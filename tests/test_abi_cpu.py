"""The C-ABI library loads without a GPU and exports every symbol include/*.h declares."""
import ctypes
import os
import re

import pytest


def _declared(repo_root):
    names = []
    inc = os.path.join(repo_root, "include")
    for fn in os.listdir(inc):
        txt = open(os.path.join(inc, fn)).read()
        txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
        names += re.findall(r"\b(?:int|const char\*|int32_t\*|void\*)\s+((?:dg[a-z]*)_[a-z0-9_]+)\s*\(", txt)
    return sorted(set(names))


def test_library_exports_header_symbols(repo_root):
    names = _declared(repo_root)
    assert "dgr_forward" in names and "dgr_backward" in names and len(names) >= 7
    lib = ctypes.CDLL(os.path.join(repo_root, "dg-mesh_b200", "libdgmesh_b200.so"))
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/ but not exported"


def test_binding_covers_header(repo_root):
    import _dgm_lib
    assert sorted(_dgm_lib.SIGNATURES) == _declared(repo_root)
    lib = _dgm_lib.lib()
    assert b"sm_90a" in lib.dgm_version()


def test_workspace_query_and_argument_errors():
    import _dgm_lib
    lib = _dgm_lib.lib()
    a, b, c = _dgm_lib.c_size_t(), _dgm_lib.c_size_t(), _dgm_lib.c_size_t()
    assert lib.dgr_workspace_sizes(1000, 64, 48, 4096, a, b, c) == 0
    assert b.value == 60 * 4096 + 128 and a.value > 1000 * 100 and c.value > 64 * 48 * 8
    assert lib.dgr_workspace_sizes(-1, 64, 48, 0, a, b, c) == -1          # DGM_E_BADARG
    # bad arguments are rejected on the host before anything touches a device
    rc = lib.dgr_forward(10, 0, 0, None, 64, 48, None, None, None, None, None, 1.0, None, None, None, None, None,
                         1.0, 1.0, 0, None, None, None, 0, None, 0, 0, None, 0, None, None, None, 0.0, 0.0, 0, None)
    assert rc == -1 and b"null" in lib.dgm_last_error()


def test_product_never_imports_oracle(repo_root):
    """The product package must not reference oracle/ (no CPU fallback, no checker in the path)."""
    pkg = os.path.join(repo_root, "dg-mesh_b200")
    for dp, _, fns in os.walk(pkg):
        for fn in fns:
            if fn.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dp, fn)).read()
                assert "oracle" not in txt.lower().replace("oracle/", "ORACLEDIR") or "import oracle" not in txt, fn
                assert "from oracle" not in txt and "import oracle" not in txt and "liboracle" not in txt, fn
