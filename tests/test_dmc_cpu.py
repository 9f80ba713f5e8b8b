"""Dual marching cubes without a GPU: the patch tables, the exact reference (tests/dmc_reference.py) against a
per-cell loop restatement and against float64 central differences, the topology of its meshes, and the host-side
refusals of the C-ABI and of DiffDMC."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from dmc_reference import (assert_same_quads, dmc_loop_reference, dmc_reference, grad_reference,
                           needed_patches, tables)
from mc_reference import LOSS_P, LOSS_W, assert_same_mesh, loss_grad, mc_reference
from test_mc_reference import noise, quantised_sphere, seam_field, single_cell, smooth_noise, sphere

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gen_mc_tables  # noqa: E402

D = 1 << 20   # a dummy address: must never be dereferenced


# ----------------------------------------------------------------------------- fields
def _axes(G):
    return np.meshgrid(*(np.linspace(-1, 1, G, dtype=np.float32),) * 3, indexing="ij")


def torus(G, R=0.5, r=0.2):
    x, y, z = _axes(G)
    q = np.sqrt(x * x + y * y) - np.float32(R)
    return (np.sqrt(q * q + z * z) - np.float32(r)).astype(np.float32)


def two_spheres(G):
    x, y, z = _axes(G)
    a = np.sqrt((x + 0.45) ** 2 + y * y + z * z) - 0.35
    b = np.sqrt((x - 0.45) ** 2 + y * y + z * z) - 0.3
    return np.minimum(a, b).astype(np.float32)


FIELDS = [
    ("sphere", sphere(12), 0.0),
    ("smooth", smooth_noise(10), 0.0),
    ("smooth_iso", smooth_noise(9, 1), -0.37),
    ("noise", noise(7), 0.0),
    ("noise_iso", noise(6, 2), 0.1),
    ("ties", quantised_sphere(11), 0.0),
    ("seams", seam_field(10), 0.0),
]


# ----------------------------------------------------------------------------- tables
def test_patch_tables():
    patch, pof, edge_lo, _ = tables()
    assert patch.shape == (256, 4, 7) and pof.shape == (256, 12)
    for case in range(256):
        loops = gen_mc_tables.case_loops(case)
        got = [sorted(int(e) for e in q if e >= 0) for q in patch[case] if (q >= 0).any()]
        assert got == [sorted(lp) for lp in loops], case                    # the patches are the generator's loops
        assert len(got) <= 4 and all(len(q) <= 7 for q in got)
        cut = {e for lp in loops for e in lp}
        for e in range(12):                                                 # every cut edge in exactly one patch
            owners = [p for p, q in enumerate(got) if e in q]
            assert len(owners) == (1 if e in cut else 0), (case, e)
            assert pof[case, e] == (owners[0] if owners else -1)
        inside = [(case >> v) & 1 for v in range(8)]
        assert cut == {e for e in range(12) if inside[gen_mc_tables.EDGES[e][0]] != inside[gen_mc_tables.EDGES[e][1]]}
    assert subprocess.call([sys.executable, os.path.join(ROOT, "tools", "gen_mc_tables.py"), "--check"]) == 0


# ----------------------------------------------------------------------------- the reference
@pytest.mark.parametrize("name,phi,iso", FIELDS)
def test_reference_equals_loop_restatement(name, phi, iso):
    ref = dmc_reference(phi, iso)
    vl, ql = dmc_loop_reference(phi, iso)
    assert len(ref.verts) and len(ref.quads)
    fl = np.concatenate([ql[:, [0, 1, 2]], ql[:, [0, 2, 3]]])
    assert_same_mesh(ref.verts, ref.faces, vl, fl)
    assert_same_quads(ref.verts, ref.quads, vl, ql)


def test_reference_single_cells_are_empty():
    """A G = 2 grid has no interior edge: no quad and no vertex, whatever the case."""
    for case in range(256):
        ref = dmc_reference(single_cell(case))
        assert len(ref.verts) == 0 and len(ref.quads) == 0


def _verts64(ref, phi):
    """The reference's vertices recomputed in float64 from phi (same cells and patches)."""
    patch, pof, edge_lo, pmask = tables()
    G = ref.G
    cells = np.stack(np.unravel_index(ref.cell, (G, G, G)), 1)
    cs = np.zeros(len(cells), np.int64)
    for c in range(8):
        n = cells + np.array([c & 1, (c >> 1) & 1, c >> 2])
        cs |= (np.asarray(phi, np.float32)[tuple(n.T)] < np.float32(ref.iso)).astype(np.int64) << c
    out = np.zeros((len(cells), 3))
    k = np.zeros(len(cells))
    for e in range(12):
        sel = pof[cs, e] == ref.patch
        a, lo = e >> 2, int(edge_lo[e])
        n = cells[sel] + np.array([lo & 1, (lo >> 1) & 1, lo >> 2])
        m = n.copy()
        m[:, a] += 1
        p0, p1 = phi[tuple(n.T)], phi[tuple(m.T)]
        pos = n.astype(np.float64)
        pos[:, a] += (ref.iso - p0) / (p1 - p0)
        out[sel] += pos
        k[sel] += 1
    return out / k[:, None] / (G - 1)


@pytest.mark.parametrize("name,phi,iso", [FIELDS[0], FIELDS[1], FIELDS[2]])
def test_reference_gradient_central_differences(name, phi, iso):
    ref = dmc_reference(phi, iso)
    p64 = phi.astype(np.float64)

    def loss(p):
        return np.sin(_verts64(ref, p) * LOSS_W + LOSS_P).sum()

    dphi, absum = grad_reference(ref, phi, loss_grad(_verts64(ref, p64)))
    nodes = np.argwhere(absum > 0)
    rng = np.random.default_rng(0)
    eps = 1e-6
    for n in nodes[rng.choice(len(nodes), min(40, len(nodes)), replace=False)]:
        n = tuple(n)
        hi, lo = p64.copy(), p64.copy()
        hi[n] += eps
        lo[n] -= eps
        fd = (loss(hi) - loss(lo)) / (2 * eps)
        assert abs(fd - dphi[n]) <= 1e-5 * max(1.0, absum[n]), (n, fd, dphi[n])


# ----------------------------------------------------------------------------- topology
def _directed_edges(faces):
    return np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])


@pytest.mark.parametrize("name,phi,iso", FIELDS)
def test_closed_and_counts(name, phi, iso):
    """Every directed edge is matched by its reverse, except where the level set leaves the grid: an unmatched
    edge joins two cells on the grid's outer faces (fields that stay inside the grid are closed)."""
    ref = dmc_reference(phi, iso)
    G = ref.G
    d = _directed_edges(ref.faces)
    fwd = d[:, 0] * len(ref.verts) + d[:, 1]
    rev = d[:, 1] * len(ref.verts) + d[:, 0]
    open_ = np.setxor1d(fwd, rev)
    cells = np.stack(np.unravel_index(ref.cell, (G, G, G)), 1)
    on_face = ((cells == 0) | (cells == G - 2)).any(1)
    assert on_face[open_ // len(ref.verts)].all() and on_face[open_ % len(ref.verts)].all()
    if name in ("sphere", "ties"):
        assert len(open_) == 0
    mc = mc_reference(phi, iso)
    nodes = np.stack(np.unravel_index(mc.node, (G, G, G)), 1)
    interior = np.ones(len(nodes), bool)
    for a in range(3):
        for o in (x for x in range(3) if x != a):
            interior &= ~((mc.axis == a) & ((nodes[:, o] < 1) | (nodes[:, o] > G - 2)))
    assert len(ref.quads) == int(interior.sum())           # one quad per interior marching-cubes vertex
    assert len(ref.faces) == 2 * len(ref.quads)
    assert np.array_equal(np.unique(ref.faces), np.arange(len(ref.verts)))     # no unreferenced vertex


@pytest.mark.parametrize("name,phi,chi", [("sphere", sphere(24), 2), ("torus", torus(32), 0),
                                          ("two_spheres", two_spheres(28), 4)])
def test_manifold_euler(name, phi, chi):
    ref = dmc_reference(phi)
    d = np.sort(_directed_edges(ref.faces), 1)
    _, cnt = np.unique(d[:, 0] * len(ref.verts) + d[:, 1], return_counts=True)
    assert (cnt == 2).all()
    assert len(ref.verts) - len(cnt) + len(ref.faces) == chi


def test_needed_patches_interior_cell():
    """A cell away from the grid's faces gives every patch a vertex."""
    patch, _, _, _ = tables()
    cs = np.arange(256)
    need = needed_patches(cs, np.full((256, 3), 3), 10)
    assert np.array_equal(need, (patch >= 0).any(2))


# ----------------------------------------------------------------------------- C-ABI and Python refusals
def _lib():
    import _dgm_lib
    return _dgm_lib.lib()


def _err(lib, rc, *words):
    msg = lib.dgm_last_error()
    assert rc == -1, (rc, msg)
    for w in words:
        assert w in msg, (w, msg)


def test_abi_signatures():
    import _dgm_lib
    lib = _lib()
    for op in ("workspace_size", "count", "emit", "backward"):
        for sfx in ("", "_batch"):
            name = f"dgdmc_{op}{sfx}"
            restype, args = _dgm_lib.SIGNATURES[name]
            assert getattr(lib, name).argtypes == args, name


def test_abi_refusals():
    import _dgm_lib
    lib = _lib()
    n = _dgm_lib.c_size_t()
    for G in (1, 801):
        _err(lib, lib.dgdmc_workspace_size(G, n), b"dgdmc_workspace_size", b"G")
    _err(lib, lib.dgdmc_workspace_size(8, None), b"dgdmc_workspace_size")
    for B in (0, 65):
        _err(lib, lib.dgdmc_workspace_size_batch(B, 8, n), b"B out of range")
        _err(lib, lib.dgdmc_count_batch(B, 8, D, 0.0, D, 1 << 40, D, None, None, None), b"B out of range")
        _err(lib, lib.dgdmc_emit_batch(B, 8, D, 0.0, D, 1 << 40, D, D, 16, D, None, 16, None), b"B out of range")
        V = (4,) * 66
        _err(lib, lib.dgdmc_backward_batch(B, 8, (_dgm_lib.c_int32 * 66)(*V), D, 0.0, D, 1 << 40, D, D, D, None),
             b"B out of range")
    _err(lib, lib.dgdmc_count(8, None, 0.0, D, 1 << 40, D, None, None, None), b"dgdmc_count")
    _err(lib, lib.dgdmc_count(8, D, 0.0, D, 1 << 40, None, None, None, None), b"null totals")
    lib.dgdmc_workspace_size(8, n)
    assert lib.dgdmc_count(8, D, 0.0, D, n.value - 1, D, None, None, None) == -2   # DGM_E_WORKSPACE
    assert b"workspace too small" in lib.dgm_last_error()
    for vcap, qcap in ((1 << 28) + 1, 16), (-1, 16), (16, 1 << 30), (16, -1):
        _err(lib, lib.dgdmc_emit(64, D, 0.0, D, 1 << 40, D, D, vcap, D, None, qcap, None), b"capacity")
    _err(lib, lib.dgdmc_emit(64, D, 0.0, D, 1 << 40, D, None, 16, D, None, 16, None), b"null output")
    _err(lib, lib.dgdmc_emit(64, D, 0.0, D, 1 << 40, D, D, 16, None, D, 16, None), b"null output")
    G = 8
    for V in (4 * (G - 1) ** 3 + 1, -1):                   # more vertices than four per cell
        _err(lib, lib.dgdmc_backward(G, V, D, 0.0, D, 1 << 40, D, D, D, None), b"V out of range")
    _err(lib, lib.dgdmc_backward(800, (1 << 28) + 1, D, 0.0, D, 1 << 40, D, D, D, None), b"V out of range")
    _err(lib, lib.dgdmc_backward(G, 5, D, 0.0, D, 1 << 40, None, D, D, None), b"null vsrc")
    _err(lib, lib.dgdmc_backward(G, 5, D, 0.0, None, 1 << 40, D, D, D, None), b"null")


def test_python_refusals():
    from diso import DiffDMC
    with pytest.raises(NotImplementedError):
        DiffDMC(dtype=torch.float64)
    m = DiffDMC()
    g = torch.zeros(8, 8, 8)
    with pytest.raises(NotImplementedError):
        m(g, deform=torch.zeros(8, 8, 8, 3))
    with pytest.raises(ValueError, match="CUDA"):
        m(g)
    with pytest.raises(ValueError, match="cubic"):
        m(torch.zeros(8, 8, 7))
    with pytest.raises(ValueError, match="batch size"):
        m.forward_batch(torch.zeros(65, 4, 4, 4))
    with pytest.raises(ValueError):
        m.forward_batch(g)
