"""Hash-grid field without a GPU: the float64 restatement (tests/hashgrid_oracle.py) against a trilinear sample and
hashes computed by hand and against central differences, the level resolutions, the dghg_ entry points' host-side
checks with their ctypes signatures, and the ValueErrors that need no device."""
import ctypes
import itertools
import math
import os
import re

import pytest
import torch

import hashgrid_oracle as ho

BOX = torch.tensor([[-1.0, -2.0, -0.5], [1.0, 2.0, 1.5]])


def _tables(G, L, T, Fe, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.rand(L, T, Fe, generator=g, dtype=torch.float64) * 2 - 1 for _ in range(G)]


def test_slots_against_hashes_by_hand():
    T = 2 ** 12
    # hashed: (i_a * 1 ^ i_b * 2654435761 ^ i_c * 805459861) mod 2^32 mod T
    for i in ((0, 0, 0), (1, 0, 0), (3, 5, 7), (2047, 1, 2048), (100000, 99999, 12345)):
        h = (i[0] ^ ((i[1] * 2654435761) % 2 ** 32) ^ ((i[2] * 805459861) % 2 ** 32)) % T
        assert int(ho.slots(torch.tensor(i), [4096] * 3, T)) == h
    # 5 * 2654435761 = 0x17156075, 7 * 805459861 = 0x50106513 (mod 2^32); 3 ^ both = 0x47050565
    assert int(ho.slots(torch.tensor((3, 5, 7)), [4096] * 3, T)) == 0x565 == 1381
    assert int(ho.slots(torch.tensor((2047, 1, 2048)), [4096] * 3, T)) == 1614
    # dense exactly at (R+1)^3 = T (R = 15), first axis fastest; hashed one node past it
    assert int(ho.slots(torch.tensor((3, 5, 7)), [15] * 3, T)) == 3 + 16 * (5 + 16 * 7)
    assert int(ho.slots(torch.tensor((15, 15, 15)), [15] * 3, T)) == T - 1
    assert int(ho.slots(torch.tensor((3, 5, 7)), [15, 15, 16], T)) == 1381
    # a space-time grid: (R+1)^2 (R_t+1) = 16 16 16 dense, 16 16 17 hashed
    assert int(ho.slots(torch.tensor((1, 2, 3)), [15, 15, 15], T)) == 1 + 16 * (2 + 16 * 3)
    assert int(ho.slots(torch.tensor((1, 2, 3)), [15, 15, 16], T)) == 1500   # 1 ^ 0x3c6ef362 ^ 0x900706bf


def test_oracle_against_a_trilinear_sample_by_hand():
    """One point of one level of the xyt grid at L = 1, R = 8, R_t = 4, and a dense xyz level."""
    T, Fe = 2 ** 12, 2
    tabs = _tables(2, 1, T, Fe, 1)
    box = torch.tensor([[0.0, 0.0, 0.0], [1.0, 1.0, 1.0]])
    x = torch.tensor([[0.3, 0.55, 1.0]])
    t = torch.tensor([[0.6]])
    got = ho.field(x, t, box, tabs, ("xyz", "xyt"), (8,), 4, 12)
    for g, (grid, R3) in enumerate((("xyz", (8, 8, 8)), ("xyt", (8, 8, 4)))):
        ax = ho.AXES[grid]
        u = [float(torch.tensor(v, dtype=torch.float32)) for v in (0.3, 0.55, 1.0, 0.6)]
        ref = torch.zeros(Fe, dtype=torch.float64)
        p = [float(torch.tensor(u[a], dtype=torch.float32) * R) for a, R in zip(ax, R3)]
        c = [min(math.floor(pi), R - 1) for pi, R in zip(p, R3)]
        w = [pi - ci for pi, ci in zip(p, c)]
        assert w[2] == 1.0 or grid == "xyt"                  # z = 1 lies on the top face: c = R - 1, w = 1
        for k in range(8):
            b = [(k >> j) & 1 for j in range(3)]
            n = [ci + bj for ci, bj in zip(c, b)]
            wk = math.prod(wj if bj else 1 - wj for wj, bj in zip(w, b))
            slot = n[0] + (R3[0] + 1) * (n[1] + (R3[1] + 1) * n[2])        # both levels are dense here
            ref += wk * tabs[g][0, slot]
        assert float((got[0, g * Fe:(g + 1) * Fe] - ref).abs().max()) < 1e-14


def test_resolutions():
    from hashgrid import HashGridField, level_resolutions
    assert HashGridField(BOX).resolutions == (16, 22, 30, 42, 58, 80, 111, 153, 212, 294, 406, 561, 776, 1072,
                                              1482, 2048)
    assert level_resolutions(1, 16, 2048) == (16,)
    assert level_resolutions(2, 16, 2048) == (16, 2048)
    f = HashGridField(BOX, grids=("xzt", "xyz"), levels=3, features=4, log2_table=12)
    assert f.grids == ("xyz", "xzt") and f.out_dim == 2 * 3 * 4
    assert [tuple(p.shape) for p in f.tables] == [(3, 4096, 4)] * 2
    assert all(float(p.detach().abs().max()) <= 1e-4 for p in f.tables)


@pytest.mark.parametrize("seed", [0, 1])
def test_oracle_gradients_against_central_differences(seed):
    """Coordinates in float64 (coord_dtype) so that x can move by 1e-6; points away from cell faces."""
    grids, res, Rt, log2T = ho.GRIDS, (3, 5), 4, 12
    tabs = _tables(4, 2, 2 ** log2T, 2, seed)
    g = torch.Generator().manual_seed(seed + 10)
    box = BOX.double()
    x = box[0] + (box[1] - box[0]) * (0.05 + 0.9 * torch.rand(6, 3, generator=g, dtype=torch.float64))
    t = torch.rand(2, 6, 1, generator=g, dtype=torch.float64)
    gout = torch.randn(2, 6, 4 * 2 * 2, generator=g, dtype=torch.float64)
    _, gx, gt = ho.field_and_grads(x, t, box, tabs, grids, res, Rt, log2T, gout, coord_dtype=torch.float64)

    def L(xx, tb):
        return float((ho.field(xx, t, box, tb, grids, res, Rt, log2T, coord_dtype=torch.float64) * gout).sum())

    h = 1e-7
    num = torch.zeros_like(x)
    for e in range(x.numel()):
        xp, xm = x.clone(), x.clone()
        xp.view(-1)[e] += h
        xm.view(-1)[e] -= h
        num.view(-1)[e] = (L(xp, tabs) - L(xm, tabs)) / (2 * h)
    assert float((num - gx).abs().max()) < 1e-6 * max(1.0, float(gx.abs().max()))
    for gi in range(4):
        hit = gt[gi].reshape(-1).nonzero()[:, 0]
        for e in hit[torch.randperm(hit.numel(), generator=g)[:10]].tolist():
            tp, tm = [p.clone() for p in tabs], [p.clone() for p in tabs]
            tp[gi].view(-1)[e] += 1e-6
            tm[gi].view(-1)[e] -= 1e-6
            d = (L(x, tp) - L(x, tm)) / 2e-6
            assert abs(d - float(gt[gi].reshape(-1)[e])) < 1e-7 * max(1.0, abs(d)), (gi, e)


def test_oracle_coordinate_gradient_outside_the_box():
    """0 strictly outside, and passed on the faces (torch.clamp)."""
    tabs = _tables(1, 2, 2 ** 12, 2, 3)
    x = torch.stack([BOX[0] - 0.5, BOX[1] + 0.5, BOX[0], BOX[1]])
    _, gx, _ = ho.field_and_grads(x, None, BOX, tabs, ("xyz",), (4, 7), 4, 12, torch.ones(4, 4, dtype=torch.float64))
    assert not gx[:2].any() and gx[2:].abs().min() > 0


# ---- the C-ABI on the host -----------------------------------------------------------------------------------------
FAKE = 0x1000
FNS = ["dghg_forward", "dghg_backward_workspace", "dghg_backward"]


def _header_params(fn):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(root, "include", "dgmesh_b200.h")).read(), flags=re.S)
    decl = re.search(r"\bint\s+" + fn + r"\s*\(([^)]*)\)", txt).group(1)
    return [(re.split(r"[\s*]+", a.strip())[-1], a.strip()) for a in decl.split(",")]


def _call(fn, res=(16, 22, 30, 42), kinds=(0, 1, 2, 3), G=None, L=None, tables=FAKE, grads=FAKE, **over):
    import _dgm_lib
    lib = _dgm_lib.lib()
    G = len(kinds) if G is None else G
    L = len(res) if L is None else L
    r = (ctypes.c_int32 * max(1, len(res)))(*res)
    k = (ctypes.c_int32 * max(1, len(kinds)))(*kinds)
    tp = (ctypes.c_void_p * 4)(*([tables] * 4))
    gp = (ctypes.c_void_p * 4)(*([grads] * 4))
    args = {"F": 2, "N": 1000, "G": G, "grids_host": ctypes.addressof(k), "L": L, "Fe": 2, "log2_table": 19,
            "res_host": ctypes.addressof(r), "R_t": 32, "ws_bytes": 1 << 40, "stream": None,
            "bytes": ctypes.pointer(ctypes.c_size_t()), "tables_host": ctypes.addressof(tp),
            "grad_tables_host": ctypes.addressof(gp), "grad_x": FAKE}
    args.update(over)
    rc = getattr(lib, fn)(*[args.get(name, FAKE) for name, _ in _header_params(fn)])
    return rc, lib.dgm_last_error()


@pytest.mark.parametrize("fn", FNS)
def test_ctypes_signature_matches_the_header(fn):
    import _dgm_lib
    res, argtypes = _dgm_lib.SIGNATURES[fn]
    params = _header_params(fn)
    assert res is ctypes.c_int and len(argtypes) == len(params)
    for (name, decl), t in zip(params, argtypes):
        if decl.startswith("size_t*"):
            assert t._type_ is ctypes.c_size_t, name
        elif "*" in decl:
            assert t is ctypes.c_void_p, name
        elif decl.startswith("size_t"):
            assert t is ctypes.c_size_t, name
        else:
            assert decl.startswith("int") and t is ctypes.c_int, name


def test_every_header_symbol_is_bound():
    import _dgm_lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(root, "include", "dgmesh_b200.h")).read(), flags=re.S)
    names = set(re.findall(r"\bdghg_\w+(?=\s*\()", txt))
    assert names == set(FNS) and names <= set(_dgm_lib.SIGNATURES)


BAD = [dict(G=0, kinds=()), dict(G=5, kinds=(0, 1, 2, 3, 3)), dict(L=0, res=()), dict(L=25, res=(16,) * 25),
       dict(Fe=3), dict(Fe=8), dict(log2_table=11), dict(log2_table=25), dict(R_t=0), dict(res=(0, 16)),
       dict(res=(16, 2 ** 24 + 1)), dict(F=-1), dict(N=-1),
       dict(F=2 ** 8, N=2 ** 17, Fe=4, kinds=(0, 1), res=(16,) * 8),            # F N G L Fe = 2^31
       dict(F=2 ** 16, N=2 ** 15, kinds=(0,), res=(16,))]                       # N F = 2^31 (F N G L Fe = 2^32)
ROWS = [(fn, b, b"bad size") for fn, b in itertools.product(FNS, BAD)]
ROWS += [(fn, b, b"bad grids") for fn, b in itertools.product(FNS, [dict(kinds=(0, 4)), dict(kinds=(-1, 0)),
                                                                   dict(kinds=(1, 0)), dict(kinds=(2, 2))])]
ROWS += [(fn, {p: None}, b"null pointer") for fn in FNS for p in ("grids_host", "res_host")]
ROWS += [(fn, {"tables_host": None}, b"null pointer") for fn in ("dghg_forward", "dghg_backward")]
ROWS += [(fn, {"tables": None}, b"null pointer") for fn in ("dghg_forward", "dghg_backward")]
ROWS += [("dghg_backward", {"grad_tables_host": None}, b"null pointer"), ("dghg_backward", {"grads": None},
                                                                          b"null pointer")]
ROWS += [(fn, {p: None}, b"null pointer") for fn, ps in (("dghg_forward", ("box", "x", "t", "out")),
                                                         ("dghg_backward", ("box", "x", "t", "grad_out", "ws")))
         for p in ps]
ROWS += [("dghg_backward_workspace", {"bytes": None}, b"null pointer")]


@pytest.mark.parametrize("fn,over,text", ROWS, ids=[f"{f}-{','.join(f'{k}={v}' for k, v in o.items())}"
                                                    for f, o, _ in ROWS])
def test_bad_argument_is_refused_on_the_host(fn, over, text):
    rc, msg = _call(fn, **over)
    assert rc == -1 and text in msg and fn.encode() in msg, (rc, msg)


def test_largest_sizes_below_the_limits_pass_the_host_checks():
    """F N G L Fe just below 2^31 is accepted; N F >= 2^31 always implies F N G L Fe >= 2^32."""
    assert _call("dghg_backward_workspace", F=2 ** 8 - 1, N=2 ** 17, Fe=4, kinds=(0, 1), res=(16,) * 8)[0] == 0
    assert _call("dghg_backward_workspace", F=2 ** 16 - 1, N=2 ** 15, kinds=(0,), res=(16,), G=1, L=1)[0] == -1
    assert _call("dghg_backward_workspace", F=2 ** 15 - 1, N=2 ** 15, kinds=(0,), res=(16,))[0] == 0
    assert _call("dghg_backward_workspace", log2_table=24, Fe=4, res=(16,) * 24)[0] == 0     # L T Fe = 1.5 2^30


def test_static_field_takes_no_t():
    """With only the xyz grid, t may be NULL; with a time grid it may not."""
    assert _call("dghg_forward", kinds=(0,), t=None, F=0)[0] == 0
    rc, msg = _call("dghg_forward", kinds=(0, 1), t=None)
    assert rc == -1 and b"null pointer" in msg


@pytest.mark.parametrize("G,L,Fe,log2T", [(1, 1, 2, 12), (4, 16, 2, 19), (3, 24, 4, 24)])
def test_short_workspace_is_refused_on_the_host(G, L, Fe, log2T):
    need = ctypes.c_size_t()
    kw = dict(kinds=tuple(range(G)), res=(16,) * L, Fe=Fe, log2_table=log2T)
    rc, _ = _call("dghg_backward_workspace", bytes=ctypes.byref(need), **kw)
    assert rc == 0 and G * L * 2 ** log2T * Fe * 8 <= need.value < G * L * 2 ** log2T * Fe * 8 + 4096
    rc, msg = _call("dghg_backward", ws_bytes=need.value - 1, **kw)
    assert rc == -2 and b"workspace too small" in msg and b"dghg_backward" in msg, (rc, msg)


def test_nothing_to_do_reads_nothing():
    """F = 0 or N = 0: the forward returns before reading a pointer other than the table array."""
    for e in (dict(F=0), dict(N=0)):
        rc, msg = _call("dghg_forward", box=None, x=None, t=None, out=None, **e)
        assert rc == 0, msg


# ---- ValueErrors that need no device -------------------------------------------------------------------------------
def test_bad_construction_is_refused():
    from hashgrid import HashGridDeformNetwork, HashGridField
    for kw in (dict(grids=()), dict(grids=("xyz", "xyz")), dict(grids=("xyw",)), dict(features=3),
               dict(features=2.0), dict(features=True), dict(levels=0), dict(levels=25), dict(log2_table=11),
               dict(log2_table=25), dict(base_resolution=0), dict(finest_resolution=8), dict(time_resolution=0),
               dict(levels=16.0)):
        with pytest.raises(ValueError):
            HashGridField(BOX, **kw)
    for b in ([[0.0] * 3], [[0.0] * 3, [0.0, 1.0, 1.0]], [[0.0] * 3, [float("inf")] * 3]):
        with pytest.raises(ValueError, match="box"):
            HashGridField(b)
    with pytest.raises(ValueError):
        HashGridDeformNetwork(BOX, W=0)


def test_cpu_tensors_and_bad_inputs_are_refused():
    from hashgrid import HashGridField
    f = HashGridField(BOX, levels=2, log2_table=12)
    x, t = torch.zeros(10, 3), torch.zeros(10, 1)
    with pytest.raises(ValueError, match="CUDA"):
        f(x, t)
    with pytest.raises(ValueError, match="grad"):
        f(x, t.requires_grad_(True))
    with pytest.raises(ValueError, match="None"):
        f(x, None)
    for xx, tt in ((torch.zeros(10, 2), torch.zeros(10, 1)), (torch.zeros(10, 3), torch.zeros(9, 1)),
                   (torch.zeros(10, 3), torch.zeros(10)), (torch.zeros(10, 3), torch.zeros(2, 10, 2))):
        with pytest.raises(ValueError):
            f(xx, tt)
    with pytest.raises(ValueError, match="float32"):
        f(x.double(), torch.zeros(10, 1))
    with pytest.raises(ValueError, match="CUDA"):
        HashGridField(BOX, grids=("xyz",), levels=2, log2_table=12)(x)
