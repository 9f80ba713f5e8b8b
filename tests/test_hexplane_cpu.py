"""HexPlane field without a GPU: the float64 restatement (tests/hexplane_oracle.py) against a bilinear formula written
out by hand and against central differences, the regulariser formulas against explicit loops, the dghp_ entry
points' host-side checks with their ctypes signatures, and the ValueErrors that need no device."""
import ctypes
import itertools
import os
import re

import pytest
import torch

import hexplane_oracle as ho

BOX = torch.tensor([[-1.0, -2.0, -0.5], [1.0, 2.0, 1.5]], dtype=torch.float64)


def _planes(S, R, Rt, C, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    for s in range(S):
        for p, (a, b) in enumerate(ho.PAIRS):
            out.append(torch.rand(Rt if b == 3 else R[s], R[s], C, generator=g, dtype=torch.float64) + 0.5)
    return out


def _bilinear(G, pa, pb):
    """G [R_b, R_a, C] at pixel coordinates (pa, pb), clamped to the plane (border padding)."""
    Rb, Ra = G.shape[0], G.shape[1]
    pa, pb = min(max(pa, 0.0), Ra - 1.0), min(max(pb, 0.0), Rb - 1.0)
    x0, y0 = min(int(pa), Ra - 2), min(int(pb), Rb - 2)
    fx, fy = pa - x0, pb - y0
    return ((1 - fx) * (1 - fy) * G[y0, x0] + fx * (1 - fy) * G[y0, x0 + 1] + (1 - fx) * fy * G[y0 + 1, x0]
            + fx * fy * G[y0 + 1, x0 + 1])


def _by_hand(x, t, planes, S, R, Rt):
    out = []
    for n in range(x.shape[0]):
        feats = []
        for s in range(S):
            pix = [float((x[n, a] - BOX[0, a]) * (R[s] - 1) / (BOX[1, a] - BOX[0, a])) for a in range(3)]
            pix.append(float(t[n, 0]) * (Rt - 1))
            f = 1
            for p, (a, b) in enumerate(ho.PAIRS):
                f = f * _bilinear(planes[6 * s + p], pix[a], pix[b])
            feats.append(f)
        out.append(torch.cat(feats))
    return torch.stack(out)


def test_oracle_against_a_bilinear_formula_by_hand():
    """Texel nodes, box faces, points outside the box and random points, times 0, 1, a time node and between."""
    S, R, Rt, C = 2, (5, 9), 5, 3
    planes = _planes(S, R, Rt, C)
    lo, hi = BOX[0], BOX[1]
    pts = [lo, hi, lo + (hi - lo) * 0.25, lo + (hi - lo) * 0.5,          # faces; nodes of both scales
           lo + (hi - lo) * torch.tensor([0.125, 0.375, 0.625]),         # nodes of the finer scale only
           lo - 0.3, hi + torch.tensor([0.1, 2.0, 0.0]), torch.tensor([0.0, 9.0, -4.0], dtype=torch.float64)]
    g = torch.Generator().manual_seed(1)
    pts += list(lo + (hi - lo) * torch.rand(6, 3, generator=g, dtype=torch.float64))
    x = torch.stack(pts)
    t = torch.tensor([0.0, 1.0, 0.5, 0.25, 0.3, 0.0, 1.0, 0.7] + [0.1 * k for k in range(6)],
                     dtype=torch.float64)[:, None]
    ref = _by_hand(x, t, planes, S, R, Rt)
    got = ho.field(x, t, BOX, planes, S)
    assert float((got - ref).abs().max()) < 1e-13
    # the batch form is the frames stacked
    t2 = torch.stack([t, t.flip(0)])
    assert torch.equal(ho.field(x, t2, BOX, planes, S)[1], ho.field(x, t.flip(0), BOX, planes, S))


def test_new_field_does_not_depend_on_time():
    from hexplane import HexPlaneField
    f = HexPlaneField(BOX.float(), channels=16, base_resolution=4, multires=(1, 2), time_resolution=5)
    assert all(bool((p == 1).all()) for i, p in enumerate(f.planes) if i % 6 in ho.TIME)
    sp = [p for i, p in enumerate(f.planes) if i % 6 in ho.SPATIAL]
    assert all(float(p.detach().min()) >= 0.1 and float(p.detach().max()) <= 0.5 for p in sp)
    assert [tuple(p.shape) for p in f.planes[:6]] == [(4, 4, 16), (4, 4, 16), (5, 4, 16), (4, 4, 16), (5, 4, 16),
                                                      (5, 4, 16)]
    x = torch.rand(7, 3, dtype=torch.float64)
    a = ho.field(x, torch.zeros(7, 1, dtype=torch.float64), BOX, [p.double() for p in f.planes], 2)
    b = ho.field(x, torch.ones(7, 1, dtype=torch.float64), BOX, [p.double() for p in f.planes], 2)
    assert torch.equal(a, b)


@pytest.mark.parametrize("seed", [0, 1])
def test_oracle_gradients_against_central_differences(seed):
    S, R, Rt, C = 2, (4, 7), 5, 2
    planes = _planes(S, R, Rt, C, seed)
    g = torch.Generator().manual_seed(seed + 10)
    x = BOX[0] + (BOX[1] - BOX[0]) * (0.05 + 0.9 * torch.rand(5, 3, generator=g, dtype=torch.float64))
    t = torch.rand(2, 5, 1, generator=g, dtype=torch.float64)
    gout = torch.randn(2, 5, S * C, generator=g, dtype=torch.float64)
    _, gx, gp = ho.field_and_grads(x, t, BOX, planes, S, gout)

    def L(xx, pl):
        return float((ho.field(xx, t, BOX, pl, S) * gout).sum())

    h = 1e-6
    num = torch.zeros_like(x)
    for e in range(x.numel()):
        xp, xm = x.clone(), x.clone()
        xp.view(-1)[e] += h
        xm.view(-1)[e] -= h
        num.view(-1)[e] = (L(xp, planes) - L(xm, planes)) / (2 * h)
    assert float((num - gx).abs().max()) < 1e-6 * max(1.0, float(gx.abs().max()))
    for i in (0, 2, 7, 11):        # a spatial and a time plane of each scale
        for e in torch.randperm(planes[i].numel(), generator=g)[:20].tolist():
            pp, pm = [p.clone() for p in planes], [p.clone() for p in planes]
            pp[i].view(-1)[e] += h
            pm[i].view(-1)[e] -= h
            d = (L(x, pp) - L(x, pm)) / (2 * h)
            assert abs(d - float(gp[i].reshape(-1)[e])) < 1e-6 * max(1.0, abs(d)), (i, e)


def test_oracle_coordinate_gradient_is_zero_outside_and_on_faces():
    S, R, Rt, C = 1, (5,), 3, 2
    planes = _planes(S, R, Rt, C, 3)
    x = torch.stack([BOX[0], BOX[1], BOX[0] - 0.5, BOX[1] + 0.5])
    t = torch.full((4, 1), 0.4, dtype=torch.float64)
    _, gx, _ = ho.field_and_grads(x, t, BOX, planes, S, torch.ones(4, C, dtype=torch.float64))
    assert not gx.any()


def test_regularisers_against_loops():
    S, R, Rt, C = 2, (3, 4), 4, 2
    planes = _planes(S, R, Rt, C, 4)
    tv = ts = l1 = 0.0
    for s in range(S):
        for p in ho.SPATIAL:
            G = planes[6 * s + p]
            Rb, Ra = G.shape[:2]
            a = sum(float(G[i + 1, j, c] - G[i, j, c]) ** 2 for i in range(Rb - 1) for j in range(Ra) for c in range(C))
            b = sum(float(G[i, j + 1, c] - G[i, j, c]) ** 2 for i in range(Rb) for j in range(Ra - 1) for c in range(C))
            tv += a / ((Rb - 1) * Ra * C) + b / (Rb * (Ra - 1) * C)
        for p in ho.TIME:
            G = planes[6 * s + p]
            Rb, Ra = G.shape[:2]
            ts += sum(float(G[i + 2, j, c] - 2 * G[i + 1, j, c] + G[i, j, c]) ** 2
                      for i in range(Rb - 2) for j in range(Ra) for c in range(C)) / ((Rb - 2) * Ra * C)
            l1 += sum(abs(1 - float(v)) for v in G.flatten()) / G.numel()
    got = [float(v) for v in ho.regularisers(planes, S)]
    assert max(abs(a - b) for a, b in zip(got, (tv, ts, l1))) < 1e-13
    # two time rows: no second difference
    assert float(ho.regularisers(_planes(1, (3,), 2, 2), 1)[1]) == 0.0
    # |1 - G| has gradient 0 at G = 1
    one = [torch.ones_like(p) for p in planes]
    _, g = ho.regularisers_and_grads(one, S, (0.0, 0.0, 1.0))
    assert not any(q.any() for q in g)


# ---- the C-ABI on the host -----------------------------------------------------------------------------------------
FAKE = 0x1000
FNS = ["dghp_forward", "dghp_backward_workspace", "dghp_backward", "dghp_reg_workspace", "dghp_reg_forward",
       "dghp_reg_backward"]


def _header_params(fn):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(root, "include", "dgmesh_b200.h")).read(), flags=re.S)
    decl = re.search(r"\bint\s+" + fn + r"\s*\(([^)]*)\)", txt).group(1)
    return [(re.split(r"[\s*]+", a.strip())[-1], a.strip()) for a in decl.split(",")]


def _call(fn, res=(64, 128), S=None, planes=FAKE, grads=FAKE, **over):
    import _dgm_lib
    lib = _dgm_lib.lib()
    S = len(res) if S is None else S
    r = (ctypes.c_int32 * max(1, len(res)))(*res)
    pl = (ctypes.c_void_p * 24)(*([planes] * 24))
    gp = (ctypes.c_void_p * 24)(*([grads] * 24))
    args = {"F": 2, "N": 1000, "S": S, "C": 32, "res_host": ctypes.addressof(r), "R_t": 25, "ws_bytes": 1 << 40,
            "stream": None, "bytes": ctypes.pointer(ctypes.c_size_t()), "planes_host": ctypes.addressof(pl),
            "grad_planes_host": ctypes.addressof(gp), "grad_x": FAKE}
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
    names = set(re.findall(r"\bdghp_\w+(?=\s*\()", txt))
    assert names == set(FNS) and names <= set(_dgm_lib.SIGNATURES)


BAD = [dict(S=0, res=()), dict(S=5, res=(4,) * 5), dict(C=8), dict(C=64), dict(R_t=1), dict(res=(1, 4)),
       dict(res=(8192, 4))]
SIZE_FNS = ["dghp_forward", "dghp_backward_workspace", "dghp_backward"]
ROWS = [(fn, b, b"bad size") for fn, b in itertools.product(FNS, BAD)]
ROWS += [(fn, b, b"bad size") for fn, b in itertools.product(SIZE_FNS, [dict(F=-1), dict(N=-1),
                                                                          dict(F=2 ** 20, N=2 ** 20)])]
ROWS += [(fn, {"res_host": None}, b"null pointer") for fn in FNS]
ROWS += [(fn, {"planes_host": None}, b"null pointer") for fn in FNS if "workspace" not in fn]
ROWS += [(fn, {"grad_planes_host": None}, b"null pointer") for fn in ("dghp_backward", "dghp_reg_backward")]
ROWS += [(fn, {"planes": None}, b"null pointer") for fn in FNS if "workspace" not in fn]
ROWS += [(fn, {"grads": None}, b"null pointer") for fn in ("dghp_backward", "dghp_reg_backward")]
ROWS += [(fn, {p: None}, b"null pointer") for fn, ps in (("dghp_forward", ("box", "x", "t", "out")),
                                                         ("dghp_backward", ("box", "x", "t", "grad_out", "ws")),
                                                         ("dghp_reg_forward", ("losses", "ws")),
                                                         ("dghp_reg_backward", ("grad_losses",))) for p in ps]
ROWS += [(fn, {"bytes": None}, b"null pointer") for fn in ("dghp_backward_workspace", "dghp_reg_workspace")]


@pytest.mark.parametrize("fn,over,text", ROWS, ids=[f"{f}-{','.join(f'{k}={v}' for k, v in o.items())}"
                                                    for f, o, _ in ROWS])
def test_bad_argument_is_refused_on_the_host(fn, over, text):
    rc, msg = _call(fn, **over)
    assert rc == -1 and text in msg and fn.encode() in msg, (rc, msg)


@pytest.mark.parametrize("fn,query", [("dghp_backward", "dghp_backward_workspace"),
                                      ("dghp_reg_forward", "dghp_reg_workspace")])
@pytest.mark.parametrize("F,N,C,res", [(1, 1, 16, (2,)), (1, 100_000, 32, (64, 128)), (8, 100_000, 16, (5, 65, 9))])
def test_short_workspace_is_refused_on_the_host(fn, query, F, N, C, res):
    need = ctypes.c_size_t()
    rc, _ = _call(query, F=F, N=N, C=C, res=res, bytes=ctypes.byref(need))
    assert rc == 0 and need.value > 0
    rc, msg = _call(fn, F=F, N=N, C=C, res=res, ws_bytes=need.value - 1)
    assert rc == -2 and b"workspace too small" in msg and fn.encode() in msg, (rc, msg)


def test_nothing_to_do_reads_nothing():
    """F = 0 or N = 0: the forward returns before reading a pointer other than the plane table."""
    for e in (dict(F=0), dict(N=0)):
        rc, msg = _call("dghp_forward", box=None, x=None, t=None, out=None, **e)
        assert rc == 0, msg


def test_backward_workspace_bytes():
    """dL/dsample [E, C], fractions, four key / id arrays per entry (E = 3 S N (1 + F)) and the cells' corner sums."""
    n = ctypes.c_size_t()
    F, N, C, res = 8, 100_000, 32, (64, 128)
    _call("dghp_backward_workspace", F=F, N=N, C=C, res=res, bytes=ctypes.byref(n))
    E = 3 * 2 * N * (1 + F)
    cells = sum(3 * (R - 1) ** 2 + 3 * (R - 1) * 24 for R in res)
    low = E * (4 * C + 8 + 16) + cells * 16 * C
    assert low <= n.value < low * 1.2


# ---- ValueErrors that need no device -------------------------------------------------------------------------------
def test_bad_construction_is_refused():
    from hexplane import HexPlaneDeformNetwork, HexPlaneField
    box = BOX.float()
    for kw in (dict(channels=8), dict(channels=16.0), dict(channels=True), dict(base_resolution=0),
               dict(base_resolution=1, multires=(1,)), dict(multires=()), dict(multires=(1, 2, 3, 4, 5)),
               dict(multires=(1.5,)), dict(time_resolution=1), dict(base_resolution=2 ** 14)):
        with pytest.raises(ValueError):
            HexPlaneField(box, **kw)
    for b in ([[0.0] * 3], [[0.0] * 3, [0.0, 1.0, 1.0]], [[0.0] * 3, [float("inf")] * 3]):
        with pytest.raises(ValueError, match="box"):
            HexPlaneField(b)
    with pytest.raises(ValueError):
        HexPlaneDeformNetwork(box, W=0)


def test_cpu_tensors_and_bad_inputs_are_refused():
    from hexplane import HexPlaneField
    f = HexPlaneField(BOX.float(), channels=16, base_resolution=4)
    x, t = torch.zeros(10, 3), torch.zeros(10, 1)
    with pytest.raises(ValueError, match="CUDA"):
        f(x, t)
    with pytest.raises(ValueError, match="CUDA"):
        f.regularisers()
    with pytest.raises(ValueError, match="grad"):
        f(x, t.requires_grad_(True))
    for xx, tt in ((torch.zeros(10, 2), torch.zeros(10, 1)), (torch.zeros(10, 3), torch.zeros(9, 1)),
                   (torch.zeros(10, 3), torch.zeros(10)), (torch.zeros(10, 3), torch.zeros(2, 10, 2))):
        with pytest.raises(ValueError):
            f(xx, tt)
    with pytest.raises(ValueError, match="float32"):
        f(x.double(), torch.zeros(10, 1))
