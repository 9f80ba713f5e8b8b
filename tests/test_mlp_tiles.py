"""Deformation / appearance MLPs, tile by tile: the persistent GEMM kernels of csrc/mlp_gemm.cuh at the row-tile
counts where their schedules wrap, against a float64 autograd reference of the same networks.

tests/test_mlp.py compares each gradient as one tensor under the 2 % bf16 bound.  That bound cannot see a single
tile: at n = 517 the last tile holds 5 rows, and at 100 000 rows one tile is 0.1 % of dW.  Here the rows are
split into groups that line up with the kernels' schedule (128-row tiles; `layer_gemm_kernel` runs min(tiles, S)
CTAs, `dw_gemm_kernel` min(tiles, S/2) x 2, S = number of SMs) and every group's gradients are checked on their
own, so a dropped, doubled or misattributed tile, row or CTA round is an error of order 1:

  * row locality, exact: dx and the outputs of a row depend on that row's x, t and upstream gradient only
    (forward GEMMs read their own row, the bf16 rounding of dZ is elementwise, dE gets two ordered adds);
  * additivity: the gradients of the groups sum to the gradient of the whole (only the fp32 summation order
    differs);
  * each group alone against the float64 reference (bf16 backward bound).

The fp64 reference is the reference module (util.load_reference_networks()) holding the same state dict, in
float64.  For the single-pass 'bf16' precision it is the same network with the forward's bf16 rounding points
(bf16 operands; tests/test_mlp.py explains why that mode is not within 2 % of the unrounded network).
"""
import importlib
import os
import subprocess
import sys
import tempfile

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if __name__ == "__main__":          # stand-alone run (the streaming-weights subprocess): the paths of conftest.py
    for _p in (ROOT, os.path.join(ROOT, "dg-mesh_b200"), os.path.join(ROOT, "tests")):
        if _p not in sys.path:
            sys.path.insert(0, _p)

import util  # noqa: E402

ref = util.load_reference_networks()

TILE = 128   # rows per activation tile (ACT_R)

# network configurations: (class, constructor keywords)
NETS = {
    "normal_blender": ("DeformNetworkNormal", dict(is_blender=True)),
    "normal_direct": ("DeformNetworkNormal", dict(is_blender=False)),
    "appearance": ("AppearanceNetwork", dict(is_blender=True)),
    "normal_6dof": ("DeformNetworkNormal", dict(is_blender=True, is_6dof=True)),
}

# row counts, resolved against the SM count S at run time (tiles = ceil(P / 128)): the edges of one tile, the
# first dw round filled (S/2 tiles) and wrapped (+1 row), the first layer round filled and wrapped, three rounds
SIZES = ("1", "127", "128", "129", "S/2*128", "S/2*128+1", "S*128", "S*128+1", "2S*128+1", "100000")


def rows_for(size, S):
    return {"S/2*128": S // 2 * TILE, "S/2*128+1": S // 2 * TILE + 1, "S*128": S * TILE, "S*128+1": S * TILE + 1,
            "2S*128+1": 2 * S * TILE + 1}.get(size) or int(size)


def sm_count():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


# ------------------------------------------------------------------------------------------------ the harness
def partition(P, S, seed=0):
    """Disjoint row groups covering 0..P-1, aligned with the kernels' schedule: [(name, sorted row indices)].
    Tile S/2 is the first tile a dw CTA takes in its second round, tile S the first a layer CTA takes in its
    second round.  Groups that do not exist at this P (or are already taken) are left out."""
    tiles = -(-P // TILE)
    taken = torch.zeros(P, dtype=torch.bool)
    groups = []

    def add(name, rows):
        rows = rows[~taken[rows]]
        if rows.numel():
            taken[rows] = True
            groups.append((name, rows))

    for name, k in (("tile 0", 0), ("last tile", tiles - 1), ("tile S/2", S // 2), ("tile S", S)):
        if 0 <= k < tiles:
            add(name, torch.arange(k * TILE, min(P, (k + 1) * TILE)))
    free = (~taken).nonzero().flatten()
    pick = torch.randperm(free.numel(), generator=torch.Generator().manual_seed(seed))[:max(1, free.numel() // 100)]
    add("scattered 1%", free[pick].sort().values)
    add("rest", (~taken).nonzero().flatten())
    return groups


def masked(g, rows):
    """The upstream gradient g with every row outside `rows` set to exactly zero."""
    m = torch.zeros_like(g)
    m[rows.to(g.device)] = g[rows.to(g.device)]
    return m


def flat(outs):
    """A network's outputs (a tensor or a tuple; the 6-dof transform is [P, 4, 4]) as one [P, C] tensor."""
    outs = outs if isinstance(outs, tuple) else (outs,)
    return torch.cat([o.reshape(o.shape[0], -1) for o in outs], -1)


def grads_of(net, x, t, gs, forward=None):
    """One forward of `net` (or `forward(net, x, t)`) at (x, t), one backward per upstream gradient in `gs`.
    Returns (outputs [P, C], [(dx, {parameter name: gradient}) per g])."""
    xr = x.detach().clone().requires_grad_(True)
    out = flat(forward(net, xr, t) if forward else net(xr, t))
    names, params = zip(*net.named_parameters())
    res = []
    for g in gs:
        gr = torch.autograd.grad(out, (xr,) + params, g, retain_graph=True)
        res.append((gr[0], dict(zip(names, gr[1:]))))
    return out.detach(), res


def make_nets(tu, key, device, seed=1):
    """(network under test, fp64 reference module with the same state dict)."""
    cls, kw = NETS[key]
    torch.manual_seed(seed)
    mine = getattr(tu, cls)(**kw).to(device)
    theirs = getattr(ref.time_utils, cls)(**kw)
    theirs.load_state_dict(mine.state_dict())
    return mine, theirs.double().to(device)


def inputs(P, uniform, seed, width):
    """x ~ 0.6 N(0, 1); t one value for every row (DG-Mesh's case) or a mix; g ~ N(0, 1) of the output width."""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(P, 3, generator=gen) * 0.6
    t = torch.full((P, 1), 0.37)
    if not uniform:
        t[::3] = torch.rand(t[::3].shape, generator=gen)
    g = torch.randn(P, width, generator=gen)
    return x, t, g


def out_width(key):
    """Columns of flat(outputs): colour 3; warp (3, or the 4 x 4 transform with is_6dof), rotation, scaling, normal."""
    cls, kw = NETS[key]
    return 3 if cls == "AppearanceNetwork" else (16 if kw.get("is_6dof") else 3) + 10


def bf16_forward(net, x, t):
    """The network with the single-pass forward's rounding points: bf16 operands of every GEMM (fp64 otherwise),
    straight-through gradients.  Not for is_6dof."""
    def bf(v):
        return v + (v.bfloat16().to(v.dtype) - v).detach()

    def pe(v, L):
        return torch.cat([v] + [f(v * 2.0 ** k) for k in range(L) for f in (torch.sin, torch.cos)], -1)

    def lin(m, h):
        return bf(h) @ bf(m.weight).t() + m.bias

    x_emb = pe(x, 10)
    t_emb = lin(net.timenet[2], torch.relu(lin(net.timenet[0], pe(t, 6)))) if net.is_blender else pe(t, 10)
    e = torch.cat([x_emb, t_emb], -1)
    h = e
    for i, l in enumerate(net.linear):
        h = torch.relu(lin(l, h))
        if i == 4:
            h = torch.cat([e, h], -1)
    if type(net).__name__ == "AppearanceNetwork":
        return torch.sigmoid(lin(net.color_warp[0], h))
    return tuple(lin(getattr(net, n), h) for n in ("gaussian_warp", "gaussian_rotation", "gaussian_scaling",
                                                    "gaussian_normal"))


def max_rel(a, b):
    """max |a - b| / max |b| (0 when both are all zero)."""
    d = float((a.double() - b.double()).abs().max()) if a.numel() else 0.0
    s = float(b.double().abs().max()) if b.numel() else 0.0
    return d / s if s > 0 else (0.0 if d == 0 else float("inf"))


def rel_l2(a, b):
    d, s = float((a.double() - b.double()).norm()), float(b.double().norm())
    return d / s if s > 0 else (0.0 if d == 0 else float("inf"))


# --------------------------------------------------------------------------------------------------- CPU
def test_harness_is_exact_on_the_reference_cpu():
    """The masking, partition and gradient helpers on the fp64 reference module: the groups' gradients sum to the
    whole to ~1e-12, an all-rows mask reproduces the unmasked gradient exactly, and dx is row-local.  A GPU
    failure below therefore points at the kernels, not at the harness."""
    torch.manual_seed(1)
    net = ref.time_utils.DeformNetworkNormal(is_blender=True).double()
    S = 2                                         # 5 tiles: tile 0, tile S/2 = 1, tile S = 2, tile 3, last tile 4
    P = 2 * S * TILE + 1
    groups = partition(P, S)
    assert [n for n, _ in groups] == ["tile 0", "last tile", "tile S/2", "tile S", "scattered 1%", "rest"]
    allrows = torch.cat([r for _, r in groups]).sort().values
    assert torch.equal(allrows, torch.arange(P))
    assert groups[1][1].tolist() == [P - 1] and groups[2][1][0] == TILE and groups[3][1][0] == 2 * TILE
    x, t, g = inputs(P, False, 3, 13)
    x, t, g = x.double(), t.double(), g.double()
    _, res = grads_of(net, x, t, [g, masked(g, torch.arange(P))] + [masked(g, r) for _, r in groups])
    (dx, full), (dx1, ones) = res[0], res[1]
    assert torch.equal(dx, dx1) and all(torch.equal(full[k], ones[k]) for k in full)
    for k in full:
        assert max_rel(sum(r[1][k] for r in res[2:]), full[k]) < 1e-12, k
    for (_, rows), (dxg, _) in zip(groups, res[2:]):
        assert torch.equal(dxg[rows], dx[rows])
        rest = torch.ones(P, dtype=torch.bool)
        rest[rows] = False
        assert not dxg[rest].any()
    # every parameter of the network takes part (a group's gradient is not trivially zero)
    assert all(res[2][1][k].abs().sum() > 0 for k in full)


# --------------------------------------------------------------------------------------------------- GPU
def _cases():
    c = []
    for prec in ("bf16x3", "bf16"):
        for size in SIZES:
            for uniform in (True, False):
                c.append(("normal_blender", size, uniform, prec))
        for key in ("normal_direct", "appearance"):
            for size in SIZES[:-1]:        # 100 000 rows: the blender network only
                c.append((key, size, False, prec))
    for size in ("129", "S*128+1"):        # single-pass bf16 has no fp64 stand-in with the screw head
        c.append(("normal_6dof", size, False, "bf16x3"))
    return c


CASES = _cases()
CASE_IDS = [f"{k}-{s}-{'uniform' if u else 'mixed'}_t-{p}" for k, s, u, p in CASES]


@pytest.fixture
def precision():
    tu = importlib.import_module("utils.time_utils")
    yield tu.set_precision
    tu.set_precision("bf16x3")


@pytest.mark.gpu
@pytest.mark.parametrize("key,size,uniform,prec", CASES, ids=CASE_IDS)
def test_rows_are_independent_and_permutable(key, size, uniform, prec, precision):
    """Bit-exact row locality.  With g zero outside a set of rows R, dx on R is bit-identical to dx from the full
    g and exactly zero elsewhere, and the outputs do not change; permuting the rows of (x, t, g) permutes the
    outputs and dx bit-identically (a row's results do not depend on its tile or its position in the tile)."""
    tu = importlib.import_module("utils.time_utils")
    precision(prec)
    P = rows_for(size, sm_count())
    mine, _ = make_nets(tu, key, "cuda")
    x, t, g = (v.cuda() for v in inputs(P, uniform, 5, out_width(key)))
    gen = torch.Generator().manual_seed(6)
    R = torch.cat([torch.arange((P - 1) // TILE * TILE, P), torch.randperm(P, generator=gen)[:max(1, P // 50)]])
    R = R.unique()
    out, [(dx, _)] = grads_of(mine, x, t, [g])
    out1, [(dx1, _)] = grads_of(mine, x, t, [masked(g, R)])
    assert torch.equal(out1, out), "outputs differ between two identical calls"
    assert torch.equal(dx1[R.cuda()], dx[R.cuda()]), "dx of a row depends on other rows' upstream gradient"
    off = torch.ones(P, dtype=torch.bool, device="cuda")
    off[R.cuda()] = False
    assert not dx1[off].any(), "rows with zero upstream gradient got a nonzero dx"
    perm = torch.randperm(P, generator=gen).cuda()
    out2, [(dx2, _)] = grads_of(mine, x[perm], t[perm], [g[perm]])
    assert torch.equal(out2, out[perm]), "outputs are not permutation-equivariant"
    assert torch.equal(dx2, dx[perm]), "dx is not permutation-equivariant"


# Per-group bound against fp64, relative L2 per parameter tensor and for dx.
GROUP_BOUND = 0.05
ADD_BOUND = 1e-5
ADD_BOUND_UNIFORM_TIMENET = 2e-2


@pytest.mark.gpu
@pytest.mark.parametrize("key,size,uniform,prec", CASES, ids=CASE_IDS)
def test_tile_gradients_add_up_and_match_fp64(key, size, uniform, prec, precision):
    """Every schedule-aligned group of rows (tile 0, the last tile, tile S/2, tile S, ~1 % scattered rows, the
    rest) on its own.

    Additivity: the groups' gradients sum to the full gradient for every parameter tensor, biases and time-net
    included (max-norm relative).  Only the fp32 summation order differs: bound 1e-5, measured <= 7.3e-7 on an
    H100 SXM (400 W).  One exception, by design: with one t for every row the time-net's backward runs on a single
    row that holds the column sum of all rows' time-feature gradients (tfeat_colsum_kernel), and that sum is
    rounded to bf16 as the time-net's dZ.  Rounding a sum is not additive, so the four time-net tensors add up to
    bf16 precision only: bound 2e-2, measured 2.0e-3 .. 6.4e-3 (two bf16 roundings, 2^-8 each).

    Against fp64: each group's gradients, alone, within the bf16 backward bound: relative L2 per tensor and for
    dx, bound 0.05; measured <= 0.0234 over all groups, networks, sizes and both precisions (whole tensors
    0.004-0.018).  A missing or doubled tile is an error of 1."""
    tu = importlib.import_module("utils.time_utils")
    precision(prec)
    S = sm_count()
    P = rows_for(size, S)
    mine, theirs = make_nets(tu, key, "cuda")
    x, t, g = (v.cuda() for v in inputs(P, uniform, 7, out_width(key)))
    groups = partition(P, S)
    gs = [g] + [masked(g, rows) for _, rows in groups]
    _, got = grads_of(mine, x, t, gs)
    fwd = bf16_forward if prec == "bf16" else None
    _, want = grads_of(theirs, x.double(), t.double(), [v.double() for v in gs], fwd)
    full = got[0][1]
    add = {k: max_rel(sum(r[1][k] for r in got[1:]), full[k]) for k in full}
    errs = {}
    for (name, _), (dx, gp), (dx64, gp64) in zip([("all", None)] + groups, got, want):
        e = {k: rel_l2(gp[k], gp64[k]) for k in gp}
        e["dx"] = rel_l2(dx, dx64)
        errs[name] = e
    worst = {n: max(e, key=e.get) for n, e in errs.items()}
    print(f"\n{key} P={P} {'uniform' if uniform else 'mixed'} t {prec}: additivity max "
          f"{max(add.values()):.2e} ({max(add, key=add.get)}); vs fp64 worst per group "
          + ", ".join(f"{n} {errs[n][k]:.4f} ({k})" for n, k in worst.items()))
    bound = {k: ADD_BOUND_UNIFORM_TIMENET if uniform and k.startswith("timenet.") else ADD_BOUND for k in add}
    bad_add = {k: v for k, v in add.items() if not v < bound[k]}
    assert not bad_add, f"group gradients do not add up to the full gradient: {bad_add}"
    bad = {(n, k): v for n, e in errs.items() for k, v in e.items() if not v < GROUP_BOUND}
    assert not bad, f"group gradients vs fp64: {bad}"


@pytest.mark.gpu
@pytest.mark.parametrize("key", list(NETS))
def test_zero_rows(key):
    """P = 0: correctly shaped empty outputs and dx, all-zero parameter gradients."""
    tu = importlib.import_module("utils.time_utils")
    mine, theirs = make_nets(tu, key, "cuda")
    x = torch.zeros(0, 3, device="cuda", requires_grad=True)
    t = torch.zeros(0, 1, device="cuda")
    outs, want = mine(x, t), theirs(x.double(), t.double())
    outs, want = (o if isinstance(o, tuple) else (o,) for o in (outs, want))
    assert [o.shape for o in outs] == [w.shape for w in want]
    sum(o.sum() for o in outs).backward()
    assert x.grad.shape == (0, 3)
    for k, p in mine.named_parameters():
        assert p.grad is not None and p.grad.shape == p.shape and not p.grad.any(), k


# ------------------------------------------------------------------------- resident vs streaming weights
STREAM_SIZE = "S*128+1"


def _stream_run(path):
    """Outputs and gradients of every network at STREAM_SIZE rows (bf16x3): returned, and saved to `path`."""
    tu = importlib.import_module("utils.time_utils")
    tu.set_precision("bf16x3")
    P = rows_for(STREAM_SIZE, sm_count())
    res = {}
    for key in NETS:
        mine, _ = make_nets(tu, key, "cuda")
        x, t, g = (v.cuda() for v in inputs(P, False, 9, out_width(key)))
        out, [(dx, gp)] = grads_of(mine, x, t, [g])
        res[key] = {"out": out.cpu(), "dx": dx.cpu(), **{k: v.cpu() for k, v in gp.items()}}
    if path:
        torch.save(res, path)
    return res


@pytest.mark.gpu
def test_resident_and_streaming_weights_agree():
    """DGMESH_B200_MLP_STREAM=1 (read once per process: a subprocess) forces the streaming layer kernel where
    the split-precision forward otherwise keeps B_hi resident in shared memory.

    The two are not bit-identical, by construction: the streaming kernel accumulates the three split-precision
    products pass by pass (all K steps of A_hi B_hi, then A_lo B_hi, then A_hi B_lo), the resident kernel K step
    by K step, so the fp32 sums round differently.  Outputs agree at fp32 level (max-norm relative bound 2e-5;
    measured 4.0e-6 on an H100 SXM).  The backward reads the bf16 (hi) activations only, and an activation that
    rounds to the neighbouring bf16 number changes the gradients at bf16 level (measured up to 3.8e-3 relative
    L2 between the variants): each variant's gradients are held to the 2 % contract against fp64 instead."""
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "stream.pt")
        env = dict(os.environ, DGMESH_B200_MLP_STREAM="1")
        flags = ["-s"] if sys.flags.no_user_site else []
        r = subprocess.run([sys.executable, *flags, os.path.abspath(__file__), path], env=env, cwd=ROOT,
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        st = torch.load(path)
    res = _stream_run(None)
    for key in NETS:
        _, theirs = make_nets(importlib.import_module("utils.time_utils"), key, "cuda")
        x, t, g = (v.cuda().double() for v in inputs(rows_for(STREAM_SIZE, sm_count()), False, 9, out_width(key)))
        out64, [(dx64, gp64)] = grads_of(theirs, x, t, [g])
        want = {"out": out64.cpu(), "dx": dx64.cpu(), **{k: v.cpu() for k, v in gp64.items()}}
        same = all(torch.equal(res[key][k], st[key][k]) for k in res[key])
        e_out = max_rel(st[key]["out"], res[key]["out"])
        errs = {(v, k): rel_l2(r[k], want[k]) for v, r in (("resident", res[key]), ("stream", st[key]))
                for k in want if k != "out"}
        print(f"\n{key}: bit-identical {same}; outputs max-rel {e_out:.2e}; gradients vs fp64: worst "
              f"{max(errs.values()):.4f}; between the variants: worst rel L2 "
              f"{max(rel_l2(st[key][k], res[key][k]) for k in want if k != 'out'):.2e}")
        assert e_out < 2e-5, key
        bad = {k: v for k, v in errs.items() if not v < 2e-2}
        assert not bad, (key, bad)


# ----------------------------------------------------------------------------------- packed-weight cache
@pytest.mark.gpu
@pytest.mark.parametrize("key", ["normal_blender", "normal_6dof"])
def test_weight_updates_reach_the_packed_weights(key):
    """The packed bf16 weights are reused while every parameter keeps its (data_ptr, _version).  Each supported
    kind of weight update must reach the kernels: after each, the outputs match the fp64 reference holding the
    updated weights, and differ from the previous outputs by far more than that bound (a stale cache fails).
    Not supported, and not tested: writes through `.data` (`p.data.mul_(2)`) leave `_version` unchanged, so the
    cache keeps serving the old weights (utils/time_utils.py)."""
    tu = importlib.import_module("utils.time_utils")
    mine, _ = make_nets(tu, key, "cuda")
    x, t, g = (v.cuda() for v in inputs(1000, False, 11, out_width(key)))

    def check(what, prev):
        theirs = getattr(ref.time_utils, NETS[key][0])(**NETS[key][1])
        theirs.load_state_dict(mine.state_dict())
        theirs = theirs.double().cuda()
        with torch.no_grad():
            want = flat(theirs(x.double(), t.double()))
        out = flat(mine(x, t)).detach()
        assert rel_l2(out, want) < 1e-4, what
        assert prev is None or rel_l2(prev, want) > 1e-3, f"{what}: the update did not change the network"
        return out

    out = check("initial", None)
    opt = torch.optim.Adam(mine.parameters(), lr=1e-2)
    (flat(mine(x, t)) * g).sum().backward()
    opt.step()
    out = check("Adam step", out)
    with torch.no_grad():
        for p in mine.parameters():
            p.mul_(1.2)
    out = check("in-place edit under no_grad", out)
    other, _ = make_nets(tu, key, "cuda", seed=2)
    mine.load_state_dict(other.state_dict())
    out = check("load_state_dict", out)
    mine.linear[3].weight = torch.nn.Parameter(torch.randn_like(mine.linear[3].weight) * 0.1)
    out = check("trunk parameter replaced by a new tensor", out)
    mine.gaussian_rotation.weight = torch.nn.Parameter(torch.randn_like(mine.gaussian_rotation.weight) * 0.5)
    check("head parameter replaced by a new tensor", out)


if __name__ == "__main__":
    _stream_run(sys.argv[1])
