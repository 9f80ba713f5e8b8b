"""Hash-grid field on the device (dg-mesh_b200/hashgrid.py, csrc/hashgrid.cu) against the float64 restatement
(tests/hashgrid_oracle.py) at N = 10^5, L = 16.

Configurations cover F = 1 and 8, Fe = 2 and 4, all four grids and ("xyz",), log2_table = 19 and 12 (at 12 most
levels hash and collide heavily).  The points are uniform in the box, 5 % outside it, 5 % on each of three faces,
some exactly on nodes of several levels, the rest random off-lattice coordinates; times are 0, 1, time nodes and
random values.  The oracle repeats the two float32 coordinate steps, so every point falls in the same cell on both
sides.  Bounds are relative to max(1, max|ref|) per tensor."""
import pytest
import torch

import hashgrid_oracle as ho

pytestmark = pytest.mark.gpu

BOX = [[-1.0, -2.0, -0.5], [1.0, 2.0, 1.5]]
N = 100_000
TOL = dict(features=2e-6, x=2e-5, tables=2e-5)
ALL = ho.GRIDS
# (F, Fe, grids, log2_table): every value of every axis at least once
CONFIGS = [(8, 2, ALL, 19), (1, 4, ALL, 12), (8, 4, ("xyz",), 12), (1, 2, ("xyz",), 19)]
WORST = {}


def _field(Fe=2, grids=ALL, log2T=19, seed=0, **kw):
    from hashgrid import HashGridField
    torch.manual_seed(seed)
    f = HashGridField(BOX, grids=grids, features=Fe, log2_table=log2T, **kw).cuda()
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for p in f.tables:       # away from the initialisation, so that every slot matters
            p.copy_(torch.rand(p.shape, generator=g) * 2 - 1)
    return f


def _points(seed=0, n=N):
    g = torch.Generator().manual_seed(seed)
    lo, hi = torch.tensor(BOX[0]), torch.tensor(BOX[1])
    x = lo + (hi - lo) * torch.rand(n, 3, generator=g)
    out = torch.rand(n, generator=g) < 0.05
    x[out] += (torch.rand(int(out.sum()), 3, generator=g) - 0.5) * 4                # outside the box
    m = n // 20
    x[m:2 * m, 0] = lo[0]                                                          # faces
    x[2 * m:3 * m, 1] = hi[1]
    x[3 * m:4 * m, 2] = lo[2]
    # nodes of the levels whose resolution divides 2^11 (16 and 2048 at the defaults): u = k / 2^11 is exact
    k = torch.randint(0, 2 ** 11 + 1, (2 * m, 3), generator=g).float()
    x[4 * m:6 * m] = lo + (hi - lo) * k / 2 ** 11
    return x.cuda()


def _times(F, seed=0, n=N, Rt=32):
    g = torch.Generator().manual_seed(100 + seed)
    t = torch.rand(F, n, 1, generator=g)
    q = n // 10
    t[:, :q] = 0.0
    t[:, q:2 * q] = 1.0
    t[:, 2 * q:3 * q] = torch.randint(0, Rt + 1, (F, q, 1), generator=g).float() / Rt
    return t.cuda()


def _rel(a, b):
    return float((a.double().cpu() - b.double().cpu()).abs().max()) / max(1.0, float(b.abs().max()))


def _note(key, e):
    WORST[key] = max(WORST.get(key, 0.0), e)
    print(f"worst {key}: {WORST[key]:.2e}")


def _run(f, x, t, gout):
    xl = x.clone().requires_grad_(True)
    for p in f.tables:
        p.grad = None
    out = f(xl, t)
    out.backward(gout)
    return out.detach(), xl.grad, [p.grad.clone() for p in f.tables]


@pytest.mark.parametrize("F,Fe,grids,log2T", CONFIGS, ids=[f"F{c[0]}-Fe{c[1]}-G{len(c[2])}-T{c[3]}" for c in CONFIGS])
def test_field_and_gradients_against_float64(F, Fe, grids, log2T):
    f = _field(Fe, grids, log2T)
    x, t = _points(), _times(F)
    gout = torch.randn(F, N, f.out_dim, generator=torch.Generator().manual_seed(7)).cuda()
    out, gx, gt = _run(f, x, t, gout)
    ref, rgx, rgt = ho.of(f, x, t, gout)
    e_f, e_x = _rel(out, ref), _rel(gx, rgx)
    e_t = max(_rel(a, b) for a, b in zip(gt, rgt))
    _note("features", e_f), _note("x", e_x), _note("tables", e_t)
    assert e_f < TOL["features"] and e_x < TOL["x"] and e_t < TOL["tables"], (e_f, e_x, e_t)
    # the coordinate gradient is zero wherever a coordinate is strictly outside the box
    lo, hi = f.box[0], f.box[1]
    outside = (x < lo) | (x > hi)
    assert not gx[outside].any()
    if F == 1:
        assert torch.equal(f(x, t[0]), out[0])
    if grids == ("xyz",):
        assert torch.equal(f(x), out[0])
        assert all(torch.equal(out[k], out[0]) for k in range(F))


def test_hot_slot_and_extreme_scales():
    """Every point at one location: about 10^5 contributions per slot; grad_out scaled by 1e30 and 1e-30; zeros;
    a NaN."""
    f = _field(2, ALL, 19, seed=2)
    x = torch.tensor([[0.1234, -0.777, 0.31]], device="cuda").expand(N, 3).contiguous()
    t = torch.full((1, N, 1), 0.4321, device="cuda")
    gout = torch.rand(1, N, f.out_dim, generator=torch.Generator().manual_seed(3)).cuda() + 0.5   # same sign
    ref, rgx, rgt = ho.of(f, x, t, gout)
    for s in (1.0, 1e30, 1e-30):
        out, gx, gt = _run(f, x, t, gout * s)
        e_t = max(_rel(a / s, b) for a, b in zip(gt, rgt))
        e_x = _rel(gx / s, rgx)
        _note("tables", e_t)
        assert all(torch.isfinite(a).all() for a in gt) and e_t < TOL["tables"] and e_x < TOL["x"], (s, e_t, e_x)
    _, gx, gt = _run(f, x, t, torch.zeros_like(gout))
    assert not gx.any() and not any(a.any() for a in gt)
    bad = gout.clone()
    bad[0, 17, 5] = float("nan")           # grid 0, level 2
    _, _, gt = _run(f, x, t, bad)
    assert not torch.isfinite(gt[0][2]).all()
    assert torch.isfinite(gt[0][3]).all() and torch.isfinite(gt[1]).all()


def test_two_runs_are_bit_identical_and_frames_are_single_frames():
    f = _field(2, ALL, 12, seed=5)
    x, t = _points(5), _times(8, 5)
    gout = torch.randn(8, N, f.out_dim, generator=torch.Generator().manual_seed(9)).cuda()
    a, b = _run(f, x, t, gout), _run(f, x, t, gout)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert all(torch.equal(p, q) for p, q in zip(a[2], b[2]))
    with torch.no_grad():
        for k in range(8):
            assert torch.equal(a[0][k], f(x, t[k])), k
        assert torch.equal(f(x, t[:1])[0], f(x, t[0]))


def test_network_against_the_oracle_encoding():
    from hashgrid import HashGridDeformNetwork
    torch.manual_seed(0)
    net = HashGridDeformNetwork(BOX, normal=True, log2_table=14).cuda()
    g = torch.Generator().manual_seed(2)
    with torch.no_grad():
        for p in net.field.tables:
            p.copy_(torch.rand(p.shape, generator=g) * 2 - 1)
    x, t = _points(8, n=20_000), _times(4, 8, n=20_000)
    outs = net(x, t)
    assert [tuple(o.shape) for o in outs] == [(4, 20_000, r) for r in (3, 4, 3, 3)]
    sum((o * o).sum() for o in outs).backward()
    got = [p.grad.clone() for p in net.parameters()]
    net.zero_grad()
    feats = ho.of(net.field, x, t)[0]
    h = net.feature_out(feats.float().cuda())
    ref = tuple(getattr(net, name)(h) for name, _ in net.heads)
    sum((o * o).sum() for o in ref).backward()
    for o, r in zip(outs, ref):
        assert _rel(o.detach(), r.detach()) < 1e-4
    for a, p in zip(got[len(net.field.tables):], list(net.parameters())[len(net.field.tables):]):
        assert _rel(a, p.grad) < 1e-3


def test_state_dict_round_trip():
    from hashgrid import HashGridDeformNetwork
    torch.manual_seed(0)
    a = HashGridDeformNetwork(BOX, log2_table=14).cuda()
    with torch.no_grad():
        for p in a.field.tables:
            p.add_(0.1 * torch.randn_like(p))
    sd = a.state_dict()
    assert "field.box" in sd and "field.tables.3" in sd and "gaussian_warp.3.weight" in sd
    torch.manual_seed(1)
    b = HashGridDeformNetwork([[0.0] * 3, [1.0] * 3], log2_table=14).cuda()
    b.load_state_dict(sd)
    x, t = _points(9, n=5000), _times(2, 9, n=5000)
    with torch.no_grad():
        assert all(torch.equal(u, v) for u, v in zip(a(x, t), b(x, t)))


def test_fused_adam_fits_a_smooth_time_varying_deformation():
    """A point set moving as d(x, t) = 0.2 sin(2 pi t + x_y) (1, 0.5, -0.5): 300 FusedAdam steps on the frame batch
    take the loss below 1 % of where it starts."""
    from hashgrid import HashGridDeformNetwork
    from optim import FusedAdam
    torch.manual_seed(0)
    net = HashGridDeformNetwork(BOX, levels=8, log2_table=15, finest_resolution=128, time_resolution=8).cuda()
    opt = FusedAdam(net.parameters(), lr=3e-3)
    g = torch.Generator().manual_seed(3)
    x = (torch.tensor(BOX[0]) + torch.rand(4000, 3, generator=g) * (torch.tensor(BOX[1]) - torch.tensor(BOX[0])))
    x = x.cuda()
    t = torch.linspace(0, 1, 8, device="cuda")[:, None, None].expand(8, 4000, 1).contiguous()
    target = 0.2 * torch.sin(2 * torch.pi * t + x[None, :, 1:2]) * torch.tensor([1.0, 0.5, -0.5], device="cuda")
    losses = []
    for _ in range(300):
        d_xyz = net(x, t)[0]
        loss = (d_xyz - target).square().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    print(f"fit: loss {losses[0]:.3e} -> {losses[-1]:.3e}")
    assert losses[-1] < 0.01 * losses[0], (losses[0], losses[-1])


def test_render_batch_takes_the_per_frame_outputs():
    import gaussian_renderer as gr
    import synth
    from hashgrid import HashGridDeformNetwork
    from test_depth_alpha_gpu import BG
    from test_normal_map_gpu import _normal_model, _pipe
    model = _normal_model(1500, seed=3)
    cams = [synth.look_at_camera(azimuth_deg=30.0 * f, elevation_deg=10.0, radius=4.0, width=64, height=48,
                                 fovx=0.6911, fovy=0.6911 * 48 / 64, device="cuda") for f in range(3)]
    xyz = model.get_xyz.detach()
    box = torch.stack([xyz.min(0).values, xyz.max(0).values]).cpu()
    torch.manual_seed(0)
    net = HashGridDeformNetwork(box, log2_table=14).cuda()
    t = torch.tensor([0.1, 0.5, 0.9], device="cuda")[:, None, None].expand(3, xyz.shape[0], 1).contiguous()
    d_xyz, d_rot, d_scale = net(xyz, t)
    assert d_xyz.shape == (3, xyz.shape[0], 3)
    pkg = gr.render_batch(cams, model, _pipe(), torch.tensor(BG, device="cuda"), 0.01 * d_xyz, 0.01 * d_rot,
                          0.01 * d_scale)
    pkg["render"].square().sum().backward()
    for i, p in enumerate(net.field.tables):
        assert p.grad is not None and torch.isfinite(p.grad).all() and p.grad.abs().sum() > 0, i


def test_refusals_on_the_device():
    f = _field(2, ALL, 12)
    x, t = _points(n=100), _times(1, n=100)[0]
    with pytest.raises(ValueError, match="grad"):
        f(x, t.clone().requires_grad_(True))
    with pytest.raises(ValueError, match="float32"):
        f(x.double(), t)
    with pytest.raises(ValueError):
        f(x, t[:50])
    with pytest.raises(ValueError, match="None"):
        f(x)
    with pytest.raises(ValueError, match="CUDA"):
        f(x.cpu(), t)
    with pytest.raises(ValueError, match="CUDA"):
        f(x, t.cpu())
