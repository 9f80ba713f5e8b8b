"""HexPlane field on the device (dg-mesh_b200/hexplane.py, csrc/hexplane.cu) against the float64 restatement
(tests/hexplane_oracle.py), at N = 10^5, S = 2, C = 16 and 32, F = 1 and 8.

The points are uniform in the box, 5 % outside it, some on the box faces and (where the field's texel nodes are
exact floats) on texel nodes; times are 0, 1, time nodes and random values.  Coordinates are multiples of
box width / 2^16, so the pixel coordinate is the same exact number in float32 and in float64: a coordinate
gradient is one-sided at a cell boundary, and a rounding on the other side of one would compare two different
cells' slopes.  Bounds are relative to max(1, max|ref|) per tensor."""
import pytest
import torch

import hexplane_oracle as ho

pytestmark = pytest.mark.gpu

BOX = [[-1.0, -2.0, -0.5], [1.0, 2.0, 1.5]]           # widths 2, 4, 2: the box scale is a power of two
# "nodes": R = 5 and 65 (R - 1 divides 2^16, so texel nodes are exact); "default": the field's defaults
CONFIGS = {"nodes": dict(base_resolution=5, multires=(1, 13)), "default": dict(base_resolution=64, multires=(1, 2))}
N = 100_000
TOL = dict(features=2e-6, x=2e-5, planes=2e-5, reg=1e-6, reg_grad=1e-6)
WORST = {}


def _field(C, cfg, seed=0):
    from hexplane import HexPlaneField
    torch.manual_seed(seed)
    f = HexPlaneField(BOX, channels=C, **CONFIGS[cfg]).cuda()
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for p in f.planes:       # away from the initialisation, so that every plane matters
            p.copy_(torch.rand(p.shape, generator=g) + 0.5)
    return f


def _points(cfg, seed=0, n=N):
    g = torch.Generator().manual_seed(seed)
    lo, hi = torch.tensor(BOX[0]), torch.tensor(BOX[1])
    k = torch.randint(0, 2 ** 16 + 1, (n, 3), generator=g).double()
    out = torch.rand(n, generator=g) < 0.05
    k[out] += torch.randint(-2 ** 15, 2 ** 15, (int(out.sum()), 3), generator=g).double() * 4    # outside the box
    m = n // 20
    k[m:2 * m, 0] = 0.0                       # faces
    k[2 * m:3 * m, 1] = 2.0 ** 16
    k[3 * m:4 * m, 2] = 0.0
    if cfg == "nodes":                        # texel nodes of both scales (every 1024 of the 2^16 steps)
        k[4 * m:6 * m] = (torch.randint(0, 65, (2 * m, 3), generator=g) * 1024).double()
    x = lo.double() + (hi - lo).double() * k / 2.0 ** 16
    assert torch.equal(x.float().double(), x)
    return x.float().cuda()


def _times(F, seed=0, n=N, Rt=25):
    g = torch.Generator().manual_seed(100 + seed)
    t = torch.rand(F, n, 1, generator=g)
    q = n // 10
    t[:, :q] = 0.0
    t[:, q:2 * q] = 1.0
    t[:, 2 * q:3 * q] = (torch.randint(0, Rt, (F, q, 1), generator=g).float() / (Rt - 1))
    return t.cuda()


def _rel(a, b):
    return float((a.double() - b.double()).abs().max()) / max(1.0, float(b.abs().max()))


def _note(key, e):
    WORST[key] = max(WORST.get(key, 0.0), e)
    print(f"worst {key}: {WORST[key]:.2e}")


def _run(f, x, t, gout):
    xl = x.clone().requires_grad_(True)
    for p in f.planes:
        p.grad = None
    out = f(xl, t)
    out.backward(gout)
    return out.detach(), xl.grad, [p.grad.clone() for p in f.planes]


@pytest.mark.parametrize("cfg", list(CONFIGS))
@pytest.mark.parametrize("C", [16, 32])
@pytest.mark.parametrize("F", [1, 8])
def test_field_and_gradients_against_float64(cfg, C, F):
    f = _field(C, cfg)
    x, t = _points(cfg), _times(F)
    gout = torch.randn(F, N, 2 * C, generator=torch.Generator().manual_seed(7)).cuda()
    out, gx, gp = _run(f, x, t, gout)
    ref, rgx, rgp = ho.field_and_grads(x, t, f.box, list(f.planes), 2, gout)
    e_f, e_x = _rel(out, ref), _rel(gx, rgx)
    e_p = max(_rel(a, b) for a, b in zip(gp, rgp))
    _note("features", e_f), _note("x", e_x), _note("planes", e_p)
    assert e_f < TOL["features"] and e_x < TOL["x"] and e_p < TOL["planes"], (e_f, e_x, e_p)
    # the coordinate gradient is zero wherever a coordinate is outside the box or on a face
    lo, hi = f.box[0], f.box[1]
    flat = ((x <= lo) | (x >= hi))
    assert not gx[flat].any()
    # the single-frame call takes [N,1] and returns [N, S C]
    if F == 1:
        assert torch.equal(f(x, t[0]), out[0])


@pytest.mark.parametrize("C", [16, 32])
def test_regularisers_against_float64(C):
    f = _field(C, "default", seed=3)
    w = (0.7, 1.3, 0.9)
    ls = f.regularisers()
    sum(wi * li for wi, li in zip(w, ls)).backward()
    ref, rg = ho.regularisers_and_grads(list(f.planes), 2, w)
    e_l = max(abs(float(a) - float(b)) / max(1.0, abs(float(b))) for a, b in zip(ls, ref))
    e_g = max(_rel(p.grad, r) for p, r in zip(f.planes, rg))
    _note("reg", e_l), _note("reg_grad", e_g)
    assert e_l < TOL["reg"] and e_g < TOL["reg_grad"], (e_l, e_g)
    # a new field: time planes all ones, so l1_time and time_smooth are 0; tv of uniform noise is positive
    from hexplane import HexPlaneField
    tv, ts, l1 = HexPlaneField(BOX, channels=C).cuda().regularisers()
    assert float(ts) == 0.0 and float(l1) == 0.0 and float(tv) > 0.0


def test_two_runs_are_bit_identical():
    f = _field(32, "default", seed=5)
    x, t = _points("default", 5), _times(8, 5)
    gout = torch.randn(8, N, 64, generator=torch.Generator().manual_seed(9)).cuda()
    a, b = _run(f, x, t, gout), _run(f, x, t, gout)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert all(torch.equal(p, q) for p, q in zip(a[2], b[2]))
    r = [f.regularisers() for _ in range(2)]
    grads = []
    for ls in r:
        for p in f.planes:
            p.grad = None
        sum(ls).backward()
        grads.append([p.grad.clone() for p in f.planes])
    assert all(torch.equal(u, v) for u, v in zip(r[0], r[1]))
    assert all(torch.equal(u, v) for u, v in zip(*grads))


@pytest.mark.parametrize("C", [16, 32])
def test_batch_frames_are_single_frames_to_the_bit(C):
    f = _field(C, "default", seed=6)
    x, t = _points("default", 6), _times(8, 6)
    with torch.no_grad():
        batch = f(x, t)
        for k in range(8):
            assert torch.equal(batch[k], f(x, t[k])), k
        assert torch.equal(f(x, t[:1])[0], f(x, t[0]))


def test_network_against_the_oracle_encoding():
    from hexplane import HexPlaneDeformNetwork
    torch.manual_seed(0)
    net = HexPlaneDeformNetwork(BOX, normal=True, channels=32).cuda()
    g = torch.Generator().manual_seed(2)
    with torch.no_grad():
        for p in net.field.planes:
            p.copy_(torch.rand(p.shape, generator=g) + 0.5)
    x, t = _points("default", 8, n=20_000), _times(4, 8, n=20_000)
    outs = net(x, t)
    assert [tuple(o.shape) for o in outs] == [(4, 20_000, r) for r in (3, 4, 3, 3)]
    sum((o * o).sum() for o in outs).backward()
    got = [p.grad.clone() for p in net.parameters()]
    net.zero_grad()
    # the same module with the encoding replaced by the oracle, in float32 after the field
    feats = ho.field(x.double(), t.double(), net.field.box.double(), [p.double() for p in net.field.planes], 2)
    h = net.feature_out(feats.float())
    ref = tuple(getattr(net, name)(h) for name, _ in net.heads)
    sum((o * o).sum() for o in ref).backward()
    for o, r in zip(outs, ref):
        assert _rel(o.detach(), r.detach()) < 1e-4
    for a, p in zip(got, net.parameters()):
        assert _rel(a, p.grad) < 1e-3


def test_state_dict_round_trip():
    from hexplane import HexPlaneDeformNetwork
    torch.manual_seed(0)
    a = HexPlaneDeformNetwork(BOX, channels=16).cuda()
    with torch.no_grad():
        for p in a.field.planes:
            p.add_(0.1 * torch.randn_like(p))
    sd = a.state_dict()
    assert "field.box" in sd and "field.planes.0" in sd
    torch.manual_seed(1)
    b = HexPlaneDeformNetwork([[0.0] * 3, [1.0] * 3], channels=16).cuda()
    b.load_state_dict(sd)
    x, t = _points("default", 9, n=5000), _times(2, 9, n=5000)
    with torch.no_grad():
        assert all(torch.equal(u, v) for u, v in zip(a(x, t), b(x, t)))


def test_fused_adam_fits_a_smooth_time_varying_deformation():
    """A point set moving as d(x, t) = 0.2 sin(2 pi t + x_y) (1, 0.5, -0.5): 300 FusedAdam steps on the frame batch
    take the loss below 1 % of where it starts."""
    from hexplane import HexPlaneDeformNetwork
    from optim import FusedAdam
    torch.manual_seed(0)
    net = HexPlaneDeformNetwork(BOX, channels=16, base_resolution=16, time_resolution=9).cuda()
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
    from hexplane import HexPlaneDeformNetwork
    from test_depth_alpha_gpu import BG
    from test_normal_map_gpu import _normal_model, _pipe
    model = _normal_model(1500, seed=3)
    cams = [synth.look_at_camera(azimuth_deg=30.0 * f, elevation_deg=10.0, radius=4.0, width=64, height=48,
                                 fovx=0.6911, fovy=0.6911 * 48 / 64, device="cuda") for f in range(3)]
    xyz = model.get_xyz.detach()
    box = torch.stack([xyz.min(0).values, xyz.max(0).values]).cpu()
    torch.manual_seed(0)
    net = HexPlaneDeformNetwork(box, channels=16).cuda()
    with torch.no_grad():   # make the field depend on time
        for p in net.field.planes:
            p.add_(0.05 * torch.randn_like(p))
    t = torch.tensor([0.1, 0.5, 0.9], device="cuda")[:, None, None].expand(3, xyz.shape[0], 1).contiguous()
    d_xyz, d_rot, d_scale = net(xyz, t)
    assert d_xyz.shape == (3, xyz.shape[0], 3)
    pkg = gr.render_batch(cams, model, _pipe(), torch.tensor(BG, device="cuda"), 0.01 * d_xyz, 0.01 * d_rot,
                          0.01 * d_scale)
    pkg["render"].square().sum().backward()
    for i, p in enumerate(net.field.planes):
        assert p.grad is not None and torch.isfinite(p.grad).all() and p.grad.abs().sum() > 0, i


def test_refusals_on_the_device():
    f = _field(16, "default")
    x, t = _points("default", n=100), _times(1, n=100)[0]
    with pytest.raises(ValueError, match="grad"):
        f(x, t.clone().requires_grad_(True))
    with pytest.raises(ValueError, match="float32"):
        f(x.double(), t)
    with pytest.raises(ValueError):
        f(x, t[:50])
    with pytest.raises(ValueError, match="CUDA"):
        f(x.cpu(), t)
