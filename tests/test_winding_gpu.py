"""Winding number, signed distance and volumetric IoU on the GPU (csrc/winding.cu, mesh_distance.winding_number /
signed_distance, mesh_metrics(iou_points=...)) against the float64 solid-angle sum of tests/winding_oracle.py.

* beta = inf: |w - w64| <= TOL_EXACT on every query farther than 1e-4 L from the surface (L the diagonal of the
  mesh's box; closer, fp32 cannot resolve the nearby faces' solid angles).
* beta = 2: |w - w64| <= TOL_BETA2 on the same queries, and on closed meshes |w| >= 0.5 agrees with the oracle's
  classification wherever the exact |w| is at least 0.05 away from 0.5.
* w is bit-identical from run to run, and whatever other points share the call (permuted or split).
* signed_distance: |sdf|, face and bary are point_mesh_distance's bit for bit, the gradients are its gradients
  with g' = sign g / (2 |sdf|), 0 on the surface, and descent moves points onto a sphere.
* IoU: 1 for a mesh against itself, 0 for disjoint boxes, V_inner / V_outer for nested icospheres."""
import math

import numpy as np
import pytest
import torch

import winding_oracle as wo

pytestmark = pytest.mark.gpu

# Every case prints its measured maxima.  On an H100 the worst were 2.5e-5 at beta = inf (one huge triangle beside
# tiny ones; 1.3e-6 elsewhere) and 2.7e-2 per layer of faces at beta = 2 (near-surface queries of closed meshes).
TOL_EXACT = 1e-4
TOL_BETA2 = 4e-2    # per layer: a mesh whose faces are all duplicated has twice the far-field error
NEAR = 1e-4         # queries within NEAR L of the surface are left out of the value checks
MARGIN = 0.05       # classification is checked where | |w64| - 0.5 | >= MARGIN


def _md():
    import mesh_distance
    return mesh_distance


def _diag(v):
    return float((v.double().max(0).values - v.double().min(0).values).norm())


def _near(v, f, Q, seed, spread=0.05):
    """Q queries: surface samples moved along their normal by up to spread L, and a tenth uniform in the box."""
    from mesh_metrics import sample_surface
    g = torch.Generator(device="cuda").manual_seed(seed)
    L = _diag(v)
    n_box = Q // 10
    p, _, nrm = sample_surface(v, f, Q - n_box, g)
    p = p + nrm * ((torch.rand(Q - n_box, 1, device="cuda", generator=g) * 2 - 1) * spread * L)
    lo, hi = v.min(0).values, v.max(0).values
    box = lo + (hi - lo) * torch.rand(n_box, 3, device="cuda", generator=g)
    return torch.cat([p, box]).float().contiguous()


def _check(name, p, v, f, closed, layers=1):
    """beta = inf and beta = 2 against the oracle (bounds times `layers`, the faces' multiplicity); returns the
    measured maxima."""
    md = _md()
    L = _diag(v)
    w_inf = md.winding_number(p, v, f, beta=math.inf)
    w_2 = md.winding_number(p, v, f)
    assert w_inf.dtype == torch.float32 and w_inf.shape == (p.shape[0],) and not w_inf.requires_grad
    assert bool(torch.isfinite(w_inf).all()) and bool(torch.isfinite(w_2).all())
    ref = wo.winding(p, v, f, device="cuda")
    d2, _, _ = md.point_mesh_distance(p, v, f)
    keep = (d2.sqrt() > NEAR * L).cpu().numpy()
    e_inf = float(np.abs(w_inf.cpu().numpy().astype(np.float64) - ref)[keep].max())
    e_2 = float(np.abs(w_2.cpu().numpy().astype(np.float64) - ref)[keep].max())
    msg = (f"{name}: Q={p.shape[0]} F={f.shape[0]} kept {int(keep.sum())}: |w - w64| beta=inf {e_inf:.2e}, "
           f"beta=2 {e_2:.2e}")
    if closed:
        sure = keep & (np.abs(np.abs(ref) - 0.5) >= MARGIN)
        inside = np.abs(ref) >= 0.5
        wrong = [int(((w.abs() >= 0.5).cpu().numpy() != inside)[sure].sum()) for w in (w_inf, w_2)]
        msg += f", {int(sure.sum())} classified, wrong (inf, 2) {wrong}, inside {int(inside.sum())}"
        assert wrong == [0, 0], wrong
    print(msg)
    assert e_inf <= layers * TOL_EXACT and e_2 <= layers * TOL_BETA2, (e_inf, e_2)
    return e_inf, e_2


# ---- meshes --------------------------------------------------------------------------------------------------------
def _cube():
    v = torch.tensor([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], dtype=torch.float32)
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    f = torch.tensor([t for a, b, c, d in quads for t in ((a, b, c), (a, c, d))], dtype=torch.int32)
    return v.cuda(), f.cuda()


def _ico(radius=1.0, faceting=1e-3):
    from test_metrics_gpu import _icosphere
    v, f = _icosphere(radius, faceting=faceting)
    return v, f.int()


def _soup(F, seed, size=0.1):
    g = torch.Generator().manual_seed(seed)
    a = torch.rand(F, 1, 3, generator=g)
    v = (a + (torch.rand(F, 3, 3, generator=g) - 0.5) * size).reshape(-1, 3)
    f = torch.arange(3 * F, dtype=torch.int32).reshape(F, 3)[torch.randperm(F, generator=g)]
    return v.cuda(), f.cuda()


def _diffmc(kind, G):
    """DiffMC mesh of a signed-distance field that is negative inside: a sphere or a torus, in [-0.9, 0.9]^3."""
    from diso import DiffMC
    x = torch.linspace(-1, 1, G, device="cuda")
    X, Y, Z = torch.meshgrid(x, x, x, indexing="ij")
    if kind == "sphere":
        phi = (X * X + Y * Y + Z * Z).sqrt() - 0.6
    elif kind == "torus":
        phi = (((X * X + Y * Y).sqrt() - 0.5) ** 2 + Z * Z).sqrt() - 0.2
    else:
        from test_meshrast_fp64 import _sdf_mesh
        v, f = _sdf_mesh(G)
        return v.cuda(), f.cuda()
    v, f = DiffMC().cuda()(phi, deform=None, isovalue=0.0)
    return ((v.detach() * 2 - 1) * 0.9).float().contiguous(), f.int().contiguous()


# ---- beta = inf and beta = 2 against the oracle ---------------------------------------------------------------------
def test_cube():
    v, f = _cube()
    p = (torch.rand(20_000, 3, generator=torch.Generator().manual_seed(0)) * 3 - 1).cuda()
    _check("cube", p, v, f, closed=True)
    w = _md().winding_number(torch.tensor([[0.5, 0.5, 0.5], [2.0, 0.5, 0.5]], device="cuda"), v, f, math.inf)
    assert abs(float(w[0]) - 1) < 1e-6 and abs(float(w[1])) < 1e-6
    w = _md().winding_number(torch.tensor([[0.5, 0.5, 0.5]], device="cuda"), v, f.flip(1).contiguous(), math.inf)
    assert abs(float(w[0]) + 1) < 1e-6


def test_icosphere():
    v, f = _ico()
    _check("icosphere", _near(v, f, 20_000, 1), v, f, closed=True)


@pytest.mark.parametrize("kind", ["sphere", "torus"])
def test_diffmc_meshes_at_64(kind):
    v, f = _diffmc(kind, 64)
    _check(f"diffmc {kind} G=64", _near(v, f, 20_000, 2), v, f, closed=True)


def test_diffmc_sphere_orientation():
    """DiffMC's triangles of a field negative inside are oriented so that w = +1 inside (counter-clockwise from
    outside); the inside test uses |w| and does not depend on it."""
    v, f = _diffmc("sphere", 64)
    w = _md().winding_number(torch.tensor([[0.0, 0.0, 0.0], [0.1, -0.2, 0.15]], device="cuda"), v, f, math.inf)
    vol = wo.polyhedron_volume(v, f)
    print(f"diffmc sphere: w at the centre {float(w[0]):+.6f}, signed volume {vol:+.4f}")
    assert abs(abs(float(w[0])) - 1) < 1e-5 and abs(abs(float(w[1])) - 1) < 1e-5
    assert (float(w[0]) > 0) == (vol > 0)


def test_open_random_soup():
    v, f = _soup(3000, 3)
    p = (torch.rand(10_000, 3, generator=torch.Generator().manual_seed(4)) * 1.2 - 0.1).cuda()
    _check("open soup", p, v, f, closed=False)


def test_duplicated_and_degenerate_faces():
    v, f = _ico(faceting=3e-3)
    n = f.shape[0]
    g = torch.Generator().manual_seed(5)
    a = torch.rand(300, 3, generator=g).cuda() * 2 - 1
    d = (torch.rand(300, 3, generator=g).cuda() - 0.5) * 0.2
    V0 = v.shape[0]
    v2 = torch.cat([v, a, a + d, a + 2.5 * d])
    i = torch.arange(300, device="cuda", dtype=torch.int32)
    collinear = torch.stack([V0 + i, V0 + 300 + i, V0 + 600 + i], 1)
    point = torch.stack([V0 + i] * 3, 1)
    f2 = torch.cat([f, f, collinear, point]).int()
    f2 = f2[torch.randperm(f2.shape[0], generator=g).cuda()].contiguous()
    p = _near(v, f, 10_000, 6)
    e = _check("duplicated + degenerate", p, v2, f2, closed=False, layers=2)
    w1 = _md().winding_number(p, v, f, math.inf)
    w2 = _md().winding_number(p, v2, f2, math.inf)
    d2, _, _ = _md().point_mesh_distance(p, v, f)
    keep = d2.sqrt() > NEAR * _diag(v)
    e2 = float((w2 - 2 * w1)[keep].abs().max())
    print(f"duplicated: |w(doubled) - 2 w| {e2:.2e} over {n} faces")
    assert e2 <= 2 * TOL_EXACT and e[0] <= 2 * TOL_EXACT


def test_huge_triangle_beside_tiny_ones_in_one_morton_cell():
    g = torch.Generator().manual_seed(14)
    n = 100_000
    c = torch.rand(n, 1, 3, generator=g, dtype=torch.float64) * 1e-6
    tiny = (c + torch.rand(n, 3, 3, generator=g, dtype=torch.float64) * 1e-7).reshape(-1, 3)
    huge = torch.tensor([[-10.0, -10.0, 0.0], [10.0, -10.0, 0.0], [0.0, 20.0, 0.0]], dtype=torch.float64)
    far = torch.tensor([[10.0, 10.0, 10.0], [10.0, 10.0, 10.0 + 1e-7], [10.0, 10.0 + 1e-7, 10.0]],
                       dtype=torch.float64)
    v = torch.cat([tiny, huge, far]).float().cuda()
    f = torch.arange(v.shape[0], dtype=torch.int32, device="cuda").reshape(-1, 3)
    f = f[torch.randperm(f.shape[0], generator=g).cuda()].contiguous()
    q = torch.rand(4000, 3, generator=g) * 4 - 2
    q[::4] = torch.rand(1000, 3, generator=g) * 4e-6 - 1e-6
    _check("huge beside tiny", q.cuda(), v, f, closed=False)


def test_queries_far_outside():
    v, f = _ico()
    g = torch.Generator().manual_seed(7)
    p = (torch.nn.functional.normalize(torch.randn(5000, 3, generator=g), dim=1) * 100 * _diag(v) + 0.3).cuda()
    _check("far queries", p, v, f, closed=True)


def test_diffmc_at_288_on_sampled_queries():
    v, f = _diffmc("sphere+torus", 288)
    assert f.shape[0] > 300_000
    p = _near(v, f, 200_000, 8)
    sel = torch.randperm(p.shape[0], generator=torch.Generator().manual_seed(9))[:2000].cuda()
    _check("diffmc G=288", p[sel].contiguous(), v, f, closed=True)
    # the sampled queries get the same bits inside the full call
    md = _md()
    for beta in (2.0, math.inf):
        assert torch.equal(md.winding_number(p, v, f, beta)[sel], md.winding_number(p[sel].contiguous(), v, f, beta))


# ---- determinism ---------------------------------------------------------------------------------------------------
def test_bit_identical_and_independent_of_the_other_queries():
    md = _md()
    v, f = _diffmc("sphere+torus", 288)
    p = _near(v, f, 200_000, 10)
    perm = torch.randperm(p.shape[0], generator=torch.Generator().manual_seed(11)).cuda()
    bits = lambda w: w.view(torch.int32)    # noqa: E731
    w = md.winding_number(p, v, f)
    assert torch.equal(bits(w), bits(md.winding_number(p, v, f)))
    assert torch.equal(bits(w[perm]), bits(md.winding_number(p[perm], v, f)))
    k = 70_001
    split = torch.cat([md.winding_number(p[:k], v, f), md.winding_number(p[k:], v, f)])
    assert torch.equal(bits(w), bits(split))
    v, f = _diffmc("torus", 64)
    p = _near(v, f, 20_000, 12)
    w = md.winding_number(p, v, f, math.inf)
    sub = perm[perm < 20_000]
    assert torch.equal(bits(w), bits(md.winding_number(p, v, f, math.inf)))
    assert torch.equal(bits(w[sub]), bits(md.winding_number(p[sub], v, f, math.inf)))


# ---- signed_distance -----------------------------------------------------------------------------------------------
def test_signed_distance_equals_point_mesh_distance_and_its_gradient():
    md = _md()
    v, f = _diffmc("sphere+torus", 288)
    p = _near(v, f, 200_000, 13)
    p = torch.cat([p, v[f[:100, 0].long()]]).contiguous()        # queries on vertices: dist2 = 0
    g = torch.randn(p.shape[0], generator=torch.Generator().manual_seed(14)).cuda()
    pp, vv = p.clone().requires_grad_(True), v.clone().requires_grad_(True)
    sdf, face, bary, w = md.signed_distance(pp, vv, f)
    assert sdf.requires_grad and not face.requires_grad and not bary.requires_grad and not w.requires_grad
    (sdf * g).sum().backward()
    qq, uu = p.clone().requires_grad_(True), v.clone().requires_grad_(True)
    d2, face2, bary2 = md.point_mesh_distance(qq, uu, f)
    assert torch.equal(sdf.detach().abs(), d2.detach().sqrt())
    assert torch.equal(face, face2) and torch.equal(bary, bary2)
    assert torch.equal(w, md.winding_number(p, v, f))
    inside = w.abs() >= 0.5
    assert torch.equal(sdf.detach() < 0, inside & (d2.detach() > 0))
    sign = torch.where(inside, -1.0, 1.0)
    dist = d2.detach().sqrt()
    g2 = torch.where(dist > 0, sign * g / (2 * dist), 0.0)
    (d2 * g2).sum().backward()
    assert torch.equal(pp.grad, qq.grad) and torch.equal(vv.grad, uu.grad)
    assert bool(torch.isfinite(pp.grad).all()) and bool(torch.isfinite(vv.grad).all())
    assert float(pp.grad[-100:].abs().max()) == 0.0
    print(f"signed distance: {int(inside.sum())} of {p.shape[0]} inside, |grad points| max "
          f"{float(pp.grad.abs().max()):.2e}")


def test_descent_moves_points_onto_a_sphere():
    md = _md()
    v, f = _ico(1.0, faceting=1e-4)
    g = torch.Generator().manual_seed(15)
    x = torch.nn.functional.normalize(torch.randn(4000, 3, generator=g), dim=1)
    x = (x * (torch.rand(4000, 1, generator=g) * 1.4 + 0.3)).cuda().requires_grad_(True)   # radii 0.3 .. 1.7
    first = None
    for _ in range(30):
        sdf, _, _, _ = md.signed_distance(x, v, f)
        if first is None:
            first = sdf.detach().clone()
        x.grad = None
        (0.5 * sdf.square()).sum().backward()
        with torch.no_grad():
            x -= 0.5 * x.grad
    sdf = md.signed_distance(x.detach(), v, f)[0]
    r = x.detach().norm(dim=1)
    print(f"descent: |sdf| {float(first.abs().max()):.3f} -> {float(sdf.abs().max()):.2e}, "
          f"radius {float(r.min()):.6f} .. {float(r.max()):.6f}, inside at start {int((first < 0).sum())}")
    assert int((first < 0).sum()) > 1000 and int((first > 0).sum()) > 1000
    assert float(sdf.abs().max()) < 1e-5 and float((r - 1).abs().max()) < 1e-3


def test_value_errors():
    md = _md()
    v, f = _cube()
    p = torch.rand(10, 3, device="cuda")
    for fn in (md.winding_number, md.signed_distance):
        for args in [(p.cpu(), v, f), (p, v.cpu(), f), (p[:, :2], v, f), (p.double(), v, f), (p, v, f[:0]),
                     (p, v, torch.cat([f, torch.tensor([[0, 1, 8]], dtype=torch.int32, device="cuda")]))]:
            with pytest.raises(ValueError):
                fn(*args)
        for beta in (0.0, -2.0, math.nan):
            with pytest.raises(ValueError):
                fn(p, v, f, beta)
    assert md.winding_number(p[:0], v, f).shape == (0,)
    sdf, face, bary, w = md.signed_distance(p[:0], v, f)
    assert sdf.shape == (0,) and face.shape == (0,) and bary.shape == (0, 3) and w.shape == (0,)
    assert torch.equal(md.winding_number(p, v, f.long()), md.winding_number(p, v, f))


# ---- mesh_metrics IoU ----------------------------------------------------------------------------------------------
def test_iou_of_a_mesh_against_itself_is_one():
    from mesh_metrics import mesh_metrics
    m = _ico()
    r = mesh_metrics(m, m, 10_000, generator=torch.Generator(device="cuda").manual_seed(1), iou_points=100_000)
    assert r["iou"] == 1.0


def test_iou_of_disjoint_meshes_is_zero():
    from mesh_metrics import mesh_metrics
    v, f = _ico()
    r = mesh_metrics((v, f), (v + 3.0, f), 10_000, generator=torch.Generator(device="cuda").manual_seed(2),
                     iou_points=100_000)
    assert r["iou"] == 0.0


def test_iou_of_nested_icospheres():
    from mesh_metrics import mesh_metrics
    a, b = _ico(1.0, 1e-4), _ico(1.05, 1e-4)
    expect = wo.polyhedron_volume(*a) / wo.polyhedron_volume(*b)
    n = 100_000
    r = mesh_metrics(a, b, 10_000, generator=torch.Generator(device="cuda").manual_seed(3), iou_points=n)
    frac = wo.polyhedron_volume(*b) / 2.1 ** 3            # the share of the box inside the outer sphere
    se = math.sqrt(expect * (1 - expect) / (n * frac))
    print(f"nested icospheres: iou {r['iou']:.5f}, V_inner / V_outer {expect:.5f}, standard error {se:.1e}")
    assert abs(r["iou"] - expect) <= 4 * se


def test_iou_leaves_every_other_metric_unchanged():
    from mesh_metrics import mesh_metrics
    a, b = _ico(1.0), _diffmc("sphere", 64)
    for surface in (False, True):
        kw = dict(thresholds=(0.05,), surface=surface)
        r0 = mesh_metrics(a, b, 20_000, generator=torch.Generator(device="cuda").manual_seed(4), **kw)
        r1 = mesh_metrics(a, b, 20_000, generator=torch.Generator(device="cuda").manual_seed(4), iou_points=50_000,
                          **kw)
        assert "iou" not in r0 and 0.0 < r1.pop("iou") < 1.0
        assert r0 == r1
