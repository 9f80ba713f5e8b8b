"""Dual marching cubes on the GPU against the exact reference (tests/dmc_reference.py).

The forward must equal the reference bit for bit: the same multiset of fp32 vertices, of oriented triangles and of
oriented quads (4-cycles), the same V, F and Q.  The backward must be within 1e-5 of the reference's sum of
|contributions| at every node, and bit-identical from run to run.  A batch item must equal the single call on it
bit for bit.  The mesh branch must run end to end with DiffDMC as its extractor."""
import importlib
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from dmc_reference import assert_same_quads, dmc_reference, grad_reference
from mc_reference import LOSS_P, LOSS_W, assert_same_mesh, loss_grad
from test_dmc_cpu import torus
from test_mc_reference import noise, quantised_sphere, seam_field, smooth_noise, sphere

pytestmark = pytest.mark.gpu


def _run(phi, iso=0.0, normalize=True, grad=True):
    """DiffDMC on phi -> (verts, faces, quads, dL/dphi of L = sum_v h(v) or None)."""
    from diso import DiffDMC
    m = DiffDMC(dtype=torch.float32)
    p = torch.from_numpy(np.ascontiguousarray(phi)).cuda().requires_grad_(grad)
    v, f = m(p, deform=None, isovalue=iso, normalize=normalize)
    assert v.dtype == torch.float32 and f.dtype == torch.int64 and f.shape[1:] == (3,)
    with torch.no_grad():
        v2, q = m(p.detach(), isovalue=iso, return_quads=True, normalize=normalize)
    assert q.dtype == torch.int64 and q.shape == (f.shape[0] // 2, 4)
    assert torch.equal(v, v2)
    dphi = None
    if grad:
        w, ph = torch.tensor(LOSS_W, device="cuda"), torch.tensor(LOSS_P, device="cuda")
        torch.sin(v.double() * w + ph).sum().backward()
        dphi = p.grad.cpu().numpy()
    return v.detach().cpu().numpy(), f.cpu().numpy(), q.cpu().numpy(), dphi


def _assert_grad_close(dphi, g, absum, scale=1.0):
    assert np.isfinite(dphi).all()
    err = np.abs(dphi.astype(np.float64) * scale - g)
    bad = err > 1e-5 * absum
    assert not bad.any(), (f"{int(bad.sum())} of {bad.size} nodes off; worst |err| / sum|c| = "
                           f"{float((err / np.maximum(absum, 1e-300)).max()):.3g}")


def _check(phi, iso=0.0, normalize=True, grad=True):
    G = phi.shape[0]
    ref = dmc_reference(phi, iso)
    v, f, q, dphi = _run(phi, iso, normalize, grad)
    want = ref.verts if normalize else ref.verts * np.float32(G - 1)
    assert len(v) == len(ref.verts) and len(f) == len(ref.faces) and len(q) == len(ref.quads)
    assert_same_mesh(v, f, want, ref.faces)
    assert_same_quads(v, q, want, ref.quads)
    if grad:
        dv = loss_grad(want) * (1 if normalize else G - 1)
        _assert_grad_close(dphi, *grad_reference(ref, phi, dv))
    return ref, v, f


def test_cuda_dmc_all_256_cases_in_the_centre_cell():
    """G = 4: the centre cell (1, 1, 1) takes each case; the other nodes get values of the same sign as the
    nearest corner of that cell, so the centre cell's patches all reach interior edges."""
    rng = np.random.default_rng(0)
    for case in range(256):
        phi = np.empty((4, 4, 4), np.float32)
        for idx in np.ndindex(4, 4, 4):
            c = sum((min(max(x - 1, 0), 1)) << b for b, x in enumerate(idx))
            val = np.float32(rng.uniform(0.05, 1.0))
            phi[idx] = -val if (case >> c) & 1 else val
        _check(phi)


@pytest.mark.parametrize("G", [9, 33, 65])
@pytest.mark.parametrize("kind", ["smooth", "seams"])
def test_cuda_dmc_exact_at_brick_and_chunk_seams(G, kind):
    _check(smooth_noise(G, G) if kind == "smooth" else seam_field(G))


@pytest.mark.parametrize("iso", [0.1, -0.37])
def test_cuda_dmc_exact_at_isovalues(iso):
    _check(smooth_noise(40, 7), iso)


@pytest.mark.parametrize("iso", [0.0, 0.125])
def test_cuda_dmc_exact_with_values_on_the_isovalue(iso):
    phi = quantised_sphere(33)
    assert (phi == np.float32(iso)).sum() > 500
    _check(phi, iso)


def test_cuda_dmc_exact_without_normalisation():
    _check(smooth_noise(33, 5), 0.1, normalize=False)


@pytest.mark.parametrize("value", [1.0, -1.0])
def test_cuda_dmc_empty_surface(value):
    phi = np.full((17, 17, 17), value, np.float32)
    v, f, q, dphi = _run(phi)
    assert v.shape == (0, 3) and f.shape == (0, 3) and q.shape == (0, 4)
    assert dphi.shape == phi.shape and not dphi.any()


@pytest.mark.parametrize("G", [8, 16, 32])
def test_cuda_dmc_independent_noise(G):
    _check(noise(G, G))


def _dpsr_field(G, n=100_000):
    """The DPSR field of points on a sphere and a torus (the shape of DG-Mesh's training fields)."""
    from nvdiffrast_utils.dpsr import DPSR
    g = torch.Generator().manual_seed(3)
    d = torch.nn.functional.normalize(torch.randn(n // 2, 3, generator=g), dim=1)
    u, w = torch.rand(n // 2, generator=g) * 6.2832, torch.rand(n // 2, generator=g) * 6.2832
    c = torch.stack([torch.cos(u), torch.sin(u), torch.zeros_like(u)], 1)
    tn = torch.cos(w)[:, None] * c + torch.sin(w)[:, None] * torch.tensor([0.0, 0, 1])
    pts = torch.cat([d * 0.2 + 0.3, (0.25 * c + 0.08 * tn) * torch.tensor([1, 1, 1.0]) + 0.6])
    nrm = torch.cat([d, tn])
    with torch.no_grad():
        phi = DPSR(res=(G, G, G), sig=2.0)(pts[None].cuda().clamp(0.02, 0.98), nrm[None].cuda())
    return phi[0].float().cpu().numpy()


@pytest.mark.parametrize("kind", ["smooth", "dpsr"])
def test_cuda_dmc_exact_at_training_size(kind):
    G = 288
    phi = smooth_noise(G, 11) if kind == "smooth" else _dpsr_field(G)
    ref, _, _ = _check(phi)
    assert len(ref.verts) > 50_000


@pytest.mark.parametrize("s", [2.0 ** -70, 2.0 ** 70])
def test_cuda_dmc_is_invariant_to_power_of_two_scale(s):
    phi = sphere(33)
    sphi = (phi * np.float32(s)).astype(np.float32)
    assert np.array_equal(sphi / np.float32(s), phi) and np.isfinite(sphi).all()
    ref = dmc_reference(phi)
    v, f, q, _ = _run(phi, grad=False)
    vs, fs, qs, dphi = _run(sphi)
    assert np.array_equal(v.view(np.uint32), vs.view(np.uint32)) and np.array_equal(f, fs) and np.array_equal(q, qs)
    g, absum = grad_reference(ref, phi, loss_grad(ref.verts))
    _assert_grad_close(dphi, g, absum, scale=s)


def test_cuda_dmc_capacity_path_equals_fresh_calls():
    """Optimistic emission with the previous capacities, and re-emission when the surface outgrew them: each
    result equals a call made with no cached capacity, bit for bit and in the same order."""
    import diso
    G = 64
    fields = [sphere(G, 0.3), sphere(G, 0.8), sphere(G, 0.3), noise(G, 5)]
    diso._caps.clear()
    seq, caps = [], []
    for phi in fields:
        caps.append(diso._caps.get(("dmc", torch.cuda.current_device(), G)))
        ref, v, f = _check(phi, grad=False)
        seq.append((v, f, len(ref.verts)))
    V = [s[2] for s in seq]
    assert caps[0] is None and V[1] > caps[1][0] and V[2] <= caps[2][0] and V[3] > caps[3][0]
    for phi, (v, f, _) in zip(fields, seq):
        diso._caps.clear()
        v1, f1, _, _ = _run(phi, grad=False)
        assert np.array_equal(v.view(np.uint32), v1.view(np.uint32)) and np.array_equal(f, f1)


def test_cuda_dmc_forward_and_backward_are_deterministic():
    phi = smooth_noise(65, 3)
    a, b = _run(phi), _run(phi)
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))


@pytest.mark.parametrize("G,B", [(64, 3), (288, 8)])
def test_cuda_dmc_batch_items_equal_single_calls(G, B):
    from diso import DiffDMC
    m = DiffDMC()
    fields = [sphere(G, 0.3 + 0.05 * k) if k % 2 else smooth_noise(G, k) for k in range(B)]
    fields[1] = np.full((G, G, G), 1.0, np.float32)               # an empty item inside the batch
    grids = torch.from_numpy(np.stack(fields)).cuda().requires_grad_(True)
    vl, fl = m.forward_batch(grids)
    w, ph = torch.tensor(LOSS_W, device="cuda"), torch.tensor(LOSS_P, device="cuda")
    sum(torch.sin(v.double() * w + ph).sum() for v in vl).backward()
    for k in range(B):
        p = grids[k].detach().clone().requires_grad_(True)
        v, f = m(p)
        torch.sin(v.double() * w + ph).sum().backward()
        assert torch.equal(v.view(torch.int32), vl[k].view(torch.int32)) and torch.equal(f, fl[k]), k
        assert torch.equal(p.grad.view(torch.int32), grids.grad[k].view(torch.int32)), k


def _gauss(n, G, R):
    from diso import DiffDMC
    from nvdiffrast_utils.dpsr import DPSR
    tu = importlib.import_module("utils.time_utils")
    d = torch.nn.functional.normalize(torch.randn(n, 3), dim=1).cuda()
    xyz = (d * R).requires_grad_(True)
    normal = d.clone().requires_grad_(True)
    thres = torch.nn.Parameter(torch.tensor(0.0, device="cuda"))
    gauss = SimpleNamespace(get_xyz=xyz, get_normal=normal, gaussian_center=torch.zeros(3, device="cuda"),
                            gaussian_scale=torch.tensor([1.0], device="cuda"), density_thres_param=thres,
                            dpsr=DPSR(res=(G, G, G), sig=2.0), diffmc=DiffDMC(dtype=torch.float32).cuda())
    back = SimpleNamespace(net=tu.DeformNetworkNormal(is_blender=True).cuda())
    back.step = lambda x, t: back.net(x, t)
    app = SimpleNamespace(net=tu.AppearanceNetwork(is_blender=True).cuda())
    app.step = lambda x, t: app.net(x, t)
    return gauss, back, app, (xyz, normal, thres)


def test_mesh_renderer_with_dual_marching_cubes():
    from test_mesh_batch_gpu import _camera
    from nvdiffrast_utils.regularizer import laplace_regularizer_const
    renderer = importlib.import_module("utils.renderer")
    torch.manual_seed(0)
    n, G, R, F, H, W = 60_000, 96, 0.6, 4, 200, 200
    gauss, back, app, params = _gauss(n, G, R)
    # single frame
    mask, img, v, f, _ = renderer.mesh_renderer(None, gauss, 0.0, 0.0, torch.tensor([0.2], device="cuda"), back,
                                                app, viewpoint_cam=_camera(0.3, H, W))
    lap = laplace_regularizer_const(v, f)
    assert torch.isfinite(lap) and float(mask.sum()) > 100
    (mask.mean() + img.mean() + lap).backward()
    for name, p in zip(("xyz", "normal", "thres"), params):
        assert p.grad is not None and torch.isfinite(p.grad).all() and float(p.grad.abs().sum()) > 0, name
        p.grad = None
    # frame batch
    shift = torch.tensor([[0.0, 0, 0], [0.05, 0, 0], [0, -0.05, 0], [0, 0, 0.04]], device="cuda")
    d_xyz = shift[:, None, :].expand(F, n, 3)
    fids = torch.tensor([[0.1], [0.3], [0.5], [0.7]], device="cuda")
    cams = [_camera(0.4 * k, H, W) for k in range(F)]
    masks, images, verts, faces, _ = renderer.mesh_renderer_batch(None, gauss, d_xyz, 0.0, fids, back, app,
                                                                  viewpoint_cams=cams)
    for k in range(F):
        r = (verts[k].detach() - shift[k]).norm(dim=1)
        assert abs(float(r.mean()) - R) < 0.03, k
    (masks.mean() + images.mean()).backward()
    for name, p in zip(("xyz", "normal", "thres"), params):
        assert p.grad is not None and torch.isfinite(p.grad).all() and float(p.grad.abs().sum()) > 0, name


def test_torus_mesh_is_closed_on_the_gpu():
    v, f, _, _ = _run(torus(48), grad=False)
    d = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    assert np.array_equal(np.sort(d[:, 0] * len(v) + d[:, 1]), np.sort(d[:, 1] * len(v) + d[:, 0]))
