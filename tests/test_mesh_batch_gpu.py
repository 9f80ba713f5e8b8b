"""Frame-batched mesh branch on the GPU: DPSR over a batch of point sets, marching cubes over a batch of grids with
one host wait, range-mode mesh rasterisation, and mesh_renderer_batch.  Every item of a batch is held to the
single-item call on that item: bit for bit where the computation is deterministic (marching cubes' vertices and
faces, the z-buffer, interpolation), within the stated rel_err where fp32 atomics sum in a varying order."""
import importlib
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import util
from oracle import meshrast_oracle as orc
from oracle.oracle import mesh_topology
from test_dpsr import _points, affine_close
from test_mc import field
from test_meshrast import _random_scene, clip_from_world

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------- DPSR
def _dpsr_case(G, n, b, sig, flip=None):
    V, N = zip(*[_points(n, 10 * G + k) for k in range(b)])
    V, N = torch.stack(V), torch.stack(N)
    if flip is not None:   # the same points as item 0 with flipped normals: the field at the origin changes sign
        V[flip], N[flip] = V[0], -N[0]
    gout = torch.randn(b, G, G, G, generator=torch.Generator().manual_seed(G)).cuda()
    return V.cuda(), N.cuda(), gout


@pytest.mark.parametrize("G,n,b", [(32, 3000, 3), (64, 20000, 3), (288, 200_000, 2)])
def test_dpsr_batch_items_equal_single_calls(G, n, b):
    from nvdiffrast_utils.dpsr import DPSR
    m = DPSR(res=(G, G, G), sig=3.0)
    V, N, gout = _dpsr_case(G, n, b, 3.0, flip=1 if b == 3 else None)
    for signed in (False, True):
        th = torch.tensor(0.05, device="cuda", requires_grad=True)
        Va, Na = V.clone().requires_grad_(True), N.clone().requires_grad_(True)
        out = m.forward_signed(Va, Na, th) if signed else m(Va, Na)
        assert out.shape == (b, G, G, G)
        (out * gout).sum().backward()
        dth = 0.0
        for k in range(b):
            tk = torch.tensor(0.05, device="cuda", requires_grad=True)
            Vk, Nk = V[k:k + 1].clone().requires_grad_(True), N[k:k + 1].clone().requires_grad_(True)
            ok = m.forward_signed(Vk, Nk, tk)[None] if signed else m(Vk, Nk)
            (ok[0] * gout[k]).sum().backward()
            # bounds ~4x the maxima of three runs on an H100 (DESIGN.md): field 4.7e-6, dV 4.1e-5, dN 1.4e-5, all at
            # G = 288; the fields and gradients are sums of fp32 atomics, whose order varies from run to run
            assert util.rel_err(out[k].detach(), ok[0].detach()) < 2e-5, (signed, k, "field")
            assert util.rel_err(Va.grad[k], Vk.grad[0]) < 2e-4, (signed, k, "dV")
            assert util.rel_err(Na.grad[k], Nk.grad[0]) < 2e-4, (signed, k, "dN")
            if signed:
                dth += float(tk.grad)
        if signed:
            assert abs(float(th.grad) - dth) <= 1e-6 * max(1.0, abs(dth)), (float(th.grad), dth)   # measured 5.3e-8
            if b == 3:   # item 1's normals are flipped: its field has the opposite sign at the origin node
                raw = m(V, N).detach()
                assert float(raw[0, 0, 0, 0]) * float(raw[1, 0, 0, 0]) < 0


def test_dpsr_batch_matches_reference_batch():
    """The batch against the reference's DPSR with test_cuda_dpsr_matches_reference's bounds.  Where oracle/_ref is
    built that is the reference's own module, called ONCE on the whole [b,nv,3] batch (item 1 the flipped-normals
    copy of item 0): it normalises every item by itself, and so does the batch.  Elsewhere it is the restatement
    tests/ref_dpsr.py, which takes one item per call."""
    from nvdiffrast_utils.dpsr import DPSR
    ref = util.load_reference_dpsr()
    whole = getattr(ref.dpsr, "__name__", "") != "ref_dpsr"
    G, n, b = 32, 3000, 3
    V, N, gout = _dpsr_case(G, n, b, 3.0, flip=1)
    Va, Na = V.clone().requires_grad_(True), N.clone().requires_grad_(True)
    phi = DPSR(res=(G, G, G), sig=3.0)(Va, Na)
    (phi * gout).sum().backward()
    spans = [(0, b)] if whole else [(k, k + 1) for k in range(b)]
    phi_ref, dV_ref, dN_ref = [], [], []
    for lo, hi in spans:
        Vb, Nb = V[lo:hi].clone().requires_grad_(True), N[lo:hi].clone().requires_grad_(True)
        p = ref.dpsr.DPSR(res=(G, G, G), sig=3.0).cuda()(Vb, Nb)
        (p * gout[lo:hi]).sum().backward()
        phi_ref.append(p.detach())
        dV_ref.append(Vb.grad)
        dN_ref.append(Nb.grad)
    phi_ref, dV_ref, dN_ref = torch.cat(phi_ref), torch.cat(dV_ref), torch.cat(dN_ref)
    for k in range(b):
        ok, info = affine_close(phi[k].detach(), phi_ref[k])
        assert ok, (k, info)
        assert util.rel_err(phi[k], phi_ref[k]) < 5e-3
        ok, info = affine_close(Na.grad[k], dN_ref[k], resid_tol=2e-3, scale_tol=1e-2)
        assert ok, (k, "dN", info)
        ok, info = affine_close(Va.grad[k], dV_ref[k], resid_tol=2e-3, scale_tol=1e-2)
        assert ok, (k, "dV", info)


def test_dpsr_batch_workspace_grows_by_one_field_per_item():
    import ctypes

    import _dgm_lib
    from nvdiffrast_utils.dpsr import _plan
    for G in (32, 288):
        plan, single = _plan(G)
        sizes = []
        for B in (1, 2, 3, 64):
            n = _dgm_lib.c_size_t()
            assert _dgm_lib.lib().dgp_batch_workspace_size(plan, B, ctypes.byref(n)) == 0
            sizes.append(n.value)
        assert sizes[0] == single
        for B, s in zip((2, 3, 64), sizes[1:]):
            assert s - single >= 4 * G ** 3 * (B - 1) and s - single < 4 * G ** 3 * (B - 1) + 4096 * B


# ---------------------------------------------------------------------------------------------- marching cubes
def _grids(G):
    empty = np.ones((G, G, G), np.float32)                       # no crossing at all
    return torch.from_numpy(np.stack([field(G, "sphere"), field(G, "torus"), field(G, "noise"), empty])).cuda()


def _count_waits(monkeypatch):
    import _dgm_lib
    lib = _dgm_lib.lib()
    real, calls = lib.dgm_notify_wait, []

    def wait(h):
        calls.append(1)
        return real(h)
    monkeypatch.setattr(lib, "dgm_notify_wait", wait)
    return calls


@pytest.mark.parametrize("G,items", [(32, (0, 1, 2, 3)), (288, (0, 2))])
def test_marching_cubes_batch_items_equal_single_calls(G, items, monkeypatch):
    import diso
    from diso import DiffMC
    mc = DiffMC()
    grids = _grids(G)[list(items)].contiguous()
    diso._caps.clear()
    waits = _count_waits(monkeypatch)
    g = grids.clone().requires_grad_(True)
    vl, fl = mc.forward_batch(g)
    assert len(waits) == 1, "one host wait per forward_batch"
    # a second call reuses the capacities; a first call with too small ones re-emits: both give the same result
    vl2, fl2 = mc.forward_batch(grids)
    for key in list(diso._caps):
        diso._caps[key] = [16, 16]
    vl3, fl3 = mc.forward_batch(grids)
    assert len(waits) == 3
    v0 = 0
    for k in range(len(items)):
        vs, fs = mc(grids[k].clone())
        assert torch.equal(vl[k], vs) and torch.equal(fl[k], fs), k
        assert torch.equal(vl2[k], vs) and torch.equal(fl3[k], fs) and torch.equal(vl3[k], vs), k
        assert fl[k].dtype == torch.int64
        if items[k] == 3:
            assert vl[k].shape == (0, 3) and fl[k].shape == (0, 3)
        if vs.shape[0]:                                              # views of one concatenated tensor
            assert vl[k].data_ptr() == vl[0].data_ptr() + 12 * v0
        v0 += vs.shape[0]
    # the per-vertex edge records of the batch are the single calls' (through the backward: one-hot dL/dverts)
    w = [torch.randn(v.shape, generator=torch.Generator().manual_seed(k)).cuda() for k, v in enumerate(vl)]
    sum((v * wk).sum() for v, wk in zip(vl, w)).backward()
    for k in range(len(items)):
        gk = grids[k].clone().requires_grad_(True)
        vs, _ = mc(gk)
        (vs * w[k]).sum().backward()
        assert util.rel_err(g.grad[k], gk.grad) < 1e-6, k


def test_marching_cubes_batch_vsrc_equals_single():
    import ctypes

    import _dgm_lib
    lib, G = _dgm_lib.lib(), 32
    grids = _grids(G)
    B = grids.shape[0]
    st = _dgm_lib.stream_ptr()

    def run(b, phi):
        n = _dgm_lib.c_size_t()
        assert lib.dgmc_workspace_size_batch(b, G, ctypes.byref(n)) == 0
        ws = torch.empty(n.value, dtype=torch.uint8, device="cuda")
        tot = torch.empty(2 * b, dtype=torch.int32, device="cuda")
        assert lib.dgmc_count_batch(b, G, phi.data_ptr(), 0.0, ws.data_ptr(), n.value, tot.data_ptr(), None, None,
                                    st) == 0
        t = tot.view(b, 2).cpu()
        V, F = int(t[:, 0].sum()), int(t[:, 1].sum())
        v = torch.empty(V, 3, device="cuda")
        src = torch.empty(V, dtype=torch.int32, device="cuda")
        f = torch.empty(F, 3, dtype=torch.int32, device="cuda")
        assert lib.dgmc_emit_batch(b, G, phi.data_ptr(), 0.0, ws.data_ptr(), n.value, v.data_ptr(), src.data_ptr(),
                                   V, f.data_ptr(), F, st) == 0
        return t, v, src, f
    t, v, src, f = run(B, grids)
    v0 = f0 = 0
    for k in range(B):
        tk, vk, sk, fk = run(1, grids[k].contiguous())
        assert torch.equal(t[k], tk[0])
        nv, nf = int(tk[0, 0]), int(tk[0, 1])
        assert torch.equal(v[v0:v0 + nv], vk) and torch.equal(src[v0:v0 + nv], sk) and torch.equal(f[f0:f0 + nf], fk)
        v0, f0 = v0 + nv, f0 + nf


# ------------------------------------------------------------------------------------------ range-mode raster
def _meshes(W, H):
    parts = [_random_scene(seed, W, H) for seed in (0, 1, 2)]
    verts = torch.cat([p[0] for p in parts])
    offs = np.cumsum([0] + [p[0].shape[0] for p in parts])
    tri = torch.cat([p[1] + int(o) for p, o in zip(parts, offs)]).int()
    attr = torch.cat([p[2] for p in parts])
    nf = [p[1].shape[0] for p in parts]
    # image 2 draws nothing: an empty range
    ranges = torch.tensor([[0, nf[0]], [nf[0], nf[1]], [0, 0], [nf[0] + nf[1], nf[2]]], dtype=torch.int32)
    return parts, verts, tri, attr, ranges, offs


@pytest.mark.parametrize("W,H", [(64, 48), (800, 800)])
def test_range_mode_equals_single_image_calls(W, H):
    import nvdiffrast.torch as dr
    parts, verts, tri, attr, ranges, offs = _meshes(W, H)
    B = ranges.shape[0]
    wimg = torch.randn(B, H, W, 3, generator=torch.Generator().manual_seed(7)).cuda()
    wrast = torch.randn(B, H, W, 4, generator=torch.Generator().manual_seed(8)).cuda()
    vb = verts.cuda().requires_grad_(True)
    ab = attr.cuda().requires_grad_(True)
    pos = clip_from_world(vb, W, H)
    rast, _ = dr.rasterize(None, pos, tri.cuda(), resolution=[H, W], ranges=ranges)
    assert rast.shape == (B, H, W, 4)
    col, _ = dr.interpolate(ab[None], rast, tri.cuda())
    col = col.detach().requires_grad_(True)
    out = dr.antialias(col, rast, pos, tri.cuda())
    ((out * wimg).sum() + (rast * wrast).sum()).backward()
    col_b = col.grad
    gv = vb.grad.clone()
    # interpolate's attribute gradient, on its own
    ab2 = attr.cuda().requires_grad_(True)
    c2, _ = dr.interpolate(ab2[None], rast.detach(), tri.cuda())
    (c2 * wimg).sum().backward()
    assert torch.equal(rast[2], torch.zeros_like(rast[2]))
    part_of = [0, 1, None, 2]
    gv_single = torch.zeros_like(gv)
    ga_single = torch.zeros_like(ab2.grad)
    for b in range(B):
        k = part_of[b]
        if k is None:
            continue
        v, t, a = parts[k]
        o = int(offs[k])
        vs = v.cuda().requires_grad_(True)
        ps = clip_from_world(vs, W, H)
        rs, _ = dr.rasterize(None, ps[None], t.cuda(), resolution=[H, W])
        expect = rs[0].detach().clone()
        hit = expect[..., 3] > 0
        expect[..., 3][hit] += float(ranges[b, 0])
        assert torch.equal(rast[b].detach(), expect), b
        asg = a.cuda().requires_grad_(True)
        cs, _ = dr.interpolate(asg[None], rs.detach(), t.cuda())
        assert torch.equal(cs[0], c2[b].detach()), b
        (cs[0] * wimg[b]).sum().backward()
        ga_single[o:o + v.shape[0]] += asg.grad
        cs = cs.detach().requires_grad_(True)
        os_ = dr.antialias(cs, rs, ps[None], t.cuda())
        assert util.rel_err(os_[0], out[b].detach()) < 1e-6, b
        ((os_[0] * wimg[b]).sum() + (rs[0] * wrast[b]).sum()).backward()
        assert util.rel_err(col_b[b], cs.grad[0]) < 1e-6, b
        gv_single[o:o + v.shape[0]] += vs.grad
        if W == 64:     # the float64 restatement, per range
            vo = v.double()
            po = clip_from_world(vo, W, H)
            ids = orc.rasterize_ids(po, t, H, W)
            ro = orc.rast_from_ids(po, t.long(), ids)
            glob = torch.where(ids >= 0, ids + int(ranges[b, 0]), ids)
            assert torch.equal(rast[b, ..., 3].long().cpu() - 1, glob), b
            assert util.rel_err(rast[b, ..., :3], ro[..., :3]) < 1e-4
            co = orc.interpolate(a.double(), ro, t.long())
            oo = orc.antialias(co, ro, po, t.long(), orc.edge_opposites(t, v.shape[0]))
            assert util.rel_err(out[b], oo) < 1e-4
    if W == 64:
        _range_mode_gradients_match_float64_restatement(parts, verts, tri, attr, ranges, offs, wimg)
    # at 800x800 a vertex's gradient sums thousands of per-pixel terms of both signs with fp32 atomics, whose order
    # differs between the batch and the single calls (measured on an H100: 8.3e-6)
    tol = 1e-6 if W * H < 10_000 else 2e-5
    assert util.rel_err(gv, gv_single) < tol
    assert util.rel_err(ab2.grad, ga_single) < tol


def _range_mode_gradients_match_float64_restatement(parts, verts, tri, attr, ranges, offs, wimg):
    """dL/dattr and dL/dpos of one range-mode pass (interpolate -> antialias) against float64 autograd through
    the restatement applied per range, with test_meshrast.py's bounds"""
    import nvdiffrast.torch as dr
    H, W = wimg.shape[1], wimg.shape[2]
    vb = verts.cuda().requires_grad_(True)
    ab = attr.cuda().requires_grad_(True)
    pos = clip_from_world(vb, W, H)
    rast, _ = dr.rasterize(None, pos, tri.cuda(), resolution=[H, W], ranges=ranges)
    col, _ = dr.interpolate(ab[None], rast, tri.cuda())
    (dr.antialias(col, rast, pos, tri.cuda()) * wimg).sum().backward()
    for b, k in ((0, 0), (1, 1), (3, 2)):
        v, t, a = parts[k]
        o, n = int(offs[k]), v.shape[0]
        vo, ao = v.double().requires_grad_(True), a.double().requires_grad_(True)
        po = clip_from_world(vo, W, H)
        ids = orc.rasterize_ids(po.detach(), t, H, W)
        ro = orc.rast_from_ids(po, t.long(), ids)
        co = orc.interpolate(ao, ro, t.long())
        (orc.antialias(co, ro, po, t.long(), orc.edge_opposites(t, n)) * wimg[b].cpu().double()).sum().backward()
        assert util.rel_err(ab.grad[o:o + n], ao.grad) < 1e-4, (b, "d/d attr")
        assert util.rel_err(vb.grad[o:o + n], vo.grad) < 2e-3, (b, "d/d vertex positions")


def _decode_ids(w):
    """triangle id + 1 from rast.w (nvdiffrast's encoding: a float up to 2^24, bit pattern 0x4a800000 + id above)"""
    w = w.contiguous()
    return torch.where(w > 16777216.0, w.view(torch.int32).long() - 0x4a800000, w.long())


def test_range_mode_triangle_ids_past_2_24():
    """A range that starts past triangle 2^24, where a float no longer holds every integer: the ids come back
    exactly, and interpolate, antialias and their gradients read the right triangles, as the single-image call on
    the same triangles does."""
    import nvdiffrast.torch as dr
    W, H = 64, 48
    v, t, a = _random_scene(0, W, H)
    n = t.shape[0]
    first = (1 << 24) + 12345
    tri = torch.zeros(first + n + 7, 3, dtype=torch.int32, device="cuda")
    tri[first:first + n] = t.cuda()
    opp_small = dr.edge_opposites(t.cuda(), v.shape[0])
    opp = torch.full_like(tri, -1)
    opp[first:first + n] = opp_small
    ranges = torch.tensor([[first, n], [0, 0]], dtype=torch.int32)
    wimg = torch.randn(H, W, 3, generator=torch.Generator().manual_seed(5)).cuda()
    res = []
    for big in (True, False):
        vs, asg = v.cuda().requires_grad_(True), a.cuda().requires_grad_(True)
        ps = clip_from_world(vs, W, H)
        if big:
            rast, _ = dr.rasterize(None, ps, tri, resolution=[H, W], ranges=ranges)
            col, _ = dr.interpolate(asg[None], rast, tri)
            out = dr.antialias(col, rast, ps, tri, topology_hash=opp)
            assert torch.equal(rast[1], torch.zeros_like(rast[1]))
        else:
            rast, _ = dr.rasterize(None, ps[None], t.cuda(), resolution=[H, W])
            col, _ = dr.interpolate(asg[None], rast, t.cuda())
            out = dr.antialias(col, rast, ps[None], t.cuda(), topology_hash=opp_small)
        (out[0] * wimg).sum().backward()
        res.append((rast[0].detach(), col[0].detach(), out[0].detach(), vs.grad, asg.grad))
    (rb, cb, ob, gvb, gab), (rs, cs, os_, gvs, gas) = res
    ids_b, ids_s = _decode_ids(rb[..., 3]), _decode_ids(rs[..., 3])
    assert int(ids_s.max()) > 0 and int(ids_b.max()) > (1 << 24)
    assert torch.equal(ids_b, torch.where(ids_s > 0, ids_s + first, ids_s))
    assert torch.equal(rb[..., :3], rs[..., :3]) and torch.equal(cb, cs)
    assert util.rel_err(ob, os_) < 1e-6
    assert util.rel_err(gab, gas) < 1e-6 and util.rel_err(gvb, gvs) < 1e-6


def test_range_mode_refuses_instanced_pos():
    import nvdiffrast.torch as dr
    _, verts, tri, _, ranges, _ = _meshes(32, 32)
    pos = clip_from_world(verts.cuda(), 32, 32)
    with pytest.raises(ValueError):
        dr.rasterize(None, torch.stack([pos, pos]), tri.cuda(), resolution=[32, 32])
    with pytest.raises(ValueError):
        dr.rasterize(None, pos[None], tri.cuda(), resolution=[32, 32], ranges=ranges)


# ------------------------------------------------------------------------------------------------------ branch
def _camera(theta, H, W):
    """a camera on a circle of radius 3 around the origin, looking at it (blender / OpenGL pose)"""
    c = np.array([3 * math.sin(theta), 0.3, 3 * math.cos(theta)], np.float32)
    z = c / np.linalg.norm(c)
    x = np.cross([0, 1, 0], z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    T = np.eye(4, dtype=np.float32)
    T[:3, 0], T[:3, 1], T[:3, 2], T[:3, 3] = x, y, z, c
    return SimpleNamespace(K=None, FoVx=0.8, FoVy=0.8, image_width=W, image_height=H, orig_transform=T)


def test_mesh_renderer_batch_per_stage_and_gradients():
    from diso import DiffMC
    from nvdiffrast_utils.dpsr import DPSR
    tu = importlib.import_module("utils.time_utils")
    renderer = importlib.import_module("utils.renderer")
    torch.manual_seed(0)
    n, G, R, F, H, W = 60_000, 96, 0.6, 4, 200, 200
    d = torch.nn.functional.normalize(torch.randn(n, 3), dim=1).cuda()
    xyz = (d * R).requires_grad_(True)
    normal = d.clone().requires_grad_(True)
    thres = torch.nn.Parameter(torch.tensor(0.0, device="cuda"))
    gauss = SimpleNamespace(get_xyz=xyz, get_normal=normal, gaussian_center=torch.zeros(3, device="cuda"),
                            gaussian_scale=torch.tensor([1.0], device="cuda"), density_thres_param=thres,
                            dpsr=DPSR(res=(G, G, G), sig=2.0), diffmc=DiffMC(dtype=torch.float32).cuda())
    back = SimpleNamespace(net=tu.DeformNetworkNormal(is_blender=True).cuda())
    back.step = lambda x, t: back.net(x, t)
    app = SimpleNamespace(net=tu.AppearanceNetwork(is_blender=True).cuda())
    app.step = lambda x, t: app.net(x, t)
    shift = torch.tensor([[0.0, 0, 0], [0.05, 0, 0], [0, -0.05, 0], [0, 0, 0.04]], device="cuda")
    d_xyz = shift[:, None, :].expand(F, n, 3)
    fids = torch.tensor([[0.1], [0.3], [0.5], [0.7]], device="cuda")
    cams = [_camera(0.4 * k, H, W) for k in range(F)]
    masks, images, verts, faces, vcol = renderer.mesh_renderer_batch(None, gauss, d_xyz, 0.0, fids, back, app,
                                                                     viewpoint_cams=cams)
    assert masks.shape == (F, H, W, 1) and images.shape == (F, 3, H, W) and len(verts) == F
    for k in range(F):
        euler, manifold, oriented = mesh_topology(verts[k].detach().cpu().numpy(), faces[k].cpu().numpy())
        assert euler == 2 and manifold and oriented, k
        r = (verts[k].detach() - shift[k]).norm(dim=1)
        assert abs(float(r.mean()) - R) < 0.03 and float(r.std()) < 0.02, k
        assert faces[k].dtype == torch.int32
        # mesh_renderer's own downstream stages on the batch's frame-k mesh
        with torch.no_grad():
            vk, fk = verts[k].detach(), faces[k]
            t = fids[k].unsqueeze(0).expand(vk.shape[0], -1)
            dx, _, _, _ = back.step(vk, t)
            ck = app.step(vk + dx, t)
            assert util.rel_err(vcol[k], ck) < 1e-5, k
            pose, K, res = renderer._camera(cams[k])
            clip, rast, topo = renderer._raster(None, vk, fk, pose, K, res)
            m3 = renderer._mask_from(rast, clip, vk, fk, topo)
            img = renderer._image_from(rast, clip, fk, ck, m3, False, topo)
            assert m3.shape == (1, H, W, 3) and img.shape == (1, 3, H, W)
            assert util.rel_err(masks[k], m3[0][..., [0]]) < 1e-5, k
            assert util.rel_err(images[k], img[0]) < 1e-5, k
        assert float(masks[k].sum()) > 100, k
    lap = sum(_laplacian(v, f) for v, f in zip(verts, faces))
    (masks.mean() + images.mean() + lap).backward()
    for name, p in (("xyz", xyz), ("normal", normal), ("thres", thres),
                    ("appearance", app.net.linear[0].weight), ("deform_back", back.net.gaussian_warp.weight)):
        assert p.grad is not None and torch.isfinite(p.grad).all() and float(p.grad.abs().sum()) > 0, name


def _laplacian(v, f):
    """a uniform Laplacian smoothness term (mean squared offset from the neighbours' mean)"""
    e = torch.cat([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]).long()
    s = torch.zeros_like(v).index_add_(0, e[:, 0], v[e[:, 1]])
    c = torch.zeros(v.shape[0], 1, device=v.device).index_add_(0, e[:, 0], torch.ones(e.shape[0], 1, device=v.device))
    return ((v - s / c.clamp_min(1)) ** 2).sum(1).mean()


def test_extract_mesh_batch_accepts_render_batch_deltas():
    from diso import DiffMC
    from nvdiffrast_utils.dpsr import DPSR
    renderer = importlib.import_module("utils.renderer")
    torch.manual_seed(1)
    n, G = 20_000, 48
    d = torch.nn.functional.normalize(torch.randn(n, 3), dim=1).cuda()
    gauss = SimpleNamespace(get_xyz=d * 0.5, get_normal=d.clone(), gaussian_center=torch.zeros(3, device="cuda"),
                            gaussian_scale=torch.tensor([1.0], device="cuda"),
                            density_thres_param=torch.tensor(0.0, device="cuda"),
                            dpsr=DPSR(res=(G, G, G), sig=2.0), diffmc=DiffMC())
    shared = torch.full((n, 3), 0.02, device="cuda")
    a = renderer.extract_mesh_batch(gauss, [shared, shared, 0.0], 0.0)
    b = renderer.extract_mesh_batch(gauss, shared, 0.0, frames=3)
    c = renderer.extract_mesh_batch(gauss, torch.stack([shared, shared, torch.zeros_like(shared)]), [0.0] * 3)
    assert len(a[0]) == len(b[0]) == len(c[0]) == 3
    for mesh in (a, b, c):
        for k in range(3):
            assert mesh[0][k].shape[0] > 100 and mesh[1][k].shape[0] > 100
            assert int(mesh[1][k].max()) < mesh[0][k].shape[0]      # indices local to the frame


def test_mesh_renderer_batch_synchronises_only_for_the_mesh_sizes():
    """Besides the marching-cubes wait (which torch does not see), the batched branch's forward makes no
    synchronising call: the per-vertex frame index and the F clip matrices are uploaded without blocking.  The
    networks here are plain element-wise functions, so that only the branch itself is observed."""
    from diso import DiffMC
    from nvdiffrast_utils.dpsr import DPSR
    renderer = importlib.import_module("utils.renderer")
    torch.manual_seed(2)
    n, G, F, H, W = 20_000, 48, 3, 64, 64
    d = torch.nn.functional.normalize(torch.randn(n, 3), dim=1).cuda()
    gauss = SimpleNamespace(get_xyz=d * 0.5, get_normal=d.clone(), gaussian_center=torch.zeros(3, device="cuda"),
                            gaussian_scale=torch.tensor([1.0], device="cuda"),
                            density_thres_param=torch.tensor(0.0, device="cuda"),
                            dpsr=DPSR(res=(G, G, G), sig=2.0), diffmc=DiffMC())
    back = SimpleNamespace(step=lambda x, t: (0.01 * x * t, None, None, None))
    app = SimpleNamespace(step=lambda x, t: torch.sigmoid(x + t))
    fids = torch.tensor([[0.1], [0.4], [0.7]], device="cuda")
    cams = [_camera(0.5 * k, H, W) for k in range(F)]
    args = (None, gauss, 0.0, 0.0, fids, back, app)
    renderer.mesh_renderer_batch(*args, viewpoint_cams=cams)          # warm-up: pinned buffers, plans, modules
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        masks, images, verts, _, _ = renderer.mesh_renderer_batch(*args, viewpoint_cams=cams)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert masks.shape == (F, H, W, 1) and len(verts) == F
