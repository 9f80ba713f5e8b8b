"""Differentiable triangle-mesh rasterisation on the GPU (SURVEY.md 8(f)-1), with the call surface of the
three nvdiffrast primitives dgmesh/utils/renderer.py:33-121 uses, so that render_mask / render_mesh read
exactly like the reference:

    rast, _ = rasterize(glctx, pos_clip, tri, resolution=[H, W])     # dr.rasterize
    out, _  = interpolate(attr[None], rast, tri)                      # dr.interpolate
    out     = antialias(color, rast, pos_clip, tri)                   # dr.antialias

`pos_clip` is [1,V,4] (or [V,4]) clip-space positions, `tri` [F,3] int32, `rast` [1,H,W,4] =
(u, v, z/w, triangle id + 1).  `glctx` is accepted and ignored: no OpenGL / CUDA-GL context is needed.
Batch size 1 (what DG-Mesh renders).  Gradients flow to `pos_clip` (through the barycentrics and through the
antialiased silhouettes), to `attr` and to `color`; csrc/meshrast.cu states the contract.  CUDA tensors
only -- no CPU fallback."""
import os
import sys

import torch

_root = os.path.dirname(os.path.abspath(__file__))
if _root not in sys.path:
    sys.path.insert(0, _root)
import _dgm_lib  # noqa: E402


def _req(t, name):
    if not t.is_cuda:
        raise ValueError(f"meshrast: {name} must be a CUDA tensor (no CPU fallback)")
    return t


def _pos2(pos):
    p = pos[0] if pos.dim() == 3 else pos
    if p.dim() != 2 or p.shape[1] != 4:
        raise ValueError("meshrast: pos must be [1,V,4] or [V,4] clip-space positions")
    return p


def _tri(tri):
    if tri.dim() != 2 or tri.shape[1] != 3:
        raise ValueError("meshrast: tri must be [F,3]")
    return tri.to(torch.int32).contiguous()


class RasterizeContext:
    """Stands where dr.RasterizeGLContext() / dr.RasterizeCudaContext() stand; holds nothing."""

    def __init__(self, *args, **kwargs):
        pass


RasterizeGLContext = RasterizeCudaContext = RasterizeContext


class _Rasterize(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pos, tri, H, W):
        p = _req(pos, "pos").contiguous().float()
        V, F = p.shape[0], tri.shape[0]
        rast = torch.empty((H, W, 4), dtype=torch.float32, device=p.device)
        zbuf = torch.empty((H * W,), dtype=torch.int64, device=p.device)
        rc = _dgm_lib.lib().dgmr_rasterize(V, F, W, H, _dgm_lib.ptr(p), _dgm_lib.ptr(tri), zbuf.data_ptr(),
                                           rast.data_ptr(), _dgm_lib.stream_ptr())
        _dgm_lib.check(rc, "dgmr_rasterize")
        ctx.save_for_backward(p, tri, rast)
        ctx.hw = (H, W)
        return rast

    @staticmethod
    def backward(ctx, grast):
        p, tri, rast = ctx.saved_tensors
        H, W = ctx.hw
        gpos = torch.zeros_like(p)
        if tri.shape[0]:
            rc = _dgm_lib.lib().dgmr_rasterize_bwd(W, H, rast.data_ptr(), tri.data_ptr(), p.data_ptr(),
                                                   grast.contiguous().float().data_ptr(), gpos.data_ptr(),
                                                   _dgm_lib.stream_ptr())
            _dgm_lib.check(rc, "dgmr_rasterize_bwd")
        return gpos, None, None, None


def rasterize(glctx, pos, tri, resolution, ranges=None, grad_db=True):
    """dr.rasterize: returns (rast [1,H,W,4], None).  The second output (screen-space derivatives of the
    barycentrics) is not used by DG-Mesh and is not produced."""
    if ranges is not None:
        raise NotImplementedError("meshrast.rasterize: range mode is not part of DG-Mesh's path")
    H, W = int(resolution[0]), int(resolution[1])
    rast = _Rasterize.apply(_pos2(pos), _tri(tri), H, W)
    return rast[None], None


class _Interpolate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, attr, rast, tri):
        a = _req(attr, "attr").contiguous().float()
        r = rast.contiguous()
        H, W = r.shape[0], r.shape[1]
        C = a.shape[1]
        out = torch.empty((H, W, C), dtype=torch.float32, device=a.device)
        rc = _dgm_lib.lib().dgmr_interpolate(W, H, C, a.data_ptr(), r.data_ptr(), _dgm_lib.ptr(tri), out.data_ptr(),
                                             _dgm_lib.stream_ptr())
        _dgm_lib.check(rc, "dgmr_interpolate")
        ctx.save_for_backward(a, r, tri)
        return out

    @staticmethod
    def backward(ctx, gout):
        a, r, tri = ctx.saved_tensors
        H, W, C = r.shape[0], r.shape[1], a.shape[1]
        need_a, need_r = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        gattr = torch.zeros_like(a) if need_a else None
        grast = torch.empty_like(r) if need_r else None
        rc = _dgm_lib.lib().dgmr_interpolate_bwd(W, H, C, a.data_ptr(), r.data_ptr(), _dgm_lib.ptr(tri),
                                                 gout.contiguous().float().data_ptr(),
                                                 gattr.data_ptr() if need_a else None,
                                                 grast.data_ptr() if need_r else None, _dgm_lib.stream_ptr())
        _dgm_lib.check(rc, "dgmr_interpolate_bwd")
        return gattr, grast, None


def interpolate(attr, rast, tri, rast_db=None, diff_attrs=None):
    """dr.interpolate: attr [1,V,C] (or [V,C]), rast [1,H,W,4] -> ([1,H,W,C], None)."""
    a = attr[0] if attr.dim() == 3 else attr
    r = rast[0] if rast.dim() == 4 else rast
    return _Interpolate.apply(a, r, _tri(tri))[None], None


def edge_opposites(tri, n_verts):
    """opp[F,3]: for edge k = (v_k, v_(k+1)%3) of triangle f, the third vertex of the OTHER triangle sharing
    that edge, or -1 for a boundary edge (sorting the 3F undirected edge keys pairs them up; a non-manifold
    edge pairs its first two users).  The silhouette test of the antialiasing pass needs it."""
    t = tri.long()
    F = t.shape[0]
    a, b = t, t[:, [1, 2, 0]]
    third = t[:, [2, 0, 1]].reshape(-1)
    key = (torch.minimum(a, b) * int(n_verts) + torch.maximum(a, b)).reshape(-1)
    order = torch.argsort(key, stable=True)    # equal keys stay in face order: the first two users pair
    ks = key[order]
    same = ks[1:] == ks[:-1]
    # first of each run of equal keys pairs with its successor
    first = torch.ones_like(ks, dtype=torch.bool)
    first[1:] = ~same
    # position i starts a pair (i, i+1): both ends learn their partner.  Written as two max-scatters over ALL
    # adjacent positions (-1 where there is no pair) so that no data-dependent size is read back by the host.
    pair = first[:-1] & same
    ia, ib = order[:-1], order[1:]
    none = torch.full_like(ia, -1)
    partner = torch.full((3 * F,), -1, dtype=torch.long, device=t.device)
    partner.scatter_reduce_(0, ia, torch.where(pair, ib, none), reduce="amax")
    partner.scatter_reduce_(0, ib, torch.where(pair, ia, none), reduce="amax")
    opp = torch.where(partner >= 0, third[partner.clamp_min(0)], torch.full_like(partner, -1))
    return opp.view(F, 3).to(torch.int32).contiguous()


class _Antialias(torch.autograd.Function):
    @staticmethod
    def forward(ctx, color, rast, pos, tri, opp):
        c = _req(color, "color").contiguous().float()
        r, p = rast.contiguous(), pos.contiguous().float()
        H, W, C = c.shape
        out = torch.empty_like(c)
        rc = _dgm_lib.lib().dgmr_antialias(W, H, C, c.data_ptr(), r.data_ptr(), _dgm_lib.ptr(p), _dgm_lib.ptr(tri),
                                           _dgm_lib.ptr(opp), out.data_ptr(), _dgm_lib.stream_ptr())
        _dgm_lib.check(rc, "dgmr_antialias")
        ctx.save_for_backward(c, r, p, tri, opp)
        return out

    @staticmethod
    def backward(ctx, gout):
        c, r, p, tri, opp = ctx.saved_tensors
        H, W, C = c.shape
        need_c, need_p = ctx.needs_input_grad[0], ctx.needs_input_grad[2]
        gcolor = torch.empty_like(c) if need_c else None
        gpos = torch.zeros_like(p) if need_p else None
        rc = _dgm_lib.lib().dgmr_antialias_bwd(W, H, C, c.data_ptr(), r.data_ptr(), p.data_ptr(), tri.data_ptr(),
                                               opp.data_ptr(), gout.contiguous().float().data_ptr(),
                                               gcolor.data_ptr() if need_c else None,
                                               gpos.data_ptr() if need_p else None, _dgm_lib.stream_ptr())
        _dgm_lib.check(rc, "dgmr_antialias_bwd")
        return gcolor, None, gpos, None, None


def antialias(color, rast, pos, tri, topology_hash=None, pos_gradient_boost=1.0):
    """dr.antialias: color [1,H,W,C], rast [1,H,W,4], pos [1,V,4] -> [1,H,W,C].  `topology_hash` may be the
    result of `edge_opposites(tri, V)` to reuse it across calls on the same mesh."""
    c = color[0] if color.dim() == 4 else color
    r = rast[0] if rast.dim() == 4 else rast
    p = _pos2(pos)
    t = _tri(tri)
    if t.shape[0] == 0:
        return c[None]
    opp = topology_hash if topology_hash is not None else edge_opposites(t, p.shape[0])
    return _Antialias.apply(c, r.detach(), p, t, opp)[None]
