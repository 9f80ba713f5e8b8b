"""Differentiable triangle-mesh rasterisation on the GPU (SURVEY.md 8(f)-1), with the call surface of the
three nvdiffrast primitives dgmesh/utils/renderer.py:33-121 uses, so that render_mask / render_mesh read
exactly like the reference:

    rast, _ = rasterize(glctx, pos_clip, tri, resolution=[H, W])     # dr.rasterize
    out, _  = interpolate(attr[None], rast, tri)                      # dr.interpolate
    out     = antialias(color, rast, pos_clip, tri)                   # dr.antialias

`pos_clip` is [1,V,4] (or [V,4]) clip-space positions, `tri` [F,3] int32, `rast` [1,H,W,4] =
(u, v, z/w, triangle id + 1).  `glctx` is accepted and ignored: no OpenGL / CUDA-GL context is needed.
One image, or B images of several meshes in one call (nvdiffrast's range mode: `ranges` [B,2]).  Gradients flow to `pos_clip` (through the barycentrics and through the
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


MAX_BATCH = 64   # images per range-mode call
MAX_TRIANGLES = 1 << 29   # rast.w holds triangle ids with nvdiffrast's encoding up to here (csrc/meshrast.cu)


def _pos2(pos):
    if pos.dim() == 3 and pos.shape[0] != 1:
        raise ValueError("meshrast: a batched pos [B,V,4] with B > 1 is nvdiffrast's instanced mode, which is not "
                         "supported; use range mode (pos [V,4] with ranges)")
    p = pos[0] if pos.dim() == 3 else pos
    if p.dim() != 2 or p.shape[1] != 4:
        raise ValueError("meshrast: pos must be [1,V,4] or [V,4] clip-space positions")
    return p


def _tri(tri):
    if tri.dim() != 2 or tri.shape[1] != 3:
        raise ValueError("meshrast: tri must be [F,3]")
    return tri.to(torch.int32).contiguous()


def _ranges(ranges, F):
    """range mode: [B,2] int32 CPU (first triangle, count) with 1 <= B <= 64, every range within [0, F]"""
    if not isinstance(ranges, torch.Tensor) or ranges.dim() != 2 or ranges.shape[1] != 2 \
            or ranges.dtype != torch.int32 or ranges.device.type != "cpu":
        raise ValueError("meshrast.rasterize: ranges must be a [B,2] int32 CPU tensor of (first triangle, count)")
    if not 1 <= ranges.shape[0] <= MAX_BATCH:
        raise ValueError(f"meshrast.rasterize: 1 <= B <= {MAX_BATCH} ranges, got {ranges.shape[0]}")
    r = ranges.contiguous()
    first, count = r[:, 0].long(), r[:, 1].long()
    if bool((first < 0).any()) or bool((count < 0).any()) or bool((first + count > F).any()):
        raise ValueError(f"meshrast.rasterize: a range runs past tri's {F} triangles")
    return r


def _image_batch(t, name, inner):
    """an image-shaped tensor [B,H,W,inner] (or [H,W,inner] for one image) -> [B,H,W,inner]"""
    if t.dim() == 3:
        t = t[None]
    if t.dim() != 4 or (inner is not None and t.shape[3] != inner):
        raise ValueError(f"meshrast: {name} must be [B,H,W,{inner if inner is not None else 'C'}]")
    if not 1 <= t.shape[0] <= MAX_BATCH:
        raise ValueError(f"meshrast: {name} holds {t.shape[0]} images, at most {MAX_BATCH} are supported")
    return t


def _call(single, batch, B, *args):
    """one launch for the B images: the single-image entry point for B = 1, its _batch form otherwise"""
    lib = _dgm_lib.lib()
    if B == 1:
        _dgm_lib.check(getattr(lib, single)(*args), single)
    else:
        _dgm_lib.check(getattr(lib, batch)(B, *args), batch)


class RasterizeContext:
    """Stands where dr.RasterizeGLContext() / dr.RasterizeCudaContext() stand; holds nothing."""

    def __init__(self, *args, **kwargs):
        pass


RasterizeGLContext = RasterizeCudaContext = RasterizeContext


class _Rasterize(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pos, tri, H, W, ranges):
        p = _req(pos, "pos").contiguous().float()
        V, F = p.shape[0], tri.shape[0]
        B = 1 if ranges is None else ranges.shape[0]
        rast = torch.empty((B, H, W, 4), dtype=torch.float32, device=p.device)
        zbuf = torch.empty((B * H * W,), dtype=torch.int64, device=p.device)
        lib, st = _dgm_lib.lib(), _dgm_lib.stream_ptr()
        if ranges is None:
            rc = lib.dgmr_rasterize(V, F, W, H, _dgm_lib.ptr(p), _dgm_lib.ptr(tri), zbuf.data_ptr(), rast.data_ptr(),
                                    st)
            _dgm_lib.check(rc, "dgmr_rasterize")
        else:
            rc = lib.dgmr_rasterize_batch(V, F, B, ranges.data_ptr(), W, H, _dgm_lib.ptr(p), _dgm_lib.ptr(tri),
                                          zbuf.data_ptr(), rast.data_ptr(), st)
            _dgm_lib.check(rc, "dgmr_rasterize_batch")
        ctx.save_for_backward(p, tri, rast)
        ctx.hw = (H, W)
        return rast

    @staticmethod
    def backward(ctx, grast):
        p, tri, rast = ctx.saved_tensors
        H, W = ctx.hw
        gpos = torch.zeros_like(p)
        if tri.shape[0]:
            _call("dgmr_rasterize_bwd", "dgmr_rasterize_bwd_batch", rast.shape[0], W, H, rast.data_ptr(),
                  tri.data_ptr(), p.data_ptr(), grast.contiguous().float().data_ptr(), gpos.data_ptr(),
                  _dgm_lib.stream_ptr())
        return gpos, None, None, None, None


def rasterize(glctx, pos, tri, resolution, ranges=None, grad_db=True):
    """dr.rasterize: returns (rast [1,H,W,4], None).  The second output (screen-space derivatives of the
    barycentrics) is not used by DG-Mesh and is not produced.

    Range mode (nvdiffrast's contract): pos [V,4], tri [F,3] with global vertex indices and ranges [B,2] int32 on
    the CPU, (first triangle, count) per image, 1 <= B <= 64 -> rast [B,H,W,4] whose triangle ids are the global
    index + 1; an empty range renders an all-zero image.  As in nvdiffrast, an id up to 2^24 is stored as a float
    and a larger one as the float with bit pattern 0x4a800000 + id (read it back with
    `w.view(torch.int32) - 0x4a800000` where w > 2^24); tri may hold up to 2^29 triangles.  A batched pos [B,V,4] (instanced mode) raises ValueError."""
    H, W = int(resolution[0]), int(resolution[1])
    t = _tri(tri)
    if t.shape[0] > MAX_TRIANGLES:
        raise ValueError(f"meshrast.rasterize: {t.shape[0]} triangles, at most 2^29 are supported")
    if ranges is None:
        return _Rasterize.apply(_pos2(pos), t, H, W, None), None
    if pos.dim() != 2:
        raise ValueError("meshrast.rasterize: range mode takes pos [V,4]")
    return _Rasterize.apply(_pos2(pos), t, H, W, _ranges(ranges, t.shape[0])), None


class _Interpolate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, attr, rast, tri):
        a = _req(attr, "attr").contiguous().float()
        r = rast.contiguous()
        B, H, W = r.shape[0], r.shape[1], r.shape[2]
        C = a.shape[1]
        out = torch.empty((B, H, W, C), dtype=torch.float32, device=a.device)
        _call("dgmr_interpolate", "dgmr_interpolate_batch", B, W, H, C, a.data_ptr(), r.data_ptr(), _dgm_lib.ptr(tri),
              out.data_ptr(), _dgm_lib.stream_ptr())
        ctx.save_for_backward(a, r, tri)
        return out

    @staticmethod
    def backward(ctx, gout):
        a, r, tri = ctx.saved_tensors
        B, H, W, C = r.shape[0], r.shape[1], r.shape[2], a.shape[1]
        need_a, need_r = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        gattr = torch.zeros_like(a) if need_a else None
        grast = torch.empty_like(r) if need_r else None
        _call("dgmr_interpolate_bwd", "dgmr_interpolate_bwd_batch", B, W, H, C, a.data_ptr(), r.data_ptr(),
              _dgm_lib.ptr(tri), gout.contiguous().float().data_ptr(), gattr.data_ptr() if need_a else None,
              grast.data_ptr() if need_r else None, _dgm_lib.stream_ptr())
        return gattr, grast, None


def interpolate(attr, rast, tri, rast_db=None, diff_attrs=None):
    """dr.interpolate: attr [1,V,C] (or [V,C]), rast [B,H,W,4] -> ([B,H,W,C], None); B > 1 is range mode, where
    every image reads the one attr.  A batched attr [B,V,C] with B > 1 (instanced mode) raises ValueError."""
    if attr.dim() == 3 and attr.shape[0] != 1:
        raise ValueError("meshrast.interpolate: a batched attr [B,V,C] with B > 1 (instanced mode) is not supported")
    a = attr[0] if attr.dim() == 3 else attr
    return _Interpolate.apply(a, _image_batch(rast, "rast", 4), _tri(tri)), None


def edge_opposites(tri, n_verts):
    """opp[F,3]: for edge k = (v_k, v_(k+1)%3) of triangle f, the third vertex of the OTHER triangle sharing
    that edge, or -1 for a boundary edge (sorting the 3F undirected edge keys pairs them up; a non-manifold
    edge pairs its first two users).  The silhouette test of the antialiasing pass needs it."""
    t = tri.long()
    F = t.shape[0]
    # column rotations written as rolls: indexing with a python list would upload the index with a blocking copy
    a, b = t, torch.roll(t, -1, 1)                 # (v1, v2, v0)
    third = torch.roll(t, -2, 1).reshape(-1)       # (v2, v0, v1)
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
        B, H, W, C = c.shape
        out = torch.empty_like(c)
        _call("dgmr_antialias", "dgmr_antialias_batch", B, W, H, C, c.data_ptr(), r.data_ptr(), _dgm_lib.ptr(p),
              _dgm_lib.ptr(tri), _dgm_lib.ptr(opp), out.data_ptr(), _dgm_lib.stream_ptr())
        ctx.save_for_backward(c, r, p, tri, opp)
        return out

    @staticmethod
    def backward(ctx, gout):
        c, r, p, tri, opp = ctx.saved_tensors
        B, H, W, C = c.shape
        need_c, need_p = ctx.needs_input_grad[0], ctx.needs_input_grad[2]
        gcolor = torch.empty_like(c) if need_c else None
        gpos = torch.zeros_like(p) if need_p else None
        _call("dgmr_antialias_bwd", "dgmr_antialias_bwd_batch", B, W, H, C, c.data_ptr(), r.data_ptr(), p.data_ptr(),
              tri.data_ptr(), opp.data_ptr(), gout.contiguous().float().data_ptr(),
              gcolor.data_ptr() if need_c else None, gpos.data_ptr() if need_p else None, _dgm_lib.stream_ptr())
        return gcolor, None, gpos, None, None


def antialias(color, rast, pos, tri, topology_hash=None, pos_gradient_boost=1.0):
    """dr.antialias: color [B,H,W,C], rast [B,H,W,4], pos [1,V,4] or [V,4] -> [B,H,W,C]; B > 1 is range mode
    (pairs of pixels never span two images).  `topology_hash` may be the result of `edge_opposites(tri, V)` to
    reuse it across calls on the same mesh.  A batched pos [B,V,4] with B > 1 (instanced mode) raises ValueError."""
    c = _image_batch(color, "color", None)
    r = _image_batch(rast, "rast", 4)
    if c.shape[:3] != r.shape[:3]:
        raise ValueError("meshrast.antialias: color and rast must cover the same [B,H,W] images")
    p = _pos2(pos)
    t = _tri(tri)
    if t.shape[0] == 0:
        return c
    opp = topology_hash if topology_hash is not None else edge_opposites(t, p.shape[0])
    return _Antialias.apply(c, r.detach(), p, t, opp)
