"""Drop-in `diff_gaussian_rasterization` backed by libdgmesh_b200.so (sm_90a).

Mirrors the reference Python surface
(dgmesh/submodules/diff-gaussian-rasterization/diff_gaussian_rasterization/__init__.py):
  GaussianRasterizationSettings  :157-169   same 12 fields, same order
  GaussianRasterizer             :171-220   forward(...) -> (color, radii), markVisible;
                                            + forward_depth_alpha(...) -> (color, radii, depth, alpha)
                                            + forward_with_camera_grad(...): gradients to the camera tensors
                                            + forward_normal(...) -> (color, radii, depth, alpha, normal)
                                            + forward_surface(...) -> (color, radii, depth, alpha, median_depth,
                                                                       distortion[, normal])
                                            + forward_features(...) -> (color, radii, depth, alpha, features)
  rasterize_gaussians / _RasterizeGaussians :21-155
  _C.rasterize_gaussians / _C.rasterize_gaussians_backward / _C.mark_visible
                                 (dgr/ext.cpp:15-19, dgr/rasterize_points.h:18-66)

Differences that are deliberate (DESIGN.md):
  * where the reference blocks on a copy of num_rendered in the middle of the forward
    (rasterizer_impl.cu:281), this enqueues the whole forward optimistically and waits only for
    an event recorded behind the tile scan (the rest stays queued); a frame that did not fit the
    instance workspace is re-run with the right capacity before the image is returned
    (`_Sizing`): every result is exact, nothing is raised later.
  * work is enqueued on the CURRENT torch stream (the reference uses the legacy
    default stream).
"""
import os
import struct
import sys
from typing import NamedTuple

import torch
import torch.nn as nn

_root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _root not in sys.path:
    sys.path.insert(0, _root)
import _dgm_lib  # noqa: E402

_ST_WORDS = 8
_MAX_FRAMES = 63


def _f32c(t, name):
    if t is None or t.numel() == 0:
        return None
    if t.dtype != torch.float32:
        raise TypeError(f"{name} must be float32")
    if not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor")
    return t.contiguous()


class _Notify:
    """Per-device early-notification object (dgm_notify_*): an event recorded right behind the tile
    scan and a device-mapped pinned mirror of the status words, read here through ctypes."""
    _per_device = {}

    def __init__(self):
        h = _dgm_lib.c_void_p()
        _dgm_lib.check(_dgm_lib.lib().dgm_notify_create(_dgm_lib.byref(h)), "dgm_notify_create")
        self.handle = h
        self.event = _dgm_lib.lib().dgm_notify_event(h)
        self.host_ptr = _dgm_lib.lib().dgm_notify_host(h)
        self.words = (_dgm_lib.c_int32 * (64 * _ST_WORDS)).from_address(self.host_ptr)

    @classmethod
    def get(cls, dev_index):
        n = cls._per_device.get(dev_index)
        if n is None:
            n = cls._per_device[dev_index] = _Notify()
        return n

    def wait(self):
        _dgm_lib.check(_dgm_lib.lib().dgm_notify_wait(self.handle), "dgm_notify_wait")


def _bits_to_float(v):
    return struct.unpack("f", struct.pack("i", int(v)))[0]


class _Sizing:
    """Capacity of the (Gaussian, tile) instance workspace and the depth-range hint, per image shape.

    The reference learns R with a blocking copy in the middle of every forward
    (rasterizer_impl.cu:281) and sizes its binning buffers exactly.  Here a forward is enqueued
    optimistically with the capacity the last frames needed (plus head-room); the tile scan
    mirrors the status words into pinned host memory and an event is recorded behind it, and the
    host waits for THAT event before returning -- the remaining 4/5 of the forward are still queued,
    so the GPU never idles.  If the frame did not fit (first frame of a shape, a close-up, after
    densification), the enqueued kernels skip themselves and the forward is re-run with the right
    capacity before the caller ever sees the image: results are exact in every case, no exception,
    no background-only frame."""
    hint = {}       # (device, W, H) -> [R capacity, depth lo, depth hi, longest tile list]

    @classmethod
    def lookup(cls, key, P):
        h = cls.hint.get(key)
        if h is None:
            return _round_cap(max(4 * P, 1 << 18)), 0.0, 0.0, 0
        return h[0], h[1], h[2], h[3]

    @classmethod
    def update(cls, key, R, lo, hi, max_tile=0):
        h = cls.hint.get(key)
        if h is None:
            if len(cls.hint) >= 64:      # bounded: image shapes seen by one process
                cls.hint.clear()
            h = cls.hint[key] = [0, 0.0, 0.0, 0]
        h[0] = max(h[0], _grow(R))
        h[3] = int(max_tile)
        if hi > lo:
            h[1], h[2] = lo, hi


def _run_sized(enqueue, key, P, dev_index, F=1):
    """enqueue(R_cap, notify, lo, hi, max_tile) -> outputs.  Returns (outputs, R of the largest frame)."""
    cap, lo, hi, mt = _Sizing.lookup(key, P)
    if torch.cuda.is_current_stream_capturing():
        # CUDA-graph capture: no host-side waiting; the capacity comes from the eager warm-up and an
        # overflow (status word 1) would replay as a background frame -- callers of graph replay check
        # `last_status()`; bench.py does
        return enqueue(cap, None, lo, hi, mt), None
    nt = _Notify.get(dev_index)
    out = enqueue(cap, nt, lo, hi, mt)
    nt.wait()
    w = nt.words
    R = max(w[_ST_WORDS * f] for f in range(F))
    ovf = any(w[_ST_WORDS * f + 1] for f in range(F))
    dlo = min((_bits_to_float(w[_ST_WORDS * f + 3]) for f in range(F) if w[_ST_WORDS * f + 4]), default=0.0)
    dhi = max((_bits_to_float(w[_ST_WORDS * f + 4]) for f in range(F) if w[_ST_WORDS * f + 4]), default=0.0)
    _Sizing.update(key, R, dlo, dhi, max(w[_ST_WORDS * f + 2] for f in range(F)))
    if ovf:
        cap, lo, hi, mt = _Sizing.lookup(key, P)
        out = enqueue(cap, nt, lo, hi, mt)   # same inputs, capacity >= R: cannot overflow again
        nt.wait()
        if any(w[_ST_WORDS * f + 1] for f in range(F)):
            raise _dgm_lib.DgmError("rasterizer: instance workspace overflow persisted after regrowth")
    return out, R


def _round_cap(c):
    # multiples of 32 instances keep every workspace array 128-byte sized, so the capacity can be
    # recovered from the byte size of the binning buffer: bytes = 60 * R_cap + 128
    return (int(c) + 31) // 32 * 32


def _grow(R):
    return _round_cap(int(R * 1.5) + (1 << 16))


def _cap_from_bytes(nbytes):
    return (int(nbytes) - 128) // 60


_ws_sizes = {}


def _sizes(P, W, H, R_cap):
    k = (P, W, H, R_cap)
    v = _ws_sizes.get(k)
    if v is None:
        gb, bb, ib = _dgm_lib.c_size_t(), _dgm_lib.c_size_t(), _dgm_lib.c_size_t()
        _dgm_lib.check(_dgm_lib.lib().dgr_workspace_sizes(P, W, H, R_cap, gb, bb, ib), "dgr_workspace_sizes")
        r = lambda x: (x + 511) // 512 * 512  # noqa: E731
        v = (gb.value, bb.value, ib.value, r(gb.value), r(bb.value), r(ib.value))
        if len(_ws_sizes) > 64:
            _ws_sizes.clear()
        _ws_sizes[k] = v
    return v


class _Workspace:
    """geom | binning | img | status carved from ONE device allocation (the three opaque buffers
    of the reference, dgr/rasterize_points.cu:68-78, kept together for the backward pass)."""
    __slots__ = ("buf", "geom", "binning", "img", "status", "gb", "bb", "ib", "R_cap", "nrm", "surf")

    def __init__(self, P, W, H, R_cap, dev):
        gb, bb, ib, ga, ba, ia = _sizes(P, W, H, R_cap)
        self.buf = torch.empty((ga + ba + ia + 64,), dtype=torch.uint8, device=dev)
        base = self.buf.data_ptr()
        self.geom, self.binning, self.img, self.status = base, base + ga, base + ga + ba, base + ga + ba + ia
        self.gb, self.bb, self.ib, self.R_cap = gb, bb, ib, R_cap
        self.nrm = None     # the normal workspace of a normal forward (_normal_ws)
        self.surf = None    # the surface workspace of a surface forward

    def status_tensor(self):
        return self.buf[-64:-32].view(torch.int32)

    # the reference-style separate byte tensors (views, no copies)
    def split(self):
        o1 = self.binning - self.geom
        o2 = self.img - self.geom
        return self.buf[:self.gb], self.buf[o1:o1 + self.bb], self.buf[o2:o2 + self.ib]


def _normal_ws_bytes(P, R_cap):
    n = _dgm_lib.c_size_t()
    _dgm_lib.check(_dgm_lib.lib().dgr_normal_workspace_size(P, R_cap, _dgm_lib.byref(n)), "dgr_normal_workspace_size")
    return n.value


def _surface_ws_bytes(W, H):
    n = _dgm_lib.c_size_t()
    _dgm_lib.check(_dgm_lib.lib().dgr_surface_workspace_size(W, H, _dgm_lib.byref(n)), "dgr_surface_workspace_size")
    return n.value


_null_segments = {}


def _enqueue(base, parts):
    """Call the narrowest entry point `base` + suffix that takes every argument segment in use.

    parts: (suffix, args) in ABI order; suffix None for the arguments every variant takes, otherwise an optional
    segment, args None when it is not in use.  The variants nest in that order: each one's argument list is the next
    narrower one's with its segment inserted (_dgm_lib.SIGNATURES), so every segment up to the widest one in use is
    passed, an unused one as the zeros / NULLs of its types there."""
    name = base
    for suffix, args in parts:
        if suffix is not None and args is not None:
            name = base + suffix
    out, narrower, done = [], base, name == base
    for suffix, args in parts:
        if suffix is None:
            out.extend(args)
        elif not done:
            wider = base + suffix
            out.extend(args if args is not None else _null_segment(wider, narrower, len(out)))
            narrower, done = wider, wider == name
    _dgm_lib.check(getattr(_dgm_lib.lib(), name)(*out), name)


def _null_segment(name, narrower, at):
    """The zeros / NULLs of the segment that `name` inserts into `narrower`'s arguments at position `at`."""
    v = _null_segments.get(name)
    if v is None:
        sig = _dgm_lib.SIGNATURES
        n = len(sig[name][1]) - len(sig[narrower][1])
        v = _null_segments[name] = tuple(None if t is _dgm_lib.P else 0.0 if t is _dgm_lib.c_float else 0
                                         for t in sig[name][1][at:at + n])
    return v


def _raw_forward(bg, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix,
                 projmatrix, tan_fovx, tan_fovy, H, W, sh, degree, campos, prefiltered, R_cap, notify=None,
                 lo=0.0, hi=0.0, out=None, max_tile=0, maps=None, nrm=None, surf=None):
    """One enqueue of the dgr_forward entry point (see `_enqueue`) that also writes `maps` = (depth, alpha) [1,H,W]
    and, with the maps, `nrm` = (normals [P,3], normal map [3,H,W]) and `surf` = (near, far, median [1,H,W],
    distortion [1,H,W]).  Returns (color, radii, workspace)."""
    if means3D.ndim != 2 or means3D.shape[1] != 3:
        raise ValueError("means3D must have dimensions (num_points, 3)")  # rasterize_points.cu:57-59
    dev = means3D.device
    P = means3D.shape[0]
    M = int(sh.shape[1]) if (sh is not None and sh.numel() != 0) else 0
    ws = _Workspace(P, W, H, R_cap, dev)
    if out is None:
        color = torch.empty((3, H, W), dtype=torch.float32, device=dev)
        radii = torch.empty((P,), dtype=torch.int32, device=dev)
    else:
        color, radii = out      # a re-run after an overflow writes the tensors of the first attempt
    p = _dgm_lib.ptr
    head = (P, degree, M, p(bg), W, H, p(means3D), p(sh), p(colors), p(opacity), p(scales), float(scale_modifier),
            p(rotations), p(cov3D_precomp), p(viewmatrix), p(projmatrix), p(campos), float(tan_fovx),
            float(tan_fovy), int(bool(prefiltered)), p(color), p(radii))
    tail = (ws.geom, ws.gb, ws.binning, ws.bb, R_cap, ws.img, ws.ib, ws.status,
            notify.host_ptr if notify else None, notify.event if notify else None, lo, hi, int(max_tile),
            _dgm_lib.stream_ptr())
    nrm_args = surf_args = None
    if nrm is not None:
        nb = _normal_ws_bytes(P, R_cap)
        ws.nrm = torch.empty((nb,), dtype=torch.uint8, device=dev)
        nrm_args = (p(nrm[0]), p(nrm[1]), ws.nrm.data_ptr(), nb)
    if surf is not None:
        sb = _surface_ws_bytes(W, H)
        ws.surf = torch.empty((sb,), dtype=torch.uint8, device=dev)
        surf_args = (float(surf[0]), float(surf[1]), p(surf[2]), p(surf[3]), ws.surf.data_ptr(), sb)
    _enqueue("dgr_forward", ((None, head), ("_aux", None if maps is None else (p(maps[0]), p(maps[1]))),
                             ("_nrm", nrm_args), ("_surf", surf_args), (None, tail)))
    return color, radii, ws


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings):
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                     cov3Ds_precomp, raster_settings)


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings):
        return _RasterizeGaussians._fwd(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                        cov3Ds_precomp, raster_settings)

    @staticmethod
    def backward(ctx, grad_out_color, _):
        return _RasterizeGaussians._bwd(ctx, grad_out_color)   # its last entry, dL/dnormals, is None here

    @staticmethod
    def _fwd(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
             raster_settings, maps=None, nrm=None, surf=None, cams=None, saved=()):
        """maps: None (colour only) or the (depth, alpha) [1,H,W] tensors the forward writes as well.
        nrm: None, or (normals [P,3], normal map [3,H,W]) for the normal map (with maps).
        surf: None, or (near, far, median [1,H,W], distortion [1,H,W]) for the surface maps (with maps).
        cams: None (the settings' camera), or the (viewmatrix, projmatrix, campos) to use instead.
        saved: more tensors to save for the backward, after (means3D, radii)."""
        rs = raster_settings
        if cams is not None:
            rs = rs._replace(viewmatrix=cams[0].detach(), projmatrix=cams[1].detach(), campos=cams[2].detach())
        means3D = _f32c(means3D, "means3D")
        if means3D is None:
            raise ValueError("means3D must have dimensions (num_points, 3)")
        t = (_f32c(rs.bg, "bg"), _f32c(sh, "sh"), _f32c(colors_precomp, "colors_precomp"),
             _f32c(opacities, "opacities"), _f32c(scales, "scales"), _f32c(rotations, "rotations"),
             _f32c(cov3Ds_precomp, "cov3D_precomp"), _f32c(rs.viewmatrix, "viewmatrix"),
             _f32c(rs.projmatrix, "projmatrix"), _f32c(rs.campos, "campos"))
        bg, sh_, col, opac, sc, rot, cov, view, proj, campos = t
        H, W = int(rs.image_height), int(rs.image_width)
        dev_index = means3D.device.index
        key = (dev_index, W, H)
        first = []

        def run(R_cap, notify, lo, hi, mt):
            o = _raw_forward(bg, means3D, col, opac, sc, rot, rs.scale_modifier, cov, view, proj, rs.tanfovx,
                             rs.tanfovy, H, W, sh_, rs.sh_degree, campos, rs.prefiltered, R_cap, notify, lo, hi,
                             first[0] if first else None, mt, maps, nrm, surf)
            if not first:
                first.append(o[:2])
            return o

        (color, radii, ws), _ = _run_sized(run, key, means3D.shape[0], dev_index)
        if rs.debug:
            torch.cuda.current_stream().synchronize()   # the reference's debug mode checks after every kernel
        ctx.raster_settings = rs
        ctx.ws = ws
        ctx.R_cap = ws.R_cap
        ctx.tensors = t
        ctx.has_m2d = means2D is not None
        ctx.save_for_backward(means3D, radii, *saved)
        ctx.mark_non_differentiable(radii)
        return color, radii

    @staticmethod
    def _bwd(ctx, grad_out_color, grad_depth=None, grad_alpha=None, cam=None, nrm=None, surf=None, abs_out=None):
        """grad_depth / grad_alpha: None, or the upstream gradients of the maps (None = unused by the loss).
        cam: None, or the _CameraGrads the backward writes the camera gradients to.
        nrm: None, or (upstream gradient of the normal map, whether dL/dnormals is needed).
        surf: None, or (near, far, upstream gradients of the median-depth and distortion maps, each None when
        unused, not both).
        abs_out: None, or the [P,3] tensor the backward writes the absolute screen-space gradient to.
        Returns the eight Gaussian inputs' gradients in the reference's order, then dL/dnormals [P,3] (or None)."""
        rs = ctx.raster_settings
        bg, sh, col, opac, sc, rot, cov, view, proj, campos = ctx.tensors
        means3D, radii = ctx.saved_tensors[:2]
        ws = ctx.ws
        P = means3D.shape[0]
        H, W = int(rs.image_height), int(rs.image_width)
        M = int(sh.shape[1]) if sh is not None else 0
        # all nine gradients in one allocation (each sub-buffer 16-byte aligned for vector stores):
        # m2d[P,3] (conic: not materialised) opac[P] col[P,3] m3d[P,3] cov[P,6] scale[P,3] rot[P,4] sh[P,M,3]
        offs, o = [], 0
        for w in (3, 0, 1, 3, 3, 6, 3, 4, 3 * M):
            offs.append(o)
            o = (o + P * w + 3) // 4 * 4
        flat = torch.empty((max(o, 1),), dtype=torch.float32, device=means3D.device)
        base = flat.data_ptr()
        ptrs = [base + 4 * x for x in offs]

        def gview(i, *shape):     # one as_strided per gradient (slice + view cost twice as much on the host)
            stride, n = [], 1
            for d in reversed(shape):
                stride.append(n)
                n *= d
            return flat.as_strided(shape, stride[::-1], offs[i])

        if grad_out_color is None:    # a depth / alpha loss only
            grad_out_color = torch.zeros((3, H, W), dtype=torch.float32, device=means3D.device)
        dpix = _f32c(grad_out_color, "grad_out_color")
        p = _dgm_lib.ptr
        head = (P, rs.sh_degree, M, p(bg), W, H, p(means3D), p(sh), p(col), p(sc), float(rs.scale_modifier), p(rot),
                p(cov), p(view), p(proj), p(campos), float(rs.tanfovx), float(rs.tanfovy), p(radii), ws.geom,
                ws.binning, ws.R_cap, ws.img, p(dpix))
        grads = (ptrs[0], None, ptrs[2], ptrs[3], ptrs[4], ptrs[5], ptrs[8] if M else None, ptrs[6], ptrs[7])
        aux = nrm_args = surf_args = dnormals = None
        if grad_depth is not None or grad_alpha is not None:
            aux = (p(_f32c(grad_depth, "grad_depth")), p(_f32c(grad_alpha, "grad_alpha")))
        if nrm is not None:
            if nrm[1]:
                dnormals = torch.empty((P, 3), dtype=torch.float32, device=means3D.device)
            nrm_args = (p(_f32c(nrm[0], "grad_normal")), p(dnormals), ws.nrm.data_ptr())
        if surf is not None:
            surf_args = (float(surf[0]), float(surf[1]), p(_f32c(surf[2], "grad_median_depth")),
                         p(_f32c(surf[3], "grad_distortion")), ws.surf.data_ptr())
        _enqueue("dgr_backward", ((None, head), ("_aux", aux), (None, grads),
                                  ("_cam", None if cam is None else cam.args()), ("_nrm", nrm_args),
                                  ("_surf", surf_args), ("_abs", None if abs_out is None else (p(abs_out),)),
                                  (None, (_dgm_lib.stream_ptr(),))))
        # same ordering as the reference (:143-153)
        return (gview(4, P, 3), gview(0, P, 3) if ctx.has_m2d else None,
                gview(8, P, M, 3) if sh is not None else None, gview(3, P, 3) if col is not None else None,
                gview(2, P, 1), gview(6, P, 3) if sc is not None else None,
                gview(7, P, 4) if rot is not None else None, gview(5, P, 6) if cov is not None else None, dnormals)


class _CameraGrads:
    """Outputs and scratch of the camera gradients of F frames: [F,16] view, [F,16] proj, [F,3] campos (one
    allocation; a gradient no camera tensor needs is passed to the library as NULL)."""

    def __init__(self, F, P, dev, need):
        n = _dgm_lib.c_size_t()
        _dgm_lib.check(_dgm_lib.lib().dgr_camera_grad_workspace_size(F, P, _dgm_lib.byref(n)),
                       "dgr_camera_grad_workspace_size")
        self.out = torch.empty((35 * F + (n.value + 3) // 4,), dtype=torch.float32, device=dev)
        self.F, self.need, self.ws_bytes = F, need, n.value
        self.view = self.out[:16 * F].view(F, 16)
        self.proj = self.out[16 * F:32 * F].view(F, 16)
        self.campos = self.out[32 * F:35 * F].view(F, 3)

    def args(self):
        """(dL_dviewmatrix, dL_dprojmatrix, dL_dcampos, cam_ws, cam_ws_bytes) of dgr_backward{,_batch}_cam."""
        outs = [t.data_ptr() if need else None for t, need in zip((self.view, self.proj, self.campos), self.need)]
        return (*outs, self.out[35 * self.F:].data_ptr(), self.ws_bytes)

    def grads(self, shapes):
        """The gradients in the shapes of the camera tensors (None where none is needed)."""
        return tuple(g.reshape(shape) if need else None
                     for g, shape, need in zip((self.view, self.proj, self.campos), shapes, self.need))


_N_STREAMS = int(os.environ.get("DGMESH_B200_STREAMS", "2"))


class _BatchWorkspace:
    """F per-frame workspaces + F status blocks in one allocation (see dgr_forward_batch)."""
    __slots__ = ("buf", "geom", "binning", "img", "status", "gs", "bs", "is_", "R_cap", "F", "nrm", "nrm_stride",
                 "surf", "surf_stride")

    def __init__(self, F, P, W, H, R_cap, dev, normal=False, surface=False):
        _, _, _, ga, ba, ia = _sizes(P, W, H, R_cap)
        self.buf = torch.empty((F * (ga + ba + ia) + 32 * F,), dtype=torch.uint8, device=dev)
        base = self.buf.data_ptr()
        self.geom, self.binning, self.img = base, base + F * ga, base + F * (ga + ba)
        self.status = base + F * (ga + ba + ia)
        self.gs, self.bs, self.is_, self.R_cap, self.F = ga, ba, ia, R_cap, F
        # F normal workspaces of a normal forward (strides multiple of 512 bytes)
        self.nrm_stride = (_normal_ws_bytes(P, R_cap) + 511) // 512 * 512 if normal else 0
        self.nrm = torch.empty((F * self.nrm_stride,), dtype=torch.uint8, device=dev) if normal else None
        # F surface workspaces of a surface forward
        self.surf_stride = (_surface_ws_bytes(W, H) + 511) // 512 * 512 if surface else 0
        self.surf = torch.empty((F * self.surf_stride,), dtype=torch.uint8, device=dev) if surface else None

    def status_tensor(self):
        return self.buf[-32 * self.F:].view(torch.int32).view(self.F, 8)

    def frame(self, f):
        """The workspace of frame f as a single-frame `_Workspace`-like view (for export_state)."""
        w = _Workspace.__new__(_Workspace)
        w.buf, w.R_cap = self.buf, self.R_cap
        w.geom, w.binning, w.img = self.geom + f * self.gs, self.binning + f * self.bs, self.img + f * self.is_
        w.status = self.status + 32 * f
        return w


_stacked = {}   # camera tensors' (address, version) -> stacked copies: a training loop reuses its cameras


def _stack_settings(settings, dev):
    key = tuple((s.viewmatrix.data_ptr(), s.viewmatrix._version, s.projmatrix.data_ptr(), s.projmatrix._version,
                 s.campos.data_ptr(), s.campos._version, float(s.tanfovx), float(s.tanfovy)) for s in settings)
    hit = _stacked.get(key)
    if hit is not None and not torch.cuda.is_current_stream_capturing():
        return hit[0]
    out = _stack_settings_uncached(settings, dev)
    if len(_stacked) >= 8:
        _stacked.clear()
    # the entry keeps the source tensors alive: their addresses cannot be recycled for other cameras while the
    # key is valid, and in-place updates move the version counters
    _stacked[key] = (out, [(s.viewmatrix, s.projmatrix, s.campos) for s in settings])
    return out


def _stack_settings_uncached(settings, dev):
    views = torch.stack([_f32c(s.viewmatrix, "viewmatrix") for s in settings]).contiguous()
    projs = torch.stack([_f32c(s.projmatrix, "projmatrix") for s in settings]).contiguous()
    cams = torch.stack([_f32c(s.campos, "campos") for s in settings]).contiguous()
    return (views, projs, cams) + _fovs(settings)


def _fovs(settings):
    """tan(fov / 2) of every frame as two host float arrays."""
    F = len(settings)
    return ((_dgm_lib.c_float * F)(*[float(s.tanfovx) for s in settings]),
            (_dgm_lib.c_float * F)(*[float(s.tanfovy) for s in settings]))


_PF_MEANS, _PF_SCALES, _PF_ROTS, _PF_OPAC, _PF_COLOR, _PF_COV = 1, 2, 4, 8, 16, 32


class _RasterizeGaussiansBatch(torch.autograd.Function):
    """F frames in one call: colors [F,3,H,W], radii [F,P].

    Every Gaussian input may be SHARED ([P,.] -- its gradient is the sum over frames, accumulated
    inside the kernels) or PER FRAME (a leading F dimension, [F,P,.] -- its gradient is [F,P,.]).
    DG-Mesh's dynamic scenes deform means / scales / rotations by the frame's time
    (gaussian_renderer/__init__.py:60-86), so those arrive per frame while opacity and SH are shared.
    means2D, if given as an [F,P,3] tensor, receives the per-frame screen-space gradients."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, settings):
        return _RasterizeGaussiansBatch._fwd(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                             cov3Ds_precomp, settings)

    @staticmethod
    def backward(ctx, grad_out_color, _):
        return _RasterizeGaussiansBatch._bwd(ctx, grad_out_color)   # its last entry, dL/dnormals, is None here

    @staticmethod
    def _fwd(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, settings,
             maps=None, nrm=None, surf=None, cams=None, saved=()):
        """maps: None (colour only) or the (depth, alpha) [F,1,H,W] tensors the forward writes as well.
        nrm: None, or (normals [P,3] shared or [F,P,3] per frame, normal maps [F,3,H,W]) (with maps).
        surf: None, or (near, far, median [F,1,H,W], distortion [F,1,H,W]) (with maps).
        cams: None (the settings' cameras), or the stacked (views [F,4,4], projs [F,4,4], campos [F,3]) to use.
        saved: more tensors to save for the backward, after (means3D, radii)."""
        rs0 = settings[0]
        F = len(settings)
        if F > _MAX_FRAMES:
            raise ValueError(f"at most {_MAX_FRAMES} frames per batch")
        for s in settings:
            if (s.image_height, s.image_width, s.sh_degree, s.scale_modifier) != \
                    (rs0.image_height, rs0.image_width, rs0.sh_degree, rs0.scale_modifier):
                raise ValueError("all frames of a batch must share image size, SH degree and scale modifier")
        means3D = _f32c(means3D, "means3D")
        if means3D is None:
            raise ValueError("means3D must have dimensions (num_points, 3)")
        t = (_f32c(rs0.bg, "bg"), _f32c(sh, "sh"), _f32c(colors_precomp, "colors_precomp"),
             _f32c(opacities, "opacities"), _f32c(scales, "scales"), _f32c(rotations, "rotations"),
             _f32c(cov3Ds_precomp, "cov3D_precomp"))
        bg, sh_, col, opac, sc, rot, cov = t
        # per-frame mask from the ranks: means [F,P,3], scales [F,P,3], rotations [F,P,4], opacities [F,P,1],
        # shs [F,P,M,3] / colors [F,P,3], cov3D [F,P,6]
        pf = 0
        for x, rank, bit in ((means3D, 3, _PF_MEANS), (sc, 3, _PF_SCALES), (rot, 3, _PF_ROTS), (opac, 3, _PF_OPAC),
                             (sh_, 4, _PF_COLOR), (col, 3, _PF_COLOR), (cov, 3, _PF_COV)):
            if x is not None and x.ndim == rank:
                if x.shape[0] != F:
                    raise ValueError("per-frame inputs must have a leading dimension equal to the number of frames")
                pf |= bit
        P = means3D.shape[-2]
        if means3D.shape[-1] != 3:
            raise ValueError("means3D must have dimensions (num_points, 3)")
        dev = means3D.device
        if cams is None:
            views, projs, cams, tx, ty = _stack_settings(settings, dev)
        else:
            views, projs, cams = (_f32c(t.detach(), n) for t, n in zip(cams, ("viewmatrix", "projmatrix", "campos")))
            tx, ty = _fovs(settings)
        H, W = int(rs0.image_height), int(rs0.image_width)
        M = int(sh_.shape[-2]) if sh_ is not None else 0
        key = (dev.index, W, H)
        p = _dgm_lib.ptr
        first = []

        def run(R_cap, notify, lo, hi, mt):
            ws = _BatchWorkspace(F, P, W, H, R_cap, dev, nrm is not None, surf is not None)
            if first:
                color, radii = first[0]
            else:
                color = torch.empty((F, 3, H, W), dtype=torch.float32, device=dev)
                radii = torch.empty((F, P), dtype=torch.int32, device=dev)
                first.append((color, radii))
            head = (F, P, rs0.sh_degree, M, p(bg), W, H, p(means3D), p(sh_), p(col), p(opac), p(sc),
                    float(rs0.scale_modifier), p(rot), p(cov), pf, p(views), p(projs), p(cams), tx, ty,
                    int(bool(rs0.prefiltered)), p(color), p(radii))
            tail = (ws.geom, ws.gs, ws.binning, ws.bs, R_cap, ws.img, ws.is_, ws.status,
                    notify.host_ptr if notify else None, notify.event if notify else None, lo, hi, int(mt),
                    _N_STREAMS, _dgm_lib.stream_ptr())
            _enqueue("dgr_forward_batch", (
                (None, head), ("_aux", None if maps is None else (p(maps[0]), p(maps[1]))),
                ("_nrm", None if nrm is None else (p(nrm[0]), int(nrm[0].ndim == 3), p(nrm[1]), ws.nrm.data_ptr(),
                                                   ws.nrm_stride)),
                ("_surf", None if surf is None else (float(surf[0]), float(surf[1]), p(surf[2]), p(surf[3]),
                                                     ws.surf.data_ptr(), ws.surf_stride)),
                (None, tail)))
            return color, radii, ws

        (color, radii, ws), _ = _run_sized(run, key, P, dev.index, F)
        ctx.ws, ctx.tensors, ctx.cams, ctx.settings = ws, t, (views, projs, cams, tx, ty), settings
        ctx.has_m2d = means2D is not None
        ctx.pf = pf
        ctx.normals_pf = int(nrm is not None and nrm[0].ndim == 3)
        ctx.save_for_backward(means3D, radii, *saved)
        ctx.mark_non_differentiable(radii)
        return color, radii

    @staticmethod
    def _bwd(ctx, grad_out_color, grad_depth=None, grad_alpha=None, cam=None, nrm=None, surf=None, abs_out=None):
        """As _RasterizeGaussians._bwd for F frames: the upstream gradients have a leading F dimension, abs_out is
        [F,P,3], and dL/dnormals is [F,P,3] for per-frame normals, else [P,3]."""
        bg, sh, col, opac, sc, rot, cov = ctx.tensors
        views, projs, cams, tx, ty = ctx.cams
        means3D, radii = ctx.saved_tensors[:2]
        ws, rs0, pf = ctx.ws, ctx.settings[0], ctx.pf
        F, P = ws.F, means3D.shape[-2]
        H, W = int(rs0.image_height), int(rs0.image_width)
        M = int(sh.shape[-2]) if sh is not None else 0

        def nf(bit):
            return F if (pf & bit) else 1

        # m2d[F,P,3] opac col m3d cov scale rot sh -- per-frame inputs get F slabs; the colour gradient (with SH
        # colours) and the cov3D gradient (without cov3D_precomp) are not returned, so they are not computed
        widths = (3 * F, nf(_PF_OPAC), 3 * nf(_PF_COLOR) if col is not None else 0, 3 * nf(_PF_MEANS),
                  6 * nf(_PF_COV) if cov is not None else 0, 3 * nf(_PF_SCALES), 4 * nf(_PF_ROTS),
                  3 * M * nf(_PF_COLOR))
        offs, o = [], 0
        for w in widths:
            offs.append(o)
            o = (o + P * w + 3) // 4 * 4
        flat = torch.empty((max(o, 1),), dtype=torch.float32, device=means3D.device)
        base = flat.data_ptr()
        ptrs = [base + 4 * x for x in offs]

        def gview(i, bit, *shape):
            if bit and (pf & bit):
                shape = (F,) + shape
            stride, n = [], 1
            for d in reversed(shape):
                stride.append(n)
                n *= d
            return flat.as_strided(shape, stride[::-1], offs[i])

        if grad_out_color is None:    # a depth / alpha loss only
            grad_out_color = torch.zeros((F, 3, H, W), dtype=torch.float32, device=means3D.device)
        dpix = _f32c(grad_out_color, "grad_out_color")
        p = _dgm_lib.ptr
        head = (F, P, rs0.sh_degree, M, p(bg), W, H, p(means3D), p(sh), p(col), p(sc), float(rs0.scale_modifier),
                p(rot), p(cov), pf, p(views), p(projs), p(cams), tx, ty, p(radii), ws.geom, ws.gs, ws.binning, ws.bs,
                ws.R_cap, ws.img, ws.is_, p(dpix))
        grads = (ptrs[0], ptrs[1], ptrs[2] if col is not None else None, ptrs[3], ptrs[4] if cov is not None else None,
                 ptrs[7] if M else None, ptrs[5], ptrs[6])
        aux = nrm_args = surf_args = dnormals = None
        if grad_depth is not None or grad_alpha is not None:
            aux = (p(_f32c(grad_depth, "grad_depth")), p(_f32c(grad_alpha, "grad_alpha")))
        if nrm is not None:
            npf = ctx.normals_pf
            if nrm[1]:
                dnormals = torch.empty((F, P, 3) if npf else (P, 3), dtype=torch.float32, device=means3D.device)
            nrm_args = (p(_f32c(nrm[0], "grad_normal")), npf, p(dnormals), ws.nrm.data_ptr(), ws.nrm_stride)
        if surf is not None:
            surf_args = (float(surf[0]), float(surf[1]), p(_f32c(surf[2], "grad_median_depth")),
                         p(_f32c(surf[3], "grad_distortion")), ws.surf.data_ptr(), ws.surf_stride)
        _enqueue("dgr_backward_batch", ((None, head), ("_aux", aux), (None, grads),
                                        ("_cam", None if cam is None else cam.args()), ("_nrm", nrm_args),
                                        ("_surf", surf_args), ("_abs", None if abs_out is None else (p(abs_out),)),
                                        (None, (_N_STREAMS, _dgm_lib.stream_ptr()))))
        return (gview(3, _PF_MEANS, P, 3), gview(0, 0, F, P, 3) if ctx.has_m2d else None,
                gview(7, _PF_COLOR, P, M, 3) if sh is not None else None,
                gview(2, _PF_COLOR, P, 3) if col is not None else None,
                gview(1, _PF_OPAC, P, 1), gview(5, _PF_SCALES, P, 3) if sc is not None else None,
                gview(6, _PF_ROTS, P, 4) if rot is not None else None,
                gview(4, _PF_COV, P, 6) if cov is not None else None, dnormals)


_MAX_FEATURES = 64


def _check_features(features, P, F=None):
    """features as a float32 CUDA tensor [P,C] (or, with F, [F,P,C]), 1 <= C <= 64."""
    f = _f32c(features, "features")
    shapes = "(num_points, C)" + (" or (num_frames, num_points, C)" if F is not None else "")
    ok = f is not None and ((f.ndim == 2 and f.shape[0] == P) or (F is not None and f.ndim == 3 and f.shape[:2] == (F, P)))
    if not ok or not 1 <= f.shape[-1] <= _MAX_FEATURES:
        raise ValueError(f"features must have dimensions {shapes}, 1 <= C <= {_MAX_FEATURES}")
    return f


class _FeatureState:
    """What the feature pass keeps for its backward: the features, and the feature workspace (the per-Gaussian
    accumulators of dL/dfeatures of every frame, dgr_feature_workspace_size bytes)."""
    __slots__ = ("feats", "per_frame", "buf", "C", "F")

    def __init__(self, feats, F, dev):
        self.feats, self.F, self.C = feats, F, int(feats.shape[-1])
        self.per_frame = int(feats.ndim == 3)
        P = feats.shape[-2]
        n = _dgm_lib.c_size_t()
        _dgm_lib.check(_dgm_lib.lib().dgr_feature_workspace_size(P, self.C, F, _dgm_lib.byref(n)),
                       "dgr_feature_workspace_size")
        self.buf = torch.empty((max(n.value, 16),), dtype=torch.uint8, device=dev)


def _ws_args(ws):
    """(geom, stride, binning, stride, R_cap, img, stride) of a single-frame or batch workspace."""
    if isinstance(ws, _BatchWorkspace):
        return ws.geom, ws.gs, ws.binning, ws.bs, ws.R_cap, ws.img, ws.is_
    return ws.geom, 0, ws.binning, 0, ws.R_cap, ws.img, 0


def _features_fwd(ws, st, W, H, fmap):
    """dgr_features_fwd over the blend of the forward that wrote `ws`: fmap [F,C,H,W] (or [C,H,W])."""
    P = st.feats.shape[-2]
    _dgm_lib.check(_dgm_lib.lib().dgr_features_fwd(st.F, P, st.C, W, H, st.feats.data_ptr(), st.per_frame,
                                                   *_ws_args(ws), fmap.data_ptr(), st.buf.data_ptr(), st.buf.numel(),
                                                   _dgm_lib.stream_ptr()), "dgr_features_fwd")


def _features_bwd(ws, st, W, H, fmap, grad, need):
    """dgr_features_bwd: adds the feature loss's share to the forward's accumulators (the rasterizer backward that
    follows carries it on) and returns dL/dfeatures (None when not `need`ed)."""
    P = st.feats.shape[-2]
    g = _f32c(grad, "grad_features")
    dfeat = torch.empty(st.feats.shape, dtype=torch.float32, device=st.feats.device) if need else None
    _dgm_lib.check(_dgm_lib.lib().dgr_features_bwd(st.F, P, st.C, W, H, st.feats.data_ptr(), st.per_frame,
                                                   *_ws_args(ws), fmap.data_ptr(), g.data_ptr(), _dgm_lib.ptr(dfeat),
                                                   st.buf.data_ptr(), st.buf.numel(), _dgm_lib.stream_ptr()),
                   "dgr_features_bwd")
    return dfeat


def _check_normals(normals, P, F=None):
    """normals as a float32 CUDA tensor [P,3] (or, with F, [P,3] shared by the frames or [F,P,3] per frame)."""
    n = _f32c(normals, "normals")
    if F is None:
        if n is None or n.shape != (P, 3):
            raise ValueError("normals must have dimensions (num_points, 3)")
    elif n is None or n.shape not in ((P, 3), (F, P, 3)):
        raise ValueError("normals must have dimensions (num_points, 3) or (num_frames, num_points, 3)")
    return n


# the outputs of the maps Functions, in order; a map the request does not ask for is None
_MAPS = ("color", "radii", "depth", "alpha", "median_depth", "distortion", "normal", "features")


def _maps_forward(ctx, batch, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                  normals, features, viewmatrix, projmatrix, campos, means2D_abs, settings, request):
    """Forward of the maps Functions (F frames when `batch`): the outputs of _MAPS."""
    ctx.set_materialize_grads(False)
    depth_alpha, surface = request
    F = len(settings) if batch else None
    lead = (F,) if batch else ()
    rs0 = settings[0] if batch else settings
    H, W = int(rs0.image_height), int(rs0.image_width)
    P, dev = means3D.shape[-2], means3D.device

    def new_map(channels):
        return torch.empty(lead + (channels, H, W), dtype=torch.float32, device=dev)

    ctx.abs_shape = lead + (P, 3)
    if means2D_abs is not None and tuple(means2D_abs.shape) != ctx.abs_shape:
        raise ValueError(f"means2D_abs must have dimensions {ctx.abs_shape}")
    maps = (new_map(1), new_map(1)) if depth_alpha else None
    nrm = None if normals is None else (_check_normals(normals, P, F), new_map(3))
    surf = None if surface is None else (surface[0], surface[1], new_map(1), new_map(1))
    st = fmap = None
    if features is not None:
        st = _FeatureState(_check_features(features, P, F), F or 1, dev)
        fmap = new_map(st.C)
    cams = None if viewmatrix is None else (viewmatrix, projmatrix, campos)
    core = _RasterizeGaussiansBatch if batch else _RasterizeGaussians
    color, radii = core._fwd(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                             settings, maps, nrm, surf, cams, () if fmap is None else (fmap,))
    if st is not None:
        _features_fwd(ctx.ws, st, W, H, fmap)
    ctx.feat, ctx.surface, ctx.frames = st, surface, F or 1
    ctx.cam_shapes = None if cams is None else tuple(t.shape for t in cams)
    return (color, radii) + (maps or (None, None)) + (surf[2:] if surf else (None, None)) + \
        (None if nrm is None else nrm[1], fmap)


def _maps_backward(ctx, core, grad_color, _, grad_depth, grad_alpha, grad_median, grad_dist, grad_normal,
                   grad_features):
    """Backward of the maps Functions: the feature pass first (it adds to the forward's accumulators), then `core`'s
    rasterizer backward with the segments the upstream gradients use."""
    *_, need_normals, need_features, need_view, need_proj, need_campos, need_abs, _, _ = ctx.needs_input_grad
    means3D = ctx.saved_tensors[0]
    dfeat = None
    if grad_features is not None:
        fmap = ctx.saved_tensors[2]
        dfeat = _features_bwd(ctx.ws, ctx.feat, fmap.shape[-1], fmap.shape[-2], fmap, grad_features, need_features)
    need = (need_view, need_proj, need_campos)
    cam = _CameraGrads(ctx.frames, means3D.shape[-2], means3D.device, need) if any(need) else None
    ab = torch.empty(ctx.abs_shape, dtype=torch.float32, device=means3D.device) if need_abs else None
    nrm = None if grad_normal is None else (grad_normal, need_normals)
    surf = None if grad_median is None and grad_dist is None else (*ctx.surface, grad_median, grad_dist)
    g = core._bwd(ctx, grad_color, grad_depth, grad_alpha, cam, nrm, surf, ab)
    return g + (dfeat,) + (cam.grads(ctx.cam_shapes) if cam else (None, None, None)) + (ab, None, None)


class _RasterizeGaussiansMaps(torch.autograd.Function):
    """`_RasterizeGaussians` + the maps a request asks for.  Inputs: the eight Gaussian tensors of
    `_RasterizeGaussians`; normals [P,3] for the normal map sum_i n_i alpha_i T_i [3,H,W] and features [P,C] for the
    feature map [C,H,W] (each None when not asked for); viewmatrix [4,4], projmatrix [4,4] and campos [3], which
    replace the settings' tensors and receive gradients (None: the settings' camera, no camera gradient);
    means2D_abs [P,3], whose gradient is the absolute screen-space gradient (or None); the settings; the request
    (depth_alpha: the depth map sum_i d_i alpha_i T_i and the alpha map 1 - T_final [1,H,W]; (near, far) for the
    median-depth and distortion maps [1,H,W], or None).  Outputs: _MAPS.  Normals, surface maps and features need
    depth_alpha; the feature map is a pass over the forward's workspaces (dgr_features_fwd / _bwd).  Gradients are
    not materialised: a map the loss does not use reaches the library as NULL, and the backward calls the narrowest
    entry point the loss needs."""

    @staticmethod
    def forward(ctx, *inputs):
        return _maps_forward(ctx, False, *inputs)

    @staticmethod
    def backward(ctx, *grads):
        return _maps_backward(ctx, _RasterizeGaussians, *grads)


class _RasterizeGaussiansBatchMaps(torch.autograd.Function):
    """`_RasterizeGaussiansMaps` for F frames over `_RasterizeGaussiansBatch`: the settings are a tuple, every map
    has a leading F dimension, normals and features are [P,.] shared by the frames (their gradient the sum over the
    frames) or [F,P,.] per frame, the cameras [F,4,4], [F,4,4], [F,3] and means2D_abs [F,P,3]."""

    @staticmethod
    def forward(ctx, *inputs):
        return _maps_forward(ctx, True, *inputs)

    @staticmethod
    def backward(ctx, *grads):
        return _maps_backward(ctx, _RasterizeGaussiansBatch, *grads)


def rasterize_gaussians_batch(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                              settings):
    return _RasterizeGaussiansBatch.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                          cov3Ds_precomp, tuple(settings))


def _exclusive_inputs(shs, colors_precomp, scales, rotations, cov3D_precomp):
    """The reference's argument-exclusivity errors (:191-195); absent inputs become empty tensors."""
    if (shs is None) == (colors_precomp is None):
        raise Exception('Please provide excatly one of either SHs or precomputed colors!')
    if ((scales is None or rotations is None) and cov3D_precomp is None) or \
            ((scales is not None or rotations is not None) and cov3D_precomp is not None):
        raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
    e = torch.Tensor([])
    return tuple(e if x is None else x for x in (shs, colors_precomp, scales, rotations, cov3D_precomp))


def _request_maps(plain, function, settings, cams, means3D, means2D, opacities, shs, colors_precomp, scales,
                  rotations, cov3D_precomp, depth_alpha, normals, surface, features, means2D_abs):
    """The rasterizers' `_maps`: the reference-shaped `plain` Function when only colour is asked for, else the maps
    `function`; the outputs by name, in _MAPS order, without the maps not asked for."""
    if features is not None and means2D_abs is not None:
        # the feature pass adds its dL/dalpha in a pass of its own, so no per-pixel total exists to take |.| of
        raise ValueError("abs_grad: the absolute screen-space gradient is not available with feature or flow maps")
    sh, col, sc, rot, cov = _exclusive_inputs(shs, colors_precomp, scales, rotations, cov3D_precomp)
    depth_alpha = bool(depth_alpha) or normals is not None or surface is not None or features is not None
    if not depth_alpha and cams[0] is None and means2D_abs is None:
        color, radii = plain.apply(means3D, means2D, sh, col, opacities, sc, rot, cov, settings)
        return {"color": color, "radii": radii}
    surface = None if surface is None else (float(surface[0]), float(surface[1]))
    out = function.apply(means3D, means2D, sh, col, opacities, sc, rot, cov, normals, features, *cams, means2D_abs,
                         settings, (depth_alpha, surface))
    return {name: t for name, t in zip(_MAPS, out) if t is not None}


class BatchGaussianRasterizer(nn.Module):
    """`GaussianRasterizer` for a batch of frames (one settings tuple per frame, same image size)."""

    def __init__(self, settings):
        super().__init__()
        self.settings = tuple(settings)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None, means2D_abs=None):
        """F frames -> (color [F,3,H,W], radii [F,P]).  means2D_abs ([F,P,3], e.g. zeros with requires_grad) receives
        in its .grad each frame's absolute screen-space gradient (see GaussianRasterizer.forward_abs_grad)."""
        if means2D_abs is not None:
            return tuple(self._maps(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp,
                                    means2D_abs=means2D_abs).values())
        if (shs is None) == (colors_precomp is None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        e = torch.Tensor([])
        return rasterize_gaussians_batch(means3D, means2D, e if shs is None else shs,
                                         e if colors_precomp is None else colors_precomp, opacities,
                                         e if scales is None else scales, e if rotations is None else rotations,
                                         e if cov3D_precomp is None else cov3D_precomp, self.settings)

    def _maps(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
              cov3D_precomp=None, depth_alpha=False, normals=None, surface=None, features=None, camera_grad=False,
              means2D_abs=None):
        """Every frame's outputs by name, in _MAPS order: "color" and "radii"; "depth" and "alpha" with depth_alpha
        or any other map; "median_depth" and "distortion" with surface = (near, far); "normal" with normals ([P,3]
        or [F,P,3]); "features" with features ([P,C] or [F,P,C]).  camera_grad: the frames' camera tensors receive
        gradients.  means2D_abs: see `forward` (not with features)."""
        cams = (None, None, None)
        if camera_grad:
            cams = tuple(torch.stack([getattr(s, k) for s in self.settings])
                         for k in ("viewmatrix", "projmatrix", "campos"))
        return _request_maps(_RasterizeGaussiansBatch, _RasterizeGaussiansBatchMaps, self.settings, cams, means3D,
                             means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp, depth_alpha,
                             normals, surface, features, means2D_abs)

    def forward_depth_alpha(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None,
                            rotations=None, cov3D_precomp=None, means2D_abs=None):
        """`forward` + the depth map sum_i d_i alpha_i T_i (view-space depth, unnormalised: expected depth is
        depth / alpha) and the alpha map 1 - T_final.  Returns (color [F,3,H,W], radii [F,P], depth [F,1,H,W],
        alpha [F,1,H,W]); both maps are differentiable.  means2D_abs: see `forward`."""
        return tuple(self._maps(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp,
                                depth_alpha=True, means2D_abs=means2D_abs).values())

    def forward_with_camera_grad(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None,
                                 rotations=None, cov3D_precomp=None, depth_alpha=False, means2D_abs=None):
        """`forward` (depth_alpha: `forward_depth_alpha`) whose result is also differentiable with respect to each
        frame's settings.viewmatrix, settings.projmatrix and settings.campos: gradients reach those tensors that
        require them (stacked with autograd).  Intrinsics (tanfovx / tanfovy) are not differentiated.
        means2D_abs: see `forward`."""
        return tuple(self._maps(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp,
                                depth_alpha=depth_alpha, camera_grad=True, means2D_abs=means2D_abs).values())

    def forward_normal(self, means3D, means2D, opacities, normals, shs=None, colors_precomp=None, scales=None,
                       rotations=None, cov3D_precomp=None, camera_grad=False, means2D_abs=None):
        """`forward_depth_alpha` + the normal maps sum_i n_i alpha_i T_i [F,3,H,W] of `normals`: [P,3] shared by
        the frames (its gradient is the sum over the frames) or [F,P,3] per frame.  The vectors are blended as
        given (see GaussianRasterizer.forward_normal).  camera_grad=True: also differentiable with respect to each
        frame's settings.viewmatrix, .projmatrix and .campos (see `forward_with_camera_grad`).  means2D_abs: see
        `forward`.  Returns (color [F,3,H,W], radii [F,P], depth [F,1,H,W], alpha [F,1,H,W], normal [F,3,H,W])."""
        if normals is None:
            raise ValueError("normals must have dimensions (num_points, 3) or (num_frames, num_points, 3)")
        return tuple(self._maps(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp,
                                normals=normals, camera_grad=camera_grad, means2D_abs=means2D_abs).values())

    def forward_surface(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None,
                        rotations=None, cov3D_precomp=None, normals=None, near=0.2, far=100.0, camera_grad=False,
                        means2D_abs=None):
        """`forward_depth_alpha` + the median-depth and distortion maps [F,1,H,W] of every frame (see
        GaussianRasterizer.forward_surface); with `normals` ([P,3] shared or [F,P,3] per frame) also the normal maps
        of `forward_normal`.  means2D_abs: see `forward`.  Returns (color [F,3,H,W], radii [F,P], depth, alpha,
        median_depth, distortion [F,1,H,W] each[, normal [F,3,H,W]]); every map is differentiable."""
        return tuple(self._maps(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp,
                                normals=normals, surface=(near, far), camera_grad=camera_grad,
                                means2D_abs=means2D_abs).values())

    def forward_features(self, means3D, means2D, opacities, features, shs=None, colors_precomp=None, scales=None,
                         rotations=None, cov3D_precomp=None, camera_grad=False, normals=None, surface=None):
        """`forward_depth_alpha` + the feature maps sum_i f_i alpha_i T_i [F,C,H,W] of `features`: [P,C] shared by
        the frames (its gradient is the sum over the frames in frame order) or [F,P,C] per frame, 1 <= C <= 64 (see
        GaussianRasterizer.forward_features).  camera_grad=True: also differentiable with respect to each frame's
        settings.viewmatrix, .projmatrix and .campos.  With `normals` ([P,3] or [F,P,3]) also the normal maps of
        `forward_normal`, with `surface` = (near, far) also the maps of `forward_surface`.  Returns (color
        [F,3,H,W], radii [F,P], depth [F,1,H,W], alpha [F,1,H,W], features [F,C,H,W][, median_depth, distortion
        [F,1,H,W]][, normal [F,3,H,W]]); every map is differentiable."""
        if features is None:
            raise ValueError(f"features must have dimensions (num_points, C) or (num_frames, num_points, C), "
                             f"1 <= C <= {_MAX_FEATURES}")
        m = self._maps(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp,
                       normals=normals, surface=surface, features=features, camera_grad=camera_grad)
        f = m.pop("features")
        out = tuple(m.values())
        return out[:4] + (f,) + out[4:]


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        # frustum test (reference :176-185)
        with torch.no_grad():
            rs = self.raster_settings
            return _C.mark_visible(positions, rs.viewmatrix, rs.projmatrix)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None):
        raster_settings = self.raster_settings
        # same argument-exclusivity errors as the reference (:191-195)
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        if shs is None:
            shs = torch.Tensor([])
        if colors_precomp is None:
            colors_precomp = torch.Tensor([])
        if scales is None:
            scales = torch.Tensor([])
        if rotations is None:
            rotations = torch.Tensor([])
        if cov3D_precomp is None:
            cov3D_precomp = torch.Tensor([])
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp,
                                   raster_settings)

    def _maps(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
              cov3D_precomp=None, depth_alpha=False, normals=None, surface=None, features=None, camera_grad=False,
              means2D_abs=None):
        """The outputs by name, in _MAPS order: "color" and "radii"; "depth" and "alpha" with depth_alpha or any
        other map; "median_depth" and "distortion" with surface = (near, far); "normal" with normals [P,3];
        "features" with features [P,C].  camera_grad: see `forward_with_camera_grad`.  means2D_abs: see
        `forward_abs_grad` (not with features)."""
        rs = self.raster_settings
        cams = (rs.viewmatrix, rs.projmatrix, rs.campos) if camera_grad else (None, None, None)
        return _request_maps(_RasterizeGaussians, _RasterizeGaussiansMaps, rs, cams, means3D, means2D, opacities, shs,
                             colors_precomp, scales, rotations, cov3D_precomp, depth_alpha, normals, surface,
                             features, means2D_abs)

    def forward_depth_alpha(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None,
                            rotations=None, cov3D_precomp=None):
        """`forward` + the depth map sum_i d_i alpha_i T_i (view-space depth, unnormalised: expected depth is
        depth / alpha) and the alpha map 1 - T_final, over the same blend as the colour image.  Returns
        (color [3,H,W], radii [P], depth [1,H,W], alpha [1,H,W]); both maps are differentiable."""
        return tuple(self._maps(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp,
                                depth_alpha=True).values())

    def forward_with_camera_grad(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None,
                                 rotations=None, cov3D_precomp=None, depth_alpha=False):
        """`forward` (depth_alpha: `forward_depth_alpha`) whose result is also differentiable with respect to
        raster_settings.viewmatrix, .projmatrix and .campos: gradients reach those of the three tensors that require
        them, e.g. for a learnable pose correction (gaussian_renderer.posed_camera).  Intrinsics (tanfovx /
        tanfovy) are not differentiated.  Returns what `forward` / `forward_depth_alpha` return."""
        return tuple(self._maps(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp,
                                depth_alpha=depth_alpha, camera_grad=True).values())

    def forward_abs_grad(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None,
                         rotations=None, cov3D_precomp=None, *, means2D_abs, depth_alpha=False, camera_grad=False):
        """`forward` (depth_alpha: `forward_depth_alpha`; camera_grad: see `forward_with_camera_grad`) whose backward
        also writes the absolute screen-space gradient (AbsGS) into means2D_abs.grad, the way it writes dL/dmean2D
        into means2D.grad.  means2D_abs is a [P,3] tensor that requires grad (e.g. zeros); its "gradient" is
        (sum_p |g_p.x|, sum_p |g_p.y|, 0) per Gaussian, g_p the part of dL/dmean2D that pixel p contributes, summed
        over every loss on the returned maps.  Unlike dL/dmean2D it does not cancel where pixels pull a Gaussian in
        opposite directions, which makes it a densification statistic that also splits large Gaussians over fine
        detail.  Returns what `forward` / `forward_depth_alpha` return."""
        return tuple(self._maps(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp,
                                depth_alpha=depth_alpha, camera_grad=camera_grad, means2D_abs=means2D_abs).values())

    def forward_normal(self, means3D, means2D, opacities, normals, shs=None, colors_precomp=None, scales=None,
                       rotations=None, cov3D_precomp=None, camera_grad=False, means2D_abs=None):
        """`forward_depth_alpha` + the normal map N = sum_i n_i alpha_i T_i [3,H,W] of the per-Gaussian 3-vectors
        `normals` [P,3], over the same blend.  The vectors are blended as given (normalise them and rotate them
        into camera space beforehand if that is what the map should show); N has no background term and is not
        normalised: N / alpha is the alpha-weighted mean normal.  camera_grad=True: also differentiable with
        respect to raster_settings.viewmatrix, .projmatrix and .campos (see `forward_with_camera_grad`).  Returns
        (color [3,H,W], radii [P], depth [1,H,W], alpha [1,H,W], normal [3,H,W]); every map is differentiable.
        means2D_abs: see `forward_abs_grad`."""
        if normals is None:
            raise ValueError("normals must have dimensions (num_points, 3)")
        return tuple(self._maps(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp,
                                normals=normals, camera_grad=camera_grad, means2D_abs=means2D_abs).values())

    def forward_surface(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None,
                        rotations=None, cov3D_precomp=None, normals=None, near=0.2, far=100.0, camera_grad=False,
                        means2D_abs=None):
        """`forward_depth_alpha` + two maps for surface regularisation (2DGS), over the same blend:
          median_depth  the view depth d_i of the last record blended while the transmittance before it is > 0.5
                        (a pixel that never falls to 0.5: its last contributor; an empty pixel: 0).  Its gradient
                        reaches the depth of that record only.
          distortion    1/2 sum_ij w_i w_j (m_i - m_j)^2 with w_i = alpha_i T_i and the normalised depth
                        m_i = far / (far - near) (1 - near / d_i), 0 < near < far.
        With `normals` [P,3] also the normal map of `forward_normal`.  camera_grad=True: also differentiable with
        respect to raster_settings.viewmatrix, .projmatrix and .campos.  Returns (color [3,H,W], radii [P], depth,
        alpha, median_depth, distortion [1,H,W] each[, normal [3,H,W]]); every map is differentiable.  means2D_abs: see
        `forward_abs_grad`."""
        return tuple(self._maps(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp,
                                normals=normals, surface=(near, far), camera_grad=camera_grad,
                                means2D_abs=means2D_abs).values())

    def forward_features(self, means3D, means2D, opacities, features, shs=None, colors_precomp=None, scales=None,
                         rotations=None, cov3D_precomp=None, camera_grad=False):
        """`forward_depth_alpha` + the feature map F_c = sum_i f_{i,c} alpha_i T_i [C,H,W] of caller-chosen
        per-Gaussian vectors `features` [P,C], 1 <= C <= 64, over the same blend (no background term, not
        normalised: F / alpha is the alpha-weighted mean), e.g. image-space motion for an optical-flow map or
        canonical coordinates for dense correspondences.  camera_grad=True: also differentiable with respect to
        raster_settings.viewmatrix, .projmatrix and .campos.  Returns (color [3,H,W], radii [P], depth [1,H,W], alpha
        [1,H,W], features [C,H,W]); every map is differentiable."""
        if features is None:
            raise ValueError(f"features must have dimensions (num_points, C), 1 <= C <= {_MAX_FEATURES}")
        return tuple(self._maps(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp,
                                features=features, camera_grad=camera_grad).values())


class _CCompat:
    """`diff_gaussian_rasterization._C` with the reference's three entry points and tuple
    layouts (dgr/rasterize_points.h:18-66).  These return num_rendered as a Python int and
    therefore synchronise, exactly like the reference binding."""

    @staticmethod
    def rasterize_gaussians(bg, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                            viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree,
                            campos, prefiltered, debug):
        a = [_f32c(x, n) for x, n in ((bg, "bg"), (means3D, "means3D"), (colors, "colors"), (opacity, "opacity"),
                                      (scales, "scales"), (rotations, "rotations"), (cov3D_precomp, "cov3D"),
                                      (viewmatrix, "view"), (projmatrix, "proj"), (sh, "sh"), (campos, "campos"))]
        bg_, m3, col, op, sc, ro, cov, view, proj, sh_, cam = a
        if m3 is None:
            raise ValueError("means3D must have dimensions (num_points, 3)")
        key = (m3.device.index, int(image_width), int(image_height))
        first = []

        def run(R_cap, notify, lo, hi, mt):
            o = _raw_forward(bg_, m3, col, op, sc, ro, scale_modifier, cov, view, proj, tan_fovx, tan_fovy,
                             int(image_height), int(image_width), sh_, degree, cam, prefiltered, R_cap, notify, lo, hi,
                             first[0] if first else None, mt)
            if not first:
                first.append(o[:2])
            return o

        (color, radii, ws), R = _run_sized(run, key, m3.shape[0], m3.device.index)
        if R is None:       # stream capture: this entry point returns R as a Python int and cannot be captured
            raise _dgm_lib.DgmError("_C.rasterize_gaussians returns num_rendered to the host: not capturable")
        # the three opaque byte tensors (views of one allocation) carry everything backward needs;
        # the capacity is implied by the size of the binning buffer
        geom, binning, img = ws.split()
        return R, color, radii, geom, binning, img

    @staticmethod
    def rasterize_gaussians_backward(bg, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp,
                                     viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color, sh, degree, campos,
                                     geomBuffer, R, binningBuffer, imageBuffer, debug):
        lib = _dgm_lib.lib()
        binning = binningBuffer
        cap = _cap_from_bytes(binning.numel())
        m3 = _f32c(means3D, "means3D")
        P = m3.shape[0]
        H, W = int(dL_dout_color.shape[1]), int(dL_dout_color.shape[2])
        sh_ = _f32c(sh, "sh")
        M = int(sh_.shape[1]) if sh_ is not None else 0
        f = dict(dtype=torch.float32, device=m3.device)
        g_m2d, g_conic, g_opac = torch.empty((P, 3), **f), torch.empty((P, 2, 2), **f), torch.empty((P, 1), **f)
        g_col, g_m3d, g_cov = torch.empty((P, 3), **f), torch.empty((P, 3), **f), torch.empty((P, 6), **f)
        g_sh, g_scale, g_rot = torch.empty((P, M, 3), **f), torch.empty((P, 3), **f), torch.empty((P, 4), **f)
        p = _dgm_lib.ptr
        rc = lib.dgr_backward(P, degree, M, p(_f32c(bg, "bg")), W, H, p(m3), p(sh_), p(_f32c(colors, "colors")),
                              p(_f32c(scales, "scales")), float(scale_modifier), p(_f32c(rotations, "rotations")),
                              p(_f32c(cov3D_precomp, "cov3D")), p(_f32c(viewmatrix, "view")),
                              p(_f32c(projmatrix, "proj")), p(_f32c(campos, "campos")), float(tan_fovx),
                              float(tan_fovy), p(radii.contiguous()), p(geomBuffer), p(binning), cap, p(imageBuffer),
                              p(_f32c(dL_dout_color, "dL_dout_color")), p(g_m2d), p(g_conic), p(g_opac), p(g_col),
                              p(g_m3d), p(g_cov), p(g_sh), p(g_scale), p(g_rot), _dgm_lib.stream_ptr())
        _dgm_lib.check(rc, "dgr_backward")
        return g_m2d, g_col, g_opac, g_m3d, g_cov, g_sh, g_scale, g_rot

    @staticmethod
    def mark_visible(means3D, viewmatrix, projmatrix):
        lib = _dgm_lib.lib()
        m3 = _f32c(means3D, "means3D")
        P = 0 if m3 is None else m3.shape[0]
        present = torch.zeros((P,), dtype=torch.bool, device=means3D.device)
        if P:
            rc = lib.dgr_mark_visible(P, m3.data_ptr(), _f32c(viewmatrix, "view").data_ptr(),
                                      _f32c(projmatrix, "proj").data_ptr(), present.data_ptr(),
                                      _dgm_lib.stream_ptr())
            _dgm_lib.check(rc, "dgr_mark_visible")
        return present


_C = _CCompat()


def export_state(P, W, H, ws, R):
    """Parity-test helper: reference-visible intermediate state of a forward as a dict of tensors."""
    lib = _dgm_lib.lib()
    dev = ws.buf.device
    R_cap = ws.R_cap
    T = ((W + 15) // 16) * ((H + 15) // 16)
    o = dict(
        depths=torch.zeros(P, device=dev), means2D=torch.zeros(P, 2, device=dev),
        cov3D=torch.zeros(P, 6, device=dev), conic_opacity=torch.zeros(P, 4, device=dev),
        rgb=torch.zeros(P, 3, device=dev), tiles_touched=torch.zeros(P, dtype=torch.int32, device=dev),
        clamped=torch.zeros(P, 3, dtype=torch.uint8, device=dev),
        point_list_keys=torch.zeros(max(R_cap, 1), dtype=torch.int64, device=dev),
        point_list=torch.zeros(max(R_cap, 1), dtype=torch.int32, device=dev),
        ranges=torch.zeros(T, 2, dtype=torch.int32, device=dev), final_T=torch.zeros(H * W, device=dev),
        n_contrib=torch.zeros(H * W, dtype=torch.int32, device=dev))
    p = _dgm_lib.ptr
    rc = lib.dgr_export_state(P, W, H, R_cap, ws.geom, ws.binning, ws.img, p(o["depths"]), p(o["means2D"]),
                              p(o["cov3D"]), p(o["conic_opacity"]), p(o["rgb"]), p(o["tiles_touched"]),
                              p(o["clamped"]), p(o["point_list_keys"]), p(o["point_list"]), p(o["ranges"]),
                              p(o["final_T"]), p(o["n_contrib"]), _dgm_lib.stream_ptr())
    _dgm_lib.check(rc, "dgr_export_state")
    o["point_list_keys"] = o["point_list_keys"][:R]
    o["point_list"] = o["point_list"][:R]
    return o
