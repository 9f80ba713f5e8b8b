"""Drop-in `diff_gaussian_rasterization` backed by libdgmesh_b200.so (sm_90a).

Mirrors the reference Python surface
(dgmesh/submodules/diff-gaussian-rasterization/diff_gaussian_rasterization/__init__.py):
  GaussianRasterizationSettings  :157-169   same 12 fields, same order
  GaussianRasterizer             :171-220   forward(...) -> (color, radii), markVisible
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
    __slots__ = ("buf", "geom", "binning", "img", "status", "gb", "bb", "ib", "R_cap")

    def __init__(self, P, W, H, R_cap, dev):
        gb, bb, ib, ga, ba, ia = _sizes(P, W, H, R_cap)
        self.buf = torch.empty((ga + ba + ia + 64,), dtype=torch.uint8, device=dev)
        base = self.buf.data_ptr()
        self.geom, self.binning, self.img, self.status = base, base + ga, base + ga + ba, base + ga + ba + ia
        self.gb, self.bb, self.ib, self.R_cap = gb, bb, ib, R_cap

    def status_tensor(self):
        return self.buf[-64:-32].view(torch.int32)

    # the reference-style separate byte tensors (views, no copies)
    def split(self):
        o1 = self.binning - self.geom
        o2 = self.img - self.geom
        return self.buf[:self.gb], self.buf[o1:o1 + self.bb], self.buf[o2:o2 + self.ib]


def _raw_forward(bg, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix,
                 projmatrix, tan_fovx, tan_fovy, H, W, sh, degree, campos, prefiltered, R_cap, notify=None,
                 lo=0.0, hi=0.0, out=None, max_tile=0):
    """One enqueue of dgr_forward.  Returns (color, radii, workspace)."""
    lib = _dgm_lib.lib()
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
    rc = lib.dgr_forward(P, degree, M, p(bg), W, H, p(means3D), p(sh), p(colors), p(opacity), p(scales),
                         float(scale_modifier), p(rotations), p(cov3D_precomp), p(viewmatrix), p(projmatrix),
                         p(campos), float(tan_fovx), float(tan_fovy), int(bool(prefiltered)), p(color), p(radii),
                         ws.geom, ws.gb, ws.binning, ws.bb, R_cap, ws.img, ws.ib, ws.status,
                         notify.host_ptr if notify else None, notify.event if notify else None, lo, hi,
                         int(max_tile), _dgm_lib.stream_ptr())
    _dgm_lib.check(rc, "dgr_forward")
    return color, radii, ws


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings):
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                     cov3Ds_precomp, raster_settings)


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings):
        rs = raster_settings
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
                             first[0] if first else None, mt)
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
        ctx.save_for_backward(means3D, radii)
        ctx.mark_non_differentiable(radii)
        return color, radii

    @staticmethod
    def backward(ctx, grad_out_color, _):
        rs = ctx.raster_settings
        bg, sh, col, opac, sc, rot, cov, view, proj, campos = ctx.tensors
        means3D, radii = ctx.saved_tensors
        ws = ctx.ws
        lib = _dgm_lib.lib()
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

        dpix = _f32c(grad_out_color, "grad_out_color")
        p = _dgm_lib.ptr
        rc = lib.dgr_backward(P, rs.sh_degree, M, p(bg), W, H, p(means3D), p(sh), p(col), p(sc),
                              float(rs.scale_modifier), p(rot), p(cov), p(view), p(proj), p(campos),
                              float(rs.tanfovx), float(rs.tanfovy), p(radii), ws.geom, ws.binning, ws.R_cap, ws.img,
                              p(dpix), ptrs[0], None, ptrs[2], ptrs[3], ptrs[4], ptrs[5],
                              ptrs[8] if M else None, ptrs[6], ptrs[7], _dgm_lib.stream_ptr())
        _dgm_lib.check(rc, "dgr_backward")
        # same ordering as the reference (:143-153)
        return (gview(4, P, 3), gview(0, P, 3) if ctx.has_m2d else None,
                gview(8, P, M, 3) if sh is not None else None, gview(3, P, 3) if col is not None else None,
                gview(2, P, 1), gview(6, P, 3) if sc is not None else None,
                gview(7, P, 4) if rot is not None else None, gview(5, P, 6) if cov is not None else None, None)


_N_STREAMS = int(os.environ.get("DGMESH_B200_STREAMS", "2"))


class _BatchWorkspace:
    """F per-frame workspaces + F status blocks in one allocation (see dgr_forward_batch)."""
    __slots__ = ("buf", "geom", "binning", "img", "status", "gs", "bs", "is_", "R_cap", "F")

    def __init__(self, F, P, W, H, R_cap, dev):
        _, _, _, ga, ba, ia = _sizes(P, W, H, R_cap)
        self.buf = torch.empty((F * (ga + ba + ia) + 32 * F,), dtype=torch.uint8, device=dev)
        base = self.buf.data_ptr()
        self.geom, self.binning, self.img = base, base + F * ga, base + F * (ga + ba)
        self.status = base + F * (ga + ba + ia)
        self.gs, self.bs, self.is_, self.R_cap, self.F = ga, ba, ia, R_cap, F

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
    F = len(settings)
    tx = (_dgm_lib.c_float * F)(*[float(s.tanfovx) for s in settings])
    ty = (_dgm_lib.c_float * F)(*[float(s.tanfovy) for s in settings])
    return views, projs, cams, tx, ty


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
        views, projs, cams, tx, ty = _stack_settings(settings, dev)
        H, W = int(rs0.image_height), int(rs0.image_width)
        M = int(sh_.shape[-2]) if sh_ is not None else 0
        key = (dev.index, W, H)
        lib = _dgm_lib.lib()
        p = _dgm_lib.ptr
        first = []

        def run(R_cap, notify, lo, hi, mt):
            ws = _BatchWorkspace(F, P, W, H, R_cap, dev)
            if first:
                color, radii = first[0]
            else:
                color = torch.empty((F, 3, H, W), dtype=torch.float32, device=dev)
                radii = torch.empty((F, P), dtype=torch.int32, device=dev)
                first.append((color, radii))
            rc = lib.dgr_forward_batch(F, P, rs0.sh_degree, M, p(bg), W, H, p(means3D), p(sh_), p(col), p(opac),
                                       p(sc), float(rs0.scale_modifier), p(rot), p(cov), pf, p(views), p(projs),
                                       p(cams), tx, ty, int(bool(rs0.prefiltered)), p(color), p(radii), ws.geom, ws.gs,
                                       ws.binning, ws.bs, R_cap, ws.img, ws.is_, ws.status,
                                       notify.host_ptr if notify else None, notify.event if notify else None, lo, hi,
                                       int(mt), _N_STREAMS, _dgm_lib.stream_ptr())
            _dgm_lib.check(rc, "dgr_forward_batch")
            return color, radii, ws

        (color, radii, ws), _ = _run_sized(run, key, P, dev.index, F)
        ctx.ws, ctx.tensors, ctx.cams, ctx.settings = ws, t, (views, projs, cams, tx, ty), settings
        ctx.has_m2d = means2D is not None
        ctx.pf = pf
        ctx.save_for_backward(means3D, radii)
        ctx.mark_non_differentiable(radii)
        return color, radii

    @staticmethod
    def backward(ctx, grad_out_color, _):
        bg, sh, col, opac, sc, rot, cov = ctx.tensors
        views, projs, cams, tx, ty = ctx.cams
        means3D, radii = ctx.saved_tensors
        ws, rs0, pf = ctx.ws, ctx.settings[0], ctx.pf
        F, P = ws.F, means3D.shape[-2]
        H, W = int(rs0.image_height), int(rs0.image_width)
        M = int(sh.shape[-2]) if sh is not None else 0

        def nf(bit):
            return F if (pf & bit) else 1

        # m2d[F,P,3] opac col m3d cov scale rot sh -- per-frame inputs get F slabs
        widths = (3 * F, nf(_PF_OPAC), 3 * (nf(_PF_COLOR) if sh is None else 1), 3 * nf(_PF_MEANS),
                  6 * nf(_PF_COV), 3 * nf(_PF_SCALES), 4 * nf(_PF_ROTS), 3 * M * nf(_PF_COLOR))
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

        dpix = _f32c(grad_out_color, "grad_out_color")
        p = _dgm_lib.ptr
        rc = _dgm_lib.lib().dgr_backward_batch(
            F, P, rs0.sh_degree, M, p(bg), W, H, p(means3D), p(sh), p(col), p(sc), float(rs0.scale_modifier), p(rot),
            p(cov), pf, p(views), p(projs), p(cams), tx, ty, p(radii), ws.geom, ws.gs, ws.binning, ws.bs, ws.R_cap,
            ws.img, ws.is_, p(dpix), ptrs[0], ptrs[1], ptrs[2], ptrs[3], ptrs[4], ptrs[7] if M else None, ptrs[5],
            ptrs[6], _N_STREAMS, _dgm_lib.stream_ptr())
        _dgm_lib.check(rc, "dgr_backward_batch")
        return (gview(3, _PF_MEANS, P, 3), gview(0, 0, F, P, 3) if ctx.has_m2d else None,
                gview(7, _PF_COLOR, P, M, 3) if sh is not None else None,
                gview(2, _PF_COLOR, P, 3) if col is not None else None,
                gview(1, _PF_OPAC, P, 1), gview(5, _PF_SCALES, P, 3) if sc is not None else None,
                gview(6, _PF_ROTS, P, 4) if rot is not None else None,
                gview(4, _PF_COV, P, 6) if cov is not None else None, None)


def rasterize_gaussians_batch(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                              settings):
    return _RasterizeGaussiansBatch.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                          cov3Ds_precomp, tuple(settings))


class BatchGaussianRasterizer(nn.Module):
    """`GaussianRasterizer` for a batch of frames (one settings tuple per frame, same image size)."""

    def __init__(self, settings):
        super().__init__()
        self.settings = tuple(settings)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None):
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
