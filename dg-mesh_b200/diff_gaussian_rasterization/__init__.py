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
                                            + forward_blend_stats(...) -> (color, radii[, depth, alpha],
                                                                           blend_weight_sum, blend_weight_max)
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
import copy
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
    """The workspaces of F frames: geom | binning | img of every frame, then the F status blocks, carved from ONE
    device allocation (the three opaque buffers of the reference, dgr/rasterize_points.cu:68-78, kept together for
    the backward pass), and the normal and surface workspaces of a forward that writes those maps.  Frame f's buffers
    start f strides in (gs, bs, is_, nrm_stride, surf_stride: the sizes rounded up to 512 bytes).  The single-frame
    entry points take the exact sizes gb, bb, ib, nrm_bytes and surf_bytes; the batch ones take the strides.
    `batch`: the workspace of a batch call, whose status words have a leading frame dimension even for F = 1."""
    __slots__ = ("buf", "geom", "binning", "img", "status", "gb", "bb", "ib", "gs", "bs", "is_", "R_cap", "F", "lead",
                 "nrm", "nrm_bytes", "nrm_stride", "surf", "surf_bytes", "surf_stride")

    def __init__(self, F, P, W, H, R_cap, dev, batch=False, normal=False, surface=False):
        self.gb, self.bb, self.ib, self.gs, self.bs, self.is_ = _sizes(P, W, H, R_cap)
        self.buf = torch.empty((F * (self.gs + self.bs + self.is_ + 32),), dtype=torch.uint8, device=dev)
        base = self.buf.data_ptr()
        self.geom, self.binning, self.img = base, base + F * self.gs, base + F * (self.gs + self.bs)
        self.status = self.img + F * self.is_
        self.R_cap, self.F, self.lead = R_cap, F, ((F,) if batch else ())
        self.nrm, self.nrm_bytes, self.nrm_stride = _side_ws(F, _normal_ws_bytes(P, R_cap), dev) if normal else \
            (None, 0, 0)
        self.surf, self.surf_bytes, self.surf_stride = _side_ws(F, _surface_ws_bytes(W, H), dev) if surface else \
            (None, 0, 0)

    def status_tensor(self):
        """The status words: [8] for a single-frame call, [F,8] for a batch."""
        o = self.status - self.buf.data_ptr()
        return self.buf[o:o + 32 * self.F].view(torch.int32).view(self.lead + (8,))

    def side_args(self):
        """(geom, stride, binning, stride, R_cap, img, stride) of the passes over this forward's blend (features,
        planar depth, blend statistics); the strides are 0 for a single-frame call."""
        if self.lead:
            return self.geom, self.gs, self.binning, self.bs, self.R_cap, self.img, self.is_
        return self.geom, 0, self.binning, 0, self.R_cap, self.img, 0

    def frame(self, f):
        """Frame f of a batch as a single-frame workspace over the same allocation (for export_state)."""
        w = copy.copy(self)
        w.geom, w.binning, w.img = self.geom + f * self.gs, self.binning + f * self.bs, self.img + f * self.is_
        w.status, w.F, w.lead = self.status + 32 * f, 1, ()
        return w

    # the reference-style separate byte tensors of a single frame (views, no copies)
    def split(self):
        o1 = self.binning - self.geom
        o2 = self.img - self.geom
        return self.buf[:self.gb], self.buf[o1:o1 + self.bb], self.buf[o2:o2 + self.ib]


def _side_ws(F, nbytes, dev):
    """(buffer, nbytes, stride) of F side workspaces of nbytes each."""
    stride = (nbytes + 511) // 512 * 512
    return torch.empty((F * stride,), dtype=torch.uint8, device=dev), nbytes, stride


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


def _forward(batch, settings, means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, maps=None,
             nrm=None, surf=None, cams=None, attempt=None):
    """Enqueue the forward of the frames of `settings` (a tuple of them with `batch`, else one) through the narrowest
    dgr_forward or dgr_forward_batch variant (see `_enqueue`) that also writes
      maps: None, or the (depth, alpha) maps [1,H,W] ([F,1,H,W] with `batch`);
      nrm: None, or (normals [P,3] (with `batch` also [F,P,3] per frame), normal maps [3,H,W] / [F,3,H,W]);
      surf: None, or (near, far, median-depth maps, distortion maps), each map as the depth map.
    The Gaussian inputs are [P,.], or with `batch` [F,P,.] per frame where their rank says so.  cams: None (the
    settings' cameras), or the (viewmatrix, projmatrix, campos) tensors to use instead, stacked with `batch`.  A frame
    that did not fit the instance workspace is re-run into the outputs of the first attempt (`_run_sized`); with
    `attempt` = (R_cap, notify, depth hint lo, hi) the forward is enqueued once, as given, and R is None.
    Returns (color, radii, workspace, R of the largest frame (None under stream capture), (means3D, the other inputs
    as the library reads them (bg, sh, colors, opacities, scales, rotations, cov3D, view, proj, campos), their
    (tanfovx, tanfovy), the per-frame mask))."""
    rs0 = settings[0] if batch else settings
    F = len(settings) if batch else 1
    if batch:
        if F > _MAX_FRAMES:
            raise ValueError(f"at most {_MAX_FRAMES} frames per batch")
        for s in settings:
            if (s.image_height, s.image_width, s.sh_degree, s.scale_modifier) != \
                    (rs0.image_height, rs0.image_width, rs0.sh_degree, rs0.scale_modifier):
                raise ValueError("all frames of a batch must share image size, SH degree and scale modifier")
    means3D = _f32c(means3D, "means3D")
    if means3D is None:
        raise ValueError("means3D must have dimensions (num_points, 3)")
    bg, sh, col, opac, sc, rot, cov = (
        _f32c(rs0.bg, "bg"), _f32c(sh, "sh"), _f32c(colors_precomp, "colors_precomp"), _f32c(opacities, "opacities"),
        _f32c(scales, "scales"), _f32c(rotations, "rotations"), _f32c(cov3Ds_precomp, "cov3D_precomp"))
    pf = 0
    if batch:
        # per-frame mask from the ranks: means [F,P,3], scales [F,P,3], rotations [F,P,4], opacities [F,P,1],
        # shs [F,P,M,3] / colors [F,P,3], cov3D [F,P,6]
        for x, rank, bit in ((means3D, 3, _PF_MEANS), (sc, 3, _PF_SCALES), (rot, 3, _PF_ROTS), (opac, 3, _PF_OPAC),
                             (sh, 4, _PF_COLOR), (col, 3, _PF_COLOR), (cov, 3, _PF_COV)):
            if x is not None and x.ndim == rank:
                if x.shape[0] != F:
                    raise ValueError("per-frame inputs must have a leading dimension equal to the number of frames")
                pf |= bit
    if means3D.shape[-1] != 3 or not batch and means3D.ndim != 2:
        raise ValueError("means3D must have dimensions (num_points, 3)")  # rasterize_points.cu:57-59
    dev = means3D.device
    if cams is not None:
        view, proj, campos = (_f32c(t.detach(), n) for t, n in zip(cams, ("viewmatrix", "projmatrix", "campos")))
        tx, ty = _fovs(settings) if batch else (rs0.tanfovx, rs0.tanfovy)
    elif batch:
        view, proj, campos, tx, ty = _stack_settings(settings, dev)
    else:
        view, proj, campos = (_f32c(rs0.viewmatrix, "viewmatrix"), _f32c(rs0.projmatrix, "projmatrix"),
                              _f32c(rs0.campos, "campos"))
        tx, ty = rs0.tanfovx, rs0.tanfovy
    P = means3D.shape[-2]
    H, W = int(rs0.image_height), int(rs0.image_width)
    M = int(sh.shape[-2]) if sh is not None else 0
    lead = (F,) if batch else ()
    p = _dgm_lib.ptr
    npf = int(nrm is not None and nrm[0].ndim == 3)
    first = []

    def run(R_cap, notify, lo, hi, mt):
        ws = _Workspace(F, P, W, H, R_cap, dev, batch, nrm is not None, surf is not None)
        if not first:    # a re-run after an overflow writes the tensors of the first attempt
            first.append((torch.empty(lead + (3, H, W), dtype=torch.float32, device=dev),
                          torch.empty(lead + (P,), dtype=torch.int32, device=dev)))
        color, radii = first[0]
        note = (notify.host_ptr, notify.event) if notify else (None, None)
        nrm_ws = None if nrm is None else ws.nrm.data_ptr()
        surf_ws = None if surf is None else ws.surf.data_ptr()
        if batch:
            head = (F, P, rs0.sh_degree, M, p(bg), W, H, p(means3D), p(sh), p(col), p(opac), p(sc),
                    float(rs0.scale_modifier), p(rot), p(cov), pf, p(view), p(proj), p(campos), tx, ty,
                    int(bool(rs0.prefiltered)), p(color), p(radii))
            tail = (ws.geom, ws.gs, ws.binning, ws.bs, R_cap, ws.img, ws.is_, ws.status, *note, lo, hi, int(mt),
                    _N_STREAMS, _dgm_lib.stream_ptr())
            nrm_args = None if nrm is None else (p(nrm[0]), npf, p(nrm[1]), nrm_ws, ws.nrm_stride)
            surf_bytes = ws.surf_stride
        else:
            head = (P, rs0.sh_degree, M, p(bg), W, H, p(means3D), p(sh), p(col), p(opac), p(sc),
                    float(rs0.scale_modifier), p(rot), p(cov), p(view), p(proj), p(campos), float(tx), float(ty),
                    int(bool(rs0.prefiltered)), p(color), p(radii))
            tail = (ws.geom, ws.gb, ws.binning, ws.bb, R_cap, ws.img, ws.ib, ws.status, *note, lo, hi, int(mt),
                    _dgm_lib.stream_ptr())
            nrm_args = None if nrm is None else (p(nrm[0]), p(nrm[1]), nrm_ws, ws.nrm_bytes)
            surf_bytes = ws.surf_bytes
        _enqueue("dgr_forward_batch" if batch else "dgr_forward", (
            (None, head), ("_aux", None if maps is None else (p(maps[0]), p(maps[1]))), ("_nrm", nrm_args),
            ("_surf", None if surf is None else (float(surf[0]), float(surf[1]), p(surf[2]), p(surf[3]), surf_ws,
                                                 surf_bytes)),
            (None, tail)))
        return color, radii, ws

    if attempt is not None:
        (color, radii, ws), R = run(*attempt, 0), None
    else:
        (color, radii, ws), R = _run_sized(run, (dev.index, W, H), P, dev.index, F)
    return color, radii, ws, R, (means3D, (bg, sh, col, opac, sc, rot, cov, view, proj, campos), (tx, ty), pf)


def _raw_forward(bg, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix,
                 projmatrix, tan_fovx, tan_fovy, H, W, sh, degree, campos, prefiltered, R_cap, notify=None, lo=0.0,
                 hi=0.0):
    """One enqueue of dgr_forward, in the reference's argument order, with capacity R_cap and the depth-range hint
    (lo, hi), and no re-run when a frame overflows: (color, radii, workspace)."""
    rs = GaussianRasterizationSettings(H, W, tan_fovx, tan_fovy, bg, scale_modifier, viewmatrix, projmatrix, degree,
                                       campos, prefiltered, False)
    color, radii, ws, _, _ = _forward(False, rs, means3D, sh, colors, opacity, scales, rotations, cov3D_precomp,
                                      attempt=(R_cap, notify, lo, hi))
    return color, radii, ws


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings):
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                     cov3Ds_precomp, raster_settings)


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings):
        return _fwd(ctx, False, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                    raster_settings)

    @staticmethod
    def backward(ctx, grad_out_color, _):
        return _bwd(ctx, grad_out_color)   # its last entry, dL/dnormals, is None here


class _CameraGrads:
    """Outputs and scratch of the camera gradients of F frames: [F,16] view, [F,16] proj, [F,3] campos and [F,2]
    tan(fov/2) (one allocation; need: which of the four are needed, a gradient no camera tensor needs is passed to
    the library as NULL)."""

    def __init__(self, F, P, dev, need):
        n = _dgm_lib.c_size_t()
        _dgm_lib.check(_dgm_lib.lib().dgr_camera_grad_workspace_size(F, P, _dgm_lib.byref(n)),
                       "dgr_camera_grad_workspace_size")
        self.out = torch.empty((37 * F + (n.value + 3) // 4,), dtype=torch.float32, device=dev)
        self.F, self.need, self.ws_bytes = F, need, n.value
        self.view = self.out[:16 * F].view(F, 16)
        self.proj = self.out[16 * F:32 * F].view(F, 16)
        self.campos = self.out[32 * F:35 * F].view(F, 3)
        self.tanfov = self.out[35 * F:37 * F].view(F, 2)

    def args(self):
        """(dL_dviewmatrix, dL_dprojmatrix, dL_dcampos, cam_ws, cam_ws_bytes) of dgr_backward{,_batch}_cam."""
        outs = [t.data_ptr() if need else None for t, need in zip((self.view, self.proj, self.campos), self.need)]
        return (*outs, self.out[37 * self.F:].data_ptr(), self.ws_bytes)

    def intr_args(self):
        """(dL_dtanfov,) of dgr_backward{,_batch}_intr, or None when no tan(fov/2) gradient is needed."""
        return (self.tanfov.data_ptr(),) if self.need[3] else None

    def grads(self, shapes):
        """The gradients in the shapes of the camera tensors (None where none is needed)."""
        return tuple(g.reshape(shape) if need else None
                     for g, shape, need in zip((self.view, self.proj, self.campos, self.tanfov), shapes, self.need))


_N_STREAMS = int(os.environ.get("DGMESH_B200_STREAMS", "2"))


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
_PF_MEAN2D = 64     # the screen-space gradients of a batch, which are per frame whatever the inputs are

# The gradient outputs of the backward entry points, in each one's argument order: (slot, floats per Gaussian (per SH
# coefficient for dL_dsh), per-frame bit, whether the entry requires it).  The slot is the output's place in the one
# gradient allocation.  An output the entry does not require is passed as NULL unless its input is given.  Like the
# reference's, dgr_backward takes every output but dL_dconic (not materialised) and dL_dsh; the batch entry points
# also skip dL_dcolor and dL_dcov3D when they are not returned.
_M2D, _CONIC, _OPAC, _COL, _M3D, _COV, _SCALE, _ROT, _SH = range(9)
_BWD_GRADS = ((_M2D, 3, 0, True), (_CONIC, 0, 0, False), (_OPAC, 1, _PF_OPAC, True), (_COL, 3, _PF_COLOR, True),
              (_M3D, 3, _PF_MEANS, True), (_COV, 6, _PF_COV, True), (_SH, 3, _PF_COLOR, False),
              (_SCALE, 3, _PF_SCALES, True), (_ROT, 4, _PF_ROTS, True))
_BWD_BATCH_GRADS = ((_M2D, 3, _PF_MEAN2D, True), (_OPAC, 1, _PF_OPAC, True), (_COL, 3, _PF_COLOR, False),
                    (_M3D, 3, _PF_MEANS, True), (_COV, 6, _PF_COV, False), (_SH, 3, _PF_COLOR, False),
                    (_SCALE, 3, _PF_SCALES, True), (_ROT, 4, _PF_ROTS, True))
_REFERENCE_ORDER = (_M3D, _M2D, _SH, _COL, _OPAC, _SCALE, _ROT, _COV)     # the reference's gradient tuple (:143-153)


def _fwd(ctx, batch, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, settings,
         maps=None, nrm=None, surf=None, cams=None, saved=()):
    """Forward of the rasterizer Functions: `_forward`, and what the backward needs kept in ctx.  saved: more
    tensors to save for the backward, after (means3D, radii)."""
    color, radii, ws, _, (means3D, ctx.tensors, ctx.fovs, ctx.pf) = _forward(
        batch, settings, means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, maps, nrm, surf,
        cams)
    if not batch and settings.debug:
        torch.cuda.current_stream().synchronize()   # the reference's debug mode checks after every kernel
    ctx.raster_settings = settings[0] if batch else settings
    ctx.ws = ws
    ctx.has_m2d = means2D is not None
    ctx.normals_pf = int(nrm is not None and nrm[0].ndim == 3)
    ctx.save_for_backward(means3D, radii, *saved)
    ctx.mark_non_differentiable(radii)
    return color, radii


def _grads(table, given, frames, F, P, M, dev):
    """The gradient outputs of `table` (_BWD_GRADS) in one allocation, each sub-buffer 16-byte aligned for vector
    stores: the outputs the entry requires or whose input is `given` (by slot), with F slabs where `frames` has
    their per-frame bit.  Returns (their pointers in argument order, NULL where there is none, the gradient of each
    given slot as a view, None elsewhere)."""
    offs, o = [None] * 9, 0
    for slot, w, bit, required in sorted(table):    # the sub-buffers in slot order
        if required or given[slot]:
            offs[slot] = o
            o = (o + P * w * (M if slot == _SH else 1) * (F if frames & bit else 1) + 3) // 4 * 4
    flat = torch.empty((max(o, 1),), dtype=torch.float32, device=dev)
    base = flat.data_ptr()
    ptrs = tuple([None if offs[slot] is None else base + 4 * offs[slot] for slot, _, _, _ in table])
    views = [None] * 9
    for slot, w, bit, _ in table:
        if given[slot]:     # one as_strided per gradient (slice + view cost twice as much on the host)
            shape, stride = ((P, M, 3), (3 * M, 3, 1)) if slot == _SH else ((P, w), (w, 1))
            if frames & bit:
                shape, stride = (F,) + shape, (P * stride[0],) + stride
            views[slot] = flat.as_strided(shape, stride, offs[slot])
    return ptrs, views


def _bwd(ctx, grad_out_color, grad_depth=None, grad_alpha=None, cam=None, nrm=None, surf=None, abs_out=None):
    """Backward of the rasterizer Functions through dgr_backward or dgr_backward_batch, the narrowest variant that
    takes every segment in use (`_enqueue`).  The upstream gradients are shaped as the forward's outputs.
    grad_depth / grad_alpha: None, or the upstream gradients of the maps (None = unused by the loss).
    cam: None, or the _CameraGrads the backward writes the camera (and intrinsics) gradients to.
    nrm: None, or (upstream gradient of the normal map, whether dL/dnormals is needed).
    surf: None, or (near, far, upstream gradients of the median-depth and distortion maps, each None when unused, not
    both).
    abs_out: None, or the [P,3] ([F,P,3] for a batch) tensor the backward writes the absolute screen-space gradient to.
    Returns the eight Gaussian inputs' gradients in the reference's order (a per-frame input's with a leading F),
    then dL/dnormals [P,3] ([F,P,3] for per-frame normals), or None."""
    rs = ctx.raster_settings
    bg, sh, col, opac, sc, rot, cov, view, proj, campos = ctx.tensors
    tx, ty = ctx.fovs
    means3D, radii = ctx.saved_tensors[:2]
    ws, pf, npf = ctx.ws, ctx.pf, ctx.normals_pf
    batch, F, P, dev = bool(ws.lead), ws.F, means3D.shape[-2], means3D.device
    H, W = int(rs.image_height), int(rs.image_width)
    M = int(sh.shape[-2]) if sh is not None else 0
    given = (ctx.has_m2d, False, True, col is not None, True, cov is not None, sc is not None, rot is not None,
             sh is not None)    # by slot: means2D, conic, opacities, colours, means3D, cov3D, scales, rotations, SH
    grads, views = _grads(_BWD_BATCH_GRADS if batch else _BWD_GRADS, given, (pf | _PF_MEAN2D) if batch else 0, F, P,
                          M, dev)
    if grad_out_color is None:    # a depth / alpha loss only
        grad_out_color = torch.zeros(ws.lead + (3, H, W), dtype=torch.float32, device=dev)
    dpix = _f32c(grad_out_color, "grad_out_color")
    p = _dgm_lib.ptr
    aux = gn = surf_args = dnormals = None
    if grad_depth is not None or grad_alpha is not None:
        aux = (p(_f32c(grad_depth, "grad_depth")), p(_f32c(grad_alpha, "grad_alpha")))
    if nrm is not None:
        if nrm[1]:
            dnormals = torch.empty((F, P, 3) if npf else (P, 3), dtype=torch.float32, device=dev)
        gn = p(_f32c(nrm[0], "grad_normal"))
    if surf is not None:
        surf_args = (float(surf[0]), float(surf[1]), p(_f32c(surf[2], "grad_median_depth")),
                     p(_f32c(surf[3], "grad_distortion")), ws.surf.data_ptr())
    if batch:
        head = (F, P, rs.sh_degree, M, p(bg), W, H, p(means3D), p(sh), p(col), p(sc), float(rs.scale_modifier),
                p(rot), p(cov), pf, p(view), p(proj), p(campos), tx, ty, p(radii), ws.geom, ws.gs, ws.binning, ws.bs,
                ws.R_cap, ws.img, ws.is_, p(dpix))
        tail = (_N_STREAMS, _dgm_lib.stream_ptr())
        nrm_args = None if nrm is None else (gn, npf, p(dnormals), ws.nrm.data_ptr(), ws.nrm_stride)
        surf_args = None if surf is None else surf_args + (ws.surf_stride,)
    else:
        head = (P, rs.sh_degree, M, p(bg), W, H, p(means3D), p(sh), p(col), p(sc), float(rs.scale_modifier), p(rot),
                p(cov), p(view), p(proj), p(campos), float(tx), float(ty), p(radii), ws.geom, ws.binning, ws.R_cap,
                ws.img, p(dpix))
        tail = (_dgm_lib.stream_ptr(),)
        nrm_args = None if nrm is None else (gn, p(dnormals), ws.nrm.data_ptr())
    _enqueue("dgr_backward_batch" if batch else "dgr_backward", (
        (None, head), ("_aux", aux), (None, grads), ("_cam", None if cam is None else cam.args()), ("_nrm", nrm_args),
        ("_surf", surf_args), ("_abs", None if abs_out is None else (p(abs_out),)),
        ("_intr", None if cam is None else cam.intr_args()), (None, tail)))
    return tuple([views[slot] for slot in _REFERENCE_ORDER]) + (dnormals,)


class _RasterizeGaussiansBatch(torch.autograd.Function):
    """F frames in one call: colors [F,3,H,W], radii [F,P].

    Every Gaussian input may be SHARED ([P,.] -- its gradient is the sum over frames, accumulated
    inside the kernels) or PER FRAME (a leading F dimension, [F,P,.] -- its gradient is [F,P,.]).
    DG-Mesh's dynamic scenes deform means / scales / rotations by the frame's time
    (gaussian_renderer/__init__.py:60-86), so those arrive per frame while opacity and SH are shared.
    means2D, if given as an [F,P,3] tensor, receives the per-frame screen-space gradients."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, settings):
        return _fwd(ctx, True, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                    settings)

    @staticmethod
    def backward(ctx, grad_out_color, _):
        return _bwd(ctx, grad_out_color)   # its last entry, dL/dnormals, is None here


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


def _features_fwd(ws, st, W, H, fmap):
    """dgr_features_fwd over the blend of the forward that wrote `ws`: fmap [F,C,H,W] (or [C,H,W])."""
    P = st.feats.shape[-2]
    _dgm_lib.check(_dgm_lib.lib().dgr_features_fwd(st.F, P, st.C, W, H, st.feats.data_ptr(), st.per_frame,
                                                   *ws.side_args(), fmap.data_ptr(), st.buf.data_ptr(), st.buf.numel(),
                                                   _dgm_lib.stream_ptr()), "dgr_features_fwd")


def _features_bwd(ws, st, W, H, fmap, grad, need):
    """dgr_features_bwd: adds the feature loss's share to the forward's accumulators (the rasterizer backward that
    follows carries it on) and returns dL/dfeatures (None when not `need`ed)."""
    P = st.feats.shape[-2]
    g = _f32c(grad, "grad_features")
    dfeat = torch.empty(st.feats.shape, dtype=torch.float32, device=st.feats.device) if need else None
    _dgm_lib.check(_dgm_lib.lib().dgr_features_bwd(st.F, P, st.C, W, H, st.feats.data_ptr(), st.per_frame,
                                                   *ws.side_args(), fmap.data_ptr(), g.data_ptr(), _dgm_lib.ptr(dfeat),
                                                   st.buf.data_ptr(), st.buf.numel(), _dgm_lib.stream_ptr()),
                   "dgr_features_bwd")
    return dfeat


def _check_pixel_weights(weights, H, W, F=None):
    """(pixel_weights as a float32 CUDA tensor, whether it is per frame): [H,W] or [1,H,W] shared by the frames, or,
    with F, [F,H,W] or [F,1,H,W] per frame."""
    shared = ((H, W), (1, H, W))
    per_frame = () if F is None else ((F, H, W), (F, 1, H, W))
    shape = tuple(weights.shape) if torch.is_tensor(weights) else None
    if shape not in shared + per_frame or weights.dtype != torch.float32:
        shapes = "(H, W) or (1, H, W)" + (" or (num_frames, H, W) or (num_frames, 1, H, W)" if F is not None else "")
        raise ValueError(f"pixel_weights must be a float32 tensor of dimensions {shapes}")
    return _f32c(weights, "pixel_weights"), int(shape not in shared)


def _blend_stats(ws, P, W, H, F, weights):
    """dgr_blend_stats over the blend of the forward that wrote `ws`: (blend_weight_sum, blend_weight_max), [P] for
    one frame (F None) or [F,P].  weights: None, or what _check_pixel_weights returns."""
    shape = (P,) if F is None else (F, P)
    out_sum, out_max = (torch.empty(shape, dtype=torch.float32, device=ws.buf.device) for _ in range(2))
    w, per_frame = (None, 0) if weights is None else weights
    _, _, binning, bs, R_cap, img, is_ = ws.side_args()
    _dgm_lib.check(_dgm_lib.lib().dgr_blend_stats(F or 1, P, W, H, binning, bs, R_cap, img, is_, _dgm_lib.ptr(w),
                                                  per_frame, out_sum.data_ptr(), out_max.data_ptr(),
                                                  _dgm_lib.stream_ptr()), "dgr_blend_stats")
    return out_sum, out_max


def _check_normals(normals, P, F=None):
    """normals as a float32 CUDA tensor [P,3] (or, with F, [P,3] shared by the frames or [F,P,3] per frame)."""
    n = _f32c(normals, "normals")
    if F is None:
        if n is None or n.shape != (P, 3):
            raise ValueError("normals must have dimensions (num_points, 3)")
    elif n is None or n.shape not in ((P, 3), (F, P, 3)):
        raise ValueError("normals must have dimensions (num_points, 3) or (num_frames, num_points, 3)")
    return n


def _camera_needs_grad(settings):
    """Whether any camera tensor of `settings` (one, or a tuple) requires grad."""
    sets = (settings,) if isinstance(settings, GaussianRasterizationSettings) else tuple(settings)
    return any(torch.is_tensor(t) and t.requires_grad
               for s in sets for t in (s.viewmatrix, s.projmatrix, s.campos, s.tanfovx, s.tanfovy))


class _GaussianPlanes(torch.autograd.Function):
    """dgr_gaussian_planes_fwd / _bwd: (means3D, scales, rotations, cov3D_precomp, settings tuple, per_frame) ->
    (planes, normals) [F,P,3]."""

    @staticmethod
    def forward(ctx, means3D, scales, rotations, cov3D_precomp, settings, per_frame):
        F, P = len(settings), means3D.shape[-2]
        rs0 = settings[0]
        m, sc, rot, cov = (_f32c(t, n) for t, n in ((means3D, "means3D"), (scales, "scales"),
                                                     (rotations, "rotations"), (cov3D_precomp, "cov3D_precomp")))
        view = torch.stack([_f32c(s.viewmatrix, "viewmatrix").reshape(16) for s in settings]).contiguous()
        fx, fy = _fovs(settings)
        planes, normals = (torch.empty((F, P, 3), dtype=torch.float32, device=m.device) for _ in range(2))
        p = _dgm_lib.ptr
        ctx.head = (F, P, int(rs0.image_width), int(rs0.image_height), p(m), p(sc), float(rs0.scale_modifier), p(rot),
                    p(cov), per_frame, p(view), fx, fy)
        _dgm_lib.check(_dgm_lib.lib().dgr_gaussian_planes_fwd(*ctx.head, p(planes), p(normals),
                                                              _dgm_lib.stream_ptr()), "dgr_gaussian_planes_fwd")
        ctx.keep = (m, sc, rot, cov, view)   # the head's pointers stay valid through the backward
        ctx.set_materialize_grads(False)
        return planes, normals

    @staticmethod
    def backward(ctx, grad_planes, grad_normals):
        m, sc, rot, cov, _ = ctx.keep
        need = ctx.needs_input_grad[:4]
        out = tuple(torch.empty(t.shape, dtype=torch.float32, device=m.device) if t is not None and n else None
                    for t, n in zip((m, sc, rot, cov), need))
        if grad_planes is None and grad_normals is None:
            return tuple(None if o is None else o.zero_() for o in out) + (None, None)
        p = _dgm_lib.ptr
        _dgm_lib.check(_dgm_lib.lib().dgr_gaussian_planes_bwd(
            *ctx.head, p(_f32c(grad_planes, "grad_planes")), p(_f32c(grad_normals, "grad_normals")),
            *map(p, out), _dgm_lib.stream_ptr()), "dgr_gaussian_planes_bwd")
        return out + (None, None)


def gaussian_planes(means3D, raster_settings, scales=None, rotations=None, cov3D_precomp=None):
    """Each Gaussian's depth plane in the camera of `raster_settings` (one GaussianRasterizationSettings, or a
    sequence of them for a batch): planes (t_z, g_u, g_v) and camera-space plane normals, [P,3] each for one
    settings and [F,P,3] for a sequence.  The depth that Gaussian i paints at pixel centre p is
    t_z + g . (p - mu2D_i), mu2D_i its screen mean; n faces the camera (see include/dgmesh_b200.h, "Planar depth",
    for the definition).  Give scales + rotations, or cov3D_precomp, as the rasterizer takes them; for a batch each
    is [P,.] shared by the frames (its gradient the sum over the frames) or [F,P,.] per frame.  Differentiable in
    the Gaussian inputs; the camera is not: a camera tensor that requires grad raises ValueError."""
    batch = not isinstance(raster_settings, GaussianRasterizationSettings)
    sets = tuple(raster_settings) if batch else (raster_settings,)
    if _camera_needs_grad(sets):
        raise ValueError("gaussian_planes: no camera gradient is formed through the planes")
    sets = _host_fovs(sets, True)[0]
    F = len(sets)
    if (scales is None or rotations is None) == (cov3D_precomp is None):
        raise ValueError("gaussian_planes: give scales and rotations, or cov3D_precomp")
    if not torch.is_tensor(means3D) or means3D.ndim not in (2, 3) or means3D.shape[-1] != 3:
        raise ValueError("means3D must have dimensions (num_points, 3)" + (" or (num_frames, num_points, 3)" if batch
                                                                          else ""))
    P = means3D.shape[-2]
    per_frame = 0
    for t, bit, w, name in ((means3D, _PF_MEANS, 3, "means3D"), (scales, _PF_SCALES, 3, "scales"),
                            (rotations, _PF_ROTS, 4, "rotations"), (cov3D_precomp, _PF_COV, 6, "cov3D_precomp")):
        if t is None:
            continue
        if tuple(t.shape) == (F, P, w) and batch:
            per_frame |= bit
        elif tuple(t.shape) != (P, w):
            raise ValueError(f"{name} must have dimensions (num_points, {w})" +
                             (f" or (num_frames, num_points, {w})" if batch else ""))
    planes, normals = _GaussianPlanes.apply(means3D, scales, rotations, cov3D_precomp, sets, per_frame)
    return (planes, normals) if batch else (planes[0], normals[0])


class _PlanarState:
    """What the planar pass keeps for its backward: the planes and the planar workspace (dgr_planar_workspace_size
    bytes: the per-Gaussian plane accumulators and the per-pixel median records of every frame)."""
    __slots__ = ("planes", "buf", "F")

    def __init__(self, planes, F, W, H, dev):
        self.planes, self.F = planes, F
        n = _dgm_lib.c_size_t()
        _dgm_lib.check(_dgm_lib.lib().dgr_planar_workspace_size(planes.shape[-2], W, H, F, _dgm_lib.byref(n)),
                       "dgr_planar_workspace_size")
        self.buf = torch.empty((max(n.value, 16),), dtype=torch.uint8, device=dev)


def _check_planes(planes, P, F=None):
    """planes as a float32 CUDA tensor [P,3] (or, with F, [F,P,3])."""
    pl = _f32c(planes, "planes")
    shape = (P, 3) if F is None else (F, P, 3)
    if pl is None or tuple(pl.shape) != shape:
        raise ValueError(f"planes must have dimensions {shape}")
    return pl


# the outputs of the maps Functions, in order; a map the request does not ask for is None
_MAPS = ("color", "radii", "depth", "alpha", "median_depth", "distortion", "normal", "features", "blend_weight_sum",
         "blend_weight_max", "planar_depth", "planar_median_depth")


def _maps_forward(ctx, batch, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                  normals, features, planes, viewmatrix, projmatrix, campos, tanfov, means2D_abs, settings, request):
    """Forward of the maps Functions (F frames when `batch`): the outputs of _MAPS."""
    ctx.set_materialize_grads(False)
    depth_alpha, surface, stats = request
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
    pst = pmaps = None
    if planes is not None:
        pst = _PlanarState(_check_planes(planes, P, F), F or 1, W, H, dev)
        pmaps = (new_map(1), new_map(1))
    cams = None if viewmatrix is None else (viewmatrix, projmatrix, campos)
    saved = (() if fmap is None else (fmap,)) + (() if pmaps is None else (pmaps[0],))
    color, radii = _fwd(ctx, batch, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        settings, maps, nrm, surf, cams, saved)
    if st is not None:
        _features_fwd(ctx.ws, st, W, H, fmap)
    if pst is not None:
        _dgm_lib.check(_dgm_lib.lib().dgr_planar_fwd(pst.F, P, W, H, pst.planes.data_ptr(), *ctx.ws.side_args(),
                                                     pmaps[0].data_ptr(), pmaps[1].data_ptr(), pst.buf.data_ptr(),
                                                     pst.buf.numel(), _dgm_lib.stream_ptr()), "dgr_planar_fwd")
    bstats = (None, None)
    if stats is not None:
        bstats = _blend_stats(ctx.ws, P, W, H, F, stats[0])
        ctx.mark_non_differentiable(radii, *bstats)
    ctx.feat, ctx.surface, ctx.frames, ctx.planar = st, surface, F or 1, pst
    ctx.cam_shapes = None if cams is None else tuple(t.shape for t in cams) + (None if tanfov is None else tanfov.shape,)
    return (color, radii) + (maps or (None, None)) + (surf[2:] if surf else (None, None)) + \
        (None if nrm is None else nrm[1], fmap) + bstats + (pmaps or (None, None))


def _maps_backward(ctx, grad_color, _, grad_depth, grad_alpha, grad_median, grad_dist, grad_normal, grad_features,
                   _bsum, _bmax, grad_pdepth, grad_pmedian):
    """Backward of the maps Functions: the feature and planar passes first (they add to the forward's accumulators),
    then the rasterizer backward with the segments the upstream gradients use."""
    *_, need_normals, need_features, need_planes, need_view, need_proj, need_campos, need_tanfov, need_abs, _, _ = \
        ctx.needs_input_grad
    means3D = ctx.saved_tensors[0]
    dfeat = dplanes = None
    if grad_features is not None:
        fmap = ctx.saved_tensors[2]
        dfeat = _features_bwd(ctx.ws, ctx.feat, fmap.shape[-1], fmap.shape[-2], fmap, grad_features, need_features)
    if grad_pdepth is not None or grad_pmedian is not None:
        pst = ctx.planar
        pdepth = ctx.saved_tensors[-1]
        H, W = pdepth.shape[-2:]
        dplanes = torch.empty(pst.planes.shape, dtype=torch.float32, device=means3D.device) if need_planes else None
        p = _dgm_lib.ptr
        _dgm_lib.check(_dgm_lib.lib().dgr_planar_bwd(
            pst.F, means3D.shape[-2], W, H, pst.planes.data_ptr(), *ctx.ws.side_args(), pdepth.data_ptr(),
            p(_f32c(grad_pdepth, "grad_planar_depth")), p(_f32c(grad_pmedian, "grad_planar_median_depth")),
            p(dplanes), pst.buf.data_ptr(), pst.buf.numel(), _dgm_lib.stream_ptr()), "dgr_planar_bwd")
    need = (need_view, need_proj, need_campos, need_tanfov)
    cam = _CameraGrads(ctx.frames, means3D.shape[-2], means3D.device, need) if any(need) else None
    ab = torch.empty(ctx.abs_shape, dtype=torch.float32, device=means3D.device) if need_abs else None
    nrm = None if grad_normal is None else (grad_normal, need_normals)
    surf = None if grad_median is None and grad_dist is None else (*ctx.surface, grad_median, grad_dist)
    g = _bwd(ctx, grad_color, grad_depth, grad_alpha, cam, nrm, surf, ab)
    return g + (dfeat, dplanes) + (cam.grads(ctx.cam_shapes) if cam else (None,) * 4) + (ab, None, None)


class _RasterizeGaussiansMaps(torch.autograd.Function):
    """`_RasterizeGaussians` + the maps a request asks for.  Inputs: the eight Gaussian tensors of
    `_RasterizeGaussians`; normals [P,3] for the normal map sum_i n_i alpha_i T_i [3,H,W] and features [P,C] for the
    feature map [C,H,W] (each None when not asked for); viewmatrix [4,4], projmatrix [4,4] and campos [3], which
    replace the settings' tensors and receive gradients (None: the settings' camera, no camera gradient); tanfov [2],
    (tan_fovx, tan_fovy) whose values the settings already carry as floats and which receives the gradient through
    the EWA covariance (or None);
    means2D_abs [P,3], whose gradient is the absolute screen-space gradient (or None); the settings; the request
    (depth_alpha: the depth map sum_i d_i alpha_i T_i and the alpha map 1 - T_final [1,H,W]; (near, far) for the
    median-depth and distortion maps [1,H,W], or None; None, or (pixel weights, per frame) from _check_pixel_weights
    or (None,) for the blend-weight statistics [P]).  Outputs: _MAPS.  Normals, surface maps and features need
    depth_alpha; the feature map and the statistics are passes over the forward's workspaces (dgr_features_fwd /
    _bwd, dgr_blend_stats), and the statistics are not differentiable.  Gradients are
    not materialised: a map the loss does not use reaches the library as NULL, and the backward calls the narrowest
    entry point the loss needs."""

    @staticmethod
    def forward(ctx, *inputs):
        return _maps_forward(ctx, False, *inputs)

    @staticmethod
    def backward(ctx, *grads):
        return _maps_backward(ctx, *grads)


class _RasterizeGaussiansBatchMaps(torch.autograd.Function):
    """`_RasterizeGaussiansMaps` for F frames over `_RasterizeGaussiansBatch`: the settings are a tuple, every map
    has a leading F dimension, normals and features are [P,.] shared by the frames (their gradient the sum over the
    frames) or [F,P,.] per frame, the cameras [F,4,4], [F,4,4], [F,3], tanfov [F,2] and means2D_abs [F,P,3]."""

    @staticmethod
    def forward(ctx, *inputs):
        return _maps_forward(ctx, True, *inputs)

    @staticmethod
    def backward(ctx, *grads):
        return _maps_backward(ctx, *grads)


def rasterize_gaussians_batch(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                              settings):
    return _RasterizeGaussiansBatch.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                          cov3Ds_precomp, tuple(settings))


class _DepthNormal(torch.autograd.Function):
    """The normals of the surface the rendered depth describes, dgr_depth_normal_fwd / _bwd: depth, alpha and
    median [F,H,W] float32 CUDA tensors (None where depth_ratio does not read them), coefs [F,4] the frames' ray
    coefficients (a float32 CPU tensor), depth_ratio in [0, 1] -> camera-space normals [F,3,H,W]."""

    @staticmethod
    def forward(ctx, depth, alpha, median, coefs, depth_ratio):
        maps = tuple(_f32c(t, n) for t, n in ((depth, "depth"), (alpha, "alpha"), (median, "median_depth")))
        F, H, W = next(t for t in maps if t is not None).shape
        out = torch.empty((F, 3, H, W), dtype=torch.float32, device=next(t for t in maps if t is not None).device)
        _dgm_lib.check(_dgm_lib.lib().dgr_depth_normal_fwd(F, W, H, depth_ratio, *map(_dgm_lib.ptr, maps),
                                                           coefs.data_ptr(), out.data_ptr(), _dgm_lib.stream_ptr()),
                       "dgr_depth_normal_fwd")
        ctx.save_for_backward(*maps)
        ctx.coefs, ctx.depth_ratio = coefs, depth_ratio
        return out

    @staticmethod
    def backward(ctx, grad_normal):
        maps = ctx.saved_tensors
        F, H, W = next(t for t in maps if t is not None).shape
        grads = tuple(torch.empty_like(t) if need else None for t, need in zip(maps, ctx.needs_input_grad[:3]))
        if any(g is not None for g in grads):
            g = _f32c(grad_normal, "grad_normal")
            _dgm_lib.check(_dgm_lib.lib().dgr_depth_normal_bwd(F, W, H, ctx.depth_ratio, *map(_dgm_lib.ptr, maps),
                                                               ctx.coefs.data_ptr(), g.data_ptr(),
                                                               *map(_dgm_lib.ptr, grads), _dgm_lib.stream_ptr()),
                           "dgr_depth_normal_bwd")
        return grads + (None, None)


def _exclusive_inputs(shs, colors_precomp, scales, rotations, cov3D_precomp):
    """The reference's argument-exclusivity errors (:191-195); absent inputs become empty tensors."""
    if (shs is None) == (colors_precomp is None):
        raise Exception('Please provide excatly one of either SHs or precomputed colors!')
    if ((scales is None or rotations is None) and cov3D_precomp is None) or \
            ((scales is not None or rotations is not None) and cov3D_precomp is not None):
        raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
    e = torch.Tensor([])
    return (e if shs is None else shs, e if colors_precomp is None else colors_precomp, e if scales is None else scales,
            e if rotations is None else rotations, e if cov3D_precomp is None else cov3D_precomp)


def _host_fovs(settings, batch=False, grad=False):
    """`settings` (a tuple of them with `batch`) whose tanfovx / tanfovy tensors are replaced by their values, read
    in one device-to-host copy, and the [2] ([F,2] with `batch`) tensor of (tanfovx, tanfovy) that takes their
    gradient when `grad` and one of them requires grad (else None).  Settings with float fields come back as they
    are."""
    sets = tuple(settings) if batch else (settings,)
    tensors = [t for s in sets for t in (s.tanfovx, s.tanfovy) if torch.is_tensor(t)]
    if not tensors:
        return settings, None
    if any(t.ndim != 0 or not t.is_floating_point() for t in tensors):
        raise ValueError("tanfovx / tanfovy must be floats or 0-dim floating-point tensors")
    dev = tensors[0].device
    fov = torch.stack([torch.stack([torch.as_tensor(t, dtype=torch.float32, device=dev)
                                    for t in (s.tanfovx, s.tanfovy)]) for s in sets])
    values = fov.detach().cpu().tolist()
    out = tuple(s._replace(tanfovx=x, tanfovy=y) for s, (x, y) in zip(sets, values))
    tanfov = (fov if batch else fov[0]) if grad and fov.requires_grad else None
    return (out if batch else out[0]), tanfov


def _request_maps(plain, function, settings, cams, means3D, means2D, opacities, shs, colors_precomp, scales,
                  rotations, cov3D_precomp, depth_alpha, normals, surface, features, means2D_abs, blend_stats=False,
                  pixel_weights=None, planes=None):
    """The rasterizers' `_maps`: the reference-shaped `plain` Function when only colour is asked for, else the maps
    `function`; the outputs by name, in _MAPS order, without the maps not asked for."""
    if planes is not None and (cams[0] is not None or _camera_needs_grad(settings)):
        raise ValueError("planar depth: no camera gradient is formed through the planes")
    if planes is not None and means2D_abs is not None:
        # the planar pass adds its dL/dalpha in a pass of its own, as the feature pass does
        raise ValueError("abs_grad: the absolute screen-space gradient is not available with planar depth")
    if features is not None and means2D_abs is not None:
        # the feature pass adds its dL/dalpha in a pass of its own, so no per-pixel total exists to take |.| of
        raise ValueError("abs_grad: the absolute screen-space gradient is not available with feature or flow maps")
    stats = None
    if blend_stats:
        batch = function is _RasterizeGaussiansBatchMaps
        rs0 = settings[0] if batch else settings
        stats = (None if pixel_weights is None else
                 _check_pixel_weights(pixel_weights, int(rs0.image_height), int(rs0.image_width),
                                      len(settings) if batch else None),)
    elif pixel_weights is not None:
        raise ValueError("pixel_weights weight the blend-weight statistics: pass blend_stats=True")
    sh, col, sc, rot, cov = _exclusive_inputs(shs, colors_precomp, scales, rotations, cov3D_precomp)
    settings, tanfov = _host_fovs(settings, function is _RasterizeGaussiansBatchMaps, cams[0] is not None)
    depth_alpha = bool(depth_alpha) or normals is not None or surface is not None or features is not None or \
        planes is not None
    if not depth_alpha and cams[0] is None and tanfov is None and means2D_abs is None and stats is None:
        color, radii = plain.apply(means3D, means2D, sh, col, opacities, sc, rot, cov, settings)
        return {"color": color, "radii": radii}
    surface = None if surface is None else (float(surface[0]), float(surface[1]))
    out = function.apply(means3D, means2D, sh, col, opacities, sc, rot, cov, normals, features, planes, *cams, tanfov,
                         means2D_abs, settings, (depth_alpha, surface, stats))
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
        sh, col, sc, rot, cov = _exclusive_inputs(shs, colors_precomp, scales, rotations, cov3D_precomp)
        return rasterize_gaussians_batch(means3D, means2D, sh, col, opacities, sc, rot, cov,
                                         _host_fovs(self.settings, True)[0])

    def _maps(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
              cov3D_precomp=None, depth_alpha=False, normals=None, surface=None, features=None, camera_grad=False,
              means2D_abs=None, blend_stats=False, pixel_weights=None, planes=None):
        """Every frame's outputs by name, in _MAPS order: "color" and "radii"; "depth" and "alpha" with depth_alpha
        or any other map; "median_depth" and "distortion" with surface = (near, far); "normal" with normals ([P,3]
        or [F,P,3]); "features" with features ([P,C] or [F,P,C]); "blend_weight_sum" and "blend_weight_max" [F,P]
        with blend_stats, weighted by pixel_weights (see `forward_blend_stats`).  camera_grad: the frames' camera
        tensors receive gradients.  means2D_abs: see `forward` (not with features)."""
        cams = (None, None, None)
        if camera_grad:
            cams = tuple(torch.stack([getattr(s, k) for s in self.settings])
                         for k in ("viewmatrix", "projmatrix", "campos"))
        return _request_maps(_RasterizeGaussiansBatch, _RasterizeGaussiansBatchMaps, self.settings, cams, means3D,
                             means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp, depth_alpha,
                             normals, surface, features, means2D_abs, blend_stats, pixel_weights, planes)

    def forward_planar(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                       cov3D_precomp=None, plane_normals=False):
        """`forward_depth_alpha` + every frame's planar-depth maps [F,1,H,W] (see GaussianRasterizer.forward_planar);
        scales, rotations and cov3D_precomp may be [P,.] shared by the frames or [F,P,.] per frame.  Returns (color
        [F,3,H,W], radii [F,P], depth, alpha, planar_depth, planar_median_depth [F,1,H,W] each[, normal
        [F,3,H,W] of the plane normals with plane_normals])."""
        planes, normals = gaussian_planes(means3D, self.settings, scales, rotations, cov3D_precomp)
        m = self._maps(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp,
                       normals=normals if plane_normals else None, planes=planes)
        keys = ("color", "radii", "depth", "alpha", "planar_depth", "planar_median_depth") + \
            (("normal",) if plane_normals else ())
        return tuple(m[k] for k in keys)

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
        require them (stacked with autograd), and each frame's tanfovx / tanfovy when they are 0-dim tensors that
        require grad (see GaussianRasterizer.forward_with_camera_grad).  means2D_abs: see `forward`."""
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

    def forward_blend_stats(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None,
                            rotations=None, cov3D_precomp=None, pixel_weights=None, depth_alpha=False,
                            camera_grad=False, means2D_abs=None):
        """`forward` (depth_alpha: `forward_depth_alpha`; camera_grad: see `forward_with_camera_grad`; means2D_abs:
        see `forward`) + each frame's blend-weight statistics blend_weight_sum and blend_weight_max [F,P] (see
        GaussianRasterizer.forward_blend_stats).  pixel_weights: None, [H,W] or [1,H,W] shared by the frames, or
        [F,H,W] or [F,1,H,W] per frame.  Returns (color [F,3,H,W], radii [F,P][, depth, alpha [F,1,H,W]],
        blend_weight_sum [F,P], blend_weight_max [F,P])."""
        return tuple(self._maps(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp,
                                depth_alpha=depth_alpha, camera_grad=camera_grad, means2D_abs=means2D_abs,
                                blend_stats=True, pixel_weights=pixel_weights).values())


class GaussianRasterizationSettings(NamedTuple):
    """The reference's settings.  tanfovx / tanfovy may also be 0-dim float tensors, e.g. to learn the focal length:
    with camera_grad (forward_with_camera_grad and the camera_grad=True methods) one that requires grad receives its
    gradient.  The kernels take the values as launch parameters, so a CUDA tensor costs one device-to-host read per
    call; Python floats cost nothing."""
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
        raster_settings = _host_fovs(self.raster_settings)[0]
        sh, col, sc, rot, cov = _exclusive_inputs(shs, colors_precomp, scales, rotations, cov3D_precomp)
        return rasterize_gaussians(means3D, means2D, sh, col, opacities, sc, rot, cov, raster_settings)

    def _maps(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
              cov3D_precomp=None, depth_alpha=False, normals=None, surface=None, features=None, camera_grad=False,
              means2D_abs=None, blend_stats=False, pixel_weights=None, planes=None):
        """The outputs by name, in _MAPS order: "color" and "radii"; "depth" and "alpha" with depth_alpha or any
        other map; "median_depth" and "distortion" with surface = (near, far); "normal" with normals [P,3];
        "features" with features [P,C]; "blend_weight_sum" and "blend_weight_max" [P] with blend_stats, weighted by
        pixel_weights (see `forward_blend_stats`).  camera_grad: see `forward_with_camera_grad`.  means2D_abs: see
        `forward_abs_grad` (not with features)."""
        rs = self.raster_settings
        cams = (rs.viewmatrix, rs.projmatrix, rs.campos) if camera_grad else (None, None, None)
        return _request_maps(_RasterizeGaussians, _RasterizeGaussiansMaps, rs, cams, means3D, means2D, opacities, shs,
                             colors_precomp, scales, rotations, cov3D_precomp, depth_alpha, normals, surface,
                             features, means2D_abs, blend_stats, pixel_weights, planes)

    def forward_planar(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                       cov3D_precomp=None, plane_normals=False):
        """`forward_depth_alpha` + two planar-depth maps (RaDe-GS / PGSR), over the same blend.  Each Gaussian paints
        the depth of its own plane (`gaussian_planes`) across its footprint instead of its centre's depth:
          planar_depth         sum_i d_i(p) alpha_i T_i (no background term, not normalised: planar_depth / alpha
                               is the expected depth)
          planar_median_depth  d_i(p) of the median record (the record `forward_surface`'s median uses; 0 where
                               nothing is blended)
        plane_normals=True: also the normal map sum_i n_i alpha_i T_i [3,H,W] of the plane normals (camera space,
        facing the camera).  Every map is differentiable in the Gaussian inputs; the camera is not (a camera tensor
        that requires grad raises ValueError).  Returns (color [3,H,W], radii [P], depth, alpha, planar_depth,
        planar_median_depth [1,H,W] each[, normal [3,H,W]])."""
        planes, normals = gaussian_planes(means3D, self.raster_settings, scales, rotations, cov3D_precomp)
        m = self._maps(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp,
                       normals=normals if plane_normals else None, planes=planes)
        keys = ("color", "radii", "depth", "alpha", "planar_depth", "planar_median_depth") + \
            (("normal",) if plane_normals else ())
        return tuple(m[k] for k in keys)

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
        them, e.g. for a learnable pose correction (gaussian_renderer.posed_camera).  raster_settings.tanfovx /
        .tanfovy given as 0-dim tensors that require grad receive dL/dtan(fov/2) through the EWA covariance: the
        focal length of its Jacobian and its 1.3 tan(fov/2) clamp.  The projection matrix, which places the 2D
        means, is a tensor of its own with its own gradient; a camera whose projmatrix and tan(fov/2) both follow a
        focal length (gaussian_renderer.posed_camera with log_focal) gets the total focal gradient as the sum of the
        two.  Returns what `forward` / `forward_depth_alpha` return."""
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

    def forward_blend_stats(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None,
                            rotations=None, cov3D_precomp=None, pixel_weights=None, depth_alpha=False,
                            camera_grad=False, means2D_abs=None):
        """`forward` (depth_alpha: `forward_depth_alpha`; camera_grad: see `forward_with_camera_grad`; means2D_abs:
        see `forward_abs_grad`) + two per-Gaussian blend-weight statistics over the same blend, w_ip = alpha_ip T_ip
        the weight Gaussian i gets at pixel p (0 where it is not blended) and e_p = pixel_weights (1 when None):
          blend_weight_sum [P]  sum_p e_p w_ip            (Mini-Splatting's / LightGaussian's importance)
          blend_weight_max [P]  max(0, max_p e_p w_ip)    (RadSplat's / Taming-3DGS's pruning criterion)
        Both are exactly 0 for a Gaussian that no pixel blends: one inside the object, one behind an opaque surface,
        or one off screen, which radii > 0 and the opacity cannot tell apart.  Weighted by 1 - mask they score how
        much background a Gaussian paints.  pixel_weights is a float32 CUDA tensor [H,W] or [1,H,W]; its values are
        not checked: a negative weight enters the sum as given and contributes 0 to the max.  The statistics are not
        differentiable and change neither the image nor any gradient; combine frames or iterations with torch
        (torch.maximum, +).  Returns (color [3,H,W], radii [P][, depth, alpha [1,H,W]], blend_weight_sum [P],
        blend_weight_max [P])."""
        return tuple(self._maps(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp,
                                depth_alpha=depth_alpha, camera_grad=camera_grad, means2D_abs=means2D_abs,
                                blend_stats=True, pixel_weights=pixel_weights).values())

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
        rs = GaussianRasterizationSettings(image_height, image_width, tan_fovx, tan_fovy, bg, scale_modifier,
                                           viewmatrix, projmatrix, degree, campos, prefiltered, debug)
        color, radii, ws, R, _ = _forward(False, rs, means3D, sh, colors, opacity, scales, rotations, cov3D_precomp)
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
