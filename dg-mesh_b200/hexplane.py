"""HexPlane / K-Planes space-time feature field (4D-GS's deformation encoding) and a DeformNetwork-shaped module on
top of it (csrc/hexplane.cu behind the C-ABI dghp_forward / dghp_backward / dghp_reg_forward / dghp_reg_backward).

    net = HexPlaneDeformNetwork(box).cuda()
    d_xyz, d_rotation, d_scaling = net(gaussians.get_xyz.detach(), t)          # t [N,1], or [F,N,1] for a batch
    tv, time_smooth, l1_time = net.field.regularisers()

A new field does not depend on time (its time planes are all ones), and nothing here changes a default of the
training script: the field is an opt-in replacement for utils.time_utils.DeformNetwork."""
import ctypes
import os
import sys

import torch
from torch import nn

_root = os.path.dirname(os.path.abspath(__file__))
if _root not in sys.path:
    sys.path.insert(0, _root)
import _dgm_lib  # noqa: E402

# plane p of a scale is the coordinate pair PAIRS[p] of (x, y, z, t); spatial planes 0, 1, 3, time planes 2, 4, 5
PAIRS = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))
SPATIAL, TIME = (0, 1, 3), (2, 4, 5)


def _int(fn, name, v, lo, hi=None):
    if isinstance(v, bool) or not isinstance(v, int) or v < lo or (hi is not None and v > hi):
        raise ValueError(f"{fn}: {name} must be an int >= {lo}" + (f" and <= {hi}" if hi is not None else "")
                         + f", not {v!r}")
    return v


def _ptrs(ts, kind=ctypes.c_void_p):
    return (kind * len(ts))(*ts)


class _Shape:
    """The plane shapes as the C-ABI takes them: (S, C, res_host, R_t)."""

    def __init__(self, field):
        self.S, self.C, self.Rt = field.S, field.channels, field.time_resolution
        self.res = _ptrs(field.resolutions, ctypes.c_int32)

    def head(self):
        return self.S, self.C, ctypes.addressof(self.res), self.Rt


class _FieldFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, shape, box, x, t, *planes):
        F, N = t.shape[0], t.shape[1]
        out = torch.empty(F, N, shape.S * shape.C, dtype=torch.float32, device=x.device)
        pp = _ptrs([p.data_ptr() for p in planes])
        _dgm_lib.check(_dgm_lib.lib().dghp_forward(F, N, *shape.head(), box.data_ptr(), x.data_ptr(), t.data_ptr(),
                                                   ctypes.addressof(pp), out.data_ptr(), _dgm_lib.stream_ptr()),
                       "dghp_forward")
        ctx.shape = shape
        ctx.save_for_backward(box, x, t, *planes)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        shape = ctx.shape
        box, x, t, *planes = ctx.saved_tensors
        F, N = t.shape[0], t.shape[1]
        lib = _dgm_lib.lib()
        grad_out = grad_out.contiguous()
        gx = torch.empty_like(x) if ctx.needs_input_grad[2] else None
        gp = [torch.empty_like(p) for p in planes]
        n = ctypes.c_size_t()
        _dgm_lib.check(lib.dghp_backward_workspace(F, N, *shape.head(), ctypes.byref(n)), "dghp_backward_workspace")
        ws = torch.empty(n.value, dtype=torch.uint8, device=x.device)
        pp, gpp = _ptrs([p.data_ptr() for p in planes]), _ptrs([g.data_ptr() for g in gp])
        _dgm_lib.check(lib.dghp_backward(F, N, *shape.head(), box.data_ptr(), x.data_ptr(), t.data_ptr(),
                                         ctypes.addressof(pp), grad_out.data_ptr(),
                                         gx.data_ptr() if gx is not None else None, ctypes.addressof(gpp),
                                         ws.data_ptr(), ws.numel(), _dgm_lib.stream_ptr()), "dghp_backward")
        return (None, None, gx, None) + tuple(gp)


class _RegFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, shape, *planes):
        lib = _dgm_lib.lib()
        dev = planes[0].device
        n = ctypes.c_size_t()
        _dgm_lib.check(lib.dghp_reg_workspace(*shape.head(), ctypes.byref(n)), "dghp_reg_workspace")
        ws = torch.empty(n.value, dtype=torch.uint8, device=dev)
        losses = torch.empty(3, dtype=torch.float32, device=dev)
        pp = _ptrs([p.data_ptr() for p in planes])
        _dgm_lib.check(lib.dghp_reg_forward(*shape.head(), ctypes.addressof(pp), losses.data_ptr(), ws.data_ptr(),
                                            ws.numel(), _dgm_lib.stream_ptr()), "dghp_reg_forward")
        ctx.shape = shape
        ctx.save_for_backward(*planes)
        return losses[0].clone(), losses[1].clone(), losses[2].clone()

    @staticmethod
    def backward(ctx, g_tv, g_ts, g_l1):
        planes = ctx.saved_tensors
        dev = planes[0].device
        g = torch.stack([t.float() if t is not None else torch.zeros((), device=dev)
                         for t in (g_tv, g_ts, g_l1)]).contiguous()
        gp = [torch.empty_like(p) for p in planes]
        pp, gpp = _ptrs([p.data_ptr() for p in planes]), _ptrs([q.data_ptr() for q in gp])
        _dgm_lib.check(_dgm_lib.lib().dghp_reg_backward(*ctx.shape.head(), ctypes.addressof(pp), g.data_ptr(),
                                                        ctypes.addressof(gpp), _dgm_lib.stream_ptr()),
                       "dghp_reg_backward")
        return (None,) + tuple(gp)


class HexPlaneField(nn.Module):
    """4D-GS's HexPlane field (the K-Planes factorisation of (x, y, z, t)): x [N,3], t [N,1] -> features [N, S C],
    or t [F,N,1] (a frame batch over the same canonical x) -> [F, N, S C].

    u = 2 (x - box_min) / (box_max - box_min) - 1 per axis and tau = 2 t - 1.  Scale s has spatial resolution
    R_s = base_resolution * multires[s] on x, y and z and time_resolution R_t (time is not scaled).  Its six planes,
    one per coordinate pair (a, b) in the order (x,y) (x,z) (x,t) (y,z) (y,t) (z,t), are parameters stored
    channels-last as [R_b, R_a, C] (`planes[6 s + p]`).  Each is sampled bilinearly as
    F.grid_sample(align_corners=True, padding_mode='border') with a on the width axis and b on the height axis, and
    f_s = prod_p sample(plane_{s,p}, u_a, u_b), channel by channel; the output is concat_s f_s.

    Initialisation (K-Planes): spatial planes uniform in [0.1, 0.5], time planes all ones (a new field does not
    depend on time).  Gradients reach every plane and x, with torch's convention of a zero coordinate gradient
    outside the box and on its faces; t takes none (a t that requires grad is refused).  The plane gradients are
    bit-identical from run to run, and each frame of a batch gives the features of that frame alone, to the bit.

    Supported: channels 16 or 32, 1 <= S <= 4, resolutions >= 2, float32 CUDA tensors; anything else raises
    ValueError.  `box` [2,3] (min row, max row) is fixed at construction and kept as a buffer (in the state_dict)."""

    def __init__(self, box, channels=32, base_resolution=64, multires=(1, 2), time_resolution=25):
        super().__init__()
        fn = "HexPlaneField"
        if isinstance(channels, bool) or not isinstance(channels, int) or channels not in (16, 32):
            raise ValueError(f"{fn}: channels must be 16 or 32, not {channels!r}")
        _int(fn, "base_resolution", base_resolution, 1)
        _int(fn, "time_resolution", time_resolution, 2)
        multires = tuple(multires)
        if not 1 <= len(multires) <= 4:
            raise ValueError(f"{fn}: multires must have 1 to 4 scales, not {len(multires)}")
        res = [_int(fn, "multires[]", m, 1) * base_resolution for m in multires]
        if min(res) < 2:
            raise ValueError(f"{fn}: every spatial resolution must be >= 2, not {res}")
        for R in res:
            if max(R, time_resolution) * R * channels >= 2 ** 31:
                raise ValueError(f"{fn}: a plane of R = {R} is too large (R max(R, R_t) C < 2^31)")
        box = torch.as_tensor(box, dtype=torch.float32).detach().clone()
        if tuple(box.shape) != (2, 3) or not bool(torch.isfinite(box).all()) or not bool((box[1] > box[0]).all()):
            raise ValueError(f"{fn}: box must be finite [2,3] (min row, max row) with max > min")
        self.channels, self.time_resolution, self.resolutions = channels, time_resolution, tuple(res)
        self.S = len(res)
        self.register_buffer("box", box)
        planes = []
        for R in res:
            for p, (a, b) in enumerate(PAIRS):
                rows = time_resolution if b == 3 else R
                if p in TIME:
                    planes.append(nn.Parameter(torch.ones(rows, R, channels)))
                else:
                    planes.append(nn.Parameter(torch.empty(rows, R, channels).uniform_(0.1, 0.5)))
        self.planes = nn.ParameterList(planes)
        self._shape = _Shape(self)

    @property
    def out_dim(self):
        return self.S * self.channels

    def _check_planes(self, fn):
        for i, p in enumerate(self.planes):
            if p.dtype != torch.float32 or not p.is_cuda:
                raise ValueError(f"{fn}: plane {i} must be a float32 CUDA tensor (there is no CPU path)")
            if not p.is_contiguous() or p.device != self.planes[0].device:
                raise ValueError(f"{fn}: planes must be contiguous and on one device")
        if self.box.device != self.planes[0].device:
            raise ValueError(f"{fn}: box is on {self.box.device}, the planes on {self.planes[0].device}")

    def forward(self, x, t):
        fn = "HexPlaneField"
        if not torch.is_tensor(x) or x.dim() != 2 or x.shape[1] != 3:
            raise ValueError(f"{fn}: x must be a tensor [N,3]")
        N = x.shape[0]
        if not torch.is_tensor(t) or t.dim() not in (2, 3) or tuple(t.shape[-2:]) != (N, 1):
            raise ValueError(f"{fn}: t must be [N,1] or [F,N,1] with N = {N}")
        if t.requires_grad:
            raise ValueError(f"{fn}: t must not require grad (the field has no gradient in t)")
        for name, v in (("x", x), ("t", t)):
            if v.dtype != torch.float32:
                raise ValueError(f"{fn}: {name} must be float32, not {v.dtype}")
            if not v.is_cuda:
                raise ValueError(f"{fn}: {name} must be a CUDA tensor (there is no CPU path)")
        self._check_planes(fn)
        if x.device != self.box.device or t.device != self.box.device:
            raise ValueError(f"{fn}: x and t must be on the field's device {self.box.device}")
        batched = t.dim() == 3
        F = t.shape[0] if batched else 1
        if 3 * self.S * N * (1 + F) >= 2 ** 31 or F * N * self.out_dim >= 2 ** 31:
            raise ValueError(f"{fn}: 3 S N (1 + F) and F N S C must be below 2^31")
        tt = t.detach().reshape(F, N).contiguous()
        out = _FieldFn.apply(self._shape, self.box, x.contiguous(), tt, *self.planes)
        return out if batched else out[0]

    def regularisers(self):
        """(tv, time_smooth, l1_time), differentiable in every plane.  For a plane G [R_b, R_a, C], each term summed
        over its planes and the scales:

            tv          (spatial planes) = mean_{i<R_b-1,j,c} (G[i+1,j,c] - G[i,j,c])^2
                                         + mean_{i,j<R_a-1,c} (G[i,j+1,c] - G[i,j,c])^2
            time_smooth (time planes, rows are time) = mean_{i<R_t-2,j,c} (G[i+2,j,c] - 2 G[i+1,j,c] + G[i,j,c])^2
            l1_time     (time planes) = mean |1 - G|    (gradient 0 at G = 1, as in torch)

        time_smooth is 0 when R_t = 2.  Every term is a mean over its differences, summed over planes and scales.
        A codebase that normalises a term differently needs its weight rescaled by the ratio: K-Planes' and 4D-GS's
        plane TV is 2 (mean over rows + mean over columns), twice tv here, while their time smoothness and L1 terms
        are the same means.  The result is bit-identical from run to run."""
        self._check_planes("HexPlaneField.regularisers")
        return _RegFn.apply(self._shape, *self.planes)


class DeformHeads(nn.Module):
    """4D-GS's deformation heads over a feature field (`field(x, t)` -> [..., field.out_dim]), shaped like
    utils.time_utils.DeformNetwork: forward(x, t) -> (d_xyz, d_rotation, d_scaling), or with normal=True
    (d_xyz, d_rotation, d_scaling, d_normal) as DeformNetworkNormal returns.  The field is followed by
    Linear(out_dim, W) and one head per output: ReLU -> Linear(W, W) -> ReLU -> Linear(W, rows).  The field is
    registered first, so parameter order and state_dict keys are field.*, feature_out.*, then the heads."""
    HEADS = (("gaussian_warp", 3), ("gaussian_rotation", 4), ("gaussian_scaling", 3))

    def __init__(self, field, normal, W):
        super().__init__()
        self.field = field
        self.feature_out = nn.Linear(field.out_dim, W)
        self.heads = self.HEADS + ((("gaussian_normal", 3),) if normal else ())
        for name, rows in self.heads:
            setattr(self, name, nn.Sequential(nn.ReLU(), nn.Linear(W, W), nn.ReLU(), nn.Linear(W, rows)))

    def forward(self, x, t):
        h = self.feature_out(self.field(x, t))
        return tuple(getattr(self, name)(h) for name, _ in self.heads)


class HexPlaneDeformNetwork(DeformHeads):
    """4D-GS's deformation network over a HexPlaneField (the DeformHeads on it), shaped like
    utils.time_utils.DeformNetwork: forward(x, t) -> (d_xyz, d_rotation, d_scaling), or with normal=True
    (d_xyz, d_rotation, d_scaling, d_normal) as DeformNetworkNormal returns.  With t [F,N,1] every output is
    [F,N,rows] (the per-frame deltas render_batch takes), the spatial planes sampled once per point for the whole
    batch.

    field_kw goes to HexPlaneField (channels, base_resolution, multires, time_resolution).  The heads are plain
    nn.Linear; every parameter is an ordinary nn.Parameter (optim.FusedAdam and state_dict work unchanged)."""

    def __init__(self, box, normal=False, W=64, **field_kw):
        _int("HexPlaneDeformNetwork", "W", W, 1)
        super().__init__(HexPlaneField(box, **field_kw), normal, W)
