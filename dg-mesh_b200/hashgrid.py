"""Multiresolution hash-grid field of (x, y, z, t) (Instant-NGP's HashGrid, and Grid4D's space-time grids) and a
DeformNetwork-shaped module on top of it (csrc/hashgrid.cu behind the C-ABI dghg_forward / dghg_backward).

    net = HashGridDeformNetwork(box).cuda()
    d_xyz, d_rotation, d_scaling = net(gaussians.get_xyz.detach(), t)          # t [N,1], or [F,N,1] for a batch

Nothing here changes a default of the training script: the field is an opt-in replacement for
utils.time_utils.DeformNetwork, next to hexplane.HexPlaneDeformNetwork."""
import ctypes
import math
import os
import sys

import torch
from torch import nn

_root = os.path.dirname(os.path.abspath(__file__))
if _root not in sys.path:
    sys.path.insert(0, _root)
import _dgm_lib  # noqa: E402
from hexplane import DeformHeads, _int, _ptrs  # noqa: E402

# the grids in their fixed order; a grid's axes are the coordinates (0..3 = x, y, z, t) its name spells
GRIDS = ("xyz", "xyt", "yzt", "xzt")
AXES = {"xyz": (0, 1, 2), "xyt": (0, 1, 3), "yzt": (1, 2, 3), "xzt": (0, 2, 3)}


def level_resolutions(levels, base_resolution, finest_resolution):
    """Instant-NGP's spatial resolutions, in float64: R_l = floor(base b^l), b = exp((ln finest - ln base) / (L - 1))
    (R_0 = base when L = 1)."""
    if levels == 1:
        return (base_resolution,)
    b = math.exp((math.log(finest_resolution) - math.log(base_resolution)) / (levels - 1))
    return tuple(int(math.floor(base_resolution * b ** l)) for l in range(levels))


class _Shape:
    """The field's shape as the C-ABI takes it: (G, grids_host, L, Fe, log2_table, res_host, R_t)."""

    def __init__(self, field):
        self.G, self.L, self.Fe = len(field.grids), field.levels, field.features
        self.log2T, self.Rt = field.log2_table, field.time_resolution
        self.kinds = _ptrs([GRIDS.index(g) for g in field.grids], ctypes.c_int32)
        self.res = _ptrs(field.resolutions, ctypes.c_int32)

    def head(self):
        return (self.G, ctypes.addressof(self.kinds), self.L, self.Fe, self.log2T, ctypes.addressof(self.res),
                self.Rt)


class _FieldFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, shape, F, box, x, t, *tables):
        N = x.shape[0]
        out = torch.empty(F, N, shape.G * shape.L * shape.Fe, dtype=torch.float32, device=x.device)
        tp = _ptrs([p.data_ptr() for p in tables])
        _dgm_lib.check(_dgm_lib.lib().dghg_forward(F, N, *shape.head(), box.data_ptr(), x.data_ptr(),
                                                   t.data_ptr() if t is not None else None, ctypes.addressof(tp),
                                                   out.data_ptr(), _dgm_lib.stream_ptr()), "dghg_forward")
        ctx.shape, ctx.F = shape, F
        ctx.save_for_backward(box, x, t, *tables)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        shape, F = ctx.shape, ctx.F
        box, x, t, *tables = ctx.saved_tensors
        N = x.shape[0]
        lib = _dgm_lib.lib()
        grad_out = grad_out.contiguous()
        gx = torch.empty_like(x) if ctx.needs_input_grad[3] else None
        gt = [torch.empty_like(p) for p in tables]
        n = ctypes.c_size_t()
        _dgm_lib.check(lib.dghg_backward_workspace(F, N, *shape.head(), ctypes.byref(n)), "dghg_backward_workspace")
        ws = torch.empty(n.value, dtype=torch.uint8, device=x.device)
        tp, gtp = _ptrs([p.data_ptr() for p in tables]), _ptrs([g.data_ptr() for g in gt])
        _dgm_lib.check(lib.dghg_backward(F, N, *shape.head(), box.data_ptr(), x.data_ptr(),
                                         t.data_ptr() if t is not None else None, ctypes.addressof(tp),
                                         grad_out.data_ptr(), gx.data_ptr() if gx is not None else None,
                                         ctypes.addressof(gtp), ws.data_ptr(), ws.numel(), _dgm_lib.stream_ptr()),
                       "dghg_backward")
        return (None, None, None, gx, None) + tuple(gt)


class HashGridField(nn.Module):
    """Multiresolution hash encoding of (x, y, z, t): x [N,3], t [N,1] -> features [N, G L Fe], or t [F,N,1] (a frame
    batch over the same canonical x) -> [F, N, G L Fe], ordered grid, then level, then feature.  t may be None only
    when grids == ("xyz",) (the static Instant-NGP encoding; the output is then [N, L Fe]).

    grids is a non-empty subset of ("xyz", "xyt", "yzt", "xzt"), kept in that fixed order whatever order it is given
    in; a grid's three axes are the coordinates its name spells, in that order.  In float32, exactly as written:
    u = (x - lo) / (hi - lo) on a spatial axis and u = t on the time axis, clamped to [0, 1].  Level l has spatial
    resolution R_l = floor(base b^l), b = exp((ln finest - ln base) / (L - 1)) (float64 on the host; `resolutions`),
    and time resolution min(R_l, time_resolution).  Per axis p = u R (float32), c = min(floor(p), R - 1), w = p - c
    (1 on the top face); the feature is the trilinear blend of the rows of the 8 nodes c + {0,1}^3.  A level's table
    has T = 2^log2_table slots: a node's slot is row-major (first axis fastest) when (R_a+1)(R_b+1)(R_c+1) <= T
    (dense), else (i_a 1 ^ i_b 2654435761 ^ i_c 805459861) mod T in uint32 (Instant-NGP's primes).

    One parameter per grid, `tables[g]` [L, T, Fe] float32 channels-last, uniform in [-1e-4, 1e-4] (Instant-NGP);
    a dense level uses a prefix of its slots.  Gradients reach the tables and x; dL/dx is 0 where u was clamped
    from strictly outside [0, 1] (it passes at 0 and 1, as torch.clamp), and t takes none (a t that requires grad is
    refused).  The table gradients are sums in int64 fixed point, bit-identical from run to run; a non-finite
    grad_out makes the affected (grid, level)'s table gradient NaN.  Each frame of a batch gives the features of
    that frame alone, to the bit.

    Supported: features 2 or 4, 1 <= levels <= 24, 12 <= log2_table <= 24, float32 CUDA tensors; anything else,
    and any L T Fe, F N G L Fe or N F at or above 2^31, raises ValueError.  `box` [2,3] (min row, max row) is fixed
    at construction and kept as a buffer (in the state_dict)."""

    def __init__(self, box, grids=GRIDS, levels=16, features=2, log2_table=19, base_resolution=16,
                 finest_resolution=2048, time_resolution=32):
        super().__init__()
        fn = "HashGridField"
        if isinstance(grids, str):
            grids = (grids,)
        grids = tuple(grids)
        if not grids or len(set(grids)) != len(grids) or any(g not in GRIDS for g in grids):
            raise ValueError(f"{fn}: grids must be a non-empty subset of {GRIDS} without repeats, not {grids!r}")
        if isinstance(features, bool) or not isinstance(features, int) or features not in (2, 4):
            raise ValueError(f"{fn}: features must be 2 or 4, not {features!r}")
        _int(fn, "levels", levels, 1, 24)
        _int(fn, "log2_table", log2_table, 12, 24)
        _int(fn, "base_resolution", base_resolution, 1, 2 ** 24)
        _int(fn, "finest_resolution", finest_resolution, base_resolution, 2 ** 24)
        _int(fn, "time_resolution", time_resolution, 1)
        if levels * 2 ** log2_table * features >= 2 ** 31:
            raise ValueError(f"{fn}: L T Fe must be below 2^31")
        box = torch.as_tensor(box, dtype=torch.float32).detach().clone()
        if tuple(box.shape) != (2, 3) or not bool(torch.isfinite(box).all()) or not bool((box[1] > box[0]).all()):
            raise ValueError(f"{fn}: box must be finite [2,3] (min row, max row) with max > min")
        self.grids = tuple(g for g in GRIDS if g in grids)
        self.levels, self.features, self.log2_table = levels, features, log2_table
        self.time_resolution = time_resolution
        self.resolutions = level_resolutions(levels, base_resolution, finest_resolution)
        self.register_buffer("box", box)
        self.tables = nn.ParameterList([nn.Parameter(torch.empty(levels, 2 ** log2_table, features).uniform_(-1e-4, 1e-4))
                                        for _ in self.grids])
        self._shape = _Shape(self)

    @property
    def out_dim(self):
        return len(self.grids) * self.levels * self.features

    def forward(self, x, t=None):
        fn = "HashGridField"
        if not torch.is_tensor(x) or x.dim() != 2 or x.shape[1] != 3:
            raise ValueError(f"{fn}: x must be a tensor [N,3]")
        N = x.shape[0]
        if t is None:
            if self.grids != ("xyz",):
                raise ValueError(f"{fn}: t may be None only when grids == ('xyz',)")
        elif not torch.is_tensor(t) or t.dim() not in (2, 3) or tuple(t.shape[-2:]) != (N, 1):
            raise ValueError(f"{fn}: t must be [N,1] or [F,N,1] with N = {N}")
        elif t.requires_grad:
            raise ValueError(f"{fn}: t must not require grad (the field has no gradient in t)")
        for name, v in (("x", x), ("t", t)):
            if v is None:
                continue
            if v.dtype != torch.float32:
                raise ValueError(f"{fn}: {name} must be float32, not {v.dtype}")
            if not v.is_cuda:
                raise ValueError(f"{fn}: {name} must be a CUDA tensor (there is no CPU path)")
        for i, p in enumerate(self.tables):
            if p.dtype != torch.float32 or not p.is_cuda:
                raise ValueError(f"{fn}: table {i} must be a float32 CUDA tensor (there is no CPU path)")
            if not p.is_contiguous() or p.device != self.box.device:
                raise ValueError(f"{fn}: tables must be contiguous and on the box's device {self.box.device}")
        if x.device != self.box.device or (t is not None and t.device != self.box.device):
            raise ValueError(f"{fn}: x and t must be on the field's device {self.box.device}")
        batched = t is not None and t.dim() == 3
        F = t.shape[0] if batched else 1
        if F * N * self.out_dim >= 2 ** 31 or N * F >= 2 ** 31:
            raise ValueError(f"{fn}: F N G L Fe and N F must be below 2^31")
        tt = t.detach().reshape(F, N).contiguous() if t is not None else None
        out = _FieldFn.apply(self._shape, F, self.box, x.contiguous(), tt, *self.tables)
        return out if batched else out[0]


class HashGridDeformNetwork(DeformHeads):
    """The deformation heads of hexplane.DeformHeads over a HashGridField, shaped like utils.time_utils.DeformNetwork:
    forward(x, t) -> (d_xyz, d_rotation, d_scaling), or with normal=True (d_xyz, d_rotation, d_scaling, d_normal) as
    DeformNetworkNormal returns.  With t [F,N,1] every output is [F,N,rows] (the per-frame deltas render_batch
    takes), the spatial grid sampled once per point for the whole batch.

    field_kw goes to HashGridField (grids, levels, features, log2_table, base_resolution, finest_resolution,
    time_resolution).  The heads are plain nn.Linear; every parameter is an ordinary nn.Parameter (optim.FusedAdam
    and state_dict work unchanged)."""

    def __init__(self, box, normal=False, W=64, **field_kw):
        _int("HashGridDeformNetwork", "W", W, 1)
        super().__init__(HashGridField(box, **field_kw), normal, W)
