"""Drop-in `utils.time_utils` (reference: dgmesh/utils/time_utils.py): DeformNetwork,
DeformNetworkNormal, DeformNetworkNormalSep, AppearanceNetwork with the SAME constructor
signatures, parameter names / shapes (state_dicts are interchangeable) and return values, but the
forward + backward run as bf16 wgmma GEMM chains inside libdgmesh_b200.so.

`utils` is a namespace package in the reference (no __init__.py) and here: with this directory
ahead of the reference's on sys.path only `utils.time_utils` is replaced.

Numerics (the reference is fp32 cuBLAS).  Default `DGMESH_B200_MLP_PRECISION=bf16x3`: the forward
runs every layer as three bf16 wgmma passes over split operands (hi + lo, fp32 accumulation), so
outputs agree with the fp32 reference to ~1e-5 and the ReLU decisions are the reference's; the
backward is single-pass bf16 and the parameter / input gradients agree to <= 2 % relative L2
(measured 0.3-1 %).  `bf16`: single-pass forward, 3x fewer MMAs; outputs ~2e-3, but ~1 % of the
ReLU signs flip and gradients differ by ~7 % (tests/test_mlp.py, DESIGN.md).  is_6dof (off in every
reference config): branch_w / branch_v run as one 6-row head of the same kernel chain, the SE(3) exponential
(utils/rigid_utils.py) is elementwise torch on the [N,6] result.

The packed bf16 operands are cached per module and rebuilt only when a parameter changed (tensor
version counters), i.e. once per optimiser step, not once per forward.  Optimiser steps, in-place edits under
torch.no_grad(), load_state_dict and assigning a new Parameter are all seen (tests/test_mlp_tiles.py).  A write
through `.data` (`p.data.mul_(2)`) is NOT: it leaves the version counter unchanged, and a module that has run a
forward keeps using the weights it packed before the write.  Update weights in place under torch.no_grad()
instead.  (The `.data` writes in DeformNetworkNormalSep's constructor run before any forward.)
"""
import ctypes
import os
import sys

import torch
import torch.nn as nn

_root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _root not in sys.path:
    sys.path.insert(0, _root)
import _dgm_lib  # noqa: E402

_sizes = None
_PRECISE = os.environ.get("DGMESH_B200_MLP_PRECISION", "bf16x3").lower() != "bf16"


def set_precision(mode):
    """'bf16x3' (default: split-precision forward) or 'bf16' (single pass)."""
    global _PRECISE
    if mode not in ("bf16x3", "bf16"):
        raise ValueError("precision must be 'bf16x3' or 'bf16'")
    _PRECISE = mode == "bf16x3"


def _pack_sizes():
    global _sizes
    if _sizes is None:
        w, b, g = _dgm_lib.c_size_t(), _dgm_lib.c_size_t(), _dgm_lib.c_size_t()
        _dgm_lib.check(_dgm_lib.lib().dgl_mlp_pack_sizes(ctypes.byref(w), ctypes.byref(b), ctypes.byref(g)),
                       "dgl_mlp_pack_sizes")
        _sizes = (w.value, b.value, g.value)
    return _sizes


def _raw_struct(cls, spec, tensors):
    """Fill a DglRaw / DglRawGrads pointer table from tensors ordered as `_TimeNet._param_list`."""
    r = cls()
    it = iter(tensors)
    if cls is _dgm_lib.DglRaw:
        r.has_timenet, r.in_t, r.sigmoid_out, r.n_heads = spec["blender"], spec["in_t"], spec["sigmoid"], len(spec["heads"])
        for i, rows in enumerate(spec["heads"]):
            r.head_rows[i] = rows
    if spec["blender"]:
        r.Wt0, r.bt0, r.Wt1, r.bt1 = (next(it).data_ptr() for _ in range(4))
    for l in range(8):
        r.W[l] = next(it).data_ptr()
        r.b[l] = next(it).data_ptr()
    for i in range(len(spec["heads"])):
        r.Wh[i] = next(it).data_ptr()
        r.bh[i] = next(it).data_ptr()
    return r


class _MLPFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, spec, train, x, t, *params):
        lib = _dgm_lib.lib()
        if not x.is_cuda:
            raise ValueError("time_utils : CUDA tensors required (no CPU fallback)")
        xc = x.detach().contiguous().float()
        tc = t.detach().contiguous().float().reshape(-1)
        P = xc.shape[0]
        if xc.dim() != 2 or xc.shape[1] != 3 or tc.shape[0] != P:
            raise ValueError("expected x [N,3] and t [N,1]")
        dev = xc.device
        st = _dgm_lib.stream_ptr()
        # packed operands: rebuilt only when some parameter was modified since they were packed
        sig = tuple((p.data_ptr(), p._version) for p in params) + (st,)
        cache = spec.get("_packed")
        if cache is not None and cache[0] == sig and not torch.cuda.is_current_stream_capturing():
            _, wbuf, bbuf, ps, raw, net = cache
        else:
            ps = [p.detach().contiguous().float() for p in params]
            wb, bb, _ = _pack_sizes()
            wbuf = torch.empty((wb,), dtype=torch.uint8, device=dev)
            bbuf = torch.empty((bb // 4,), dtype=torch.float32, device=dev)
            raw = _raw_struct(_dgm_lib.DglRaw, spec, ps)
            net = _dgm_lib.DglNet()
            _dgm_lib.check(lib.dgl_mlp_pack(ctypes.byref(raw), wbuf.data_ptr(), bbuf.data_ptr(), ctypes.byref(net),
                                            st), "dgl_mlp_pack")
            spec["_packed"] = (sig, wbuf, bbuf, ps, raw, net)
        net.precise = int(_PRECISE)
        train = int(train)   # decided by the caller: grad mode is always off inside Function.forward
        nbytes = _dgm_lib.c_size_t()
        _dgm_lib.check(lib.dgl_mlp_workspace(P, train, ctypes.byref(nbytes)), "dgl_mlp_workspace")
        ws = torch.empty((nbytes.value,), dtype=torch.uint8, device=dev)
        out = torch.empty((P, 16), dtype=torch.float32, device=dev)
        if P:
            _dgm_lib.check(lib.dgl_mlp_forward(ctypes.byref(net), P, xc.data_ptr(), tc.data_ptr(), out.data_ptr(),
                                               train, ws.data_ptr(), nbytes.value, st), "dgl_mlp_forward")
        ctx.spec, ctx.net, ctx.raw, ctx.keep = spec, net, raw, (wbuf, bbuf, ps)
        ctx.x_needs_grad = x.requires_grad
        ctx.save_for_backward(xc, out, ws)
        return out

    @staticmethod
    def backward(ctx, g_out):
        lib = _dgm_lib.lib()
        xc, out, ws = ctx.saved_tensors
        P, dev, spec = xc.shape[0], xc.device, ctx.spec
        _, _, gb = _pack_sizes()
        gbuf = torch.empty((gb // 4,), dtype=torch.float32, device=dev)
        grads = _dgm_lib.DglGrads()
        _dgm_lib.check(lib.dgl_mlp_grad_pointers(gbuf.data_ptr(), ctypes.byref(grads)), "dgl_mlp_grad_pointers")
        ps = ctx.keep[2]
        outs = [torch.empty_like(p) for p in ps]
        dx = torch.empty_like(xc) if ctx.x_needs_grad else None
        st = _dgm_lib.stream_ptr()
        if P:
            g = g_out.contiguous().float()
            _dgm_lib.check(lib.dgl_mlp_backward(ctypes.byref(ctx.net), P, xc.data_ptr(), out.data_ptr(), g.data_ptr(),
                                                ws.data_ptr(), ws.numel(), ctypes.byref(grads),
                                                dx.data_ptr() if dx is not None else None, st), "dgl_mlp_backward")
        else:
            gbuf.zero_()
        rg = _raw_struct(_dgm_lib.DglRawGrads, spec, outs)
        _dgm_lib.check(lib.dgl_mlp_unpack_grads(ctypes.byref(ctx.raw), gbuf.data_ptr(), ctypes.byref(rg), st),
                       "dgl_mlp_unpack_grads")
        return (None, None, dx, None) + tuple(outs)


class _TimeNet(nn.Module):
    """Shared trunk; subclasses declare their heads (name, rows) in output order."""
    HEADS = ()
    SIGMOID = False

    def __init__(self, D=8, W=256, input_ch=3, output_ch=59, multires=10, is_blender=False, is_6dof=False):
        super().__init__()
        if D != 8 or W != 256 or multires != 10:
            raise NotImplementedError("time_utils : D=8, W=256, multires=10 (the reference defaults) only")
        self.D, self.W, self.input_ch, self.output_ch = D, W, input_ch, output_ch
        self.t_multires = 6 if is_blender else 10
        self.skips = [D // 2]
        xyz_input_ch, time_input_ch = 63, 2 * self.t_multires + 1
        self.input_ch = xyz_input_ch + time_input_ch
        # same construction order as the reference -> identical default initialisation under a seed
        if is_blender:
            self.time_out = 30
            self.timenet = nn.Sequential(nn.Linear(time_input_ch, 256), nn.ReLU(inplace=True),
                                         nn.Linear(256, self.time_out))
            in0 = xyz_input_ch + self.time_out
        else:
            in0 = self.input_ch
        self.linear = nn.ModuleList([nn.Linear(in0, W)] + [
            nn.Linear(W, W) if i not in self.skips else nn.Linear(W + in0, W) for i in range(D - 1)])
        self.is_blender, self.is_6dof = is_blender, is_6dof
        # is_6dof (time_utils.py:96-98,169-171): the translation head is replaced by a screw axis (branch_w,
        # branch_v); the kernel sees ONE 6-row head whose weights are the two branches stacked
        self._screw = bool(is_6dof) and self.HEADS[0][0] == "gaussian_warp"
        self._make_heads(W)
        rows = [r for _, r in self.HEADS]
        if self._screw:
            rows[0] = 6
        self._spec = dict(blender=int(is_blender), in_t=in0 - xyz_input_ch, sigmoid=int(self.SIGMOID), heads=rows)

    def _make_heads(self, W):
        for name, rows in self.HEADS:
            if self._screw and name == "gaussian_warp":   # same construction order as the reference
                self.branch_w = nn.Linear(W, 3)
                self.branch_v = nn.Linear(W, 3)
            else:
                setattr(self, name, nn.Linear(W, rows))

    def _head_params(self):
        ps = []
        for name, _ in self.HEADS:
            if self._screw and name == "gaussian_warp":
                ps += [torch.cat([self.branch_w.weight, self.branch_v.weight], 0),
                       torch.cat([self.branch_w.bias, self.branch_v.bias], 0)]
            else:
                h = getattr(self, name)
                h = h[0] if isinstance(h, nn.Sequential) else h
                ps += [h.weight, h.bias]
        return ps

    def _param_list(self):
        ps = []
        if self.is_blender:
            ps += [self.timenet[0].weight, self.timenet[0].bias, self.timenet[2].weight, self.timenet[2].bias]
        for l in self.linear:
            ps += [l.weight, l.bias]
        return ps + self._head_params()

    def _warp(self, first):
        """d_xyz from the first head: a translation, or (is_6dof) the SE(3) transform of a screw motion."""
        if not self._screw:
            return first
        from utils.rigid_utils import exp_se3
        w, v = first[:, :3], first[:, 3:6]
        theta = torch.norm(w, dim=-1, keepdim=True)
        w = w / theta + 1e-5                     # as written in the reference (time_utils.py:119-123)
        v = v / theta + 1e-5
        return exp_se3(torch.cat([w, v], dim=-1), theta)

    def _run(self, x, t):
        params = self._param_list()
        train = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params))
        out = _MLPFunction.apply(self._spec, train, x, t, *params)
        cols, o = [], 0
        for r in self._spec["heads"]:
            cols.append(out[:, o:o + r])
            o += r
        return cols


class DeformNetwork(_TimeNet):
    HEADS = (("gaussian_warp", 3), ("gaussian_rotation", 4), ("gaussian_scaling", 3))

    def forward(self, x, t):
        d_xyz, rotation, scaling = self._run(x, t)
        return self._warp(d_xyz), rotation, scaling


class DeformNetworkNormal(_TimeNet):
    # construction order of the reference: warp, rotation, scaling, normal (time_utils.py:171-176)
    HEADS = (("gaussian_warp", 3), ("gaussian_rotation", 4), ("gaussian_scaling", 3), ("gaussian_normal", 3))

    def forward(self, x, t):
        d_xyz, rotation, scaling, normal = self._run(x, t)
        return self._warp(d_xyz), rotation, scaling, normal


class DeformNetworkNormalSep(_TimeNet):
    HEADS = (("gaussian_normal", 3),)

    def _make_heads(self, W):
        super()._make_heads(W)
        self.gaussian_normal.weight.data.zero_()   # time_utils.py:247-249
        self.gaussian_normal.bias.data.zero_()

    def forward(self, x, t):
        return self._run(x, t)[0]


class AppearanceNetwork(_TimeNet):
    HEADS = (("color_warp", 3),)
    SIGMOID = True

    def __init__(self, D=8, W=256, input_ch=3, output_ch=59, multires=10, is_blender=False):
        super().__init__(D, W, input_ch, output_ch, multires, is_blender, False)

    def _make_heads(self, W):
        self.color_warp = nn.Sequential(nn.Linear(W, 3), nn.Sigmoid())   # time_utils.py:306-309

    def forward(self, x, t):
        return self._run(x, t)[0]
