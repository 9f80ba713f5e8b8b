"""Drop-in `nvdiffrast_utils.dpsr.DPSR` backed by libdgmesh_b200.so (sm_90a kernels + cuFFT).

Mirrors dgmesh/nvdiffrast_utils/dpsr.py:10-70:
    DPSR(res, sig=10, scale=True, shift=True);  forward(V[b,nv,3], N[b,nv,3]) -> phi[b,*res]
Only the configuration DG-Mesh uses is implemented natively: 3-D cubic grids, batch 1,
scale=True, shift=True (gaussian_model_dpsr_dynamic_anchor.py:79).  Anything else raises.

`DPSR.forward_signed(V, N, thres)` additionally fuses what `mesh_renderer` does right after the
solve (utils/renderer.py:163-168: sign fix from psr[0,0,0,0], subtract the density threshold) and
thereby removes the reference's host synchronisation.
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

_plans = {}  # (device index, G) -> (plan handle, workspace bytes): cuFFT plans belong to a device


def _plan(G):
    key = (torch.cuda.current_device(), G)
    if key not in _plans:
        h, nbytes = ctypes.c_void_p(), _dgm_lib.c_size_t()
        _dgm_lib.check(_dgm_lib.lib().dgp_plan_create(G, ctypes.byref(h), ctypes.byref(nbytes)), "dgp_plan_create")
        _plans[key] = (h, nbytes.value)
    return _plans[key]


class _DPSRFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, V, N, thres, G, sig, mode):
        if V.dim() != 2 or V.shape[1] != 3 or V.shape != N.shape:
            raise ValueError("DPSR: V and N must both be [nv, 3]")
        if not V.is_cuda:
            raise ValueError("DPSR: CUDA tensors required (no CPU fallback)")
        Vc, Nc = V.contiguous().float(), N.contiguous().float()
        plan, nbytes = _plan(G)
        ws = torch.empty((nbytes,), dtype=torch.uint8, device=V.device)
        out = torch.empty((G, G, G), dtype=torch.float32, device=V.device)
        th = thres.reshape(1).contiguous().float() if mode else None
        rc = _dgm_lib.lib().dgp_forward(plan, Vc.shape[0], float(sig), Vc.data_ptr(), Nc.data_ptr(), mode,
                                        th.data_ptr() if mode else None, out.data_ptr(), ws.data_ptr(), nbytes,
                                        _dgm_lib.stream_ptr())
        _dgm_lib.check(rc, "dgp_forward")
        ctx.save_for_backward(Vc, Nc, ws)
        ctx.G, ctx.mode, ctx.th_shape = G, mode, (thres.shape if mode else None)
        return out

    @staticmethod
    def backward(ctx, g):
        Vc, Nc, ws = ctx.saved_tensors
        plan, nbytes = _plan(ctx.G)
        dV, dN = torch.empty_like(Vc), torch.empty_like(Nc)
        dth = torch.empty((1,), dtype=torch.float32, device=Vc.device) if ctx.mode else None
        rc = _dgm_lib.lib().dgp_backward(plan, Vc.shape[0], Vc.data_ptr(), Nc.data_ptr(), ctx.mode,
                                         g.contiguous().float().data_ptr(), dV.data_ptr(), dN.data_ptr(),
                                         dth.data_ptr() if ctx.mode else None, ws.data_ptr(), nbytes,
                                         _dgm_lib.stream_ptr())
        _dgm_lib.check(rc, "dgp_backward")
        return dV, dN, (dth.reshape(ctx.th_shape) if ctx.mode else None), None, None, None


class DPSR(nn.Module):
    def __init__(self, res, sig=10, scale=True, shift=True):
        super().__init__()
        if len(res) != 3 or not (res[0] == res[1] == res[2]) or res[0] % 2:
            raise NotImplementedError("DPSR : cubic 3-D grids with an even resolution only")
        if not (scale and shift):
            raise NotImplementedError("DPSR : scale=True, shift=True only (DG-Mesh's configuration)")
        self.res, self.sig, self.dim = tuple(res), sig, 3
        self.scale, self.shift = scale, shift

    def _check(self, V, N):
        assert V.shape == N.shape  # dpsr.py:34
        if V.dim() != 3 or V.shape[0] != 1:
            raise NotImplementedError("DPSR : batch size 1 only")

    def forward(self, V, N):
        """phi [1, G, G, G] exactly as the reference returns it."""
        self._check(V, N)
        return _DPSRFunction.apply(V[0], N[0], None, self.res[0], self.sig, 0).unsqueeze(0)

    def forward_signed(self, V, N, thres):
        """(psr * sign - thres) [G, G, G] of mesh_renderer (utils/renderer.py:163-169), no host sync."""
        self._check(V, N)
        return _DPSRFunction.apply(V[0], N[0], thres, self.res[0], self.sig, 1)
