"""Drop-in `nvdiffrast_utils.dpsr.DPSR` backed by libdgmesh_b200.so (sm_90a kernels + cuFFT).

Mirrors dgmesh/nvdiffrast_utils/dpsr.py:10-70:
    DPSR(res, sig=10, scale=True, shift=True);  forward(V[b,nv,3], N[b,nv,3]) -> phi[b,*res]
Only the configuration DG-Mesh uses is implemented natively: 3-D cubic grids, scale=True, shift=True
(gaussian_model_dpsr_dynamic_anchor.py:79).  Anything else raises.  A batch (1 <= b <= 64) runs in one call:
every item is normalised on its own, as the reference does, and only each item's field outlives the forward.

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

MAX_BATCH = 64
_plans = {}  # (device index, G) -> (plan handle, workspace bytes): cuFFT plans belong to a device


def _plan(G):
    key = (torch.cuda.current_device(), G)
    if key not in _plans:
        h, nbytes = ctypes.c_void_p(), _dgm_lib.c_size_t()
        _dgm_lib.check(_dgm_lib.lib().dgp_plan_create(G, ctypes.byref(h), ctypes.byref(nbytes)), "dgp_plan_create")
        _plans[key] = (h, nbytes.value)
    return _plans[key]


def _workspace_bytes(plan, nbytes, B):
    if B == 1:
        return nbytes
    b = _dgm_lib.c_size_t()
    _dgm_lib.check(_dgm_lib.lib().dgp_batch_workspace_size(plan, B, ctypes.byref(b)), "dgp_batch_workspace_size")
    return b.value


class _DPSRFunction(torch.autograd.Function):
    """V, N [B, nv, 3] -> [B, G, G, G]; B = 1 runs the single-item entry points."""

    @staticmethod
    def forward(ctx, V, N, thres, G, sig, mode):
        if V.dim() != 3 or V.shape[2] != 3 or V.shape != N.shape:
            raise ValueError("DPSR: V and N must both be [b, nv, 3]")
        if not 1 <= V.shape[0] <= MAX_BATCH:
            raise ValueError(f"DPSR: batch size must be in [1, {MAX_BATCH}], got {V.shape[0]}")
        if not V.is_cuda:
            raise ValueError("DPSR: CUDA tensors required (no CPU fallback)")
        Vc, Nc = V.contiguous().float(), N.contiguous().float()
        B, nv = Vc.shape[0], Vc.shape[1]
        plan, nbytes = _plan(G)
        nbytes = _workspace_bytes(plan, nbytes, B)
        ws = torch.empty((nbytes,), dtype=torch.uint8, device=V.device)
        out = torch.empty((B, G, G, G), dtype=torch.float32, device=V.device)
        th = thres.reshape(1).contiguous().float() if mode else None
        lib = _dgm_lib.lib()
        args = (nv, float(sig), Vc.data_ptr(), Nc.data_ptr(), mode, th.data_ptr() if mode else None, out.data_ptr(),
                ws.data_ptr(), nbytes, _dgm_lib.stream_ptr())
        if B == 1:
            _dgm_lib.check(lib.dgp_forward(plan, *args), "dgp_forward")
        else:
            _dgm_lib.check(lib.dgp_forward_batch(plan, B, *args), "dgp_forward_batch")
        ctx.save_for_backward(Vc, Nc, ws)
        ctx.G, ctx.mode, ctx.th_shape = G, mode, (thres.shape if mode else None)
        return out

    @staticmethod
    def backward(ctx, g):
        Vc, Nc, ws = ctx.saved_tensors
        B, nv = Vc.shape[0], Vc.shape[1]
        plan, _ = _plan(ctx.G)
        dV, dN = torch.empty_like(Vc), torch.empty_like(Nc)
        dth = torch.empty((B,), dtype=torch.float32, device=Vc.device) if ctx.mode else None
        lib = _dgm_lib.lib()
        args = (nv, Vc.data_ptr(), Nc.data_ptr(), ctx.mode, g.contiguous().float().data_ptr(), dV.data_ptr(),
                dN.data_ptr(), dth.data_ptr() if ctx.mode else None, ws.data_ptr(), ws.numel(), _dgm_lib.stream_ptr())
        if B == 1:
            _dgm_lib.check(lib.dgp_backward(plan, *args), "dgp_backward")
        else:
            _dgm_lib.check(lib.dgp_backward_batch(plan, B, *args), "dgp_backward_batch")
        # every item has its own sign and offset but all share the threshold: its gradient is the items' sum
        dthres = (dth.sum() if B > 1 else dth).reshape(ctx.th_shape) if ctx.mode else None
        return dV, dN, dthres, None, None, None


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
        if V.dim() != 3:
            raise NotImplementedError("DPSR : V and N must be [b, nv, 3]")

    def forward(self, V, N):
        """phi [b, G, G, G] exactly as the reference returns it: each item shifted and scaled by its own mean and
        phi[k,0,0,0]."""
        self._check(V, N)
        return _DPSRFunction.apply(V, N, None, self.res[0], self.sig, 0)

    def forward_signed(self, V, N, thres):
        """(psr * sign - thres) of mesh_renderer (utils/renderer.py:163-169), no host sync: [G, G, G] for b = 1,
        [b, G, G, G] for b > 1.  Every item takes its sign from its own psr[k,0,0,0] (the reference reads item 0's
        only), so item k equals the b = 1 call on item k; all items share `thres`."""
        self._check(V, N)
        out = _DPSRFunction.apply(V, N, thres, self.res[0], self.sig, 1)
        return out[0] if V.shape[0] == 1 else out
