"""Stand-in for the third-party `diso` package as DG-Mesh uses it
(`from diso import DiffDMC, DiffMC`, dgmesh/scene/gaussian_model_dpsr_dynamic_anchor.py:40,84;
`gaussians.diffmc(psr, deform=None, isovalue=0.0)`, dgmesh/utils/renderer.py:171).

`diso` is not vendored with the reference and cannot be installed offline, so this follows the
CONTRACT visible at those call sites -- grid [G,G,G] fp32 -> (verts [V,3] fp32 in [0,1]^3, faces
[F,3] integer), differentiable w.r.t. the grid -- with our own sm_90a marching cubes.  Vertex and
face ORDER are this implementation's (parity with diso is unpinned; see DESIGN.md)."""
import os
import sys

import torch
import torch.nn as nn

_root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _root not in sys.path:
    sys.path.insert(0, _root)
import _dgm_lib  # noqa: E402


_caps = {}      # (device, G) -> [V capacity, F capacity] of the previous surfaces (+ head-room)
_notify = {}    # device -> (handle, event, host pointer, ctypes view): early notification of {V, F}


def _notifier(dev_index):
    n = _notify.get(dev_index)
    if n is None:
        lib = _dgm_lib.lib()
        h = _dgm_lib.c_void_p()
        _dgm_lib.check(lib.dgm_notify_create(_dgm_lib.byref(h)), "dgm_notify_create")
        host = lib.dgm_notify_host(h)
        n = _notify[dev_index] = (h, lib.dgm_notify_event(h), host, (_dgm_lib.c_int32 * 2).from_address(host))
    return n


class _MCFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, grid, isovalue, normalize):
        if grid.dim() != 3 or not (grid.shape[0] == grid.shape[1] == grid.shape[2]):
            raise ValueError("DiffMC: cubic grid [G, G, G] expected")
        if not grid.is_cuda:
            raise ValueError("DiffMC: CUDA tensor required (no CPU fallback)")
        lib = _dgm_lib.lib()
        g = grid.contiguous().float()
        G, dev = g.shape[0], g.device
        nbytes = _dgm_lib.c_size_t()
        _dgm_lib.check(lib.dgmc_workspace_size(G, nbytes), "dgmc_workspace_size")
        ws = torch.empty((nbytes.value,), dtype=torch.uint8, device=dev)
        totals = torch.empty((2,), dtype=torch.int32, device=dev)
        st = _dgm_lib.stream_ptr()
        handle, event, host_ptr, words = _notifier(dev.index)
        _dgm_lib.check(lib.dgmc_count(G, g.data_ptr(), float(isovalue), ws.data_ptr(), nbytes.value,
                                      totals.data_ptr(), host_ptr, event, st), "dgmc_count")
        # Output sizes are data dependent (the reference's diso sizes its outputs with a host read too).  The
        # emission is enqueued OPTIMISTICALLY with the capacities the previous surface needed, THEN the host
        # waits for {V, F} (mirrored into pinned memory behind the count pass): the GPU keeps working while
        # the host waits, and only a surface that outgrew the capacity is emitted a second time.
        key = (dev.index, G)
        cap = _caps.get(key)

        def emit(vc, fc):
            v = torch.empty((vc, 3), dtype=torch.float32, device=dev)
            f = torch.empty((fc, 3), dtype=torch.int32, device=dev)
            _dgm_lib.check(lib.dgmc_emit(G, g.data_ptr(), float(isovalue), ws.data_ptr(), nbytes.value,
                                         _dgm_lib.ptr(v), vc, _dgm_lib.ptr(f), fc, st), "dgmc_emit")
            return v, f

        out = emit(*cap) if cap else None
        _dgm_lib.check(lib.dgm_notify_wait(handle), "dgm_notify_wait")
        V, F = int(words[0]), int(words[1])
        if out is None or V > cap[0] or F > cap[1]:
            out = emit(V, F) if (V or F) else (torch.empty((0, 3), dtype=torch.float32, device=dev),
                                               torch.empty((0, 3), dtype=torch.int32, device=dev))
        if len(_caps) > 32:
            _caps.clear()
        _caps[key] = [max(cap[0] if cap else 0, int(V * 1.25) + 1024), max(cap[1] if cap else 0, int(F * 1.25) + 1024)]
        verts, faces = out[0][:V], out[1][:F]
        if not normalize:
            verts = verts * float(G - 1)
        ctx.save_for_backward(g, ws)
        ctx.iso, ctx.normalize, ctx.nbytes, ctx.V = float(isovalue), normalize, nbytes.value, V
        ctx.mark_non_differentiable(faces)
        return verts, faces

    @staticmethod
    def backward(ctx, dverts, _):
        g, ws = ctx.saved_tensors
        G = g.shape[0]
        dphi = torch.empty_like(g)
        dv = dverts.contiguous().float()
        if not ctx.normalize:
            dv = dv * float(G - 1)
        _dgm_lib.check(_dgm_lib.lib().dgmc_backward(G, ctx.V, g.data_ptr(), ctx.iso, ws.data_ptr(), ctx.nbytes,
                                                    _dgm_lib.ptr(dv), dphi.data_ptr(), _dgm_lib.stream_ptr()),
                       "dgmc_backward")
        return dphi, None, None


class DiffMC(nn.Module):
    def __init__(self, dtype=torch.float32):
        super().__init__()
        if dtype != torch.float32:
            raise NotImplementedError("DiffMC : float32 only (what DG-Mesh instantiates)")

    def forward(self, grid, deform=None, isovalue=0.0, normalize=True):
        if deform is not None:
            raise NotImplementedError("DiffMC : deform=None only (what DG-Mesh passes)")
        verts, faces = _MCFunction.apply(grid, float(isovalue), bool(normalize))
        return verts, faces.long()


class DiffDMC(nn.Module):
    """Imported but never instantiated by DG-Mesh (gaussian_model_dpsr_dynamic_anchor.py:40)."""

    def __init__(self, *a, **k):
        super().__init__()
        raise NotImplementedError("DiffDMC is not part of the DG-Mesh hot path")
