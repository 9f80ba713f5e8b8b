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


_caps = {}      # (device, G), or (device, G, B) for a batch -> [V capacity, F capacity] of the previous surfaces
                # (+ head-room)
_MAX_VERTS = 1 << 29   # dgmc_emit packs vertex indices into 29 bits (include/dgmesh_b200.h), a batch's total too
MAX_BATCH = 64  # grids per forward_batch call
_notify = {}    # device -> (handle, event, host pointer, ctypes view): early notification of {V_k, F_k}


def _notifier(dev_index):
    n = _notify.get(dev_index)
    if n is None:
        lib = _dgm_lib.lib()
        h = _dgm_lib.c_void_p()
        _dgm_lib.check(lib.dgm_notify_create(_dgm_lib.byref(h)), "dgm_notify_create")
        host = lib.dgm_notify_host(h)
        n = _notify[dev_index] = (h, lib.dgm_notify_event(h), host,
                                  (_dgm_lib.c_int32 * (2 * MAX_BATCH)).from_address(host))
    return n


class _MCFunction(torch.autograd.Function):
    """grid [B, G, G, G] -> (verts [sum V_k, 3], faces [sum F_k, 3] with item-local indices, counts [B, 2] on the
    host); B = 1 runs the single-grid entry points."""

    @staticmethod
    def forward(ctx, grid, isovalue, normalize):
        if grid.dim() != 4 or not (grid.shape[1] == grid.shape[2] == grid.shape[3]):
            raise ValueError("DiffMC: cubic grid [G, G, G] expected")
        if not 1 <= grid.shape[0] <= MAX_BATCH:
            raise ValueError(f"DiffMC: batch size must be in [1, {MAX_BATCH}], got {grid.shape[0]}")
        if not grid.is_cuda:
            raise ValueError("DiffMC: CUDA tensor required (no CPU fallback)")
        lib = _dgm_lib.lib()
        g = grid.contiguous().float()
        B, G, dev = g.shape[0], g.shape[1], g.device
        nbytes = _dgm_lib.c_size_t()
        if B == 1:
            _dgm_lib.check(lib.dgmc_workspace_size(G, nbytes), "dgmc_workspace_size")
        else:
            _dgm_lib.check(lib.dgmc_workspace_size_batch(B, G, nbytes), "dgmc_workspace_size_batch")
        ws = torch.empty((nbytes.value,), dtype=torch.uint8, device=dev)
        totals = torch.empty((2 * B,), dtype=torch.int32, device=dev)
        st = _dgm_lib.stream_ptr()
        handle, event, host_ptr, words = _notifier(dev.index)
        if B == 1:
            _dgm_lib.check(lib.dgmc_count(G, g.data_ptr(), float(isovalue), ws.data_ptr(), nbytes.value,
                                          totals.data_ptr(), host_ptr, event, st), "dgmc_count")
        else:
            _dgm_lib.check(lib.dgmc_count_batch(B, G, g.data_ptr(), float(isovalue), ws.data_ptr(), nbytes.value,
                                                totals.data_ptr(), host_ptr, event, st), "dgmc_count_batch")
        # Output sizes are data dependent (the reference's diso sizes its outputs with a host read too).  The
        # emission is enqueued OPTIMISTICALLY with the capacities the previous surface needed, THEN the host
        # waits for {V, F} (mirrored into pinned memory behind the count pass): the GPU keeps working while
        # the host waits, and only a surface that outgrew the capacity is emitted a second time.
        key = (dev.index, G) if B == 1 else (dev.index, G, B)
        cap = _caps.get(key)

        def emit(vc, fc):
            v = torch.empty((vc, 3), dtype=torch.float32, device=dev)
            src = torch.empty((vc,), dtype=torch.int32, device=dev)   # each vertex's grid edge, for the backward
            f = torch.empty((fc, 3), dtype=torch.int32, device=dev)
            if vc or fc:
                if B == 1:
                    _dgm_lib.check(lib.dgmc_emit(G, g.data_ptr(), float(isovalue), ws.data_ptr(), nbytes.value,
                                                 _dgm_lib.ptr(v), _dgm_lib.ptr(src), vc, _dgm_lib.ptr(f), fc, st),
                                   "dgmc_emit")
                else:
                    _dgm_lib.check(lib.dgmc_emit_batch(B, G, g.data_ptr(), float(isovalue), ws.data_ptr(),
                                                       nbytes.value, _dgm_lib.ptr(v), _dgm_lib.ptr(src), vc,
                                                       _dgm_lib.ptr(f), fc, st), "dgmc_emit_batch")
            return v, src, f

        out = emit(*cap) if cap else None
        _dgm_lib.check(lib.dgm_notify_wait(handle), "dgm_notify_wait")
        counts = [(int(words[2 * k]), int(words[2 * k + 1])) for k in range(B)]
        V, F = sum(c[0] for c in counts), sum(c[1] for c in counts)
        if out is None or V > cap[0] or F > cap[1]:
            out = emit(V, F)      # V beyond what dgmc_emit can index is refused there (DgmError)
        if len(_caps) > 32:
            _caps.clear()
        _caps[key] = [min(max(cap[0] if cap else 0, int(V * 1.25) + 1024), _MAX_VERTS),
                      max(cap[1] if cap else 0, int(F * 1.25) + 1024)]
        verts, vsrc, faces = out[0][:V], out[1][:V], out[2][:F]
        if not normalize:
            verts = verts * float(G - 1)
        ctx.save_for_backward(g, vsrc)
        ctx.iso, ctx.normalize, ctx.counts = float(isovalue), normalize, counts
        ctx.mark_non_differentiable(faces)
        return verts, faces, torch.tensor(counts, dtype=torch.int64).reshape(B, 2)

    @staticmethod
    def backward(ctx, dverts, _, __):
        g, vsrc = ctx.saved_tensors
        B, G = g.shape[0], g.shape[1]
        dphi = torch.empty_like(g)
        dv = dverts.contiguous().float()
        if not ctx.normalize:
            dv = dv * float(G - 1)
        lib = _dgm_lib.lib()
        if B == 1:
            rc = lib.dgmc_backward(G, ctx.counts[0][0], g.data_ptr(), ctx.iso, _dgm_lib.ptr(vsrc), _dgm_lib.ptr(dv),
                                   dphi.data_ptr(), _dgm_lib.stream_ptr())
            _dgm_lib.check(rc, "dgmc_backward")
        else:
            nv = (_dgm_lib.c_int32 * B)(*[c[0] for c in ctx.counts])
            rc = lib.dgmc_backward_batch(B, G, nv, g.data_ptr(), ctx.iso, _dgm_lib.ptr(vsrc), _dgm_lib.ptr(dv),
                                         dphi.data_ptr(), _dgm_lib.stream_ptr())
            _dgm_lib.check(rc, "dgmc_backward_batch")
        return dphi, None, None


class DiffMC(nn.Module):
    def __init__(self, dtype=torch.float32):
        super().__init__()
        if dtype != torch.float32:
            raise NotImplementedError("DiffMC : float32 only (what DG-Mesh instantiates)")

    def forward(self, grid, deform=None, isovalue=0.0, normalize=True):
        if deform is not None:
            raise NotImplementedError("DiffMC : deform=None only (what DG-Mesh passes)")
        if grid.dim() != 3:
            raise ValueError("DiffMC: cubic grid [G, G, G] expected")
        verts, faces, _ = _MCFunction.apply(grid[None], float(isovalue), bool(normalize))
        return verts, faces.long()

    def forward_batch(self, grids, isovalue=0.0, normalize=True):
        """grids [B,G,G,G] (1 <= B <= 64) -> (verts list, faces list): item k's vertices and faces are exactly what
        `forward(grids[k])` gives, as views of one concatenated tensor each (faces int64, indices local to the item).
        One count pass, one emission and ONE host wait for the whole batch."""
        if grids.dim() != 4:
            raise ValueError("DiffMC.forward_batch: grids [B, G, G, G] expected")
        verts, faces, counts = _MCFunction.apply(grids, float(isovalue), bool(normalize))
        faces = faces.long()
        vl, fl, v0, f0 = [], [], 0, 0
        for nv, nf in counts.tolist():
            vl.append(verts[v0:v0 + nv])
            fl.append(faces[f0:f0 + nf])
            v0, f0 = v0 + nv, f0 + nf
        return vl, fl


class DiffDMC(nn.Module):
    """Imported but never instantiated by DG-Mesh (gaussian_model_dpsr_dynamic_anchor.py:40)."""

    def __init__(self, *a, **k):
        super().__init__()
        raise NotImplementedError("DiffDMC is not part of the DG-Mesh hot path")
