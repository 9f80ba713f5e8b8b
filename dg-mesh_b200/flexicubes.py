"""FlexiCubes (Shen et al., SIGGRAPH 2023; the extractor of nvdiffrec and kaolin) on sm_90a: dual marching cubes
with learnable node offsets, crossing and vertex weights and a weighted quad split, forward and backward.

`FlexiCubes()(scalar_field, deform=None, beta=None, alpha=None, gamma_f=None, isovalue=0.0, training=False,
normalize=True)` -> (vertices [V,3] or [V+Q,3] fp32, faces [2Q,3] or [4Q,3] int64, L_dev [sum_v k_v] fp32).

- Grid, corners, edges, cases, patches, "inside" (phi < isovalue) and which patches get a vertex are
  `diso.DiffDMC`'s, so V and Q are too.
- s = phi - isovalue.  Node n sits at n + deform[n] (grid units; `deform` [G,G,G,3]).  The raw per-cell weights
  `beta` [G-1,G-1,G-1,12], `alpha` [..,8] and `gamma_f` [G-1,G-1,G-1] are indexed by this project's numbering
  (corner r = (i + (r&1), j + ((r>>1)&1), k + (r>>2)); edge e = 4 axis + combo) and activated as kaolin does:
  beta = 1 + 0.99 tanh(b), alpha = 1 + 0.99 tanh(a), gamma = 0.005 + 0.99 sigmoid(g).  None is raw 0.
- Crossing on cut edge e with lower / upper corners r0 / r1: w0 = alpha[r0] s(n0), w1 = alpha[r1] s(n1),
  t = w0 / (w0 - w1), u_e = x0 + t (x1 - x0).
- Dual vertex: (sum_e beta[e] u_e) / (sum_e beta[e]), summed in increasing edge id, then divided by G - 1
  (normalize=False multiplies back by G - 1).  With neutral weights, no deform and isovalue 0 the vertices equal
  DiffDMC's bit for bit.
- training=False: each quad (q0,q1,q2,q3) of DiffDMC gives (q0,q1,q2), (q0,q2,q3) when gamma0 gamma2 >=
  gamma1 gamma3 (DiffDMC's faces with neutral weights), else (q0,q1,q3), (q1,q2,q3); no gradient to gamma_f.
- training=True: quad q gets a centre vertex at row V + q, m = (g02 (v0+v2)/2 + g13 (v1+v3)/2) / (g02 + g13 +
  1e-8) (g02 = gamma0 gamma2, g13 = gamma1 gamma3), and the triangles (q0,q1,m), (q1,q2,m), (q2,q3,m), (q3,q0,m).
- L_dev: for every dual vertex and every crossing of its patch, |d_e - mean_e d_e| with d_e = |u_e - v| in output
  units, in vertex order, then increasing edge id.  The gradient of |.| at 0 is 0.
- Gradients flow from the vertices and L_dev to scalar_field, deform, alpha, beta and (training) gamma_f, only to
  those autograd asks for; none flows to isovalue.  The backward is bit-identical from run to run.
The mesh is closed but, like DiffDMC's, not always edge-manifold (kaolin's ambiguity table is not applied).  Reading
L_dev's length back costs one host wait more than DiffDMC's forward."""
import os
import sys

import torch
import torch.nn as nn

_root = os.path.dirname(os.path.abspath(__file__))
if _root not in sys.path:
    sys.path.insert(0, _root)
import _dgm_lib  # noqa: E402
import diso  # noqa: E402

SLOTS = 7   # crossings per patch, at most
_MAX_VERTS = 1 << 28   # dgfc_emit: V_cap <= 2^28


class _FCFunction(torch.autograd.Function):
    """phi [G,G,G] and the optional offsets and raw weights -> (normalised verts [V (+Q), 3], faces int32, L_dev
    padded [V, SLOTS], crossings per vertex [V])."""

    @staticmethod
    def forward(ctx, phi, deform, alpha, beta, gamma_f, isovalue, training, normalize):
        lib = _dgm_lib.lib()
        G, dev = phi.shape[0], phi.device
        ws, nbytes = diso._DMC.workspace(lib, 1, G, dev)
        totals = torch.empty((2,), dtype=torch.int32, device=dev)
        st = _dgm_lib.stream_ptr()
        handle, event, host_ptr, words = diso._notifier(dev.index)
        _dgm_lib.check(lib.dgdmc_count(G, phi.data_ptr(), float(isovalue), ws.data_ptr(), nbytes, totals.data_ptr(),
                                       host_ptr, event, st), "dgdmc_count")
        weights = [_dgm_lib.ptr(t) for t in (deform, alpha, beta, gamma_f)]

        def emit(vc, qc):   # optimistic, as diso's extractors (diso._MCFunction.forward)
            v = torch.empty((vc + (qc if training else 0), 3), dtype=torch.float32, device=dev)
            src = torch.empty((vc,), dtype=torch.int32, device=dev)
            ld = torch.empty((vc, SLOTS), dtype=torch.float32, device=dev)
            vk = torch.empty((vc,), dtype=torch.int32, device=dev)
            f = torch.empty(((4 if training else 2) * qc, 3), dtype=torch.int32, device=dev)
            q = torch.empty((qc, 4), dtype=torch.int32, device=dev)
            if vc or qc:
                _dgm_lib.check(lib.dgfc_emit(G, phi.data_ptr(), float(isovalue), *weights, int(training),
                                             int(normalize), ws.data_ptr(), nbytes, _dgm_lib.ptr(v),
                                             _dgm_lib.ptr(src), _dgm_lib.ptr(ld), _dgm_lib.ptr(vk), vc,
                                             _dgm_lib.ptr(f), _dgm_lib.ptr(q), qc, st), "dgfc_emit")
            return v, src, ld, vk, f, q

        key = ("fc", dev.index, G, bool(training))
        cap = diso._caps.get(key)
        out = emit(*cap) if cap else None
        _dgm_lib.check(lib.dgm_notify_wait(handle), "dgm_notify_wait")
        V, Q = int(words[0]), int(words[1])
        if out is None or V > cap[0] or Q > cap[1]:
            out = emit(V, Q)
        diso._remember_caps(key, cap, V, Q, _MAX_VERTS)
        v, src, ld, vk, f, q = out
        verts = v[:V + (Q if training else 0)]
        faces = f[:(4 if training else 2) * Q]
        ctx.save_for_backward(phi, deform, alpha, beta, gamma_f, verts, src[:V], q[:Q])
        ctx.V, ctx.Q, ctx.iso, ctx.training, ctx.normalize = V, Q, float(isovalue), bool(training), bool(normalize)
        ctx.mark_non_differentiable(faces, vk)
        return verts, faces, ld[:V], vk[:V]

    @staticmethod
    def backward(ctx, dverts, _, dldev, __):
        phi, deform, alpha, beta, gamma_f, verts, vsrc, quads = ctx.saved_tensors
        G, V, Q, training = phi.shape[0], ctx.V, ctx.Q, ctx.training
        need = ctx.needs_input_grad
        dv = torch.zeros_like(verts) if dverts is None else dverts.contiguous().float()
        dld = None if dldev is None else dldev.contiguous().float()
        dphi = torch.empty_like(phi)
        outs = [torch.empty_like(t) if (t is not None and need[i + 1]) else None
                for i, t in enumerate((deform, alpha, beta, gamma_f))]
        if not training:
            outs[3] = None
        lib = _dgm_lib.lib()
        nbytes = _dgm_lib.c_size_t()
        _dgm_lib.check(lib.dgfc_backward_workspace_size(G, V, Q, int(training), _dgm_lib.byref(nbytes)),
                       "dgfc_backward_workspace_size")
        ws = torch.empty((nbytes.value,), dtype=torch.uint8, device=phi.device)
        _dgm_lib.check(lib.dgfc_backward(G, V, Q, phi.data_ptr(), ctx.iso,
                                         *[_dgm_lib.ptr(t) for t in (deform, alpha, beta, gamma_f)],
                                         int(training), int(ctx.normalize), _dgm_lib.ptr(verts), _dgm_lib.ptr(vsrc),
                                         _dgm_lib.ptr(quads), _dgm_lib.ptr(dv), _dgm_lib.ptr(dld), ws.data_ptr(),
                                         nbytes.value, dphi.data_ptr(), *[_dgm_lib.ptr(t) for t in outs],
                                         _dgm_lib.stream_ptr()), "dgfc_backward")
        return (dphi if need[0] else None), *outs, None, None, None


def _check(name, t, shape, dev):
    if t is None:
        return None
    if not isinstance(t, torch.Tensor) or t.dtype != torch.float32:
        raise ValueError(f"FlexiCubes: {name} must be a float32 tensor")
    if tuple(t.shape) != shape:
        raise ValueError(f"FlexiCubes: {name} must have shape {list(shape)}, got {list(t.shape)}")
    if t.device != dev:
        raise ValueError(f"FlexiCubes: {name} must be on {dev}, like the scalar field")
    return t.contiguous()


class FlexiCubes(nn.Module):
    """The FlexiCubes extractor defined in this module's docstring."""

    def forward(self, scalar_field, deform=None, beta=None, alpha=None, gamma_f=None, isovalue=0.0, training=False,
                normalize=True):
        phi = scalar_field
        if not isinstance(phi, torch.Tensor) or phi.dim() != 3 or not (phi.shape[0] == phi.shape[1] == phi.shape[2]):
            raise ValueError("FlexiCubes: cubic grid [G, G, G] expected")
        if phi.dtype != torch.float32:
            raise ValueError("FlexiCubes: float32 scalar field expected")
        G = phi.shape[0]
        if not 2 <= G <= 800:
            raise ValueError(f"FlexiCubes: 2 <= G <= 800 required, got {G}")
        c = (G - 1,) * 3
        deform = _check("deform", deform, (G, G, G, 3), phi.device)
        beta = _check("beta", beta, c + (12,), phi.device)
        alpha = _check("alpha", alpha, c + (8,), phi.device)
        gamma_f = _check("gamma_f", gamma_f, c, phi.device)
        if not phi.is_cuda:
            raise ValueError("FlexiCubes: CUDA tensor required (no CPU fallback)")
        verts, faces, ld, vk = _FCFunction.apply(phi.contiguous(), deform, alpha, beta, gamma_f, float(isovalue),
                                                 bool(training), bool(normalize))
        if not normalize:
            verts = verts * float(G - 1)
        L_dev = ld[torch.arange(SLOTS, device=ld.device) < vk[:, None]]
        return verts, faces.long(), L_dev
