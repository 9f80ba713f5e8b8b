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
                # (+ head-room); dual marching cubes keys ("dmc", device, G[, B]) -> [V capacity, Q capacity]
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


def _remember_caps(key, cap, V, P, max_verts):
    """The capacities the next call at `key` emits with: the counts V, P plus a quarter and 1024, never below the
    previous capacities `cap`, V at most max_verts."""
    if len(_caps) > 32:
        _caps.clear()
    _caps[key] = [min(max(cap[0] if cap else 0, int(V * 1.25) + 1024), max_verts),
                  max(cap[1] if cap else 0, int(P * 1.25) + 1024)]


class _Extractor:
    """The C entry points of one surface extractor.  Both count {V_k, P_k} per item (P: faces of marching cubes,
    quads of dual marching cubes), emit optimistically into caller capacities and map dL/dverts to dL/dphi; the
    dual extractor writes 2 triangles per quad (and, on request, the quads) and its backward takes a workspace."""

    def __init__(self, name, prefix, max_verts, dual):
        self.name, self.prefix, self.max_verts, self.dual = name, prefix, max_verts, dual

    def fn(self, lib, B, op):
        return getattr(lib, f"{self.prefix}_{op}" + ("" if B == 1 else "_batch"))

    def workspace(self, lib, B, G, dev):
        nbytes = _dgm_lib.c_size_t()
        args = (G, nbytes) if B == 1 else (B, G, nbytes)
        _dgm_lib.check(self.fn(lib, B, "workspace_size")(*args),
                       f"{self.prefix}_workspace_size" + ("" if B == 1 else "_batch"))
        return torch.empty((nbytes.value,), dtype=torch.uint8, device=dev), nbytes.value


_MC = _Extractor("DiffMC", "dgmc", _MAX_VERTS, False)
_DMC = _Extractor("DiffDMC", "dgdmc", 1 << 28, True)   # dgdmc_emit: V_cap <= 2^28


class _MCFunction(torch.autograd.Function):
    """grid [B, G, G, G] -> (verts [sum V_k, 3], faces [sum F_k, 3] with item-local indices, quads [sum Q_k, 4]
    (dual marching cubes with want_quads, else empty), counts [B, 2] on the host: {V_k, F_k}, or {V_k, Q_k} for
    dual marching cubes); B = 1 runs the single-grid entry points."""

    @staticmethod
    def forward(ctx, grid, isovalue, normalize, kind, want_quads):
        name = kind.name
        if grid.dim() != 4 or not (grid.shape[1] == grid.shape[2] == grid.shape[3]):
            raise ValueError(f"{name}: cubic grid [G, G, G] expected")
        if not 1 <= grid.shape[0] <= MAX_BATCH:
            raise ValueError(f"{name}: batch size must be in [1, {MAX_BATCH}], got {grid.shape[0]}")
        if not grid.is_cuda:
            raise ValueError(f"{name}: CUDA tensor required (no CPU fallback)")
        lib = _dgm_lib.lib()
        g = grid.contiguous().float()
        B, G, dev = g.shape[0], g.shape[1], g.device
        ws, nbytes = kind.workspace(lib, B, G, dev)
        totals = torch.empty((2 * B,), dtype=torch.int32, device=dev)
        st = _dgm_lib.stream_ptr()
        handle, event, host_ptr, words = _notifier(dev.index)
        lead = (G,) if B == 1 else (B, G)
        _dgm_lib.check(kind.fn(lib, B, "count")(*lead, g.data_ptr(), float(isovalue), ws.data_ptr(), nbytes,
                                                totals.data_ptr(), host_ptr, event, st),
                       f"{kind.prefix}_count" + ("" if B == 1 else "_batch"))
        # Output sizes are data dependent (the reference's diso sizes its outputs with a host read too).  The
        # emission is enqueued OPTIMISTICALLY with the capacities the previous surface needed, THEN the host
        # waits for the counts (mirrored into pinned memory behind the count pass): the GPU keeps working while
        # the host waits, and only a surface that outgrew the capacity is emitted a second time.
        key = ((dev.index, G) if B == 1 else (dev.index, G, B))
        if kind.dual:
            key = ("dmc",) + key
        cap = _caps.get(key)

        def emit(vc, pc):
            v = torch.empty((vc, 3), dtype=torch.float32, device=dev)
            src = torch.empty((vc,), dtype=torch.int32, device=dev)   # each vertex's grid edge / cell, for the backward
            f = torch.empty(((2 * pc if kind.dual else pc), 3), dtype=torch.int32, device=dev)
            q = torch.empty((pc if want_quads else 0, 4), dtype=torch.int32, device=dev)
            if vc or pc:
                out = (_dgm_lib.ptr(f), _dgm_lib.ptr(q), pc) if kind.dual else (_dgm_lib.ptr(f), pc)
                _dgm_lib.check(kind.fn(lib, B, "emit")(*lead, g.data_ptr(), float(isovalue), ws.data_ptr(), nbytes,
                                                       _dgm_lib.ptr(v), _dgm_lib.ptr(src), vc, *out, st),
                               f"{kind.prefix}_emit" + ("" if B == 1 else "_batch"))
            return v, src, f, q

        out = emit(*cap) if cap else None
        _dgm_lib.check(lib.dgm_notify_wait(handle), "dgm_notify_wait")
        counts = [(int(words[2 * k]), int(words[2 * k + 1])) for k in range(B)]
        V, P = sum(c[0] for c in counts), sum(c[1] for c in counts)
        if out is None or V > cap[0] or P > cap[1] or (want_quads and out[3].shape[0] < P):
            out = emit(V, P)      # V beyond what the emission can index is refused there (DgmError)
        _remember_caps(key, cap, V, P, kind.max_verts)
        verts, vsrc = out[0][:V], out[1][:V]
        faces, quads = out[2][:(2 * P if kind.dual else P)], out[3][:P]
        if not normalize:
            verts = verts * float(G - 1)
        ctx.save_for_backward(g, vsrc)
        ctx.iso, ctx.normalize, ctx.counts, ctx.kind = float(isovalue), normalize, counts, kind
        ctx.mark_non_differentiable(faces, quads)
        return verts, faces, quads, torch.tensor(counts, dtype=torch.int64).reshape(B, 2)

    @staticmethod
    def backward(ctx, dverts, _, __, ___):
        g, vsrc = ctx.saved_tensors
        B, G, kind = g.shape[0], g.shape[1], ctx.kind
        dphi = torch.empty_like(g)
        dv = dverts.contiguous().float()
        if not ctx.normalize:
            dv = dv * float(G - 1)
        lib = _dgm_lib.lib()
        nv = ctx.counts[0][0] if B == 1 else (_dgm_lib.c_int32 * B)(*[c[0] for c in ctx.counts])
        lead = (G, nv) if B == 1 else (B, G, nv)
        ws = ()
        if kind.dual:   # the backward's own workspace: the forward's is released with the forward
            wsb, nbytes = kind.workspace(lib, B, G, g.device)
            ws = (wsb.data_ptr(), nbytes)
        rc = kind.fn(lib, B, "backward")(*lead, g.data_ptr(), ctx.iso, *ws, _dgm_lib.ptr(vsrc), _dgm_lib.ptr(dv),
                                         dphi.data_ptr(), _dgm_lib.stream_ptr())
        _dgm_lib.check(rc, f"{kind.prefix}_backward" + ("" if B == 1 else "_batch"))
        return dphi, None, None, None, None


def _split(counts, verts, faces, per):
    """Item k's views of the concatenated verts and faces (per faces per counted primitive)."""
    vl, fl, v0, f0 = [], [], 0, 0
    for nv, nf in counts.tolist():
        vl.append(verts[v0:v0 + nv])
        fl.append(faces[f0:f0 + per * nf])
        v0, f0 = v0 + nv, f0 + per * nf
    return vl, fl


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
        verts, faces, _, _ = _MCFunction.apply(grid[None], float(isovalue), bool(normalize), _MC, False)
        return verts, faces.long()

    def forward_batch(self, grids, isovalue=0.0, normalize=True):
        """grids [B,G,G,G] (1 <= B <= 64) -> (verts list, faces list): item k's vertices and faces are exactly what
        `forward(grids[k])` gives, as views of one concatenated tensor each (faces int64, indices local to the item).
        One count pass, one emission and ONE host wait for the whole batch."""
        if grids.dim() != 4:
            raise ValueError("DiffMC.forward_batch: grids [B, G, G, G] expected")
        verts, faces, _, counts = _MCFunction.apply(grids, float(isovalue), bool(normalize), _MC, False)
        return _split(counts, verts, faces.long(), 1)


class DiffDMC(nn.Module):
    """Differentiable dual marching cubes (Nielson 2004) on sm_90a, with DiffMC's calling convention:
    `forward(grid, deform=None, isovalue=0.0, return_quads=False, normalize=True)` -> (verts [V,3] fp32 in
    [0,1]^3, faces [2Q,3] int64), or (verts, quads [Q,4] int64) with return_quads=True.

    - A node is inside when phi < isovalue; corners, edges and cases are those of marching cubes.
    - A cell's patches are the loops of its marching-cubes case (tools/gen_mc_tables.py): at most 4 per cell
      and 7 edges per patch, with the same ambiguous-face rule, so neighbouring cells agree.
    - A patch's vertex is the mean of its edge crossings (each one DiffMC's vertex on that edge), summed in fp32
      in increasing edge id, divided by the edge count, then by G - 1.  Only patches with an interior edge (one
      whose four cells lie in the grid) get a vertex, so no vertex is unreferenced.
    - Every sign-changing interior edge gives one quad over its four cells' vertices in cyclic order, oriented
      like DiffMC (normal from the inside node to the outside one), split into (q0,q1,q2), (q0,q2,q3) at the
      lowest cell q0.  Edges on the grid's outer faces give nothing.
    - The mesh of a closed level set is closed (every directed edge is matched by its reverse) but not always
      edge-manifold: where both cells beside an ambiguous face keep the face's two segments in one patch, a dual
      edge is shared by four triangles.
    - dL/dgrid flows through each crossing, weighted 1/k in a k-edge patch; none flows to isovalue.  The
      backward is bit-identical from run to run.
    Vertex and face order are this implementation's (parity with diso is unpinned)."""

    def __init__(self, dtype=torch.float32):
        super().__init__()
        if dtype != torch.float32:
            raise NotImplementedError("DiffDMC : float32 only (what DG-Mesh instantiates)")

    def forward(self, grid, deform=None, isovalue=0.0, return_quads=False, normalize=True):
        if deform is not None:
            raise NotImplementedError("DiffDMC : deform=None only")
        if grid.dim() != 3:
            raise ValueError("DiffDMC: cubic grid [G, G, G] expected")
        verts, faces, quads, _ = _MCFunction.apply(grid[None], float(isovalue), bool(normalize), _DMC,
                                                   bool(return_quads))
        return verts, (quads if return_quads else faces).long()

    def forward_batch(self, grids, isovalue=0.0, normalize=True):
        """grids [B,G,G,G] (1 <= B <= 64) -> (verts list, faces list): item k's vertices and faces are exactly what
        `forward(grids[k])` gives, as views of one concatenated tensor each (faces int64, indices local to the item).
        One count pass, one emission and ONE host wait for the whole batch."""
        if grids.dim() != 4:
            raise ValueError("DiffDMC.forward_batch: grids [B, G, G, G] expected")
        verts, faces, _, counts = _MCFunction.apply(grids, float(isovalue), bool(normalize), _DMC, False)
        return _split(counts, verts, faces.long(), 2)
