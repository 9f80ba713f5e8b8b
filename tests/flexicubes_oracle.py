"""Vectorised torch float64 restatement of FlexiCubes (dg-mesh_b200/flexicubes.py, csrc/flexicubes.cu) on CPU.

The topology (which patches get a vertex, the quads in DiffDMC's orientation) and the vertex keys (cell, patch) are
tests/dmc_reference.py's; everything else follows the definition in flexicubes.py in float64 from the given inputs,
and its gradients come from autograd.  Vertex rows are dmc_reference's (cell-major, increasing patch); quad q's
centre vertex, in training mode, is row V + q of dmc_reference's quad order."""
import numpy as np
import torch

from dmc_reference import cell_cases, dmc_reference, tables


class FCRef:
    """verts [V (+Q), 3], faces [2Q or 4Q, 3] int64, L_dev [sum k_v], and the topology: dmc (the DMCRef), k [V]
    (crossings per vertex) and, in inference mode, near_tie [Q] (|g0 g2 - g1 g3| <= 1e-5 max)."""


def _safe_norm(x):
    sq = (x * x).sum(-1)
    pos = sq > 0
    return torch.where(pos, torch.sqrt(torch.where(pos, sq, torch.ones_like(sq))), torch.zeros_like(sq))


def flexicubes(phi, deform=None, beta=None, alpha=None, gamma_f=None, iso=0.0, training=False, normalize=True,
               dmc=None):
    """phi [G,G,G] (its float32 signs fix the topology) and the optional inputs, any float dtype; the outputs are
    float64 and differentiable in every tensor input that requires grad."""
    _, pof, edge_lo, _ = tables()
    phi_np = phi.detach().float().numpy()
    G = phi_np.shape[0]
    if dmc is None:
        dmc = dmc_reference(phi_np, iso)
    V, Q = len(dmc.verts), len(dmc.quads)
    cells = np.stack(np.unravel_index(dmc.cell, (G, G, G)), 1)                      # [V, 3]
    cs = cell_cases(phi_np < np.float32(iso))[tuple(cells.T)] if V else np.zeros(0, np.int64)
    member = torch.from_numpy(pof[cs] == dmc.patch[:, None]) if V else torch.zeros(0, 12, dtype=torch.bool)
    k = member.sum(1)
    wc = torch.from_numpy(np.ravel_multi_index(cells.T, (G - 1,) * 3) if V else np.zeros(0, np.int64))
    s = phi.double().reshape(-1) - float(np.float32(iso))
    grid = torch.stack(torch.meshgrid(*(torch.arange(G, dtype=torch.float64),) * 3, indexing="ij"), -1).reshape(-1, 3)
    x = grid if deform is None else grid + deform.double().reshape(-1, 3)
    al = (torch.ones(V, 8, dtype=torch.float64) if alpha is None
          else 1 + 0.99 * torch.tanh(alpha.double().reshape(-1, 8)[wc]))
    be = (torch.ones(V, 12, dtype=torch.float64) if beta is None
          else 1 + 0.99 * torch.tanh(beta.double().reshape(-1, 12)[wc]))
    ct = torch.from_numpy(cells)
    u, lo_r, hi_r = [], [], []
    for e in range(12):
        a, lo = e >> 2, int(edge_lo[e])
        hi = lo + (1 << a)
        n0 = ct + torch.tensor([lo & 1, (lo >> 1) & 1, lo >> 2])
        n1 = n0.clone()
        n1[:, a] += 1
        i0 = (n0[:, 0] * G + n0[:, 1]) * G + n0[:, 2]
        i1 = (n1[:, 0] * G + n1[:, 1]) * G + n1[:, 2]
        w0, w1 = al[:, lo] * s[i0], al[:, hi] * s[i1]
        den = torch.where(member[:, e], w0 - w1, torch.ones_like(w0))
        t = torch.where(member[:, e], w0 / den, torch.zeros_like(w0))
        u.append(x[i0] + t[:, None] * (x[i1] - x[i0]))
    u = torch.stack(u, 1)                                                           # [V, 12, 3]
    bm = torch.where(member, be, torch.zeros_like(be))
    v = (bm[:, :, None] * u).sum(1) / bm.sum(1, keepdim=True)                      # grid units
    scale = 1.0 / (G - 1) if normalize else 1.0
    d = _safe_norm(u - v[:, None, :]) * scale
    mean = torch.where(member, d, torch.zeros_like(d)).sum(1) / k.clamp(min=1)
    L_dev = (d - mean[:, None]).abs()[member]
    verts = v * scale
    quads = torch.from_numpy(dmc.quads)
    gam = (torch.full((V,), 0.5, dtype=torch.float64) if gamma_f is None
           else 0.005 + 0.99 * torch.sigmoid(gamma_f.double().reshape(-1)[wc]))
    out = FCRef()
    out.dmc, out.k = dmc, k.numpy()
    if Q:
        g = gam[quads]
        g02, g13 = g[:, 0] * g[:, 2], g[:, 1] * g[:, 3]
    if not training:
        if Q:
            a02 = (g02 >= g13).detach().numpy()[:, None]
            q = dmc.quads
            faces = np.concatenate([np.where(a02, q[:, [0, 1, 2]], q[:, [0, 1, 3]]),
                                    np.where(a02, q[:, [0, 2, 3]], q[:, [1, 2, 3]])], 1).reshape(-1, 3)
            mx = torch.maximum(g02, g13).detach()
            out.near_tie = ((g02 - g13).abs().detach() <= 1e-5 * mx).numpy()
        else:
            faces, out.near_tie = np.zeros((0, 3), np.int64), np.zeros(0, bool)
    else:
        if Q:
            vq = verts[quads]                                                       # [Q, 4, 3]
            m = ((g02[:, None] * (vq[:, 0] + vq[:, 2]) / 2 + g13[:, None] * (vq[:, 1] + vq[:, 3]) / 2)
                 / (g02 + g13 + 1e-8)[:, None])
            verts = torch.cat([verts, m])
            mid = V + np.arange(Q)
            q = dmc.quads
            faces = np.stack([np.stack([q[:, n], q[:, (n + 1) % 4], mid], 1) for n in range(4)], 1).reshape(-1, 3)
        else:
            faces = np.zeros((0, 3), np.int64)
    out.verts, out.faces, out.L_dev = verts, faces.astype(np.int64), L_dev
    return out
