"""Float64 statement of the hash-grid field (dg-mesh_b200/hashgrid.py, csrc/hashgrid.cu): the two coordinate steps
(u = (x - lo) / (hi - lo), clamped; p = u R) in float32 exactly as specified, the slot arithmetic in int64 masked to
32 bits, the blend, dL/dx and the table gradients (index_add_) in float64."""
import torch

GRIDS = ("xyz", "xyt", "yzt", "xzt")
AXES = {"xyz": (0, 1, 2), "xyt": (0, 1, 3), "yzt": (1, 2, 3), "xzt": (0, 2, 3)}
PRIMES = (1, 2654435761, 805459861)
M32 = 0xFFFFFFFF


def slots(idx, R3, T):
    """idx [..., 3] int64 node indices, R3 the three axis resolutions -> slots [...] int64."""
    if (R3[0] + 1) * (R3[1] + 1) * (R3[2] + 1) <= T:
        return idx[..., 0] + (R3[0] + 1) * (idx[..., 1] + (R3[1] + 1) * idx[..., 2])
    h = ((idx[..., 0] * PRIMES[0]) & M32) ^ ((idx[..., 1] * PRIMES[1]) & M32) ^ ((idx[..., 2] * PRIMES[2]) & M32)
    return h & (T - 1)


def coords(x, t, box, coord_dtype=torch.float32):
    """u [F,N,4] (clamped) and du/dx [N,3] (0 where the unclamped u is outside [0, 1]), in coord_dtype."""
    lo, hi = box[0].to(coord_dtype), box[1].to(coord_dtype)
    w = hi - lo
    raw = (x.to(coord_dtype) - lo) / w
    u = raw.clamp(0, 1)
    dudx = torch.where((raw >= 0) & (raw <= 1), 1 / w.double(), torch.zeros((), dtype=torch.float64))
    F, N = t.shape[0], x.shape[0]
    tt = t.reshape(F, N).to(coord_dtype).clamp(0, 1)
    return torch.cat([u[None].expand(F, N, 3), tt[..., None]], -1), dudx


def _cell(u, grid, R, Rt):
    """u [F,N,4] -> (node indices [F,N,8,3] int64, weights [F,N,8], dweights/dw [F,N,8,3], R3)."""
    ax = AXES[grid]
    R3 = [Rt if a == 3 else R for a in ax]
    c, w = [], []
    for a, Ra in zip(ax, R3):
        p = u[..., a] * Ra                                   # one rounded product in u's dtype
        ci = torch.clamp(torch.floor(p), max=Ra - 1)
        c.append(ci.long())
        w.append((p - ci).double())
    corners = torch.tensor([[(k >> j) & 1 for j in range(3)] for k in range(8)])          # [8, 3]
    idx = torch.stack(c, -1)[..., None, :] + corners                                     # [F,N,8,3]
    fac = [torch.where(corners[:, j].bool(), w[j][..., None], 1 - w[j][..., None]) for j in range(3)]
    sgn = corners.double() * 2 - 1
    wt = fac[0] * fac[1] * fac[2]
    dwt = torch.stack([sgn[:, 0] * fac[1] * fac[2], sgn[:, 1] * fac[0] * fac[2], sgn[:, 2] * fac[0] * fac[1]], -1)
    return idx, wt, dwt, R3


def field_and_grads(x, t, box, tables, grids, resolutions, time_resolution, log2_table, grad_out=None,
                    coord_dtype=torch.float32):
    """x [N,3], t [F,N,1] or [N,1] or None (xyz only), tables: one [L, T, Fe] per grid.  Returns (features
    [F,N,G L Fe] or [N, G L Fe], dL/dx [N,3], [dL/dtable]) in float64 for L = sum grad_out * features; the gradients
    are None without grad_out."""
    batched = t is not None and t.dim() == 3
    N = x.shape[0]
    t3 = (t if batched else t[None]) if t is not None else torch.zeros(1, N, 1)
    F = t3.shape[0]
    u, dudx = coords(x.detach().cpu(), t3.detach().cpu(), box.detach().cpu(), coord_dtype)
    T = 2 ** log2_table
    tabs = [p.detach().cpu().double() for p in tables]
    L, Fe = tabs[0].shape[0], tabs[0].shape[2]
    go = None
    if grad_out is not None:
        go = grad_out.detach().cpu().double()
        go = (go if batched else go[None]).reshape(F, N, len(grids), L, Fe)
    out = torch.zeros(F, N, len(grids), L, Fe, dtype=torch.float64)
    gx = torch.zeros(N, 3, dtype=torch.float64)
    gt = [torch.zeros_like(p) for p in tabs]
    for g, grid in enumerate(grids):
        for l, R in enumerate(resolutions):
            idx, wt, dwt, R3 = _cell(u, grid, R, min(R, time_resolution))
            s = slots(idx, R3, T)                                                # [F,N,8]
            rows = tabs[g][l][s]                                                 # [F,N,8,Fe]
            out[:, :, g, l] = (wt[..., None] * rows).sum(2)
            if go is None:
                continue
            gg = go[:, :, g, l]                                                  # [F,N,Fe]
            gt[g][l].index_add_(0, s.reshape(-1), (wt[..., None] * gg[:, :, None]).reshape(-1, Fe))
            sk = (rows * gg[:, :, None]).sum(-1)                                 # [F,N,8]
            dw = (sk[..., None] * dwt).sum(2)                                    # [F,N,3]
            for j, a in enumerate(AXES[grid]):
                if a < 3:
                    gx[:, a] += (dw[..., j] * R3[j]).sum(0) * dudx[:, a]
    out = out.reshape(F, N, -1)
    out = out if batched else out[0]
    return (out, gx, gt) if go is not None else (out, None, None)


def field(x, t, box, tables, grids, resolutions, time_resolution, log2_table, coord_dtype=torch.float32):
    return field_and_grads(x, t, box, tables, grids, resolutions, time_resolution, log2_table,
                           coord_dtype=coord_dtype)[0]


def of(f, x, t, grad_out=None):
    """field_and_grads for a HashGridField f."""
    return field_and_grads(x, t, f.box, list(f.tables), f.grids, f.resolutions, f.time_resolution, f.log2_table,
                           grad_out)
