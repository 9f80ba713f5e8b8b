"""Float64 statement of the HexPlane field and its regularisers (dg-mesh_b200/hexplane.py, csrc/hexplane.cu), through
F.grid_sample on channels-first copies of the planes; its autograd gives the reference gradients."""
import torch
import torch.nn.functional as Fn

PAIRS = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))
SPATIAL, TIME = (0, 1, 3), (2, 4, 5)


def field(x, t, box, planes, S):
    """x [N,3], t [F,N,1] (or [N,1]), box [2,3], planes: 6 S tensors [R_b, R_a, C] -> [F,N,S C] (or [N,S C]) in the
    dtype of the planes."""
    dt = planes[0].dtype
    batched = t.dim() == 3
    t3 = t if batched else t[None]
    Fr, N = t3.shape[0], x.shape[0]
    lo, hi = box[0].to(dt), box[1].to(dt)
    u = 2 * (x.to(dt) - lo) / (hi - lo) - 1                      # [N,3]
    tau = 2 * t3.to(dt) - 1                                     # [F,N,1]
    coords = torch.cat([u[None].expand(Fr, N, 3), tau], -1).reshape(Fr * N, 4)
    out = []
    for s in range(S):
        f = None
        for p, (a, b) in enumerate(PAIRS):
            G = planes[6 * s + p].permute(2, 0, 1)[None]         # [1, C, R_b, R_a]
            grid = torch.stack([coords[:, a], coords[:, b]], -1)[None, :, None]   # [1, M, 1, 2]: (width, height)
            v = Fn.grid_sample(G, grid, mode="bilinear", padding_mode="border", align_corners=True)
            v = v[0, :, :, 0].T                                   # [M, C]
            f = v if f is None else f * v
        out.append(f)
    res = torch.cat(out, -1).reshape(Fr, N, -1)
    return res if batched else res[0]


def regularisers(planes, S):
    """(tv, time_smooth, l1_time), each a sum over planes and scales of means (time_smooth 0 when R_t = 2)."""
    tv = ts = l1 = 0
    for s in range(S):
        for p in SPATIAL:
            G = planes[6 * s + p]
            tv = tv + (G[1:] - G[:-1]).square().mean() + (G[:, 1:] - G[:, :-1]).square().mean()
        for p in TIME:
            G = planes[6 * s + p]
            if G.shape[0] > 2:
                ts = ts + (G[2:] - 2 * G[1:-1] + G[:-2]).square().mean()
            l1 = l1 + (1 - G).abs().mean()
    z = planes[0].new_zeros(())
    return tuple(v if torch.is_tensor(v) else z for v in (tv, ts, l1))


def field_and_grads(x, t, box, planes, S, grad_out):
    """(features, dL/dx, [dL/dplane]) in float64 for L = sum grad_out * features."""
    xd = x.detach().double().requires_grad_(True)
    pd = [p.detach().double().requires_grad_(True) for p in planes]
    out = field(xd, t.detach().double(), box.double(), pd, S)
    gx, *gp = torch.autograd.grad(out, [xd] + pd, grad_out.double())
    return out.detach(), gx, gp


def regularisers_and_grads(planes, S, weights):
    pd = [p.detach().double().requires_grad_(True) for p in planes]
    ls = regularisers(pd, S)
    total = sum(w * v for w, v in zip(weights, ls))
    gp = torch.autograd.grad(total, pd)
    return [v.detach() for v in ls], gp
