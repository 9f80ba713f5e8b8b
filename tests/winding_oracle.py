"""float64 restatement of the generalized winding number (csrc/winding.cu, mesh_distance.winding_number): the exact
solid-angle sum over all faces, in chunks (torch float64 on any device, so large meshes can be checked on the GPU),
and, in numpy, Barill et al. 2018's order-1 moments of a cluster of faces, their merge and the far-field term."""
import numpy as np
import torch


def _np(x, dtype=np.float64):
    if hasattr(x, "detach"):
        x = x.detach().cpu().numpy()
    return np.asarray(x, dtype=dtype)


def _t(x, device, dtype=torch.float64):
    return torch.as_tensor(_np(x, np.float64 if dtype == torch.float64 else np.int64), dtype=dtype, device=device)


def solid_angles(q, v, f, device="cpu"):
    """[Q, F] float64 solid angles 2 atan2(det[a b c], |a||b||c| + (a.b)|c| + (b.c)|a| + (c.a)|b|), a, b, c = the
    face's vertices minus q; 0 where det is exactly 0 (as the kernel).  Computed in torch on `device`."""
    q, v, f = _t(q, device), _t(v, device), _t(f, device, torch.int64)
    a = v[f[:, 0]][None] - q[:, None]
    b = v[f[:, 1]][None] - q[:, None]
    c = v[f[:, 2]][None] - q[:, None]
    det = (a * torch.linalg.cross(b, c)).sum(2)
    la, lb, lc = (x.norm(dim=2) for x in (a, b, c))
    den = la * lb * lc + (a * b).sum(2) * lc + (b * c).sum(2) * la + (c * a).sum(2) * lb
    return torch.where(det == 0.0, torch.zeros_like(det), 2.0 * torch.atan2(det, den))


def winding(q, v, f, device="cpu", pairs=1 << 22):
    """[Q] numpy float64 exact generalized winding number: the sum of the solid angles over all faces / 4 pi, in
    chunks of about `pairs` (query, face) pairs."""
    q = _np(q)
    F = len(_np(f, np.int64))
    step = max(1, pairs // max(F, 1))
    out = np.empty(len(q))
    for i in range(0, len(q), step):
        out[i:i + step] = (solid_angles(q[i:i + step], v, f, device).sum(1) / (4 * np.pi)).cpu().numpy()
    return out


def moments(v, f):
    """Order-1 expansion of the cluster of faces f: (p~ [3], N [3], M [3,3], r, A) with a_t n_t = 1/2 (b-a) x (c-a),
    A = sum |a_t n_t|, p~ = sum |a_t n_t| x_t / A (x_t the centroid), N = sum a_t n_t, M = sum (x_t - p~) (a_t n_t)^T
    and r = max |vertex - p~|."""
    v, f = _np(v), _np(f, np.int64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    n = 0.5 * np.cross(b - a, c - a)
    area = np.linalg.norm(n, axis=1)
    x = (a + b + c) / 3
    A = area.sum()
    p = (area[:, None] * x).sum(0) / A
    M = np.einsum("ti,tj->ij", x - p, n)
    r = np.linalg.norm(v[np.unique(f)] - p, axis=1).max()
    return p, n.sum(0), M, r, A


def merge(e0, e1):
    """The expansion of the union of two clusters from theirs, as csrc/winding.cu merges child records: p~ the
    area-weighted mean, N the sum, M re-centred, M = M0 + (p~0 - p~) N0^T + M1 + (p~1 - p~) N1^T, and the child
    bound r = max(|p~0 - p~| + r0, |p~1 - p~| + r1)."""
    (p0, n0, m0, r0, a0), (p1, n1, m1, r1, a1) = e0, e1
    A = a0 + a1
    p = (a0 * p0 + a1 * p1) / A
    M = m0 + np.outer(p0 - p, n0) + m1 + np.outer(p1 - p, n1)
    r = max(np.linalg.norm(p0 - p) + r0, np.linalg.norm(p1 - p) + r1)
    return p, n0 + n1, M, r, A


def far_field(q, p, N, M):
    """[Q] order-1 far-field winding number of a cluster (p~, N, M) at q: the Taylor expansion of the dipole kernel
    (x - q) / |x - q|^3 about p~, (y.N / d^3 + tr M / d^3 - 3 y^T M y / d^5) / 4 pi with y = p~ - q, d = |y|."""
    y = _np(p)[None] - _np(q)
    d = np.linalg.norm(y, axis=1)
    yMy = np.einsum("qi,ij,qj->q", y, M, y)
    return (y @ N / d ** 3 + np.trace(M) / d ** 3 - 3 * yMy / d ** 5) / (4 * np.pi)


def polyhedron_volume(v, f):
    """Signed volume of a closed, consistently oriented mesh (divergence theorem): sum a . (b x c) / 6."""
    v, f = _np(v), _np(f, np.int64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    return float(np.einsum("tk,tk->t", a, np.cross(b, c)).sum() / 6)
