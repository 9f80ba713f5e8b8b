"""Mesh-to-mesh metrics of DG-Mesh's evaluation: Chamfer distance and the approximate EMD between surface samples
(PointFlow's `cd` and `emd_approx`, on metrics.pytorch_structural_losses), plus F-score, normal consistency and,
optionally, volumetric IoU.

Meshes are (verts [V,3], faces [F,3]) in the caller's units: nothing is normalised, aligned or cleaned.  Sampling is
plain torch (it is not a hot path); the distances, the closest points on a surface and the matching run on this
package's sm_90a kernels."""
import math
import os
import sys

import torch

_root = os.path.dirname(os.path.abspath(__file__))
if _root not in sys.path:
    sys.path.insert(0, _root)
from metrics.pytorch_structural_losses.match_cost import match_cost  # noqa: E402
from metrics.pytorch_structural_losses.nn_distance import nn_distance_with_indices  # noqa: E402
from mesh_distance import point_mesh_distance, winding_number  # noqa: E402


def sample_surface(verts, faces, n, generator=None):
    """(points [n,3], face_index [n] int64, normals [n,3]): n points uniform in area over the mesh.

    The face is drawn by inverse CDF over the float64 cumulative face areas with torch.rand(generator=...); the
    point inside it from two more uniforms u, v, reflected as trimesh does (u + v > 1 -> 1 - u, 1 - v), at
    a + u (b - a) + v (c - a).  normals are the unit face normals (right-handed in the face's vertex order).  Points
    and normals have verts' dtype and device; the random numbers come from `generator`'s device (verts' device
    without one).  Raises ValueError for bad shapes, n < 1 or a mesh of zero total area."""
    if not torch.is_tensor(verts) or verts.dim() != 2 or verts.shape[1] != 3 or not verts.is_floating_point():
        raise ValueError("sample_surface: verts must be a floating-point tensor [V, 3]")
    if not torch.is_tensor(faces) or faces.dim() != 2 or faces.shape[1] != 3 or faces.shape[0] < 1 or \
            faces.is_floating_point():
        raise ValueError("sample_surface: faces must be an integer tensor [F, 3] with F >= 1")
    if isinstance(n, bool) or not isinstance(n, int) or n < 1:
        raise ValueError("sample_surface: n must be an int >= 1")
    f = faces.to(verts.device, torch.int64)
    a, b, c = verts[f[:, 0]], verts[f[:, 1]], verts[f[:, 2]]
    cross = torch.linalg.cross(b - a, c - a)
    area = 0.5 * torch.linalg.norm(cross.double(), dim=1)
    cdf = torch.cumsum(area, 0)
    total = float(cdf[-1])
    if not (total > 0.0 and math.isfinite(total)):
        raise ValueError("sample_surface: the mesh has zero (or non-finite) total area")
    rdev = generator.device if generator is not None else verts.device
    r = torch.rand(n, dtype=torch.float64, generator=generator, device=rdev).to(verts.device)
    # first face whose cumulative area exceeds r * total: never a zero-area face
    face = torch.searchsorted(cdf, r * total, right=True).clamp_(max=f.shape[0] - 1)
    uv = torch.rand(n, 2, dtype=verts.dtype, generator=generator, device=rdev).to(verts.device)
    flip = uv.sum(1) > 1
    uv[flip] = 1 - uv[flip]
    u, v = uv[:, :1], uv[:, 1:]
    points = a[face] + u * (b[face] - a[face]) + v * (c[face] - a[face])
    normals = torch.nn.functional.normalize(cross, dim=1)[face]
    return points, face, normals


def _mesh(m, name):
    if not isinstance(m, (tuple, list)) or len(m) != 2:
        raise ValueError(f"mesh_metrics: {name} must be a pair (verts [V,3], faces [F,3])")
    return m


def _face_normals(verts, faces):
    """Unit normals of every face, as sample_surface computes them (zero for a face without area)."""
    f = faces.to(verts.device, torch.int64)
    a, b, c = verts[f[:, 0]], verts[f[:, 1]], verts[f[:, 2]]
    return torch.nn.functional.normalize(torch.linalg.cross(b - a, c - a), dim=1)


def mesh_metrics(pred, gt, n_points, thresholds=(), generator=None, surface=False, iou_points=0):
    """Sample n_points on each mesh (sample_surface, pred first) and compare the samples.

    pred, gt: (verts [V,3], faces [F,3]); the samples go to the device of pred's verts, which must be CUDA.
    Returns a dict of floats:
      chamfer_l2 = mean dist1 + mean dist2 (squared nearest-neighbour distances; PointFlow's `cd`),
      chamfer_l1 = (mean sqrt(dist1) + mean sqrt(dist2)) / 2,
      emd = match_cost / n_points (PointFlow's `emd_approx`),
      normal_consistency = (mean |n_pred . n_gt[nearest]| + mean |n_gt . n_pred[nearest]|) / 2,
    and dicts precision, recall, fscore keyed by each threshold tau: precision = share of pred samples within tau
    of the gt samples (distance < tau), recall the converse, fscore = 2 P R / (P + R) (0 when P + R = 0).

    With surface=True each mesh's samples are measured against the other mesh's surface (mesh_distance's closest
    points) instead of against its samples: dist1 / dist2 above become squared point-to-mesh distances, so the
    sampling noise of the other mesh drops out (a mesh against itself scores 0 up to rounding), and
    normal_consistency takes the normal of the closest face.  The samples are drawn with the same calls in the same
    order in both modes, so with the same generator both measure the same points; emd is the same in both.

    With iou_points > 0 the dict also has iou = |inside_pred and inside_gt| / |inside_pred or inside_gt| (0.0 when
    no point is inside either mesh) over iou_points points uniform in the union of the two meshes' axis-aligned
    boxes, drawn with the same generator after the surface samples, so every other entry is the same as with
    iou_points = 0.  A point is inside a mesh when |winding_number| >= 0.5 (beta = 2): right for closed meshes of
    either consistent orientation, graceful on open ones.  Its standard error is about sqrt(iou (1 - iou) / n_in),
    n_in the points inside either mesh."""
    if isinstance(iou_points, bool) or not isinstance(iou_points, int) or iou_points < 0:
        raise ValueError("mesh_metrics: iou_points must be an int >= 0")
    pv, pf = _mesh(pred, "pred")
    gv, gf = _mesh(gt, "gt")
    p, _, pn = sample_surface(pv, pf, n_points, generator)
    g, _, gn = sample_surface(gv.to(pv.device), gf, n_points, generator)
    x1, x2 = p.float()[None].contiguous(), g.float()[None].contiguous()
    if surface:
        pv32, gv32 = pv.detach().to(p.device, torch.float32), gv.detach().to(p.device, torch.float32)
        with torch.no_grad():
            d1, f1, _ = point_mesh_distance(x1[0], gv32, gf.to(p.device))
            d2, f2, _ = point_mesh_distance(x2[0], pv32, pf.to(p.device))
        d1, d2 = d1.double(), d2.double()
        n1, n2 = _face_normals(gv.to(p.device), gf)[f1].to(pn.dtype), _face_normals(pv, pf)[f2].to(gn.dtype)
    else:
        d1, i1, d2, i2 = nn_distance_with_indices(x1, x2)
        d1, d2, i1, i2 = d1[0].double(), d2[0].double(), i1[0], i2[0]
        n1, n2 = gn[i1], pn[i2]
    s1, s2 = d1.sqrt(), d2.sqrt()
    with torch.no_grad():
        emd = float(match_cost(x1, x2)[0]) / n_points
    nc = 0.5 * (float((pn * n1).sum(1).abs().mean()) + float((gn * n2).sum(1).abs().mean()))
    out = {"chamfer_l2": float(d1.mean() + d2.mean()), "chamfer_l1": 0.5 * float(s1.mean() + s2.mean()),
           "emd": emd, "normal_consistency": nc, "precision": {}, "recall": {}, "fscore": {}}
    for tau in thresholds:
        P, R = float((s1 < tau).double().mean()), float((s2 < tau).double().mean())
        out["precision"][tau], out["recall"][tau] = P, R
        out["fscore"][tau] = 2 * P * R / (P + R) if P + R > 0 else 0.0
    if iou_points > 0:
        out["iou"] = _iou(pv, pf, gv, gf, iou_points, generator)
    return out


def _iou(pv, pf, gv, gf, n, generator):
    dev = pv.device
    pv32, gv32 = pv.detach().to(dev, torch.float32), gv.detach().to(dev, torch.float32)
    lo = torch.minimum(pv32.min(0).values, gv32.min(0).values).double()
    hi = torch.maximum(pv32.max(0).values, gv32.max(0).values).double()
    rdev = generator.device if generator is not None else dev
    r = torch.rand(n, 3, dtype=torch.float64, generator=generator, device=rdev).to(dev)
    x = (lo + (hi - lo) * r).float().contiguous()
    a = winding_number(x, pv32, pf.to(dev)).abs() >= 0.5
    b = winding_number(x, gv32, gf.to(dev)).abs() >= 0.5
    union = int((a | b).sum())
    return int((a & b).sum()) / union if union > 0 else 0.0
