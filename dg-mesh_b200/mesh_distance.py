"""Point-to-mesh distance: the closest point of a triangle mesh to every query point, differentiable in the points and
the vertices (csrc/mesh_distance.cu behind the C-ABI dgpm_forward / dgpm_backward); the generalized winding number
and the signed distance it gives (csrc/winding.cu behind dgpm_winding).

A BVH over the faces is built on the device on every call; nothing is kept between calls."""
import ctypes
import os
import sys

import torch

_root = os.path.dirname(os.path.abspath(__file__))
if _root not in sys.path:
    sys.path.insert(0, _root)
import _dgm_lib  # noqa: E402


def _check(points, verts, faces, fn="point_mesh_distance"):
    for name, t in (("points", points), ("verts", verts), ("faces", faces)):
        if not torch.is_tensor(t):
            raise ValueError(f"{fn}: {name} must be a tensor")
        if t.dim() != 2 or t.shape[1] != 3:
            raise ValueError(f"{fn}: {name} must have shape [N, 3], not {tuple(t.shape)}")
        if not t.is_cuda:
            raise ValueError(f"{fn}: {name} must be a CUDA tensor (there is no CPU path)")
    for name, t in (("points", points), ("verts", verts)):
        if t.dtype != torch.float32:
            raise ValueError(f"{fn}: {name} must be float32, not {t.dtype}")
    if faces.dtype not in (torch.int32, torch.int64):
        raise ValueError(f"{fn}: faces must be int32 or int64, not {faces.dtype}")
    if not (points.device == verts.device == faces.device):
        raise ValueError(f"{fn}: points, verts and faces are on {points.device}, {verts.device} and {faces.device}")
    V, F = verts.shape[0], faces.shape[0]
    if V < 1 or F < 1:
        raise ValueError(f"{fn}: the mesh needs at least one vertex and one face (V = {V}, F = {F})")
    if max(3 * V, 3 * F, 3 * points.shape[0]) >= 2 ** 31:
        raise ValueError(f"{fn}: 3 V, 3 F and 3 Q must be below 2^31")
    lo, hi = torch.stack(torch.aminmax(faces)).tolist()
    if lo < 0 or hi >= V:
        raise ValueError(f"{fn}: face indices must lie in [0, {V}), found [{lo}, {hi}]")
    return points.detach().contiguous(), verts.detach().contiguous(), faces.detach().to(torch.int32).contiguous()


def _workspace(name, V, F, Q, device):
    n = ctypes.c_size_t()
    _dgm_lib.check(getattr(_dgm_lib.lib(), name)(V, F, Q, ctypes.byref(n)), name)
    return torch.empty(n.value, dtype=torch.uint8, device=device)


class PointMeshDistance(torch.autograd.Function):
    @staticmethod
    def forward(ctx, points, verts, faces):
        p, v, f = _check(points, verts, faces)
        Q, V, F = p.shape[0], v.shape[0], f.shape[0]
        dist2 = torch.empty(Q, dtype=torch.float32, device=p.device)
        face = torch.empty(Q, dtype=torch.int64, device=p.device)
        bary = torch.empty(Q, 3, dtype=torch.float32, device=p.device)
        if Q > 0:
            ws = _workspace("dgpm_forward_workspace", V, F, Q, p.device)
            _dgm_lib.check(_dgm_lib.lib().dgpm_forward(V, F, Q, v.data_ptr(), f.data_ptr(), p.data_ptr(),
                                                       dist2.data_ptr(), face.data_ptr(), bary.data_ptr(),
                                                       ws.data_ptr(), ws.numel(), _dgm_lib.stream_ptr()),
                           "dgpm_forward")
        ctx.mark_non_differentiable(face, bary)
        ctx.save_for_backward(p, v, f, face, bary)
        return dist2, face, bary

    @staticmethod
    def backward(ctx, grad_dist2, _grad_face, _grad_bary):
        p, v, f, face, bary = ctx.saved_tensors
        Q, V, F = p.shape[0], v.shape[0], f.shape[0]
        grad_points = torch.empty_like(p)
        grad_verts = torch.empty_like(v)
        if Q == 0 or grad_dist2 is None:
            return grad_points.zero_(), grad_verts.zero_(), None
        _distance_backward(p, v, f, face, bary, grad_dist2.float().contiguous(), grad_points, grad_verts)
        return grad_points, grad_verts, None


def _distance_backward(p, v, f, face, bary, g, grad_points, grad_verts):
    """dgpm_backward: the gradients of sum g dist2 at fixed (face, bary), written into grad_points and grad_verts."""
    Q, V, F = p.shape[0], v.shape[0], f.shape[0]
    ws = _workspace("dgpm_backward_workspace", V, F, Q, p.device)
    _dgm_lib.check(_dgm_lib.lib().dgpm_backward(V, F, Q, v.data_ptr(), f.data_ptr(), p.data_ptr(), face.data_ptr(),
                                                bary.data_ptr(), g.data_ptr(), grad_points.data_ptr(),
                                                grad_verts.data_ptr(), ws.data_ptr(), ws.numel(),
                                                _dgm_lib.stream_ptr()), "dgpm_backward")


def point_mesh_distance(points, verts, faces):
    """(dist2 [Q], face [Q] int64, bary [Q,3]): the closest point of the mesh (verts [V,3], faces [F,3]) to each of
    points [Q,3].

    dist2 is the squared distance to the closest point, face the triangle it lies on (exact ties go to the lowest
    face index; a point equal to a vertex gets dist2 = 0 and the lowest-index face around that vertex), and bary its
    weights w >= 0 (summing to 1 up to rounding) on that triangle's vertices.  The closest points are

        c = (bary[:, :, None] * verts[faces[face]]).sum(1)

    which, written so in torch, is differentiable in verts at fixed weights.  dist2 is differentiable in points and
    verts: d dist2 / d points = 2 (p - c), and -2 w_k (p - c) into the triangle's k-th vertex (exact wherever the
    closest point is unique).  face and bary are not differentiable.  Triangles with collinear or coincident vertices
    count as their longest edge or their point.

    points and verts are float32, faces int32 or int64, all CUDA tensors on one device; F >= 1.  Face indices outside
    [0, V) are refused: they are checked on the device with one min / max and one read of the result on the host,
    so a call synchronises once.  Anything else raises ValueError."""
    return PointMeshDistance.apply(points, verts, faces)


def _winding(points, verts, faces, beta, fn, closest):
    """dgpm_winding on checked inputs: ((p, v, f), winding [Q], (dist2, face, bary) or three Nones)."""
    if isinstance(beta, bool) or not isinstance(beta, (int, float)) or not ctypes.c_float(beta).value > 0:
        raise ValueError(f"{fn}: beta must be a number > 0 in float32 (math.inf for the exact sum), not {beta!r}")
    p, v, f = _check(points, verts, faces, fn)
    Q, V, F = p.shape[0], v.shape[0], f.shape[0]
    w = torch.empty(Q, dtype=torch.float32, device=p.device)
    out = (torch.empty(Q, dtype=torch.float32, device=p.device), torch.empty(Q, dtype=torch.int64, device=p.device),
           torch.empty(Q, 3, dtype=torch.float32, device=p.device)) if closest else (None, None, None)
    if Q > 0:
        ws = _workspace("dgpm_winding_workspace", V, F, Q, p.device)
        ptr = [None if t is None else t.data_ptr() for t in out]
        _dgm_lib.check(_dgm_lib.lib().dgpm_winding(V, F, Q, v.data_ptr(), f.data_ptr(), p.data_ptr(), float(beta),
                                                   w.data_ptr(), *ptr, ws.data_ptr(), ws.numel(),
                                                   _dgm_lib.stream_ptr()), "dgpm_winding")
    return (p, v, f), w, out


def winding_number(points, verts, faces, beta=2.0):
    """winding [Q] float32: the generalized winding number (Jacobson et al. 2013) of the mesh (verts [V,3],
    faces [F,3]) at each of points [Q,3],

        w(q) = 1 / (4 pi) sum over faces of the solid angle the face subtends at q,

    each solid angle 2 atan2(det[a b c], |a||b||c| + (a.b)|c| + (b.c)|a| + (c.a)|b|) with a, b, c the face's vertices
    minus q, in the order the face lists them.  w = +1 inside a closed mesh whose faces are counter-clockwise seen
    from outside (the right-hand normal of sample_surface points out), -1 inside one oriented the other way, 0
    outside; on open, non-manifold or self-intersecting meshes (TSDF holes, triangle soups) it degrades smoothly
    instead of flipping as ray parity or the closest face's normal do, so |w| >= 0.5 is a robust inside test.  A face
    for which det is exactly 0 adds 0: a query on a face, edge or vertex, and faces with coincident or collinear
    vertices.

    beta trades accuracy for time (Barill et al. 2018): a cluster of faces whose area-weighted centroid is farther
    than beta times its radius from q adds its order-1 far-field expansion instead of its faces.  At beta = 2 the
    error is largest for queries near the surface (measured up to 2.7e-2 on closed meshes, far below the 0.5 of
    the inside test) and falls as (radius / distance)^2; beta = math.inf never takes the far field and gives the
    exact sum of fp32 solid angles (accumulated in float64, within 1e-4 away from the surface), at the cost of F
    solid angles per query.  The result is
    bit-identical from run to run and does not depend on which other points share the call.

    Not differentiable.  Accuracy is fp32's: within about 1e-4 of the mesh's extent from the surface the sign of a
    nearby face's solid angle is not reliable.  The inputs are checked as in point_mesh_distance (one host read);
    beta must be > 0 (NaN is refused).  Anything else raises ValueError."""
    with torch.no_grad():
        return _winding(points, verts, faces, beta, "winding_number", False)[1]


class SignedDistance(torch.autograd.Function):
    @staticmethod
    def forward(ctx, points, verts, faces, beta):
        (p, v, f), w, (dist2, face, bary) = _winding(points, verts, faces, beta, "signed_distance", True)
        dist = dist2.sqrt()
        sign = torch.where(w.abs() >= 0.5, -1.0, 1.0)
        sdf = sign * dist
        ctx.mark_non_differentiable(face, bary, w)
        ctx.save_for_backward(p, v, f, face, bary, dist, sign)
        return sdf, face, bary, w

    @staticmethod
    def backward(ctx, grad_sdf, _grad_face, _grad_bary, _grad_w):
        p, v, f, face, bary, dist, sign = ctx.saved_tensors
        grad_points = torch.zeros_like(p)
        grad_verts = torch.zeros_like(v)
        if p.shape[0] == 0 or grad_sdf is None:
            return grad_points, grad_verts, None, None
        # d sdf = s d dist2 / (2 sqrt dist2) at fixed sign; 0 where dist2 = 0
        g = torch.where(dist > 0, sign * grad_sdf.float() / (2 * dist), 0.0).contiguous()
        _distance_backward(p, v, f, face, bary, g, grad_points, grad_verts)
        return grad_points, grad_verts, None, None


def signed_distance(points, verts, faces, beta=2.0):
    """(sdf [Q], face [Q] int64, bary [Q,3], winding [Q]): the signed distance from each of points [Q,3] to the mesh
    (verts [V,3], faces [F,3]), negative inside.

    A point is inside when |winding| >= 0.5 (winding_number with the same beta), so the sign is right for closed
    meshes of either consistent orientation and degrades gracefully on open ones.  sdf = -sqrt(dist2) inside and
    +sqrt(dist2) outside, where dist2, face and bary are point_mesh_distance's, bit for bit, from the same BVH build
    (one dgpm_winding call).  sdf is differentiable in points and verts with the sign held fixed: the gradient is
    point_mesh_distance's for dist2 with g' = sign g / (2 |sdf|), and 0 where the point lies on the surface
    (dist2 = 0), so no NaN appears.  face, bary and winding are not differentiable.  Checks and errors as in
    winding_number."""
    return SignedDistance.apply(points, verts, faces, beta)
