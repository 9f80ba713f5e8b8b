"""Drop-in `gaussian_renderer` (reference: dgmesh/gaussian_renderer/__init__.py:32-119).

`render(viewpoint_camera, pc, pipe, bg_color, d_xyz, d_rotation, d_scaling, is_6dof=False,
scaling_modifier=1.0, override_color=None)` keeps its signature and its four-key result dict
("render", "viewspace_points", "visibility_filter", "radii"); the rasterizer underneath is the
sm_90a one (diff_gaussian_rasterization in this package).  `render_batch` is the multi-frame
variant used for data-parallel training over frames (one call, one gradient accumulation).
`render_depth_alpha` (and `render_batch(..., depth_alpha=True)`) add the differentiable "depth" map
(sum_i d_i alpha_i T_i, unnormalised view-space depth) and "alpha" map (accumulated opacity 1 - T_final).
`render_camera_grad` (and `render_batch(..., camera_grad=True)`) also pass gradients to the camera's
world_view_transform, full_proj_transform and camera_center; `posed_camera` makes those three differentiable
functions of an se(3) pose correction.
`render_normal` (and `render_batch(..., normals=True)`) add the differentiable "normal" map
(sum_i n_i alpha_i T_i of the Gaussians' unit normals, in camera or world space) to the depth / alpha maps.
`render_features` (and `render_batch(..., features=...)`) add the differentiable "features" map of caller-chosen
per-Gaussian vectors; `render_flow` (and `render_batch(..., flow_to=...)`) the optical-flow map "flow" between two
times and cameras.
`render_abs_grad` (and `abs_grad=True` on `render_depth_alpha`, `render_camera_grad`, `render_normal`,
`render_surface` and `render_batch`) also return "viewspace_points_abs", whose .grad receives the absolute
screen-space gradient (AbsGS) next to "viewspace_points"'s dL/dmean2D."""
import math

import torch

from diff_gaussian_rasterization import (BatchGaussianRasterizer, GaussianRasterizationSettings,
                                         GaussianRasterizer)


def quaternion_multiply(q1, q2):
    w1, x1, y1, z1 = q1[..., 0], q1[..., 1], q1[..., 2], q1[..., 3]
    w2, x2, y2, z2 = q2[..., 0], q2[..., 1], q2[..., 2], q2[..., 3]
    return torch.stack((w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                        w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2), dim=-1)


def _settings(cam, pc, pipe, bg_color, scaling_modifier):
    return GaussianRasterizationSettings(
        image_height=int(cam.image_height), image_width=int(cam.image_width),
        tanfovx=math.tan(cam.FoVx * 0.5), tanfovy=math.tan(cam.FoVy * 0.5), bg=bg_color,
        scale_modifier=scaling_modifier, viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform,
        sh_degree=pc.active_sh_degree, campos=cam.camera_center, prefiltered=False, debug=pipe.debug)


def _gaussian_inputs(cam, pc, pipe, d_xyz, d_rotation, d_scaling, is_6dof, scaling_modifier, override_color):
    """The tensors the rasterizer consumes, assembled exactly as the reference does (:66-104)."""
    if is_6dof:
        if torch.is_tensor(d_xyz) is False:
            means3D = pc.get_xyz
        else:
            from utils.rigid_utils import from_homogenous, to_homogenous
            means3D = from_homogenous(torch.bmm(d_xyz, to_homogenous(pc.get_xyz).unsqueeze(-1)).squeeze(-1))
    else:
        means3D = pc.get_xyz + d_xyz
    kw = dict(means3D=means3D, opacities=pc.get_opacity)
    if pipe.compute_cov3D_python:
        kw["cov3D_precomp"] = pc.get_covariance(scaling_modifier)
    else:
        kw["scales"] = pc.get_scaling + d_scaling
        kw["rotations"] = pc.get_rotation + d_rotation
    if override_color is None:
        if pipe.convert_SHs_python:
            from utils.sh_utils import eval_sh
            shs_view = pc.get_features.transpose(1, 2).view(-1, 3, (pc.max_sh_degree + 1) ** 2)
            dir_pp = (pc.get_xyz - cam.camera_center.repeat(pc.get_features.shape[0], 1))
            dir_pp_normalized = dir_pp / dir_pp.norm(dim=1, keepdim=True)
            sh2rgb = eval_sh(pc.active_sh_degree, shs_view, dir_pp_normalized)
            kw["colors_precomp"] = torch.clamp_min(sh2rgb + 0.5, 0.0)
        else:
            kw["shs"] = pc.get_features
    else:
        kw["colors_precomp"] = override_color
    return kw


def render(viewpoint_camera, pc, pipe, bg_color, d_xyz, d_rotation, d_scaling, is_6dof=False, scaling_modifier=1.0,
           override_color=None):
    """Render the scene.  Background tensor (bg_color) must be on GPU!"""
    return _render(viewpoint_camera, pc, pipe, bg_color, d_xyz, d_rotation, d_scaling, is_6dof, scaling_modifier,
                   override_color, False)


def render_depth_alpha(viewpoint_camera, pc, pipe, bg_color, d_xyz, d_rotation, d_scaling, is_6dof=False,
                       scaling_modifier=1.0, override_color=None, abs_grad=False):
    """`render` + "depth" [1,H,W] (sum_i d_i alpha_i T_i; divide by alpha for the expected depth) and
    "alpha" [1,H,W] (1 - T_final), both differentiable, e.g. for a foreground-mask loss on the Gaussians.
    abs_grad=True: see `render_abs_grad`."""
    return _render(viewpoint_camera, pc, pipe, bg_color, d_xyz, d_rotation, d_scaling, is_6dof, scaling_modifier,
                   override_color, True, abs_grad=abs_grad)


def render_camera_grad(viewpoint_camera, pc, pipe, bg_color, d_xyz, d_rotation, d_scaling, is_6dof=False,
                       scaling_modifier=1.0, override_color=None, depth_alpha=False, abs_grad=False):
    """`render` (depth_alpha: `render_depth_alpha`) whose result is also differentiable with respect to the
    camera's world_view_transform, full_proj_transform and camera_center, e.g. those of `posed_camera`.  The field
    of view is not differentiated.  abs_grad=True: see `render_abs_grad`."""
    return _render(viewpoint_camera, pc, pipe, bg_color, d_xyz, d_rotation, d_scaling, is_6dof, scaling_modifier,
                   override_color, depth_alpha, camera_grad=True, abs_grad=abs_grad)


def render_abs_grad(viewpoint_camera, pc, pipe, bg_color, d_xyz, d_rotation, d_scaling, is_6dof=False,
                    scaling_modifier=1.0, override_color=None, depth_alpha=False, camera_grad=False):
    """`render` (depth_alpha: `render_depth_alpha`; camera_grad: `render_camera_grad`) + "viewspace_points_abs"
    [N,3], a zero tensor like "viewspace_points" whose .grad receives, per Gaussian, the absolute screen-space
    gradient (AbsGS): (sum_p |g_p.x|, sum_p |g_p.y|, 0) with g_p the part of dL/dmean2D that pixel p contributes.
    Pixels that pull a Gaussian in opposite directions cancel in "viewspace_points".grad but not here, so a large
    Gaussian over fine detail still reaches the densification threshold.  Use it where the reference uses
    "viewspace_points": gaussians.add_densification_stats(pkg["viewspace_points_abs"], pkg["visibility_filter"])
    (it reads only .grad[:, :2] of the tensor it is given).  The threshold that suits the statistic is the training
    recipe's choice; densify_and_prune is unchanged."""
    return _render(viewpoint_camera, pc, pipe, bg_color, d_xyz, d_rotation, d_scaling, is_6dof, scaling_modifier,
                   override_color, depth_alpha, camera_grad=camera_grad, abs_grad=True)


def render_normal(viewpoint_camera, pc, pipe, bg_color, d_xyz, d_rotation, d_scaling, d_normal=0.0, is_6dof=False,
                  scaling_modifier=1.0, override_color=None, space="camera", camera_grad=False, abs_grad=False):
    """`render_depth_alpha` + "normal" [3,H,W]: sum_i n_i alpha_i T_i over the same blend, n_i = normalize(
    pc.get_normal + d_normal), the oriented normals DG-Mesh builds its surface from.  space="camera" rotates them
    into the camera frame (n @ world_view_transform[:3,:3], so that a `posed_camera` also gets the rotation's
    gradient), space="world" leaves them as they are.  The map has no background term and is not normalised:
    normal / alpha is the alpha-weighted mean normal.  camera_grad=True: see `render_camera_grad`.  Every map is
    differentiable; the normal map's gradient reaches pc.get_normal and d_normal directly, and every other input
    through the blend.  abs_grad=True: see `render_abs_grad`."""
    if is_6dof:
        raise NotImplementedError("render_normal: normals under the per-Gaussian SE(3) deformation (is_6dof)")
    n = _normals(viewpoint_camera, pc, d_normal, space)
    return _render(viewpoint_camera, pc, pipe, bg_color, d_xyz, d_rotation, d_scaling, is_6dof, scaling_modifier,
                   override_color, True, camera_grad=camera_grad, normals=n, abs_grad=abs_grad)


def render_surface(viewpoint_camera, pc, pipe, bg_color, d_xyz, d_rotation, d_scaling, near=0.2, far=100.0,
                   normals=False, d_normal=0.0, space="camera", is_6dof=False, scaling_modifier=1.0,
                   override_color=None, camera_grad=False, abs_grad=False):
    """`render_depth_alpha` + "median_depth" [1,H,W] (the view depth where the transmittance crosses 0.5; 0 where
    nothing is blended) and "distortion" [1,H,W] (2DGS's 1/2 sum_ij w_i w_j (m_i - m_j)^2 over the blend weights
    w_i = alpha_i T_i, m_i the depth normalised between `near` and `far`), for depth-normal consistency and
    distortion losses.  normals=True also adds "normal" (see `render_normal`, with `d_normal` and `space`).
    camera_grad=True: see `render_camera_grad`.  Every map is differentiable.  abs_grad=True: see
    `render_abs_grad`."""
    if is_6dof:
        raise NotImplementedError("render_surface: surface maps under the per-Gaussian SE(3) deformation (is_6dof)")
    n = _normals(viewpoint_camera, pc, d_normal, space) if normals else None
    return _render(viewpoint_camera, pc, pipe, bg_color, d_xyz, d_rotation, d_scaling, is_6dof, scaling_modifier,
                   override_color, True, camera_grad=camera_grad, normals=n, surface=(near, far), abs_grad=abs_grad)


def render_features(viewpoint_camera, pc, pipe, bg_color, d_xyz, d_rotation, d_scaling, features, is_6dof=False,
                    scaling_modifier=1.0, override_color=None, camera_grad=False, abs_grad=False):
    """`render_depth_alpha` + "features" [C,H,W]: sum_i f_i alpha_i T_i over the same blend of the caller's per-Gaussian
    vectors `features` [N,C], 1 <= C <= 64 (e.g. pc.get_xyz for canonical-coordinate maps).  No background term and
    no normalisation: features / alpha is the alpha-weighted mean.  Works under is_6dof (the features are the
    caller's).  camera_grad=True: see `render_camera_grad`.  Every map is differentiable; the feature map's gradient
    reaches `features` directly and every other input through the blend.  abs_grad=True raises ValueError: the
    feature pass has no per-pixel total of dL/dmean2D to take |.| of."""
    return _render(viewpoint_camera, pc, pipe, bg_color, d_xyz, d_rotation, d_scaling, is_6dof, scaling_modifier,
                   override_color, True, camera_grad=camera_grad, features=features, abs_grad=abs_grad)


FLOW_NEAR = 0.2   # the rasterizer's near cut-off (view depth): a Gaussian nearer than this in either camera has no flow


def _project(cam, x):
    """The rasterizer's projection of points x [..., N, 3] into `cam` (full_proj_transform, perspective divide, then
    ((ndc + 1) S - 1) / 2), in pixels [..., N, 2], and their view depth [..., N]; torch ops, differentiable in x and in
    the camera's matrices."""
    xh = torch.cat([x, torch.ones_like(x[..., :1])], -1)
    ph = xh @ cam.full_proj_transform
    z = (xh @ cam.world_view_transform)[..., 2]
    ndc = ph[..., :2] / (ph[..., 3:] + 1e-7)
    S = torch.tensor([cam.image_width, cam.image_height], dtype=x.dtype, device=x.device)
    return ((ndc + 1) * S - 1) * 0.5, z


def flow_features(cam, cam_to, x, x_to):
    """Per-Gaussian image displacement pi_to(x_to) - pi(x) [..., N, 2] in pixels (pi: `_project` into `cam`, pi_to into
    `cam_to`); exactly 0, with no gradient, for a Gaussian whose view depth is <= FLOW_NEAR in either camera."""
    p, z = _project(cam, x)
    p_to, z_to = _project(cam_to, x_to)
    ok = ((z > FLOW_NEAR) & (z_to > FLOW_NEAR))[..., None]
    return torch.where(ok, p_to - p, torch.zeros_like(p))


def render_flow(viewpoint_camera, cam_to, pc, pipe, bg_color, d_xyz, d_rotation, d_scaling, d_xyz_to,
                scaling_modifier=1.0, override_color=None, camera_grad=False, abs_grad=False):
    """`render_depth_alpha` + "flow" [2,H,W]: the optical flow from `viewpoint_camera` at the time of the deformation
    (d_xyz, d_rotation, d_scaling) to `cam_to` at the time of d_xyz_to, over viewpoint_camera's blend:
        flow = sum_i (pi_to(x_i + d_xyz_to,i) - pi(x_i + d_xyz_i)) alpha_i T_i   (pixels; flow / alpha is the mean)
    with pi the rasterizer's own projection (see `_project`), computed with torch ops so that the gradient reaches
    both deformations and both cameras (e.g. `posed_camera`s).  A Gaussian whose view depth in either camera is <= 0.2
    (FLOW_NEAR, the rasterizer's near cut-off) contributes zero flow and receives no flow gradient.  Supervise
    flow / alpha (or flow against alpha times an estimate) with an off-line optical-flow estimate.  abs_grad=True
    raises ValueError, as for `render_features`."""
    x = pc.get_xyz
    f = flow_features(viewpoint_camera, cam_to, x + d_xyz, x + d_xyz_to)
    out = _render(viewpoint_camera, pc, pipe, bg_color, d_xyz, d_rotation, d_scaling, False, scaling_modifier,
                  override_color, True, camera_grad=camera_grad, features=f, abs_grad=abs_grad)
    out["flow"] = out.pop("features")
    return out


def _normals(cam, pc, d_normal, space):
    """normalize(pc.get_normal + d_normal) ([N,3], or [F,N,3] for a per-frame d_normal), in camera or world space;
    cam: one camera, or a list of F cameras for [F,N,3] camera-space normals."""
    if space not in ("camera", "world"):
        raise ValueError('space must be "camera" or "world"')
    n = torch.nn.functional.normalize(pc.get_normal + d_normal, dim=-1)
    if space == "world":
        return n
    if isinstance(cam, (list, tuple)):   # row vectors: n_cam = n_world R^T, R^T = world_view_transform[:3,:3]
        rot = torch.stack([c.world_view_transform[:3, :3] for c in cam])
        return n @ rot if n.ndim == 3 else torch.einsum("nj,fjk->fnk", n, rot)
    return n @ cam.world_view_transform[:3, :3]


class _PosedCamera:
    """`camera` with its pose corrected by exp(delta) in the camera frame (see posed_camera)."""

    def __init__(self, camera, delta):
        self._camera = camera
        E = _se3_exp(delta.to(camera.world_view_transform.dtype))
        # world_view_transform is the world-to-camera matrix transposed: (E C)^T = C^T E^T
        self.world_view_transform = camera.world_view_transform @ E.transpose(0, 1)
        self.full_proj_transform = self.world_view_transform @ camera.projection_matrix
        self.camera_center = torch.linalg.inv(self.world_view_transform)[3, :3]

    def __getattr__(self, name):
        return getattr(self._camera, name)


def posed_camera(camera, delta):
    """A camera-like object whose world_view_transform, full_proj_transform (= world_view_transform @
    camera.projection_matrix) and camera_center (= inverse(world_view_transform)[3, :3]) are differentiable
    functions of the se(3) correction delta [6] = (w, v): the world-to-camera transform becomes exp(delta) times
    the camera's, with rotation vector w and translation part v expressed in the camera frame.  Every other
    attribute is the camera's.  delta = 0 gives the camera's own pose."""
    return _PosedCamera(camera, delta)


def _se3_exp(delta):
    """[6] (w, v) -> [4,4] exp of the twist, [[R, V v], [0, 1]] with R = I + A W + B W^2, V = I + B W + C W^2,
    W = skew(w), |w| = theta, A = sin(theta)/theta, B = (1 - cos(theta))/theta^2, C = (theta - sin(theta))/theta^3
    (their series for small theta, where the closed forms cancel)."""
    from utils.rigid_utils import rp_to_se3, skew
    w, v = delta[:3], delta[3:]
    th2 = (w * w).sum()
    small = th2 < 1e-2
    th = torch.sqrt(torch.where(small, torch.ones_like(th2), th2))   # the closed forms see no theta near 0
    A = torch.where(small, 1 - th2 / 6 * (1 - th2 / 20 * (1 - th2 / 42)), torch.sin(th) / th)
    B = torch.where(small, 0.5 * (1 - th2 / 12 * (1 - th2 / 30 * (1 - th2 / 56))), (1 - torch.cos(th)) / (th * th))
    C = torch.where(small, (1 - th2 / 20 * (1 - th2 / 42 * (1 - th2 / 72))) / 6, (th - torch.sin(th)) / (th * th * th))
    Wm = skew(w[None])[0]
    W2 = Wm @ Wm
    eye = torch.eye(3, dtype=delta.dtype, device=delta.device)
    R = eye + A * Wm + B * W2
    V = eye + B * Wm + C * W2
    return rp_to_se3(R[None], (V @ v)[None, :, None])[0]


def _viewspace_points(shape, dtype):
    """Zero tensor whose gradient receives a screen-space statistic of the 2D means (densification)."""
    t = torch.zeros(shape, dtype=dtype, requires_grad=True, device="cuda") + 0
    try:
        t.retain_grad()
    except Exception:
        pass
    return t


def _render(viewpoint_camera, pc, pipe, bg_color, d_xyz, d_rotation, d_scaling, is_6dof, scaling_modifier,
            override_color, depth_alpha, camera_grad=False, normals=None, surface=None, features=None, abs_grad=False):
    # zero tensor whose gradient receives the 2D (screen-space) mean gradients (densification statistics)
    screenspace_points = torch.zeros_like(pc.get_xyz, dtype=pc.get_xyz.dtype, requires_grad=True,
                                          device="cuda") + 0
    try:
        screenspace_points.retain_grad()
    except Exception:
        pass
    rasterizer = GaussianRasterizer(raster_settings=_settings(viewpoint_camera, pc, pipe, bg_color, scaling_modifier))
    kw = _gaussian_inputs(viewpoint_camera, pc, pipe, d_xyz, d_rotation, d_scaling, is_6dof, scaling_modifier,
                          override_color)
    points_abs = _viewspace_points(pc.get_xyz.shape, pc.get_xyz.dtype) if abs_grad else None
    maps = rasterizer._maps(means2D=screenspace_points, depth_alpha=depth_alpha, camera_grad=camera_grad,
                            normals=normals, surface=surface, features=features, means2D_abs=points_abs, **kw)
    return _result(maps, screenspace_points, points_abs)


def _result(maps, screenspace_points, points_abs):
    """The result dict of `render` / `render_batch` from the rasterizer's maps by name."""
    res = {"render": maps.pop("color"), "viewspace_points": screenspace_points, "visibility_filter": maps["radii"] > 0}
    res.update(maps)
    if points_abs is not None:
        res["viewspace_points_abs"] = points_abs
    return res


def render_batch(cameras, pc, pipe, bg_color, d_xyz, d_rotation, d_scaling, scaling_modifier=1.0, depth_alpha=False,
                 camera_grad=False, normals=False, d_normal=0.0, normal_space="camera", surface=False, near=0.2,
                 far=100.0, features=None, flow_to=None, abs_grad=False):
    """F training frames in one call -> images [F,3,H,W]; the keys of `render` with a leading frame dimension.

    DG-Mesh deforms the Gaussians by each frame's own time (dgmesh/train.py:157-178): pass `d_xyz`,
    `d_rotation`, `d_scaling` as [F,N,.] tensors (or lists of F per-frame tensors, e.g. the deformation
    network's outputs for t_k = fid_k) and every frame renders xyz + d_xyz[k], rotation + d_rotation[k],
    scaling + d_scaling[k] -- bit-identical to F calls of `render`, with the binning chains of later frames
    overlapped with the blend kernels of earlier ones.  [N,.] deltas (or 0.0, the warm-up phase) apply to
    every frame.  Opacity and SH are shared; their gradients are summed over the frames inside the kernels.
    depth_alpha=True adds "depth" and "alpha" [F,1,H,W] (see `render_depth_alpha`); camera_grad=True passes
    gradients to every camera's world_view_transform, full_proj_transform and camera_center (see
    `render_camera_grad`).  normals=True adds "normal" [F,3,H,W] (and "depth", "alpha"; see `render_normal`), with
    `d_normal` given like the other deltas and the normals in `normal_space` ("camera": each frame's own).
    surface=True adds "median_depth" and "distortion" [F,1,H,W] (and "depth", "alpha"; see `render_surface`, with
    `near` and `far`).  features ([N,C] shared or [F,N,C] per frame, 1 <= C <= 64) adds "features" [F,C,H,W] (see
    `render_features`); flow_to = (cameras_to, d_xyz_to) adds "flow" [F,2,H,W], frame k's flow from cameras[k] at its
    own deformation to cameras_to[k] at d_xyz_to[k] (see `render_flow`; d_xyz_to given like d_xyz).  Both compose
    with each other (one pass over C + 2 channels) and with the other maps; they add "depth" and "alpha".
    abs_grad=True adds "viewspace_points_abs" [F,N,3] (see `render_abs_grad`), each frame's statistic in its slab;
    not with features or flow_to (ValueError)."""
    F, N = len(cameras), pc.get_xyz.shape[0]
    screenspace_points = torch.zeros((F, N, 3), dtype=pc.get_xyz.dtype, requires_grad=True, device="cuda") + 0
    try:
        screenspace_points.retain_grad()
    except Exception:
        pass
    sets = [_settings(c, pc, pipe, bg_color, scaling_modifier) for c in cameras]

    def per_frame(d):
        if isinstance(d, (list, tuple)):
            if len(d) != F:
                raise ValueError("per-frame deltas: one entry per camera")
            return torch.stack([x if torch.is_tensor(x) else torch.zeros_like(pc.get_xyz[:, :1]) + x for x in d])
        return d

    d_xyz, d_rotation, d_scaling = per_frame(d_xyz), per_frame(d_rotation), per_frame(d_scaling)
    if isinstance(d_normal, (list, tuple)):   # scalar entries as [N,3], to stack with the tensor ones
        d_normal = [x if torch.is_tensor(x) else torch.zeros_like(pc.get_xyz) + x for x in d_normal]
    nrm = _normals(list(cameras), pc, per_frame(d_normal), normal_space) if normals else None
    if pipe.compute_cov3D_python or pipe.convert_SHs_python:
        raise NotImplementedError("render_batch: the python covariance / SH paths are per-camera; use render()")
    kw = dict(means3D=pc.get_xyz + d_xyz, opacities=pc.get_opacity, scales=pc.get_scaling + d_scaling,
              rotations=pc.get_rotation + d_rotation, shs=pc.get_features)
    rasterizer = BatchGaussianRasterizer(sets)
    points_abs = _viewspace_points((F, N, 3), pc.get_xyz.dtype) if abs_grad else None
    feats, C = _batch_features(cameras, pc, F, d_xyz, features, flow_to, per_frame)
    maps = rasterizer._maps(means2D=screenspace_points, depth_alpha=depth_alpha, camera_grad=camera_grad, normals=nrm,
                            surface=(near, far) if surface else None, features=feats, means2D_abs=points_abs, **kw)
    if feats is not None:
        fm = maps.pop("features")
        if features is not None:
            maps["features"] = fm[:, :C]
        if flow_to is not None:
            maps["flow"] = fm[:, C:]
    return _result(maps, screenspace_points, points_abs)


def _batch_features(cameras, pc, F, d_xyz, features, flow_to, per_frame):
    """The per-Gaussian vectors of render_batch's feature pass ([N,C'] or [F,N,C']) and C, the caller's channels in
    front of the two flow channels; (None, 0) when there is neither."""
    if features is None and flow_to is None:
        return None, 0
    parts = []
    C = 0
    if features is not None:
        C = int(features.shape[-1])
        parts.append(features)
    if flow_to is not None:
        cams_to, d_xyz_to = flow_to
        if len(cams_to) != F:
            raise ValueError("flow_to: one target camera per camera")
        x = pc.get_xyz
        x0 = (x + d_xyz).expand(F, -1, -1) if not torch.is_tensor(d_xyz) or d_xyz.ndim < 3 else x + d_xyz
        d_to = per_frame(d_xyz_to)
        x1 = (x + d_to).expand(F, -1, -1) if not torch.is_tensor(d_to) or d_to.ndim < 3 else x + d_to
        parts.append(torch.stack([flow_features(cameras[k], cams_to[k], x0[k], x1[k]) for k in range(F)]))
    if len(parts) == 2 and parts[0].ndim == 2:
        parts[0] = parts[0].expand(F, -1, -1)
    return (torch.cat(parts, -1) if len(parts) == 2 else parts[0]).contiguous(), C
