"""Drop-in `gaussian_renderer` (reference: dgmesh/gaussian_renderer/__init__.py:32-119).

`render(viewpoint_camera, pc, pipe, bg_color, d_xyz, d_rotation, d_scaling, is_6dof=False,
scaling_modifier=1.0, override_color=None)` keeps its signature and its four-key result dict
("render", "viewspace_points", "visibility_filter", "radii"); the rasterizer underneath is the
sm_90a one (diff_gaussian_rasterization in this package).  `render_batch` is the multi-frame
variant used for data-parallel training over frames (one call, one gradient accumulation)."""
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
    rendered_image, radii = rasterizer(means2D=screenspace_points, **kw)
    return {"render": rendered_image, "viewspace_points": screenspace_points, "visibility_filter": radii > 0,
            "radii": radii}


def render_batch(cameras, pc, pipe, bg_color, d_xyz, d_rotation, d_scaling, scaling_modifier=1.0):
    """F training frames in one call -> images [F,3,H,W]; the keys of `render` with a leading frame dimension.

    DG-Mesh deforms the Gaussians by each frame's own time (dgmesh/train.py:157-178): pass `d_xyz`,
    `d_rotation`, `d_scaling` as [F,N,.] tensors (or lists of F per-frame tensors, e.g. the deformation
    network's outputs for t_k = fid_k) and every frame renders xyz + d_xyz[k], rotation + d_rotation[k],
    scaling + d_scaling[k] -- bit-identical to F calls of `render`, with the binning chains of later frames
    overlapped with the blend kernels of earlier ones.  [N,.] deltas (or 0.0, the warm-up phase) apply to
    every frame.  Opacity and SH are shared; their gradients are summed over the frames inside the kernels."""
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
    if pipe.compute_cov3D_python or pipe.convert_SHs_python:
        raise NotImplementedError("render_batch: the python covariance / SH paths are per-camera; use render()")
    kw = dict(means3D=pc.get_xyz + d_xyz, opacities=pc.get_opacity, scales=pc.get_scaling + d_scaling,
              rotations=pc.get_rotation + d_rotation, shs=pc.get_features)
    images, radii = BatchGaussianRasterizer(sets)(means2D=screenspace_points, **kw)
    return {"render": images, "viewspace_points": screenspace_points, "visibility_filter": radii > 0, "radii": radii}
