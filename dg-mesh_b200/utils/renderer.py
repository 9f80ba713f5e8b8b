"""Drop-in `utils.renderer` (reference: dgmesh/utils/renderer.py:33-233): Gaussians -> DPSR indicator grid ->
marching cubes -> per-vertex colour -> mesh rasterisation (mask + image), i.e. the whole mesh branch of the
training step.  Same signatures, same return values.

What changes underneath: DPSR and marching cubes are the sm_90a kernels of this package; when
`gaussians.dpsr` is this package's DPSR, the sign fix + threshold that follow the solve (reference
:163-168) are fused into it, which removes the host read of psr[0,0,0,0].  The mesh RASTERISATION
(`render_mask` / `render_mesh`, reference :33-121: nvdiffrast's rasterize / interpolate / antialias on an
OpenGL context) runs on this package's CUDA triangle rasteriser (`nvdiffrast.torch` here is
dg-mesh_b200/nvdiffrast -> meshrast.py): no GL context, and `mesh_renderer` rasterises the mesh ONCE for the
mask and the image (the reference rasterises it twice)."""
import math

import torch

import nvdiffrast.torch as dr

SMALL_NUMBER = 1e-6

# camera-convention changes of dgmesh/nvdiffrast_utils/util.py:470-475 (the reference module itself imports the
# third-party nvdiffrast and imageio packages at import time, so the constants are restated here)
_B2CV = ((1.0, 0.0, 0.0, 0.0), (0.0, -1.0, 0.0, 0.0), (0.0, 0.0, -1.0, 0.0), (0.0, 0.0, 0.0, 1.0))


def _blender2opencv(device):
    return torch.tensor(_B2CV, dtype=torch.float32, device=device)


def K_to_projection(K, H, W, n=0.001, f=10.0):
    """nvdiffrast_utils/util.py:484-490 (argument names as there: it is called with (K, height, width)).
    The four intrinsics are read on the host: a device-resident K costs ONE copy here (the reference's
    element-wise float() reads are four blocking copies); the result lives where K lived."""
    k = K.detach().cpu() if K.is_cuda else K
    fu, fv, cu, cv = float(k[0, 0]), float(k[1, 1]), float(k[0, 2]), float(k[1, 2])
    return torch.tensor([[2 * fu / W, 0, -2 * cu / W + 1, 0], [0, 2 * fv / H, 2 * cv / H - 1, 0],
                         [0, 0, -(f + n) / (f - n), -2 * f * n / (f - n)], [0, 0, -1, 0]],
                        dtype=torch.float32, device=K.device)


def transform_pos(mtx, pos):
    """(x, y, z) -> (x, y, z, 1) @ mtx^T, [1, N, 4] (nvdiffrast_utils/util.py:493-497)."""
    posw = torch.cat([pos, torch.ones([pos.shape[0], 1], device=pos.device)], axis=1)
    return torch.matmul(posw, mtx.t())[None, ...]


def _clip_matrix(pose, K, resolution):
    """projection @ pose; camera matrices that arrive on the host are multiplied there (no kernel, no blocking
    read)"""
    proj = K_to_projection(K, resolution[0], resolution[1])
    return proj.to(pose.device) @ pose


def _clip(mesh_v_pos, pose, K, resolution):
    return transform_pos(_clip_matrix(pose, K, resolution).to(mesh_v_pos.device), mesh_v_pos)


def _upload(t, device):
    """a host tensor to `device` without waiting for the stream: pinned, asynchronous"""
    return t.pin_memory().to(device, non_blocking=True) if torch.device(device).type == "cuda" else t.to(device)


def _raster(glctx, mesh_v_pos, mesh_t_pos_idx, pose, K, resolution):
    v_pos_clip = _clip(mesh_v_pos, pose, K, resolution)
    rast_out, _ = dr.rasterize(glctx, v_pos_clip, mesh_t_pos_idx, resolution=resolution)
    topo = dr.edge_opposites(mesh_t_pos_idx, mesh_v_pos.shape[0]) if mesh_t_pos_idx.shape[0] else None
    return v_pos_clip, rast_out, topo


# _mask_from and _image_from take rast [B,H,W,4] (one image, or B of range mode) and return masks [B,H,W,3] and
# images [B,3,H,W]; the single-image callers take [0]
def _mask_from(rast_out, v_pos_clip, mesh_v_pos, mesh_t_pos_idx, topo):
    vtx_color = torch.ones(mesh_v_pos.shape, dtype=torch.float, device=v_pos_clip.device)
    color, _ = dr.interpolate(vtx_color[None, ...], rast_out, mesh_t_pos_idx)
    color = dr.antialias(color, rast_out, v_pos_clip, mesh_t_pos_idx, topology_hash=topo)
    return torch.flip(color, dims=[1])


def _image_from(rast_out, v_pos_clip, mesh_t_pos_idx, vtx_color, mask, whitebackground, topo):
    output, _ = dr.interpolate(vtx_color[None, ...], rast_out, mesh_t_pos_idx)
    output = dr.antialias(output, rast_out, v_pos_clip, mesh_t_pos_idx, topology_hash=topo)
    output = torch.flip(output, dims=[1])
    output.masked_fill_(~mask.bool(), 1 if whitebackground else 0)   # output[~mask] = bg, without a sync
    return torch.clamp(output, 0.0, 1.0).permute(0, 3, 1, 2)


def render_mask(glctx, mesh_v_pos, mesh_t_pos_idx, pose, K, resolution=[800, 800]):
    """reference :33-66 -> mask [H, W, 3]"""
    v_pos_clip, rast_out, topo = _raster(glctx, mesh_v_pos, mesh_t_pos_idx, pose, K, resolution)
    return _mask_from(rast_out, v_pos_clip, mesh_v_pos, mesh_t_pos_idx, topo)[0]


def render_mesh(glctx, mesh_v_pos, mesh_t_pos_idx, vtx_color, pose, K, resolution=[800, 800], whitebackground=False):
    """reference :69-121 -> image [3, H, W]"""
    v_pos_clip, rast_out, topo = _raster(glctx, mesh_v_pos, mesh_t_pos_idx, pose, K, resolution)
    mask = _mask_from(rast_out, v_pos_clip, mesh_v_pos, mesh_t_pos_idx, topo)
    return _image_from(rast_out, v_pos_clip, mesh_t_pos_idx, vtx_color, mask, whitebackground, topo)[0]


def _dpsr_inputs(gaussians, d_xyz, d_normal, freeze_pos):
    """DPSR's points in [0, 1] and its normals: [N,3], or [F,N,3] for [F,N,3] deltas (reference :150-161)"""
    if freeze_pos:
        dpsr_points = gaussians.get_xyz.detach() + d_xyz.detach()
    else:
        dpsr_points = gaussians.get_xyz + d_xyz
    dpsr_points = (dpsr_points - gaussians.gaussian_center) / gaussians.gaussian_scale  # [-1, 1]
    dpsr_points = dpsr_points / 2.0 + 0.5                                                 # [0, 1]
    dpsr_points = torch.clamp(dpsr_points, SMALL_NUMBER, 1 - SMALL_NUMBER)
    return dpsr_points, gaussians.get_normal + d_normal


def _to_world(verts, gaussians):
    verts = verts * 2.0 - 1.0  # [-1, 1]
    return verts * gaussians.gaussian_scale + gaussians.gaussian_center


def extract_mesh(gaussians, d_xyz, d_normal, freeze_pos=False):
    """Gaussians (+ deltas) -> (verts [V,3] float32 in world space, faces [F,3] int32): reference :150-175."""
    dpsr_points, normals = _dpsr_inputs(gaussians, d_xyz, d_normal, freeze_pos)
    if hasattr(gaussians.dpsr, "forward_signed"):
        psr = gaussians.dpsr.forward_signed(dpsr_points.unsqueeze(0), normals.unsqueeze(0),
                                            gaussians.density_thres_param)
    else:  # a reference DPSR module: same arithmetic, with its host synchronisation
        psr = gaussians.dpsr(dpsr_points.unsqueeze(0), normals.unsqueeze(0))
        sign = psr[0, 0, 0, 0].detach()  # Sign for Diso is opposite to dpsr
        psr = psr * (-1 if sign < 0 else 1)
        psr = (psr - gaussians.density_thres_param).squeeze(0)
    verts, faces = gaussians.diffmc(psr, deform=None, isovalue=0.0)
    verts = _to_world(verts, gaussians)
    return verts.to(torch.float32), faces.to(torch.int32)


def _frame_deltas(d, F, like, name):
    """a delta as render_batch takes it -- [F,N,3], a list of F ([N,3] or scalars), or one shared [N,3] / scalar --
    as [F,N,3] (a shared delta is expanded, not copied)"""
    if isinstance(d, (list, tuple)):
        if len(d) != F:
            raise ValueError(f"{name}: {len(d)} per-frame entries for {F} frames")
        return torch.stack([x if torch.is_tensor(x) else torch.zeros_like(like) + x for x in d])
    if torch.is_tensor(d) and d.dim() == 3:
        if d.shape[0] != F:
            raise ValueError(f"{name}: {d.shape[0]} per-frame entries for {F} frames")
        return d
    d = d if torch.is_tensor(d) else torch.zeros_like(like) + d
    return d.expand(F, *like.shape)


def _frame_count(*ds):
    counts = {len(d) if isinstance(d, (list, tuple)) else d.shape[0] for d in ds
              if isinstance(d, (list, tuple)) or (torch.is_tensor(d) and d.dim() == 3)}
    if len(counts) > 1:
        raise ValueError(f"per-frame deltas: mismatched frame counts {sorted(counts)}")
    return counts.pop() if counts else None


def extract_mesh_batch(gaussians, d_xyz, d_normal, freeze_pos=False, frames=None):
    """`extract_mesh` for F frames in one call: (verts list, faces list), frame k's mesh from xyz + d_xyz[k] and
    normal + d_normal[k].  The deltas are given as render_batch takes them: [F,N,3], a list of F, or a shared
    [N,3] / 0.0 (`frames` gives F when no delta is per frame).  One DPSR.forward_signed over the F point sets --
    every frame's field takes its sign from its own psr[k,0,0,0] -- and one DiffMC.forward_batch, so the branch
    waits for the host once.  The lists hold views of one vertex tensor and one face tensor (int32, indices local
    to the frame)."""
    F = _frame_count(d_xyz, d_normal)
    if F is None:
        F = 1 if frames is None else int(frames)
    elif frames is not None and int(frames) != F:
        raise ValueError(f"extract_mesh_batch: frames={frames} but the deltas hold {F} frames")
    like = gaussians.get_xyz
    d_xyz, d_normal = _frame_deltas(d_xyz, F, like, "d_xyz"), _frame_deltas(d_normal, F, like, "d_normal")
    dpsr_points, normals = _dpsr_inputs(gaussians, d_xyz, d_normal, freeze_pos)
    if hasattr(gaussians.dpsr, "forward_signed"):
        psr = gaussians.dpsr.forward_signed(dpsr_points, normals, gaussians.density_thres_param)
        psr = psr.reshape(F, *psr.shape[-3:])
    else:  # a reference DPSR module: every frame's own sign, without a host read
        psr = gaussians.dpsr(dpsr_points, normals)
        sign = torch.where(psr[:, :1, :1, :1].detach() < 0, -1.0, 1.0)
        psr = psr * sign - gaussians.density_thres_param
    verts, faces = gaussians.diffmc.forward_batch(psr, isovalue=0.0)
    counts = [v.shape[0] for v in verts]
    verts = _to_world(torch.cat(verts), gaussians).to(torch.float32)
    return list(torch.split(verts, counts)), [f.to(torch.int32) for f in faces]


def extract_gaussian_mesh(gaussians, d_xyz, d_rotation, d_scaling, level, resolution, is_6dof=False, cutoff=3.0):
    """The counterpart of `extract_mesh` from the Gaussians' own density: the level set phi = `level` of their
    opacity field (opacity_field.opacity_field) on a `resolution`^3 grid over the box [c - s, c + s]
    (c = gaussians.gaussian_center, s = gaussians.gaussian_scale), as (verts [V,3] float32 in world space, faces
    [F,3] int32).  The Gaussians are deformed by (d_xyz, d_rotation, d_scaling, is_6dof) exactly as `render` deforms
    them.  Marching cubes runs on level - phi, so that the outside is positive as in `extract_mesh`'s field and the
    faces are oriented the same way.  The vertices are differentiable in the Gaussians' means, scales, rotations and
    opacities (and whatever the deltas depend on)."""
    from gaussian_renderer import _gaussian_geometry
    from opacity_field import opacity_field
    means3D, scales, rotations = _gaussian_geometry(gaussians, d_xyz, d_rotation, d_scaling, is_6dof)
    dev = means3D.device
    c = torch.as_tensor(gaussians.gaussian_center, dtype=torch.float32, device=dev).reshape(-1)
    s = torch.as_tensor(gaussians.gaussian_scale, dtype=torch.float32, device=dev).reshape(-1)
    box = torch.stack([(c - s).expand(3), (c + s).expand(3)]).detach()
    phi = opacity_field(means3D, scales, rotations, gaussians.get_opacity, box, resolution, cutoff=cutoff)
    verts, faces = gaussians.diffmc(level - phi, deform=None, isovalue=0.0)
    verts = verts * 2.0 - 1.0  # [-1, 1]
    verts = verts * gaussians.gaussian_scale + gaussians.gaussian_center
    return verts.to(torch.float32), faces.to(torch.int32)


TSDF_CHUNK = 16   # cameras rendered per render_batch call in extract_tsdf_mesh


def extract_tsdf_mesh(cameras, gaussians, pipe, bg_color, d_xyz, d_rotation, d_scaling, resolution, sdf_trunc=None,
                      depth_max=math.inf, depth_ratio=0.0, alpha_min=0.5, is_6dof=False, color=True, box=None,
                      **options):
    """The mesh 2DGS-style pipelines export: the Gaussians deformed once by (d_xyz, d_rotation, d_scaling), i.e. at
    one time t, rendered from every camera in `cameras` (render_batch under no_grad, TSDF_CHUNK cameras at a
    time), each view's surface depth fused into a tsdf.TSDFVolume of `resolution`^3 nodes, and
    TSDFVolume.extract_mesh: (verts [V,3] float32 in world space, faces [F,3] int32, vertex colours [V,3] or None).

    Surface depth: s = (1 - depth_ratio) depth / alpha (0 where alpha == 0) + depth_ratio median_depth, as
    gaussian_renderer.depth_normal forms it; pixels with alpha < alpha_min get 0 (unobserved).  planar=True fuses
    the planar-depth maps instead (render_batch(..., planar=True): each Gaussian's depth on its own plane, so tilted
    surfaces are not stair-stepped): (1 - depth_ratio) planar_depth / alpha + depth_ratio planar_median_depth.
    (planar is taken as a keyword option so that the positional parameters and their defaults stay those of the
    established signature; any other option raises TypeError.)  color=True fuses
    "render" as the colour (so bg_color shows where alpha < 1).  box: [2,3] (lo, hi), by default c -/+ s with
    c = gaussians.gaussian_center and s = gaussians.gaussian_scale, as extract_gaussian_mesh; sdf_trunc: by default
    5 node spacings along the box's largest axis.  Under is_6dof the deformed centres are handed to the rasterizer
    as the offset from get_xyz, which may differ from them in the last bit.  Not differentiable."""
    from gaussian_renderer import _gaussian_means, render_batch
    from tsdf import TSDFVolume
    planar = bool(options.pop("planar", False))
    if options:
        raise TypeError(f"extract_tsdf_mesh: unexpected keyword arguments {sorted(options)}")
    with torch.no_grad():
        dev = gaussians.get_xyz.device
        if box is None:
            c = torch.as_tensor(gaussians.gaussian_center, dtype=torch.float32, device=dev).reshape(-1)
            s = torch.as_tensor(gaussians.gaussian_scale, dtype=torch.float32, device=dev).reshape(-1)
            box = torch.stack([(c - s).expand(3), (c + s).expand(3)])
        box = torch.as_tensor(box, dtype=torch.float32, device=dev).reshape(2, 3)
        if sdf_trunc is None:
            sdf_trunc = 5.0 * float((box[1] - box[0]).max()) / (resolution - 1)
        vol = TSDFVolume(box, resolution, sdf_trunc, depth_max, color=color)
        if is_6dof:
            d_xyz = _gaussian_means(gaussians, d_xyz, True) - gaussians.get_xyz
        cameras = list(cameras)
        for k in range(0, len(cameras), TSDF_CHUNK):
            cams = cameras[k:k + TSDF_CHUNK]
            out = render_batch(cams, gaussians, pipe, bg_color, d_xyz, d_rotation, d_scaling, depth_alpha=True,
                               surface=depth_ratio > 0 and not planar, planar=planar)
            depth = surface_depth(out, depth_ratio, alpha_min, planar)
            vol.integrate(cams, depth, out["render"] if color else None)
        return vol.extract_mesh()


def surface_depth(maps, depth_ratio=0.0, alpha_min=0.5, planar=False):
    """The depth extract_tsdf_mesh fuses, from render_batch's (or render_surface's) "depth", "alpha" and, when
    depth_ratio > 0, "median_depth": (1 - r) depth / alpha (0 where alpha == 0) + r median_depth, and 0 where
    alpha < alpha_min.  planar=True reads "planar_depth" and "planar_median_depth" (render_batch(..., planar=True)
    or render_planar) in their place."""
    alpha = maps["alpha"]
    depth, median = ("planar_depth", "planar_median_depth") if planar else ("depth", "median_depth")
    e = torch.where(alpha > 0, maps[depth] / torch.where(alpha > 0, alpha, torch.ones_like(alpha)),
                    torch.zeros_like(alpha))
    s = e if depth_ratio == 0 else (1.0 - depth_ratio) * e + depth_ratio * maps[median]
    return torch.where(alpha >= alpha_min, s, torch.zeros_like(s)).contiguous()


def mesh_renderer(glctx, gaussians, d_xyz, d_normal, fid, deform_back, appearance, freeze_pos=False,
                  whitebackground=False, viewpoint_cam=None):
    """Gaussian mesh renderer (reference :124-233)."""
    verts, faces = extract_mesh(gaussians, d_xyz, d_normal, freeze_pos)
    # Deform mesh vertices back to the canonical mesh and query vertex colour
    N = verts.shape[0]
    time_input = fid.unsqueeze(0).expand(N, -1)
    mesh_deform_back_dxyz, _, _, _ = deform_back.step(verts.detach(), time_input)
    mesh_canonical_xyz = verts + mesh_deform_back_dxyz
    vtx_color = appearance.step(mesh_canonical_xyz, time_input)
    if viewpoint_cam is None:
        return verts, faces, vtx_color
    pose, K, res = _camera(viewpoint_cam)
    # one rasterisation serves the mask and the image (reference: render_mask + render_mesh rasterise twice)
    v_pos_clip, rast_out, topo = _raster(glctx, verts, faces, pose, K, res)
    mask3 = _mask_from(rast_out, v_pos_clip, verts, faces, topo)
    mesh_image = _image_from(rast_out, v_pos_clip, faces, vtx_color, mask3, whitebackground, topo)
    return mask3[0][..., [0]], mesh_image[0], verts, faces, vtx_color


def _camera(viewpoint_cam):
    """(pose, K, [H, W]) of a camera as mesh_renderer renders it.
    The camera is host data (numpy / python floats): intrinsics, pose and their product are formed on the host
    in float32 and uploaded once.  The reference moves them to the GPU first and then inverts two 4x4 matrices
    and reads four intrinsics back there -- six blocking round trips in the middle of the mesh branch."""
    if viewpoint_cam.K is not None:
        K = torch.as_tensor(viewpoint_cam.K).detach().float().cpu()
    else:
        import math
        # utils/graphics_utils.fov2focal (:103-104)
        focalx = viewpoint_cam.image_width / (2 * math.tan(viewpoint_cam.FoVx / 2))
        focaly = viewpoint_cam.image_height / (2 * math.tan(viewpoint_cam.FoVy / 2))
        K = torch.tensor([[focalx, 0, viewpoint_cam.image_width / 2], [0, focaly, viewpoint_cam.image_height / 2],
                          [0, 0, 1]]).float()
    c2w_blender = torch.as_tensor(viewpoint_cam.orig_transform).detach().float().cpu()   # blender/OpenGL camera
    b2cv = _blender2opencv("cpu")
    c2w_opencv = c2w_blender @ b2cv
    pose = torch.inverse(b2cv) @ torch.inverse(c2w_opencv)                    # = w2c in the blender convention
    return pose, K, [viewpoint_cam.image_height, viewpoint_cam.image_width]


def mesh_renderer_batch(glctx, gaussians, d_xyz, d_normal, fids, deform_back, appearance, freeze_pos=False,
                        whitebackground=False, viewpoint_cams=None):
    """`mesh_renderer` for F frames in one call.  fids: [F,1] (or a list of F [1] tensors), each frame's time; the
    deltas as `extract_mesh_batch` takes them.  Returns (verts, faces, vtx_color) lists, or with F cameras
    (masks [F,H,W,1], images [F,3,H,W], verts, faces, vtx_color).  Frame k's result is what mesh_renderer gives for
    frame k on the same mesh: deform_back.step and appearance.step each run once over the F frames' vertices (each
    row at its own frame's time), and one range-mode rasterisation of the F meshes, every one in its own camera's
    clip space, serves the masks and the images.  The cameras must share one resolution (ValueError)."""
    fids = torch.stack(list(fids)) if isinstance(fids, (list, tuple)) else fids
    fids = fids.reshape(fids.shape[0], -1)
    F = fids.shape[0]
    if viewpoint_cams is not None:
        viewpoint_cams = list(viewpoint_cams)
        if len(viewpoint_cams) != F:
            raise ValueError(f"mesh_renderer_batch: {len(viewpoint_cams)} cameras for {F} frames")
        cams = [_camera(c) for c in viewpoint_cams]
        if len({tuple(int(x) for x in c[2]) for c in cams}) > 1:
            raise ValueError("mesh_renderer_batch: the cameras must share one resolution")
    verts, faces = extract_mesh_batch(gaussians, d_xyz, d_normal, freeze_pos, frames=F)
    counts = [v.shape[0] for v in verts]
    verts_all = torch.cat(verts)
    # what is built from the frames' sizes (their vertex counts, the F clip matrices) is uploaded from pinned memory
    # without blocking, so the marching cubes' totals stay the branch's only host wait
    time_input = torch.repeat_interleave(fids, _upload(torch.tensor(counts, dtype=torch.int64), fids.device), dim=0,
                                         output_size=verts_all.shape[0])
    mesh_deform_back_dxyz, _, _, _ = deform_back.step(verts_all.detach(), time_input)
    vtx_color_all = appearance.step(verts_all + mesh_deform_back_dxyz, time_input)
    vtx_color = list(torch.split(vtx_color_all, counts))
    if viewpoint_cams is None:
        return verts, faces, vtx_color
    res = cams[0][2]
    mtx = _upload(torch.stack([_clip_matrix(pose, K, res) for pose, K, _ in cams]), verts_all.device)
    pos = torch.cat([transform_pos(m, v)[0] for m, v in zip(mtx, verts)])
    voff = [0]
    for n in counts[:-1]:
        voff.append(voff[-1] + n)
    tri = torch.cat([f + o for f, o in zip(faces, voff)]).to(torch.int32)
    nf = [f.shape[0] for f in faces]
    ranges = torch.tensor([[sum(nf[:k]), nf[k]] for k in range(F)], dtype=torch.int32)
    rast, _ = dr.rasterize(glctx, pos, tri, resolution=res, ranges=ranges)
    topo = dr.edge_opposites(tri, pos.shape[0]) if tri.shape[0] else None
    mask3 = _mask_from(rast, pos, verts_all, tri, topo)
    images = _image_from(rast, pos, tri, vtx_color_all, mask3, whitebackground, topo)
    return mask3[..., :1], images, verts, faces, vtx_color

def __getattr__(name):
    """Names this drop-in does not define (`mesh_shape_renderer`, `pointcloud_renderer`: PyTorch3D /
    matplotlib visualisation helpers used by render_test.py / render_trajectory.py, outside the hot
    path) resolve to the reference's own `utils/renderer.py`, found through the merged `utils` package
    path that launch.install() sets up (this directory first, the reference's second)."""
    import importlib.util
    import os
    import sys
    pkg = sys.modules.get("utils")
    here = os.path.dirname(os.path.abspath(__file__))
    for d in list(getattr(pkg, "__path__", [])):
        cand = os.path.join(d, "renderer.py")
        if os.path.abspath(d) != here and os.path.exists(cand):
            mod = sys.modules.get("_reference_utils_renderer")
            if mod is None:
                spec = importlib.util.spec_from_file_location("_reference_utils_renderer", cand)
                mod = importlib.util.module_from_spec(spec)
                sys.modules["_reference_utils_renderer"] = mod
                spec.loader.exec_module(mod)
            if hasattr(mod, name):
                return getattr(mod, name)
    raise AttributeError(f"module 'utils.renderer' has no attribute {name!r}")
