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


def _raster(glctx, mesh_v_pos, mesh_t_pos_idx, pose, K, resolution):
    proj = K_to_projection(K, resolution[0], resolution[1])
    # camera matrices that arrive on the host are multiplied there: one small upload, no kernel, no blocking read
    mtx = (proj.to(pose.device) @ pose).to(mesh_v_pos.device)
    v_pos_clip = transform_pos(mtx, mesh_v_pos)
    rast_out, _ = dr.rasterize(glctx, v_pos_clip, mesh_t_pos_idx, resolution=resolution)
    topo = dr.edge_opposites(mesh_t_pos_idx, mesh_v_pos.shape[0]) if mesh_t_pos_idx.shape[0] else None
    return v_pos_clip, rast_out, topo


def _mask_from(rast_out, v_pos_clip, mesh_v_pos, mesh_t_pos_idx, topo):
    vtx_color = torch.ones(mesh_v_pos.shape, dtype=torch.float, device=v_pos_clip.device)
    color, _ = dr.interpolate(vtx_color[None, ...], rast_out, mesh_t_pos_idx)
    color = dr.antialias(color, rast_out, v_pos_clip, mesh_t_pos_idx, topology_hash=topo)
    return torch.flip(color[0, :, :], dims=[0])


def _image_from(rast_out, v_pos_clip, mesh_t_pos_idx, vtx_color, mask, whitebackground, topo):
    output, _ = dr.interpolate(vtx_color[None, ...], rast_out, mesh_t_pos_idx)
    output = dr.antialias(output, rast_out, v_pos_clip, mesh_t_pos_idx, topology_hash=topo)
    output = torch.flip(output, dims=[1])[0]
    output[~mask.bool()] = 1 if whitebackground else 0
    return torch.clamp(output, 0.0, 1.0).permute(2, 0, 1)


def render_mask(glctx, mesh_v_pos, mesh_t_pos_idx, pose, K, resolution=[800, 800]):
    """reference :33-66 -> mask [H, W, 3]"""
    v_pos_clip, rast_out, topo = _raster(glctx, mesh_v_pos, mesh_t_pos_idx, pose, K, resolution)
    return _mask_from(rast_out, v_pos_clip, mesh_v_pos, mesh_t_pos_idx, topo)


def render_mesh(glctx, mesh_v_pos, mesh_t_pos_idx, vtx_color, pose, K, resolution=[800, 800], whitebackground=False):
    """reference :69-121 -> image [3, H, W]"""
    v_pos_clip, rast_out, topo = _raster(glctx, mesh_v_pos, mesh_t_pos_idx, pose, K, resolution)
    mask = _mask_from(rast_out, v_pos_clip, mesh_v_pos, mesh_t_pos_idx, topo)
    return _image_from(rast_out, v_pos_clip, mesh_t_pos_idx, vtx_color, mask, whitebackground, topo)


def extract_mesh(gaussians, d_xyz, d_normal, freeze_pos=False):
    """Gaussians (+ deltas) -> (verts [V,3] float32 in world space, faces [F,3] int32): reference :150-175."""
    if freeze_pos:
        dpsr_points = gaussians.get_xyz.detach() + d_xyz.detach()
    else:
        dpsr_points = gaussians.get_xyz + d_xyz
    dpsr_points = (dpsr_points - gaussians.gaussian_center) / gaussians.gaussian_scale  # [-1, 1]
    dpsr_points = dpsr_points / 2.0 + 0.5                                                 # [0, 1]
    dpsr_points = torch.clamp(dpsr_points, SMALL_NUMBER, 1 - SMALL_NUMBER)
    normals = gaussians.get_normal + d_normal
    if hasattr(gaussians.dpsr, "forward_signed"):
        psr = gaussians.dpsr.forward_signed(dpsr_points.unsqueeze(0), normals.unsqueeze(0),
                                            gaussians.density_thres_param)
    else:  # a reference DPSR module: same arithmetic, with its host synchronisation
        psr = gaussians.dpsr(dpsr_points.unsqueeze(0), normals.unsqueeze(0))
        sign = psr[0, 0, 0, 0].detach()  # Sign for Diso is opposite to dpsr
        psr = psr * (-1 if sign < 0 else 1)
        psr = (psr - gaussians.density_thres_param).squeeze(0)
    verts, faces = gaussians.diffmc(psr, deform=None, isovalue=0.0)
    verts = verts * 2.0 - 1.0  # [-1, 1]
    verts = verts * gaussians.gaussian_scale + gaussians.gaussian_center
    return verts.to(torch.float32), faces.to(torch.int32)


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
    # The camera is host data (numpy / python floats): intrinsics, pose and their product are formed on the host
    # in float32 and uploaded once.  The reference moves them to the GPU first and then inverts two 4x4 matrices
    # and reads four intrinsics back there -- six blocking round trips in the middle of the mesh branch.
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
    res = [viewpoint_cam.image_height, viewpoint_cam.image_width]
    # one rasterisation serves the mask and the image (reference: render_mask + render_mesh rasterise twice)
    v_pos_clip, rast_out, topo = _raster(glctx, verts, faces, pose, K, res)
    mask3 = _mask_from(rast_out, v_pos_clip, verts, faces, topo)
    mesh_image = _image_from(rast_out, v_pos_clip, faces, vtx_color, mask3, whitebackground, topo)
    return mask3[..., [0]], mesh_image, verts, faces, vtx_color

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
