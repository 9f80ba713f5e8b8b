"""ctypes binding of libdgmesh_b200.so (the C-ABI in include/dgmesh_b200.h).

PyTorch only supplies device memory (`tensor.data_ptr()`) and the CUDA stream; all
compute is in the shared library.  There is NO fallback: if the library is missing
or a call fails, an exception is raised.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdgmesh_b200.so")
# experiments only: an alternative build of the same library (never a different implementation)
LIB_PATH = os.environ.get("DGMESH_B200_LIB", LIB_PATH)

c_void_p, c_int, c_float, c_size_t, c_int64 = (ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t,
                                               ctypes.c_int64)
c_int32, byref = ctypes.c_int32, ctypes.byref
P = c_void_p  # every device pointer crosses the boundary as a plain address

# name -> (restype, argtypes); must list every symbol declared in include/dgmesh_b200.h
SIGNATURES = {
    "dgm_version": (ctypes.c_char_p, []),
    "dgm_last_error": (ctypes.c_char_p, []),
    "dgr_workspace_sizes": (c_int, [c_int, c_int, c_int, c_int64, ctypes.POINTER(c_size_t),
                                    ctypes.POINTER(c_size_t), ctypes.POINTER(c_size_t)]),
    "dgm_notify_create": (c_int, [ctypes.POINTER(c_void_p)]),
    "dgm_notify_host": (c_void_p, [P]),
    "dgm_notify_event": (c_void_p, [P]),
    "dgm_notify_wait": (c_int, [P]),
    "dgm_notify_destroy": (c_int, [P]),
    "dgr_forward": (c_int, [c_int, c_int, c_int, P, c_int, c_int, P, P, P, P, P, c_float, P, P, P, P, P,
                            c_float, c_float, c_int, P, P, P, c_size_t, P, c_size_t, c_int64, P, c_size_t, P, P, P,
                            c_float, c_float, c_int, P]),
    "dgr_backward": (c_int, [c_int, c_int, c_int, P, c_int, c_int, P, P, P, P, c_float, P, P, P, P, P,
                             c_float, c_float, P, P, P, c_int64, P, P, P, P, P, P, P, P, P, P, P, P]),
    "dgr_forward_batch": (c_int, [c_int, c_int, c_int, c_int, P, c_int, c_int, P, P, P, P, P, c_float, P, P, c_int,
                                  P, P, P, P, P, c_int, P, P, P, c_size_t, P, c_size_t, c_int64, P, c_size_t, P, P, P,
                                  c_float, c_float, c_int, c_int, P]),
    "dgr_backward_batch": (c_int, [c_int, c_int, c_int, c_int, P, c_int, c_int, P, P, P, P, c_float, P, P, c_int,
                                   P, P, P, P, P, P, P, c_size_t, P, c_size_t, c_int64, P, c_size_t, P, P, P, P, P, P,
                                   P, P, P, c_int, P]),
    # the *_aux variants: their counterpart's arguments + two [.., H, W] maps (see include/dgmesh_b200.h)
    "dgr_forward_aux": (c_int, [c_int, c_int, c_int, P, c_int, c_int, P, P, P, P, P, c_float, P, P, P, P, P,
                                c_float, c_float, c_int, P, P, P, P, P, c_size_t, P, c_size_t, c_int64, P, c_size_t,
                                P, P, P, c_float, c_float, c_int, P]),
    "dgr_backward_aux": (c_int, [c_int, c_int, c_int, P, c_int, c_int, P, P, P, P, c_float, P, P, P, P, P,
                                 c_float, c_float, P, P, P, c_int64, P, P, P, P, P, P, P, P, P, P, P, P, P, P]),
    "dgr_forward_batch_aux": (c_int, [c_int, c_int, c_int, c_int, P, c_int, c_int, P, P, P, P, P, c_float, P, P,
                                      c_int, P, P, P, P, P, c_int, P, P, P, P, P, c_size_t, P, c_size_t, c_int64, P,
                                      c_size_t, P, P, P, c_float, c_float, c_int, c_int, P]),
    "dgr_backward_batch_aux": (c_int, [c_int, c_int, c_int, c_int, P, c_int, c_int, P, P, P, P, c_float, P, P,
                                       c_int, P, P, P, P, P, P, P, c_size_t, P, c_size_t, c_int64, P, c_size_t, P,
                                       P, P, P, P, P, P, P, P, P, P, c_int, P]),
    # the *_cam variants: their *_aux counterpart's arguments + three camera gradients and a workspace
    "dgr_camera_grad_workspace_size": (c_int, [c_int, c_int, ctypes.POINTER(c_size_t)]),
    "dgr_backward_cam": (c_int, [c_int, c_int, c_int, P, c_int, c_int, P, P, P, P, c_float, P, P, P, P, P,
                                 c_float, c_float, P, P, P, c_int64, P, P, P, P, P, P, P, P, P, P, P, P, P,
                                 P, P, P, P, c_size_t, P]),
    "dgr_backward_batch_cam": (c_int, [c_int, c_int, c_int, c_int, P, c_int, c_int, P, P, P, P, c_float, P, P,
                                       c_int, P, P, P, P, P, P, P, c_size_t, P, c_size_t, c_int64, P, c_size_t, P,
                                       P, P, P, P, P, P, P, P, P, P, P, P, P, P, c_size_t, c_int, P]),
    # the *_nrm variants: the normal map (forward: *_aux + normals, out_normal, workspace; backward: *_cam +
    # the map's gradient, dL/dnormals, workspace)
    "dgr_normal_workspace_size": (c_int, [c_int, c_int64, ctypes.POINTER(c_size_t)]),
    "dgr_forward_nrm": (c_int, [c_int, c_int, c_int, P, c_int, c_int, P, P, P, P, P, c_float, P, P, P, P, P,
                                c_float, c_float, c_int, P, P, P, P, P, P, P, c_size_t, P, c_size_t, P, c_size_t,
                                c_int64, P, c_size_t, P, P, P, c_float, c_float, c_int, P]),
    "dgr_backward_nrm": (c_int, [c_int, c_int, c_int, P, c_int, c_int, P, P, P, P, c_float, P, P, P, P, P,
                                 c_float, c_float, P, P, P, c_int64, P, P, P, P, P, P, P, P, P, P, P, P, P,
                                 P, P, P, P, c_size_t, P, P, P, P]),
    "dgr_forward_batch_nrm": (c_int, [c_int, c_int, c_int, c_int, P, c_int, c_int, P, P, P, P, P, c_float, P, P,
                                      c_int, P, P, P, P, P, c_int, P, P, P, P, P, c_int, P, P, c_size_t, P,
                                      c_size_t, P, c_size_t, c_int64, P, c_size_t, P, P, P, c_float, c_float, c_int,
                                      c_int, P]),
    "dgr_backward_batch_nrm": (c_int, [c_int, c_int, c_int, c_int, P, c_int, c_int, P, P, P, P, c_float, P, P,
                                       c_int, P, P, P, P, P, P, P, c_size_t, P, c_size_t, c_int64, P, c_size_t, P,
                                       P, P, P, P, P, P, P, P, P, P, P, P, P, P, c_size_t, P, c_int, P, P,
                                       c_size_t, c_int, P]),
    "dgr_mark_visible": (c_int, [c_int, P, P, P, P, P]),
    "dgr_export_state": (c_int, [c_int, c_int, c_int, c_int64, P, P, P] + [P] * 12 + [P]),
    "dgk_workspace_size": (c_int, [c_int, ctypes.POINTER(c_size_t)]),
    "dgk_dist2": (c_int, [c_int, P, P, P, c_size_t, P]),
    "dgk_nearest": (c_int, [c_int, P, c_int, P, P, P, P]),
    "dgp_plan_create": (c_int, [c_int, ctypes.POINTER(c_void_p), ctypes.POINTER(c_size_t)]),
    "dgp_plan_destroy": (c_int, [P]),
    "dgp_forward": (c_int, [P, c_int, ctypes.c_double, P, P, c_int, P, P, P, c_size_t, P]),
    "dgp_backward": (c_int, [P, c_int, P, P, c_int, P, P, P, P, P, c_size_t, P]),
    "dgp_batch_workspace_size": (c_int, [P, c_int, ctypes.POINTER(c_size_t)]),
    "dgp_forward_batch": (c_int, [P, c_int, c_int, ctypes.c_double, P, P, c_int, P, P, P, c_size_t, P]),
    "dgp_backward_batch": (c_int, [P, c_int, c_int, P, P, c_int, P, P, P, P, P, c_size_t, P]),
    "dgmc_workspace_size": (c_int, [c_int, ctypes.POINTER(c_size_t)]),
    "dgmc_count": (c_int, [c_int, P, c_float, P, c_size_t, P, P, P, P]),
    "dgmc_emit": (c_int, [c_int, P, c_float, P, c_size_t, P, P, c_int64, P, c_int64, P]),
    "dgmc_backward": (c_int, [c_int, c_int, P, c_float, P, P, P, P]),
    "dgdmc_workspace_size": (c_int, [c_int, ctypes.POINTER(c_size_t)]),
    "dgdmc_workspace_size_batch": (c_int, [c_int, c_int, ctypes.POINTER(c_size_t)]),
    "dgdmc_count": (c_int, [c_int, P, c_float, P, c_size_t, P, P, P, P]),
    "dgdmc_count_batch": (c_int, [c_int, c_int, P, c_float, P, c_size_t, P, P, P, P]),
    "dgdmc_emit": (c_int, [c_int, P, c_float, P, c_size_t, P, P, c_int64, P, P, c_int64, P]),
    "dgdmc_emit_batch": (c_int, [c_int, c_int, P, c_float, P, c_size_t, P, P, c_int64, P, P, c_int64, P]),
    "dgdmc_backward": (c_int, [c_int, c_int, P, c_float, P, c_size_t, P, P, P, P]),
    "dgdmc_backward_batch": (c_int, [c_int, c_int, P, P, c_float, P, c_size_t, P, P, P, P]),
    "dgfc_emit": (c_int, [c_int, P, c_float, P, P, P, P, c_int, c_int, P, c_size_t, P, P, P, P, c_int64, P, P,
                          c_int64, P]),
    "dgfc_backward_workspace_size": (c_int, [c_int, c_int, c_int, c_int, ctypes.POINTER(c_size_t)]),
    "dgfc_backward": (c_int, [c_int, c_int, c_int, P, c_float, P, P, P, P, c_int, c_int, P, P, P, P, P, P, c_size_t,
                              P, P, P, P, P, P]),
    "dgmc_workspace_size_batch": (c_int, [c_int, c_int, ctypes.POINTER(c_size_t)]),
    "dgmc_count_batch": (c_int, [c_int, c_int, P, c_float, P, c_size_t, P, P, P, P]),
    "dgmc_emit_batch": (c_int, [c_int, c_int, P, c_float, P, c_size_t, P, P, c_int64, P, c_int64, P]),
    "dgmc_backward_batch": (c_int, [c_int, c_int, P, P, c_float, P, P, P, P]),
    "dgl_gemm_ws_bytes": (c_int, [c_int, c_int, c_int, ctypes.POINTER(c_size_t)]),
    "dgl_gemm_bf16": (c_int, [c_int, c_int, c_int, P, c_int, P, c_int, P, c_int, P, c_int, P, c_size_t, P]),
    "dgl_gemm_tn_bf16": (c_int, [c_int, c_int, c_int, P, c_int, P, c_int, P, c_int, c_int, P, c_size_t, P]),
    "dgl_mlp_pack_sizes": (c_int, [ctypes.POINTER(c_size_t), ctypes.POINTER(c_size_t), ctypes.POINTER(c_size_t)]),
    "dgl_mlp_pack": (c_int, [P, P, P, P, P]),
    "dgl_mlp_grad_pointers": (c_int, [P, P]),
    "dgl_mlp_unpack_grads": (c_int, [P, P, P, P]),
    "dgl_mlp_workspace": (c_int, [c_int, c_int, ctypes.POINTER(c_size_t)]),
    "dgl_mlp_forward": (c_int, [P, c_int, P, P, P, c_int, P, c_size_t, P]),
    "dgl_mlp_backward": (c_int, [P, c_int, P, P, P, P, c_size_t, P, P, P]),
    "dgl_laplacian_workspace": (c_int, [c_int, ctypes.POINTER(c_size_t)]),
    "dgl_laplacian_forward": (c_int, [c_int, c_int, P, P, P, P, c_size_t, P]),
    "dgl_laplacian_backward": (c_int, [c_int, c_int, P, P, P, P, c_size_t, P]),
    "dgmr_rasterize": (c_int, [c_int, c_int, c_int, c_int, P, P, P, P, P]),
    "dgmr_rasterize_bwd": (c_int, [c_int, c_int, P, P, P, P, P, P]),
    "dgmr_interpolate": (c_int, [c_int, c_int, c_int, P, P, P, P, P]),
    "dgmr_interpolate_bwd": (c_int, [c_int, c_int, c_int, P, P, P, P, P, P, P]),
    "dgmr_antialias": (c_int, [c_int, c_int, c_int, P, P, P, P, P, P, P]),
    "dgmr_antialias_bwd": (c_int, [c_int, c_int, c_int, P, P, P, P, P, P, P, P, P]),
    "dgmr_rasterize_batch": (c_int, [c_int, c_int, c_int, P, c_int, c_int, P, P, P, P, P]),
    "dgmr_rasterize_bwd_batch": (c_int, [c_int, c_int, c_int, P, P, P, P, P, P]),
    "dgmr_interpolate_batch": (c_int, [c_int, c_int, c_int, c_int, P, P, P, P, P]),
    "dgmr_interpolate_bwd_batch": (c_int, [c_int, c_int, c_int, c_int, P, P, P, P, P, P, P]),
    "dgmr_antialias_batch": (c_int, [c_int, c_int, c_int, c_int, P, P, P, P, P, P, P]),
    "dgmr_antialias_bwd_batch": (c_int, [c_int, c_int, c_int, c_int, P, P, P, P, P, P, P, P, P]),
    "dgd_workspace_size": (c_int, [c_int, ctypes.POINTER(c_size_t)]),
    "dgd_plan": (c_int, [c_int, P, P, P, P, c_float, c_float, ctypes.c_double, ctypes.c_double, c_int, c_float, P,
                         c_size_t, P, P]),
    "dgd_split_stds": (c_int, [c_int, P, P, c_size_t, P, P]),
    "dgd_apply": (c_int, [c_int, c_int, P, P, P, P, c_size_t, P]),
    "dgx_allreduce_nvls": (c_int, [P, c_size_t, P, c_int, c_int, ctypes.c_uint32, c_float, c_int, P]),
    "dgm_profile_enable": (c_int, [c_int]),
    "dgloss_workspace_size": (c_int, [c_int, c_int, ctypes.POINTER(c_size_t)]),
    "dgloss_forward": (c_int, [c_int, c_int, P, P, c_float, c_int, P, P, c_size_t, P]),
    "dgloss_backward": (c_int, [c_int, c_int, P, P, c_float, c_int, P, P, P, c_size_t, P]),
    "dgm_profile_read": (c_int, [ctypes.POINTER(c_float), c_int]),
    "dgm_timeline_read": (c_int, [ctypes.POINTER(c_float), ctypes.POINTER(c_float), ctypes.POINTER(c_int), c_int]),
}


def _surf(nrm_name, at, extra):
    """The *_surf variant of a *_nrm entry: its arguments with `extra` inserted at position `at`."""
    args = SIGNATURES[nrm_name][1]
    return (c_int, args[:at] + extra + args[at:])


# the *_surf variants: the median-depth and distortion maps (forward: *_nrm + near, far, the two maps and the
# surface workspace after the normal workspace; backward: *_nrm + near, far, the maps' gradients and the workspace)
SIGNATURES.update({
    "dgr_surface_workspace_size": (c_int, [c_int, c_int, ctypes.POINTER(c_size_t)]),
    "dgr_forward_surf": _surf("dgr_forward_nrm", 28, [c_float, c_float, P, P, P, c_size_t]),
    "dgr_backward_surf": _surf("dgr_backward_nrm", -1, [c_float, c_float, P, P, P]),
    "dgr_forward_batch_surf": _surf("dgr_forward_batch_nrm", 31, [c_float, c_float, P, P, P, c_size_t]),
    "dgr_backward_batch_surf": _surf("dgr_backward_batch_nrm", -2, [c_float, c_float, P, P, P, c_size_t]),
})
# the absolute screen-space gradient: the *_surf backward + the [P,3] / [F,P,3] output before the stream arguments
SIGNATURES.update({
    "dgr_backward_abs": _surf("dgr_backward_surf", -1, [P]),
    "dgr_backward_batch_abs": _surf("dgr_backward_batch_surf", -2, [P]),
})
# the intrinsics gradient: the *_abs backward + the [2] / [F,2] dL/dtan(fov/2) output before the stream arguments
SIGNATURES.update({
    "dgr_backward_intr": _surf("dgr_backward_abs", -1, [P]),
    "dgr_backward_batch_intr": _surf("dgr_backward_batch_abs", -2, [P]),
})

# the feature-map pass over an earlier forward's workspaces: (F, P, C, W, H, features, per_frame, geom, stride,
# binning, stride, R_cap, img, stride) + forward: out_map, feat_ws, bytes / backward: map, dL_dmap, dL_dfeatures,
# feat_ws, bytes; + stream
_FEAT_HEAD = [c_int, c_int, c_int, c_int, c_int, P, c_int, P, c_size_t, P, c_size_t, c_int64, P, c_size_t]
SIGNATURES.update({
    "dgr_feature_workspace_size": (c_int, [c_int, c_int, c_int, ctypes.POINTER(c_size_t)]),
    "dgr_features_fwd": (c_int, _FEAT_HEAD + [P, P, c_size_t, P]),
    "dgr_features_bwd": (c_int, _FEAT_HEAD + [P, P, P, P, c_size_t, P]),
})
# planar depth: the plane op (F, P, W, H, means3D, scales, scale_modifier, rotations, cov3D_precomp, per_frame,
# viewmatrices, tan_fovx_host, tan_fovy_host) + forward: planes, normals / backward: dL_dplanes, dL_dnormals,
# dL_dmeans3D, dL_dscales, dL_drotations, dL_dcov3D; the pass (F, P, W, H, planes, geom, stride, binning, stride,
# R_cap, img, stride) + forward: planar_depth, planar_median, ws, bytes / backward: planar_depth, dL_dplanar_depth,
# dL_dplanar_median, dL_dplanes, ws, bytes; + stream
_PLANE_HEAD = [c_int, c_int, c_int, c_int, P, P, c_float, P, P, c_int, P, P, P]
_PLANAR_HEAD = [c_int, c_int, c_int, c_int, P, P, c_size_t, P, c_size_t, c_int64, P, c_size_t]
SIGNATURES.update({
    "dgr_gaussian_planes_fwd": (c_int, _PLANE_HEAD + [P, P, P]),
    "dgr_gaussian_planes_bwd": (c_int, _PLANE_HEAD + [P, P, P, P, P, P, P]),
    "dgr_planar_workspace_size": (c_int, [c_int, c_int, c_int, c_int, ctypes.POINTER(c_size_t)]),
    "dgr_planar_fwd": (c_int, _PLANAR_HEAD + [P, P, P, c_size_t, P]),
    "dgr_planar_bwd": (c_int, _PLANAR_HEAD + [P, P, P, P, P, c_size_t, P]),
})
# blend-weight statistics: (F, P, W, H, binning, stride, R_cap, img, stride, pixel_weights, weights_per_frame,
# out_sum, out_max, stream)
SIGNATURES["dgr_blend_stats"] = (c_int, [c_int, c_int, c_int, c_int, P, c_size_t, c_int64, P, c_size_t, P, c_int,
                                         P, P, P])
# depth normals: (F, W, H, depth_ratio, depth, alpha, median, coefs_host) + forward: out_normal / backward: dL_dnormal,
# dL_ddepth, dL_dalpha, dL_dmedian; + stream
_DN_HEAD = [c_int, c_int, c_int, c_float, P, P, P, P]
SIGNATURES.update({
    "dgr_depth_normal_fwd": (c_int, _DN_HEAD + [P, P]),
    "dgr_depth_normal_bwd": (c_int, _DN_HEAD + [P, P, P, P, P]),
})



class DgoTensor(ctypes.Structure):
    """Mirror of `struct DgoTensor` (one tensor of a fused Adam step)."""
    _fields_ = [("p", c_void_p), ("g", c_void_p), ("m", c_void_p), ("v", c_void_p), ("n", c_int64),
                ("row_width", c_int), ("step_size", c_float), ("inv_bc2_sqrt", c_float), ("eps", c_float)]


DGO_MAX_TENSORS = 32
# the optimiser step: (n_tensors, tensors_host, beta1, beta2, row_radii, zero_grad, stream); the densification
# statistics: (F, P, grad, abs_grad, grad_stride, radii, radii_stride, accum, accum_abs, denom, max_radii2D, stream)
SIGNATURES.update({
    "dgo_adam_step": (c_int, [c_int, ctypes.POINTER(DgoTensor), ctypes.c_double, ctypes.c_double, P, c_int, P]),
    "dgo_densify_stats": (c_int, [c_int, c_int, P, P, c_int64, P, c_int64, P, P, P, P, P]),
})

# the opacity field: (P, G, means3D, scales, rotations, opacities, box, cutoff, scale_modifier, pair_cap, ws, bytes)
# + forward: phi, pairs_host, pairs_event / backward: dL_dphi, dL_dmeans3D, dL_dscales, dL_drotations,
# dL_dopacities; + stream
_OF_HEAD = [c_int, c_int, P, P, P, P, P, c_float, c_float, c_int64, P, c_size_t]
SIGNATURES.update({
    "dgf_workspace_size": (c_int, [c_int, c_int, c_int64, ctypes.POINTER(c_size_t)]),
    "dgf_forward": (c_int, _OF_HEAD + [P, P, P, P]),
    "dgf_backward": (c_int, _OF_HEAD + [P, P, P, P, P, P]),
})
# TSDF fusion: (G, box, F, W, H, views_host, coefs_host, depth, color, sdf_trunc, depth_max, tsdf, weight,
# color_grid, stream)
SIGNATURES["dgt_integrate"] = (c_int, [c_int, P, c_int, c_int, c_int, P, P, P, P, c_float, c_float, P, P, P, P])

# structural losses: (B, N, M, xyz1, xyz2) + nn_distance: dist1, idx1, dist2, idx2 / its backward: idx1, idx2,
# grad_dist1, grad_dist2, grad_xyz1, grad_xyz2, ws, bytes / match_cost: cost, ws, bytes / its backward: grad_cost,
# grad_xyz1, grad_xyz2, ws, bytes; + stream
_DGE_SIZE = (c_int, [c_int, c_int, c_int, ctypes.POINTER(c_size_t)])
SIGNATURES.update({
    "dge_nn_distance": (c_int, [c_int, c_int, c_int, P, P, P, P, P, P, P]),
    "dge_nn_distance_workspace": _DGE_SIZE,
    "dge_nn_distance_bwd": (c_int, [c_int, c_int, c_int, P, P, P, P, P, P, P, P, P, c_size_t, P]),
    "dge_match_cost_workspace": _DGE_SIZE,
    "dge_match_cost": (c_int, [c_int, c_int, c_int, P, P, P, P, c_size_t, P]),
    "dge_match_cost_bwd": (c_int, [c_int, c_int, c_int, P, P, P, P, P, P, c_size_t, P]),
})

# point-to-mesh distance: (V, F, Q) + forward: verts, faces, points, dist2, face, bary, ws, bytes / backward: verts,
# faces, points, face, bary, grad_dist2, grad_points, grad_verts, ws, bytes; + stream
SIGNATURES.update({
    "dgpm_forward_workspace": _DGE_SIZE,
    "dgpm_forward": (c_int, [c_int, c_int, c_int, P, P, P, P, P, P, P, c_size_t, P]),
    "dgpm_backward_workspace": _DGE_SIZE,
    "dgpm_backward": (c_int, [c_int, c_int, c_int, P, P, P, P, P, P, P, P, P, c_size_t, P]),
    # winding: verts, faces, points, beta, winding, dist2, face, bary, ws, bytes
    "dgpm_winding_workspace": _DGE_SIZE,
    "dgpm_winding": (c_int, [c_int, c_int, c_int, P, P, P, c_float, P, P, P, P, P, c_size_t, P]),
})

# deformation regularisers: the graph (P, K, weight_lambda, points, index, dist2, weight, inv_offsets, inv_pairs, ws,
# bytes, stream); the losses (F, P, K, index, weight, [inv_offsets, inv_pairs,] xyz_a, rot_a, xyz_b, rot_b) +
# forward: losses, ws, bytes / backward: grad_losses, four gradients, ws, bytes; + stream
SIGNATURES.update({
    "dgkg_workspace": (c_int, [c_int, c_int, ctypes.POINTER(c_size_t)]),
    "dgkg_build": (c_int, [c_int, c_int, c_float, P, P, P, P, P, P, P, c_size_t, P]),
    "dgdr_forward_workspace": _DGE_SIZE,
    "dgdr_forward": (c_int, [c_int, c_int, c_int, P, P, P, P, P, P, P, P, c_size_t, P]),
    "dgdr_backward_workspace": _DGE_SIZE,
    "dgdr_backward": (c_int, [c_int, c_int, c_int, P, P, P, P, P, P, P, P, P, P, P, P, P, P, c_size_t, P]),
})

# HexPlane field: (F, N, S, C, res_host, R_t) + forward: box, x, t, planes_host, out / backward: box, x, t,
# planes_host, grad_out, grad_x, grad_planes_host, ws, bytes; the regularisers (S, C, res_host, R_t, planes_host) +
# forward: losses, ws, bytes / backward: grad_losses, grad_planes_host; + stream
_HP_HEAD = [c_int, c_int, c_int, c_int, P, c_int]
SIGNATURES.update({
    "dghp_forward": (c_int, _HP_HEAD + [P, P, P, P, P, P]),
    "dghp_backward_workspace": (c_int, _HP_HEAD + [ctypes.POINTER(c_size_t)]),
    "dghp_backward": (c_int, _HP_HEAD + [P, P, P, P, P, P, P, P, c_size_t, P]),
    "dghp_reg_workspace": (c_int, _HP_HEAD[2:] + [ctypes.POINTER(c_size_t)]),
    "dghp_reg_forward": (c_int, _HP_HEAD[2:] + [P, P, P, c_size_t, P]),
    "dghp_reg_backward": (c_int, _HP_HEAD[2:] + [P, P, P, P]),
})

# hash-grid field: (F, N, G, grids_host, L, Fe, log2_table, res_host, R_t) + forward: box, x, t, tables_host, out /
# backward: box, x, t, tables_host, grad_out, grad_x, grad_tables_host, ws, bytes; + stream
_HG_HEAD = [c_int, c_int, c_int, P, c_int, c_int, c_int, P, c_int]
SIGNATURES.update({
    "dghg_forward": (c_int, _HG_HEAD + [P, P, P, P, P, P]),
    "dghg_backward_workspace": (c_int, _HG_HEAD + [ctypes.POINTER(c_size_t)]),
    "dghg_backward": (c_int, _HG_HEAD + [P, P, P, P, P, P, P, P, c_size_t, P]),
})

KERNEL_NAMES = ["preprocess", "tile_scan", "scatter", "sort_pack", "render_fwd", "render_bwd", "preprocess_bwd",
                "count", "normal_grad_finish", "median_grad", "feature_fwd", "feature_bwd", "feature_grad_finish",
                "blend_stats"]


def profile_read():
    """{kernel name: ms of its most recent launch} (synchronises the profiling events)."""
    buf = (c_float * 16)()
    check(lib().dgm_profile_read(buf, 16), "dgm_profile_read")
    return {n: float(buf[i]) for i, n in enumerate(KERNEL_NAMES) if buf[i] >= 0}



class DglNet(ctypes.Structure):
    """Mirror of `struct DglNet` (include/dgmesh_b200.h)."""
    _fields_ = [("has_timenet", c_int), ("in_t", c_int), ("n_out", c_int), ("sigmoid_out", c_int),
                ("W", c_void_p * 8), ("WT", c_void_p * 8), ("b", c_void_p * 8),
                ("Wh", c_void_p), ("WhT", c_void_p), ("bh", c_void_p),
                ("Wt0", c_void_p), ("bt0", c_void_p), ("Wt1", c_void_p), ("Wt1T", c_void_p), ("bt1", c_void_p),
                ("precise", c_int), ("Wlo", c_void_p * 8), ("Whlo", c_void_p), ("Wt0lo", c_void_p),
                ("Wt1lo", c_void_p)]


class DglRaw(ctypes.Structure):
    """Mirror of `struct DglRaw` (reference-shaped fp32 parameters)."""
    _fields_ = [("has_timenet", c_int), ("in_t", c_int), ("sigmoid_out", c_int), ("n_heads", c_int),
                ("head_rows", c_int * 4), ("W", c_void_p * 8), ("b", c_void_p * 8), ("Wh", c_void_p * 4),
                ("bh", c_void_p * 4), ("Wt0", c_void_p), ("bt0", c_void_p), ("Wt1", c_void_p), ("bt1", c_void_p)]


class DglRawGrads(ctypes.Structure):
    _fields_ = [("W", c_void_p * 8), ("b", c_void_p * 8), ("Wh", c_void_p * 4), ("bh", c_void_p * 4),
                ("Wt0", c_void_p), ("bt0", c_void_p), ("Wt1", c_void_p), ("bt1", c_void_p)]


class DgdField(ctypes.Structure):
    """Mirror of `struct DgdField` (densify_and_prune gather)."""
    _fields_ = [("src", c_void_p), ("m1_src", c_void_p), ("m2_src", c_void_p), ("dst", c_void_p),
                ("m1_dst", c_void_p), ("m2_dst", c_void_p), ("width", c_int), ("role", c_int)]


class DglGrads(ctypes.Structure):
    """Mirror of `struct DglGrads`."""
    _fields_ = [("dW", c_void_p * 8), ("db", c_void_p * 8), ("dWh", c_void_p), ("dbh", c_void_p),
                ("dWt0", c_void_p), ("dbt0", c_void_p), ("dWt1", c_void_p), ("dbt1", c_void_p)]


_lib = None


class DgmError(RuntimeError):
    pass


def lib():
    """Load (once) and return the ctypes handle; raises if the CUDA library is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise DgmError(
                f"{LIB_PATH} not found: build it with `make` (or __graft_entry__.build()). "
                "dgmesh_b200 has no CPU / PyTorch fallback.")
        h = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(h, name)  # AttributeError if the symbol is missing
            fn.restype = res
            fn.argtypes = args
        _lib = h
    return _lib


def check(rc, what):
    if rc != 0:
        msg = lib().dgm_last_error().decode()
        raise DgmError(f"{what} failed (code {rc}): {msg}")


def ptr(t):
    """Device address of a tensor, or None (NULL) for an absent / zero-element tensor
    (the reference signals "absent" with zero-element tensors, dgr/.../__init__.py:197-207)."""
    if t is None or t.numel() == 0:
        return None
    return t.data_ptr()


_raw_stream = None


def stream_ptr():
    """cudaStream_t of torch's current stream on the current device.  `torch.cuda.current_stream()` builds a
    Stream object (~28 us); the raw query is ~1 us -- this is called twice per rendered frame."""
    global _raw_stream
    import torch
    if _raw_stream is None:
        _raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", False)
    if _raw_stream:
        return _raw_stream(torch.cuda.current_device())
    return torch.cuda.current_stream().cuda_stream
