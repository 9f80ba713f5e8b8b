// raster_kernels.h -- host-side launch interface between api.cu and the kernel files.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>

namespace dgm {

struct FwdArgs {
  int P, D, M;
  const float* background;
  int W, H;
  const float *means3D, *shs, *colors_precomp, *opacities, *scales;
  float scale_modifier;
  const float *rotations, *cov3D_precomp, *viewmatrix, *projmatrix, *cam_pos;
  float tan_fovx, tan_fovy;
  int prefiltered;
  float* out_color;
  int* radii;
  // optional [H,W] depth and alpha maps (NULL: not rendered; both NULL: the colour-only blend kernel).
  // With out_depth the blend records carry the view depth, which a depth backward needs
  float *out_depth, *out_alpha;
  void *geom_ws, *binning_ws, *img_ws;
  int64_t R_cap;
  int32_t* status;
  // optional: host-mapped (pinned) copy of the status words, written by the tile scan, and the
  // depth range of an earlier frame (hint_hi > hint_lo enables the fused preprocess + count)
  int32_t* status_host;
  float hint_lo, hint_hi;
  int hint_max_tile;         // longest per-tile list of an earlier frame (status word 2), 0: unknown
  cudaEvent_t status_event;  // recorded right after the tile scan (may be null)
  // optional [3,H,W] normal map sum_i n_i alpha_i T_i of the [P,3] `normals` (NULL: not rendered).  Its records
  // and per-Gaussian gradient accumulator live in nrm_ws (NrmWS); a normal forward is also a depth forward
  const float* normals = nullptr;
  float* out_normal = nullptr;
  void* nrm_ws = nullptr;
  // optional [H,W] median-depth and depth-distortion maps (surf_ws non-NULL: the surface forward, which writes
  // the per-pixel state of SurfWS and each map whose pointer is non-NULL); also a depth forward.
  // surf_k = far near / (far - near) of the normalised depth (see surf_m)
  float *out_median = nullptr, *out_distortion = nullptr;
  void* surf_ws = nullptr;
  float surf_k = 0.f;
};

struct BwdArgs {
  int P, D, M;
  const float* background;
  int W, H;
  const float *means3D, *shs, *colors_precomp, *scales;
  float scale_modifier;
  const float *rotations, *cov3D_precomp, *viewmatrix, *projmatrix, *cam_pos;
  const float *tan_fovx, *tan_fovy;  // host arrays, one value per frame
  const int* radii;
  void *geom_ws, *binning_ws, *img_ws;
  int64_t R_cap;
  const float* dL_dpix;
  // optional [H,W] upstream gradients of the depth and alpha maps (both NULL: the colour-only kernels)
  const float *dL_ddepth, *dL_dalpha;
  float *dL_dmean2D, *dL_dconic, *dL_dopacity, *dL_dcolor, *dL_dmean3D, *dL_dcov3D, *dL_dsh, *dL_dscale, *dL_drot;
  // launch_preprocess_bwd covers F frames (1 <= F <= PB_MAX_FRAMES) in one launch: frame f reads the camera at
  // index f (viewmatrix + 16 f, ..., tan_fovx[f]), its workspace at geom_ws + f * geom_stride, radii + f * P,
  // and the slab f of each input whose DGR_PF_* bit is set in per_frame.  dL_dmean2D (and dL_dconic) are
  // [F,P,.]; every other gradient is [F,P,.] when its bit is set and the sum over the frames otherwise.
  // launch_render_bwd reads one frame: frame 0 of the above.
  int F, per_frame;
  size_t geom_stride;
  // optional camera gradients, [F,16], [F,16], [F,3] (all NULL: no camera gradient).  cam_ws is the
  // [F][ceil(P/32)][CAM_TERMS] scratch of the per-warp partials (camera_ws_bytes)
  float *dL_dview = nullptr, *dL_dproj = nullptr, *dL_dcampos = nullptr;
  float* cam_ws = nullptr;
  // optional [F,2] dL/dtan_fovx, dL/dtan_fovy through the EWA covariance (NULL: not formed).  Needs cam_ws of
  // intrinsics_ws_bytes: the intrinsics partials [F][ceil(P/32)][INTR_TERMS] follow the camera partials
  float* dL_dtanfov = nullptr;
  // optional [3,H,W] upstream gradient of the normal map (NULL: the kernels above).  launch_render_bwd adds
  // dL/dnormal into the accumulator of nrm_ws (frame 0); launch_normal_grad_finish reads and re-zeroes the
  // accumulators of the F frames (nrm_ws + f * nrm_stride) and writes dL_dnormals ([F,P,3] with
  // normals_per_frame, else the [P,3] sum over the frames; NULL: only re-zeroes)
  const float* dL_dnormal = nullptr;
  float* dL_dnormals = nullptr;
  void* nrm_ws = nullptr;
  size_t nrm_stride = 0;
  int normals_per_frame = 0;
  // optional [H,W] upstream gradients of the median-depth and distortion maps (NULL: unused), with the surface
  // workspace of the frame's surface forward (surf_k as in FwdArgs).  dL_ddistortion selects the surface blend
  // backward; dL_dmedian adds median_grad_kernel.  Either one sets preprocess_bwd's depth_grad
  const float *dL_dmedian = nullptr, *dL_ddistortion = nullptr;
  void* surf_ws = nullptr;
  float surf_k = 0.f;
  // optional [P,3] absolute screen-space gradient of frame 0 (NULL: not formed): launch_render_bwd adds
  // (sum |dL/dmean2D.x| per pixel, the same of .y) into it with the ABS instances; the caller zeroes it first
  float* dL_dmean2D_abs = nullptr;
};
#define PB_MAX_FRAMES 64

// The workspaces of F frames an earlier forward wrote, which a side pass (features, planar depth, blend statistics)
// reads: frame f's at geom_ws + f * geom_stride, ... (strides 0 for one frame; blend statistics reads no geom_ws)
struct ForwardWS {
  int F, P, W, H;
  void *geom_ws, *binning_ws, *img_ws;
  size_t geom_stride, binning_stride, img_stride;
  int64_t R_cap;
};
// feature maps (raster_feat.cu): features [P,C], or [F,P,C] with per_frame; out_map / map / dL_dmap [F,C,H,W].
// feat_ws holds F per-Gaussian accumulators of dL/dfeatures, feature_ws_stride(P, C) bytes apart: the forward
// clears them, the backward adds into them and launch_features_bwd's finish re-zeroes them while it writes
// dL_dfeatures ([F,P,C] with per_frame, else the [P,C] sum over the frames; NULL: only re-zeroes)
struct FeatArgs : ForwardWS {
  int C;
  const float* features;
  int per_frame;
  float* out_map;           // forward
  const float *map, *dL_dmap;  // backward
  float* dL_dfeatures;      // backward
  void* feat_ws;
};
size_t feature_ws_stride(int P, int C);
cudaError_t launch_features_fwd(const FeatArgs& a, cudaStream_t s);  // raster_feat.cu
cudaError_t launch_features_bwd(const FeatArgs& a, cudaStream_t s);  // raster_feat.cu
// blend-weight statistics (raster_stats.cu): pixel_weights NULL, [H,W] or, with weights_per_frame, [F,H,W];
// out_sum / out_max [F,P], zeroed by the launch
struct StatsArgs : ForwardWS {
  const float* pixel_weights;
  int weights_per_frame;
  float *out_sum, *out_max;
};
cudaError_t launch_blend_stats(const StatsArgs& a, cudaStream_t s);  // raster_stats.cu
// per-Gaussian depth planes (gaussian_planes.cu): F <= PB_MAX_FRAMES cameras (viewmatrix [F,16] on the device, the
// tangents by value); inputs [P,.] or, with their DGR_PF_* bit in per_frame, [F,P,.]; planes / normals [F,P,3]
struct PlaneCams {
  float tanx[64], tany[64];  // PB_MAX_FRAMES
};
struct PlaneArgs {
  int F, P, W, H;
  const float *means3D, *scales, *rotations, *cov3D_precomp;  // scales + rotations, or cov3D_precomp
  float scale_modifier;
  int per_frame;
  const float* viewmatrix;
  PlaneCams cams;
  float *planes, *normals;                                          // forward
  const float *dL_dplanes, *dL_dnormals;                            // backward (either may be NULL)
  float *dL_dmeans3D, *dL_dscales, *dL_drotations, *dL_dcov3D;      // backward (NULL: not written)
};
cudaError_t launch_gaussian_planes_fwd(const PlaneArgs& a, cudaStream_t s);  // gaussian_planes.cu
cudaError_t launch_gaussian_planes_bwd(const PlaneArgs& a, cudaStream_t s);  // gaussian_planes.cu
// planar-depth maps (raster_planar.cu): planes [F,P,3]; maps [F,1,H,W]; planar_ws holds F per-frame workspaces
// planar_ws_stride(P, W, H) bytes apart (a plane accumulator per Gaussian and the median record per pixel)
struct PlanarArgs : ForwardWS {
  const float* planes;
  float *out_depth, *out_median;                     // forward
  const float *depth, *dL_ddepth, *dL_dmedian;       // backward (each gradient may be NULL)
  float* dL_dplanes;                                 // backward
  void* planar_ws;
};
size_t planar_ws_stride(int P, int W, int H);
cudaError_t launch_planar_fwd(const PlanarArgs& a, cudaStream_t s);  // raster_planar.cu
cudaError_t launch_planar_bwd(const PlanarArgs& a, cudaStream_t s);  // raster_planar.cu
// camera terms per (frame, Gaussian) and per partial: dL/dview[4k+j] (j < 3) at 3k+j, dL/dproj[4k+{0,1,3}] at
// 12+3k+{0,1,2}, dL/dcampos at 24..26
#define CAM_TERMS 27
inline size_t camera_ws_bytes(int F, int P) { return (size_t)F * ((P + 31) / 32) * CAM_TERMS * sizeof(float); }
// intrinsics terms (dL/dtan_fovx, dL/dtan_fovy), partials after the camera partials
#define INTR_TERMS 2
inline size_t intrinsics_ws_bytes(int F, int P) {
  return camera_ws_bytes(F, P) + (size_t)F * ((P + 31) / 32) * INTR_TERMS * sizeof(float);
}

// event pairs around kernels (see dgm_profile_enable in include/dgmesh_b200.h)
struct Profiler {
  int on = 0;  // 1: last duration per kernel id;  2: timeline (every launch since enable, any stream)
  cudaEvent_t ev[16][2] = {};
  bool used[16] = {};
  static const int TL_CAP = 512;
  cudaEvent_t tl_ev[TL_CAP][2] = {};
  int tl_id[TL_CAP] = {};
  int tl_n = 0;
  void begin(int k, cudaStream_t s) {
    if (on == 1) cudaEventRecord(ev[k][0], s);
    if (on == 2 && tl_n < TL_CAP) {
      if (!tl_ev[tl_n][0]) cudaEventCreate(&tl_ev[tl_n][0]), cudaEventCreate(&tl_ev[tl_n][1]);
      tl_id[tl_n] = k;
      cudaEventRecord(tl_ev[tl_n][0], s);
    }
  }
  void end(int k, cudaStream_t s) {
    if (on == 1) {
      cudaEventRecord(ev[k][1], s);
      used[k] = true;
    }
    if (on == 2 && tl_n < TL_CAP) cudaEventRecord(tl_ev[tl_n++][1], s);
  }
};
extern Profiler g_prof;

// A forward is launch_binning then launch_render (launch_forward: both on one stream).  A backward of F frames is
// launch_render_bwd (+ launch_median_grad) per frame, then launch_preprocess_bwd (+ launch_normal_grad_finish) once.
// launch_render_bwd picks the blend instance and calls launch_blend_bwd (raster_bwd_blend.cuh) through the entry of
// the file that compiles that instance: launch_render_bwd_{nrm,surf,abs}.
cudaError_t launch_forward(const FwdArgs& a, cudaStream_t s);
cudaError_t launch_binning(const FwdArgs& a, cudaStream_t s);
cudaError_t launch_render(const FwdArgs& a, cudaStream_t s);
cudaError_t launch_render_bwd(const BwdArgs& a, cudaStream_t s);
cudaError_t launch_preprocess_bwd(const BwdArgs& a, cudaStream_t s);
cudaError_t launch_render_bwd_nrm(const BwdArgs& a, cudaStream_t s);  // raster_nrm_bwd.cu
cudaError_t launch_normal_grad_finish(const BwdArgs& a, cudaStream_t s);  // raster_nrm_bwd.cu
cudaError_t launch_render_bwd_surf(const BwdArgs& a, cudaStream_t s);  // raster_surf_bwd.cu
cudaError_t launch_median_grad(const BwdArgs& a, cudaStream_t s);      // raster_surf_bwd.cu
cudaError_t launch_render_bwd_abs(const BwdArgs& a, cudaStream_t s);   // raster_abs_bwd.cu
cudaError_t launch_mark_visible(int P, const float* means3D, const float* view, const float* proj, uint8_t* present,
                                cudaStream_t s);
cudaError_t launch_export_state(int P, int W, int H, int64_t R_cap, const void* geom_ws, const void* binning_ws,
                                const void* img_ws, float* depths, float* means2D, float* cov3D, float* conic_opacity,
                                float* rgb, uint32_t* tiles_touched, uint8_t* clamped, uint64_t* point_list_keys,
                                uint32_t* point_list, uint32_t* ranges, float* final_T, uint32_t* n_contrib,
                                cudaStream_t s);

}  // namespace dgm
