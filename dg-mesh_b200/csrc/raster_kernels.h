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
  void *geom_ws, *binning_ws, *img_ws;
  int64_t R_cap;
  int32_t* status;
  // optional: host-mapped (pinned) copy of the status words, written by the tile scan, and the
  // depth range of an earlier frame (hint_hi > hint_lo enables the fused preprocess + count)
  int32_t* status_host;
  float hint_lo, hint_hi;
  int hint_max_tile;         // longest per-tile list of an earlier frame (status word 2), 0: unknown
  cudaEvent_t status_event;  // recorded right after the tile scan (may be null)
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
  float *dL_dmean2D, *dL_dconic, *dL_dopacity, *dL_dcolor, *dL_dmean3D, *dL_dcov3D, *dL_dsh, *dL_dscale, *dL_drot;
  // launch_preprocess_bwd covers F frames (1 <= F <= PB_MAX_FRAMES) in one launch: frame f reads the camera at
  // index f (viewmatrix + 16 f, ..., tan_fovx[f]), its workspace at geom_ws + f * geom_stride, radii + f * P,
  // and the slab f of each input whose DGR_PF_* bit is set in per_frame.  dL_dmean2D (and dL_dconic) are
  // [F,P,.]; every other gradient is [F,P,.] when its bit is set and the sum over the frames otherwise.
  // launch_render_bwd reads one frame: frame 0 of the above.
  int F, per_frame;
  size_t geom_stride;
};
#define PB_MAX_FRAMES 64

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

cudaError_t launch_forward(const FwdArgs& a, cudaStream_t s);
cudaError_t launch_backward(const BwdArgs& a, cudaStream_t s);
cudaError_t launch_binning(const FwdArgs& a, cudaStream_t s);
cudaError_t launch_render(const FwdArgs& a, cudaStream_t s);
cudaError_t launch_render_bwd(const BwdArgs& a, cudaStream_t s);
cudaError_t launch_preprocess_bwd(const BwdArgs& a, cudaStream_t s);
cudaError_t launch_mark_visible(int P, const float* means3D, const float* view, const float* proj, uint8_t* present,
                                cudaStream_t s);
cudaError_t launch_export_state(int P, int W, int H, int64_t R_cap, const void* geom_ws, const void* binning_ws,
                                const void* img_ws, float* depths, float* means2D, float* cov3D, float* conic_opacity,
                                float* rgb, uint32_t* tiles_touched, uint8_t* clamped, uint64_t* point_list_keys,
                                uint32_t* point_list, uint32_t* ranges, float* final_T, uint32_t* n_contrib,
                                cudaStream_t s);

}  // namespace dgm
