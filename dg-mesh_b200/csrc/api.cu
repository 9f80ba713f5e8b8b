// api.cu -- the C-ABI of libdgmesh_b200.so (see include/dgmesh_b200.h).
#include "../../include/dgmesh_b200.h"
#include "common.cuh"
#include "raster_kernels.h"
#include "knn_kernels.h"
#include "dpsr_kernels.h"
#include "mc_kernels.h"
#include "loss_kernels.h"
#include "mlp_kernels.h"
#include "densify_kernels.h"
#include "meshrast_kernels.h"
#include "nvls_kernels.h"

#include <string.h>
#include <stdlib.h>
#include <mutex>
#include <map>

namespace {
thread_local char g_last_error[256] = "";
int check(cudaError_t e) {
  if (e == cudaSuccess) return DGM_OK;
  strncpy(g_last_error, cudaGetErrorString(e), sizeof(g_last_error) - 1);
  return DGM_E_LAUNCH;
}
int bad(const char* msg) {
  strncpy(g_last_error, msg, sizeof(g_last_error) - 1);
  return DGM_E_BADARG;
}
}  // namespace

namespace dgm {
Profiler g_prof;
// programmatic dependent launch between the rasterizer's kernels: DGMESH_B200_PDL=1 turns it on.
// Off by default: early-resident dependents hold CTA slots / shared memory while the predecessor's
// tail is still running, and the launch gaps it could hide are a small part of a frame.
int g_pdl = [] {
  const char* e = getenv("DGMESH_B200_PDL");
  return (e && e[0] == '1') ? 1 : 0;
}();
// ---- state export (parity tests): rebuild the reference-visible views from the
// private workspaces.  point_list_keys is reconstructed as (tile << 32 | depth bits),
// the key the reference sorts on (rasterizer_impl.cu:98-106).
__global__ void export_keys_kernel(int T, const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list,
                                   const float* __restrict__ depths, uint64_t* __restrict__ keys) {
  const int t = blockIdx.x;
  if (t >= T) return;
  const uint2 r = ranges[t];
  for (uint32_t i = r.x + threadIdx.x; i < r.y; i += blockDim.x)
    keys[i] = ((uint64_t)t << 32) | (uint64_t)__float_as_uint(depths[point_list[i]]);
}

cudaError_t launch_export_state(int P, int W, int H, int64_t R_cap, const void* geom_ws, const void* binning_ws,
                                const void* img_ws, float* depths, float* means2D, float* cov3D, float* conic_opacity,
                                float* rgb, uint32_t* tiles_touched, uint8_t* clamped, uint64_t* point_list_keys,
                                uint32_t* point_list, uint32_t* ranges, float* final_T, uint32_t* n_contrib,
                                cudaStream_t s) {
  const unsigned gx = (W + TILE_X - 1) / TILE_X, gy = (H + TILE_Y - 1) / TILE_Y;
  const int T = gx * gy;
  const size_t npix = (size_t)W * H;
  GeomWS g = GeomWS::from((char*)geom_ws, P);
  ImgWS im = ImgWS::from((char*)img_ws, npix, T);
  BinWS b = BinWS::from((char*)binning_ws, (size_t)R_cap);
  const cudaMemcpyKind k = cudaMemcpyDeviceToDevice;
  if (depths) cudaMemcpyAsync(depths, g.depths, sizeof(float) * P, k, s);
  if (means2D) cudaMemcpyAsync(means2D, g.means2D, sizeof(float2) * P, k, s);
  if (cov3D) cudaMemcpyAsync(cov3D, g.cov3D, sizeof(float) * 6 * P, k, s);
  if (conic_opacity) cudaMemcpyAsync(conic_opacity, g.conic_opacity, sizeof(float4) * P, k, s);
  if (rgb) cudaMemcpyAsync(rgb, g.rgb, sizeof(float) * 3 * P, k, s);
  if (tiles_touched) cudaMemcpyAsync(tiles_touched, g.tiles_touched, sizeof(uint32_t) * P, k, s);
  if (clamped) cudaMemcpyAsync(clamped, g.clamped, 3 * (size_t)P, k, s);
  if (ranges) cudaMemcpyAsync(ranges, im.ranges, sizeof(uint2) * T, k, s);
  if (final_T) cudaMemcpyAsync(final_T, im.final_T, sizeof(float) * npix, k, s);
  if (n_contrib) cudaMemcpyAsync(n_contrib, im.n_contrib, sizeof(uint32_t) * npix, k, s);
  // the caller sizes point_list / keys by the R it read from the status block (R <= R_cap)
  if (point_list_keys) export_keys_kernel<<<T, 128, 0, s>>>(T, im.ranges, b.point_list, g.depths, point_list_keys);
  if (point_list) {
    // copy only the populated prefix: R is the end of the last non-empty range; copy R_cap is safe too
    cudaMemcpyAsync(point_list, b.point_list, sizeof(uint32_t) * (size_t)R_cap, k, s);
  }
  return cudaGetLastError();
}
}  // namespace dgm

extern "C" {

const char* dgm_version(void) { return "dgmesh_b200 0.1 sm_90a"; }
const char* dgm_last_error(void) { return g_last_error; }

int dgr_workspace_sizes(int P, int W, int H, int64_t R_cap, size_t* geom_bytes, size_t* binning_bytes,
                        size_t* img_bytes) {
  if (P < 0 || W <= 0 || H <= 0 || R_cap < 0) return bad("dgr_workspace_sizes: negative size");
  const unsigned gx = (W + TILE_X - 1) / TILE_X, gy = (H + TILE_Y - 1) / TILE_Y;
  size_t gb, bb, ib;
  dgm::GeomWS::from(nullptr, (size_t)P, &gb);
  dgm::BinWS::from(nullptr, (size_t)R_cap, &bb);
  dgm::ImgWS::from(nullptr, (size_t)W * H, (size_t)gx * gy, &ib);
  if (geom_bytes) *geom_bytes = gb;
  if (binning_bytes) *binning_bytes = bb;
  if (img_bytes) *img_bytes = ib;
  return DGM_OK;
}

int dgr_forward(int P, int D, int M, const float* background, int W, int H, const float* means3D, const float* shs,
                const float* colors_precomp, const float* opacities, const float* scales, float scale_modifier,
                const float* rotations, const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                const float* cam_pos, float tan_fovx, float tan_fovy, int prefiltered, float* out_color, int* radii,
                void* geom_ws, size_t geom_bytes, void* binning_ws, size_t binning_bytes, int64_t R_cap, void* img_ws,
                size_t img_bytes, int32_t* status, int32_t* status_host, void* status_event, float depth_hint_lo,
                float depth_hint_hi, int max_tile_hint, void* stream) {
  if (P < 0 || W <= 0 || H <= 0 || R_cap < 0) return bad("dgr_forward: negative size");
  if (!background || !viewmatrix || !projmatrix || !cam_pos || !out_color || !status)
    return bad("dgr_forward: null required pointer");
  if (P > 0) {
    if (!means3D || !opacities) return bad("dgr_forward: means3D / opacities missing");
    if ((shs == nullptr) == (colors_precomp == nullptr)) return bad("dgr_forward: exactly one of shs / colors_precomp");
    if (((scales == nullptr) || (rotations == nullptr)) == (cov3D_precomp == nullptr))
      return bad("dgr_forward: exactly one of scales+rotations / cov3D_precomp");
    if (shs && (M <= 0 || M > 16 || (D + 1) * (D + 1) > M || D < 0 || D > 3))
      return bad("dgr_forward: SH degree / coefficient count");
  }
  if (P == 0) {
    // the reference skips the whole pipeline and returns the zero-initialised image
    // (rasterize_points.cu:64,80: torch::full(0.0) and `if (P != 0)`)
    cudaMemsetAsync(out_color, 0, sizeof(float) * 3 * (size_t)W * H, (cudaStream_t)stream);
    cudaMemsetAsync(status, 0, sizeof(int32_t) * DGR_STATUS_WORDS, (cudaStream_t)stream);
    if (status_host) memset(status_host, 0, sizeof(int32_t) * DGR_STATUS_WORDS);
    if (status_event) cudaEventRecord((cudaEvent_t)status_event, (cudaStream_t)stream);
    return check(cudaGetLastError());
  }
  size_t gb, bb, ib;
  dgr_workspace_sizes(P, W, H, R_cap, &gb, &bb, &ib);
  if (geom_bytes < gb || binning_bytes < bb || img_bytes < ib || !geom_ws || !binning_ws || !img_ws) {
    strncpy(g_last_error, "dgr_forward: workspace too small", sizeof(g_last_error) - 1);
    return DGM_E_WORKSPACE;
  }
  dgm::FwdArgs a;
  a.P = P; a.D = D; a.M = M; a.background = background; a.W = W; a.H = H;
  a.means3D = means3D; a.shs = shs; a.colors_precomp = colors_precomp; a.opacities = opacities;
  a.scales = scales; a.scale_modifier = scale_modifier; a.rotations = rotations; a.cov3D_precomp = cov3D_precomp;
  a.viewmatrix = viewmatrix; a.projmatrix = projmatrix; a.cam_pos = cam_pos;
  a.tan_fovx = tan_fovx; a.tan_fovy = tan_fovy; a.prefiltered = prefiltered;
  a.out_color = out_color; a.radii = radii;
  a.geom_ws = geom_ws; a.binning_ws = binning_ws; a.img_ws = img_ws; a.R_cap = R_cap; a.status = status;
  a.status_host = status_host; a.status_event = (cudaEvent_t)status_event;
  a.hint_lo = depth_hint_lo; a.hint_hi = depth_hint_hi; a.hint_max_tile = max_tile_hint;
  return check(dgm::launch_forward(a, (cudaStream_t)stream));
}

int dgr_backward(int P, int D, int M, const float* background, int W, int H, const float* means3D, const float* shs,
                 const float* colors_precomp, const float* scales, float scale_modifier, const float* rotations,
                 const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                 float tan_fovx, float tan_fovy, const int* radii, void* geom_ws, void* binning_ws, int64_t R_cap,
                 void* img_ws, const float* dL_dpix, float* dL_dmean2D, float* dL_dconic, float* dL_dopacity,
                 float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale,
                 float* dL_drot, void* stream) {
  if (P < 0 || W <= 0 || H <= 0 || R_cap < 0) return bad("dgr_backward: negative size");
  if (P == 0) return DGM_OK;
  if (!background || !means3D || !viewmatrix || !projmatrix || !cam_pos || !geom_ws || !binning_ws || !img_ws ||
      !dL_dpix || !dL_dmean2D || !dL_dopacity || !dL_dcolor || !dL_dmean3D || !dL_dcov3D || !dL_dscale ||
      !dL_drot)
    return bad("dgr_backward: null required pointer");
  if (shs && !dL_dsh) return bad("dgr_backward: dL_dsh missing");
  dgm::BwdArgs a;
  a.P = P; a.D = D; a.M = M; a.background = background; a.W = W; a.H = H;
  a.means3D = means3D; a.shs = shs; a.colors_precomp = colors_precomp; a.scales = scales;
  a.scale_modifier = scale_modifier; a.rotations = rotations; a.cov3D_precomp = cov3D_precomp;
  a.viewmatrix = viewmatrix; a.projmatrix = projmatrix; a.cam_pos = cam_pos;
  a.tan_fovx = &tan_fovx; a.tan_fovy = &tan_fovy; a.radii = radii;
  a.geom_ws = geom_ws; a.binning_ws = binning_ws; a.img_ws = img_ws; a.R_cap = R_cap;
  a.dL_dpix = dL_dpix; a.dL_dmean2D = dL_dmean2D; a.dL_dconic = dL_dconic; a.dL_dopacity = dL_dopacity;
  a.dL_dcolor = dL_dcolor; a.dL_dmean3D = dL_dmean3D; a.dL_dcov3D = dL_dcov3D; a.dL_dsh = dL_dsh;
  a.dL_dscale = dL_dscale; a.dL_drot = dL_drot;
  a.F = 1; a.per_frame = 0; a.geom_stride = 0;
  return check(dgm::launch_backward(a, (cudaStream_t)stream));
}

namespace {
// Internal streams for the frame batches (created once per process).
//   hi[]  high priority: the short, latency-bound kernels (preprocess / binning / sort)
//   lo[]  low priority : the blend kernels, each of which fills the GPU on its own; two streams,
//         alternating frames, so the next kernel's CTAs fill the SMs while the previous one's tail drains
// A frame's binning chain runs on hi[f % NH] and its blend kernel on lo behind an event.  The block
// scheduler serves pending high-priority CTAs first, so the binning chains of the NEXT frames slip
// through while the blend kernel of the current frame is running (they are latency-bound and cost
// the issue-bound blend kernel almost nothing) instead of queueing behind its 2 500 CTAs.
struct BatchStreams {
  static const int NH = 4;
  cudaStream_t hi[NH] = {}, lo[2] = {};
  cudaEvent_t fork = nullptr, done_hi[NH] = {}, done_lo[2] = {}, ready[NH] = {};
  bool ok = false;
  std::mutex mu;  // one batch call at a time per device (the events above are shared)
  bool init() {
    if (ok) return true;
    int least = 0, greatest = 0;
    if (cudaDeviceGetStreamPriorityRange(&least, &greatest) != cudaSuccess) return false;
    for (int i = 0; i < NH; ++i) {
      if (cudaStreamCreateWithPriority(&hi[i], cudaStreamNonBlocking, greatest) != cudaSuccess) return false;
      if (cudaEventCreateWithFlags(&done_hi[i], cudaEventDisableTiming) != cudaSuccess) return false;
      if (cudaEventCreateWithFlags(&ready[i], cudaEventDisableTiming) != cudaSuccess) return false;
    }
    if (cudaEventCreateWithFlags(&fork, cudaEventDisableTiming) != cudaSuccess) return false;
    for (int i = 0; i < 2; ++i) {
      if (cudaStreamCreateWithPriority(&lo[i], cudaStreamNonBlocking, least) != cudaSuccess) return false;
      if (cudaEventCreateWithFlags(&done_lo[i], cudaEventDisableTiming) != cudaSuccess) return false;
    }
    ok = true;
    return true;
  }
};
// one set per device, created on first use
std::mutex g_bs_mu;
std::map<int, BatchStreams*> g_bs_map;
BatchStreams* batch_streams() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  std::lock_guard<std::mutex> lk(g_bs_mu);
  BatchStreams*& p = g_bs_map[dev];
  if (!p) p = new BatchStreams();
  return p->init() ? p : nullptr;
}

dgm::FwdArgs fwd_args(int P, int D, int M, const float* background, int W, int H, const float* means3D,
                      const float* shs, const float* colors_precomp, const float* opacities, const float* scales,
                      float scale_modifier, const float* rotations, const float* cov3D_precomp,
                      const float* viewmatrix, const float* projmatrix, const float* cam_pos, float tan_fovx,
                      float tan_fovy, int prefiltered, float* out_color, int* radii, void* geom_ws, void* binning_ws,
                      int64_t R_cap, void* img_ws, int32_t* status, int32_t* status_host, float hint_lo,
                      float hint_hi, int hint_max_tile) {
  dgm::FwdArgs a;
  a.P = P; a.D = D; a.M = M; a.background = background; a.W = W; a.H = H;
  a.means3D = means3D; a.shs = shs; a.colors_precomp = colors_precomp; a.opacities = opacities;
  a.scales = scales; a.scale_modifier = scale_modifier; a.rotations = rotations; a.cov3D_precomp = cov3D_precomp;
  a.viewmatrix = viewmatrix; a.projmatrix = projmatrix; a.cam_pos = cam_pos;
  a.tan_fovx = tan_fovx; a.tan_fovy = tan_fovy; a.prefiltered = prefiltered;
  a.out_color = out_color; a.radii = radii;
  a.geom_ws = geom_ws; a.binning_ws = binning_ws; a.img_ws = img_ws; a.R_cap = R_cap; a.status = status;
  a.status_host = status_host; a.status_event = nullptr; a.hint_lo = hint_lo; a.hint_hi = hint_hi;
  a.hint_max_tile = hint_max_tile;
  return a;
}
}  // namespace

int dgr_forward_batch(int F, int P, int D, int M, const float* background, int W, int H, const float* means3D,
                      const float* shs, const float* colors_precomp, const float* opacities, const float* scales,
                      float scale_modifier, const float* rotations, const float* cov3D_precomp, int per_frame,
                      const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                      const float* tan_fovx_host, const float* tan_fovy_host, int prefiltered, float* out_color,
                      int* radii, void* geom_ws, size_t geom_stride, void* binning_ws, size_t binning_stride,
                      int64_t R_cap, void* img_ws, size_t img_stride, int32_t* status, int32_t* status_host,
                      void* status_event, float depth_hint_lo, float depth_hint_hi, int max_tile_hint, int n_streams,
                      void* stream) {
  if (F <= 0 || !tan_fovx_host || !tan_fovy_host || !viewmatrices || !projmatrices || !cam_poses)
    return bad("dgr_forward_batch: bad argument");
  size_t gb, bb, ib;
  if (dgr_workspace_sizes(P, W, H, R_cap, &gb, &bb, &ib) != DGM_OK) return DGM_E_BADARG;
  if (geom_stride < gb || binning_stride < bb || img_stride < ib || (geom_stride | binning_stride | img_stride) & 127) {
    strncpy(g_last_error, "dgr_forward_batch: workspace stride too small / unaligned", sizeof(g_last_error) - 1);
    return DGM_E_WORKSPACE;
  }
  cudaStream_t main_s = (cudaStream_t)stream;
  const bool multi = n_streams > 1 && F > 1 && P > 0;
  const int NH = multi ? (n_streams > BatchStreams::NH ? BatchStreams::NH : n_streams) : 0;
  // per-frame inputs (bit set in per_frame) advance by one [P, .] slab per frame
  auto pf = [&](const float* p, int bit, size_t width, int f) {
    return (p && (per_frame & bit)) ? p + (size_t)f * P * width : p;
  };
  const size_t cw = shs ? (size_t)M * 3 : 3;
  if (!multi) {
    int rc = DGM_OK;
    for (int f = 0; f < F && rc == DGM_OK; ++f)
      rc = dgr_forward(P, D, M, background, W, H, pf(means3D, DGR_PF_MEANS, 3, f), pf(shs, DGR_PF_COLOR, cw, f),
                       pf(colors_precomp, DGR_PF_COLOR, 3, f), pf(opacities, DGR_PF_OPAC, 1, f),
                       pf(scales, DGR_PF_SCALES, 3, f), scale_modifier, pf(rotations, DGR_PF_ROTS, 4, f),
                       pf(cov3D_precomp, DGR_PF_COV, 6, f), viewmatrices + 16 * f, projmatrices + 16 * f,
                       cam_poses + 3 * f, tan_fovx_host[f], tan_fovy_host[f], prefiltered,
                       out_color + (size_t)f * 3 * W * H, radii ? radii + (size_t)f * P : nullptr,
                       (char*)geom_ws + f * geom_stride, geom_stride, (char*)binning_ws + f * binning_stride,
                       binning_stride, R_cap, (char*)img_ws + f * img_stride, img_stride,
                       status + f * DGR_STATUS_WORDS, status_host ? status_host + f * DGR_STATUS_WORDS : nullptr,
                       (f == F - 1) ? status_event : nullptr, depth_hint_lo, depth_hint_hi, max_tile_hint, main_s);
    return rc;
  }
  if (!background || !out_color || !status || !means3D || !opacities) return bad("dgr_forward_batch: null required pointer");
  if ((shs == nullptr) == (colors_precomp == nullptr)) return bad("dgr_forward_batch: exactly one of shs / colors_precomp");
  if (((scales == nullptr) || (rotations == nullptr)) == (cov3D_precomp == nullptr))
    return bad("dgr_forward_batch: exactly one of scales+rotations / cov3D_precomp");
  if (shs && (M <= 0 || M > 16 || (D + 1) * (D + 1) > M || D < 0 || D > 3))
    return bad("dgr_forward_batch: SH degree / coefficient count");
  BatchStreams* bs = batch_streams();
  if (!bs) return check(cudaGetLastError());
  std::lock_guard<std::mutex> lk(bs->mu);
  cudaEventRecord(bs->fork, main_s);
  for (int i = 0; i < NH; ++i) cudaStreamWaitEvent(bs->hi[i], bs->fork, 0);
  for (int i = 0; i < 2; ++i) cudaStreamWaitEvent(bs->lo[i], bs->fork, 0);
  cudaError_t e = cudaSuccess;
  for (int f = 0; f < F && e == cudaSuccess; ++f) {
    const int i = f % NH;
    cudaStream_t lo = bs->lo[f & 1];
    const dgm::FwdArgs a = fwd_args(
        P, D, M, background, W, H, pf(means3D, DGR_PF_MEANS, 3, f), pf(shs, DGR_PF_COLOR, cw, f),
        pf(colors_precomp, DGR_PF_COLOR, 3, f), pf(opacities, DGR_PF_OPAC, 1, f), pf(scales, DGR_PF_SCALES, 3, f),
        scale_modifier, pf(rotations, DGR_PF_ROTS, 4, f), pf(cov3D_precomp, DGR_PF_COV, 6, f), viewmatrices + 16 * f,
        projmatrices + 16 * f, cam_poses + 3 * f, tan_fovx_host[f], tan_fovy_host[f], prefiltered,
        out_color + (size_t)f * 3 * W * H, radii ? radii + (size_t)f * P : nullptr, (char*)geom_ws + f * geom_stride,
        (char*)binning_ws + f * binning_stride, R_cap, (char*)img_ws + f * img_stride, status + f * DGR_STATUS_WORDS,
        status_host ? status_host + f * DGR_STATUS_WORDS : nullptr, depth_hint_lo, depth_hint_hi, max_tile_hint);
    e = dgm::launch_binning(a, bs->hi[i]);
    cudaEventRecord(bs->ready[i], bs->hi[i]);
    cudaStreamWaitEvent(lo, bs->ready[i], 0);
    if (e == cudaSuccess) e = dgm::launch_render(a, lo);
  }
  // the binning chains finish long before the blend kernels: the caller's status event fires then
  for (int i = 0; i < NH; ++i) {
    cudaEventRecord(bs->done_hi[i], bs->hi[i]);
    cudaStreamWaitEvent(main_s, bs->done_hi[i], 0);
  }
  if (status_event) cudaEventRecord((cudaEvent_t)status_event, main_s);
  for (int i = 0; i < 2; ++i) {
    cudaEventRecord(bs->done_lo[i], bs->lo[i]);
    cudaStreamWaitEvent(main_s, bs->done_lo[i], 0);
  }
  return check(e != cudaSuccess ? e : cudaGetLastError());
}

int dgr_backward_batch(int F, int P, int D, int M, const float* background, int W, int H, const float* means3D,
                       const float* shs, const float* colors_precomp, const float* scales, float scale_modifier,
                       const float* rotations, const float* cov3D_precomp, int per_frame, const float* viewmatrices,
                       const float* projmatrices, const float* cam_poses, const float* tan_fovx_host,
                       const float* tan_fovy_host, const int* radii, void* geom_ws, size_t geom_stride,
                       void* binning_ws, size_t binning_stride, int64_t R_cap, void* img_ws, size_t img_stride,
                       const float* dL_dpix, float* dL_dmean2D, float* dL_dopacity, float* dL_dcolor,
                       float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot,
                       int n_streams, void* stream) {
  if (F <= 0 || P < 0 || W <= 0 || H <= 0 || R_cap < 0) return bad("dgr_backward_batch: bad size");
  if (F > PB_MAX_FRAMES) return bad("dgr_backward_batch: more than 64 frames");
  if (P == 0) return DGM_OK;
  if (!background || !means3D || !viewmatrices || !projmatrices || !cam_poses || !tan_fovx_host || !tan_fovy_host ||
      !geom_ws || !binning_ws || !img_ws || !dL_dpix || !dL_dmean2D || !dL_dopacity || (!shs && !dL_dcolor) ||
      !dL_dmean3D || (cov3D_precomp && !dL_dcov3D) || !dL_dscale || !dL_drot || (shs && !dL_dsh))
    return bad("dgr_backward_batch: null required pointer");
  // the render_bwd kernels alternate two low-priority streams (the next one's CTAs fill the SMs while the
  // previous one's tail drains); one per-Gaussian kernel for all frames follows once both have finished
  const bool multi = n_streams > 1 && F > 1;
  cudaStream_t main_s = (cudaStream_t)stream;
  BatchStreams* bs = nullptr;
  std::unique_lock<std::mutex> lk;
  if (multi) {
    bs = batch_streams();
    if (!bs) return check(cudaGetLastError());
    lk = std::unique_lock<std::mutex>(bs->mu);
    cudaEventRecord(bs->fork, main_s);
    for (int i = 0; i < 2; ++i) cudaStreamWaitEvent(bs->lo[i], bs->fork, 0);
  }
  dgm::BwdArgs a;
  a.P = P; a.D = D; a.M = M; a.background = background; a.W = W; a.H = H;
  a.means3D = means3D; a.shs = shs; a.colors_precomp = colors_precomp; a.scales = scales;
  a.scale_modifier = scale_modifier; a.rotations = rotations; a.cov3D_precomp = cov3D_precomp;
  a.viewmatrix = viewmatrices; a.projmatrix = projmatrices; a.cam_pos = cam_poses;
  a.tan_fovx = tan_fovx_host; a.tan_fovy = tan_fovy_host; a.radii = radii;
  a.geom_ws = geom_ws; a.binning_ws = binning_ws; a.img_ws = img_ws; a.R_cap = R_cap; a.dL_dpix = dL_dpix;
  a.dL_dmean2D = dL_dmean2D; a.dL_dconic = nullptr; a.dL_dopacity = dL_dopacity; a.dL_dcolor = dL_dcolor;
  a.dL_dmean3D = dL_dmean3D; a.dL_dcov3D = dL_dcov3D; a.dL_dsh = dL_dsh;
  a.dL_dscale = dL_dscale; a.dL_drot = dL_drot;
  a.F = F; a.per_frame = per_frame; a.geom_stride = geom_stride;
  cudaError_t e = cudaSuccess;
  for (int f = 0; f < F && e == cudaSuccess; ++f) {
    dgm::BwdArgs af = a;  // launch_render_bwd reads frame 0 of its arguments
    af.geom_ws = (char*)geom_ws + f * geom_stride; af.binning_ws = (char*)binning_ws + f * binning_stride;
    af.img_ws = (char*)img_ws + f * img_stride; af.dL_dpix = dL_dpix + (size_t)f * 3 * W * H;
    e = dgm::launch_render_bwd(af, multi ? bs->lo[f & 1] : main_s);
  }
  if (multi) {
    for (int i = 0; i < 2; ++i) {
      cudaEventRecord(bs->done_lo[i], bs->lo[i]);
      cudaStreamWaitEvent(main_s, bs->done_lo[i], 0);
    }
  }
  if (e == cudaSuccess) e = dgm::launch_preprocess_bwd(a, main_s);
  return check(e != cudaSuccess ? e : cudaGetLastError());
}

int dgr_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix, uint8_t* present,
                     void* stream) {
  if (P < 0) return bad("dgr_mark_visible: negative size");
  if (P > 0 && (!means3D || !viewmatrix || !projmatrix || !present)) return bad("dgr_mark_visible: null pointer");
  return check(dgm::launch_mark_visible(P, means3D, viewmatrix, projmatrix, present, (cudaStream_t)stream));
}

int dgr_export_state(int P, int W, int H, int64_t R_cap, const void* geom_ws, const void* binning_ws,
                     const void* img_ws, float* depths, float* means2D, float* cov3D, float* conic_opacity, float* rgb,
                     uint32_t* tiles_touched, uint8_t* clamped, uint64_t* point_list_keys, uint32_t* point_list,
                     uint32_t* ranges, float* final_T, uint32_t* n_contrib, void* stream) {
  if (P < 0 || W <= 0 || H <= 0 || R_cap < 0 || !geom_ws || !binning_ws || !img_ws)
    return bad("dgr_export_state: bad argument");
  return check(dgm::launch_export_state(P, W, H, R_cap, geom_ws, binning_ws, img_ws, depths, means2D, cov3D,
                                        conic_opacity, rgb, tiles_touched, clamped, point_list_keys, point_list,
                                        ranges, final_T, n_contrib, (cudaStream_t)stream));
}

int dgk_workspace_size(int P, size_t* bytes) {
  if (P < 0 || !bytes) return bad("dgk_workspace_size: bad argument");
  dgm::KnnWS::from(nullptr, (size_t)P, P ? dgm::knn_cub_bytes(P) : 0, bytes);
  return DGM_OK;
}

int dgk_dist2(int P, const float* points, float* mean_dist2, void* ws, size_t ws_bytes, void* stream) {
  if (P < 0) return bad("dgk_dist2: negative size");
  if (P == 0) return DGM_OK;
  if (!points || !mean_dist2 || !ws) return bad("dgk_dist2: null pointer");
  size_t need;
  dgk_workspace_size(P, &need);
  if (ws_bytes < need) {
    strncpy(g_last_error, "dgk_dist2: workspace too small", sizeof(g_last_error) - 1);
    return DGM_E_WORKSPACE;
  }
  return check(dgm::launch_knn(P, points, mean_dist2, ws, (cudaStream_t)stream));
}

int dgk_nearest(int Q, const float* queries, int R, const float* refs, float* dist2, int64_t* index, void* stream) {
  if (Q < 0 || R < 1) return bad("dgk_nearest: Q >= 0 and R >= 1 required");
  if (Q == 0) return DGM_OK;
  if (!queries || !refs || !dist2 || !index) return bad("dgk_nearest: null pointer");
  return check(dgm::launch_nearest(Q, queries, R, refs, dist2, (long long*)index, (cudaStream_t)stream));
}

int dgp_plan_create(int G, void** plan, size_t* ws_bytes) {
  if (G < 4 || (G & 1) || !plan) return bad("dgp_plan_create: G must be even and >= 4");
  size_t work = 0;
  if (dgm::dpsr_plan_create(G, plan, &work) != 0) {
    strncpy(g_last_error, "dgp_plan_create: cuFFT plan creation failed", sizeof(g_last_error) - 1);
    return DGM_E_LAUNCH;
  }
  if (ws_bytes) dgm::DpsrWS::from(nullptr, G, work, ws_bytes);
  return DGM_OK;
}

int dgp_plan_destroy(void* plan) {
  dgm::dpsr_plan_destroy(plan);
  return DGM_OK;
}

static int dgp_check(void* plan, size_t ws_bytes, void* ws) {
  if (!plan || !ws) return bad("dpsr: null plan / workspace");
  size_t need;
  dgm::DpsrWS::from(nullptr, dgm::dpsr_plan_res(plan), dgm::dpsr_plan_work(plan), &need);
  if (ws_bytes < need) {
    strncpy(g_last_error, "dpsr: workspace too small", sizeof(g_last_error) - 1);
    return DGM_E_WORKSPACE;
  }
  return DGM_OK;
}

int dgp_forward(void* plan, int N, double sig, const float* V, const float* Nrm, int mode, const float* thres,
                float* out, void* ws, size_t ws_bytes, void* stream) {
  int rc = dgp_check(plan, ws_bytes, ws);
  if (rc != DGM_OK) return rc;
  if (N < 0 || !out || (N > 0 && (!V || !Nrm)) || (mode && !thres)) return bad("dgp_forward: bad argument");
  return check(dgm::launch_dpsr_forward(plan, N, sig, V, Nrm, mode, thres, out, ws, (cudaStream_t)stream));
}

int dgp_backward(void* plan, int N, const float* V, const float* Nrm, int mode, const float* dL_dout, float* dV,
                 float* dN, float* dthres, void* ws, size_t ws_bytes, void* stream) {
  int rc = dgp_check(plan, ws_bytes, ws);
  if (rc != DGM_OK) return rc;
  if (N < 0 || !dL_dout || (N > 0 && (!V || !Nrm || !dV || !dN))) return bad("dgp_backward: bad argument");
  return check(dgm::launch_dpsr_backward(plan, N, V, Nrm, mode, dL_dout, dV, dN, dthres, ws, (cudaStream_t)stream));
}

int dgmc_workspace_size(int G, size_t* bytes) {
  if (G < 2 || G > 800 || !bytes) return bad("dgmc_workspace_size: bad argument (2 <= G <= 800)");
  dgm::McWS::from(nullptr, G, bytes);
  return DGM_OK;
}

static int dgmc_check(int G, const float* phi, void* ws, size_t ws_bytes) {
  if (G < 2 || G > 800 || !phi || !ws) return bad("marching cubes: bad argument (2 <= G <= 800)");
  size_t need;
  dgm::McWS::from(nullptr, G, &need);
  if (ws_bytes < need) {
    strncpy(g_last_error, "marching cubes: workspace too small", sizeof(g_last_error) - 1);
    return DGM_E_WORKSPACE;
  }
  return DGM_OK;
}

int dgmc_count(int G, const float* phi, float iso, void* ws, size_t ws_bytes, int32_t* totals, int32_t* totals_host,
               void* totals_event, void* stream) {
  int rc = dgmc_check(G, phi, ws, ws_bytes);
  if (rc != DGM_OK) return rc;
  if (!totals) return bad("dgmc_count: null totals");
  return check(dgm::launch_mc_count(G, phi, iso, ws, totals, totals_host, (cudaEvent_t)totals_event,
                                    (cudaStream_t)stream));
}

int dgmc_emit(int G, const float* phi, float iso, void* ws, size_t ws_bytes, float* verts, int64_t V_cap,
              int32_t* faces, int64_t F_cap, void* stream) {
  int rc = dgmc_check(G, phi, ws, ws_bytes);
  if (rc != DGM_OK) return rc;
  if (V_cap < 0 || F_cap < 0 || (V_cap > 0 && !verts) || (F_cap > 0 && !faces)) return bad("dgmc_emit: bad argument");
  return check(dgm::launch_mc_emit(G, phi, iso, ws, verts, V_cap, faces, F_cap, (cudaStream_t)stream));
}

int dgmc_backward(int G, int V, const float* phi, float iso, void* ws, size_t ws_bytes, const float* dL_dverts,
                  float* dL_dphi, void* stream) {
  int rc = dgmc_check(G, phi, ws, ws_bytes);
  if (rc != DGM_OK) return rc;
  if (!dL_dphi || V < 0 || (V > 0 && !dL_dverts)) return bad("dgmc_backward: bad argument");
  return check(dgm::launch_mc_backward(G, V, phi, iso, ws, dL_dverts, dL_dphi, (cudaStream_t)stream));
}

int dgl_gemm_ws_bytes(int M, int N, int K, size_t* bytes) {
  if (M <= 0 || N <= 0 || K <= 0 || !bytes) return bad("dgl_gemm_ws_bytes: bad argument");
  *bytes = dgm::gemm_test_ws_bytes(M, N > 256 ? N : 256, K);
  return DGM_OK;
}

int dgl_gemm_bf16(int M, int N, int K, const void* A, int lda, const void* B, int ldb, const float* bias, int relu,
                  float* C, int ldc, void* ws, size_t ws_bytes, void* stream) {
  if (M <= 0 || N <= 0 || N > 256 || K <= 0 || !A || !B || !C || !ws) return bad("dgl_gemm_bf16: bad argument");
  if (ldc < (N + 3) / 4 * 4 || (ldc & 3)) return bad("dgl_gemm_bf16: ldc must be a multiple of 4 and >= N rounded up to 4");
  if (ws_bytes < dgm::gemm_test_ws_bytes(M, 256, K)) {
    strncpy(g_last_error, "dgl_gemm_bf16: workspace too small", sizeof(g_last_error) - 1);
    return DGM_E_WORKSPACE;
  }
  return check(dgm::launch_gemm_test(M, N, K, A, lda, B, ldb, bias, relu, C, ldc, ws, (cudaStream_t)stream));
}

int dgl_gemm_tn_bf16(int P, int Mf, int Nf, const void* X, int ldx, const void* Y, int ldy, float* C, int ldc,
                     int transpose_out, void* ws, size_t ws_bytes, void* stream) {
  if (P <= 0 || Mf <= 0 || Mf > 256 || Nf <= 0 || Nf > 256 || !X || !Y || !C || !ws)
    return bad("dgl_gemm_tn_bf16: bad argument");
  if (ws_bytes < dgm::gemm_test_ws_bytes(P, 256, 256)) {
    strncpy(g_last_error, "dgl_gemm_tn_bf16: workspace too small", sizeof(g_last_error) - 1);
    return DGM_E_WORKSPACE;
  }
  return check(dgm::launch_gemm_tn_test(P, Mf, Nf, X, ldx, Y, ldy, C, ldc, transpose_out, ws, (cudaStream_t)stream));
}

int dgl_mlp_pack_sizes(size_t* w_bytes, size_t* b_bytes, size_t* g_bytes) {
  dgm::mlp_pack_sizes(w_bytes, b_bytes, g_bytes);
  return DGM_OK;
}

static int raw_ok(const DglRaw* r) {
  if (!r || r->n_heads < 1 || r->n_heads > 4 || r->in_t < 1 || r->in_t > 30) return 0;
  int rows = 0;
  for (int h = 0; h < r->n_heads; ++h) rows += r->head_rows[h];
  return rows >= 1 && rows <= 16;
}

int dgl_mlp_pack(const DglRaw* raw, void* wbuf, float* bbuf, DglNet* net_out, void* stream) {
  if (!raw_ok(raw) || !wbuf || !bbuf || !net_out) return bad("dgl_mlp_pack: bad argument");
  return check(dgm::launch_mlp_pack(*raw, wbuf, bbuf, net_out, (cudaStream_t)stream));
}

int dgl_mlp_grad_pointers(float* gbuf, DglGrads* grads_out) {
  if (!gbuf || !grads_out) return bad("dgl_mlp_grad_pointers: null pointer");
  dgm::mlp_grad_pointers(gbuf, grads_out);
  return DGM_OK;
}

int dgl_mlp_unpack_grads(const DglRaw* raw, const float* gbuf, const DglRawGrads* out, void* stream) {
  if (!raw_ok(raw) || !gbuf || !out) return bad("dgl_mlp_unpack_grads: bad argument");
  return check(dgm::launch_mlp_unpack_grads(*raw, gbuf, *out, (cudaStream_t)stream));
}

int dgl_mlp_workspace(int P, int train, size_t* bytes) {
  if (P < 0 || !bytes) return bad("dgl_mlp_workspace: bad argument");
  *bytes = dgm::mlp_workspace_bytes(P, train);
  return DGM_OK;
}

static int dgl_check(const DglNet* n, int P, const void* ws, size_t ws_bytes, int train) {
  if (!n || P <= 0 || !ws) return bad("mlp: bad argument");
  if (n->n_out < 1 || n->n_out > 16 || n->in_t < 1 || n->in_t > 32 || !n->Wh || !n->bh) return bad("mlp: bad net");
  for (int l = 0; l < 8; ++l)
    if (!n->W[l] || !n->b[l]) return bad("mlp: missing layer");
  if (n->has_timenet && (!n->Wt0 || !n->bt0 || !n->Wt1 || !n->bt1)) return bad("mlp: missing timenet");
  if (n->precise) {
    for (int l = 0; l < 8; ++l)
      if (!n->Wlo[l]) return bad("mlp: precise forward without residual operands");
    if (!n->Whlo || (n->has_timenet && (!n->Wt0lo || !n->Wt1lo))) return bad("mlp: precise forward without residual operands");
  }
  if (ws_bytes < dgm::mlp_workspace_bytes(P, train)) {
    strncpy(g_last_error, "mlp: workspace too small", sizeof(g_last_error) - 1);
    return DGM_E_WORKSPACE;
  }
  return DGM_OK;
}

int dgl_mlp_forward(const DglNet* net, int P, const float* x, const float* t, float* out, int train, void* ws,
                    size_t ws_bytes, void* stream) {
  int rc = dgl_check(net, P, ws, ws_bytes, train);
  if (rc != DGM_OK) return rc;
  if (!x || !t || !out) return bad("dgl_mlp_forward: null pointer");
  return check(dgm::launch_mlp_forward(*net, P, x, t, out, train, ws, (cudaStream_t)stream));
}

int dgl_mlp_backward(const DglNet* net, int P, const float* x, const float* out, const float* g_out, void* ws,
                     size_t ws_bytes, const DglGrads* grads, float* dx, void* stream) {
  int rc = dgl_check(net, P, ws, ws_bytes, 1);
  if (rc != DGM_OK) return rc;
  if (!x || !out || !g_out || !grads) return bad("dgl_mlp_backward: null pointer");
  for (int l = 0; l < 8; ++l)
    if (!net->WT[l] || !grads->dW[l] || !grads->db[l]) return bad("dgl_mlp_backward: missing transposed weights / grads");
  if (!net->WhT || !grads->dWh || !grads->dbh) return bad("dgl_mlp_backward: missing head buffers");
  if (net->has_timenet && (!net->Wt1T || !grads->dWt0 || !grads->dbt0 || !grads->dWt1 || !grads->dbt1))
    return bad("dgl_mlp_backward: missing timenet buffers");
  return check(dgm::launch_mlp_backward(*net, P, x, out, g_out, ws, *grads, dx, (cudaStream_t)stream));
}

int dgloss_workspace_size(int H, int W, size_t* bytes) {
  if (H <= 0 || W <= 0 || !bytes) return bad("dgloss_workspace_size: bad argument");
  *bytes = dgm::loss_workspace_bytes(H, W);
  return DGM_OK;
}

int dgloss_forward(int H, int W, const float* img, const float* gt, float lambda_dssim, int mode, float* out3, void* ws,
                   size_t ws_bytes, void* stream) {
  if (H <= 0 || W <= 0 || !img || !gt || !out3 || !ws) return bad("dgloss_forward: bad argument");
  if (ws_bytes < dgm::loss_workspace_bytes(H, W)) {
    strncpy(g_last_error, "dgloss_forward: workspace too small", sizeof(g_last_error) - 1);
    return DGM_E_WORKSPACE;
  }
  return check(dgm::launch_loss_forward(H, W, img, gt, lambda_dssim, mode, out3, ws, (cudaStream_t)stream));
}

int dgloss_backward(int H, int W, const float* img, const float* gt, float lambda_dssim, int mode,
                    const float* dL_dloss, float* dL_dimg, void* ws, size_t ws_bytes, void* stream) {
  if (H <= 0 || W <= 0 || !img || !gt || !dL_dimg || !ws) return bad("dgloss_backward: bad argument");
  if (ws_bytes < dgm::loss_workspace_bytes(H, W)) {
    strncpy(g_last_error, "dgloss_backward: workspace too small", sizeof(g_last_error) - 1);
    return DGM_E_WORKSPACE;
  }
  return check(dgm::launch_loss_backward(H, W, img, gt, lambda_dssim, mode, dL_dloss, dL_dimg, ws, (cudaStream_t)stream));
}

int dgl_laplacian_workspace(int V, size_t* bytes) {
  if (V < 0 || !bytes) return bad("dgl_laplacian_workspace: bad argument");
  *bytes = dgm::laplacian_ws_bytes(V);
  return DGM_OK;
}
int dgl_laplacian_forward(int V, int F, const float* verts, const int32_t* tri, float* out, void* ws,
                          size_t ws_bytes, void* stream) {
  if (V < 0 || F < 0 || !out || !ws || (V > 0 && !verts) || (F > 0 && !tri)) return bad("dgl_laplacian_forward: bad argument");
  if (ws_bytes < dgm::laplacian_ws_bytes(V)) {
    strncpy(g_last_error, "dgl_laplacian_forward: workspace too small", sizeof(g_last_error) - 1);
    return DGM_E_WORKSPACE;
  }
  return check(dgm::launch_laplacian_forward(V, F, verts, tri, out, ws, (cudaStream_t)stream));
}
int dgl_laplacian_backward(int V, int F, const int32_t* tri, const float* dL_dloss, float* dverts, void* ws,
                           size_t ws_bytes, void* stream) {
  if (V < 0 || F < 0 || !ws || (V > 0 && !dverts) || (F > 0 && !tri)) return bad("dgl_laplacian_backward: bad argument");
  if (ws_bytes < dgm::laplacian_ws_bytes(V)) {
    strncpy(g_last_error, "dgl_laplacian_backward: workspace too small", sizeof(g_last_error) - 1);
    return DGM_E_WORKSPACE;
  }
  if (V == 0) return DGM_OK;
  return check(dgm::launch_laplacian_backward(V, F, tri, dL_dloss, dverts, ws, (cudaStream_t)stream));
}

int dgmr_rasterize(int V, int F, int W, int H, const float* pos, const int32_t* tri, void* zbuf, float* rast,
                   void* stream) {
  if (V < 0 || F < 0 || W <= 0 || H <= 0 || !zbuf || !rast || (F > 0 && (!pos || !tri)))
    return bad("dgmr_rasterize: bad argument");
  return check(dgm::launch_mr_rasterize(V, F, W, H, pos, tri, zbuf, rast, (cudaStream_t)stream));
}
int dgmr_rasterize_bwd(int W, int H, const float* rast, const int32_t* tri, const float* pos, const float* grast,
                       float* gpos, void* stream) {
  if (W <= 0 || H <= 0 || !rast || !tri || !pos || !grast || !gpos) return bad("dgmr_rasterize_bwd: bad argument");
  return check(dgm::launch_mr_rasterize_bwd(W, H, rast, tri, pos, grast, gpos, (cudaStream_t)stream));
}
int dgmr_interpolate(int W, int H, int C, const float* attr, const float* rast, const int32_t* tri, float* out,
                     void* stream) {
  if (W <= 0 || H <= 0 || C < 1 || !attr || !rast || !tri || !out) return bad("dgmr_interpolate: bad argument");
  return check(dgm::launch_mr_interpolate(W, H, C, attr, rast, tri, out, (cudaStream_t)stream));
}
int dgmr_interpolate_bwd(int W, int H, int C, const float* attr, const float* rast, const int32_t* tri,
                         const float* gout, float* gattr, float* grast, void* stream) {
  if (W <= 0 || H <= 0 || C < 1 || !attr || !rast || !tri || !gout) return bad("dgmr_interpolate_bwd: bad argument");
  return check(dgm::launch_mr_interpolate_bwd(W, H, C, attr, rast, tri, gout, gattr, grast, (cudaStream_t)stream));
}
int dgmr_antialias(int W, int H, int C, const float* color, const float* rast, const float* pos,
                   const int32_t* tri, const int32_t* opp, float* out, void* stream) {
  if (W <= 0 || H <= 0 || C < 1 || !color || !rast || !pos || !tri || !opp || !out)
    return bad("dgmr_antialias: bad argument");
  return check(dgm::launch_mr_antialias(W, H, C, color, rast, pos, tri, opp, out, (cudaStream_t)stream));
}
int dgmr_antialias_bwd(int W, int H, int C, const float* color, const float* rast, const float* pos,
                       const int32_t* tri, const int32_t* opp, const float* gout, float* gcolor, float* gpos,
                       void* stream) {
  if (W <= 0 || H <= 0 || C < 1 || !color || !rast || !pos || !tri || !opp || !gout)
    return bad("dgmr_antialias_bwd: bad argument");
  return check(dgm::launch_mr_antialias_bwd(W, H, C, color, rast, pos, tri, opp, gout, gcolor, gpos,
                                            (cudaStream_t)stream));
}

int dgd_workspace_size(int P, size_t* bytes) {
  if (P <= 0 || !bytes) return bad("dgd_workspace_size: bad argument");
  *bytes = dgm::densify_ws_bytes(P);
  return DGM_OK;
}

static int dgd_check(int P, const void* ws, size_t ws_bytes) {
  if (P <= 0 || !ws) return bad("densify: bad argument");
  if (ws_bytes < dgm::densify_ws_bytes(P)) {
    strncpy(g_last_error, "densify: workspace too small", sizeof(g_last_error) - 1);
    return DGM_E_WORKSPACE;
  }
  return DGM_OK;
}

int dgd_plan(int P, const float* xyz_gradient_accum, const float* denom, const float* scaling_raw,
             const float* opacity_raw, float max_grad, float min_opacity, float extent, float percent_dense,
             int size_prune, float max_screen_size, void* ws, size_t ws_bytes, int32_t* counts, void* stream) {
  int rc = dgd_check(P, ws, ws_bytes);
  if (rc != DGM_OK) return rc;
  if (!xyz_gradient_accum || !denom || !scaling_raw || !opacity_raw || !counts) return bad("dgd_plan: null pointer");
  return check(dgm::launch_densify_plan(P, xyz_gradient_accum, denom, scaling_raw, opacity_raw, max_grad, min_opacity,
                                        extent, percent_dense, size_prune, max_screen_size, ws, counts,
                                        (cudaStream_t)stream));
}

int dgd_split_stds(int P, const float* scaling_raw, void* ws, size_t ws_bytes, float* stds, void* stream) {
  int rc = dgd_check(P, ws, ws_bytes);
  if (rc != DGM_OK) return rc;
  if (!scaling_raw || !stds) return bad("dgd_split_stds: null pointer");
  return check(dgm::launch_densify_stds(P, scaling_raw, ws, stds, (cudaStream_t)stream));
}

int dgd_apply(int P, int n_fields, const DgdField* fields_host, const float* rotation_raw, const float* samples,
              void* ws, size_t ws_bytes, void* stream) {
  int rc = dgd_check(P, ws, ws_bytes);
  if (rc != DGM_OK) return rc;
  if (n_fields < 1 || n_fields > DGD_MAX_FIELDS || !fields_host || !rotation_raw) return bad("dgd_apply: bad argument");
  dgm::DensifyTables t = {};
  t.n_fields = n_fields;
  t.rotation_raw = rotation_raw;
  int cols = 0;
  for (int i = 0; i < n_fields; ++i) {
    const DgdField& f = fields_host[i];
    if (!f.src || !f.dst || f.width < 1 || ((f.m1_src == nullptr) != (f.m1_dst == nullptr)) ||
        ((f.m1_src == nullptr) != (f.m2_src == nullptr)) || ((f.m1_dst == nullptr) != (f.m2_dst == nullptr)))
      return bad("dgd_apply: bad field");
    t.f[i].src = f.src; t.f[i].m1_src = f.m1_src; t.f[i].m2_src = f.m2_src;
    t.f[i].dst = f.dst; t.f[i].m1_dst = f.m1_dst; t.f[i].m2_dst = f.m2_dst;
    t.f[i].width = f.width; t.f[i].role = f.role;
    cols += f.width;
  }
  if (cols > 64) return bad("dgd_apply: more than 64 parameter columns");
  return check(dgm::launch_densify_apply(P, t, samples, ws, (cudaStream_t)stream));
}

int dgx_allreduce_nvls(float* multicast_ptr, size_t n_floats, void* signal_pads_dev, int rank, int world,
                       uint32_t epoch, float scale, int blocks, void* stream) {
  if (!multicast_ptr || !signal_pads_dev || world < 1 || rank < 0 || rank >= world || blocks < 1 || (n_floats & 3) ||
      ((uintptr_t)multicast_ptr & 15) || epoch == 0)
    return bad("dgx_allreduce_nvls: bad argument");
  return check(dgm::launch_nvls_allreduce(multicast_ptr, n_floats, (uint32_t* const*)signal_pads_dev, rank, world,
                                          epoch, scale, blocks, (cudaStream_t)stream));
}

// ---- early notification objects: an event + a device-mapped pinned status mirror.  These are the
// only resources the library creates on request (host memory and an event, no device memory).
struct DgmNotify {
  cudaEvent_t ev;
  int32_t* host;
};

int dgm_notify_create(void** handle) {
  if (!handle) return bad("dgm_notify_create: null handle");
  DgmNotify* n = new DgmNotify();
  if (cudaEventCreateWithFlags(&n->ev, cudaEventDisableTiming) != cudaSuccess ||
      cudaHostAlloc((void**)&n->host, sizeof(int32_t) * DGR_STATUS_WORDS * 64,
                    cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) {
    delete n;
    return check(cudaGetLastError());
  }
  memset(n->host, 0, sizeof(int32_t) * DGR_STATUS_WORDS * 64);
  *handle = n;
  return DGM_OK;
}
int32_t* dgm_notify_host(void* handle) { return handle ? ((DgmNotify*)handle)->host : nullptr; }
void* dgm_notify_event(void* handle) { return handle ? (void*)((DgmNotify*)handle)->ev : nullptr; }
int dgm_notify_wait(void* handle) {
  if (!handle) return bad("dgm_notify_wait: null handle");
  return check(cudaEventSynchronize(((DgmNotify*)handle)->ev));
}
int dgm_notify_destroy(void* handle) {
  if (!handle) return DGM_OK;
  DgmNotify* n = (DgmNotify*)handle;
  cudaEventDestroy(n->ev);
  cudaFreeHost(n->host);
  delete n;
  return DGM_OK;
}

int dgm_profile_enable(int on) {
  using dgm::g_prof;
  if (on && !g_prof.ev[0][0]) {
    for (int k = 0; k < DGM_K_COUNT; ++k)
      for (int j = 0; j < 2; ++j)
        if (cudaEventCreate(&g_prof.ev[k][j]) != cudaSuccess) return check(cudaGetLastError());
  }
  g_prof.on = on;
  g_prof.tl_n = 0;
  for (int k = 0; k < DGM_K_COUNT; ++k) g_prof.used[k] = false;
  return DGM_OK;
}

int dgm_timeline_read(float* begin_ms, float* end_ms, int* kernel_ids, int cap) {
  using dgm::g_prof;
  if (!begin_ms || !end_ms || !kernel_ids || cap < 0) return bad("dgm_timeline_read: bad argument");
  if (cudaDeviceSynchronize() != cudaSuccess) return check(cudaGetLastError());
  const int n = g_prof.tl_n < cap ? g_prof.tl_n : cap;
  for (int i = 0; i < n; ++i) {
    kernel_ids[i] = g_prof.tl_id[i];
    cudaEventElapsedTime(&begin_ms[i], g_prof.tl_ev[0][0], g_prof.tl_ev[i][0]);
    cudaEventElapsedTime(&end_ms[i], g_prof.tl_ev[0][0], g_prof.tl_ev[i][1]);
  }
  cudaGetLastError();
  return n;
}

int dgm_profile_read(float* ms_host, int n) {
  using dgm::g_prof;
  if (!ms_host || n < 0) return bad("dgm_profile_read: bad argument");
  for (int k = 0; k < n && k < DGM_K_COUNT; ++k) {
    ms_host[k] = -1.f;
    if (!g_prof.used[k]) continue;
    if (cudaEventSynchronize(g_prof.ev[k][1]) != cudaSuccess) return check(cudaGetLastError());
    float ms = -1.f;
    if (cudaEventElapsedTime(&ms, g_prof.ev[k][0], g_prof.ev[k][1]) != cudaSuccess) return check(cudaGetLastError());
    ms_host[k] = ms;
  }
  return DGM_OK;
}

}  // extern "C"
