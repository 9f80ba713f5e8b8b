// api.cu -- the C-ABI of libdgmesh_b200.so (see include/dgmesh_b200.h).
#include "../../include/dgmesh_b200.h"
#include "common.cuh"
#include "raster_kernels.h"
#include "depth_normal_kernels.h"
#include "knn_kernels.h"
#include "dpsr_kernels.h"
#include "mc_kernels.h"
#include "flexicubes_kernels.h"
#include "loss_kernels.h"
#include "mlp_kernels.h"
#include "densify_kernels.h"
#include "optim_kernels.h"
#include "opacity_field_kernels.h"
#include "tsdf_kernels.h"
#include "metrics_kernels.h"
#include "mesh_distance_kernels.h"
#include "deform_reg_kernels.h"
#include "hexplane_kernels.h"
#include "hashgrid_kernels.h"
#include "meshrast_kernels.h"
#include "nvls_kernels.h"

#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <mutex>
#include <map>
#include <math.h>

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

int dgr_normal_workspace_size(int P, int64_t R_cap, size_t* bytes) {
  if (P < 0 || R_cap < 0 || !bytes) return bad("dgr_normal_workspace_size: bad argument");
  dgm::NrmWS::from(nullptr, (size_t)P, (size_t)R_cap, bytes);
  return DGM_OK;
}

int dgr_surface_workspace_size(int W, int H, size_t* bytes) {
  if (W <= 0 || H <= 0 || !bytes) return bad("dgr_surface_workspace_size: bad argument");
  dgm::SurfWS::from(nullptr, (size_t)W * H, bytes);
  return DGM_OK;
}

namespace {
// near / far of the normalised depth: DGM_OK, or the error to return
int surface_range(float near_, float far_) {
  if (!(near_ > 0.0f) || !(far_ > near_) || !(far_ < INFINITY)) return bad("dgr_*_surf: need 0 < near < far");
  return DGM_OK;
}

// k = far near / (far - near) of the normalised depth (see surf_m), rounded as the CPU oracle rounds it
float surf_k(float near_, float far_) {
  const float mk = far_ / (far_ - near_);
  return mk * near_;
}

// the surface-map arguments of a forward (any output non-NULL): DGM_OK, or the error to return
int surface_args(int W, int H, float near_, float far_, void* surf_ws, size_t surf_ws_bytes) {
  const int rc = surface_range(near_, far_);
  if (rc != DGM_OK) return rc;
  size_t need;
  if (dgr_surface_workspace_size(W, H, &need) != DGM_OK) return DGM_E_BADARG;
  if (!surf_ws || surf_ws_bytes < need) {
    strncpy(g_last_error, "dgr_forward_surf: surface workspace too small", sizeof(g_last_error) - 1);
    return DGM_E_WORKSPACE;
  }
  return DGM_OK;
}

// the normal-map arguments of a forward: DGM_OK, or the error to return
int normal_args(int P, int64_t R_cap, const float* normals, float* out_normal, void* nrm_ws, size_t nrm_ws_bytes) {
  if (!out_normal || P == 0) return DGM_OK;
  if (!normals) return bad("dgr_forward_nrm: normals missing");
  size_t need;
  dgr_normal_workspace_size(P, R_cap, &need);
  if (!nrm_ws || nrm_ws_bytes < need) {
    strncpy(g_last_error, "dgr_forward_nrm: normal workspace too small", sizeof(g_last_error) - 1);
    return DGM_E_WORKSPACE;
  }
  return DGM_OK;
}

// the Gaussian inputs of a forward of P > 0 Gaussians: DGM_OK, or the error to return (`who` names the entry point)
int gaussian_args(const char* who, int D, int M, const float* means3D, const float* shs, const float* colors_precomp,
                  const float* opacities, const float* scales, const float* rotations, const float* cov3D_precomp) {
  const char* e = nullptr;
  if (!means3D || !opacities) e = "means3D / opacities missing";
  else if ((shs == nullptr) == (colors_precomp == nullptr)) e = "exactly one of shs / colors_precomp";
  else if (((scales == nullptr) || (rotations == nullptr)) == (cov3D_precomp == nullptr))
    e = "exactly one of scales+rotations / cov3D_precomp";
  else if (shs && (M <= 0 || M > 16 || (D + 1) * (D + 1) > M || D < 0 || D > 3)) e = "SH degree / coefficient count";
  if (!e) return DGM_OK;
  char msg[128];
  snprintf(msg, sizeof(msg), "%s: %s", who, e);
  return bad(msg);
}

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

// a frame of no Gaussian: the reference skips the whole pipeline and returns the zero-initialised image
// (rasterize_points.cu:64,80: torch::full(0.0) and `if (P != 0)`)
cudaError_t zero_frame(const dgm::FwdArgs& a, cudaStream_t s) {
  const size_t map = sizeof(float) * (size_t)a.W * a.H;
  cudaMemsetAsync(a.out_color, 0, 3 * map, s);
  if (a.out_depth) cudaMemsetAsync(a.out_depth, 0, map, s);
  if (a.out_alpha) cudaMemsetAsync(a.out_alpha, 0, map, s);
  if (a.out_normal) cudaMemsetAsync(a.out_normal, 0, 3 * map, s);
  if (a.out_median) cudaMemsetAsync(a.out_median, 0, map, s);
  if (a.out_distortion) cudaMemsetAsync(a.out_distortion, 0, map, s);
  cudaMemsetAsync(a.status, 0, sizeof(int32_t) * DGR_STATUS_WORDS, s);
  if (a.status_host) memset(a.status_host, 0, sizeof(int32_t) * DGR_STATUS_WORDS);
  if (a.status_event) cudaEventRecord(a.status_event, s);
  return cudaGetLastError();
}

// The forward of F frames whose arguments have been checked, in the layout of dgr_forward_batch_surf (one frame: the
// arguments of dgr_forward_surf with F = 1, strides 0 and one stream).  Frame f reads camera f and the slab f of each
// per-frame input, and writes its maps, radii and status words at f times their size and its workspaces at f times
// their stride.  With one stream (or one frame, or no Gaussian) the frames run in order on the caller's stream and
// status_event is recorded after the last frame's tile scan; otherwise they run on the BatchStreams.
int forward_frames(int F, int P, int D, int M, const float* background, int W, int H, const float* means3D,
                   const float* shs, const float* colors_precomp, const float* opacities, const float* scales,
                   float scale_modifier, const float* rotations, const float* cov3D_precomp, int per_frame,
                   const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                   const float* tan_fovx_host, const float* tan_fovy_host, int prefiltered, float* out_color,
                   int* radii, float* out_depth, float* out_alpha, const float* normals, int normals_per_frame,
                   float* out_normal, void* nrm_ws, size_t nrm_ws_stride, float near_, float far_,
                   float* out_median, float* out_distortion, void* surf_ws, size_t surf_ws_stride, void* geom_ws,
                   size_t geom_stride, void* binning_ws, size_t binning_stride, int64_t R_cap, void* img_ws,
                   size_t img_stride, int32_t* status, int32_t* status_host, void* status_event,
                   float depth_hint_lo, float depth_hint_hi, int max_tile_hint, int n_streams, void* stream) {
  const size_t npix = (size_t)W * H, cw = shs ? (size_t)M * 3 : 3;
  const bool surf = out_median || out_distortion;
  // frame f of: an input whose bit is set in per_frame ([F,P,width]), a [F,c,H,W] map, a workspace
  auto pf = [&](const float* p, int bit, size_t width, int f) {
    return (p && (per_frame & bit)) ? p + (size_t)f * P * width : p;
  };
  auto map = [&](float* p, size_t c, int f) { return p ? p + f * c * npix : p; };
  auto ws = [](void* p, size_t stride, int f) { return p ? (void*)((char*)p + f * stride) : p; };
  auto frame = [&](int f) {
    dgm::FwdArgs a;
    a.P = P; a.D = D; a.M = M; a.background = background; a.W = W; a.H = H;
    a.means3D = pf(means3D, DGR_PF_MEANS, 3, f); a.shs = pf(shs, DGR_PF_COLOR, cw, f);
    a.colors_precomp = pf(colors_precomp, DGR_PF_COLOR, 3, f); a.opacities = pf(opacities, DGR_PF_OPAC, 1, f);
    a.scales = pf(scales, DGR_PF_SCALES, 3, f); a.scale_modifier = scale_modifier;
    a.rotations = pf(rotations, DGR_PF_ROTS, 4, f); a.cov3D_precomp = pf(cov3D_precomp, DGR_PF_COV, 6, f);
    a.viewmatrix = viewmatrices + 16 * f; a.projmatrix = projmatrices + 16 * f; a.cam_pos = cam_poses + 3 * f;
    a.tan_fovx = tan_fovx_host[f]; a.tan_fovy = tan_fovy_host[f]; a.prefiltered = prefiltered;
    a.out_color = map(out_color, 3, f); a.radii = radii ? radii + (size_t)f * P : nullptr;
    a.out_depth = map(out_depth, 1, f); a.out_alpha = map(out_alpha, 1, f);
    a.geom_ws = ws(geom_ws, geom_stride, f); a.binning_ws = ws(binning_ws, binning_stride, f);
    a.img_ws = ws(img_ws, img_stride, f); a.R_cap = R_cap;
    a.status = status + f * DGR_STATUS_WORDS; a.status_host = status_host ? status_host + f * DGR_STATUS_WORDS : nullptr;
    a.status_event = nullptr; a.hint_lo = depth_hint_lo; a.hint_hi = depth_hint_hi; a.hint_max_tile = max_tile_hint;
    if (out_normal) {
      a.normals = (normals && normals_per_frame) ? normals + (size_t)f * P * 3 : normals;
      a.out_normal = map(out_normal, 3, f); a.nrm_ws = ws(nrm_ws, nrm_ws_stride, f);
    }
    if (surf) {
      a.out_median = map(out_median, 1, f); a.out_distortion = map(out_distortion, 1, f);
      a.surf_ws = ws(surf_ws, surf_ws_stride, f); a.surf_k = surf_k(near_, far_);
    }
    return a;
  };
  cudaStream_t main_s = (cudaStream_t)stream;
  cudaError_t e = cudaSuccess;
  if (n_streams <= 1 || F == 1 || P == 0) {
    for (int f = 0; f < F && e == cudaSuccess; ++f) {
      dgm::FwdArgs a = frame(f);
      if (f == F - 1) a.status_event = (cudaEvent_t)status_event;
      e = P > 0 ? dgm::launch_forward(a, main_s) : zero_frame(a, main_s);
    }
    return check(e);
  }
  const int NH = n_streams > BatchStreams::NH ? BatchStreams::NH : n_streams;
  BatchStreams* bs = batch_streams();
  if (!bs) return check(cudaGetLastError());
  std::lock_guard<std::mutex> lk(bs->mu);
  cudaEventRecord(bs->fork, main_s);
  for (int i = 0; i < NH; ++i) cudaStreamWaitEvent(bs->hi[i], bs->fork, 0);
  for (int i = 0; i < 2; ++i) cudaStreamWaitEvent(bs->lo[i], bs->fork, 0);
  for (int f = 0; f < F && e == cudaSuccess; ++f) {
    const int i = f % NH;
    cudaStream_t lo = bs->lo[f & 1];
    const dgm::FwdArgs a = frame(f);
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
}  // namespace

int dgr_forward_surf(int P, int D, int M, const float* background, int W, int H, const float* means3D,
                     const float* shs, const float* colors_precomp, const float* opacities, const float* scales,
                     float scale_modifier, const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                     const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy, int prefiltered,
                     float* out_color, int* radii, float* out_depth, float* out_alpha, const float* normals,
                     float* out_normal, void* nrm_ws, size_t nrm_ws_bytes, float near_, float far_,
                     float* out_median, float* out_distortion, void* surf_ws, size_t surf_ws_bytes, void* geom_ws,
                     size_t geom_bytes, void* binning_ws, size_t binning_bytes, int64_t R_cap, void* img_ws,
                     size_t img_bytes, int32_t* status, int32_t* status_host, void* status_event,
                     float depth_hint_lo, float depth_hint_hi, int max_tile_hint, void* stream) {
  if (P < 0 || W <= 0 || H <= 0 || R_cap < 0) return bad("dgr_forward: negative size");
  if (!background || !viewmatrix || !projmatrix || !cam_pos || !out_color || !status)
    return bad("dgr_forward: null required pointer");
  int rc = normal_args(P, R_cap, normals, out_normal, nrm_ws, nrm_ws_bytes);
  if (rc != DGM_OK) return rc;
  if ((out_median || out_distortion) && (rc = surface_args(W, H, near_, far_, surf_ws, surf_ws_bytes)) != DGM_OK)
    return rc;
  if (P > 0) {
    rc = gaussian_args("dgr_forward", D, M, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp);
    if (rc != DGM_OK) return rc;
    size_t gb, bb, ib;
    dgr_workspace_sizes(P, W, H, R_cap, &gb, &bb, &ib);
    if (geom_bytes < gb || binning_bytes < bb || img_bytes < ib || !geom_ws || !binning_ws || !img_ws) {
      strncpy(g_last_error, "dgr_forward: workspace too small", sizeof(g_last_error) - 1);
      return DGM_E_WORKSPACE;
    }
  }
  return forward_frames(1, P, D, M, background, W, H, means3D, shs, colors_precomp, opacities, scales, scale_modifier,
                        rotations, cov3D_precomp, 0, viewmatrix, projmatrix, cam_pos, &tan_fovx, &tan_fovy,
                        prefiltered, out_color, radii, out_depth, out_alpha, normals, 0, out_normal, nrm_ws, 0, near_,
                        far_, out_median, out_distortion, surf_ws, 0, geom_ws, 0, binning_ws, 0, R_cap, img_ws, 0,
                        status, status_host, status_event, depth_hint_lo, depth_hint_hi, max_tile_hint, 1, stream);
}

int dgr_forward_nrm(int P, int D, int M, const float* background, int W, int H, const float* means3D,
                    const float* shs, const float* colors_precomp, const float* opacities, const float* scales,
                    float scale_modifier, const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                    const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy, int prefiltered,
                    float* out_color, int* radii, float* out_depth, float* out_alpha, const float* normals,
                    float* out_normal, void* nrm_ws, size_t nrm_ws_bytes, void* geom_ws, size_t geom_bytes,
                    void* binning_ws, size_t binning_bytes, int64_t R_cap, void* img_ws, size_t img_bytes,
                    int32_t* status, int32_t* status_host, void* status_event, float depth_hint_lo,
                    float depth_hint_hi, int max_tile_hint, void* stream) {
  return dgr_forward_surf(P, D, M, background, W, H, means3D, shs, colors_precomp, opacities, scales, scale_modifier,
                          rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, prefiltered,
                          out_color, radii, out_depth, out_alpha, normals, out_normal, nrm_ws, nrm_ws_bytes, 0.f, 0.f,
                          nullptr, nullptr, nullptr, 0, geom_ws, geom_bytes, binning_ws, binning_bytes, R_cap, img_ws,
                          img_bytes, status, status_host, status_event, depth_hint_lo, depth_hint_hi, max_tile_hint,
                          stream);
}

int dgr_forward_aux(int P, int D, int M, const float* background, int W, int H, const float* means3D,
                    const float* shs, const float* colors_precomp, const float* opacities, const float* scales,
                    float scale_modifier, const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                    const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy, int prefiltered,
                    float* out_color, int* radii, float* out_depth, float* out_alpha, void* geom_ws,
                    size_t geom_bytes, void* binning_ws, size_t binning_bytes, int64_t R_cap, void* img_ws,
                    size_t img_bytes, int32_t* status, int32_t* status_host, void* status_event,
                    float depth_hint_lo, float depth_hint_hi, int max_tile_hint, void* stream) {
  return dgr_forward_surf(P, D, M, background, W, H, means3D, shs, colors_precomp, opacities, scales, scale_modifier,
                          rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, prefiltered,
                          out_color, radii, out_depth, out_alpha, nullptr, nullptr, nullptr, 0, 0.f, 0.f, nullptr,
                          nullptr, nullptr, 0, geom_ws, geom_bytes, binning_ws, binning_bytes, R_cap, img_ws,
                          img_bytes, status, status_host, status_event, depth_hint_lo, depth_hint_hi, max_tile_hint,
                          stream);
}

int dgr_forward(int P, int D, int M, const float* background, int W, int H, const float* means3D, const float* shs,
                const float* colors_precomp, const float* opacities, const float* scales, float scale_modifier,
                const float* rotations, const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                const float* cam_pos, float tan_fovx, float tan_fovy, int prefiltered, float* out_color, int* radii,
                void* geom_ws, size_t geom_bytes, void* binning_ws, size_t binning_bytes, int64_t R_cap, void* img_ws,
                size_t img_bytes, int32_t* status, int32_t* status_host, void* status_event, float depth_hint_lo,
                float depth_hint_hi, int max_tile_hint, void* stream) {
  return dgr_forward_aux(P, D, M, background, W, H, means3D, shs, colors_precomp, opacities, scales, scale_modifier,
                         rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, prefiltered,
                         out_color, radii, nullptr, nullptr, geom_ws, geom_bytes, binning_ws, binning_bytes, R_cap,
                         img_ws, img_bytes, status, status_host, status_event, depth_hint_lo, depth_hint_hi,
                         max_tile_hint, stream);
}

int dgr_forward_batch_surf(int F, int P, int D, int M, const float* background, int W, int H,
                           const float* means3D, const float* shs, const float* colors_precomp,
                           const float* opacities, const float* scales, float scale_modifier, const float* rotations,
                           const float* cov3D_precomp, int per_frame, const float* viewmatrices,
                           const float* projmatrices, const float* cam_poses, const float* tan_fovx_host,
                           const float* tan_fovy_host, int prefiltered, float* out_color, int* radii,
                           float* out_depth, float* out_alpha, const float* normals, int normals_per_frame,
                           float* out_normal, void* nrm_ws, size_t nrm_ws_stride, float near_, float far_,
                           float* out_median, float* out_distortion, void* surf_ws, size_t surf_ws_stride,
                           void* geom_ws, size_t geom_stride, void* binning_ws, size_t binning_stride,
                           int64_t R_cap, void* img_ws, size_t img_stride, int32_t* status, int32_t* status_host,
                           void* status_event, float depth_hint_lo, float depth_hint_hi, int max_tile_hint,
                           int n_streams, void* stream) {
  if (F <= 0 || !tan_fovx_host || !tan_fovy_host || !viewmatrices || !projmatrices || !cam_poses)
    return bad("dgr_forward_batch: bad argument");
  size_t gb, bb, ib;
  if (dgr_workspace_sizes(P, W, H, R_cap, &gb, &bb, &ib) != DGM_OK) return DGM_E_BADARG;
  if (geom_stride < gb || binning_stride < bb || img_stride < ib || (geom_stride | binning_stride | img_stride) & 127) {
    strncpy(g_last_error, "dgr_forward_batch: workspace stride too small / unaligned", sizeof(g_last_error) - 1);
    return DGM_E_WORKSPACE;
  }
  int rc;
  if (out_normal) {
    if ((rc = normal_args(P, R_cap, normals, out_normal, nrm_ws, nrm_ws_stride)) != DGM_OK) return rc;
    if (nrm_ws_stride & 127) return bad("dgr_forward_batch_nrm: normal workspace stride unaligned");
  }
  if (out_median || out_distortion) {
    if ((rc = surface_args(W, H, near_, far_, surf_ws, surf_ws_stride)) != DGM_OK) return rc;
    if (surf_ws_stride & 127) return bad("dgr_forward_batch_surf: surface workspace stride unaligned");
  }
  if (!background || !out_color || !status) return bad("dgr_forward_batch: null required pointer");
  if (P > 0) {
    rc = gaussian_args("dgr_forward_batch", D, M, means3D, shs, colors_precomp, opacities, scales, rotations,
                       cov3D_precomp);
    if (rc != DGM_OK) return rc;
    if (!geom_ws || !binning_ws || !img_ws) {
      strncpy(g_last_error, "dgr_forward_batch: workspace missing", sizeof(g_last_error) - 1);
      return DGM_E_WORKSPACE;
    }
  }
  return forward_frames(F, P, D, M, background, W, H, means3D, shs, colors_precomp, opacities, scales, scale_modifier,
                        rotations, cov3D_precomp, per_frame, viewmatrices, projmatrices, cam_poses, tan_fovx_host,
                        tan_fovy_host, prefiltered, out_color, radii, out_depth, out_alpha, normals, normals_per_frame,
                        out_normal, nrm_ws, nrm_ws_stride, near_, far_, out_median, out_distortion, surf_ws,
                        surf_ws_stride, geom_ws, geom_stride, binning_ws, binning_stride, R_cap, img_ws, img_stride,
                        status, status_host, status_event, depth_hint_lo, depth_hint_hi, max_tile_hint, n_streams,
                        stream);
}

int dgr_forward_batch_nrm(int F, int P, int D, int M, const float* background, int W, int H, const float* means3D,
                          const float* shs, const float* colors_precomp, const float* opacities, const float* scales,
                          float scale_modifier, const float* rotations, const float* cov3D_precomp, int per_frame,
                          const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                          const float* tan_fovx_host, const float* tan_fovy_host, int prefiltered, float* out_color,
                          int* radii, float* out_depth, float* out_alpha, const float* normals, int normals_per_frame,
                          float* out_normal, void* nrm_ws, size_t nrm_ws_stride, void* geom_ws, size_t geom_stride,
                          void* binning_ws, size_t binning_stride, int64_t R_cap, void* img_ws, size_t img_stride,
                          int32_t* status, int32_t* status_host, void* status_event, float depth_hint_lo,
                          float depth_hint_hi, int max_tile_hint, int n_streams, void* stream) {
  return dgr_forward_batch_surf(F, P, D, M, background, W, H, means3D, shs, colors_precomp, opacities, scales,
                                scale_modifier, rotations, cov3D_precomp, per_frame, viewmatrices, projmatrices,
                                cam_poses, tan_fovx_host, tan_fovy_host, prefiltered, out_color, radii, out_depth,
                                out_alpha, normals, normals_per_frame, out_normal, nrm_ws, nrm_ws_stride, 0.f, 0.f,
                                nullptr, nullptr, nullptr, 0, geom_ws, geom_stride, binning_ws, binning_stride, R_cap,
                                img_ws, img_stride, status, status_host, status_event, depth_hint_lo, depth_hint_hi,
                                max_tile_hint, n_streams, stream);
}

int dgr_forward_batch_aux(int F, int P, int D, int M, const float* background, int W, int H, const float* means3D,
                          const float* shs, const float* colors_precomp, const float* opacities, const float* scales,
                          float scale_modifier, const float* rotations, const float* cov3D_precomp, int per_frame,
                          const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                          const float* tan_fovx_host, const float* tan_fovy_host, int prefiltered, float* out_color,
                          int* radii, float* out_depth, float* out_alpha, void* geom_ws, size_t geom_stride,
                          void* binning_ws, size_t binning_stride, int64_t R_cap, void* img_ws, size_t img_stride,
                          int32_t* status, int32_t* status_host, void* status_event, float depth_hint_lo,
                          float depth_hint_hi, int max_tile_hint, int n_streams, void* stream) {
  return dgr_forward_batch_nrm(F, P, D, M, background, W, H, means3D, shs, colors_precomp, opacities, scales,
                               scale_modifier, rotations, cov3D_precomp, per_frame, viewmatrices, projmatrices,
                               cam_poses, tan_fovx_host, tan_fovy_host, prefiltered, out_color, radii, out_depth,
                               out_alpha, nullptr, 0, nullptr, nullptr, 0, geom_ws, geom_stride, binning_ws,
                               binning_stride, R_cap, img_ws, img_stride, status, status_host, status_event,
                               depth_hint_lo, depth_hint_hi, max_tile_hint, n_streams, stream);
}

int dgr_forward_batch(int F, int P, int D, int M, const float* background, int W, int H, const float* means3D,
                      const float* shs, const float* colors_precomp, const float* opacities, const float* scales,
                      float scale_modifier, const float* rotations, const float* cov3D_precomp, int per_frame,
                      const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                      const float* tan_fovx_host, const float* tan_fovy_host, int prefiltered, float* out_color,
                      int* radii, void* geom_ws, size_t geom_stride, void* binning_ws, size_t binning_stride,
                      int64_t R_cap, void* img_ws, size_t img_stride, int32_t* status, int32_t* status_host,
                      void* status_event, float depth_hint_lo, float depth_hint_hi, int max_tile_hint, int n_streams,
                      void* stream) {
  return dgr_forward_batch_aux(F, P, D, M, background, W, H, means3D, shs, colors_precomp, opacities, scales,
                               scale_modifier, rotations, cov3D_precomp, per_frame, viewmatrices, projmatrices,
                               cam_poses, tan_fovx_host, tan_fovy_host, prefiltered, out_color, radii, nullptr,
                               nullptr, geom_ws, geom_stride, binning_ws, binning_stride, R_cap, img_ws, img_stride,
                               status, status_host, status_event, depth_hint_lo, depth_hint_hi, max_tile_hint,
                               n_streams, stream);
}

int dgr_camera_grad_workspace_size(int F, int P, size_t* bytes) {
  if (F <= 0 || P < 0 || !bytes) return bad("dgr_camera_grad_workspace_size: bad argument");
  *bytes = dgm::intrinsics_ws_bytes(F, P);  // enough for the pose and the intrinsics outputs
  return DGM_OK;
}

namespace {
// the camera-gradient arguments of dgr_backward{,_batch}_cam and of dL_dtanfov (dgr_backward{,_batch}_intr): DGM_OK,
// or the error to return.  The pose outputs alone need the workspace of their partials, dL_dtanfov that of both
int camera_args(int F, int P, float* dL_dview, float* dL_dproj, float* dL_dcampos, float* dL_dtanfov, void* cam_ws,
                size_t cam_ws_bytes, cudaStream_t s) {
  if (!dL_dview && !dL_dproj && !dL_dcampos && !dL_dtanfov) return DGM_OK;
  if (P == 0) {  // no Gaussian: the camera gradients are zero
    if (dL_dview) cudaMemsetAsync(dL_dview, 0, sizeof(float) * 16 * F, s);
    if (dL_dproj) cudaMemsetAsync(dL_dproj, 0, sizeof(float) * 16 * F, s);
    if (dL_dcampos) cudaMemsetAsync(dL_dcampos, 0, sizeof(float) * 3 * F, s);
    if (dL_dtanfov) cudaMemsetAsync(dL_dtanfov, 0, sizeof(float) * INTR_TERMS * F, s);
    return check(cudaGetLastError());
  }
  if (!cam_ws || cam_ws_bytes < (dL_dtanfov ? dgm::intrinsics_ws_bytes(F, P) : dgm::camera_ws_bytes(F, P))) {
    strncpy(g_last_error, "dgr_backward_cam: camera-gradient workspace too small", sizeof(g_last_error) - 1);
    return DGM_E_WORKSPACE;
  }
  return DGM_OK;
}

// The backward of F frames of P > 0 Gaussians whose arguments have been checked, in the layout of
// dgr_backward_batch_intr plus the [P,4] dL_dconic of a single frame (one frame: the arguments of dgr_backward_intr
// with F = 1, strides 0 and one stream).  Each frame's blend backward (+ median gradient), then one per-Gaussian
// backward for all frames (+ the normal gradients) on the caller's stream.
int backward_frames(int F, int P, int D, int M, const float* background, int W, int H, const float* means3D,
                    const float* shs, const float* colors_precomp, const float* scales, float scale_modifier,
                    const float* rotations, const float* cov3D_precomp, int per_frame, const float* viewmatrices,
                    const float* projmatrices, const float* cam_poses, const float* tan_fovx_host,
                    const float* tan_fovy_host, const int* radii, void* geom_ws, size_t geom_stride,
                    void* binning_ws, size_t binning_stride, int64_t R_cap, void* img_ws, size_t img_stride,
                    const float* dL_dpix, const float* dL_ddepth, const float* dL_dalpha, float* dL_dmean2D,
                    float* dL_dconic, float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D,
                    float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dviewmatrix, float* dL_dprojmatrix,
                    float* dL_dcampos, void* cam_ws, const float* dL_dnormal_maps, int normals_per_frame,
                    float* dL_dnormals, void* nrm_ws, size_t nrm_ws_stride, float near_, float far_,
                    const float* dL_dmedian, const float* dL_ddistortion, void* surf_ws, size_t surf_ws_stride,
                    float* dL_dmean2D_abs, float* dL_dtanfov, int n_streams, void* stream) {
  // the render_bwd kernels alternate two low-priority streams (the next one's CTAs fill the SMs while the
  // previous one's tail drains); one per-Gaussian kernel for all frames follows once both have finished
  const bool multi = n_streams > 1 && F > 1;
  cudaStream_t main_s = (cudaStream_t)stream;
  // the kernels of every frame add into its slab: zeroed on the call's stream, before the fork
  if (dL_dmean2D_abs) cudaMemsetAsync(dL_dmean2D_abs, 0, sizeof(float) * 3 * (size_t)F * P, main_s);
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
  a.dL_ddepth = dL_ddepth; a.dL_dalpha = dL_dalpha; a.dL_dmean2D = dL_dmean2D; a.dL_dconic = dL_dconic;
  a.dL_dopacity = dL_dopacity; a.dL_dcolor = dL_dcolor; a.dL_dmean3D = dL_dmean3D; a.dL_dcov3D = dL_dcov3D;
  a.dL_dsh = dL_dsh; a.dL_dscale = dL_dscale; a.dL_drot = dL_drot;
  a.F = F; a.per_frame = per_frame; a.geom_stride = geom_stride;
  a.dL_dview = dL_dviewmatrix; a.dL_dproj = dL_dprojmatrix; a.dL_dcampos = dL_dcampos; a.cam_ws = (float*)cam_ws;
  a.dL_dtanfov = dL_dtanfov;
  if (dL_dnormal_maps) {
    a.dL_dnormal = dL_dnormal_maps; a.dL_dnormals = dL_dnormals; a.nrm_ws = nrm_ws; a.nrm_stride = nrm_ws_stride;
    a.normals_per_frame = normals_per_frame;
  }
  if (dL_dmedian || dL_ddistortion) {
    a.dL_dmedian = dL_dmedian; a.dL_ddistortion = dL_ddistortion; a.surf_ws = surf_ws;
    a.surf_k = surf_k(near_, far_);
  }
  cudaError_t e = cudaSuccess;
  for (int f = 0; f < F && e == cudaSuccess; ++f) {
    dgm::BwdArgs af = a;  // launch_render_bwd reads frame 0 of its arguments
    af.geom_ws = (char*)geom_ws + f * geom_stride; af.binning_ws = (char*)binning_ws + f * binning_stride;
    af.img_ws = (char*)img_ws + f * img_stride; af.dL_dpix = dL_dpix + (size_t)f * 3 * W * H;
    if (dL_ddepth) af.dL_ddepth = dL_ddepth + (size_t)f * W * H;
    if (dL_dalpha) af.dL_dalpha = dL_dalpha + (size_t)f * W * H;
    if (dL_dnormal_maps) {
      af.dL_dnormal = dL_dnormal_maps + (size_t)f * 3 * W * H;
      af.nrm_ws = (char*)nrm_ws + f * nrm_ws_stride;
    }
    if (dL_dmedian) af.dL_dmedian = dL_dmedian + (size_t)f * W * H;
    if (dL_ddistortion) af.dL_ddistortion = dL_ddistortion + (size_t)f * W * H;
    if (a.surf_ws) af.surf_ws = (char*)surf_ws + f * surf_ws_stride;
    if (dL_dmean2D_abs) af.dL_dmean2D_abs = dL_dmean2D_abs + (size_t)f * 3 * P;
    cudaStream_t fs = multi ? bs->lo[f & 1] : main_s;
    e = dgm::launch_render_bwd(af, fs);
    if (e == cudaSuccess && dL_dmedian) e = dgm::launch_median_grad(af, fs);
  }
  if (multi) {
    for (int i = 0; i < 2; ++i) {
      cudaEventRecord(bs->done_lo[i], bs->lo[i]);
      cudaStreamWaitEvent(main_s, bs->done_lo[i], 0);
    }
  }
  if (e == cudaSuccess) e = dgm::launch_preprocess_bwd(a, main_s);
  if (e == cudaSuccess && dL_dnormal_maps) e = dgm::launch_normal_grad_finish(a, main_s);
  return check(e != cudaSuccess ? e : cudaGetLastError());
}
}  // namespace

int dgr_backward_intr(int P, int D, int M, const float* background, int W, int H, const float* means3D,
                      const float* shs, const float* colors_precomp, const float* scales, float scale_modifier,
                      const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                      const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy, const int* radii,
                      void* geom_ws, void* binning_ws, int64_t R_cap, void* img_ws, const float* dL_dpix,
                      const float* dL_ddepth, const float* dL_dalpha, float* dL_dmean2D, float* dL_dconic,
                      float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                      float* dL_dscale, float* dL_drot, float* dL_dviewmatrix, float* dL_dprojmatrix,
                      float* dL_dcampos, void* cam_ws, size_t cam_ws_bytes, const float* dL_dnormal_map,
                      float* dL_dnormals, void* nrm_ws, float near_, float far_, const float* dL_dmedian,
                      const float* dL_ddistortion, void* surf_ws, float* dL_dmean2D_abs, float* dL_dtanfov,
                      void* stream) {
  if (P < 0 || W <= 0 || H <= 0 || R_cap < 0) return bad("dgr_backward: negative size");
  if (dL_dmedian || dL_ddistortion) {
    const int rc = surface_range(near_, far_);
    if (rc != DGM_OK) return rc;
    if (!surf_ws) return bad("dgr_backward_surf: surface workspace missing");
  }
  const int rc = camera_args(1, P, dL_dviewmatrix, dL_dprojmatrix, dL_dcampos, dL_dtanfov, cam_ws, cam_ws_bytes,
                             (cudaStream_t)stream);
  if (rc != DGM_OK) return rc;
  if (P == 0) return DGM_OK;
  if (dL_dnormal_map && !nrm_ws) return bad("dgr_backward_nrm: normal workspace missing");
  if (!background || !means3D || !viewmatrix || !projmatrix || !cam_pos || !geom_ws || !binning_ws || !img_ws ||
      !dL_dpix || !dL_dmean2D || !dL_dopacity || !dL_dcolor || !dL_dmean3D || !dL_dcov3D || !dL_dscale ||
      !dL_drot)
    return bad("dgr_backward: null required pointer");
  if (shs && !dL_dsh) return bad("dgr_backward: dL_dsh missing");
  return backward_frames(1, P, D, M, background, W, H, means3D, shs, colors_precomp, scales, scale_modifier, rotations,
                         cov3D_precomp, 0, viewmatrix, projmatrix, cam_pos, &tan_fovx, &tan_fovy, radii, geom_ws, 0,
                         binning_ws, 0, R_cap, img_ws, 0, dL_dpix, dL_ddepth, dL_dalpha, dL_dmean2D, dL_dconic,
                         dL_dopacity, dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, dL_dviewmatrix,
                         dL_dprojmatrix, dL_dcampos, cam_ws, dL_dnormal_map, 0, dL_dnormals, nrm_ws, 0, near_, far_,
                         dL_dmedian, dL_ddistortion, surf_ws, 0, dL_dmean2D_abs, dL_dtanfov, 1, stream);
}

int dgr_backward_abs(int P, int D, int M, const float* background, int W, int H, const float* means3D,
                     const float* shs, const float* colors_precomp, const float* scales, float scale_modifier,
                     const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                     const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy, const int* radii,
                     void* geom_ws, void* binning_ws, int64_t R_cap, void* img_ws, const float* dL_dpix,
                     const float* dL_ddepth, const float* dL_dalpha, float* dL_dmean2D, float* dL_dconic,
                     float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                     float* dL_dscale, float* dL_drot, float* dL_dviewmatrix, float* dL_dprojmatrix,
                     float* dL_dcampos, void* cam_ws, size_t cam_ws_bytes, const float* dL_dnormal_map,
                     float* dL_dnormals, void* nrm_ws, float near_, float far_, const float* dL_dmedian,
                     const float* dL_ddistortion, void* surf_ws, float* dL_dmean2D_abs, void* stream) {
  return dgr_backward_intr(P, D, M, background, W, H, means3D, shs, colors_precomp, scales, scale_modifier, rotations,
                           cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_ws,
                           binning_ws, R_cap, img_ws, dL_dpix, dL_ddepth, dL_dalpha, dL_dmean2D, dL_dconic,
                           dL_dopacity, dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, dL_dviewmatrix,
                           dL_dprojmatrix, dL_dcampos, cam_ws, cam_ws_bytes, dL_dnormal_map, dL_dnormals, nrm_ws,
                           near_, far_, dL_dmedian, dL_ddistortion, surf_ws, dL_dmean2D_abs, nullptr, stream);
}

int dgr_backward_surf(int P, int D, int M, const float* background, int W, int H, const float* means3D,
                      const float* shs, const float* colors_precomp, const float* scales, float scale_modifier,
                      const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                      const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy, const int* radii,
                      void* geom_ws, void* binning_ws, int64_t R_cap, void* img_ws, const float* dL_dpix,
                      const float* dL_ddepth, const float* dL_dalpha, float* dL_dmean2D, float* dL_dconic,
                      float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                      float* dL_dscale, float* dL_drot, float* dL_dviewmatrix, float* dL_dprojmatrix,
                      float* dL_dcampos, void* cam_ws, size_t cam_ws_bytes, const float* dL_dnormal_map,
                      float* dL_dnormals, void* nrm_ws, float near_, float far_, const float* dL_dmedian,
                      const float* dL_ddistortion, void* surf_ws, void* stream) {
  return dgr_backward_abs(P, D, M, background, W, H, means3D, shs, colors_precomp, scales, scale_modifier, rotations,
                          cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_ws,
                          binning_ws, R_cap, img_ws, dL_dpix, dL_ddepth, dL_dalpha, dL_dmean2D, dL_dconic,
                          dL_dopacity, dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, dL_dviewmatrix,
                          dL_dprojmatrix, dL_dcampos, cam_ws, cam_ws_bytes, dL_dnormal_map, dL_dnormals, nrm_ws,
                          near_, far_, dL_dmedian, dL_ddistortion, surf_ws, nullptr, stream);
}

int dgr_backward_nrm(int P, int D, int M, const float* background, int W, int H, const float* means3D,
                     const float* shs, const float* colors_precomp, const float* scales, float scale_modifier,
                     const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                     const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy, const int* radii,
                     void* geom_ws, void* binning_ws, int64_t R_cap, void* img_ws, const float* dL_dpix,
                     const float* dL_ddepth, const float* dL_dalpha, float* dL_dmean2D, float* dL_dconic,
                     float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                     float* dL_dscale, float* dL_drot, float* dL_dviewmatrix, float* dL_dprojmatrix,
                     float* dL_dcampos, void* cam_ws, size_t cam_ws_bytes, const float* dL_dnormal_map,
                     float* dL_dnormals, void* nrm_ws, void* stream) {
  return dgr_backward_surf(P, D, M, background, W, H, means3D, shs, colors_precomp, scales, scale_modifier,
                           rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii,
                           geom_ws, binning_ws, R_cap, img_ws, dL_dpix, dL_ddepth, dL_dalpha, dL_dmean2D, dL_dconic,
                           dL_dopacity, dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, dL_dviewmatrix,
                           dL_dprojmatrix, dL_dcampos, cam_ws, cam_ws_bytes, dL_dnormal_map, dL_dnormals, nrm_ws,
                           0.f, 0.f, nullptr, nullptr, nullptr, stream);
}

int dgr_backward_cam(int P, int D, int M, const float* background, int W, int H, const float* means3D,
                     const float* shs, const float* colors_precomp, const float* scales, float scale_modifier,
                     const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                     const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy, const int* radii,
                     void* geom_ws, void* binning_ws, int64_t R_cap, void* img_ws, const float* dL_dpix,
                     const float* dL_ddepth, const float* dL_dalpha, float* dL_dmean2D, float* dL_dconic,
                     float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                     float* dL_dscale, float* dL_drot, float* dL_dviewmatrix, float* dL_dprojmatrix,
                     float* dL_dcampos, void* cam_ws, size_t cam_ws_bytes, void* stream) {
  return dgr_backward_nrm(P, D, M, background, W, H, means3D, shs, colors_precomp, scales, scale_modifier, rotations,
                          cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_ws,
                          binning_ws, R_cap, img_ws, dL_dpix, dL_ddepth, dL_dalpha, dL_dmean2D, dL_dconic,
                          dL_dopacity, dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, dL_dviewmatrix,
                          dL_dprojmatrix, dL_dcampos, cam_ws, cam_ws_bytes, nullptr, nullptr, nullptr, stream);
}

int dgr_backward_aux(int P, int D, int M, const float* background, int W, int H, const float* means3D,
                     const float* shs, const float* colors_precomp, const float* scales, float scale_modifier,
                     const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                     const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy, const int* radii,
                     void* geom_ws, void* binning_ws, int64_t R_cap, void* img_ws, const float* dL_dpix,
                     const float* dL_ddepth, const float* dL_dalpha, float* dL_dmean2D, float* dL_dconic,
                     float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                     float* dL_dscale, float* dL_drot, void* stream) {
  return dgr_backward_cam(P, D, M, background, W, H, means3D, shs, colors_precomp, scales, scale_modifier, rotations,
                          cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_ws,
                          binning_ws, R_cap, img_ws, dL_dpix, dL_ddepth, dL_dalpha, dL_dmean2D, dL_dconic,
                          dL_dopacity, dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, nullptr, nullptr,
                          nullptr, nullptr, 0, stream);
}

int dgr_backward(int P, int D, int M, const float* background, int W, int H, const float* means3D, const float* shs,
                 const float* colors_precomp, const float* scales, float scale_modifier, const float* rotations,
                 const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                 float tan_fovx, float tan_fovy, const int* radii, void* geom_ws, void* binning_ws, int64_t R_cap,
                 void* img_ws, const float* dL_dpix, float* dL_dmean2D, float* dL_dconic, float* dL_dopacity,
                 float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale,
                 float* dL_drot, void* stream) {
  return dgr_backward_aux(P, D, M, background, W, H, means3D, shs, colors_precomp, scales, scale_modifier, rotations,
                          cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, radii, geom_ws,
                          binning_ws, R_cap, img_ws, dL_dpix, nullptr, nullptr, dL_dmean2D, dL_dconic, dL_dopacity,
                          dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, stream);
}

int dgr_backward_batch_intr(int F, int P, int D, int M, const float* background, int W, int H,
                            const float* means3D, const float* shs, const float* colors_precomp, const float* scales,
                            float scale_modifier, const float* rotations, const float* cov3D_precomp, int per_frame,
                            const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                            const float* tan_fovx_host, const float* tan_fovy_host, const int* radii, void* geom_ws,
                            size_t geom_stride, void* binning_ws, size_t binning_stride, int64_t R_cap, void* img_ws,
                            size_t img_stride, const float* dL_dpix, const float* dL_ddepth, const float* dL_dalpha,
                            float* dL_dmean2D, float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D,
                            float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dviewmatrix,
                            float* dL_dprojmatrix, float* dL_dcampos, void* cam_ws, size_t cam_ws_bytes,
                            const float* dL_dnormal_maps, int normals_per_frame, float* dL_dnormals, void* nrm_ws,
                            size_t nrm_ws_stride, float near_, float far_, const float* dL_dmedian,
                            const float* dL_ddistortion, void* surf_ws, size_t surf_ws_stride, float* dL_dmean2D_abs,
                            float* dL_dtanfov, int n_streams, void* stream) {
  if (F <= 0 || P < 0 || W <= 0 || H <= 0 || R_cap < 0) return bad("dgr_backward_batch: bad size");
  if (F > PB_MAX_FRAMES) return bad("dgr_backward_batch: more than 64 frames");
  const bool surf = dL_dmedian || dL_ddistortion;
  if (surf) {
    const int rc = surface_range(near_, far_);
    if (rc != DGM_OK) return rc;
    size_t need;
    dgr_surface_workspace_size(W, H, &need);
    if (!surf_ws || (surf_ws_stride & 127) || (F > 1 && surf_ws_stride < need))
      return bad("dgr_backward_batch_surf: surface workspace missing / stride too small or unaligned");
  }
  const int rc = camera_args(F, P, dL_dviewmatrix, dL_dprojmatrix, dL_dcampos, dL_dtanfov, cam_ws, cam_ws_bytes,
                             (cudaStream_t)stream);
  if (rc != DGM_OK) return rc;
  if (P == 0) return DGM_OK;
  if (dL_dnormal_maps && (!nrm_ws || (nrm_ws_stride & 127)))
    return bad("dgr_backward_batch_nrm: normal workspace missing / stride unaligned");
  if (!background || !means3D || !viewmatrices || !projmatrices || !cam_poses || !tan_fovx_host || !tan_fovy_host ||
      !geom_ws || !binning_ws || !img_ws || !dL_dpix || !dL_dmean2D || !dL_dopacity || (!shs && !dL_dcolor) ||
      !dL_dmean3D || (cov3D_precomp && !dL_dcov3D) || !dL_dscale || !dL_drot || (shs && !dL_dsh))
    return bad("dgr_backward_batch: null required pointer");
  return backward_frames(F, P, D, M, background, W, H, means3D, shs, colors_precomp, scales, scale_modifier, rotations,
                         cov3D_precomp, per_frame, viewmatrices, projmatrices, cam_poses, tan_fovx_host, tan_fovy_host,
                         radii, geom_ws, geom_stride, binning_ws, binning_stride, R_cap, img_ws, img_stride, dL_dpix,
                         dL_ddepth, dL_dalpha, dL_dmean2D, nullptr, dL_dopacity, dL_dcolor, dL_dmean3D, dL_dcov3D,
                         dL_dsh, dL_dscale, dL_drot, dL_dviewmatrix, dL_dprojmatrix, dL_dcampos, cam_ws,
                         dL_dnormal_maps, normals_per_frame, dL_dnormals, nrm_ws, nrm_ws_stride, near_, far_,
                         dL_dmedian, dL_ddistortion, surf_ws, surf_ws_stride, dL_dmean2D_abs, dL_dtanfov, n_streams,
                         stream);
}

int dgr_backward_batch_abs(int F, int P, int D, int M, const float* background, int W, int H,
                           const float* means3D, const float* shs, const float* colors_precomp, const float* scales,
                           float scale_modifier, const float* rotations, const float* cov3D_precomp, int per_frame,
                           const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                           const float* tan_fovx_host, const float* tan_fovy_host, const int* radii, void* geom_ws,
                           size_t geom_stride, void* binning_ws, size_t binning_stride, int64_t R_cap, void* img_ws,
                           size_t img_stride, const float* dL_dpix, const float* dL_ddepth, const float* dL_dalpha,
                           float* dL_dmean2D, float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D,
                           float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dviewmatrix,
                           float* dL_dprojmatrix, float* dL_dcampos, void* cam_ws, size_t cam_ws_bytes,
                           const float* dL_dnormal_maps, int normals_per_frame, float* dL_dnormals, void* nrm_ws,
                           size_t nrm_ws_stride, float near_, float far_, const float* dL_dmedian,
                           const float* dL_ddistortion, void* surf_ws, size_t surf_ws_stride, float* dL_dmean2D_abs,
                           int n_streams, void* stream) {
  return dgr_backward_batch_intr(F, P, D, M, background, W, H, means3D, shs, colors_precomp, scales, scale_modifier,
                                 rotations, cov3D_precomp, per_frame, viewmatrices, projmatrices, cam_poses,
                                 tan_fovx_host, tan_fovy_host, radii, geom_ws, geom_stride, binning_ws,
                                 binning_stride, R_cap, img_ws, img_stride, dL_dpix, dL_ddepth, dL_dalpha, dL_dmean2D,
                                 dL_dopacity, dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot,
                                 dL_dviewmatrix, dL_dprojmatrix, dL_dcampos, cam_ws, cam_ws_bytes, dL_dnormal_maps,
                                 normals_per_frame, dL_dnormals, nrm_ws, nrm_ws_stride, near_, far_, dL_dmedian,
                                 dL_ddistortion, surf_ws, surf_ws_stride, dL_dmean2D_abs, nullptr, n_streams, stream);
}

int dgr_backward_batch_surf(int F, int P, int D, int M, const float* background, int W, int H,
                            const float* means3D, const float* shs, const float* colors_precomp, const float* scales,
                            float scale_modifier, const float* rotations, const float* cov3D_precomp, int per_frame,
                            const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                            const float* tan_fovx_host, const float* tan_fovy_host, const int* radii, void* geom_ws,
                            size_t geom_stride, void* binning_ws, size_t binning_stride, int64_t R_cap, void* img_ws,
                            size_t img_stride, const float* dL_dpix, const float* dL_ddepth, const float* dL_dalpha,
                            float* dL_dmean2D, float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D,
                            float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dviewmatrix,
                            float* dL_dprojmatrix, float* dL_dcampos, void* cam_ws, size_t cam_ws_bytes,
                            const float* dL_dnormal_maps, int normals_per_frame, float* dL_dnormals, void* nrm_ws,
                            size_t nrm_ws_stride, float near_, float far_, const float* dL_dmedian,
                            const float* dL_ddistortion, void* surf_ws, size_t surf_ws_stride, int n_streams,
                            void* stream) {
  return dgr_backward_batch_abs(F, P, D, M, background, W, H, means3D, shs, colors_precomp, scales, scale_modifier,
                                rotations, cov3D_precomp, per_frame, viewmatrices, projmatrices, cam_poses,
                                tan_fovx_host, tan_fovy_host, radii, geom_ws, geom_stride, binning_ws,
                                binning_stride, R_cap, img_ws, img_stride, dL_dpix, dL_ddepth, dL_dalpha, dL_dmean2D,
                                dL_dopacity, dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot,
                                dL_dviewmatrix, dL_dprojmatrix, dL_dcampos, cam_ws, cam_ws_bytes, dL_dnormal_maps,
                                normals_per_frame, dL_dnormals, nrm_ws, nrm_ws_stride, near_, far_, dL_dmedian,
                                dL_ddistortion, surf_ws, surf_ws_stride, nullptr, n_streams, stream);
}

int dgr_backward_batch_nrm(int F, int P, int D, int M, const float* background, int W, int H, const float* means3D,
                           const float* shs, const float* colors_precomp, const float* scales, float scale_modifier,
                           const float* rotations, const float* cov3D_precomp, int per_frame,
                           const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                           const float* tan_fovx_host, const float* tan_fovy_host, const int* radii, void* geom_ws,
                           size_t geom_stride, void* binning_ws, size_t binning_stride, int64_t R_cap, void* img_ws,
                           size_t img_stride, const float* dL_dpix, const float* dL_ddepth, const float* dL_dalpha,
                           float* dL_dmean2D, float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D,
                           float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dviewmatrix,
                           float* dL_dprojmatrix, float* dL_dcampos, void* cam_ws, size_t cam_ws_bytes,
                           const float* dL_dnormal_maps, int normals_per_frame, float* dL_dnormals, void* nrm_ws,
                           size_t nrm_ws_stride, int n_streams, void* stream) {
  return dgr_backward_batch_surf(F, P, D, M, background, W, H, means3D, shs, colors_precomp, scales, scale_modifier,
                                 rotations, cov3D_precomp, per_frame, viewmatrices, projmatrices, cam_poses,
                                 tan_fovx_host, tan_fovy_host, radii, geom_ws, geom_stride, binning_ws,
                                 binning_stride, R_cap, img_ws, img_stride, dL_dpix, dL_ddepth, dL_dalpha,
                                 dL_dmean2D, dL_dopacity, dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale,
                                 dL_drot, dL_dviewmatrix, dL_dprojmatrix, dL_dcampos, cam_ws, cam_ws_bytes,
                                 dL_dnormal_maps, normals_per_frame, dL_dnormals, nrm_ws, nrm_ws_stride, 0.f, 0.f,
                                 nullptr, nullptr, nullptr, 0, n_streams, stream);
}

int dgr_backward_batch_cam(int F, int P, int D, int M, const float* background, int W, int H, const float* means3D,
                           const float* shs, const float* colors_precomp, const float* scales, float scale_modifier,
                           const float* rotations, const float* cov3D_precomp, int per_frame,
                           const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                           const float* tan_fovx_host, const float* tan_fovy_host, const int* radii, void* geom_ws,
                           size_t geom_stride, void* binning_ws, size_t binning_stride, int64_t R_cap, void* img_ws,
                           size_t img_stride, const float* dL_dpix, const float* dL_ddepth, const float* dL_dalpha,
                           float* dL_dmean2D, float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D,
                           float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dviewmatrix,
                           float* dL_dprojmatrix, float* dL_dcampos, void* cam_ws, size_t cam_ws_bytes, int n_streams,
                           void* stream) {
  return dgr_backward_batch_nrm(F, P, D, M, background, W, H, means3D, shs, colors_precomp, scales, scale_modifier,
                                rotations, cov3D_precomp, per_frame, viewmatrices, projmatrices, cam_poses,
                                tan_fovx_host, tan_fovy_host, radii, geom_ws, geom_stride, binning_ws, binning_stride,
                                R_cap, img_ws, img_stride, dL_dpix, dL_ddepth, dL_dalpha, dL_dmean2D, dL_dopacity,
                                dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, dL_dviewmatrix,
                                dL_dprojmatrix, dL_dcampos, cam_ws, cam_ws_bytes, nullptr, 0, nullptr, nullptr, 0,
                                n_streams, stream);
}

int dgr_backward_batch_aux(int F, int P, int D, int M, const float* background, int W, int H, const float* means3D,
                           const float* shs, const float* colors_precomp, const float* scales, float scale_modifier,
                           const float* rotations, const float* cov3D_precomp, int per_frame,
                           const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                           const float* tan_fovx_host, const float* tan_fovy_host, const int* radii, void* geom_ws,
                           size_t geom_stride, void* binning_ws, size_t binning_stride, int64_t R_cap, void* img_ws,
                           size_t img_stride, const float* dL_dpix, const float* dL_ddepth, const float* dL_dalpha,
                           float* dL_dmean2D, float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D,
                           float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot, int n_streams,
                           void* stream) {
  return dgr_backward_batch_cam(F, P, D, M, background, W, H, means3D, shs, colors_precomp, scales, scale_modifier,
                                rotations, cov3D_precomp, per_frame, viewmatrices, projmatrices, cam_poses,
                                tan_fovx_host, tan_fovy_host, radii, geom_ws, geom_stride, binning_ws, binning_stride,
                                R_cap, img_ws, img_stride, dL_dpix, dL_ddepth, dL_dalpha, dL_dmean2D, dL_dopacity,
                                dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, nullptr, nullptr,
                                nullptr, nullptr, 0, n_streams, stream);
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
  return dgr_backward_batch_aux(F, P, D, M, background, W, H, means3D, shs, colors_precomp, scales, scale_modifier,
                                rotations, cov3D_precomp, per_frame, viewmatrices, projmatrices, cam_poses,
                                tan_fovx_host, tan_fovy_host, radii, geom_ws, geom_stride, binning_ws,
                                binning_stride, R_cap, img_ws, img_stride, dL_dpix, nullptr, nullptr, dL_dmean2D,
                                dL_dopacity, dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot,
                                n_streams, stream);
}

int dgr_feature_workspace_size(int P, int C, int F, size_t* bytes) {
  if (P < 0 || C < 1 || C > 64 || F < 1 || F > PB_MAX_FRAMES || !bytes)
    return bad("dgr_feature_workspace_size: bad argument");
  *bytes = (size_t)F * dgm::feature_ws_stride(P, C);
  return DGM_OK;
}

namespace {
// The workspaces of F frames an earlier forward wrote, as a side-pass entry point (who) takes them: DGM_OK with ws
// filled in, or the error to return (nothing is launched).  The pass's own pointers are checked with them (own_ptrs:
// none is NULL).  max_F: PB_MAX_FRAMES for the passes whose workspaces are sized per frame, 65535 (grid.y) for
// blend statistics, which reads no geometry workspace (geom false: geom_ws and geom_stride are not checked).
int forward_ws_args(const char* who, int max_F, bool geom, int F, int P, int W, int H, void* geom_ws,
                    size_t geom_stride, void* binning_ws, size_t binning_stride, int64_t R_cap, void* img_ws,
                    size_t img_stride, bool own_ptrs, dgm::ForwardWS& ws) {
  char msg[128];
  if (F < 1 || F > max_F || P < 0 || W <= 0 || H <= 0 || R_cap < 0)
    return snprintf(msg, sizeof(msg), "%s: bad size", who), bad(msg);
  if ((geom && !geom_ws) || !binning_ws || !img_ws || !own_ptrs)
    return snprintf(msg, sizeof(msg), "%s: null pointer", who), bad(msg);
  if (F > 1) {
    size_t gb, bb, ib;
    dgr_workspace_sizes(P, W, H, R_cap, &gb, &bb, &ib);
    if ((geom && (geom_stride < gb || geom_stride % 128)) || binning_stride < bb || img_stride < ib ||
        binning_stride % 128 || img_stride % 128)
      return snprintf(msg, sizeof(msg), "%s: workspace stride too small or not a multiple of 128", who), bad(msg);
  }
  ws.F = F, ws.P = P, ws.W = W, ws.H = H;
  ws.geom_ws = geom_ws, ws.binning_ws = binning_ws, ws.img_ws = img_ws;
  ws.geom_stride = F > 1 ? geom_stride : 0, ws.binning_stride = F > 1 ? binning_stride : 0;
  ws.img_stride = F > 1 ? img_stride : 0;
  ws.R_cap = R_cap;
  return DGM_OK;
}

// the arguments shared by dgr_features_fwd / _bwd: DGM_OK, or the error to return (nothing is launched)
int feature_args(const char* who, int F, int P, int C, int W, int H, const float* features, int per_frame,
                 void* geom_ws, size_t geom_stride, void* binning_ws, size_t binning_stride, int64_t R_cap,
                 void* img_ws, size_t img_stride, void* feat_ws, size_t feat_ws_bytes, dgm::FeatArgs& a) {
  char msg[128];
  if (C < 1 || C > 64) return snprintf(msg, sizeof(msg), "%s: need 1 <= C <= 64", who), bad(msg);
  a = {};
  const int rc = forward_ws_args(who, PB_MAX_FRAMES, true, F, P, W, H, geom_ws, geom_stride, binning_ws,
                                 binning_stride, R_cap, img_ws, img_stride, features && feat_ws, a);
  if (rc != DGM_OK) return rc;
  if (reinterpret_cast<uintptr_t>(feat_ws) % 16) return snprintf(msg, sizeof(msg), "%s: misaligned workspace", who), bad(msg);
  size_t need;
  dgr_feature_workspace_size(P, C, F, &need);
  if (feat_ws_bytes < need) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: feature workspace too small", who);
    return DGM_E_WORKSPACE;
  }
  a.C = C, a.features = features, a.per_frame = per_frame ? 1 : 0, a.feat_ws = feat_ws;
  return DGM_OK;
}
}  // namespace

int dgr_features_fwd(int F, int P, int C, int W, int H, const float* features, int features_per_frame, void* geom_ws,
                     size_t geom_stride, void* binning_ws, size_t binning_stride, int64_t R_cap, void* img_ws,
                     size_t img_stride, float* out_map, void* feat_ws, size_t feat_ws_bytes, void* stream) {
  dgm::FeatArgs a;
  const int rc = feature_args("dgr_features_fwd", F, P, C, W, H, features, features_per_frame, geom_ws, geom_stride,
                              binning_ws, binning_stride, R_cap, img_ws, img_stride, feat_ws, feat_ws_bytes, a);
  if (rc != DGM_OK) return rc;
  if (!out_map) return bad("dgr_features_fwd: null pointer");
  a.out_map = out_map;
  return check(dgm::launch_features_fwd(a, (cudaStream_t)stream));
}

int dgr_features_bwd(int F, int P, int C, int W, int H, const float* features, int features_per_frame, void* geom_ws,
                     size_t geom_stride, void* binning_ws, size_t binning_stride, int64_t R_cap, void* img_ws,
                     size_t img_stride, const float* map, const float* dL_dmap, float* dL_dfeatures, void* feat_ws,
                     size_t feat_ws_bytes, void* stream) {
  dgm::FeatArgs a;
  const int rc = feature_args("dgr_features_bwd", F, P, C, W, H, features, features_per_frame, geom_ws, geom_stride,
                              binning_ws, binning_stride, R_cap, img_ws, img_stride, feat_ws, feat_ws_bytes, a);
  if (rc != DGM_OK) return rc;
  if (!map || !dL_dmap) return bad("dgr_features_bwd: null pointer");
  a.map = map, a.dL_dmap = dL_dmap, a.dL_dfeatures = dL_dfeatures;
  return check(dgm::launch_features_bwd(a, (cudaStream_t)stream));
}

namespace {
// the arguments shared by dgr_gaussian_planes_fwd / _bwd: DGM_OK or DGM_E_BADARG (nothing is launched)
int plane_args(const char* who, int F, int P, int W, int H, const float* means3D, const float* scales,
               const float* rotations, const float* cov3D_precomp, int per_frame, const float* view,
               const float* tanx, const float* tany, dgm::PlaneArgs& a) {
  char msg[128];
  if (F < 1 || F > PB_MAX_FRAMES || P < 0 || W <= 0 || H <= 0 || (per_frame & ~DGR_PF_ALL))
    return snprintf(msg, sizeof(msg), "%s: bad size", who), bad(msg);
  if (!means3D || !view || !tanx || !tany || (cov3D_precomp ? (scales || rotations) : (!scales || !rotations)))
    return snprintf(msg, sizeof(msg), "%s: null pointer (or both scales / rotations and cov3D_precomp)", who), bad(msg);
  for (int f = 0; f < F; ++f)
    if (!(tanx[f] > 0.0f) || !(tany[f] > 0.0f)) return snprintf(msg, sizeof(msg), "%s: bad tan_fov", who), bad(msg);
  a = {};
  a.F = F, a.P = P, a.W = W, a.H = H;
  a.means3D = means3D, a.scales = scales, a.rotations = rotations, a.cov3D_precomp = cov3D_precomp;
  a.per_frame = per_frame, a.viewmatrix = view;
  for (int f = 0; f < F; ++f) a.cams.tanx[f] = tanx[f], a.cams.tany[f] = tany[f];
  return DGM_OK;
}

// the arguments shared by dgr_planar_fwd / _bwd (as feature_args)
int planar_args(const char* who, int F, int P, int W, int H, const float* planes, void* geom_ws, size_t geom_stride,
                void* binning_ws, size_t binning_stride, int64_t R_cap, void* img_ws, size_t img_stride,
                void* planar_ws, size_t planar_ws_bytes, dgm::PlanarArgs& a) {
  char msg[128];
  a = {};
  const int rc = forward_ws_args(who, PB_MAX_FRAMES, true, F, P, W, H, geom_ws, geom_stride, binning_ws,
                                 binning_stride, R_cap, img_ws, img_stride, planes && planar_ws, a);
  if (rc != DGM_OK) return rc;
  if (reinterpret_cast<uintptr_t>(planar_ws) % 16)
    return snprintf(msg, sizeof(msg), "%s: misaligned workspace", who), bad(msg);
  size_t need;
  dgr_planar_workspace_size(P, W, H, F, &need);
  if (planar_ws_bytes < need) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: planar workspace too small", who);
    return DGM_E_WORKSPACE;
  }
  a.planes = planes, a.planar_ws = planar_ws;
  return DGM_OK;
}
}  // namespace

int dgr_gaussian_planes_fwd(int F, int P, int W, int H, const float* means3D, const float* scales,
                            float scale_modifier, const float* rotations, const float* cov3D_precomp, int per_frame,
                            const float* viewmatrices, const float* tan_fovx_host, const float* tan_fovy_host,
                            float* planes, float* normals, void* stream) {
  dgm::PlaneArgs a;
  const int rc = plane_args("dgr_gaussian_planes_fwd", F, P, W, H, means3D, scales, rotations, cov3D_precomp,
                            per_frame, viewmatrices, tan_fovx_host, tan_fovy_host, a);
  if (rc != DGM_OK) return rc;
  if (!planes || !normals) return bad("dgr_gaussian_planes_fwd: null pointer");
  a.scale_modifier = scale_modifier, a.planes = planes, a.normals = normals;
  return check(dgm::launch_gaussian_planes_fwd(a, (cudaStream_t)stream));
}

int dgr_gaussian_planes_bwd(int F, int P, int W, int H, const float* means3D, const float* scales,
                            float scale_modifier, const float* rotations, const float* cov3D_precomp, int per_frame,
                            const float* viewmatrices, const float* tan_fovx_host, const float* tan_fovy_host,
                            const float* dL_dplanes, const float* dL_dnormals, float* dL_dmeans3D,
                            float* dL_dscales, float* dL_drotations, float* dL_dcov3D_precomp, void* stream) {
  dgm::PlaneArgs a;
  const int rc = plane_args("dgr_gaussian_planes_bwd", F, P, W, H, means3D, scales, rotations, cov3D_precomp,
                            per_frame, viewmatrices, tan_fovx_host, tan_fovy_host, a);
  if (rc != DGM_OK) return rc;
  a.scale_modifier = scale_modifier, a.dL_dplanes = dL_dplanes, a.dL_dnormals = dL_dnormals;
  a.dL_dmeans3D = dL_dmeans3D, a.dL_dscales = dL_dscales, a.dL_drotations = dL_drotations;
  a.dL_dcov3D = dL_dcov3D_precomp;
  return check(dgm::launch_gaussian_planes_bwd(a, (cudaStream_t)stream));
}

int dgr_planar_workspace_size(int P, int W, int H, int F, size_t* bytes) {
  if (P < 0 || W <= 0 || H <= 0 || F < 1 || F > PB_MAX_FRAMES || !bytes)
    return bad("dgr_planar_workspace_size: bad argument");
  *bytes = (size_t)F * dgm::planar_ws_stride(P, W, H);
  return DGM_OK;
}

int dgr_planar_fwd(int F, int P, int W, int H, const float* planes, void* geom_ws, size_t geom_stride,
                   void* binning_ws, size_t binning_stride, int64_t R_cap, void* img_ws, size_t img_stride,
                   float* planar_depth, float* planar_median, void* planar_ws, size_t planar_ws_bytes, void* stream) {
  dgm::PlanarArgs a;
  const int rc = planar_args("dgr_planar_fwd", F, P, W, H, planes, geom_ws, geom_stride, binning_ws, binning_stride,
                             R_cap, img_ws, img_stride, planar_ws, planar_ws_bytes, a);
  if (rc != DGM_OK) return rc;
  if (!planar_depth || !planar_median) return bad("dgr_planar_fwd: null pointer");
  a.out_depth = planar_depth, a.out_median = planar_median;
  return check(dgm::launch_planar_fwd(a, (cudaStream_t)stream));
}

int dgr_planar_bwd(int F, int P, int W, int H, const float* planes, void* geom_ws, size_t geom_stride,
                   void* binning_ws, size_t binning_stride, int64_t R_cap, void* img_ws, size_t img_stride,
                   const float* planar_depth, const float* dL_dplanar_depth, const float* dL_dplanar_median,
                   float* dL_dplanes, void* planar_ws, size_t planar_ws_bytes, void* stream) {
  dgm::PlanarArgs a;
  const int rc = planar_args("dgr_planar_bwd", F, P, W, H, planes, geom_ws, geom_stride, binning_ws, binning_stride,
                             R_cap, img_ws, img_stride, planar_ws, planar_ws_bytes, a);
  if (rc != DGM_OK) return rc;
  if (dL_dplanar_depth && !planar_depth) return bad("dgr_planar_bwd: null pointer");
  a.depth = planar_depth, a.dL_ddepth = dL_dplanar_depth, a.dL_dmedian = dL_dplanar_median;
  a.dL_dplanes = dL_dplanes;
  return check(dgm::launch_planar_bwd(a, (cudaStream_t)stream));
}

int dgr_blend_stats(int F, int P, int W, int H, void* binning_ws, size_t binning_stride, int64_t R_cap,
                    void* img_ws, size_t img_stride, const float* pixel_weights, int weights_per_frame,
                    float* out_sum, float* out_max, void* stream) {
  dgm::StatsArgs a = {};
  // grid.y counts the frames and is limited to 65535
  const int rc = forward_ws_args("dgr_blend_stats", 65535, false, F, P, W, H, nullptr, 0, binning_ws, binning_stride,
                                 R_cap, img_ws, img_stride, out_sum && out_max, a);
  if (rc != DGM_OK) return rc;
  a.pixel_weights = pixel_weights, a.weights_per_frame = (pixel_weights && weights_per_frame) ? 1 : 0;
  a.out_sum = out_sum, a.out_max = out_max;
  return check(dgm::launch_blend_stats(a, (cudaStream_t)stream));
}

namespace {
// the arguments shared by dgr_depth_normal_fwd / _bwd: DGM_OK, or the error to return (nothing is launched)
int depth_normal_args(const char* who, int F, int W, int H, float depth_ratio, const float* depth, const float* alpha,
                      const float* median, const float* coefs_host) {
  char msg[128];
  // grid.y counts 16-row tiles and is limited to 65535
  if (F < 1 || W < 1 || H < 1 || H > 65535 * 16) return snprintf(msg, sizeof(msg), "%s: bad size", who), bad(msg);
  if (!(depth_ratio >= 0.0f && depth_ratio <= 1.0f))
    return snprintf(msg, sizeof(msg), "%s: need 0 <= depth_ratio <= 1", who), bad(msg);
  if (!coefs_host || (depth_ratio < 1.0f && (!depth || !alpha)) || (depth_ratio > 0.0f && !median))
    return snprintf(msg, sizeof(msg), "%s: null pointer", who), bad(msg);
  return DGM_OK;
}
}  // namespace

int dgr_depth_normal_fwd(int F, int W, int H, float depth_ratio, const float* depth, const float* alpha,
                         const float* median, const float* coefs_host, float* out_normal, void* stream) {
  const int rc = depth_normal_args("dgr_depth_normal_fwd", F, W, H, depth_ratio, depth, alpha, median, coefs_host);
  if (rc != DGM_OK) return rc;
  if (!out_normal) return bad("dgr_depth_normal_fwd: null pointer");
  return check(dgm::launch_depth_normal_fwd(F, W, H, depth_ratio, depth, alpha, median, coefs_host, out_normal,
                                            (cudaStream_t)stream));
}

int dgr_depth_normal_bwd(int F, int W, int H, float depth_ratio, const float* depth, const float* alpha,
                         const float* median, const float* coefs_host, const float* dL_dnormal, float* dL_ddepth,
                         float* dL_dalpha, float* dL_dmedian, void* stream) {
  const int rc = depth_normal_args("dgr_depth_normal_bwd", F, W, H, depth_ratio, depth, alpha, median, coefs_host);
  if (rc != DGM_OK) return rc;
  if (!dL_dnormal) return bad("dgr_depth_normal_bwd: null pointer");
  if ((depth_ratio == 1.0f && (dL_ddepth || dL_dalpha)) || (depth_ratio == 0.0f && dL_dmedian))
    return bad("dgr_depth_normal_bwd: a gradient of a map depth_ratio does not read must be NULL");
  if (!dL_ddepth && !dL_dalpha && !dL_dmedian) return DGM_OK;
  return check(dgm::launch_depth_normal_bwd(F, W, H, depth_ratio, depth, alpha, median, coefs_host, dL_dnormal,
                                            dL_ddepth, dL_dalpha, dL_dmedian, (cudaStream_t)stream));
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
  return check(dgm::launch_nearest(1, Q, queries, R, refs, dist2, (long long*)index, (cudaStream_t)stream));
}

int dgp_plan_create(int G, void** plan, size_t* ws_bytes) {
  if (G < 4 || (G & 1) || !plan) return bad("dgp_plan_create: G must be even and >= 4");
  size_t work = 0;
  if (dgm::dpsr_plan_create(G, plan, &work) != 0) {
    strncpy(g_last_error, "dgp_plan_create: cuFFT plan creation failed", sizeof(g_last_error) - 1);
    return DGM_E_LAUNCH;
  }
  if (ws_bytes) dgm::DpsrWS::from(nullptr, G, work, 1, ws_bytes);
  return DGM_OK;
}

int dgp_plan_destroy(void* plan) {
  dgm::dpsr_plan_destroy(plan);
  return DGM_OK;
}

int dgp_batch_workspace_size(void* plan, int B, size_t* bytes) {
  if (!plan || !bytes) return bad("dgp_batch_workspace_size: null plan / bytes");
  if (B < 1 || B > dgm::DPSR_MAX_BATCH) return bad("dgp_batch_workspace_size: B out of range (1 <= B <= 64)");
  dgm::DpsrWS::from(nullptr, dgm::dpsr_plan_res(plan), dgm::dpsr_plan_work(plan), B, bytes);
  return DGM_OK;
}

static int dgp_check(const char* fn, void* plan, int B, size_t ws_bytes, void* ws) {
  char msg[160];
  if (!plan || !ws) {
    snprintf(msg, sizeof(msg), "%s: null plan / workspace", fn);
    return bad(msg);
  }
  if (B < 1 || B > dgm::DPSR_MAX_BATCH) {
    snprintf(msg, sizeof(msg), "%s: B out of range (1 <= B <= 64)", fn);
    return bad(msg);
  }
  size_t need;
  dgm::DpsrWS::from(nullptr, dgm::dpsr_plan_res(plan), dgm::dpsr_plan_work(plan), B, &need);
  if (ws_bytes < need) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: workspace too small", fn);
    return DGM_E_WORKSPACE;
  }
  return DGM_OK;
}

int dgp_forward_batch(void* plan, int B, int N, double sig, const float* V, const float* Nrm, int mode,
                      const float* thres, float* out, void* ws, size_t ws_bytes, void* stream) {
  int rc = dgp_check("dgp_forward_batch", plan, B, ws_bytes, ws);
  if (rc != DGM_OK) return rc;
  if (N < 0 || !out || (N > 0 && (!V || !Nrm)) || (mode && !thres)) return bad("dgp_forward_batch: bad argument");
  return check(dgm::launch_dpsr_forward(plan, B, N, sig, V, Nrm, mode, thres, out, ws, (cudaStream_t)stream));
}

int dgp_backward_batch(void* plan, int B, int N, const float* V, const float* Nrm, int mode, const float* dL_dout,
                       float* dV, float* dN, float* dthres, void* ws, size_t ws_bytes, void* stream) {
  int rc = dgp_check("dgp_backward_batch", plan, B, ws_bytes, ws);
  if (rc != DGM_OK) return rc;
  if (N < 0 || !dL_dout || (N > 0 && (!V || !Nrm || !dV || !dN))) return bad("dgp_backward_batch: bad argument");
  return check(dgm::launch_dpsr_backward(plan, B, N, V, Nrm, mode, dL_dout, dV, dN, dthres, ws,
                                         (cudaStream_t)stream));
}

int dgp_forward(void* plan, int N, double sig, const float* V, const float* Nrm, int mode, const float* thres,
                float* out, void* ws, size_t ws_bytes, void* stream) {
  int rc = dgp_check("dpsr", plan, 1, ws_bytes, ws);
  if (rc != DGM_OK) return rc;
  if (N < 0 || !out || (N > 0 && (!V || !Nrm)) || (mode && !thres)) return bad("dgp_forward: bad argument");
  return check(dgm::launch_dpsr_forward(plan, 1, N, sig, V, Nrm, mode, thres, out, ws, (cudaStream_t)stream));
}

int dgp_backward(void* plan, int N, const float* V, const float* Nrm, int mode, const float* dL_dout, float* dV,
                 float* dN, float* dthres, void* ws, size_t ws_bytes, void* stream) {
  int rc = dgp_check("dpsr", plan, 1, ws_bytes, ws);
  if (rc != DGM_OK) return rc;
  if (N < 0 || !dL_dout || (N > 0 && (!V || !Nrm || !dV || !dN))) return bad("dgp_backward: bad argument");
  return check(dgm::launch_dpsr_backward(plan, 1, N, V, Nrm, mode, dL_dout, dV, dN, dthres, ws, (cudaStream_t)stream));
}

int dgmc_workspace_size(int G, size_t* bytes) {
  if (G < 2 || G > 800 || !bytes) return bad("dgmc_workspace_size: bad argument (2 <= G <= 800)");
  dgm::McWS::from(nullptr, G, 1, bytes);
  return DGM_OK;
}

int dgmc_workspace_size_batch(int B, int G, size_t* bytes) {
  if (B < 1 || B > dgm::MC_MAX_BATCH) return bad("dgmc_workspace_size_batch: B out of range (1 <= B <= 64)");
  if (G < 2 || G > 800 || !bytes) return bad("dgmc_workspace_size_batch: bad argument (2 <= G <= 800)");
  dgm::McWS::from(nullptr, G, B, bytes);
  return DGM_OK;
}

static int dgmc_check(const char* fn, int B, int G, const float* phi, void* ws, size_t ws_bytes) {
  char msg[160];
  if (B < 1 || B > dgm::MC_MAX_BATCH) {
    snprintf(msg, sizeof(msg), "%s: B out of range (1 <= B <= 64)", fn);
    return bad(msg);
  }
  if (G < 2 || G > 800 || !phi || !ws) {
    snprintf(msg, sizeof(msg), "%s: bad argument (2 <= G <= 800)", fn);
    return bad(msg);
  }
  size_t need;
  dgm::McWS::from(nullptr, G, B, &need);
  if (ws_bytes < need) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: workspace too small", fn);
    return DGM_E_WORKSPACE;
  }
  return DGM_OK;
}

static int dgmc_count_call(const char* fn, int B, int G, const float* phi, float iso, void* ws, size_t ws_bytes,
                           int32_t* totals, int32_t* totals_host, void* totals_event, void* stream) {
  int rc = dgmc_check(fn, B, G, phi, ws, ws_bytes);
  if (rc != DGM_OK) return rc;
  if (!totals) return bad(B == 1 ? "dgmc_count: null totals" : "dgmc_count_batch: null totals");
  return check(dgm::launch_mc_count(B, G, phi, iso, ws, totals, totals_host, (cudaEvent_t)totals_event,
                                    (cudaStream_t)stream));
}

int dgmc_count(int G, const float* phi, float iso, void* ws, size_t ws_bytes, int32_t* totals, int32_t* totals_host,
               void* totals_event, void* stream) {
  return dgmc_count_call("marching cubes", 1, G, phi, iso, ws, ws_bytes, totals, totals_host, totals_event, stream);
}

int dgmc_count_batch(int B, int G, const float* phi, float iso, void* ws, size_t ws_bytes, int32_t* totals,
                     int32_t* totals_host, void* totals_event, void* stream) {
  return dgmc_count_call("dgmc_count_batch", B, G, phi, iso, ws, ws_bytes, totals, totals_host, totals_event,
                         stream);
}

static int dgmc_emit_call(const char* fn, int B, int G, const float* phi, float iso, void* ws, size_t ws_bytes,
                          float* verts, int32_t* vsrc, int64_t V_cap, int32_t* faces, int64_t F_cap, void* stream) {
  char msg[160];
  // vertex indices are packed into 29 bits and face counts are int32: larger capacities could never be filled
  if (V_cap < 0 || V_cap > dgm::MC_MAX_VERTS || F_cap < 0 || F_cap > INT32_MAX) {
    snprintf(msg, sizeof(msg), "%s: capacity out of range (V_cap <= 2^29, F_cap < 2^31)", fn);
    return bad(msg);
  }
  if ((V_cap > 0 && (!verts || !vsrc)) || (F_cap > 0 && !faces)) {
    snprintf(msg, sizeof(msg), "%s: null output", fn);
    return bad(msg);
  }
  int rc = dgmc_check(B == 1 ? "marching cubes" : fn, B, G, phi, ws, ws_bytes);
  if (rc != DGM_OK) return rc;
  return check(dgm::launch_mc_emit(B, G, phi, iso, ws, verts, vsrc, V_cap, faces, F_cap, (cudaStream_t)stream));
}

int dgmc_emit(int G, const float* phi, float iso, void* ws, size_t ws_bytes, float* verts, int32_t* vsrc,
              int64_t V_cap, int32_t* faces, int64_t F_cap, void* stream) {
  return dgmc_emit_call("dgmc_emit", 1, G, phi, iso, ws, ws_bytes, verts, vsrc, V_cap, faces, F_cap, stream);
}

int dgmc_emit_batch(int B, int G, const float* phi, float iso, void* ws, size_t ws_bytes, float* verts,
                    int32_t* vsrc, int64_t V_cap, int32_t* faces, int64_t F_cap, void* stream) {
  return dgmc_emit_call("dgmc_emit_batch", B, G, phi, iso, ws, ws_bytes, verts, vsrc, V_cap, faces, F_cap, stream);
}

// V_host[B]: each item's vertex count (from dgmc_count / dgmc_count_batch)
static int dgmc_backward_call(const char* fn, int B, int G, const int32_t* V_host, const float* phi, float iso,
                              const int32_t* vsrc, const float* dL_dverts, float* dL_dphi, void* stream) {
  char msg[160];
  if (B < 1 || B > dgm::MC_MAX_BATCH) {
    snprintf(msg, sizeof(msg), "%s: B out of range (1 <= B <= 64)", fn);
    return bad(msg);
  }
  if (G < 2 || G > 800 || !phi || !dL_dphi || !V_host) {
    snprintf(msg, sizeof(msg), "%s: bad argument (2 <= G <= 800)", fn);
    return bad(msg);
  }
  // each V_k comes from dgmc_count: at most one vertex per grid edge; the batch within the 29-bit packing of dgmc_emit
  const long long edges = 3ll * G * G * (G - 1);
  dgm::McItems it;
  it.B = B;
  long long total = 0;
  for (int k = 0; k < B; ++k) {
    it.voff[k] = (int)total;
    if (V_host[k] < 0 || V_host[k] > edges || total + V_host[k] > dgm::MC_MAX_VERTS) {
      snprintf(msg, sizeof(msg), "%s: V out of range", fn);
      return bad(msg);
    }
    total += V_host[k];
  }
  it.voff[B] = (int)total;
  if (total > 0 && (!vsrc || !dL_dverts)) {
    snprintf(msg, sizeof(msg), "%s: null vsrc / dL_dverts", fn);
    return bad(msg);
  }
  return check(dgm::launch_mc_backward(G, it, phi, iso, vsrc, dL_dverts, dL_dphi, (cudaStream_t)stream));
}

int dgmc_backward(int G, int V, const float* phi, float iso, const int32_t* vsrc, const float* dL_dverts,
                  float* dL_dphi, void* stream) {
  return dgmc_backward_call("dgmc_backward", 1, G, &V, phi, iso, vsrc, dL_dverts, dL_dphi, stream);
}

int dgmc_backward_batch(int B, int G, const int32_t* V_host, const float* phi, float iso, const int32_t* vsrc,
                        const float* dL_dverts, float* dL_dphi, void* stream) {
  return dgmc_backward_call("dgmc_backward_batch", B, G, V_host, phi, iso, vsrc, dL_dverts, dL_dphi, stream);
}

// dual marching cubes: the same conventions as dgmc_*, with dual vertices and quads in place of vertices and faces
static int dgdmc_size(const char* fn, int B, int G, size_t* bytes) {
  char msg[160];
  if (B < 1 || B > dgm::MC_MAX_BATCH) {
    snprintf(msg, sizeof(msg), "%s: B out of range (1 <= B <= 64)", fn);
    return bad(msg);
  }
  if (G < 2 || G > 800 || !bytes) {
    snprintf(msg, sizeof(msg), "%s: bad argument (2 <= G <= 800)", fn);
    return bad(msg);
  }
  dgm::DmcWS::from(nullptr, G, B, bytes);
  return DGM_OK;
}

int dgdmc_workspace_size(int G, size_t* bytes) { return dgdmc_size("dgdmc_workspace_size", 1, G, bytes); }
int dgdmc_workspace_size_batch(int B, int G, size_t* bytes) {
  return dgdmc_size("dgdmc_workspace_size_batch", B, G, bytes);
}

static int dgdmc_check(const char* fn, int B, int G, const float* phi, void* ws, size_t ws_bytes) {
  char msg[160];
  size_t need;
  int rc = dgdmc_size(fn, B, G, &need);
  if (rc != DGM_OK) return rc;
  if (!phi || !ws) {
    snprintf(msg, sizeof(msg), "%s: bad argument (null grid or workspace)", fn);
    return bad(msg);
  }
  if (ws_bytes < need) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: workspace too small", fn);
    return DGM_E_WORKSPACE;
  }
  return DGM_OK;
}

static int dgdmc_count_call(const char* fn, int B, int G, const float* phi, float iso, void* ws, size_t ws_bytes,
                            int32_t* totals, int32_t* totals_host, void* totals_event, void* stream) {
  int rc = dgdmc_check(fn, B, G, phi, ws, ws_bytes);
  if (rc != DGM_OK) return rc;
  if (!totals) {
    char msg[160];
    snprintf(msg, sizeof(msg), "%s: null totals", fn);
    return bad(msg);
  }
  return check(dgm::launch_dmc_count(B, G, phi, iso, ws, totals, totals_host, (cudaEvent_t)totals_event,
                                     (cudaStream_t)stream));
}

int dgdmc_count(int G, const float* phi, float iso, void* ws, size_t ws_bytes, int32_t* totals, int32_t* totals_host,
                void* totals_event, void* stream) {
  return dgdmc_count_call("dgdmc_count", 1, G, phi, iso, ws, ws_bytes, totals, totals_host, totals_event, stream);
}

int dgdmc_count_batch(int B, int G, const float* phi, float iso, void* ws, size_t ws_bytes, int32_t* totals,
                      int32_t* totals_host, void* totals_event, void* stream) {
  return dgdmc_count_call("dgdmc_count_batch", B, G, phi, iso, ws, ws_bytes, totals, totals_host, totals_event,
                          stream);
}

static int dgdmc_emit_call(const char* fn, int B, int G, const float* phi, float iso, void* ws, size_t ws_bytes,
                           float* verts, int32_t* vsrc, int64_t V_cap, int32_t* faces, int32_t* quads, int64_t Q_cap,
                           void* stream) {
  char msg[160];
  if (V_cap < 0 || V_cap > dgm::DMC_MAX_VERTS || Q_cap < 0 || Q_cap > dgm::DMC_MAX_QUADS) {
    snprintf(msg, sizeof(msg), "%s: capacity out of range (V_cap <= 2^28, Q_cap < 2^30)", fn);
    return bad(msg);
  }
  if ((V_cap > 0 && (!verts || !vsrc)) || (Q_cap > 0 && !faces)) {
    snprintf(msg, sizeof(msg), "%s: null output", fn);
    return bad(msg);
  }
  int rc = dgdmc_check(fn, B, G, phi, ws, ws_bytes);
  if (rc != DGM_OK) return rc;
  return check(dgm::launch_dmc_emit(B, G, phi, iso, ws, verts, vsrc, V_cap, faces, quads, Q_cap,
                                    (cudaStream_t)stream));
}

int dgdmc_emit(int G, const float* phi, float iso, void* ws, size_t ws_bytes, float* verts, int32_t* vsrc,
               int64_t V_cap, int32_t* faces, int32_t* quads, int64_t Q_cap, void* stream) {
  return dgdmc_emit_call("dgdmc_emit", 1, G, phi, iso, ws, ws_bytes, verts, vsrc, V_cap, faces, quads, Q_cap, stream);
}

int dgdmc_emit_batch(int B, int G, const float* phi, float iso, void* ws, size_t ws_bytes, float* verts,
                     int32_t* vsrc, int64_t V_cap, int32_t* faces, int32_t* quads, int64_t Q_cap, void* stream) {
  return dgdmc_emit_call("dgdmc_emit_batch", B, G, phi, iso, ws, ws_bytes, verts, vsrc, V_cap, faces, quads, Q_cap,
                         stream);
}

static int dgdmc_backward_call(const char* fn, int B, int G, const int32_t* V_host, const float* phi, float iso,
                               void* ws, size_t ws_bytes, const int32_t* vsrc, const float* dL_dverts,
                               float* dL_dphi, void* stream) {
  char msg[160];
  int rc = dgdmc_check(fn, B, G, phi, ws, ws_bytes);
  if (rc != DGM_OK) return rc;
  if (!dL_dphi || !V_host) {
    snprintf(msg, sizeof(msg), "%s: bad argument (null dL_dphi or V)", fn);
    return bad(msg);
  }
  // each V_k comes from dgdmc_count: at most four dual vertices per cell, the batch within DMC_MAX_VERTS
  const long long cells = 4ll * (G - 1) * (G - 1) * (G - 1);
  dgm::McItems it;
  it.B = B;
  long long total = 0;
  for (int k = 0; k < B; ++k) {
    it.voff[k] = (int)total;
    if (V_host[k] < 0 || V_host[k] > cells || total + V_host[k] > dgm::DMC_MAX_VERTS) {
      snprintf(msg, sizeof(msg), "%s: V out of range", fn);
      return bad(msg);
    }
    total += V_host[k];
  }
  it.voff[B] = (int)total;
  if (total > 0 && (!vsrc || !dL_dverts)) {
    snprintf(msg, sizeof(msg), "%s: null vsrc / dL_dverts", fn);
    return bad(msg);
  }
  return check(dgm::launch_dmc_backward(G, it, phi, iso, ws, vsrc, dL_dverts, dL_dphi, (cudaStream_t)stream));
}

int dgdmc_backward(int G, int V, const float* phi, float iso, void* ws, size_t ws_bytes, const int32_t* vsrc,
                   const float* dL_dverts, float* dL_dphi, void* stream) {
  return dgdmc_backward_call("dgdmc_backward", 1, G, &V, phi, iso, ws, ws_bytes, vsrc, dL_dverts, dL_dphi, stream);
}

int dgdmc_backward_batch(int B, int G, const int32_t* V_host, const float* phi, float iso, void* ws, size_t ws_bytes,
                         const int32_t* vsrc, const float* dL_dverts, float* dL_dphi, void* stream) {
  return dgdmc_backward_call("dgdmc_backward_batch", B, G, V_host, phi, iso, ws, ws_bytes, vsrc, dL_dverts, dL_dphi,
                             stream);
}

// FlexiCubes: dual marching cubes' count (dgdmc_count) and workspace, with weighted crossings and vertices, node
// offsets and the gamma split
static int dgfc_weights(const char* fn, const float* alpha, const float* beta, const float* gamma_f, int training,
                        const float* dalpha, const float* dbeta, const float* dgamma) {
  char msg[160];
  if ((dalpha && !alpha) || (dbeta && !beta) || (dgamma && !gamma_f)) {
    snprintf(msg, sizeof(msg), "%s: a gradient was requested for a null weight", fn);
    return bad(msg);
  }
  if (dgamma && !training) {
    snprintf(msg, sizeof(msg), "%s: dL_dgamma is only defined in training mode", fn);
    return bad(msg);
  }
  return DGM_OK;
}

int dgfc_emit(int G, const float* phi, float iso, const float* deform, const float* alpha, const float* beta,
              const float* gamma_f, int training, int normalize, void* ws, size_t ws_bytes, float* verts,
              int32_t* vsrc, float* ldev, int32_t* vk, int64_t V_cap, int32_t* faces, int32_t* quads, int64_t Q_cap,
              void* stream) {
  const char* fn = "dgfc_emit";
  char msg[160];
  const long long q_max = training ? dgm::FC_MAX_QUADS_TRAINING : dgm::DMC_MAX_QUADS;
  if (V_cap < 0 || V_cap > dgm::DMC_MAX_VERTS || Q_cap < 0 || Q_cap > q_max) {
    snprintf(msg, sizeof(msg), "%s: capacity out of range (V_cap <= 2^28, Q_cap < 2^30, < 2^29 in training)", fn);
    return bad(msg);
  }
  if ((V_cap > 0 && (!verts || !vsrc || !ldev || !vk)) || (Q_cap > 0 && (!faces || !quads))) {
    snprintf(msg, sizeof(msg), "%s: null output", fn);
    return bad(msg);
  }
  int rc = dgdmc_check(fn, 1, G, phi, ws, ws_bytes);
  if (rc != DGM_OK) return rc;
  const dgm::FcParams w{deform, alpha, beta, gamma_f};
  return check(dgm::launch_fc_emit(G, phi, iso, w, training != 0, normalize != 0, ws, verts, vsrc, ldev, vk, V_cap,
                                   faces, quads, Q_cap, (cudaStream_t)stream));
}

static int dgfc_counts(const char* fn, int G, int V, int Q, int training) {
  char msg[160];
  const long long G1 = G - 1;
  const long long q_max = training ? dgm::FC_MAX_QUADS_TRAINING : dgm::DMC_MAX_QUADS;
  if (G < 2 || G > 800) {
    snprintf(msg, sizeof(msg), "%s: bad argument (2 <= G <= 800)", fn);
    return bad(msg);
  }
  if (V < 0 || V > 4 * G1 * G1 * G1 || V > dgm::DMC_MAX_VERTS || Q < 0 || Q > 3ll * G * G * G1 || Q > q_max) {
    snprintf(msg, sizeof(msg), "%s: V or Q out of range", fn);
    return bad(msg);
  }
  return DGM_OK;
}

int dgfc_backward_workspace_size(int G, int V, int Q, int training, size_t* bytes) {
  int rc = dgfc_counts("dgfc_backward_workspace_size", G, V, Q, training);
  if (rc != DGM_OK) return rc;
  if (!bytes) return bad("dgfc_backward_workspace_size: null bytes");
  *bytes = dgm::fc_backward_ws_bytes(G, V, Q, training != 0);
  return DGM_OK;
}

int dgfc_backward(int G, int V, int Q, const float* phi, float iso, const float* deform, const float* alpha,
                  const float* beta, const float* gamma_f, int training, int normalize, const float* verts,
                  const int32_t* vsrc, const int32_t* quads, const float* dL_dverts, const float* dL_dldev, void* ws,
                  size_t ws_bytes, float* dL_dphi, float* dL_ddeform, float* dL_dalpha, float* dL_dbeta,
                  float* dL_dgamma, void* stream) {
  const char* fn = "dgfc_backward";
  char msg[160];
  int rc = dgfc_counts(fn, G, V, Q, training);
  if (rc != DGM_OK) return rc;
  if (!phi || !ws || !dL_dphi || (dL_ddeform && !deform)) {
    snprintf(msg, sizeof(msg), "%s: bad argument (null grid, workspace or dL_dphi, or dL_ddeform without deform)", fn);
    return bad(msg);
  }
  rc = dgfc_weights(fn, alpha, beta, gamma_f, training, dL_dalpha, dL_dbeta, dL_dgamma);
  if (rc != DGM_OK) return rc;
  if ((V > 0 && (!vsrc || !dL_dverts)) || (training && V > 0 && !verts) || (training && Q > 0 && !quads)) {
    snprintf(msg, sizeof(msg), "%s: null verts / vsrc / quads / dL_dverts", fn);
    return bad(msg);
  }
  if (ws_bytes < dgm::fc_backward_ws_bytes(G, V, Q, training != 0)) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: workspace too small", fn);
    return DGM_E_WORKSPACE;
  }
  const dgm::FcParams w{deform, alpha, beta, gamma_f};
  return check(dgm::launch_fc_backward(G, V, Q, phi, iso, w, training != 0, normalize != 0, verts, vsrc, quads,
                                       dL_dverts, dL_dldev, ws, dL_dphi, dL_ddeform, dL_dalpha, dL_dbeta, dL_dgamma,
                                       (cudaStream_t)stream));
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

// the B images of a call: 1 <= B <= 64, and for the rasteriser ranges[B][2] = (first triangle, count) within F
static int dgmr_batch(const char* fn, int B) {
  char msg[160];
  if (B < 1 || B > dgm::MR_MAX_BATCH) {
    snprintf(msg, sizeof(msg), "%s: B out of range (1 <= B <= 64)", fn);
    return bad(msg);
  }
  return DGM_OK;
}

static int dgmr_ranges(int B, int F, const int32_t* ranges, dgm::MrRanges& R) {
  int rc = dgmr_batch("dgmr_rasterize_batch", B);
  if (rc != DGM_OK) return rc;
  if (!ranges) return bad("dgmr_rasterize_batch: null ranges");
  R.B = B;
  long long total = 0;
  for (int b = 0; b < B; ++b) {
    const long long first = ranges[2 * b], count = ranges[2 * b + 1];
    if (first < 0 || count < 0 || first + count > F)
      return bad("dgmr_rasterize_batch: a range runs past F (0 <= first, 0 <= count, first + count <= F)");
    R.start[b] = (int)first;
    R.off[b] = (int)total;
    total += count;
    if (total > INT32_MAX) return bad("dgmr_rasterize_batch: more than 2^31 - 1 triangles in all ranges");
  }
  R.off[B] = (int)total;
  return DGM_OK;
}

static int dgmr_rasterize_call(const char* fn, int V, int F, int W, int H, const float* pos, const int32_t* tri,
                               void* zbuf, float* rast, const dgm::MrRanges& R, void* stream) {
  char msg[160];
  if (V < 0 || F < 0 || W <= 0 || H <= 0 || !zbuf || !rast || (F > 0 && (!pos || !tri))) {
    snprintf(msg, sizeof(msg), "%s: bad argument", fn);
    return bad(msg);
  }
  if (F > dgm::MR_MAX_TRIANGLES) {
    snprintf(msg, sizeof(msg), "%s: F beyond 2^29 triangles (the largest id rast holds)", fn);
    return bad(msg);
  }
  return check(dgm::launch_mr_rasterize(R, W, H, pos, tri, zbuf, rast, (cudaStream_t)stream));
}

int dgmr_rasterize(int V, int F, int W, int H, const float* pos, const int32_t* tri, void* zbuf, float* rast,
                   void* stream) {
  dgm::MrRanges R;
  R.B = 1;
  R.start[0] = 0;
  R.off[0] = 0;
  R.off[1] = F > 0 ? F : 0;
  return dgmr_rasterize_call("dgmr_rasterize", V, F, W, H, pos, tri, zbuf, rast, R, stream);
}
int dgmr_rasterize_batch(int V, int F, int B, const int32_t* ranges, int W, int H, const float* pos,
                         const int32_t* tri, void* zbuf, float* rast, void* stream) {
  dgm::MrRanges R;
  int rc = dgmr_ranges(B, F, ranges, R);
  if (rc != DGM_OK) return rc;
  return dgmr_rasterize_call("dgmr_rasterize_batch", V, F, W, H, pos, tri, zbuf, rast, R, stream);
}

static int dgmr_rasterize_bwd_call(const char* fn, int B, int W, int H, const float* rast, const int32_t* tri,
                                   const float* pos, const float* grast, float* gpos, void* stream) {
  char msg[160];
  int rc = dgmr_batch(fn, B);
  if (rc != DGM_OK) return rc;
  if (W <= 0 || H <= 0 || !rast || !tri || !pos || !grast || !gpos) {
    snprintf(msg, sizeof(msg), "%s: bad argument", fn);
    return bad(msg);
  }
  return check(dgm::launch_mr_rasterize_bwd(B, W, H, rast, tri, pos, grast, gpos, (cudaStream_t)stream));
}
int dgmr_rasterize_bwd(int W, int H, const float* rast, const int32_t* tri, const float* pos, const float* grast,
                       float* gpos, void* stream) {
  return dgmr_rasterize_bwd_call("dgmr_rasterize_bwd", 1, W, H, rast, tri, pos, grast, gpos, stream);
}
int dgmr_rasterize_bwd_batch(int B, int W, int H, const float* rast, const int32_t* tri, const float* pos,
                             const float* grast, float* gpos, void* stream) {
  return dgmr_rasterize_bwd_call("dgmr_rasterize_bwd_batch", B, W, H, rast, tri, pos, grast, gpos, stream);
}

static int dgmr_interpolate_call(const char* fn, int B, int W, int H, int C, const float* attr, const float* rast,
                                 const int32_t* tri, float* out, void* stream) {
  char msg[160];
  int rc = dgmr_batch(fn, B);
  if (rc != DGM_OK) return rc;
  if (W <= 0 || H <= 0 || C < 1 || !attr || !rast || !tri || !out) {
    snprintf(msg, sizeof(msg), "%s: bad argument", fn);
    return bad(msg);
  }
  return check(dgm::launch_mr_interpolate(B, W, H, C, attr, rast, tri, out, (cudaStream_t)stream));
}
int dgmr_interpolate(int W, int H, int C, const float* attr, const float* rast, const int32_t* tri, float* out,
                     void* stream) {
  return dgmr_interpolate_call("dgmr_interpolate", 1, W, H, C, attr, rast, tri, out, stream);
}
int dgmr_interpolate_batch(int B, int W, int H, int C, const float* attr, const float* rast, const int32_t* tri,
                           float* out, void* stream) {
  return dgmr_interpolate_call("dgmr_interpolate_batch", B, W, H, C, attr, rast, tri, out, stream);
}

static int dgmr_interpolate_bwd_call(const char* fn, int B, int W, int H, int C, const float* attr, const float* rast,
                                     const int32_t* tri, const float* gout, float* gattr, float* grast,
                                     void* stream) {
  char msg[160];
  int rc = dgmr_batch(fn, B);
  if (rc != DGM_OK) return rc;
  if (W <= 0 || H <= 0 || C < 1 || !attr || !rast || !tri || !gout) {
    snprintf(msg, sizeof(msg), "%s: bad argument", fn);
    return bad(msg);
  }
  return check(dgm::launch_mr_interpolate_bwd(B, W, H, C, attr, rast, tri, gout, gattr, grast, (cudaStream_t)stream));
}
int dgmr_interpolate_bwd(int W, int H, int C, const float* attr, const float* rast, const int32_t* tri,
                         const float* gout, float* gattr, float* grast, void* stream) {
  return dgmr_interpolate_bwd_call("dgmr_interpolate_bwd", 1, W, H, C, attr, rast, tri, gout, gattr, grast, stream);
}
int dgmr_interpolate_bwd_batch(int B, int W, int H, int C, const float* attr, const float* rast, const int32_t* tri,
                               const float* gout, float* gattr, float* grast, void* stream) {
  return dgmr_interpolate_bwd_call("dgmr_interpolate_bwd_batch", B, W, H, C, attr, rast, tri, gout, gattr, grast,
                                   stream);
}

static int dgmr_antialias_call(const char* fn, int B, int W, int H, int C, const float* color, const float* rast,
                               const float* pos, const int32_t* tri, const int32_t* opp, float* out, void* stream) {
  char msg[160];
  int rc = dgmr_batch(fn, B);
  if (rc != DGM_OK) return rc;
  if (W <= 0 || H <= 0 || C < 1 || !color || !rast || !pos || !tri || !opp || !out) {
    snprintf(msg, sizeof(msg), "%s: bad argument", fn);
    return bad(msg);
  }
  return check(dgm::launch_mr_antialias(B, W, H, C, color, rast, pos, tri, opp, out, (cudaStream_t)stream));
}
int dgmr_antialias(int W, int H, int C, const float* color, const float* rast, const float* pos,
                   const int32_t* tri, const int32_t* opp, float* out, void* stream) {
  return dgmr_antialias_call("dgmr_antialias", 1, W, H, C, color, rast, pos, tri, opp, out, stream);
}
int dgmr_antialias_batch(int B, int W, int H, int C, const float* color, const float* rast, const float* pos,
                         const int32_t* tri, const int32_t* opp, float* out, void* stream) {
  return dgmr_antialias_call("dgmr_antialias_batch", B, W, H, C, color, rast, pos, tri, opp, out, stream);
}

static int dgmr_antialias_bwd_call(const char* fn, int B, int W, int H, int C, const float* color, const float* rast,
                                   const float* pos, const int32_t* tri, const int32_t* opp, const float* gout,
                                   float* gcolor, float* gpos, void* stream) {
  char msg[160];
  int rc = dgmr_batch(fn, B);
  if (rc != DGM_OK) return rc;
  if (W <= 0 || H <= 0 || C < 1 || !color || !rast || !pos || !tri || !opp || !gout) {
    snprintf(msg, sizeof(msg), "%s: bad argument", fn);
    return bad(msg);
  }
  return check(dgm::launch_mr_antialias_bwd(B, W, H, C, color, rast, pos, tri, opp, gout, gcolor, gpos,
                                            (cudaStream_t)stream));
}
int dgmr_antialias_bwd(int W, int H, int C, const float* color, const float* rast, const float* pos,
                       const int32_t* tri, const int32_t* opp, const float* gout, float* gcolor, float* gpos,
                       void* stream) {
  return dgmr_antialias_bwd_call("dgmr_antialias_bwd", 1, W, H, C, color, rast, pos, tri, opp, gout, gcolor, gpos,
                                 stream);
}
int dgmr_antialias_bwd_batch(int B, int W, int H, int C, const float* color, const float* rast, const float* pos,
                             const int32_t* tri, const int32_t* opp, const float* gout, float* gcolor, float* gpos,
                             void* stream) {
  return dgmr_antialias_bwd_call("dgmr_antialias_bwd_batch", B, W, H, C, color, rast, pos, tri, opp, gout, gcolor,
                                 gpos, stream);
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
             const float* opacity_raw, float max_grad, float min_opacity, double extent, double percent_dense,
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

int dgo_adam_step(int n_tensors, const DgoTensor* tensors_host, double beta1, double beta2,
                  const int32_t* row_radii, int zero_grad, void* stream) {
  if (n_tensors < 1 || n_tensors > DGO_MAX_TENSORS) return bad("dgo_adam_step: need 1 <= n_tensors <= 32");
  if (!tensors_host) return bad("dgo_adam_step: null tensor table");
  if (!(beta1 >= 0.0 && beta1 < 1.0 && beta2 >= 0.0 && beta2 < 1.0)) return bad("dgo_adam_step: need 0 <= beta < 1");
  dgm::AdamTable tab = {};
  tab.w1 = (float)(1.0 - beta1);
  tab.beta2 = (float)beta2;
  tab.w2 = (float)(1.0 - beta2);
  int64_t rows = -1, chunks = 0;
  for (int i = 0; i < n_tensors; ++i) {
    const DgoTensor& t = tensors_host[i];
    if (!t.p || !t.g || !t.m || !t.v) return bad("dgo_adam_step: null p / g / m / v pointer");
    if (t.n < 0) return bad("dgo_adam_step: negative element count");
    if (row_radii) {
      if (t.row_width < 1 || t.n % t.row_width) return bad("dgo_adam_step: n is not a multiple of row_width");
      if (rows >= 0 && t.n / t.row_width != rows) return bad("dgo_adam_step: row counts differ under one row mask");
      rows = t.n / t.row_width;
    }
    if (t.n == 0) continue;
    chunks += (t.n + ADAM_CHUNK - 1) / ADAM_CHUNK;
    if (chunks > INT32_MAX) return bad("dgo_adam_step: more than 2^31 - 1 chunks");
    tab.t[tab.n_tensors] = t;
    tab.chunk_end[tab.n_tensors++] = (int)chunks;
  }
  if (tab.n_tensors == 0) return DGM_OK;
  return check(dgm::launch_adam_step(tab, row_radii, zero_grad, (cudaStream_t)stream));
}

int dgo_densify_stats(int F, int P, const float* viewspace_grad, const float* viewspace_abs_grad,
                      int64_t grad_stride, const int32_t* radii, int64_t radii_stride, float* xyz_gradient_accum,
                      float* xyz_gradient_accum_abs, float* denom, float* max_radii2D, void* stream) {
  if (F < 1 || P < 0) return bad("dgo_densify_stats: bad size");
  if (P > 0 && (!viewspace_grad || !radii || !xyz_gradient_accum || !denom))
    return bad("dgo_densify_stats: null pointer");
  if ((viewspace_abs_grad == nullptr) != (xyz_gradient_accum_abs == nullptr))
    return bad("dgo_densify_stats: the abs gradient and its accumulator come together");
  if (F > 1 && (grad_stride < 3 * (int64_t)P || radii_stride < P)) return bad("dgo_densify_stats: stride too small");
  return check(dgm::launch_densify_stats(F, P, viewspace_grad, viewspace_abs_grad, grad_stride, radii, radii_stride,
                                         xyz_gradient_accum, xyz_gradient_accum_abs, denom, max_radii2D,
                                         (cudaStream_t)stream));
}

int dgx_allreduce_nvls(float* multicast_ptr, size_t n_floats, void* signal_pads_dev, int rank, int world,
                       uint32_t epoch, float scale, int blocks, void* stream) {
  if (!multicast_ptr || !signal_pads_dev || world < 1 || rank < 0 || rank >= world || blocks < 1 || (n_floats & 3) ||
      ((uintptr_t)multicast_ptr & 15) || epoch == 0)
    return bad("dgx_allreduce_nvls: bad argument");
  return check(dgm::launch_nvls_allreduce(multicast_ptr, n_floats, (uint32_t* const*)signal_pads_dev, rank, world,
                                          epoch, scale, blocks, (cudaStream_t)stream));
}

// ---- opacity field.  The checks shared by the three entry points: DGM_OK, or the error to return.
static int dgf_sizes(const char* fn, int P, int G, int64_t pair_cap) {
  char msg[160];
  if (P < 0 || G < 2 || G > OF_MAX_G || pair_cap < 0 || pair_cap > INT32_MAX) {
    snprintf(msg, sizeof(msg), "%s: bad size (P >= 0, 2 <= G <= %d, 0 <= pair_cap <= 2^31 - 1)", fn, OF_MAX_G);
    return bad(msg);
  }
  return DGM_OK;
}

static int dgf_args(const char* fn, int P, int G, const float* means3D, const float* scales, const float* rotations,
                    const float* opacities, const float* box, float cutoff, float scale_modifier, int64_t pair_cap,
                    const void* ws, size_t ws_bytes, dgm::OfParams& p) {
  char msg[160];
  int rc = dgf_sizes(fn, P, G, pair_cap);
  if (rc != DGM_OK) return rc;
  if (!box || !ws || (P > 0 && (!means3D || !scales || !rotations || !opacities))) {
    snprintf(msg, sizeof(msg), "%s: null pointer", fn);
    return bad(msg);
  }
  if (!(cutoff > 0.f) || !isfinite(cutoff) || !(scale_modifier > 0.f) || !isfinite(scale_modifier)) {
    snprintf(msg, sizeof(msg), "%s: cutoff and scale_modifier must be finite and > 0", fn);
    return bad(msg);
  }
  size_t need;
  dgm::OfWS::from(nullptr, P, G, pair_cap, &need);
  if (ws_bytes < need) {
    snprintf(g_last_error, sizeof(g_last_error), "%s: workspace too small (%zu < %zu bytes)", fn, ws_bytes, need);
    return DGM_E_WORKSPACE;
  }
  const double k2 = (double)cutoff * cutoff, e0 = exp(-0.5 * k2);
  p = dgm::OfParams{P, G, means3D, scales, rotations, opacities, box, scale_modifier, (float)k2, (float)e0,
                    (float)(1.0 / (1.0 - e0))};
  return DGM_OK;
}

int dgf_workspace_size(int P, int G, int64_t pair_cap, size_t* bytes) {
  const int rc = dgf_sizes("dgf_workspace_size", P, G, pair_cap);
  if (rc != DGM_OK) return rc;
  if (!bytes) return bad("dgf_workspace_size: null pointer");
  dgm::OfWS::from(nullptr, P, G, pair_cap, bytes);
  return DGM_OK;
}

int dgf_forward(int P, int G, const float* means3D, const float* scales, const float* rotations,
                const float* opacities, const float* box, float cutoff, float scale_modifier, int64_t pair_cap,
                void* ws, size_t ws_bytes, float* phi, int32_t* pairs_host, void* pairs_event, void* stream) {
  dgm::OfParams p;
  const int rc = dgf_args("dgf_forward", P, G, means3D, scales, rotations, opacities, box, cutoff, scale_modifier,
                          pair_cap, ws, ws_bytes, p);
  if (rc != DGM_OK) return rc;
  if (!phi) return bad("dgf_forward: null pointer");
  return check(dgm::launch_of_forward(p, pair_cap, ws, phi, pairs_host, (cudaEvent_t)pairs_event,
                                      (cudaStream_t)stream));
}

int dgf_backward(int P, int G, const float* means3D, const float* scales, const float* rotations,
                 const float* opacities, const float* box, float cutoff, float scale_modifier, int64_t pair_cap,
                 void* ws, size_t ws_bytes, const float* dL_dphi, float* dL_dmeans3D, float* dL_dscales,
                 float* dL_drotations, float* dL_dopacities, void* stream) {
  dgm::OfParams p;
  const int rc = dgf_args("dgf_backward", P, G, means3D, scales, rotations, opacities, box, cutoff, scale_modifier,
                          pair_cap, ws, ws_bytes, p);
  if (rc != DGM_OK) return rc;
  if (!dL_dphi || (P > 0 && (!dL_dmeans3D || !dL_dscales || !dL_drotations || !dL_dopacities)))
    return bad("dgf_backward: null pointer");
  return check(dgm::launch_of_backward(p, pair_cap, ws, dL_dphi, dL_dmeans3D, dL_dscales, dL_drotations,
                                       dL_dopacities, (cudaStream_t)stream));
}

// ---- TSDF fusion.  Every argument is checked here, before any device work.
int dgt_integrate(int G, const float* box, int F, int W, int H, const float* views_host, const float* coefs_host,
                  const float* depth, const float* color, float sdf_trunc, float depth_max, float* tsdf,
                  float* weight, float* color_grid, void* stream) {
  char msg[160];
  if (G < 2 || G > TSDF_MAX_G || F < 1 || W < 1 || H < 1) {
    snprintf(msg, sizeof(msg), "dgt_integrate: bad size (2 <= G <= %d, F, W, H >= 1)", TSDF_MAX_G);
    return bad(msg);
  }
  if (!(sdf_trunc > 0.f) || !isfinite(sdf_trunc)) return bad("dgt_integrate: sdf_trunc must be finite and > 0");
  if (!(depth_max > 0.f)) return bad("dgt_integrate: depth_max must be > 0 (+inf allowed)");
  if (!box || !views_host || !coefs_host || !depth || !tsdf || !weight) return bad("dgt_integrate: null pointer");
  if (!color != !color_grid) return bad("dgt_integrate: color and color_grid must be both NULL or both non-NULL");
  for (int f = 0; f < F; ++f) {
    if (coefs_host[4 * (size_t)f] == 0.f || coefs_host[4 * (size_t)f + 2] == 0.f) {
      snprintf(msg, sizeof(msg), "dgt_integrate: frame %d has a zero ray coefficient a_x or a_y", f);
      return bad(msg);
    }
  }
  const dgm::TsdfArgs a = {G, F, W, H, box, views_host, coefs_host, depth, color, sdf_trunc, depth_max, tsdf,
                           weight, color_grid};
  return check(dgm::launch_tsdf_integrate(a, (cudaStream_t)stream));
}

// ---- structural losses (nn_distance, match_cost).  Every argument is checked here, before any device work.
namespace {
int dge_sizes(const char* fn, int B, int N, int M) {
  char msg[160];
  // B on gridDim.z / y; 3 B N, 3 B M (coordinate indices and the CSR keys) in 31 bits
  if (B < 1 || N < 1 || M < 1 || B > 65535 || 3 * (int64_t)B * N > INT32_MAX || 3 * (int64_t)B * M > INT32_MAX) {
    snprintf(msg, sizeof(msg), "%s: bad size (1 <= B <= 65535, N, M >= 1, 3 B N and 3 B M < 2^31)", fn);
    return bad(msg);
  }
  return DGM_OK;
}
int dge_short(const char* fn, size_t ws_bytes, size_t need) {
  snprintf(g_last_error, sizeof(g_last_error), "%s: workspace too small (%zu < %zu bytes)", fn, ws_bytes, need);
  return DGM_E_WORKSPACE;
}
}  // namespace

int dge_nn_distance(int B, int N, int M, const float* xyz1, const float* xyz2, float* dist1, int64_t* idx1,
                    float* dist2, int64_t* idx2, void* stream) {
  const int rc = dge_sizes("dge_nn_distance", B, N, M);
  if (rc != DGM_OK) return rc;
  if (!xyz1 || !xyz2 || !dist1 || !idx1 || !dist2 || !idx2) return bad("dge_nn_distance: null pointer");
  return check(dgm::launch_nn_distance(B, N, M, xyz1, xyz2, dist1, (long long*)idx1, dist2, (long long*)idx2,
                                       (cudaStream_t)stream));
}

int dge_nn_distance_workspace(int B, int N, int M, size_t* bytes) {
  const int rc = dge_sizes("dge_nn_distance_workspace", B, N, M);
  if (rc != DGM_OK) return rc;
  if (!bytes) return bad("dge_nn_distance_workspace: null pointer");
  dgm::NnWS::from(nullptr, B, N, M, dgm::nn_cub_bytes(B, N, M), bytes);
  return DGM_OK;
}

int dge_nn_distance_bwd(int B, int N, int M, const float* xyz1, const float* xyz2, const int64_t* idx1,
                        const int64_t* idx2, const float* grad_dist1, const float* grad_dist2, float* grad_xyz1,
                        float* grad_xyz2, void* ws, size_t ws_bytes, void* stream) {
  const int rc = dge_sizes("dge_nn_distance_bwd", B, N, M);
  if (rc != DGM_OK) return rc;
  if (!xyz1 || !xyz2 || !idx1 || !idx2 || !grad_dist1 || !grad_dist2 || !grad_xyz1 || !grad_xyz2 || !ws)
    return bad("dge_nn_distance_bwd: null pointer");
  size_t need;
  dge_nn_distance_workspace(B, N, M, &need);
  if (ws_bytes < need) return dge_short("dge_nn_distance_bwd", ws_bytes, need);
  return check(dgm::launch_nn_distance_bwd(B, N, M, xyz1, xyz2, (const long long*)idx1, (const long long*)idx2,
                                           grad_dist1, grad_dist2, grad_xyz1, grad_xyz2, ws, (cudaStream_t)stream));
}

int dge_match_cost_workspace(int B, int N, int M, size_t* bytes) {
  const int rc = dge_sizes("dge_match_cost_workspace", B, N, M);
  if (rc != DGM_OK) return rc;
  if (!bytes) return bad("dge_match_cost_workspace: null pointer");
  dgm::MatchWS::from(nullptr, B, N, M, bytes);
  return DGM_OK;
}

int dge_match_cost(int B, int N, int M, const float* xyz1, const float* xyz2, float* cost, void* ws,
                   size_t ws_bytes, void* stream) {
  const int rc = dge_sizes("dge_match_cost", B, N, M);
  if (rc != DGM_OK) return rc;
  if (!xyz1 || !xyz2 || !cost || !ws) return bad("dge_match_cost: null pointer");
  size_t need;
  dge_match_cost_workspace(B, N, M, &need);
  if (ws_bytes < need) return dge_short("dge_match_cost", ws_bytes, need);
  return check(dgm::launch_match_cost(B, N, M, xyz1, xyz2, cost, ws, (cudaStream_t)stream));
}

int dge_match_cost_bwd(int B, int N, int M, const float* xyz1, const float* xyz2, const float* grad_cost,
                       float* grad_xyz1, float* grad_xyz2, void* ws, size_t ws_bytes, void* stream) {
  const int rc = dge_sizes("dge_match_cost_bwd", B, N, M);
  if (rc != DGM_OK) return rc;
  if (!xyz1 || !xyz2 || !grad_cost || !grad_xyz1 || !grad_xyz2 || !ws) return bad("dge_match_cost_bwd: null pointer");
  size_t need;
  dge_match_cost_workspace(B, N, M, &need);
  if (ws_bytes < need) return dge_short("dge_match_cost_bwd", ws_bytes, need);
  return check(dgm::launch_match_cost_bwd(B, N, M, xyz1, xyz2, grad_cost, grad_xyz1, grad_xyz2, ws,
                                          (cudaStream_t)stream));
}

// ---- point-to-mesh distance.  Every argument is checked here, before any device work.
namespace {
int dgpm_sizes(const char* fn, int V, int F, int Q) {
  char msg[160];
  // 3 V, 3 F, 3 Q coordinate / index offsets and the 3 Q backward entries in 31 bits
  if (V < 1 || F < 1 || Q < 0 || 3 * (int64_t)V > INT32_MAX || 3 * (int64_t)F > INT32_MAX ||
      3 * (int64_t)Q > INT32_MAX) {
    snprintf(msg, sizeof(msg), "%s: bad size (V, F >= 1, Q >= 0, 3 V, 3 F and 3 Q < 2^31)", fn);
    return bad(msg);
  }
  return DGM_OK;
}
}  // namespace

int dgpm_forward_workspace(int V, int F, int Q, size_t* bytes) {
  const int rc = dgpm_sizes("dgpm_forward_workspace", V, F, Q);
  if (rc != DGM_OK) return rc;
  if (!bytes) return bad("dgpm_forward_workspace: null pointer");
  dgm::PmFwdWS::from(nullptr, F, Q, dgm::pm_fwd_cub_bytes(F, Q), bytes);
  return DGM_OK;
}

int dgpm_forward(int V, int F, int Q, const float* verts, const int32_t* faces, const float* points, float* dist2,
                 int64_t* face, float* bary, void* ws, size_t ws_bytes, void* stream) {
  const int rc = dgpm_sizes("dgpm_forward", V, F, Q);
  if (rc != DGM_OK) return rc;
  if (Q == 0) return DGM_OK;
  if (!verts || !faces || !points || !dist2 || !face || !bary || !ws) return bad("dgpm_forward: null pointer");
  size_t need;
  dgpm_forward_workspace(V, F, Q, &need);
  if (ws_bytes < need) return dge_short("dgpm_forward", ws_bytes, need);
  return check(dgm::launch_point_mesh_distance(F, Q, verts, faces, points, dist2, (long long*)face, bary, ws,
                                               (cudaStream_t)stream));
}

int dgpm_backward_workspace(int V, int F, int Q, size_t* bytes) {
  const int rc = dgpm_sizes("dgpm_backward_workspace", V, F, Q);
  if (rc != DGM_OK) return rc;
  if (!bytes) return bad("dgpm_backward_workspace: null pointer");
  dgm::PmBwdWS::from(nullptr, Q, dgm::pm_bwd_cub_bytes(V, Q), bytes);
  return DGM_OK;
}

int dgpm_backward(int V, int F, int Q, const float* verts, const int32_t* faces, const float* points,
                  const int64_t* face, const float* bary, const float* grad_dist2, float* grad_points,
                  float* grad_verts, void* ws, size_t ws_bytes, void* stream) {
  const int rc = dgpm_sizes("dgpm_backward", V, F, Q);
  if (rc != DGM_OK) return rc;
  if (Q == 0) return DGM_OK;
  if (!verts || !faces || !points || !face || !bary || !grad_dist2 || !grad_points || !grad_verts || !ws)
    return bad("dgpm_backward: null pointer");
  size_t need;
  dgpm_backward_workspace(V, F, Q, &need);
  if (ws_bytes < need) return dge_short("dgpm_backward", ws_bytes, need);
  return check(dgm::launch_point_mesh_distance_bwd(V, Q, verts, faces, points, (const long long*)face, bary,
                                                   grad_dist2, grad_points, grad_verts, ws, (cudaStream_t)stream));
}

int dgpm_winding_workspace(int V, int F, int Q, size_t* bytes) {
  const int rc = dgpm_sizes("dgpm_winding_workspace", V, F, Q);
  if (rc != DGM_OK) return rc;
  if (!bytes) return bad("dgpm_winding_workspace: null pointer");
  dgm::WnWS::from(nullptr, F, Q, dgm::pm_fwd_cub_bytes(F, Q), bytes);
  return DGM_OK;
}

int dgpm_winding(int V, int F, int Q, const float* verts, const int32_t* faces, const float* points, float beta,
                 float* winding, float* dist2, int64_t* face, float* bary, void* ws, size_t ws_bytes, void* stream) {
  const int rc = dgpm_sizes("dgpm_winding", V, F, Q);
  if (rc != DGM_OK) return rc;
  if (!(beta > 0.f)) return bad("dgpm_winding: beta must be > 0 (+inf for the exact sum)");
  if (Q == 0) return DGM_OK;
  if (!verts || !faces || !points || !winding || !ws) return bad("dgpm_winding: null pointer");
  if (!dist2 != !face || !dist2 != !bary) return bad("dgpm_winding: dist2, face and bary must be all NULL or none");
  size_t need;
  dgpm_winding_workspace(V, F, Q, &need);
  if (ws_bytes < need) return dge_short("dgpm_winding", ws_bytes, need);
  return check(dgm::launch_winding_number(F, Q, verts, faces, points, beta, winding, dist2, (long long*)face, bary,
                                          ws, (cudaStream_t)stream));
}

// ---- deformation regularisers and their K-nearest-neighbour graph.  Every argument is checked here, before any
// device work.
namespace {
int dgdr_sizes(const char* fn, int F, int P, int K) {
  char msg[200];
  // 3 P K pair offsets and 4 F P state offsets in 31 bits
  if (K < 1 || K > KG_MAX_K || P < 0 || F < 0 || (P > 0 && P <= K) || 3 * (int64_t)P * K > INT32_MAX ||
      4 * (int64_t)F * P > INT32_MAX) {
    snprintf(msg, sizeof(msg), "%s: bad size (1 <= K <= 32, P = 0 or P > K, F >= 0, 3 P K and 4 F P < 2^31)", fn);
    return bad(msg);
  }
  return DGM_OK;
}
}  // namespace

int dgkg_workspace(int P, int K, size_t* bytes) {
  const int rc = dgdr_sizes("dgkg_workspace", 1, P, K);
  if (rc != DGM_OK) return rc;
  if (!bytes) return bad("dgkg_workspace: null pointer");
  dgm::KgWS::from(nullptr, P, K, dgm::kg_cub_bytes(P, K), bytes);
  return DGM_OK;
}

int dgkg_build(int P, int K, float weight_lambda, const float* points, int32_t* index, float* dist2, float* weight,
               int32_t* inv_offsets, int32_t* inv_pairs, void* ws, size_t ws_bytes, void* stream) {
  const int rc = dgdr_sizes("dgkg_build", 1, P, K);
  if (rc != DGM_OK) return rc;
  if (!(weight_lambda >= 0.f) || isinf(weight_lambda)) return bad("dgkg_build: bad weight_lambda (finite, >= 0)");
  if (P == 0) return DGM_OK;
  if (!points || !index || !dist2 || !weight || !inv_offsets || !inv_pairs || !ws)
    return bad("dgkg_build: null pointer");
  size_t need;
  dgkg_workspace(P, K, &need);
  if (ws_bytes < need) return dge_short("dgkg_build", ws_bytes, need);
  return check(dgm::launch_knn_graph(P, K, weight_lambda, points, index, dist2, weight, inv_offsets, inv_pairs, ws,
                                     (cudaStream_t)stream));
}

int dgdr_forward_workspace(int F, int P, int K, size_t* bytes) {
  const int rc = dgdr_sizes("dgdr_forward_workspace", F, P, K);
  if (rc != DGM_OK) return rc;
  if (!bytes) return bad("dgdr_forward_workspace: null pointer");
  dgm::DrWS::from(nullptr, F, P, false, bytes);
  return DGM_OK;
}

int dgdr_forward(int F, int P, int K, const int32_t* index, const float* weight, const float* xyz_a,
                 const float* rot_a, const float* xyz_b, const float* rot_b, float* losses, void* ws, size_t ws_bytes,
                 void* stream) {
  const int rc = dgdr_sizes("dgdr_forward", F, P, K);
  if (rc != DGM_OK) return rc;
  if (F == 0 || P == 0) return DGM_OK;
  if (!index || !weight || !xyz_a || !rot_a || !xyz_b || !rot_b || !losses || !ws)
    return bad("dgdr_forward: null pointer");
  size_t need;
  dgdr_forward_workspace(F, P, K, &need);
  if (ws_bytes < need) return dge_short("dgdr_forward", ws_bytes, need);
  return check(dgm::launch_deform_reg_fwd(F, P, K, index, weight, xyz_a, rot_a, xyz_b, rot_b, losses, ws,
                                          (cudaStream_t)stream));
}

int dgdr_backward_workspace(int F, int P, int K, size_t* bytes) {
  const int rc = dgdr_sizes("dgdr_backward_workspace", F, P, K);
  if (rc != DGM_OK) return rc;
  if (!bytes) return bad("dgdr_backward_workspace: null pointer");
  dgm::DrWS::from(nullptr, F, P, true, bytes);
  return DGM_OK;
}

int dgdr_backward(int F, int P, int K, const int32_t* index, const float* weight, const int32_t* inv_offsets,
                  const int32_t* inv_pairs, const float* xyz_a, const float* rot_a, const float* xyz_b,
                  const float* rot_b, const float* grad_losses, float* grad_xyz_a, float* grad_rot_a,
                  float* grad_xyz_b, float* grad_rot_b, void* ws, size_t ws_bytes, void* stream) {
  const int rc = dgdr_sizes("dgdr_backward", F, P, K);
  if (rc != DGM_OK) return rc;
  if (F == 0 || P == 0) return DGM_OK;
  if (!index || !weight || !inv_offsets || !inv_pairs || !xyz_a || !rot_a || !xyz_b || !rot_b || !grad_losses || !ws)
    return bad("dgdr_backward: null pointer");
  size_t need;
  dgdr_backward_workspace(F, P, K, &need);
  if (ws_bytes < need) return dge_short("dgdr_backward", ws_bytes, need);
  return check(dgm::launch_deform_reg_bwd(F, P, K, index, weight, inv_offsets, inv_pairs, xyz_a, rot_a, xyz_b, rot_b,
                                          grad_losses, grad_xyz_a, grad_rot_a, grad_xyz_b, grad_rot_b, ws,
                                          (cudaStream_t)stream));
}

// ---- HexPlane field and its regularisers.  Every argument is checked here, before any device work.
namespace {
int dghp_field(const char* fn, int S, int C, const int32_t* res_host, int R_t, dgm::HpField& f) {
  char msg[200];
  if (S < 1 || S > HP_MAX_S || (C != 16 && C != 32) || R_t < 2) {
    snprintf(msg, sizeof(msg), "%s: bad size (1 <= S <= 4, C = 16 or 32, R_t >= 2)", fn);
    return bad(msg);
  }
  if (!res_host) {
    snprintf(msg, sizeof(msg), "%s: null pointer (res_host)", fn);
    return bad(msg);
  }
  memset(&f, 0, sizeof(f));
  f.S = S, f.C = C, f.Rt = R_t;
  for (int s = 0; s < S; ++s) {
    const int64_t R = res_host[s];
    if (R < 2 || R * R * C > INT32_MAX || (int64_t)R_t * R * C > INT32_MAX) {
      snprintf(msg, sizeof(msg), "%s: bad size (resolutions >= 2, R R C and R_t R C < 2^31)", fn);
      return bad(msg);
    }
    f.R[s] = (int)R;
  }
  return DGM_OK;
}

int dghp_sizes(const char* fn, int F, int N, int S, int C) {
  char msg[200];
  if (F < 0 || N < 0 || 3 * (int64_t)S * N * (1 + (int64_t)F) > INT32_MAX || (int64_t)F * N * S * C > INT32_MAX) {
    snprintf(msg, sizeof(msg), "%s: bad size (F, N >= 0, 3 S N (1 + F) and F N S C < 2^31)", fn);
    return bad(msg);
  }
  return DGM_OK;
}

// the field's shape and, when planes_host is given, its 6 S plane pointers (none may be NULL)
int dghp_args(const char* fn, int F, int N, int S, int C, const int32_t* res_host, int R_t,
              const float* const* planes_host, dgm::HpField& f) {
  int rc = dghp_field(fn, S, C, res_host, R_t, f);
  if (rc == DGM_OK) rc = dghp_sizes(fn, F, N, S, C);
  if (rc != DGM_OK || !planes_host) return rc;
  for (int p = 0; p < HP_PLANES * S; ++p) {
    if (!planes_host[p]) {
      char msg[200];
      snprintf(msg, sizeof(msg), "%s: null pointer (plane %d)", fn, p);
      return bad(msg);
    }
    f.p[p] = planes_host[p];
  }
  return DGM_OK;
}

int dghp_grads(const char* fn, int S, float* const* grad_planes_host, dgm::HpGrads& g) {
  char msg[200];
  for (int p = 0; p < HP_PLANES * S; ++p) {
    if (!grad_planes_host[p]) {
      snprintf(msg, sizeof(msg), "%s: null pointer (plane gradient %d)", fn, p);
      return bad(msg);
    }
    g.p[p] = grad_planes_host[p];
  }
  return DGM_OK;
}
}  // namespace

int dghp_forward(int F, int N, int S, int C, const int32_t* res_host, int R_t, const float* box, const float* x,
                 const float* t, const float* const* planes_host, float* out, void* stream) {
  dgm::HpField f;
  if (!planes_host) return bad("dghp_forward: null pointer");
  const int rc = dghp_args("dghp_forward", F, N, S, C, res_host, R_t, planes_host, f);
  if (rc != DGM_OK) return rc;
  if (F == 0 || N == 0) return DGM_OK;
  if (!box || !x || !t || !out) return bad("dghp_forward: null pointer");
  return check(dgm::launch_hexplane_fwd(F, N, f, box, x, t, out, (cudaStream_t)stream));
}

int dghp_backward_workspace(int F, int N, int S, int C, const int32_t* res_host, int R_t, size_t* bytes) {
  dgm::HpField f;
  const int rc = dghp_args("dghp_backward_workspace", F, N, S, C, res_host, R_t, nullptr, f);
  if (rc != DGM_OK) return rc;
  if (!bytes) return bad("dghp_backward_workspace: null pointer");
  const size_t E = dgm::hp_entries(F, N, S), cells = dgm::hp_cells(f);
  dgm::HpWS::from(nullptr, E, cells, C, E ? dgm::hp_cub_bytes(E, cells) : 0, bytes);
  return DGM_OK;
}

int dghp_backward(int F, int N, int S, int C, const int32_t* res_host, int R_t, const float* box, const float* x,
                  const float* t, const float* const* planes_host, const float* grad_out, float* grad_x,
                  float* const* grad_planes_host, void* ws, size_t ws_bytes, void* stream) {
  dgm::HpField f;
  dgm::HpGrads g;
  if (!planes_host || !grad_planes_host) return bad("dghp_backward: null pointer");
  int rc = dghp_args("dghp_backward", F, N, S, C, res_host, R_t, planes_host, f);
  if (rc == DGM_OK) rc = dghp_grads("dghp_backward", S, grad_planes_host, g);
  if (rc != DGM_OK) return rc;
  if (F > 0 && N > 0) {
    if (!box || !x || !t || !grad_out || !ws) return bad("dghp_backward: null pointer");
    size_t need;
    dghp_backward_workspace(F, N, S, C, res_host, R_t, &need);
    if (ws_bytes < need) return dge_short("dghp_backward", ws_bytes, need);
  }
  return check(dgm::launch_hexplane_bwd(F, N, f, box, x, t, grad_out, grad_x, g, ws, (cudaStream_t)stream));
}

int dghp_reg_workspace(int S, int C, const int32_t* res_host, int R_t, size_t* bytes) {
  dgm::HpField f;
  const int rc = dghp_field("dghp_reg_workspace", S, C, res_host, R_t, f);
  if (rc != DGM_OK) return rc;
  if (!bytes) return bad("dghp_reg_workspace: null pointer");
  *bytes = dgm::hp_reg_ws_bytes(f);
  return DGM_OK;
}

int dghp_reg_forward(int S, int C, const int32_t* res_host, int R_t, const float* const* planes_host, float* losses,
                     void* ws, size_t ws_bytes, void* stream) {
  dgm::HpField f;
  if (!planes_host) return bad("dghp_reg_forward: null pointer");
  const int rc = dghp_args("dghp_reg_forward", 0, 0, S, C, res_host, R_t, planes_host, f);
  if (rc != DGM_OK) return rc;
  if (!losses || !ws) return bad("dghp_reg_forward: null pointer");
  const size_t need = dgm::hp_reg_ws_bytes(f);
  if (ws_bytes < need) return dge_short("dghp_reg_forward", ws_bytes, need);
  return check(dgm::launch_hexplane_reg_fwd(f, losses, ws, (cudaStream_t)stream));
}

int dghp_reg_backward(int S, int C, const int32_t* res_host, int R_t, const float* const* planes_host,
                      const float* grad_losses, float* const* grad_planes_host, void* stream) {
  dgm::HpField f;
  dgm::HpGrads g;
  if (!planes_host || !grad_planes_host) return bad("dghp_reg_backward: null pointer");
  int rc = dghp_args("dghp_reg_backward", 0, 0, S, C, res_host, R_t, planes_host, f);
  if (rc == DGM_OK) rc = dghp_grads("dghp_reg_backward", S, grad_planes_host, g);
  if (rc != DGM_OK) return rc;
  if (!grad_losses) return bad("dghp_reg_backward: null pointer");
  return check(dgm::launch_hexplane_reg_bwd(f, grad_losses, g, (cudaStream_t)stream));
}

// ---- hash-grid field.  Every argument is checked here, before any device work.
namespace {
// the field's shape (kinds, resolutions, dense levels) and, when tables_host is given, its G table pointers
int dghg_args(const char* fn, int F, int N, int G, const int32_t* grids_host, int L, int Fe, int log2_table,
              const int32_t* res_host, int R_t, const float* const* tables_host, dgm::HgField& f) {
  char msg[200];
  if (G < 1 || G > HG_MAX_G || L < 1 || L > HG_MAX_L || (Fe != 2 && Fe != 4) || log2_table < 12 || log2_table > 24 ||
      R_t < 1) {
    snprintf(msg, sizeof(msg), "%s: bad size (1 <= G <= 4, 1 <= L <= 24, Fe = 2 or 4, 12 <= log2_table <= 24, R_t >= 1)",
             fn);
    return bad(msg);
  }
  if (!grids_host || !res_host) {
    snprintf(msg, sizeof(msg), "%s: null pointer (%s)", fn, grids_host ? "res_host" : "grids_host");
    return bad(msg);
  }
  const int64_t T = (int64_t)1 << log2_table, GLFe = (int64_t)G * L * Fe;
  if (F < 0 || N < 0 || (int64_t)L * T * Fe >= ((int64_t)1 << 31) || (int64_t)F * N * GLFe >= ((int64_t)1 << 31) ||
      (int64_t)N * F >= ((int64_t)1 << 31)) {
    snprintf(msg, sizeof(msg), "%s: bad size (F, N >= 0; L T Fe, F N G L Fe and N F < 2^31)", fn);
    return bad(msg);
  }
  memset(&f, 0, sizeof(f));
  f.G = G, f.L = L, f.Fe = Fe, f.log2T = log2_table;
  for (int g = 0; g < G; ++g) {
    if (grids_host[g] < 0 || grids_host[g] > 3 || (g > 0 && grids_host[g] <= grids_host[g - 1])) {
      snprintf(msg, sizeof(msg), "%s: bad grids (kinds 0 xyz, 1 xyt, 2 yzt, 3 xzt, strictly increasing)", fn);
      return bad(msg);
    }
    f.kind[g] = grids_host[g];
  }
  for (int l = 0; l < L; ++l) {
    if (res_host[l] < 1 || res_host[l] > (1 << 24)) {
      snprintf(msg, sizeof(msg), "%s: bad size (level resolutions in [1, 2^24])", fn);
      return bad(msg);
    }
    f.R[l] = res_host[l];
    f.Rt[l] = res_host[l] < R_t ? res_host[l] : R_t;
  }
  for (int g = 0; g < G; ++g)
    for (int l = 0; l < L; ++l) {
      const int64_t r = f.R[l] + 1, rc = (f.kind[g] == 0 ? f.R[l] : f.Rt[l]) + 1;
      if (r * r * rc <= T) f.dense[g] |= 1u << l;
    }
  if (!tables_host) return DGM_OK;
  for (int g = 0; g < G; ++g) {
    if (!tables_host[g]) {
      snprintf(msg, sizeof(msg), "%s: null pointer (table %d)", fn, g);
      return bad(msg);
    }
    f.tab[g] = tables_host[g];
  }
  return DGM_OK;
}

bool dghg_timed(const dgm::HgField& f) { return f.kind[f.G - 1] != 0; }
}  // namespace

int dghg_forward(int F, int N, int G, const int32_t* grids_host, int L, int Fe, int log2_table,
                 const int32_t* res_host, int R_t, const float* box, const float* x, const float* t,
                 const float* const* tables_host, float* out, void* stream) {
  dgm::HgField f;
  if (!tables_host) return bad("dghg_forward: null pointer");
  const int rc = dghg_args("dghg_forward", F, N, G, grids_host, L, Fe, log2_table, res_host, R_t, tables_host, f);
  if (rc != DGM_OK) return rc;
  if (F == 0 || N == 0) return DGM_OK;
  if (!box || !x || (!t && dghg_timed(f)) || !out) return bad("dghg_forward: null pointer");
  return check(dgm::launch_hashgrid_fwd(F, N, f, box, x, t, out, (cudaStream_t)stream));
}

int dghg_backward_workspace(int F, int N, int G, const int32_t* grids_host, int L, int Fe, int log2_table,
                            const int32_t* res_host, int R_t, size_t* bytes) {
  dgm::HgField f;
  const int rc = dghg_args("dghg_backward_workspace", F, N, G, grids_host, L, Fe, log2_table, res_host, R_t, nullptr, f);
  if (rc != DGM_OK) return rc;
  if (!bytes) return bad("dghg_backward_workspace: null pointer");
  *bytes = dgm::hg_ws_bytes(f);
  return DGM_OK;
}

int dghg_backward(int F, int N, int G, const int32_t* grids_host, int L, int Fe, int log2_table,
                  const int32_t* res_host, int R_t, const float* box, const float* x, const float* t,
                  const float* const* tables_host, const float* grad_out, float* grad_x,
                  float* const* grad_tables_host, void* ws, size_t ws_bytes, void* stream) {
  dgm::HgField f;
  dgm::HgGrads g;
  if (!tables_host || !grad_tables_host) return bad("dghg_backward: null pointer");
  const int rc = dghg_args("dghg_backward", F, N, G, grids_host, L, Fe, log2_table, res_host, R_t, tables_host, f);
  if (rc != DGM_OK) return rc;
  for (int i = 0; i < G; ++i) {
    if (!grad_tables_host[i]) {
      char msg[200];
      snprintf(msg, sizeof(msg), "dghg_backward: null pointer (table gradient %d)", i);
      return bad(msg);
    }
    g.tab[i] = grad_tables_host[i];
  }
  if (F > 0 && N > 0) {
    if (!box || !x || (!t && dghg_timed(f)) || !grad_out || !ws) return bad("dghg_backward: null pointer");
    const size_t need = dgm::hg_ws_bytes(f);
    if (ws_bytes < need) return dge_short("dghg_backward", ws_bytes, need);
  }
  return check(dgm::launch_hashgrid_bwd(F, N, f, box, x, t, grad_out, grad_x, g, ws, (cudaStream_t)stream));
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
