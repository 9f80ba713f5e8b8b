// raster_bwd.cu -- backward pass of the tile-based 3D-Gaussian rasterizer for sm_90a.
//
//   render_bwd_kernel      gradient of the alpha-composite (role of renderCUDA,
//                          dgr/cuda_rasterizer/backward.cu:399-557)
//   preprocess_bwd_kernel  chain rule to means3D / scales / rotations / SH / opacity
//                          (computeCov2DCUDA + preprocessCUDA, backward.cu:144-396, fused), one
//                          launch for all frames of a batch (CAM: + per-warp partials of the camera gradients)
//   camera_grad_finish_kernel  sums the camera-gradient partials of each frame
//
// The reference issues 9 global float atomics per contributing (pixel, Gaussian)
// pair.  Here the per-Gaussian gradient is written as nine pixel sums over each warp's
// 8x4 block: six moments of w = G * dL/dG (w, w dx, w dy, w dx^2, w dx dy, w dy^2) and
// three colour weights.  Each moment is a polynomial in the pixel's offset (u, v) from
// the block centre, so a lane only stages its two scalars (w, alpha T) per record in
// shared memory; once per chunk of records the warp contracts them (one record per lane
// pair, against the fixed u, v and the staged dL/dpixel) and adds the nine sums into a
// per-tile shared-memory accumulator.  The tile flushes once per (tile, Gaussian) with
// vector reductions (red.global.add.v4.f32) into a [P,12] accumulator that the fused
// preprocess-backward consumes and re-zeroes (render_bwd_kernel<true> also forms dL/d(depth) of the depth map,
// a fourth colour weight, into float 9).  The per-pair arithmetic follows the
// reference's back-to-front recurrence; only the summation order differs (the
// reference's own order is non-deterministic).
//
// render_bwd_kernel and its one launcher, launch_blend_bwd, are in raster_bwd_blend.cuh.  This file compiles the
// colour-only and depth/alpha instances; the normal-map instance and normal_grad_finish_kernel are compiled in
// raster_nrm_bwd.cu, the median-depth / distortion instances and median_grad_kernel in raster_surf_bwd.cu, the
// instances with the absolute screen-space gradient in raster_abs_bwd.cu.  launch_render_bwd below picks the instance
// and hands the call to the file that holds it.
#include "../../include/dgmesh_b200.h"
#include "common.cuh"
#include "raster_math.cuh"
#include "raster_kernels.h"

#include "raster_bwd_blend.cuh"

namespace dgm {

// ===================================================== preprocess (bwd) ====
// SH colour gradient (backward.cu:20-139): returns the dL/d(mean) contribution as (x, y, z) * w, the caller forming
// the products (fused into its sum).  dL/dsh is the outer product dL_dsh[k][ch] = w[k] * dRGB[ch] (w[k] = 0 for
// k >= (deg + 1)^2); the caller forms it from the two factors.
__device__ __forceinline__ float4 sh_backward(int deg, const float3 pos, const float3 campos, const float* sh,
                                              const uint8_t* clamped, const float3 dL_dcolor, float* w /*[16]*/,
                                              float* dRGB /*[3]*/) {
  const float3 dir_orig = make_float3(pos.x - campos.x, pos.y - campos.y, pos.z - campos.z);
  const float len = sqrtf(dir_orig.x * dir_orig.x + dir_orig.y * dir_orig.y + dir_orig.z * dir_orig.z);
  const float x = dir_orig.x / len, y = dir_orig.y / len, z = dir_orig.z / len;
  dRGB[0] = dL_dcolor.x * (clamped[0] ? 0 : 1);
  dRGB[1] = dL_dcolor.y * (clamped[1] ? 0 : 1);
  dRGB[2] = dL_dcolor.z * (clamped[2] ? 0 : 1);
  float ddir[3] = {0.f, 0.f, 0.f};  // dL/d(dir) accumulated over channels
#pragma unroll
  for (int k = 0; k < 16; ++k) w[k] = 0.f;
  w[0] = kSH0;
  float xx = 0, yy = 0, zz = 0, xy = 0, yz = 0, xz = 0;
  if (deg > 0) {
    w[1] = -kSH1 * y;
    w[2] = kSH1 * z;
    w[3] = -kSH1 * x;
    if (deg > 1) {
      xx = x * x, yy = y * y, zz = z * z;
      xy = x * y, yz = y * z, xz = x * z;
      w[4] = kSH2[0] * xy;
      w[5] = kSH2[1] * yz;
      w[6] = kSH2[2] * (2.f * zz - xx - yy);
      w[7] = kSH2[3] * xz;
      w[8] = kSH2[4] * (xx - yy);
      if (deg > 2) {
        w[9] = kSH3[0] * y * (3.f * xx - yy);
        w[10] = kSH3[1] * xy * z;
        w[11] = kSH3[2] * y * (4.f * zz - xx - yy);
        w[12] = kSH3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy);
        w[13] = kSH3[4] * x * (4.f * zz - xx - yy);
        w[14] = kSH3[5] * z * (xx - yy);
        w[15] = kSH3[6] * x * (xx - 3.f * yy);
      }
    }
  }
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    float dx = 0.f, dy = 0.f, dz = 0.f;
    if (deg > 0) {
      dx = -kSH1 * sh[3 * 3 + ch];
      dy = -kSH1 * sh[1 * 3 + ch];
      dz = kSH1 * sh[2 * 3 + ch];
      if (deg > 1) {
        dx += kSH2[0] * y * sh[4 * 3 + ch] + kSH2[2] * 2.f * -x * sh[6 * 3 + ch] + kSH2[3] * z * sh[7 * 3 + ch] +
              kSH2[4] * 2.f * x * sh[8 * 3 + ch];
        dy += kSH2[0] * x * sh[4 * 3 + ch] + kSH2[1] * z * sh[5 * 3 + ch] + kSH2[2] * 2.f * -y * sh[6 * 3 + ch] +
              kSH2[4] * 2.f * -y * sh[8 * 3 + ch];
        dz += kSH2[1] * y * sh[5 * 3 + ch] + kSH2[2] * 2.f * 2.f * z * sh[6 * 3 + ch] + kSH2[3] * x * sh[7 * 3 + ch];
        if (deg > 2) {
          dx += (kSH3[0] * sh[9 * 3 + ch] * 3.f * 2.f * xy + kSH3[1] * sh[10 * 3 + ch] * yz +
                 kSH3[2] * sh[11 * 3 + ch] * -2.f * xy + kSH3[3] * sh[12 * 3 + ch] * -3.f * 2.f * xz +
                 kSH3[4] * sh[13 * 3 + ch] * (-3.f * xx + 4.f * zz - yy) + kSH3[5] * sh[14 * 3 + ch] * 2.f * xz +
                 kSH3[6] * sh[15 * 3 + ch] * 3.f * (xx - yy));
          dy += (kSH3[0] * sh[9 * 3 + ch] * 3.f * (xx - yy) + kSH3[1] * sh[10 * 3 + ch] * xz +
                 kSH3[2] * sh[11 * 3 + ch] * (-3.f * yy + 4.f * zz - xx) +
                 kSH3[3] * sh[12 * 3 + ch] * -3.f * 2.f * yz + kSH3[4] * sh[13 * 3 + ch] * -2.f * xy +
                 kSH3[5] * sh[14 * 3 + ch] * -2.f * yz + kSH3[6] * sh[15 * 3 + ch] * -3.f * 2.f * xy);
          dz += (kSH3[1] * sh[10 * 3 + ch] * xy + kSH3[2] * sh[11 * 3 + ch] * 4.f * 2.f * yz +
                 kSH3[3] * sh[12 * 3 + ch] * 3.f * (2.f * zz - xx - yy) +
                 kSH3[4] * sh[13 * 3 + ch] * 4.f * 2.f * xz + kSH3[5] * sh[14 * 3 + ch] * (xx - yy));
        }
      }
    }
    ddir[0] += dx * dRGB[ch];
    ddir[1] += dy * dRGB[ch];
    ddir[2] += dz * dRGB[ch];
  }
  // through the normalisation dir = v / |v| (auxiliary.h:112-122)
  const float3 vv = dir_orig;
  const float sum2 = vv.x * vv.x + vv.y * vv.y + vv.z * vv.z;
  const float invsum32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
  float4 r;
  r.x = (+sum2 - vv.x * vv.x) * ddir[0] - vv.y * vv.x * ddir[1] - vv.z * vv.x * ddir[2];
  r.y = -vv.x * vv.y * ddir[0] + (sum2 - vv.y * vv.y) * ddir[1] - vv.z * vv.y * ddir[2];
  r.z = -vv.x * vv.z * ddir[0] - vv.y * vv.z * ddir[1] + (sum2 - vv.z * vv.z) * ddir[2];
  r.w = invsum32;
  return r;
}

// ---- per-Gaussian backward of a frame batch (F = 1: one frame).  A block covers NG Gaussians x FB frames per
// pass (FB * NG = NT): warp w takes 32 consecutive Gaussians of frame f0 + w % FB, so per-frame slabs load
// coalesced.  Every output is staged per (frame, Gaussian) in shared memory and written as rows of consecutive
// floats (every store of a warp covers 128 consecutive bytes): gradients of per-frame inputs by the warp that
// staged them, to the frame's slab; gradients of inputs shared by the frames by the whole block once per pass,
// summed over the frames in frame order f = 0, 1, ..., F - 1 (the rounding of F - 1 sequential fp32
// additions).  The SH gradient is staged as its two factors w[16], dRGB[3] and the products are formed by the
// writing thread.
//
// The kernel streams about 220 B per (frame, Gaussian) against a few hundred flops, so it is bound by how many
// bytes are in flight.  A thread therefore issues every load it needs at its top, before the visibility test,
// which only selects the results (a culled Gaussian's gradients are zero).  With sh_smem the block's SH
// coefficients (shared by the frames, 16 per Gaussian) arrive with one bulk copy issued at block start; it
// overlaps the per-frame loads, and the frames' threads read them from shared memory.
// staging slots: the SH factors w[16] and dRGB[3], opacity, colour, mean, scale, rotation, cov3D, 2D mean
#define SL_W 0
#define SL_RGB 16
#define SL_OPAC 19
#define SL_COL 20
#define SL_MEAN 23
#define SL_SCALE 26
#define SL_ROT 29
#define SL_COV 33
#define SL_M2D 39
#define SL_COUNT 42
// CAM: the 27 camera-gradient terms of each (frame, Gaussian), in the order of a camera partial (CAM_* below)
#define SL_CAM 42

// frames per pass of a 256-thread block (one frame: any block size)
static __host__ __device__ inline int pb_frames_per_pass(int F) { return F >= 8 ? 8 : F >= 4 ? 4 : F >= 2 ? 2 : 1; }

// dynamic shared memory of an NT-thread block: the block's SH coefficients (with sh_smem), then the staging area
// (+ CAM_TERMS slots for the camera terms)
static inline size_t pb_smem_bytes(int NT, int F, int M, bool sh_smem, bool cam = false) {
  return (sh_smem ? (size_t)(NT / pb_frames_per_pass(F)) * M * 12 : 0) +
         (size_t)(SL_COUNT + (cam ? CAM_TERMS : 0)) * (NT + 1) * 4;
}

struct PbCams {  // per frame: tan(fov / 2) and focal lengths in pixels
  float tanx[PB_MAX_FRAMES], tany[PB_MAX_FRAMES], fx[PB_MAX_FRAMES], fy[PB_MAX_FRAMES];
};

// NT threads per block.  One frame runs as 128-thread blocks, 3 per SM (the register budget of the one-frame math
// without a cap); a batch as 256-thread blocks, 2 per SM, 128 registers, 8 frames per pass (with CAM 1 per SM: at
// 128 registers the camera terms spill).
// sh_smem: M = 16 and shs is shared by the frames (or there is one frame).
// CAM: also the camera gradients.  Each (frame, Gaussian) stages its CAM_TERMS camera terms; each frame-warp sums
// its 32 Gaussians' terms in Gaussian order into one partial per (frame, 32-Gaussian group), cam_part
// [F][ceil(P/32)][CAM_TERMS], which camera_grad_finish_kernel sums per frame.  Both launch shapes give a warp 32
// consecutive Gaussians of one frame, so the partials do not depend on the shape.
template <int NT, int MIN_BLOCKS, bool CAM>
__global__ void __launch_bounds__(NT, MIN_BLOCKS) preprocess_bwd_kernel(
    int F, int P, int D, int M, int per_frame, const float* __restrict__ means3D, const int* __restrict__ radii,
    const float* __restrict__ shs, int sh_smem, const float* __restrict__ scales,
    const float* __restrict__ rotations, float scale_modifier, const float* __restrict__ cov3D_precomp,
    const float* __restrict__ views, const float* __restrict__ projs, const float* __restrict__ cam_poses,
    const PbCams cams, char* geom_ws, size_t geom_stride, float* __restrict__ dL_dmean2D,
    float* __restrict__ dL_dconic, float* __restrict__ dL_dopacity, float* __restrict__ dL_dcolor,
    float* __restrict__ dL_dmean3D, float* __restrict__ dL_dcov3D, float* __restrict__ dL_dsh,
    float* __restrict__ dL_dscale, float* __restrict__ dL_drot, int depth_grad, float* __restrict__ cam_part) {
  constexpr int PB_STRIDE = NT + 1;  // floats per staging slot: NT (frame, Gaussian) values, + 1 so that slot k starts in bank k
  extern __shared__ __align__(16) float s_dyn[];  // [NG][M * 3] SH coefficients (with sh_smem), then the staging area
  __shared__ __align__(8) uint64_t s_bar;
  pdl_wait();
  pdl_launch();
  const int FB = pb_frames_per_pass(F), NG = NT / FB;
  const int tid = threadIdx.x, wid = tid >> 5;
  const int fi = wid % FB, gl = (wid / FB) * 32 + (tid & 31);
  const int g0 = blockIdx.x * NG, g = g0 + gl, nval = min(NG, P - g0);
  // outputs summed over the frames (DGR_PF_* bits; with one frame every output is that frame's).  dL_dcolor
  // follows the colour input's bit, except with SH colours, where it is [P,3] scratch
  const int sum = F > 1 ? (DGR_PF_ALL & ~per_frame) : 0;
  const bool sum_col = dL_dcolor && F > 1 && (shs || (sum & DGR_PF_COLOR));
  const bool sum_sh = shs && (sum & DGR_PF_COLOR);
  const int ncoef = (D + 1) * (D + 1);
  float* const s_stage = s_dyn + (sh_smem ? NG * 48 : 0);
  float* const stage = s_stage + fi * NG + gl;
  if (sh_smem) {
    if (tid == 0) {
      mbar_init(&s_bar, 1);
      mbar_fence_init();
    }
    __syncthreads();
    if (tid == 0) {
      mbar_expect_tx(&s_bar, nval * 192u);
      tma_load_1d(s_dyn, shs + (size_t)g0 * 48, nval * 192u, &s_bar);
    }
  }

  for (int f0 = 0; f0 < F; f0 += FB) {
    const int f = f0 + fi;
    if (f < F && g < P) {
      const size_t fg = (size_t)f * P + g;
      auto slab = [&](const float* p, int bit, int width) {
        return (per_frame & bit) ? p + (size_t)f * P * width : p;
      };
      const GeomWS gw = GeomWS::from(geom_ws + f * geom_stride, P);
      // ---- every load of this (frame, Gaussian), issued before any of them is used
      const bool visible = (radii ? radii[fg] : gw.radii[g]) > 0;
      const float4 a0 = gw.grad_acc[3 * g + 0], a1 = gw.grad_acc[3 * g + 1], a2 = gw.grad_acc[3 * g + 2];
      const float* mp = slab(means3D, DGR_PF_MEANS, 3) + 3 * g;
      const float3 mean = make_float3(mp[0], mp[1], mp[2]);
      float cov3D[6];
      if (cov3D_precomp) {
        const float* c = slab(cov3D_precomp, DGR_PF_COV, 6) + 6 * g;
#pragma unroll
        for (int k = 0; k < 6; ++k) cov3D[k] = c[k];
      } else {  // the workspace's rows are 8-byte aligned
        const float2* c = reinterpret_cast<const float2*>(gw.cov3D + 6 * g);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const float2 v = c[k];
          cov3D[2 * k] = v.x;
          cov3D[2 * k + 1] = v.y;
        }
      }
      const float* sc_f = scales ? slab(scales, DGR_PF_SCALES, 3) : nullptr;
      const float* rot_f = rotations ? slab(rotations, DGR_PF_ROTS, 4) : nullptr;
      if (sc_f) {  // parked in the slots of their gradients until the EWA gradient is done (register budget)
        const float4 q = __ldg(reinterpret_cast<const float4*>(rot_f) + g);
#pragma unroll
        for (int k = 0; k < 3; ++k) stage[(SL_SCALE + k) * PB_STRIDE] = sc_f[3 * g + k];
        stage[(SL_ROT + 0) * PB_STRIDE] = q.x;
        stage[(SL_ROT + 1) * PB_STRIDE] = q.y;
        stage[(SL_ROT + 2) * PB_STRIDE] = q.z;
        stage[(SL_ROT + 3) * PB_STRIDE] = q.w;
      }
      // clear the accumulators written by render_bwd_kernel
      gw.grad_acc[3 * g + 0] = make_float4(0, 0, 0, 0);
      gw.grad_acc[3 * g + 1] = make_float4(0, 0, 0, 0);
      gw.grad_acc[3 * g + 2] = make_float4(0, 0, 0, 0);
      const float3 dcon = make_float3(a0.z, a0.w, a1.x);  // (xx, xy, yy) slots .x .y .w of the reference float4
      // the 2D mean and colour gradients are read back from the staging area where they are used (fewer live
      // registers through the EWA gradient)
      stage[(SL_M2D + 0) * PB_STRIDE] = a0.x;
      stage[(SL_M2D + 1) * PB_STRIDE] = a0.y;
      stage[(SL_M2D + 2) * PB_STRIDE] = 0.f;
      if (dL_dconic) reinterpret_cast<float4*>(dL_dconic)[fg] = make_float4(dcon.x, dcon.y, 0.f, dcon.z);
      stage[SL_OPAC * PB_STRIDE] = a1.y;
      stage[(SL_COL + 0) * PB_STRIDE] = a1.z;
      stage[(SL_COL + 1) * PB_STRIDE] = a1.w;
      stage[(SL_COL + 2) * PB_STRIDE] = a2.x;
      stage[SL_MEAN * PB_STRIDE] = a2.y;  // dL/d(depth), until dL/dmean3D takes the slot

      float dcov[6] = {0, 0, 0, 0, 0, 0};
      float3 dmean = make_float3(0, 0, 0);
      float3 dscale = make_float3(0, 0, 0);
      float4 drot = make_float4(0, 0, 0, 0);
      float w[16], dRGB[3] = {0.f, 0.f, 0.f};
#pragma unroll
      for (int k = 0; k < 16; ++k) w[k] = 0.f;
      {
        const float* view = views + 16 * f;
        const float* proj = projs + 16 * f;
        const float focal_x = cams.fx[f], focal_y = cams.fy[f], tan_fovx = cams.tanx[f], tan_fovy = cams.tany[f];
        // ---------------- gradient through the 2D covariance / conic (backward.cu:144-274)
        EwaFrame fr;
        ewa_frame(mean, focal_x, focal_y, tan_fovx, tan_fovy, cov3D, view, fr);
        const float limx = 1.3f * tan_fovx, limy = 1.3f * tan_fovy;
        const float x_grad_mul = fr.txtz < -limx || fr.txtz > limx ? 0 : 1;
        const float y_grad_mul = fr.tytz < -limy || fr.tytz > limy ? 0 : 1;
        const float3 c2 = ewa_cov2d(fr);
        const float a = c2.x, b = c2.y, c = c2.z;
        const float denom = a * c - b * b;
        float dL_da = 0, dL_db = 0, dL_dc = 0;
        const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
        const Mat3& T = fr.T;
        const Mat3& Vrk = fr.Vrk;
        if (denom2inv != 0) {
          dL_da = denom2inv * (-c * c * dcon.x + 2 * b * c * dcon.y + (denom - a * c) * dcon.z);
          dL_dc = denom2inv * (-a * a * dcon.z + 2 * a * b * dcon.y + (denom - a * c) * dcon.x);
          dL_db = denom2inv * 2 * (b * c * dcon.x - (denom + 2 * b * b) * dcon.y + a * b * dcon.z);
          dcov[0] = (T.c[0][0] * T.c[0][0] * dL_da + T.c[0][0] * T.c[1][0] * dL_db + T.c[1][0] * T.c[1][0] * dL_dc);
          dcov[3] = (T.c[0][1] * T.c[0][1] * dL_da + T.c[0][1] * T.c[1][1] * dL_db + T.c[1][1] * T.c[1][1] * dL_dc);
          dcov[5] = (T.c[0][2] * T.c[0][2] * dL_da + T.c[0][2] * T.c[1][2] * dL_db + T.c[1][2] * T.c[1][2] * dL_dc);
          dcov[1] = 2 * T.c[0][0] * T.c[0][1] * dL_da + (T.c[0][0] * T.c[1][1] + T.c[0][1] * T.c[1][0]) * dL_db +
                    2 * T.c[1][0] * T.c[1][1] * dL_dc;
          dcov[2] = 2 * T.c[0][0] * T.c[0][2] * dL_da + (T.c[0][0] * T.c[1][2] + T.c[0][2] * T.c[1][0]) * dL_db +
                    2 * T.c[1][0] * T.c[1][2] * dL_dc;
          dcov[4] = 2 * T.c[0][2] * T.c[0][1] * dL_da + (T.c[0][1] * T.c[1][2] + T.c[0][2] * T.c[1][1]) * dL_db +
                    2 * T.c[1][1] * T.c[1][2] * dL_dc;
        }
        const float dL_dT00 = 2 * (T.c[0][0] * Vrk.c[0][0] + T.c[0][1] * Vrk.c[0][1] + T.c[0][2] * Vrk.c[0][2]) * dL_da +
                              (T.c[1][0] * Vrk.c[0][0] + T.c[1][1] * Vrk.c[0][1] + T.c[1][2] * Vrk.c[0][2]) * dL_db;
        const float dL_dT01 = 2 * (T.c[0][0] * Vrk.c[1][0] + T.c[0][1] * Vrk.c[1][1] + T.c[0][2] * Vrk.c[1][2]) * dL_da +
                              (T.c[1][0] * Vrk.c[1][0] + T.c[1][1] * Vrk.c[1][1] + T.c[1][2] * Vrk.c[1][2]) * dL_db;
        const float dL_dT02 = 2 * (T.c[0][0] * Vrk.c[2][0] + T.c[0][1] * Vrk.c[2][1] + T.c[0][2] * Vrk.c[2][2]) * dL_da +
                              (T.c[1][0] * Vrk.c[2][0] + T.c[1][1] * Vrk.c[2][1] + T.c[1][2] * Vrk.c[2][2]) * dL_db;
        const float dL_dT10 = 2 * (T.c[1][0] * Vrk.c[0][0] + T.c[1][1] * Vrk.c[0][1] + T.c[1][2] * Vrk.c[0][2]) * dL_dc +
                              (T.c[0][0] * Vrk.c[0][0] + T.c[0][1] * Vrk.c[0][1] + T.c[0][2] * Vrk.c[0][2]) * dL_db;
        const float dL_dT11 = 2 * (T.c[1][0] * Vrk.c[1][0] + T.c[1][1] * Vrk.c[1][1] + T.c[1][2] * Vrk.c[1][2]) * dL_dc +
                              (T.c[0][0] * Vrk.c[1][0] + T.c[0][1] * Vrk.c[1][1] + T.c[0][2] * Vrk.c[1][2]) * dL_db;
        const float dL_dT12 = 2 * (T.c[1][0] * Vrk.c[2][0] + T.c[1][1] * Vrk.c[2][1] + T.c[1][2] * Vrk.c[2][2]) * dL_dc +
                              (T.c[0][0] * Vrk.c[2][0] + T.c[0][1] * Vrk.c[2][1] + T.c[0][2] * Vrk.c[2][2]) * dL_db;
        // camera term c of this (frame, Gaussian); a culled Gaussian's are zero
        auto cam = [&](int c, float v) { stage[(SL_CAM + c) * PB_STRIDE] = visible ? v : 0.f; };
        if (CAM) {  // view, through W in T = W J (T.c[r][k] = sum_j J.c[r][j] W.c[j][k], W.c[j][k] = v[4k+j])
          const float t_z = fr.t.z;
          const float J00 = focal_x / t_z, J11 = focal_y / t_z;
          const float J02 = -(focal_x * fr.t.x) / (t_z * t_z), J12 = -(focal_y * fr.t.y) / (t_z * t_z);
          const float dT0[3] = {dL_dT00, dL_dT01, dL_dT02}, dT1[3] = {dL_dT10, dL_dT11, dL_dT12};
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            stage[(SL_CAM + 3 * k + 0) * PB_STRIDE] = J00 * dT0[k];
            stage[(SL_CAM + 3 * k + 1) * PB_STRIDE] = J11 * dT1[k];
            stage[(SL_CAM + 3 * k + 2) * PB_STRIDE] = fmaf(J02, dT0[k], J12 * dT1[k]);
          }
        }
        const Mat3& Wm = fr.W;
        const float dL_dJ00 = Wm.c[0][0] * dL_dT00 + Wm.c[0][1] * dL_dT01 + Wm.c[0][2] * dL_dT02;
        const float dL_dJ02 = Wm.c[2][0] * dL_dT00 + Wm.c[2][1] * dL_dT01 + Wm.c[2][2] * dL_dT02;
        const float dL_dJ11 = Wm.c[1][0] * dL_dT10 + Wm.c[1][1] * dL_dT11 + Wm.c[1][2] * dL_dT12;
        const float dL_dJ12 = Wm.c[2][0] * dL_dT10 + Wm.c[2][1] * dL_dT11 + Wm.c[2][2] * dL_dT12;
        const float tz = 1.f / fr.t.z;
        const float tz2 = tz * tz;
        const float tz3 = tz2 * tz;
        const float dL_dtx = x_grad_mul * -focal_x * tz2 * dL_dJ02;
        const float dL_dty = y_grad_mul * -focal_y * tz2 * dL_dJ12;
        const float dL_dtz = -focal_x * tz2 * dL_dJ00 - focal_y * tz2 * dL_dJ11 + (2 * focal_x * fr.t.x) * tz3 * dL_dJ02 +
                             (2 * focal_y * fr.t.y) * tz3 * dL_dJ12;
        dmean = xform_vec4x3_T(make_float3(dL_dtx, dL_dty, dL_dtz), view);
        if (CAM) {  // view, through t = W m + v[12..14]: dL/dv[4k+j] = dL/dt_j mh_k (+ the W term staged above)
          const float dtz = depth_grad ? dL_dtz + stage[SL_MEAN * PB_STRIDE] : dL_dtz;  // depth = t_z
          const float dt[3] = {dL_dtx, dL_dty, dtz}, mh[3] = {mean.x, mean.y, mean.z};
#pragma unroll
          for (int k = 0; k < 3; ++k)
#pragma unroll
            for (int j = 0; j < 3; ++j) cam(3 * k + j, fmaf(dt[j], mh[k], stage[(SL_CAM + 3 * k + j) * PB_STRIDE]));
#pragma unroll
          for (int j = 0; j < 3; ++j) cam(9 + j, dt[j]);
        }

        // ---------------- screen-space mean -> 3D mean (backward.cu:366-381)
        const float4 m_hom = xform4x4(mean, proj);
        const float m_w = 1.0f / (m_hom.w + 0.0000001f);
        const float mul1 = (proj[0] * mean.x + proj[4] * mean.y + proj[8] * mean.z + proj[12]) * m_w * m_w;
        const float mul2 = (proj[1] * mean.x + proj[5] * mean.y + proj[9] * mean.z + proj[13]) * m_w * m_w;
        float3 dm;
        const float2 dm2 = make_float2(stage[SL_M2D * PB_STRIDE], stage[(SL_M2D + 1) * PB_STRIDE]);
        dm.x = (proj[0] * m_w - proj[3] * mul1) * dm2.x + (proj[1] * m_w - proj[3] * mul2) * dm2.y;
        dm.y = (proj[4] * m_w - proj[7] * mul1) * dm2.x + (proj[5] * m_w - proj[7] * mul2) * dm2.y;
        dm.z = (proj[8] * m_w - proj[11] * mul1) * dm2.x + (proj[9] * m_w - proj[11] * mul2) * dm2.y;
        dmean.x += dm.x;
        dmean.y += dm.y;
        dmean.z += dm.z;
        if (CAM) {  // projection: dL/dproj[4k+i] = (g.x m_w, g.y m_w, -(g.x mul1 + g.y mul2))_i mh_k, i = 0, 1, 3
          const float gp[3] = {dm2.x * m_w, dm2.y * m_w, -fmaf(dm2.x, mul1, dm2.y * mul2)};
          const float mh[4] = {mean.x, mean.y, mean.z, 1.0f};
#pragma unroll
          for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int i = 0; i < 3; ++i) cam(12 + 3 * k + i, gp[i] * mh[k]);
        }
        // depth map: dL/d(depth) (grad_acc float 9) through depth = p_view.z, the third row of the view
        // transform (xform4x3).  Only when the backward carries one: adding 0 would turn -0 into +0
        if (depth_grad) {
          const float dd = stage[SL_MEAN * PB_STRIDE];
          dmean.x += dd * view[2];
          dmean.y += dd * view[6];
          dmean.z += dd * view[10];
        }

        // ---------------- 3D covariance -> scale / rotation (backward.cu:279-341)
        if (sc_f) {
          const float3 sc = make_float3(stage[SL_SCALE * PB_STRIDE], stage[(SL_SCALE + 1) * PB_STRIDE],
                                        stage[(SL_SCALE + 2) * PB_STRIDE]);
          const float4 q = make_float4(stage[SL_ROT * PB_STRIDE], stage[(SL_ROT + 1) * PB_STRIDE],
                                       stage[(SL_ROT + 2) * PB_STRIDE], stage[(SL_ROT + 3) * PB_STRIDE]);
          const float r = q.x, x = q.y, y = q.z, z = q.w;
          Mat3 R;
          quat_to_R(q, R);
          const float3 s = make_float3(scale_modifier * sc.x, scale_modifier * sc.y, scale_modifier * sc.z);
          Mat3 S;
#pragma unroll
          for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) S.c[i][j] = (i == j) ? 1.0f : 0.0f;
          S.c[0][0] = s.x;
          S.c[1][1] = s.y;
          S.c[2][2] = s.z;
          const Mat3 Mm = mat3_mul(S, R);
          Mat3 dSig;
          dSig.c[0][0] = dcov[0];
          dSig.c[0][1] = 0.5f * dcov[1];
          dSig.c[0][2] = 0.5f * dcov[2];
          dSig.c[1][0] = 0.5f * dcov[1];
          dSig.c[1][1] = dcov[3];
          dSig.c[1][2] = 0.5f * dcov[4];
          dSig.c[2][0] = 0.5f * dcov[2];
          dSig.c[2][1] = 0.5f * dcov[4];
          dSig.c[2][2] = dcov[5];
          Mat3 M2;
#pragma unroll
          for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) M2.c[i][j] = 2.0f * Mm.c[i][j];
          const Mat3 dL_dM = mat3_mul(M2, dSig);
          const Mat3 Rt = mat3_T(R);
          Mat3 dMt = mat3_T(dL_dM);
          dscale.x = Rt.c[0][0] * dMt.c[0][0] + Rt.c[0][1] * dMt.c[0][1] + Rt.c[0][2] * dMt.c[0][2];
          dscale.y = Rt.c[1][0] * dMt.c[1][0] + Rt.c[1][1] * dMt.c[1][1] + Rt.c[1][2] * dMt.c[1][2];
          dscale.z = Rt.c[2][0] * dMt.c[2][0] + Rt.c[2][1] * dMt.c[2][1] + Rt.c[2][2] * dMt.c[2][2];
#pragma unroll
          for (int j = 0; j < 3; ++j) {
            dMt.c[0][j] *= s.x;
            dMt.c[1][j] *= s.y;
            dMt.c[2][j] *= s.z;
          }
          drot.x = 2 * z * (dMt.c[0][1] - dMt.c[1][0]) + 2 * y * (dMt.c[2][0] - dMt.c[0][2]) +
                   2 * x * (dMt.c[1][2] - dMt.c[2][1]);
          drot.y = 2 * y * (dMt.c[1][0] + dMt.c[0][1]) + 2 * z * (dMt.c[2][0] + dMt.c[0][2]) +
                   2 * r * (dMt.c[1][2] - dMt.c[2][1]) - 4 * x * (dMt.c[2][2] + dMt.c[1][1]);
          drot.z = 2 * x * (dMt.c[1][0] + dMt.c[0][1]) + 2 * r * (dMt.c[2][0] - dMt.c[0][2]) +
                   2 * z * (dMt.c[1][2] + dMt.c[2][1]) - 4 * y * (dMt.c[2][2] + dMt.c[0][0]);
          drot.w = 2 * r * (dMt.c[0][1] - dMt.c[1][0]) + 2 * x * (dMt.c[2][0] + dMt.c[0][2]) +
                   2 * y * (dMt.c[1][2] + dMt.c[2][1]) - 4 * z * (dMt.c[1][1] + dMt.c[0][0]);
        }
        // a culled Gaussian's gradients are zero: the visibility test selects the results
        auto vis = [&](float v) { return visible ? v : 0.f; };
#pragma unroll
        for (int k = 0; k < 6; ++k) stage[(SL_COV + k) * PB_STRIDE] = vis(dcov[k]);
        stage[(SL_SCALE + 0) * PB_STRIDE] = vis(dscale.x);
        stage[(SL_SCALE + 1) * PB_STRIDE] = vis(dscale.y);
        stage[(SL_SCALE + 2) * PB_STRIDE] = vis(dscale.z);
        stage[(SL_ROT + 0) * PB_STRIDE] = vis(drot.x);
        stage[(SL_ROT + 1) * PB_STRIDE] = vis(drot.y);
        stage[(SL_ROT + 2) * PB_STRIDE] = vis(drot.z);
        stage[(SL_ROT + 3) * PB_STRIDE] = vis(drot.w);

        // ---------------- SH colour (backward.cu:20-139, 383-385)
        if (shs) {
          const float3 cp = make_float3(cam_poses[3 * f], cam_poses[3 * f + 1], cam_poses[3 * f + 2]);
          float sh[48];
          if (!sh_smem) {
            load_sh(slab(shs, DGR_PF_COLOR, M * 3), g, M, ncoef, sh);
          } else {
            mbar_wait(&s_bar, 0);
            const float4* v = reinterpret_cast<const float4*>(s_dyn + gl * 48);
#pragma unroll
            for (int i = 0; i < 12; ++i) {
              const float4 t = v[i];
              sh[4 * i + 0] = t.x;
              sh[4 * i + 1] = t.y;
              sh[4 * i + 2] = t.z;
              sh[4 * i + 3] = t.w;
            }
          }
          const float3 dcol = make_float3(stage[SL_COL * PB_STRIDE], stage[(SL_COL + 1) * PB_STRIDE],
                                          stage[(SL_COL + 2) * PB_STRIDE]);
          const float4 dms = sh_backward(D, mean, cp, sh, gw.clamped + 3 * g, dcol, w, dRGB);
          // explicit fused sums: the camera term below takes the products too, which would otherwise change
          // whether the compiler fuses them here (dL/dmean3D must not depend on CAM)
          dmean.x = fmaf(dms.x, dms.w, dmean.x);
          dmean.y = fmaf(dms.y, dms.w, dmean.y);
          dmean.z = fmaf(dms.z, dms.w, dmean.z);
          if (CAM) {  // the SH direction is mean - campos
            cam(24, -(dms.x * dms.w));
            cam(25, -(dms.y * dms.w));
            cam(26, -(dms.z * dms.w));
          }
        } else if (CAM) {
          cam(24, 0.f);
          cam(25, 0.f);
          cam(26, 0.f);
        }
#pragma unroll
        for (int k = 0; k < 16; ++k) stage[(SL_W + k) * PB_STRIDE] = vis(w[k]);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) stage[(SL_RGB + ch) * PB_STRIDE] = vis(dRGB[ch]);
        stage[(SL_MEAN + 0) * PB_STRIDE] = vis(dmean.x);
        stage[(SL_MEAN + 1) * PB_STRIDE] = vis(dmean.y);
        stage[(SL_MEAN + 2) * PB_STRIDE] = vis(dmean.z);
      }
    }
    // ---- per-frame outputs: each warp writes the rows of its own 32 Gaussians as soon as it has staged them
    // (element e = q * width + c of the warp's slice is row q, column c: every store of the warp covers 128
    // consecutive bytes), without waiting for the rest of the block
    if (f < F) {  // uniform per warp
      __syncwarp();
      const int gw0 = (wid / FB) * 32, nw = min(32, P - g0 - gw0);
      const float* ws = s_stage + fi * NG + gw0;
      auto own = [&](float* out, int width, auto value) {
        float* dst = out + ((size_t)f * P + g0 + gw0) * width;
#pragma unroll 4
        for (int j = 0; j < width; ++j) {
          const int e = (tid & 31) + 32 * j, q = e / width, c = e - q * width;
          if (q < nw) dst[e] = value(ws, q, c);
        }
      };
      auto staged = [](int slot) {
        return [=](const float* st, int q, int c) { return st[(slot + c) * PB_STRIDE + q]; };
      };
      own(dL_dmean2D, 3, staged(SL_M2D));
      if (!(sum & DGR_PF_OPAC)) own(dL_dopacity, 1, staged(SL_OPAC));
      if (dL_dcolor && !sum_col) own(dL_dcolor, 3, staged(SL_COL));
      if (!(sum & DGR_PF_MEANS)) own(dL_dmean3D, 3, staged(SL_MEAN));
      if (dL_dcov3D && !(sum & DGR_PF_COV)) own(dL_dcov3D, 6, staged(SL_COV));
      if (!(sum & DGR_PF_SCALES)) own(dL_dscale, 3, staged(SL_SCALE));
      if (!(sum & DGR_PF_ROTS)) own(dL_drot, 4, staged(SL_ROT));
      // dL_dsh[k][ch] = w[k] dRGB[ch]; 0 for the coefficients k >= ncoef that the SH degree does not use
      if (shs && !sum_sh)
        own(dL_dsh, 3 * M, [=](const float* st, int q, int c) {
          const int k = c / 3;
          return k < ncoef ? __fmul_rn(st[(SL_W + k) * PB_STRIDE + q], st[(SL_RGB + c - 3 * k) * PB_STRIDE + q]) : 0.f;
        });
      // camera partial of this (frame, 32-Gaussian group): lane c sums term c over the group in Gaussian order
      if (CAM && nw > 0 && (tid & 31) < CAM_TERMS) {
        const int c = tid & 31;
        const float* src = ws + (SL_CAM + c) * PB_STRIDE;
        float acc = src[0];
        for (int q = 1; q < nw; ++q) acc += src[q];
        cam_part[((size_t)f * ((P + 31) >> 5) + ((g0 + gw0) >> 5)) * CAM_TERMS + c] = acc;
      }
      __syncwarp();
    }
    if (!sum && !sum_col) continue;  // uniform: nothing is summed over the frames
    __syncthreads();
    // ---- outputs summed over the frames: the block sums this pass's frames into its rows, in frame order,
    // continuing from the value the previous pass stored.  value(q, c, i) is frame i's staged value
    const int nf = min(FB, F - f0);
    auto sum_rows = [&](float* out, int width, auto value) {
      float* dst = out + (size_t)g0 * width;
      for (int e = tid; e < nval * width; e += NT) {
        const int q = e / width, c = e - q * width;
        float v[8];  // FB <= 8: every frame's value is read before the sequential sum
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = i < nf ? value(q, c, i) : 0.f;
        float acc = f0 ? dst[e] : v[0];
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (i < nf && (f0 || i > 0)) acc = acc + v[i];
        dst[e] = acc;
      }
    };
    auto summed = [&](int slot) {
      return [=](int q, int c, int i) { return s_stage[(slot + c) * PB_STRIDE + i * NG + q]; };
    };
    if (sum & DGR_PF_OPAC) sum_rows(dL_dopacity, 1, summed(SL_OPAC));
    if (sum_col) sum_rows(dL_dcolor, 3, summed(SL_COL));
    if (sum & DGR_PF_MEANS) sum_rows(dL_dmean3D, 3, summed(SL_MEAN));
    if ((sum & DGR_PF_COV) && dL_dcov3D) sum_rows(dL_dcov3D, 6, summed(SL_COV));
    if (sum & DGR_PF_SCALES) sum_rows(dL_dscale, 3, summed(SL_SCALE));
    if (sum & DGR_PF_ROTS) sum_rows(dL_drot, 4, summed(SL_ROT));
    // each product rounded before it is added; 0 for k >= ncoef
    if (sum_sh)
      sum_rows(dL_dsh, 3 * M, [=](int q, int c, int i) {
        const int k = c / 3;
        return k < ncoef ? __fmul_rn(s_stage[(SL_W + k) * PB_STRIDE + i * NG + q],
                                     s_stage[(SL_RGB + c - 3 * k) * PB_STRIDE + i * NG + q])
                         : 0.f;
      });
    __syncthreads();  // the next pass overwrites the staging area
  }
}

// Camera gradients of frame blockIdx.x from its ceil(P/32) = G partials (preprocess_bwd_kernel<.., true>): thread
// (r, c) of the 32 x CAM_TERMS block sums term c of the partials r, r + 32, r + 64, ... in that order (a warp reads
// 32 consecutive floats), then thread c sums the 32 row sums in row order.  The order depends on P only.
__global__ void __launch_bounds__(32 * CAM_TERMS) camera_grad_finish_kernel(int G, const float* __restrict__ part,
                                                                            float* __restrict__ dL_dview,
                                                                            float* __restrict__ dL_dproj,
                                                                            float* __restrict__ dL_dcampos) {
  __shared__ float s_row[32][CAM_TERMS];
  const int f = blockIdx.x, t = threadIdx.x, r = t / CAM_TERMS, c = t - r * CAM_TERMS;
  const float* p = part + (size_t)f * G * CAM_TERMS + c;
  float acc = 0.f;
#pragma unroll 8
  for (int i = r; i < G; i += 32) acc += p[(size_t)i * CAM_TERMS];
  s_row[r][c] = acc;
  __syncthreads();
  if (t >= 35) return;
  // output t: dL/dview[t] (t < 16), dL/dproj[t - 16] (t < 32), dL/dcampos[t - 32]; -1: structurally zero
  int src;
  if (t < 16) src = (t & 3) == 3 ? -1 : 3 * (t >> 2) + (t & 3);
  else if (t < 32) src = ((t - 16) & 3) == 2 ? -1 : 12 + 3 * ((t - 16) >> 2) + min((t - 16) & 3, 2);
  else src = 24 + t - 32;
  float v = 0.f;
  if (src >= 0) {
    v = s_row[0][src];
    for (int q = 1; q < 32; ++q) v += s_row[q][src];
  }
  if (t < 16) {
    if (dL_dview) dL_dview[16 * f + t] = v;
  } else if (t < 32) {
    if (dL_dproj) dL_dproj[16 * f + t - 16] = v;
  } else if (dL_dcampos) {
    dL_dcampos[3 * f + t - 32] = v;
  }
}

// gradient of the alpha-compositing (fills the GPU); leaves the per-Gaussian moments in grad_acc.  The instance follows
// the rule of launch_blend_bwd
cudaError_t launch_render_bwd(const BwdArgs& a, cudaStream_t s) {
  if (a.dL_dmean2D_abs) return launch_render_bwd_abs(a, s);  // raster_abs_bwd.cu
  if (a.dL_ddistortion) return launch_render_bwd_surf(a, s);  // raster_surf_bwd.cu
  if (a.dL_dnormal) return launch_render_bwd_nrm(a, s);  // raster_nrm_bwd.cu
  return (a.dL_ddepth || a.dL_dalpha) ? launch_blend_bwd<true, false, false, false>(a, s)
                                      : launch_blend_bwd<false, false, false, false>(a, s);
}

// chain rule from the moments to the inputs, all frames of a batch in one launch (after every frame's
// render_bwd_kernel)
cudaError_t launch_preprocess_bwd(const BwdArgs& a, cudaStream_t s) {
  if (a.P == 0) return cudaSuccess;
  if (a.F < 1 || a.F > PB_MAX_FRAMES) return cudaErrorInvalidValue;
  PbCams c = {};
  for (int f = 0; f < a.F; ++f) {
    c.tanx[f] = a.tan_fovx[f];
    c.tany[f] = a.tan_fovy[f];
    c.fx[f] = a.W / (2.0f * a.tan_fovx[f]);
    c.fy[f] = a.H / (2.0f * a.tan_fovy[f]);
  }
  auto one = preprocess_bwd_kernel<128, 3, false>, batch = preprocess_bwd_kernel<256, 2, false>;
  auto one_cam = preprocess_bwd_kernel<128, 3, true>, batch_cam = preprocess_bwd_kernel<256, 1, true>;
  static unsigned long long attr = 0;  // per device
  if (once_per_device(attr)) {
    // the largest staging area + SH tile (2 or 3 frames: 128 Gaussians per block) exceeds 48 KB
    cudaFuncSetAttribute(one, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pb_smem_bytes(128, 1, 16, true));
    cudaFuncSetAttribute(batch, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pb_smem_bytes(256, 2, 16, true));
    cudaFuncSetAttribute(one_cam, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)pb_smem_bytes(128, 1, 16, true, true));
    cudaFuncSetAttribute(batch_cam, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)pb_smem_bytes(256, 2, 16, true, true));
  }
  const bool cam = a.dL_dview || a.dL_dproj || a.dL_dcampos;
  if (cam && !a.cam_ws) return cudaErrorInvalidValue;
  // 16 SH coefficients per Gaussian are read as 16-byte vectors throughout (load_sh): 192-byte rows, aligned
  const bool sh_smem = a.shs && a.M == 16 && (a.F == 1 || !(a.per_frame & DGR_PF_COLOR));
  const int nt = a.F == 1 ? 128 : 256, ng = nt / pb_frames_per_pass(a.F);
  auto k = a.F == 1 ? (cam ? one_cam : one) : (cam ? batch_cam : batch);
  g_prof.begin(6, s);  // with camera gradients, the time includes the finishing kernel
  launch_pdl(k, dim3((a.P + ng - 1) / ng), dim3(nt), pb_smem_bytes(nt, a.F, a.M, sh_smem, cam), s, a.F, a.P, a.D,
             a.M, a.per_frame, a.means3D, a.radii, a.shs, sh_smem ? 1 : 0, a.scales, a.rotations, a.scale_modifier,
             a.cov3D_precomp, a.viewmatrix, a.projmatrix, a.cam_pos, c, (char*)a.geom_ws, a.geom_stride,
             a.dL_dmean2D, a.dL_dconic, a.dL_dopacity, a.dL_dcolor, a.dL_dmean3D, a.dL_dcov3D, a.dL_dsh, a.dL_dscale,
             a.dL_drot, (a.dL_ddepth || a.dL_dmedian || a.dL_ddistortion) ? 1 : 0, a.cam_ws);
  if (cam)
    camera_grad_finish_kernel<<<a.F, 32 * CAM_TERMS, 0, s>>>((a.P + 31) / 32, a.cam_ws, a.dL_dview, a.dL_dproj,
                                                              a.dL_dcampos);
  g_prof.end(6, s);
  return cudaGetLastError();
}

}  // namespace dgm
