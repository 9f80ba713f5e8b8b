// raster_feat.cu -- feature maps of caller-chosen per-Gaussian vectors (DESIGN.md §4, "Feature maps and flow"),
// sm_90a.  A pass over the workspaces an existing forward left behind (sorted blend records, tile ranges,
// tile order, n_contrib); no existing kernel or workspace layout changes.
//
//   feature_fwd_kernel          F_c(pix) = sum_i f_{i,c} alpha_i T_i over the colour image's own blend
//   feature_bwd_kernel          dL/dalpha_i (as the six moments, into floats 0-5 of grad_acc) and
//                               dL/df_{i,c} = sum over pixels of alpha_i T_i dL/dF_c (into the feature workspace)
//   feature_grad_finish_kernel  dL/dfeatures from the accumulators of every frame, which it re-zeroes
//
// One CTA per (tile, group of FG = 4 channels, frame): grid (T, ceil(C / 4), F).  Each CTA walks its tile's records
// with the side passes' side_walk (raster_walk.cuh), so the transmittance it sees is the forward's bit for bit,
// gathering the group's four feature values of each record from f[id] (a float4 per record in shared memory), so
// no workspace depends on the record capacity.
#include "../../include/dgmesh_b200.h"
#include "common.cuh"
#include "raster_kernels.h"
#include "raster_walk.cuh"

namespace dgm {

#define FG 4  // channels per group (one float4 per record; the four dL/dF rows of contract_chunk<true>)

namespace {

// this frame's records of the group: positions [base, base + cnt) of the tile, into shared memory
__device__ __forceinline__ void load_feature_batch(const BinWS& b, uint32_t first, int cnt, const float* feats, int C,
                                                   int c0, float4* s_geo, float4* s_con, float4* s_f, uint32_t tid) {
  if ((int)tid < cnt) {
    const size_t r = (size_t)first + tid;
    s_geo[tid] = b.inst_geo[r];
    s_con[tid] = b.inst_attr[2 * r];
    const uint32_t id = __float_as_uint(b.inst_attr[2 * r + 1].w);
    const float* f = feats + (size_t)id * C + c0;
    const int n = min(FG, C - c0);
    float v[FG];
#pragma unroll
    for (int k = 0; k < FG; ++k) v[k] = k < n ? __ldg(f + k) : 0.0f;
    s_f[tid] = make_float4(v[0], v[1], v[2], v[3]);
  }
}

}  // namespace

// features [P,C] (per frame: frame f at features + f P C); out [F,C,H,W].  Frame f's workspaces at
// img_ws + f img_stride, bin_ws + f bin_stride.
__global__ void __launch_bounds__(256, 4) feature_fwd_kernel(int W, int H, int P, int C, const char* img_ws,
                                                             size_t img_stride, const char* bin_ws, size_t bin_stride,
                                                             int64_t R_cap, const float* __restrict__ features,
                                                             int per_frame, float* __restrict__ out) {
  __shared__ __align__(16) float4 s_geo[RB];
  __shared__ __align__(16) float4 s_con[RB];
  __shared__ __align__(16) float4 s_f[RB];
  __shared__ int s_maxc;

  const int f = blockIdx.z, c0 = blockIdx.y * FG;
  SideTile t(W, H, f, img_ws, img_stride, bin_ws, bin_stride, R_cap);
  t.find_stops(&s_maxc, [] {});
  const size_t npix = (size_t)W * H;
  const float* feats = features + (per_frame ? (size_t)f * P * C : 0);

  float T = 1.0f, F0 = 0.f, F1 = 0.f, F2 = 0.f, F3 = 0.f;
  // (the record callable's capture order sets nvcc's register assignment of the sums: compare SASS when changing it)
  side_walk(
      t, s_geo, s_con,
      [&](int base, int cnt) {
        load_feature_batch(t.b, t.range.x + base, cnt, feats, C, c0, s_geo, s_con, s_f, t.tid);
      },
      [&F3, &F2, &F1, &F0, &T](int, int j, float opac, float np, bool pre) {
        if (pre) {
          const float alpha = fminf(0.99f, __fmul_rn(opac, expf(-np)));
          if (!(alpha < 1.0f / 255.0f)) {
            const float4 fv = s_f[j];
            F0 = __fmaf_rn(T, __fmul_rn(alpha, fv.x), F0);
            F1 = __fmaf_rn(T, __fmul_rn(alpha, fv.y), F1);
            F2 = __fmaf_rn(T, __fmul_rn(alpha, fv.z), F2);
            F3 = __fmaf_rn(T, __fmul_rn(alpha, fv.w), F3);
            T = __fmul_rn(T, __fadd_rn(1.0f, -alpha));
          }
        }
      },
      [](int) {});
  if (t.inside) {
    float* o = out + ((size_t)f * C + c0) * npix + t.pix_id;
    const float v[FG] = {F0, F1, F2, F3};
#pragma unroll
    for (int k = 0; k < FG; ++k)
      if (c0 + k < C) o[k * npix] = v[k];
  }
}

// dL/dalpha_i += T_i sum_c (f_{i,c} - F_behind,c) dL/dF_c, walked front to back with the forward's T: the part of
// the map behind record i is T_i F_behind = F - Pref_i, Pref_i the map's prefix through record i, accumulated
// exactly as the forward accumulates the map, so dL/dalpha_i = sum_c dL/dF_c (T_i f_c - (F_c - Pref_i,c) / (1 - a)).
// side_bwd_walk (raster_walk.cuh) contracts w = G dL/dG and alpha T with dL/dF of the group's four channels in its
// four rows: the six moments go to floats 0-5 of grad_acc (dL/dmean2D, dL/dconic, dL/dopacity, as the blend
// backward forms them), the four weight sums to the feature accumulator of the frame (feat_ws + f ws_stride,
// [P, Cp] floats, Cp = C rounded up to 4).  Dynamic shared memory: STAGE_BYTES.
__global__ void __launch_bounds__(256, 2) feature_bwd_kernel(int W, int H, int P, int C, char* geom_ws,
                                                             size_t geom_stride, const char* img_ws, size_t img_stride,
                                                             const char* bin_ws, size_t bin_stride, int64_t R_cap,
                                                             const float* __restrict__ features, int per_frame,
                                                             const float* __restrict__ fmap,
                                                             const float* __restrict__ dL_dfmap, char* feat_ws,
                                                             size_t ws_stride) {
  constexpr int ACC_STRIDE = acc_stride<true>();
  __shared__ __align__(16) float4 s_geo[RB];
  __shared__ __align__(16) float4 s_con[RB];
  __shared__ __align__(16) float4 s_f[RB];
  __shared__ __align__(16) uint32_t s_id[RB];
  __shared__ float s_acc[RB * ACC_STRIDE];
  __shared__ __align__(16) float s_dlp[8][FG][32];
  __shared__ int s_maxc;
  extern __shared__ __align__(16) float s_stage[];  // [8 warps][CHUNK][SLOT_F]

  const int f = blockIdx.z, c0 = blockIdx.y * FG;
  const int Cp = (C + FG - 1) / FG * FG;
  SideTile t(W, H, f, img_ws, img_stride, bin_ws, bin_stride, R_cap);
  const size_t npix = (size_t)W * H;
  float4* const grad_acc = GeomWS::from(geom_ws + f * geom_stride, P).grad_acc;
  float* const facc = reinterpret_cast<float*>(feat_ws + f * ws_stride);
  const float* feats = features + (per_frame ? (size_t)f * P * C : 0);

  float g[FG], Fm[FG], Pf[FG];
  side_bwd_walk(
      t, W, H, &s_maxc, s_geo, s_con, s_id, s_acc, s_dlp, s_stage, grad_acc,
      [&] {  // the group's upstream gradient (the dL/dpixel rows of the contraction) and map values of this pixel
#pragma unroll
        for (int k = 0; k < FG; ++k) {
          const bool ok = t.inside && c0 + k < C;
          const size_t o = ((size_t)f * C + c0 + k) * npix + t.pix_id;
          g[k] = ok ? dL_dfmap[o] : 0.0f;
          Fm[k] = ok ? fmap[o] : 0.0f;
          Pf[k] = 0.0f;
          s_dlp[t.wid][k][t.lane] = g[k];
        }
      },
      [&](int base, int cnt) {
        load_feature_batch(t.b, t.range.x + base, cnt, feats, C, c0, s_geo, s_con, s_f, t.tid);
        if ((int)t.tid < cnt)
          s_id[t.tid] = __float_as_uint(t.b.inst_attr[2 * ((size_t)t.range.x + base + t.tid) + 1].w);
      },
      [&](int j, float alpha, float T, bool act) {
        const float4 fv = s_f[j];
        const float fa[FG] = {fv.x, fv.y, fv.z, fv.w};
        const float r1 = __fdividef(1.0f, 1.0f - alpha);
        float dLa = 0.0f;
#pragma unroll
        for (int c = 0; c < FG; ++c) {
          const float pn = __fmaf_rn(T, __fmul_rn(alpha, fa[c]), Pf[c]);
          Pf[c] = act ? pn : Pf[c];
          dLa = fmaf(g[c], fmaf(T, fa[c], -(Fm[c] - Pf[c]) * r1), dLa);
        }
        return dLa;
      },
      [&](int, uint32_t id, const float* a) { red_add_v4(facc + (size_t)id * Cp + c0, a[6], a[7], a[8], a[9]); });
}

// dL/dfeatures from the feature accumulators of F frames, one thread per (Gaussian, padded channel): per_frame,
// out[f][g][c] = acc_f[g][c]; else out[g][c] = the sum over the frames in frame order.  Every accumulator is
// re-zeroed for the next backward (out NULL: only that).
__global__ void __launch_bounds__(256) feature_grad_finish_kernel(int F, int P, int C, char* feat_ws,
                                                                  size_t ws_stride, int per_frame,
                                                                  float* __restrict__ out) {
  const int Cp = (C + FG - 1) / FG * FG;
  const size_t e = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (e >= (size_t)P * Cp) return;
  const size_t g = e / Cp;
  const int c = (int)(e - g * Cp);
  float sum = 0.0f;
  for (int f = 0; f < F; ++f) {
    float* acc = reinterpret_cast<float*>(feat_ws + f * ws_stride) + e;
    const float v = *acc;
    *acc = 0.0f;
    if (per_frame) {
      if (out && c < C) out[((size_t)f * P + g) * C + c] = v;
    } else {
      sum = f == 0 ? v : sum + v;
    }
  }
  if (!per_frame && out && c < C) out[g * C + c] = sum;
}

size_t feature_ws_stride(int P, int C) {
  const size_t Cp = (size_t)(C + FG - 1) / FG * FG;
  return (sizeof(float) * (size_t)P * Cp + 127) / 128 * 128;
}

cudaError_t launch_features_fwd(const FeatArgs& a, cudaStream_t s) {
  if (a.P == 0) return cudaSuccess;
  const unsigned gx = (a.W + TILE_X - 1) / TILE_X, gy = (a.H + TILE_Y - 1) / TILE_Y;
  const size_t stride = feature_ws_stride(a.P, a.C);
  // the backward adds into the accumulators: they start at zero
  cudaMemsetAsync(a.feat_ws, 0, stride * a.F, s);
  g_prof.begin(10, s);
  feature_fwd_kernel<<<dim3(gx * gy, (a.C + FG - 1) / FG, a.F), 256, 0, s>>>(
      a.W, a.H, a.P, a.C, (const char*)a.img_ws, a.img_stride, (const char*)a.binning_ws, a.binning_stride, a.R_cap,
      a.features, a.per_frame, a.out_map);
  g_prof.end(10, s);
  return cudaGetLastError();
}

cudaError_t launch_features_bwd(const FeatArgs& a, cudaStream_t s) {
  side_bwd_attributes<feature_bwd_kernel>();
  if (a.P == 0) return cudaSuccess;
  const unsigned gx = (a.W + TILE_X - 1) / TILE_X, gy = (a.H + TILE_Y - 1) / TILE_Y;
  const size_t stride = feature_ws_stride(a.P, a.C);
  g_prof.begin(11, s);
  feature_bwd_kernel<<<dim3(gx * gy, (a.C + FG - 1) / FG, a.F), 256, STAGE_BYTES, s>>>(
      a.W, a.H, a.P, a.C, (char*)a.geom_ws, a.geom_stride, (const char*)a.img_ws, a.img_stride,
      (const char*)a.binning_ws, a.binning_stride, a.R_cap, a.features, a.per_frame, a.map, a.dL_dmap,
      (char*)a.feat_ws, stride);
  g_prof.end(11, s);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const size_t n = (size_t)a.P * ((a.C + FG - 1) / FG * FG);
  g_prof.begin(12, s);
  feature_grad_finish_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a.F, a.P, a.C, (char*)a.feat_ws, stride,
                                                                         a.per_frame, a.dL_dfeatures);
  g_prof.end(12, s);
  return cudaGetLastError();
}

}  // namespace dgm
