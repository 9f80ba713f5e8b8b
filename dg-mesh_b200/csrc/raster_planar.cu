// raster_planar.cu -- the planar-depth maps (DESIGN.md §4, "Planar depth"), sm_90a.  A pass over the workspaces an
// existing forward left behind, like the feature pass (raster_feat.cu); no existing kernel or workspace layout
// changes.  Record i paints the depth of its plane (gaussian_planes.cu) at the pixel centre p,
// d_i(p) = t_z + g . (p - mu2D_i), mu2D_i the record's own screen mean (inst_geo.xy):
//
//   planar_fwd_kernel          planar_depth = sum_i d_i(p) alpha_i T_i and planar_median_depth = d_i(p) of the last
//                              record blended while T > 0.5, over the colour image's own blend; the median record's
//                              id per pixel into the planar workspace
//   planar_bwd_kernel          dL/dalpha_i (the six moments, into floats 0-5 of grad_acc), -g sum e into floats 0-1
//                              (dL/dmean2D) and (sum e, sum e dx, sum e dy), e = alpha T dL/dD, into the plane
//                              accumulator of the frame
//   planar_median_grad_kernel  the same two terms of dL/dmedian at each pixel's median record
//   planar_grad_finish_kernel  dL/dplanes from the accumulators, which it re-zeroes
//
// One CTA per (tile, frame), walked with side_walk (raster_walk.cuh), so T is the forward's bit for bit.
#include "../../include/dgmesh_b200.h"
#include "common.cuh"
#include "raster_kernels.h"
#include "raster_walk.cuh"

namespace dgm {

namespace {

// frame f's planar workspace: the plane accumulator [P] float4 (sum e, sum e dx, sum e dy, 0), then the median
// record's id per pixel (0xFFFFFFFF: none)
struct PlanarWS {
  float4* acc;
  uint32_t* median_id;
  __host__ __device__ static PlanarWS from(char* base, size_t P) {
    PlanarWS w;
    w.acc = reinterpret_cast<float4*>(base);
    w.median_id = reinterpret_cast<uint32_t*>(base + (P * sizeof(float4) + 127) / 128 * 128);
    return w;
  }
};

__device__ __forceinline__ void load_planar_batch(const BinWS& b, uint32_t first, int cnt, const float* planes,
                                                  float4* s_geo, float4* s_con, float4* s_pl, uint32_t* s_id,
                                                  uint32_t tid) {
  if ((int)tid < cnt) {
    const size_t r = (size_t)first + tid;
    s_geo[tid] = b.inst_geo[r];
    s_con[tid] = b.inst_attr[2 * r];
    const uint32_t id = __float_as_uint(b.inst_attr[2 * r + 1].w);
    const float* p = planes + 3 * (size_t)id;
    s_pl[tid] = make_float4(__ldg(p), __ldg(p + 1), __ldg(p + 2), 0.0f);
    s_id[tid] = id;
  }
}

// d_i(p) with explicit rounding (the oracle repeats it): t_z + g_u (px - mu_x) + g_v (py - mu_y)
__device__ __forceinline__ float plane_depth(float4 pl, float4 geo, float px, float py) {
  return __fmaf_rn(pl.z, __fsub_rn(py, geo.y), __fmaf_rn(pl.y, __fsub_rn(px, geo.x), pl.x));
}

}  // namespace

size_t planar_ws_stride(int P, int W, int H) {
  return ((size_t)P * sizeof(float4) + 127) / 128 * 128 + ((size_t)W * H * sizeof(uint32_t) + 127) / 128 * 128;
}

// planes [F,P,3]; out_depth / out_median [F,1,H,W]
__global__ void __launch_bounds__(256, 4) planar_fwd_kernel(int W, int H, int P, const char* img_ws, size_t img_stride,
                                                            const char* bin_ws, size_t bin_stride, int64_t R_cap,
                                                            const float* __restrict__ planes, char* pl_ws,
                                                            size_t ws_stride, float* __restrict__ out_depth,
                                                            float* __restrict__ out_median) {
  __shared__ __align__(16) float4 s_geo[RB];
  __shared__ __align__(16) float4 s_con[RB];
  __shared__ __align__(16) float4 s_pl[RB];
  __shared__ __align__(16) uint32_t s_id[RB];
  __shared__ int s_maxc;

  const int f = blockIdx.z;
  SideTile t(W, H, f, img_ws, img_stride, bin_ws, bin_stride, R_cap);
  t.find_stops(&s_maxc, [] {});
  const size_t npix = (size_t)W * H;
  const float* pl = planes + (size_t)f * P * 3;
  const float px = -t.npx2.x, py = -t.npy2.x;

  float T = 1.0f, D = 0.0f, Med = 0.0f;
  uint32_t mid = 0xFFFFFFFFu;
  side_walk(
      t, s_geo, s_con,
      [&](int base, int cnt) { load_planar_batch(t.b, t.range.x + base, cnt, pl, s_geo, s_con, s_pl, s_id, t.tid); },
      [&](int, int j, float opac, float np, bool pre) {
        if (pre) {
          const float alpha = fminf(0.99f, __fmul_rn(opac, expf(-np)));
          if (!(alpha < 1.0f / 255.0f)) {
            const float d = plane_depth(s_pl[j], s_geo[j], px, py);
            D = __fmaf_rn(T, __fmul_rn(alpha, d), D);
            if (T > 0.5f) {
              Med = d;
              mid = s_id[j];
            }
            T = __fmul_rn(T, __fadd_rn(1.0f, -alpha));
          }
        }
      },
      [](int) {});
  if (t.inside) {
    out_depth[(size_t)f * npix + t.pix_id] = D;
    out_median[(size_t)f * npix + t.pix_id] = Med;
    PlanarWS::from(pl_ws + f * ws_stride, P).median_id[t.pix_id] = mid;
  }
}

// dL/dalpha_i += dL/dD (T_i d_i(p) - (D - Pref_i) / (1 - alpha_i)), walked front to back with the forward's T by
// side_bwd_walk (raster_walk.cuh), as feature_bwd_kernel is.  The four dL/dpixel rows of contract_chunk<true> are
// dL/dD, dL/dD u', dL/dD v', 0 with (u', v') = p minus the TILE's centre (the warps' sums meet in one per-tile
// accumulator, so their offsets must share an origin); at the flush sum e (p - mu) = (S_u' - Gx' S, S_v' - Gy' S),
// (Gx', Gy') = mu minus the tile's centre.
__global__ void __launch_bounds__(256, 2) planar_bwd_kernel(int W, int H, int P, char* geom_ws, size_t geom_stride,
                                                            const char* img_ws, size_t img_stride, const char* bin_ws,
                                                            size_t bin_stride, int64_t R_cap,
                                                            const float* __restrict__ planes,
                                                            const float* __restrict__ dmap,
                                                            const float* __restrict__ dL_ddmap, char* pl_ws,
                                                            size_t ws_stride) {
  constexpr int ACC_STRIDE = acc_stride<true>();
  __shared__ __align__(16) float4 s_geo[RB];
  __shared__ __align__(16) float4 s_con[RB];
  __shared__ __align__(16) float4 s_pl[RB];
  __shared__ __align__(16) uint32_t s_id[RB];
  __shared__ float s_acc[RB * ACC_STRIDE];
  __shared__ __align__(16) float s_dlp[8][4][32];
  __shared__ int s_maxc;
  extern __shared__ __align__(16) float s_stage[];  // [8 warps][CHUNK][SLOT_F]

  const int f = blockIdx.z;
  SideTile t(W, H, f, img_ws, img_stride, bin_ws, bin_stride, R_cap);
  const size_t npix = (size_t)W * H;
  float4* const grad_acc = GeomWS::from(geom_ws + f * geom_stride, P).grad_acc;
  float4* const pacc = PlanarWS::from(pl_ws + f * ws_stride, P).acc;
  const float* pl = planes + (size_t)f * P * 3;
  const unsigned gx = (W + TILE_X - 1) / TILE_X;
  const float tcx = (t.tile % gx) * TILE_X + 0.5f * (TILE_X - 1), tcy = (t.tile / gx) * TILE_Y + 0.5f * (TILE_Y - 1);
  const float px = -t.npx2.x, py = -t.npy2.x;

  float g, Dm, Pf = 0.0f;
  side_bwd_walk(
      t, W, H, &s_maxc, s_geo, s_con, s_id, s_acc, s_dlp, s_stage, grad_acc,
      [&] {
        const size_t o = (size_t)f * npix + t.pix_id;
        g = t.inside ? dL_ddmap[o] : 0.0f, Dm = t.inside ? dmap[o] : 0.0f;
        s_dlp[t.wid][0][t.lane] = g;
        s_dlp[t.wid][1][t.lane] = g * (px - tcx);
        s_dlp[t.wid][2][t.lane] = g * (py - tcy);
        s_dlp[t.wid][3][t.lane] = 0.0f;
      },
      [&](int base, int cnt) { load_planar_batch(t.b, t.range.x + base, cnt, pl, s_geo, s_con, s_pl, s_id, t.tid); },
      [&](int j, float alpha, float T, bool act) {
        const float d = plane_depth(s_pl[j], s_geo[j], px, py);
        const float r1 = __fdividef(1.0f, 1.0f - alpha);
        const float pn = __fmaf_rn(T, __fmul_rn(alpha, d), Pf);
        Pf = act ? pn : Pf;
        return g * fmaf(T, d, -(Dm - Pf) * r1);
      },
      [&](int r, uint32_t id, const float* a) {  // the plane sums, and -g sum e for dL/dmean2D
        const float4 ge = s_geo[r], p4 = s_pl[r];
        red_add_v4(reinterpret_cast<float*>(pacc + id), a[6], fmaf(-(ge.x - tcx), a[6], a[7]),
                   fmaf(-(ge.y - tcy), a[6], a[8]), 0.0f);
        return make_float2(p4.y * a[6], p4.z * a[6]);
      });
}

// one thread per (frame, pixel): dL/dmedian of each pixel into its median record's plane accumulator
// (g, g dx, g dy) and dL/dmean2D (-g_plane g, as the flush scales it)
__global__ void __launch_bounds__(256) planar_median_grad_kernel(int F, int W, int H, int P, char* geom_ws,
                                                                 size_t geom_stride, const float* __restrict__ planes,
                                                                 const float* __restrict__ dL_dmedian, char* pl_ws,
                                                                 size_t ws_stride) {
  const size_t npix = (size_t)W * H;
  const size_t e = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (e >= (size_t)F * npix) return;
  const int f = (int)(e / npix);
  const uint32_t pix = (uint32_t)(e - (size_t)f * npix);
  const PlanarWS pw = PlanarWS::from(pl_ws + f * ws_stride, P);
  const uint32_t id = pw.median_id[pix];
  const float g = dL_dmedian[e];
  if (id == 0xFFFFFFFFu || g == 0.0f) return;
  const GeomWS gw = GeomWS::from(geom_ws + f * geom_stride, P);
  const float2 mu = gw.means2D[id];
  const float* p = planes + 3 * ((size_t)f * P + id);
  const float dx = (float)(pix % W) - mu.x, dy = (float)(pix / W) - mu.y;
  float* acc = reinterpret_cast<float*>(pw.acc + id);
  atomicAdd(acc, g);
  atomicAdd(acc + 1, g * dx);
  atomicAdd(acc + 2, g * dy);
  float* ga = reinterpret_cast<float*>(gw.grad_acc + 3 * (size_t)id);
  atomicAdd(ga, -0.5f * W * p[1] * g);
  atomicAdd(ga + 1, -0.5f * H * p[2] * g);
}

// dL/dplanes [F,P,3] from the accumulators (NULL: only re-zeroes them)
__global__ void __launch_bounds__(256) planar_grad_finish_kernel(int F, int P, char* pl_ws, size_t ws_stride,
                                                                 float* __restrict__ out) {
  const size_t e = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (e >= (size_t)F * P) return;
  const int f = (int)(e / P);
  const size_t i = e - (size_t)f * P;
  float4* acc = PlanarWS::from(pl_ws + f * ws_stride, P).acc + i;
  const float4 v = *acc;
  *acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (out) out[3 * e] = v.x, out[3 * e + 1] = v.y, out[3 * e + 2] = v.z;
}

cudaError_t launch_planar_fwd(const PlanarArgs& a, cudaStream_t s) {
  if (a.P == 0) return cudaSuccess;
  const unsigned gx = (a.W + TILE_X - 1) / TILE_X, gy = (a.H + TILE_Y - 1) / TILE_Y;
  const size_t stride = planar_ws_stride(a.P, a.W, a.H);
  // the backward adds into the accumulators: they start at zero (each frame's, stride bytes apart)
  cudaError_t e = cudaMemset2DAsync(a.planar_ws, stride, 0, (size_t)a.P * sizeof(float4), a.F, s);
  if (e != cudaSuccess) return e;
  planar_fwd_kernel<<<dim3(gx * gy, 1, a.F), 256, 0, s>>>(a.W, a.H, a.P, (const char*)a.img_ws, a.img_stride,
                                                          (const char*)a.binning_ws, a.binning_stride, a.R_cap,
                                                          a.planes, (char*)a.planar_ws, stride, a.out_depth,
                                                          a.out_median);
  return cudaGetLastError();
}

cudaError_t launch_planar_bwd(const PlanarArgs& a, cudaStream_t s) {
  side_bwd_attributes<planar_bwd_kernel>();
  if (a.P == 0) return cudaSuccess;
  const unsigned gx = (a.W + TILE_X - 1) / TILE_X, gy = (a.H + TILE_Y - 1) / TILE_Y;
  const size_t stride = planar_ws_stride(a.P, a.W, a.H);
  cudaError_t e;
  if (a.dL_ddepth) {
    planar_bwd_kernel<<<dim3(gx * gy, 1, a.F), 256, STAGE_BYTES, s>>>(
        a.W, a.H, a.P, (char*)a.geom_ws, a.geom_stride, (const char*)a.img_ws, a.img_stride,
        (const char*)a.binning_ws, a.binning_stride, a.R_cap, a.planes, a.depth, a.dL_ddepth, (char*)a.planar_ws,
        stride);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
  }
  if (a.dL_dmedian) {
    const size_t n = (size_t)a.F * a.W * a.H;
    planar_median_grad_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(
        a.F, a.W, a.H, a.P, (char*)a.geom_ws, a.geom_stride, a.planes, a.dL_dmedian, (char*)a.planar_ws, stride);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
  }
  const size_t n = (size_t)a.F * a.P;
  planar_grad_finish_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a.F, a.P, (char*)a.planar_ws, stride,
                                                                        a.dL_dplanes);
  return cudaGetLastError();
}

}  // namespace dgm
