// raster_stats.cu -- per-Gaussian blend-weight statistics (DESIGN.md §4, "Blend-weight statistics"), sm_90a.  A
// pass over the workspaces an existing forward left behind (sorted blend records, tile ranges, tile order,
// n_contrib); no existing kernel or workspace layout changes.
//
//   blend_stats_kernel  sum_i = sum_p e_p alpha_ip T_ip and max_i = max(0, max_p e_p alpha_ip T_ip) over the colour
//                       image's own blend, e_p an optional per-pixel weight (1 when absent)
//
// One CTA per (tile, frame): grid (T, F).  The walk is the side passes' side_walk (raster_walk.cuh), so T is the
// forward's bit for bit.
#include "../../include/dgmesh_b200.h"
#include "common.cuh"
#include "raster_kernels.h"
#include "raster_walk.cuh"

namespace dgm {

// Each blended (pixel, record) pair gives v = e_p alpha T.  Per record the warp forms the total of v over its 32
// pixels (a fixed butterfly) and the maximum (__reduce_max_sync on the bits: v is clamped to >= 0 first, and the
// order of non-negative floats is that of their bits) into its own slots s_sum / s_max [warp][record].  After the
// batch, thread r combines slot r of the 8 warps in warp order, so a tile's totals do not depend on scheduling,
// and issues at most one red.add into out_sum and one atomicMax into out_max (as uint bits) per record, none for
// a zero total.  The outputs must be zero beforehand.  weights: NULL, [H,W] (w_stride 0) or frame f's map at
// weights + f w_stride.
__global__ void __launch_bounds__(256, 4) blend_stats_kernel(int W, int H, int P, const char* img_ws,
                                                             size_t img_stride, const char* bin_ws, size_t bin_stride,
                                                             int64_t R_cap, const float* __restrict__ weights,
                                                             size_t w_stride, float* __restrict__ out_sum,
                                                             unsigned* __restrict__ out_max) {
  __shared__ __align__(16) float4 s_geo[RB];
  __shared__ __align__(16) float4 s_con[RB];
  __shared__ uint32_t s_id[RB];
  __shared__ float s_sum[8][RB];
  __shared__ unsigned s_max[8][RB];
  __shared__ int s_maxc;

  const int f = blockIdx.y;
  SideTile t(W, H, f, img_ws, img_stride, bin_ws, bin_stride, R_cap);
  const float e = (weights && t.inside) ? weights[f * w_stride + t.pix_id] : 1.0f;
  t.find_stops(&s_maxc, [&] {
    for (int i = t.tid; i < 8 * RB; i += 256) {  // the flush re-zeroes the slots it reads
      (&s_sum[0][0])[i] = 0.0f;
      (&s_max[0][0])[i] = 0u;
    }
  });
  float* const my_sum = s_sum[t.wid];
  unsigned* const my_max = s_max[t.wid];

  float T = 1.0f;
  side_walk(
      t, s_geo, s_con,
      [&](int base, int cnt) {
        if ((int)t.tid < cnt) {
          const size_t r = (size_t)t.range.x + base + t.tid;
          s_geo[t.tid] = t.b.inst_geo[r];
          s_con[t.tid] = t.b.inst_attr[2 * r];
          s_id[t.tid] = __float_as_uint(t.b.inst_attr[2 * r + 1].w);
        }
      },
      [&](int, int j, float opac, float np, bool pre) {
        float v = 0.0f;
        if (pre) {
          const float alpha = fminf(0.99f, __fmul_rn(opac, expf(-np)));
          if (!(alpha < 1.0f / 255.0f)) {
            v = __fmul_rn(e, __fmul_rn(alpha, T));
            T = __fmul_rn(T, __fadd_rn(1.0f, -alpha));
          }
        }
        const unsigned vb = v > 0.0f ? __float_as_uint(v) : 0u;
        // (uniform per warp) a record no pixel of the warp blends leaves its slots at zero
        if (__ballot_sync(0xffffffffu, v != 0.0f) != 0u) {
          float s = v;
#pragma unroll
          for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
          const unsigned m = __reduce_max_sync(0xffffffffu, vb);
          if (t.lane == 0) my_sum[j] = s, my_max[j] = m;
        }
      },
      [&](int cnt) {
        __syncthreads();
        // ---- flush this batch: one total per record, the 8 warps in warp order
        if ((int)t.tid < cnt) {
          float s = 0.0f;
          unsigned m = 0u;
#pragma unroll
          for (int w = 0; w < 8; ++w) {
            s += s_sum[w][t.tid];
            m = max(m, s_max[w][t.tid]);
            s_sum[w][t.tid] = 0.0f;
            s_max[w][t.tid] = 0u;
          }
          const size_t id = (size_t)f * P + s_id[t.tid];
          if (s != 0.0f) atomicAdd(out_sum + id, s);
          if (m != 0u) atomicMax(out_max + id, m);
        }
      });
}

cudaError_t launch_blend_stats(const StatsArgs& a, cudaStream_t s) {
  const size_t bytes = sizeof(float) * (size_t)a.F * a.P;
  cudaMemsetAsync(a.out_sum, 0, bytes, s);
  cudaMemsetAsync(a.out_max, 0, bytes, s);
  if (a.P == 0) return cudaGetLastError();
  const unsigned gx = (a.W + TILE_X - 1) / TILE_X, gy = (a.H + TILE_Y - 1) / TILE_Y;
  g_prof.begin(13, s);
  blend_stats_kernel<<<dim3(gx * gy, a.F), 256, 0, s>>>(
      a.W, a.H, a.P, (const char*)a.img_ws, a.img_stride, (const char*)a.binning_ws, a.binning_stride, a.R_cap,
      a.pixel_weights, a.weights_per_frame ? (size_t)a.W * a.H : 0, a.out_sum, reinterpret_cast<unsigned*>(a.out_max));
  g_prof.end(13, s);
  return cudaGetLastError();
}

}  // namespace dgm
