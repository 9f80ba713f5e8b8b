// raster_fwd.cu -- forward pass of the tile-based 3D-Gaussian rasterizer for sm_90a.
//
// Pipeline (one stream, no host synchronisation):
//   memset(tile counters) -> preprocess_kernel -> tile_scan_kernel -> scatter_kernel
//   -> tile_sort_pack_kernel -> render_fwd_kernel (<true>: + the depth and alpha maps; <true, true>: + the normal map;
//      <true, *, true>: + the median-depth and distortion maps)
//
// Results are those of the reference forward (dgr/cuda_rasterizer/forward.cu:155-374,
// rasterizer_impl.cu:198-336): identical radii / tiles_touched / per-tile sorted
// lists / n_contrib, image within fp32 rounding.  The design differs:
//   * no global 64-bit radix sort and no prefix sum over Gaussians: instances are
//     counted per tile, each tile segment is sorted on its own in shared memory by
//     (depth bits, gaussian id) which is exactly the order the reference's stable
//     sort on (tile | depth) yields (emission order == gaussian id);
//   * the sorted segment is materialised as packed records that the blend kernels
//     stream with 1-D TMA bulk copies (cp.async.bulk + mbarrier) instead of gathering
//     per-Gaussian attributes from three arrays in both passes;
//   * each warp owns an 8x4 pixel block and first culls the batch against a
//     conservative alpha >= 1/255 extent, so only Gaussians that can contribute to
//     the block enter the blend loop (the skipped ones are exactly those the
//     reference `continue`s over, so results are unchanged).
#include <stdio.h>
#include "common.cuh"
#include "raster_math.cuh"
#include "raster_kernels.h"

namespace dgm {

// =========================================================== preprocess ====
// One thread per Gaussian (forward.cu:155-256).  Besides the reference outputs it
// clears the backward accumulators and tracks the depth range of the visible set.
//
// Binning = one MSD counting pass on (tile, depth bucket) + tiny sorts (DESIGN.md):
//   count_kernel    hist[tile][bucket] += 1 per (Gaussian, tile) instance, bucket = linear
//                   quantisation of the view depth into DEPTH_BUCKETS slots.  ~T*256 counters
//                   -> no hot addresses (returning atomics on T counters serialise at ~64
//                   cycles/op on the busiest tiles, ncu r1a)
//   tile_scan_kernel  exclusive offsets of every (tile, bucket) block + tile ranges
//   scatter_kernel  keys into their block (cursor = the offset table itself)
//   tile_sort_pack_kernel  sorts every block on its own (a handful of keys in spread-out scenes, thousands in
//                   dense ones: insertion / register / warp / CTA regimes per block) and packs the blend records
#define DEPTH_BUCKETS 256

struct PreOut {
  uint2 rmin, rmax;
  uint32_t ntiles;
};

__device__ __forceinline__ bool preprocess_one(
    int idx, int D, int M, const float* __restrict__ means3D, const float* __restrict__ scales, float scale_modifier,
    const float* __restrict__ rotations, const float* __restrict__ opacities, const float* __restrict__ shs,
    const float* __restrict__ cov3D_precomp, const float* __restrict__ colors_precomp, const float* viewmatrix,
    const float* projmatrix, const float* cam_pos, int W, int H, float tan_fovx, float tan_fovy, float focal_x,
    float focal_y, int* __restrict__ radii_out, const GeomWS& g, unsigned gx, unsigned gy, int prefiltered,
    PreOut& o) {
  g.radii[idx] = 0;
  if (radii_out) radii_out[idx] = 0;
  g.tiles_touched[idx] = 0;
  g.grad_acc[3 * idx + 0] = make_float4(0, 0, 0, 0);
  g.grad_acc[3 * idx + 1] = make_float4(0, 0, 0, 0);
  g.grad_acc[3 * idx + 2] = make_float4(0, 0, 0, 0);
  const float3 p_orig = make_float3(means3D[3 * idx], means3D[3 * idx + 1], means3D[3 * idx + 2]);
  // near culling (auxiliary.h:139-164)
  const float4 p_hom = xform4x4(p_orig, projmatrix);
  const float p_w = 1.0f / (p_hom.w + 0.0000001f);
  const float3 p_proj = make_float3(p_hom.x * p_w, p_hom.y * p_w, p_hom.z * p_w);
  const float3 p_view = xform4x3(p_orig, viewmatrix);
  if (p_view.z <= 0.2f) {
    if (prefiltered) {
      printf("Point is filtered although prefiltered is set. This shouldn't happen!");
      __trap();
    }
    return false;
  }
  const float* cov3D;
  if (cov3D_precomp != nullptr) {
    cov3D = cov3D_precomp + idx * 6;
  } else {
    const float3 sc = make_float3(scales[3 * idx], scales[3 * idx + 1], scales[3 * idx + 2]);
    const float4 q = __ldg(reinterpret_cast<const float4*>(rotations) + idx);
    cov3d_from_scale_rot(sc, scale_modifier, q, g.cov3D + idx * 6);
    cov3D = g.cov3D + idx * 6;
  }
  EwaFrame fr;
  ewa_frame(p_orig, focal_x, focal_y, tan_fovx, tan_fovy, cov3D, viewmatrix, fr);
  const float3 cov = ewa_cov2d(fr);
  // invert (EWA), forward.cu:217-221
  const float det = (cov.x * cov.z - cov.y * cov.y);
  if (det == 0.0f) return false;
  const float det_inv = 1.f / det;
  const float3 conic = make_float3(cov.z * det_inv, -cov.y * det_inv, cov.x * det_inv);
  // screen-space extent from the larger eigenvalue, forward.cu:227-235
  const float mid = 0.5f * (cov.x + cov.z);
  const float lambda1 = mid + sqrtf(max(0.1f, mid * mid - det));
  const float lambda2 = mid - sqrtf(max(0.1f, mid * mid - det));
  const float my_radius = ceilf(3.f * sqrtf(max(lambda1, lambda2)));
  const float2 point_image = make_float2(ndc_to_pix(p_proj.x, W), ndc_to_pix(p_proj.y, H));
  tile_rect(point_image, my_radius, o.rmin, o.rmax, gx, gy);
  if ((o.rmax.x - o.rmin.x) * (o.rmax.y - o.rmin.y) == 0) return false;
  if (colors_precomp == nullptr) {
    bool cl[3];
    float sh[48];
    load_sh(shs, idx, M, (D + 1) * (D + 1), sh);
    const float3 cp = make_float3(cam_pos[0], cam_pos[1], cam_pos[2]);
    const float3 c = sh_to_rgb(D, p_orig, cp, sh, cl);
    g.clamped[3 * idx + 0] = cl[0];
    g.clamped[3 * idx + 1] = cl[1];
    g.clamped[3 * idx + 2] = cl[2];
    g.rgb[3 * idx + 0] = c.x;
    g.rgb[3 * idx + 1] = c.y;
    g.rgb[3 * idx + 2] = c.z;
  }
  g.depths[idx] = p_view.z;
  g.radii[idx] = my_radius;
  if (radii_out) radii_out[idx] = my_radius;
  g.means2D[idx] = point_image;
  g.conic_opacity[idx] = make_float4(conic.x, conic.y, conic.z, opacities[idx]);
  o.ntiles = (o.rmax.y - o.rmin.y) * (o.rmax.x - o.rmin.x);
  g.tiles_touched[idx] = o.ntiles;
  return true;
}

// call f(tile, payload) once per tile of each lane's rectangle; rectangles larger than 32
// tiles are spread over the whole warp (payload of the owning lane is broadcast)
template <typename F>
__device__ __forceinline__ void for_each_tile_warp(const uint2 rmin, const uint2 rmax, uint32_t ntiles, unsigned gx,
                                                   unsigned lane, unsigned long long payload, F&& f) {
  const bool big = ntiles > 32;
  if (ntiles && !big) {
    for (unsigned y = rmin.y; y < rmax.y; ++y)
      for (unsigned x = rmin.x; x < rmax.x; ++x) f(y * gx + x, payload);
  }
  unsigned bigmask = __ballot_sync(0xffffffffu, big);
  while (bigmask) {
    const int src = __ffs(bigmask) - 1;
    bigmask &= bigmask - 1;
    const unsigned x0 = __shfl_sync(0xffffffffu, rmin.x, src), y0 = __shfl_sync(0xffffffffu, rmin.y, src);
    const unsigned x1 = __shfl_sync(0xffffffffu, rmax.x, src), y1 = __shfl_sync(0xffffffffu, rmax.y, src);
    const unsigned long long pl = __shfl_sync(0xffffffffu, payload, src);
    const unsigned w = x1 - x0, n = w * (y1 - y0);
    for (unsigned k = lane; k < n; k += 32) f((y0 + k / w) * gx + (x0 + k % w), pl);
  }
}

// depth -> bucket; monotone non-decreasing in the depth (same code in count and scatter).  The
// range is either this frame's own (read from depth_range after preprocess) or a HINT passed by the
// caller (the range of an earlier frame): any monotone map gives the same final order, the range
// only decides how evenly the buckets fill, so a stale hint costs balance, never correctness.
struct DepthBuckets {
  float dmin, scale;
  __device__ __forceinline__ DepthBuckets(float lo, float hi) { set(lo, hi); }
  __device__ __forceinline__ DepthBuckets(const uint32_t* depth_range, int use_hint, float lo, float hi) {
    if (use_hint) set(lo, hi);
    else set(__uint_as_float(~depth_range[0]), __uint_as_float(depth_range[1]));
  }
  __device__ __forceinline__ void set(float lo, float hi) {
    dmin = lo;
    scale = (hi > lo) ? (float)DEPTH_BUCKETS / (hi - lo) : 0.0f;
  }
  __device__ __forceinline__ unsigned of(float depth) const {
    const float x = (depth - dmin) * scale;
    return min((unsigned)(DEPTH_BUCKETS - 1), (unsigned)max(x, 0.0f));
  }
};

// COUNT: the (tile, depth bucket) histogram of count_kernel is built here as well (needs the
// bucket range before the kernel starts, i.e. a hint)
template <bool COUNT>
__global__ void __launch_bounds__(256) preprocess_kernel(
    int P, int D, int M, const float* __restrict__ means3D, const float* __restrict__ scales, float scale_modifier,
    const float* __restrict__ rotations, const float* __restrict__ opacities, const float* __restrict__ shs,
    const float* __restrict__ cov3D_precomp, const float* __restrict__ colors_precomp,
    const float* __restrict__ viewmatrix, const float* __restrict__ projmatrix, const float* __restrict__ cam_pos,
    int W, int H, float tan_fovx, float tan_fovy, float focal_x, float focal_y, int* __restrict__ radii_out,
    GeomWS g, unsigned gx, unsigned gy, uint32_t* __restrict__ depth_range, uint32_t* __restrict__ scan_flags,
    int32_t* __restrict__ status, int prefiltered, uint32_t* __restrict__ hist, float hint_lo, float hint_hi) {
  __shared__ float s_cam[36];
  const unsigned tid = threadIdx.x;
  pdl_wait();
  pdl_launch();
  if (blockIdx.x == 0 && tid < 8) {  // state consumed by tile_scan_kernel, which runs after this grid
    scan_flags[tid] = 0;
    status[tid] = 0;
  }
  if (tid < 16) s_cam[tid] = viewmatrix[tid];
  else if (tid < 32) s_cam[tid] = projmatrix[tid - 16];
  else if (tid < 35) s_cam[tid] = cam_pos[tid - 32];
  __syncthreads();
  const int idx = blockIdx.x * 256 + tid;
  PreOut o;
  o.rmin = o.rmax = make_uint2(0, 0);
  o.ntiles = 0;
  bool ok = false;
  if (idx < P)
    ok = preprocess_one(idx, D, M, means3D, scales, scale_modifier, rotations, opacities, shs, cov3D_precomp,
                        colors_precomp, s_cam, s_cam + 16, s_cam + 32, W, H, tan_fovx, tan_fovy, focal_x, focal_y,
                        radii_out, g, gx, gy, prefiltered, o);
  // depth range of the visible Gaussians (positive floats order like their bit patterns);
  // depth_range = { max of ~bits (i.e. the minimum), max of bits }, both zero-initialised
  uint32_t dmax = ok ? __float_as_uint(g.depths[idx]) : 0u;
  uint32_t dmin_inv = ok ? ~dmax : 0u;
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    dmax = max(dmax, __shfl_xor_sync(0xffffffffu, dmax, off));
    dmin_inv = max(dmin_inv, __shfl_xor_sync(0xffffffffu, dmin_inv, off));
  }
  if ((tid & 31) == 0 && dmax) {
    atomicMax(&depth_range[0], dmin_inv);
    atomicMax(&depth_range[1], dmax);
  }
  if (COUNT) {
    const DepthBuckets db(hint_lo, hint_hi);
    const unsigned long long bucket = ok ? db.of(g.depths[idx]) : 0u;
    for_each_tile_warp(o.rmin, o.rmax, ok ? o.ntiles : 0u, gx, tid & 31, bucket, [&](unsigned t, unsigned long long b) {
      atomicAdd(&hist[(size_t)t * DEPTH_BUCKETS + (unsigned)b], 1u);
    });
  }
}

// ================================================================ count ====
__global__ void __launch_bounds__(256) count_kernel(int P, GeomWS g, uint32_t* __restrict__ hist,
                                                    const uint32_t* __restrict__ depth_range, unsigned gx,
                                                    unsigned gy) {
  pdl_wait();
  pdl_launch();
  const int idx = blockIdx.x * 256 + threadIdx.x;
  const unsigned lane = threadIdx.x & 31;
  const DepthBuckets db(depth_range, 0, 0.f, 0.f);
  uint2 rmin = make_uint2(0, 0), rmax = make_uint2(0, 0);
  uint32_t ntiles = 0;
  unsigned long long bucket = 0;
  if (idx < P) {
    const int r = g.radii[idx];
    if (r > 0) {
      tile_rect(g.means2D[idx], r, rmin, rmax, gx, gy);
      ntiles = (rmax.y - rmin.y) * (rmax.x - rmin.x);
      bucket = db.of(g.depths[idx]);
    }
  }
  for_each_tile_warp(rmin, rmax, ntiles, gx, lane, bucket, [&](unsigned t, unsigned long long b) {
    atomicAdd(&hist[(size_t)t * DEPTH_BUCKETS + (unsigned)b], 1u);
  });
}

// ============================================================ tile scan ====
// hist[T, B] ((tile, depth bucket) counts) -> in place: exclusive prefix over the buckets of
// each tile; then the last CTA to finish scans the T tile totals into ranges[t] =
// [start, end) (what identifyTileRanges, rasterizer_impl.cu:116-138, derives from the
// sorted keys), writes R / overflow into `status`, and orders the tiles by decreasing
// list length (coarse, by power-of-two bucket) so the blend kernels start their longest
// tiles first.  CTA = 32 tiles x 8 bucket groups.
__global__ void __launch_bounds__(256) tile_scan_kernel(int T, uint32_t* __restrict__ hist,
                                                        uint32_t* __restrict__ tile_total, uint2* __restrict__ ranges,
                                                        uint32_t* __restrict__ tile_order,
                                                        uint32_t* __restrict__ flags, int32_t* __restrict__ status,
                                                        long long R_cap, const uint32_t* __restrict__ depth_range,
                                                        volatile int32_t* __restrict__ status_host) {
  __shared__ uint32_t s_part[8][33];
  __shared__ uint32_t s_warp[32];
  __shared__ uint32_t s_bucket[33];
  __shared__ uint32_t s_carry, s_last;
  const int tid = threadIdx.x;
  pdl_wait();
  pdl_launch();
  {
    const int tx = tid & 31, seg = tid >> 5;
    const int t = blockIdx.x * 32 + tx;
    // this thread owns DEPTH_BUCKETS/8 = 32 consecutive buckets (128 B) of tile t
    uint4* row = reinterpret_cast<uint4*>(hist + (size_t)(t < T ? t : 0) * DEPTH_BUCKETS + seg * (DEPTH_BUCKETS / 8));
    uint4 v[8];
    uint32_t sum = 0;
    if (t < T) {
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        v[c] = row[c];
        sum += v[c].x + v[c].y + v[c].z + v[c].w;
      }
    }
    s_part[seg][tx] = sum;
    __syncthreads();
    uint32_t run = 0;
    for (int k = 0; k < seg; ++k) run += s_part[k][tx];
    if (t < T) {
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        uint4 o;
        o.x = run;
        run += v[c].x;
        o.y = run;
        run += v[c].y;
        o.z = run;
        run += v[c].z;
        o.w = run;
        run += v[c].w;
        row[c] = o;
      }
      if (seg == 7) tile_total[t] = run;  // the last segment ends with the tile total
    }
  }
  // ---- last CTA done: scan of the column totals
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = (atomicAdd(&flags[0], 1u) == gridDim.x - 1) ? 1u : 0u;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const int lane = tid & 31, wid = tid >> 5;
  if (tid == 0) s_carry = 0;
  if (tid < 33) s_bucket[tid] = 0;
  __syncthreads();
  uint32_t local_max = 0;
  for (int base = 0; base < T; base += 256) {
    const int t = base + tid;
    const uint32_t c = (t < T) ? __ldcg(tile_total + t) : 0u;
    local_max = max(local_max, c);
    if (t < T) atomicAdd(&s_bucket[c ? 32 - __clz(c) : 0], 1u);  // bucket b holds 2^(b-1) <= c < 2^b
    uint32_t v = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t n = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += n;
    }
    if (lane == 31) s_warp[wid] = v;
    __syncthreads();
    if (wid == 0) {
      uint32_t w = lane < 8 ? s_warp[lane] : 0;
#pragma unroll
      for (int o = 1; o < 8; o <<= 1) {
        const uint32_t n = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += n;
      }
      if (lane < 8) s_warp[lane] = w;
    }
    __syncthreads();
    const uint32_t incl = s_carry + (wid ? s_warp[wid - 1] : 0u) + v;
    if (t < T) ranges[t] = c ? make_uint2(incl - c, incl) : make_uint2(0u, 0u);
    __syncthreads();
    if (tid == 255) s_carry = incl;
    __syncthreads();
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) local_max = max(local_max, __shfl_xor_sync(0xffffffffu, local_max, o));
  if (lane == 0) atomicMax(reinterpret_cast<unsigned*>(status + 2), local_max);
  // tile order: longest bucket first
  if (tid == 0) {
    uint32_t acc = 0;
    for (int b = 32; b >= 0; --b) {
      const uint32_t n = s_bucket[b];
      s_bucket[b] = acc;
      acc += n;
    }
    status[0] = (int32_t)s_carry;
    status[1] = ((long long)s_carry > R_cap) ? 1 : 0;
    // this frame's depth range (float bits; 0 / 0 when nothing is visible): the next call's hint
    status[3] = depth_range[1] ? (int32_t)~depth_range[0] : 0;
    status[4] = (int32_t)depth_range[1];
  }
  __syncthreads();
  if (tid == 0 && status_host) {
    // the caller's host-mapped copy (it waits for an event recorded behind this kernel)
    status_host[0] = (int32_t)s_carry;
    status_host[1] = ((long long)s_carry > R_cap) ? 1 : 0;
    status_host[2] = *reinterpret_cast<volatile int32_t*>(status + 2);
    status_host[3] = status[3];
    status_host[4] = status[4];
    __threadfence_system();
  }
  for (int t = tid; t < T; t += 256) {
    const uint32_t c = __ldcg(tile_total + t);
    const uint32_t pos = atomicAdd(&s_bucket[c ? 32 - __clz(c) : 0], 1u);
    tile_order[pos] = (uint32_t)t;
  }
}

// ============================================================== scatter ====
// Emit one (depth bits << 32 | gaussian id) key per (Gaussian, tile) instance into its
// (tile, bucket) block (role of duplicateWithKeys, rasterizer_impl.cu:70-111; the tile id
// is implied by the segment, so the 64-bit word carries the gaussian id instead).  The
// offset table doubles as the cursor: afterwards hist[t][b] is the END of block b.
__global__ void __launch_bounds__(256) scatter_kernel(int P, GeomWS g, const uint2* __restrict__ ranges,
                                                      uint32_t* __restrict__ hist,
                                                      const uint32_t* __restrict__ depth_range,
                                                      unsigned long long* __restrict__ keys, unsigned gx, unsigned gy,
                                                      const int32_t* __restrict__ status, int use_hint,
                                                      float hint_lo, float hint_hi) {
  pdl_wait();
  pdl_launch();
  if (status[1]) return;  // overflow: nothing may be written
  const int idx = blockIdx.x * 256 + threadIdx.x;
  const unsigned lane = threadIdx.x & 31;
  const DepthBuckets db(depth_range, use_hint, hint_lo, hint_hi);
  uint2 rmin = make_uint2(0, 0), rmax = make_uint2(0, 0);
  unsigned long long key = 0;
  uint32_t ntiles = 0;
  if (idx < P) {
    const int r = g.radii[idx];
    if (r > 0) {
      tile_rect(g.means2D[idx], r, rmin, rmax, gx, gy);
      ntiles = (rmax.y - rmin.y) * (rmax.x - rmin.x);
      key = ((unsigned long long)__float_as_uint(g.depths[idx]) << 32) | (unsigned)idx;
    }
  }
  for_each_tile_warp(rmin, rmax, ntiles, gx, lane, key, [&](unsigned t, unsigned long long k64) {
    const unsigned b = db.of(__uint_as_float((unsigned)(k64 >> 32)));
    const uint32_t pos = ranges[t].x + atomicAdd(&hist[(size_t)t * DEPTH_BUCKETS + b], 1u);
    keys[pos] = k64;
  });
}

// ======================================================= tile sort+pack ====
// One CTA per tile (longest lists first): the segment is already partitioned into DEPTH_BUCKETS depth-ordered
// blocks (scatter left each block's END in hist); sort every block by (depth bits, gaussian id) -- which is
// exactly the order the reference's stable sort on (tile | depth) yields -- then write point_list and the packed
// blend records.  Block sizes vary by orders of magnitude between scenes: a spread-out scene (C2) has ~1 key per
// block, an object that fills a seventh of the image (what DG-Mesh trains on) has thousands of keys per tile in
// a few dozen blocks.
//   * A tile is processed in RUNS of consecutive blocks that fit the 24 KB key stage (eight CTAs per SM whatever
//     the scene): load the run, sort its blocks, pack its records, next run.  A tile of any length is handled at
//     full occupancy; only a single block longer than the stage is sorted in place in global memory.
//   * Four sort regimes, chosen per BLOCK:
//       <= 8 keys      insertion sort by the block's own thread
//       <= 32 keys     one warp, keys in registers, bitonic network over shuffles
//       <= 2048 keys   one warp, bitonic network in shared memory (normalised: all comparators ascending, so
//                      virtual +inf padding never moves and any length works)
//       larger         the whole CTA
//     Thread (warp w, lane l) owns block 8 l + w, so depth-adjacent (similarly full) blocks land in different
//     warps; a warp finds the blocks it has to sort cooperatively with one ballot over its own lanes.
#define SORT_STAGE_KEYS 3072  // 24 KB
#define INSERT_SORT_MAX 8     // longest block one thread sorts by insertion
#define WARP_SORT_MAX 2048    // longest block one warp sorts

__device__ __forceinline__ void cmpswap(unsigned long long* a, uint32_t lo, uint32_t hi, uint32_t n) {
  if (hi < n) {
    const unsigned long long x = a[lo], y = a[hi];
    if (x > y) {
      a[lo] = y;
      a[hi] = x;
    }
  }
}

// normalised bitonic sort of a[0..n) by `nthreads` cooperating threads (WARP: one warp, __syncwarp between
// steps; otherwise the whole CTA, __syncthreads)
template <bool WARP>
__device__ __forceinline__ void bitonic_sort_any(unsigned long long* a, uint32_t n, uint32_t tid, uint32_t nthreads) {
  if (n < 2) return;
  const uint32_t lm = 32 - __clz(n - 1);  // m = 1 << lm = next power of two >= n
  const uint32_t half = 1u << (lm - 1);
  for (uint32_t lk = 1; lk <= lm; ++lk) {  // merge size k = 1 << lk
    const uint32_t hk = 1u << (lk - 1);
    // mirror step: i -> (block base + off, block base + k - 1 - off)
    for (uint32_t i = tid; i < half; i += nthreads) {
      const uint32_t off = i & (hk - 1), base = (i >> (lk - 1)) << lk;
      cmpswap(a, base + off, base + (hk << 1) - 1 - off, n);
    }
    if (WARP) __syncwarp(); else __syncthreads();
    for (uint32_t j = hk >> 1; j >= 1; j >>= 1) {
      for (uint32_t i = tid; i < half; i += nthreads) {
        const uint32_t lo = ((i & ~(j - 1)) << 1) | (i & (j - 1));
        cmpswap(a, lo, lo + j, n);
      }
      if (WARP) __syncwarp(); else __syncthreads();
    }
  }
}

// a[0..n), n <= 32: one key per lane, bitonic network over shuffles (padding = all ones sorts last)
__device__ __forceinline__ void warp_sort32(unsigned long long* a, uint32_t n, uint32_t lane) {
  unsigned long long x = lane < n ? a[lane] : ~0ull;
#pragma unroll
  for (uint32_t k = 2; k <= 32; k <<= 1) {
#pragma unroll
    for (uint32_t j = k >> 1; j > 0; j >>= 1) {
      const unsigned long long y = __shfl_xor_sync(0xffffffffu, x, j);
      const bool take_min = ((lane & j) == 0) == ((lane & k) == 0);
      x = take_min ? (x < y ? x : y) : (x < y ? y : x);
    }
  }
  if (lane < n) a[lane] = x;
}

struct PackRec {
  uint32_t id;
  float4 geo, attr0, attr1, nrm;
};
// rec_depth: the view-space depths when the forward renders depth (stored in the record's .w), else NULL;
// normals: the [P,3] normals when it renders the normal map (record of the normal stream), else NULL
__device__ __forceinline__ PackRec pack_record(unsigned long long k, const GeomWS& g, const float* __restrict__ colors,
                                               const float* __restrict__ rec_depth,
                                               const float* __restrict__ normals) {
  PackRec r;
  r.id = (uint32_t)(k & 0xffffffffull);
  const float2 xy = g.means2D[r.id];
  const float4 co = g.conic_opacity[r.id];
  const float c0 = colors[3 * r.id], c1 = colors[3 * r.id + 1], c2 = colors[3 * r.id + 2];
  // 2*(ln(255 o) + margin): the level of q = -2 power below which alpha >= 1/255 is possible
  // (see cull_keep); -1 when the opacity alone rules it out, +inf for a degenerate conic
  float q2tau;
  const float tau = __logf(255.0f * co.w) + 0.02f;
  const float det = co.x * co.z - co.y * co.y;
  if (!(tau > 0.0f)) q2tau = -1.0f;
  else if (!(det > 0.0f) || !(co.x > 0.0f) || !(co.z > 0.0f) || !isfinite(det) || !isfinite(tau)) q2tau = 3.0e38f;
  else q2tau = 2.0f * tau;
  r.geo = make_float4(xy.x, xy.y, q2tau, rec_depth ? rec_depth[r.id] : 0.0f);
  r.attr0 = co;
  r.attr1 = make_float4(c0, c1, c2, __uint_as_float(r.id));
  if (normals) r.nrm = make_float4(normals[3 * r.id], normals[3 * r.id + 1], normals[3 * r.id + 2], 0.0f);
  return r;
}
__device__ __forceinline__ void store_record(const BinWS& b, size_t o, const PackRec& r, float4* __restrict__ inst_nrm) {
  b.point_list[o] = r.id;
  b.inst_geo[o] = r.geo;
  b.inst_attr[2 * o] = r.attr0;
  b.inst_attr[2 * o + 1] = r.attr1;
  if (inst_nrm) inst_nrm[o] = r.nrm;
}
// records of sorted keys a[0..cnt) -> instance slots first + i; two keys per thread in flight
__device__ __forceinline__ void pack_run(const unsigned long long* a, uint32_t cnt, size_t first, const GeomWS& g,
                                         const float* __restrict__ colors, const float* __restrict__ rec_depth,
                                         const BinWS& b, uint32_t tid, const float* __restrict__ normals,
                                         float4* __restrict__ inst_nrm) {
  uint32_t i = tid;
  for (; i + 256 < cnt; i += 512) {
    const PackRec r0 = pack_record(a[i], g, colors, rec_depth, normals),
                  r1 = pack_record(a[i + 256], g, colors, rec_depth, normals);
    store_record(b, first + i, r0, inst_nrm);
    store_record(b, first + i + 256, r1, inst_nrm);
  }
  if (i < cnt) store_record(b, first + i, pack_record(a[i], g, colors, rec_depth, normals), inst_nrm);
}

// DEPTH: the records carry the view depth (rec_depth = the depths of the geom workspace) for the depth map;
// the colour-only instance ignores rec_depth and stores 0.
// NRM (with DEPTH): also the normal stream, inst_nrm[o] = {normals[id], 0} in the final sorted order; the other
// instances ignore normals and inst_nrm
template <bool DEPTH, bool NRM = false>
__global__ void __launch_bounds__(256) tile_sort_pack_kernel(const uint2* __restrict__ ranges,
                                                             const uint32_t* __restrict__ tile_order,
                                                             unsigned long long* __restrict__ keys,
                                                             const uint32_t* __restrict__ hist, GeomWS g,
                                                             const float* __restrict__ colors_precomp,
                                                             const float* __restrict__ rec_depth, BinWS b,
                                                             const int32_t* __restrict__ status,
                                                             const float* __restrict__ normals,
                                                             float4* __restrict__ inst_nrm) {
  __shared__ __align__(16) unsigned long long s_keys[SORT_STAGE_KEYS];
  __shared__ uint32_t s_end[DEPTH_BUCKETS + 1];  // s_end[k] = start of block k, s_end[k + 1] = its end
  pdl_wait();
  pdl_launch();
  if (status[1]) return;
  const uint32_t tile = tile_order[blockIdx.x];  // longest lists first (shorter tail in dense scenes)
  const uint2 range = ranges[tile];
  const uint32_t n = range.y - range.x;
  if (n == 0) return;
  const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const uint32_t mine = lane * 8 + wid;  // the block this thread owns
  unsigned long long* seg = keys + range.x;
  const float* colors = colors_precomp ? colors_precomp : g.rgb;
  if (!DEPTH) rec_depth = nullptr;
  if (!NRM) normals = nullptr, inst_nrm = nullptr;
  // (scatter left the block END, relative to the segment, in hist)
  s_end[mine + 1] = hist[(size_t)tile * DEPTH_BUCKETS + mine];
  if (tid == 0) s_end[0] = 0;
  __syncthreads();
  const uint32_t bstart = s_end[mine], blen = s_end[mine + 1] - bstart;

  uint32_t k0 = 0;
  while (k0 < DEPTH_BUCKETS) {
    const uint32_t start = s_end[k0];
    if (start == n) break;  // only empty blocks left
    // blocks [k0, k1) fit the stage (s_end is monotone: the predicate holds on a prefix of [k0, 256))
    const uint32_t fit = __syncthreads_count(tid >= k0 && s_end[tid + 1] - start <= SORT_STAGE_KEYS);
    if (fit == 0) {  // block k0 alone is longer than the stage: sort it where it lies (rare)
      const uint32_t len = s_end[k0 + 1] - start;
      bitonic_sort_any<false>(seg + start, len, tid, 256);
      pack_run(seg + start, len, (size_t)range.x + start, g, colors, rec_depth, b, tid, normals, inst_nrm);
      k0 += 1;
      continue;
    }
    const uint32_t k1 = k0 + fit, cnt = s_end[k1] - start;
    for (uint32_t i = tid; i < cnt; i += 256) s_keys[i] = seg[start + i];
    const bool in_run = mine >= k0 && mine < k1;
    const uint32_t len = in_run ? blen : 0;
    const int any_huge = __syncthreads_or(len > WARP_SORT_MAX);  // also: the stage is loaded
    unsigned long long* a = s_keys + (bstart - start);           // this thread's block (valid when in_run)
    if (len > 1 && len <= INSERT_SORT_MAX) {
      for (uint32_t i = 1; i < len; ++i) {
        const unsigned long long key = a[i];
        uint32_t j = i;
        while (j > 0 && a[j - 1] > key) {
          a[j] = a[j - 1];
          --j;
        }
        a[j] = key;
      }
    }
    // blocks of this warp's lanes that need the whole warp
    uint32_t coop = __ballot_sync(0xffffffffu, len > INSERT_SORT_MAX && len <= WARP_SORT_MAX);
    while (coop) {
      const uint32_t l = __ffs(coop) - 1;
      coop &= coop - 1;
      const uint32_t s0 = __shfl_sync(0xffffffffu, bstart, l) - start, ln = __shfl_sync(0xffffffffu, len, l);
      if (ln <= 32) warp_sort32(s_keys + s0, ln, lane);
      else bitonic_sort_any<true>(s_keys + s0, ln, lane, 32);
    }
    if (any_huge) {  // uniform loop: every thread sees the same sizes
      __syncthreads();
      for (uint32_t k = k0; k < k1; ++k) {
        const uint32_t s0 = s_end[k], ln = s_end[k + 1] - s0;
        if (ln > WARP_SORT_MAX) bitonic_sort_any<false>(s_keys + (s0 - start), ln, tid, 256);
      }
    }
    __syncthreads();
    pack_run(s_keys, cnt, (size_t)range.x + start, g, colors, rec_depth, b, tid, normals, inst_nrm);
    k0 = k1;
    if (k0 < DEPTH_BUCKETS) __syncthreads();  // the stage is overwritten by the next run
  }
}

// =============================================================== render ====
// One CTA per 16x16 tile, one thread per pixel, warp = 8x4 pixel block
// (semantics of renderCUDA, forward.cu:261-374).
#define RB 256  // records per batch (== reference BLOCK_SIZE staging granularity)

#ifdef DGM_COUNT_PAIRS
// diagnostic build only (tools/pair_stats.py): [0] (warp, Gaussian) pairs evaluated after the cull,
// [1] those in which at least one lane blended the Gaussian, [2] (warp, Gaussian) pairs before the cull
__device__ unsigned long long g_dbg_pairs[4];
#endif

// AUX: also the depth map sum_i d_i alpha_i T_i (d_i = the record's .w) and the alpha map 1 - T_final, each
// written when its pointer is non-NULL.  The colour-only instance (AUX = false) ignores both pointers.
// NRM (with AUX): also the [3,H,W] normal map sum_i n_i alpha_i T_i (out_normal, may be NULL) of the normal
// stream inst_nrm, a third record stream that arrives on the same mbarrier (its stage exists in that instance only)
// SURF (with AUX; needs the records of a depth forward): also the median depth (d of the last record blended with
// T > 0.5 before it, 0 where none) and the distortion sum_i w_i (m_i^2 A_i + M2_i - 2 m_i M1_i), w_i = alpha_i T_i,
// m_i = surf_m(d_i, d of the tile's first record), A_i / M1_i / M2_i = the sums of w_j / w_j m_j / w_j m_j^2 over
// j < i (= 1/2 sum_ij w_i w_j (m_i - m_j)^2).  Always writes the median record's id and the totals M1, M2 (surf_id,
// surf_mom) for the backward; out_median and out_dist may be NULL
template <bool AUX, bool NRM = false, bool SURF = false>
__global__ void __launch_bounds__(256, AUX ? 4 : 5) render_fwd_kernel(const uint2* __restrict__ ranges,
                                                         const uint32_t* __restrict__ tile_order,
                                                         const float4* __restrict__ inst_geo,
                                                         const float4* __restrict__ inst_attr, int W, int H,
                                                         const float* __restrict__ bg_color,
                                                         float* __restrict__ final_T, uint32_t* __restrict__ n_contrib,
                                                         float* __restrict__ out_color,
                                                         const int32_t* __restrict__ status,
                                                         float* __restrict__ out_depth, float* __restrict__ out_alpha,
                                                         const float4* __restrict__ inst_nrm,
                                                         float* __restrict__ out_normal,
                                                         uint32_t* __restrict__ surf_id, float2* __restrict__ surf_mom,
                                                         float* __restrict__ out_median, float* __restrict__ out_dist,
                                                         float surf_k) {
  __shared__ __align__(128) float4 s_geo[2][RB];
  __shared__ __align__(128) float4 s_attr[2][2 * RB];
  __shared__ __align__(8) uint64_t s_bar[2];
  __shared__ __align__(128) float4 s_nrm[NRM ? 2 * RB : 1];  // [2][RB] (NRM only)

  pdl_wait();
  pdl_launch();
  const unsigned gx = (W + TILE_X - 1) / TILE_X;
  const unsigned tile = tile_order[blockIdx.x];  // longest lists first
  const unsigned tx = tile % gx, ty = tile / gx;
  const unsigned tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  // warp -> 8x4 block inside the tile; lane -> pixel inside the block
  const int wx0 = tx * TILE_X + (wid & 1) * 8, wy0 = ty * TILE_Y + (wid >> 1) * 4;
  const int px = wx0 + (lane & 7), py = wy0 + (lane >> 3);
  const bool inside = px < W && py < H;
  const uint32_t pix_id = W * py + px;
  const float pixfx = (float)px, pixfy = (float)py;
  const float bx0 = (float)wx0, bx1 = (float)(wx0 + 7), by0 = (float)wy0, by1 = (float)(wy0 + 3);
  const float2 npx2 = make_float2(-pixfx, -pixfx), npy2 = make_float2(-pixfy, -pixfy);

  uint2 range = ranges[tile];
  if (status[1]) range = make_uint2(0, 0);
  const int total = range.y - range.x;
  const int rounds = (total + RB - 1) / RB;
  const float dref = (SURF && total > 0) ? inst_geo[range.x].w : 1.0f;  // reference depth of surf_m (SURF only)

  if (tid == 0) {
    mbar_init(&s_bar[0], 1);
    mbar_init(&s_bar[1], 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (tid == 0 && rounds > 0) {
    const uint32_t nb = min(RB, total);
    mbar_expect_tx(&s_bar[0], nb * (NRM ? 64u : 48u));
    tma_load_1d(&s_geo[0][0], inst_geo + range.x, nb * 16u, &s_bar[0]);
    tma_load_1d(&s_attr[0][0], inst_attr + 2 * (size_t)range.x, nb * 32u, &s_bar[0]);
    if (NRM) tma_load_1d(&s_nrm[0], inst_nrm + range.x, nb * 16u, &s_bar[0]);
  }

  bool done = !inside;
  float T = 1.0f;
  uint32_t last_contributor = 0;
  float C0 = 0.f, C1 = 0.f, C2 = 0.f;
  float Dp = 0.f;                    // depth (AUX only)
  float N0 = 0.f, N1 = 0.f, N2 = 0.f;  // normal (NRM only)
  float SA = 0.f, SM1 = 0.f, SM2 = 0.f, Dist = 0.f, Med = 0.f;  // running sums, distortion, median (SURF only)
  uint32_t med_id = 0xFFFFFFFFu;

  for (int i = 0; i < rounds; ++i) {
    const int st = i & 1;
    mbar_wait(&s_bar[st], (i >> 1) & 1);
    // block-wide exit vote (forward.cu:309-311); also fences reuse of the other stage
    const int num_done = __syncthreads_count(done);
    if (num_done == TILE_PIX) break;
    const int base = i * RB;
    const int nb = min(RB, total - base);
    if (tid == 0 && i + 1 < rounds) {
      const int nbase = base + RB;
      const uint32_t nn = min(RB, total - nbase);
      mbar_expect_tx(&s_bar[st ^ 1], nn * (NRM ? 64u : 48u));
      tma_load_1d(&s_geo[st ^ 1][0], inst_geo + range.x + nbase, nn * 16u, &s_bar[st ^ 1]);
      tma_load_1d(&s_attr[st ^ 1][0], inst_attr + 2 * ((size_t)range.x + nbase), nn * 32u, &s_bar[st ^ 1]);
      if (NRM) tma_load_1d(&s_nrm[(st ^ 1) * RB], inst_nrm + range.x + nbase, nn * 16u, &s_bar[st ^ 1]);
    }
    if (__all_sync(0xffffffffu, done)) continue;  // whole 8x4 block finished

    // ---- cull this batch against the warp's pixel block
    unsigned keep[RB / 32];
#pragma unroll
    for (int k = 0; k < RB / 32; ++k) {
      const int r = k * 32 + lane;
      bool kp = false;
      if (r < nb) {
        kp = cull_keep(s_geo[st][r], s_attr[st][2 * r], bx0, bx1, by0, by1);
      }
      keep[k] = __ballot_sync(0xffffffffu, kp);
    }
#ifdef DGM_COUNT_PAIRS
    if (lane == 0) atomicAdd(&g_dbg_pairs[2], (unsigned long long)nb);
#endif
    // ---- blend the survivors front to back, two records per iteration: the quadratic
    // forms of both are evaluated side by side (pair_npow), the order-dependent
    // transmittance update stays scalar.
#pragma unroll
    for (int k = 0; k < RB / 32; ++k) {
      unsigned mask = keep[k];
      if (mask == 0) continue;
      if (__all_sync(0xffffffffu, done)) break;
      while (mask) {
        const int bA = __ffs(mask) - 1;
        mask &= mask - 1;
        const bool two = mask != 0;
        const int bB = two ? __ffs(mask) - 1 : bA;
        mask &= mask - 1;  // no-op when mask is already 0
        const int jA = k * 32 + bA, jB = k * 32 + bB;
        const float4 geA = s_geo[st][jA], geB = s_geo[st][jB];
        const float4 coA = s_attr[st][2 * jA], coB = s_attr[st][2 * jB];
        const float2 npow = pair_npow(geA, geB, coA, coB, npx2, npy2);
#ifdef DGM_COUNT_PAIRS
        const uint32_t lc_before = last_contributor;
#endif
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const float np = q ? npow.y : npow.x;
          const float opac = q ? coB.w : coA.w;
          const int j = q ? jB : jA;
#ifdef DGM_COUNT_PAIRS
          const uint32_t lc0 = last_contributor;
#endif
          if ((q == 0 || two) && !done && !(np < 0.0f)) {  // reference: if (power > 0) continue
            const float alpha = fminf(0.99f, __fmul_rn(opac, expf(-np)));
            if (!(alpha < 1.0f / 255.0f)) {
              const float test_T = __fmul_rn(T, __fadd_rn(1.0f, -alpha));
              if (test_T < 0.0001f) {
                done = true;
              } else {
                const float4 col = s_attr[st][2 * j + 1];
                C0 = __fmaf_rn(T, __fmul_rn(alpha, col.x), C0);
                C1 = __fmaf_rn(T, __fmul_rn(alpha, col.y), C1);
                C2 = __fmaf_rn(T, __fmul_rn(alpha, col.z), C2);
                if (AUX) Dp = __fmaf_rn(T, __fmul_rn(alpha, s_geo[st][j].w), Dp);
                if (NRM) {
                  const float4 n = s_nrm[st * RB + j];
                  N0 = __fmaf_rn(T, __fmul_rn(alpha, n.x), N0);
                  N1 = __fmaf_rn(T, __fmul_rn(alpha, n.y), N1);
                  N2 = __fmaf_rn(T, __fmul_rn(alpha, n.z), N2);
                }
                if (SURF) {
                  const float d = s_geo[st][j].w;
                  const float w = __fmul_rn(alpha, T), m = surf_m(d, dref, surf_k);
                  const float wm = __fmul_rn(w, m);
                  // w (m (m A - 2 M1) + M2)
                  Dist = __fmaf_rn(w, __fmaf_rn(m, __fmaf_rn(m, SA, __fmul_rn(-2.0f, SM1)), SM2), Dist);
                  SA = __fadd_rn(SA, w);
                  SM1 = __fadd_rn(SM1, wm);
                  SM2 = __fmaf_rn(wm, m, SM2);
                  if (T > 0.5f) {
                    Med = d;
                    med_id = __float_as_uint(s_attr[st][2 * j + 1].w);
                  }
                }
                T = test_T;
                last_contributor = base + j + 1;
              }
            }
          }
#ifdef DGM_COUNT_PAIRS
          if (q == 0 || two) {
            const bool any = __any_sync(0xffffffffu, last_contributor != lc0);
            if (lane == 0) {
              atomicAdd(&g_dbg_pairs[0], 1ull);
              if (any) atomicAdd(&g_dbg_pairs[1], 1ull);
            }
          }
#endif
        }
#ifdef DGM_COUNT_PAIRS
        (void)lc_before;
#endif
      }
    }
  }
  if (inside) {
    final_T[pix_id] = T;
    n_contrib[pix_id] = last_contributor;
    const size_t HW = (size_t)H * W;
    out_color[0 * HW + pix_id] = C0 + T * bg_color[0];
    out_color[1 * HW + pix_id] = C1 + T * bg_color[1];
    out_color[2 * HW + pix_id] = C2 + T * bg_color[2];
    if (AUX) {
      if (out_depth) out_depth[pix_id] = Dp;
      if (out_alpha) out_alpha[pix_id] = __fadd_rn(1.0f, -T);
    }
    if (NRM && out_normal) {
      out_normal[0 * HW + pix_id] = N0;
      out_normal[1 * HW + pix_id] = N1;
      out_normal[2 * HW + pix_id] = N2;
    }
    if (SURF) {
      surf_id[pix_id] = med_id;
      surf_mom[pix_id] = make_float2(SM1, SM2);
      if (out_median) out_median[pix_id] = Med;
      if (out_dist) out_dist[pix_id] = Dist;
    }
  }
}

#ifdef DGM_COUNT_PAIRS
}  // namespace dgm
extern "C" int dgm_debug_pair_counters(unsigned long long* out4, int reset) {
  cudaDeviceSynchronize();
  if (out4) cudaMemcpyFromSymbol(out4, dgm::g_dbg_pairs, sizeof(unsigned long long) * 4);
  if (reset) {
    unsigned long long z[4] = {0, 0, 0, 0};
    cudaMemcpyToSymbol(dgm::g_dbg_pairs, z, sizeof(z));
  }
  return 0;
}
namespace dgm {
#endif

// frustum test only (rasterizer_impl.cu:54-66)
__global__ void __launch_bounds__(256) mark_visible_kernel(int P, const float* __restrict__ means3D,
                                                           const float* __restrict__ viewmatrix,
                                                           const float* __restrict__ projmatrix,
                                                           uint8_t* __restrict__ present) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= P) return;
  const float3 p = make_float3(means3D[3 * idx], means3D[3 * idx + 1], means3D[3 * idx + 2]);
  const float3 pv = xform4x3(p, viewmatrix);
  present[idx] = (pv.z <= 0.2f) ? 0 : 1;
}

// ------------------------------------------------------------ launchers ----
cudaError_t launch_forward(const FwdArgs& a, cudaStream_t s) {
  cudaError_t e = launch_binning(a, s);
  return e != cudaSuccess ? e : launch_render(a, s);
}

// preprocess + per-tile binning / sort / record packing: short, latency-bound kernels
cudaError_t launch_binning(const FwdArgs& a, cudaStream_t s) {
  const unsigned gx = (a.W + TILE_X - 1) / TILE_X, gy = (a.H + TILE_Y - 1) / TILE_Y;
  const int T = gx * gy;
  GeomWS g = GeomWS::from((char*)a.geom_ws, a.P);
  ImgWS im = ImgWS::from((char*)a.img_ws, (size_t)a.W * a.H, T);
  BinWS b = BinWS::from((char*)a.binning_ws, (size_t)a.R_cap);
  const float focal_y = a.H / (2.0f * a.tan_fovy);
  const float focal_x = a.W / (2.0f * a.tan_fovx);
  const int pblocks = (a.P + 255) / 256;
  // (tile, bucket) counters + the two depth-range words that follow them
  cudaMemsetAsync(im.hist, 0, sizeof(uint32_t) * ((size_t)T * DEPTH_BUCKETS + 8), s);
  const int use_hint = (a.hint_hi > a.hint_lo) ? 1 : 0;
  g_prof.begin(0, s);
  if (use_hint) {
    launch_pdl(preprocess_kernel<true>, dim3(pblocks), dim3(256), 0, s, a.P, a.D, a.M, a.means3D, a.scales,
               a.scale_modifier, a.rotations, a.opacities, a.shs, a.cov3D_precomp, a.colors_precomp, a.viewmatrix,
               a.projmatrix, a.cam_pos, a.W, a.H, a.tan_fovx, a.tan_fovy, focal_x, focal_y, a.radii, g, gx, gy,
               im.depth_range, im.scan_flags, a.status, a.prefiltered, im.hist, a.hint_lo, a.hint_hi);
    g_prof.end(0, s);
  } else {
    launch_pdl(preprocess_kernel<false>, dim3(pblocks), dim3(256), 0, s, a.P, a.D, a.M, a.means3D, a.scales,
               a.scale_modifier, a.rotations, a.opacities, a.shs, a.cov3D_precomp, a.colors_precomp, a.viewmatrix,
               a.projmatrix, a.cam_pos, a.W, a.H, a.tan_fovx, a.tan_fovy, focal_x, focal_y, a.radii, g, gx, gy,
               im.depth_range, im.scan_flags, a.status, a.prefiltered, im.hist, 0.f, 0.f);
    g_prof.end(0, s);
    g_prof.begin(7, s);
    launch_pdl(count_kernel, dim3(pblocks), dim3(256), 0, s, a.P, g, im.hist, (const uint32_t*)im.depth_range, gx, gy);
    g_prof.end(7, s);
  }
  g_prof.begin(1, s);
  launch_pdl(tile_scan_kernel, dim3((T + 31) / 32), dim3(256), 0, s, T, im.hist, im.tile_total, im.ranges,
             im.tile_order, im.scan_flags, a.status, (long long)a.R_cap, (const uint32_t*)im.depth_range,
             (volatile int32_t*)a.status_host);
  g_prof.end(1, s);
  if (a.status_event) cudaEventRecord(a.status_event, s);
  g_prof.begin(2, s);
  launch_pdl(scatter_kernel, dim3(pblocks), dim3(256), 0, s, a.P, g, (const uint2*)im.ranges, im.hist,
             (const uint32_t*)im.depth_range, b.keys, gx, gy, (const int32_t*)a.status, use_hint, a.hint_lo, a.hint_hi);
  g_prof.end(2, s);
  g_prof.begin(3, s);
  // (a.hint_max_tile is advisory and no longer needed: the kernel walks a tile in stage-sized runs)
  // the normal map adds the normal stream to the depth records; the surface maps blend the depth records
  const bool nrm = a.out_normal, depth = a.out_depth || a.surf_ws || nrm;
  NrmWS n = {};
  if (nrm) {  // the backward's accumulator starts at zero
    n = NrmWS::from((char*)a.nrm_ws, a.P, (size_t)a.R_cap);
    cudaMemsetAsync(n.acc, 0, sizeof(float4) * (size_t)a.P, s);
  }
  launch_pdl(nrm ? tile_sort_pack_kernel<true, true> : depth ? tile_sort_pack_kernel<true> : tile_sort_pack_kernel<false>,
             dim3(T), dim3(256), 0, s, (const uint2*)im.ranges, (const uint32_t*)im.tile_order, b.keys,
             (const uint32_t*)im.hist, g, a.colors_precomp, depth ? (const float*)g.depths : nullptr, b,
             (const int32_t*)a.status, nrm ? a.normals : nullptr, n.inst_nrm);
  g_prof.end(3, s);
  return cudaGetLastError();
}

// the alpha-compositing kernel (fills the GPU): render_fwd_kernel<AUX, NRM, SURF> with NRM = out_normal, SURF =
// surf_ws, AUX = out_depth || out_alpha || NRM || SURF; the arguments of a map the instance does not write are NULL
cudaError_t launch_render(const FwdArgs& a, cudaStream_t s) {
  const unsigned gx = (a.W + TILE_X - 1) / TILE_X, gy = (a.H + TILE_Y - 1) / TILE_Y;
  const int T = gx * gy;
  ImgWS im = ImgWS::from((char*)a.img_ws, (size_t)a.W * a.H, T);
  BinWS b = BinWS::from((char*)a.binning_ws, (size_t)a.R_cap);
  const bool nrm = a.out_normal, surf = a.surf_ws, aux = a.out_depth || a.out_alpha || nrm || surf;
  NrmWS n = {};
  if (nrm) n = NrmWS::from((char*)a.nrm_ws, a.P, (size_t)a.R_cap);
  SurfWS sw = {};
  if (surf) sw = SurfWS::from((char*)a.surf_ws, (size_t)a.W * a.H);
  auto k = surf ? (nrm ? render_fwd_kernel<true, true, true> : render_fwd_kernel<true, false, true>)
           : nrm ? render_fwd_kernel<true, true>
           : aux ? render_fwd_kernel<true>
                 : render_fwd_kernel<false>;
  g_prof.begin(4, s);
  launch_pdl(k, dim3(T), dim3(256), 0, s, (const uint2*)im.ranges, (const uint32_t*)im.tile_order,
             (const float4*)b.inst_geo, (const float4*)b.inst_attr, a.W, a.H, a.background, im.final_T, im.n_contrib,
             a.out_color, (const int32_t*)a.status, a.out_depth, a.out_alpha, (const float4*)n.inst_nrm, a.out_normal,
             sw.median_id, sw.moments, surf ? a.out_median : nullptr, surf ? a.out_distortion : nullptr,
             surf ? a.surf_k : 0.f);
  g_prof.end(4, s);
  return cudaGetLastError();
}

cudaError_t launch_mark_visible(int P, const float* means3D, const float* view, const float* proj, uint8_t* present,
                                cudaStream_t s) {
  if (P > 0) mark_visible_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, means3D, view, proj, present);
  return cudaGetLastError();
}

}  // namespace dgm
