// raster_walk.cuh -- the walk of the side passes (feature_fwd_kernel, feature_bwd_kernel in raster_feat.cu,
// blend_stats_kernel in raster_stats.cu): passes over the workspaces an existing forward left behind (sorted blend
// records, tile ranges, tile order, n_contrib).  The walk repeats the forward's blend operation for operation (same
// quadratic form, alpha, 1/255 skip and stop at n_contrib), so the transmittance a side pass sees is the forward's
// bit for bit.
#pragma once
#include "raster_bwd_blend.cuh"

namespace dgm {

// A side-pass CTA's tile of one frame (frame f's workspaces at img_ws + f img_stride, bin_ws + f bin_stride) with
// the blend kernels' CTA -> tile -> warp block -> pixel mapping (tile_order; 8x4 pixels per warp).
struct SideTile {
  ImgWS im;
  BinWS b;
  unsigned tile, tid, lane, wid;
  int wx0, wy0;
  bool inside;
  uint32_t pix_id;
  float bx0, bx1, by0, by1;
  float2 npx2, npy2;
  uint2 range;
  int total, last, wmax, maxc;  // set by find_stops

  __device__ __forceinline__ SideTile(int W, int H, int f, const char* img_ws, size_t img_stride, const char* bin_ws,
                                      size_t bin_stride, int64_t R_cap) {
    const unsigned gx = (W + TILE_X - 1) / TILE_X, gy = (H + TILE_Y - 1) / TILE_Y;
    const size_t npix = (size_t)W * H;
    im = ImgWS::from(const_cast<char*>(img_ws) + f * img_stride, npix, (size_t)gx * gy);
    b = BinWS::from(const_cast<char*>(bin_ws) + f * bin_stride, (size_t)R_cap);
    tile = im.tile_order[blockIdx.x];
    const unsigned tx = tile % gx, ty = tile / gx;
    tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    wx0 = tx * TILE_X + (wid & 1) * 8, wy0 = ty * TILE_Y + (wid >> 1) * 4;
    const int px = wx0 + (lane & 7), py = wy0 + (lane >> 3);
    inside = px < W && py < H;
    pix_id = W * py + px;
    bx0 = (float)wx0, bx1 = (float)(wx0 + 7), by0 = (float)wy0, by1 = (float)(wy0 + 3);
    npx2 = make_float2(-(float)px, -(float)px), npy2 = make_float2(-(float)py, -(float)py);
  }

  // The tile's records and the positions past which the forward blended nothing: last for the pixel, wmax over the
  // warp, maxc over the CTA, capped at the tile's record count.  Called by the whole CTA (s_maxc a __shared__ int);
  // init() stores the kernel's initial shared memory, which the barriers here publish.
  template <class Init> __device__ __forceinline__ void find_stops(int* s_maxc, Init init) {
    range = im.ranges[tile];
    total = range.y - range.x;
    last = inside ? (int)im.n_contrib[pix_id] : 0;
    wmax = last;
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
    init();
    if (tid == 0) *s_maxc = 0;
    __syncthreads();
    int v = last;
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
    if (lane == 0) atomicMax(s_maxc, v);
    __syncthreads();
    maxc = min(*s_maxc, total);
  }
};

// Walk the tile's records front to back in batches of RB.  stage(base, cnt) puts positions [base, base + cnt) of
// the tile into shared memory, at least their inst_geo into s_geo and inst_attr[2 r] into s_con.  Each warp then
// pairs the records its block keeps (cull_keep) and calls record(q, j, opac, np, pre) for each of a pair (q = 0,
// then 1): record j of the batch, np = -power at the pixel (pair_npow), pre when the forward reached j with power
// <= 0.  record forms alpha = min(0.99, opac exp(-np)) and skips alpha < 1/255 itself, branching or branch-free as
// its kernel needs.  end(cnt) closes the batch; it starts with a barrier if it reads what other warps wrote.
template <class Stage, class Record, class End>
__device__ __forceinline__ void side_walk(const SideTile& t, const float4* s_geo, const float4* s_con, Stage stage,
                                          Record record, End end) {
  for (int base = 0; base < t.maxc; base += RB) {
    const int cnt = min(RB, t.maxc - base);
    __syncthreads();  // the previous batch is no longer read
    stage(base, cnt);
    __syncthreads();
    if (base < t.wmax) {  // (uniform per warp) something left for this warp's pixels
#pragma unroll 1
      for (int k = 0; k < RB / 32; ++k) {
        const int r = k * 32 + t.lane;
        const bool kp = r < cnt && base + r < t.wmax && cull_keep(s_geo[r], s_con[r], t.bx0, t.bx1, t.by0, t.by1);
        unsigned mask = __ballot_sync(0xffffffffu, kp);
        while (mask) {
          const int bA = __ffs(mask) - 1;
          mask &= mask - 1;
          const bool two = mask != 0;
          const int bB = two ? __ffs(mask) - 1 : bA;
          mask &= mask - 1;
          const int jA = k * 32 + bA, jB = k * 32 + bB;
          const float4 geA = s_geo[jA], geB = s_geo[jB];
          const float4 coA = s_con[jA], coB = s_con[jB];
          const float2 npow = pair_npow(geA, geB, coA, coB, t.npx2, t.npy2);
#pragma unroll
          for (int q = 0; q < 2; ++q) {
            const float np = q ? npow.y : npow.x;
            const float opac = q ? coB.w : coA.w;
            const int j = q ? jB : jA;
            record(q, j, opac, np, (q == 0 || two) && base + j < t.last && !(np < 0.0f));
          }
        }
      }
    }
    end(cnt);
  }
}

}  // namespace dgm
