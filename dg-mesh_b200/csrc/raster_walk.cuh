// raster_walk.cuh -- the walk of the side passes (the feature kernels in raster_feat.cu, the planar kernels in
// raster_planar.cu, blend_stats_kernel in raster_stats.cu): passes over the workspaces an existing forward left
// behind (sorted blend records, tile ranges, tile order, n_contrib).  The walk repeats the forward's blend operation
// for operation (same quadratic form, alpha, 1/255 skip and stop at n_contrib), so the transmittance a side pass sees
// is the forward's bit for bit.  The side passes' backward kernels share side_bwd_walk on top of it.
#pragma once
#include <type_traits>
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

// The backward walk of a side pass (feature_bwd_kernel, planar_bwd_kernel), called by the whole CTA: side_walk with
// the forward's T and its branch-free alpha / 1/255 gate.  Each warp stages w = G dL/dG and alpha T of the records
// it blends in its CHUNK slots of s_stage (STAGE_BYTES of dynamic shared memory) and contracts them with its four
// dL/dpixel rows s_dlp[wid] (contract_chunk<true>) when a pair leaves no room for another and at the batch's end.
// After the batch's barrier each record's six moments go to floats 0-5 of grad_acc, as the blend backward turns them
// into dL/dmean2D, dL/dconic and dL/dopacity.  A CTA whose pixels blend nothing returns before rows().
//   rows()                     the warp's dL/dpixel rows into s_dlp[wid], and the per-pixel values dla reads
//   stage(base, cnt)           as side_walk's, and each record's Gaussian id into s_id
//   dla(j, alpha, T, act)      dL/dalpha of record j at the pixel; advances the kernel's prefix of its map when act
//                              (the pixel blends the record)
//   flush(r, id, a)            adds record r's own totals a[6..9] into the kernel's accumulator; returns void, or a
//                              float2 that the flush adds to dL/dmean2D's two sums before their W/2, H/2 scale
template <class Rows, class Stage, class DLa, class Flush>
__device__ __forceinline__ void side_bwd_walk(SideTile& t, int W, int H, int* s_maxc, const float4* s_geo,
                                              const float4* s_con, const uint32_t* s_id, float* s_acc,
                                              float (*s_dlp)[4][32], float* s_stage, float4* grad_acc, Rows rows,
                                              Stage stage, DLa dla, Flush flush) {
  constexpr int ACC_STRIDE = acc_stride<true>();
  const float cx = t.wx0 + 3.5f, cy = t.wy0 + 1.5f;  // centre of the warp's block
  t.find_stops(s_maxc, [&] {
    for (int i = t.tid; i < RB * ACC_STRIDE; i += 256) s_acc[i] = 0.f;
  });
  if (t.maxc == 0) return;  // uniform per CTA
  rows();
  float* const stg = s_stage + t.wid * (CHUNK * SLOT_F);
  int nslot = 0, rec = 0;  // staged records; the record of slot lane & 15
  float T = 1.0f;

  side_walk(
      t, s_geo, s_con, stage,
      [&](int q, int j, float opac, float np, bool pre) {
        const float G = expf(-np);
        const float alpha = fminf(0.99f, __fmul_rn(opac, G));
        const bool act = pre && !(alpha < 1.0f / 255.0f);
        const float dLa = dla(j, alpha, T, act);
        const float w = act ? (G * opac) * dLa : 0.0f;
        const float aT = act ? alpha * T : 0.0f;
        T = act ? __fmul_rn(T, __fadd_rn(1.0f, -alpha)) : T;
        if (__any_sync(0xffffffffu, act)) {
          stg[nslot * SLOT_F + t.lane] = w;
          stg[nslot * SLOT_F + 32 + t.lane] = aT;
          if ((int)(t.lane & 15) == nslot) rec = j;
          ++nslot;
        }
        if (q == 1 && nslot > CHUNK - 2) {  // the pair is staged and there is no room for another
          __syncwarp();
          contract_chunk<true>(stg, &s_dlp[t.wid][0][0], nslot, rec, t.lane, s_geo, cx, cy, s_acc);
          __syncwarp();
          nslot = 0;
        }
      },
      [&](int cnt) {
        if (nslot > 0) {  // the batch's records must be in s_acc before the flush
          __syncwarp();
          contract_chunk<true>(stg, &s_dlp[t.wid][0][0], nslot, rec, t.lane, s_geo, cx, cy, s_acc);
          __syncwarp();
          nslot = 0;
        }
        __syncthreads();
        // ---- flush this batch: the moments as the blend backward turns them into gradients, and the kernel's sums
        if ((int)t.tid < cnt) {
          float* acc = &s_acc[t.tid * ACC_STRIDE];
          float a[ACC_STRIDE];
          bool nz = false;
#pragma unroll
          for (int q = 0; q < ACC_STRIDE; ++q) {
            a[q] = acc[q];
            nz |= (a[q] != 0.f);
            acc[q] = 0.f;
          }
          if (nz) {
            const float ddelx_dx = 0.5 * W;
            const float ddely_dy = 0.5 * H;
            const float4 con_o = s_con[t.tid];
            const uint32_t id = s_id[t.tid];
            float sx = con_o.x * a[1] + con_o.y * a[2], sy = con_o.z * a[2] + con_o.y * a[1];
            if constexpr (std::is_void_v<decltype(flush(t.tid, id, a))>) {
              flush(t.tid, id, a);
            } else {
              const float2 m = flush(t.tid, id, a);
              sx += m.x, sy += m.y;
            }
            const float g_mx = -ddelx_dx * sx;
            const float g_my = -ddely_dy * sy;
            const float g_op = (con_o.w != 0.0f) ? a[0] / con_o.w : 0.0f;
            float* dst = reinterpret_cast<float*>(grad_acc + 3 * (size_t)id);
            red_add_v4(dst, g_mx, g_my, -0.5f * a[3], -0.5f * a[4]);
            red_add_v2(dst + 4, -0.5f * a[5], g_op);
          }
        }
      });
}

// a side-pass backward kernel's launch attributes, once per device: the staging areas' STAGE_BYTES of dynamic
// shared memory and the largest shared-memory carveout
template <auto Kernel> void side_bwd_attributes() {
  static unsigned long long attr = 0;  // per device
  if (once_per_device(attr)) {
    cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, STAGE_BYTES);
    cudaFuncSetAttribute(Kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  }
}

}  // namespace dgm
