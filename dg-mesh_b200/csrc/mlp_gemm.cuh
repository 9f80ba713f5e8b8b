// mlp_gemm.cuh -- the two tensor-core kernels of the deformation / appearance MLPs (Hopper wgmma, bf16
// operands, fp32 accumulators in registers), built around ONE global data layout.
//
// Blocked ("K-blocked") bf16 layout.  A matrix with F feature columns (F % 8 == 0) is stored in row
// tiles of R rows:  element (row, f) lives at
//     tile(row / R) * tile_stride  +  ((f / 8) * R + row % R) * 8 + f % 8            [elements]
// i.e. per tile, per 8-feature block ("kb"), R units of 16 bytes.  Activations use R = 128 (one tile =
// one 128-point M tile), weight matrices a single tile with R = number of output rows.
// Why: (1) a K-chunk of a tile (8 kbs) is ONE contiguous piece of memory that is already in the wgmma
// no-swizzle core-matrix order (wgmma.cuh), so an operand stage is filled by a single 1-D bulk copy
// (cp.async.bulk + mbarrier complete_tx) issued by one thread -- no per-thread address arithmetic,
// no tensor maps; (2) the epilogue's stores are coalesced (a warp's 4-byte stores for one column pair
// cover 8 consecutive rows = 128 contiguous bytes); (3) the SAME stored activations serve as MN-major
// operands of the weight-gradient GEMM (contraction over the points), so no transposed copies are ever
// written.
//
//   layer_gemm_kernel   D[rows, N] = A[rows, K] . B[N, K]^T          (forward layers, dZ back-propagation)
//       persistent CTAs (one per SM) over the 128-row tiles; warp-specialised:
//         warps 0-7  two consumer warpgroups; each multiplies 64 rows of the tile (wgmma m64nNk16,
//                    N <= 256, accumulators in registers) and runs the epilogue of its rows (bias / ReLU /
//                    ReLU bit-mask -> blocked bf16 store, fp32 store or fp32 reduction)
//         warp 8     producer: per 16-wide K step one bulk copy for A and one for B into a 16-stage ring;
//                    it runs ahead into the next tile while the consumers run their epilogue
//       The producer warpgroup (warps 8-11) hands its registers to the consumers (setmaxnreg): a 64 x 256
//       fp32 accumulator takes 128 registers per thread.
//   dw_gemm_kernel      C[Mf, Nf] += X[rows, Mf]^T . Y[rows, Nf]     (weight gradients)
//       both operands MN-major straight from the blocked activations; each CTA accumulates its share
//       of the row tiles in registers and adds its partial result to C once (red.global.add).
// N is a template parameter (the accumulator count is part of the wgmma instruction); the host
// dispatches on N = 16, 32, ..., 256 (DGM_GEMM_NS).
#pragma once
#include "wgmma.cuh"

namespace dgm {

#define ACT_R 128             // rows per activation tile
#define KB_ELEMS (ACT_R * 8)  // elements of one 8-feature block of an activation tile (2 KB)
#define DGM_GEMM_NS(X) \
  X(16) X(32) X(48) X(64) X(80) X(96) X(112) X(128) X(144) X(160) X(176) X(192) X(208) X(224) X(240) X(256)

// view of a blocked activation matrix: pointer to tile 0, elements between tiles, first kb used
struct BlkView {
  const __nv_bfloat16* p;
  size_t tile_stride;
  int kb0;
};

struct LayerArgs {
  BlkView A;                  // [tiles*128, K]
  const __nv_bfloat16* B;     // blocked single tile, R = N rows: [K/8][N][8]
  int K, N;                   // K % 16 == 0, N % 16 == 0, 16 <= N <= 256
  int tiles;                  // 128-row tiles
  const int* tiles_dev;       // optional: device-side cap on `tiles` (decided by an earlier kernel of the stream)
  int rows_valid;             // rows < rows_valid are written to the fp32 output
  const float* bias;          // [N] or null
  int relu;
  const uint32_t* mask_bits;  // null: none; else ReLU mask of a previous output: bit j of word
                              // [(tile*8 + c/32)*128 + row] keeps column c = 32*(c/32) + j
  uint32_t* mask_out;         // null: none; else write this output's (value > 0) bits in that layout
  __nv_bfloat16* out;         // blocked output (N columns from out_kb0) or null
  size_t out_tile_stride;
  int out_kb0;
  float* out_f32;             // row-major [rows, ld_f32] or null; first n_f32 columns
  int ld_f32, n_f32, atomic;  // atomic: accumulate with red.global.add
  // split precision ("bf16x3"): operands are pairs hi + lo of bf16 numbers (lo = the rounding
  // residual of hi), the product is A_hi B_hi + A_lo B_hi + A_hi B_lo accumulated in fp32 -- three
  // passes over K into the same accumulator, ~16 mantissa bits per operand.  A_lo / B_lo have
  // the geometry of A / B; out_lo (optional) receives the residual of the bf16 output.
  const __nv_bfloat16* A_lo;  // null: single pass
  const __nv_bfloat16* B_lo;
  __nv_bfloat16* out_lo;
};

#define GEMM_THREADS 384        // two consumer warpgroups (warps 0-7) + the producer warpgroup (warps 8-11)
#define GEMM_PRODUCER_WARP 8
#define GEMM_CONSUMER_WARPS 8   // a ring stage is free once every consumer warp has released it
#define GEMM_PRODUCER_REGS 40   // 4 warps x 40 + 8 warps x 232 registers x 32 lanes <= 64 K
#define GEMM_CONSUMER_REGS 232
// One ring stage per 16-wide K step (one wgmma per consumer warpgroup and stage): every wgmma is issued on a
// warp-uniform path, whatever K is.
#define LG_STAGES 16
#define LG_A_BYTES (ACT_R * 16 * 2)  // 4 KB: 128 rows x 16 K
#define LG_STAGE_BYTES (LG_A_BYTES + 256 * 16 * 2)  // + up to 256 rows x 16 K of B
#define LG_SMEM (LG_STAGES * LG_STAGE_BYTES + 1024)
// RESIDENT variant (RES = true; split-precision layers whose weight matrix fits 128 KB, i.e. every 256x256 layer):
// in the streaming variant such a layer re-fetches the weights through L2 for every tile and pass (704 KB per
// 128-row tile).  Here B_hi is loaded into shared memory ONCE per CTA; the ring carries only what changes per
// tile, in 16 KB stages: one 16-wide K step of A_hi, A_lo and B_lo -- the three products of a K step are issued
// back to back (A_hi B_hi, A_lo B_hi, A_hi B_lo), so A_hi is fetched once, not twice.  L2 traffic per tile:
// 704 -> 384 KB.  (Single-pass launches keep the streaming variant.)
#define LGR_B_BYTES 131072
#define LGR_STAGES 5
#define LGR_STAGE_BYTES 16384
#define LGR_SMEM (LGR_B_BYTES + LGR_STAGES * LGR_STAGE_BYTES + 1024)
#define LG_MAX_STAGES 16

__device__ __forceinline__ void producer_regs() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(GEMM_PRODUCER_REGS));
}
__device__ __forceinline__ void consumer_regs() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(GEMM_CONSUMER_REGS));
}

// one arrival per consumer warp: the warpgroup's wgmma reading the stage has completed
__device__ __forceinline__ void release_stage(uint64_t* bar, int lane) {
  __syncwarp();
  if (lane == 0) mbar_arrive(bar);
}

template <bool RES, int NT>
__global__ void __launch_bounds__(GEMM_THREADS, 1) layer_gemm_kernel(const LayerArgs g) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t s_full[LG_MAX_STAGES], s_empty[LG_MAX_STAGES], s_bres;
  __shared__ float s_bias[256];
  constexpr int NST = RES ? LGR_STAGES : LG_STAGES;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t ring = (smem_u32(smem_raw) + 1023u) & ~1023u;  // 1 KB aligned operand ring
  const uint32_t sLG = ring;                                      // streaming variant
  const uint32_t sBres = ring, sStage = ring + LGR_B_BYTES;      // resident variant

  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < NST; ++s) {
      mbar_init(&s_full[s], 1);
      mbar_init(&s_empty[s], GEMM_CONSUMER_WARPS);
    }
    mbar_init(&s_bres, 1);
    mbar_fence_init();
  }
  for (int i = tid; i < 256; i += GEMM_THREADS) s_bias[i] = (g.bias && i < g.N) ? g.bias[i] : 0.f;
  __syncthreads();

  const int nkb = g.K >> 3;  // 8-wide k blocks
  const int nks = nkb >> 1;  // 16-wide K steps
  const int npasses = g.A_lo ? 3 : 1;
  const int n_tiles = g.tiles_dev ? min(g.tiles, *g.tiles_dev) : g.tiles;
  const int my_tiles = (n_tiles > (int)blockIdx.x) ? (n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;

  if (warp >= GEMM_PRODUCER_WARP) {
    // ------------------------------------------------------------ producer
    producer_regs();
    if (warp != GEMM_PRODUCER_WARP) return;
    if (RES && lane == 0) {
      if (my_tiles > 0) {  // the resident weights, once
        const uint32_t bytes = (uint32_t)nkb * g.N * 16;
        mbar_expect_tx(&s_bres, bytes);
        for (uint32_t off = 0; off < bytes; off += 32768u)
          tma_load_1d_u32(sBres + off, reinterpret_cast<const uint8_t*>(g.B) + off, min(32768u, bytes - off), &s_bres);
      }
      uint32_t it = 0;
      for (int i = 0; i < my_tiles; ++i) {
        const int tile = blockIdx.x + i * gridDim.x;
        const size_t a_off = (size_t)tile * g.A.tile_stride + (size_t)g.A.kb0 * KB_ELEMS;
        const uint32_t bl_bytes = (uint32_t)g.N * 32;  // two k blocks of B_lo
        for (int c = 0; c < nks; ++c, ++it) {
          const int st = it % NST;
          mbar_wait(&s_empty[st], ((it / NST) & 1) ^ 1);
          mbar_expect_tx(&s_full[st], 2 * 4096u + bl_bytes);
          const uint32_t dst = sStage + st * LGR_STAGE_BYTES;
          tma_load_1d_u32(dst, g.A.p + a_off + (size_t)c * 2 * KB_ELEMS, 4096u, &s_full[st]);
          tma_load_1d_u32(dst + 4096u, g.A_lo + a_off + (size_t)c * 2 * KB_ELEMS, 4096u, &s_full[st]);
          tma_load_1d_u32(dst + 8192u, g.B_lo + (size_t)c * 2 * g.N * 8, bl_bytes, &s_full[st]);
        }
      }
    } else if (!RES && lane == 0) {
      uint32_t it = 0;
      for (int i = 0; i < my_tiles; ++i) {
        const int tile = blockIdx.x + i * gridDim.x;
        const size_t a_off = (size_t)tile * g.A.tile_stride + (size_t)g.A.kb0 * KB_ELEMS;
        for (int pass = 0; pass < npasses; ++pass) {
          // pass 0: A_hi B_hi, pass 1: A_lo B_hi, pass 2: A_hi B_lo
          const __nv_bfloat16* a_tile = ((pass == 1) ? g.A_lo : g.A.p) + a_off;
          const __nv_bfloat16* b_mat = (pass == 2) ? g.B_lo : g.B;
          const uint32_t b_bytes = (uint32_t)g.N * 32;  // two k blocks of B
          for (int c = 0; c < nks; ++c, ++it) {
            const int st = it % LG_STAGES;
            mbar_wait(&s_empty[st], ((it / LG_STAGES) & 1) ^ 1);
            mbar_expect_tx(&s_full[st], LG_A_BYTES + b_bytes);
            const uint32_t dst = sLG + st * LG_STAGE_BYTES;
            tma_load_1d_u32(dst, a_tile + (size_t)c * 2 * KB_ELEMS, LG_A_BYTES, &s_full[st]);
            tma_load_1d_u32(dst + LG_A_BYTES, b_mat + (size_t)c * 2 * g.N * 8, b_bytes, &s_full[st]);
          }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------- consumers (warpgroups 0 and 1)
  consumer_regs();
  const int wg = warp >> 2;                               // rows 64 wg .. 64 wg + 63 of every tile
  const uint32_t a_half = (uint32_t)wg * 64 * 16;         // byte offset of those rows in a K-major A stage
  const uint32_t lbo_b = g.N * 16;                        // K-major B: N rows per k block
  const int quad = lane & 3;
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's rows: r0 and r0 + 8
  constexpr int NQ = (NT + 31) / 32;                       // 32-column groups (ReLU-mask words)
  float acc[NT / 2];
  uint32_t it = 0;
  for (int i = 0; i < my_tiles; ++i) {
    const int tile = blockIdx.x + i * gridDim.x;
    int prev = -1;  // ring stage still read by the wgmma group in flight
    if (RES) {
      if (i == 0) mbar_wait(&s_bres, 0);
      for (int c = 0; c < nks; ++c, ++it) {
        const int st = it % NST;
        mbar_wait(&s_full[st], (it / NST) & 1);
        const uint32_t base = sStage + st * LGR_STAGE_BYTES;
        const uint64_t da_hi = wgmma::smem_desc(base + a_half, ACT_R * 16, 128);
        const uint64_t da_lo = wgmma::smem_desc(base + 4096u + a_half, ACT_R * 16, 128);
        const uint64_t db_hi = wgmma::smem_desc(sBres + (uint32_t)(2 * c) * lbo_b, lbo_b, 128);
        const uint64_t db_lo = wgmma::smem_desc(base + 8192u, lbo_b, 128);
        wgmma::fence();
        wgmma::mma_bf16<NT, 0>(acc, da_hi, db_hi, c != 0);
        wgmma::mma_bf16<NT, 0>(acc, da_lo, db_hi, 1);
        wgmma::mma_bf16<NT, 0>(acc, da_hi, db_lo, 1);
        wgmma::commit();
        wgmma::wait<1>();
        if (prev >= 0) release_stage(&s_empty[prev], lane);
        prev = st;
      }
    } else {
      for (int pc = 0; pc < npasses * nks; ++pc, ++it) {
        const int st = it % LG_STAGES;
        mbar_wait(&s_full[st], (it / LG_STAGES) & 1);
        const uint32_t base = sLG + st * LG_STAGE_BYTES;
        wgmma::fence();
        wgmma::mma_bf16<NT, 0>(acc, wgmma::smem_desc(base + a_half, ACT_R * 16, 128),
                               wgmma::smem_desc(base + LG_A_BYTES, lbo_b, 128), pc != 0);
        wgmma::commit();
        wgmma::wait<1>();
        if (prev >= 0) release_stage(&s_empty[prev], lane);
        prev = st;
      }
    }
    wgmma::wait<0>();
    wgmma::fence_operands(acc);
    if (prev >= 0) release_stage(&s_empty[prev], lane);

    // ---- epilogue: this thread holds columns 8 j + 2 quad + {0, 1} of rows r0 and r0 + 8; one 32-column group
    // (one ReLU-mask word per row) at a time
    __nv_bfloat16* ot = g.out ? g.out + (size_t)tile * g.out_tile_stride : nullptr;
    __nv_bfloat16* ol = g.out_lo ? g.out_lo + (size_t)tile * g.out_tile_stride : nullptr;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = r0 + 8 * h;
      const size_t row = (size_t)tile * ACT_R + r;
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        const uint32_t mb = g.mask_bits ? g.mask_bits[((size_t)tile * 8 + q) * ACT_R + r] : 0xffffffffu;
        uint32_t pos = 0;
#pragma unroll
        for (int j = 4 * q; j < 4 * q + 4 && j < NT / 8; ++j) {
          const int col = 8 * j + 2 * quad;
          const int bit = col & 31;
          float v0 = acc[4 * j + 2 * h] + s_bias[col], v1 = acc[4 * j + 2 * h + 1] + s_bias[col + 1];
          if (g.relu) {
            v0 = fmaxf(v0, 0.0f);
            v1 = fmaxf(v1, 0.0f);
          }
          v0 = ((mb >> bit) & 1u) ? v0 : 0.0f;
          v1 = ((mb >> (bit + 1)) & 1u) ? v1 : 0.0f;
          pos |= ((v0 > 0.0f ? 1u : 0u) << bit) | ((v1 > 0.0f ? 1u : 0u) << (bit + 1));
          if (ot) {
            const __nv_bfloat162 hi = __floats2bfloat162_rn(v0, v1);
            const size_t off = ((size_t)(g.out_kb0 + j) * ACT_R + r) * 8 + 2 * quad;
            *reinterpret_cast<__nv_bfloat162*>(ot + off) = hi;
            if (ol) {  // the rounding residual as a second bf16 number
              const float2 hf = __bfloat1622float2(hi);
              *reinterpret_cast<__nv_bfloat162*>(ol + off) = __floats2bfloat162_rn(v0 - hf.x, v1 - hf.y);
            }
          }
          if (g.out_f32 && row < (size_t)g.rows_valid && col < g.n_f32) {
            float* dst = g.out_f32 + row * g.ld_f32 + col;
            if (col + 1 < g.n_f32) {
              if (g.atomic) red_add_v2(dst, v0, v1);
              else *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
            } else {
              if (g.atomic) atomicAdd(dst, v0);
              else *dst = v0;
            }
          }
        }
        if (g.mask_out) {  // uniform: the four threads of a quad hold the row's 32 columns together
          pos |= __shfl_xor_sync(0xffffffffu, pos, 1);
          pos |= __shfl_xor_sync(0xffffffffu, pos, 2);
          if (quad == 0) g.mask_out[((size_t)tile * 8 + q) * ACT_R + r] = pos;
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
struct DwArgs {
  BlkView X;      // rows x 256 features: CTA (blockIdx.y) takes features [X.kb0*8 + 128*blockIdx.y, +128)
  BlkView Y;      // rows x N features from Y.kb0
  int N;          // multiple of 16, <= 256
  int tiles;
  const int* tiles_dev;  // optional device-side cap on `tiles`
  float* C;       // fp32, leading dimension ld (even)
  int ld;
  int transpose;  // 0: C[m, n] (m = X feature, n = Y feature);  1: C[n, m]
  int m_valid;    // X features >= m_valid are not written
  int n_valid;
  // optional bias gradients from the operand tiles already staged in shared memory (the first consumer
  // warpgroup sums them while its wgmma runs): colsum_x[f] += sum over rows of X[:, f] (f relative to the view)
  // for this CTA's 128 features, colsum_y[f] += sum over rows of Y[:, f] (N <= 128; CTAs with blockIdx.y == 0
  // only)
  float* colsum_x;
  float* colsum_y;
};

#define DW_STAGES 2
#define DW_A_BYTES (128 * ACT_R * 2)  // 32 KB: 128 features x 128 rows
#define DW_B_BYTES (256 * ACT_R * 2)  // 64 KB
#define DW_SMEM (DW_STAGES * (DW_A_BYTES + DW_B_BYTES) + 1024)

template <int NT>
__global__ void __launch_bounds__(GEMM_THREADS, 1) dw_gemm_kernel(const DwArgs g) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t s_full[DW_STAGES], s_empty[DW_STAGES];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t ring = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sA = ring, sB = ring + DW_STAGES * DW_A_BYTES;
  const bool sum_x = g.colsum_x != nullptr, sum_y = g.colsum_y != nullptr && blockIdx.y == 0 && g.N <= 128;
  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < DW_STAGES; ++s) {
      mbar_init(&s_full[s], 1);
      mbar_init(&s_empty[s], GEMM_CONSUMER_WARPS);
    }
    mbar_fence_init();
  }
  __syncthreads();
  const int n_tiles = g.tiles_dev ? min(g.tiles, *g.tiles_dev) : g.tiles;
  const int my_tiles = (n_tiles > (int)blockIdx.x) ? (n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  const int m0 = blockIdx.y * 128;  // first X feature of this CTA

  if (warp >= GEMM_PRODUCER_WARP) {
    producer_regs();
    if (warp == GEMM_PRODUCER_WARP && lane == 0) {
      for (int i = 0; i < my_tiles; ++i) {
        const int tile = blockIdx.x + i * gridDim.x;
        const int st = i % DW_STAGES;
        mbar_wait(&s_empty[st], ((i / DW_STAGES) & 1) ^ 1);
        const uint32_t a_bytes = 16 * (ACT_R * 16), b_bytes = (g.N >> 3) * (ACT_R * 16);
        mbar_expect_tx(&s_full[st], a_bytes + b_bytes);
        tma_load_1d_u32(sA + st * DW_A_BYTES,
                        g.X.p + (size_t)tile * g.X.tile_stride + (size_t)(g.X.kb0 + (m0 >> 3)) * KB_ELEMS, a_bytes,
                        &s_full[st]);
        tma_load_1d_u32(sB + st * DW_B_BYTES, g.Y.p + (size_t)tile * g.Y.tile_stride + (size_t)g.Y.kb0 * KB_ELEMS,
                        b_bytes, &s_full[st]);
      }
    }
    return;
  }
  consumer_regs();
  if (my_tiles == 0) return;

  // -------------------------------------------------------------- consumers (warpgroups 0 and 1)
  // both operands MN-major: core matrix = 8 rows (K) x 8 features; K groups 128 B apart (LBO), feature
  // groups one kb = 2 KB apart (SBO).  Warpgroup wg takes the CTA's features 64 wg .. 64 wg + 63.
  const int wg = warp >> 2;
  const bool sums = (sum_x || sum_y) && wg == 0;
  // column sums: 8 threads per 8-feature block, 16 rows each (conflict-free LDS.128)
  const int kb = tid >> 3, sub = tid & 7;
  float ax[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, ay[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const bool do_y = sum_y && kb < (g.N >> 3);
  const uint8_t* ring_p = reinterpret_cast<const uint8_t*>(smem_raw) + (ring - smem_u32(smem_raw));
  float acc[NT / 2];
  int prev = -1;
  for (int i = 0; i < my_tiles; ++i) {
    const int st = i % DW_STAGES;
    mbar_wait(&s_full[st], (i / DW_STAGES) & 1);
    wgmma::fence();
#pragma unroll
    for (int ks = 0; ks < ACT_R / 16; ++ks) {
      const uint64_t da = wgmma::smem_desc(sA + st * DW_A_BYTES + wg * 8 * (ACT_R * 16) + ks * 256, 128, ACT_R * 16);
      const uint64_t db = wgmma::smem_desc(sB + st * DW_B_BYTES + ks * 256, 128, ACT_R * 16);
      wgmma::mma_bf16<NT, 1>(acc, da, db, (i | ks) != 0);
    }
    wgmma::commit();
    if (sums) {  // ---- column sums of the staged operand tiles while the tensor core multiplies them
      const uint8_t* pa = ring_p + st * DW_A_BYTES + kb * (ACT_R * 16);
      const uint8_t* pb = ring_p + DW_STAGES * DW_A_BYTES + st * DW_B_BYTES + kb * (ACT_R * 16);
#pragma unroll 4
      for (int r = sub; r < ACT_R; r += 8) {
        if (sum_x) {
          const uint4 v = *reinterpret_cast<const uint4*>(pa + r * 16);
          const __nv_bfloat162* p2 = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float2 f = __bfloat1622float2(p2[q]);
            ax[2 * q] += f.x;
            ax[2 * q + 1] += f.y;
          }
        }
        if (do_y) {
          const uint4 v = *reinterpret_cast<const uint4*>(pb + r * 16);
          const __nv_bfloat162* p2 = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float2 f = __bfloat1622float2(p2[q]);
            ay[2 * q] += f.x;
            ay[2 * q + 1] += f.y;
          }
        }
      }
    }
    wgmma::wait<1>();
    if (prev >= 0) release_stage(&s_empty[prev], lane);
    prev = st;
  }
  wgmma::wait<0>();
  wgmma::fence_operands(acc);
  release_stage(&s_empty[prev], lane);

  if (sums) {
    // the 8 threads of a feature block are consecutive lanes
#pragma unroll
    for (int q = 0; q < 8; ++q) {
#pragma unroll
      for (int o = 1; o < 8; o <<= 1) {
        ax[q] += __shfl_xor_sync(0xffffffffu, ax[q], o);
        ay[q] += __shfl_xor_sync(0xffffffffu, ay[q], o);
      }
    }
    if (sub == 0) {
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        if (sum_x) atomicAdd(&g.colsum_x[m0 + kb * 8 + q], ax[q]);
        if (do_y) atomicAdd(&g.colsum_y[kb * 8 + q], ay[q]);
      }
    }
  }
  // ---- epilogue: accumulator rows are X features, columns Y features
  const int quad = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
    if (m >= g.m_valid) continue;
#pragma unroll
    for (int j = 0; j < NT / 8; ++j) {
      const int n = 8 * j + 2 * quad;
      const float a0 = acc[4 * j + 2 * h], a1 = acc[4 * j + 2 * h + 1];
      if (!g.transpose) {
        float* dst = g.C + (size_t)m * g.ld + n;
        if (n + 1 < g.n_valid) red_add_v2(dst, a0, a1);
        else if (n < g.n_valid) atomicAdd(dst, a0);
      } else {
        if (n < g.n_valid) atomicAdd(g.C + (size_t)n * g.ld + m, a0);
        if (n + 1 < g.n_valid) atomicAdd(g.C + (size_t)(n + 1) * g.ld + m, a1);
      }
    }
  }
}

}  // namespace dgm
