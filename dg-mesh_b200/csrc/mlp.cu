// mlp.cu -- deformation / appearance MLPs on the Hopper tensor cores (wgmma).
//
// The networks (dgmesh/utils/time_utils.py): DeformNetwork / DeformNetworkNormal /
// DeformNetworkNormalSep / AppearanceNetwork share one trunk --
//   x_emb = pe(x, 10) [63], t_emb = pe(t, 6) [13] -> timenet 13->256->30 (is_blender)
//                            or pe(t, 10) [21]                       (otherwise)
//   h = [x_emb, t_emb] -> 8 x (Linear + ReLU), width 256, [x_emb, t_emb] re-concatenated after
//   layer 4 (time_utils.py:178-188) -> linear heads (13 / 3 / 10 outputs, sigmoid for colour)
// -- and run here as a chain of the two GEMM kernels of mlp_gemm.cuh over BLOCKED bf16 activations
// (layout: mlp_gemm.cuh).  Activation buffers, Pp = P rounded up to 128 rows:
//   A5 [Pp, 352] : features 0..62 x_emb | 63: 0 | 64..64+in_t-1 time features | ..95: 0 | 96..351 h4
//                  (layer 0 reads the first 12 kbs; the skip layer reads all 44: no concat copy)
//   T0 [Pp, 16], T1 [Pp, 256] (timenet), H[l] [Pp, 256]
// Training keeps every activation (they double as the MN-major operands of the weight-gradient
// GEMMs -- no transposed copies); inference ping-pongs two buffers.
#include <stdlib.h>

#include "mlp_gemm.cuh"
#include "mlp_kernels.h"

namespace dgm {

#define XE 63      // x embedding width
#define TCOL 64    // first feature of the time block
#define K0 96      // padded width of [x_emb, t features]
#define K5 352     // skip layer input width
#define WID 256

static int g_sms = 0;
static int sm_count() {
  if (!g_sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_sms <= 0) g_sms = DGM_NUM_SMS;
  }
  return g_sms;
}

typedef void (*LayerKernel)(const LayerArgs);
typedef void (*DwKernel)(const DwArgs);
static LayerKernel layer_kernel(bool resident, int N) {
  switch (N) {
#define DGM_CASE(n) \
  case n: return resident ? layer_gemm_kernel<true, n> : layer_gemm_kernel<false, n>;
    DGM_GEMM_NS(DGM_CASE)
#undef DGM_CASE
  }
  return nullptr;
}
static DwKernel dw_kernel(int N) {
  switch (N) {
#define DGM_CASE(n) \
  case n: return dw_gemm_kernel<n>;
    DGM_GEMM_NS(DGM_CASE)
#undef DGM_CASE
  }
  return nullptr;
}

cudaError_t launch_layer_gemm(const LayerArgs& g, cudaStream_t s) {
  static unsigned long long attr = 0;  // per device
  if (once_per_device(attr)) {
    for (int n = 16; n <= 256; n += 16) {
      cudaFuncSetAttribute(layer_kernel(false, n), cudaFuncAttributeMaxDynamicSharedMemorySize, LG_SMEM);
      cudaFuncSetAttribute(layer_kernel(true, n), cudaFuncAttributeMaxDynamicSharedMemorySize, LGR_SMEM);
    }
  }
  if (g.tiles <= 0) return cudaSuccess;
  if (g.N % 16 != 0 || g.N < 16 || g.N > 256 || g.K % 16 != 0 || g.K <= 0) return cudaErrorInvalidValue;
  // split-precision layers whose weights fit 128 KB keep B_hi in shared memory for the CTA's lifetime (every
  // 256-wide layer; the K = 320 skip layer streams).  Single-pass launches (the backward, bf16 mode) stay on the
  // streaming variant.  DGMESH_B200_MLP_STREAM=1 forces the streaming variant everywhere (A/B comparison).
  static const bool force_stream = [] {
    const char* e = getenv("DGMESH_B200_MLP_STREAM");
    return e && e[0] == '1';
  }();
  const bool resident = !force_stream && g.A_lo != nullptr && (size_t)(g.K >> 3) * g.N * 16 <= LGR_B_BYTES;
  layer_kernel(resident, g.N)<<<min(g.tiles, sm_count()), GEMM_THREADS, resident ? LGR_SMEM : LG_SMEM, s>>>(g);
  return cudaGetLastError();
}

// X has 256 features (two 128-feature halves -> grid.y = 2)
cudaError_t launch_dw_gemm(const DwArgs& g, cudaStream_t s) {
  static unsigned long long attr = 0;  // per device
  if (once_per_device(attr))
    for (int n = 16; n <= 256; n += 16)
      cudaFuncSetAttribute(dw_kernel(n), cudaFuncAttributeMaxDynamicSharedMemorySize, DW_SMEM);
  if (g.tiles <= 0) return cudaSuccess;
  if (g.N % 16 != 0 || g.N < 16 || g.N > 256) return cudaErrorInvalidValue;
  dim3 grid(min(g.tiles, max(1, sm_count() / 2)), 2);
  dw_kernel(g.N)<<<grid, GEMM_THREADS, DW_SMEM, s>>>(g);
  return cudaGetLastError();
}

struct MlpBufs {
  __nv_bfloat16 *A5, *T0, *T1, *H[8];  // H[4] = A5 viewed from kb 12
  __nv_bfloat16 *dZ[2], *dZh, *dZt1;
  uint32_t *M[8], *Mt1;                 // ReLU masks as bits, [tiles][8][128] words (training only)
  float* dE;                            // [Pp, 96] fp32 row-major: gradient w.r.t. the embedded inputs
  // split-precision forward: rounding residuals of A5 / T0 / T1 and of the running hidden activation
  __nv_bfloat16 *A5lo, *T0lo, *T1lo, *Hlo[2];
  // uniform-time shortcut: tu[0] = 1 when every row has the same t (decided on the device), tu[1] = tiles the
  // time-net kernels process (1 or all); tsum[32] = column sums of the time-feature gradients
  int* tu;
  float* tsum;
  int Pp, tiles;
  static MlpBufs carve_all(char* base, int P, int train, size_t* bytes) {
    char* p = base;
    MlpBufs b;
    const size_t Pp = ((size_t)P + ACT_R - 1) / ACT_R * ACT_R;
    b.Pp = (int)Pp;
    b.tiles = (int)(Pp / ACT_R);
    b.A5 = carve<__nv_bfloat16>(p, Pp * K5);
    b.T0 = carve<__nv_bfloat16>(p, Pp * 16);
    b.T1 = carve<__nv_bfloat16>(p, Pp * WID);
    b.A5lo = carve<__nv_bfloat16>(p, Pp * K5);
    b.T0lo = carve<__nv_bfloat16>(p, Pp * 16);
    b.T1lo = carve<__nv_bfloat16>(p, Pp * WID);
    b.Hlo[0] = carve<__nv_bfloat16>(p, Pp * WID);
    b.Hlo[1] = carve<__nv_bfloat16>(p, Pp * WID);
    b.tu = carve<int>(p, 32);
    b.tsum = carve<float>(p, 32);
    if (train) {
      for (int l = 0; l < 8; ++l) b.H[l] = (l == 4) ? b.A5 : carve<__nv_bfloat16>(p, Pp * WID);
      for (int i = 0; i < 2; ++i) b.dZ[i] = carve<__nv_bfloat16>(p, Pp * WID);
      b.dZh = carve<__nv_bfloat16>(p, Pp * 16);
      b.dZt1 = carve<__nv_bfloat16>(p, Pp * 32);
      b.dE = carve<float>(p, Pp * K0);
      for (int l = 0; l < 8; ++l) b.M[l] = carve<uint32_t>(p, Pp * 8);
      b.Mt1 = carve<uint32_t>(p, Pp * 8);
    } else {
      __nv_bfloat16* ping = carve<__nv_bfloat16>(p, Pp * WID);
      __nv_bfloat16* pong = carve<__nv_bfloat16>(p, Pp * WID);
      for (int l = 0; l < 8; ++l) b.H[l] = (l == 4) ? b.A5 : ((l & 1) ? pong : ping);
      b.dZ[0] = b.dZ[1] = b.dZh = b.dZt1 = nullptr;
      b.dE = nullptr;
      for (int l = 0; l < 8; ++l) b.M[l] = nullptr;
      b.Mt1 = nullptr;
    }
    if (bytes) *bytes = size_t(p - base) + 128;
    return b;
  }
  // blocked views
  BlkView h(int l) const {  // output of layer l
    return (l == 4) ? BlkView{A5, (size_t)K5 * ACT_R, K0 / 8} : BlkView{H[l], (size_t)WID * ACT_R, 0};
  }
  BlkView a5() const { return BlkView{A5, (size_t)K5 * ACT_R, 0}; }
  // residual buffer with the geometry of h(l): layer l's output residual / layer l+1's input residual
  __nv_bfloat16* hlo(int l) const { return (l == 4) ? A5lo : Hlo[l & 1]; }
};

__device__ __forceinline__ uint4 pack8(const float* v) {
  uint4 pk;
  __nv_bfloat162* p2 = reinterpret_cast<__nv_bfloat162*>(&pk);
#pragma unroll
  for (int q = 0; q < 4; ++q) p2[q] = __floats2bfloat162_rn(v[2 * q], v[2 * q + 1]);
  return pk;
}
// address of the 16-byte unit (row, kb) of a blocked activation with F features
__device__ __forceinline__ uint4* blk_unit(__nv_bfloat16* base, int F, int row, int kb) {
  return reinterpret_cast<uint4*>(base + (size_t)(row / ACT_R) * F * ACT_R + ((size_t)kb * ACT_R + row % ACT_R) * 8);
}

// positional encodings (time_utils.py:8-55): [v, sin(v 2^0), cos(v 2^0), ..., sin(v 2^(L-1)), cos(v 2^(L-1))]
// One thread per row (padding rows get zeros); writes the x block (+ direct time features) of A5 and T0.
// residuals of pack8(v): lo[i] = bf16(v[i] - float(bf16(v[i])))
__device__ __forceinline__ uint4 pack8_lo(const float* v) {
  float r[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) r[i] = v[i] - __bfloat162float(__float2bfloat16_rn(v[i]));
  return pack8(r);
}

__global__ void __launch_bounds__(256) pe_kernel(int P, int Pp, const float* __restrict__ x,
                                                 const float* __restrict__ t, int has_timenet, int t_freqs,
                                                 __nv_bfloat16* __restrict__ A5, __nv_bfloat16* __restrict__ T0,
                                                 __nv_bfloat16* __restrict__ A5lo, __nv_bfloat16* __restrict__ T0lo) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= Pp) return;
  const bool ok = p < P;
  float e[K0];
#pragma unroll
  for (int i = 0; i < K0; ++i) e[i] = 0.f;
  float te[24];
#pragma unroll
  for (int i = 0; i < 24; ++i) te[i] = 0.f;
  if (ok) {
    const float v[3] = {x[3 * p], x[3 * p + 1], x[3 * p + 2]};
#pragma unroll
    for (int c = 0; c < 3; ++c) e[c] = v[c];
#pragma unroll
    for (int f = 0; f < 10; ++f) {
      const float fr = (float)(1 << f);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float s, co;
        sincosf(v[c] * fr, &s, &co);
        e[3 + 6 * f + c] = s;
        e[3 + 6 * f + 3 + c] = co;
      }
    }
    const float tv = t[p];
    te[0] = tv;
    for (int f = 0; f < t_freqs; ++f) {
      float s, co;
      sincosf(tv * (float)(1 << f), &s, &co);
      te[1 + 2 * f] = s;
      te[2 + 2 * f] = co;
    }
    if (!has_timenet) {
#pragma unroll
      for (int i = 0; i < 21; ++i) e[TCOL + i] = te[i];
    }
  }
  const int nkb = has_timenet ? TCOL / 8 : K0 / 8;  // with a timenet its GEMM writes kbs 8..11
#pragma unroll
  for (int kb = 0; kb < K0 / 8; ++kb)
    if (kb < nkb) {
      *blk_unit(A5, K5, p, kb) = pack8(e + 8 * kb);
      if (A5lo) *blk_unit(A5lo, K5, p, kb) = pack8_lo(e + 8 * kb);
    }
  if (has_timenet) {
    *blk_unit(T0, 16, p, 0) = pack8(te);
    *blk_unit(T0, 16, p, 1) = pack8(te + 8);
    if (T0lo) {
      *blk_unit(T0lo, 16, p, 0) = pack8_lo(te);
      *blk_unit(T0lo, 16, p, 1) = pack8_lo(te + 8);
    }
  }
}

// gradient of the heads' pre-activation: dZh = g (* y (1 - y) for the sigmoid colour head), blocked [Pp,16]
__global__ void __launch_bounds__(256) head_grad_kernel(int P, int Pp, int n_out, int sigmoid,
                                                        const float* __restrict__ g, const float* __restrict__ y,
                                                        __nv_bfloat16* __restrict__ dZh) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= Pp) return;
  float v[16];
#pragma unroll
  for (int o = 0; o < 16; ++o) {
    float w = 0.f;
    if (p < P && o < n_out) {
      w = g[(size_t)p * 16 + o];
      if (sigmoid) {
        const float yy = y[(size_t)p * 16 + o];
        w *= yy * (1.f - yy);
      }
    }
    v[o] = w;
  }
  *blk_unit(dZh, 16, p, 0) = pack8(v);
  *blk_unit(dZh, 16, p, 1) = pack8(v + 8);
}

__global__ void __launch_bounds__(256) sigmoid_kernel(int n, float* __restrict__ y) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = 1.f / (1.f + expf(-y[i]));
}

// dE[:, 64:96] (fp32 row-major) -> dZt1 blocked [Pp, 32] (features >= n_t are zero)
__global__ void __launch_bounds__(256) tfeat_grad_kernel(int Pp, int n_t, const int* __restrict__ tu,
                                                         const float* __restrict__ dE,
                                                         __nv_bfloat16* __restrict__ dZ) {
  if (tu[0]) return;  // uniform time: tfeat_colsum / tfeat_row0 produce the single row that matters
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= Pp) return;
  float v[32];
#pragma unroll
  for (int o = 0; o < 32; ++o) v[o] = (o < n_t) ? dE[(size_t)p * K0 + TCOL + o] : 0.f;
#pragma unroll
  for (int kb = 0; kb < 4; ++kb) *blk_unit(dZ, 32, p, kb) = pack8(v + 8 * kb);
}

// dx = dE . d pe(x) / dx
__global__ void __launch_bounds__(256) pe_backward_kernel(int P, const float* __restrict__ x,
                                                          const float* __restrict__ dE, float* __restrict__ dx) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const float* g = dE + (size_t)p * K0;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v = x[3 * p + c];
    float acc = g[c];
#pragma unroll
    for (int f = 0; f < 10; ++f) {
      const float fr = (float)(1 << f);
      float s, co;
      sincosf(v * fr, &s, &co);
      acc += fr * (g[3 + 6 * f + c] * co - g[3 + 6 * f + 3 + c] * s);
    }
    dx[3 * p + c] = acc;
  }
}

// ---- uniform time: DG-Mesh evaluates a network at ONE time for all points of a frame (train.py:158-172:
// fid.expand(N, -1), plus at most one shared noise scalar).  The time-net (t -> 256 -> 30 features) then produces
// the same row N times: ~8 % of an MLP evaluation at 200k points, all of it HBM traffic.  The decision is made on
// the device (no host read, exact in both cases): when every t equals t[0] the time-net kernels process tile 0
// only and the 30 features are broadcast to all rows; in the backward the rows' feature gradients are summed
// into row 0 first (the time-net is shared, so the sum of per-row backward passes is the backward of the sum).
__global__ void __launch_bounds__(1024) t_uniform_kernel(int P, int tiles, const float* __restrict__ t,
                                                         int* __restrict__ tu, float* __restrict__ tsum) {
  const uint32_t t0 = __float_as_uint(t[0]);
  int diff = 0;
  for (int p = threadIdx.x; p < P; p += blockDim.x) diff |= (__float_as_uint(t[p]) != t0);
  diff = __syncthreads_or(diff);
  if (threadIdx.x == 0) {
    tu[0] = diff ? 0 : 1;
    tu[1] = diff ? tiles : 1;
  }
  if (threadIdx.x < 32) tsum[threadIdx.x] = 0.f;
}

// time features of row 0 (A5 k-blocks TCOL/8 .. +3, hi and lo) -> every other row
__global__ void __launch_bounds__(256) tfeat_broadcast_kernel(int Pp, const int* __restrict__ tu,
                                                              __nv_bfloat16* __restrict__ A5,
                                                              __nv_bfloat16* __restrict__ A5lo) {
  if (!tu[0]) return;
  const int p = blockIdx.x * blockDim.x + threadIdx.x + 1;
  if (p >= Pp) return;
#pragma unroll
  for (int kb = TCOL / 8; kb < K0 / 8; ++kb) {
    *blk_unit(A5, K5, p, kb) = *blk_unit(A5, K5, 0, kb);
    if (A5lo) *blk_unit(A5lo, K5, p, kb) = *blk_unit(A5lo, K5, 0, kb);
  }
}

// uniform time, backward: tsum[o] += sum over rows of dE[:, TCOL + o]
__global__ void __launch_bounds__(256) tfeat_colsum_kernel(int Pp, int n_t, const int* __restrict__ tu,
                                                           const float* __restrict__ dE, float* __restrict__ tsum) {
  if (!tu[0]) return;
  __shared__ float s_part[8][32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  // a warp reads 32 consecutive time-feature gradients of one row per step (coalesced 128 B)
  float acc = 0.f;
  for (int p = blockIdx.x * 8 + wid; p < Pp; p += gridDim.x * 8)
    if (lane < n_t) acc += dE[(size_t)p * K0 + TCOL + lane];
  s_part[wid][lane] = acc;
  __syncthreads();
  if (wid == 0) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) v += s_part[w][lane];
    if (lane < n_t) atomicAdd(&tsum[lane], v);
  }
}
// uniform time, backward: tile 0 of dZt1 = [tsum; 0; 0; ...]
__global__ void __launch_bounds__(ACT_R) tfeat_row0_kernel(const int* __restrict__ tu, const float* __restrict__ tsum,
                                                           __nv_bfloat16* __restrict__ dZ) {
  if (!tu[0]) return;
  const int p = threadIdx.x;
  float v[32];
#pragma unroll
  for (int o = 0; o < 32; ++o) v[o] = (p == 0) ? tsum[o] : 0.f;
#pragma unroll
  for (int kb = 0; kb < 4; ++kb) *blk_unit(dZ, 32, p, kb) = pack8(v + 8 * kb);
}

#define CK(call)                      \
  do {                                \
    cudaError_t e_ = (call);          \
    if (e_ != cudaSuccess) return e_; \
  } while (0)

typedef const __nv_bfloat16* CB;

static LayerArgs layer(const BlkView& A, int K, CB B, int N, int tiles) {
  LayerArgs g = {};
  g.A = A; g.K = K; g.B = B; g.N = N; g.tiles = tiles;
  return g;
}

cudaError_t launch_mlp_forward(const DglNet& n, int P, const float* x, const float* t, float* out, int train,
                               void* ws, cudaStream_t s) {
  MlpBufs b = MlpBufs::carve_all((char*)ws, P, train, nullptr);
  const int Pp = b.Pp, tiles = b.tiles;
  const bool hp = n.precise != 0;  // split-precision forward (bf16x3)
  pe_kernel<<<(Pp + 255) / 256, 256, 0, s>>>(P, Pp, x, t, n.has_timenet, n.has_timenet ? 6 : 10, b.A5, b.T0,
                                             hp ? b.A5lo : nullptr, hp ? b.T0lo : nullptr);
  if (n.has_timenet) {
    t_uniform_kernel<<<1, 1024, 0, s>>>(P, tiles, t, b.tu, b.tsum);
    LayerArgs g = layer(BlkView{b.T0, (size_t)16 * ACT_R, 0}, 16, (CB)n.Wt0, WID, tiles);
    g.tiles_dev = b.tu + 1;  // tile 0 only when every row has the same t
    g.bias = n.bt0; g.relu = 1; g.out = b.T1; g.out_tile_stride = (size_t)WID * ACT_R;
    g.mask_out = b.Mt1;
    if (hp) { g.A_lo = b.T0lo; g.B_lo = (CB)n.Wt0lo; g.out_lo = b.T1lo; }
    CK(launch_layer_gemm(g, s));
    g = layer(BlkView{b.T1, (size_t)WID * ACT_R, 0}, WID, (CB)n.Wt1, 32, tiles);  // 30 outputs padded to 32
    g.tiles_dev = b.tu + 1;
    g.bias = n.bt1; g.out = b.A5; g.out_tile_stride = (size_t)K5 * ACT_R; g.out_kb0 = TCOL / 8;
    if (hp) { g.A_lo = b.T1lo; g.B_lo = (CB)n.Wt1lo; g.out_lo = b.A5lo; }
    CK(launch_layer_gemm(g, s));
    tfeat_broadcast_kernel<<<(Pp + 255) / 256, 256, 0, s>>>(Pp, b.tu, b.A5, hp ? b.A5lo : nullptr);
  }
  for (int l = 0; l < 8; ++l) {
    const BlkView A = (l == 0 || l == 5) ? b.a5() : b.h(l - 1);
    const int K = (l == 0) ? K0 : (l == 5 ? K5 : WID);
    LayerArgs g = layer(A, K, (CB)n.W[l], WID, tiles);
    g.bias = n.b[l]; g.relu = 1;
    const BlkView o = b.h(l);
    g.out = const_cast<__nv_bfloat16*>(o.p); g.out_tile_stride = o.tile_stride; g.out_kb0 = o.kb0;
    g.mask_out = b.M[l];
    if (hp) {
      g.A_lo = (l == 0 || l == 5) ? b.A5lo : b.hlo(l - 1);
      g.B_lo = (CB)n.Wlo[l];
      g.out_lo = b.hlo(l);
    }
    CK(launch_layer_gemm(g, s));
  }
  LayerArgs g = layer(b.h(7), WID, (CB)n.Wh, 16, tiles);
  g.bias = n.bh; g.out_f32 = out; g.ld_f32 = 16; g.n_f32 = 16; g.rows_valid = P;
  if (hp) { g.A_lo = b.hlo(7); g.B_lo = (CB)n.Whlo; }
  CK(launch_layer_gemm(g, s));
  if (n.sigmoid_out) sigmoid_kernel<<<(P * 16 + 255) / 256, 256, 0, s>>>(P * 16, out);
  return cudaGetLastError();
}

// weight gradient C[256 (X features), N (Y features)] (+)= X^T Y, or its transpose
static cudaError_t dw(const BlkView& X, const BlkView& Y, int N, int tiles, float* C, int ld, int transpose,
                      cudaStream_t s, float* colsum_x = nullptr, float* colsum_y = nullptr,
                      const int* tiles_dev = nullptr) {
  DwArgs g = {};
  g.X = X; g.Y = Y; g.N = N; g.tiles = tiles; g.tiles_dev = tiles_dev; g.C = C; g.ld = ld; g.transpose = transpose;
  g.m_valid = WID; g.n_valid = N;
  g.colsum_x = colsum_x; g.colsum_y = colsum_y;  // bias gradients ride along (no separate column-sum pass)
  return launch_dw_gemm(g, s);
}

bool grads_are_packed(const DglGrads& g);
size_t packed_grad_total_bytes();

cudaError_t launch_mlp_backward(const DglNet& n, int P, const float* x, const float* out, const float* g_out,
                                void* ws, const DglGrads& gr, float* dx, cudaStream_t s) {
  MlpBufs b = MlpBufs::carve_all((char*)ws, P, 1, nullptr);
  const int Pp = b.Pp, tiles = b.tiles;
  const size_t HS = (size_t)WID * ACT_R;  // tile stride of a 256-feature activation
  cudaMemsetAsync(b.dE, 0, sizeof(float) * (size_t)Pp * K0, s);
  if (grads_are_packed(gr)) {
    // the usual case (dgl_mlp_grad_pointers): one contiguous buffer, one memset
    cudaMemsetAsync(gr.dW[0], 0, packed_grad_total_bytes(), s);
  } else {
    for (int l = 0; l < 8; ++l) {
      const int K = (l == 0) ? K0 : (l == 5 ? K5 : WID);
      cudaMemsetAsync(gr.dW[l], 0, sizeof(float) * WID * K, s);
      cudaMemsetAsync(gr.db[l], 0, sizeof(float) * WID, s);
    }
    cudaMemsetAsync(gr.dWh, 0, sizeof(float) * 16 * WID, s);
    cudaMemsetAsync(gr.dbh, 0, sizeof(float) * 16, s);
    if (n.has_timenet) {
      cudaMemsetAsync(gr.dWt0, 0, sizeof(float) * WID * 16, s);
      cudaMemsetAsync(gr.dbt0, 0, sizeof(float) * WID, s);
      cudaMemsetAsync(gr.dWt1, 0, sizeof(float) * 32 * WID, s);
      cudaMemsetAsync(gr.dbt1, 0, sizeof(float) * 32, s);
    }
  }
  // heads: dWh[16,256] = dZh^T . H7 (computed transposed: X = H7), dbh, dZ7 = (dZh . Wh) * relu'(H7)
  const BlkView vZh{b.dZh, (size_t)16 * ACT_R, 0};
  head_grad_kernel<<<(Pp + 255) / 256, 256, 0, s>>>(P, Pp, n.n_out, n.sigmoid_out, g_out, out, b.dZh);
  CK(dw(b.h(7), vZh, 16, tiles, gr.dWh, WID, 1, s, nullptr, gr.dbh));
  int cur = 0;
  {
    LayerArgs g = layer(vZh, 16, (CB)n.WhT, WID, tiles);
    g.mask_bits = b.M[7];
    g.out = b.dZ[cur]; g.out_tile_stride = HS;
    CK(launch_layer_gemm(g, s));
  }
  for (int l = 7; l >= 0; --l) {
    // dZ[cur] = dL/d(pre-activation of layer l)
    const BlkView vZ{b.dZ[cur], HS, 0};
    if (l == 0 || l == 5) {
      CK(dw(vZ, b.a5(), K0, tiles, gr.dW[l], (l == 0) ? K0 : K5, 0, s, gr.db[l]));  // columns of [x_emb, t]; db[l]
      if (l == 5) CK(dw(vZ, b.h(4), WID, tiles, gr.dW[l] + K0, K5, 0, s));          // columns of h4
    } else {
      CK(dw(vZ, b.h(l - 1), WID, tiles, gr.dW[l], WID, 0, s, gr.db[l]));
    }
    if (l == 0 || l == 5) {  // gradient w.r.t. the embedded inputs (no ReLU in front of them)
      const CB We = (l == 0) ? (CB)n.WT[0] : (CB)n.WT[5] + (size_t)WID * WID;  // [256/8][96][8]
      LayerArgs g = layer(vZ, WID, We, K0, tiles);
      g.out_f32 = b.dE; g.ld_f32 = K0; g.n_f32 = K0; g.atomic = 1; g.rows_valid = Pp;
      CK(launch_layer_gemm(g, s));
    }
    if (l > 0) {
      LayerArgs g = layer(vZ, WID, (CB)n.WT[l], WID, tiles);  // for l == 5 the h4 part comes first
      g.mask_bits = b.M[l - 1];
      g.out = b.dZ[cur ^ 1]; g.out_tile_stride = HS;
      CK(launch_layer_gemm(g, s));
      cur ^= 1;
    }
  }
  if (n.has_timenet) {
    const BlkView vT1{b.T1, HS, 0}, vZt1{b.dZt1, (size_t)32 * ACT_R, 0};
    // per-row feature gradients, or (uniform time, flag on the device) their column sums in row 0 of tile 0
    cudaMemsetAsync(b.tsum, 0, 32 * sizeof(float), s);
    tfeat_grad_kernel<<<(Pp + 255) / 256, 256, 0, s>>>(Pp, n.in_t, b.tu, b.dE, b.dZt1);
    tfeat_colsum_kernel<<<min(4 * sm_count(), (Pp + 7) / 8), 256, 0, s>>>(Pp, n.in_t, b.tu, b.dE, b.tsum);
    tfeat_row0_kernel<<<1, ACT_R, 0, s>>>(b.tu, b.tsum, b.dZt1);
    const int* td = b.tu + 1;
    CK(dw(vT1, vZt1, 32, tiles, gr.dWt1, WID, 1, s, nullptr, gr.dbt1, td));  // dWt1[32,256] = dZt1^T . T1 (transposed form)
    LayerArgs g = layer(vZt1, 32, (CB)n.Wt1T, WID, tiles);
    g.tiles_dev = td;
    g.mask_bits = b.Mt1;
    g.out = b.dZ[cur ^ 1]; g.out_tile_stride = HS;
    CK(launch_layer_gemm(g, s));
    CK(dw(BlkView{b.dZ[cur ^ 1], HS, 0}, BlkView{b.T0, (size_t)16 * ACT_R, 0}, 16, tiles, gr.dWt0, 16, 0, s,
          gr.dbt0, nullptr, td));
  }
  if (dx) pe_backward_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, x, b.dE, dx);
  return cudaGetLastError();
}

size_t mlp_workspace_bytes(int P, int train) {
  size_t bytes;
  MlpBufs::carve_all(nullptr, P, train, &bytes);
  return bytes;
}

// ------------------------------------------------------------------ stand-alone GEMM entry points (tests)
// row-major bf16 [rows, ld] (cols valid) -> blocked with R-row tiles and Fp features (zero padded)
__global__ void rm_to_blk_kernel(const __nv_bfloat16* __restrict__ src, int rows, int cols, int ld, int R, int Fp,
                                 int rows_pad, __nv_bfloat16* __restrict__ dst) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)rows_pad * Fp) return;
  const int row = (int)(i / Fp), f = (int)(i % Fp);
  const __nv_bfloat16 v = (row < rows && f < cols) ? src[(size_t)row * ld + f] : __float2bfloat16_rn(0.f);
  dst[(size_t)(row / R) * Fp * R + ((size_t)(f >> 3) * R + row % R) * 8 + (f & 7)] = v;
}

size_t gemm_test_ws_bytes(int M, int N, int K) {
  const size_t Mp = ((size_t)M + ACT_R - 1) / ACT_R * ACT_R, Np = ((size_t)N + 15) / 16 * 16,
               Kp = ((size_t)K + 15) / 16 * 16;
  return (Mp * Kp + Np * Kp + Mp * 256 + Mp * Np) * 2 + 1024;
}

// C[M,N] = A[M,K] . B[N,K]^T through layer_gemm_kernel
cudaError_t launch_gemm_test(int M, int N, int K, const void* A, int lda, const void* B, int ldb, const float* bias,
                             int relu, float* C, int ldc, void* ws, cudaStream_t s) {
  const int Mp = (M + ACT_R - 1) / ACT_R * ACT_R, Np = (N + 15) / 16 * 16, Kp = (K + 15) / 16 * 16;
  char* p = (char*)ws;
  __nv_bfloat16* Ab = carve<__nv_bfloat16>(p, (size_t)Mp * Kp);
  __nv_bfloat16* Bb = carve<__nv_bfloat16>(p, (size_t)Np * Kp);
  rm_to_blk_kernel<<<(unsigned)(((size_t)Mp * Kp + 255) / 256), 256, 0, s>>>((CB)A, M, K, lda, ACT_R, Kp, Mp, Ab);
  rm_to_blk_kernel<<<(unsigned)(((size_t)Np * Kp + 255) / 256), 256, 0, s>>>((CB)B, N, K, ldb, Np, Kp, Np, Bb);
  LayerArgs g = layer(BlkView{Ab, (size_t)Kp * ACT_R, 0}, Kp, Bb, Np, Mp / ACT_R);
  g.bias = bias; g.relu = relu;
  g.out_f32 = C; g.ld_f32 = ldc; g.n_f32 = N; g.rows_valid = M;
  // the bias vector has N entries; the kernel reads bias[i] for i < g.N = Np: guard with a padded copy
  if (bias && Np != N) {
    float* bp = carve<float>(p, 256);
    cudaMemsetAsync(bp, 0, 256 * sizeof(float), s);
    cudaMemcpyAsync(bp, bias, sizeof(float) * N, cudaMemcpyDeviceToDevice, s);
    g.bias = bp;
  }
  return launch_layer_gemm(g, s);
}

// C[Mf,Nf] (+)= X[P,Mf]^T . Y[P,Nf] through dw_gemm_kernel (Mf <= 256, Nf <= 256)
cudaError_t launch_gemm_tn_test(int P, int Mf, int Nf, const void* X, int ldx, const void* Y, int ldy, float* C,
                                int ldc, int transpose, void* ws, cudaStream_t s) {
  const int Pp = (P + ACT_R - 1) / ACT_R * ACT_R, Np = (Nf + 15) / 16 * 16;
  char* p = (char*)ws;
  __nv_bfloat16* Xb = carve<__nv_bfloat16>(p, (size_t)Pp * 256);
  __nv_bfloat16* Yb = carve<__nv_bfloat16>(p, (size_t)Pp * Np);
  rm_to_blk_kernel<<<(unsigned)(((size_t)Pp * 256 + 255) / 256), 256, 0, s>>>((CB)X, P, Mf, ldx, ACT_R, 256, Pp, Xb);
  rm_to_blk_kernel<<<(unsigned)(((size_t)Pp * Np + 255) / 256), 256, 0, s>>>((CB)Y, P, Nf, ldy, ACT_R, Np, Pp, Yb);
  DwArgs g = {};
  g.X = BlkView{Xb, (size_t)256 * ACT_R, 0};
  g.Y = BlkView{Yb, (size_t)Np * ACT_R, 0};
  g.N = Np; g.tiles = Pp / ACT_R; g.C = C; g.ld = ldc; g.transpose = transpose;
  g.m_valid = Mf; g.n_valid = transpose ? Nf : (Nf + 3) / 4 * 4;
  return launch_dw_gemm(g, s);
}

}  // namespace dgm

// =====================================================================================
// Parameter packing: reference-shaped fp32 parameters (nn.Linear weights [out, in]) -> the blocked
// bf16 operands of DglNet, and packed fp32 gradients -> reference-shaped gradients.
// Column map of an input-facing matrix: c < 63 -> c ; 63 <= c < 63+in_t -> c + 1 ; beyond (the
// hidden part of the skip layer) -> 96 + (c - 63 - in_t).
// =====================================================================================
namespace dgm {

__device__ __forceinline__ int map_col(int c, int in_t, int mapped) {
  if (!mapped) return c;
  if (c < XE) return c;
  if (c < XE + in_t) return c + 1;
  return K0 + (c - XE - in_t);
}

// One table-driven launch packs (or unpacks) every matrix and bias of a network.
// Weight entry: src fp32 [rows, kin] (nn.Linear layout [out, in]) -> blocked bf16 operands (mlp_gemm.cuh):
//   forward  B operand  dst : single tile of Rf rows (outputs), element (o, k) at ((k/8)*Rf + o)*8 + k%8
//   backward B operand  dstT: rows = inputs j, contraction index = outputs o:
//            element (j, o) at ((o/8)*Rt + j)*8 + o%8.  For the input-facing layers the input columns
//            split into the [x_emb, t] block (j < 96, Rt = 96, at dstT_e) and the hidden block
//            (j >= 96 -> j - 96, Rt = 256, at dstT).
struct PackEntry {
  const float* src;          // pack: raw weight / bias;  unpack: packed fp32 gradient
  float* dst_f32;            // bias copy / unpacked gradient
  __nv_bfloat16 *dst, *dstT, *dstT_e;
  __nv_bfloat16* dst_lo;     // forward operand of the split-precision path: bf16(w - float(bf16(w)))
  int rows, kin, mapped, r0, Rf, Rt, kpad, is_bias;
};
#define PACK_MAX 32
struct PackTable {
  PackEntry e[PACK_MAX];
  int n, in_t;
};

__global__ void __launch_bounds__(256) pack_all_kernel(const PackTable t) {
  const PackEntry& E = t.e[blockIdx.y];
  const int total = E.rows * E.kin;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    if (E.is_bias) {
      E.dst_f32[i] = E.src[i];
      continue;
    }
    const int r = i / E.kin, c = i % E.kin;
    const int cc = map_col(c, t.in_t, E.mapped), o = E.r0 + r;
    const __nv_bfloat16 v = __float2bfloat16_rn(E.src[i]);
    E.dst[((size_t)(cc >> 3) * E.Rf + o) * 8 + (cc & 7)] = v;
    if (E.dst_lo)
      E.dst_lo[((size_t)(cc >> 3) * E.Rf + o) * 8 + (cc & 7)] = __float2bfloat16_rn(E.src[i] - __bfloat162float(v));
    if (E.mapped) {
      if (cc < K0) {
        if (E.dstT_e) E.dstT_e[((size_t)(o >> 3) * K0 + cc) * 8 + (o & 7)] = v;
      } else if (E.dstT) {
        E.dstT[((size_t)(o >> 3) * WID + (cc - K0)) * 8 + (o & 7)] = v;
      }
    } else if (E.dstT) {
      E.dstT[((size_t)(o >> 3) * E.Rt + cc) * 8 + (o & 7)] = v;
    }
  }
}
// packed fp32 gradients (row-major [*, kpad], row offset r0) -> reference-shaped [rows, kin]; biases copied
__global__ void __launch_bounds__(256) unpack_all_kernel(const PackTable t) {
  const PackEntry& E = t.e[blockIdx.y];
  const int total = E.rows * E.kin;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    if (E.is_bias) {
      E.dst_f32[i] = E.src[i];
      continue;
    }
    const int r = i / E.kin, c = i % E.kin;
    E.dst_f32[i] = E.src[(size_t)(E.r0 + r) * E.kpad + map_col(c, t.in_t, E.mapped)];
  }
}

// fixed layout of the packed buffers (elements)
struct PackLayout {
  size_t W[8], WT[8], Wh, WhT, Wt0, Wt1, Wt1T, w_total;  // bf16 elements
  size_t Wlo[8], Whlo, Wt0lo, Wt1lo;                      // residual forward operands (split precision)
  size_t b[8], bh, bt0, bt1, b_total;                     // fp32 elements
  // gradient buffer (fp32 elements): same matrices, no transposes
  size_t gW[8], gb[8], gWh, gbh, gWt0, gbt0, gWt1, gbt1, g_total;
  PackLayout() {
    size_t o = 0;
    auto take = [&](size_t n) { size_t r = o; o += (n + 63) / 64 * 64; return r; };
    for (int l = 0; l < 8; ++l) {
      const size_t K = (l == 0) ? K0 : (l == 5 ? K5 : WID);
      W[l] = take(WID * K);
      WT[l] = take(WID * K);
    }
    Wh = take(16 * WID); WhT = take(16 * WID);
    Wt0 = take(WID * 16); Wt1 = take(32 * WID); Wt1T = take(32 * WID);
    for (int l = 0; l < 8; ++l) Wlo[l] = take(WID * ((l == 0) ? K0 : (l == 5 ? K5 : WID)));
    Whlo = take(16 * WID); Wt0lo = take(WID * 16); Wt1lo = take(32 * WID);
    w_total = o;
    o = 0;
    for (int l = 0; l < 8; ++l) b[l] = take(WID);
    bh = take(16); bt0 = take(WID); bt1 = take(32);
    b_total = o;
    o = 0;
    for (int l = 0; l < 8; ++l) {
      const size_t K = (l == 0) ? K0 : (l == 5 ? K5 : WID);
      gW[l] = take(WID * K);
      gb[l] = take(WID);
    }
    gWh = take(16 * WID); gbh = take(16); gWt0 = take(WID * 16); gbt0 = take(WID); gWt1 = take(32 * WID);
    gbt1 = take(32);
    g_total = o;
  }
};
static const PackLayout& layout() {
  static PackLayout L;
  return L;
}

void mlp_pack_sizes(size_t* w_bytes, size_t* b_bytes, size_t* g_bytes) {
  const PackLayout& L = layout();
  if (w_bytes) *w_bytes = L.w_total * 2;
  if (b_bytes) *b_bytes = L.b_total * 4;
  if (g_bytes) *g_bytes = L.g_total * 4;
}

static int in_width(const DglRaw& r) { return XE + r.in_t; }

cudaError_t launch_mlp_pack(const DglRaw& r, void* wbuf, float* bbuf, DglNet* net, cudaStream_t s) {
  const PackLayout& L = layout();
  __nv_bfloat16* w = (__nv_bfloat16*)wbuf;
  cudaMemsetAsync(wbuf, 0, L.w_total * 2, s);
  cudaMemsetAsync(bbuf, 0, L.b_total * 4, s);
  net->has_timenet = r.has_timenet; net->in_t = r.in_t; net->sigmoid_out = r.sigmoid_out;
  const size_t NONE = (size_t)-1;
  auto at = [&](size_t off) { return off == NONE ? (__nv_bfloat16*)nullptr : w + off; };
  PackTable T = {};
  T.in_t = r.in_t;
  auto pack = [&](const float* src, int rows, int kin, int mapped, int r0, int Rf, size_t dst, size_t dstT, int Rt,
                  size_t dstT_e, size_t dst_lo) {
    PackEntry& E = T.e[T.n++];
    E.src = src; E.rows = rows; E.kin = kin; E.mapped = mapped; E.r0 = r0; E.Rf = Rf;
    E.dst = w + dst; E.dstT = at(dstT); E.Rt = Rt; E.dstT_e = at(dstT_e); E.dst_lo = w + dst_lo;
  };
  auto bias = [&](const float* src, int n_el, float* dst) {
    PackEntry& E = T.e[T.n++];
    E.src = src; E.rows = 1; E.kin = n_el; E.dst_f32 = dst; E.is_bias = 1;
  };
  for (int l = 0; l < 8; ++l) {
    const int kin = (l == 0) ? in_width(r) : (l == 5 ? in_width(r) + WID : WID);
    // WT[0] holds only the [x_emb, t] block; WT[5] the hidden block followed by the [x_emb, t] block
    if (l == 0) pack(r.W[l], WID, kin, 1, 0, WID, L.W[l], NONE, 0, L.WT[l], L.Wlo[l]);
    else if (l == 5) pack(r.W[l], WID, kin, 1, 0, WID, L.W[l], L.WT[l], WID, L.WT[l] + (size_t)WID * WID, L.Wlo[l]);
    else pack(r.W[l], WID, kin, 0, 0, WID, L.W[l], L.WT[l], WID, NONE, L.Wlo[l]);
    bias(r.b[l], WID, bbuf + L.b[l]);
    net->W[l] = w + L.W[l]; net->WT[l] = w + L.WT[l]; net->b[l] = bbuf + L.b[l];
    net->Wlo[l] = w + L.Wlo[l];
  }
  int r0 = 0;
  for (int h = 0; h < r.n_heads; ++h) {
    pack(r.Wh[h], r.head_rows[h], WID, 0, r0, 16, L.Wh, L.WhT, WID, NONE, L.Whlo);
    bias(r.bh[h], r.head_rows[h], bbuf + L.bh + r0);
    r0 += r.head_rows[h];
  }
  net->n_out = r0;
  net->Wh = w + L.Wh; net->WhT = w + L.WhT; net->bh = bbuf + L.bh;
  net->Whlo = w + L.Whlo; net->Wt0lo = w + L.Wt0lo; net->Wt1lo = w + L.Wt1lo;
  net->precise = 1;  // the caller may clear it to run the single-pass bf16 forward
  if (r.has_timenet) {
    pack(r.Wt0, WID, 13, 0, 0, WID, L.Wt0, NONE, 0, NONE, L.Wt0lo);
    pack(r.Wt1, r.in_t, WID, 0, 0, 32, L.Wt1, L.Wt1T, WID, NONE, L.Wt1lo);
    bias(r.bt0, WID, bbuf + L.bt0);
    bias(r.bt1, r.in_t, bbuf + L.bt1);
    net->Wt0 = w + L.Wt0; net->Wt1 = w + L.Wt1; net->Wt1T = w + L.Wt1T;
    net->bt0 = bbuf + L.bt0; net->bt1 = bbuf + L.bt1;
  } else {
    net->Wt0 = net->Wt1 = net->Wt1T = nullptr;
    net->bt0 = net->bt1 = nullptr;
  }
  pack_all_kernel<<<dim3(32, T.n), 256, 0, s>>>(T);
  return cudaGetLastError();
}

size_t packed_grad_total_bytes() { return layout().g_total * sizeof(float); }

// true when `g` is the pointer table of ONE packed buffer starting at g.dW[0]
bool grads_are_packed(const DglGrads& g) {
  const PackLayout& L = layout();
  if (L.gW[0] != 0 || !g.dW[0]) return false;
  float* base = g.dW[0];
  for (int l = 0; l < 8; ++l)
    if (g.dW[l] != base + L.gW[l] || g.db[l] != base + L.gb[l]) return false;
  return g.dWh == base + L.gWh && g.dbh == base + L.gbh && g.dWt0 == base + L.gWt0 && g.dbt0 == base + L.gbt0 &&
         g.dWt1 == base + L.gWt1 && g.dbt1 == base + L.gbt1;
}

void mlp_grad_pointers(float* gbuf, DglGrads* g) {
  const PackLayout& L = layout();
  for (int l = 0; l < 8; ++l) {
    g->dW[l] = gbuf + L.gW[l];
    g->db[l] = gbuf + L.gb[l];
  }
  g->dWh = gbuf + L.gWh; g->dbh = gbuf + L.gbh;
  g->dWt0 = gbuf + L.gWt0; g->dbt0 = gbuf + L.gbt0; g->dWt1 = gbuf + L.gWt1; g->dbt1 = gbuf + L.gbt1;
}

// packed gradients -> tensors shaped like the reference parameters (DglRawGrads mirrors DglRaw)
cudaError_t launch_mlp_unpack_grads(const DglRaw& r, const float* gbuf, const DglRawGrads& o, cudaStream_t s) {
  const PackLayout& L = layout();
  PackTable T = {};
  T.in_t = r.in_t;
  auto unpack = [&](size_t src, int kpad, int r0, int rows, int kin, int mapped, float* dst) {
    PackEntry& E = T.e[T.n++];
    E.src = gbuf + src; E.kpad = kpad; E.r0 = r0; E.rows = rows; E.kin = kin; E.mapped = mapped; E.dst_f32 = dst;
  };
  auto bias = [&](size_t src, int n_el, float* dst) {
    PackEntry& E = T.e[T.n++];
    E.src = gbuf + src; E.rows = 1; E.kin = n_el; E.dst_f32 = dst; E.is_bias = 1;
  };
  for (int l = 0; l < 8; ++l) {
    const int kin = (l == 0) ? in_width(r) : (l == 5 ? in_width(r) + WID : WID);
    const int kpad = (l == 0) ? K0 : (l == 5 ? K5 : WID);
    unpack(L.gW[l], kpad, 0, WID, kin, l == 0 || l == 5, o.W[l]);
    bias(L.gb[l], WID, o.b[l]);
  }
  int r0 = 0;
  for (int h = 0; h < r.n_heads; ++h) {
    unpack(L.gWh, WID, r0, r.head_rows[h], WID, 0, o.Wh[h]);
    bias(L.gbh + r0, r.head_rows[h], o.bh[h]);
    r0 += r.head_rows[h];
  }
  if (r.has_timenet) {
    unpack(L.gWt0, 16, 0, WID, 13, 0, o.Wt0);
    unpack(L.gWt1, WID, 0, r.in_t, WID, 0, o.Wt1);
    bias(L.gbt0, WID, o.bt0);
    bias(L.gbt1, r.in_t, o.bt1);
  }
  unpack_all_kernel<<<dim3(32, T.n), 256, 0, s>>>(T);
  return cudaGetLastError();
}

}  // namespace dgm
