// hashgrid.cu -- the multiresolution hash encoding of (x, y, z, t) (Instant-NGP's HashGrid on x, y, z and Grid4D's
// space-time grids on (x, y, t), (y, z, t), (x, z, t)), forward and backward (include/dgmesh_b200.h "dghg_" states
// the definition).
//
//   * Layout: grid g's table is channels-last [L, T, Fe], so a corner is one float2 (Fe = 2) or float4 (Fe = 4) load.
//   * Thread mapping: one thread per (point, level), Lp lanes a point (Lp the power of two >= L, so a point's lanes
//     sit in one warp).  A thread takes its level of every grid: the spatial grid once for the whole batch (its
//     features written into every frame's output), each time grid once per frame.  The 8 corner slots are computed
//     first and the 8 loads issued together before any is used: the gather is latency-bound.
//   * Backward, x: each thread sums its level's terms over the grids in order and the frames in frame order (the
//     spatial grid takes the frames' grad_out summed in frame order), and a fixed shuffle tree adds the point's
//     levels.  No atomics.
//   * Backward, tables, without float atomics: a pre-pass takes M = max |grad_out| per (grid, level) as an integer
//     atomicMax on the float bits (order-independent).  Every contribution g w (float32) is scaled by 2^s, rounded
//     to int64 and added with red.global.add.u64, with s chosen so that count M 2^s < 2^61 (count = F N, and a
//     point's corner weights sum to 1, so no slot and no partial sum can overflow).  Integer addition is associative:
//     the sums do not depend on the order of the adds.  A last pass writes float(double(sum) 2^-s), or NaN for every
//     slot of a (grid, level) whose M is not finite.
#include "common.cuh"
#include "hashgrid_kernels.h"

namespace dgm {

#define HG_BLOCK 256

namespace {

// the coordinate (0..3 = x, y, z, t) of axis a of grid kind k: xyz (0 1 2), xyt (0 1 3), yzt (1 2 3), xzt (0 2 3)
__device__ __forceinline__ int hg_axis(int kind, int a) {
  constexpr uint32_t AX = (0u | 1u << 2 | 2u << 4) | (0u | 1u << 2 | 3u << 4) << 6 | (1u | 2u << 2 | 3u << 4) << 12 |
                          (0u | 2u << 2 | 3u << 4) << 18;
  return (int)((AX >> (6 * kind + 2 * a)) & 3u);
}

// u = clamp((x - lo) / (hi - lo), 0, 1) per spatial axis, and du/dx = 1 / (hi - lo) where the unclamped u is in
// [0, 1] (torch.clamp's convention), else 0
__device__ __forceinline__ void hg_point(const float* __restrict__ box, const float* __restrict__ x, int n, float u[4],
                                         float dudx[3]) {
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float lo = __ldg(box + a), w = __ldg(box + 3 + a) - lo;
    const float raw = (__ldg(x + 3 * (size_t)n + a) - lo) / w;
    u[a] = fminf(fmaxf(raw, 0.f), 1.f);
    dudx[a] = (raw >= 0.f && raw <= 1.f) ? 1.f / w : 0.f;
  }
  u[3] = 0.f;
}

__device__ __forceinline__ float hg_time(float t) { return fminf(fmaxf(t, 0.f), 1.f); }

// the cell of level l of grid g: the 8 corner slots (corner k = c + (k & 1, k >> 1 & 1, k >> 2 & 1)), the fractions
// w and each axis's resolution
struct HgCell {
  uint32_t slot[8];
  float w[3];
  int R[3];
};

__device__ __forceinline__ void hg_cell(const HgField& f, int g, int l, const float u[4], HgCell& c) {
  const int kind = f.kind[g];
  int i[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int ax = hg_axis(kind, a);
    const int R = ax == 3 ? f.Rt[l] : f.R[l];
    const float ua = ax == 0 ? u[0] : ax == 1 ? u[1] : ax == 2 ? u[2] : u[3];  // selects, not a local array
    const float p = __fmul_rn(ua, (float)R);  // never contracted: w below is p - c of the rounded product
    const int ci = min((int)floorf(p), R - 1);
    c.w[a] = p - (float)ci;
    c.R[a] = R;
    i[a] = ci;
  }
  const bool dense = (f.dense[g] >> l) & 1u;
  const uint32_t mask = (1u << f.log2T) - 1u;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const uint32_t n0 = i[0] + (k & 1), n1 = i[1] + (k >> 1 & 1), n2 = i[2] + (k >> 2 & 1);
    c.slot[k] = dense ? n0 + (uint32_t)(c.R[0] + 1) * (n1 + (uint32_t)(c.R[1] + 1) * n2)
                      : (n0 ^ n1 * 2654435761u ^ n2 * 805459861u) & mask;
  }
}

// corner k's trilinear factors: a[j] = w_j or 1 - w_j
__device__ __forceinline__ void hg_factors(const HgCell& c, int k, float a[3]) {
#pragma unroll
  for (int j = 0; j < 3; ++j) a[j] = (k >> j & 1) ? c.w[j] : 1.f - c.w[j];
}

// element g of a by-value pointer array, by selects (a dynamic index would copy the kernel parameter to the stack)
template <typename P>
__device__ __forceinline__ P hg_pick(const P (&a)[HG_MAX_G], int g) {
  return g == 0 ? a[0] : g == 1 ? a[1] : g == 2 ? a[2] : a[3];
}

template <int FE>
__device__ __forceinline__ void hg_load(const float* p, float (&r)[FE]) {
  if constexpr (FE == 2) {
    const float2 q = __ldg(reinterpret_cast<const float2*>(p));
    r[0] = q.x, r[1] = q.y;
  } else {
    const float4 q = __ldg(reinterpret_cast<const float4*>(p));
    r[0] = q.x, r[1] = q.y, r[2] = q.z, r[3] = q.w;
  }
}

template <int FE>
__device__ __forceinline__ void hg_store(float* p, const float (&r)[FE]) {
  if constexpr (FE == 2) *reinterpret_cast<float2*>(p) = make_float2(r[0], r[1]);
  else *reinterpret_cast<float4*>(p) = make_float4(r[0], r[1], r[2], r[3]);
}

// the 8 corner rows of a cell, all loads issued before any is used
template <int FE>
__device__ __forceinline__ void hg_gather(const float* __restrict__ tab, const HgCell& c, float (&r)[8][FE]) {
#pragma unroll
  for (int k = 0; k < 8; ++k) hg_load<FE>(tab + (size_t)c.slot[k] * FE, r[k]);
}

template <int FE>
__global__ void __launch_bounds__(HG_BLOCK) hg_fwd_kernel(int F, int N, int lp_log2, HgField f,
                                                          const float* __restrict__ box, const float* __restrict__ x,
                                                          const float* __restrict__ t, float* __restrict__ out) {
  const size_t gid = (size_t)blockIdx.x * HG_BLOCK + threadIdx.x;
  const int n = (int)(gid >> lp_log2), l = (int)(gid & ((1u << lp_log2) - 1u));
  if (n >= N || l >= f.L) return;
  float u[4], dudx[3];
  hg_point(box, x, n, u, dudx);
  const size_t T = (size_t)1 << f.log2T, row = (size_t)f.G * f.L * FE;
  for (int g = 0; g < f.G; ++g) {
    const float* tab = hg_pick(f.tab, g) + (size_t)l * T * FE;
    const bool timed = f.kind[g] != 0;
    const size_t col = ((size_t)g * f.L + l) * FE;
    for (int fr = 0; fr < (timed ? F : 1); ++fr) {
      if (timed) u[3] = hg_time(__ldg(t + (size_t)fr * N + n));
      HgCell c;
      hg_cell(f, g, l, u, c);
      float r[8][FE];
      hg_gather<FE>(tab, c, r);
      float o[FE];
#pragma unroll
      for (int j = 0; j < FE; ++j) o[j] = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        float a[3];
        hg_factors(c, k, a);
        const float wk = a[0] * a[1] * a[2];
#pragma unroll
        for (int j = 0; j < FE; ++j) o[j] += wk * r[k][j];
      }
      if (timed) {
        hg_store<FE>(out + ((size_t)fr * N + n) * row + col, o);
      } else {
        for (int f2 = 0; f2 < F; ++f2) hg_store<FE>(out + ((size_t)f2 * N + n) * row + col, o);
      }
    }
  }
}

// M per (grid, level) as the bits of max |grad_out| (NaN above +inf above every finite value): a block's maxima in
// shared memory, then one global atomicMax per (block, grid, level)
template <int FE>
__global__ void __launch_bounds__(HG_BLOCK) hg_max_kernel(size_t rows, int GL, const float* __restrict__ grad_out,
                                                          uint32_t* __restrict__ mbits) {
  __shared__ uint32_t sm[HG_MAX_G * HG_MAX_L];
  for (int i = threadIdx.x; i < GL; i += HG_BLOCK) sm[i] = 0u;
  __syncthreads();
  for (size_t r = (size_t)blockIdx.x * HG_BLOCK + threadIdx.x; r < rows; r += (size_t)gridDim.x * HG_BLOCK) {
    float v[FE];
    hg_load<FE>(grad_out + r * FE, v);
    uint32_t m = 0u;
#pragma unroll
    for (int j = 0; j < FE; ++j) m = max(m, __float_as_uint(v[j]) & 0x7fffffffu);
    if (m) atomicMax(&sm[r % GL], m);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < GL; i += HG_BLOCK)
    if (sm[i]) atomicMax(mbits + i, sm[i]);
}

// s with count M 2^s < 2^61 for M < 2^e (frexp's exponent of M, from its bits) and count <= 2^k
__device__ __forceinline__ int hg_shift(uint32_t mbits, unsigned long long count) {
  const int ef = (int)(mbits >> 23);
  const int e = ef ? ef - 126 : (mbits ? -117 - __clz((int)mbits) : 0);
  const int k = count > 1 ? 64 - __clzll(count - 1) : 0;
  return 61 - k - e;
}

// 2^s as a double, from its bits (|s| stays far inside the normal range: -190 < s < 210)
__device__ __forceinline__ double hg_pow2(int s) { return __longlong_as_double((long long)(s + 1023) << 52); }

__device__ __forceinline__ bool hg_finite(uint32_t mbits) { return mbits < 0x7f800000u; }

template <int FE>
__global__ void __launch_bounds__(HG_BLOCK, 2) hg_bwd_kernel(int F, int N, int lp_log2, HgField f,
                                                          const float* __restrict__ box, const float* __restrict__ x,
                                                          const float* __restrict__ t,
                                                          const float* __restrict__ grad_out, float* __restrict__ grad_x,
                                                          const uint32_t* __restrict__ mbits,
                                                          unsigned long long* __restrict__ acc) {
  const size_t gid = (size_t)blockIdx.x * HG_BLOCK + threadIdx.x;
  const int Lp = 1 << lp_log2;
  const int n = (int)(gid >> lp_log2), l = (int)(gid & (Lp - 1));
  const bool valid = n < N && l < f.L;  // every lane stays for the shuffle tree below
  float dx[3] = {0.f, 0.f, 0.f};
  if (valid) {
    float u[4], dudx[3];
    hg_point(box, x, n, u, dudx);
    const size_t T = (size_t)1 << f.log2T, row = (size_t)f.G * f.L * FE;
    const unsigned long long count = (unsigned long long)F * N;
    for (int g = 0; g < f.G; ++g) {
      const int gl = g * f.L + l;
      const uint32_t m = __ldg(mbits + gl);
      const bool finite = hg_finite(m);
      const double scale = hg_pow2(hg_shift(m, count));
      const float* tab = hg_pick(f.tab, g) + (size_t)l * T * FE;
      unsigned long long* a64 = acc + (size_t)gl * T * FE;
      const bool timed = f.kind[g] != 0;
      float gs[FE];
#pragma unroll
      for (int j = 0; j < FE; ++j) gs[j] = 0.f;
      for (int fr = 0; fr < F; ++fr) {
        float gv[FE];
        hg_load<FE>(grad_out + ((size_t)fr * N + n) * row + (size_t)gl * FE, gv);
        if (!timed) {  // the spatial grid: the frames' grad_out summed in frame order, one pass after the loop
#pragma unroll
          for (int j = 0; j < FE; ++j) gs[j] += gv[j];
          if (fr + 1 < F) continue;
#pragma unroll
          for (int j = 0; j < FE; ++j) gv[j] = gs[j];
        } else {
          u[3] = hg_time(__ldg(t + (size_t)fr * N + n));
        }
        HgCell c;
        hg_cell(f, g, l, u, c);
        if (grad_x) {
          float r[8][FE];
          hg_gather<FE>(tab, c, r);
          float dw[3] = {0.f, 0.f, 0.f};
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            float a[3];
            hg_factors(c, k, a);
            float sk = 0.f;
#pragma unroll
            for (int j = 0; j < FE; ++j) sk += gv[j] * r[k][j];
            const float s0 = (k & 1) ? sk : -sk, s1 = (k & 2) ? sk : -sk, s2 = (k & 4) ? sk : -sk;
            dw[0] += s0 * (a[1] * a[2]);
            dw[1] += s1 * (a[0] * a[2]);
            dw[2] += s2 * (a[0] * a[1]);
          }
#pragma unroll
          for (int a = 0; a < 3; ++a) {
            const int ax = hg_axis(f.kind[g], a);
            const float d = dw[a] * (float)c.R[a];
            if (ax == 0) dx[0] += d * dudx[0];
            else if (ax == 1) dx[1] += d * dudx[1];
            else if (ax == 2) dx[2] += d * dudx[2];
          }
        }
        if (finite) {
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            float a[3];
            hg_factors(c, k, a);
            const float wk = a[0] * a[1] * a[2];
#pragma unroll
            for (int j = 0; j < FE; ++j) {
              const long long q = __double2ll_rn((double)(gv[j] * wk) * scale);
              if (q) atomicAdd(a64 + (size_t)c.slot[k] * FE + j, (unsigned long long)q);
            }
          }
        }
      }
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a)
    for (int off = Lp / 2; off >= 1; off >>= 1) dx[a] += __shfl_xor_sync(0xffffffffu, dx[a], off, Lp);
  if (valid && l == 0 && grad_x) {
    grad_x[3 * (size_t)n] = dx[0];
    grad_x[3 * (size_t)n + 1] = dx[1];
    grad_x[3 * (size_t)n + 2] = dx[2];
  }
}

// every table entry: float(double(sum) 2^-s), or NaN across a (grid, level) whose M is not finite
__global__ void __launch_bounds__(HG_BLOCK) hg_finish_kernel(int F, int N, HgField f, const uint32_t* __restrict__ mbits,
                                                             const long long* __restrict__ acc, HgGrads g) {
  const int shift = f.log2T + (f.Fe == 4 ? 2 : 1);  // log2 (T Fe): entries per (grid, level)
  const size_t level = (size_t)1 << shift, total = (size_t)f.G * f.L * level;
  const unsigned long long count = (unsigned long long)F * N;
  for (size_t e = (size_t)blockIdx.x * HG_BLOCK + threadIdx.x; e < total; e += (size_t)gridDim.x * HG_BLOCK) {
    const int gl = (int)(e >> shift), gr = gl / f.L;
    const uint32_t m = __ldg(mbits + gl);
    const float v = hg_finite(m) ? (float)((double)__ldg(acc + e) * hg_pow2(-hg_shift(m, count))) : __int_as_float(0x7fc00000);
    hg_pick(g.tab, gr)[e - (size_t)gr * f.L * level] = v;
  }
}

int hg_lp_log2(int L) {
  int k = 0;
  while ((1 << k) < L) ++k;
  return k;
}

unsigned hg_stride_blocks(size_t work) {
  const size_t b = (work + HG_BLOCK - 1) / HG_BLOCK;
  return (unsigned)(b < 132 * 16 ? (b ? b : 1) : 132 * 16);
}

}  // namespace

size_t hg_ws_bytes(const HgField& f) {
  char* p = nullptr;
  carve<long long>(p, ((size_t)f.G * f.L << f.log2T) * f.Fe);
  carve<uint32_t>(p, (size_t)f.G * f.L);
  return size_t(p) + 128;
}

cudaError_t launch_hashgrid_fwd(int F, int N, const HgField& f, const float* box, const float* x, const float* t,
                                float* out, cudaStream_t s) {
  if (F == 0 || N == 0) return cudaSuccess;
  const int lp = hg_lp_log2(f.L);
  const unsigned blocks = (unsigned)((((size_t)N << lp) + HG_BLOCK - 1) / HG_BLOCK);
  if (f.Fe == 2) hg_fwd_kernel<2><<<blocks, HG_BLOCK, 0, s>>>(F, N, lp, f, box, x, t, out);
  else hg_fwd_kernel<4><<<blocks, HG_BLOCK, 0, s>>>(F, N, lp, f, box, x, t, out);
  return cudaGetLastError();
}

cudaError_t launch_hashgrid_bwd(int F, int N, const HgField& f, const float* box, const float* x, const float* t,
                                const float* grad_out, float* grad_x, const HgGrads& g, void* ws, cudaStream_t s) {
  const size_t per_grid = ((size_t)f.L << f.log2T) * f.Fe;
  if (F == 0 || N == 0) {  // nothing sampled: every table gradient is 0
    for (int i = 0; i < f.G; ++i) cudaMemsetAsync(g.tab[i], 0, per_grid * sizeof(float), s);
    return cudaGetLastError();
  }
  char* p = (char*)ws;
  const size_t entries = (size_t)f.G * per_grid, GL = (size_t)f.G * f.L;
  long long* acc = carve<long long>(p, entries);
  uint32_t* mbits = carve<uint32_t>(p, GL);
  cudaMemsetAsync(acc, 0, entries * sizeof(long long), s);
  cudaMemsetAsync(mbits, 0, GL * sizeof(uint32_t), s);
  const size_t rows = (size_t)F * N * GL;
  const int lp = hg_lp_log2(f.L);
  const unsigned blocks = (unsigned)((((size_t)N << lp) + HG_BLOCK - 1) / HG_BLOCK);
  unsigned long long* acc_u = reinterpret_cast<unsigned long long*>(acc);
  if (f.Fe == 2) {
    hg_max_kernel<2><<<hg_stride_blocks(rows), HG_BLOCK, 0, s>>>(rows, (int)GL, grad_out, mbits);
    hg_bwd_kernel<2><<<blocks, HG_BLOCK, 0, s>>>(F, N, lp, f, box, x, t, grad_out, grad_x, mbits, acc_u);
  } else {
    hg_max_kernel<4><<<hg_stride_blocks(rows), HG_BLOCK, 0, s>>>(rows, (int)GL, grad_out, mbits);
    hg_bwd_kernel<4><<<blocks, HG_BLOCK, 0, s>>>(F, N, lp, f, box, x, t, grad_out, grad_x, mbits, acc_u);
  }
  hg_finish_kernel<<<hg_stride_blocks(entries), HG_BLOCK, 0, s>>>(F, N, f, mbits, acc, g);
  return cudaGetLastError();
}

}  // namespace dgm
