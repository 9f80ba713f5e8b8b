// hexplane.cu -- the HexPlane / K-Planes space-time feature field of 4D-GS, forward and backward, and its three
// plane regularisers (include/dgmesh_b200.h "dghp_" states the definitions).
//
//   * Layout: plane (s, p) is channels-last [R_b, R_a, C], so one corner's C channels are one line.  A thread owns
//     four channels of one point (C / 4 threads a point): every corner is one float4 load and the threads of a point
//     read one contiguous line.  The pixel coordinate of an axis is (x - lo) (R - 1) / (hi - lo), clamped to
//     [0, R - 1] (grid_sample's align_corners=True, padding_mode='border'); time's is t (R_t - 1), clamped.
//   * Forward: per (point, scale) the three spatial planes are sampled once, A = s0 s1 s3; per frame the three time
//     planes, and the feature is A (s2 s4 s5).  Nothing is stored for the backward.
//   * Backward, one pass per (point, channel quad): the six samples are recomputed, dL/dsample_p = g prod_{q != p}
//     s_q with the spatial ones summed over the frames in frame order (dL/dA = sum_f g_f T_f), and dL/dx is the
//     channel sum through each plane's bilinear derivative, the clamp (0 outside the box and on its faces, as in
//     torch) and the box scale, reduced over the point's threads by a fixed shuffle tree.  Each (plane, entry) --
//     entry = point for a spatial plane, (frame, point) for a time plane -- stages dL/dsample [C], its bilinear
//     fractions and the key of its cell.
//   * Plane gradients without float atomics: one CUB stable radix sort of the entry ids by global cell id (a short
//     key: key_bits of the cell count), then one thread per (cell, channel quad) sums its entries' four corner
//     terms in increasing entry id, and one thread per (texel, channel quad) adds its four adjacent cells' corner
//     sums in a fixed order.  Bit-identical from run to run.
//   * Regularisers: one kernel per direction over every texel of every plane.  The forward's CTAs write partial
//     sums; the CTA that finishes last (an integer ticket) adds them in a fixed order, in double.  The
//     backward is the stencils' gather, one thread per (texel, channel quad).
#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"
#include "csr_inverse.cuh"
#include "hexplane_kernels.h"

namespace dgm {

#define HP_BLOCK 256

namespace {

__host__ __device__ __forceinline__ bool hp_time_plane(int p) { return p == 2 || p == 4 || p == 5; }
__host__ __device__ __forceinline__ int hp_rows(const HpField& f, int s, int p) { return hp_time_plane(p) ? f.Rt : f.R[s]; }

// the global id of plane (s, p)'s first cell; cells of a plane are (R_b - 1) (R_a - 1), row-major
__host__ __device__ inline size_t hp_cell_base(const HpField& f, int plane) {
  size_t c = 0;
  for (int q = 0; q < plane; ++q) c += (size_t)(hp_rows(f, q / HP_PLANES, q % HP_PLANES) - 1) * (f.R[q / HP_PLANES] - 1);
  return c;
}

struct Bl {
  int off;  // element offset of the cell's (row y0, column x0) corner
  int Ra;   // row length in texels
  float fx, fy;
};

__device__ __forceinline__ float hp_pix(float v, float lo, float scale, int R, float& clip) {
  const float p = (v - lo) * scale;
  const float hi = (float)(R - 1);
  clip = (p > 0.f && p < hi) ? 1.f : 0.f;  // torch: the border counts as outside (zero coordinate gradient)
  return fminf(fmaxf(p, 0.f), hi);
}

__device__ __forceinline__ Bl hp_cell(float pa, float pb, int Ra, int Rb, int C, int& cell) {
  const int x0 = min((int)pa, Ra - 2), y0 = min((int)pb, Rb - 2);
  cell = y0 * (Ra - 1) + x0;
  return {(y0 * Ra + x0) * C, Ra, pa - (float)x0, pb - (float)y0};
}

__device__ __forceinline__ float4 f4(float a) { return make_float4(a, a, a, a); }
__device__ __forceinline__ float4 operator*(float4 a, float4 b) { return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }
__device__ __forceinline__ float4 operator+(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ float4 operator-(float4 a, float4 b) { return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }
__device__ __forceinline__ float dot4(float4 a, float4 b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }

// bilinear sample of four channels at channel offset c4, and (optionally) its derivatives along a and b in pixels
template <bool DERIV>
__device__ __forceinline__ float4 hp_sample(const float* __restrict__ plane, const Bl& b, int C, int c4, float4* da,
                                            float4* db) {
  const float4* q = reinterpret_cast<const float4*>(plane + b.off + c4);
  const int row = b.Ra * C / 4;
  const float4 v00 = __ldg(q), v01 = __ldg(q + C / 4), v10 = __ldg(q + row), v11 = __ldg(q + row + C / 4);
  const float4 gx = f4(1.f - b.fx), fx = f4(b.fx), gy = f4(1.f - b.fy), fy = f4(b.fy);
  if (DERIV) {
    *da = gy * (v01 - v00) + fy * (v11 - v10);
    *db = gx * (v10 - v00) + fx * (v11 - v01);
  }
  return gy * (gx * v00 + fx * v01) + fy * (gx * v10 + fx * v11);
}

// the clamped pixel coordinates of point n at scale s, with clip(x) (R - 1) / (hi - lo) per spatial axis in dpix
__device__ __forceinline__ void hp_coords(const HpField& f, int s, const float* __restrict__ box,
                                          const float* __restrict__ x, int n, float pix[3], float dpix[3]) {
  const int R = f.R[s];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float lo = __ldg(box + a), hi = __ldg(box + 3 + a);
    const float scale = (float)(R - 1) / (hi - lo);
    float clip;
    pix[a] = hp_pix(__ldg(x + 3 * (size_t)n + a), lo, scale, R, clip);
    dpix[a] = clip * scale;
  }
}

__device__ __forceinline__ float hp_tpix(const HpField& f, float t) {
  return fminf(fmaxf(t * (float)(f.Rt - 1), 0.f), (float)(f.Rt - 1));
}

template <int C>
__global__ void __launch_bounds__(HP_BLOCK) hp_fwd_kernel(int F, int N, HpField f, const float* __restrict__ box,
                                                          const float* __restrict__ x, const float* __restrict__ t,
                                                          float* __restrict__ out) {
  constexpr int G = C / 4;
  const size_t gid = (size_t)blockIdx.x * HP_BLOCK + threadIdx.x;
  const int n = (int)(gid / G), c4 = 4 * (int)(gid % G);
  if (n >= N) return;
  const size_t SC = (size_t)f.S * C;
  for (int s = 0; s < f.S; ++s) {
    float pix[3], dpix[3];
    hp_coords(f, s, box, x, n, pix, dpix);
    const int R = f.R[s];
    int cell;
    const float4 s0 = hp_sample<false>(f.p[6 * s + 0], hp_cell(pix[0], pix[1], R, R, C, cell), C, c4, nullptr, nullptr);
    const float4 s1 = hp_sample<false>(f.p[6 * s + 1], hp_cell(pix[0], pix[2], R, R, C, cell), C, c4, nullptr, nullptr);
    const float4 s3 = hp_sample<false>(f.p[6 * s + 3], hp_cell(pix[1], pix[2], R, R, C, cell), C, c4, nullptr, nullptr);
    const float4 A = s0 * s1 * s3;
    for (int fr = 0; fr < F; ++fr) {
      const float pt = hp_tpix(f, __ldg(t + (size_t)fr * N + n));
      const float4 s2 = hp_sample<false>(f.p[6 * s + 2], hp_cell(pix[0], pt, R, f.Rt, C, cell), C, c4, nullptr, nullptr);
      const float4 s4 = hp_sample<false>(f.p[6 * s + 4], hp_cell(pix[1], pt, R, f.Rt, C, cell), C, c4, nullptr, nullptr);
      const float4 s5 = hp_sample<false>(f.p[6 * s + 5], hp_cell(pix[2], pt, R, f.Rt, C, cell), C, c4, nullptr, nullptr);
      *reinterpret_cast<float4*>(out + ((size_t)fr * N + n) * SC + (size_t)s * C + c4) = A * (s2 * s4 * s5);
    }
  }
}

// one (plane, entry)'s staging: dL/dsample (every thread its quad), and once per entry its fractions and cell key
__device__ __forceinline__ void hp_stage(const HpWS& w, size_t e, int C, int c4, float4 d, const Bl& b, uint32_t key) {
  *reinterpret_cast<float4*>(w.stage + e * C + c4) = d;
  if (c4 == 0) {
    w.frac[e] = make_float2(b.fx, b.fy);
    w.keys_in[e] = key;
    w.vals_in[e] = (uint32_t)e;
  }
}

template <int C>
__global__ void __launch_bounds__(HP_BLOCK) hp_bwd_kernel(int F, int N, HpField f, const float* __restrict__ box,
                                                          const float* __restrict__ x, const float* __restrict__ t,
                                                          const float* __restrict__ grad_out,
                                                          float* __restrict__ grad_x, HpWS w) {
  constexpr int G = C / 4;
  const size_t gid = (size_t)blockIdx.x * HP_BLOCK + threadIdx.x;
  const bool valid = gid / G < (size_t)N;  // a point's G threads are all valid or all not (G divides 32)
  const int n = valid ? (int)(gid / G) : N - 1, c4 = 4 * (int)(gid % G);
  const size_t SC = (size_t)f.S * C, FN = (size_t)F * N;
  float dx[3] = {0.f, 0.f, 0.f};
  for (int s = 0; s < f.S; ++s) {
    float pix[3], dpix[3];
    hp_coords(f, s, box, x, n, pix, dpix);
    const int R = f.R[s];
    // entries of scale s: planes 0, 1 (N each), 2 (F N), 3 (N), 4, 5 (F N each)
    const size_t eb = (size_t)s * (3 * (size_t)N + 3 * FN);
    const size_t e0 = eb, e1 = eb + N, e2 = eb + 2 * (size_t)N, e3 = e2 + FN, e4 = e3 + N, e5 = e4 + FN;
    uint32_t cb[HP_PLANES];
#pragma unroll
    for (int p = 0; p < HP_PLANES; ++p) cb[p] = (uint32_t)hp_cell_base(f, 6 * s + p);
    int k0, k1, k3;
    const Bl b0 = hp_cell(pix[0], pix[1], R, R, C, k0), b1 = hp_cell(pix[0], pix[2], R, R, C, k1),
             b3 = hp_cell(pix[1], pix[2], R, R, C, k3);
    float4 d0a, d0b, d1a, d1b, d3a, d3b;
    const float4 s0 = hp_sample<true>(f.p[6 * s + 0], b0, C, c4, &d0a, &d0b);
    const float4 s1 = hp_sample<true>(f.p[6 * s + 1], b1, C, c4, &d1a, &d1b);
    const float4 s3 = hp_sample<true>(f.p[6 * s + 3], b3, C, c4, &d3a, &d3b);
    const float4 A = s0 * s1 * s3;
    float4 GA = f4(0.f);
    float tx = 0.f, ty = 0.f, tz = 0.f;
    for (int fr = 0; fr < F; ++fr) {
      const size_t fn = (size_t)fr * N + n;
      const float4 g = __ldg(reinterpret_cast<const float4*>(grad_out + fn * SC + (size_t)s * C + c4));
      const float pt = hp_tpix(f, __ldg(t + fn));
      int k2, k4, k5;
      const Bl b2 = hp_cell(pix[0], pt, R, f.Rt, C, k2), b4 = hp_cell(pix[1], pt, R, f.Rt, C, k4),
               b5 = hp_cell(pix[2], pt, R, f.Rt, C, k5);
      float4 e2a, e4a, e5a, unused;
      const float4 s2 = hp_sample<true>(f.p[6 * s + 2], b2, C, c4, &e2a, &unused);
      const float4 s4 = hp_sample<true>(f.p[6 * s + 4], b4, C, c4, &e4a, &unused);
      const float4 s5 = hp_sample<true>(f.p[6 * s + 5], b5, C, c4, &e5a, &unused);
      GA = GA + g * (s2 * s4 * s5);
      const float4 gA = g * A;
      const float4 q2 = gA * (s4 * s5), q4 = gA * (s2 * s5), q5 = gA * (s2 * s4);
      if (valid) {
        hp_stage(w, e2 + fn, C, c4, q2, b2, cb[2] + k2);
        hp_stage(w, e4 + fn, C, c4, q4, b4, cb[4] + k4);
        hp_stage(w, e5 + fn, C, c4, q5, b5, cb[5] + k5);
      }
      tx += dot4(q2, e2a);
      ty += dot4(q4, e4a);
      tz += dot4(q5, e5a);
    }
    const float4 q0 = GA * (s1 * s3), q1 = GA * (s0 * s3), q3 = GA * (s0 * s1);
    if (valid) {
      hp_stage(w, e0 + n, C, c4, q0, b0, cb[0] + k0);
      hp_stage(w, e1 + n, C, c4, q1, b1, cb[1] + k1);
      hp_stage(w, e3 + n, C, c4, q3, b3, cb[3] + k3);
    }
    dx[0] += (tx + dot4(q0, d0a) + dot4(q1, d1a)) * dpix[0];
    dx[1] += (ty + dot4(q0, d0b) + dot4(q3, d3a)) * dpix[1];
    dx[2] += (tz + dot4(q1, d1b) + dot4(q3, d3b)) * dpix[2];
  }
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int off = G / 2; off >= 1; off >>= 1) dx[a] += __shfl_xor_sync(0xffffffffu, dx[a], off, G);
  if (valid && c4 == 0 && grad_x) {
    grad_x[3 * (size_t)n] = dx[0];
    grad_x[3 * (size_t)n + 1] = dx[1];
    grad_x[3 * (size_t)n + 2] = dx[2];
  }
}

// one thread per (cell, channel quad): the cell's four corner sums over its entries in increasing entry id
template <int C>
__global__ void __launch_bounds__(HP_BLOCK) hp_cell_kernel(size_t cells, size_t E, HpWS w) {
  constexpr int G = C / 4;
  const size_t gid = (size_t)blockIdx.x * HP_BLOCK + threadIdx.x;
  if (gid >= cells * G) return;
  const size_t c = gid / G;
  const int c4 = 4 * (int)(gid % G);
  const int lo = lower_bound_u32(w.keys_out, (int)E, (uint32_t)c),
            hi = lower_bound_u32(w.keys_out, (int)E, (uint32_t)c + 1u);
  float4 a00 = f4(0.f), a01 = f4(0.f), a10 = f4(0.f), a11 = f4(0.f);
  for (int j = lo; j < hi; ++j) {
    const size_t e = __ldg(w.vals_out + j);
    const float2 fr = w.frac[e];
    const float4 d = *reinterpret_cast<const float4*>(w.stage + e * C + c4);
    const float gx = 1.f - fr.x, gy = 1.f - fr.y;
    a00 = a00 + f4(gx * gy) * d;
    a01 = a01 + f4(fr.x * gy) * d;
    a10 = a10 + f4(gx * fr.y) * d;
    a11 = a11 + f4(fr.x * fr.y) * d;
  }
  float4* o = reinterpret_cast<float4*>(w.cell_acc + c * 4 * C + c4);
  o[0] = a00;
  o[G] = a01;
  o[2 * G] = a10;
  o[3 * G] = a11;
}

// grid (texel blocks, 6 S): texel (ty, tx) of plane (s, p) adds the corner sums of the cells (ty-1, tx-1),
// (ty-1, tx), (ty, tx-1), (ty, tx), in that order
template <int C>
__global__ void __launch_bounds__(HP_BLOCK) hp_texel_kernel(HpField f, HpGrads g, const float* __restrict__ cell_acc) {
  constexpr int G = C / 4;
  const int plane = blockIdx.y, s = plane / HP_PLANES, p = plane % HP_PLANES;
  const int Ra = f.R[s], Rb = hp_rows(f, s, p);
  const size_t gid = (size_t)blockIdx.x * HP_BLOCK + threadIdx.x;
  if (gid >= (size_t)Ra * Rb * G) return;
  const int texel = (int)(gid / G), c4 = 4 * (int)(gid % G);
  const int ty = texel / Ra, tx = texel % Ra;
  const size_t cb = hp_cell_base(f, plane);
  const int Rc = Ra - 1;
  auto corner = [&](int cy, int cx, int k) {
    return *reinterpret_cast<const float4*>(cell_acc + ((cb + (size_t)cy * Rc + cx) * 4 + k) * C + c4);
  };
  float4 v = f4(0.f);
  if (ty > 0 && tx > 0) v = v + corner(ty - 1, tx - 1, 3);
  if (ty > 0 && tx < Rc) v = v + corner(ty - 1, tx, 2);
  if (ty < Rb - 1 && tx > 0) v = v + corner(ty, tx - 1, 1);
  if (ty < Rb - 1 && tx < Rc) v = v + corner(ty, tx, 0);
  *reinterpret_cast<float4*>(g.p[plane] + (size_t)texel * C + c4) = v;
}

// ---- regularisers

// grid (blocks of the largest plane, 6 S): partial[plane, block] = (tv rows, tv columns) of a spatial plane or
// (time smoothness, l1) of a time plane, unnormalised; the last CTA to finish writes the three means' sums
__global__ void __launch_bounds__(HP_BLOCK) hp_reg_fwd_kernel(HpField f, float2* __restrict__ partial,
                                                              unsigned* __restrict__ ticket, float* __restrict__ losses) {
  __shared__ float red[2][HP_BLOCK / 32];
  __shared__ bool last;
  const int G = f.C / 4;
  const int plane = blockIdx.y, s = plane / HP_PLANES, p = plane % HP_PLANES;
  const int Ra = f.R[s], Rb = hp_rows(f, s, p);
  const size_t gid = (size_t)blockIdx.x * HP_BLOCK + threadIdx.x;
  const size_t row = (size_t)Ra * f.C;
  float a = 0.f, b = 0.f;
  if (gid < (size_t)Ra * Rb * G) {
    const int texel = (int)(gid / G), c4 = 4 * (int)(gid % G);
    const int ty = texel / Ra, tx = texel % Ra;
    const float* q = f.p[plane] + (size_t)texel * f.C + c4;
    const float4 v = __ldg(reinterpret_cast<const float4*>(q));
    if (!hp_time_plane(p)) {
      if (ty + 1 < Rb) {
        const float4 d = __ldg(reinterpret_cast<const float4*>(q + row)) - v;
        a = dot4(d, d);
      }
      if (tx + 1 < Ra) {
        const float4 d = __ldg(reinterpret_cast<const float4*>(q + f.C)) - v;
        b = dot4(d, d);
      }
    } else {
      if (ty + 2 < Rb) {
        const float4 d = __ldg(reinterpret_cast<const float4*>(q + 2 * row)) -
                         f4(2.f) * __ldg(reinterpret_cast<const float4*>(q + row)) + v;
        a = dot4(d, d);
      }
      b = fabsf(1.f - v.x) + fabsf(1.f - v.y) + fabsf(1.f - v.z) + fabsf(1.f - v.w);
    }
  }
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, off);
    b += __shfl_xor_sync(0xffffffffu, b, off);
  }
  if ((threadIdx.x & 31) == 0) red[0][threadIdx.x >> 5] = a, red[1][threadIdx.x >> 5] = b;
  __syncthreads();
  if (threadIdx.x == 0) {
    float ta = 0.f, tb = 0.f;
    for (int k = 0; k < HP_BLOCK / 32; ++k) ta += red[0][k], tb += red[1][k];
    partial[(size_t)plane * gridDim.x + blockIdx.x] = make_float2(ta, tb);
    __threadfence();
    last = atomicAdd(ticket, 1u) == gridDim.x * gridDim.y - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  // thread k adds partials k, k + HP_BLOCK, ... of every plane, each plane's sums divided by its counts, and a fixed
  // shared-memory tree adds the threads
  __shared__ double acc[3][HP_BLOCK];
  double tv = 0.0, ts = 0.0, l1 = 0.0;
  for (int pl = 0; pl < (int)gridDim.y; ++pl) {
    const int ps = pl / HP_PLANES, pp = pl % HP_PLANES;
    const double ra = f.R[ps], rb = hp_rows(f, ps, pp), C = f.C;
    double sa = 0.0, sb = 0.0;
    for (unsigned k = threadIdx.x; k < gridDim.x; k += HP_BLOCK) {
      const volatile float* v = (const volatile float*)(partial + (size_t)pl * gridDim.x + k);
      sa += v[0], sb += v[1];
    }
    if (!hp_time_plane(pp)) {
      tv += sa / ((rb - 1) * ra * C) + sb / (rb * (ra - 1) * C);
    } else {
      if (rb > 2) ts += sa / ((rb - 2) * ra * C);
      l1 += sb / (rb * ra * C);
    }
  }
  acc[0][threadIdx.x] = tv, acc[1][threadIdx.x] = ts, acc[2][threadIdx.x] = l1;
  __syncthreads();
  for (int h = HP_BLOCK / 2; h >= 1; h >>= 1) {
    if (threadIdx.x < h)
      for (int c = 0; c < 3; ++c) acc[c][threadIdx.x] += acc[c][threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x < 3) losses[threadIdx.x] = (float)acc[threadIdx.x][0];
}

__device__ __forceinline__ float4 hp_ld(const float* q) { return __ldg(reinterpret_cast<const float4*>(q)); }

// grid (blocks of the largest plane, 6 S): the stencils' gradient at every texel, gathered
__global__ void __launch_bounds__(HP_BLOCK) hp_reg_bwd_kernel(HpField f, const float* __restrict__ grad_losses,
                                                              HpGrads g) {
  const int G = f.C / 4;
  const int plane = blockIdx.y, s = plane / HP_PLANES, p = plane % HP_PLANES;
  const int Ra = f.R[s], Rb = hp_rows(f, s, p);
  const size_t gid = (size_t)blockIdx.x * HP_BLOCK + threadIdx.x;
  if (gid >= (size_t)Ra * Rb * G) return;
  const int texel = (int)(gid / G), c4 = 4 * (int)(gid % G);
  const int ty = texel / Ra, tx = texel % Ra;
  const size_t row = (size_t)Ra * f.C;
  const float* q = f.p[plane] + (size_t)texel * f.C + c4;
  const float4 v = hp_ld(q);
  const float C = (float)f.C;
  float4 out = f4(0.f);
  if (!hp_time_plane(p)) {
    // d/dG of mean (G[i+1] - G[i])^2 over rows and of mean (G[j+1] - G[j])^2 over columns
    const float wr = 2.f * __ldg(grad_losses) / ((float)(Rb - 1) * (float)Ra * C);
    const float wc = 2.f * __ldg(grad_losses) / ((float)Rb * (float)(Ra - 1) * C);
    float4 r = f4(0.f), c = f4(0.f);
    if (ty > 0) r = r + (v - hp_ld(q - row));
    if (ty + 1 < Rb) r = r - (hp_ld(q + row) - v);
    if (tx > 0) c = c + (v - hp_ld(q - f.C));
    if (tx + 1 < Ra) c = c - (hp_ld(q + f.C) - v);
    out = f4(wr) * r + f4(wc) * c;
  } else {
    // D(k) = G[k+2] - 2 G[k+1] + G[k], 0 <= k <= Rb - 3; row ty takes D(ty - 2) - 2 D(ty - 1) + D(ty)
    if (Rb > 2) {
      const float ws = 2.f * __ldg(grad_losses + 1) / ((float)(Rb - 2) * (float)Ra * C);
      auto D = [&](int k) {
        const float* b = q + (ptrdiff_t)(k - ty) * (ptrdiff_t)row;
        return hp_ld(b + 2 * row) - f4(2.f) * hp_ld(b + row) + hp_ld(b);
      };
      float4 d = f4(0.f);
      if (ty >= 2) d = d + D(ty - 2);
      if (ty >= 1 && ty - 1 <= Rb - 3) d = d - f4(2.f) * D(ty - 1);
      if (ty <= Rb - 3) d = d + D(ty);
      out = f4(ws) * d;
    }
    // d/dG mean |1 - G| = -sign(1 - G) / count, 0 at G = 1
    const float wl = __ldg(grad_losses + 2) / ((float)Rb * (float)Ra * C);
    auto sg = [](float u) { return u < 1.f ? -1.f : (u > 1.f ? 1.f : 0.f); };
    out = out + f4(wl) * make_float4(sg(v.x), sg(v.y), sg(v.z), sg(v.w));
  }
  *reinterpret_cast<float4*>(g.p[plane] + (size_t)texel * f.C + c4) = out;
}

size_t hp_max_texels(const HpField& f) {
  size_t m = 0;
  for (int s = 0; s < f.S; ++s) {
    const size_t R = f.R[s], t = R * (R > (size_t)f.Rt ? R : (size_t)f.Rt);
    m = t > m ? t : m;
  }
  return m;
}

}  // namespace

size_t hp_entries(int F, int N, int S) { return (size_t)S * 3 * (size_t)N * (1 + (size_t)F); }
size_t hp_cells(const HpField& f) { return hp_cell_base(f, HP_PLANES * f.S); }

size_t hp_cub_bytes(size_t E, size_t cells) {
  size_t b = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, b, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                  (uint32_t*)nullptr, (int)E, 0, key_bits(cells));
  return b;
}

HpWS HpWS::from(char* base, size_t E, size_t cells, int C, size_t cub_bytes, size_t* bytes) {
  char* p = base;
  HpWS w;
  w.stage = carve<float>(p, E * C);
  w.frac = carve<float2>(p, E);
  w.keys_in = carve<uint32_t>(p, E);
  w.keys_out = carve<uint32_t>(p, E);
  w.vals_in = carve<uint32_t>(p, E);
  w.vals_out = carve<uint32_t>(p, E);
  w.cell_acc = carve<float>(p, cells * 4 * C);
  w.cub_temp = carve<char>(p, cub_bytes);
  w.cub_bytes = cub_bytes;
  if (bytes) *bytes = size_t(p - base) + 128;
  return w;
}

cudaError_t launch_hexplane_fwd(int F, int N, const HpField& f, const float* box, const float* x, const float* t,
                                float* out, cudaStream_t s) {
  if (F == 0 || N == 0) return cudaSuccess;
  const size_t threads = (size_t)N * (f.C / 4);
  const unsigned blocks = (unsigned)((threads + HP_BLOCK - 1) / HP_BLOCK);
  if (f.C == 16) hp_fwd_kernel<16><<<blocks, HP_BLOCK, 0, s>>>(F, N, f, box, x, t, out);
  else hp_fwd_kernel<32><<<blocks, HP_BLOCK, 0, s>>>(F, N, f, box, x, t, out);
  return cudaGetLastError();
}

template <int C>
static void hp_bwd_launch(int F, int N, const HpField& f, const float* box, const float* x, const float* t,
                          const float* grad_out, float* grad_x, const HpGrads& g, HpWS& w, size_t E, size_t cells,
                          cudaStream_t s) {
  constexpr int G = C / 4;
  hp_bwd_kernel<C><<<(unsigned)(((size_t)N * G + HP_BLOCK - 1) / HP_BLOCK), HP_BLOCK, 0, s>>>(F, N, f, box, x, t,
                                                                                             grad_out, grad_x, w);
  size_t tb = w.cub_bytes;
  cub::DeviceRadixSort::SortPairs(w.cub_temp, tb, w.keys_in, w.keys_out, w.vals_in, w.vals_out, (int)E, 0,
                                  key_bits(cells), s);
  hp_cell_kernel<C><<<(unsigned)((cells * G + HP_BLOCK - 1) / HP_BLOCK), HP_BLOCK, 0, s>>>(cells, E, w);
  const dim3 grid((unsigned)((hp_max_texels(f) * G + HP_BLOCK - 1) / HP_BLOCK), HP_PLANES * f.S);
  hp_texel_kernel<C><<<grid, HP_BLOCK, 0, s>>>(f, g, w.cell_acc);
}

cudaError_t launch_hexplane_bwd(int F, int N, const HpField& f, const float* box, const float* x, const float* t,
                                const float* grad_out, float* grad_x, const HpGrads& g, void* ws, cudaStream_t s) {
  const size_t E = hp_entries(F, N, f.S), cells = hp_cells(f);
  if (F == 0 || N == 0) {  // no entries: every plane gradient is 0
    for (int p = 0; p < HP_PLANES * f.S; ++p) {
      const size_t rows = (p % HP_PLANES == 2 || p % HP_PLANES >= 4) ? f.Rt : f.R[p / HP_PLANES];
      cudaMemsetAsync(g.p[p], 0, rows * f.R[p / HP_PLANES] * f.C * sizeof(float), s);
    }
    return cudaGetLastError();
  }
  HpWS w = HpWS::from((char*)ws, E, cells, f.C, hp_cub_bytes(E, cells));
  if (f.C == 16) hp_bwd_launch<16>(F, N, f, box, x, t, grad_out, grad_x, g, w, E, cells, s);
  else hp_bwd_launch<32>(F, N, f, box, x, t, grad_out, grad_x, g, w, E, cells, s);
  return cudaGetLastError();
}

size_t hp_reg_blocks(const HpField& f) { return (hp_max_texels(f) * (f.C / 4) + HP_BLOCK - 1) / HP_BLOCK; }

size_t hp_reg_ws_bytes(const HpField& f) {
  char* p = nullptr;
  carve<float2>(p, hp_reg_blocks(f) * HP_PLANES * f.S);
  carve<unsigned>(p, 1);
  return size_t(p) + 128;
}

cudaError_t launch_hexplane_reg_fwd(const HpField& f, float* losses, void* ws, cudaStream_t s) {
  char* p = (char*)ws;
  const size_t nblk = hp_reg_blocks(f);
  float2* partial = carve<float2>(p, nblk * HP_PLANES * f.S);
  unsigned* ticket = carve<unsigned>(p, 1);
  cudaMemsetAsync(ticket, 0, sizeof(unsigned), s);
  hp_reg_fwd_kernel<<<dim3((unsigned)nblk, HP_PLANES * f.S), HP_BLOCK, 0, s>>>(f, partial, ticket, losses);
  return cudaGetLastError();
}

cudaError_t launch_hexplane_reg_bwd(const HpField& f, const float* grad_losses, const HpGrads& g, cudaStream_t s) {
  hp_reg_bwd_kernel<<<dim3((unsigned)hp_reg_blocks(f), HP_PLANES * f.S), HP_BLOCK, 0, s>>>(f, grad_losses, g);
  return cudaGetLastError();
}

}  // namespace dgm
