// raster_bwd.cu -- backward pass of the tile-based 3D-Gaussian rasterizer for sm_90a.
//
//   render_bwd_kernel      gradient of the alpha-composite (role of renderCUDA,
//                          dgr/cuda_rasterizer/backward.cu:399-557)
//   preprocess_bwd_kernel  chain rule to means3D / scales / rotations / SH / opacity
//                          (computeCov2DCUDA + preprocessCUDA, backward.cu:144-396, fused)
//
// The reference issues 9 global float atomics per contributing (pixel, Gaussian)
// pair.  Here each warp (8x4 pixels) reduces its 32 partial gradients with a
// transposing butterfly (14 shuffles for 9 values), adds the 9 sums into a per-tile
// shared-memory accumulator, and the tile flushes once per (tile, Gaussian) with
// vector reductions (red.global.add.v4.f32) into a [P,12] accumulator that the fused
// preprocess-backward consumes and re-zeroes.  The per-pair arithmetic follows the
// reference's back-to-front recurrence; only the summation order differs (the
// reference's own order is non-deterministic).
#include "common.cuh"
#include "raster_math.cuh"
#include "raster_kernels.h"

namespace dgm {

#define RB 256
#define ACC_STRIDE 9

// Reduce the 9 partial gradients of TWO Gaussians (A, B) over the 32 lanes of a warp with a
// transposing butterfly: at each level a lane keeps half of its values and trades the other
// half with its partner, so 16 values cost 8+4+2+1+1 = 16 shuffles (+5 for the pair of 9th
// values) instead of 2 x 9 x 5 = 90 for naive per-value reductions.
// On return, for lanes with (lane & 1) == 0: r8 = total of value ((lane>>1)&7) of Gaussian
// (lane>>4); r9 = total of value 8 of Gaussian (lane>>4) on every lane.
__device__ __forceinline__ void warp_reduce_pair(const float (&vK)[9], const float (&vS)[9], unsigned lane, float& r8,
                                                 float& r9) {
  // vK: the 9 values of the Gaussian this lane's half KEEPS (A on lanes 0-15, B on lanes 16-31),
  // vS: those of the Gaussian it SENDS to the other half -- arranged by the caller, so the first
  // (widest) butterfly stage needs no selects
  const unsigned FULL = 0xffffffffu;
  float a[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) a[k] = vK[k] + __shfl_xor_sync(FULL, vS[k], 16);
  float b[4];
  {
    const bool up = lane & 8;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float send = up ? a[k] : a[k + 4];
      const float keep = up ? a[k + 4] : a[k];
      b[k] = keep + __shfl_xor_sync(FULL, send, 8);
    }
  }
  float c[2];
  {
    const bool up = lane & 4;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const float send = up ? b[k] : b[k + 2];
      const float keep = up ? b[k + 2] : b[k];
      c[k] = keep + __shfl_xor_sync(FULL, send, 4);
    }
  }
  float d;
  {
    const bool up = lane & 2;
    const float send = up ? c[0] : c[1];
    const float keep = up ? c[1] : c[0];
    d = keep + __shfl_xor_sync(FULL, send, 2);
  }
  d += __shfl_xor_sync(FULL, d, 1);
  r8 = d;
  float e = vK[8] + __shfl_xor_sync(FULL, vS[8], 16);
  e += __shfl_xor_sync(FULL, e, 8);
  e += __shfl_xor_sync(FULL, e, 4);
  e += __shfl_xor_sync(FULL, e, 2);
  e += __shfl_xor_sync(FULL, e, 1);
  r9 = e;
}

__global__ void __launch_bounds__(256, 4) render_bwd_kernel(
    const uint2* __restrict__ ranges, const uint32_t* __restrict__ tile_order, const float4* __restrict__ inst_geo,
    const float4* __restrict__ inst_attr,
    int W, int H, const float* __restrict__ bg_color, const float* __restrict__ final_Ts,
    const uint32_t* __restrict__ n_contrib, const float* __restrict__ dL_dpixels, float4* __restrict__ grad_acc) {
  __shared__ __align__(128) float4 s_geo[2][RB];
  __shared__ __align__(128) float4 s_attr[2][2 * RB];
  __shared__ float s_acc[RB * ACC_STRIDE];
  __shared__ __align__(8) uint64_t s_bar[2];
  __shared__ int s_maxc;

  pdl_wait();
  pdl_launch();
  const unsigned gx = (W + TILE_X - 1) / TILE_X;
  const unsigned tile = tile_order[blockIdx.x];  // longest lists first
  const unsigned tx = tile % gx, ty = tile / gx;
  const unsigned tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int wx0 = tx * TILE_X + (wid & 1) * 8, wy0 = ty * TILE_Y + (wid >> 1) * 4;
  const int px = wx0 + (lane & 7), py = wy0 + (lane >> 3);
  const bool inside = px < W && py < H;
  const uint32_t pix_id = W * py + px;
  const float pixfx = (float)px, pixfy = (float)py;
  const float bx0 = (float)wx0, bx1 = (float)(wx0 + 7), by0 = (float)wy0, by1 = (float)(wy0 + 3);
  const float2 npx2 = make_float2(-pixfx, -pixfx), npy2 = make_float2(-pixfy, -pixfy);

  const uint2 range = ranges[tile];
  const int total = range.y - range.x;
  if (total == 0) return;  // uniform per CTA

  const float T_final = inside ? final_Ts[pix_id] : 0;
  float T = T_final;
  const int last_contributor = inside ? (int)n_contrib[pix_id] : 0;

  if (tid == 0) {
    s_maxc = 0;
    mbar_init(&s_bar[0], 1);
    mbar_init(&s_bar[1], 1);
    mbar_fence_init();
  }
  for (int i = tid; i < RB * ACC_STRIDE; i += 256) s_acc[i] = 0.f;
  __syncthreads();
  // positions >= max over the warp / tile of n_contrib can be skipped altogether
  int wmax = last_contributor;
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
  if (lane == 0) atomicMax(&s_maxc, wmax);
  __syncthreads();
  const int maxc = min(s_maxc, total);
  const int rounds = (maxc + RB - 1) / RB;
  if (rounds == 0) return;

  // batch i covers positions [hi_i - cnt_i, hi_i), hi_0 = maxc, walking towards the front
  if (tid == 0) {
    const int hi = maxc, lo = max(0, hi - RB);
    const uint32_t cnt = hi - lo;
    mbar_expect_tx(&s_bar[0], cnt * 48u);
    tma_load_1d(&s_geo[0][0], inst_geo + range.x + lo, cnt * 16u, &s_bar[0]);
    tma_load_1d(&s_attr[0][0], inst_attr + 2 * ((size_t)range.x + lo), cnt * 32u, &s_bar[0]);
  }

  float dLp0 = 0.f, dLp1 = 0.f, dLp2 = 0.f;
  if (inside) {
    const size_t HW = (size_t)H * W;
    dLp0 = dL_dpixels[0 * HW + pix_id];
    dLp1 = dL_dpixels[1 * HW + pix_id];
    dLp2 = dL_dpixels[2 * HW + pix_id];
  }
  float bg_dot_dpixel = 0;
  bg_dot_dpixel += bg_color[0] * dLp0;
  bg_dot_dpixel += bg_color[1] * dLp1;
  bg_dot_dpixel += bg_color[2] * dLp2;

  const float mTb = -T_final * bg_dot_dpixel;  // background term of dL/dalpha, times 1/(1-alpha) per record
  float accum0 = 0.f, accum1 = 0.f, accum2 = 0.f;  // colour composited behind the current record
  // d(pixel coordinate)/d(NDC), backward.cu:457-458 (double literal 0.5)
  const float ddelx_dx = 0.5 * W;
  const float ddely_dy = 0.5 * H;

  for (int i = 0; i < rounds; ++i) {
    const int st = i & 1;
    const int hi = maxc - i * RB, lo = max(0, hi - RB);
    const int cnt = hi - lo;
    mbar_wait(&s_bar[st], (i >> 1) & 1);
    __syncthreads();  // previous batch fully flushed; other stage free
    if (tid == 0 && i + 1 < rounds) {
      const int nhi = lo, nlo = max(0, nhi - RB);
      const uint32_t ncnt = nhi - nlo;
      mbar_expect_tx(&s_bar[st ^ 1], ncnt * 48u);
      tma_load_1d(&s_geo[st ^ 1][0], inst_geo + range.x + nlo, ncnt * 16u, &s_bar[st ^ 1]);
      tma_load_1d(&s_attr[st ^ 1][0], inst_attr + 2 * ((size_t)range.x + nlo), ncnt * 32u, &s_bar[st ^ 1]);
    }
    // ---- cull (same conservative extent test as the forward pass)
    unsigned keep[RB / 32];
#pragma unroll
    for (int k = 0; k < RB / 32; ++k) {
      const int r = k * 32 + lane;
      bool kp = false;
      if (r < cnt && (lo + r) < wmax) {
        kp = cull_keep(s_geo[st][r], s_attr[st][2 * r], bx0, bx1, by0, by1);
      }
      keep[k] = __ballot_sync(0xffffffffu, kp);
    }
    // ---- back to front, two records per iteration (two-lane quadratic form, one
    // butterfly reduction for both).  A is the record nearer the back (processed first).
    // Per lane only MOMENTS of w = G * dL/dG are accumulated (w, w dx, w dy, w dx^2, w dx dy,
    // w dy^2) plus the colour weights; the per-Gaussian factors (conic, opacity, viewport
    // scale) are applied once per (tile, Gaussian) at flush time.  Branch-free: inactive
    // lanes are masked with selects.
#pragma unroll
    for (int k = RB / 32 - 1; k >= 0; --k) {
      unsigned mask = keep[k];
      while (mask) {
        const int bA = 31 - __clz(mask);
        mask &= ~(1u << bA);
        const bool two = mask != 0;
        const int bB = two ? 31 - __clz(mask) : bA;
        mask &= ~(1u << bB);
        const int jA = k * 32 + bA, jB = k * 32 + bB;
        const float4 geA = s_geo[st][jA], geB = s_geo[st][jB];
        const float4 coA = s_attr[st][2 * jA], coB = s_attr[st][2 * jB];
        const float2 dx2 = add2_rn(make_float2(geA.x, geB.x), npx2);
        const float2 dy2 = add2_rn(make_float2(geA.y, geB.y), npy2);
        float2 m1 = mul2_rn(dy2, make_float2(coA.z, coB.z));
        const float2 m2 = mul2_rn(dx2, make_float2(coA.x, coB.x));
        m1 = mul2_rn(dy2, m1);
        const float2 sq = fma2_rn(dx2, m2, m1);
        float2 m3 = mul2_rn(dx2, make_float2(coA.y, coB.y));
        m3 = mul2_rn(dy2, m3);
        const float2 npow = fma2_rn(sq, make_float2(0.5f, 0.5f), m3);  // = -power
        // order-dependent part (scalar): transmittance and the colour behind each record
        float wq[2], atq[2];
        bool contrib = false;
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const float np = q ? npow.y : npow.x;
          const float opac = q ? coB.w : coA.w;
          const int j = q ? jB : jA;
          const float4 col = s_attr[st][2 * j + 1];
          // reference: contributor (0-based position) < last_contributor, power <= 0, alpha >= 1/255
          const bool pre = (q == 0 || two) && (lo + j) < last_contributor && !(np < 0.0f);
          const float G = expf(-np);
          const float alpha = fminf(0.99f, opac * G);
          const bool act = pre && !(alpha < 1.0f / 255.0f);
          contrib |= act;
          const float r = __fdividef(1.0f, 1.0f - alpha);
          const float a_eff = act ? alpha : 0.0f;  // inactive lanes leave every state variable unchanged
          T *= act ? r : 1.0f;
          const float d0 = col.x - accum0, d1 = col.y - accum1, d2 = col.z - accum2;
          float dLa = d0 * dLp0;
          dLa = fmaf(d1, dLp1, dLa);
          dLa = fmaf(d2, dLp2, dLa);
          dLa = fmaf(dLa, T, mTb * r);
          wq[q] = act ? (G * opac) * dLa : 0.0f;
          atq[q] = a_eff * T;
          // colour behind the NEXT record: alpha c + (1 - alpha) accum  (backward.cu:507, evaluated eagerly)
          accum0 = fmaf(a_eff, d0, accum0);
          accum1 = fmaf(a_eff, d1, accum1);
          accum2 = fmaf(a_eff, d2, accum2);
        }
        // moments of w for both records at once (packed).  Component .x is the record this lane's half
        // keeps in the reduction (A on lanes 0-15, B on lanes 16-31), .y the one it hands over.
        float v[2][9];
        {
          const bool up = lane & 16;
          const float2 w2 = up ? make_float2(wq[1], wq[0]) : make_float2(wq[0], wq[1]);
          const float2 at2 = up ? make_float2(atq[1], atq[0]) : make_float2(atq[0], atq[1]);
          const float2 ex2 = up ? make_float2(dx2.y, dx2.x) : dx2;
          const float2 ey2 = up ? make_float2(dy2.y, dy2.x) : dy2;
          const float2 wx = mul2_rn(w2, ex2), wy = mul2_rn(w2, ey2);
          const float2 wxx = mul2_rn(wx, ex2), wxy = mul2_rn(wx, ey2), wyy = mul2_rn(wy, ey2);
          const float2 c0 = mul2_rn(at2, make_float2(dLp0, dLp0)), c1 = mul2_rn(at2, make_float2(dLp1, dLp1)),
                       c2 = mul2_rn(at2, make_float2(dLp2, dLp2));
          v[0][0] = w2.x, v[1][0] = w2.y;
          v[0][1] = wx.x, v[1][1] = wx.y;
          v[0][2] = wy.x, v[1][2] = wy.y;
          v[0][3] = wxx.x, v[1][3] = wxx.y;
          v[0][4] = wxy.x, v[1][4] = wxy.y;
          v[0][5] = wyy.x, v[1][5] = wyy.y;
          v[0][6] = c0.x, v[1][6] = c0.y;
          v[0][7] = c1.x, v[1][7] = c1.y;
          v[0][8] = c2.x, v[1][8] = c2.y;
        }
        if (__any_sync(0xffffffffu, contrib)) {
          float r8, r9;
          warp_reduce_pair(v[0], v[1], lane, r8, r9);
          const int jj = (lane & 16) ? jB : jA;
          float* acc = &s_acc[jj * ACC_STRIDE];
          // a lone record (two == false) reduces against zeros: only its own half is added
          if ((lane & 1) == 0 && (two || !(lane & 16))) atomicAdd(&acc[(lane >> 1) & 7], r8);
          if ((lane & 15) == 1 && (two || !(lane & 16))) atomicAdd(&acc[8], r9);
        }
      }
    }
    __syncthreads();
    // ---- flush this batch: one vector reduction triple per (tile, Gaussian)
    if ((int)tid < cnt) {
      float* acc = &s_acc[tid * ACC_STRIDE];
      float a[9];
      bool nz = false;
#pragma unroll
      for (int q = 0; q < 9; ++q) {
        a[q] = acc[q];
        nz |= (a[q] != 0.f);
        acc[q] = 0.f;
      }
      if (nz) {
        // moments -> gradients (backward.cu:531-554): a[0..5] = sums of w, w dx, w dy, w dx^2, w dx dy, w dy^2
        const float4 con_o = s_attr[st][2 * tid];
        const uint32_t id = __float_as_uint(s_attr[st][2 * tid + 1].w);
        const float g_mx = -ddelx_dx * (con_o.x * a[1] + con_o.y * a[2]);
        const float g_my = -ddely_dy * (con_o.z * a[2] + con_o.y * a[1]);
        const float g_op = (con_o.w != 0.0f) ? a[0] / con_o.w : 0.0f;
        float* dst = reinterpret_cast<float*>(grad_acc + 3 * (size_t)id);
        red_add_v4(dst, g_mx, g_my, -0.5f * a[3], -0.5f * a[4]);
        red_add_v4(dst + 4, -0.5f * a[5], g_op, a[6], a[7]);
        atomicAdd(dst + 8, a[8]);
      }
    }
  }
}

// ===================================================== preprocess (bwd) ====
// SH colour gradient (backward.cu:20-139): returns dL/d(mean) contribution, writes dL_dsh.
__device__ __forceinline__ float3 sh_backward(int deg, const float3 pos, const float3 campos, const float* sh,
                                              const uint8_t* clamped, const float3 dL_dcolor, float* dL_dsh) {
  const float3 dir_orig = make_float3(pos.x - campos.x, pos.y - campos.y, pos.z - campos.z);
  const float len = sqrtf(dir_orig.x * dir_orig.x + dir_orig.y * dir_orig.y + dir_orig.z * dir_orig.z);
  const float x = dir_orig.x / len, y = dir_orig.y / len, z = dir_orig.z / len;
  float dRGB[3] = {dL_dcolor.x, dL_dcolor.y, dL_dcolor.z};
  dRGB[0] *= clamped[0] ? 0 : 1;
  dRGB[1] *= clamped[1] ? 0 : 1;
  dRGB[2] *= clamped[2] ? 0 : 1;
  float ddir[3] = {0.f, 0.f, 0.f};  // dL/d(dir) accumulated over channels
  float w[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) w[k] = 0.f;
  w[0] = kSH0;
  float xx = 0, yy = 0, zz = 0, xy = 0, yz = 0, xz = 0;
  if (deg > 0) {
    w[1] = -kSH1 * y;
    w[2] = kSH1 * z;
    w[3] = -kSH1 * x;
    if (deg > 1) {
      xx = x * x, yy = y * y, zz = z * z;
      xy = x * y, yz = y * z, xz = x * z;
      w[4] = kSH2[0] * xy;
      w[5] = kSH2[1] * yz;
      w[6] = kSH2[2] * (2.f * zz - xx - yy);
      w[7] = kSH2[3] * xz;
      w[8] = kSH2[4] * (xx - yy);
      if (deg > 2) {
        w[9] = kSH3[0] * y * (3.f * xx - yy);
        w[10] = kSH3[1] * xy * z;
        w[11] = kSH3[2] * y * (4.f * zz - xx - yy);
        w[12] = kSH3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy);
        w[13] = kSH3[4] * x * (4.f * zz - xx - yy);
        w[14] = kSH3[5] * z * (xx - yy);
        w[15] = kSH3[6] * x * (xx - 3.f * yy);
      }
    }
  }
  const int ncoef = (deg + 1) * (deg + 1);
#pragma unroll
  for (int k = 0; k < 16; ++k) {
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) dL_dsh[k * 3 + ch] = (k < ncoef) ? w[k] * dRGB[ch] : 0.f;
  }

#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    float dx = 0.f, dy = 0.f, dz = 0.f;
    if (deg > 0) {
      dx = -kSH1 * sh[3 * 3 + ch];
      dy = -kSH1 * sh[1 * 3 + ch];
      dz = kSH1 * sh[2 * 3 + ch];
      if (deg > 1) {
        dx += kSH2[0] * y * sh[4 * 3 + ch] + kSH2[2] * 2.f * -x * sh[6 * 3 + ch] + kSH2[3] * z * sh[7 * 3 + ch] +
              kSH2[4] * 2.f * x * sh[8 * 3 + ch];
        dy += kSH2[0] * x * sh[4 * 3 + ch] + kSH2[1] * z * sh[5 * 3 + ch] + kSH2[2] * 2.f * -y * sh[6 * 3 + ch] +
              kSH2[4] * 2.f * -y * sh[8 * 3 + ch];
        dz += kSH2[1] * y * sh[5 * 3 + ch] + kSH2[2] * 2.f * 2.f * z * sh[6 * 3 + ch] + kSH2[3] * x * sh[7 * 3 + ch];
        if (deg > 2) {
          dx += (kSH3[0] * sh[9 * 3 + ch] * 3.f * 2.f * xy + kSH3[1] * sh[10 * 3 + ch] * yz +
                 kSH3[2] * sh[11 * 3 + ch] * -2.f * xy + kSH3[3] * sh[12 * 3 + ch] * -3.f * 2.f * xz +
                 kSH3[4] * sh[13 * 3 + ch] * (-3.f * xx + 4.f * zz - yy) + kSH3[5] * sh[14 * 3 + ch] * 2.f * xz +
                 kSH3[6] * sh[15 * 3 + ch] * 3.f * (xx - yy));
          dy += (kSH3[0] * sh[9 * 3 + ch] * 3.f * (xx - yy) + kSH3[1] * sh[10 * 3 + ch] * xz +
                 kSH3[2] * sh[11 * 3 + ch] * (-3.f * yy + 4.f * zz - xx) +
                 kSH3[3] * sh[12 * 3 + ch] * -3.f * 2.f * yz + kSH3[4] * sh[13 * 3 + ch] * -2.f * xy +
                 kSH3[5] * sh[14 * 3 + ch] * -2.f * yz + kSH3[6] * sh[15 * 3 + ch] * -3.f * 2.f * xy);
          dz += (kSH3[1] * sh[10 * 3 + ch] * xy + kSH3[2] * sh[11 * 3 + ch] * 4.f * 2.f * yz +
                 kSH3[3] * sh[12 * 3 + ch] * 3.f * (2.f * zz - xx - yy) +
                 kSH3[4] * sh[13 * 3 + ch] * 4.f * 2.f * xz + kSH3[5] * sh[14 * 3 + ch] * (xx - yy));
        }
      }
    }
    ddir[0] += dx * dRGB[ch];
    ddir[1] += dy * dRGB[ch];
    ddir[2] += dz * dRGB[ch];
  }
  // through the normalisation dir = v / |v| (auxiliary.h:112-122)
  const float3 vv = dir_orig;
  const float sum2 = vv.x * vv.x + vv.y * vv.y + vv.z * vv.z;
  const float invsum32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
  float3 r;
  r.x = ((+sum2 - vv.x * vv.x) * ddir[0] - vv.y * vv.x * ddir[1] - vv.z * vv.x * ddir[2]) * invsum32;
  r.y = (-vv.x * vv.y * ddir[0] + (sum2 - vv.y * vv.y) * ddir[1] - vv.z * vv.y * ddir[2]) * invsum32;
  r.z = (-vv.x * vv.z * ddir[0] - vv.y * vv.z * ddir[1] + (sum2 - vv.z * vv.z) * ddir[2]) * invsum32;
  return r;
}

// write v, or add it to what the buffer holds (never reads the buffer unless accumulating)
__device__ __forceinline__ void acc_store(float* p, float v, int accumulate) { *p = accumulate ? *p + v : v; }

// `accumulate` bits (DGR_PF_* of include/dgmesh_b200.h): which parameter-gradient outputs are summed
#define ACC_MEANS 1
#define ACC_SCALES 2
#define ACC_ROTS 4
#define ACC_OPAC 8
#define ACC_COLOR 16  // dL_dsh / dL_dcolor
#define ACC_COV 32
#define ACC_ALL 63

__global__ void __launch_bounds__(128) preprocess_bwd_kernel(
    int P, int D, int M, const float* __restrict__ means3D, const int* __restrict__ radii,
    const float* __restrict__ shs, const float* __restrict__ scales, const float* __restrict__ rotations,
    float scale_modifier, const float* __restrict__ cov3D_precomp, const float* __restrict__ view,
    const float* __restrict__ proj, float focal_x, float focal_y, float tan_fovx, float tan_fovy,
    const float* __restrict__ cam_pos, GeomWS g, float* __restrict__ dL_dmean2D, float* __restrict__ dL_dconic,
    float* __restrict__ dL_dopacity, float* __restrict__ dL_dcolor, float* __restrict__ dL_dmean3D,
    float* __restrict__ dL_dcov3D, float* __restrict__ dL_dsh, float* __restrict__ dL_dscale,
    float* __restrict__ dL_drot, int accumulate) {
  pdl_wait();
  pdl_launch();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= P) return;
  const bool visible = radii[idx] > 0;
  // fetch + clear the accumulators written by render_bwd_kernel
  const float4 a0 = g.grad_acc[3 * idx + 0], a1 = g.grad_acc[3 * idx + 1], a2 = g.grad_acc[3 * idx + 2];
  g.grad_acc[3 * idx + 0] = make_float4(0, 0, 0, 0);
  g.grad_acc[3 * idx + 1] = make_float4(0, 0, 0, 0);
  g.grad_acc[3 * idx + 2] = make_float4(0, 0, 0, 0);
  const float2 dm2 = make_float2(a0.x, a0.y);
  const float3 dcon = make_float3(a0.z, a0.w, a1.x);  // (xx, xy, yy) slots .x .y .w of the reference float4
  const float dop = a1.y;
  const float3 dcol = make_float3(a1.z, a1.w, a2.x);

  dL_dmean2D[3 * idx + 0] = dm2.x;
  dL_dmean2D[3 * idx + 1] = dm2.y;
  dL_dmean2D[3 * idx + 2] = 0.f;
  if (dL_dconic) reinterpret_cast<float4*>(dL_dconic)[idx] = make_float4(dcon.x, dcon.y, 0.f, dcon.z);
  // parameter gradients: written, or (frame batches) added to the running sum over frames
  if (accumulate == ACC_ALL && !visible) return;  // a culled Gaussian adds nothing
  acc_store(&dL_dopacity[idx], dop, accumulate & ACC_OPAC);
  acc_store(&dL_dcolor[3 * idx + 0], dcol.x, accumulate & ACC_COLOR);
  acc_store(&dL_dcolor[3 * idx + 1], dcol.y, accumulate & ACC_COLOR);
  acc_store(&dL_dcolor[3 * idx + 2], dcol.z, accumulate & ACC_COLOR);

  float dcov[6] = {0, 0, 0, 0, 0, 0};
  float3 dmean = make_float3(0, 0, 0);
  float3 dscale = make_float3(0, 0, 0);
  float4 drot = make_float4(0, 0, 0, 0);

  if (!visible) {
    if (dL_dsh && !(accumulate & ACC_COLOR)) {
      float* dst = dL_dsh + (size_t)idx * M * 3;
      if (M == 16) {
#pragma unroll
        for (int i = 0; i < 12; ++i) reinterpret_cast<float4*>(dst)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      } else {
        for (int k = 0; k < M * 3; ++k) dst[k] = 0.f;
      }
    }
  } else {
    const float3 mean = make_float3(means3D[3 * idx], means3D[3 * idx + 1], means3D[3 * idx + 2]);
    const float* cov3D = cov3D_precomp ? cov3D_precomp + 6 * idx : g.cov3D + 6 * idx;
    // ---------------- gradient through the 2D covariance / conic (backward.cu:144-274)
    EwaFrame fr;
    ewa_frame(mean, focal_x, focal_y, tan_fovx, tan_fovy, cov3D, view, fr);
    const float limx = 1.3f * tan_fovx, limy = 1.3f * tan_fovy;
    const float x_grad_mul = fr.txtz < -limx || fr.txtz > limx ? 0 : 1;
    const float y_grad_mul = fr.tytz < -limy || fr.tytz > limy ? 0 : 1;
    const float3 c2 = ewa_cov2d(fr);
    const float a = c2.x, b = c2.y, c = c2.z;
    const float denom = a * c - b * b;
    float dL_da = 0, dL_db = 0, dL_dc = 0;
    const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
    const Mat3& T = fr.T;
    const Mat3& Vrk = fr.Vrk;
    if (denom2inv != 0) {
      dL_da = denom2inv * (-c * c * dcon.x + 2 * b * c * dcon.y + (denom - a * c) * dcon.z);
      dL_dc = denom2inv * (-a * a * dcon.z + 2 * a * b * dcon.y + (denom - a * c) * dcon.x);
      dL_db = denom2inv * 2 * (b * c * dcon.x - (denom + 2 * b * b) * dcon.y + a * b * dcon.z);
      dcov[0] = (T.c[0][0] * T.c[0][0] * dL_da + T.c[0][0] * T.c[1][0] * dL_db + T.c[1][0] * T.c[1][0] * dL_dc);
      dcov[3] = (T.c[0][1] * T.c[0][1] * dL_da + T.c[0][1] * T.c[1][1] * dL_db + T.c[1][1] * T.c[1][1] * dL_dc);
      dcov[5] = (T.c[0][2] * T.c[0][2] * dL_da + T.c[0][2] * T.c[1][2] * dL_db + T.c[1][2] * T.c[1][2] * dL_dc);
      dcov[1] = 2 * T.c[0][0] * T.c[0][1] * dL_da + (T.c[0][0] * T.c[1][1] + T.c[0][1] * T.c[1][0]) * dL_db +
                2 * T.c[1][0] * T.c[1][1] * dL_dc;
      dcov[2] = 2 * T.c[0][0] * T.c[0][2] * dL_da + (T.c[0][0] * T.c[1][2] + T.c[0][2] * T.c[1][0]) * dL_db +
                2 * T.c[1][0] * T.c[1][2] * dL_dc;
      dcov[4] = 2 * T.c[0][2] * T.c[0][1] * dL_da + (T.c[0][1] * T.c[1][2] + T.c[0][2] * T.c[1][1]) * dL_db +
                2 * T.c[1][1] * T.c[1][2] * dL_dc;
    }
    const float dL_dT00 = 2 * (T.c[0][0] * Vrk.c[0][0] + T.c[0][1] * Vrk.c[0][1] + T.c[0][2] * Vrk.c[0][2]) * dL_da +
                          (T.c[1][0] * Vrk.c[0][0] + T.c[1][1] * Vrk.c[0][1] + T.c[1][2] * Vrk.c[0][2]) * dL_db;
    const float dL_dT01 = 2 * (T.c[0][0] * Vrk.c[1][0] + T.c[0][1] * Vrk.c[1][1] + T.c[0][2] * Vrk.c[1][2]) * dL_da +
                          (T.c[1][0] * Vrk.c[1][0] + T.c[1][1] * Vrk.c[1][1] + T.c[1][2] * Vrk.c[1][2]) * dL_db;
    const float dL_dT02 = 2 * (T.c[0][0] * Vrk.c[2][0] + T.c[0][1] * Vrk.c[2][1] + T.c[0][2] * Vrk.c[2][2]) * dL_da +
                          (T.c[1][0] * Vrk.c[2][0] + T.c[1][1] * Vrk.c[2][1] + T.c[1][2] * Vrk.c[2][2]) * dL_db;
    const float dL_dT10 = 2 * (T.c[1][0] * Vrk.c[0][0] + T.c[1][1] * Vrk.c[0][1] + T.c[1][2] * Vrk.c[0][2]) * dL_dc +
                          (T.c[0][0] * Vrk.c[0][0] + T.c[0][1] * Vrk.c[0][1] + T.c[0][2] * Vrk.c[0][2]) * dL_db;
    const float dL_dT11 = 2 * (T.c[1][0] * Vrk.c[1][0] + T.c[1][1] * Vrk.c[1][1] + T.c[1][2] * Vrk.c[1][2]) * dL_dc +
                          (T.c[0][0] * Vrk.c[1][0] + T.c[0][1] * Vrk.c[1][1] + T.c[0][2] * Vrk.c[1][2]) * dL_db;
    const float dL_dT12 = 2 * (T.c[1][0] * Vrk.c[2][0] + T.c[1][1] * Vrk.c[2][1] + T.c[1][2] * Vrk.c[2][2]) * dL_dc +
                          (T.c[0][0] * Vrk.c[2][0] + T.c[0][1] * Vrk.c[2][1] + T.c[0][2] * Vrk.c[2][2]) * dL_db;
    const Mat3& Wm = fr.W;
    const float dL_dJ00 = Wm.c[0][0] * dL_dT00 + Wm.c[0][1] * dL_dT01 + Wm.c[0][2] * dL_dT02;
    const float dL_dJ02 = Wm.c[2][0] * dL_dT00 + Wm.c[2][1] * dL_dT01 + Wm.c[2][2] * dL_dT02;
    const float dL_dJ11 = Wm.c[1][0] * dL_dT10 + Wm.c[1][1] * dL_dT11 + Wm.c[1][2] * dL_dT12;
    const float dL_dJ12 = Wm.c[2][0] * dL_dT10 + Wm.c[2][1] * dL_dT11 + Wm.c[2][2] * dL_dT12;
    const float tz = 1.f / fr.t.z;
    const float tz2 = tz * tz;
    const float tz3 = tz2 * tz;
    const float dL_dtx = x_grad_mul * -focal_x * tz2 * dL_dJ02;
    const float dL_dty = y_grad_mul * -focal_y * tz2 * dL_dJ12;
    const float dL_dtz = -focal_x * tz2 * dL_dJ00 - focal_y * tz2 * dL_dJ11 + (2 * focal_x * fr.t.x) * tz3 * dL_dJ02 +
                         (2 * focal_y * fr.t.y) * tz3 * dL_dJ12;
    dmean = xform_vec4x3_T(make_float3(dL_dtx, dL_dty, dL_dtz), view);

    // ---------------- screen-space mean -> 3D mean (backward.cu:366-381)
    const float4 m_hom = xform4x4(mean, proj);
    const float m_w = 1.0f / (m_hom.w + 0.0000001f);
    const float mul1 = (proj[0] * mean.x + proj[4] * mean.y + proj[8] * mean.z + proj[12]) * m_w * m_w;
    const float mul2 = (proj[1] * mean.x + proj[5] * mean.y + proj[9] * mean.z + proj[13]) * m_w * m_w;
    float3 dm;
    dm.x = (proj[0] * m_w - proj[3] * mul1) * dm2.x + (proj[1] * m_w - proj[3] * mul2) * dm2.y;
    dm.y = (proj[4] * m_w - proj[7] * mul1) * dm2.x + (proj[5] * m_w - proj[7] * mul2) * dm2.y;
    dm.z = (proj[8] * m_w - proj[11] * mul1) * dm2.x + (proj[9] * m_w - proj[11] * mul2) * dm2.y;
    dmean.x += dm.x;
    dmean.y += dm.y;
    dmean.z += dm.z;

    // ---------------- SH colour (backward.cu:20-139, 383-385)
    if (shs) {
      const float3 cp = make_float3(cam_pos[0], cam_pos[1], cam_pos[2]);
      float sh[48], dsh[48];
      load_sh(shs, idx, M, (D + 1) * (D + 1), sh);
      const float3 dms = sh_backward(D, mean, cp, sh, g.clamped + 3 * idx, dcol, dsh);
      dmean.x += dms.x;
      dmean.y += dms.y;
      dmean.z += dms.z;
      float* dst = dL_dsh + (size_t)idx * M * 3;
      if (M == 16) {
#pragma unroll
        for (int i = 0; i < 12; ++i) {
          float4 o = make_float4(dsh[4 * i], dsh[4 * i + 1], dsh[4 * i + 2], dsh[4 * i + 3]);
          if (accumulate & ACC_COLOR) {
            const float4 old = reinterpret_cast<float4*>(dst)[i];
            o.x += old.x, o.y += old.y, o.z += old.z, o.w += old.w;
          }
          reinterpret_cast<float4*>(dst)[i] = o;
        }
      } else {
#pragma unroll
        for (int i = 0; i < 48; ++i)
          if (i < M * 3) acc_store(&dst[i], dsh[i], accumulate & ACC_COLOR);
      }
    }
    // ---------------- 3D covariance -> scale / rotation (backward.cu:279-341)
    if (scales) {
      const float3 sc = make_float3(scales[3 * idx], scales[3 * idx + 1], scales[3 * idx + 2]);
      const float4 q = __ldg(reinterpret_cast<const float4*>(rotations) + idx);
      const float r = q.x, x = q.y, y = q.z, z = q.w;
      Mat3 R;
      quat_to_R(q, R);
      const float3 s = make_float3(scale_modifier * sc.x, scale_modifier * sc.y, scale_modifier * sc.z);
      Mat3 S;
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) S.c[i][j] = (i == j) ? 1.0f : 0.0f;
      S.c[0][0] = s.x;
      S.c[1][1] = s.y;
      S.c[2][2] = s.z;
      const Mat3 Mm = mat3_mul(S, R);
      Mat3 dSig;
      dSig.c[0][0] = dcov[0];
      dSig.c[0][1] = 0.5f * dcov[1];
      dSig.c[0][2] = 0.5f * dcov[2];
      dSig.c[1][0] = 0.5f * dcov[1];
      dSig.c[1][1] = dcov[3];
      dSig.c[1][2] = 0.5f * dcov[4];
      dSig.c[2][0] = 0.5f * dcov[2];
      dSig.c[2][1] = 0.5f * dcov[4];
      dSig.c[2][2] = dcov[5];
      Mat3 M2;
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) M2.c[i][j] = 2.0f * Mm.c[i][j];
      const Mat3 dL_dM = mat3_mul(M2, dSig);
      const Mat3 Rt = mat3_T(R);
      Mat3 dMt = mat3_T(dL_dM);
      dscale.x = Rt.c[0][0] * dMt.c[0][0] + Rt.c[0][1] * dMt.c[0][1] + Rt.c[0][2] * dMt.c[0][2];
      dscale.y = Rt.c[1][0] * dMt.c[1][0] + Rt.c[1][1] * dMt.c[1][1] + Rt.c[1][2] * dMt.c[1][2];
      dscale.z = Rt.c[2][0] * dMt.c[2][0] + Rt.c[2][1] * dMt.c[2][1] + Rt.c[2][2] * dMt.c[2][2];
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        dMt.c[0][j] *= s.x;
        dMt.c[1][j] *= s.y;
        dMt.c[2][j] *= s.z;
      }
      drot.x = 2 * z * (dMt.c[0][1] - dMt.c[1][0]) + 2 * y * (dMt.c[2][0] - dMt.c[0][2]) +
               2 * x * (dMt.c[1][2] - dMt.c[2][1]);
      drot.y = 2 * y * (dMt.c[1][0] + dMt.c[0][1]) + 2 * z * (dMt.c[2][0] + dMt.c[0][2]) +
               2 * r * (dMt.c[1][2] - dMt.c[2][1]) - 4 * x * (dMt.c[2][2] + dMt.c[1][1]);
      drot.z = 2 * x * (dMt.c[1][0] + dMt.c[0][1]) + 2 * r * (dMt.c[2][0] - dMt.c[0][2]) +
               2 * z * (dMt.c[1][2] + dMt.c[2][1]) - 4 * y * (dMt.c[2][2] + dMt.c[0][0]);
      drot.w = 2 * r * (dMt.c[0][1] - dMt.c[1][0]) + 2 * x * (dMt.c[2][0] + dMt.c[0][2]) +
               2 * y * (dMt.c[1][2] + dMt.c[2][1]) - 4 * z * (dMt.c[1][1] + dMt.c[0][0]);
    }
  }
  acc_store(&dL_dmean3D[3 * idx + 0], dmean.x, accumulate & ACC_MEANS);
  acc_store(&dL_dmean3D[3 * idx + 1], dmean.y, accumulate & ACC_MEANS);
  acc_store(&dL_dmean3D[3 * idx + 2], dmean.z, accumulate & ACC_MEANS);
#pragma unroll
  for (int k = 0; k < 6; ++k) acc_store(&dL_dcov3D[6 * idx + k], dcov[k], accumulate & ACC_COV);
  acc_store(&dL_dscale[3 * idx + 0], dscale.x, accumulate & ACC_SCALES);
  acc_store(&dL_dscale[3 * idx + 1], dscale.y, accumulate & ACC_SCALES);
  acc_store(&dL_dscale[3 * idx + 2], dscale.z, accumulate & ACC_SCALES);
  {
    float4 o = drot;
    if (accumulate & ACC_ROTS) {
      const float4 old = reinterpret_cast<float4*>(dL_drot)[idx];
      o.x += old.x, o.y += old.y, o.z += old.z, o.w += old.w;
    }
    reinterpret_cast<float4*>(dL_drot)[idx] = o;
  }
}

cudaError_t launch_backward(const BwdArgs& a, cudaStream_t s) {
  cudaError_t e = launch_render_bwd(a, s);
  return e != cudaSuccess ? e : launch_preprocess_bwd(a, s);
}

// gradient of the alpha-compositing (fills the GPU); leaves the per-Gaussian moments in grad_acc
cudaError_t launch_render_bwd(const BwdArgs& a, cudaStream_t s) {
  if (a.P == 0) return cudaSuccess;
  const unsigned gx = (a.W + TILE_X - 1) / TILE_X, gy = (a.H + TILE_Y - 1) / TILE_Y;
  const int T = gx * gy;
  GeomWS g = GeomWS::from((char*)a.geom_ws, a.P);
  ImgWS im = ImgWS::from((char*)a.img_ws, (size_t)a.W * a.H, T);
  BinWS b = BinWS::from((char*)a.binning_ws, (size_t)a.R_cap);
  g_prof.begin(5, s);
  launch_pdl(render_bwd_kernel, dim3(T), dim3(256), 0, s, (const uint2*)im.ranges, (const uint32_t*)im.tile_order,
             (const float4*)b.inst_geo, (const float4*)b.inst_attr, a.W, a.H, a.background, (const float*)im.final_T,
             (const uint32_t*)im.n_contrib, a.dL_dpix, g.grad_acc);
  g_prof.end(5, s);
  return cudaGetLastError();
}

// chain rule from the moments to the inputs (short); with a.accumulate it adds to the outputs, so
// the calls of a frame batch must be ordered (same stream)
cudaError_t launch_preprocess_bwd(const BwdArgs& a, cudaStream_t s) {
  if (a.P == 0) return cudaSuccess;
  GeomWS g = GeomWS::from((char*)a.geom_ws, a.P);
  const float focal_y = a.H / (2.0f * a.tan_fovy);
  const float focal_x = a.W / (2.0f * a.tan_fovx);
  const int* radii = a.radii ? a.radii : g.radii;
  g_prof.begin(6, s);
  launch_pdl(preprocess_bwd_kernel, dim3((a.P + 127) / 128), dim3(128), 0, s, a.P, a.D, a.M, a.means3D, radii, a.shs,
             a.scales, a.rotations, a.scale_modifier, a.cov3D_precomp, a.viewmatrix, a.projmatrix, focal_x, focal_y,
             a.tan_fovx, a.tan_fovy, a.cam_pos, g, a.dL_dmean2D, a.dL_dconic, a.dL_dopacity, a.dL_dcolor, a.dL_dmean3D,
             a.dL_dcov3D, a.dL_dsh, a.dL_dscale, a.dL_drot, a.accumulate);
  g_prof.end(6, s);
  return cudaGetLastError();
}

}  // namespace dgm
