// raster_bwd.cu -- backward pass of the tile-based 3D-Gaussian rasterizer for sm_90a.
//
//   render_bwd_kernel      gradient of the alpha-composite (role of renderCUDA,
//                          dgr/cuda_rasterizer/backward.cu:399-557)
//   preprocess_bwd_kernel  chain rule to means3D / scales / rotations / SH / opacity
//                          (computeCov2DCUDA + preprocessCUDA, backward.cu:144-396, fused), one
//                          launch for all frames of a batch
//
// The reference issues 9 global float atomics per contributing (pixel, Gaussian)
// pair.  Here the per-Gaussian gradient is written as nine pixel sums over each warp's
// 8x4 block: six moments of w = G * dL/dG (w, w dx, w dy, w dx^2, w dx dy, w dy^2) and
// three colour weights.  Each moment is a polynomial in the pixel's offset (u, v) from
// the block centre, so a lane only stages its two scalars (w, alpha T) per record in
// shared memory; once per chunk of records the warp contracts them (one record per lane
// pair, against the fixed u, v and the staged dL/dpixel) and adds the nine sums into a
// per-tile shared-memory accumulator.  The tile flushes once per (tile, Gaussian) with
// vector reductions (red.global.add.v4.f32) into a [P,12] accumulator that the fused
// preprocess-backward consumes and re-zeroes (render_bwd_kernel<true> also forms dL/d(depth) of the depth map,
// a fourth colour weight, into float 9).  The per-pair arithmetic follows the
// reference's back-to-front recurrence; only the summation order differs (the
// reference's own order is non-deterministic).
#include "../../include/dgmesh_b200.h"
#include "common.cuh"
#include "raster_math.cuh"
#include "raster_kernels.h"

namespace dgm {

#define RB 256          // records per TMA batch
#define CHUNK 16        // records a warp stages before contracting them
#define SLOT_F 68       // floats per staged record: w[32], alpha T[32], and 16 B that put the 16 slots in distinct banks
#define STAGE_BYTES (8 * CHUNK * SLOT_F * 4)  // dynamic shared memory: one staging area per warp

// floats per record in the per-tile accumulator: the nine sums, + dL/d(depth) with depth and alpha
template <bool AUX> constexpr int acc_stride() { return AUX ? 10 : 9; }

// Contract the first n staged records of a warp into s_acc.  Slot k holds w and alpha T of the 32 pixels
// (pixel = lane of the staging warp: column lane & 7, row lane >> 3) of record `rec` (held by lanes k and
// k + 16).  Lane l sums slot l & 15 over pixel rows 2h, 2h+1, h = l >> 4, as pixel offsets u, v from the
// block centre (exact in fp32), then expands the moments about the Gaussian's offset (Gx, Gy) from that
// centre: sum w dx = Gx S_1 - S_u, sum w dx^2 = Gx^2 S_1 - 2 Gx S_u + S_uu, ...  The two lanes of a slot
// trade half of their nine partial sums, so each adds 5 or 4 totals (shared-memory float atomics are
// compare-and-swap loops on sm_90).  Every lane computes; only the lanes of the n filled slots add.
// AUX: dlp has a fourth row, dL/d(depth); its weight sum alpha T dL/dD is the tenth total (slot 9), added
// by lane h = 1, which then adds 5 totals too.
template <bool AUX>
__device__ __forceinline__ void contract_chunk(const float* stage, const float* dlp, int n, int rec, unsigned lane,
                                               const float4* geo, float cx, float cy, float* s_acc) {
  constexpr int NCH = AUX ? 4 : 3;
  const int k = lane & 15, h = lane >> 4;
  const float4* w4 = reinterpret_cast<const float4*>(stage + k * SLOT_F + 16 * h);  // w of this half's 16 pixels
  const float4* a4 = w4 + 8;                                                        // alpha T of the same
  const float4* d4 = reinterpret_cast<const float4*>(dlp + 16 * h);                 // dlp is [NCH][32]
  float c[NCH];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 t = a4[i];
    const float at[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) {
      const float4 e = d4[8 * ch + i];
      const float dl[4] = {e.x, e.y, e.z, e.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) c[ch] = (i == 0 && j == 0) ? at[j] * dl[j] : fmaf(at[j], dl[j], c[ch]);
    }
  }
  // per pixel row r: pixels 8r .. 8r+7 of this half at u = -3.5 .. 3.5, folded about the centre column
  float sw[2], su[2], suu[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const float4 p = w4[2 * r], q = w4[2 * r + 1];
    const float w[8] = {p.x, p.y, p.z, p.w, q.x, q.y, q.z, q.w};
    float a[4], d[4];  // w(u) + w(-u), w(u) - w(-u) for u = m + 0.5
#pragma unroll
    for (int m = 0; m < 4; ++m) a[m] = w[4 + m] + w[3 - m], d[m] = w[4 + m] - w[3 - m];
    sw[r] = (a[0] + a[1]) + (a[2] + a[3]);
    su[r] = fmaf(3.5f, d[3], fmaf(2.5f, d[2], fmaf(1.5f, d[1], 0.5f * d[0])));
    suu[r] = fmaf(12.25f, a[3], fmaf(6.25f, a[2], fmaf(2.25f, a[1], 0.25f * a[0])));
  }
  const float v0 = 2 * h - 1.5f, v1 = 2 * h - 0.5f;
  const float S1 = sw[0] + sw[1], Su = su[0] + su[1], Suu = suu[0] + suu[1];
  const float Sv = fmaf(v1, sw[1], v0 * sw[0]), Suv = fmaf(v1, su[1], v0 * su[0]);
  const float Svv = fmaf(v1 * v1, sw[1], (v0 * v0) * sw[0]);
  const float4 g = geo[rec];
  const float Gx = g.x - cx, Gy = g.y - cy;
  const float my = fmaf(Gy, S1, -Sv);
  const float m[10] = {S1, fmaf(Gx, S1, -Su), my, fmaf(Gx, fmaf(Gx, S1, -2.0f * Su), Suu),
                       fmaf(Gx, my, fmaf(-Gy, Su, Suv)), fmaf(Gy, fmaf(Gy, S1, -2.0f * Sv), Svv),
                       c[0], c[1], c[2], AUX ? c[NCH - 1] : 0.0f};
  float* acc = &s_acc[rec * acc_stride<AUX>() + 5 * h];  // lane h = 0 adds moments 0-4, h = 1 moments 5-8 (9)
#pragma unroll
  for (int q = 0; q < 5; ++q) {
    const float keep = h ? m[q + 5] : m[q], send = h ? m[q] : m[q + 5];
    const float tot = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    if (k < n && (AUX || q < 4 || h == 0)) atomicAdd(&acc[q], tot);
  }
}

// AUX: the upstream gradients of the depth map (needs the records of a depth forward: depth in .w) and of
// the alpha map, each NULL when the loss does not use it.  dL/d(depth_i) goes to float 9 of grad_acc.
template <bool AUX>
__global__ void __launch_bounds__(256, AUX ? 2 : 3) render_bwd_kernel(
    const uint2* __restrict__ ranges, const uint32_t* __restrict__ tile_order, const float4* __restrict__ inst_geo,
    const float4* __restrict__ inst_attr,
    int W, int H, const float* __restrict__ bg_color, const float* __restrict__ final_Ts,
    const uint32_t* __restrict__ n_contrib, const float* __restrict__ dL_dpixels, float4* __restrict__ grad_acc,
    const float* __restrict__ dL_ddepth, const float* __restrict__ dL_dalpha) {
  constexpr int ACC_STRIDE = acc_stride<AUX>();
  __shared__ __align__(128) float4 s_geo[2][RB];
  __shared__ __align__(128) float4 s_attr[2][2 * RB];
  __shared__ float s_acc[RB * ACC_STRIDE];
  __shared__ __align__(16) float s_dlp[8][AUX ? 4 : 3][32];  // dL/dpixel of each warp's 32 pixels, per colour (+ depth)
  __shared__ __align__(8) uint64_t s_bar[2];
  __shared__ int s_maxc;
  extern __shared__ __align__(16) float s_stage[];  // [8 warps][CHUNK][SLOT_F]

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
  const float cx = wx0 + 3.5f, cy = wy0 + 1.5f;  // centre of the warp's block
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

  float dLp0 = 0.f, dLp1 = 0.f, dLp2 = 0.f, dLD = 0.f, dLA = 0.f;
  if (inside) {
    const size_t HW = (size_t)H * W;
    dLp0 = dL_dpixels[0 * HW + pix_id];
    dLp1 = dL_dpixels[1 * HW + pix_id];
    dLp2 = dL_dpixels[2 * HW + pix_id];
    if (AUX && dL_ddepth) dLD = dL_ddepth[pix_id];
    if (AUX && dL_dalpha) dLA = dL_dalpha[pix_id];
  }
  s_dlp[wid][0][lane] = dLp0;
  s_dlp[wid][1][lane] = dLp1;
  s_dlp[wid][2][lane] = dLp2;
  if (AUX) s_dlp[wid][AUX ? 3 : 0][lane] = dLD;
  float* const stage = s_stage + wid * (CHUNK * SLOT_F);
  int nslot = 0, rec = 0;  // staged records; the record of slot lane & 15
  float bg_dot_dpixel = 0;
  bg_dot_dpixel += bg_color[0] * dLp0;
  bg_dot_dpixel += bg_color[1] * dLp1;
  bg_dot_dpixel += bg_color[2] * dLp2;

  // background term of dL/dalpha, times 1/(1-alpha) per record; the alpha map A = 1 - T_final adds
  // dL/dA T_final / (1 - alpha) in the same form
  const float mTb = -T_final * (AUX ? bg_dot_dpixel - dLA : bg_dot_dpixel);
  float accum0 = 0.f, accum1 = 0.f, accum2 = 0.f;  // colour composited behind the current record
  float accumD = 0.f;                              // depth composited behind it (AUX only)

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
    // ---- cull (same conservative extent test as the forward pass); lane k keeps the ballot of
    // records [32k, 32k + 32), so that the k loop below stays rolled and its body (with the
    // contraction) is emitted once
    unsigned keep_k = 0;
#pragma unroll
    for (int k = 0; k < RB / 32; ++k) {
      const int r = k * 32 + lane;
      bool kp = false;
      if (r < cnt && (lo + r) < wmax) {
        kp = cull_keep(s_geo[st][r], s_attr[st][2 * r], bx0, bx1, by0, by1);
      }
      const unsigned b = __ballot_sync(0xffffffffu, kp);
      if (lane == k) keep_k = b;
    }
    // ---- back to front, two records per iteration (two-lane quadratic form).  A is the record
    // nearer the back (processed first).  Per lane only w = G * dL/dG and alpha T are formed and
    // staged; the moments are formed by contract_chunk, the per-Gaussian factors (conic, opacity,
    // viewport scale) once per (tile, Gaussian) at flush time.  Branch-free: inactive lanes are
    // masked with selects.
#pragma unroll 1
    for (int k = RB / 32 - 1; k >= 0; --k) {
      unsigned mask = __shfl_sync(0xffffffffu, keep_k, k);
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
          const float r = __fdividef(1.0f, 1.0f - alpha);
          const float a_eff = act ? alpha : 0.0f;  // inactive lanes leave every state variable unchanged
          T *= act ? r : 1.0f;
          const float d0 = col.x - accum0, d1 = col.y - accum1, d2 = col.z - accum2;
          const float dD = AUX ? s_geo[st][j].w - accumD : 0.0f;
          float dLa = d0 * dLp0;
          dLa = fmaf(d1, dLp1, dLa);
          dLa = fmaf(d2, dLp2, dLa);
          if (AUX) dLa = fmaf(dD, dLD, dLa);
          dLa = fmaf(dLa, T, mTb * r);
          const float w = act ? (G * opac) * dLa : 0.0f;
          // colour behind the NEXT record: alpha c + (1 - alpha) accum  (backward.cu:507, evaluated eagerly)
          accum0 = fmaf(a_eff, d0, accum0);
          accum1 = fmaf(a_eff, d1, accum1);
          accum2 = fmaf(a_eff, d2, accum2);
          if (AUX) accumD = fmaf(a_eff, dD, accumD);
          // only records with a contributing lane take a slot (the others add exact zeros)
          if (__any_sync(0xffffffffu, act)) {
            stage[nslot * SLOT_F + lane] = w;
            stage[nslot * SLOT_F + 32 + lane] = a_eff * T;
            if ((int)(lane & 15) == nslot) rec = j;
            ++nslot;
          }
        }
        if (nslot > CHUNK - 2) {  // no room for another pair
          __syncwarp();
          contract_chunk<AUX>(stage, &s_dlp[wid][0][0], nslot, rec, lane, s_geo[st], cx, cy, s_acc);
          __syncwarp();
          nslot = 0;
        }
      }
    }
    if (nslot > 0) {  // the batch's records must be in s_acc before the flush
      __syncwarp();
      contract_chunk<AUX>(stage, &s_dlp[wid][0][0], nslot, rec, lane, s_geo[st], cx, cy, s_acc);
      nslot = 0;
    }
    __syncthreads();
    // ---- flush this batch: one vector reduction triple per (tile, Gaussian)
    if ((int)tid < cnt) {
      float* acc = &s_acc[tid * ACC_STRIDE];
      float a[ACC_STRIDE];
      bool nz = false;
#pragma unroll
      for (int q = 0; q < ACC_STRIDE; ++q) {
        a[q] = acc[q];
        nz |= (a[q] != 0.f);
        acc[q] = 0.f;
      }
      if (nz) {
        // moments -> gradients (backward.cu:531-554): a[0..5] = sums of w, w dx, w dy, w dx^2, w dx dy, w dy^2
        // d(pixel coordinate)/d(NDC), backward.cu:457-458 (double literal 0.5)
        const float ddelx_dx = 0.5 * W;
        const float ddely_dy = 0.5 * H;
        const float4 con_o = s_attr[st][2 * tid];
        const uint32_t id = __float_as_uint(s_attr[st][2 * tid + 1].w);
        const float g_mx = -ddelx_dx * (con_o.x * a[1] + con_o.y * a[2]);
        const float g_my = -ddely_dy * (con_o.z * a[2] + con_o.y * a[1]);
        const float g_op = (con_o.w != 0.0f) ? a[0] / con_o.w : 0.0f;
        float* dst = reinterpret_cast<float*>(grad_acc + 3 * (size_t)id);
        red_add_v4(dst, g_mx, g_my, -0.5f * a[3], -0.5f * a[4]);
        red_add_v4(dst + 4, -0.5f * a[5], g_op, a[6], a[7]);
        if (AUX) red_add_v2(dst + 8, a[8], a[AUX ? 9 : 8]);
        else atomicAdd(dst + 8, a[8]);
      }
    }
  }
}

// ===================================================== preprocess (bwd) ====
// SH colour gradient (backward.cu:20-139): returns dL/d(mean) contribution.  dL/dsh is the outer product
// dL_dsh[k][ch] = w[k] * dRGB[ch] (w[k] = 0 for k >= (deg + 1)^2); the caller forms it from the two factors.
__device__ __forceinline__ float3 sh_backward(int deg, const float3 pos, const float3 campos, const float* sh,
                                              const uint8_t* clamped, const float3 dL_dcolor, float* w /*[16]*/,
                                              float* dRGB /*[3]*/) {
  const float3 dir_orig = make_float3(pos.x - campos.x, pos.y - campos.y, pos.z - campos.z);
  const float len = sqrtf(dir_orig.x * dir_orig.x + dir_orig.y * dir_orig.y + dir_orig.z * dir_orig.z);
  const float x = dir_orig.x / len, y = dir_orig.y / len, z = dir_orig.z / len;
  dRGB[0] = dL_dcolor.x * (clamped[0] ? 0 : 1);
  dRGB[1] = dL_dcolor.y * (clamped[1] ? 0 : 1);
  dRGB[2] = dL_dcolor.z * (clamped[2] ? 0 : 1);
  float ddir[3] = {0.f, 0.f, 0.f};  // dL/d(dir) accumulated over channels
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

// ---- per-Gaussian backward of a frame batch (F = 1: one frame).  A block covers NG Gaussians x FB frames per
// pass (FB * NG = NT): warp w takes 32 consecutive Gaussians of frame f0 + w % FB, so per-frame slabs load
// coalesced.  Every output is staged per (frame, Gaussian) in shared memory and written as rows of consecutive
// floats (every store of a warp covers 128 consecutive bytes): gradients of per-frame inputs by the warp that
// staged them, to the frame's slab; gradients of inputs shared by the frames by the whole block once per pass,
// summed over the frames in frame order f = 0, 1, ..., F - 1 (the rounding of F - 1 sequential fp32
// additions).  The SH gradient is staged as its two factors w[16], dRGB[3] and the products are formed by the
// writing thread.
//
// The kernel streams about 220 B per (frame, Gaussian) against a few hundred flops, so it is bound by how many
// bytes are in flight.  A thread therefore issues every load it needs at its top, before the visibility test,
// which only selects the results (a culled Gaussian's gradients are zero).  With sh_smem the block's SH
// coefficients (shared by the frames, 16 per Gaussian) arrive with one bulk copy issued at block start; it
// overlaps the per-frame loads, and the frames' threads read them from shared memory.
// staging slots: the SH factors w[16] and dRGB[3], opacity, colour, mean, scale, rotation, cov3D, 2D mean
#define SL_W 0
#define SL_RGB 16
#define SL_OPAC 19
#define SL_COL 20
#define SL_MEAN 23
#define SL_SCALE 26
#define SL_ROT 29
#define SL_COV 33
#define SL_M2D 39
#define SL_COUNT 42

// frames per pass of a 256-thread block (one frame: any block size)
static __host__ __device__ inline int pb_frames_per_pass(int F) { return F >= 8 ? 8 : F >= 4 ? 4 : F >= 2 ? 2 : 1; }

// dynamic shared memory of an NT-thread block: the block's SH coefficients (with sh_smem), then the staging area
static inline size_t pb_smem_bytes(int NT, int F, int M, bool sh_smem) {
  return (sh_smem ? (size_t)(NT / pb_frames_per_pass(F)) * M * 12 : 0) + (size_t)SL_COUNT * (NT + 1) * 4;
}

struct PbCams {  // per frame: tan(fov / 2) and focal lengths in pixels
  float tanx[PB_MAX_FRAMES], tany[PB_MAX_FRAMES], fx[PB_MAX_FRAMES], fy[PB_MAX_FRAMES];
};

// NT threads per block.  One frame runs as 128-thread blocks, 3 per SM (the register budget of the one-frame math
// without a cap); a batch as 256-thread blocks, 2 per SM, 128 registers, 8 frames per pass.
// sh_smem: M = 16 and shs is shared by the frames (or there is one frame).
template <int NT, int MIN_BLOCKS>
__global__ void __launch_bounds__(NT, MIN_BLOCKS) preprocess_bwd_kernel(
    int F, int P, int D, int M, int per_frame, const float* __restrict__ means3D, const int* __restrict__ radii,
    const float* __restrict__ shs, int sh_smem, const float* __restrict__ scales,
    const float* __restrict__ rotations, float scale_modifier, const float* __restrict__ cov3D_precomp,
    const float* __restrict__ views, const float* __restrict__ projs, const float* __restrict__ cam_poses,
    const PbCams cams, char* geom_ws, size_t geom_stride, float* __restrict__ dL_dmean2D,
    float* __restrict__ dL_dconic, float* __restrict__ dL_dopacity, float* __restrict__ dL_dcolor,
    float* __restrict__ dL_dmean3D, float* __restrict__ dL_dcov3D, float* __restrict__ dL_dsh,
    float* __restrict__ dL_dscale, float* __restrict__ dL_drot, int depth_grad) {
  constexpr int PB_STRIDE = NT + 1;  // floats per staging slot: NT (frame, Gaussian) values, + 1 so that slot k starts in bank k
  extern __shared__ __align__(16) float s_dyn[];  // [NG][M * 3] SH coefficients (with sh_smem), then the staging area
  __shared__ __align__(8) uint64_t s_bar;
  pdl_wait();
  pdl_launch();
  const int FB = pb_frames_per_pass(F), NG = NT / FB;
  const int tid = threadIdx.x, wid = tid >> 5;
  const int fi = wid % FB, gl = (wid / FB) * 32 + (tid & 31);
  const int g0 = blockIdx.x * NG, g = g0 + gl, nval = min(NG, P - g0);
  // outputs summed over the frames (DGR_PF_* bits; with one frame every output is that frame's).  dL_dcolor
  // follows the colour input's bit, except with SH colours, where it is [P,3] scratch
  const int sum = F > 1 ? (DGR_PF_ALL & ~per_frame) : 0;
  const bool sum_col = dL_dcolor && F > 1 && (shs || (sum & DGR_PF_COLOR));
  const bool sum_sh = shs && (sum & DGR_PF_COLOR);
  const int ncoef = (D + 1) * (D + 1);
  float* const s_stage = s_dyn + (sh_smem ? NG * 48 : 0);
  float* const stage = s_stage + fi * NG + gl;
  if (sh_smem) {
    if (tid == 0) {
      mbar_init(&s_bar, 1);
      mbar_fence_init();
    }
    __syncthreads();
    if (tid == 0) {
      mbar_expect_tx(&s_bar, nval * 192u);
      tma_load_1d(s_dyn, shs + (size_t)g0 * 48, nval * 192u, &s_bar);
    }
  }

  for (int f0 = 0; f0 < F; f0 += FB) {
    const int f = f0 + fi;
    if (f < F && g < P) {
      const size_t fg = (size_t)f * P + g;
      auto slab = [&](const float* p, int bit, int width) {
        return (per_frame & bit) ? p + (size_t)f * P * width : p;
      };
      const GeomWS gw = GeomWS::from(geom_ws + f * geom_stride, P);
      // ---- every load of this (frame, Gaussian), issued before any of them is used
      const bool visible = (radii ? radii[fg] : gw.radii[g]) > 0;
      const float4 a0 = gw.grad_acc[3 * g + 0], a1 = gw.grad_acc[3 * g + 1], a2 = gw.grad_acc[3 * g + 2];
      const float* mp = slab(means3D, DGR_PF_MEANS, 3) + 3 * g;
      const float3 mean = make_float3(mp[0], mp[1], mp[2]);
      float cov3D[6];
      if (cov3D_precomp) {
        const float* c = slab(cov3D_precomp, DGR_PF_COV, 6) + 6 * g;
#pragma unroll
        for (int k = 0; k < 6; ++k) cov3D[k] = c[k];
      } else {  // the workspace's rows are 8-byte aligned
        const float2* c = reinterpret_cast<const float2*>(gw.cov3D + 6 * g);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const float2 v = c[k];
          cov3D[2 * k] = v.x;
          cov3D[2 * k + 1] = v.y;
        }
      }
      const float* sc_f = scales ? slab(scales, DGR_PF_SCALES, 3) : nullptr;
      const float* rot_f = rotations ? slab(rotations, DGR_PF_ROTS, 4) : nullptr;
      if (sc_f) {  // parked in the slots of their gradients until the EWA gradient is done (register budget)
        const float4 q = __ldg(reinterpret_cast<const float4*>(rot_f) + g);
#pragma unroll
        for (int k = 0; k < 3; ++k) stage[(SL_SCALE + k) * PB_STRIDE] = sc_f[3 * g + k];
        stage[(SL_ROT + 0) * PB_STRIDE] = q.x;
        stage[(SL_ROT + 1) * PB_STRIDE] = q.y;
        stage[(SL_ROT + 2) * PB_STRIDE] = q.z;
        stage[(SL_ROT + 3) * PB_STRIDE] = q.w;
      }
      // clear the accumulators written by render_bwd_kernel
      gw.grad_acc[3 * g + 0] = make_float4(0, 0, 0, 0);
      gw.grad_acc[3 * g + 1] = make_float4(0, 0, 0, 0);
      gw.grad_acc[3 * g + 2] = make_float4(0, 0, 0, 0);
      const float3 dcon = make_float3(a0.z, a0.w, a1.x);  // (xx, xy, yy) slots .x .y .w of the reference float4
      // the 2D mean and colour gradients are read back from the staging area where they are used (fewer live
      // registers through the EWA gradient)
      stage[(SL_M2D + 0) * PB_STRIDE] = a0.x;
      stage[(SL_M2D + 1) * PB_STRIDE] = a0.y;
      stage[(SL_M2D + 2) * PB_STRIDE] = 0.f;
      if (dL_dconic) reinterpret_cast<float4*>(dL_dconic)[fg] = make_float4(dcon.x, dcon.y, 0.f, dcon.z);
      stage[SL_OPAC * PB_STRIDE] = a1.y;
      stage[(SL_COL + 0) * PB_STRIDE] = a1.z;
      stage[(SL_COL + 1) * PB_STRIDE] = a1.w;
      stage[(SL_COL + 2) * PB_STRIDE] = a2.x;
      stage[SL_MEAN * PB_STRIDE] = a2.y;  // dL/d(depth), until dL/dmean3D takes the slot

      float dcov[6] = {0, 0, 0, 0, 0, 0};
      float3 dmean = make_float3(0, 0, 0);
      float3 dscale = make_float3(0, 0, 0);
      float4 drot = make_float4(0, 0, 0, 0);
      float w[16], dRGB[3] = {0.f, 0.f, 0.f};
#pragma unroll
      for (int k = 0; k < 16; ++k) w[k] = 0.f;
      {
        const float* view = views + 16 * f;
        const float* proj = projs + 16 * f;
        const float focal_x = cams.fx[f], focal_y = cams.fy[f], tan_fovx = cams.tanx[f], tan_fovy = cams.tany[f];
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
        const float2 dm2 = make_float2(stage[SL_M2D * PB_STRIDE], stage[(SL_M2D + 1) * PB_STRIDE]);
        dm.x = (proj[0] * m_w - proj[3] * mul1) * dm2.x + (proj[1] * m_w - proj[3] * mul2) * dm2.y;
        dm.y = (proj[4] * m_w - proj[7] * mul1) * dm2.x + (proj[5] * m_w - proj[7] * mul2) * dm2.y;
        dm.z = (proj[8] * m_w - proj[11] * mul1) * dm2.x + (proj[9] * m_w - proj[11] * mul2) * dm2.y;
        dmean.x += dm.x;
        dmean.y += dm.y;
        dmean.z += dm.z;
        // depth map: dL/d(depth) (grad_acc float 9) through depth = p_view.z, the third row of the view
        // transform (xform4x3).  Only when the backward carries one: adding 0 would turn -0 into +0
        if (depth_grad) {
          const float dd = stage[SL_MEAN * PB_STRIDE];
          dmean.x += dd * view[2];
          dmean.y += dd * view[6];
          dmean.z += dd * view[10];
        }

        // ---------------- 3D covariance -> scale / rotation (backward.cu:279-341)
        if (sc_f) {
          const float3 sc = make_float3(stage[SL_SCALE * PB_STRIDE], stage[(SL_SCALE + 1) * PB_STRIDE],
                                        stage[(SL_SCALE + 2) * PB_STRIDE]);
          const float4 q = make_float4(stage[SL_ROT * PB_STRIDE], stage[(SL_ROT + 1) * PB_STRIDE],
                                       stage[(SL_ROT + 2) * PB_STRIDE], stage[(SL_ROT + 3) * PB_STRIDE]);
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
        // a culled Gaussian's gradients are zero: the visibility test selects the results
        auto vis = [&](float v) { return visible ? v : 0.f; };
#pragma unroll
        for (int k = 0; k < 6; ++k) stage[(SL_COV + k) * PB_STRIDE] = vis(dcov[k]);
        stage[(SL_SCALE + 0) * PB_STRIDE] = vis(dscale.x);
        stage[(SL_SCALE + 1) * PB_STRIDE] = vis(dscale.y);
        stage[(SL_SCALE + 2) * PB_STRIDE] = vis(dscale.z);
        stage[(SL_ROT + 0) * PB_STRIDE] = vis(drot.x);
        stage[(SL_ROT + 1) * PB_STRIDE] = vis(drot.y);
        stage[(SL_ROT + 2) * PB_STRIDE] = vis(drot.z);
        stage[(SL_ROT + 3) * PB_STRIDE] = vis(drot.w);

        // ---------------- SH colour (backward.cu:20-139, 383-385)
        if (shs) {
          const float3 cp = make_float3(cam_poses[3 * f], cam_poses[3 * f + 1], cam_poses[3 * f + 2]);
          float sh[48];
          if (!sh_smem) {
            load_sh(slab(shs, DGR_PF_COLOR, M * 3), g, M, ncoef, sh);
          } else {
            mbar_wait(&s_bar, 0);
            const float4* v = reinterpret_cast<const float4*>(s_dyn + gl * 48);
#pragma unroll
            for (int i = 0; i < 12; ++i) {
              const float4 t = v[i];
              sh[4 * i + 0] = t.x;
              sh[4 * i + 1] = t.y;
              sh[4 * i + 2] = t.z;
              sh[4 * i + 3] = t.w;
            }
          }
          const float3 dcol = make_float3(stage[SL_COL * PB_STRIDE], stage[(SL_COL + 1) * PB_STRIDE],
                                          stage[(SL_COL + 2) * PB_STRIDE]);
          const float3 dms = sh_backward(D, mean, cp, sh, gw.clamped + 3 * g, dcol, w, dRGB);
          dmean.x += dms.x;
          dmean.y += dms.y;
          dmean.z += dms.z;
        }
#pragma unroll
        for (int k = 0; k < 16; ++k) stage[(SL_W + k) * PB_STRIDE] = vis(w[k]);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) stage[(SL_RGB + ch) * PB_STRIDE] = vis(dRGB[ch]);
        stage[(SL_MEAN + 0) * PB_STRIDE] = vis(dmean.x);
        stage[(SL_MEAN + 1) * PB_STRIDE] = vis(dmean.y);
        stage[(SL_MEAN + 2) * PB_STRIDE] = vis(dmean.z);
      }
    }
    // ---- per-frame outputs: each warp writes the rows of its own 32 Gaussians as soon as it has staged them
    // (element e = q * width + c of the warp's slice is row q, column c: every store of the warp covers 128
    // consecutive bytes), without waiting for the rest of the block
    if (f < F) {  // uniform per warp
      __syncwarp();
      const int gw0 = (wid / FB) * 32, nw = min(32, P - g0 - gw0);
      const float* ws = s_stage + fi * NG + gw0;
      auto own = [&](float* out, int width, auto value) {
        float* dst = out + ((size_t)f * P + g0 + gw0) * width;
#pragma unroll 4
        for (int j = 0; j < width; ++j) {
          const int e = (tid & 31) + 32 * j, q = e / width, c = e - q * width;
          if (q < nw) dst[e] = value(ws, q, c);
        }
      };
      auto staged = [](int slot) {
        return [=](const float* st, int q, int c) { return st[(slot + c) * PB_STRIDE + q]; };
      };
      own(dL_dmean2D, 3, staged(SL_M2D));
      if (!(sum & DGR_PF_OPAC)) own(dL_dopacity, 1, staged(SL_OPAC));
      if (dL_dcolor && !sum_col) own(dL_dcolor, 3, staged(SL_COL));
      if (!(sum & DGR_PF_MEANS)) own(dL_dmean3D, 3, staged(SL_MEAN));
      if (dL_dcov3D && !(sum & DGR_PF_COV)) own(dL_dcov3D, 6, staged(SL_COV));
      if (!(sum & DGR_PF_SCALES)) own(dL_dscale, 3, staged(SL_SCALE));
      if (!(sum & DGR_PF_ROTS)) own(dL_drot, 4, staged(SL_ROT));
      // dL_dsh[k][ch] = w[k] dRGB[ch]; 0 for the coefficients k >= ncoef that the SH degree does not use
      if (shs && !sum_sh)
        own(dL_dsh, 3 * M, [=](const float* st, int q, int c) {
          const int k = c / 3;
          return k < ncoef ? __fmul_rn(st[(SL_W + k) * PB_STRIDE + q], st[(SL_RGB + c - 3 * k) * PB_STRIDE + q]) : 0.f;
        });
      __syncwarp();
    }
    if (!sum && !sum_col) continue;  // uniform: nothing is summed over the frames
    __syncthreads();
    // ---- outputs summed over the frames: the block sums this pass's frames into its rows, in frame order,
    // continuing from the value the previous pass stored.  value(q, c, i) is frame i's staged value
    const int nf = min(FB, F - f0);
    auto sum_rows = [&](float* out, int width, auto value) {
      float* dst = out + (size_t)g0 * width;
      for (int e = tid; e < nval * width; e += NT) {
        const int q = e / width, c = e - q * width;
        float v[8];  // FB <= 8: every frame's value is read before the sequential sum
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = i < nf ? value(q, c, i) : 0.f;
        float acc = f0 ? dst[e] : v[0];
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (i < nf && (f0 || i > 0)) acc = acc + v[i];
        dst[e] = acc;
      }
    };
    auto summed = [&](int slot) {
      return [=](int q, int c, int i) { return s_stage[(slot + c) * PB_STRIDE + i * NG + q]; };
    };
    if (sum & DGR_PF_OPAC) sum_rows(dL_dopacity, 1, summed(SL_OPAC));
    if (sum_col) sum_rows(dL_dcolor, 3, summed(SL_COL));
    if (sum & DGR_PF_MEANS) sum_rows(dL_dmean3D, 3, summed(SL_MEAN));
    if ((sum & DGR_PF_COV) && dL_dcov3D) sum_rows(dL_dcov3D, 6, summed(SL_COV));
    if (sum & DGR_PF_SCALES) sum_rows(dL_dscale, 3, summed(SL_SCALE));
    if (sum & DGR_PF_ROTS) sum_rows(dL_drot, 4, summed(SL_ROT));
    // each product rounded before it is added; 0 for k >= ncoef
    if (sum_sh)
      sum_rows(dL_dsh, 3 * M, [=](int q, int c, int i) {
        const int k = c / 3;
        return k < ncoef ? __fmul_rn(s_stage[(SL_W + k) * PB_STRIDE + i * NG + q],
                                     s_stage[(SL_RGB + c - 3 * k) * PB_STRIDE + i * NG + q])
                         : 0.f;
      });
    __syncthreads();  // the next pass overwrites the staging area
  }
}

cudaError_t launch_backward(const BwdArgs& a, cudaStream_t s) {
  cudaError_t e = launch_render_bwd(a, s);
  return e != cudaSuccess ? e : launch_preprocess_bwd(a, s);
}

// gradient of the alpha-compositing (fills the GPU); leaves the per-Gaussian moments in grad_acc
cudaError_t launch_render_bwd(const BwdArgs& a, cudaStream_t s) {
  static unsigned long long attr = 0;  // per device
  if (once_per_device(attr)) {
    // the staging area takes the kernel past 48 KB of shared memory; 3 CTAs per SM need the largest carveout
    for (auto k : {render_bwd_kernel<false>, render_bwd_kernel<true>}) {
      cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, STAGE_BYTES);
      cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    }
  }
  if (a.P == 0) return cudaSuccess;
  const unsigned gx = (a.W + TILE_X - 1) / TILE_X, gy = (a.H + TILE_Y - 1) / TILE_Y;
  const int T = gx * gy;
  GeomWS g = GeomWS::from((char*)a.geom_ws, a.P);
  ImgWS im = ImgWS::from((char*)a.img_ws, (size_t)a.W * a.H, T);
  BinWS b = BinWS::from((char*)a.binning_ws, (size_t)a.R_cap);
  const bool aux = a.dL_ddepth || a.dL_dalpha;
  g_prof.begin(5, s);
  launch_pdl(aux ? render_bwd_kernel<true> : render_bwd_kernel<false>, dim3(T), dim3(256), STAGE_BYTES, s,
             (const uint2*)im.ranges, (const uint32_t*)im.tile_order, (const float4*)b.inst_geo,
             (const float4*)b.inst_attr, a.W, a.H, a.background, (const float*)im.final_T,
             (const uint32_t*)im.n_contrib, a.dL_dpix, g.grad_acc, a.dL_ddepth, a.dL_dalpha);
  g_prof.end(5, s);
  return cudaGetLastError();
}

// chain rule from the moments to the inputs, all frames of a batch in one launch (after every frame's
// render_bwd_kernel)
cudaError_t launch_preprocess_bwd(const BwdArgs& a, cudaStream_t s) {
  if (a.P == 0) return cudaSuccess;
  if (a.F < 1 || a.F > PB_MAX_FRAMES) return cudaErrorInvalidValue;
  PbCams c = {};
  for (int f = 0; f < a.F; ++f) {
    c.tanx[f] = a.tan_fovx[f];
    c.tany[f] = a.tan_fovy[f];
    c.fx[f] = a.W / (2.0f * a.tan_fovx[f]);
    c.fy[f] = a.H / (2.0f * a.tan_fovy[f]);
  }
  auto one = preprocess_bwd_kernel<128, 3>, batch = preprocess_bwd_kernel<256, 2>;
  static unsigned long long attr = 0;  // per device
  if (once_per_device(attr)) {
    // the largest staging area + SH tile (2 or 3 frames: 128 Gaussians per block) exceeds 48 KB
    cudaFuncSetAttribute(one, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pb_smem_bytes(128, 1, 16, true));
    cudaFuncSetAttribute(batch, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pb_smem_bytes(256, 2, 16, true));
  }
  // 16 SH coefficients per Gaussian are read as 16-byte vectors throughout (load_sh): 192-byte rows, aligned
  const bool sh_smem = a.shs && a.M == 16 && (a.F == 1 || !(a.per_frame & DGR_PF_COLOR));
  const int nt = a.F == 1 ? 128 : 256, ng = nt / pb_frames_per_pass(a.F);
  g_prof.begin(6, s);
  launch_pdl(a.F == 1 ? one : batch, dim3((a.P + ng - 1) / ng), dim3(nt), pb_smem_bytes(nt, a.F, a.M, sh_smem), s,
             a.F, a.P, a.D, a.M, a.per_frame, a.means3D, a.radii, a.shs, sh_smem ? 1 : 0, a.scales, a.rotations,
             a.scale_modifier, a.cov3D_precomp, a.viewmatrix, a.projmatrix, a.cam_pos, c, (char*)a.geom_ws,
             a.geom_stride, a.dL_dmean2D, a.dL_dconic, a.dL_dopacity, a.dL_dcolor, a.dL_dmean3D, a.dL_dcov3D,
             a.dL_dsh, a.dL_dscale, a.dL_drot, a.dL_ddepth ? 1 : 0);
  g_prof.end(6, s);
  return cudaGetLastError();
}

}  // namespace dgm
