// raster_bwd_blend.cuh -- the blend backward kernel (render_bwd_kernel) of the tile-based 3D-Gaussian rasterizer and
// its launcher (launch_blend_bwd), shared by raster_bwd.cu (the colour-only and depth/alpha instances),
// raster_nrm_bwd.cu (the normal-map instance), raster_surf_bwd.cu (the median-depth / distortion instances) and
// raster_abs_bwd.cu (the instances with the absolute screen-space gradient), each in its own translation unit so that
// the other kernels of raster_bwd.cu compile as they did without them.
// See raster_bwd.cu for the design of the kernel.
#pragma once
#include "common.cuh"
#include "raster_kernels.h"
#include "raster_math.cuh"

namespace dgm {

#define RB 256          // records per TMA batch
#define CHUNK 16        // records a warp stages before contracting them
#define SLOT_F 68       // floats per staged record: w[32], alpha T[32], and 16 B that put the 16 slots in distinct banks
#define STAGE_BYTES (8 * CHUNK * SLOT_F * 4)  // dynamic shared memory: one staging area per warp

// floats per record in the per-tile accumulator: the nine sums, + dL/d(depth) with depth and alpha, + the three
// dL/dnormal sums with the normal map, + the two distortion sums S_A, S_M with the surface maps, + the two sums
// of |dL/dmean2D| per pixel with the absolute screen-space gradient (ABS)
template <bool AUX, bool NRM = false, bool SURF = false, bool ABS = false> constexpr int acc_stride() {
  return (NRM ? 13 : AUX ? 10 : 9) + (SURF ? 2 : 0) + (ABS ? 2 : 0);
}
// rows of dL/dpixel per warp: colour, + depth, + normal, + the two distortion rows (A, M1) dL/d(distortion)
template <bool AUX, bool NRM = false, bool SURF = false> constexpr int dlp_rows() {
  return (NRM ? 7 : AUX ? 4 : 3) + (SURF ? 2 : 0);
}

// The normal (NRM) and surface (SURF) instances keep their per-tile accumulator, their dL/dpixel rows and the
// normal stream (NRM) in the dynamic shared memory, behind the staging area (the static arrays of the normal
// instance would pass 48 KB; with static arrays the surface instance spills): offsets and size in floats
template <bool NRM, bool SURF = false, bool ABS = false> struct DynSmem {
  static constexpr int ACC = STAGE_BYTES / 4;                                // s_acc [RB][acc_stride]
  static constexpr int DLP = ACC + RB * acc_stride<true, NRM, SURF, ABS>();  // s_dlp [8 warps][dlp_rows][32]
  static constexpr int REF = DLP + 8 * dlp_rows<true, NRM, SURF>() * 32;   // the tile's reference depth (SURF only)
  static constexpr int REC = REF + (SURF ? 4 : 0);                         // s_nrm [2][RB] float4 (16-byte aligned)
  static constexpr int BYTES = (REC + (NRM ? 2 * RB * 4 : 0)) * 4;
};

// Contract the first n staged records of a warp into s_acc.  Slot k holds w and alpha T of the 32 pixels
// (pixel = lane of the staging warp: column lane & 7, row lane >> 3) of record `rec` (held by lanes k and
// k + 16).  Lane l sums slot l & 15 over pixel rows 2h, 2h+1, h = l >> 4, as pixel offsets u, v from the
// block centre (exact in fp32), then expands the moments about the Gaussian's offset (Gx, Gy) from that
// centre: sum w dx = Gx S_1 - S_u, sum w dx^2 = Gx^2 S_1 - 2 Gx S_u + S_uu, ...  The two lanes of a slot
// trade half of their nine partial sums, so each adds 5 or 4 totals (shared-memory float atomics are
// compare-and-swap loops on sm_90).  Every lane computes; only the lanes of the n filled slots add.
// AUX: dlp has a fourth row, dL/d(depth); its weight sum alpha T dL/dD is the tenth total (slot 9), added
// by lane h = 1, which then adds 5 totals too.
// NRM (with AUX): rows 4-6 are dL/dnormal; their weight sums are totals 10-12.  Lane h = 0 adds totals 0-6,
// lane h = 1 totals 7-12.
// SURF (with AUX): the last two rows are A dL/dS and M1 dL/dS (S the distortion map); their weight sums S_A, S_M are
// the last two totals (10-11, or 13-14 with NRM).  Lane h = 0 adds 6 (8) totals, lane h = 1 the other 6 (7).
// ABS: two more totals behind all of the above, sum |w (c.x dx + c.y dy)| and sum |w (c.y dx + c.z dy)| over the
// pixels (c the record's conic in attr), formed pixel by pixel: |.| does not pass through the moments.  Each lane
// adds one total more.
template <bool AUX, bool NRM = false, bool SURF = false, bool ABS = false>
__device__ __forceinline__ void contract_chunk(const float* stage, const float* dlp, int n, int rec, unsigned lane,
                                               const float4* geo, float cx, float cy, float* s_acc,
                                               const float4* attr = nullptr) {
  constexpr int NCH = dlp_rows<AUX, NRM, SURF>();
  constexpr int HALF = (SURF ? (NRM ? 8 : 6) : NRM ? 7 : 5) + (ABS ? 1 : 0);  // totals of lane h = 0
  constexpr int LAST = acc_stride<AUX, NRM, SURF, ABS>() - HALF;               // totals of lane h = 1
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
  float m[2 * HALF] = {S1, fmaf(Gx, S1, -Su), my, fmaf(Gx, fmaf(Gx, S1, -2.0f * Su), Suu),
                       fmaf(Gx, my, fmaf(-Gy, Su, Suv)), fmaf(Gy, fmaf(Gy, S1, -2.0f * Sv), Svv),
                       c[0], c[1], c[2], AUX ? c[AUX ? 3 : 0] : 0.0f};
#pragma unroll
  for (int ch = 4; ch < NCH; ++ch) m[6 + ch] = c[ch];  // NRM: the normal weights, totals 10-12; SURF: S_A, S_M
  if (ABS) {
    // at pixel (u, v): c.x dx + c.y dy = X_v - c.x u with X_v = c.x Gx + c.y (Gy - v), c.y dx + c.z dy = Y_v - c.y u
    constexpr int S = acc_stride<AUX, NRM, SURF>();
    const float4 co = attr[2 * rec];
    float ax = 0.0f, ay = 0.0f;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float4 p = w4[2 * r], q = w4[2 * r + 1];
      const float w[8] = {p.x, p.y, p.z, p.w, q.x, q.y, q.z, q.w};
      const float dy = Gy - (r ? v1 : v0);
      const float X = fmaf(co.x, Gx, co.y * dy), Y = fmaf(co.y, Gx, co.z * dy);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float u = j - 3.5f;
        ax += fabsf(w[j] * fmaf(-co.x, u, X));
        ay += fabsf(w[j] * fmaf(-co.y, u, Y));
      }
    }
    m[ABS ? S : 0] = ax;
    m[ABS ? S + 1 : 0] = ay;
  }
  // lane h = 0 adds moments 0-4, h = 1 moments 5-8 (9) (NRM: totals 0-6 and 7-12)
  float* acc = &s_acc[rec * acc_stride<AUX, NRM, SURF, ABS>() + HALF * h];
#pragma unroll
  for (int q = 0; q < HALF; ++q) {
    const float keep = h ? m[q + HALF] : m[q], send = h ? m[q] : m[q + HALF];
    const float tot = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    if (k < n && (q < LAST || h == 0)) atomicAdd(&acc[q], tot);
  }
}

// AUX: the upstream gradients of the depth map (needs the records of a depth forward: depth in .w) and of
// the alpha map, each NULL when the loss does not use it.  dL/d(depth_i) goes to float 9 of grad_acc.
// NRM (with AUX): also the upstream gradient of the [3,H,W] normal map (non-NULL); the records' normals stream
// from inst_nrm and dL/dn_i = sum over pixels of alpha_i T_i dL/dN goes to nrm_acc[id] (NrmWS::acc).  Dynamic
// shared memory: DynSmem<NRM, SURF, ABS>::BYTES with NRM or SURF, else STAGE_BYTES (launch_blend_bwd).
// SURF (with AUX): also the upstream gradient dL/dS of the distortion map (non-NULL), with the totals {M1, M2} of the
// surface forward (surf_mom), A = 1 - T_final and m_i = surf_m(d_i, d of the tile's first record, surf_k).  Through alpha the distortion acts as one more colour channel of
// "colour" g_i = m_i^2 A - 2 m_i M1 + M2 and no background; through the depth, dL/dm_i = 2 (m_i S_A - S_M) with
// S_A, S_M = sum over pixels of alpha_i T_i A dL/dS and alpha_i T_i M1 dL/dS, chained through dm/dd = k / d^2 into
// float 9 of grad_acc (the reference depth drops out: the distortion depends on differences of m only).
// ABS (any of the above): also the absolute screen-space gradient, abs_out[id] += (sum over pixels of |dL/dmean2D.x|
// per pixel, the same of .y), into the [P,3] abs_out (.z untouched), which the caller zeroes.
template <bool AUX, bool NRM = false, bool SURF = false, bool ABS = false>
__global__ void __launch_bounds__(256, AUX || ABS ? 2 : 3) render_bwd_kernel(
    const uint2* __restrict__ ranges, const uint32_t* __restrict__ tile_order, const float4* __restrict__ inst_geo,
    const float4* __restrict__ inst_attr,
    int W, int H, const float* __restrict__ bg_color, const float* __restrict__ final_Ts,
    const uint32_t* __restrict__ n_contrib, const float* __restrict__ dL_dpixels, float4* __restrict__ grad_acc,
    const float* __restrict__ dL_ddepth, const float* __restrict__ dL_dalpha, const float* __restrict__ dL_dnormal,
    const float4* __restrict__ inst_nrm, float4* __restrict__ nrm_acc, const float* __restrict__ dL_ddist,
    const float2* __restrict__ surf_mom, float surf_k, float* __restrict__ abs_out) {
  constexpr int ACC_STRIDE = acc_stride<AUX, NRM, SURF, ABS>();
  constexpr int SB = acc_stride<AUX, NRM, SURF>();  // the totals before the two ABS totals
  constexpr int NCH = dlp_rows<AUX, NRM, SURF>();  // rows of s_dlp
  constexpr int SROW = NRM ? 7 : 4;                // first distortion row of s_dlp (SURF only)
  __shared__ __align__(128) float4 s_geo[2][RB];
  __shared__ __align__(128) float4 s_attr[2][2 * RB];
  constexpr bool DYN = NRM || SURF;  // s_acc and s_dlp in the dynamic shared memory
  __shared__ float s_acc_st[DYN ? 1 : RB * ACC_STRIDE];
  __shared__ __align__(16) float s_dlp_st[DYN ? 1 : 8][NCH][32];  // dL/dpixel of each warp's 32 pixels, per colour (+ depth)
  __shared__ __align__(8) uint64_t s_bar[2];
  __shared__ int s_maxc;
  extern __shared__ __align__(16) float s_stage[];  // [8 warps][CHUNK][SLOT_F] (NRM / SURF: then s_acc, s_dlp, s_nrm)
  using DS = DynSmem<NRM, SURF, ABS>;
  float* const s_acc = DYN ? s_stage + DS::ACC : s_acc_st;
  float(*const s_dlp)[NCH][32] = DYN ? reinterpret_cast<float(*)[NCH][32]>(s_stage + DS::DLP) : s_dlp_st;
  float4* const s_nrm = reinterpret_cast<float4*>(s_stage + DS::REC);  // [2][RB] (NRM only)
  float* const s_dref = s_stage + DS::REF;  // (SURF only; read where used: no register to hold)

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

  if (SURF && tid == 0) *s_dref = inst_geo[range.x].w;
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
    mbar_expect_tx(&s_bar[0], cnt * (NRM ? 64u : 48u));
    tma_load_1d(&s_geo[0][0], inst_geo + range.x + lo, cnt * 16u, &s_bar[0]);
    tma_load_1d(&s_attr[0][0], inst_attr + 2 * ((size_t)range.x + lo), cnt * 32u, &s_bar[0]);
    if (NRM) tma_load_1d(&s_nrm[0], inst_nrm + range.x + lo, cnt * 16u, &s_bar[0]);
  }

  float dLp0 = 0.f, dLp1 = 0.f, dLp2 = 0.f, dLD = 0.f, dLA = 0.f;
  float dLN0 = 0.f, dLN1 = 0.f, dLN2 = 0.f;  // normal map (NRM only)
  // distortion map (SURF only): the pixel's totals A, M1, M2 times dL/dS, so that dL/dS g_i = m_i (m_i cA + cM1x2) + cM2
  float cA = 0.f, cM1 = 0.f, cM2 = 0.f;
  if (inside) {
    const size_t HW = (size_t)H * W;
    dLp0 = dL_dpixels[0 * HW + pix_id];
    dLp1 = dL_dpixels[1 * HW + pix_id];
    dLp2 = dL_dpixels[2 * HW + pix_id];
    if (AUX && dL_ddepth) dLD = dL_ddepth[pix_id];
    if (AUX && dL_dalpha) dLA = dL_dalpha[pix_id];
    if (NRM) {
      dLN0 = dL_dnormal[0 * HW + pix_id];
      dLN1 = dL_dnormal[1 * HW + pix_id];
      dLN2 = dL_dnormal[2 * HW + pix_id];
    }
    if (SURF) {
      const float2 mom = surf_mom[pix_id];
      const float dLS = dL_ddist[pix_id];
      cA = (1.0f - T_final) * dLS;
      cM1 = mom.x * dLS;
      cM2 = mom.y * dLS;
    }
  }
  s_dlp[wid][0][lane] = dLp0;
  s_dlp[wid][1][lane] = dLp1;
  s_dlp[wid][2][lane] = dLp2;
  if (AUX) s_dlp[wid][AUX ? 3 : 0][lane] = dLD;
  if (NRM) {
    s_dlp[wid][NRM ? 4 : 0][lane] = dLN0;
    s_dlp[wid][NRM ? 5 : 0][lane] = dLN1;
    s_dlp[wid][NRM ? 6 : 0][lane] = dLN2;
  }
  if (SURF) {
    s_dlp[wid][SURF ? SROW : 0][lane] = cA;
    s_dlp[wid][SURF ? SROW + 1 : 0][lane] = cM1;
  }
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
  float accumN0 = 0.f, accumN1 = 0.f, accumN2 = 0.f;  // normal composited behind it (NRM only)
  float accumG = 0.f;  // dL/dS times the distortion "colour" composited behind it (SURF only)

  for (int i = 0; i < rounds; ++i) {
    const int st = i & 1;
    const int hi = maxc - i * RB, lo = max(0, hi - RB);
    const int cnt = hi - lo;
    mbar_wait(&s_bar[st], (i >> 1) & 1);
    __syncthreads();  // previous batch fully flushed; other stage free
    if (tid == 0 && i + 1 < rounds) {
      const int nhi = lo, nlo = max(0, nhi - RB);
      const uint32_t ncnt = nhi - nlo;
      mbar_expect_tx(&s_bar[st ^ 1], ncnt * (NRM ? 64u : 48u));
      tma_load_1d(&s_geo[st ^ 1][0], inst_geo + range.x + nlo, ncnt * 16u, &s_bar[st ^ 1]);
      tma_load_1d(&s_attr[st ^ 1][0], inst_attr + 2 * ((size_t)range.x + nlo), ncnt * 32u, &s_bar[st ^ 1]);
      if (NRM) tma_load_1d(&s_nrm[(st ^ 1) * RB], inst_nrm + range.x + nlo, ncnt * 16u, &s_bar[st ^ 1]);
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
        const float2 npow = pair_npow(geA, geB, coA, coB, npx2, npy2);
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
          float dN0 = 0.0f, dN1 = 0.0f, dN2 = 0.0f;
          if (NRM) {
            const float4 nv = s_nrm[st * RB + j];
            dN0 = nv.x - accumN0, dN1 = nv.y - accumN1, dN2 = nv.z - accumN2;
          }
          float dG = 0.0f;
          if (SURF) {
            const float m = surf_m(s_geo[st][j].w, *s_dref, surf_k);
            // cA and cM1 are read back from their dL/dpixel rows (held in registers, they make this instance spill)
            const float a_ = s_dlp[wid][SURF ? SROW : 0][lane], m1_ = s_dlp[wid][SURF ? SROW + 1 : 0][lane];
            dG = fmaf(m, fmaf(m, a_, -2.0f * m1_), cM2) - accumG;  // dL/dS (g_i - G_behind)
          }
          float dLa = d0 * dLp0;
          dLa = fmaf(d1, dLp1, dLa);
          dLa = fmaf(d2, dLp2, dLa);
          if (AUX) dLa = fmaf(dD, dLD, dLa);
          if (NRM) {
            dLa = fmaf(dN0, dLN0, dLa);
            dLa = fmaf(dN1, dLN1, dLa);
            dLa = fmaf(dN2, dLN2, dLa);
          }
          if (SURF) dLa += dG;
          dLa = fmaf(dLa, T, mTb * r);
          const float w = act ? (G * opac) * dLa : 0.0f;
          // colour behind the NEXT record: alpha c + (1 - alpha) accum  (backward.cu:507, evaluated eagerly)
          accum0 = fmaf(a_eff, d0, accum0);
          accum1 = fmaf(a_eff, d1, accum1);
          accum2 = fmaf(a_eff, d2, accum2);
          if (AUX) accumD = fmaf(a_eff, dD, accumD);
          if (NRM) {
            accumN0 = fmaf(a_eff, dN0, accumN0);
            accumN1 = fmaf(a_eff, dN1, accumN1);
            accumN2 = fmaf(a_eff, dN2, accumN2);
          }
          if (SURF) accumG = fmaf(a_eff, dG, accumG);
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
          contract_chunk<AUX, NRM, SURF, ABS>(stage, &s_dlp[wid][0][0], nslot, rec, lane, s_geo[st], cx, cy, s_acc,
                                              s_attr[st]);
          __syncwarp();
          nslot = 0;
        }
      }
    }
    if (nslot > 0) {  // the batch's records must be in s_acc before the flush
      __syncwarp();
      contract_chunk<AUX, NRM, SURF, ABS>(stage, &s_dlp[wid][0][0], nslot, rec, lane, s_geo[st], cx, cy, s_acc,
                                          s_attr[st]);
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
        if (SURF) {  // dL/dd += 2 (m S_A - S_M) dm/dd, dm/dd = k / d^2
          const float d = s_geo[st][tid].w, rd = __frcp_rn(d);
          const float m = surf_m(d, *s_dref, surf_k);
          const float dm_dd = surf_k * (rd * rd);
          const float g_m = 2.0f * fmaf(m, a[SB - 2], -a[SB - 1]);
          red_add_v2(dst + 8, a[8], fmaf(g_m, dm_dd, a[AUX ? 9 : 8]));
        } else if (AUX) red_add_v2(dst + 8, a[8], a[AUX ? 9 : 8]);
        else atomicAdd(dst + 8, a[8]);
        if (NRM) red_add_v4(reinterpret_cast<float*>(nrm_acc + id), a[NRM ? 10 : 0], a[NRM ? 11 : 0],
                            a[NRM ? 12 : 0], 0.0f);
        if (ABS) {  // rows of 12 bytes: 8-byte aligned for even id only, so two scalar reductions, not one v2
          float* o = abs_out + 3 * (size_t)id;
          atomicAdd(o, ddelx_dx * a[ABS ? SB : 0]);
          atomicAdd(o + 1, ddely_dy * a[ABS ? SB + 1 : 0]);
        }
      }
    }
  }
}

// The blend backward of one frame (frame 0 of a) with render_bwd_kernel<AUX, NRM, SURF, ABS>.  launch_render_bwd picks
// the instance: NRM = dL_dnormal, SURF = dL_ddistortion, ABS = dL_dmean2D_abs, AUX = dL_ddepth || dL_dalpha || NRM ||
// SURF; the arguments of a map the instance does not read are NULL.  Each instance is instantiated in one translation
// unit only (see the file comment).
template <bool AUX, bool NRM, bool SURF, bool ABS>
cudaError_t launch_blend_bwd(const BwdArgs& a, cudaStream_t s) {
  auto k = render_bwd_kernel<AUX, NRM, SURF, ABS>;
  constexpr size_t smem = (NRM || SURF) ? (size_t)DynSmem<NRM, SURF, ABS>::BYTES : (size_t)STAGE_BYTES;
  static unsigned long long attr = 0;  // per device
  if (once_per_device(attr)) {
    // the staging area takes every instance past 48 KB of shared memory; 2 or 3 CTAs per SM need the largest carveout
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  }
  if (a.P == 0) return cudaSuccess;
  const unsigned gx = (a.W + TILE_X - 1) / TILE_X, gy = (a.H + TILE_Y - 1) / TILE_Y;
  const int T = gx * gy;
  GeomWS g = GeomWS::from((char*)a.geom_ws, a.P);
  ImgWS im = ImgWS::from((char*)a.img_ws, (size_t)a.W * a.H, T);
  BinWS b = BinWS::from((char*)a.binning_ws, (size_t)a.R_cap);
  NrmWS n = {};
  if (NRM) n = NrmWS::from((char*)a.nrm_ws, a.P, (size_t)a.R_cap);
  SurfWS sw = {};
  if (SURF) sw = SurfWS::from((char*)a.surf_ws, (size_t)a.W * a.H);
  g_prof.begin(5, s);
  launch_pdl(k, dim3(T), dim3(256), smem, s, (const uint2*)im.ranges, (const uint32_t*)im.tile_order,
             (const float4*)b.inst_geo, (const float4*)b.inst_attr, a.W, a.H, a.background, (const float*)im.final_T,
             (const uint32_t*)im.n_contrib, a.dL_dpix, g.grad_acc, AUX ? a.dL_ddepth : nullptr,
             AUX ? a.dL_dalpha : nullptr, NRM ? a.dL_dnormal : nullptr, (const float4*)n.inst_nrm, n.acc,
             SURF ? a.dL_ddistortion : nullptr, (const float2*)sw.moments, SURF ? a.surf_k : 0.f,
             ABS ? a.dL_dmean2D_abs : nullptr);
  g_prof.end(5, s);
  return cudaGetLastError();
}

}  // namespace dgm
