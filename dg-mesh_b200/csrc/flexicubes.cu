// flexicubes.cu -- FlexiCubes (Shen et al. 2023) on the topology of dual marching cubes (dmc.cu), forward and
// backward, for one G^3 grid.
//
// Cells, cases, patches, which patches get a vertex, V and Q are dual marching cubes' (launch_dmc_count; the emission
// reuses launch_dmc_emit for vsrc, cvid and the oriented quads).  On top of that, with s = phi - iso, node n at
// x_n = n + deform[n] and kaolin's activations of the raw per-cell weights:
//   crossing   w0 = alpha[r0] s(n0), w1 = alpha[r1] s(n1), t = w0 / (w0 - w1), u = x0 + t (x1 - x0)
//   vertex     v = (sum_e beta[e] u_e) / (sum_e beta[e]), summed in increasing edge id, / (G - 1)
//   split      inference: (q0,q1,q2), (q0,q2,q3) when g0 g2 >= g1 g3, else (q0,q1,q3), (q1,q2,q3);
//              training: a centre vertex m = (g02 (v0 + v2) / 2 + g13 (v1 + v3) / 2) / (g02 + g13 + 1e-8) at row
//              V + q and four triangles around it
//   L_dev      |d_e - mean d| per crossing of every patch, d_e = |u_e - v| in output units
// With neutral weights, no offsets and iso = 0 every operation rounds as dmc.cu's, so the vertices are DiffDMC's.
// Forward:  fc_vertex_kernel (one thread per vertex: position, L_dev) and fc_split_kernel (one thread per quad).
// Backward: fc_quad_bwd_kernel (training: one thread per quad, the centre vertex's partials to its four corners and
// their cells' gamma, into P[Q, 4]); fc_cell_bwd_kernel (one thread per cell: every crossing's adjoint, including
// L_dev's and the centre vertices' (gathered through vq), and dalpha, dbeta, dgamma, written for every cell);
// fc_node_bwd_kernel (one thread per node: its <= 24 crossing records in a fixed order into dphi and ddeform).
// No float atomics: the gradients are bit-identical from run to run.
#include "common.cuh"
#include "dmc_cell.cuh"
#include "flexicubes_kernels.h"
#include "mc_kernels.h"
#include "mc_sweep.cuh"

namespace dgm {

__device__ __forceinline__ float fc_tanh_act(float a) { return 1.f + 0.99f * tanhf(a); }         // alpha, beta
__device__ __forceinline__ float fc_tanh_der(float a) { const float h = tanhf(a); return 0.99f * (1.f - h * h); }
__device__ __forceinline__ float fc_sig(float g) { return 1.f / (1.f + expf(-g)); }
__device__ __forceinline__ float fc_gamma_act(float g) { return 0.005f + 0.99f * fc_sig(g); }

// a cell's corners: s = phi - iso, position in grid units, alpha
struct FcCell {
  float s[8], x[8][3], al[8];
};

__device__ __forceinline__ size_t fc_wcell(int G, int i, int j, int k) {
  return ((size_t)i * (G - 1) + j) * (G - 1) + k;
}

__device__ __forceinline__ void fc_load(int G, float iso, const float* __restrict__ phi, const FcParams& w, int i,
                                        int j, int k, FcCell& c) {
  const size_t wc = fc_wcell(G, i, j, k);
#pragma unroll
  for (int r = 0; r < 8; ++r) {  // corner r = (i + (r & 1), j + ((r >> 1) & 1), k + (r >> 2))
    const int ni = i + (r & 1), nj = j + ((r >> 1) & 1), nk = k + (r >> 2);
    const size_t n = ((size_t)ni * G + nj) * G + nk;
    c.s[r] = phi[n] - iso;
    c.x[r][0] = (float)ni;
    c.x[r][1] = (float)nj;
    c.x[r][2] = (float)nk;
    if (w.deform) {
      c.x[r][0] += w.deform[3 * n + 0];
      c.x[r][1] += w.deform[3 * n + 1];
      c.x[r][2] += w.deform[3 * n + 2];
    }
    c.al[r] = w.alpha ? fc_tanh_act(w.alpha[wc * 8 + r]) : 1.f;
  }
}

__device__ __forceinline__ unsigned fc_case(const FcCell& c) {
  unsigned cs = 0;
#pragma unroll
  for (int r = 0; r < 8; ++r) cs |= (unsigned)(c.s[r] < 0.f) << r;  // s < 0 exactly when phi < iso
  return cs;
}

__device__ __forceinline__ void fc_load_beta(const FcParams& w, size_t wc, unsigned pmk, float be[12]) {
#pragma unroll
  for (int e = 0; e < 12; ++e) be[e] = (w.beta && ((pmk >> e) & 1u)) ? fc_tanh_act(w.beta[wc * 12 + e]) : 1.f;
}

// the crossing on edge e: returns t, writes u (grid units)
__device__ __forceinline__ float fc_cross(const FcCell& c, int e, float u[3]) {
  const int lo = mc_edge_lo(e), hi = lo + (1 << (e >> 2));
  const float w0 = c.al[lo] * c.s[lo], w1 = c.al[hi] * c.s[hi];
  const float t = w0 / (w0 - w1);
#pragma unroll
  for (int a = 0; a < 3; ++a) u[a] = c.x[lo][a] + t * (c.x[hi][a] - c.x[lo][a]);
  return t;
}

// the dual vertex of the patch with edge mask pmk (grid units); returns sum beta
__device__ __forceinline__ float fc_vertex(const FcCell& c, const float be[12], unsigned pmk, float v[3]) {
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, bs = 0.f;
#pragma unroll
  for (int e = 0; e < 12; ++e) {
    if ((pmk >> e) & 1u) {
      float u[3];
      fc_cross(c, e, u);
      s0 += be[e] * u[0];
      s1 += be[e] * u[1];
      s2 += be[e] * u[2];
      bs += be[e];
    }
  }
  v[0] = s0 / bs;
  v[1] = s1 / bs;
  v[2] = s2 / bs;
  return bs;
}

__device__ __forceinline__ float fc_norm(const float u[3], const float v[3]) {
  const float dx = u[0] - v[0], dy = u[1] - v[1], dz = u[2] - v[2];
  return sqrtf(dx * dx + dy * dy + dz * dz);
}

// one thread per vertex (V = min(V_counted, V_cap)): position (normalised), L_dev of its crossings (padded to
// FC_SLOTS) and its crossing count
__global__ void __launch_bounds__(256) fc_vertex_kernel(int G, float iso, const float* __restrict__ phi, FcParams w,
                                                        const long long* __restrict__ item_off, long long V_cap,
                                                        const int32_t* __restrict__ vsrc, float lsc,
                                                        float* __restrict__ verts, float* __restrict__ ldev,
                                                        int32_t* __restrict__ vk) {
  const long long V = min(item_off[1], V_cap);
  const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const uint32_t src = (uint32_t)vsrc[v], id = src >> 2;
  const int p = (int)(src & 3u);
  const int i = (int)(id / ((uint32_t)G * G)), j = (int)((id / G) % G), k = (int)(id % G);
  FcCell c;
  fc_load(G, iso, phi, w, i, j, k, c);
  const unsigned pmk = (unsigned)(__ldg(&g_dmc_pmask[fc_case(c)]) >> (16 * p)) & 0xfffu;
  float be[12], vg[3];
  fc_load_beta(w, fc_wcell(G, i, j, k), pmk, be);
  fc_vertex(c, be, pmk, vg);
  const float gm1 = (float)(G - 1);
#pragma unroll
  for (int a = 0; a < 3; ++a) verts[3 * v + a] = vg[a] / gm1;
  float dd[12], dsum = 0.f;
#pragma unroll
  for (int e = 0; e < 12; ++e) {
    dd[e] = 0.f;
    if ((pmk >> e) & 1u) {
      float u[3];
      fc_cross(c, e, u);
      dd[e] = fc_norm(u, vg) * lsc;
      dsum += dd[e];
    }
  }
  const int kk = __popc(pmk);
  const float mean = dsum / (float)kk;
  float* out = ldev + (size_t)v * FC_SLOTS;
  int slot = 0;
#pragma unroll
  for (int e = 0; e < 12; ++e)
    if ((pmk >> e) & 1u) out[slot++] = fabsf(dd[e] - mean);
  for (; slot < FC_SLOTS; ++slot) out[slot] = 0.f;
  vk[v] = kk;
}

__device__ __forceinline__ float fc_gamma_of(int G, const float* __restrict__ gamma, int32_t src) {
  if (!gamma) return 0.5f;
  const uint32_t id = (uint32_t)src >> 2;
  const int i = (int)(id / ((uint32_t)G * G)), j = (int)((id / G) % G), k = (int)(id % G);
  return fc_gamma_act(gamma[fc_wcell(G, i, j, k)]);
}

// one thread per quad (DiffDMC's order and orientation): the gamma split, or the centre vertex and four
// triangles.  Nothing is written when the vertices did not fit (the caller emits again).
__global__ void __launch_bounds__(256) fc_split_kernel(int G, const float* __restrict__ gamma,
                                                       const long long* __restrict__ item_off, long long V_cap,
                                                       long long Q_cap, bool training,
                                                       const int32_t* __restrict__ vsrc,
                                                       const int32_t* __restrict__ quads, float* verts,
                                                       int32_t* __restrict__ faces) {
  const long long V = item_off[1], Q = min(item_off[3], Q_cap);
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= Q || V > V_cap) return;
  int32_t qv[4];
  float gm[4];
#pragma unroll
  for (int n = 0; n < 4; ++n) {
    qv[n] = quads[4 * q + n];
    gm[n] = fc_gamma_of(G, gamma, vsrc[qv[n]]);
  }
  const float g02 = gm[0] * gm[2], g13 = gm[1] * gm[3];
  if (!training) {
    int32_t* f = faces + 6 * q;
    const bool d02 = g02 >= g13;
    f[0] = qv[0];
    f[1] = qv[1];
    f[2] = d02 ? qv[2] : qv[3];
    f[3] = d02 ? qv[0] : qv[1];
    f[4] = qv[2];
    f[5] = qv[3];
    return;
  }
  const long long m = V + q;
  const float den = g02 + g13 + 1e-8f;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float A = (verts[3 * (size_t)qv[0] + a] + verts[3 * (size_t)qv[2] + a]) * 0.5f;
    const float B = (verts[3 * (size_t)qv[1] + a] + verts[3 * (size_t)qv[3] + a]) * 0.5f;
    verts[3 * m + a] = (g02 * A + g13 * B) / den;
  }
  int32_t* f = faces + 12 * q;
#pragma unroll
  for (int n = 0; n < 4; ++n) {
    f[3 * n + 0] = qv[n];
    f[3 * n + 1] = qv[(n + 1) & 3];
    f[3 * n + 2] = (int32_t)m;
  }
}

__device__ __forceinline__ int fc_pick(const int x[3], int a) { return a == 0 ? x[0] : (a == 1 ? x[1] : x[2]); }

// training backward, one thread per quad: P[4q + n] = (dL/d v_n from the centre vertex, dL/d gamma of v_n's cell);
// vq[v_n * 12 + le] = 4q + n, le the edge of the quad in v_n's cell
__global__ void __launch_bounds__(256) fc_quad_bwd_kernel(int G, const float* __restrict__ gamma, int V, int Q,
                                                          const int32_t* __restrict__ vsrc,
                                                          const int32_t* __restrict__ quads,
                                                          const float* __restrict__ verts,
                                                          const float* __restrict__ dverts, float4* __restrict__ P,
                                                          int32_t* __restrict__ vq) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= Q) return;
  int32_t qv[4];
  int cc[4][3];
  float gm[4];
#pragma unroll
  for (int n = 0; n < 4; ++n) {
    qv[n] = quads[4 * (size_t)q + n];
    const int32_t src = vsrc[qv[n]];
    const uint32_t id = (uint32_t)src >> 2;
    cc[n][0] = (int)(id / ((uint32_t)G * G));
    cc[n][1] = (int)((id / G) % G);
    cc[n][2] = (int)(id % G);
    gm[n] = fc_gamma_of(G, gamma, src);
  }
  const float g02 = gm[0] * gm[2], g13 = gm[1] * gm[3];
  const float den = g02 + g13 + 1e-8f;
  float s02 = 0.f, s13 = 0.f, gmv[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float A = (verts[3 * (size_t)qv[0] + a] + verts[3 * (size_t)qv[2] + a]) * 0.5f;
    const float B = (verts[3 * (size_t)qv[1] + a] + verts[3 * (size_t)qv[3] + a]) * 0.5f;
    const float m = (g02 * A + g13 * B) / den;
    gmv[a] = dverts[3 * ((size_t)V + q) + a];
    s02 += gmv[a] * (A - m);
    s13 += gmv[a] * (B - m);
  }
  const float h02 = g02 * 0.5f / den, h13 = g13 * 0.5f / den;
  s02 /= den;
  s13 /= den;
  P[4 * (size_t)q + 0] = make_float4(gmv[0] * h02, gmv[1] * h02, gmv[2] * h02, gm[2] * s02);
  P[4 * (size_t)q + 2] = make_float4(gmv[0] * h02, gmv[1] * h02, gmv[2] * h02, gm[0] * s02);
  P[4 * (size_t)q + 1] = make_float4(gmv[0] * h13, gmv[1] * h13, gmv[2] * h13, gm[3] * s13);
  P[4 * (size_t)q + 3] = make_float4(gmv[0] * h13, gmv[1] * h13, gmv[2] * h13, gm[1] * s13);
  // the edge's axis a: the one along which q0's and q2's cells agree; the other two are b = a + 1, c = a + 2
  const int a = cc[0][0] == cc[2][0] ? 0 : (cc[0][1] == cc[2][1] ? 1 : 2);
  const int b = (a + 1) % 3, c = (a + 2) % 3;
#pragma unroll
  for (int n = 0; n < 4; ++n) {
    const int rb = 1 - (fc_pick(cc[n], b) - fc_pick(cc[0], b)), rc = 1 - (fc_pick(cc[n], c) - fc_pick(cc[0], c));
    const int le = 4 * a + (a == 1 ? (rc | (rb << 1)) : (rb | (rc << 1)));
    vq[(size_t)qv[n] * 12 + le] = 4 * q + n;
  }
}

// one thread per cell: the adjoints of every crossing of every patch with a vertex -> X[2 (v FC_SLOTS + slot)] =
// (dL/dphi(n0), dL/dphi(n1), t, dL/du.x), (dL/du.y, dL/du.z, -, -); dalpha, dbeta, dgamma of every cell
__global__ void __launch_bounds__(256) fc_cell_bwd_kernel(
    int G, float iso, const float* __restrict__ phi, FcParams w, bool training, float lsc,
    const unsigned long long* __restrict__ cvid, const float* __restrict__ dverts, const float* __restrict__ dldev,
    const float4* __restrict__ P, const int32_t* __restrict__ vq, float4* __restrict__ X, float* __restrict__ dalpha,
    float* __restrict__ dbeta, float* __restrict__ dgamma) {
  const size_t G1 = (size_t)(G - 1);
  const size_t wc = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (wc >= G1 * G1 * G1) return;
  const int i = (int)(wc / (G1 * G1)), j = (int)((wc / G1) % G1), k = (int)(wc % G1);
  unsigned cs = 0;
#pragma unroll
  for (int r = 0; r < 8; ++r)
    cs |= (unsigned)(phi[((size_t)(i + (r & 1)) * G + j + ((r >> 1) & 1)) * G + k + (r >> 2)] < iso) << r;
  const unsigned long long pm = __ldg(&g_dmc_pmask[cs]);
  const unsigned im = dmc_interior_edges(G, i, j, k);
  const unsigned need = (cs == 0u || cs == 255u) ? 0u : dmc_need(pm, im);
  float ga[8], gb[12], gg = 0.f;
#pragma unroll
  for (int r = 0; r < 8; ++r) ga[r] = 0.f;
#pragma unroll
  for (int e = 0; e < 12; ++e) gb[e] = 0.f;
  if (need) {
    FcCell c;
    fc_load(G, iso, phi, w, i, j, k, c);
    const float gm1 = (float)(G - 1);
    const uint32_t first = (uint32_t)cvid[((size_t)i * G + j) * G + k];
#pragma unroll 1
    for (int p = 0; p < 4; ++p) {
      if (!((need >> p) & 1u)) continue;
      const size_t v = first + (uint32_t)__popc(need & ((1u << p) - 1u));
      const unsigned pmk = (unsigned)(pm >> (16 * p)) & 0xfffu;
      float be[12], vg[3], gv[3];
      fc_load_beta(w, wc, pmk, be);
      const float bs = fc_vertex(c, be, pmk, vg);
#pragma unroll
      for (int a = 0; a < 3; ++a) gv[a] = dverts[3 * v + a];
      if (training) {
#pragma unroll
        for (int e = 0; e < 12; ++e) {
          if (((pmk & im) >> e) & 1u) {  // each interior edge of the patch is one quad's corner
            const float4 pq = P[vq[v * 12 + e]];
            gv[0] += pq.x;
            gv[1] += pq.y;
            gv[2] += pq.z;
            gg += pq.w;
          }
        }
      }
#pragma unroll
      for (int a = 0; a < 3; ++a) gv[a] /= gm1;  // w.r.t. the vertex in grid units
      // L_dev: entry_e = |d_e - mean d|; gd_e = dL/dd_e = g_e sgn_e - (sum_j g_j sgn_j) / k
      const int kk = __popc(pmk);
      float dd[12], mean = 0.f, sg = 0.f;
#pragma unroll
      for (int e = 0; e < 12; ++e) dd[e] = 0.f;
      if (dldev) {
        float dsum = 0.f;
#pragma unroll
        for (int e = 0; e < 12; ++e) {
          if ((pmk >> e) & 1u) {
            float u[3];
            fc_cross(c, e, u);
            dd[e] = fc_norm(u, vg) * lsc;
            dsum += dd[e];
          }
        }
        mean = dsum / (float)kk;
        int slot = 0;
#pragma unroll
        for (int e = 0; e < 12; ++e) {
          if ((pmk >> e) & 1u) {
            const float g = dldev[v * FC_SLOTS + slot++], x = dd[e] - mean;
            sg += x > 0.f ? g : (x < 0.f ? -g : 0.f);
          }
        }
        sg /= (float)kk;
        // the vertex's own share: d_e moves with -grad_u
        slot = 0;
#pragma unroll
        for (int e = 0; e < 12; ++e) {
          if ((pmk >> e) & 1u) {
            float u[3];
            fc_cross(c, e, u);
            const float g = dldev[v * FC_SLOTS + slot++], x = dd[e] - mean;
            const float gd = (x > 0.f ? g : (x < 0.f ? -g : 0.f)) - sg;
            const float n = fc_norm(u, vg);
            if (n > 0.f) {
              const float f = gd * lsc / n;
#pragma unroll
              for (int a = 0; a < 3; ++a) gv[a] -= f * (u[a] - vg[a]);
            }
          }
        }
      }
      int slot = 0;
#pragma unroll
      for (int e = 0; e < 12; ++e) {
        if ((pmk >> e) & 1u) {
          const int lo = mc_edge_lo(e), hi = lo + (1 << (e >> 2));
          float u[3], gu[3];
          const float t = fc_cross(c, e, u);
          const float wb = be[e] / bs;
          float gbe = 0.f;
#pragma unroll
          for (int a = 0; a < 3; ++a) {
            gu[a] = wb * gv[a];
            gbe += gv[a] * (u[a] - vg[a]);
          }
          gb[e] = gbe / bs;
          if (dldev) {
            const float g = dldev[v * FC_SLOTS + slot], x = dd[e] - mean;
            const float gd = (x > 0.f ? g : (x < 0.f ? -g : 0.f)) - sg;
            const float n = fc_norm(u, vg);
            if (n > 0.f) {
              const float f = gd * lsc / n;
#pragma unroll
              for (int a = 0; a < 3; ++a) gu[a] += f * (u[a] - vg[a]);
            }
          }
          float gt = 0.f;
#pragma unroll
          for (int a = 0; a < 3; ++a) gt += gu[a] * (c.x[hi][a] - c.x[lo][a]);
          const float w0 = c.al[lo] * c.s[lo], w1 = c.al[hi] * c.s[hi], d = w0 - w1;
          const float gw0 = gt * (-w1 / d) / d, gw1 = gt * (w0 / d) / d;  // dt/dw0 = -w1 / d^2, dt/dw1 = w0 / d^2
          ga[lo] += gw0 * c.s[lo];
          ga[hi] += gw1 * c.s[hi];
          float4* rec = X + 2 * (v * FC_SLOTS + slot);
          rec[0] = make_float4(gw0 * c.al[lo], gw1 * c.al[hi], t, gu[0]);
          rec[1] = make_float4(gu[1], gu[2], 0.f, 0.f);
          ++slot;
        }
      }
    }
  }
  if (dalpha) {
#pragma unroll
    for (int r = 0; r < 8; ++r) dalpha[wc * 8 + r] = ga[r] == 0.f ? 0.f : ga[r] * fc_tanh_der(w.alpha[wc * 8 + r]);
  }
  if (dbeta) {
#pragma unroll
    for (int e = 0; e < 12; ++e) dbeta[wc * 12 + e] = gb[e] == 0.f ? 0.f : gb[e] * fc_tanh_der(w.beta[wc * 12 + e]);
  }
  if (dgamma) {
    float d = 0.f;
    if (gg != 0.f) {
      const float sg = fc_sig(w.gamma[wc]);
      d = gg * 0.99f * sg * (1.f - sg);
    }
    dgamma[wc] = d;
  }
}

// dL/dphi and dL/ddeform at one node: the six grid edges at the node, along -x, +x, -y, +y, -z, +z; on each cut one
// the four cells around it (those in the grid), in a fixed order, each through its patch of that edge when the
// patch has a vertex (the cell order of dmc_backward_kernel).  Every node is written.
__global__ void __launch_bounds__(256) fc_node_bwd_kernel(int G, const float* __restrict__ phi, float iso,
                                                          const unsigned long long* __restrict__ cvid,
                                                          const float4* __restrict__ X, float* __restrict__ dphi,
                                                          float* __restrict__ ddeform) {
  const size_t G3 = (size_t)G * G * G;
  const size_t m = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= G3) return;
  const int mi = (int)(m / ((size_t)G * G)), mj = (int)((m / G) % G), mk = (int)(m % G);
  const size_t st[3] = {(size_t)G * G, (size_t)G, 1};
  const int mc[3] = {mi, mj, mk};
  float f[3][3][3];
  f[1][1][1] = phi[m];
  const bool sc = f[1][1][1] < iso;
  bool any = false;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
#pragma unroll
    for (int sd = 0; sd < 2; ++sd) {
      const bool ok = sd ? mc[a] + 1 < G : mc[a] >= 1;
      const float val = ok ? phi[sd ? m + st[a] : m - st[a]] : 0.f;
      any |= ok && ((val < iso) != sc);
    }
  }
  if (!any) {
    dphi[m] = 0.f;
    if (ddeform) ddeform[3 * m] = ddeform[3 * m + 1] = ddeform[3 * m + 2] = 0.f;
    return;
  }
#pragma unroll
  for (int di = 0; di < 3; ++di)
#pragma unroll
    for (int dj = 0; dj < 3; ++dj)
#pragma unroll
      for (int dk = 0; dk < 3; ++dk) {
        const int ni = mi + di - 1, nj = mj + dj - 1, nk = mk + dk - 1;
        const bool ok = ni >= 0 && ni < G && nj >= 0 && nj < G && nk >= 0 && nk < G;
        f[di][dj][dk] = ok ? phi[((size_t)ni * G + nj) * G + nk] : 0.f;
      }
  float acc = 0.f, dx[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int b = (a + 1) % 3, c = (a + 2) % 3;
#pragma unroll
    for (int sd = 0; sd < 2; ++sd) {  // sd = 0: the edge (m - e_a, m), m its upper node; sd = 1: (m, m + e_a)
      if (!(sd ? mc[a] + 1 < G : mc[a] >= 1)) continue;
      const int oa = sd ? 2 : 0;
      const float po = a == 0 ? f[oa][1][1] : (a == 1 ? f[1][oa][1] : f[1][1][oa]);
      if ((po < iso) == sc) continue;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int db = q & 1, dc = q >> 1;
        int o[3];
        o[a] = sd ? 0 : -1;
        o[b] = -db;
        o[c] = -dc;
        const int ci = mi + o[0], cj = mj + o[1], ck = mk + o[2];
        if (ci < 0 || cj < 0 || ck < 0 || ci > G - 2 || cj > G - 2 || ck > G - 2) continue;
        unsigned cs = 0;
#pragma unroll
        for (int cr = 0; cr < 8; ++cr)
          cs |= (unsigned)(f[o[0] + 1 + (cr & 1)][o[1] + 1 + ((cr >> 1) & 1)][o[2] + 1 + (cr >> 2)] < iso) << cr;
        const int lo_e = 4 * a + (a == 1 ? (dc | (db << 1)) : (db | (dc << 1)));
        const unsigned p = (unsigned)(__ldg(&g_dmc_pof[cs]) >> (4 * lo_e)) & 15u;
        const unsigned long long pm = __ldg(&g_dmc_pmask[cs]);
        const unsigned need = dmc_need(pm, dmc_interior_edges(G, ci, cj, ck));
        if (!(need & (1u << p))) continue;
        const size_t cell = ((size_t)ci * G + cj) * G + ck;
        const size_t v = (uint32_t)cvid[cell] + (uint32_t)__popc(need & ((1u << p) - 1u));
        const unsigned pmk = (unsigned)(pm >> (16 * p)) & 0xfffu;
        const size_t slot = (size_t)__popc(pmk & ((1u << lo_e) - 1u));
        const float4 r0 = X[2 * (v * FC_SLOTS + slot)], r1 = X[2 * (v * FC_SLOTS + slot) + 1];
        acc += sd ? r0.x : r0.y;  // sd = 1: m is the edge's lower node n0
        const float wgt = sd ? 1.f - r0.z : r0.z;
        dx[0] += wgt * r0.w;
        dx[1] += wgt * r1.x;
        dx[2] += wgt * r1.y;
      }
    }
  }
  dphi[m] = acc;
  if (ddeform) {
    ddeform[3 * m + 0] = dx[0];
    ddeform[3 * m + 1] = dx[1];
    ddeform[3 * m + 2] = dx[2];
  }
}

cudaError_t launch_fc_emit(int G, const float* phi, float iso, const FcParams& w, bool training, bool normalize,
                           void* ws, float* verts, int32_t* vsrc, float* ldev, int32_t* vk, long long V_cap,
                           int32_t* faces, int32_t* quads, long long Q_cap, cudaStream_t s) {
  cudaError_t e = upload_dmc_tables();
  if (e != cudaSuccess) return e;
  e = launch_dmc_emit(1, G, phi, iso, ws, verts, vsrc, V_cap, faces, quads, Q_cap, s);
  if (e != cudaSuccess) return e;
  DmcWS dw = DmcWS::from((char*)ws, G, 1);
  const float lsc = normalize ? 1.f / (float)(G - 1) : 1.f;
  if (V_cap > 0)
    fc_vertex_kernel<<<(unsigned)((V_cap + 255) / 256), 256, 0, s>>>(G, iso, phi, w, dw.item_off, V_cap, vsrc, lsc,
                                                                      verts, ldev, vk);
  if (Q_cap > 0)
    fc_split_kernel<<<(unsigned)((Q_cap + 255) / 256), 256, 0, s>>>(G, w.gamma, dw.item_off, V_cap, Q_cap, training,
                                                                     vsrc, quads, verts, faces);
  return cudaGetLastError();
}

struct FcBwdWS {
  DmcWS dmc;
  float4* X;    // [V FC_SLOTS, 2]: every crossing's record
  int32_t* vq;  // [V, 12] (training): the quad corner of every (vertex, interior edge)
  float4* P;    // [Q, 4] (training): the centre vertices' partials
  static FcBwdWS from(char* base, int G, long long V, long long Q, bool training, size_t* bytes = nullptr) {
    FcBwdWS w;
    size_t db;
    w.dmc = DmcWS::from(base, G, 1, &db);
    char* p = base + db;
    w.X = carve<float4>(p, (size_t)V * FC_SLOTS * 2);
    w.vq = carve<int32_t>(p, training ? (size_t)V * 12 : 0);
    w.P = carve<float4>(p, training ? (size_t)Q * 4 : 0);
    if (bytes) *bytes = size_t(p - base) + 128;
    return w;
  }
};

size_t fc_backward_ws_bytes(int G, long long V, long long Q, bool training) {
  size_t b;
  FcBwdWS::from(nullptr, G, V, Q, training, &b);
  return b;
}

cudaError_t launch_fc_backward(int G, int V, int Q, const float* phi, float iso, const FcParams& w, bool training,
                               bool normalize, const float* verts, const int32_t* vsrc, const int32_t* quads,
                               const float* dverts, const float* dldev, void* ws, float* dphi, float* ddeform,
                               float* dalpha, float* dbeta, float* dgamma, cudaStream_t s) {
  cudaError_t e = upload_dmc_tables();
  if (e != cudaSuccess) return e;
  FcBwdWS b = FcBwdWS::from((char*)ws, G, V, Q, training);
  McItems it;
  it.B = 1;
  it.voff[0] = 0;
  it.voff[1] = V;
  launch_dmc_first_vertex(G, it, vsrc, b.dmc.cvid, s);
  if (training && Q > 0)
    fc_quad_bwd_kernel<<<(Q + 255) / 256, 256, 0, s>>>(G, w.gamma, V, Q, vsrc, quads, verts, dverts, b.P, b.vq);
  const size_t G1 = (size_t)(G - 1), cells = G1 * G1 * G1, G3 = (size_t)G * G * G;
  const float lsc = normalize ? 1.f / (float)(G - 1) : 1.f;
  fc_cell_bwd_kernel<<<(unsigned)((cells + 255) / 256), 256, 0, s>>>(G, iso, phi, w, training, lsc, b.dmc.cvid,
                                                                      dverts, dldev, b.P, b.vq, b.X, dalpha, dbeta,
                                                                      dgamma);
  fc_node_bwd_kernel<<<(unsigned)((G3 + 255) / 256), 256, 0, s>>>(G, phi, iso, b.dmc.cvid, b.X, dphi, ddeform);
  return cudaGetLastError();
}

}  // namespace dgm
