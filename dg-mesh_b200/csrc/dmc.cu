// dmc.cu -- differentiable dual marching cubes (Nielson 2004) on a G^3 scalar grid, forward and backward.
//
// Stands in for `diso.DiffDMC`.  A cell's surface patches are the loops of its marching-cubes case
// (tools/gen_mc_tables.py: DMC_PATCH, DMC_PATCH_OF_EDGE); every patch that has an interior edge (one whose four
// incident cells all lie in the grid) gets one dual vertex, the fp32 mean of its edge crossings, summed in
// increasing edge id.  Every sign-changing interior edge gives one quad over the four cells around it, split
// into two triangles at its lowest cell.  Same brick sweep as mc.cu (mc_sweep.cuh) and the same protocol:
//   count   per brick: ONE packed (dual vertices | quads << 32) total                               [reads phi once]
//   scan    the brick totals and the item totals (launch_mc_scan_totals, shared with marching cubes)
//   emit    only bricks that own something re-read it: dual vertices, vsrc = cell * 4 + patch, cvid[cell] =
//           first vertex | case << 32 (sparse), and each quad as the reference lowest cell * 3 + axis, owned by
//           the cell whose edge 4 * axis + 3 it is
//   resolve one thread per quad turns the reference into two triangles (and the quad) through cvid
// Backward: vsrc rebuilds every cell's first vertex; then one thread per NODE gathers, in a fixed order, the
// <= 24 (cell, patch) terms of its six edges: the gradient is bit-identical from run to run, no float atomics.
#include "common.cuh"
#include "dmc_cell.cuh"
#include "mc_kernels.h"
#include "mc_sweep.cuh"

namespace dgm {

// quads a cell owns: its cut interior edges 3, 7, 11 (the x, y and z edges through corner 7)
#define DMC_QUAD_EDGES 0x888u

// dual vertices | quads << 16 of cell (i, j, k) of case cs (0 for a node that is not a cell's lowest corner)
__device__ __forceinline__ unsigned dmc_cell_count(int G, int i, int j, int k, unsigned cs) {
  if (cs == 0u || cs == 255u) return 0u;
  const unsigned long long pm = __ldg(&g_dmc_pmask[cs]);
  const unsigned im = dmc_interior_edges(G, i, j, k);
  return (unsigned)__popc(dmc_need(pm, im)) | ((unsigned)__popc(dmc_cut(pm) & im & DMC_QUAD_EDGES) << 16);
}

__global__ void __launch_bounds__(32 * MC_WARPS) dmc_count_kernel(McGeom g, size_t nall, const float* __restrict__ phi,
                                                                  float iso,
                                                                  unsigned long long* __restrict__ blk_counts) {
  const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const size_t brick = (size_t)blockIdx.x * MC_WARPS + wid;
  if (brick >= nall) return;
  const size_t item = brick / g.nbricks;
  McBrick B;
  mc_load_brick(g, brick - item * g.nbricks, lane, phi + item * g.G * g.G * g.G, B);
  {
    bool neg, pos;
    mc_brick_sides(g, B, lane, iso, neg, pos);
    if (!(__any_sync(0xffffffffu, neg) && __any_sync(0xffffffffu, pos))) {
      if (lane == 0) blk_counts[brick] = 0ull;
      return;
    }
  }
  unsigned c = 0;  // dual vertices | quads << 16: <= 1024 / 768 per brick
#pragma unroll
  for (int r = 0; r < MC_BJ; ++r) {
    unsigned mask, cs;
    mc_classify(g, B, r, iso, mask, cs);
    c += dmc_cell_count(g.G, B.i, B.j0 + r, B.k, cs);
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if (lane == 0) blk_counts[brick] = (unsigned long long)(c & 0xffffu) | ((unsigned long long)(c >> 16) << 32);
}

// item k's dual vertices and quads follow those of items 0..k-1 (item_off); cvid, vsrc and the quad references are
// local to the item
__global__ void __launch_bounds__(32 * MC_WARPS) dmc_emit_kernel(
    McGeom g, int items, const float* __restrict__ phi, float iso, const unsigned long long* __restrict__ blk_counts,
    const unsigned long long* __restrict__ blk_offsets, const long long* __restrict__ item_off,
    unsigned long long* __restrict__ cvid, float* __restrict__ verts, int32_t* __restrict__ vsrc, long long V_cap,
    int32_t* __restrict__ faces, long long Q_cap) {
  const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const size_t brick = (size_t)blockIdx.x * MC_WARPS + wid;
  if (brick >= (size_t)items * g.nbricks || blk_counts[brick] == 0) return;
  const size_t item = brick / g.nbricks, G3 = (size_t)g.G * g.G * g.G;
  McBrick B;
  mc_load_brick(g, brick - item * g.nbricks, lane, phi + item * G3, B);
  unsigned css[MC_BJ];
  unsigned mine = 0;
#pragma unroll
  for (int r = 0; r < MC_BJ; ++r) {
    unsigned mask;
    mc_classify(g, B, r, iso, mask, css[r]);
    mine += dmc_cell_count(g.G, B.i, B.j0 + r, B.k, css[r]);
  }
  unsigned inc = mine;  // inclusive prefix over the lanes (order inside the brick: lane-major, then r)
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned up = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= (unsigned)o) inc += up;
  }
  if (mine == 0) return;
  const unsigned excl = inc - mine;
  const unsigned long long base = blk_offsets[brick] - blk_offsets[item * g.nbricks];
  unsigned long long vl = (base & 0xffffffffull) + (excl & 0xffffu);  // the item's own vertex index
  const long long v0 = item_off[item];                               // + vl: the batch's vertex index
  long long q = item_off[items + 1 + item] + (long long)(base >> 32) + (excl >> 16);
  const int G = g.G;
  const float gm1 = (float)(G - 1);
#pragma unroll
  for (int r = 0; r < MC_BJ; ++r) {
    const unsigned cs = css[r];
    if (cs == 0u || cs == 255u) continue;
    const int j = B.j0 + r;
    const unsigned long long pm = __ldg(&g_dmc_pmask[cs]);
    const unsigned im = dmc_interior_edges(G, B.i, j, B.k);
    const unsigned need = dmc_need(pm, im), qm = dmc_cut(pm) & im & DMC_QUAD_EDGES;
    const size_t id = ((size_t)B.i * G + j) * G + B.k;
    if (need) {
      cvid[item * G3 + id] = vl | ((unsigned long long)cs << 32);
      const unsigned long long pof = __ldg(&g_dmc_pof[cs]);
      // corner c = (i + (c & 1), j + ((c >> 1) & 1), k + (c >> 2)), as mc_classify
      const float v[8] = {B.a[0][r], B.a[1][r], B.a[0][r + 1], B.a[1][r + 1],
                          B.z[0][r], B.z[1][r], B.z[0][r + 1], B.z[1][r + 1]};
      float s[4][3];
#pragma unroll
      for (int p = 0; p < 4; ++p) s[p][0] = s[p][1] = s[p][2] = 0.f;
#pragma unroll
      for (int e = 0; e < 12; ++e) {  // every crossing exactly as mc.cu computes its vertex, added in edge order
        const unsigned pe = (unsigned)(pof >> (4 * e)) & 15u;
        if (pe < 4u) {
          const int a = e >> 2, lo = mc_edge_lo(e), hi = lo + (1 << a);
          const float t = (iso - v[lo]) / (v[hi] - v[lo]);
          float pos[3] = {(float)(B.i + (lo & 1)), (float)(j + ((lo >> 1) & 1)), (float)(B.k + (lo >> 2))};
          pos[a] += t;
#pragma unroll
          for (int p = 0; p < 4; ++p)
            if (pe == (unsigned)p) {
              s[p][0] += pos[0];
              s[p][1] += pos[1];
              s[p][2] += pos[2];
            }
        }
      }
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        if (need & (1u << p)) {
          const long long vv = v0 + (long long)vl;
          if (vv < V_cap) {
            const float kf = (float)__popc((unsigned)(pm >> (16 * p)) & 0xfffu);
            verts[3 * vv + 0] = s[p][0] / kf / gm1;  // IEEE divisions: identical to the numpy restatement
            verts[3 * vv + 1] = s[p][1] / kf / gm1;
            verts[3 * vv + 2] = s[p][2] / kf / gm1;
            vsrc[vv] = (int32_t)(id * 4 + p);  // < 4 G^3 < 2^31 for G <= 800
          }
          ++vl;
        }
      }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (qm & (8u << (4 * a))) {
        if (q < Q_cap) faces[6 * q] = (int32_t)(id * 3 + a);  // resolved by dmc_resolve_kernel
        ++q;
      }
    }
  }
}

// one thread per quad: the reference lowest cell * 3 + axis a -> the four cells around the edge through that
// cell's corner 7 along a, in cyclic order c, c + e_b, c + e_b + e_c, c + e_c ((a, b, c) cyclic: normal +a),
// reversed when the edge's lower node is outside, so that the normal points from the inside node to the outside
// one; triangles (q0, q1, q2), (q0, q2, q3).  qoff = item_off + items + 1: the batch's first quad of every item.
__global__ void __launch_bounds__(256) dmc_resolve_kernel(int G, int items, const long long* __restrict__ qoff,
                                                          long long Q_cap, const unsigned long long* __restrict__ cvid,
                                                          int32_t* __restrict__ faces, int32_t* __restrict__ quads) {
  const long long n = min(qoff[items], Q_cap);
  const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= n) return;
  int lo = 0, hi = items - 1;  // the item of quad x: the last k with qoff[k] <= x
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (qoff[mid] <= x) lo = mid;
    else hi = mid - 1;
  }
  const size_t G3 = (size_t)G * G * G;
  cvid += (size_t)lo * G3;
  const uint32_t ref = (uint32_t)faces[6 * x];
  const uint32_t c = ref / 3;
  const int a = (int)(ref % 3);
  const int ci = (int)(c / ((uint32_t)G * G)), cj = (int)((c / G) % G), ck = (int)(c % G);
  // e_b and e_c: b = (a + 1) % 3, c = (a + 2) % 3
  const int bi = a == 2, bj = a == 0, bk = a == 1, ei = a == 1, ej = a == 2, ek = a == 0;
  const size_t sb = (size_t)bi * G * G + (size_t)bj * G + bk, sc = (size_t)ei * G * G + (size_t)ej * G + ek;
  // local edge of the cell at offset (db, dc) from c: the edge's lower node is at (1 - db, 1 - dc) across the
  // edge; combo bit 0 belongs to the lower-numbered of b and c (c when a = 1)
  auto le = [&](int db, int dc) {
    const int rb = 1 - db, rc = 1 - dc;
    return 4 * a + (a == 1 ? (rc | (rb << 1)) : (rb | (rc << 1)));
  };
  const unsigned long long w0 = cvid[c];
  const uint32_t q0 = dmc_vertex_of(G, w0, ci, cj, ck, le(0, 0));
  const uint32_t q1 = dmc_vertex_of(G, cvid[c + sb], ci + bi, cj + bj, ck + bk, le(1, 0));
  const uint32_t q2 = dmc_vertex_of(G, cvid[c + sb + sc], ci + bi + ei, cj + bj + ej, ck + bk + ek, le(1, 1));
  const uint32_t q3 = dmc_vertex_of(G, cvid[c + sc], ci + ei, cj + ej, ck + ek, le(0, 1));
  // corner e_b + e_c of cell c is the edge's lower node: corner id (1 << b) | (1 << c) = 7 - (1 << a)
  const bool in = ((w0 >> 32) >> (7 - (1 << a))) & 1ull;
  const uint32_t o1 = in ? q1 : q3, o3 = in ? q3 : q1;
  int32_t* f = faces + 6 * x;
  f[0] = (int32_t)q0;
  f[1] = (int32_t)o1;
  f[2] = (int32_t)q2;
  f[3] = (int32_t)q0;
  f[4] = (int32_t)q2;
  f[5] = (int32_t)o3;
  if (quads) {
    quads[4 * x + 0] = (int32_t)q0;
    quads[4 * x + 1] = (int32_t)o1;
    quads[4 * x + 2] = (int32_t)q2;
    quads[4 * x + 3] = (int32_t)o3;
  }
}

// the backward's cell table: cvid[cell] = the cell's first dual vertex (item-local), from vsrc (a cell's vertices
// are consecutive, in increasing patch)
__global__ void __launch_bounds__(256) dmc_first_vertex_kernel(size_t G3, McItems it,
                                                               const int32_t* __restrict__ vsrc,
                                                               unsigned long long* __restrict__ cvid) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= it.voff[it.B]) return;
  int lo = 0, hi = it.B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (it.voff[mid] <= v) lo = mid;
    else hi = mid - 1;
  }
  const uint32_t cell = (uint32_t)vsrc[v] >> 2;
  if (v == it.voff[lo] || ((uint32_t)vsrc[v - 1] >> 2) != cell) cvid[(size_t)lo * G3 + cell] = (unsigned)(v - it.voff[lo]);
}

// dL/dphi at one node: the six grid edges at the node, along -x, +x, -y, +y, -z, +z; on each cut one the four
// cells around it (those in the grid), in a fixed order; a cell contributes through its patch of that edge when
// the patch has a dual vertex: d vert / d t = 1 / (k (G - 1)) along the edge for a k-edge patch, and dt / d phi as
// in mc.cu.  Every node is written.
__global__ void __launch_bounds__(256) dmc_backward_kernel(int G, McItems it, const float* __restrict__ phi, float iso,
                                                           const unsigned long long* __restrict__ cvid,
                                                           const float* __restrict__ dverts,
                                                           float* __restrict__ dphi) {
  const size_t G3 = (size_t)G * G * G;
  const size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= (size_t)it.B * G3) return;
  const int item = (int)(x / G3);
  const size_t m = x - (size_t)item * G3;
  phi += (size_t)item * G3;
  cvid += (size_t)item * G3;
  const int mi = (int)(m / ((size_t)G * G)), mj = (int)((m / G) % G), mk = (int)(m % G);
  const size_t st[3] = {(size_t)G * G, (size_t)G, 1};
  const int mc[3] = {mi, mj, mk};
  // f[di][dj][dk] = phi at (mi + di - 1, mj + dj - 1, mk + dk - 1) when that node is in the grid
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
    dphi[x] = 0.f;
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
  const float gm1 = (float)(G - 1);
  const int voff = it.voff[item];
  float acc = 0.f;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int b = (a + 1) % 3, c = (a + 2) % 3;
#pragma unroll
    for (int sd = 0; sd < 2; ++sd) {  // sd = 0: the edge (m - e_a, m), m its upper node; sd = 1: (m, m + e_a)
      if (!(sd ? mc[a] + 1 < G : mc[a] >= 1)) continue;
      const int oa = sd ? 2 : 0;  // the other node, index along a in f
      const float po = a == 0 ? f[oa][1][1] : (a == 1 ? f[1][oa][1] : f[1][1][oa]);
      if ((po < iso) == sc) continue;
      const float p0 = sd ? f[1][1][1] : po, p1 = sd ? po : f[1][1][1];
      const float d = p1 - p0;
      const float t = (iso - p0) / d, u = (p1 - iso) / d;
      const float dt = sd ? -u / d : -t / d;  // d t / d phi(m)
#pragma unroll
      for (int q = 0; q < 4; ++q) {  // the cell at offset (-db, -dc) across the edge from its lower node
        const int db = q & 1, dc = q >> 1;
        int o[3];           // the cell's lowest corner, offset from m
        o[a] = sd ? 0 : -1;
        o[b] = -db;
        o[c] = -dc;
        const int ci = mi + o[0], cj = mj + o[1], ck = mk + o[2];
        if (ci < 0 || cj < 0 || ck < 0 || ci > G - 2 || cj > G - 2 || ck > G - 2) continue;
        unsigned cs = 0;
#pragma unroll
        for (int cr = 0; cr < 8; ++cr)
          cs |= (unsigned)(f[o[0] + 1 + (cr & 1)][o[1] + 1 + ((cr >> 1) & 1)][o[2] + 1 + (cr >> 2)] < iso) << cr;
        const int rb = db, rc = dc;  // the edge's lower node in the cell, across the edge
        const int lo_e = 4 * a + (a == 1 ? (rc | (rb << 1)) : (rb | (rc << 1)));
        const unsigned p = (unsigned)(__ldg(&g_dmc_pof[cs]) >> (4 * lo_e)) & 15u;
        const unsigned long long pm = __ldg(&g_dmc_pmask[cs]);
        const unsigned need = dmc_need(pm, dmc_interior_edges(G, ci, cj, ck));
        if (!(need & (1u << p))) continue;
        const size_t cell = ((size_t)ci * G + cj) * G + ck;
        const int v = voff + (int)((uint32_t)cvid[cell] + (uint32_t)__popc(need & ((1u << p) - 1u)));
        const float kf = (float)__popc((unsigned)(pm >> (16 * p)) & 0xfffu);
        acc += dverts[3 * (size_t)v + a] / gm1 / kf * dt;
      }
    }
  }
  dphi[x] = acc;
}

DmcWS DmcWS::from(char* base, int G, int B, size_t* bytes) {
  char* p = base;
  DmcWS w;
  const size_t n = (size_t)G * G * G, nb = (size_t)B * mc_num_blocks(G);
  w.blk_counts = carve<unsigned long long>(p, nb);
  w.blk_offsets = carve<unsigned long long>(p, nb);
  w.item_off = carve<long long>(p, 2 * (size_t)B + 2);
  w.cub_bytes = mc_cub_bytes(nb);
  w.cub_temp = carve<char>(p, w.cub_bytes);
  w.cvid = carve<unsigned long long>(p, (size_t)B * n);  // sparse: only cells with dual vertices are written or read
  if (bytes) *bytes = size_t(p - base) + 128;
  return w;
}

cudaError_t launch_dmc_count(int B, int G, const float* phi, float iso, void* ws, int32_t* totals,
                             int32_t* totals_host, cudaEvent_t ev, cudaStream_t s) {
  cudaError_t e = upload_dmc_tables();
  if (e != cudaSuccess) return e;
  DmcWS w = DmcWS::from((char*)ws, G, B);
  const McGeom g = mc_geom(G);
  const size_t nb = mc_num_blocks(G), nall = (size_t)B * nb;
  dmc_count_kernel<<<(unsigned)((nall + MC_WARPS - 1) / MC_WARPS), 32 * MC_WARPS, 0, s>>>(g, nall, phi, iso,
                                                                                           w.blk_counts);
  return launch_mc_scan_totals(B, nb, w.blk_counts, w.blk_offsets, w.item_off, w.cub_temp, w.cub_bytes, totals,
                               totals_host, ev, s);
}

cudaError_t launch_dmc_emit(int B, int G, const float* phi, float iso, void* ws, float* verts, int32_t* vsrc,
                            long long V_cap, int32_t* faces, int32_t* quads, long long Q_cap, cudaStream_t s) {
  DmcWS w = DmcWS::from((char*)ws, G, B);
  const McGeom g = mc_geom(G);
  const size_t nall = (size_t)B * mc_num_blocks(G);
  dmc_emit_kernel<<<(unsigned)((nall + MC_WARPS - 1) / MC_WARPS), 32 * MC_WARPS, 0, s>>>(
      g, B, phi, iso, w.blk_counts, w.blk_offsets, w.item_off, w.cvid, verts, vsrc, V_cap, faces, Q_cap);
  if (Q_cap > 0)
    dmc_resolve_kernel<<<(unsigned)((Q_cap + 255) / 256), 256, 0, s>>>(G, B, w.item_off + B + 1, Q_cap, w.cvid,
                                                                       faces, quads);
  return cudaGetLastError();
}

void launch_dmc_first_vertex(int G, const McItems& it, const int32_t* vsrc, unsigned long long* cvid,
                             cudaStream_t s) {
  const int V = it.voff[it.B];
  if (V > 0) dmc_first_vertex_kernel<<<(V + 255) / 256, 256, 0, s>>>((size_t)G * G * G, it, vsrc, cvid);
}

cudaError_t launch_dmc_backward(int G, const McItems& it, const float* phi, float iso, void* ws, const int32_t* vsrc,
                                const float* dverts, float* dphi, cudaStream_t s) {
  cudaError_t e = upload_dmc_tables();
  if (e != cudaSuccess) return e;
  DmcWS w = DmcWS::from((char*)ws, G, it.B);
  const size_t G3 = (size_t)G * G * G, n = (size_t)it.B * G3;
  launch_dmc_first_vertex(G, it, vsrc, w.cvid, s);
  dmc_backward_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(G, it, phi, iso, w.cvid, dverts, dphi);
  return cudaGetLastError();
}

}  // namespace dgm
