// mc.cu -- differentiable marching cubes on a G^3 scalar grid (iso-surface extraction + backward).
//
// Stands in for `diso.DiffMC.__call__(grid, deform=None, isovalue=0.0)` as DG-Mesh calls it
// (dgmesh/utils/renderer.py:171, dgmesh/scene/gaussian_model_dpsr_dynamic_anchor.py:704,851):
//   phi[G,G,G] fp32 -> verts[V,3] in [0,1]^3 (grid index / (G-1)), faces[F,3] int32.
// `diso` is a third-party CUDA package that is not in the reference tree (SURVEY.md 8(c)): its
// vertex / face ORDER cannot be reproduced, only the surface.  Case tables are derived by
// tools/gen_mc_tables.py (watertight by construction).
//
// Warp-per-brick sweep.  A BRICK is 8 (j) x 32 (k) nodes of one i-plane; a warp owns one brick: lane = k, and
// every lane loads the 9 rows (j .. j+8) of planes i and i+1 at its k -- 18 independent, fully coalesced loads
// in flight per lane, 2.25 loads per node instead of 8 -- the k+1 neighbours come from the next lane by shuffle
// (lane 31 fetches its own).  No shared memory, no CTA barrier.  Hierarchical counting instead of a per-node scan:
//   count   per brick: ONE packed (vertices | triangles << 32) total                              [reads phi once]
//   scan    cub::DeviceScan over the n/256 brick totals (library primitive), totals -> device + mapped host
//   emit    only warps whose brick owns something re-read it (a few % of the grid): a warp prefix sum gives
//           every vertex its index; vertices are written, the owner table vid[node] = first vertex |
//           edge mask << 29 is filled SPARSELY (only nodes that own vertices are ever looked up), faces are
//           written as encoded owner references (node * 3 + axis), and vsrc[v] remembers each vertex's edge
//           (a caller-owned [V_cap] array: V reaches ~1.45 G^3 on independent noise, up to 3 G^2 (G - 1))
//   resolve 3F threads turn the owner references into vertex indices through vid[]
// Backward: one thread per VERTEX (vsrc), d verts / d phi through t = (iso - phi0) / (phi1 - phi0).
// Scratch traffic is 8 B per brick instead of 26 B per node: the sweep is bound by reading phi once
// (4 G^3 bytes, SURVEY.md 8(d)) rather than by its own bookkeeping.
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "mc_kernels.h"
#include "mc_sweep.cuh"
#include "mc_tables.h"

namespace dgm {

// case tables in GLOBAL memory, read through the read-only path: the case index differs from lane to lane, and a
// __constant__ access with divergent addresses is replayed once per distinct address (measured: the emit pass
// spent most of its time there); L1-cached loads are not
__device__ unsigned char g_ntri[256];
__device__ signed char g_tri[256][MC_MAX_TRI * 3];
__device__ __forceinline__ unsigned mc_ntri(unsigned cs) { return (cs == 0u || cs == 255u) ? 0u : __ldg(&g_ntri[cs]); }

size_t mc_num_blocks(int G) { return mc_geom(G).nbricks; }
// a batch of grids phi[items, G, G, G] is swept as items * nbricks bricks; brick b belongs to item b / nbricks
__global__ void __launch_bounds__(32 * MC_WARPS) mc_count_kernel(McGeom g, size_t nall, const float* __restrict__ phi,
                                                                 float iso,
                                                                 unsigned long long* __restrict__ blk_counts) {
  const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const size_t brick = (size_t)blockIdx.x * MC_WARPS + wid;
  if (brick >= nall) return;
  const size_t item = brick / g.nbricks;
  McBrick B;
  mc_load_brick(g, brick - item * g.nbricks, lane, phi + item * g.G * g.G * g.G, B);
  // the common case (>95 % of a 288^3 grid): every value the brick touches lies on one side of the level set --
  // nothing to classify.  Lanes look at their own valid values (lane 31 also at its k + 1 column).
  {
    bool neg = false, pos = false;
#pragma unroll
    for (int r = 0; r <= MC_BJ; ++r) {
      const bool jin = B.j0 + r < g.G;
#pragma unroll
      for (int pl = 0; pl < 2; ++pl) {
        const bool ok = jin && B.kin && (pl == 0 || B.xi);
        const bool s = B.a[pl][r] < iso;
        neg |= ok && s;
        pos |= ok && !s;
        if (lane == 31) {
          const bool okz = jin && B.zk && (pl == 0 || B.xi);
          const bool sz = B.z[pl][r] < iso;
          neg |= okz && sz;
          pos |= okz && !sz;
        }
      }
    }
    if (!(__any_sync(0xffffffffu, neg) && __any_sync(0xffffffffu, pos))) {
      if (lane == 0) blk_counts[brick] = 0ull;
      return;
    }
  }
  unsigned c = 0;  // vertices | triangles << 16: <= 768 / 1280 per brick
#pragma unroll
  for (int r = 0; r < MC_BJ; ++r) {
    unsigned mask, cs;
    mc_classify(g, B, r, iso, mask, cs);
    c += __popc(mask) | (mc_ntri(cs) << 16);
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if (lane == 0) blk_counts[brick] = (unsigned long long)(c & 0xffffu) | ((unsigned long long)(c >> 16) << 32);
}

// {V_k, F_k} of every item -> the workspace's item offsets (emit and resolve), the caller's device pairs and their
// host-mapped mirror.  The difference of the packed prefix at an item's two ends is exactly V_k + 2^32 F_k
// (V_k < 2^32), whatever the earlier items carried from the vertex half into the face half of the packed scan.
__global__ void mc_totals_kernel(int B, size_t nb, const unsigned long long* __restrict__ counts,
                                 const unsigned long long* __restrict__ offsets, long long* __restrict__ item_off,
                                 int32_t* __restrict__ totals, volatile int32_t* __restrict__ totals_host) {
  long long vo = 0, fo = 0;
  for (int k = 0; k < B; ++k) {
    const unsigned long long lo = offsets[k * nb];
    const unsigned long long hi = k + 1 < B ? offsets[(k + 1) * nb] : offsets[B * nb - 1] + counts[B * nb - 1];
    const unsigned long long d = hi - lo;
    const int32_t V = (int32_t)(d & 0xffffffffull), F = (int32_t)(d >> 32);
    item_off[k] = vo;
    item_off[B + 1 + k] = fo;
    vo += V;
    fo += F;
    totals[2 * k] = V;
    totals[2 * k + 1] = F;
    if (totals_host) {
      totals_host[2 * k] = V;
      totals_host[2 * k + 1] = F;
    }
  }
  item_off[B] = vo;
  item_off[2 * B + 1] = fo;
  if (totals_host) __threadfence_system();
}

// item k's vertices and faces follow those of items 0..k-1 (item_off); vid, vsrc and the face references are local
// to the item, so item k's slice is what the item alone gives
__global__ void __launch_bounds__(32 * MC_WARPS) mc_emit_kernel(
    McGeom g, int items, const float* __restrict__ phi, float iso, const unsigned long long* __restrict__ blk_counts,
    const unsigned long long* __restrict__ blk_offsets, const long long* __restrict__ item_off,
    uint32_t* __restrict__ vid, float* __restrict__ verts, int32_t* __restrict__ vsrc, long long V_cap,
    int32_t* __restrict__ faces, long long F_cap) {
  const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const size_t brick = (size_t)blockIdx.x * MC_WARPS + wid;
  if (brick >= (size_t)items * g.nbricks || blk_counts[brick] == 0) return;  // nothing owned here (most bricks)
  const size_t item = brick / g.nbricks, G3 = (size_t)g.G * g.G * g.G;
  McBrick B;
  mc_load_brick(g, brick - item * g.nbricks, lane, phi + item * G3, B);
  unsigned masks = 0, css[MC_BJ];  // 3 bits of mask per node, packed
  unsigned mine = 0;
#pragma unroll
  for (int r = 0; r < MC_BJ; ++r) {
    unsigned mask;
    mc_classify(g, B, r, iso, mask, css[r]);
    masks |= mask << (3 * r);
    mine += __popc(mask) | (mc_ntri(css[r]) << 16);
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
  long long f = item_off[items + 1 + item] + (long long)(base >> 32) + (excl >> 16);
  const int G = g.G;
  const float gm1 = (float)(G - 1);
#pragma unroll
  for (int r = 0; r < MC_BJ; ++r) {
    const unsigned mask = (masks >> (3 * r)) & 7u, cs = css[r];
    if (mask == 0 && cs == 0) continue;
    const int j = B.j0 + r;
    const size_t id = ((size_t)B.i * G + j) * G + B.k;
    if (mask) {
      vid[item * G3 + id] = (uint32_t)vl | (mask << 29);
      const float p0 = B.a[0][r];
      const float p1[3] = {B.a[1][r], B.a[0][r + 1], B.z[0][r]};
      const float basep[3] = {(float)B.i, (float)j, (float)B.k};
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        if (mask & (1u << a)) {
          const long long v = v0 + (long long)vl;
          if (v < V_cap) {
            const float t = (iso - p0) / (p1[a] - p0);
            float pos[3] = {basep[0], basep[1], basep[2]};
            pos[a] += t;
            verts[3 * v + 0] = pos[0] / gm1;  // IEEE division: identical to the numpy restatement
            verts[3 * v + 1] = pos[1] / gm1;
            verts[3 * v + 2] = pos[2] / gm1;
            vsrc[v] = (int32_t)(id * 3 + a);  // < 3 G^3 < 2^31 for G <= 800
          }
          ++vl;
        }
      }
    }
    const int nt = (int)mc_ntri(cs);
    for (int t = 0; t < nt; ++t, ++f) {
      if (f >= F_cap) break;
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const int e = __ldg(&g_tri[cs][3 * t + q]);
        const int c = mc_edge_lo(e), axis = e >> 2;
        const size_t owner = ((size_t)(B.i + (c & 1)) * G + (j + ((c >> 1) & 1))) * G + (B.k + (c >> 2));
        faces[3 * f + q] = (int32_t)(owner * 3 + axis);  // resolved by mc_resolve_kernel
      }
    }
  }
}

// foff = item_off + items + 1: the batch's first face of every item, and the total
__global__ void __launch_bounds__(256) mc_resolve_kernel(int items, size_t G3, const long long* __restrict__ foff,
                                                         long long F_cap, const uint32_t* __restrict__ vid,
                                                         int32_t* __restrict__ faces) {
  const long long n = 3 * min(foff[items], F_cap);
  const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= n) return;
  int lo = 0, hi = items - 1;  // the item of face x / 3: the last k with foff[k] <= x / 3
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (foff[mid] <= x / 3) lo = mid;
    else hi = mid - 1;
  }
  const uint32_t e = (uint32_t)faces[x];
  const uint32_t w = vid[(size_t)lo * G3 + e / 3];
  faces[x] = (int32_t)((w & 0x1fffffffu) + __popc((w >> 29) & ((1u << (e % 3)) - 1u)));
}

// dL/dphi += dL/dverts . d verts/d phi   (only the coordinate along the edge moves); one thread per vertex
// item k's vertices are [it.voff[k], it.voff[k + 1]) of the batch, its grids phi / dphi + k G^3
__global__ void __launch_bounds__(256) mc_backward_kernel(int G, McItems it, const float* __restrict__ phi, float iso,
                                                          const int32_t* __restrict__ vsrc,
                                                          const float* __restrict__ dverts,
                                                          float* __restrict__ dphi) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= it.voff[it.B]) return;
  int lo = 0, hi = it.B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (it.voff[mid] <= v) lo = mid;
    else hi = mid - 1;
  }
  const size_t G3 = (size_t)G * G * G;
  phi += lo * G3;
  dphi += lo * G3;
  const uint32_t e = (uint32_t)vsrc[v];
  const size_t id = e / 3;
  const int a = (int)(e % 3);
  const size_t nb = id + (a == 0 ? (size_t)G * G : (a == 1 ? (size_t)G : 1));
  const float p0 = phi[id], p1 = phi[nb];
  const float d = p1 - p0;
  // dt/dp0 = -(1 - t)/d, dt/dp1 = -t/d, with t = (iso - p0)/d the forward's t bit for bit and 1 - t taken from the
  // other end of the edge, (p1 - iso)/d: 1.f - t would lose the digits of 1 - t when t is near 1 (up to 1e-3
  // relative error measured on smooth fields).  The textbook (iso - p1)/d^2 form squares d, which is subnormal or
  // zero for |d| below ~1e-19 and infinite above ~1.8e19; this one is as scale-invariant as the forward.
  const float t = (iso - p0) / d, u = (p1 - iso) / d;
  const float gr = dverts[3 * (size_t)v + a] / (float)(G - 1);
  atomicAdd(&dphi[id], -gr * u / d);
  atomicAdd(&dphi[nb], -gr * t / d);
}

static unsigned long long g_tables_uploaded = 0;  // per device
static cudaError_t upload_tables() {
  if (!once_per_device(g_tables_uploaded)) return cudaSuccess;
  cudaError_t e = cudaMemcpyToSymbol(g_ntri, MC_NTRI, sizeof(MC_NTRI));
  if (e == cudaSuccess) e = cudaMemcpyToSymbol(g_tri, MC_TRI, sizeof(MC_TRI));
  for (int i = 0; i < 12 && e == cudaSuccess; ++i) {  // the closed form must be the generated table
    const int axis = i >> 2, k = i & 3;
    const int lo = axis == 0 ? (k << 1) : (axis == 1 ? ((k & 1) | ((k & 2) << 1)) : k);
    if (lo != MC_EDGE_LO[i]) e = cudaErrorInvalidValue;
  }
  if (e != cudaSuccess) g_tables_uploaded = 0;  // retry on the next call
  return e;
}

size_t mc_cub_bytes(size_t n) {
  size_t bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                (int)n);
  return bytes;
}

McWS McWS::from(char* base, int G, int B, size_t* bytes) {
  char* p = base;
  McWS w;
  const size_t n = (size_t)G * G * G, nb = (size_t)B * mc_num_blocks(G);
  w.blk_counts = carve<unsigned long long>(p, nb);
  w.blk_offsets = carve<unsigned long long>(p, nb);
  w.item_off = carve<long long>(p, 2 * (size_t)B + 2);
  w.cub_bytes = mc_cub_bytes(nb);
  w.cub_temp = carve<char>(p, w.cub_bytes);
  w.vid = carve<uint32_t>(p, (size_t)B * n);    // sparse: only entries of vertex-owning nodes are ever written or read
  if (bytes) *bytes = size_t(p - base) + 128;
  return w;
}

cudaError_t launch_mc_scan_totals(int B, size_t nb, unsigned long long* blk_counts,
                                  unsigned long long* blk_offsets, long long* item_off, void* cub_temp,
                                  size_t cub_bytes, int32_t* totals, int32_t* totals_host, cudaEvent_t ev,
                                  cudaStream_t s) {
  size_t tb = cub_bytes;
  cub::DeviceScan::ExclusiveSum(cub_temp, tb, blk_counts, blk_offsets, (int)(B * nb), s);
  mc_totals_kernel<<<1, 1, 0, s>>>(B, nb, blk_counts, blk_offsets, item_off, totals, (volatile int32_t*)totals_host);
  if (ev) cudaEventRecord(ev, s);
  return cudaGetLastError();
}

cudaError_t launch_mc_count(int B, int G, const float* phi, float iso, void* ws, int32_t* totals,
                            int32_t* totals_host, cudaEvent_t ev, cudaStream_t s) {
  cudaError_t e = upload_tables();
  if (e != cudaSuccess) return e;
  McWS w = McWS::from((char*)ws, G, B);
  const McGeom g = mc_geom(G);
  const size_t nb = mc_num_blocks(G), nall = (size_t)B * nb;
  mc_count_kernel<<<(unsigned)((nall + MC_WARPS - 1) / MC_WARPS), 32 * MC_WARPS, 0, s>>>(g, nall, phi, iso,
                                                                                          w.blk_counts);
  return launch_mc_scan_totals(B, nb, w.blk_counts, w.blk_offsets, w.item_off, w.cub_temp, w.cub_bytes, totals,
                               totals_host, ev, s);
}

cudaError_t launch_mc_emit(int B, int G, const float* phi, float iso, void* ws, float* verts, int32_t* vsrc,
                           long long V_cap, int32_t* faces, long long F_cap, cudaStream_t s) {
  McWS w = McWS::from((char*)ws, G, B);
  const McGeom g = mc_geom(G);
  const size_t nall = (size_t)B * mc_num_blocks(G);
  mc_emit_kernel<<<(unsigned)((nall + MC_WARPS - 1) / MC_WARPS), 32 * MC_WARPS, 0, s>>>(
      g, B, phi, iso, w.blk_counts, w.blk_offsets, w.item_off, w.vid, verts, vsrc, V_cap, faces, F_cap);
  if (F_cap > 0)
    mc_resolve_kernel<<<(unsigned)((3 * F_cap + 255) / 256), 256, 0, s>>>(B, (size_t)G * G * G, w.item_off + B + 1,
                                                                          F_cap, w.vid, faces);
  return cudaGetLastError();
}

cudaError_t launch_mc_backward(int G, const McItems& it, const float* phi, float iso, const int32_t* vsrc,
                               const float* dverts, float* dphi, cudaStream_t s) {
  const size_t n = (size_t)it.B * G * G * G;
  const int V = it.voff[it.B];
  cudaMemsetAsync(dphi, 0, sizeof(float) * n, s);
  if (V > 0) mc_backward_kernel<<<(V + 255) / 256, 256, 0, s>>>(G, it, phi, iso, vsrc, dverts, dphi);
  return cudaGetLastError();
}

}  // namespace dgm
