// mesh_distance.cu -- the closest point of a triangle mesh to each of Q query points, and the gradient of the squared
// distance in the points and the vertices (include/dgmesh_b200.h "dgpm_").
//
//   * BVH, rebuilt on the device on every call: a linear BVH (Karras 2012, "Maximizing parallelism in the
//     construction of BVHs, octrees and k-d trees").  knn.cu's bounds and Morton kernels give each triangle
//     centroid a 30-bit code; a stable CUB radix sort orders (code, face) pairs; runs of PM_LEAF = 4 consecutive
//     triangles form the leaves, whose key is (code of the first triangle << 32 | leaf index), so equal codes are
//     split by index and every key is distinct.  One thread per internal node finds its range and split from the
//     keys alone; the boxes are refitted bottom-up with one arrival counter per internal node (the second arrival
//     merges).  Min and max do not depend on the arrival order, so the tree is the same bits from run to run.
//     Four triangles per leaf: a leaf visit costs four closest-point tests against one box pair per internal node,
//     and the tree has a quarter of the nodes of one triangle per leaf.
//   * Query: the queries are put in Morton order the same way (in their own box) and one thread per query walks
//     the tree with a stack, nearer child first; the order only groups similar walks into a warp (2x faster for
//     10^6 queries on 5.2 M faces, tools/mesh_distance_bench.py) and every query's result is computed alone.  A child is skipped only when its
//     box is strictly farther than the best squared distance so far, and a triangle is taken when (d, face) is
//     lexicographically smaller than the best, so the result is the minimum of (d, face) over all triangles: exact
//     ties go to the lowest face index whatever the visiting order.
//   * Stack bound: the keys are distinct 64-bit integers whose two top bits are 0 (codes < 2^30), and the tree is
//     their binary radix tree, so the common-prefix length strictly grows from an internal node to an internal
//     child and lies in [2, 63]: at most 62 internal nodes on any root-to-leaf path.  Every stack entry is the far
//     child of a distinct ancestor of the node being visited, so the stack never holds more than 61 entries;
//     PM_STACK = 64.
//   * Closest point: Ericson's region method ("Real-Time Collision Detection", 5.1.5), every region's offset taken
//     from a vertex of that region, so a query equal to a vertex has a zero offset.  A triangle that is degenerate
//     in fp32 (|ab x ac|^2 <= 1e-10 |ab|^2 |ac|^2: collinear or coincident vertices) is the union of its three edges,
//     i.e. its longest edge or its single point, and its weights are put on the longest edge; the union of the
//     edges also covers a face region whose fp32 weights come out outside the triangle.
//   * Backward, for dist2 only: grad_points[q] = 2 g[q] (p_q - c_q), and grad_verts[v] = -sum over the entries
//     (q, k) with faces[face[q]][k] = v of bary[q][k] grad_points[q], gathered through csr_inverse.cuh (no float
//     atomics; segments summed in increasing entry 3 q + k).
#include <cfloat>
#include <climits>
#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"
#include "csr_inverse.cuh"
#include "knn_kernels.h"
#include "mesh_distance_kernels.h"

namespace dgm {

#define PM_DEGENERATE 1e-10f  // sin^2 of the triangle's angle at a below which it is a set of segments

__device__ __forceinline__ float3 pm_sub(float3 a, float3 b) { return make_float3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ float pm_dot(float3 a, float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
// a - t b
__device__ __forceinline__ float3 pm_axpy(float3 a, float t, float3 b) {
  return make_float3(a.x - t * b.x, a.y - t * b.y, a.z - t * b.z);
}

size_t pm_fwd_cub_bytes(int F, int Q) {
  size_t a = 0, b = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, a, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                  (const uint32_t*)nullptr, (uint32_t*)nullptr, F, 0, 30);
  cub::DeviceRadixSort::SortPairs(nullptr, b, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                  (const uint32_t*)nullptr, (uint32_t*)nullptr, Q, 0, 30);
  return a > b ? a : b;
}

PmFwdWS PmFwdWS::from(char* base, size_t F, size_t Q, size_t cub_bytes, size_t* bytes) {
  char* p = base;
  const size_t L = (F + PM_LEAF - 1) / PM_LEAF;
  PmFwdWS w;
  w.cent = carve<float>(p, 3 * F);
  w.bounds = carve<uint32_t>(p, 8);
  w.codes = carve<uint32_t>(p, F);
  w.codes_sorted = carve<uint32_t>(p, F);
  w.idx = carve<uint32_t>(p, F);
  w.order = carve<uint32_t>(p, F);
  w.tri = carve<float>(p, 12 * F);
  w.nodes = carve<PmNode>(p, L > 1 ? L - 1 : 1);
  w.leaf_parent = carve<int>(p, L);
  w.counter = carve<int>(p, L > 1 ? L - 1 : 1);
  w.qbounds = carve<uint32_t>(p, 8);
  w.qcodes = carve<uint32_t>(p, Q);
  w.qcodes_sorted = carve<uint32_t>(p, Q);
  w.qidx = carve<uint32_t>(p, Q);
  w.qorder = carve<uint32_t>(p, Q);
  w.cub_temp = carve<char>(p, cub_bytes);
  w.cub_bytes = cub_bytes;
  if (bytes) *bytes = size_t(p - base) + 128;
  return w;
}

size_t pm_bwd_cub_bytes(int V, int Q) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                  (const uint32_t*)nullptr, (uint32_t*)nullptr, 3 * Q, 0, key_bits((size_t)V));
  return bytes;
}

PmBwdWS PmBwdWS::from(char* base, size_t Q, size_t cub_bytes, size_t* bytes) {
  char* p = base;
  PmBwdWS w;
  w.keys_in = carve<uint32_t>(p, 3 * Q);
  w.keys_out = carve<uint32_t>(p, 3 * Q);
  w.vals_in = carve<uint32_t>(p, 3 * Q);
  w.vals_out = carve<uint32_t>(p, 3 * Q);
  w.cub_temp = carve<char>(p, cub_bytes);
  w.cub_bytes = cub_bytes;
  if (bytes) *bytes = size_t(p - base) + 128;
  return w;
}

__device__ __forceinline__ float3 pm_vert(const float* __restrict__ verts, int i) {
  return make_float3(verts[3 * (size_t)i], verts[3 * (size_t)i + 1], verts[3 * (size_t)i + 2]);
}

__global__ void __launch_bounds__(256) pm_centroid_kernel(int F, const float* __restrict__ verts,
                                                          const int32_t* __restrict__ faces,
                                                          float* __restrict__ cent) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const float3 a = pm_vert(verts, faces[3 * (size_t)f]), b = pm_vert(verts, faces[3 * (size_t)f + 1]),
               c = pm_vert(verts, faces[3 * (size_t)f + 2]);
  cent[3 * (size_t)f] = (a.x + b.x + c.x) * (1.f / 3.f);
  cent[3 * (size_t)f + 1] = (a.y + b.y + c.y) * (1.f / 3.f);
  cent[3 * (size_t)f + 2] = (a.z + b.z + c.z) * (1.f / 3.f);
}

// key of leaf l: (Morton code of its first triangle, l)
__device__ __forceinline__ unsigned long long pm_key(const uint32_t* __restrict__ codes, int l) {
  return ((unsigned long long)codes[(size_t)l * PM_LEAF] << 32) | (unsigned)l;
}

// Karras 2012, algorithm 2: internal node i of L leaves; children >= 0 are internal nodes, ~l is leaf l
__global__ void __launch_bounds__(256) pm_build_kernel(int L, const uint32_t* __restrict__ codes,
                                                       PmNode* __restrict__ nodes, int* __restrict__ leaf_parent) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L - 1) return;
  const unsigned long long ki = pm_key(codes, i);
  auto delta = [&](int j) -> int { return (j < 0 || j >= L) ? -1 : __clzll(ki ^ pm_key(codes, j)); };
  const int d = delta(i + 1) > delta(i - 1) ? 1 : -1;
  const int dmin = delta(i - d);
  int lmax = 2;
  while (delta(i + lmax * d) > dmin) lmax <<= 1;
  int l = 0;
  for (int t = lmax >> 1; t >= 1; t >>= 1)
    if (delta(i + (l + t) * d) > dmin) l += t;
  const int j = i + l * d;
  const int dnode = delta(j);
  int s = 0;
  for (int div = 2, t = l;; div <<= 1) {
    t = (l + div - 1) / div;
    if (delta(i + (s + t) * d) > dnode) s += t;
    if (t <= 1) break;
  }
  const int gamma = i + s * d + min(d, 0);
  const bool left_leaf = min(i, j) == gamma, right_leaf = max(i, j) == gamma + 1;
  nodes[i].child[0] = left_leaf ? ~gamma : gamma;
  nodes[i].child[1] = right_leaf ? ~(gamma + 1) : gamma + 1;
  if (left_leaf) leaf_parent[gamma] = i << 1;
  else nodes[gamma].parent = i << 1;
  if (right_leaf) leaf_parent[gamma + 1] = (i << 1) | 1;
  else nodes[gamma + 1].parent = (i << 1) | 1;
  if (i == 0) nodes[0].parent = -1;
}

// One thread per leaf: copy its triangles in Morton order into tri (three float4: a, b, c, face index), take their
// box, and climb while this thread is the second arrival at the parent.
__global__ void __launch_bounds__(256) pm_refit_kernel(int F, int L, const float* __restrict__ verts,
                                                       const int32_t* __restrict__ faces,
                                                       const uint32_t* __restrict__ order, float4* __restrict__ tri,
                                                       PmNode* nodes, const int* __restrict__ leaf_parent,
                                                       int* __restrict__ counter) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= L) return;
  float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  for (int t = l * PM_LEAF; t < min(F, (l + 1) * PM_LEAF); ++t) {
    const int f = (int)order[t];
    float x[9];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float3 v = pm_vert(verts, faces[3 * (size_t)f + k]);
      x[3 * k] = v.x;
      x[3 * k + 1] = v.y;
      x[3 * k + 2] = v.z;
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      mn[k % 3] = fminf(mn[k % 3], x[k]);
      mx[k % 3] = fmaxf(mx[k % 3], x[k]);
    }
    tri[3 * (size_t)t] = make_float4(x[0], x[1], x[2], x[3]);
    tri[3 * (size_t)t + 1] = make_float4(x[4], x[5], x[6], x[7]);
    tri[3 * (size_t)t + 2] = make_float4(x[8], __int_as_float(f), 0.f, 0.f);
  }
  int p = L > 1 ? leaf_parent[l] : -1;
  while (p >= 0) {
    const int node = p >> 1, side = p & 1;
    float* b = nodes[node].box[side];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      b[c] = mn[c];
      b[3 + c] = mx[c];
    }
    __threadfence();
    if (atomicAdd(&counter[node], 1) == 0) return;  // the sibling's thread arrives second and merges
    const float* o = nodes[node].box[side ^ 1];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      mn[c] = fminf(mn[c], __ldcg(o + c));
      mx[c] = fmaxf(mx[c], __ldcg(o + 3 + c));
    }
    p = __ldcg(&nodes[node].parent);
  }
}

// squared distance of ap - t ab, t = clamp(ap . ab / |ab|^2, 0, 1) (0 for a zero-length segment)
__device__ __forceinline__ float pm_segment(float3 ap, float3 ab, float& t) {
  const float den = pm_dot(ab, ab);
  t = den > 0.f ? fminf(fmaxf(pm_dot(ap, ab) / den, 0.f), 1.f) : 0.f;
  const float3 e = pm_axpy(ap, t, ab);
  return pm_dot(e, e);
}

// the triangle as the union of its edges ab (from a), bc (from b) and ca (from c); the first of equal distances
__device__ __forceinline__ float pm_edges(float3 p, float3 a, float3 b, float3 c, float& u, float& v, float& w) {
  float t;
  float best = pm_segment(pm_sub(p, a), pm_sub(b, a), t);
  u = 1.f - t, v = t, w = 0.f;
  float d = pm_segment(pm_sub(p, b), pm_sub(c, b), t);
  if (d < best) best = d, u = 0.f, v = 1.f - t, w = t;
  d = pm_segment(pm_sub(p, c), pm_sub(a, c), t);
  if (d < best) best = d, u = t, v = 0.f, w = 1.f - t;
  return best;
}

// The weights of a point u a + v b + w c of a degenerate triangle are not unique; re-express it on the longest edge
// (the first of equal lengths in the order ab, bc, ca), so that the gradient goes to that edge's endpoints
// whichever edge was nearest.  A triangle of three equal vertices keeps the weights (1, 0, 0).
__device__ __forceinline__ void pm_on_longest_edge(float3 a, float3 b, float3 c, float& u, float& v, float& w) {
  const float3 ab = pm_sub(b, a), bc = pm_sub(c, b), ca = pm_sub(a, c);
  const float lab = pm_dot(ab, ab), lbc = pm_dot(bc, bc), lca = pm_dot(ca, ca);
  const float3 q = make_float3(u * a.x + v * b.x + w * c.x, u * a.y + v * b.y + w * c.y, u * a.z + v * b.z + w * c.z);
  float t;
  if (lab >= lbc && lab >= lca) {
    t = lab > 0.f ? fminf(fmaxf(pm_dot(pm_sub(q, a), ab) / lab, 0.f), 1.f) : 0.f;
    u = 1.f - t, v = t, w = 0.f;
  } else if (lbc >= lca) {
    t = fminf(fmaxf(pm_dot(pm_sub(q, b), bc) / lbc, 0.f), 1.f);
    u = 0.f, v = 1.f - t, w = t;
  } else {
    t = fminf(fmaxf(pm_dot(pm_sub(q, c), ca) / lca, 0.f), 1.f);
    u = t, v = 0.f, w = 1.f - t;
  }
}

// Squared distance from p to triangle (a, b, c) and the weights of its closest point u a + v b + w c.  The region
// tests are Ericson's; the edge parameters divide by the edge's own squared length, and the face weights are those
// of p's projection onto the plane, measured from a: both stay accurate when p is far from a small triangle, where
// Ericson's vb / (va + vb + vc) loses the digits that cancel in va, vb and vc.
__device__ __forceinline__ float pm_closest(float3 p, float3 a, float3 b, float3 c, float& u, float& v, float& w) {
  const float3 ab = pm_sub(b, a), ac = pm_sub(c, a);
  const float3 n = make_float3(ab.y * ac.z - ab.z * ac.y, ab.z * ac.x - ab.x * ac.z, ab.x * ac.y - ab.y * ac.x);
  const float lab = pm_dot(ab, ab), lac = pm_dot(ac, ac), nn = pm_dot(n, n);
  if (!(nn > PM_DEGENERATE * lab * lac)) {
    const float d = pm_edges(p, a, b, c, u, v, w);
    pm_on_longest_edge(a, b, c, u, v, w);
    return d;
  }
  const float3 ap = pm_sub(p, a);
  const float d1 = pm_dot(ab, ap), d2 = pm_dot(ac, ap);
  if (d1 <= 0.f && d2 <= 0.f) {  // vertex a
    u = 1.f, v = 0.f, w = 0.f;
    return pm_dot(ap, ap);
  }
  const float3 bp = pm_sub(p, b);
  const float d3 = pm_dot(ab, bp), d4 = pm_dot(ac, bp);
  if (d3 >= 0.f && d4 <= d3) {  // vertex b
    u = 0.f, v = 1.f, w = 0.f;
    return pm_dot(bp, bp);
  }
  const float vc = d1 * d4 - d3 * d2;
  if (vc <= 0.f && d1 >= 0.f && d3 <= 0.f) {  // edge ab
    const float t = fminf(d1 / lab, 1.f);
    u = 1.f - t, v = t, w = 0.f;
    const float3 e = pm_axpy(ap, t, ab);
    return pm_dot(e, e);
  }
  const float3 cp = pm_sub(p, c);
  const float d5 = pm_dot(ab, cp), d6 = pm_dot(ac, cp);
  if (d6 >= 0.f && d5 <= d6) {  // vertex c
    u = 0.f, v = 0.f, w = 1.f;
    return pm_dot(cp, cp);
  }
  const float vb = d5 * d2 - d1 * d6;
  if (vb <= 0.f && d2 >= 0.f && d6 <= 0.f) {  // edge ac
    const float t = fminf(d2 / lac, 1.f);
    u = 1.f - t, v = 0.f, w = t;
    const float3 e = pm_axpy(ap, t, ac);
    return pm_dot(e, e);
  }
  const float va = d3 * d6 - d5 * d4;
  if (va <= 0.f && d4 - d3 >= 0.f && d5 - d6 >= 0.f) {  // edge bc
    const float3 bc = pm_sub(c, b);
    const float lbc = pm_dot(bc, bc), t = lbc > 0.f ? fminf(fmaxf(pm_dot(bp, bc) / lbc, 0.f), 1.f) : 0.f;
    u = 0.f, v = 1.f - t, w = t;
    const float3 e = pm_axpy(bp, t, bc);
    return pm_dot(e, e);
  }
  // face: the projection q of p, a + v ab + w ac with v = ((aq x ac) . n) / |n|^2, w = ((ab x aq) . n) / |n|^2
  const float inv = 1.f / nn;
  const float3 aq = pm_axpy(ap, pm_dot(ap, n) * inv, n);
  const float3 x = make_float3(aq.y * ac.z - aq.z * ac.y, aq.z * ac.x - aq.x * ac.z, aq.x * ac.y - aq.y * ac.x);
  const float3 y = make_float3(ab.y * aq.z - ab.z * aq.y, ab.z * aq.x - ab.x * aq.z, ab.x * aq.y - ab.y * aq.x);
  v = pm_dot(x, n) * inv, w = pm_dot(y, n) * inv;
  if (!(v >= 0.f && w >= 0.f && v + w <= 1.f)) return pm_edges(p, a, b, c, u, v, w);
  u = 1.f - v - w;
  const float3 e = pm_axpy(pm_axpy(ap, v, ab), w, ac);
  return pm_dot(e, e);
}

struct PmBest {
  float d, u, v, w;
  int f;
};

__device__ __forceinline__ void pm_leaf(int l, int F, const float4* __restrict__ tri, float3 p, PmBest& best) {
  for (int t = l * PM_LEAF; t < min(F, (l + 1) * PM_LEAF); ++t) {
    const float4 r0 = __ldg(tri + 3 * (size_t)t), r1 = __ldg(tri + 3 * (size_t)t + 1),
                 r2 = __ldg(tri + 3 * (size_t)t + 2);
    float u, v, w;
    const float d = pm_closest(p, make_float3(r0.x, r0.y, r0.z), make_float3(r0.w, r1.x, r1.y),
                               make_float3(r1.z, r1.w, r2.x), u, v, w);
    const int f = __float_as_int(r2.y);
    if (d < best.d || (d == best.d && f < best.f)) best = {d, u, v, w, f};
  }
}

__device__ __forceinline__ float pm_box_d2(float x0, float y0, float z0, float x1, float y1, float z1, float3 p) {
  const float dx = fmaxf(fmaxf(x0 - p.x, p.x - x1), 0.f), dy = fmaxf(fmaxf(y0 - p.y, p.y - y1), 0.f),
              dz = fmaxf(fmaxf(z0 - p.z, p.z - z1), 0.f);
  return dx * dx + dy * dy + dz * dz;
}

// thread t takes query qorder[t], so a warp's queries are Morton neighbours and walk much the same part of the tree
__global__ void __launch_bounds__(128) pm_query_kernel(int Q, int F, int L, const float* __restrict__ points,
                                                       const uint32_t* __restrict__ qorder,
                                                       const float4* __restrict__ tri,
                                                       const PmNode* __restrict__ nodes, float* __restrict__ dist2,
                                                       long long* __restrict__ face, float* __restrict__ bary) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= Q) return;
  const int q = (int)qorder[t];
  const float3 p = make_float3(points[3 * (size_t)q], points[3 * (size_t)q + 1], points[3 * (size_t)q + 2]);
  PmBest best = {__int_as_float(0x7f800000), 0.f, 0.f, 0.f, INT_MAX};
  if (L == 1) {
    pm_leaf(0, F, tri, p, best);
  } else {
    int stack_node[PM_STACK];
    float stack_d[PM_STACK];
    int sp = 0, node = 0;
    while (true) {
      const float4* r = reinterpret_cast<const float4*>(nodes + node);
      const float4 q0 = __ldg(r), q1 = __ldg(r + 1), q2 = __ldg(r + 2), q3 = __ldg(r + 3);
      int cl = __float_as_int(q3.x), cr = __float_as_int(q3.y);
      float dl = pm_box_d2(q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, p), dr = pm_box_d2(q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, p);
      if (dr < dl) {  // nearer child first; the left one on a tie
        const int ci = cl;
        cl = cr, cr = ci;
        const float di = dl;
        dl = dr, dr = di;
      }
      bool go_l = !(dl > best.d), go_r = !(dr > best.d);
      if (go_l && cl < 0) {
        pm_leaf(~cl, F, tri, p, best);
        go_l = false;
        go_r = !(dr > best.d);
      }
      if (go_r && cr < 0) {
        pm_leaf(~cr, F, tri, p, best);
        go_r = false;
      }
      if (go_l) {
        if (go_r) {
          stack_node[sp] = cr;
          stack_d[sp++] = dr;
        }
        node = cl;
        continue;
      }
      if (go_r) {
        node = cr;
        continue;
      }
      while (sp > 0 && stack_d[sp - 1] > best.d) --sp;
      if (sp == 0) break;
      node = stack_node[--sp];
    }
  }
  dist2[q] = best.d;
  face[q] = best.f;
  bary[3 * (size_t)q] = best.u;
  bary[3 * (size_t)q + 1] = best.v;
  bary[3 * (size_t)q + 2] = best.w;
}

void pm_build(int F, int Q, const float* verts, const int32_t* faces, const float* points, const PmFwdWS& w,
              cudaStream_t s) {
  const int L = (F + PM_LEAF - 1) / PM_LEAF;
  cudaMemsetAsync(w.bounds, 0, 8 * sizeof(uint32_t), s);
  cudaMemsetAsync(w.qbounds, 0, 8 * sizeof(uint32_t), s);
  if (L > 1) cudaMemsetAsync(w.counter, 0, (L - 1) * sizeof(int), s);
  pm_centroid_kernel<<<(F + 255) / 256, 256, 0, s>>>(F, verts, faces, w.cent);
  knn_bounds_kernel<<<min(592, (F + 255) / 256), 256, 0, s>>>(F, w.cent, w.bounds);
  knn_morton_kernel<<<(F + 255) / 256, 256, 0, s>>>(F, w.cent, w.bounds, w.codes, w.idx);
  size_t tb = w.cub_bytes;
  cub::DeviceRadixSort::SortPairs(w.cub_temp, tb, w.codes, w.codes_sorted, w.idx, w.order, F, 0, 30, s);
  if (L > 1) pm_build_kernel<<<(L - 1 + 255) / 256, 256, 0, s>>>(L, w.codes_sorted, w.nodes, w.leaf_parent);
  pm_refit_kernel<<<(L + 255) / 256, 256, 0, s>>>(F, L, verts, faces, w.order, (float4*)w.tri, w.nodes,
                                                  w.leaf_parent, w.counter);
  knn_bounds_kernel<<<min(592, (Q + 255) / 256), 256, 0, s>>>(Q, points, w.qbounds);
  knn_morton_kernel<<<(Q + 255) / 256, 256, 0, s>>>(Q, points, w.qbounds, w.qcodes, w.qidx);
  tb = w.cub_bytes;
  cub::DeviceRadixSort::SortPairs(w.cub_temp, tb, w.qcodes, w.qcodes_sorted, w.qidx, w.qorder, Q, 0, 30, s);
}

void pm_query(int F, int Q, const float* points, const PmFwdWS& w, float* dist2, long long* face, float* bary,
              cudaStream_t s) {
  const int L = (F + PM_LEAF - 1) / PM_LEAF;
  pm_query_kernel<<<(Q + 127) / 128, 128, 0, s>>>(Q, F, L, points, w.qorder, (const float4*)w.tri, w.nodes, dist2,
                                                  face, bary);
}

cudaError_t launch_point_mesh_distance(int F, int Q, const float* verts, const int32_t* faces, const float* points,
                                       float* dist2, long long* face, float* bary, void* ws, cudaStream_t s) {
  if (Q == 0) return cudaSuccess;
  const PmFwdWS w = PmFwdWS::from((char*)ws, F, Q, pm_fwd_cub_bytes(F, Q));
  pm_build(F, Q, verts, faces, points, w, s);
  pm_query(F, Q, points, w, dist2, face, bary, s);
  return cudaGetLastError();
}

// grad_points[q] = 2 g[q] (p - c), p - c = (p - a) - v (b - a) - w (c - a); and the (vertex, entry 3 q + k) pairs
__global__ void __launch_bounds__(256) pm_grad_points_kernel(int Q, const float* __restrict__ verts,
                                                             const int32_t* __restrict__ faces,
                                                             const float* __restrict__ points,
                                                             const long long* __restrict__ face,
                                                             const float* __restrict__ bary,
                                                             const float* __restrict__ g,
                                                             float* __restrict__ grad_points,
                                                             uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= Q) return;
  const size_t f = (size_t)face[q];
  const int i0 = faces[3 * f], i1 = faces[3 * f + 1], i2 = faces[3 * f + 2];
  const float3 a = pm_vert(verts, i0), p = pm_vert(points, q);
  const float3 e = pm_axpy(pm_axpy(pm_sub(p, a), bary[3 * (size_t)q + 1], pm_sub(pm_vert(verts, i1), a)),
                           bary[3 * (size_t)q + 2], pm_sub(pm_vert(verts, i2), a));
  const float s = 2.f * g[q];
  grad_points[3 * (size_t)q] = s * e.x;
  grad_points[3 * (size_t)q + 1] = s * e.y;
  grad_points[3 * (size_t)q + 2] = s * e.z;
  keys[3 * (size_t)q] = (uint32_t)i0;
  keys[3 * (size_t)q + 1] = (uint32_t)i1;
  keys[3 * (size_t)q + 2] = (uint32_t)i2;
#pragma unroll
  for (int k = 0; k < 3; ++k) vals[3 * (size_t)q + k] = (uint32_t)(3 * q + k);
}

// grad_verts[v] = -sum over v's segment of the sorted pairs, in increasing entry e = 3 q + k, of bary[e] grad_points[q]
__global__ void __launch_bounds__(256) pm_grad_verts_kernel(int V, int n, const uint32_t* __restrict__ keys,
                                                            const uint32_t* __restrict__ vals,
                                                            const float* __restrict__ bary,
                                                            const float* __restrict__ grad_points,
                                                            float* __restrict__ grad_verts) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int lo = lower_bound_u32(keys, n, (uint32_t)v), hi = lower_bound_u32(keys, n, (uint32_t)v + 1u);
  float gx = 0.f, gy = 0.f, gz = 0.f;
  for (int j = lo; j < hi; ++j) {
    const uint32_t e = vals[j];
    const size_t q = e / 3;
    const float w = bary[e];
    gx -= w * grad_points[3 * q];
    gy -= w * grad_points[3 * q + 1];
    gz -= w * grad_points[3 * q + 2];
  }
  grad_verts[3 * (size_t)v] = gx;
  grad_verts[3 * (size_t)v + 1] = gy;
  grad_verts[3 * (size_t)v + 2] = gz;
}

cudaError_t launch_point_mesh_distance_bwd(int V, int Q, const float* verts, const int32_t* faces,
                                           const float* points, const long long* face, const float* bary,
                                           const float* grad_dist2, float* grad_points, float* grad_verts, void* ws,
                                           cudaStream_t s) {
  if (Q == 0) return cudaSuccess;
  PmBwdWS w = PmBwdWS::from((char*)ws, Q, pm_bwd_cub_bytes(V, Q));
  pm_grad_points_kernel<<<(Q + 255) / 256, 256, 0, s>>>(Q, verts, faces, points, face, bary, grad_dist2,
                                                        grad_points, w.keys_in, w.vals_in);
  size_t tb = w.cub_bytes;
  cub::DeviceRadixSort::SortPairs(w.cub_temp, tb, w.keys_in, w.keys_out, w.vals_in, w.vals_out, 3 * Q, 0,
                                  key_bits((size_t)V), s);
  pm_grad_verts_kernel<<<(V + 255) / 256, 256, 0, s>>>(V, 3 * Q, w.keys_out, w.vals_out, bary, grad_points,
                                                       grad_verts);
  return cudaGetLastError();
}

}  // namespace dgm
