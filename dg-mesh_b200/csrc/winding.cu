// winding.cu -- the generalized winding number of a triangle mesh at Q query points (Jacobson et al. 2013), evaluated
// on mesh_distance.cu's BVH with Barill et al. 2018's order-1 far-field expansion (include/dgmesh_b200.h
// "dgpm_winding").
//
//   * Build: pm_build, exactly as dgpm_forward (the same kernels, launches and workspace prefix), so the optional
//     closest points of dgpm_winding are dgpm_forward's bit for bit.
//   * Expansions (wn_refit_kernel): for each child cluster of every internal node, with t over its triangles,
//     a_t n_t = 1/2 (b - a) x (c - a), A = sum |a_t n_t| and x_t the triangle's centroid:
//       p~ = sum |a_t n_t| x_t / A (the child's box centre when A = 0),  N = sum a_t n_t,
//       M = sum (x_t - p~) (a_t n_t)^T,  r >= max over the cluster's vertices of |v - p~|.
//     A leaf takes its triangles directly and r = max |v - p~|; a merge takes the two stored child records,
//     p~ = (A0 p~0 + A1 p~1) / A, M = M0 + (p~0 - p~) N0^T + M1 + (p~1 - p~) N1^T and the child bound
//     r = max(|p~0 - p~| + r0, |p~1 - p~| + r1).  Sums run in float64 from the stored fp32 records and are rounded
//     to fp32 (r upward).  Bottom-up with one arrival counter per internal node, as pm_refit_kernel: the second
//     arrival merges child 0 then child 1 from memory, so the records are the same bits whichever thread merges.
//   * Query (wn_query_kernel): one thread per query in the forward's Morton order, the same 64-entry stack as
//     pm_query_kernel (each entry is child 1 of a distinct ancestor, so the bound stated in mesh_distance.cu holds).
//     At a node, child 0 is handled before child 1: a child with |q - p~| > beta r adds its far-field term
//       (u . N + (tr M - 3 u^T M u) / d) / d^2,  d = |p~ - q|, u = (p~ - q) / d
//     (the solid angle of the order-1 Taylor expansion of the dipole kernel (x - q) / |x - q|^3 about p~); a leaf
//     child adds its triangles' exact solid angles 2 atan2(det[a b c], |a||b||c| + (a.b)|c| + (b.c)|a| + (c.a)|b|),
//     a, b, c the vertices minus q, and 0 where det is exactly 0 (a query on a face, edge or vertex, and
//     coincident or collinear vertices); an internal child is descended into (child 1 waits on the stack when both
//     are).  The terms are fp32 and are added to one float64 sum per thread in that fixed order, so w depends only
//     on the tree and the query: bit-identical from run to run and whatever the other queries of the call.
//     beta = +inf never takes the far field (r = 0 gives inf * 0 = NaN, which compares false as well): the exact
//     sum over all faces.
//   * w = sum / (4 pi), stored as fp32.
#include <cfloat>
#include <cmath>

#include "common.cuh"
#include "mesh_distance_kernels.h"

namespace dgm {

WnWS WnWS::from(char* base, size_t F, size_t Q, size_t cub_bytes, size_t* bytes) {
  WnWS w;
  w.pm = PmFwdWS::from(base, F, Q, cub_bytes);
  char* p = w.pm.cub_temp + cub_bytes;
  const size_t L = (F + PM_LEAF - 1) / PM_LEAF;
  w.nodes = carve<WnNode>(p, L > 1 ? L - 1 : 1);
  w.counter = carve<int>(p, L > 1 ? L - 1 : 1);
  if (bytes) *bytes = size_t(p - base) + 128;
  return w;
}

// a child's record, written to or read from slot k of a WnNode
struct WnExp {
  float p[3], r, n[3], a, m[9];
};

__device__ __forceinline__ void wn_store(WnNode* nd, int k, const WnExp& e) {
  nd->pr[k] = make_float4(e.p[0], e.p[1], e.p[2], e.r);
  nd->na[k] = make_float4(e.n[0], e.n[1], e.n[2], e.a);
#pragma unroll
  for (int i = 0; i < 9; ++i) nd->m[k][i] = e.m[i];
}

__device__ __forceinline__ WnExp wn_load(const WnNode* nd, int k) {
  WnExp e;
  const float4 pr = __ldcg(&nd->pr[k]), na = __ldcg(&nd->na[k]);
  e.p[0] = pr.x, e.p[1] = pr.y, e.p[2] = pr.z, e.r = pr.w;
  e.n[0] = na.x, e.n[1] = na.y, e.n[2] = na.z, e.a = na.w;
#pragma unroll
  for (int i = 0; i < 9; ++i) e.m[i] = __ldcg(&nd->m[k][i]);
  return e;
}

// p~ of a cluster: sum_area_x / A, or its box (pm_refit_kernel's, [min xyz, max xyz]) centre when A = 0
__device__ __forceinline__ void wn_centre(double A, const double* ax, const float* box, float* p) {
#pragma unroll
  for (int c = 0; c < 3; ++c) p[c] = A > 0.0 ? (float)(ax[c] / A) : 0.5f * (box[c] + box[3 + c]);
}

// One thread per leaf: the leaf's expansion from its triangles (tri, in Morton order), then climb while this thread
// is the second arrival at the parent, merging the parent's two stored child records.
__global__ void __launch_bounds__(256) wn_refit_kernel(int F, int L, const float4* __restrict__ tri,
                                                       const PmNode* __restrict__ pnodes,
                                                       const int* __restrict__ leaf_parent, WnNode* nodes,
                                                       int* __restrict__ counter) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= L) return;
  const int t0 = l * PM_LEAF, t1 = min(F, (l + 1) * PM_LEAF);
  int p = leaf_parent[l];
  WnExp e;
  {
    double A = 0.0, ax[3] = {0.0, 0.0, 0.0}, n[3] = {0.0, 0.0, 0.0};
    for (int t = t0; t < t1; ++t) {
      const float4 r0 = __ldg(tri + 3 * (size_t)t), r1 = __ldg(tri + 3 * (size_t)t + 1),
                   r2 = __ldg(tri + 3 * (size_t)t + 2);
      const double a[3] = {r0.x, r0.y, r0.z}, b[3] = {r0.w, r1.x, r1.y}, c[3] = {r1.z, r1.w, r2.x};
      const double u[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]}, v[3] = {c[0] - a[0], c[1] - a[1], c[2] - a[2]};
      const double nt[3] = {0.5 * (u[1] * v[2] - u[2] * v[1]), 0.5 * (u[2] * v[0] - u[0] * v[2]),
                            0.5 * (u[0] * v[1] - u[1] * v[0])};
      const double at = sqrt(nt[0] * nt[0] + nt[1] * nt[1] + nt[2] * nt[2]);
      A += at;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        ax[k] += at * ((a[k] + b[k] + c[k]) / 3.0);
        n[k] += nt[k];
      }
    }
    wn_centre(A, ax, pnodes[p >> 1].box[p & 1], e.p);
    double m[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, r2max = 0.0;
    for (int t = t0; t < t1; ++t) {
      const float4 r0 = __ldg(tri + 3 * (size_t)t), r1 = __ldg(tri + 3 * (size_t)t + 1),
                   r2 = __ldg(tri + 3 * (size_t)t + 2);
      const double a[3] = {r0.x, r0.y, r0.z}, b[3] = {r0.w, r1.x, r1.y}, c[3] = {r1.z, r1.w, r2.x};
      const double u[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]}, v[3] = {c[0] - a[0], c[1] - a[1], c[2] - a[2]};
      const double nt[3] = {0.5 * (u[1] * v[2] - u[2] * v[1]), 0.5 * (u[2] * v[0] - u[0] * v[2]),
                            0.5 * (u[0] * v[1] - u[1] * v[0])};
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const double xi = (a[i] + b[i] + c[i]) / 3.0 - e.p[i];
#pragma unroll
        for (int j = 0; j < 3; ++j) m[3 * i + j] += xi * nt[j];
      }
      const double* vs[3] = {a, b, c};
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double dx = vs[k][0] - e.p[0], dy = vs[k][1] - e.p[1], dz = vs[k][2] - e.p[2];
        r2max = fmax(r2max, dx * dx + dy * dy + dz * dz);
      }
    }
    e.r = __double2float_ru(sqrt(r2max));
    e.a = (float)A;
#pragma unroll
    for (int k = 0; k < 3; ++k) e.n[k] = (float)n[k];
#pragma unroll
    for (int k = 0; k < 9; ++k) e.m[k] = (float)m[k];
  }
  while (true) {
    const int node = p >> 1, side = p & 1;
    wn_store(nodes + node, side, e);
    nodes[node].child[side] = pnodes[node].child[side];
    __threadfence();
    if (atomicAdd(&counter[node], 1) == 0) return;  // the sibling's thread arrives second and merges
    p = pnodes[node].parent;
    if (p < 0) return;  // the root's own expansion is never read
    const WnExp c0 = wn_load(nodes + node, 0), c1 = wn_load(nodes + node, 1);
    const double A = (double)c0.a + (double)c1.a;
    double ax[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) ax[k] = (double)c0.a * c0.p[k] + (double)c1.a * c1.p[k];
    wn_centre(A, ax, pnodes[p >> 1].box[p & 1], e.p);
    double d0[3], d1[3], l0 = 0.0, l1 = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      d0[k] = (double)c0.p[k] - e.p[k];
      d1[k] = (double)c1.p[k] - e.p[k];
      l0 += d0[k] * d0[k];
      l1 += d1[k] * d1[k];
    }
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j)
        e.m[3 * i + j] = (float)((double)c0.m[3 * i + j] + d0[i] * c0.n[j] + (double)c1.m[3 * i + j] +
                                 d1[i] * c1.n[j]);
#pragma unroll
    for (int k = 0; k < 3; ++k) e.n[k] = (float)((double)c0.n[k] + (double)c1.n[k]);
    e.a = (float)A;
    e.r = __double2float_ru(fmax(sqrt(l0) + c0.r, sqrt(l1) + c1.r));
  }
}

// the exact solid angles of leaf l's triangles seen from q, added to s in triangle order
__device__ __forceinline__ void wn_leaf(int l, int F, const float4* __restrict__ tri, float3 q, double& s) {
  for (int t = l * PM_LEAF; t < min(F, (l + 1) * PM_LEAF); ++t) {
    const float4 r0 = __ldg(tri + 3 * (size_t)t), r1 = __ldg(tri + 3 * (size_t)t + 1),
                 r2 = __ldg(tri + 3 * (size_t)t + 2);
    const float3 a = make_float3(r0.x - q.x, r0.y - q.y, r0.z - q.z),
                 b = make_float3(r0.w - q.x, r1.x - q.y, r1.y - q.z),
                 c = make_float3(r1.z - q.x, r1.w - q.y, r2.x - q.z);
    const float det = a.x * (b.y * c.z - b.z * c.y) + a.y * (b.z * c.x - b.x * c.z) + a.z * (b.x * c.y - b.y * c.x);
    if (det == 0.f) continue;
    const float la = sqrtf(a.x * a.x + a.y * a.y + a.z * a.z), lb = sqrtf(b.x * b.x + b.y * b.y + b.z * b.z),
                lc = sqrtf(c.x * c.x + c.y * c.y + c.z * c.z);
    const float den = la * lb * lc + (a.x * b.x + a.y * b.y + a.z * b.z) * lc +
                      (b.x * c.x + b.y * c.y + b.z * c.z) * la + (c.x * a.x + c.y * a.y + c.z * a.z) * lb;
    s += (double)(2.f * atan2f(det, den));
  }
}

// child k of nd: its far-field term when |q - p~| > beta r (returns true), else nothing (returns false)
__device__ __forceinline__ bool wn_far(const WnNode* __restrict__ nd, int k, float3 q, float beta, double& s) {
  const float4 pr = __ldg(&nd->pr[k]);
  const float x = pr.x - q.x, y = pr.y - q.y, z = pr.z - q.z, d2 = x * x + y * y + z * z, br = beta * pr.w;
  if (!(d2 > br * br)) return false;
  const float4 na = __ldg(&nd->na[k]);
  const float* m = nd->m[k];
  const float inv = rsqrtf(d2), ux = x * inv, uy = y * inv, uz = z * inv;
  const float mu0 = __ldg(m) * ux + __ldg(m + 1) * uy + __ldg(m + 2) * uz,
              mu1 = __ldg(m + 3) * ux + __ldg(m + 4) * uy + __ldg(m + 5) * uz,
              mu2 = __ldg(m + 6) * ux + __ldg(m + 7) * uy + __ldg(m + 8) * uz;
  const float tr = __ldg(m) + __ldg(m + 4) + __ldg(m + 8), umu = ux * mu0 + uy * mu1 + uz * mu2;
  const float un = ux * na.x + uy * na.y + uz * na.z;
  s += (double)((un + (tr - 3.f * umu) * inv) * inv * inv);
  return true;
}

// thread t takes query qorder[t] (pm_query_kernel's order)
__global__ void __launch_bounds__(128) wn_query_kernel(int Q, int F, int L, const float* __restrict__ points,
                                                       const uint32_t* __restrict__ qorder,
                                                       const float4* __restrict__ tri,
                                                       const WnNode* __restrict__ nodes, float beta,
                                                       float* __restrict__ winding) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= Q) return;
  const int qi = (int)qorder[t];
  const float3 q = make_float3(points[3 * (size_t)qi], points[3 * (size_t)qi + 1], points[3 * (size_t)qi + 2]);
  double s = 0.0;
  if (L == 1) {
    wn_leaf(0, F, tri, q, s);
  } else {
    int stack[PM_STACK];
    int sp = 0, node = 0;
    while (true) {
      const WnNode* nd = nodes + node;
      const int2 ch = __ldg(reinterpret_cast<const int2*>(nd->child));
      int next = -1;
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        if (wn_far(nd, k, q, beta, s)) continue;
        const int c = k == 0 ? ch.x : ch.y;
        if (c < 0) wn_leaf(~c, F, tri, q, s);
        else if (next < 0) next = c;
        else stack[sp++] = c;
      }
      if (next >= 0) {
        node = next;
        continue;
      }
      if (sp == 0) break;
      node = stack[--sp];
    }
  }
  winding[qi] = (float)(s * (0.25 / M_PI));
}

cudaError_t launch_winding_number(int F, int Q, const float* verts, const int32_t* faces, const float* points,
                                  float beta, float* winding, float* dist2, long long* face, float* bary, void* ws,
                                  cudaStream_t s) {
  if (Q == 0) return cudaSuccess;
  const WnWS w = WnWS::from((char*)ws, F, Q, pm_fwd_cub_bytes(F, Q));
  const int L = (F + PM_LEAF - 1) / PM_LEAF;
  pm_build(F, Q, verts, faces, points, w.pm, s);
  if (L > 1) {
    cudaMemsetAsync(w.counter, 0, (L - 1) * sizeof(int), s);
    wn_refit_kernel<<<(L + 255) / 256, 256, 0, s>>>(F, L, (const float4*)w.pm.tri, w.pm.nodes, w.pm.leaf_parent,
                                                    w.nodes, w.counter);
  }
  if (dist2) pm_query(F, Q, points, w.pm, dist2, face, bary, s);
  wn_query_kernel<<<(Q + 127) / 128, 128, 0, s>>>(Q, F, L, points, w.pm.qorder, (const float4*)w.pm.tri, w.nodes,
                                                  beta, winding);
  return cudaGetLastError();
}

}  // namespace dgm
