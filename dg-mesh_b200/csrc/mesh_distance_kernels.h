// mesh_distance_kernels.h -- host-side launch interface of mesh_distance.cu (closest points on a triangle mesh,
// include/dgmesh_b200.h "dgpm_")
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace dgm {

#define PM_LEAF 4    // triangles per BVH leaf (consecutive in Morton order)
#define PM_STACK 64  // traversal stack entries; mesh_distance.cu states the bound

// one internal node of the BVH: the boxes of both children (so a visit reads one 64-byte record and tests two boxes),
// the children (>= 0 internal, ~l for leaf l) and the parent ((parent << 1) | side, -1 at the root)
struct alignas(16) PmNode {
  float box[2][6];  // [child][min xyz, max xyz]
  int child[2];
  int parent;
  int pad;
};

// forward: the BVH, rebuilt on every call, and the queries' Morton order
struct PmFwdWS {
  float* cent;              // [F,3] triangle centroids
  uint32_t *bounds, *codes, *codes_sorted, *idx, *order;
  uint32_t *qbounds, *qcodes, *qcodes_sorted, *qidx, *qorder;
  float* tri;               // [F,12] triangles in Morton order: a, b, c, face index (three float4)
  PmNode* nodes;            // [L-1], L = ceil(F / PM_LEAF) leaves
  int* leaf_parent;         // [L]
  int* counter;             // [L-1] refit arrivals
  char* cub_temp;
  size_t cub_bytes;
  static PmFwdWS from(char* base, size_t F, size_t Q, size_t cub_bytes, size_t* bytes = nullptr);
};
size_t pm_fwd_cub_bytes(int F, int Q);
// the BVH over the faces and the queries' Morton order, into w (Q >= 1); then the closest-point query on them
void pm_build(int F, int Q, const float* verts, const int32_t* faces, const float* points, const PmFwdWS& w,
              cudaStream_t s);
void pm_query(int F, int Q, const float* points, const PmFwdWS& w, float* dist2, long long* face, float* bary,
              cudaStream_t s);

// Barill et al. 2018's order-1 expansions of both children of one internal node (parallel to PmNode): centroid p~
// and radius r, zeroth moment N = sum a_t n_t and total area A, first moment M = sum a_t (x_t - p~) n_t^T (row
// major), and the children again, so a winding visit reads this record alone
struct alignas(16) WnNode {
  float4 pr[2];     // [child] p~ xyz, r
  float4 na[2];     // [child] N xyz, A
  float m[2][9];    // [child] M
  int child[2];     // as PmNode::child
};

// winding number: the forward's BVH and query order, then the expansions with their own refit arrivals
struct WnWS {
  PmFwdWS pm;
  WnNode* nodes;    // [L-1]
  int* counter;     // [L-1]
  static WnWS from(char* base, size_t F, size_t Q, size_t cub_bytes, size_t* bytes = nullptr);
};

// backward: the CSR inverse of the 3Q (vertex, entry) pairs
struct PmBwdWS {
  uint32_t *keys_in, *keys_out, *vals_in, *vals_out;
  char* cub_temp;
  size_t cub_bytes;
  static PmBwdWS from(char* base, size_t Q, size_t cub_bytes, size_t* bytes = nullptr);
};
size_t pm_bwd_cub_bytes(int V, int Q);

cudaError_t launch_point_mesh_distance(int F, int Q, const float* verts, const int32_t* faces, const float* points,
                                       float* dist2, long long* face, float* bary, void* ws, cudaStream_t s);
// winding [Q] and, when dist2 is not null, launch_point_mesh_distance's outputs from the same build (ws: WnWS)
cudaError_t launch_winding_number(int F, int Q, const float* verts, const int32_t* faces, const float* points,
                                  float beta, float* winding, float* dist2, long long* face, float* bary, void* ws,
                                  cudaStream_t s);
cudaError_t launch_point_mesh_distance_bwd(int V, int Q, const float* verts, const int32_t* faces,
                                           const float* points, const long long* face, const float* bary,
                                           const float* grad_dist2, float* grad_points, float* grad_verts, void* ws,
                                           cudaStream_t s);

}  // namespace dgm
