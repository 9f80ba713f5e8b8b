// mc_kernels.h -- host-side interface of mc.cu
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace dgm {
// vid packs a vertex index into its low 29 bits (the owned-edge mask takes the top 3): V <= 2^29
// (a batch's total too: the emit's capacity check is on the batch's vertex index)
constexpr long long MC_MAX_VERTS = 1ll << 29;
// a batch is B grids phi[B,G,G,G], 1 <= B <= MC_MAX_BATCH; B = 1 is the single grid
constexpr int MC_MAX_BATCH = 64;
struct McWS {
  unsigned long long *blk_counts, *blk_offsets;  // per brick of 8 x 32 nodes: (vertices | triangles << 32), exclusive scan
  long long* item_off;                            // [2B + 2]: first vertex of every item and V; first face and F
  uint32_t* vid;                                  // [B n] sparse: the item's first vertex index | owned-edge mask << 29
  char* cub_temp;
  size_t cub_bytes;
  static McWS from(char* base, int G, int B = 1, size_t* bytes = nullptr);
};
// item k's vertices are [voff[k], voff[k + 1]) of the batch (passed by value: B <= 64)
struct McItems {
  int B;
  int voff[MC_MAX_BATCH + 1];
};
size_t mc_num_blocks(int G);
// totals[2B] = {V_k, F_k} of every item (and totals_host, when given, behind ev)
cudaError_t launch_mc_count(int B, int G, const float* phi, float iso, void* ws, int32_t* totals,
                            int32_t* totals_host, cudaEvent_t ev, cudaStream_t s);
// vsrc[V_cap]: node * 3 + axis of every vertex (node local to its item), read back by the backward
cudaError_t launch_mc_emit(int B, int G, const float* phi, float iso, void* ws, float* verts, int32_t* vsrc,
                           long long V_cap, int32_t* faces, long long F_cap, cudaStream_t s);
cudaError_t launch_mc_backward(int G, const McItems& it, const float* phi, float iso, const int32_t* vsrc,
                               const float* dverts, float* dphi, cudaStream_t s);
}  // namespace dgm
