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
// the exclusive scan of B * nb packed brick totals and the item totals behind it (shared by marching cubes and
// dual marching cubes)
cudaError_t launch_mc_scan_totals(int B, size_t nb, unsigned long long* blk_counts,
                                  unsigned long long* blk_offsets, long long* item_off, void* cub_temp,
                                  size_t cub_bytes, int32_t* totals, int32_t* totals_host, cudaEvent_t ev,
                                  cudaStream_t s);
size_t mc_cub_bytes(size_t n);
// totals[2B] = {V_k, F_k} of every item (and totals_host, when given, behind ev)
cudaError_t launch_mc_count(int B, int G, const float* phi, float iso, void* ws, int32_t* totals,
                            int32_t* totals_host, cudaEvent_t ev, cudaStream_t s);
// vsrc[V_cap]: node * 3 + axis of every vertex (node local to its item), read back by the backward
cudaError_t launch_mc_emit(int B, int G, const float* phi, float iso, void* ws, float* verts, int32_t* vsrc,
                           long long V_cap, int32_t* faces, long long F_cap, cudaStream_t s);
cudaError_t launch_mc_backward(int G, const McItems& it, const float* phi, float iso, const int32_t* vsrc,
                               const float* dverts, float* dphi, cudaStream_t s);

// Dual marching cubes (dmc.cu).  cvid packs a cell's first dual vertex (low 32 bits) and its case (bits 32..39);
// vertex indices stay below 2^28 so that cell * 4 + patch and the counts fit their int32 records.
constexpr long long DMC_MAX_VERTS = 1ll << 28;
constexpr long long DMC_MAX_QUADS = (1ll << 30) - 1;  // faces = 2 quads < 2^31
struct DmcWS {
  unsigned long long *blk_counts, *blk_offsets;  // per brick: (dual vertices | quads << 32), exclusive scan
  long long* item_off;                            // [2B + 2]: first vertex of every item and V; first quad and Q
  unsigned long long* cvid;                       // [B n] sparse: first dual vertex of a cell | case << 32
  char* cub_temp;
  size_t cub_bytes;
  static DmcWS from(char* base, int G, int B = 1, size_t* bytes = nullptr);
};
// totals[2B] = {V_k, Q_k} of every item (and totals_host, when given, behind ev)
cudaError_t launch_dmc_count(int B, int G, const float* phi, float iso, void* ws, int32_t* totals,
                             int32_t* totals_host, cudaEvent_t ev, cudaStream_t s);
// verts[V_cap,3], vsrc[V_cap] = cell * 4 + patch (cell local to its item), faces[2 Q_cap, 3], quads[Q_cap, 4] or null
cudaError_t launch_dmc_emit(int B, int G, const float* phi, float iso, void* ws, float* verts, int32_t* vsrc,
                            long long V_cap, int32_t* faces, int32_t* quads, long long Q_cap, cudaStream_t s);
// cvid[cell] = the first dual vertex of every cell with one (item-local), rebuilt from vsrc
void launch_dmc_first_vertex(int G, const McItems& it, const int32_t* vsrc, unsigned long long* cvid,
                             cudaStream_t s);
// ws: any workspace of the batch's size (the backward rebuilds the cells' first vertices from vsrc)
cudaError_t launch_dmc_backward(int G, const McItems& it, const float* phi, float iso, void* ws, const int32_t* vsrc,
                                const float* dverts, float* dphi, cudaStream_t s);
}  // namespace dgm
