// dmc_cell.cuh -- the per-cell rules of dual marching cubes, shared by dmc.cu and flexicubes.cu: the patch tables,
// which edges of a cell are interior, which patches get a vertex, the cut edges of a case and the vertex of a
// patch.  Each translation unit holds its own copy of the device tables and uploads it once per device.
#pragma once
#include "common.cuh"
#include "mc_tables.h"

namespace dgm {

// per case, built from DMC_PATCH_OF_EDGE: the patch of every edge as 12 nibbles (15: the edge is not cut), and
// the 12-bit edge mask of each patch at bits 16 p
static __device__ unsigned long long g_dmc_pof[256];
static __device__ unsigned long long g_dmc_pmask[256];

// bit e: edge e of cell (i, j, k) is interior -- its two coordinates across the edge, cell + combo bit, lie in
// [1, G - 2].  Edge e = 4 * axis + combo, combo bit 0 / 1 for the lower / higher of the other two axes.
__device__ __forceinline__ unsigned dmc_interior_edges(int G, int i, int j, int k) {
  const bool lo0 = i >= 1, lo1 = j >= 1, lo2 = k >= 1, hi0 = i <= G - 3, hi1 = j <= G - 3, hi2 = k <= G - 3;
  unsigned m = 0;
#pragma unroll
  for (int e = 0; e < 12; ++e) {
    const int a = e >> 2;
    const bool b0 = a == 0 ? ((e & 1) ? hi1 : lo1) : ((e & 1) ? hi0 : lo0);
    const bool b1 = a == 2 ? ((e & 2) ? hi1 : lo1) : ((e & 2) ? hi2 : lo2);
    m |= (unsigned)(b0 && b1) << e;
  }
  return m;
}

// the patches of case cs with a dual vertex: those with an interior edge
__device__ __forceinline__ unsigned dmc_need(unsigned long long pm, unsigned imask) {
  unsigned need = 0;
#pragma unroll
  for (int p = 0; p < 4; ++p) need |= (unsigned)((((unsigned)(pm >> (16 * p))) & imask & 0xfffu) != 0) << p;
  return need;
}

// the cut edges of a case (union of its patches)
__device__ __forceinline__ unsigned dmc_cut(unsigned long long pm) {
  return (unsigned)(pm | (pm >> 16) | (pm >> 32) | (pm >> 48)) & 0xfffu;
}

// dual vertex (item-local) of the patch of cell `c` (cell coordinates ci, cj, ck) that contains local edge le
__device__ __forceinline__ uint32_t dmc_vertex_of(int G, unsigned long long w, int ci, int cj, int ck, int le) {
  const unsigned cs = (unsigned)(w >> 32) & 255u;
  const unsigned p = (unsigned)(__ldg(&g_dmc_pof[cs]) >> (4 * le)) & 15u;
  const unsigned need = dmc_need(__ldg(&g_dmc_pmask[cs]), dmc_interior_edges(G, ci, cj, ck));
  return (uint32_t)w + (uint32_t)__popc(need & ((1u << p) - 1u));
}

static unsigned long long g_dmc_tables_uploaded = 0;  // per device
static cudaError_t upload_dmc_tables() {
  if (!once_per_device(g_dmc_tables_uploaded)) return cudaSuccess;
  unsigned long long pof[256], pmask[256];
  for (int cs = 0; cs < 256; ++cs) {
    pof[cs] = ~0ull;
    pmask[cs] = 0;
    for (int e = 0; e < 12; ++e) {
      const int p = DMC_PATCH_OF_EDGE[cs][e];
      if (p >= 0) {
        pof[cs] &= ~(15ull << (4 * e)) | ((unsigned long long)p << (4 * e));
        pmask[cs] |= 1ull << (16 * p + e);
      }
    }
  }
  cudaError_t e = cudaMemcpyToSymbol(g_dmc_pof, pof, sizeof(pof));
  if (e == cudaSuccess) e = cudaMemcpyToSymbol(g_dmc_pmask, pmask, sizeof(pmask));
  if (e != cudaSuccess) g_dmc_tables_uploaded = 0;  // retry on the next call
  return e;
}

}  // namespace dgm
