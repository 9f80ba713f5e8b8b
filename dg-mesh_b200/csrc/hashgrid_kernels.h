// hashgrid_kernels.h -- host-side launch interface of hashgrid.cu (the multiresolution hash encoding of (x, y, z, t)
// and its gradients); include/dgmesh_b200.h "dghg_"
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace dgm {

#define HG_MAX_G 4
#define HG_MAX_L 24

// the grids of one field: grid g is of kind kind[g] (0 xyz, 1 xyt, 2 yzt, 3 xzt) with table tab[g], [L, T, Fe]
// channels-last, T = 2^log2T; level l has spatial resolution R[l] and time resolution Rt[l] = min(R[l], R_t); bit l
// of dense[g] is set when level l of grid g indexes its nodes densely.  Passed to the kernels by value.
struct HgField {
  const float* tab[HG_MAX_G];
  int kind[HG_MAX_G];
  int R[HG_MAX_L], Rt[HG_MAX_L];
  uint32_t dense[HG_MAX_G];
  int G, L, Fe, log2T;
};
struct HgGrads {
  float* tab[HG_MAX_G];
};

// backward workspace: the int64 fixed-point accumulator [G, L, T, Fe] and max|grad_out| per (grid, level) as float
// bits [G, L]
size_t hg_ws_bytes(const HgField& f);

cudaError_t launch_hashgrid_fwd(int F, int N, const HgField& f, const float* box, const float* x, const float* t,
                                float* out, cudaStream_t s);
cudaError_t launch_hashgrid_bwd(int F, int N, const HgField& f, const float* box, const float* x, const float* t,
                                const float* grad_out, float* grad_x, const HgGrads& g, void* ws, cudaStream_t s);

}  // namespace dgm
