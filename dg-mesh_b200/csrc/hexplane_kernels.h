// hexplane_kernels.h -- host-side launch interface of hexplane.cu (the HexPlane / K-Planes space-time feature field,
// its gradients and its plane regularisers); include/dgmesh_b200.h "dghp_"
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace dgm {

#define HP_MAX_S 4
#define HP_PLANES 6  // (x,y) (x,z) (x,t) (y,z) (y,t) (z,t); spatial 0, 1, 3, time 2, 4, 5

// the planes of one field: plane (s, p) is p[6 s + p], channels-last [R_b, R_a, C]; R[s] is scale s's spatial
// resolution, Rt the time resolution of every scale.  Passed to the kernels by value.
struct HpField {
  const float* p[HP_MAX_S * HP_PLANES];
  int R[HP_MAX_S];
  int Rt, S, C;
};
struct HpGrads {
  float* p[HP_MAX_S * HP_PLANES];
};

// backward: every (plane, entry)'s dL/dsample [C] and bilinear fractions, the entries' cell keys sorted (stably)
// with their ids, and each cell's four corner sums [cells, 4, C]; entries of plane (s, p) are the N points
// (spatial) or the F N (frame, point) pairs (time), in that order, planes in (s, p) order
struct HpWS {
  float* stage;      // [E, C]
  float2* frac;      // [E]
  uint32_t *keys_in, *keys_out, *vals_in, *vals_out;  // [E]
  float* cell_acc;   // [cells, 4, C]
  char* cub_temp;
  size_t cub_bytes;
  static HpWS from(char* base, size_t E, size_t cells, int C, size_t cub_bytes, size_t* bytes = nullptr);
};
size_t hp_entries(int F, int N, int S);
size_t hp_cells(const HpField& f);
size_t hp_cub_bytes(size_t E, size_t cells);

cudaError_t launch_hexplane_fwd(int F, int N, const HpField& f, const float* box, const float* x, const float* t,
                                float* out, cudaStream_t s);
cudaError_t launch_hexplane_bwd(int F, int N, const HpField& f, const float* box, const float* x, const float* t,
                                const float* grad_out, float* grad_x, const HpGrads& g, void* ws, cudaStream_t s);

// regularisers: each CTA's partial sums, and a counter that elects the CTA which adds them up
size_t hp_reg_blocks(const HpField& f);
size_t hp_reg_ws_bytes(const HpField& f);
cudaError_t launch_hexplane_reg_fwd(const HpField& f, float* losses, void* ws, cudaStream_t s);
cudaError_t launch_hexplane_reg_bwd(const HpField& f, const float* grad_losses, const HpGrads& g, cudaStream_t s);

}  // namespace dgm
