// flexicubes_kernels.h -- host-side interface of flexicubes.cu
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace dgm {
// training mode adds one centre vertex and two more triangles per quad: Q_cap < 2^29 keeps the 4 Q triangles
// below 2^31 and every vertex index (V + Q < 2^28 + 2^29) inside int32
constexpr long long FC_MAX_QUADS_TRAINING = (1ll << 29) - 1;
constexpr int FC_SLOTS = 7;  // crossings per patch, at most

// the raw per-node offsets and per-cell weights; a null pointer is the neutral value (raw 0, offset 0)
struct FcParams {
  const float *deform, *alpha, *beta, *gamma;
};

// after launch_dmc_count on ws: verts[V_cap (+ Q_cap in training), 3] (normalised), vsrc[V_cap],
// ldev[V_cap, FC_SLOTS] (L_dev per crossing, padded), vk[V_cap] (crossings per vertex), faces[(2 | 4) Q_cap, 3],
// quads[Q_cap, 4]
cudaError_t launch_fc_emit(int G, const float* phi, float iso, const FcParams& w, bool training, bool normalize,
                           void* ws, float* verts, int32_t* vsrc, float* ldev, int32_t* vk, long long V_cap,
                           int32_t* faces, int32_t* quads, long long Q_cap, cudaStream_t s);
size_t fc_backward_ws_bytes(int G, long long V, long long Q, bool training);
// dverts[V (+ Q), 3] w.r.t. the normalised vertices, dldev[V, FC_SLOTS] or null; ddeform, dalpha, dbeta, dgamma
// may be null (not computed), dgamma must be null in inference mode
cudaError_t launch_fc_backward(int G, int V, int Q, const float* phi, float iso, const FcParams& w, bool training,
                               bool normalize, const float* verts, const int32_t* vsrc, const int32_t* quads,
                               const float* dverts, const float* dldev, void* ws, float* dphi, float* ddeform,
                               float* dalpha, float* dbeta, float* dgamma, cudaStream_t s);
}  // namespace dgm
