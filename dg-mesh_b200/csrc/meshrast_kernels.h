// meshrast_kernels.h -- host-side launch interface of meshrast.cu
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>

namespace dgm {
// B images rendered in one call (nvdiffrast's range mode), 1 <= B <= MR_MAX_BATCH; every buffer of the images is
// [B, H, W, ...] and B = 1 is the single image.  Image b draws triangles [start[b], start[b] + off[b + 1] - off[b]);
// the ranges are passed by value (B <= 64 keeps them small), so no copy is enqueued.
constexpr int MR_MAX_BATCH = 64;
// triangle ids are stored in rast.w with nvdiffrast's encoding (meshrast.cu), whose bit pattern stays a finite float
// up to 0x7f7fffff - 0x4a800000 ids; F and every range end are held to 2^29, below that
constexpr int MR_MAX_TRIANGLES = 1 << 29;
struct MrRanges {
  int B;
  int start[MR_MAX_BATCH];
  int off[MR_MAX_BATCH + 1];  // prefix sum of the counts
};
cudaError_t launch_mr_rasterize(const MrRanges& R, int W, int H, const float* pos, const int* tri, void* zbuf,
                                float* rast, cudaStream_t s);
cudaError_t launch_mr_rasterize_bwd(int B, int W, int H, const float* rast, const int* tri, const float* pos,
                                    const float* grast, float* gpos, cudaStream_t s);
cudaError_t launch_mr_interpolate(int B, int W, int H, int C, const float* attr, const float* rast, const int* tri,
                                  float* out, cudaStream_t s);
cudaError_t launch_mr_interpolate_bwd(int B, int W, int H, int C, const float* attr, const float* rast,
                                      const int* tri, const float* gout, float* gattr, float* grast, cudaStream_t s);
cudaError_t launch_mr_antialias(int B, int W, int H, int C, const float* color, const float* rast, const float* pos,
                                const int* tri, const int* opp, float* out, cudaStream_t s);
cudaError_t launch_mr_antialias_bwd(int B, int W, int H, int C, const float* color, const float* rast,
                                    const float* pos, const int* tri, const int* opp, const float* gout,
                                    float* gcolor, float* gpos, cudaStream_t s);
}  // namespace dgm
