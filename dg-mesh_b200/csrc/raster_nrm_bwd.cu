// raster_nrm_bwd.cu -- backward of the normal map (DESIGN.md §4, "Normal maps") for sm_90a.
//
//   render_bwd_kernel<true, true>  the blend backward with the normal map: also dL/dn_i = sum over pixels of
//                                  alpha_i T_i dL/dN into the normal workspace's per-Gaussian accumulator
//   normal_grad_finish_kernel      dL/dnormals from the accumulators of every frame, which it re-zeroes
//
// launch_render_bwd_nrm launches the blend instance through launch_blend_bwd (raster_bwd_blend.cuh).  Kept apart from
// raster_bwd.cu so that the kernels there compile exactly as they do without the normal map.
#include "../../include/dgmesh_b200.h"
#include "common.cuh"
#include "raster_kernels.h"
#include "raster_bwd_blend.cuh"

namespace dgm {

// dL/dnormals from the normal accumulators of F frames (frame f's normal workspace at nrm_ws + f * stride), one
// thread per Gaussian: per_frame, out[f][g] = acc_f[g]; else out[g] = the sum over the frames in frame order.
// Every accumulator is re-zeroed for the next backward (out NULL: only that).
__global__ void __launch_bounds__(256) normal_grad_finish_kernel(int F, int P, char* nrm_ws, size_t stride,
                                                                 int per_frame, float* __restrict__ out) {
  const int g = blockIdx.x * 256 + threadIdx.x;
  if (g >= P) return;
  float3 sum = make_float3(0.f, 0.f, 0.f);
  for (int f = 0; f < F; ++f) {
    float4* acc = NrmWS::from(nrm_ws + f * stride, P, 0).acc + g;
    const float4 v = *acc;
    *acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (per_frame) {
      if (out) {
        float* o = out + 3 * ((size_t)f * P + g);
        o[0] = v.x, o[1] = v.y, o[2] = v.z;
      }
    } else if (f == 0) {
      sum = make_float3(v.x, v.y, v.z);
    } else {
      sum = make_float3(sum.x + v.x, sum.y + v.y, sum.z + v.z);
    }
  }
  if (!per_frame && out) out[3 * g] = sum.x, out[3 * g + 1] = sum.y, out[3 * g + 2] = sum.z;
}

// the blend backward of one frame with the normal map (launch_render_bwd with a.dL_dnormal)
cudaError_t launch_render_bwd_nrm(const BwdArgs& a, cudaStream_t s) {
  return launch_blend_bwd<true, true, false, false>(a, s);
}

// after the blend backward of every frame: dL/dnormals, and the accumulators back to zero
cudaError_t launch_normal_grad_finish(const BwdArgs& a, cudaStream_t s) {
  if (a.P == 0) return cudaSuccess;
  g_prof.begin(8, s);
  normal_grad_finish_kernel<<<(a.P + 255) / 256, 256, 0, s>>>(a.F, a.P, (char*)a.nrm_ws, a.nrm_stride,
                                                              a.normals_per_frame, a.dL_dnormals);
  g_prof.end(8, s);
  return cudaGetLastError();
}

}  // namespace dgm
