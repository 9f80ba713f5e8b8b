// raster_surf_bwd.cu -- backward of the median-depth and depth-distortion maps (DESIGN.md §4, "Median depth and
// distortion") for sm_90a.
//
//   render_bwd_kernel<true, false, true>  the blend backward with the distortion map (+ the depth / alpha maps)
//   render_bwd_kernel<true, true, true>   the same with the normal map
//   median_grad_kernel                    dL/dd of each pixel's median record: the median depth is piecewise
//                                         constant in alpha, so its gradient reaches the depth of one record only
//
// launch_render_bwd_surf picks one of the two blend instances and launches it through launch_blend_bwd
// (raster_bwd_blend.cuh).  Kept apart from raster_bwd.cu and raster_nrm_bwd.cu so that the kernels there compile
// exactly as they do without the surface maps.
#include "../../include/dgmesh_b200.h"
#include "common.cuh"
#include "raster_kernels.h"
#include "raster_bwd_blend.cuh"

namespace dgm {

// one thread per pixel: grad_acc[id] float 9 (dL/d(depth)) += dL/dmedian of every pixel whose median record is id
__global__ void __launch_bounds__(256) median_grad_kernel(int npix, const uint32_t* __restrict__ median_id,
                                                          const float* __restrict__ dL_dmedian,
                                                          float4* __restrict__ grad_acc) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= npix) return;
  const uint32_t id = median_id[i];
  const float g = dL_dmedian[i];
  if (id != 0xFFFFFFFFu && g != 0.0f) atomicAdd(reinterpret_cast<float*>(grad_acc + 3 * (size_t)id) + 9, g);
}

// the blend backward of one frame with the distortion map (launch_render_bwd with a.dL_ddistortion)
cudaError_t launch_render_bwd_surf(const BwdArgs& a, cudaStream_t s) {
  return a.dL_dnormal ? launch_blend_bwd<true, true, true, false>(a, s) : launch_blend_bwd<true, false, true, false>(a, s);
}

// dL/dmedian into the depth gradient of the median records (one frame: frame 0 of the arguments); after the frame's
// forward and before preprocess_bwd, which reads float 9 of grad_acc
cudaError_t launch_median_grad(const BwdArgs& a, cudaStream_t s) {
  if (a.P == 0) return cudaSuccess;
  const int npix = a.W * a.H;
  const SurfWS sw = SurfWS::from((char*)a.surf_ws, (size_t)npix);
  GeomWS g = GeomWS::from((char*)a.geom_ws, a.P);
  g_prof.begin(9, s);
  median_grad_kernel<<<(npix + 255) / 256, 256, 0, s>>>(npix, sw.median_id, a.dL_dmedian, g.grad_acc);
  g_prof.end(9, s);
  return cudaGetLastError();
}

}  // namespace dgm
