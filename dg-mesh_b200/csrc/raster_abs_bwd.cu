// raster_abs_bwd.cu -- the blend backward with the absolute screen-space gradient (AbsGS; DESIGN.md §4, "Absolute
// screen-space gradients") for sm_90a.
//
//   render_bwd_kernel<*, *, *, true>  the blend backward of each existing combination (colour, depth / alpha,
//                                     + normal map, + surface maps, + both) that also adds, per Gaussian, the sums
//                                     over pixels of |dL/dmean2D.x| and |dL/dmean2D.y| of each pixel's term
//
// launch_render_bwd_abs picks one of the five and launches it through launch_blend_bwd (raster_bwd_blend.cuh).  Kept
// apart from raster_bwd.cu, raster_nrm_bwd.cu and raster_surf_bwd.cu so that the kernels there compile exactly as they
// do without the statistic.
#include "../../include/dgmesh_b200.h"
#include "common.cuh"
#include "raster_kernels.h"
#include "raster_bwd_blend.cuh"

namespace dgm {

// the blend backward of one frame with a.dL_dmean2D_abs (launch_render_bwd); the other arguments pick the instance
// by the rule of launch_blend_bwd
cudaError_t launch_render_bwd_abs(const BwdArgs& a, cudaStream_t s) {
  if (a.dL_ddistortion)
    return a.dL_dnormal ? launch_blend_bwd<true, true, true, true>(a, s) : launch_blend_bwd<true, false, true, true>(a, s);
  if (a.dL_dnormal) return launch_blend_bwd<true, true, false, true>(a, s);
  return (a.dL_ddepth || a.dL_dalpha) ? launch_blend_bwd<true, false, false, true>(a, s)
                                      : launch_blend_bwd<false, false, false, true>(a, s);
}

}  // namespace dgm
