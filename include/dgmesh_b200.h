/*
 * dgmesh_b200.h -- C-ABI of the H100-native DG-Mesh hot path (libdgmesh_b200.so).
 *
 * Drop-in boundary: every entry point below stands in for one native interface
 * of the reference (Isabella98Liu/DG-Mesh @ 754f42c); the reference file:line it
 * replaces is cited on each declaration.  Conventions (all entry points):
 *
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless
 *     the name ends in `_host`; no torch / C++ types cross this boundary;
 *   - the library never allocates, never frees and never synchronises: the
 *     caller owns all memory (query-then-call workspaces) and passes the CUDA
 *     stream (`void* stream` == cudaStream_t) the work is enqueued on;
 *   - "absent" optional inputs are NULL (the reference passes zero-element
 *     tensors whose data_ptr is null, dgr/rasterize_points.cu:84-103);
 *   - return value: 0 on success, a negative DGM_E_* code on a host-detectable
 *     error (bad argument, launch failure).  Device-side conditions (workspace
 *     overflow) are reported through the `status` words, see dgr_forward.
 *
 * Layouts are the reference's: row-major contiguous fp32 / int32 tensors.
 */
#ifndef DGMESH_B200_H_
#define DGMESH_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DGM_OK 0
#define DGM_E_BADARG (-1)
#define DGM_E_WORKSPACE (-2) /* a workspace is smaller than the query says */
#define DGM_E_LAUNCH (-3)    /* cudaGetLastError() != cudaSuccess after enqueue */

/* library / build identification ("dgmesh_b200 <ver> sm_90a") */
const char* dgm_version(void);
/* cudaGetErrorString of the last launch error seen by this thread (or "") */
const char* dgm_last_error(void);

/* Early-notification object for dgr_forward / dgr_forward_batch (see there): a CUDA event
 * plus a pinned, device-mapped host array of 64 status blocks (int32[64 * DGR_STATUS_WORDS]).
 * Stands in for the reference's blocking cudaMemcpy of num_rendered
 * (rasterizer_impl.cu:281): the caller waits for the event instead, with the rest of the
 * forward already queued.  dgm_notify_wait = cudaEventSynchronize. */
int dgm_notify_create(void** handle);
int32_t* dgm_notify_host(void* handle);
void* dgm_notify_event(void* handle);
int dgm_notify_wait(void* handle);
int dgm_notify_destroy(void* handle);

/* ------------------------------------------------------------------------
 * Differentiable 3D-Gaussian rasterizer
 * replaces CudaRasterizer::Rasterizer (dgr/cuda_rasterizer/rasterizer.h:20-86,
 * implementation dgr/cuda_rasterizer/rasterizer_impl.cu:198-336, 340-434) and
 * the torch binding dgr/rasterize_points.cu:35-217.
 * ------------------------------------------------------------------------ */

/* device status block written by dgr_forward (int32[DGR_STATUS_WORDS]) */
#define DGR_STATUS_WORDS 8
#define DGR_ST_NUM_RENDERED 0 /* R = sum of tiles touched (reference: num_rendered,
                                 rasterizer_impl.cu:281) -- stays on the device */
#define DGR_ST_OVERFLOW 1     /* 1 if R > R_cap: binning + blend were skipped */
#define DGR_ST_MAX_TILE 2     /* longest per-tile list (diagnostic) */
#define DGR_ST_DEPTH_LO 3     /* float bits: smallest / largest view depth of the visible set; */
#define DGR_ST_DEPTH_HI 4     /* feed them to the next call as depth_hint_lo / depth_hint_hi   */

/* Workspace sizes for P Gaussians, W x H image and room for R_cap
 * (Gaussian, tile) instances.  Mirrors required<GeometryState/ImageState/
 * BinningState>() (rasterizer_impl.h:66-72).  The three buffers play the role
 * of the reference's geomBuffer / binningBuffer / imgBuffer byte tensors
 * (rasterize_points.cu:68-78); their internal layout is private to this
 * library (see DESIGN.md) and they must be handed unchanged to dgr_backward. */
int dgr_workspace_sizes(int P, int W, int H, int64_t R_cap,
                        size_t* geom_bytes, size_t* binning_bytes, size_t* img_bytes);

/* Forward: preprocess -> per-tile binning/sort -> alpha-composite.
 * Same inputs / outputs as Rasterizer::forward (rasterizer.h:28-52):
 *   P, D (active SH degree), M (SH coeffs per Gaussian, 0 if shs == NULL)
 *   background[3], means3D[P,3], shs[P,M,3] | colors_precomp[P,3],
 *   opacities[P], scales[P,3] + rotations[P,4] | cov3D_precomp[P,6],
 *   viewmatrix[16], projmatrix[16] (row-vector convention, read column-major,
 *   auxiliary.h:58-77), cam_pos[3]
 *   -> out_color[3,H,W], radii[P] (int32; may be NULL)
 * No host synchronisation: where the reference copies num_rendered to the host
 * (rasterizer_impl.cu:281) this writes it to status[DGR_ST_NUM_RENDERED].  If
 * R exceeds R_cap, status[DGR_ST_OVERFLOW] = 1, out_color is filled with the
 * background and the caller must retry with a larger R_cap.
 * Early notification (optional, so that the caller can retry BEFORE anyone consumes
 * the image -- the drop-in Python layer always does):
 *   status_host   pinned, device-mapped host memory int32[DGR_STATUS_WORDS] or NULL: the
 *                 tile-scan kernel stores the status words there as well;
 *   status_event  cudaEvent_t or NULL: recorded on `stream` right behind the tile scan,
 *                 i.e. after ~1/5 of the forward -- waiting for it leaves the scatter /
 *                 sort / blend kernels queued, so the GPU does not idle.
 * depth_hint_lo < depth_hint_hi (view-depth range of an earlier, similar frame, from
 * status[DGR_ST_DEPTH_LO/HI]) lets preprocess build the (tile, depth-bucket) histogram
 * itself (one kernel less); the hint only affects bucket balance, never the result.
 * Pass 0, 0 when there is none.  max_tile_hint (status[DGR_ST_MAX_TILE] of an earlier frame, 0 = unknown)
 * is advisory: like the depth hint it can only affect speed (the per-tile sort walks a list of any
 * length in 3072-key shared-memory stages and currently ignores it). */
int dgr_forward(int P, int D, int M,
                const float* background, int W, int H,
                const float* means3D, const float* shs, const float* colors_precomp,
                const float* opacities, const float* scales, float scale_modifier,
                const float* rotations, const float* cov3D_precomp,
                const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                float tan_fovx, float tan_fovy, int prefiltered,
                float* out_color, int* radii,
                void* geom_ws, size_t geom_bytes,
                void* binning_ws, size_t binning_bytes, int64_t R_cap,
                void* img_ws, size_t img_bytes,
                int32_t* status, int32_t* status_host, void* status_event,
                float depth_hint_lo, float depth_hint_hi, int max_tile_hint, void* stream);

/* Backward: same contract as Rasterizer::backward (rasterizer.h:54-84).  All
 * nine gradient outputs are fully written (zeros for culled Gaussians), the
 * caller does NOT need to zero them (the reference requires zero-filled
 * tensors, rasterize_points.cu:151-159).
 *   dL_dpix[3,H,W] -> dL_dmean2D[P,3] (.xy written, .z = 0), dL_dconic[P,4] (may be NULL),
 *   dL_dopacity[P], dL_dcolor[P,3], dL_dmean3D[P,3], dL_dcov3D[P,6],
 *   dL_dsh[P,M,3] (may be NULL when shs == NULL), dL_dscale[P,3], dL_drot[P,4] */
int dgr_backward(int P, int D, int M,
                 const float* background, int W, int H,
                 const float* means3D, const float* shs, const float* colors_precomp,
                 const float* scales, float scale_modifier, const float* rotations,
                 const float* cov3D_precomp,
                 const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                 float tan_fovx, float tan_fovy, const int* radii,
                 void* geom_ws, void* binning_ws, int64_t R_cap, void* img_ws,
                 const float* dL_dpix,
                 float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                 float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                 float* dL_dscale, float* dL_drot,
                 void* stream);

/* ------------------------------------------------------------------------
 * Frame batches (data parallelism over training frames, SURVEY.md 8(e)): F cameras
 * rendered over ONE set of Gaussians, or -- what DG-Mesh's dynamic scenes need, where every
 * frame has its own time and therefore its own deformed means / scales / rotations
 * (dgmesh/train.py:157-178, gaussian_renderer/__init__.py:60-86) -- over per-frame slabs:
 * `per_frame` is a mask of DGR_PF_* bits; an input whose bit is set is [F,P,.] (frame f reads
 * slab f) and its gradient is [F,P,.], written per frame; inputs whose bit is clear are shared
 * [P,.] and their gradients are SUMMED over the frames.  No reference counterpart -- the reference renders
 * one frame per call (dgmesh/train.py:150-178); this is F x dgr_forward / dgr_backward
 * with (a) one host call, (b) consecutive frames enqueued on alternating internal side
 * streams forked from / joined to `stream`, so the short latency-bound kernels of frame
 * f+1 overlap the blend kernels of frame f, and (c) parameter gradients SUMMED over the
 * frames inside the kernels (what autograd's per-frame accumulation computes).
 *   per-frame inputs : viewmatrices[F,16], projmatrices[F,16], cam_poses[F,3] (device);
 *                      tan_fovx_host[F], tan_fovy_host[F] (HOST arrays)
 *   per-frame outputs: out_color[F,3,H,W], radii[F,P], status[F,DGR_STATUS_WORDS]
 *   workspaces       : frame f uses geom_ws + f*geom_stride, ... (each stride >= the size
 *                      reported by dgr_workspace_sizes, multiple of 128)
 * backward: dL_dpix[F,3,H,W] -> dL_dmean2D[F,P,3] per frame; dL_dopacity[P], dL_dcolor[P,3],
 * dL_dmean3D[P,3], dL_dcov3D[P,6], dL_dsh[P,M,3], dL_dscale[P,3], dL_drot[P,4] summed over
 * frames in frame order (fully written, no zero-fill needed).  With shs, dL_dcolor is [P,3] summed
 * over the frames whatever the mask, and may be NULL; without cov3D_precomp, dL_dcov3D may be NULL.
 * Both are intermediate gradients that only a caller inspecting them needs.  The per-Gaussian part
 * of the backward runs once for all frames after every frame's blend backward; at most 64 frames.
 * n_streams: 1..4 side streams.
 * ------------------------------------------------------------------------ */
#define DGR_PF_MEANS 1
#define DGR_PF_SCALES 2
#define DGR_PF_ROTS 4
#define DGR_PF_OPAC 8
#define DGR_PF_COLOR 16 /* shs or colors_precomp */
#define DGR_PF_COV 32
#define DGR_PF_ALL 63
int dgr_forward_batch(int F, int P, int D, int M,
                      const float* background, int W, int H,
                      const float* means3D, const float* shs, const float* colors_precomp,
                      const float* opacities, const float* scales, float scale_modifier,
                      const float* rotations, const float* cov3D_precomp, int per_frame,
                      const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                      const float* tan_fovx_host, const float* tan_fovy_host, int prefiltered,
                      float* out_color, int* radii,
                      void* geom_ws, size_t geom_stride,
                      void* binning_ws, size_t binning_stride, int64_t R_cap,
                      void* img_ws, size_t img_stride,
                      int32_t* status, int32_t* status_host, void* status_event,
                      float depth_hint_lo, float depth_hint_hi, int max_tile_hint, int n_streams, void* stream);

int dgr_backward_batch(int F, int P, int D, int M,
                       const float* background, int W, int H,
                       const float* means3D, const float* shs, const float* colors_precomp,
                       const float* scales, float scale_modifier, const float* rotations,
                       const float* cov3D_precomp, int per_frame,
                       const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                       const float* tan_fovx_host, const float* tan_fovy_host, const int* radii,
                       void* geom_ws, size_t geom_stride, void* binning_ws, size_t binning_stride,
                       int64_t R_cap, void* img_ws, size_t img_stride,
                       const float* dL_dpix,
                       float* dL_dmean2D, float* dL_dopacity, float* dL_dcolor,
                       float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                       float* dL_dscale, float* dL_drot,
                       int n_streams, void* stream);

/* ------------------------------------------------------------------------
 * Depth and alpha maps.  The four *_aux entry points take exactly the arguments of their
 * counterparts above plus, per pixel of the same front-to-back blend as the colour image
 * (same alpha_i, transmittance T_i, early stop and n_contrib):
 *   forward, after radii:    out_depth, out_alpha  [H,W] (batch: [F,H,W])
 *       depth = sum_i d_i alpha_i T_i   (d_i = view-space depth p_view.z; unnormalised, no
 *                                        background term: expected depth is depth / alpha)
 *       alpha = 1 - T_final              (T_final: the transmittance applied to the background)
 *   backward, after dL_dpix: dL_ddepth, dL_dalpha  [H,W] (batch: [F,H,W])
 * Each pointer may be NULL on its own; all NULL runs the colour-only kernels and is exactly the
 * counterpart above (which calls this path with NULLs).  A non-NULL dL_ddepth requires workspaces
 * written by a forward with a non-NULL out_depth: only that forward stores each Gaussian's depth
 * in the blend records the backward reads.  The depth gradient reaches dL_dmean3D through
 * p_view.z; summed over frames or per frame exactly like the rest of dL_dmean3D.
 * ------------------------------------------------------------------------ */
int dgr_forward_aux(int P, int D, int M,
                    const float* background, int W, int H,
                    const float* means3D, const float* shs, const float* colors_precomp,
                    const float* opacities, const float* scales, float scale_modifier,
                    const float* rotations, const float* cov3D_precomp,
                    const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                    float tan_fovx, float tan_fovy, int prefiltered,
                    float* out_color, int* radii, float* out_depth, float* out_alpha,
                    void* geom_ws, size_t geom_bytes,
                    void* binning_ws, size_t binning_bytes, int64_t R_cap,
                    void* img_ws, size_t img_bytes,
                    int32_t* status, int32_t* status_host, void* status_event,
                    float depth_hint_lo, float depth_hint_hi, int max_tile_hint, void* stream);

int dgr_backward_aux(int P, int D, int M,
                     const float* background, int W, int H,
                     const float* means3D, const float* shs, const float* colors_precomp,
                     const float* scales, float scale_modifier, const float* rotations,
                     const float* cov3D_precomp,
                     const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                     float tan_fovx, float tan_fovy, const int* radii,
                     void* geom_ws, void* binning_ws, int64_t R_cap, void* img_ws,
                     const float* dL_dpix, const float* dL_ddepth, const float* dL_dalpha,
                     float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                     float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                     float* dL_dscale, float* dL_drot,
                     void* stream);

int dgr_forward_batch_aux(int F, int P, int D, int M,
                          const float* background, int W, int H,
                          const float* means3D, const float* shs, const float* colors_precomp,
                          const float* opacities, const float* scales, float scale_modifier,
                          const float* rotations, const float* cov3D_precomp, int per_frame,
                          const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                          const float* tan_fovx_host, const float* tan_fovy_host, int prefiltered,
                          float* out_color, int* radii, float* out_depth, float* out_alpha,
                          void* geom_ws, size_t geom_stride,
                          void* binning_ws, size_t binning_stride, int64_t R_cap,
                          void* img_ws, size_t img_stride,
                          int32_t* status, int32_t* status_host, void* status_event,
                          float depth_hint_lo, float depth_hint_hi, int max_tile_hint, int n_streams,
                          void* stream);

int dgr_backward_batch_aux(int F, int P, int D, int M,
                           const float* background, int W, int H,
                           const float* means3D, const float* shs, const float* colors_precomp,
                           const float* scales, float scale_modifier, const float* rotations,
                           const float* cov3D_precomp, int per_frame,
                           const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                           const float* tan_fovx_host, const float* tan_fovy_host, const int* radii,
                           void* geom_ws, size_t geom_stride, void* binning_ws, size_t binning_stride,
                           int64_t R_cap, void* img_ws, size_t img_stride,
                           const float* dL_dpix, const float* dL_ddepth, const float* dL_dalpha,
                           float* dL_dmean2D, float* dL_dopacity, float* dL_dcolor,
                           float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                           float* dL_dscale, float* dL_drot,
                           int n_streams, void* stream);

/* ------------------------------------------------------------------------
 * Camera gradients.  dgr_backward_cam / dgr_backward_batch_cam take exactly the arguments of their
 * *_aux counterparts plus, after dL_drot:
 *   dL_dviewmatrix [F,16], dL_dprojmatrix [F,16], dL_dcampos [F,3]   (F = 1 for dgr_backward_cam)
 *       the gradients of the 16 stored floats of each frame's viewmatrix / projmatrix (the layout
 *       the kernels read, t_i = sum_k view[4k+i] mh_k) and of its campos.  view[3], view[7],
 *       view[11], view[15] and projmatrix[2], [6], [10], [14] do not enter the render: exactly 0.
 *       With precomputed colours dL_dcampos is exactly 0.  tan_fovx / tan_fovy are
 *       differentiated by dgr_backward_intr / dgr_backward_batch_intr (below).
 *   cam_ws, cam_ws_bytes: scratch of dgr_camera_grad_workspace_size(F, P) bytes (too small: an error
 *       return, DGM_E_WORKSPACE).  That size also covers the intrinsics output of the *_intr calls.
 * Each output pointer may be NULL on its own; all three NULL is the *_aux call.  No atomics and no
 * host synchronisation: for the same per-Gaussian moments (render backward output) the camera
 * gradients are bit-identical from call to call, and a batch gives those of F one-frame calls.
 * ------------------------------------------------------------------------ */
int dgr_camera_grad_workspace_size(int F, int P, size_t* bytes);

int dgr_backward_cam(int P, int D, int M,
                     const float* background, int W, int H,
                     const float* means3D, const float* shs, const float* colors_precomp,
                     const float* scales, float scale_modifier, const float* rotations,
                     const float* cov3D_precomp,
                     const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                     float tan_fovx, float tan_fovy, const int* radii,
                     void* geom_ws, void* binning_ws, int64_t R_cap, void* img_ws,
                     const float* dL_dpix, const float* dL_ddepth, const float* dL_dalpha,
                     float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                     float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                     float* dL_dscale, float* dL_drot,
                     float* dL_dviewmatrix, float* dL_dprojmatrix, float* dL_dcampos,
                     void* cam_ws, size_t cam_ws_bytes, void* stream);

int dgr_backward_batch_cam(int F, int P, int D, int M,
                           const float* background, int W, int H,
                           const float* means3D, const float* shs, const float* colors_precomp,
                           const float* scales, float scale_modifier, const float* rotations,
                           const float* cov3D_precomp, int per_frame,
                           const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                           const float* tan_fovx_host, const float* tan_fovy_host, const int* radii,
                           void* geom_ws, size_t geom_stride, void* binning_ws, size_t binning_stride,
                           int64_t R_cap, void* img_ws, size_t img_stride,
                           const float* dL_dpix, const float* dL_ddepth, const float* dL_dalpha,
                           float* dL_dmean2D, float* dL_dopacity, float* dL_dcolor,
                           float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                           float* dL_dscale, float* dL_drot,
                           float* dL_dviewmatrices, float* dL_dprojmatrices, float* dL_dcam_poses,
                           void* cam_ws, size_t cam_ws_bytes, int n_streams, void* stream);

/* ------------------------------------------------------------------------
 * Normal maps.  Over the same blend as the colour image (same alpha_i, T_i, early stop and
 * n_contrib), the [3,H,W] map N = sum_i n_i alpha_i T_i of caller-supplied per-Gaussian 3-vectors
 * n_i (used as given: no normalisation, no rotation; no background term: N / alpha is the
 * alpha-weighted mean normal).
 *   dgr_normal_workspace_size: bytes of one frame's normal workspace (the records' normal stream
 *       and a per-Gaussian gradient accumulator) for P Gaussians and instance capacity R_cap.
 *   dgr_forward_nrm / dgr_forward_batch_nrm: the arguments of the *_aux counterparts plus, after
 *       out_alpha:
 *         normals [P,3] (batch: [F,P,3] when normals_per_frame is non-zero; a flag of its own, the
 *             DGR_PF_* mask is unchanged),
 *         out_normal [3,H,W] (batch: [F,3,H,W]; NULL: exactly the *_aux call),
 *         nrm_ws, nrm_ws_bytes (batch: frame f's workspace at nrm_ws + f * nrm_ws_stride, the stride
 *             a multiple of 128 and at least the size; too small: DGM_E_WORKSPACE).
 *       A normal forward is also a depth forward (its records carry the depth; out_depth may be
 *       NULL) and clears the workspace's accumulator (asynchronously).
 *   dgr_backward_nrm / dgr_backward_batch_nrm: the arguments of the *_cam counterparts (the camera
 *       outputs and cam_ws may be NULL) plus, after cam_ws_bytes:
 *         dL_dnormal_map [3,H,W] (batch: [F,3,H,W]; NULL: exactly the *_cam call),
 *         (batch: normals_per_frame, as in the forward)
 *         dL_dnormals [P,3], or [F,P,3] with normals_per_frame (the shared normals' gradient is the
 *             sum over the frames in frame order); may be NULL,
 *         nrm_ws (batch: nrm_ws, nrm_ws_stride): the workspaces the forward wrote.
 *       The accumulators are zero again when the call's work completes, with or without dL_dnormals.
 *       Gaussians in no blend record get exact zeros.  The normal loss reaches every other input
 *       and the camera gradients through dL/dalpha_i.
 * No call allocates or synchronises.
 * ------------------------------------------------------------------------ */
int dgr_normal_workspace_size(int P, int64_t R_cap, size_t* bytes);

int dgr_forward_nrm(int P, int D, int M,
                    const float* background, int W, int H,
                    const float* means3D, const float* shs, const float* colors_precomp,
                    const float* opacities, const float* scales, float scale_modifier,
                    const float* rotations, const float* cov3D_precomp,
                    const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                    float tan_fovx, float tan_fovy, int prefiltered,
                    float* out_color, int* radii, float* out_depth, float* out_alpha,
                    const float* normals, float* out_normal, void* nrm_ws, size_t nrm_ws_bytes,
                    void* geom_ws, size_t geom_bytes,
                    void* binning_ws, size_t binning_bytes, int64_t R_cap,
                    void* img_ws, size_t img_bytes,
                    int32_t* status, int32_t* status_host, void* status_event,
                    float depth_hint_lo, float depth_hint_hi, int max_tile_hint, void* stream);

int dgr_backward_nrm(int P, int D, int M,
                     const float* background, int W, int H,
                     const float* means3D, const float* shs, const float* colors_precomp,
                     const float* scales, float scale_modifier, const float* rotations,
                     const float* cov3D_precomp,
                     const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                     float tan_fovx, float tan_fovy, const int* radii,
                     void* geom_ws, void* binning_ws, int64_t R_cap, void* img_ws,
                     const float* dL_dpix, const float* dL_ddepth, const float* dL_dalpha,
                     float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                     float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                     float* dL_dscale, float* dL_drot,
                     float* dL_dviewmatrix, float* dL_dprojmatrix, float* dL_dcampos,
                     void* cam_ws, size_t cam_ws_bytes,
                     const float* dL_dnormal_map, float* dL_dnormals, void* nrm_ws, void* stream);

int dgr_forward_batch_nrm(int F, int P, int D, int M,
                          const float* background, int W, int H,
                          const float* means3D, const float* shs, const float* colors_precomp,
                          const float* opacities, const float* scales, float scale_modifier,
                          const float* rotations, const float* cov3D_precomp, int per_frame,
                          const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                          const float* tan_fovx_host, const float* tan_fovy_host, int prefiltered,
                          float* out_color, int* radii, float* out_depth, float* out_alpha,
                          const float* normals, int normals_per_frame, float* out_normal,
                          void* nrm_ws, size_t nrm_ws_stride,
                          void* geom_ws, size_t geom_stride,
                          void* binning_ws, size_t binning_stride, int64_t R_cap,
                          void* img_ws, size_t img_stride,
                          int32_t* status, int32_t* status_host, void* status_event,
                          float depth_hint_lo, float depth_hint_hi, int max_tile_hint, int n_streams,
                          void* stream);

int dgr_backward_batch_nrm(int F, int P, int D, int M,
                           const float* background, int W, int H,
                           const float* means3D, const float* shs, const float* colors_precomp,
                           const float* scales, float scale_modifier, const float* rotations,
                           const float* cov3D_precomp, int per_frame,
                           const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                           const float* tan_fovx_host, const float* tan_fovy_host, const int* radii,
                           void* geom_ws, size_t geom_stride, void* binning_ws, size_t binning_stride,
                           int64_t R_cap, void* img_ws, size_t img_stride,
                           const float* dL_dpix, const float* dL_ddepth, const float* dL_dalpha,
                           float* dL_dmean2D, float* dL_dopacity, float* dL_dcolor,
                           float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                           float* dL_dscale, float* dL_drot,
                           float* dL_dviewmatrices, float* dL_dprojmatrices, float* dL_dcam_poses,
                           void* cam_ws, size_t cam_ws_bytes,
                           const float* dL_dnormal_maps, int normals_per_frame, float* dL_dnormals,
                           void* nrm_ws, size_t nrm_ws_stride, int n_streams, void* stream);

/* ------------------------------------------------------------------------
 * Median-depth and depth-distortion maps (2DGS).  Over the same blend as the colour image
 * (same alpha_i, T_i, early stop and n_contrib), with w_i = alpha_i T_i, d_i = p_view.z and the
 * normalised depth m_i = far / (far - near) (1 - near / d_i):
 *   median     [H,W]  d_i of the last blended record whose T before blending is > 0.5 (a pixel
 *                     whose T never reaches 0.5: its last contributor; nothing blended: 0)
 *   distortion [H,W]  1/2 sum_ij w_i w_j (m_i - m_j)^2, computed front to back as
 *                     sum_i w_i (m_i^2 A_i + M2_i - 2 m_i M1_i), A_i, M1_i, M2_i the sums of w_j,
 *                     w_j m_j, w_j m_j^2 over j < i
 *   dgr_surface_workspace_size: bytes of one frame's surface workspace for a W x H image (the
 *       median record's Gaussian id and the totals M1, M2 per pixel, about 12 B per pixel).
 *   dgr_forward_surf / dgr_forward_batch_surf: the arguments of the *_nrm counterparts plus, after
 *       nrm_ws_bytes (batch: nrm_ws_stride):
 *         near, far (0 < near < far; 2DGS uses 0.2 and 100),
 *         out_median, out_distortion [H,W] (batch: [F,H,W]),
 *         surf_ws, surf_ws_bytes (batch: frame f's workspace at surf_ws + f * surf_ws_stride, the stride
 *             a multiple of 128 and at least the size; too small: DGM_E_WORKSPACE).
 *       A surface forward is also a depth forward (out_depth may be NULL).
 *   dgr_backward_surf / dgr_backward_batch_surf: the arguments of the *_nrm counterparts (the normal
 *       pointers may be NULL) plus, after nrm_ws (batch: nrm_ws_stride):
 *         near, far (as in the forward),
 *         dL_dmedian, dL_ddistortion [H,W] (batch: [F,H,W]),
 *         surf_ws (batch: surf_ws, surf_ws_stride): the workspaces the forward wrote.
 *       dL/dmedian reaches the depth of each pixel's median record only (the median is piecewise
 *       constant in alpha); the distortion loss reaches every input through dL/dalpha_i and the
 *       depths.  Both reach dL_dmean3D (per frame or summed over the frames like the rest of it) and,
 *       with the camera outputs, the camera gradients.
 * Each surface pointer may be NULL on its own; all NULL is exactly the *_nrm call (near, far and the
 * surface workspace are then ignored).  Bad near / far: DGM_E_BADARG before any device work.
 * No call allocates or synchronises.
 * ------------------------------------------------------------------------ */
int dgr_surface_workspace_size(int W, int H, size_t* bytes);

int dgr_forward_surf(int P, int D, int M,
                     const float* background, int W, int H,
                     const float* means3D, const float* shs, const float* colors_precomp,
                     const float* opacities, const float* scales, float scale_modifier,
                     const float* rotations, const float* cov3D_precomp,
                     const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                     float tan_fovx, float tan_fovy, int prefiltered,
                     float* out_color, int* radii, float* out_depth, float* out_alpha,
                     const float* normals, float* out_normal, void* nrm_ws, size_t nrm_ws_bytes,
                     float near, float far, float* out_median, float* out_distortion,
                     void* surf_ws, size_t surf_ws_bytes,
                     void* geom_ws, size_t geom_bytes,
                     void* binning_ws, size_t binning_bytes, int64_t R_cap,
                     void* img_ws, size_t img_bytes,
                     int32_t* status, int32_t* status_host, void* status_event,
                     float depth_hint_lo, float depth_hint_hi, int max_tile_hint, void* stream);

int dgr_backward_surf(int P, int D, int M,
                      const float* background, int W, int H,
                      const float* means3D, const float* shs, const float* colors_precomp,
                      const float* scales, float scale_modifier, const float* rotations,
                      const float* cov3D_precomp,
                      const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                      float tan_fovx, float tan_fovy, const int* radii,
                      void* geom_ws, void* binning_ws, int64_t R_cap, void* img_ws,
                      const float* dL_dpix, const float* dL_ddepth, const float* dL_dalpha,
                      float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                      float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                      float* dL_dscale, float* dL_drot,
                      float* dL_dviewmatrix, float* dL_dprojmatrix, float* dL_dcampos,
                      void* cam_ws, size_t cam_ws_bytes,
                      const float* dL_dnormal_map, float* dL_dnormals, void* nrm_ws,
                      float near, float far, const float* dL_dmedian, const float* dL_ddistortion,
                      void* surf_ws, void* stream);

int dgr_forward_batch_surf(int F, int P, int D, int M,
                           const float* background, int W, int H,
                           const float* means3D, const float* shs, const float* colors_precomp,
                           const float* opacities, const float* scales, float scale_modifier,
                           const float* rotations, const float* cov3D_precomp, int per_frame,
                           const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                           const float* tan_fovx_host, const float* tan_fovy_host, int prefiltered,
                           float* out_color, int* radii, float* out_depth, float* out_alpha,
                           const float* normals, int normals_per_frame, float* out_normal,
                           void* nrm_ws, size_t nrm_ws_stride,
                           float near, float far, float* out_median, float* out_distortion,
                           void* surf_ws, size_t surf_ws_stride,
                           void* geom_ws, size_t geom_stride,
                           void* binning_ws, size_t binning_stride, int64_t R_cap,
                           void* img_ws, size_t img_stride,
                           int32_t* status, int32_t* status_host, void* status_event,
                           float depth_hint_lo, float depth_hint_hi, int max_tile_hint, int n_streams,
                           void* stream);

int dgr_backward_batch_surf(int F, int P, int D, int M,
                            const float* background, int W, int H,
                            const float* means3D, const float* shs, const float* colors_precomp,
                            const float* scales, float scale_modifier, const float* rotations,
                            const float* cov3D_precomp, int per_frame,
                            const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                            const float* tan_fovx_host, const float* tan_fovy_host, const int* radii,
                            void* geom_ws, size_t geom_stride, void* binning_ws, size_t binning_stride,
                            int64_t R_cap, void* img_ws, size_t img_stride,
                            const float* dL_dpix, const float* dL_ddepth, const float* dL_dalpha,
                            float* dL_dmean2D, float* dL_dopacity, float* dL_dcolor,
                            float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                            float* dL_dscale, float* dL_drot,
                            float* dL_dviewmatrices, float* dL_dprojmatrices, float* dL_dcam_poses,
                            void* cam_ws, size_t cam_ws_bytes,
                            const float* dL_dnormal_maps, int normals_per_frame, float* dL_dnormals,
                            void* nrm_ws, size_t nrm_ws_stride,
                            float near, float far, const float* dL_dmedian, const float* dL_ddistortion,
                            void* surf_ws, size_t surf_ws_stride, int n_streams, void* stream);

/* ------------------------------------------------------------------------
 * Absolute screen-space gradients (AbsGS, "homodirectional" gradient; gsplat's absgrad).  For Gaussian i
 * and pixel p let g_ip be the summand the blend backward adds to dL/dmean2D for that pair
 * (dL/dG dG/d(delx, dely) (W/2, H/2), the reference's backward.cu:531-554), from every loss the call
 * carries: colour, depth, alpha, normal and distortion (through dL/dalpha).  The median depth's
 * gradient reaches the depth only and adds nothing.  The statistic is
 *   dL_dmean2D_abs[i] = (sum_p |g_ip.x|, sum_p |g_ip.y|, 0)
 * which, unlike dL/dmean2D, does not cancel over pixels that pull a Gaussian in opposite directions.
 *   dgr_backward_abs / dgr_backward_batch_abs: the arguments of dgr_backward_surf /
 *       dgr_backward_batch_surf plus, after surf_ws (batch: surf_ws_stride):
 *         dL_dmean2D_abs [P,3] (batch: [F,P,3], frame f's statistic in slab f).
 *       The output is fully written (zeroed on the call's stream, then added to): no zero-fill needed.
 *       A Gaussian without a blend record gets exact zeros.  Every other output is that of the *_surf
 *       call.  It needs nothing but what any forward of this library leaves behind.
 * dL_dmean2D_abs NULL is exactly the *_surf call.  The argument checks are those of the *_surf call,
 * before any device work.  No call allocates or synchronises.
 * ------------------------------------------------------------------------ */
int dgr_backward_abs(int P, int D, int M,
                     const float* background, int W, int H,
                     const float* means3D, const float* shs, const float* colors_precomp,
                     const float* scales, float scale_modifier, const float* rotations,
                     const float* cov3D_precomp,
                     const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                     float tan_fovx, float tan_fovy, const int* radii,
                     void* geom_ws, void* binning_ws, int64_t R_cap, void* img_ws,
                     const float* dL_dpix, const float* dL_ddepth, const float* dL_dalpha,
                     float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                     float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                     float* dL_dscale, float* dL_drot,
                     float* dL_dviewmatrix, float* dL_dprojmatrix, float* dL_dcampos,
                     void* cam_ws, size_t cam_ws_bytes,
                     const float* dL_dnormal_map, float* dL_dnormals, void* nrm_ws,
                     float near, float far, const float* dL_dmedian, const float* dL_ddistortion,
                     void* surf_ws, float* dL_dmean2D_abs, void* stream);

int dgr_backward_batch_abs(int F, int P, int D, int M,
                           const float* background, int W, int H,
                           const float* means3D, const float* shs, const float* colors_precomp,
                           const float* scales, float scale_modifier, const float* rotations,
                           const float* cov3D_precomp, int per_frame,
                           const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                           const float* tan_fovx_host, const float* tan_fovy_host, const int* radii,
                           void* geom_ws, size_t geom_stride, void* binning_ws, size_t binning_stride,
                           int64_t R_cap, void* img_ws, size_t img_stride,
                           const float* dL_dpix, const float* dL_ddepth, const float* dL_dalpha,
                           float* dL_dmean2D, float* dL_dopacity, float* dL_dcolor,
                           float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                           float* dL_dscale, float* dL_drot,
                           float* dL_dviewmatrices, float* dL_dprojmatrices, float* dL_dcam_poses,
                           void* cam_ws, size_t cam_ws_bytes,
                           const float* dL_dnormal_maps, int normals_per_frame, float* dL_dnormals,
                           void* nrm_ws, size_t nrm_ws_stride,
                           float near, float far, const float* dL_dmedian, const float* dL_ddistortion,
                           void* surf_ws, size_t surf_ws_stride, float* dL_dmean2D_abs, int n_streams,
                           void* stream);

/* ------------------------------------------------------------------------
 * Focal-length (intrinsics) gradients.  dgr_backward_intr / dgr_backward_batch_intr take the arguments of
 * dgr_backward_abs / dgr_backward_batch_abs plus, after dL_dmean2D_abs:
 *   dL_dtanfov [F,2] (F = 1 for dgr_backward_intr): (dL/dtan_fovx, dL/dtan_fovy) of each frame through
 *       the EWA covariance, i.e. through everything the kernels take from tan_fovx / tan_fovy: the
 *       focal lengths f = W / (2 tan_fovx), H / (2 tan_fovy) of the Jacobian J and the 1.3 tan(fov/2)
 *       clamp of the view-space position.  The projection matrix (which places the 2D means) is an
 *       input of its own: its path is dL_dprojmatrix.  A camera whose projmatrix and tan(fov/2) both
 *       follow the focal length gets the total focal gradient as the sum of the two.
 *       The pose outputs may be NULL; cam_ws must then still be given (dgr_camera_grad_workspace_size
 *       bytes; too small: DGM_E_WORKSPACE).  P = 0: exact zeros.  Summed without atomics in a fixed
 *       order: bit-identical from call to call, a batch gives those of F one-frame calls, and every
 *       other output is bit-identical to the *_abs call's.
 * dL_dtanfov NULL is exactly the *_abs call.  No call allocates or synchronises.
 * ------------------------------------------------------------------------ */
int dgr_backward_intr(int P, int D, int M,
                      const float* background, int W, int H,
                      const float* means3D, const float* shs, const float* colors_precomp,
                      const float* scales, float scale_modifier, const float* rotations,
                      const float* cov3D_precomp,
                      const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                      float tan_fovx, float tan_fovy, const int* radii,
                      void* geom_ws, void* binning_ws, int64_t R_cap, void* img_ws,
                      const float* dL_dpix, const float* dL_ddepth, const float* dL_dalpha,
                      float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                      float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                      float* dL_dscale, float* dL_drot,
                      float* dL_dviewmatrix, float* dL_dprojmatrix, float* dL_dcampos,
                      void* cam_ws, size_t cam_ws_bytes,
                      const float* dL_dnormal_map, float* dL_dnormals, void* nrm_ws,
                      float near, float far, const float* dL_dmedian, const float* dL_ddistortion,
                      void* surf_ws, float* dL_dmean2D_abs, float* dL_dtanfov, void* stream);

int dgr_backward_batch_intr(int F, int P, int D, int M,
                            const float* background, int W, int H,
                            const float* means3D, const float* shs, const float* colors_precomp,
                            const float* scales, float scale_modifier, const float* rotations,
                            const float* cov3D_precomp, int per_frame,
                            const float* viewmatrices, const float* projmatrices, const float* cam_poses,
                            const float* tan_fovx_host, const float* tan_fovy_host, const int* radii,
                            void* geom_ws, size_t geom_stride, void* binning_ws, size_t binning_stride,
                            int64_t R_cap, void* img_ws, size_t img_stride,
                            const float* dL_dpix, const float* dL_ddepth, const float* dL_dalpha,
                            float* dL_dmean2D, float* dL_dopacity, float* dL_dcolor,
                            float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                            float* dL_dscale, float* dL_drot,
                            float* dL_dviewmatrices, float* dL_dprojmatrices, float* dL_dcam_poses,
                            void* cam_ws, size_t cam_ws_bytes,
                            const float* dL_dnormal_maps, int normals_per_frame, float* dL_dnormals,
                            void* nrm_ws, size_t nrm_ws_stride,
                            float near, float far, const float* dL_dmedian, const float* dL_ddistortion,
                            void* surf_ws, size_t surf_ws_stride, float* dL_dmean2D_abs, float* dL_dtanfov,
                            int n_streams, void* stream);

/* ------------------------------------------------------------------------
 * Feature maps.  Over the same blend as the colour image of an EARLIER forward (same alpha_i, T_i, 1/255 skip,
 * early stop and n_contrib), the [C,H,W] map F_c = sum_i f_{i,c} alpha_i T_i of caller-chosen per-Gaussian
 * vectors f [P,C], 1 <= C <= 64 (no background term, no normalisation: F / alpha is the alpha-weighted mean).
 * The calls are a pass over the workspaces that forward left behind and change none of them except grad_acc:
 *   any forward of this library -- dgr_forward, *_aux, *_nrm, *_surf, or their batch forms -- whose
 *   geom / binning / img workspaces (frame f's at geom_ws + f * geom_stride, ...; F = 1: the strides are
 *   ignored) are passed unchanged.  An overflowed forward must have been re-run before.
 *   dgr_feature_workspace_size: bytes of the feature workspace of F frames (a per-Gaussian accumulator of
 *       dL/dfeatures per frame; it does not depend on R_cap).
 *   dgr_features_fwd: features [P,C] (or [F,P,C] when features_per_frame is non-zero) -> out_map [F,C,H,W];
 *       clears the feature workspace's accumulators (asynchronously).
 *   dgr_features_bwd: the same features and workspaces, the forward's map [F,C,H,W] and its upstream
 *       gradient dL_dmap [F,C,H,W] -> dL_dfeatures [P,C] (the sum over the frames in frame order), or
 *       [F,P,C] with features_per_frame; may be NULL.  It adds the feature loss's share of dL/dmean2D,
 *       dL/dconic and dL/dopacity to the forward's per-Gaussian accumulators, which only the backward of the
 *       same forward reads: enqueue dgr_features_bwd BEFORE the matching dgr_backward* call on the same
 *       stream, and always follow it with that call (with zero dL_dpix if the loss uses no other map).  That
 *       call carries the feature loss to every Gaussian input and, with its camera outputs, to the cameras.
 *       The feature workspace's accumulators are zero again when the call's work completes.
 * Bad C, F outside 1..64, a NULL required pointer or a stride below the forward's workspace size:
 * DGM_E_BADARG; a feature workspace below the query: DGM_E_WORKSPACE; both before any device work.
 * No call allocates or synchronises.
 * ------------------------------------------------------------------------ */
int dgr_feature_workspace_size(int P, int C, int F, size_t* bytes);

int dgr_features_fwd(int F, int P, int C, int W, int H, const float* features, int features_per_frame,
                     void* geom_ws, size_t geom_stride, void* binning_ws, size_t binning_stride, int64_t R_cap,
                     void* img_ws, size_t img_stride, float* out_map, void* feat_ws, size_t feat_ws_bytes,
                     void* stream);

int dgr_features_bwd(int F, int P, int C, int W, int H, const float* features, int features_per_frame,
                     void* geom_ws, size_t geom_stride, void* binning_ws, size_t binning_stride, int64_t R_cap,
                     void* img_ws, size_t img_stride, const float* map, const float* dL_dmap,
                     float* dL_dfeatures, void* feat_ws, size_t feat_ws_bytes, void* stream);

/* ------------------------------------------------------------------------
 * Planar depth (RaDe-GS / PGSR unbiased depth).  Each Gaussian i of frame f gets a depth plane in screen space,
 * with V the world-to-camera rotation (rows (view[0], view[4], view[8]), (view[1], view[5], view[9]),
 * (view[2], view[6], view[10])), t = V m + (view[12], view[13], view[14]) formed as preprocess forms it,
 * fx = W / (2 tan_fovx), fy = H / (2 tan_fovy), r = (tx_c / t_z, ty_c / t_z, 1) with the EWA clamp (1.3 tan_fov),
 * A = V adj(Sigma) V^T (Sigma the rasterizer's 3D covariance: (S R)^T (S R) from the un-normalised quaternion with
 * scale_modifier, or cov3D_precomp), a = A r, q = r^T a:
 *   slope   g = -t_z (a_x / fx, a_y / fy) / q (depth units per pixel), scaled by PLANE_MAX_TILT / tau when
 *           tau = |(a_x, a_y)| / q > PLANE_MAX_TILT
 *   normal  n = -a / |a| (camera space, facing the camera: (0, 0, -1) for a plane facing it)
 *   planes[f,i] = (t_z, g_u, g_v), normals[f,i] = n;  q <= 0: g = 0, n = 0;  t_z <= 0.2: (t_z, 0, 0), n = 0;
 *   no gradient flows in either case.
 * The depth of record i at pixel centre p is d_i(p) = t_z + g . (p - mu2D_i), mu2D_i its screen mean.
 *   dgr_gaussian_planes_fwd / _bwd: means3D, and scales + rotations or cov3D_precomp ([P,.], or [F,P,.] when
 *       the input's DGR_PF_* bit is set in per_frame), viewmatrices [F,16] (device), tan_fovx / tan_fovy [F]
 *       (host) -> planes, normals [F,P,3]; the backward takes dL_dplanes, dL_dnormals [F,P,3] (either may be
 *       NULL) -> dL_dmeans3D, dL_dscales, dL_drotations or dL_dcov3D_precomp (shared inputs: the sum over the
 *       frames in frame order; per-frame ones per frame; NULL: not written).  No camera gradient is formed.
 *   dgr_planar_workspace_size: bytes of the planar workspace of F frames.
 *   dgr_planar_fwd: over the same blend as the colour image of an EARLIER forward (as dgr_features_fwd), planes
 *       [F,P,3] -> planar_depth = sum_i d_i(p) alpha_i T_i and planar_median = d_i(p) of the last record blended
 *       while T > 0.5 (0 where nothing is blended), each [F,1,H,W]; clears the workspace's accumulators.
 *   dgr_planar_bwd: the same planes and workspaces, the forward's planar_depth and the upstream gradients of the
 *       two maps (either may be NULL) -> dL_dplanes [F,P,3] (may be NULL).  Adds the maps' share of dL/dmean2D,
 *       dL/dconic and dL/dopacity to the forward's accumulators: enqueue it BEFORE the matching dgr_backward*
 *       call and always follow it with that call, as dgr_features_bwd.
 * Bad sizes, F outside 1..64, NULL required pointers or short strides: DGM_E_BADARG; a planar workspace below the
 * query: DGM_E_WORKSPACE; both before any device work.  No call allocates or synchronises.
 * ------------------------------------------------------------------------ */
#define PLANE_MAX_TILT 10.0f
int dgr_gaussian_planes_fwd(int F, int P, int W, int H, const float* means3D, const float* scales,
                            float scale_modifier, const float* rotations, const float* cov3D_precomp, int per_frame,
                            const float* viewmatrices, const float* tan_fovx_host, const float* tan_fovy_host,
                            float* planes, float* normals, void* stream);

int dgr_gaussian_planes_bwd(int F, int P, int W, int H, const float* means3D, const float* scales,
                            float scale_modifier, const float* rotations, const float* cov3D_precomp, int per_frame,
                            const float* viewmatrices, const float* tan_fovx_host, const float* tan_fovy_host,
                            const float* dL_dplanes, const float* dL_dnormals, float* dL_dmeans3D,
                            float* dL_dscales, float* dL_drotations, float* dL_dcov3D_precomp, void* stream);

int dgr_planar_workspace_size(int P, int W, int H, int F, size_t* bytes);

int dgr_planar_fwd(int F, int P, int W, int H, const float* planes, void* geom_ws, size_t geom_stride,
                   void* binning_ws, size_t binning_stride, int64_t R_cap, void* img_ws, size_t img_stride,
                   float* planar_depth, float* planar_median, void* planar_ws, size_t planar_ws_bytes, void* stream);

int dgr_planar_bwd(int F, int P, int W, int H, const float* planes, void* geom_ws, size_t geom_stride,
                   void* binning_ws, size_t binning_stride, int64_t R_cap, void* img_ws, size_t img_stride,
                   const float* planar_depth, const float* dL_dplanar_depth, const float* dL_dplanar_median,
                   float* dL_dplanes, void* planar_ws, size_t planar_ws_bytes, void* stream);

/* ------------------------------------------------------------------------
 * Blend-weight statistics.  Over the same blend as the colour image of an EARLIER forward (same alpha_i, T_i, 1/255
 * skip and n_contrib), per frame f and Gaussian i, with w_ip = alpha_ip T_ip (T_ip the transmittance before record
 * i is blended at pixel p) and e_p an optional per-pixel weight (1 when pixel_weights is NULL):
 *   out_sum[f,i] = sum_p e_p w_ip            out_max[f,i] = max(0, max_p e_p w_ip)
 * both [F,P] float32 and exactly 0 for a Gaussian no pixel blends (pruning / importance statistics; a negative
 * weight enters the sum as given and contributes 0 to the max).  pixel_weights is NULL, [H,W] shared by the frames,
 * or [F,H,W] when weights_per_frame is non-zero.  The call is a pass over the binning and img workspaces of any
 * forward of this library -- dgr_forward, *_aux, *_nrm, *_surf, or their batch forms -- passed unchanged (frame
 * f's at binning_ws + f * binning_stride, ...; F = 1: the strides are ignored).  An overflowed forward must have
 * been re-run before.  It zeroes both outputs on the stream itself, reads the workspaces and writes nothing else.
 * out_max is the same from run to run bit for bit; out_sum's per-Gaussian total over tiles is a float atomic sum.
 * Bad F, P, W or H, a NULL workspace or output, or a stride below the forward's workspace size (or not a multiple
 * of 128): DGM_E_BADARG before any device work.  It does not allocate or synchronise.
 * ------------------------------------------------------------------------ */
int dgr_blend_stats(int F, int P, int W, int H, void* binning_ws, size_t binning_stride, int64_t R_cap,
                    void* img_ws, size_t img_stride, const float* pixel_weights, int weights_per_frame,
                    float* out_sum, float* out_max, void* stream);

/* ------------------------------------------------------------------------
 * Depth normals: the normals of the surface the rendered depth describes (2DGS's depth_to_normal), for
 * the depth-normal consistency loss against the rendered normal map.  No reference counterpart.
 * Per frame f (maps [F,H,W], frame f at offset f*H*W; r = depth_ratio in [0, 1]):
 *   surface depth s = (1 - r) E + r M, E = depth / alpha where alpha > 0 and 0 elsewhere, M = median;
 *   depth and alpha are not read when r == 1 (may be NULL), median is not read when r == 0 (may be NULL);
 *   the rasterizer's pixel rays: X/Z = ax u + bx, Y/Z = ay v + by at pixel centre (u, v), with
 *   coefs_host [F,4] = (ax, bx, ay, by) per frame (HOST memory, read during the call; for a centred pinhole
 *   ax = 2 tanfovx / W, bx = (1/W - 1) tanfovx, likewise y with H);
 *   P(u,v) = s (ax u + bx, ay v + by, 1) and, for 0 < u < W-1, 0 < v < H-1,
 *   normal = normalize(sign(ax ay) cross(P(u,v+1) - P(u,v-1), P(u+1,v) - P(u-1,v))) -- camera space,
 *   (0, 0, -1) for a plane facing the camera; 0 on the image border and where the cross product is exactly 0.
 *   dgr_depth_normal_fwd: -> out_normal [F,3,H,W].
 *   dgr_depth_normal_bwd: dL_dnormal [F,3,H,W] -> dL_ddepth = (1 - r) / alpha dL/ds and
 *       dL_dalpha = -(1 - r) depth / alpha^2 dL/ds (both 0 where alpha == 0), dL_dmedian = r dL/ds, each
 *       [F,H,W] and written in full.  A gradient may be NULL when not wanted, and must be NULL for a map r does
 *       not read.  No atomics: the result is the same bit for bit from run to run.
 * Bad F, W, H, r outside [0, 1] or a NULL required pointer: DGM_E_BADARG before any device work.  Neither call
 * allocates or synchronises.
 * ------------------------------------------------------------------------ */
int dgr_depth_normal_fwd(int F, int W, int H, float depth_ratio, const float* depth, const float* alpha,
                         const float* median, const float* coefs_host, float* out_normal, void* stream);

int dgr_depth_normal_bwd(int F, int W, int H, float depth_ratio, const float* depth, const float* alpha,
                         const float* median, const float* coefs_host, const float* dL_dnormal, float* dL_ddepth,
                         float* dL_dalpha, float* dL_dmedian, void* stream);

/* Frustum test, Rasterizer::markVisible (rasterizer.h:22-27,
 * rasterizer_impl.cu:54-66,141-153): present[P] (uint8 bool). */
int dgr_mark_visible(int P, const float* means3D, const float* viewmatrix,
                     const float* projmatrix, uint8_t* present, void* stream);

/* Introspection for parity tests: export the reference-visible intermediate
 * state of the last forward from the private workspaces into caller arrays
 * laid out as in the reference's GeometryState / BinningState / ImageState
 * (rasterizer_impl.h:30-63).  Any output pointer may be NULL.
 *   depths[P], means2D[P,2], cov3D[P,6], conic_opacity[P,4], rgb[P,3],
 *   tiles_touched[P] (u32), clamped[P,3] (u8),
 *   point_list_keys[R] (u64: tile<<32 | depth bits), point_list[R] (u32),
 *   ranges[T,2] (u32), final_T[H*W], n_contrib[H*W] (u32)               */
int dgr_export_state(int P, int W, int H, int64_t R_cap,
                     const void* geom_ws, const void* binning_ws, const void* img_ws,
                     float* depths, float* means2D, float* cov3D, float* conic_opacity,
                     float* rgb, uint32_t* tiles_touched, uint8_t* clamped,
                     uint64_t* point_list_keys, uint32_t* point_list,
                     uint32_t* ranges, float* final_T, uint32_t* n_contrib,
                     void* stream);

/* ------------------------------------------------------------------------
 * simple-knn: mean squared distance to the 3 nearest neighbours of every point.
 * replaces SimpleKNN::knn / distCUDA2 (dgmesh/submodules/simple-knn/simple_knn.cu:185-221,
 * spatial.cu:15-26, ext.cpp:15-17).  points[P,3] fp32 -> mean_dist2[P] fp32.
 * Unlike the reference (two blocking D2H copies, simple_knn.cu:196-200) nothing
 * synchronises with the host.
 * ------------------------------------------------------------------------ */
int dgk_workspace_size(int P, size_t* bytes);
int dgk_dist2(int P, const float* points, float* mean_dist2,
              void* ws, size_t ws_bytes, void* stream);

/* Cross-set nearest neighbour, K = 1: for every query the squared distance to, and the index of, its
 * nearest reference point (ties: lowest index).  Replaces `pytorch3d.ops.knn_points(p1, p2, K=1)` as
 * anchor_mesh calls it (dgmesh/scene/gaussian_model_dpsr_dynamic_anchor.py:761): queries[Q,3],
 * refs[R,3] fp32 -> dist2[Q] fp32, index[Q] int64.  R >= 1. */
int dgk_nearest(int Q, const float* queries, int R, const float* refs,
                float* dist2, int64_t* index, void* stream);

/* ------------------------------------------------------------------------
 * DPSR -- differentiable Poisson surface reconstruction on a G^3 periodic grid.
 * replaces DPSR.forward (dgmesh/nvdiffrast_utils/dpsr.py:28-70) with point_rasterize /
 * grid_interp / spec_gaussian_filter / fftfreqs (dgmesh/nvdiffrast_utils/dpsr_utils.py:25-197)
 * and the autograd graph PyTorch builds through them.  One item here; the _batch calls below take B.
 *   V[N,3] in (0,1), Nrm[N,3]  ->  out[G,G,G]
 *   mode 0: out = phi exactly as DPSR.forward returns it (shifted, scaled by -0.5/|phi[0,0,0]|)
 *   mode 1: out = psr * sign - thres[0] as mesh_renderer forms it (dgmesh/utils/renderer.py:
 *           163-168) without the reference's host read of psr[0,0,0,0]; thres is a device scalar
 * The plan owns the cuFFT handles (the one-time setup the reference leaves to torch.fft's plan
 * cache); all device memory, including the FFT work area, is the caller's workspace, which must
 * be passed unchanged from dgp_forward to dgp_backward (it holds the field for the backward pass).
 * backward: dL_dout[G,G,G] -> dV[N,3], dN[N,3], dthres[1] (mode 1; may be NULL).
 * ------------------------------------------------------------------------ */
int dgp_plan_create(int G, void** plan, size_t* ws_bytes);
int dgp_plan_destroy(void* plan);
int dgp_forward(void* plan, int N, double sig, const float* V, const float* Nrm, int mode,
                const float* thres, float* out, void* ws, size_t ws_bytes, void* stream);
int dgp_backward(void* plan, int N, const float* V, const float* Nrm, int mode,
                 const float* dL_dout, float* dV, float* dN, float* dthres,
                 void* ws, size_t ws_bytes, void* stream);
/* DPSR over a batch of B point sets (the reference's DPSR.forward(V[b,nv,3], N[b,nv,3])), 1 <= B <= 64; B out
 * of range, a NULL pointer or a short workspace is refused on the host before any device work.
 *   V[B,N,3], Nrm[B,N,3]  ->  out[B,G,G,G]; every item is normalised on its own (its own offset and its own
 *   phi[k,0,0,0] scale, or in mode 1 its own sign from psr[k,0,0,0]); item k equals the single call on item k.
 *   All items share thres[0] (mode 1).
 * dgp_batch_workspace_size: bytes of a B-item workspace for the plan's G.  Only each item's field (4 G^3 bytes)
 * and a few scalars outlive the forward; the spectra, the normals grid and the FFT work area are scratch that
 * the items reuse one after another, so the size is the single-item size plus 4 G^3 (B - 1) bytes (at G = 288:
 * 0.86 GB + 95.6 MB per further item).  B = 1 gives dgp_plan_create's ws_bytes.  dgp_forward_batch and
 * dgp_backward_batch must be given the same workspace.
 * dgp_backward_batch: dL_dout[B,G,G,G] -> dV[B,N,3], dN[B,N,3], dthres[B] (mode 1: each item's own dL/dthres,
 * which the caller sums for the shared threshold; may be NULL).
 * dgp_forward / dgp_backward are the B = 1 calls of the same launchers. */
int dgp_batch_workspace_size(void* plan, int B, size_t* bytes);
int dgp_forward_batch(void* plan, int B, int N, double sig, const float* V, const float* Nrm, int mode,
                      const float* thres, float* out, void* ws, size_t ws_bytes, void* stream);
int dgp_backward_batch(void* plan, int B, int N, const float* V, const float* Nrm, int mode,
                       const float* dL_dout, float* dV, float* dN, float* dthres,
                       void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------
 * Differentiable marching cubes.  Stands in for diso.DiffMC.__call__(grid, deform=None,
 * isovalue) as called at dgmesh/utils/renderer.py:171 and
 * dgmesh/scene/gaussian_model_dpsr_dynamic_anchor.py:704,851 (third-party package, not in the
 * reference tree: only the CONTRACT at the call sites is reproduced, see DESIGN.md).
 *   phi[G,G,G] fp32, iso  ->  verts[V,3] fp32 in [0,1]^3 (index/(G-1)), faces[F,3] int32
 * V and F are data dependent.  dgmc_count sweeps the grid once and writes totals[2] = {V, F} to a device
 * int32 pair and, when given, to a pinned device-mapped host pair (`totals_host`, e.g. dgm_notify_host) with
 * `totals_event` (a cudaEvent_t) recorded behind it; dgmc_emit writes up to V_cap vertices (verts[V_cap,3] and
 * vsrc[V_cap], each vertex's grid edge as node * 3 + axis, which the backward reads) and F_cap faces
 * (bounds enforced on the device), so a caller may enqueue it OPTIMISTICALLY with the capacities of the previous
 * call before it knows V and F, wait for the event, and re-run dgmc_emit only if something did not fit -- the
 * drop-in Python layer does that; the reference's diso synchronises to size its outputs as well.
 * V is at most one vertex per grid edge, 3 G^2 (G-1) (independent noise reaches ~1.45 G^3).
 * G <= 800 (face references are packed into int32), V_cap <= 2^29 (vertex indices are packed into 29 bits),
 * F_cap < 2^31; a V the packing cannot hold is reported by dgmc_count and refused by dgmc_emit.
 * dgmc_backward: dL_dverts[V,3] -> dL_dphi[G,G,G] (fully written); V as returned by dgmc_count, vsrc as
 * written by dgmc_emit.  It needs no workspace.
 * ------------------------------------------------------------------------ */
int dgmc_workspace_size(int G, size_t* bytes);
int dgmc_count(int G, const float* phi, float iso, void* ws, size_t ws_bytes,
               int32_t* totals, int32_t* totals_host, void* totals_event, void* stream);
int dgmc_emit(int G, const float* phi, float iso, void* ws, size_t ws_bytes,
              float* verts, int32_t* vsrc, int64_t V_cap, int32_t* faces, int64_t F_cap, void* stream);
int dgmc_backward(int G, int V, const float* phi, float iso, const int32_t* vsrc,
                  const float* dL_dverts, float* dL_dphi, void* stream);
/* Marching cubes over a batch of B grids phi[B,G,G,G], 1 <= B <= 64 (B out of range, a NULL pointer or a short
 * workspace is refused on the host before any device work).  The count pass sweeps all B grids in one launch,
 * one scan covers the B grids' brick totals, and one kernel writes totals[B,2] = {V_k, F_k} of every item (and
 * the same pairs to totals_host behind totals_event: dgm_notify_host has room for 256 pairs).  dgmc_emit_batch
 * writes the items one after another -- item k's vertices start at V_0 + .. + V_(k-1), its faces at
 * F_0 + .. + F_(k-1) -- with face indices LOCAL to the item and vsrc local to the item's grid, so item k's slice
 * is exactly what dgmc_emit gives for grid k.  The capacities bound the batch's totals: the 29-bit vertex
 * packing limits the WHOLE batch to V_0 + .. + V_(B-1) <= 2^29 vertices (V_cap <= 2^29), and F_cap < 2^31.
 * dgmc_backward_batch: V_host[B] (host) = the items' vertex counts from totals; dL_dverts[V,3] of the concatenated
 * vertices -> dL_dphi[B,G,G,G] (fully written), one launch.
 * dgmc_workspace_size_batch at B = 1 equals dgmc_workspace_size, and every further item adds its own vertex-owner
 * table (4 G^3 bytes) and brick totals: about 97 MB per item at G = 288.  The single-grid entry points are the
 * B = 1 calls of the same launchers. */
int dgmc_workspace_size_batch(int B, int G, size_t* bytes);
int dgmc_count_batch(int B, int G, const float* phi, float iso, void* ws, size_t ws_bytes,
                     int32_t* totals, int32_t* totals_host, void* totals_event, void* stream);
int dgmc_emit_batch(int B, int G, const float* phi, float iso, void* ws, size_t ws_bytes,
                    float* verts, int32_t* vsrc, int64_t V_cap, int32_t* faces, int64_t F_cap, void* stream);
int dgmc_backward_batch(int B, int G, const int32_t* V_host, const float* phi, float iso, const int32_t* vsrc,
                        const float* dL_dverts, float* dL_dphi, void* stream);

/* ------------------------------------------------------------------------
 * Differentiable dual marching cubes (Nielson 2004).  Stands in for diso.DiffDMC(grid, isovalue):
 *   phi[G,G,G] fp32, iso  ->  verts[V,3] fp32 in [0,1]^3, faces[2Q,3] int32 and, optionally, quads[Q,4] int32
 * Definition:
 *   - A node is inside when phi < iso; corners, edges and case index are those of mc_tables.h.
 *   - The patches of a case are the loops of tools/gen_mc_tables.py (DMC_PATCH, DMC_PATCH_OF_EDGE): at most 4
 *     per case and 7 edges per patch; an ambiguous face separates the inside corners, as in marching cubes.
 *   - A cut edge's crossing is marching cubes' vertex in grid units: t = (iso - p0)/(p1 - p0); pos = n;
 *     pos[axis] += t.  A patch's dual vertex is the fp32 sum of its crossings in increasing edge id, divided by
 *     its edge count, then by G - 1.  A patch gets a vertex only when one of its edges is interior (its four
 *     incident cells lie in the grid), so no vertex is unreferenced.
 *   - Every sign-changing interior edge gives one quad: the dual vertices of the four cells around it (each
 *     cell's patch containing the edge) in cyclic order, oriented so the normal points from the inside node to
 *     the outside one (as dgmc_*), starting at the lowest cell q0; triangles (q0,q1,q2), (q0,q2,q3).  Edges on
 *     the grid's outer faces give nothing.  Q equals the number of interior marching-cubes vertices.
 *   - Closed (every directed edge is matched by its reverse) but not always edge-manifold: in 36 ambiguous
 *     (case, face) pairs one patch holds both segments of the face, and where the cells on both sides do that,
 *     one dual edge is shared by four triangles.
 *   - dL/dphi flows through each crossing's t with weight 1/k per crossing of a k-edge patch; nothing flows to
 *     iso.  The backward gathers the <= 24 (cell, patch) terms of every node in a fixed order, without float
 *     atomics: its result is bit-identical from run to run.
 * Calls, as dgmc_*: dgdmc_count writes totals[2] = {V, Q} (and the same pair to totals_host behind
 * totals_event); dgdmc_emit writes up to V_cap vertices (verts, and vsrc[V_cap] = cell * 4 + patch, which the
 * backward reads) and up to Q_cap quads (faces[2 Q_cap, 3]; quads[Q_cap, 4] when not NULL), capacities enforced
 * on the device, so it may be enqueued optimistically and re-run when something did not fit.
 * Limits: 2 <= G <= 800; V is at most 4 (G-1)^3 and Q at most 3 G^2 (G-1); V_cap <= 2^28 (a cell's first
 * vertex and cell * 4 + patch are packed into 32-bit records), Q_cap < 2^30 (2 Q triangles < 2^31).
 * dgdmc_backward: dL_dverts[V,3] -> dL_dphi[G,G,G] (fully written), V as returned by dgdmc_count, vsrc as
 * written by dgdmc_emit; it takes a workspace of dgdmc_workspace_size bytes, which need not be the forward's.
 * The _batch forms take B grids phi[B,G,G,G], 1 <= B <= 64, with the layout of dgmc_*_batch: item k's
 * vertices and quads follow those of items 0..k-1, indices local to the item, and item k's slice is exactly
 * what the single call gives for grid k; V_host[B] are the items' vertex counts.  The workspace holds the
 * brick totals and an 8-byte record per cell: about 191 MB per item at G = 288.  Bad arguments are refused on
 * the host before any device work.
 * ------------------------------------------------------------------------ */
int dgdmc_workspace_size(int G, size_t* bytes);
int dgdmc_workspace_size_batch(int B, int G, size_t* bytes);
int dgdmc_count(int G, const float* phi, float iso, void* ws, size_t ws_bytes,
                int32_t* totals, int32_t* totals_host, void* totals_event, void* stream);
int dgdmc_count_batch(int B, int G, const float* phi, float iso, void* ws, size_t ws_bytes,
                      int32_t* totals, int32_t* totals_host, void* totals_event, void* stream);
int dgdmc_emit(int G, const float* phi, float iso, void* ws, size_t ws_bytes, float* verts, int32_t* vsrc,
               int64_t V_cap, int32_t* faces, int32_t* quads, int64_t Q_cap, void* stream);
int dgdmc_emit_batch(int B, int G, const float* phi, float iso, void* ws, size_t ws_bytes, float* verts,
                     int32_t* vsrc, int64_t V_cap, int32_t* faces, int32_t* quads, int64_t Q_cap, void* stream);
int dgdmc_backward(int G, int V, const float* phi, float iso, void* ws, size_t ws_bytes, const int32_t* vsrc,
                   const float* dL_dverts, float* dL_dphi, void* stream);
int dgdmc_backward_batch(int B, int G, const int32_t* V_host, const float* phi, float iso, void* ws, size_t ws_bytes,
                         const int32_t* vsrc, const float* dL_dverts, float* dL_dphi, void* stream);

/* ------------------------------------------------------------------------
 * FlexiCubes (Shen et al. 2023; the extractor of nvdiffrec and kaolin) on the topology of dgdmc_*:
 *   phi[G,G,G] fp32, iso, deform[G,G,G,3], alpha[G-1,G-1,G-1,8], beta[G-1,G-1,G-1,12], gamma_f[G-1,G-1,G-1]
 *   ->  verts[V (+ Q),3] fp32 in [0,1]^3, faces[2Q (4Q),3] int32, L_dev per crossing
 * Definition:
 *   - Grid, corners, edges, cases, patches, "inside" (phi < iso) and which patches get a vertex are dgdmc_*'s, so
 *     V and Q are what dgdmc_count returns; its workspace is the emission's.
 *   - s = phi - iso; node n sits at x_n = n + deform[n] (grid units; NULL: 0).  The raw per-cell weights are
 *     indexed by corner r = (i + (r&1), j + ((r>>1)&1), k + (r>>2)) and edge e = 4 axis + combo, and activated as
 *     kaolin does: beta = 1 + 0.99 tanh(b), alpha = 1 + 0.99 tanh(a), gamma = 0.005 + 0.99 sigmoid(g); NULL is raw
 *     0 (beta = alpha = 1, gamma = 1/2).
 *   - Crossing on cut edge e, lower / upper corners r0 / r1: w0 = alpha[r0] s(n0), w1 = alpha[r1] s(n1),
 *     t = w0 / (w0 - w1), u_e = x0 + t (x1 - x0).
 *   - Dual vertex: (sum_e beta[e] u_e) / (sum_e beta[e]), summed in fp32 in increasing edge id, then / (G - 1).
 *     With neutral weights, no deform and iso = 0 every operation rounds as dgdmc_*'s: the vertices are equal.
 *   - Inference (training = 0): each quad (q0,q1,q2,q3) of dgdmc_emit, a vertex's gamma its cell's, gives
 *     (q0,q1,q2), (q0,q2,q3) when gamma0 gamma2 >= gamma1 gamma3 (dgdmc's split), else (q0,q1,q3), (q1,q2,q3).
 *   - Training (training = 1): quad q gets a centre vertex at row V + q, m = (g02 (v0+v2)/2 + g13 (v1+v3)/2) /
 *     (g02 + g13 + 1e-8), g02 = gamma0 gamma2, g13 = gamma1 gamma3, and faces (q0,q1,m), (q1,q2,m), (q2,q3,m),
 *     (q3,q0,m).
 *   - L_dev: for each vertex v and each crossing of its patch, |d_e - mean_e d_e|, d_e = |u_e - v| in output units
 *     (normalize = 1: / (G - 1)), written to ldev[v, slot] (slot: rank of e among the patch's edges, at most 7;
 *     unused slots 0), with the crossing count in vk[v].
 * dgfc_emit, after dgdmc_count on ws: verts[V_cap (+ Q_cap in training), 3], vsrc[V_cap] (as dgdmc_emit),
 * ldev[V_cap, 7], vk[V_cap], faces[(2 | 4) Q_cap, 3], quads[Q_cap, 4] (dgdmc's oriented quads, read by the
 * backward).  Capacities are enforced on the device, so it may be enqueued optimistically and re-run.
 * Limits: as dgdmc_*; in training Q_cap < 2^29, so V + Q < 2^28 + 2^29 vertex indices and 4 Q < 2^31 triangles.
 * dgfc_backward: dL_dverts[V (+ Q), 3] w.r.t. the normalised vertices and dL_dldev[V, 7] (or NULL) ->
 * dL_dphi[G,G,G], and, each when not NULL, dL_ddeform[G,G,G,3], dL_dalpha, dL_dbeta, dL_dgamma (training only)
 * w.r.t. the raw inputs, every element written (zero away from the surface).  verts, vsrc and quads are the
 * emission's; V and Q are dgdmc_count's.  Nothing flows to iso; the gradient at |.| = 0 is 0.  Every gradient is
 * gathered in a fixed order, without float atomics: bit-identical from run to run.  Its workspace is
 * dgfc_backward_workspace_size(G, V, Q, training) bytes: dgdmc's plus 56 bytes per vertex, and 48 more per vertex
 * and 64 per quad in training.  Bad arguments are refused on the host before any device work.
 * ------------------------------------------------------------------------ */
int dgfc_emit(int G, const float* phi, float iso, const float* deform, const float* alpha, const float* beta,
              const float* gamma_f, int training, int normalize, void* ws, size_t ws_bytes, float* verts,
              int32_t* vsrc, float* ldev, int32_t* vk, int64_t V_cap, int32_t* faces, int32_t* quads, int64_t Q_cap,
              void* stream);
int dgfc_backward_workspace_size(int G, int V, int Q, int training, size_t* bytes);
int dgfc_backward(int G, int V, int Q, const float* phi, float iso, const float* deform, const float* alpha,
                  const float* beta, const float* gamma_f, int training, int normalize, const float* verts,
                  const int32_t* vsrc, const int32_t* quads, const float* dL_dverts, const float* dL_dldev, void* ws,
                  size_t ws_bytes, float* dL_dphi, float* dL_ddeform, float* dL_dalpha, float* dL_dbeta,
                  float* dL_dgamma, void* stream);

/* ------------------------------------------------------------------------
 * Tensor-core GEMM building blocks of the MLPs (wgmma, bf16 operands, fp32 accumulation in
 * registers), exposed stand-alone for the parity tests (torch.matmul on the same bf16 operands is the
 * oracle).  The networks below drive the same two kernels on activations kept in the library's
 * blocked layout; these entry points first copy the row-major operands into that layout inside
 * `ws` (dgl_gemm_ws_bytes(M, N, K), with M = the long dimension).
 *   dgl_gemm_bf16   : C[M,N] (fp32, ldc) = A[M,K] (bf16, lda) * B[N,K]^T (bf16, ldb) [+ bias[N]] [ReLU]
 *                     N <= 256; writes columns [0, N rounded up to 4)         (layer kernel)
 *   dgl_gemm_tn_bf16: C[Mf,Nf] += X[P,Mf]^T * Y[P,Nf]   (or C[Nf,Mf] when transpose_out); Mf, Nf <= 256;
 *                     accumulates into C with fp32 reductions                 (weight-gradient kernel)
 * ------------------------------------------------------------------------ */
int dgl_gemm_ws_bytes(int M, int N, int K, size_t* bytes);
int dgl_gemm_bf16(int M, int N, int K, const void* A, int lda, const void* B, int ldb,
                  const float* bias, int relu, float* C, int ldc, void* ws, size_t ws_bytes, void* stream);
int dgl_gemm_tn_bf16(int P, int Mf, int Nf, const void* X, int ldx, const void* Y, int ldy, float* C, int ldc,
                     int transpose_out, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------
 * Deformation / appearance MLPs (dgmesh/utils/time_utils.py:58-323: DeformNetwork,
 * DeformNetworkNormal, DeformNetworkNormalSep, AppearanceNetwork; driven through
 * DeformModel*.step / AppearanceModel.step, dgmesh/scene/deform_model.py, appearance_model.py).
 * The reference runs ~30 fp32 cuBLAS / elementwise kernels per call; here the whole network is a
 * chain of bf16 wgmma GEMMs (fp32 accumulation) with fused bias / ReLU epilogues.
 *
 * DglNet describes one network with PACKED parameters (built by dgl_mlp_pack): bf16 weights in the
 * blocked operand layout of the GEMM kernels (dg-mesh_b200/csrc/mlp_gemm.cuh: element (row, k) of
 * an R-row matrix at ((k/8)*R + row)*8 + k%8) and fp32 biases.  Input columns: 0..62 pe(x,10) |
 * 63 zero | 64.. time features | zero pad to 96; the skip layer (index 5) sees those 96 columns
 * followed by the 256 hidden units.
 *   x[P,3], t[P] fp32  ->  out[P,16] fp32 (first n_out columns valid; column order = the
 *   reference's heads concatenated: warp 3, rotation 4, scaling 3, normal 3 / colour 3)
 * train != 0 additionally stores what dgl_mlp_backward needs in the workspace.
 * backward: g_out[P,16] -> every weight / bias gradient in the packed fp32 layouts of DglGrads
 * (fully written) and dx[P,3] (may be NULL).
 * ------------------------------------------------------------------------ */
typedef struct DglNet {
  int has_timenet;   /* is_blender: pe(t,6) -> 13 -> 256 -> 30 ; else pe(t,10) = 21 features */
  int in_t;          /* 30 or 21 */
  int n_out;         /* <= 16 */
  int sigmoid_out;   /* AppearanceNetwork */
  const void* W[8];  /* forward operand: 256 rows (outputs) x Kpad_l, Kpad = 96, 256 x4, 352, 256 x2 */
  const void* WT[8]; /* backward operand: rows = inputs, K = the 256 outputs.  WT[0]: the 96 [x_emb,t]
                        rows only; WT[5]: the 256 hidden rows, then (at +65536 elements) the 96 rows */
  const float* b[8];
  const void* Wh;    /* 16 rows x 256 */
  const void* WhT;   /* 256 rows x 16 */
  const float* bh;   /* [16] */
  const void* Wt0;   /* 256 rows x 16    timenet.0 (13 -> 256), input padded to 16 */
  const float* bt0;
  const void* Wt1;   /* 32 rows x 256    timenet.2 (256 -> 30), output padded to 32 */
  const void* Wt1T;  /* 256 rows x 32 */
  const float* bt1;  /* [32] */
  /* Forward precision.  precise != 0 ("bf16x3", what dgl_mlp_pack sets): every forward operand is a
   * PAIR of bf16 numbers hi + lo (lo = rounding residual) and each layer accumulates
   * A_hi B_hi + A_lo B_hi + A_hi B_lo in fp32 -- three wgmma passes into one accumulator, ~16
   * mantissa bits per operand, so activations and ReLU decisions match the reference's fp32 cuBLAS
   * to ~1e-5 (a single bf16 pass differs by ~2e-3, enough to flip ReLU signs and move the gradients
   * by ~7 %, see DESIGN.md).  precise == 0: single bf16 pass (3x fewer MMAs).  The backward pass is
   * bf16 in both modes.  The *lo tables have the layout of W / Wh / Wt0 / Wt1. */
  int precise;
  const void* Wlo[8];
  const void* Whlo;
  const void* Wt0lo;
  const void* Wt1lo;
} DglNet;

typedef struct DglGrads {
  float* dW[8];      /* fp32 [256, Kpad_l] */
  float* db[8];      /* [256] */
  float* dWh;        /* [16, 256] */
  float* dbh;        /* [16] */
  float* dWt0;       /* [256, 16] */
  float* dbt0;       /* [256] */
  float* dWt1;       /* [32, 256] */
  float* dbt1;       /* [32] */
} DglGrads;

/* Reference-shaped parameters (fp32, nn.Linear layout [out, in]); DglRawGrads has the same shape
 * with writable pointers.  Heads are listed in output-column order (n_heads <= 4). */
typedef struct DglRaw {
  int has_timenet, in_t, sigmoid_out, n_heads;
  int head_rows[4];
  const float* W[8];   /* linear.l.weight: [256, 63+in_t], [256,256] x4, [256, 63+in_t+256], [256,256] x2 */
  const float* b[8];
  const float* Wh[4];  /* e.g. gaussian_warp [3,256], gaussian_rotation [4,256], ... */
  const float* bh[4];
  const float *Wt0, *bt0, *Wt1, *bt1;  /* timenet.0 [256,13], timenet.2 [in_t,256] */
} DglRaw;
typedef struct DglRawGrads {
  float* W[8];
  float* b[8];
  float* Wh[4];
  float* bh[4];
  float *Wt0, *bt0, *Wt1, *bt1;
} DglRawGrads;

/* byte sizes of the packed bf16 weight buffer, the packed fp32 bias buffer and the packed fp32
 * gradient buffer (fixed for this architecture) */
int dgl_mlp_pack_sizes(size_t* w_bytes, size_t* b_bytes, size_t* g_bytes);
/* fill wbuf / bbuf from the raw parameters and write the DglNet pointer table (host struct) */
int dgl_mlp_pack(const DglRaw* raw, void* wbuf, float* bbuf, DglNet* net_out, void* stream);
/* pointer table into a packed gradient buffer, and its scatter into reference-shaped tensors */
int dgl_mlp_grad_pointers(float* gbuf, DglGrads* grads_out);
int dgl_mlp_unpack_grads(const DglRaw* raw, const float* gbuf, const DglRawGrads* out, void* stream);

int dgl_mlp_workspace(int P, int train, size_t* bytes);
int dgl_mlp_forward(const DglNet* net, int P, const float* x, const float* t, float* out,
                    int train, void* ws, size_t ws_bytes, void* stream);
int dgl_mlp_backward(const DglNet* net, int P, const float* x, const float* out, const float* g_out,
                     void* ws, size_t ws_bytes, const DglGrads* grads, float* dx, void* stream);

/* ------------------------------------------------------------------------
 * Image loss of the training step (next-tier row SURVEY.md 8(f)-3):
 *   loss = (1 - lambda) * mean|img - gt| + lambda * (1 - SSIM(img, gt))        (mode 0)
 * as dgmesh/train.py:308-311 composes l1_loss and ssim (dgmesh/utils/loss_utils.py:18-19, 39-76:
 * 11x11 Gaussian window, sigma 1.5, zero padding, C1 = 0.01^2, C2 = 0.03^2); mode 1 returns the
 * SSIM value itself (the stand-alone `ssim()` of the reference).  img, gt: [3,H,W] fp32.
 *   forward : out3 = {loss (or ssim in mode 1), l1, ssim} on the device (no host read); keeps three
 *             partial-derivative maps in `ws` for the backward call
 *   backward: dL_dimg[3,H,W] = dL_dloss[0] * d out3[0] / d img   (dL_dloss NULL = 1)
 * ------------------------------------------------------------------------ */
int dgloss_workspace_size(int H, int W, size_t* bytes);
int dgloss_forward(int H, int W, const float* img, const float* gt, float lambda_dssim, int mode,
                   float* out3, void* ws, size_t ws_bytes, void* stream);
int dgloss_backward(int H, int W, const float* img, const float* gt, float lambda_dssim, int mode,
                    const float* dL_dloss, float* dL_dimg, void* ws, size_t ws_bytes, void* stream);

/* Laplacian mesh regulariser (umbrella operator) of the mesh branch:
 * nvdiffrast_utils.regularizer.laplace_regularizer_const(verts, faces)
 * (dgmesh/nvdiffrast_utils/regularizer.py:40-59, used at dgmesh/train.py:277-283).
 *   verts[V,3], tri[F,3] int32 -> out[1] = mean((T / max(n, 1))^2); the workspace carries the
 *   per-vertex state to dgl_laplacian_backward: dL_dloss[1] (NULL = 1) -> dverts[V,3] (fully written). */
int dgl_laplacian_workspace(int V, size_t* bytes);
int dgl_laplacian_forward(int V, int F, const float* verts, const int32_t* tri, float* out, void* ws,
                          size_t ws_bytes, void* stream);
int dgl_laplacian_backward(int V, int F, const int32_t* tri, const float* dL_dloss, float* dverts, void* ws,
                           size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------
 * Differentiable triangle-mesh rasterisation (next-tier row SURVEY.md 8(f)-1): the three primitives
 * dgmesh/utils/renderer.py:33-121 (render_mask / render_mesh) takes from nvdiffrast --
 * dr.rasterize, dr.interpolate, dr.antialias -- forward and backward, one image (batch 1).
 * nvdiffrast is third-party and not in the reference tree: the CONTRACT of those calls is reproduced
 * (dg-mesh_b200/csrc/meshrast.cu states it), parity is geometric (DESIGN.md).
 *   pos[V,4]  clip-space positions (x, y, z, w), tri[F,3] int32, image H x W, row 0 = NDC y -1
 *   rast[H,W,4] = (u, v, z/w, triangle id + 1; all zero where nothing is hit)
 *   dgmr_rasterize      zbuf: caller scratch of 8 * H * W bytes
 *   dgmr_rasterize_bwd  grast[H,W,4] (only .xy used) -> gpos[V,4] ACCUMULATED (caller zero-fills)
 *   dgmr_interpolate    attr[V,C] -> out[H,W,C]
 *   dgmr_interpolate_bwd  gout[H,W,C] -> gattr[V,C] ACCUMULATED (may be NULL), grast[H,W,4] written (may be NULL)
 *   dgmr_antialias      color[H,W,C], opp[F,3] (vertex opposite edge k = (v_k, v_k+1) in the neighbouring
 *                       triangle, -1 on a boundary) -> out[H,W,C]
 *   dgmr_antialias_bwd  gout -> gcolor[H,W,C] written (may be NULL), gpos[V,4] ACCUMULATED (may be NULL)
 * ------------------------------------------------------------------------ */
int dgmr_rasterize(int V, int F, int W, int H, const float* pos, const int32_t* tri, void* zbuf, float* rast,
                   void* stream);
int dgmr_rasterize_bwd(int W, int H, const float* rast, const int32_t* tri, const float* pos, const float* grast,
                       float* gpos, void* stream);
int dgmr_interpolate(int W, int H, int C, const float* attr, const float* rast, const int32_t* tri, float* out,
                     void* stream);
int dgmr_interpolate_bwd(int W, int H, int C, const float* attr, const float* rast, const int32_t* tri,
                         const float* gout, float* gattr, float* grast, void* stream);
int dgmr_antialias(int W, int H, int C, const float* color, const float* rast, const float* pos,
                   const int32_t* tri, const int32_t* opp, float* out, void* stream);
int dgmr_antialias_bwd(int W, int H, int C, const float* color, const float* rast, const float* pos,
                       const int32_t* tri, const int32_t* opp, const float* gout, float* gcolor, float* gpos,
                       void* stream);
/* Range mode (nvdiffrast's way of rendering several meshes into a batch of images): B images, 1 <= B <= 64.
 *   ranges[B,2] int32 on the HOST = (first triangle, count) of image b within tri[F,3]; every range must lie in
 *   [0, F] (else DGM_E_BADARG before any device work).  The ranges are passed to the kernel by value.
 *   dgmr_rasterize_batch   zbuf: 8 * B * H * W bytes -> rast[B,H,W,4], triangle ids GLOBAL + 1; an empty range
 *                          gives an all-zero image
 *   rast.w (both modes) holds id + 1 as nvdiffrast encodes it: a float up to 2^24, above that the float whose bit
 *   pattern is 0x4a800000 + (id + 1); F <= 2^29 (larger F is refused).
 *   the other _batch calls take rast[B,H,W,4] and images [B,H,W,C] and the same pos[V,4] / attr[V,C] / tri for
 *   every image; gradients of pos and attr accumulate over the images.  Antialiasing pairs pixels within an
 *   image only.  The single-image entry points are the B = 1 calls of the same launchers. */
int dgmr_rasterize_batch(int V, int F, int B, const int32_t* ranges, int W, int H, const float* pos,
                         const int32_t* tri, void* zbuf, float* rast, void* stream);
int dgmr_rasterize_bwd_batch(int B, int W, int H, const float* rast, const int32_t* tri, const float* pos,
                             const float* grast, float* gpos, void* stream);
int dgmr_interpolate_batch(int B, int W, int H, int C, const float* attr, const float* rast, const int32_t* tri,
                           float* out, void* stream);
int dgmr_interpolate_bwd_batch(int B, int W, int H, int C, const float* attr, const float* rast,
                               const int32_t* tri, const float* gout, float* gattr, float* grast, void* stream);
int dgmr_antialias_batch(int B, int W, int H, int C, const float* color, const float* rast, const float* pos,
                         const int32_t* tri, const int32_t* opp, float* out, void* stream);
int dgmr_antialias_bwd_batch(int B, int W, int H, int C, const float* color, const float* rast, const float* pos,
                             const int32_t* tri, const int32_t* opp, const float* gout, float* gcolor,
                             float* gpos, void* stream);

/* ------------------------------------------------------------------------
 * Adaptive density control on the device (next-tier row SURVEY.md 8(f)-2): the whole of
 * GaussianModelDPSRDynamicAnchor.densify_and_prune
 * (dgmesh/scene/gaussian_model_dpsr_dynamic_anchor.py:469-551: densify_and_clone, densify_and_split
 * with N = 2, prune; built on cat_tensors_to_optimizer :403-428, _prune_optimizer :383-401,
 * densification_postfix :430-452) as one plan and one gather over the seven parameter tensors and
 * both Adam moments.  Same survivors, same final row order
 * [kept originals | clones | first split copies | second split copies], same values.
 *   dgd_plan        xyz_gradient_accum[P], denom[P], _scaling[P,3], _opacity[P] (raw, pre-activation)
 *                   -> counts[4] on the device = {kept originals, clones, split-selected, children per copy};
 *                   the new model has counts[0] + counts[1] + 2 * counts[3] rows.  size_prune = the
 *                   reference's `if max_screen_size:` branch.  The caller reads counts (the one host read).
 *                   extent and percent_dense are doubles because the reference forms percent_dense * extent
 *                   and 0.1 * extent in Python double, which torch rounds once to float32 to compare.
 *   dgd_split_stds  stds[2 * counts[2], 3] = get_scaling[selected].repeat(2, 1): feed torch.normal(0, stds)
 *                   so the generator is consumed exactly as by the reference (:463-465)
 *   dgd_apply       fields_host: up to DGD_MAX_FIELDS tensors [P, width] with optional Adam moments,
 *                   role 1 = xyz, 2 = _scaling, 0 = copied as is; samples[2 * counts[2], 3];
 *                   rotation_raw[P,4].  Writes every row of every output tensor.
 * ------------------------------------------------------------------------ */
#define DGD_MAX_FIELDS 8
typedef struct DgdField {
  const float* src;     /* [P, width] */
  const float* m1_src;  /* Adam exp_avg    [P, width] or NULL */
  const float* m2_src;  /* Adam exp_avg_sq [P, width] or NULL */
  float* dst;           /* [n_out, width] */
  float* m1_dst;
  float* m2_dst;
  int width;
  int role;             /* 0 plain, 1 xyz, 2 scaling */
} DgdField;
int dgd_workspace_size(int P, size_t* bytes);
int dgd_plan(int P, const float* xyz_gradient_accum, const float* denom, const float* scaling_raw,
             const float* opacity_raw, float max_grad, float min_opacity, double extent, double percent_dense,
             int size_prune, float max_screen_size, void* ws, size_t ws_bytes, int32_t* counts, void* stream);
int dgd_split_stds(int P, const float* scaling_raw, void* ws, size_t ws_bytes, float* stds, void* stream);
int dgd_apply(int P, int n_fields, const DgdField* fields_host, const float* rotation_raw, const float* samples,
              void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------
 * Optimiser step and densification statistics: what a training iteration does after loss.backward().
 *
 * dgo_adam_step: the Adam update of up to DGO_MAX_TENSORS float32 tensors in ONE launch, element for element
 * the arithmetic of torch.optim.Adam's single-tensor path (no weight decay, no amsgrad, no maximize; the
 * operation-by-operation statement is at the top of csrc/optim.cu):
 *     m = m + (1 - beta1) (g - m);  v = beta2 v + (1 - beta2) g g;
 *     p = p - step_size * m / (sqrt(v) * inv_bc2_sqrt + eps)
 * The descriptors are read on the host during the call and travel to the kernel by value: no device table, no
 * upload.  beta1 and beta2 are doubles because torch forms 1 - beta in double before it rounds to float32.
 *   row_radii  NULL: every element is updated.  Otherwise int32 [rows]: element e of a tensor belongs to row
 *              e / row_width, and a row is updated iff row_radii[row] > 0 (sparse Adam as in the official 3DGS
 *              code: a hidden row keeps p, m and v bit for bit, its moments do not decay, the step count is
 *              global).  Then every tensor needs row_width > 0, n % row_width == 0 and the same n / row_width.
 *   zero_grad  != 0: g is set to zero in the same pass (also in hidden rows), although it is declared const.
 * n_tensors outside 1..DGO_MAX_TENSORS, a NULL p / g / m / v, n < 0 or a violated row rule: DGM_E_BADARG before
 * any device work.  A tensor with n == 0 is skipped.  16-byte accesses for a tensor whose four pointers are
 * 16-byte aligned and whose n % 4 == 0, 4-byte accesses otherwise.
 *
 * dgo_densify_stats: GaussianModelDPSRDynamicAnchor.add_densification_stats
 * (gaussian_model_dpsr_dynamic_anchor.py:679-682) and train.py:491-496's max_radii2D update with no boolean-mask
 * indexing, hence no host read.  For f = 0 .. F-1 in order, for every row with radii[f][i] > 0:
 *     xyz_gradient_accum[i] += sqrt(gx^2 + gy^2) of viewspace_grad[f][i];  denom[i] += 1;
 *     max_radii2D[i] = max(max_radii2D[i], (float)radii[f][i])
 * and, when viewspace_abs_grad and xyz_gradient_accum_abs are given (both or neither), the same norm of the
 * absolute gradient (AbsGS) into its own accumulator.  Frame f's gradients are at viewspace_grad + f * grad_stride
 * ([P,3] floats each, the same stride for the abs gradient), its radii at radii + f * radii_stride; F = 1 ignores
 * the strides.  max_radii2D may be NULL (not updated: the reference's method leaves it to its caller).  A row no
 * frame shows is not written.
 * ------------------------------------------------------------------------ */
#define DGO_MAX_TENSORS 32
typedef struct DgoTensor {
  float* p;            /* parameter   [n] */
  const float* g;      /* gradient    [n] */
  float* m;            /* exp_avg     [n] */
  float* v;            /* exp_avg_sq  [n] */
  int64_t n;
  int row_width;       /* elements per row; read only with row_radii */
  float step_size;     /* lr / (1 - beta1^step), formed in double */
  float inv_bc2_sqrt;  /* 1 / sqrt(1 - beta2^step), formed in double */
  float eps;
} DgoTensor;
int dgo_adam_step(int n_tensors, const DgoTensor* tensors_host, double beta1, double beta2,
                  const int32_t* row_radii, int zero_grad, void* stream);
int dgo_densify_stats(int F, int P, const float* viewspace_grad, const float* viewspace_abs_grad,
                      int64_t grad_stride, const int32_t* radii, int64_t radii_stride, float* xyz_gradient_accum,
                      float* xyz_gradient_accum_abs, float* denom, float* max_radii2D, void* stream);

/* ------------------------------------------------------------------------
 * Data-parallel exchange (SURVEY.md 8(e)): in-place all-reduce (sum, then * scale) of ONE flat fp32 buffer
 * that lives in symmetric memory mapped through an NVSwitch multicast object -- the reduction is done BY THE
 * SWITCH (multimem.ld_reduce of this rank's slice, multimem.st of the result to every replica), one kernel,
 * two flag barriers across the ranks.  No reference counterpart (the reference is single-GPU); replaces the
 * ncclAllReduce this path would otherwise issue.
 *   multicast_ptr   the multicast (NVLS) address of the buffer; n_floats a multiple of 4, buffer 16-B aligned
 *   signal_pads_dev device array of `world` pointers to the ranks' signal pads (uint32, symmetric memory),
 *                   each at least `blocks * world` words, zero before the first call
 *   epoch           starts at 1 and must advance by 2 per call on all ranks alike (flags are never reset)
 *   blocks          CTAs (<= signal-pad words / world); the same value on every rank
 * ------------------------------------------------------------------------ */
int dgx_allreduce_nvls(float* multicast_ptr, size_t n_floats, void* signal_pads_dev, int rank, int world,
                       uint32_t epoch, float scale, int blocks, void* stream);

/* ------------------------------------------------------------------------
 * Measurement hooks (bench.py roofline leg).  Off by default.  When enabled the
 * library records a CUDA event pair around each of its kernels ON THE LAUNCHING
 * STREAM; dgm_profile_read synchronises those events (the only call in this
 * library that waits on the device) and returns the duration in ms of the most
 * recent launch of kernel k, k in DGM_K_*; -1 if it never ran.
 * ------------------------------------------------------------------------ */
#define DGM_K_PREPROCESS 0
#define DGM_K_TILE_SCAN 1
#define DGM_K_SCATTER 2
#define DGM_K_SORT_PACK 3
#define DGM_K_RENDER_FWD 4
#define DGM_K_RENDER_BWD 5
#define DGM_K_PREPROCESS_BWD 6
#define DGM_K_COUNT_TILES 7
#define DGM_K_NORMAL_GRAD_FINISH 8
#define DGM_K_MEDIAN_GRAD 9
#define DGM_K_COUNT 16
int dgm_profile_enable(int on);
int dgm_profile_read(float* ms_host, int n);
/* dgm_profile_enable(2) = timeline mode: every rasterizer kernel launched afterwards (any stream,
 * including the internal streams of the _batch calls) is bracketed by timing events.
 * dgm_timeline_read synchronises the device and returns the number of launches recorded;
 * begin/end are milliseconds relative to the first recorded launch ("begin" = the launch reached
 * the front of its stream).  Diagnostic only (tools/batch_timeline.py). */
int dgm_timeline_read(float* begin_ms, float* end_ms, int* kernel_ids, int cap);

/* ------------------------------------------------------------------------
 * Opacity field of the Gaussians on a grid (csrc/opacity_field.cu), differentiable in means, scales, rotations
 * and opacities:
 *   phi(x) = sum_i o_i g_k(q_i(x)),  q_i(x) = |M_i^-T (x - mu_i)|^2,  M_i = diag(m s_i) R(q_i)  (Sigma = M^T M, the
 *   rasterizer's covariance of the un-normalised quaternion),  g_k(q) = max(0, (e^{-q/2} - e^{-k^2/2}) /
 *   (1 - e^{-k^2/2})).
 * phi[G,G,G] fp32, phi[i,j,k] = phi(lo + (hi - lo) (i, j, k) / (G - 1)), i along x: the layout and vertex convention
 * of dgmc_*.  box is a DEVICE pointer to {lo x, lo y, lo z, hi x, hi y, hi z}; it is never read on the host.
 * means3D [P,3], scales [P,3], rotations [P,4] (r, x, y, z), opacities [P] (or [P,1]).  A Gaussian with a singular M
 * (a zero scale, a zero quaternion) contributes nothing and receives zero gradient.
 * The (Gaussian, 8^3-node brick) pair count is data dependent.  dgf_forward writes it to `pairs_host` (pinned,
 * device-mapped int32[2], e.g. dgm_notify_host: {pairs, 0}, pairs = -1 beyond 2^31 - 1) with `pairs_event` recorded
 * behind it, early in the chain; if pairs > pair_cap, the stages after the count do nothing and phi is not written:
 * the caller waits for the event and calls dgf_forward again with a workspace for pair_cap >= pairs (the result is
 * the same bits as a call sized right the first time).  dgf_backward reads the workspace of the forward that
 * produced phi (same arguments, same pair_cap) and writes all four gradients in full.
 * Bounds: 2 <= G <= 1024, 0 <= pair_cap <= 2^31 - 1, cutoff k > 0 and scale_modifier m > 0, both finite.
 * ------------------------------------------------------------------------ */
int dgf_workspace_size(int P, int G, int64_t pair_cap, size_t* bytes);
int dgf_forward(int P, int G, const float* means3D, const float* scales, const float* rotations,
                const float* opacities, const float* box, float cutoff, float scale_modifier, int64_t pair_cap,
                void* ws, size_t ws_bytes, float* phi, int32_t* pairs_host, void* pairs_event, void* stream);
int dgf_backward(int P, int G, const float* means3D, const float* scales, const float* rotations,
                 const float* opacities, const float* box, float cutoff, float scale_modifier, int64_t pair_cap,
                 void* ws, size_t ws_bytes, const float* dL_dphi, float* dL_dmeans3D, float* dL_dscales,
                 float* dL_drotations, float* dL_dopacities, void* stream);

/* ------------------------------------------------------------------------
 * TSDF fusion of depth maps into a dense truncated signed-distance volume (csrc/tsdf.cu): Open3D's projective
 * TSDF (nearest pixel, uniform weights, positive in front of the surface).
 * Grid: G nodes per axis over box = {lo x, lo y, lo z, hi x, hi y, hi z} (a DEVICE pointer, as dgf_forward takes
 * it); node (i, j, k) is at lo + (hi - lo) (i, j, k) / (G - 1), i along x, flat index (i G + j) G + k: the layout
 * and vertex convention of dgf_forward and dgmc_*.
 * State, caller-owned, integrated in place: tsdf [G,G,G] (start at 1), weight [G,G,G] (start at 0), optionally
 * color_grid [3,G,G,G] planar (start at 0).
 * Frame f: views_host [F,16] = world_view_transform (row-vector convention: p = (x, 1) V), coefs_host [F,4] =
 * (a_x, b_x, a_y, b_y) of the pixel rays exactly as dgr_depth_normal_fwd takes them; depth [F,H,W] and color
 * [F,3,H,W] on the device.  Per node, for f = 0 .. F-1 in order, in fp32, every product, sum, difference and
 * quotient rounded once and nothing contracted (fl(.) below):
 *   x = fl(lo + fl(fl(fl(hi - lo) * i) / (G - 1)))   per axis (i, j, k exactly converted to float)
 *   p_c = fl(fl(fl(fl(x V[0][c]) + fl(y V[1][c])) + fl(z V[2][c])) + V[3][c])   c = 0, 1, 2;  z_c = p_2
 *   skip unless z_c > 0
 *   u = fl(fl(fl(p_0 / z_c) - b_x) / a_x),  v = fl(fl(fl(p_1 / z_c) - b_y) / a_y)
 *   iu = floor(fl(u + 0.5)), iv = floor(fl(v + 0.5));  skip unless 0 <= iu < W and 0 <= iv < H
 *   D = depth[f, iv, iu];  skip unless D is finite and 0 < D <= depth_max
 *   sdf = fl(D - z_c);  skip if sdf < -sdf_trunc
 *   t = min(1, fl(sdf / sdf_trunc)),  w' = fl(w + 1)
 *   tsdf = fl(fl(fl(tsdf w) + t) / w'),  color_c = fl(fl(fl(color_c w) + color[f, c, iv, iu]) / w'),  w = w'
 * Weights are exact integers (below 2^24), and the result depends only on the sequence of frames: F frames in one
 * call, in any split over several calls, or one call per frame give the same bits.  No atomics: bit-identical
 * from run to run.  views_host and coefs_host are HOST memory read during the call; the call neither allocates
 * nor synchronises.
 * DGM_E_BADARG before any device work for: G outside [2, 1024]; F, W or H < 1; sdf_trunc not finite or <= 0;
 * depth_max NaN or <= 0 (+inf is allowed); a zero a_x or a_y; a NULL required pointer; color and color_grid not
 * both NULL or both non-NULL.
 * ------------------------------------------------------------------------ */
int dgt_integrate(int G, const float* box, int F, int W, int H, const float* views_host, const float* coefs_host,
                  const float* depth, const float* color, float sdf_trunc, float depth_max, float* tsdf,
                  float* weight, float* color_grid, void* stream);

/* ------------------------------------------------------------------------
 * Structural losses of mesh evaluation: PointFlow's nn_distance and match_cost (DG-Mesh:
 * dgmesh/metrics/pytorch_structural_losses, nndistance.cu and approxmatch.cu), batched.
 * xyz1 [B,N,3] and xyz2 [B,M,3] fp32 on the device; each batch item is independent, and B items in one call give
 * the same bits as B calls of one item.  No float atomics: every output is bit-identical from run to run.  Nothing
 * allocates or synchronises with the host.  DGM_E_BADARG before any device work for: B, N or M < 1, B > 65535,
 * 3 B N or 3 B M >= 2^31, or a NULL pointer; a workspace below its query: DGM_E_WORKSPACE, also before any
 * device work.
 *
 * dge_nn_distance: dist1 [B,N] = squared distance from each point of set 1 to its nearest point in set 2 of the
 * same item, idx1 [B,N] its index (int64, local to the item; ties: lowest index); dist2 / idx2 [B,M] the same from
 * set 2 to set 1.  The squared distance is ((dx^2 + dy^2) + dz^2) with fused multiply-adds, d = query - reference
 * (dgk_nearest is the B = 1, one-direction case and gives the same bits).
 * dge_nn_distance_bwd: with g1 = grad_dist1 [B,N], g2 = grad_dist2 [B,M] (both required),
 *   grad_xyz1[k] = 2 g1[k] (xyz1[k] - xyz2[idx1[k]]) - sum_{l: idx2[l] = k} 2 g2[l] (xyz2[l] - xyz1[k]),
 *   and symmetrically grad_xyz2; the sums run in increasing l.  Workspace: dge_nn_distance_workspace.
 *
 * dge_match_cost: Fan et al.'s approximate matching cost, per item (n = N, m = M, d_kl the squared distance):
 *   remainL[k] = multiL, remainR[l] = multiR; n >= m: multiL = 1, multiR = float(n / m), else multiL = float(m / n),
 *   multiR = 1 (integer divisions);
 *   for j = 7, 6, ..., -2, level = -4^j (0 at j = -2), e_kl = exp(level d_kl) (__expf):
 *     ratioL[k] = remainL[k] / (1e-9 + sum_l e_kl remainR[l])
 *     s_l = remainR[l] sum_k e_kl ratioL[k];  ratioR[l] = min(remainR[l] / (s_l + 1e-9), 1) remainR[l];
 *     remainR[l] = max(0, remainR[l] - s_l)
 *     w_kl = e_kl ratioL[k] ratioR[l];  remainL[k] = max(0, remainL[k] - sum_l w_kl);  match_kl += w_kl
 *   cost[b] = sum_kl match_kl sqrt(d_kl).
 * The matching is not stored: the workspace keeps ratioL and ratioR of every level (10 B (N + M) floats) plus
 * chunk partials, and dge_match_cost_bwd rebuilds match from them, so it needs the workspace of the dge_match_cost
 * call on the same xyz1 / xyz2, untouched.  dge_match_cost_bwd: with match held constant,
 *   grad_xyz1[k] = grad_cost[b] sum_l match_kl (xyz1[k] - xyz2[l]) / max(sqrt(d_kl), 1e-20),
 *   grad_xyz2[l] = grad_cost[b] sum_k match_kl (xyz2[l] - xyz1[k]) / max(sqrt(d_kl), 1e-20)
 * (the reference's matchcostgrad, not the total derivative of the cost).  grad_cost [B] on the device.
 * ------------------------------------------------------------------------ */
int dge_nn_distance(int B, int N, int M, const float* xyz1, const float* xyz2, float* dist1, int64_t* idx1,
                    float* dist2, int64_t* idx2, void* stream);
int dge_nn_distance_workspace(int B, int N, int M, size_t* bytes);
int dge_nn_distance_bwd(int B, int N, int M, const float* xyz1, const float* xyz2, const int64_t* idx1,
                        const int64_t* idx2, const float* grad_dist1, const float* grad_dist2, float* grad_xyz1,
                        float* grad_xyz2, void* ws, size_t ws_bytes, void* stream);
int dge_match_cost_workspace(int B, int N, int M, size_t* bytes);
int dge_match_cost(int B, int N, int M, const float* xyz1, const float* xyz2, float* cost, void* ws,
                   size_t ws_bytes, void* stream);
int dge_match_cost_bwd(int B, int N, int M, const float* xyz1, const float* xyz2, const float* grad_cost,
                       float* grad_xyz1, float* grad_xyz2, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------
 * Point-to-mesh distance: the closest point of one triangle mesh to each of Q query points.
 * verts [V,3] fp32, faces [F,3] int32, points [Q,3] fp32, all on the device.  Every face index must lie in [0, V);
 * the kernels do not check it (an index outside reads outside verts).  Nothing allocates or synchronises with the
 * host.  DGM_E_BADARG before any device work for: V or F < 1, Q < 0, 3 V, 3 F or 3 Q >= 2^31, or a NULL pointer; a
 * workspace below its query: DGM_E_WORKSPACE, also before any device work.  Q = 0 returns DGM_OK and does nothing
 * (no pointer is read).
 *
 * dgpm_forward: for every query q,
 *   dist2[q] = min over faces f of the squared distance from points[q] to triangle f,
 *   face[q] (int64) = the f of the minimum, ties (equal fp32 distances) going to the lowest f,
 *   bary[q] [3] = weights w >= 0 summing to 1 up to rounding, with closest point
 *     c_q = w0 verts[faces[f][0]] + w1 verts[faces[f][1]] + w2 verts[faces[f][2]].
 * The closest point is computed from a vertex of its region, so a query equal to a vertex of the mesh has
 * dist2 = 0 exactly and the lowest-index face incident to it.  A triangle degenerate in fp32 (collinear or
 * coincident vertices) is measured as its longest edge or its point, with its weights on that edge.  The BVH over
 * the faces and the queries' Morton order are built in the workspace on every call; the outputs are bit-identical
 * from run to run.  Workspace: dgpm_forward_workspace (depends on F and Q).
 * dgpm_backward: with g = grad_dist2 [Q] and face / bary from dgpm_forward on the same inputs,
 *   grad_points[q] = 2 g[q] (points[q] - c_q),
 *   grad_verts[v] = - sum over (q, k) with faces[face[q]][k] = v of 2 g[q] bary[q][k] (points[q] - c_q),
 * the exact derivative of dist2 wherever the closest point is unique.  The sum runs in increasing 3 q + k, without
 * float atomics (bit-identical from run to run); vertices no query touches get 0.  Both outputs are written, not
 * accumulated.  Workspace: dgpm_backward_workspace (depends on V and Q).
 * ------------------------------------------------------------------------ */
int dgpm_forward_workspace(int V, int F, int Q, size_t* bytes);
int dgpm_forward(int V, int F, int Q, const float* verts, const int32_t* faces, const float* points, float* dist2,
                 int64_t* face, float* bary, void* ws, size_t ws_bytes, void* stream);
int dgpm_backward_workspace(int V, int F, int Q, size_t* bytes);
int dgpm_backward(int V, int F, int Q, const float* verts, const int32_t* faces, const float* points,
                  const int64_t* face, const float* bary, const float* grad_dist2, float* grad_points,
                  float* grad_verts, void* ws, size_t ws_bytes, void* stream);

/* dgpm_winding: the generalized winding number (Jacobson et al. 2013) of the mesh at every query q,
 *   winding[q] = (1 / 4 pi) sum over faces f of Omega_f(q),
 *   Omega_f(q) = 2 atan2(det[a b c], |a||b||c| + (a.b)|c| + (b.c)|a| + (c.a)|b|), a, b, c = the face's vertices
 *   in the order faces[f][0..2], minus points[q],
 * with Omega_f(q) = 0 where det[a b c] is exactly 0 (a query on a face, edge or vertex, and faces with coincident
 * or collinear vertices add nothing).  Orientation: winding = +1 inside a closed mesh whose faces are
 * counter-clockwise seen from outside (right-hand normal (b - a) x (c - a) pointing out), -1 inside one oriented
 * the other way, 0 outside; open, non-manifold or self-intersecting meshes give values in between that degrade
 * smoothly.  The sum is evaluated on dgpm_forward's BVH with Barill et al. 2018's order-1 expansion of every child
 * cluster (area-weighted centroid p~, radius r bounding its vertices): a cluster with |points[q] - p~| > beta r
 * adds its far-field term instead of its faces.  beta > 0 and not NaN; beta = +inf never takes the far field and
 * gives the exact sum of the fp32 solid angles (accumulated in float64).  The result is bit-identical from run to
 * run and does not depend on the other queries of the call.
 * dist2, face and bary are all NULL (winding only) or all non-NULL: then they are dgpm_forward's outputs, bit for
 * bit, from the same build.  DGM_E_BADARG also for beta <= 0 or NaN, or for only some of dist2, face, bary NULL.
 * Workspace: dgpm_winding_workspace (depends on F and Q; dgpm_forward's plus the expansions).
 * ------------------------------------------------------------------------ */
int dgpm_winding_workspace(int V, int F, int Q, size_t* bytes);
int dgpm_winding(int V, int F, int Q, const float* verts, const int32_t* faces, const float* points, float beta,
                 float* winding, float* dist2, int64_t* face, float* bary, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------
 * Deformation regularisers (Dynamic 3D Gaussians' local rigidity, rotation similarity and isometry) over an exact
 * K-nearest-neighbour graph of the Gaussians.  All pointers are device memory.  Nothing allocates or synchronises
 * with the host.  DGM_E_BADARG before any device work for: K outside [1, 32], P < 0, 0 < P <= K, 3 P K >= 2^31,
 * F < 0 or 4 F P >= 2^31, a negative or non-finite weight_lambda, or a NULL pointer; a workspace below its query:
 * DGM_E_WORKSPACE, also before any device work.  P = 0 (or F = 0) returns DGM_OK and does nothing (no pointer is
 * read).
 *
 * dgkg_build: the graph of points [P,3] fp32.
 *   index [P,K] int32: the K nearest other points of each point, ascending in (dist2, original index); only the point
 *     itself is excluded, so exact duplicates are neighbours at distance 0, and equal distances go to the lowest
 *     index.  dist2 [P,K] = fmaf(dz, dz, fmaf(dy, dy, dx dx)) with d = x_j - x_i (the bits of dgk_nearest).
 *   weight [P,K] = expf(-weight_lambda dist2).
 *   inv_offsets [P+1], inv_pairs [P K] int32: the inverse graph as a CSR over targets.  The pair ids p = i K + k
 *     with index[p] = j are inv_pairs[inv_offsets[j] .. inv_offsets[j+1]), in increasing p.
 *   The result is exact and bit-identical from run to run.  Workspace: dgkg_workspace (depends on P and K).
 * dgdr_forward: with the graph's index and weight, state a (xyz_a [P,3], rot_a [P,4]) and F states b (xyz_b [F,P,3],
 *   rot_b [F,P,4]), quaternions raw (w, x, y, z) and normalised inside as q / max(|q|, 1e-12), and per pair
 *   (i, j = index[i,k], w = weight[i,k]): r_i = n(q_b,i) (x) conj(n(q_a,i)), da = x_a,j - x_a,i, db = x_b,j - x_b,i,
 *     losses[0][f] = rigid = sum w sqrt(|R(r_i)^T db - da|^2 + 1e-20) / (P K)
 *     losses[1][f] = rot   = sum w sqrt(|r_j - r_i|^2 + 1e-20) / (P K)
 *     losses[2][f] = iso   = sum | |da| - |db| | / (P K)
 *   (losses [3,F]).  Workspace: dgdr_forward_workspace (depends on F and P).
 * dgdr_backward: grad_losses [3,F] -> grad_xyz_a [P,3], grad_rot_a [P,4] (summed over the frames in frame order),
 *   grad_xyz_b [F,P,3], grad_rot_b [F,P,4].  Each output may be NULL (not computed); the others are written, not
 *   accumulated.  At the kinks the gradient is torch's: 0 through |x| at x = 0 and through |v| at v = 0.  The j-side
 *   terms are gathered through inv_offsets / inv_pairs, without float atomics: bit-identical from run to run, and a
 *   frame of a batch gives the bits of the same frame alone.  Workspace: dgdr_backward_workspace (depends on F and P).
 * ------------------------------------------------------------------------ */
int dgkg_workspace(int P, int K, size_t* bytes);
int dgkg_build(int P, int K, float weight_lambda, const float* points, int32_t* index, float* dist2, float* weight,
               int32_t* inv_offsets, int32_t* inv_pairs, void* ws, size_t ws_bytes, void* stream);
int dgdr_forward_workspace(int F, int P, int K, size_t* bytes);
int dgdr_forward(int F, int P, int K, const int32_t* index, const float* weight, const float* xyz_a,
                 const float* rot_a, const float* xyz_b, const float* rot_b, float* losses, void* ws, size_t ws_bytes,
                 void* stream);
int dgdr_backward_workspace(int F, int P, int K, size_t* bytes);
int dgdr_backward(int F, int P, int K, const int32_t* index, const float* weight, const int32_t* inv_offsets,
                  const int32_t* inv_pairs, const float* xyz_a, const float* rot_a, const float* xyz_b,
                  const float* rot_b, const float* grad_losses, float* grad_xyz_a, float* grad_rot_a,
                  float* grad_xyz_b, float* grad_rot_b, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------
 * HexPlane / K-Planes space-time feature field (4D-GS).  Device pointers, except res_host [S] (the spatial
 * resolution of each scale), planes_host and grad_planes_host [6 S] (host arrays of device pointers).  Nothing
 * allocates or synchronises with the host.  DGM_E_BADARG before any device work for: S outside [1, 4], C not 16 or
 * 32, a resolution below 2, R R C or R_t R C >= 2^31 for a plane, N < 0, F < 0, 3 S N (1 + F) >= 2^31,
 * F N S C >= 2^31, or a NULL pointer; a workspace below its query: DGM_E_WORKSPACE.  F = 0 or N = 0 writes nothing
 * (the backward zeroes the plane gradients).
 *
 * The field: x [N,3] canonical positions, t [F,N] times, box [6] = (lo xyz, hi xyz) device floats.  Plane (s, p),
 * p over the pairs (a, b) = (x,y) (x,z) (x,t) (y,z) (y,t) (z,t), is planes_host[6 s + p], channels-last [R_b, R_a, C]
 * with R_x = R_y = R_z = res_host[s] and R_t.  Each plane is sampled bilinearly as grid_sample(align_corners=True,
 * padding_mode='border'): pixel coordinate (x - lo) (R - 1) / (hi - lo) along a spatial axis and t (R_t - 1) along
 * time, clamped to [0, R - 1]; a indexes the columns (width), b the rows.
 *   out[f, n, s C + c] = prod_p sample_{s,p}(f, n)[c]   (out [F,N,S C]; computed as (s0 s1 s3) (s2 s4 s5)).
 * dghp_forward keeps nothing for the backward.
 * dghp_backward: grad_out [F,N,S C] -> grad_x [N,3] (NULL: not computed) and every plane's gradient
 *   (grad_planes_host, each written, not accumulated).  The coordinate gradient is torch's: 0 outside the box and
 *   on its faces.  The plane gradients are gathered through a stable sort of the samples by bilinear cell, without
 *   float atomics: bit-identical from run to run.  Workspace: dghp_backward_workspace (depends on F, N and the
 *   planes' shapes).
 * dghp_reg_forward: losses [3] = (tv, time_smooth, l1_time), each summed over its planes and the scales, for G
 *   [R_b, R_a, C]:
 *     tv          (spatial planes): mean_{i<R_b-1,j,c} (G[i+1,j,c] - G[i,j,c])^2 + mean_{i,j<R_a-1,c} (G[i,j+1,c] - G[i,j,c])^2
 *     time_smooth (time planes):    mean_{i<R_t-2,j,c} (G[i+2,j,c] - 2 G[i+1,j,c] + G[i,j,c])^2   (0 when R_t = 2)
 *     l1_time     (time planes):    mean |1 - G|
 *   The partial sums are added in a fixed order (bit-identical from run to run).  Workspace: dghp_reg_workspace.
 * dghp_reg_backward: grad_losses [3] (device) -> every plane's gradient (written, not accumulated); d|1 - G|/dG is 0
 *   at G = 1.
 * ------------------------------------------------------------------------ */
int dghp_forward(int F, int N, int S, int C, const int32_t* res_host, int R_t, const float* box, const float* x,
                 const float* t, const float* const* planes_host, float* out, void* stream);
int dghp_backward_workspace(int F, int N, int S, int C, const int32_t* res_host, int R_t, size_t* bytes);
int dghp_backward(int F, int N, int S, int C, const int32_t* res_host, int R_t, const float* box, const float* x,
                  const float* t, const float* const* planes_host, const float* grad_out, float* grad_x,
                  float* const* grad_planes_host, void* ws, size_t ws_bytes, void* stream);
int dghp_reg_workspace(int S, int C, const int32_t* res_host, int R_t, size_t* bytes);
int dghp_reg_forward(int S, int C, const int32_t* res_host, int R_t, const float* const* planes_host, float* losses,
                     void* ws, size_t ws_bytes, void* stream);
int dghp_reg_backward(int S, int C, const int32_t* res_host, int R_t, const float* const* planes_host,
                      const float* grad_losses, float* const* grad_planes_host, void* stream);

/* ------------------------------------------------------------------------
 * Multiresolution hash-grid field of (x, y, z, t) (Instant-NGP's HashGrid; Grid4D's space-time grids).  Device
 * pointers, except grids_host [G], res_host [L], tables_host and grad_tables_host [G] (host arrays).  Nothing
 * allocates or synchronises with the host.  DGM_E_BADARG before any device work for: G outside [1, 4], L outside
 * [1, 24], Fe not 2 or 4, log2_table outside [12, 24], R_t < 1, a level resolution outside [1, 2^24], grids_host
 * not strictly increasing kinds in [0, 3], F < 0, N < 0, L T Fe >= 2^31, F N G L Fe >= 2^31, N F >= 2^31, or a NULL
 * pointer (t may be NULL when no grid uses time); a workspace below its query: DGM_E_WORKSPACE.  F = 0 or N = 0
 * writes nothing (the backward zeroes the table gradients).
 *
 * The field: x [N,3] canonical positions, t [F,N] times, box [6] = (lo xyz, hi xyz) device floats.  Grid g is of
 * kind grids_host[g]: 0 = xyz, 1 = xyt, 2 = yzt, 3 = xzt, its three axes the coordinates the name spells, in order.
 * Its table tables_host[g] is [L, T, Fe] float32, T = 2^log2_table.  In float32, exactly as written (no fast math):
 *   u = (x - lo) / (hi - lo) per spatial axis, u = t on the time axis, then u = min(max(u, 0), 1);
 *   per axis of level l, with R = res_host[l] (spatial) or min(res_host[l], R_t) (time):
 *     p = u R (one rounded product), c = min(floor(p), R - 1), w = p - c (exact; 1 on the top face);
 *   the 8 nodes c + {0,1}^3 have slots
 *     dense level, (R_a + 1)(R_b + 1)(R_c + 1) <= T: i_a + (R_a + 1) (i_b + (R_b + 1) i_c)   (first axis fastest)
 *     hashed level, otherwise:  (i_a * 1 ^ i_b * 2654435761 ^ i_c * 805459861) mod T        (uint32 wrap-around)
 *   out[f, n, (g L + l) Fe + e] = sum over the 8 nodes of the trilinear weight times table_g[l, slot, e]
 *   (out [F,N,G L Fe]: grid, then level, then feature; the spatial grid is the same in every frame).
 * dghg_forward keeps nothing for the backward.
 * dghg_backward: grad_out [F,N,G L Fe] -> grad_x [N,3] (NULL: not computed) and every table's gradient
 *   (grad_tables_host, each written, not accumulated; a dense level's unused slots are 0).  dL/dx passes through each
 *   grid's spatial axes and is 0 where the unclamped u is outside [0, 1] (it passes at u = 0 and u = 1, as
 *   torch.clamp); t takes none.  The table gradients are sums in int64 fixed point at a power-of-two scale chosen
 *   per (grid, level) from max |grad_out|, so they are bit-identical from run to run; a non-finite grad_out in a
 *   (grid, level) makes that level's table gradient NaN.  Workspace: dghg_backward_workspace (G L T Fe 8 bytes and
 *   a little more; independent of F and N).
 * ------------------------------------------------------------------------ */
int dghg_forward(int F, int N, int G, const int32_t* grids_host, int L, int Fe, int log2_table,
                 const int32_t* res_host, int R_t, const float* box, const float* x, const float* t,
                 const float* const* tables_host, float* out, void* stream);
int dghg_backward_workspace(int F, int N, int G, const int32_t* grids_host, int L, int Fe, int log2_table,
                            const int32_t* res_host, int R_t, size_t* bytes);
int dghg_backward(int F, int N, int G, const int32_t* grids_host, int L, int Fe, int log2_table,
                  const int32_t* res_host, int R_t, const float* box, const float* x, const float* t,
                  const float* const* tables_host, const float* grad_out, float* grad_x,
                  float* const* grad_tables_host, void* ws, size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DGMESH_B200_H_ */
