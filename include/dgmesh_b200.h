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
 * frames (fully written, no zero-fill needed).  n_streams: 1..4 side streams.
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
 * and the autograd graph PyTorch builds through them.  Batch size 1 (what DG-Mesh uses).
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

/* ------------------------------------------------------------------------
 * Differentiable marching cubes.  Stands in for diso.DiffMC.__call__(grid, deform=None,
 * isovalue) as called at dgmesh/utils/renderer.py:171 and
 * dgmesh/scene/gaussian_model_dpsr_dynamic_anchor.py:704,851 (third-party package, not in the
 * reference tree: only the CONTRACT at the call sites is reproduced, see DESIGN.md).
 *   phi[G,G,G] fp32, iso  ->  verts[V,3] fp32 in [0,1]^3 (index/(G-1)), faces[F,3] int32
 * V and F are data dependent.  dgmc_count sweeps the grid once and writes totals[2] = {V, F} to a device
 * int32 pair and, when given, to a pinned device-mapped host pair (`totals_host`, e.g. dgm_notify_host) with
 * `totals_event` (a cudaEvent_t) recorded behind it; dgmc_emit writes up to V_cap vertices and F_cap faces
 * (bounds enforced on the device), so a caller may enqueue it OPTIMISTICALLY with the capacities of the previous
 * call before it knows V and F, wait for the event, and re-run dgmc_emit only if something did not fit -- the
 * drop-in Python layer does that; the reference's diso synchronises to size its outputs as well.
 * G <= 800 (face references are packed into int32).
 * dgmc_backward: dL_dverts[V,3] -> dL_dphi[G,G,G] (fully written); V as returned by dgmc_count.
 * ------------------------------------------------------------------------ */
int dgmc_workspace_size(int G, size_t* bytes);
int dgmc_count(int G, const float* phi, float iso, void* ws, size_t ws_bytes,
               int32_t* totals, int32_t* totals_host, void* totals_event, void* stream);
int dgmc_emit(int G, const float* phi, float iso, void* ws, size_t ws_bytes,
              float* verts, int64_t V_cap, int32_t* faces, int64_t F_cap, void* stream);
int dgmc_backward(int G, int V, const float* phi, float iso, void* ws, size_t ws_bytes,
                  const float* dL_dverts, float* dL_dphi, void* stream);

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
             const float* opacity_raw, float max_grad, float min_opacity, float extent, float percent_dense,
             int size_prune, float max_screen_size, void* ws, size_t ws_bytes, int32_t* counts, void* stream);
int dgd_split_stds(int P, const float* scaling_raw, void* ws, size_t ws_bytes, float* stds, void* stream);
int dgd_apply(int P, int n_fields, const DgdField* fields_host, const float* rotation_raw, const float* samples,
              void* ws, size_t ws_bytes, void* stream);

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
#define DGM_K_COUNT 16
int dgm_profile_enable(int on);
int dgm_profile_read(float* ms_host, int n);
/* dgm_profile_enable(2) = timeline mode: every rasterizer kernel launched afterwards (any stream,
 * including the internal streams of the _batch calls) is bracketed by timing events.
 * dgm_timeline_read synchronises the device and returns the number of launches recorded;
 * begin/end are milliseconds relative to the first recorded launch ("begin" = the launch reached
 * the front of its stream).  Diagnostic only (tools/batch_timeline.py). */
int dgm_timeline_read(float* begin_ms, float* end_ms, int* kernel_ids, int cap);

#ifdef __cplusplus
}
#endif
#endif /* DGMESH_B200_H_ */
