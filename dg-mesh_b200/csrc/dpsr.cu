// dpsr.cu -- Differentiable Poisson Surface Reconstruction (spectral solve), forward + backward.
//
// Reference: dgmesh/nvdiffrast_utils/dpsr.py:28-70 (DPSR.forward) and
// dgmesh/nvdiffrast_utils/dpsr_utils.py:25-197 (fftfreqs, spec_gaussian_filter, grid_interp,
// point_rasterize), which run ~25 PyTorch index / elementwise kernels around torch.fft and
// build an (N*24, 5) int64 index tensor per call.  Here:
//   scatter   one kernel: trilinear splat of the normals into ras[3,G,G,G] (fp32 atomics)
//   rfftn     cuFFT R2C, batch 3 (library call, as the north star specifies)
//   spectral  ONE pass: Gaussian filter x divergence x inverse Laplacian, DC = 0
//             (dpsr.py:41-52: ~10 elementwise kernels + a 289 MB intermediate)
//   irfftn    cuFFT C2R
//   gather    trilinear read-back at the points + block reduction of their mean
//   finalize  shift / scale (dpsr.py:57-69), optionally with the sign fix and threshold that
//             mesh_renderer applies afterwards (utils/renderer.py:163-168) fused in, which
//             removes the reference's host synchronisation on psr[0,0,0,0]
// Backward is the hand-derived adjoint of the same chain (the spectral solve is a real,
// shift-invariant linear map, so its adjoint is the solve with the conjugate transfer function).
//
// Index / weight arithmetic follows the reference's fp32 operation order (pts / cubesize with
// cubesize = fp32(1/G), floor / ceil / fmod) so that points on cell boundaries land in the same cells.
#include <cufft.h>

#include "common.cuh"
#include "dpsr_kernels.h"

namespace dgm {

// trilinear stencil of one point: base cell ind0, wrapped upper cell ind1, fractional weights
struct Stencil {
  int i0[3], i1[3];
  float w0[3], w1[3];  // weight of the lower / upper node along each axis
  float g0[3], g1[3];  // d w0 / d p, d w1 / d p  (torch: d|x|/dx = sign(x), 0 at x == 0)
};

__device__ __forceinline__ Stencil make_stencil(const float* p, int G, float cs) {
  Stencil s;
  const float size = (float)G;
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const float t = p[d] / cs;                    // dpsr_utils.py:158 (division by fp32(1/G))
    const float fl = floorf(t), ce = ceilf(t);
    s.i0[d] = (int)fl;
    s.i1[d] = (int)fmodf(ce, size);               // periodic wrap-around, :159
    // explicit roundings: an FMA-contracted p - fl*cs keeps the unrounded product and can flip the
    // SIGN of a ~1e-9 difference for points on grid nodes when 1/G is not a power of two
    const float xyz0 = __fmul_rn(fl, cs), xyz1 = __fmul_rn(fl + 1.0f, cs);
    const float d1 = __fsub_rn(p[d], xyz1), d0 = __fsub_rn(p[d], xyz0);
    s.w0[d] = fabsf(d1) / cs;                     // weight of node ind0 uses the OPPOSITE corner, :168-174
    s.w1[d] = fabsf(d0) / cs;
    const float inv_cs = 1.0f / cs;
    s.g0[d] = d1 > 0.f ? inv_cs : (d1 < 0.f ? -inv_cs : 0.f);
    s.g1[d] = d0 > 0.f ? inv_cs : (d0 < 0.f ? -inv_cs : 0.f);  // a point exactly on a node: 0, like autograd
    s.i0[d] = min(max(s.i0[d], 0), G - 1);        // points are clamped to (0,1) by the caller
  }
  return s;
}

// ------------------------------------------------------------------ scatter (point_rasterize)
__global__ void __launch_bounds__(256) dpsr_scatter_kernel(int N, int G, float cs, const float* __restrict__ V,
                                                           const float* __restrict__ Nrm, float* __restrict__ ras) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= N) return;
  const float pt[3] = {V[3 * p], V[3 * p + 1], V[3 * p + 2]};
  const float nv[3] = {Nrm[3 * p], Nrm[3 * p + 1], Nrm[3 * p + 2]};
  const Stencil s = make_stencil(pt, G, cs);
  const size_t G3 = (size_t)G * G * G;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int a = c >> 2, b = (c >> 1) & 1, d = c & 1;
    const int ix = a ? s.i1[0] : s.i0[0], iy = b ? s.i1[1] : s.i0[1], iz = d ? s.i1[2] : s.i0[2];
    const float w = (a ? s.w1[0] : s.w0[0]) * (b ? s.w1[1] : s.w0[1]) * (d ? s.w1[2] : s.w0[2]);
    const size_t cell = ((size_t)ix * G + iy) * G + iz;
    atomicAdd(&ras[cell], w * nv[0]);
    atomicAdd(&ras[G3 + cell], w * nv[1]);
    atomicAdd(&ras[2 * G3 + cell], w * nv[2]);
  }
}

// filter LUT: spec_gaussian_filter (dpsr_utils.py:58-64) depends on |omega|^2 = integer only;
// evaluated in fp64 and rounded to fp32 exactly like `spec_gaussian_filter(...).float()` (dpsr.py:21)
__global__ void dpsr_filter_lut_kernel(int n, int G, double sig, float* __restrict__ lut) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double dis = sqrt((double)i);
  const double a = sig * 2.0 * dis / (double)G;
  lut[i] = (float)exp(-0.5 * a * a);
}

__device__ __forceinline__ int fft_freq(int i, int G) { return (i < (G + 1) / 2) ? i : i - G; }  // np.fft.fftfreq(G, 1/G)

// ------------------------------------------------------------------ spectral solve (dpsr.py:41-52)
// spec[c][x][y][z] (z < G/2+1) -> phi_hat[x][y][z] = sum_c (-i w_c) G N_c / (Lap + 1e-6), DC = 0.
// adjoint != 0: in = D_hat (one field), out_c = conj(H_c) D_hat for the three channels.
__global__ void __launch_bounds__(256) dpsr_spectral_kernel(int G, const float* __restrict__ lut,
                                                            const float2* __restrict__ in, float2* __restrict__ out,
                                                            int adjoint) {
  const int Gh = G / 2 + 1;
  const size_t n = (size_t)G * G * Gh;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int z = (int)(i % Gh), y = (int)((i / Gh) % G), x = (int)(i / ((size_t)Gh * G));
  const int fx = fft_freq(x, G), fy = fft_freq(y, G), fz = z;  // rfftfreq: 0..G/2
  const float tw = (float)(2.0 * 3.141592653589793);           // omega *= 2*np.pi in fp32 (dpsr.py:44)
  const float wx = (float)fx * tw, wy = (float)fy * tw, wz = (float)fz * tw;
  const float g = lut[fx * fx + fy * fy + fz * fz];
  const float lap = -(wx * wx + wy * wy + wz * wz);
  const float den = lap + 1e-6f;
  const bool dc = (x == 0 && y == 0 && z == 0);
  if (!adjoint) {
    // DivN = sum_c (im_c, -re_c) * G * w_c  (i.e. -i w_c N_c), dpsr.py:47
    float re = 0.f, im = 0.f;
    const float w[3] = {wx, wy, wz};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float2 s = in[(size_t)c * n + i];
      re += (s.y * g) * w[c];
      im += (-(s.x * g)) * w[c];
    }
    out[i] = dc ? make_float2(0.f, 0.f) : make_float2(re / den, im / den);
  } else {
    // conj(H_c) = (+i w_c G) / den :  (re, im) -> (-im, re) * w_c G / den
    const float2 d = in[i];
    const float w[3] = {wx, wy, wz};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float k = dc ? 0.f : (w[c] * g) / den;
      out[(size_t)c * n + i] = make_float2(-d.y * k, d.x * k);
    }
  }
}

// ------------------------------------------------------------------ gather (grid_interp) + mean
__global__ void __launch_bounds__(256) dpsr_gather_mean_kernel(int N, int G, float cs, float inv_n3,
                                                               const float* __restrict__ V,
                                                               const float* __restrict__ phi_raw,
                                                               double* __restrict__ sum) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  float fv = 0.f;
  if (p < N) {
    const float pt[3] = {V[3 * p], V[3 * p + 1], V[3 * p + 2]};
    const Stencil s = make_stencil(pt, G, cs);
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const int a = c >> 2, b = (c >> 1) & 1, d = c & 1;
      const int ix = a ? s.i1[0] : s.i0[0], iy = b ? s.i1[1] : s.i0[1], iz = d ? s.i1[2] : s.i0[2];
      const float w = (a ? s.w1[0] : s.w0[0]) * (b ? s.w1[1] : s.w0[1]) * (d ? s.w1[2] : s.w0[2]);
      fv += (phi_raw[((size_t)ix * G + iy) * G + iz] * inv_n3) * w;
    }
  }
  double v = (double)fv;
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __shared__ double s_w[8];
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0;
    for (int w = 0; w < 8; ++w) t += s_w[w];
    atomicAdd(sum, t);
  }
}

// ------------------------------------------------------------------ finalize (dpsr.py:57-69)
// phi = irfftn scale * raw;  phi -= mean_p fv;  fv0 = phi[0,0,0];  out = -phi / |fv0| * 0.5
// mode 1 (mesh_renderer, utils/renderer.py:163-168): out = 0.5 * phi / fv0 - thres, which is the
// reference's   psr * sign(...) - density_thres   without reading psr[0,0,0,0] on the host.
// scal[0] = offset, scal[1] = fv0 (kept for the backward pass).
__global__ void __launch_bounds__(256) dpsr_finalize_kernel(size_t n, int N, float inv_n3,
                                                            const float* __restrict__ phi_raw,
                                                            const double* __restrict__ sum, int mode,
                                                            const float* __restrict__ thres, float* __restrict__ out,
                                                            float* __restrict__ scal) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const float offset = (float)(*sum / (double)N);
  const float fv0 = phi_raw[0] * inv_n3 - offset;
  if (i == 0) {
    scal[0] = offset;
    scal[1] = fv0;
  }
  if (i >= n) return;
  const float phi = phi_raw[i] * inv_n3 - offset;
  out[i] = mode ? (0.5f * phi / fv0 - thres[0]) : (-phi / fabsf(fv0) * 0.5f);
}

// ================================================================== backward
// 1. g = dL/dout -> dphi (grid), with the contributions through fv0 and through the mean shift.
//    out = k * phi1 with k = -0.5/|fv0| (mode 0) or 0.5/fv0 (mode 1); phi1 = phi - offset.
//    Two-pass: (a) reduce A = sum g_i, B = sum g_i phi1_i over i >= 1 ; (b) write dphi.
__global__ void __launch_bounds__(256) dpsr_bwd_reduce_kernel(size_t n, float inv_n3, const float* __restrict__ g,
                                                              const float* __restrict__ phi_raw,
                                                              const float* __restrict__ scal,
                                                              double* __restrict__ red) {
  const float offset = scal[0];
  double a = 0, b = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (i == 0) continue;  // out_0 is constant: see dpsr_bwd_dphi_kernel
    const float gi = g[i];
    a += gi;
    b += (double)gi * (double)(phi_raw[i] * inv_n3 - offset);
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  __shared__ double s_a[8], s_b[8];
  if ((threadIdx.x & 31) == 0) {
    s_a[threadIdx.x >> 5] = a;
    s_b[threadIdx.x >> 5] = b;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double ta = 0, tb = 0;
    for (int w = 0; w < 8; ++w) ta += s_a[w], tb += s_b[w];
    atomicAdd(&red[0], ta);
    atomicAdd(&red[1], tb);
  }
}

// dphi_i = k g_i for i >= 1, dphi_0 = dfv0; doffset = -(sum_i dphi_i); dthres = -sum g (mode 1).
// coef[0] = doffset / N  (the gradient every point's interpolated value receives).
// out_0 = k * fv0 is constant (-0.5 sign(fv0), or 0.5 - thres), so g_0 reaches nothing but thres: its direct term
// k g_0 and its term through fv0, dk g_0 fv0, cancel exactly.  Both are left out (A and B skip i = 0) instead of
// leaving the rounding of that cancellation in every gradient.
__global__ void __launch_bounds__(256) dpsr_bwd_dphi_kernel(size_t n, int N, const float* __restrict__ g,
                                                            const float* __restrict__ scal,
                                                            const double* __restrict__ red, int mode,
                                                            float* __restrict__ dphi, float* __restrict__ coef,
                                                            float* __restrict__ dthres) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const float fv0 = scal[1];
  const float k = mode ? 0.5f / fv0 : -0.5f / fabsf(fv0);
  // d out_i / d fv0 = phi1_i * dk/dfv0;  dk/dfv0 = -0.5/fv0^2 (mode 1),  +0.5 sign(fv0)/fv0^2 (mode 0)
  const float dk = mode ? -0.5f / (fv0 * fv0) : 0.5f * (fv0 > 0.f ? 1.f : -1.f) / (fv0 * fv0);
  const float dfv0 = (float)(red[1] * (double)dk);
  if (i == 0) {
    const double sum_dphi = (double)k * red[0] + (double)dfv0;
    coef[0] = (float)(-sum_dphi / (double)N);
    if (dthres) dthres[0] = mode ? (float)(-(red[0] + (double)g[0])) : 0.f;
  }
  if (i >= n) return;
  dphi[i] = i == 0 ? dfv0 : k * g[i];
}

// 2. every point's interpolated value fv_p gets the same gradient c = doffset/N:
//    dphi += c * w_pk at the stencil cells (atomics);  dV_p = c * sum_k (dw_pk/dV) phi[cell]
__global__ void __launch_bounds__(256) dpsr_bwd_interp_kernel(int N, int G, float cs, float inv_n3,
                                                              const float* __restrict__ V,
                                                              const float* __restrict__ phi_raw,
                                                              const float* __restrict__ coef,
                                                              float* __restrict__ dphi, float* __restrict__ dV) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= N) return;
  const float c = coef[0];
  const float pt[3] = {V[3 * p], V[3 * p + 1], V[3 * p + 2]};
  const Stencil s = make_stencil(pt, G, cs);
  float gv[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const int a = q >> 2, b = (q >> 1) & 1, d = q & 1;
    const int ix = a ? s.i1[0] : s.i0[0], iy = b ? s.i1[1] : s.i0[1], iz = d ? s.i1[2] : s.i0[2];
    const float ux = a ? s.w1[0] : s.w0[0], uy = b ? s.w1[1] : s.w0[1], uz = d ? s.w1[2] : s.w0[2];
    const size_t cell = ((size_t)ix * G + iy) * G + iz;
    atomicAdd(&dphi[cell], c * (ux * uy * uz));
    const float ph = phi_raw[cell] * inv_n3;
    gv[0] += (a ? s.g1[0] : s.g0[0]) * uy * uz * ph;
    gv[1] += (b ? s.g1[1] : s.g0[1]) * ux * uz * ph;
    gv[2] += (d ? s.g1[2] : s.g0[2]) * ux * uy * ph;
  }
  dV[3 * p + 0] = c * gv[0];
  dV[3 * p + 1] = c * gv[1];
  dV[3 * p + 2] = c * gv[2];
}

// 3. adjoint of point_rasterize: dN_pc = sum_k w_pk dras_c[cell];  dV_p += sum_k sum_c dw_pk/dV N_pc dras_c[cell]
//    (dras holds the UNSCALED C2R output; inv_n3 applies the irfftn normalisation)
__global__ void __launch_bounds__(256) dpsr_bwd_points_kernel(int N, int G, float cs, float inv_n3,
                                                              const float* __restrict__ V,
                                                              const float* __restrict__ Nrm,
                                                              const float* __restrict__ dras,
                                                              float* __restrict__ dV, float* __restrict__ dN) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= N) return;
  const float pt[3] = {V[3 * p], V[3 * p + 1], V[3 * p + 2]};
  const float nv[3] = {Nrm[3 * p], Nrm[3 * p + 1], Nrm[3 * p + 2]};
  const Stencil s = make_stencil(pt, G, cs);
  const size_t G3 = (size_t)G * G * G;
  float gn[3] = {0.f, 0.f, 0.f}, gv[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const int a = q >> 2, b = (q >> 1) & 1, d = q & 1;
    const int ix = a ? s.i1[0] : s.i0[0], iy = b ? s.i1[1] : s.i0[1], iz = d ? s.i1[2] : s.i0[2];
    const float ux = a ? s.w1[0] : s.w0[0], uy = b ? s.w1[1] : s.w0[1], uz = d ? s.w1[2] : s.w0[2];
    const size_t cell = ((size_t)ix * G + iy) * G + iz;
    const float r0 = dras[cell] * inv_n3, r1 = dras[G3 + cell] * inv_n3, r2 = dras[2 * G3 + cell] * inv_n3;
    const float w = ux * uy * uz;
    gn[0] += w * r0;
    gn[1] += w * r1;
    gn[2] += w * r2;
    const float dot = nv[0] * r0 + nv[1] * r1 + nv[2] * r2;
    gv[0] += (a ? s.g1[0] : s.g0[0]) * uy * uz * dot;
    gv[1] += (b ? s.g1[1] : s.g0[1]) * ux * uz * dot;
    gv[2] += (d ? s.g1[2] : s.g0[2]) * ux * uy * dot;
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    dN[3 * p + c] = gn[c];
    dV[3 * p + c] += gv[c];
  }
}

// ------------------------------------------------------------------ host side
// B items: phi_raw, red and scal are per item (item k at k * G^3, 4 k, 8 k) and outlive the forward; the rest is
// scratch that the stages of one item use and the next item reuses.  B = 1 is the single-item layout.
DpsrWS DpsrWS::from(char* base, int G, size_t fft_bytes, int B, size_t* bytes) {
  char* p = base;
  DpsrWS w;
  const size_t G3 = (size_t)G * G * G, Gs = (size_t)G * G * (G / 2 + 1);
  w.ras = carve<float>(p, 3 * G3);        // normals grid (fwd) / dras (bwd)
  w.spec = carve<float2>(p, 3 * Gs);      // spectra of the three channels
  w.phi_hat = carve<float2>(p, Gs);       // solved field, half spectrum
  w.phi_raw = carve<float>(p, (size_t)B * G3);  // unscaled C2R output (kept for the backward pass)
  w.dphi = carve<float>(p, G3);
  w.lut = carve<float>(p, 3 * (size_t)(G / 2 + 1) * (G / 2 + 1) + 8);
  w.red = carve<double>(p, 4 * (size_t)B);  // [0] sum of fv (fwd);  [1..2] A, B (bwd)
  w.scal = carve<float>(p, 8 * (size_t)B);  // offset, fv0, coef
  w.fft_work = carve<char>(p, fft_bytes);
  if (bytes) *bytes = size_t(p - base) + 128;
  return w;
}

struct DpsrPlan {
  int G;
  cufftHandle r2c3, r2c1, c2r1, c2r3;
  size_t work;
};

int dpsr_plan_create(int G, void** out, size_t* work_bytes) {
  DpsrPlan* pl = new DpsrPlan();
  pl->G = G;
  int n[3] = {G, G, G};
  size_t ws[4] = {0, 0, 0, 0};
  cufftHandle* h[4] = {&pl->r2c3, &pl->r2c1, &pl->c2r1, &pl->c2r3};
  const cufftType ty[4] = {CUFFT_R2C, CUFFT_R2C, CUFFT_C2R, CUFFT_C2R};
  const int batch[4] = {3, 1, 1, 3};
  const int rdist = G * G * G, cdist = G * G * (G / 2 + 1);
  for (int i = 0; i < 4; ++i) {
    if (cufftCreate(h[i]) != CUFFT_SUCCESS) return -1;
    cufftSetAutoAllocation(*h[i], 0);  // the caller provides the work area
    const int idist = (ty[i] == CUFFT_R2C) ? rdist : cdist, odist = (ty[i] == CUFFT_R2C) ? cdist : rdist;
    if (cufftMakePlanMany(*h[i], 3, n, nullptr, 1, idist, nullptr, 1, odist, ty[i], batch[i], &ws[i]) != CUFFT_SUCCESS)
      return -1;
  }
  pl->work = ws[0];
  for (int i = 1; i < 4; ++i) pl->work = ws[i] > pl->work ? ws[i] : pl->work;
  *out = pl;
  if (work_bytes) *work_bytes = pl->work;
  return 0;
}

void dpsr_plan_destroy(void* plan) {
  DpsrPlan* pl = (DpsrPlan*)plan;
  if (!pl) return;
  cufftDestroy(pl->r2c3);
  cufftDestroy(pl->r2c1);
  cufftDestroy(pl->c2r1);
  cufftDestroy(pl->c2r3);
  delete pl;
}

size_t dpsr_plan_work(void* plan) { return ((DpsrPlan*)plan)->work; }
int dpsr_plan_res(void* plan) { return ((DpsrPlan*)plan)->G; }

static bool use(cufftHandle h, void* work, cudaStream_t s) {
  return cufftSetStream(h, s) == CUFFT_SUCCESS && cufftSetWorkArea(h, work) == CUFFT_SUCCESS;
}

// items are V[B,N,3], Nrm[B,N,3] -> out[B,G,G,G]; each item runs the whole chain on the shared scratch
cudaError_t launch_dpsr_forward(void* plan, int B, int N, double sig, const float* V, const float* Nrm, int mode,
                                const float* thres, float* out, void* ws, cudaStream_t s) {
  DpsrPlan* pl = (DpsrPlan*)plan;
  const int G = pl->G;
  DpsrWS w = DpsrWS::from((char*)ws, G, pl->work, B);
  const size_t G3 = (size_t)G * G * G, Gs = (size_t)G * G * (G / 2 + 1);
  const float cs = 1.0f / (float)G;  // torch: cubesize = 1.0 / size (fp32)
  const float inv_n3 = (float)(1.0 / (double)G3);
  const int nlut = 3 * (G / 2 + 1) * (G / 2 + 1);
  cudaMemsetAsync(w.red, 0, sizeof(double) * 4 * B, s);
  dpsr_filter_lut_kernel<<<(nlut + 255) / 256, 256, 0, s>>>(nlut, G, sig, w.lut);
  for (int k = 0; k < B; ++k) {
    const float *Vk = V + (size_t)k * N * 3, *Nk = Nrm + (size_t)k * N * 3;
    float* phi_raw = w.phi_raw + (size_t)k * G3;
    double* red = w.red + 4 * k;
    cudaMemsetAsync(w.ras, 0, sizeof(float) * 3 * G3, s);
    if (N > 0) dpsr_scatter_kernel<<<(N + 255) / 256, 256, 0, s>>>(N, G, cs, Vk, Nk, w.ras);
    if (!use(pl->r2c3, w.fft_work, s) || cufftExecR2C(pl->r2c3, w.ras, (cufftComplex*)w.spec) != CUFFT_SUCCESS)
      return cudaErrorUnknown;
    dpsr_spectral_kernel<<<(unsigned)((Gs + 255) / 256), 256, 0, s>>>(G, w.lut, w.spec, w.phi_hat, 0);
    if (!use(pl->c2r1, w.fft_work, s) || cufftExecC2R(pl->c2r1, (cufftComplex*)w.phi_hat, phi_raw) != CUFFT_SUCCESS)
      return cudaErrorUnknown;
    if (N > 0)
      dpsr_gather_mean_kernel<<<(N + 255) / 256, 256, 0, s>>>(N, G, cs, inv_n3, Vk, phi_raw, red);
    dpsr_finalize_kernel<<<(unsigned)((G3 + 255) / 256), 256, 0, s>>>(G3, N > 0 ? N : 1, inv_n3, phi_raw, red, mode,
                                                                      thres, out + (size_t)k * G3, w.scal + 8 * k);
  }
  return cudaGetLastError();
}

// g[B,G,G,G] -> dV[B,N,3], dN[B,N,3], dthres[B] (each item's own dL/dthres; may be NULL)
cudaError_t launch_dpsr_backward(void* plan, int B, int N, const float* V, const float* Nrm, int mode, const float* g,
                                 float* dV, float* dN, float* dthres, void* ws, cudaStream_t s) {
  DpsrPlan* pl = (DpsrPlan*)plan;
  const int G = pl->G;
  DpsrWS w = DpsrWS::from((char*)ws, G, pl->work, B);
  const size_t G3 = (size_t)G * G * G, Gs = (size_t)G * G * (G / 2 + 1);
  const float cs = 1.0f / (float)G;
  const float inv_n3 = (float)(1.0 / (double)G3);
  cudaMemsetAsync(w.red, 0, sizeof(double) * 4 * B, s);
  for (int k = 0; k < B; ++k) {
    const float *Vk = V + (size_t)k * N * 3, *Nk = Nrm + (size_t)k * N * 3, *gk = g + (size_t)k * G3;
    float *dVk = dV + (size_t)k * N * 3, *dNk = dN + (size_t)k * N * 3;
    const float* phi_raw = w.phi_raw + (size_t)k * G3;
    double* red = w.red + 4 * k;
    float* scal = w.scal + 8 * k;
    dpsr_bwd_reduce_kernel<<<592, 256, 0, s>>>(G3, inv_n3, gk, phi_raw, scal, red);
    dpsr_bwd_dphi_kernel<<<(unsigned)((G3 + 255) / 256), 256, 0, s>>>(G3, N > 0 ? N : 1, gk, scal, red, mode, w.dphi,
                                                                      scal + 2, dthres ? dthres + k : nullptr);
    if (N > 0)
      dpsr_bwd_interp_kernel<<<(N + 255) / 256, 256, 0, s>>>(N, G, cs, inv_n3, Vk, phi_raw, scal + 2, w.dphi, dVk);
    // adjoint spectral solve: rfftn(dphi) -> conj(H_c) -> irfftn per channel (into the ras buffer)
    if (!use(pl->r2c1, w.fft_work, s) || cufftExecR2C(pl->r2c1, w.dphi, (cufftComplex*)w.phi_hat) != CUFFT_SUCCESS)
      return cudaErrorUnknown;
    dpsr_spectral_kernel<<<(unsigned)((Gs + 255) / 256), 256, 0, s>>>(G, w.lut, w.phi_hat, w.spec, 1);
    if (!use(pl->c2r3, w.fft_work, s) || cufftExecC2R(pl->c2r3, (cufftComplex*)w.spec, w.ras) != CUFFT_SUCCESS)
      return cudaErrorUnknown;
    if (N > 0)
      dpsr_bwd_points_kernel<<<(N + 255) / 256, 256, 0, s>>>(N, G, cs, inv_n3, Vk, Nk, w.ras, dVk, dNk);
  }
  return cudaGetLastError();
}

}  // namespace dgm
