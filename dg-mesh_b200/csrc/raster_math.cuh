// raster_math.cuh -- per-Gaussian projection math shared by forward and backward.
//
// The expressions below follow the reference's evaluation ORDER (not its code):
// tile keys and sort indices must be bit-exact (SURVEY.md 7 "Hard parts"), and
// under nvcc's default -fmad=true the FMA contraction pattern is decided by the
// shape of each expression.  3x3 products are therefore written as the same
// left-associated three-term sums glm uses (column-major, m[col][row]) including
// the structurally-zero terms; see DESIGN.md "bit-exactness".
#pragma once
#include "common.cuh"

namespace dgm {

// spherical-harmonics constants (values of the real SH basis, degree <= 3)
__device__ const float kSH0 = 0.28209479177387814f;
__device__ const float kSH1 = 0.4886025119029199f;
__device__ const float kSH2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                  -1.0925484305920792f, 0.5462742152960396f};
__device__ const float kSH3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                                  0.3731763325901154f,  -0.4570457994644658f, 1.445305721320277f,
                                  -0.5900435899266435f};

// two-lane fp32 arithmetic with explicit rounding (one rounded operation per lane; Hopper has no
// packed fp32x2 instructions, so each lane is a scalar FADD / FMUL / FFMA that cannot be re-associated)
__device__ __forceinline__ float2 add2_rn(float2 a, float2 b) {
  return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
}
__device__ __forceinline__ float2 mul2_rn(float2 a, float2 b) {
  return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
}
__device__ __forceinline__ float2 fma2_rn(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

// The quadratic form of two blend records A, B (geo: mean in .xy; con: conic in .xyz) at the pixel (-npx, -npy),
// side by side.  The operation sequence (which product is fused into which FMA) is the one nvcc emits for the
// reference's renderCUDA (forward.cu:330-352), written with explicit-rounding intrinsics so it cannot be
// re-associated: every blend kernel and side pass sees the same value, = -power (exactly).
__device__ __forceinline__ float2 pair_npow(float4 geA, float4 geB, float4 coA, float4 coB, float2 npx2,
                                            float2 npy2) {
  const float2 dx = add2_rn(make_float2(geA.x, geB.x), npx2);
  const float2 dy = add2_rn(make_float2(geA.y, geB.y), npy2);
  float2 m1 = mul2_rn(dy, make_float2(coA.z, coB.z));
  const float2 m2 = mul2_rn(dx, make_float2(coA.x, coB.x));
  m1 = mul2_rn(dy, m1);
  const float2 sq = fma2_rn(dx, m2, m1);
  float2 m3 = mul2_rn(dx, make_float2(coA.y, coB.y));
  m3 = mul2_rn(dy, m3);
  return fma2_rn(sq, make_float2(0.5f, 0.5f), m3);
}

struct Mat3 {  // column-major like glm: c[col][row]
  float c[3][3];
};

__device__ __forceinline__ Mat3 mat3_mul(const Mat3& a, const Mat3& b) {
  Mat3 r;
#pragma unroll
  for (int col = 0; col < 3; ++col)
#pragma unroll
    for (int row = 0; row < 3; ++row)
      r.c[col][row] = a.c[0][row] * b.c[col][0] + a.c[1][row] * b.c[col][1] + a.c[2][row] * b.c[col][2];
  return r;
}
__device__ __forceinline__ Mat3 mat3_T(const Mat3& a) {
  Mat3 r;
#pragma unroll
  for (int col = 0; col < 3; ++col)
#pragma unroll
    for (int row = 0; row < 3; ++row) r.c[col][row] = a.c[row][col];
  return r;
}

// viewmatrix / projmatrix are stored transposed (row-vector convention) and read
// column-major: auxiliary.h:58-99
__device__ __forceinline__ float3 xform4x3(const float3& p, const float* m) {
  return make_float3(m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12],
                     m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13],
                     m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14]);
}
__device__ __forceinline__ float4 xform4x4(const float3& p, const float* m) {
  return make_float4(m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12],
                     m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13],
                     m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14],
                     m[3] * p.x + m[7] * p.y + m[11] * p.z + m[15]);
}
__device__ __forceinline__ float3 xform_vec4x3_T(const float3& p, const float* m) {
  return make_float3(m[0] * p.x + m[1] * p.y + m[2] * p.z, m[4] * p.x + m[5] * p.y + m[6] * p.z,
                     m[8] * p.x + m[9] * p.y + m[10] * p.z);
}

// NDC -> pixel; evaluated in double exactly like auxiliary.h:41-44 (double literals)
__device__ __forceinline__ float ndc_to_pix(float v, int S) { return ((v + 1.0) * S - 1.0) * 0.5; }

// tile rectangle touched by a disc of integer radius (auxiliary.h:46-56)
__device__ __forceinline__ void tile_rect(const float2 p, int max_radius, uint2& rmin, uint2& rmax,
                                          unsigned gx, unsigned gy) {
  rmin.x = min(gx, max((int)0, (int)((p.x - max_radius) / TILE_X)));
  rmin.y = min(gy, max((int)0, (int)((p.y - max_radius) / TILE_Y)));
  rmax.x = min(gx, max((int)0, (int)((p.x + max_radius + TILE_X - 1) / TILE_X)));
  rmax.y = min(gy, max((int)0, (int)((p.y + max_radius + TILE_Y - 1) / TILE_Y)));
}

// rotation (from the UN-normalised quaternion, forward.cu:126-139) scaled by S -> M = S*R
__device__ __forceinline__ void quat_to_R(const float4 q, Mat3& R) {
  const float r = q.x, x = q.y, y = q.z, z = q.w;
  R.c[0][0] = 1.f - 2.f * (y * y + z * z);
  R.c[0][1] = 2.f * (x * y - r * z);
  R.c[0][2] = 2.f * (x * z + r * y);
  R.c[1][0] = 2.f * (x * y + r * z);
  R.c[1][1] = 1.f - 2.f * (x * x + z * z);
  R.c[1][2] = 2.f * (y * z - r * x);
  R.c[2][0] = 2.f * (x * z - r * y);
  R.c[2][1] = 2.f * (y * z + r * x);
  R.c[2][2] = 1.f - 2.f * (x * x + y * y);
}

// world-space covariance from scale + quaternion (forward.cu:118-152): Sigma = (S R)^T (S R)
__device__ __forceinline__ void cov3d_from_scale_rot(const float3 scale, float mod, const float4 rot, float* cov3D) {
  Mat3 S;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) S.c[i][j] = (i == j) ? 1.0f : 0.0f;
  S.c[0][0] = mod * scale.x;
  S.c[1][1] = mod * scale.y;
  S.c[2][2] = mod * scale.z;
  Mat3 R;
  quat_to_R(rot, R);
  Mat3 M = mat3_mul(S, R);
  Mat3 Sigma = mat3_mul(mat3_T(M), M);
  cov3D[0] = Sigma.c[0][0];
  cov3D[1] = Sigma.c[0][1];
  cov3D[2] = Sigma.c[0][2];
  cov3D[3] = Sigma.c[1][1];
  cov3D[4] = Sigma.c[1][2];
  cov3D[5] = Sigma.c[2][2];
}

// EWA projection pieces shared by forward (cov2D) and backward (its gradient):
// clamped view-space mean t, T = W*J, Vrk (forward.cu:74-113, backward.cu:144-201)
struct EwaFrame {
  float3 t;          // clamped view-space position
  float txtz, tytz;  // unclamped ratios (for the gradient mask)
  Mat3 W, T, Vrk;
};
__device__ __forceinline__ void ewa_frame(const float3& mean, float fx, float fy, float tan_fovx, float tan_fovy,
                                          const float* cov3D, const float* view, EwaFrame& f) {
  float3 t = xform4x3(mean, view);
  const float limx = 1.3f * tan_fovx;
  const float limy = 1.3f * tan_fovy;
  f.txtz = t.x / t.z;
  f.tytz = t.y / t.z;
  t.x = min(limx, max(-limx, f.txtz)) * t.z;
  t.y = min(limy, max(-limy, f.tytz)) * t.z;
  f.t = t;
  Mat3 J;
  J.c[0][0] = fx / t.z;
  J.c[0][1] = 0.0f;
  J.c[0][2] = -(fx * t.x) / (t.z * t.z);
  J.c[1][0] = 0.0f;
  J.c[1][1] = fy / t.z;
  J.c[1][2] = -(fy * t.y) / (t.z * t.z);
  J.c[2][0] = 0;
  J.c[2][1] = 0;
  J.c[2][2] = 0;
  f.W.c[0][0] = view[0];
  f.W.c[0][1] = view[4];
  f.W.c[0][2] = view[8];
  f.W.c[1][0] = view[1];
  f.W.c[1][1] = view[5];
  f.W.c[1][2] = view[9];
  f.W.c[2][0] = view[2];
  f.W.c[2][1] = view[6];
  f.W.c[2][2] = view[10];
  f.T = mat3_mul(f.W, J);
  f.Vrk.c[0][0] = cov3D[0];
  f.Vrk.c[0][1] = cov3D[1];
  f.Vrk.c[0][2] = cov3D[2];
  f.Vrk.c[1][0] = cov3D[1];
  f.Vrk.c[1][1] = cov3D[3];
  f.Vrk.c[1][2] = cov3D[4];
  f.Vrk.c[2][0] = cov3D[2];
  f.Vrk.c[2][1] = cov3D[4];
  f.Vrk.c[2][2] = cov3D[5];
}
// cov2D = T^T Vrk^T T, plus the 0.3 px low-pass on the diagonal; returns (xx, xy, yy)
__device__ __forceinline__ float3 ewa_cov2d(const EwaFrame& f) {
  Mat3 cov = mat3_mul(mat3_mul(mat3_T(f.T), mat3_T(f.Vrk)), f.T);
  cov.c[0][0] += 0.3f;
  cov.c[1][1] += 0.3f;
  return make_float3(cov.c[0][0], cov.c[0][1], cov.c[1][1]);
}

// view-dependent colour from SH (forward.cu:20-71).  sh points at this Gaussian's
// [M,3] coefficients.  clamped[3] receives the "negative before clamp" flags.
__device__ __forceinline__ float3 sh_to_rgb(int deg, const float3 pos, const float3 campos, const float* sh,
                                            bool* clamped) {
  float3 dir = make_float3(pos.x - campos.x, pos.y - campos.y, pos.z - campos.z);
  {
    const float tx = dir.x * dir.x, ty = dir.y * dir.y, tz = dir.z * dir.z;
    const float len = sqrtf(tx + ty + tz);
    dir.x = dir.x / len;
    dir.y = dir.y / len;
    dir.z = dir.z / len;
  }
  float res[3];
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    float r = kSH0 * sh[0 * 3 + ch];
    if (deg > 0) {
      const float x = dir.x, y = dir.y, z = dir.z;
      r = r - kSH1 * y * sh[1 * 3 + ch] + kSH1 * z * sh[2 * 3 + ch] - kSH1 * x * sh[3 * 3 + ch];
      if (deg > 1) {
        const float xx = x * x, yy = y * y, zz = z * z;
        const float xy = x * y, yz = y * z, xz = x * z;
        r = r + kSH2[0] * xy * sh[4 * 3 + ch] + kSH2[1] * yz * sh[5 * 3 + ch] +
            kSH2[2] * (2.0f * zz - xx - yy) * sh[6 * 3 + ch] + kSH2[3] * xz * sh[7 * 3 + ch] +
            kSH2[4] * (xx - yy) * sh[8 * 3 + ch];
        if (deg > 2) {
          r = r + kSH3[0] * y * (3.0f * xx - yy) * sh[9 * 3 + ch] + kSH3[1] * xy * z * sh[10 * 3 + ch] +
              kSH3[2] * y * (4.0f * zz - xx - yy) * sh[11 * 3 + ch] +
              kSH3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * sh[12 * 3 + ch] +
              kSH3[4] * x * (4.0f * zz - xx - yy) * sh[13 * 3 + ch] + kSH3[5] * z * (xx - yy) * sh[14 * 3 + ch] +
              kSH3[6] * x * (xx - 3.0f * yy) * sh[15 * 3 + ch];
        }
      }
    }
    r += 0.5f;
    clamped[ch] = (r < 0);
    res[ch] = fmaxf(r, 0.0f);
  }
  return make_float3(res[0], res[1], res[2]);
}

// Exact test "can this Gaussian reach alpha >= 1/255 on any pixel of the block [bx0,bx1]x[by0,by1]?":
// minimise q(d) = a dx^2 + 2 b dx dy + c dy^2 (= -2 power) over the box of offsets d = g - p.  The
// minimiser of a convex quadratic with its centre outside the box lies on an edge facing the centre,
// so at most two clamped 1-D minimisations are needed.  geo.z holds 2*(ln(255 o) + margin)
// (negative: never visible; +inf: degenerate conic, never culled); the margin (0.02 on tau) dwarfs
// the fp32 rounding of the blend, so a culled record is one the reference `continue`s over.
__device__ __forceinline__ bool cull_keep(const float4 geo, const float4 con_o, float bx0, float bx1, float by0,
                                          float by1) {
  const float X0 = geo.x - bx1, X1 = geo.x - bx0, Y0 = geo.y - by1, Y1 = geo.y - by0;
  const float ex = fminf(fmaxf(0.0f, X0), X1), ey = fminf(fmaxf(0.0f, Y0), Y1);  // box point nearest the centre
  const float a = con_o.x, b = con_o.y, c = con_o.z;
  // edge dx = ex: dy* = clamp(-b ex / c);  edge dy = ey: dx* = clamp(-b ey / a)
  const float dy1 = fminf(fmaxf(__fdividef(-b * ex, c), Y0), Y1);
  const float dx2 = fminf(fmaxf(__fdividef(-b * ey, a), X0), X1);
  const float q1 = a * ex * ex + 2.0f * b * ex * dy1 + c * dy1 * dy1;
  const float q2 = a * dx2 * dx2 + 2.0f * b * dx2 * ey + c * ey * ey;
  // a facing edge exists only where the box does not straddle the centre on that axis
  float qmin = 0.0f;
  if (ex != 0.0f && ey != 0.0f) qmin = fminf(q1, q2);
  else if (ex != 0.0f) qmin = q1;
  else if (ey != 0.0f) qmin = q2;
  return !(qmin > geo.z);
}

// this Gaussian's SH coefficients -> registers (only the first ncoef*3 values are valid)
__device__ __forceinline__ void load_sh(const float* __restrict__ shs, size_t idx, int M, int ncoef, float* s) {
  const float* src = shs + idx * (size_t)M * 3;
  if (M == 16) {  // 192-byte records: 16-byte aligned vector loads, all independent
    const float4* v = reinterpret_cast<const float4*>(src);
    const int nv = (ncoef * 3 + 3) >> 2;
#pragma unroll
    for (int i = 0; i < 12; ++i) {
      if (i < nv) {
        const float4 q = __ldg(v + i);
        s[4 * i + 0] = q.x;
        s[4 * i + 1] = q.y;
        s[4 * i + 2] = q.z;
        s[4 * i + 3] = q.w;
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < 48; ++i)
      if (i < ncoef * 3) s[i] = __ldg(src + i);
  }
}

}  // namespace dgm
