// mc_sweep.cuh -- the warp-per-brick sweep of a G^3 grid shared by marching cubes (mc.cu) and dual marching
// cubes (dmc.cu): brick geometry, the brick loader and the per-node classifier.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace dgm {

// corner of edge e = 4 * axis + combo with the lower index (MC_EDGE_LO of mc_tables.h, in closed form)
__device__ __forceinline__ int mc_edge_lo(int e) {
  const int axis = e >> 2, k = e & 3;
  return axis == 0 ? (k << 1) : (axis == 1 ? ((k & 1) | ((k & 2) << 1)) : k);
}

#define MC_WARPS 8  // bricks (warps) per CTA
#define MC_BJ 8     // j-rows per brick

struct McGeom {
  int G, spr, njb;   // grid size, k-chunks per row = ceil(G / 32), j-blocks per plane = ceil(G / MC_BJ)
  size_t nbricks;    // G * njb * spr
};
__host__ __device__ inline McGeom mc_geom(int G) {
  McGeom g;
  g.G = G;
  g.spr = (G + 31) / 32;
  g.njb = (G + MC_BJ - 1) / MC_BJ;
  g.nbricks = (size_t)G * g.njb * g.spr;
  return g;
}

// one lane's view of its brick: phi at (i + p, j0 + r, k) and at k + 1, r = 0..MC_BJ (out of range = 0)
struct McBrick {
  int i, j0, k;
  bool xi, zk, kin;
  float a[2][MC_BJ + 1], z[2][MC_BJ + 1];
};

__device__ __forceinline__ void mc_load_brick(const McGeom& g, size_t brick, unsigned lane,
                                              const float* __restrict__ phi, McBrick& B) {
  const int G = g.G;
  const int kc = (int)(brick % g.spr);
  const size_t t = brick / g.spr;
  B.j0 = (int)(t % g.njb) * MC_BJ;
  B.i = (int)(t / g.njb);
  B.k = kc * 32 + (int)lane;
  B.kin = B.k < G;
  B.xi = B.i + 1 < G;
  B.zk = B.k + 1 < G;
  const float* base = phi + ((size_t)B.i * G + B.j0) * G + B.k;
  const size_t sx = (size_t)G * G;
#pragma unroll
  for (int r = 0; r <= MC_BJ; ++r) {
    const bool jin = B.j0 + r < G;
    B.a[0][r] = (jin && B.kin) ? base[(size_t)r * G] : 0.f;
    B.a[1][r] = (jin && B.kin && B.xi) ? base[sx + (size_t)r * G] : 0.f;
  }
  // the k + 1 column: lanes 0..30 take their neighbour's value, lane 31 reads the next chunk's first element
#pragma unroll
  for (int r = 0; r <= MC_BJ; ++r) {
    const bool jin = B.j0 + r < G;
    float e0 = 0.f, e1 = 0.f;
    if (lane == 31 && jin && B.zk) {
      e0 = base[(size_t)r * G + 1];
      if (B.xi) e1 = base[sx + (size_t)r * G + 1];
    }
    const float n0 = __shfl_down_sync(0xffffffffu, B.a[0][r], 1), n1 = __shfl_down_sync(0xffffffffu, B.a[1][r], 1);
    B.z[0][r] = lane == 31 ? e0 : n0;
    B.z[1][r] = lane == 31 ? e1 : n1;
  }
}

// node r of the lane: owned-edge mask (bit a: the edge towards +axis a carries a vertex) and cell case
__device__ __forceinline__ void mc_classify(const McGeom& g, const McBrick& B, int r, float iso, unsigned& mask,
                                            unsigned& cs) {
  mask = cs = 0;
  const int j = B.j0 + r;
  if (!B.kin || j >= g.G) return;
  const bool yj = j + 1 < g.G;
  const float v0 = B.a[0][r], v1 = B.a[1][r], v2 = B.a[0][r + 1], v3 = B.a[1][r + 1];
  const float v4 = B.z[0][r], v5 = B.z[1][r], v6 = B.z[0][r + 1], v7 = B.z[1][r + 1];
  const bool s0 = v0 < iso;
  if (B.xi && ((v1 < iso) != s0)) mask |= 1;
  if (yj && ((v2 < iso) != s0)) mask |= 2;
  if (B.zk && ((v4 < iso) != s0)) mask |= 4;
  if (B.xi && yj && B.zk) {  // corner c = (i + (c & 1), j + ((c >> 1) & 1), k + (c >> 2))
    cs = (unsigned)s0 | ((unsigned)(v1 < iso) << 1) | ((unsigned)(v2 < iso) << 2) | ((unsigned)(v3 < iso) << 3) |
         ((unsigned)(v4 < iso) << 4) | ((unsigned)(v5 < iso) << 5) | ((unsigned)(v6 < iso) << 6) |
         ((unsigned)(v7 < iso) << 7);
  }
}

// the common case (>95 % of a 288^3 grid): every value the brick touches lies on one side of the level set --
// nothing to classify.  Lanes look at their own valid values (lane 31 also at its k + 1 column): neg / pos is set
// when one of them lies below / at or above iso.
__device__ __forceinline__ void mc_brick_sides(const McGeom& g, const McBrick& B, unsigned lane, float iso, bool& neg,
                                               bool& pos) {
  neg = pos = false;
#pragma unroll
  for (int r = 0; r <= MC_BJ; ++r) {
    const bool jin = B.j0 + r < g.G;
#pragma unroll
    for (int pl = 0; pl < 2; ++pl) {
      const bool ok = jin && B.kin && (pl == 0 || B.xi);
      const bool s = B.a[pl][r] < iso;
      neg |= ok && s;
      pos |= ok && !s;
      if (lane == 31) {
        const bool okz = jin && B.zk && (pl == 0 || B.xi);
        const bool sz = B.z[pl][r] < iso;
        neg |= okz && sz;
        pos |= okz && !sz;
      }
    }
  }
}

}  // namespace dgm
