// common.cuh -- shared device helpers + private workspace layouts (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ < 900)
#error "dgmesh_b200 is written for sm_90a (Hopper H100)"
#endif

#define DGM_NUM_SMS 132          // H100 SXM
#define TILE_X 16                // reference BLOCK_X / BLOCK_Y (dgr/cuda_rasterizer/config.h:16-17)
#define TILE_Y 16
#define TILE_PIX (TILE_X * TILE_Y)

namespace dgm {

// ---------------------------------------------------------------- layouts --
template <typename T>
__host__ __device__ inline T* carve(char*& p, size_t count) {
  uintptr_t a = (reinterpret_cast<uintptr_t>(p) + 127) & ~uintptr_t(127);
  T* r = reinterpret_cast<T*>(a);
  p = reinterpret_cast<char*>(r + count);
  return r;
}

// per-Gaussian state (plays the role of GeometryState, rasterizer_impl.h:30-45)
struct GeomWS {
  float* depths;          // [P]
  uint8_t* clamped;       // [P,3]
  int* radii;             // [P]
  float2* means2D;        // [P]
  float* cov3D;           // [P,6]
  float4* conic_opacity;  // [P]
  float* rgb;             // [P,3]
  uint32_t* tiles_touched;// [P]
  float4* grad_acc;       // [P,3] backward accumulators: {m2d.x,m2d.y,con.x,con.y},{con.w,opac,r,g},{b,-,-,-}
  __host__ __device__ static GeomWS from(char* base, size_t P, size_t* bytes = nullptr) {
    char* p = base;
    GeomWS g;
    g.depths = carve<float>(p, P);
    g.clamped = carve<uint8_t>(p, 3 * P);
    g.radii = carve<int>(p, P);
    g.means2D = carve<float2>(p, P);
    g.cov3D = carve<float>(p, 6 * P);
    g.conic_opacity = carve<float4>(p, P);
    g.rgb = carve<float>(p, 3 * P);
    g.tiles_touched = carve<uint32_t>(p, P);
    g.grad_acc = carve<float4>(p, 3 * P);
    if (bytes) *bytes = size_t(p - base) + 128;
    return g;
  }
};

// per-image state (ImageState, rasterizer_impl.h:47-54) + binning tables
struct ImgWS {
  float* final_T;        // [H*W]
  uint32_t* n_contrib;   // [H*W]
  uint2* ranges;         // [T]
  uint32_t* hist;        // [T, 256] (tile, depth bucket) counts -> block offsets -> block ends
  uint32_t* depth_range; // [8]  {~min depth bits, max depth bits} of the visible set (follows hist: one memset)
  uint32_t* tile_total;  // [T] instances per tile
  uint32_t* tile_order;  // [T] tile ids, longest list first (launch order of the blend kernels)
  uint32_t* scan_flags;  // [8]  completion ticket of tile_scan_kernel
  __host__ __device__ static ImgWS from(char* base, size_t npix, size_t T, size_t* bytes = nullptr) {
    char* p = base;
    ImgWS w;
    w.final_T = carve<float>(p, npix);
    w.n_contrib = carve<uint32_t>(p, npix);
    w.ranges = carve<uint2>(p, T);
    w.hist = carve<uint32_t>(p, T * 256 + 8);
    w.depth_range = w.hist + T * 256;
    w.tile_total = carve<uint32_t>(p, T);
    w.tile_order = carve<uint32_t>(p, T);
    w.scan_flags = carve<uint32_t>(p, 8);
    if (bytes) *bytes = size_t(p - base) + 128;
    return w;
  }
};

// per-instance state (BinningState, rasterizer_impl.h:56-64).  Instead of a
// global 64-bit radix sort the tile segments are sorted independently; the
// sorted segments are additionally materialised as packed, streamable records
// so that both blend kernels read them with linear bulk copies.
struct BinWS {
  unsigned long long* keys;  // [R] unsorted (depth_bits<<32 | gaussian) inside each tile segment
  uint32_t* point_list;      // [R] sorted gaussian ids (== reference point_list)
  float4* inst_geo;          // [R]   {mean2D.x, mean2D.y, 2 ln(255 o) cull level, -}
  float4* inst_attr;         // [2R]  {conic.x, conic.y, conic.z, opacity}, {r, g, b, id bits}
  __host__ __device__ static BinWS from(char* base, size_t R, size_t* bytes = nullptr) {
    char* p = base;
    BinWS b;
    b.keys = carve<unsigned long long>(p, R);
    b.point_list = carve<uint32_t>(p, R);
    b.inst_geo = carve<float4>(p, R);
    b.inst_attr = carve<float4>(p, 2 * R);
    if (bytes) *bytes = size_t(p - base) + 128;
    return b;
  }
};

// ------------------------------------------------------- mbarrier / TMA ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// 1-D TMA bulk copy global -> shared::cta, completion on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(smem_dst)),
      "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

__device__ __forceinline__ void tma_load_1d_u32(uint32_t smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_dst),
      "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// ------------------------------------------- programmatic dependent launch ----
// A kernel launched with launch_pdl() may become resident while its predecessor on the stream is
// still running; it must call pdl_wait() before reading anything the predecessor wrote (the wait
// returns once the predecessor grid has completed and its memory is visible).  pdl_launch() lets
// the NEXT kernel's CTAs be scheduled as this grid's last wave drains.  Both are no-ops for a
// kernel launched the ordinary way.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// vector float reductions to global memory (sm_90+): one L2 atomic transaction for 4 floats
__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d)
               : "memory");
}
__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {  // 8-byte aligned
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}


#ifdef __CUDACC__
// host: launch `k` with the programmatic-stream-serialization attribute (pdl != 0) or plainly
extern int g_pdl;  // api.cu; DGMESH_B200_PDL=0 disables
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*k)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = g_pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, k, KArgs(args)...);
}
#endif

// One-time per-DEVICE initialisation (constant / global tables, function attributes are per device: a process
// that touches a second GPU must repeat them there).  `done` is a bit mask of device ordinals; returns true the
// first time it is called on the current device.  Not atomic: a benign race repeats an idempotent upload.
inline bool once_per_device(unsigned long long& done) {
  int d = 0;
  cudaGetDevice(&d);
  if (d < 0 || d >= 64) return true;
  if ((done >> d) & 1ull) return false;
  done |= 1ull << d;
  return true;
}

}  // namespace dgm
