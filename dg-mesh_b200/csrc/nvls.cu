// nvls.cu -- the data-parallel exchange as our own kernel over NVLink / NVSwitch (SURVEY.md 8(e)).
//
// The one collective of the path is an all-reduce (sum) of ONE flat fp32 gradient buffer
// [canonical-Gaussian gradients || MLP gradients] (23.6 MB at C2, 60 MB at C4).  At these sizes NCCL's
// all-reduce is latency-bound.  With the buffer in symmetric memory mapped through an NVSwitch MULTICAST object,
// the reduction is done by the switch itself:
//     rank r owns slice r of the buffer:  v = multimem.ld_reduce.add(slice r)    -- the switch fetches the N
//                                                                                   replicas, adds them, returns one
//                                         multimem.st(slice r, v)                -- the switch writes v to all N
// so every GPU receives the buffer once and sends it once (2 x bytes / N per direction and rank), in ONE
// kernel bracketed by two flag barriers across the ranks (signal pads in the peers' symmetric memory).
// The caller (dg-mesh_b200/dp.py) allocates the buffer with torch's symmetric-memory allocator and passes
// the multicast address and the table of signal-pad addresses; nothing here allocates or synchronises.
#include "common.cuh"
#include "nvls_kernels.h"

namespace dgm {

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// Cross-rank barrier by ONE block: thread t < world raises flag (my rank) in rank t's pad and waits for flag (t)
// in its own.  Flags carry the epoch, so pads are never reset.  Our flags start NVLS_PAD_SKIP words into the pad:
// the first words belong to the allocator's own barrier channels.
__device__ __forceinline__ void rank_barrier(uint32_t* const* __restrict__ pads, int rank, int world, uint32_t epoch) {
  if ((int)threadIdx.x < world) {
    __threadfence_system();
    const int t = threadIdx.x;
    st_release_sys(pads[t] + NVLS_PAD_SKIP + rank, epoch);
    const uint32_t* mine = pads[rank] + NVLS_PAD_SKIP + t;
    while (ld_acquire_sys(mine) != epoch) {
    }
  }
  __syncthreads();
}

// per-device grid bookkeeping (one process drives one GPU; launches of this kernel must be stream-ordered with
// respect to each other -- one all-reduce at a time per device; epochs start at 1)
__device__ unsigned int g_nvls_go;       // epoch of the last start barrier block 0 has passed
__device__ unsigned int g_nvls_arrived;  // blocks that have finished their slice

__device__ __forceinline__ float4 mm_ld_reduce(const float* p) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ void mm_st(float* p, float4 v, float scale) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x * scale),
               "f"(v.y * scale), "f"(v.z * scale), "f"(v.w * scale)
               : "memory");
}

// Grid of many blocks (enough requests in flight to fill the links), but only block 0 talks to the peers at the
// start (the others wait for its local go flag) and only the LAST block to finish talks to them at the end, so
// nothing requires the blocks to be co-resident and the pads hold `world` flags whatever the grid.
__global__ void __launch_bounds__(512) nvls_allreduce_kernel(float* __restrict__ mc, size_t n_vec4,
                                                             uint32_t* const* __restrict__ pads, int rank, int world,
                                                             uint32_t epoch, float scale) {
  __shared__ unsigned int s_last;
  // start: everyone's local contributions are complete (stream order on each rank) and visible (system fence)
  if (blockIdx.x == 0) {
    rank_barrier(pads, rank, world, epoch);
    if (threadIdx.x == 0) {
      __threadfence();
      atomicExch(&g_nvls_go, epoch);
    }
  } else {
    if (threadIdx.x == 0) {
      while (*(volatile unsigned int*)&g_nvls_go != epoch) {
      }
      __threadfence();
    }
    __syncthreads();
  }
  const size_t per = (n_vec4 + world - 1) / world;
  const size_t lo = per * rank, hi = min(n_vec4, lo + per);
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  size_t i = lo + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + 3 * stride < hi; i += 4 * stride) {  // four requests in flight per thread
    float* p0 = mc + 4 * i;
    float* p1 = mc + 4 * (i + stride);
    float* p2 = mc + 4 * (i + 2 * stride);
    float* p3 = mc + 4 * (i + 3 * stride);
    const float4 v0 = mm_ld_reduce(p0), v1 = mm_ld_reduce(p1), v2 = mm_ld_reduce(p2), v3 = mm_ld_reduce(p3);
    mm_st(p0, v0, scale);
    mm_st(p1, v1, scale);
    mm_st(p2, v2, scale);
    mm_st(p3, v3, scale);
  }
  for (; i < hi; i += stride) mm_st(mc + 4 * i, mm_ld_reduce(mc + 4 * i), scale);
  // end: every slice has been written to every replica before anyone reads the result.  The last block of this
  // rank to finish tells the peers and waits for theirs; the kernel (hence the stream) completes after it.
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(&g_nvls_arrived, 1u) == gridDim.x - 1) ? 1u : 0u;
  __syncthreads();
  if (s_last) {
    if (threadIdx.x == 0) {
      g_nvls_arrived = 0;
      g_nvls_go = 0;  // every block of this launch is past the start: the next launch (any buffer, any epoch >= 1)
                      // must not find a stale go value equal to its own epoch
    }
    rank_barrier(pads, rank, world, epoch + 1);
  }
}

cudaError_t launch_nvls_allreduce(float* multicast_ptr, size_t n_floats, uint32_t* const* signal_pads_dev, int rank,
                                  int world, uint32_t epoch, float scale, int blocks, cudaStream_t s) {
  nvls_allreduce_kernel<<<blocks, 512, 0, s>>>(multicast_ptr, n_floats / 4, signal_pads_dev, rank, world, epoch, scale);
  return cudaGetLastError();
}

}  // namespace dgm
