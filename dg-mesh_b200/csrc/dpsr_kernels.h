// dpsr_kernels.h -- host-side interface of dpsr.cu
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace dgm {
struct DpsrWS {
  float* ras;
  float2* spec;
  float2* phi_hat;
  float* phi_raw;
  float* dphi;
  float* lut;
  double* red;
  float* scal;
  char* fft_work;
  static DpsrWS from(char* base, int G, size_t fft_bytes, int B = 1, size_t* bytes = nullptr);
};
int dpsr_plan_create(int G, void** out, size_t* work_bytes);
void dpsr_plan_destroy(void* plan);
size_t dpsr_plan_work(void* plan);
int dpsr_plan_res(void* plan);
// B items of N points each (1 <= B <= DPSR_MAX_BATCH); B = 1 is the single-item call
constexpr int DPSR_MAX_BATCH = 64;
cudaError_t launch_dpsr_forward(void* plan, int B, int N, double sig, const float* V, const float* Nrm, int mode,
                                const float* thres, float* out, void* ws, cudaStream_t s);
cudaError_t launch_dpsr_backward(void* plan, int B, int N, const float* V, const float* Nrm, int mode, const float* g,
                                 float* dV, float* dN, float* dthres, void* ws, cudaStream_t s);
}  // namespace dgm
