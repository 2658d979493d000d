// Shared device/host helpers for libskd_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>

namespace skd {

constexpr int kNumSMs = 132;           // H100 SXM; grids are sized in multiples of this

// thread-local last-error text, exposed through skd_last_error()
void set_error(const char* where, cudaError_t err);
void set_error_msg(const char* where, const char* msg);
// 1: TMA tensor maps use CU_TENSOR_MAP_DATA_TYPE_TFLOAT32, 0: FLOAT32 (wgmma then ignores the low 13 mantissa bits)
extern int g_tf32_tma_type;

// Reference convention (libs/src/bn.cu:244-249): every launcher returns 1 on success, 0 on a CUDA error.
extern unsigned long long g_kernel_launches;     // kernels this library launched (skd_kernel_launches())
inline int finish(const char* where, int kernels = 1) {
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) { set_error(where, err); return 0; }
  g_kernel_launches += (unsigned long long)kernels;
  return 1;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide sum of two values; result valid in every thread. `sh` must hold 64 floats.
__device__ __forceinline__ float2 block_sum2(float a, float b, float* sh) {
  a = warp_sum(a); b = warp_sum(b);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (lane == 0) { sh[wid] = a; sh[32 + wid] = b; }
  __syncthreads();
  a = lane < nw ? sh[lane] : 0.f;
  b = lane < nw ? sh[32 + lane] : 0.f;
  a = warp_sum(a); b = warp_sum(b);
  return make_float2(a, b);
}

__device__ __forceinline__ float4 ld_stream(const float4* p) {   // read-once data: bypass L1 allocation
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}

enum Act : int { ACT_NONE = 0, ACT_LEAKY = 1, ACT_ELU = 2, ACT_RELU = 3 };

__device__ __forceinline__ float act_fwd(float z, int act, float slope) {
  if (act == ACT_LEAKY) return z < 0.f ? z * slope : z;
  if (act == ACT_RELU) return fmaxf(z, 0.f);
  if (act == ACT_ELU) return z < 0.f ? expm1f(z) : z;
  return z;
}

}  // namespace skd
