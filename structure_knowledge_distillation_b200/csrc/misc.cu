// Error reporting + small weight-repacking kernels of libskd_b200.so.
#include <cstring>

#include "common.cuh"
#include "skd.h"
#include "sm90_ptx.cuh"

namespace skd {
static thread_local char g_err[256] = "";
int g_tf32_tma_type = 1;
unsigned long long g_kernel_launches = 0;
void set_error(const char* where, cudaError_t err) { snprintf(g_err, sizeof g_err, "%s: %s", where, cudaGetErrorString(err)); }
void set_error_msg(const char* where, const char* msg) { snprintf(g_err, sizeof g_err, "%s: %s", where, msg); }
}  // namespace skd

using namespace skd;

namespace {
__global__ void __launch_bounds__(256)
flip_transpose_kernel(int Cout, int Cin, int KH, int KW, const float* __restrict__ w, float* __restrict__ wt, int rnd) {
  const long long total = (long long)Cout * KH * KW * Cin;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    // i indexes wt[ci][kh][kw][co]
    const int co = (int)(i % Cout); long long r = i / Cout;
    const int kw = (int)(r % KW); r /= KW; const int kh = (int)(r % KH); const int ci = (int)(r / KH);
    float v = __ldg(w + (((size_t)co * KH + (KH - 1 - kh)) * KW + (KW - 1 - kw)) * Cin + ci);
    wt[i] = rnd ? ptx::round_tf32(v) : v;
  }
}
__global__ void __launch_bounds__(256) round_kernel(long long n, const float* __restrict__ s, float* __restrict__ d) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    d[i] = ptx::round_tf32(s[i]);
}
__global__ void __launch_bounds__(256) split_kernel(long long n4, const float4* __restrict__ s, float4* __restrict__ hi, float4* __restrict__ lo) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = s[i]; float4 h, l;
    h.x = ptx::round_tf32(v.x); h.y = ptx::round_tf32(v.y); h.z = ptx::round_tf32(v.z); h.w = ptx::round_tf32(v.w);
    l.x = ptx::round_tf32(v.x - h.x); l.y = ptx::round_tf32(v.y - h.y); l.z = ptx::round_tf32(v.z - h.z); l.w = ptx::round_tf32(v.w - h.w);
    if (hi) hi[i] = h;
    lo[i] = l;
  }
}
int blocks_for(long long n) { long long b = (n + 255) / 256; if (b > kNumSMs * 16) b = kNumSMs * 16; if (b < 1) b = 1; return (int)b; }
}  // namespace

extern "C" const char* skd_last_error(void) { return skd::g_err; }
extern "C" int skd_version(void) { return 90; }
extern "C" long long skd_kernel_launches(void) { return (long long)skd::g_kernel_launches; }
extern "C" void skd_set_tf32_tma_type(int use_tfloat32_type) { skd::g_tf32_tma_type = use_tfloat32_type ? 1 : 0; }

extern "C" int skd_weight_flip_transpose(int Cout, int Cin, int KH, int KW, const float* w, float* wt, int round_tf32, cudaStream_t st) {
  flip_transpose_kernel<<<blocks_for((long long)Cout * Cin * KH * KW), 256, 0, st>>>(Cout, Cin, KH, KW, w, wt, round_tf32);
  return finish("skd_weight_flip_transpose");
}
extern "C" int skd_round_tf32(long long n, const float* src, float* dst, cudaStream_t st) {
  if (n <= 0) return 1;
  round_kernel<<<blocks_for(n), 256, 0, st>>>(n, src, dst);
  return finish("skd_round_tf32");
}
extern "C" int skd_split_tf32(long long n, const float* src, float* hi, float* lo, cudaStream_t st) {
  // hi may be NULL: a TFLOAT32 tensor map rounds the original tensor to exactly that value on load, only lo must exist in memory
  if (n % 4 || ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(hi) | reinterpret_cast<uintptr_t>(lo)) & 15)) {
    set_error_msg("skd_split_tf32", "n must be a multiple of 4 and the pointers 16-byte aligned"); return 0;
  }
  if (n <= 0) return 1;
  split_kernel<<<blocks_for(n / 4), 256, 0, st>>>(n / 4, reinterpret_cast<const float4*>(src), reinterpret_cast<float4*>(hi), reinterpret_cast<float4*>(lo));
  return finish("skd_split_tf32");
}
