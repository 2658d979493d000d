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

// scipy.ndimage.zoom(order=1, prefilter=False, mode='constant') along one axis (ohem.cu's threshold grid, eval.cu's multi-scale
// image): ratio (in - 1) / (out - 1) first (1 for a single output point), source coordinate o * ratio in double, both
// neighbours and their weights.  A coordinate past in - 1 -- rounding can put the last output point there, e.g.
// 767 * (1023 / 767) = 1023.0000000000001 -- lies outside the input, and mode 'constant' reads 0 for it.
struct ZoomAxis {
  double c, t, w0;     // coordinate, weight of i1 (c - i0), weight of i0 (1 - t)
  int i0, i1;
  bool outside;
};
__host__ __device__ __forceinline__ double zoom_ratio(int n_in, int n_out) {
  return n_out > 1 ? (double)(n_in - 1) / (double)(n_out - 1) : 1.0;
}
__device__ __forceinline__ ZoomAxis zoom_axis(int o, double ratio, int n_in) {
  ZoomAxis a;
  a.c = __dmul_rn((double)o, ratio);
  a.outside = a.c > (double)(n_in - 1);
  a.i0 = (int)floor(a.c);
  a.i1 = min(a.i0 + 1, n_in - 1);
  a.t = __dsub_rn(a.c, (double)a.i0);
  a.w0 = __dsub_rn(1.0, a.t);
  return a;
}
// value * w_y * w_x, summed neighbour by neighbour in scipy's order (NI_ZoomShift); no FMA contraction
__device__ __forceinline__ double zoom_lerp(double p00, double p01, double p10, double p11, const ZoomAxis& y, const ZoomAxis& x) {
  double a = __dmul_rn(__dmul_rn(p00, y.w0), x.w0);
  a = __dadd_rn(a, __dmul_rn(__dmul_rn(p01, y.w0), x.t));
  a = __dadd_rn(a, __dmul_rn(__dmul_rn(p10, y.t), x.w0));
  a = __dadd_rn(a, __dmul_rn(__dmul_rn(p11, y.t), x.t));
  return a;
}

// bilinear (align_corners) value of one plane p (pixel stride sp, h x w) at (y, x) of the up-/down-sampled grid, ry = (h - 1) / (H - 1):
// ATen's source-index rule (eval.cu's score accumulation, espnet.cu's teacher resample)
__device__ __forceinline__ float up_at(const float* __restrict__ p, long long sp, int h, int w, float ry, float rx, int y, int x) {
  const float fy = y * ry, fx = x * rx;
  const int y0 = min((int)fy, h - 1), x0 = min((int)fx, w - 1);
  const int y1i = min(y0 + 1, h - 1), x1i = min(x0 + 1, w - 1);
  const float ly = fy - y0, lx = fx - x0;
  const float v00 = __ldg(p + ((long long)y0 * w + x0) * sp), v01 = __ldg(p + ((long long)y0 * w + x1i) * sp);
  const float v10 = __ldg(p + ((long long)y1i * w + x0) * sp), v11 = __ldg(p + ((long long)y1i * w + x1i) * sp);
  return (1.f - ly) * ((1.f - lx) * v00 + lx * v01) + ly * ((1.f - lx) * v10 + lx * v11);
}

// bilinear (align_corners) source index pair and weights of output coordinate dst: v = l0 * src[i0] + l1 * src[i1], with ATen's
// area_pixel_compute_source_index(align_corners=True): src = scale * dst, scale = (in - 1) / (out - 1)
struct Bilin { int i0, i1; float l0, l1; };
__device__ __forceinline__ Bilin bilin(int dst, float scale, int in) {
  const float src = scale * (float)dst;
  Bilin b;
  b.i0 = (int)src; if (b.i0 > in - 1) b.i0 = in - 1;
  b.i1 = b.i0 + (b.i0 < in - 1 ? 1 : 0);
  b.l1 = src - (float)b.i0; b.l0 = 1.f - b.l1;
  return b;
}

// softmax probability of class lab at the upsampled pixel (by, bx) of logits L (strides sn, sc, sp over image, class, pixel; w source
// columns), with exactly the DSN row kernel's arithmetic (losses.cu): the two source rows blended first, then the two columns, __expf,
// times the reciprocal of the sum.  OHEM ranks these values on its threshold grid (ohem.cu) and the row kernel keeps a pixel when its
// value is <= the threshold: where a grid point lies on a pixel, both must compute the same bits, or the pixel that defines the
// threshold can come out above it and be dropped.
template <int CT>
__device__ __forceinline__ float up_label_prob(const float* __restrict__ L, long long sn, long long sc, long long sp, int n, int C,
                                               int w, Bilin by, Bilin bx, int lab) {
  const float* b0 = L + n * sn + (long long)by.i0 * w * sp;
  const float* b1 = L + n * sn + (long long)by.i1 * w * sp;
  const long long x0 = (long long)bx.i0 * sp, x1 = (long long)bx.i1 * sp;
  float v[CT];
  float m = -INFINITY;
#pragma unroll
  for (int c = 0; c < CT; ++c) if (c < C) {
    const long long o = (long long)c * sc;
    const float r0 = by.l0 * __ldg(b0 + x0 + o) + by.l1 * __ldg(b1 + x0 + o);
    const float r1 = by.l0 * __ldg(b0 + x1 + o) + by.l1 * __ldg(b1 + x1 + o);
    v[c] = bx.l0 * r0 + bx.l1 * r1;
    m = fmaxf(m, v[c]);
  }
  float z = 0.f, e = 0.f;
#pragma unroll
  for (int c = 0; c < CT; ++c) if (c < C) { v[c] = __expf(v[c] - m); z += v[c]; if (c == lab) e = v[c]; }
  return e * (1.f / z);
}

// Cityscapes label id -> train id (reference dataset/datasets.py:146-151, ids 0..33; everything else passes through).  The one
// copy of the table: augment.cu maps labels with it, skd_cityscapes_id_tables derives the reverse (train id -> label id) map
// that evaluation writes test-split predictions with.
#define SKD_CITYSCAPES_TRAINID {255, 255, 255, 255, 255, 255, 255, 0, 1, 255, 255, 2, 3, 4, 255, 255, 255, 5, 255, 6, 7, 8, 9, 10, \
                                11, 12, 13, 14, 15, 255, 255, 16, 17, 18}
constexpr int kCityscapesIds = 34;

enum Act : int { ACT_NONE = 0, ACT_LEAKY = 1, ACT_ELU = 2, ACT_RELU = 3 };

__device__ __forceinline__ float act_fwd(float z, int act, float slope) {
  if (act == ACT_LEAKY) return z < 0.f ? z * slope : z;
  if (act == ACT_RELU) return fmaxf(z, 0.f);
  if (act == ACT_ELU) return z < 0.f ? expm1f(z) : z;
  return z;
}

}  // namespace skd
