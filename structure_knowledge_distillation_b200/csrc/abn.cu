// Fused BatchNorm(+|w|+eps affine)+activation kernels for sm_90a.
//
// Part A: drop-in replacements for the reference's only native component, libs/src/bn.cu, behind the very same
//         raw-pointer C ABI (libs/src/bn.h:7-19): tensors are NCHW viewed as (N, C, S), fp32.
//         The reference launches ONE block per channel (bn.cu:237-300) -> at C=64 only 64 of 132 SMs work and the
//         variance costs a second full pass.  Here every channel is reduced by a thread-block CLUSTER whose CTAs
//         combine their partials through distributed shared memory: no workspace, no atomics, deterministic,
//         single pass (shifted sums), float4 streaming loads, grid = C x cluster >= 2 waves of 132 SMs.
// Part B: the NHWC (channels-last) kernels the H100 path itself uses between wgmma convolutions:
//         split-row partial statistics -> finalize (+running stats, +folded scale/shift) -> one fused
//         apply(+activation, +residual add, +Dropout2d channel mask) pass; and the matching backward.
#include <cooperative_groups.h>

#include "common.cuh"
#include "skd.h"
#include "sm90_ptx.cuh"

namespace cg = cooperative_groups;
using namespace skd;

namespace {

constexpr int kRedThreads = 512;
constexpr int kMaxCluster = 8;

__host__ int pick_cluster(int C, long long per_channel_elems) {
  // enough CTAs for >= 2 waves, but never split a channel finer than ~4K elements per CTA
  int want = (2 * kNumSMs + C - 1) / C;
  long long cap = per_channel_elems / 4096;
  if (cap < 1) cap = 1;
  int cl = want < (int)cap ? want : (int)cap;
  if (cl > kMaxCluster) cl = kMaxCluster;
  int p = 1;
  while (p * 2 <= cl) p *= 2;          // power of two keeps the grid a multiple of the cluster size
  return p;
}

template <typename Kernel, typename... Args>
cudaError_t launch_cluster(Kernel k, dim3 grid, dim3 block, int cluster, cudaStream_t stream, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = 0; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cluster; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, k, args...);
}

// Combine (a,b) partials of all CTAs of the cluster; valid in rank 0 only (thread 0).
__device__ __forceinline__ float2 cluster_sum2(float a, float b) {
  __shared__ float sh[64];
  __shared__ float2 part;
  cg::cluster_group cluster = cg::this_cluster();
  float2 r = block_sum2(a, b, sh);
  if (threadIdx.x == 0) part = r;
  cluster.sync();
  float2 tot = make_float2(0.f, 0.f);
  if (cluster.block_rank() == 0 && threadIdx.x == 0) {
    for (unsigned i = 0; i < cluster.num_blocks(); ++i) {
      const float2* rp = cluster.map_shared_rank(&part, i);
      float2 v = *rp;
      tot.x += v.x; tot.y += v.y;
    }
  }
  cluster.sync();                       // keep every CTA's smem alive until rank 0 has read it
  return tot;
}

// ------------------------------------------------------------------------------------------------
// Part A: (N, C, S) kernels
// ------------------------------------------------------------------------------------------------
// One pass: sums of (x-K) and (x-K)^2 with K = first element of the channel (same for all CTAs).
__global__ void __launch_bounds__(kRedThreads)
nchw_mean_var_kernel(const float* __restrict__ x, float* __restrict__ mean, float* __restrict__ var,
                     int N, int C, int S, int cl, int vec) {
  const int c = blockIdx.x / cl, rank = blockIdx.x % cl;
  const float K = __ldg(x + (size_t)c * S);
  float s1 = 0.f, s2 = 0.f;
  if (vec) {
    const int S4 = S >> 2;
    const long long tot4 = (long long)N * S4;
    for (long long j = (long long)rank * blockDim.x + threadIdx.x; j < tot4; j += (long long)cl * blockDim.x) {
      const int n = (int)(j / S4), s4 = (int)(j - (long long)n * S4);
      float4 v = ld_stream(reinterpret_cast<const float4*>(x + ((size_t)n * C + c) * S) + s4);
      float d0 = v.x - K, d1 = v.y - K, d2 = v.z - K, d3 = v.w - K;
      s1 += (d0 + d1) + (d2 + d3);
      s2 += (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
    }
  } else {
    const long long tot = (long long)N * S;
    for (long long j = (long long)rank * blockDim.x + threadIdx.x; j < tot; j += (long long)cl * blockDim.x) {
      const int n = (int)(j / S), s = (int)(j - (long long)n * S);
      float d = __ldg(x + ((size_t)n * C + c) * S + s) - K;
      s1 += d; s2 += d * d;
    }
  }
  float2 t = cluster_sum2(s1, s2);
  if (rank == 0 && threadIdx.x == 0) {
    const float inv = 1.f / ((float)N * (float)S);
    const float m = t.x * inv;
    mean[c] = K + m;
    var[c] = fmaxf(t.y * inv - m * m, 0.f);     // biased variance (bn.cu:132)
  }
}

__global__ void __launch_bounds__(256)
nchw_forward_kernel(const float* x, const float* __restrict__ mean, const float* __restrict__ var,
                    const float* __restrict__ weight, const float* __restrict__ bias, float* y, float* z,
                    float eps, int N, int C, int S, int vec) {
  const int c = blockIdx.x;
  const float m = mean[c], v = var[c];
  const float invstd = (v != 0.f || eps != 0.f) ? 1.f / sqrtf(v + eps) : 0.f;     // bn.cu:148-151
  const float gamma = weight ? fabsf(weight[c]) + eps : 1.f;                       // bn.cu:153
  const float beta = bias ? bias[c] : 0.f;
  const bool same = (y == z);
  if (vec) {
    const int S4 = S >> 2;
    const long long tot4 = (long long)N * S4;
    for (long long j = (long long)blockIdx.y * blockDim.x + threadIdx.x; j < tot4; j += (long long)gridDim.y * blockDim.x) {
      const int n = (int)(j / S4), s4 = (int)(j - (long long)n * S4);
      const size_t off = ((size_t)n * C + c) * S + 4 * (size_t)s4;
      float4 a = *reinterpret_cast<const float4*>(x + off), yy, zz;
      yy.x = (a.x - m) * invstd; yy.y = (a.y - m) * invstd; yy.z = (a.z - m) * invstd; yy.w = (a.w - m) * invstd;
      zz.x = yy.x * gamma + beta; zz.y = yy.y * gamma + beta; zz.z = yy.z * gamma + beta; zz.w = yy.w * gamma + beta;
      if (!same) *reinterpret_cast<float4*>(y + off) = yy;
      *reinterpret_cast<float4*>(z + off) = zz;
    }
  } else {
    const long long tot = (long long)N * S;
    for (long long j = (long long)blockIdx.y * blockDim.x + threadIdx.x; j < tot; j += (long long)gridDim.y * blockDim.x) {
      const int n = (int)(j / S), s = (int)(j - (long long)n * S);
      const size_t off = ((size_t)n * C + c) * S + s;
      const float yy = (x[off] - m) * invstd;
      if (!same) y[off] = yy;
      z[off] = yy * gamma + beta;
    }
  }
}

__global__ void __launch_bounds__(kRedThreads)
nchw_edz_eydz_kernel(const float* __restrict__ z, const float* __restrict__ dz, const float* __restrict__ weight,
                     const float* __restrict__ bias, float* __restrict__ edz, float* __restrict__ eydz, float eps,
                     int N, int C, int S, int cl, int vec) {
  const int c = blockIdx.x / cl, rank = blockIdx.x % cl;
  const float gamma = weight ? fabsf(weight[c]) + eps : 1.f;
  const float beta = bias ? bias[c] : 0.f;
  float s1 = 0.f, s2 = 0.f;
  if (vec) {
    const int S4 = S >> 2;
    const long long tot4 = (long long)N * S4;
    for (long long j = (long long)rank * blockDim.x + threadIdx.x; j < tot4; j += (long long)cl * blockDim.x) {
      const int n = (int)(j / S4), s4 = (int)(j - (long long)n * S4);
      const size_t off = ((size_t)n * C + c) * S;
      float4 a = ld_stream(reinterpret_cast<const float4*>(z + off) + s4);
      float4 g = ld_stream(reinterpret_cast<const float4*>(dz + off) + s4);
      s1 += (g.x + g.y) + (g.z + g.w);
      s2 += ((a.x - beta) / gamma * g.x + (a.y - beta) / gamma * g.y) + ((a.z - beta) / gamma * g.z + (a.w - beta) / gamma * g.w);
    }
  } else {
    const long long tot = (long long)N * S;
    for (long long j = (long long)rank * blockDim.x + threadIdx.x; j < tot; j += (long long)cl * blockDim.x) {
      const int n = (int)(j / S), s = (int)(j - (long long)n * S);
      const size_t off = ((size_t)n * C + c) * S + s;
      const float g = dz[off];
      s1 += g; s2 += (z[off] - beta) / gamma * g;
    }
  }
  float2 t = cluster_sum2(s1, s2);
  if (rank == 0 && threadIdx.x == 0) {
    const float inv = 1.f / ((float)N * (float)S);
    edz[c] = t.x * inv; eydz[c] = t.y * inv;
  }
}

__global__ void __launch_bounds__(256)
nchw_backward_kernel(const float* __restrict__ dz, const float* __restrict__ z, const float* __restrict__ var,
                     const float* __restrict__ weight, const float* __restrict__ bias,
                     const float* __restrict__ edz, const float* __restrict__ eydz, float* __restrict__ dx,
                     float* dweight, float* dbias, float eps, int N, int C, int S, int vec) {
  const int c = blockIdx.x;
  const float e1 = edz[c], e2 = eydz[c];
  const float gamma = weight ? fabsf(weight[c]) + eps : 1.f;
  const float beta = bias ? bias[c] : 0.f;
  if (dx) {
    const float v = var[c];
    const float invstd = (v != 0.f || eps != 0.f) ? 1.f / sqrtf(v + eps) : 0.f;
    const float mul = gamma * invstd;
    if (vec) {
      const int S4 = S >> 2;
      const long long tot4 = (long long)N * S4;
      for (long long j = (long long)blockIdx.y * blockDim.x + threadIdx.x; j < tot4; j += (long long)gridDim.y * blockDim.x) {
        const int n = (int)(j / S4), s4 = (int)(j - (long long)n * S4);
        const size_t off = ((size_t)n * C + c) * S + 4 * (size_t)s4;
        float4 g = ld_stream(reinterpret_cast<const float4*>(dz + off));
        float4 a = ld_stream(reinterpret_cast<const float4*>(z + off));
        float4 o;
        o.x = (g.x - e1 - (a.x - beta) / gamma * e2) * mul; o.y = (g.y - e1 - (a.y - beta) / gamma * e2) * mul;
        o.z = (g.z - e1 - (a.z - beta) / gamma * e2) * mul; o.w = (g.w - e1 - (a.w - beta) / gamma * e2) * mul;
        *reinterpret_cast<float4*>(dx + off) = o;
      }
    } else {
      const long long tot = (long long)N * S;
      for (long long j = (long long)blockIdx.y * blockDim.x + threadIdx.x; j < tot; j += (long long)gridDim.y * blockDim.x) {
        const int n = (int)(j / S), s = (int)(j - (long long)n * S);
        const size_t off = ((size_t)n * C + c) * S + s;
        dx[off] = (dz[off] - e1 - (z[off] - beta) / gamma * e2) * mul;
      }
    }
  }
  if (blockIdx.y == 0 && threadIdx.x == 0) {              // bn.cu:214-230: += into caller-zeroed buffers
    const float norm = (float)N * (float)S;
    if (dweight) {
      const float w = weight[c];
      if (w > 0.f) dweight[c] += e2 * norm; else if (w < 0.f) dweight[c] -= e2 * norm;
    }
    if (dbias) dbias[c] += e1 * norm;
  }
}

// elementwise activation helpers (bn.cu:302-377); op: 0 leaky fwd (x<0 -> x*slope), 1 leaky bwd, 2 elu fwd,
// 3 elu bwd, 4 elu inverse
template <int OP>
__global__ void __launch_bounds__(256) act_kernel(int n, float* __restrict__ x, float* __restrict__ dx, float slope) {
  const int n4 = n >> 2;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += gridDim.x * blockDim.x) {
    float4 a = reinterpret_cast<float4*>(x)[i];
    float* p = reinterpret_cast<float*>(&a);
    if (OP == 1 || OP == 3) {
      float4 g = reinterpret_cast<float4*>(dx)[i];
      float* q = reinterpret_cast<float*>(&g);
#pragma unroll
      for (int k = 0; k < 4; ++k) if (p[k] < 0.f) q[k] = OP == 1 ? q[k] * slope : q[k] * (p[k] + 1.f);
      reinterpret_cast<float4*>(dx)[i] = g;
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (p[k] < 0.f) p[k] = OP == 0 ? p[k] * slope : (OP == 2 ? expf(p[k]) - 1.f : log1pf(p[k]));
      reinterpret_cast<float4*>(x)[i] = a;
    }
  }
  for (int i = (n4 << 2) + blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float v = x[i];
    if (v < 0.f) {
      if (OP == 0) x[i] = v * slope;
      else if (OP == 1) dx[i] *= slope;
      else if (OP == 2) x[i] = expf(v) - 1.f;
      else if (OP == 3) dx[i] *= (v + 1.f);
      else x[i] = log1pf(v);
    }
  }
}

template <int OP>
int launch_act(int n, float* x, float* dx, float slope, cudaStream_t st, const char* name) {
  if (n <= 0) return 1;
  if ((reinterpret_cast<uintptr_t>(x) & 15) || (dx && (reinterpret_cast<uintptr_t>(dx) & 15))) {
    set_error_msg(name, "pointer not 16-byte aligned"); return 0;
  }
  int blocks = (n / 4 + 255) / 256;
  if (blocks < 1) blocks = 1;
  if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
  act_kernel<OP><<<blocks, 256, 0, st>>>(n, x, dx, slope);
  return finish(name);
}

int vec_ok(int S, const void* a, const void* b, const void* c) {
  return (S % 4 == 0) && !((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c)) & 15);
}

int elementwise_grid_y(int C, long long per_channel) {
  long long want = (4LL * kNumSMs + C - 1) / C;
  long long cap = (per_channel / 4 + 255) / 256;
  if (cap < 1) cap = 1;
  if (want > cap) want = cap;
  if (want < 1) want = 1;
  if (want > 65535) want = 65535;
  return (int)want;
}

// ------------------------------------------------------------------------------------------------
// Part B: NHWC kernels.  x is [P][C] (P = N*H*W rows), C % 4 == 0.
// ------------------------------------------------------------------------------------------------
// Shifted one-pass sums lose (m / std)^2 of float's precision, m = mean - K: ~3e-6 of the variance when the first row lies a few std
// from the mean, 1e-4 at 16 std, 1e-3 at 100.  The same pass therefore also keeps the sums in double, and a channel whose first row
// lies more than kShiftStd std from the mean takes its statistics from those; every other channel keeps the float result.
constexpr float kShiftStd = 8.f;

// partial[r][c] = (sum_rows (x-K), sum_rows (x-K)^2) over the rows owned by split r, K = x[0][c], in float; partial_d[r][c] the same
// sums in double
__global__ void __launch_bounds__(256)
nhwc_stats_partial_kernel(const float* __restrict__ x, float2* __restrict__ partial, double2* __restrict__ partial_d, long long P,
                          int C) {
  __shared__ float4 sh1[256], sh2[256];
  __shared__ double4 shd1[256], shd2[256];
  const int C4 = C >> 2;
  const int TC = C4 < 256 ? C4 : 256;                   // threads across channels
  const int TR = 256 / TC;                              // rows in flight per block
  const int tx = threadIdx.x % TC, ty = threadIdx.x / TC;
  const int c4 = blockIdx.y * TC + tx;
  const bool active = c4 < C4 && ty < TR;
  float4 K = active ? __ldg(reinterpret_cast<const float4*>(x) + c4) : make_float4(0, 0, 0, 0);
  float4 s1 = make_float4(0, 0, 0, 0), s2 = make_float4(0, 0, 0, 0);
  double4 d1 = make_double4(0, 0, 0, 0), d2 = d1;
  if (active) {
    const long long rows_per = (P + gridDim.x - 1) / gridDim.x;
    const long long r0 = (long long)blockIdx.x * rows_per;
    long long r1 = r0 + rows_per; if (r1 > P) r1 = P;
    const float4* base = reinterpret_cast<const float4*>(x) + c4;
    long long r = r0 + ty;
#define ACCD(v, f) { const double e = (double)v.f - (double)K.f; d1.f += e; d2.f = fma(e, e, d2.f); }
#define ACC(v) { float a = v.x - K.x, b = v.y - K.y, c = v.z - K.z, d = v.w - K.w; \
                 s1.x += a; s1.y += b; s1.z += c; s1.w += d; s2.x += a * a; s2.y += b * b; s2.z += c * c; s2.w += d * d; \
                 ACCD(v, x) ACCD(v, y) ACCD(v, z) ACCD(v, w) }
    for (; r + 3LL * TR < r1; r += 4LL * TR) {          // 4 independent 16B loads in flight per thread
      float4 v0 = ld_stream(base + r * C4), v1 = ld_stream(base + (r + TR) * C4);
      float4 v2 = ld_stream(base + (r + 2LL * TR) * C4), v3 = ld_stream(base + (r + 3LL * TR) * C4);
      ACC(v0) ACC(v1) ACC(v2) ACC(v3)
    }
    for (; r < r1; r += TR) { float4 v = ld_stream(base + r * C4); ACC(v) }
#undef ACC
#undef ACCD
  }
  sh1[threadIdx.x] = s1; sh2[threadIdx.x] = s2; shd1[threadIdx.x] = d1; shd2[threadIdx.x] = d2;
  __syncthreads();
  if (ty == 0 && active) {
    for (int k = 1; k < TR; ++k) {
      float4 a = sh1[k * TC + tx], b = sh2[k * TC + tx];
      s1.x += a.x; s1.y += a.y; s1.z += a.z; s1.w += a.w; s2.x += b.x; s2.y += b.y; s2.z += b.z; s2.w += b.w;
      const double4 p = shd1[k * TC + tx], q = shd2[k * TC + tx];
      d1.x += p.x; d1.y += p.y; d1.z += p.z; d1.w += p.w; d2.x += q.x; d2.y += q.y; d2.z += q.z; d2.w += q.w;
    }
    float2* out = partial + (size_t)blockIdx.x * C + 4 * (size_t)c4;
    out[0] = make_float2(s1.x, s2.x); out[1] = make_float2(s1.y, s2.y);
    out[2] = make_float2(s1.z, s2.z); out[3] = make_float2(s1.w, s2.w);
    double2* od = partial_d + (size_t)blockIdx.x * C + 4 * (size_t)c4;
    od[0] = make_double2(d1.x, d2.x); od[1] = make_double2(d1.y, d2.y);
    od[2] = make_double2(d1.z, d2.z); od[3] = make_double2(d1.w, d2.w);
  }
}

// mean/var from the split partials (+ running-stat EMA, + folded scale/shift for the apply pass)
__global__ void nhwc_stats_finalize_kernel(const float* __restrict__ x, const float2* __restrict__ partial,
                                           const double2* __restrict__ partial_d, int R, int C, float count,
                                           const float* __restrict__ weight, const float* __restrict__ bias, float eps,
                                           float momentum, float* running_mean, float* running_var, float* __restrict__ mean,
                                           float* __restrict__ var, float* __restrict__ scale, float* __restrict__ shift) {
  // one WARP per channel (8 channels per block): the R (~600) split partials of a channel are read by 32 lanes -- ~19 dependent loads
  // per thread instead of 37 -- and folded with shuffles (the 2-block version was latency-bound, 58 times a step)
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (c >= C) return;
  float s1 = 0.f, s2 = 0.f;
  for (int r = lane; r < R; r += 32) { float2 p = partial[(size_t)r * C + c]; s1 += p.x; s2 += p.y; }
  s1 = warp_sum(s1); s2 = warp_sum(s2);
  const float K = x[c];
  const float m = s1 / count;
  float mu = K + m;
  float v = fmaxf(__fsub_rn(s2 / count, __fmul_rn(m, m)), 0.f);   // product and difference rounded separately, never fused
  if (fabsf(m) > kShiftStd * sqrtf(v)) {                           // the whole warp: the same s1, s2 in every lane
    double t1 = 0.0, t2 = 0.0;
    for (int r = lane; r < R; r += 32) { const double2 p = partial_d[(size_t)r * C + c]; t1 += p.x; t2 += p.y; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { t1 += __shfl_xor_sync(0xffffffffu, t1, o); t2 += __shfl_xor_sync(0xffffffffu, t2, o); }
    const double md = t1 / (double)count;
    mu = (float)((double)K + md);
    v = (float)fmax(t2 / (double)count - md * md, 0.0);
  }
  if (lane != 0) return;
  mean[c] = mu; var[c] = v;
  if (running_mean) {                                              // libs/functions.py:90-91
    running_mean[c] = running_mean[c] * (1.f - momentum) + momentum * mu;
    running_var[c] = running_var[c] * (1.f - momentum) + momentum * v * (count > 1.f ? count / (count - 1.f) : 1.f);   // n/(n-1) (functions.py:91); a single sample keeps the biased value instead of 0 * inf
  }
  const float invstd = 1.f / sqrtf(v + eps);
  const float gamma = weight ? fabsf(weight[c]) + eps : 1.f;
  const float sc = gamma * invstd;
  scale[c] = sc;
  shift[c] = (bias ? bias[c] : 0.f) - mu * sc;
}

// scale/shift from given (running) statistics: eval-mode ABN and BN folding for the frozen teacher
__global__ void nhwc_fold_kernel(int C, const float* __restrict__ mean, const float* __restrict__ var,
                                 const float* __restrict__ weight, const float* __restrict__ bias, float eps,
                                 float* __restrict__ scale, float* __restrict__ shift) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float invstd = 1.f / sqrtf(var[c] + eps);
  const float gamma = weight ? fabsf(weight[c]) + eps : 1.f;
  const float sc = gamma * invstd;
  scale[c] = sc; shift[c] = (bias ? bias[c] : 0.f) - mean[c] * sc;
}

// out = act(x*scale + shift (+ residual)) (* chan_mul[n][c])
__global__ void __launch_bounds__(256)
nhwc_apply_kernel(const float* __restrict__ x, float* __restrict__ out, int out_pitch4, long long total4, int C4, int S,
                  const float* __restrict__ scale, const float* __restrict__ shift, int act, float slope,
                  const float* __restrict__ residual, const float* __restrict__ chan_mul, int round_out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / C4;
    const int c4 = (int)(i - row * C4);
    float4 v = ld_stream(reinterpret_cast<const float4*>(x) + i);
    const float4 sc = __ldg(reinterpret_cast<const float4*>(scale) + c4);
    const float4 sf = __ldg(reinterpret_cast<const float4*>(shift) + c4);
    v.x = v.x * sc.x + sf.x; v.y = v.y * sc.y + sf.y; v.z = v.z * sc.z + sf.z; v.w = v.w * sc.w + sf.w;
    if (residual) {
      float4 r = ld_stream(reinterpret_cast<const float4*>(residual) + i);
      v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
    }
    v.x = act_fwd(v.x, act, slope); v.y = act_fwd(v.y, act, slope);
    v.z = act_fwd(v.z, act, slope); v.w = act_fwd(v.w, act, slope);
    if (chan_mul) {
      const long long n = row / S;
      const float4 m = __ldg(reinterpret_cast<const float4*>(chan_mul) + n * C4 + c4);
      v.x *= m.x; v.y *= m.y; v.z *= m.z; v.w *= m.w;
    }
    if (round_out) { v.x = ptx::round_tf32(v.x); v.y = ptx::round_tf32(v.y); v.z = ptx::round_tf32(v.z); v.w = ptx::round_tf32(v.w); }
    reinterpret_cast<float4*>(out)[row * out_pitch4 + c4] = v;
  }
}

__device__ __forceinline__ float dact(float o, float g, int act, float slope) {
  // derivative through the activation, sign taken from the stored output (valid for relu / leaky with slope>0)
  if (act == ACT_RELU) return o > 0.f ? g : 0.f;
  if (act == ACT_LEAKY) return o < 0.f ? g * slope : g;
  if (act == ACT_ELU) return o < 0.f ? g * (o + 1.f) : g;
  return g;
}

// The stored output is act(.) * chan_mul: ELU's derivative (o + 1 where o < 0) needs o before the mask.  A zero mask zeroes g,
// so its o does not matter.  (relu / leaky only read the sign, which a positive mask keeps.)
__device__ __forceinline__ void unmask(float4& o, const float4 m) {
  o.x = m.x != 0.f ? o.x / m.x : 0.f; o.y = m.y != 0.f ? o.y / m.y : 0.f;
  o.z = m.z != 0.f ? o.z / m.z : 0.f; o.w = m.w != 0.f ? o.w / m.w : 0.f;
}

// partial[r][c] = (sum dz, sum y*dz), dz = dout * chan_mul * act'(out / chan_mul), y = (x-mean)*invstd
__global__ void __launch_bounds__(256)
nhwc_bwd_partial_kernel(const float* __restrict__ x, const float* __restrict__ out, const float* __restrict__ dout,
                        float2* __restrict__ partial, long long P, int C, int S, const float* __restrict__ mean,
                        const float* __restrict__ var, float eps, int act, float slope,
                        const float* __restrict__ chan_mul, const float* __restrict__ scale, const float* __restrict__ shift) {
  // out == nullptr: the activation's sign is recomputed as x*scale + shift -- the very FMA the apply pass evaluated, so the mask
  // is bit-identical -- and the stored activation output is not read at all (layers without a fused residual: 4 reads instead of 6
  // over the two backward passes)
  __shared__ float4 sh1[256], sh2[256];
  const int C4 = C >> 2;
  const int TC = C4 < 256 ? C4 : 256;
  const int TR = 256 / TC;
  const int tx = threadIdx.x % TC, ty = threadIdx.x / TC;
  const int c4 = blockIdx.y * TC + tx;
  const bool active = c4 < C4 && ty < TR;
  float4 s1 = make_float4(0, 0, 0, 0), s2 = make_float4(0, 0, 0, 0);
  if (active) {
    const float4 mu = __ldg(reinterpret_cast<const float4*>(mean) + c4);
    float4 is = __ldg(reinterpret_cast<const float4*>(var) + c4);
    is.x = 1.f / sqrtf(is.x + eps); is.y = 1.f / sqrtf(is.y + eps); is.z = 1.f / sqrtf(is.z + eps); is.w = 1.f / sqrtf(is.w + eps);
    float4 sc = make_float4(0, 0, 0, 0), sf = sc;
    if (!out) { sc = __ldg(reinterpret_cast<const float4*>(scale) + c4); sf = __ldg(reinterpret_cast<const float4*>(shift) + c4); }
    const long long rows_per = (P + gridDim.x - 1) / gridDim.x;
    const long long r0 = (long long)blockIdx.x * rows_per;
    long long r1 = r0 + rows_per; if (r1 > P) r1 = P;
    for (long long r = r0 + ty; r < r1; r += TR) {
      const long long i = r * C4 + c4;
      float4 xv = ld_stream(reinterpret_cast<const float4*>(x) + i);
      float4 ov;
      if (out) ov = ld_stream(reinterpret_cast<const float4*>(out) + i);
      else { ov.x = xv.x * sc.x + sf.x; ov.y = xv.y * sc.y + sf.y; ov.z = xv.z * sc.z + sf.z; ov.w = xv.w * sc.w + sf.w; }
      float4 g = ld_stream(reinterpret_cast<const float4*>(dout) + i);
      if (chan_mul) {
        const float4 m = __ldg(reinterpret_cast<const float4*>(chan_mul) + (r / S) * C4 + c4);
        g.x *= m.x; g.y *= m.y; g.z *= m.z; g.w *= m.w;
        if (act == ACT_ELU) unmask(ov, m);
      }
      g.x = dact(ov.x, g.x, act, slope); g.y = dact(ov.y, g.y, act, slope);
      g.z = dact(ov.z, g.z, act, slope); g.w = dact(ov.w, g.w, act, slope);
      s1.x += g.x; s1.y += g.y; s1.z += g.z; s1.w += g.w;
      s2.x += (xv.x - mu.x) * is.x * g.x; s2.y += (xv.y - mu.y) * is.y * g.y;
      s2.z += (xv.z - mu.z) * is.z * g.z; s2.w += (xv.w - mu.w) * is.w * g.w;
    }
  }
  sh1[threadIdx.x] = s1; sh2[threadIdx.x] = s2;
  __syncthreads();
  if (ty == 0 && active) {
    for (int k = 1; k < TR; ++k) {
      float4 a = sh1[k * TC + tx], b = sh2[k * TC + tx];
      s1.x += a.x; s1.y += a.y; s1.z += a.z; s1.w += a.w; s2.x += b.x; s2.y += b.y; s2.z += b.z; s2.w += b.w;
    }
    float2* o = partial + (size_t)blockIdx.x * C + 4 * (size_t)c4;
    o[0] = make_float2(s1.x, s2.x); o[1] = make_float2(s1.y, s2.y);
    o[2] = make_float2(s1.z, s2.z); o[3] = make_float2(s1.w, s2.w);
  }
}

__global__ void nhwc_bwd_finalize_kernel(const float2* __restrict__ partial, int R, int C, float count,
                                         const float* __restrict__ weight, float* __restrict__ edz,
                                         float* __restrict__ eydz, float* __restrict__ dweight,
                                         float* __restrict__ dbias) {
  // one warp per channel, 8 channels per block (see nhwc_stats_finalize_kernel)
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (c >= C) return;
  float s1 = 0.f, s2 = 0.f;
  for (int r = lane; r < R; r += 32) { float2 p = partial[(size_t)r * C + c]; s1 += p.x; s2 += p.y; }
  s1 = warp_sum(s1); s2 = warp_sum(s2);
  if (lane != 0) return;
  edz[c] = s1 / count; eydz[c] = s2 / count;
  if (dweight) { const float w = weight[c]; dweight[c] = w > 0.f ? s2 : (w < 0.f ? -s2 : 0.f); }   // bn.cu:217-223
  if (dbias) dbias[c] = s1;
}

// dx = (dz - edz - y*eydz) * gamma*invstd ; dres = dz
// The launch makes gridDim.x * blockDim.x a multiple of C4 whenever it can, so a thread meets ONE channel quad in every iteration of its
// grid-stride loop: the per-channel terms fold once into dx = k1*(dz - edz) - k2*(x - mean) (a version that re-derives them per
// element -- a 64-bit division, five parameter loads, four rsqrt -- is issue-bound).
__global__ void __launch_bounds__(256)
nhwc_bwd_dx_kernel(const float* __restrict__ x, const float* __restrict__ out, const float* __restrict__ dout,
                   float* __restrict__ dx, float* __restrict__ dres, long long total4, int C4, int S,
                   const float* __restrict__ mean, const float* __restrict__ var, const float* __restrict__ weight,
                   const float* __restrict__ edz, const float* __restrict__ eydz, float eps, int act, float slope,
                   const float* __restrict__ chan_mul, int round_out, const float* __restrict__ scale, const float* __restrict__ shift) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const bool fixed_c = (stride % C4) == 0;
  float4 k1, k2, mu, e1, sc, sf;
  auto coeffs = [&](int c4) {
    mu = __ldg(reinterpret_cast<const float4*>(mean) + c4);
    const float4 vv = __ldg(reinterpret_cast<const float4*>(var) + c4);
    e1 = __ldg(reinterpret_cast<const float4*>(edz) + c4);
    const float4 e2 = __ldg(reinterpret_cast<const float4*>(eydz) + c4);
    const float4 w = weight ? __ldg(reinterpret_cast<const float4*>(weight) + c4) : make_float4(1, 1, 1, 1);
#define KK(f) { const float is = 1.f / sqrtf(vv.f + eps); const float gm = weight ? fabsf(w.f) + eps : 1.f; \
                k1.f = gm * is; k2.f = is * e2.f * gm * is; }
    KK(x) KK(y) KK(z) KK(w)
#undef KK
    if (!out) { sc = __ldg(reinterpret_cast<const float4*>(scale) + c4); sf = __ldg(reinterpret_cast<const float4*>(shift) + c4); }
  };
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  int c4 = (int)(i % C4);
  if (fixed_c && i < total4) coeffs(c4);
  for (; i < total4; i += stride) {
    if (!fixed_c) { c4 = (int)(i % C4); coeffs(c4); }
    float4 xv = ld_stream(reinterpret_cast<const float4*>(x) + i);
    float4 ov;
    if (out) ov = ld_stream(reinterpret_cast<const float4*>(out) + i);
    else { ov.x = xv.x * sc.x + sf.x; ov.y = xv.y * sc.y + sf.y; ov.z = xv.z * sc.z + sf.z; ov.w = xv.w * sc.w + sf.w; }   // sign of the activation input, recomputed (see nhwc_bwd_partial_kernel)
    float4 g = ld_stream(reinterpret_cast<const float4*>(dout) + i);
    if (chan_mul) {
      const long long row = i / C4;
      const float4 m = __ldg(reinterpret_cast<const float4*>(chan_mul) + (row / S) * C4 + c4);
      g.x *= m.x; g.y *= m.y; g.z *= m.z; g.w *= m.w;
      if (act == ACT_ELU) unmask(ov, m);
    }
    g.x = dact(ov.x, g.x, act, slope); g.y = dact(ov.y, g.y, act, slope);
    g.z = dact(ov.z, g.z, act, slope); g.w = dact(ov.w, g.w, act, slope);
    if (dres) reinterpret_cast<float4*>(dres)[i] = g;
    float4 o;
    o.x = fmaf(g.x - e1.x, k1.x, -(xv.x - mu.x) * k2.x); o.y = fmaf(g.y - e1.y, k1.y, -(xv.y - mu.y) * k2.y);
    o.z = fmaf(g.z - e1.z, k1.z, -(xv.z - mu.z) * k2.z); o.w = fmaf(g.w - e1.w, k1.w, -(xv.w - mu.w) * k2.w);
    if (round_out) { o.x = ptx::round_tf32(o.x); o.y = ptx::round_tf32(o.y); o.z = ptx::round_tf32(o.z); o.w = ptx::round_tf32(o.w); }
    reinterpret_cast<float4*>(dx)[i] = o;
  }
}

int ew_blocks(long long total4) {
  long long b = (total4 + 255) / 256;
  if (b > kNumSMs * 16) b = kNumSMs * 16;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace

// ---------------------------------------------------------------------------------------------------
// C ABI -- Part A (replaces libs/src/bn.h:7-19 one for one)
// ---------------------------------------------------------------------------------------------------
extern "C" int skd_bn_mean_var_cuda(int N, int C, int S, const float* x, float* mean, float* var, cudaStream_t st) {
  if (N <= 0 || C <= 0 || S <= 0) return 1;
  const int cl = pick_cluster(C, (long long)N * S);
  cudaError_t e = launch_cluster(nchw_mean_var_kernel, dim3(C * cl), dim3(kRedThreads), cl, st, x, mean, var, N, C, S, cl, vec_ok(S, x, nullptr, nullptr));
  if (e != cudaSuccess) { set_error("skd_bn_mean_var_cuda", e); return 0; }
  return finish("skd_bn_mean_var_cuda");
}

extern "C" int skd_bn_forward_cuda(int N, int C, int S, const float* x, const float* mean, const float* var,
                                   const float* weight, const float* bias, float* y, float* z, float eps,
                                   cudaStream_t st) {
  if (N <= 0 || C <= 0 || S <= 0) return 1;
  nchw_forward_kernel<<<dim3(C, elementwise_grid_y(C, (long long)N * S)), 256, 0, st>>>(x, mean, var, weight, bias, y, z,
                                                                                         eps, N, C, S, vec_ok(S, x, y, z));
  return finish("skd_bn_forward_cuda");
}

extern "C" int skd_bn_edz_eydz_cuda(int N, int C, int S, const float* z, const float* dz, const float* weight,
                                    const float* bias, float* edz, float* eydz, float eps, cudaStream_t st) {
  if (N <= 0 || C <= 0 || S <= 0) return 1;
  const int cl = pick_cluster(C, (long long)N * S);
  cudaError_t e = launch_cluster(nchw_edz_eydz_kernel, dim3(C * cl), dim3(kRedThreads), cl, st, z, dz, weight, bias, edz,
                                 eydz, eps, N, C, S, cl, vec_ok(S, z, dz, nullptr));
  if (e != cudaSuccess) { set_error("skd_bn_edz_eydz_cuda", e); return 0; }
  return finish("skd_bn_edz_eydz_cuda");
}

extern "C" int skd_bn_backward_cuda(int N, int C, int S, const float* dz, const float* z, const float* var,
                                    const float* weight, const float* bias, const float* edz, const float* eydz,
                                    float* dx, float* dweight, float* dbias, float eps, cudaStream_t st) {
  if (N <= 0 || C <= 0 || S <= 0) return 1;
  nchw_backward_kernel<<<dim3(C, elementwise_grid_y(C, (long long)N * S)), 256, 0, st>>>(dz, z, var, weight, bias, edz, eydz,
                                                                                          dx, dweight, dbias, eps, N, C, S, vec_ok(S, dz, z, dx));
  return finish("skd_bn_backward_cuda");
}

extern "C" int skd_leaky_relu_cuda(int N, float* x, float slope, cudaStream_t st) {
  return launch_act<0>(N, x, nullptr, slope, st, "skd_leaky_relu_cuda");
}
extern "C" int skd_leaky_relu_backward_cuda(int N, const float* x, float* dx, float slope, cudaStream_t st) {
  return launch_act<1>(N, const_cast<float*>(x), dx, slope, st, "skd_leaky_relu_backward_cuda");
}
extern "C" int skd_elu_cuda(int N, float* x, cudaStream_t st) { return launch_act<2>(N, x, nullptr, 0.f, st, "skd_elu_cuda"); }
extern "C" int skd_elu_backward_cuda(int N, const float* x, float* dx, cudaStream_t st) {
  return launch_act<3>(N, const_cast<float*>(x), dx, 0.f, st, "skd_elu_backward_cuda");
}
extern "C" int skd_elu_inv_cuda(int N, float* x, cudaStream_t st) { return launch_act<4>(N, x, nullptr, 0.f, st, "skd_elu_inv_cuda"); }

// ---------------------------------------------------------------------------------------------------
// C ABI -- Part B (NHWC)
// ---------------------------------------------------------------------------------------------------
extern "C" int skd_abn_num_splits(long long P, int C) {
  // row splits so that splits * channel-chunks ~ 4 waves, each split >= 32 rows
  const int chunks = (C / 4 + 255) / 256;
  long long r = (4LL * skd::kNumSMs + chunks - 1) / chunks;
  long long cap = (P + 31) / 32;
  if (r > cap) r = cap;
  if (r < 1) r = 1;
  return (int)r;
}

static int nhwc_check(const char* name, int C, const void* a, const void* b, const void* c) {
  if (C % 4 != 0) { set_error_msg(name, "C must be a multiple of 4 for the NHWC path"); return 0; }
  if ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c)) & 15) {
    set_error_msg(name, "pointer not 16-byte aligned"); return 0;
  }
  return 1;
}

extern "C" int skd_abn_stats_nhwc(long long P, int C, const float* x, const float* weight, const float* bias,
                                  float eps, float momentum, float* running_mean, float* running_var, float* mean,
                                  float* var, float* scale, float* shift, float* workspace, int splits,
                                  cudaStream_t st) {
  if (!nhwc_check("skd_abn_stats_nhwc", C, x, workspace, nullptr)) return 0;
  if (P <= 0) return 1;
  const int chunks = (C / 4 + 255) / 256;
  float2* part = reinterpret_cast<float2*>(workspace);
  double2* part_d = reinterpret_cast<double2*>(workspace + (size_t)splits * C * 2);
  nhwc_stats_partial_kernel<<<dim3(splits, chunks), 256, 0, st>>>(x, part, part_d, P, C);
  nhwc_stats_finalize_kernel<<<(C + 7) / 8, 256, 0, st>>>(x, part, part_d, splits, C, (float)P, weight, bias, eps, momentum,
                                                             running_mean, running_var, mean, var, scale, shift);
  return finish("skd_abn_stats_nhwc", 2);
}

extern "C" int skd_abn_fold(int C, const float* mean, const float* var, const float* weight, const float* bias, float eps,
                            float* scale, float* shift, cudaStream_t st) {
  nhwc_fold_kernel<<<(C + 127) / 128, 128, 0, st>>>(C, mean, var, weight, bias, eps, scale, shift);
  return finish("skd_abn_fold");
}

extern "C" int skd_abn_apply_nhwc(long long P, int C, int S, const float* x, float* out, int out_pitch, const float* scale,
                                  const float* shift, int act, float slope, const float* residual,
                                  const float* chan_mul, int round_tf32, cudaStream_t st) {
  if (!nhwc_check("skd_abn_apply_nhwc", C, x, out, residual)) return 0;
  if (out_pitch % 4) { set_error_msg("skd_abn_apply_nhwc", "out_pitch must be a multiple of 4"); return 0; }
  if (P <= 0) return 1;
  const long long total4 = P * (C / 4);
  nhwc_apply_kernel<<<ew_blocks(total4), 256, 0, st>>>(x, out, out_pitch / 4, total4, C / 4, S, scale, shift, act, slope, residual,
                                                      chan_mul, round_tf32);
  return finish("skd_abn_apply_nhwc");
}

extern "C" int skd_abn_bwd_reduce_nhwc(long long P, int C, int S, const float* x, const float* out, const float* dout,
                                       const float* mean, const float* var, const float* weight, float eps, int act,
                                       float slope, const float* chan_mul, float* edz, float* eydz, float* dweight,
                                       float* dbias, float* workspace, int splits, const float* scale, const float* shift,
                                       cudaStream_t st) {
  if (!nhwc_check("skd_abn_bwd_reduce_nhwc", C, x, out, dout)) return 0;
  if (!out && (!scale || !shift || act == ACT_ELU)) { set_error_msg("skd_abn_bwd_reduce_nhwc", "out == NULL needs scale/shift and a sign-only activation"); return 0; }
  if (P <= 0) return 1;
  const int chunks = (C / 4 + 255) / 256;
  nhwc_bwd_partial_kernel<<<dim3(splits, chunks), 256, 0, st>>>(x, out, dout, reinterpret_cast<float2*>(workspace), P, C, S,
                                                               mean, var, eps, act, slope, chan_mul, scale, shift);
  nhwc_bwd_finalize_kernel<<<(C + 7) / 8, 256, 0, st>>>(reinterpret_cast<const float2*>(workspace), splits, C, (float)P,
                                                           weight, edz, eydz, dweight, dbias);
  return finish("skd_abn_bwd_reduce_nhwc", 2);
}

extern "C" int skd_abn_bwd_dx_nhwc(long long P, int C, int S, const float* x, const float* out, const float* dout,
                                   float* dx, float* dres, const float* mean, const float* var, const float* weight,
                                   const float* edz, const float* eydz, float eps, int act, float slope,
                                   const float* chan_mul, int round_tf32, const float* scale, const float* shift, cudaStream_t st) {
  if (!nhwc_check("skd_abn_bwd_dx_nhwc", C, x, dx, dres)) return 0;
  if (!out && (!scale || !shift || act == ACT_ELU)) { set_error_msg("skd_abn_bwd_dx_nhwc", "out == NULL needs scale/shift and a sign-only activation"); return 0; }
  if (P <= 0) return 1;
  const long long total4 = P * (C / 4);
  nhwc_bwd_dx_kernel<<<ew_blocks(total4), 256, 0, st>>>(x, out, dout, dx, dres, total4, C / 4, S, mean, var, weight, edz,
                                                       eydz, eps, act, slope, chan_mul, round_tf32, scale, shift);
  return finish("skd_abn_bwd_dx_nhwc");
}
