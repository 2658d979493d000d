// MobileNetV2 student (networks/mobilenet.py): the depthwise 3x3 convolution (groups = C) -- forward with the following BatchNorm's
// statistics accumulated in the same pass, data gradient as a gather, weight gradient as per-block partials reduced in a second
// pass -- and BatchNorm + ReLU6 / linear BatchNorm (+ residual) apply and backward passes.
//
// All tensors are fp32 NHWC with C a multiple of 4: a thread owns four consecutive channels and reads a pixel's slice of them as
// one float4 (every MobileNetV2 width is a multiple of 8).  A depthwise output element is 9 multiply-adds over the same channel of
// its input, so the pass is bound by HBM, not by arithmetic; the tensor cores have nothing to do here.
//
// Every reduction adds in a fixed order (rows split by (P, C) alone, partials in double, splits summed in order by a finalize
// pass), with no atomics, so two runs give bit-identical results.
#include <cstdint>
#include <initializer_list>

#include "common.cuh"
#include "skd.h"

using namespace skd;

namespace {

constexpr int kThreads = 256;
constexpr int kStatBlocks = 4 * kNumSMs;    // row splits of the statistics / BatchNorm backward reductions (per channel chunk)
constexpr int kWgradBlocks = 2 * kNumSMs;   // ... of the weight gradient (nine partials per channel: a smaller workspace)

// A block's channel-group chunk and its share of the rows: tc threads across groups of 4 channels, tr rows in flight
struct Tile4 {
  int tc, tr, tx, ty, c;     // c: first of the thread's four channels
  long long r0, r1;
  bool active;
};
__device__ __forceinline__ Tile4 tile4_of(long long P, int C) {
  const int c4 = C >> 2;
  Tile4 t;
  t.tc = c4 < kThreads ? c4 : kThreads;
  t.tr = kThreads / t.tc;
  t.tx = threadIdx.x % t.tc; t.ty = threadIdx.x / t.tc;
  t.c = (blockIdx.y * t.tc + t.tx) * 4;
  t.active = t.ty < t.tr && t.c < C;
  const long long per = (P + gridDim.x - 1) / gridDim.x;
  t.r0 = (long long)blockIdx.x * per;
  t.r1 = t.r0 + per < P ? t.r0 + per : P;
  return t;
}

int chunks_of(int C) {
  const int c4 = C / 4, tc = c4 < kThreads ? c4 : kThreads;
  return (c4 + tc - 1) / tc;
}

int splits_of(long long P, int C, int blocks) {
  const int chunks = chunks_of(C);
  long long r = (blocks + chunks - 1) / chunks;
  const long long cap = (P + 31) / 32;
  if (r > cap) r = cap;
  return (int)(r < 1 ? 1 : r);
}

int ew_grid(long long total) {
  long long b = (total + kThreads - 1) / kThreads;
  if (b > kNumSMs * 16) b = kNumSMs * 16;
  return (int)(b < 1 ? 1 : b);
}

bool aligned16(const void* p) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

__device__ __forceinline__ float lane(const float4& v, int j) { return j == 0 ? v.x : j == 1 ? v.y : j == 2 ? v.z : v.w; }
__device__ __forceinline__ void set_lane(float4& v, int j, float s) {
  if (j == 0) v.x = s; else if (j == 1) v.y = s; else if (j == 2) v.z = s; else v.w = s;
}
__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ float4 fma4(float4 a, float4 b, float4 c) {
  return make_float4(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y), fmaf(a.z, b.z, c.z), fmaf(a.w, b.w, c.w));
}

// Depthwise geometry: input N x H x W, output N x OH x OW, C channels; 3x3 taps at dilation d, padding d, stride s in {1, 2}
struct DwGeom {
  int N, H, W, C, OH, OW, s, d;
};

// the thread's four channels of the (C, 1, 3, 3) weight, tap-major: w[tap] = (w[c][tap], ..., w[c + 3][tap])
__device__ __forceinline__ void load_taps(const float* __restrict__ weight, int c, float4 (&w)[9]) {
#pragma unroll
  for (int k = 0; k < 9; ++k)
    w[k] = make_float4(weight[(c + 0) * 9 + k], weight[(c + 1) * 9 + k], weight[(c + 2) * 9 + k], weight[(c + 3) * 9 + k]);
}

// y[n][oy][ox][c] = sum_{ky, kx} w[c][ky][kx] * x[n][oy*s - d + ky*d][ox*s - d + kx*d][c] (taps outside the map read zero), taps in
// row-major order.  kStats: partial[split][c] = (sum y, sum y^2) over the block's rows, for the BatchNorm that follows.
template <bool kStats>
__global__ void __launch_bounds__(kThreads)
dw_fwd_kernel(DwGeom g, const float* __restrict__ x, const float* __restrict__ weight, float* __restrict__ y,
              double2* __restrict__ partial) {
  __shared__ double2 sh[kStats ? 4 : 1][kThreads];
  const long long P = (long long)g.N * g.OH * g.OW;
  const Tile4 t = tile4_of(P, g.C);
  double s1[4] = {0.0, 0.0, 0.0, 0.0}, s2[4] = {0.0, 0.0, 0.0, 0.0};
  if (t.active) {
    float4 w[9];
    load_taps(weight, t.c, w);
    for (long long r = t.r0 + t.ty; r < t.r1; r += t.tr) {
      const int ox = (int)(r % g.OW); const long long q = r / g.OW;
      const int oy = (int)(q % g.OH), n = (int)(q / g.OH);
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) {
        const int iy = oy * g.s - g.d + ky * g.d;
        if (iy < 0 || iy >= g.H) continue;
        const float* row = x + ((long long)n * g.H + iy) * g.W * g.C + t.c;
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const int ix = ox * g.s - g.d + kx * g.d;
          if (ix < 0 || ix >= g.W) continue;
          acc = fma4(w[ky * 3 + kx], ld4(row + (long long)ix * g.C), acc);
        }
      }
      st4(y + r * g.C + t.c, acc);
      if (kStats) {
#pragma unroll
        for (int j = 0; j < 4; ++j) { const double v = lane(acc, j); s1[j] += v; s2[j] += v * v; }
      }
    }
  }
  if constexpr (kStats) {
#pragma unroll
    for (int j = 0; j < 4; ++j) sh[j][threadIdx.x] = make_double2(s1[j], s2[j]);
    __syncthreads();
    if (t.ty == 0 && t.active) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        double a = s1[j], b = s2[j];
        for (int k = 1; k < t.tr; ++k) { const double2 p = sh[j][k * t.tc + t.tx]; a += p.x; b += p.y; }
        partial[(long long)blockIdx.x * g.C + t.c + j] = make_double2(a, b);
      }
    }
  }
}

// mean, biased variance; running statistics with the unbiased variance n / (n - 1) and momentum, as torch's BatchNorm2d (the same
// arithmetic as skd_bnprelu_stats)
__global__ void stats_finalize_kernel(int R, int C, const double2* __restrict__ partial, double count, float momentum,
                                      float* __restrict__ running_mean, float* __restrict__ running_var, long long* nbt,
                                      float* __restrict__ mean, float* __restrict__ var) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c == 0 && nbt) *nbt += 1;
  if (c >= C) return;
  double s1 = 0.0, s2 = 0.0;
  for (int r = 0; r < R; ++r) { const double2 p = partial[(long long)r * C + c]; s1 += p.x; s2 += p.y; }
  const double m = s1 / count;
  double v = s2 / count - m * m;
  if (v < 0.0) v = 0.0;
  mean[c] = (float)m; var[c] = (float)v;
  if (running_mean) {
    const float ub = (float)(count > 1.0 ? v * count / (count - 1.0) : v);
    running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)m;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * ub;
  }
}

// dx[n][iy][ix][c] = sum over the taps (ky, kx) whose output pixel oy = (iy + d - ky*d) / s, ox = (ix + d - kx*d) / s is whole and
// inside the output map of w[c][ky][kx] * dy[n][oy][ox][c]: a gather, one thread per input element group, taps in row-major order
__global__ void __launch_bounds__(kThreads)
dw_dgrad_kernel(DwGeom g, const float* __restrict__ dy, const float* __restrict__ weight, float* __restrict__ dx) {
  const long long P = (long long)g.N * g.H * g.W;
  const Tile4 t = tile4_of(P, g.C);
  if (!t.active) return;
  float4 w[9];
  load_taps(weight, t.c, w);
  for (long long r = t.r0 + t.ty; r < t.r1; r += t.tr) {
    const int ix = (int)(r % g.W); const long long q = r / g.W;
    const int iy = (int)(q % g.H), n = (int)(q / g.H);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int ty = iy + g.d - ky * g.d;
      if (ty < 0 || ty % g.s) continue;
      const int oy = ty / g.s;
      if (oy >= g.OH) continue;
      const float* row = dy + ((long long)n * g.OH + oy) * g.OW * g.C + t.c;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int tx = ix + g.d - kx * g.d;
        if (tx < 0 || tx % g.s) continue;
        const int ox = tx / g.s;
        if (ox >= g.OW) continue;
        acc = fma4(w[ky * 3 + kx], ld4(row + (long long)ox * g.C), acc);
      }
    }
    st4(dx + r * g.C + t.c, acc);
  }
}

// partial[split][tap][c] = sum over the block's output pixels p of dy[p][c] * x[p + offset(tap)][c]: fp32 per thread, the block's
// threads added in double in row order
__global__ void __launch_bounds__(kThreads)
dw_wgrad_kernel(DwGeom g, const float* __restrict__ x, const float* __restrict__ dy, double* __restrict__ partial) {
  __shared__ float4 sh[kThreads];
  const long long P = (long long)g.N * g.OH * g.OW;
  const Tile4 t = tile4_of(P, g.C);
  float4 acc[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (t.active) {
    for (long long r = t.r0 + t.ty; r < t.r1; r += t.tr) {
      const int ox = (int)(r % g.OW); const long long q = r / g.OW;
      const int oy = (int)(q % g.OH), n = (int)(q / g.OH);
      const float4 gv = ld4(dy + r * g.C + t.c);
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) {
        const int iy = oy * g.s - g.d + ky * g.d;
        if (iy < 0 || iy >= g.H) continue;
        const float* row = x + ((long long)n * g.H + iy) * g.W * g.C + t.c;
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const int ix = ox * g.s - g.d + kx * g.d;
          if (ix < 0 || ix >= g.W) continue;
          acc[ky * 3 + kx] = fma4(gv, ld4(row + (long long)ix * g.C), acc[ky * 3 + kx]);
        }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    sh[threadIdx.x] = acc[k];
    __syncthreads();
    if (t.ty == 0 && t.active) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        double s = lane(acc[k], j);
        for (int i = 1; i < t.tr; ++i) s += (double)lane(sh[i * t.tc + t.tx], j);
        partial[((long long)blockIdx.x * 9 + k) * g.C + t.c + j] = s;
      }
    }
    __syncthreads();
  }
}

// dweight[c][tap] ((C, 1, 3, 3) layout) = the splits' partials summed in split order
__global__ void wgrad_finalize_kernel(int R, int C, const double* __restrict__ partial, float* __restrict__ dweight) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C * 9) return;
  const int c = i / 9, k = i - c * 9;
  double s = 0.0;
  for (int r = 0; r < R; ++r) s += partial[((long long)r * 9 + k) * C + c];
  dweight[i] = (float)s;
}

// ---- BatchNorm + ReLU6 / linear BatchNorm (+ residual) ----
__device__ __forceinline__ float bn_invstd(float var, float eps) { return 1.f / sqrtf(var + eps); }

// z = (x - mean) * invstd * w + b, rounded step by step so that the apply pass and the backward passes (which recompute z for the
// ReLU6 mask) agree bit for bit
__device__ __forceinline__ float bn_z(float x, float m, float is, float w, float b) {
  return __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(x, m), is), w), b);
}

// the gradient passes through ReLU6 where 0 < z < 6 (strictly, as torch's hardtanh_backward); everywhere for the linear BatchNorm
__device__ __forceinline__ float act_grad(float z, float g, int relu6) { return !relu6 || (z > 0.f && z < 6.f) ? g : 0.f; }

struct BnAct {
  const float *mean, *var, *w, *b;
  float eps;
  int relu6;
};

// out = relu6(z) or z + residual, four channels per thread
__global__ void __launch_bounds__(kThreads)
bnact_apply_kernel(long long P, int C, const float* __restrict__ x, int ldx, BnAct a, const float* __restrict__ res, int ldr,
                   float* __restrict__ out, int ldo) {
  const int c4 = C >> 2;
  const long long total = P * c4;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
    const int c = (int)(i % c4) * 4; const long long r = i / c4;
    const float4 xv = ld4(x + r * ldx + c);
    const float4 rv = res ? ld4(res + r * ldr + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 y;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float z = bn_z(lane(xv, j), a.mean[c + j], bn_invstd(a.var[c + j], a.eps), a.w[c + j], a.b[c + j]);
      set_lane(y, j, a.relu6 ? fminf(fmaxf(z, 0.f), 6.f) : (res ? __fadd_rn(lane(rv, j), z) : z));
    }
    st4(out + r * ldo + c, y);
  }
}

// partial[split][c] = (sum dz, sum dz * xhat), dz = dout * act'(z)
__global__ void __launch_bounds__(kThreads)
bnact_bwd_partial_kernel(long long P, int C, const float* __restrict__ x, int ldx, const float* __restrict__ dout, int ldd, BnAct a,
                         double2* __restrict__ partial) {
  __shared__ double2 sh[4][kThreads];
  const Tile4 t = tile4_of(P, C);
  double s1[4] = {0.0, 0.0, 0.0, 0.0}, s2[4] = {0.0, 0.0, 0.0, 0.0};
  if (t.active) {
    float m[4], is[4], wc[4], bc[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      m[j] = a.mean[t.c + j]; is[j] = bn_invstd(a.var[t.c + j], a.eps); wc[j] = a.w[t.c + j]; bc[j] = a.b[t.c + j];
    }
    for (long long r = t.r0 + t.ty; r < t.r1; r += t.tr) {
      const float4 xv = ld4(x + r * ldx + t.c), gv = ld4(dout + r * ldd + t.c);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float xs = lane(xv, j);
        const float dz = act_grad(bn_z(xs, m[j], is[j], wc[j], bc[j]), lane(gv, j), a.relu6);
        s1[j] += (double)dz;
        s2[j] += (double)dz * (double)((xs - m[j]) * is[j]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) sh[j][threadIdx.x] = make_double2(s1[j], s2[j]);
  __syncthreads();
  if (t.ty == 0 && t.active) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      double p1 = s1[j], p2 = s2[j];
      for (int k = 1; k < t.tr; ++k) { const double2 p = sh[j][k * t.tc + t.tx]; p1 += p.x; p2 += p.y; }
      partial[(long long)blockIdx.x * C + t.c + j] = make_double2(p1, p2);
    }
  }
}

// dweight = sum dz * xhat, dbias = sum dz (each may be NULL); coef = (mean dz, mean dz * xhat) for the dx pass
__global__ void bnact_bwd_finalize_kernel(int R, int C, const double2* __restrict__ partial, double count, float* __restrict__ dweight,
                                          float* __restrict__ dbias, float* __restrict__ coef) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double s1 = 0.0, s2 = 0.0;
  for (int r = 0; r < R; ++r) { const double2 p = partial[(long long)r * C + c]; s1 += p.x; s2 += p.y; }
  if (dweight) dweight[c] = (float)s2;
  if (dbias) dbias[c] = (float)s1;
  coef[c] = (float)(s1 / count); coef[C + c] = (float)(s2 / count);
}

// dx = w * invstd * (dz - mean dz - xhat * mean(dz xhat)) with batch statistics, w * invstd * dz with running statistics
__global__ void __launch_bounds__(kThreads)
bnact_dx_kernel(long long P, int C, const float* __restrict__ x, int ldx, const float* __restrict__ dout, int ldd, BnAct a, int training,
                const float* __restrict__ coef, float* __restrict__ dx, int lddx) {
  const int c4 = C >> 2;
  const long long total = P * c4;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
    const int c = (int)(i % c4) * 4; const long long r = i / c4;
    const float4 xv = ld4(x + r * ldx + c), gv = ld4(dout + r * ldd + c);
    float4 d;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float m = a.mean[c + j], is = bn_invstd(a.var[c + j], a.eps), wc = a.w[c + j];
      const float xs = lane(xv, j);
      const float dz = act_grad(bn_z(xs, m, is, wc, a.b[c + j]), lane(gv, j), a.relu6);
      float v;
      if (!training) v = dz * (wc * is);
      else v = (dz - coef[c + j] - (xs - m) * is * coef[C + c + j]) * (wc * is);
      set_lane(d, j, v);
    }
    st4(dx + r * lddx + c, d);
  }
}

bool dw_geom(const char* where, int N, int H, int W, int C, int stride, int dilation, DwGeom& g) {
  if (N <= 0 || H <= 0 || W <= 0 || C <= 0 || C % 4 || (stride != 1 && stride != 2) || dilation < 1) {
    set_error_msg(where, "depthwise 3x3: needs C a multiple of 4, stride 1 or 2, dilation >= 1 (padding = dilation)");
    return false;
  }
  g = DwGeom{N, H, W, C, (H - 1) / stride + 1, (W - 1) / stride + 1, stride, dilation};
  return true;
}

bool bn_shape_ok(long long P, int C, std::initializer_list<int> pitches, std::initializer_list<const void*> ptrs) {
  if (P <= 0 || C <= 0 || C % 4) return false;
  for (int ld : pitches) if (ld < C || ld % 4) return false;
  for (const void* p : ptrs) if (!aligned16(p)) return false;
  return true;
}

}  // namespace

extern "C" long long skd_mbv2_workspace_doubles(long long P, int C) {
  const long long stats = 2LL * splits_of(P, C, kStatBlocks) * C, wgrad = 9LL * splits_of(P, C, kWgradBlocks) * C;
  return stats > wgrad ? stats : wgrad;
}

extern "C" int skd_dwconv3x3_fwd(int N, int H, int W, int C, int stride, int dilation, const float* x, const float* weight, float* y,
                                 float momentum, float* running_mean, float* running_var, long long* num_batches_tracked, float* mean,
                                 float* var, double* workspace, cudaStream_t st) {
  DwGeom g;
  if (!dw_geom("skd_dwconv3x3_fwd", N, H, W, C, stride, dilation, g)) return 0;
  if (!aligned16(x) || !aligned16(y)) { set_error_msg("skd_dwconv3x3_fwd", "x / y must be 16-byte aligned"); return 0; }
  const long long P = (long long)N * g.OH * g.OW;
  const dim3 grid(splits_of(P, C, kStatBlocks), chunks_of(C));
  if (!mean) {
    dw_fwd_kernel<false><<<grid, kThreads, 0, st>>>(g, x, weight, y, nullptr);
    return finish("skd_dwconv3x3_fwd");
  }
  double2* part = reinterpret_cast<double2*>(workspace);
  dw_fwd_kernel<true><<<grid, kThreads, 0, st>>>(g, x, weight, y, part);
  stats_finalize_kernel<<<(C + 127) / 128, 128, 0, st>>>(grid.x, C, part, (double)P, momentum, running_mean, running_var,
                                                          num_batches_tracked, mean, var);
  return finish("skd_dwconv3x3_fwd", 2);
}

extern "C" int skd_dwconv3x3_dgrad(int N, int H, int W, int C, int stride, int dilation, const float* dy, const float* weight, float* dx,
                                   cudaStream_t st) {
  DwGeom g;
  if (!dw_geom("skd_dwconv3x3_dgrad", N, H, W, C, stride, dilation, g)) return 0;
  if (!aligned16(dy) || !aligned16(dx)) { set_error_msg("skd_dwconv3x3_dgrad", "dy / dx must be 16-byte aligned"); return 0; }
  const long long P = (long long)N * H * W;
  dw_dgrad_kernel<<<dim3(splits_of(P, C, kStatBlocks), chunks_of(C)), kThreads, 0, st>>>(g, dy, weight, dx);
  return finish("skd_dwconv3x3_dgrad");
}

extern "C" int skd_dwconv3x3_wgrad(int N, int H, int W, int C, int stride, int dilation, const float* x, const float* dy, float* dweight,
                                   double* workspace, cudaStream_t st) {
  DwGeom g;
  if (!dw_geom("skd_dwconv3x3_wgrad", N, H, W, C, stride, dilation, g)) return 0;
  if (!aligned16(x) || !aligned16(dy)) { set_error_msg("skd_dwconv3x3_wgrad", "x / dy must be 16-byte aligned"); return 0; }
  const long long P = (long long)N * g.OH * g.OW;
  const dim3 grid(splits_of(P, C, kWgradBlocks), chunks_of(C));
  dw_wgrad_kernel<<<grid, kThreads, 0, st>>>(g, x, dy, workspace);
  wgrad_finalize_kernel<<<(C * 9 + 255) / 256, 256, 0, st>>>(grid.x, C, workspace, dweight);
  return finish("skd_dwconv3x3_wgrad", 2);
}

extern "C" int skd_bnact_apply(long long P, int C, int relu6, const float* x, int ldx, const float* mean, const float* var,
                               const float* weight, const float* bias, float eps, const float* residual, int ldr, float* out, int ldo,
                               cudaStream_t st) {
  if (!bn_shape_ok(P, C, {ldx, ldo, residual ? ldr : C}, {x, out, residual}) || (relu6 && residual)) {
    set_error_msg("skd_bnact_apply", "bad shape (C and pitches multiples of 4, 16-byte aligned rows; no residual with ReLU6)");
    return 0;
  }
  const BnAct a{mean, var, weight, bias, eps, relu6};
  bnact_apply_kernel<<<ew_grid(P * (C / 4)), kThreads, 0, st>>>(P, C, x, ldx, a, residual, ldr, out, ldo);
  return finish("skd_bnact_apply");
}

extern "C" int skd_bnact_bwd_reduce(long long P, int C, int relu6, const float* x, int ldx, const float* dout, int ldd, const float* mean,
                                    const float* var, const float* weight, const float* bias, float eps, float* dweight, float* dbias,
                                    float* coef, double* workspace, cudaStream_t st) {
  if (!bn_shape_ok(P, C, {ldx, ldd}, {x, dout})) { set_error_msg("skd_bnact_bwd_reduce", "bad shape"); return 0; }
  const BnAct a{mean, var, weight, bias, eps, relu6};
  const dim3 grid(splits_of(P, C, kStatBlocks), chunks_of(C));
  double2* part = reinterpret_cast<double2*>(workspace);
  bnact_bwd_partial_kernel<<<grid, kThreads, 0, st>>>(P, C, x, ldx, dout, ldd, a, part);
  bnact_bwd_finalize_kernel<<<(C + 127) / 128, 128, 0, st>>>(grid.x, C, part, (double)P, dweight, dbias, coef);
  return finish("skd_bnact_bwd_reduce", 2);
}

extern "C" int skd_bnact_bwd_dx(long long P, int C, int relu6, const float* x, int ldx, const float* dout, int ldd, const float* mean,
                                const float* var, const float* weight, const float* bias, float eps, int training, const float* coef,
                                float* dx, int lddx, cudaStream_t st) {
  if (!bn_shape_ok(P, C, {ldx, ldd, lddx}, {x, dout, dx})) { set_error_msg("skd_bnact_bwd_dx", "bad shape"); return 0; }
  const BnAct a{mean, var, weight, bias, eps, relu6};
  bnact_dx_kernel<<<ew_grid(P * (C / 4)), kThreads, 0, st>>>(P, C, x, ldx, dout, ldd, a, training, coef, dx, lddx);
  return finish("skd_bnact_bwd_dx");
}
