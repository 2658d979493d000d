// ESPNet-C student (networks/espnet.py): BatchNorm + PReLU in NHWC with row pitch (channel slices of concat buffers are addressed
// through an offset pointer), the ESP module's combine (hierarchical feature fusion + concatenation + residual) fused with the
// BatchNorm statistics, its backward fused with the BatchNorm + PReLU input-gradient pass, and the input projection (3x3 / stride 2
// average pooling of the image straight into a concat buffer's channel slice), and the teacher's resample onto the student's grid.
// The full ESPNet's decoder adds plain BatchNorm (the BN + PReLU kernels with alpha == NULL) and the adjoint of the bilinear resample
// (the discriminator sees the full-resolution student logits resized onto the teacher's grid).
//
// Every reduction adds in a fixed order (row splits fixed by (P, C), partials in double, split order in the finalize pass), so
// two runs of a step give bit-identical results.  The kernels are scalar per channel: ESPNet-C's channel counts (19, 25, 131, ...)
// are not multiples of 4, and these passes are a small part of a distillation step whose teacher does ~170x the arithmetic.
#include "common.cuh"
#include "skd.h"

using namespace skd;

namespace {

constexpr int kThreads = 256;

// The ESP module's five branch outputs (d1: n1 channels, pitch ld1; d2 / d4 / d8 / d16: n channels, pitch ldn) and the optional
// residual (the block input, nOut = n1 + 4n channels, pitch ldr).
struct EspSrc {
  const float *d1, *d2, *d4, *d8, *d16, *res;
  int ld1, ldn, ldr, n1, n;
};

// combine[c] = [d1 | a1 | a2 | a3 | a4][c] (+ residual[c]) with a1 = d2, a2 = a1 + d4, a3 = a2 + d8, a4 = a3 + d16: the additions of the
// plain-torch module, in its order
__device__ __forceinline__ float esp_combine_at(const EspSrc& s, long long row, int c) {
  float v;
  if (c < s.n1) {
    v = s.d1[row * s.ld1 + c];
  } else {
    const int j = (c - s.n1) / s.n, k = (c - s.n1) - j * s.n;
    const long long o = row * s.ldn + k;
    v = s.d2[o];
    if (j >= 1) v = __fadd_rn(v, s.d4[o]);
    if (j >= 2) v = __fadd_rn(v, s.d8[o]);
    if (j >= 3) v = __fadd_rn(v, s.d16[o]);
  }
  if (s.res) v = __fadd_rn(s.res[row * s.ldr + c], v);
  return v;
}

__device__ __forceinline__ float bn_invstd(float var, float eps) { return 1.f / sqrtf(var + eps); }

// PReLU slope of channel c; alpha == NULL is plain BatchNorm (slope 1: every product below with it is exact, so z and dz pass unchanged)
__device__ __forceinline__ float slope_of(const float* __restrict__ alpha, int c) { return alpha ? alpha[c] : 1.f; }

// BatchNorm output before the PReLU, z = (x - mean) * invstd * w + b, rounded step by step so that the apply pass and the backward
// passes (which recompute z for the PReLU mask) agree bit for bit
__device__ __forceinline__ float bn_z(float x, float m, float is, float w, float b) {
  return __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(x, m), is), w), b);
}

struct Tile {             // a block's channel chunk and its share of the rows
  int tc, tr, tx, ty, c;
  long long r0, r1;
  bool active;
};
__device__ __forceinline__ Tile tile_of(long long P, int C) {
  Tile t;
  t.tc = C < kThreads ? C : kThreads;
  t.tr = kThreads / t.tc;
  t.tx = threadIdx.x % t.tc; t.ty = threadIdx.x / t.tc;
  t.c = blockIdx.y * t.tc + t.tx;
  t.active = t.ty < t.tr && t.c < C;
  const long long per = (P + gridDim.x - 1) / gridDim.x;
  t.r0 = (long long)blockIdx.x * per;
  t.r1 = t.r0 + per < P ? t.r0 + per : P;
  return t;
}

// partial[split][c] = (sum x, sum x^2) over the split's rows.  kCombine: x is the ESP combine, computed here and written to out.
template <bool kCombine>
__global__ void __launch_bounds__(kThreads)
stats_partial_kernel(long long P, int C, const float* __restrict__ x, int ldx, EspSrc src, float* __restrict__ out, int ldo,
                     double2* __restrict__ partial) {
  __shared__ double2 sh[kThreads];
  const Tile t = tile_of(P, C);
  double s1 = 0.0, s2 = 0.0;
  if (t.active) {
    for (long long r = t.r0 + t.ty; r < t.r1; r += t.tr) {
      float v;
      if (kCombine) { v = esp_combine_at(src, r, t.c); out[r * ldo + t.c] = v; }
      else v = x[r * ldx + t.c];
      s1 += (double)v; s2 += (double)v * (double)v;
    }
  }
  if (!partial) return;
  sh[threadIdx.x] = make_double2(s1, s2);
  __syncthreads();
  if (t.ty == 0 && t.active) {
    for (int k = 1; k < t.tr; ++k) { const double2 p = sh[k * t.tc + t.tx]; s1 += p.x; s2 += p.y; }
    partial[(long long)blockIdx.x * C + t.c] = make_double2(s1, s2);
  }
}

// mean, biased variance; running statistics with the unbiased variance n / (n - 1) and momentum, as torch's BatchNorm2d
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

// out[r][c] = prelu(bn(x[r][c])) for c < C, 0 for C <= c < Cw (the zero channel padding the next convolution reads)
__global__ void __launch_bounds__(kThreads)
apply_kernel(long long P, int C, int Cw, const float* __restrict__ x, int ldx, const float* __restrict__ mean,
             const float* __restrict__ var, const float* __restrict__ w, const float* __restrict__ b, const float* __restrict__ alpha,
             float eps, float* __restrict__ out, int ldo) {
  const long long total = P * Cw;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
    const int c = (int)(i % Cw); const long long r = i / Cw;
    float y = 0.f;
    if (c < C) {
      const float z = bn_z(x[r * ldx + c], mean[c], bn_invstd(var[c], eps), w[c], b[c]);
      y = z > 0.f ? z : __fmul_rn(slope_of(alpha, c), z);
    }
    out[r * ldo + c] = y;
  }
}

// partial[split][c] = (sum dz, sum dz * xhat, sum_{z <= 0} z * dout), dz = dout * prelu'(z) (torch's PReLU: slope where z <= 0)
__global__ void __launch_bounds__(kThreads)
bwd_partial_kernel(long long P, int C, const float* __restrict__ x, int ldx, const float* __restrict__ dout, int ldd,
                   const float* __restrict__ mean, const float* __restrict__ var, const float* __restrict__ w,
                   const float* __restrict__ b, const float* __restrict__ alpha, float eps, double* __restrict__ partial) {
  __shared__ double sh[3][kThreads];
  const Tile t = tile_of(P, C);
  double s1 = 0.0, s2 = 0.0, s3 = 0.0;
  if (t.active) {
    const float m = mean[t.c], is = bn_invstd(var[t.c], eps), wc = w[t.c], bc = b[t.c], a = slope_of(alpha, t.c);
    for (long long r = t.r0 + t.ty; r < t.r1; r += t.tr) {
      const float xv = x[r * ldx + t.c], g = dout[r * ldd + t.c];
      const float z = bn_z(xv, m, is, wc, bc);
      const float dz = z > 0.f ? g : a * g;
      s1 += (double)dz;
      s2 += (double)dz * (double)((xv - m) * is);
      if (!(z > 0.f)) s3 += (double)z * (double)g;
    }
  }
  sh[0][threadIdx.x] = s1; sh[1][threadIdx.x] = s2; sh[2][threadIdx.x] = s3;
  __syncthreads();
  if (t.ty == 0 && t.active) {
    for (int k = 1; k < t.tr; ++k) { const int j = k * t.tc + t.tx; s1 += sh[0][j]; s2 += sh[1][j]; s3 += sh[2][j]; }
    double* o = partial + ((long long)blockIdx.x * C + t.c) * 3;
    o[0] = s1; o[1] = s2; o[2] = s3;
  }
}

// dweight = sum dz * xhat, dbias = sum dz, dalpha = sum_{z <= 0} z * dout (each may be NULL); coef = (mean dz, mean dz * xhat) for the
// input-gradient pass
__global__ void bwd_finalize_kernel(int R, int C, const double* __restrict__ partial, double count, float* __restrict__ dweight,
                                    float* __restrict__ dbias, float* __restrict__ dalpha, float* __restrict__ coef) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double s1 = 0.0, s2 = 0.0, s3 = 0.0;
  for (int r = 0; r < R; ++r) { const double* p = partial + ((long long)r * C + c) * 3; s1 += p[0]; s2 += p[1]; s3 += p[2]; }
  if (dweight) dweight[c] = (float)s2;
  if (dbias) dbias[c] = (float)s1;
  if (dalpha) dalpha[c] = (float)s3;
  coef[c] = (float)(s1 / count); coef[C + c] = (float)(s2 / count);
}

struct BnArgs {
  const float *x, *dout, *mean, *var, *w, *b, *alpha, *coef;
  int ldx, ldd, C, training;
  float eps;
};

// input gradient of prelu(bn(x)) at (r, c): w * invstd * (dz - mean dz - xhat * mean(dz xhat)) with batch statistics, w * invstd * dz
// with running statistics
__device__ __forceinline__ float bn_dx_at(const BnArgs& a, long long r, int c) {
  const float xv = a.x[r * a.ldx + c], g = a.dout[r * a.ldd + c];
  const float m = a.mean[c], is = bn_invstd(a.var[c], a.eps), wc = a.w[c];
  const float z = bn_z(xv, m, is, wc, a.b[c]);
  const float dz = z > 0.f ? g : slope_of(a.alpha, c) * g;
  if (!a.training) return dz * (wc * is);
  const float xhat = (xv - m) * is;
  return (dz - a.coef[c] - xhat * a.coef[a.C + c]) * (wc * is);
}

__global__ void __launch_bounds__(kThreads)
dx_kernel(long long P, int Cw, BnArgs a, float* __restrict__ dx, int lddx) {
  const long long total = P * Cw;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
    const int c = (int)(i % Cw); const long long r = i / Cw;
    dx[r * lddx + c] = c < a.C ? bn_dx_at(a, r, c) : 0.f;
  }
}

// Backward of the ESP combine, fused with the BatchNorm + PReLU input gradient: g = d(combine); d(d1) = g[0:n1]; the HFF branches get
// the suffix sums over their slices, d16 = g4, d8 = g3 + g4, d4 = g2 + (g3 + g4), d2 = g1 + (g2 + g3 + g4); dres = g (residual).  Pad
// channels of the branch gradients (up to their pitches) are written as zeros.  Thread j of a row: j < ld1 -> d1 channel j,
// else HFF index k = j - ld1 < ldn.
__global__ void __launch_bounds__(kThreads)
esp_dx_kernel(long long P, BnArgs a, int n1, int n, float* __restrict__ dd1, int ld1, float* __restrict__ dd2, float* __restrict__ dd4,
              float* __restrict__ dd8, float* __restrict__ dd16, int ldn, float* __restrict__ dres, int ldr) {
  const int J = ld1 + ldn;
  const long long total = P * J;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
    const int j = (int)(i % J); const long long r = i / J;
    if (j < ld1) {
      float v = 0.f;
      if (j < n1) { v = bn_dx_at(a, r, j); if (dres) dres[r * ldr + j] = v; }
      dd1[r * ld1 + j] = v;
      continue;
    }
    const int k = j - ld1;
    const long long o = r * ldn + k;
    if (k >= n) { dd2[o] = 0.f; dd4[o] = 0.f; dd8[o] = 0.f; dd16[o] = 0.f; continue; }
    float g[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int c = n1 + q * n + k;
      g[q] = bn_dx_at(a, r, c);
      if (dres) dres[r * ldr + c] = g[q];
    }
    float s = g[3];
    dd16[o] = s;
    s = __fadd_rn(g[2], s); dd8[o] = s;
    s = __fadd_rn(g[1], s); dd4[o] = s;
    s = __fadd_rn(g[0], s); dd2[o] = s;
  }
}

// nn.AvgPool2d(3, stride 2, padding 1) (count_include_pad: divide by 9), one output element per thread, taps summed row by row
__global__ void __launch_bounds__(kThreads)
avgpool3s2_kernel(int N, int H, int W, int C, const float* __restrict__ src, int lds, int OH, int OW, float* __restrict__ dst, int ldd) {
  const long long total = (long long)N * OH * OW * C;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
    const int c = (int)(i % C); long long r = i / C;
    const int ox = (int)(r % OW); r /= OW;
    const int oy = (int)(r % OH); const int nimg = (int)(r / OH);
    float s = 0.f;
    for (int ky = 0; ky < 3; ++ky) {
      const int y = 2 * oy - 1 + ky;
      if (y < 0 || y >= H) continue;
      for (int kx = 0; kx < 3; ++kx) {
        const int x = 2 * ox - 1 + kx;
        if (x < 0 || x >= W) continue;
        s = __fadd_rn(s, src[(((long long)nimg * H + y) * W + x) * lds + c]);
      }
    }
    dst[(((long long)nimg * OH + oy) * OW + ox) * ldd + c] = s / 9.f;
  }
}

// out[n][y][x][c] = bilinear (align_corners) resize of src (n, c, h, w; strides sn / sc / sp) to H x W, one output element per thread
__global__ void __launch_bounds__(kThreads)
resample_kernel(int N, int C, int h, int w, const float* __restrict__ src, long long sn, long long sc, long long sp, int H, int W,
                float* __restrict__ out) {
  const long long total = (long long)N * H * W * C;
  const float ry = H > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f, rx = W > 1 ? (float)(w - 1) / (float)(W - 1) : 0.f;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
    const int c = (int)(i % C); long long r = i / C;
    const int x = (int)(r % W); r /= W;
    const int y = (int)(r % H); const int n = (int)(r / H);
    out[i] = up_at(src + n * sn + c * sc, sp, h, w, ry, rx, y, x);
  }
}

// Adjoint of resample_kernel (d src from d out), as a gather: one thread per source element (n, y, x, c) sums, in ascending (oy, ox)
// order, wy * wx * dout over the output pixels whose four taps include (y, x).  The weights are resample_kernel's, recomputed with
// its arithmetic (up_at); a clamped tap (y0 == y1 at the last row / column) receives both of its weights.  No atomics: the result
// does not depend on scheduling.  dout is dense NHWC [N][H][W][C]; dsrc is NHWC with pixel pitch lds.
__device__ __forceinline__ float adj_weight(int o, float r, int n, int i) {
  const float f = o * r;
  const int i0 = min((int)f, n - 1), i1 = min(i0 + 1, n - 1);
  const float l = f - i0;
  return (i0 == i ? 1.f - l : 0.f) + (i1 == i ? l : 0.f);
}

__global__ void __launch_bounds__(kThreads)
resample_adjoint_kernel(int N, int C, int h, int w, const float* __restrict__ dout, int H, int W, float* __restrict__ dsrc, int lds) {
  const long long total = (long long)N * h * w * C;
  const float ry = H > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f, rx = W > 1 ? (float)(w - 1) / (float)(W - 1) : 0.f;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
    const int c = (int)(i % C); long long r = i / C;
    const int x = (int)(r % w); r /= w;
    const int y = (int)(r % h); const int n = (int)(r / h);
    // output rows / columns that can reach y / x: o * ry in (y - 1, y + 1], widened by one for the float rounding of o * ry
    const int oy0 = ry > 0.f ? max(0, (int)floorf((y - 1) / ry) - 1) : 0, oy1 = ry > 0.f ? min(H - 1, (int)ceilf((y + 1) / ry) + 1) : H - 1;
    const int ox0 = rx > 0.f ? max(0, (int)floorf((x - 1) / rx) - 1) : 0, ox1 = rx > 0.f ? min(W - 1, (int)ceilf((x + 1) / rx) + 1) : W - 1;
    float acc = 0.f;
    for (int oy = oy0; oy <= oy1; ++oy) {
      const float wy = adj_weight(oy, ry, h, y);
      if (wy == 0.f) continue;
      const float* row = dout + (((long long)n * H + oy) * W) * C + c;
      float s = 0.f;
      for (int ox = ox0; ox <= ox1; ++ox) {
        const float wx = adj_weight(ox, rx, w, x);
        if (wx != 0.f) s = __fadd_rn(s, __fmul_rn(wx, row[(long long)ox * C]));
      }
      acc = __fadd_rn(acc, __fmul_rn(wy, s));
    }
    dsrc[(((long long)n * h + y) * w + x) * lds + c] = acc;
  }
}

int ew_grid(long long total) {
  long long b = (total + kThreads - 1) / kThreads;
  if (b > kNumSMs * 16) b = kNumSMs * 16;
  return (int)(b < 1 ? 1 : b);
}

int stat_splits(long long P, int C) {
  const int tc = C < kThreads ? C : kThreads;
  const int chunks = (C + tc - 1) / tc;
  long long r = (4LL * kNumSMs + chunks - 1) / chunks;
  const long long cap = (P + 31) / 32;
  if (r > cap) r = cap;
  return (int)(r < 1 ? 1 : r);
}

dim3 stat_grid(long long P, int C) {
  const int tc = C < kThreads ? C : kThreads;
  return dim3(stat_splits(P, C), (C + tc - 1) / tc);
}

}  // namespace

extern "C" long long skd_bnprelu_workspace_doubles(long long P, int C) { return 3LL * stat_splits(P, C) * C; }

extern "C" int skd_bnprelu_stats(long long P, int C, const float* x, int ldx, float momentum, float* running_mean, float* running_var,
                                 long long* num_batches_tracked, float* mean, float* var, double* workspace, cudaStream_t st) {
  if (P <= 0 || C <= 0 || ldx < C) { set_error_msg("skd_bnprelu_stats", "bad shape"); return 0; }
  const dim3 g = stat_grid(P, C);
  EspSrc none{};
  stats_partial_kernel<false><<<g, kThreads, 0, st>>>(P, C, x, ldx, none, nullptr, 0, reinterpret_cast<double2*>(workspace));
  stats_finalize_kernel<<<(C + 127) / 128, 128, 0, st>>>(g.x, C, reinterpret_cast<const double2*>(workspace), (double)P, momentum,
                                                          running_mean, running_var, num_batches_tracked, mean, var);
  return finish("skd_bnprelu_stats", 2);
}

extern "C" int skd_esp_combine(long long P, int n1, int n, const float* d1, int ld1, const float* d2, const float* d4, const float* d8,
                               const float* d16, int ldn, const float* residual, int ldr, float* out, int ldo, float momentum,
                               float* running_mean, float* running_var, long long* num_batches_tracked, float* mean, float* var,
                               double* workspace, cudaStream_t st) {
  const int C = n1 + 4 * n;
  if (P <= 0 || n1 <= 0 || n <= 0 || ld1 < n1 || ldn < n || ldo < C || (residual && ldr < C)) {
    set_error_msg("skd_esp_combine", "bad shape"); return 0;
  }
  const EspSrc s{d1, d2, d4, d8, d16, residual, ld1, ldn, ldr, n1, n};
  const dim3 g = stat_grid(P, C);
  double2* part = mean ? reinterpret_cast<double2*>(workspace) : nullptr;
  stats_partial_kernel<true><<<g, kThreads, 0, st>>>(P, C, nullptr, 0, s, out, ldo, part);
  if (!mean) return finish("skd_esp_combine");
  stats_finalize_kernel<<<(C + 127) / 128, 128, 0, st>>>(g.x, C, part, (double)P, momentum, running_mean, running_var,
                                                          num_batches_tracked, mean, var);
  return finish("skd_esp_combine", 2);
}

extern "C" int skd_bnprelu_apply(long long P, int C, const float* x, int ldx, const float* mean, const float* var, const float* weight,
                                 const float* bias, const float* alpha, float eps, float* out, int ldo, int out_channels, cudaStream_t st) {
  if (P <= 0 || C <= 0 || ldx < C || out_channels < C || ldo < out_channels) { set_error_msg("skd_bnprelu_apply", "bad shape"); return 0; }
  apply_kernel<<<ew_grid(P * out_channels), kThreads, 0, st>>>(P, C, out_channels, x, ldx, mean, var, weight, bias, alpha, eps, out, ldo);
  return finish("skd_bnprelu_apply");
}

extern "C" int skd_bnprelu_bwd_reduce(long long P, int C, const float* x, int ldx, const float* dout, int ldd, const float* mean,
                                      const float* var, const float* weight, const float* bias, const float* alpha, float eps,
                                      float* dweight, float* dbias, float* dalpha, float* coef, double* workspace, cudaStream_t st) {
  if (P <= 0 || C <= 0 || ldx < C || ldd < C) { set_error_msg("skd_bnprelu_bwd_reduce", "bad shape"); return 0; }
  const dim3 g = stat_grid(P, C);
  bwd_partial_kernel<<<g, kThreads, 0, st>>>(P, C, x, ldx, dout, ldd, mean, var, weight, bias, alpha, eps, workspace);
  bwd_finalize_kernel<<<(C + 127) / 128, 128, 0, st>>>(g.x, C, workspace, (double)P, dweight, dbias, dalpha, coef);
  return finish("skd_bnprelu_bwd_reduce", 2);
}

extern "C" int skd_bnprelu_bwd_dx(long long P, int C, const float* x, int ldx, const float* dout, int ldd, const float* mean,
                                  const float* var, const float* weight, const float* bias, const float* alpha, float eps, int training,
                                  const float* coef, float* dx, int lddx, int dx_channels, cudaStream_t st) {
  if (P <= 0 || C <= 0 || dx_channels < C || lddx < dx_channels) { set_error_msg("skd_bnprelu_bwd_dx", "bad shape"); return 0; }
  const BnArgs a{x, dout, mean, var, weight, bias, alpha, coef, ldx, ldd, C, training, eps};
  dx_kernel<<<ew_grid(P * dx_channels), kThreads, 0, st>>>(P, dx_channels, a, dx, lddx);
  return finish("skd_bnprelu_bwd_dx");
}

extern "C" int skd_esp_bwd_dx(long long P, int n1, int n, const float* x, int ldx, const float* dout, int ldd, const float* mean,
                              const float* var, const float* weight, const float* bias, const float* alpha, float eps, int training,
                              const float* coef, float* dd1, int ld1, float* dd2, float* dd4, float* dd8, float* dd16, int ldn,
                              float* dres, int ldr, cudaStream_t st) {
  const int C = n1 + 4 * n;
  if (P <= 0 || n1 <= 0 || n <= 0 || ld1 < n1 || ldn < n || (dres && ldr < C)) { set_error_msg("skd_esp_bwd_dx", "bad shape"); return 0; }
  const BnArgs a{x, dout, mean, var, weight, bias, alpha, coef, ldx, ldd, C, training, eps};
  esp_dx_kernel<<<ew_grid(P * (ld1 + ldn)), kThreads, 0, st>>>(P, a, n1, n, dd1, ld1, dd2, dd4, dd8, dd16, ldn, dres, ldr);
  return finish("skd_esp_bwd_dx");
}

extern "C" int skd_resample_bilinear_nhwc(int N, int C, int h, int w, const float* src, long long sn, long long sc, long long sp, int H,
                                          int W, float* out, cudaStream_t st) {
  if (N <= 0 || C <= 0 || h <= 0 || w <= 0 || H <= 0 || W <= 0) { set_error_msg("skd_resample_bilinear_nhwc", "bad shape"); return 0; }
  resample_kernel<<<ew_grid((long long)N * H * W * C), kThreads, 0, st>>>(N, C, h, w, src, sn, sc, sp, H, W, out);
  return finish("skd_resample_bilinear_nhwc");
}

extern "C" int skd_resample_bilinear_adjoint_nhwc(int N, int C, int h, int w, const float* dout, int H, int W, float* dsrc, int lds,
                                                  cudaStream_t st) {
  if (N <= 0 || C <= 0 || h <= 0 || w <= 0 || H <= 0 || W <= 0 || lds < C) {
    set_error_msg("skd_resample_bilinear_adjoint_nhwc", "bad shape"); return 0;
  }
  resample_adjoint_kernel<<<ew_grid((long long)N * h * w * C), kThreads, 0, st>>>(N, C, h, w, dout, H, W, dsrc, lds);
  return finish("skd_resample_bilinear_adjoint_nhwc");
}

extern "C" int skd_avgpool3x3s2(int N, int H, int W, int C, const float* src, int lds, float* dst, int ldd, cudaStream_t st) {
  if (N <= 0 || H <= 0 || W <= 0 || C <= 0 || lds < C || ldd < C) { set_error_msg("skd_avgpool3x3s2", "bad shape"); return 0; }
  const int OH = (H - 1) / 2 + 1, OW = (W - 1) / 2 + 1;
  avgpool3s2_kernel<<<ew_grid((long long)N * OH * OW * C), kThreads, 0, st>>>(N, H, W, C, src, lds, OH, OW, dst, ldd);
  return finish("skd_avgpool3x3s2");
}
