// SIMT direct convolutions (NHWC, fp32 FMA) for the shapes the wgmma path does not take:
//   * the 3-channel stem convolution (Cin=3: K=27, nothing for a tensor core to chew on; HBM-bound on its output)
//   * strided data-gradients (two student convs) until they move to the sub-grid wgmma formulation
// They are also the on-device cross-check for the tensor-core kernels in tests (exact fp32 accumulation order aside).
#include "common.cuh"
#include "skd.h"

using namespace skd;

namespace {

struct Geo { int N, H, W, Cin, OH, OW, Cout, KH, KW, stride, pad, dil; };

// thread <-> (pixel, co); x reads are warp-broadcast, w reads hit L1
__global__ void __launch_bounds__(256)
direct_fwd_kernel(Geo g, const float* __restrict__ x, int ldx, const float* __restrict__ w, float* __restrict__ y, int ldy,
                  const float* __restrict__ scale, const float* __restrict__ shift, int act, float slope) {
  const long long total = (long long)g.N * g.OH * g.OW * g.Cout;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int co = (int)(i % g.Cout); long long p = i / g.Cout;
    const int ox = (int)(p % g.OW); long long r = p / g.OW; const int oy = (int)(r % g.OH), n = (int)(r / g.OH);
    float acc = 0.f;
    for (int kh = 0; kh < g.KH; ++kh) {
      const int iy = oy * g.stride - g.pad + kh * g.dil;
      if (iy < 0 || iy >= g.H) continue;
      for (int kw = 0; kw < g.KW; ++kw) {
        const int ix = ox * g.stride - g.pad + kw * g.dil;
        if (ix < 0 || ix >= g.W) continue;
        const float* xp = x + (((size_t)n * g.H + iy) * g.W + ix) * ldx;
        const float* wp = w + ((size_t)co * g.KH * g.KW + kh * g.KW + kw) * g.Cin;
        for (int ci = 0; ci < g.Cin; ++ci) acc = fmaf(__ldg(xp + ci), __ldg(wp + ci), acc);
      }
    }
    if (scale) acc *= __ldg(scale + co);
    if (shift) acc += __ldg(shift + co);
    y[p * ldy + co] = act_fwd(acc, act, slope);
  }
}

// dx[n,iy,ix,ci] = sum_{kh,kw,co} dy[n,oy,ox,co] * w[co,kh,kw,ci],  iy = oy*s - p + kh*d
__global__ void __launch_bounds__(256)
direct_dgrad_kernel(Geo g, const float* __restrict__ dy, int ldy, const float* __restrict__ w, float* __restrict__ dx, int ldx) {
  const long long total = (long long)g.N * g.H * g.W * g.Cin;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ci = (int)(i % g.Cin); long long p = i / g.Cin;
    const int ix = (int)(p % g.W); long long r = p / g.W; const int iy = (int)(r % g.H), n = (int)(r / g.H);
    float acc = 0.f;
    for (int kh = 0; kh < g.KH; ++kh) {
      const int ty = iy + g.pad - kh * g.dil;
      if (ty < 0 || ty % g.stride) continue;
      const int oy = ty / g.stride;
      if (oy >= g.OH) continue;
      for (int kw = 0; kw < g.KW; ++kw) {
        const int tx = ix + g.pad - kw * g.dil;
        if (tx < 0 || tx % g.stride) continue;
        const int ox = tx / g.stride;
        if (ox >= g.OW) continue;
        const float* dp = dy + (((size_t)n * g.OH + oy) * g.OW + ox) * ldy;
        const float* wp = w + (size_t)(kh * g.KW + kw) * g.Cin + ci;
        const size_t wstride = (size_t)g.KH * g.KW * g.Cin;
        for (int co = 0; co < g.Cout; ++co) acc = fmaf(__ldg(dp + co), __ldg(wp + co * wstride), acc);
      }
    }
    dx[p * ldx + ci] = acc;
  }
}

// The two reductions below give each output column group ONE CTA that walks all pixels and adds its warps' partials in fixed order:
// deterministic (a training run is bit-reproducible), and -- unlike a cluster-wide reduction -- they need no co-scheduled SMs, so they
// still slip in beside the persistent convolution kernels of the overlapping streams.
constexpr int kWgWarps = 16;

// dw[co,kh,kw,ci] = sum_pixels dy[p,co] * x[p shifted, ci]: one CTA per (tap, 32 input channels, 32 output channels).  Lane = input
// channel (coalesced x reads), warp = pixel phase; each lane keeps the 32 output channels' sums, the dy row arrives by one coalesced load
// and warp shuffles.
__global__ void __launch_bounds__(kWgWarps * 32)
direct_wgrad_kernel(Geo g, const float* __restrict__ x, int ldx, const float* __restrict__ dy, int ldy, float* __restrict__ dw) {
  __shared__ float red[kWgWarps / 2][32][33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int ci_tiles = (g.Cin + 31) / 32, co_tiles = (g.Cout + 31) / 32;
  const int cot = blockIdx.x % co_tiles, r0 = blockIdx.x / co_tiles;
  const int cit = r0 % ci_tiles, tap = r0 / ci_tiles;
  const int kh = tap / g.KW, kw = tap - kh * g.KW;
  const int ci = cit * 32 + lane, co_lane = cot * 32 + lane;
  const long long P = (long long)g.N * g.OH * g.OW;
  float acc[32];
#pragma unroll
  for (int c = 0; c < 32; ++c) acc[c] = 0.f;
  long long p = warp;
  int ox = (int)(p % g.OW); long long r = p / g.OW; int oy = (int)(r % g.OH), n = (int)(r / g.OH);
  for (; p < P; p += kWgWarps) {
    const int iy = oy * g.stride - g.pad + kh * g.dil, ix = ox * g.stride - g.pad + kw * g.dil;
    if (iy >= 0 && iy < g.H && ix >= 0 && ix < g.W) {                     // warp-uniform
      const float xv = ci < g.Cin ? __ldg(x + (((size_t)n * g.H + iy) * g.W + ix) * ldx + ci) : 0.f;
      const float dv = co_lane < g.Cout ? __ldg(dy + p * ldy + co_lane) : 0.f;
#pragma unroll
      for (int c = 0; c < 32; ++c) acc[c] = fmaf(__shfl_sync(0xffffffffu, dv, c), xv, acc[c]);
    }
    ox += kWgWarps;
    while (ox >= g.OW) { ox -= g.OW; if (++oy == g.OH) { oy = 0; ++n; } }
  }
  // warps w and w + 8 first, then the eight sums in order
  constexpr int H = kWgWarps / 2;
  if (warp >= H) {
#pragma unroll
    for (int c = 0; c < 32; ++c) red[warp - H][c][lane] = acc[c];
  }
  __syncthreads();
  if (warp < H) {
#pragma unroll
    for (int c = 0; c < 32; ++c) red[warp][c][lane] = acc[c] + red[warp][c][lane];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 32 * 32; i += kWgWarps * 32) {
    const int c = i >> 5, l = i & 31, co = cot * 32 + c, cc = cit * 32 + l;
    if (co >= g.Cout || cc >= g.Cin) continue;
    float t = red[0][c][l];
    for (int w = 1; w < H; ++w) t += red[w][c][l];
    dw[((size_t)co * g.KH * g.KW + tap) * g.Cin + cc] = t;
  }
}

// db[c] (+)= sum_rows dy[row][c]  (conv bias gradient; also used for the 19-class heads): 32 columns x 32 row lanes per CTA
__global__ void __launch_bounds__(1024)
colsum_kernel(const float* __restrict__ dy, int ldy, long long P, int C, float* __restrict__ db, int accumulate) {
  __shared__ float sh[32][33];
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int lane_r = threadIdx.x >> 5;
  float a = 0.f;
  if (c < C) for (long long p = lane_r; p < P; p += 32) a += __ldg(dy + p * ldy + c);
  sh[lane_r][threadIdx.x & 31] = a;
  __syncthreads();
  if (lane_r == 0 && c < C) {
    for (int k = 1; k < 32; ++k) a += sh[k][threadIdx.x & 31];
    db[c] = accumulate ? db[c] + a : a;
  }
}

// Explicit im2col for tiny-Cin convolutions (the 3-channel stem): col[p][(kh*KW+kw)*Cin + ci], zero padded to Kp columns.
// With K = 27 a tensor-core implicit GEMM would spend 9 mostly-empty K steps per tile; one dense 32-wide K step on this
// matrix (134 MB at batch 8) is 5x cheaper, and the weight gradient becomes a single-tap GEMM over the same matrix.
// CIN / KHW > 0: compile-time channel count and (square) filter size -- the index arithmetic (six divisions per element) folds into
// multiplies; 0: run-time values.  The stem convolution (3 channels, 3x3) is the only caller on the path.
template <int CIN, int KHW>
__global__ void __launch_bounds__(256)
im2col_small_kernel(Geo g, const float* __restrict__ x, int ldx, float* __restrict__ col, int Kp) {
  if (CIN > 0) { g.Cin = CIN; g.KH = KHW; g.KW = KHW; }
  const long long total = (long long)g.N * g.OH * g.OW * (Kp / 4);
  const int K = g.KH * g.KW * g.Cin;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int k4 = (int)(i % (Kp / 4)); const long long p = i / (Kp / 4);
    const int ox = (int)(p % g.OW); const long long r = p / g.OW; const int oy = (int)(r % g.OH), n = (int)(r / g.OH);
    float v[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int k = k4 * 4 + t;
      float val = 0.f;
      if (k < K) {
        const int ci = k % g.Cin, tap = k / g.Cin, kh = tap / g.KW, kw = tap - kh * g.KW;
        const int iy = oy * g.stride - g.pad + kh * g.dil, ix = ox * g.stride - g.pad + kw * g.dil;
        if (iy >= 0 && iy < g.H && ix >= 0 && ix < g.W) val = __ldg(x + (((size_t)n * g.H + iy) * g.W + ix) * ldx + ci);
      }
      v[t] = val;
    }
    reinterpret_cast<float4*>(col)[i] = make_float4(v[0], v[1], v[2], v[3]);
  }
}

int ew_blocks(long long total) {
  long long b = (total + 255) / 256;
  if (b > kNumSMs * 32) b = kNumSMs * 32;
  if (b < 1) b = 1;
  return (int)b;
}

Geo make_geo(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil) {
  Geo g; g.N = N; g.H = H; g.W = W; g.Cin = Cin; g.Cout = Cout; g.KH = KH; g.KW = KW; g.stride = stride; g.pad = pad; g.dil = dil;
  g.OH = (H + 2 * pad - dil * (KH - 1) - 1) / stride + 1; g.OW = (W + 2 * pad - dil * (KW - 1) - 1) / stride + 1;
  return g;
}

}  // namespace

extern "C" int skd_conv2d_fwd_direct(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil,
                                     const float* x, int ldx, const float* w, float* y, int ldy, const float* scale,
                                     const float* shift, int act, float slope, cudaStream_t st) {
  const Geo g = make_geo(N, H, W, Cin, Cout, KH, KW, stride, pad, dil);
  if (g.OH <= 0 || g.OW <= 0) return 1;
  direct_fwd_kernel<<<ew_blocks((long long)N * g.OH * g.OW * Cout), 256, 0, st>>>(g, x, ldx, w, y, ldy, scale, shift, act, slope);
  return finish("skd_conv2d_fwd_direct");
}

extern "C" int skd_conv2d_dgrad_direct(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil,
                                       const float* dy, int ldy, const float* w, float* dx, int ldx, cudaStream_t st) {
  const Geo g = make_geo(N, H, W, Cin, Cout, KH, KW, stride, pad, dil);
  direct_dgrad_kernel<<<ew_blocks((long long)N * H * W * Cin), 256, 0, st>>>(g, dy, ldy, w, dx, ldx);
  return finish("skd_conv2d_dgrad_direct");
}

extern "C" int skd_conv2d_wgrad_direct(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil,
                                       const float* x, int ldx, const float* dy, int ldy, float* dw, cudaStream_t st) {
  const Geo g = make_geo(N, H, W, Cin, Cout, KH, KW, stride, pad, dil);
  direct_wgrad_kernel<<<KH * KW * ((Cin + 31) / 32) * ((Cout + 31) / 32), kWgWarps * 32, 0, st>>>(g, x, ldx, dy, ldy, dw);
  return finish("skd_conv2d_wgrad_direct");
}

static int colsum_launch(long long P, int C, const float* dy, int ldy, float* db, bool accumulate, cudaStream_t st) {
  colsum_kernel<<<(C + 31) / 32, 1024, 0, st>>>(dy, ldy, P, C, db, accumulate ? 1 : 0);
  return finish("skd_colsum");
}
extern "C" int skd_colsum(long long P, int C, const float* dy, int ldy, float* db, cudaStream_t st) { return colsum_launch(P, C, dy, ldy, db, false, st); }
// db += column sums (the bias gradient of the second and third discriminator pass of a phase accumulates in place)
extern "C" int skd_colsum_acc(long long P, int C, const float* dy, int ldy, float* db, cudaStream_t st) { return colsum_launch(P, C, dy, ldy, db, true, st); }

extern "C" int skd_im2col_small(int N, int H, int W, int Cin, int KH, int KW, int stride, int pad, int dil, const float* x, int ldx,
                                float* col, int Kp, cudaStream_t st) {
  if (Kp % 4 || Kp < KH * KW * Cin) { set_error_msg("skd_im2col_small", "Kp must be a multiple of 4 and >= KH*KW*Cin"); return 0; }
  const Geo g = make_geo(N, H, W, Cin, 1, KH, KW, stride, pad, dil);
  const int blocks = ew_blocks((long long)N * g.OH * g.OW * (Kp / 4));
  if (Cin == 3 && KH == 3 && KW == 3) im2col_small_kernel<3, 3><<<blocks, 256, 0, st>>>(g, x, ldx, col, Kp);
  else im2col_small_kernel<0, 0><<<blocks, 256, 0, st>>>(g, x, ldx, col, Kp);
  return finish("skd_im2col_small");
}
