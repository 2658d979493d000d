// Distillation / task losses for sm_90a (HBM- or latency-bound: SIMT, coalesced, fused; no tensor cores here).
//   * pixel-wise (Pi):  utils/criterion.py:211-226   softmax(T) . log_softmax(S), batch-summed, / (W*H)
//   * pair-wise  (Pa):  utils/criterion.py:228-245 + utils/utils.py:170-183 (ceil-mode max-pool, detached L2 norm,
//                       node affinity, squared difference) -- SIMT path for <= ~1.2k nodes; the 8 385-node regime is
//                       the wgmma kernel in pairwise_sm100.cu
//   * DSN cross entropy: utils/criterion.py:168-188   bilinear(align_corners) upsample + log-softmax + NLL(ignore)
//                       fused so the 2 x 318 MB upsampled logits are never materialised.
// Tensors are addressed with explicit element strides (sn, sc, sp) over (image, channel, pixel) so both NCHW
// (reference layout) and NHWC (our conv layout) feed the same kernels.
#include "common.cuh"
#include "skd.h"

using namespace skd;

namespace {

constexpr int kMaxClasses = 32;

struct Strides { long long sn, sc, sp; };

// deterministic two-stage scalar reduction: per-block partials (double) -> fixed-order final sum
__global__ void finalize_sum_kernel(const double* __restrict__ part, int n, double scale, float* __restrict__ out,
                                    const double* __restrict__ denom_part, int use_denom, float* __restrict__ denom_out) {
  __shared__ double sh[2][32];
  double a = 0.0, b = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) { a += part[i]; if (use_denom) b += denom_part[i]; }
  for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
  if ((threadIdx.x & 31) == 0) { sh[0][threadIdx.x >> 5] = a; sh[1][threadIdx.x >> 5] = b; }
  __syncthreads();
  if (threadIdx.x == 0) {
    a = 0.0; b = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { a += sh[0][i]; b += sh[1][i]; }
    if (use_denom) { out[0] = (float)(a * scale / b); denom_out[0] = (float)b; }
    else out[0] = (float)(a * scale);
  }
}

__device__ __forceinline__ double block_sum_d(double v, double* sh) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x == 0) for (int i = 0; i < (int)((blockDim.x + 31) >> 5); ++i) t += sh[i];
  return t;
}

// ------------------------------------------------------------------------------------------------
// Pixel-wise
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
pixelwise_fwd_kernel(const float* __restrict__ S, const float* __restrict__ T, int N, int C, int HW, Strides ss,
                     Strides ts, double* __restrict__ part) {
  __shared__ double sh[32];
  double acc = 0.0;
  const long long total = (long long)N * HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(i / HW), p = (int)(i - (long long)n * HW);
    const float* sp = S + n * ss.sn + p * ss.sp;
    const float* tp = T + n * ts.sn + p * ts.sp;
    float s[kMaxClasses], t[kMaxClasses];
    float ms = -INFINITY, mt = -INFINITY;
#pragma unroll
    for (int c = 0; c < kMaxClasses; ++c) if (c < C) {
      s[c] = __ldg(sp + c * ss.sc); t[c] = __ldg(tp + c * ts.sc);
      ms = fmaxf(ms, s[c]); mt = fmaxf(mt, t[c]);
    }
    float zs = 0.f, zt = 0.f, dot = 0.f;
#pragma unroll
    for (int c = 0; c < kMaxClasses; ++c) if (c < C) {
      const float et = __expf(t[c] - mt);
      zt += et; zs += __expf(s[c] - ms); dot += et * (s[c] - ms);
    }
    // -sum_c p_T,c * (s_c - ms - log zs) = log zs - dot/zt
    acc += (double)(__logf(zs) - dot / zt);
  }
  double t = block_sum_d(acc, sh);
  if (threadIdx.x == 0) part[blockIdx.x] = t;
}

// dS = g * (softmax(S) - softmax(T)) * inv_hw
__global__ void __launch_bounds__(256)
pixelwise_bwd_kernel(const float* __restrict__ S, const float* __restrict__ T, float* __restrict__ dS, int N, int C,
                     int HW, Strides ss, Strides ts, Strides ds, const float* __restrict__ gout, float mult) {
  const float g = __ldg(gout) * mult;
  const long long total = (long long)N * HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(i / HW), p = (int)(i - (long long)n * HW);
    const float* sp = S + n * ss.sn + p * ss.sp;
    const float* tp = T + n * ts.sn + p * ts.sp;
    float s[kMaxClasses], t[kMaxClasses];
    float ms = -INFINITY, mt = -INFINITY;
#pragma unroll
    for (int c = 0; c < kMaxClasses; ++c) if (c < C) {
      s[c] = __ldg(sp + c * ss.sc); t[c] = __ldg(tp + c * ts.sc);
      ms = fmaxf(ms, s[c]); mt = fmaxf(mt, t[c]);
    }
    float zs = 0.f, zt = 0.f;
#pragma unroll
    for (int c = 0; c < kMaxClasses; ++c) if (c < C) {
      s[c] = __expf(s[c] - ms); t[c] = __expf(t[c] - mt); zs += s[c]; zt += t[c];
    }
    const float rs = 1.f / zs, rt = 1.f / zt;
    float* dp = dS + n * ds.sn + p * ds.sp;
#pragma unroll
    for (int c = 0; c < kMaxClasses; ++c) if (c < C) dp[c * ds.sc] = g * (s[c] * rs - t[c] * rt);
  }
}

// ------------------------------------------------------------------------------------------------
// DSN cross-entropy with fused align_corners bilinear upsampling
// ------------------------------------------------------------------------------------------------
struct Bilin { int i0, i1; float l0, l1; };                 // v = l0*src[i0] + l1*src[i1]
__device__ __forceinline__ Bilin bilin(int dst, float scale, int in) {
  // ATen area_pixel_compute_source_index(align_corners=True): src = scale*dst, scale=(in-1)/(out-1)
  const float src = scale * (float)dst;
  Bilin b;
  b.i0 = (int)src; if (b.i0 > in - 1) b.i0 = in - 1;
  b.i1 = b.i0 + (b.i0 < in - 1 ? 1 : 0);
  b.l1 = src - (float)b.i0; b.l0 = 1.f - b.l1;
  return b;
}

// logits of one upsampled pixel + its log-sum-exp
__device__ __forceinline__ float up_logits(const float* __restrict__ L, Strides st, int n, int C, int w, Bilin by, Bilin bx,
                                           float* v) {
  const float* b = L + n * st.sn;
  const float* p00 = b + ((long long)by.i0 * w + bx.i0) * st.sp; const float* p01 = b + ((long long)by.i0 * w + bx.i1) * st.sp;
  const float* p10 = b + ((long long)by.i1 * w + bx.i0) * st.sp; const float* p11 = b + ((long long)by.i1 * w + bx.i1) * st.sp;
  float m = -INFINITY;
#pragma unroll
  for (int c = 0; c < kMaxClasses; ++c) if (c < C) {
    const long long o = c * st.sc;
    v[c] = by.l0 * (bx.l0 * __ldg(p00 + o) + bx.l1 * __ldg(p01 + o)) + by.l1 * (bx.l0 * __ldg(p10 + o) + bx.l1 * __ldg(p11 + o));
    m = fmaxf(m, v[c]);
  }
  float z = 0.f;
#pragma unroll
  for (int c = 0; c < kMaxClasses; ++c) if (c < C) z += __expf(v[c] - m);
  return m + __logf(z);
}

__global__ void __launch_bounds__(256)
dsn_ce_fwd_kernel(const float* __restrict__ L0, const float* __restrict__ L1, Strides s0, Strides s1,
                  const long long* __restrict__ labels, int N, int C, int h, int w, int H, int W, int ignore, float w0,
                  float w1, double* __restrict__ part_loss, double* __restrict__ part_cnt) {
  __shared__ double sh[32];
  const float sy = H > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f, sx = W > 1 ? (float)(w - 1) / (float)(W - 1) : 0.f;
  double acc = 0.0, cnt = 0.0;
  const long long total = (long long)N * H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int X = (int)(i % W); const long long r = i / W; const int Y = (int)(r % H), n = (int)(r / H);
    const long long lab = labels[i];
    if (lab == ignore) continue;
    const Bilin by = bilin(Y, sy, h), bx = bilin(X, sx, w);
    float v[kMaxClasses];
    float lse = up_logits(L0, s0, n, C, w, by, bx, v);
    float loss = 0.f, pick = 0.f;
#pragma unroll
    for (int c = 0; c < kMaxClasses; ++c) if (c == (int)lab) pick = v[c];
    loss = w0 * (lse - pick);
    if (L1) {
      lse = up_logits(L1, s1, n, C, w, by, bx, v);
#pragma unroll
      for (int c = 0; c < kMaxClasses; ++c) if (c == (int)lab) pick = v[c];
      loss += w1 * (lse - pick);
    }
    acc += (double)loss; cnt += 1.0;
  }
  double t = block_sum_d(acc, sh);
  double u = block_sum_d(cnt, sh);
  if (threadIdx.x == 0) { part_loss[blockIdx.x] = t; part_cnt[blockIdx.x] = u; }
}

// Backward, phase 1: for one output row Y of one image: G[c][X] = softmax - onehot (0 if ignored), then reduce along
// X into the w source columns:  T1[n][Y][x][c] = sum_X wx(x;X) G[c][X].   One block per (Y, n, head).
// The X that feed source column x are contiguous runs (i0 is monotonic in X): those with i0 == x (weight wa = l0, plus l1 where
// the right neighbour is clamped onto the same column) and those with i0 == x-1 (weight wb = l1).  The run starts first[x] are
// found once per chunk, so a (x, c) pair is ~2*W/w shared-memory FMAs.  Lanes run over c (odd row pitch: conflict-free).
// LOSS = true: the same pass also produces the loss (it has every pixel's log-sum-exp in hand): the training forward then IS the
// backward's first phase, and the backward proper is only phase 2 -- one softmax over the 2 x 8 x 512 x 1024 upsampled pixels per
// step instead of two (skd_dsn_ce_fwd_train / skd_dsn_ce_bwd_cols).
// Round 2b: 512 threads and <= 64 registers (two blocks per SM, so one block's reduction phase overlaps the other's softmax phase);
// the two source rows of the logits are blended ONCE per block into shared memory (row[x][c] = ly0 * L[y0][x][c] + ly1 * L[y1][x][c]),
// so a pixel is 2 x C shared-memory reads instead of 4 x C global ones, and the softmax reuses exp(v - max) for the gradient (C
// exponentials per pixel instead of 2 C).  CT: compile-time class bound (19 for Cityscapes; 32 generic).
constexpr int kRowsThreads = 512;
template <bool LOSS, int CT>
__global__ void __launch_bounds__(kRowsThreads, 2)
dsn_ce_bwd_rows_kernel(const float* __restrict__ L0, const float* __restrict__ L1, Strides s0, Strides s1,
                       const long long* __restrict__ labels, int N, int C, int h, int w, int H, int W, int ignore,
                       float* __restrict__ T1, int chunk, double* __restrict__ part_loss, double* __restrict__ part_cnt, float w0, float w1) {
  __shared__ double shd[32];
  double loss_acc = 0.0, cnt_acc = 0.0;
  extern __shared__ float G[];                                 // [C][chunk|1], wa[chunk], wb[chunk], first[w+2], row[w][C]
  const int pitch = chunk | 1;
  float* wa = G + (size_t)C * pitch;
  float* wb = wa + chunk;
  int* first = reinterpret_cast<int*>(wb + chunk);
  float* row = reinterpret_cast<float*>(first + w + 2);
  const int Y = blockIdx.x, n = blockIdx.y, head = blockIdx.z;
  const float* L = head == 0 ? L0 : L1;
  const Strides st = head == 0 ? s0 : s1;
  const float sy = H > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f, sx = W > 1 ? (float)(w - 1) / (float)(W - 1) : 0.f;
  const Bilin by = bilin(Y, sy, h);
  float* out = T1 + (((size_t)head * N + n) * H + Y) * (size_t)C * w;
  {
    const float* b0 = L + n * st.sn + (long long)by.i0 * w * st.sp;
    const float* b1 = L + n * st.sn + (long long)by.i1 * w * st.sp;
    for (int i = threadIdx.x; i < w * C; i += blockDim.x) {
      const int x = i / C, c = i - x * C;
      const long long o = (long long)x * st.sp + (long long)c * st.sc;
      row[i] = by.l0 * __ldg(b0 + o) + by.l1 * __ldg(b1 + o);
    }
  }
  for (int X0 = 0; X0 < W; X0 += chunk) {
    const int X1 = min(W, X0 + chunk);
    __syncthreads();
    for (int x = threadIdx.x; x <= w; x += blockDim.x) first[x] = X1 - X0;
    __syncthreads();
    for (int X = X0 + threadIdx.x; X < X1; X += blockDim.x) {
      const long long lab = labels[((long long)n * H + Y) * W + X];
      const Bilin bx = bilin(X, sx, w);
      const int j = X - X0;
      wa[j] = bx.l0 + (bx.i1 == bx.i0 ? bx.l1 : 0.f);
      wb[j] = bx.i1 == bx.i0 ? 0.f : bx.l1;
      const int prev = X == X0 ? -1 : bilin(X - 1, sx, w).i0;
      for (int x = prev + 1; x <= bx.i0; ++x) first[x] = j;     // first X of the chunk with i0 >= x
      if (lab == ignore) {
#pragma unroll
        for (int c = 0; c < CT; ++c) if (c < C) G[c * pitch + j] = 0.f;
      } else {
        const float* r0 = row + bx.i0 * C;
        const float* r1 = row + bx.i1 * C;
        float v[CT];
        float m = -INFINITY, pick = 0.f;
#pragma unroll
        for (int c = 0; c < CT; ++c) if (c < C) {
          v[c] = bx.l0 * r0[c] + bx.l1 * r1[c];
          m = fmaxf(m, v[c]);
          if (c == (int)lab) pick = v[c];
        }
        float z = 0.f;
#pragma unroll
        for (int c = 0; c < CT; ++c) if (c < C) { v[c] = __expf(v[c] - m); z += v[c]; }
        const float rz = 1.f / z;
#pragma unroll
        for (int c = 0; c < CT; ++c) if (c < C) G[c * pitch + j] = v[c] * rz - (c == (int)lab ? 1.f : 0.f);
        if (LOSS) { loss_acc += (double)(m + __logf(z) - pick); cnt_acc += 1.0; }
      }
    }
    __syncthreads();
    for (int pair = threadIdx.x; pair < C * w; pair += blockDim.x) {
      const int x = pair / C, c = pair - x * C;
      const float* g = G + c * pitch;
      float a = 0.f;
      for (int j = first[x]; j < first[x + 1]; ++j) a += wa[j] * g[j];
      if (x > 0) for (int j = first[x - 1]; j < first[x]; ++j) a += wb[j] * g[j];
      if (X0 == 0) out[pair] = a; else out[pair] += a;
    }
  }
  if (LOSS) {                                                    // fixed-order partials: one per (head, image, output row)
    const double tl = block_sum_d(loss_acc, shd);
    const double tc = block_sum_d(cnt_acc, shd);
    if (threadIdx.x == 0) {
      const size_t idx = ((size_t)head * N + n) * H + Y;
      part_loss[idx] = tl * (double)(head == 0 ? w0 : w1);
      part_cnt[idx] = head == 0 ? tc : 0.0;
    }
  }
}

// Backward, phase 2: dL[n][c][y][x] = g*wh/count * sum_Y wy(y;Y) T1[n][Y][x][c]
__global__ void __launch_bounds__(256)
dsn_ce_bwd_cols_kernel(const float* __restrict__ T1, float* __restrict__ d0, float* __restrict__ d1, Strides a0, Strides a1,
                       int N, int C, int h, int w, int H, const float* __restrict__ gout, const float* __restrict__ count,
                       float w0, float w1) {
  const float sy = H > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f;
  const long long per = (long long)N * h * C * w;
  const int heads = d1 ? 2 : 1;
  const float gc = __ldg(gout) / __ldg(count);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < per * heads; i += (long long)gridDim.x * blockDim.x) {
    const int head = (int)(i / per); long long r = i - (long long)head * per;
    const int c = (int)(r % C); r /= C; const int x = (int)(r % w); r /= w; const int y = (int)(r % h); const int n = (int)(r / h);
    int lo = sy > 0.f ? (int)floorf((float)(y - 1) / sy) : 0, hi = sy > 0.f ? (int)ceilf((float)(y + 1) / sy) : H - 1;
    lo = max(lo - 1, 0); hi = min(hi + 1, H - 1);
    const float* src = T1 + (((size_t)head * N + n) * H) * (size_t)C * w + (size_t)x * C + c;
    float a = 0.f;
    for (int Y = lo; Y <= hi; ++Y) {
      const Bilin by = bilin(Y, sy, h);
      float wgt = 0.f;
      if (by.i0 == y) wgt += by.l0;
      if (by.i1 == y) wgt += by.l1;
      a += wgt * __ldg(src + (size_t)Y * C * w);
    }
    const Strides st = head == 0 ? a0 : a1;
    float* dst = head == 0 ? d0 : d1;
    dst[n * st.sn + c * st.sc + ((long long)y * w + x) * st.sp] = a * gc * (head == 0 ? w0 : w1);
  }
}

// ------------------------------------------------------------------------------------------------
// Pair-wise: ceil-mode max pooling (+argmax), detached-norm normalisation, affinity, squared difference
// ------------------------------------------------------------------------------------------------
// one block per (node, image, channel-chunk of 64): 64 channel lanes x 4 window lanes
__global__ void __launch_bounds__(256)
pa_pool_kernel(const float* __restrict__ F, Strides st, int C, int H, int W, int ph, int pw, int nh, int nw,
               float* __restrict__ pooled, int* __restrict__ argmax) {
  __shared__ float sv[256]; __shared__ int si[256];
  const int node = blockIdx.x, n = blockIdx.y;
  const int cx = threadIdx.x & 63, lane = threadIdx.x >> 6;
  const int c = blockIdx.z * 64 + cx;
  const int ny = node / nw, nx = node - ny * nw;
  const int y0 = ny * ph, x0 = nx * pw, y1 = min(H, y0 + ph), x1 = min(W, x0 + pw);
  const int ww = x1 - x0, cnt = (y1 - y0) * ww;
  float best = -INFINITY; int bi = y0 * W + x0;
  if (c < C) {
    const float* base = F + n * st.sn + c * st.sc;
    for (int k = lane; k < cnt; k += 4) {
      const int y = y0 + k / ww, x = x0 + k % ww;
      const float v = __ldg(base + ((long long)y * W + x) * st.sp);
      if (v > best || (v != v)) { best = v; bi = y * W + x; }       // first max wins inside a lane (k ascending)
    }
  }
  sv[threadIdx.x] = best; si[threadIdx.x] = bi;
  __syncthreads();
  if (lane == 0 && c < C) {
    for (int l = 1; l < 4; ++l) {
      const float v = sv[l * 64 + cx]; const int i = si[l * 64 + cx];
      if (v > best || (v == best && i < bi)) { best = v; bi = i; }   // ties -> smallest index (ATen scan order)
    }
    const size_t o = ((size_t)n * (nh * nw) + node) * C + c;
    pooled[o] = best; if (argmax) argmax[o] = bi;
  }
}

// NHWC variant: 16 channel quads (float4) x 16 window lanes per block -- 4x the loads in flight of the scalar kernel above, which
// walks a 32 x 64 pixel window (pool_scale 0.5) with 4 lanes of dependent scalar loads
__global__ void __launch_bounds__(256)
pa_pool_nhwc_kernel(const float* __restrict__ F, long long sn, int pitch, int C, int H, int W, int ph, int pw, int nh, int nw,
                    float* __restrict__ pooled, int* __restrict__ argmax) {
  __shared__ float4 sv[256]; __shared__ int4 si[256];
  const int node = blockIdx.x, n = blockIdx.y;
  const int cq = threadIdx.x & 15, lane = threadIdx.x >> 4;
  const int c = blockIdx.z * 64 + cq * 4;
  const int ny = node / nw, nx = node - ny * nw;
  const int y0 = ny * ph, x0 = nx * pw, y1 = min(H, y0 + ph), x1 = min(W, x0 + pw);
  const int ww = x1 - x0, cnt = (y1 - y0) * ww;
  float4 best = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
  const int i0 = y0 * W + x0;
  int4 bi = make_int4(i0, i0, i0, i0);
  if (c < C) {
    const float* base = F + n * sn + c;
#define PA_UPD(f, v, idx) if (v > best.f || (v != v)) { best.f = v; bi.f = idx; }
    for (int k = lane; k < cnt; k += 16) {                        // first max wins inside a lane (k ascending)
      const int y = y0 + k / ww, x = x0 + k % ww, idx = y * W + x;
      const float4 v = __ldg(reinterpret_cast<const float4*>(base + (long long)idx * pitch));
      PA_UPD(x, v.x, idx) PA_UPD(y, v.y, idx) PA_UPD(z, v.z, idx) PA_UPD(w, v.w, idx)
    }
#undef PA_UPD
  }
  sv[threadIdx.x] = best; si[threadIdx.x] = bi;
  __syncthreads();
  if (lane == 0 && c < C) {
#define PA_MRG(f) if (v.f > best.f || (v.f == best.f && i.f < bi.f)) { best.f = v.f; bi.f = i.f; }
    for (int l = 1; l < 16; ++l) {                                // ties -> smallest index (ATen scan order)
      const float4 v = sv[l * 16 + cq]; const int4 i = si[l * 16 + cq];
      PA_MRG(x) PA_MRG(y) PA_MRG(z) PA_MRG(w)
    }
#undef PA_MRG
    const size_t o = ((size_t)n * (nh * nw) + node) * C + c;
    *reinterpret_cast<float4*>(pooled + o) = best;
    if (argmax) *reinterpret_cast<int4*>(argmax + o) = bi;
  }
}

// rnorm[n][node] = 1 / (sqrt(sum_c f^2) + 1e-8)     (utils.py:170-171; eps OUTSIDE the sqrt)
__global__ void pa_rnorm_kernel(const float* __restrict__ pooled, int C, float* __restrict__ rnorm) {
  const float* p = pooled + (size_t)blockIdx.x * C;
  float a = 0.f;
  for (int c = threadIdx.x; c < C; c += 32) { const float v = p[c]; a += v * v; }
  a = warp_sum(a);
  if (threadIdx.x == 0) rnorm[blockIdx.x] = 1.f / (sqrtf(a) + 1e-8f);
}

// 32x32 tile of E = A_T - A_S for one image, A = (f_m . f_n) * rnorm_m * rnorm_n.  Accumulates sum E^2.
constexpr int kPT = 32, kPK = 32;
__device__ __forceinline__ float pa_tile_dot(const float* __restrict__ P, int C, int nodes, int m0, int n0,
                                             float (*sa)[kPK + 1], float (*sb)[kPK + 1]) {
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;          // 32 x 8 threads, each thread 4 rows
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int k0 = 0; k0 < C; k0 += kPK) {
    __syncthreads();
    for (int r = ty; r < kPT; r += 8) {
      const int k = k0 + tx;
      sa[r][tx] = (m0 + r < nodes && k < C) ? __ldg(P + (size_t)(m0 + r) * C + k) : 0.f;
      sb[r][tx] = (n0 + r < nodes && k < C) ? __ldg(P + (size_t)(n0 + r) * C + k) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kPK; ++k) {
      const float b = sb[tx][k];
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[j] += sa[ty + 8 * j][k] * b;
    }
  }
  // return through registers: caller reads acc via lambda-less trick -> we pack into smem instead
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 4; ++j) sa[ty + 8 * j][tx] = acc[j];
  __syncthreads();
  return 0.f;
}

__global__ void __launch_bounds__(256)
pa_gram_kernel(const float* __restrict__ PS, const float* __restrict__ PT, const float* __restrict__ rS,
               const float* __restrict__ rT, int CS, int CT, int nodes, float* __restrict__ E, double* __restrict__ part) {
  __shared__ float sa[kPT][kPK + 1], sb[kPT][kPK + 1];
  __shared__ float res[kPT][kPK + 1];
  __shared__ double sh[32];
  const int n = blockIdx.z, m0 = blockIdx.y * kPT, n0 = blockIdx.x * kPT;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  pa_tile_dot(PT + (size_t)n * nodes * CT, CT, nodes, m0, n0, sa, sb);
#pragma unroll
  for (int j = 0; j < 4; ++j) res[ty + 8 * j][tx] = sa[ty + 8 * j][tx];
  pa_tile_dot(PS + (size_t)n * nodes * CS, CS, nodes, m0, n0, sa, sb);
  double acc = 0.0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int m = m0 + ty + 8 * j, q = n0 + tx;
    if (m < nodes && q < nodes) {
      const float at = res[ty + 8 * j][tx] * rT[(size_t)n * nodes + m] * rT[(size_t)n * nodes + q];
      const float as = sa[ty + 8 * j][tx] * rS[(size_t)n * nodes + m] * rS[(size_t)n * nodes + q];
      const float e = at - as;
      if (E) E[((size_t)n * nodes + m) * nodes + q] = e;
      acc += (double)e * (double)e;
    }
  }
  double t = block_sum_d(acc, sh);
  if (threadIdx.x == 0) part[((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = t;
}

// dpooled_S[n][m][c] = coef * rS[m] * sum_q E[m][q] * rS[q] * PS[q][c],   coef = -4*g/(nodes^2 * N)
__global__ void __launch_bounds__(256)
pa_bwd_kernel(const float* __restrict__ E, const float* __restrict__ PS, const float* __restrict__ rS, int CS, int nodes,
              int N, const float* __restrict__ gout, float* __restrict__ dpooled) {
  __shared__ float se[kPT][kPK + 1], sp[kPK][kPT + 1];
  const int n = blockIdx.z, m0 = blockIdx.y * kPT, c0 = blockIdx.x * kPT;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const float coef = -4.f * __ldg(gout) / ((float)nodes * (float)nodes * (float)N);
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int q0 = 0; q0 < nodes; q0 += kPK) {
    __syncthreads();
    for (int r = ty; r < kPT; r += 8) {
      const int q = q0 + tx;
      se[r][tx] = (m0 + r < nodes && q < nodes) ? E[((size_t)n * nodes + m0 + r) * nodes + q] : 0.f;
      const int qq = q0 + r, c = c0 + tx;
      sp[r][tx] = (qq < nodes && c < CS) ? PS[((size_t)n * nodes + qq) * CS + c] * rS[(size_t)n * nodes + qq] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kPK; ++k) {
      const float b = sp[k][tx];
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[j] += se[ty + 8 * j][k] * b;
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int m = m0 + ty + 8 * j, c = c0 + tx;
    if (m < nodes && c < CS) dpooled[((size_t)n * nodes + m) * CS + c] = coef * rS[(size_t)n * nodes + m] * acc[j];
  }
}

// scatter the pooled gradient to the arg-max positions of the (pre-zeroed) feature gradient
__global__ void pa_scatter_kernel(const float* __restrict__ dpooled, const int* __restrict__ argmax, int C, int nodes, int N,
                                  float* __restrict__ dF, Strides st) {
  const long long total = (long long)N * nodes * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C); const long long r = i / C; const int n = (int)(r / nodes);
    dF[n * st.sn + c * st.sc + (long long)argmax[i] * st.sp] = dpooled[i];
  }
}

int red_blocks(long long total) {
  long long b = (total + 255) / 256;
  if (b > kNumSMs * 4) b = kNumSMs * 4;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace

extern "C" int skd_loss_max_partials(void) { return kNumSMs * 4; }

extern "C" int skd_pixelwise_fwd(int N, int C, int HW, const float* S, long long s_sn, long long s_sc, long long s_sp,
                                 const float* T, long long t_sn, long long t_sc, long long t_sp, float inv_hw,
                                 float* loss, double* workspace, cudaStream_t st) {
  if (C > kMaxClasses) { set_error_msg("skd_pixelwise_fwd", "C > 32 classes unsupported"); return 0; }
  const int blocks = red_blocks((long long)N * HW);
  pixelwise_fwd_kernel<<<blocks, 256, 0, st>>>(S, T, N, C, HW, Strides{s_sn, s_sc, s_sp}, Strides{t_sn, t_sc, t_sp}, workspace);
  finalize_sum_kernel<<<1, 256, 0, st>>>(workspace, blocks, (double)inv_hw, loss, nullptr, 0, nullptr);
  return finish("skd_pixelwise_fwd", 2);
}

extern "C" int skd_pixelwise_bwd(int N, int C, int HW, const float* S, long long s_sn, long long s_sc, long long s_sp,
                                 const float* T, long long t_sn, long long t_sc, long long t_sp, float* dS,
                                 long long d_sn, long long d_sc, long long d_sp, const float* grad_out, float inv_hw,
                                 cudaStream_t st) {
  if (C > kMaxClasses) { set_error_msg("skd_pixelwise_bwd", "C > 32 classes unsupported"); return 0; }
  pixelwise_bwd_kernel<<<red_blocks((long long)N * HW), 256, 0, st>>>(S, T, dS, N, C, HW, Strides{s_sn, s_sc, s_sp},
                                                                     Strides{t_sn, t_sc, t_sp}, Strides{d_sn, d_sc, d_sp},
                                                                     grad_out, inv_hw);
  return finish("skd_pixelwise_bwd");
}

extern "C" int skd_dsn_ce_fwd(int N, int C, int h, int w, int H, int W, const float* L0, long long a_sn, long long a_sc,
                              long long a_sp, const float* L1, long long b_sn, long long b_sc, long long b_sp,
                              const long long* labels, int ignore_index, float w0, float w1, float* loss, float* count,
                              double* workspace, cudaStream_t st) {
  if (C > kMaxClasses) { set_error_msg("skd_dsn_ce_fwd", "C > 32 classes unsupported"); return 0; }
  const int blocks = red_blocks((long long)N * H * W);
  dsn_ce_fwd_kernel<<<blocks, 256, 0, st>>>(L0, L1, Strides{a_sn, a_sc, a_sp}, Strides{b_sn, b_sc, b_sp}, labels, N, C, h, w,
                                           H, W, ignore_index, w0, w1, workspace, workspace + blocks);
  finalize_sum_kernel<<<1, 256, 0, st>>>(workspace, blocks, 1.0, loss, workspace + blocks, 1, count);
  return finish("skd_dsn_ce_fwd", 2);
}

extern "C" long long skd_dsn_ce_bwd_workspace_floats(int N, int C, int w, int H, int heads) {
  return (long long)heads * N * H * C * w;
}

static int dsn_rows_launch(bool with_loss, int N, int C, int h, int w, int H, int W, const float* L0, Strides a, const float* L1, Strides b,
                           const long long* labels, int ignore_index, float w0, float w1, float* T1, double* part_loss, double* part_cnt,
                           cudaStream_t st, const char* who) {
  const int heads = L1 ? 2 : 1;
  int chunk = W < 1024 ? W : 1024;
  const size_t smem = ((size_t)C * (chunk | 1) + 2 * (size_t)chunk + (size_t)w + 2 + (size_t)w * C) * sizeof(float);
  if (smem > 200 * 1024) { set_error_msg(who, "source width too large for one block's shared memory"); return 0; }
  static bool attr_done = false;
  if (!attr_done) {
    cudaFuncSetAttribute(dsn_ce_bwd_rows_kernel<false, 19>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(dsn_ce_bwd_rows_kernel<true, 19>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(dsn_ce_bwd_rows_kernel<false, kMaxClasses>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(dsn_ce_bwd_rows_kernel<true, kMaxClasses>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    attr_done = true;
  }
  const dim3 grid(H, N, heads);
#define SKD_DSN_ROWS(LOSSF, CTV, PL, PC) \
  dsn_ce_bwd_rows_kernel<LOSSF, CTV><<<grid, kRowsThreads, smem, st>>>(L0, L1, a, b, labels, N, C, h, w, H, W, ignore_index, T1, chunk, PL, PC, w0, w1)
  if (with_loss) { if (C <= 19) SKD_DSN_ROWS(true, 19, part_loss, part_cnt); else SKD_DSN_ROWS(true, kMaxClasses, part_loss, part_cnt); }
  else { if (C <= 19) SKD_DSN_ROWS(false, 19, nullptr, nullptr); else SKD_DSN_ROWS(false, kMaxClasses, nullptr, nullptr); }
#undef SKD_DSN_ROWS
  return 1;
}

extern "C" int skd_dsn_ce_bwd(int N, int C, int h, int w, int H, int W, const float* L0, long long a_sn, long long a_sc,
                              long long a_sp, const float* L1, long long b_sn, long long b_sc, long long b_sp,
                              const long long* labels, int ignore_index, float w0, float w1, const float* grad_out,
                              const float* count, float* d0, float* d1, float* workspace, cudaStream_t st) {
  if (C > kMaxClasses) { set_error_msg("skd_dsn_ce_bwd", "C > 32 classes unsupported"); return 0; }
  const int heads = L1 ? 2 : 1;
  if (!dsn_rows_launch(false, N, C, h, w, H, W, L0, Strides{a_sn, a_sc, a_sp}, L1, Strides{b_sn, b_sc, b_sp}, labels, ignore_index, w0, w1, workspace,
                       nullptr, nullptr, st, "skd_dsn_ce_bwd")) return 0;
  const long long tot = (long long)heads * N * h * C * w;
  dsn_ce_bwd_cols_kernel<<<red_blocks(tot), 256, 0, st>>>(workspace, d0, L1 ? d1 : nullptr, Strides{a_sn, a_sc, a_sp},
                                                         Strides{b_sn, b_sc, b_sp}, N, C, h, w, H, grad_out, count, w0, w1);
  return finish("skd_dsn_ce_bwd", 2);
}

// Training forward: loss and valid-pixel count AND the backward's row-phase result (rows_ws: skd_dsn_ce_bwd_workspace_floats) in one
// pass over the upsampled pixels; partials: 2 * heads * N * H doubles.
extern "C" long long skd_dsn_ce_train_partials(int N, int H, int heads) { return 2LL * heads * N * H; }

extern "C" int skd_dsn_ce_fwd_train(int N, int C, int h, int w, int H, int W, const float* L0, long long a_sn, long long a_sc,
                                    long long a_sp, const float* L1, long long b_sn, long long b_sc, long long b_sp,
                                    const long long* labels, int ignore_index, float w0, float w1, float* loss, float* count,
                                    double* partials, float* rows_ws, cudaStream_t st) {
  if (C > kMaxClasses) { set_error_msg("skd_dsn_ce_fwd_train", "C > 32 classes unsupported"); return 0; }
  const int heads = L1 ? 2 : 1;
  const int np = heads * N * H;
  if (!dsn_rows_launch(true, N, C, h, w, H, W, L0, Strides{a_sn, a_sc, a_sp}, L1, Strides{b_sn, b_sc, b_sp}, labels, ignore_index, w0, w1, rows_ws,
                       partials, partials + np, st, "skd_dsn_ce_fwd_train")) return 0;
  finalize_sum_kernel<<<1, 256, 0, st>>>(partials, np, 1.0, loss, partials + np, 1, count);
  return finish("skd_dsn_ce_fwd_train", 2);
}

// Backward after skd_dsn_ce_fwd_train: only the column phase (d logits = g / count * U_y^T rows_ws)
extern "C" int skd_dsn_ce_bwd_cols(int N, int C, int h, int w, int H, const float* rows_ws, long long a_sn, long long a_sc, long long a_sp,
                                   long long b_sn, long long b_sc, long long b_sp, int heads, float w0, float w1, const float* grad_out,
                                   const float* count, float* d0, float* d1, cudaStream_t st) {
  const long long tot = (long long)heads * N * h * C * w;
  dsn_ce_bwd_cols_kernel<<<red_blocks(tot), 256, 0, st>>>(rows_ws, d0, heads == 2 ? d1 : nullptr, Strides{a_sn, a_sc, a_sp},
                                                         Strides{b_sn, b_sc, b_sp}, N, C, h, w, H, grad_out, count, w0, w1);
  return finish("skd_dsn_ce_bwd_cols");
}

extern "C" int skd_pairwise_pool(int N, int C, int H, int W, const float* F, long long sn, long long sc, long long sp,
                                 int ph, int pw, float* pooled, int* argmax, float* rnorm, cudaStream_t st) {
  if (ph <= 0 || pw <= 0) { set_error_msg("skd_pairwise_pool", "pool window is empty (scale too small)"); return 0; }
  const int nh = (H + ph - 1) / ph, nw = (W + pw - 1) / pw;
  if (sc == 1 && C % 4 == 0 && sp % 4 == 0 && sn % 4 == 0 && sp < (1LL << 31) &&
      !((reinterpret_cast<uintptr_t>(F) | reinterpret_cast<uintptr_t>(pooled) | reinterpret_cast<uintptr_t>(argmax)) & 15))
    pa_pool_nhwc_kernel<<<dim3(nh * nw, N, (C + 63) / 64), 256, 0, st>>>(F, sn, (int)sp, C, H, W, ph, pw, nh, nw, pooled, argmax);
  else
    pa_pool_kernel<<<dim3(nh * nw, N, (C + 63) / 64), 256, 0, st>>>(F, Strides{sn, sc, sp}, C, H, W, ph, pw, nh, nw, pooled, argmax);
  pa_rnorm_kernel<<<N * nh * nw, 32, 0, st>>>(pooled, C, rnorm);
  return finish("skd_pairwise_pool", 2);
}

extern "C" long long skd_pairwise_gram_partials(int N, int nodes) {
  const long long t = (nodes + kPT - 1) / kPT;
  return (long long)N * t * t;
}

extern "C" int skd_pairwise_gram(int N, int nodes, int CS, int CT, const float* pooled_S, const float* pooled_T,
                                 const float* rnorm_S, const float* rnorm_T, float* E, float* loss, double* workspace,
                                 cudaStream_t st) {
  const int t = (nodes + kPT - 1) / kPT;
  pa_gram_kernel<<<dim3(t, t, N), 256, 0, st>>>(pooled_S, pooled_T, rnorm_S, rnorm_T, CS, CT, nodes, E, workspace);
  const double scale = 1.0 / ((double)nodes * (double)nodes) / (double)N;          // utils.py:181
  finalize_sum_kernel<<<1, 256, 0, st>>>(workspace, N * t * t, scale, loss, nullptr, 0, nullptr);
  return finish("skd_pairwise_gram", 2);
}

extern "C" int skd_pairwise_scatter(int N, int nodes, int CS, const float* dpooled, const int* argmax, float* dF, long long sn,
                                    long long sc, long long sp, cudaStream_t st) {
  pa_scatter_kernel<<<red_blocks((long long)N * nodes * CS), 256, 0, st>>>(dpooled, argmax, CS, nodes, N, dF, Strides{sn, sc, sp});
  return finish("skd_pairwise_scatter");
}

extern "C" int skd_pairwise_bwd(int N, int nodes, int CS, const float* E, const float* pooled_S, const float* rnorm_S,
                                const int* argmax, const float* grad_out, float* dpooled, float* dF, long long sn,
                                long long sc, long long sp, cudaStream_t st) {
  const int t = (nodes + kPT - 1) / kPT;
  pa_bwd_kernel<<<dim3((CS + kPT - 1) / kPT, t, N), 256, 0, st>>>(E, pooled_S, rnorm_S, CS, nodes, N, grad_out, dpooled);
  pa_scatter_kernel<<<red_blocks((long long)N * nodes * CS), 256, 0, st>>>(dpooled, argmax, CS, nodes, N, dF, Strides{sn, sc, sp});
  return finish("skd_pairwise_bwd", 2);
}
