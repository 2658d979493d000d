// SAGAN discriminator of the holistic (Ho) loss on sm_90a -- everything around its tensor-core convolutions:
//
//   networks/spectral.py:23-35          skd_sn_power_iter / skd_sn_weight_grad   (cluster + DSMEM power iteration)
//   networks/sagan_models.py:147,157    skd_bn2d_*                               (BatchNorm2d(19), batch statistics)
//   networks/sagan_models.py:31-40      skd_attn_fwd / _tangent_fwd / _bwd       (softmax(Q K^T) V, gamma * o + x)
//   networks/sagan_models.py:140,166    skd_disc_last_*                          (the 4x4 "last" conv, Cout = 1)
//   utils/criterion.py:98-120           skd_gp_norms / skd_gp_direction          (WGAN-GP)
//   utils/criterion.py:129-166          skd_adv_loss                             (wgan / hinge adversarial losses)
//
// The 4x4 stride-2 spectral-norm convolutions and the 1x1 q/k/v projections run on the wgmma implicit-GEMM kernel
// (conv_sm100.cu, split-precision 3xTF32); the data gradient of a 4x4/s2/p1 convolution is ONE 3x3 stride-1 convolution of
// dy producing the four input-pixel parity classes as 4*Cin channels (weights from skd_disc_dgrad_weight_prep), un-shuffled
// (and multiplied by the LeakyReLU mask of the layer below) by skd_disc_dgrad_unshuffle.
//
// WGAN-GP needs d/dtheta of |d(sum D(x))/dx|: the reference gets it from autograd's double backward.  Here it is "reverse
// over forward" (oracle/gp_dual.py states and pins the math): a tangent (JVP) pass along v = c_n * g_n followed by ONE
// reverse pass over the joint (primal, tangent) graph.  Convolutions are bilinear, so the joint pass is the ordinary
// backward over a batch of 2B rows ([primal | tangent]); LeakyReLU contributes its mask to both halves; only the softmax
// attention and the batch-statistics BatchNorm have genuinely second-order terms, implemented below.
#include <cooperative_groups.h>

#include "common.cuh"
#include "skd.h"
#include "sm90_ptx.cuh"

namespace cg = cooperative_groups;
using namespace skd;

namespace {

int blocks_for(long long n, int per_block = 256) {
  long long b = (n + per_block - 1) / per_block;
  if (b > kNumSMs * 8) b = kNumSMs * 8;
  if (b < 1) b = 1;
  return (int)b;
}

__device__ __forceinline__ float lo_part(float v) { return ptx::round_tf32(v - ptx::round_tf32(v)); }

__device__ __forceinline__ float block_sum(float a, float* sh64) { return block_sum2(a, 0.f, sh64).x; }

// C[M][N] = sum_k a(i,k) * b(k,j) by the whole CTA (256 threads as 16 x 16): thread (ty, tx) owns rows ty + 16*ii and columns
// tx + 16*jj (interleaved: the lanes of a warp read consecutive columns).  Operands are shared-memory accessors.
template <int TM, int TN, class FA, class FB, class FS>
__device__ __forceinline__ void block_gemm(int M, int N, int K, FA a, FB b, FS store) {
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  for (int m0 = 0; m0 < M; m0 += 16 * TM) {
    for (int n0 = 0; n0 < N; n0 += 16 * TN) {
      if (m0 + ty >= M || n0 + tx >= N) continue;
      int ri[TM], cj[TN];
#pragma unroll
      for (int ii = 0; ii < TM; ++ii) ri[ii] = min(m0 + ty + 16 * ii, M - 1);
#pragma unroll
      for (int jj = 0; jj < TN; ++jj) cj[jj] = min(n0 + tx + 16 * jj, N - 1);
      float acc[TM][TN];
#pragma unroll
      for (int ii = 0; ii < TM; ++ii)
#pragma unroll
        for (int jj = 0; jj < TN; ++jj) acc[ii][jj] = 0.f;
      for (int k = 0; k < K; ++k) {
        float av[TM], bv[TN];
#pragma unroll
        for (int ii = 0; ii < TM; ++ii) av[ii] = a(ri[ii], k);
#pragma unroll
        for (int jj = 0; jj < TN; ++jj) bv[jj] = b(k, cj[jj]);
#pragma unroll
        for (int ii = 0; ii < TM; ++ii)
#pragma unroll
          for (int jj = 0; jj < TN; ++jj) acc[ii][jj] = fmaf(av[ii], bv[jj], acc[ii][jj]);
      }
#pragma unroll
      for (int ii = 0; ii < TM; ++ii)
#pragma unroll
        for (int jj = 0; jj < TN; ++jj) {
          const int i = m0 + ty + 16 * ii, j = n0 + tx + 16 * jj;
          if (i < M && j < N) store(i, j, acc[ii][jj]);
        }
    }
  }
}

// The same product on the tensor cores: mma.sync m16n8k8 TF32 in split precision (a_lo*b_hi + a_hi*b_lo + a_hi*b_hi, fp32-grade like
// the 3xTF32 convolutions), operands through the same shared-memory accessors.  Warp tiles of 16 x 8*NT, eight warps round-robin.
// The attention products are 32..1024 positions wide (n x n x d scores, n x C x n values): far below one wgmma tile pipeline's
// start-up cost, so the warp-level MMA is the tensor-core path that fits them.
__device__ __forceinline__ void mma_m16n8k8_tf32(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

template <int NT, class FA, class FB, class FS>
__device__ __forceinline__ void block_gemm_tc(int M, int N, int K, FA a, FB b, FS store) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int mt = (M + 15) / 16, nt = (N + 8 * NT - 1) / (8 * NT);
  for (int tile = warp; tile < mt * nt; tile += nw) {
    const int m0 = (tile / nt) * 16, n0 = (tile % nt) * 8 * NT;
    const int r0 = min(m0 + g, M - 1), r1 = min(m0 + g + 8, M - 1);
    int cn[NT];
#pragma unroll
    for (int j = 0; j < NT; ++j) cn[j] = min(n0 + 8 * j + g, N - 1);
    float acc[NT][4];
#pragma unroll
    for (int j = 0; j < NT; ++j) { acc[j][0] = 0.f; acc[j][1] = 0.f; acc[j][2] = 0.f; acc[j][3] = 0.f; }
    for (int k0 = 0; k0 < K; k0 += 8) {
      const bool va = k0 + t < K, vb = k0 + t + 4 < K;
      const int ka = min(k0 + t, K - 1), kb = min(k0 + t + 4, K - 1);
      float af[4];
      af[0] = va ? a(r0, ka) : 0.f; af[1] = va ? a(r1, ka) : 0.f; af[2] = vb ? a(r0, kb) : 0.f; af[3] = vb ? a(r1, kb) : 0.f;
      uint32_t ah[4], al[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) { const float h = ptx::round_tf32(af[q]); ah[q] = __float_as_uint(h); al[q] = __float_as_uint(ptx::round_tf32(af[q] - h)); }
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        const float b0 = va ? b(ka, cn[j]) : 0.f, b1 = vb ? b(kb, cn[j]) : 0.f;
        const float h0 = ptx::round_tf32(b0), h1 = ptx::round_tf32(b1);
        const uint32_t bh[2] = {__float_as_uint(h0), __float_as_uint(h1)};
        const uint32_t bl[2] = {__float_as_uint(ptx::round_tf32(b0 - h0)), __float_as_uint(ptx::round_tf32(b1 - h1))};
        mma_m16n8k8_tf32(acc[j], al, bh);
        mma_m16n8k8_tf32(acc[j], ah, bl);
        mma_m16n8k8_tf32(acc[j], ah, bh);
      }
    }
#pragma unroll
    for (int j = 0; j < NT; ++j) {
      const int col = n0 + 8 * j + 2 * t;
      if (m0 + g < M) { if (col < N) store(m0 + g, col, acc[j][0]); if (col + 1 < N) store(m0 + g, col + 1, acc[j][1]); }
      if (m0 + g + 8 < M) { if (col < N) store(m0 + g + 8, col, acc[j][2]); if (col + 1 < N) store(m0 + g + 8, col + 1, acc[j][3]); }
    }
  }
}

// tc != 0: tensor cores (mma.sync, split precision); 0: the SIMT fp32 product (kept as the cross-check; skd_set_attn_tensor_cores)
template <int TM, int TN, class FA, class FB, class FS>
__device__ __forceinline__ void attn_gemm(int tc, int M, int N, int K, FA a, FB b, FS store) {
  if (tc) block_gemm_tc<4>(M, N, K, a, b, store);
  else block_gemm<TM, TN>(M, N, K, a, b, store);
}

int g_attn_tc = 1;

// ====================================================================================================================
// Spectral normalisation (networks/spectral.py:23-35)
// ====================================================================================================================
constexpr int kSnThreads = 512, kSnCluster = 8, kSnMaxK = 8192, kSnMaxRows = 256;

// One power iteration by ONE cluster of 8 CTAs: each CTA owns Cout/8 rows of W; W^T u is combined through distributed shared
// memory, then v = normalize(W^T u), s = W v (own rows), u = normalize(s), sigma = u . s.  W is [Cout][taps][Cin] (OHWI);
// v is kept in the reference's flattening order (ci * taps + tap: `w.view(height, -1)` of a (Cout,Cin,KH,KW) tensor).
__global__ void __launch_bounds__(kSnThreads)
sn_power_iter_kernel(int Cout, int taps, int Cin, const float* __restrict__ w, float* u, float* v, float* u_save, float* v_save,
                     float* sigma, float* inv_vec, int vec_len) {
  cg::cluster_group cluster = cg::this_cluster();
  __shared__ float s_t[kSnMaxK];
  __shared__ float s_s[kSnMaxRows];
  __shared__ float s_red[64];
  __shared__ float s_part;
  const int K = taps * Cin;
  const int rank = (int)cluster.block_rank();
  const int R = (Cout + kSnCluster - 1) / kSnCluster;
  const int row0 = min(rank * R, Cout), row1 = min(Cout, row0 + R);
  for (int k = threadIdx.x; k < K; k += kSnThreads) {
    float acc = 0.f;
    for (int r = row0; r < row1; ++r) acc = fmaf(__ldg(w + (size_t)r * K + k), u[r], acc);
    s_t[k] = acc;
  }
  cluster.sync();
  float loc[kSnMaxK / kSnThreads];
  float n2 = 0.f;
  int cnt = 0;
  for (int k = threadIdx.x; k < K; k += kSnThreads) {
    float tot = 0.f;
    for (int rk = 0; rk < kSnCluster; ++rk) tot += cluster.map_shared_rank(s_t, rk)[k];
    loc[cnt++] = tot;
    n2 = fmaf(tot, tot, n2);
  }
  n2 = block_sum(n2, s_red);
  cluster.sync();                                   // every CTA has read every partial before s_t is overwritten
  const float inv_t = 1.f / (sqrtf(n2) + 1e-12f);   // l2normalize: v / (|v| + eps), spectral.py:10-11
  cnt = 0;
  for (int k = threadIdx.x; k < K; k += kSnThreads) {
    const float vv = loc[cnt++] * inv_t;
    s_t[k] = vv;
    if (rank == 0) {
      const int kr = (k % Cin) * taps + k / Cin;
      v[kr] = vv;
      if (v_save) v_save[kr] = vv;
    }
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = row0 + warp; r < row1; r += kSnThreads / 32) {
    float acc = 0.f;
    for (int k = lane; k < K; k += 32) acc = fmaf(__ldg(w + (size_t)r * K + k), s_t[k], acc);
    acc = warp_sum(acc);
    if (lane == 0) s_s[r - row0] = acc;
  }
  __syncthreads();
  float q = 0.f;
  for (int i = threadIdx.x; i < row1 - row0; i += kSnThreads) q = fmaf(s_s[i], s_s[i], q);
  q = block_sum(q, s_red);
  if (threadIdx.x == 0) s_part = q;
  cluster.sync();
  float tot = 0.f;
  for (int rk = 0; rk < kSnCluster; ++rk) tot += *cluster.map_shared_rank(&s_part, rk);
  cluster.sync();                                   // keep every CTA's shared memory alive until all peers have read it
  const float inv_s = 1.f / (sqrtf(tot) + 1e-12f);
  for (int i = threadIdx.x; i < row1 - row0; i += kSnThreads) {
    const float uu = s_s[i] * inv_s;
    u[row0 + i] = uu;
    if (u_save) u_save[row0 + i] = uu;
  }
  const float sg = tot * inv_s;                     // u . (W v) = |Wv|^2 / (|Wv| + eps)
  if (rank == 0) {
    if (threadIdx.x == 0) sigma[0] = sg;
    for (int i = threadIdx.x; i < vec_len; i += kSnThreads) inv_vec[i] = 1.f / sg;
  }
}

// ---- the same iteration for SEVERAL layers at once, spread over the whole GPU (the discriminator's four layers per forward) ----
// The cluster kernel above keeps one layer on 8 SMs: the 512 x 4096 matrix of l4 is two passes over 8 MB through 8 SMs.
// Here every phase is a grid over all layers: (1) partial W^T u per 32-row block, (2) v = normalize(sum of partials) [fixed order],
// (3) s = W v, one warp per row, (4) u = normalize(s), sigma = u . s.  Deterministic (no atomics): replicas of a data-parallel
// job keep bit-identical u, v.
constexpr int kSnBatchMax = 8, kSnRowBlock = 32, kSnKBlock = 1024;
struct SnLayer {
  int Cout, taps, Cin, K, vec_len, n_rb, n_kb, blk1, blk3;     // blk1 / blk3: first block of this layer in phase 1 / 3
  const float* w; float *u, *v, *u_save, *v_save, *sigma, *inv_vec;
  float *tpart, *vlin, *s;                                      // workspace: [n_rb][K], [K], [Cout]
};
struct SnBatch { int n; SnLayer L[kSnBatchMax]; };

__device__ __forceinline__ int sn_find_layer(const SnBatch& b, int blk, bool phase3) {
  int l = 0;
  for (int i = 1; i < b.n; ++i) if (blk >= (phase3 ? b.L[i].blk3 : b.L[i].blk1)) l = i;
  return l;
}

__global__ void __launch_bounds__(256)
sn_phase1_kernel(const __grid_constant__ SnBatch b) {
  __shared__ float su[kSnRowBlock];
  const int li = sn_find_layer(b, blockIdx.x, false);
  const SnLayer& L = b.L[li];
  const int rel = blockIdx.x - L.blk1, rb = rel / L.n_kb, kb = rel - rb * L.n_kb;
  const int r0 = rb * kSnRowBlock, r1 = min(L.Cout, r0 + kSnRowBlock);
  if (threadIdx.x < r1 - r0) su[threadIdx.x] = L.u[r0 + threadIdx.x];
  __syncthreads();
  const int k0 = kb * kSnKBlock + threadIdx.x;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  const float* wp = L.w + (size_t)r0 * L.K;
  for (int r = 0; r < r1 - r0; ++r, wp += L.K) {
    const float ur = su[r];
#pragma unroll
    for (int j = 0; j < 4; ++j) { const int k = k0 + j * 256; if (k < L.K) acc[j] = fmaf(__ldg(wp + k), ur, acc[j]); }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) { const int k = k0 + j * 256; if (k < L.K) L.tpart[(size_t)rb * L.K + k] = acc[j]; }
}

__global__ void __launch_bounds__(1024)
sn_phase2_kernel(const __grid_constant__ SnBatch b) {
  __shared__ float s_t[kSnMaxK];
  __shared__ float s_red[64];
  const SnLayer& L = b.L[blockIdx.x];
  float n2 = 0.f;
  for (int k = threadIdx.x; k < L.K; k += 1024) {
    float tot = 0.f;
    for (int rb = 0; rb < L.n_rb; ++rb) tot += L.tpart[(size_t)rb * L.K + k];
    s_t[k] = tot; n2 = fmaf(tot, tot, n2);
  }
  n2 = block_sum(n2, s_red);
  const float inv_t = 1.f / (sqrtf(n2) + 1e-12f);   // l2normalize: v / (|v| + eps), spectral.py:10-11
  for (int k = threadIdx.x; k < L.K; k += 1024) {
    const float vv = s_t[k] * inv_t;
    L.vlin[k] = vv;
    const int kr = (k % L.Cin) * L.taps + k / L.Cin;            // the reference's flattening of (Cout, Cin, KH, KW).view(Cout, -1)
    L.v[kr] = vv;
    if (L.v_save) L.v_save[kr] = vv;
  }
}

__global__ void __launch_bounds__(256)
sn_phase3_kernel(const __grid_constant__ SnBatch b) {
  const int li = sn_find_layer(b, blockIdx.x, true);
  const SnLayer& L = b.L[li];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = (blockIdx.x - L.blk3) * 8 + warp;
  if (r >= L.Cout) return;
  const float* wp = L.w + (size_t)r * L.K;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  int k = lane;
  for (; k + 96 < L.K; k += 128) {
    a0 = fmaf(__ldg(wp + k), L.vlin[k], a0); a1 = fmaf(__ldg(wp + k + 32), L.vlin[k + 32], a1);
    a2 = fmaf(__ldg(wp + k + 64), L.vlin[k + 64], a2); a3 = fmaf(__ldg(wp + k + 96), L.vlin[k + 96], a3);
  }
  for (; k < L.K; k += 32) a0 = fmaf(__ldg(wp + k), L.vlin[k], a0);
  const float acc = warp_sum((a0 + a1) + (a2 + a3));
  if (lane == 0) L.s[r] = acc;
}

__global__ void __launch_bounds__(256)
sn_phase4_kernel(const __grid_constant__ SnBatch b) {
  __shared__ float s_red[64];
  const SnLayer& L = b.L[blockIdx.x];
  float q = 0.f;
  for (int i = threadIdx.x; i < L.Cout; i += 256) { const float sv = L.s[i]; q = fmaf(sv, sv, q); }
  const float tot = block_sum(q, s_red);
  const float inv_s = 1.f / (sqrtf(tot) + 1e-12f);
  for (int i = threadIdx.x; i < L.Cout; i += 256) {
    const float uu = L.s[i] * inv_s;
    L.u[i] = uu;
    if (L.u_save) L.u_save[i] = uu;
  }
  const float sg = tot * inv_s;                     // u . (W v) = |Wv|^2 / (|Wv| + eps)
  if (threadIdx.x == 0) L.sigma[0] = sg;
  for (int i = threadIdx.x; i < L.vec_len; i += 256) L.inv_vec[i] = 1.f / sg;
}

constexpr int kDotBlocks = 296;
// <dWn, W> over the valid (un-padded) entries; deterministic: fixed per-block partials, the last block adds them in order
__global__ void __launch_bounds__(256)
sn_grad_dot_kernel(int Cout, int taps, int Cin, int Cin_p, const float* __restrict__ dwn, const float* __restrict__ w, double* ws) {
  __shared__ double sh[256];
  __shared__ bool last;
  const long long total = (long long)Cout * taps * Cin;
  double acc = 0.0;
  const long long step = (long long)gridDim.x * 256;
  for (long long i0 = (long long)blockIdx.x * 256 + threadIdx.x; i0 < total; i0 += 4 * step) {
    float a[4], b[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long i = i0 + j * step;
      const bool ok = i < total;
      const int ci = ok ? (int)(i % Cin) : 0; const long long rt = ok ? i / Cin : 0;
      a[j] = ok ? __ldg(dwn + rt * Cin_p + ci) : 0.f; b[j] = ok ? __ldg(w + i) : 0.f;
    }
    acc += ((double)a[0] * (double)b[0] + (double)a[1] * (double)b[1]) + ((double)a[2] * (double)b[2] + (double)a[3] * (double)b[3]);
  }
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o]; __syncthreads(); }
  unsigned* counter = reinterpret_cast<unsigned*>(ws + 1 + kDotBlocks);
  if (threadIdx.x == 0) {
    ws[1 + blockIdx.x] = sh[0];
    __threadfence();
    last = (atomicAdd(counter, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (last && threadIdx.x == 0) {
    __threadfence();
    double t = 0.0;
    for (unsigned b = 0; b < gridDim.x; ++b) t += reinterpret_cast<volatile double*>(ws)[1 + b];
    ws[0] = t;
    *counter = 0u;                                  // self-resetting: the workspace only has to be zero the first time
  }
}

// dW = dWn / sigma - <dWn, W> / sigma^2 * u v^T   (sigma = u^T W v with u, v constant: spectral.py:34-35)
__global__ void __launch_bounds__(256)
sn_grad_apply_kernel(int Cout, int taps, int Cin, int Cin_p, const float* __restrict__ dwn, const float* __restrict__ u,
                     const float* __restrict__ v, const float* __restrict__ sigma, const double* __restrict__ ws, float* dw, int accumulate) {
  const long long total = (long long)Cout * taps * Cin;
  const float sg = sigma[0];
  const float coef = (float)(ws[0] / ((double)sg * (double)sg));
  const float inv = 1.f / sg;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int ci = (int)(i % Cin); const long long rt = i / Cin;
    const int tap = (int)(rt % taps), co = (int)(rt / taps);
    const float g = __ldg(dwn + rt * Cin_p + ci) * inv - coef * __ldg(u + co) * __ldg(v + ci * taps + tap);
    dw[i] = accumulate ? dw[i] + g : g;
  }
}

// w [Cout][taps][Cin] -> channel-padded copy (TMA rounds it to TF32 on load: the "hi" part) and its TF32 "lo" part
__global__ void __launch_bounds__(256)
weight_prep_kernel(long long rows, int Cin, int Cin_p, const float* __restrict__ w, float* __restrict__ wp, float* __restrict__ wlo) {
  const long long total = rows * Cin_p;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int ci = (int)(i % Cin_p); const long long r = i / Cin_p;
    const float val = ci < Cin ? __ldg(w + r * Cin + ci) : 0.f;
    wp[i] = val;
    if (wlo) wlo[i] = lo_part(val);
  }
}

// data-gradient weights of a 4x4 / stride 2 / pad 1 convolution as ONE 3x3 stride-1 convolution of dy:
//   wd[(py*2+px)*Cin_p + ci][ty+1][tx+1][co] = w[co][py + 1 - 2 ty][px + 1 - 2 tx][ci]   (zero where the tap does not exist)
// input pixel (2j+py, 2i+px) receives dy rows j+ty, ty in {-1,0,1}: ky = 2j + py + 1 - 2 (j + ty).
__global__ void __launch_bounds__(256)
dgrad_weight_prep_kernel(int Cout, int Cin, int Cin_p, const float* __restrict__ w, float* __restrict__ wd, float* __restrict__ wlo) {
  const long long total = 4LL * Cin_p * 9 * Cout;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int co = (int)(i % Cout); long long r = i / Cout;
    const int tx = (int)(r % 3) - 1; r /= 3;
    const int ty = (int)(r % 3) - 1; r /= 3;
    const int ci = (int)(r % Cin_p); const int cls = (int)(r / Cin_p);
    const int py = cls >> 1, px = cls & 1;
    const int ky = py + 1 - 2 * ty, kx = px + 1 - 2 * tx;
    float val = 0.f;
    if (ci < Cin && ky >= 0 && ky < 4 && kx >= 0 && kx < 4) val = __ldg(w + (((size_t)co * 4 + ky) * 4 + kx) * Cin + ci);
    wd[i] = val;
    if (wlo) wlo[i] = lo_part(val);
  }
}

// ====================================================================================================================
// BatchNorm2d with batch statistics on <= 32 channels (nn.BatchNorm2d(19), sagan_models.py:147)
// ====================================================================================================================
constexpr int kBnBlocks = 296;

// per-channel sums over pixels of up to three products; lane = channel, warp = pixel.
//   MODE 0: S1 = sum x,      S2 = sum x^2                                  (x strided)                 -> statistics
//   MODE 1: S1 = sum a,      S2 = sum a * xhat,   S3 = sum a * b (b may be NULL)   (a, b dense [P][ld])
// The last block folds the fixed-order partials: MODE 0 -> mean, rstd, running statistics; MODE 1 -> sums[3][32].
template <int MODE>
__global__ void __launch_bounds__(256)
bn2d_reduce_kernel(int N, int C, int HW, const float* __restrict__ x, long long sn, long long sc, long long sp,
                   const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ a, const float* __restrict__ b2,
                   int ld, float eps, float momentum, float* running_mean, float* running_var, long long* nbt, float* out_mean,
                   float* out_rstd, float* sums, double* ws) {
  __shared__ double sh[8][3][32];
  __shared__ bool last;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long P = (long long)N * HW;
  double s1 = 0.0, s2 = 0.0, s3 = 0.0;
  if (lane < C) {
    const float m = MODE ? mean[lane] : 0.f, r = MODE ? rstd[lane] : 0.f;
    // four pixels per iteration: 4-12 independent loads in flight per lane (one pixel per iteration is latency-bound)
    const long long step = (long long)gridDim.x * 8;
    for (long long p0 = (long long)blockIdx.x * 8 + warp; p0 < P; p0 += 4 * step) {
      float xv[4], av[4], bv[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const long long p = p0 + j * step;
        const bool ok = p < P;
        const long long n = ok ? p / HW : 0, q = ok ? p - n * HW : 0;
        xv[j] = ok ? __ldg(x + n * sn + lane * sc + q * sp) : 0.f;
        av[j] = (MODE && ok) ? __ldg(a + p * ld + lane) : 0.f;
        bv[j] = (MODE && ok && b2) ? __ldg(b2 + p * ld + lane) : 0.f;
        if (MODE && !ok) xv[j] = m;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (MODE == 0) { s1 += xv[j]; s2 += (double)xv[j] * xv[j]; }
        else { s1 += av[j]; s2 += (double)(av[j] * ((xv[j] - m) * r)); s3 += (double)(av[j] * bv[j]); }
      }
    }
  }
  sh[warp][0][lane] = s1; sh[warp][1][lane] = s2; sh[warp][2][lane] = s3;
  __syncthreads();
  unsigned* counter = reinterpret_cast<unsigned*>(ws + (size_t)kBnBlocks * 96);
  if (threadIdx.x < 96) {
    const int k = threadIdx.x / 32, c = threadIdx.x % 32;
    double t = 0.0;
    for (int w8 = 0; w8 < 8; ++w8) t += sh[w8][k][c];
    ws[(size_t)blockIdx.x * 96 + threadIdx.x] = t;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = (atomicAdd(counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!last) return;
  __threadfence();
  if (threadIdx.x < 96) {
    const int k = threadIdx.x / 32, c = threadIdx.x % 32;
    double t = 0.0;
    for (unsigned bb = 0; bb < gridDim.x; ++bb) t += reinterpret_cast<volatile double*>(ws)[(size_t)bb * 96 + threadIdx.x];
    sh[0][k][c] = t;
  }
  __syncthreads();
  if (threadIdx.x < C) {
    const int c = threadIdx.x;
    if (MODE == 0) {
      const double mu = sh[0][0][c] / (double)P;
      double var = sh[0][1][c] / (double)P - mu * mu;
      if (var < 0.0) var = 0.0;
      out_mean[c] = (float)mu;
      out_rstd[c] = (float)(1.0 / sqrt(var + (double)eps));
      if (running_mean) {                            // nn.BatchNorm2d training-mode update: unbiased variance, momentum 0.1
        running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)mu;
        const double unb = P > 1 ? var * (double)P / (double)(P - 1) : var;
        running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unb;
      }
    } else {
      sums[c] = (float)sh[0][0][c]; sums[32 + c] = (float)sh[0][1][c]; sums[64 + c] = (float)sh[0][2][c];
    }
  }
  if (threadIdx.x == 0) { *counter = 0u; if (MODE == 0 && nbt) *nbt += 1; }
}

// out[p][c] = gamma (x - mean) rstd + beta  (c < C; channels C..Cp-1 are zero: 16-byte pixel rows for TMA)
__global__ void __launch_bounds__(256)
bn2d_apply_kernel(int N, int C, int HW, const float* __restrict__ x, long long sn, long long sc, long long sp,
                  const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ weight,
                  const float* __restrict__ bias, float* __restrict__ out, float* __restrict__ out_lo, int Cp) {
  const long long total = (long long)N * HW * Cp;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % Cp); const long long p = i / Cp;
    float val = 0.f;
    if (c < C) {
      const long long n = p / HW, q = p - n * HW;
      val = (__ldg(x + n * sn + c * sc + q * sp) - mean[c]) * rstd[c] * (weight ? weight[c] : 1.f) + (bias ? bias[c] : 0.f);
    }
    out[i] = val;
    if (out_lo) out_lo[i] = lo_part(val);
  }
}

// F(a) = gamma rstd (a - mean(a) - xhat mean(a xhat)): the input gradient of batch-statistics BN and -- its Jacobian being
// symmetric -- also its forward-mode tangent.  sums = {sum a, sum a xhat} from bn2d_reduce_kernel<1>.  Output strided.
__global__ void __launch_bounds__(256)
bn2d_jacobian_kernel(int N, int C, int HW, const float* __restrict__ x, long long sn, long long sc, long long sp,
                     const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ weight,
                     const float* __restrict__ a, int ld, const float* __restrict__ sums, float* __restrict__ out, long long on,
                     long long oc, long long op, int Cq, float* __restrict__ out_lo) {
  const long long P = (long long)N * HW;
  const long long total = P * Cq;
  const float invP = 1.f / (float)P;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % Cq); const long long p = i / Cq;
    const long long n = p / HW, q = p - n * HW;
    float val = 0.f;
    if (c < C) {
      const float xh = (__ldg(x + n * sn + c * sc + q * sp) - mean[c]) * rstd[c];
      val = (weight ? weight[c] : 1.f) * rstd[c] * (__ldg(a + p * ld + c) - sums[c] * invP - xh * sums[32 + c] * invP);
    }
    out[n * on + c * oc + q * op] = val;
    if (out_lo) out_lo[n * on + c * oc + q * op] = lo_part(val);
  }
}

// dgamma (+)= sum gh xhat + sum gth t0,  dbeta (+)= sum gh,  t0 = rstd (xdot - mean(xdot) - xhat mean(xdot xhat))
//   sums_g  = {S gh, S gh xhat};  sums_t = {S gth, S gth xhat, S gth xdot} (NULL: first order);  sums_v = {S xdot, S xdot xhat}
__global__ void bn2d_param_grad_kernel(int C, long long P, const float* __restrict__ rstd, const float* __restrict__ sums_g,
                                       const float* __restrict__ sums_t, const float* __restrict__ sums_v, float* dgamma, float* dbeta,
                                       int accumulate) {
  const int c = threadIdx.x;
  if (c >= C) return;
  float g = sums_g[32 + c];
  if (sums_t) {
    const float invP = 1.f / (float)P;
    g += rstd[c] * (sums_t[64 + c] - sums_v[c] * invP * sums_t[c] - sums_v[32 + c] * invP * sums_t[32 + c]);
  }
  const float bq = sums_g[c];
  if (dgamma) dgamma[c] = accumulate ? dgamma[c] + g : g;
  if (dbeta) dbeta[c] = accumulate ? dbeta[c] + bq : bq;
}

// ====================================================================================================================
// pointwise preprocessing of preprocess_GAN_mode 2 (nn.Tanh) and 3 (lambda x: 2 * (x / 255 - 0.5)), sagan_models.py:149-152
// ====================================================================================================================
// Mode 3 keeps the reference's operation order in fp32 with IEEE division (torch's CPU `x / 255` is a true division, not a
// multiply by the reciprocal); the explicit _rn intrinsics keep the compiler from contracting the steps into one FMA.
__device__ __forceinline__ float pointwise_prep(int mode, float x) {
  return mode == 2 ? tanhf(x) : __fmul_rn(2.f, __fsub_rn(__fdiv_rn(x, 255.f), 0.5f));
}

// out[p][c] = f(x) for c < C; channels C..Cp-1 zero (the same output contract as bn2d_apply_kernel)
__global__ void __launch_bounds__(256)
pointwise_prep_kernel(int mode, int N, int C, int HW, const float* __restrict__ x, long long sn, long long sc, long long sp,
                      float* __restrict__ out, float* __restrict__ out_lo, int Cp) {
  const long long total = (long long)N * HW * Cp;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % Cp); const long long p = i / Cp;
    float val = 0.f;
    if (c < C) {
      const long long n = p / HW, q = p - n * HW;
      val = pointwise_prep(mode, __ldg(x + n * sn + c * sc + q * sp));
    }
    out[i] = val;
    if (out_lo) out_lo[i] = lo_part(val);
  }
}

// out = f'(x) * a.  Mode 2: torch's tanh_backward a * (1 - y^2) with y = tanhf(x) in full fp32 (exactly 0 where tanhf saturates
// to +-1).  Mode 3: autograd's order for 2 * (x / 255 - 0.5): (a * 2) / 255.  The Jacobian is diagonal, hence its own transpose:
// the same kernel gives the input gradient and the forward-mode tangent.  a dense [N*HW][ld], out strided; channels C..Cq-1 zero.
__global__ void __launch_bounds__(256)
pointwise_prep_jacobian_kernel(int mode, int N, int C, int HW, const float* __restrict__ x, long long sn, long long sc, long long sp,
                               const float* __restrict__ a, int ld, float* __restrict__ out, long long on, long long oc, long long op,
                               int Cq, float* __restrict__ out_lo) {
  const long long total = (long long)N * HW * Cq;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % Cq); const long long p = i / Cq;
    const long long n = p / HW, q = p - n * HW;
    float val = 0.f;
    if (c < C) {
      const float g = __ldg(a + p * ld + c);
      if (mode == 2) {
        const float y = tanhf(__ldg(x + n * sn + c * sc + q * sp));
        val = __fmul_rn(g, __fsub_rn(1.f, __fmul_rn(y, y)));
      } else {
        val = __fdiv_rn(__fmul_rn(g, 2.f), 255.f);
      }
    }
    out[n * on + c * oc + q * op] = val;
    if (out_lo) out_lo[n * on + c * oc + q * op] = lo_part(val);
  }
}

// ====================================================================================================================
// element-wise glue around the convolutions
// ====================================================================================================================
// out = in * leaky'(ref)   (the mask is recovered from the sign of the post-activation output; ref repeats every `period` elements:
// the tangent half of a [primal | tangent] batch uses the primal mask)
__global__ void __launch_bounds__(256)
mask_mul_kernel(long long n4, long long period4, const float4* __restrict__ ref, const float4* __restrict__ in, float4* __restrict__ out,
                float4* __restrict__ out_lo, float slope) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
    const float4 r = __ldg(ref + (i % period4)), v = __ldg(in + i);
    float4 o;
    o.x = r.x > 0.f ? v.x : v.x * slope; o.y = r.y > 0.f ? v.y : v.y * slope;
    o.z = r.z > 0.f ? v.z : v.z * slope; o.w = r.w > 0.f ? v.w : v.w * slope;
    out[i] = o;
    if (out_lo) out_lo[i] = make_float4(lo_part(o.x), lo_part(o.y), lo_part(o.z), lo_part(o.w));
  }
}

// parity-class channels [B][Hj][Wj][4*Cp] -> dx [B][H][W][Cq] (x leaky mask of ref [Bref][H][W][C], ref may be NULL)
__global__ void __launch_bounds__(256)
dgrad_unshuffle_kernel(int B, int H, int W, int C, int Cp, int Hj, int Wj, const float* __restrict__ d2s, const float* __restrict__ ref,
                       int Bref, float slope, float* __restrict__ out, int Cq, float* __restrict__ out_lo) {
  const long long total = (long long)B * H * W * Cq;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % Cq); long long r = i / Cq;
    const int xx = (int)(r % W); r /= W;
    const int yy = (int)(r % H); const int b = (int)(r / H);
    float val = 0.f;
    if (c < C) {
      val = __ldg(d2s + (((size_t)b * Hj + (yy >> 1)) * Wj + (xx >> 1)) * (4 * Cp) + ((yy & 1) * 2 + (xx & 1)) * Cp + c);
      if (ref) {
        const float rv = __ldg(ref + (((size_t)(b % Bref) * H + yy) * W + xx) * C + c);
        if (!(rv > 0.f)) val *= slope;
      }
    }
    out[i] = val;
    if (out_lo) out_lo[i] = lo_part(val);
  }
}

// ====================================================================================================================
// the "last" convolution: Cout = 1, KH x KW window, no padding (sagan_models.py:140)
// ====================================================================================================================
__global__ void __launch_bounds__(256)
last_fwd_kernel(int H, int W, int C, int KH, int KW, int OH, int OW, const float* __restrict__ x, const float* __restrict__ w,
                int w_row, const float* __restrict__ bias, float* __restrict__ out) {
  __shared__ float sh[64];
  const int o = blockIdx.x;
  const int ox = o % OW, oy = (o / OW) % OH, b = o / (OW * OH);
  const int len = KH * KW * C;
  float acc = 0.f;
  for (int i = threadIdx.x; i < len; i += 256) {
    const int c = i % C, kx = (i / C) % KW, ky = i / (C * KW);
    acc = fmaf(__ldg(x + (((size_t)b * H + oy + ky) * W + ox + kx) * C + c), __ldg(w + (size_t)ky * w_row + kx * C + c), acc);
  }
  acc = block_sum(acc, sh);
  if (threadIdx.x == 0) out[o] = acc + (bias ? bias[0] : 0.f);
}

__global__ void __launch_bounds__(256)
last_dgrad_kernel(int B, int H, int W, int C, int KH, int KW, int OH, int OW, const float* __restrict__ gout, const float* __restrict__ w,
                  int w_row, float* __restrict__ gx, float* __restrict__ gx_lo) {
  const long long total = (long long)B * H * W * C;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % C); long long r = i / C;
    const int xx = (int)(r % W); r /= W;
    const int yy = (int)(r % H); const int b = (int)(r / H);
    float acc = 0.f;
    for (int oy = max(0, yy - KH + 1); oy <= min(yy, OH - 1); ++oy)
      for (int ox = max(0, xx - KW + 1); ox <= min(xx, OW - 1); ++ox)
        acc = fmaf(gout ? __ldg(gout + ((size_t)b * OH + oy) * OW + ox) : 1.f, __ldg(w + (size_t)(yy - oy) * w_row + (xx - ox) * C + c), acc);
    gx[i] = acc;
    if (gx_lo) gx_lo[i] = lo_part(acc);
  }
}

__global__ void __launch_bounds__(256)
last_wgrad_kernel(int B, int H, int W, int C, int KH, int KW, int OH, int OW, const float* __restrict__ x, const float* __restrict__ gout,
                  float* gw, int w_row, float* gbias, int accumulate) {
  const int len = KH * KW * C;
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i < len) {
    const int c = i % C, kx = (i / C) % KW, ky = i / (C * KW);
    float acc = 0.f;
    for (int b = 0; b < B; ++b)
      for (int oy = 0; oy < OH; ++oy)
        for (int ox = 0; ox < OW; ++ox)
          acc = fmaf(gout ? __ldg(gout + ((size_t)b * OH + oy) * OW + ox) : 1.f, __ldg(x + (((size_t)b * H + oy + ky) * W + ox + kx) * C + c), acc);
    float* dst = gw + (size_t)ky * w_row + kx * C + c;
    *dst = accumulate ? *dst + acc : acc;
  }
  if (gbias && blockIdx.x == 0 && threadIdx.x == 0) {
    float s = 0.f;
    for (int o = 0; o < B * OH * OW; ++o) s += gout ? __ldg(gout + o) : 1.f;
    gbias[0] = accumulate ? gbias[0] + s : s;
  }
}

// ====================================================================================================================
// adversarial losses (utils/criterion.py:129-166) and the WGAN-GP penalty (:98-120)
// ====================================================================================================================
// type 0: wgan-gp  loss = -mean(real) + mean(fake);  1: hinge  mean(relu(1-real)) + mean(relu(1+fake));  2: generator  -mean(fake)
__global__ void adv_loss_kernel(int n, const float* __restrict__ real, const float* __restrict__ fake, int type, float* loss,
                                float* g_real, float* g_fake) {
  __shared__ float sh[64];
  float acc = 0.f;
  const float inv = 1.f / (float)n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    float gr = 0.f, gf = 0.f;
    if (type == 0) { acc += fake[i] - real[i]; gr = -inv; gf = inv; }
    else if (type == 1) {
      const float a = 1.f - real[i], bq = 1.f + fake[i];
      acc += fmaxf(a, 0.f) + fmaxf(bq, 0.f);
      gr = a > 0.f ? -inv : 0.f; gf = bq > 0.f ? inv : 0.f;
    } else { acc -= fake[i]; gf = -inv; }
    if (g_real) g_real[i] = gr;
    if (g_fake) g_fake[i] = gf;
  }
  acc = block_sum(acc, sh);
  if (threadIdx.x == 0) loss[0] = acc * inv;
}

__global__ void __launch_bounds__(1024)
gp_norm_kernel(long long len, const float* __restrict__ g, float* __restrict__ norms) {
  __shared__ double sh[1024];
  const float* p = g + (size_t)blockIdx.x * len;
  double acc = 0.0;
  for (long long i = threadIdx.x; i < len; i += 1024) { const float t = __ldg(p + i); acc += (double)t * t; }
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) { if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o]; __syncthreads(); }
  if (threadIdx.x == 0) norms[blockIdx.x] = (float)sqrt(sh[0]);
}
__global__ void gp_loss_kernel(int B, const float* __restrict__ norms, float lambda_gp, float* loss) {
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int b = 0; b < B; ++b) { const float d = norms[b] - 1.f; s = fmaf(d, d, s); }
    loss[0] = lambda_gp * s / (float)B;
  }
}
// v_n = upstream * 2 lambda / B * (|g_n| - 1) / |g_n| * g_n : the constant tangent direction of the penalty's parameter gradient
__global__ void __launch_bounds__(256)
gp_direction_kernel(int B, long long len, const float* __restrict__ g, const float* __restrict__ norms, float lambda_gp,
                    const float* __restrict__ upstream, float* __restrict__ v) {
  const int b = blockIdx.y;
  const float nn = norms[b];
  const float c = (upstream ? upstream[0] : 1.f) * 2.f * lambda_gp / (float)B * (nn - 1.f) / nn;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < len; i += (long long)gridDim.x * 256)
    v[(size_t)b * len + i] = c * __ldg(g + (size_t)b * len + i);
}

// ====================================================================================================================
// Self attention core (sagan_models.py:31-40): A = softmax(Q K^T) (no 1/sqrt(d)), O = A V, y = gamma O + x
// rows are positions: qkv [B*n][ldq] = [q (d) | k (d) | v (C)], x / o / y [B*n][C]
// ====================================================================================================================
constexpr int kAttnMaxN = 128;
constexpr int kAttnFwdSlice = 64, kAttnBwdSlice = 32;

__device__ __forceinline__ void load_rows(float* dst, int ldd, const float* __restrict__ src, long long lds, int rows, int cols, float mul = 1.f) {
  for (int i = threadIdx.x; i < rows * cols; i += blockDim.x) {
    const int r = i / cols, c = i - r * cols;
    dst[r * ldd + c] = src ? __ldg(src + (long long)r * lds + c) * mul : 0.f;
  }
}

// softmax over each row of s[n][ld] in place (warp per row)
__device__ __forceinline__ void softmax_rows(float* s, int n, int ld) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int i = warp; i < n; i += nw) {
    float* row = s + i * ld;
    float m = -INFINITY;
    for (int j = lane; j < n; j += 32) m = fmaxf(m, row[j]);
    m = warp_max(m);
    float sum = 0.f;
    for (int j = lane; j < n; j += 32) { const float e = __expf(row[j] - m); row[j] = e; sum += e; }
    sum = warp_sum(sum);
    const float inv = 1.f / sum;
    for (int j = lane; j < n; j += 32) row[j] *= inv;
  }
}

// grid (B, C / 64).  Every slice CTA recomputes the n x n scores (n^2 d MACs, less than its n^2 64 share of A V).
__global__ void __launch_bounds__(256)
attn_fwd_kernel(int n, int C, int d, const float* __restrict__ qkv, int ldq, const float* __restrict__ x, const float* __restrict__ gamma,
                float* __restrict__ attn, float* __restrict__ o, float* __restrict__ y, float* __restrict__ y_lo, int tc) {
  extern __shared__ float smem[];
  const int b = blockIdx.x, sl = blockIdx.y;
  const int ldA = n + 1, ldD = d + 1, CS = kAttnFwdSlice;
  float* sA = smem;                       // [n][n+1]
  float* sQ = sA + n * ldA;               // [n][d+1]
  float* sK = sQ + n * ldD;               // [n][d+1]
  float* sV = sK + n * ldD;               // [n][CS+1]
  const float* base = qkv + (size_t)b * n * ldq;
  load_rows(sQ, ldD, base, ldq, n, d);
  load_rows(sK, ldD, base + d, ldq, n, d);
  const int c0 = sl * CS, cw = min(CS, C - c0);
  load_rows(sV, CS + 1, base + 2 * d + c0, ldq, n, cw);
  __syncthreads();
  attn_gemm<4, 4>(tc, n, n, d, [&](int i, int k) { return sQ[i * ldD + k]; }, [&](int k, int j) { return sK[j * ldD + k]; },
                   [&](int i, int j, float v) { sA[i * ldA + j] = v; });
  __syncthreads();
  softmax_rows(sA, n, ldA);
  __syncthreads();
  if (sl == 0 && attn)
    for (int i = threadIdx.x; i < n * n; i += 256) attn[(size_t)b * n * n + i] = sA[(i / n) * ldA + (i % n)];
  const float gm = gamma[0];
  attn_gemm<4, 4>(tc, n, cw, n, [&](int i, int k) { return sA[i * ldA + k]; }, [&](int k, int j) { return sV[k * (CS + 1) + j]; },
                   [&](int i, int j, float v) {
                     const size_t idx = ((size_t)b * n + i) * C + c0 + j;
                     if (o) o[idx] = v;
                     const float yy = fmaf(gm, v, __ldg(x + idx));
                     y[idx] = yy;
                     if (y_lo) y_lo[idx] = lo_part(yy);
                   });
}

// Forward-mode tangent: Sdot = Qdot K^T + Q Kdot^T, Adot = A (Sdot - rowsum(A Sdot)), Odot = Adot V + A Vdot, ydot = gamma Odot + xdot
__global__ void __launch_bounds__(256)
attn_tangent_kernel(int n, int C, int d, const float* __restrict__ qkv, const float* __restrict__ tqkv, int ldq,
                    const float* __restrict__ attn, const float* __restrict__ tx, const float* __restrict__ gamma, float* __restrict__ dattn,
                    float* __restrict__ to, float* __restrict__ ty, float* __restrict__ ty_lo, int tc) {
  extern __shared__ float smem[];
  const int b = blockIdx.x, sl = blockIdx.y;
  const int ldA = n + 1, ldD = d + 1, CS = kAttnFwdSlice, ldV = CS + 1;
  float* sA = smem;                       // [n][n+1]
  float* sdA = sA + n * ldA;              // [n][n+1]
  float* sQ = sdA + n * ldA;              // q, k, qdot, kdot: 4 x [n][d+1]; later reused for the V / Vdot slices
  float* sK = sQ + n * ldD;
  float* sTQ = sK + n * ldD;
  float* sTK = sTQ + n * ldD;
  const float* base = qkv + (size_t)b * n * ldq;
  const float* tbase = tqkv + (size_t)b * n * ldq;
  load_rows(sA, ldA, attn + (size_t)b * n * n, n, n, n);
  load_rows(sQ, ldD, base, ldq, n, d);
  load_rows(sK, ldD, base + d, ldq, n, d);
  load_rows(sTQ, ldD, tbase, ldq, n, d);
  load_rows(sTK, ldD, tbase + d, ldq, n, d);
  __syncthreads();
  attn_gemm<4, 4>(tc, n, n, 2 * d,
                   [&](int i, int k) { return k < d ? sTQ[i * ldD + k] : sQ[i * ldD + k - d]; },
                   [&](int k, int j) { return k < d ? sK[j * ldD + k] : sTK[j * ldD + k - d]; },
                   [&](int i, int j, float v) { sdA[i * ldA + j] = v; });
  __syncthreads();
  {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = warp; i < n; i += 8) {
      float r = 0.f;
      for (int j = lane; j < n; j += 32) r = fmaf(sA[i * ldA + j], sdA[i * ldA + j], r);
      r = warp_sum(r);
      for (int j = lane; j < n; j += 32) sdA[i * ldA + j] = sA[i * ldA + j] * (sdA[i * ldA + j] - r);
    }
  }
  __syncthreads();
  if (sl == 0 && dattn)
    for (int i = threadIdx.x; i < n * n; i += 256) dattn[(size_t)b * n * n + i] = sdA[(i / n) * ldA + (i % n)];
  float* sV = sQ;                          // the q/k region is free now: 4 n (d+1) >= 2 n 65 floats is checked by the launcher
  float* sTV = sV + n * ldV;
  const int c0 = sl * CS, cw = min(CS, C - c0);
  load_rows(sV, ldV, base + 2 * d + c0, ldq, n, cw);
  load_rows(sTV, ldV, tbase + 2 * d + c0, ldq, n, cw);
  __syncthreads();
  const float gm = gamma[0];
  attn_gemm<4, 4>(tc, n, cw, 2 * n,
                   [&](int i, int k) { return k < n ? sdA[i * ldA + k] : sA[i * ldA + k - n]; },
                   [&](int k, int j) { return k < n ? sV[k * ldV + j] : sTV[(k - n) * ldV + j]; },
                   [&](int i, int j, float v) {
                     const size_t idx = ((size_t)b * n + i) * C + c0 + j;
                     to[idx] = v;
                     const float yy = fmaf(gm, v, __ldg(tx + idx));
                     ty[idx] = yy;
                     if (ty_lo) ty_lo[idx] = lo_part(yy);
                   });
}

// Backward stage 1, grid (B, C / 32): everything that is sliced by value channel.
//   gV    = A^T Go + Adot^T Gto            gVdot^ = A^T Gto                       (written to gqkv / gtqkv, value columns)
//   Abar1 = Go V^T + Gto Vdot^T  (partial) G      = Gto V^T  (partial: adjoint of Adot)   -> ws[b][slice][2][n][n]
//   ggamma partial = <gy, O> + <gty, Odot>                                                -> gpart[b][slice]
// with Go = gamma gy, Gto = gamma gty.  DUAL = false: first-order backward (no tangent terms).
template <bool DUAL>
__global__ void __launch_bounds__(256)
attn_bwd1_kernel(int n, int C, int d, const float* __restrict__ qkv, const float* __restrict__ tqkv, int ldq, const float* __restrict__ attn,
                 const float* __restrict__ dattn, const float* __restrict__ o, const float* __restrict__ to, const float* __restrict__ gamma,
                 const float* __restrict__ gy, const float* __restrict__ gty, float* __restrict__ gqkv, float* __restrict__ gtqkv,
                 float* __restrict__ ws, float* __restrict__ gpart, int tc) {
  extern __shared__ float smem[];
  __shared__ float red[64];
  const int b = blockIdx.x, sl = blockIdx.y, nsl = gridDim.y;
  const int ldA = n + 1, CS = kAttnBwdSlice, ldV = CS + 1;
  float* sA = smem;                                   // [n][n+1]
  float* sdA = sA + n * ldA;                          // [n][n+1]   (DUAL)
  float* sGO = DUAL ? sdA + n * ldA : sdA;            // gamma gy   [n][33]
  float* sV = sGO + n * ldV;
  float* sGTO = sV + n * ldV;                         // (DUAL)
  float* sTV = sGTO + n * ldV;                        // (DUAL)
  const int c0 = sl * CS, cw = min(CS, C - c0);
  const float gm = gamma[0];
  const size_t row0 = (size_t)b * n;
  load_rows(sA, ldA, attn + row0 * n, n, n, n);
  load_rows(sGO, ldV, gy ? gy + row0 * C + c0 : nullptr, C, n, cw, gm);
  load_rows(sV, ldV, qkv + row0 * ldq + 2 * d + c0, ldq, n, cw);
  if (DUAL) {
    load_rows(sdA, ldA, dattn + row0 * n, n, n, n);
    load_rows(sGTO, ldV, gty + row0 * C + c0, C, n, cw, gm);
    load_rows(sTV, ldV, tqkv + row0 * ldq + 2 * d + c0, ldq, n, cw);
  }
  float gp = 0.f;
  for (int i = threadIdx.x; i < n * cw; i += 256) {
    const int r = i / cw, c = i - r * cw;
    const size_t idx = (row0 + r) * C + c0 + c;
    if (gy) gp = fmaf(__ldg(gy + idx), __ldg(o + idx), gp);
    if (DUAL) gp = fmaf(__ldg(gty + idx), __ldg(to + idx), gp);
  }
  gp = block_sum(gp, red);
  if (threadIdx.x == 0) gpart[b * nsl + sl] = gp;
  __syncthreads();
  // gV[j][c] = sum_i A[i][j] Go[i][c] (+ Adot[i][j] Gto[i][c])
  attn_gemm<4, 2>(tc, n, cw, DUAL ? 2 * n : n,
                   [&](int j, int k) { return (!DUAL || k < n) ? sA[k * ldA + j] : sdA[(k - n) * ldA + j]; },
                   [&](int k, int c) { return (!DUAL || k < n) ? sGO[k * ldV + c] : sGTO[(k - n) * ldV + c]; },
                   [&](int j, int c, float v) { gqkv[(row0 + j) * ldq + 2 * d + c0 + c] = v; });
  if (DUAL)
    attn_gemm<4, 2>(tc, n, cw, n, [&](int j, int k) { return sA[k * ldA + j]; }, [&](int k, int c) { return sGTO[k * ldV + c]; },
                     [&](int j, int c, float v) { gtqkv[(row0 + j) * ldq + 2 * d + c0 + c] = v; });
  float* w1 = ws + (((size_t)b * nsl + sl) * 2) * n * n;
  // Abar1[i][j] = sum_c Go[i][c] V[j][c] (+ Gto[i][c] Vdot[j][c])
  attn_gemm<4, 4>(tc, n, n, DUAL ? 2 * cw : cw,
                   [&](int i, int k) { return (!DUAL || k < cw) ? sGO[i * ldV + k] : sGTO[i * ldV + k - cw]; },
                   [&](int k, int j) { return (!DUAL || k < cw) ? sV[j * ldV + k] : sTV[j * ldV + k - cw]; },
                   [&](int i, int j, float v) { w1[i * n + j] = v; });
  if (DUAL)
    attn_gemm<4, 4>(tc, n, n, cw, [&](int i, int k) { return sGTO[i * ldV + k]; }, [&](int k, int j) { return sV[j * ldV + k]; },
                     [&](int i, int j, float v) { w1[(size_t)n * n + i * n + j] = v; });
}

// Backward stage 2, grid (B): the n x n part.
//   g = rowsum(A G), St^ = A (G - g)                       (adjoint of Sdot)
//   Abar = Abar1 + G (Sdot - r) - g Sdot,  r = rowsum(A Sdot)
//   Sbar = A (Abar - rowsum(A Abar))
//   gQ = Sbar K + St^ Kdot, gK = Sbar^T Q + St^^T Qdot, gQdot^ = St^ K, gKdot^ = St^^T Q
//   ggamma (+)= sum of all partials (block 0; fixed order)
template <bool DUAL>
__global__ void __launch_bounds__(256)
attn_bwd2_kernel(int B, int n, int d, int nsl, const float* __restrict__ qkv, const float* __restrict__ tqkv, int ldq,
                 const float* __restrict__ attn, const float* __restrict__ ws, const float* __restrict__ gpart, float* __restrict__ gqkv,
                 float* __restrict__ gtqkv, float* ggamma, int accumulate, int tc) {
  extern __shared__ float smem[];
  const int b = blockIdx.x;
  const int ldA = n + 1, ldD = d + 1;
  float* sGS = smem;                                  // Sbar          [n][n+1]
  float* sGT = sGS + n * ldA;                         // Sdot -> St^   [n][n+1]  (DUAL)
  float* sQ = DUAL ? sGT + n * ldA : sGT;
  float* sK = sQ + n * ldD;
  float* sTQ = sK + n * ldD;                          // (DUAL)
  float* sTK = sTQ + n * ldD;                         // (DUAL)
  const size_t row0 = (size_t)b * n;
  load_rows(sQ, ldD, qkv + row0 * ldq, ldq, n, d);
  load_rows(sK, ldD, qkv + row0 * ldq + d, ldq, n, d);
  if (DUAL) {
    load_rows(sTQ, ldD, tqkv + row0 * ldq, ldq, n, d);
    load_rows(sTK, ldD, tqkv + row0 * ldq + d, ldq, n, d);
  }
  __syncthreads();
  if (DUAL) {
    attn_gemm<4, 4>(tc, n, n, 2 * d,
                     [&](int i, int k) { return k < d ? sTQ[i * ldD + k] : sQ[i * ldD + k - d]; },
                     [&](int k, int j) { return k < d ? sK[j * ldD + k] : sTK[j * ldD + k - d]; },
                     [&](int i, int j, float v) { sGT[i * ldA + j] = v; });
    __syncthreads();
  }
  {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int kPer = kAttnMaxN / 32;
    for (int i = warp; i < n; i += 8) {
      float a[kPer], ab[kPer], G[kPer], sd[kPer];
      float r = 0.f, g = 0.f;
#pragma unroll
      for (int t = 0; t < kPer; ++t) {
        const int j = lane + 32 * t;
        a[t] = ab[t] = G[t] = sd[t] = 0.f;
        if (j < n) {
          a[t] = __ldg(attn + (row0 + i) * n + j);
          for (int s = 0; s < nsl; ++s) {
            const float* w1 = ws + (((size_t)b * nsl + s) * 2) * n * n;
            ab[t] += __ldg(w1 + i * n + j);
            if (DUAL) G[t] += __ldg(w1 + (size_t)n * n + i * n + j);
          }
          if (DUAL) { sd[t] = sGT[i * ldA + j]; r = fmaf(a[t], sd[t], r); g = fmaf(a[t], G[t], g); }
        }
      }
      if (DUAL) { r = warp_sum(r); g = warp_sum(g); }
      float aa = 0.f;
#pragma unroll
      for (int t = 0; t < kPer; ++t) {
        if (DUAL) ab[t] += G[t] * (sd[t] - r) - g * sd[t];
        aa = fmaf(a[t], ab[t], aa);
      }
      aa = warp_sum(aa);
#pragma unroll
      for (int t = 0; t < kPer; ++t) {
        const int j = lane + 32 * t;
        if (j < n) {
          sGS[i * ldA + j] = a[t] * (ab[t] - aa);
          if (DUAL) sGT[i * ldA + j] = a[t] * (G[t] - g);
        }
      }
    }
  }
  __syncthreads();
  attn_gemm<4, 2>(tc, n, d, DUAL ? 2 * n : n,
                   [&](int i, int k) { return (!DUAL || k < n) ? sGS[i * ldA + k] : sGT[i * ldA + k - n]; },
                   [&](int k, int c) { return (!DUAL || k < n) ? sK[k * ldD + c] : sTK[(k - n) * ldD + c]; },
                   [&](int i, int c, float v) { gqkv[(row0 + i) * ldq + c] = v; });
  attn_gemm<4, 2>(tc, n, d, DUAL ? 2 * n : n,
                   [&](int j, int k) { return (!DUAL || k < n) ? sGS[k * ldA + j] : sGT[(k - n) * ldA + j]; },
                   [&](int k, int c) { return (!DUAL || k < n) ? sQ[k * ldD + c] : sTQ[(k - n) * ldD + c]; },
                   [&](int j, int c, float v) { gqkv[(row0 + j) * ldq + d + c] = v; });
  if (DUAL) {
    attn_gemm<4, 2>(tc, n, d, n, [&](int i, int k) { return sGT[i * ldA + k]; }, [&](int k, int c) { return sK[k * ldD + c]; },
                     [&](int i, int c, float v) { gtqkv[(row0 + i) * ldq + c] = v; });
    attn_gemm<4, 2>(tc, n, d, n, [&](int j, int k) { return sGT[k * ldA + j]; }, [&](int k, int c) { return sQ[k * ldD + c]; },
                     [&](int j, int c, float v) { gtqkv[(row0 + j) * ldq + d + c] = v; });
  }
  if (b == 0 && threadIdx.x == 0 && ggamma) {
    float t = 0.f;
    for (int i = 0; i < B * nsl; ++i) t += gpart[i];
    ggamma[0] = accumulate ? ggamma[0] + t : t;
  }
}

// --------------------------------------------------------------------------------------------------------------------
// Row-stripe attention for n > 128 (and for every n under skd_set_attn_tiled(1)).  The kernels above hold whole n x n tiles
// in shared memory; these hold stripes of R query rows ([R][n+1] each, R = 16 or 8) and stream K / Kdot / V / Vdot through
// 64-row tiles, so shared memory grows with n, not n^2.  Products accumulate tile by tile into shared memory (each output
// element is owned by one thread of one attn_gemm call, and every call is fenced by __syncthreads), in a fixed order.
// --------------------------------------------------------------------------------------------------------------------
constexpr int kAttnTiledMaxN = 1024, kAttnKeyTile = 64, kAttnKeyRows = 32;

// softmax over each of `rows` rows of s[rows][ld], `cols` entries each (warp per row)
__device__ __forceinline__ void softmax_stripe(float* s, int rows, int cols, int ld) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int i = warp; i < rows; i += nw) {
    float* row = s + i * ld;
    float m = -INFINITY;
    for (int j = lane; j < cols; j += 32) m = fmaxf(m, row[j]);
    m = warp_max(m);
    float sum = 0.f;
    for (int j = lane; j < cols; j += 32) { const float e = __expf(row[j] - m); row[j] = e; sum += e; }
    sum = warp_sum(sum);
    const float inv = 1.f / sum;
    for (int j = lane; j < cols; j += 32) row[j] *= inv;
  }
}

__device__ __forceinline__ void zero_smem(float* p, int len) {
  for (int i = threadIdx.x; i < len; i += blockDim.x) p[i] = 0.f;
}

// grid (B, n / R, C / 64): S stripe = Q_rows K^T (K in 64-row tiles), row softmax, A stripe out, O = A V (V in 64-row tiles)
__global__ void __launch_bounds__(256)
attn_fwd_tiled_kernel(int n, int C, int d, int R, const float* __restrict__ qkv, int ldq, const float* __restrict__ x,
                      const float* __restrict__ gamma, float* __restrict__ attn, float* __restrict__ o, float* __restrict__ y,
                      float* __restrict__ y_lo, int tc) {
  extern __shared__ float smem[];
  const int b = blockIdx.x, i0 = blockIdx.y * R, sl = blockIdx.z;
  const int rr = min(R, n - i0), ldS = n + 1, ldD = d + 1, ldV = kAttnFwdSlice + 1, KT = kAttnKeyTile;
  float* sS = smem;                       // [R][n+1]  scores, then A
  float* sQ = sS + R * ldS;               // [R][d+1]
  float* sO = sQ + R * ldD;               // [R][65]   O accumulator
  float* sT = sO + R * ldV;               // [64][65]  a K tile, later a V tile
  const float* base = qkv + (size_t)b * n * ldq;
  load_rows(sQ, ldD, base + (size_t)i0 * ldq, ldq, rr, d);
  zero_smem(sO, R * ldV);
  for (int j0 = 0; j0 < n; j0 += KT) {
    const int jw = min(KT, n - j0);
    __syncthreads();
    load_rows(sT, ldD, base + (size_t)j0 * ldq + d, ldq, jw, d);
    __syncthreads();
    attn_gemm<1, 4>(tc, rr, jw, d, [&](int i, int k) { return sQ[i * ldD + k]; }, [&](int k, int j) { return sT[j * ldD + k]; },
                     [&](int i, int j, float v) { sS[i * ldS + j0 + j] = v; });
  }
  __syncthreads();
  softmax_stripe(sS, rr, n, ldS);
  __syncthreads();
  if (sl == 0 && attn)
    for (int t = threadIdx.x; t < rr * n; t += 256) attn[((size_t)b * n + i0) * n + t] = sS[(t / n) * ldS + t % n];
  const int c0 = sl * kAttnFwdSlice, cw = min(kAttnFwdSlice, C - c0);
  for (int j0 = 0; j0 < n; j0 += KT) {
    const int jw = min(KT, n - j0);
    __syncthreads();
    load_rows(sT, ldV, base + (size_t)j0 * ldq + 2 * d + c0, ldq, jw, cw);
    __syncthreads();
    attn_gemm<1, 4>(tc, rr, cw, jw, [&](int i, int k) { return sS[i * ldS + j0 + k]; }, [&](int k, int c) { return sT[k * ldV + c]; },
                     [&](int i, int c, float v) { sO[i * ldV + c] += v; });
  }
  __syncthreads();
  const float gm = gamma[0];
  for (int t = threadIdx.x; t < rr * cw; t += 256) {
    const int i = t / cw, c = t - i * cw;
    const size_t idx = ((size_t)b * n + i0 + i) * C + c0 + c;
    const float v = sO[i * ldV + c];
    if (o) o[idx] = v;
    const float yy = fmaf(gm, v, __ldg(x + idx));
    y[idx] = yy;
    if (y_lo) y_lo[idx] = lo_part(yy);
  }
}

// grid (B, n / R, C / 64): Sdot stripe = Qdot K^T + Q Kdot^T, Adot = A (Sdot - rowsum(A Sdot)), Odot = Adot V + A Vdot
__global__ void __launch_bounds__(256)
attn_tangent_tiled_kernel(int n, int C, int d, int R, const float* __restrict__ qkv, const float* __restrict__ tqkv, int ldq,
                          const float* __restrict__ attn, const float* __restrict__ tx, const float* __restrict__ gamma,
                          float* __restrict__ dattn, float* __restrict__ to, float* __restrict__ ty, float* __restrict__ ty_lo, int tc) {
  extern __shared__ float smem[];
  const int b = blockIdx.x, i0 = blockIdx.y * R, sl = blockIdx.z;
  const int rr = min(R, n - i0), ldS = n + 1, ldD = d + 1, ldV = kAttnFwdSlice + 1, KT = kAttnKeyTile;
  float* sA = smem;                       // [R][n+1]
  float* sdA = sA + R * ldS;              // [R][n+1]  Sdot, then Adot
  float* sQ = sdA + R * ldS;              // [R][d+1]
  float* sTQ = sQ + R * ldD;              // [R][d+1]
  float* sO = sTQ + R * ldD;              // [R][65]   Odot accumulator
  float* sT = sO + R * ldV;               // 2 x [64][65]: K | Kdot tiles, later V | Vdot tiles
  float* sT2 = sT + KT * ldV;
  const float* base = qkv + (size_t)b * n * ldq;
  const float* tbase = tqkv + (size_t)b * n * ldq;
  load_rows(sA, ldS, attn + ((size_t)b * n + i0) * n, n, rr, n);
  load_rows(sQ, ldD, base + (size_t)i0 * ldq, ldq, rr, d);
  load_rows(sTQ, ldD, tbase + (size_t)i0 * ldq, ldq, rr, d);
  zero_smem(sO, R * ldV);
  for (int j0 = 0; j0 < n; j0 += KT) {
    const int jw = min(KT, n - j0);
    __syncthreads();
    load_rows(sT, ldD, base + (size_t)j0 * ldq + d, ldq, jw, d);
    load_rows(sT2, ldD, tbase + (size_t)j0 * ldq + d, ldq, jw, d);
    __syncthreads();
    attn_gemm<1, 4>(tc, rr, jw, 2 * d,
                     [&](int i, int k) { return k < d ? sTQ[i * ldD + k] : sQ[i * ldD + k - d]; },
                     [&](int k, int j) { return k < d ? sT[j * ldD + k] : sT2[j * ldD + k - d]; },
                     [&](int i, int j, float v) { sdA[i * ldS + j0 + j] = v; });
  }
  __syncthreads();
  {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = warp; i < rr; i += 8) {
      float r = 0.f;
      for (int j = lane; j < n; j += 32) r = fmaf(sA[i * ldS + j], sdA[i * ldS + j], r);
      r = warp_sum(r);
      for (int j = lane; j < n; j += 32) sdA[i * ldS + j] = sA[i * ldS + j] * (sdA[i * ldS + j] - r);
    }
  }
  __syncthreads();
  if (sl == 0 && dattn)
    for (int t = threadIdx.x; t < rr * n; t += 256) dattn[((size_t)b * n + i0) * n + t] = sdA[(t / n) * ldS + t % n];
  const int c0 = sl * kAttnFwdSlice, cw = min(kAttnFwdSlice, C - c0);
  for (int j0 = 0; j0 < n; j0 += KT) {
    const int jw = min(KT, n - j0);
    __syncthreads();
    load_rows(sT, ldV, base + (size_t)j0 * ldq + 2 * d + c0, ldq, jw, cw);
    load_rows(sT2, ldV, tbase + (size_t)j0 * ldq + 2 * d + c0, ldq, jw, cw);
    __syncthreads();
    attn_gemm<1, 4>(tc, rr, cw, 2 * jw,
                     [&](int i, int k) { return k < jw ? sdA[i * ldS + j0 + k] : sA[i * ldS + j0 + k - jw]; },
                     [&](int k, int c) { return k < jw ? sT[k * ldV + c] : sT2[(k - jw) * ldV + c]; },
                     [&](int i, int c, float v) { sO[i * ldV + c] += v; });
  }
  __syncthreads();
  const float gm = gamma[0];
  for (int t = threadIdx.x; t < rr * cw; t += 256) {
    const int i = t / cw, c = t - i * cw;
    const size_t idx = ((size_t)b * n + i0 + i) * C + c0 + c;
    const float v = sO[i * ldV + c];
    to[idx] = v;
    const float yy = fmaf(gm, v, __ldg(tx + idx));
    ty[idx] = yy;
    if (ty_lo) ty_lo[idx] = lo_part(yy);
  }
}

// Backward stage 1, grid (B, n / R): everything indexed by query row i.
//   Abar = Go V^T + Gto Vdot^T + G (Sdot - r) - g Sdot,  G = Gto V^T,  r = rowsum(A Sdot),  g = rowsum(A G)   (Go = gamma gy, ...)
//   Sbar = A (Abar - rowsum(A Abar)),  St^ = A (G - g)                                          -> sbar / stbar [B][n][n]
//   gQ = Sbar K + St^ Kdot,  gQdot^ = St^ K                                                     -> gqkv / gtqkv, query columns
//   per-row ggamma partials <gy, O> + <gty, Odot>                                               -> gpart [B][n]
// V / Vdot and Go / Gto are streamed in 64 x 64 tiles; K / Kdot in 64-row tiles.  DUAL = false: first-order backward.
template <bool DUAL>
__global__ void __launch_bounds__(256)
attn_bwd_rows_kernel(int n, int C, int d, int R, const float* __restrict__ qkv, const float* __restrict__ tqkv, int ldq,
                     const float* __restrict__ attn, const float* __restrict__ o, const float* __restrict__ to, const float* __restrict__ gamma,
                     const float* __restrict__ gy, const float* __restrict__ gty, float* __restrict__ gqkv, float* __restrict__ gtqkv,
                     float* __restrict__ sbar, float* __restrict__ stbar, float* __restrict__ gpart, int tc) {
  extern __shared__ float smem[];
  const int b = blockIdx.x, i0 = blockIdx.y * R;
  const int rr = min(R, n - i0), ldS = n + 1, ldD = d + 1, CS = kAttnFwdSlice, ldV = CS + 1, KT = kAttnKeyTile;
  float* p = smem;
  float* sA = p;   p += R * ldS;          // [R][n+1]
  float* sAb = p;  p += R * ldS;          // Abar, then Sbar
  float* sG = p;                          // G, then St^   (DUAL)
  float* sSd = p + R * ldS;               // Sdot          (DUAL)
  if (DUAL) p += 2 * R * ldS;
  float* sGO = p;  p += R * ldV;          // [R][65] gamma gy, one 64-channel chunk
  float* sGTO = p; if (DUAL) p += R * ldV;
  float* sQ = p;                          // q / qdot rows (DUAL: for Sdot)
  float* sTQ = p + R * ldD;
  if (DUAL) p += 2 * R * ldD;
  float* sAcc = p; p += R * ldD;          // gQ
  float* sAccT = p; if (DUAL) p += R * ldD;   // gQdot^
  float* sT = p;                          // 2 x [64][65] tiles
  float* sT2 = sT + KT * ldV;
  const float* base = qkv + (size_t)b * n * ldq;
  const float* tbase = DUAL ? tqkv + (size_t)b * n * ldq : nullptr;
  const size_t grow0 = (size_t)b * n + i0;
  const float gm = gamma[0];
  load_rows(sA, ldS, attn + grow0 * n, n, rr, n);
  zero_smem(sAb, (DUAL ? 2 : 1) * R * ldS);
  zero_smem(sAcc, (DUAL ? 2 : 1) * R * ldD);
  if (DUAL) {
    load_rows(sQ, ldD, base + (size_t)i0 * ldq, ldq, rr, d);
    load_rows(sTQ, ldD, tbase + (size_t)i0 * ldq, ldq, rr, d);
    for (int j0 = 0; j0 < n; j0 += KT) {
      const int jw = min(KT, n - j0);
      __syncthreads();
      load_rows(sT, ldD, base + (size_t)j0 * ldq + d, ldq, jw, d);
      load_rows(sT2, ldD, tbase + (size_t)j0 * ldq + d, ldq, jw, d);
      __syncthreads();
      attn_gemm<1, 4>(tc, rr, jw, 2 * d,
                       [&](int i, int k) { return k < d ? sTQ[i * ldD + k] : sQ[i * ldD + k - d]; },
                       [&](int k, int j) { return k < d ? sT[j * ldD + k] : sT2[j * ldD + k - d]; },
                       [&](int i, int j, float v) { sSd[i * ldS + j0 + j] = v; });
    }
  }
  // Abar1[i][j] = sum_c Go[i][c] V[j][c] (+ Gto[i][c] Vdot[j][c]),  G[i][j] = sum_c Gto[i][c] V[j][c]
  for (int c0 = 0; c0 < C; c0 += CS) {
    const int cw = min(CS, C - c0);
    __syncthreads();
    load_rows(sGO, ldV, gy ? gy + grow0 * C + c0 : nullptr, C, rr, cw, gm);
    if (DUAL) load_rows(sGTO, ldV, gty + grow0 * C + c0, C, rr, cw, gm);
    for (int j0 = 0; j0 < n; j0 += KT) {
      const int jw = min(KT, n - j0);
      __syncthreads();
      load_rows(sT, ldV, base + (size_t)j0 * ldq + 2 * d + c0, ldq, jw, cw);
      if (DUAL) load_rows(sT2, ldV, tbase + (size_t)j0 * ldq + 2 * d + c0, ldq, jw, cw);
      __syncthreads();
      attn_gemm<1, 4>(tc, rr, jw, DUAL ? 2 * cw : cw,
                       [&](int i, int k) { return (!DUAL || k < cw) ? sGO[i * ldV + k] : sGTO[i * ldV + k - cw]; },
                       [&](int k, int j) { return (!DUAL || k < cw) ? sT[j * ldV + k] : sT2[j * ldV + k - cw]; },
                       [&](int i, int j, float v) { sAb[i * ldS + j0 + j] += v; });
      if (DUAL)
        attn_gemm<1, 4>(tc, rr, jw, cw, [&](int i, int k) { return sGTO[i * ldV + k]; }, [&](int k, int j) { return sT[j * ldV + k]; },
                         [&](int i, int j, float v) { sG[i * ldS + j0 + j] += v; });
    }
  }
  __syncthreads();
  {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = warp; i < rr; i += 8) {
      float* a = sA + i * ldS;
      float* ab = sAb + i * ldS;
      float r = 0.f, g = 0.f;
      if (DUAL) {
        for (int j = lane; j < n; j += 32) { r = fmaf(a[j], sSd[i * ldS + j], r); g = fmaf(a[j], sG[i * ldS + j], g); }
        r = warp_sum(r); g = warp_sum(g);
      }
      float aa = 0.f;
      for (int j = lane; j < n; j += 32) {
        if (DUAL) { const float sd = sSd[i * ldS + j]; ab[j] += sG[i * ldS + j] * (sd - r) - g * sd; }
        aa = fmaf(a[j], ab[j], aa);
      }
      aa = warp_sum(aa);
      float* gsb = sbar + (grow0 + i) * n;
      for (int j = lane; j < n; j += 32) {
        const float s = a[j] * (ab[j] - aa);
        ab[j] = s;
        gsb[j] = s;
        if (DUAL) {
          const float st = a[j] * (sG[i * ldS + j] - g);
          sG[i * ldS + j] = st;
          stbar[(grow0 + i) * n + j] = st;
        }
      }
      float gp = 0.f;
      for (int c = lane; c < C; c += 32) {
        const size_t idx = (grow0 + i) * C + c;
        if (gy) gp = fmaf(__ldg(gy + idx), __ldg(o + idx), gp);
        if (DUAL) gp = fmaf(__ldg(gty + idx), __ldg(to + idx), gp);
      }
      gp = warp_sum(gp);
      if (lane == 0) gpart[grow0 + i] = gp;
    }
  }
  // gQ[i] = sum_j Sbar[i][j] K[j] (+ St^[i][j] Kdot[j]),  gQdot^[i] = sum_j St^[i][j] K[j]
  for (int j0 = 0; j0 < n; j0 += KT) {
    const int jw = min(KT, n - j0);
    __syncthreads();
    load_rows(sT, ldD, base + (size_t)j0 * ldq + d, ldq, jw, d);
    if (DUAL) load_rows(sT2, ldD, tbase + (size_t)j0 * ldq + d, ldq, jw, d);
    __syncthreads();
    attn_gemm<1, 4>(tc, rr, d, DUAL ? 2 * jw : jw,
                     [&](int i, int k) { return (!DUAL || k < jw) ? sAb[i * ldS + j0 + k] : sG[i * ldS + j0 + k - jw]; },
                     [&](int k, int c) { return (!DUAL || k < jw) ? sT[k * ldD + c] : sT2[(k - jw) * ldD + c]; },
                     [&](int i, int c, float v) { sAcc[i * ldD + c] += v; });
    if (DUAL)
      attn_gemm<1, 4>(tc, rr, d, jw, [&](int i, int k) { return sG[i * ldS + j0 + k]; }, [&](int k, int c) { return sT[k * ldD + c]; },
                       [&](int i, int c, float v) { sAccT[i * ldD + c] += v; });
  }
  __syncthreads();
  for (int t = threadIdx.x; t < rr * d; t += 256) {
    const int i = t / d, c = t - i * d;
    gqkv[(grow0 + i) * ldq + c] = sAcc[i * ldD + c];
    if (DUAL) gtqkv[(grow0 + i) * ldq + c] = sAccT[i * ldD + c];
  }
}

// Backward stage 2, grid (B, n / 32, 1 + C / 64): everything indexed by key row j, as X^T P (+ Y^T PT) and X^T PT over query
// tiles i of 32 rows:
//   z = 0:      gK = St^^T Qdot + Sbar^T Q,  gKdot^ = St^^T Q      (X, Y = stbar, sbar; P, PT = qdot, q.  First order: Sbar^T Q)
//   z = 1 + s:  gV = A^T Go + Adot^T Gto,    gVdot^ = A^T Gto      (X, Y = attn, dattn; P, PT = gamma gy, gamma gty; slice s)
// Block (0, 0, 0) also sums the per-row ggamma partials (fixed order).
template <bool DUAL>
__global__ void __launch_bounds__(256)
attn_bwd_keys_kernel(int B, int n, int C, int d, const float* __restrict__ qkv, const float* __restrict__ tqkv, int ldq,
                     const float* __restrict__ attn, const float* __restrict__ dattn, const float* __restrict__ gamma,
                     const float* __restrict__ gy, const float* __restrict__ gty, const float* __restrict__ sbar,
                     const float* __restrict__ stbar, const float* __restrict__ gpart, float* __restrict__ gqkv, float* __restrict__ gtqkv,
                     float* ggamma, int accumulate, int tc) {
  extern __shared__ float smem[];
  __shared__ float red[64];
  constexpr int RJ = kAttnKeyRows, IT = kAttnKeyRows, ldX = RJ + 1, ldP = kAttnFwdSlice + 1;
  const int b = blockIdx.x, j0 = blockIdx.y * RJ, z = blockIdx.z;
  const int rw = min(RJ, n - j0);
  float* sX = smem;                       // [IT][33]  X[i][j]
  float* sY = sX + IT * ldX;              // [IT][33]  Y[i][j]   (DUAL)
  float* sP = sY + IT * ldX;              // [IT][65]  P[i][c]
  float* sPT = sP + IT * ldP;             // [IT][65]  PT[i][c]  (DUAL)
  float* sAcc = sPT + IT * ldP;           // [32][65]
  float* sAccT = sAcc + RJ * ldP;         // [32][65]  (DUAL)
  const float gm = gamma[0];
  const size_t nn = (size_t)b * n * n;
  const float *X, *Y = nullptr, *P, *PT = nullptr;
  int cw, pcol, ocol;
  long long ldp;
  float mul;
  if (z == 0) {
    cw = d; pcol = 0; ocol = d; ldp = ldq; mul = 1.f;
    const float* q = qkv + (size_t)b * n * ldq;
    if (DUAL) { X = stbar + nn; Y = sbar + nn; P = tqkv + (size_t)b * n * ldq; PT = q; }
    else { X = sbar + nn; P = q; }
  } else {
    X = attn + nn;
    if (DUAL) Y = dattn + nn;
    const int c0 = (z - 1) * kAttnFwdSlice;
    cw = min(kAttnFwdSlice, C - c0); pcol = c0; ocol = 2 * d + c0; ldp = C; mul = gm;
    P = gy ? gy + (size_t)b * n * C : nullptr; PT = DUAL ? gty + (size_t)b * n * C : nullptr;
  }
  zero_smem(sAcc, 2 * RJ * ldP);
  for (int i0 = 0; i0 < n; i0 += IT) {
    const int iw = min(IT, n - i0);
    __syncthreads();
    load_rows(sX, ldX, X + (size_t)i0 * n + j0, n, iw, rw);
    load_rows(sP, ldP, P ? P + (size_t)i0 * ldp + pcol : nullptr, ldp, iw, cw, mul);
    if (DUAL) {
      load_rows(sY, ldX, Y + (size_t)i0 * n + j0, n, iw, rw);
      load_rows(sPT, ldP, PT + (size_t)i0 * ldp + pcol, ldp, iw, cw, mul);
    }
    __syncthreads();
    attn_gemm<1, 4>(tc, rw, cw, DUAL ? 2 * iw : iw,
                     [&](int j, int k) { return (!DUAL || k < iw) ? sX[k * ldX + j] : sY[(k - iw) * ldX + j]; },
                     [&](int k, int c) { return (!DUAL || k < iw) ? sP[k * ldP + c] : sPT[(k - iw) * ldP + c]; },
                     [&](int j, int c, float v) { sAcc[j * ldP + c] += v; });
    if (DUAL)
      attn_gemm<1, 4>(tc, rw, cw, iw, [&](int j, int k) { return sX[k * ldX + j]; }, [&](int k, int c) { return sPT[k * ldP + c]; },
                       [&](int j, int c, float v) { sAccT[j * ldP + c] += v; });
  }
  __syncthreads();
  for (int t = threadIdx.x; t < rw * cw; t += 256) {
    const int j = t / cw, c = t - j * cw;
    const size_t row = (size_t)b * n + j0 + j;
    gqkv[row * ldq + ocol + c] = sAcc[j * ldP + c];
    if (DUAL) gtqkv[row * ldq + ocol + c] = sAccT[j * ldP + c];
  }
  if (ggamma && b == 0 && blockIdx.y == 0 && z == 0) {
    float t = 0.f;
    for (int i = threadIdx.x; i < B * n; i += 256) t += gpart[i];
    t = block_sum(t, red);
    if (threadIdx.x == 0) ggamma[0] = accumulate ? ggamma[0] + t : t;
  }
}

template <typename Kernel>
bool set_smem(Kernel k, size_t bytes, const char* who) {
  if (bytes > 232448) { set_error_msg(who, "attention tile exceeds the 227 KB of shared memory (n <= 1024, d <= 64)"); return false; }
  cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e != cudaSuccess) { set_error(who, e); return false; }
  return true;
}

bool attn_shape_ok(int B, int n, int C, int d, int ldq, const char* who) {
  if (B <= 0 || n <= 0 || n > kAttnTiledMaxN || d <= 0 || d > 64 || C <= 0 || ldq < 2 * d + C) {
    set_error_msg(who, "unsupported attention shape (1 <= n <= 1024 positions, d <= 64, ldq >= 2d + C)");
    return false;
  }
  return true;
}

int g_attn_tiled = 0;

constexpr size_t kAttnSmemMax = 232448;

// The whole-tile kernels for n <= 128 where their tiles fit shared memory (whole_tile_bytes; at n = 128 the tangent and the joint
// backward of d = 64 do not); the row-stripe kernels for everything else, and for every n under skd_set_attn_tiled(1).
bool attn_use_tiled(int n, size_t whole_tile_bytes) { return n > kAttnMaxN || whole_tile_bytes > kAttnSmemMax || g_attn_tiled; }

// rows per stripe: 16, or 8 where 16 would not fit (floats(R) = the kernel's shared-memory floats).  8 always fits: the
// static_asserts below check the largest kernels at n = kAttnTiledMaxN, d = 64, so raising the bound fails to compile first.
template <class F>
int attn_stripe_rows(F floats) { return floats(16) * 4 <= kAttnSmemMax ? 16 : 8; }

constexpr size_t attn_fwd_tiled_floats(int R, int n, int d, bool tangent) {
  const size_t ldS = n + 1, ldD = d + 1, ldV = kAttnFwdSlice + 1;
  return (tangent ? 2 : 1) * R * ldS + (tangent ? 2 : 1) * R * ldD + R * ldV + (tangent ? 2 : 1) * kAttnKeyTile * ldV;
}

constexpr size_t attn_bwd_rows_floats(int R, int n, int d, bool dual) {
  const size_t ldS = n + 1, ldD = d + 1, ldV = kAttnFwdSlice + 1;
  return (dual ? 4 : 2) * R * ldS + (dual ? 2 : 1) * R * ldV + (dual ? 4 : 1) * R * ldD + 2 * kAttnKeyTile * ldV;
}

static_assert(attn_fwd_tiled_floats(8, kAttnTiledMaxN, 64, true) * 4 <= kAttnSmemMax, "tangent stripe of 8 rows must fit at the bound");
static_assert(attn_bwd_rows_floats(8, kAttnTiledMaxN, 64, true) * 4 <= kAttnSmemMax, "joint backward stripe of 8 rows must fit at the bound");

constexpr size_t kAttnKeysBytes = (2 * kAttnKeyRows * (kAttnKeyRows + 1) + 4 * kAttnKeyRows * (kAttnFwdSlice + 1)) * 4;

}  // namespace

// ---------------------------------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------------------------------
extern "C" int skd_sn_power_iter(int Cout, int taps, int Cin, const float* w_bar, float* u, float* v, float* u_save, float* v_save,
                                 float* sigma, float* inv_sigma_vec, int vec_len, cudaStream_t st) {
  const char* who = "skd_sn_power_iter";
  if (taps * Cin > kSnMaxK || Cout > kSnCluster * kSnMaxRows || Cout <= 0) { set_error_msg(who, "weight matrix too large (K <= 8192, Cout <= 2048)"); return 0; }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(kSnCluster); cfg.blockDim = dim3(kSnThreads); cfg.dynamicSmemBytes = 0; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = kSnCluster; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, sn_power_iter_kernel, Cout, taps, Cin, w_bar, u, v, u_save, v_save, sigma, inv_sigma_vec, vec_len);
  if (e != cudaSuccess) { set_error(who, e); return 0; }
  return finish(who);
}

static long long sn_layer_ws_floats(int Cout, int K) {
  const long long n_rb = (Cout + kSnRowBlock - 1) / kSnRowBlock;
  return ((n_rb + 1) * K + Cout + 3) / 4 * 4;
}

extern "C" long long skd_sn_power_iter_batched_workspace_floats(int n_layers, const skd_sn_layer* layers) {
  long long t = 0;
  for (int i = 0; i < n_layers; ++i) t += sn_layer_ws_floats(layers[i].Cout, layers[i].taps * layers[i].Cin);
  return t;
}

extern "C" int skd_sn_power_iter_batched(int n_layers, const skd_sn_layer* layers, float* workspace, cudaStream_t st) {
  const char* who = "skd_sn_power_iter_batched";
  if (n_layers <= 0) return 1;
  if (n_layers > kSnBatchMax) { set_error_msg(who, "at most 8 layers per call"); return 0; }
  SnBatch b; b.n = n_layers;
  int blk1 = 0, blk3 = 0;
  float* ws = workspace;
  for (int i = 0; i < n_layers; ++i) {
    const skd_sn_layer& in = layers[i];
    SnLayer& L = b.L[i];
    L.Cout = in.Cout; L.taps = in.taps; L.Cin = in.Cin; L.K = in.taps * in.Cin; L.vec_len = in.vec_len;
    if (L.K > kSnMaxK || L.K <= 0 || L.Cout <= 0) { set_error_msg(who, "weight matrix too large (K <= 8192)"); return 0; }
    L.n_rb = (L.Cout + kSnRowBlock - 1) / kSnRowBlock; L.n_kb = (L.K + kSnKBlock - 1) / kSnKBlock;
    L.blk1 = blk1; blk1 += L.n_rb * L.n_kb;
    L.blk3 = blk3; blk3 += (L.Cout + 7) / 8;
    L.w = in.w_bar; L.u = in.u; L.v = in.v; L.u_save = in.u_save; L.v_save = in.v_save; L.sigma = in.sigma; L.inv_vec = in.inv_sigma_vec;
    L.tpart = ws; L.vlin = ws + (size_t)L.n_rb * L.K; L.s = L.vlin + L.K;
    ws += sn_layer_ws_floats(L.Cout, L.K);
  }
  sn_phase1_kernel<<<blk1, 256, 0, st>>>(b);
  sn_phase2_kernel<<<n_layers, 1024, 0, st>>>(b);
  sn_phase3_kernel<<<blk3, 256, 0, st>>>(b);
  sn_phase4_kernel<<<n_layers, 256, 0, st>>>(b);
  return finish(who, 4);
}

extern "C" long long skd_sn_weight_grad_workspace_doubles(void) { return 1 + kDotBlocks + 1; }

extern "C" int skd_sn_weight_grad(int Cout, int taps, int Cin, int Cin_p, const float* d_wn, const float* w_bar, const float* u,
                                  const float* v, const float* sigma, float* d_w, int accumulate, double* workspace, cudaStream_t st) {
  sn_grad_dot_kernel<<<kDotBlocks, 256, 0, st>>>(Cout, taps, Cin, Cin_p, d_wn, w_bar, workspace);
  sn_grad_apply_kernel<<<blocks_for((long long)Cout * taps * Cin), 256, 0, st>>>(Cout, taps, Cin, Cin_p, d_wn, u, v, sigma, workspace, d_w, accumulate);
  return finish("skd_sn_weight_grad", 2);
}

extern "C" int skd_disc_weight_prep(long long rows, int Cin, int Cin_p, const float* w, float* w_pad, float* w_lo, cudaStream_t st) {
  weight_prep_kernel<<<blocks_for(rows * Cin_p), 256, 0, st>>>(rows, Cin, Cin_p, w, w_pad, w_lo);
  return finish("skd_disc_weight_prep");
}

extern "C" int skd_disc_dgrad_weight_prep(int Cout, int Cin, int Cin_p, const float* w, float* wd, float* wd_lo, cudaStream_t st) {
  dgrad_weight_prep_kernel<<<blocks_for(36LL * Cin_p * Cout), 256, 0, st>>>(Cout, Cin, Cin_p, w, wd, wd_lo);
  return finish("skd_disc_dgrad_weight_prep");
}

extern "C" long long skd_bn2d_workspace_doubles(void) { return (long long)kBnBlocks * 96 + 1; }

extern "C" int skd_bn2d_stats(int N, int C, int HW, const float* x, long long sn, long long sc, long long sp, float eps, float momentum,
                              float* running_mean, float* running_var, long long* num_batches_tracked, float* mean, float* rstd,
                              double* workspace, cudaStream_t st) {
  if (C > 32 || C <= 0) { set_error_msg("skd_bn2d_stats", "C must be in 1..32"); return 0; }
  bn2d_reduce_kernel<0><<<kBnBlocks, 256, 0, st>>>(N, C, HW, x, sn, sc, sp, nullptr, nullptr, nullptr, nullptr, 0, eps, momentum, running_mean,
                                                   running_var, num_batches_tracked, mean, rstd, nullptr, workspace);
  return finish("skd_bn2d_stats");
}

extern "C" int skd_bn2d_apply(int N, int C, int HW, const float* x, long long sn, long long sc, long long sp, const float* mean,
                              const float* rstd, const float* weight, const float* bias, float* out, float* out_lo, int Cp, cudaStream_t st) {
  bn2d_apply_kernel<<<blocks_for((long long)N * HW * Cp), 256, 0, st>>>(N, C, HW, x, sn, sc, sp, mean, rstd, weight, bias, out, out_lo, Cp);
  return finish("skd_bn2d_apply");
}

extern "C" int skd_bn2d_reduce(int N, int C, int HW, const float* x, long long sn, long long sc, long long sp, const float* mean,
                               const float* rstd, const float* a, const float* b, int ld, float* sums, double* workspace, cudaStream_t st) {
  if (C > 32 || C <= 0) { set_error_msg("skd_bn2d_reduce", "C must be in 1..32"); return 0; }
  bn2d_reduce_kernel<1><<<kBnBlocks, 256, 0, st>>>(N, C, HW, x, sn, sc, sp, mean, rstd, a, b, ld, 0.f, 0.f, nullptr, nullptr, nullptr, nullptr,
                                                   nullptr, sums, workspace);
  return finish("skd_bn2d_reduce");
}

extern "C" int skd_bn2d_jacobian(int N, int C, int HW, const float* x, long long sn, long long sc, long long sp, const float* mean,
                                 const float* rstd, const float* weight, const float* a, int ld, const float* sums, float* out, long long on,
                                 long long oc, long long op, int Cq, float* out_lo, cudaStream_t st) {
  bn2d_jacobian_kernel<<<blocks_for((long long)N * HW * Cq), 256, 0, st>>>(N, C, HW, x, sn, sc, sp, mean, rstd, weight, a, ld, sums, out, on, oc, op,
                                                                          Cq, out_lo);
  return finish("skd_bn2d_jacobian");
}

extern "C" int skd_bn2d_param_grad(int C, long long P, const float* rstd, const float* sums_g, const float* sums_t, const float* sums_v,
                                   float* dgamma, float* dbeta, int accumulate, cudaStream_t st) {
  bn2d_param_grad_kernel<<<1, 32, 0, st>>>(C, P, rstd, sums_g, sums_t, sums_v, dgamma, dbeta, accumulate);
  return finish("skd_bn2d_param_grad");
}

extern "C" int skd_disc_pointwise_prep(int mode, int N, int C, int HW, const float* x, long long sn, long long sc, long long sp, float* out,
                                       float* out_lo, int Cp, cudaStream_t st) {
  if (mode != 2 && mode != 3) { set_error_msg("skd_disc_pointwise_prep", "mode must be 2 (tanh) or 3 (rescale)"); return 0; }
  if (C <= 0 || Cp < C) { set_error_msg("skd_disc_pointwise_prep", "need 0 < C <= Cp"); return 0; }
  pointwise_prep_kernel<<<blocks_for((long long)N * HW * Cp), 256, 0, st>>>(mode, N, C, HW, x, sn, sc, sp, out, out_lo, Cp);
  return finish("skd_disc_pointwise_prep");
}

extern "C" int skd_disc_pointwise_prep_jacobian(int mode, int N, int C, int HW, const float* x, long long sn, long long sc, long long sp,
                                                const float* a, int ld, float* out, long long on, long long oc, long long op, int Cq,
                                                float* out_lo, cudaStream_t st) {
  if (mode != 2 && mode != 3) { set_error_msg("skd_disc_pointwise_prep_jacobian", "mode must be 2 (tanh) or 3 (rescale)"); return 0; }
  if (C <= 0 || Cq < C || ld < C) { set_error_msg("skd_disc_pointwise_prep_jacobian", "need 0 < C <= Cq and C <= ld"); return 0; }
  pointwise_prep_jacobian_kernel<<<blocks_for((long long)N * HW * Cq), 256, 0, st>>>(mode, N, C, HW, x, sn, sc, sp, a, ld, out, on, oc, op, Cq,
                                                                                    out_lo);
  return finish("skd_disc_pointwise_prep_jacobian");
}

extern "C" int skd_disc_mask_mul(long long n, long long period, const float* ref, const float* in, float* out, float* out_lo, float slope,
                                 cudaStream_t st) {
  if (n % 4 || period % 4 || ((reinterpret_cast<uintptr_t>(ref) | reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out) |
                              reinterpret_cast<uintptr_t>(out_lo)) & 15)) {
    set_error_msg("skd_disc_mask_mul", "sizes must be multiples of 4 and pointers 16-byte aligned"); return 0;
  }
  if (n <= 0) return 1;
  mask_mul_kernel<<<blocks_for(n / 4), 256, 0, st>>>(n / 4, period / 4, reinterpret_cast<const float4*>(ref), reinterpret_cast<const float4*>(in),
                                                     reinterpret_cast<float4*>(out), reinterpret_cast<float4*>(out_lo), slope);
  return finish("skd_disc_mask_mul");
}

extern "C" int skd_disc_dgrad_unshuffle(int B, int H, int W, int C, int Cp, const float* d2s, const float* ref, int ref_batch, float slope,
                                        float* out, int Cq, float* out_lo, cudaStream_t st) {
  const int Hj = (H + 1) / 2, Wj = (W + 1) / 2;
  dgrad_unshuffle_kernel<<<blocks_for((long long)B * H * W * Cq), 256, 0, st>>>(B, H, W, C, Cp, Hj, Wj, d2s, ref, ref_batch > 0 ? ref_batch : B, slope,
                                                                               out, Cq, out_lo);
  return finish("skd_disc_dgrad_unshuffle");
}

extern "C" int skd_disc_last_fwd(int B, int H, int W, int C, int KH, int KW, const float* x, const float* w, int w_row, const float* bias,
                                 float* out, cudaStream_t st) {
  const int OH = H - KH + 1, OW = W - KW + 1;
  if (OH <= 0 || OW <= 0) { set_error_msg("skd_disc_last_fwd", "window larger than the map"); return 0; }
  last_fwd_kernel<<<B * OH * OW, 256, 0, st>>>(H, W, C, KH, KW, OH, OW, x, w, w_row, bias, out);
  return finish("skd_disc_last_fwd");
}

extern "C" int skd_disc_last_dgrad(int B, int H, int W, int C, int KH, int KW, const float* gout, const float* w, int w_row, float* gx,
                                   float* gx_lo, cudaStream_t st) {
  const int OH = H - KH + 1, OW = W - KW + 1;
  last_dgrad_kernel<<<blocks_for((long long)B * H * W * C), 256, 0, st>>>(B, H, W, C, KH, KW, OH, OW, gout, w, w_row, gx, gx_lo);
  return finish("skd_disc_last_dgrad");
}

extern "C" int skd_disc_last_wgrad(int B, int H, int W, int C, int KH, int KW, const float* x, const float* gout, float* gw, int w_row,
                                   float* gbias, int accumulate, cudaStream_t st) {
  const int OH = H - KH + 1, OW = W - KW + 1;
  last_wgrad_kernel<<<(KH * KW * C + 255) / 256, 256, 0, st>>>(B, H, W, C, KH, KW, OH, OW, x, gout, gw, w_row, gbias, accumulate);
  return finish("skd_disc_last_wgrad");
}

extern "C" int skd_adv_loss(int n, const float* real, const float* fake, int type, float* loss, float* g_real, float* g_fake, cudaStream_t st) {
  adv_loss_kernel<<<1, 128, 0, st>>>(n, real, fake, type, loss, g_real, g_fake);
  return finish("skd_adv_loss");
}

extern "C" int skd_gp_norms(int B, long long len, const float* g, float lambda_gp, float* norms, float* loss, cudaStream_t st) {
  gp_norm_kernel<<<B, 1024, 0, st>>>(len, g, norms);
  gp_loss_kernel<<<1, 32, 0, st>>>(B, norms, lambda_gp, loss);
  return finish("skd_gp_norms", 2);
}

extern "C" int skd_gp_direction(int B, long long len, const float* g, const float* norms, float lambda_gp, const float* upstream, float* v,
                                cudaStream_t st) {
  int bx = blocks_for(len); if (bx > 64) bx = 64;
  gp_direction_kernel<<<dim3(bx, B), 256, 0, st>>>(B, len, g, norms, lambda_gp, upstream, v);
  return finish("skd_gp_direction");
}

extern "C" void skd_set_attn_tensor_cores(int on) { g_attn_tc = on ? 1 : 0; }

extern "C" void skd_set_attn_tiled(int force) { g_attn_tiled = force ? 1 : 0; }

extern "C" int skd_attn_fwd(int B, int n, int C, int d, const float* qkv, int ldq, const float* x, const float* gamma, float* attn, float* o,
                            float* y, float* y_lo, cudaStream_t st) {
  const char* who = "skd_attn_fwd";
  if (!attn_shape_ok(B, n, C, d, ldq, who)) return 0;
  const size_t bytes = ((size_t)n * (n + 1) + 2 * (size_t)n * (d + 1) + (size_t)n * (kAttnFwdSlice + 1)) * 4;
  if (attn_use_tiled(n, bytes)) {
    const int R = attn_stripe_rows([&](int r) { return attn_fwd_tiled_floats(r, n, d, false); });
    const size_t tb = attn_fwd_tiled_floats(R, n, d, false) * 4;
    if (!set_smem(attn_fwd_tiled_kernel, tb, who)) return 0;
    attn_fwd_tiled_kernel<<<dim3(B, (n + R - 1) / R, (C + kAttnFwdSlice - 1) / kAttnFwdSlice), 256, tb, st>>>(
        n, C, d, R, qkv, ldq, x, gamma, attn, o, y, y_lo, g_attn_tc);
    return finish(who);
  }
  if (!set_smem(attn_fwd_kernel, bytes, who)) return 0;
  attn_fwd_kernel<<<dim3(B, (C + kAttnFwdSlice - 1) / kAttnFwdSlice), 256, bytes, st>>>(n, C, d, qkv, ldq, x, gamma, attn, o, y, y_lo, g_attn_tc);
  return finish(who);
}

extern "C" int skd_attn_tangent_fwd(int B, int n, int C, int d, const float* qkv, const float* tqkv, int ldq, const float* attn,
                                    const float* tx, const float* gamma, float* dattn, float* to, float* ty, float* ty_lo, cudaStream_t st) {
  const char* who = "skd_attn_tangent_fwd";
  if (!attn_shape_ok(B, n, C, d, ldq, who)) return 0;
  size_t region = 4 * (size_t)n * (d + 1), need = 2 * (size_t)n * (kAttnFwdSlice + 1);
  if (region < need) region = need;
  const size_t bytes = (2 * (size_t)n * (n + 1) + region) * 4;
  if (attn_use_tiled(n, bytes)) {
    const int R = attn_stripe_rows([&](int r) { return attn_fwd_tiled_floats(r, n, d, true); });
    const size_t tb = attn_fwd_tiled_floats(R, n, d, true) * 4;
    if (!set_smem(attn_tangent_tiled_kernel, tb, who)) return 0;
    attn_tangent_tiled_kernel<<<dim3(B, (n + R - 1) / R, (C + kAttnFwdSlice - 1) / kAttnFwdSlice), 256, tb, st>>>(
        n, C, d, R, qkv, tqkv, ldq, attn, tx, gamma, dattn, to, ty, ty_lo, g_attn_tc);
    return finish(who);
  }
  if (!set_smem(attn_tangent_kernel, bytes, who)) return 0;
  attn_tangent_kernel<<<dim3(B, (C + kAttnFwdSlice - 1) / kAttnFwdSlice), 256, bytes, st>>>(n, C, d, qkv, tqkv, ldq, attn, tx, gamma, dattn, to, ty, ty_lo, g_attn_tc);
  return finish(who);
}

// The row-stripe backward: Sbar, St^ [B][n][n] and per-row ggamma partials.  For n <= 128 the larger of both paths' sizes: which
// path runs there also depends on d, the mode (first order / joint) and skd_set_attn_tiled.
extern "C" long long skd_attn_bwd_workspace_floats(int B, int n, int C) {
  const long long tiled = 2LL * B * n * n + (long long)B * n;
  if (n > kAttnMaxN) return tiled;
  const long long nsl = (C + kAttnBwdSlice - 1) / kAttnBwdSlice;
  const long long whole = (long long)B * nsl * 2 * n * n + (long long)B * nsl;
  return whole > tiled ? whole : tiled;
}

extern "C" int skd_attn_bwd(int B, int n, int C, int d, const float* qkv, int ldq, const float* attn, const float* o, const float* gamma,
                            const float* gy, const float* tqkv, const float* dattn, const float* to, const float* gty, float* gqkv,
                            float* gtqkv, float* ggamma, int accumulate, float* workspace, cudaStream_t st) {
  const char* who = "skd_attn_bwd";
  if (!attn_shape_ok(B, n, C, d, ldq, who)) return 0;
  const bool dual = gty != nullptr;
  if (dual && !(tqkv && dattn && to && gtqkv)) { set_error_msg(who, "the joint backward needs tqkv, dattn, to and gtqkv"); return 0; }
  const size_t b1 = ((dual ? 2 : 1) * (size_t)n * (n + 1) + (dual ? 4 : 2) * (size_t)n * (kAttnBwdSlice + 1)) * 4;
  const size_t b2 = ((dual ? 2 : 1) * (size_t)n * (n + 1) + (dual ? 4 : 2) * (size_t)n * (d + 1)) * 4;
  if (attn_use_tiled(n, b1 > b2 ? b1 : b2)) {
    const size_t nn = (size_t)B * n * n;
    float *sbar = workspace, *stbar = workspace + nn, *gpart = workspace + 2 * nn;
    const int R = attn_stripe_rows([&](int r) { return attn_bwd_rows_floats(r, n, d, dual); });
    const size_t rb = attn_bwd_rows_floats(R, n, d, dual) * 4;
    const dim3 g1(B, (n + R - 1) / R), g2(B, (n + kAttnKeyRows - 1) / kAttnKeyRows, 1 + (C + kAttnFwdSlice - 1) / kAttnFwdSlice);
    if (dual) {
      if (!set_smem(attn_bwd_rows_kernel<true>, rb, who) || !set_smem(attn_bwd_keys_kernel<true>, kAttnKeysBytes, who)) return 0;
      attn_bwd_rows_kernel<true><<<g1, 256, rb, st>>>(n, C, d, R, qkv, tqkv, ldq, attn, o, to, gamma, gy, gty, gqkv, gtqkv, sbar, stbar, gpart, g_attn_tc);
      attn_bwd_keys_kernel<true><<<g2, 256, kAttnKeysBytes, st>>>(B, n, C, d, qkv, tqkv, ldq, attn, dattn, gamma, gy, gty, sbar, stbar, gpart, gqkv,
                                                                  gtqkv, ggamma, accumulate, g_attn_tc);
    } else {
      if (!set_smem(attn_bwd_rows_kernel<false>, rb, who) || !set_smem(attn_bwd_keys_kernel<false>, kAttnKeysBytes, who)) return 0;
      attn_bwd_rows_kernel<false><<<g1, 256, rb, st>>>(n, C, d, R, qkv, nullptr, ldq, attn, o, nullptr, gamma, gy, nullptr, gqkv, nullptr, sbar, nullptr,
                                                       gpart, g_attn_tc);
      attn_bwd_keys_kernel<false><<<g2, 256, kAttnKeysBytes, st>>>(B, n, C, d, qkv, nullptr, ldq, attn, nullptr, gamma, gy, nullptr, sbar, nullptr, gpart,
                                                                   gqkv, nullptr, ggamma, accumulate, g_attn_tc);
    }
    return finish(who, 2);
  }
  const int nsl = (C + kAttnBwdSlice - 1) / kAttnBwdSlice;
  float* gpart = workspace + (size_t)B * nsl * 2 * n * n;
  if (dual) {
    if (!set_smem(attn_bwd1_kernel<true>, b1, who) || !set_smem(attn_bwd2_kernel<true>, b2, who)) return 0;
    attn_bwd1_kernel<true><<<dim3(B, nsl), 256, b1, st>>>(n, C, d, qkv, tqkv, ldq, attn, dattn, o, to, gamma, gy, gty, gqkv, gtqkv, workspace, gpart, g_attn_tc);
    attn_bwd2_kernel<true><<<B, 256, b2, st>>>(B, n, d, nsl, qkv, tqkv, ldq, attn, workspace, gpart, gqkv, gtqkv, ggamma, accumulate, g_attn_tc);
  } else {
    if (!set_smem(attn_bwd1_kernel<false>, b1, who) || !set_smem(attn_bwd2_kernel<false>, b2, who)) return 0;
    attn_bwd1_kernel<false><<<dim3(B, nsl), 256, b1, st>>>(n, C, d, qkv, nullptr, ldq, attn, nullptr, o, nullptr, gamma, gy, nullptr, gqkv, nullptr, workspace, gpart, g_attn_tc);
    attn_bwd2_kernel<false><<<B, 256, b2, st>>>(B, n, d, nsl, qkv, nullptr, ldq, attn, workspace, gpart, gqkv, nullptr, ggamma, accumulate, g_attn_tc);
  }
  return finish(who, 2);
}
