// Pair-wise affinity loss at large node counts (pool_scale -> 1/65: 8 385 nodes per image) on wgmma.
//   utils/utils.py:173-183:  A = f^T f / (|f_m| |f_n|) per image,  loss = sum (A_T - A_S)^2 / nodes^2 / N
// Formulation: with X = [ fT*rT | fS*rS ] and W = [ fT*rT | -fS*rS ] (K = C_T + C_S) the difference matrix is ONE K-major
// GEMM  E = X W^T, so the tensor-core kernel of conv_sm100.cu is used as a plain NT GEMM (skd_gemm_nt_sm100) with the L2
// reduction (sum E^2) fused into its epilogue; E itself (2.25 GB at 8x8385^2) is written only when a backward will follow.
// Backward: dpooled_S = -4 g /(nodes^2 N) * rS_m * (E (fS*rS)) -- a second NT GEMM per image with E as the A operand.
#include "common.cuh"
#include "skd.h"

using namespace skd;

namespace {

__global__ void __launch_bounds__(256)
pa_concat_norm_kernel(const float* __restrict__ pS, const float* __restrict__ pT, const float* __restrict__ rS,
                      const float* __restrict__ rT, long long rows, int CS, int CT, float* __restrict__ X, float* __restrict__ Wn) {
  const int K = CS + CT;
  const long long total = rows * K;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / K; const int k = (int)(i - r * K);
    float v, w;
    if (k < CT) { v = __ldg(pT + r * CT + k) * __ldg(rT + r); w = v; }
    else { v = __ldg(pS + r * CS + (k - CT)) * __ldg(rS + r); w = -v; }
    X[i] = v; Wn[i] = w;
  }
}

// Bt[c][m] = pS[m][c] * rS[m]   (one image; pitch ld >= nodes, tail zero)
__global__ void __launch_bounds__(256)
pa_transpose_norm_kernel(const float* __restrict__ pS, const float* __restrict__ rS, int nodes, int CS, int ld, float* __restrict__ Bt) {
  __shared__ float tile[32][33];
  const int m0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int r = ty; r < 32; r += 8) {
    const int m = m0 + r, c = c0 + tx;
    tile[r][tx] = (m < nodes && c < CS) ? pS[(size_t)m * CS + c] * rS[m] : 0.f;
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const int c = c0 + r, m = m0 + tx;
    if (c < CS && m < ld) Bt[(size_t)c * ld + m] = tile[tx][r];
  }
}

__global__ void __launch_bounds__(256)
pa_scale_kernel(const float* __restrict__ G, const float* __restrict__ rS, long long rows, int CS, float coef_mul, const float* __restrict__ gout,
                float* __restrict__ dpooled) {
  const float coef = coef_mul * __ldg(gout);
  const long long total = rows * CS;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    dpooled[i] = coef * __ldg(rS + i / CS) * G[i];
}

__global__ void pa_finalize_kernel(const double* __restrict__ acc, double scale, float* __restrict__ loss) { loss[0] = (float)(acc[0] * scale); }

__global__ void __launch_bounds__(256) zero_pad_cols_kernel(float* __restrict__ E, long long rows, int nodes, int ld) {
  const int pad = ld - nodes;
  const long long total = rows * pad;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    E[(i / pad) * ld + nodes + (int)(i % pad)] = 0.f;
}

int blocks_for(long long n) { long long b = (n + 255) / 256; if (b > kNumSMs * 16) b = kNumSMs * 16; if (b < 1) b = 1; return (int)b; }

}  // namespace

extern "C" int skd_gemm_nt_sm100(int M, int Ncols, int K, const float* A, int lda, const float* B, float* D, int ldd, double* sumsq, cudaStream_t st);

extern "C" long long skd_pairwise_affinity_sm100_workspace_floats(int N, int nodes, int CS, int CT) {
  return 2LL * N * nodes * (CS + CT);
}

extern "C" int skd_pairwise_affinity_sm100(int N, int nodes, int CS, int CT, const float* pooled_S, const float* pooled_T,
                                           const float* rnorm_S, const float* rnorm_T, float* E, int ldE, float* loss,
                                           float* workspace, double* acc, cudaStream_t st) {
  const char* who = "skd_pairwise_affinity_sm100";
  const int K = CS + CT;
  if (K % 4 || (E && (ldE % 4 || ldE < nodes))) { set_error_msg(who, "C_S + C_T and the pitch of E must be multiples of 4"); return 0; }
  const long long rows = (long long)N * nodes;
  float* X = workspace; float* Wn = workspace + rows * K;
  if (cudaMemsetAsync(acc, 0, sizeof(double), st) != cudaSuccess) return finish(who);
  pa_concat_norm_kernel<<<blocks_for(rows * K), 256, 0, st>>>(pooled_S, pooled_T, rnorm_S, rnorm_T, rows, CS, CT, X, Wn);
  if (E && ldE > nodes) zero_pad_cols_kernel<<<blocks_for(rows * (ldE - nodes)), 256, 0, st>>>(E, rows, nodes, ldE);
  for (int n = 0; n < N; ++n) {
    const float* Xn = X + (size_t)n * nodes * K; const float* Wi = Wn + (size_t)n * nodes * K;
    if (!skd_gemm_nt_sm100(nodes, nodes, K, Xn, K, Wi, E ? E + (size_t)n * nodes * ldE : nullptr, ldE, acc, st)) return 0;
  }
  pa_finalize_kernel<<<1, 1, 0, st>>>(acc, 1.0 / ((double)nodes * (double)nodes) / (double)N, loss);
  return finish(who, 3);
}

extern "C" long long skd_pairwise_affinity_bwd_sm100_workspace_floats(int N, int nodes, int CS, int ldE) {
  return (long long)CS * ldE + (long long)N * nodes * CS;
}

extern "C" int skd_pairwise_affinity_bwd_sm100(int N, int nodes, int CS, const float* E, int ldE, const float* pooled_S,
                                               const float* rnorm_S, const float* grad_out, float* dpooled, float* workspace,
                                               cudaStream_t st) {
  const char* who = "skd_pairwise_affinity_bwd_sm100";
  if (CS % 4 || ldE % 4) { set_error_msg(who, "C_S and the pitch of E must be multiples of 4"); return 0; }
  float* Bt = workspace; float* G = workspace + (size_t)CS * ldE;
  for (int n = 0; n < N; ++n) {
    pa_transpose_norm_kernel<<<dim3((ldE + 31) / 32, (CS + 31) / 32), 256, 0, st>>>(pooled_S + (size_t)n * nodes * CS, rnorm_S + (size_t)n * nodes,
                                                                                  nodes, CS, ldE, Bt);
    if (!skd_gemm_nt_sm100(nodes, CS, ldE, E + (size_t)n * nodes * ldE, ldE, Bt, G + (size_t)n * nodes * CS, CS, nullptr, st)) return 0;
  }
  pa_scale_kernel<<<blocks_for((long long)N * nodes * CS), 256, 0, st>>>(G, rnorm_S, (long long)N * nodes, CS,
                                                                        -4.f / ((float)nodes * (float)nodes * (float)N), grad_out, dpooled);
  return finish(who, N + 1);
}
