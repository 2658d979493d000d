// Feature-level distillation baselines for sm_90a (HBM-bound SIMT passes, no tensor cores):
//   * attention transfer (AT, Zagoruyko & Komodakis): q = mean_c(a_c^2) per pixel, q^ = q / max(||q||_2, 1e-12) per sample,
//     L = mean over N*H*W of (q^_S - q^_T)^2 -- the authors' at(x) = F.normalize(x.pow(2).mean(1).view(N, -1));
//   * MIMIC (Li et al.): L = mean of (r - f_T)^2 over the adapter output r, F.mse_loss.
// Feature maps are fp32 NHWC rows of C channels at a row pitch (the teacher's x4 is a channel slice of the PSP concat buffer), read in
// float4 groups when C, the pitch and the base are 16-byte aligned.  Every reduction runs in a fixed order (warp butterflies, per-block
// partials summed by one block) with no atomics, so two calls give bit-identical results.
#include "common.cuh"
#include "skd.h"

using namespace skd;

namespace {

constexpr float kNormEps = 1e-12f;    // F.normalize's eps
constexpr int kRedThreads = 1024;

__host__ __device__ inline bool vec4_ok(const void* p, int C, int ld) {
  return C % 4 == 0 && ld % 4 == 0 && (reinterpret_cast<uintptr_t>(p) & 15) == 0;
}

__device__ __forceinline__ double block_sum_double(double v, double* sh) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += sh[i];   // every thread, same order
  return t;
}

// q[i] = mean_c a[i][c]^2, one warp per pixel row; blockIdx.y selects the student (0) or the teacher (1) map
__global__ void __launch_bounds__(256)
at_map_kernel(long long P, const float* __restrict__ S, int CS, int lds, int vs, const float* __restrict__ T, int CT, int ldt, int vt,
              float* __restrict__ q) {
  const bool teacher = blockIdx.y == 1;
  const float* a = teacher ? T : S;
  const int C = teacher ? CT : CS, ld = teacher ? ldt : lds;
  const bool vec = teacher ? vt : vs;
  float* out = q + (teacher ? P : 0);
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long i = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); i < P; i += warps) {
    const float* row = a + i * ld;
    float s = 0.f;
    if (vec) {
      const float4* r4 = reinterpret_cast<const float4*>(row);
      for (int j = lane; j < C / 4; j += 32) {
        const float4 v = ld_stream(r4 + j);
        s = fmaf(v.x, v.x, s); s = fmaf(v.y, v.y, s); s = fmaf(v.z, v.z, s); s = fmaf(v.w, v.w, s);
      }
    } else {
      for (int c = lane; c < C; c += 32) { const float v = __ldg(row + c); s = fmaf(v, v, s); }
    }
    s = warp_sum(s);
    if (lane == 0) out[i] = s / (float)C;
  }
}

// per (sample, map): norm = ||q||_2 (double sum), q^ = q / max(norm, eps) in place
__global__ void __launch_bounds__(kRedThreads)
at_norm_kernel(int N, int HW, float* __restrict__ q, float* __restrict__ norms) {
  __shared__ double sh[32];
  const int n = blockIdx.x, t = blockIdx.y;
  float* row = q + ((long long)t * N + n) * HW;
  double acc = 0.0;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) { const double v = row[p]; acc += v * v; }
  const float norm = (float)sqrt(block_sum_double(acc, sh));
  const float d = fmaxf(norm, kNormEps);
  for (int p = threadIdx.x; p < HW; p += blockDim.x) row[p] = row[p] / d;
  if (threadIdx.x == 0) norms[t * N + n] = norm;
}

// loss = sum (q^_S - q^_T)^2 / (N * HW), one block
__global__ void __launch_bounds__(kRedThreads)
at_loss_kernel(long long P, const float* __restrict__ qhat, float* __restrict__ loss) {
  __shared__ double sh[32];
  double acc = 0.0;
  for (long long i = threadIdx.x; i < P; i += blockDim.x) { const float d = qhat[i] - qhat[P + i]; acc += (double)d * d; }
  const double s = block_sum_double(acc, sh);
  if (threadIdx.x == 0) loss[0] = (float)(s / (double)P);
}

// per sample: h = 2 (q^_S - q^_T) / (N * HW) * dL and g = (h - q^_S <q^_S, h>) / ||q_S|| -- or h / eps where the norm is clamped, whose
// gradient F.normalize's clamp_min stops
__global__ void __launch_bounds__(kRedThreads)
at_bwd_g_kernel(int N, int HW, const float* __restrict__ qhat, const float* __restrict__ norms, const float* __restrict__ gout,
                float* __restrict__ g) {
  __shared__ double sh[32];
  const int n = blockIdx.x;
  const long long P = (long long)N * HW;
  const float* qs = qhat + (long long)n * HW;
  const float* qt = qhat + P + (long long)n * HW;
  const float coef = 2.f * __ldg(gout) / (float)P;
  const float norm = norms[n];
  float* gr = g + (long long)n * HW;
  if (norm < kNormEps) {
    for (int p = threadIdx.x; p < HW; p += blockDim.x) gr[p] = coef * (qs[p] - qt[p]) / kNormEps;
    return;
  }
  double acc = 0.0;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) acc += (double)qs[p] * (double)(coef * (qs[p] - qt[p]));
  const float dot = (float)block_sum_double(acc, sh);
  for (int p = threadIdx.x; p < HW; p += blockDim.x) gr[p] = (coef * (qs[p] - qt[p]) - qs[p] * dot) / norm;
}

// dA[i][c] = (2 / C) a[i][c] g[i], one thread per channel group
__global__ void __launch_bounds__(256)
at_bwd_dx_kernel(long long P, int C, const float* __restrict__ a, int lda, const float* __restrict__ g, float* __restrict__ da, int ldd,
                 int vec) {
  const float k = 2.f / (float)C;
  const int G = vec ? C / 4 : C;
  const long long total = P * G;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long i = e / G;
    const int j = (int)(e - i * G);
    const float s = k * __ldg(g + i);
    if (vec) {
      const float4 v = ld_stream(reinterpret_cast<const float4*>(a + i * lda) + j);
      reinterpret_cast<float4*>(da + i * ldd)[j] = make_float4(v.x * s, v.y * s, v.z * s, v.w * s);
    } else {
      da[i * ldd + j] = __ldg(a + i * lda + j) * s;
    }
  }
}

// per-block partial sums of (r - t)^2
__global__ void __launch_bounds__(256)
mse_partial_kernel(long long P, int C, const float* __restrict__ r, int ldr, const float* __restrict__ t, int ldt, int vec,
                   double* __restrict__ part) {
  __shared__ double sh[32];
  const int G = vec ? C / 4 : C;
  const long long total = P * G;
  double acc = 0.0;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long i = e / G;
    const int j = (int)(e - i * G);
    if (vec) {
      const float4 a = ld_stream(reinterpret_cast<const float4*>(r + i * ldr) + j);
      const float4 b = ld_stream(reinterpret_cast<const float4*>(t + i * ldt) + j);
      const float dx = a.x - b.x, dy = a.y - b.y, dz = a.z - b.z, dw = a.w - b.w;
      acc += (double)(dx * dx) + (double)(dy * dy) + (double)(dz * dz) + (double)(dw * dw);
    } else {
      const float d = __ldg(r + i * ldr + j) - __ldg(t + i * ldt + j);
      acc += (double)(d * d);
    }
  }
  const double s = block_sum_double(acc, sh);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}

__global__ void __launch_bounds__(kRedThreads)
mse_finalize_kernel(const double* __restrict__ part, int n, double inv_numel, float* __restrict__ loss) {
  __shared__ double sh[32];
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) acc += part[i];
  const double s = block_sum_double(acc, sh);
  if (threadIdx.x == 0) loss[0] = (float)(s * inv_numel);
}

// dR = 2 (r - t) / numel * dL
__global__ void __launch_bounds__(256)
mse_bwd_kernel(long long P, int C, const float* __restrict__ r, int ldr, const float* __restrict__ t, int ldt, const float* __restrict__ gout,
               float inv_numel, float* __restrict__ dr, int ldd, int vec) {
  const float k = 2.f * __ldg(gout) * inv_numel;
  const int G = vec ? C / 4 : C;
  const long long total = P * G;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long i = e / G;
    const int j = (int)(e - i * G);
    if (vec) {
      const float4 a = ld_stream(reinterpret_cast<const float4*>(r + i * ldr) + j);
      const float4 b = ld_stream(reinterpret_cast<const float4*>(t + i * ldt) + j);
      reinterpret_cast<float4*>(dr + i * ldd)[j] = make_float4((a.x - b.x) * k, (a.y - b.y) * k, (a.z - b.z) * k, (a.w - b.w) * k);
    } else {
      dr[i * ldd + j] = (__ldg(r + i * ldr + j) - __ldg(t + i * ldt + j)) * k;
    }
  }
}

int grid_for(long long work, int per_block) {
  long long b = (work + per_block - 1) / per_block;
  if (b > kNumSMs * 4) b = kNumSMs * 4;
  return b < 1 ? 1 : (int)b;
}

bool check_rows(const char* who, long long P, int C, int ld) {
  if (P < 1 || C < 1 || ld < C) { set_error_msg(who, "empty map or row pitch smaller than the channel count"); return false; }
  return true;
}

}  // namespace

extern "C" int skd_at_fwd(int N, int HW, int CS, const float* S, int lds, int CT, const float* T, int ldt, float* qhat, float* norms,
                          float* loss, cudaStream_t st) {
  const long long P = (long long)N * HW;
  if (!check_rows("skd_at_fwd", P, CS, lds) || !check_rows("skd_at_fwd", P, CT, ldt)) return 0;
  at_map_kernel<<<dim3(grid_for(P, 8), 2), 256, 0, st>>>(P, S, CS, lds, vec4_ok(S, CS, lds), T, CT, ldt, vec4_ok(T, CT, ldt), qhat);
  at_norm_kernel<<<dim3(N, 2), kRedThreads, 0, st>>>(N, HW, qhat, norms);
  at_loss_kernel<<<1, kRedThreads, 0, st>>>(P, qhat, loss);
  return finish("skd_at_fwd", 3);
}

extern "C" int skd_at_bwd(int N, int HW, int C, const float* S, int lds, const float* qhat, const float* norms, const float* grad_out,
                          float* g, float* dS, int ldd, cudaStream_t st) {
  const long long P = (long long)N * HW;
  if (!check_rows("skd_at_bwd", P, C, lds) || !check_rows("skd_at_bwd", P, C, ldd)) return 0;
  const int vec = vec4_ok(S, C, lds) && vec4_ok(dS, C, ldd);
  at_bwd_g_kernel<<<N, kRedThreads, 0, st>>>(N, HW, qhat, norms, grad_out, g);
  at_bwd_dx_kernel<<<grid_for(P * (vec ? C / 4 : C), 256), 256, 0, st>>>(P, C, S, lds, g, dS, ldd, vec);
  return finish("skd_at_bwd", 2);
}

extern "C" int skd_mse_fwd(long long P, int C, const float* R, int ldr, const float* T, int ldt, float* loss, double* workspace,
                           cudaStream_t st) {
  if (!check_rows("skd_mse_fwd", P, C, ldr) || !check_rows("skd_mse_fwd", P, C, ldt)) return 0;
  const int vec = vec4_ok(R, C, ldr) && vec4_ok(T, C, ldt);
  const int blocks = grid_for(P * (vec ? C / 4 : C), 256);
  mse_partial_kernel<<<blocks, 256, 0, st>>>(P, C, R, ldr, T, ldt, vec, workspace);
  mse_finalize_kernel<<<1, kRedThreads, 0, st>>>(workspace, blocks, 1.0 / ((double)P * C), loss);
  return finish("skd_mse_fwd", 2);
}

extern "C" int skd_mse_bwd(long long P, int C, const float* R, int ldr, const float* T, int ldt, const float* grad_out, float* dR,
                           int ldd, cudaStream_t st) {
  if (!check_rows("skd_mse_bwd", P, C, ldr) || !check_rows("skd_mse_bwd", P, C, ldt) || !check_rows("skd_mse_bwd", P, C, ldd)) return 0;
  const int vec = vec4_ok(R, C, ldr) && vec4_ok(T, C, ldt) && vec4_ok(dR, C, ldd);
  mse_bwd_kernel<<<grid_for(P * (vec ? C / 4 : C), 256), 256, 0, st>>>(P, C, R, ldr, T, ldt, grad_out,
                                                                       (float)(1.0 / ((double)P * C)), dR, ldd, vec);
  return finish("skd_mse_bwd");
}
