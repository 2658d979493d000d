// Channel-wise distillation (CWD, Shu et al., ICCV 2021) for sm_90a (HBM-bound SIMT passes, no tensor cores):
//   p_{n,c,i} = softmax over the H*W positions i of x_{n,c,i} / tau, for the student map S and the (frozen) teacher map T,
//   L = tau^2 / (N*C) * sum_{n,c,i} pT (log pT - log pS),   dL/dS = tau / (N*C) * (pS - pT) * dL_out.
// The log-probabilities are z - lse(z), z = x / tau, with lse taken max-subtracted, so a pS that underflows to 0 still has a finite
// log (softmax(...).log() would give -inf there and inf / NaN in the loss).
//
// Maps come as (image, channel, pixel) strides, so NCHW logits, NHWC logits at a pitch and NHWC feature rows (channel slices of a
// concat buffer included) all run in place.  Three thread mappings, chosen from the strides:
//   CH   channels contiguous: lanes over 32 channels, the 8 warps over pixel stripes;
//   CH4  the same with float4 channel groups (C, the pitches and the bases 16-byte aligned): lanes over 128 channels;
//   PX   anything else (NCHW: pixels contiguous): lanes over pixel stripes, the 8 warps over 8 channels.
// CH and CH4 give every channel the same pixel order and the same stripe reduction, so alignment never changes a bit of the result.
// Forward: (1) per (map, n, c, chunk) the pair (max z, sum exp(z - max)) -- online, the sum in double; (2) the pairs of each
// (map, n, c) combined over chunks in order into lse, kept for the backward; (3) per (n, c, chunk) the KL sum in double; (4) one block
// sums those in a fixed order.  Each map is read twice, the backward reads S and T once and writes dS once; no probability map is
// stored.  z = x / tau is one rounded product (never fused into the subtraction of lse), so HW = 1 or S = T give exactly 0.
// The pixel chunking depends on (N, C, HW) only, nothing is atomic: two calls give bit-identical results.
#include <cmath>

#include "common.cuh"
#include "skd.h"

using namespace skd;

namespace {

constexpr int kThreads = 256;
constexpr int kFinThreads = 1024;
constexpr int kMinChunk = 64;                 // pixels per chunk at least
constexpr long long kTargetCtas = 8LL * kNumSMs;

enum Mode { CH = 0, CH4 = 1, PX = 2 };
template <int M> struct Map;
template <> struct Map<CH>  { static constexpr int kTileC = 32,  kStripes = 8,  kVpt = 1; };
template <> struct Map<CH4> { static constexpr int kTileC = 128, kStripes = 8,  kVpt = 4; };
template <> struct Map<PX>  { static constexpr int kTileC = 8,   kStripes = 32, kVpt = 1; };

struct Strides { long long n, c, p; };
struct Plan { int N, C, HW, chunks, len; };   // chunk k covers pixels [k * len, min((k + 1) * len, HW))

Plan make_plan(int N, int C, int HW) {
  const long long tiles = (long long)N * ((C + 31) / 32);
  long long k = (kTargetCtas + tiles - 1) / tiles;
  const long long kmax = (HW + kMinChunk - 1) / kMinChunk;
  if (k > kmax) k = kmax;
  if (k < 1) k = 1;
  const int len = (int)((HW + k - 1) / k);
  return Plan{N, C, HW, (HW + len - 1) / len, len};
}

// this thread's channel slot and pixel stripe
template <int M> __device__ __forceinline__ int slot() { return M == PX ? (threadIdx.x >> 5) : (threadIdx.x & 31); }
template <int M> __device__ __forceinline__ int stripe() { return M == PX ? (threadIdx.x & 31) : (threadIdx.x >> 5); }

// the kVpt values of channels c .. c + kVpt - 1 at pixel p
template <int M>
__device__ __forceinline__ void load(const float* __restrict__ base, Strides s, int c, long long p, float* v) {
  const float* a = base + c * s.c + p * s.p;
  if constexpr (M == CH4) {
    const float4 q = __ldg(reinterpret_cast<const float4*>(a));
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
  } else {
    v[0] = __ldg(a);
  }
}

// (m, s) <- the pair of {m, s} and {m2, s2}; an empty pair (s = 0) changes nothing
__device__ __forceinline__ void combine(double& m, double& s, double m2, double s2) {
  if (s2 == 0.0) return;
  if (m2 > m) { s = s * exp(m - m2) + s2; m = m2; }
  else        { s += s2 * exp(m2 - m); }
}

// (1): blockIdx = (chunk, channel tile, map * N + n); part[map][n][chunk][C] = (max z, sum exp(z - max)) over the chunk
template <int M>
__global__ void __launch_bounds__(kThreads)
cwd_stats_kernel(Plan pl, const float* __restrict__ S, Strides ss, const float* __restrict__ T, Strides ts, double invtau,
                 double2* __restrict__ part) {
  using G = Map<M>;
  __shared__ double2 sh[G::kStripes][G::kTileC];
  const int map = blockIdx.z / pl.N, n = blockIdx.z - map * pl.N;
  const float* x = (map ? T : S) + n * (map ? ts.n : ss.n);
  const Strides st = map ? ts : ss;
  const int c0 = blockIdx.y * G::kTileC + slot<M>() * G::kVpt;
  const long long p0 = (long long)blockIdx.x * pl.len, p1 = min(p0 + pl.len, (long long)pl.HW);
  double m[G::kVpt], s[G::kVpt];
#pragma unroll
  for (int v = 0; v < G::kVpt; ++v) { m[v] = -INFINITY; s[v] = 0.0; }
  if (c0 < pl.C) {
#pragma unroll 2
    for (long long p = p0 + stripe<M>(); p < p1; p += G::kStripes) {
      float a[G::kVpt];
      load<M>(x, st, c0, p, a);
#pragma unroll
      for (int v = 0; v < G::kVpt; ++v) {
        const double z = __dmul_rn((double)a[v], invtau);
        if (z > m[v]) { s[v] = s[v] * (double)expf((float)(m[v] - z)) + 1.0; m[v] = z; }
        else          { s[v] += (double)expf((float)(z - m[v])); }
      }
    }
  }
#pragma unroll
  for (int v = 0; v < G::kVpt; ++v) sh[stripe<M>()][slot<M>() * G::kVpt + v] = make_double2(m[v], s[v]);
  __syncthreads();
  const int c = blockIdx.y * G::kTileC + threadIdx.x;
  if (threadIdx.x < G::kTileC && c < pl.C) {
    double mm = -INFINITY, ss2 = 0.0;
    for (int k = 0; k < G::kStripes; ++k) combine(mm, ss2, sh[k][threadIdx.x].x, sh[k][threadIdx.x].y);
    part[(((long long)map * pl.N + n) * pl.chunks + blockIdx.x) * pl.C + c] = make_double2(mm, ss2);
  }
}

// (2): lse[map][n][c] = max + log(sum), the chunks combined in order
__global__ void __launch_bounds__(kThreads)
cwd_lse_kernel(Plan pl, const double2* __restrict__ part, double* __restrict__ lse) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // (map * N + n) * C + c
  if (i >= 2LL * pl.N * pl.C) return;
  const long long mn = i / pl.C, c = i - mn * pl.C;
  const double2* q = part + mn * pl.chunks * pl.C + c;
  double m = -INFINITY, s = 0.0;
  for (int k = 0; k < pl.chunks; ++k) combine(m, s, q[(long long)k * pl.C].x, q[(long long)k * pl.C].y);
  lse[i] = m + log(s);
}

// (3): blockIdx = (chunk, channel tile, n); kl[n][chunk][C] = sum over the chunk of pT (log pT - log pS), terms with pT = 0 giving 0
template <int M>
__global__ void __launch_bounds__(kThreads)
cwd_kl_kernel(Plan pl, const float* __restrict__ S, Strides ss, const float* __restrict__ T, Strides ts, double invtau,
              const double* __restrict__ lse, double* __restrict__ kl) {
  using G = Map<M>;
  __shared__ double sh[G::kStripes][G::kTileC];
  const int n = blockIdx.z;
  const float* xs = S + n * ss.n;
  const float* xt = T + n * ts.n;
  const int c0 = blockIdx.y * G::kTileC + slot<M>() * G::kVpt;
  const long long p0 = (long long)blockIdx.x * pl.len, p1 = min(p0 + pl.len, (long long)pl.HW);
  double acc[G::kVpt];
#pragma unroll
  for (int v = 0; v < G::kVpt; ++v) acc[v] = 0.0;
  if (c0 < pl.C) {
    double ls[G::kVpt], lt[G::kVpt];
#pragma unroll
    for (int v = 0; v < G::kVpt; ++v) {
      ls[v] = lse[(long long)n * pl.C + c0 + v];
      lt[v] = lse[((long long)pl.N + n) * pl.C + c0 + v];
    }
#pragma unroll 4
    for (long long p = p0 + stripe<M>(); p < p1; p += G::kStripes) {
      float a[G::kVpt], b[G::kVpt];
      load<M>(xs, ss, c0, p, a);
      load<M>(xt, ts, c0, p, b);
#pragma unroll
      for (int v = 0; v < G::kVpt; ++v) {
        const double qs = __dmul_rn((double)a[v], invtau) - ls[v], qt = __dmul_rn((double)b[v], invtau) - lt[v];
        const double pt = (double)expf((float)qt);
        acc[v] += pt > 0.0 ? pt * (qt - qs) : 0.0;
      }
    }
  }
#pragma unroll
  for (int v = 0; v < G::kVpt; ++v) sh[stripe<M>()][slot<M>() * G::kVpt + v] = acc[v];
  __syncthreads();
  const int c = blockIdx.y * G::kTileC + threadIdx.x;
  if (threadIdx.x < G::kTileC && c < pl.C) {
    double t = 0.0;
    for (int k = 0; k < G::kStripes; ++k) t += sh[k][threadIdx.x];
    kl[((long long)n * pl.chunks + blockIdx.x) * pl.C + c] = t;
  }
}

// (4): loss = scale * sum of the n partials, one block: thread t sums t, t + 1024, ..., then a fixed butterfly and warp order
__global__ void __launch_bounds__(kFinThreads)
cwd_loss_kernel(const double* __restrict__ kl, long long n, double scale, float* __restrict__ loss) {
  __shared__ double sh[32];
  double acc = 0.0;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) acc += kl[i];
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < kFinThreads / 32; ++i) t += sh[i];
    loss[0] = (float)(t * scale);
  }
}

// backward: dS = tau / (N*C) * dL_out * (pS - pT), pS and pT recomputed from the maps and lse
template <int M>
__global__ void __launch_bounds__(kThreads)
cwd_bwd_kernel(Plan pl, const float* __restrict__ S, Strides ss, const float* __restrict__ T, Strides ts, double invtau,
               const double* __restrict__ lse, const float* __restrict__ gout, float coef, float* __restrict__ dS, Strides ds) {
  using G = Map<M>;
  const int n = blockIdx.z;
  const int c0 = blockIdx.y * G::kTileC + slot<M>() * G::kVpt;
  if (c0 >= pl.C) return;
  const float* xs = S + n * ss.n;
  const float* xt = T + n * ts.n;
  float* d = dS + n * ds.n + c0 * ds.c;
  const float k = coef * __ldg(gout);
  double ls[G::kVpt], lt[G::kVpt];
#pragma unroll
  for (int v = 0; v < G::kVpt; ++v) {
    ls[v] = lse[(long long)n * pl.C + c0 + v];
    lt[v] = lse[((long long)pl.N + n) * pl.C + c0 + v];
  }
  const long long p0 = (long long)blockIdx.x * pl.len, p1 = min(p0 + pl.len, (long long)pl.HW);
#pragma unroll 4
  for (long long p = p0 + stripe<M>(); p < p1; p += G::kStripes) {
    float a[G::kVpt], b[G::kVpt], r[G::kVpt];
    load<M>(xs, ss, c0, p, a);
    load<M>(xt, ts, c0, p, b);
#pragma unroll
    for (int v = 0; v < G::kVpt; ++v)
      r[v] = k * (expf((float)(__dmul_rn((double)a[v], invtau) - ls[v])) - expf((float)(__dmul_rn((double)b[v], invtau) - lt[v])));
    if constexpr (M == CH4) reinterpret_cast<float4*>(d + p * ds.p)[0] = make_float4(r[0], r[1], r[2], r[3]);
    else d[p * ds.p] = r[0];
  }
}

bool aligned4(const void* p, Strides s) {
  return (reinterpret_cast<uintptr_t>(p) & 15) == 0 && s.n % 4 == 0 && s.p % 4 == 0;
}

// CH when every map has contiguous channels (C > 1), CH4 when they are float4-aligned too, else PX
int pick_mode(int C, const void* a, Strides sa, const void* b, Strides sb, const void* c = nullptr, Strides sc = Strides{0, 1, 0}) {
  if (C == 1 || sa.c != 1 || sb.c != 1 || sc.c != 1) return PX;
  return C % 4 == 0 && aligned4(a, sa) && aligned4(b, sb) && (c == nullptr || aligned4(c, sc)) ? CH4 : CH;
}

int tile_c(int mode) { return mode == CH4 ? Map<CH4>::kTileC : mode == CH ? Map<CH>::kTileC : Map<PX>::kTileC; }

bool check(const char* who, int N, int C, int HW, float tau) {
  if (N < 1 || C < 1 || HW < 1) { set_error_msg(who, "empty map"); return false; }
  if (2LL * N > 65535) { set_error_msg(who, "more than 32767 images"); return false; }
  if (!(tau > 0.f) || !std::isfinite(tau)) { set_error_msg(who, "the temperature must be finite and > 0"); return false; }
  return true;
}

}  // namespace

extern "C" long long skd_cwd_workspace(int N, int C, int HW) {
  if (N < 1 || C < 1 || HW < 1) return 0;
  return 4LL * N * make_plan(N, C, HW).chunks * C;
}

extern "C" int skd_cwd_fwd(int N, int C, int HW, const float* S, long long s_sn, long long s_sc, long long s_sp, const float* T,
                           long long t_sn, long long t_sc, long long t_sp, float tau, float* loss, double* lse, double* workspace,
                           cudaStream_t st) {
  if (!check("skd_cwd_fwd", N, C, HW, tau)) return 0;
  const Plan pl = make_plan(N, C, HW);
  const Strides ss{s_sn, s_sc, s_sp}, ts{t_sn, t_sc, t_sp};
  const double invtau = 1.0 / (double)tau;
  const int mode = pick_mode(C, S, ss, T, ts);
  const unsigned ct = (unsigned)((C + tile_c(mode) - 1) / tile_c(mode));
  double2* part = reinterpret_cast<double2*>(workspace);
  const dim3 gs(pl.chunks, ct, 2 * N), gk(pl.chunks, ct, N);
  if (mode == CH4) cwd_stats_kernel<CH4><<<gs, kThreads, 0, st>>>(pl, S, ss, T, ts, invtau, part);
  else if (mode == CH) cwd_stats_kernel<CH><<<gs, kThreads, 0, st>>>(pl, S, ss, T, ts, invtau, part);
  else cwd_stats_kernel<PX><<<gs, kThreads, 0, st>>>(pl, S, ss, T, ts, invtau, part);
  cwd_lse_kernel<<<(unsigned)((2LL * N * C + kThreads - 1) / kThreads), kThreads, 0, st>>>(pl, part, lse);
  if (mode == CH4) cwd_kl_kernel<CH4><<<gk, kThreads, 0, st>>>(pl, S, ss, T, ts, invtau, lse, workspace);
  else if (mode == CH) cwd_kl_kernel<CH><<<gk, kThreads, 0, st>>>(pl, S, ss, T, ts, invtau, lse, workspace);
  else cwd_kl_kernel<PX><<<gk, kThreads, 0, st>>>(pl, S, ss, T, ts, invtau, lse, workspace);
  cwd_loss_kernel<<<1, kFinThreads, 0, st>>>(workspace, (long long)N * pl.chunks * C, (double)tau * tau / ((double)N * C), loss);
  return finish("skd_cwd_fwd", 4);
}

extern "C" int skd_cwd_bwd(int N, int C, int HW, const float* S, long long s_sn, long long s_sc, long long s_sp, const float* T,
                           long long t_sn, long long t_sc, long long t_sp, float tau, const double* lse, const float* grad_out, float* dS,
                           long long d_sn, long long d_sc, long long d_sp, cudaStream_t st) {
  if (!check("skd_cwd_bwd", N, C, HW, tau)) return 0;
  const Plan pl = make_plan(N, C, HW);
  const Strides ss{s_sn, s_sc, s_sp}, ts{t_sn, t_sc, t_sp}, ds{d_sn, d_sc, d_sp};
  const double invtau = 1.0 / (double)tau;
  const int mode = pick_mode(C, S, ss, T, ts, dS, ds);
  const dim3 g(pl.chunks, (unsigned)((C + tile_c(mode) - 1) / tile_c(mode)), N);
  const float coef = (float)((double)tau / ((double)N * C));
  if (mode == CH4) cwd_bwd_kernel<CH4><<<g, kThreads, 0, st>>>(pl, S, ss, T, ts, invtau, lse, grad_out, coef, dS, ds);
  else if (mode == CH) cwd_bwd_kernel<CH><<<g, kThreads, 0, st>>>(pl, S, ss, T, ts, invtau, lse, grad_out, coef, dS, ds);
  else cwd_bwd_kernel<PX><<<g, kThreads, 0, st>>>(pl, S, ss, T, ts, invtau, lse, grad_out, coef, dS, ds);
  return finish("skd_cwd_bwd");
}
