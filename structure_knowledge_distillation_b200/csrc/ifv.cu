// Intra-class feature variation distillation (IFVD, Wang et al., ECCV 2020) for sm_90a (HBM-bound SIMT passes, no tensor cores).
// Per feature level, for the student map S (C_S channels) and the frozen teacher map T (C_T channels) on one h x w grid, with the
// step's labels taken down to that grid by torch's legacy nearest rule:
//   cnt[n,k] = #{i : lab_i = k},  P[n,k] = sum_{lab_i = k} f_i / (cnt[n,k] + 1e-6)          (separately for S and T)
//   cos_i = (f_i . P[n, lab_i]) / (max(|f_i|, eps) max(|P|, eps)),  eps = 1e-8               (torch's cosine_similarity)
//   L = 1 / (N h w) * sum over the pixels with a label in [0, K) of (cos_S,i - cos_T,i)^2   (other pixels add exactly 0)
// The gradient reaches S through its own cosine and through the prototypes (every pixel of class k feeds P_S[n,k]):
//   dS_i = a_i P_k - b_i f_i + Q_k / (cnt_k + 1e-6),   g_i = 2 (cos_S,i - cos_T,i) dL_out / (N h w),
//   a_i = g_i / (nf_i np_k),  b_i = g_i cos_i / (nf_i |f_i|),  nf = max(|f|, eps),  np = max(|P|, eps),
//   Q_k = A_k / np_k - P_k B_k / (np_k |P_k|),  A_k = sum_{lab_i = k} (g_i / nf_i) f_i,  B_k = sum_{lab_i = k} g_i cos_i.
//
// Passes.  Forward: the class sums of S and then of T (one kernel, w = 1) -> prototypes, counts and |P|^2 per class; one warp per pixel
// for both dot products and |f|^2 -> cos_S, d = cos_S - cos_T and |f_S| kept per pixel, sum d^2 in a fixed order.  Backward: the
// same class-sum kernel on S with the weights (g / nf, g cos) -> Q, then one elementwise pass.  Each map is read twice forward, S twice
// and dS written once backward; no per-pixel copy of a prototype is stored.
//
// Maps are NHWC rows at a pitch (channel slices of concat buffers included): (image, pixel) strides, channels contiguous.  Lane l of a
// warp always owns channels 4l .. 4l + 3 (+ 128 j); the float4 path (C % 4 == 0, bases and strides 16-byte aligned) only widens the
// loads, so it gives the bits of the scalar path.  The class sums accumulate in double in per-warp shared-memory rows, classes in
// groups of at most 12 (any K <= 255), per (n, pixel chunk, 128-channel tile); warps and chunks are combined in a fixed order.  Nothing
// is atomic and the chunking depends on the shape only: two calls give bit-identical results.
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "skd.h"

using namespace skd;

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kTileC = 128;                     // channels per class-sum block: 4 per lane
constexpr int kMaxGroup = 12;                   // classes per class-sum block: 12 * 8 warps * 128 doubles = 96 KB of shared memory
constexpr int kMinChunk = 256;                  // pixels per class-sum chunk at least
constexpr int kFinThreads = 128;
constexpr long long kTargetCtas = 8LL * kNumSMs;
constexpr int kPixBlocks = 16 * kNumSMs;        // warp-per-pixel passes: grid-stride over N * h * w
constexpr double kEps = 1e-8;                   // cosine_similarity's clamp of each norm
constexpr double kCntEps = 1e-6;                // IFVD's prototype denominator

struct Map { const float* x; long long sn, sp; int C; };
struct Plan { int N, HW, K, C, chunks, len, groups, kg; };   // chunk j covers pixels [j * len, min((j + 1) * len, HW))
struct Wts { const float* pix; const float* gout; double scale; long long nhw; };   // pix == nullptr: w = u = 1

Plan sum_plan(int N, int HW, int K, int C) {
  const int groups = (K + kMaxGroup - 1) / kMaxGroup, kg = (K + groups - 1) / groups;
  const long long tiles = (long long)N * ((C + kTileC - 1) / kTileC) * groups;
  long long k = (kTargetCtas + tiles - 1) / tiles;
  const long long kmax = (HW + kMinChunk - 1) / kMinChunk;
  if (k > kmax) k = kmax;
  if (k < 1) k = 1;
  const int len = (int)((HW + k - 1) / k);
  return Plan{N, HW, K, C, (HW + len - 1) / len, len, groups, kg};
}

size_t sum_smem(const Plan& pl) { return (size_t)pl.kg * kWarps * (kTileC + 1) * sizeof(double); }
// doubles of part + cpart, rounded up to 16 bytes so that what follows them is float4-aligned
long long part_doubles(const Plan& pl) { return ((long long)pl.N * pl.chunks * pl.K * ((long long)pl.C + 1) + 1) / 2 * 2; }
int pix_blocks(long long nhw) { return (int)std::min<long long>((nhw + kWarps - 1) / kWarps, kPixBlocks); }

// the 4 values of channels c .. c + 3 of row `a` (0 past C)
template <bool V4>
__device__ __forceinline__ void load4(const float* __restrict__ a, int c, int C, float* v) {
  if constexpr (V4) {
    if (c < C) {
      const float4 q = __ldg(reinterpret_cast<const float4*>(a + c));
      v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
    } else {
      v[0] = v[1] = v[2] = v[3] = 0.f;
    }
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = c + j < C ? __ldg(a + c + j) : 0.f;
  }
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// labels (N, H, W) int64 -> (N, h, w) int32 by F.interpolate(mode="nearest")'s rule: src = min(floor(dst * (float(in) / out)), in - 1),
// the product one fp32 rounding; labels outside the int32 range become -1 (ignored like any label outside [0, K))
__global__ void labels_nearest_kernel(int N, int H, int W, const long long* __restrict__ lab, int h, int w, float sy, float sx,
                                      int* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)N * h * w) return;
  const int x = (int)(i % w), y = (int)((i / w) % h), n = (int)(i / ((long long)w * h));
  const int ys = min((int)floorf(__fmul_rn((float)y, sy)), H - 1), xs = min((int)floorf(__fmul_rn((float)x, sx)), W - 1);
  const long long v = lab[((long long)n * H + ys) * W + xs];
  out[i] = (v < 0 || v > 0x7fffffffLL) ? -1 : (int)v;
}

// blockIdx = (chunk, channel tile, n * groups + group): per class k of the group and channel c of the tile, sum over the chunk's
// pixels of class k of w_i * f_i[c] -> part[n][chunk][k][C]; the tile-0 blocks also sum u_i -> cpart[n][chunk][k]
template <bool V4>
__global__ void __launch_bounds__(kThreads)
ifv_class_sum_kernel(Plan pl, const int* __restrict__ lab, Map m, Wts wt, double* __restrict__ part, double* __restrict__ cpart) {
  extern __shared__ double sh[];                      // [kg][kWarps][kTileC] feature sums, then [kWarps][kg] weight sums
  double* shc = sh + (size_t)pl.kg * kWarps * kTileC;
  const int chunk = blockIdx.x, tile = blockIdx.y, n = blockIdx.z / pl.groups, grp = blockIdx.z - n * pl.groups;
  const int k0 = grp * pl.kg, nk = min(pl.kg, pl.K - k0);
  for (int i = threadIdx.x; i < pl.kg * kWarps * (kTileC + 1); i += kThreads) sh[i] = 0.0;
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c0 = tile * kTileC + lane * 4;
  const bool counts = tile == 0 && lane == 0;
  const float* x = m.x + n * m.sn;
  const long long base = (long long)n * pl.HW;
  const double g0 = wt.pix != nullptr ? wt.scale * (double)__ldg(wt.gout) : 1.0;
  const long long p0 = (long long)chunk * pl.len, p1 = min(p0 + pl.len, (long long)pl.HW);
#pragma unroll 2
  for (long long p = p0 + warp; p < p1; p += kWarps) {
    const int k = __ldg(lab + base + p) - k0;           // the same for the whole warp
    if ((unsigned)k >= (unsigned)nk) continue;
    double w = 1.0, u = 1.0;
    if (wt.pix != nullptr) {
      const double g = g0 * (double)__ldg(wt.pix + wt.nhw + base + p);
      w = g / fmax((double)__ldg(wt.pix + 2 * wt.nhw + base + p), kEps);
      u = g * (double)__ldg(wt.pix + base + p);
    }
    float v[4];
    load4<V4>(x + p * m.sp, c0, m.C, v);
    double* a = sh + ((size_t)k * kWarps + warp) * kTileC + lane;     // slot j * 32 + lane holds channel c0 + j
#pragma unroll
    for (int j = 0; j < 4; ++j) a[j * 32] = fma(w, (double)v[j], a[j * 32]);
    if (counts) shc[warp * pl.kg + k] += u;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < nk * kTileC; e += kThreads) {
    const int kk = e / kTileC, cc = e - kk * kTileC, c = tile * kTileC + cc;
    if (c >= m.C) continue;
    const int s = (cc & 3) * 32 + (cc >> 2);
    double t = 0.0;
    for (int w = 0; w < kWarps; ++w) t += sh[((size_t)kk * kWarps + w) * kTileC + s];
    part[(((long long)n * pl.chunks + chunk) * pl.K + k0 + kk) * m.C + c] = t;
  }
  if (tile == 0) {
    for (int kk = threadIdx.x; kk < nk; kk += kThreads) {
      double t = 0.0;
      for (int w = 0; w < kWarps; ++w) t += shc[w * pl.kg + kk];
      cpart[((long long)n * pl.chunks + chunk) * pl.K + k0 + kk] = t;
    }
  }
}

// fixed-order sum of one double over a kFinThreads block; valid in thread 0
__device__ __forceinline__ double block_sum_d(double v, double* sh) {
  v = warp_sum_d(v);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x == 0)
    for (int i = 0; i < kFinThreads / 32; ++i) t += sh[i];
  return t;
}

// forward, one block per (n, k): the chunks combined in order -> P[n][k][C] = sum / (cnt + 1e-6) (fp32), pn2[n][k] = |P|^2 of those
// fp32 values, and cnt[n][k] when `cnt` is given
__global__ void __launch_bounds__(kFinThreads)
ifv_proto_kernel(Plan pl, const double* __restrict__ part, const double* __restrict__ cpart, float* __restrict__ P,
                 double* __restrict__ cnt, double* __restrict__ pn2) {
  __shared__ double sh[kFinThreads / 32];
  const long long nk = blockIdx.x;
  const long long n = nk / pl.K, k = nk - n * pl.K;
  double c = 0.0;
  for (int j = 0; j < pl.chunks; ++j) c += cpart[(n * pl.chunks + j) * pl.K + k];
  const double den = c + kCntEps;
  double acc = 0.0;
  for (int ch = threadIdx.x; ch < pl.C; ch += kFinThreads) {
    double s = 0.0;
    for (int j = 0; j < pl.chunks; ++j) s += part[((n * pl.chunks + j) * pl.K + k) * pl.C + ch];
    const float p = (float)(s / den);
    P[nk * pl.C + ch] = p;
    acc = fma((double)p, (double)p, acc);
  }
  const double t = block_sum_d(acc, sh);
  if (threadIdx.x == 0) {
    pn2[nk] = t;
    if (cnt != nullptr) cnt[nk] = c;
  }
}

// backward, one block per (n, k): A (part) and B (cpart) combined in order -> Qs[n][k][C] = Q_k / (cnt + 1e-6)
__global__ void __launch_bounds__(kFinThreads)
ifv_q_kernel(Plan pl, const double* __restrict__ part, const double* __restrict__ cpart, const float* __restrict__ P,
             const double* __restrict__ cnt, const double* __restrict__ pn2, float* __restrict__ Qs) {
  const long long nk = blockIdx.x;
  const long long n = nk / pl.K, k = nk - n * pl.K;
  double B = 0.0;
  for (int j = 0; j < pl.chunks; ++j) B += cpart[(n * pl.chunks + j) * pl.K + k];
  const double pn = sqrt(pn2[nk]), np = fmax(pn, kEps), den = cnt[nk] + kCntEps;
  const double bp = pn > 0.0 ? B / (np * pn) : 0.0;
  for (int ch = threadIdx.x; ch < pl.C; ch += kFinThreads) {
    double A = 0.0;
    for (int j = 0; j < pl.chunks; ++j) A += part[((n * pl.chunks + j) * pl.K + k) * pl.C + ch];
    Qs[nk * pl.C + ch] = (float)((A / np - (double)P[nk * pl.C + ch] * bp) / den);
  }
}

// per lane: (f . p, f . f) over its channels of row x against the prototype row pr
template <bool V4>
__device__ __forceinline__ void dot_row(const float* __restrict__ x, const float* __restrict__ pr, int C, double& fp, double& ff) {
  for (int c = (threadIdx.x & 31) * 4; c < C; c += 128) {
    float v[4], q[4];
    load4<V4>(x, c, C, v);
    load4<V4>(pr, c, C, q);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      fp = fma((double)v[j], (double)q[j], fp);
      ff = fma((double)v[j], (double)v[j], ff);
    }
  }
}

// one warp per pixel i (grid-stride): pix[0][i] = cos_S, pix[1][i] = cos_S - cos_T, pix[2][i] = |f_S| (all 0 for an ignored pixel);
// lpart[block] = sum of (cos_S - cos_T)^2 over the block's pixels, warps in order
template <bool V4>
__global__ void __launch_bounds__(kThreads)
ifv_cos_kernel(int N, int HW, int K, const int* __restrict__ lab, Map s, Map t, const float* __restrict__ PS, const float* __restrict__ PT,
               const double* __restrict__ pn2S, const double* __restrict__ pn2T, float* __restrict__ pix, double* __restrict__ lpart) {
  __shared__ double sh[kWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long nhw = (long long)N * HW;
  double l2 = 0.0;
  for (long long i = (long long)blockIdx.x * kWarps + warp; i < nhw; i += (long long)gridDim.x * kWarps) {
    const int k = __ldg(lab + i);
    if (k < 0 || k >= K) {
      if (lane == 0) pix[i] = pix[nhw + i] = pix[2 * nhw + i] = 0.f;
      continue;
    }
    const long long n = i / HW, p = i - n * HW, nk = n * K + k;
    double fs = 0.0, ss = 0.0, ft = 0.0, tt = 0.0;
    dot_row<V4>(s.x + n * s.sn + p * s.sp, PS + nk * s.C, s.C, fs, ss);
    dot_row<V4>(t.x + n * t.sn + p * t.sp, PT + nk * t.C, t.C, ft, tt);
    fs = warp_sum_d(fs); ss = warp_sum_d(ss); ft = warp_sum_d(ft); tt = warp_sum_d(tt);
    const double ns = sqrt(ss);
    const double cs = fs / (fmax(ns, kEps) * fmax(sqrt(pn2S[nk]), kEps));
    const double ct = ft / (fmax(sqrt(tt), kEps) * fmax(sqrt(pn2T[nk]), kEps));
    const double d = cs - ct;
    if (lane == 0) {
      pix[i] = (float)cs; pix[nhw + i] = (float)d; pix[2 * nhw + i] = (float)ns;
      l2 = fma(d, d, l2);
    }
  }
  if (lane == 0) sh[warp] = l2;
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0;
    for (int w = 0; w < kWarps; ++w) a += sh[w];
    lpart[blockIdx.x] = a;
  }
}

// loss = scale * sum of the n block partials, in order
__global__ void __launch_bounds__(kFinThreads)
ifv_loss_kernel(const double* __restrict__ lpart, int n, double scale, float* __restrict__ loss) {
  __shared__ double sh[kFinThreads / 32];
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += kFinThreads) acc += lpart[i];
  const double t = block_sum_d(acc, sh);
  if (threadIdx.x == 0) loss[0] = (float)(t * scale);
}

// backward, one warp per pixel: dS_i = a_i P_k - b_i f_i + Qs_k at dS's strides (0 for an ignored pixel)
template <bool V4>
__global__ void __launch_bounds__(kThreads)
ifv_grad_kernel(int N, int HW, int K, const int* __restrict__ lab, Map s, const float* __restrict__ PS, const double* __restrict__ pn2S,
                const float* __restrict__ pix, const float* __restrict__ Qs, const float* __restrict__ gout, double scale,
                float* __restrict__ dS, long long d_sn, long long d_sp) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long nhw = (long long)N * HW;
  const double g0 = scale * (double)__ldg(gout);
  for (long long i = (long long)blockIdx.x * kWarps + warp; i < nhw; i += (long long)gridDim.x * kWarps) {
    const int k = __ldg(lab + i);
    const long long n = i / HW, p = i - n * HW;
    float* dst = dS + n * d_sn + p * d_sp;
    const bool valid = k >= 0 && k < K;
    double a = 0.0, b = 0.0;
    const long long nk = n * K + (valid ? k : 0);
    if (valid) {
      const double g = g0 * (double)__ldg(pix + nhw + i), fn = (double)__ldg(pix + 2 * nhw + i), nf = fmax(fn, kEps);
      a = g / (nf * fmax(sqrt(pn2S[nk]), kEps));
      b = fn > 0.0 ? g * (double)__ldg(pix + i) / (nf * fn) : 0.0;
    }
    const float* x = s.x + n * s.sn + p * s.sp;
    for (int c = lane * 4; c < s.C; c += 128) {
      float r[4] = {0.f, 0.f, 0.f, 0.f};
      if (valid) {
        float f[4], pk[4], q[4];
        load4<V4>(x, c, s.C, f);
        load4<V4>(PS + nk * s.C, c, s.C, pk);
        load4<V4>(Qs + nk * s.C, c, s.C, q);
#pragma unroll
        for (int j = 0; j < 4; ++j) r[j] = (float)fma(a, (double)pk[j], fma(-b, (double)f[j], (double)q[j]));
      }
      if constexpr (V4) {
        *reinterpret_cast<float4*>(dst + c) = make_float4(r[0], r[1], r[2], r[3]);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (c + j < s.C) dst[c + j] = r[j];
      }
    }
  }
}

bool aligned4(const void* p, long long sn, long long sp, int C) {
  return (reinterpret_cast<uintptr_t>(p) & 15) == 0 && sn % 4 == 0 && sp % 4 == 0 && C % 4 == 0;
}

bool check(const char* who, int N, int HW, int K, int CS, int CT) {
  if (N < 1 || HW < 1 || CS < 1 || CT < 1) { set_error_msg(who, "empty map"); return false; }
  if (K < 1 || K > 255) { set_error_msg(who, "the class count must be in [1, 255]"); return false; }
  if ((long long)N * ((K + kMaxGroup - 1) / kMaxGroup) > 65535) { set_error_msg(who, "too many images"); return false; }
  return true;
}

template <bool V4>
bool class_sum(const Plan& pl, const int* lab, Map m, Wts wt, double* part, double* cpart, cudaStream_t st, const char* who) {
  static bool attr = false;                           // once, for the largest class group
  if (!attr) {
    const cudaError_t e = cudaFuncSetAttribute(ifv_class_sum_kernel<V4>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               (int)((size_t)kMaxGroup * kWarps * (kTileC + 1) * sizeof(double)));
    if (e != cudaSuccess) { set_error(who, e); return false; }
    attr = true;
  }
  const dim3 g(pl.chunks, (pl.C + kTileC - 1) / kTileC, pl.N * pl.groups);
  ifv_class_sum_kernel<V4><<<g, kThreads, sum_smem(pl), st>>>(pl, lab, m, wt, part, cpart);
  return true;
}

bool class_sum_any(const Plan& pl, const int* lab, Map m, Wts wt, double* part, double* cpart, cudaStream_t st, const char* who) {
  return aligned4(m.x, m.sn, m.sp, m.C) ? class_sum<true>(pl, lab, m, wt, part, cpart, st, who)
                                        : class_sum<false>(pl, lab, m, wt, part, cpart, st, who);
}

}  // namespace

extern "C" int skd_labels_nearest(int N, int H, int W, const long long* labels, int h, int w, int* out, cudaStream_t st) {
  if (N < 1 || H < 1 || W < 1 || h < 1 || w < 1) { set_error_msg("skd_labels_nearest", "empty label map"); return 0; }
  const long long total = (long long)N * h * w;
  labels_nearest_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(N, H, W, labels, h, w, (float)H / (float)h,
                                                                          (float)W / (float)w, out);
  return finish("skd_labels_nearest");
}

// [part | cpart] of the larger map's class sums, the loss partials, then N * K * max(CS, CT) floats (P_T forward, Q backward)
extern "C" long long skd_ifv_workspace(int N, int HW, int K, int CS, int CT) {
  if (N < 1 || HW < 1 || K < 1 || CS < 1 || CT < 1) return 0;
  const long long parts = std::max(part_doubles(sum_plan(N, HW, K, CS)), part_doubles(sum_plan(N, HW, K, CT)));
  return parts + kPixBlocks + ((long long)N * K * std::max(CS, CT) + 1) / 2;
}

extern "C" int skd_ifv_fwd(int N, int HW, int K, const int* lab, const float* S, int CS, long long s_sn, long long s_sp, const float* T,
                           int CT, long long t_sn, long long t_sp, float* loss, float* PS, double* stats, float* pix, double* workspace,
                           cudaStream_t st) {
  if (!check("skd_ifv_fwd", N, HW, K, CS, CT)) return 0;
  const Plan ps = sum_plan(N, HW, K, CS), pt = sum_plan(N, HW, K, CT);
  const long long parts = std::max(part_doubles(ps), part_doubles(pt));
  double* lpart = workspace + parts;
  float* PT = reinterpret_cast<float*>(lpart + kPixBlocks);
  const Map ms{S, s_sn, s_sp, CS}, mt{T, t_sn, t_sp, CT};
  const Wts ones{nullptr, nullptr, 0.0, 0};
  double* cnt = stats;
  double* pn2S = stats + (long long)N * K;
  double* pn2T = stats + 2LL * N * K;
  if (!class_sum_any(ps, lab, ms, ones, workspace, workspace + (long long)N * ps.chunks * K * CS, st, "skd_ifv_fwd")) return 0;
  ifv_proto_kernel<<<N * K, kFinThreads, 0, st>>>(ps, workspace, workspace + (long long)N * ps.chunks * K * CS, PS, cnt, pn2S);
  if (!class_sum_any(pt, lab, mt, ones, workspace, workspace + (long long)N * pt.chunks * K * CT, st, "skd_ifv_fwd")) return 0;
  ifv_proto_kernel<<<N * K, kFinThreads, 0, st>>>(pt, workspace, workspace + (long long)N * pt.chunks * K * CT, PT, nullptr, pn2T);
  const long long nhw = (long long)N * HW;
  const int nb = pix_blocks(nhw);
  if (aligned4(S, s_sn, s_sp, CS) && aligned4(T, t_sn, t_sp, CT))
    ifv_cos_kernel<true><<<nb, kThreads, 0, st>>>(N, HW, K, lab, ms, mt, PS, PT, pn2S, pn2T, pix, lpart);
  else
    ifv_cos_kernel<false><<<nb, kThreads, 0, st>>>(N, HW, K, lab, ms, mt, PS, PT, pn2S, pn2T, pix, lpart);
  ifv_loss_kernel<<<1, kFinThreads, 0, st>>>(lpart, nb, 1.0 / (double)nhw, loss);
  return finish("skd_ifv_fwd", 6);
}

extern "C" int skd_ifv_bwd(int N, int HW, int K, const int* lab, const float* S, int CS, long long s_sn, long long s_sp, const float* PS,
                           const double* stats, const float* pix, const float* grad_out, float* dS, long long d_sn, long long d_sp,
                           double* workspace, cudaStream_t st) {
  if (!check("skd_ifv_bwd", N, HW, K, CS, CS)) return 0;
  const Plan ps = sum_plan(N, HW, K, CS);
  const long long nhw = (long long)N * HW;
  const double scale = 2.0 / (double)nhw;
  const Map ms{S, s_sn, s_sp, CS};
  const Wts wt{pix, grad_out, scale, nhw};
  double* cpart = workspace + (long long)N * ps.chunks * K * CS;
  float* Qs = reinterpret_cast<float*>(workspace + part_doubles(ps) + kPixBlocks);
  if (!class_sum_any(ps, lab, ms, wt, workspace, cpart, st, "skd_ifv_bwd")) return 0;
  ifv_q_kernel<<<N * K, kFinThreads, 0, st>>>(ps, workspace, cpart, PS, stats, stats + (long long)N * K, Qs);
  const int nb = pix_blocks(nhw);
  if (aligned4(S, s_sn, s_sp, CS) && aligned4(dS, d_sn, d_sp, CS))
    ifv_grad_kernel<true><<<nb, kThreads, 0, st>>>(N, HW, K, lab, ms, PS, stats + (long long)N * K, pix, Qs, grad_out, scale, dS, d_sn, d_sp);
  else
    ifv_grad_kernel<false><<<nb, kThreads, 0, st>>>(N, HW, K, lab, ms, PS, stats + (long long)N * K, pix, Qs, grad_out, scale, dS, d_sn,
                                                    d_sp);
  return finish("skd_ifv_bwd", 3);
}
