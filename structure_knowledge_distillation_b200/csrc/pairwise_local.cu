// Local pair-wise affinity distillation for sm_90a (SIMT, fp32 FMA, no tensor cores): the pair-wise (Pa) term with each pooled node
// connected to its k x k neighbours at dilation d instead of to every node, so it runs at one node per pixel.
//   a_ij = (f_i . f_j) * rn_i * rn_j,  rn = 1 / (||f||_2 + 1e-8) (the global form's detached norm, losses.cu)
//   E[i][o] = a^T_ij - a^S_ij for offset o = (t + r) * k + (u + r), j = (y + t d, x + u d), t, u in -r..r, r = (k - 1) / 2;
//             E[i][o] = 0 where j lies outside the h x w grid
//   loss    = sum E^2 / (N * P),  P = (sum_y c_h(y)) * (sum_x c_w(x)) connected ordered pairs per image
//   dpooled_S[i] = -4 g / (N * P) * rn_i * sum_o E[i][o] * rn_j f_j  (the window is symmetric: j in W(i) <=> i in W(j), E_ij = E_ji)
// Tiling: one CTA per (image, residue class (y mod d, x mod d), 8 x 8 tile of that class's sub-grid), so the halo is r nodes whatever
// d is.  The tile's rows plus the halo pass through shared memory in 16-channel chunks; each thread holds the (node, offset) dot products
// of one node and a quarter of the offsets in registers.  Nothing of size nodes^2 exists; the loss partials (one double per CTA) are
// summed in a fixed order, so two calls give bit-identical results.
#include "common.cuh"
#include "skd.h"

using namespace skd;

namespace {

constexpr int kTile = 8;                      // 8 x 8 nodes of one residue class per CTA
constexpr int kTileNodes = kTile * kTile;
constexpr int kThreads = 256;
constexpr int kGroups = kThreads / kTileNodes;   // forward: 4 offset groups per node
constexpr int kCC = 16;                       // channels per shared-memory chunk
constexpr int kFwdLd = kCC + 4;               // forward halo row stride: float4-aligned, 8 consecutive rows hit distinct banks
constexpr int kBwdLd = kCC + 1;               // backward halo row stride: lanes differ in the channel

struct TileGeom {
  int h, w, d, ry, rx, ty0, tx0;              // grid, dilation, residue class, tile origin in the class's sub-grid
};

__device__ __forceinline__ TileGeom tile_geom(int h, int w, int d, int tiles_x) {
  TileGeom g;
  g.h = h; g.w = w; g.d = d;
  g.ry = blockIdx.y / d; g.rx = blockIdx.y - g.ry * d;
  g.ty0 = (blockIdx.x / tiles_x) * kTile; g.tx0 = (blockIdx.x % tiles_x) * kTile;
  return g;
}

// node index of the tile-relative position (a, b) (halo included: a, b in -R .. kTile - 1 + R), or -1 outside the grid
__device__ __forceinline__ int node_at(const TileGeom& g, int a, int b) {
  const int sy = g.ty0 + a, sx = g.tx0 + b;
  if (sy < 0 || sx < 0) return -1;
  const int y = g.ry + g.d * sy, x = g.rx + g.d * sx;
  return (y < g.h && x < g.w) ? y * g.w + x : -1;
}

// channels c0 .. c0 + kCC - 1 of the tile's rows and halo (zero outside the grid and past C), scaled by rn when given
template <int K, int LD>
__device__ __forceinline__ void load_halo(float* sm, const TileGeom& g, const float* __restrict__ P, int C, int c0,
                                          const float* __restrict__ rn) {
  constexpr int R = (K - 1) / 2, HW = kTile + 2 * R;
  for (int i = threadIdx.x; i < HW * HW * kCC; i += kThreads) {
    const int a = i / kCC, c = i - a * kCC;
    const int hy = a / HW, hx = a - hy * HW;
    const int j = node_at(g, hy - R, hx - R);
    float v = 0.f;
    if (j >= 0 && c0 + c < C) {
      v = __ldg(P + (size_t)j * C + c0 + c);
      if (rn) v *= __ldg(rn + j);
    }
    sm[a * LD + c] = v;
  }
}

// acc[q] = f_i . f_j over all C channels for the offsets o0 .. o0 + OPT - 1 (< K^2) of this thread's node
template <int K, int OPT>
__device__ __forceinline__ void local_dots(float (&acc)[OPT], float* sm, const TileGeom& g, const float* __restrict__ P, int C,
                                           int self, int o0) {
  constexpr int R = (K - 1) / 2, HW = kTile + 2 * R;
#pragma unroll
  for (int q = 0; q < OPT; ++q) acc[q] = 0.f;
  for (int c0 = 0; c0 < C; c0 += kCC) {
    __syncthreads();
    load_halo<K, kFwdLd>(sm, g, P, C, c0, nullptr);
    __syncthreads();
    float4 ctr[kCC / 4];
#pragma unroll
    for (int v = 0; v < kCC / 4; ++v) ctr[v] = *reinterpret_cast<const float4*>(sm + self * kFwdLd + 4 * v);
#pragma unroll
    for (int q = 0; q < OPT; ++q) {
      const int o = o0 + q;
      if (o < K * K) {                                   // warp-uniform: the offset group is constant over a warp
        const int oy = o / K, ox = o - oy * K;
        const float* row = sm + (self + (oy - R) * HW + (ox - R)) * kFwdLd;
        float s = acc[q];
#pragma unroll
        for (int v = 0; v < kCC / 4; ++v) {
          const float4 b = *reinterpret_cast<const float4*>(row + 4 * v);
          s = fmaf(ctr[v].x, b.x, s); s = fmaf(ctr[v].y, b.y, s); s = fmaf(ctr[v].z, b.z, s); s = fmaf(ctr[v].w, b.w, s);
        }
        acc[q] = s;
      }
    }
  }
}

template <int K>
__global__ void __launch_bounds__(kThreads, 1)
pa_local_fwd_kernel(const float* __restrict__ pS, const float* __restrict__ pT, const float* __restrict__ rS,
                    const float* __restrict__ rT, int CS, int CT, int h, int w, int d, int tiles_x, float* __restrict__ E,
                    double* __restrict__ part) {
  constexpr int R = (K - 1) / 2, HW = kTile + 2 * R, K2 = K * K, OPT = (K2 + kGroups - 1) / kGroups;
  __shared__ __align__(16) float sm[HW * HW * kFwdLd];
  __shared__ double red[kThreads / 32];
  const TileGeom g = tile_geom(h, w, d, tiles_x);
  const int n = blockIdx.z, nodes = h * w;
  const int p = threadIdx.x % kTileNodes, grp = threadIdx.x / kTileNodes;
  const int py = p / kTile, px = p - py * kTile;
  const int self = (py + R) * HW + px + R, o0 = grp * OPT;
  const int i = node_at(g, py, px);
  const size_t img = (size_t)n * nodes;

  float aT[OPT], aS[OPT];
  local_dots<K, OPT>(aT, sm, g, pT + img * CT, CT, self, o0);
  local_dots<K, OPT>(aS, sm, g, pS + img * CS, CS, self, o0);

  double sq = 0.0;
  if (i >= 0) {
    const float rTi = __ldg(rT + img + i), rSi = __ldg(rS + img + i);
#pragma unroll
    for (int q = 0; q < OPT; ++q) {
      const int o = o0 + q;
      if (o < K2) {
        const int oy = o / K, ox = o - oy * K;
        const int j = node_at(g, py + oy - R, px + ox - R);
        float e = 0.f;
        if (j >= 0) e = aT[q] * rTi * __ldg(rT + img + j) - aS[q] * rSi * __ldg(rS + img + j);
        if (E) E[(img + i) * K2 + o] = e;
        sq += (double)e * (double)e;
      }
    }
  }
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sq;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int k = 0; k < kThreads / 32; ++k) t += red[k];
    part[((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = t;
  }
}

// loss = scale * sum of the partials, one block in a fixed order
__global__ void __launch_bounds__(256) pa_local_finalize_kernel(const double* __restrict__ part, int n, double scale, float* __restrict__ loss) {
  __shared__ double sh[8];
  double a = 0.0;
  for (int k = threadIdx.x; k < n; k += 256) a += part[k];
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = a;
  __syncthreads();
  if (threadIdx.x == 0) {
    a = 0.0;
    for (int k = 0; k < 8; ++k) a += sh[k];
    loss[0] = (float)(a * scale);
  }
}

// dpooled_S[i][c] = coef * rS_i * sum_o E[i][o] * rS_j pS[j][c]: 16 channel lanes x 16 node groups, 4 of the tile's nodes per thread
template <int K>
__global__ void __launch_bounds__(kThreads)
pa_local_bwd_kernel(const float* __restrict__ E, const float* __restrict__ pS, const float* __restrict__ rS, int CS, int h, int w,
                    int d, int tiles_x, float scale, const float* __restrict__ gout, float* __restrict__ dpooled) {
  constexpr int R = (K - 1) / 2, HW = kTile + 2 * R, K2 = K * K, NPT = kTileNodes / (kThreads / kCC);
  __shared__ float sm[HW * HW * kBwdLd];
  const TileGeom g = tile_geom(h, w, d, tiles_x);
  const int n = blockIdx.z, nodes = h * w;
  const size_t img = (size_t)n * nodes;
  const int c = threadIdx.x % kCC, grp = threadIdx.x / kCC;
  const float coef = scale * __ldg(gout);
  int node[NPT], self[NPT];
#pragma unroll
  for (int k = 0; k < NPT; ++k) {
    const int p = grp + k * (kThreads / kCC), py = p / kTile, px = p - py * kTile;
    node[k] = node_at(g, py, px);
    self[k] = (py + R) * HW + px + R;
  }
  for (int c0 = 0; c0 < CS; c0 += kCC) {
    __syncthreads();
    load_halo<K, kBwdLd>(sm, g, pS + img * CS, CS, c0, rS + img);
    __syncthreads();
#pragma unroll
    for (int k = 0; k < NPT; ++k) {
      if (node[k] < 0) continue;
      const float* e = E + (img + node[k]) * K2;
      float acc = 0.f;
#pragma unroll 5
      for (int o = 0; o < K2; ++o) {
        const int oy = o / K, ox = o - oy * K;
        acc = fmaf(__ldg(e + o), sm[(self[k] + (oy - R) * HW + (ox - R)) * kBwdLd + c], acc);
      }
      if (c0 + c < CS) dpooled[(img + node[k]) * CS + c0 + c] = coef * __ldg(rS + img + node[k]) * acc;
    }
  }
}

// sum over positions 0 <= y < L of #{t in -r..r : 0 <= y + t d < L}
long long axis_pairs(int L, int r, int d) {
  long long s = 0;
  for (int y = 0; y < L; ++y)
    for (int t = -r; t <= r; ++t) s += (y + t * d >= 0 && y + t * d < L);
  return s;
}

bool check_args(const char* who, int N, int h, int w, int CS, int CT, int k, int d) {
  if (N < 1 || h < 1 || w < 1 || CS < 1 || CT < 1) { set_error_msg(who, "empty input"); return false; }
  if (k < 3 || k > 15 || k % 2 == 0) { set_error_msg(who, "window must be odd, 3..15"); return false; }
  if (d < 1 || d > 8) { set_error_msg(who, "dilation must be 1..8"); return false; }
  if ((long long)h * w > (1LL << 30) / 225) { set_error_msg(who, "grid too large"); return false; }
  return true;
}

dim3 local_grid(int N, int h, int w, int d, int* tiles_x) {
  const int hs = (h + d - 1) / d, ws = (w + d - 1) / d;            // residue class 0 has the largest sub-grid
  *tiles_x = (ws + kTile - 1) / kTile;
  return dim3(((hs + kTile - 1) / kTile) * *tiles_x, d * d, N);
}

template <int K>
void launch_fwd(dim3 grid, int tiles_x, const float* pS, const float* pT, const float* rS, const float* rT, int CS, int CT, int h, int w,
                int d, float* E, double* part, cudaStream_t st) {
  pa_local_fwd_kernel<K><<<grid, kThreads, 0, st>>>(pS, pT, rS, rT, CS, CT, h, w, d, tiles_x, E, part);
}

template <int K>
void launch_bwd(dim3 grid, int tiles_x, const float* E, const float* pS, const float* rS, int CS, int h, int w, int d, float scale,
                const float* gout, float* dpooled, cudaStream_t st) {
  pa_local_bwd_kernel<K><<<grid, kThreads, 0, st>>>(E, pS, rS, CS, h, w, d, tiles_x, scale, gout, dpooled);
}

#define SKD_PA_LOCAL_DISPATCH(k, CALL)                                                                   \
  switch (k) {                                                                                           \
    case 3: CALL(3); break; case 5: CALL(5); break; case 7: CALL(7); break; case 9: CALL(9); break;      \
    case 11: CALL(11); break; case 13: CALL(13); break; default: CALL(15); break;                        \
  }

}  // namespace

extern "C" long long skd_pairwise_local_pairs(int h, int w, int k, int d) {
  return axis_pairs(h, (k - 1) / 2, d) * axis_pairs(w, (k - 1) / 2, d);
}

extern "C" long long skd_pairwise_local_partials(int N, int h, int w, int k, int d) {
  if (d < 1) return 0;
  int tiles_x;
  const dim3 g = local_grid(N, h, w, d, &tiles_x);
  return (long long)g.x * g.y * g.z;
}

extern "C" int skd_pairwise_local_fwd(int N, int h, int w, int CS, int CT, const float* pooled_S, const float* pooled_T,
                                      const float* rnorm_S, const float* rnorm_T, int k, int d, float* E, float* loss, double* partials,
                                      cudaStream_t st) {
  const char* who = "skd_pairwise_local_fwd";
  if (!check_args(who, N, h, w, CS, CT, k, d)) return 0;
  int tiles_x;
  const dim3 grid = local_grid(N, h, w, d, &tiles_x);
#define SKD_FWD(K) launch_fwd<K>(grid, tiles_x, pooled_S, pooled_T, rnorm_S, rnorm_T, CS, CT, h, w, d, E, partials, st)
  SKD_PA_LOCAL_DISPATCH(k, SKD_FWD)
#undef SKD_FWD
  const double pairs = (double)skd_pairwise_local_pairs(h, w, k, d);
  pa_local_finalize_kernel<<<1, 256, 0, st>>>(partials, (int)(grid.x * grid.y * grid.z), 1.0 / ((double)N * pairs), loss);
  return finish(who, 2);
}

extern "C" int skd_pairwise_local_bwd(int N, int h, int w, int CS, const float* E, const float* pooled_S, const float* rnorm_S, int k,
                                      int d, const float* grad_out, float* dpooled, cudaStream_t st) {
  const char* who = "skd_pairwise_local_bwd";
  if (!check_args(who, N, h, w, CS, 1, k, d)) return 0;
  int tiles_x;
  const dim3 grid = local_grid(N, h, w, d, &tiles_x);
  const float scale = (float)(-4.0 / ((double)N * (double)skd_pairwise_local_pairs(h, w, k, d)));
#define SKD_BWD(K) launch_bwd<K>(grid, tiles_x, E, pooled_S, rnorm_S, CS, h, w, d, scale, grad_out, dpooled, st)
  SKD_PA_LOCAL_DISPATCH(k, SKD_BWD)
#undef SKD_BWD
  return finish(who);
}
