// NHWC pooling / resampling / optimizer kernels for sm_90a (all HBM- or latency-bound; float4 over channels).
//   * 3x3 s2 p1 ceil-mode max-pool of the ResNet stem          networks/pspnet_combine.py:130
//   * AdaptiveAvgPool2d(1/2/3/6) of the PSP module               networks/pspnet_combine.py:103
//   * bilinear(align_corners) upsampling of the PSP priors, written straight into their channel slice of the
//     concat buffer (no torch.cat pass)                           networks/pspnet_combine.py:110-111
//   * momentum-SGD with weight decay over one flat parameter buffer   networks/kd_model.py:74,171
#include "common.cuh"
#include "skd.h"

using namespace skd;

namespace {

__host__ __device__ inline int pool_out_ceil(int in, int k, int s, int p) {
  int o = (in + 2 * p - k + s - 1) / s + 1;
  if ((o - 1) * s >= in + p) --o;                      // ATen pooling_output_shape, ceil_mode
  return o;
}

// grid (rows, slices of a row): ~4 float4 per thread and slice
dim3 row_grid(int rows, int per_row) {
  int ys = (per_row + 1023) / 1024;
  if (ys < 1) ys = 1;
  if (ys > 64) ys = 64;
  return dim3((unsigned)rows, (unsigned)ys);
}

int ew_blocks(long long total) {
  long long b = (total + 255) / 256;
  if (b > kNumSMs * 16) b = kNumSMs * 16;
  if (b < 1) b = 1;
  return (int)b;
}

__device__ __forceinline__ void max4(float4& best, int4& bi, const float4 v, int idx) {
  if (v.x > best.x || v.x != v.x) { best.x = v.x; bi.x = idx; }
  if (v.y > best.y || v.y != v.y) { best.y = v.y; bi.y = idx; }
  if (v.z > best.z || v.z != v.z) { best.z = v.z; bi.z = idx; }
  if (v.w > best.w || v.w != v.w) { best.w = v.w; bi.w = idx; }
}

// One block per (output row, slice of the row): the (n, y) decomposition is done once per block and the inner index is 32-bit (the
// flat 64-bit i -> (n, y, x, c4) chain of divisions costs more issue slots than the memory traffic).
__global__ void __launch_bounds__(256)
maxpool_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, unsigned char* __restrict__ arg, int N, int H, int W,
                   int C4, int OH, int OW) {
  const int row = blockIdx.x, n = row / OH, oy = row - n * OH;
  const int per = OW * C4;
  const float4* xin = reinterpret_cast<const float4*>(x) + (long long)n * H * W * C4;
  const long long obase = (long long)row * per;
  for (int j = blockIdx.y * blockDim.x + threadIdx.x; j < per; j += gridDim.y * blockDim.x) {
    const int ox = j / C4, c4 = j - ox * C4;
    float4 best = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY); int4 bi = make_int4(0, 0, 0, 0);
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int iy = oy * 2 - 1 + ky;
      if (iy < 0 || iy >= H) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int ix = ox * 2 - 1 + kx;
        if (ix < 0 || ix >= W) continue;
        max4(best, bi, __ldg(xin + ((long long)iy * W + ix) * C4 + c4), ky * 3 + kx);
      }
    }
    reinterpret_cast<float4*>(y)[obase + j] = best;
    reinterpret_cast<uchar4*>(arg)[obase + j] = make_uchar4(bi.x, bi.y, bi.z, bi.w);
  }
}

// gather form: every input element looks at the <=4 windows that cover it
__global__ void __launch_bounds__(256)
maxpool_bwd_kernel(const float* __restrict__ dy, const unsigned char* __restrict__ arg, float* __restrict__ dx, int N, int H,
                   int W, int C4, int OH, int OW) {
  const int row = blockIdx.x, n = row / H, iy = row - n * H;
  const int per = W * C4;
  const long long ibase = (long long)row * per, nbase = (long long)n * OH * OW * C4;
  for (int j = blockIdx.y * blockDim.x + threadIdx.x; j < per; j += gridDim.y * blockDim.x) {
    const int ix = j / C4, c4 = j - ix * C4;
    float4 g = make_float4(0, 0, 0, 0);
    for (int oy = iy / 2; oy <= (iy + 1) / 2 && oy < OH; ++oy) {
      const int ky = iy - (oy * 2 - 1);
      if (ky < 0 || ky > 2) continue;
      for (int ox = (ix) / 2; ox <= (ix + 1) / 2 && ox < OW; ++ox) {
        const int kx = ix - (ox * 2 - 1);
        if (kx < 0 || kx > 2) continue;
        const long long o = nbase + ((long long)oy * OW + ox) * C4 + c4;
        const uchar4 a = reinterpret_cast<const uchar4*>(arg)[o];
        const float4 d = __ldg(reinterpret_cast<const float4*>(dy) + o);
        const int k = ky * 3 + kx;
        if (a.x == k) g.x += d.x;
        if (a.y == k) g.y += d.y;
        if (a.z == k) g.z += d.z;
        if (a.w == k) g.w += d.w;
      }
    }
    reinterpret_cast<float4*>(dx)[ibase + j] = g;
  }
}

// ---- PSP pyramid: all bins of all levels in one launch -------------------------------------------------
struct Pyramid { int levels; int size[4]; int first_bin[5]; };

__device__ __forceinline__ void bin_of(const Pyramid& p, int bin, int& lvl, int& by, int& bx) {
  lvl = 0;
  while (lvl + 1 < p.levels && bin >= p.first_bin[lvl + 1]) ++lvl;
  const int b = bin - p.first_bin[lvl];
  by = b / p.size[lvl]; bx = b - by * p.size[lvl];
}
__device__ __forceinline__ int bin_lo(int i, int in, int s) { return (i * in) / s; }                  // floor
__device__ __forceinline__ int bin_hi(int i, int in, int s) { return ((i + 1) * in + s - 1) / s; }    // ceil

// Separable pyramid pooling, one pass over the feature map for ALL levels:
//   stage 1: rowbins[n][y][xb][c] = sum_{x in x-bin xb} x[n][y][x][c]      (xb runs over the 1+2+3+6 x-bins of all levels)
//   stage 2: pooled[n][bin][c]    = sum_{y in y-bin} rowbins[n][y][xb(bin)][c] / area
constexpr int kMaxXBins = 16, kMaxXSegs = 32;
// x-bins of all levels expressed over the segments between their sorted distinct end points: every x lies in exactly one segment,
// bin b = segments [fs[b], ls[b]).  One add per loaded value instead of one compare per (value, bin).
struct XBins { int n, nseg; int seg_lo[kMaxXSegs + 1]; int fs[kMaxXBins]; int ls[kMaxXBins]; };

// block = 64 channel quads (float4) x 4 x-lanes (adjacent threads: a warp reads 4 pixels x 128 contiguous bytes); lanes are folded
// with two shuffles per segment.  (Walking a row with scalar loads and 12 compares per value is issue-bound.)
__global__ void __launch_bounds__(256)
psp_rowbins_kernel(const float* __restrict__ x, int pitch, int C, int H, int W, XBins xb, float* __restrict__ rowbins) {
  const int y = blockIdx.x, n = blockIdx.y, xl = threadIdx.x & 3, cq = threadIdx.x >> 2;
  const int c = (blockIdx.z * 64 + cq) * 4;
  const bool active = c < C;
  float4 acc[kMaxXBins];
#pragma unroll
  for (int b = 0; b < kMaxXBins; ++b) acc[b] = make_float4(0.f, 0.f, 0.f, 0.f);
  const float* base = x + ((size_t)n * H + y) * W * pitch + (active ? c : 0);
  for (int sgm = 0; sgm < xb.nseg; ++sgm) {
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    if (active)
      for (int xx = xb.seg_lo[sgm] + xl; xx < xb.seg_lo[sgm + 1]; xx += 4) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(base + (size_t)xx * pitch));
        a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
      }
#pragma unroll
    for (int o = 1; o < 4; o <<= 1) {
      a.x += __shfl_xor_sync(0xffffffffu, a.x, o); a.y += __shfl_xor_sync(0xffffffffu, a.y, o);
      a.z += __shfl_xor_sync(0xffffffffu, a.z, o); a.w += __shfl_xor_sync(0xffffffffu, a.w, o);
    }
#pragma unroll
    for (int b = 0; b < kMaxXBins; ++b)
      if (b < xb.n && sgm >= xb.fs[b] && sgm < xb.ls[b]) { acc[b].x += a.x; acc[b].y += a.y; acc[b].z += a.z; acc[b].w += a.w; }
  }
  if (xl == 0 && active) {
    float* out = rowbins + (((size_t)n * H + y) * xb.n) * C + c;
#pragma unroll
    for (int b = 0; b < kMaxXBins; ++b) if (b < xb.n) *reinterpret_cast<float4*>(out + (size_t)b * C) = acc[b];
  }
}

__global__ void __launch_bounds__(256)
psp_colbins_kernel(const float* __restrict__ rowbins, int C, int H, int W, Pyramid p, int nxb, float* __restrict__ pooled) {
  const int bin = blockIdx.x, n = blockIdx.y, c = blockIdx.z * 256 + threadIdx.x;
  if (c >= C) return;
  int lvl, by, bx; bin_of(p, bin, lvl, by, bx);
  const int s = p.size[lvl];
  int xoff = 0;
  for (int l = 0; l < lvl; ++l) xoff += p.size[l];
  const int y0 = bin_lo(by, H, s), y1 = bin_hi(by, H, s), x0 = bin_lo(bx, W, s), x1 = bin_hi(bx, W, s);
  const float* src = rowbins + ((size_t)n * H * nxb + (xoff + bx)) * C + c;
  float a = 0.f;
  for (int y = y0; y < y1; ++y) a += __ldg(src + (size_t)y * nxb * C);
  pooled[((size_t)n * gridDim.x + bin) * C + c] = a / (float)((y1 - y0) * (x1 - x0));
}

// dx[n][y][x][c] = sum over bins containing (y,x) of dpooled/area.  Bin extents come from tables in the kernel parameters (the version
// that re-derived them with integer divisions per element and candidate bin spent ~3 600 instructions per float4).
struct PyrBins { int levels; int size[4]; int first_bin[4]; int lo_y[4][6], hi_y[4][6], lo_x[4][6], hi_x[4][6]; };

__global__ void __launch_bounds__(256)
psp_pool_bwd_kernel(const float* __restrict__ dpooled, int C4, int H, int W, int N, PyrBins p, int nbins,
                    float* __restrict__ dx) {
  const int row = blockIdx.x, n = row / H, yy = row - n * H;
  const int per = W * C4;
  const float4* dp = reinterpret_cast<const float4*>(dpooled) + (size_t)n * nbins * C4;
  const long long obase = (long long)row * per;
  for (int j = blockIdx.y * blockDim.x + threadIdx.x; j < per; j += gridDim.y * blockDim.x) {
    const int xx = j / C4, c4 = j - xx * C4;
    float4 g = make_float4(0, 0, 0, 0);
#pragma unroll
    for (int l = 0; l < 4; ++l) {
      if (l >= p.levels) break;
      const int s = p.size[l];
#pragma unroll
      for (int by = 0; by < 6; ++by) {
        if (by >= s || yy < p.lo_y[l][by] || yy >= p.hi_y[l][by]) continue;
#pragma unroll
        for (int bx = 0; bx < 6; ++bx) {
          if (bx >= s || xx < p.lo_x[l][bx] || xx >= p.hi_x[l][bx]) continue;
          const float inv = 1.f / (float)((p.hi_y[l][by] - p.lo_y[l][by]) * (p.hi_x[l][bx] - p.lo_x[l][bx]));
          const float4 d = __ldg(dp + (size_t)(p.first_bin[l] + by * s + bx) * C4 + c4);
          g.x += d.x * inv; g.y += d.y * inv; g.z += d.z * inv; g.w += d.w * inv;
        }
      }
    }
    reinterpret_cast<float4*>(dx)[obase + j] = g;
  }
}

struct Lin { int i0, i1; float l0, l1; };
__device__ __forceinline__ Lin lin(int dst, int in, int out) {
  const float scale = out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.f;
  const float src = scale * (float)dst;
  Lin b; b.i0 = (int)src; if (b.i0 > in - 1) b.i0 = in - 1;
  b.i1 = b.i0 + (b.i0 < in - 1 ? 1 : 0); b.l1 = src - (float)b.i0; b.l0 = 1.f - b.l1;
  return b;
}

// out[n][y][x][coff + c] = bilinear(src[n][s][s][c]), src = stage output [N][nbins_total][C] slice at first_bin
__global__ void __launch_bounds__(256)
psp_up_fwd_kernel(const float* __restrict__ src, int C4, int s, int nb_total, int first_bin, float* __restrict__ out,
                  int out_pitch4, int coff4, int N, int H, int W) {
  const int row = blockIdx.x, n = row / H, yy = row - n * H;
  const int per = W * C4;
  const Lin by = lin(yy, s, H);
  const float4* b = reinterpret_cast<const float4*>(src) + ((size_t)n * nb_total + first_bin) * C4;
  const float4* r0 = b + (size_t)(by.i0 * s) * C4;
  const float4* r1 = b + (size_t)(by.i1 * s) * C4;
  float4* orow = reinterpret_cast<float4*>(out) + (size_t)row * W * out_pitch4 + coff4;
  const float scale = W > 1 ? (float)(s - 1) / (float)(W - 1) : 0.f;
  for (int j = blockIdx.y * blockDim.x + threadIdx.x; j < per; j += gridDim.y * blockDim.x) {
    const int xx = j / C4, c4 = j - xx * C4;
    const float sx = scale * (float)xx;                                  // lin(xx, s, W) with the scale hoisted
    int i0 = (int)sx; if (i0 > s - 1) i0 = s - 1;
    const int i1 = i0 + (i0 < s - 1 ? 1 : 0);
    const float l1 = sx - (float)i0, l0 = 1.f - l1;
    const float4 v00 = __ldg(r0 + (size_t)i0 * C4 + c4), v01 = __ldg(r0 + (size_t)i1 * C4 + c4);
    const float4 v10 = __ldg(r1 + (size_t)i0 * C4 + c4), v11 = __ldg(r1 + (size_t)i1 * C4 + c4);
    float4 o;
    o.x = by.l0 * (l0 * v00.x + l1 * v01.x) + by.l1 * (l0 * v10.x + l1 * v11.x);
    o.y = by.l0 * (l0 * v00.y + l1 * v01.y) + by.l1 * (l0 * v10.y + l1 * v11.y);
    o.z = by.l0 * (l0 * v00.z + l1 * v01.z) + by.l1 * (l0 * v10.z + l1 * v11.z);
    o.w = by.l0 * (l0 * v00.w + l1 * v01.w) + by.l1 * (l0 * v10.w + l1 * v11.w);
    orow[(size_t)xx * out_pitch4 + c4] = o;
  }
}

// Bilinear-upsample backward, separable:  dsrc[n][iy][ix][c] = sum_y wy(y,iy) * ( sum_x wx(x,ix) * dout[n][y][x][coff+c] )
//   stage 1 (per output row y): T[n][y][ix][c] for the s source columns;   stage 2: weighted sum over the rows.
__global__ void __launch_bounds__(256)
psp_up_bwd_rows_kernel(const float* __restrict__ dout, int pitch, int coff, int C, int s, float* __restrict__ T, int H, int W) {
  __shared__ float sv[3][6][64];
  const int y = blockIdx.x, n = blockIdx.y, cx = threadIdx.x & 63, lane = threadIdx.x >> 6, c = blockIdx.z * 64 + cx;
  float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (c < C) {
    const float* base = dout + ((size_t)n * H + y) * W * pitch + coff + c;
    for (int xx = lane; xx < W; xx += 4) {
      const float v = __ldg(base + (size_t)xx * pitch);
      const Lin bx = lin(xx, s, W);
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        float wgt = 0.f;
        if (bx.i0 == k) wgt += bx.l0;
        if (bx.i1 == k) wgt += bx.l1;
        acc[k] += wgt * v;
      }
    }
  }
  if (lane > 0) {
#pragma unroll
    for (int k = 0; k < 6; ++k) sv[lane - 1][k][cx] = acc[k];
  }
  __syncthreads();
  if (lane == 0 && c < C) {
#pragma unroll
    for (int k = 0; k < 6; ++k) if (k < s) T[(((size_t)n * H + y) * s + k) * C + c] = acc[k] + sv[0][k][cx] + sv[1][k][cx] + sv[2][k][cx];
  }
}

__global__ void __launch_bounds__(256)
psp_up_bwd_cols_kernel(const float* __restrict__ T, int C, int s, int nb_total, int first_bin, float* __restrict__ dsrc, int H) {
  const int bin = blockIdx.x, n = blockIdx.y, c = blockIdx.z * 256 + threadIdx.x;
  if (c >= C) return;
  const int iy = bin / s, ix = bin - iy * s;
  float a = 0.f;
  for (int y = 0; y < H; ++y) {
    const Lin by = lin(y, s, H);
    float wy = 0.f;
    if (by.i0 == iy) wy += by.l0;
    if (by.i1 == iy) wy += by.l1;
    if (wy != 0.f) a += wy * __ldg(T + (((size_t)n * H + y) * s + ix) * C + c);
  }
  dsrc[((size_t)n * nb_total + first_bin + bin) * C + c] = a;
}

// strided channel-slice copy: dst[row][doff + c] = src[row][soff + c]
__global__ void __launch_bounds__(256)
slice_copy_kernel(const float* __restrict__ src, int spitch4, int soff4, float* __restrict__ dst, int dpitch4, int doff4,
                  long long rows, int C4) {
  const long long total = rows * C4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / C4; const int c4 = (int)(i - r * C4);
    reinterpret_cast<float4*>(dst)[r * dpitch4 + doff4 + c4] = ld_stream(reinterpret_cast<const float4*>(src) + r * spitch4 + soff4 + c4);
  }
}

// v = mu*v + (g + wd*p) ; p -= lr*v   (torch.optim.SGD, dampening 0, first step v = g + wd*p)
__global__ void __launch_bounds__(256)
sgd_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ v, long long n4, long long n,
           const float* __restrict__ lr_ptr, float momentum, float wd, int first, float gscale) {
  const float lr = __ldg(lr_ptr);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 pp = reinterpret_cast<float4*>(p)[i];
    const float4 gg = ld_stream(reinterpret_cast<const float4*>(g) + i);
    float4 vv = first ? make_float4(0, 0, 0, 0) : reinterpret_cast<float4*>(v)[i];
#define UPD(f) { const float d = gg.f * gscale + wd * pp.f; vv.f = first ? d : momentum * vv.f + d; pp.f -= lr * vv.f; }
    UPD(x) UPD(y) UPD(z) UPD(w)
#undef UPD
    reinterpret_cast<float4*>(v)[i] = vv; reinterpret_cast<float4*>(p)[i] = pp;
  }
  for (long long i = n4 * 4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float d = g[i] * gscale + wd * p[i];
    const float nv = first ? d : momentum * v[i] + d;
    v[i] = nv; p[i] -= lr * nv;
  }
}

// ---- data-parallel SGD over NVSwitch multicast ------------------------------------------------------------------------------
// The gradient exchange of the path (utils/parallel.py:54-63,155: mean over GPUs of per-GPU gradients) fused with the optimizer:
// rank r owns a contiguous range of the flat buffers.  For every float4 of its range it issues ONE multimem.ld_reduce on the
// multicast address of the symmetric gradient buffer -- the NVSwitch fetches that float4 from every GPU and adds them in the
// switch (NVLS), so the sum arrives over this GPU's links once instead of world-1 times -- applies momentum-SGD with 1/world folded
// in, and writes the new parameters with ONE multimem.st on the multicast address of the symmetric parameter buffer, which the
// switch replicates into every GPU's copy.  A reduce-scatter, the update and an all-gather in a single pass; the momentum buffer
// is touched only by the owner (1/world of the optimizer traffic per GPU); every replica receives bit-identical parameters.
__device__ __forceinline__ float4 multimem_ld_reduce_add(const float* mc) {
  float4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(mc) : "memory");
  return r;
}
__device__ __forceinline__ void multimem_st(float* mc, float4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__global__ void __launch_bounds__(256)
sgd_nvls_kernel(long long lo4, long long hi4, float* __restrict__ p_mc, const float* __restrict__ g_mc, const float* __restrict__ p_local,
                float* __restrict__ v, const float* __restrict__ lr_ptr, float momentum, float wd, float gscale) {
  const float lr = __ldg(lr_ptr);
  for (long long i = lo4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < hi4; i += (long long)gridDim.x * blockDim.x) {
    const float4 gg = multimem_ld_reduce_add(g_mc + 4 * i);
    float4 pp = reinterpret_cast<const float4*>(p_local)[i];
    float4 vv = reinterpret_cast<float4*>(v)[i];
#define UPD(f) { const float d = gg.f * gscale + wd * pp.f; vv.f = momentum * vv.f + d; pp.f -= lr * vv.f; }
    UPD(x) UPD(y) UPD(z) UPD(w)
#undef UPD
    reinterpret_cast<float4*>(v)[i] = vv;
    multimem_st(p_mc + 4 * i, pp);
  }
  __threadfence_system();
}

Pyramid make_pyramid(int levels, const int* sizes) {
  Pyramid p; p.levels = levels; p.first_bin[0] = 0;
  for (int i = 0; i < 4; ++i) p.size[i] = i < levels ? sizes[i] : 1;
  for (int i = 0; i < levels; ++i) p.first_bin[i + 1] = p.first_bin[i] + sizes[i] * sizes[i];
  return p;
}

}  // namespace

extern "C" int skd_pool_out_size_ceil(int in, int k, int s, int p) { return pool_out_ceil(in, k, s, p); }

extern "C" int skd_maxpool3x3s2_fwd(int N, int H, int W, int C, const float* x, float* y, unsigned char* argmax,
                                    cudaStream_t st) {
  if (C % 4) { set_error_msg("skd_maxpool3x3s2_fwd", "C % 4 != 0"); return 0; }
  const int OH = pool_out_ceil(H, 3, 2, 1), OW = pool_out_ceil(W, 3, 2, 1);
  maxpool_fwd_kernel<<<row_grid(N * OH, OW * (C / 4)), 256, 0, st>>>(x, y, argmax, N, H, W, C / 4, OH, OW);
  return finish("skd_maxpool3x3s2_fwd");
}

extern "C" int skd_maxpool3x3s2_bwd(int N, int H, int W, int C, const float* dy, const unsigned char* argmax, float* dx,
                                    cudaStream_t st) {
  if (C % 4) { set_error_msg("skd_maxpool3x3s2_bwd", "C % 4 != 0"); return 0; }
  const int OH = pool_out_ceil(H, 3, 2, 1), OW = pool_out_ceil(W, 3, 2, 1);
  maxpool_bwd_kernel<<<row_grid(N * H, W * (C / 4)), 256, 0, st>>>(dy, argmax, dx, N, H, W, C / 4, OH, OW);
  return finish("skd_maxpool3x3s2_bwd");
}

extern "C" long long skd_psp_pool_workspace_floats(int N, int H, int C, int levels, const int* sizes) {
  int nxb = 0;
  for (int i = 0; i < levels; ++i) nxb += sizes[i];
  return (long long)N * H * nxb * C;
}

extern "C" int skd_psp_pool_fwd(int N, int H, int W, int C, const float* x, int x_pitch, int levels, const int* sizes,
                                float* pooled, float* workspace, cudaStream_t st) {
  if (levels < 1 || levels > 4) { set_error_msg("skd_psp_pool_fwd", "1..4 pyramid levels"); return 0; }
  const Pyramid p = make_pyramid(levels, sizes);
  if (C % 4 || x_pitch % 4 || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(workspace) & 15)) {
    set_error_msg("skd_psp_pool_fwd", "C / pitch must be multiples of 4 floats and pointers 16-byte aligned"); return 0;
  }
  XBins xb; xb.n = 0;
  int lo[kMaxXBins], hi[kMaxXBins], pts[2 * kMaxXBins + 2], np = 0;
  for (int l = 0; l < levels; ++l)
    for (int b = 0; b < sizes[l]; ++b) {
      if (xb.n >= kMaxXBins) { set_error_msg("skd_psp_pool_fwd", "more than 16 x-bins over all levels"); return 0; }
      lo[xb.n] = (b * W) / sizes[l]; hi[xb.n] = ((b + 1) * W + sizes[l] - 1) / sizes[l];
      pts[np++] = lo[xb.n]; pts[np++] = hi[xb.n]; ++xb.n;
    }
  for (int i = 1; i < np; ++i) { const int v = pts[i]; int j = i - 1; while (j >= 0 && pts[j] > v) { pts[j + 1] = pts[j]; --j; } pts[j + 1] = v; }
  int nu = 0;
  for (int i = 0; i < np; ++i) if (nu == 0 || pts[i] != pts[nu - 1]) pts[nu++] = pts[i];
  if (nu - 1 > kMaxXSegs) { set_error_msg("skd_psp_pool_fwd", "more than 32 x segments"); return 0; }
  xb.nseg = nu - 1;
  for (int i = 0; i <= kMaxXSegs; ++i) xb.seg_lo[i] = pts[i < nu ? i : nu - 1];
  for (int b = 0; b < kMaxXBins; ++b) {
    xb.fs[b] = 0; xb.ls[b] = 0;
    if (b >= xb.n) continue;
    for (int i = 0; i < nu; ++i) { if (pts[i] == lo[b]) xb.fs[b] = i; if (pts[i] == hi[b]) xb.ls[b] = i; }
  }
  psp_rowbins_kernel<<<dim3(H, N, (C + 255) / 256), 256, 0, st>>>(x, x_pitch, C, H, W, xb, workspace);
  psp_colbins_kernel<<<dim3(p.first_bin[levels], N, (C + 255) / 256), 256, 0, st>>>(workspace, C, H, W, p, xb.n, pooled);
  return finish("skd_psp_pool_fwd", 2);
}

extern "C" int skd_psp_pool_bwd(int N, int H, int W, int C, const float* dpooled, int levels, const int* sizes, float* dx,
                                cudaStream_t st) {
  if (C % 4 || levels < 1 || levels > 4) { set_error_msg("skd_psp_pool_bwd", "C % 4 != 0 or bad levels"); return 0; }
  const Pyramid p = make_pyramid(levels, sizes);
  PyrBins pb; pb.levels = levels;
  for (int l = 0; l < 4; ++l) {
    pb.size[l] = l < levels ? sizes[l] : 1; pb.first_bin[l] = l < levels ? p.first_bin[l] : 0;
    if (pb.size[l] > 6) { set_error_msg("skd_psp_pool_bwd", "pyramid level size must be <= 6"); return 0; }
    for (int b = 0; b < 6; ++b) {
      const bool ok = l < levels && b < sizes[l];
      pb.lo_y[l][b] = ok ? (b * H) / sizes[l] : 0; pb.hi_y[l][b] = ok ? ((b + 1) * H + sizes[l] - 1) / sizes[l] : 0;
      pb.lo_x[l][b] = ok ? (b * W) / sizes[l] : 0; pb.hi_x[l][b] = ok ? ((b + 1) * W + sizes[l] - 1) / sizes[l] : 0;
    }
  }
  psp_pool_bwd_kernel<<<row_grid(N * H, W * (C / 4)), 256, 0, st>>>(dpooled, C / 4, H, W, N, pb, p.first_bin[levels], dx);
  return finish("skd_psp_pool_bwd");
}

extern "C" int skd_psp_upsample_fwd(int N, int H, int W, int C, int s, const float* src, int nbins_total, int first_bin,
                                    float* out, int out_pitch, int chan_off, cudaStream_t st) {
  if (C % 4 || out_pitch % 4 || chan_off % 4) { set_error_msg("skd_psp_upsample_fwd", "channel counts must be multiples of 4"); return 0; }
  psp_up_fwd_kernel<<<row_grid(N * H, W * (C / 4)), 256, 0, st>>>(src, C / 4, s, nbins_total, first_bin, out,
                                                                 out_pitch / 4, chan_off / 4, N, H, W);
  return finish("skd_psp_upsample_fwd");
}

extern "C" long long skd_psp_upsample_bwd_workspace_floats(int N, int H, int C, int s) { return (long long)N * H * s * C; }

extern "C" int skd_psp_upsample_bwd(int N, int H, int W, int C, int s, const float* dout, int dout_pitch, int chan_off,
                                    float* dsrc, int nbins_total, int first_bin, float* workspace, cudaStream_t st) {
  if (s < 1 || s > 6) { set_error_msg("skd_psp_upsample_bwd", "pyramid level size must be 1..6"); return 0; }
  psp_up_bwd_rows_kernel<<<dim3(H, N, (C + 63) / 64), 256, 0, st>>>(dout, dout_pitch, chan_off, C, s, workspace, H, W);
  psp_up_bwd_cols_kernel<<<dim3(s * s, N, (C + 255) / 256), 256, 0, st>>>(workspace, C, s, nbins_total, first_bin, dsrc, H);
  return finish("skd_psp_upsample_bwd", 2);
}

extern "C" int skd_slice_copy(long long rows, int C, const float* src, int src_pitch, int src_off, float* dst, int dst_pitch,
                              int dst_off, cudaStream_t st) {
  if ((C | src_pitch | src_off | dst_pitch | dst_off) % 4) { set_error_msg("skd_slice_copy", "multiples of 4 channels only"); return 0; }
  slice_copy_kernel<<<ew_blocks(rows * (C / 4)), 256, 0, st>>>(src, src_pitch / 4, src_off / 4, dst, dst_pitch / 4, dst_off / 4,
                                                              rows, C / 4);
  return finish("skd_slice_copy");
}

extern "C" int skd_sgd_step(long long n, float* param, const float* grad, float* momentum_buf, const float* lr, float momentum,
                            float weight_decay, int first_step, float grad_scale, cudaStream_t st) {
  if (n <= 0) return 1;
  const bool al = !((reinterpret_cast<uintptr_t>(param) | reinterpret_cast<uintptr_t>(grad) | reinterpret_cast<uintptr_t>(momentum_buf)) & 15);
  const long long n4 = al ? n / 4 : 0;
  sgd_kernel<<<ew_blocks(n / 4 + 1), 256, 0, st>>>(param, grad, momentum_buf, n4, n, lr, momentum, weight_decay, first_step, grad_scale);
  return finish("skd_sgd_step");
}

extern "C" int skd_sgd_step_nvls(long long lo, long long hi, float* param_mc, const float* grad_mc, const float* param_local, float* momentum_buf,
                                 const float* lr, float momentum, float weight_decay, float grad_scale, cudaStream_t st) {
  const char* who = "skd_sgd_step_nvls";
  if (hi <= lo) return 1;
  if ((lo | hi) & 3 || ((reinterpret_cast<uintptr_t>(param_mc) | reinterpret_cast<uintptr_t>(grad_mc) | reinterpret_cast<uintptr_t>(param_local) |
                         reinterpret_cast<uintptr_t>(momentum_buf)) & 15) || !param_mc || !grad_mc) {
    set_error_msg(who, "range bounds must be multiples of 4 floats, buffers 16-byte aligned, multicast addresses non-null"); return 0;
  }
  const long long n4 = (hi - lo) / 4;
  long long blocks = (n4 + 255) / 256;
  if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
  sgd_nvls_kernel<<<(int)blocks, 256, 0, st>>>(lo / 4, hi / 4, param_mc, grad_mc, param_local, momentum_buf, lr, momentum, weight_decay, grad_scale);
  return finish(who);
}
