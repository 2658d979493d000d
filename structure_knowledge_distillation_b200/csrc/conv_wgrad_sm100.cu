// wgmma weight-gradient convolution for sm_90a (cuDNN wgrad in the reference, reached through autograd of every
// nn.Conv2d of the student: networks/kd_model.py:150 G_loss.backward()).
//
//   dW[co][tap][ci] = sum_{pixels p} dY[p][co] * X[p shifted by tap][ci]
//
// GEMM view: M = Cout (128 per tile), N = Cin (<= 128 per tile, one filter tap per tile), K = pixels.  Both operands lie in HBM with
// the channels contiguous (NHWC), i.e. MN-major, and wgmma takes tf32 operands only K-major.  So per pipeline stage TMA drops
// 32-channel x 32-pixel boxes (128B-swizzled, one pixel per 128-byte row) of dY and X into a raw stage, the two consumer warpgroups
// transpose them into K-major 128B-swizzled tiles (one channel per 128-byte row, double-buffered so the transposition of the next
// K-block overlaps the wgmmas of this one) and release the raw stage at once; each warpgroup then issues 4 x wgmma.m64nNk8.tf32 for
// its 64 Cout rows.  Split-K over pixel blocks gives >= 2 waves of work units; fp32 partials go to a workspace and a deterministic
// reduction adds them in fixed order.
#include <cuda.h>

#include "common.cuh"
#include "skd.h"
#include "sm90_ptx.cuh"

using namespace skd;

namespace {

constexpr int kBlockM = 128;               // Cout per tile
constexpr int kKPix = 32;                  // pixels per pipeline stage (one 128-byte K row of the transposed tiles)
constexpr int kThreads = 384;              // producer warpgroup + 2 consumer warpgroups
constexpr int kChunkBytes = 32 * kKPix * 4;        // one 32-channel x 32-pixel box
constexpr int kMaxStages = 4;

struct WgArgs {
  int N, OH, OW, Cout, Cin, KH, KW, stride, pad, dil;
  int BHk, BWk, kb_x, kb_y;                // pixel K-blocks per image
  int m_tiles, n_tiles, taps, splits, kb_total, kb_per_split;
  float* ws;                               // [splits][Cout][taps*Cin]
  int linear;                              // K-blocks are 32 consecutive output pixels (dY as a [P][Cout] matrix, X through TMA im2col)
};

template <int BLOCK_N>
struct WCfg {
  static constexpr int kABytes = 4 * kChunkBytes;                    // 128 co
  static constexpr int kBBytes = (BLOCK_N / 32) * kChunkBytes;
  static constexpr int kStageBytes = kABytes + kBBytes;              // raw (pixel-major) stage; the transposed set has the same size
  static constexpr int kFit = (232448 - 2 * kStageBytes - 1024 - 256) / kStageBytes;
  static constexpr int kStages = kFit > kMaxStages ? kMaxStages : kFit;
  static constexpr int kSmemBytes = (kStages + 2) * kStageBytes + 1024 + 256;
  static_assert(kStages >= 2, "at least two pipeline stages");
};

// raw box (pixel rows of 32 channels, 128B swizzle) -> K-major tile (channel rows of 32 pixels, 128B swizzle); unit = 4 pixels x 4 channels
__device__ __forceinline__ void transpose_tile(const uint8_t* raw, uint8_t* dst, int rows, int t) {
  for (int u = t; u < rows * 2; u += 256) {
    const int pg = u & 7, cg = u >> 3;
    const uint8_t* src = raw + (cg >> 3) * kChunkBytes;
    float4 r[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int p = 4 * pg + i;
      r[i] = *reinterpret_cast<const float4*>(src + p * 128 + ((((cg & 7) ^ (p & 7))) << 4));
    }
    const int c = 4 * cg;
    *reinterpret_cast<float4*>(dst + (c + 0) * 128 + ((pg ^ ((c + 0) & 7)) << 4)) = make_float4(r[0].x, r[1].x, r[2].x, r[3].x);
    *reinterpret_cast<float4*>(dst + (c + 1) * 128 + ((pg ^ ((c + 1) & 7)) << 4)) = make_float4(r[0].y, r[1].y, r[2].y, r[3].y);
    *reinterpret_cast<float4*>(dst + (c + 2) * 128 + ((pg ^ ((c + 2) & 7)) << 4)) = make_float4(r[0].z, r[1].z, r[2].z, r[3].z);
    *reinterpret_cast<float4*>(dst + (c + 3) * 128 + ((pg ^ ((c + 3) & 7)) << 4)) = make_float4(r[0].w, r[1].w, r[2].w, r[3].w);
  }
}

template <int BLOCK_N>
__global__ void __launch_bounds__(kThreads, 1)
conv_wgrad_sm90_kernel(const __grid_constant__ CUtensorMap tmap_dy, const __grid_constant__ CUtensorMap tmap_x, const WgArgs a) {
  using C = WCfg<BLOCK_N>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // keep the pointer in the shared address space (integer round trips make nvcc emit generic LD/ST instead of LDS/STS)
  const uint32_t raw_addr = ptx::smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
  uint8_t* sets = smem + C::kStages * C::kStageBytes;                // 2 transposed {A, B} sets
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sets + 2 * C::kStageBytes);
  uint64_t* empty_bar = full_bar + kMaxStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmap_dy); ptx::prefetch_tmap(&tmap_x);
    for (int s = 0; s < C::kStages; ++s) { ptx::mbar_init(&full_bar[s], 1); ptx::mbar_init(&empty_bar[s], 1); }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  const int tiles = a.m_tiles * a.taps * a.n_tiles;
  const int units = tiles * a.splits;
  const int kb_per_img = a.kb_x * a.kb_y;

  if (warp < 4) {
    // ===================== TMA producer =====================
    // all-out-of-range channel chunks (Cout or Cin < tile) are not issued
    if (threadIdx.x == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int u = blockIdx.x; u < units; u += gridDim.x) {
        const int split = u / tiles, tile = u - split * tiles;
        const int mt = tile / (a.taps * a.n_tiles), r = tile - mt * (a.taps * a.n_tiles);
        const int tap = r / a.n_tiles, nt = r - tap * a.n_tiles;
        const int kh = tap / a.KW, kw = tap - kh * a.KW;
        const int kb0 = split * a.kb_per_split;
        const int kb1 = min(a.kb_total, kb0 + a.kb_per_split);
        const int a_chunks = min(4, (a.Cout - mt * kBlockM + 31) / 32);
        const int b_chunks = max(0, min(BLOCK_N / 32, (a.Cin - nt * BLOCK_N + 31) / 32));
        for (int kb = kb0; kb < kb1; ++kb) {
          ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * C::kStageBytes;
          uint8_t* sb = sa + C::kABytes;
          ptx::mbar_expect_tx(&full_bar[stage], (uint32_t)((a_chunks + b_chunks) * kChunkBytes));
          if (a.linear) {
            const int p0 = kb * kKPix;
            const int img = p0 / (a.OH * a.OW), r2 = p0 - img * (a.OH * a.OW);
            const int oy = r2 / a.OW, ox = r2 - oy * a.OW;
            for (int c = 0; c < a_chunks; ++c)
              ptx::tma_load_4d(sa + c * kChunkBytes, &tmap_dy, &full_bar[stage], mt * kBlockM + c * 32, p0, 0, 0);
            for (int c = 0; c < b_chunks; ++c)
              ptx::tma_load_im2col_4d(sb + c * kChunkBytes, &tmap_x, &full_bar[stage], nt * BLOCK_N + c * 32, ox * a.stride - a.pad,
                                      oy * a.stride - a.pad, img, (uint16_t)(kw * a.dil), (uint16_t)(kh * a.dil));
          } else {
            const int img = kb / kb_per_img, q = kb - img * kb_per_img;
            const int by = q / a.kb_x, bx = q - by * a.kb_x;
            const int oy0 = by * a.BHk, ox0 = bx * a.BWk;
            for (int c = 0; c < a_chunks; ++c)
              ptx::tma_load_4d(sa + c * kChunkBytes, &tmap_dy, &full_bar[stage], mt * kBlockM + c * 32, ox0, oy0, img);
            for (int c = 0; c < b_chunks; ++c)
              ptx::tma_load_4d(sb + c * kChunkBytes, &tmap_x, &full_bar[stage], nt * BLOCK_N + c * 32,
                               ox0 * a.stride - a.pad + kw * a.dil, oy0 * a.stride - a.pad + kh * a.dil, img);
          }
          if (++stage == C::kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers =====================
    const int t = threadIdx.x - 128;                           // 0..255
    const int g = t >> 7;                                      // warpgroup: Cout rows 64g .. 64g+63 of the tile
    const int wq = warp & 3;
    const int r_lo = g * 64 + wq * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);
    const size_t kdim = (size_t)a.taps * a.Cin;
    float acc[BLOCK_N / 2];
    int stage = 0; uint32_t phase = 0; uint32_t it = 0;        // it: K-blocks consumed so far (transposed-set parity)
    for (int u = blockIdx.x; u < units; u += gridDim.x) {
      const int split = u / tiles, tile = u - split * tiles;
      const int mt = tile / (a.taps * a.n_tiles), r = tile - mt * (a.taps * a.n_tiles);
      const int tap = r / a.n_tiles, nt = r - tap * a.n_tiles;
      const int kb0 = split * a.kb_per_split;
      const int nkb = min(a.kb_total, kb0 + a.kb_per_split) - kb0;
      for (int k = 0; k < nkb; ++k, ++it) {
        uint8_t* set = sets + (it & 1) * C::kStageBytes;
        ptx::mbar_wait(&full_bar[stage], phase);
        ptx::wgmma_wait<1>();                                  // this warpgroup's wgmmas of two K-blocks ago (same set) are done
        ptx::named_bar_sync(1, 256);                           // ... and the other warpgroup's
        const uint8_t* raw = smem + stage * C::kStageBytes;
        transpose_tile(raw, set, kBlockM, t);
        transpose_tile(raw + C::kABytes, set + C::kABytes, BLOCK_N, t);
        ptx::fence_proxy_async();                              // generic-proxy writes -> visible to the wgmma (async proxy) reads
        ptx::named_bar_sync(1, 256);
        if (t == 0) ptx::mbar_arrive(&empty_bar[stage]);       // raw stage consumed
        const uint32_t sa = ptx::smem_u32(set) + (uint32_t)(g * 64 * 128);
        const uint32_t sb = ptx::smem_u32(set) + (uint32_t)C::kABytes;
        ptx::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kKPix / 8; ++kk)
          ptx::wgmma_tf32<BLOCK_N>(acc, ptx::make_wgmma_desc_sw128(sa + kk * 32), ptx::make_wgmma_desc_sw128(sb + kk * 32), (k | kk) != 0 ? 1u : 0u);
        ptx::wgmma_commit();
        if (++stage == C::kStages) { stage = 0; phase ^= 1; }
      }
      ptx::wgmma_wait<0>();
      ptx::fence_regs(acc);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int co = mt * kBlockM + r_lo + 8 * h;
        if (co >= a.Cout) continue;
        float* orow = a.ws + ((size_t)split * a.Cout + co) * kdim + (size_t)tap * a.Cin;
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const int ci = nt * BLOCK_N + 8 * j + cq;            // even; Cin % 4 == 0, so ci + 1 < Cin too
          if (ci < a.Cin) *reinterpret_cast<float2*>(orow + ci) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256)
splitk_reduce_kernel(const float* __restrict__ ws, float* __restrict__ dw, long long n4, int splits) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 a = reinterpret_cast<const float4*>(ws)[i];
    for (int s = 1; s < splits; ++s) {
      const float4 b = reinterpret_cast<const float4*>(ws)[(long long)s * n4 + i];
      a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    }
    reinterpret_cast<float4*>(dw)[i] = a;
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr; static bool tried = false;
  if (!tried) {
    tried = true; void* p = nullptr; cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

struct Plan { int OH, OW, BHk, BWk, kb_x, kb_y, kb_total, bn, m_tiles, n_tiles, taps, splits, kb_per_split, linear; };

int g_wgrad_linear = 1;

Plan make_plan(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil) {
  Plan p;
  p.OH = (H + 2 * pad - dil * (KH - 1) - 1) / stride + 1; p.OW = (W + 2 * pad - dil * (KW - 1) - 1) / stride + 1;
  const int cand[4][2] = {{4, 8}, {8, 4}, {2, 16}, {1, 32}};        // 32-pixel K blocks in the rectangular fallback mode
  long long best = -1;
  for (auto& c : cand) {
    const long long t = (long long)((p.OH + c[0] - 1) / c[0]) * ((p.OW + c[1] - 1) / c[1]);
    if (best < 0 || t < best) { best = t; p.BHk = c[0]; p.BWk = c[1]; }
  }
  p.bn = Cin > 64 ? 128 : (Cin > 32 ? 64 : 32);
  p.kb_x = (p.OW + p.BWk - 1) / p.BWk; p.kb_y = (p.OH + p.BHk - 1) / p.BHk;
  p.kb_total = N * p.kb_x * p.kb_y;
  const int up_h = pad - (KH - 1) * dil, up_w = pad - (KW - 1) * dil;
  p.linear = g_wgrad_linear && pad <= 128 && up_h >= -128 && up_w >= -128 && stride <= 8 && (long long)N * p.OH * p.OW < (1LL << 31);
  if (p.linear) p.kb_total = (int)(((long long)N * p.OH * p.OW + kKPix - 1) / kKPix);
  p.m_tiles = (Cout + kBlockM - 1) / kBlockM; p.n_tiles = (Cin + p.bn - 1) / p.bn; p.taps = KH * KW;
  const int tiles = p.m_tiles * p.n_tiles * p.taps;
  const int slots = kNumSMs;                                 // persistent CTAs
  // split-K: work units = tiles x K ranges over a persistent grid of kNumSMs CTAs.  Pick the split count whose unit count fills
  // whole waves best (a unit count just past a whole number of waves leaves
  // most SMs idle in the last round), fewer splits on ties (each split writes a partial dW plane)
  int cap = p.kb_total / 16; if (cap < 1) cap = 1;          // at least 16 k-blocks per unit
  int hi = (4 * slots + tiles - 1) / tiles; if (hi > cap) hi = cap; if (hi < 1) hi = 1;
  int best_sp = 1; double best_eff = -1.0;
  for (int sp = 1; sp <= hi; ++sp) {
    const int kps = (p.kb_total + sp - 1) / sp;
    const int real = (p.kb_total + kps - 1) / kps;             // splits that actually get work
    const long long units = (long long)tiles * real;
    const long long waves = (units + slots - 1) / slots;
    double eff = (double)units / (double)(waves * slots);
    if (units < slots) eff = (double)units / slots * 0.999;       // less than one wave: more units is better
    if (eff > best_eff + 0.02) { best_eff = eff; best_sp = real; }
  }
  int splits = best_sp;
  p.kb_per_split = (p.kb_total + splits - 1) / splits;
  p.splits = (p.kb_total + p.kb_per_split - 1) / p.kb_per_split;
  return p;
}

template <int BLOCK_N>
int launch(const CUtensorMap& tdy, const CUtensorMap& tx, const WgArgs& a, int units, cudaStream_t st) {
  using C = WCfg<BLOCK_N>;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(conv_wgrad_sm90_kernel<BLOCK_N>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmemBytes);
    if (e != cudaSuccess) { set_error("skd_conv2d_wgrad_sm100(attr)", e); return 0; }
    attr = true;
  }
  const int grid = units < kNumSMs ? units : kNumSMs;
  conv_wgrad_sm90_kernel<BLOCK_N><<<grid, kThreads, C::kSmemBytes, st>>>(tdy, tx, a);
  return finish("skd_conv2d_wgrad_sm100");
}

}  // namespace

extern "C" void skd_set_wgrad_linear(int on) { g_wgrad_linear = on ? 1 : 0; }

extern "C" long long skd_conv2d_wgrad_sm100_workspace_floats(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride,
                                                             int pad, int dil) {
  const Plan p = make_plan(N, H, W, Cin, Cout, KH, KW, stride, pad, dil);
  return (long long)p.splits * Cout * KH * KW * Cin;
}

extern "C" int skd_conv2d_wgrad_sm100(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil,
                                      const float* x, int ldx, const float* dy, int ldy, float* dw, float* workspace,
                                      cudaStream_t st) {
  const char* who = "skd_conv2d_wgrad_sm100";
  if (Cin % 4 || Cout % 4 || ldx % 4 || ldy % 4 || ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dy) |
                                                     reinterpret_cast<uintptr_t>(dw) | reinterpret_cast<uintptr_t>(workspace)) & 15)) {
    set_error_msg(who, "channel counts / pitches must be multiples of 4 floats and pointers 16-byte aligned (TMA)");
    return 0;
  }
  const Plan p = make_plan(N, H, W, Cin, Cout, KH, KW, stride, pad, dil);
  if (p.OH <= 0 || p.OW <= 0 || N <= 0) return 1;
  EncodeTiledFn enc = get_encode();
  if (!enc) { set_error_msg(who, "cuTensorMapEncodeTiled unavailable (no CUDA driver)"); return 0; }
  const CUtensorMapDataType dt = skd::g_tf32_tma_type ? CU_TENSOR_MAP_DATA_TYPE_TFLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  CUtensorMap tdy, tx;
  if (p.linear) {
    typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const int*,
                                       const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                       CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static EncodeIm2colFn enc_i2c = nullptr;
    if (!enc_i2c) {
      void* fp = nullptr; cudaDriverEntryPointQueryResult q;
      if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &fp, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
        enc_i2c = reinterpret_cast<EncodeIm2colFn>(fp);
    }
    if (!enc_i2c) { set_error_msg(who, "cuTensorMapEncodeIm2col unavailable"); return 0; }
    const long long P = (long long)N * p.OH * p.OW;
    {
      cuuint64_t dims[4] = {(cuuint64_t)Cout, (cuuint64_t)P, 1, 1};
      cuuint64_t strides[3] = {(cuuint64_t)ldy * 4, (cuuint64_t)P * ldy * 4, (cuuint64_t)P * ldy * 4};
      cuuint32_t box[4] = {32, (cuuint32_t)kKPix, 1, 1};
      cuuint32_t es[4] = {1, 1, 1, 1};
      CUresult r = enc(&tdy, dt, 4, const_cast<float*>(dy), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                       CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) { set_error_msg(who, "cuTensorMapEncodeTiled(dy, linear) failed"); return 0; }
    }
    {
      cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
      cuuint64_t strides[3] = {(cuuint64_t)ldx * 4, (cuuint64_t)W * ldx * 4, (cuuint64_t)H * W * ldx * 4};
      int lower[2] = {-pad, -pad};
      int upper[2] = {pad - (KW - 1) * dil, pad - (KH - 1) * dil};
      cuuint32_t es[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
      CUresult r = enc_i2c(&tx, dt, 4, const_cast<float*>(x), dims, strides, lower, upper, 32, (cuuint32_t)kKPix, es,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) { set_error_msg(who, "cuTensorMapEncodeIm2col(x) failed"); return 0; }
    }
  } else {
  {
    cuuint64_t dims[4] = {(cuuint64_t)Cout, (cuuint64_t)p.OW, (cuuint64_t)p.OH, (cuuint64_t)N};
    cuuint64_t strides[3] = {(cuuint64_t)ldy * 4, (cuuint64_t)p.OW * ldy * 4, (cuuint64_t)p.OH * p.OW * ldy * 4};
    cuuint32_t box[4] = {32, (cuuint32_t)p.BWk, (cuuint32_t)p.BHk, 1};
    cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult r = enc(&tdy, dt, 4, const_cast<float*>(dy), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error_msg(who, "cuTensorMapEncodeTiled(dy) failed"); return 0; }
  }
  {
    cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t strides[3] = {(cuuint64_t)ldx * 4, (cuuint64_t)W * ldx * 4, (cuuint64_t)H * W * ldx * 4};
    cuuint32_t box[4] = {32, (cuuint32_t)(p.BWk * stride), (cuuint32_t)(p.BHk * stride), 1};
    cuuint32_t es[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
    CUresult r = enc(&tx, dt, 4, const_cast<float*>(x), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error_msg(who, "cuTensorMapEncodeTiled(x) failed"); return 0; }
  }
  }
  WgArgs a;
  a.N = N; a.OH = p.OH; a.OW = p.OW; a.Cout = Cout; a.Cin = Cin; a.KH = KH; a.KW = KW; a.stride = stride; a.pad = pad; a.dil = dil;
  a.BHk = p.BHk; a.BWk = p.BWk; a.kb_x = p.kb_x; a.kb_y = p.kb_y; a.m_tiles = p.m_tiles; a.n_tiles = p.n_tiles; a.taps = p.taps;
  a.splits = p.splits; a.kb_total = p.kb_total; a.kb_per_split = p.kb_per_split;
  a.ws = p.splits == 1 ? dw : workspace;
  a.linear = p.linear;
  const int units = p.m_tiles * p.n_tiles * p.taps * p.splits;
  int ok;
  switch (p.bn) {
    case 128: ok = launch<128>(tdy, tx, a, units, st); break;
    case 64: ok = launch<64>(tdy, tx, a, units, st); break;
    default: ok = launch<32>(tdy, tx, a, units, st); break;
  }
  if (!ok) return 0;
  if (p.splits > 1) {
    const long long n4 = (long long)Cout * KH * KW * Cin / 4;
    long long b = (n4 + 255) / 256; if (b > kNumSMs * 8) b = kNumSMs * 8; if (b < 1) b = 1;
    splitk_reduce_kernel<<<(int)b, 256, 0, st>>>(workspace, dw, n4, p.splits);
  }
  return finish(who);
}
