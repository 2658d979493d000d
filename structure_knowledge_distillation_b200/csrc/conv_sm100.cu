// wgmma implicit-GEMM 2-D convolution for sm_90a (replaces every cuDNN nn.Conv2d call of
// networks/pspnet_combine.py on the hot path: forward here; dgrad reuses this kernel on the output gradient with
// flipped/transposed weights; wgrad is conv_wgrad_sm100.cu).
//
//   D[M = N*OH*OW pixels][Cout] = sum_{tap, ci}  X[pixel shifted by tap][ci] * W[Cout][tap][ci]
//
// Layout: activations NHWC fp32 (row pitch ld*, so channel slices of a concat buffer are addressable in place),
// weights [Cout][KH][KW][Cin] (K-major), fp32 storage, TF32 tensor-core math with fp32 accumulation in registers.
//
// One persistent CTA per SM, three warpgroups:
//   warpgroup 0     TMA producer (one thread): per (tap, 32-channel chunk) one A box of X -- 128 consecutive output pixels in TMA
//                   im2col mode (tap shift / padding / stride / dilation in the tensor map, out-of-bounds = hardware zero fill),
//                   a flat [pixels][C] box for 1x1 convs, or a BH x BW rectangle in tiled mode -- plus one 3-D box
//                   {32ch, 1 tap, BLOCK_N} of W, both 128B-swizzled K-major, landing on a full[] mbarrier of a multi-stage ring.
//                   Split precision (3xTF32): the stage also holds the low parts of both operands.
//   warpgroups 1-2  consumers: warpgroup g owns GEMM rows 64g .. 64g+63 of the 128-pixel tile; 4 x wgmma.m64nNk8.tf32 per stage
//                   (x3 for split precision), accumulator in registers, the stage released one stage later (one wgmma batch in
//                   flight); epilogue straight from the registers: per-channel scale/shift (folded BN or bias), residual add,
//                   ReLU / leaky-ReLU / ELU, optional TF32 rounding and fused sum of squares, global stores.
#include <cuda.h>

#include "common.cuh"
#include "skd.h"
#include "sm90_ptx.cuh"

using namespace skd;

namespace {

constexpr int kBlockM = 128;
constexpr int kBlockK = 32;                 // fp32 elements = 128 B = one swizzle row
constexpr int kWgmmaK = 8;                  // tf32
constexpr int kThreads = 384;               // producer warpgroup + 2 consumer warpgroups
constexpr int kABytes = kBlockM * kBlockK * 4;

struct ConvArgs {
  int N, OH, OW, Cout, Cin;
  int KH, KW, stride, pad, dil;
  int BH, BW, tiles_x, tiles_y;
  int m_tiles, n_tiles, k_chunks;
  float* y; int ldy; long long y_row, y_img;   // output element (img, oy, ox, c) at y[img * y_img + oy * y_row + ox * ldy + c]
  const float* scale; const float* shift;
  const float* residual; int ldr;
  int act; float slope; int round_out;
  double* sumsq;                   // optional: += sum of squares of every valid output element (fused L2 reduction)
  int no_store;                    // 1: the output tensor is not written at all (reduction-only epilogue)
  int nstages;                     // A/B pipeline stages in use
  int kc_outer;                    // K loop order: 1 = channel chunk outermost / taps innermost, 0 = taps outermost
  int reverse;                     // walk the tile list back to front (alternated per layer so a layer starts on the
                                   // activations its producer wrote last, which are still in L2)
  int im2col, rOH, rOW;            // im2col mode: M tiles are 128 consecutive output pixels of the real (rOH x rOW) maps
  int splits, k_per_split;         // split-K (few tiles, long K: the discriminator's 4x4 convolutions on 4x8 .. 16x32 maps): unit = (tile, K range),
  long long split_stride;          //   raw fp32 partials go to y + split * split_stride; splitk_epilogue_kernel adds them and applies the epilogue
};

template <int BLOCK_N, bool SPLIT>
struct Cfg {
  static constexpr int kBBytes = BLOCK_N * kBlockK * 4;
  static constexpr int kStageBytes = (kABytes + kBBytes) * (SPLIT ? 2 : 1);   // split precision: {x_hi, w_hi, x_lo, w_lo}
  static constexpr int kFixedBytes = 1024 /*align slack*/ + 256 /*barriers*/;
  static constexpr int kFit = (232448 - kFixedBytes) / kStageBytes;
  static constexpr int kStages = kFit > 8 ? 8 : kFit;
  static constexpr int kSmemBytes = kStages * kStageBytes + kFixedBytes;
  static_assert(kStages >= 2, "at least two pipeline stages");
  static_assert(kSmemBytes <= 232448, "exceeds the 227 KB of shared memory a CTA may use");
};

__device__ __forceinline__ float epi_act(float v, int act, float slope) {
  if (act == ACT_RELU) return fmaxf(v, 0.f);
  if (act == ACT_LEAKY) return v < 0.f ? v * slope : v;
  if (act == ACT_ELU) return v < 0.f ? expm1f(v) : v;
  return v;
}

template <int BLOCK_N, bool SPLIT>
__global__ void __launch_bounds__(kThreads, 1)
conv_fwd_sm90_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                     const __grid_constant__ CUtensorMap tmap_x2, const __grid_constant__ CUtensorMap tmap_w2, const ConvArgs a) {
  using C = Cfg<BLOCK_N, SPLIT>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // keep the pointer in the shared address space (integer round trips make nvcc emit generic LD/ST instead of LDS/STS)
  const uint32_t raw_addr = ptx::smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C::kStages * C::kStageBytes);
  uint64_t* empty_bar = full_bar + C::kStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmap_x);
    ptx::prefetch_tmap(&tmap_w);
    for (int s = 0; s < C::kStages; ++s) { ptx::mbar_init(&full_bar[s], 1); ptx::mbar_init(&empty_bar[s], 8); }   // one arrival per consumer warp
    ptx::fence_barrier_init();
  }
  __syncthreads();

  const int total_tiles = a.m_tiles * a.n_tiles * a.splits;     // work units: (tile, K range); the K ranges of a tile are consecutive units
  const int taps = a.KH * a.KW;
  const int k_iters = taps * a.k_chunks;
  const int tiles_per_img = a.tiles_x * a.tiles_y;

  if (warp < 4) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int tu = a.reverse ? total_tiles - 1 - tile : tile;
        const int tl = tu / a.splits, sp = tu - tl * a.splits;
        const int mt = tl / a.n_tiles, nt = tl - mt * a.n_tiles;
        const int img = mt / tiles_per_img, rem = mt - img * tiles_per_img;
        const int ty = rem / a.tiles_x, tx = rem - ty * a.tiles_x;
        const int iy0 = ty * a.BH * a.stride - a.pad, ix0 = tx * a.BW * a.stride - a.pad;
        // im2col: first output pixel of the tile (n, p, q) -> filter-origin input coordinates
        int in0 = 0, ip0 = 0, iq0 = 0;
        if (a.im2col) {
          const int m0 = mt * kBlockM;
          in0 = m0 / (a.rOH * a.rOW);
          const int r2 = m0 - in0 * (a.rOH * a.rOW);
          ip0 = (r2 / a.rOW) * a.stride - a.pad;
          iq0 = (r2 % a.rOW) * a.stride - a.pad;
        }
        // kc_outer: channel chunk outermost, filter taps innermost -- the taps of one chunk re-read (shifted) the same input lines,
        // L2 hits whatever Cin is; taps outermost streams Cin * 128 pixels per CTA between reuses.
        const int n_inner = a.kc_outer ? taps : a.k_chunks;
        const int k0 = sp * a.k_per_split, k1 = min(k_iters, k0 + a.k_per_split);
        for (int k = k0; k < k1; ++k) {
          const int io = k / n_inner, ii = k - io * n_inner;
          const int kc = a.kc_outer ? io : ii, tap = a.kc_outer ? ii : io;
          const int kh = tap / a.KW, kw = tap - kh * a.KW;
          ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * C::kStageBytes;
          ptx::mbar_expect_tx(&full_bar[stage], (uint32_t)C::kStageBytes);
#pragma unroll
          for (int part = 0; part < (SPLIT ? 2 : 1); ++part) {
            const CUtensorMap* mx = part ? &tmap_x2 : &tmap_x;
            const CUtensorMap* mw = part ? &tmap_w2 : &tmap_w;
            uint8_t* pa = sa + part * (kABytes + C::kBBytes);
            uint8_t* pb = pa + kABytes;
            if (a.im2col)
              ptx::tma_load_im2col_4d(pa, mx, &full_bar[stage], kc * kBlockK, iq0, ip0, in0, (uint16_t)(kw * a.dil), (uint16_t)(kh * a.dil));
            else
              ptx::tma_load_4d(pa, mx, &full_bar[stage], kc * kBlockK, ix0 + kw * a.dil, iy0 + kh * a.dil, img);
            ptx::tma_load_3d(pb, mw, &full_bar[stage], kc * kBlockK, tap, nt * BLOCK_N);
          }
          if (++stage == a.nstages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers: warpgroup g = rows 64g .. 64g+63 of the tile =====================
    const int g = (warp >> 2) - 1;
    const int wq = warp & 3;
    const int r_lo = g * 64 + wq * 16 + (lane >> 2);          // tile rows of this thread's fragment: r_lo and r_lo + 8
    const int cq = 2 * (lane & 3);                             // first of the thread's two columns in every 8-column group
    constexpr int R = BLOCK_N / 2;
    float acc[R];
    float tot[SPLIT ? R : 1];
    double sq_acc = 0.0;
    int stage = 0; uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int tu = a.reverse ? total_tiles - 1 - tile : tile;
      const int tl = tu / a.splits, sp = tu - tl * a.splits;
      const int mt = tl / a.n_tiles, nt = tl - mt * a.n_tiles;
      const int nk = min(k_iters, (sp + 1) * a.k_per_split) - sp * a.k_per_split;      // K steps of this unit
      if constexpr (SPLIT) {
#pragma unroll
        for (int i = 0; i < R; ++i) tot[i] = 0.f;
      }
      int prev_stage = -1;
      for (int k = 0; k < nk; ++k) {
        ptx::mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = ptx::smem_u32(smem + stage * C::kStageBytes) + (uint32_t)(g * 64 * 128);
        const uint32_t sb = ptx::smem_u32(smem + stage * C::kStageBytes) + (uint32_t)kABytes;
        ptx::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kBlockK / kWgmmaK; ++kk) {
          const uint64_t da = ptx::make_wgmma_desc_sw128(sa + kk * kWgmmaK * 4);
          const uint64_t db = ptx::make_wgmma_desc_sw128(sb + kk * kWgmmaK * 4);
          if constexpr (SPLIT) {
            // split precision: this stage's x_hi*w_hi + x_lo*w_hi + x_hi*w_lo in a fresh accumulator, added to the running total with
            // round-to-nearest fp32 adds below (the tensor core truncates on every accumulate: over hundreds of K steps that, not the
            // operand split, would limit the "fp32-grade" layers)
            constexpr uint32_t kLo = kABytes + C::kBBytes;
            ptx::wgmma_tf32<BLOCK_N>(acc, da, db, kk != 0 ? 1u : 0u);
            ptx::wgmma_tf32<BLOCK_N>(acc, ptx::make_wgmma_desc_sw128(sa + kLo + kk * kWgmmaK * 4), db, 1u);
            ptx::wgmma_tf32<BLOCK_N>(acc, da, ptx::make_wgmma_desc_sw128(sb + kLo + kk * kWgmmaK * 4), 1u);
          } else {
            ptx::wgmma_tf32<BLOCK_N>(acc, da, db, (k | kk) != 0 ? 1u : 0u);
          }
        }
        ptx::wgmma_commit();
        if constexpr (SPLIT) {
          ptx::wgmma_wait<0>();
          ptx::fence_regs(acc);
#pragma unroll
          for (int i = 0; i < R; ++i) tot[i] += acc[i];
          if (lane == 0) ptx::mbar_arrive(&empty_bar[stage]);
        } else {
          ptx::wgmma_wait<1>();                                  // the previous stage's wgmmas are done: release its buffers
          if (prev_stage >= 0 && lane == 0) ptx::mbar_arrive(&empty_bar[prev_stage]);
          prev_stage = stage;
        }
        if (++stage == a.nstages) { stage = 0; phase ^= 1; }
      }
      if constexpr (!SPLIT) {
        ptx::wgmma_wait<0>();
        ptx::fence_regs(acc);
        if (prev_stage >= 0 && lane == 0) ptx::mbar_arrive(&empty_bar[prev_stage]);
      }
      if constexpr (SPLIT) {
#pragma unroll
        for (int i = 0; i < R; ++i) acc[i] = tot[i];
      }
      const float* v = acc;

      // ---- epilogue straight from the fragment ----
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = r_lo + 8 * h;
        const int img = mt / tiles_per_img, rem = mt - img * tiles_per_img;
        const int ty = rem / a.tiles_x, tx = rem - ty * a.tiles_x;
        const int dy = row / a.BW, dx = row - dy * a.BW;
        const int oy = ty * a.BH + dy, ox = tx * a.BW + dx;
        if (oy >= a.OH || ox >= a.OW) continue;
        float* yrow = a.y + (size_t)sp * a.split_stride + (size_t)img * a.y_img + (size_t)oy * a.y_row + (size_t)ox * a.ldy;
        const float* rrow = a.residual ? a.residual + (((size_t)img * a.OH + oy) * a.OW + ox) * a.ldr : nullptr;
        float part = 0.f;
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const int c = nt * BLOCK_N + 8 * j + cq;
          if (c >= a.Cout) continue;
          const bool two = c + 1 < a.Cout;
          float v0 = v[4 * j + 2 * h], v1 = v[4 * j + 2 * h + 1];
          if (a.scale) { v0 *= __ldg(a.scale + c); if (two) v1 *= __ldg(a.scale + c + 1); }
          if (a.shift) { v0 += __ldg(a.shift + c); if (two) v1 += __ldg(a.shift + c + 1); }
          if (rrow) { v0 += __ldg(rrow + c); if (two) v1 += __ldg(rrow + c + 1); }
          v0 = epi_act(v0, a.act, a.slope); v1 = epi_act(v1, a.act, a.slope);
          if (a.round_out) { v0 = ptx::round_tf32(v0); v1 = ptx::round_tf32(v1); }
          if (a.sumsq) part = fmaf(v0, v0, two ? fmaf(v1, v1, part) : part);
          if (a.no_store) continue;
          if (two && !((reinterpret_cast<uintptr_t>(yrow + c)) & 7)) {
            *reinterpret_cast<float2*>(yrow + c) = make_float2(v0, v1);
          } else {
            yrow[c] = v0;
            if (two) yrow[c + 1] = v1;
          }
        }
        sq_acc += (double)part;                                 // fp32 within a row of the tile, fp64 across rows and tiles
      }
    }
    if (a.sumsq) {
      for (int o = 16; o > 0; o >>= 1) sq_acc += __shfl_xor_sync(0xffffffffu, sq_acc, o);
      if (lane == 0) atomicAdd(a.sumsq, sq_acc);
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const int*,
                                   const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeIm2colFn get_encode_im2col() {
  static EncodeIm2colFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeIm2colFn>(p);
  }
  return fn;
}
int g_conv_im2col = 1;
int g_tile_order = 0;             // 0 front-to-back, 1 back-to-front, 2 alternate per launch
int g_tile_flip = 0;
int g_k_order = 0;                // 0: by working set (channel chunks outermost when Cin >= 2048); 1: taps outermost; 2: chunks outermost

EncodeTiledFn get_encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}


bool encode(CUtensorMap* m, int rank, const void* base, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
            const cuuint32_t* box, const cuuint32_t* estr, const char* who) {
  EncodeTiledFn fn = get_encode_tiled();
  if (!fn) { set_error_msg(who, "cuTensorMapEncodeTiled unavailable (no CUDA driver)"); return false; }
  CUresult r = fn(m, g_tf32_tma_type ? CU_TENSOR_MAP_DATA_TYPE_TFLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank,
                  const_cast<void*>(base), dims, strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[160];
    snprintf(buf, sizeof buf, "cuTensorMapEncodeTiled failed (CUresult %d)", (int)r);
    set_error_msg(who, buf);
    return false;
  }
  return true;
}

void pick_rect(int OH, int OW, int stride, int* BH, int* BW) {
  const int cand[6][2] = {{8, 16}, {4, 32}, {16, 8}, {2, 64}, {32, 4}, {1, 128}};
  long long best = -1;
  for (auto& c : cand) {
    if (c[0] * stride > 256 || c[1] * stride > 256) continue;
    const long long t = (long long)((OH + c[0] - 1) / c[0]) * ((OW + c[1] - 1) / c[1]);
    if (best < 0 || t < best) { best = t; *BH = c[0]; *BW = c[1]; }
  }
}

template <int BLOCK_N, bool SPLIT>
int launch(const CUtensorMap& tx, const CUtensorMap& tw, const CUtensorMap& tx2, const CUtensorMap& tw2, const ConvArgs& a_in, cudaStream_t st) {
  using C = Cfg<BLOCK_N, SPLIT>;
  ConvArgs a = a_in;
  a.nstages = C::kStages;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(conv_fwd_sm90_kernel<BLOCK_N, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmemBytes);
    if (e != cudaSuccess) { set_error("skd_conv2d_fwd_sm100(attr)", e); return 0; }
    attr = true;
  }
  int grid = a.m_tiles * a.n_tiles * a.splits;
  if (grid > kNumSMs) grid = kNumSMs;
  conv_fwd_sm90_kernel<BLOCK_N, SPLIT><<<grid, kThreads, C::kSmemBytes, st>>>(tx, tw, tx2, tw2, a);
  return finish("skd_conv2d_fwd_sm100");
}

}  // namespace

extern "C" void skd_set_conv_im2col(int on) { g_conv_im2col = on ? 1 : 0; }
extern "C" void skd_set_conv_tile_order(int mode) { g_tile_order = mode; g_tile_flip = 0; }
extern "C" void skd_set_conv_k_order(int mode) { g_k_order = mode; }

// ---- split-K for convolutions with few output tiles and a long K loop (the discriminator: 256 .. 4096 output pixels, K up to 4096) ----
// Without it a 4x8-pixel map at batch 8 is 2 x 2 tiles: 4 of 132 SMs walk 128 K steps each.  Units = tiles x K ranges fill the
// machine; the raw partial tiles go to a caller-provided workspace and one elementwise pass adds them in fixed order and applies
// the epilogue (scale / shift / residual / activation).
static int plan_splits(long long tiles, int k_iters) {
  if (tiles * 2 > kNumSMs || k_iters < 8) return 1;
  int splits = (int)((kNumSMs + tiles - 1) / tiles);
  const int cap = k_iters / 4;                                  // at least 4 K steps per unit
  if (splits > cap) splits = cap;
  if (splits < 2) return 1;
  const int kps = (k_iters + splits - 1) / splits;
  return (k_iters + kps - 1) / kps;                              // no empty range
}

__global__ void __launch_bounds__(256)
splitk_epilogue_kernel(const float* __restrict__ ws, long long plane, int splits, long long P, int C4, int ldw4, float* __restrict__ y, int ldy4,
                       const float* __restrict__ scale, const float* __restrict__ shift, const float* __restrict__ residual, int ldr4,
                       int act, float slope) {
  const long long total = P * C4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long p = i / C4; const int c4 = (int)(i - p * C4);
    const float4* src = reinterpret_cast<const float4*>(ws) + p * ldw4 + c4;
    float4 v = src[0];
    for (int s2 = 1; s2 < splits; ++s2) {
      const float4 b = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(src) + (long long)s2 * plane);
      v.x += b.x; v.y += b.y; v.z += b.z; v.w += b.w;
    }
    if (scale) { const float4 sc = __ldg(reinterpret_cast<const float4*>(scale) + c4); v.x *= sc.x; v.y *= sc.y; v.z *= sc.z; v.w *= sc.w; }
    if (shift) { const float4 sh = __ldg(reinterpret_cast<const float4*>(shift) + c4); v.x += sh.x; v.y += sh.y; v.z += sh.z; v.w += sh.w; }
    if (residual) { const float4 r = __ldg(reinterpret_cast<const float4*>(residual) + p * ldr4 + c4); v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w; }
    v.x = act_fwd(v.x, act, slope); v.y = act_fwd(v.y, act, slope); v.z = act_fwd(v.z, act, slope); v.w = act_fwd(v.w, act, slope);
    reinterpret_cast<float4*>(y)[p * ldy4 + c4] = v;
  }
}

static int conv_fwd_impl(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil,
                         const float* x, const float* x_lo, int ldx, const float* w, const float* w_lo, float* y, int ldy, long long y_row, long long y_img, int oh_req,
                         int ow_req, double* sumsq, int no_store, const float* scale, const float* shift, const float* residual, int ldr, int act, float slope,
                         int round_tf32, cudaStream_t st, float* split_ws = nullptr, long long split_ws_floats = 0) {
  const char* who = "skd_conv2d_fwd_sm100";
  if (Cin % 4 || ldx % 4 || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(w) & 15)) {
    set_error_msg(who, "Cin and the input pitch must be multiples of 4 floats and pointers 16-byte aligned (TMA)");
    return 0;
  }
  // oh_req/ow_req > 0: caller-chosen output extent (rows/cols past the natural size read zero-filled input: far-end padding)
  const int OH = oh_req > 0 ? oh_req : (H + 2 * pad - dil * (KH - 1) - 1) / stride + 1;
  const int OW = ow_req > 0 ? ow_req : (W + 2 * pad - dil * (KW - 1) - 1) / stride + 1;
  if (OH <= 0 || OW <= 0 || N <= 0) return 1;
  ConvArgs a;
  a.Cout = Cout; a.Cin = Cin; a.KH = KH; a.KW = KW; a.stride = stride; a.pad = pad; a.dil = dil;
  a.rOH = OH; a.rOW = OW; a.im2col = 0;
  // tile geometry of the M (pixel) dimension:
  //   flat   : 1x1/stride-1 convolutions are plain GEMMs over the [N*H*W][C] matrix -> tiles of 128 consecutive pixels;
  //   im2col : TMA im2col mode walks 128 consecutive OUTPUT pixels across rows and images (halo = hardware zero fill);
  //   rect   : BH x BW rectangles of one image through the tiled TMA mode (ragged edges waste up to ~19% at 65x129).
  // output addressed as y[n*y_img + oy*y_row + ox*ldy + c]; anything but the dense NHWC strides (e.g. an every-other-pixel
  // sub-grid written by the strided data-gradient) forces rectangular tiles
  const bool strided_out = (y_row != (long long)OW * ldy) || (y_img != (long long)OH * y_row);
  const bool flat = !strided_out && (KH == 1 && KW == 1 && stride == 1 && pad == 0);
  const long long P = (long long)N * OH * OW;
  // TMA im2col bounding box: the last filter origin is dim - 1 + upper.  A caller-chosen extent moves it so that exactly OH x OW
  // origins exist (rows / columns past the input read hardware zero fill)
  const int up_h = oh_req > 0 ? (OH - 1) * stride - pad - (H - 1) : pad - (KH - 1) * dil;
  const int up_w = ow_req > 0 ? (OW - 1) * stride - pad - (W - 1) : pad - (KW - 1) * dil;
  const bool can_im2col = !flat && !strided_out && g_conv_im2col && get_encode_im2col() && pad <= 128 && up_h >= -128 && up_w >= -128 && up_h <= 127 &&
                          up_w <= 127 && stride <= 8 &&
                          P < (1LL << 31) && (KH - 1) * dil < 65536;
  int vN = N, vH = H, vW = W;                                // geometry of the tiled-mode input view
  if (flat) { vN = 1; vH = 1; vW = (int)P; a.N = 1; a.OH = 1; a.OW = (int)P; a.BH = 1; a.BW = 128; }
  else if (can_im2col) { a.im2col = 1; a.N = 1; a.OH = 1; a.OW = (int)P; a.BH = 1; a.BW = 128; }
  else { a.N = N; a.OH = OH; a.OW = OW; pick_rect(OH, OW, stride, &a.BH, &a.BW); }
  a.tiles_x = (a.OW + a.BW - 1) / a.BW; a.tiles_y = (a.OH + a.BH - 1) / a.BH;
  a.m_tiles = a.N * a.tiles_x * a.tiles_y;
  a.k_chunks = (Cin + kBlockK - 1) / kBlockK;
  a.y = y; a.ldy = ldy; a.scale = scale; a.shift = shift; a.residual = residual; a.ldr = ldr;
  a.act = act; a.slope = slope; a.round_out = round_tf32;
  a.y_row = strided_out ? y_row : (long long)a.OW * ldy; a.y_img = strided_out ? y_img : (long long)a.OH * a.OW * ldy;
  // N tile: at most 128 channels, so that a consumer thread's fragment (64 fp32, 128 with the split-precision running total) stays in
  // registers
  const int bn = Cout > 64 ? 128 : (Cout > 32 ? 64 : 32);
  a.n_tiles = (Cout + bn - 1) / bn;
  const bool kc_outer = (g_k_order == 2) || (g_k_order == 0 && KH * KW > 1 && Cin >= 2048);
  // split-K: flat / im2col tile modes only, channel counts and pitches that are whole float4s, a workspace from the caller
  a.splits = 1; a.k_per_split = KH * KW * a.k_chunks; a.split_stride = 0;
  const int ldw = (Cout + 3) / 4 * 4;
  int splits = 1;
  if (split_ws && (flat || a.im2col) && !sumsq && !no_store && Cout % 4 == 0 && ldy % 4 == 0 && !(reinterpret_cast<uintptr_t>(y) & 15) &&
      !((reinterpret_cast<uintptr_t>(scale) | reinterpret_cast<uintptr_t>(shift)) & 15) &&
      (!residual || (ldr % 4 == 0 && !(reinterpret_cast<uintptr_t>(residual) & 15))))
    splits = plan_splits((long long)a.m_tiles * a.n_tiles, KH * KW * a.k_chunks);
  if (splits > 1 && (long long)splits * P * ldw > split_ws_floats) splits = 1;
  if (splits > 1) {
    a.splits = splits; a.k_per_split = (KH * KW * a.k_chunks + splits - 1) / splits; a.split_stride = P * ldw;
    a.y = split_ws; a.ldy = ldw; a.y_row = (long long)a.OW * ldw; a.y_img = (long long)a.OH * a.OW * ldw;
    a.scale = nullptr; a.shift = nullptr; a.residual = nullptr; a.ldr = 0; a.act = 0; a.round_out = 0;
  }

  CUtensorMap tx, tw, tx2, tw2;
  auto encode_x = [&](CUtensorMap* m, const float* ptr) -> bool {
    if (a.im2col) {
      cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
      cuuint64_t strides[3] = {(cuuint64_t)ldx * 4, (cuuint64_t)W * ldx * 4, (cuuint64_t)H * W * ldx * 4};
      int lower[2] = {-pad, -pad};                             // (W, H): filter origin of the first output pixel
      int upper[2] = {up_w, up_h};                             // last filter origin = dim-1 + upper
      cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
      CUresult r = get_encode_im2col()(m, g_tf32_tma_type ? CU_TENSOR_MAP_DATA_TYPE_TFLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4,
                                       const_cast<float*>(ptr), dims, strides, lower, upper, (cuuint32_t)kBlockK, (cuuint32_t)kBlockM, estr,
                                       CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) { set_error_msg(who, "cuTensorMapEncodeIm2col failed"); return false; }
      return true;
    }
    cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)vW, (cuuint64_t)vH, (cuuint64_t)vN};
    cuuint64_t strides[3] = {(cuuint64_t)ldx * 4, (cuuint64_t)vW * ldx * 4, (cuuint64_t)vH * vW * ldx * 4};
    cuuint32_t box[4] = {(cuuint32_t)kBlockK, (cuuint32_t)(a.BW * stride), (cuuint32_t)(a.BH * stride), 1};
    cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
    return encode(m, 4, ptr, dims, strides, box, estr, who);
  };
  auto encode_w = [&](CUtensorMap* m, const float* ptr) -> bool {
    cuuint64_t dims[3] = {(cuuint64_t)Cin, (cuuint64_t)(KH * KW), (cuuint64_t)Cout};
    cuuint64_t strides[2] = {(cuuint64_t)Cin * 4, (cuuint64_t)KH * KW * Cin * 4};
    cuuint32_t box[3] = {(cuuint32_t)kBlockK, 1, (cuuint32_t)bn};
    cuuint32_t estr[3] = {1, 1, 1};
    return encode(m, 3, ptr, dims, strides, box, estr, who);
  };
  if (!encode_x(&tx, x) || !encode_w(&tw, w)) return 0;
  tx2 = tx; tw2 = tw;
  const bool split3 = x_lo && w_lo;
  if (split3) {                                          // split-precision operands: three MMAs per K step
    if ((reinterpret_cast<uintptr_t>(x_lo) | reinterpret_cast<uintptr_t>(w_lo)) & 15) { set_error_msg(who, "x_lo / w_lo not 16-byte aligned"); return 0; }
    if (!encode_x(&tx2, x_lo) || !encode_w(&tw2, w_lo)) return 0;
  }
  a.kc_outer = kc_outer;
  a.reverse = (g_tile_order == 2) ? (g_tile_flip ^= 1) : g_tile_order;
  a.nstages = 0; a.sumsq = sumsq; a.no_store = no_store;
  if (strided_out && residual) { set_error_msg(who, "strided output takes no residual"); return 0; }
  int ok;
  switch (bn) {
    case 128: ok = split3 ? launch<128, true>(tx, tw, tx2, tw2, a, st) : launch<128, false>(tx, tw, tx2, tw2, a, st); break;
    case 64: ok = split3 ? launch<64, true>(tx, tw, tx2, tw2, a, st) : launch<64, false>(tx, tw, tx2, tw2, a, st); break;
    default: ok = split3 ? launch<32, true>(tx, tw, tx2, tw2, a, st) : launch<32, false>(tx, tw, tx2, tw2, a, st); break;
  }
  if (!ok || a.splits == 1) return ok;
  const long long tot4 = P * (Cout / 4);
  long long blocks = (tot4 + 255) / 256; if (blocks > kNumSMs * 8) blocks = kNumSMs * 8; if (blocks < 1) blocks = 1;
  splitk_epilogue_kernel<<<(int)blocks, 256, 0, st>>>(split_ws, a.split_stride, a.splits, P, Cout / 4, ldw / 4, y, ldy / 4, scale, shift, residual,
                                                     ldr / 4, act, slope);
  return finish("skd_conv2d_fwd_sm100(split-K epilogue)");
}

extern "C" int skd_conv2d_fwd_sm100(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil,
                                    const float* x, int ldx, const float* w, float* y, int ldy, const float* scale,
                                    const float* shift, const float* residual, int ldr, int act, float slope,
                                    int round_tf32, cudaStream_t st) {
  const int OH = (H + 2 * pad - dil * (KH - 1) - 1) / stride + 1, OW = (W + 2 * pad - dil * (KW - 1) - 1) / stride + 1;
  return conv_fwd_impl(N, H, W, Cin, Cout, KH, KW, stride, pad, dil, x, nullptr, ldx, w, nullptr, y, ldy, (long long)OW * ldy, (long long)OH * OW * ldy, 0, 0, nullptr, 0,
                       scale, shift, residual, ldr, act, slope, round_tf32, st);
}

extern "C" int skd_conv2d_fwd_sm100_strided(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil,
                                            const float* x, int ldx, const float* w, float* y, long long y_pix, long long y_row,
                                            long long y_img, int out_h, int out_w, int round_tf32, cudaStream_t st) {
  return conv_fwd_impl(N, H, W, Cin, Cout, KH, KW, stride, pad, dil, x, nullptr, ldx, w, nullptr, y, (int)y_pix, y_row, y_img, out_h, out_w, nullptr, 0, nullptr, nullptr, nullptr, 0,
                       0, 0.f, round_tf32, st);
}

// GEMM view of the same kernel for the pair-wise affinity (utils/utils.py:173-183): D[M][Ncols] = A[M][K] * B[Ncols][K]^T with both
// operands K-major; optional output, optional fused sum of squares.
extern "C" int skd_gemm_nt_sm100(int M, int Ncols, int K, const float* A, int lda, const float* B, float* D, int ldd, double* sumsq,
                                 cudaStream_t st) {
  return conv_fwd_impl(1, 1, M, K, Ncols, 1, 1, 1, 0, 1, A, nullptr, lda, B, nullptr, D, ldd, (long long)M * ldd, (long long)M * ldd, 0, 0, sumsq,
                       D == nullptr ? 1 : 0, nullptr, nullptr, nullptr, 0, 0, 0.f, 0, st);
}

// Split-precision ("3xTF32") forward: x = x_hi + x_lo, w = w_hi + w_lo (each part exactly representable in TF32); the kernel
// accumulates x_hi*w_hi + x_lo*w_hi + x_hi*w_lo per K step and adds the steps with fp32 adds -> fp32-grade result at 3x the tensor work.
// Used for the student's stem, layer1 and layer2, where train-mode BN amplifies operand rounding the most (DESIGN.md "TF32 and parity").
extern "C" int skd_conv2d_fwd_sm100_3xtf32(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil,
                                           const float* x_hi, const float* x_lo, int ldx, const float* w_hi, const float* w_lo,
                                           float* y, int ldy, const float* scale, const float* shift, int act, float slope,
                                           cudaStream_t st) {
  const int OH = (H + 2 * pad - dil * (KH - 1) - 1) / stride + 1, OW = (W + 2 * pad - dil * (KW - 1) - 1) / stride + 1;
  return conv_fwd_impl(N, H, W, Cin, Cout, KH, KW, stride, pad, dil, x_hi, x_lo, ldx, w_hi, w_lo, y, ldy, (long long)OW * ldy,
                       (long long)OH * OW * ldy, 0, 0, nullptr, 0, scale, shift, nullptr, 0, act, slope, 0, st);
}

// General entry (discriminator path, networks/sagan_models.py): optional split-precision operands (x_lo / w_lo NULL -> plain TF32),
// optional output extent (out_h / out_w > 0: rows / columns past the natural size see zero-filled input), fused per-channel
// scale / shift, residual add and activation.
extern "C" int skd_conv2d_fwd_sm100_ex(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil, const float* x,
                                       const float* x_lo, int ldx, const float* w, const float* w_lo, float* y, int ldy, int out_h, int out_w,
                                       const float* scale, const float* shift, const float* residual, int ldr, int act, float slope,
                                       cudaStream_t st) {
  const int OH = out_h > 0 ? out_h : (H + 2 * pad - dil * (KH - 1) - 1) / stride + 1;
  const int OW = out_w > 0 ? out_w : (W + 2 * pad - dil * (KW - 1) - 1) / stride + 1;
  if ((x_lo == nullptr) != (w_lo == nullptr)) { set_error_msg("skd_conv2d_fwd_sm100_ex", "x_lo and w_lo must be given together"); return 0; }
  return conv_fwd_impl(N, H, W, Cin, Cout, KH, KW, stride, pad, dil, x, x_lo, ldx, w, w_lo, y, ldy, (long long)OW * ldy, (long long)OH * OW * ldy,
                       out_h, out_w, nullptr, 0, scale, shift, residual, ldr, act, slope, 0, st);
}

// The same convolution with split-K where the tile count is small (plan_splits): `workspace` holds the partial planes.
extern "C" long long skd_conv2d_fwd_sm100_splitk_workspace_floats(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad,
                                                                 int dil, int out_h, int out_w) {
  const int OH = out_h > 0 ? out_h : (H + 2 * pad - dil * (KH - 1) - 1) / stride + 1;
  const int OW = out_w > 0 ? out_w : (W + 2 * pad - dil * (KW - 1) - 1) / stride + 1;
  if (OH <= 0 || OW <= 0 || N <= 0 || Cout % 4) return 0;
  const long long P = (long long)N * OH * OW;
  const int bn = Cout > 64 ? 128 : (Cout > 32 ? 64 : 32);
  const long long tiles = ((P + kBlockM - 1) / kBlockM) * ((Cout + bn - 1) / bn);
  const int splits = plan_splits(tiles, KH * KW * ((Cin + kBlockK - 1) / kBlockK));
  return splits > 1 ? (long long)splits * P * Cout : 0;
}

extern "C" int skd_conv2d_fwd_sm100_splitk(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil, const float* x,
                                           const float* x_lo, int ldx, const float* w, const float* w_lo, float* y, int ldy, int out_h, int out_w,
                                           const float* scale, const float* shift, const float* residual, int ldr, int act, float slope,
                                           float* workspace, long long workspace_floats, cudaStream_t st) {
  const int OH = out_h > 0 ? out_h : (H + 2 * pad - dil * (KH - 1) - 1) / stride + 1;
  const int OW = out_w > 0 ? out_w : (W + 2 * pad - dil * (KW - 1) - 1) / stride + 1;
  if ((x_lo == nullptr) != (w_lo == nullptr)) { set_error_msg("skd_conv2d_fwd_sm100_splitk", "x_lo and w_lo must be given together"); return 0; }
  if (workspace && (reinterpret_cast<uintptr_t>(workspace) & 15)) { set_error_msg("skd_conv2d_fwd_sm100_splitk", "workspace not 16-byte aligned"); return 0; }
  return conv_fwd_impl(N, H, W, Cin, Cout, KH, KW, stride, pad, dil, x, x_lo, ldx, w, w_lo, y, ldy, (long long)OW * ldy, (long long)OH * OW * ldy,
                       out_h, out_w, nullptr, 0, scale, shift, residual, ldr, act, slope, 0, st, workspace, workspace_floats);
}
