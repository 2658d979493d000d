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
//   TMA_EPI         (short-K flat / im2col launches with a residual) the residual comes in and the output goes out through a
//                   shared-memory tile: thread 32 of warpgroup 0 loads the tile's residual by TMA while the K loop runs, and each
//                   consumer warpgroup hands its finished 64 rows to one TMA store and starts the next tile's wgmmas without waiting.
//   BLOCK_M = 256   (flat / im2col, BLOCK_N 128) 256-pixel tiles: the producer loads A as two 128-row boxes, warpgroup g owns
//                   rows 128g .. 128g+127 as two m64 sub-tiles sharing each B read, so a stage brings 48 KB for twice the MMA work
//                   of a 32 KB 128-row stage.  setmaxnreg moves registers from the producer warpgroup to the two accumulators.
#include <cuda.h>

#include "common.cuh"
#include "skd.h"
#include "sm90_ptx.cuh"

using namespace skd;

namespace {

constexpr int kBlockM = 128;                // rows of one A box (and of the default tile; a 256-row tile is two boxes)
constexpr int kBlockK = 32;                 // fp32 elements = 128 B = one swizzle row
constexpr int kWgmmaK = 8;                  // tf32
constexpr int kThreads = 384;               // producer warpgroup + 2 consumer warpgroups
constexpr int kBoxBytes = kBlockM * kBlockK * 4;
constexpr int kProducerRegs = 40;           // BLOCK_M = 256: per-thread registers of the producer / consumer warpgroups after
constexpr int kConsumerRegs = 232;          //   setmaxnreg; 128 * 40 + 256 * 232 = 64 512 <= the 65 536 of the SM
constexpr int kTmaEpiMaxK = 16;             // longest K loop (taps x 32-channel chunks) that takes the TMA epilogue
constexpr int kTile256MinK = 2;             // K loops (taps x 32-channel chunks) that take 256-row tiles: at least 2 steps,
constexpr int kTile256OneNMinK = 18;        //   and 18 .. 72 steps for a launch with a single N tile
constexpr int kTile256OneNMaxK = 72;
constexpr int kEpiBoxBytes = 64 * kBlockK * 4;   // TMA epilogue box: 64 rows x 32 channels

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

template <int BLOCK_M, int BLOCK_N, bool SPLIT, bool TMA_EPI>
struct Cfg {
  static_assert(!(SPLIT && TMA_EPI), "the TMA epilogue serves single-precision launches only");
  static_assert(BLOCK_M == kBlockM || (BLOCK_M == 2 * kBlockM && BLOCK_N == 128 && !SPLIT && !TMA_EPI),
                "256-row tiles: BLOCK_N 128, single precision, register epilogue");
  static constexpr int kMS = BLOCK_M / kBlockM;                // m64 sub-tiles per consumer warpgroup
  static constexpr int kABytes = BLOCK_M * kBlockK * 4;
  static constexpr int kBBytes = BLOCK_N * kBlockK * 4;
  static constexpr int kStageBytes = (kABytes + kBBytes) * (SPLIT ? 2 : 1);   // split precision: {x_hi, w_hi, x_lo, w_lo}
  // TMA epilogue: ring of output tiles (128 rows x BLOCK_N fp32, 32-channel x 64-row boxes of 128B-swizzled rows), taken out of the
  // 227 KB before the operand stages are counted
  static constexpr int kEpiBufs = TMA_EPI ? 2 : 0;
  static constexpr int kEpiBytes = kBlockM * BLOCK_N * 4;
  static constexpr int kFixedBytes = 1024 /*align slack*/ + 256 /*barriers*/;
  static constexpr int kFit = (232448 - kFixedBytes - kEpiBufs * kEpiBytes) / kStageBytes;
  static constexpr int kStages = kFit > 8 ? 8 : kFit;
  static constexpr int kSmemBytes = kStages * kStageBytes + kEpiBufs * kEpiBytes + kFixedBytes;
  static_assert(kStages >= 2, "at least two pipeline stages");
  static_assert(2 * (kStages + kEpiBufs) * 8 <= 256, "barriers");
  static_assert(kSmemBytes <= 232448, "exceeds the 227 KB of shared memory a CTA may use");
};

__device__ __forceinline__ float epi_act(float v, int act, float slope) {
  if (act == ACT_RELU) return fmaxf(v, 0.f);
  if (act == ACT_LEAKY) return v < 0.f ? v * slope : v;
  if (act == ACT_ELU) return v < 0.f ? expm1f(v) : v;
  return v;
}

// TMA epilogue (TMA_EPI): tile buffer eb of the ring holds the tile's residual (loaded by TMA; epi_full[eb] completes when it has
// landed) and then its output (stored by TMA from the same positions; epi_empty[eb] gets one arrival per consumer warpgroup once
// its store has read the buffer).  The output may be the residual itself (Bottleneck.frozen adds in place).  That stays safe:
// a tile reads its residual only from the rows and channels it writes, its load has completed (epi_full) before its own store is
// issued, and no two tiles of a launch write the same element.
template <int BLOCK_M, int BLOCK_N, bool SPLIT, bool TMA_EPI>
__global__ void __launch_bounds__(kThreads, 1)
conv_fwd_sm90_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                     const __grid_constant__ CUtensorMap tmap_x2, const __grid_constant__ CUtensorMap tmap_w2,
                     const __grid_constant__ CUtensorMap tmap_r, const __grid_constant__ CUtensorMap tmap_y, const ConvArgs a) {
  using C = Cfg<BLOCK_M, BLOCK_N, SPLIT, TMA_EPI>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // keep the pointer in the shared address space (integer round trips make nvcc emit generic LD/ST instead of LDS/STS)
  const uint32_t raw_addr = ptx::smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
  uint8_t* epi_smem = smem + C::kStages * C::kStageBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(epi_smem + C::kEpiBufs * C::kEpiBytes);
  uint64_t* empty_bar = full_bar + C::kStages;
  uint64_t* epi_full = empty_bar + C::kStages;
  uint64_t* epi_empty = epi_full + C::kEpiBufs;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmap_x);
    ptx::prefetch_tmap(&tmap_w);
    for (int s = 0; s < C::kStages; ++s) { ptx::mbar_init(&full_bar[s], 1); ptx::mbar_init(&empty_bar[s], 8); }   // one arrival per consumer warp
    if constexpr (TMA_EPI) {
      ptx::prefetch_tmap(&tmap_y);
      ptx::prefetch_tmap(&tmap_r);
      for (int b = 0; b < C::kEpiBufs; ++b) { ptx::mbar_init(&epi_full[b], 1); ptx::mbar_init(&epi_empty[b], 2); }   // one arrival per consumer warpgroup
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  const int total_tiles = a.m_tiles * a.n_tiles * a.splits;     // work units: (tile, K range); the K ranges of a tile are consecutive units
  const int taps = a.KH * a.KW;
  const int k_iters = taps * a.k_chunks;
  const int tiles_per_img = a.tiles_x * a.tiles_y;

  if (warp < 4) {
    // ===================== TMA producer =====================
    if constexpr (C::kMS > 1) ptx::setmaxnreg_dec<kProducerRegs>();
    if (threadIdx.x == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int tu = a.reverse ? total_tiles - 1 - tile : tile;
        const int tl = tu / a.splits, sp = tu - tl * a.splits;
        const int mt = tl / a.n_tiles, nt = tl - mt * a.n_tiles;
        const int img = mt / tiles_per_img, rem = mt - img * tiles_per_img;
        const int ty = rem / a.tiles_x, tx = rem - ty * a.tiles_x;
        const int iy0 = ty * a.BH * a.stride - a.pad, ix0 = tx * a.BW * a.stride - a.pad;
        // im2col: first output pixel of each A box (n, p, q) -> filter-origin input coordinates
        int in0[C::kMS] = {}, ip0[C::kMS] = {}, iq0[C::kMS] = {};
        if (a.im2col) {
#pragma unroll
          for (int b = 0; b < C::kMS; ++b) {
            const int m0 = mt * BLOCK_M + b * kBlockM;
            in0[b] = m0 / (a.rOH * a.rOW);
            const int r2 = m0 - in0[b] * (a.rOH * a.rOW);
            ip0[b] = (r2 / a.rOW) * a.stride - a.pad;
            iq0[b] = (r2 % a.rOW) * a.stride - a.pad;
          }
        }
        // 256-row tiles (flat / im2col, a.OW = P): a second box that starts past P is not loaded.  Its rows of the stage keep
        // whatever an earlier stage left there; a GEMM row depends on its own A row only, and rows past P are never stored.
        const int boxes = (C::kMS > 1 && mt * BLOCK_M + kBlockM >= a.OW) ? 1 : C::kMS;
        const uint32_t stage_tx = (uint32_t)(C::kStageBytes - (C::kMS - boxes) * kBoxBytes);
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
          ptx::mbar_expect_tx(&full_bar[stage], stage_tx);
#pragma unroll
          for (int part = 0; part < (SPLIT ? 2 : 1); ++part) {
            const CUtensorMap* mx = part ? &tmap_x2 : &tmap_x;
            const CUtensorMap* mw = part ? &tmap_w2 : &tmap_w;
            uint8_t* pa = sa + part * (C::kABytes + C::kBBytes);
            uint8_t* pb = pa + C::kABytes;
#pragma unroll
            for (int b = 0; b < C::kMS; ++b) {
              if (b >= boxes) break;
              if (a.im2col)
                ptx::tma_load_im2col_4d(pa + b * kBoxBytes, mx, &full_bar[stage], kc * kBlockK, iq0[b], ip0[b], in0[b], (uint16_t)(kw * a.dil),
                                        (uint16_t)(kh * a.dil));
              else
                ptx::tma_load_4d(pa + b * kBoxBytes, mx, &full_bar[stage], kc * kBlockK, ix0 + b * kBlockM + kw * a.dil, iy0 + kh * a.dil, img);
            }
            ptx::tma_load_3d(pb, mw, &full_bar[stage], kc * kBlockK, tap, nt * BLOCK_N);
          }
          if (++stage == a.nstages) { stage = 0; phase ^= 1; }
        }
      }
    }
    if constexpr (TMA_EPI) {
      // residual loader, a thread of its own so that waiting for a free tile buffer never holds up the operand loads.  Boxes of 32
      // channels x 64 rows, one 64-row half per consumer warpgroup; boxes wholly past P or Cout are not loaded (nobody stores them)
      if (threadIdx.x == 32) {
        const int P = a.OW;                                          // flat / im2col: one row of P pixels
        int eb = 0; uint32_t ephase = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
          const int tu = a.reverse ? total_tiles - 1 - tile : tile;
          const int mt = tu / a.n_tiles, nt = tu - mt * a.n_tiles;
          ptx::mbar_wait(&epi_empty[eb], ephase ^ 1);
          uint32_t bytes = 0;
          for (int h = 0; h < 2; ++h)
            for (int j = 0; j < BLOCK_N / kBlockK; ++j)
              if (mt * kBlockM + 64 * h < P && nt * BLOCK_N + kBlockK * j < a.Cout) bytes += kEpiBoxBytes;
          ptx::mbar_expect_tx(&epi_full[eb], bytes);
          uint8_t* buf = epi_smem + eb * C::kEpiBytes;
          for (int h = 0; h < 2; ++h)
            for (int j = 0; j < BLOCK_N / kBlockK; ++j)
              if (mt * kBlockM + 64 * h < P && nt * BLOCK_N + kBlockK * j < a.Cout)
                ptx::tma_load_2d(buf + (h * (BLOCK_N / kBlockK) + j) * kEpiBoxBytes, &tmap_r, &epi_full[eb], nt * BLOCK_N + kBlockK * j,
                                 mt * kBlockM + 64 * h);
          if (++eb == C::kEpiBufs) { eb = 0; ephase ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers: warpgroup g = rows 64g .. 64g+63 of the tile (128g .. 128g+127 at BLOCK_M 256) =====================
    if constexpr (C::kMS > 1) ptx::setmaxnreg_inc<kConsumerRegs>();
    constexpr int MS = C::kMS;
    const int g = (warp >> 2) - 1;
    const int wq = warp & 3;
    const int r_lo = g * 64 * MS + wq * 16 + (lane >> 2);     // tile rows of this thread's fragment of sub-tile s: r_lo + 64s + {0, 8}
    const int cq = 2 * (lane & 3);                             // first of the thread's two columns in every 8-column group
    constexpr int R = BLOCK_N / 2;
    float acc[MS][R];
    float tot[SPLIT ? R : 1];
    double sq_acc = 0.0;
    int stage = 0; uint32_t phase = 0;
    int eb = 0; uint32_t ephase = 0;                           // TMA epilogue: tile buffer of the current tile
    const bool epi_leader = (threadIdx.x & 127) == 0;          //   the thread that issues its warpgroup's stores
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
        const uint32_t sa = ptx::smem_u32(smem + stage * C::kStageBytes) + (uint32_t)(g * MS * 64 * 128);
        const uint32_t sb = ptx::smem_u32(smem + stage * C::kStageBytes) + (uint32_t)C::kABytes;
        ptx::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kBlockK / kWgmmaK; ++kk) {
          // sub-tile s: the warpgroup's rows 64s .. 64s+63, each its own accumulator through the same k8 sequence, one B read for all
          uint64_t da[MS];
#pragma unroll
          for (int s = 0; s < MS; ++s) da[s] = ptx::make_wgmma_desc_sw128(sa + s * 64 * 128 + kk * kWgmmaK * 4);
          const uint64_t db = ptx::make_wgmma_desc_sw128(sb + kk * kWgmmaK * 4);
          if constexpr (SPLIT) {
            // split precision: this stage's x_hi*w_hi + x_lo*w_hi + x_hi*w_lo in a fresh accumulator, added to the running total with
            // round-to-nearest fp32 adds below (the tensor core truncates on every accumulate: over hundreds of K steps that, not the
            // operand split, would limit the "fp32-grade" layers)
            constexpr uint32_t kLo = C::kABytes + C::kBBytes;
            ptx::wgmma_tf32<BLOCK_N>(acc[0], da[0], db, kk != 0 ? 1u : 0u);
            ptx::wgmma_tf32<BLOCK_N>(acc[0], ptx::make_wgmma_desc_sw128(sa + kLo + kk * kWgmmaK * 4), db, 1u);
            ptx::wgmma_tf32<BLOCK_N>(acc[0], da[0], ptx::make_wgmma_desc_sw128(sb + kLo + kk * kWgmmaK * 4), 1u);
          } else {
#pragma unroll
            for (int s = 0; s < MS; ++s) ptx::wgmma_tf32<BLOCK_N>(acc[s], da[s], db, (k | kk) != 0 ? 1u : 0u);
          }
        }
        ptx::wgmma_commit();
        if constexpr (SPLIT) {
          ptx::wgmma_wait<0>();
          ptx::fence_regs(acc[0]);
#pragma unroll
          for (int i = 0; i < R; ++i) tot[i] += acc[0][i];
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
#pragma unroll
        for (int s = 0; s < MS; ++s) ptx::fence_regs(acc[s]);
        if (prev_stage >= 0 && lane == 0) ptx::mbar_arrive(&empty_bar[prev_stage]);
      }
      if constexpr (SPLIT) {
#pragma unroll
        for (int i = 0; i < R; ++i) acc[0][i] = tot[i];
      }

      // ---- epilogue from the fragment ----
      // the thread's two output rows of sub-tile s (fragment rows r_lo + 64s and r_lo + 64s + 8); in[s][h] = false past the output
      bool in[MS][2];
      float* yrow[MS][2];
      const float* rrow[MS][2];
#pragma unroll
      for (int s = 0; s < MS; ++s) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = r_lo + 64 * s + 8 * h;
          const int img = mt / tiles_per_img, rem = mt - img * tiles_per_img;
          const int ty = rem / a.tiles_x, tx = rem - ty * a.tiles_x;
          const int dy = row / a.BW, dx = row - dy * a.BW;
          const int oy = ty * a.BH + dy, ox = tx * a.BW + dx;
          in[s][h] = oy < a.OH && ox < a.OW;
          yrow[s][h] = a.y + (size_t)sp * a.split_stride + (size_t)img * a.y_img + (size_t)oy * a.y_row + (size_t)ox * a.ldy;
          rrow[s][h] = in[s][h] && a.residual ? a.residual + (((size_t)img * a.OH + oy) * a.OW + ox) * a.ldr : nullptr;
        }
      }
      // Pass 1: scale, shift and residual, each read in full at the thread's columns and then applied in place, before anything is
      // stored.  The output may alias what these read, so the compiler keeps every read after the stores that precede it: reads
      // interleaved with the stores wait one global-memory latency per column pair (a 1x1 convolution with a residual then runs at
      // a fraction of the DRAM rate), while a pass with no store in it has all its reads in flight at once.  __fmul_rn / __fadd_rn
      // keep the product and each sum separately rounded (no contraction into an FMA), in the order scale, shift, residual.
      // Columns past Cout read nothing; their values are never stored.  A per-channel operand is read once for both sub-tiles.
      const int c0 = nt * BLOCK_N + cq;
      float t[BLOCK_N / 4];                                      // one operand at the thread's columns c0 + 8j + {0, 1}
      auto gather = [&](const float* p) {
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const int c = c0 + 8 * j;
          t[2 * j] = c < a.Cout ? __ldg(p + c) : 0.f;
          t[2 * j + 1] = c + 1 < a.Cout ? __ldg(p + c + 1) : 0.f;
        }
      };
      if (a.scale) {
        gather(a.scale);
#pragma unroll
        for (int s = 0; s < MS; ++s)
#pragma unroll
          for (int i = 0; i < R; ++i) acc[s][i] = __fmul_rn(acc[s][i], t[(i >> 2) * 2 + (i & 1)]);
      }
      if (a.shift) {
        gather(a.shift);
#pragma unroll
        for (int s = 0; s < MS; ++s)
#pragma unroll
          for (int i = 0; i < R; ++i) acc[s][i] = __fadd_rn(acc[s][i], t[(i >> 2) * 2 + (i & 1)]);
      }
      if constexpr (TMA_EPI) {
        float* v = acc[0];
        // The residual and the output share the tile buffer: the thread reads the residual at its own fragment positions and writes
        // the finished values back to the same positions, so the two passes need no barrier between them.  Position of fragment row
        // rl and column c: box c / 32 of the warpgroup's half, row rl of 128 B, 16-byte chunk (c % 32) / 4 XOR rl % 8 (SWIZZLE_128B,
        // which also spreads the float2 accesses of a warp over all banks).
        uint8_t* half = epi_smem + eb * C::kEpiBytes + g * (C::kEpiBytes / 2);
        const uint32_t frag = (uint32_t)((wq * 16 + (lane >> 2)) * 128 + (cq & 3) * 4);
        auto at = [&](int h, int j) -> float2* {
          return reinterpret_cast<float2*>(half + (j >> 2) * kEpiBoxBytes + frag + h * 8 * 128 +
                                           ((((j & 3) * 2 + (cq >> 2)) ^ (lane >> 2)) << 4));
        };
        // the previous tile's stores have had this tile's K loop to read their buffer: hand it to the residual loader
        if (epi_leader && tile != blockIdx.x) {
          ptx::bulk_wait_group_read<0>();
          ptx::mbar_arrive(&epi_empty[eb == 0 ? C::kEpiBufs - 1 : eb - 1]);
        }
        ptx::mbar_wait(&epi_full[eb], ephase);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int j = 0; j < BLOCK_N / 8; ++j) {
            const float2 r = *at(h, j);
            v[4 * j + 2 * h] = __fadd_rn(v[4 * j + 2 * h], r.x);
            v[4 * j + 2 * h + 1] = __fadd_rn(v[4 * j + 2 * h + 1], r.y);
          }
        }
        // Pass 2: activation, rounding, sum of squares (from the registers), values into the buffer
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float part = 0.f;
#pragma unroll
          for (int j = 0; j < BLOCK_N / 8; ++j) {
            const int c = c0 + 8 * j;
            float v0 = v[4 * j + 2 * h], v1 = v[4 * j + 2 * h + 1];
            v0 = epi_act(v0, a.act, a.slope); v1 = epi_act(v1, a.act, a.slope);
            if (a.round_out) { v0 = ptx::round_tf32(v0); v1 = ptx::round_tf32(v1); }
            if (a.sumsq && c < a.Cout) part = fmaf(v0, v0, c + 1 < a.Cout ? fmaf(v1, v1, part) : part);
            *at(h, j) = make_float2(v0, v1);
          }
          if (in[0][h]) sq_acc += (double)part;
        }
        // one TMA store per 32-channel box of the warpgroup's 64 rows; the tensor map clips rows past P and channels past Cout
        ptx::fence_proxy_async();
        ptx::named_bar_sync(1 + g, 128);
        if (epi_leader) {
          const int row0 = mt * kBlockM + 64 * g;
          if (row0 < a.OW)
            for (int j = 0; j < BLOCK_N / kBlockK; ++j)
              if (nt * BLOCK_N + kBlockK * j < a.Cout) ptx::tma_store_2d(&tmap_y, half + j * kEpiBoxBytes, nt * BLOCK_N + kBlockK * j, row0);
          ptx::bulk_commit_group();
        }
        if (++eb == C::kEpiBufs) { eb = 0; ephase ^= 1; }
      } else {
#pragma unroll
        for (int s = 0; s < MS; ++s) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (!rrow[s][h]) continue;
            gather(rrow[s][h]);
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j) {
              acc[s][4 * j + 2 * h] = __fadd_rn(acc[s][4 * j + 2 * h], t[2 * j]);
              acc[s][4 * j + 2 * h + 1] = __fadd_rn(acc[s][4 * j + 2 * h + 1], t[2 * j + 1]);
            }
          }
        }
        // Pass 2: activation, rounding, sum of squares, stores.  One copy of the pass per activation, chosen once per tile: with the
        // activation chosen per value, the inlined ELU made every column pair 2 KB of code, and a 256-row tile's epilogue took
        // 50 - 58 us instead of 8 (DESIGN.md §3.1, §6).
        auto pass2 = [&](auto act) {
#pragma unroll
          for (int s = 0; s < MS; ++s) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              if (!in[s][h]) continue;
              float part = 0.f;
#pragma unroll
              for (int j = 0; j < BLOCK_N / 8; ++j) {
                const int c = c0 + 8 * j;
                if (c >= a.Cout) continue;
                const bool two = c + 1 < a.Cout;
                float v0 = act(acc[s][4 * j + 2 * h]), v1 = act(acc[s][4 * j + 2 * h + 1]);
                if (a.round_out) { v0 = ptx::round_tf32(v0); v1 = ptx::round_tf32(v1); }
                if (a.sumsq) part = fmaf(v0, v0, two ? fmaf(v1, v1, part) : part);
                if (a.no_store) continue;
                float* y = yrow[s][h];
                if (two && !((reinterpret_cast<uintptr_t>(y + c)) & 7)) {
                  *reinterpret_cast<float2*>(y + c) = make_float2(v0, v1);
                } else {
                  y[c] = v0;
                  if (two) y[c + 1] = v1;
                }
              }
              sq_acc += (double)part;                           // fp32 within a row of the tile, fp64 across rows and tiles
            }
          }
        };
        switch (a.act) {
          case ACT_RELU: pass2([](float v) { return epi_act(v, ACT_RELU, 0.f); }); break;
          case ACT_LEAKY: pass2([&](float v) { return epi_act(v, ACT_LEAKY, a.slope); }); break;
          case ACT_ELU: pass2([](float v) { return epi_act(v, ACT_ELU, 0.f); }); break;
          default: pass2([](float v) { return v; }); break;
        }
      }
    }
    if constexpr (TMA_EPI) {
      if (epi_leader) ptx::bulk_wait_group<0>();                // the last stores read shared memory until they complete
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
int g_tile_m = 0;                 // 0: 256-row tiles by the launch's shape; 1: always 128; 2: 256 wherever the 256-row path can run
int g_last_plan[7] = {0, 0, 0, 0, 0, 0, 0};   // what conv_fwd_impl chose for its last launch (skd_conv_fwd_last_plan)

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


// Operand maps round to TF32 on load (CU_TENSOR_MAP_DATA_TYPE_TFLOAT32 under g_tf32_tma_type); epilogue maps (residual, output) are
// FLOAT32 and move the values unchanged.
CUtensorMapDataType operand_type() { return g_tf32_tma_type ? CU_TENSOR_MAP_DATA_TYPE_TFLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32; }

bool encode(CUtensorMap* m, CUtensorMapDataType type, int rank, const void* base, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
            const cuuint32_t* box, const cuuint32_t* estr, const char* who) {
  EncodeTiledFn fn = get_encode_tiled();
  if (!fn) { set_error_msg(who, "cuTensorMapEncodeTiled unavailable (no CUDA driver)"); return false; }
  CUresult r = fn(m, type, (cuuint32_t)rank,
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

template <int BLOCK_M, int BLOCK_N, bool SPLIT, bool TMA_EPI>
int launch(const CUtensorMap& tx, const CUtensorMap& tw, const CUtensorMap& tx2, const CUtensorMap& tw2, const CUtensorMap& tr,
           const CUtensorMap& ty, const ConvArgs& a_in, cudaStream_t st) {
  using C = Cfg<BLOCK_M, BLOCK_N, SPLIT, TMA_EPI>;
  ConvArgs a = a_in;
  a.nstages = C::kStages;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(conv_fwd_sm90_kernel<BLOCK_M, BLOCK_N, SPLIT, TMA_EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         C::kSmemBytes);
    if (e != cudaSuccess) { set_error("skd_conv2d_fwd_sm100(attr)", e); return 0; }
    attr = true;
  }
  int grid = a.m_tiles * a.n_tiles * a.splits;
  if (grid > kNumSMs) grid = kNumSMs;
  conv_fwd_sm90_kernel<BLOCK_M, BLOCK_N, SPLIT, TMA_EPI><<<grid, kThreads, C::kSmemBytes, st>>>(tx, tw, tx2, tw2, tr, ty, a);
  return finish("skd_conv2d_fwd_sm100");
}

template <int BLOCK_N>
int launch_n(bool split3, bool tma_epi, const CUtensorMap& tx, const CUtensorMap& tw, const CUtensorMap& tx2, const CUtensorMap& tw2,
             const CUtensorMap& tr, const CUtensorMap& ty, const ConvArgs& a, cudaStream_t st) {
  if (split3) return launch<kBlockM, BLOCK_N, true, false>(tx, tw, tx2, tw2, tr, ty, a, st);
  if (tma_epi) return launch<kBlockM, BLOCK_N, false, true>(tx, tw, tx2, tw2, tr, ty, a, st);
  return launch<kBlockM, BLOCK_N, false, false>(tx, tw, tx2, tw2, tr, ty, a, st);
}

// ---------------------------------------------------------------------------------------------------
// Chained bottleneck 1x1 pair (frozen teacher): block i's conv3 and block i+1's conv1 in one launch.
//   y3 = relu(conv1x1(x3, w3) * scale3 + shift3 + residual)       (Cin3 -> Cout3; y3 may be the residual itself)
//   y1 = relu(conv1x1(y3, w1) * scale1 + shift1)                   (Cout3 -> Cout1 <= 256)
// Per flat 128-pixel tile the consumers walk conv3's output channels in chunks of kChainBN3: the conv3 K loop, the TMA epilogue of
// conv_fwd_sm90_kernel (residual loaded into a tile buffer by thread 32, the same float operations, a TMA store of the 64 rows of the
// warpgroup), and the finished values -- rounded as the TFLOAT32 tensor map of the unfused conv1 would round them -- into a K-major
// SWIZZLE_128B staging buffer that is conv1's A operand for the chunk's 64 channels of K.  conv1's weights stream through the
// operand ring after the chunk's conv3 stages.  conv1's accumulators stay in registers across the chunks; its register epilogue
// runs after the last one.  Both outputs equal the two unfused launches bit for bit: the same k8 wgmma sequences per element
// (conv1's K in ascending 32-channel chunks, m64n128 per 128 output channels as the unfused BLOCK_N 128 tiles), and the same
// epilogue arithmetic.  What it saves is reading y3 back from HBM and one launch per bottleneck.
// ---------------------------------------------------------------------------------------------------
constexpr int kChainBN3 = 64;                    // conv3 output channels per chunk = conv1 K per chunk

struct ChainArgs {
  int P, Cin3, Cout3;
  const float* scale3; const float* shift3;
  const float* scale1; const float* shift1;
  float* y1; int ldy1;
  int round_stage;                               // 1: conv1 operand rounded to nearest TF32 (the TFLOAT32 operand maps); 0: raw fp32
  int nstages;
};

template <int COUT1>
struct ChainCfg {
  static_assert(COUT1 == 64 || COUT1 == 128 || COUT1 == 256, "conv1 output channels: 64, 128 or 256");
  static constexpr int kN1 = COUT1 > 128 ? 128 : COUT1;        // conv1 wgmma width: the unfused launch's BLOCK_N
  static constexpr int kNT1 = COUT1 / kN1;                     // conv1 accumulators per consumer thread
  static constexpr int kA3Bytes = kBlockM * kBlockK * 4;
  static constexpr int kB3Bytes = kChainBN3 * kBlockK * 4;
  static constexpr int kB1Bytes = COUT1 * kBlockK * 4;
  static constexpr int kStageBytes = kA3Bytes + kB3Bytes > kB1Bytes ? kA3Bytes + kB3Bytes : kB1Bytes;
  static constexpr int kTileBytes = kBlockM * kChainBN3 * 4;   // one residual / output tile buffer, and the staging buffer
  static constexpr int kEpiBufs = 2;
  static constexpr int kFixedBytes = 1024 /*align slack*/ + 256 /*barriers*/;
  static constexpr int kFit = (232448 - kFixedBytes - (kEpiBufs + 1) * kTileBytes) / kStageBytes;
  static constexpr int kStages = kFit > 8 ? 8 : kFit;
  static constexpr int kSmemBytes = kStages * kStageBytes + (kEpiBufs + 1) * kTileBytes + kFixedBytes;
  static_assert(kStages >= 3, "operand ring");
  static_assert(2 * (kStages + kEpiBufs) * 8 <= 256, "barriers");
  static_assert(kSmemBytes <= 232448, "exceeds the 227 KB of shared memory a CTA may use");
};

template <int COUT1>
__global__ void __launch_bounds__(kThreads, 1)
conv1x1_chain_sm90_kernel(const __grid_constant__ CUtensorMap tmap_x3, const __grid_constant__ CUtensorMap tmap_w3,
                          const __grid_constant__ CUtensorMap tmap_w1, const __grid_constant__ CUtensorMap tmap_r,
                          const __grid_constant__ CUtensorMap tmap_y3, const ChainArgs a) {
  using C = ChainCfg<COUT1>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t raw_addr = ptx::smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
  uint8_t* epi_smem = smem + C::kStages * C::kStageBytes;
  uint8_t* stg_smem = epi_smem + C::kEpiBufs * C::kTileBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(stg_smem + C::kTileBytes);
  uint64_t* empty_bar = full_bar + C::kStages;
  uint64_t* epi_full = empty_bar + C::kStages;
  uint64_t* epi_empty = epi_full + C::kEpiBufs;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmap_x3);
    ptx::prefetch_tmap(&tmap_w3);
    ptx::prefetch_tmap(&tmap_w1);
    ptx::prefetch_tmap(&tmap_r);
    ptx::prefetch_tmap(&tmap_y3);
    for (int s = 0; s < C::kStages; ++s) { ptx::mbar_init(&full_bar[s], 1); ptx::mbar_init(&empty_bar[s], 8); }
    for (int b = 0; b < C::kEpiBufs; ++b) { ptx::mbar_init(&epi_full[b], 1); ptx::mbar_init(&epi_empty[b], 2); }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  const int m_tiles = (a.P + kBlockM - 1) / kBlockM;
  const int chunks = a.Cout3 / kChainBN3;
  const int k3 = (a.Cin3 + kBlockK - 1) / kBlockK;
  constexpr int k1 = kChainBN3 / kBlockK;

  if (warp < 4) {
    ptx::setmaxnreg_dec<kProducerRegs>();
    if (threadIdx.x == 0) {
      // operand producer: per chunk, k3 stages of {x3 box, w3 box}, then k1 stages of one w1 box (all conv1 output channels)
      int stage = 0; uint32_t phase = 0;
      for (int mt = blockIdx.x; mt < m_tiles; mt += gridDim.x) {
        for (int c = 0; c < chunks; ++c) {
          for (int k = 0; k < k3; ++k) {
            ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
            uint8_t* sa = smem + stage * C::kStageBytes;
            ptx::mbar_expect_tx(&full_bar[stage], C::kA3Bytes + C::kB3Bytes);
            ptx::tma_load_2d(sa, &tmap_x3, &full_bar[stage], k * kBlockK, mt * kBlockM);
            ptx::tma_load_2d(sa + C::kA3Bytes, &tmap_w3, &full_bar[stage], k * kBlockK, c * kChainBN3);
            if (++stage == a.nstages) { stage = 0; phase ^= 1; }
          }
          for (int k = 0; k < k1; ++k) {
            ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
            ptx::mbar_expect_tx(&full_bar[stage], C::kB1Bytes);
            ptx::tma_load_2d(smem + stage * C::kStageBytes, &tmap_w1, &full_bar[stage], (c * k1 + k) * kBlockK, 0);
            if (++stage == a.nstages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    if (threadIdx.x == 32) {
      // residual loader: one tile buffer per chunk, 32-channel x 64-row boxes; a 64-row half wholly past P is not loaded
      int eb = 0; uint32_t ephase = 0;
      for (int mt = blockIdx.x; mt < m_tiles; mt += gridDim.x) {
        const uint32_t bytes = (mt * kBlockM + 64 < a.P ? 2 : 1) * k1 * kEpiBoxBytes;
        for (int c = 0; c < chunks; ++c) {
          ptx::mbar_wait(&epi_empty[eb], ephase ^ 1);
          ptx::mbar_expect_tx(&epi_full[eb], bytes);
          uint8_t* buf = epi_smem + eb * C::kTileBytes;
          for (int h = 0; h < 2; ++h)
            for (int j = 0; j < k1; ++j)
              if (mt * kBlockM + 64 * h < a.P)
                ptx::tma_load_2d(buf + (h * k1 + j) * kEpiBoxBytes, &tmap_r, &epi_full[eb], c * kChainBN3 + kBlockK * j, mt * kBlockM + 64 * h);
          if (++eb == C::kEpiBufs) { eb = 0; ephase ^= 1; }
        }
      }
    }
  } else {
    ptx::setmaxnreg_inc<kConsumerRegs>();
    constexpr int N1 = C::kN1, NT1 = C::kNT1;
    const int g = (warp >> 2) - 1;
    const int wq = warp & 3;
    const int r_lo = g * 64 + wq * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);
    float acc1[NT1][N1 / 2];
    float acc3[kChainBN3 / 2];
    int stage = 0; uint32_t phase = 0;
    int eb = 0; uint32_t ephase = 0;
    bool first_chunk = true;
    const bool epi_leader = (threadIdx.x & 127) == 0;
    // the warpgroup's 64 rows of the staging buffer: conv1's A operand, boxes of 32 channels as in the tile buffers
    uint8_t* stg = stg_smem + g * (C::kTileBytes / 2);
    const uint32_t stg_addr = ptx::smem_u32(stg);
    const uint32_t frag = (uint32_t)((wq * 16 + (lane >> 2)) * 128 + (cq & 3) * 4);
    auto at = [&](uint8_t* half, int h, int j) -> float2* {     // fragment position (row half h, column group j), SWIZZLE_128B
      return reinterpret_cast<float2*>(half + (j >> 2) * kEpiBoxBytes + frag + h * 8 * 128 + ((((j & 3) * 2 + (cq >> 2)) ^ (lane >> 2)) << 4));
    };
    float t[N1 / 4];
    auto gather = [&](const float* p, int c0, int n) {
#pragma unroll
      for (int j = 0; j < n / 8; ++j) { t[2 * j] = __ldg(p + c0 + 8 * j); t[2 * j + 1] = __ldg(p + c0 + 8 * j + 1); }
    };
    for (int mt = blockIdx.x; mt < m_tiles; mt += gridDim.x) {
      int prev_stage = -1;
      auto release_prev = [&]() {
        if (prev_stage >= 0 && lane == 0) ptx::mbar_arrive(&empty_bar[prev_stage]);
      };
      for (int c = 0; c < chunks; ++c) {
        // ---- conv3, output channels c*64 .. c*64+63 ----
        for (int k = 0; k < k3; ++k) {
          ptx::mbar_wait(&full_bar[stage], phase);
          const uint32_t base = ptx::smem_u32(smem + stage * C::kStageBytes);
          const uint32_t sa = base + (uint32_t)(g * 64 * 128), sb = base + (uint32_t)C::kA3Bytes;
          ptx::wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < kBlockK / kWgmmaK; ++kk)
            ptx::wgmma_tf32<kChainBN3>(acc3, ptx::make_wgmma_desc_sw128(sa + kk * kWgmmaK * 4), ptx::make_wgmma_desc_sw128(sb + kk * kWgmmaK * 4),
                                      (k | kk) != 0 ? 1u : 0u);
          ptx::wgmma_commit();
          ptx::wgmma_wait<1>();
          release_prev();
          prev_stage = stage;
          if (++stage == a.nstages) { stage = 0; phase ^= 1; }
        }
        ptx::wgmma_wait<0>();
        ptx::fence_regs(acc3);
#pragma unroll
        for (int n = 0; n < NT1; ++n) ptx::fence_regs(acc1[n]);
        release_prev();
        prev_stage = -1;

        // ---- conv3 epilogue: scale, shift, residual, ReLU (conv_fwd_sm90_kernel's TMA epilogue, BLOCK_N 64) ----
        const int c0 = c * kChainBN3 + cq;
        gather(a.scale3, c0, kChainBN3);
#pragma unroll
        for (int i = 0; i < kChainBN3 / 2; ++i) acc3[i] = __fmul_rn(acc3[i], t[(i >> 2) * 2 + (i & 1)]);
        gather(a.shift3, c0, kChainBN3);
#pragma unroll
        for (int i = 0; i < kChainBN3 / 2; ++i) acc3[i] = __fadd_rn(acc3[i], t[(i >> 2) * 2 + (i & 1)]);
        uint8_t* half = epi_smem + eb * C::kTileBytes + g * (C::kTileBytes / 2);
        if (epi_leader && !first_chunk) {                       // the previous chunk's stores have read their buffer
          ptx::bulk_wait_group_read<0>();
          ptx::mbar_arrive(&epi_empty[eb == 0 ? C::kEpiBufs - 1 : eb - 1]);
        }
        first_chunk = false;
        ptx::mbar_wait(&epi_full[eb], ephase);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int j = 0; j < kChainBN3 / 8; ++j) {
            const float2 r = *at(half, h, j);
            float v0 = __fadd_rn(acc3[4 * j + 2 * h], r.x), v1 = __fadd_rn(acc3[4 * j + 2 * h + 1], r.y);
            v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f);
            *at(half, h, j) = make_float2(v0, v1);
            if (a.round_stage) { v0 = ptx::round_tf32(v0); v1 = ptx::round_tf32(v1); }
            *at(stg, h, j) = make_float2(v0, v1);
          }
        }
        // the tile buffer goes to the TMA store and the staging buffer to the tensor core: both read through the async proxy
        ptx::fence_proxy_async();
        ptx::named_bar_sync(1 + g, 128);
        if (epi_leader) {
          const int row0 = mt * kBlockM + 64 * g;
          if (row0 < a.P)
            for (int j = 0; j < k1; ++j) ptx::tma_store_2d(&tmap_y3, half + j * kEpiBoxBytes, c * kChainBN3 + kBlockK * j, row0);
          ptx::bulk_commit_group();
        }
        if (++eb == C::kEpiBufs) { eb = 0; ephase ^= 1; }

        // ---- conv1, K = channels c*64 .. c*64+63 of y3, from the staging buffer ----
        for (int kb = 0; kb < k1; ++kb) {
          ptx::mbar_wait(&full_bar[stage], phase);
          const uint32_t sb = ptx::smem_u32(smem + stage * C::kStageBytes);
          ptx::wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < kBlockK / kWgmmaK; ++kk) {
            const uint64_t da = ptx::make_wgmma_desc_sw128(stg_addr + kb * kEpiBoxBytes + kk * kWgmmaK * 4);
#pragma unroll
            for (int n = 0; n < NT1; ++n)
              ptx::wgmma_tf32<N1>(acc1[n], da, ptx::make_wgmma_desc_sw128(sb + n * N1 * 128 + kk * kWgmmaK * 4), (c | kb | kk) != 0 ? 1u : 0u);
          }
          ptx::wgmma_commit();
          ptx::wgmma_wait<1>();
          release_prev();
          prev_stage = stage;
          if (++stage == a.nstages) { stage = 0; phase ^= 1; }
        }
      }
      ptx::wgmma_wait<0>();
#pragma unroll
      for (int n = 0; n < NT1; ++n) ptx::fence_regs(acc1[n]);
      release_prev();

      // ---- conv1 epilogue: scale, shift, ReLU, stores (conv_fwd_sm90_kernel's register epilogue) ----
#pragma unroll
      for (int n = 0; n < NT1; ++n) {
        const int c0 = n * N1 + cq;
        gather(a.scale1, c0, N1);
#pragma unroll
        for (int i = 0; i < N1 / 2; ++i) acc1[n][i] = __fmul_rn(acc1[n][i], t[(i >> 2) * 2 + (i & 1)]);
        gather(a.shift1, c0, N1);
#pragma unroll
        for (int i = 0; i < N1 / 2; ++i) acc1[n][i] = __fadd_rn(acc1[n][i], t[(i >> 2) * 2 + (i & 1)]);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = mt * kBlockM + r_lo + 8 * h;
          if (row >= a.P) continue;
          float* y = a.y1 + (size_t)row * a.ldy1 + c0;
#pragma unroll
          for (int j = 0; j < N1 / 8; ++j)
            *reinterpret_cast<float2*>(y + 8 * j) = make_float2(fmaxf(acc1[n][4 * j + 2 * h], 0.f), fmaxf(acc1[n][4 * j + 2 * h + 1], 0.f));
        }
      }
    }
    if (epi_leader) ptx::bulk_wait_group<0>();
  }
}

template <int COUT1>
int launch_chain(const CUtensorMap& tx3, const CUtensorMap& tw3, const CUtensorMap& tw1, const CUtensorMap& tr, const CUtensorMap& ty3,
                 const ChainArgs& a_in, cudaStream_t st) {
  using C = ChainCfg<COUT1>;
  ChainArgs a = a_in;
  a.nstages = C::kStages;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(conv1x1_chain_sm90_kernel<COUT1>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmemBytes);
    if (e != cudaSuccess) { set_error("skd_conv1x1_chain_sm100(attr)", e); return 0; }
    attr = true;
  }
  const int m_tiles = (a.P + kBlockM - 1) / kBlockM;
  conv1x1_chain_sm90_kernel<COUT1><<<m_tiles < kNumSMs ? m_tiles : kNumSMs, kThreads, C::kSmemBytes, st>>>(tx3, tw3, tw1, tr, ty3, a);
  return finish("skd_conv1x1_chain_sm100");
}

int g_conv_chain = 0;              // 0: frozen bottlenecks chain conv3 into the next block's conv1; 1: never

}  // namespace

extern "C" void skd_set_conv_im2col(int on) { g_conv_im2col = on ? 1 : 0; }
extern "C" void skd_set_conv_tile_order(int mode) { g_tile_order = mode; g_tile_flip = 0; }
extern "C" void skd_set_conv_k_order(int mode) { g_k_order = mode; }
extern "C" void skd_set_conv_tile_m(int mode) { g_tile_m = mode; }
extern "C" void skd_set_conv_chain(int mode) { g_conv_chain = mode; }
extern "C" int skd_conv_chain_mode(void) { return g_conv_chain; }
extern "C" void skd_conv_fwd_last_plan(int* out) { for (int i = 0; i < 7; ++i) out[i] = g_last_plan[i]; }

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
      CUresult r = get_encode_im2col()(m, operand_type(), 4,
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
    return encode(m, operand_type(), 4, ptr, dims, strides, box, estr, who);
  };
  auto encode_w = [&](CUtensorMap* m, const float* ptr) -> bool {
    cuuint64_t dims[3] = {(cuuint64_t)Cin, (cuuint64_t)(KH * KW), (cuuint64_t)Cout};
    cuuint64_t strides[2] = {(cuuint64_t)Cin * 4, (cuuint64_t)KH * KW * Cin * 4};
    cuuint32_t box[3] = {(cuuint32_t)kBlockK, 1, (cuuint32_t)bn};
    cuuint32_t estr[3] = {1, 1, 1};
    return encode(m, operand_type(), 3, ptr, dims, strides, box, estr, who);
  };
  if (!encode_x(&tx, x) || !encode_w(&tw, w)) return 0;
  tx2 = tx; tw2 = tw;
  const bool split3 = x_lo && w_lo;
  if (split3) {                                          // split-precision operands: three MMAs per K step
    if ((reinterpret_cast<uintptr_t>(x_lo) | reinterpret_cast<uintptr_t>(w_lo)) & 15) { set_error_msg(who, "x_lo / w_lo not 16-byte aligned"); return 0; }
    if (!encode_x(&tx2, x_lo) || !encode_w(&tw2, w_lo)) return 0;
  }
  // TMA epilogue: short-K launches with a residual (the teacher's bottleneck conv3), whose time goes to reading the residual and
  // writing the output rather than to the K loop.  Without a residual, or with a longer K loop, the register epilogue and the deeper
  // operand ring the tile buffers would cost are faster (DESIGN.md §6).  It needs the [P][Cout] pixel rows of the flat / im2col tile
  // modes (so no strided output), a plain fp32 output (no split-K partials, no reduction-only launch) and pitches and pointers TMA can
  // address (whole float4s, 16-byte aligned).
  const bool tma_epi = (flat || a.im2col) && a.splits == 1 && !no_store && !split3 && residual &&
                       KH * KW * a.k_chunks <= kTmaEpiMaxK && ldy % 4 == 0 && !(reinterpret_cast<uintptr_t>(y) & 15) &&
                       ldr % 4 == 0 && !(reinterpret_cast<uintptr_t>(residual) & 15);
  CUtensorMap tr{}, ty{};
  if (tma_epi) {
    auto encode_rows = [&](CUtensorMap* m, const float* ptr, int ld) -> bool {
      cuuint64_t dims[2] = {(cuuint64_t)Cout, (cuuint64_t)P};
      cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
      cuuint32_t box[2] = {(cuuint32_t)kBlockK, 64};
      cuuint32_t estr[2] = {1, 1};
      return encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, ptr, dims, strides, box, estr, who);
    };
    if (!encode_rows(&ty, y, ldy) || !encode_rows(&tr, residual, ldr)) return 0;
  }
  // 256-row tiles (two 128-row A boxes per stage, same maps): a 48 KB stage carries twice the MMA work of a 32 KB 128-row stage, and
  // the operand bytes per FLOP bound both tile shapes (DESIGN.md §3.1, §6).  Measured: with more than one N tile 256 rows won at
  // every K from 2 to 1152 steps; with a single N tile they won at K = 18 and 72 and lost at K = 16 (1x1 512->128) and K = 288
  // (3x3 1024->128).  And only where the halved unit count costs no extra time in ragged waves of 132 CTAs: a 256-row unit took
  // 1.3 - 1.8 times a 128-row unit of the same launch, so the 256-row waves, counted at 1.8 each, must not outlast the 128-row waves.
  const bool tile256_legal = (flat || a.im2col) && bn == 128 && !split3 && a.splits == 1 && !tma_epi && !sumsq && !no_store;
  const long long units128 = (long long)a.m_tiles * a.n_tiles, units256 = (P + 2 * kBlockM - 1) / (2 * kBlockM) * a.n_tiles;
  const long long waves128 = (units128 + kNumSMs - 1) / kNumSMs, waves256 = (units256 + kNumSMs - 1) / kNumSMs;
  const int k_steps = KH * KW * a.k_chunks;
  const bool tile256 = tile256_legal && g_tile_m != 1 &&
                       (g_tile_m == 2 ||
                        (k_steps >= kTile256MinK && (a.n_tiles > 1 || (k_steps >= kTile256OneNMinK && k_steps <= kTile256OneNMaxK)) &&
                         9 * waves256 <= 5 * waves128));
  if (tile256) { a.BW = 2 * kBlockM; a.tiles_x = (a.OW + a.BW - 1) / a.BW; a.m_tiles = a.tiles_x; }
  a.kc_outer = kc_outer;
  a.reverse = (g_tile_order == 2) ? (g_tile_flip ^= 1) : g_tile_order;
  a.nstages = 0; a.sumsq = sumsq; a.no_store = no_store;
  if (strided_out && residual) { set_error_msg(who, "strided output takes no residual"); return 0; }
  const int plan[7] = {flat ? 0 : (a.im2col ? 1 : 2), tile256 ? 2 * kBlockM : kBlockM, bn, a.splits, tma_epi ? 1 : 0, kc_outer ? 1 : 0, a.reverse};
  for (int i = 0; i < 7; ++i) g_last_plan[i] = plan[i];
  int ok;
  switch (bn) {
    case 128:
      ok = tile256 ? launch<2 * kBlockM, 128, false, false>(tx, tw, tx2, tw2, tr, ty, a, st) : launch_n<128>(split3, tma_epi, tx, tw, tx2, tw2, tr, ty, a, st);
      break;
    case 64: ok = launch_n<64>(split3, tma_epi, tx, tw, tx2, tw2, tr, ty, a, st); break;
    default: ok = launch_n<32>(split3, tma_epi, tx, tw, tx2, tw2, tr, ty, a, st); break;
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

// The strided-output form with split-precision operands (ESPNet's 2x2 / stride-2 transposed convolution: a 1x1 GEMM per output-row
// parity written straight onto the every-other-row sub-grid, fp32-grade like skd_conv2d_fwd_sm100_3xtf32).
extern "C" int skd_conv2d_fwd_sm100_strided_3xtf32(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil,
                                                   const float* x_hi, const float* x_lo, int ldx, const float* w_hi, const float* w_lo,
                                                   float* y, long long y_pix, long long y_row, long long y_img, cudaStream_t st) {
  if (!x_lo || !w_lo) { set_error_msg("skd_conv2d_fwd_sm100_strided_3xtf32", "x_lo and w_lo are required"); return 0; }
  return conv_fwd_impl(N, H, W, Cin, Cout, KH, KW, stride, pad, dil, x_hi, x_lo, ldx, w_hi, w_lo, y, (int)y_pix, y_row, y_img, 0, 0, nullptr, 0,
                       nullptr, nullptr, nullptr, 0, 0, 0.f, 0, st);
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

// Chained frozen-bottleneck pair (conv1x1_chain_sm90_kernel): y3 = relu(x3 * w3 * scale3 + shift3 + residual) over P pixel rows
// (y3 may be the residual), then y1 = relu(y3 * w1 * scale1 + shift1) in the same launch.
extern "C" int skd_conv1x1_chain_sm100(int P, int Cin3, int Cout3, int Cout1, const float* x3, int ldx3, const float* w3, const float* scale3,
                                       const float* shift3, const float* residual, int ldr, float* y3, int ldy3, const float* w1,
                                       const float* scale1, const float* shift1, float* y1, int ldy1, cudaStream_t st) {
  const char* who = "skd_conv1x1_chain_sm100";
  if (P <= 0) return 1;
  if (Cin3 % 4 || Cout3 % kChainBN3 || !(Cout1 == 64 || Cout1 == 128 || Cout1 == 256) || ldx3 % 4 || ldr % 4 || ldy3 % 4 || ldy1 % 2) {
    set_error_msg(who, "Cin3 and the pitches must be multiples of 4 floats, Cout3 a multiple of 64, Cout1 64, 128 or 256");
    return 0;
  }
  if ((reinterpret_cast<uintptr_t>(x3) | reinterpret_cast<uintptr_t>(w3) | reinterpret_cast<uintptr_t>(residual) | reinterpret_cast<uintptr_t>(y3) |
       reinterpret_cast<uintptr_t>(w1)) & 15 || (reinterpret_cast<uintptr_t>(y1) & 7) || !scale3 || !shift3 || !scale1 || !shift1) {
    set_error_msg(who, "operands 16-byte aligned (y1 8-byte), scale and shift of both convolutions required");
    return 0;
  }
  auto rows = [&](CUtensorMap* m, CUtensorMapDataType type, const float* ptr, int cols, int nrows, int ld, int box_rows) -> bool {
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)nrows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
    cuuint32_t box[2] = {(cuuint32_t)kBlockK, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    return encode(m, type, 2, ptr, dims, strides, box, estr, who);
  };
  CUtensorMap tx3, tw3, tw1, tr, ty3;
  if (!rows(&tx3, operand_type(), x3, Cin3, P, ldx3, kBlockM) || !rows(&tw3, operand_type(), w3, Cin3, Cout3, Cin3, kChainBN3) ||
      !rows(&tw1, operand_type(), w1, Cout3, Cout1, Cout3, Cout1) || !rows(&tr, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, residual, Cout3, P, ldr, 64) ||
      !rows(&ty3, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, y3, Cout3, P, ldy3, 64))
    return 0;
  ChainArgs a;
  a.P = P; a.Cin3 = Cin3; a.Cout3 = Cout3;
  a.scale3 = scale3; a.shift3 = shift3; a.scale1 = scale1; a.shift1 = shift1;
  a.y1 = y1; a.ldy1 = ldy1;
  a.round_stage = g_tf32_tma_type ? 1 : 0;
  a.nstages = 0;
  switch (Cout1) {
    case 64: return launch_chain<64>(tx3, tw3, tw1, tr, ty3, a, st);
    case 128: return launch_chain<128>(tx3, tw3, tw1, tr, ty3, a, st);
    default: return launch_chain<256>(tx3, tw3, tw1, tr, ty3, a, st);
  }
}
