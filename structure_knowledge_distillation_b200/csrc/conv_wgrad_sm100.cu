// wgmma weight-gradient convolution for sm_90a (cuDNN wgrad in the reference, reached through autograd of every
// nn.Conv2d of the student: networks/kd_model.py:150 G_loss.backward()).
//
//   dW[co][tap][ci] = sum_{pixels p} dY[p][co] * X[p shifted by tap][ci]
//
// GEMM view: M = Cout (128 per tile), N = Cin (<= 128 per tile, one filter tap per tile), K = pixels.  Both operands lie in HBM with
// the channels contiguous (NHWC), i.e. MN-major, and TF32 wgmma takes a shared-memory operand only K-major.  Per pipeline stage TMA
// drops 32-channel x 32-pixel boxes (128B-swizzled, one pixel per 128-byte row) of dY and X into a raw stage.
//  * dY is the A operand and goes to the tensor core from registers: each consumer thread loads its A fragments straight from the raw
//    box (no transposed copy), so a dY box is never rewritten, however many taps and Cin tiles read it.
//  * X is the B operand: warps 1-3 of the producer warpgroup transpose it into a ring of K-major 128B-swizzled tiles (one channel per
//    128-byte row) with its own full / empty barriers, so the transposition of later K-blocks runs while the consumers' wgmmas run.
//  * The raw stage is released once the three transposer warps have read X and the eight consumer warps have loaded their fragments.
// Each consumer warpgroup issues 4 x wgmma.m64nNk8.tf32 per K-block for its 64 Cout rows.  Split-K over pixel blocks gives >= 2 waves
// of work units; fp32 partials go to a workspace and a deterministic reduction adds them in fixed order.
// Pairs (BLOCK_N 128, Cout >= 256): two units of adjacent full Cout tiles with the same (split, tap, Cin tile) run on one CTA of a
// launch of their own, before the launch of the single units.  The stage holds both dY boxes and one X box, X is transposed once
// for 256 Cout rows, and each consumer warpgroup computes one of the two units as two m64 sub-tiles against the same X tile.  Each
// dW element is the same k8 MMA sequence over the same operands either way, so pairing never changes a bit.
// Per-warpgroup pairs (Cout <= 64, BLOCK_N <= 64): any two units share a CTA, each on its own consumer warpgroup with its own dY and
// X boxes, so no MMA row is out of range and two waves of units fit in one (kWgPair below).
#include <cuda.h>

#include "common.cuh"
#include "skd.h"
#include "sm90_ptx.cuh"

using namespace skd;

namespace {

constexpr int kBlockM = 128;               // Cout per tile
constexpr int kKPix = 32;                  // pixels per pipeline stage (one 128-byte K row of the transposed tiles)
constexpr int kThreads = 384;              // producer warpgroup (TMA thread + 3 transposer warps) + 2 consumer warpgroups
constexpr int kTransposeThreads = 96;
constexpr int kChunkBytes = 32 * kKPix * 4;        // one 32-channel x 32-pixel box
constexpr int kMaxStages = 4;
constexpr int kSets = 3;                   // transposed X sets
constexpr int kProducerRegs = 48;          // pair kernel: per-thread registers of the producer / consumer warpgroups after
constexpr int kConsumerRegs = 224;         //   setmaxnreg; 128 * 48 + 256 * 224 = 63 488 <= the 168 * 384 the launch holds

struct WgArgs {
  int N, OH, OW, Cout, Cin, KH, KW, stride, pad, dil;
  int BHk, BWk, kb_x, kb_y;                // pixel K-blocks per image
  int m_tiles, n_tiles, taps, splits, kb_total, kb_per_split;
  float* ws;                               // [splits][Cout][taps*Cin]
  int linear;                              // K-blocks are 32 consecutive output pixels (dY as a [P][Cout] matrix, X through TMA im2col)
  int m_pairs;                             // pairs of full Cout tiles (2i, 2i + 1) per (split, tap, nt) that may run as one unit
  int pairs;                               // pair units: kCoutPair runs them in a launch of their own before the single units,
                                           //   kWgPair at the head of its one launch
  int items;                               // work units of this launch
};

// Work-unit kinds of a launch.
//  kSingle:   one unit per work item; consumer warpgroup g computes Cout rows 64 g .. 64 g + 63 of the unit's tile.
//  kCoutPair: every item is two units of adjacent full Cout tiles with the same (split, tap, nt), i.e. the same X box; the raw
//             stage holds their two dY boxes (256 Cout) and consumer warpgroup g computes Cout tile mt + g as two m64 sub-tiles.
//  kWgPair:   Cout <= 64: an item is any two units (or one), each on its own consumer warpgroup, so no MMA row is out of range; the
//             stage holds a dY box (chunks 2 g, 2 g + 1) and an X box per warpgroup, and each X set two transposed tiles.
enum : int { kSingle = 0, kCoutPair = 1, kWgPair = 2 };

template <int BLOCK_N, int KIND>
struct WCfg {
  static constexpr int kABytes = 4 * kChunkBytes;                    // 128 co
  static constexpr int kARegion = (KIND == kCoutPair ? 2 : 1) * kABytes;
  static constexpr int kBBytes = (BLOCK_N / 32) * kChunkBytes;       // one X box; its transposed tile has the same size
  static constexpr int kBRegion = (KIND == kWgPair ? 2 : 1) * kBBytes;   // X boxes of a stage = one transposed X set
  static constexpr int kStageBytes = kARegion + kBRegion;            // raw (pixel-major) stage
  static constexpr int kFit = (232448 - kSets * kBRegion - 1024 - 256) / kStageBytes;
  static constexpr int kStages = kFit > kMaxStages ? kMaxStages : kFit;
  static constexpr int kSmemBytes = kStages * kStageBytes + kSets * kBRegion + 1024 + 256;
  static_assert(kStages >= 2, "at least two pipeline stages");
};

struct Unit { int split, mt, nt, tap, pair; };

// index u over (split, Cout tile row of m, tap, nt), split-major
__device__ __forceinline__ Unit decode_tile(const WgArgs& a, int u, int m) {
  const int tiles = m * a.taps * a.n_tiles;
  Unit w;
  w.split = u / tiles;
  const int tile = u - w.split * tiles;
  w.mt = tile / (a.taps * a.n_tiles);
  const int r = tile - w.mt * (a.taps * a.n_tiles);
  w.tap = r / a.n_tiles;
  w.nt = r - w.tap * a.n_tiles;
  w.pair = 0;
  return w;
}

// kCoutPair launch: item i is group i of (split, Cout tile pair, tap, nt), w.mt the pair's first tile.  kSingle launch: both units
// of every group the pair launch left out, then the units of Cout tiles in no pair (an odd or ragged last tile); with m_pairs = 0
// that is (split, mt, tap, nt) order.  kWgPair: item i < pairs is units 2i and 2i + 1 of that order, item i >= pairs unit pairs + i
// alone (w[1].split = -1).  Every unit computes its dW block over its split's K-blocks whether it runs paired or not.
template <int KIND>
__device__ __forceinline__ void decode_item(const WgArgs& a, int i, Unit (&w)[2]) {
  w[1].split = -1;
  if constexpr (KIND == kCoutPair) {
    w[0] = decode_tile(a, i, a.m_pairs);
    w[0].mt *= 2; w[0].pair = 1;
  } else if constexpr (KIND == kWgPair) {
    w[0] = decode_tile(a, i < a.pairs ? 2 * i : a.pairs + i, a.m_tiles);
    if (i < a.pairs) w[1] = decode_tile(a, 2 * i + 1, a.m_tiles);
  } else {
    const int unpaired = 2 * (a.splits * a.m_pairs * a.taps * a.n_tiles - a.pairs);
    if (i < unpaired) { w[0] = decode_tile(a, a.pairs + (i >> 1), a.m_pairs); w[0].mt = 2 * w[0].mt + (i & 1); return; }
    w[0] = decode_tile(a, i - unpaired, a.m_tiles - 2 * a.m_pairs);
    w[0].mt += 2 * a.m_pairs;
  }
}

// K-blocks of a unit (0 for an absent one) and its first
__device__ __forceinline__ int unit_kblocks(const WgArgs& a, const Unit& w, int& kb0) {
  if (w.split < 0) { kb0 = 0; return 0; }
  kb0 = w.split * a.kb_per_split;
  return min(a.kb_total, kb0 + a.kb_per_split) - kb0;
}

// X box (pixel rows of 32 channels, 128B swizzle) -> K-major tile (channel rows of 32 pixels, 128B swizzle); unit = 4 pixels x 4
// channels, read as 4 float4 (one per pixel row) and written as 4 float4 (one per channel row).  Unit u: q = u & 7, channel group
// cg = 8 (u >> 6) + q, pixel group pg = q ^ ((u >> 3) & 7).  A quarter-warp (one 128-bit wavefront) holds q = 0..7 with the rest of
// u fixed, and both its 16-byte slot maps are permutations of 0..7 (enumerated on the host), so neither side has bank conflicts:
// reads (cg & 7) ^ ((4 pg + i) & 7) = q ^ 4 ((q ^ s) & 1) ^ i, writes pg ^ ((4 cg + e) & 7) = q ^ s ^ 4 (q & 1) ^ e.
template <int BLOCK_N>
__device__ __forceinline__ void transpose_x(const uint8_t* raw, uint8_t* dst, int t) {
  for (int u = t; u < BLOCK_N * 2; u += kTransposeThreads) {
    const int q = u & 7, pg = q ^ ((u >> 3) & 7), cg = ((u >> 6) << 3) + q;
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

struct Ring { int stage; uint32_t phase; int xs; uint32_t xphase; int prev_xs; };

// One consumer warpgroup's share of a work unit: NSUB m64 sub-tiles read from the 64-row blocks rb0 .. rb0 + NSUB - 1 of the
// stage's dY boxes (off: the fragment offsets of row block rb0), all against the transposed X tile at x_off in the X set.  They
// are Cout rows co_row .. co_row + 64 NSUB - 1 of the unit's tile.
template <int BLOCK_N, int KIND, int NSUB>
__device__ __forceinline__ void consume_unit(const WgArgs& a, const Unit& w, int co_row, int x_off, const uint32_t (&off)[4], int co_lane,
                                             int lane, uint8_t* smem, uint8_t* sets, uint64_t* full_bar, uint64_t* empty_bar,
                                             uint64_t* xfull_bar, uint64_t* xempty_bar, Ring& q) {
  using C = WCfg<BLOCK_N, KIND>;
  const int kb0 = w.split * a.kb_per_split;                    // a present unit
  const int nkb = min(a.kb_total, kb0 + a.kb_per_split) - kb0;
  float acc[NSUB][BLOCK_N / 2];
  uint32_t fa[NSUB][16], fb[NSUB][16];                         // A fragments of two K-blocks: loads for k + 1 leave k's in-flight operands alone
  auto kblock = [&](uint32_t (&f)[NSUB][16], int k) {
    ptx::mbar_wait(&full_bar[q.stage], q.phase);
    const uint8_t* raw = smem + q.stage * C::kStageBytes;
    // fragment kk: a0 / a1 = rows h 0 / 1 at pixel 8kk + j, a2 / a3 the same at pixel 8kk + j + 4; sub-tile s two chunks further
#pragma unroll
    for (int s = 0; s < NSUB; ++s) {
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int r = 0; r < 4; ++r)
          f[s][4 * kk + r] = *reinterpret_cast<const uint32_t*>(raw + off[2 * (r & 1) + (r >> 1)] + 2 * kChunkBytes * s + 1024 * kk +
                                                                512 * (r >> 1));
      }
    }
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(&empty_bar[q.stage]);
    if (++q.stage == C::kStages) { q.stage = 0; q.phase ^= 1; }
    ptx::mbar_wait(&xfull_bar[q.xs], q.xphase);
    const uint32_t sb = ptx::smem_u32(sets + q.xs * C::kBRegion + x_off);
    ptx::wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kKPix / 8; ++kk) {
#pragma unroll
      for (int s = 0; s < NSUB; ++s)
        ptx::wgmma_tf32_rs<BLOCK_N>(acc[s], f[s][4 * kk], f[s][4 * kk + 1], f[s][4 * kk + 2], f[s][4 * kk + 3],
                                    ptx::make_wgmma_desc_sw128(sb + kk * 32), (k | kk) != 0 ? 1u : 0u);
    }
    ptx::wgmma_commit();
    if constexpr (NSUB == 1) {
      ptx::wgmma_wait<1>();                                    // the previous K-block's wgmmas are done: its fragments and X tile are free
      if (q.prev_xs >= 0) { __syncwarp(); if (lane == 0) ptx::mbar_arrive(&xempty_bar[q.prev_xs]); }
      q.prev_xs = q.xs;
    } else {
      ptx::wgmma_wait<0>();                                    // one fragment set: this K-block's wgmmas are done
      __syncwarp(); if (lane == 0) ptx::mbar_arrive(&xempty_bar[q.xs]);
    }
    if (++q.xs == kSets) { q.xs = 0; q.xphase ^= 1; }
  };
  int k = 0;
  if constexpr (NSUB == 1) {
    for (; k + 1 < nkb; k += 2) { kblock(fa, k); kblock(fb, k + 1); }
    if (k < nkb) kblock(fa, k);                                // odd count: fa's last wgmmas were retired by fb's wait
  } else {
    // 128 accumulators leave no room for a second fragment set; the other warpgroup's wgmmas cover this one's fragment loads
    for (; k < nkb; ++k) kblock(fa, k);
  }
  ptx::wgmma_wait<0>();
  if (q.prev_xs >= 0) { __syncwarp(); if (lane == 0) ptx::mbar_arrive(&xempty_bar[q.prev_xs]); q.prev_xs = -1; }
  const size_t kdim = (size_t)a.taps * a.Cin;
  const int cq = 2 * (lane & 3);
#pragma unroll
  for (int s = 0; s < NSUB; ++s) {
    ptx::fence_regs(acc[s]);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int co = w.mt * kBlockM + co_row + 64 * s + co_lane + 4 * h;
      if (co >= a.Cout) continue;
      float* orow = a.ws + ((size_t)w.split * a.Cout + co) * kdim + (size_t)w.tap * a.Cin;
#pragma unroll
      for (int jj = 0; jj < BLOCK_N / 8; ++jj) {
        const int ci = w.nt * BLOCK_N + 8 * jj + cq;           // even; Cin % 4 == 0, so ci + 1 < Cin too
        if (ci < a.Cin) *reinterpret_cast<float2*>(orow + ci) = make_float2(acc[s][4 * jj + 2 * h], acc[s][4 * jj + 2 * h + 1]);
      }
    }
  }
}

// kWgPair: the stages of an item past this warpgroup's own unit (the other unit is longer, or this one is absent) are released
// without MMAs, so that every stage and X set still gets its 8 consumer-warp arrivals.
template <int BLOCK_N, int KIND>
__device__ __forceinline__ void skip_kblocks(int n, int lane, uint64_t* full_bar, uint64_t* empty_bar, uint64_t* xfull_bar,
                                             uint64_t* xempty_bar, Ring& q) {
  using C = WCfg<BLOCK_N, KIND>;
  for (int k = 0; k < n; ++k) {
    ptx::mbar_wait(&full_bar[q.stage], q.phase);
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(&empty_bar[q.stage]);
    if (++q.stage == C::kStages) { q.stage = 0; q.phase ^= 1; }
    ptx::mbar_wait(&xfull_bar[q.xs], q.xphase);
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(&xempty_bar[q.xs]);
    if (++q.xs == kSets) { q.xs = 0; q.xphase ^= 1; }
  }
}

template <int BLOCK_N, int KIND>
__global__ void __launch_bounds__(kThreads, 1)
conv_wgrad_sm90_kernel(const __grid_constant__ CUtensorMap tmap_dy, const __grid_constant__ CUtensorMap tmap_x, const WgArgs a) {
  using C = WCfg<BLOCK_N, KIND>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // keep the pointer in the shared address space (integer round trips make nvcc emit generic LD/ST instead of LDS/STS)
  const uint32_t raw_addr = ptx::smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
  uint8_t* sets = smem + C::kStages * C::kStageBytes;                // kSets transposed X tiles
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sets + kSets * C::kBRegion);
  uint64_t* empty_bar = full_bar + kMaxStages;
  uint64_t* xfull_bar = empty_bar + kMaxStages;
  uint64_t* xempty_bar = xfull_bar + kSets;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmap_dy); ptx::prefetch_tmap(&tmap_x);
    // one arrival per warp: raw stage <- 3 transposer + 8 consumer warps, X set full <- 3 transposer warps, empty <- 8 consumer warps
    for (int s = 0; s < C::kStages; ++s) { ptx::mbar_init(&full_bar[s], 1); ptx::mbar_init(&empty_bar[s], 11); }
    for (int s = 0; s < kSets; ++s) { ptx::mbar_init(&xfull_bar[s], 3); ptx::mbar_init(&xempty_bar[s], 8); }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  const int kb_per_img = a.kb_x * a.kb_y;

  if (warp < 4) {
    if constexpr (KIND == kCoutPair) ptx::setmaxnreg_dec<kProducerRegs>();
    if (warp == 0) {
      // ===================== TMA producer =====================
      // all-out-of-range channel chunks (Cout or Cin < tile) are not issued; a Cout pair's two tiles are full and adjacent, so its
      // eight dY chunks are one run of Cout; a kWgPair unit (Cout <= 64, at most two chunks) loads into chunks 2 x, 2 x + 1
      if (threadIdx.x == 0) {
        int stage = 0; uint32_t phase = 0;
        // one unit's K-block kb into the stage's dY chunks at sa and X box at sb
        auto issue = [&](const Unit& w, int kb, uint8_t* sa, uint8_t* sb, int a_chunks, int b_chunks, uint64_t* bar) {
          const int kh = w.tap / a.KW, kw = w.tap - kh * a.KW;
          if (a.linear) {
            const int p0 = kb * kKPix;
            const int img = p0 / (a.OH * a.OW), r2 = p0 - img * (a.OH * a.OW);
            const int oy = r2 / a.OW, ox = r2 - oy * a.OW;
            for (int c = 0; c < a_chunks; ++c)
              ptx::tma_load_4d(sa + c * kChunkBytes, &tmap_dy, bar, w.mt * kBlockM + c * 32, p0, 0, 0);
            for (int c = 0; c < b_chunks; ++c)
              ptx::tma_load_im2col_4d(sb + c * kChunkBytes, &tmap_x, bar, w.nt * BLOCK_N + c * 32, ox * a.stride - a.pad,
                                      oy * a.stride - a.pad, img, (uint16_t)(kw * a.dil), (uint16_t)(kh * a.dil));
          } else {
            const int img = kb / kb_per_img, q = kb - img * kb_per_img;
            const int by = q / a.kb_x, bx = q - by * a.kb_x;
            const int oy0 = by * a.BHk, ox0 = bx * a.BWk;
            for (int c = 0; c < a_chunks; ++c)
              ptx::tma_load_4d(sa + c * kChunkBytes, &tmap_dy, bar, w.mt * kBlockM + c * 32, ox0, oy0, img);
            for (int c = 0; c < b_chunks; ++c)
              ptx::tma_load_4d(sb + c * kChunkBytes, &tmap_x, bar, w.nt * BLOCK_N + c * 32, ox0 * a.stride - a.pad + kw * a.dil,
                               oy0 * a.stride - a.pad + kh * a.dil, img);
          }
        };
        auto chunks = [&](const Unit& w, int& a_chunks, int& b_chunks) {
          a_chunks = KIND == kCoutPair ? 8 : min(4, (a.Cout - w.mt * kBlockM + 31) / 32);
          b_chunks = max(0, min(BLOCK_N / 32, (a.Cin - w.nt * BLOCK_N + 31) / 32));
        };
        for (int i = blockIdx.x; i < a.items; i += gridDim.x) {
          Unit w[2];
          decode_item<KIND>(a, i, w);
          if constexpr (KIND == kWgPair) {
            int kb0[2], nkb[2], a_chunks[2], b_chunks[2];
#pragma unroll
            for (int x = 0; x < 2; ++x) { nkb[x] = unit_kblocks(a, w[x], kb0[x]); chunks(w[x], a_chunks[x], b_chunks[x]); }
            const int nk = max(nkb[0], nkb[1]);
            for (int k = 0; k < nk; ++k) {
              ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
              uint32_t bytes = 0;
#pragma unroll
              for (int x = 0; x < 2; ++x)
                if (k < nkb[x]) bytes += (uint32_t)((a_chunks[x] + b_chunks[x]) * kChunkBytes);
              ptx::mbar_expect_tx(&full_bar[stage], bytes);
#pragma unroll
              for (int x = 0; x < 2; ++x)
                if (k < nkb[x])
                  issue(w[x], kb0[x] + k, smem + stage * C::kStageBytes + x * 2 * kChunkBytes,
                        smem + stage * C::kStageBytes + C::kARegion + x * C::kBBytes, a_chunks[x], b_chunks[x], &full_bar[stage]);
              if (++stage == C::kStages) { stage = 0; phase ^= 1; }
            }
          } else {
            int a_chunks, b_chunks;
            chunks(w[0], a_chunks, b_chunks);
            const int kb0 = w[0].split * a.kb_per_split;
            const int kb1 = min(a.kb_total, kb0 + a.kb_per_split);
            for (int kb = kb0; kb < kb1; ++kb) {
              ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
              uint8_t* sa = smem + stage * C::kStageBytes;
              ptx::mbar_expect_tx(&full_bar[stage], (uint32_t)((a_chunks + b_chunks) * kChunkBytes));
              issue(w[0], kb, sa, sa + C::kARegion, a_chunks, b_chunks, &full_bar[stage]);
              if (++stage == C::kStages) { stage = 0; phase ^= 1; }
            }
          }
        }
      }
    } else {
      // ===================== X transposer (warps 1-3) =====================
      const int t = threadIdx.x - 32;                            // 0..95
      int stage = 0; uint32_t phase = 0; int xs = 0; uint32_t xphase = 0;
      for (int i = blockIdx.x; i < a.items; i += gridDim.x) {
        Unit w[2];
        decode_item<KIND>(a, i, w);
        int kb0, nkb[2] = {0, 0};
        if constexpr (KIND == kWgPair) {
          nkb[0] = unit_kblocks(a, w[0], kb0);
          nkb[1] = unit_kblocks(a, w[1], kb0);
        } else {
          kb0 = w[0].split * a.kb_per_split;
          nkb[0] = min(a.kb_total, kb0 + a.kb_per_split) - kb0;
        }
        const int nk = max(nkb[0], nkb[1]);
        for (int k = 0; k < nk; ++k) {
          ptx::mbar_wait(&full_bar[stage], phase);
          ptx::mbar_wait(&xempty_bar[xs], xphase ^ 1);
          const uint8_t* raw = smem + stage * C::kStageBytes + C::kARegion;
          if constexpr (KIND == kWgPair) {
            if (k < nkb[0]) transpose_x<BLOCK_N>(raw, sets + xs * C::kBRegion, t);
            if (k < nkb[1]) transpose_x<BLOCK_N>(raw + C::kBBytes, sets + xs * C::kBRegion + C::kBBytes, t);
          } else {
            transpose_x<BLOCK_N>(raw, sets + xs * C::kBRegion, t);
          }
          ptx::fence_proxy_async();                              // generic-proxy writes -> visible to the wgmma (async proxy) reads
          __syncwarp();
          if (lane == 0) { ptx::mbar_arrive(&empty_bar[stage]); ptx::mbar_arrive(&xfull_bar[xs]); }
          if (++stage == C::kStages) { stage = 0; phase ^= 1; }
          if (++xs == kSets) { xs = 0; xphase ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers =====================
    if constexpr (KIND == kCoutPair) ptx::setmaxnreg_inc<kConsumerRegs>();
    const int g = (threadIdx.x - 128) >> 7;                    // warpgroup
    const int wq = warp & 3, c8 = lane >> 2, j = lane & 3;
    // MMA row 16 wq + 8 h + c8 of an m64 sub-tile holds Cout 32 (wq >> 1) + 16 (c8 >> 2) + 8 (wq & 1) + 4 h + (c8 & 3) of its 64: with
    // the fragment's k = j (+4) that puts the 32 lanes of every fragment load on 32 different banks (16-byte slot 4 (c8 >> 2) + 2 (wq & 1)
    // + h of the 32-channel box, XOR pixel & 7 = j or j + 4: bank bits 4 / 3-2 / 1-0 = c8 >> 2 / j / c8 & 3, enumerated on the host).
    // Cout = MMA row would put each load's lanes on 16 banks, two per bank.  Each dW element is still the same k8 MMA sequence over
    // the same operands, only on another row of the tensor core.
    const int co_lane = 32 * (wq >> 1) + 16 * (c8 >> 2) + 8 * (wq & 1) + (c8 & 3);   // + 64 row block + 4 h
    const int rb0 = KIND == kCoutPair ? 2 * g : g;             // first 64-row block of the stage's dY boxes
    uint32_t off[4];                                           // byte offsets in the raw stage of (h, pixel & 4) for pixel 4i + j
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int slot = 4 * (c8 >> 2) + 2 * (wq & 1) + h;
      const int base = (2 * rb0 + (wq >> 1)) * kChunkBytes + j * 128 + 4 * (c8 & 3);
      off[2 * h] = base + ((slot ^ j) << 4);
      off[2 * h + 1] = base + ((slot ^ j ^ 4) << 4);
    }
    Ring q{0, 0u, 0, 0u, -1};
    // one accumulator width per kernel: with both in one consumer ptxas serializes every wgmma of the kernel
    for (int i = blockIdx.x; i < a.items; i += gridDim.x) {
      Unit w[2];
      decode_item<KIND>(a, i, w);
      if constexpr (KIND == kWgPair) {
        int kb0;
        const int n0 = unit_kblocks(a, w[0], kb0), n1 = unit_kblocks(a, w[1], kb0), n = g ? n1 : n0;
        const Unit wu = g ? w[1] : w[0];
        if (n) consume_unit<BLOCK_N, KIND, 1>(a, wu, 0, g * C::kBBytes, off, co_lane, lane, smem, sets, full_bar, empty_bar, xfull_bar,
                                              xempty_bar, q);
        skip_kblocks<BLOCK_N, KIND>(max(n0, n1) - n, lane, full_bar, empty_bar, xfull_bar, xempty_bar, q);
      } else {
        consume_unit<BLOCK_N, KIND, KIND == kCoutPair ? 2 : 1>(a, w[0], 64 * rb0, 0, off, co_lane, lane, smem, sets, full_bar, empty_bar,
                                                               xfull_bar, xempty_bar, q);
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
int g_last_plan[3] = {0, 0, 0};   // what skd_conv2d_wgrad_sm100 chose for its last launch (skd_conv_wgrad_last_plan)
int g_wgrad_pairing = 1;
int g_last_pairs = 0;             // pair units of the last launch (skd_conv_wgrad_last_pairs)

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

// Pair units of a call (WgArgs::pairs).  Mode 0: none; 2: every legal pair; 1: the count that minimises the predicted time, in
// single-unit times, of a static stride over at most kNumSMs CTAs.
// kCoutPair: the pair launch followed by the single launch, ceil(pairs / kNumSMs) kPairCost + ceil(singles / kNumSMs).  Measured on
// an H100 (700 W, batch 8, tools/conv_wgrad_bench.py) a pair cost 1.18-1.24 single units at the 3x3 shapes and 1.50 at the 1x1
// 256->512; 1.4 and 1.2 pick the same pair counts for every weight gradient of the benchmark step.
// kWgPair: one launch whose CTA 0 runs the most items and the most pairs, ceil(items / grid) + (kWgPairCost - 1) ceil(pairs / grid);
// its two units share no operand, and a pair measured 1.80-1.89 single units (layer1 and stem conv2 64->64, same card and tool).
// Ties take more pairs (less work in all).
constexpr double kPairCost = 1.4;
constexpr double kWgPairCost = 1.8;

int choose_wg_pairs(int units, int mode) {
  if (mode == 0 || units < 2) return 0;
  if (mode == 2) return units / 2;
  int best = 0; double best_t = 1e30;
  for (int P = 0; P <= units / 2; ++P) {
    const int items = units - P, grid = items < kNumSMs ? items : kNumSMs;
    const double t = (double)((items + grid - 1) / grid) + (kWgPairCost - 1.0) * (double)((P + grid - 1) / grid);
    if (t < best_t + 1e-9) { if (t < best_t) best_t = t; best = P; }
  }
  return best;
}

int choose_pairs(const Plan& p, int m_pairs, int mode) {
  const int groups = p.splits * m_pairs * p.taps * p.n_tiles;
  if (mode == 0 || groups == 0) return 0;
  if (mode == 2) return groups;
  const int units = p.m_tiles * p.n_tiles * p.taps * p.splits;
  int best = 0; double best_t = 1e30;
  for (int P = 0; P <= groups; ++P) {
    const double t = kPairCost * ((P + kNumSMs - 1) / kNumSMs) + (double)((units - 2 * P + kNumSMs - 1) / kNumSMs);
    if (t < best_t + 1e-9) { if (t < best_t) best_t = t; best = P; }
  }
  return best;
}

template <int BLOCK_N, int KIND>
int launch(const CUtensorMap& tdy, const CUtensorMap& tx, const WgArgs& a, cudaStream_t st) {
  using C = WCfg<BLOCK_N, KIND>;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(conv_wgrad_sm90_kernel<BLOCK_N, KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         C::kSmemBytes);
    if (e != cudaSuccess) { set_error("skd_conv2d_wgrad_sm100(attr)", e); return 0; }
    attr = true;
  }
  const int grid = a.items < kNumSMs ? a.items : kNumSMs;
  conv_wgrad_sm90_kernel<BLOCK_N, KIND><<<grid, kThreads, C::kSmemBytes, st>>>(tdy, tx, a);
  return finish("skd_conv2d_wgrad_sm100");
}

}  // namespace

extern "C" void skd_set_wgrad_linear(int on) { g_wgrad_linear = on ? 1 : 0; }
extern "C" void skd_conv_wgrad_last_plan(int* out) { for (int i = 0; i < 3; ++i) out[i] = g_last_plan[i]; }
extern "C" void skd_set_wgrad_pairing(int mode) { g_wgrad_pairing = mode < 0 ? 0 : (mode > 2 ? 2 : mode); }
extern "C" void skd_conv_wgrad_last_pairs(int* out) { out[0] = g_last_pairs; }

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
  g_last_plan[0] = p.bn; g_last_plan[1] = p.linear; g_last_plan[2] = p.splits;
  int ok = 1;
  if (Cout <= 64 && p.bn <= 64) {
    // one 64-row block per unit: any two units share a CTA, one per consumer warpgroup (BLOCK_N 128 would leave 2 stages)
    a.m_pairs = 0;
    a.pairs = choose_wg_pairs(units, g_wgrad_pairing);
    a.items = units - a.pairs;
    g_last_pairs = a.pairs;
    if (a.pairs) ok = p.bn == 64 ? launch<64, kWgPair>(tdy, tx, a, st) : launch<32, kWgPair>(tdy, tx, a, st);
    else ok = p.bn == 64 ? launch<64, kSingle>(tdy, tx, a, st) : launch<32, kSingle>(tdy, tx, a, st);
  } else {
    // pairs of Cout tiles share their X box: BLOCK_N 128 only, full tiles only (a ragged or odd last tile runs single)
    a.m_pairs = p.bn == 128 ? (Cout / kBlockM) / 2 : 0;
    a.pairs = choose_pairs(p, a.m_pairs, g_wgrad_pairing);
    if (a.pairs == 0) a.m_pairs = 0;
    const int singles = units - 2 * a.pairs;
    g_last_pairs = a.pairs;
    if (a.pairs) { a.items = a.pairs; ok = launch<128, kCoutPair>(tdy, tx, a, st); }
    a.items = singles;
    if (ok && singles) switch (p.bn) {
      case 128: ok = launch<128, kSingle>(tdy, tx, a, st); break;
      case 64: ok = launch<64, kSingle>(tdy, tx, a, st); break;
      default: ok = launch<32, kSingle>(tdy, tx, a, st); break;
    }
  }
  if (!ok) return 0;
  if (p.splits > 1) {
    const long long n4 = (long long)Cout * KH * KW * Cin / 4;
    long long b = (n4 + 255) / 256; if (b > kNumSMs * 8) b = kNumSMs * 8; if (b < 1) b = 1;
    splitk_reduce_kernel<<<(int)b, 256, 0, st>>>(workspace, dw, n4, p.splits);
  }
  return finish(who);
}
