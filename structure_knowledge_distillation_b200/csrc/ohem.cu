// Online hard-example mining (OhemCrossEntropy2d, utils/criterion.py:11-90) for sm_90a: the threshold pass.
//   * grid sample: the reference zooms the full-resolution softmax with scipy.ndimage.zoom(order=1) and the labels with
//     zoom(order=0) to a 1/factor grid (criterion.py:20-24), then reads the zoomed probability of the zoomed label.  One thread
//     per grid point restates that exactly: source coordinate o * r in double with r = (in - 1) / (out - 1), mode 'constant'
//     (a coordinate past in - 1 reads 0 for probability AND label), order 0 = floor(c + 0.5), order 1 = the four neighbours
//     combined in double in scipy's summation order.  The four full-resolution probabilities come straight from the
//     low-resolution logits (align_corners upsample, fp32 softmax), so nothing at full resolution is materialised; they are computed
//     as the row kernel that applies the mask computes them (common.cuh up_label_prob), so a grid point that lies on a pixel holds
//     that pixel's probability bit for bit.
//   * radix select: the exact k-th smallest zoomed probability (criterion.py:41-47) over the float bits (probabilities are >= 0,
//     so their bit patterns order like the values; invalid points hold +inf and sort last), four 8-bit passes of integer
//     histograms -- deterministic, multi-CTA, and without a host round trip, so the step stays capturable in a CUDA graph.
// The masked cross entropy that consumes the threshold is the DSN row kernel of losses.cu (skd_ohem_dsn_ce_fwd_train).
#include "common.cuh"
#include "skd.h"

using namespace skd;

namespace {

constexpr int kMaxClasses = 32;
constexpr int kBins = 256;

__global__ void __launch_bounds__(256)
ohem_grid_kernel(const float* __restrict__ L, long long sn, long long sc, long long sp, const long long* __restrict__ labels,
                 int N, int C, int h, int w, int H, int W, int gh, int gw, int ignore, float* __restrict__ pred,
                 long long* __restrict__ glabels, int* __restrict__ nvalid) {
  // scipy's zoom arithmetic (common.cuh: zoom_ratio / zoom_axis / zoom_lerp)
  const double ry = zoom_ratio(H, gh), rx = zoom_ratio(W, gw);
  const float sy = H > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f, sx = W > 1 ? (float)(w - 1) / (float)(W - 1) : 0.f;
  const long long total = (long long)N * gh * gw;
  int valid = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int gx = (int)(i % gw); const long long r = i / gw; const int gy = (int)(r % gh), n = (int)(r / gh);
    const ZoomAxis ay = zoom_axis(gy, ry, H), ax = zoom_axis(gx, rx, W);
    const bool outside = ay.outside || ax.outside;                             // mode 'constant', cval 0
    long long lab = 0;
    if (!outside) {
      int iy = (int)floor(__dadd_rn(ay.c, 0.5)), ix = (int)floor(__dadd_rn(ax.c, 0.5));
      iy = min(iy, H - 1); ix = min(ix, W - 1);
      lab = labels[((long long)n * H + iy) * W + ix];
    }
    if (glabels) glabels[i] = lab;
    float v = INFINITY;
    if (lab != ignore) {
      ++valid;
      v = 0.f;
      if (!outside) {
        const int lb = (int)lab;
        // p[lab] at the four full-resolution pixels, computed as the row kernel that applies the mask computes them
        const Bilin by0 = bilin(ay.i0, sy, h), by1 = bilin(ay.i1, sy, h), bx0 = bilin(ax.i0, sx, w), bx1 = bilin(ax.i1, sx, w);
        const double p00 = up_label_prob<kMaxClasses>(L, sn, sc, sp, n, C, w, by0, bx0, lb);
        const double p01 = up_label_prob<kMaxClasses>(L, sn, sc, sp, n, C, w, by0, bx1, lb);
        const double p10 = up_label_prob<kMaxClasses>(L, sn, sc, sp, n, C, w, by1, bx0, lb);
        const double p11 = up_label_prob<kMaxClasses>(L, sn, sc, sp, n, C, w, by1, bx1, lb);
        v = (float)zoom_lerp(p00, p01, p10, p11, ay, ax);                     // the zoomed array has the input's dtype
      }
    }
    pred[i] = v;
  }
  for (int o = 16; o > 0; o >>= 1) valid += __shfl_xor_sync(0xffffffffu, valid, o);
  if ((threadIdx.x & 31) == 0 && valid) atomicAdd(nvalid, valid);
}

// state: [0] prefix bits found so far, [1] rank still to find inside the prefix, [2] 1 = threshold already decided
__global__ void __launch_bounds__(256)
ohem_hist_kernel(const float* __restrict__ vals, long long n, int pass, const unsigned* __restrict__ state, unsigned* __restrict__ hist) {
  __shared__ unsigned sh[kBins];
  if (pass > 0 && state[2]) return;
  for (int i = threadIdx.x; i < kBins; i += blockDim.x) sh[i] = 0;
  __syncthreads();
  const int shift = 24 - 8 * pass;
  const unsigned mask = pass == 0 ? 0u : (0xFFFFFFFFu << (shift + 8));
  const unsigned prefix = pass == 0 ? 0u : state[0];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned b = __float_as_uint(__ldg(vals + i));
    if ((b & mask) == prefix) atomicAdd(&sh[(b >> shift) & 0xFFu], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kBins; i += blockDim.x)
    if (sh[i]) atomicAdd(&hist[i], sh[i]);
}

// one thread walks the 256 bins: the digit whose cumulative count passes the rank.  Pass 0 first applies the rule of
// criterion.py:36-47 (1.0 when min_kept >= num_valid, thresh when min_kept <= 0); pass 3 writes max(thresh, k-th value)
__global__ void ohem_select_kernel(const unsigned* __restrict__ hist, int pass, const int* __restrict__ nvalid, int min_kept,
                                   float thresh, unsigned* __restrict__ state, float* __restrict__ threshold) {
  if (threadIdx.x != 0) return;
  if (pass == 0) {
    const int nv = *nvalid;
    state[0] = 0u; state[2] = 0u;
    if (min_kept >= nv) { *threshold = 1.f; state[2] = 1u; return; }
    if (min_kept <= 0) { *threshold = thresh; state[2] = 1u; return; }
    state[1] = (unsigned)(min(nv, min_kept) - 1);
  } else if (state[2]) {
    return;
  }
  const int shift = 24 - 8 * pass;
  unsigned k = state[1], cum = 0u;
  int d = 0;
  for (; d < kBins - 1; ++d) {
    if (cum + hist[d] > k) break;
    cum += hist[d];
  }
  state[0] |= (unsigned)d << shift;
  state[1] = k - cum;
  if (pass == 3) {
    const float v = __uint_as_float(state[0]);
    *threshold = v > thresh ? v : thresh;
  }
}

int grid_blocks(long long total) {
  long long b = (total + 255) / 256;
  if (b > kNumSMs * 8) b = kNumSMs * 8;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace

extern "C" int skd_ohem_grid_sample(int N, int C, int h, int w, int H, int W, int gh, int gw, const float* logits, long long sn,
                                    long long sc, long long sp, const long long* labels, int ignore_index, float* pred,
                                    long long* grid_labels, int* nvalid, cudaStream_t st) {
  if (C > kMaxClasses) { set_error_msg("skd_ohem_grid_sample", "C > 32 classes unsupported"); return 0; }
  if (gh < 1 || gw < 1) { set_error_msg("skd_ohem_grid_sample", "empty threshold grid (factor larger than the label map)"); return 0; }
  cudaMemsetAsync(nvalid, 0, sizeof(int), st);
  const long long total = (long long)N * gh * gw;
  ohem_grid_kernel<<<grid_blocks(total), 256, 0, st>>>(logits, sn, sc, sp, labels, N, C, h, w, H, W, gh, gw, ignore_index, pred,
                                                       grid_labels, nvalid);
  return finish("skd_ohem_grid_sample");
}

extern "C" long long skd_ohem_threshold_workspace_ints(void) { return 4LL * kBins + 4; }

extern "C" int skd_ohem_threshold(long long n, const float* pred, const int* nvalid, int min_kept, float thresh, float* threshold,
                                  int* workspace, cudaStream_t st) {
  unsigned* hist = reinterpret_cast<unsigned*>(workspace);
  unsigned* state = hist + 4 * kBins;
  cudaMemsetAsync(hist, 0, 4 * kBins * sizeof(unsigned), st);
  const int blocks = grid_blocks(n);
  for (int pass = 0; pass < 4; ++pass) {
    ohem_hist_kernel<<<blocks, 256, 0, st>>>(pred, n, pass, state, hist + pass * kBins);
    ohem_select_kernel<<<1, 32, 0, st>>>(hist + pass * kBins, pass, nvalid, min_kept, thresh, state, threshold);
  }
  return finish("skd_ohem_threshold", 8);
}
