// Evaluation kernels (networks/evaluate.py:75-206): bilinear (align_corners) up-sampling of the class scores of one tile
// accumulated into the full-image score buffer (predict_sliding :86-113 / predict_whole :115-122), then arg-max and the confusion
// matrix (get_confusion_matrix :143-160, ignore label 255) -- no score tensor ever goes to the host.
// Multi-scale / flip evaluation (predict_multiscale :115-134) and test-split prediction maps (:187-191, dataset/datasets.py:234-250):
//   * zoom_image_kernel: scipy.ndimage.zoom(image, (1, 1, s, s), order=1, prefilter=False) bit for bit (common.cuh zoom_*), written
//     as the network's 4-channel NHWC input, with the mirrored copy as batch item 1;
//   * upsample_acc_kernel<kWeightedPair>: 0.5 * (up(L0) + up(L1) mirrored) of that batch-2 forward, in the reference's order;
//   * argmax_lut_kernel: the whole-image prediction map (train ids or, through a table, Cityscapes label ids) + the confusion matrix;
//   * cs_test_preprocess_kernel: CSDataTestSet's mean subtraction in double and bottom / right zero padding.
#include "common.cuh"
#include "skd.h"

using namespace skd;

namespace {

enum AccMode : int { kPlain = 0, kWeighted = 1, kWeightedPair = 2 };

// full[(y1+y)*W + x1+x][c] += bilinear(logits)[c][y][x] for y < vh, x < vw (the tile may be padded beyond the image: only the valid
// part is accumulated, evaluate.py:106-110).  kWeighted: += weight * up(L0); kWeightedPair: += weight * 0.5f * (up(L0)[y][x] +
// up(L1)[y][TW-1-x]) with L1 = the forward of the mirrored image (batch item 1, `sn` floats further), evaluate.py:130-131
template <int MODE>
__global__ void __launch_bounds__(256)
upsample_acc_kernel(int C, int h, int w, const float* __restrict__ L, long long sn, long long sc, long long sp, int TH, int TW, int vh,
                    int vw, float* __restrict__ full, int W, int y1, int x1, float weight) {
  const long long total = (long long)vh * vw * C;
  const float ry = TH > 1 ? (float)(h - 1) / (float)(TH - 1) : 0.f, rx = TW > 1 ? (float)(w - 1) / (float)(TW - 1) : 0.f;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % C); const long long r = i / C;
    const int x = (int)(r % vw), y = (int)(r / vw);
    const float v = up_at(L + c * sc, sp, h, w, ry, rx, y, x);
    float* dst = full + ((long long)(y1 + y) * W + x1 + x) * C + c;
    if (MODE == kPlain) {
      *dst += v;
    } else if (MODE == kWeighted) {
      *dst += weight * v;
    } else {
      const float m = up_at(L + sn + c * sc, sp, h, w, ry, rx, y, TW - 1 - x);
      *dst += weight * (0.5f * (v + m));
    }
  }
}

__global__ void __launch_bounds__(256)
argmax_confusion_kernel(int H, int W, int C, const float* __restrict__ full, const long long* __restrict__ gt, long long gt_row, int vh,
                        int vw, int ignore, unsigned long long* conf, unsigned char* __restrict__ pred) {
  const long long total = (long long)vh * vw;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int x = (int)(i % vw), y = (int)(i / vw);
    const float* p = full + ((long long)y * W + x) * C;
    int best = 0; float bv = p[0];
    for (int c = 1; c < C; ++c) { const float v = p[c]; if (v > bv) { bv = v; best = c; } }     // first maximum, like np.argmax
    if (pred) pred[(long long)y * W + x] = (unsigned char)best;
    if (gt) {
      const long long g = gt[(long long)y * gt_row + x];
      if (g != ignore && g >= 0 && g < C) atomicAdd(conf + g * C + best, 1ull);
    }
  }
}

int blocks_for(long long n) { long long b = (n + 255) / 256; if (b > kNumSMs * 8) b = kNumSMs * 8; if (b < 1) b = 1; return (int)b; }

// argmax_confusion_kernel over the union of two regions: the prediction map pred[ph][pw] (whole image, evaluate.py:187-191; through
// `lut` when given, :188) and the confusion matrix of the valid region vh x vw (:194-198)
__global__ void __launch_bounds__(256)
argmax_lut_kernel(int W, int C, const float* __restrict__ full, const long long* __restrict__ gt, long long gt_row, int vh, int vw, int ignore,
                  unsigned long long* conf, unsigned char* __restrict__ pred, int ph, int pw, const unsigned char* __restrict__ lut, int rh, int rw) {
  const long long total = (long long)rh * rw;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int x = (int)(i % rw), y = (int)(i / rw);
    const float* p = full + ((long long)y * W + x) * C;
    int best = 0; float bv = p[0];
    for (int c = 1; c < C; ++c) { const float v = p[c]; if (v > bv) { bv = v; best = c; } }     // first maximum, like np.argmax
    if (pred && y < ph && x < pw) pred[(long long)y * pw + x] = lut ? __ldg(lut + best) : (unsigned char)best;
    if (gt && y < vh && x < vw) {
      const long long g = gt[(long long)y * gt_row + x];
      if (g != ignore && g >= 0 && g < C) atomicAdd(conf + g * C + best, 1ull);
    }
  }
}

// scipy.ndimage.zoom(image, (1, 1, s, s), order=1, prefilter=False) of the float32 (1, 3, H, W) image (evaluate.py:127) -> out[y][x] =
// (c0, c1, c2, 0), the 4-channel NHWC input Res_pspnet.forward takes; flip: out[OH*OW + y*OW + OW-1-x] gets the same pixel (:130)
__global__ void __launch_bounds__(256)
zoom_image_kernel(const float* __restrict__ img, int H, int W, int OH, int OW, double ry, double rx, int flip, float4* __restrict__ out) {
  const long long total = (long long)OH * OW, plane = (long long)H * W;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int x = (int)(i % OW), y = (int)(i / OW);
    const ZoomAxis ay = zoom_axis(y, ry, H), ax = zoom_axis(x, rx, W);
    float v[3] = {0.f, 0.f, 0.f};                                             // mode 'constant': outside reads 0
    if (!ay.outside && !ax.outside) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float* p = img + c * plane;
        v[c] = (float)zoom_lerp(__ldg(p + (long long)ay.i0 * W + ax.i0), __ldg(p + (long long)ay.i0 * W + ax.i1),
                                __ldg(p + (long long)ay.i1 * W + ax.i0), __ldg(p + (long long)ay.i1 * W + ax.i1), ay, ax);
      }
    }
    const float4 o = make_float4(v[0], v[1], v[2], 0.f);
    out[i] = o;
    if (flip) out[total + (long long)y * OW + (OW - 1 - x)] = o;
  }
}

struct Mean3 { double m[3]; };

// CSDataTestSet.__getitem__ after cv2.imread (dataset/datasets.py:239-249): float32 image minus the mean tuple (numpy computes in
// double and rounds once to float32), zero padding on the bottom / right up to (OH, OW), HWC -> CHW
__global__ void __launch_bounds__(256)
cs_test_preprocess_kernel(const unsigned char* __restrict__ img, int H, int W, int OH, int OW, Mean3 mean, float* __restrict__ out) {
  const long long plane = (long long)OH * OW, total = 3 * plane;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int c = (int)(i / plane); const long long r = i - c * plane;
    const int x = (int)(r % OW), y = (int)(r / OW);
    float v = 0.f;
    if (y < H && x < W) {
      const double m = c == 0 ? mean.m[0] : (c == 1 ? mean.m[1] : mean.m[2]);
      v = __double2float_rn(__dsub_rn((double)__ldg(img + ((long long)y * W + x) * 3 + c), m));
    }
    out[i] = v;
  }
}

}  // namespace

extern "C" int skd_eval_upsample_accumulate(int C, int h, int w, const float* logits, long long sc, long long sp, int tile_h, int tile_w,
                                            int valid_h, int valid_w, float* full, int W, int y1, int x1, cudaStream_t st) {
  if (valid_h <= 0 || valid_w <= 0) return 1;
  upsample_acc_kernel<kPlain><<<blocks_for((long long)valid_h * valid_w * C), 256, 0, st>>>(C, h, w, logits, 0, sc, sp, tile_h, tile_w, valid_h,
                                                                                           valid_w, full, W, y1, x1, 1.f);
  return finish("skd_eval_upsample_accumulate");
}

extern "C" int skd_eval_argmax_confusion(int H, int W, int C, const float* full, const long long* gt, long long gt_row, int valid_h,
                                         int valid_w, int ignore_index, long long* confusion, unsigned char* pred, cudaStream_t st) {
  if (valid_h <= 0 || valid_w <= 0) return 1;
  argmax_confusion_kernel<<<blocks_for((long long)valid_h * valid_w), 256, 0, st>>>(H, W, C, full, gt, gt_row, valid_h, valid_w, ignore_index,
                                                                                   reinterpret_cast<unsigned long long*>(confusion), pred);
  return finish("skd_eval_argmax_confusion");
}

extern "C" int skd_eval_upsample_accumulate_ms(int C, int h, int w, const float* logits, long long sn, long long sc, long long sp, int tile_h,
                                               int tile_w, int valid_h, int valid_w, float* full, int W, float weight, int paired,
                                               cudaStream_t st) {
  if (valid_h <= 0 || valid_w <= 0) return 1;
  if (valid_w > tile_w || valid_h > tile_h) { set_error_msg("skd_eval_upsample_accumulate_ms", "valid region larger than the tile"); return 0; }
  const int blocks = blocks_for((long long)valid_h * valid_w * C);
  if (paired)
    upsample_acc_kernel<kWeightedPair><<<blocks, 256, 0, st>>>(C, h, w, logits, sn, sc, sp, tile_h, tile_w, valid_h, valid_w, full, W, 0, 0,
                                                               weight);
  else
    upsample_acc_kernel<kWeighted><<<blocks, 256, 0, st>>>(C, h, w, logits, sn, sc, sp, tile_h, tile_w, valid_h, valid_w, full, W, 0, 0, weight);
  return finish("skd_eval_upsample_accumulate_ms");
}

extern "C" int skd_eval_argmax_confusion_lut(int H, int W, int C, const float* full, const long long* gt, long long gt_row, int valid_h,
                                             int valid_w, int ignore_index, long long* confusion, unsigned char* pred, int pred_h, int pred_w,
                                             const unsigned char* lut, cudaStream_t st) {
  if (lut && C > 256) { set_error_msg("skd_eval_argmax_confusion_lut", "a label table needs C <= 256"); return 0; }
  if (!gt) valid_h = valid_w = 0;
  if (!pred) pred_h = pred_w = 0;
  if (valid_h > H || valid_w > W || pred_h > H || pred_w > W) {
    set_error_msg("skd_eval_argmax_confusion_lut", "region larger than the score buffer");
    return 0;
  }
  const int rh = max(valid_h, pred_h), rw = max(valid_w, pred_w);
  if (rh <= 0 || rw <= 0) return 1;
  argmax_lut_kernel<<<blocks_for((long long)rh * rw), 256, 0, st>>>(W, C, full, gt, gt_row, valid_h, valid_w, ignore_index,
                                                                  reinterpret_cast<unsigned long long*>(confusion), pred, pred_h, pred_w, lut,
                                                                  rh, rw);
  return finish("skd_eval_argmax_confusion_lut");
}

extern "C" int skd_eval_zoom_image(int H, int W, const float* image, int out_h, int out_w, int flip, float* out, cudaStream_t st) {
  if (H < 1 || W < 1 || out_h < 1 || out_w < 1) { set_error_msg("skd_eval_zoom_image", "empty image"); return 0; }
  zoom_image_kernel<<<blocks_for((long long)out_h * out_w), 256, 0, st>>>(image, H, W, out_h, out_w, zoom_ratio(H, out_h), zoom_ratio(W, out_w),
                                                                        flip, reinterpret_cast<float4*>(out));
  return finish("skd_eval_zoom_image");
}

extern "C" int skd_cs_test_preprocess(int H, int W, const unsigned char* image, const double* mean_bgr, int out_h, int out_w, float* out,
                                      cudaStream_t st) {
  if (out_h < H || out_w < W) { set_error_msg("skd_cs_test_preprocess", "output smaller than the image (the test set pads, never crops)"); return 0; }
  Mean3 m;
  for (int c = 0; c < 3; ++c) m.m[c] = mean_bgr[c];
  cs_test_preprocess_kernel<<<blocks_for(3LL * out_h * out_w), 256, 0, st>>>(image, H, W, out_h, out_w, m, out);
  return finish("skd_cs_test_preprocess");
}

extern "C" int skd_cityscapes_id_tables(unsigned char* to_train, unsigned char* to_label) {
  static const unsigned char kTrainIdHost[kCityscapesIds] = SKD_CITYSCAPES_TRAINID;
  for (int i = 0; i < 256; ++i) {
    to_train[i] = i < kCityscapesIds ? kTrainIdHost[i] : (unsigned char)i;
    to_label[i] = (unsigned char)i;
  }
  // id2trainId(..., reverse=True) (evaluate.py:30-38): label_copy[label == train] = id over the table in order, the last id wins
  for (int id = 0; id < kCityscapesIds; ++id) to_label[kTrainIdHost[id]] = (unsigned char)id;
  return 1;
}
