// Training augmentation on the GPU: ONE kernel per batch does what `CSDataSet.__getitem__` / `VOCDataSet.__getitem__` do on the CPU
// after the two cv2.imread calls (reference dataset/datasets.py:45-81, 175-206): label table (Cityscapes id -> trainId; VOC: none),
// cv2.resize (uint8 INTER_LINEAR for the image, INTER_NEAREST for the label) by the drawn scale factor, mean subtraction, zero /
// ignore-label padding to the crop size, crop, mirror, HWC -> CHW.  Only the crop's pixels are ever computed: the reference resizes
// the whole 1024 x 2048 image (up to 2150 x 4301) and then throws away all but 512 x 1024 of it.
//
// Mean subtraction is (float)((double)p - mean[c]) with the mean in double.  numpy's `float32 image -= mean` subtracts in float32 for
// a float32 mean (then p - m is exact in double, since p is an integer in 0..255, and the one rounding is float32's: bit-identical)
// and in double for a tuple of Python numbers (VOCDataSet's default (128, 128, 128)); the caller passes the mean with numpy's type.
//
// Bit-exact with OpenCV's fixed-point path (modules/imgproc/src/resize.cpp, opencv-python 4.13.0 in this image; restated in
// oracle/dataset_port.py and pinned there against cv2 and against the unmodified reference loader):
//   dsize = cvRound(size * f);  scale = 1 / f (double)
//   fx = float((dx + 0.5) * scale - 0.5);  sx = floor(fx);  fx -= sx;  sx < 0 -> (0, 0);  sx >= W - 1 -> (W - 1, 0)        [columns]
//   rows: same, source rows clipped to [0, H - 1], weights kept
//   a = short(round((1 - fx) * 2048)), short(round(fx * 2048));   row value r = S[sx] * a0 + S[sx + 1] * a1   (int32)
//   out = uint8(( ((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16) + 2 ) >> 2)
//   nearest: min(floor(d * scale), size - 1)
// Double / float operations are issued with explicit round-to-nearest intrinsics so that no FMA contraction changes a rounding.
// HBM-bound and tiny: per 8 x 512 x 1024 batch it reads <= 4 source pixels per output pixel (L2-resident rows) and writes 67 MB.
#include "common.cuh"
#include "skd.h"

using namespace skd;

namespace {
constexpr int kMaxSamples = 32;

struct DevSample {
  const unsigned char* image; const unsigned char* label;
  double inv;                                     // 1 / f_scale
  int src_h, src_w, scaled_h, scaled_w, h_off, w_off, flip, scale_on;
};
struct DevBatch { DevSample s[kMaxSamples]; double mean[3]; int ignore_label; unsigned char table[256]; };

__device__ __forceinline__ void linear_coef(int d, double inv, int size, bool reset_at_border, int& s, int& c0, int& c1) {
  float f = __double2float_rn(__dadd_rn(__dmul_rn(__dadd_rn((double)d, 0.5), inv), -0.5));
  s = __float2int_rd(f);
  f = __fsub_rn(f, (float)s);
  if (reset_at_border) {
    if (s < 0) { f = 0.f; s = 0; }
    if (s >= size - 1) { f = 0.f; s = size - 1; }
  }
  c0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
  c1 = __float2int_rn(__fmul_rn(f, 2048.f));
}

template <typename LabelT>
__global__ void __launch_bounds__(256)
cs_augment_kernel(const __grid_constant__ DevBatch b, int crop_h, int crop_w, float* __restrict__ images, LabelT* __restrict__ labels) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, n = blockIdx.z;
  if (x >= crop_w) return;
  const DevSample& sp = b.s[n];
  const int cx = sp.flip < 0 ? crop_w - 1 - x : x;                 // mirror acts on the cropped image (datasets.py:203-206)
  const int py = sp.h_off + y, px = sp.w_off + cx;                 // position in the padded, scaled image
  float v0 = 0.f, v1 = 0.f, v2 = 0.f;                              // pad value of the mean-subtracted image (datasets.py:186-188)
  int lab = b.ignore_label;
  if (py < sp.scaled_h && px < sp.scaled_w) {
    int p0, p1, p2, l;
    if (sp.scale_on) {
      int sx, sy, a0, a1, b0, b1;
      linear_coef(px, sp.inv, sp.src_w, true, sx, a0, a1);
      linear_coef(py, sp.inv, sp.src_h, false, sy, b0, b1);
      const int sx1 = min(sx + 1, sp.src_w - 1);
      const int y0 = min(max(sy, 0), sp.src_h - 1), y1 = min(max(sy + 1, 0), sp.src_h - 1);
      const unsigned char* r0 = sp.image + (size_t)y0 * sp.src_w * 3;
      const unsigned char* r1 = sp.image + (size_t)y1 * sp.src_w * 3;
      int o[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const int h0 = (int)r0[sx * 3 + c] * a0 + (int)r0[sx1 * 3 + c] * a1;
        const int h1 = (int)r1[sx * 3 + c] * a0 + (int)r1[sx1 * 3 + c] * a1;
        o[c] = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
        o[c] = min(max(o[c], 0), 255);
      }
      p0 = o[0]; p1 = o[1]; p2 = o[2];
      const int nx = min(__double2int_rd(__dmul_rn((double)px, sp.inv)), sp.src_w - 1);
      const int ny = min(__double2int_rd(__dmul_rn((double)py, sp.inv)), sp.src_h - 1);
      l = sp.label[(size_t)ny * sp.src_w + nx];
    } else {
      const unsigned char* r = sp.image + ((size_t)py * sp.src_w + px) * 3;
      p0 = r[0]; p1 = r[1]; p2 = r[2];
      l = sp.label[(size_t)py * sp.src_w + px];
    }
    v0 = __double2float_rn(__dsub_rn((double)p0, b.mean[0]));
    v1 = __double2float_rn(__dsub_rn((double)p1, b.mean[1]));
    v2 = __double2float_rn(__dsub_rn((double)p2, b.mean[2]));
    lab = b.table[l];
  }
  const size_t plane = (size_t)crop_h * crop_w, o = (size_t)y * crop_w + x;
  float* img = images + (size_t)n * 3 * plane + o;
  img[0] = v0; img[plane] = v1; img[2 * plane] = v2;
  labels[(size_t)n * plane + o] = (LabelT)lab;
}

// `who`: the C entry point whose name errors are reported under
int augment_batch(const char* who, int n, const skd_cs_sample* samples, int crop_h, int crop_w, const double* mean_bgr,
                  const unsigned char* label_table, int ignore_label, float* images, void* labels, int labels_int64, cudaStream_t st) {
  if (n <= 0) return 1;
  if (!samples || !mean_bgr || !images || !labels || crop_h <= 0 || crop_w <= 0) { set_error_msg(who, "bad arguments"); return 0; }
  const size_t plane = (size_t)crop_h * crop_w;
  int kernels = 0;
  for (int base = 0; base < n; base += kMaxSamples) {
    const int cnt = n - base < kMaxSamples ? n - base : kMaxSamples;
    DevBatch b;
    for (int i = 0; i < cnt; ++i) {
      const skd_cs_sample& s = samples[base + i];
      const bool scale_on = s.f_scale > 0.0;
      if (!s.image || !s.label || s.src_h <= 0 || s.src_w <= 0 || s.h_off < 0 || s.w_off < 0) { set_error_msg(who, "bad sample"); return 0; }
      DevSample& d = b.s[i];
      d.image = s.image; d.label = s.label; d.src_h = s.src_h; d.src_w = s.src_w;
      d.scale_on = scale_on ? 1 : 0;
      d.inv = scale_on ? 1.0 / s.f_scale : 1.0;
      d.scaled_h = scale_on ? s.scaled_h : s.src_h; d.scaled_w = scale_on ? s.scaled_w : s.src_w;
      d.h_off = s.h_off; d.w_off = s.w_off; d.flip = s.flip;
    }
    for (int c = 0; c < 3; ++c) b.mean[c] = mean_bgr[c];
    b.ignore_label = ignore_label;
    for (int i = 0; i < 256; ++i) b.table[i] = label_table ? label_table[i] : (unsigned char)i;
    const dim3 grid((crop_w + 255) / 256, crop_h, cnt);
    float* img = images + (size_t)base * 3 * plane;
    if (labels_int64) cs_augment_kernel<long long><<<grid, 256, 0, st>>>(b, crop_h, crop_w, img, reinterpret_cast<long long*>(labels) + (size_t)base * plane);
    else cs_augment_kernel<float><<<grid, 256, 0, st>>>(b, crop_h, crop_w, img, reinterpret_cast<float*>(labels) + (size_t)base * plane);
    ++kernels;
  }
  return finish(who, kernels);
}
}  // namespace

extern "C" int skd_augment_batch(int n, const skd_cs_sample* samples, int crop_h, int crop_w, const double* mean_bgr,
                                 const unsigned char* label_table, int ignore_label, float* images, void* labels, int labels_int64,
                                 cudaStream_t st) {
  return augment_batch("skd_augment_batch", n, samples, crop_h, crop_w, mean_bgr, label_table, ignore_label, images, labels,
                       labels_int64, st);
}

// datasets.py:146-151: Cityscapes label ids -> train ids (ids >= 34 pass through), the mean as given in float32
extern "C" int skd_cs_augment_batch(int n, const skd_cs_sample* samples, int crop_h, int crop_w, const float* mean_bgr, int ignore_label,
                                    float* images, void* labels, int labels_int64, cudaStream_t st) {
  if (n <= 0) return 1;
  if (!mean_bgr) { set_error_msg("skd_cs_augment_batch", "bad arguments"); return 0; }
  unsigned char to_train[256], to_label[256];
  skd_cityscapes_id_tables(to_train, to_label);
  const double mean[3] = {mean_bgr[0], mean_bgr[1], mean_bgr[2]};
  return augment_batch("skd_cs_augment_batch", n, samples, crop_h, crop_w, mean, to_train, ignore_label, images, labels, labels_int64, st);
}
