/* libskd_b200.so -- C ABI of the Hopper-native (sm_90a) structured-distillation step.
 *
 * Drop-in boundary for the hot path of irfanICMLL/structure_knowledge_distillation (NetModel.optimize_parameters,
 * networks/kd_model.py:167-173).  Conventions are the reference's own native-ABI conventions
 * (libs/src/bn.h:7-19, libs/src/bn.cu:237-300, libs/src/lib_cffi.cpp:36-111):
 *   - plain pointers and sizes only, fp32 data, no torch types;
 *   - every function returns 1 on success and 0 on error (the Python side turns 0 into
 *     RuntimeError("CUDA Error encountered in <fn>"), libs/functions.py:13-16); skd_last_error() gives the text;
 *   - no allocation, no synchronisation, no hidden state: the caller owns and pre-sizes every buffer (workspaces
 *     included) and picks the stream; a NULL pointer means "tensor absent" (no affine / gradient not wanted);
 *   - re-entrant and device-agnostic: work is issued on the caller's current device.
 * Activation codes: 0 none, 1 leaky_relu(slope), 2 elu, 3 relu.
 * "NHWC" tensors are [N*H*W rows][C] with an explicit row pitch in floats where noted (channel slices of a concat
 * buffer are addressed in place).  (sn, sc, sp) are element strides over (image, channel, pixel).
 */
#ifndef SKD_B200_H_
#define SKD_B200_H_

#include <cuda_runtime_api.h>

#ifdef __cplusplus
extern "C" {
#endif

const char* skd_last_error(void);
int skd_version(void);
long long skd_kernel_launches(void);   /* number of kernels this library has launched in this process */

/* ---- A. InPlace-ABN native ABI: one-for-one replacements of libs/src/bn.h:7-19 ((N, C, S) NCHW views) ---- */
/* replaces _bn_mean_var_cuda  (bn.h:7,  bn.cu:125-138,237-250): per-channel mean and BIASED variance */
int skd_bn_mean_var_cuda(int N, int C, int S, const float* x, float* mean, float* var, cudaStream_t);
/* replaces _bn_forward_cuda   (bn.h:8-9, bn.cu:140-165,252-268): y=(x-mean)*rsqrt(var+eps); z=y*(|w|+eps)+b; y,z may alias x */
int skd_bn_forward_cuda(int N, int C, int S, const float* x, const float* mean, const float* var, const float* weight,
                        const float* bias, float* y, float* z, float eps, cudaStream_t);
/* replaces _bn_edz_eydz_cuda  (bn.h:10-11, bn.cu:167-184,270-283): edz=mean(dz), eydz=mean(y*dz), y recovered from z */
int skd_bn_edz_eydz_cuda(int N, int C, int S, const float* z, const float* dz, const float* weight, const float* bias,
                         float* edz, float* eydz, float eps, cudaStream_t);
/* replaces _bn_backward_cuda  (bn.h:12-14, bn.cu:186-232,285-300): dx; dweight/dbias are += into caller-zeroed buffers */
int skd_bn_backward_cuda(int N, int C, int S, const float* dz, const float* z, const float* var, const float* weight,
                         const float* bias, const float* edz, const float* eydz, float* dx, float* dweight, float* dbias,
                         float eps, cudaStream_t);
/* replace _leaky_relu_cuda, _leaky_relu_backward_cuda, _elu_cuda, _elu_backward_cuda, _elu_inv_cuda (bn.h:15-19, bn.cu:302-377) */
int skd_leaky_relu_cuda(int N, float* x, float slope, cudaStream_t);
int skd_leaky_relu_backward_cuda(int N, const float* x, float* dx, float slope, cudaStream_t);
int skd_elu_cuda(int N, float* x, cudaStream_t);
int skd_elu_backward_cuda(int N, const float* x, float* dx, cudaStream_t);
int skd_elu_inv_cuda(int N, float* x, cudaStream_t);

/* ---- B. fused NHWC ABN used between the wgmma convolutions (same math: libs/functions.py:81-109,113-162) ---- */
int skd_abn_num_splits(long long P, int C);   /* workspace = splits*C*6 floats (stats), splits*C*2 floats (bwd reduce) */
/* batch stats of x[P][C] -> mean,var (biased); running EMA with n/(n-1) (functions.py:90-91); scale=(|w|+eps)*rsqrt(var+eps),
   shift=b-mean*scale for the apply pass.  One pass of sums shifted by the first row, kept in float and in double; a channel whose
   first row lies more than 8 std from its mean takes the double sums.  workspace: 16-byte aligned */
int skd_abn_stats_nhwc(long long P, int C, const float* x, const float* weight, const float* bias, float eps, float momentum,
                       float* running_mean, float* running_var, float* mean, float* var, float* scale, float* shift,
                       float* workspace, int splits, cudaStream_t);
/* eval-mode / frozen-teacher folding of running statistics into scale/shift */
int skd_abn_fold(int C, const float* mean, const float* var, const float* weight, const float* bias, float eps, float* scale,
                 float* shift, cudaStream_t);
/* out = act(x*scale+shift (+residual)) (*chan_mul[n][c] : Dropout2d mask, S = rows per image); out_pitch in floats;
   round_tf32: store TF32 values rounded to nearest even (the tensor feeds a tensor-core convolution) */
int skd_abn_apply_nhwc(long long P, int C, int S, const float* x, float* out, int out_pitch, const float* scale,
                       const float* shift, int act, float slope, const float* residual, const float* chan_mul,
                       int round_tf32, cudaStream_t);
/* edz, eydz (means) and dweight=sign(w)*sum(y*dz), dbias=sum(dz) (bn.cu:214-230); dz = dout*chan_mul*act'(out).
   out may be NULL for sign-only activations without a fused residual (none / relu / leaky): the sign is then recomputed from
   x*scale + shift (the apply pass's own FMA) and the stored activation output is never read. */
int skd_abn_bwd_reduce_nhwc(long long P, int C, int S, const float* x, const float* out, const float* dout, const float* mean,
                            const float* var, const float* weight, float eps, int act, float slope, const float* chan_mul,
                            float* edz, float* eydz, float* dweight, float* dbias, float* workspace, int splits,
                            const float* scale, const float* shift, cudaStream_t);
/* dx = (dz - edz - y*eydz)*(|w|+eps)*rsqrt(var+eps); dres = dz (gradient of the residual input), either may be NULL... dx not */
int skd_abn_bwd_dx_nhwc(long long P, int C, int S, const float* x, const float* out, const float* dout, float* dx, float* dres,
                        const float* mean, const float* var, const float* weight, const float* edz, const float* eydz,
                        float eps, int act, float slope, const float* chan_mul, int round_tf32, const float* scale,
                        const float* shift, cudaStream_t);

/* ---- C. losses ---- */
int skd_loss_max_partials(void);              /* doubles of workspace the reductions below may use (x2 for dsn_ce) */
/* CriterionPixelWise.forward (utils/criterion.py:219-226): loss = inv_hw * sum_pixels -softmax(T).log_softmax(S) */
int skd_pixelwise_fwd(int N, int C, int HW, const float* S, long long s_sn, long long s_sc, long long s_sp, const float* T,
                      long long t_sn, long long t_sc, long long t_sp, float inv_hw, float* loss, double* workspace, cudaStream_t);
int skd_pixelwise_bwd(int N, int C, int HW, const float* S, long long s_sn, long long s_sc, long long s_sp, const float* T,
                      long long t_sn, long long t_sc, long long t_sp, float* dS, long long d_sn, long long d_sc, long long d_sp,
                      const float* grad_out, float inv_hw, cudaStream_t);
/* CriterionDSN.forward (utils/criterion.py:179-188): w0*CE(up(L0)) + w1*CE(up(L1)), bilinear align_corners to (H,W),
   ignore_index, mean over valid pixels; L1 may be NULL.  count receives the number of valid pixels. */
int skd_dsn_ce_fwd(int N, int C, int h, int w, int H, int W, const float* L0, long long a_sn, long long a_sc, long long a_sp,
                   const float* L1, long long b_sn, long long b_sc, long long b_sp, const long long* labels, int ignore_index,
                   float w0, float w1, float* loss, float* count, double* workspace, cudaStream_t);
long long skd_dsn_ce_bwd_workspace_floats(int N, int C, int w, int H, int heads);
int skd_dsn_ce_bwd(int N, int C, int h, int w, int H, int W, const float* L0, long long a_sn, long long a_sc, long long a_sp,
                   const float* L1, long long b_sn, long long b_sc, long long b_sp, const long long* labels, int ignore_index,
                   float w0, float w1, const float* grad_out, const float* count, float* d0, float* d1, float* workspace,
                   cudaStream_t);
/* training forward = loss + count + the backward's row phase in ONE pass over the upsampled pixels (one softmax per pixel and step
   instead of two); skd_dsn_ce_bwd_cols finishes the backward from `rows_ws` (skd_dsn_ce_bwd_workspace_floats floats) */
long long skd_dsn_ce_train_partials(int N, int H, int heads);       /* doubles */
int skd_dsn_ce_fwd_train(int N, int C, int h, int w, int H, int W, const float* logits0, long long a_sn, long long a_sc, long long a_sp,
                         const float* logits1, long long b_sn, long long b_sc, long long b_sp, const long long* labels, int ignore_index,
                         float w0, float w1, float* loss, float* count, double* partials, float* rows_ws, cudaStream_t);
int skd_dsn_ce_bwd_cols(int N, int C, int h, int w, int H, const float* rows_ws, long long a_sn, long long a_sc, long long a_sp,
                        long long b_sn, long long b_sc, long long b_sp, int heads, float w0, float w1, const float* grad_out,
                        const float* count, float* d0, float* d1, cudaStream_t);
/* Class-weighted forms (CrossEntropyLoss(weight=class_weight, ignore_index) per head): class_weight is a device array of C floats;
   loss = w0 * sum_i cw[y_i] nll0_i / sum_i cw[y_i] + w1 * sum_i cw[y_i] nll1_i / sum_i cw[y_i] over the pixels whose label is
   not ignore_index, and count receives sum_i cw[y_i].  The backward of the training forward is skd_dsn_ce_bwd_cols.
   A label outside [0, C) that is not ignore_index does not index the table: its weight is 0.
   If sum_i cw[y_i] = 0 (every label ignored, or every present class weighted 0) the loss is NaN and the gradient 0. */
int skd_dsn_ce_fwd_weighted(int N, int C, int h, int w, int H, int W, const float* L0, long long a_sn, long long a_sc, long long a_sp,
                            const float* L1, long long b_sn, long long b_sc, long long b_sp, const long long* labels, int ignore_index,
                            float w0, float w1, float* loss, float* count, double* workspace, const float* class_weight, cudaStream_t);
int skd_dsn_ce_fwd_train_weighted(int N, int C, int h, int w, int H, int W, const float* logits0, long long a_sn, long long a_sc,
                                  long long a_sp, const float* logits1, long long b_sn, long long b_sc, long long b_sp,
                                  const long long* labels, int ignore_index, float w0, float w1, float* loss, float* count,
                                  double* partials, float* rows_ws, const float* class_weight, cudaStream_t);
/* OhemCrossEntropy2d / CriterionOhemDSN (utils/criterion.py:11-90, 190-209), with no host round trip.
   skd_ohem_grid_sample replaces find_threshold's scipy zooms (criterion.py:20-35): for every point of the gh x gw grid (Python
   round(H / factor), round(W / factor)) it writes the zoomed probability of the zoomed label (+inf where that label is
   ignore_index) to pred[N*gh*gw], the zoomed label to grid_labels (may be NULL) and the number of valid points to *nvalid.
   The probabilities come from the low-resolution logits (align_corners upsample to (H, W), fp32 softmax). */
int skd_ohem_grid_sample(int N, int C, int h, int w, int H, int W, int gh, int gw, const float* logits, long long sn, long long sc,
                         long long sp, const long long* labels, int ignore_index, float* pred, long long* grid_labels, int* nvalid,
                         cudaStream_t);
/* criterion.py:36-47 (np.partition): threshold = 1 when min_kept >= *nvalid, else thresh raised to the (min_kept-1)-th smallest
   pred when that is larger and min_kept > 0 (min_kept = the reference's min_kept // factor^2).  Exact radix select on the device. */
long long skd_ohem_threshold_workspace_ints(void);
int skd_ohem_threshold(long long n, const float* pred, const int* nvalid, int min_kept, float thresh, float* threshold,
                       int* workspace, cudaStream_t);
/* criterion.py:65-90 + 203-209: w0 * CE over the valid pixels with p[label] <= *threshold (head 0) + w1 * CE over the valid
   pixels (head 1, logits1 may be NULL), each mean over its own count, fused with the backward's row phase like
   skd_dsn_ce_fwd_train.  counts[4]: kept, valid (head 1), and the two denominators skd_ohem_dsn_ce_bwd_cols reads. */
int skd_ohem_dsn_ce_fwd_train(int N, int C, int h, int w, int H, int W, const float* logits0, long long a_sn, long long a_sc,
                              long long a_sp, const float* logits1, long long b_sn, long long b_sc, long long b_sp,
                              const long long* labels, int ignore_index, float w0, float w1, const float* threshold, float* loss,
                              float* counts, double* partials, float* rows_ws, cudaStream_t);
int skd_ohem_dsn_ce_bwd_cols(int N, int C, int h, int w, int H, const float* rows_ws, long long a_sn, long long a_sc, long long a_sp,
                             long long b_sn, long long b_sc, long long b_sp, int heads, float w0, float w1, const float* grad_out,
                             const float* counts, float* d0, float* d1, cudaStream_t);
/* CriterionPairWiseforWholeFeatAfterPool.forward (utils/criterion.py:236-245) + sim_dis_compute (utils/utils.py:170-183):
   pool: ceil-mode max pool kernel=stride=(ph,pw) -> pooled[N][nodes][C], argmax (pixel index, may be NULL), rnorm[N][nodes] */
int skd_pairwise_pool(int N, int C, int H, int W, const float* F, long long sn, long long sc, long long sp, int ph, int pw,
                      float* pooled, int* argmax, float* rnorm, cudaStream_t);
long long skd_pairwise_gram_partials(int N, int nodes);
/* E[N][nodes][nodes] = A_T - A_S (may be NULL), loss = sum E^2 / nodes^2 / N */
int skd_pairwise_gram(int N, int nodes, int CS, int CT, const float* pooled_S, const float* pooled_T, const float* rnorm_S,
                      const float* rnorm_T, float* E, float* loss, double* workspace, cudaStream_t);
/* dpooled_S, then scattered through argmax into the pre-zeroed feature gradient dF */
int skd_pairwise_bwd(int N, int nodes, int CS, const float* E, const float* pooled_S, const float* rnorm_S, const int* argmax,
                     const float* grad_out, float* dpooled, float* dF, long long sn, long long sc, long long sp, cudaStream_t);

/* dF[argmax] = dpooled on a pre-zeroed feature gradient (second half of skd_pairwise_bwd) */
int skd_pairwise_scatter(int N, int nodes, int CS, const float* dpooled, const int* argmax, float* dF, long long sn, long long sc,
                         long long sp, cudaStream_t);
/* wgmma path for large node counts (pool_scale -> 1/65: 8 385 nodes): E = [fT^|fS^] [fT^|-fS^]^T as one K-major TF32 GEMM per image with
   the L2 reduction fused into the epilogue; E ([N][nodes][ldE], ldE % 4 == 0) may be NULL when no backward follows.  acc: 1 double. */
long long skd_pairwise_affinity_sm100_workspace_floats(int N, int nodes, int CS, int CT);
int skd_pairwise_affinity_sm100(int N, int nodes, int CS, int CT, const float* pooled_S, const float* pooled_T, const float* rnorm_S,
                                const float* rnorm_T, float* E, int ldE, float* loss, float* workspace, double* acc, cudaStream_t);
long long skd_pairwise_affinity_bwd_sm100_workspace_floats(int N, int nodes, int CS, int ldE);
int skd_pairwise_affinity_bwd_sm100(int N, int nodes, int CS, const float* E, int ldE, const float* pooled_S, const float* rnorm_S,
                                    const float* grad_out, float* dpooled, float* workspace, cudaStream_t);
/* the wgmma conv kernel as a plain NT GEMM: D[M][Ncols] = A[M][K] B[Ncols][K]^T (D may be NULL), sumsq += sum D^2 (may be NULL) */
int skd_gemm_nt_sm100(int M, int Ncols, int K, const float* A, int lda, const float* B, float* D, int ldd, double* sumsq, cudaStream_t);

/* ---- D. convolutions (every nn.Conv2d of networks/pspnet_combine.py; cuDNN in the reference) ---- */
/* wgmma implicit GEMM: y = act((conv(x,w))*scale + shift + residual); w is [Cout][KH][KW][Cin]; Cin % 4 == 0 */
int skd_conv2d_fwd_sm100(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil, const float* x,
                         int ldx, const float* w, float* y, int ldy, const float* scale, const float* shift,
                         const float* residual, int ldr, int act, float slope, int round_tf32, cudaStream_t);
/* split-precision forward (x = x_hi + x_lo, w = w_hi + w_lo, all four TF32-exact): three accumulation passes in one launch, fp32-grade
   result; skd_split_tf32 produces the parts (hi = rn_tf32(v), lo = rn_tf32(v - hi), round-to-nearest-even like the TMA conversion) */
int skd_conv2d_fwd_sm100_3xtf32(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil, const float* x_hi,
                                const float* x_lo, int ldx, const float* w_hi, const float* w_lo, float* y, int ldy, const float* scale,
                                const float* shift, int act, float slope, cudaStream_t);
int skd_split_tf32(long long n, const float* src, float* hi, float* lo, cudaStream_t);
/* general form of the wgmma forward (discriminator path): optional split-precision operands (x_lo / w_lo both NULL -> plain TF32),
   optional output extent (out_h / out_w > 0: positions past the natural size read zero-filled input), fused scale / shift / residual / act */
int skd_conv2d_fwd_sm100_ex(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil, const float* x,
                            const float* x_lo, int ldx, const float* w, const float* w_lo, float* y, int ldy, int out_h, int out_w,
                            const float* scale, const float* shift, const float* residual, int ldr, int act, float slope, cudaStream_t);
/* the same convolution with split-K when it has too few output tiles to fill the GPU (the discriminator's 4x4/s2 convolutions on
   4x8 .. 16x32 maps: K up to 4096 on 2..8 tiles): work units are (tile, K range), raw partial tiles go to `workspace`
   (skd_conv2d_fwd_sm100_splitk_workspace_floats; 0 = no split, then identical to _ex) and one pass adds them in fixed order and
   applies scale / shift / residual / act */
long long skd_conv2d_fwd_sm100_splitk_workspace_floats(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil,
                                                       int out_h, int out_w);
int skd_conv2d_fwd_sm100_splitk(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil, const float* x,
                                const float* x_lo, int ldx, const float* w, const float* w_lo, float* y, int ldy, int out_h, int out_w,
                                const float* scale, const float* shift, const float* residual, int ldr, int act, float slope,
                                float* workspace, long long workspace_floats, cudaStream_t);

/* same kernel, output written through explicit element strides y[n*y_img + oy*y_row + ox*y_pix + c] (every-other-pixel sub-grids:
   the data gradient of a stride-2 convolution is 4 stride-1 convolutions of dy, one per input-pixel parity class) */
int skd_conv2d_fwd_sm100_strided(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil, const float* x,
                                 int ldx, const float* w, float* y, long long y_pix, long long y_row, long long y_img, int out_h, int out_w,
                                 int round_tf32, cudaStream_t);   /* out_h/out_w > 0 override the output extent (far-end zero padding) */
/* the strided-output form with split-precision operands (x_lo, w_lo required; skd_split_tf32 makes them) */
int skd_conv2d_fwd_sm100_strided_3xtf32(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil,
                                        const float* x_hi, const float* x_lo, int ldx, const float* w_hi, const float* w_lo, float* y,
                                        long long y_pix, long long y_row, long long y_img, cudaStream_t);
/* wgmma weight gradient: dw[Cout][KH][KW][Cin] = sum_pixels dy[p][co] * x[p+tap][ci]; workspace from the size query */
long long skd_conv2d_wgrad_sm100_workspace_floats(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil);
int skd_conv2d_wgrad_sm100(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil, const float* x,
                           int ldx, const float* dy, int ldy, float* dw, float* workspace, cudaStream_t);
/* SIMT direct forms (3-channel stem, strided dgrad, cross-checks) */
int skd_conv2d_fwd_direct(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil, const float* x,
                          int ldx, const float* w, float* y, int ldy, const float* scale, const float* shift, int act,
                          float slope, cudaStream_t);
int skd_conv2d_dgrad_direct(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil,
                            const float* dy, int ldy, const float* w, float* dx, int ldx, cudaStream_t);
int skd_conv2d_wgrad_direct(int N, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dil, const float* x,
                            int ldx, const float* dy, int ldy, float* dw, cudaStream_t);
int skd_colsum(long long P, int C, const float* dy, int ldy, float* db, cudaStream_t);
int skd_colsum_acc(long long P, int C, const float* dy, int ldy, float* db, cudaStream_t);   /* db += (bias gradients accumulated over passes) */
/* explicit im2col for tiny-Cin convolutions (3-channel stem): col[N*OH*OW][Kp], k = (kh*KW+kw)*Cin+ci, zero padded to Kp */
int skd_im2col_small(int N, int H, int W, int Cin, int KH, int KW, int stride, int pad, int dil, const float* x, int ldx, float* col,
                     int Kp, cudaStream_t);
/* wt[Cin][KH][KW][Cout] = w[Cout][KH-1-kh][KW-1-kw][Cin] (dgrad of a stride-1 conv == forward conv with wt, pad' = d*(K-1)-pad) */
int skd_weight_flip_transpose(int Cout, int Cin, int KH, int KW, const float* w, float* wt, int round_tf32, cudaStream_t);
int skd_round_tf32(long long n, const float* src, float* dst, cudaStream_t);
void skd_set_tf32_tma_type(int use_tfloat32_type);
void skd_set_wgrad_linear(int on);     /* 1 (default): wgrad K-blocks are 32 consecutive pixels (im2col TMA); 0: 4x8 pixel rectangles */
void skd_set_conv_tile_order(int mode); /* 0 (default) front-to-back, 1 back-to-front, 2 alternate per launch (a consumer starts on
                                          the tail its producer left in L2) */
void skd_set_conv_k_order(int mode);   /* K loop of k>1 convolutions: 0 (default) by working set, 1 taps outermost, 2 channel chunks outermost */
void skd_set_conv_im2col(int on);      /* 1 (default): TMA im2col-mode M tiles for k>1 / strided convs; 0: rectangular tiled-mode tiles */
void skd_set_conv_tile_m(int mode);    /* wgmma conv M tile: 0 (default) 256 rows for long-K launches with Cout > 128 that fill waves as
                                          well as 128 rows do; 1 always 128; 2 256 wherever that path can run (flat / im2col, Cout > 64,
                                          TF32, no split-K, register epilogue, an output tensor) */
/* two frozen bottleneck 1x1 convolutions in one launch, over P pixel rows:
     y3 = relu(conv1x1(x3, w3) * scale3 + shift3 + residual)   w3 [Cout3][Cin3], y3 may be the residual itself
     y1 = relu(conv1x1(y3, w1) * scale1 + shift1)              w1 [Cout1][Cout3]
   both bit for bit what two skd_conv2d_fwd_sm100 launches compute.  Cout3 % 64 == 0, Cout1 in {64, 128, 256} */
int skd_conv1x1_chain_sm100(int P, int Cin3, int Cout3, int Cout1, const float* x3, int ldx3, const float* w3, const float* scale3,
                            const float* shift3, const float* residual, int ldr, float* y3, int ldy3, const float* w1,
                            const float* scale1, const float* shift1, float* y1, int ldy1, cudaStream_t);
/* what the host-side dispatch chose for the last wgmma forward launch (any skd_conv2d_fwd_sm100* entry or skd_gemm_nt_sm100):
   out[7] = {M tile mode (0 flat, 1 im2col, 2 rect), tile rows (128 or 256), BLOCK_N, K splits, TMA epilogue, channel chunks outermost
   (kc_outer), tile order reversed}.  Reports only; launches are unchanged. */
void skd_conv_fwd_last_plan(int* out);
/* the same for the last skd_conv2d_wgrad_sm100: out[3] = {BLOCK_N, linear 32-pixel K blocks, K splits} */
void skd_conv_wgrad_last_plan(int* out);
/* weight-gradient work units run two to a CTA: for Cout >= 256 (BLOCK_N 128) two adjacent full 128-row Cout tiles with the same
   split, tap and Cin tile, sharing one X transposition; for Cout <= 64 (BLOCK_N <= 64) any two units, one per consumer warpgroup.
   Every dW bit is the same in all modes.  0: never; 1 (default): the number of pairs that minimises the predicted makespan over the
   persistent CTAs; 2: every such pair */
void skd_set_wgrad_pairing(int mode);
/* the number of pair units of the last skd_conv2d_wgrad_sm100: out[0] */
void skd_conv_wgrad_last_pairs(int* out);
void skd_set_conv_chain(int mode);     /* frozen bottlenecks: 0 (default) chain conv3 with the next block's conv1 where the shapes allow; 1 never */
int skd_conv_chain_mode(void);

/* ---- E. pooling / resampling / optimiser ---- */
int skd_pool_out_size_ceil(int in, int k, int s, int p);
int skd_maxpool3x3s2_fwd(int N, int H, int W, int C, const float* x, float* y, unsigned char* argmax, cudaStream_t);
int skd_maxpool3x3s2_bwd(int N, int H, int W, int C, const float* dy, const unsigned char* argmax, float* dx, cudaStream_t);
long long skd_psp_pool_workspace_floats(int N, int H, int C, int levels, const int* sizes);
int skd_psp_pool_fwd(int N, int H, int W, int C, const float* x, int x_pitch, int levels, const int* sizes, float* pooled,
                     float* workspace, cudaStream_t);
int skd_psp_pool_bwd(int N, int H, int W, int C, const float* dpooled, int levels, const int* sizes, float* dx, cudaStream_t);
int skd_psp_upsample_fwd(int N, int H, int W, int C, int s, const float* src, int nbins_total, int first_bin, float* out,
                         int out_pitch, int chan_off, cudaStream_t);
long long skd_psp_upsample_bwd_workspace_floats(int N, int H, int C, int s);
int skd_psp_upsample_bwd(int N, int H, int W, int C, int s, const float* dout, int dout_pitch, int chan_off, float* dsrc,
                         int nbins_total, int first_bin, float* workspace, cudaStream_t);
/* dst[r][dst_off + c] = src[r][src_off + c], c < C; float4 accesses when every count / offset / pitch is a multiple of 4, else scalar */
int skd_slice_copy(long long rows, int C, const float* src, int src_pitch, int src_off, float* dst, int dst_pitch, int dst_off, cudaStream_t);
/* G_solver.step (networks/kd_model.py:74,171): v = mu*v + (g*grad_scale + wd*p); p -= lr*v; lr read from device memory */
int skd_sgd_step(long long n, float* param, const float* grad, float* momentum_buf, const float* lr, float momentum,
                 float weight_decay, int first_step, float grad_scale, cudaStream_t);
/* The same update fused with the data-parallel gradient exchange over NVSwitch multicast (replaces Reduce.apply + the per-GPU
   optimizer of utils/parallel.py:54-63,155 + kd_model.py:171): the calling rank owns elements [lo, hi) of the flat buffers (multiples of
   4): g = multimem.ld_reduce.add over every rank's gradient (summed inside the switch), momentum-SGD with grad_scale = 1/world, new
   parameters multimem.st-broadcast to every rank.  param_mc / grad_mc: MULTICAST addresses of the symmetric parameter / gradient
   buffers (element 0); param_local: this rank's own copy; momentum_buf: local, only [lo, hi) is used.  The caller brackets the call
   with two cross-rank barriers (gradients complete before, parameters complete after). */
int skd_sgd_step_nvls(long long lo, long long hi, float* param_mc, const float* grad_mc, const float* param_local, float* momentum_buf,
                      const float* lr, float momentum, float weight_decay, float grad_scale, cudaStream_t);


/* ---- F. SAGAN discriminator of the holistic loss (networks/sagan_models.py:9-41,105-168, networks/spectral.py:23-35) and the
        adversarial criteria (utils/criterion.py:92-166).  Activations are NHWC rows [positions][channels].  "+=" outputs honour
        `accumulate` (the reference's native convention: caller-zeroed dweight/dbias, libs/src/bn.cu:214-230). ---- */
/* SpectralNorm._update_u_v (spectral.py:23-35), ONE power iteration: v <- normalize(W^T u), u <- normalize(W v), sigma = u.(W v).
   w_bar is [Cout][taps][Cin] (OHWI storage of the (Cout,Cin,KH,KW) parameter); v keeps the reference's flattening (ci*taps + tap).
   u, v advance in place; u_save / v_save (may be NULL) receive copies for the backward; inv_sigma_vec[vec_len] is filled with
   1/sigma (per-channel epilogue scale of the convolution: conv(x, w_bar/sigma) = conv(x, w_bar)/sigma).  One cluster of 8 CTAs. */
int skd_sn_power_iter(int Cout, int taps, int Cin, const float* w_bar, float* u, float* v, float* u_save, float* v_save, float* sigma,
                      float* inv_sigma_vec, int vec_len, cudaStream_t);
/* The same iteration for several layers in one call (the discriminator's four spectral-norm layers per forward), each phase a
   grid over all layers and the whole GPU (the single-layer entry keeps a layer on one 8-CTA cluster).  Deterministic (fixed-order partial sums, no atomics).  `layers` is a HOST array. */
typedef struct skd_sn_layer {
  int Cout, taps, Cin, vec_len;
  const float* w_bar; float* u; float* v; float* u_save; float* v_save; float* sigma; float* inv_sigma_vec;
} skd_sn_layer;
long long skd_sn_power_iter_batched_workspace_floats(int n_layers, const skd_sn_layer* layers);
int skd_sn_power_iter_batched(int n_layers, const skd_sn_layer* layers, float* workspace, cudaStream_t);
/* d_w (+)= d_wn/sigma - <d_wn, w_bar>/sigma^2 * u v^T : gradient through w_bar/sigma with u, v constant (spectral.py:34-35).
   d_wn is [Cout][taps][Cin_p] (channel-padded wgrad output), d_w / w_bar [Cout][taps][Cin]. */
long long skd_sn_weight_grad_workspace_doubles(void);      /* zero-initialised once by the caller; self-resetting */
int skd_sn_weight_grad(int Cout, int taps, int Cin, int Cin_p, const float* d_wn, const float* w_bar, const float* u, const float* v,
                       const float* sigma, float* d_w, int accumulate, double* workspace, cudaStream_t);
/* w [rows][Cin] -> channel-padded copy [rows][Cin_p] (+ its TF32 "lo" part, may be NULL) */
int skd_disc_weight_prep(long long rows, int Cin, int Cin_p, const float* w, float* w_pad, float* w_lo, cudaStream_t);
/* data-gradient weights of a 4x4 / stride 2 / pad 1 convolution as ONE 3x3 stride-1 convolution of dy whose 4*Cin_p output channels
   are the four input-pixel parity classes: wd[(py*2+px)*Cin_p+ci][3][3][Cout] */
int skd_disc_dgrad_weight_prep(int Cout, int Cin, int Cin_p, const float* w, float* wd, float* wd_lo, cudaStream_t);
/* un-shuffle that convolution's output d2s [B][ceil(H/2)][ceil(W/2)][4*Cp] into dx [B][H][W][Cq] (channels >= C zero), multiplied by
   the LeakyReLU mask recovered from ref [ref_batch][H][W][C] (post-activation output of the layer below; NULL: no mask) */
int skd_disc_dgrad_unshuffle(int B, int H, int W, int C, int Cp, const float* d2s, const float* ref, int ref_batch, float slope, float* out,
                             int Cq, float* out_lo, cudaStream_t);
/* out = in * leaky'(ref[i % period]) (+ TF32 lo part) */
int skd_disc_mask_mul(long long n, long long period, const float* ref, const float* in, float* out, float* out_lo, float slope, cudaStream_t);
/* nn.BatchNorm2d(C <= 32) with batch statistics (sagan_models.py:147): x addressed by (sn, sc, sp) strides */
long long skd_bn2d_workspace_doubles(void);                /* zero-initialised once by the caller; self-resetting */
int skd_bn2d_stats(int N, int C, int HW, const float* x, long long sn, long long sc, long long sp, float eps, float momentum,
                   float* running_mean, float* running_var, long long* num_batches_tracked, float* mean, float* rstd, double* workspace,
                   cudaStream_t);
int skd_bn2d_apply(int N, int C, int HW, const float* x, long long sn, long long sc, long long sp, const float* mean, const float* rstd,
                   const float* weight, const float* bias, float* out, float* out_lo, int Cp, cudaStream_t);
/* sums[0..31] = sum a, sums[32..63] = sum a*xhat, sums[64..95] = sum a*b (b may be NULL); a, b dense [N*HW][ld] */
int skd_bn2d_reduce(int N, int C, int HW, const float* x, long long sn, long long sc, long long sp, const float* mean, const float* rstd,
                    const float* a, const float* b, int ld, float* sums, double* workspace, cudaStream_t);
/* out = gamma rstd (a - mean(a) - xhat mean(a xhat)): BN's input gradient and (symmetric Jacobian) its forward-mode tangent */
int skd_bn2d_jacobian(int N, int C, int HW, const float* x, long long sn, long long sc, long long sp, const float* mean, const float* rstd,
                      const float* weight, const float* a, int ld, const float* sums, float* out, long long on, long long oc, long long op,
                      int Cq, float* out_lo, cudaStream_t);
/* dgamma (+)= sum gh xhat [+ sum gth t0], dbeta (+)= sum gh; sums_t / sums_v NULL for the first-order backward */
int skd_bn2d_param_grad(int C, long long P, const float* rstd, const float* sums_g, const float* sums_t, const float* sums_v, float* dgamma,
                        float* dbeta, int accumulate, cudaStream_t);
/* preprocess_GAN_mode 2 / 3 (sagan_models.py:149-152), no parameters: mode 2 out = tanhf(x); mode 3 out = 2 * (x / 255 - 0.5) in the
   reference's fp32 operation order (IEEE division).  Same addressing and output as skd_bn2d_apply: x by (sn, sc, sp) strides, out
   [N*HW][Cp] with channels >= C zero, out_lo (may be NULL) its TF32 lo part */
int skd_disc_pointwise_prep(int mode, int N, int C, int HW, const float* x, long long sn, long long sc, long long sp, float* out, float* out_lo,
                            int Cp, cudaStream_t);
/* out = J a with the diagonal Jacobian of that map at x: mode 2 a * (1 - tanhf(x)^2), mode 3 (a * 2) / 255.  a dense [N*HW][ld]; out by
   (on, oc, op) strides over Cq channels (channels >= C zero), out_lo may be NULL -- as skd_bn2d_jacobian */
int skd_disc_pointwise_prep_jacobian(int mode, int N, int C, int HW, const float* x, long long sn, long long sc, long long sp, const float* a,
                                     int ld, float* out, long long on, long long oc, long long op, int Cq, float* out_lo, cudaStream_t);
/* Self_Attn core (sagan_models.py:31-40): A = softmax(Q K^T) (no 1/sqrt(d)), O = A V, y = gamma O + x.
   qkv [B*n][ldq] = [q(d) | k(d) | v(C)] (the three 1x1 convolutions as one GEMM), x / o / y [B*n][C], attn [B][n][n]; n <= 1024, d <= 64.
   n <= 128 runs whole n x n tiles per CTA; n > 128 runs stripes of query rows with keys / values streamed in tiles. */
void skd_set_attn_tensor_cores(int on);   /* 1 (default): the attention products on mma.sync TF32 in split precision; 0: SIMT fp32 (cross-check) */
void skd_set_attn_tiled(int force);       /* 1: the row-stripe kernels for every n (cross-checks and timing at n <= 128); 0 (default): only for n > 128 */
int skd_attn_fwd(int B, int n, int C, int d, const float* qkv, int ldq, const float* x, const float* gamma, float* attn, float* o, float* y,
                 float* y_lo, cudaStream_t);
/* forward-mode tangent along (tqkv, tx): dattn = Adot, to = Odot, ty = gamma Odot + tx */
int skd_attn_tangent_fwd(int B, int n, int C, int d, const float* qkv, const float* tqkv, int ldq, const float* attn, const float* tx,
                         const float* gamma, float* dattn, float* to, float* ty, float* ty_lo, cudaStream_t);
/* backward: gy = adjoint of y (NULL: zero).  gty != NULL selects the JOINT backward of (y, ydot) used by the WGAN-GP penalty
   (oracle/gp_dual.py attn_joint_backward); gqkv / gtqkv receive the adjoints of qkv / tqkv, ggamma (+)= dgamma */
long long skd_attn_bwd_workspace_floats(int B, int n, int C);
int skd_attn_bwd(int B, int n, int C, int d, const float* qkv, int ldq, const float* attn, const float* o, const float* gamma,
                 const float* gy, const float* tqkv, const float* dattn, const float* to, const float* gty, float* gqkv, float* gtqkv,
                 float* ggamma, int accumulate, float* workspace, cudaStream_t);
/* the "last" convolution (sagan_models.py:140: Conv2d(C, 1, 4), no padding): w [KH][KW][C] with row pitch w_row floats */
int skd_disc_last_fwd(int B, int H, int W, int C, int KH, int KW, const float* x, const float* w, int w_row, const float* bias, float* out,
                      cudaStream_t);
int skd_disc_last_dgrad(int B, int H, int W, int C, int KH, int KW, const float* gout, const float* w, int w_row, float* gx, float* gx_lo,
                        cudaStream_t);                       /* gout NULL: all ones */
int skd_disc_last_wgrad(int B, int H, int W, int C, int KH, int KW, const float* x, const float* gout, float* gw, int w_row, float* gbias,
                        int accumulate, cudaStream_t);
/* CriterionAdv / CriterionAdvForG (utils/criterion.py:129-166): type 0 wgan-gp, 1 hinge, 2 generator; also d loss / d out */
int skd_adv_loss(int n, const float* real, const float* fake, int type, float* loss, float* g_real, float* g_fake, cudaStream_t);
/* CriterionAdditionalGP (utils/criterion.py:98-120): norms[b] = |g_b|, loss = lambda * mean (|g_b| - 1)^2 */
int skd_gp_norms(int B, long long len, const float* g, float lambda_gp, float* norms, float* loss, cudaStream_t);
/* v_b = upstream * 2 lambda / B * (|g_b| - 1) / |g_b| * g_b  (upstream: device scalar or NULL) */
int skd_gp_direction(int B, long long len, const float* g, const float* norms, float lambda_gp, const float* upstream, float* v, cudaStream_t);

/* ---- G. evaluation (networks/evaluate.py:75-206): full [H][W][C] += bilinear(align_corners) up-sampling of one tile's class scores
        (C, h, w; strides sc, sp) to tile_h x tile_w, valid part only, placed at (y1, x1); then arg-max + confusion matrix (+=),
        labels == ignore_index skipped; pred (uint8 [H][W]) optional ---- */
int skd_eval_upsample_accumulate(int C, int h, int w, const float* logits, long long sc, long long sp, int tile_h, int tile_w, int valid_h,
                                 int valid_w, float* full, int W, int y1, int x1, cudaStream_t);
int skd_eval_argmax_confusion(int H, int W, int C, const float* full, const long long* gt, long long gt_row, int valid_h, int valid_w,
                              int ignore_index, long long* confusion, unsigned char* pred, cudaStream_t);
/* predict_multiscale (networks/evaluate.py:115-134), whole-image tiles placed at (0, 0):
   skd_eval_zoom_image replaces scipy.ndimage.zoom(image, (1, 1, s, s), order=1, prefilter=False) (:127) bit for bit, including mode
   'constant''s zero line where a rounded source coordinate passes the last row / column; image is float32 (1, 3, H, W) contiguous,
   out_h / out_w = round(H * s), round(W * s); out is the 4-channel NHWC network input [1 + flip][out_h][out_w][4] (channel 3 zero),
   item 1 the mirror image[:, :, :, ::-1] (:130) when flip != 0.
   skd_eval_upsample_accumulate_ms: full += weight * up(L0) (paired = 0) or full += weight * 0.5f * (up(L0)[y][x] + up(L1)[y][tile_w-1-x])
   (paired = 1, :131), L1 = batch item 1 of the logits (sn floats after L0); weight = 1 / len(scales) (:133). */
int skd_eval_zoom_image(int H, int W, const float* image, int out_h, int out_w, int flip, float* out, cudaStream_t);
int skd_eval_upsample_accumulate_ms(int C, int h, int w, const float* logits, long long sn, long long sc, long long sp, int tile_h,
                                    int tile_w, int valid_h, int valid_w, float* full, int W, float weight, int paired, cudaStream_t);
/* arg-max of the whole score buffer into pred [pred_h][pred_w] (evaluate.py:187-191, before the `size` crop of :194), through the
   256-entry device table lut when given (train id -> Cityscapes label id for type='test', :188); confusion += over the valid region
   only, as skd_eval_argmax_confusion.  gt / pred may be NULL. */
int skd_eval_argmax_confusion_lut(int H, int W, int C, const float* full, const long long* gt, long long gt_row, int valid_h, int valid_w,
                                  int ignore_index, long long* confusion, unsigned char* pred, int pred_h, int pred_w,
                                  const unsigned char* lut, cudaStream_t);
/* HOST tables, 256 entries each: label id -> train id (dataset/datasets.py:146-151, the table skd_cs_augment_batch applies) and its
   reverse, train id -> label id, as id2trainId(..., reverse=True) builds it (evaluate.py:30-38, 188) */
int skd_cityscapes_id_tables(unsigned char* to_train, unsigned char* to_label);

/* ---- Cityscapes training augmentation on the device (csrc/augment.cu) --------------------------------------------------------------
   Replaces the per-sample CPU work of `CSDataSet.__getitem__` after cv2.imread (reference dataset/datasets.py:175-206):
   id -> trainId table (:161-169), `generate_scale_label` = cv2.resize INTER_LINEAR / INTER_NEAREST by f_scale (:155-159), float32 mean
   subtraction (:180-181), padding with 0 / ignore_label (:183-193), crop (:196-200), HWC -> CHW (:202), mirror (:203-206) -- bit-exact
   with opencv's uint8 fixed-point resize.  The host draws the random numbers in the reference's order
   (structure_knowledge_distillation_b200/dataset/datasets.py::draw_augmentation) and passes them here.  `samples` and `mean_bgr` are
   HOST arrays; image / label pointers inside are DEVICE pointers to the raw decoded files (uint8 H x W x 3 BGR interleaved, uint8 H x W).
   images: device [n][3][crop_h][crop_w] float32; labels: device [n][crop_h][crop_w], float32 (what __getitem__ returns) or int64
   (what `NetModel.set_input` turns them into, kd_model.py:105). */
typedef struct skd_cs_sample {
  const unsigned char* image; const unsigned char* label;
  int src_h, src_w;
  double f_scale;               /* 0.7 + randint(0, 14) / 10.0 (VOC: 0.5 + randint(0, 11) / 10.0); <= 0: no resize (scale=False) */
  int scaled_h, scaled_w;       /* cvRound(src * f_scale) (ignored without resize) */
  int h_off, w_off;             /* crop origin inside the padded, scaled image */
  int flip;                     /* -1: mirror, +1: keep */
} skd_cs_sample;
int skd_cs_augment_batch(int n, const skd_cs_sample* samples, int crop_h, int crop_w, const float* mean_bgr, int ignore_label,
                         float* images, void* labels, int labels_int64, cudaStream_t);
/* The same kernel for any data set (`VOCDataSet.__getitem__`, dataset/datasets.py:45-81, and the above): label_table is a HOST
   uint8[256] applied to every raw label (NULL: labels pass through, as VOC's class ids 0..20 and 255 do); mean_bgr is HOST, 3
   doubles, and the image value is (float)((double)x - mean_bgr[c]), i.e. numpy's `float32 image -= mean` for a float32 mean (pass
   it rounded to float32) and for a tuple of Python numbers (pass it as is).  skd_cs_augment_batch is this call with the Cityscapes
   table (ids >= 34 pass through) and its float32 mean. */
int skd_augment_batch(int n, const skd_cs_sample* samples, int crop_h, int crop_w, const double* mean_bgr,
                      const unsigned char* label_table, int ignore_label, float* images, void* labels, int labels_int64, cudaStream_t);
/* `CSDataTestSet.__getitem__` after cv2.imread (dataset/datasets.py:234-250): image (device, uint8 H x W x 3 BGR) -> out (device,
   float32 [3][out_h][out_w]), value (float)((double)x - mean_bgr[c]) -- the reference subtracts a tuple of Python floats, i.e. in
   double -- and zero padding on the bottom / right; out_h = max(H, crop_h), out_w = max(W, crop_w) (no crop).  mean_bgr: HOST, 3. */
int skd_cs_test_preprocess(int H, int W, const unsigned char* image, const double* mean_bgr, int out_h, int out_w, float* out, cudaStream_t);

/* ---- H. ESPNet-C student (networks/espnet.py, csrc/espnet.cu).  NHWC rows [P = N*H*W][...] with explicit row pitches in floats;
        a channel slice of a concat buffer is passed as a pointer to its first channel.  Plain affine BatchNorm2d (gamma = w, not
        ABN's |w| + eps) followed by a per-channel PReLU (y = z if z > 0 else alpha * z).  Fixed-order reductions throughout. ---- */
long long skd_bnprelu_workspace_doubles(long long P, int C);   /* workspace of the statistics / backward reductions below */
/* replaces nn.BatchNorm2d's training-mode statistics: mean, biased var; running_mean / running_var (may be NULL) updated with momentum
   and the unbiased variance n / (n - 1); *num_batches_tracked += 1 (may be NULL) */
int skd_bnprelu_stats(long long P, int C, const float* x, int ldx, float momentum, float* running_mean, float* running_var,
                      long long* num_batches_tracked, float* mean, float* var, double* workspace, cudaStream_t);
/* replaces ESPNet's torch.cat([d1, a1, a2, a3, a4], 1) (+ input) with a1 = d2, a2 = a1 + d4, a3 = a2 + d8, a4 = a3 + d16: writes the
   combine [P][n1 + 4n] to out and, when mean != NULL, the BatchNorm statistics of it in the same pass (as skd_bnprelu_stats).
   d1 has pitch ld1, d2..d16 pitch ldn, residual (may be NULL) pitch ldr */
int skd_esp_combine(long long P, int n1, int n, const float* d1, int ld1, const float* d2, const float* d4, const float* d8,
                    const float* d16, int ldn, const float* residual, int ldr, float* out, int ldo, float momentum,
                    float* running_mean, float* running_var, long long* num_batches_tracked, float* mean, float* var,
                    double* workspace, cudaStream_t);
/* alpha == NULL in the apply, backward reduce and dx passes below is plain BatchNorm2d without the PReLU (the full ESPNet's `br`):
   slope 1, no dalpha.  Non-NULL alpha computes exactly what it did before this mode existed. */
/* replaces BatchNorm2d + PReLU forward: out = prelu((x - mean) * w * rsqrt(var + eps) + b) for C channels, zeros in channels
   C .. out_channels - 1 (the channel padding the next convolution reads).  Eval mode passes the running statistics. */
int skd_bnprelu_apply(long long P, int C, const float* x, int ldx, const float* mean, const float* var, const float* weight,
                      const float* bias, const float* alpha, float eps, float* out, int ldo, int out_channels, cudaStream_t);
/* backward reduce pass: dweight = sum dz * xhat, dbias = sum dz, dalpha = sum_{z <= 0} z * dout (each may be NULL), dz = dout * prelu'(z);
   coef[2C] = (mean dz, mean dz * xhat) for the dx pass */
int skd_bnprelu_bwd_reduce(long long P, int C, const float* x, int ldx, const float* dout, int ldd, const float* mean, const float* var,
                           const float* weight, const float* bias, const float* alpha, float eps, float* dweight, float* dbias,
                           float* dalpha, float* coef, double* workspace, cudaStream_t);
/* dx pass: dx = w * rsqrt(var + eps) * (dz - coef[c] - xhat * coef[C + c]) (training) or w * rsqrt(var + eps) * dz (running
   statistics); channels C .. dx_channels - 1 are written as zeros */
int skd_bnprelu_bwd_dx(long long P, int C, const float* x, int ldx, const float* dout, int ldd, const float* mean, const float* var,
                       const float* weight, const float* bias, const float* alpha, float eps, int training, const float* coef, float* dx,
                       int lddx, int dx_channels, cudaStream_t);
/* the same dx pass over an ESP combine (x = the combine, C = n1 + 4n), written as the branch gradients: dd1 = g[0:n1],
   dd16 = g4, dd8 = g3 + g4, dd4 = g2 + g3 + g4, dd2 = g1 + ... + g4 (suffix sums of the HFF slices g1..g4), pad channels up to the
   pitches zero; dres (may be NULL) = g, the gradient of the residual input */
int skd_esp_bwd_dx(long long P, int n1, int n, const float* x, int ldx, const float* dout, int ldd, const float* mean, const float* var,
                   const float* weight, const float* bias, const float* alpha, float eps, int training, const float* coef, float* dd1,
                   int ld1, float* dd2, float* dd4, float* dd8, float* dd16, int ldn, float* dres, int ldr, cudaStream_t);
/* replaces ESPNet's InputProjectionA step nn.AvgPool2d(3, stride=2, padding=1) (count_include_pad): src [N][H][W] pitch lds, C
   channels -> dst [N][(H+1)/2][(W+1)/2] pitch ldd; forward only (the image needs no gradient) */
int skd_avgpool3x3s2(int N, int H, int W, int C, const float* src, int lds, float* dst, int ldd, cudaStream_t);
/* replaces F.interpolate(t, (H, W), mode='bilinear', align_corners=True) of the teacher's logits / feature (NetModel puts them on
   the student's grid): src (N, C, h, w) with element strides (sn, sc, sp) -> out dense NHWC [N][H][W][C]; forward only */
int skd_resample_bilinear_nhwc(int N, int C, int h, int w, const float* src, long long sn, long long sc, long long sp, int H, int W,
                               float* out, cudaStream_t);
/* adjoint of skd_resample_bilinear_nhwc: dsrc (N, C, h, w; NHWC, pixel pitch lds) = the transpose of the resize applied to dout
   (dense NHWC [N][H][W][C]).  A gather in fixed order (no atomics): two calls give bit-identical results.  The full ESPNet's
   discriminator input is its logits resized onto the teacher's grid; this is the gradient of that resize. */
int skd_resample_bilinear_adjoint_nhwc(int N, int C, int h, int w, const float* dout, int H, int W, float* dsrc, int lds, cudaStream_t);

/* ---- I. MobileNetV2 student (networks/mobilenet.py, csrc/mobilenet.cu).  fp32 NHWC, C a multiple of 4, rows 16-byte aligned.
        Fixed-order reductions (double partials, no atomics): two runs give bit-identical results. ---- */
/* workspace of the reductions below over P rows (the depthwise forward statistics and weight gradient: P = N * OH * OW) of C channels */
long long skd_mbv2_workspace_doubles(long long P, int C);
/* replaces nn.Conv2d(C, C, 3, stride, padding=dilation, dilation, groups=C, bias=False) forward: x dense [N][H][W][C], weight the
   (C, 1, 3, 3) parameter, y dense [N][OH][OW][C] with OH = (H - 1) / stride + 1.  stride 1 or 2.  When mean != NULL, the following
   BatchNorm2d's training statistics of y are formed in the same pass (as skd_bnprelu_stats: running statistics and counter may be NULL) */
int skd_dwconv3x3_fwd(int N, int H, int W, int C, int stride, int dilation, const float* x, const float* weight, float* y, float momentum,
                      float* running_mean, float* running_var, long long* num_batches_tracked, float* mean, float* var, double* workspace,
                      cudaStream_t);
/* its data gradient dx [N][H][W][C] from dy [N][OH][OW][C]: a gather, one thread per input element group, no atomics */
int skd_dwconv3x3_dgrad(int N, int H, int W, int C, int stride, int dilation, const float* dy, const float* weight, float* dx, cudaStream_t);
/* its weight gradient dweight (C, 1, 3, 3) = sum over output pixels of dy * x at each tap: per-block partials in the workspace, then
   one fixed-order reduction */
int skd_dwconv3x3_wgrad(int N, int H, int W, int C, int stride, int dilation, const float* x, const float* dy, float* dweight,
                        double* workspace, cudaStream_t);
/* BatchNorm2d (mean / var as skd_bnprelu_stats gives them, or the running statistics) followed by ReLU6 (relu6 = 1: clamp to [0, 6]) or
   by nothing (relu6 = 0), plus residual (may be NULL; linear mode only): out = z + residual, the projection of an inverted residual */
int skd_bnact_apply(long long P, int C, int relu6, const float* x, int ldx, const float* mean, const float* var, const float* weight,
                    const float* bias, float eps, const float* residual, int ldr, float* out, int ldo, cudaStream_t);
/* backward reduce pass: dweight = sum dz * xhat, dbias = sum dz (each may be NULL), dz = dout where 0 < z < 6 (ReLU6; z recomputed from
   x) or dout (linear); coef[2C] = (mean dz, mean dz * xhat) for the dx pass.  The residual's gradient is dout itself. */
int skd_bnact_bwd_reduce(long long P, int C, int relu6, const float* x, int ldx, const float* dout, int ldd, const float* mean,
                         const float* var, const float* weight, const float* bias, float eps, float* dweight, float* dbias, float* coef,
                         double* workspace, cudaStream_t);
/* dx pass: w * rsqrt(var + eps) * (dz - coef[c] - xhat * coef[C + c]) (training) or w * rsqrt(var + eps) * dz (running statistics) */
int skd_bnact_bwd_dx(long long P, int C, int relu6, const float* x, int ldx, const float* dout, int ldd, const float* mean, const float* var,
                     const float* weight, const float* bias, float eps, int training, const float* coef, float* dx, int lddx, cudaStream_t);

/* ---- J. feature-level distillation baselines (csrc/feature_kd.cu).  Maps are fp32 NHWC rows [P = N*H*W][C] at a row pitch in floats
        (ld >= C; channel slices of a concat buffer in place), read in float4 groups when C, the pitch and the base are 16-byte aligned.
        Fixed-order reductions, no atomics: two calls give bit-identical results. ---- */
/* attention transfer, at(x) = F.normalize(x.pow(2).mean(1).view(N, -1)): q = mean_c a_c^2 per pixel of the student map S (CS channels)
   and the teacher map T (CT channels, same N and HW); qhat [2][N*HW] = q / max(||q||_2, 1e-12) per sample (student, then teacher),
   norms [2][N] = ||q||_2; loss = mean over N*HW of (qhat_S - qhat_T)^2 */
int skd_at_fwd(int N, int HW, int CS, const float* S, int lds, int CT, const float* T, int ldt, float* qhat, float* norms, float* loss,
               cudaStream_t);
/* its gradient dS = (2 / C) a_c g with g = (h - qhat_S <qhat_S, h>) / ||q_S|| (h / 1e-12 where the norm is below the clamp),
   h = 2 (qhat_S - qhat_T) / (N*HW) * grad_out[0]; g: N*HW floats of workspace; dS at pitch ldd */
int skd_at_bwd(int N, int HW, int C, const float* S, int lds, const float* qhat, const float* norms, const float* grad_out, float* g,
               float* dS, int ldd, cudaStream_t);
/* MIMIC's F.mse_loss(R, T): loss = mean of (R - T)^2 over P*C; workspace: skd_loss_max_partials() doubles */
int skd_mse_fwd(long long P, int C, const float* R, int ldr, const float* T, int ldt, float* loss, double* workspace, cudaStream_t);
/* its gradient dR = 2 (R - T) / (P*C) * grad_out[0], at pitch ldd */
int skd_mse_bwd(long long P, int C, const float* R, int ldr, const float* T, int ldt, const float* grad_out, float* dR, int ldd,
                cudaStream_t);

/* ---- K. local pair-wise distillation (csrc/pairwise_local.cu): the pair-wise term with node i = (y, x) of the pooled h x w grid
        connected to j = (y + t d, x + u d), t, u in -r..r (r = (k - 1) / 2, j = i included) inside the grid.  Inputs are
        skd_pairwise_pool's dense rows pooled[N][h*w][C] (any C >= 1) and rnorm[N][h*w]; k odd in 3..15, d in 1..8.  fp32 FMA dot
        products, fixed-order double reduction of the loss, no atomics, no allocation: two calls give bit-identical results. ---- */
/* connected ordered pairs per image, P = (sum_y c_h(y)) * (sum_x c_w(x)), c_h(y) = #{t : 0 <= y + t d < h} */
long long skd_pairwise_local_pairs(int h, int w, int k, int d);
/* doubles of `partials` skd_pairwise_local_fwd needs */
long long skd_pairwise_local_partials(int N, int h, int w, int k, int d);
/* loss = sum over pairs of (a^T_ij - a^S_ij)^2 / (N * P), a_ij = (f_i . f_j) rnorm_i rnorm_j; E[N][h*w][k*k] (may be NULL) receives
   a^T - a^S at offset o = (t + r) k + (u + r), 0 where j lies outside the grid */
int skd_pairwise_local_fwd(int N, int h, int w, int CS, int CT, const float* pooled_S, const float* pooled_T, const float* rnorm_S,
                           const float* rnorm_T, int k, int d, float* E, float* loss, double* partials, cudaStream_t);
/* dpooled[N][h*w][CS] = -4 grad_out[0] / (N * P) * rnorm_S[i] * sum_o E[i][o] rnorm_S[j] pooled_S[j]; skd_pairwise_scatter finishes
   the feature gradient */
int skd_pairwise_local_bwd(int N, int h, int w, int CS, const float* E, const float* pooled_S, const float* rnorm_S, int k, int d,
                           const float* grad_out, float* dpooled, cudaStream_t);

/* ---- L. channel-wise distillation (csrc/cwd.cu): p = softmax over the HW positions of x / tau per (image, channel) of the student
        map S and the teacher map T, both N x C x HW at (image, channel, pixel) strides (NCHW, NHWC, pitched NHWC, channel slices);
        loss = tau^2 / (N*C) * sum pT (log pT - log pS), log p = x / tau - lse max-subtracted.  Any C >= 1 and HW >= 1 (N <= 32767).
        Fixed-order double reductions, no atomics, no allocation: two calls give bit-identical results. ---- */
/* doubles of `workspace` skd_cwd_fwd needs: 4 * N * C * chunks, the pixel chunks a function of (N, C, HW) */
long long skd_cwd_workspace(int N, int C, int HW);
/* loss[0]; lse [2][N][C] doubles (student, then teacher): the log-sum-exp of x / tau per (map, n, c), kept for the backward */
int skd_cwd_fwd(int N, int C, int HW, const float* S, long long s_sn, long long s_sc, long long s_sp, const float* T, long long t_sn,
                long long t_sc, long long t_sp, float tau, float* loss, double* lse, double* workspace, cudaStream_t);
/* dS = tau / (N*C) * grad_out[0] * (pS - pT), pS and pT recomputed from the maps and lse, at dS's strides */
int skd_cwd_bwd(int N, int C, int HW, const float* S, long long s_sn, long long s_sc, long long s_sp, const float* T, long long t_sn,
                long long t_sc, long long t_sp, float tau, const double* lse, const float* grad_out, float* dS, long long d_sn,
                long long d_sc, long long d_sp, cudaStream_t);

/* ---- M. intra-class feature variation distillation (csrc/ifv.cu): per image n and class k in [0, K), 1 <= K <= 255, the prototype
        P[n,k] = sum of the features of the pixels labelled k / (count + 1e-6), separately for the student map S (CS channels) and the
        teacher map T (CT channels), both N x HW NHWC rows at (image, pixel) strides with contiguous channels (pitches and channel
        slices allowed); cos_i = cosine_similarity(f_i, P[n, lab_i]) (eps 1e-8); loss = sum over the pixels labelled in [0, K) of
        (cos_S - cos_T)^2 / (N * HW).  Pixels with another label add exactly 0 to the loss and the gradient.  Fixed-order double
        reductions, no atomics, no allocation: two calls give bit-identical results. ---- */
/* out[N][h][w] int32 = labels[N][H][W] (contiguous int64) at F.interpolate(mode="nearest")'s source pixel
   min(floor(dst * (float(in) / out)), in - 1), the product rounded once in fp32; labels outside the int32 range become -1 */
int skd_labels_nearest(int N, int H, int W, const long long* labels, int h, int w, int* out, cudaStream_t);
/* doubles of `workspace` skd_ifv_fwd and skd_ifv_bwd need */
long long skd_ifv_workspace(int N, int HW, int K, int CS, int CT);
/* lab[N][HW] int32 (skd_labels_nearest's map) -> loss[0]; PS [N][K][CS] fp32 (the student's prototypes); stats [3][N][K] doubles:
   the counts, |P_S|^2 and |P_T|^2; pix [3][N][HW] fp32: cos_S, cos_S - cos_T and |f_S| (0 for an ignored pixel) */
int skd_ifv_fwd(int N, int HW, int K, const int* lab, const float* S, int CS, long long s_sn, long long s_sp, const float* T, int CT,
                long long t_sn, long long t_sp, float* loss, float* PS, double* stats, float* pix, double* workspace, cudaStream_t);
/* dS = grad_out[0] * d loss / d S (through the student's cosines and its prototypes) from what skd_ifv_fwd kept, at dS's strides */
int skd_ifv_bwd(int N, int HW, int K, const int* lab, const float* S, int CS, long long s_sn, long long s_sp, const float* PS,
                const double* stats, const float* pix, const float* grad_out, float* dS, long long d_sn, long long d_sp,
                double* workspace, cudaStream_t);

#ifdef __cplusplus
}
#endif
#endif /* SKD_B200_H_ */
