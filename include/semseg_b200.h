/*
 * semseg_b200 — C-ABI of the B200-native hot path of hszhao/semseg.
 *
 * Plain pointers and sizes only: no ATen / pybind types cross this boundary. Every entry point
 * takes device pointers, a cudaStream_t passed as void*, returns 0 on success or a negative
 * SEMSEG_E_* code, and never throws; semseg_last_error() returns the message of the last failure
 * on the calling thread. All kernels are sm_90a-only; there is no CPU fallback behind this ABI.
 *
 * What each group replaces in the reference (paths relative to the hszhao/semseg tree):
 *   - semseg_psamask_*        : lib/psa/src/gpu/operator.h:3-4 (psamask_forward_cuda / psamask_backward_cuda,
 *                               kernels lib/psa/src/gpu/psamask_cuda.cu:8-128) bound by
 *                               lib/psa/functions/psamask.py:19-35.
 *   - semseg_conv_*           : the cuDNN convolutions behind nn.Conv2d at model/resnet.py:63-69,108-113,133-137
 *                               (after the dilation patch model/pspnet.py:49-58), the heads
 *                               model/pspnet.py:65-69,73-77 and PSA 1x1s model/psanet.py:24-51.
 *   - semseg_bn_*             : nn.BatchNorm2d / nn.SyncBatchNorm (training + eval) and the in-place ReLU and
 *                               residual add around them, model/resnet.py:77-92.
 *   - semseg_pack_* / layout  : NCHW fp32 <-> NHWC bf16 at the module boundary (model/pspnet.py:80-105).
 *   - semseg_ppm_* / pool     : model/pspnet.py:12-26 (AdaptiveAvgPool2d, bilinear upsample, concat),
 *                               nn.MaxPool2d at model/resnet.py:115.
 *   - semseg_upsample_ce_*    : F.interpolate + CrossEntropyLoss + argmax, model/pspnet.py:94-103.
 *                               semseg_upsample_ce_ohem_*: the same with an OHEM cross-entropy criterion.
 *                               semseg_upsample_ce_{,ohem_}weighted_*: class weights / label smoothing.
 *                               semseg_upsample_ce_dice_*: soft Dice loss, alone or plus cross-entropy.
 *                               semseg_upsample_ce_rmi_*: RMI loss with its BCE term, optionally plus cross-entropy.
 *                               semseg_upsample_ce_focal_*: softmax focal loss, with or without class weights.
 *                               semseg_upsample_ce_relax_*: boundary label relaxation, with or without class
 *                               weights.
 *                               semseg_upsample_ce_lovasz_*: Lovász-Softmax, alone or plus cross-entropy, on
 *                               semseg_segsort_u32_pairs (segmented stable radix sort).
 *                               semseg_upsample_kd_*: pixel-wise distillation from a teacher's logits.
 *                               semseg_upsample_ce_unbiased_*, semseg_upsample_unkd_*: MiB's class-incremental
 *                               cross-entropy and distillation from the previous step's logits.
 *                               semseg_upsample_pl_*: confidence-masked pseudo-labels from a teacher's logits.
 *                               semseg_upsample_ce_entropy_*: entropy minimisation, plus cross-entropy.
 *                               semseg_gated_crf_*: the Gated CRF loss's pairwise term (csrc/crf.cu).
 *                               semseg_abl_*: the Active Boundary Loss term (csrc/boundary.cu).
 *   - semseg_window_*         : the post-network steps of sliding-window evaluation (tool/test.py:122-178): the eval
 *                               logit upsample (model/pspnet.py:95, tool/test.py:138), softmax and flip averaging
 *                               (tool/test.py:139-141), the overlap accumulation and normalisation
 *                               (tool/test.py:163-176) and the per-scale resize into the running total
 *                               (tool/test.py:177, 202).
 *                               semseg_window_scores_mc: the same scores averaged over Monte Carlo dropout draws,
 *                               with the mean sample entropy.
 *   - semseg_anomaly_*        : anomaly segmentation on the evaluation scores (max-logit, energy, standardized
 *                               max-logit) and its AUROC / AP / FPR95, with semseg_window_scores_stats.
 *   - semseg_densecrf_*       : dense CRF refinement of the evaluation scores (pydensecrf's DenseCRF2D with a Gaussian
 *                               and a bilateral Potts kernel), on a device permutohedral lattice.
 *   - semseg_augment          : tool/train.py:194-212's transform chains (util/transform.py), one launch per batch.
 *   - semseg_strong_augment   : the strong (colour jitter, grayscale, blur) student view of mean-teacher training.
 *
 * Activations are NHWC bf16 in HBM; "pitch" arguments are the distance between consecutive pixels in
 * elements (>= channels; lets a kernel read/write a channel slice of a wider concat buffer).
 */
#ifndef SEMSEG_B200_H
#define SEMSEG_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SEMSEG_OK 0
#define SEMSEG_E_INVALID (-1)  /* bad argument (shape, alignment, null pointer) */
#define SEMSEG_E_CUDA (-2)     /* CUDA runtime / driver error (message in semseg_last_error) */
#define SEMSEG_E_UNSUPPORTED (-3)

#define SEMSEG_MAX_TAPS 9

const char* semseg_last_error(void);
int semseg_abi_version(void);
/* Number of kernels this library has launched since load (bench.py reports it as gpu_launches). */
long long semseg_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * PSA mask (collect / distribute), fp32 NCHW exactly as the reference.
 *   psa_type 0 = collect, 1 = distribute (lib/psa/functions/psamask.py:9).
 *   fwd: in  [N, mH*mW, H, W] -> out [N, H*W, H, W]; every element of out is written (zeros included),
 *        so the caller does NOT need to pre-zero it (the reference requires a zeroed buffer).
 *   bwd: dout [N, H*W, H, W] -> din [N, mH*mW, H, W]; every element of din is written.
 */
int semseg_psamask_fwd(int psa_type, const float* in, float* out, int N, int H, int W, int mH, int mW,
                       void* stream);
int semseg_psamask_bwd(int psa_type, const float* dout, float* din, int N, int H, int W, int mH, int mW,
                       void* stream);

/* ------------------------------------------------------------------------------------------------
 * Fused point-wise spatial attention (model/psanet.py:81-91: psa_mask -> softmax(dim=1) -> bmm, SURVEY.md §8 f2): the
 * [N, HW, HW] attention map never exists in HBM.
 *   attn  fp32 NHWC [N, H*W, a_pitch] (a_pitch >= mH*mW): the attention logits as the 1x1 conv's F32 epilogue writes them
 *   feat / out / dout  activations NHWC [N, H*W, C] (C = 512), plain bf16 or split (hi, lo)
 *   stats fp32 [N, H*W, 2] = (max, 1/sum) of every target's softmax (written by mode 0, read by the backward calls)
 * semseg_psa_attend  mode 0: out[t,:]   = scale * sum_s P[t,s] * feat[s,:]   (forward; P = softmax over sources s)
 *                    mode 1: out[s,:]   = scale * sum_t P[t,s] * feat[t,:]   (feature gradient: pass dout as feat)
 * semseg_psa_attend_bwd_attn: dattn (same shape as attn, every element written: zero where the mask window gives no
 *   gradient) = P * (scale * dout . feat^T - rowsum(dout * out)) scattered back through the mask index map.
 * psa_type 0 = collect, 1 = distribute (lib/psa/functions/psamask.py:9). */
int semseg_psa_attend(int mode, int psa_type, const float* attn, int a_pitch, const void* feat, const void* feat_lo,
                      int feat_pitch, float* stats, void* out, void* out_lo, int out_pitch, int N, int H, int W, int mH,
                      int mW, int C, float scale, void* stream);
int semseg_psa_attend_bwd_attn(int psa_type, const float* attn, int a_pitch, const float* stats, const void* feat,
                               const void* feat_lo, int feat_pitch, const void* out, const void* out_lo, int out_pitch,
                               const void* dout, const void* dout_lo, int dout_pitch, float* dattn, int N, int H, int W,
                               int mH, int mW, int C, float scale, void* stream);

/* The same two operations for every option of the reference's PSA module (model/psanet.py:76-84). `form` is a bit mask:
 *   SEMSEG_PSA_DENSE      compact=True: mH*mW == H*W and a_pitch >= H*W; the owner's attention vector is indexed by the
 *                         other pixel's flat position (collect: L[t,s] = attn[t][s], distribute: L[t,s] = attn[s][t]);
 *                         every element of dattn is written from it. Without the bit: the odd mH x mW window above.
 *   SEMSEG_PSA_NO_SOFTMAX psa_softmax=False: P = L. stats may be NULL and are neither written nor read; in the logit
 *                         gradient dattn = scale * dout . feat^T scattered back, and out / out_lo may be NULL.
 * form 0 is semseg_psa_attend / semseg_psa_attend_bwd_attn, bit for bit. */
#define SEMSEG_PSA_DENSE 1
#define SEMSEG_PSA_NO_SOFTMAX 2
int semseg_psa_attend_ex(int mode, int psa_type, int form, const float* attn, int a_pitch, const void* feat,
                         const void* feat_lo, int feat_pitch, float* stats, void* out, void* out_lo, int out_pitch, int N,
                         int H, int W, int mH, int mW, int C, float scale, void* stream);
int semseg_psa_attend_bwd_attn_ex(int psa_type, int form, const float* attn, int a_pitch, const float* stats,
                                  const void* feat, const void* feat_lo, int feat_pitch, const void* out,
                                  const void* out_lo, int out_pitch, const void* dout, const void* dout_lo, int dout_pitch,
                                  float* dattn, int N, int H, int W, int mH, int mW, int C, float scale, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Implicit-GEMM convolution on wgmma tensor cores (bf16 operands, fp32 accumulation in registers).
 *
 * One descriptor drives fprop and dgrad (dgrad = fprop of dY with the transposed/flipped packed
 * weights). The output pixel grid is [N, H, W]; tap t reads input pixel
 * (n*img_mul + img_add[t], h + dh[t], w + dw[t]) of an input tensor [Nin, Hin, Win, Cin] with zero fill
 * outside it, multiplied by packed-weight slab wtap[t] of a [n_wtaps][Cout_rows][Cin_cols] bf16 tensor.
 */
enum {
  SEMSEG_EPI_RAW = 0,    /* y = bf16(acc); optional per-tile BN partial statistics */
  SEMSEG_EPI_AFFINE = 1, /* y = bf16(act(acc*scale[c] + shift[c] + residual)); scale/shift/residual optional */
  SEMSEG_EPI_F32 = 2     /* out_f32[pixel*out_pitch + c] = acc + shift[c] (bias), c < Cout */
};

typedef struct semseg_conv_desc {
  /* output pixel grid and GEMM sizes */
  int32_t N, H, W;
  int32_t Cin, Cout;
  /* input tensor (bf16 NHWC) */
  const void* x;
  int32_t Nin, Hin, Win, x_pitch;
  /* packed weights (bf16 [n_wtaps][w_rows][w_cols], w_cols contiguous) */
  const void* w;
  int32_t n_wtaps, w_rows, w_cols;
  /* taps */
  int32_t taps;
  int32_t dh[SEMSEG_MAX_TAPS], dw[SEMSEG_MAX_TAPS], wtap[SEMSEG_MAX_TAPS];
  int32_t img_mul, img_add[SEMSEG_MAX_TAPS];
  /* epilogue */
  int32_t epi_mode;
  int32_t relu;
  void* y; /* bf16 NHWC output (RAW / AFFINE) */
  int32_t y_pitch;
  const float* scale;   /* [Cout] or NULL */
  const float* shift;   /* [Cout] or NULL (bias in F32 mode) */
  const void* residual; /* bf16 NHWC [N,H,W,*] or NULL */
  int32_t res_pitch;
  float* out_f32; /* F32 mode output */
  int32_t out_pitch;
  /* RAW mode statistics: stats_partial [rows][3][Cout] = per epilogue-warp (sum, sum of squares, count) of the stored
   * bf16 outputs per channel, rows = semseg_conv_stats_rows(); NULL to skip. The kernel zeroes and fills every row. */
  float* stats_partial;
  /* bf16x3 operand mode (split storage): lo planes of x / y / residual (same shapes and pitches as the hi planes);
   * all NULL for plain bf16. With x_lo set, w must hold the lo slab directly behind the hi slab (w_split != 0,
   * semseg_pack_item.split != 0) and every K block is accumulated as x_hi*w_hi + x_lo*w_hi + x_hi*w_lo;
   * statistics are those of hi + lo. */
  const void* x_lo;
  void* y_lo;
  const void* residual_lo;
  int32_t w_split;
  /* K slicing (F32 epilogue only; 0 or 1 = off): the K blocks (64-channel block x tap) are cut into k_slices ranges,
   * slice s writes its fp32 partial to out_f32 + s*slice_stride (elements); the bias is added by slice 0 only. Used by
   * the bf16x3 mode to bound the length of one tensor-core accumulation chain (semseg_conv_k_slices,
   * semseg_conv_splitk_finish). */
  int32_t k_slices;
  int64_t slice_stride;
  /* e4m3 operand mode (eval convs of semseg_b200/fp8.py; e4m3 = 1, or 2 for the unpromoted accumulation that
   * tools/probe_accum.py measures against it): x is e4m3 NHWC [Nin,Hin,Win,x_pitch] bytes and w an
   * e4m3 slab [n_wtaps][w_rows][w_cols] (semseg_fp8_pack_weights); a K block is 128 channels and (e4m3 = 1) the
   * tensor-core partial of every K block is added into the fp32 accumulator (promotion). AFFINE epilogue only, which writes y (bf16, may be
   * NULL) and / or y8: e4m3 NHWC [N,H,W,y8_pitch] bytes of sat_e4m3(v * y8_qscale), v the bf16 epilogue's fp32 value.
   * Dequantisation (s_x * s_w[c]) is folded into scale[c] by the caller. Requires Cin % 128 == 0, Cout % 64 == 0, x_pitch,
   * w_cols, y8_pitch multiples of 16 (bytes), and no split operands, K slicing or statistics. */
  int32_t e4m3;
  void* y8;
  int32_t y8_pitch;
  float y8_qscale;
} semseg_conv_desc;

/* Number of K slices such that one slice holds at most max_kblocks K blocks (64-channel block x tap). */
int semseg_conv_k_slices(int Cin, int taps, int max_kblocks);
/* Sum the k_slices fp32 partials [k_slices][M][part_pitch] of a K-sliced conv in fp32 (round-to-nearest) and finish
 * like the conv epilogue would have: RAW (y = sum; optional statistics rows [rows][3][C] = (sum, sum of squares, count)
 * per pixel chunk, rows = semseg_conv_splitk_rows(M)) or AFFINE (y = act(sum*scale + shift + residual)). y (and the
 * residual) may be split (hi, lo) or plain. C % 64 == 0. */
int semseg_conv_splitk_rows(int M);
int semseg_conv_splitk_finish(const float* partial, int k_slices, long long slice_stride, int part_pitch, int M, int C,
                              int epi_mode, int relu, const float* scale, const float* shift, const void* residual,
                              const void* residual_lo, int res_pitch, void* y, void* y_lo, int y_pitch,
                              float* stats_partial, void* stream);
/* Rows of the statistics buffer (= 4 x CTAs launched) for an [N,H,W] x Cout output. */
int semseg_conv_stats_rows(int N, int H, int W, int Cout);
int semseg_conv_fprop(const semseg_conv_desc* d, void* stream);

/* wgrad: dw_partial[split][tap][co][ci] (fp32) = sum over the split's pixels of dy[p, co] * x[p + off(tap), ci].
 * Returns the number of splits through *n_splits (query with dw_partial == NULL first; the buffer must hold
 * n_splits*taps*Cout*Cin floats). */
typedef struct semseg_wgrad_desc {
  int32_t N, H, W;
  int32_t Cin, Cout;
  const void* x; /* bf16 NHWC [Nin,Hin,Win,*] */
  int32_t Nin, Hin, Win, x_pitch;
  const void* dy; /* bf16 NHWC [N,H,W,*] */
  int32_t dy_pitch;
  int32_t taps;
  int32_t dh[SEMSEG_MAX_TAPS], dw[SEMSEG_MAX_TAPS];
  int32_t img_mul, img_add[SEMSEG_MAX_TAPS];
  float* dw_partial;
  int32_t n_splits; /* in: 0 = let the library choose; out (via semseg_conv_wgrad_splits) */
  /* bf16x3 operand mode: lo planes of x and dy (both or neither); dy_hi*x_hi + dy_lo*x_hi + dy_hi*x_lo. */
  const void* x_lo;
  const void* dy_lo;
} semseg_wgrad_desc;

int semseg_conv_wgrad_splits(const semseg_wgrad_desc* d);
int semseg_conv_wgrad(const semseg_wgrad_desc* d, void* stream);
/* dw_oihw[co][ci][tap] (+)= sum_s dw_partial[s][tap][co][ci]; accumulate != 0 adds to the existing values. */
int semseg_wgrad_reduce(const float* dw_partial, int n_splits, int taps, int Cout, int Cin, float* dw_oihw,
                        int accumulate, void* stream);

/* Weight packing: fp32 OIHW [Cout][Cin][taps] -> the bf16 operand slabs of the conv kernels, for every conv of a model
 * in one launch (torch re-packs after each optimizer step). `items` is an array in DEVICE memory, sorted by tile0; an
 * item's tiles are its 32 x 32 (co, ci) blocks: tiles_ci = ceil(cols_f / 32) per row of ceil(cols_d / 32) rows.
 *   wf bf16 [taps][Cout][cols_f]  (wf[t][co][ci], zero padded)   — fprop B operand
 *   wd bf16 [taps][Cin][cols_d]   (wd[t][ci][co], zero padded)   — dgrad B operand
 *   wp bf16 [Cout][32]            (wp[co][t*Cin + ci], columns 9*Cin..31 zero; taps == 9 and Cin <= 3 only) — the stem
 *                                 conv as a 1x1 conv over semseg_im2col3x3s2 patches
 * cols_* = Cin / Cout rounded up to 8; wd and wp may be NULL. */
typedef struct semseg_pack_item {
  const float* w;
  void* wf;
  void* wd;
  void* wp;
  int Cout, Cin, taps;
  int cols_f, cols_d;
  int tile0, tiles_ci;
  int split; /* != 0: lo slabs follow the hi slabs (wf + taps*Cout*cols_f, wd + taps*Cin*cols_d, wp + Cout*32) */
} semseg_pack_item;
int semseg_pack_weights_multi(const semseg_pack_item* items_dev, int n_items, int n_tiles, int max_taps, void* stream);

/* ------------------------------------------------------------------------------------------------
 * FP8 (e4m3) eval support (csrc/fp8.cu). One quantisation formula throughout: q = sat_e4m3(v * qscale) with
 * qscale = 448 / amax computed in fp32, round to nearest even, saturating to +-448 (NaN stays NaN).
 *   semseg_fp8_quantize: bf16 NHWC x [M pixels][x_pitch] -> e4m3 y [M][y_pitch], C channels, q(x * qscale).
 *   semseg_fp8_amax    : amax_bits[0] = max(amax_bits[0], max |x| as fp32 bits) over a bf16 NHWC tensor; |x| bit
 *                        patterns order as integers, so the running maximum over calls is exact and order-free.
 *                        NaN inputs are ignored.
 *   semseg_fp8_pack_weights: fp32 OIHW w [Cout][Cin][taps] -> e4m3 slab wf [taps][Cout][Cin] = q(w) with the
 *                        per-output-channel qscale = 448 / amax_c, and the dequantisation scale scale_w[c] = amax_c / 448
 *                        (amax_c = max |w| of output channel c; an all-zero channel uses amax_c = 448).
 *                        Cin % 16 == 0; one launch per conv, at freeze time.
 * Pitches are in elements; C % 16 == 0, pitches multiples of 16. */
int semseg_fp8_quantize(const void* x, int x_pitch, void* y, int y_pitch, long long M, int C, float qscale,
                        void* stream);
int semseg_fp8_amax(const void* x, int x_pitch, long long M, int C, unsigned int* amax_bits, void* stream);
int semseg_fp8_pack_weights(const float* w, int Cout, int Cin, int taps, void* wf, float* scale_w, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Layout conversion at the module boundary.
 */
int semseg_nchw_f32_to_nhwc_bf16(const float* in, void* out, void* out_lo, int N, int C, int H, int W, int out_pitch,
                                 void* stream);
int semseg_nhwc_bf16_to_nchw_f32(const void* in, const void* in_lo, float* out, int N, int C, int H, int W,
                                 int in_pitch, void* stream);
int semseg_nhwc_f32_to_nchw_f32(const float* in, float* out, int N, int C, int H, int W, int in_pitch,
                                void* stream);

/* Stem conv (3x3, stride 2, pad 1, Cin <= 3 — model/resnet.py:106-108) as a 1x1 conv over input patches:
 *   out[n, ho, wo, (r*3+s)*Cin + c] = x[n, 2ho-1+r, 2wo-1+s, c], zero outside the image and for columns >= 9*Cin;
 *   out is [N, (H-1)/2+1, (W-1)/2+1, 32] bf16. x is NHWC bf16 with x_pitch >= 4 (the first Cin channels are read). */
int semseg_im2col3x3s2(const void* x, int x_pitch, int N, int H, int W, int Cin, void* out, void* stream);

/* Input gradient of that stem conv (the adjoint of semseg_im2col3x3s2 + the patch-slab product), fp32 NCHW:
 *   dx[n, c, y, x] = sum_{(r, s, ho, wo): 2ho-1+r = y, 2wo-1+s = x} sum_k dy[n, ho, wo, k] * w[k, c, r, s]
 * dy     : bf16 NHWC [N, Ho, Wo, >= Cout] with dy_pitch (a multiple of 8, 16-byte aligned); dy_lo its lo plane in
 *          bf16x3 (same pitch), else NULL
 * wp     : the patch slab bf16 [Cout][32], column (r*3+s)*Cin + c = w[:, c, r, s]; with wp_split = 1 its lo slab follows
 *          (required exactly when dy_lo is given: the three products hi*hi + lo*hi + hi*lo)
 * dx_nchw: fp32 [N, Cin, H, W], every element written; Ho = (H-1)/2+1, Wo = (W-1)/2+1, 1 <= Cin <= 3, Cout = 64.
 * Deterministic: fp32 accumulation in a fixed order, no atomics. */
int semseg_stem_dgrad3x3s2(const void* dy, const void* dy_lo, int dy_pitch, int N, int Ho, int Wo, int H, int W, int Cin,
                           int Cout, const void* wp, int wp_split, float* dx_nchw, void* stream);

/* 2x2 phase decomposition used to run stride-2 convolutions (model/resnet.py:108 conv1, layer2.0 conv2 and
 * downsample) on the stride-1 tensor-core kernel:
 *   xp [4][N][Hh][Wh][C], Hh = (H+1)/2:  xp[ph*2+pw][n][i][j] = x[n][2i+ph][2j+pw] (zero outside x). */
int semseg_space_to_phases(const void* x, int x_pitch, int N, int H, int W, int C, void* xp, void* stream);
int semseg_phases_to_space(const void* xp, int N, int H, int W, int C, void* x, void* stream);

/* ------------------------------------------------------------------------------------------------
 * BatchNorm (training statistics, apply, backward) on NHWC bf16 tensors, fp32 statistics.
 */
/* Merge the conv epilogue's per-CTA partials [rows][3][C] (Chan) into per-channel (mean, M2, count): out_stats [3][C]. */
int semseg_bn_merge_partials(const float* stats_partial, int rows, int C, float* out_stats, void* stream);
/* Scratch floats of the two-stage backward reductions (bn_bwd_reduce, bn_bwd_frozen) for an [M][C] tensor. */
long long semseg_bn_workspace_floats(int M, int C);
/* Merge R rank-stat blocks [R][3][C] (R = 1 without SyncBN) and finalise:
 *   mean_invstd [3][C] = (mean, 1/sqrt(var+eps), total samples per channel over all ranks — every finalize entry point
 *   writes the three rows); scale_shift [2][C] with scale = gamma*invstd, shift = beta - mean*scale;
 *   running_mean/var updated in place (momentum, unbiased var) when non-NULL. */
int semseg_bn_finalize(const float* rank_stats, int R, int C, const float* gamma, const float* beta, float eps,
                       float momentum, float* running_mean, float* running_var, float* mean_invstd,
                       float* scale_shift, void* stream);
/* Peer exchange (SyncBatchNorm over NVLink peer memory instead of NCCL, inside the kernel): the arguments
 * (peer_bufs, world, rank, slot, slot_floats, seq_ptr) that semseg_bn_finalize_partials and semseg_bn_bwd_reduce take.
 * peer_bufs == NULL: a single rank, and the other five are ignored. Otherwise peer_bufs[world] (world <= 8, rank < world)
 * are device pointers into every rank's symmetric (peer-mapped) allocation: a zero-initialised buffer of
 * n_slots*world*slot_floats 8-byte words. Every value travels as one {fp32, sequence number} word that the sender stores
 * into sub-block `rank` of the slot in every peer's buffer; the receiver polls its own memory (flag-in-data, no fences).
 * `slot` must be unique per exchange within a step; the sequence number is the uint32 read from the device address
 * seq_ptr when the kernel runs, strictly increasing per step and the same on every rank (a device-resident step
 * counter, so that a captured CUDA graph with baked-in slots can be replayed). */
/* Merge the per-CTA conv partials [rows][3][C] and finalise in one launch, like semseg_bn_merge_partials +
 * semseg_bn_finalize (R = 1). With peers, this rank's (mean, M2, n) [3][C] (3*C <= slot_floats) is exchanged and the
 * ranks' moments are merged in rank order before the finalise; every rank computes the same bits. */
int semseg_bn_finalize_partials(const float* stats_partial, int rows, int C, const float* gamma, const float* beta,
                                float eps, float momentum, float* running_mean, float* running_var, float* mean_invstd,
                                float* scale_shift, void* const* peer_bufs, int world, int rank, int slot,
                                int slot_floats, const void* seq_ptr, void* stream);
/* Eval-mode folding: scale = gamma/sqrt(var+eps), shift = beta - mean*scale. */
int semseg_bn_fold_eval(const float* gamma, const float* beta, const float* running_mean,
                        const float* running_var, float eps, int C, float* scale_shift, void* stream);
/* y = act(x*scale[c] + shift[c] + residual). */
int semseg_bn_apply(const void* x, const void* x_lo, int x_pitch, const float* scale_shift, const void* residual,
                    const void* residual_lo, int res_pitch, void* y, void* y_lo, int y_pitch, int M, int C, int relu,
                    void* stream);
/* Backward reduce: with dz = dy * (y > 0 if relu) and xhat = (x - mean)*invstd,
 *   sums [2][C] = this rank's (sum dz, sum dz*xhat). y may be NULL when relu == 0; when relu != 0 and y == NULL the mask
 *   is recomputed as fma(x, scale, shift) > 0 from scale_shift [2][C] (valid when the forward had no residual).
 *   With peers (see the peer exchange above; 2*C <= slot_floats), sums_total [2][C] = the sums added over the ranks in
 *   rank order; without, sums_total may be NULL and is not written. */
int semseg_bn_bwd_reduce(const void* dy, const void* dy_lo, int dy_pitch, const void* y, const void* y_lo, int y_pitch,
                         const void* x, const void* x_lo, int x_pitch, const float* mean_invstd,
                         const float* scale_shift, int M, int C, int relu, float* workspace,
                         long long workspace_floats, float* sums, float* sums_total, void* const* peer_bufs,
                         int world, int rank, int slot, int slot_floats, const void* seq_ptr, void* stream);
/* Backward apply: dx = gamma*invstd*(dz - sum_dz/count - xhat*sum_dzxhat/count);
 *   dres (optional) = dz; dgamma = sum_dzxhat, dbeta = sum_dz written to dgamma_dbeta [2][C].
 *   count = total number of samples per channel across all ranks; count <= 0 takes it from mean_invstd row 2 (what
 *   the forward exchange measured: correct also when the ranks hold different numbers of pixels, as torch SyncBN). */
int semseg_bn_bwd_apply(const void* dy, const void* dy_lo, int dy_pitch, const void* y, const void* y_lo, int y_pitch,
                        const void* x, const void* x_lo, int x_pitch, const float* mean_invstd, const float* gamma,
                        const float* scale_shift, const float* sums, float count, int M, int C, int relu, void* dx,
                        void* dx_lo, int dx_pitch, void* dres, void* dres_lo, int dres_pitch, float* dgamma_dbeta,
                        void* stream);
/* Frozen BatchNorm backward (BN normalised with its running statistics inside a network that trains), one pass.
 *   scale = gamma/sqrt(running_var+eps), shift = beta - running_mean*scale (gamma / beta may be NULL: 1 / 0);
 *   dz = dy * (y > 0 if relu); d_raw = dz*scale; dres (optional) = dz;
 *   sums [2][C] (optional) = (sum dz, sum dz*xhat) = (dbeta, dgamma), xhat = (raw - running_mean)/sqrt(running_var+eps),
 *   reduced in a fixed order (deterministic) through `workspace` (semseg_bn_workspace_floats(M, C) floats).
 *   The mask comes from y, or — relu with y == NULL, valid when the forward had no residual — from
 *   fma(raw, scale, shift) > 0. raw == NULL: the sum dz*xhat row is zero. sums == NULL: no reduction, no workspace. */
int semseg_bn_bwd_frozen(const void* dy, const void* dy_lo, int dy_pitch, const void* y, const void* y_lo, int y_pitch,
                         const void* raw, const void* raw_lo, int raw_pitch, const float* gamma, const float* beta,
                         const float* running_mean, const float* running_var, float eps, int M, int C, int relu,
                         void* d_raw, void* d_raw_lo, int d_raw_pitch, void* dres, void* dres_lo, int dres_pitch,
                         float* workspace, long long workspace_floats, float* sums, void* stream);
/* out = a + b (merges gradient branches; split-aware, unlike an elementwise add of the two planes). */
int semseg_add_act(const void* a, const void* a_lo, int a_pitch, const void* b, const void* b_lo, int b_pitch,
                   void* out, void* out_lo, int out_pitch, int M, int C, void* stream);
/* out[n, p, c] = x[n, p, c] * scale[n*C + c] for p < HW: nn.Dropout2d's per-(image, channel) factor
 * (model/pspnet.py:68,76) and its backward. */
int semseg_scale_nc(const void* x, const void* x_lo, int x_pitch, const float* scale, void* out, void* out_lo,
                    int out_pitch, int N, int HW, int C, void* stream);
/* Feature perturbation (UniMatch's FP stream). Fork: x holds N images [N][HW][x_pitch], out 2N [2N][HW][out_pitch];
 * out[n] = x[n] and out[N + n] = x[n] * scale[n*C + c], each computed in fp32 from x (hi + lo) and stored by the
 * activation store, so the second half is bit-equal to semseg_scale_nc(x, scale) and scale = 1 gives equal halves.
 * Fold (its backward): d holds 2N images, out N; out[n] = d[n] + scale[n*C + c] * d[N + n] in fp32 (product and sum
 * each rounded to nearest, no fma), rounded once to the activation form. Both: C % 8 == 0, pitches multiples of 8 and
 * at least C, 16-byte aligned bases and scale, one storage form (plain or split) for input and output. */
int semseg_fp_fork(const void* x, const void* x_lo, int x_pitch, const float* scale, void* out, void* out_lo,
                   int out_pitch, int N, int HW, int C, void* stream);
int semseg_fp_fold(const void* d, const void* d_lo, int d_pitch, const float* scale, void* out, void* out_lo,
                   int out_pitch, int N, int HW, int C, void* stream);
/* The same with the first N of M >= N images perturbed (UniMatch's two strong streams, the first one perturbed).
 * Fork: x holds M images, out M + N; out[m] = x[m] and out[M + n] = x[n] * scale[n*C + c] for n < N. Fold: d holds
 * M + N images, out M; out[m] = d[m], plus scale[n*C + c] * d[M + n] for n < N, in the arithmetic above, rounded once.
 * The other rules are the ones above; M = N gives semseg_fp_fork / semseg_fp_fold's results bit for bit. */
int semseg_fp_fork_prefix(const void* x, const void* x_lo, int x_pitch, const float* scale, void* out, void* out_lo,
                          int out_pitch, int M, int N, int HW, int C, void* stream);
int semseg_fp_fold_prefix(const void* d, const void* d_lo, int d_pitch, const float* scale, void* out, void* out_lo,
                          int out_pitch, int M, int N, int HW, int C, void* stream);
/* fp32 rows [M][in_pitch] (C columns used) -> activation rows [M][out_pitch], columns C..Cp-1 zero (Cp % 8 == 0). */
int semseg_f32_to_act(const float* in, int in_pitch, void* out, void* out_lo, int out_pitch, long long M, int C,
                      int Cp, void* stream);
/* activation rows [M][in_pitch] (C % 8 == 0 columns) -> fp32 rows [M][out_pitch]. */
int semseg_act_to_f32(const void* in, const void* in_lo, int in_pitch, float* out, int out_pitch, long long M, int C,
                      void* stream);

/* ------------------------------------------------------------------------------------------------
 * nn.MaxPool2d(kernel_size=3, stride=2, padding=1) on NHWC bf16 (model/resnet.py:115): y [N,Ho,Wo,C] with
 * Ho = (H-1)/2+1; argcode uint8 [N,Ho,Wo,C] (or NULL) = window position 0..8 of the arg-max (first maximum in window
 * order, as ATen). Backward gathers with those codes: dx [N,H,W,C] dense, deterministic, no atomics.
 */
int semseg_maxpool3x3s2_fwd(const void* x, const void* x_lo, void* y, void* y_lo, void* argcode, int N, int H, int W,
                            int C, void* stream);
int semseg_maxpool3x3s2_bwd(const void* argcode, const void* dy, const void* dy_lo, void* dx, void* dx_lo, int N,
                            int H, int W, int C, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Pyramid pooling module data movement (model/pspnet.py:12-26), NHWC bf16, all bins in one launch.
 *   bins[nb] = pooled sizes (1,2,3,6); per-bin tensors are [N][b][b][channels] contiguous bf16.
 *   ppm_pool            : pooled_k = AdaptiveAvgPool2d(b_k)(x), window [floor(i*H/b), ceil((i+1)*H/b)).
 *   ppm_pool_bwd        : dx (dense, every element written) = sum_k adjoint of the pooling applied to dpooled_k.
 *   ppm_pool_bwd        : dx = adjoint of ppm_pool (+ `add` [N,H,W,add_pitch], nullable: the identity branch of the
 *                         concat, so the two gradients of x are summed in this kernel instead of by autograd).
 *   ppm_upsample_concat : out[..., 0:C] = x; out[..., C + k*Cr : C + (k+1)*Cr] = bilinear(align_corners=True) of
 *                         feats_k to H x W (the torch.cat of model/pspnet.py:26 written in place).
 *   ppm_upsample_bwd    : dfeats_k = adjoint of the bilinear upsample applied to dout[..., c_off + k*Cr : ...].
 */
int semseg_ppm_pool(const void* x, const void* x_lo, int x_pitch, int N, int H, int W, int C, const int* bins,
                    void* const* pooled, void* const* pooled_lo, int nb, void* stream);
int semseg_ppm_pool_bwd(void* const* dpooled, void* const* dpooled_lo, const int* bins, int nb, int N, int H, int W,
                        int C, void* dx, void* dx_lo, int dx_pitch, const void* add, const void* add_lo, int add_pitch,
                        void* stream);
int semseg_ppm_upsample_concat(const void* x, const void* x_lo, int x_pitch, void* const* feats, void* const* feats_lo,
                               const int* bins, int nb, int N, int H, int W, int C, int Cr, void* out, void* out_lo,
                               int out_pitch, void* stream);
int semseg_ppm_upsample_bwd(const void* dout, const void* dout_lo, int dout_pitch, int c_off, void* const* dfeats,
                            void* const* dfeats_lo, const int* bins, int nb, int N, int H, int W, int Cr, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Bilinear resize, align_corners=True, of an NHWC activation [N,Hi,Wi,C] -> [N,Ho,Wo,C] (F.interpolate at
 * model/psanet.py:61,97) and its adjoint (dy [N,Ho,Wo,C] -> dx [N,Hi,Wi,C]; a deterministic gather, no atomics).
 */
int semseg_resize_bilinear_fwd(const void* x, const void* x_lo, int x_pitch, int N, int Hi, int Wi, int C, int Ho,
                               int Wo, void* y, void* y_lo, int y_pitch, void* stream);
int semseg_resize_bilinear_bwd(const void* dy, const void* dy_lo, int dy_pitch, int N, int Hi, int Wi, int C, int Ho,
                               int Wo, void* dx, void* dx_lo, int dx_pitch, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Fused logit upsample (bilinear, align_corners=True, x8; the zoom entry points below take zoom 1, 2, 4 or 8) +
 * cross-entropy (ignore_index, mean over valid
 * pixels) + argmax: F.interpolate + CrossEntropyLoss + max(1) of model/pspnet.py:94-103 without the
 * [N, classes, Ho, Wo] tensor. Requires Ho = 8(h-1)+1, Wo = 8(w-1)+1 (zoom_factor 8), classes <= 256.
 *   logits fp32 NHWC [N,h,w,C] (pitch), target int64 [N,Ho,Wo].
 *   fwd: loss_out[0] = mean CE, loss_out[1] = number of non-ignored pixels; argmax int64 [N,Ho,Wo] (or NULL);
 *        lse fp32 [N,Ho,Wo] (saved for backward); workspace: semseg_upsample_ce_workspace_floats() floats.
 *   bwd: dlogits fp32 [N,h,w,C] (dense, every element written) = grad_out[0] * d(mean CE)/dlogits;
 *        workspace: semseg_upsample_ce_bwd_workspace_floats() floats (row-reduced intermediate [N][Ho][w][C]).
 */
long long semseg_upsample_ce_workspace_floats(int N, int Ho, int Wo);
int semseg_upsample_ce_fwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                           int Ho, int Wo, int ignore_index, float* workspace, float* loss_out, int64_t* argmax,
                           float* lse, void* stream);
long long semseg_upsample_ce_bwd_workspace_floats(int N, int Ho, int w, int C);
int semseg_upsample_ce_bwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                           int Ho, int Wo, int ignore_index, const float* lse, const float* loss_info,
                           const float* grad_out, float* workspace, float* dlogits, void* stream);
/* The same at zoom factor `zoom` in {1, 2, 4, 8}: requires Ho = zoom(h-1)+1, Wo = zoom(w-1)+1 (zoom 1: no
 * interpolation, plain cross-entropy + argmax of the logits). The forward workspace holds 2 floats per forward CTA,
 * N * ((Ho-1)/zoom+1) * ceil(Wo/128) CTAs; the backward one [N][(Ho-1)/zoom+1][2][w][C] floats. The workspace functions
 * return -1 for a zoom outside {1, 2, 4, 8}. Zoom 8 is exactly the entry points above. */
long long semseg_upsample_ce_zoom_workspace_floats(int N, int Ho, int Wo, int zoom);
int semseg_upsample_ce_zoom_fwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                                int Ho, int Wo, int zoom, int ignore_index, float* workspace, float* loss_out,
                                int64_t* argmax, float* lse, void* stream);
long long semseg_upsample_ce_zoom_bwd_workspace_floats(int N, int Ho, int w, int C, int zoom);
int semseg_upsample_ce_zoom_bwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                                int Ho, int Wo, int zoom, int ignore_index, const float* lse, const float* loss_info,
                                const float* grad_out, float* workspace, float* dlogits, void* stream);
/* OHEM cross-entropy (semseg_b200/losses.py OhemCrossEntropyLoss) on the same fused upsample at zoom `zoom`: with
 * p_t = softmax(v)[target] and nll = -log_softmax(v)[target] per valid pixel (target != ignore_index, 0 <= target < C),
 * k = min(min_kept, n_v - 1) over the n_v valid pixels, thr = max(thresh, k-th smallest p_t (0-based)), the loss is the
 * mean nll over the kept pixels, p_t < thr; 0 (and a zero gradient) when none is kept. Requires 0 <= thresh <= 1,
 * min_kept >= 0. The selection is exact and runs on the device (no host synchronisation; graph-capturable).
 *   fwd: loss_out[0] = mean nll over the kept pixels, loss_out[1] = kept count; argmax (or NULL) and lse as above;
 *        pt, nll fp32 [N,Ho,Wo] (pt = -1, nll = 0 where the pixel is not valid); thr fp32 [1] = the threshold.
 *        workspace: semseg_upsample_ce_ohem_workspace_floats() floats.
 *   bwd: dlogits as above, with every pixel whose pt is not below *thr treated as ignored (the forward's kept set);
 *        workspace: semseg_upsample_ce_ohem_bwd_workspace_floats() floats (the same as the zoom backward's). */
long long semseg_upsample_ce_ohem_workspace_floats(int N, int Ho, int Wo, int zoom);
int semseg_upsample_ce_ohem_fwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                                int Ho, int Wo, int zoom, int ignore_index, float thresh, int min_kept,
                                float* workspace, float* loss_out, int64_t* argmax, float* lse, float* pt, float* nll,
                                float* thr, void* stream);
long long semseg_upsample_ce_ohem_bwd_workspace_floats(int N, int Ho, int w, int C, int zoom);
int semseg_upsample_ce_ohem_bwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                                int Ho, int Wo, int zoom, int ignore_index, const float* lse, const float* pt,
                                const float* thr, const float* loss_info, const float* grad_out, float* workspace,
                                float* dlogits, void* stream);
/* Class-weighted and label-smoothed cross-entropy (nn.CrossEntropyLoss(weight, ignore_index, reduction='mean',
 * label_smoothing)) on the same fused upsample at zoom `zoom`. class_weight fp32 [C] on the device (NULL = all ones;
 * read at every launch, so a CUDA graph sees in-place edits), label_smoothing eps in [0, 1]. With w_t the weight of a
 * valid pixel's target, W = sum_c w_c and lse = logsumexp_c v_c:
 *   loss_pix = (1-eps) w_t (lse - v_t) + (eps/C) sum_c w_c (lse - v_c),  loss = sum over valid pixels / D, D = sum w_t;
 * loss 0 and an exactly zero gradient when D = 0 (where torch gives nan). Out-of-range targets are ignored.
 *   fwd: loss_out[0] = loss, loss_out[1] = D; argmax (or NULL) and lse as above; workspace:
 *        semseg_upsample_ce_weighted_workspace_floats() floats (the zoom forward's).
 *   bwd: dlogits fp32 [N,h,w,C] = grad_out[0] * dloss/dlogits; workspace:
 *        semseg_upsample_ce_weighted_bwd_workspace_floats() floats (the zoom backward's). Same width limit as the zoom
 *        backward.
 * Weighted OHEM (losses.OhemCrossEntropyLoss(weight=...)): the OHEM entry points with nll = w_t (lse - v_t); the
 * selection on p_t is unweighted and the loss is the plain mean of w_t * nll over the kept pixels. Workspaces are the
 * OHEM ones. All of these reject a bad shape, zoom, option or null output before any CUDA call. */
long long semseg_upsample_ce_weighted_workspace_floats(int N, int Ho, int Wo, int zoom);
int semseg_upsample_ce_weighted_fwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                                    int Ho, int Wo, int zoom, int ignore_index, const float* class_weight,
                                    float label_smoothing, float* workspace, float* loss_out, int64_t* argmax,
                                    float* lse, void* stream);
long long semseg_upsample_ce_weighted_bwd_workspace_floats(int N, int Ho, int w, int C, int zoom);
int semseg_upsample_ce_weighted_bwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                                    int Ho, int Wo, int zoom, int ignore_index, const float* class_weight,
                                    float label_smoothing, const float* lse, const float* loss_info,
                                    const float* grad_out, float* workspace, float* dlogits, void* stream);
int semseg_upsample_ce_ohem_weighted_fwd(const float* logits, int pitch, int N, int h, int w, int C,
                                         const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                         float thresh, int min_kept, const float* class_weight, float* workspace,
                                         float* loss_out, int64_t* argmax, float* lse, float* pt, float* nll,
                                         float* thr, void* stream);
int semseg_upsample_ce_ohem_weighted_bwd(const float* logits, int pitch, int N, int h, int w, int C,
                                         const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                         const float* class_weight, const float* lse, const float* pt,
                                         const float* thr, const float* loss_info, const float* grad_out,
                                         float* workspace, float* dlogits, void* stream);
/* Soft Dice loss, alone or plus cross-entropy (semseg_b200/losses.py DiceLoss), on the same fused upsample at zoom
 * `zoom`. With p = softmax(v) and sums over every valid pixel (target != ignore_index, 0 <= target < C) of every image:
 *   n_c = #{t = c},  I_c = sum p_c [t = c],  S_c = sum p_c + n_c,  dice_c = (2 I_c + smooth) / max(S_c + smooth, eps)
 *   loss = (1/C) sum_{c: n_c > 0} (1 - dice_c) + ce_weight * CE,   CE = mean over the valid pixels of lse - v_t
 * loss 0 and an exactly zero gradient when no pixel is valid. smooth, eps, ce_weight finite and >= 0. The staged rows
 * take 12 bytes per pixel: Wo <= 229376 / (12 zoom), i.e. 2389 at zoom 8; a wider target is rejected before any launch.
 *   fwd: loss_out[0] = loss, loss_out[1] = number of valid pixels; argmax (or NULL) and lse as the zoom forward's
 *        (the same bits); table fp32 [5C+2] = alpha[C], beta[C], I[C], S[C], n[C], ce_weight / n_valid, 1 (the
 *        gradient coefficients and the per-class statistics, written on the device: graph-capturable);
 *        workspace: semseg_upsample_ce_dice_workspace_floats() floats, 8-byte aligned.
 *   bwd: dlogits fp32 [N,h,w,C] = grad_out[0] * dloss/dlogits from the forward's lse and table; workspace:
 *        semseg_upsample_ce_dice_bwd_workspace_floats() floats.
 * Both reject a bad shape, zoom, option, width or null output before any CUDA call; the workspace functions return -1
 * for a zoom outside {1, 2, 4, 8}. */
long long semseg_upsample_ce_dice_workspace_floats(int N, int Ho, int Wo, int C, int zoom);
int semseg_upsample_ce_dice_fwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                                int Ho, int Wo, int zoom, int ignore_index, float smooth, float eps, float ce_weight,
                                float* workspace, float* loss_out, int64_t* argmax, float* lse, float* table,
                                void* stream);
long long semseg_upsample_ce_dice_bwd_workspace_floats(int N, int Ho, int Wo, int w, int C, int zoom);
int semseg_upsample_ce_dice_bwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                                int Ho, int Wo, int zoom, int ignore_index, const float* lse, const float* table,
                                const float* grad_out, float* workspace, float* dlogits, void* stream);
/* Region Mutual Information loss (Zhao, Wang, Cai, NeurIPS 2019; semseg_b200/losses.py RMILoss) with its sigmoid BCE
 * term and optionally cross-entropy, on the same fused upsample at zoom `zoom`, in the authors' default configuration
 * (average pooling 4, radius 3, lambda_way 1, clip 1e-6: fixed). For the upsampled logits z and the target t:
 *   v = [t != ignore_index and 0 <= t < C],  y_c = [t = c] v,  s_c = sigmoid(z_c),  q_c = s_c v + 1e-6
 *   BCE = sum_{pixels, c} v (softplus(z_c) - y_c z_c) / (n_valid + 1)
 *   Y, Q = 4x4 average pools (stride 4, no padding) of y, q: [N][C][Hp][Wp], Hp = Ho / 4, Wp = Wo / 4 (floor)
 *   a_k, b_k = the 3x3 neighbourhoods (row-major (dy, dx)) of pooled cell k = (i, j), i < Hp-2, j < Wp-2, of Y and Q;
 *   K = (Hp-2)(Wp-2); centred a~, b~ (fp64): S_aa, S_bb, S_ab = sum_k a~a~', b~b~', a~b~' (9x9, not divided by K)
 *   P = S_bb + pos_alpha I,  A = S_aa - S_ab P^-1 S_ab',  r[n,c] = 1/2 log det(A + pos_alpha I)   (Cholesky)
 *   RMI = sum_c ((1/N) sum_n r[n,c]) / 9,   loss = bce_weight BCE + (1 - bce_weight) RMI + ce_weight CE
 * CE = mean over the valid pixels of lse - z_t (0 with none). 0 <= bce_weight <= 1, pos_alpha finite > 0, ce_weight
 * finite >= 0, Ho and Wo >= 12. The backward's rows kernel stages 8 bytes per pixel: Wo <= 229376 / (8 zoom), i.e.
 * 3584 at zoom 8; wider targets are rejected before any launch.
 *   fwd: loss_out fp32 [5] = (loss, n_valid, BCE, RMI, CE); argmax (or NULL) and lse as the zoom forward's (the same
 *        bits); pooled fp32 [2][N][C][Hp][Wp] = Y then Q (kept for the backward: 2 N C Hp Wp floats, 268 MB at
 *        16 x 150 x 473^2); table fp32 [semseg_upsample_ce_rmi_table_floats()] = per (n, c) a 184-float record
 *        (T [9][18] = [G_ab' | 2 G_bb] row-major, mean a [9], mean b [9], r, 3 zeros), then 4 scalars for the backward
 *        (ce_weight / n_valid, 1, bce_weight / (n_valid + 1), (1 - bce_weight) / (144 N)); written on the device:
 *        graph-capturable. workspace: semseg_upsample_ce_rmi_workspace_floats() floats, 8-byte aligned: the raw fp64
 *        moment sums [N*C][189] first (sum a[9], sum b[9], a a' upper triangle row-major [45], b b' the same [45],
 *        a b' [9][9]), then r fp64 [N*C], then the CE and BCE partials.
 *   bwd: dlogits fp32 [N,h,w,C] = grad_out[0] * dloss/dlogits from the forward's lse, pooled maps and table, with
 *        G_ab = -M S_ab P^-1, G_bb = 1/2 P^-1 S_ab' M S_ab P^-1, M = (A + pos_alpha I)^-1; workspace:
 *        semseg_upsample_ce_rmi_bwd_workspace_floats() floats (the transpose-upsample rows, then dr/dQ [N][C][Hp][Wp]).
 * Both reject a bad shape, zoom, option, width, null pointer or misalignment before any CUDA call; the workspace
 * functions return -1 for a zoom outside {1, 2, 4, 8}. */
long long semseg_upsample_ce_rmi_workspace_floats(int N, int Ho, int Wo, int C, int zoom);
long long semseg_upsample_ce_rmi_table_floats(int N, int C);
int semseg_upsample_ce_rmi_fwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                               int Ho, int Wo, int zoom, int ignore_index, float bce_weight, float pos_alpha,
                               float ce_weight, float* workspace, float* loss_out, int64_t* argmax, float* lse,
                               float* pooled, float* table, void* stream);
long long semseg_upsample_ce_rmi_bwd_workspace_floats(int N, int Ho, int Wo, int w, int C, int zoom);
int semseg_upsample_ce_rmi_bwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                               int Ho, int Wo, int zoom, int ignore_index, const float* lse, const float* pooled,
                               const float* table, const float* grad_out, float* workspace, float* dlogits,
                               void* stream);
/* Softmax focal loss (Lin et al., ICCV 2017; semseg_b200/losses.py FocalLoss) on the same fused upsample at zoom
 * `zoom`. class_weight fp32 [C] on the device (NULL = all ones; read at every launch, so a CUDA graph sees in-place
 * edits), gamma finite and >= 0. Per valid pixel (target != ignore_index, 0 <= target < C), with p = softmax(v),
 * q = 1 - p_t and nll = -log p_t:
 *   l = w_t q^gamma nll,   loss = sum over valid pixels of l / n_valid   (the pixel count, not sum w_t),
 *   dl/dv_c = w_t M (p_c - [c = t]),   M = q^gamma + gamma p_t q^(gamma-1) nll,
 * with torch.pow's 0^0 = 1 (at q = 0: l = 0, M = 1 when gamma = 0 and 0 otherwise); loss 0 and an exactly zero gradient
 * when no pixel is valid. q = (sum_{c != t} e_c) / (sum_c e_c), so it keeps its relative accuracy as p_t -> 1. The
 * backward's staged rows take 12 bytes per pixel: the Dice width limit, Wo <= 229376 / (12 zoom), 2389 at zoom 8.
 *   fwd: loss_out[0] = loss, loss_out[1] = n_valid; argmax (or NULL) and lse as the zoom forward's (the same bits);
 *        mod fp32 [N,Ho,Wo] = w_t M per pixel, 0 where the pixel is not valid (kept for the backward); workspace:
 *        semseg_upsample_ce_focal_workspace_floats() floats (the zoom forward's).
 *   bwd: dlogits fp32 [N,h,w,C] = grad_out[0] * dloss/dlogits from the forward's lse, mod and loss_out; workspace:
 *        semseg_upsample_ce_focal_bwd_workspace_floats() floats (the zoom backward's).
 * Both reject a bad shape, zoom, gamma, width, alignment or null output before any CUDA call. */
long long semseg_upsample_ce_focal_workspace_floats(int N, int Ho, int Wo, int zoom);
int semseg_upsample_ce_focal_fwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                                 int Ho, int Wo, int zoom, int ignore_index, const float* class_weight, float gamma,
                                 float* workspace, float* loss_out, int64_t* argmax, float* lse, float* mod,
                                 void* stream);
long long semseg_upsample_ce_focal_bwd_workspace_floats(int N, int Ho, int w, int C, int zoom);
int semseg_upsample_ce_focal_bwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                                 int Ho, int Wo, int zoom, int ignore_index, const float* lse, const float* mod,
                                 const float* loss_info, const float* grad_out, float* workspace, float* dlogits,
                                 void* stream);
/* Boundary label relaxation (Zhu et al., CVPR 2019; semseg_b200/losses.py BoundaryRelaxationLoss) on the same fused
 * upsample at zoom `zoom`. class_weight fp32 [C] on the device (NULL = all ones; read at every launch), border in
 * [0, 4]. A label is valid when it is != ignore_index and in [0, C). For a valid pixel i, S_i is the set of valid labels
 * in the (2 border + 1)^2 window of the target centred on i, clipped to the image; with p = softmax(v):
 *   l_i = -log sum_{c in S_i} p_c,   omega_i = (1/|S_i|) sum_{c in S_i} w_c,   loss = sum_i omega_i l_i / D,
 *   D = sum_i omega_i,   dl_i/dv_c = p_c - [c in S_i] p_c / (1 - R_i),   R_i = sum_{c not in S_i} p_c,
 * loss 0 and an exactly zero gradient when D = 0. l_i is taken as log1p(e_R / e_S) from the two sums of exp and keeps
 * its relative accuracy when small; it and its gradient are exactly 0 when S_i holds every class. The backward's
 * staged rows take 12 bytes per pixel: the Dice width limit, Wo <= 229376 / (12 zoom), 2389 at zoom 8.
 *   fwd: loss_out[0] = loss, loss_out[1] = D; argmax (or NULL) and lse as the zoom forward's (the same bits); sets int32
 *        [semseg_upsample_ce_relax_sets_words()] = each pixel's label set (tag, omega, mask words) and lq fp32
 *        [N,Ho,Wo] = log2(R / (1 - R)) per valid pixel, both kept for the backward; workspace:
 *        semseg_upsample_ce_relax_workspace_floats() floats (the zoom forward's).
 *   bwd: dlogits fp32 [N,h,w,C] = grad_out[0] * dloss/dlogits from the forward's lse, sets, lq and loss_out; workspace:
 *        semseg_upsample_ce_relax_bwd_workspace_floats() floats (the zoom backward's).
 * Both reject a bad shape, zoom, border, width, alignment or null pointer before any CUDA call; sets_words returns -1
 * for a bad size. No host synchronisation (graph-capturable), no float atomics: deterministic. */
long long semseg_upsample_ce_relax_workspace_floats(int N, int Ho, int Wo, int zoom);
long long semseg_upsample_ce_relax_sets_words(int N, int Ho, int Wo, int C);
int semseg_upsample_ce_relax_fwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                                 int Ho, int Wo, int zoom, int ignore_index, int border, const float* class_weight,
                                 float* workspace, float* loss_out, int64_t* argmax, float* lse, int32_t* sets,
                                 float* lq, void* stream);
long long semseg_upsample_ce_relax_bwd_workspace_floats(int N, int Ho, int w, int C, int zoom);
int semseg_upsample_ce_relax_bwd(const float* logits, int pitch, int N, int h, int w, int C, int Ho, int Wo, int zoom,
                                 const float* lse, const int32_t* sets, const float* lq, const float* loss_info,
                                 const float* grad_out, float* workspace, float* dlogits, void* stream);
/* The SegPGD attack loss (Gu et al., ECCV 2022; semseg_b200/adversarial.py) on the same fused upsample at zoom `zoom`.
 * Per valid pixel j (target != ignore_index, 0 <= target < C), with pred_j the first-maximum argmax of the upsampled
 * logits computed in the same pass and nll_j = lse_j - v_{j,target} (the plain forward's bits):
 *   w_j = (1 - lambda) if pred_j == target_j else lambda,   loss = sum_j w_j nll_j / n_valid,
 * the weights constants (no gradient through the argmax); loss 0 and an exactly zero gradient when no pixel is valid.
 * lambda finite in [0, 1] (the attack's lambda_t = (t - 1) / (2T) at iteration t = 1..T).
 *   fwd: loss_out[0] = loss, loss_out[1] = n_valid; argmax (or NULL) and lse as the zoom forward's (the same bits);
 *        mod fp32 [N,Ho,Wo] = w_j, 0 where the pixel is not valid; workspace: semseg_upsample_ce_zoom_workspace_floats()
 *        floats.
 *   bwd: semseg_upsample_ce_focal_bwd(logits, ..., lse, mod, loss_out, ...) gives grad_out[0] * dloss/dlogits
 *        = grad_out[0] sum_j w_j (p_c - [c = target_j]) / n_valid.
 * Wo has the focal width limit (2389 at zoom 8). A bad shape, zoom, lambda, width, alignment or null pointer is rejected
 * before any CUDA call. */
int semseg_upsample_segpgd_fwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                               int Ho, int Wo, int zoom, int ignore_index, float lambda, float* workspace,
                               float* loss_out, int64_t* argmax, float* lse, float* mod, void* stream);
/* Lovász-Softmax loss (Berman et al., CVPR 2018), alone or plus cross-entropy (semseg_b200/losses.py
 * LovaszSoftmaxLoss), on the same fused upsample at zoom `zoom`. p = softmax(v) as the Dice passes compute it. A segment
 * is one class over every valid pixel of the call (per_image = 0, S = C segments of L = N*Ho*Wo pixels) or one (image,
 * class) pair (per_image = 1, S = N*C, L = Ho*Wo). Per segment, fg_i = [t_i = c], e_i = |fg_i - p_ic| (fp32),
 * G = sum fg_i, the valid pixels sorted by e descending with ties by flat pixel index n*Ho*Wo + y*Wo + x ascending:
 *   J_k = 1 - (G - A_k) / (G + B_k)  (A_k, B_k: fg / bg pixels among the first k; integer counts, fp64 J),  J_0 = 0
 *   loss_seg = sum_k e_(k) (J_k - J_{k-1})
 * classes_all = 0 ('present') averages over the segments with G > 0, classes_all = 1 over every segment of a scope
 * (call or image) with a valid pixel; per_image averages the images' means over all N images. Plus ce_weight * CE (the
 * mean over the call's valid pixels); loss 0 and an exactly zero gradient when no pixel is valid. The gradient holds the
 * sort order fixed: gamma_ic = w_seg g_k sign(p_ic - fg_i) (sign(0) = 0),
 *   dL/dv_ic = p_ic (gamma_ic - sum_c' p_ic' gamma_ic') + (ce_weight / n_valid) (p_ic - fg_i).
 * Wo has the Dice limit (2389 at zoom 8) and N*Ho*Wo < 2^31; a bad shape, option or width is rejected before any launch.
 *   fwd: loss_out[0] = loss, loss_out[1] = number of valid pixels; argmax (or NULL) and lse as the zoom forward's
 *        (the same bits); gamma fp32 [N*Ho*Wo*C + 2] = w_seg g_k per pixel and class ([pixel][class], unsigned: the
 *        backward applies the sign), then ce_weight / n_valid and 1; keep it for the backward.
 *        workspace: semseg_upsample_ce_lovasz_workspace_floats() floats, 8-byte aligned, about (16 S L + 1 KB * S *
 *        ceil(L / 4096)) bytes. After the call its words [0, S*L) hold each considered segment's sorted keys
 *        (0x7FFFFFFF - bits(e), 0xFFFFFFFF for invalid pixels, which sort last) and [S*L, 2*S*L) their payloads
 *        ((pixel index << 1) | fg); the segments of skipped (not considered) scopes are not written.
 *   bwd: dlogits fp32 [N,h,w,C] = grad_out[0] * dloss/dlogits from the forward's lse and gamma; workspace:
 *        semseg_upsample_ce_lovasz_bwd_workspace_floats() floats.
 * The workspace functions return -1 for a bad zoom, size or per_image. */
long long semseg_upsample_ce_lovasz_workspace_floats(int N, int Ho, int Wo, int C, int zoom, int per_image);
int semseg_upsample_ce_lovasz_fwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                                  int Ho, int Wo, int zoom, int ignore_index, int classes_all, int per_image,
                                  float ce_weight, float* workspace, float* loss_out, int64_t* argmax, float* lse,
                                  float* gamma, void* stream);
long long semseg_upsample_ce_lovasz_bwd_workspace_floats(int N, int Ho, int Wo, int w, int C, int zoom);
int semseg_upsample_ce_lovasz_bwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                                  int Ho, int Wo, int zoom, int ignore_index, const float* lse, const float* gamma,
                                  const float* grad_out, float* workspace, float* dlogits, void* stream);
/* Pixel-wise knowledge distillation (semseg_b200/losses.py DistillationLoss) on the same fused upsample at zoom `zoom`:
 * student and teacher are fp32 NHWC [N,h,w,C] maps, each with its own pitch (>= C), both upsampled as the zoom forward
 * upsamples (zoom 1: the maps themselves). With T = temperature > 0, p = softmax(s/T), q = softmax(t/T) per output pixel
 * and P = N*Ho*Wo (every pixel; there is no target):
 *   KL = (1/P) sum_pix sum_c q_c (log q_c - log p_c),  log p_c = (s_c - max s)/T - log sum_c' exp((s_c' - max s)/T)
 * so s = t gives a KL and a gradient of exactly 0. The backward stages 8 bytes per pixel: Wo <= 2560 at zoom 8.
 *   fwd: kl_out[0] = KL, kl_out[1] = P; lse fp32 [N,Ho,Wo,2] = (lse(s/T), lse(t/T)) per pixel, keep it for the backward;
 *        workspace: semseg_upsample_kd_workspace_floats() floats.
 *   bwd: ADDS grad_out[0] * kd_weight * T * (p_c - q_c) / P, the gradient of kd_weight * T^2 * KL with respect to the
 *        student map, into dlogits fp32 [N,h,w,C] (dense), which the caller has filled (e.g. with the cross-entropy
 *        gradient); the teacher gets no gradient. workspace: semseg_upsample_kd_bwd_workspace_floats() floats.
 * Both reject a bad shape, zoom, temperature, kd_weight, pitch, width or null pointer before any CUDA call; the workspace
 * functions return -1 for a zoom outside {1, 2, 4, 8} or a bad size. No host synchronisation (graph-capturable), no
 * atomics: deterministic. */
long long semseg_upsample_kd_workspace_floats(int N, int Ho, int Wo, int zoom);
int semseg_upsample_kd_fwd(const float* student, int pitch_s, const float* teacher, int pitch_t, int N, int h, int w,
                           int C, int Ho, int Wo, int zoom, float temperature, float* workspace, float* kl_out,
                           float* lse, void* stream);
long long semseg_upsample_kd_bwd_workspace_floats(int N, int Ho, int w, int C, int zoom);
int semseg_upsample_kd_bwd(const float* student, int pitch_s, const float* teacher, int pitch_t, int N, int h, int w,
                           int C, int Ho, int Wo, int zoom, float temperature, float kd_weight, const float* lse,
                           const float* grad_out, float* workspace, float* dlogits, void* stream);
/* Class-incremental training (MiB, Cermelli et al., CVPR 2020; semseg_b200/losses.py IncrementalLoss) on the same fused
 * upsample at zoom `zoom`: a student of C classes, the previous step's network (the teacher) of C_old, 2 <= C_old < C
 * <= 256. Class 0 is the background, [0, C_old) the old classes, [C_old, C) the new ones; lse_A(x) = log sum_{c in A}
 * exp(x_c), each subset's sum against its own maximum (a confident new-class pixel labelled background gives a large
 * finite loss). Both backward rows kernels stage 12 bytes per pixel: the Dice width limit, Wo <= 2389 at zoom 8.
 * Unbiased cross-entropy, per valid pixel (target != ignore_index, 0 <= target < C):
 *   l = lse_all(s) - lse_old(s) for target < C_old (old labels count as background), lse_all(s) - s_target otherwise;
 *   loss = mean over the valid pixels (0 with a zero gradient when there is none);
 *   dl/ds_c = p_c - [target < C_old][c < C_old] exp(s_c - lse_old) - [target >= C_old][c = target].
 *   fwd: loss_out[0] = loss, loss_out[1] = n_valid; argmax (or NULL) over all C classes and lse as the zoom forward's;
 *        lse_old fp32 [N,Ho,Wo] = lse_old(s) per pixel (keep both for the backward); workspace:
 *        semseg_upsample_ce_unbiased_workspace_floats() floats.
 *   bwd: dlogits fp32 [N,h,w,C] = grad_out[0] * dloss/dlogits; workspace: semseg_upsample_ce_unbiased_bwd_workspace_floats().
 * Unbiased distillation: the teacher is an fp32 NHWC [N,h,w,C_old] map with its own pitch (>= C_old), upsampled as the
 * student. With q = softmax(alpha t) over the C_old classes (alpha finite and > 0), B = {0} u [C_old, C), per pixel
 * (every pixel, no target):
 *   k = -(1/C_old) [ q_0 (lse_B(s) - lse_all(s)) + sum_{c=1}^{C_old-1} q_c (s_c - lse_all(s)) ],  KD = mean of k over the
 *   P = N*Ho*Wo pixels;  dKD/ds_c = (p_c - q_0 exp(s_c - lse_B)) / (C_old P) for c in B, (p_c - q_c) / (C_old P) else.
 *   fwd: loss_out[0] = KD, loss_out[1] = P; lse fp32 [N,Ho,Wo,3] = (lse_all(s), lse_B(s), lse(alpha t)) per pixel, keep
 *        it for the backward; workspace: semseg_upsample_unkd_workspace_floats() floats.
 *   bwd: ADDS grad_out[0] * kd_weight * dKD/ds into dlogits fp32 [N,h,w,C] (dense), which the caller has filled (with the
 *        unbiased cross-entropy gradient); the teacher gets no gradient. workspace:
 *        semseg_upsample_unkd_bwd_workspace_floats() floats.
 * All four reject a bad shape, zoom, C_old, alpha, kd_weight, pitch, width or null pointer before any CUDA call; the
 * workspace functions return -1 for a zoom outside {1, 2, 4, 8} or a bad size. No host synchronisation
 * (graph-capturable), no atomics: deterministic. */
long long semseg_upsample_ce_unbiased_workspace_floats(int N, int Ho, int Wo, int zoom);
int semseg_upsample_ce_unbiased_fwd(const float* logits, int pitch, int N, int h, int w, int C, int C_old,
                                    const int64_t* target, int Ho, int Wo, int zoom, int ignore_index, float* workspace,
                                    float* loss_out, int64_t* argmax, float* lse, float* lse_old, void* stream);
long long semseg_upsample_ce_unbiased_bwd_workspace_floats(int N, int Ho, int w, int C, int zoom);
int semseg_upsample_ce_unbiased_bwd(const float* logits, int pitch, int N, int h, int w, int C, int C_old,
                                    const int64_t* target, int Ho, int Wo, int zoom, int ignore_index, const float* lse,
                                    const float* lse_old, const float* loss_info, const float* grad_out,
                                    float* workspace, float* dlogits, void* stream);
long long semseg_upsample_unkd_workspace_floats(int N, int Ho, int Wo, int zoom);
int semseg_upsample_unkd_fwd(const float* student, int pitch_s, const float* teacher, int pitch_t, int N, int h, int w,
                             int C, int C_old, int Ho, int Wo, int zoom, float alpha, float* workspace, float* loss_out,
                             float* lse, void* stream);
long long semseg_upsample_unkd_bwd_workspace_floats(int N, int Ho, int w, int C, int zoom);
int semseg_upsample_unkd_bwd(const float* student, int pitch_s, const float* teacher, int pitch_t, int N, int h, int w,
                             int C, int C_old, int Ho, int Wo, int zoom, float alpha, float kd_weight, const float* lse,
                             const float* grad_out, float* workspace, float* dlogits, void* stream);
/* Cross-image relational distillation (semseg_b200/losses.py DistillationLoss relation_weight; CIRKD's mini-batch
 * pixel-to-pixel term). Features are NHWC bf16 [B,h,w,C] activations (lo == NULL: plain; else the split form), C = 512.
 *   nodes:     node (a,b) of image n max-pools rows [p a, min(p a + p, h)) x columns [p b, min(p b + p, w)) per channel
 *              (max_pool2d(p, p, ceil_mode=True)); M = ceil(h/p) ceil(w/p), 1 <= p <= 16. Each node is divided by its
 *              fp32 L2 norm (Sigma x^2 in a fixed order); a node with norm < 1e-12 is the zero vector. Written as the bf16
 *              operand nodes [B,M,512] (dense, 16-byte aligned), plus nodes_lo (bf16(v - hi)) when non-NULL. With argmax
 *              (uint8 [B,M,512], 16-byte aligned) and inv_norm (fp32 [B,M]) it also saves the window offset
 *              (row-major, first maximum) of every (node, channel) maximum and 1/|x| (0 for a zero node).
 *   kl_fwd:    with X_i, Y_i the student / teacher nodes of image i and tau = temperature > 0,
 *              S_ij = X_i X_j^T / tau, T_ij = Y_i Y_j^T / tau, P = row-softmax(S), Q = row-softmax(T),
 *              loss[0] = tau^2 / (B^2 M) sum_{i,j} sum_rows KL(Q_ij,row || P_ij,row)     (all ordered pairs)
 *              lse fp32 [B,B,M,2] = (lse of the row of S_ij, of T_ij) per (i, j, row): keep it for the backward.
 *              workspace: semseg_relation_workspace_floats(B, M) floats, 8-byte aligned. Both node sets share one form.
 *   kl_bwd:    dnodes fp32 [B,M,512] = grad_out[0] d loss / d X (the student nodes; the teacher gets none), written.
 *   nodes_bwd: dfeat [B,h,w,512] (its own form and pitch) = the gradient of the features through the normalisation and
 *              the saved maxima; every element is written (zero off the maxima and for zero nodes).
 * Every entry point rejects a null pointer, a bad shape, C != 512, a pool outside [1, 16], a bad temperature, a pitch
 * that is not a multiple of 8 or below C, or a misaligned pointer before any CUDA call. No host synchronisation
 * (graph-capturable), no atomics: deterministic. semseg_relation_workspace_floats returns -1 for a bad size. */
int semseg_relation_nodes(const void* feat, const void* feat_lo, int pitch, int B, int h, int w, int C, int pool,
                          void* nodes, void* nodes_lo, unsigned char* argmax, float* inv_norm, void* stream);
long long semseg_relation_workspace_floats(int B, int M);
int semseg_relation_kl_fwd(const void* xs, const void* xs_lo, const void* xt, const void* xt_lo, int B, int M, int C,
                           float temperature, float* workspace, float* lse, float* loss, void* stream);
int semseg_relation_kl_bwd(const void* xs, const void* xs_lo, const void* xt, const void* xt_lo, int B, int M, int C,
                           float temperature, const float* lse, const float* grad_out, float* dnodes, void* stream);
int semseg_relation_nodes_bwd(const void* feat, const void* feat_lo, int pitch, int B, int h, int w, int C, int pool,
                              const unsigned char* argmax, const float* inv_norm, const float* dnodes, void* dfeat,
                              void* dfeat_lo, int dfeat_pitch, void* stream);
/* Confidence-masked pseudo-label cross-entropy (semseg_b200/losses.py PseudoLabelLoss) on the same fused upsample at
 * zoom `zoom`: student and teacher fp32 NHWC [N,h,w,C] maps, each with its own pitch (>= C), both upsampled as the zoom
 * forward upsamples. Per output pixel, L = {0 <= target < C, target != ignore_index}, U = {target == ignore_index},
 * yhat = argmax_c t_c (first maximum), conf = 1 / sum_c exp(t_c - t_yhat):
 *   loss = ce_weight (1/|L|) sum_L (lse(s) - s_target) + pl_weight (1/|U|) sum_{U, conf >= threshold} (lse(s) - s_yhat)
 * A term whose set is empty is 0 with a zero gradient; other out-of-range targets belong to neither set. threshold is
 * any finite float (<= 0: every U pixel, > 1: none), pl_weight / ce_weight finite and >= 0.
 *   fwd: loss_out fp32 [6] = (CE mean over L, |L|, PL sum / |U|, |U|, 0, 1), so loss = ce_weight loss_out[0] +
 *        pl_weight loss_out[2]; argmax (or NULL) and lse as the zoom forward's (the same bits); eff_target int64
 *        [N,Ho,Wo] = target on L, yhat on confident U, -1 elsewhere; weight fp32 [N,Ho,Wo] = ce_weight/|L| on L,
 *        pl_weight/|U| on confident U, 0 elsewhere. workspace: semseg_upsample_pl_workspace_floats() floats, 8-byte
 *        aligned.
 *   bwd: semseg_upsample_ce_focal_bwd(student, ..., eff_target, ..., ignore_index = -1, lse, mod = weight,
 *        loss_info = loss_out + 4, ...) gives grad_out[0] * dloss/dstudent = sum_p weight_p (p_c - [c = eff_p]).
 * Wo has the Dice limit (2389 at zoom 8). A bad shape, zoom, pitch, option, width, alignment or null pointer is rejected
 * before any CUDA call; the workspace function returns -1 for a bad zoom or size. No host synchronisation; the counts
 * are integer atomics and the sums fixed-order: deterministic. */
long long semseg_upsample_pl_workspace_floats(int N, int Ho, int Wo, int zoom);
int semseg_upsample_pl_fwd(const float* student, int pitch_s, const float* teacher, int pitch_t, int N, int h, int w,
                           int C, const int64_t* target, int Ho, int Wo, int zoom, int ignore_index, float threshold,
                           float pl_weight, float ce_weight, float* workspace, float* loss_out, int64_t* argmax,
                           float* lse, int64_t* eff_target, float* weight, void* stream);
/* The mixed form (CutMix / ClassMix, semseg_b200/losses.py MixPseudoLabelLoss): semseg_upsample_pl_fwd with the teacher
 * of each output pixel (n, i, j) taken from image n's map or its partner (n + 1) mod N's, as mix_mask uint8
 * [N, 8(h-1)+1, 8(w-1)+1] (semseg_mix_apply's mask on the input grid) says at input pixel (i 8/zoom, j 8/zoom). Per
 * pixel, yhat and conf are the bits semseg_upsample_pl_fwd computes for that teacher image; target is the mixed target.
 * The same workspace, outputs, backward and checks, and a null mask is rejected. */
int semseg_upsample_pl_mix_fwd(const float* student, int pitch_s, const float* teacher, int pitch_t, int N, int h,
                               int w, int C, const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                               float threshold, float pl_weight, float ce_weight, const uint8_t* mix_mask,
                               float* workspace, float* loss_out, int64_t* argmax, float* lse, int64_t* eff_target,
                               float* weight, void* stream);
/* Entropy minimisation plus cross-entropy (TENT, ADVENT's MinEnt, entropy regularisation; semseg_b200/losses.py
 * EntropyLoss) on the same fused upsample at zoom `zoom`. Per output pixel, with s the upsampled logits,
 * L = {0 <= target < C, target != ignore_index}, U = {target == ignore_index}, p = softmax(s), lse = logsumexp(s) and
 * H = lse - sum_c p_c s_c (natural log):
 *   loss = ce_weight (1/|L|) sum_L (lse - s_target) + ent_weight (1/|U|) sum_U H
 *   dloss/ds_c = ce_weight/|L| (p_c - [c = t]) on L,   -ent_weight/|U| p_c (s_c - lse + H) = ent_weight/|U| p_c (mu - s_c)
 *   on U, with mu = sum_c p_c s_c the softmax-expected logit.
 * A term whose set is empty is 0 with an exactly zero gradient; other out-of-range targets belong to neither set. With
 * m the pixel's max (at class a), S_o = sum_{c != a} exp(s_c - m), S = 1 + S_o and D = sum_c exp(s_c - m) (s_c - m) <= 0:
 * H = log1p(S_o) - D / S (finite, >= 0 and relatively accurate however far the logits saturate) and mu = m + D / S
 * (= s_c exactly for constant logits: a zero gradient).
 *   fwd: loss_out fp32 [6] = (CE mean over L, |L|, H mean over U, |U|, 0, 1), so loss = ce_weight loss_out[0] +
 *        ent_weight loss_out[2]; argmax (or NULL) and lse as the zoom forward's (the same bits); mu fp32 [N,Ho,Wo] per
 *        pixel (kept for the backward); workspace: semseg_upsample_ce_entropy_workspace_floats() floats.
 *   bwd: dlogits fp32 [N,h,w,C] = grad_out[0] * dloss/dlogits from the forward's lse, mu and loss_out (|L|, |U|);
 *        ent_weight / ce_weight finite and >= 0; workspace: semseg_upsample_ce_entropy_bwd_workspace_floats() floats.
 * The backward's staged rows take 12 bytes per pixel: the Dice width limit, Wo <= 229376 / (12 zoom), 2389 at zoom 8;
 * both directions reject a wider target. A bad shape, zoom, pitch, weight, width, alignment or null pointer is rejected
 * before any CUDA call; the workspace functions return -1 for a bad zoom or size. No atomics, no host synchronisation:
 * deterministic. */
long long semseg_upsample_ce_entropy_workspace_floats(int N, int Ho, int Wo, int zoom);
int semseg_upsample_ce_entropy_fwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                                   int Ho, int Wo, int zoom, int ignore_index, float* workspace, float* loss_out,
                                   int64_t* argmax, float* lse, float* mu, void* stream);
long long semseg_upsample_ce_entropy_bwd_workspace_floats(int N, int Ho, int w, int C, int zoom);
int semseg_upsample_ce_entropy_bwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                                   int Ho, int Wo, int zoom, int ignore_index, float ent_weight, float ce_weight,
                                   const float* lse, const float* mu, const float* loss_info, const float* grad_out,
                                   float* workspace, float* dlogits, void* stream);
/* Gated CRF loss (Obukhov et al., 2019; semseg_b200/losses.py GatedCRFLoss), the pairwise term, on the loss grid
 * Hg x Wg = zoom (h-1)+1 x zoom (w-1)+1 of the fp32 NHWC logits [N,h,w,pitch] (zoom 1: the logits grid itself; zoom
 * > 1: the tail's bilinear xZ upsample, align_corners). The image is fp32 NCHW [N,3,H,W], normalised as
 * (rgb255 - mean) / std, with H = istride (Hg-1)+1 and W = istride (Wg-1)+1: grid pixel (y, x) takes its colour
 * rgb = (image[.., istride y, istride x] std + mean) / 255. With p_i = softmax over the classes at grid pixel i,
 * W(i) the (2 radius+1)^2 window around i without i and without pixels outside the grid, and positions in grid units:
 *   k_ij = exp(-|pos_i - pos_j|^2 / (2 sigma_xy^2) - |rgb_i - rgb_j|^2 / (2 sigma_rgb^2))
 *   G_ic = sum_{j in W(i)} k_ij p_jc,   S_i = sum_c p_ic G_ic,   CRF = (1/P) sum_i sum_{j in W(i)} k_ij (1 - p_i.p_j)
 *   dCRF/ds_ic = -(2/P) p_ic (G_ic - S_i),   P = N Hg Wg.
 *   fwd: lse fp32 [N,Hg,Wg], the per-pixel logsumexp on the grid: the zoom forward's lse (input), or, with compute_lse
 *        (zoom 1 only), written here; s_out fp32 [N,Hg,Wg] = S (kept for the backward); loss_out fp32 [2] = (CRF, P)
 *        through the tail's fp64 reduce; workspace: semseg_gated_crf_workspace_floats() floats (2 per 16x16 tile).
 *   bwd: ADDS grad_out[0] * crf_weight * dCRF/dlogits into dlogits fp32 [N,h,w,C] (written before, e.g. by the
 *        cross-entropy backward); workspace: semseg_gated_crf_bwd_workspace_floats() floats, 0 at zoom 1, else
 *        N C Wg (Hg + h): the per-class output-resolution terms [N,Hg,Wg,C] and their row adjoint [N,h,Wg,C] (21
 *        classes at 16 x 473^2, zoom 8: 0.34 GB; 150 classes: 2.4 GB).
 * Limits: C <= 256, radius in [1, 8], sigmas finite and > 0, mean finite, std finite and > 0, crf_weight finite and
 * >= 0, Hg <= 65535 * 16; any grid width. A bad argument is rejected before any CUDA call; the workspace functions return
 * -1 for a bad zoom or size. No atomics, no host synchronisation: deterministic, and graph-capturable. */
long long semseg_gated_crf_workspace_floats(int N, int h, int w, int zoom);
int semseg_gated_crf_fwd(const float* logits, int pitch, int N, int h, int w, int C, int zoom, float* lse,
                         int compute_lse, const float* image, int H, int W, int istride, int radius, float sigma_xy,
                         float sigma_rgb, float mean0, float mean1, float mean2, float std0, float std1, float std2,
                         float* workspace, float* s_out, float* loss_out, void* stream);
long long semseg_gated_crf_bwd_workspace_floats(int N, int h, int w, int C, int zoom);
int semseg_gated_crf_bwd(const float* logits, int pitch, int N, int h, int w, int C, int zoom, const float* lse,
                         const float* image, int H, int W, int istride, int radius, float sigma_xy, float sigma_rgb,
                         float mean0, float mean1, float mean2, float std0, float std1, float std2, const float* s_in,
                         float crf_weight, const float* grad_out, float* workspace, float* dlogits, void* stream);
/* Active Boundary Loss (Wang et al., AAAI 2022; semseg_b200/losses.py ActiveBoundaryLoss), the boundary term, on the
 * loss grid Hg x Wg = zoom (h-1)+1 x zoom (w-1)+1 of the fp32 NHWC logits [N,h,w,pitch] (zoom 1: the logits grid
 * itself; zoom > 1: the tail's bilinear xZ upsample, align_corners), with the target int64 [N,Hg,Wg]. Per image, with
 * p = softmax of the grid logits s and KL(a|b) = sum_c a_c (log a_c - log b_c):
 *   GT boundary: t(y,x) != t(y+1,x), t(y,x) != t(y,x+1) or t(y,x) == ignore_index;
 *   D = fp32(max(sqrt(e) - 1, 0)), e the exact squared distance to the image's nearest GT-boundary pixel (+inf on an
 *     image without one: it selects nothing);
 *   k(y,x) = KL(p_yx | p_y+1,x) + KL(p_yx | p_y,x+1) (0 past the last row / column); t_0 = 1e-5, t_j+1 = 1.2 t_j in
 *     fp64, compared as fp32; j* = the smallest j < 256 with #(k > t_j) <= max_n_ratio Hg Wg over the call (255 if
 *     none); B(p) = some pixel of p's 3x3 neighbourhood has k > t_j*;
 *   neighbours n_0..n_7 at (+1,0) (-1,0) (0,-1) (0,+1) (-1,+1) (+1,+1) (-1,-1) (+1,-1), 8 = p itself; dir(p) = the
 *     first argmin of D over the nine (out-of-image: +inf); p is selected if B(p), dir != 8 and D(p) is finite;
 *   z_j = KL(p_nj | p) (an out-of-image n_j replicates the edge), y_dir = 1 - label_smoothing, y_j = label_smoothing
 *     / 8 elsewhere, l = -sum_j y_j log softmax(z)_j, w = min(D, max_clip_dist) / max_clip_dist;
 *   ABL = (1/M) sum over the M selected pixels of w l (0 when M = 0); dz_j/ds_p,c = p_c - p_nj,c (n_j detached).
 *   fwd: lse fp32 [N,Hg,Wg], the grid's per-pixel logsumexp (the zoom forward's); state: semseg_abl_workspace_floats
 *        (pass 0) floats, kept for the backward, P = N Hg Wg, in 4-byte words: D fp32 [P] at 0, k fp32 [P] at P, w dl/dz
 *        fp32 [P][8] at 2P (written for the selected pixels), code uint8 [P] at 10P (dir | B << 4 | selected << 5; dir
 *        15 on an image without a GT boundary), the level histogram int32 [257] at 10P + ceil(P/4), then j* int32 and
 *        the bits of t_j*, then the per-tile partials (16 x 473^2 images: 0.15 GB); loss_out fp32 [2] = (ABL, M)
 *        through the tail's fp64 reduce.
 *   bwd: ADDS grad_out[0] * abl_weight * dABL/dlogits into dlogits fp32 [N,h,w,C] (written before, e.g. by the
 *        cross-entropy backward), from the forward's lse, state and loss_out (loss_info); workspace:
 *        semseg_abl_workspace_floats (pass 1) floats, 0 at zoom 1, else N C Wg (Hg + h), the output-resolution
 *        gradient and its row adjoint (21 classes at 16 x 473^2, zoom 8: 0.34 GB; 150 classes: 2.4 GB).
 * Limits: C <= 256, N <= 65535, Hg <= 65535 * 16, max_n_ratio in [0, 1], max_clip_dist finite and > 0,
 * label_smoothing in [0, 1], abl_weight finite and >= 0. A bad argument is rejected before any CUDA call; the
 * workspace function returns -1 for a bad zoom, size or pass. The histogram counts with integer atomics; no other
 * atomics, no host synchronisation: deterministic, and graph-capturable. */
long long semseg_abl_workspace_floats(int N, int h, int w, int C, int zoom, int pass);
int semseg_abl_fwd(const float* logits, int pitch, int N, int h, int w, int C, int zoom, const float* lse,
                   const void* target_i64, long long ignore_index, double max_n_ratio, float max_clip_dist,
                   float label_smoothing, float* state, float* loss_out, void* stream);
int semseg_abl_bwd(const float* logits, int pitch, int N, int h, int w, int C, int zoom, const float* lse,
                   const float* state, const float* loss_info, float abl_weight, const float* grad_out,
                   float* workspace, float* dlogits, void* stream);
/* Mixed-sample masks and batches (csrc/mix.cu) for mean-teacher training. Image n is mixed with its partner
 * pi(n) = (n + 1) mod N; uniforms fp32 [N, ustride] hold u0 (apply), u1 (area), u2 (ratio), u3 (row), u4 (column) and,
 * for ClassMix, class priorities u[n, 5 + c]; image n is mixed iff (double) u0 < p.
 *   mix_argmax_x8: teacher fp32 NHWC [N,h,w,C] (pitch >= C, C <= 256) -> argmax uint8 [N, 8(h-1)+1, 8(w-1)+1], the
 *                  first maximum after the x8 bilinear (align_corners) upsample, bit-equal to semseg_upsample_pl_fwd's
 *                  yhat at zoom 8; present uint32 [N, 8]: the classes that occur in each image's argmax, as bits.
 *   mix_select   : selected uint32 [N, 8] = the ceil(k/2) of each image's k present classes with the smallest
 *                  (u[n, 5 + c], c), lexicographically (ustride >= 5 + C).
 *   mix_apply    : M (mask uint8 [N,H,W], 1 = from the partner), x_mixed fp32 NCHW [N,Cin,H,W] = M ? x[pi(n)] : x[n],
 *                  y_mixed int64 [N,Ho,Wo] = y[pi(n)] where M at input pixel (i 8/zoom, j 8/zoom), else y[n]
 *                  (H-1, W-1 multiples of 8, Ho = zoom(H-1)/8 + 1). M = 0 on an image that is not mixed; else
 *                  SEMSEG_MIX_CUTMIX: M = 1 on rows [y0, y0+bh) and columns [x0, x0+bw), in fp64 with every operation
 *                    correctly rounded: a = ((area_lo + (area_hi - area_lo) u1) H) W, rho = ratio_lo + (ratio_hi -
 *                    ratio_lo) u2, bw = min(W, max(1, floor(sqrt(a / rho)))), bh = min(H, max(1, floor(sqrt(a rho)))),
 *                    x0 = min(W - bw, floor(u4 (W - bw + 1))), y0 = min(H - bh, floor(u3 (H - bh + 1)));
 *                  SEMSEG_MIX_CLASSMIX: M = 1 where argmax[pi(n)] is in selected[pi(n)].
 *                  p in [0, 1], 0 < area_lo <= area_hi <= 1, 0 < ratio_lo <= ratio_hi; the outputs may not alias x, y.
 * Bad arguments are rejected before any CUDA call. No host synchronisation; deterministic. */
#define SEMSEG_MIX_CUTMIX 0
#define SEMSEG_MIX_CLASSMIX 1
int semseg_mix_argmax_x8(const float* teacher, int pitch, int N, int h, int w, int C, uint8_t* argmax,
                         uint32_t* present, void* stream);
int semseg_mix_select(const float* uniforms, int ustride, const uint32_t* present, int N, int C, uint32_t* selected,
                      void* stream);
int semseg_mix_apply(int mode, const float* x, int N, int Cin, int H, int W, const int64_t* y, int Ho, int Wo, int zoom,
                     const float* uniforms, int ustride, double p, double area_lo, double area_hi, double ratio_lo,
                     double ratio_hi, const uint8_t* argmax, const uint32_t* selected, uint8_t* mask,
                     float* x_mixed, int64_t* y_mixed, void* stream);
/* The strong view of mean-teacher training (csrc/strong.cu, semseg_b200/augment.py StrongAugment): colour jitter,
 * grayscale and Gaussian blur of x fp32 NCHW [N,3,H,W] (normalised) -> out (same shape, not aliasing x). Image n uses
 * uniforms u[n, 0..11] (fp32 [N, ustride], ustride >= 12); a comparison "u < p" is made as (double) u < p. Per image:
 *   1. v = clamp((x std_c + mean_c) / 255, 0, 1) in fp32. This and every later step run only when at least one operation
 *      below applies; an image with none applied is copied bit for bit.
 *   2. Colour jitter iff u0 < p_jitter. Factors in fp64, rounded once to fp32: brightness b = lo + (hi - lo) u1 with
 *      [lo, hi] = [max(0, 1 - B), 1 + B], contrast c by u2 and saturation s by u3 alike, hue h = -H + 2H u4. An operation
 *      of strength 0 is skipped. Order: ascending (u5..u8, index). torchvision.transforms.v2.functional's float forms:
 *      brightness clamp(b v); contrast clamp(c v + (1 - c) m), m = the image mean of gray(v) at that point of the chain;
 *      saturation clamp(s v + (1 - s) gray(v)); hue _rgb2hsv, h <- (h + hue) mod 1, _hsv2rgb.
 *      gray = 0.2989 r + 0.587 g + 0.114 b.
 *   3. Grayscale iff u9 < p_gray: every channel becomes gray(v).
 *   4. Blur iff u10 < p_blur: sigma = fp32(sigma_lo + (sigma_hi - sigma_lo) u11) (fp64, rounded once),
 *      r = min(ceil(3 sigma), ceil(3 sigma_hi)), taps exp(-k^2 / 2 sigma^2), k = -r..r, normalised; separable, with
 *      reflect-101 borders (the edge pixel is not repeated): torchvision's gaussian_blur(v, [2r+1]*2, [sigma]*2).
 *   5. out = (255 v - mean_c) / std_c.
 * workspace: N ceil(H/32) ceil(W/32) floats (per-tile partial sums of the contrast mean). Strengths finite >= 0 with
 * hue <= 0.5, probabilities in [0, 1], 0 < sigma_lo <= sigma_hi <= 5, std > 0, H and W > ceil(3 sigma_hi). Two launches,
 * fixed geometry, no atomics, deterministic, no host synchronisation. Bad arguments are rejected before any CUDA call. */
int semseg_strong_augment(const float* x, int N, int C, int H, int W, const float* uniforms, int ustride,
                          double brightness, double contrast, double saturation, double hue, double p_jitter,
                          double p_gray, double p_blur, double sigma_lo, double sigma_hi, const float* mean3,
                          const float* std3, float* workspace, float* out, void* stream);
/* Segmented stable radix sort (csrc/segsort.cu): S segments of L (uint32 key, uint32 payload) pairs, [S][L], each sorted
 * in place by key ascending, equal keys in input order. keys_alt / vals_alt: scratch of the same size. skip: NULL, or
 * int [S] on the device, a non-zero entry leaves that segment untouched. workspace:
 * semseg_segsort_u32_pairs_workspace_bytes() bytes = 1 KB * S * ceil(L / 4096). No host synchronisation, fixed launch
 * geometry (graph-capturable), deterministic. 0 < L < 2^31; the workspace function returns -1 for bad sizes. */
long long semseg_segsort_u32_pairs_workspace_bytes(int S, long long L);
int semseg_segsort_u32_pairs(unsigned* keys, unsigned* vals, unsigned* keys_alt, unsigned* vals_alt, int S,
                             long long L, const int* skip, void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Sliding-window evaluation after the network (semseg_b200/inference.py, exact=False). No tensor cores, no atomics.
 *   window_scores     : logits fp32 NHWC [G (+G mirrored crops when flip), h, w, C] (pitch >= C; with flip, images
 *                       G..2G-1 are the mirrors of 0..G-1) -> out fp32 [G, C, crop_h, crop_w] (contiguous) =
 *                       softmax over C of the x8 bilinear (align_corners=True) upsample, averaged with the mirrored
 *                       crop's scores as (p + p_mirror) * 0.5 when flip. Requires crop = 8(h-1)+1 x 8(w-1)+1 and
 *                       C <= 256. The upsampled logits are never stored.
 *   window_accumulate : scores fp32 [ny*nx, C, crop_h, crop_w] of a scale's crop grid in row-major order, crop origins
 *                       ys[ny] / xs[nx] (host arrays, at most 256 each: ascending, first 0, last full - crop, gaps <=
 *                       crop) on the padded [full_h, full_w] image -> canvas fp64 [C, img_h, img_w] = the un-padded
 *                       window at (top, left) of the fp64 sum of the covering crops' scores in grid order, divided by
 *                       their count. Every element written once; bit-identical to the sequential accumulation.
 *   window_resize_add : total fp64 [C, Ho, Wo] += bilinear resize (align_corners=False, half-pixel centres, fp64 as
 *                       ATen's upsample_bilinear2d) of canvas fp64 [C, Hi, Wi].
 */
int semseg_window_scores(const float* logits, int pitch, int G, int h, int w, int C, int flip, float* out, int crop_h,
                         int crop_w, void* stream);
int semseg_window_accumulate(const float* scores, int C, int crop_h, int crop_w, const int* ys, int ny, const int* xs,
                             int nx, int full_h, int full_w, int top, int left, int img_h, int img_w, double* canvas,
                             void* stream);
int semseg_window_resize_add(const double* canvas, int C, int Hi, int Wi, double* total, int Ho, int Wo, void* stream);
/* window_scores_stats: window_scores with the same arguments, writing out fp32 [G, C + 2, crop_h, crop_w]: channels
 * 0..C-1 bit-identical to window_scores', then ML = max_c v and LSE = max + log(sum_c exp(v - max)) of the same
 * upsampled logits v, each flip-averaged as (a + a_mirror) * 0.5 when flip. window_accumulate and window_resize_add
 * take the C + 2 channels unchanged. */
int semseg_window_scores_stats(const float* logits, int pitch, int G, int h, int w, int C, int flip, float* out,
                               int crop_h, int crop_w, void* stream);
/* window_scores_mc: Monte Carlo dropout scores. logits fp32 [T][G (+G mirrors when flip)][h][w][pitch] (T draws of one
 * batch's low-resolution logits, each draw laid out as window_scores' input) -> out fp32 [G, C + 1, crop_h, crop_w]:
 * channels 0..C-1 = (sum_t p_t) * (1/T), p_t draw t's flip-averaged scores with window_scores' arithmetic, summed in draw
 * order; channel C = the same mean of the flip-averaged sample entropy H_t = log S - sum_c q_c (v_c - max) of the
 * upsampled logits v (S = sum_c exp(v_c - max), q = the softmax). T = 1 gives score channels bit-identical to
 * window_scores'. The upsampled logits are never stored; each element of out is written once; no atomics
 * (deterministic). Same checks as window_scores, plus 1 <= T <= 128. window_accumulate and window_resize_add take the
 * C + 1 channels unchanged. */
int semseg_window_scores_mc(const float* logits, int pitch, int T, int G, int h, int w, int C, int flip, float* out,
                            int crop_h, int crop_w, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Anomaly segmentation (semseg_b200/anomaly.py; csrc/anomaly.cu). No host synchronisation, no float atomics:
 * deterministic. Bad arguments (null pointers, sizes, options) are rejected before any CUDA call; the workspace
 * queries return -1 for bad sizes.
 *   class_moments : pred int64 [P] (the argmax), ml fp64 [P] (the ML plane) -> moments fp64 [3][C] += (sum ML,
 *                   sum ML^2, pixel count) per class c = pred; predictions outside [0, C) are not counted.
 *                   workspace: class_moments_workspace_bytes(P, C) = 24 C ceil(P / 2048) bytes. 1 <= C <= 4096.
 *   sml           : standardized max-logit of one H x W image: S = (ml - mean[pred]) / std[pred] (mean, std: fp64 [C]
 *                   on the device; a prediction outside [0, C) gives NaN), then boundary_iterations Jacobi suppression
 *                   steps i at width r_i = boundary_width - i floor(boundary_width / boundary_iterations): a pixel whose
 *                   (2 r_i + 1)^2 window, clipped to the image, holds another prediction takes the mean of S over the
 *                   non-boundary pixels of its clipped 3x3 neighbourhood (kept if there are none); then
 *                   T = sum g S(p + d (a, b)) / sum g over the taps inside the image, a, b in [-k/2, k/2],
 *                   g = exp(-(a^2 + b^2) / 2 sigma^2), d = smooth_dilation; out fp32 [H, W] = -T. fp64 throughout.
 *                   1 <= smooth_kernel <= 63 odd, sigma finite > 0, dilation >= 1, boundary_width >= 1 when
 *                   boundary_iterations > 0. workspace: sml_workspace_bytes(H, W) = 40 H W bytes.
 *   metrics       : score fp32 [n], label [n] (uint8 when label_bytes = 1, int64 when 8; 1 = anomaly, 0 = inlier,
 *                   ignore_index = void) -> out fp64 [3] = (AUROC, AP, FPR95), info int64 [3] = (positives, negatives,
 *                   error bits: 1 = a label other than 0, 1, ignore_index; 2 = a non-finite score on a non-void pixel).
 *                   Non-void pixels sorted by score descending, equal scores (-0.0 = +0.0) one group g with cumulative
 *                   TP_g, FP_g: AUROC = sum_g (FP_g - FP_g-1)(TP_g-1 + TP_g) / 2PN (Mann-Whitney, ties 1/2),
 *                   AP = sum_g (TP_g - TP_g-1) / P * TP_g / (TP_g + FP_g), FPR95 = FP_g / N at the first g with
 *                   TP_g >= 0.95 P. NaN without positives or without negatives. 0 < n < 2^31.
 *                   workspace: metrics_workspace_bytes(n), about 16 n bytes.
 */
long long semseg_anomaly_class_moments_workspace_bytes(long long P, int C);
int semseg_anomaly_class_moments(const long long* pred, const double* ml, long long P, int C, void* workspace,
                                 double* moments, void* stream);
long long semseg_anomaly_sml_workspace_bytes(int H, int W);
int semseg_anomaly_sml(const double* ml, const long long* pred, int H, int W, int C, const double* mean,
                       const double* std, int boundary_width, int boundary_iterations, int smooth_kernel,
                       double smooth_sigma, int smooth_dilation, void* workspace, float* out, void* stream);
long long semseg_anomaly_metrics_workspace_bytes(long long n);
int semseg_anomaly_metrics(const float* score, const void* label, int label_bytes, long long n,
                           long long ignore_index, void* workspace, double* out, long long* info, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Dense CRF refinement of one image (Krähenbühl & Koltun 2011; semseg_b200/densecrf.py DenseCRF; csrc/densecrf.cu):
 * Potts mean field with a smoothness kernel exp(-|p_i - p_j|^2 / 2 pos_xy_std^2) (d = 2) and an appearance kernel
 * exp(-|p_i - p_j|^2 / 2 bi_xy_std^2 - |I_i - I_j|^2 / 2 bi_rgb_std^2) (d = 5), each on a permutohedral lattice and
 * symmetrically normalised: K~ v = n * K (n * v), n = (K 1 + 1e-20)^-1/2. Pixel i = y W + x has position (x, y) and
 * colour I_i = image[i][0..2], clamped to [0, 255].
 *   lattice_bytes : size of the lattice buffer of an H x W image; both lattices at their worst case V = N (d+1) plus the
 *                   build's scratch, about 700 bytes per pixel (1.5 GB at 2048 x 1024).
 *   build         : image fp32 HWC [H][W][3] -> lattice. The first two int32 of the lattice are then V_s and V_a, the
 *                   vertex counts, read back once to size the value buffers. Lattice keys pack the d stored coordinates
 *                   into 64 bits with per-coordinate widths from their range (image size and standard deviations); a
 *                   configuration that needs more than 64 bits, or a coordinate range beyond +-2^52, is rejected.
 *                   0 < H W, 6 H W < 2^31.
 *   values_floats : values workspace of meanfield / filter = 2 (V_s + V_a) C floats (two [V][C] buffers per kernel).
 *   meanfield     : prob fp32 [H W][C] (class-contiguous) -> Q fp32 [H W][C]: Q0 = softmax(log max(prob, clip)), then
 *                   `iterations` times Q <- softmax(log max(prob, clip) + pos_weight K~_s Q + bi_weight K~_a Q). A
 *                   kernel of weight 0 is skipped. FLT_MIN <= clip < 1 (the log is taken in fp32), weights finite
 *                   and >= 0, iterations >= 0.
 *   filter        : out fp32 [H W][C] = K~ in for kernel 0 (smoothness) or 1 (appearance).
 *   keys          : out int32 [V][d] = the vertex keys of kernel 0 or 1 (the first d lattice coordinates, in key order),
 *                   given the standard deviations of the build.
 * V_s / V_a passed to meanfield, filter and keys are the build's. Deterministic (no float atomics, every result
 * written once); the build reads nothing back to the host. Bad arguments (empty images, non-finite or non-positive
 * standard deviations, negative or non-finite weights, iterations < 0, clip outside [FLT_MIN, 1), key overflow, null
 * pointers) are rejected before any CUDA call.
 */
long long semseg_densecrf_lattice_bytes(int H, int W);
int semseg_densecrf_build(const float* image, int H, int W, double pos_xy_std, double bi_xy_std, double bi_rgb_std,
                          void* lattice, void* stream);
long long semseg_densecrf_values_floats(int H, int W, int Vs, int Va, int C);
int semseg_densecrf_meanfield(const void* lattice, int H, int W, int Vs, int Va, const float* prob, int C, double clip,
                              int iterations, double pos_weight, double bi_weight, float* values, float* Q,
                              void* stream);
int semseg_densecrf_filter(const void* lattice, int H, int W, int Vs, int Va, int kernel, const float* in, int C,
                           float* values, float* out, void* stream);
int semseg_densecrf_keys(const void* lattice, int H, int W, int Vs, int Va, int kernel, double pos_xy_std,
                         double bi_xy_std, double bi_rgb_std, int* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Step glue: per-class intersection / union / target areas (util/util.py:55-67, called at tool/train.py:286,375).
 *   counts int32 [3][K] (zeroed by the call): [0] = #(pred == target == k), [1] = #(pred == k) with pred forced to
 *   ignore_index where target == ignore_index, [2] = #(target == k); union = [1] + [2] - [0].
 *   write_back != 0 also stores the masked prediction (the reference masks `output` in place). 1 <= K <= 4096; n == 0
 *   (pred and target may then be null) gives zero counts.
 */
int semseg_iou_hist(void* pred_i64, const void* target_i64, long long n, int K, long long ignore_index, int write_back,
                    int* counts, void* stream);
/* Boundary IoU (Cheng et al., CVPR 2021; semseg_b200/metrics.py boundaryIoUGPU) of pred and target int64 [N,H,W]:
 *   a pixel of label c lies in its map's band if its (2d+1)^2 window holds another label or reaches outside the image
 *   (the per-class mask padded by 1 and 3x3-eroded d times, subtracted from the mask); in the target ignore_index is a
 *   label of its own. Over the pixels whose target is not ignore_index, counts int32 [3][K] (zeroed by the call):
 *   [0] = #(pred == target == k, both in band), [1] = #(pred == k in band), [2] = #(target == k in band); union =
 *   [1] + [2] - [0]. Labels outside [0, K) are not counted; labels are compared saturated to int32.
 *   workspace: 4 N H W int32 (the row-window minima and maxima of both maps). 1 <= K <= 4096, d >= 1.
 */
int semseg_boundary_iou_hist(const void* pred_i64, const void* target_i64, int N, int H, int W, int K,
                             long long ignore_index, int d, int* workspace, int* counts, void* stream);

/* ------------------------------------------------------------------------------------------------
 * torch.optim.SGD (momentum, dampening, weight decay, nesterov; tool/train.py:140,274-276) over every parameter tensor in
 * one launch. items_dev: device array sorted by chunk0 (an item's chunks are consecutive blocks of
 * semseg_sgd_chunk_elems() elements); grad_ptrs_dev: device array of n_items gradient pointers (0 = no gradient this
 * step: the parameter is skipped); hyper: per-group hyper-parameters, passed by value, with nesterov a bit mask (bit g:
 * group g uses Nesterov momentum). `first` != 0 initialises the momentum buffer with the (decayed) gradient, as torch
 * does on a parameter's first step with a gradient under a non-zero momentum. In a group whose momentum is 0 the buffer
 * is neither read nor written (it may be null), as torch leaves it.
 */
#define SEMSEG_SGD_MAX_GROUPS 16
typedef struct semseg_sgd_item {
  float* w;
  float* buf;
  long long n;
  int group;
  int chunk0;
  int first;
  int reserved;
} semseg_sgd_item;
typedef struct semseg_sgd_hyper {
  float lr[SEMSEG_SGD_MAX_GROUPS];
  float momentum[SEMSEG_SGD_MAX_GROUPS];
  float weight_decay[SEMSEG_SGD_MAX_GROUPS];
  float dampening[SEMSEG_SGD_MAX_GROUPS];
  int nesterov;
} semseg_sgd_hyper;
int semseg_sgd_chunk_elems(void);
int semseg_sgd_multi(const semseg_sgd_item* items_dev, const void* grad_ptrs_dev, int n_items, int n_chunks,
                     const semseg_sgd_hyper* hyper, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Exponential moving average of a model's weights (semseg_b200/optim.py ModelEMA) over every tensor in one launch, on
 * semseg_sgd_multi's table layout (an item's chunks are consecutive blocks of semseg_sgd_chunk_elems() elements,
 * items_dev sorted by chunk0, 8-byte aligned). kind SEMSEG_EMA_LERP_F32: shadow <- lerp(shadow, source, 1 - decay) on
 * fp32, in torch.lerp's two-branch form (weight < 0.5: e + weight (w - e); else w - (w - e) (1 - weight)), so the bits
 * equal torch._foreach_lerp_(shadow, source, 1 - decay); decay 0 copies, decay 1 leaves the shadow as it is.
 * kind SEMSEG_EMA_COPY_I64: the n int64 elements are copied (BatchNorm's num_batches_tracked). Element-wise and
 * deterministic; a null table, counts <= 0, decay outside [0, 1] or a misaligned table is rejected before any CUDA call.
 */
#define SEMSEG_EMA_LERP_F32 0
#define SEMSEG_EMA_COPY_I64 1
typedef struct semseg_ema_item {
  void* shadow;
  const void* source;
  long long n;
  int kind;
  int chunk0;
} semseg_ema_item;
int semseg_ema_multi(const semseg_ema_item* items_dev, int n_items, int n_chunks, double decay, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Training-batch augmentation: tool/train.py:194-201's RandScale -> RandRotate -> RandomGaussianBlur ->
 * RandomHorizontalFlip -> Crop -> ToTensor -> Normalize (util/transform.py) with the parameters drawn on the host, in
 * ONE launch over decoded uint8 images. `data` holds every sample's uint8 RGB HWC image and uint8 HW label at the byte
 * offsets of its descriptor. Per output pixel: crop/pad -> flip -> 5x5 Gaussian (reflect-101 at the rotated image's
 * edges) -> cv2's fixed-point warpAffine (AB_BITS 10, border = mean / ignore_label) -> cv2's resize (INTER_LINEAR image,
 * INTER_NEAREST label) of the source; a stage whose flag is off (or rh,rw == h,w for the resize) is skipped. Nothing at
 * resized or rotated resolution is written. Outputs: out_img fp32 [N,3,crop_h,crop_w] = (v - mean[c]) / std[c],
 * out_lab int64 [N,crop_h,crop_w]. desc_host (validated before any CUDA call) and desc_dev hold the same n entries.
 * Validation mode is the same call with every stage off and centred offsets.
 */
typedef struct semseg_augment_desc {
  long long img_off;   /* byte offset of the uint8 RGB HWC image in data */
  long long lab_off;   /* byte offset of the uint8 HW label in data */
  int h, w;            /* source size */
  int rh, rw;          /* resized size; equal to (h, w) = cv2's copy, no interpolation */
  double scale_y;      /* 1 / fy: source step per resized pixel (cv2's scale_y) */
  double scale_x;      /* 1 / fx */
  double m[6];         /* inverse affine map resized <- rotated, row-major 2x3 (cv2.invertAffineTransform) */
  int rotate, blur, flip;
  int pad_top, pad_left;   /* leading padding: max(crop - resized, 0) / 2 */
  int off_y, off_x;        /* crop offsets in the padded frame */
  int reserved;
} semseg_augment_desc;
int semseg_augment(const void* data, long long data_bytes, const semseg_augment_desc* desc_host,
                   const semseg_augment_desc* desc_dev, int n, int crop_h, int crop_w, const float* mean3,
                   const float* std3, int ignore_label, float* out_img, long long* out_lab, void* stream);

/* ------------------------------------------------------------------------------------------------
 * L-infinity PGD / SegPGD attack steps (semseg_b200/adversarial.py) on the network's fp32 NCHW input [N,3,H,W] in the
 * normalised space it sees. Per channel c, from the attack's eps, alpha and the trainer's mean / std in 0-255 pixel
 * units, computed on the host in fp64 and rounded to fp32 once:
 *   step[c] = alpha / std_c,  eps[c] = eps / std_c,  lo[c] = (0 - mean_c) / std_c,  hi[c] = (255 - mean_c) / std_c.
 * Every operation below is one fp32 round-to-nearest in the order written, without FMA contraction, so the results are
 * bit-identical to the same formula in torch fp32 (s = sign(g) with sign(0) = 0, as torch.sign):
 *   semseg_adv_step : v = x + step s;  v = min(max(v, x0 - eps), x0 + eps);  out = min(max(v, lo), hi)
 *                     (step s is exact; out may be x: the step runs in place)
 *   semseg_adv_start: out = min(max(min(max(x0 + eps (2u - 1), x0 - eps), x0 + eps), lo), hi)
 *                     (u: uniforms in [0, 1) of the input's shape, drawn by the caller)
 * Both reject a null pointer, a tensor that is not 4-byte aligned, a bad shape (3N <= 65535) or constants that are not
 * finite, a negative step or eps, or lo > hi, before any CUDA call. */
typedef struct semseg_adv_box {
  float step[3];
  float eps[3];
  float lo[3];
  float hi[3];
} semseg_adv_box;
int semseg_adv_step(const float* x, const float* grad, const float* x0, float* out, int N, int H, int W,
                    const semseg_adv_box* box, void* stream);
int semseg_adv_start(const float* x0, const float* u, float* out, int N, int H, int W, const semseg_adv_box* box,
                     void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SEMSEG_B200_H */
