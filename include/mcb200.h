/* mcb200.h — C ABI of libmcb200.so: the H100 (sm_90a) hot path of neptune-ai/open-solution-mapping-challenge.
 *
 * The reference is 100 % Python; every FLOP of its hot path runs inside torch 0.3.1 / cuDNN / scipy / skimage /
 * pydensecrf calls.  This header is what a Python host binds (ctypes, see INTEGRATION.md) in place of those library
 * calls.  Each entry point cites the reference call site it replaces as  file:line  of the reference repository.
 *
 * Conventions
 *   - every function returns 0 on success, a negative MCB_ERR_* code on failure; mcb_last_error() returns a
 *     thread-local message (the Python layer raises RuntimeError with it, matching the reference's exceptions);
 *   - the caller owns all memory: device pointers allocated by the host framework; the library never allocates or
 *     frees device memory and keeps no pointer after returning;
 *   - all work is enqueued asynchronously on `stream` (a cudaStream_t passed as void*); no hidden synchronisation;
 *   - activations are NHWC bf16, dense; conv weights are bf16 [ky][kx][cout][cin] ("tap-major");
 *     weight gradients are fp32 in the same layout; vectors (bias, BN parameters, statistics) are fp32;
 *   - there is no CPU fallback: without a CUDA device every compute entry point fails with MCB_ERR_CUDA.
 */
#ifndef MCB200_H_
#define MCB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MCB_OK 0
#define MCB_ERR_INVALID (-1)
#define MCB_ERR_CUDA (-2)
#define MCB_ERR_UNSUPPORTED (-3)

const char* mcb_last_error(void);
int mcb_version(void);
/* zero-fill of an accumulation buffer as a memset on `stream` (gradient arena, statistic sums) */
int mcb_zero_bytes(void* p, size_t bytes, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Convolutions as wgmma implicit GEMMs (TMA-fed, register accumulators).
 * Replaces nn.Conv2d / nn.ConvTranspose2d forward + autograd backward at
 *   src/unet_models.py:21-34 (conv3x3, ConvRelu), :125-150 (DecoderBlockV2), :360-383 (encoder stages, final),
 *   torchvision/models/resnet.py BasicBlock / Bottleneck (used at src/unet_models.py:344-352).
 * ---------------------------------------------------------------------------------------------------------------- */

typedef struct {
  const void* x[2];   /* NHWC bf16 inputs; x[1] != NULL fuses torch.cat([x0, x1], 1) (src/unet_models.py:395-399) */
  int cin[2];         /* channels of x[0], x[1] (32, or multiples of 64) */
  int n, h, w;        /* input batch, height, width */
  const void* weight; /* bf16 [ksize*ksize][cout][cin0+cin1] */
  int cout;
  int ksize;          /* 1 or 3; padding = ksize / 2 */
  int stride;         /* 1 or 2 */
  const float* bias;  /* fp32 [cout] or NULL */
  int relu;           /* fuse ReLU (ConvRelu, src/unet_models.py:25-34) */
  float* stats;       /* fp32 [2*cout] or NULL: += per-channel sum / sum of squares of the stored (bf16) outputs:
                         the BatchNorm batch statistics of the layer that follows */
  void* y;            /* NHWC bf16 [n][h/stride][w/stride][cout] */
  /* inference-mode BatchNorm / residual folded into the epilogue: y = relu?(acc*scale[c] + bias[c] + residual) */
  const float* scale;   /* fp32 [cout] or NULL */
  const void* residual; /* NHWC bf16 like y, or NULL */
} mcb_conv_fwd_args;
int mcb_conv_fwd(const mcb_conv_fwd_args* a, void* stream);

typedef struct {
  const void* dy;        /* NHWC bf16 [n][h/stride][w/stride][cout] */
  int n, h, w;           /* dims of dx (the conv input) */
  const void* weight;    /* bf16 [ksize*ksize][cout][cin_total] */
  int cout, cin_total;
  int ci_off, cin;       /* dx covers weight input channels [ci_off, ci_off+cin) (one source of a fused concat) */
  int ksize, stride;
  void* dx;              /* NHWC bf16 [n][h][w][cin] */
  const void* relu_mask; /* NHWC bf16 like dx or NULL: dx is zeroed where relu_mask <= 0 (backward of the ReLU that
                            produced the conv input) */
  int accumulate;        /* dx += (TMA reduce-add) instead of dx = */
  /* optional fused backward of the conv-BatchNorm-ReLU unit whose output is this conv's input (relu_mask must then be
     NULL: the ReLU mask is that unit's own output sign, recomputed from its BatchNorm input bn_z exactly as the
     forward did):   y = fma(bn_z, bn_gamma*bn_invstd, bn_beta - bn_mean*bn_gamma*bn_invstd);  g = dy_in * (y > 0);
     dx = g;  bn_dbeta[c] += sum g;  bn_dgamma[c] += sum g * (bn_z - bn_mean[c]) * bn_invstd[c]   (sums over the
     STORED bf16 g).  bn_z: NHWC bf16 like dx; all NULL to disable */
  const void* bn_z;
  const float* bn_mean;
  const float* bn_invstd;
  float* bn_dbeta;
  float* bn_dgamma;
  const float* bn_gamma;
  const float* bn_beta;
  float* dx_channel_sum; /* fp32 [cin] or NULL (needs relu_mask, no accumulate): += sum over pixels of the stored dx, i.e.
                            the bias gradient of the conv+bias+ReLU layer that produced this conv's input */
} mcb_conv_dgrad_args;
int mcb_conv_dgrad(const mcb_conv_dgrad_args* a, void* stream);

typedef struct {
  const void* dy;     /* NHWC bf16 [n][h/stride][w/stride][cout] */
  const void* x;      /* NHWC bf16 [n][h][w][cin] */
  int n, h, w;
  int cout, cin_total;
  int ci_off, cin;    /* x supplies weight input channels [ci_off, ci_off+cin) */
  int ksize, stride;
  float* dw;          /* fp32 [ksize*ksize][cout][cin_total], accumulated (+=); zero it first */
} mcb_conv_wgrad_args;
int mcb_conv_wgrad(const mcb_conv_wgrad_args* a, void* stream);

/* nn.ConvTranspose2d(kernel_size=4, stride=2, padding=1) (src/unet_models.py:138-139) as four sub-pixel phases, or, with
   ksize = 3, nn.ConvTranspose2d(kernel_size=3, stride=2, padding=1, output_padding=1) (the UNet11 DecoderBlock,
   src/unet_models.py:42-53); both map h x w to 2h x 2w.  ksize is the last field so that a zeroed struct (ksize 0)
   keeps meaning the 4x4 kernel */
typedef struct {
  const void* x;      /* NHWC bf16 [n][h][w][cin] */
  int n, h, w, cin;
  const void* weight; /* bf16 [ksize*ksize][cout][cin] */
  int cout;
  const float* bias;
  int relu;
  void* y;            /* NHWC bf16 [n][2h][2w][cout] */
  int ksize;          /* 3 or 4; 0 means 4 */
} mcb_convt_fwd_args;
int mcb_convt_fwd(const mcb_convt_fwd_args* a, void* stream);

typedef struct {
  const void* dy;     /* NHWC bf16 [n][2h][2w][cout] */
  int n, h, w, cin;
  const void* weight; /* bf16 [ksize*ksize][cout][cin] */
  int cout;
  void* dx;           /* NHWC bf16 [n][h][w][cin] */
  const void* relu_mask;
  int accumulate;
  float* dx_channel_sum; /* as in mcb_conv_dgrad_args */
  int ksize;          /* 3 or 4; 0 means 4 */
} mcb_convt_dgrad_args;
int mcb_convt_dgrad(const mcb_convt_dgrad_args* a, void* stream);

typedef struct {
  const void* dy;     /* NHWC bf16 [n][2h][2w][cout] */
  const void* x;      /* NHWC bf16 [n][h][w][cin] */
  int n, h, w, cin, cout;
  float* dw;          /* fp32 [ksize*ksize][cout][cin], accumulated */
  int ksize;          /* 3 or 4; 0 means 4 */
} mcb_convt_wgrad_args;
int mcb_convt_wgrad(const mcb_convt_wgrad_args* a, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * HBM-bound glue kernels of the train / inference step (16-byte vectorised NHWC bf16 passes).
 * ---------------------------------------------------------------------------------------------------------------- */

/* API-edge layout conversion: the reference hands the net NCHW fp32 (src/steps/pytorch/models.py:76-92) */
int mcb_nchw_f32_to_nhwc_bf16(const float* x, void* y, int n, int c, int h, int w, void* stream);
int mcb_nhwc_bf16_to_nchw_f32(const void* x, float* y, int n, int c, int h, int w, void* stream);

/* ResNet stem, encoder.conv1 = Conv2d(3, 64, 7, stride 2, pad 3) (src/unet_models.py:360): im2col into a
 * [n*h/2*w/2][192] bf16 matrix (k = (ky*7+kx)*3 + c, zero-padded 147 -> 192) fed to mcb_conv_fwd as a 1x1 conv.
 * The master weight is fp32 [49][64][3]; pack/unpack convert to/from the GEMM operand [64][192]. */
int mcb_stem_im2col(const float* x_nchw, void* col, int n, int h, int w, void* stream);
int mcb_stem_pack_weight(const float* w, void* w_packed, void* stream);
int mcb_stem_unpack_wgrad(const float* dw_packed, float* dw, void* stream); /* dw += */

/* VGG input conv, encoder.0 = Conv2d(3, 64, 3, padding 1) + ReLU at full resolution (src/unet_models.py:68,90 and
 * :252,256): im2col into a [n*h*w][32] bf16 matrix (k = (ky*3+kx)*3 + c for k < 27, zero for k = 27..31; pixels outside
 * the image read zero) fed to mcb_conv_fwd / mcb_conv_wgrad as a 1x1 conv.  The master weight is fp32 [9][64][3];
 * pack/unpack convert to/from the GEMM operand [64][32].  No data gradient: the input is the image. */
int mcb_vgg_input_im2col(const float* x_nchw, void* col, int n, int h, int w, void* stream);
int mcb_vgg_input_pack_weight(const float* w, void* w_packed, void* stream);
int mcb_vgg_input_unpack_wgrad(const float* dw_packed, float* dw, void* stream); /* dw += */

/* nn.BatchNorm2d (eps 1e-5, momentum 0.1; torchvision resnet blocks).  Training: `stats` is what mcb_conv_fwd
 * accumulated; finalize turns it into the per-channel affine + saved mean / invstd and updates the running stats. */
int mcb_bn_finalize(const float* stats, long count, const float* gamma, const float* beta, float* running_mean,
                    float* running_var, float momentum, float eps, float* scale, float* shift, float* mean,
                    float* invstd, int c, void* stream);
int mcb_bn_eval_params(const float* gamma, const float* beta, const float* running_mean, const float* running_var,
                       float eps, float* scale, float* shift, int c, void* stream);
/* y = [relu](z*scale + shift [+ residual*res_scale + res_shift | + residual]) — BN + residual add + ReLU in one pass */
int mcb_bn_apply(const void* z, const float* scale, const float* shift, const void* residual, const float* res_scale,
                 const float* res_shift, int relu, void* y, long pixels, int c, void* stream);
/* training-mode BN + residual + ReLU with the finalisation folded in (no separate mcb_bn_finalize launch): the affine is
 * derived in-kernel from `stats`; mean / invstd are published for the backward pass and the running statistics updated.
 * res_bn != NULL: the residual is a raw conv output with its own training-mode BN (ResNet downsample branch). */
typedef struct {
  const float* stats;  /* fp32 [2c] sum, sum of squares (from mcb_conv_fwd) */
  const float* gamma;
  const float* beta;
  float* running_mean; /* may be NULL */
  float* running_var;
  float* mean;         /* out, fp32 [c] */
  float* invstd;       /* out, fp32 [c] */
} mcb_bn_train;
int mcb_bn_train_apply(const void* z, const mcb_bn_train* bn, const void* residual, const mcb_bn_train* res_bn, int relu,
                       void* y, long pixels, int c, float momentum, float eps, void* stream);
/* Synchronised BatchNorm (one process per GPU): `stats` has been all-reduced over the ranks and stat_count = the GLOBAL
   number of pixels per channel; `pixels` stays the local extent of z / y */
int mcb_bn_train_apply_global(const void* z, const mcb_bn_train* bn, const void* residual, const mcb_bn_train* res_bn,
                              int relu, void* y, long pixels, long stat_count, int c, float momentum, float eps,
                              void* stream);
/* backward: g = dy * (y_mask > 0);  dbeta += sum g;  dgamma += sum g * xhat */
int mcb_bn_bwd_reduce(const void* dy, const void* y_mask, const void* z, const float* mean, const float* invstd,
                      float* dbeta, float* dgamma, long pixels, int c, void* stream);
/* dz = gamma*invstd*(g - dbeta/M - xhat*dgamma/M); g_out (optional) receives g (= or +=) for the residual branch */
int mcb_bn_bwd_apply(const void* dy, const void* y_mask, const void* z, const float* mean, const float* invstd,
                     const float* gamma, const float* dbeta, const float* dgamma, void* dz, void* g_out,
                     int g_accumulate, long pixels, int c, void* stream);
/* synchronised variant: dbeta / dgamma all-reduced over the ranks, M = stat_count (global pixels per channel) */
int mcb_bn_bwd_apply_global(const void* dy, const void* y_mask, const void* z, const float* mean, const float* invstd,
                            const float* gamma, const float* dbeta, const float* dgamma, void* dz, void* g_out,
                            int g_accumulate, long pixels, long stat_count, int c, void* stream);
/* out[c] += sum over pixels of x[.., c]  (conv bias gradients) */
int mcb_channel_sum(const void* x, float* out, long pixels, int c, void* stream);
/* the fixed-order sum that finishes every cross-CTA reduction of the library (csrc/detsum.cuh), over rows the caller
 * provides: out[(i / inner) * out_stride + i % inner] += sum over r < nrows of rows[r * row_stride + i], i < n */
int mcb_det_sum_f32(const float* rows, int nrows, long row_stride, long n, long inner, float* out, long out_stride,
                    void* stream);

/* nn.MaxPool2d(2, 2) (src/unet_models.py:356,363,392); backward routes to the first maximum like torch */
int mcb_maxpool2_fwd(const void* x, void* y, int n, int h, int w, int c, void* stream);
int mcb_maxpool2_bwd(const void* x, const void* dy, void* dx, int accumulate, int n, int h, int w, int c,
                     void* stream);
/* VGG encoders (src/unet_models.py:90-105, :296-310): y = relu(conv + b) [n, h, w, c] feeds both pool(y) and a decoder
 * concat.  On entry g holds the concat's data gradient; in place g = bf16(g + routed dpool) * (y > 0) (dpool to the
 * first maximum of each window), and db += the per-channel sums of the stored bf16 g (the conv's bias gradient, summed
 * like mcb_conv_dgrad's dx_channel_sum; fixed-order, run-to-run identical).  g must not alias y or dpool. */
int mcb_maxpool2_bwd_skip_relu(const void* y, const void* dpool, void* g, float* db, int n, int h, int w, int c,
                               void* stream);

/* final = Conv2d(32, 2, 1) (src/unet_models.py:383,403): NHWC bf16 -> NCHW fp32 logits; backward also applies
 * dec0's ReLU mask (x is dec0's output) */
int mcb_final_conv_fwd(const void* x, const float* w, const float* b, float* logits, int n, int h, int wd, int c, int k,
                       void* stream);
int mcb_final_conv_bwd(const void* x, const float* w, const float* dlogits, void* dx, float* dw, float* db, int n,
                       int h, int wd, int c, int k, void* stream);

/* torch.optim.Adam with L2 (src/models.py:57,287-292) over one flat fp32 arena; refreshes the bf16 operand copy.
   The betas are double: the bias corrections 1 - beta^t are taken from them in double, as torch does; the moment
   updates use them rounded to fp32 */
int mcb_adam_step(float* p, const float* g, float* m, float* v, void* p_bf16, long n, float lr, double beta1,
                  double beta2, float eps, float weight_decay, int step, float grad_scale, void* stream);
/* same update with the step-dependent scalars read from DEVICE memory: hyper = {lr, 1-beta1^t, sqrt(1-beta2^t)}
   (fp32[3]), so the launch can be captured once into a CUDA graph and replayed every step */
int mcb_adam_step_dyn(float* p, const float* g, float* m, float* v, void* p_bf16, long n, const float* hyper,
                      float beta1, float beta2, float eps, float weight_decay, float grad_scale, void* stream);
int mcb_cast_f32_bf16(const float* x, void* y, long n, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Losses (src/models.py:310-454, src/steps/pytorch/validation.py:8-28), two phases around the global sums
 * sums[4] = { sum p1*t, sum p1, sum t, sum w*ce } (fp64, zero before phase 1, all-reduce between phases under DDP).
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct {
  const float* logits; /* fp32 NCHW [n][2][h][w] */
  const float* target; /* fp32 NCHW [n][3][h][w] (mask, distance, size) for mode 0; [n][1][h][w] for mode 1 */
  int n, h, w;
  int mode;            /* 0: PyTorchUNetWeighted (weighted CE + Dice); 1: PyTorchUNet (plain CE) */
  float w0, sigma;     /* neptune.yaml:55-56 */
  float size_c;        /* C = sqrt(image_h*image_w)/2 from the CONFIGURED size (src/models.py:373-381) */
  float dice_weight, ce_weight, dice_smooth;
  int dice_activation; /* mode 0's Dice probability of class 1 (src/models.py:438-443): 0 softmax, 1 sigmoid(z1); any
                          other value is rejected.  Mode 1 ignores it.  It is the last field so that a zeroed struct
                          keeps meaning the softmax Dice */
} mcb_loss_args;
int mcb_loss_partials(const mcb_loss_args* a, double* sums, void* stream);
int mcb_loss_grad(const mcb_loss_args* a, const double* sums, long global_pixels, float grad_scale, float* dlogits,
                  float* loss_out, void* stream);
/* numpy softmax over the class axis (src/utils.py:231-273 at src/models.py:88-92) */
int mcb_softmax2(const float* logits, float* probs, int n, int h, int w, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Per-pixel mask post-processing (src/postprocessing.py:48-258, src/utils.py:328-339), batched: a "plane" is one
 * (image, layer) 2-D map; all planes of a batch are processed by one call.  Integer / bool outputs and the float64
 * resize are bit-exact against the reference path (scipy.ndimage / skimage as restated in oracle/post_oracle.py).
 * ---------------------------------------------------------------------------------------------------------------- */

/* resize_image (src/postprocessing.py:48-61) -> skimage.transform.resize(mode='constant'), n-D branch:
 * x fp32 [n][c][hi][wi] -> y fp64 [n][c][ho][wo]; minmax_ws: fp32 [2*n] scratch */
int mcb_resize_bilinear_f64(const float* x, double* y, float* minmax_ws, int n, int c, int hi, int wi, int ho, int wo,
                            void* stream);
/* categorize_multilayer_image (src/postprocessing.py:77-84): out uint8 [n][layers][h][w] = prob[layer_channel[l]] >
 * thresholds[l]; prob fp32 or fp64 [n][c][h][w] */
int mcb_threshold_layers(const void* prob, int prob_is_f64, const double* thresholds, const int* layer_channel,
                         uint8_t* out, int n, int c, int layers, int h, int w, void* stream);
/* label / label_multilayer_image (src/utils.py:328-330, src/postprocessing.py:127-132) -> scipy.ndimage.label:
 * 4-connectivity, labels 1..K in raster order of each component's first pixel, int32.
 * mask uint8 or int32 [planes][h][w]; workspace int32 [planes*h*w]; counts int32 [planes] (K per plane) or NULL */
int mcb_ccl_label(const void* mask, int mask_is_i32, int* labels, int* workspace, int* counts, int planes, int h, int w,
                  void* stream);
/* skimage.morphology.erosion / dilation with rectangle(size, size) (src/postprocessing.py:135-180): uint8 or int32 */
int mcb_morph_rect(const void* in, void* out, int is_i32, int is_dilation, int size, int planes, int h, int w,
                   void* stream);
/* add_dropped_objects (src/utils.py:333-339), per 2-D plane; workspace int32 [2*planes*h*w] */
int mcb_add_dropped_objects(const uint8_t* original, const uint8_t* processed, uint8_t* out, int* workspace, int planes,
                            int h, int w, void* stream);
/* skimage <= 0.17 binary_erosion (ndi.binary_erosion, border_value=True) / binary_dilation with rectangle(size, size)
 * (src/preparation.py:170-186) on {0,1} uint8 planes; differs from mcb_morph_rect only in an even erosion's centre */
int mcb_binary_morph_rect(const uint8_t* in, uint8_t* out, int is_dilation, int size, int planes, int h, int w,
                          void* stream);
/* build_score (src/postprocessing.py:228-236): scores[offsets[p] + l - 1] = mean(prob[labels == l]) * sqrt(area);
 * offsets int32 [planes] (exclusive prefix of the per-plane label counts); sums/counts/scores sized total_instances */
int mcb_instance_scores(const int* labels, const void* prob, int prob_is_f64, const int* offsets, double* sums,
                        int* counts, double* scores, int total_instances, int planes, int h, int w, void* stream);
/* same, without a host round trip: one CTA per plane, scores written at scores[plane*kcap + l - 1] for
 * l <= min(counts[plane], kcap); counts = labels per plane (from mcb_ccl_label); workspaces sized planes*kcap */
int mcb_instance_scores_strided(const int* labels, const void* prob, int prob_is_f64, const int* counts, double* scores,
                                double* gsum_ws, int* gcnt_ws, int kcap, int planes, int h, int w, void* stream);

/* dense_crf (src/postprocessing.py:183-225 -> pydensecrf DenseCRF2D: unary_from_softmax, addPairwiseGaussian,
 * addPairwiseBilateral, inference(iterations)); 2 labels, Potts compatibility, symmetric normalisation, Gaussian
 * kernels evaluated exactly inside a 13x13 window.  PARITY UNPINNED (pydensecrf absent; see oracle/post_oracle.py).
 * probs fp32 [n][2][h][w]; rgb uint8 [n][h][w][3]; out fp32 [n][2][h][w]; workspace fp32 [3*n*2*h*w] */
int mcb_crf_rgb_from_normalized(const float* img_nchw, uint8_t* rgb, int n, int h, int w, void* stream);
int mcb_dense_crf(const float* probs, const uint8_t* rgb, float* out, float* workspace, int n, int h, int w,
                  float compat_gaussian, float sxy_gaussian, float compat_bilateral, float sxy_bilateral, float srgb,
                  int iterations, void* stream);

/* Marker-based watershed on -prob, 4-connectivity.  NOT in the reference (SURVEY.md 0.4); semantics defined by
 * oracle/post_oracle.py::minimax_watershed (minimax flooding cost, geodesic tie-break, smallest label), PARITY UNPINNED.
 * prob fp32|fp64, markers int32 (0 = none), mask uint8, labels int32, all [planes][h][w]; workspace int32 [3*planes*h*w] */
int mcb_watershed(const void* prob, int prob_is_f64, const int* markers, const uint8_t* mask, int* labels,
                  int* workspace, int planes, int h, int w, int levels, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Callers on either side of the per-pixel chain (SURVEY.md 8f-2 / 8f-3) and categorize_image.
 * ---------------------------------------------------------------------------------------------------------------- */

/* categorize_image (src/postprocessing.py:64-74) -> np.argmax(image, axis=0): prob fp32|fp64 [n][c][h][w] -> int64
 * [n][h][w]; first maximum, NaN counts as the maximum (numpy semantics) */
int mcb_argmax_channels(const void* prob, int prob_is_f64, long long* out, int n, int c, int h, int w, void* stream);

/* test_time_augmentation_transform (src/loaders.py:470-480) for nv (image, variant) pairs: out[v] =
 * rot90(flip(x[img_of[v]]), k); code[v] = k | flip << 2 (k quarter turns counter-clockwise; flip 0 none, 1 up-down,
 * 2 left-right).  x fp32 [n][c][h][w], out fp32 [nv][c][h][w] (h == w when k is odd) */
int mcb_tta_transform(const float* x, float* out, const int* img_of, const int* code, int nv, int c, int h, int w,
                      void* stream);
/* The variant rows of the TTA loaders before their pad / resize: test_time_augmentation_transform
 * (src/loaders.py:477-487) with its colour-shift branch, color_seq (src/augmentation.py:12-31), on the decoded tiles.
 * images uint8 [n][h][w][3] RGB -> out uint8 [nv][h][w][3], row v from tile src[v]; code[v] = geometry (bits 0-3, as
 * mcb_tta_transform) | colour branch << 4 (0 none; 1-3 Add to H, S or V through cv2's RGB2HSV / HSV2RGB; 4-6 Add to
 * R, G or B) | value << 8 (0-255; clipped at 255 after the add).  Bit-exact to cv2 4.x's vector body on every pixel
 * (h == w when k is odd) */
int mcb_tta_variants_u8(const uint8_t* images, uint8_t* out, const int* src, const int* code, int nv, int h, int w,
                        void* stream);
/* TestTimeAugmentationAggregator.transform + test_time_augmentation_inverse_transform (src/loaders.py:437-497) in one
 * pass: out[i] = agg over the variants v of image i of flip(rot90(pred[v], -k)); pred fp32 [nv][c][h][w] holds class
 * probabilities, or logits when from_logits (the class softmax of src/models.py:88-92 is then taken in registers).
 * var_start int32 [n+1], var_index int32 [nv]; method 0 gmean, 1 mean, 2 max, 3 min; out fp32 [n][c][h][w]; c <= 8 */
int mcb_tta_aggregate(const float* pred, int from_logits, const int* var_start, const int* var_index, const int* code,
                      float* out, int n, int c, int h, int w, int method, void* stream);

/* Instance emission (src/utils.py:61-127; src/postprocessing.py:284-352).  An instance is (plane, label); its slot is
 * offsets[plane] + label - 1 with offsets the exclusive prefix of counts (labels per plane, from mcb_ccl_label).
 * geometry: geo int32 [total][5] = {area, rmin, rmax, cmin, cmax} (caller initialises {0, INT_MAX, -1, INT_MAX, -1});
 * with prob (fp32|fp64 planes aligned with labels): psum fp64 [total] (zeroed) and pmax int64 [total] (order-preserving
 * integer image of the fp64 maximum -- bits b >= 0 stay, b < 0 become b ^ 0x7FFFFFFFFFFFFFFF -- initialised to that of
 * -inf; an fp32 input widens exactly, so the maximum is exact in either precision) */
int mcb_instance_geometry(const int* labels, const void* prob, int prob_is_f64, const int* offsets, const int* counts,
                          int* geo, double* psum, long long* pmax, int planes, int h, int w, void* stream);
/* COCO run-length encoding of every instance mask (pycocotools rleEncode on the Fortran-ordered mask,
 * src/utils.py:118-120).  One task per (instance, bounding-box column), listed in (instance, column) order by the caller
 * (task_slot, task_x: int32 [ntasks]).  Pass write=0 fills task_n[t] = number of value changes of the column-major scan
 * inside that column; the caller prefix-sums it into task_start; pass write=1 stores the change positions (x*h + y) at
 * changes[task_start[t]...] and sets spans[slot] when a run of ones covers several columns (rleToBbox then reports the
 * full height).  inst_plane int32 [instances] = plane of each slot; geo from mcb_instance_geometry */
int mcb_rle_walk(const int* labels, const int* offsets, const int* geo, const int* inst_plane, const int* task_slot,
                 const int* task_x, const int* task_start, int* task_n, int* changes, int* spans, int ntasks, int h, int w,
                 int write, void* stream);
/* run lengths from change positions: instance `slot` owns counts [out_start[slot] + slot, +nchanges[slot] + 1);
 * slot_of_count int32 [total_counts]; cnts uint32 [total_counts] */
int mcb_rle_counts(const int* changes, const int* nchanges, const int* out_start, const int* slot_of_count,
                   uint32_t* cnts, long total_counts, int hw, void* stream);
/* intersection pixel counts between the instances of two label planes of one image (the IoU matrix of
 * remove_overlapping_masks, src/postprocessing.py:355-386): inter int32 [ka][kb], zeroed by the caller */
int mcb_pair_intersections(const int* labels_a, const int* labels_b, int* inter, int ka, int kb, int h, int w,
                           void* stream);
/* get_contour_length (src/postprocessing.py:340-352): mask pixels with a 4-neighbour outside the mask, per instance;
 * clen int32 [total], zeroed by the caller */
int mcb_contour_length(const int* labels, const int* offsets, const int* counts, int* clen, int planes, int h, int w,
                       void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Input side (SURVEY.md 8f-4): the step right before the network.
 * ---------------------------------------------------------------------------------------------------------------- */

/* padding_seq (src/augmentation.py:40-86 -> cv2.copyMakeBorder, pad_mode 0 = BORDER_REPLICATE, 1 = BORDER_REFLECT_101)
 * + transforms.ToTensor + transforms.Normalize (src/loaders.py:311-317): img uint8 [n][h][w][3] -> out fp32
 * [n][3][h + 2 pad_h][w + 2 pad_w]; mean3 / std3 are HOST pointers to three floats; bit-exact fp32 */
int mcb_image_pad_normalize(const uint8_t* img, float* out, int n, int h, int w, int pad_h, int pad_w, int pad_mode,
                            const float* mean3, const float* std3, void* stream);
/* transforms.Resize on a PIL image (src/loaders.py:287-305, loader_mode 'resize') = Pillow ImagingResample, BILINEAR,
 * 8 bits per channel: horizontal pass into tmp uint8 [n][h][out_w][c], vertical pass into out uint8 [n][out_h][out_w][c];
 * coef_* int32 [out][ksize] = Pillow's 22-bit fixed-point filter rows, bounds_* int32 [out][2] = (first tap, taps),
 * computed by the caller like precompute_coeffs / normalize_coeffs_8bpc (mcb200.preparation does); bit-exact */
int mcb_pil_resize_bilinear_u8(const uint8_t* in, uint8_t* tmp, uint8_t* out, const int* coef_h, const int* bounds_h,
                               int ksize_h, const int* coef_v, const int* bounds_v, int ksize_v, int n, int h, int w,
                               int c, int out_h, int out_w, void* stream);
/* update_distances + clean_distances (src/preparation.py:151-168): masks uint8 [k][h][w] (one plane per building of ONE
 * image); dist_sum fp16 [h][w] = d_nearest + d_second (one building counts twice, none gives 0),
 * second_nearest fp64 [h][w]; distances are scipy.ndimage.distance_transform_edt(1 - mask), exact, including an
 * empty plane (a building eroded to nothing), for which scipy, with no background pixel, gives sqrt((y + 1)^2 + x^2);
 * workspace int32 [k][h][w] */
int mcb_edt_two_nearest(const uint8_t* masks, int k, int h, int w, int* workspace, void* dist_sum_f16,
                        double* second_nearest, void* stream);
/* get_size_matrix (src/preparation.py:189-195): labels int32 [h][w] (mcb_ccl_label), area int32 [labels] -> int64 [h][w] */
/* the same over n images: image i takes the instances [image_off[i], image_off[i + 1]) of a list whose entry k is plane
 * plane_index[k] of masks (uint8 [planes][h][w]; identity when plane_index is NULL); plane_stats (NULL, or
 * mcb_plane_stats of masks) bounds each plane's columns; an empty plane is scipy's all-foreground transform
 * sqrt((y + 1)^2 + x^2).  workspace int32 [k][h][w]; dist_sum fp16 / second_nearest fp64 [n][h][w] */
int mcb_edt_two_nearest_batched(const uint8_t* masks, const int* plane_index, const int* image_off,
                                const int* plane_stats, int k, int n, int h, int w, int* workspace, void* dist_sum_f16,
                                double* second_nearest, void* stream);
int mcb_size_matrix(const int* labels, const int* area, long long* out, int h, int w, void* stream);
/* get_size_matrix of n label planes (mcb_ccl_label numbering per plane); area_ws int32 [n][h][w] workspace */
int mcb_size_matrix_batched(const int* labels, int* area_ws, long long* out, int n, int h, int w, void* stream);
/* the target tensor of MetadataImageSegmentationDatasetDistances (src/loaders.py:141-171), deterministic part:
 * mask uint8 [n][h][w], dist fp16 [n][h][w], sizes int64 [n][h][w] -> fp32 [n][3][h + 2 pad_h][w + 2 pad_w] =
 * {mask, uint8(uint16(dist)), uint8(uint16(sqrt(uint16(sizes))))}, padded like the image */
int mcb_target_channels(const uint8_t* mask, const void* dist_f16, const long long* sizes, float* out, int n, int h, int w,
                        int pad_h, int pad_w, int pad_mode, void* stream);
/* the target tensor from augmented uint8 planes (src/loaders.py:159-165: to_pil, to_monochrome, to_tensor, cat):
 * planes uint8 [n][h][w][c] (c = 3: mask, distances, sizes; c = 1: mask) -> fp32 [n][c][h + 2 pad_h][w + 2 pad_w],
 * padded like the image (padding_seq of the crop-and-pad validation loaders) */
int mcb_target_channels_u8(const uint8_t* planes, float* out, int n, int h, int w, int c, int pad_h, int pad_w,
                           int pad_mode, void* stream);

/* one sample of the training augmentation: fast_seq (src/augmentation.py:5-10) and crop_seq's RandomCropFixedSize
 * (:34-37, :91-135), one deterministic draw applied to every array of the sample (ImgAug,
 * src/steps/pytorch/utils.py:108-129).  Flip bits: 1 = Fliplr, 2 = Flipud. */
typedef struct {
  double inv[9];   /* output (x, y) -> input (column, row) map of skimage warp: np.linalg.inv of the Affine matrix */
  int warp;        /* 0: the sample is not warped (no Affine child drawn); 1: warp through inv */
  int pre_flip;    /* flips drawn before the Affine child */
  int post_flip;   /* flips drawn after it (all flips when warp = 0) */
  int top, left;   /* crop offset (0, 0 in resize mode) */
  int reserved;
} mcb_augment_row;
/* the augmenters of the training loaders (src/loaders.py:140-159, 236-237, 261, 277-278, 302) for a batch:
 * img uint8 [n][h][w][3], mask uint8 [n][h][w], dist / size uint16 [n][h][w] (both or neither: the distance loaders'
 * Di / Si after their astype casts) -> img_out uint8 [n][out_h][out_w][3], tgt_out uint8 [n][out_h][out_w][c]
 * (c = 3: mask, distances, sizes; c = 1 without dist / size), every pixel cropped, flipped and warped like
 * imgaug 0.2.5's Affine over skimage.transform.warp (order 1, constant 0, fp64, clipped to each array's input range,
 * truncated to its dtype), uint16 planes then wrapped to uint8 like to_pil (src/utils.py:284-289).
 * rows: HOST array [n] (checked, then passed to the kernels by value); range_ws uint32 [n][8] workspace. */
int mcb_augment_warp(const uint8_t* img, const uint8_t* mask, const uint16_t* dist, const uint16_t* size,
                     const mcb_augment_row* rows, int n, int h, int w, int out_h, int out_w, unsigned* range_ws,
                     uint8_t* img_out, uint8_t* tgt_out, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Synchronised BatchNorm over NVLink peer memory (SURVEY.md 8e collective (2)): one-shot all-reduce of a small fp32
 * vector.  `partial` = this rank's partial sums (local memory, this exchange at [offset, offset+count)).  peer_recv:
 * DEVICE array of `world` pointers, entry r = rank r's symmetric receive buffer as mapped in this process (caller's
 * plumbing, e.g. torch symmetric memory): per rank [world][stride] pairs of (fp32 value, uint32 stamp), zeroed once.
 * The kernel pushes (partial[offset + c], *step) into slot [rank] of every peer, polls its own slots for this step's
 * stamp and writes out[c] = sum over ranks (in rank order); optionally out2_first[c] / out2_second[c - split] =
 * scale2 * out[c].  *step is the device-resident step stamp (mcb_sync_step_bump at the start of every step; never 0).
 * Asynchronous on `stream`, capturable.
 * ---------------------------------------------------------------------------------------------------------------- */
int mcb_sync_step_bump(unsigned* step, void* stream);
int mcb_sync_exchange(const float* partial, void* const* peer_recv, int rank, int world, long stride, long offset,
                      int count, const unsigned* step, float* out, float* out2_first, float* out2_second, int split,
                      float scale2, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * COCO segmentation evaluation (src/cocoeval.py, csrc/evaluation.cu)
 * ---------------------------------------------------------------------------------------------------------------- */
/* mask IoU of (detection, ground truth) pairs, pycocotools rleIou as src/cocoeval.py:196 calls it
 * (maskUtils.iou(d, g, iscrowd)): run lists dt_cnts / gt_cnts uint32 (COCO column-major RLE counts), RLE r owning
 * [starts[r], starts[r + 1]) (int64); gt_crowd uint8 per ground-truth RLE (union = detection area when set).
 * Pair p (int32 pair_dt / pair_gt, bounding boxes already found to overlap by the caller) writes
 * iou[pair_out[p]] = i / u (fp64), 0 when the masks do not intersect.  Entries of pairs not listed are the caller's
 * (zero: pycocotools' bounding-box gate).  One thread per pair. */
int mcb_rle_pair_iou(const uint32_t* dt_cnts, const long long* dt_starts, const uint32_t* gt_cnts,
                     const long long* gt_starts, const uint8_t* gt_crowd, const int* pair_dt, const int* pair_gt,
                     const long long* pair_out, double* iou, int npairs, void* stream);
/* get_iou over get_iou_matrix (src/postprocessing.py:306-328): out[r] = max of iou[row_off[r], row_off[r + 1]) (fp64),
 * NaN for an empty row (no ground truth of the instance's image and category: the reference's `None`).
 * row_off int64 [rows + 1].  One thread per row. */
int mcb_iou_row_max(const double* iou, const long long* row_off, int rows, double* out, void* stream);
/* COCOeval.evaluateImg (src/cocoeval.py:242-320) for every (unit, area range); a unit is one (image, category) with
 * nd[u] detections (score-ordered, already cut to maxDets[-1]) at dt_off[u] and ng[u] ground truths (file order) at
 * gt_off[u]; its IoU table is iou[iou_off[u] + d * ng[u] + g].  dt_id int64, dt_area fp64; gt_id int64, gt_crowd uint8
 * (iscrowd = ignore), gt_area fp64 (the JSON area); area_rng fp64 [A][2] (both bounds inclusive); thr fp64 [T]
 * (T <= 32).  Outputs: dt_match int64 [A][T][d_total] (matched ground-truth id, 0 = none), dt_ignore uint8
 * [A][T][d_total], gt_ignore uint8 [A][g_total] (in the stable `_ignore` order); gt_taken uint8 [A][T][g_total] is
 * workspace, zeroed by the caller.  One warp per (unit, area range), one lane per threshold. */
int mcb_coco_match(const double* iou, const long long* iou_off, const int* nd, const int* ng, const long long* dt_off,
                   const long long* dt_id, const double* dt_area, const long long* gt_off, const long long* gt_id,
                   const uint8_t* gt_crowd, const double* gt_area, const double* area_rng, const double* thr, int units,
                   int A, int T, long long d_total, long long g_total, long long* dt_match, uint8_t* dt_ignore,
                   uint8_t* gt_ignore, uint8_t* gt_taken, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Second-level scoring model (src/models.py:212-282, csrc/forest.cu; the importers are mcb200.forest)
 * ---------------------------------------------------------------------------------------------------------------- */
#define MCB_FOREST_SKLEARN 0      /* RandomForestRegressor.predict */
#define MCB_FOREST_LIGHTGBM 1     /* Booster.predict of an L2 regression model */
#define MCB_FOREST_DEFAULT_LEFT 2 /* flag bit: a missing value goes left (LightGBM's kDefaultLeftMask) */
#define MCB_FOREST_MISSING_ZERO 1 /* (flags >> 2) & 3, LightGBM's MissingType */
#define MCB_FOREST_MISSING_NAN 2
/* ScoringRandomForest.transform / ScoringLightGBM.transform (src/models.py:232-243, 267-278): out fp64 [rows] =
 * (0.0 + leaf of tree 0 + leaf of tree 1 + ... in tree order) [/ n_trees when average], for the row-major fp64 feature
 * matrix x [rows][n_features].  One node format for both libraries: node n has feature[n] (int32), threshold[n]
 * (fp64), left[n] / right[n] (int32: a node index, or ~k for leaf_value[k]) and flags[n] (uint8, LightGBM's
 * decision_type layout without the categorical bit); tree_root int32 [n_trees] is a node index or ~k for a one-leaf
 * tree.  The forest must be acyclic (mcb200.forest validates it).  semantics MCB_FOREST_SKLEARN: x is cast to float32,
 * NaN follows DEFAULT_LEFT, else x <= threshold.  MCB_FOREST_LIGHTGBM: |x| <= (double)1e-35f becomes 0.0, NaN under a
 * missing type other than NaN becomes 0.0, a zero under MISSING_ZERO or a NaN under MISSING_NAN follows DEFAULT_LEFT,
 * else x <= threshold.  work fp64 [chunk_trees * rows] is caller-owned: the trees are traversed chunk by chunk, one
 * thread per (tree, row), and each row's running sum is carried across chunks in out. */
int mcb_forest_predict(const double* x, int rows, int n_features, const int* tree_root, int n_trees, const int* feature,
                       const double* threshold, const int* left, const int* right, const uint8_t* flags,
                       const double* leaf_value, int semantics, int average, double* work, int chunk_trees, double* out,
                       void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Target preparation from COCO polygons (src/preparation.py:18-198, csrc/polygon.cu)
 * ---------------------------------------------------------------------------------------------------------------- */
/* pycocotools maskApi.c rleFrPoly + rleDecode (cocomask.frPyObjects(polys, h, w) then decode), bit-exact.  The host
 * scales the vertices, (int)(5 x + .5), and passes one row per edge of the closed polygons: edge_xy int32 [edges][4] =
 * (xs, ys, xe, ye), edge_pt int64 [edges + 1] = first upsampled point of each edge (max(|dx|, |dy|) + 1 per edge,
 * points = edge_pt[edges]), edge_plane int32 [edges] = the polygon's output plane (consecutive polygons differ).
 * bits uint32 [planes][ceil(h*w / 32)] workspace; out uint8 [planes][h][w] row-major. */
int mcb_rasterize_polygons(const int* edge_xy, const long long* edge_pt, const int* edge_plane, int edges,
                           long long points, uint32_t* bits, uint8_t* out, int planes, int h, int w, void* stream);
/* per uint8 plane: stats int32 [count][4] = (pixel count, any pixel at least `border` away from every edge
 * (not is_on_border(m, border), src/preparation.py:197-198), first column, last column with a pixel (w, -1 if none)) */
int mcb_plane_stats(const uint8_t* planes, int count, int h, int w, int border, int* stats, void* stream);
/* out[g] = union of the planes index[group_off[g] .. group_off[g + 1]) of `planes`, uint8 {0,1} [groups][h][w] */
int mcb_plane_union(const uint8_t* planes, const int* index, const int* group_off, int groups, int h, int w,
                    uint8_t* out, void* stream);
/* mask_overlayed = np.where(mask_c, category_nr[c], mask_overlayed) over c (src/preparation.py:50-78):
 * cat_masks uint8 [n][categories][h][w], category_nr int32 [categories] (device) -> out uint8 [n][h][w] */
int mcb_category_overlay(const uint8_t* cat_masks, const int* category_nr, int categories, int n, int h, int w,
                         uint8_t* out, void* stream);
/* the border class (src/preparation.py:83-86) in place: where second_nearest < border_width and the class is even
 * (numpy's bool & ~uint8), the class becomes the image's max + 1 */
int mcb_border_class(uint8_t* mask, const double* second_nearest, int n, int h, int w, double border_width,
                     void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * JPEG decode (csrc/jpeg.cu; the host side that parses the files and lays out these tables is mcb200.jpeg)
 * Sequential Huffman JPEG, 8-bit, one scan, 1 or 3 components each sampled at 1 or 1/2 of the largest factor, bit-exact
 * to libjpeg-turbo (islow IDCT, fancy upsampling).  All int32 tables are device memory:
 *   images [n][36]   = ncomp, mcux, hmax, vmax, first segment, segment count, then per component (10 words): h, v, blocks_w, blocks_h, first block of
 *                      the component in `coef` / `planes`, downsampled width, downsampled height, DC table slot, AC
 *                      table slot (image * 8 + class * 4 + id), 0.  Blocks and segments of an image are consecutive,
 *                      images in order.
 *   segments [s][5]  = image, byte offset in `data`, byte count, first MCU, MCU count (an image, or one restart
 *                      interval; bytes unstuffed, restart markers removed)
 *   huff [slot][804] = 512 lookahead entries (length << 8 | symbol for codes of at most 9 bits, else 0), maxcode[18]
 *                      by length (index 17 a sentinel), value offset[18] by length, symbols[256]
 *   qt [n][3][64]    = quantisation tables in natural order, per component
 *   tables [4][256]  = jdcolor.c's Cr->R, Cb->B, Cr->G, Cb->G tables
 * ---------------------------------------------------------------------------------------------------------------- */
/* entropy decode, one thread per segment, one CTA per image: coef int16 [blocks][64] (natural order, padding blocks of the MCUs included);
 * status int32 [n] is zeroed, then set non-zero for an image whose data ends inside a segment (1), holds a code no table
 * has (2) or runs a coefficient index past 63 (3).  No segment is read past its byte count. */
int mcb_jpeg_entropy_decode(const uint8_t* data, const int* segments, int nseg, const int* images, const int* huff,
                            int n, int16_t* coef, int* status, void* stream);
/* bits per subsequence of the parallel entropy decode (a compile-time constant of the library) */
int mcb_jpeg_subsequence_bits(void);
/* entropy decode with the same inputs and the same coef and status as mcb_jpeg_entropy_decode, parallel inside each
 * segment: a segment of B bytes is cut into S = mcb_jpeg_subsequence_bits()-bit subsequences, decoded speculatively,
 * resolved in order (a guess that proves wrong is decoded again, so a stream that never resynchronises costs about
 * one serial decode) and written out; a segment given one subsequence is decoded whole by one thread.  Three launches,
 * no memset, no allocation, no host synchronisation; capturable into a CUDA graph.  A segment must be shorter than
 * 2^28 bytes, and one image may have at most 65535 * 128 subsequences.
 *   sub_first int32 [nseg + 1]  first subsequence of each segment, numbered across the batch (prefix sum of the counts);
 *                               a segment's count is 1 or ceil(8 * B / S) (mcb200.jpeg splits segments of more than 16)
 *   max_image_subs              the most subsequences of any one image (sizes the grid)
 *   workspace int32 [16 + 16 * sub_first[nseg]]  caller-owned; words 0..3 count the speculated entry states that held,
 *                               were corrected, the longest run of consecutive corrections and the exact re-decodes
 *                               of a segment's error or last block; the rest is per-subsequence state
 * coef is fully written (every block zeroed first); status as mcb_jpeg_entropy_decode. */
int mcb_jpeg_entropy_decode_parallel(const uint8_t* data, const int* segments, int nseg, const int* images,
                                     const int* huff, int n, const int* sub_first, int max_image_subs, int* workspace,
                                     int16_t* coef, int* status, void* stream);
/* dequantisation + libjpeg's jpeg_idct_islow per block -> planes uint8 [blocks][8][8] */
int mcb_jpeg_idct(const int16_t* coef, const int* qt, const int* images, int n, int n_blocks, uint8_t* planes,
                  void* stream);
/* libjpeg-turbo's fancy upsampling + ycc_rgb_convert (grayscale replicated) -> out uint8 [n][h][w][3] */
int mcb_jpeg_upsample_rgb(const uint8_t* planes, const int* images, const int* tables, int n, int h, int w,
                          uint8_t* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MCB200_H_ */
