/*
 * atomai_b200.h — C ABI of libatomai_b200.so (sm_90a only).
 *
 * Drop-in boundary for the AtomAI data-parallel hot path (SURVEY.md §8b).  The
 * reference (pycroscopy/atomai v0.8.1) has no FFI of its own: every entry point
 * below replaces a stock torch op call site inside the reference's nn.Modules,
 * cited per function as /root/reference-relative file:line.
 *
 * Conventions
 *  - All pointers are DEVICE pointers unless the name ends in _host.
 *  - Activations are NHWC fp32 ("pixel-major"): element (n,h,w,c) lives at
 *    ((n*H + h)*W + w)*ld + c, ld >= C (ld lets a tensor be a channel slice).
 *  - Every launch goes to `stream` (a cudaStream_t passed as void*).
 *  - Sums across CTAs (BatchNorm statistics and backward sums, weight gradients, losses) are
 *    added in a fixed order, so repeating a call on the same inputs gives bit-identical
 *    results.  Their partials live in a library-internal device workspace per (device, stream),
 *    allocated on first use and grown when a larger launch needs it; calls on different streams
 *    may run concurrently.
 *  - The caller owns every buffer; the library never allocates caller-visible
 *    memory.  Return value: 0 = ok, non-zero = error, text via
 *    atomai_b200_last_error() (thread-local).  No exceptions cross the ABI.
 *  - math: 0 = exact fp32 FFMA kernels, 1 = TF32 wgmma tensor-core kernels
 *    (fp32 accumulate in registers), 2 = the same kernels with every operand split into
 *    hi = rn_tf32(v) and lo = v - hi.  Forward / data gradient: per k-step one TF32 MMA on
 *    (a_hi, w_hi) plus one bf16 MMA that adds a_lo*w + a_hi*w_lo; weight gradient: three TF32
 *    MMAs (hi, hi), (lo, hi), (hi, lo).  lo*lo is not formed.  Per element,
 *    |y - y_exact| <= (2^-18 + (K+2) 2^-23) * (sum |x||w| + |b|) for K = taps * Cin (pixels
 *    for the weight gradient), against 2^-10 + (K+2) 2^-23 in mode 1 and (K+2) 2^-24 in
 *    mode 0 (tests/test_conv_exact_gpu.py).  There is no CPU path.
 */
#ifndef ATOMAI_B200_H
#define ATOMAI_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AB_MATH_FP32 0
#define AB_MATH_TF32 1
#define AB_MATH_TF32X3 2 /* split operands: a_hi*w_hi + a_lo*w + a_hi*w_lo (see `math` above) */

#define AB_ACT_LRELU 0
#define AB_ACT_TANH 1
#define AB_ACT_RBF 2      /* y = lrelu * exp(-0.5 * max(x, 0))        (Gram epilogue)      */
#define AB_ACT_MATERN25 3 /* y = lrelu * (1 + s + s^2/3) exp(-s), s = sqrt(5 max(x, 0))   */

#define AB_WMODE_FWD 0   /* weights as used by the forward conv           */
#define AB_WMODE_DGRAD 1 /* flipped + transposed weights for data-gradient */

/* One input source of a convolution.  The loader applies, in this order:
 * per-channel affine (BatchNorm normalise-on-load), 2x2 max-pool OR 2x upsampling, zero padding.
 * Replaces the separate BatchNorm2d / F.max_pool2d / F.interpolate / torch.cat passes of
 * atomai/nets/blocks.py:73,130-131 and atomai/nets/fcnn.py:123-138. */
typedef struct {
  const float* ptr;   /* NHWC base                                          */
  const float* scale; /* [C] or NULL                                        */
  const float* shift; /* [C] or NULL                                        */
  int32_t C;          /* channels taken from this source                    */
  int32_t ld;         /* pixel stride in floats                             */
  int32_t pool;       /* 1: source is (2H,2W); 2x2 max taken after affine;
                         2 / 3: source is (H/2,W/2); bilinear (align_corners=0) /
                         nearest 2x upsampling on load (H, W even)          */
  int32_t reserved;
} ab_src_t;

/* Convolution descriptor: stride 1, "same" zero padding (pad = dil*(ks/2)),
 * ks in {1,3}; 1-D signals are H = 1 with ks_h = 1. */
typedef struct {
  int32_t N, H, W;     /* output (= input) spatial extent                   */
  int32_t Cout;
  int32_t ks_h, ks_w;  /* 1 or 3 each                                       */
  int32_t dil;
  int32_t nsrc;        /* 1 or 2 (2 = concat-free torch.cat([s0, s1], 1))   */
  ab_src_t src[2];
  float lrelu;         /* LeakyReLU slope; 1.0f = identity, 0.0f = ReLU     */
  int32_t math;        /* AB_MATH_*                                         */
  int32_t out_nchw;    /* 1: store output as NCHW (for flatten -> Linear)   */
  int32_t act;         /* AB_ACT_LRELU (uses .lrelu) or AB_ACT_TANH         */
} ab_conv_t;

const char* atomai_b200_version(void);
const char* atomai_b200_last_error(void);
/* 1 if the wgmma kernels can run on `device` (compute capability 9.x). */
int atomai_b200_device_ok(int device);

/* ---- weight preparation -------------------------------------------------
 * OIHW fp32 (nn.Conv2d.weight, atomai/nets/blocks.py:63-67) -> kernel layout.
 * FP32: [tap][Cin][Cout];  TF32: K-chunked UMMA core-matrix blobs, RN-rounded.
 * Cin/Cout here are the forward layer's; mode AB_WMODE_DGRAD emits the
 * flipped/transposed operator.  `out` must hold ab_prep_weights_elems(). */
int64_t atomai_b200_prep_weights_elems(int Cout, int Cin, int ks_h, int ks_w, int mode, int math);
int atomai_b200_prep_weights(const float* w_oihw, int Cout, int Cin, int ks_h, int ks_w,
                             int mode, int math, float* out, void* stream);

/* ---- convolution forward (also used for dgrad with AB_WMODE_DGRAD weights) --
 * y = lrelu(conv(x) + bias); optional per-channel (sum, sum^2) of y into
 * stats[2*Cout] (double, caller zeroes; added to in a fixed order, see Conventions).
 * Replaces nn.Conv2d + nn.LeakyReLU (+ the statistics pass of nn.BatchNorm2d):
 * atomai/nets/blocks.py:61-76 (ConvBlock), :302-319 (DilatedBlock),
 * :130-132 (UpsampleBlock 1x1), atomai/nets/fcnn.py:115 (px head). */
int atomai_b200_conv_fwd(const ab_conv_t* d, const float* w_prepped, const float* bias,
                         float* y, int ld_y, double* stats, void* stream);
/* 1 if the tensor-core (AB_MATH_TF32) kernel takes this descriptor: which = 0 forward / dgrad
 * (atomai_b200_conv_fwd), 1 weight gradient (atomai_b200_conv_wgrad).  Callers fall back to
 * AB_MATH_FP32 (exact SIMT kernels) for the rest — thin channel counts, odd strides. */
int atomai_b200_conv_supported(const ab_conv_t* d, int which);
/* scratch/occupancy query so the caller can report launch geometry */
int atomai_b200_conv_info(const ab_conv_t* d, int* grid, int* block, int* smem_bytes);

/* ---- weight gradient ------------------------------------------------------
 * dW[co][ci][ky][kx] += sum_p dy[p][co] * x[p + tap][ci]  (OIHW fp32, caller
 * zeroes), x seen through the same loader as the forward.  Replaces autograd's
 * cuDNN bwd-filter for atomai/trainers/trainer.py:206. */
int atomai_b200_conv_wgrad(const ab_conv_t* d, const float* dy, int ld_dy,
                           float* dw_oihw, void* stream);

/* ---- BatchNorm ------------------------------------------------------------
 * finalize: stats -> (scale, shift) used by the next loader, saved (mean,
 * invstd), running-stat update (momentum, unbiased var) — nn.BatchNorm2d
 * training semantics, atomai/nets/blocks.py:73.  training=0: scale/shift from
 * running stats.  */
int atomai_b200_bn_finalize(const double* stats, int C, double count, const float* gamma,
                            const float* beta, float* running_mean, float* running_var,
                            float momentum, float eps, int training, float* scale,
                            float* shift, float* mean, float* invstd, void* stream);
/* y = a*scale + shift  (materialise a BN output when a module boundary needs it) */
int atomai_b200_affine(const float* a, int ld_a, const float* scale, const float* shift,
                       float* y, int ld_y, int64_t npix, int C, int out_nchw_hw, void* stream);
/* backward, pass 1: sums[0:C] = sum dY, sums[C:2C] = sum dY*xhat (double, caller zeroes) */
int atomai_b200_bn_bwd_reduce(const float* dy, int ld_dy, const float* a, int ld_a,
                              const float* mean, const float* invstd, int64_t npix, int C,
                              double* sums, void* stream);
/* backward, pass 2 (+LeakyReLU backward, + bias gradient):
 *   g    = bn ? scale*(dY - s1/M - xhat*s2/M) : dY        [+ extra if given]
 *   dpre = act'(a) * g   (lrelu' from sign(a), tanh' = 1-a^2)   [+ extra if given]
 *   dbias[c] += sum dpre  (double, caller zeroes; may be NULL)
 * `extra` carries DilatedBlock's direct taps (atomai/nets/blocks.py:321-329). */
int atomai_b200_bn_lrelu_bwd(const float* dy, int ld_dy, const float* a, int ld_a,
                             const float* mean, const float* invstd, const float* scale,
                             const double* sums, double count, const float* extra, int ld_extra,
                             int act, float lrelu, float* dpre, int ld_dpre, double* dbias,
                             int64_t npix, int C, void* stream);

/* ---- pooling / upsampling ---------------------------------------------------
 * F.max_pool2d(2,2) atomai/nets/fcnn.py:123-127 ; F.interpolate(x2, bilinear
 * align_corners=False | nearest) atomai/nets/blocks.py:130-131. */
int atomai_b200_pool2x2_fwd(const float* a, int ld_a, const float* scale, const float* shift,
                            float* y, int ld_y, int N, int Ho, int Wo, int C, void* stream);
/* dfull (+)= scatter(dpooled) to the first-max position of the affine'd window */
int atomai_b200_pool2x2_bwd(const float* dp, int ld_dp, const float* a, int ld_a,
                            const float* scale, const float* shift, float* dfull, int ld_df,
                            int accumulate, int N, int Ho, int Wo, int C, void* stream);
/* the same, and — when `sums` is given — the BatchNorm-backward reductions of the finished
 * gradient (sums[0:C] += sum dY, sums[C:2C] += sum dY*xhat, as atomai_b200_bn_bwd_reduce) in the
 * same pass: valid when this call is the last contribution to dfull.  C/4 a power of two. */
int atomai_b200_pool2x2_bwd_bn(const float* dp, int ld_dp, const float* a, int ld_a,
                               const float* scale, const float* shift, float* dfull, int ld_df,
                               int accumulate, int N, int Ho, int Wo, int C, const float* mean,
                               const float* invstd, double* sums, void* stream);
int atomai_b200_upsample2x_fwd(const float* x, int ld_x, float* y, int ld_y, int N, int h, int w,
                               int C, int bilinear, void* stream);
int atomai_b200_upsample2x_bwd(const float* dy, int ld_dy, float* dx, int ld_dx, int N, int h,
                               int w, int C, int bilinear, void* stream);
/* ImSpec encoder_downsampling (atomai/nets/ed.py:66-79): y (N, H/sh, W/sw, C) = average over each
 * sh x sw window of x (N, H, W, C), floor semantics; sum in row-major order times 1/(sh*sw).
 * Images use (s, s), spectra stored as (N, 1, L, 1) use (1, s).  Forward only. */
int atomai_b200_avgpool_fwd(const float* x, int ld_x, float* y, int ld_y, int N, int H, int W, int C,
                            int sh, int sw, void* stream);
/* 1-D decoder_upsampling (atomai/nets/ed.py:151-154): nearest x2 along the width of (N, 1, w, C)
 * -> (N, 1, 2w, C), and its adjoint dx[i] = dy[2i] + dy[2i+1]. */
int atomai_b200_upsample_w2x_fwd(const float* x, int ld_x, float* y, int ld_y, int N, int w, int C,
                                 void* stream);
int atomai_b200_upsample_w2x_bwd(const float* dy, int ld_dy, float* dx, int ld_dx, int N, int w, int C,
                                 void* stream);
/* ResBlock tail (atomai/nets/blocks.py:199-214): y = LeakyReLU(a*scale + shift + res) in one
 * pass; scale/shift (the BatchNorm affine) and res (the residual) may be NULL.  Backward mask:
 * g = dy * LeakyReLU'(y), read from sign(y) (slope > 0). */
int atomai_b200_affine_res_act(const float* a, int ld_a, const float* scale, const float* shift,
                               const float* res, int ld_res, float lrelu, float* y, int ld_y,
                               int64_t npix, int C, void* stream);
int atomai_b200_lrelu_mask_bwd(const float* dy, int ld_dy, const float* y, int ld_y, float lrelu,
                               float* g, int ld_g, int64_t npix, int C, void* stream);
/* F.interpolate(size = factor * (h, w), mode = bilinear (align_corners=False) | nearest) of the
 * ResHedNet side outputs (atomai/nets/fcnn.py:292-293) and its adjoint (dx zeroed by the caller,
 * accumulated with atomics). */
int atomai_b200_resize_fwd(const float* x, int ld_x, float* y, int ld_y, int N, int h, int w, int C,
                           int factor, int bilinear, void* stream);
int atomai_b200_resize_bwd(const float* dy, int ld_dy, float* dx, int ld_dx, int N, int h, int w,
                           int C, int factor, int bilinear, void* stream);
/* MobileNetV2 (Regressor / Classifier backbone, atomai/nets/blocks.py:376-387), mobilenet.cu.
 * 3x3 convolution, pad 1, stride 1 or 2, output (N, (H-1)/stride+1, (W-1)/stride+1, Cout): dense
 * (w: Cout x Cin x 3 x 3, the stem) or depthwise (Cin == Cout, w: C x 1 x 3 x 3).  The input is
 * read as act(x) = [relu6 if clip](x*scale + shift) (scale/shift may be NULL); stats (2*Cout
 * doubles, zeroed by the caller, may be NULL) receive the BatchNorm sums (sum y, sum y^2) of the
 * raw output.  wgrad adds sum over pixels of dy * act(x) into dw (zeroed by the caller); dgrad is
 * the depthwise data gradient w.r.t. act(x) (gather, no atomics).  Every cross-CTA sum is ordered. */
int atomai_b200_conv3x3_fwd(const float* x, int ld_x, const float* scale, const float* shift,
                            int clip, const float* w, int depthwise, float* y, int ld_y, int N,
                            int H, int W, int Cin, int Cout, int stride, double* stats,
                            void* stream);
int atomai_b200_conv3x3_wgrad(const float* dy, int ld_dy, const float* x, int ld_x,
                              const float* scale, const float* shift, int clip, int depthwise,
                              float* dw, int N, int H, int W, int Cin, int Cout, int stride,
                              void* stream);
int atomai_b200_dw3x3_dgrad(const float* dy, int ld_dy, const float* w, float* dx, int ld_dx,
                            int N, int H, int W, int C, int stride, void* stream);
/* BatchNorm -> ReLU6 backward, first pass: g = dy * [0 < a*scale + shift < 6] and
 * sums += (sum g, sum g * (a - mean) * invstd) per channel (2*C doubles); the apply is
 * atomai_b200_bn_lrelu_bwd on g with slope 1.  hw > 0: dy is the (N, C) gradient of an average
 * pool over hw pixels per image (row stride ld_dy), read as dy[n][c] / hw at every pixel. */
int atomai_b200_relu6_bwd_reduce(const float* dy, int ld_dy, const float* a, int ld_a,
                                 const float* scale, const float* shift, const float* mean,
                                 const float* invstd, float* g, int ld_g, int64_t npix, int C,
                                 int hw, double* sums, void* stream);
/* y = relu6(a*scale + shift) */
int atomai_b200_affine_relu6(const float* a, int ld_a, const float* scale, const float* shift,
                             float* y, int ld_y, int64_t npix, int C, void* stream);
/* y (N, C) = mean over the HW pixels of relu6(a*scale + shift) (AdaptiveAvgPool2d(1)); backward
 * g (N, HW, C) = dy / HW */
int atomai_b200_avgpool_relu6_fwd(const float* a, int ld_a, const float* scale, const float* shift,
                                  float* y, int N, int HW, int C, void* stream);
int atomai_b200_avgpool_bwd(const float* dy, float* g, int ld_g, int N, int HW, int C,
                            void* stream);
/* LogSoftmax(dim=1) of a contiguous (B, C) matrix and its backward dx = dy - exp(y) sum(dy) */
int atomai_b200_log_softmax_fwd(const float* x, float* y, int B, int C, void* stream);
int atomai_b200_log_softmax_bwd(const float* y, const float* dy, float* dx, int B, int C,
                                void* stream);
/* mean NLL loss of (B, C) log-probabilities and int64 targets: loss (1 float, may be NULL) =
 * -mean_i logp[i][t_i] (NaN for a target outside [0, C)); dlogp (may be NULL) = -g/B at the
 * targets, 0 elsewhere, g read from gscale_dev (NULL: 1). */
int atomai_b200_nll_fwd_bwd(const float* logp, const int64_t* target, int B, int C, float* loss,
                            float* dlogp, const float* gscale_dev, void* stream);
/* y[n][c][r] = x[n][r][c]: NHWC <-> NCHW around `x.reshape(-1, C*H*W)` -> nn.Linear
 * (atomai/nets/ed.py:77-79, 284-287, 516-517). */
int atomai_b200_transpose(const float* x, float* y, int N, int R, int Cc, void* stream);
/* dst[p][0:C] (+)= src[p][0:C] — gradient routing between channel slices */
int atomai_b200_add_slice(const float* src, int ld_s, float* dst, int ld_d, int accumulate,
                          int64_t npix, int C, void* stream);
/* out = sum_l (pre_l + a_l + [bn_l(a_l)]) — DilatedBlock.forward, blocks.py:321-329 */
int atomai_b200_dilated_sum(const float* const* a_ptrs, const float* const* scale_ptrs,
                            const float* const* shift_ptrs, int nlayers, float lrelu, float* out,
                            int64_t n_elems, int C, void* stream);

/* ---- losses -----------------------------------------------------------------
 * nn.CrossEntropyLoss (mean) over NHWC logits + int64 labels:
 * atomai/losses_metrics/losses.py:154-155, called at trainers/trainer.py:205.
 * loss_sum: double[1] (nullable; caller zeroes); dlogits (nullable) = (softmax-onehot)*g with
 * g = gscale * (gscale_dev ? *gscale_dev : 1) — the device scalar carries autograd's upstream
 * gradient without a host sync. */
int atomai_b200_ce_fwd_bwd(const float* logits, int ld, const int64_t* labels, int64_t npix,
                           int C, double* loss_sum, float* dlogits, int ld_d, float gscale,
                           const float* gscale_dev, void* stream);
/* kind 0: MSE (losses.py:163-164), 1: BCE-with-logits (losses.py:157-158); elementwise over n */
int atomai_b200_pointwise_loss(const float* pred, const float* target, int64_t n, int kind,
                               double* loss_sum, float* dpred, float gscale,
                               const float* gscale_dev, void* stream);
/* Dice loss (atomai/losses_metrics/losses.py:53-89) over NHWC logits of an N x H x W batch.
 * C > 1: softmax probabilities, int64 labels (N, H, W); the reference sums over dims (0, 2), so
 * there are K = C*W cells (class, image column).  C == 1: probabilities [sigmoid, 1 - sigmoid],
 * targets [y == 1, y == 0] of (N, 1, H, W) labels (float if label_float, else int64), K = 2.
 * dice_sums writes cells[0:K] = I = sum p*t and cells[K:2K] = S = sum (p + t) (double, ordered
 * cross-CTA sums, C <= 16, 2*C*ceil(W/32)*32 <= 2^21; N = 0 zeroes them).  dice_finalize: loss[0] = 1 - mean 2I/(S+eps)
 * and coef[0:K] = -(2/K)/(S+eps), coef[K:2K] = (2/K) I/(S+eps)^2 (nullable).  dice_bwd:
 * dlogits = g * dL/dlogits with dL/dp = t*coef[k] + coef[K+k], chained through the softmax /
 * sigmoid, g = gscale * (gscale_dev ? *gscale_dev : 1). */
int atomai_b200_dice_sums(const float* logits, int ld, const void* labels, int label_float, int N,
                          int H, int W, int C, double* cells, void* stream);
int atomai_b200_dice_finalize(const double* cells, int K, float eps, float* loss, float* coef,
                              void* stream);
int atomai_b200_dice_bwd(const float* logits, int ld, const void* labels, int label_float, int N,
                         int H, int W, int C, const float* coef, float* dlogits, int ld_d,
                         float gscale, const float* gscale_dev, void* stream);
/* Focal loss (losses.py:13-50) from the BCE-with-logits sum of atomai_b200_pointwise_loss(kind 1):
 * CE = *bce_sum / count, pt = exp(-CE), loss[0] = alpha (1-pt)^gamma CE, factor[0] = dloss/dCE
 * (nullable) — the device scale of the BCE gradient. */
int atomai_b200_focal_finalize(const double* bce_sum, double count, float alpha, float gamma,
                               float* loss, float* factor, void* stream);

/* ---- segmentation accuracy -----------------------------------------------------
 * Mean IoU (atomai/losses_metrics/metrics.py:16-95).  iou_hist: counts[nc*true + pred] += pixels
 * (int64, nc*nc, caller zeroes; nc = max(C, 2), C <= 64), pred = sum_c c*[softmax_c > thresh]
 * (0 if above C-1) for C > 1, [sigmoid > thresh] for C == 1 (activation = 0: the raw values
 * instead of softmax / sigmoid); labels int64 or float
 * (label_float, truncated); pixels whose label is outside [0, nc) are skipped.
 * iou_finalize: iou[0] = mean_c diag / (rowsum + colsum - diag + 1e-10) in float32. */
int atomai_b200_iou_hist(const float* logits, int ld, const void* labels, int label_float,
                         int64_t npix, int C, int activation, float thresh, int64_t* counts,
                         void* stream);
int atomai_b200_iou_finalize(const int64_t* counts, int nc, float* iou, void* stream);

/* ---- optimizer --------------------------------------------------------------
 * torch.optim.Adam step over a table of tensors (trainers/trainer.py:207,539).
 * table: n rows of {param*, grad*, exp_avg*, exp_avg_sq*, numel} packed as int64[5]. */
int atomai_b200_adam_multi(const int64_t* table_dev, int n, int64_t max_numel, float lr,
                           float beta1, float beta2, float eps, float weight_decay, int step,
                           float grad_scale, void* stream);

/* ---- VAE / rVAE ---------------------------------------------------------------
 * Skinny Linear layers of convEncoderNet/convDecoderNet/SignalEncoder
 * (atomai/nets/ed.py:64,273-274,503-505): y[B][O] = x[B][K] W[O][K]^T + b. */
int atomai_b200_linear_fwd(const float* x, const float* w, const float* b, float* y, int B,
                           int K, int O, void* stream);
/* dx[B][K] = dy[B][O] W[O][K] (nullable) ; dW[O][K] = dy^T x ; db[O] = sum_B dy */
int atomai_b200_linear_bwd(const float* x, const float* w, const float* dy, float* dx,
                           float* dw, float* db, int B, int K, int O, void* stream);
/* General strided fp32 GEMM used by the skinny/odd-shaped Linear layers:
 *   C[m][n] (+)= act( sum_k A[m*a_sm + k*a_sk] * B[k*b_sk + n*b_sn] + bias[n] )
 * accumulate = 1 adds to C (C += act(A.B + bias)), 0 overwrites it.  split_k > 1
 * distributes K over CTAs with atomic accumulation (then act must be identity); the
 * effective split also depends on K (K <= 16 always runs as one split), and both
 * give the same result up to the order of the fp32 sums.  A and B may be NULL when
 * K = 0 (C (+)= act(bias)). */
int atomai_b200_gemm(const float* A, int64_t a_sm, int64_t a_sk, const float* B, int64_t b_sk,
                     int64_t b_sn, float* C, int64_t c_sm, int M, int N, int K, const float* bias,
                     int act, float slope, int accumulate, int split_k, void* stream);
/* coord_latent + transform_coordinates fused (atomai/nets/ed.py:672-687,
 * atomai/utils/coords.py:47-83, models/dgm/rvae.py:118-145): the (B,HW,2) coordinate
 * grid is generated on the fly from (phi, dx) and never materialised.
 *   h0[b*HW + p][:] = act( Wc @ (R(phi_b) g_p + dx_b) + bc + Wz @ z_b ),  act = tanh or id */
typedef struct {
  int32_t B, H, W, zdim, hid, tanh_act;
  const float* z;   /* [B][zdim]                                   */
  const float* phi; /* [B] or NULL                                 */
  const float* dx;  /* [B][2] or NULL                              */
  const float* wc;  /* [hid][2]    coord_latent.fc_coord.weight    */
  const float* bc;  /* [hid]       coord_latent.fc_coord.bias      */
  const float* wz;  /* [hid][zdim] coord_latent.fc_latent.weight   */
} ab_coordlat_t;
int atomai_b200_coord_latent_fwd(const ab_coordlat_t* d, float* h0, void* stream);
/* dpre0: gradient w.r.t. the pre-activation of h0 [B*HW][hid]; every output accumulates
 * (caller zeroes): dwc[hid][2], dbc[hid], sb[B][hid] (= sum_p dpre0, for dWz / dz via
 * atomai_b200_gemm), dphi[B], ddx[B][2] (either may be NULL). */
int atomai_b200_coord_latent_bwd(const ab_coordlat_t* d, const float* dpre0, float* dwc,
                                 float* dbc, float* sb, float* dphi, float* ddx, void* stream);
/* ELBO pieces (atomai/losses_metrics/vi_losses.py:13-57,77-137):
 * out[0] = sum_b 0.5*sum_px (xhat-x)^2 ; dxhat = (xhat - x)*gscale (nullable). */
int atomai_b200_sqerr_reduce(const float* x, const float* xhat, int64_t n, double* out,
                             float* dxhat, float gscale, const float* gscale_dev, void* stream);

/* ---- joint (continuous + Gumbel-softmax) latent block of jVAE / jrVAE ------------------------
 * (atomai/models/dgm/jvae.py:103-131, jrvae.py:117-151, trainers/vitrainer.py:236-248,
 * losses_metrics/vi_losses.py:40-84,140-221).  Per row b of B, with D = sum of the head sizes:
 *   alpha = softmax(logits) per head (fp32, max subtracted)
 *   z     = mu + exp(logsd) * eps                                   (Dc continuous columns)
 *   g     = -log(-log(u + 1e-12) + 1e-12),  u = caller's uniform or hash(seed, b*D + j)
 *   zd    = softmax((log(alpha + 1e-12) + g) / tau) per head
 *   zdec  = [z[coord:], zd]  (B x (Dc - coord + D): the decoder input),  phi = z[:, 0] and
 *           dx = z[:, 1:3] * dx_prior when coord is 1 / 3 (rDecoderNet's rotation / translation)
 *   kl[0] = mean_b kld_normal(z columns coord>0 ? 1.. : 0..) + (coord ? mean_b kld_rot(logsd[:,0]) : 0)
 *   kl[1] = sum_heads mean_b sum_j alpha (log(alpha + 1e-12) - log(1/D_h + 1e-12))
 * The KL sums run in fp64 in a fixed order in one CTA (no atomics): one input, one output bit
 * pattern.  Limits: 1 <= Dc <= 32, coord in {0, 1, 3} < Dc, 1 <= D <= 64 (any number of heads).
 * mode AB_JLAT_ALPHAS computes alpha only (mu, logsd, eps, u, zdec, phi, dx, kl unused). */
#define AB_JLAT_MAX_CONT 32
#define AB_JLAT_MAX_DISC 64
#define AB_JLAT_ALPHAS 0
#define AB_JLAT_SAMPLE 1
typedef struct {
  int32_t B, Dc, coord, nheads;
  int32_t heads[AB_JLAT_MAX_DISC]; /* head sizes D_1..D_nheads */
  float tau, phi_prior, dx_prior;
} ab_jlat_t;
/* u: [B][D] or NULL (then the hash generator with `seed`); phi, dx: [B], [B][2] when coord > 0;
 * kl: float[2] or NULL */
int atomai_b200_jlatent_fwd(const ab_jlat_t* d, int mode, const float* mu, const float* logsd,
                            const float* logits, const float* eps, const float* u, uint64_t seed,
                            float* alpha, float* zdec, float* phi, float* dx, float* kl,
                            void* stream);
/* Gradients of the forward above (same inputs, same noise) from dzdec, dphi, ddx, dalpha and
 * gkl = d loss / d kl[0..1] (each nullable = zero); overwrites dmu, dlogsd ([B][Dc], unused in
 * mode AB_JLAT_ALPHAS) and dlogits ([B][D]). */
int atomai_b200_jlatent_bwd(const ab_jlat_t* d, int mode, const float* mu, const float* logsd,
                            const float* logits, const float* eps, const float* u, uint64_t seed,
                            const float* dzdec, const float* dphi, const float* ddx,
                            const float* dalpha, const float* gkl, float* dmu, float* dlogsd,
                            float* dlogits, void* stream);

/* ---- DKL ----------------------------------------------------------------------
 * Dense Gram K[i][j] = os * k(||(x1_i - x2_j) * inv_ls||), kind 0 = RBF,
 * 1 = Matern-2.5 (gpytorch RBFKernel/MaternKernel/ScaleKernel as configured at
 * atomai/nets/gp.py:41-46, :100-111).  x: [n][d] row-major fp32, inv_ls: [d].
 * math: AB_MATH_TF32 / AB_MATH_TF32X3 run the contraction on the tensor-core convolution kernel
 * with the exponentiation in its register epilogue, AB_MATH_FP32 on exact FFMA tiles.
 * `workspace` (256 B aligned, >= atomai_b200_gram_workspace_bytes) is caller-owned scratch
 * for the scaled/augmented operands; the library allocates nothing. */
int64_t atomai_b200_gram_workspace_bytes(int n1, int n2, int d);
int atomai_b200_gram(const float* x1, const float* x2, const float* inv_ls, float outputscale,
                     int n1, int n2, int d, int kind, int math, float* K, int64_t ldk,
                     void* workspace, int64_t workspace_bytes, void* stream);
/* GP predictive mean without the cross-Gram (csrc/gpr.cu):
 *   y[i] = c + outputscale * sum_j k(||(xq_i - x_j) * inv_ls||) * alpha_j
 * for nq query points xq: [nq][d] against n training points x: [n][d] (fp32, row-major),
 * inv_ls: [d], 1 <= d <= 4, kind as atomai_b200_gram.  alpha: [n] and y: [nq] are double.  k is
 * evaluated in fp32 from the coordinate differences; each y[i] is accumulated in double in a fixed
 * order of j that does not depend on nq, so a query gets identical bits however the queries are
 * batched.  The nq x n matrix is never formed. */
int atomai_b200_gram_matvec(const float* xq, const float* x, const float* inv_ls,
                            const double* alpha, double c, double outputscale, int nq, int n, int d,
                            int kind, double* y, void* stream);
/* Exact-GP training Gram in double (csrc/gpr.cu): K[i][j] = outputscale * k(||(x_i - x_j) * inv_ls||)
 * + noise [i == j] for x: [n][d] double, 1 <= d <= 4, kind as atomai_b200_gram, from coordinate
 * differences (exactly symmetric, no norm-expansion cancellation).  K: [n][ldk] double. */
int atomai_b200_gram_f64(const double* x, const double* inv_ls, double outputscale, double noise,
                         int n, int d, int kind, double* K, int64_t ldk, void* stream);
/* Its adjoint for an upstream gradient G: [n][ldg] double, with t_ijk = (x_ik - x_jk) inv_ls_k,
 * k_ij = k(r_ij^2) and m_ij = -2 dk/dr^2 (RBF: k; Matern-2.5: 5/3 (1 + s) exp(-s)):
 * out[k] = sum_ij G_ij m_ij t_ijk^2 (k < d), out[d] = sum_ij G_ij k_ij, out[d + 1] = sum_i G_ii,
 * i.e. dL/dls_k = os out[k] / ls_k, dL/dos = out[d], dL/dnoise = out[d + 1].  Double sums in a
 * fixed order (bit-identical on repeat). */
int atomai_b200_gram_f64_adjoint(const double* x, const double* inv_ls, int n, int d, int kind,
                                 const double* G, int64_t ldg, double* out, void* stream);

/* ---- prediction front-end / data path (SURVEY.md 8f) -----------------------------
 * prob[p][c] = softmax_c(logits[p][:]) (mode 0) | sigmoid (1) | exp (2) | identity (3) over NHWC
 * pixels, and mask[p][c] = prob > thresh (uint8, nullable): SegPredictor.forward_ +
 * cv_thresh in one pass (atomai/predictors/predictor.py:209-231, atomai/utils/img.py:554-564). */
int atomai_b200_prob_mask(const float* logits, int ld, int64_t npix, int C, int mode, float thresh,
                          float* prob, int ld_p, uint8_t* mask, void* stream);
/* out[k] = img[f_k, sx_k:sx_k+r, sy_k:sy_k+r, :] for the K rows {f, sx, sy} of `table` (int32,
 * device); nanflag[k] = 1 if the window holds a NaN (nullable; caller zeroes).  Sub-image
 * extraction of atomai/utils/img.py:138-180, 298-350 as one gather. */
int atomai_b200_gather_windows(const float* img, int n, int h, int w, int c, const int32_t* table,
                               int K, int r, float* out, int32_t* nanflag, void* stream);
/* out[k] = the ph x pw x c window of a row-major image whose rows hold w * c elements, starting at
 * element offs[k] (int64, device), for the K windows; a bit copy of elements of elem_bytes in
 * {1, 2, 4, 8}.  The patches of extract_patches_ (atomai/utils/img.py:353-389), whose offsets
 * are drawn on the host. */
int atomai_b200_gather_patches(const void* img, int elem_bytes, int w, int c, const int64_t* offs,
                               int K, int ph, int pw, void* out, void* stream);
/* ---- lattice masks of utils.imgen (atomai/utils/imgen.py:82-229) ------------------------------
 * atoms: K rows of AB_IMGEN_ATOM_INTS int32 {frame, channel, r0, c0, nr, nc, tpl, sr, sc}: the
 * atom's clamped slice rows r0 .. r0+nr-1, columns c0 .. c0+nc-1, and its template element for
 * slice pixel (i, j) at tpl + i * sr + j * sc (stride 0 broadcasts).  frames: F rows of
 * AB_IMGEN_FRAME_INTS int64 {h, w, C, out offset, owner offset}, offsets in elements; the frame's
 * owner map is C planes of h x w int32 and its output h x w x (C [+ 1]) elements.
 * imgen_owner: owner[pixel] = max(owner, atom + 1) over each atom's slice (caller zeroes owner).
 * imgen_fill: every class channel of every pixel = the bits of its owner's template element, or 0;
 * background = 1: float64, a last channel 1 - sum of the class channels (numpy's pairwise order,
 * recursive above 128 channels), then every negative value set to 0.  max_pix = the largest h * w. */
#define AB_IMGEN_ATOM_INTS 9
#define AB_IMGEN_FRAME_INTS 5
int atomai_b200_imgen_owner(const int32_t* atoms, int K, const int64_t* frames, int32_t* owner,
                            void* stream);
int atomai_b200_imgen_fill(const int32_t* atoms, const int64_t* frames, int F, int64_t max_pix,
                           const int32_t* owner, const void* tpl, int elem_bytes, int background,
                           void* out, void* stream);
/* ---- blob filtering of utils.filter_cells[_] (atomai/utils/img.py:567-625) --------------------
 * For every frame of the row-major (n, h, w) stack `img` (h * w < 2^31): a pixel is foreground
 * when img > im_thresh (float32 pixels against (float)im_thresh, the others in double; NaN is
 * background); the 4-connected components of the foreground are labelled; a component is dropped
 * when its pixel count c has c > blob_thresh (above != 0) or c < blob_thresh (above == 0), compared
 * in double, so a NaN blob_thresh keeps every component; out = 1 on the pixels of kept components,
 * 0 elsewhere, in out_dtype.  Frames never join.  labels and counts are caller-owned n * h * w int32
 * workspaces, overwritten: afterwards labels[pixel] is the smallest frame-local linear index of the
 * pixel's component (-1 on the background) and counts[root] the component's size at that index.
 * dtype: AB_BLOB_U8 .. AB_BLOB_F64; out_dtype: any AB_BLOB_* code.  All passes run on `stream`. */
#define AB_BLOB_U8 0
#define AB_BLOB_I16 1
#define AB_BLOB_U16 2
#define AB_BLOB_F32 3
#define AB_BLOB_F64 4
#define AB_BLOB_I32 5
int atomai_b200_blob_filter(const void* img, int dtype, int64_t n, int h, int w, double im_thresh,
                            double blob_thresh, int above, int32_t* labels, int32_t* counts,
                            void* out, int out_dtype, void* stream);
/* ---- 2-D FFTs of utils.FFTmask / FFTsub (atomai/utils/img.py:455-486) ------------------------
 * float64 complex transforms of one row-major (h, w) array; each side is in [1, AB_FFT_MAX_SIDE]
 * or a power of two up to AB_FFT_MAX_POW2.  Lengths that are not powers of two run by Bluestein's
 * chirp-z method.  `work` is caller-owned device scratch of at least
 * atomai_b200_fft2_workspace_bytes(h, w) bytes (-1 for an unsupported side), 256 B aligned.
 * Element dtypes: AB_FFT_U8 .. AB_FFT_C128 (bool as AB_FFT_U8).  All passes run on `stream`.
 * fft2_mask: F2 = fftshift(fft2(img)); F3 = F2 except F3 = F2 * (1 - disk) at (r0 + y, c0 + x),
 *   0 <= x, y < 2l, disk = (x + 1 - l)^2 + (y + 1 - l)^2 <= l^2 (l = 0: F3 = F2).  f2 and f3 are
 *   (h, w) complex64 (c64 != 0, each component rounded once) or complex128.
 * fft2_sub: recon = Re(ifft2(ifftshift(spec))) with the 1 / (h w) scale, spec complex64 or
 *   complex128; d = |img - recon|; out = (d - min d) / (max d - min d) in float64 (NaN-propagating
 *   extremes, a constant d gives NaN), stored as float32 (out_f32 != 0) or float64. */
#define AB_FFT_U8 0
#define AB_FFT_I8 1
#define AB_FFT_I16 2
#define AB_FFT_U16 3
#define AB_FFT_I32 4
#define AB_FFT_U32 5
#define AB_FFT_I64 6
#define AB_FFT_U64 7
#define AB_FFT_F16 8
#define AB_FFT_F32 9
#define AB_FFT_F64 10
#define AB_FFT_C64 11
#define AB_FFT_C128 12
#define AB_FFT_MAX_SIDE 4096
#define AB_FFT_MAX_POW2 8192
int64_t atomai_b200_fft2_workspace_bytes(int h, int w);
int atomai_b200_fft2_mask(const void* img, int dtype, int h, int w, int r0, int c0, int l,
                          void* f2, void* f3, int c64, void* work, int64_t work_bytes,
                          void* stream);
int atomai_b200_fft2_sub(const void* img, int img_dtype, const void* spec, int spec_dtype, int h,
                         int w, void* out, int out_f32, void* work, int64_t work_bytes,
                         void* stream);
/* 2-D Gaussian peak refinement (atomai/utils/coords.py:152-231, predictors/predictor.py:609-619):
 * for each of the K rows {frame, row0, col0, d} of `atoms` (int32, device) one least-squares fit of
 *   offset + amp exp(-(a (x-xo)^2 + 2 b (x-xo)(y-yo) + c (y-yo)^2))
 * to the window img[frame, row0:row0+2d, col0:col0+2d] of the fp32 (n, H, W) stack, in fp64, by
 * MINPACK lmdif as scipy.optimize.curve_fit runs it (start (img[d, d], d, d, 1, 1, 0, 0) in window
 * coordinates, maxfev 1600).  popt: K x 7 doubles {amp, xo, yo, sigma_x, sigma_y, theta, offset};
 * info: MINPACK's info (1..8, 0 when (2d)^2 < 7) or one of AB_REFINE_*; nfev (nullable): function
 * evaluations.  row0 < 0 skips an atom.  Every d must lie in [1, dmax], 1 <= dmax <= 16. */
#define AB_REFINE_SKIPPED -1   /* row0 < 0: not fitted                                    */
#define AB_REFINE_NONFINITE -2 /* the window holds a NaN or an infinity                   */
#define AB_REFINE_BAD_ATOM -3  /* frame or window outside the stack, or d outside [1, dmax] */
int atomai_b200_peak_refine(const float* img, int n, int H, int W, const int32_t* atoms, int K,
                            int dmax, double* popt, int32_t* info, int32_t* nfev, void* stream);
/* Per-sample VAE reconstruction loss (atomai/losses_metrics/vi_losses.py:13-37) over B rows of D
 * elements: kind 0 out[b] += 0.5*sum (xhat-x)^2, kind 1 out[b] += sum BCE-with-logits(xhat, x)
 * (double, nullable, caller zeroes); dxhat (nullable) = gvec[b] * d loss_b / d xhat. */
int atomai_b200_rowloss(const float* x, const float* xhat, int B, int64_t D, int kind, double* out,
                        float* dxhat, const float* gvec, void* stream);
/* In-place inverted dropout a <- a * m / (1 - p), m = [hash(seed, element index) >= p]
 * (nn.Dropout of ConvBlock, atomai/nets/blocks.py:68-69; the same call with the same seed applies
 * the mask to a gradient).  stats (nullable, double[2C], caller zeroes) receives the per-channel
 * sum and sum of squares of the result. */
int atomai_b200_dropout(float* a, int ld, int64_t npix, int C, float p, uint64_t seed,
                        double* stats, void* stream);

/* On-the-fly augmentation of a batch of (n, h, w) images (+ int64 label maps, nullable) entirely in
 * HBM: the reference's datatransform sequence (atomai/transforms/imaug.py:109-358) as three passes.
 * params: n x 16 floats per image {flip code, gauss var, poisson vals, s&p amount, blur sigma,
 * gamma, background amp, x0, y0, a*ln2/fwhm^2, b*ln2/fwhm^2, ...} drawn by the caller; row_shift
 * (nullable): n x h jitter roll amounts; scratch: n*h*w floats; minmax: 2 floats (device). */
int atomai_b200_augment(const float* x, float* y, float* scratch, const int64_t* lab_in,
                        int64_t* lab_out, const float* params, const int32_t* row_shift, int n,
                        int h, int w, float in_min, float in_max, uint64_t seed, float* minmax,
                        void* stream);

/* ---- k-means and Gaussian-mixture EM over a sub-image stack (csrc/stat.cu) ---------------------
 * X: N x d fp32 row-major; mu (d): the column mean, subtracted on every load (X is never copied);
 * 1 <= K <= 64 components.  Row sums go through the ordered per-CTA slots: identical bits on repeat.
 * estep: s_nk = sum_j A_kj x_nj (+ B_kj x_nj^2 in mode 0) on centred rows, then per mode
 *   0 GMM:     l_nk = s_nk + cst_k; resp (N x K, nullable) = softmax_k l, labels (nullable) = argmax,
 *              out[0] = sum_n logsumexp_k l_nk;
 *   1 k-means: dist_nk = ||x_n||^2 + s_nk + cst_k; labels (in: previous labels, out: first argmin),
 *              rowval (nullable) = min distance, out[0] = sum of min distances, *changes (nullable)
 *              += number of rows whose label changed;
 *   2 k-means++ candidates: D (N x K) = dist, out[k] = sum_n min(closest_n, D_nk).
 * accum: sx (K x d) = sum_n r_nk x_n, sxx (K x d, nullable) = sum_n r_nk x_n^2, nk (K, nullable) =
 *   sum_n r_nk (float64) with r = resp (N x K) if given, else one-hot labels if given, else r_n0 = 1
 *   (mu may be NULL: raw X).
 * gmm_params: sklearn's diag (spherical = 0) / spherical M-step from accum's sums of centred X:
 *   nk + 10 eps, means, covs (K x d or K, + reg_covar), weights (nk / N if init, else normalised),
 *   and the E-step operands A = means * prec, B = -prec / 2, cst = log N(0) constant + log weight.
 * kmeans_centres: c_new = sx / nk (empty clusters keep c_old), *shift = sum ||c_new - c_old||^2;
 *   sx == NULL: c_new holds the centres already.  Both form A = -2 c, cst = ||c||^2.
 * kpp_candidates: ntr <= 32 indices drawn with hash_uniform(counter + t, seed): proportional to
 *   closest (numpy searchsorted over its fixed-order prefix sum), uniform if closest == NULL;
 *   chunk_ws: atomai_b200_stat_kpp_chunks(N) doubles.
 * estep / accum `math` (AB_MATH_*): FP32 exact FFMA kernels; TF32 / TF32X3 the wgmma kernels
 *   (TF32X3: split operands, three MMAs per product).
 * gather_rows: out (n x d) = X[idx] - mu.  kpp_commit: best = first argmin of pot (ntr),
 *   closest = min(closest, D[:, best]), centre (d) = cand[best]. */
int atomai_b200_stat_estep(const float* X, const float* mu, int N, int d, int K, int mode,
                           const float* A, const float* B, const float* cst, const float* closest,
                           float* resp, int* labels, float* rowval, float* D, double* out,
                           double* changes, int math, void* stream);
int atomai_b200_stat_accum(const float* X, const float* mu, int N, int d, int K, const float* resp,
                           const int* labels, double* sx, double* sxx, double* nk, int math,
                           void* stream);
int atomai_b200_stat_gmm_params(const double* sx, const double* sxx, const double* nk, int N, int d,
                                int K, int spherical, double reg_covar, int init, float* means,
                                float* covs, float* weights, float* A, float* B, float* cst,
                                void* stream);
int atomai_b200_stat_kmeans_centres(const double* sx, const double* nk, const float* c_old,
                                    float* c_new, int K, int d, float* A, float* cst, double* shift,
                                    void* stream);
int64_t atomai_b200_stat_kpp_chunks(int N);
int atomai_b200_stat_kpp_candidates(const float* closest, int N, int ntr, uint64_t seed,
                                    uint64_t counter, double* chunk_ws, int* idx, void* stream);
int atomai_b200_stat_gather_rows(const float* X, const float* mu, int d, const int* idx, int n,
                                 float* out, void* stream);
int atomai_b200_stat_kpp_commit(const float* D, int ntr, const double* pot, float* closest, int N,
                                const float* cand, int d, float* centre, void* stream);

/* ---- PCA / NMF / FastICA passes over a sub-image stack (csrc/decomp.cu) ----------------------
 * X: N x d fp32 row-major, read in place; mu (d, nullable): subtracted on every load.  Exact fp32
 * FFMA for the contractions over X, float64 for everything else; the set_math mode does not apply.
 * Row sums go through the ordered per-CTA slots: identical bits on repeat.  1 <= K <= 64.
 * gram: rows = 0: G (d x d) = (X - mu)^T (X - mu); rows = 1: G (N x N) = (X - mu)(X - mu)^T;
 *   float64, exactly symmetric (upper-triangle tiles, mirrored).
 * project: out[n * ldo + k] = sum_j (X_nj - mu_j) B_kj for the K rows of B (K x d fp32).
 * nmf_w: one coordinate-descent sweep (sklearn's _update_cdnmf_fast, Frobenius, no regularisation)
 *   of W (N x K fp32, in place) against H (K x d fp32) and HHt (K x K float64), with XHt = X H^T
 *   formed per row tile; out (K * K + 1 doubles) = [W^T W of the updated W, violation].
 * nmf_h: the same sweep of H (K x d, in place) from WtX (K x d float64, sum_n W_nk X_n:
 *   atomai_b200_stat_accum with resp = W, mu = NULL) and WtW (K x K); out = [H H^T, violation].
 * ica_step: X1 (N x K fp32 row-major: the whitened samples), W (K x K float64); with
 *   g = tanh(W x1) per sample, out (K * K + K doubles) = [sum_n g x1^T, sum_n (1 - g^2)].
 * slot_doubles: the ordered-slot workspace (doubles) a call takes, op 0/1 gram (rows = op),
 *   2 nmf_w, 3 nmf_h, 4 ica_step; -1 for bad arguments. */
int64_t atomai_b200_decomp_slot_doubles(int op, int N, int d, int K);
int atomai_b200_decomp_gram(const float* X, const float* mu, int N, int d, int rows, double* G,
                            void* stream);
int atomai_b200_decomp_project(const float* X, const float* mu, int N, int d, int K, const float* B,
                               float* out, int ldo, void* stream);
int atomai_b200_decomp_nmf_w(const float* X, int N, int d, int K, const float* H, const double* HHt,
                             float* W, double* out, void* stream);
int atomai_b200_decomp_nmf_h(const double* WtX, const double* WtW, int d, int K, float* H,
                             double* out, void* stream);
int atomai_b200_decomp_ica_step(const float* X1, int N, int K, const double* W, double* out,
                                void* stream);

/* ---- bond graphs and rings of atomic lattices (csrc/graph.cu) --------------------------------
 * pos: N x 3 float64 (Å); cls (N int32, nullable = all 0) indexes the C x C float64 cutoff table
 * `cut`; frame (N int32, nullable = all 0) keeps the frames of a batch apart.  Grid: cell side
 * `side` (>= every cutoff), origin lo_host[3] and dims_host[3] cells (HOST arrays).
 * cell_keys: keys[i] = ((frame * nz + cz) * ny + cy) * nx + cx; the caller sorts them stably
 *   (keys ascending, perm = the atom of each sorted key, int64).
 * bonds: rowptr == NULL: out[i] = degree of i; else out[rowptr[i] ...] = the atoms bonded to i,
 *   ascending.  Bonded: i != j and |p_i - p_j| <= cut[cls_i * C + cls_j].
 * hops: one level of the hop table.  Rows bptr/ball hold packed words (id << 5 | hops), sorted;
 *   level 0 is {u << 5} per atom.  optr == NULL: cnt[u] = length of u's next-level row (the union of
 *   u's row and its bonded atoms' rows + 1 hop, least hops per id); else out[optr[u] ...] = that
 *   row.  N < 2^26.
 * rings: the hop table of radius max_depth / 2 in bptr/ball; 3 <= max_depth <= AB_GRAPH_MAX_RING.
 *   ring_base == NULL: cnt[3 r ...] = (rings, their atoms, search steps) of root r; else root r's
 *   rings in discovery order go to lens[ring_base[r] ...] and atoms[atom_base[r] ...].
 * ring_filter: keep[r] = 0 when two atoms j < k of ring r (atoms[off[r] ...], lens[r] atoms) are
 *   fewer than min(k - j, lens[r] - k + j) hops apart, else 1. */
#define AB_GRAPH_MAX_RING 32
int atomai_b200_graph_cell_keys(const double* pos, const int* frame, int N, const double* lo_host,
                                double side, const int64_t* dims_host, int64_t* keys,
                                void* stream);
int atomai_b200_graph_bonds(const double* pos, const int* cls, const int* frame, int N,
                            const int64_t* keys, const int64_t* perm, const double* cut, int C,
                            const double* lo_host, double side, const int64_t* dims_host,
                            const int64_t* rowptr, int* out, void* stream);
int atomai_b200_graph_hops(const int64_t* rowptr, const int* cols, int N, const int64_t* bptr,
                           const uint32_t* ball, const int64_t* optr, uint32_t* out, int64_t* cnt,
                           void* stream);
int atomai_b200_graph_rings(const int64_t* rowptr, const int* cols, int N, const int64_t* bptr,
                            const uint32_t* ball, int max_depth, const int64_t* ring_base,
                            const int64_t* atom_base, int* lens, int* atoms, int64_t* cnt,
                            void* stream);
int atomai_b200_graph_ring_filter(const int64_t* off, const int* lens, const int* atoms,
                                  int64_t R, const int64_t* bptr, const uint32_t* ball,
                                  unsigned char* keep, void* stream);

/* ---- neighbour searches of atomic coordinates (csrc/coords.cu) ------------------------------
 * pos: N x 3 float64, binned by graph_cell_keys into the grid (lo_host, side, dims_host; HOST
 * arrays) with keys / perm the stably sorted keys and the atom of each.  foff (F + 1 int64) holds
 * the first sorted key of every frame; the atoms of a batch are stored frame by frame.  Distances
 * are float64, unfused; an equal distance goes to the lower index.  Every query comes with its
 * cell (3 int64), which coords_cells writes for N points of the same grid.
 * knn: the k nearest atoms with d < ub (ub = +inf: no bound) of query i (qpos Q x 3) in frame
 *   qframe[i] (nullable with foff = NULL: one frame of N atoms): oidx / odist (Q x k) ascending,
 *   -1 / +inf where fewer are found.  1 <= k <= AB_COORDS_MAX_K.
 * ball: the atoms with d < rmax of every query (side >= rmax, one frame).  rowptr == NULL:
 *   cnt[i] = their number; else oidx / odist[rowptr[i] ...] = them, in scan order.
 * walk: for start s (start S x 3 with z = 0, cells scell) and frame f = 0 ... F-1 (atom cells
 *   pcell): the nearest atom j of
 *   frame f with d < rmax to the walk's position; out[(s F + f) 4 ...] = (f, j, row0, col0) when
 *   numpy's slice [cx - half : cx + half, cy - half : cy + half] of an H x W image, cx, cy the
 *   half-to-even rounded (x, y) of j, is r x r (the walk then moves to j), else (f, -1, -1, -1).
 * dbscan_roots: parent[i] = the least core index of i's component for a core point of the CSR
 *   (rowptr, cols) neighbourhoods (row length + 1 >= min_samples), -1 otherwise.  flag: 1 int of
 *   device scratch.  Synchronises the stream once per round.
 * dbscan_labels: labels[i] = rank[root] of i's root, or of the least root among a border point's
 *   core neighbours, else -1. */
#define AB_COORDS_MAX_K 32
int atomai_b200_coords_cells(const double* pos, int N, const double* lo_host, double side,
                             const int64_t* dims_host, int64_t* cells, void* stream);
int atomai_b200_coords_knn(const double* qpos, const int64_t* qcell, const int* qframe, int Q,
                           const double* pos, int N, const int64_t* keys, const int64_t* perm,
                           const int64_t* foff, const double* lo_host, double side,
                           const int64_t* dims_host, int k, double ub, int* oidx, double* odist,
                           void* stream);
int atomai_b200_coords_ball(const double* qpos, const int64_t* qcell, int Q, const double* pos,
                            int N, const int64_t* keys, const int64_t* perm,
                            const double* lo_host, double side, const int64_t* dims_host,
                            double rmax, const int64_t* rowptr, int* oidx, double* odist,
                            int64_t* cnt, void* stream);
int atomai_b200_coords_walk(const double* start, const int64_t* scell, int S, const double* pos,
                            const int64_t* pcell, const int64_t* keys, const int64_t* perm,
                            const int64_t* foff, int F, const double* lo_host, double side,
                            const int64_t* dims_host, double rmax, int64_t H, int64_t W,
                            int64_t half, int64_t r, int* out, void* stream);
int atomai_b200_coords_dbscan_roots(const int64_t* rowptr, const int* cols, int N,
                                    int min_samples, int* parent, int* flag, void* stream);
int atomai_b200_coords_dbscan_labels(const int64_t* rowptr, const int* cols, int N,
                                     const int* parent, const int64_t* rank, int64_t* labels,
                                     void* stream);

/* ---- multi-GPU: small all-reduce over NVLink peer memory (csrc/p2p.cu) -----------------
 * Every rank exposes a zero-initialised mailbox (atomai_b200_p2p_data_bytes) and flag buffer
 * (atomai_b200_p2p_flag_bytes) to its peers (CUDA IPC: atomai_b200_ipc_export gives the 64-byte
 * handle of the enclosing allocation + the offset inside it, atomai_b200_ipc_import maps it for the
 * current device with peer access); data_ptrs / flag_ptrs are HOST arrays of
 * the `world` mapped device pointers in rank order.  All ranks call with the same, strictly
 * increasing `epoch`.  allreduce: vals[0:n] <- sum over ranks (n <= 1024 doubles).
 * bn_finalize: the same exchange fused with atomai_b200_bn_finalize(training = 1) —
 * synchronised BatchNorm statistics without an NCCL launch per layer. */
int atomai_b200_ipc_export(const void* ptr, unsigned char* handle64, int64_t* offset);
int atomai_b200_ipc_import(const unsigned char* handle64, int64_t offset, void** ptr_out);
int64_t atomai_b200_p2p_data_bytes(int world);
int64_t atomai_b200_p2p_flag_bytes(int world);
int atomai_b200_p2p_allreduce(void* const* data_ptrs_host, void* const* flag_ptrs_host, int world,
                              int rank, uint64_t epoch, double* vals, int n, void* stream);
int atomai_b200_p2p_bn_finalize(void* const* data_ptrs_host, void* const* flag_ptrs_host, int world,
                                int rank, uint64_t epoch, double* stats, int C, double count,
                                const float* gamma, const float* beta, float* running_mean,
                                float* running_var, float momentum, float eps, float* scale,
                                float* shift, float* mean, float* invstd, void* stream);

/* ---- self-test hooks (tests only) ------------------------------------------------ */
/* TMA probe (dev only): one cp.async.bulk.tensor of a {32 ch, TWp, THp, 1} box at (c0, w0, h0, n0)
 * of an NHWC fp32 tensor (out-of-range coordinates are zero-filled) into shared memory at
 * `smem_offset` past a 1024 B boundary, swizzle_mode 0 none / 1 32B / 2 64B / 3 128B /
 * 4 128B_ATOM_32B; `out` receives the raw shared-memory image (TWp*THp*32 floats). */
int atomai_b200_selftest_tma(const float* x, int N, int H, int W, int C, int c0, int w0, int h0,
                             int n0, int TWp, int THp, int swizzle_mode, int smem_offset,
                             float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ATOMAI_B200_H */
