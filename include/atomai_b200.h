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
 * cross-CTA sums, C <= 16, 2*C*ceil(W/32)*32 <= 2^21).  dice_finalize: loss[0] = 1 - mean 2I/(S+eps)
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
 * split_k > 1 distributes K over CTAs with atomic accumulation (then act must be
 * identity and C pre-initialised, e.g. with the bias). */
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
