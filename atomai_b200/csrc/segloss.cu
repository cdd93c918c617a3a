// segloss.cu — the segmentation objectives beyond cross-entropy:
//   dice      Sørensen–Dice loss (atomai/losses_metrics/losses.py:53-89): per-cell sums
//             I = sum p*t, S = sum (p + t) in one pass over the logits, a one-CTA finalise of the
//             loss and of the per-cell backward coefficients, and an elementwise backward that
//             recomputes the softmax / sigmoid
//   focal     focal loss (losses.py:13-50) is a scalar function of the mean BCE-with-logits; the
//             BCE sum and its gradient come from pointwise_loss (elementwise.cu), only the scalar
//             transform and its derivative factor live here
//   IoU       mean Intersection over Union (atomai/losses_metrics/metrics.py:16-95): thresholded
//             class decision + confusion histogram in one pass, finalised on the device
// All HBM-bound; the logits are read where the network leaves them (NHWC, pixel stride ld).
#include "common.cuh"

namespace {

constexpr int kT = 256;
constexpr int kCols = 32;                  // image columns per dice CTA (one per lane)
constexpr int kLanes = kT / kCols;         // rows processed side by side (one per warp)
constexpr int64_t kDiceWsDoubles = 1 << 21;  // cap of the dice partials: 16 MB per stream

// the class decision of SegPredictor / Locator: prob > thresh with the arithmetic of
// prob_mask_kernel (frontend.cu), so that predict() and the accuracy agree on every pixel
__device__ __forceinline__ float softmax_max(const float* x, int C) {
  float mx = x[0];
  for (int c = 1; c < C; ++c) mx = fmaxf(mx, x[c]);
  return mx;
}
__device__ __forceinline__ float softmax_den(const float* x, int C, float mx) {
  float s = 0.f;
  for (int c = 0; c < C; ++c) s += expf(x[c] - mx);
  return s;
}
__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + expf(-x)); }

__device__ __forceinline__ int64_t label_at(const void* labels, int label_float, int64_t p) {
  // true.long() of the reference: float labels truncate toward zero
  return label_float ? (int64_t)__ldg(static_cast<const float*>(labels) + p)
                     : __ldg(static_cast<const int64_t*>(labels) + p);
}

// ---------------------------------------------------------------- dice, multi-class
// labels (N, H, W): the reference sums over dims (0, 2) of the (N, C, H, W) product, so there is
// one (I, S) cell per (class, image column).  CTA (bx, by): columns [32 bx, 32 bx + 32) of the row
// chunk by; lane = column, warp = row phase.  Per-thread float sums live in shared memory
// (thread-private), the 8 warps are added in warp order, and the CTA's 2 C x 32 partials go to
// slot `by` of group `bx` of an ordered cross-CTA sum.
__global__ void __launch_bounds__(kT) dice_sums_kernel(const float* __restrict__ logits, int ld,
                                                       const void* __restrict__ labels,
                                                       int label_float, int rows, int W, int C,
                                                       double* __restrict__ cells, Ordered red) {
  extern __shared__ float s_acc[];         // [2][C][kT]: I then S
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int w = blockIdx.x * kCols + lane;
  for (int i = threadIdx.x; i < 2 * C * kT; i += kT) s_acc[i] = 0.f;
  __syncthreads();
  const int r0 = (int)((int64_t)rows * blockIdx.y / gridDim.y);
  const int r1 = (int)((int64_t)rows * (blockIdx.y + 1) / gridDim.y);
  if (w < W) {
    for (int r = r0 + warp; r < r1; r += kLanes) {
      const int64_t p = (int64_t)r * W + w;
      const float* x = logits + p * ld;
      const int64_t y = label_at(labels, label_float, p);
      const float mx = softmax_max(x, C);
      const float inv = 1.f / softmax_den(x, C, mx);
      for (int c = 0; c < C; ++c) {
        const float pr = expf(x[c] - mx) * inv;
        const float t = (y == c) ? 1.f : 0.f;
        s_acc[c * kT + threadIdx.x] += pr * t;
        s_acc[(C + c) * kT + threadIdx.x] += pr + t;
      }
    }
  }
  __syncthreads();
  const int n = 2 * C * kCols;
  double* slot = ordered_slot(red, blockIdx.x, gridDim.y, blockIdx.y, n);
  for (int i = threadIdx.x; i < n; i += kT) {
    const int kc = i / kCols, l = i - kc * kCols;
    float s = 0.f;
    for (int q = 0; q < kLanes; ++q) s += s_acc[kc * kT + q * kCols + l];
    slot[i] = (double)s;
  }
  __shared__ unsigned s_last;
  const int K = C * W;
  ordered_finish(red, blockIdx.x, gridDim.y, n, threadIdx.x, kT, gridDim.y, [] { __syncthreads(); },
                 [&](int i, double v) {
                   const int kc = i / kCols, l = i - kc * kCols;
                   const int k = kc / C, c = kc - k * C;
                   const int ww = blockIdx.x * kCols + l;
                   if (ww < W) cells[k * K + c * W + ww] = v;
                 },
                 &s_last);
}

// ---------------------------------------------------------------- dice, binary
// one logit channel, labels (N, 1, H, W): probabilities [sigmoid, 1 - sigmoid], targets
// [y == 1, y == 0], dims (0, 2, 3) -> two cells
__global__ void __launch_bounds__(kT) dice_sums_bin_kernel(const float* __restrict__ logits, int ld,
                                                           const void* __restrict__ labels,
                                                           int label_float, int64_t npix,
                                                           double* __restrict__ cells,
                                                           Ordered red) {
  float a[4] = {0.f, 0.f, 0.f, 0.f};  // I0, I1, S0, S1
  for (int64_t p = blockIdx.x * (int64_t)kT + threadIdx.x; p < npix; p += (int64_t)gridDim.x * kT) {
    const float s = sigmoid_f(logits[p * ld]);
    const int64_t y = label_at(labels, label_float, p);
    const float t0 = y == 1 ? 1.f : 0.f, t1 = y == 0 ? 1.f : 0.f;
    const float q = 1.f - s;
    a[0] += s * t0;
    a[1] += q * t1;
    a[2] += s + t0;
    a[3] += q + t1;
  }
  __shared__ float wred[4][kT / 32];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float v = warp_sum(a[k]);
    if ((threadIdx.x & 31) == 0) wred[k][threadIdx.x >> 5] = v;
  }
  __syncthreads();
  if (threadIdx.x < 4) {
    float t = 0.f;
    for (int i = 0; i < kT / 32; ++i) t += wred[threadIdx.x][i];
    ordered_slot(red, 0, gridDim.x, blockIdx.x, 4)[threadIdx.x] = (double)t;
  }
  __shared__ unsigned s_last;
  ordered_finish(red, 0, gridDim.x, 4, threadIdx.x, kT, gridDim.x, [] { __syncthreads(); },
                 [&](int i, double v) { cells[i] = v; }, &s_last);
}

// loss = 1 - mean_k 2 I_k / (S_k + eps); coef[k] = A_k, coef[K + k] = B_k with
// dL/dp = t A + B:  A = -(2/K) / (S + eps),  B = (2/K) I / (S + eps)^2
__global__ void __launch_bounds__(kT) dice_finalize_kernel(const double* __restrict__ cells, int K,
                                                           double eps, float* __restrict__ loss,
                                                           float* __restrict__ coef) {
  double acc = 0.0;
  const double g = 2.0 / K;
  for (int k = threadIdx.x; k < K; k += kT) {
    const double I = cells[k], d = cells[K + k] + eps;
    acc += 2.0 * I / d;
    if (coef) {
      coef[k] = (float)(-g / d);
      coef[K + k] = (float)(g * I / (d * d));
    }
  }
  __shared__ double wred[kT / 32];
  acc = warp_sum_d(acc);
  if ((threadIdx.x & 31) == 0) wred[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < kT / 32; ++i) t += wred[i];
    if (loss) *loss = (float)(1.0 - t / K);
  }
}

// dlogits = g * dL/dlogits: softmax chain dx_j = p_j (G_j - sum_c p_c G_c), sigmoid chain
// dx = s (1 - s) (G_0 - G_1), with G = t A + B of the pixel's cells
__global__ void __launch_bounds__(kT) dice_bwd_kernel(const float* __restrict__ logits, int ld,
                                                      const void* __restrict__ labels,
                                                      int label_float, int64_t npix, int W, int C,
                                                      const float* __restrict__ coef,
                                                      float* __restrict__ dlogits, int ld_d,
                                                      float gscale, const float* gscale_dev) {
  if (gscale_dev) gscale *= __ldg(gscale_dev);
  const int K = C == 1 ? 2 : C * W;
  for (int64_t p = blockIdx.x * (int64_t)kT + threadIdx.x; p < npix; p += (int64_t)gridDim.x * kT) {
    const float* x = logits + p * ld;
    float* d = dlogits + p * ld_d;
    const int64_t y = label_at(labels, label_float, p);
    if (C == 1) {
      const float s = sigmoid_f(x[0]);
      const float G0 = (y == 1 ? __ldg(coef) : 0.f) + __ldg(coef + 2);
      const float G1 = (y == 0 ? __ldg(coef + 1) : 0.f) + __ldg(coef + 3);
      d[0] = s * (1.f - s) * (G0 - G1) * gscale;
      continue;
    }
    const int w = (int)(p % W);
    const float mx = softmax_max(x, C);
    const float inv = 1.f / softmax_den(x, C, mx);
    float dot = 0.f;
    for (int c = 0; c < C; ++c) {
      const int k = c * W + w;
      const float G = (y == c ? __ldg(coef + k) : 0.f) + __ldg(coef + K + k);
      dot += expf(x[c] - mx) * inv * G;
    }
    for (int c = 0; c < C; ++c) {
      const int k = c * W + w;
      const float G = (y == c ? __ldg(coef + k) : 0.f) + __ldg(coef + K + k);
      d[c] = expf(x[c] - mx) * inv * (G - dot) * gscale;
    }
  }
}

// ---------------------------------------------------------------- focal
// CE = bce_sum / count, pt = exp(-CE), loss = alpha (1 - pt)^gamma CE,
// factor = dloss/dCE = alpha [(1 - pt)^gamma + gamma pt (1 - pt)^(gamma - 1) CE]
__global__ void focal_finalize_kernel(const double* bce_sum, double count, double alpha,
                                      double gamma, float* loss, float* factor) {
  const double ce = *bce_sum / count, pt = exp(-ce), q = 1.0 - pt;
  if (loss) *loss = (float)(alpha * pow(q, gamma) * ce);
  if (factor) {
    const double tail = gamma == 0.0 ? 0.0 : gamma * pt * pow(q, gamma - 1.0) * ce;
    *factor = (float)(alpha * (pow(q, gamma) + tail));
  }
}

// ---------------------------------------------------------------- IoU
// Per pixel: predicted class = sum_c c [p_c > thresh], 0 if above C - 1 (C > 1), or
// [sigmoid > thresh] (C = 1, two classes), p = softmax / sigmoid (or the raw values without
// `activation`); true class outside [0, nc) is ignored.  Bin
// nc * true + pred of a per-CTA shared histogram (one atomic per distinct bin and warp), then
// integer atomics into the int64 counts (integer sums do not depend on the order).
__global__ void __launch_bounds__(kT) iou_hist_kernel(const float* __restrict__ logits, int ld,
                                                      const void* __restrict__ labels,
                                                      int label_float, int64_t npix, int C,
                                                      int activation, float thresh,
                                                      unsigned long long* __restrict__ counts) {
  extern __shared__ unsigned s_hist[];
  const int nc = C == 1 ? 2 : C;
  for (int i = threadIdx.x; i < nc * nc; i += kT) s_hist[i] = 0u;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  for (int64_t base = blockIdx.x * (int64_t)kT + (threadIdx.x & ~31); base < npix;
       base += (int64_t)gridDim.x * kT) {
    const int64_t p = base + lane;
    int key = -1;
    if (p < npix) {
      const float* x = logits + p * ld;
      int pred = 0;
      if (C == 1) {
        pred = (activation ? sigmoid_f(x[0]) : x[0]) > thresh ? 1 : 0;
      } else if (activation) {
        const float mx = softmax_max(x, C);
        const float s = softmax_den(x, C, mx);
        for (int c = 0; c < C; ++c) pred += (expf(x[c] - mx) / s > thresh) ? c : 0;
        if (pred > C - 1) pred = 0;
      } else {
        for (int c = 0; c < C; ++c) pred += (x[c] > thresh) ? c : 0;
        if (pred > C - 1) pred = 0;
      }
      const int64_t y = label_at(labels, label_float, p);
      if (y >= 0 && y < nc) key = (int)y * nc + pred;
    }
    const unsigned peers = __match_any_sync(0xffffffffu, key);
    if (key >= 0 && lane == __ffs(peers) - 1) atomicAdd(&s_hist[key], (unsigned)__popc(peers));
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nc * nc; i += kT)
    if (s_hist[i]) atomicAdd(counts + i, (unsigned long long)s_hist[i]);
}

// the reference's float32 formula: jcd = diag / (rowsum + colsum - diag + 1e-10), mean over classes
__global__ void iou_finalize_kernel(const int64_t* __restrict__ counts, int nc, float* iou) {
  float sum = 0.f;
  for (int i = 0; i < nc; ++i) {
    int64_t a = 0, b = 0;
    for (int j = 0; j < nc; ++j) {
      a += counts[i * nc + j];
      b += counts[j * nc + i];
    }
    const float d = (float)counts[i * nc + i];
    sum += d / ((float)a + (float)b - d + 1e-10f);
  }
  *iou = sum / (float)nc;
}

}  // namespace

#define STREAM ((cudaStream_t)stream)

extern "C" {

int atomai_b200_dice_sums(const float* logits, int ld, const void* labels, int label_float, int N,
                          int H, int W, int C, double* cells, void* stream) {
  // an empty batch has no logits or labels to point at (torch gives empty tensors a null pointer)
  AB_CHECK(cells && N >= 0 && H > 0 && W > 0 && C >= 1 && ld >= C && (N == 0 || (logits && labels)),
           "dice_sums: bad arguments");
  AB_CHECK(C <= 16, "dice_sums: %d classes (at most 16)", C);
  AB_CHECK(C == 1 || !label_float, "dice_sums: multi-class labels must be int64");
  if (N == 0) {  // every sum is empty: the cells are zero and the loss is 1 - mean(0 / eps) = 1
    const int64_t K = C == 1 ? 2 : (int64_t)C * W;
    AB_CUDA(cudaMemsetAsync(cells, 0, 2 * K * sizeof(double), STREAM));
    return 0;
  }
  Ordered red;
  if (C == 1) {
    const int64_t npix = (int64_t)N * H * W;
    const int g = ab_grid(npix, kT, 8);
    if (ab_ordered_ws(STREAM, (int64_t)g * 4, 1, &red)) return 1;
    dice_sums_bin_kernel<<<g, kT, 0, STREAM>>>(logits, ld, labels, label_float, npix, cells, red);
    AB_LAUNCH_CHECK();
    return 0;
  }
  // groups of 32 columns; row chunks (slots) until about 4 CTAs per SM, at least 8 rows per chunk,
  // and at most kDiceWsDoubles partials (each row chunk holds 2 C x ceil(W/32)*32 of them)
  const int64_t rows = (int64_t)N * H;
  const int ncb = (W + kCols - 1) / kCols;
  const int64_t per_chunk = 2LL * C * kCols * ncb;
  AB_CHECK(per_chunk <= kDiceWsDoubles && ncb <= 4096,
           "dice_sums: %d classes x %d columns exceed the partial-sum workspace", C, W);
  AB_CHECK(rows <= 0x7fffffff, "dice_sums: too many rows");
  int64_t ny = ((int64_t)ab_num_sms() * 4 + ncb - 1) / ncb;
  ny = ny < (rows + kLanes - 1) / kLanes ? ny : (rows + kLanes - 1) / kLanes;
  ny = ny < kDiceWsDoubles / per_chunk ? ny : kDiceWsDoubles / per_chunk;
  ny = ny < 65535 ? ny : 65535;
  if (ny < 1) ny = 1;
  if (ab_ordered_ws(STREAM, ny * per_chunk, ncb, &red)) return 1;
  dice_sums_kernel<<<dim3(ncb, (unsigned)ny), kT, 2 * C * kT * sizeof(float), STREAM>>>(
      logits, ld, labels, label_float, (int)rows, W, C, cells, red);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_dice_finalize(const double* cells, int K, float eps, float* loss, float* coef,
                              void* stream) {
  AB_CHECK(cells && K > 0, "dice_finalize: bad arguments");
  dice_finalize_kernel<<<1, kT, 0, STREAM>>>(cells, K, (double)eps, loss, coef);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_dice_bwd(const float* logits, int ld, const void* labels, int label_float, int N,
                         int H, int W, int C, const float* coef, float* dlogits, int ld_d,
                         float gscale, const float* gscale_dev, void* stream) {
  AB_CHECK(coef && N >= 0 && H > 0 && W > 0 && C >= 1 && ld >= C && ld_d >= C &&
               (N == 0 || (logits && labels && dlogits)),
           "dice_bwd: bad arguments");
  AB_CHECK(C == 1 || !label_float, "dice_bwd: multi-class labels must be int64");
  const int64_t npix = (int64_t)N * H * W;
  if (npix == 0) return 0;
  dice_bwd_kernel<<<ab_grid(npix, kT, 8), kT, 0, STREAM>>>(logits, ld, labels, label_float, npix, W, C,
                                                     coef, dlogits, ld_d, gscale, gscale_dev);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_focal_finalize(const double* bce_sum, double count, float alpha, float gamma,
                               float* loss, float* factor, void* stream) {
  AB_CHECK(bce_sum && count > 0 && gamma >= 0.f, "focal_finalize: bad arguments");
  focal_finalize_kernel<<<1, 1, 0, STREAM>>>(bce_sum, count, (double)alpha, (double)gamma, loss,
                                             factor);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_iou_hist(const float* logits, int ld, const void* labels, int label_float,
                         int64_t npix, int C, int activation, float thresh, int64_t* counts,
                         void* stream) {
  AB_CHECK(logits && labels && counts && C >= 1 && ld >= C && npix >= 0, "iou_hist: bad arguments");
  AB_CHECK(C <= 64, "iou_hist: %d classes (at most 64)", C);
  if (npix == 0) return 0;
  const int nc = C == 1 ? 2 : C;
  iou_hist_kernel<<<ab_grid(npix, kT, 8), kT, nc * nc * sizeof(unsigned), STREAM>>>(
      logits, ld, labels, label_float, npix, C, activation, thresh,
      reinterpret_cast<unsigned long long*>(counts));
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_iou_finalize(const int64_t* counts, int nc, float* iou, void* stream) {
  AB_CHECK(counts && iou && nc >= 2, "iou_finalize: bad arguments");
  iou_finalize_kernel<<<1, 1, 0, STREAM>>>(counts, nc, iou);
  AB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
