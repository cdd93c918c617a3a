// frontend.cu — the steps either side of the network on the prediction / data path (SURVEY.md §8f)
// and training-mode dropout:
//   prob_mask       softmax / sigmoid over NHWC logits + thresholded binary mask per class in one
//                   pass (SegPredictor.forward_ + cv_thresh: atomai/predictors/predictor.py:209-231,
//                   atomai/utils/img.py:554-564) — the Locator then labels the masks on the host
//   gather          sub-image extraction around atom coordinates as one gather
//                   (atomai/utils/img.py:138-180, 298-350) with a per-window NaN flag, and the
//                   patches of extract_patches_ (atomai/utils/img.py:353-389) as a bit copy
//   dropout         in-place inverted dropout from a counter-based hash RNG (nn.Dropout in
//                   ConvBlock, atomai/nets/blocks.py:68-69) + per-channel sums for BatchNorm / bias
// All HBM-bound elementwise work: coalesced loads, one pass.
#include "common.cuh"

namespace {

constexpr int kT = 256;

__global__ void __launch_bounds__(kT) prob_mask_kernel(const float* __restrict__ logits, int ld,
                                                        int64_t npix, int C, int mode, float thresh,
                                                        float* __restrict__ prob, int ld_p,
                                                        uint8_t* __restrict__ mask) {
  for (int64_t p = blockIdx.x * (int64_t)kT + threadIdx.x; p < npix; p += (int64_t)gridDim.x * kT) {
    const float* x = logits + p * ld;
    float* o = prob + p * ld_p;
    if (mode == 0) {               // softmax over the C channels of this pixel
      float mx = x[0];
      for (int c = 1; c < C; ++c) mx = fmaxf(mx, x[c]);
      float s = 0.f;
      for (int c = 0; c < C; ++c) s += expf(x[c] - mx);
      for (int c = 0; c < C; ++c) {
        const float v = expf(x[c] - mx) / s;
        o[c] = v;
        if (mask) mask[p * C + c] = v > thresh ? 1 : 0;
      }
    } else {
      for (int c = 0; c < C; ++c) {
        const float v = mode == 1 ? 1.f / (1.f + expf(-x[c])) : (mode == 2 ? expf(x[c]) : x[c]);
        o[c] = v;
        if (mask) mask[p * C + c] = v > thresh ? 1 : 0;
      }
    }
  }
}

// one block per window: out[k][i][j][:] = img[origin_k + i * w * c + j * c + :] for a ph x pw
// window of c channels.  The origin is the element offset offs[k] when given, else it comes from
// the int32 row {f, sx, sy} of `table`.  T is a float (NaN flag per window) or an unsigned integer
// of the element's size (a bit copy, no flag).
template <typename T>
__global__ void __launch_bounds__(kT) gather_kernel(const T* __restrict__ img, int h, int w, int c,
                                                    const int32_t* __restrict__ table,
                                                    const int64_t* __restrict__ offs, int ph, int pw,
                                                    T* __restrict__ out,
                                                    int32_t* __restrict__ nanflag) {
  const int k = blockIdx.x;
  const int64_t row = (int64_t)w * c;
  const T* base = img + (offs ? offs[k]
                              : ((int64_t)table[3 * k] * h + table[3 * k + 1]) * row +
                                    (int64_t)table[3 * k + 2] * c);
  const int pwc = pw * c, n = ph * pwc;
  T* o = out + (int64_t)k * n;
  int bad = 0;
  for (int e = threadIdx.x; e < n; e += kT) {
    const int i = e / pwc, jc = e - i * pwc;
    const T v = base[i * row + jc];
    o[e] = v;
    bad |= (v != v);
  }
  if (nanflag && __syncthreads_or(bad) && threadIdx.x == 0) nanflag[k] = 1;
}

__global__ void __launch_bounds__(kT) dropout_kernel(float* __restrict__ a, int ld, int64_t npix,
                                                      int C, float p, float inv_keep, uint64_t seed,
                                                      double* __restrict__ stats) {
  extern __shared__ float s_part[];   // [2][C] block partials
  for (int i = threadIdx.x; i < 2 * C; i += kT) s_part[i] = 0.f;
  __syncthreads();
  const int64_t total = npix * C;
  for (int64_t e = blockIdx.x * (int64_t)kT + threadIdx.x; e < total; e += (int64_t)gridDim.x * kT) {
    const int64_t pix = e / C;
    const int c = (int)(e - pix * C);
    float* q = a + pix * ld + c;
    const float v = hash_uniform((uint64_t)e, seed) < p ? 0.f : *q * inv_keep;
    *q = v;
    if (stats) {
      atomicAdd(&s_part[c], v);
      atomicAdd(&s_part[C + c], v * v);
    }
  }
  if (stats) {
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * C; i += kT) atomicAdd(stats + i, (double)s_part[i]);
  }
}

// per-sample reconstruction loss of the VAEs (atomai/losses_metrics/vi_losses.py:13-37):
// kind 0: out[b] = 0.5 * sum_j (xhat - x)^2 ; kind 1: sum_j BCE-with-logits(xhat, x).
// grid = (chunks, B), scalar loads; one double atomic per block, so out is not bitwise
// reproducible when a row has more than one chunk.
// dxhat (nullable) = gvec[b] * dloss/dxhat.
__global__ void __launch_bounds__(kT) rowloss_kernel(const float* __restrict__ x,
                                                      const float* __restrict__ xhat, int64_t D,
                                                      int kind, double* __restrict__ out,
                                                      float* __restrict__ dxhat,
                                                      const float* __restrict__ gvec) {
  const int b = blockIdx.y;
  const float* xr = x + (int64_t)b * D;
  const float* hr = xhat + (int64_t)b * D;
  float* dr = dxhat ? dxhat + (int64_t)b * D : nullptr;
  const float g = gvec ? gvec[b] : 1.f;
  float acc = 0.f;
  for (int64_t j = blockIdx.x * (int64_t)kT + threadIdx.x; j < D; j += (int64_t)gridDim.x * kT) {
    const float t = xr[j], p = hr[j];
    if (kind == 0) {
      const float d = p - t;
      acc = fmaf(0.5f * d, d, acc);
      if (dr) dr[j] = g * d;
    } else {   // max(p, 0) - p t + log(1 + exp(-|p|))
      acc += fmaxf(p, 0.f) - p * t + log1pf(expf(-fabsf(p)));
      if (dr) dr[j] = g * (1.f / (1.f + expf(-p)) - t);
    }
  }
  if (out) {
    acc = warp_sum(acc);
    __shared__ float s_w[kT / 32];
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float tot = 0.f;
      for (int i = 0; i < kT / 32; ++i) tot += s_w[i];
      atomicAdd(out + b, (double)tot);
    }
  }
}

}  // namespace

extern "C" {

int atomai_b200_prob_mask(const float* logits, int ld, int64_t npix, int C, int mode, float thresh,
                          float* prob, int ld_p, uint8_t* mask, void* stream) {
  AB_CHECK(logits && prob && C > 0 && ld >= C && ld_p >= C, "prob_mask: bad arguments");
  AB_CHECK(mode >= 0 && mode <= 3, "prob_mask: mode=%d", mode);
  if (npix == 0) return 0;
  prob_mask_kernel<<<ab_grid(npix, kT, 16), kT, 0, (cudaStream_t)stream>>>(logits, ld, npix, C, mode,
                                                                     thresh, prob, ld_p, mask);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_gather_windows(const float* img, int n, int h, int w, int c, const int32_t* table,
                               int K, int r, float* out, int32_t* nanflag, void* stream) {
  AB_CHECK(img && table && out && n > 0 && h > 0 && w > 0 && c > 0 && r > 0 && r <= h && r <= w,
           "gather_windows: bad arguments");
  if (K == 0) return 0;
  gather_kernel<float><<<K, kT, 0, (cudaStream_t)stream>>>(img, h, w, c, table, nullptr, r, r, out,
                                                           nanflag);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_gather_patches(const void* img, int elem_bytes, int w, int c, const int64_t* offs,
                               int K, int ph, int pw, void* out, void* stream) {
  AB_CHECK(img && offs && out && w > 0 && c > 0 && K >= 0 && ph > 0 && pw > 0 && pw <= w &&
               (int64_t)ph * pw * c <= INT32_MAX,
           "gather_patches: bad arguments");
  if (K == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  switch (elem_bytes) {
    case 1:
      gather_kernel<uint8_t><<<K, kT, 0, st>>>((const uint8_t*)img, 0, w, c, nullptr, offs, ph, pw,
                                               (uint8_t*)out, nullptr);
      break;
    case 2:
      gather_kernel<uint16_t><<<K, kT, 0, st>>>((const uint16_t*)img, 0, w, c, nullptr, offs, ph,
                                                pw, (uint16_t*)out, nullptr);
      break;
    case 4:
      gather_kernel<uint32_t><<<K, kT, 0, st>>>((const uint32_t*)img, 0, w, c, nullptr, offs, ph,
                                                pw, (uint32_t*)out, nullptr);
      break;
    case 8:
      gather_kernel<unsigned long long><<<K, kT, 0, st>>>((const unsigned long long*)img, 0, w, c,
                                                          nullptr, offs, ph, pw,
                                                          (unsigned long long*)out, nullptr);
      break;
    default: AB_CHECK(false, "gather_patches: element size %d not in {1, 2, 4, 8}", elem_bytes);
  }
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_rowloss(const float* x, const float* xhat, int B, int64_t D, int kind, double* out,
                        float* dxhat, const float* gvec, void* stream) {
  AB_CHECK(x && xhat && B >= 0 && D > 0 && (kind == 0 || kind == 1), "rowloss: bad arguments");
  AB_CHECK(B <= 65535, "rowloss: batch too large for one launch");
  if (B == 0) return 0;
  int gx = (int)((D + kT * 8 - 1) / (kT * 8));
  gx = gx < 1 ? 1 : (gx > 64 ? 64 : gx);
  rowloss_kernel<<<dim3(gx, B), kT, 0, (cudaStream_t)stream>>>(x, xhat, D, kind, out, dxhat, gvec);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_dropout(float* a, int ld, int64_t npix, int C, float p, uint64_t seed,
                        double* stats, void* stream) {
  AB_CHECK(a && C > 0 && ld >= C && p >= 0.f && p < 1.f, "dropout: bad arguments (p=%f)", p);
  AB_CHECK(C <= 4096, "dropout: too many channels");
  if (npix == 0) return 0;
  dropout_kernel<<<ab_grid(npix * C, kT, 16), kT, 2 * C * sizeof(float), (cudaStream_t)stream>>>(
      a, ld, npix, C, p, 1.f / (1.f - p), seed, stats);
  AB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
