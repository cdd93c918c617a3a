// elementwise.cu — the HBM-bound kernels around the convolutions: BatchNorm finalize / backward,
// LeakyReLU backward, 2x2 max-pool, bilinear/nearest x2 upsampling, gradient routing, the
// DilatedBlock sum, losses and the fused multi-tensor Adam step.  All are coalesced along the
// channel axis of the NHWC activations (float4 when C % 4 == 0) and grid-sized as a multiple of
// the SM count.  Per-channel reductions go warp/CTA-local first and finish with an ordered
// cross-CTA sum in double per channel.
//
// Reference call sites: nn.BatchNorm2d atomai/nets/blocks.py:73; nn.LeakyReLU :70;
// F.max_pool2d atomai/nets/fcnn.py:123-127; F.interpolate atomai/nets/blocks.py:130-131;
// DilatedBlock.forward blocks.py:321-329; nn.CrossEntropyLoss / BCEWithLogits / MSE
// atomai/losses_metrics/losses.py:154-164; torch.optim.Adam atomai/trainers/trainer.py:539.
#include <initializer_list>

#include "common.cuh"

namespace {

constexpr int kT = 256;

// workspace of an ordered cross-CTA sum of n values per CTA for a launch of grid_for() CTAs
int red_ws(cudaStream_t stream, int n, Ordered* red) {
  return ab_ordered_ws(stream, (int64_t)ab_num_sms() * 8 * n, 1, red);
}

inline int grid_for(int64_t work_items, int per_block = kT) {
  int64_t b = (work_items + per_block - 1) / per_block;
  const int64_t cap = (int64_t)ab_num_sms() * 8;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

// ---------------------------------------------------------------- BatchNorm finalize
__global__ void bn_finalize_kernel(const double* stats, int C, double count, const float* gamma,
                                   const float* beta, float* rmean, float* rvar, float momentum,
                                   float eps, int training, float* scale, float* shift,
                                   float* mean_o, float* invstd_o) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float mean, var_b;
  if (training) {
    const double m = stats[c] / count;
    double v = stats[C + c] / count - m * m;
    if (v < 0) v = 0;
    mean = (float)m;
    var_b = (float)v;
    if (rmean) {
      const double unb = count > 1 ? v * count / (count - 1) : v;
      rmean[c] = (1.f - momentum) * rmean[c] + momentum * mean;
      rvar[c] = (1.f - momentum) * rvar[c] + momentum * (float)unb;
    }
  } else {
    mean = rmean[c];
    var_b = rvar[c];
  }
  const float invstd = rsqrtf(var_b + eps);
  const float g = gamma ? gamma[c] : 1.f, b = beta ? beta[c] : 0.f;
  scale[c] = g * invstd;
  shift[c] = b - mean * g * invstd;
  if (mean_o) mean_o[c] = mean;
  if (invstd_o) invstd_o[c] = invstd;
}

// ---------------------------------------------------------------- y = a*scale + shift
__global__ void affine_kernel(const float* __restrict__ a, int ld_a, const float* scale,
                              const float* shift, float* __restrict__ y, int ld_y, int64_t npix,
                              int C, int hw_nchw) {
  const int64_t total = npix * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int64_t pix = i / C;
    float v = a[pix * ld_a + c];
    if (scale) v = fmaf(v, scale[c], shift[c]);
    if (hw_nchw) {
      const int64_t n = pix / hw_nchw, r = pix % hw_nchw;
      y[(n * C + c) * hw_nchw + r] = v;
    } else {
      y[pix * ld_y + c] = v;
    }
  }
}

// ---------------------------------------------------------------- per-channel reductions
// Thread layout: CW = pow2 >= C (<= 256) channel lanes, R = 256/CW pixel rows per CTA step.
struct ChanLayout {
  int CW, R;
};
inline ChanLayout chan_layout(int C) {
  int cw = 1;
  while (cw < C) cw <<= 1;
  ChanLayout l;
  l.CW = cw;
  l.R = kT / cw;
  return l;
}

// The CTA's per-channel totals go into its slot of an ordered cross-CTA sum (common.cuh), so the
// result does not depend on which CTA finishes first.
__device__ __forceinline__ void block_chan_reduce2(float v1, float v2, int cx, int py, int CW,
                                                   int R, int C, double* out1, double* out2,
                                                   const Ordered& red) {
  __shared__ float s1[kT], s2[kT];
  s1[py * CW + cx] = v1;
  s2[py * CW + cx] = v2;
  __syncthreads();
  if (py == 0 && cx < C) {
    float a = 0.f, b = 0.f;
    for (int r = 0; r < R; ++r) {
      a += s1[r * CW + cx];
      b += s2[r * CW + cx];
    }
    double* slot = ordered_slot(red, 0, gridDim.x, blockIdx.x, 2 * C);
    slot[cx] = a;
    slot[C + cx] = b;
  }
  __shared__ unsigned s_last;
  ordered_finish(red, 0, gridDim.x, 2 * C, threadIdx.x, kT, gridDim.x, [] { __syncthreads(); },
                 [&](int i, double v) {
                   double* o = i < C ? out1 : out2;
                   if (o) o[i < C ? i : i - C] += v;
                 },
                 &s_last);
}

__global__ void __launch_bounds__(kT) bn_bwd_reduce_kernel(const float* __restrict__ dy, int ld_dy,
                                                           const float* __restrict__ a, int ld_a,
                                                           const float* mean, const float* invstd,
                                                           int64_t npix, int C, int CW, int R,
                                                           double* sums, Ordered red) {
  const int cx = threadIdx.x % CW, py = threadIdx.x / CW;
  float s1 = 0.f, s2 = 0.f;
  if (cx < C) {
    const float m = mean[cx], is = invstd[cx];
    for (int64_t p = (int64_t)blockIdx.x * R + py; p < npix; p += (int64_t)gridDim.x * R) {
      const float g = dy[p * ld_dy + cx];
      const float xh = (a[p * ld_a + cx] - m) * is;
      s1 += g;
      s2 = fmaf(g, xh, s2);
    }
  }
  block_chan_reduce2(s1, s2, cx, py, CW, R, C, sums, sums + C, red);
}

__global__ void __launch_bounds__(kT)
    bn_lrelu_bwd_kernel(const float* __restrict__ dy, int ld_dy, const float* __restrict__ a,
                        int ld_a, const float* mean, const float* invstd, const float* scale,
                        const double* sums, double count, const float* __restrict__ extra,
                        int ld_extra, int act, float alpha, float* __restrict__ dpre, int ld_dpre,
                        double* dbias, int64_t npix, int C, int CW, int R, Ordered red) {
  const int cx = threadIdx.x % CW, py = threadIdx.x / CW;
  float sb = 0.f;
  if (cx < C) {
    float m = 0.f, is = 0.f, sc = 1.f, k1 = 0.f, k2 = 0.f;
    const bool bn = scale != nullptr;
    if (bn) {
      m = mean[cx];
      is = invstd[cx];
      sc = scale[cx];
      k1 = (float)(sums[cx] / count);
      k2 = (float)(sums[C + cx] / count);
    }
    for (int64_t p = (int64_t)blockIdx.x * R + py; p < npix; p += (int64_t)gridDim.x * R) {
      const float av = a[p * ld_a + cx];
      float g = dy ? dy[p * ld_dy + cx] : 0.f;
      if (bn) {
        const float xh = (av - m) * is;
        g = sc * (g - k1 - xh * k2);
      }
      float ex = 0.f;
      if (extra) {
        ex = extra[p * ld_extra + cx];
        g += ex;
      }
      const float d = g * act_grad_from_out(av, act, alpha) + ex;
      dpre[p * ld_dpre + cx] = d;
      sb += d;
    }
  }
  if (dbias) block_chan_reduce2(sb, 0.f, cx, py, CW, R, C, dbias, nullptr, red);
}

// ---------------------------------------------------------------- 2x2 max pool
__global__ void pool_fwd_kernel(const float* __restrict__ a, int ld_a, const float* scale,
                                const float* shift, float* __restrict__ y, int ld_y, int N, int Ho,
                                int Wo, int C) {
  const int64_t total = (int64_t)N * Ho * Wo * C;
  const int W2 = 2 * Wo, H2 = 2 * Ho;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    int64_t r = i / C;
    const int wo = (int)(r % Wo); r /= Wo;
    const int ho = (int)(r % Ho);
    const int n = (int)(r / Ho);
    const float sc = scale ? scale[c] : 1.f, sh = scale ? shift[c] : 0.f;
    const float* b = a + (((int64_t)n * H2 + 2 * ho) * W2 + 2 * wo) * ld_a + c;
    const float v0 = fmaf(b[0], sc, sh), v1 = fmaf(b[ld_a], sc, sh);
    const float v2 = fmaf(b[(int64_t)W2 * ld_a], sc, sh);
    const float v3 = fmaf(b[(int64_t)W2 * ld_a + ld_a], sc, sh);
    y[(((int64_t)n * Ho + ho) * Wo + wo) * ld_y + c] = fmaxf(fmaxf(v0, v1), fmaxf(v2, v3));
  }
}

__global__ void pool_bwd_kernel(const float* __restrict__ dp, int ld_dp,
                                const float* __restrict__ a, int ld_a, const float* scale,
                                const float* shift, float* __restrict__ df, int ld_df,
                                int accumulate, int N, int Ho, int Wo, int C) {
  const int64_t total = (int64_t)N * Ho * Wo * C;
  const int W2 = 2 * Wo, H2 = 2 * Ho;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    int64_t r = i / C;
    const int wo = (int)(r % Wo); r /= Wo;
    const int ho = (int)(r % Ho);
    const int n = (int)(r / Ho);
    const float sc = scale ? scale[c] : 1.f, sh = scale ? shift[c] : 0.f;
    const int64_t base = ((int64_t)n * H2 + 2 * ho) * W2 + 2 * wo;
    const int64_t off[4] = {0, 1, W2, (int64_t)W2 + 1};
    int best = 0;
    float bv = fmaf(a[(base + off[0]) * ld_a + c], sc, sh);
#pragma unroll
    for (int k = 1; k < 4; ++k) {
      const float v = fmaf(a[(base + off[k]) * ld_a + c], sc, sh);
      if (v > bv) {  // first maximum wins, as in ATen's max_pool2d
        bv = v;
        best = k;
      }
    }
    const float g = dp[(((int64_t)n * Ho + ho) * Wo + wo) * ld_dp + c];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float* o = df + (base + off[k]) * ld_df + c;
      const float v = (k == best) ? g : 0.f;
      *o = accumulate ? *o + v : v;
    }
  }
}

// ---------------------------------------------------------------- x2 upsampling
__device__ __forceinline__ void up_src(int o, int n, int& i0, int& i1, float& l1) {
  // align_corners=False, scale 2: src = max(o/2 - 0.25, 0)
  float s = 0.5f * o - 0.25f;
  if (s < 0.f) s = 0.f;
  i0 = (int)s;
  l1 = s - i0;
  i1 = i0 + 1 < n ? i0 + 1 : n - 1;
}

// (1-lh)((1-lw)a + lw b) + lh((1-lw)c + lw d), with the FMAs spelled out: each sum is one FMA of
// its first product onto the rounded second product.  Left to the compiler, the contraction
// differed between the two kernels below (whether lh / lw are constants or not); this is the
// form the 2x2-block kernel has always computed, and both kernels now give its bits.
__device__ __forceinline__ float bil_mix(float a, float b, float c, float d, float lh, float lw) {
  const float top = fmaf(1.f - lw, a, __fmul_rn(lw, b));
  const float bot = fmaf(1.f - lw, c, __fmul_rn(lw, d));
  return fmaf(1.f - lh, top, __fmul_rn(lh, bot));
}

__global__ void upsample_fwd_kernel(const float* __restrict__ x, int ld_x, float* __restrict__ y,
                                    int ld_y, int N, int h, int w, int C, int bilinear) {
  const int H = 2 * h, W = 2 * w;
  const int64_t total = (int64_t)N * H * W * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    int64_t r = i / C;
    const int ow = (int)(r % W); r /= W;
    const int oh = (int)(r % H);
    const int n = (int)(r / H);
    float v;
    const float* xb = x + (int64_t)n * h * w * ld_x + c;
    if (bilinear) {
      int h0, h1, w0, w1;
      float lh, lw;
      up_src(oh, h, h0, h1, lh);
      up_src(ow, w, w0, w1, lw);
      const float x00 = xb[((int64_t)h0 * w + w0) * ld_x], x01 = xb[((int64_t)h0 * w + w1) * ld_x];
      const float x10 = xb[((int64_t)h1 * w + w0) * ld_x], x11 = xb[((int64_t)h1 * w + w1) * ld_x];
      v = bil_mix(x00, x01, x10, x11, lh, lw);
    } else {
      v = xb[((int64_t)(oh >> 1) * w + (ow >> 1)) * ld_x];
    }
    y[(((int64_t)n * H + oh) * W + ow) * ld_y + c] = v;
  }
}

// adjoint of the above: gather form, <= 4 taps per axis
__device__ __forceinline__ int up_adj(int i, int n, int* o, float* wt) {
  int k = 0;
  if (i >= 1) { o[k] = 2 * i - 1; wt[k++] = 0.25f; }
  o[k] = 2 * i; wt[k++] = (i == 0) ? 1.0f : 0.75f;
  o[k] = 2 * i + 1; wt[k++] = (i == n - 1) ? 1.0f : 0.75f;
  if (i <= n - 2) { o[k] = 2 * i + 2; wt[k++] = 0.25f; }
  return k;
}

__global__ void upsample_bwd_kernel(const float* __restrict__ dy, int ld_dy, float* __restrict__ dx,
                                    int ld_dx, int N, int h, int w, int C, int bilinear) {
  const int H = 2 * h, W = 2 * w;
  const int64_t total = (int64_t)N * h * w * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    int64_t r = i / C;
    const int iw = (int)(r % w); r /= w;
    const int ih = (int)(r % h);
    const int n = (int)(r / h);
    const float* db = dy + (int64_t)n * H * W * ld_dy + c;
    float acc = 0.f;
    if (bilinear) {
      int oh[4], ow[4];
      float wh[4], ww[4];
      const int nh = up_adj(ih, h, oh, wh), nw = up_adj(iw, w, ow, ww);
      for (int a = 0; a < nh; ++a) {
        float rowacc = 0.f;
        for (int b = 0; b < nw; ++b) rowacc = fmaf(ww[b], db[((int64_t)oh[a] * W + ow[b]) * ld_dy], rowacc);
        acc = fmaf(wh[a], rowacc, acc);
      }
    } else {
      const int64_t b0 = ((int64_t)(2 * ih) * W + 2 * iw) * ld_dy;
      // (top pair) + (bottom pair), as the float4 kernel sums them
      acc = (db[b0] + db[b0 + ld_dy]) + (db[b0 + (int64_t)W * ld_dy] + db[b0 + (int64_t)W * ld_dy + ld_dy]);
    }
    dx[(((int64_t)n * h + ih) * w + iw) * ld_dx + c] = acc;
  }
}

__global__ void add_slice_kernel(const float* __restrict__ src, int ld_s, float* __restrict__ dst,
                                 int ld_d, int accumulate, int64_t npix, int C) {
  const int64_t total = npix * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int64_t p = i / C;
    const float v = src[p * ld_s + c];
    float* o = dst + p * ld_d + c;
    *o = accumulate ? *o + v : v;
  }
}

constexpr int kMaxDil = 8;
struct DilPtrs {
  const float* a[kMaxDil];
  const float* scale[kMaxDil];
  const float* shift[kMaxDil];
};
__global__ void dilated_sum_kernel(DilPtrs P, int nl, float alpha, float* __restrict__ out,
                                   int64_t n, int C) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    float acc = 0.f;
    for (int l = 0; l < nl; ++l) {
      const float av = P.a[l][i];
      const float pre = av > 0.f ? av : av / alpha;
      acc += pre + av;
      if (P.scale[l]) acc += fmaf(av, P.scale[l][c], P.shift[l][c]);
    }
    out[i] = acc;
  }
}

// ---------------------------------------------------------------- losses
__global__ void __launch_bounds__(kT) ce_kernel(const float* __restrict__ logits, int ld,
                                                const int64_t* __restrict__ labels, int64_t npix,
                                                int C, double* loss_sum,
                                                float* __restrict__ dlogits, int ld_d,
                                                float gscale, const float* gscale_dev, Ordered red) {
  float local = 0.f;
  if (gscale_dev) gscale *= __ldg(gscale_dev);
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < npix;
       p += (int64_t)gridDim.x * blockDim.x) {
    const float* l = logits + p * ld;
    float m = l[0];
    for (int c = 1; c < C; ++c) m = fmaxf(m, l[c]);
    float s = 0.f;
    for (int c = 0; c < C; ++c) s += __expf(l[c] - m);
    const float lse = m + __logf(s);
    const int y = (int)labels[p];
    local += lse - l[y];
    if (dlogits) {
      const float inv = 1.f / s;
      for (int c = 0; c < C; ++c) {
        const float pr = __expf(l[c] - m) * inv;
        dlogits[p * ld_d + c] = (pr - (c == y ? 1.f : 0.f)) * gscale;
      }
    }
  }
  __shared__ float wred[kT / 32];
  const float ws = warp_sum(local);
  if ((threadIdx.x & 31) == 0) wred[threadIdx.x >> 5] = ws;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < kT / 32; ++i) t += wred[i];
    if (loss_sum) ordered_slot(red, 0, gridDim.x, blockIdx.x, 1)[0] = (double)t;
  }
  __shared__ unsigned s_last;
  if (loss_sum)
    ordered_finish(red, 0, gridDim.x, 1, threadIdx.x, kT, gridDim.x, [] { __syncthreads(); },
                   [&](int, double v) { *loss_sum += v; }, &s_last);
}

__global__ void __launch_bounds__(kT) pointwise_loss_kernel(const float* __restrict__ pred,
                                                            const float* __restrict__ tgt,
                                                            int64_t n, int kind, double* loss_sum,
                                                            float* __restrict__ dpred,
                                                            float gscale,
                                                            const float* gscale_dev, Ordered red) {
  float local = 0.f;
  if (gscale_dev) gscale *= __ldg(gscale_dev);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const float x = pred[i], t = tgt[i];
    if (kind == 0) {
      const float d = x - t;
      local = fmaf(d, d, local);
      if (dpred) dpred[i] = 2.f * d * gscale;
    } else {  // BCE with logits: max(x,0) - x*t + log(1 + exp(-|x|))
      local += fmaxf(x, 0.f) - x * t + log1pf(__expf(-fabsf(x)));
      if (dpred) dpred[i] = (1.f / (1.f + __expf(-x)) - t) * gscale;
    }
  }
  __shared__ float wred[kT / 32];
  const float ws = warp_sum(local);
  if ((threadIdx.x & 31) == 0) wred[threadIdx.x >> 5] = ws;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < kT / 32; ++i) t += wred[i];
    if (loss_sum) ordered_slot(red, 0, gridDim.x, blockIdx.x, 1)[0] = (double)t;
  }
  __shared__ unsigned s_last;
  if (loss_sum)
    ordered_finish(red, 0, gridDim.x, 1, threadIdx.x, kT, gridDim.x, [] { __syncthreads(); },
                   [&](int, double v) { *loss_sum += v; }, &s_last);
}

__global__ void __launch_bounds__(kT) sqerr_kernel(const float* __restrict__ x,
                                                   const float* __restrict__ xhat, int64_t n,
                                                   double* out, float* __restrict__ dxhat,
                                                   float gscale, const float* gscale_dev, Ordered red) {
  float local = 0.f;
  if (gscale_dev) gscale *= __ldg(gscale_dev);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const float d = xhat[i] - x[i];
    local = fmaf(d, d, local);
    if (dxhat) dxhat[i] = d * gscale;
  }
  __shared__ float wred[kT / 32];
  const float ws = warp_sum(local);
  if ((threadIdx.x & 31) == 0) wred[threadIdx.x >> 5] = ws;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < kT / 32; ++i) t += wred[i];
    if (out) ordered_slot(red, 0, gridDim.x, blockIdx.x, 1)[0] = 0.5 * (double)t;
  }
  __shared__ unsigned s_last;
  if (out)
    ordered_finish(red, 0, gridDim.x, 1, threadIdx.x, kT, gridDim.x, [] { __syncthreads(); },
                   [&](int, double v) { *out += v; }, &s_last);
}

// ---------------------------------------------------------------- Adam (multi-tensor)
__global__ void adam_multi_kernel(const int64_t* __restrict__ table, float lr, float b1, float b2,
                                  float eps, float wd, float bc1, float bc2_sqrt,
                                  float grad_scale) {
  const int64_t* row = table + (int64_t)blockIdx.y * 5;
  float* p = reinterpret_cast<float*>(row[0]);
  const float* g = reinterpret_cast<const float*>(row[1]);
  float* m = reinterpret_cast<float*>(row[2]);
  float* v = reinterpret_cast<float*>(row[3]);
  const int64_t n = row[4];
  const float step = lr / bc1;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    float gi = g[i] * grad_scale;
    if (wd != 0.f) gi = fmaf(wd, p[i], gi);
    const float mi = b1 * m[i] + (1.f - b1) * gi;
    const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    const float denom = sqrtf(vi) / bc2_sqrt + eps;
    p[i] = p[i] - step * (mi / denom);
  }
}


// ================================================================= float4 fast paths
// Used when C % 4 == 0, every pixel stride % 4 == 0 and all pointers are 16 B aligned (always the
// case for the UNet path).  Index math is 32-bit with shift/mask when C/4 is a power of two.
struct VIdx {
  int C4;
  int shift;  // log2(C4) or -1
  __device__ __forceinline__ void split(uint32_t i, uint32_t& pix, int& c4) const {
    if (shift >= 0) { pix = i >> shift; c4 = (int)(i & (uint32_t)(C4 - 1)); }
    else { pix = i / (uint32_t)C4; c4 = (int)(i - pix * (uint32_t)C4); }
  }
};
inline VIdx make_vidx(int C) {
  VIdx v; v.C4 = C / 4; v.shift = -1;
  for (int s = 0; s < 12; ++s) if ((1 << s) == v.C4) v.shift = s;
  return v;
}
inline bool vec_ok(int C, std::initializer_list<const void*> ptrs, std::initializer_list<int> lds,
                   int64_t total4) {
  if (C % 4 != 0 || total4 >= (int64_t)1 << 31) return false;
  for (auto p : ptrs) if (p && ((uintptr_t)p & 15)) return false;
  for (auto l : lds) if (l % 4 != 0) return false;
  return true;
}
__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 f4fma(float4 a, float4 s, float4 t) {
  return make_float4(fmaf(a.x, s.x, t.x), fmaf(a.y, s.y, t.y), fmaf(a.z, s.z, t.z), fmaf(a.w, s.w, t.w));
}
__device__ __forceinline__ float4 f4max(float4 a, float4 b) {
  return make_float4(fmaxf(a.x, b.x), fmaxf(a.y, b.y), fmaxf(a.z, b.z), fmaxf(a.w, b.w));
}
__device__ __forceinline__ float4 f4add(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }

__global__ void __launch_bounds__(kT) affine_vec_kernel(const float* __restrict__ a, int ld_a, const float* scale,
                                  const float* shift, float* __restrict__ y, int ld_y, uint32_t total, VIdx ix) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    uint32_t pix; int c4; ix.split(i, pix, c4);
    float4 v = ld4(a + (size_t)pix * ld_a + c4 * 4);
    if (scale) v = f4fma(v, ld4(scale + c4 * 4), ld4(shift + c4 * 4));
    *reinterpret_cast<float4*>(y + (size_t)pix * ld_y + c4 * 4) = v;
  }
}

__global__ void __launch_bounds__(kT) add_slice_vec_kernel(const float* __restrict__ src, int ld_s, float* __restrict__ dst,
                                     int ld_d, int accumulate, uint32_t total, VIdx ix) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    uint32_t pix; int c4; ix.split(i, pix, c4);
    float4 v = ld4(src + (size_t)pix * ld_s + c4 * 4);
    float4* o = reinterpret_cast<float4*>(dst + (size_t)pix * ld_d + c4 * 4);
    if (accumulate) v = f4add(v, *o);
    *o = v;
  }
}

// per-channel reductions: thread = (c4 lane cx, pixel row py), CW4 = pow2 >= C4, R = 256 / CW4
__device__ __forceinline__ void block_chan_reduce_vec(float4 v1, float4 v2, int cx, int py, int CW, int R, int C4,
                                                      double* out1, double* out2, const Ordered& red) {
  __shared__ float4 s1[kT], s2[kT];
  s1[py * CW + cx] = v1;
  s2[py * CW + cx] = v2;
  __syncthreads();
  if (py == 0 && cx < C4) {
    float4 a = make_float4(0, 0, 0, 0), b = a;
    for (int r = 0; r < R; ++r) { a = f4add(a, s1[r * CW + cx]); b = f4add(b, s2[r * CW + cx]); }
    double* slot = ordered_slot(red, 0, gridDim.x, blockIdx.x, 8 * C4);
    slot[cx * 4] = a.x; slot[cx * 4 + 1] = a.y; slot[cx * 4 + 2] = a.z; slot[cx * 4 + 3] = a.w;
    double* s2_ = slot + 4 * C4;
    s2_[cx * 4] = b.x; s2_[cx * 4 + 1] = b.y; s2_[cx * 4 + 2] = b.z; s2_[cx * 4 + 3] = b.w;
  }
  __shared__ unsigned s_last;
  const int C = 4 * C4;
  ordered_finish(red, 0, gridDim.x, 2 * C, threadIdx.x, kT, gridDim.x, [] { __syncthreads(); },
                 [&](int i, double v) {
                   double* o = i < C ? out1 : out2;
                   if (o) o[i < C ? i : i - C] += v;
                 },
                 &s_last);
}

__global__ void __launch_bounds__(kT) bn_bwd_reduce_vec_kernel(const float* __restrict__ dy, int ld_dy, const float* __restrict__ a,
                                         int ld_a, const float* mean, const float* invstd, int64_t npix, int C4,
                                         int CW, int R, double* sums, Ordered red) {
  const int cx = threadIdx.x % CW, py = threadIdx.x / CW;
  float4 s1 = make_float4(0, 0, 0, 0), s2 = s1;
  if (cx < C4) {
    const float4 m = ld4(mean + cx * 4), is = ld4(invstd + cx * 4);
    for (int64_t p = (int64_t)blockIdx.x * R + py; p < npix; p += (int64_t)gridDim.x * R) {
      const float4 g = ld4(dy + p * ld_dy + cx * 4), av = ld4(a + p * ld_a + cx * 4);
      s1 = f4add(s1, g);
      s2.x = fmaf(g.x, (av.x - m.x) * is.x, s2.x); s2.y = fmaf(g.y, (av.y - m.y) * is.y, s2.y);
      s2.z = fmaf(g.z, (av.z - m.z) * is.z, s2.z); s2.w = fmaf(g.w, (av.w - m.w) * is.w, s2.w);
    }
  }
  block_chan_reduce_vec(s1, s2, cx, py, CW, R, C4, sums, sums + C4 * 4, red);
}

__device__ __forceinline__ float bwd1(float g, float av, bool bn, float m, float is, float sc, float k1, float k2,
                                      float ex, bool has_ex, int act, float alpha) {
  if (bn) g = sc * (g - k1 - (av - m) * is * k2);
  if (has_ex) g += ex;
  return g * act_grad_from_out(av, act, alpha) + (has_ex ? ex : 0.f);
}

__global__ void __launch_bounds__(kT) bn_lrelu_bwd_vec_kernel(const float* __restrict__ dy, int ld_dy, const float* __restrict__ a, int ld_a,
                                        const float* mean, const float* invstd, const float* scale, const double* sums,
                                        double count, const float* __restrict__ extra, int ld_extra, int act, float alpha,
                                        float* __restrict__ dpre, int ld_dpre, double* dbias, int64_t npix, int C4,
                                        int CW, int R, Ordered red) {
  const int cx = threadIdx.x % CW, py = threadIdx.x / CW;
  float4 sb = make_float4(0, 0, 0, 0);
  if (cx < C4) {
    const bool bn = scale != nullptr, has_ex = extra != nullptr;
    float4 m = sb, is = sb, sc = sb, k1 = sb, k2 = sb;
    if (bn) {
      const int C = C4 * 4, c = cx * 4;
      m = ld4(mean + c); is = ld4(invstd + c); sc = ld4(scale + c);
      k1 = make_float4((float)(sums[c] / count), (float)(sums[c + 1] / count), (float)(sums[c + 2] / count), (float)(sums[c + 3] / count));
      k2 = make_float4((float)(sums[C + c] / count), (float)(sums[C + c + 1] / count), (float)(sums[C + c + 2] / count), (float)(sums[C + c + 3] / count));
    }
    for (int64_t p = (int64_t)blockIdx.x * R + py; p < npix; p += (int64_t)gridDim.x * R) {
      const float4 av = ld4(a + p * ld_a + cx * 4);
      const float4 g = dy ? ld4(dy + p * ld_dy + cx * 4) : make_float4(0, 0, 0, 0);
      const float4 ex = has_ex ? ld4(extra + p * ld_extra + cx * 4) : make_float4(0, 0, 0, 0);
      float4 d;
      d.x = bwd1(g.x, av.x, bn, m.x, is.x, sc.x, k1.x, k2.x, ex.x, has_ex, act, alpha);
      d.y = bwd1(g.y, av.y, bn, m.y, is.y, sc.y, k1.y, k2.y, ex.y, has_ex, act, alpha);
      d.z = bwd1(g.z, av.z, bn, m.z, is.z, sc.z, k1.z, k2.z, ex.z, has_ex, act, alpha);
      d.w = bwd1(g.w, av.w, bn, m.w, is.w, sc.w, k1.w, k2.w, ex.w, has_ex, act, alpha);
      *reinterpret_cast<float4*>(dpre + p * ld_dpre + cx * 4) = d;
      sb = f4add(sb, d);
    }
  }
  if (dbias) block_chan_reduce_vec(sb, make_float4(0, 0, 0, 0), cx, py, CW, R, C4, dbias, nullptr, red);
}

__global__ void __launch_bounds__(kT) pool_fwd_vec_kernel(const float* __restrict__ a, int ld_a, const float* scale, const float* shift,
                                    float* __restrict__ y, int ld_y, int Ho, int Wo, uint32_t total, VIdx ix) {
  const int W2 = 2 * Wo;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    uint32_t pix; int c4; ix.split(i, pix, c4);
    const uint32_t wo = pix % Wo, r = pix / Wo, ho = r % Ho, n = r / Ho;
    float4 sc = make_float4(1, 1, 1, 1), sh = make_float4(0, 0, 0, 0);
    if (scale) { sc = ld4(scale + c4 * 4); sh = ld4(shift + c4 * 4); }
    const float* b = a + (((size_t)n * 2 * Ho + 2 * ho) * W2 + 2 * wo) * ld_a + c4 * 4;
    const float4 v = f4max(f4max(f4fma(ld4(b), sc, sh), f4fma(ld4(b + ld_a), sc, sh)),
                           f4max(f4fma(ld4(b + (size_t)W2 * ld_a), sc, sh), f4fma(ld4(b + (size_t)W2 * ld_a + ld_a), sc, sh)));
    *reinterpret_cast<float4*>(y + (size_t)pix * ld_y + c4 * 4) = v;
  }
}

__device__ __forceinline__ void pick4(float v0, float v1, float v2, float v3, float g, float& o0, float& o1, float& o2, float& o3) {
  int best = 0; float bv = v0;
  if (v1 > bv) { bv = v1; best = 1; }
  if (v2 > bv) { bv = v2; best = 2; }
  if (v3 > bv) { bv = v3; best = 3; }
  o0 = best == 0 ? g : 0.f; o1 = best == 1 ? g : 0.f; o2 = best == 2 ? g : 0.f; o3 = best == 3 ? g : 0.f;
}

// STATS: the gradient written here is the LAST contribution to d loss / d BN-output of this
// tensor, so the BatchNorm-backward reductions (sum dY, sum dY*xhat — bn_bwd_reduce) ride along
// and that separate pass over dY and a is not needed.  Requires C4 to be a power of two dividing
// the block (a thread's channel quad is then a loop constant).
template <bool STATS>
__global__ void __launch_bounds__(kT) pool_bwd_vec_kernel(const float* __restrict__ dp, int ld_dp, const float* __restrict__ a, int ld_a,
                                    const float* scale, const float* shift, float* __restrict__ df, int ld_df,
                                    int accumulate, int Ho, int Wo, uint32_t total, VIdx ix,
                                    const float* mean, const float* invstd, double* sums, Ordered red) {
  const int W2 = 2 * Wo;
  float4 s1 = make_float4(0, 0, 0, 0), s2 = s1, mu = s1, is = s1;
  if (STATS) {
    const int c4 = (int)(threadIdx.x & (uint32_t)(ix.C4 - 1));
    mu = ld4(mean + c4 * 4);
    is = ld4(invstd + c4 * 4);
  }
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    uint32_t pix; int c4; ix.split(i, pix, c4);
    const uint32_t wo = pix % Wo, r = pix / Wo, ho = r % Ho, n = r / Ho;
    float4 sc = make_float4(1, 1, 1, 1), sh = make_float4(0, 0, 0, 0);
    if (scale) { sc = ld4(scale + c4 * 4); sh = ld4(shift + c4 * 4); }
    const size_t base = ((size_t)n * 2 * Ho + 2 * ho) * W2 + 2 * wo;
    const size_t off[4] = {0, 1, (size_t)W2, (size_t)W2 + 1};
    float4 raw[4], v[4], o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      raw[k] = ld4(a + (base + off[k]) * ld_a + c4 * 4);
      v[k] = f4fma(raw[k], sc, sh);
    }
    const float4 g = ld4(dp + (size_t)pix * ld_dp + c4 * 4);
    pick4(v[0].x, v[1].x, v[2].x, v[3].x, g.x, o[0].x, o[1].x, o[2].x, o[3].x);
    pick4(v[0].y, v[1].y, v[2].y, v[3].y, g.y, o[0].y, o[1].y, o[2].y, o[3].y);
    pick4(v[0].z, v[1].z, v[2].z, v[3].z, g.z, o[0].z, o[1].z, o[2].z, o[3].z);
    pick4(v[0].w, v[1].w, v[2].w, v[3].w, g.w, o[0].w, o[1].w, o[2].w, o[3].w);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float4* q = reinterpret_cast<float4*>(df + (base + off[k]) * ld_df + c4 * 4);
      const float4 t = accumulate ? f4add(*q, o[k]) : o[k];
      *q = t;
      if (STATS) {
        s1 = f4add(s1, t);
        s2.x = fmaf(t.x, (raw[k].x - mu.x) * is.x, s2.x); s2.y = fmaf(t.y, (raw[k].y - mu.y) * is.y, s2.y);
        s2.z = fmaf(t.z, (raw[k].z - mu.z) * is.z, s2.z); s2.w = fmaf(t.w, (raw[k].w - mu.w) * is.w, s2.w);
      }
    }
  }
  if (STATS) {
    const int C4 = ix.C4, cx = threadIdx.x & (C4 - 1), py = threadIdx.x / C4;
    block_chan_reduce_vec(s1, s2, cx, py, C4, kT / C4, C4, sums, sums + C4 * 4, red);
  }
}

// One thread per LOW-res pixel and 4 channels: the 2 x 2 output block it covers comes from its
// 3 x 3 (edge-clamped) neighbourhood — 9 loads and one set of index arithmetic per four outputs
// (the per-output kernel above spends 4 loads and three integer divisions on each).  Same
// expression per output as up_src / the scalar kernel, so results are bit-identical.
__global__ void __launch_bounds__(kT) upsample_fwd_blk_kernel(const float* __restrict__ x, int ld_x,
                                                                float* __restrict__ y, int ld_y, int h,
                                                                int w, int bilinear, uint32_t total,
                                                                VIdx ix) {
  const int W = 2 * w;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    uint32_t pix; int c4; ix.split(i, pix, c4);
    const uint32_t iw = pix % (uint32_t)w, r = pix / (uint32_t)w, ih = r % (uint32_t)h, n = r / (uint32_t)h;
    const float* xb = x + (size_t)n * h * w * ld_x + c4 * 4;
    float* yb = y + ((size_t)(n * 2 * h + 2 * ih) * W + 2 * iw) * ld_y + c4 * 4;
    const size_t yrow = (size_t)W * ld_y;
    if (!bilinear) {
      const float4 v = ld4(xb + ((size_t)ih * w + iw) * ld_x);
      *reinterpret_cast<float4*>(yb) = v;
      *reinterpret_cast<float4*>(yb + ld_y) = v;
      *reinterpret_cast<float4*>(yb + yrow) = v;
      *reinterpret_cast<float4*>(yb + yrow + ld_y) = v;
      continue;
    }
    const int hm = ih > 0 ? (int)ih - 1 : 0, hp = (int)ih + 1 < h ? (int)ih + 1 : h - 1;
    const int wm = iw > 0 ? (int)iw - 1 : 0, wp = (int)iw + 1 < w ? (int)iw + 1 : w - 1;
    const float* rm = xb + (size_t)hm * w * ld_x;
    const float* r0 = xb + (size_t)ih * w * ld_x;
    const float* rp = xb + (size_t)hp * w * ld_x;
    const float4 mm = ld4(rm + (size_t)wm * ld_x), m0 = ld4(rm + (size_t)iw * ld_x), mp = ld4(rm + (size_t)wp * ld_x);
    const float4 zm = ld4(r0 + (size_t)wm * ld_x), z0 = ld4(r0 + (size_t)iw * ld_x), zp = ld4(r0 + (size_t)wp * ld_x);
    const float4 pm = ld4(rp + (size_t)wm * ld_x), p0 = ld4(rp + (size_t)iw * ld_x), pp = ld4(rp + (size_t)wp * ld_x);
    // even output index 2i: (x[i-1], x[i], l = 0.75)  [i = 0: l = 0];  odd 2i+1: (x[i], x[i+1], l = 0.25)
    const float lhe = ih > 0 ? 0.75f : 0.f, lwe = iw > 0 ? 0.75f : 0.f;
    auto mix4 = [&](float4 a, float4 b, float4 c, float4 d, float lh, float lw) {
      return make_float4(bil_mix(a.x, b.x, c.x, d.x, lh, lw), bil_mix(a.y, b.y, c.y, d.y, lh, lw),
                         bil_mix(a.z, b.z, c.z, d.z, lh, lw), bil_mix(a.w, b.w, c.w, d.w, lh, lw));
    };
    *reinterpret_cast<float4*>(yb) = mix4(mm, m0, zm, z0, lhe, lwe);
    *reinterpret_cast<float4*>(yb + ld_y) = mix4(m0, mp, z0, zp, lhe, 0.25f);
    *reinterpret_cast<float4*>(yb + yrow) = mix4(zm, z0, pm, p0, 0.25f, lwe);
    *reinterpret_cast<float4*>(yb + yrow + ld_y) = mix4(z0, zp, p0, pp, 0.25f, 0.25f);
  }
}

__global__ void __launch_bounds__(kT) upsample_bwd_vec_kernel(const float* __restrict__ dy, int ld_dy, float* __restrict__ dx, int ld_dx,
                                        int h, int w, int bilinear, uint32_t total, VIdx ix) {
  const int H = 2 * h, W = 2 * w;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    uint32_t pix; int c4; ix.split(i, pix, c4);
    const uint32_t iw = pix % w, r = pix / w, ih = r % h, n = r / h;
    const float* db = dy + (size_t)n * H * W * ld_dy + c4 * 4;
    float4 acc = make_float4(0, 0, 0, 0);
    if (bilinear) {
      int oh[4], ow[4]; float wh[4], ww[4];
      const int nh = up_adj((int)ih, h, oh, wh), nw = up_adj((int)iw, w, ow, ww);
      for (int a = 0; a < nh; ++a) {
        float4 row = make_float4(0, 0, 0, 0);
        for (int b = 0; b < nw; ++b) {
          const float4 g = ld4(db + ((size_t)oh[a] * W + ow[b]) * ld_dy);
          row.x = fmaf(ww[b], g.x, row.x); row.y = fmaf(ww[b], g.y, row.y);
          row.z = fmaf(ww[b], g.z, row.z); row.w = fmaf(ww[b], g.w, row.w);
        }
        acc.x = fmaf(wh[a], row.x, acc.x); acc.y = fmaf(wh[a], row.y, acc.y);
        acc.z = fmaf(wh[a], row.z, acc.z); acc.w = fmaf(wh[a], row.w, acc.w);
      }
    } else {
      const size_t b0 = ((size_t)(2 * ih) * W + 2 * iw) * ld_dy;
      acc = f4add(f4add(ld4(db + b0), ld4(db + b0 + ld_dy)),
                  f4add(ld4(db + b0 + (size_t)W * ld_dy), ld4(db + b0 + (size_t)W * ld_dy + ld_dy)));
    }
    *reinterpret_cast<float4*>(dx + (size_t)pix * ld_dx + c4 * 4) = acc;
  }
}

// batched 2-D transpose: y[n][c][r] = x[n][r][c]  (NHWC <-> NCHW around flatten/Linear)
__global__ void transpose_kernel(const float* __restrict__ x, float* __restrict__ y, int R, int Cc) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const float* xb = x + (size_t)n * R * Cc;
  float* yb = y + (size_t)n * R * Cc;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (r < R && c < Cc) ? xb[(size_t)r * Cc + c] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (r < R && c < Cc) yb[(size_t)c * R + r] = tile[threadIdx.x][i];
  }
}

}  // namespace

#define STREAM ((cudaStream_t)stream)

extern "C" {

int atomai_b200_bn_finalize(const double* stats, int C, double count, const float* gamma,
                            const float* beta, float* running_mean, float* running_var,
                            float momentum, float eps, int training, float* scale, float* shift,
                            float* mean, float* invstd, void* stream) {
  AB_CHECK(C > 0, "bn_finalize: C=%d", C);
  AB_CHECK(training || (running_mean && running_var), "bn_finalize: eval needs running stats");
  bn_finalize_kernel<<<(C + 127) / 128, 128, 0, STREAM>>>(stats, C, count, gamma, beta,
                                                          running_mean, running_var, momentum,
                                                          eps, training, scale, shift, mean,
                                                          invstd);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_affine(const float* a, int ld_a, const float* scale, const float* shift, float* y,
                       int ld_y, int64_t npix, int C, int out_nchw_hw, void* stream) {
  if (npix * C == 0) return 0;
  if (!out_nchw_hw && vec_ok(C, {a, y, scale, shift}, {ld_a, ld_y}, npix * C / 4)) {
    affine_vec_kernel<<<grid_for(npix * C / 4), kT, 0, STREAM>>>(a, ld_a, scale, shift, y, ld_y,
                                                               (uint32_t)(npix * C / 4), make_vidx(C));
    AB_LAUNCH_CHECK();
    return 0;
  }
  affine_kernel<<<grid_for(npix * C), kT, 0, STREAM>>>(a, ld_a, scale, shift, y, ld_y, npix, C,
                                                       out_nchw_hw);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_bn_bwd_reduce(const float* dy, int ld_dy, const float* a, int ld_a,
                              const float* mean, const float* invstd, int64_t npix, int C,
                              double* sums, void* stream) {
  if (npix == 0) return 0;
  if (C <= 4 * kT && vec_ok(C, {dy, a, mean, invstd}, {ld_dy, ld_a}, npix)) {
    const ChanLayout l4 = chan_layout(C / 4);
    Ordered red;
    if (red_ws(STREAM, 2 * C, &red)) return 1;
    bn_bwd_reduce_vec_kernel<<<grid_for(npix, l4.R * 8), kT, 0, STREAM>>>(
        dy, ld_dy, a, ld_a, mean, invstd, npix, C / 4, l4.CW, l4.R, sums, red);
    AB_LAUNCH_CHECK();
    return 0;
  }
  AB_CHECK(C <= kT, "bn_bwd_reduce: C=%d unsupported (max %d, or %d when C %% 4 == 0)", C, kT, 4 * kT);
  const ChanLayout l = chan_layout(C);
  Ordered red;
  if (red_ws(STREAM, 2 * C, &red)) return 1;
  bn_bwd_reduce_kernel<<<grid_for(npix, l.R * 8), kT, 0, STREAM>>>(dy, ld_dy, a, ld_a, mean,
                                                                  invstd, npix, C, l.CW, l.R,
                                                                  sums, red);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_bn_lrelu_bwd(const float* dy, int ld_dy, const float* a, int ld_a,
                             const float* mean, const float* invstd, const float* scale,
                             const double* sums, double count, const float* extra, int ld_extra,
                             int act, float lrelu, float* dpre, int ld_dpre, double* dbias,
                             int64_t npix, int C, void* stream) {
  if (npix == 0) return 0;
  Ordered red = {nullptr, nullptr};
  if (dbias && red_ws(STREAM, 2 * C, &red)) return 1;
  if (C <= 4 * kT && vec_ok(C, {dy, a, mean, invstd, scale, extra, dpre}, {dy ? ld_dy : 0, ld_a, extra ? ld_extra : 0, ld_dpre}, npix)) {
    const ChanLayout l4 = chan_layout(C / 4);
    bn_lrelu_bwd_vec_kernel<<<grid_for(npix, l4.R * 8), kT, 0, STREAM>>>(
        dy, ld_dy, a, ld_a, mean, invstd, scale, sums, count, extra, ld_extra, act, lrelu, dpre,
        ld_dpre, dbias, npix, C / 4, l4.CW, l4.R, red);
    AB_LAUNCH_CHECK();
    return 0;
  }
  AB_CHECK(C <= kT, "bn_lrelu_bwd: C=%d unsupported (max %d, or %d when C %% 4 == 0)", C, kT, 4 * kT);
  const ChanLayout l = chan_layout(C);
  bn_lrelu_bwd_kernel<<<grid_for(npix, l.R * 8), kT, 0, STREAM>>>(
      dy, ld_dy, a, ld_a, mean, invstd, scale, sums, count, extra, ld_extra, act, lrelu, dpre,
      ld_dpre, dbias, npix, C, l.CW, l.R, red);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_pool2x2_fwd(const float* a, int ld_a, const float* scale, const float* shift,
                            float* y, int ld_y, int N, int Ho, int Wo, int C, void* stream) {
  const int64_t total = (int64_t)N * Ho * Wo * C;
  if (total == 0) return 0;
  if (vec_ok(C, {a, y, scale, shift}, {ld_a, ld_y}, total / 4)) {
    pool_fwd_vec_kernel<<<grid_for(total / 4), kT, 0, STREAM>>>(a, ld_a, scale, shift, y, ld_y, Ho, Wo,
                                                              (uint32_t)(total / 4), make_vidx(C));
    AB_LAUNCH_CHECK();
    return 0;
  }
  pool_fwd_kernel<<<grid_for(total), kT, 0, STREAM>>>(a, ld_a, scale, shift, y, ld_y, N, Ho, Wo,
                                                      C);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_pool2x2_bwd_bn(const float* dp, int ld_dp, const float* a, int ld_a,
                               const float* scale, const float* shift, float* dfull, int ld_df,
                               int accumulate, int N, int Ho, int Wo, int C, const float* mean,
                               const float* invstd, double* sums, void* stream) {
  const int64_t total = (int64_t)N * Ho * Wo * C;
  if (total == 0) return 0;
  const bool stats = sums != nullptr;
  AB_CHECK(!stats || (mean && invstd), "pool2x2_bwd_bn: statistics need mean and invstd");
  if (vec_ok(C, {dp, a, dfull, scale, shift}, {ld_dp, ld_a, ld_df}, total / 4)) {
    const VIdx ix = make_vidx(C);
    if (stats) {
      AB_CHECK(ix.shift >= 0 && ix.C4 <= kT && ((uintptr_t)mean & 15) == 0 && ((uintptr_t)invstd & 15) == 0,
               "pool2x2_bwd_bn: fused statistics need C/4 = power of two <= %d (C=%d)", kT, C);
      Ordered red;
      if (red_ws(STREAM, 2 * C, &red)) return 1;
      pool_bwd_vec_kernel<true><<<grid_for(total / 4), kT, 0, STREAM>>>(
          dp, ld_dp, a, ld_a, scale, shift, dfull, ld_df, accumulate, Ho, Wo, (uint32_t)(total / 4), ix,
          mean, invstd, sums, red);
    } else {
      pool_bwd_vec_kernel<false><<<grid_for(total / 4), kT, 0, STREAM>>>(
          dp, ld_dp, a, ld_a, scale, shift, dfull, ld_df, accumulate, Ho, Wo, (uint32_t)(total / 4), ix,
          nullptr, nullptr, nullptr, Ordered{nullptr, nullptr});
    }
    AB_LAUNCH_CHECK();
    return 0;
  }
  AB_CHECK(!stats, "pool2x2_bwd_bn: fused statistics need the float4 path (C=%d)", C);
  pool_bwd_kernel<<<grid_for(total), kT, 0, STREAM>>>(dp, ld_dp, a, ld_a, scale, shift, dfull,
                                                      ld_df, accumulate, N, Ho, Wo, C);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_pool2x2_bwd(const float* dp, int ld_dp, const float* a, int ld_a,
                            const float* scale, const float* shift, float* dfull, int ld_df,
                            int accumulate, int N, int Ho, int Wo, int C, void* stream) {
  return atomai_b200_pool2x2_bwd_bn(dp, ld_dp, a, ld_a, scale, shift, dfull, ld_df, accumulate, N, Ho,
                                    Wo, C, nullptr, nullptr, nullptr, stream);
}

int atomai_b200_upsample2x_fwd(const float* x, int ld_x, float* y, int ld_y, int N, int h, int w,
                               int C, int bilinear, void* stream) {
  const int64_t total = (int64_t)N * 4 * h * w * C;
  if (total == 0) return 0;
  if (vec_ok(C, {x, y}, {ld_x, ld_y}, total / 4)) {
    const int64_t lo = (int64_t)N * h * w * (C / 4);        // one thread per low-res float4
    upsample_fwd_blk_kernel<<<grid_for(lo), kT, 0, STREAM>>>(x, ld_x, y, ld_y, h, w, bilinear,
                                                            (uint32_t)lo, make_vidx(C));
    AB_LAUNCH_CHECK();
    return 0;
  }
  upsample_fwd_kernel<<<grid_for(total), kT, 0, STREAM>>>(x, ld_x, y, ld_y, N, h, w, C, bilinear);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_upsample2x_bwd(const float* dy, int ld_dy, float* dx, int ld_dx, int N, int h,
                               int w, int C, int bilinear, void* stream) {
  const int64_t total = (int64_t)N * h * w * C;
  if (total == 0) return 0;
  if (vec_ok(C, {dy, dx}, {ld_dy, ld_dx}, total / 4)) {
    upsample_bwd_vec_kernel<<<grid_for(total / 4), kT, 0, STREAM>>>(dy, ld_dy, dx, ld_dx, h, w, bilinear,
                                                                  (uint32_t)(total / 4), make_vidx(C));
    AB_LAUNCH_CHECK();
    return 0;
  }
  upsample_bwd_kernel<<<grid_for(total), kT, 0, STREAM>>>(dy, ld_dy, dx, ld_dx, N, h, w, C,
                                                          bilinear);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_add_slice(const float* src, int ld_s, float* dst, int ld_d, int accumulate,
                          int64_t npix, int C, void* stream) {
  if (npix * C == 0) return 0;
  if (vec_ok(C, {src, dst}, {ld_s, ld_d}, npix * C / 4)) {
    add_slice_vec_kernel<<<grid_for(npix * C / 4), kT, 0, STREAM>>>(src, ld_s, dst, ld_d, accumulate,
                                                                  (uint32_t)(npix * C / 4), make_vidx(C));
    AB_LAUNCH_CHECK();
    return 0;
  }
  add_slice_kernel<<<grid_for(npix * C), kT, 0, STREAM>>>(src, ld_s, dst, ld_d, accumulate, npix,
                                                          C);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_dilated_sum(const float* const* a_ptrs, const float* const* scale_ptrs,
                            const float* const* shift_ptrs, int nlayers, float lrelu, float* out,
                            int64_t n_elems, int C, void* stream) {
  AB_CHECK(nlayers >= 1 && nlayers <= kMaxDil, "dilated_sum: nlayers=%d (max %d)", nlayers,
           kMaxDil);
  AB_CHECK(lrelu != 0.f, "dilated_sum: LeakyReLU slope 0 is not invertible");
  DilPtrs P;
  for (int l = 0; l < kMaxDil; ++l) {
    P.a[l] = l < nlayers ? a_ptrs[l] : nullptr;
    P.scale[l] = (l < nlayers && scale_ptrs) ? scale_ptrs[l] : nullptr;
    P.shift[l] = (l < nlayers && shift_ptrs) ? shift_ptrs[l] : nullptr;
  }
  if (n_elems == 0) return 0;
  dilated_sum_kernel<<<grid_for(n_elems), kT, 0, STREAM>>>(P, nlayers, lrelu, out, n_elems, C);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_ce_fwd_bwd(const float* logits, int ld, const int64_t* labels, int64_t npix, int C,
                           double* loss_sum, float* dlogits, int ld_d, float gscale,
                           const float* gscale_dev, void* stream) {
  if (npix == 0) return 0;
  Ordered red = {nullptr, nullptr};
  if (loss_sum && red_ws(STREAM, 1, &red)) return 1;
  ce_kernel<<<grid_for(npix), kT, 0, STREAM>>>(logits, ld, labels, npix, C, loss_sum, dlogits,
                                               ld_d, gscale, gscale_dev, red);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_pointwise_loss(const float* pred, const float* target, int64_t n, int kind,
                               double* loss_sum, float* dpred, float gscale,
                               const float* gscale_dev, void* stream) {
  AB_CHECK(kind == 0 || kind == 1, "pointwise_loss: kind=%d", kind);
  if (n == 0) return 0;
  Ordered red = {nullptr, nullptr};
  if (loss_sum && red_ws(STREAM, 1, &red)) return 1;
  pointwise_loss_kernel<<<grid_for(n), kT, 0, STREAM>>>(pred, target, n, kind, loss_sum, dpred,
                                                        gscale, gscale_dev, red);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_sqerr_reduce(const float* x, const float* xhat, int64_t n, double* out,
                             float* dxhat, float gscale, const float* gscale_dev, void* stream) {
  if (n == 0) return 0;
  Ordered red = {nullptr, nullptr};
  if (out && red_ws(STREAM, 1, &red)) return 1;
  sqerr_kernel<<<grid_for(n), kT, 0, STREAM>>>(x, xhat, n, out, dxhat, gscale, gscale_dev, red);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_transpose(const float* x, float* y, int N, int R, int Cc, void* stream) {
  AB_CHECK(x && y && N >= 0 && R > 0 && Cc > 0, "transpose: bad arguments");
  if (N == 0) return 0;
  AB_CHECK(N <= 65535 && (R + 31) / 32 <= 65535, "transpose: grid too large");
  dim3 grid((Cc + 31) / 32, (R + 31) / 32, N), block(32, 8);
  transpose_kernel<<<grid, block, 0, STREAM>>>(x, y, R, Cc);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_adam_multi(const int64_t* table_dev, int n, int64_t max_numel, float lr,
                           float beta1, float beta2, float eps, float weight_decay, int step,
                           float grad_scale, void* stream) {
  if (n == 0 || max_numel == 0) return 0;
  AB_CHECK(step >= 1, "adam: step=%d", step);
  AB_CHECK(n <= 65535, "adam: too many tensors (%d)", n);
  const float bc1 = 1.f - powf(beta1, (float)step);
  const float bc2 = 1.f - powf(beta2, (float)step);
  int gx = (int)((max_numel + kT * 4 - 1) / (kT * 4));
  if (gx > 64) gx = 64;
  if (gx < 1) gx = 1;
  dim3 grid(gx, n);
  adam_multi_kernel<<<grid, kT, 0, STREAM>>>(table_dev, lr, beta1, beta2, eps, weight_decay, bc1,
                                             sqrtf(bc2), grad_scale);
  AB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
