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
#include "common.cuh"

namespace {

constexpr int kT = 256;
constexpr int kCtasPerSm = 8;  // grid cap of every launch here (ab_grid)

// workspace of an ordered cross-CTA sum of n values per CTA for a launch of ab_grid() CTAs
int red_ws(cudaStream_t stream, int n, Ordered* red) {
  return ab_ordered_ws(stream, (int64_t)ab_num_sms() * kCtasPerSm * n, 1, red);
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
// Each kernel below runs W = 4 channels per thread on the float4 path and W = 1 otherwise
// (common.cuh: Lanes, ChanIdx, vec_ok); the grid-stride loop walks (pixel, channel group) items.
// hw_nchw (W = 1 only): y is written NCHW with hw_nchw pixels per image.
template <int W>
__global__ void __launch_bounds__(kT) affine_kernel(const float* __restrict__ a, int ld_a,
                                                    const float* scale, const float* shift,
                                                    float* __restrict__ y, int ld_y,
                                                    typename ChanIdx<W>::I total, ChanIdx<W> ix,
                                                    int hw_nchw) {
  using I = typename ChanIdx<W>::I;
  for (I i = blockIdx.x * (I)blockDim.x + threadIdx.x; i < total; i += (I)gridDim.x * blockDim.x) {
    I pix; int c; ix.split(i, pix, c);
    Lanes<W> v = lanes_ld<W>(a + (size_t)pix * ld_a + c);
    if (scale) {
      const Lanes<W> s = lanes_ld<W>(scale + c), t = lanes_ld<W>(shift + c);
#pragma unroll
      for (int k = 0; k < W; ++k) v[k] = fmaf(v[k], s[k], t[k]);
    }
    if constexpr (W == 1) {
      if (hw_nchw) {
        const int64_t n = pix / hw_nchw, r = pix % hw_nchw;
        y[(n * ix.C + c) * hw_nchw + r] = v[0];
        continue;
      }
    }
    lanes_at<W>(y + (size_t)pix * ld_y + c) = v;
  }
}

// ---------------------------------------------------------------- per-channel reductions
// Thread layout: CW = pow2 >= CG (<= 256) lanes of W channels each (CG = C / W channel groups),
// R = 256/CW pixel rows per CTA step.
struct ChanLayout {
  int CW, R;
};
inline ChanLayout chan_layout(int CG) {
  int cw = 1;
  while (cw < CG) cw <<= 1;
  ChanLayout l;
  l.CW = cw;
  l.R = kT / cw;
  return l;
}

// The CTA's per-channel totals (rows r = 0..R-1 in order) go into its slot of an ordered cross-CTA
// sum (common.cuh): C sums of v1, then C sums of v2.  The result does not depend on which CTA
// finishes first.
template <int W>
__device__ __forceinline__ void block_chan_reduce(Lanes<W> v1, Lanes<W> v2, int cx, int py, int CW,
                                                  int R, int CG, double* out1, double* out2,
                                                  const Ordered& red) {
  __shared__ Lanes<W> s1[kT], s2[kT];
  s1[py * CW + cx] = v1;
  s2[py * CW + cx] = v2;
  __syncthreads();
  const int C = W * CG;
  if (py == 0 && cx < CG) {
    Lanes<W> a = lanes_fill<W>(0.f), b = a;
    for (int r = 0; r < R; ++r) {
      const Lanes<W> x1 = s1[r * CW + cx], x2 = s2[r * CW + cx];
#pragma unroll
      for (int k = 0; k < W; ++k) { a[k] += x1[k]; b[k] += x2[k]; }
    }
    double* slot = ordered_slot(red, 0, gridDim.x, blockIdx.x, 2 * C);
#pragma unroll
    for (int k = 0; k < W; ++k) { slot[cx * W + k] = a[k]; slot[C + cx * W + k] = b[k]; }
  }
  __shared__ unsigned s_last;
  ordered_finish(red, 0, gridDim.x, 2 * C, threadIdx.x, kT, gridDim.x, [] { __syncthreads(); },
                 [&](int i, double v) {
                   double* o = i < C ? out1 : out2;
                   if (o) o[i < C ? i : i - C] += v;
                 },
                 &s_last);
}

template <int W>
__global__ void __launch_bounds__(kT) bn_bwd_reduce_kernel(const float* __restrict__ dy, int ld_dy,
                                                           const float* __restrict__ a, int ld_a,
                                                           const float* mean, const float* invstd,
                                                           int64_t npix, int CG, int CW, int R,
                                                           double* sums, Ordered red) {
  const int cx = threadIdx.x % CW, py = threadIdx.x / CW, c = cx * W;
  Lanes<W> s1 = lanes_fill<W>(0.f), s2 = s1;
  if (cx < CG) {
    const Lanes<W> m = lanes_ld<W>(mean + c), is = lanes_ld<W>(invstd + c);
    for (int64_t p = (int64_t)blockIdx.x * R + py; p < npix; p += (int64_t)gridDim.x * R) {
      const Lanes<W> g = lanes_ld<W>(dy + p * ld_dy + c), av = lanes_ld<W>(a + p * ld_a + c);
#pragma unroll
      for (int k = 0; k < W; ++k) {
        s1[k] += g[k];
        s2[k] = fmaf(g[k], (av[k] - m[k]) * is[k], s2[k]);
      }
    }
  }
  block_chan_reduce<W>(s1, s2, cx, py, CW, R, CG, sums, sums + W * CG, red);
}

__device__ __forceinline__ float bwd1(float g, float av, bool bn, float m, float is, float sc, float k1, float k2,
                                      float ex, bool has_ex, int act, float alpha) {
  if (bn) g = sc * (g - k1 - (av - m) * is * k2);
  if (has_ex) g += ex;
  return g * act_grad_from_out(av, act, alpha) + (has_ex ? ex : 0.f);
}

template <int W>
__global__ void __launch_bounds__(kT)
    bn_lrelu_bwd_kernel(const float* __restrict__ dy, int ld_dy, const float* __restrict__ a,
                        int ld_a, const float* mean, const float* invstd, const float* scale,
                        const double* sums, double count, const float* __restrict__ extra,
                        int ld_extra, int act, float alpha, float* __restrict__ dpre, int ld_dpre,
                        double* dbias, int64_t npix, int CG, int CW, int R, Ordered red) {
  const int cx = threadIdx.x % CW, py = threadIdx.x / CW, c = cx * W;
  Lanes<W> sb = lanes_fill<W>(0.f);
  if (cx < CG) {
    const bool bn = scale != nullptr, has_ex = extra != nullptr;
    Lanes<W> m = sb, is = sb, sc = sb, k1 = sb, k2 = sb;
    if (bn) {
      const int C = W * CG;
      m = lanes_ld<W>(mean + c);
      is = lanes_ld<W>(invstd + c);
      sc = lanes_ld<W>(scale + c);
#pragma unroll
      for (int k = 0; k < W; ++k) {
        k1[k] = (float)(sums[c + k] / count);
        k2[k] = (float)(sums[C + c + k] / count);
      }
    }
    for (int64_t p = (int64_t)blockIdx.x * R + py; p < npix; p += (int64_t)gridDim.x * R) {
      const Lanes<W> av = lanes_ld<W>(a + p * ld_a + c);
      const Lanes<W> g = dy ? lanes_ld<W>(dy + p * ld_dy + c) : lanes_fill<W>(0.f);
      const Lanes<W> ex = has_ex ? lanes_ld<W>(extra + p * ld_extra + c) : lanes_fill<W>(0.f);
      Lanes<W> d;
#pragma unroll
      for (int k = 0; k < W; ++k)
        d[k] = bwd1(g[k], av[k], bn, m[k], is[k], sc[k], k1[k], k2[k], ex[k], has_ex, act, alpha);
      lanes_at<W>(dpre + p * ld_dpre + c) = d;
#pragma unroll
      for (int k = 0; k < W; ++k) sb[k] += d[k];
    }
  }
  if (dbias) block_chan_reduce<W>(sb, lanes_fill<W>(0.f), cx, py, CW, R, CG, dbias, nullptr, red);
}

// ---------------------------------------------------------------- 2x2 max pool
template <int W>
__global__ void __launch_bounds__(kT) pool_fwd_kernel(const float* __restrict__ a, int ld_a,
                                                      const float* scale, const float* shift,
                                                      float* __restrict__ y, int ld_y, int Ho,
                                                      int Wo, typename ChanIdx<W>::I total,
                                                      ChanIdx<W> ix) {
  using I = typename ChanIdx<W>::I;
  const int W2 = 2 * Wo;
  for (I i = blockIdx.x * (I)blockDim.x + threadIdx.x; i < total; i += (I)gridDim.x * blockDim.x) {
    I pix; int c; ix.split(i, pix, c);
    const I wo = pix % (I)Wo, r = pix / (I)Wo, ho = r % (I)Ho, n = r / (I)Ho;
    Lanes<W> sc = lanes_fill<W>(1.f), sh = lanes_fill<W>(0.f);
    if (scale) { sc = lanes_ld<W>(scale + c); sh = lanes_ld<W>(shift + c); }
    const float* b = a + (((size_t)n * 2 * Ho + 2 * ho) * W2 + 2 * wo) * ld_a + c;
    const Lanes<W> v0 = lanes_ld<W>(b), v1 = lanes_ld<W>(b + ld_a);
    const Lanes<W> v2 = lanes_ld<W>(b + (size_t)W2 * ld_a), v3 = lanes_ld<W>(b + (size_t)W2 * ld_a + ld_a);
    Lanes<W> v;
#pragma unroll
    for (int k = 0; k < W; ++k)
      v[k] = fmaxf(fmaxf(fmaf(v0[k], sc[k], sh[k]), fmaf(v1[k], sc[k], sh[k])),
                   fmaxf(fmaf(v2[k], sc[k], sh[k]), fmaf(v3[k], sc[k], sh[k])));
    lanes_at<W>(y + (size_t)pix * ld_y + c) = v;
  }
}

// the gradient g goes to the first maximum of the window, as in ATen's max_pool2d
__device__ __forceinline__ void pick4(float v0, float v1, float v2, float v3, float g, float& o0, float& o1, float& o2, float& o3) {
  int best = 0; float bv = v0;
  if (v1 > bv) { bv = v1; best = 1; }
  if (v2 > bv) { bv = v2; best = 2; }
  if (v3 > bv) { bv = v3; best = 3; }
  o0 = best == 0 ? g : 0.f; o1 = best == 1 ? g : 0.f; o2 = best == 2 ? g : 0.f; o3 = best == 3 ? g : 0.f;
}

// STATS: the gradient written here is the LAST contribution to d loss / d BN-output of this
// tensor, so the BatchNorm-backward reductions (sum dY, sum dY*xhat — bn_bwd_reduce) ride along
// and that separate pass over dY and a is not needed.  Float4 path only; requires C/4 to be a
// power of two dividing the block (a thread's channel quad is then a loop constant).
template <int W, bool STATS>
__global__ void __launch_bounds__(kT) pool_bwd_kernel(const float* __restrict__ dp, int ld_dp, const float* __restrict__ a, int ld_a,
                                    const float* scale, const float* shift, float* __restrict__ df, int ld_df,
                                    int accumulate, int Ho, int Wo, typename ChanIdx<W>::I total, ChanIdx<W> ix,
                                    const float* mean, const float* invstd, double* sums, Ordered red) {
  static_assert(!STATS || W == 4, "fused statistics run on the float4 path only");
  using I = typename ChanIdx<W>::I;
  const int W2 = 2 * Wo;
  Lanes<W> s1 = lanes_fill<W>(0.f), s2 = s1, mu = s1, is = s1;
  if constexpr (STATS) {
    const int c = (int)(threadIdx.x & (uint32_t)(ix.C4 - 1)) * 4;
    mu = lanes_ld<W>(mean + c);
    is = lanes_ld<W>(invstd + c);
  }
  for (I i = blockIdx.x * (I)blockDim.x + threadIdx.x; i < total; i += (I)gridDim.x * blockDim.x) {
    I pix; int c; ix.split(i, pix, c);
    const I wo = pix % (I)Wo, r = pix / (I)Wo, ho = r % (I)Ho, n = r / (I)Ho;
    Lanes<W> sc = lanes_fill<W>(1.f), sh = lanes_fill<W>(0.f);
    if (scale) { sc = lanes_ld<W>(scale + c); sh = lanes_ld<W>(shift + c); }
    const size_t base = ((size_t)n * 2 * Ho + 2 * ho) * W2 + 2 * wo;
    const size_t off[4] = {0, 1, (size_t)W2, (size_t)W2 + 1};
    Lanes<W> raw[4], v[4], o[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      raw[q] = lanes_ld<W>(a + (base + off[q]) * ld_a + c);
#pragma unroll
      for (int k = 0; k < W; ++k) v[q][k] = fmaf(raw[q][k], sc[k], sh[k]);
    }
    const Lanes<W> g = lanes_ld<W>(dp + (size_t)pix * ld_dp + c);
#pragma unroll
    for (int k = 0; k < W; ++k)
      pick4(v[0][k], v[1][k], v[2][k], v[3][k], g[k], o[0][k], o[1][k], o[2][k], o[3][k]);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      Lanes<W>& dst = lanes_at<W>(df + (base + off[q]) * ld_df + c);
      Lanes<W> t = o[q];
      if (accumulate) {
        const Lanes<W> prev = dst;
#pragma unroll
        for (int k = 0; k < W; ++k) t[k] = prev[k] + o[q][k];
      }
      dst = t;
      if constexpr (STATS) {
#pragma unroll
        for (int k = 0; k < W; ++k) {
          s1[k] += t[k];
          s2[k] = fmaf(t[k], (raw[q][k] - mu[k]) * is[k], s2[k]);
        }
      }
    }
  }
  if constexpr (STATS) {
    const int C4 = ix.C4, cx = threadIdx.x & (C4 - 1), py = threadIdx.x / C4;
    block_chan_reduce<W>(s1, s2, cx, py, C4, kT / C4, C4, sums, sums + C4 * 4, red);
  }
}

// ---------------------------------------------------------------- x2 upsampling
// (1-lh)((1-lw)a + lw b) + lh((1-lw)c + lw d), with the FMAs spelled out: each sum is one FMA of
// its first product onto the rounded second product, so the bits do not depend on how the
// compiler would contract the expression.
__device__ __forceinline__ float bil_mix(float a, float b, float c, float d, float lh, float lw) {
  const float top = fmaf(1.f - lw, a, __fmul_rn(lw, b));
  const float bot = fmaf(1.f - lw, c, __fmul_rn(lw, d));
  return fmaf(1.f - lh, top, __fmul_rn(lh, bot));
}

// One thread per LOW-res pixel and W channels: the 2 x 2 output block it covers comes from its
// 3 x 3 (edge-clamped) neighbourhood — 9 loads and one set of index arithmetic per four outputs.
// align_corners = False, scale 2: even output 2i mixes (x[i-1], x[i]) with weight 0.75 on x[i]
// (i = 0: weight 0 on the clamped x[-1] = x[0]), odd 2i+1 mixes (x[i], x[i+1]) with weight 0.25.
template <int W>
__global__ void __launch_bounds__(kT) upsample_fwd_kernel(const float* __restrict__ x, int ld_x,
                                                          float* __restrict__ y, int ld_y, int h,
                                                          int w, int bilinear,
                                                          typename ChanIdx<W>::I total,
                                                          ChanIdx<W> ix) {
  using I = typename ChanIdx<W>::I;
  const int W2 = 2 * w;
  for (I i = blockIdx.x * (I)blockDim.x + threadIdx.x; i < total; i += (I)gridDim.x * blockDim.x) {
    I pix; int c; ix.split(i, pix, c);
    const I iw = pix % (I)w, r = pix / (I)w, ih = r % (I)h, n = r / (I)h;
    const float* xb = x + (size_t)n * h * w * ld_x + c;
    float* yb = y + ((size_t)(n * 2 * h + 2 * ih) * W2 + 2 * iw) * ld_y + c;
    const size_t yrow = (size_t)W2 * ld_y;
    if (!bilinear) {
      const Lanes<W> v = lanes_ld<W>(xb + ((size_t)ih * w + iw) * ld_x);
      lanes_at<W>(yb) = v;
      lanes_at<W>(yb + ld_y) = v;
      lanes_at<W>(yb + yrow) = v;
      lanes_at<W>(yb + yrow + ld_y) = v;
      continue;
    }
    const int hm = ih > 0 ? (int)ih - 1 : 0, hp = (int)ih + 1 < h ? (int)ih + 1 : h - 1;
    const int wm = iw > 0 ? (int)iw - 1 : 0, wp = (int)iw + 1 < w ? (int)iw + 1 : w - 1;
    const float* rm = xb + (size_t)hm * w * ld_x;
    const float* r0 = xb + (size_t)ih * w * ld_x;
    const float* rp = xb + (size_t)hp * w * ld_x;
    const Lanes<W> mm = lanes_ld<W>(rm + (size_t)wm * ld_x), m0 = lanes_ld<W>(rm + (size_t)iw * ld_x), mp = lanes_ld<W>(rm + (size_t)wp * ld_x);
    const Lanes<W> zm = lanes_ld<W>(r0 + (size_t)wm * ld_x), z0 = lanes_ld<W>(r0 + (size_t)iw * ld_x), zp = lanes_ld<W>(r0 + (size_t)wp * ld_x);
    const Lanes<W> pm = lanes_ld<W>(rp + (size_t)wm * ld_x), p0 = lanes_ld<W>(rp + (size_t)iw * ld_x), pp = lanes_ld<W>(rp + (size_t)wp * ld_x);
    const float lhe = ih > 0 ? 0.75f : 0.f, lwe = iw > 0 ? 0.75f : 0.f;
    auto mix = [&](const Lanes<W>& a, const Lanes<W>& b, const Lanes<W>& c, const Lanes<W>& d, float lh, float lw) {
      Lanes<W> o;
#pragma unroll
      for (int k = 0; k < W; ++k) o[k] = bil_mix(a[k], b[k], c[k], d[k], lh, lw);
      return o;
    };
    lanes_at<W>(yb) = mix(mm, m0, zm, z0, lhe, lwe);
    lanes_at<W>(yb + ld_y) = mix(m0, mp, z0, zp, lhe, 0.25f);
    lanes_at<W>(yb + yrow) = mix(zm, z0, pm, p0, 0.25f, lwe);
    lanes_at<W>(yb + yrow + ld_y) = mix(z0, zp, p0, pp, 0.25f, 0.25f);
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

template <int W>
__global__ void __launch_bounds__(kT) upsample_bwd_kernel(const float* __restrict__ dy, int ld_dy,
                                                          float* __restrict__ dx, int ld_dx, int h,
                                                          int w, int bilinear,
                                                          typename ChanIdx<W>::I total,
                                                          ChanIdx<W> ix) {
  using I = typename ChanIdx<W>::I;
  const int H2 = 2 * h, W2 = 2 * w;
  for (I i = blockIdx.x * (I)blockDim.x + threadIdx.x; i < total; i += (I)gridDim.x * blockDim.x) {
    I pix; int c; ix.split(i, pix, c);
    const I iw = pix % (I)w, r = pix / (I)w, ih = r % (I)h, n = r / (I)h;
    const float* db = dy + (size_t)n * H2 * W2 * ld_dy + c;
    Lanes<W> acc = lanes_fill<W>(0.f);
    if (bilinear) {
      int oh[4], ow[4]; float wh[4], ww[4];
      const int nh = up_adj((int)ih, h, oh, wh), nw = up_adj((int)iw, w, ow, ww);
      for (int a = 0; a < nh; ++a) {
        Lanes<W> row = lanes_fill<W>(0.f);
        for (int b = 0; b < nw; ++b) {
          const Lanes<W> g = lanes_ld<W>(db + ((size_t)oh[a] * W2 + ow[b]) * ld_dy);
#pragma unroll
          for (int k = 0; k < W; ++k) row[k] = fmaf(ww[b], g[k], row[k]);
        }
#pragma unroll
        for (int k = 0; k < W; ++k) acc[k] = fmaf(wh[a], row[k], acc[k]);
      }
    } else {  // (top pair) + (bottom pair)
      const size_t b0 = ((size_t)(2 * ih) * W2 + 2 * iw) * ld_dy;
      const Lanes<W> t0 = lanes_ld<W>(db + b0), t1 = lanes_ld<W>(db + b0 + ld_dy);
      const Lanes<W> b0v = lanes_ld<W>(db + b0 + (size_t)W2 * ld_dy), b1v = lanes_ld<W>(db + b0 + (size_t)W2 * ld_dy + ld_dy);
#pragma unroll
      for (int k = 0; k < W; ++k) acc[k] = (t0[k] + t1[k]) + (b0v[k] + b1v[k]);
    }
    lanes_at<W>(dx + (size_t)pix * ld_dx + c) = acc;
  }
}

template <int W>
__global__ void __launch_bounds__(kT) add_slice_kernel(const float* __restrict__ src, int ld_s,
                                                       float* __restrict__ dst, int ld_d,
                                                       int accumulate, typename ChanIdx<W>::I total,
                                                       ChanIdx<W> ix) {
  using I = typename ChanIdx<W>::I;
  for (I i = blockIdx.x * (I)blockDim.x + threadIdx.x; i < total; i += (I)gridDim.x * blockDim.x) {
    I pix; int c; ix.split(i, pix, c);
    Lanes<W> v = lanes_ld<W>(src + (size_t)pix * ld_s + c);
    Lanes<W>& o = lanes_at<W>(dst + (size_t)pix * ld_d + c);
    if (accumulate) {
      const Lanes<W> prev = o;
#pragma unroll
      for (int k = 0; k < W; ++k) v[k] = v[k] + prev[k];
    }
    o = v;
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
// CTA total of every thread's `local`, times `mul`, into the CTA's ordered slot; the last CTA adds
// the slots in order to *out (nothing is summed when out is null)
__device__ __forceinline__ void cta_sum_ordered(float local, double mul, double* out,
                                                const Ordered& red) {
  if (!out) return;
  __shared__ float wred[kT / 32];
  const float ws = warp_sum(local);
  if ((threadIdx.x & 31) == 0) wred[threadIdx.x >> 5] = ws;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < kT / 32; ++i) t += wred[i];
    ordered_slot(red, 0, gridDim.x, blockIdx.x, 1)[0] = mul * (double)t;
  }
  __shared__ unsigned s_last;
  ordered_finish(red, 0, gridDim.x, 1, threadIdx.x, kT, gridDim.x, [] { __syncthreads(); },
                 [&](int, double v) { *out += v; }, &s_last);
}

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
  cta_sum_ordered(local, 1.0, loss_sum, red);
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
  cta_sum_ordered(local, 1.0, loss_sum, red);
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
  cta_sum_ordered(local, 0.5, out, red);
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

// The entry points below run their kernel at W = 4 when vec_ok() holds and at W = 1 otherwise
// (by_width); the launch geometry of each width is part of the result (ordered sums).
int atomai_b200_affine(const float* a, int ld_a, const float* scale, const float* shift, float* y,
                       int ld_y, int64_t npix, int C, int out_nchw_hw, void* stream) {
  if (npix * C == 0) return 0;
  const bool vec = !out_nchw_hw && vec_ok(C, {a, y, scale, shift}, {ld_a, ld_y}, npix * C / 4);
  return by_width(vec, [&](auto vw) {
    constexpr int W = decltype(vw)::value;
    affine_kernel<W><<<ab_grid(npix * C / W, kT, kCtasPerSm), kT, 0, STREAM>>>(
        a, ld_a, scale, shift, y, ld_y, npix * C / W, ChanIdx<W>(C), out_nchw_hw);
    AB_LAUNCH_CHECK();
    return 0;
  });
}

int atomai_b200_bn_bwd_reduce(const float* dy, int ld_dy, const float* a, int ld_a,
                              const float* mean, const float* invstd, int64_t npix, int C,
                              double* sums, void* stream) {
  if (npix == 0) return 0;
  const bool vec = C <= 4 * kT && vec_ok(C, {dy, a, mean, invstd}, {ld_dy, ld_a}, npix);
  return by_width(vec, [&](auto vw) {
    constexpr int W = decltype(vw)::value;
    AB_CHECK(C <= W * kT, "bn_bwd_reduce: C=%d unsupported (max %d, or %d when C %% 4 == 0)", C, kT, 4 * kT);
    const ChanLayout l = chan_layout(C / W);
    Ordered red;
    if (red_ws(STREAM, 2 * C, &red)) return 1;
    bn_bwd_reduce_kernel<W><<<ab_grid(npix, l.R * 8, kCtasPerSm), kT, 0, STREAM>>>(
        dy, ld_dy, a, ld_a, mean, invstd, npix, C / W, l.CW, l.R, sums, red);
    AB_LAUNCH_CHECK();
    return 0;
  });
}

int atomai_b200_bn_lrelu_bwd(const float* dy, int ld_dy, const float* a, int ld_a,
                             const float* mean, const float* invstd, const float* scale,
                             const double* sums, double count, const float* extra, int ld_extra,
                             int act, float lrelu, float* dpre, int ld_dpre, double* dbias,
                             int64_t npix, int C, void* stream) {
  if (npix == 0) return 0;
  Ordered red = {nullptr, nullptr};
  if (dbias && red_ws(STREAM, 2 * C, &red)) return 1;
  const bool vec = C <= 4 * kT && vec_ok(C, {dy, a, mean, invstd, scale, extra, dpre},
                                         {dy ? ld_dy : 0, ld_a, extra ? ld_extra : 0, ld_dpre}, npix);
  return by_width(vec, [&](auto vw) {
    constexpr int W = decltype(vw)::value;
    AB_CHECK(C <= W * kT, "bn_lrelu_bwd: C=%d unsupported (max %d, or %d when C %% 4 == 0)", C, kT, 4 * kT);
    const ChanLayout l = chan_layout(C / W);
    bn_lrelu_bwd_kernel<W><<<ab_grid(npix, l.R * 8, kCtasPerSm), kT, 0, STREAM>>>(
        dy, ld_dy, a, ld_a, mean, invstd, scale, sums, count, extra, ld_extra, act, lrelu, dpre,
        ld_dpre, dbias, npix, C / W, l.CW, l.R, red);
    AB_LAUNCH_CHECK();
    return 0;
  });
}

int atomai_b200_pool2x2_fwd(const float* a, int ld_a, const float* scale, const float* shift,
                            float* y, int ld_y, int N, int Ho, int Wo, int C, void* stream) {
  const int64_t total = (int64_t)N * Ho * Wo * C;
  if (total == 0) return 0;
  return by_width(vec_ok(C, {a, y, scale, shift}, {ld_a, ld_y}, total / 4), [&](auto vw) {
    constexpr int W = decltype(vw)::value;
    pool_fwd_kernel<W><<<ab_grid(total / W, kT, kCtasPerSm), kT, 0, STREAM>>>(
        a, ld_a, scale, shift, y, ld_y, Ho, Wo, total / W, ChanIdx<W>(C));
    AB_LAUNCH_CHECK();
    return 0;
  });
}

int atomai_b200_pool2x2_bwd_bn(const float* dp, int ld_dp, const float* a, int ld_a,
                               const float* scale, const float* shift, float* dfull, int ld_df,
                               int accumulate, int N, int Ho, int Wo, int C, const float* mean,
                               const float* invstd, double* sums, void* stream) {
  const int64_t total = (int64_t)N * Ho * Wo * C;
  if (total == 0) return 0;
  const bool stats = sums != nullptr;
  AB_CHECK(!stats || (mean && invstd), "pool2x2_bwd_bn: statistics need mean and invstd");
  const bool vec = vec_ok(C, {dp, a, dfull, scale, shift}, {ld_dp, ld_a, ld_df}, total / 4);
  return by_width(vec, [&](auto vw) {
    constexpr int W = decltype(vw)::value;
    const ChanIdx<W> ix(C);
    const int grid = ab_grid(total / W, kT, kCtasPerSm);
    if constexpr (W == 4) {
      if (stats) {
        AB_CHECK(ix.shift >= 0 && ix.C4 <= kT && ((uintptr_t)mean & 15) == 0 && ((uintptr_t)invstd & 15) == 0,
                 "pool2x2_bwd_bn: fused statistics need C/4 = power of two <= %d (C=%d)", kT, C);
        Ordered red;
        if (red_ws(STREAM, 2 * C, &red)) return 1;
        pool_bwd_kernel<4, true><<<grid, kT, 0, STREAM>>>(
            dp, ld_dp, a, ld_a, scale, shift, dfull, ld_df, accumulate, Ho, Wo, total / 4, ix,
            mean, invstd, sums, red);
        AB_LAUNCH_CHECK();
        return 0;
      }
    }
    AB_CHECK(!stats, "pool2x2_bwd_bn: fused statistics need the float4 path (C=%d)", C);
    pool_bwd_kernel<W, false><<<grid, kT, 0, STREAM>>>(
        dp, ld_dp, a, ld_a, scale, shift, dfull, ld_df, accumulate, Ho, Wo, total / W, ix,
        nullptr, nullptr, nullptr, Ordered{nullptr, nullptr});
    AB_LAUNCH_CHECK();
    return 0;
  });
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
  return by_width(vec_ok(C, {x, y}, {ld_x, ld_y}, total / 4), [&](auto vw) {
    constexpr int W = decltype(vw)::value;
    const int64_t lo = (int64_t)N * h * w * (C / W);  // one thread per low-res pixel and W channels
    upsample_fwd_kernel<W><<<ab_grid(lo, kT, kCtasPerSm), kT, 0, STREAM>>>(
        x, ld_x, y, ld_y, h, w, bilinear, lo, ChanIdx<W>(C));
    AB_LAUNCH_CHECK();
    return 0;
  });
}

int atomai_b200_upsample2x_bwd(const float* dy, int ld_dy, float* dx, int ld_dx, int N, int h,
                               int w, int C, int bilinear, void* stream) {
  const int64_t total = (int64_t)N * h * w * C;
  if (total == 0) return 0;
  return by_width(vec_ok(C, {dy, dx}, {ld_dy, ld_dx}, total / 4), [&](auto vw) {
    constexpr int W = decltype(vw)::value;
    upsample_bwd_kernel<W><<<ab_grid(total / W, kT, kCtasPerSm), kT, 0, STREAM>>>(
        dy, ld_dy, dx, ld_dx, h, w, bilinear, total / W, ChanIdx<W>(C));
    AB_LAUNCH_CHECK();
    return 0;
  });
}

int atomai_b200_add_slice(const float* src, int ld_s, float* dst, int ld_d, int accumulate,
                          int64_t npix, int C, void* stream) {
  if (npix * C == 0) return 0;
  return by_width(vec_ok(C, {src, dst}, {ld_s, ld_d}, npix * C / 4), [&](auto vw) {
    constexpr int W = decltype(vw)::value;
    add_slice_kernel<W><<<ab_grid(npix * C / W, kT, kCtasPerSm), kT, 0, STREAM>>>(
        src, ld_s, dst, ld_d, accumulate, npix * C / W, ChanIdx<W>(C));
    AB_LAUNCH_CHECK();
    return 0;
  });
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
  dilated_sum_kernel<<<ab_grid(n_elems, kT, kCtasPerSm), kT, 0, STREAM>>>(P, nlayers, lrelu, out, n_elems, C);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_ce_fwd_bwd(const float* logits, int ld, const int64_t* labels, int64_t npix, int C,
                           double* loss_sum, float* dlogits, int ld_d, float gscale,
                           const float* gscale_dev, void* stream) {
  if (npix == 0) return 0;
  Ordered red = {nullptr, nullptr};
  if (loss_sum && red_ws(STREAM, 1, &red)) return 1;
  ce_kernel<<<ab_grid(npix, kT, kCtasPerSm), kT, 0, STREAM>>>(logits, ld, labels, npix, C, loss_sum, dlogits,
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
  pointwise_loss_kernel<<<ab_grid(n, kT, kCtasPerSm), kT, 0, STREAM>>>(pred, target, n, kind, loss_sum, dpred,
                                                        gscale, gscale_dev, red);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_sqerr_reduce(const float* x, const float* xhat, int64_t n, double* out,
                             float* dxhat, float gscale, const float* gscale_dev, void* stream) {
  if (n == 0) return 0;
  Ordered red = {nullptr, nullptr};
  if (out && red_ws(STREAM, 1, &red)) return 1;
  sqerr_kernel<<<ab_grid(n, kT, kCtasPerSm), kT, 0, STREAM>>>(x, xhat, n, out, dxhat, gscale, gscale_dev, red);
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
