// mobilenet.cu — the MobileNetV2 pieces the convolution engine does not cover
// (torchvision.models.mobilenet_v2 as used by atomai/nets/blocks.py:376-387, Regressor / Classifier):
//   * the 3x3 / pad-1 convolutions with stride 1 or 2: the dense stem (small Cin) and the depthwise
//     layers of the inverted-residual blocks.  Forward applies the producer's pending
//     relu6(scale*x + shift) on load (zero padding is that of the activated tensor) and writes the
//     raw output plus its BatchNorm sums; the depthwise data gradient is a gather; both weight
//     gradients sum per-CTA partials;
//   * BatchNorm -> ReLU6 backward: g = dy * [0 < scale*a + shift < 6] and the BatchNorm-backward
//     sums of g; the apply is atomai_b200_bn_lrelu_bwd with slope 1;
//   * relu6(scale*a + shift) written out, for the 1x1 tensor-core layers that read it;
//   * AdaptiveAvgPool2d(1) of relu6(scale*a + shift) and its backward;
//   * LogSoftmax(dim=1) and the mean NLL loss of the classifier head.
// Every cross-CTA sum (BatchNorm statistics and backward sums, weight gradients, the loss) goes
// through the ordered per-CTA slots of common.cuh: same input, same bits, no float atomics.
// Layout: NHWC fp32, one thread per (pixel, channel) with 32 consecutive channels per warp.
#include "common.cuh"

namespace {

constexpr int kT = 256;   // 8 warps: 8 pixel rows x 32 channel lanes
constexpr int kLanes = 32;
constexpr int kRows = kT / kLanes;

// CTAs along the pixel axis for a (pixels x channel groups) launch: a function of the shape and the
// SM count only, so the ordered sums are reproducible
inline int grid_rows(int64_t rows, int groups) {
  int64_t b = (rows + kRows - 1) / kRows;
  int64_t cap = (int64_t)ab_num_sms() * 8 / groups;
  if (cap < 1) cap = 1;
  if (b > cap) b = cap;
  return b < 1 ? 1 : (int)b;
}

__device__ __forceinline__ float load_act(const float* p, const float* scale, const float* shift,
                                          int clip, int c) {
  float v = __ldg(p);
  if (scale) v = fmaf(v, __ldg(scale + c), __ldg(shift + c));
  if (clip) v = fminf(fmaxf(v, 0.f), 6.f);
  return v;
}

// (v1, v2) of lane cx, row py -> ordered sums out[c0 + cx] and out[C + c0 + cx] of slot group
// `group` (one slot per CTA along x)
__device__ __forceinline__ void chan_reduce2(float v1, float v2, int c0, int C, double* out,
                                             const Ordered& red, int group) {
  __shared__ float s[2][kRows][kLanes];
  __shared__ unsigned s_last;
  const int tid = threadIdx.x, cx = tid % kLanes, py = tid / kLanes;
  s[0][py][cx] = v1;
  s[1][py][cx] = v2;
  __syncthreads();
  if (tid < 2 * kLanes) {
    const int k = tid / kLanes, l = tid % kLanes;
    float a = 0.f;
    for (int r = 0; r < kRows; ++r) a += s[k][r][l];
    ordered_slot(red, group, gridDim.x, blockIdx.x, 2 * kLanes)[tid] = a;
  }
  ordered_finish(red, group, gridDim.x, 2 * kLanes, tid, kT, gridDim.x, [] { __syncthreads(); },
                 [&](int i, double v) {
                   const int c = c0 + i % kLanes;
                   if (c < C) out[(i / kLanes) * C + c] += v;
                 },
                 &s_last);
}

struct Conv3Params {
  const float* x; int ld_x;
  const float* scale; const float* shift; int clip;
  const float* w; int depthwise;
  float* y; int ld_y;
  const float* dy; int ld_dy;
  float* dw;
  int N, H, W, Cin, Cout, stride, Ho, Wo;
  double* stats;
  Ordered red;
};

// y = conv3x3(act(x)), pad 1, stride s; dense (w: Cout x Cin x 3 x 3) or depthwise (Cout == Cin,
// w: C x 1 x 3 x 3)
__global__ void __launch_bounds__(kT) conv3_fwd_kernel(const Conv3Params p) {
  const int cx = threadIdx.x % kLanes, py = threadIdx.x / kLanes;
  const int co = blockIdx.y * kLanes + cx;
  const int64_t npix = (int64_t)p.N * p.Ho * p.Wo;
  float s1 = 0.f, s2 = 0.f;
  if (co < p.Cout) {
    for (int64_t q = (int64_t)blockIdx.x * kRows + py; q < npix; q += (int64_t)gridDim.x * kRows) {
      const int wo = (int)(q % p.Wo);
      const int64_t t = q / p.Wo;
      const int ho = (int)(t % p.Ho), n = (int)(t / p.Ho);
      float acc = 0.f;
      for (int kh = 0; kh < 3; ++kh) {
        const int hi = ho * p.stride - 1 + kh;
        if (hi < 0 || hi >= p.H) continue;
        for (int kw = 0; kw < 3; ++kw) {
          const int wi = wo * p.stride - 1 + kw;
          if (wi < 0 || wi >= p.W) continue;
          const float* xp = p.x + ((int64_t)(n * p.H + hi) * p.W + wi) * p.ld_x;
          if (p.depthwise) {
            acc = fmaf(__ldg(p.w + co * 9 + kh * 3 + kw), load_act(xp + co, p.scale, p.shift, p.clip, co),
                       acc);
          } else {
            for (int ci = 0; ci < p.Cin; ++ci)
              acc = fmaf(__ldg(p.w + ((int64_t)co * p.Cin + ci) * 9 + kh * 3 + kw),
                         load_act(xp + ci, p.scale, p.shift, p.clip, ci), acc);
          }
        }
      }
      p.y[q * p.ld_y + co] = acc;
      s1 += acc;
      s2 = fmaf(acc, acc, s2);
    }
  }
  if (p.stats) chan_reduce2(s1, s2, blockIdx.y * kLanes, p.Cout, p.stats, p.red, blockIdx.y);
}

// dw[co][ci][kh][kw] += sum over output pixels of dy * act(x); one input channel per blockIdx.z
// (dense) or the lane's own channel (depthwise)
__global__ void __launch_bounds__(kT) conv3_wgrad_kernel(const Conv3Params p) {
  const int cx = threadIdx.x % kLanes, py = threadIdx.x / kLanes;
  const int co = blockIdx.y * kLanes + cx;
  const int ci = p.depthwise ? co : (int)blockIdx.z;
  const int64_t npix = (int64_t)p.N * p.Ho * p.Wo;
  float acc[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) acc[k] = 0.f;
  if (co < p.Cout) {
    for (int64_t q = (int64_t)blockIdx.x * kRows + py; q < npix; q += (int64_t)gridDim.x * kRows) {
      const int wo = (int)(q % p.Wo);
      const int64_t t = q / p.Wo;
      const int ho = (int)(t % p.Ho), n = (int)(t / p.Ho);
      const float g = __ldg(p.dy + q * p.ld_dy + co);
#pragma unroll
      for (int kh = 0; kh < 3; ++kh) {
        const int hi = ho * p.stride - 1 + kh;
        if (hi < 0 || hi >= p.H) continue;
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
          const int wi = wo * p.stride - 1 + kw;
          if (wi < 0 || wi >= p.W) continue;
          const float* xp = p.x + ((int64_t)(n * p.H + hi) * p.W + wi) * p.ld_x + ci;
          acc[kh * 3 + kw] = fmaf(g, load_act(xp, p.scale, p.shift, p.clip, ci), acc[kh * 3 + kw]);
        }
      }
    }
  }
  __shared__ float s[9][kRows][kLanes];
  __shared__ unsigned s_last;
#pragma unroll
  for (int k = 0; k < 9; ++k) s[k][py][cx] = acc[k];
  __syncthreads();
  const int group = blockIdx.z * gridDim.y + blockIdx.y;
  const int tid = threadIdx.x;
  for (int i = tid; i < 9 * kLanes; i += kT) {
    const int k = i / kLanes, l = i % kLanes;
    float a = 0.f;
    for (int r = 0; r < kRows; ++r) a += s[k][r][l];
    ordered_slot(p.red, group, gridDim.x, blockIdx.x, 9 * kLanes)[i] = a;
  }
  const int c0 = blockIdx.y * kLanes;
  const int cin_w = p.depthwise ? 1 : p.Cin, ci_w = p.depthwise ? 0 : (int)blockIdx.z;
  ordered_finish(p.red, group, gridDim.x, 9 * kLanes, tid, kT, gridDim.x, [] { __syncthreads(); },
                 [&](int i, double v) {
                   const int c = c0 + i % kLanes;
                   if (c < p.Cout) p.dw[((int64_t)c * cin_w + ci_w) * 9 + i / kLanes] += (float)v;
                 },
                 &s_last);
}

// dx[n][hi][wi][c] = sum over the taps that read (hi, wi) of w[c][kh][kw] * dy[n][ho][wo][c]
__global__ void __launch_bounds__(kT) dw_dgrad_kernel(const Conv3Params p) {
  const int64_t total = (int64_t)p.N * p.H * p.W * p.Cout;
  for (int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x; i < total; i += (int64_t)gridDim.x * kT) {
    const int c = (int)(i % p.Cout);
    const int64_t pix = i / p.Cout;
    const int wi = (int)(pix % p.W);
    const int64_t t = pix / p.W;
    const int hi = (int)(t % p.H), n = (int)(t / p.H);
    float acc = 0.f;
    for (int kh = 0; kh < 3; ++kh) {
      const int th = hi + 1 - kh;
      if (th < 0 || th % p.stride) continue;
      const int ho = th / p.stride;
      if (ho >= p.Ho) continue;
      for (int kw = 0; kw < 3; ++kw) {
        const int tw = wi + 1 - kw;
        if (tw < 0 || tw % p.stride) continue;
        const int wo = tw / p.stride;
        if (wo >= p.Wo) continue;
        acc = fmaf(__ldg(p.w + c * 9 + kh * 3 + kw),
                   __ldg(p.dy + ((int64_t)(n * p.Ho + ho) * p.Wo + wo) * p.ld_dy + c), acc);
      }
    }
    p.y[pix * p.ld_y + c] = acc;
  }
}

// g = dy * [0 < scale*a + shift < 6]; sums += (sum g, sum g * (a - mean) * invstd) per channel.
// hw > 0: dy is the (N, C) gradient of the average pool over hw pixels per image, spread as dy / hw
// on the fly (AdaptiveAvgPool2d backward fused with the BatchNorm-backward reduction)
__global__ void __launch_bounds__(kT)
    relu6_bwd_reduce_kernel(const float* __restrict__ dy, int ld_dy, const float* __restrict__ a,
                            int ld_a, const float* scale, const float* shift, const float* mean,
                            const float* invstd, float* __restrict__ g, int ld_g, int64_t npix,
                            int C, int hw, double* sums, Ordered red) {
  const int cx = threadIdx.x % kLanes, py = threadIdx.x / kLanes;
  const int c = blockIdx.y * kLanes + cx;
  float s1 = 0.f, s2 = 0.f;
  if (c < C) {
    const float sc = scale[c], sh = shift[c], m = mean[c], is = invstd[c];
    const float inv_hw = hw > 0 ? 1.f / (float)hw : 1.f;
    for (int64_t q = (int64_t)blockIdx.x * kRows + py; q < npix; q += (int64_t)gridDim.x * kRows) {
      const float av = a[q * ld_a + c];
      const float y = fmaf(av, sc, sh);
      const float d = hw > 0 ? dy[(q / hw) * ld_dy + c] * inv_hw : dy[q * ld_dy + c];
      const float v = (y > 0.f && y < 6.f) ? d : 0.f;
      g[q * ld_g + c] = v;
      s1 += v;
      s2 = fmaf(v, (av - m) * is, s2);
    }
  }
  chan_reduce2(s1, s2, blockIdx.y * kLanes, C, sums, red, blockIdx.y);
}

__global__ void __launch_bounds__(kT)
    affine_relu6_kernel(const float* __restrict__ a, int ld_a, const float* scale, const float* shift,
                        float* __restrict__ y, int ld_y, int64_t npix, int C) {
  const int64_t total = npix * C;
  for (int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x; i < total; i += (int64_t)gridDim.x * kT) {
    const int c = (int)(i % C);
    const int64_t q = i / C;
    y[q * ld_y + c] = fminf(fmaxf(fmaf(a[q * ld_a + c], scale[c], shift[c]), 0.f), 6.f);
  }
}

// y[n][c] = mean over the HW pixels of image n of relu6(scale*a + shift), summed in pixel order
__global__ void __launch_bounds__(kT)
    avgpool_relu6_kernel(const float* __restrict__ a, int ld_a, const float* scale,
                         const float* shift, float* __restrict__ y, int N, int HW, int C) {
  const int64_t total = (int64_t)N * C;
  for (int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x; i < total; i += (int64_t)gridDim.x * kT) {
    const int c = (int)(i % C);
    const int64_t n = i / C;
    const float sc = scale ? scale[c] : 1.f, sh = scale ? shift[c] : 0.f;
    const float* ap = a + n * HW * ld_a + c;
    float s = 0.f;
    for (int r = 0; r < HW; ++r) s += fminf(fmaxf(fmaf(ap[(int64_t)r * ld_a], sc, sh), 0.f), 6.f);
    y[i] = s / (float)HW;
  }
}

__global__ void __launch_bounds__(kT)
    avgpool_bwd_kernel(const float* __restrict__ dy, float* __restrict__ g, int ld_g, int N, int HW,
                       int C) {
  const int64_t total = (int64_t)N * HW * C;
  const float inv = 1.f / (float)HW;
  for (int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x; i < total; i += (int64_t)gridDim.x * kT) {
    const int c = (int)(i % C);
    const int64_t q = i / C;
    g[q * ld_g + c] = dy[(q / HW) * C + c] * inv;
  }
}

// one warp per row of the (B, C) matrix
__global__ void __launch_bounds__(kT)
    log_softmax_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int C) {
  const int lane = threadIdx.x % 32;
  for (int64_t row = (blockIdx.x * (int64_t)kT + threadIdx.x) / 32; row < B;
       row += (int64_t)gridDim.x * kT / 32) {
    const float* xr = x + row * C;
    float m = -INFINITY;
    for (int c = lane; c < C; c += 32) m = fmaxf(m, xr[c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s += expf(xr[c] - m);
    s = warp_sum(s);
    const float lse = logf(s);
    for (int c = lane; c < C; c += 32) y[row * C + c] = xr[c] - m - lse;
  }
}

// dx = dy - exp(y) * sum(dy)
__global__ void __launch_bounds__(kT)
    log_softmax_bwd_kernel(const float* __restrict__ y, const float* __restrict__ dy,
                           float* __restrict__ dx, int B, int C) {
  const int lane = threadIdx.x % 32;
  for (int64_t row = (blockIdx.x * (int64_t)kT + threadIdx.x) / 32; row < B;
       row += (int64_t)gridDim.x * kT / 32) {
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s += dy[row * C + c];
    s = warp_sum(s);
    for (int c = lane; c < C; c += 32) dx[row * C + c] = dy[row * C + c] - expf(y[row * C + c]) * s;
  }
}

// loss = -mean_i logp[i][t_i] in one CTA (fixed summation order); a target outside [0, C) gives NaN
__global__ void __launch_bounds__(kT)
    nll_fwd_kernel(const float* __restrict__ logp, const int64_t* __restrict__ tgt, int B, int C,
                   float* loss) {
  __shared__ double s[kT];
  double a = 0.0;
  for (int i = threadIdx.x; i < B; i += kT) {
    const int64_t t = tgt[i];
    a += (t >= 0 && t < C) ? (double)logp[(int64_t)i * C + t] : (double)NAN;
  }
  s[threadIdx.x] = a;
  __syncthreads();
  for (int h = kT / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) s[threadIdx.x] += s[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) *loss = (float)(-s[0] / (double)B);
}

// dlogp[i][c] = -g / B at c == t_i, else 0 (g: upstream gradient read from device memory)
__global__ void __launch_bounds__(kT)
    nll_bwd_kernel(const int64_t* __restrict__ tgt, int B, int C, const float* gdev,
                   float* __restrict__ d) {
  const float v = -(gdev ? *gdev : 1.f) / (float)B;
  const int64_t total = (int64_t)B * C;
  for (int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x; i < total; i += (int64_t)gridDim.x * kT) {
    const int c = (int)(i % C);
    d[i] = tgt[i / C] == c ? v : 0.f;
  }
}

int conv3_setup(Conv3Params& p, const float* x, int ld_x, const float* scale, const float* shift,
                int clip, const float* w, int depthwise, int N, int H, int W, int Cin, int Cout,
                int stride, const char* who) {
  AB_CHECK(x && w && N >= 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0, "%s: bad arguments", who);
  AB_CHECK(stride == 1 || stride == 2, "%s: stride %d (1 or 2)", who, stride);
  AB_CHECK(!depthwise || Cin == Cout, "%s: depthwise needs Cin == Cout (%d, %d)", who, Cin, Cout);
  AB_CHECK(ld_x >= Cin, "%s: ld_x=%d < Cin=%d", who, ld_x, Cin);
  AB_CHECK((scale == nullptr) == (shift == nullptr), "%s: scale and shift go together", who);
  p = Conv3Params{};
  p.x = x; p.ld_x = ld_x; p.scale = scale; p.shift = shift; p.clip = clip ? 1 : 0;
  p.w = w; p.depthwise = depthwise ? 1 : 0;
  p.N = N; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout; p.stride = stride;
  p.Ho = (H - 1) / stride + 1;
  p.Wo = (W - 1) / stride + 1;
  return 0;
}

}  // namespace

extern "C" {

#define STREAM ((cudaStream_t)stream)

int atomai_b200_conv3x3_fwd(const float* x, int ld_x, const float* scale, const float* shift,
                            int clip, const float* w, int depthwise, float* y, int ld_y, int N,
                            int H, int W, int Cin, int Cout, int stride, double* stats,
                            void* stream) {
  Conv3Params p;
  if (conv3_setup(p, x, ld_x, scale, shift, clip, w, depthwise, N, H, W, Cin, Cout, stride,
                  "conv3x3_fwd"))
    return 1;
  AB_CHECK(y && ld_y >= Cout, "conv3x3_fwd: bad output (ld_y=%d, Cout=%d)", ld_y, Cout);
  p.y = y; p.ld_y = ld_y; p.stats = stats;
  const int64_t npix = (int64_t)N * p.Ho * p.Wo;
  if (npix == 0) return 0;
  const int gy = (Cout + kLanes - 1) / kLanes, gx = grid_rows(npix, gy);
  if (stats && ab_ordered_ws(STREAM, (int64_t)gx * gy * 2 * kLanes, gy, &p.red)) return 1;
  conv3_fwd_kernel<<<dim3(gx, gy), kT, 0, STREAM>>>(p);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_conv3x3_wgrad(const float* dy, int ld_dy, const float* x, int ld_x,
                              const float* scale, const float* shift, int clip, int depthwise,
                              float* dw, int N, int H, int W, int Cin, int Cout, int stride,
                              void* stream) {
  Conv3Params p;
  if (conv3_setup(p, x, ld_x, scale, shift, clip, dw, depthwise, N, H, W, Cin, Cout, stride,
                  "conv3x3_wgrad"))
    return 1;
  AB_CHECK(dy && ld_dy >= Cout, "conv3x3_wgrad: bad dy (ld_dy=%d, Cout=%d)", ld_dy, Cout);
  p.dy = dy; p.ld_dy = ld_dy; p.dw = dw;
  const int64_t npix = (int64_t)N * p.Ho * p.Wo;
  if (npix == 0) return 0;
  const int gy = (Cout + kLanes - 1) / kLanes, gz = depthwise ? 1 : Cin;
  AB_CHECK(gz <= 65535, "conv3x3_wgrad: Cin=%d", Cin);
  const int gx = grid_rows(npix, gy * gz);
  if (ab_ordered_ws(STREAM, (int64_t)gx * gy * gz * 9 * kLanes, gy * gz, &p.red)) return 1;
  conv3_wgrad_kernel<<<dim3(gx, gy, gz), kT, 0, STREAM>>>(p);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_dw3x3_dgrad(const float* dy, int ld_dy, const float* w, float* dx, int ld_dx,
                            int N, int H, int W, int C, int stride, void* stream) {
  Conv3Params p;
  if (conv3_setup(p, dy, ld_dy, nullptr, nullptr, 0, w, 1, N, H, W, C, C, stride, "dw3x3_dgrad"))
    return 1;
  AB_CHECK(dx && ld_dx >= C, "dw3x3_dgrad: bad dx (ld_dx=%d, C=%d)", ld_dx, C);
  p.dy = dy; p.ld_dy = ld_dy; p.y = dx; p.ld_y = ld_dx;
  const int64_t total = (int64_t)N * H * W * C;
  if (total == 0) return 0;
  dw_dgrad_kernel<<<ab_grid(total, kT, 16), kT, 0, STREAM>>>(p);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_relu6_bwd_reduce(const float* dy, int ld_dy, const float* a, int ld_a,
                                 const float* scale, const float* shift, const float* mean,
                                 const float* invstd, float* g, int ld_g, int64_t npix, int C,
                                 int hw, double* sums, void* stream) {
  AB_CHECK(dy && a && scale && shift && mean && invstd && g && sums && C > 0 && npix >= 0,
           "relu6_bwd_reduce: bad arguments");
  AB_CHECK(hw >= 0 && (hw == 0 || npix % hw == 0), "relu6_bwd_reduce: hw=%d does not divide npix", hw);
  if (npix == 0) return 0;
  const int gy = (C + kLanes - 1) / kLanes, gx = grid_rows(npix, gy);
  Ordered red;
  if (ab_ordered_ws(STREAM, (int64_t)gx * gy * 2 * kLanes, gy, &red)) return 1;
  relu6_bwd_reduce_kernel<<<dim3(gx, gy), kT, 0, STREAM>>>(dy, ld_dy, a, ld_a, scale, shift, mean,
                                                          invstd, g, ld_g, npix, C, hw, sums, red);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_affine_relu6(const float* a, int ld_a, const float* scale, const float* shift,
                             float* y, int ld_y, int64_t npix, int C, void* stream) {
  AB_CHECK(a && scale && shift && y && C > 0 && npix >= 0, "affine_relu6: bad arguments");
  if (npix == 0) return 0;
  affine_relu6_kernel<<<ab_grid(npix * C, kT, 16), kT, 0, STREAM>>>(a, ld_a, scale, shift, y, ld_y, npix, C);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_avgpool_relu6_fwd(const float* a, int ld_a, const float* scale, const float* shift,
                                  float* y, int N, int HW, int C, void* stream) {
  AB_CHECK(a && y && N >= 0 && HW > 0 && C > 0, "avgpool_relu6_fwd: bad arguments");
  AB_CHECK((scale == nullptr) == (shift == nullptr), "avgpool_relu6_fwd: scale and shift go together");
  if (N == 0) return 0;
  avgpool_relu6_kernel<<<ab_grid((int64_t)N * C, kT, 16), kT, 0, STREAM>>>(a, ld_a, scale, shift, y, N, HW, C);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_avgpool_bwd(const float* dy, float* g, int ld_g, int N, int HW, int C,
                            void* stream) {
  AB_CHECK(dy && g && N >= 0 && HW > 0 && C > 0 && ld_g >= C, "avgpool_bwd: bad arguments");
  if (N == 0) return 0;
  avgpool_bwd_kernel<<<ab_grid((int64_t)N * HW * C, kT, 16), kT, 0, STREAM>>>(dy, g, ld_g, N, HW, C);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_log_softmax_fwd(const float* x, float* y, int B, int C, void* stream) {
  AB_CHECK(x && y && B >= 0 && C > 0, "log_softmax_fwd: bad arguments");
  if (B == 0) return 0;
  log_softmax_fwd_kernel<<<ab_grid((int64_t)B * 32, kT, 16), kT, 0, STREAM>>>(x, y, B, C);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_log_softmax_bwd(const float* y, const float* dy, float* dx, int B, int C,
                                void* stream) {
  AB_CHECK(y && dy && dx && B >= 0 && C > 0, "log_softmax_bwd: bad arguments");
  if (B == 0) return 0;
  log_softmax_bwd_kernel<<<ab_grid((int64_t)B * 32, kT, 16), kT, 0, STREAM>>>(y, dy, dx, B, C);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_nll_fwd_bwd(const float* logp, const int64_t* target, int B, int C, float* loss,
                            float* dlogp, const float* gscale_dev, void* stream) {
  AB_CHECK(target && B > 0 && C > 0 && (loss || dlogp), "nll_fwd_bwd: bad arguments");
  if (loss) {
    AB_CHECK(logp, "nll_fwd_bwd: the loss needs logp");
    nll_fwd_kernel<<<1, kT, 0, STREAM>>>(logp, target, B, C, loss);
    AB_LAUNCH_CHECK();
  }
  if (dlogp) {
    nll_bwd_kernel<<<ab_grid((int64_t)B * C, kT, 16), kT, 0, STREAM>>>(target, B, C, gscale_dev, dlogp);
    AB_LAUNCH_CHECK();
  }
  return 0;
}

}  // extern "C"
