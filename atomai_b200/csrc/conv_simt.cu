// conv_simt.cu — exact-fp32 (FFMA) convolution family: forward/dgrad and weight-gradient for ANY
// channel count (Cin = 1 first layer, Cout = nb_classes head, 1-D signals as H = 1), reading its
// input through the same normalise-on-load source loader as the tensor-core path.  This is the
// AB_MATH_FP32 math mode: bit-for-bit it is still not the CPU reference (different summation
// order) but it carries no TF32 rounding, so it is the mode the 1e-3 logit parity bound is pinned
// with.  It also serves every layer shape the tensor-core kernels do not take (C % 8 != 0, Cout % 16).
//
// Replaces nn.Conv2d/nn.Conv1d (+bias, LeakyReLU, BN statistics) of atomai/nets/blocks.py:61-76,
// :302-319, :130-132 and autograd's bwd-filter for atomai/trainers/trainer.py:206.
#include "common.cuh"

namespace {

// ------------------------------------------------------------------ forward
// CTA: 256 threads, output tile 8 rows x 32 cols (or 1 x 256 for 1-D), COT = 16 couts per pass.
// thread -> 4 consecutive-w pixels x 4 couts... laid out as: pg = tid % 64 (8 rows x 8 groups of
// 4 px), cg = tid / 64 (4 groups of 4 couts).
constexpr int F_TH = 8, F_TW = 32, F_COT = 16, F_CIT = 8, F_THREADS = 256;

struct ConvSimtParams {
  SrcSet S;
  int N, H, W, Cout;
  int th, tw, dil;
  const float* w;  // [tap][Cin][Cout]
  const float* bias;
  float alpha;
  int act;
  float* out;
  int ld_out;
  int out_nchw;
  double* stats;
  int tiles_h, tiles_w;
  int c0;          // thin-channel kernels: first output channel of this launch's channel block
  Ordered red;     // quad-lane / tile kernels: ordered sum of the per-warp statistics
};

__global__ void __launch_bounds__(F_THREADS) conv_simt_fwd_kernel(const ConvSimtParams p) {
  extern __shared__ float sm[];
  const int taps = p.th * p.tw;
  const int ph = p.dil * (p.th >> 1), pw = p.dil * (p.tw >> 1);
  const int THp = F_TH + 2 * ph, TWp = F_TW + 2 * pw;
  float* s_in = sm;                             // [F_CIT][THp][TWp]
  float* s_w = sm + F_CIT * THp * TWp;          // [taps][F_CIT][F_COT]
  __shared__ float s_red[2 * F_COT];

  const int tile = blockIdx.x;
  const int tw_i = tile % p.tiles_w;
  const int th_i = (tile / p.tiles_w) % p.tiles_h;
  const int n = tile / (p.tiles_w * p.tiles_h);
  const int h0 = th_i * F_TH, w0 = tw_i * F_TW;
  const int co0 = blockIdx.y * F_COT;

  const int tid = threadIdx.x;
  const int pg = tid & 63, cg = tid >> 6;
  const int r = pg >> 3, wq = (pg & 7) * 4;  // row in tile, first of 4 pixels
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int k = 0; k < 4; ++k) acc[i][k] = 0.f;

  const int Cin = p.S.Ctot;
  for (int ci0 = 0; ci0 < Cin; ci0 += F_CIT) {
    __syncthreads();
    for (int i = tid; i < F_CIT * THp * TWp; i += F_THREADS) {
      const int ww = i % TWp, hh = (i / TWp) % THp, c = i / (TWp * THp);
      float v = 0.f;
      if (ci0 + c < Cin) v = load_src1(p.S, n, h0 - ph + hh, w0 - pw + ww, p.H, p.W, ci0 + c);
      s_in[i] = v;
    }
    for (int i = tid; i < taps * F_CIT * F_COT; i += F_THREADS) {
      const int co = i % F_COT, c = (i / F_COT) % F_CIT, t = i / (F_COT * F_CIT);
      float v = 0.f;
      if (ci0 + c < Cin && co0 + co < p.Cout)
        v = __ldg(p.w + ((size_t)t * Cin + ci0 + c) * p.Cout + co0 + co);
      s_w[i] = v;
    }
    __syncthreads();
    const int cmax = min(F_CIT, Cin - ci0);
    for (int c = 0; c < cmax; ++c) {
      for (int t = 0; t < taps; ++t) {
        const int ty = t / p.tw, tx = t - ty * p.tw;
        const float* ip = s_in + (c * THp + r + ty * p.dil) * TWp + wq + tx * p.dil;
        const float4 wv = *reinterpret_cast<const float4*>(s_w + (t * F_CIT + c) * F_COT + cg * 4);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float x = ip[i];
          acc[i][0] = fmaf(x, wv.x, acc[i][0]);
          acc[i][1] = fmaf(x, wv.y, acc[i][1]);
          acc[i][2] = fmaf(x, wv.z, acc[i][2]);
          acc[i][3] = fmaf(x, wv.w, acc[i][3]);
        }
      }
    }
  }

  // epilogue
  float ssum[4] = {0, 0, 0, 0}, ssq[4] = {0, 0, 0, 0};
  const int gh = h0 + r;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int gw = w0 + wq + i;
    const bool valid = gh < p.H && gw < p.W;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int co = co0 + cg * 4 + k;
      if (co < p.Cout) {
        float v = acc[i][k] + (p.bias ? __ldg(p.bias + co) : 0.f);
        v = act_f(v, p.act, p.alpha);
        if (valid) {
          if (!p.out_nchw)
            p.out[(((size_t)n * p.H + gh) * p.W + gw) * p.ld_out + co] = v;
          else
            p.out[(((size_t)n * p.Cout + co) * p.H + gh) * p.W + gw] = v;
          ssum[k] += v;
          ssq[k] += v * v;
        }
      }
    }
  }
  if (p.stats) {
    if (tid < 2 * F_COT) s_red[tid] = 0.f;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float a = warp_sum(ssum[k]), b = warp_sum(ssq[k]);
      if ((tid & 31) == 0) {
        atomicAdd(&s_red[cg * 4 + k], a);
        atomicAdd(&s_red[F_COT + cg * 4 + k], b);
      }
    }
    __syncthreads();
    if (tid < F_COT && co0 + tid < p.Cout) {
      atomicAdd(p.stats + co0 + tid, (double)s_red[tid]);
      atomicAdd(p.stats + p.Cout + co0 + tid, (double)s_red[F_COT + tid]);
    }
  }
}


// ------------------------------------------------------------------ thin-channel specialisations
// The first layer (Cin = 1, 3x3) and the pixel-wise head / its data-gradient (1x1 with <= 4 or
// from <= 4 channels) are pure HBM streams: one thread per pixel, all output channels in
// registers, weights broadcast from shared memory, float4 stores.
template <int CO>
__global__ void __launch_bounds__(256) conv_pix_kernel(const ConvSimtParams p, int vec_in) {
  extern __shared__ float s_w[];                 // [taps][Cin][CO] (zero padded to CO)
  __shared__ float s_red[2 * CO];
  const int taps = p.th * p.tw, Cin = p.S.Ctot;
  const int c0 = p.c0, nco = min(CO, p.Cout - c0);     // this launch's channel block
  for (int i = threadIdx.x; i < taps * Cin * CO; i += blockDim.x) {
    const int co = i % CO, r = i / CO;
    s_w[i] = co < nco ? __ldg(p.w + (size_t)r * p.Cout + c0 + co) : 0.f;
  }
  if (threadIdx.x < 2 * CO) s_red[threadIdx.x] = 0.f;
  __syncthreads();
  float bias[CO];
#pragma unroll
  for (int k = 0; k < CO; ++k) bias[k] = (p.bias && k < nco) ? __ldg(p.bias + c0 + k) : 0.f;
  float ssum[CO], ssq[CO];
#pragma unroll
  for (int k = 0; k < CO; ++k) { ssum[k] = 0.f; ssq[k] = 0.f; }
  const int64_t npix = (int64_t)p.N * p.H * p.W;
  // 1x1 kernel on one plain source (the pixel-wise head and its data gradient): no halo, so the
  // pending BatchNorm affine folds into the staged weights — w'[c][k] = w[c][k]*scale[c],
  // b'[k] = b[k] + sum_c w[c][k]*shift[c] — and the loop is pointer + loads + FMAs (the generic
  // loader below re-derives source, bounds and affine for every 4 channels)
  const bool direct = taps == 1 && p.S.nsrc == 1 && p.S.s[0].pool == 0;
  if (direct) {
    const SrcDev sd = p.S.s[0];
    if (sd.scale) {
#pragma unroll
      for (int k = 0; k < CO; ++k) {
        float t = 0.f;
        for (int c = 0; c < Cin; ++c) t = fmaf(s_w[c * CO + k], __ldg(sd.shift + c), t);
        bias[k] += t;
      }
      __syncthreads();
      for (int i = threadIdx.x; i < Cin * CO; i += blockDim.x) s_w[i] *= __ldg(sd.scale + i / CO);
      __syncthreads();
    }
    for (int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < npix;
         pix += (int64_t)gridDim.x * blockDim.x) {
      const float* xp = sd.ptr + pix * sd.ld;
      float acc[CO];
#pragma unroll
      for (int k = 0; k < CO; ++k) acc[k] = bias[k];
      if (vec_in) {
        for (int c = 0; c < Cin; c += 4) {
          const float4 x = __ldg(reinterpret_cast<const float4*>(xp + c));
          const float* wt = s_w + c * CO;
#pragma unroll
          for (int k = 0; k < CO; ++k)
            acc[k] = fmaf(x.x, wt[k], fmaf(x.y, wt[CO + k], fmaf(x.z, wt[2 * CO + k], fmaf(x.w, wt[3 * CO + k], acc[k]))));
        }
      } else {
        for (int c = 0; c < Cin; ++c) {
          const float x = __ldg(xp + c);
#pragma unroll
          for (int k = 0; k < CO; ++k) acc[k] = fmaf(x, s_w[c * CO + k], acc[k]);
        }
      }
#pragma unroll
      for (int k = 0; k < CO; ++k) {
        acc[k] = act_f(acc[k], p.act, p.alpha);
        ssum[k] += acc[k];
        ssq[k] = fmaf(acc[k], acc[k], ssq[k]);
      }
      if (!p.out_nchw) {
        float* o = p.out + pix * p.ld_out + c0;
        if (CO % 4 == 0 && nco == CO && (p.ld_out & 3) == 0 && (c0 & 3) == 0) {
#pragma unroll
          for (int k = 0; k < CO; k += 4)
            *reinterpret_cast<float4*>(o + k) = make_float4(acc[k], acc[k + 1], acc[k + 2], acc[k + 3]);
        } else {
#pragma unroll
          for (int k = 0; k < CO; ++k)
            if (k < nco) o[k] = acc[k];
        }
      } else {
        const size_t hw = (size_t)p.H * p.W;
        const int64_t n = pix / (int64_t)hw, r = pix - n * (int64_t)hw;
#pragma unroll
        for (int k = 0; k < CO; ++k)
          if (k < nco) p.out[((size_t)n * p.Cout + c0 + k) * hw + (size_t)r] = acc[k];
      }
    }
  }
  const int ph = p.dil * (p.th >> 1), pw = p.dil * (p.tw >> 1);
  const uint32_t uW = p.W, uHW = (uint32_t)p.H * p.W;      // npix < 2^32 (checked by the launcher)
  for (int64_t pix = direct ? npix : (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < npix;
       pix += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t up = (uint32_t)pix;                     // 32-bit divisions: ~20 instrs, not ~150
    const int n = (int)(up / uHW);
    const uint32_t rem = up - (uint32_t)n * uHW;
    const int h = (int)(rem / uW);
    const int w = (int)(rem - (uint32_t)h * uW);
    float acc[CO];
#pragma unroll
    for (int k = 0; k < CO; ++k) acc[k] = bias[k];
    for (int t = 0; t < taps; ++t) {
      const int ty = t / p.tw, tx = t - ty * p.tw;
      const int hh = h - ph + ty * p.dil, ww = w - pw + tx * p.dil;
      const float* wt = s_w + (size_t)t * Cin * CO;
      if (vec_in) {
        for (int c = 0; c < Cin; c += 4) {
          const float4 x = load_src4(p.S, n, hh, ww, p.H, p.W, c);
#pragma unroll
          for (int k = 0; k < CO; ++k)
            acc[k] = fmaf(x.x, wt[c * CO + k], fmaf(x.y, wt[(c + 1) * CO + k],
                     fmaf(x.z, wt[(c + 2) * CO + k], fmaf(x.w, wt[(c + 3) * CO + k], acc[k]))));
        }
      } else {
        for (int c = 0; c < Cin; ++c) {
          const float x = load_src1(p.S, n, hh, ww, p.H, p.W, c);
#pragma unroll
          for (int k = 0; k < CO; ++k) acc[k] = fmaf(x, wt[c * CO + k], acc[k]);
        }
      }
    }
#pragma unroll
    for (int k = 0; k < CO; ++k) {
      acc[k] = act_f(acc[k], p.act, p.alpha);
      ssum[k] += acc[k];
      ssq[k] = fmaf(acc[k], acc[k], ssq[k]);
    }
    if (!p.out_nchw) {
      float* o = p.out + pix * p.ld_out + c0;
      if (CO % 4 == 0 && nco == CO && (p.ld_out & 3) == 0 && (c0 & 3) == 0) {
#pragma unroll
        for (int k = 0; k < CO; k += 4)
          *reinterpret_cast<float4*>(o + k) = make_float4(acc[k], acc[k + 1], acc[k + 2], acc[k + 3]);
      } else {
#pragma unroll
        for (int k = 0; k < CO; ++k)
          if (k < nco) o[k] = acc[k];
      }
    } else {
      const size_t hw = (size_t)p.H * p.W;
#pragma unroll
      for (int k = 0; k < CO; ++k)
        if (k < nco) p.out[((size_t)n * p.Cout + c0 + k) * hw + (size_t)h * p.W + w] = acc[k];
    }
  }
  if (p.stats) {
#pragma unroll
    for (int k = 0; k < CO; ++k) {
      const float a = warp_sum(ssum[k]), b = warp_sum(ssq[k]);
      if ((threadIdx.x & 31) == 0) {
        atomicAdd(&s_red[k], a);
        atomicAdd(&s_red[CO + k], b);
      }
    }
    __syncthreads();
    if (threadIdx.x < CO && threadIdx.x < nco) {
      atomicAdd(p.stats + c0 + threadIdx.x, (double)s_red[threadIdx.x]);
      atomicAdd(p.stats + p.Cout + c0 + threadIdx.x, (double)s_red[CO + threadIdx.x]);
    }
  }
}

// First layer (Cin = 1, 3x3, one un-pooled source): an HBM stream that writes 16x more than it
// reads.  Each thread owns two horizontally adjacent output pixels: 3 x 4 input samples from
// L1, the 9 x CO weights as float4 broadcasts from shared memory (shared by both pixels), CO x 2
// accumulators in registers, 2 x CO/4 float4 stores; BN statistics ride along in registers.
template <int CO>
__global__ void __launch_bounds__(256, 2) conv_c1_kernel(const ConvSimtParams p) {
  __shared__ float4 s_w[9 * CO / 4];            // [tap][co]
  __shared__ float4 s_b[CO / 4];
  __shared__ float s_red[2 * CO];
  const int c0 = p.c0;                                           // channel block of this launch
  for (int i = threadIdx.x; i < 9 * CO; i += blockDim.x)         // packed [tap][Cin = 1][Cout]
    reinterpret_cast<float*>(s_w)[i] = __ldg(p.w + (size_t)(i / CO) * p.Cout + c0 + (i % CO));
  if (threadIdx.x < CO)
    reinterpret_cast<float*>(s_b)[threadIdx.x] = p.bias ? __ldg(p.bias + c0 + threadIdx.x) : 0.f;
  if (threadIdx.x < 2 * CO) s_red[threadIdx.x] = 0.f;
  __syncthreads();
  const SrcDev sd = p.S.s[0];
  float sc = 1.f, sh = 0.f;
  if (sd.scale) { sc = __ldg(sd.scale); sh = __ldg(sd.shift); }
  float ssum[CO], ssq[CO];
#pragma unroll
  for (int k = 0; k < CO; ++k) { ssum[k] = 0.f; ssq[k] = 0.f; }
  const int H = p.H, W = p.W, d = p.dil;
  const uint32_t Wh = (uint32_t)(W + 1) >> 1, per_img = Wh * (uint32_t)H;
  const uint32_t total = per_img * (uint32_t)p.N;
  const bool fast = p.act == AB_ACT_LRELU && p.alpha >= 0.f && p.alpha <= 1.f;
  const uint32_t stride = gridDim.x * blockDim.x;
  // input patch of a pixel pair (w, w+1): rows h-d, h, h+d x columns {w-d, w, w+d} (+1 for the
  // second pixel), zero padded; fetched one iteration ahead so the loads overlap the FMAs
  auto fetch = [&](uint32_t idx, float (&x0)[9], float (&x1)[9], uint32_t& n, int& h, int& w) {
    n = idx / per_img;
    const uint32_t rem = idx - n * per_img;
    h = (int)(rem / Wh);
    w = (int)(rem - (uint32_t)h * Wh) * 2;
#pragma unroll
    for (int ty = 0; ty < 3; ++ty) {
      const int hh = h + (ty - 1) * d;
      const bool rok = (unsigned)hh < (unsigned)H;
      const float* rowp = sd.ptr + ((size_t)n * H + (rok ? hh : 0)) * W * sd.ld;
#pragma unroll
      for (int tx = 0; tx < 3; ++tx) {
        const int w0 = w + (tx - 1) * d, w1 = w0 + 1;
        const bool ok0 = rok && (unsigned)w0 < (unsigned)W, ok1 = rok && (unsigned)w1 < (unsigned)W;
        x0[ty * 3 + tx] = ok0 ? fmaf(__ldg(rowp + (size_t)w0 * sd.ld), sc, sh) : 0.f;
        x1[ty * 3 + tx] = ok1 ? fmaf(__ldg(rowp + (size_t)w1 * sd.ld), sc, sh) : 0.f;
      }
    }
  };
  uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
  float nx0[9], nx1[9];
  uint32_t nn = 0; int nh = 0, nw = 0;
  if (idx < total) fetch(idx, nx0, nx1, nn, nh, nw);
  for (; idx < total; idx += stride) {
    float x0[9], x1[9];
#pragma unroll
    for (int t = 0; t < 9; ++t) { x0[t] = nx0[t]; x1[t] = nx1[t]; }
    const uint32_t n = nn; const int h = nh, w = nw;
    if (idx + stride < total) fetch(idx + stride, nx0, nx1, nn, nh, nw);
    float a0[CO], a1[CO];
#pragma unroll
    for (int k4 = 0; k4 < CO / 4; ++k4) {
      const float4 bv = s_b[k4];
      a0[k4 * 4] = bv.x; a0[k4 * 4 + 1] = bv.y; a0[k4 * 4 + 2] = bv.z; a0[k4 * 4 + 3] = bv.w;
      a1[k4 * 4] = bv.x; a1[k4 * 4 + 1] = bv.y; a1[k4 * 4 + 2] = bv.z; a1[k4 * 4 + 3] = bv.w;
    }
#pragma unroll
    for (int t = 0; t < 9; ++t) {
#pragma unroll
      for (int k4 = 0; k4 < CO / 4; ++k4) {
        const float4 wv = s_w[t * (CO / 4) + k4];
        a0[k4 * 4 + 0] = fmaf(x0[t], wv.x, a0[k4 * 4 + 0]); a1[k4 * 4 + 0] = fmaf(x1[t], wv.x, a1[k4 * 4 + 0]);
        a0[k4 * 4 + 1] = fmaf(x0[t], wv.y, a0[k4 * 4 + 1]); a1[k4 * 4 + 1] = fmaf(x1[t], wv.y, a1[k4 * 4 + 1]);
        a0[k4 * 4 + 2] = fmaf(x0[t], wv.z, a0[k4 * 4 + 2]); a1[k4 * 4 + 2] = fmaf(x1[t], wv.z, a1[k4 * 4 + 2]);
        a0[k4 * 4 + 3] = fmaf(x0[t], wv.w, a0[k4 * 4 + 3]); a1[k4 * 4 + 3] = fmaf(x1[t], wv.w, a1[k4 * 4 + 3]);
      }
    }
    const bool two = w + 1 < W;
#pragma unroll
    for (int k = 0; k < CO; ++k) {
      a0[k] = fast ? fmaxf(a0[k], a0[k] * p.alpha) : act_f(a0[k], p.act, p.alpha);
      a1[k] = fast ? fmaxf(a1[k], a1[k] * p.alpha) : act_f(a1[k], p.act, p.alpha);
      if (!two) a1[k] = 0.f;
      ssum[k] += a0[k] + a1[k];
      ssq[k] = fmaf(a0[k], a0[k], fmaf(a1[k], a1[k], ssq[k]));
    }
    float* o = p.out + (((size_t)n * H + h) * W + w) * p.ld_out + c0;
#pragma unroll
    for (int k = 0; k < CO; k += 4) {
      *reinterpret_cast<float4*>(o + k) = make_float4(a0[k], a0[k + 1], a0[k + 2], a0[k + 3]);
      if (two)
        *reinterpret_cast<float4*>(o + p.ld_out + k) = make_float4(a1[k], a1[k + 1], a1[k + 2], a1[k + 3]);
    }
  }
  if (p.stats) {
#pragma unroll
    for (int k = 0; k < CO; ++k) {
      const float a = warp_sum(ssum[k]), b = warp_sum(ssq[k]);
      if ((threadIdx.x & 31) == 0) {
        atomicAdd(&s_red[k], a);
        atomicAdd(&s_red[CO + k], b);
      }
    }
    __syncthreads();
    if (threadIdx.x < CO) {
      atomicAdd(p.stats + c0 + threadIdx.x, (double)s_red[threadIdx.x]);
      atomicAdd(p.stats + p.Cout + c0 + threadIdx.x, (double)s_red[CO + threadIdx.x]);
    }
  }
}

// First layer, tile version (dilation 1): a CTA of 8 warps owns a 64 x 16 output tile whose
// 66 x 18 input halo tile (affine applied, zero padded) sits in shared memory; the NEXT tile's
// halo is fetched into registers before the current one is computed.  Lane l of a warp = pixel
// l >> 2 of an 8-pixel run x channel quad l & 3, so every STG.128 of a warp writes 8 whole pixels
// = 512 contiguous bytes (the pair-per-thread kernel above writes 16-byte pieces 128 bytes
// apart), the thread's 9 x 4 weights live in registers for the
// whole kernel, and walking down the 16 rows costs 3 broadcast LDS per 36 FFMA.  Accumulation
// order per output (bias, then taps 0..8 with fmaf) is the pair kernel's: results are identical.
constexpr int C1T_W = 64, C1T_H = 16, C1T_PW = C1T_W + 2, C1T_PH = C1T_H + 2;
constexpr int C1T_ELEMS = C1T_PW * C1T_PH, C1T_PER_THREAD = (C1T_ELEMS + 255) / 256;

struct C1Tile { int n, h0, w0; };
__device__ __forceinline__ C1Tile c1_tile(int tile, int tiles_w, int tiles_hw) {
  C1Tile t;
  t.n = tile / tiles_hw;
  const int rem = tile - t.n * tiles_hw;
  const int th = rem / tiles_w;
  t.h0 = th * C1T_H;
  t.w0 = (rem - th * tiles_w) * C1T_W;
  return t;
}
// halo tile of `t` -> registers (element e = tid + i*256 of the 66 x 18 tile)
__device__ __forceinline__ void c1_fetch(const SrcDev& sd, float sc, float sh, int H, int W,
                                         const C1Tile& t, float (&r)[C1T_PER_THREAD]) {
#pragma unroll
  for (int i = 0; i < C1T_PER_THREAD; ++i) {
    const int e = threadIdx.x + i * 256;
    const int row = e / C1T_PW, col = e - row * C1T_PW;
    const int gh = t.h0 - 1 + row, gw = t.w0 - 1 + col;
    const bool ok = e < C1T_ELEMS && (unsigned)gh < (unsigned)H && (unsigned)gw < (unsigned)W;
    r[i] = ok ? fmaf(__ldg(sd.ptr + (((size_t)t.n * H + gh) * W + gw) * sd.ld), sc, sh) : 0.f;
  }
}
__device__ __forceinline__ void c1_stage(float* s_x, const float (&r)[C1T_PER_THREAD]) {
#pragma unroll
  for (int i = 0; i < C1T_PER_THREAD; ++i) {
    const int e = threadIdx.x + i * 256;
    if (e < C1T_ELEMS) s_x[e] = r[i];
  }
}

template <int FAST>
__global__ void __launch_bounds__(256) conv_c1_tile_kernel(const ConvSimtParams p, int tiles_w,
                                                           int tiles_hw, int num_tiles) {
  __shared__ float s_x[C1T_ELEMS];
  __shared__ unsigned s_last;
  const int c0 = p.c0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int px = lane >> 2, q = lane & 3;
  const int col = warp * 8 + px;                                   // column inside the tile
  float wr[9][4], bq[4];
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int k = 0; k < 4; ++k) wr[t][k] = __ldg(p.w + (size_t)t * p.Cout + c0 + q * 4 + k);
#pragma unroll
  for (int k = 0; k < 4; ++k) bq[k] = p.bias ? __ldg(p.bias + c0 + q * 4 + k) : 0.f;
  const SrcDev sd = p.S.s[0];
  float sc = 1.f, sh = 0.f;
  if (sd.scale) { sc = __ldg(sd.scale); sh = __ldg(sd.shift); }
  const int H = p.H, W = p.W;
  float ssum[4] = {0.f, 0.f, 0.f, 0.f}, ssq[4] = {0.f, 0.f, 0.f, 0.f};
  float nxt[C1T_PER_THREAD];
  int tile = blockIdx.x;
  C1Tile cur = c1_tile(tile < num_tiles ? tile : 0, tiles_w, tiles_hw);
  if (tile < num_tiles) c1_fetch(sd, sc, sh, H, W, cur, nxt);
  for (; tile < num_tiles; tile += gridDim.x) {
    __syncthreads();                     // every warp is done with the previous tile's halo
    c1_stage(s_x, nxt);
    __syncthreads();
    const C1Tile me = cur;
    const int tn = tile + gridDim.x;
    if (tn < num_tiles) {
      cur = c1_tile(tn, tiles_w, tiles_hw);
      c1_fetch(sd, sc, sh, H, W, cur, nxt);
    }
    const int gw = me.w0 + col;
    if (gw < W) {
      const float* sp = s_x + col;
      float x0[3], x1[3], x2[3];
#pragma unroll
      for (int j = 0; j < 3; ++j) { x0[j] = sp[j]; x1[j] = sp[C1T_PW + j]; }
      float* o = p.out + (((size_t)me.n * H + me.h0) * W + gw) * p.ld_out + c0 + q * 4;
      const size_t row_stride = (size_t)W * p.ld_out;
      const int rows = min(C1T_H, H - me.h0);
#pragma unroll 4
      for (int r = 0; r < rows; ++r) {
#pragma unroll
        for (int j = 0; j < 3; ++j) x2[j] = sp[(r + 2) * C1T_PW + j];
        float a[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          float v = bq[k];
          v = fmaf(x0[0], wr[0][k], v); v = fmaf(x0[1], wr[1][k], v); v = fmaf(x0[2], wr[2][k], v);
          v = fmaf(x1[0], wr[3][k], v); v = fmaf(x1[1], wr[4][k], v); v = fmaf(x1[2], wr[5][k], v);
          v = fmaf(x2[0], wr[6][k], v); v = fmaf(x2[1], wr[7][k], v); v = fmaf(x2[2], wr[8][k], v);
          v = FAST ? fmaxf(v, v * p.alpha) : act_f(v, p.act, p.alpha);
          ssum[k] += v;
          ssq[k] = fmaf(v, v, ssq[k]);
          a[k] = v;
        }
        *reinterpret_cast<float4*>(o + r * row_stride) = make_float4(a[0], a[1], a[2], a[3]);
#pragma unroll
        for (int j = 0; j < 3; ++j) { x0[j] = x1[j]; x1[j] = x2[j]; }
      }
    }
  }
  if (p.stats) {
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float a = ssum[k], b = ssq[k];
#pragma unroll
      for (int m = 4; m <= 16; m <<= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, m);
        b += __shfl_xor_sync(0xffffffffu, b, m);
      }
      if (lane < 4) {   // one slot per warp, added in (CTA, warp) order
        double* slot = ordered_slot(p.red, 0, gridDim.x * 8, blockIdx.x * 8 + (threadIdx.x >> 5), 32);
        slot[q * 4 + k] = a;
        slot[16 + q * 4 + k] = b;
      }
    }
    ordered_finish(p.red, 0, gridDim.x * 8, 32, threadIdx.x, 256, gridDim.x, [] { __syncthreads(); },
                   [&](int i, double v) { p.stats[(i < 16 ? c0 : p.Cout + c0 - 16) + i] += v; },
                   &s_last);
  }
}

int launch_conv_c1_tile(const ConvSimtParams& p, cudaStream_t stream) {
  const int tiles_w = (p.W + C1T_W - 1) / C1T_W, tiles_h = (p.H + C1T_H - 1) / C1T_H;
  const int64_t tiles = (int64_t)p.N * tiles_w * tiles_h;
  AB_CHECK(tiles < (1ll << 31), "conv_c1: too many tiles");
  int64_t blocks = tiles;
  const int64_t cap = (int64_t)ab_num_sms() * 3;
  if (blocks > cap) blocks = cap;
  const bool fast = p.act == AB_ACT_LRELU && p.alpha >= 0.f && p.alpha <= 1.f;
  ConvSimtParams q = p;
  if (p.stats && ab_ordered_ws(stream, blocks * 8 * 32, 1, &q.red)) return 1;
  if (fast)
    conv_c1_tile_kernel<1><<<(unsigned)blocks, 256, 0, stream>>>(q, tiles_w, tiles_w * tiles_h, (int)tiles);
  else
    conv_c1_tile_kernel<0><<<(unsigned)blocks, 256, 0, stream>>>(q, tiles_w, tiles_w * tiles_h, (int)tiles);
  AB_LAUNCH_CHECK();
  return 0;
}

template <int CO>
int launch_conv_c1(const ConvSimtParams& p, cudaStream_t stream) {
  const int64_t pairs = (int64_t)p.N * p.H * ((p.W + 1) / 2);
  AB_CHECK(pairs < (1ll << 31), "conv_c1: too many pixels");
  int64_t blocks = (pairs + 255) / 256;
  const int64_t cap = (int64_t)ab_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  conv_c1_kernel<CO><<<(unsigned)blocks, 256, 0, stream>>>(p);
  AB_LAUNCH_CHECK();
  return 0;
}

// Pixel-wise 1x1 convolution onto 16 channels from a few (<= 8) input channels — the data
// gradient of the classification head (nb_classes -> 16) — in the quad-lane layout: lane = pixel
// l >> 2 of an 8-pixel run x output quad l & 3.  The thread keeps its Cin x 4 weights in
// registers, the 4 lanes of a pixel share its input loads (one broadcast request), and each
// STG.128 of a warp writes 512 contiguous bytes (the thread-per-pixel kernel below writes 16-byte
// pieces 64 bytes apart).  Same per-output fmaf order as conv_pix_kernel's direct path.
template <int CIN_MAX>
__global__ void __launch_bounds__(256) conv_pix_quad_kernel(const ConvSimtParams p) {
  __shared__ unsigned s_last;
  const int lane = threadIdx.x & 31;
  const int px = lane >> 2, q = lane & 3;
  const int Cin = p.S.Ctot;
  const SrcDev sd = p.S.s[0];
  float wr[CIN_MAX][4], bq[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) bq[k] = p.bias ? __ldg(p.bias + q * 4 + k) : 0.f;
#pragma unroll
  for (int c = 0; c < CIN_MAX; ++c)
#pragma unroll
    for (int k = 0; k < 4; ++k) wr[c][k] = c < Cin ? __ldg(p.w + (size_t)c * p.Cout + q * 4 + k) : 0.f;
  if (sd.scale) {           // pending affine folded into weights and bias (as conv_pix_kernel does)
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float t = 0.f;
#pragma unroll
      for (int c = 0; c < CIN_MAX; ++c)
        if (c < Cin) t = fmaf(wr[c][k], __ldg(sd.shift + c), t);
      bq[k] += t;
    }
#pragma unroll
    for (int c = 0; c < CIN_MAX; ++c)
      if (c < Cin) {
        const float sc = __ldg(sd.scale + c);
#pragma unroll
        for (int k = 0; k < 4; ++k) wr[c][k] *= sc;
      }
  }
  const int64_t npix = (int64_t)p.N * p.H * p.W;
  float ssum[4] = {0.f, 0.f, 0.f, 0.f}, ssq[4] = {0.f, 0.f, 0.f, 0.f};
  const int64_t stride = (int64_t)gridDim.x * (blockDim.x >> 2);
#pragma unroll 4
  for (int64_t pix = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 2; pix < npix; pix += stride) {
    const float* xp = sd.ptr + pix * sd.ld;
    float a[4] = {bq[0], bq[1], bq[2], bq[3]};
#pragma unroll
    for (int c = 0; c < CIN_MAX; ++c)
      if (c < Cin) {
        const float x = __ldg(xp + c);
#pragma unroll
        for (int k = 0; k < 4; ++k) a[k] = fmaf(x, wr[c][k], a[k]);
      }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      a[k] = act_f(a[k], p.act, p.alpha);
      ssum[k] += a[k];
      ssq[k] = fmaf(a[k], a[k], ssq[k]);
    }
    *reinterpret_cast<float4*>(p.out + pix * p.ld_out + q * 4) = make_float4(a[0], a[1], a[2], a[3]);
  }
  (void)px;
  if (p.stats) {
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float a = ssum[k], b = ssq[k];
#pragma unroll
      for (int m = 4; m <= 16; m <<= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, m);
        b += __shfl_xor_sync(0xffffffffu, b, m);
      }
      if (lane < 4) {   // one slot per warp, added in (CTA, warp) order
        double* slot = ordered_slot(p.red, 0, gridDim.x * 8, blockIdx.x * 8 + (threadIdx.x >> 5), 32);
        slot[q * 4 + k] = a;
        slot[16 + q * 4 + k] = b;
      }
    }
    ordered_finish(p.red, 0, gridDim.x * 8, 32, threadIdx.x, 256, gridDim.x, [] { __syncthreads(); },
                   [&](int i, double v) { p.stats[(i < 16 ? 0 : p.Cout - 16) + i] += v; }, &s_last);
  }
}

static bool pix_quad_enabled() {
  const char* e = getenv("ATOMAI_B200_PIX_QUAD");
  return !(e && e[0] == '0');
}

int launch_conv_pix_quad(const ConvSimtParams& p, cudaStream_t stream) {
  const int64_t npix = (int64_t)p.N * p.H * p.W;
  int64_t blocks = (npix * 4 + 256 * 8 - 1) / (256 * 8);
  const int64_t cap = (int64_t)ab_num_sms() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  ConvSimtParams q = p;
  if (p.stats && ab_ordered_ws(stream, blocks * 8 * 32, 1, &q.red)) return 1;
  if (p.S.Ctot <= 4) conv_pix_quad_kernel<4><<<(unsigned)blocks, 256, 0, stream>>>(q);
  else conv_pix_quad_kernel<8><<<(unsigned)blocks, 256, 0, stream>>>(q);
  AB_LAUNCH_CHECK();
  return 0;
}

template <int CO>
int launch_conv_pix(const ConvSimtParams& p, cudaStream_t stream) {
  const int taps = p.th * p.tw, Cin = p.S.Ctot;
  const size_t smem = (size_t)taps * Cin * CO * sizeof(float);
  const int64_t npix = (int64_t)p.N * p.H * p.W;
  AB_CHECK(npix < (1ll << 32), "conv_pix: too many pixels");
  int vec = (Cin % 4 == 0);
  for (int i = 0; i < p.S.nsrc; ++i)
    if (p.S.s[i].C % 4 != 0 || p.S.s[i].ld % 4 != 0 || ((uintptr_t)p.S.s[i].ptr & 15)) vec = 0;
  int64_t blocks = (npix + 256 * 4 - 1) / (256 * 4);
  const int64_t cap = (int64_t)ab_num_sms() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  conv_pix_kernel<CO><<<(unsigned)blocks, 256, smem, stream>>>(p, vec);
  AB_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------ weight gradient
// grid: (pixel ranges, taps, co-tiles*ci-tiles).  CTA accumulates dW[co 0..63][ci 0..63] of one
// tap over its pixel range in registers (thread: 4 co x 4 ci), pixels streamed through smem in
// slabs of 64, then atomically adds into dW (OIHW).
constexpr int G_PX = 64, G_CT = 64, G_THREADS = 256;

struct WgradSimtParams {
  SrcSet S;
  int N, H, W, Cout;
  int th, tw, dil;
  const float* dy;
  int ld_dy;
  float* dw;  // OIHW
  int64_t npix;
  int px_per_cta;
  int co_tiles, ci_tiles;
  Ordered red;     // quad-lane / tile kernels: ordered sum of the per-warp partial dW
};

__global__ void __launch_bounds__(G_THREADS) conv_simt_wgrad_kernel(const WgradSimtParams p) {
  __shared__ float s_dy[G_PX][G_CT + 4];
  __shared__ float s_x[G_PX][G_CT + 4];
  const int t = blockIdx.y;
  const int ty = t / p.tw, tx = t - ty * p.tw;
  const int co_t = blockIdx.z / p.ci_tiles, ci_t = blockIdx.z % p.ci_tiles;
  const int co0 = co_t * G_CT, ci0 = ci_t * G_CT;
  const int Cin = p.S.Ctot;
  const int dh = (ty - (p.th >> 1)) * p.dil, dwid = (tx - (p.tw >> 1)) * p.dil;
  const int tid = threadIdx.x;
  const int a = tid >> 4, b = tid & 15;  // co group, ci group (4 each)
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int k = 0; k < 4; ++k) acc[i][k] = 0.f;

  const int64_t p_begin = (int64_t)blockIdx.x * p.px_per_cta;
  int64_t p_end = p_begin + p.px_per_cta;
  if (p_end > p.npix) p_end = p.npix;
  for (int64_t pb = p_begin; pb < p_end; pb += G_PX) {
    __syncthreads();
    for (int i = tid; i < G_PX * G_CT; i += G_THREADS) {
      const int c = i % G_CT, q = i / G_CT;
      const int64_t pix = pb + q;
      float vd = 0.f, vx = 0.f;
      if (pix < p_end) {
        if (co0 + c < p.Cout) vd = __ldg(p.dy + pix * p.ld_dy + co0 + c);
        if (ci0 + c < Cin) {
          const int w = (int)(pix % p.W);
          const int h = (int)((pix / p.W) % p.H);
          const int n = (int)(pix / ((int64_t)p.W * p.H));
          vx = load_src1(p.S, n, h + dh, w + dwid, p.H, p.W, ci0 + c);
        }
      }
      s_dy[q][c] = vd;
      s_x[q][c] = vx;
    }
    __syncthreads();
#pragma unroll 4
    for (int q = 0; q < G_PX; ++q) {
      const float4 d4 = *reinterpret_cast<const float4*>(&s_dy[q][a * 4]);
      const float4 x4 = *reinterpret_cast<const float4*>(&s_x[q][b * 4]);
      const float dv[4] = {d4.x, d4.y, d4.z, d4.w};
      const float xv[4] = {x4.x, x4.y, x4.z, x4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[i][k] = fmaf(dv[i], xv[k], acc[i][k]);
    }
  }
  const int taps = p.th * p.tw;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int co = co0 + a * 4 + i;
    if (co >= p.Cout) continue;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int ci = ci0 + b * 4 + k;
      if (ci < Cin) atomicAdd(p.dw + ((size_t)co * Cin + ci) * taps + t, acc[i][k]);
    }
  }
}

// ------------------------------------------------------------------ weight gradient, tiny shapes
// First layer (Cin = 1) and the pixel-wise head (Cout = nb_classes): the 64 x 64 register tiling
// above would waste > 95 % of its FMAs, so here every thread walks pixels and keeps the whole
// CO x CI x TW slice of dW in registers; one warp-shuffle reduction + atomics per CTA at the end.
// grid: (pixel ranges, tap rows (ks_h), co-groups * ci-groups).
// Weight gradient of the same layer: dW[co][0][ty][tx] = sum_p dy[p][co] * x[p + tap].  Thread =
// two adjacent pixels x CO/2 output channels (blockIdx.y picks the half): the 3 x 4 input patch
// is shared by both pixels, dy comes in as float4, the 9 x CO/2 partial sums live in registers.
template <int CO>
__global__ void __launch_bounds__(256, 2) wgrad_c1_kernel(const WgradSimtParams p) {
  constexpr int CH = CO / 2;
  const int co0 = blockIdx.y * CH;
  const SrcDev sd = p.S.s[0];
  float sc = 1.f, sh = 0.f;
  if (sd.scale) { sc = __ldg(sd.scale); sh = __ldg(sd.shift); }
  float acc[CH][9];
#pragma unroll
  for (int a = 0; a < CH; ++a)
#pragma unroll
    for (int t = 0; t < 9; ++t) acc[a][t] = 0.f;
  const int H = p.H, W = p.W, d = p.dil;
  const uint32_t Wh = (uint32_t)(W + 1) >> 1, per_img = Wh * (uint32_t)H;
  const uint32_t total = per_img * (uint32_t)p.N;
  for (uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += gridDim.x * blockDim.x) {
    const uint32_t n = idx / per_img, rem = idx - n * per_img;
    const int h = (int)(rem / Wh), w = (int)(rem - (uint32_t)h * Wh) * 2;
    const bool two = w + 1 < W;
    const float* dyp = p.dy + (((size_t)n * H + h) * W + w) * p.ld_dy + co0;
    float d0[CH], d1[CH];
#pragma unroll
    for (int a = 0; a < CH; a += 4) {
      const float4 v0 = __ldg(reinterpret_cast<const float4*>(dyp + a));
      float4 v1 = make_float4(0.f, 0.f, 0.f, 0.f);
      if (two) v1 = __ldg(reinterpret_cast<const float4*>(dyp + p.ld_dy + a));
      d0[a] = v0.x; d0[a + 1] = v0.y; d0[a + 2] = v0.z; d0[a + 3] = v0.w;
      d1[a] = v1.x; d1[a + 1] = v1.y; d1[a + 2] = v1.z; d1[a + 3] = v1.w;
    }
#pragma unroll
    for (int ty = 0; ty < 3; ++ty) {
      const int hh = h + (ty - 1) * d;
      const bool rok = (unsigned)hh < (unsigned)H;
      const float* rowp = sd.ptr + ((size_t)n * H + (rok ? hh : 0)) * W * sd.ld;
#pragma unroll
      for (int tx = 0; tx < 3; ++tx) {
        const int w0 = w + (tx - 1) * d, w1 = w0 + 1;
        const bool ok0 = rok && (unsigned)w0 < (unsigned)W, ok1 = rok && (unsigned)w1 < (unsigned)W;
        const float x0 = ok0 ? fmaf(__ldg(rowp + (size_t)w0 * sd.ld), sc, sh) : 0.f;
        const float x1 = ok1 ? fmaf(__ldg(rowp + (size_t)w1 * sd.ld), sc, sh) : 0.f;
#pragma unroll
        for (int a = 0; a < CH; ++a)
          acc[a][ty * 3 + tx] = fmaf(d0[a], x0, fmaf(d1[a], x1, acc[a][ty * 3 + tx]));
      }
    }
  }
  __shared__ float s_acc[CH * 9];
  for (int i = threadIdx.x; i < CH * 9; i += blockDim.x) s_acc[i] = 0.f;
  __syncthreads();
#pragma unroll
  for (int a = 0; a < CH; ++a)
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const float v = warp_sum(acc[a][t]);
      if ((threadIdx.x & 31) == 0) atomicAdd(&s_acc[a * 9 + t], v);
    }
  __syncthreads();
  for (int i = threadIdx.x; i < CH * 9; i += blockDim.x)
    atomicAdd(p.dw + (size_t)(co0 + i / 9) * 9 + i % 9, s_acc[i]);   // OIHW with Cin = 1
}

// First-layer weight gradient, tile version (same CTA tile, halo staging and lane mapping as
// conv_c1_tile_kernel): a thread accumulates dW[4 channels of its quad][9 taps] over its pixels,
// so all 16 channels go in ONE pass over dy (the pair kernel above reads dy twice, 8 channels
// per pass) with 512-byte coalesced LDG.128 rows.
__global__ void __launch_bounds__(256) wgrad_c1_tile_kernel(const WgradSimtParams p, int tiles_w,
                                                            int tiles_hw, int num_tiles) {
  __shared__ float s_x[C1T_ELEMS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int px = lane >> 2, q = lane & 3;
  const int col = warp * 8 + px;
  const SrcDev sd = p.S.s[0];
  float sc = 1.f, sh = 0.f;
  if (sd.scale) { sc = __ldg(sd.scale); sh = __ldg(sd.shift); }
  const int H = p.H, W = p.W;
  float acc[4][9];
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int t = 0; t < 9; ++t) acc[k][t] = 0.f;
  float nxt[C1T_PER_THREAD];
  int tile = blockIdx.x;
  C1Tile cur = c1_tile(tile < num_tiles ? tile : 0, tiles_w, tiles_hw);
  if (tile < num_tiles) c1_fetch(sd, sc, sh, H, W, cur, nxt);
  for (; tile < num_tiles; tile += gridDim.x) {
    __syncthreads();
    c1_stage(s_x, nxt);
    __syncthreads();
    const C1Tile me = cur;
    const int tn = tile + gridDim.x;
    if (tn < num_tiles) {
      cur = c1_tile(tn, tiles_w, tiles_hw);
      c1_fetch(sd, sc, sh, H, W, cur, nxt);
    }
    const int gw = me.w0 + col;
    if (gw < W) {
      const float* sp = s_x + col;
      float x0[3], x1[3], x2[3];
#pragma unroll
      for (int j = 0; j < 3; ++j) { x0[j] = sp[j]; x1[j] = sp[C1T_PW + j]; }
      const float* dyp = p.dy + (((size_t)me.n * H + me.h0) * W + gw) * p.ld_dy + q * 4;
      const size_t row_stride = (size_t)W * p.ld_dy;
      const int rows = min(C1T_H, H - me.h0);
#pragma unroll 4
      for (int r = 0; r < rows; ++r) {
        const float4 d4 = __ldg(reinterpret_cast<const float4*>(dyp + r * row_stride));
#pragma unroll
        for (int j = 0; j < 3; ++j) x2[j] = sp[(r + 2) * C1T_PW + j];
        const float dv[4] = {d4.x, d4.y, d4.z, d4.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
#pragma unroll
          for (int j = 0; j < 3; ++j) {
            acc[k][j] = fmaf(dv[k], x0[j], acc[k][j]);
            acc[k][3 + j] = fmaf(dv[k], x1[j], acc[k][3 + j]);
            acc[k][6 + j] = fmaf(dv[k], x2[j], acc[k][6 + j]);
          }
        }
#pragma unroll
        for (int j = 0; j < 3; ++j) { x0[j] = x1[j]; x1[j] = x2[j]; }
      }
    }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      float v = acc[k][t];
#pragma unroll
      for (int m = 4; m <= 16; m <<= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
      if (lane < 4)     // one slot per warp, added in (CTA, warp) order
        ordered_slot(p.red, 0, gridDim.x * 8, blockIdx.x * 8 + warp, 16 * 9)[(q * 4 + k) * 9 + t] = v;
    }
  __shared__ unsigned s_last;
  ordered_finish(p.red, 0, gridDim.x * 8, 16 * 9, threadIdx.x, 256, gridDim.x, [] { __syncthreads(); },
                 [&](int i, double v) { p.dw[i] += (float)v; }, &s_last);   // OIHW, Cin = 1
}

int launch_wgrad_c1_tile(const WgradSimtParams& p, cudaStream_t stream) {
  const int tiles_w = (p.W + C1T_W - 1) / C1T_W, tiles_h = (p.H + C1T_H - 1) / C1T_H;
  const int64_t tiles = (int64_t)p.N * tiles_w * tiles_h;
  AB_CHECK(tiles < (1ll << 31), "wgrad_c1: too many tiles");
  int64_t blocks = tiles;
  const int64_t cap = (int64_t)ab_num_sms() * 3;
  if (blocks > cap) blocks = cap;
  WgradSimtParams q = p;
  if (ab_ordered_ws(stream, blocks * 8 * 16 * 9, 1, &q.red)) return 1;
  wgrad_c1_tile_kernel<<<(unsigned)blocks, 256, 0, stream>>>(q, tiles_w, tiles_w * tiles_h, (int)tiles);
  AB_LAUNCH_CHECK();
  return 0;
}

// the tile kernels want dilation 1 and rows that fill most of the 64-pixel tile width
static bool c1_tile_ok(int dil, int W) {
  if (const char* e = getenv("ATOMAI_B200_C1_TILE"))
    if (e[0] == '0') return false;
  const int tiles_w = (W + C1T_W - 1) / C1T_W;
  return dil == 1 && tiles_w * C1T_W - W <= W / 4;
}

template <int CO>
int launch_wgrad_c1(const WgradSimtParams& p, cudaStream_t stream) {
  const int64_t pairs = (int64_t)p.N * p.H * ((p.W + 1) / 2);
  AB_CHECK(pairs < (1ll << 31), "wgrad_c1: too many pixels");
  int64_t bx = (pairs + 256 * 8 - 1) / (256 * 8);
  const int64_t cap = (int64_t)ab_num_sms() * 4;
  if (bx > cap) bx = cap;
  if (bx < 1) bx = 1;
  dim3 grid((unsigned)bx, 2, 1);
  wgrad_c1_kernel<CO><<<grid, 256, 0, stream>>>(p);
  AB_LAUNCH_CHECK();
  return 0;
}

template <int CO, int CI, int TH, int TW>
__global__ void __launch_bounds__(256) wgrad_small_kernel(const WgradSimtParams p, int co_groups) {
  const int cog = blockIdx.z % co_groups, cig = blockIdx.z / co_groups;
  const int co0 = cog * CO, ci0 = cig * CI;
  const int Cin = p.S.Ctot;
  float acc[CO][CI][TH * TW];
#pragma unroll
  for (int a = 0; a < CO; ++a)
#pragma unroll
    for (int b = 0; b < CI; ++b)
#pragma unroll
      for (int t = 0; t < TH * TW; ++t) acc[a][b][t] = 0.f;
  const uint32_t uW = p.W, uHW = (uint32_t)p.H * p.W;      // npix < 2^32 (checked by the launcher)
  // float4 loads when the channel group is whole, aligned and inside one source
  const bool dy_vec = CO % 4 == 0 && co0 + CO <= p.Cout && (p.ld_dy & 3) == 0 &&
                      ((uintptr_t)(p.dy + co0) & 15) == 0;
  const bool x_vec = CI % 4 == 0 && ci0 + CI <= Cin && p.S.nsrc == 1 && (p.S.s[0].ld & 3) == 0 &&
                     ((uintptr_t)p.S.s[0].ptr & 15) == 0 && (p.S.s[0].C & 3) == 0;
  for (int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < p.npix;
       pix += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t up = (uint32_t)pix;
    const int n = (int)(up / uHW);
    const uint32_t rem = up - (uint32_t)n * uHW;
    const int h = (int)(rem / uW);
    const int w = (int)(rem - (uint32_t)h * uW);
    float d[CO];
    if (dy_vec) {
#pragma unroll
      for (int a = 0; a < CO; a += 4) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(p.dy + pix * p.ld_dy + co0 + a));
        d[a] = v.x; d[a + 1] = v.y; d[a + 2] = v.z; d[a + 3] = v.w;
      }
    } else {
#pragma unroll
      for (int a = 0; a < CO; ++a)
        d[a] = (co0 + a < p.Cout) ? __ldg(p.dy + pix * p.ld_dy + co0 + a) : 0.f;
    }
#pragma unroll
    for (int ty = 0; ty < TH; ++ty) {
      const int hh = h + (ty - (TH >> 1)) * p.dil;
#pragma unroll
      for (int tx = 0; tx < TW; ++tx) {
        const int ww = w + (tx - (TW >> 1)) * p.dil;
        float x[CI];
        if (x_vec) {
#pragma unroll
          for (int b = 0; b < CI; b += 4) {
            const float4 v = load_src4(p.S, n, hh, ww, p.H, p.W, ci0 + b);
            x[b] = v.x; x[b + 1] = v.y; x[b + 2] = v.z; x[b + 3] = v.w;
          }
        } else {
#pragma unroll
          for (int b = 0; b < CI; ++b)
            x[b] = (ci0 + b < Cin) ? load_src1(p.S, n, hh, ww, p.H, p.W, ci0 + b) : 0.f;
        }
#pragma unroll
        for (int b = 0; b < CI; ++b)
#pragma unroll
          for (int a = 0; a < CO; ++a)
            acc[a][b][ty * TW + tx] = fmaf(d[a], x[b], acc[a][b][ty * TW + tx]);
      }
    }
  }
  constexpr int NA = CO * CI * TH * TW;
  __shared__ float s_acc[NA];
  for (int i = threadIdx.x; i < NA; i += blockDim.x) s_acc[i] = 0.f;
  __syncthreads();
#pragma unroll
  for (int a = 0; a < CO; ++a)
#pragma unroll
    for (int b = 0; b < CI; ++b)
#pragma unroll
      for (int t = 0; t < TH * TW; ++t) {
        const float v = warp_sum(acc[a][b][t]);
        if ((threadIdx.x & 31) == 0) atomicAdd(&s_acc[(a * CI + b) * (TH * TW) + t], v);
      }
  __syncthreads();
  for (int i = threadIdx.x; i < NA; i += blockDim.x) {
    const int t = i % (TH * TW), b = (i / (TH * TW)) % CI, a = i / (TH * TW * CI);
    if (co0 + a < p.Cout && ci0 + b < Cin)
      atomicAdd(p.dw + ((size_t)(co0 + a) * Cin + ci0 + b) * (TH * TW) + t, s_acc[i]);
  }
}

// Weight gradient of a pixel-wise head with <= 4 outputs from 16 input channels (16 -> nb_classes,
// 1x1), quad-lane layout: lane = pixel l >> 2 x input quad l & 3, so the 16-channel activation is
// read with 512-byte coalesced LDG.128 rows (thread-per-pixel: four 16-byte pieces 64 bytes
// apart per thread); the <= 4 dy values of a pixel are one broadcast request per quad.
__global__ void __launch_bounds__(256) wgrad_pix_quad_kernel(const WgradSimtParams p) {
  const int lane = threadIdx.x & 31;
  const int q = lane & 3;
  const int Cout = p.Cout;
  const SrcDev sd = p.S.s[0];
  float4 sc = make_float4(1.f, 1.f, 1.f, 1.f), sh = make_float4(0.f, 0.f, 0.f, 0.f);
  if (sd.scale) {
    sc = __ldg(reinterpret_cast<const float4*>(sd.scale + q * 4));
    sh = __ldg(reinterpret_cast<const float4*>(sd.shift + q * 4));
  }
  float acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
  const int64_t stride = (int64_t)gridDim.x * (blockDim.x >> 2);
#pragma unroll 4
  for (int64_t pix = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 2; pix < p.npix; pix += stride) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(sd.ptr + pix * sd.ld + q * 4));
    const float x[4] = {fmaf(v.x, sc.x, sh.x), fmaf(v.y, sc.y, sh.y), fmaf(v.z, sc.z, sh.z),
                        fmaf(v.w, sc.w, sh.w)};
    const float* dyp = p.dy + pix * p.ld_dy;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const float d = a < Cout ? __ldg(dyp + a) : 0.f;
#pragma unroll
      for (int b = 0; b < 4; ++b) acc[a][b] = fmaf(d, x[b], acc[a][b]);
    }
  }
  __syncthreads();
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      float v = acc[a][b];
#pragma unroll
      for (int m = 4; m <= 16; m <<= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
      if (lane < 4)     // one slot per warp, added in (CTA, warp) order
        ordered_slot(p.red, 0, gridDim.x * 8, blockIdx.x * 8 + (threadIdx.x >> 5), 64)[a * 16 + q * 4 + b] = v;
    }
  __shared__ unsigned s_last;
  ordered_finish(p.red, 0, gridDim.x * 8, 64, threadIdx.x, 256, gridDim.x, [] { __syncthreads(); },
                 [&](int i, double v) { if ((i >> 4) < Cout) p.dw[(size_t)(i >> 4) * 16 + (i & 15)] += (float)v; },
                 &s_last);                                            // OIHW with 1x1 taps
}

int launch_wgrad_pix_quad(const WgradSimtParams& p, cudaStream_t stream) {
  int64_t blocks = (p.npix * 4 + 256 * 8 - 1) / (256 * 8);
  const int64_t cap = (int64_t)ab_num_sms() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  WgradSimtParams q = p;
  if (ab_ordered_ws(stream, blocks * 8 * 64, 1, &q.red)) return 1;
  wgrad_pix_quad_kernel<<<(unsigned)blocks, 256, 0, stream>>>(q);
  AB_LAUNCH_CHECK();
  return 0;
}

template <int CO, int CI, int TH, int TW>
int launch_wgrad_small(const WgradSimtParams& p, cudaStream_t stream) {
  AB_CHECK(p.npix < (1ll << 32), "wgrad_small: too many pixels");
  AB_CHECK(p.th == TH && p.tw == TW, "wgrad_small: kernel %dx%d != %dx%d", p.th, p.tw, TH, TW);
  const int co_groups = (p.Cout + CO - 1) / CO, ci_groups = (p.S.Ctot + CI - 1) / CI;
  int64_t bx = (p.npix + 256 * 16 - 1) / (256 * 16);
  const int64_t cap = (int64_t)ab_num_sms() * 4;
  if (bx > cap) bx = cap;
  if (bx < 1) bx = 1;
  dim3 grid((unsigned)bx, 1, co_groups * ci_groups);
  wgrad_small_kernel<CO, CI, TH, TW><<<grid, 256, 0, stream>>>(p, co_groups);
  AB_LAUNCH_CHECK();
  return 0;
}

// W[co][ci][ty][tx] -> [tap][Cin][Cout] (FWD) ; dgrad: out[tap][co][ci] with flipped taps
__global__ void pack_weights_simt_kernel(const float* __restrict__ w, int Cout, int Cin, int th,
                                         int tw, int mode, float* __restrict__ out,
                                         int64_t total) {
  const int taps = th * tw;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    if (mode == AB_WMODE_FWD) {
      const int co = i % Cout, ci = (i / Cout) % Cin, t = (int)(i / ((int64_t)Cout * Cin));
      out[i] = w[((int64_t)co * Cin + ci) * taps + t];
    } else {  // conv input = dy (Cout ch), output = dx (Cin ch): out[tap][co][ci]
      const int ci = i % Cin, co = (i / Cin) % Cout, t = (int)(i / ((int64_t)Cout * Cin));
      out[i] = w[((int64_t)co * Cin + ci) * taps + (taps - 1 - t)];
    }
  }
}

}  // namespace

int ab_pack_weights_simt(const float* w, int Cout, int Cin, int th, int tw, int mode, float* out,
                         cudaStream_t stream) {
  const int64_t total = (int64_t)Cout * Cin * th * tw;
  const int threads = 256;
  int64_t blocks = (total + threads - 1) / threads;
  if (blocks > 4096) blocks = 4096;
  pack_weights_simt_kernel<<<(int)blocks, threads, 0, stream>>>(w, Cout, Cin, th, tw, mode, out,
                                                                total);
  AB_LAUNCH_CHECK();
  return 0;
}

int ab_conv_simt_fwd(const ab_conv_t* d, const float* w, const float* bias, float* y, int ld_y,
                     double* stats, cudaStream_t stream) {
  ConvSimtParams p;
  if (ab_make_srcset(d, &p.S)) return 1;
  p.N = d->N; p.H = d->H; p.W = d->W; p.Cout = d->Cout;
  p.th = d->ks_h; p.tw = d->ks_w; p.dil = d->dil;
  p.w = w; p.bias = bias; p.alpha = d->lrelu; p.act = d->act; p.out = y; p.ld_out = ld_y;
  p.out_nchw = d->out_nchw; p.stats = stats;
  p.tiles_h = (d->H + F_TH - 1) / F_TH;
  p.tiles_w = (d->W + F_TW - 1) / F_TW;
  // thin-channel specialisations (first layer, pixel-wise head and its data-gradient)
  {
    const int Cin = p.S.Ctot, taps = d->ks_h * d->ks_w;
    p.c0 = 0;
    if (Cin == 1 && d->ks_h == 3 && d->ks_w == 3 && d->Cout % 16 == 0 && d->Cout <= 256 &&
        p.S.nsrc == 1 && !p.S.s[0].pool && !d->out_nchw && ld_y % 4 == 0 && ((uintptr_t)y & 15) == 0 &&
        d->N * (int64_t)d->H * d->W > 0) {
      // first layer of every net (Unet 1 -> 16, ImSpec 1 -> 64, VAE 1 -> 128): one launch per block
      // of 16 output channels, the single-channel input stays in L2 between them
      const bool tile = c1_tile_ok(d->dil, d->W);
      for (p.c0 = 0; p.c0 < d->Cout; p.c0 += 16)
        if (tile ? launch_conv_c1_tile(p, stream) : launch_conv_c1<16>(p, stream)) return 1;
      return 0;
    }
    if (d->N * (int64_t)d->H * d->W > 0) {
      // pixel-wise kernels: weights in shared memory ([taps][Cin][CO] floats), all CO outputs of a
      // pixel in registers.  Heads with <= 4 outputs take any Cin up to 1024 taps*channels (the
      // rDecoder's 128 -> 1 output layer); wider outputs from <= 64 taps*channels run as blocks of
      // 32 channels (the 1 -> 128 data-gradient of that layer)
      if (d->Cout <= 4 && taps * Cin <= 1024) return launch_conv_pix<4>(p, stream);
      if (taps * Cin <= 64) {
        if (d->Cout == 8) return launch_conv_pix<8>(p, stream);
        if (d->Cout == 16 && taps == 1 && Cin <= 8 && p.S.nsrc == 1 && !p.S.s[0].pool && !d->out_nchw &&
            ld_y % 4 == 0 && ((uintptr_t)y & 15) == 0 && pix_quad_enabled())
          return launch_conv_pix_quad(p, stream);
        if (d->Cout == 16) return launch_conv_pix<16>(p, stream);
        if (d->Cout % 32 == 0 && d->Cout <= 256 && !d->out_nchw) {
          for (p.c0 = 0; p.c0 < d->Cout; p.c0 += 32)
            if (launch_conv_pix<32>(p, stream)) return 1;
          return 0;
        }
      }
    }
    p.c0 = 0;
  }
  const int ph = d->dil * (d->ks_h >> 1), pw = d->dil * (d->ks_w >> 1);
  const int smem = (F_CIT * (F_TH + 2 * ph) * (F_TW + 2 * pw) + d->ks_h * d->ks_w * F_CIT * F_COT) *
                   (int)sizeof(float);
  AB_CHECK(smem <= 200 * 1024, "conv_simt: dilation %d too large", d->dil);
  static unsigned char optin[64];
  if (smem > 48 * 1024 &&
      ab_optin_smem(reinterpret_cast<const void*>(conv_simt_fwd_kernel), 200 * 1024, optin))
    return 1;
  const int64_t tiles = (int64_t)d->N * p.tiles_h * p.tiles_w;
  AB_CHECK(tiles < (1ll << 31), "conv_simt: too many tiles");
  if (tiles == 0) return 0;
  dim3 grid((unsigned)tiles, (d->Cout + F_COT - 1) / F_COT);
  conv_simt_fwd_kernel<<<grid, F_THREADS, smem, stream>>>(p);
  AB_LAUNCH_CHECK();
  return 0;
}

int ab_conv_simt_wgrad(const ab_conv_t* d, const float* dy, int ld_dy, float* dw,
                       cudaStream_t stream) {
  WgradSimtParams p;
  if (ab_make_srcset(d, &p.S)) return 1;
  p.N = d->N; p.H = d->H; p.W = d->W; p.Cout = d->Cout;
  p.th = d->ks_h; p.tw = d->ks_w; p.dil = d->dil;
  p.dy = dy; p.ld_dy = ld_dy; p.dw = dw;
  p.npix = (int64_t)d->N * d->H * d->W;
  if (p.npix == 0) return 0;
  p.co_tiles = (d->Cout + G_CT - 1) / G_CT;
  p.ci_tiles = (p.S.Ctot + G_CT - 1) / G_CT;
  p.px_per_cta = 0;
  if (p.S.Ctot == 1 && d->ks_w == 3 && d->ks_h == 3 && d->Cout == 16 && p.S.nsrc == 1 &&
      !p.S.s[0].pool && ld_dy % 4 == 0 && ((uintptr_t)dy & 15) == 0)
    return c1_tile_ok(d->dil, d->W) ? launch_wgrad_c1_tile(p, stream) : launch_wgrad_c1<16>(p, stream);
  if (p.S.Ctot <= 2 && d->ks_w == 3 && d->ks_h == 3) return launch_wgrad_small<8, 1, 3, 3>(p, stream);
  if (p.S.Ctot <= 2 && d->ks_w == 3 && d->ks_h == 1) return launch_wgrad_small<16, 1, 1, 3>(p, stream);
  if (p.S.Ctot <= 2 && d->ks_w == 1 && d->ks_h == 1) return launch_wgrad_small<16, 2, 1, 1>(p, stream);
  if (d->Cout <= 4 && d->ks_w == 1 && d->ks_h == 1 && p.S.Ctot == 16 && p.S.nsrc == 1 && !p.S.s[0].pool &&
      (p.S.s[0].ld & 3) == 0 && ((uintptr_t)p.S.s[0].ptr & 15) == 0 &&
      (!p.S.s[0].scale || (((uintptr_t)p.S.s[0].scale | (uintptr_t)p.S.s[0].shift) & 15) == 0) &&
      pix_quad_enabled())
    return launch_wgrad_pix_quad(p, stream);
  if (d->Cout <= 4 && d->ks_w == 1 && d->ks_h == 1) return launch_wgrad_small<4, 16, 1, 1>(p, stream);
  if (d->Cout <= 4 && d->ks_w == 3 && d->ks_h == 3) return launch_wgrad_small<4, 4, 3, 3>(p, stream);
  if (d->Cout <= 4 && d->ks_w == 3 && d->ks_h == 1) return launch_wgrad_small<4, 4, 1, 3>(p, stream);
  const int taps = d->ks_h * d->ks_w;
  const int64_t per_range_ctas = (int64_t)taps * p.co_tiles * p.ci_tiles;
  int64_t ranges = (4ll * ab_num_sms() + per_range_ctas - 1) / per_range_ctas;  // ~4 waves
  int64_t max_ranges = (p.npix + G_PX - 1) / G_PX;
  if (ranges > max_ranges) ranges = max_ranges;
  if (ranges < 1) ranges = 1;
  int64_t ppc = (p.npix + ranges - 1) / ranges;
  ppc = (ppc + G_PX - 1) / G_PX * G_PX;
  ranges = (p.npix + ppc - 1) / ppc;
  p.px_per_cta = (int)ppc;
  dim3 grid((unsigned)ranges, taps, p.co_tiles * p.ci_tiles);
  conv_simt_wgrad_kernel<<<grid, G_THREADS, 0, stream>>>(p);
  AB_LAUNCH_CHECK();
  return 0;
}
