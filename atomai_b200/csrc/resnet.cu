// resnet.cu — the element-wise pieces of the ResBlock networks (SegResNet / ResHedNet):
//   * y = LeakyReLU(a*scale + shift + residual): the BatchNorm -> (+ residual) -> LeakyReLU tail of
//     atomai/nets/blocks.py:199-214 in ONE pass over HBM (the reference runs three), and its
//     backward mask g = dy * LeakyReLU'(y);
//   * F.interpolate(size = integer multiple, mode = bilinear (align_corners=False) | nearest) of
//     atomai/nets/fcnn.py:292-293 (ResHedNet side outputs, x2 and x4) and its adjoint.
// All HBM-bound, grid-stride, scalar (the side outputs have nb_classes = 1..3 channels) with a
// float4 path when C % 4 == 0.
#include "common.cuh"

namespace {

constexpr int kT = 256;

// W = 4 channels per thread on the float4 path, W = 1 otherwise (common.cuh: Lanes, ChanIdx)
template <int W>
__global__ void __launch_bounds__(kT)
    affine_res_act_kernel(const float* __restrict__ a, int ld_a, const float* __restrict__ scale,
                          const float* __restrict__ shift, const float* __restrict__ res,
                          int ld_res, float slope, float* __restrict__ y, int ld_y,
                          typename ChanIdx<W>::I total, ChanIdx<W> ix) {
  using I = typename ChanIdx<W>::I;
  for (I i = blockIdx.x * (I)kT + threadIdx.x; i < total; i += (I)gridDim.x * kT) {
    I pix; int c; ix.split(i, pix, c);
    Lanes<W> v = lanes_ld<W>(a + (size_t)pix * ld_a + c);
    if (scale) {
      const Lanes<W> s = lanes_ld<W>(scale + c), t = lanes_ld<W>(shift + c);
#pragma unroll
      for (int k = 0; k < W; ++k) v[k] = fmaf(v[k], s[k], t[k]);
    }
    if (res) {
      const Lanes<W> r = lanes_ld<W>(res + (size_t)pix * ld_res + c);
#pragma unroll
      for (int k = 0; k < W; ++k) v[k] += r[k];
    }
#pragma unroll
    for (int k = 0; k < W; ++k) v[k] = v[k] > 0.f ? v[k] : v[k] * slope;
    lanes_at<W>(y + (size_t)pix * ld_y + c) = v;
  }
}

__global__ void __launch_bounds__(kT)
    lrelu_mask_bwd_kernel(const float* __restrict__ dy, int ld_dy, const float* __restrict__ y,
                          int ld_y, float slope, float* __restrict__ g, int ld_g, int64_t npix,
                          int C) {
  const int64_t total = npix * C;
  for (int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x; i < total; i += (int64_t)gridDim.x * kT) {
    const int c = (int)(i % C);
    const int64_t pix = i / C;
    const float d = dy[pix * ld_dy + c];
    g[pix * ld_g + c] = y[pix * ld_y + c] > 0.f ? d : d * slope;
  }
}

// source coordinate of output index o (PyTorch area_pixel_compute_source_index, align_corners=False)
__device__ __forceinline__ void bil_src(int o, int f, int in, int& i0, int& i1, float& l1) {
  float s = (1.f / (float)f) * ((float)o + 0.5f) - 0.5f;   // ATen: scale * (dst + 0.5) - 0.5
  s = s < 0.f ? 0.f : s;
  i0 = (int)s;
  i1 = i0 + (i0 < in - 1 ? 1 : 0);
  l1 = s - (float)i0;
}

__global__ void __launch_bounds__(kT)
    resize_fwd_kernel(const float* __restrict__ x, int ld_x, float* __restrict__ y, int ld_y, int N,
                      int h, int w, int C, int f, int bilinear) {
  const int H = h * f, W = w * f;
  const int64_t total = (int64_t)N * H * W * C;
  for (int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x; i < total; i += (int64_t)gridDim.x * kT) {
    const int c = (int)(i % C);
    int64_t r = i / C;
    const int ow = (int)(r % W); r /= W;
    const int oh = (int)(r % H);
    const int n = (int)(r / H);
    const float* xb = x + (size_t)n * h * w * ld_x + c;
    float v;
    if (bilinear) {
      int h0, h1, w0, w1; float lh, lw;
      bil_src(oh, f, h, h0, h1, lh);
      bil_src(ow, f, w, w0, w1, lw);
      const float v00 = xb[((size_t)h0 * w + w0) * ld_x], v01 = xb[((size_t)h0 * w + w1) * ld_x];
      const float v10 = xb[((size_t)h1 * w + w0) * ld_x], v11 = xb[((size_t)h1 * w + w1) * ld_x];
      // same association as ATen's upsample_bilinear2d: h0lambda*(w0lambda*v00 + w1lambda*v01) + ...
      v = (1.f - lh) * ((1.f - lw) * v00 + lw * v01) + lh * ((1.f - lw) * v10 + lw * v11);
    } else {
      v = xb[((size_t)(oh / f) * w + (ow / f)) * ld_x];
    }
    y[(((size_t)n * H + oh) * W + ow) * ld_y + c] = v;
  }
}

// adjoint: dx (zeroed by the caller) += scatter(dy)
__global__ void __launch_bounds__(kT)
    resize_bwd_kernel(const float* __restrict__ dy, int ld_dy, float* __restrict__ dx, int ld_dx,
                      int N, int h, int w, int C, int f, int bilinear) {
  const int H = h * f, W = w * f;
  const int64_t total = (int64_t)N * H * W * C;
  for (int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x; i < total; i += (int64_t)gridDim.x * kT) {
    const int c = (int)(i % C);
    int64_t r = i / C;
    const int ow = (int)(r % W); r /= W;
    const int oh = (int)(r % H);
    const int n = (int)(r / H);
    const float g = dy[(((size_t)n * H + oh) * W + ow) * ld_dy + c];
    float* db = dx + (size_t)n * h * w * ld_dx + c;
    if (bilinear) {
      int h0, h1, w0, w1; float lh, lw;
      bil_src(oh, f, h, h0, h1, lh);
      bil_src(ow, f, w, w0, w1, lw);
      atomicAdd(db + ((size_t)h0 * w + w0) * ld_dx, (1.f - lh) * (1.f - lw) * g);
      atomicAdd(db + ((size_t)h0 * w + w1) * ld_dx, (1.f - lh) * lw * g);
      atomicAdd(db + ((size_t)h1 * w + w0) * ld_dx, lh * (1.f - lw) * g);
      atomicAdd(db + ((size_t)h1 * w + w1) * ld_dx, lh * lw * g);
    } else {
      atomicAdd(db + ((size_t)(oh / f) * w + (ow / f)) * ld_dx, g);
    }
  }
}

}  // namespace

extern "C" {

#define STREAM ((cudaStream_t)stream)

int atomai_b200_affine_res_act(const float* a, int ld_a, const float* scale, const float* shift,
                               const float* res, int ld_res, float lrelu, float* y, int ld_y,
                               int64_t npix, int C, void* stream) {
  AB_CHECK(a && y && C > 0 && npix >= 0, "affine_res_act: bad arguments");
  AB_CHECK((scale == nullptr) == (shift == nullptr), "affine_res_act: scale and shift go together");
  if (npix == 0) return 0;
  const bool vec = vec_ok(C, {a, y, scale, shift, res}, {ld_a, ld_y, res ? ld_res : 0}, npix * C / 4);
  return by_width(vec, [&](auto vw) {
    constexpr int W = decltype(vw)::value;
    affine_res_act_kernel<W><<<ab_grid(npix * C / W, kT, 16), kT, 0, STREAM>>>(
        a, ld_a, scale, shift, res, ld_res, lrelu, y, ld_y, npix * C / W, ChanIdx<W>(C));
    AB_LAUNCH_CHECK();
    return 0;
  });
}

int atomai_b200_lrelu_mask_bwd(const float* dy, int ld_dy, const float* y, int ld_y, float lrelu,
                               float* g, int ld_g, int64_t npix, int C, void* stream) {
  AB_CHECK(dy && y && g && C > 0 && npix >= 0, "lrelu_mask_bwd: bad arguments");
  AB_CHECK(lrelu > 0.f, "lrelu_mask_bwd: the mask is read from sign(y), which needs slope > 0");
  if (npix == 0) return 0;
  lrelu_mask_bwd_kernel<<<ab_grid(npix * C, kT, 16), kT, 0, STREAM>>>(dy, ld_dy, y, ld_y, lrelu, g, ld_g,
                                                              npix, C);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_resize_fwd(const float* x, int ld_x, float* y, int ld_y, int N, int h, int w, int C,
                           int factor, int bilinear, void* stream) {
  AB_CHECK(x && y && factor >= 1 && C > 0, "resize_fwd: bad arguments");
  if ((int64_t)N * h * w == 0) return 0;
  resize_fwd_kernel<<<ab_grid((int64_t)N * h * w * factor * factor * C, kT, 16), kT, 0, STREAM>>>(
      x, ld_x, y, ld_y, N, h, w, C, factor, bilinear);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_resize_bwd(const float* dy, int ld_dy, float* dx, int ld_dx, int N, int h, int w,
                           int C, int factor, int bilinear, void* stream) {
  AB_CHECK(dy && dx && factor >= 1 && C > 0, "resize_bwd: bad arguments");
  if ((int64_t)N * h * w == 0) return 0;
  resize_bwd_kernel<<<ab_grid((int64_t)N * h * w * factor * factor * C, kT, 16), kT, 0, STREAM>>>(
      dy, ld_dy, dx, ld_dx, N, h, w, C, factor, bilinear);
  AB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
