// ed_ops.cu — the resampling steps of the ImSpec encoder / decoder options
// (atomai/nets/ed.py:66-79, 141-157):
//   * avgpool_fwd: F.avg_pool2d(x, s, s) of an image, or F.avg_pool1d(x, s, s) of a spectrum stored
//     as (N, 1, L, 1), on an NHWC tensor with window (sh, sw) and floor semantics (trailing rows and
//     columns that do not fill a window are dropped).  Each output is the sum of its window in
//     row-major order times 1/(sh*sw).  Forward only: it pools the network input, which carries no
//     gradient on these paths.
//   * upsample_w2x_fwd / _bwd: F.interpolate(scale_factor=2, mode="nearest") of a 1-D signal stored
//     as (N, 1, w, C), and its adjoint (the sum of each output pair).
// HBM-bound, grid-stride, one thread per output element, coalesced along the channel axis.
#include "common.cuh"

namespace {

constexpr int kT = 256;

__global__ void __launch_bounds__(kT)
    avgpool_fwd_kernel(const float* __restrict__ x, int ld_x, float* __restrict__ y, int ld_y,
                       int N, int H, int W, int C, int sh, int sw) {
  const int Ho = H / sh, Wo = W / sw;
  const int64_t total = (int64_t)N * Ho * Wo * C;
  const float inv = 1.f / (float)(sh * sw);
  for (int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x; i < total; i += (int64_t)gridDim.x * kT) {
    const int c = (int)(i % C);
    int64_t r = i / C;
    const int wo = (int)(r % Wo); r /= Wo;
    const int ho = (int)(r % Ho);
    const int n = (int)(r / Ho);
    const float* xb = x + (((int64_t)n * H + (int64_t)ho * sh) * W + (int64_t)wo * sw) * ld_x + c;
    float acc = 0.f;
    for (int a = 0; a < sh; ++a)
      for (int b = 0; b < sw; ++b) acc += xb[((int64_t)a * W + b) * ld_x];
    y[(((int64_t)n * Ho + ho) * Wo + wo) * ld_y + c] = acc * inv;
  }
}

__global__ void __launch_bounds__(kT)
    upsample_w2x_fwd_kernel(const float* __restrict__ x, int ld_x, float* __restrict__ y, int ld_y,
                            int64_t rows_out, int C) {
  // rows_out = N * 2w output positions; output position p reads input position p / 2 (same n)
  const int64_t total = rows_out * C;
  for (int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x; i < total; i += (int64_t)gridDim.x * kT) {
    const int c = (int)(i % C);
    const int64_t p = i / C;
    y[p * ld_y + c] = x[(p >> 1) * ld_x + c];
  }
}

__global__ void __launch_bounds__(kT)
    upsample_w2x_bwd_kernel(const float* __restrict__ dy, int ld_dy, float* __restrict__ dx,
                            int ld_dx, int64_t rows_in, int C) {
  const int64_t total = rows_in * C;
  for (int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x; i < total; i += (int64_t)gridDim.x * kT) {
    const int c = (int)(i % C);
    const int64_t p = i / C;
    dx[p * ld_dx + c] = dy[(2 * p) * ld_dy + c] + dy[(2 * p + 1) * ld_dy + c];
  }
}

}  // namespace

extern "C" {

#define STREAM ((cudaStream_t)stream)

int atomai_b200_avgpool_fwd(const float* x, int ld_x, float* y, int ld_y, int N, int H, int W, int C,
                            int sh, int sw, void* stream) {
  AB_CHECK(x && y && N >= 0 && H >= 0 && W >= 0 && C > 0 && ld_x >= C && ld_y >= C,
           "avgpool_fwd: bad arguments");
  AB_CHECK(sh >= 1 && sw >= 1, "avgpool_fwd: window (%d, %d) must be positive", sh, sw);
  const int64_t total = (int64_t)N * (H / sh) * (W / sw) * C;
  if (total == 0) return 0;
  avgpool_fwd_kernel<<<ab_grid(total, kT, 16), kT, 0, STREAM>>>(x, ld_x, y, ld_y, N, H, W, C, sh, sw);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_upsample_w2x_fwd(const float* x, int ld_x, float* y, int ld_y, int N, int w, int C,
                                 void* stream) {
  AB_CHECK(x && y && N >= 0 && w >= 0 && C > 0 && ld_x >= C && ld_y >= C,
           "upsample_w2x_fwd: bad arguments");
  const int64_t rows = (int64_t)N * 2 * w;
  if (rows == 0) return 0;
  upsample_w2x_fwd_kernel<<<ab_grid(rows * C, kT, 16), kT, 0, STREAM>>>(x, ld_x, y, ld_y, rows, C);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_upsample_w2x_bwd(const float* dy, int ld_dy, float* dx, int ld_dx, int N, int w, int C,
                                 void* stream) {
  AB_CHECK(dy && dx && N >= 0 && w >= 0 && C > 0 && ld_dy >= C && ld_dx >= C,
           "upsample_w2x_bwd: bad arguments");
  const int64_t rows = (int64_t)N * w;
  if (rows == 0) return 0;
  upsample_w2x_bwd_kernel<<<ab_grid(rows * C, kT, 16), kT, 0, STREAM>>>(dy, ld_dy, dx, ld_dx, rows, C);
  AB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
