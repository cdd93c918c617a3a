// gram.cu — dense deep-kernel Gram matrix K[i][j] = os * k(|| (x1_i - x2_j) * inv_ls ||).
// The squared distance is ONE contraction over augmented operands,
//     a' = [a/l, ||a/l||^2, 1, 0..]   b' = [-2 b/l, 1, ||b/l||^2, 0..]   =>  a'.b' = ||a/l - b/l||^2
// (row norms by warp shuffles while scaling), so the -2ab^T term, both norms and the
// exponentiation ride on the tensor-core convolution kernel as a 1x1 convolution with an RBF /
// Matern "activation" in its register epilogue: x1 rows = pixels of a (1, n1/8, 8, K') image, column
// blocks of <= 128 rows of x2 = output channels.  The n1 x n2 matrix is written exactly once.
// AB_MATH_FP32 (and the < 8-row / < 16-column remainders of the tensor path) use the exact FFMA
// tile kernel below.
// RBF / Matern-2.5 / outputscale follow gpytorch's public kernel definitions as configured at
// atomai/nets/gp.py:41-46 and :100-111 (gpytorch itself is not vendored by the reference).
#include <cstdlib>
#include "common.cuh"


// implemented in conv_tc.cu
int64_t ab_pack_weights_tc_elems(int Cout, int Cin, int th, int tw, int mode, int x3);
int ab_pack_weights_tc(const float* w, int Cout, int Cin, int th, int tw, int mode, int x3,
                       float* out, cudaStream_t stream);
int ab_conv_tc_fwd(const ab_conv_t* d, const float* wblob, const float* bias, float* y, int ld_y,
                   double* stats, cudaStream_t stream);

namespace {

constexpr int TM = 64, TN = 64, TK = 16, GT = 256;
constexpr int kColBlock = 128;      // max output channels (rows of K) per tensor-core launch

// one warp per row: out[row] = [x*inv_ls * fac, (side 0: |.|^2, 1) | (side 1: 1, |.|^2), 0-pad]
__global__ void augment_kernel(const float* __restrict__ x, const float* __restrict__ inv_ls,
                               int n, int d, int Kp, int side, float* __restrict__ out) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= n) return;
  float acc = 0.f;
  const float fac = side ? -2.f : 1.f;
  for (int k = lane; k < Kp; k += 32) {
    float v = 0.f;
    if (k < d) {
      v = x[(int64_t)row * d + k] * inv_ls[k];
      acc = fmaf(v, v, acc);
      v *= fac;
    }
    out[(int64_t)row * Kp + k] = v;
  }
  acc = warp_sum(acc);
  if (lane == 0) {
    out[(int64_t)row * Kp + d + (side ? 1 : 0)] = acc;
    out[(int64_t)row * Kp + d + (side ? 0 : 1)] = 1.f;
  }
}

__global__ void __launch_bounds__(GT)
    gram_kernel(const float* __restrict__ a, const float* __restrict__ b, int n1, int n2, int d,
                float os, int kind, float* __restrict__ K, int64_t ldk) {
  __shared__ float sA[TK][TM + 4];
  __shared__ float sB[TK][TN + 4];
  const int m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
  const int tid = threadIdx.x;
  const int tm = (tid >> 4) * 4, tn = (tid & 15) * 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < d; k0 += TK) {
    __syncthreads();
    for (int i = tid; i < TM * TK; i += GT) {
      const int k = i % TK, m = i / TK;
      sA[k][m] = (m0 + m < n1 && k0 + k < d) ? __ldg(a + (int64_t)(m0 + m) * d + k0 + k) : 0.f;
      sB[k][m] = (n0 + m < n2 && k0 + k < d) ? __ldg(b + (int64_t)(n0 + m) * d + k0 + k) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < TK; ++k) {
      const float4 a4 = *reinterpret_cast<const float4*>(&sA[k][tm]);
      const float4 b4 = *reinterpret_cast<const float4*>(&sB[k][tn]);
      const float av[4] = {a4.x, a4.y, a4.z, a4.w};
      const float bv[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + tm + i;
    if (m >= n1) continue;
    float out[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) out[j] = act_f(acc[i][j], kind == 0 ? AB_ACT_RBF : AB_ACT_MATERN25, os);
    float* o = K + (int64_t)m * ldk + n0 + tn;
    if (n0 + tn + 3 < n2 && ((ldk & 3) == 0) && (((uintptr_t)o & 15) == 0)) {
      *reinterpret_cast<float4*>(o) = make_float4(out[0], out[1], out[2], out[3]);
    } else {
      for (int j = 0; j < 4; ++j)
        if (n0 + tn + j < n2) o[j] = out[j];
    }
  }
}

int gram_simt(const float* a, const float* b, int n1, int n2, int Kp, float os, int kind, float* K,
              int64_t ldk, cudaStream_t st) {
  if (n1 <= 0 || n2 <= 0) return 0;
  dim3 grid((n2 + TN - 1) / TN, (n1 + TM - 1) / TM);
  AB_CHECK(grid.y <= 65535, "gram: n1 too large for one launch");
  gram_kernel<<<grid, GT, 0, st>>>(a, b, n1, n2, Kp, os, kind, K, ldk);
  AB_LAUNCH_CHECK();
  return 0;
}

inline int64_t align256(int64_t v) { return (v + 255) & ~(int64_t)255; }
// K' = d + 2 padded to the conv kernel's k-chunk (32 channels once there is more than one chunk)
inline int aug_k(int d) { return d + 2 <= 8 ? 8 : (d + 2 <= 16 ? 16 : (d + 2 + 31) & ~31); }

}  // namespace

extern "C" int64_t atomai_b200_gram_workspace_bytes(int n1, int n2, int d) {
  if (n1 < 0 || n2 < 0 || d <= 0) return -1;
  const int Kp = aug_k(d);
  return align256((int64_t)n1 * Kp * 4) + align256((int64_t)n2 * Kp * 4) +
         align256(ab_pack_weights_tc_elems(kColBlock, Kp, 1, 1, AB_WMODE_FWD, 1) * 4) + 256;
}

extern "C" int atomai_b200_gram(const float* x1, const float* x2, const float* inv_ls,
                                float outputscale, int n1, int n2, int d, int kind, int math,
                                float* K, int64_t ldk, void* workspace, int64_t workspace_bytes,
                                void* stream) {
  AB_CHECK(x1 && x2 && inv_ls && K && workspace, "gram: null pointer");
  AB_CHECK(n1 >= 0 && n2 >= 0 && d > 0 && ldk >= n2, "gram: bad dims n1=%d n2=%d d=%d", n1, n2, d);
  AB_CHECK(kind == 0 || kind == 1, "gram: kind=%d", kind);
  AB_CHECK(math == AB_MATH_FP32 || math == AB_MATH_TF32 || math == AB_MATH_TF32X3, "gram: math=%d",
           math);
  AB_CHECK(workspace_bytes >= atomai_b200_gram_workspace_bytes(n1, n2, d) &&
               ((uintptr_t)workspace & 255) == 0,
           "gram: workspace too small or unaligned (need %lld bytes, 256 B aligned)",
           (long long)atomai_b200_gram_workspace_bytes(n1, n2, d));
  if (n1 == 0 || n2 == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int Kp = aug_k(d);
  char* ws = static_cast<char*>(workspace);
  float* a = reinterpret_cast<float*>(ws);
  float* b = reinterpret_cast<float*>(ws + align256((int64_t)n1 * Kp * 4));
  float* blob = reinterpret_cast<float*>(ws + align256((int64_t)n1 * Kp * 4) +
                                         align256((int64_t)n2 * Kp * 4));
  augment_kernel<<<(n1 + 7) / 8, 256, 0, st>>>(x1, inv_ls, n1, d, Kp, 0, a);
  AB_LAUNCH_CHECK();
  augment_kernel<<<(n2 + 7) / 8, 256, 0, st>>>(x2, inv_ls, n2, d, Kp, 1, b);
  AB_LAUNCH_CHECK();
  const int act = kind == 0 ? AB_ACT_RBF : AB_ACT_MATERN25;
  int n1m = 0, n2m = 0;
  if (math != AB_MATH_FP32 && ldk < (1ll << 31)) {
    n1m = n1 & ~15;
    n2m = n2 & ~7;
  }
  if (n1m > 0 && n2m > 0) {
    // tensor path: the rows of x2 are the pixels of a (1, n2m/8, 8, K') image, row blocks of <= 128
    // rows of x1 the output channels, stored "NCHW" with the channel pitch = ldk: lane l of an
    // epilogue warp holds K[r][c + l], so every store instruction writes 128 contiguous bytes of a
    // row of K (the NHWC form would write 16 B to 32 different rows per instruction)
    ab_conv_t cd;
    memset(&cd, 0, sizeof(cd));
    cd.N = 1; cd.H = n2m / 8; cd.W = 8;
    cd.ks_h = cd.ks_w = 1; cd.dil = 1; cd.nsrc = 1;
    cd.src[0].ptr = b; cd.src[0].C = Kp; cd.src[0].ld = Kp;
    cd.lrelu = outputscale; cd.math = math; cd.act = act; cd.out_nchw = 1;
    const int x3 = math == AB_MATH_TF32X3;
    // rows of K per launch: as wide as the consumer's accumulator registers allow — wide N amortises
    // the A-operand reads and the per-tile handshakes
    int blk = kColBlock;
    if (const char* e = getenv("ATOMAI_B200_GRAM_BLOCK")) blk = atoi(e);
    if (blk < 16 || blk > kColBlock || blk % 16 != 0) blk = kColBlock;
    for (int r0 = 0; r0 < n1m; r0 += blk) {
      const int rb = (n1m - r0) < blk ? (n1m - r0) : blk;
      cd.Cout = rb;
      if (ab_pack_weights_tc(a + (int64_t)r0 * Kp, rb, Kp, 1, 1, AB_WMODE_FWD, x3, blob, st)) return 1;
      if (ab_conv_tc_fwd(&cd, blob, nullptr, K + (int64_t)r0 * ldk, -(int)ldk, nullptr, st)) return 1;
    }
  }
  // exact FFMA tiles: everything (fp32 math) or the right / bottom remainders of the tensor path
  if (gram_simt(a, b + (int64_t)n2m * Kp, n1m, n2 - n2m, Kp, outputscale, kind, K + n2m, ldk, st))
    return 1;
  if (gram_simt(a + (int64_t)n1m * Kp, b, n1 - n1m, n2, Kp, outputscale, kind,
                K + (int64_t)n1m * ldk, ldk, st))
    return 1;
  return 0;
}
