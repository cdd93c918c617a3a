// gpr.cu — GP predictive mean without the cross-Gram:
//     y[i] = c + os * sum_j k(||(xq_i - x_j) * inv_ls||) * alpha_j
// for n_q query points against n training points of dimension d = 1..4 (the Reconstructor's
// predict over every pixel of an image: 512^2 queries x 26 k training pixels would be a 27 GB
// n_q x n matrix).  With d <= 4 there is no contraction worth a tensor core: per (i, j) pair the
// work is d subtractions, d scalings, d FMAs, one expf (plus one sqrtf for Matern), one fp32 -> fp64
// conversion and one fp64 FMA, so the kernel is SIMT and bound by the MUFU / conversion pipes.
//
// Tiling: a CTA owns kQB = kThreads * kQPT query points (kQPT per thread, held in registers, strided
// by kThreads so the loads coalesce) and walks the training points through shared memory, kTile
// at a time; every thread reads the same staged point (broadcast).  The j range is cut into fixed
// chunks of kChunk points.  Each thread sums one chunk into a fresh float64 partial (in increasing
// j) and the chunk partials are added in chunk order, starting from zero.  When the query blocks
// alone do not fill the GPU, CTAs along grid.y take runs of chunks and store each chunk partial in
// an ordered slot (common.cuh); the last CTA of a query block adds the slots in chunk order.  Both
// paths perform the same additions in the same order, so the result depends neither on the split
// nor on how the queries are batched, and a repeated call gives identical bits.
//
// The same file holds the training side of the exact GP: the float64 N x N Gram (+ noise on the
// diagonal) and its hyper-parameter adjoint, both from coordinate differences (no norm expansion,
// whose cancellation on pixel coordinates makes an fp32 Gram indefinite) and in float64 throughout,
// so the Cholesky sees a matrix that is symmetric positive definite to float64 rounding.
#include "common.cuh"

namespace {

constexpr int kThreads = 128;
constexpr int kQPT = 2;                    // query points per thread
constexpr int kQB = kThreads * kQPT;       // query points per CTA
constexpr int kTile = 256;                 // training points staged per pass
constexpr int kChunk = 1024;               // training points per float64 partial
constexpr int64_t kMaxSlotDoubles = 1ll << 24;   // ordered-slot workspace cap (128 MB)
constexpr int kMaxOrderedGroups = 4096;          // ticket groups of ab_ordered_ws

template <int D, int ACT>
__global__ void __launch_bounds__(kThreads, 8)
    gram_matvec_kernel(const float* __restrict__ xq, const float* __restrict__ x,
                       const float* __restrict__ inv_ls, const double* __restrict__ alpha,
                       double c, double os, int nq, int n, int nch, int cpc, Ordered ord,
                       double* __restrict__ y) {
  __shared__ float sx[kTile][D];
  __shared__ double sa[kTile];
  __shared__ unsigned s_last;
  const int tid = threadIdx.x;
  const int q0 = blockIdx.x * kQB;
  float il[D];
#pragma unroll
  for (int k = 0; k < D; ++k) il[k] = __ldg(inv_ls + k);
  float q[kQPT][D];
#pragma unroll
  for (int p = 0; p < kQPT; ++p) {
    const int i = q0 + p * kThreads + tid;
#pragma unroll
    for (int k = 0; k < D; ++k) q[p][k] = i < nq ? __ldg(xq + (int64_t)i * D + k) : 0.f;
  }
  double tot[kQPT];
#pragma unroll
  for (int p = 0; p < kQPT; ++p) tot[p] = 0.0;
  const bool split = gridDim.y > 1;
  const int ch0 = blockIdx.y * cpc;
  const int ch1 = min(ch0 + cpc, nch);
  for (int ch = ch0; ch < ch1; ++ch) {
    double acc[kQPT];
#pragma unroll
    for (int p = 0; p < kQPT; ++p) acc[p] = 0.0;
    const int j1 = min((ch + 1) * kChunk, n);
    for (int t0 = ch * kChunk; t0 < j1; t0 += kTile) {
      const int m = min(kTile, j1 - t0);
      __syncthreads();
      for (int e = tid; e < m * D; e += kThreads) sx[e / D][e % D] = __ldg(x + (int64_t)t0 * D + e);
      for (int e = tid; e < m; e += kThreads) sa[e] = __ldg(alpha + t0 + e);
      __syncthreads();
#pragma unroll 4
      for (int jj = 0; jj < m; ++jj) {
        float xs[D];
#pragma unroll
        for (int k = 0; k < D; ++k) xs[k] = sx[jj][k];
        const double a = sa[jj];
#pragma unroll
        for (int p = 0; p < kQPT; ++p) {
          float r2 = 0.f;
#pragma unroll
          for (int k = 0; k < D; ++k) {
            const float t = (q[p][k] - xs[k]) * il[k];
            r2 = fmaf(t, t, r2);
          }
          acc[p] = fma((double)act_f(r2, ACT, 1.f), a, acc[p]);
        }
      }
    }
    if (split) {
      double* slot = ordered_slot(ord, blockIdx.x, nch, ch, kQB);
#pragma unroll
      for (int p = 0; p < kQPT; ++p) slot[p * kThreads + tid] = acc[p];
    } else {
#pragma unroll
      for (int p = 0; p < kQPT; ++p) tot[p] += acc[p];
    }
  }
  if (!split) {
#pragma unroll
    for (int p = 0; p < kQPT; ++p) {
      const int i = q0 + p * kThreads + tid;
      if (i < nq) y[i] = c + os * tot[p];
    }
    return;
  }
  ordered_finish(ord, blockIdx.x, nch, kQB, tid, kThreads, gridDim.y, [] { __syncthreads(); },
                 [&](int e, double v) {
                   if (q0 + e < nq) y[q0 + e] = c + os * v;
                 },
                 &s_last);
}

template <int D>
int launch_d(int act, dim3 grid, cudaStream_t st, const float* xq, const float* x,
             const float* inv_ls, const double* alpha, double c, double os, int nq, int n, int nch,
             int cpc, const Ordered& ord, double* y) {
  if (act == AB_ACT_RBF)
    gram_matvec_kernel<D, AB_ACT_RBF><<<grid, kThreads, 0, st>>>(xq, x, inv_ls, alpha, c, os, nq, n,
                                                                  nch, cpc, ord, y);
  else
    gram_matvec_kernel<D, AB_ACT_MATERN25><<<grid, kThreads, 0, st>>>(xq, x, inv_ls, alpha, c, os,
                                                                       nq, n, nch, cpc, ord, y);
  AB_LAUNCH_CHECK();
  return 0;
}

}  // namespace

extern "C" int atomai_b200_gram_matvec(const float* xq, const float* x, const float* inv_ls,
                                       const double* alpha, double c, double outputscale, int nq,
                                       int n, int d, int kind, double* y, void* stream) {
  AB_CHECK(nq >= 0 && n >= 0 && d >= 1 && d <= 4, "gram_matvec: bad dims nq=%d n=%d d=%d (d in 1..4)",
           nq, n, d);
  AB_CHECK(kind == 0 || kind == 1, "gram_matvec: kind=%d", kind);
  AB_CHECK(y && (nq == 0 || xq) && inv_ls && (n == 0 || (x && alpha)), "gram_matvec: null pointer");
  if (nq == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int qblocks = (nq + kQB - 1) / kQB;
  const int nch = n > 0 ? (n + kChunk - 1) / kChunk : 1;
  AB_CHECK(qblocks <= 2147483647 / kQB, "gram_matvec: nq too large");
  // split the chunks over grid.y until about four resident waves of CTAs (8 per SM: <= 64
  // registers at 128 threads), as far as the chunks, the slot workspace and its ticket groups (one
  // per query block) allow; the sums do not depend on it
  const int64_t target = (int64_t)ab_num_sms() * 8 * 4;
  int64_t sy = (target + qblocks - 1) / qblocks;
  if (sy > nch) sy = nch;
  if ((int64_t)qblocks * nch * kQB > kMaxSlotDoubles || sy > 65535 || qblocks > kMaxOrderedGroups)
    sy = 1;
  const int cpc = (int)((nch + sy - 1) / sy);
  sy = (nch + cpc - 1) / cpc;
  Ordered ord{nullptr, nullptr};
  if (sy > 1 && ab_ordered_ws(st, (int64_t)qblocks * nch * kQB, qblocks, &ord)) return 1;
  const dim3 grid((unsigned)qblocks, (unsigned)sy);
  const int act = kind == 0 ? AB_ACT_RBF : AB_ACT_MATERN25;
  switch (d) {
    case 1: return launch_d<1>(act, grid, st, xq, x, inv_ls, alpha, c, outputscale, nq, n, nch, cpc, ord, y);
    case 2: return launch_d<2>(act, grid, st, xq, x, inv_ls, alpha, c, outputscale, nq, n, nch, cpc, ord, y);
    case 3: return launch_d<3>(act, grid, st, xq, x, inv_ls, alpha, c, outputscale, nq, n, nch, cpc, ord, y);
    default: return launch_d<4>(act, grid, st, xq, x, inv_ls, alpha, c, outputscale, nq, n, nch, cpc, ord, y);
  }
}

// ---------------------------------------------------------------- float64 training Gram + adjoint
namespace {

constexpr int kGT = 256;            // adjoint: 8 warps, one training row per warp

// k(r^2) / os and m = -2 dk/dr^2 / os in float64: RBF exp(-r^2/2) (m = k); Matern-2.5
// (1 + s + s^2/3) exp(-s), m = 5/3 (1 + s) exp(-s), s = sqrt(5 r^2)
template <int ACT>
__device__ __forceinline__ void k64(double r2, double& k, double& m) {
  if (ACT == AB_ACT_RBF) {
    k = exp(-0.5 * r2);
    m = k;
  } else {
    const double s = sqrt(5.0 * r2), e = exp(-s);
    k = (1.0 + s + (5.0 / 3.0) * r2) * e;
    m = (5.0 / 3.0) * (1.0 + s) * e;
  }
}

template <int D>
__device__ __forceinline__ double r2_diff(const double* __restrict__ x, int i, int j,
                                          const double* il, double* t) {
  double r2 = 0.0;
#pragma unroll
  for (int k = 0; k < D; ++k) {
    t[k] = (__ldg(x + (int64_t)i * D + k) - __ldg(x + (int64_t)j * D + k)) * il[k];
    r2 = fma(t[k], t[k], r2);
  }
  return r2;
}

// K[i][j] = os k(r_ij^2) + noise [i == j]; 32 x 8 threads per CTA, lanes along j (coalesced rows)
template <int D, int ACT>
__global__ void __launch_bounds__(256) gram_f64_kernel(const double* __restrict__ x,
                                                       const double* __restrict__ inv_ls, double os,
                                                       double noise, int n, double* __restrict__ K,
                                                       int64_t ldk) {
  const int j = blockIdx.x * 32 + threadIdx.x, i = blockIdx.y * 8 + threadIdx.y;
  if (i >= n || j >= n) return;
  double il[D], t[D], k, m;
#pragma unroll
  for (int q = 0; q < D; ++q) il[q] = __ldg(inv_ls + q);
  k64<ACT>(r2_diff<D>(x, i, j, il, t), k, m);
  K[(int64_t)i * ldk + j] = os * k + (i == j ? noise : 0.0);
}

// out[0..D-1] = sum_ij G_ij m_ij t_ijk^2, out[D] = sum_ij G_ij k_ij, out[D+1] = sum_i G_ii (unit
// outputscale).  Each lane sums its columns of one row in increasing j, the lanes by a fixed
// shuffle tree, the warps of a CTA in warp order, the CTAs in CTA order (ordered slots).
template <int D, int ACT>
__global__ void __launch_bounds__(kGT) gram_f64_adjoint_kernel(const double* __restrict__ x,
                                                               const double* __restrict__ inv_ls,
                                                               int n, const double* __restrict__ G,
                                                               int64_t ldg, Ordered ord,
                                                               double* __restrict__ out) {
  constexpr int NV = D + 2;
  __shared__ double part[kGT / 32][NV];
  __shared__ unsigned s_last;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * (kGT / 32) + warp;
  double il[D], acc[NV];
#pragma unroll
  for (int q = 0; q < D; ++q) il[q] = __ldg(inv_ls + q);
#pragma unroll
  for (int v = 0; v < NV; ++v) acc[v] = 0.0;
  if (i < n) {
    for (int j = lane; j < n; j += 32) {
      double t[D], k, m;
      k64<ACT>(r2_diff<D>(x, i, j, il, t), k, m);
      const double g = __ldg(G + (int64_t)i * ldg + j);
#pragma unroll
      for (int q = 0; q < D; ++q) acc[q] = fma(g * m, t[q] * t[q], acc[q]);
      acc[D] = fma(g, k, acc[D]);
      if (j == i) acc[D + 1] += g;
    }
  }
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    const double s = warp_sum_d(acc[v]);
    if (lane == 0) part[warp][v] = s;
  }
  __syncthreads();
  if (threadIdx.x < NV) {
    double s = 0.0;
    for (int w = 0; w < kGT / 32; ++w) s += part[w][threadIdx.x];
    ordered_slot(ord, 0, gridDim.x, blockIdx.x, NV)[threadIdx.x] = s;
  }
  ordered_finish(ord, 0, gridDim.x, NV, threadIdx.x, kGT, gridDim.x, [] { __syncthreads(); },
                 [&](int v, double s) { out[v] = s; }, &s_last);
}

template <int D>
int gram_f64_d(int act, const double* x, const double* inv_ls, double os, double noise, int n,
               double* K, int64_t ldk, cudaStream_t st) {
  const dim3 grid((n + 31) / 32, (n + 7) / 8), block(32, 8);
  if (act == AB_ACT_RBF)
    gram_f64_kernel<D, AB_ACT_RBF><<<grid, block, 0, st>>>(x, inv_ls, os, noise, n, K, ldk);
  else
    gram_f64_kernel<D, AB_ACT_MATERN25><<<grid, block, 0, st>>>(x, inv_ls, os, noise, n, K, ldk);
  AB_LAUNCH_CHECK();
  return 0;
}

template <int D>
int gram_f64_adjoint_d(int act, const double* x, const double* inv_ls, int n, const double* G,
                       int64_t ldg, double* out, cudaStream_t st) {
  const int nb = (n + kGT / 32 - 1) / (kGT / 32);
  Ordered ord;
  if (ab_ordered_ws(st, (int64_t)nb * (D + 2), 1, &ord)) return 1;
  if (act == AB_ACT_RBF)
    gram_f64_adjoint_kernel<D, AB_ACT_RBF><<<nb, kGT, 0, st>>>(x, inv_ls, n, G, ldg, ord, out);
  else
    gram_f64_adjoint_kernel<D, AB_ACT_MATERN25><<<nb, kGT, 0, st>>>(x, inv_ls, n, G, ldg, ord, out);
  AB_LAUNCH_CHECK();
  return 0;
}

}  // namespace

extern "C" int atomai_b200_gram_f64(const double* x, const double* inv_ls, double outputscale,
                                    double noise, int n, int d, int kind, double* K, int64_t ldk,
                                    void* stream) {
  AB_CHECK(n >= 0 && d >= 1 && d <= 4 && ldk >= n, "gram_f64: bad dims n=%d d=%d (d in 1..4)", n, d);
  AB_CHECK(kind == 0 || kind == 1, "gram_f64: kind=%d", kind);
  AB_CHECK(n == 0 || (x && inv_ls && K), "gram_f64: null pointer");
  AB_CHECK((n + 7) / 8 <= 65535, "gram_f64: n=%d too large", n);
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int act = kind == 0 ? AB_ACT_RBF : AB_ACT_MATERN25;
  switch (d) {
    case 1: return gram_f64_d<1>(act, x, inv_ls, outputscale, noise, n, K, ldk, st);
    case 2: return gram_f64_d<2>(act, x, inv_ls, outputscale, noise, n, K, ldk, st);
    case 3: return gram_f64_d<3>(act, x, inv_ls, outputscale, noise, n, K, ldk, st);
    default: return gram_f64_d<4>(act, x, inv_ls, outputscale, noise, n, K, ldk, st);
  }
}

extern "C" int atomai_b200_gram_f64_adjoint(const double* x, const double* inv_ls, int n, int d,
                                            int kind, const double* G, int64_t ldg, double* out,
                                            void* stream) {
  AB_CHECK(n >= 1 && d >= 1 && d <= 4 && ldg >= n, "gram_f64_adjoint: bad dims n=%d d=%d", n, d);
  AB_CHECK(kind == 0 || kind == 1, "gram_f64_adjoint: kind=%d", kind);
  AB_CHECK(x && inv_ls && G && out, "gram_f64_adjoint: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int act = kind == 0 ? AB_ACT_RBF : AB_ACT_MATERN25;
  switch (d) {
    case 1: return gram_f64_adjoint_d<1>(act, x, inv_ls, n, G, ldg, out, st);
    case 2: return gram_f64_adjoint_d<2>(act, x, inv_ls, n, G, ldg, out, st);
    case 3: return gram_f64_adjoint_d<3>(act, x, inv_ls, n, G, ldg, out, st);
    default: return gram_f64_adjoint_d<4>(act, x, inv_ls, n, G, ldg, out, st);
  }
}
