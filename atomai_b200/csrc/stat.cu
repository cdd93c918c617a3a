// stat.cu — k-means (k-means++ seeding, Lloyd) and diagonal / spherical Gaussian-mixture EM over a
// stack of flattened sub-images X (N x d, fp32, row-major: the (N, r, r, c) gather output).
//
// X is never copied: every kernel reads it through `mu`, the column mean, subtracted on load
// (sklearn centres X before k-means; the GMM scores are shift invariant, and centring keeps the
// ||x||^2 - 2 x.c + ||c||^2 expansion away from cancellation).
//
//   estep   one pass over X: per row and component s_k = sum_j A_kj x_j + B_kj x_j^2 (fp32, fixed
//           j order), then per row either the GMM log-sum-exp (responsibilities, argmax, log_prob_norm)
//           or the k-means argmin (label, squared distance), or the k-means++ candidate potentials.
//   accum   one pass over X: per component sum_n r_nk, sum_n r_nk x_n, sum_n r_nk x_n^2 with r either
//           soft responsibilities, hard labels, or all ones (column mean / variance).
//   gmm_params / kmeans_centres   O(K d) finalisation of the M-step / the Lloyd update.
//
// Determinism: row sums never use floating-point atomics.  `accum` sums fixed chunks of kRowChunk
// rows in fp32 in row order and the chunk partials in chunk order in float64 through the ordered
// slots of common.cuh; `estep` sums its per-row scalars per CTA in row order and the CTAs in CTA
// order the same way.  The chunking depends on N only, so a repeated fit gives identical bits on any
// GPU (permuting the rows reorders the fp32 sums and so can change the last bits).  The only atomics
// add integer counts (label changes), which are exact.
//
// Arithmetic (`math`, the library's AB_MATH_*): the two contractions, N x 2d . 2d x K for the
// E-step and K x N . N x 2d for the M-step, run on wgmma (estep_tc_kernel / accum_tc_kernel, K
// padded to the MMA N of 16, 32 or 64) under AB_MATH_TF32X3 (split operands, fp32-level accuracy)
// and AB_MATH_TF32, and as exact fp32 FFMA on the CUDA cores (estep_kernel / accum_kernel) under
// AB_MATH_FP32.  Either way: fp32 dot products over d and fp32 sums over a chunk's rows (as
// sklearn's float32 BLAS calls), float64 where chunks are combined.
#include <float.h>
#include <math.h>
#include "common.cuh"
#include "wgmma.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kRows = 64;          // estep: rows per CTA
constexpr int kCols = 32;          // column tile of both passes
constexpr int kAccRows = 32;       // accum: rows staged per pass
constexpr int kRowChunk = 4096;    // accum: rows per fp32 partial (fixed: the sums depend on it)
constexpr int kSumChunk = 1024;    // k-means++: rows per D^2 prefix chunk
constexpr int kMaxK = 64;

enum { kModeGMM = 0, kModeKMeans = 1, kModeKPP = 2 };

// first index of the smallest (lt = true) / largest value over the warp; lanes hold (v, i)
__device__ __forceinline__ void warp_arg(float& v, int& i, bool lt) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    const bool better = lt ? (ov < v) : (ov > v);
    if (better || (ov == v && oi < i)) {
      v = ov;
      i = oi;
    }
  }
}

// Per-row finish of an E-step tile of kRows rows: sc (row stride ld) holds the scores s_nk, rq the
// squared row norms.  One warp per row, lanes over components; the CTA's per-row values are summed
// in row order into its ordered slot.  Called by all NT threads of the CTA.
template <int MODE, int NT>
__device__ __forceinline__ void estep_rows(float* sc, int ld, const float* rq, int64_t r0, int N,
                                           int K, const float* __restrict__ cst,
                                           const float* __restrict__ closest, float* resp,
                                           int* labels, float* rowval, float* D, const Ordered& ord,
                                           double* out, double* changes, int* s_changed,
                                           unsigned* s_last) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // one warp per row: lanes over components
  int changed = 0;
  for (int rr = warp; rr < kRows; rr += NT / 32) {
    const int64_t n = r0 + rr;
    const bool live = n < N;
    if (MODE == kModeGMM) {
      float v[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int k = lane + 32 * h;
        v[h] = k < K ? sc[rr * ld + k] + __ldg(cst + k) : -INFINITY;
      }
      float bv = v[0] >= v[1] ? v[0] : v[1];
      int bi = v[0] >= v[1] ? lane : lane + 32;
      warp_arg(bv, bi, false);
      float s = 0.f;
#pragma unroll
      for (int h = 0; h < 2; ++h) s += lane + 32 * h < K ? expf(v[h] - bv) : 0.f;
      const float lse = bv + logf(warp_sum(s));
      if (live) {
        if (resp) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int k = lane + 32 * h;
            if (k < K) resp[n * K + k] = expf(v[h] - lse);
          }
        }
        if (labels && lane == 0) labels[n] = bi;
      }
      if (lane == 0) sc[rr * ld] = live ? lse : 0.f;
    } else if (MODE == kModeKMeans) {
      float v[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int k = lane + 32 * h;
        v[h] = k < K ? fmaxf(rq[rr] + sc[rr * ld + k] + __ldg(cst + k), 0.f) : INFINITY;
      }
      float bv = v[0] <= v[1] ? v[0] : v[1];
      int bi = v[0] <= v[1] ? lane : lane + 32;
      warp_arg(bv, bi, true);
      if (live && lane == 0) {
        if (labels[n] != bi) ++changed;
        labels[n] = bi;
        if (rowval) rowval[n] = bv;
      }
      __syncwarp();
      if (lane == 0) sc[rr * ld] = live ? bv : 0.f;
    } else {
      float v[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int k = lane + 32 * h;
        v[h] = 0.f;
        if (k < K && live) {
          const float dist = fmaxf(rq[rr] + sc[rr * ld + k] + __ldg(cst + k), 0.f);
          D[n * K + k] = dist;
          v[h] = fminf(__ldg(closest + n), dist);
        }
      }
      __syncwarp();
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (lane + 32 * h < K) sc[rr * ld + lane + 32 * h] = v[h];
    }
  }
  if (MODE == kModeKMeans && changes) {
    if (changed) atomicAdd(s_changed, changed);
  }
  __syncthreads();
  const int nv = MODE == kModeKPP ? K : 1;
  if (tid < nv) {
    double s = 0.0;
    for (int rr = 0; rr < kRows; ++rr) s += (double)sc[rr * ld + tid];
    ordered_slot(ord, 0, gridDim.x, blockIdx.x, nv)[tid] = s;
  }
  if (MODE == kModeKMeans && changes && tid == 0 && *s_changed) atomicAdd(changes, (double)*s_changed);
  ordered_finish(ord, 0, gridDim.x, nv, tid, NT, gridDim.x, [] { __syncthreads(); },
                 [&](int i, double s) { out[i] = s; }, s_last);
}

// KPT components per thread: 16 component groups x 16 row groups, 4 rows per thread
template <int KPT, int MODE>
__global__ void __launch_bounds__(kThreads)
    estep_kernel(const float* __restrict__ X, const float* __restrict__ mu, int N, int d, int K,
                 const float* __restrict__ A, const float* __restrict__ B,
                 const float* __restrict__ cst, const float* __restrict__ closest,
                 float* __restrict__ resp, int* __restrict__ labels, float* __restrict__ rowval,
                 float* __restrict__ D, Ordered ord, double* __restrict__ out,
                 double* __restrict__ changes) {
  constexpr int KP = 16 * KPT;
  __shared__ float xs[kRows][kCols + 1];
  __shared__ float as[KP][kCols + 1];
  __shared__ float bs[MODE == kModeGMM ? KP : 1][kCols + 1];
  __shared__ float sc[kRows][KP + 1];
  __shared__ float rq[kRows];
  __shared__ int s_changed;
  __shared__ unsigned s_last;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rg = tid & 15, kg = tid >> 4;
  const int64_t r0 = (int64_t)blockIdx.x * kRows;
  if (tid == 0) s_changed = 0;

  float acc[4][KPT], sq[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    sq[i] = 0.f;
#pragma unroll
    for (int q = 0; q < KPT; ++q) acc[i][q] = 0.f;
  }
  for (int j0 = 0; j0 < d; j0 += kCols) {
    __syncthreads();
#pragma unroll
    for (int e = tid; e < kRows * kCols; e += kThreads) {
      const int rr = e / kCols, cc = e % kCols, j = j0 + cc;
      const int64_t row = r0 + rr;
      xs[rr][cc] = (row < N && j < d) ? __ldg(X + row * d + j) - __ldg(mu + j) : 0.f;
    }
    for (int e = tid; e < KP * kCols; e += kThreads) {
      const int k = e / kCols, cc = e % kCols, j = j0 + cc;
      const bool ok = k < K && j < d;
      as[k][cc] = ok ? __ldg(A + (int64_t)k * d + j) : 0.f;
      if (MODE == kModeGMM) bs[k][cc] = ok ? __ldg(B + (int64_t)k * d + j) : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int jj = 0; jj < kCols; ++jj) {
      float a[KPT], b[KPT];
#pragma unroll
      for (int q = 0; q < KPT; ++q) {
        a[q] = as[kg + 16 * q][jj];
        b[q] = MODE == kModeGMM ? bs[kg + 16 * q][jj] : 0.f;
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float x = xs[rg + 16 * i][jj], x2 = x * x;
        if (MODE != kModeGMM) sq[i] = fmaf(x, x, sq[i]);
#pragma unroll
        for (int q = 0; q < KPT; ++q) {
          acc[i][q] = fmaf(a[q], x, acc[i][q]);
          if (MODE == kModeGMM) acc[i][q] = fmaf(b[q], x2, acc[i][q]);
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int q = 0; q < KPT; ++q) sc[rg + 16 * i][kg + 16 * q] = acc[i][q];
    if (kg == 0) rq[rg + 16 * i] = sq[i];
  }
  __syncthreads();

  estep_rows<MODE, kThreads>(&sc[0][0], KP + 1, rq, r0, N, K, cst, closest, resp, labels, rowval,
                             D, ord, out, changes, &s_changed, &s_last);
}

// grid (column blocks, row chunks); warp w owns components w, w + 8, ...; lane = column
template <int KW>
__global__ void __launch_bounds__(kThreads)
    accum_kernel(const float* __restrict__ X, const float* __restrict__ mu, int N, int d, int K,
                 const float* __restrict__ resp, const int* __restrict__ labels, int want_sq,
                 Ordered ord, double* __restrict__ sx, double* __restrict__ sxx,
                 double* __restrict__ nk) {
  constexpr int KP = 8 * KW;
  constexpr int NV = 2 * kCols + 1;  // per component: kCols sums, kCols square sums, the count
  __shared__ float xs[kAccRows][kCols + 1];
  __shared__ float rs[kAccRows][KP];
  __shared__ unsigned s_last;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int j0 = blockIdx.x * kCols;
  const int64_t c0 = (int64_t)blockIdx.y * kRowChunk;
  const int64_t c1 = min((int64_t)N, c0 + kRowChunk);
  float s[KW], q[KW], c[KW];
#pragma unroll
  for (int i = 0; i < KW; ++i) s[i] = q[i] = c[i] = 0.f;
  for (int64_t r0 = c0; r0 < c1; r0 += kAccRows) {
    __syncthreads();
#pragma unroll
    for (int e = tid; e < kAccRows * kCols; e += kThreads) {
      const int rr = e / kCols, cc = e % kCols, j = j0 + cc;
      const int64_t row = r0 + rr;
      float v = 0.f;
      if (row < c1 && j < d) {
        v = __ldg(X + row * d + j);
        if (mu) v -= __ldg(mu + j);
      }
      xs[rr][cc] = v;
    }
    for (int e = tid; e < kAccRows * KP; e += kThreads) {
      const int rr = e / KP, k = e % KP;
      const int64_t row = r0 + rr;
      float v = 0.f;
      if (row < c1 && k < K) {
        if (resp) v = __ldg(resp + row * K + k);
        else if (labels) v = __ldg(labels + row) == k ? 1.f : 0.f;
        else v = k == 0 ? 1.f : 0.f;
      }
      rs[rr][k] = v;
    }
    __syncthreads();
#pragma unroll 4
    for (int rr = 0; rr < kAccRows; ++rr) {
      const float x = xs[rr][lane], x2 = x * x;
#pragma unroll
      for (int i = 0; i < KW; ++i) {
        const float r = rs[rr][warp + 8 * i];
        s[i] = fmaf(r, x, s[i]);
        if (want_sq) q[i] = fmaf(r, x2, q[i]);
        c[i] += r;
      }
    }
  }
  double* slot = ordered_slot(ord, blockIdx.x, gridDim.y, blockIdx.y, K * NV);
#pragma unroll
  for (int i = 0; i < KW; ++i) {
    const int k = warp + 8 * i;
    if (k < K) {
      slot[k * NV + lane] = s[i];
      slot[k * NV + kCols + lane] = q[i];
      if (lane == 0) slot[k * NV + 2 * kCols] = c[i];
    }
  }
  ordered_finish(ord, blockIdx.x, gridDim.y, K * NV, tid, kThreads, gridDim.y,
                 [] { __syncthreads(); },
                 [&](int i, double v) {
                   const int k = i / NV, e = i % NV;
                   if (e < kCols) {
                     if (j0 + e < d) sx[(int64_t)k * d + j0 + e] = v;
                   } else if (e < 2 * kCols) {
                     if (sxx && j0 + e - kCols < d) sxx[(int64_t)k * d + j0 + e - kCols] = v;
                   } else if (nk && blockIdx.x == 0) {
                     nk[k] = v;
                   }
                 },
                 &s_last);
}

// ---------------------------------------------------------------- tensor-core (wgmma) passes
// One warpgroup per CTA, operands staged K-major without swizzle (core matrices of 8 rows x 16 B,
// kmaj_off) and read by m64nNk8 TF32 MMAs, fp32 accumulation.  Every value is stored RN-rounded to
// TF32 (hi) and, under tf32x3, also its exact remainder rounded again (lo); per k-step the products
// (hi, hi), (hi, lo) and (lo, hi) are issued.  The x^2 operand is formed by the loader.  Each stage
// is loaded into registers while the previous stage's MMAs run.
constexpr int kTcThreads = 128;
constexpr int kTcK = 16;                          // k extent of a stage (features / rows)
constexpr int kTcSbo = (kTcK / 4) * 128 + 32;     // bytes per 8-row group (+32: bank spread)

__device__ __forceinline__ uint32_t tf32b(float x) { return __float_as_uint(x) + 0x1000u; }
__device__ __forceinline__ float tf32_lo(float x) { return x - __uint_as_float(tf32b(x) & 0xFFFFE000u); }
__device__ __forceinline__ uint32_t kmaj_off(int r, int k) {
  return (uint32_t)((r >> 3) * kTcSbo + (k >> 2) * 128 + (r & 7) * 16 + (k & 3) * 4);
}
// hi part at base, lo part at base + lo_off (x3 only)
__device__ __forceinline__ void put_split(uint32_t base, uint32_t lo_off, int r, int k, float v,
                                          bool x3) {
  const uint32_t a = base + kmaj_off(r, k);
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(tf32b(v)) : "memory");
  if (x3) asm volatile("st.shared.b32 [%0], %1;" ::"r"(a + lo_off), "r"(tf32b(tf32_lo(v))) : "memory");
}
template <int NB, bool X3>
__device__ __forceinline__ void mma_split(float (&acc)[NB / 2], uint32_t a, uint32_t a_lo, uint32_t b,
                                          uint32_t b_lo) {
  const uint64_t ah = wgmma_desc(a, 128, kTcSbo), bh = wgmma_desc(b, 128, kTcSbo);
  Wgmma<NB>::tf32(acc, ah, bh, 1u);
  if (X3) {
    Wgmma<NB>::tf32(acc, ah, wgmma_desc(b + b_lo, 128, kTcSbo), 1u);
    Wgmma<NB>::tf32(acc, wgmma_desc(a + a_lo, 128, kTcSbo), bh, 1u);
  }
}

// E-step: M = 64 rows, N = NB >= K components (padded with zero operands), k = features.
// Loader: thread t owns row t / 2, features 8 (t % 2) .. +8 of the stage; component operands
// e = t + 128 i -> (component e / 16, feature e % 16).
template <int NB, int MODE, bool X3>
__global__ void __launch_bounds__(kTcThreads)
    estep_tc_kernel(const float* __restrict__ X, const float* __restrict__ mu, int N, int d, int K,
                    const float* __restrict__ A, const float* __restrict__ B,
                    const float* __restrict__ cst, const float* __restrict__ closest,
                    float* __restrict__ resp, int* __restrict__ labels, float* __restrict__ rowval,
                    float* __restrict__ D, Ordered ord, double* __restrict__ out,
                    double* __restrict__ changes) {
  constexpr bool GMM = MODE == kModeGMM;
  constexpr int XB = 8 * kTcSbo, CB = (NB / 8) * kTcSbo;
  constexpr int NX = GMM ? 2 : 1;                          // x and x^2 operands
  constexpr int STAGE = 2 * NX * (XB + CB);                // [x|x2][hi|lo] then [A|B][hi|lo]
  constexpr int SCB = kRows * (NB + 1) * 4;
  constexpr int CPT = NB * kTcK / kTcThreads;              // component operand values per thread
  __shared__ __align__(128) unsigned char smem[STAGE > SCB ? STAGE : SCB];
  __shared__ float rq[kRows];
  __shared__ int s_changed;
  __shared__ unsigned s_last;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t r0 = (int64_t)blockIdx.x * kRows;
  constexpr bool use_lo = X3;
  if (tid == 0) s_changed = 0;
  const uint32_t sb = smem_u32(smem);
  const uint32_t sx = sb, sx2 = sb + 2 * XB, sa = sb + 2 * NX * XB, sbb = sa + 2 * CB;
  const int lr = tid >> 1, lc = (tid & 1) * 8;
  const int64_t row = r0 + lr;
  float acc[NB / 2];
#pragma unroll
  for (int i = 0; i < NB / 2; ++i) acc[i] = 0.f;
  float sq = 0.f;
  float xv[8], av[CPT], bv[CPT];
  auto load = [&](int j0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int j = j0 + lc + i;
      xv[i] = (row < N && j < d) ? __ldg(X + row * d + j) - __ldg(mu + j) : 0.f;
    }
#pragma unroll
    for (int i = 0; i < CPT; ++i) {
      const int e = tid + kTcThreads * i, k = e / kTcK, j = j0 + e % kTcK;
      const bool ok = k < K && j < d;
      av[i] = ok ? __ldg(A + (int64_t)k * d + j) : 0.f;
      bv[i] = (GMM && ok) ? __ldg(B + (int64_t)k * d + j) : 0.f;
    }
  };
  load(0);
  for (int j0 = 0; j0 < d; j0 += kTcK) {
    __syncthreads();                                       // previous stage's MMAs have retired
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float x = xv[i], x2 = x * x;
      if (!GMM) sq = fmaf(x, x, sq);
      put_split(sx, XB, lr, lc + i, x, use_lo);
      if (GMM) put_split(sx2, XB, lr, lc + i, x2, use_lo);
    }
#pragma unroll
    for (int i = 0; i < CPT; ++i) {
      const int e = tid + kTcThreads * i;
      put_split(sa, CB, e / kTcK, e % kTcK, av[i], use_lo);
      if (GMM) put_split(sbb, CB, e / kTcK, e % kTcK, bv[i], use_lo);
    }
    fence_proxy_async_smem();
    __syncthreads();
    wgmma_fence();
    wgmma_fence_regs(acc);
#pragma unroll
    for (int ks = 0; ks < kTcK / 8; ++ks) {
      mma_split<NB, X3>(acc, sx + ks * 256, XB, sa + ks * 256, CB);
      if (GMM) mma_split<NB, X3>(acc, sx2 + ks * 256, XB, sbb + ks * 256, CB);
    }
    wgmma_commit();
    if (j0 + kTcK < d) load(j0 + kTcK);
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
  }
  // rows' squared norms: the two loader threads of a row add their halves in a fixed order
  const float other = __shfl_xor_sync(0xffffffffu, sq, 1);
  __syncthreads();
  float* sc = reinterpret_cast<float*>(smem);
  if ((tid & 1) == 0) rq[lr] = sq + other;
#pragma unroll
  for (int j = 0; j < NB / 8; ++j) {
    const int r = 16 * warp + (lane >> 2), c = 8 * j + 2 * (lane & 3);
    sc[r * (NB + 1) + c] = acc[4 * j];
    sc[r * (NB + 1) + c + 1] = acc[4 * j + 1];
    sc[(r + 8) * (NB + 1) + c] = acc[4 * j + 2];
    sc[(r + 8) * (NB + 1) + c + 1] = acc[4 * j + 3];
  }
  __syncthreads();
  estep_rows<MODE, kTcThreads>(sc, NB + 1, rq, r0, N, K, cst, closest, resp, labels, rowval, D, ord,
                               out, changes, &s_changed, &s_last);
}

// M-step: M = 64 feature columns, N = NB >= K components, k = rows.  grid (column blocks of 64, row
// chunks of kRowChunk); the chunk partials go through the ordered slots like accum_kernel's.
// Loader: x values e = t + 128 i -> (row e / 64, column e % 64); weights e -> (row e / NB,
// component e % NB), so thread t always holds component t % NB and sums its count in row order.
constexpr int kTcCols = 64;
template <int NB, bool X3, bool SQ>
__global__ void __launch_bounds__(kTcThreads)
    accum_tc_kernel(const float* __restrict__ X, const float* __restrict__ mu, int N, int d, int K,
                    const float* __restrict__ resp, const int* __restrict__ labels, Ordered ord,
                    double* __restrict__ sx, double* __restrict__ sxx, double* __restrict__ nk) {
  constexpr int NV = 2 * kTcCols + 1;
  constexpr int XB = 8 * kTcSbo, RB = (NB / 8) * kTcSbo;
  constexpr int XPT = kTcCols * kTcK / kTcThreads, RPT = NB * kTcK / kTcThreads;
  __shared__ __align__(128) unsigned char smem[4 * XB + 2 * RB];
  __shared__ float cnt[kTcThreads];
  __shared__ unsigned s_last;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int j0 = blockIdx.x * kTcCols;
  const int64_t c0 = (int64_t)blockIdx.y * kRowChunk;
  const int64_t c1 = min((int64_t)N, c0 + kRowChunk);
  constexpr bool use_lo = X3, sqm = SQ;
  const uint32_t sb = smem_u32(smem);
  const uint32_t s_x = sb, s_x2 = sb + 2 * XB, s_r = sb + 4 * XB;
  float accs[NB / 2], accq[NB / 2];
#pragma unroll
  for (int i = 0; i < NB / 2; ++i) accs[i] = accq[i] = 0.f;
  float c = 0.f;
  float xv[XPT], rv[RPT];
  auto load = [&](int64_t n0) {
#pragma unroll
    for (int i = 0; i < XPT; ++i) {
      const int e = tid + kTcThreads * i, j = j0 + e % kTcCols;
      const int64_t n = n0 + e / kTcCols;
      float v = 0.f;
      if (n < c1 && j < d) {
        v = __ldg(X + n * d + j);
        if (mu) v -= __ldg(mu + j);
      }
      xv[i] = v;
    }
#pragma unroll
    for (int i = 0; i < RPT; ++i) {
      const int e = tid + kTcThreads * i, k = e % NB;
      const int64_t n = n0 + e / NB;
      float v = 0.f;
      if (n < c1 && k < K) {
        if (resp) v = __ldg(resp + n * K + k);
        else if (labels) v = __ldg(labels + n) == k ? 1.f : 0.f;
        else v = k == 0 ? 1.f : 0.f;
      }
      rv[i] = v;
    }
  };
  load(c0);
  for (int64_t n0 = c0; n0 < c1; n0 += kTcK) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < XPT; ++i) {
      const int e = tid + kTcThreads * i;
      put_split(s_x, XB, e % kTcCols, e / kTcCols, xv[i], use_lo);
      if (sqm) put_split(s_x2, XB, e % kTcCols, e / kTcCols, xv[i] * xv[i], use_lo);
    }
#pragma unroll
    for (int i = 0; i < RPT; ++i) {
      const int e = tid + kTcThreads * i;
      put_split(s_r, RB, e % NB, e / NB, rv[i], use_lo);
      c += rv[i];
    }
    fence_proxy_async_smem();
    __syncthreads();
    wgmma_fence();
    wgmma_fence_regs(accs);
    wgmma_fence_regs(accq);
#pragma unroll
    for (int ks = 0; ks < kTcK / 8; ++ks) {
      mma_split<NB, X3>(accs, s_x + ks * 256, XB, s_r + ks * 256, RB);
      if (SQ) mma_split<NB, X3>(accq, s_x2 + ks * 256, XB, s_r + ks * 256, RB);
    }
    wgmma_commit();
    if (n0 + kTcK < c1) load(n0 + kTcK);
    wgmma_wait<0>();
    wgmma_fence_regs(accs);
    wgmma_fence_regs(accq);
  }
  cnt[tid] = c;
  __syncthreads();
  double* slot = ordered_slot(ord, blockIdx.x, gridDim.y, blockIdx.y, K * NV);
#pragma unroll
  for (int j = 0; j < NB / 8; ++j) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int m = 16 * warp + (lane >> 2) + 8 * (e >> 1), k = 8 * j + 2 * (lane & 3) + (e & 1);
      if (k < K) {
        slot[k * NV + m] = accs[4 * j + e];
        slot[k * NV + kTcCols + m] = accq[4 * j + e];
      }
    }
  }
  if (tid < K) {
    float t = 0.f;
    for (int i = tid; i < kTcThreads; i += NB) t += cnt[i];
    slot[tid * NV + 2 * kTcCols] = t;
  }
  ordered_finish(ord, blockIdx.x, gridDim.y, K * NV, tid, kTcThreads, gridDim.y,
                 [] { __syncthreads(); },
                 [&](int i, double v) {
                   const int k = i / NV, e = i % NV;
                   if (e < kTcCols) {
                     if (j0 + e < d) sx[(int64_t)k * d + j0 + e] = v;
                   } else if (e < 2 * kTcCols) {
                     if (sxx && j0 + e - kTcCols < d) sxx[(int64_t)k * d + j0 + e - kTcCols] = v;
                   } else if (nk && blockIdx.x == 0) {
                     nk[k] = v;
                   }
                 },
                 &s_last);
}

// fixed-shape tree over the CTA (deterministic)
__device__ double block_sum_d(double v, double* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int o = kThreads / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

// one CTA per component: sklearn's _estimate_gaussian_parameters + _compute_precision_cholesky
// (diag / spherical) in float64, and the E-step operands A = mean * prec, B = -prec / 2,
// cst = -(d log 2 pi + sum mean^2 prec) / 2 + log det(prec_chol) + log weight
__global__ void __launch_bounds__(kThreads)
    gmm_params_kernel(const double* __restrict__ sx, const double* __restrict__ sxx,
                      const double* __restrict__ nk, int N, int d, int K, int spherical,
                      double reg, int init, float* __restrict__ means, float* __restrict__ covs,
                      float* __restrict__ weights, float* __restrict__ A, float* __restrict__ B,
                      float* __restrict__ cst) {
  __shared__ double red[kThreads];
  const int k = blockIdx.x, t = threadIdx.x;
  const double eps10 = 10.0 * (double)FLT_EPSILON;
  double tot = 0.0;
  for (int i = 0; i < K; ++i) tot += __ldg(nk + i) + eps10;
  const double n = __ldg(nk + k) + eps10;
  const double w = n / (init ? (double)N : tot);
  const double* px = sx + (int64_t)k * d;
  const double* pxx = sxx + (int64_t)k * d;
  auto var_of = [&](int j) {
    const double m = px[j] / n;
    return pxx[j] / n - 2.0 * m * (px[j] / n) + m * m + reg;
  };
  double sph = 0.0;
  if (spherical) {
    double a = 0.0;
    for (int j = t; j < d; j += kThreads) a += var_of(j);
    sph = block_sum_d(a, red) / d;
  }
  double ld = 0.0, m2p = 0.0;
  for (int j = t; j < d; j += kThreads) {
    const double m = px[j] / n, v = spherical ? sph : var_of(j), p = 1.0 / v;
    means[(int64_t)k * d + j] = (float)m;
    if (!spherical) covs[(int64_t)k * d + j] = (float)v;
    A[(int64_t)k * d + j] = (float)(m * p);
    B[(int64_t)k * d + j] = (float)(-0.5 * p);
    ld += log(1.0 / sqrt(v));
    m2p += m * m * p;
  }
  ld = block_sum_d(ld, red);
  m2p = block_sum_d(m2p, red);
  if (t == 0) {
    if (spherical) covs[k] = (float)sph;
    weights[k] = (float)w;
    cst[k] = (float)(-0.5 * (d * 1.8378770664093453 + m2p) + ld + log(w));
  }
}

// one CTA per centre: c_new = sx / nk (an empty cluster keeps its centre), the squared shift summed
// over centres in order into *shift; A = -2 c, cst = ||c||^2 for the next assignment.  sx == NULL:
// c_new already holds the centres, only A and cst are formed.
__global__ void __launch_bounds__(kThreads)
    kmeans_centres_kernel(const double* __restrict__ sx, const double* __restrict__ nk,
                          const float* __restrict__ c_old, float* __restrict__ c_new, int d,
                          float* __restrict__ A, float* __restrict__ cst, Ordered ord,
                          double* __restrict__ shift) {
  __shared__ double red[kThreads];
  __shared__ unsigned s_last;
  const int k = blockIdx.x, t = threadIdx.x;
  double cc = 0.0, sh = 0.0;
  const double n = sx ? __ldg(nk + k) : 0.0;
  for (int j = t; j < d; j += kThreads) {
    const int64_t e = (int64_t)k * d + j;
    float c;
    if (sx) {
      c = n > 0.0 ? (float)(sx[e] / n) : c_old[e];
      c_new[e] = c;
      const double dd = (double)c - (double)c_old[e];
      sh += dd * dd;
    } else {
      c = c_new[e];
    }
    A[e] = -2.f * c;
    cc += (double)c * c;
  }
  cc = block_sum_d(cc, red);
  sh = block_sum_d(sh, red);
  if (t == 0) cst[k] = (float)cc;
  if (!shift) return;
  if (t == 0) ordered_slot(ord, 0, gridDim.x, k, 1)[0] = sh;
  ordered_finish(ord, 0, gridDim.x, 1, t, kThreads, gridDim.x, [] { __syncthreads(); },
                 [&](int, double s) { *shift = s; }, &s_last);
}

// k-means++: per chunk of kSumChunk rows, the sum of D^2 (each thread 4 consecutive rows, then a
// fixed tree)
__global__ void __launch_bounds__(kThreads)
    chunk_sum_kernel(const float* __restrict__ v, int N, double* __restrict__ out) {
  __shared__ double red[kThreads];
  const int64_t base = (int64_t)blockIdx.x * kSumChunk + threadIdx.x * 4;
  double s = 0.0;
#pragma unroll
  for (int i = 0; i < 4; ++i)
    if (base + i < N) s += (double)__ldg(v + base + i);
  s = block_sum_d(s, red);
  if (threadIdx.x == 0) out[blockIdx.x] = s;
}

// candidate t: u = hash_uniform(counter + t, seed); index = first i with prefix_D2[i] >= u * total
// (numpy searchsorted 'left' over the cumulative sum), or floor(u N) when closest == NULL.  The
// prefix is the chunk sums in order, then the rows of the chosen chunk in order.
__global__ void candidates_kernel(const float* __restrict__ closest, int N,
                                  const double* __restrict__ csum, int nch, int ntr,
                                  uint64_t seed, uint64_t counter, int* __restrict__ idx) {
  const int t = threadIdx.x;
  if (t >= ntr) return;
  const float u = hash_uniform(counter + t, seed);
  if (!closest) {
    idx[t] = min((int)(u * (double)N), N - 1);
    return;
  }
  double tot = 0.0;
  for (int c = 0; c < nch; ++c) tot += csum[c];
  const double r = (double)u * tot;
  double pre = 0.0;
  int c = 0;
  while (c < nch - 1 && pre + csum[c] < r) pre += csum[c++];
  const int64_t i0 = (int64_t)c * kSumChunk, i1 = min((int64_t)N, i0 + kSumChunk);
  int64_t i = i0;
  for (; i < i1 - 1; ++i) {
    pre += (double)closest[i];
    if (pre >= r) break;
  }
  idx[t] = (int)i;
}

__global__ void gather_rows_kernel(const float* __restrict__ X, const float* __restrict__ mu, int d,
                                   const int* __restrict__ idx, float* __restrict__ out) {
  const int64_t row = __ldg(idx + blockIdx.y);
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < d; j += gridDim.x * blockDim.x)
    out[(int64_t)blockIdx.y * d + j] = __ldg(X + row * d + j) - __ldg(mu + j);
}

// keep the candidate of least potential (first on ties, like numpy's argmin): closest <- min(closest,
// D[:, best]); CTA 0 copies the candidate into `centre`
__global__ void __launch_bounds__(kThreads)
    kpp_commit_kernel(const float* __restrict__ D, int ntr, const double* __restrict__ pot,
                      float* __restrict__ closest, int N, const float* __restrict__ cand, int d,
                      float* __restrict__ centre) {
  int best = 0;
  for (int t = 1; t < ntr; ++t)
    if (pot[t] < pot[best]) best = t;
  for (int64_t n = (int64_t)blockIdx.x * kThreads + threadIdx.x; n < N;
       n += (int64_t)gridDim.x * kThreads)
    closest[n] = fminf(closest[n], D[n * ntr + best]);
  if (blockIdx.x == 0)
    for (int j = threadIdx.x; j < d; j += kThreads) centre[j] = cand[(int64_t)best * d + j];
}

template <int MODE>
int estep_mode(int kpt, dim3 grid, cudaStream_t st, const float* X, const float* mu, int N, int d,
               int K, const float* A, const float* B, const float* cst, const float* closest,
               float* resp, int* labels, float* rowval, float* D, const Ordered& ord, double* out,
               double* changes) {
#define AB_ESTEP(KPT)                                                                             \
  estep_kernel<KPT, MODE><<<grid, kThreads, 0, st>>>(X, mu, N, d, K, A, B, cst, closest, resp,   \
                                                     labels, rowval, D, ord, out, changes)
  if (kpt == 1) AB_ESTEP(1);
  else if (kpt == 2) AB_ESTEP(2);
  else AB_ESTEP(4);
#undef AB_ESTEP
  AB_LAUNCH_CHECK();
  return 0;
}

}  // namespace

extern "C" int atomai_b200_stat_estep(const float* X, const float* mu, int N, int d, int K, int mode,
                                      const float* A, const float* B, const float* cst,
                                      const float* closest, float* resp, int* labels,
                                      float* rowval, float* D, double* out, double* changes,
                                      int math, void* stream) {
  AB_CHECK(N >= 1 && d >= 1 && K >= 1 && K <= kMaxK, "stat_estep: bad dims N=%d d=%d K=%d (K <= %d)",
           N, d, K, kMaxK);
  AB_CHECK(mode >= kModeGMM && mode <= kModeKPP, "stat_estep: mode=%d", mode);
  AB_CHECK(X && mu && A && cst && out, "stat_estep: null pointer");
  AB_CHECK(mode != kModeGMM || B, "stat_estep: GMM mode needs B");
  AB_CHECK(mode != kModeKMeans || labels, "stat_estep: k-means mode needs labels");
  AB_CHECK(mode != kModeKPP || (closest && D), "stat_estep: k-means++ mode needs closest and D");
  cudaStream_t st = (cudaStream_t)stream;
  const int nb = (N + kRows - 1) / kRows;
  const int nv = mode == kModeKPP ? K : 1;
  Ordered ord;
  if (ab_ordered_ws(st, (int64_t)nb * nv, 1, &ord)) return 1;
  const dim3 grid(nb);
  if (math != AB_MATH_FP32) {
    const int x3 = math == AB_MATH_TF32X3;
#define AB_ESTEP_TC3(NB, MODE, X3)                                                            \
  estep_tc_kernel<NB, MODE, X3><<<grid, kTcThreads, 0, st>>>(X, mu, N, d, K, A, B, cst, closest, \
                                                             resp, labels, rowval, D, ord, out,   \
                                                             changes)
#define AB_ESTEP_TC(NB, MODE) \
  { if (x3) AB_ESTEP_TC3(NB, MODE, true); else AB_ESTEP_TC3(NB, MODE, false); }
#define AB_ESTEP_TC_NB(MODE)            \
  if (K <= 16) AB_ESTEP_TC(16, MODE)     \
  else if (K <= 32) AB_ESTEP_TC(32, MODE) \
  else AB_ESTEP_TC(64, MODE)
    if (mode == kModeGMM) { AB_ESTEP_TC_NB(kModeGMM) }
    else if (mode == kModeKMeans) { AB_ESTEP_TC_NB(kModeKMeans) }
    else { AB_ESTEP_TC_NB(kModeKPP) }
#undef AB_ESTEP_TC_NB
#undef AB_ESTEP_TC
#undef AB_ESTEP_TC3
    AB_LAUNCH_CHECK();
    return 0;
  }
  const int kpt = K <= 16 ? 1 : (K <= 32 ? 2 : 4);
  if (mode == kModeGMM)
    return estep_mode<kModeGMM>(kpt, grid, st, X, mu, N, d, K, A, B, cst, closest, resp, labels,
                                rowval, D, ord, out, changes);
  if (mode == kModeKMeans)
    return estep_mode<kModeKMeans>(kpt, grid, st, X, mu, N, d, K, A, B, cst, closest, resp, labels,
                                   rowval, D, ord, out, changes);
  return estep_mode<kModeKPP>(kpt, grid, st, X, mu, N, d, K, A, B, cst, closest, resp, labels,
                              rowval, D, ord, out, changes);
}

extern "C" int atomai_b200_stat_accum(const float* X, const float* mu, int N, int d, int K,
                                      const float* resp, const int* labels, double* sx,
                                      double* sxx, double* nk, int math, void* stream) {
  AB_CHECK(N >= 1 && d >= 1 && K >= 1 && K <= kMaxK, "stat_accum: bad dims N=%d d=%d K=%d (K <= %d)",
           N, d, K, kMaxK);
  AB_CHECK(X && sx, "stat_accum: null pointer");
  const int cols = math == AB_MATH_FP32 ? kCols : kTcCols;
  const int ncb = (d + cols - 1) / cols, nch = (N + kRowChunk - 1) / kRowChunk;
  AB_CHECK(ncb <= 4096 && nch <= 65535, "stat_accum: d=%d or N=%d too large", d, N);
  cudaStream_t st = (cudaStream_t)stream;
  Ordered ord;
  if (math != AB_MATH_FP32) {
    if (ab_ordered_ws(st, (int64_t)ncb * nch * K * (2 * kTcCols + 1), ncb, &ord)) return 1;
    const dim3 grid(ncb, nch);
    const int x3 = math == AB_MATH_TF32X3, sq = sxx != nullptr;
#define AB_ACCUM_TC3(NB, X3, SQ)                                                             \
  accum_tc_kernel<NB, X3, SQ><<<grid, kTcThreads, 0, st>>>(X, mu, N, d, K, resp, labels, ord, sx, \
                                                           sxx, nk)
#define AB_ACCUM_TC(NB)                                                  \
  if (x3) { if (sq) AB_ACCUM_TC3(NB, true, true); else AB_ACCUM_TC3(NB, true, false); } \
  else { if (sq) AB_ACCUM_TC3(NB, false, true); else AB_ACCUM_TC3(NB, false, false); }
    if (K <= 16) { AB_ACCUM_TC(16) }
    else if (K <= 32) { AB_ACCUM_TC(32) }
    else { AB_ACCUM_TC(64) }
#undef AB_ACCUM_TC
#undef AB_ACCUM_TC3
    AB_LAUNCH_CHECK();
    return 0;
  }
  if (ab_ordered_ws(st, (int64_t)ncb * nch * K * (2 * kCols + 1), ncb, &ord)) return 1;
  const dim3 grid(ncb, nch);
  const int sq = sxx != nullptr;
#define AB_ACCUM(KW) \
  accum_kernel<KW><<<grid, kThreads, 0, st>>>(X, mu, N, d, K, resp, labels, sq, ord, sx, sxx, nk)
  if (K <= 8) AB_ACCUM(1);
  else if (K <= 16) AB_ACCUM(2);
  else if (K <= 32) AB_ACCUM(4);
  else AB_ACCUM(8);
#undef AB_ACCUM
  AB_LAUNCH_CHECK();
  return 0;
}

extern "C" int atomai_b200_stat_gmm_params(const double* sx, const double* sxx, const double* nk,
                                           int N, int d, int K, int spherical, double reg_covar,
                                           int init, float* means, float* covs, float* weights,
                                           float* A, float* B, float* cst, void* stream) {
  AB_CHECK(N >= 1 && d >= 1 && K >= 1 && K <= kMaxK, "stat_gmm_params: bad dims N=%d d=%d K=%d", N,
           d, K);
  AB_CHECK(sx && sxx && nk && means && covs && weights && A && B && cst,
           "stat_gmm_params: null pointer");
  gmm_params_kernel<<<K, kThreads, 0, (cudaStream_t)stream>>>(
      sx, sxx, nk, N, d, K, spherical, reg_covar, init, means, covs, weights, A, B, cst);
  AB_LAUNCH_CHECK();
  return 0;
}

extern "C" int atomai_b200_stat_kmeans_centres(const double* sx, const double* nk,
                                               const float* c_old, float* c_new, int K, int d,
                                               float* A, float* cst, double* shift, void* stream) {
  AB_CHECK(K >= 1 && K <= kMaxK && d >= 1, "stat_kmeans_centres: bad dims K=%d d=%d", K, d);
  AB_CHECK(c_new && A && cst && (!sx || (nk && c_old && shift)), "stat_kmeans_centres: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  Ordered ord{nullptr, nullptr};
  if (sx && ab_ordered_ws(st, K, 1, &ord)) return 1;
  kmeans_centres_kernel<<<K, kThreads, 0, st>>>(sx, nk, c_old, c_new, d, A, cst, ord,
                                                sx ? shift : nullptr);
  AB_LAUNCH_CHECK();
  return 0;
}

extern "C" int atomai_b200_stat_kpp_candidates(const float* closest, int N, int ntr, uint64_t seed,
                                               uint64_t counter, double* chunk_ws, int* idx,
                                               void* stream) {
  AB_CHECK(N >= 1 && ntr >= 1 && ntr <= 32, "stat_kpp_candidates: N=%d ntr=%d", N, ntr);
  AB_CHECK(idx && (!closest || chunk_ws), "stat_kpp_candidates: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int nch = (N + kSumChunk - 1) / kSumChunk;
  if (closest) {
    chunk_sum_kernel<<<nch, kThreads, 0, st>>>(closest, N, chunk_ws);
    AB_LAUNCH_CHECK();
  }
  candidates_kernel<<<1, 32, 0, st>>>(closest, N, chunk_ws, nch, ntr, seed, counter, idx);
  AB_LAUNCH_CHECK();
  return 0;
}

extern "C" int64_t atomai_b200_stat_kpp_chunks(int N) {
  return N >= 1 ? (N + kSumChunk - 1) / kSumChunk : 0;
}

extern "C" int atomai_b200_stat_gather_rows(const float* X, const float* mu, int d, const int* idx,
                                            int n, float* out, void* stream) {
  AB_CHECK(d >= 1 && n >= 1 && n <= 65535, "stat_gather_rows: d=%d n=%d", d, n);
  AB_CHECK(X && mu && idx && out, "stat_gather_rows: null pointer");
  const dim3 grid((d + kThreads - 1) / kThreads, n);
  gather_rows_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(X, mu, d, idx, out);
  AB_LAUNCH_CHECK();
  return 0;
}

extern "C" int atomai_b200_stat_kpp_commit(const float* D, int ntr, const double* pot,
                                           float* closest, int N, const float* cand, int d,
                                           float* centre, void* stream) {
  AB_CHECK(N >= 1 && d >= 1 && ntr >= 1 && ntr <= kMaxK, "stat_kpp_commit: N=%d d=%d ntr=%d", N, d,
           ntr);
  AB_CHECK(D && pot && closest && cand && centre, "stat_kpp_commit: null pointer");
  const int64_t nb = (N + kThreads - 1) / kThreads;
  kpp_commit_kernel<<<(unsigned)(nb < 1024 ? nb : 1024), kThreads, 0, (cudaStream_t)stream>>>(
      D, ntr, pot, closest, N, cand, d, centre);
  AB_LAUNCH_CHECK();
  return 0;
}
