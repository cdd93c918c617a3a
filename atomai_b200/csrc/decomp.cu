// decomp.cu — the passes of PCA, NMF (coordinate descent) and FastICA over a stack of flattened
// sub-images X (N x d, fp32, row-major), read in place.
//
//   gram        G = (X - mu)^T (X - mu) (d x d) or (X - mu)(X - mu)^T (N x N), float64, symmetric:
//               only the upper-triangle 64 x 64 tiles are computed; each is written and mirrored.
//   project     out = (X - mu) B^T for up to 64 rows of B (k x d); out (N x k) fp32 with any ld.
//   nmf_w       per row tile: XHt = X H^T, then sklearn's coordinate-descent sweep of the tile's rows
//               of W (rows are independent, so the component-outer / sample-inner loop of
//               _update_cdnmf_fast gives the same result row by row), W written back, W^T W and the
//               projected-gradient violation summed.
//   nmf_h       the same sweep over the d columns of H from W^T X (atomai_b200_stat_accum with resp =
//               W) and W^T W; H written back, H H^T and the violation summed.
//   ica_step    one FastICA (parallel, logcosh) pass over the whitened samples X1 (N x k):
//               y = W x1, g = tanh(y); sums of g x1^T (k x k) and of 1 - g^2 (k).
//
// Arithmetic: exact fp32 FFMA for the contractions over X (the library's set_math mode does not
// apply here), float64 for the coordinate descent, the FastICA step and every sum across rows.  The
// Gram flushes its fp32 tile accumulators into float64 registers every kFlush contraction steps.
//
// Determinism: no floating-point atomics.  Cross-CTA sums go through the ordered slots of
// common.cuh and every partition (Gram chunks, row tiles, sample chunks) depends on the shapes only,
// so a repeated call gives identical bits on any GPU.
#include <math.h>
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kMaxK = 64;
constexpr int kStage = 32;           // project / nmf_w: features per stage

// ---------------------------------------------------------------- Gram
constexpr int kT = 64;               // output tile
constexpr int kK = 16;               // contraction stage
constexpr int kTp = kT + 4;          // smem row (16-byte aligned)
constexpr int kFlush = 256;          // fp32 steps between float64 flushes
constexpr int kGramMinChunk = 1024;  // least contraction length per CTA
constexpr int kGramCtas = 1024;      // CTAs the chunking aims for

struct GramPlan {
  int m, nt, ntiles, nch;
  int64_t L, chunk;
};

// rows = 0: G = Xc^T Xc (m = d, contraction over the N rows); rows = 1: G = Xc Xc^T (m = N, over d)
GramPlan gram_plan(int N, int d, int rows) {
  GramPlan p;
  p.m = rows ? N : d;
  p.L = rows ? d : N;
  p.nt = (p.m + kT - 1) / kT;
  p.ntiles = p.nt * (p.nt + 1) / 2;
  int64_t n = (p.L + kGramMinChunk - 1) / kGramMinChunk;
  const int64_t want = (kGramCtas + p.ntiles - 1) / p.ntiles;
  if (n > want) n = want;
  if (n < 1) n = 1;
  int64_t c = (p.L + n - 1) / n;
  p.chunk = (c + kK - 1) / kK * kK;
  p.nch = (int)((p.L + p.chunk - 1) / p.chunk);
  return p;
}

// grid (upper tiles, contraction chunks); thread (ty, tx) owns outputs (4 ty + a, 4 tx + b).
// Operand e = t + 256 i of a stage: ROWS ? (p = e / 16, c = e % 16) : (c = e / 64, p = e % 64), so
// the global loads run along X's rows either way.
template <bool ROWS>
__global__ void __launch_bounds__(kThreads)
    gram_kernel(const float* __restrict__ X, const float* __restrict__ mu, int N, int d, GramPlan P,
                Ordered ord, double* __restrict__ G) {
  __shared__ __align__(16) float as[kK][kTp];
  __shared__ __align__(16) float bs[kK][kTp];
  __shared__ unsigned s_last;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  int ti = 0, r = blockIdx.x;
  while (r >= P.nt - ti) r -= P.nt - ti++;
  const int tj = ti + r;
  const int p0 = ti * kT, q0 = tj * kT;
  const int64_t c0 = (int64_t)blockIdx.y * P.chunk;
  const int64_t c1 = min(P.L, c0 + P.chunk);
  float av[4], bv[4];
  auto fetch = [&](int64_t cs, int o0, float* v, int e) {
    const int p = ROWS ? e / kK : e % kT, c = ROWS ? e % kK : e / kT;
    const int64_t cc = cs + c;
    const int pp = o0 + p;
    float x = 0.f;
    if (pp < P.m && cc < c1) {
      const int64_t row = ROWS ? pp : cc;
      const int64_t col = ROWS ? cc : pp;
      x = __ldg(X + row * d + col);
      if (mu) x -= __ldg(mu + col);
    }
    *v = x;
  };
  auto load = [&](int64_t cs) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      fetch(cs, p0, av + i, tid + kThreads * i);
      fetch(cs, q0, bv + i, tid + kThreads * i);
    }
  };
  float acc[4][4];
  double accd[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.f, accd[a][b] = 0.0;
  load(c0);
  int steps = 0;
  for (int64_t cs = c0; cs < c1; cs += kK) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = tid + kThreads * i;
      const int p = ROWS ? e / kK : e % kT, c = ROWS ? e % kK : e / kT;
      as[c][p] = av[i];
      bs[c][p] = bv[i];
    }
    __syncthreads();
    if (cs + kK < c1) load(cs + kK);
#pragma unroll
    for (int c = 0; c < kK; ++c) {
      const float4 a4 = *reinterpret_cast<const float4*>(&as[c][4 * ty]);
      const float4 b4 = *reinterpret_cast<const float4*>(&bs[c][4 * tx]);
      const float a[4] = {a4.x, a4.y, a4.z, a4.w}, b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if ((steps += kK) == kFlush) {
      steps = 0;
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) accd[i][j] += acc[i][j], acc[i][j] = 0.f;
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) accd[i][j] += acc[i][j];
  const int64_t m = P.m;
  auto put = [&](int p, int q, double v) {
    if (p < m && q < m) {
      G[(int64_t)p * m + q] = v;
      if (ti != tj) G[(int64_t)q * m + p] = v;
    }
  };
  if (P.nch == 1) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) put(p0 + 4 * ty + i, q0 + 4 * tx + j, accd[i][j]);
    return;
  }
  double* slot = ordered_slot(ord, blockIdx.x, P.nch, blockIdx.y, kT * kT);
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) slot[(4 * ty + i) * kT + 4 * tx + j] = accd[i][j];
  ordered_finish(ord, blockIdx.x, P.nch, kT * kT, tid, kThreads, P.nch, [] { __syncthreads(); },
                 [&](int e, double v) { put(p0 + e / kT, q0 + e % kT, v); }, &s_last);
}

// ---------------------------------------------------------------- row tiles: (X - mu) B^T
// KP = components padded to 16 / 32 / 64; thread (rg, kg) = (t / (KP/4), t % (KP/4)) owns rows
// 4 rg .. +3 and components 4 kg .. +3 of a tile of kRowsOf(KP) = 4096 / KP rows, so a small K gets
// a tall tile and every thread the same 16 FMAs per feature.
template <int KP>
struct RowTile {
  static constexpr int KG = KP / 4, RG = kThreads / KG, ROWS = 4 * RG;
  static constexpr int XS = ROWS * (kStage + 1), BS = kStage * (KP + 4);   // floats
};

// acc[i][q] = sum_j (x[r0 + 4 rg + i, j] - mu_j) B[4 kg + q, j] (fp32, j in order); xs / bs: smem
template <int KP>
__device__ __forceinline__ void row_tile_dot(const float* __restrict__ X,
                                             const float* __restrict__ mu, int N, int d, int K,
                                             const float* __restrict__ B, int64_t r0, float* xs,
                                             float* bs, float (&acc)[4][4]) {
  using T = RowTile<KP>;
  // loader: thread t stages column t % 32 of rows (components) t / 32 + 8 i
  constexpr int RS = kThreads / kStage, XPT = T::ROWS / RS, BPT = KP / RS;
  const int tid = threadIdx.x, kg = tid % T::KG, rg = tid / T::KG;
  const int lr = tid / kStage, lc = tid % kStage;
  const int xrows = (int)min((int64_t)T::ROWS, (int64_t)N - r0) - lr;
  const float* xsrc = X + (r0 + lr) * d + lc;
  const float* bsrc = B + (int64_t)lr * d + lc;
  float xv[XPT], bv[BPT];
  auto load = [&](int j0) {
    const bool col = j0 + lc < d;
    const float m = (mu && col) ? __ldg(mu + j0 + lc) : 0.f;
    const float* p = xsrc + j0;
#pragma unroll
    for (int i = 0; i < XPT; ++i, p += (int64_t)RS * d) xv[i] = (col && RS * i < xrows) ? __ldg(p) - m : 0.f;
    p = bsrc + j0;
#pragma unroll
    for (int i = 0; i < BPT; ++i, p += (int64_t)RS * d) bv[i] = (col && lr + RS * i < K) ? __ldg(p) : 0.f;
  };
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[i][q] = 0.f;
  load(0);
  for (int j0 = 0; j0 < d; j0 += kStage) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < XPT; ++i) xs[(lr + RS * i) * (kStage + 1) + lc] = xv[i];
#pragma unroll
    for (int i = 0; i < BPT; ++i) bs[lc * (KP + 4) + lr + RS * i] = bv[i];
    __syncthreads();
    if (j0 + kStage < d) load(j0 + kStage);
#pragma unroll 8
    for (int jj = 0; jj < kStage; ++jj) {
      const float4 b4 = *reinterpret_cast<const float4*>(bs + jj * (KP + 4) + 4 * kg);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float x = xs[(4 * rg + i) * (kStage + 1) + jj];
        acc[i][0] = fmaf(x, b4.x, acc[i][0]);
        acc[i][1] = fmaf(x, b4.y, acc[i][1]);
        acc[i][2] = fmaf(x, b4.z, acc[i][2]);
        acc[i][3] = fmaf(x, b4.w, acc[i][3]);
      }
    }
  }
}

template <int KP>
__global__ void __launch_bounds__(kThreads)
    project_kernel(const float* __restrict__ X, const float* __restrict__ mu, int N, int d, int K,
                   const float* __restrict__ B, float* __restrict__ out, int ldo) {
  using T = RowTile<KP>;
  __shared__ __align__(16) float xs[T::XS];
  __shared__ __align__(16) float bs[T::BS];
  const int tid = threadIdx.x, kg = tid % T::KG, rg = tid / T::KG;
  const int64_t r0 = (int64_t)blockIdx.x * T::ROWS;
  float acc[4][4];
  row_tile_dot<KP>(X, mu, N, d, K, B, r0, xs, bs, acc);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t row = r0 + 4 * rg + i;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int k = 4 * kg + q;
      if (row < N && k < K) out[row * ldo + k] = acc[i][q];
    }
  }
}

// ---------------------------------------------------------------- NMF coordinate descent
// sklearn's _update_cdnmf_fast for one row w (K <= KP values, the rest zero) against the Gram hh
// (KP x KP float64 in smem, zero-padded): components in order, grad = -xht(t) + sum_r hh[t][r] w[r],
// projected gradient min(0, grad) where w[t] == 0, w[t] = max(w[t] - grad / hh[t][t], 0).
template <int KP, class Xht>
__device__ __forceinline__ double cd_sweep(float (&w)[KP], int K, const double* hh, Xht xht) {
  double viol = 0.0;
#pragma unroll
  for (int t = 0; t < KP; ++t) {
    if (t < K) {
      double grad = -xht(t);
#pragma unroll
      for (int r = 0; r < KP; ++r) grad = fma(hh[t * KP + r], (double)w[r], grad);
      const double pg = w[t] == 0.f ? fmin(0.0, grad) : grad;
      viol += fabs(pg);
      const double hess = hh[t * KP + t];
      if (hess != 0.0) w[t] = (float)fmax((double)w[t] - grad / hess, 0.0);
    }
  }
  return viol;
}

// Shared memory of the two sweep kernels (dynamic): [hh: KP*KP double][viol: ROWS double]
// [work: max(row-tile stage, ROWS x (KP + 1) floats)]
template <int KP>
constexpr int sweep_smem_bytes() {
  using T = RowTile<KP>;
  constexpr int stage = (T::XS + T::BS) * 4, vals = T::ROWS * (KP + 1) * 4;
  return KP * KP * 8 + T::ROWS * 8 + (stage > vals ? stage : vals);
}

template <int KP>
__device__ __forceinline__ void load_gram_smem(const double* __restrict__ g, int K, double* hh) {
  for (int e = threadIdx.x; e < KP * KP; e += kThreads) {
    const int a = e / KP, b = e % KP;
    hh[e] = (a < K && b < K) ? __ldg(g + a * K + b) : 0.0;
  }
}

// After the sweep: vals (ROWS x (KP + 1) floats) hold the tile's updated rows (zero where invalid),
// viol the per-row violations.  Emits sum_rows v v^T (K x K) and the violation (value K * K) through
// the ordered slots, CTA order.
template <int KP>
__device__ __forceinline__ void emit_gram_viol(const float* vals, const double* viol, int K,
                                               const Ordered& ord, double* __restrict__ out,
                                               unsigned* s_last) {
  constexpr int ROWS = RowTile<KP>::ROWS, EPT = (KP * KP + kThreads - 1) / kThreads;
  const int tid = threadIdx.x, nv = K * K + 1;
  double* slot = ordered_slot(ord, 0, gridDim.x, blockIdx.x, nv);
#pragma unroll
  for (int q = 0; q < EPT; ++q) {
    const int e = tid + kThreads * q, a = e / KP, b = e % KP;
    if (e < KP * KP && a < K && b < K) {
      double s = 0.0;
      for (int r = 0; r < ROWS; ++r)
        s = fma((double)vals[r * (KP + 1) + a], (double)vals[r * (KP + 1) + b], s);
      slot[a * K + b] = s;
    }
  }
  if (tid == 0) {
    double s = 0.0;
    for (int r = 0; r < ROWS; ++r) s += viol[r];
    slot[K * K] = s;
  }
  ordered_finish(ord, 0, gridDim.x, nv, tid, kThreads, gridDim.x, [] { __syncthreads(); },
                 [&](int i, double v) { out[i] = v; }, s_last);
}

template <int KP>
__global__ void __launch_bounds__(kThreads)
    nmf_w_kernel(const float* __restrict__ X, int N, int d, int K, const float* __restrict__ H,
                 const double* __restrict__ HHt, float* __restrict__ W, Ordered ord,
                 double* __restrict__ out) {
  using T = RowTile<KP>;
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ unsigned s_last;
  double* hh = reinterpret_cast<double*>(smem);
  double* viol = hh + KP * KP;
  float* work = reinterpret_cast<float*>(viol + T::ROWS);
  const int tid = threadIdx.x, kg = tid % T::KG, rg = tid / T::KG;
  const int64_t r0 = (int64_t)blockIdx.x * T::ROWS;
  load_gram_smem<KP>(HHt, K, hh);
  float acc[4][4];
  row_tile_dot<KP>(X, nullptr, N, d, K, H, r0, work, work + T::XS, acc);
  __syncthreads();
  float* sc = work;                                  // XHt rows, then the updated W rows
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int q = 0; q < 4; ++q) sc[(4 * rg + i) * (KP + 1) + 4 * kg + q] = acc[i][q];
  __syncthreads();
  if (tid < T::ROWS) {
    const int64_t row = r0 + tid;
    float w[KP];
    double v = 0.0;
#pragma unroll
    for (int t = 0; t < KP; ++t) w[t] = (row < N && t < K) ? W[row * K + t] : 0.f;
    if (row < N) {
      v = cd_sweep<KP>(w, K, hh, [&](int t) { return (double)sc[tid * (KP + 1) + t]; });
#pragma unroll
      for (int t = 0; t < KP; ++t)
        if (t < K) W[row * K + t] = w[t];
    }
#pragma unroll
    for (int t = 0; t < KP; ++t) sc[tid * (KP + 1) + t] = w[t];
    viol[tid] = v;
  }
  __syncthreads();
  emit_gram_viol<KP>(sc, viol, K, ord, out, &s_last);
}

// columns c0 + t (t < ROWS) of H (K x d), one per thread
template <int KP>
__global__ void __launch_bounds__(kThreads)
    nmf_h_kernel(const double* __restrict__ WtX, const double* __restrict__ WtW, int d, int K,
                 float* __restrict__ H, Ordered ord, double* __restrict__ out) {
  using T = RowTile<KP>;
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ unsigned s_last;
  double* hh = reinterpret_cast<double*>(smem);
  double* viol = hh + KP * KP;
  float* sc = reinterpret_cast<float*>(viol + T::ROWS);
  const int tid = threadIdx.x;
  load_gram_smem<KP>(WtW, K, hh);
  __syncthreads();
  if (tid < T::ROWS) {
    const int64_t col = (int64_t)blockIdx.x * T::ROWS + tid;
    float h[KP];
    double v = 0.0;
#pragma unroll
    for (int t = 0; t < KP; ++t) h[t] = (col < d && t < K) ? H[t * d + col] : 0.f;
    if (col < d) {
      v = cd_sweep<KP>(h, K, hh, [&](int t) { return __ldg(WtX + t * d + col); });
#pragma unroll
      for (int t = 0; t < KP; ++t)
        if (t < K) H[t * d + col] = h[t];
    }
#pragma unroll
    for (int t = 0; t < KP; ++t) sc[tid * (KP + 1) + t] = h[t];
    viol[tid] = v;
  }
  __syncthreads();
  emit_gram_viol<KP>(sc, viol, K, ord, out, &s_last);
}

// ---------------------------------------------------------------- FastICA step
constexpr int kIcaTile = 64;     // samples per smem tile
constexpr int kIcaChunk = 512;   // samples per CTA (fixed: the sums depend on it)

template <int KP>
constexpr int ica_smem_bytes() {
  return KP * KP * 8 + kIcaTile * (KP + 1) * 8 + kIcaTile * (KP + 1) * 4;
}

// thread t: sample t % 64 and components t / 64 + 4 q of a tile for y and g; entries (e / KP,
// e % KP), e = t + 256 q of sum g x1^T; t < K also the sum of 1 - g^2.  All float64.
template <int KP>
__global__ void __launch_bounds__(kThreads)
    ica_step_kernel(const float* __restrict__ X1, int N, int K, const double* __restrict__ Wm,
                    Ordered ord, double* __restrict__ out) {
  constexpr int EPT = (KP * KP + kThreads - 1) / kThreads;
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ unsigned s_last;
  double* ws = reinterpret_cast<double*>(smem);
  double* gs = ws + KP * KP;
  float* xs = reinterpret_cast<float*>(gs + kIcaTile * (KP + 1));
  const int tid = threadIdx.x, s = tid % kIcaTile, ig = tid / kIcaTile;
  load_gram_smem<KP>(Wm, K, ws);
  double accg[EPT], acch = 0.0;
#pragma unroll
  for (int q = 0; q < EPT; ++q) accg[q] = 0.0;
  const int64_t n0 = (int64_t)blockIdx.x * kIcaChunk;
  const int64_t n1 = min((int64_t)N, n0 + kIcaChunk);
  for (int64_t t0 = n0; t0 < n1; t0 += kIcaTile) {
    const int nv = (int)min((int64_t)kIcaTile, n1 - t0);
    __syncthreads();
    for (int e = tid; e < kIcaTile * KP; e += kThreads) {
      const int r = e / KP, k = e % KP;
      xs[r * (KP + 1) + k] = (r < nv && k < K) ? __ldg(X1 + (t0 + r) * K + k) : 0.f;
    }
    __syncthreads();
    for (int i = ig; i < KP; i += kThreads / kIcaTile) {
      double y = 0.0;
      for (int j = 0; j < K; ++j) y = fma(ws[i * KP + j], (double)xs[s * (KP + 1) + j], y);
      gs[s * (KP + 1) + i] = (s < nv && i < K) ? tanh(y) : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < EPT; ++q) {
      const int e = tid + kThreads * q, a = e / KP, b = e % KP;
      if (e < KP * KP)
        for (int r = 0; r < nv; ++r)
          accg[q] = fma(gs[r * (KP + 1) + a], (double)xs[r * (KP + 1) + b], accg[q]);
    }
    if (tid < K)
      for (int r = 0; r < nv; ++r) {
        const double g = gs[r * (KP + 1) + tid];
        acch += 1.0 - g * g;
      }
  }
  const int nvals = K * K + K;
  double* slot = ordered_slot(ord, 0, gridDim.x, blockIdx.x, nvals);
#pragma unroll
  for (int q = 0; q < EPT; ++q) {
    const int e = tid + kThreads * q, a = e / KP, b = e % KP;
    if (e < KP * KP && a < K && b < K) slot[a * K + b] = accg[q];
  }
  if (tid < K) slot[K * K + tid] = acch;
  ordered_finish(ord, 0, gridDim.x, nvals, tid, kThreads, gridDim.x, [] { __syncthreads(); },
                 [&](int i, double v) { out[i] = v; }, &s_last);
}

int kp_of(int K) { return K <= 16 ? 16 : (K <= 32 ? 32 : 64); }

template <int KP>
int64_t sweep_ctas(int rows) {
  return (rows + RowTile<KP>::ROWS - 1) / RowTile<KP>::ROWS;
}

int64_t sweep_ctas(int KP, int rows) {
  return KP == 16 ? sweep_ctas<16>(rows) : (KP == 32 ? sweep_ctas<32>(rows) : sweep_ctas<64>(rows));
}

}  // namespace

extern "C" int64_t atomai_b200_decomp_slot_doubles(int op, int N, int d, int K) {
  if (N < 1 || d < 1 || K < 1 || K > kMaxK) return -1;
  switch (op) {
    case 0:
    case 1: {
      const GramPlan P = gram_plan(N, d, op);
      return P.nch > 1 ? (int64_t)P.ntiles * P.nch * kT * kT : 0;
    }
    case 2: return sweep_ctas(kp_of(K), N) * (K * K + 1);
    case 3: return sweep_ctas(kp_of(K), d) * (K * K + 1);
    case 4: return (int64_t)((N + kIcaChunk - 1) / kIcaChunk) * (K * K + K);
    default: return -1;
  }
}

extern "C" int atomai_b200_decomp_gram(const float* X, const float* mu, int N, int d, int rows,
                                       double* G, void* stream) {
  AB_CHECK(N >= 1 && d >= 1 && (rows == 0 || rows == 1), "decomp_gram: N=%d d=%d rows=%d", N, d,
           rows);
  AB_CHECK(X && G, "decomp_gram: null pointer");
  const GramPlan P = gram_plan(N, d, rows);
  AB_CHECK(P.nch <= 65535 && P.ntiles <= (int64_t)1 << 30, "decomp_gram: N=%d d=%d too large", N, d);
  cudaStream_t st = (cudaStream_t)stream;
  Ordered ord{nullptr, nullptr};
  if (P.nch > 1 && ab_ordered_ws(st, (int64_t)P.ntiles * P.nch * kT * kT, P.ntiles, &ord)) return 1;
  const dim3 grid(P.ntiles, P.nch);
  if (rows) gram_kernel<true><<<grid, kThreads, 0, st>>>(X, mu, N, d, P, ord, G);
  else gram_kernel<false><<<grid, kThreads, 0, st>>>(X, mu, N, d, P, ord, G);
  AB_LAUNCH_CHECK();
  return 0;
}

extern "C" int atomai_b200_decomp_project(const float* X, const float* mu, int N, int d, int K,
                                          const float* B, float* out, int ldo, void* stream) {
  AB_CHECK(N >= 1 && d >= 1 && K >= 1 && K <= kMaxK && ldo >= K,
           "decomp_project: N=%d d=%d K=%d (<= %d) ldo=%d", N, d, K, kMaxK, ldo);
  AB_CHECK(X && B && out, "decomp_project: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int KP = kp_of(K);
  const unsigned grid = (unsigned)sweep_ctas(KP, N);
  if (KP == 16) project_kernel<16><<<grid, kThreads, 0, st>>>(X, mu, N, d, K, B, out, ldo);
  else if (KP == 32) project_kernel<32><<<grid, kThreads, 0, st>>>(X, mu, N, d, K, B, out, ldo);
  else project_kernel<64><<<grid, kThreads, 0, st>>>(X, mu, N, d, K, B, out, ldo);
  AB_LAUNCH_CHECK();
  return 0;
}

#define AB_DYN_LAUNCH(KERN, BYTES, GRID, ...)                                   \
  do {                                                                          \
    static unsigned char done[64] = {0};                                        \
    if (ab_optin_smem((const void*)KERN, BYTES, done)) return 1;                \
    KERN<<<GRID, kThreads, BYTES, st>>>(__VA_ARGS__);                           \
  } while (0)

extern "C" int atomai_b200_decomp_nmf_w(const float* X, int N, int d, int K, const float* H,
                                        const double* HHt, float* W, double* out, void* stream) {
  AB_CHECK(N >= 1 && d >= 1 && K >= 1 && K <= kMaxK, "decomp_nmf_w: N=%d d=%d K=%d (<= %d)", N, d,
           K, kMaxK);
  AB_CHECK(X && H && HHt && W && out, "decomp_nmf_w: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int KP = kp_of(K);
  const int64_t grid = sweep_ctas(KP, N);
  Ordered ord;
  if (ab_ordered_ws(st, grid * (K * K + 1), 1, &ord)) return 1;
  if (KP == 16) AB_DYN_LAUNCH(nmf_w_kernel<16>, sweep_smem_bytes<16>(), grid, X, N, d, K, H, HHt, W, ord, out);
  else if (KP == 32) AB_DYN_LAUNCH(nmf_w_kernel<32>, sweep_smem_bytes<32>(), grid, X, N, d, K, H, HHt, W, ord, out);
  else AB_DYN_LAUNCH(nmf_w_kernel<64>, sweep_smem_bytes<64>(), grid, X, N, d, K, H, HHt, W, ord, out);
  AB_LAUNCH_CHECK();
  return 0;
}

extern "C" int atomai_b200_decomp_nmf_h(const double* WtX, const double* WtW, int d, int K,
                                        float* H, double* out, void* stream) {
  AB_CHECK(d >= 1 && K >= 1 && K <= kMaxK, "decomp_nmf_h: d=%d K=%d (<= %d)", d, K, kMaxK);
  AB_CHECK(WtX && WtW && H && out, "decomp_nmf_h: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int KP = kp_of(K);
  const int64_t grid = sweep_ctas(KP, d);
  Ordered ord;
  if (ab_ordered_ws(st, grid * (K * K + 1), 1, &ord)) return 1;
  if (KP == 16) AB_DYN_LAUNCH(nmf_h_kernel<16>, sweep_smem_bytes<16>(), grid, WtX, WtW, d, K, H, ord, out);
  else if (KP == 32) AB_DYN_LAUNCH(nmf_h_kernel<32>, sweep_smem_bytes<32>(), grid, WtX, WtW, d, K, H, ord, out);
  else AB_DYN_LAUNCH(nmf_h_kernel<64>, sweep_smem_bytes<64>(), grid, WtX, WtW, d, K, H, ord, out);
  AB_LAUNCH_CHECK();
  return 0;
}

extern "C" int atomai_b200_decomp_ica_step(const float* X1, int N, int K, const double* W,
                                           double* out, void* stream) {
  AB_CHECK(N >= 1 && K >= 1 && K <= kMaxK, "decomp_ica_step: N=%d K=%d (<= %d)", N, K, kMaxK);
  AB_CHECK(X1 && W && out, "decomp_ica_step: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int KP = kp_of(K);
  const int64_t grid = (N + kIcaChunk - 1) / kIcaChunk;
  Ordered ord;
  if (ab_ordered_ws(st, grid * (K * K + K), 1, &ord)) return 1;
  if (KP == 16) AB_DYN_LAUNCH(ica_step_kernel<16>, ica_smem_bytes<16>(), grid, X1, N, K, W, ord, out);
  else if (KP == 32) AB_DYN_LAUNCH(ica_step_kernel<32>, ica_smem_bytes<32>(), grid, X1, N, K, W, ord, out);
  else AB_DYN_LAUNCH(ica_step_kernel<64>, ica_smem_bytes<64>(), grid, X1, N, K, W, ord, out);
  AB_LAUNCH_CHECK();
  return 0;
}
