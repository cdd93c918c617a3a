// fft.cu — float64 complex 2-D FFTs for utils.FFTmask / FFTsub (atomai/utils/img.py:455-486).
//
// A 2-D transform of an (h, w) image runs as four passes on the caller's stream:
//   rows    fft_rows_kernel: the w-point transform of each of the h rows, in shared memory,
//           fused with the load (dtype promotion to complex double, or the ifftshift of a spectrum)
//   T       fft_transpose_kernel: a 32 x 32-tiled transpose of the (h, w) workspace to (w, h)
//   rows    fft_rows_kernel again: the h-point transform of each of the w rows, in place
//   store   fft_transpose_kernel back to (h, w), fused with the endpoint: fftshift, the disk
//           mask and the complex64 rounding of FFTmask's F2 and F3 (written from the same read),
//           or FFTsub's |src - Re(recon)| with each tile's float64 min and max
// FFTsub then reduces the tile extremes in one CTA and normalises in a last elementwise pass:
// no atomics anywhere, so repeated calls give identical bits.
//
// Every row transform is a power-of-two radix-2 transform of L points in shared memory (one row
// per CTA at a time).  A length n that is not a power of two runs by Bluestein's chirp-z method
// through the same code with L = next_pow2(2n - 1): x[k] w[k] is convolved with conj(w) by two
// L-point transforms, w[k] = exp(-i pi k^2 / n).  The inverse transform is conj(F(conj(x))), the
// forward transform with conjugate twiddles; its 1 / (h w) scale is applied at the store.
// Twiddles exp(-2 pi i t / Lmax) and chirps are computed with sincospi of exactly reduced
// arguments: t / Lmax is exact, and k^2 is reduced mod 2n in integers before the division.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace {

constexpr int kRowThreads = 512;
constexpr int kTile = 32;
constexpr int kTileRows = 8;
constexpr int kReduceThreads = 1024;

__device__ __forceinline__ double2 cmul(double2 a, double2 b) {
  return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
__device__ __forceinline__ double2 cconj(double2 a) { return make_double2(a.x, -a.y); }

// element i of a row-major array of dtype `code`, as complex double (exact for every code)
__device__ __forceinline__ double2 load_c(const void* p, int code, int64_t i) {
  switch (code) {
    case AB_FFT_U8: return make_double2((double)((const uint8_t*)p)[i], 0.0);
    case AB_FFT_I8: return make_double2((double)((const int8_t*)p)[i], 0.0);
    case AB_FFT_I16: return make_double2((double)((const int16_t*)p)[i], 0.0);
    case AB_FFT_U16: return make_double2((double)((const uint16_t*)p)[i], 0.0);
    case AB_FFT_I32: return make_double2((double)((const int32_t*)p)[i], 0.0);
    case AB_FFT_U32: return make_double2((double)((const uint32_t*)p)[i], 0.0);
    case AB_FFT_I64: return make_double2((double)((const int64_t*)p)[i], 0.0);
    case AB_FFT_U64: return make_double2((double)((const uint64_t*)p)[i], 0.0);
    case AB_FFT_F16: return make_double2((double)__half2float(((const __half*)p)[i]), 0.0);
    case AB_FFT_F32: return make_double2((double)((const float*)p)[i], 0.0);
    case AB_FFT_F64: return make_double2(((const double*)p)[i], 0.0);
    case AB_FFT_C64: {
      const float2 v = ((const float2*)p)[i];
      return make_double2((double)v.x, (double)v.y);
    }
    default: return ((const double2*)p)[i];
  }
}

__device__ __forceinline__ unsigned brev_idx(unsigned k, int log2L) {
  return log2L ? __brev(k) >> (32 - log2L) : 0u;
}

// in-place radix-2 decimation-in-time transform of s[0, L) (input in bit-reversed order, output
// in natural order); tw[t] = exp(-2 pi i t / Lmax), t < Lmax / 2.  Synchronises before and after.
__device__ void fft_pow2(double2* s, int L, const double2* __restrict__ tw, int Lmax) {
  for (int half = 1; half < L; half <<= 1) {
    __syncthreads();
    const int step = Lmax / (2 * half);
    for (int b = threadIdx.x; b < L / 2; b += blockDim.x) {
      const int j = b & (half - 1);
      const int i0 = ((b - j) << 1) + j, i1 = i0 + half;
      const double2 u = s[i0], v = cmul(s[i1], __ldg(tw + j * step));
      s[i0] = make_double2(u.x + v.x, u.y + v.y);
      s[i1] = make_double2(u.x - v.x, u.y - v.y);
    }
  }
  __syncthreads();
}

// bit-reversal permutation of s[0, L) in place: each pair is swapped by one thread
__device__ void bitrev_swap(double2* s, int L, int log2L) {
  __syncthreads();
  for (int k = threadIdx.x; k < L; k += blockDim.x) {
    const int r = (int)brev_idx((unsigned)k, log2L);
    if (k < r) {
      const double2 t = s[k];
      s[k] = s[r];
      s[r] = t;
    }
  }
}

__global__ void fft_twiddle_kernel(double2* __restrict__ tw, int Lmax) {
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < Lmax / 2; t += gridDim.x * blockDim.x) {
    double sn, cs;
    sincospi(2.0 * t / Lmax, &sn, &cs);   // 2t / Lmax is exact
    tw[t] = make_double2(cs, -sn);
  }
}

// Bluestein tables of length n: chirp[k] = exp(-i pi k^2 / n) (k < n), and bfft = F_L(b) / L of
// b[m] = conj(chirp[|m|]) for |m| < n, laid out circularly in L points.  One CTA.
__global__ void __launch_bounds__(kRowThreads)
    fft_chirp_kernel(int n, int L, int log2L, const double2* __restrict__ tw, int Lmax,
                     double2* __restrict__ chirp, double2* __restrict__ bfft) {
  extern __shared__ double2 s[];
  for (int m = threadIdx.x; m < L; m += blockDim.x) {
    const int k = m < n ? m : (m > L - n ? L - m : -1);
    double2 b = make_double2(0.0, 0.0);
    if (k >= 0) {
      const int64_t q = ((int64_t)k * k) % (2 * (int64_t)n);   // exp(-i pi k^2/n) has period 2n
      double sn, cs;
      sincospi((double)q / n, &sn, &cs);
      b = make_double2(cs, sn);
      if (m < n) chirp[m] = make_double2(cs, -sn);
    }
    s[brev_idx((unsigned)m, log2L)] = b;
  }
  fft_pow2(s, L, tw, Lmax);
  const double inv = 1.0 / L;   // exact: L is a power of two
  for (int m = threadIdx.x; m < L; m += blockDim.x)
    bfft[m] = make_double2(s[m].x * inv, s[m].y * inv);
}

struct RowPass {
  const void* src;   // rows x n elements of dtype `code` (row-major)
  int code;
  int rows, n;
  int row_shift, col_shift;   // element (r, k) loads src[(r + row_shift) % rows][(k + col_shift) % n]
  int inverse;                // conj on load and on store
  int L, log2L, bluestein;
  const double2* tw;
  int Lmax;
  const double2* chirp;
  const double2* bfft;
  double2* dst;               // rows x n complex double; may alias src when code == AB_FFT_C128
};

__global__ void __launch_bounds__(kRowThreads) fft_rows_kernel(RowPass p) {
  extern __shared__ double2 s[];
  const int n = p.n, L = p.L;
  for (int r = blockIdx.x; r < p.rows; r += gridDim.x) {
    __syncthreads();   // the previous row's stores have read s
    const int64_t src_row = (int64_t)((r + p.row_shift) % p.rows) * n;
    for (int k = threadIdx.x; k < L; k += blockDim.x) {
      double2 x = make_double2(0.0, 0.0);
      if (k < n) {
        int c = k + p.col_shift;
        if (c >= n) c -= n;
        x = load_c(p.src, p.code, src_row + c);
        if (p.inverse) x = cconj(x);
        if (p.bluestein) x = cmul(x, p.chirp[k]);
      }
      s[brev_idx((unsigned)k, p.log2L)] = x;
    }
    fft_pow2(s, L, p.tw, p.Lmax);
    if (p.bluestein) {
      // c = conj(F_L(conj(A B / L))): the inverse transform of the product, by the forward one
      for (int k = threadIdx.x; k < L; k += blockDim.x) s[k] = cconj(cmul(s[k], p.bfft[k]));
      bitrev_swap(s, L, p.log2L);
      fft_pow2(s, L, p.tw, p.Lmax);
    }
    double2* out = p.dst + (int64_t)r * n;
    for (int k = threadIdx.x; k < n; k += blockDim.x) {
      double2 y = s[k];
      if (p.bluestein) y = cmul(cconj(y), p.chirp[k]);
      out[k] = p.inverse ? cconj(y) : y;
    }
  }
}

enum StoreMode { kPlain = 0, kMask = 1, kSub = 2 };

struct TransposePass {
  const double2* src;   // R x C complex double
  int R, C;
  double2* dst;         // kPlain: C x R complex double
  // kMask: src is the (w, h) spectrum; (i, j) = ((q + h/2) % h, (p + w/2) % w) of the (h, w)
  // outputs, F3 = F2 * (1 - disk) inside the box [r0, r0 + 2l) x [c0, c0 + 2l)
  void* f2;
  void* f3;
  int c64, r0, c0, l;
  // kSub: src is the (w, h) inverse without its scale; d = |img - Re(src) * scale| into diff
  const void* img;
  int img_code;
  double scale;
  double* diff;
  double2* tile_minmax;   // one {min, max} per tile
};

// NaN-propagating extremes, like numpy's amin / amax
__device__ __forceinline__ double nan_min(double a, double b) { return (b < a || b != b) ? b : a; }
__device__ __forceinline__ double nan_max(double a, double b) { return (b > a || b != b) ? b : a; }

template <int MODE>
__global__ void __launch_bounds__(kTile * kTileRows) fft_transpose_kernel(TransposePass t) {
  __shared__ double2 tile[kTile][kTile + 1];
  __shared__ double2 red[kTile * kTileRows / 32];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int tiles_c = (t.C + kTile - 1) / kTile;
  const int p0 = (blockIdx.x / tiles_c) * kTile, q0 = (blockIdx.x % tiles_c) * kTile;
  for (int rr = ty; rr < kTile; rr += kTileRows) {
    const int p = p0 + rr, q = q0 + tx;
    if (p < t.R && q < t.C) tile[rr][tx] = t.src[(int64_t)p * t.C + q];
  }
  __syncthreads();
  double mn = __longlong_as_double(0x7ff0000000000000ll), mx = -mn;   // +inf, -inf
  for (int cc = ty; cc < kTile; cc += kTileRows) {
    const int q = q0 + cc, p = p0 + tx;   // output (q, p) = src (p, q)
    if (q >= t.C || p >= t.R) continue;
    const double2 v = tile[tx][cc];
    if (MODE == kPlain) {
      t.dst[(int64_t)q * t.R + p] = v;
    } else if (MODE == kMask) {
      // src is (w, h): p runs over the w axis, q over the h axis
      const int h = t.C, w = t.R;
      int i = q + h / 2, j = p + w / 2;
      if (i >= h) i -= h;
      if (j >= w) j -= w;
      double2 g = v;
      const int y = i - t.r0, x = j - t.c0;
      if (y >= 0 && y < 2 * t.l && x >= 0 && x < 2 * t.l) {
        const int64_t dy = y + 1 - t.l, dx = x + 1 - t.l;
        const double keep = (dx * dx + dy * dy <= (int64_t)t.l * t.l) ? 0.0 : 1.0;
        g = cmul(v, make_double2(keep, 0.0));   // numpy's F3 * (1 - mask), NaN and signs included
      }
      const int64_t o = (int64_t)i * w + j;
      if (t.c64) {
        ((float2*)t.f2)[o] = make_float2((float)v.x, (float)v.y);
        ((float2*)t.f3)[o] = make_float2((float)g.x, (float)g.y);
      } else {
        ((double2*)t.f2)[o] = v;
        ((double2*)t.f3)[o] = g;
      }
    } else {
      const int w = t.R;
      const int64_t o = (int64_t)q * w + p;
      const double2 a = load_c(t.img, t.img_code, o);
      const double d = hypot(a.x - v.x * t.scale, a.y);
      t.diff[o] = d;
      mn = nan_min(mn, d);
      mx = nan_max(mx, d);
    }
  }
  if (MODE == kSub) {
    for (int off = 16; off; off >>= 1) {
      mn = nan_min(mn, __shfl_xor_sync(0xffffffffu, mn, off));
      mx = nan_max(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    }
    const int warp = (ty * kTile + tx) / 32;
    if (tx % 32 == 0) red[warp] = make_double2(mn, mx);
    __syncthreads();
    if (ty == 0 && tx == 0) {
      double2 m = red[0];
      for (int k = 1; k < kTile * kTileRows / 32; ++k)
        m = make_double2(nan_min(m.x, red[k].x), nan_max(m.y, red[k].y));
      t.tile_minmax[blockIdx.x] = m;
    }
  }
}

// {min, max} over the tiles' extremes, one CTA; exact, so independent of the order
__global__ void __launch_bounds__(kReduceThreads)
    fft_minmax_kernel(const double2* __restrict__ part, int n, double2* __restrict__ out) {
  __shared__ double2 red[kReduceThreads / 32];
  double mn = __longlong_as_double(0x7ff0000000000000ll), mx = -mn;
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    mn = nan_min(mn, part[k].x);
    mx = nan_max(mx, part[k].y);
  }
  for (int off = 16; off; off >>= 1) {
    mn = nan_min(mn, __shfl_xor_sync(0xffffffffu, mn, off));
    mx = nan_max(mx, __shfl_xor_sync(0xffffffffu, mx, off));
  }
  if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = make_double2(mn, mx);
  __syncthreads();
  if (threadIdx.x == 0) {
    double2 m = red[0];
    for (int k = 1; k < kReduceThreads / 32; ++k)
      m = make_double2(nan_min(m.x, red[k].x), nan_max(m.y, red[k].y));
    *out = m;
  }
}

// out = (d - min) / (max - min), numpy's (diff - amin) / amax(diff - amin) in float64
template <typename O>
__global__ void fft_normalise_kernel(const double* __restrict__ diff, int64_t n,
                                     const double2* __restrict__ minmax, O* __restrict__ out) {
  const double2 m = *minmax;
  const double range = m.y - m.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x)
    out[i] = (O)((diff[i] - m.x) / range);
}

int log2_of(int L) {
  int k = 0;
  while ((1 << k) < L) ++k;
  return k;
}
bool is_pow2(int n) { return n > 0 && (n & (n - 1)) == 0; }
int transform_len(int n) { return is_pow2(n) ? n : 1 << log2_of(2 * n - 1); }
bool side_ok(int n) { return n >= 1 && (n <= AB_FFT_MAX_SIDE || (is_pow2(n) && n <= AB_FFT_MAX_POW2)); }
int64_t align256(int64_t b) { return (b + 255) & ~(int64_t)255; }

// workspace carve-up: two (h, w) complex double planes, twiddles, the Bluestein tables of both
// sides, the tile extremes and the global extremes
struct Work {
  double2 *a, *b, *tw, *chirp_w, *bfft_w, *chirp_h, *bfft_h, *part, *minmax;
};

int64_t carve(int h, int w, char* base, Work* o) {
  const int Lw = transform_len(w), Lh = transform_len(h), Lmax = Lw > Lh ? Lw : Lh;
  const int64_t tiles = (int64_t)((h + kTile - 1) / kTile) * ((w + kTile - 1) / kTile);
  const int64_t n[9] = {(int64_t)h * w, (int64_t)h * w, Lmax / 2 > 0 ? Lmax / 2 : 1,
                        is_pow2(w) ? 0 : w, is_pow2(w) ? 0 : Lw, is_pow2(h) ? 0 : h,
                        is_pow2(h) ? 0 : Lh, tiles, 1};
  double2** slot[9] = {&o->a, &o->b, &o->tw, &o->chirp_w, &o->bfft_w, &o->chirp_h, &o->bfft_h,
                       &o->part, &o->minmax};
  int64_t off = 0;
  for (int k = 0; k < 9; ++k) {
    if (base) *slot[k] = n[k] ? (double2*)(base + off) : nullptr;
    off += align256(n[k] * (int64_t)sizeof(double2));
  }
  return off;
}

int run_rows(RowPass p, cudaStream_t st) {
  static unsigned char optin[64];
  const int smem = p.L * (int)sizeof(double2);
  if (smem > 48 * 1024 &&
      ab_optin_smem(reinterpret_cast<const void*>(fft_rows_kernel),
                    AB_FFT_MAX_POW2 * (int)sizeof(double2), optin))
    return 1;
  const int per_sm = smem > 0 ? (200 * 1024) / smem : 8;
  fft_rows_kernel<<<ab_grid(p.rows, 1, per_sm < 1 ? 1 : (per_sm > 8 ? 8 : per_sm)), kRowThreads,
                    smem, st>>>(p);
  AB_LAUNCH_CHECK();
  return 0;
}

int run_chirp(int n, const Work& wk, int Lmax, double2* chirp, double2* bfft, cudaStream_t st) {
  static unsigned char optin[64];
  const int L = transform_len(n), smem = L * (int)sizeof(double2);
  if (smem > 48 * 1024 &&
      ab_optin_smem(reinterpret_cast<const void*>(fft_chirp_kernel),
                    AB_FFT_MAX_POW2 * (int)sizeof(double2), optin))
    return 1;
  fft_chirp_kernel<<<1, kRowThreads, smem, st>>>(n, L, log2_of(L), wk.tw, Lmax, chirp, bfft);
  AB_LAUNCH_CHECK();
  return 0;
}

// the transform of an (h, w) array, leaving the (w, h) transposed spectrum in wk.b: spectrum
// (kr, kc) at wk.b[kc * h + kr].  `inverse` conjugates the twiddles (no scale);
// the first pass loads src[(r + row_shift) % h][(k + col_shift) % w].
int fft2_passes(const void* src, int code, int h, int w, int row_shift, int col_shift,
                int inverse, const Work& wk, cudaStream_t st) {
  const int Lw = transform_len(w), Lh = transform_len(h), Lmax = Lw > Lh ? Lw : Lh;
  fft_twiddle_kernel<<<(Lmax / 2 + 255) / 256 + 1, 256, 0, st>>>(wk.tw, Lmax);
  AB_LAUNCH_CHECK();
  if (!is_pow2(w) && run_chirp(w, wk, Lmax, wk.chirp_w, wk.bfft_w, st)) return 1;
  if (!is_pow2(h) && run_chirp(h, wk, Lmax, wk.chirp_h, wk.bfft_h, st)) return 1;
  RowPass p{src, code, h, w, row_shift, col_shift, inverse, Lw, log2_of(Lw), !is_pow2(w),
            wk.tw, Lmax, wk.chirp_w, wk.bfft_w, wk.a};
  if (run_rows(p, st)) return 1;
  TransposePass t{};
  t.src = wk.a;
  t.R = h;
  t.C = w;
  t.dst = wk.b;
  const int64_t tiles = (int64_t)((h + kTile - 1) / kTile) * ((w + kTile - 1) / kTile);
  fft_transpose_kernel<kPlain><<<(unsigned)tiles, dim3(kTile, kTileRows), 0, st>>>(t);
  AB_LAUNCH_CHECK();
  RowPass q{wk.b, AB_FFT_C128, w, h, 0, 0, inverse, Lh, log2_of(Lh), !is_pow2(h),
            wk.tw, Lmax, wk.chirp_h, wk.bfft_h, wk.b};
  return run_rows(q, st);
}

int check_args(const char* what, int h, int w, int code, void* work, int64_t work_bytes) {
  AB_CHECK(side_ok(h) && side_ok(w),
           "%s: sides must be in [1, %d] or powers of two up to %d, got %d x %d", what,
           AB_FFT_MAX_SIDE, AB_FFT_MAX_POW2, h, w);
  AB_CHECK(code >= AB_FFT_U8 && code <= AB_FFT_C128, "%s: dtype code %d", what, code);
  AB_CHECK(work && work_bytes >= carve(h, w, nullptr, nullptr),
           "%s: workspace of %lld bytes, %lld needed", what, (long long)work_bytes,
           (long long)carve(h, w, nullptr, nullptr));
  return 0;
}

}  // namespace

extern "C" {

int64_t atomai_b200_fft2_workspace_bytes(int h, int w) {
  if (!side_ok(h) || !side_ok(w)) return -1;
  return carve(h, w, nullptr, nullptr);
}

int atomai_b200_fft2_mask(const void* img, int dtype, int h, int w, int r0, int c0, int l,
                          void* f2, void* f3, int c64, void* work, int64_t work_bytes,
                          void* stream) {
  if (check_args("fft2_mask", h, w, dtype, work, work_bytes)) return 1;
  AB_CHECK(img && f2 && f3, "fft2_mask: null pointer");
  AB_CHECK(l >= 0 && l <= 4096, "fft2_mask: mask half-width %d", l);
  cudaStream_t st = (cudaStream_t)stream;
  Work wk;
  carve(h, w, (char*)work, &wk);
  if (fft2_passes(img, dtype, h, w, 0, 0, 0, wk, st)) return 1;
  TransposePass t{};
  t.src = wk.b;
  t.R = w;
  t.C = h;
  t.f2 = f2;
  t.f3 = f3;
  t.c64 = c64;
  t.r0 = r0;
  t.c0 = c0;
  t.l = l;
  const int64_t tiles = (int64_t)((h + kTile - 1) / kTile) * ((w + kTile - 1) / kTile);
  fft_transpose_kernel<kMask><<<(unsigned)tiles, dim3(kTile, kTileRows), 0, st>>>(t);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_fft2_sub(const void* img, int img_dtype, const void* spec, int spec_dtype, int h,
                         int w, void* out, int out_f32, void* work, int64_t work_bytes,
                         void* stream) {
  if (check_args("fft2_sub", h, w, img_dtype, work, work_bytes)) return 1;
  AB_CHECK(spec_dtype == AB_FFT_C64 || spec_dtype == AB_FFT_C128,
           "fft2_sub: spectrum dtype code %d", spec_dtype);
  AB_CHECK(img && spec && out, "fft2_sub: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  Work wk;
  carve(h, w, (char*)work, &wk);
  // the ifftshift is the load's shift by (h/2, w/2)
  if (fft2_passes(spec, spec_dtype, h, w, h / 2, w / 2, 1, wk, st)) return 1;
  TransposePass t{};
  t.src = wk.b;
  t.R = w;
  t.C = h;
  t.img = img;
  t.img_code = img_dtype;
  t.scale = 1.0 / ((double)h * (double)w);
  t.diff = (double*)wk.a;
  t.tile_minmax = wk.part;
  const int64_t tiles = (int64_t)((h + kTile - 1) / kTile) * ((w + kTile - 1) / kTile);
  fft_transpose_kernel<kSub><<<(unsigned)tiles, dim3(kTile, kTileRows), 0, st>>>(t);
  AB_LAUNCH_CHECK();
  fft_minmax_kernel<<<1, kReduceThreads, 0, st>>>(wk.part, (int)tiles, wk.minmax);
  AB_LAUNCH_CHECK();
  const int64_t n = (int64_t)h * w;
  const int grid = ab_grid(n, 256 * 8, 8);
  if (out_f32)
    fft_normalise_kernel<float><<<grid, 256, 0, st>>>((const double*)wk.a, n, wk.minmax, (float*)out);
  else
    fft_normalise_kernel<double><<<grid, 256, 0, st>>>((const double*)wk.a, n, wk.minmax, (double*)out);
  AB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
