// augment.cu — on-the-fly training-data augmentation on the GPU (SURVEY.md §8f rank 3).
// The reference's `datatransform` (atomai/transforms/imaug.py:20-358) loops over the images of
// a batch in numpy/cv2/skimage on the CPU, round-tripping device -> host -> device every step.
// Here the batch never leaves HBM; the reference's sequence
//     min-max normalise -> rotation/flip -> gauss -> jitter -> poisson -> salt&pepper -> blur ->
//     contrast (gamma) -> background -> min-max normalise
// runs as three HBM-bound passes with per-image parameters drawn on the host:
//   pass A  gather (flip / rot90 / per-row jitter roll) + normalise + the three noise models
//   pass B  Gaussian blur (truncate = 4 sigma, reflect boundary like scipy.ndimage) + gamma +
//           additive 2-D Gaussian background + global min / max (atomics)
//   pass C  final min-max normalisation
// Random numbers come from a counter-based hash of (seed, image, pixel): streams differ from
// numpy's by construction (SURVEY.md §8c: stream-level RNG parity is not required); the
// distributions follow skimage.util.random_noise / numpy.random.poisson as the reference uses them.
#include "common.cuh"

namespace {

constexpr int kT = 256;
constexpr int kNP = 16;   // floats per image in the parameter table (see ab_aug_params below)

// per-image parameters (host-drawn): [0] flip type (-1, 0, 1: cv2.flip codes; 2: rot90 ccw;
// 3: rot90 cw; 9: none)  [1] gauss variance (0 = off)  [2] poisson `vals` (0 = off)
// [3] s&p amount (0 = off)  [4] blur sigma (0 = off)  [5] gamma (0 = off)
// [6..10] background: amplitude, x0, y0, a / fwhm^2 * ln2, b / fwhm^2 * ln2   [11] jitter lambda
__device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__device__ __forceinline__ float u01(uint64_t key) {       // (0, 1]
  return ((float)(uint32_t)(mix64(key) >> 40) + 1.0f) * (1.0f / 16777216.0f);
}
__device__ __forceinline__ float normal01(uint64_t key) {
  const float u1 = u01(key), u2 = u01(key ^ 0x9E3779B97F4A7C15ull);
  return sqrtf(-2.f * logf(u1)) * cospif(2.f * u2);
}
// Poisson(lam): Knuth's product method below 30, rounded normal approximation above
__device__ __forceinline__ float poisson(float lam, uint64_t key) {
  if (lam <= 0.f) return 0.f;
  if (lam < 30.f) {
    const float L = expf(-lam);
    float p = 1.f;
    int k = 0;
    do {
      ++k;
      p *= u01(key + (uint64_t)k * 0xD1B54A32D192ED03ull);
    } while (p > L && k < 200);
    return (float)(k - 1);
  }
  return fmaxf(0.f, rintf(lam + sqrtf(lam) * normal01(key)));
}

__global__ void __launch_bounds__(kT) aug_pass_a(const float* __restrict__ x, float* __restrict__ y,
                                                  const int64_t* __restrict__ lab_in,
                                                  int64_t* __restrict__ lab_out,
                                                  const float* __restrict__ prm,
                                                  const int* __restrict__ row_shift, int n, int h,
                                                  int w, float lo, float inv_range, uint64_t seed) {
  const int64_t total = (int64_t)n * h * w;
  for (int64_t e = blockIdx.x * (int64_t)kT + threadIdx.x; e < total; e += (int64_t)gridDim.x * kT) {
    const int i = (int)(e / ((int64_t)h * w));
    const int r = (int)((e / w) % h), c = (int)(e % w);
    const float* P = prm + (int64_t)i * kNP;
    const int ft = (int)P[0];
    // output (r, c) <- source (sr, sc) of the flip / rotation (square images for rot90)
    int sr = r, sc = c;
    if (ft == 0) sr = h - 1 - r;                       // cv2.flip(.., 0): vertical
    else if (ft == 1) sc = w - 1 - c;                  // horizontal
    else if (ft == -1) { sr = h - 1 - r; sc = w - 1 - c; }
    else if (ft == 2) { sr = c; sc = w - 1 - r; }      // ROTATE_90_COUNTERCLOCKWISE
    else if (ft == 3) { sr = h - 1 - c; sc = r; }      // ROTATE_90_CLOCKWISE
    if (lab_out) lab_out[e] = lab_in[((int64_t)i * h + sr) * w + sc];
    // jitter: np.roll(row, z) of the (already flipped) image: out[c] = in[(c - z) mod w]
    int jc = c;
    if (row_shift) {
      const int z = row_shift[(int64_t)i * h + r] % w;
      jc = (c - z + w) % w;
      // the roll applies to the flipped image, so map the rolled column through the flip again
      sr = r; sc = jc;
      if (ft == 0) sr = h - 1 - r;
      else if (ft == 1) sc = w - 1 - jc;
      else if (ft == -1) { sr = h - 1 - r; sc = w - 1 - jc; }
      else if (ft == 2) { sr = jc; sc = w - 1 - r; }
      else if (ft == 3) { sr = h - 1 - jc; sc = r; }
    }
    float v = (x[((int64_t)i * h + sr) * w + sc] - lo) * inv_range;
    const uint64_t key = seed * 0x9E3779B97F4A7C15ull + (uint64_t)e * 4u;
    if (P[1] > 0.f) v = fminf(fmaxf(v + sqrtf(P[1]) * normal01(key), 0.f), 1.f);   // gaussian, clip
    if (P[2] > 0.f) v = poisson(v * P[2], key + 1) / P[2];
    if (P[3] > 0.f) {                                                               // salt & pepper
      const float u = u01(key + 2);
      if (u <= P[3]) v = u01(key + 3) <= 0.5f ? 1.f : 0.f;
    }
    y[e] = v;
  }
}

__device__ __forceinline__ void atomic_minmax(float* mn, float* mx, float v) {
  // values here can be negative (background): order-preserving integer trick
  int* imn = reinterpret_cast<int*>(mn);
  int* imx = reinterpret_cast<int*>(mx);
  if (v >= 0.f) {
    atomicMin(imn, __float_as_int(v));
    atomicMax(imx, __float_as_int(v));
  } else {
    atomicMax(reinterpret_cast<unsigned int*>(imn), __float_as_uint(v));
    atomicMin(reinterpret_cast<unsigned int*>(imx), __float_as_uint(v));
  }
}

__global__ void __launch_bounds__(kT) aug_pass_b(const float* __restrict__ x, float* __restrict__ y,
                                                  const float* __restrict__ prm, int n, int h, int w,
                                                  float* __restrict__ minmax) {
  const int64_t total = (int64_t)n * h * w;
  float lmn = 3.4e38f, lmx = -3.4e38f;
  for (int64_t e = blockIdx.x * (int64_t)kT + threadIdx.x; e < total; e += (int64_t)gridDim.x * kT) {
    const int i = (int)(e / ((int64_t)h * w));
    const int r = (int)((e / w) % h), c = (int)(e % w);
    const float* P = prm + (int64_t)i * kNP;
    const float* img = x + (int64_t)i * h * w;
    float v;
    const float sigma = P[4];
    if (sigma > 0.f) {
      // scipy.ndimage.gaussian_filter: separable kernel, radius int(4 sigma + 0.5), 'reflect'
      const int rad = (int)(4.f * sigma + 0.5f);
      const float inv2 = -0.5f / (sigma * sigma);
      float num = 0.f, den = 0.f;
      for (int dy = -rad; dy <= rad; ++dy) {
        int rr = r + dy;
        while (rr < 0 || rr >= h) rr = rr < 0 ? -rr - 1 : 2 * h - 1 - rr;
        const float wy = expf(inv2 * dy * dy);
        float rown = 0.f, rowd = 0.f;
        for (int dx = -rad; dx <= rad; ++dx) {
          int cc = c + dx;
          while (cc < 0 || cc >= w) cc = cc < 0 ? -cc - 1 : 2 * w - 1 - cc;
          const float wx = expf(inv2 * dx * dx);
          rown = fmaf(wx, img[(int64_t)rr * w + cc], rown);
          rowd += wx;
        }
        num = fmaf(wy, rown / rowd, num);
        den += wy;
      }
      v = num / den;
    } else {
      v = img[(int64_t)r * w + c];
    }
    if (P[5] > 0.f) v = powf(fmaxf(v, 0.f), P[5]);                 // exposure.adjust_gamma
    if (P[6] != 0.f) {                                            // asymmetric 2-D Gaussian
      const float xs = (float)r * ((float)h / (float)(h - 1 > 0 ? h - 1 : 1));   // np.linspace(0, h, h)
      const float ys = (float)c * ((float)w / (float)(w - 1 > 0 ? w - 1 : 1));
      v += P[6] * expf(-(P[9] * (xs - P[7]) * (xs - P[7]) + P[10] * (ys - P[8]) * (ys - P[8])));
    }
    y[e] = v;
    lmn = fminf(lmn, v);
    lmx = fmaxf(lmx, v);
  }
  for (int o = 16; o > 0; o >>= 1) {
    lmn = fminf(lmn, __shfl_xor_sync(0xffffffffu, lmn, o));
    lmx = fmaxf(lmx, __shfl_xor_sync(0xffffffffu, lmx, o));
  }
  if ((threadIdx.x & 31) == 0 && lmn <= lmx) atomic_minmax(minmax, minmax + 1, lmn), atomic_minmax(minmax, minmax + 1, lmx);
}

__global__ void __launch_bounds__(kT) aug_pass_c(float* __restrict__ y, int64_t total,
                                                  const float* __restrict__ minmax) {
  const float lo = minmax[0], inv = 1.f / (minmax[1] - minmax[0]);
  for (int64_t e = blockIdx.x * (int64_t)kT + threadIdx.x; e < total; e += (int64_t)gridDim.x * kT)
    y[e] = (y[e] - lo) * inv;
}

}  // namespace

extern "C" int atomai_b200_augment(const float* x, float* y, float* scratch, const int64_t* lab_in,
                                   int64_t* lab_out, const float* params, const int* row_shift,
                                   int n, int h, int w, float in_min, float in_max, uint64_t seed,
                                   float* minmax, void* stream) {
  AB_CHECK(x && y && scratch && params && minmax && n > 0 && h > 0 && w > 0, "augment: bad arguments");
  AB_CHECK((lab_in == nullptr) == (lab_out == nullptr), "augment: label in/out mismatch");
  AB_CHECK(in_max > in_min, "augment: constant input batch");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t total = (int64_t)n * h * w;
  const float init[2] = {3.4e38f, -3.4e38f};
  AB_CUDA(cudaMemcpyAsync(minmax, init, sizeof(init), cudaMemcpyHostToDevice, st));
  aug_pass_a<<<ab_grid(total, kT, 16), kT, 0, st>>>(x, scratch, lab_in, lab_out, params, row_shift, n, h, w,
                                            in_min, 1.f / (in_max - in_min), seed);
  AB_LAUNCH_CHECK();
  aug_pass_b<<<ab_grid(total, kT, 16), kT, 0, st>>>(scratch, y, params, n, h, w, minmax);
  AB_LAUNCH_CHECK();
  aug_pass_c<<<ab_grid(total, kT, 16), kT, 0, st>>>(y, total, minmax);
  AB_LAUNCH_CHECK();
  return 0;
}
