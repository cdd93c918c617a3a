// imgen.cu — lattice masks of utils.imgen: every atom writes a template (the class's mask, pre-cast
// on the host to the output dtype) into its slice of a frame, and the last atom in input order
// wins over its whole slice, zero corners included.
//
//   owner   one warp per atom: atomicMax(owner[frame][ch][row][col], atom + 1) over the atom's
//           clamped slice.  An integer max does not depend on the order of the atomics, so the
//           owner of every pixel (0: none) is independent of the launch configuration.
//   fill    one thread per pixel of a frame (grid.y = frame): every class channel gets the bits of
//           its owner's template element, or zero; with `background` the output is float64 with
//           one more channel, 1 - the class channels summed in numpy's pairwise order (any count), and every
//           negative value clamped to 0.
//
// A template is read as tpl[off + (row - r0) * sr + (col - c0) * sc]: a stride of 0 broadcasts a
// template axis of length 1 over the slice, as numpy's assignment does.
#include "common.cuh"

namespace {

constexpr int kT = 256;
constexpr int kAtomInts = AB_IMGEN_ATOM_INTS;
constexpr int kFrameInts = AB_IMGEN_FRAME_INTS;
constexpr int kPairwiseBlock = 128;   // numpy's PW_BLOCKSIZE
constexpr int kPairwiseDepth = 32;    // > log2(INT_MAX / 64): every split leaves at least 64

__global__ void __launch_bounds__(kT) imgen_owner_kernel(const int32_t* __restrict__ atoms, int K,
                                                         const int64_t* __restrict__ frames,
                                                         int32_t* __restrict__ owner) {
  const int a = blockIdx.x * (kT / 32) + (threadIdx.x >> 5);
  if (a >= K) return;
  const int32_t* at = atoms + (int64_t)a * kAtomInts;
  const int f = at[0], ch = at[1], r0 = at[2], c0 = at[3], nr = at[4], nc = at[5];
  const int64_t* fr = frames + (int64_t)f * kFrameInts;
  const int64_t h = fr[0], w = fr[1];
  int32_t* own = owner + fr[4] + ((int64_t)ch * h + r0) * w + c0;
  for (int e = threadIdx.x & 31; e < nr * nc; e += 32) {
    const int i = e / nc, j = e - i * nc;
    atomicMax(own + i * w + j, a + 1);
  }
}

// T: an unsigned integer of the element's size (the copy is a bit copy); kBackground: T holds
// float64 bits and the frame gets the background channel.
template <typename T, bool kBackground>
__global__ void __launch_bounds__(kT) imgen_fill_kernel(const int32_t* __restrict__ atoms,
                                                        const int64_t* __restrict__ frames,
                                                        const int32_t* __restrict__ owner,
                                                        const T* __restrict__ tpl,
                                                        T* __restrict__ out) {
  const int64_t* fr = frames + (int64_t)blockIdx.y * kFrameInts;
  const int64_t w = fr[1], npix = fr[0] * w;
  const int C = (int)fr[2];
  const int cout = C + (kBackground ? 1 : 0);
  const int32_t* own = owner + fr[4];
  for (int64_t p = blockIdx.x * (int64_t)kT + threadIdx.x; p < npix; p += (int64_t)gridDim.x * kT) {
    const int64_t row = p / w, col = p - row * w;
    T* o = out + fr[3] + p * cout;
    // the class-channel value of this pixel; written (clamped at 0 with a background) on the way
    auto value = [&](int c) -> T {
      const int a = own[c * npix + p];
      T v = 0;
      if (a) {
        const int32_t* at = atoms + (int64_t)(a - 1) * kAtomInts;
        v = tpl[at[6] + (row - at[2]) * at[7] + (col - at[3]) * at[8]];
      }
      if constexpr (kBackground) {
        o[c] = __longlong_as_double((long long)v) < 0.0 ? 0ull : v;
      } else {
        o[c] = v;
      }
      return v;
    };
    if constexpr (!kBackground) {
      for (int c = 0; c < C; ++c) value(c);
    } else {
      // numpy's pairwise sum.  A block of at most 128 values: below 8 a running sum from 0.0;
      // from 8 on, eight accumulators over the whole groups of 8, a fixed tree over them, then the
      // rest in order.  More than 128 values: the sums of two halves split at a multiple of 8,
      // recursively; an explicit stack walks that tree left to right, visiting each channel once.
      auto dv = [&](int c) { return __longlong_as_double((long long)value(c)); };
      auto block = [&](int lo, int n) {
        const int n8 = n >= 8 ? n - n % 8 : 0;
        double t = 0.0;
        if (n8) {
          double r[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) r[j] = dv(lo + j);
          for (int b = 8; b < n8; b += 8) {
#pragma unroll
            for (int j = 0; j < 8; ++j) r[j] += dv(lo + b + j);
          }
          t = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
        }
        for (int c = lo + n8; c < lo + n; ++c) t += dv(c);
        return t;
      };
      auto half = [](int n) { return n / 2 - (n / 2) % 8; };
      double s;
      if (C <= kPairwiseBlock) {
        s = block(0, C);
      } else {
        int slo[kPairwiseDepth], sn[kPairwiseDepth];
        double left[kPairwiseDepth];
        unsigned right = 0;   // bit d: node d has summed its left half
        int d = 0;
        slo[0] = 0;
        sn[0] = C;
        for (;;) {
          for (; sn[d] > kPairwiseBlock; ++d) {
            slo[d + 1] = slo[d];
            sn[d + 1] = half(sn[d]);
            right &= ~(1u << d);
          }
          s = block(slo[d], sn[d]);
          while (d > 0) {
            --d;
            if (!(right >> d & 1u)) {   // left half done: walk the right half next
              left[d] = s;
              right |= 1u << d;
              slo[d + 1] = slo[d] + half(sn[d]);
              sn[d + 1] = sn[d] - half(sn[d]);
              ++d;
              break;
            }
            s = left[d] + s;
          }
          if (d == 0) break;
        }
      }
      const double bg = 1.0 - s;
      o[C] = bg < 0.0 ? 0ull : (T)__double_as_longlong(bg);
    }
  }
}

template <typename T, bool kBackground>
void launch_fill(const int32_t* atoms, const int64_t* frames, int F, int64_t max_pix,
                 const int32_t* owner, const void* tpl, void* out, cudaStream_t st) {
  const dim3 grid(ab_grid(max_pix, kT, 8), F);
  imgen_fill_kernel<T, kBackground><<<grid, kT, 0, st>>>(atoms, frames, owner, (const T*)tpl,
                                                         (T*)out);
}

}  // namespace

extern "C" {

int atomai_b200_imgen_owner(const int32_t* atoms, int K, const int64_t* frames, int32_t* owner,
                            void* stream) {
  AB_CHECK(K >= 0 && (K == 0 || (atoms && frames && owner)), "imgen_owner: bad arguments");
  if (K == 0) return 0;
  const int per = kT / 32;
  imgen_owner_kernel<<<(K + per - 1) / per, kT, 0, (cudaStream_t)stream>>>(atoms, K, frames, owner);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_imgen_fill(const int32_t* atoms, const int64_t* frames, int F, int64_t max_pix,
                           const int32_t* owner, const void* tpl, int elem_bytes, int background,
                           void* out, void* stream) {
  AB_CHECK(frames && owner && out && F > 0 && F <= 65535 && max_pix >= 0,
           "imgen_fill: bad arguments (F=%d)", F);
  AB_CHECK(!background || elem_bytes == 8, "imgen_fill: the background channel needs float64");
  if (max_pix == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  switch (elem_bytes) {
    case 1: launch_fill<uint8_t, false>(atoms, frames, F, max_pix, owner, tpl, out, st); break;
    case 2: launch_fill<uint16_t, false>(atoms, frames, F, max_pix, owner, tpl, out, st); break;
    case 4: launch_fill<uint32_t, false>(atoms, frames, F, max_pix, owner, tpl, out, st); break;
    case 8:
      if (background)
        launch_fill<unsigned long long, true>(atoms, frames, F, max_pix, owner, tpl, out, st);
      else
        launch_fill<unsigned long long, false>(atoms, frames, F, max_pix, owner, tpl, out, st);
      break;
    default: AB_CHECK(false, "imgen_fill: element size %d not in {1, 2, 4, 8}", elem_bytes);
  }
  AB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
