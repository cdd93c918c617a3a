// common.cuh — error plumbing, PTX wrappers (mbarrier / bulk copy) and
// the shared "source loader" used by every convolution-family kernel.
// sm_90a only.  Test infrastructure lives elsewhere; this is product code.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/atomai_b200.h"

// ---------------------------------------------------------------- host errors
void ab_set_error(const char* fmt, ...);
#define AB_CHECK(cond, ...)            \
  do {                                 \
    if (!(cond)) {                     \
      ab_set_error(__VA_ARGS__);       \
      return 1;                        \
    }                                  \
  } while (0)
#define AB_CUDA(expr)                                                              \
  do {                                                                             \
    cudaError_t _e = (expr);                                                       \
    if (_e != cudaSuccess) {                                                       \
      ab_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, \
                   __LINE__);                                                      \
      return 1;                                                                    \
    }                                                                              \
  } while (0)
#define AB_LAUNCH_CHECK() AB_CUDA(cudaGetLastError())

int ab_num_sms();  // cached SM count of the current device
// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is per device: `done` is a per-kernel table
// indexed by the current device (set once per device, benign if two threads race)
int ab_optin_smem(const void* func, int bytes, unsigned char* done);

// ---------------------------------------------------------------- device utils
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ float to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
__device__ __forceinline__ float lrelu_f(float v, float a) { return v > 0.f ? v : v * a; }
// forward activation and its derivative expressed through the OUTPUT value a = act(pre)
// AB_ACT_RBF / AB_ACT_MATERN25: v is a squared scaled distance, slope the outputscale
// (gpytorch RBFKernel / MaternKernel(nu=2.5) under a ScaleKernel, atomai/nets/gp.py:41-46,100-111)
__device__ __forceinline__ float act_f(float v, int act, float slope) {
  if (act == AB_ACT_TANH) return tanhf(v);
  if (act == AB_ACT_RBF) return slope * expf(-0.5f * fmaxf(v, 0.f));
  if (act == AB_ACT_MATERN25) {
    const float d2 = fmaxf(v, 0.f);
    const float s5r = 2.2360679775f * sqrtf(d2);
    return slope * (1.f + s5r + 1.6666666667f * d2) * expf(-s5r);
  }
  return v > 0.f ? v : v * slope;
}
__device__ __forceinline__ float act_grad_from_out(float a, int act, float slope) {
  return act == AB_ACT_TANH ? 1.f - a * a : (a > 0.f ? 1.f : slope);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Counter-based RNG shared by dropout and the Gumbel noise of the joint VAEs: a 64-bit mix of the
// counter and the seed (splitmix64 finaliser), top 24 bits -> uniform in [0, 1)
__device__ __forceinline__ float hash_uniform(uint64_t idx, uint64_t seed) {
  uint64_t z = idx + seed * 0x9E3779B97F4A7C15ull + 0xD1B54A32D192ED03ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (float)(uint32_t)(z >> 40) * (1.0f / 16777216.0f);
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
// try_wait with a suspend-time hint: the hardware parks the thread until the phase completes (or the
// hint expires) instead of returning at once, so a waiting warp does not hammer the shared-memory
// pipe the tensor core reads its operands through.
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity), "r"(200000u)
      : "memory");
  return ok;
}
// Bounded wait: a protocol bug must surface as a trapped launch, never a hung GPU.
__device__ __forceinline__ uint64_t global_timer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  uint64_t t0 = 0;
  while (!mbar_try_wait(bar, parity)) {
    // wall-clock bound (20 s), not a spin count: under a profiler's instrumented replay a healthy
    // kernel can run two orders of magnitude slower, and the suspend hint is only an upper limit
    if ((++spins & 255u) == 0) {
      const uint64_t now = global_timer_ns();
      if (t0 == 0) t0 = now;
      if (now - t0 > 20000000000ull) {
        printf("atomai_b200: mbarrier wait timed out (block %d thread %d bar %u parity %u)\n",
               blockIdx.x, threadIdx.x, bar, parity);
        __trap();
      }
    }
  }
}
// The same bound without the diagnostic printf: a function call between wgmma issue and
// wgmma.wait would make ptxas serialise the warpgroup MMAs.
__device__ __forceinline__ void mbar_wait_quiet(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  uint64_t t0 = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 255u) == 0) {
      const uint64_t now = global_timer_ns();
      if (t0 == 0) t0 = now;
      if (now - t0 > 20000000000ull) __trap();
    }
  }
}
__device__ __forceinline__ void prefetch_l2(const void* p) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// generic-proxy smem writes -> visible to the async proxy (wgmma / bulk copies)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// 1-D bulk copy global -> shared, completion counted on an mbarrier (bytes % 16 == 0)
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes,
                                         uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(dst_smem),
      "l"(src), "r"(bytes), "r"(bar)
      : "memory");
}

// One leader lane of a fully converged warp (the same lane every time): code around it stays
// warp-uniform, so descriptors live in uniform registers and no waterfall loops are generated.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// two floats -> packed bf16x2 (lo half = first argument), round to nearest even
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// ---------------------------------------------------------------- source loader
struct SrcDev {
  const float* ptr;
  const float* scale;
  const float* shift;
  int C;
  int ld;
  int pool;
};
struct SrcSet {
  SrcDev s[2];
  int nsrc;
  int Ctot;
};

// ---- 2x upsampling on load (F.interpolate(scale_factor=2, mode), atomai/nets/blocks.py:130-131,
// fused into the consumer convolution's loader: source code pool = AB_SRC_UP_BILINEAR / _NEAREST,
// the source tensor is (H/2, W/2)).  For output coordinate o of an axis with n_lo low-res samples:
// the two contributing samples and the weight of the second (align_corners = False:
// src = (o + 0.5)/2 - 0.5 clamped at 0 -> even o = 2i: 0.25 x[i-1] + 0.75 x[i], odd: 0.75 x[i] +
// 0.25 x[i+1], edges clamped).
#define AB_SRC_POOL 1
#define AB_SRC_UP_BILINEAR 2
#define AB_SRC_UP_NEAREST 3
__device__ __forceinline__ void up2_coord(int o, int n_lo, bool bilinear, int& i0, int& i1,
                                          float& l1) {
  const int i = o >> 1;
  if (!bilinear) { i0 = i1 = i; l1 = 0.f; return; }
  if (o & 1) { i0 = i; i1 = min(i + 1, n_lo - 1); l1 = 0.25f; }
  else { i0 = max(i - 1, 0); i1 = i; l1 = 0.75f; }     // (o = 0: i0 = i1 = 0, any weight gives x[0])
}
__device__ __forceinline__ float lerp2(float v00, float v01, float v10, float v11, float lh,
                                       float lw) {
  // same association as ATen's upsample_bilinear2d kernel
  return (1.f - lh) * ((1.f - lw) * v00 + lw * v01) + lh * ((1.f - lw) * v10 + lw * v11);
}
__device__ __forceinline__ float4 lerp2_4(float4 a, float4 b, float4 c, float4 d, float lh, float lw) {
  return make_float4(lerp2(a.x, b.x, c.x, d.x, lh, lw), lerp2(a.y, b.y, c.y, d.y, lh, lw),
                     lerp2(a.z, b.z, c.z, d.z, lh, lw), lerp2(a.w, b.w, c.w, d.w, lh, lw));
}
// upsampled value (before the affine) of 4 channels at hi-res pixel (n, h, w) of an H x W grid
__device__ __forceinline__ float4 load_up4(const float* __restrict__ ptr_c, int ld, int mode, int n,
                                           int h, int w, int H, int W) {
  const int Hl = H >> 1, Wl = W >> 1;
  int h0, h1, w0, w1;
  float lh, lw;
  up2_coord(h, Hl, mode == AB_SRC_UP_BILINEAR, h0, h1, lh);
  up2_coord(w, Wl, mode == AB_SRC_UP_BILINEAR, w0, w1, lw);
  const float* r0 = ptr_c + (size_t)(n * Hl + h0) * Wl * ld;
  const float* r1 = ptr_c + (size_t)(n * Hl + h1) * Wl * ld;
  const float4 a = __ldg(reinterpret_cast<const float4*>(r0 + (size_t)w0 * ld));
  if (mode != AB_SRC_UP_BILINEAR) return a;
  const float4 b = __ldg(reinterpret_cast<const float4*>(r0 + (size_t)w1 * ld));
  const float4 c = __ldg(reinterpret_cast<const float4*>(r1 + (size_t)w0 * ld));
  const float4 d = __ldg(reinterpret_cast<const float4*>(r1 + (size_t)w1 * ld));
  return lerp2_4(a, b, c, d, lh, lw);
}

static __device__ __noinline__ float4 load_up4_noinline(const float* __restrict__ ptr_c, int ld, int mode,
                                                 int n, int h, int w, int H, int W) {
  return load_up4(ptr_c, ld, mode, n, h, w, H, W);
}
static __device__ __noinline__ float load_up1_noinline(const float* __restrict__ ptr_c, int ld, int mode,
                                                int n, int h, int w, int H, int W) {
  const int Hl = H >> 1, Wl = W >> 1;
  int h0, h1, w0, w1;
  float lh, lw;
  up2_coord(h, Hl, mode == AB_SRC_UP_BILINEAR, h0, h1, lh);
  up2_coord(w, Wl, mode == AB_SRC_UP_BILINEAR, w0, w1, lw);
  const float* r0 = ptr_c + (size_t)(n * Hl + h0) * Wl * ld;
  const float* r1 = ptr_c + (size_t)(n * Hl + h1) * Wl * ld;
  return lerp2(__ldg(r0 + (size_t)w0 * ld), __ldg(r0 + (size_t)w1 * ld), __ldg(r1 + (size_t)w0 * ld),
               __ldg(r1 + (size_t)w1 * ld), lh, lw);
}

// 4 consecutive channels [c, c+4) of the logical (post-affine, post-pool, zero padded)
// input at pixel (n, h, w) of an H x W grid.  c must be a multiple of 4 and every source's
// C a multiple of 4 on this vector path.
__device__ __forceinline__ float4 load_src4(const SrcSet& S, int n, int h, int w, int H, int W,
                                            int c) {
  float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
  if ((unsigned)h >= (unsigned)H || (unsigned)w >= (unsigned)W) return r;
  const SrcDev* s = &S.s[0];
  if (S.nsrc > 1 && c >= S.s[0].C) {
    s = &S.s[1];
    c -= S.s[0].C;
  }
  float4 sc = make_float4(1.f, 1.f, 1.f, 1.f), sh = make_float4(0.f, 0.f, 0.f, 0.f);
  if (s->scale) {
    sc = __ldg(reinterpret_cast<const float4*>(s->scale + c));
    sh = __ldg(reinterpret_cast<const float4*>(s->shift + c));
  }
  if (s->pool >= AB_SRC_UP_BILINEAR) {
    // out of line: inlined, the four extra loads and the interpolation cost the thin-channel
    // kernels 12-20 registers (conv_pix<16>: 128 -> 148, one CTA per SM instead of two)
    const float4 v = load_up4_noinline(s->ptr + c, s->ld, s->pool, n, h, w, H, W);
    r.x = fmaf(v.x, sc.x, sh.x);
    r.y = fmaf(v.y, sc.y, sh.y);
    r.z = fmaf(v.z, sc.z, sh.z);
    r.w = fmaf(v.w, sc.w, sh.w);
  } else if (!s->pool) {
    const float4 v = __ldg(
        reinterpret_cast<const float4*>(s->ptr + ((size_t)(n * H + h) * W + w) * s->ld + c));
    r.x = fmaf(v.x, sc.x, sh.x);
    r.y = fmaf(v.y, sc.y, sh.y);
    r.z = fmaf(v.z, sc.z, sh.z);
    r.w = fmaf(v.w, sc.w, sh.w);
  } else {
    const int H2 = 2 * H, W2 = 2 * W;
    const float* base = s->ptr + ((size_t)(n * H2 + 2 * h) * W2 + 2 * w) * s->ld + c;
    const float4 v0 = __ldg(reinterpret_cast<const float4*>(base));
    const float4 v1 = __ldg(reinterpret_cast<const float4*>(base + s->ld));
    const float4 v2 = __ldg(reinterpret_cast<const float4*>(base + (size_t)W2 * s->ld));
    const float4 v3 = __ldg(reinterpret_cast<const float4*>(base + (size_t)W2 * s->ld + s->ld));
    r.x = fmaxf(fmaxf(fmaf(v0.x, sc.x, sh.x), fmaf(v1.x, sc.x, sh.x)),
                fmaxf(fmaf(v2.x, sc.x, sh.x), fmaf(v3.x, sc.x, sh.x)));
    r.y = fmaxf(fmaxf(fmaf(v0.y, sc.y, sh.y), fmaf(v1.y, sc.y, sh.y)),
                fmaxf(fmaf(v2.y, sc.y, sh.y), fmaf(v3.y, sc.y, sh.y)));
    r.z = fmaxf(fmaxf(fmaf(v0.z, sc.z, sh.z), fmaf(v1.z, sc.z, sh.z)),
                fmaxf(fmaf(v2.z, sc.z, sh.z), fmaf(v3.z, sc.z, sh.z)));
    r.w = fmaxf(fmaxf(fmaf(v0.w, sc.w, sh.w), fmaf(v1.w, sc.w, sh.w)),
                fmaxf(fmaf(v2.w, sc.w, sh.w), fmaf(v3.w, sc.w, sh.w)));
  }
  return r;
}

// scalar variant (any channel count; used by the exact-fp32 kernels for odd C)
__device__ __forceinline__ float load_src1(const SrcSet& S, int n, int h, int w, int H, int W,
                                           int c) {
  if ((unsigned)h >= (unsigned)H || (unsigned)w >= (unsigned)W) return 0.f;
  const SrcDev* s = &S.s[0];
  if (S.nsrc > 1 && c >= S.s[0].C) {
    s = &S.s[1];
    c -= S.s[0].C;
  }
  float sc = 1.f, sh = 0.f;
  if (s->scale) {
    sc = __ldg(s->scale + c);
    sh = __ldg(s->shift + c);
  }
  if (s->pool >= AB_SRC_UP_BILINEAR)
    return fmaf(load_up1_noinline(s->ptr + c, s->ld, s->pool, n, h, w, H, W), sc, sh);
  if (!s->pool) {
    return fmaf(__ldg(s->ptr + ((size_t)(n * H + h) * W + w) * s->ld + c), sc, sh);
  }
  const int H2 = 2 * H, W2 = 2 * W;
  const float* base = s->ptr + ((size_t)(n * H2 + 2 * h) * W2 + 2 * w) * s->ld + c;
  const float v0 = fmaf(__ldg(base), sc, sh), v1 = fmaf(__ldg(base + s->ld), sc, sh);
  const float v2 = fmaf(__ldg(base + (size_t)W2 * s->ld), sc, sh);
  const float v3 = fmaf(__ldg(base + (size_t)W2 * s->ld + s->ld), sc, sh);
  return fmaxf(fmaxf(v0, v1), fmaxf(v2, v3));
}

int ab_make_srcset(const ab_conv_t* d, SrcSet* out);  // validates + converts (host)

// ---------------------------------------------------------------- ordered cross-CTA sums
// Run-to-run deterministic replacement for "one atomicAdd per CTA (or warp) and value": floating-
// point addition is not associative, so sums whose order depends on which CTA finishes first
// differ in the last bits from run to run, and training (Adam on gradients that are pure rounding,
// e.g. a conv bias in front of BatchNorm) amplifies that.  Instead every contributing slot stores
// its n partials; the last CTA to finish adds all slots in slot order and adds the result to dst.
struct Ordered {
  double* slots;     // [groups][slots per group][n]
  unsigned* ticket;  // [groups], zero between launches
};
// host: workspace of the current device and `stream` for `n_doubles` partials and `groups`
// tickets (thread-safe; launches on other streams use other workspaces)
int ab_ordered_ws(cudaStream_t stream, int64_t n_doubles, int groups, Ordered* out);
__device__ __forceinline__ double* ordered_slot(const Ordered& o, int group, int nslots, int slot,
                                                int n) {
  return o.slots + ((size_t)group * nslots + slot) * n;
}
// Called by all `nt` threads (index t) of the CTA's participating group after its partials are
// stored; bar() synchronises that group; add(i, sum) receives the ordered total of value i.
template <class Bar, class Add>
__device__ __forceinline__ void ordered_finish(const Ordered& o, int group, int nslots, int n,
                                               int t, int nt, int nctas, Bar bar, Add add,
                                               unsigned* s_flag) {
  __threadfence();
  bar();
  if (t == 0) *s_flag = atomicAdd(o.ticket + group, 1u) == (unsigned)nctas - 1u;
  bar();
  if (*s_flag) {
    __threadfence();
    const double* base = o.slots + (size_t)group * nslots * n;
    for (int i = t; i < n; i += nt) {
      double sum = 0.0;
      for (int s = 0; s < nslots; ++s) sum += __ldcg(base + (size_t)s * n + i);
      add(i, sum);
    }
    if (t == 0) o.ticket[group] = 0u;
  }
}
