// wgrad_tc.cu — convolution weight gradient on the Hopper tensor cores (wgmma, TF32 operands, fp32
// accumulators in registers).
//
//   dW[co][ci][ty][tx] = sum_p dy[p][co] * x[p + (ty, tx) * dil][ci]        (SURVEY.md §2.4 K7)
//
// The reduction (GEMM K) runs over pixels.  wgmma reads 32-bit operands K-major only, so the
// loaders transpose the channel-contiguous NHWC data while they stage it: a tile of 64 pixels
// (8 x 8) becomes, per operand, rows = channels with the pixels along K, stored as no-swizzle core
// matrices (8 rows x 4 pixels, LBO = 128 B between neighbouring pixel quads, SBO = one padded
// 8-row group).  One CTA is one warpgroup and owns one tap, one block of 64 output channels (M),
// one block of CIB input channels (N) and a contiguous range of pixel tiles; the x tile it stages
// is already shifted by its tap, so every tap is the same GEMM D[co][ci] += dy^T x over the range.
// The accumulators are flushed once into dW (OIHW), summed over the ranges in a fixed order.
// Staging of tile i + 1 (global loads, TF32 rounding, x3 split) overlaps the MMAs of tile i through a two-stage ring.
//
// Replaces autograd's cuDNN bwd-filter behind loss.backward(), atomai/trainers/trainer.py:206.
#include <cstdlib>
#include "common.cuh"
#include "wgmma.cuh"

namespace {

constexpr int kTile = 8;                      // 8 x 8 pixel tiles: K = 64 per stage
constexpr int kPix = kTile * kTile;
constexpr int kThreads = 128;                 // one warpgroup
constexpr int kM = 64;                        // output channels per CTA (wgmma M)
constexpr int kSbo = (kPix / 4) * 128 + 32;   // one 8-row group: 16 pixel quads, padded (bank spread)

struct WgradTcParams {
  SrcSet S;
  int N, H, W, Cout, Cin;
  int taps_h, taps_w, dil;
  const float* dy;
  int ld_dy;
  float* dw;
  int tiles_h, tiles_w, num_tiles;
  int cib;               // input channels per CTA (wgmma N: 16, 32 or 64)
  int n_cib, n_cob;      // input / output channel blocks
  int ranges;            // pixel-tile ranges per (tap, co block, ci block)
  int a_bytes, b_bytes;  // one operand part (dy^T / x^T) of a stage
  int stage_bytes;       // [dy_hi][x_hi] (x3: [dy_hi][dy_lo][x_hi][x_lo])
  int x3;                // AB_MATH_TF32X3: every value split into rn_tf32(v) and the exact remainder;
                         // per k-step the pairs (hi, hi), (lo, hi), (hi, lo) are issued
  Ordered red;           // per (tap, channel block pair): ordered sum of the ranges' partial dW
};

// RN-to-TF32: the tensor core reads the upper 19 bits only (see conv_tc.cu tf32_bits)
__device__ __forceinline__ uint32_t tf32b(float x) { return __float_as_uint(x) + 0x1000u; }
__device__ __forceinline__ float lo_part(float x) {
  return x - __uint_as_float(tf32b(x) & 0xFFFFE000u);
}
// byte offset of (row r, pixel k) in the K-major core-matrix layout of one operand part
__device__ __forceinline__ uint32_t kmaj_off(int r, int k) {
  return (uint32_t)((r >> 3) * kSbo + (k >> 2) * 128 + (r & 7) * 16 + (k & 3) * 4);
}
// 4 consecutive channels (rows r0..r0+3) of pixel k: hi part, and the lo part at +lo_off (x3)
__device__ __forceinline__ void put4(uint32_t base, int r0, int k, float4 v, bool x3, uint32_t lo_off) {
  const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t a = base + kmaj_off(r0 + i, k);
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(tf32b(e[i])) : "memory");
    if (x3) asm volatile("st.shared.b32 [%0], %1;" ::"r"(a + lo_off), "r"(tf32b(lo_part(e[i]))) : "memory");
  }
}

template <int CIB>
__global__ void __launch_bounds__(kThreads) wgrad_tc_kernel(const WgradTcParams p) {
  constexpr int R = CIB / 2;
  constexpr int QX = CIB / 4;                 // x quads per pixel
  constexpr int ND = kPix * (kM / 4) / kThreads;   // dy float4 per thread per tile (8)
  constexpr int NX = kPix * QX / kThreads;         // x float4 per thread per tile (2..8)
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x;

  // grid: x = pixel range, y = (tap, co block, ci block)
  int blk = blockIdx.y;
  const int cbi = blk % p.n_cib; blk /= p.n_cib;
  const int cob = blk % p.n_cob; blk /= p.n_cob;
  const int t = blk;
  const int ty = t / p.taps_w, tx = t - ty * p.taps_w;
  const int co0 = cob * kM, ci0 = cbi * CIB;
  const int dh = (ty - (p.taps_h >> 1)) * p.dil, dwo = (tx - (p.taps_w >> 1)) * p.dil;
  const int t_begin = (int)((int64_t)p.num_tiles * blockIdx.x / p.ranges);
  const int t_end = (int)((int64_t)p.num_tiles * (blockIdx.x + 1) / p.ranges);
  const int tpi = p.tiles_h * p.tiles_w;
  const bool x3 = p.x3 != 0;
  const int H = p.H, W = p.W;
  const uint32_t a_lo = x3 ? (uint32_t)p.a_bytes : 0u;                     // dy_hi -> dy_lo
  const uint32_t b_off = (uint32_t)p.a_bytes * (x3 ? 2 : 1);              // stage -> x_hi
  const uint32_t b_lo = x3 ? (uint32_t)p.b_bytes : 0u;                     // x_hi -> x_lo

  float4 dv[ND], xv[NX];
  auto load = [&](int tile) {
    const int n = tile / tpi, rem = tile - n * tpi;
    const int h0 = (rem / p.tiles_w) * kTile, w0 = (rem % p.tiles_w) * kTile;
#pragma unroll
    for (int i = 0; i < ND; ++i) {
      const int e = tid + kThreads * i;
      const int k = (e >> 6) * 4 + (e & 3), q = (e >> 2) & 15;
      const int gh = h0 + (k >> 3), gw = w0 + (k & 7), co = co0 + 4 * q;
      dv[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (gh < H && gw < W && co < p.Cout)
        dv[i] = __ldg(reinterpret_cast<const float4*>(p.dy + ((size_t)(n * H + gh) * W + gw) * p.ld_dy + co));
    }
#pragma unroll
    for (int i = 0; i < NX; ++i) {
      const int e = tid + kThreads * i;
      const int k = (e / (4 * QX)) * 4 + (e & 3), q = (e >> 2) % QX;
      const int ci = ci0 + 4 * q;
      xv[i] = ci < p.Cin ? load_src4(p.S, n, h0 + (k >> 3) + dh, w0 + (k & 7) + dwo, H, W, ci)
                         : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto store = [&](uint32_t st) {
#pragma unroll
    for (int i = 0; i < ND; ++i) {
      const int e = tid + kThreads * i;
      put4(st, 4 * ((e >> 2) & 15), (e >> 6) * 4 + (e & 3), dv[i], x3, a_lo);
    }
#pragma unroll
    for (int i = 0; i < NX; ++i) {
      const int e = tid + kThreads * i;
      put4(st + b_off, 4 * ((e >> 2) % QX), (e / (4 * QX)) * 4 + (e & 3), xv[i], x3, b_lo);
    }
  };

  float acc[R];
#pragma unroll
  for (int i = 0; i < R; ++i) acc[i] = 0.f;
  const uint64_t tmpl = wgmma_desc(0, 128, kSbo);
  if (t_begin < t_end) load(t_begin);
  int it = 0;
  for (int tile = t_begin; tile < t_end; ++tile, ++it) {
    const uint32_t st = sbase + (uint32_t)(it & 1) * p.stage_bytes;
    store(st);
    fence_proxy_async_smem();
    __syncthreads();
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < kPix / 8; ++ks) {
      const uint32_t a = st + ks * 256, b = st + b_off + ks * 256;
      Wgmma<CIB>::tf32(acc, tmpl | (a >> 4), tmpl | (b >> 4), 1u);
      if (x3) {
        Wgmma<CIB>::tf32(acc, tmpl | ((a + a_lo) >> 4), tmpl | (b >> 4), 1u);
        Wgmma<CIB>::tf32(acc, tmpl | (a >> 4), tmpl | ((b + b_lo) >> 4), 1u);
      }
    }
    wgmma_commit();
    if (tile + 1 < t_end) load(tile + 1);     // global loads in flight while the MMAs run
    wgmma_wait<1>();                           // the group of tile - 1 (the other stage) retired
    __syncthreads();
  }
  wgmma_wait<0>();
  wgmma_fence_regs(acc);
  // this CTA's partial D[64][CIB] (row-major) into its slot; the last range of the group adds the
  // ranges in order into dW
  const int warp = tid >> 5, lane = tid & 31;
  const int taps = p.taps_h * p.taps_w;
  constexpr int n = kM * CIB;
  double* slot = ordered_slot(p.red, blockIdx.y, gridDim.x, blockIdx.x, n);
#pragma unroll
  for (int j = 0; j < R / 4; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < 2; ++e)
        slot[(16 * warp + (lane >> 2) + 8 * h) * CIB + 8 * j + 2 * (lane & 3) + e] = acc[4 * j + 2 * h + e];
  __shared__ unsigned s_last;
  ordered_finish(p.red, blockIdx.y, gridDim.x, n, tid, kThreads, gridDim.x, [] { __syncthreads(); },
                 [&](int i, double v) {
                   const int co = co0 + i / CIB, ci = ci0 + i % CIB;
                   if (co < p.Cout && ci < p.Cin) p.dw[((size_t)co * p.Cin + ci) * taps + t] += (float)v;
                 },
                 &s_last);
}

int wgrad_plan(const ab_conv_t* d, WgradTcParams* p, int* smem_bytes) {
  if (ab_make_srcset(d, &p->S)) return 1;
  p->N = d->N; p->H = d->H; p->W = d->W; p->Cout = d->Cout; p->Cin = p->S.Ctot;
  p->taps_h = d->ks_h; p->taps_w = d->ks_w; p->dil = d->dil;
  p->x3 = d->math == AB_MATH_TF32X3 ? 1 : 0;
  AB_CHECK(d->ks_w <= 4 && d->ks_h <= 4, "wgrad_tc: kernel %dx%d too large", d->ks_h, d->ks_w);
  p->tiles_h = (d->H + kTile - 1) / kTile;
  p->tiles_w = (d->W + kTile - 1) / kTile;
  const int64_t nt = (int64_t)d->N * p->tiles_h * p->tiles_w;
  AB_CHECK(nt < (1ll << 31) / 4096, "wgrad_tc: too many tiles");
  p->num_tiles = (int)nt;
  p->cib = p->Cin <= 16 ? 16 : (p->Cin <= 32 ? 32 : 64);
  p->n_cib = (p->Cin + p->cib - 1) / p->cib;
  p->n_cob = (d->Cout + kM - 1) / kM;
  p->a_bytes = (kM / 8) * kSbo;
  p->b_bytes = (p->cib / 8) * kSbo;
  p->stage_bytes = ((p->a_bytes + p->b_bytes) * (p->x3 ? 2 : 1) + 127) & ~127;
  *smem_bytes = 2 * p->stage_bytes;
  // about six CTAs per SM in total (two waves of the three that fit at N = 64): a CTA is one
  // warpgroup that waits on its own global loads, so latency is hidden by resident CTAs; every
  // CTA keeps at least a few tiles
  const int groups = d->ks_h * d->ks_w * p->n_cob * p->n_cib;
  int ranges = (6 * ab_num_sms() + groups - 1) / groups;
  if (ranges > p->num_tiles / 4) ranges = p->num_tiles / 4;
  if (ranges < 1) ranges = 1;
  p->ranges = ranges;
  return 0;
}

template <int CIB>
int launch(const WgradTcParams& p, int smem, cudaStream_t stream) {
  // opted in once per device for the largest plan of this N (tf32x3 stages), not for the first
  const int max_smem = 2 * ((((kM + CIB) / 8) * kSbo * 2 + 127) & ~127);
  AB_CHECK(smem <= max_smem, "wgrad_tc: %d B of shared memory exceeds the plan bound", smem);
  static unsigned char optin[64];
  if (ab_optin_smem(reinterpret_cast<const void*>(wgrad_tc_kernel<CIB>), max_smem, optin)) return 1;
  const dim3 grid(p.ranges, p.taps_h * p.taps_w * p.n_cob * p.n_cib);
  WgradTcParams q = p;
  if (ab_ordered_ws(stream, (int64_t)grid.x * grid.y * kM * CIB, grid.y, &q.red)) return 1;
  wgrad_tc_kernel<CIB><<<grid, kThreads, smem, stream>>>(q);
  AB_LAUNCH_CHECK();
  return 0;
}

}  // namespace

int ab_wgrad_tc_supported(const ab_conv_t* d) {
  for (int i = 0; i < d->nsrc; ++i) {
    if (d->src[i].C % 4 != 0 || d->src[i].ld % 4 != 0) return 0;
    if (((uintptr_t)d->src[i].ptr & 15) != 0) return 0;
  }
  if (d->Cout % 4 != 0) return 0;
  if (d->ks_w > 4 || d->ks_h > 4) return 0;
  WgradTcParams p;
  int smem = 0;
  if (wgrad_plan(d, &p, &smem)) return 0;
  return 1;
}

int ab_conv_tc_wgrad(const ab_conv_t* d, const float* dy, int ld_dy, float* dw,
                     cudaStream_t stream) {
  WgradTcParams p;
  int smem = 0;
  if (wgrad_plan(d, &p, &smem)) return 1;
  AB_CHECK(((uintptr_t)dy & 15) == 0 && ld_dy % 4 == 0, "wgrad_tc: unaligned dy");
  p.dy = dy; p.ld_dy = ld_dy; p.dw = dw;
  if (p.num_tiles == 0) return 0;
  if (p.cib == 16) return launch<16>(p, smem, stream);
  if (p.cib == 32) return launch<32>(p, smem, stream);
  return launch<64>(p, smem, stream);
}
