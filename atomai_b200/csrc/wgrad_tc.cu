// wgrad_tc.cu — convolution weight gradient on the Hopper tensor cores (wgmma, TF32 operands, fp32
// accumulators in registers).
//
//   dW[co][ci][ty][tx] = sum_p dy[p][co] * x[p + (ty, tx) * dil][ci]        (SURVEY.md §2.4 K7)
//
// The reduction (GEMM K) runs over pixels.  wgmma reads 32-bit operands K-major only, so the
// loaders transpose the channel-contiguous NHWC data while they stage it: a tile of 64 pixels
// (8 x 8) becomes, per operand, rows = channels with the pixels along K, stored as no-swizzle core
// matrices (8 rows x 4 pixels, LBO = 128 B between neighbouring pixel quads, SBO = one padded
// 8-row group).  Pixel k = 8 * row + col, so one k-step (8 pixels) is one image row of the tile.
//
// A work unit is one kernel column tx (all taps_h taps of it, or one tap when the halo would be too
// tall), one block of output and one of input channels, and a contiguous range of pixel tiles.
// dy is staged once per tile; x is staged once per tile as a halo of 8 + dil * (taps_h - 1) rows,
// already shifted by the column's tx * dil, and tap ty reads it from its own start address
// (ty * dil rows = 2 * ty * dil core matrices further along K), so all taps of the column share
// both staged operands and keep one accumulator set each.
// The wider channel side goes on the wgmma M rows: when the output channels are few and the input
// channels more, the unit computes dW^T[ci][co] (A = x^T, B = dy^T) instead of dW[co][ci].
// Each unit's accumulators are flushed once into its per-range slot; wgrad_sum_kernel adds each
// group's slots in range order into dW (OIHW), so the result does not depend on which CTA finishes
// first or on which CTA ran which unit.
//
// A CTA is warp-specialised and loops over work units:
//   warps 0-3  consumer  waits for a full stage, issues every (k-step, tap) MMA of the tile as one
//                        wgmma group, and releases the stage once the next group is committed and
//                        wgmma_wait<1> has retired this one; flushes a unit's accumulators
//   warps 4-7  loaders   global float4 loads -> BN affine / 2x2 max-pool -> RN-to-TF32 (and the lo
//                        part in x3) -> transposing stores into a free stage of the ring
// Stages hand off through per-stage full / empty mbarriers, so the loaders run up to a ring ahead
// of the MMAs and neither side waits at a CTA-wide barrier.
//
// Replaces autograd's cuDNN bwd-filter behind loss.backward(), atomai/trainers/trainer.py:206.
#include <cstdlib>
#include "common.cuh"
#include "wgmma.cuh"

namespace {

constexpr int kTile = 8;                      // 8 x 8 pixel tiles: K = 64 per stage
constexpr int kPix = kTile * kTile;
constexpr int kWg = 128;                      // threads of a warpgroup
constexpr int kThreads = 2 * kWg;             // consumer warpgroup + loader warpgroup
// Two CTAs per SM are launched at 65536 / (2 * 256 threads) = 128 registers; setmaxnreg gives the
// consumer room for its accumulators and the loaders room for a tile of float4s in flight.  The
// widest unit (N = 64, three taps: 3 x 32 accumulators, 18 float4 per loader thread) does not fit
// that split without spills (ptxas, CUDA 12.9), so it runs one CTA per SM at full registers.
constexpr int kRegsCons = 136, kRegsLoad = 120;
static_assert(kRegsCons + kRegsLoad <= 2 * 65536 / (2 * kThreads), "register budget");
__host__ __device__ constexpr int ctas_per_sm(int nb, int th) { return nb == 64 && th == 3 ? 1 : 2; }
constexpr int kM = 64;                        // wgmma M: channels of the M side per unit
constexpr int kMaxDil = 1;                    // column units (TH = 3) up to this dilation: 10 halo rows
                                              // (a taller halo's loads do not fit in registers at N = 64)
constexpr int kMaxStages = 4;
constexpr int kCtlBytes = 128;                // full[kMaxStages], empty[kMaxStages] mbarriers
// shared memory per CTA that lets `ctas` CTAs share an SM (228 KB, 1 KB reserved per CTA)
constexpr int smem_budget(int ctas) { return 228 * 1024 / ctas - 1024; }
// SBO of an operand part spanning `rows` pixel rows (two 16-B pixel quads per row): one 8-row
// group, padded by 32 B (bank spread)
__host__ __device__ constexpr int sbo_bytes(int rows) { return rows * 2 * 128 + 32; }

// how the loaders read x: every source plain, every source 2x2 max-pooled, or any other mix
// (upsampling on load) through the general load_src4
enum { kXPlain = 0, kXPool = 1, kXGeneral = 2 };

struct WgradTcParams {
  SrcSet S;
  int N, H, W, Cout, Cin;
  int taps_h, taps_w, dil;
  const float* dy;
  int ld_dy;
  float* dw;
  int tiles_h, tiles_w, num_tiles;
  int th;                // kernel rows per unit: taps_h (one whole kernel column) or 1
  int x_rows;            // pixel rows of the staged x halo: 8 + dil * (th - 1)
  int trans;             // 1: D = dW^T[ci][co] (M = input channels), 0: D = dW[co][ci]
  int nb;                // wgmma N (16, 32 or 64): input channels per unit, output channels if trans
  int n_dyb, n_xb;       // output / input channel blocks
  int groups;            // (tap rows, tx, channel blocks) groups
  int ranges;            // pixel-tile ranges per group; a work unit is (range, group)
  int dy_bytes, x_bytes; // one operand part (dy^T / x^T) of a stage
  int stage_bytes;       // [dy_hi][x_hi] (x3: [dy_hi][dy_lo][x_hi][x_lo])
  int stages;            // ring depth
  int xmode;             // kXPlain / kXPool / kXGeneral
  int x3;                // AB_MATH_TF32X3: every value split into rn_tf32(v) and the exact remainder;
                         // per k-step the pairs (hi, hi), (dy lo, x hi), (dy hi, x lo) are issued
  Ordered red;           // slots [group][range][TH x 64 x nb]
};

// RN-to-TF32: the tensor core reads the upper 19 bits only (see conv_tc.cu tf32_bits)
__device__ __forceinline__ uint32_t tf32b(float x) { return __float_as_uint(x) + 0x1000u; }
__device__ __forceinline__ float lo_part(float x) {
  return x - __uint_as_float(tf32b(x) & 0xFFFFE000u);
}
// byte offset of (row r, pixel k) in the K-major core-matrix layout of one operand part
__device__ __forceinline__ uint32_t kmaj_off(int r, int k, int sbo) {
  return (uint32_t)((r >> 3) * sbo + (k >> 2) * 128 + (r & 7) * 16 + (k & 3) * 4);
}
// 4 consecutive channels (rows r0..r0+3) of pixel k: hi part, and the lo part at +lo_off (x3)
__device__ __forceinline__ void put4(uint32_t base, int sbo, int r0, int k, float4 v, bool x3,
                                     uint32_t lo_off) {
  const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t a = base + kmaj_off(r0 + i, k, sbo);
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(tf32b(e[i])) : "memory");
    if (x3) asm volatile("st.shared.b32 [%0], %1;" ::"r"(a + lo_off), "r"(tf32b(lo_part(e[i]))) : "memory");
  }
}
__device__ __forceinline__ float4 affine4(float4 v, float4 sc, float4 sh) {
  return make_float4(fmaf(v.x, sc.x, sh.x), fmaf(v.y, sc.y, sh.y), fmaf(v.z, sc.z, sh.z),
                     fmaf(v.w, sc.w, sh.w));
}
__device__ __forceinline__ float4 max4(float4 a, float4 b, float4 c, float4 d) {
  return make_float4(fmaxf(fmaxf(a.x, b.x), fmaxf(c.x, d.x)), fmaxf(fmaxf(a.y, b.y), fmaxf(c.y, d.y)),
                     fmaxf(fmaxf(a.z, b.z), fmaxf(c.z, d.z)), fmaxf(fmaxf(a.w, b.w), fmaxf(c.w, d.w)));
}
__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// What a work unit covers
struct Unit {
  int group, range, t_begin, t_end;
  int co0, ci0;   // first output / input channel
  int ty0, tx;    // first kernel row, kernel column
};
template <int NB, int TH, bool TRANS>
__device__ __forceinline__ Unit unit_of(const WgradTcParams& p, int u) {
  constexpr int DYC = TRANS ? NB : kM, XC = TRANS ? kM : NB;
  Unit w;
  w.group = u % p.groups;
  w.range = u / p.groups;
  int blk = w.group;
  const int xb = blk % p.n_xb; blk /= p.n_xb;
  const int dyb = blk % p.n_dyb; blk /= p.n_dyb;
  w.tx = blk % p.taps_w;
  w.ty0 = (blk / p.taps_w) * TH;
  w.co0 = dyb * DYC;
  w.ci0 = xb * XC;
  w.t_begin = (int)((int64_t)p.num_tiles * w.range / p.ranges);
  w.t_end = (int)((int64_t)p.num_tiles * (w.range + 1) / p.ranges);
  return w;
}

// Loader warpgroup, the tiles of one unit.  A thread's channel quad is the same for every float4
// it stages (the warpgroup's 128 threads cover whole pixel quads of <= 32 channel quads), so its
// source, affine and validity are fixed per unit and only the pixel moves: pixel k0 + step * i.
// Plain and pooled sources are read from clamped addresses without branches and masked after,
// so all of a tile's loads are in flight together.
template <int NB, int TH, bool TRANS, int XMODE>
__device__ __forceinline__ void load_unit(const WgradTcParams& p, const Unit& w, uint32_t sbase,
                                          uint32_t bar_full, uint32_t bar_empty, int& st,
                                          uint32_t& ph) {
  constexpr int DYC = TRANS ? NB : kM, XC = TRANS ? kM : NB;
  constexpr int QD = DYC / 4, QX = XC / 4;          // channel quads per pixel
  constexpr int XR = kTile + kMaxDil * (TH - 1);    // most x rows staged
  constexpr int SBO_D = sbo_bytes(kTile);
  constexpr int ND = kPix * QD / kWg;                         // dy float4 per thread per tile
  constexpr int NX = (XR * kTile * QX + kWg - 1) / kWg;       // x float4 per thread (at most)
  constexpr int KSD = kWg / QD, KSX = kWg / QX;               // pixel step between a thread's float4s
  static_assert(KSD % kTile == 0 && KSX % kTile == 0, "a thread's pixels share one tile column");
  const int tid = threadIdx.x - kWg;
  const int H = p.H, W = p.W;
  const bool x3 = p.x3 != 0;
  const int sbo_x = sbo_bytes(p.x_rows);
  const int x_elems = p.x_rows * kTile * QX;
  const uint32_t d_lo = x3 ? (uint32_t)p.dy_bytes : 0u;
  const uint32_t x_off = (uint32_t)p.dy_bytes * (x3 ? 2 : 1);
  const uint32_t x_lo = x3 ? (uint32_t)p.x_bytes : 0u;
  const int tpi = p.tiles_h * p.tiles_w;
  const int dh = (w.ty0 - (p.taps_h >> 1)) * p.dil, dwo = (w.tx - (p.taps_w >> 1)) * p.dil;

  // dy: channel quad qd, pixels kd0 + KSD * i
  const int qd = (tid >> 2) % QD, kd0 = (tid / (4 * QD)) * 4 + (tid & 3);
  const int co = w.co0 + 4 * qd;
  const bool d_ok = co < p.Cout;
  const float* dyp = p.dy + (d_ok ? co : 0);
  // x: channel quad qx of source `si`, pixels kx0 + KSX * i
  const int qx = (tid >> 2) % QX, kx0 = (tid / (4 * QX)) * 4 + (tid & 3);
  const int ci = w.ci0 + 4 * qx;
  const bool x_ok = ci < p.Cin;
  const int si = p.S.nsrc > 1 && ci >= p.S.s[0].C ? 1 : 0;
  const int c = x_ok ? ci - (si ? p.S.s[0].C : 0) : 0;
  const float* xp = (si ? p.S.s[1].ptr : p.S.s[0].ptr) + c;
  const int ld = si ? p.S.s[1].ld : p.S.s[0].ld;
  const float* scp = si ? p.S.s[1].scale : p.S.s[0].scale;
  const float* shp = si ? p.S.s[1].shift : p.S.s[0].shift;
  float4 sc = make_float4(1.f, 1.f, 1.f, 1.f), sh = make_float4(0.f, 0.f, 0.f, 0.f);
  if (XMODE != kXGeneral && scp) {
    sc = ldg4(scp + c);
    sh = ldg4(shp + c);
  }

  for (int tile = w.t_begin; tile < w.t_end; ++tile) {
    const int n = tile / tpi, rem = tile - n * tpi;
    const int h0 = (rem / p.tiles_w) * kTile, w0 = (rem % p.tiles_w) * kTile;
    float4 dv[ND], xv[NX];
    {
      const int gw = w0 + (kd0 & 7), gwc = min(gw, W - 1);
#pragma unroll
      for (int i = 0; i < ND; ++i) {
        const int gh = h0 + (kd0 >> 3) + (KSD / kTile) * i, ghc = min(gh, H - 1);
        dv[i] = ldg4(dyp + ((size_t)(n * H + ghc) * W + gwc) * p.ld_dy);
      }
    }
    {
      const int gw = w0 + (kx0 & 7) + dwo, gwc = min(max(gw, 0), W - 1);
#pragma unroll
      for (int i = 0; i < NX; ++i) {
        const int gh = h0 + (kx0 >> 3) + (KSX / kTile) * i + dh, ghc = min(max(gh, 0), H - 1);
        if (XMODE == kXPlain) {
          xv[i] = ldg4(xp + ((size_t)(n * H + ghc) * W + gwc) * ld);
        } else if (XMODE == kXPool) {
          const size_t rs = (size_t)(2 * W) * ld;
          const float* b = xp + ((size_t)(n * 2 * H + 2 * ghc) * (2 * W) + 2 * gwc) * ld;
          xv[i] = max4(affine4(ldg4(b), sc, sh), affine4(ldg4(b + ld), sc, sh),
                       affine4(ldg4(b + rs), sc, sh), affine4(ldg4(b + rs + ld), sc, sh));
        } else {
          xv[i] = x_ok ? load_src4(p.S, n, gh, gw, H, W, ci) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
    }
    // mask: out-of-image pixels and channels past Cout / Cin are zero (load_src4 semantics)
    const int gwd = w0 + (kd0 & 7), gwx = w0 + (kx0 & 7) + dwo;
#pragma unroll
    for (int i = 0; i < ND; ++i) {
      const int gh = h0 + (kd0 >> 3) + (KSD / kTile) * i;
      if (!(d_ok && gh < H && gwd < W)) dv[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int i = 0; i < NX; ++i) {
      const int gh = h0 + (kx0 >> 3) + (KSX / kTile) * i + dh;
      const bool in = x_ok && (unsigned)gh < (unsigned)H && (unsigned)gwx < (unsigned)W;
      if (XMODE == kXPlain) xv[i] = in ? affine4(xv[i], sc, sh) : make_float4(0.f, 0.f, 0.f, 0.f);
      else if (XMODE == kXPool && !in) xv[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }

    mbar_wait_quiet(bar_empty + st * 8, ph ^ 1);
    const uint32_t sa = sbase + (uint32_t)st * p.stage_bytes;
    // Channel rows past Cout / Cin are never staged: they only feed accumulator rows or columns
    // that the flush drops.
    if (d_ok) {
#pragma unroll
      for (int i = 0; i < ND; ++i) put4(sa, SBO_D, 4 * qd, kd0 + KSD * i, dv[i], x3, d_lo);
    }
    if (x_ok) {
#pragma unroll
      for (int i = 0; i < NX; ++i)
        if (tid + kWg * i < x_elems) put4(sa + x_off, sbo_x, 4 * qx, kx0 + KSX * i, xv[i], x3, x_lo);
    }
    fence_proxy_async_smem();
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(bar_full + st * 8);
    if (++st == p.stages) { st = 0; ph ^= 1; }
  }
}

// Consumer warpgroup, the tiles of one unit: acc[j] accumulates tap ty0 + j over the unit's tiles
// in tile order, k-steps in order, then its fp32 partial D[TH][64][NB] goes to the unit's slot.
template <int NB, int TH, bool TRANS>
__device__ __forceinline__ void mma_unit(const WgradTcParams& p, const Unit& w, uint32_t sbase,
                                         uint32_t bar_full, uint32_t bar_empty, int& st, uint32_t& ph) {
  constexpr int R = NB / 2;
  constexpr int SBO_D = sbo_bytes(kTile);
  const bool x3 = p.x3 != 0;
  const uint32_t d_lo = x3 ? (uint32_t)p.dy_bytes : 0u;
  const uint32_t x_off = (uint32_t)p.dy_bytes * (x3 ? 2 : 1);
  const uint32_t x_lo = x3 ? (uint32_t)p.x_bytes : 0u;
  const uint64_t dtmpl = wgmma_desc(0, 128, SBO_D), xtmpl = wgmma_desc(0, 128, sbo_bytes(p.x_rows));
  float acc[TH][R];
#pragma unroll
  for (int j = 0; j < TH; ++j)
#pragma unroll
    for (int i = 0; i < R; ++i) acc[j][i] = 0.f;
  uint32_t prev = 0;   // empty barrier of the stage whose MMAs are still in flight
  for (int tile = w.t_begin; tile < w.t_end; ++tile) {
    mbar_wait_quiet(bar_full + st * 8, ph);
    const uint32_t sa = sbase + (uint32_t)st * p.stage_bytes;
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < kPix / 8; ++ks) {
#pragma unroll
      for (int j = 0; j < TH; ++j) {
        // k-step ks of tap ty0 + j: image row ks of dy, halo row ks + j * dil of x
        const uint32_t da = sa + ks * 256, xa = sa + x_off + (ks + j * p.dil) * 256;
        const uint64_t dyh = dtmpl | (da >> 4), xh = xtmpl | (xa >> 4);
        if (TRANS) Wgmma<NB>::tf32(acc[j], xh, dyh, 1u);
        else Wgmma<NB>::tf32(acc[j], dyh, xh, 1u);
        if (x3) {
          const uint64_t dyl = dtmpl | ((da + d_lo) >> 4), xl = xtmpl | ((xa + x_lo) >> 4);
          if (TRANS) {
            Wgmma<NB>::tf32(acc[j], xh, dyl, 1u);
            Wgmma<NB>::tf32(acc[j], xl, dyh, 1u);
          } else {
            Wgmma<NB>::tf32(acc[j], dyl, xh, 1u);
            Wgmma<NB>::tf32(acc[j], dyh, xl, 1u);
          }
        }
      }
    }
    wgmma_commit();
    wgmma_wait<1>();          // the previous tile's group retired: its stage is free
    consumer_release(prev);
    prev = bar_empty + st * 8;
    if (++st == p.stages) { st = 0; ph ^= 1; }
  }
  wgmma_wait<0>();
  consumer_release(prev);
#pragma unroll
  for (int j = 0; j < TH; ++j) wgmma_fence_regs(acc[j]);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double* slot = ordered_slot(p.red, w.group, p.ranges, w.range, TH * kM * NB);
#pragma unroll
  for (int j = 0; j < TH; ++j)
#pragma unroll
    for (int c = 0; c < R / 4; ++c)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          slot[(j * kM + 16 * warp + (lane >> 2) + 8 * h) * NB + 8 * c + 2 * (lane & 3) + e] =
              acc[j][4 * c + 2 * h + e];
}

template <int NB, int TH, bool TRANS, int XMODE>
__device__ __forceinline__ void loader(const WgradTcParams& p, uint32_t sbase, uint32_t bar_full,
                                       uint32_t bar_empty) {
  int st = 0;
  uint32_t ph = 0;
  for (int u = blockIdx.x; u < p.groups * p.ranges; u += gridDim.x)
    load_unit<NB, TH, TRANS, XMODE>(p, unit_of<NB, TH, TRANS>(p, u), sbase, bar_full, bar_empty, st, ph);
}

// NB = wgmma N, TH = kernel rows per unit (1 or 3), TRANS = input channels on M.  Units
// u = blockIdx.x + k * gridDim.x run in order, unit u = (range u / groups, group u % groups), so
// the CTAs running at one time read neighbouring pixels and share dy and x through L2.
template <int NB, int TH, bool TRANS>
__global__ void __launch_bounds__(kThreads, ctas_per_sm(NB, TH)) wgrad_tc_kernel(const WgradTcParams p) {
  constexpr bool kSplitRegs = ctas_per_sm(NB, TH) == 2;
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t bar_full = smem_u32(smem), bar_empty = bar_full + kMaxStages * 8;
  const uint32_t sbase = smem_u32(smem) + kCtlBytes;
  if (threadIdx.x == 0) {
    for (int i = 0; i < p.stages; ++i) {
      mbar_init(bar_full + i * 8, kWg / 32);
      mbar_init(bar_empty + i * 8, kWg / 32);
    }
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x >= kWg) {
    if constexpr (kSplitRegs) setmaxnreg_dec<kRegsLoad>();
    if (p.xmode == kXPlain) loader<NB, TH, TRANS, kXPlain>(p, sbase, bar_full, bar_empty);
    else if (p.xmode == kXPool) loader<NB, TH, TRANS, kXPool>(p, sbase, bar_full, bar_empty);
    else loader<NB, TH, TRANS, kXGeneral>(p, sbase, bar_full, bar_empty);
  } else {
    if constexpr (kSplitRegs) setmaxnreg_inc<kRegsCons>();
    int st = 0;
    uint32_t ph = 0;
    for (int u = blockIdx.x; u < p.groups * p.ranges; u += gridDim.x)
      mma_unit<NB, TH, TRANS>(p, unit_of<NB, TH, TRANS>(p, u), sbase, bar_full, bar_empty, st, ph);
  }
}

// dW += the sum of a group's slots over its ranges in range order (the ordered_finish order), one
// thread per value: every group's sum runs in parallel instead of in the group's last CTA
__global__ void __launch_bounds__(256) wgrad_sum_kernel(const WgradTcParams p) {
  const int n = p.th * kM * p.nb;
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  int blk = blockIdx.y;
  const int xb = blk % p.n_xb; blk /= p.n_xb;
  const int dyb = blk % p.n_dyb; blk /= p.n_dyb;
  const int tx = blk % p.taps_w;
  const int ty = (blk / p.taps_w) * p.th + i / (kM * p.nb);
  const int m = (i / p.nb) % kM, c = i % p.nb;
  const int co = dyb * (p.trans ? p.nb : kM) + (p.trans ? c : m);
  const int ci = xb * (p.trans ? kM : p.nb) + (p.trans ? m : c);
  if (co >= p.Cout || ci >= p.Cin) return;
  const double* v = ordered_slot(p.red, blockIdx.y, p.ranges, 0, n) + i;
  double sum = 0.0;
  for (int s = 0; s < p.ranges; ++s) sum += __ldcg(v + (size_t)s * n);
  p.dw[(((size_t)co * p.Cin + ci) * p.taps_h + ty) * p.taps_w + tx] += (float)sum;
}

// wgmma N for a channel count: 16, 32 or 64 (blocks of 64 beyond)
int chan_block(int c) { return c <= 16 ? 16 : (c <= 32 ? 32 : 64); }

// bytes of one stage: [dy_hi][x_hi] (x3: [dy_hi][dy_lo][x_hi][x_lo]), 128-B aligned
constexpr int stage_bytes(int dyc, int xc, int x_rows, bool x3) {
  return (((dyc / 8) * sbo_bytes(kTile) + (xc / 8) * sbo_bytes(x_rows)) * (x3 ? 2 : 1) + 127) & ~127;
}
// ring depth: as many stages (up to kMaxStages) as fit `ctas` CTAs per SM, at least two
constexpr int ring_stages(int stage, int ctas) {
  return (smem_budget(ctas) - kCtlBytes) / stage >= kMaxStages ? kMaxStages
         : (smem_budget(ctas) - kCtlBytes) / stage < 2     ? 2
                                                           : (smem_budget(ctas) - kCtlBytes) / stage;
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
  // orientation: the one that issues fewer padded MMA rows and columns (a tie keeps dW[co][ci]);
  // dW^T only wins with at most 32 output channels, so its N is 16 or 32
  const auto padded = [](int c, int b) { return (int64_t)((c + b - 1) / b) * b; };
  const int64_t work = padded(p->Cout, kM) * padded(p->Cin, chan_block(p->Cin));
  const int64_t work_t = padded(p->Cin, kM) * padded(p->Cout, chan_block(p->Cout));
  p->trans = work_t < work ? 1 : 0;
  p->nb = chan_block(p->trans ? p->Cout : p->Cin);
  const int dyc = p->trans ? p->nb : kM, xc = p->trans ? kM : p->nb;
  p->n_dyb = (p->Cout + dyc - 1) / dyc;
  p->n_xb = (p->Cin + xc - 1) / xc;
  // a 3-tap column shares one x halo when it stays short; other kernels run a unit per tap row
  p->th = d->ks_h == 3 && d->dil <= kMaxDil ? 3 : 1;
  p->x_rows = kTile + d->dil * (p->th - 1);
  p->groups = (p->taps_h / p->th) * p->taps_w * p->n_dyb * p->n_xb;
  p->dy_bytes = (dyc / 8) * sbo_bytes(kTile);
  p->x_bytes = (xc / 8) * sbo_bytes(p->x_rows);
  p->stage_bytes = stage_bytes(dyc, xc, p->x_rows, p->x3 != 0);
  p->stages = ring_stages(p->stage_bytes, ctas_per_sm(p->nb, p->th));
  *smem_bytes = kCtlBytes + p->stages * p->stage_bytes;
  bool plain = true, pool = true;
  for (int i = 0; i < p->S.nsrc; ++i) {
    plain = plain && p->S.s[i].pool == 0;
    pool = pool && p->S.s[i].pool == AB_SRC_POOL;
  }
  p->xmode = plain ? kXPlain : (pool ? kXPool : kXGeneral);
  // Pixel-range partition: what one CTA per tap and per (64 output, chan_block(Cin) input) channel
  // block pair needs for about six CTAs per SM; every range keeps at least a few tiles.  It does
  // not depend on the orientation or on how many taps a unit runs, and each dW element is the
  // ordered sum of its ranges' fp32 partials, so every plan computes the same bits for a given
  // shape.
  const int per_tap_groups = d->ks_h * d->ks_w * ((p->Cout + kM - 1) / kM) *
                             ((p->Cin + chan_block(p->Cin) - 1) / chan_block(p->Cin));
  int ranges = (6 * ab_num_sms() + per_tap_groups - 1) / per_tap_groups;
  if (ranges > p->num_tiles / 4) ranges = p->num_tiles / 4;
  if (ranges < 1) ranges = 1;
  p->ranges = ranges;
  return 0;
}

template <int NB, int TH, bool TRANS>
int launch(const WgradTcParams& p, int smem, cudaStream_t stream) {
  // opted in once per device for the largest plan of this instantiation (tf32x3 stages, tallest halo)
  constexpr int dyc = TRANS ? NB : kM, xc = TRANS ? kM : NB;
  constexpr int ctas = ctas_per_sm(NB, TH);
  constexpr int x3_ring = ring_stages(stage_bytes(dyc, xc, kTile + kMaxDil * (TH - 1), true), ctas) *
                          stage_bytes(dyc, xc, kTile + kMaxDil * (TH - 1), true);
  constexpr int tf32_ring = ring_stages(stage_bytes(dyc, xc, kTile + kMaxDil * (TH - 1), false), ctas) *
                            stage_bytes(dyc, xc, kTile + kMaxDil * (TH - 1), false);
  constexpr int max_smem = kCtlBytes + (x3_ring > tf32_ring ? x3_ring : tf32_ring);
  AB_CHECK(smem <= max_smem, "wgrad_tc: %d B of shared memory exceeds the plan bound", smem);
  const auto kernel = wgrad_tc_kernel<NB, TH, TRANS>;
  static unsigned char optin[64];
  if (ab_optin_smem(reinterpret_cast<const void*>(kernel), max_smem, optin)) return 1;
  const int units = p.groups * p.ranges, n = TH * kM * NB;
  int per_sm = 0;
  AB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, smem));
  AB_CHECK(per_sm >= 1, "wgrad_tc: %d B of shared memory leave no CTA per SM", smem);
  const int grid = units < per_sm * ab_num_sms() ? units : per_sm * ab_num_sms();
  WgradTcParams q = p;
  if (ab_ordered_ws(stream, (int64_t)units * n, p.groups, &q.red)) return 1;
  kernel<<<grid, kThreads, smem, stream>>>(q);
  AB_LAUNCH_CHECK();
  wgrad_sum_kernel<<<dim3((n + 255) / 256, p.groups), 256, 0, stream>>>(q);
  AB_LAUNCH_CHECK();
  return 0;
}

template <int TH>
int launch_th(const WgradTcParams& p, int smem, cudaStream_t stream) {
  if (p.trans) return p.nb == 16 ? launch<16, TH, true>(p, smem, stream) : launch<32, TH, true>(p, smem, stream);
  if (p.nb == 16) return launch<16, TH, false>(p, smem, stream);
  if (p.nb == 32) return launch<32, TH, false>(p, smem, stream);
  return launch<64, TH, false>(p, smem, stream);
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
  return p.th == 3 ? launch_th<3>(p, smem, stream) : launch_th<1>(p, smem, stream);
}
