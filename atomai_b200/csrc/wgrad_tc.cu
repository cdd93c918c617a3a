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
// One CTA is one warpgroup and owns one kernel column tx (all taps_h taps of it, or one tap when
// the halo would be too tall), one block of output and one of input channels, and a contiguous
// range of pixel tiles.  dy is staged once per tile; x is staged once per tile as a halo of
// 8 + dil * (taps_h - 1) rows, already shifted by the column's tx * dil, and tap ty reads it from
// its own start address (ty * dil rows = 2 * ty * dil core matrices further along K), so all taps
// of the column share both staged operands and keep one accumulator set each.
// The wider channel side goes on the wgmma M rows: when the output channels are few and the input
// channels more, the CTA computes dW^T[ci][co] (A = x^T, B = dy^T) instead of dW[co][ci].
// The accumulators are flushed once into per-range slots; wgrad_sum_kernel adds each group's slots
// in range order into dW (OIHW), so the result does not depend on which CTA finishes first.
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
constexpr int kM = 64;                        // wgmma M: channels of the M side per CTA
constexpr int kMaxDil = 1;                    // column CTAs (TH = 3) up to this dilation: 10 halo rows
                                              // (a taller halo's loads do not fit in registers at N = 64)
// SBO of an operand part spanning `rows` pixel rows (two 16-B pixel quads per row): one 8-row
// group, padded by 32 B (bank spread)
__host__ __device__ constexpr int sbo_bytes(int rows) { return rows * 2 * 128 + 32; }

struct WgradTcParams {
  SrcSet S;
  int N, H, W, Cout, Cin;
  int taps_h, taps_w, dil;
  const float* dy;
  int ld_dy;
  float* dw;
  int tiles_h, tiles_w, num_tiles;
  int th;                // kernel rows per CTA: taps_h (one whole kernel column) or 1
  int x_rows;            // pixel rows of the staged x halo: 8 + dil * (th - 1)
  int trans;             // 1: D = dW^T[ci][co] (M = input channels), 0: D = dW[co][ci]
  int nb;                // wgmma N (16, 32 or 64): input channels per CTA, output channels if trans
  int n_dyb, n_xb;       // output / input channel blocks
  int ranges;            // pixel-tile ranges per (tap rows, tx, channel blocks)
  int dy_bytes, x_bytes; // one operand part (dy^T / x^T) of a stage
  int stage_bytes;       // [dy_hi][x_hi] (x3: [dy_hi][dy_lo][x_hi][x_lo])
  int x3;                // AB_MATH_TF32X3: every value split into rn_tf32(v) and the exact remainder;
                         // per k-step the pairs (hi, hi), (dy lo, x hi), (dy hi, x lo) are issued
  Ordered red;           // slots [group = (tap rows, tx, channel blocks)][range][TH x 64 x nb]
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

// NB = wgmma N, TH = kernel rows per CTA (1 or 3), TRANS = input channels on M
template <int NB, int TH, bool TRANS>
__global__ void __launch_bounds__(kThreads) wgrad_tc_kernel(const WgradTcParams p) {
  constexpr int R = NB / 2;
  constexpr int DYC = TRANS ? NB : kM;             // output channels per CTA
  constexpr int XC = TRANS ? kM : NB;              // input channels per CTA
  constexpr int QD = DYC / 4, QX = XC / 4;         // channel quads per pixel
  constexpr int XR = kTile + kMaxDil * (TH - 1);   // most x rows staged
  constexpr int SBO_D = sbo_bytes(kTile);
  constexpr int ND = kPix * QD / kThreads;                          // dy float4 per thread per tile
  constexpr int NX = (XR * kTile * QX + kThreads - 1) / kThreads;   // x float4 per thread (at most)
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x;

  // grid: x = (tap rows, tx, dy block, x block), y = pixel range: the CTAs that read the same
  // pixels are launched together and share dy and x through L2
  int blk = blockIdx.x;
  const int xb = blk % p.n_xb; blk /= p.n_xb;
  const int dyb = blk % p.n_dyb; blk /= p.n_dyb;
  const int tx = blk % p.taps_w;
  const int ty0 = (blk / p.taps_w) * TH;
  const int co0 = dyb * DYC, ci0 = xb * XC;
  const int dh = (ty0 - (p.taps_h >> 1)) * p.dil, dwo = (tx - (p.taps_w >> 1)) * p.dil;
  const int t_begin = (int)((int64_t)p.num_tiles * blockIdx.y / p.ranges);
  const int t_end = (int)((int64_t)p.num_tiles * (blockIdx.y + 1) / p.ranges);
  const int tpi = p.tiles_h * p.tiles_w;
  const bool x3 = p.x3 != 0;
  const int H = p.H, W = p.W;
  const int sbo_x = sbo_bytes(p.x_rows);
  const int x_elems = p.x_rows * kTile * QX;                              // float4 of one x halo
  const uint32_t d_lo = x3 ? (uint32_t)p.dy_bytes : 0u;                   // dy_hi -> dy_lo
  const uint32_t x_off = (uint32_t)p.dy_bytes * (x3 ? 2 : 1);             // stage -> x_hi
  const uint32_t x_lo = x3 ? (uint32_t)p.x_bytes : 0u;                    // x_hi -> x_lo

  // Channel rows past Cout / Cin are never staged: they only feed accumulator rows or columns that
  // the flush drops.
  float4 dv[ND], xv[NX];
  auto load = [&](int tile) {
    const int n = tile / tpi, rem = tile - n * tpi;
    const int h0 = (rem / p.tiles_w) * kTile, w0 = (rem % p.tiles_w) * kTile;
#pragma unroll
    for (int i = 0; i < ND; ++i) {
      const int e = tid + kThreads * i;
      const int k = (e / (4 * QD)) * 4 + (e & 3), q = (e >> 2) % QD;
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
      xv[i] = e < x_elems && ci < p.Cin
                  ? load_src4(p.S, n, h0 + (k >> 3) + dh, w0 + (k & 7) + dwo, H, W, ci)
                  : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto store = [&](uint32_t st) {
#pragma unroll
    for (int i = 0; i < ND; ++i) {
      const int e = tid + kThreads * i, q = (e >> 2) % QD;
      if (co0 + 4 * q < p.Cout) put4(st, SBO_D, 4 * q, (e / (4 * QD)) * 4 + (e & 3), dv[i], x3, d_lo);
    }
#pragma unroll
    for (int i = 0; i < NX; ++i) {
      const int e = tid + kThreads * i, q = (e >> 2) % QX;
      if (e < x_elems && ci0 + 4 * q < p.Cin)
        put4(st + x_off, sbo_x, 4 * q, (e / (4 * QX)) * 4 + (e & 3), xv[i], x3, x_lo);
    }
  };

  float acc[TH][R];
#pragma unroll
  for (int j = 0; j < TH; ++j)
#pragma unroll
    for (int i = 0; i < R; ++i) acc[j][i] = 0.f;
  const uint64_t dtmpl = wgmma_desc(0, 128, SBO_D), xtmpl = wgmma_desc(0, 128, sbo_x);
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
#pragma unroll
      for (int j = 0; j < TH; ++j) {
        // k-step ks of tap ty0 + j: image row ks of dy, halo row ks + j * dil of x
        const uint32_t da = st + ks * 256, xa = st + x_off + (ks + j * p.dil) * 256;
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
    if (tile + 1 < t_end) load(tile + 1);     // global loads in flight while the MMAs run
    wgmma_wait<1>();                           // the group of tile - 1 (the other stage) retired
    __syncthreads();
  }
  wgmma_wait<0>();
#pragma unroll
  for (int j = 0; j < TH; ++j) wgmma_fence_regs(acc[j]);
  // this CTA's partial D[TH][64][NB] (row-major) into its slot; wgrad_sum_kernel adds the slots
  const int warp = tid >> 5, lane = tid & 31;
  double* slot = ordered_slot(p.red, blockIdx.x, p.ranges, blockIdx.y, TH * kM * NB);
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
  // a 3-tap column shares one x halo when it stays short; other kernels run a CTA per tap row
  p->th = d->ks_h == 3 && d->dil <= kMaxDil ? 3 : 1;
  p->x_rows = kTile + d->dil * (p->th - 1);
  p->dy_bytes = (dyc / 8) * sbo_bytes(kTile);
  p->x_bytes = (xc / 8) * sbo_bytes(p->x_rows);
  p->stage_bytes = ((p->dy_bytes + p->x_bytes) * (p->x3 ? 2 : 1) + 127) & ~127;
  *smem_bytes = 2 * p->stage_bytes;
  // Pixel-range partition: what one CTA per tap and per (64 output, chan_block(Cin) input) channel
  // block pair needs for about six CTAs per SM; every CTA keeps at least a few tiles.  It does not
  // depend on the orientation or on how many taps a CTA runs, and each dW element is the ordered
  // sum of its ranges' fp32 partials, so every plan computes the same bits for a given shape.
  // Column CTAs therefore number about two per SM (six / three taps).
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
  constexpr int max_smem =
      2 * ((((dyc / 8) * sbo_bytes(kTile) + (xc / 8) * sbo_bytes(kTile + kMaxDil * (TH - 1))) * 2 + 127) & ~127);
  AB_CHECK(smem <= max_smem, "wgrad_tc: %d B of shared memory exceeds the plan bound", smem);
  static unsigned char optin[64];
  if (ab_optin_smem(reinterpret_cast<const void*>(wgrad_tc_kernel<NB, TH, TRANS>), max_smem, optin)) return 1;
  const int groups = (p.taps_h / TH) * p.taps_w * p.n_dyb * p.n_xb, n = TH * kM * NB;
  WgradTcParams q = p;
  if (ab_ordered_ws(stream, (int64_t)groups * p.ranges * n, groups, &q.red)) return 1;
  wgrad_tc_kernel<NB, TH, TRANS><<<dim3(groups, p.ranges), kThreads, smem, stream>>>(q);
  AB_LAUNCH_CHECK();
  wgrad_sum_kernel<<<dim3((n + 255) / 256, groups), 256, 0, stream>>>(q);
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
