// conv_tc.cu — implicit-GEMM convolution on the Hopper tensor cores (wgmma, TF32 operands, fp32
// accumulators in registers).  One persistent, warp-specialised CTA per SM, two pipelines that
// work on alternate tiles, each with its own consumer and loader warpgroup:
//
//   warps 0-3, 4-7    consumer g   wgmma for every (k-chunk, tap, k-step) of pipeline g's tiles, then
//                                  the epilogue from the accumulator registers: bias + activation ->
//                                  NHWC/NCHW store + BN statistics; refills its own weight ring
//                                  (streamed weights) with cp.async.bulk of the pre-packed blob
//   warps 8-11, 12-15 loaders g    HBM/L2 (or a TMA-staged raw tile) -> regs -> [BN affine, 2x2
//                                  max-pool, zero pad, RN->TF32] -> smem for pipeline g
//
// While one consumer waits for a stage or runs its epilogue, the other keeps the tensor core fed.
//
// GEMM view (SURVEY.md §8a): M = 64 output pixels (an 8 x 8 tile = one m64 wgmma row block, or
// 8 x 16 as two sub-tiles when N <= 64), N = Cout (<= 128 per launch; wider layers run one launch
// per 128 channels), K = taps * Cin.  The tile height is set by the register file: the whole
// 512-thread kernel is compiled for 128 registers per thread, so the consumer keeps at most 64
// fp32 accumulators.  The activation halo tile is loaded ONCE per k-chunk and re-used by all nine
// taps: it is stored as K-major no-swizzle core matrices, one plane per 4 channels, rows = halo
// pixels at 16 B pitch.  A tap is then just a different start address ((ty*d*TWp + tx*d) * 16 B)
// with SBO = TWp*16 B (next image row = next 8-row group) and LBO = plane stride (next 4
// channels).  No im2col buffer ever exists.
//
// Replaces nn.Conv2d(+bias) -> nn.LeakyReLU -> (batch statistics of) nn.BatchNorm2d of
// atomai/nets/blocks.py:61-76,302-319, the preceding BatchNorm2d/max_pool2d/cat passes
// (normalise-on-load, atomai/nets/fcnn.py:123-138) and, with flipped weights, autograd's dgrad.
#include <cuda.h>

#include <cstdio>
#include <cstdlib>
#include <type_traits>
#include "common.cuh"
#include "wgmma.cuh"

namespace {

constexpr int kTileH = 8;
constexpr int kTileW = 8;
constexpr int kNumEpiWarps = 4;     // warps per consumer warpgroup
constexpr int kNumConsWarps = 2 * kNumEpiWarps;
constexpr int kFirstLoadWarp = kNumConsWarps;
constexpr int kNumLoadWarps = 8;
constexpr int kThreads = (kFirstLoadWarp + kNumLoadWarps) * 32;
// register split between the warpgroups (2 * (consumer + loader) * 128 threads = 64K registers).
// The kernel is launched at 128 registers per thread and setmaxnreg moves them between the
// warpgroups.  The loaders keep 120 (their U <= kMaxU staged float4s); the consumers get the
// rest, 136.  More does not help them: with CUDA 12.9 ptxas kept the consumer code within about
// 136 registers even when setmaxnreg allowed 160 or 232, and those splits only made the kernel's
// stack frame larger.
constexpr int kRegsCons = 136, kRegsLoad = 120;
static_assert(2 * (kRegsCons + kRegsLoad) <= 512, "register budget");
constexpr int kMaxN = 128;          // output channels per launch (accumulator registers)
constexpr int kMaxAStages = 4;
constexpr int kMaxBStages = 32;     // streamed weights: bytes in flight must cover the L2 latency
constexpr int kMaxRStages = 8;      // TMA mode: raw activation tiles in flight (two rings of n_r/2)
constexpr int kGroupThreads = 128;  // loader threads per group (2 groups of 4 warps)
constexpr int kMaxU = 12;           // register-staged 16B elements per loader thread per chunk

struct ConvTcParams {
  SrcSet S;
  int N, H, W, Cout;
  int n0, nn;        // output channels [n0, n0 + nn) of this launch
  int taps_h, taps_w, dil;
  const float* wblob;
  const float* bias;
  float alpha;
  int act;
  float* out;
  int ld_out;
  int out_nchw;
  int64_t nchw_stride; // out_nchw: elements between channel planes (H*W, or the caller's row pitch)
  double* stats;
  Ordered red;       // stats: ordered sum of the per-CTA partials
  int tiles_h, tiles_w, num_tiles;
  int KC;            // channels per k-chunk (8, 16 or 32)
  int n_chunks;      // Ctot / KC
  int TWp, THp, HP;  // halo tile extent and pixel count
  int plane_bytes;   // stride between 4-channel planes (== 128/P mod 128 -> conflict-free STS)
  int a_stage_bytes, b_stage_bytes;
  int n_a, n_b;      // pipeline depths
  int sub;           // 8-pixel-wide sub-tiles per CTA tile (1 or 2): M = 128*sub per weight stage
  int w_resident;    // 1: all weights live in shared memory for the whole kernel
  int w_bytes;       // taps * Ctot * Cout * 4  (x3: twice that — hi and lo parts)
  int x3;            // AB_MATH_TF32X3: every k-step issues a second, bf16 MMA (K = 16) on an operand
                     // pair ([a_lo | a_hi] x [w ; w_lo]) that adds the two cross terms of the split
  int corr_off;      // x3: byte offset of the correction planes inside an activation stage
  // TMA mode (resident weights, un-pooled sources): cp.async.bulk.tensor copies the raw NHWC halo
  // tile {KC channels, TWp, THp} (out-of-image pixels zero-filled by the copy engine) into a ring
  // of raw stages; the "loader" warps then only transform shared memory -> shared memory (affine,
  // border mask, TF32 rounding / x3 split into the MMA planes).  Bytes in flight are bounded by
  // the raw ring (up to 8 stages) instead of by loader registers.
  int tma;
  int raw_bytes;     // HP * KC * 4
  int n_r;           // raw stages (two rings of n_r/2)
  // tiles per consumer pass (1 or 2).  2: a consumer takes two of its tiles at once, k-chunk by
  // k-chunk, and issues every (tap, k-step) MMA of one tile right after the same MMA of the
  // other, so two independent accumulator chains hide each other's wgmma latency.  Every tile
  // keeps its own accumulators, MMA order and place in the statistics token sequence, so outputs
  // and statistics are bit-identical to pair = 1.
  int pair;
};

struct __align__(8) SharedCtl {
  uint64_t full_a[kMaxAStages], empty_a[kMaxAStages];
  uint64_t full_b[kMaxBStages];
  uint64_t raw_full[kMaxRStages], raw_empty[kMaxRStages];
  uint64_t w_full;
  unsigned red_last;
};

// named barriers (id 0 = __syncthreads, 1 = the consumers' final statistics sum)
constexpr int kStatBar = 2;   // 2..5: consumer 0 -> 1 statistics token of warp w, 6..9: 1 -> 0

// Streamed-weight refill issued by one thread of a consumer warpgroup.  The copies are predicated
// instead of branched on: a divergent branch while MMAs are in flight makes ptxas serialise them.
__device__ __forceinline__ void expect_tx_if(uint32_t pred, uint32_t bar, uint32_t bytes) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %0, 0;\n\t"
      "@p mbarrier.arrive.expect_tx.shared::cta.b64 _, [%1], %2;\n\t}" ::"r"(pred), "r"(bar), "r"(bytes)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s_if(uint32_t pred, uint32_t dst_smem, const void* src,
                                            uint32_t bytes, uint32_t bar) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %0, 0;\n\t"
      "@p cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%1], [%2], %3, [%4];\n\t}" ::
          "r"(pred), "r"(dst_smem), "l"(src), "r"(bytes), "r"(bar)
      : "memory");
}

// The tile loop of consumer warpgroup `pipe`, specialised on (N = output channels of this launch,
// 8-pixel sub-tiles).  Consumer g owns the tiles with CTA-local index = g (mod 2), the operand
// ring half g (filled by loader group g) and the weight ring half g.  A k-chunk (resident weights)
// or a tap (streamed weights) is one wgmma group; a stage is handed back when the group after its
// last use has been issued and the one using it has retired (wgmma.wait_group 1), so the tensor
// core always has the next group queued.  A streamed weight stage is refilled at that point by
// the consumer's first thread with the piece it holds next (n_b/2 pieces ahead): the retired group
// was issued by all four warps, so none of them still waits for the stage's previous contents.
// PAIR = 2 (resident weights, see ConvTcParams::pair) runs its own pass loop below and shares the
// epilogue and the statistics hand-off with the one-tile loop.
template <int N, int SUB, int PAIR, int PIPE>
__device__ __forceinline__ void consumer_loop(const ConvTcParams& p, SharedCtl* ctl, uint32_t a_base,
                                              uint32_t b_base, float* s_stats, const float* s_bias) {
  // PIPE is a template parameter: control flow that depends on the thread index puts the MMAs on
  // a divergent path for ptxas, which then serialises them (C7520)
  constexpr int pipe = PIPE;
  constexpr int R = N / 2;
  const int warp = (threadIdx.x >> 5) & (kNumEpiWarps - 1), lane = threadIdx.x & 31;
  const uint32_t leader = (threadIdx.x & (kNumEpiWarps * 32 - 1)) == 0 ? 1u : 0u;
  const uint32_t ring_n = p.n_a / 2, nb2 = p.n_b / 2;
  const int ksteps = p.KC >> 3;
  const int th = p.taps_h, tw = p.taps_w, taps = th * tw;
  const bool x3 = p.x3 != 0, res = p.w_resident != 0;
  const uint32_t wmult = x3 ? 2u : 1u;
  const uint32_t piece = (uint32_t)p.Cout * 32;                     // bytes of one (k-step, tap) piece
  const uint32_t corr_w = res ? (uint32_t)taps * piece : piece;      // main -> correction piece
  const uint32_t b_n0 = (uint32_t)p.n0 * 16;
  const uint64_t a_tmpl = wgmma_desc(0, p.plane_bytes, p.TWp * 16);
  const uint64_t b_tmpl = wgmma_desc(0, p.Cout * 16, 128);
  const uint32_t mb_off = 8u * p.TWp * 16, sb_off = kTileW * 16;
  const uint32_t bar_full_a = smem_u32(&ctl->full_a[0]), bar_empty_a = smem_u32(&ctl->empty_a[0]);
  const uint32_t bar_full_b = smem_u32(&ctl->full_b[0]);
  const int tpi = p.tiles_w * p.tiles_h;
  const bool fast = p.act == AB_ACT_LRELU && p.alpha >= 0.f && p.alpha <= 1.f;
  const float alpha = p.alpha;
  float* my_stats = s_stats + warp * 2 * p.Cout;
  const int tile_step = 2 * gridDim.x;
  const uint32_t ring0 = pipe * ring_n, b_ring0 = pipe * nb2;
  uint32_t s_a = 0, p_a = 0, s_b = 0, p_b = 0;
  // streamed weights: copy the piece `ahead` pieces after (r_tile, r_ch, r_t) of this consumer's
  // sequence into weight stage `stage`
  auto refill_b = [&](uint32_t stage, int r_tile, int r_ch, int r_t, int ahead) {
    r_t += ahead;
    while (r_t >= taps) {
      r_t -= taps;
      if (++r_ch == p.n_chunks) { r_ch = 0; r_tile += tile_step; }
    }
    if (r_tile < p.num_tiles) {
      // piece (k-step s, kind, tap) of the blob lives at ((s*wmult + kind)*taps + tap); the stage
      // holds [k-step][kind] pieces
      const uint32_t bar = bar_full_b + (b_ring0 + stage) * 8;
      expect_tx_if(leader, bar, p.b_stage_bytes);
      for (int ks = 0; ks < ksteps; ++ks)
        for (uint32_t kd = 0; kd < wmult; ++kd)
          bulk_g2s_if(leader, b_base + (b_ring0 + stage) * p.b_stage_bytes + (ks * wmult + kd) * piece,
                      p.wblob + ((((size_t)r_ch * ksteps + ks) * wmult + kd) * taps + r_t) * (piece >> 2),
                      piece, bar);
    }
  };
  if (res) {
    mbar_wait_quiet(smem_u32(&ctl->w_full), 0);
  } else {
    for (uint32_t i = 0; i < nb2; ++i) refill_b(i, blockIdx.x + pipe * gridDim.x, 0, 0, (int)i);
  }
  constexpr int MB = kTileH / 8;               // m64 row blocks per sub-tile
  float acc[SUB][MB][R];

  // ---------------- epilogue: registers -> bias + activation -> global store + BN statistics
  const int c_lane = 2 * (lane & 3);
  // a tile's channel sums, added once the token arrives.  After the butterfly every lane of a
  // channel pair holds the same sums, so column group j is kept by the lanes with
  // lane >> 2 == j % 8 only: R / 32 groups per lane instead of R / 4
  constexpr int JL = (R / 4 + 7) / 8;
  // tile `tl`'s epilogue from accumulators `a`; `real` = false: the dropped second tile of a
  // paired pass, which stores nothing.  Its channel sums go to `st` for add_stats.
  auto epilogue = [&](float (&a)[SUB][MB][R], const int tl, const bool real, float (&st)[JL][4]) {
    const int n = tl / tpi, rem = tl - n * tpi;
    const int th_i = rem / p.tiles_w, tw_i = rem - th_i * p.tiles_w;
    // compiled once for the plain LeakyReLU and once for every other activation: the per-element
    // activation switch of the general case, unrolled over the tile, is what the epilogue spilled
    auto body = [&](auto fast_tag) {
      constexpr bool FAST = decltype(fast_tag)::value;
#pragma unroll
      for (int j = 0; j < R / 4; ++j) {
        const int c = p.n0 + 8 * j + c_lane;
        const float b0 = s_bias[c], b1 = s_bias[c + 1];
        float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
#pragma unroll
        for (int s = 0; s < SUB; ++s)
#pragma unroll
          for (int mb = 0; mb < MB; ++mb)
#pragma unroll
            for (int hrow = 0; hrow < 2; ++hrow) {
              const int gh = th_i * kTileH + mb * 8 + 2 * warp + hrow;
              const int gw = (tw_i * SUB + s) * kTileW + (lane >> 2);
              const bool valid = real && gh < p.H && gw < p.W;
              float v0 = a[s][mb][4 * j + 2 * hrow] + b0, v1 = a[s][mb][4 * j + 2 * hrow + 1] + b1;
              if (FAST) {
                v0 = fmaxf(v0, v0 * alpha);
                v1 = fmaxf(v1, v1 * alpha);
              } else if (p.act == AB_ACT_RBF) {     // alpha * exp(-x/2) as one FMUL + EX2
                v0 = alpha * exp2f(-0.72134752f * fmaxf(v0, 0.f));
                v1 = alpha * exp2f(-0.72134752f * fmaxf(v1, 0.f));
              } else {
                v0 = act_f(v0, p.act, alpha);
                v1 = act_f(v1, p.act, alpha);
              }
              v0 = valid ? v0 : 0.f;
              v1 = valid ? v1 : 0.f;
              if (valid) {
                const size_t pix = ((size_t)n * p.H + gh) * p.W + gw;
                if (!p.out_nchw) {
                  *reinterpret_cast<float2*>(p.out + pix * p.ld_out + c) = make_float2(v0, v1);
                } else {
                  const size_t hw = (size_t)p.nchw_stride;
                  float* o = p.out + ((size_t)n * p.Cout + c) * hw + (size_t)gh * p.W + gw;
                  o[0] = v0;
                  o[hw] = v1;
                }
              }
              s0 += v0; s1 += v1;
              q0 = fmaf(v0, v0, q0); q1 = fmaf(v1, v1, q1);
            }
        if (p.stats) {   // the 8 lanes sharing (lane & 3) hold the same two channels
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) {
            s0 += __shfl_xor_sync(0xffffffffu, s0, o);
            s1 += __shfl_xor_sync(0xffffffffu, s1, o);
            q0 += __shfl_xor_sync(0xffffffffu, q0, o);
            q1 += __shfl_xor_sync(0xffffffffu, q1, o);
          }
          if ((lane >> 2) == (j & 7)) {
            st[j >> 3][0] = s0; st[j >> 3][1] = s1; st[j >> 3][2] = q0; st[j >> 3][3] = q1;
          }
        }
      }
    };
    if (fast) body(std::true_type{});
    else body(std::false_type{});
  };
  // tile `tl`'s statistics.  Warp w of both consumers adds into s_stats[w] in tile order, as one
  // consumer did: wait for the other consumer's previous tile, add, pass the token on.  The token
  // is a named barrier of the two warps (bar.arrive by the passing warp, bar.sync by the waiting
  // one): a spin on shared memory here puts the next tile's MMAs on a divergent path for ptxas
  auto add_stats = [&](const int tl, const float (&st)[JL][4]) {
    if (tl != (int)blockIdx.x) named_bar_sync(kStatBar + (PIPE ? 0 : kNumEpiWarps) + warp, 64);
#pragma unroll
    for (int jl = 0; jl < JL; ++jl) {
      const int j = 8 * jl + (lane >> 2);
      if (j < R / 4) {
        const int c = p.n0 + 8 * j + c_lane;
        my_stats[c] += st[jl][0];
        my_stats[c + 1] += st[jl][1];
        my_stats[p.Cout + c] += st[jl][2];
        my_stats[p.Cout + c + 1] += st[jl][3];
      }
    }
    if (tl + (int)gridDim.x < p.num_tiles)
      named_bar_arrive(kStatBar + (PIPE ? kNumEpiWarps : 0) + warp, 64);
  };

  auto tile_fn = [&](const int tile) {
    uint32_t pend_a = 0, accum = 0;
    bool pend_b = false;
    for (int ch = 0; ch < p.n_chunks; ++ch) {
      if (pend_a && ring_n == 1) {
        // one operand stage per pipeline: the stage this chunk needs is the one still held for
        // the previous chunk, so its MMAs must retire before it can go back to the loaders
        wgmma_wait<0>();
        consumer_release(pend_a);
        pend_a = 0;
      }
      mbar_wait_quiet(bar_full_a + (ring0 + s_a) * 8, p_a);
      const uint32_t a_stage = a_base + (ring0 + s_a) * p.a_stage_bytes;
      for (int t = 0; t < taps; ++t) {
        const int ty = t / tw, tx = t - ty * tw;
        uint32_t b_stage = 0;
        if (!res) {
          if (pend_b && nb2 == 1) {   // the same for a one-stage weight ring
            wgmma_wait<0>();
            refill_b((s_b + nb2 - 1) % nb2, tile, ch, t, (int)nb2 - 1);
            pend_b = false;
          }
          mbar_wait_quiet(bar_full_b + (b_ring0 + s_b) * 8, p_b);
          b_stage = b_base + (b_ring0 + s_b) * p.b_stage_bytes;
        }
        const uint32_t a_tap = a_stage + (uint32_t)(ty * p.TWp + tx) * p.dil * 16;
        wgmma_fence();
        for (int ks = 0; ks < ksteps; ++ks) {
          const uint32_t a_k = a_tap + ks * 2u * p.plane_bytes;
          const uint32_t b_k = b_n0 + (res ? b_base + ((uint32_t)(ch * ksteps + ks) * wmult * taps + t) * piece
                                           : b_stage + ks * wmult * piece);
          const uint64_t bd = b_tmpl | (b_k >> 4);
#pragma unroll
          for (int s = 0; s < SUB; ++s)
#pragma unroll
            for (int mb = 0; mb < MB; ++mb)
              Wgmma<N>::tf32(acc[s][mb], a_tmpl | ((a_k + mb * mb_off + s * sb_off) >> 4), bd, accum);
          if (x3) {   // + a_lo*w + a_hi*w_lo: one bf16 MMA (K = 16) on the correction planes
            const uint64_t bc = b_tmpl | ((b_k + corr_w) >> 4);
#pragma unroll
            for (int s = 0; s < SUB; ++s)
#pragma unroll
              for (int mb = 0; mb < MB; ++mb)
                Wgmma<N>::bf16(acc[s][mb], a_tmpl | ((a_k + p.corr_off + mb * mb_off + s * sb_off) >> 4),
                               bc, 1u);
          }
          accum = 1u;
        }
        // resident weights: one group per k-chunk; streamed: one per tap (its weight stage goes
        // back as soon as possible, the ring may hold fewer stages than there are taps)
        if (res && t != taps - 1) continue;
        wgmma_commit();
        wgmma_wait<1>();
        consumer_release(pend_a);
        if (pend_b) refill_b((s_b + nb2 - 1) % nb2, tile, ch, t, (int)nb2 - 1);
        pend_a = 0;
        pend_b = false;
        if (!res) {
          pend_b = true;
          if (++s_b == nb2) { s_b = 0; p_b ^= 1; }
        }
        if (t == taps - 1) {
          pend_a = bar_empty_a + (ring0 + s_a) * 8;
          if (++s_a == ring_n) { s_a = 0; p_a ^= 1; }
        }
      }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int s = 0; s < SUB; ++s)
#pragma unroll
      for (int mb = 0; mb < MB; ++mb) wgmma_fence_regs(acc[s][mb]);
    consumer_release(pend_a);
    if (pend_b) refill_b((s_b + nb2 - 1) % nb2, tile + tile_step, 0, 0, (int)nb2 - 1);

    float st[JL][4];
    epilogue(acc, tile, true, st);
    if (p.stats) add_stats(tile, st);
  };

  if constexpr (PAIR == 1) {
    for (int tile = blockIdx.x + pipe * gridDim.x; tile < p.num_tiles; tile += tile_step) tile_fn(tile);
  } else {
    // A pass takes the consumer's tiles k and k + 1 (tile, tile + tile_step); the loaders stage
    // them k-chunk by k-chunk, one operand stage each, so a pass holds both stages of its
    // pipeline and every k-chunk group retires right after its commit (the other pipeline keeps
    // the tensor core busy meanwhile; a wgmma wait at the top of the chunk instead makes ptxas
    // serialise the MMAs).  A lone last tile is staged twice and the second result dropped, so
    // no MMA or wgmma wait depends on whether the pass has two tiles.  Both tiles' epilogues run
    // before the first statistics add: accumulators read after the lane-dependent adds also
    // serialise the MMAs.
    float pacc[2][SUB][MB][R];
    auto pass_fn = [&](const int tile) {
      const bool two = tile + tile_step < p.num_tiles;
      uint32_t accum = 0;
      for (int ch = 0; ch < p.n_chunks; ++ch) {
        uint32_t a_stage[2], empty[2];
#pragma unroll
        for (int w = 0; w < 2; ++w) {
          mbar_wait_quiet(bar_full_a + (ring0 + s_a) * 8, p_a);
          a_stage[w] = a_base + (ring0 + s_a) * p.a_stage_bytes;
          empty[w] = bar_empty_a + (ring0 + s_a) * 8;
          if (++s_a == ring_n) { s_a = 0; p_a ^= 1; }
        }
        for (int t = 0; t < taps; ++t) {
          const int ty = t / tw, tx = t - ty * tw;
          const uint32_t tap_off = (uint32_t)(ty * p.TWp + tx) * p.dil * 16;
          wgmma_fence();
          for (int ks = 0; ks < ksteps; ++ks) {
            const uint32_t a_k = tap_off + ks * 2u * p.plane_bytes;
            const uint32_t b_k = b_n0 + b_base + ((uint32_t)(ch * ksteps + ks) * wmult * taps + t) * piece;
            const uint64_t bd = b_tmpl | (b_k >> 4);
#pragma unroll
            for (int w = 0; w < 2; ++w)
#pragma unroll
              for (int s = 0; s < SUB; ++s)
#pragma unroll
                for (int mb = 0; mb < MB; ++mb)
                  Wgmma<N>::tf32(pacc[w][s][mb],
                                 a_tmpl | ((a_stage[w] + a_k + mb * mb_off + s * sb_off) >> 4), bd, accum);
            if (x3) {
              const uint64_t bc = b_tmpl | ((b_k + corr_w) >> 4);
#pragma unroll
              for (int w = 0; w < 2; ++w)
#pragma unroll
                for (int s = 0; s < SUB; ++s)
#pragma unroll
                  for (int mb = 0; mb < MB; ++mb)
                    Wgmma<N>::bf16(pacc[w][s][mb],
                                   a_tmpl | ((a_stage[w] + a_k + p.corr_off + mb * mb_off + s * sb_off) >> 4),
                                   bc, 1u);
            }
            accum = 1u;
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        consumer_release(empty[0]);
        consumer_release(empty[1]);
      }
#pragma unroll
      for (int w = 0; w < 2; ++w)
#pragma unroll
        for (int s = 0; s < SUB; ++s)
#pragma unroll
          for (int mb = 0; mb < MB; ++mb) wgmma_fence_regs(pacc[w][s][mb]);
      float st[2][JL][4];
#pragma unroll
      for (int w = 0; w < 2; ++w) epilogue(pacc[w], tile + w * tile_step, w == 0 || two, st[w]);
      if (p.stats) {
        add_stats(tile, st[0]);
        if (two) add_stats(tile + tile_step, st[1]);
      }
    };
    for (int tile = blockIdx.x + pipe * gridDim.x; tile < p.num_tiles; tile += 2 * tile_step) pass_fn(tile);
  }
  if (p.stats) {   // this CTA's partial = the four warps' sums in warp order, then ordered over CTAs
    constexpr int kNt = kNumConsWarps * 32;
    auto bar = [] { asm volatile("bar.sync 1, %0;" ::"n"(kNt) : "memory"); };
    bar();
    const int t = threadIdx.x, n = 2 * p.nn;
    double* slot = ordered_slot(p.red, 0, gridDim.x, blockIdx.x, n);
    for (int i = t; i < n; i += kNt) {
      const int c = i < p.nn ? p.n0 + i : p.Cout + p.n0 + (i - p.nn);
      double v = 0.0;
      for (int w = 0; w < kNumEpiWarps; ++w) v += (double)s_stats[w * 2 * p.Cout + c];
      slot[i] = v;
    }
    ordered_finish(p.red, 0, gridDim.x, n, t, kNt, gridDim.x, bar,
                   [&](int i, double v) {
                     p.stats[i < p.nn ? p.n0 + i : p.Cout + p.n0 + (i - p.nn)] += v;
                   },
                   &ctl->red_last);
  }
}

// RN-to-TF32 of an fp32 bit pattern for a tensor-core operand: the tensor core reads only the upper
// 19 bits, so adding half an ulp of the 10-bit mantissa (round-half-away, like cvt.rna) is enough
// and costs one integer add instead of cvt.rna.tf32's four-instruction emulation.
__device__ __forceinline__ uint32_t tf32_bits(float x) { return __float_as_uint(x) + 0x1000u; }

// Activation loader of one group (4 warps), specialised on U = 16-byte elements per thread per
// chunk.  Element u of a thread is halo pixel q0 + u*QS of plane j for every chunk, so its pixel
// offset relative to the tile origin and its smem slot are loop constants; only element U-1 can be
// absent (HP is not a multiple of QS), every other load/store is unconditional.
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "r"(addr));
  return v;
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* tm, int c0, int c1,
                                            int c2, int c3, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%2, %3, %4, %5}], [%6];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(tm)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(bar)
      : "memory");
}

template <int U, int PAIR>
__device__ __forceinline__ void loader_loop(const ConvTcParams& p, SharedCtl* ctl,
                                            uint32_t a_base, uint32_t raw_base, int grp,
                                            const CUtensorMap* tm0, const CUtensorMap* tm1) {
  const int lane = threadIdx.x & 31;
  const int gt = threadIdx.x - (kFirstLoadWarp + grp * 4) * 32;   // 0..127
  const int P = p.KC >> 2;                   // planes per chunk (2, 4 or 8)
  const int j = gt & (P - 1);                // this thread's plane (constant: 128 % P == 0)
  const int QS = kGroupThreads / P;          // halo pixels advanced per u
  const int q0 = gt / P;
  const int H = p.H, W = p.W;
  uint32_t pix[U], hw[U];
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const int q = q0 + u * QS;
    const bool v = q < p.HP;
    const int hh = v ? q / p.TWp : 0;
    const int ww = v ? q - hh * p.TWp : 0;
    pix[u] = (uint32_t)(hh * W + ww);
    hw[u] = ((uint32_t)hh << 16) | (uint32_t)ww;
  }
  const uint32_t last_valid = (q0 + (U - 1) * QS) < p.HP ? 1u : 0u;
  const uint32_t dst0 = a_base + j * p.plane_bytes + q0 * 16;
  const uint32_t qs16 = QS * 16;
  const uint32_t bar_full_a = smem_u32(&ctl->full_a[0]), bar_empty_a = smem_u32(&ctl->empty_a[0]);
  const int tpi = p.tiles_w * p.tiles_h;
  const float inv_tpi = 1.f / (float)tpi, inv_tw = 1.f / (float)p.tiles_w;
  const int n_chunks = p.n_chunks;
  const uint32_t n_a = p.n_a;
  // group g stages every chunk of the tiles with CTA-local index = g (mod 2) into its own half of
  // the stage ring, for consumer g
  const int tile_step = 2 * gridDim.x;
  const uint32_t ring_n = n_a / 2;
  const uint32_t ring0 = grp * ring_n;
  int tile = blockIdx.x + grp * gridDim.x;
  // PAIR = 2: a pass covers the group's tiles `tile` and tile + tile_step, k-chunk by k-chunk in
  // the order its consumer takes them: pass chunk ch is k-chunk ch / 2 of the pass's tile ch % 2
  // (`tile` again when tile + tile_step is past the end)
  const int n_chunks_eff = n_chunks * PAIR;
  auto tile_of = [&](int r_tile, int r_ch) {
    return PAIR == 2 && (r_ch & 1) && r_tile + tile_step < p.num_tiles ? r_tile + tile_step : r_tile;
  };
  // x3: besides the TF32 planes every element also goes, as bf16, into the correction planes of
  // its k-step: plane 2*ks holds the low parts a - rn_tf32(a) of the 8 channels, plane 2*ks + 1
  // the high parts (one 16-byte row per pixel each = one K-major core-matrix row of a K = 16 MMA).
  const bool x3 = p.x3 != 0;
  const uint32_t corr_dst0 = a_base + p.corr_off + (j >> 1) * 2 * p.plane_bytes + q0 * 16 + (j & 1) * 8;
  // TMA mode: this group's half of the raw ring, and this thread's first row inside a raw tile
  const uint32_t rn = (uint32_t)p.n_r / 2, rr0 = grp * rn;
  const uint32_t rowb = (uint32_t)p.KC * 4;
  const uint32_t raw_src0 = raw_base + q0 * rowb + j * 16;
  const uint32_t bar_raw_full = smem_u32(&ctl->raw_full[0]), bar_raw_empty = smem_u32(&ctl->raw_empty[0]);
  uint32_t rst = 0, rph = 0;
  // TMA mode: thread 0 of the group copies the raw tile of its k-chunk (r_tile, r_ch) into raw
  // stage rs: one cp.async.bulk.tensor, box {KC channels, TWp, THp} at (c, w_org, h_org, n);
  // coordinates outside the image are zero-filled by the copy engine
  auto issue_raw = [&](int r_tile, int r_ch, uint32_t rs) {
    const int n = r_tile / tpi, rem = r_tile - n * tpi;
    const int th_i = rem / p.tiles_w, tw_i = rem - th_i * p.tiles_w;
    const int h_org = th_i * kTileH - p.dil * (p.taps_h >> 1);
    const int w_org = tw_i * kTileW * p.sub - p.dil * (p.taps_w >> 1);
    const uint32_t bar = bar_raw_full + (rr0 + rs) * 8;
    mbar_arrive_expect_tx(bar, p.raw_bytes);
    const int c = r_ch * p.KC, c_split = p.S.nsrc > 1 ? p.S.s[0].C : (1 << 30);
    tma_load_4d(raw_base + (rr0 + rs) * p.raw_bytes, c < c_split ? tm0 : tm1,
                c < c_split ? c : c - c_split, w_org, h_org, n, bar);
  };
  // the group's k-chunk `ahead` chunks after (r_tile, r_ch), or r_tile >= num_tiles past its last
  auto chunk_after = [&](int& r_tile, int& r_ch, int ahead) {
    r_ch += ahead;
    while (r_ch >= n_chunks_eff) { r_ch -= n_chunks_eff; r_tile += PAIR * tile_step; }
  };
  if (p.tma && gt == 0) {   // the first rn chunks; after that, one per transformed chunk
    for (uint32_t i = 0; i < rn; ++i) {
      int r_tile = tile, r_ch = 0;
      chunk_after(r_tile, r_ch, (int)i);
      if (r_tile < p.num_tiles) issue_raw(tile_of(r_tile, r_ch), r_ch / PAIR, i);
    }
  }
  int ch = 0;
  uint32_t st = 0, ph = 1;   // stage / empty-phase of the current chunk
  for (;;) {
    while (ch >= n_chunks_eff) { ch -= n_chunks_eff; tile += PAIR * tile_step; }
    if (tile >= p.num_tiles) break;
    const int ch_real = ch / PAIR;
    const int cur = tile_of(tile, ch);   // the tile this chunk belongs to
    // cur -> (n, th_i, tw_i) without integer division
    int n = __float2int_rz((float)cur * inv_tpi);
    n += ((n + 1) * tpi <= cur) - (n * tpi > cur);
    const int rem = cur - n * tpi;
    int th_i = __float2int_rz((float)rem * inv_tw);
    th_i += ((th_i + 1) * p.tiles_w <= rem) - (th_i * p.tiles_w > rem);
    const int tw_i = rem - th_i * p.tiles_w;
    const int h_org = th_i * kTileH - p.dil * (p.taps_h >> 1);
    const int w_org = tw_i * kTileW * p.sub - p.dil * (p.taps_w >> 1);
    int c = ch_real * p.KC + j * 4;
    const SrcDev* sp = &p.S.s[0];
    if (p.S.nsrc > 1 && c >= p.S.s[0].C) {
      sp = &p.S.s[1];
      c -= p.S.s[0].C;
    }
    const uint32_t ld = sp->ld;
    const bool pool = sp->pool != 0;            // any on-load resampling (2x2 max or 2x upsampling)
    const int up_mode = sp->pool >= AB_SRC_UP_BILINEAR ? sp->pool : 0;
    const bool has_aff = sp->scale != nullptr;
    float4 sc = make_float4(1.f, 1.f, 1.f, 1.f), sh = make_float4(0.f, 0.f, 0.f, 0.f);
    if (has_aff) {
      sc = __ldg(reinterpret_cast<const float4*>(sp->scale + c));
      sh = __ldg(reinterpret_cast<const float4*>(sp->shift + c));
    }
    const float* base = sp->ptr + c;
    float4 v[U];
    const bool interior = h_org >= 0 && w_org >= 0 && h_org + p.THp <= H && w_org + p.TWp <= W;
    if (p.tma) {
      // the copy engine has staged the raw tile (zero-filled outside the image): registers <-
      // shared memory, then hand the raw stage straight back to the producer
      mbar_wait_quiet(bar_raw_full + (rr0 + rst) * 8, rph);
      const uint32_t rsrc = raw_src0 + (rr0 + rst) * p.raw_bytes;
#pragma unroll
      for (int u = 0; u < U; ++u)
        v[u] = (u < U - 1 || last_valid) ? lds128(rsrc + u * QS * rowb) : make_float4(0.f, 0.f, 0.f, 0.f);
      if (has_aff) {
        if (interior) {
#pragma unroll
          for (int u = 0; u < U; ++u) {
            v[u].x = fmaf(v[u].x, sc.x, sh.x);
            v[u].y = fmaf(v[u].y, sc.y, sh.y);
            v[u].z = fmaf(v[u].z, sc.z, sh.z);
            v[u].w = fmaf(v[u].w, sc.w, sh.w);
          }
        } else {      // zero padding applies AFTER the affine: mask the out-of-image pixels
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int gh = h_org + (int)(hw[u] >> 16), gw = w_org + (int)(hw[u] & 0xFFFFu);
            const bool ok = (unsigned)gh < (unsigned)H && (unsigned)gw < (unsigned)W;
            v[u].x = ok ? fmaf(v[u].x, sc.x, sh.x) : 0.f;
            v[u].y = ok ? fmaf(v[u].y, sc.y, sh.y) : 0.f;
            v[u].z = ok ? fmaf(v[u].z, sc.z, sh.z) : 0.f;
            v[u].w = ok ? fmaf(v[u].w, sc.w, sh.w) : 0.f;
          }
        }
      }
    } else if (!pool && interior) {
      // fast path (~90 % of the tiles of a 512^2 image): one IMAD.WIDE + LDG.128 per element
      const float* tb = base + ((size_t)(n * H + h_org) * W + w_org) * ld;
#pragma unroll
      for (int u = 0; u < U; ++u) v[u] = __ldg(reinterpret_cast<const float4*>(tb + pix[u] * ld));
      if (has_aff) {
#pragma unroll
        for (int u = 0; u < U; ++u) {
          v[u].x = fmaf(v[u].x, sc.x, sh.x);
          v[u].y = fmaf(v[u].y, sc.y, sh.y);
          v[u].z = fmaf(v[u].z, sc.z, sh.z);
          v[u].w = fmaf(v[u].w, sc.w, sh.w);
        }
      }
    } else if (!pool) {
      const size_t img = (size_t)n * H;
      uint32_t okmask = 0;
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int gh = h_org + (int)(hw[u] >> 16), gw = w_org + (int)(hw[u] & 0xFFFFu);
        const bool ok = (unsigned)gh < (unsigned)H && (unsigned)gw < (unsigned)W;
        const int ghc = min(max(gh, 0), H - 1), gwc = min(max(gw, 0), W - 1);
        v[u] = __ldg(reinterpret_cast<const float4*>(base + ((img + ghc) * W + gwc) * ld));
        okmask |= (ok ? 1u : 0u) << u;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const bool ok = (okmask >> u) & 1u;
        v[u].x = ok ? fmaf(v[u].x, sc.x, sh.x) : 0.f;
        v[u].y = ok ? fmaf(v[u].y, sc.y, sh.y) : 0.f;
        v[u].z = ok ? fmaf(v[u].z, sc.z, sh.z) : 0.f;
        v[u].w = ok ? fmaf(v[u].w, sc.w, sh.w) : 0.f;
      }
    } else if (up_mode) {
      // 2x upsampling on load (the decoder's second source, atomai/nets/blocks.py:130-131 +
      // fcnn.py:131-138): the (H/2, W/2) tensor is interpolated while the halo tile is staged,
      // so the 4x larger upsampled tensor is never written or re-read
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int gh = h_org + (int)(hw[u] >> 16), gw = w_org + (int)(hw[u] & 0xFFFFu);
        const bool ok = (unsigned)gh < (unsigned)H && (unsigned)gw < (unsigned)W;
        const int ghc = min(max(gh, 0), H - 1), gwc = min(max(gw, 0), W - 1);
        const float4 a = load_up4(base, (int)ld, up_mode, n, ghc, gwc, H, W);
        v[u] = make_float4(ok ? fmaf(a.x, sc.x, sh.x) : 0.f, ok ? fmaf(a.y, sc.y, sh.y) : 0.f,
                           ok ? fmaf(a.z, sc.z, sh.z) : 0.f, ok ? fmaf(a.w, sc.w, sh.w) : 0.f);
      }
    } else {
      const int H2 = 2 * H, W2 = 2 * W;
      const size_t img = (size_t)n * H2;
      const size_t rs = (size_t)W2 * ld;
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int gh = h_org + (int)(hw[u] >> 16), gw = w_org + (int)(hw[u] & 0xFFFFu);
        const bool ok = (unsigned)gh < (unsigned)H && (unsigned)gw < (unsigned)W;
        const int ghc = min(max(gh, 0), H - 1), gwc = min(max(gw, 0), W - 1);
        const float* q0p = base + ((img + 2 * ghc) * W2 + 2 * gwc) * ld;
        const float4 a0 = __ldg(reinterpret_cast<const float4*>(q0p));
        const float4 a1 = __ldg(reinterpret_cast<const float4*>(q0p + ld));
        const float4 a2 = __ldg(reinterpret_cast<const float4*>(q0p + rs));
        const float4 a3 = __ldg(reinterpret_cast<const float4*>(q0p + rs + ld));
        const float mx = fmaxf(fmaxf(fmaf(a0.x, sc.x, sh.x), fmaf(a1.x, sc.x, sh.x)),
                               fmaxf(fmaf(a2.x, sc.x, sh.x), fmaf(a3.x, sc.x, sh.x)));
        const float my = fmaxf(fmaxf(fmaf(a0.y, sc.y, sh.y), fmaf(a1.y, sc.y, sh.y)),
                               fmaxf(fmaf(a2.y, sc.y, sh.y), fmaf(a3.y, sc.y, sh.y)));
        const float mz = fmaxf(fmaxf(fmaf(a0.z, sc.z, sh.z), fmaf(a1.z, sc.z, sh.z)),
                               fmaxf(fmaf(a2.z, sc.z, sh.z), fmaf(a3.z, sc.z, sh.z)));
        const float mw = fmaxf(fmaxf(fmaf(a0.w, sc.w, sh.w), fmaf(a1.w, sc.w, sh.w)),
                               fmaxf(fmaf(a2.w, sc.w, sh.w), fmaf(a3.w, sc.w, sh.w)));
        v[u] = make_float4(ok ? mx : 0.f, ok ? my : 0.f, ok ? mz : 0.f, ok ? mw : 0.f);
      }
    }
    mbar_wait_quiet(bar_empty_a + (ring0 + st) * 8, ph);
    const uint32_t dst = dst0 + (ring0 + st) * p.a_stage_bytes;
    if (x3) {
      const uint32_t cdst = corr_dst0 + (ring0 + st) * p.a_stage_bytes;
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const float hx = __uint_as_float(tf32_bits(v[u].x) & 0xFFFFE000u);
        const float hy = __uint_as_float(tf32_bits(v[u].y) & 0xFFFFE000u);
        const float hz = __uint_as_float(tf32_bits(v[u].z) & 0xFFFFE000u);
        const float hw_ = __uint_as_float(tf32_bits(v[u].w) & 0xFFFFE000u);
        const uint32_t l01 = pack_bf16x2(v[u].x - hx, v[u].y - hy);
        const uint32_t l23 = pack_bf16x2(v[u].z - hz, v[u].w - hw_);
        const uint32_t h01 = pack_bf16x2(hx, hy), h23 = pack_bf16x2(hz, hw_);
        const uint32_t ok = u == U - 1 ? last_valid : 1u;
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %5, 0;\n\t"
            "@p st.shared.v2.b32 [%0], {%1, %2};\n\t"
            "@p st.shared.v2.b32 [%6], {%3, %4};\n\t}" ::"r"(cdst + u * qs16),
            "r"(l01), "r"(l23), "r"(h01), "r"(h23), "r"(ok),
            "r"(cdst + u * qs16 + (uint32_t)p.plane_bytes)
            : "memory");
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      asm volatile(
          "{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %5, 0;\n\t"
          "@p st.shared.v4.b32 [%0], {%1, %2, %3, %4};\n\t}" ::"r"(dst + u * qs16),
          "r"(tf32_bits(v[u].x)), "r"(tf32_bits(v[u].y)), "r"(tf32_bits(v[u].z)),
          "r"(tf32_bits(v[u].w)), "r"(u == U - 1 ? last_valid : 1u)
          : "memory");
    }
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_full_a + (ring0 + st) * 8);
    if (p.tma) {   // the raw tile has been consumed (the stores above depend on every load of it)
      if (lane == 0) mbar_arrive(bar_raw_empty + (rr0 + rst) * 8);
      if (gt == 0) {   // once all four warps have read it, the stage takes the chunk rn later
        int r_tile = tile, r_ch = ch;
        chunk_after(r_tile, r_ch, (int)rn);
        if (r_tile < p.num_tiles) {
          mbar_wait_quiet(bar_raw_empty + (rr0 + rst) * 8, rph);
          issue_raw(tile_of(r_tile, r_ch), r_ch / PAIR, rst);
        }
      }
      if (++rst == rn) { rst = 0; rph ^= 1; }
    }
    // advance to this group's next chunk
    ++ch;
    if (++st == ring_n) { st = 0; ph ^= 1; }
  }
}

// consumer warpgroup PIPE: the instantiation for this launch's output channels and sub-tiles
template <int PIPE>
__device__ __forceinline__ void conv_consumer(const ConvTcParams& p, SharedCtl* ctl, uint32_t a_base,
                                              uint32_t b_base, float* s_stats, const float* s_bias) {
#define AB_CONS_CASE(NN, S, T) \
  case NN: consumer_loop<NN, S, T, PIPE>(p, ctl, a_base, b_base, s_stats, s_bias); break;
  if (p.pair == 2) {
    switch (p.nn) {
      AB_CONS_CASE(16, 1, 2) AB_CONS_CASE(32, 1, 2)
      default: __trap();
    }
  } else if (p.sub == 2) {
    switch (p.nn) {
      AB_CONS_CASE(16, 2, 1) AB_CONS_CASE(32, 2, 1) AB_CONS_CASE(48, 2, 1) AB_CONS_CASE(64, 2, 1)
      default: __trap();
    }
  } else {
    switch (p.nn) {
      AB_CONS_CASE(16, 1, 1) AB_CONS_CASE(32, 1, 1) AB_CONS_CASE(48, 1, 1) AB_CONS_CASE(64, 1, 1)
      AB_CONS_CASE(80, 1, 1) AB_CONS_CASE(96, 1, 1) AB_CONS_CASE(112, 1, 1) AB_CONS_CASE(128, 1, 1)
      default: __trap();
    }
  }
#undef AB_CONS_CASE
}

constexpr int kCtlBytes = 1024;     // SharedCtl, then the statistics / bias block
static_assert(sizeof(SharedCtl) <= kCtlBytes, "SharedCtl must fit below the statistics block");

__global__ void __launch_bounds__(kThreads, 1)
    conv_tc_kernel(const ConvTcParams p, const __grid_constant__ CUtensorMap tm0,
                   const __grid_constant__ CUtensorMap tm1) {
  extern __shared__ __align__(1024) uint8_t smem[];
  SharedCtl* ctl = reinterpret_cast<SharedCtl*>(smem);
  float* s_stats = reinterpret_cast<float*>(smem + kCtlBytes);  // [4 warps][2][Cout]
  const uint32_t stats_bytes = (kNumEpiWarps * 2 + 1) * p.Cout * sizeof(float);   // + bias copy
  float* s_bias = s_stats + kNumEpiWarps * 2 * p.Cout;
  const uint32_t a_base = smem_u32(smem) + ((kCtlBytes + stats_bytes + 127) & ~127u);
  const uint32_t b_base = a_base + p.n_a * p.a_stage_bytes;
  const uint32_t raw_base = (b_base + p.w_bytes + 127) & ~127u;      // TMA mode (resident weights)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.n_a; ++i) {
      mbar_init(smem_u32(&ctl->full_a[i]), kNumLoadWarps / 2);
      mbar_init(smem_u32(&ctl->empty_a[i]), kNumEpiWarps);
    }
    for (int i = 0; i < p.n_b; ++i) mbar_init(smem_u32(&ctl->full_b[i]), 1);
    for (int i = 0; i < kMaxRStages; ++i) {
      mbar_init(smem_u32(&ctl->raw_full[i]), 1);
      mbar_init(smem_u32(&ctl->raw_empty[i]), kNumLoadWarps / 2);
    }
    mbar_init(smem_u32(&ctl->w_full), 1);
    fence_barrier_init();
  }
  if (warp < kNumEpiWarps) {
    for (int i = lane; i < 2 * p.Cout; i += 32) s_stats[warp * 2 * p.Cout + i] = 0.f;
    if (warp == 0)
      for (int i = lane; i < p.Cout; i += 32) s_bias[i] = p.bias ? __ldg(p.bias + i) : 0.f;
  }
  __syncthreads();

  if (warp >= kFirstLoadWarp) {
    setmaxnreg_dec<kRegsLoad>();
    // ===================== activation loaders =====================
    // Two groups of 4 warps; group g stages every k-chunk of the tiles with local index = g
    // (mod 2), so two chunks are always in flight per SM.  Per thread the (halo row, halo col) of
    // each of its <= kMaxU 16-byte elements is fixed for the whole kernel (no divisions in the
    // loop); loads are issued branch-free from clamped addresses and masked afterwards, so the
    // compiler keeps all of them in flight before the first use.
    const int grp = (warp - kFirstLoadWarp) >> 2;
    const int U = (p.HP * (p.KC >> 2) + kGroupThreads - 1) / kGroupThreads;   // <= kMaxU (plan)
    if (p.pair == 2) {   // the plan pairs only these element counts
      switch (U) {
        case 2: loader_loop<2, 2>(p, ctl, a_base, raw_base, grp, &tm0, &tm1); break;
        case 4: loader_loop<4, 2>(p, ctl, a_base, raw_base, grp, &tm0, &tm1); break;
        default: __trap();
      }
    } else switch (U) {
#define AB_LOAD_CASE(K) case K: loader_loop<K, 1>(p, ctl, a_base, raw_base, grp, &tm0, &tm1); break;
      AB_LOAD_CASE(1) AB_LOAD_CASE(2) AB_LOAD_CASE(3) AB_LOAD_CASE(4) AB_LOAD_CASE(5) AB_LOAD_CASE(6)
      AB_LOAD_CASE(7) AB_LOAD_CASE(8) AB_LOAD_CASE(9) AB_LOAD_CASE(10) AB_LOAD_CASE(11)
      AB_LOAD_CASE(12)
#undef AB_LOAD_CASE
      default: __trap();
    }
  } else {
    // ===================== consumers: wgmma + epilogue =====================
    if (p.w_resident && threadIdx.x == 0) {
      // the packed blob is already in shared-memory order: copy it once, in 16 KB pieces
      const uint32_t bar = smem_u32(&ctl->w_full);
      mbar_arrive_expect_tx(bar, p.w_bytes);
      for (int off = 0; off < p.w_bytes; off += 16384) {
        const int n = min(16384, p.w_bytes - off);
        bulk_g2s(b_base + off, reinterpret_cast<const char*>(p.wblob) + off, n, bar);
      }
    }
    // one branch per consumer ahead of setmaxnreg (.sync.aligned: each warpgroup is converged
    // after it), so nothing in a consumer's wgmma code depends on the thread index
    if (warp < kNumEpiWarps) {
      setmaxnreg_inc<kRegsCons>();
      conv_consumer<0>(p, ctl, a_base, b_base, s_stats, s_bias);
    } else {
      setmaxnreg_inc<kRegsCons>();
      conv_consumer<1>(p, ctl, a_base, b_base, s_stats, s_bias);
    }
  }
  __syncthreads();
}

// ---------------------------------------------------------------- weight packing (TF32 blobs)
// blob[k-step s (8 channels)][tap][plane j (2)][n][4]  <-  W, RN-rounded to TF32.  One (s, tap)
// piece is a ready-made K-major B operand for one wgmma (N rows x 8 k).
//   FWD  : B[n = co][k = ci]            = W[co][ci][ty][tx]
//   DGRAD: B[n = ci][k = co] (roles swap) = W[co][ci][Th-1-ty][Tw-1-tx]
// x3 (AB_MATH_TF32X3): blob[k-step][kind (main, corr)][tap][plane][n][4 words]: the main piece as
// above (hi = rn_tf32(W)); the correction piece is the K-major bf16 B operand of a K = 16 MMA,
// plane 0 = bf16(W) of the k-step's 8 channels (meets the activations' low parts), plane 1 =
// bf16(W - hi) (meets their high parts): a_hi*w_hi + (a_lo*w + a_hi*w_lo) ~ 2^-20 relative.
__global__ void pack_weights_tc_kernel(const float* __restrict__ w, int Cout, int Cin, int th,
                                       int tw, int mode, int x3, float* __restrict__ out,
                                       int64_t total) {
  const int taps = th * tw;
  const int Nn = mode == AB_WMODE_FWD ? Cout : Cin;   // GEMM N (rows of B)
  const int Kk = mode == AB_WMODE_FWD ? Cin : Cout;   // GEMM K per tap
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i;
    const int e = r % 4; r /= 4;
    const int nn = r % Nn; r /= Nn;
    const int j = r % 2; r /= 2;
    const int t = r % taps; r /= taps;
    int kind = 0;
    if (x3) { kind = r % 2; r /= 2; }
    const int ks = (int)r;
    const int ty = t / tw, tx = t % tw;
    auto wv = [&](int k) -> float {
      if (k >= Kk) return 0.f;
      return mode == AB_WMODE_FWD
                 ? w[(((int64_t)nn * Cin + k) * th + ty) * tw + tx]
                 : w[(((int64_t)k * Cin + nn) * th + (th - 1 - ty)) * tw + (tw - 1 - tx)];
    };
    if (!kind) {
      out[i] = to_tf32(wv(ks * 8 + j * 4 + e));
    } else {   // word e of plane j holds channels ks*8 + 2e, 2e + 1 as bf16 (j: 0 = W, 1 = W - hi)
      const float v0 = wv(ks * 8 + 2 * e), v1 = wv(ks * 8 + 2 * e + 1);
      const float a0 = j ? v0 - to_tf32(v0) : v0, a1 = j ? v1 - to_tf32(v1) : v1;
      out[i] = __uint_as_float(pack_bf16x2(a0, a1));
    }
  }
}

int pick_kc(int Ctot) { return Ctot % 32 == 0 ? 32 : (Ctot % 16 == 0 ? 16 : 8); }

}  // namespace

// exported to api.cu ---------------------------------------------------------------
int ab_conv_tc_supported(const ab_conv_t* d) {
  int ctot = 0;
  for (int i = 0; i < d->nsrc; ++i) {
    if (d->src[i].C % 4 != 0 || d->src[i].ld % 4 != 0) return 0;
    if (((uintptr_t)d->src[i].ptr & 15) != 0) return 0;
    ctot += d->src[i].C;
  }
  if (ctot % 8 != 0) return 0;
  if (d->Cout % 16 != 0 || d->Cout < 16 || d->Cout > 256) return 0;
  return 1;
}

int64_t ab_pack_weights_tc_elems(int Cout, int Cin, int th, int tw, int mode, int x3) {
  const int Nn = mode == AB_WMODE_FWD ? Cout : Cin;
  const int Kk = mode == AB_WMODE_FWD ? Cin : Cout;
  return (int64_t)(Kk / 8) * th * tw * 8 * Nn * (x3 ? 2 : 1);
}

int ab_pack_weights_tc(const float* w, int Cout, int Cin, int th, int tw, int mode, int x3,
                       float* out, cudaStream_t stream) {
  const int Kk = mode == AB_WMODE_FWD ? Cin : Cout;
  AB_CHECK(Kk % 8 == 0, "tf32 weight pack: K=%d not a multiple of 8", Kk);
  const int64_t total = ab_pack_weights_tc_elems(Cout, Cin, th, tw, mode, x3);
  const int threads = 256;
  const int blocks = (int)((total + threads - 1) / threads);
  pack_weights_tc_kernel<<<blocks > 4096 ? 4096 : blocks, threads, 0, stream>>>(
      w, Cout, Cin, th, tw, mode, x3, out, total);
  AB_LAUNCH_CHECK();
  return 0;
}

// Environment overrides of the tile-plan search, read once per plan (the tests set them between
// calls to force every plan variant; tools/plan_ab.py and tools/show_plans.py sweep them).
struct PlanKnobs {
  int budget = 224 * 1024;   // ATOMAI_B200_SMEM_KB (64..224): shared memory the plan may use
  int na4 = 3;               // ATOMAI_B200_NA4: operand-ring preference bits (see conv_tc_plan)
  int min_nr = 4;            // ATOMAI_B200_MIN_NR (>= 2): fewest raw stages of a TMA plan
  int attempt = -1, kc = 0;  // ATOMAI_B200_PLAN="<attempt>,<KC>": pin the weight mode / k-chunk
  bool tma = true;           // ATOMAI_B200_TMA=0: register-staged loaders only
  int res_na4 = -1;          // ATOMAI_B200_RES_NA4=0/1: resident n_a = 4 rule for no / every layer
  int tma_min_kc = 16;       // ATOMAI_B200_TMA_KC8 (set): TMA plans may use 32-byte box rows
  bool pair = true;          // ATOMAI_B200_PAIR=0: thin layers take one tile per consumer pass
  bool log = false;          // ATOMAI_B200_PLAN_LOG (set): print every plan to stderr
};

static PlanKnobs plan_knobs() {
  PlanKnobs k;
  if (const char* e = getenv("ATOMAI_B200_SMEM_KB")) {
    const int kb = atoi(e);
    if (kb >= 64 && kb <= 224) k.budget = kb * 1024;
  }
  if (const char* e = getenv("ATOMAI_B200_NA4")) k.na4 = atoi(e);
  if (const char* e = getenv("ATOMAI_B200_MIN_NR")) k.min_nr = atoi(e) < 2 ? 2 : atoi(e);
  if (const char* e = getenv("ATOMAI_B200_PLAN")) sscanf(e, "%d,%d", &k.attempt, &k.kc);
  if (const char* e = getenv("ATOMAI_B200_TMA")) k.tma = e[0] != '0';
  if (const char* e = getenv("ATOMAI_B200_RES_NA4")) k.res_na4 = e[0] == '1' ? 1 : 0;
  if (getenv("ATOMAI_B200_TMA_KC8")) k.tma_min_kc = 8;
  if (const char* e = getenv("ATOMAI_B200_PAIR")) k.pair = e[0] != '0';
  k.log = getenv("ATOMAI_B200_PLAN_LOG") != nullptr;
  return k;
}

// Operand and weight stages of a k-chunk of KC channels: P = KC/4 planes of HP pixels x 16 B, the
// plane stride padded so that the P planes start 128/P bytes apart mod 128 (spread over the
// banks); x3 doubles both for the bf16 correction planes.  false: more 16-byte elements than the
// register-staged loaders hold.
struct Chunk { int KC, plane, a_stage, b_stage; };

static bool chunk_stages(int HP, int KC, int Cout, int x3, Chunk* c) {
  const int P = KC / 4;
  if (HP * P > kMaxU * kGroupThreads) return false;
  int plane = HP * 16;
  const int want = (128 / P) % 128;
  plane += ((want - plane % 128) + 128) % 128;
  *c = {KC, plane, P * plane * (x3 ? 2 : 1), KC * Cout * 4 * (x3 ? 2 : 1)};
  return true;
}

static void set_chunk(ConvTcParams* p, const Chunk& c) {
  p->KC = c.KC; p->plane_bytes = c.plane; p->a_stage_bytes = c.a_stage; p->b_stage_bytes = c.b_stage;
  p->corr_off = c.KC / 4 * c.plane;
}

// Shared memory of everything but the stages: the statistics / control block and, for resident
// weights, the whole packed weight blob
static int fixed_smem(const ConvTcParams& p, int stats_bytes, int resident) {
  return stats_bytes + (resident ? (p.w_bytes + 127) & ~127 : 0);
}

static int plan_smem(const ConvTcParams& p, int stats_bytes) {
  return fixed_smem(p, stats_bytes, p.w_resident) + p.n_a * p.a_stage_bytes + p.n_b * p.b_stage_bytes +
         p.n_r * p.raw_bytes + (p.tma ? 128 : 0);
}

static int conv_tc_plan(const ab_conv_t* d, ConvTcParams* p, int* smem_bytes) {
  SrcSet S;
  if (ab_make_srcset(d, &S)) return 1;
  const PlanKnobs k = plan_knobs();
  p->S = S;
  p->N = d->N; p->H = d->H; p->W = d->W; p->Cout = d->Cout;
  p->taps_h = d->ks_h; p->taps_w = d->ks_w; p->dil = d->dil;
  p->alpha = d->lrelu;
  p->act = d->act;
  p->out_nchw = d->out_nchw;
  const int taps = d->ks_h * d->ks_w;
  p->x3 = d->math == AB_MATH_TF32X3 ? 1 : 0;
  p->w_bytes = taps * S.Ctot * d->Cout * 4 * (p->x3 ? 2 : 1);
  // 1 CTA / SM: 227 KB of dynamic shared memory are addressable (226 KB opted in below);
  // the plan uses k.budget of them
  // Operand-ring preference.  Every pipeline owns n_a/2 operand stages; with n_a = 2 the loader
  // group and the consumer strictly alternate on a pipeline (stage -> MMA -> stage ...) and only
  // the *other* pipeline hides the hand-over.  Buying the deeper ring with 8-channel k-chunks does
  // not pay when the loaders are the heavy side (pooled sources, register-staged resident
  // layers), so pass 0 of the search only drops to KC = 8 for streamed-weight layers with plain
  // sources.
  // k.na4 bit 0: resident-weight plans prefer n_a = 4 over more raw TMA stages;
  // bit 1: streamed-weight plans prefer n_a = 4 over a larger k-chunk / more weight stages.
  // TMA mode needs at least k.min_nr raw stages (two rings of min_nr/2), else the plan stays
  // register-staged: with one raw stage per pipeline every k-chunk pays the full HBM latency
  bool any_pool = false;
  for (int i = 0; i < S.nsrc; ++i) any_pool = any_pool || S.s[i].pool != 0;
  const int stats_bytes = (((kNumEpiWarps * 2 + 1) * d->Cout * 4 + 127) & ~127) + kCtlBytes + 128;
  // Try, in order of preference: (resident weights, 1 sub-tile), (streamed weights, 2 sub-tiles
  // so that every weight stage feeds M = 256), (streamed, 1 sub-tile).
  bool ok = false;
  // Resident weights that leave only n_a = 2 vs streamed weights with n_a = 4: streaming wins only
  // where the weight ring gets deep enough to cover the L2 latency, i.e. for the two-source
  // decoder convolution onto <= 32 channels.  So: for that layer class a resident plan must reach
  // n_a = 4, else a streamed plan with >= 12 weight stages is preferred; the resident n_a = 2 plan
  // stays the fallback.  ATOMAI_B200_RES_NA4 = 0 disables, = 1 applies the rule to every layer.
  int strict0 = (p->x3 && S.nsrc == 2 && !any_pool && taps == 9 && d->Cout <= 32) ? 1 : 0;
  if (k.res_na4 >= 0) strict0 = k.res_na4;
  for (int strict = strict0; strict >= 0 && !ok; --strict)
  for (int attempt = 0; attempt < 3 && !ok; ++attempt) {
    if (k.attempt >= 0 && attempt != k.attempt) continue;
    const int resident = attempt == 0;
    const int sub = attempt == 1 ? 2 : 1;
    if (sub == 2 && (d->Cout > kMaxN / 2 || d->W <= kTileW)) continue;   // SUB * N accumulators
    p->tiles_h = (d->H + kTileH - 1) / kTileH;
    p->tiles_w = (d->W + kTileW * sub - 1) / (kTileW * sub);
    p->THp = kTileH + d->dil * (d->ks_h - 1);
    p->TWp = kTileW * sub + d->dil * (d->ks_w - 1);
    p->HP = p->THp * p->TWp;
    const int avail = k.budget - fixed_smem(*p, stats_bytes, resident);
    // pass 0 (only when this weight mode prefers deep operand rings, or for a strict resident
    // plan) accepts a k-chunk only if it leaves room for n_a = 4; pass 1 is the plain "largest
    // k-chunk with n_a >= 2" search
    for (int pass = (k.na4 & (resident ? 1 : 2)) ? 0 : 1; pass < 2 && !ok; ++pass)
    for (int KC = pick_kc(S.Ctot); KC >= 8 && !ok; KC >>= 1) {
      const int need_a = pass == 0 || (strict && resident) ? 4 : 2;
      Chunk c;
      if (S.Ctot % KC != 0 || (k.kc > 0 && KC != k.kc) || !chunk_stages(p->HP, KC, d->Cout, p->x3, &c))
        continue;
      if (need_a == 4 && KC < 16 && (resident || any_pool)) continue;
      int n_b = 0;
      if (!resident) {
        // weight stages: cover the L2 latency, leave room for the activation stages
        n_b = ((avail - need_a * c.a_stage) / c.b_stage) & ~1;      // two rings of n_b/2 stages
        if (n_b > kMaxBStages) n_b = kMaxBStages;
        if (n_b < (strict ? 12 : 4)) continue;
      }
      const int na = (avail - n_b * c.b_stage) / c.a_stage;
      if (na < need_a) continue;
      set_chunk(p, c);
      p->n_a = (na > kMaxAStages ? kMaxAStages : na) & ~1;   // two rings of n_a/2 stages
      p->n_b = n_b; p->sub = sub; p->w_resident = resident;
      p->tma = 0; p->n_r = 0; p->raw_bytes = 0;
      ok = true;
    }
    // TMA mode (resident weights, un-pooled sources, sources split on a chunk boundary): choose
    // the (KC, operand stages, raw stages) with the most raw bytes in flight
    if (ok && resident && k.tma && !S.s[0].pool && !(S.nsrc > 1 && S.s[1].pool)) {
      int best_bytes = 0;
      for (int KC = pick_kc(S.Ctot); KC >= k.tma_min_kc; KC >>= 1) {
        Chunk c;
        if (S.Ctot % KC != 0 || (S.nsrc > 1 && S.s[0].C % KC != 0) || (k.kc > 0 && KC != k.kc) ||
            !chunk_stages(p->HP, KC, d->Cout, p->x3, &c))
          continue;
        const int raw = p->HP * KC * 4;
        if (raw % 128 != 0) continue;
        for (int na = 4; na >= ((k.na4 & 1) ? 4 : 2); na -= 2) {
          int nr = ((avail - na * c.a_stage) / raw) & ~1;
          if (nr > kMaxRStages) nr = kMaxRStages;
          if (nr < k.min_nr) continue;
          // raw bytes in flight decide; with the n_a = 4 preference a double-buffered operand
          // ring outranks any number of raw stages
          const int score = nr * raw + (na == 4 ? ((k.na4 & 1) ? (1 << 24) : 1) : 0);
          if (score > best_bytes) {
            best_bytes = score;
            set_chunk(p, c);
            p->n_a = na; p->n_r = nr; p->raw_bytes = raw; p->tma = 1;
          }
        }
      }
    }
  }
  AB_CHECK(ok, "conv_tc: no shared-memory plan (Cin=%d Cout=%d dil=%d)", S.Ctot, d->Cout, d->dil);
  p->num_tiles = d->N * p->tiles_h * p->tiles_w;
  p->n_chunks = S.Ctot / p->KC;
  // Thin 3x3 layers (one launch of <= 32 channels: at most 32 accumulator registers per tile)
  // issue the MMAs of two tiles back to back.  A pass holds one operand stage per tile, so the
  // pipeline's ring must have two; a pipeline needs two tiles for a pass to add a chain (with
  // num_tiles <= 2 * grid every pass would be a lone tile, staged and multiplied twice); the
  // loader has paired instantiations for 2 and 4 elements per thread only (KC = 8 / 16 at
  // dilation 1).  A 1x1 layer's k-chunk is too few MMAs to pay for retiring every group before
  // the next chunk is staged.
  {
    const int u = (p->HP * (p->KC >> 2) + kGroupThreads - 1) / kGroupThreads;
    const int sms = ab_num_sms(), grid = p->num_tiles < sms ? p->num_tiles : sms;
    p->pair = (k.pair && p->w_resident && p->sub == 1 && d->Cout <= 32 && p->n_a == 4 && taps > 1 &&
               p->num_tiles > 2 * grid && (u == 2 || u == 4)) ? 2 : 1;
  }
  AB_CHECK(p->plane_bytes / 16 < (1 << 14) && p->TWp < (1 << 14), "conv_tc: descriptor overflow");
  *smem_bytes = plan_smem(*p, stats_bytes);
  if (k.log)
    fprintf(stderr,
            "conv_tc plan: %dx%d Cin=%d Cout=%d taps=%d x3=%d | resident=%d sub=%d KC=%d n_a=%d "
            "n_b=%d tma=%d n_r=%d a_stage=%d smem=%d\n",
            d->H, d->W, S.Ctot, d->Cout, taps, p->x3, p->w_resident, p->sub, p->KC, p->n_a, p->n_b,
            p->tma, p->n_r, p->a_stage_bytes, *smem_bytes);
  if (k.log)
    fprintf(stderr, "conv_tc tile: 8x%d px, %d tile(s) per consumer pass\n", kTileW * p->sub, p->pair);
  return 0;
}

// 4-D tensor map {C, W, H, N} of one NHWC source (pixel stride ld) with box {KC, TWp, THp, 1}
static int make_src_tmap(const SrcDev& s, int N, int H, int W, int KC, int TWp, int THp,
                         CUtensorMap* out) {
  typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static EncodeTiledFn encode = nullptr;
  if (!encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    AB_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
    AB_CHECK(fn != nullptr && q == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available");
    encode = reinterpret_cast<EncodeTiledFn>(fn);
  }
  const cuuint64_t dims[4] = {(cuuint64_t)s.C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  const cuuint64_t strides[3] = {(cuuint64_t)s.ld * 4, (cuuint64_t)W * s.ld * 4,
                                 (cuuint64_t)H * W * s.ld * 4};
  const cuuint32_t box[4] = {(cuuint32_t)KC, (cuuint32_t)TWp, (cuuint32_t)THp, 1};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  const CUresult r = encode(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(s.ptr), dims,
                            strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  AB_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  return 0;
}

int ab_conv_tc_info(const ab_conv_t* d, int* grid, int* block, int* smem_bytes) {
  ConvTcParams p;
  if (conv_tc_plan(d, &p, smem_bytes)) return 1;
  const int sms = ab_num_sms();
  *grid = p.num_tiles < sms ? p.num_tiles : sms;
  *block = kThreads;
  return 0;
}

int ab_conv_tc_fwd(const ab_conv_t* d, const float* wblob, const float* bias, float* y, int ld_y,
                   double* stats, cudaStream_t stream) {
  ConvTcParams p;
  int smem_bytes = 0;
  if (conv_tc_plan(d, &p, &smem_bytes)) return 1;
  AB_CHECK(((uintptr_t)wblob & 15) == 0 && ((uintptr_t)y & 15) == 0 && (d->out_nchw || ld_y % 4 == 0),
           "conv_tc: unaligned weight blob / output");
  p.wblob = wblob; p.bias = bias; p.out = y; p.ld_out = ld_y; p.stats = stats;
  // NCHW output: ld_y < 0 gives the pitch between channel planes (the Gram kernel writes
  // K[row = channel][col = pixel] with the caller's leading dimension); default H*W
  p.nchw_stride = (d->out_nchw && ld_y < 0) ? -(int64_t)ld_y : (int64_t)d->H * d->W;
  static unsigned char optin[64];
  if (ab_optin_smem(reinterpret_cast<const void*>(conv_tc_kernel), 226 * 1024, optin)) return 1;
  const int sms = ab_num_sms();
  const int grid = p.num_tiles < sms ? p.num_tiles : sms;
  if (grid == 0) return 0;
  if (stats && ab_ordered_ws(stream, (int64_t)grid * 2 * kMaxN, 1, &p.red)) return 1;
  CUtensorMap tm0, tm1;
  memset(&tm0, 0, sizeof(tm0));
  memset(&tm1, 0, sizeof(tm1));
  if (p.tma) {
    if (make_src_tmap(p.S.s[0], p.N, p.H, p.W, p.KC, p.TWp, p.THp, &tm0)) return 1;
    if (p.S.nsrc > 1 && make_src_tmap(p.S.s[1], p.N, p.H, p.W, p.KC, p.TWp, p.THp, &tm1)) return 1;
  }
  // one launch per <= 128 output channels (the consumer's accumulator registers)
  for (int n0 = 0; n0 < d->Cout; n0 += kMaxN) {
    p.n0 = n0;
    p.nn = d->Cout - n0 < kMaxN ? d->Cout - n0 : kMaxN;
    conv_tc_kernel<<<grid, kThreads, smem_bytes, stream>>>(p, tm0, tm1);
    AB_LAUNCH_CHECK();
  }
  return 0;
}
