// vae.cu — the non-convolutional pieces of the VAE / rVAE / ImSpec / DKL paths:
//   * a strided fp32 GEMM with optional split-K (skinny nn.Linear layers: 524288 -> latent
//     heads of convEncoderNet, latent -> 524288 of convDecoderNet, the fcFeatureExtractor MLP);
//   * coord_latent fused with transform_coordinates (rVAE spatial decoder, first layer).
// Reference call sites: atomai/nets/ed.py:64,273-274,503-505 (Linear), :672-687 (coord_latent),
// atomai/utils/coords.py:47-83, atomai/models/dgm/rvae.py:118-145, atomai/nets/gp.py:14-26.
#include "common.cuh"

namespace {

constexpr int TM = 64, TN = 64, TK = 16, GT = 256;

struct GemmParams {
  const float* A; int64_t a_sm, a_sk;
  const float* B; int64_t b_sk, b_sn;
  float* C; int64_t c_sm;
  int M, N, K;
  const float* bias;
  int act; float slope;
  int accumulate;  // C += act(A.B + bias) (plain add when split_k == 1, atomics otherwise)
  int split_k, k_per_split;
};

// C tile 64x64, 256 threads, 4x4 micro-tile.  Tile loads walk the contiguous axis of each
// operand with consecutive threads (decided from the strides) so they stay coalesced for
// NN / NT / TN shapes alike.
__global__ void __launch_bounds__(GT) gemm_kernel(const GemmParams p) {
  __shared__ float sA[TK][TM + 4];
  __shared__ float sB[TK][TN + 4];
  const int m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
  const int k_begin = blockIdx.z * p.k_per_split;
  const int k_end = min(p.K, k_begin + p.k_per_split);
  const int tid = threadIdx.x;
  const int tm = (tid >> 4) * 4, tn = (tid & 15) * 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  const bool a_k_fast = p.a_sk == 1;  // A contiguous along k
  const bool b_n_fast = p.b_sn == 1;  // B contiguous along n

  for (int k0 = k_begin; k0 < k_end; k0 += TK) {
    __syncthreads();
    for (int i = tid; i < TM * TK; i += GT) {
      int m, k;
      if (a_k_fast) { k = i % TK; m = i / TK; } else { m = i % TM; k = i / TM; }
      float v = 0.f;
      if (m0 + m < p.M && k0 + k < k_end) v = __ldg(p.A + (int64_t)(m0 + m) * p.a_sm + (int64_t)(k0 + k) * p.a_sk);
      sA[k][m] = v;
    }
    for (int i = tid; i < TN * TK; i += GT) {
      int n, k;
      if (b_n_fast) { n = i % TN; k = i / TN; } else { k = i % TK; n = i / TK; }
      float v = 0.f;
      if (n0 + n < p.N && k0 + k < k_end) v = __ldg(p.B + (int64_t)(k0 + k) * p.b_sk + (int64_t)(n0 + n) * p.b_sn);
      sB[k][n] = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < TK; ++k) {
      const float4 a4 = *reinterpret_cast<const float4*>(&sA[k][tm]);
      const float4 b4 = *reinterpret_cast<const float4*>(&sB[k][tn]);
      const float av[4] = {a4.x, a4.y, a4.z, a4.w};
      const float bv[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + tm + i;
    if (m >= p.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tn + j;
      if (n >= p.N) continue;
      float* c = p.C + (int64_t)m * p.c_sm + n;
      if (p.split_k > 1) {
        // C already holds the bias (bias_fill_kernel) unless accumulating; then the first K
        // slice adds it, so that C += A.B + bias on every path
        float v = acc[i][j];
        if (p.accumulate && p.bias && blockIdx.z == 0) v += __ldg(p.bias + n);
        atomicAdd(c, v);
      } else {
        float v = acc[i][j] + (p.bias ? __ldg(p.bias + n) : 0.f);
        v = act_f(v, p.act, p.slope);
        *c = p.accumulate ? *c + v : v;
      }
    }
  }
}

__global__ void bias_fill_kernel(float* C, int64_t c_sm, int M, int N, const float* bias) {
  const int64_t total = (int64_t)M * N;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int n = (int)(i % N);
    C[(i / N) * c_sm + n] = bias ? bias[n] : 0.f;
  }
}


// ---------------------------------------------------------------- skinny nn.Linear (O <= 16)
// The latent heads of the VAE / ImSpec encoders (atomai/nets/ed.py:64,273-274: 262144..524288
// inputs -> 2..13 outputs) are pure HBM streams over the activations: B x K floats read once,
// a handful of outputs.  The 64x64 GEMM tile above wastes 59/64 of its B-operand lanes on them and
// reads x in 64-byte pieces;
// these kernels read x / write dx as whole rows of float4 and keep the O-wide side in shared
// memory or registers.
constexpr int SK_T = 256;          // threads
constexpr int SK_KS = 1024;        // k per CTA (one float4 per thread)
constexpr int SK_MAXO = 16;

// y[b][o] (+)= sum_{k in slice} x[b][k] w[o][k]: CTA = one k-slice, thread = 4 k, loop over rows;
// per row a warp reduces its O partial sums with shuffles and adds them into y (pre-filled with the
// bias by the caller)
__global__ void __launch_bounds__(SK_T) skinny_fwd_kernel(const float* __restrict__ x,
                                                           const float* __restrict__ w,
                                                           float* __restrict__ y, int B, int K, int O) {
  const int k = blockIdx.x * SK_KS + threadIdx.x * 4;
  const bool in = k < K;                     // K % 4 == 0: a thread's 4 k are all in or all out
  float4 wv[SK_MAXO];
#pragma unroll
  for (int o = 0; o < SK_MAXO; ++o)
    wv[o] = (in && o < O) ? __ldg(reinterpret_cast<const float4*>(w + (size_t)o * K + k))
                          : make_float4(0.f, 0.f, 0.f, 0.f);
  __shared__ float s_part[SK_T / 32][SK_MAXO];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int b = blockIdx.y; b < B; b += gridDim.y) {
    const float4 xv = in ? __ldg(reinterpret_cast<const float4*>(x + (size_t)b * K + k))
                         : make_float4(0.f, 0.f, 0.f, 0.f);
    float acc[SK_MAXO];
#pragma unroll
    for (int o = 0; o < SK_MAXO; ++o)
      acc[o] = fmaf(xv.x, wv[o].x, fmaf(xv.y, wv[o].y, fmaf(xv.z, wv[o].z, xv.w * wv[o].w)));
#pragma unroll
    for (int o = 0; o < SK_MAXO; ++o) {
      if (o < O) {
        float a = acc[o];
#pragma unroll
        for (int sft = 16; sft >= 1; sft >>= 1) a += __shfl_xor_sync(0xffffffffu, a, sft);
        if (lane == 0) s_part[warp][o] = a;
      }
    }
    __syncthreads();
    if (threadIdx.x < O) {
      float t = 0.f;
#pragma unroll
      for (int wi = 0; wi < SK_T / 32; ++wi) t += s_part[wi][threadIdx.x];
      atomicAdd(y + (size_t)b * O + threadIdx.x, t);
    }
    __syncthreads();
  }
}

// dx[b][k] = sum_o dy[b][o] w[o][k]   and   dw[o][k] = sum_b dy[b][o] x[b][k]  in ONE pass over the
// rows: a thread owns 4 consecutive k (its w in registers), dy lives in shared memory
constexpr int SK_TB = 128, SK_KSB = 512;   // backward: 128 threads x 4 k (two O-wide float4 sets per thread)
template <int MAXO>
__global__ void __launch_bounds__(SK_TB) skinny_bwd_kernel(const float* __restrict__ x,
                                                           const float* __restrict__ w,
                                                           const float* __restrict__ dy,
                                                           float* __restrict__ dx,
                                                           float* __restrict__ dw, int B, int K, int O) {
  extern __shared__ float s_dy[];            // [B][O]
  for (int i = threadIdx.x; i < B * O; i += SK_TB) s_dy[i] = __ldg(dy + i);
  __syncthreads();
  const int k = blockIdx.x * SK_KSB + threadIdx.x * 4;
  if (k >= K) return;
  float4 wv[MAXO], gw[MAXO];
#pragma unroll
  for (int o = 0; o < MAXO; ++o) {
    wv[o] = (dx && o < O) ? __ldg(reinterpret_cast<const float4*>(w + (size_t)o * K + k))
                          : make_float4(0.f, 0.f, 0.f, 0.f);
    gw[o] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  constexpr int RB = 4;                      // rows in flight
  for (int b0 = 0; b0 < B; b0 += RB) {
    float4 xv[RB];
    if (dw) {
#pragma unroll
      for (int r = 0; r < RB; ++r)
        xv[r] = b0 + r < B ? __ldg(reinterpret_cast<const float4*>(x + (size_t)(b0 + r) * K + k))
                           : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int r = 0; r < RB; ++r) {
      if (b0 + r >= B) break;
      const float* d = s_dy + (b0 + r) * O;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int o = 0; o < MAXO; ++o) {
        if (o < O) {
          const float g = d[o];
          if (dw) {
            gw[o].x = fmaf(g, xv[r].x, gw[o].x); gw[o].y = fmaf(g, xv[r].y, gw[o].y);
            gw[o].z = fmaf(g, xv[r].z, gw[o].z); gw[o].w = fmaf(g, xv[r].w, gw[o].w);
          }
          acc.x = fmaf(g, wv[o].x, acc.x); acc.y = fmaf(g, wv[o].y, acc.y);
          acc.z = fmaf(g, wv[o].z, acc.z); acc.w = fmaf(g, wv[o].w, acc.w);
        }
      }
      if (dx) *reinterpret_cast<float4*>(dx + (size_t)(b0 + r) * K + k) = acc;
    }
  }
  if (dw) {
#pragma unroll
    for (int o = 0; o < MAXO; ++o)
      if (o < O) *reinterpret_cast<float4*>(dw + (size_t)o * K + k) = gw[o];
  }
}

inline bool skinny_ok(const void* a, const void* b, const void* c, int B, int K, int O) {
  const auto al = [](const void* p) { return p == nullptr || ((uintptr_t)p & 15) == 0; };
  return O >= 1 && O <= SK_MAXO && K % 4 == 0 && K >= 4 * SK_KS && B >= 1 && al(a) && al(b) && al(c);
}

// ---------------------------------------------------------------- coord_latent
struct CoordDev {
  int B, H, W, zdim, hid, tanh_act;
  const float *z, *phi, *dx, *wc, *bc, *wz;
};

__device__ __forceinline__ void grid_xy(const CoordDev& d, int p, float& gx, float& gy) {
  // imcoordgrid (atomai/utils/coords.py:47-54): x = linspace(-1,1,H)[i] slowest, y = linspace(1,-1,W)[j]
  const int i = p / d.W, j = p - i * d.W;
  gx = d.H > 1 ? -1.f + 2.f * i / (float)(d.H - 1) : -1.f;
  gy = d.W > 1 ? 1.f - 2.f * j / (float)(d.W - 1) : 1.f;
}
// per-sample part of transform_coordinates (hoisted out of the pixel loops: sincosf alone was a
// third of the instructions of these kernels)
struct Xf { float c, s, tx, ty; };
__device__ __forceinline__ Xf xform_setup(const CoordDev& d, int b) {
  Xf t; t.c = 1.f; t.s = 0.f; t.tx = 0.f; t.ty = 0.f;
  if (d.phi) { sincosf(d.phi[b], &t.s, &t.c); }
  if (d.dx) { t.tx = d.dx[b * 2]; t.ty = d.dx[b * 2 + 1]; }
  return t;
}
__device__ __forceinline__ void xform(const CoordDev& d, const Xf& t, float gx, float gy, float& x,
                                      float& y) {
  // coord @ [[c, s], [-s, c]] + dx  (atomai/utils/coords.py:78-83)
  x = gx * t.c - gy * t.s;
  y = gx * t.s + gy * t.c;
  if (d.dx) { x += t.tx; y += t.ty; }
}

// grid: (pixel chunks, B); block 128 threads = hidden lanes (hid <= 1024 handled by a loop)
__global__ void coord_latent_fwd_kernel(const CoordDev d, float* __restrict__ h0, int px_per_cta) {
  extern __shared__ float s_hz[];  // [hid]: bc + Wz z_b
  const int b = blockIdx.y, HW = d.H * d.W;
  for (int h = threadIdx.x; h < d.hid; h += blockDim.x) {
    float acc = d.bc ? d.bc[h] : 0.f;
    for (int k = 0; k < d.zdim; ++k) acc = fmaf(d.wz[h * d.zdim + k], d.z[b * d.zdim + k], acc);
    s_hz[h] = acc;
  }
  __syncthreads();
  const int p0 = blockIdx.x * px_per_cta, p1 = min(HW, p0 + px_per_cta);
  const Xf t = xform_setup(d, b);
  // (the common hid <= blockDim case keeps the thread's two coordinate weights in registers)
  const int h_own = threadIdx.x < d.hid ? threadIdx.x : 0;
  const float w0 = d.wc[h_own * 2], w1 = d.wc[h_own * 2 + 1], hz = s_hz[h_own];
  for (int p = p0; p < p1; ++p) {
    float gx, gy, x, y;
    grid_xy(d, p, gx, gy);
    xform(d, t, gx, gy, x, y);
    float* o = h0 + ((int64_t)b * HW + p) * d.hid;
    if (d.hid <= (int)blockDim.x) {
      if (threadIdx.x < d.hid) {
        const float v = fmaf(w0, x, fmaf(w1, y, hz));
        o[threadIdx.x] = d.tanh_act ? tanhf(v) : v;
      }
    } else {
      for (int h = threadIdx.x; h < d.hid; h += blockDim.x) {
        float v = fmaf(d.wc[h * 2], x, fmaf(d.wc[h * 2 + 1], y, s_hz[h]));
        o[h] = d.tanh_act ? tanhf(v) : v;
      }
    }
  }
}

__global__ void coord_latent_bwd_kernel(const CoordDev d, const float* __restrict__ dpre,
                                        float* dwc, float* dbc, float* sb, float* dphi,
                                        float* ddx, int px_per_cta) {
  extern __shared__ float s_red[];  // [3][blockDim] scratch for (gxsum, gysum, gphi)
  const int b = blockIdx.y, HW = d.H * d.W;
  const int p0 = blockIdx.x * px_per_cta, p1 = min(HW, p0 + px_per_cta);
  float a_dx = 0.f, a_dy = 0.f, a_phi = 0.f;
  // per hidden lane partials (thread h owns lanes h, h+blockDim, ...; hid <= 4*blockDim)
  float s0[4] = {0, 0, 0, 0}, sx[4] = {0, 0, 0, 0}, sy[4] = {0, 0, 0, 0};
  const Xf t = xform_setup(d, b);
  const float c = t.c, s = t.s;
  for (int p = p0; p < p1; ++p) {
    float gx, gy, x, y;
    grid_xy(d, p, gx, gy);
    xform(d, t, gx, gy, x, y);
    const float* g = dpre + ((int64_t)b * HW + p) * d.hid;
    float px = 0.f, py = 0.f;
    int u = 0;
    for (int h = threadIdx.x; h < d.hid; h += blockDim.x, ++u) {
      const float gv = g[h];
      s0[u] += gv;
      sx[u] = fmaf(gv, x, sx[u]);
      sy[u] = fmaf(gv, y, sy[u]);
      px = fmaf(gv, d.wc[h * 2], px);
      py = fmaf(gv, d.wc[h * 2 + 1], py);
    }
    // this thread's share of d(loss)/d(x', y') for pixel p; reduced over threads at the end
    a_dx += px;
    a_dy += py;
    a_phi += px * (-gx * s - gy * c) + py * (gx * c - gy * s);
  }
  int u = 0;
  for (int h = threadIdx.x; h < d.hid; h += blockDim.x, ++u) {
    atomicAdd(dbc + h, s0[u]);
    atomicAdd(dwc + h * 2, sx[u]);
    atomicAdd(dwc + h * 2 + 1, sy[u]);
    atomicAdd(sb + (int64_t)b * d.hid + h, s0[u]);
  }
  s_red[threadIdx.x] = a_dx;
  s_red[blockDim.x + threadIdx.x] = a_dy;
  s_red[2 * blockDim.x + threadIdx.x] = a_phi;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t0 = 0.f, t1 = 0.f, t2 = 0.f;
    for (int i = 0; i < (int)blockDim.x; ++i) {
      t0 += s_red[i];
      t1 += s_red[blockDim.x + i];
      t2 += s_red[2 * blockDim.x + i];
    }
    if (ddx) { atomicAdd(ddx + b * 2, t0); atomicAdd(ddx + b * 2 + 1, t1); }
    if (dphi) atomicAdd(dphi + b, t2);
  }
}

int to_dev(const ab_coordlat_t* d, CoordDev* o) {
  AB_CHECK(d && d->B > 0 && d->H > 0 && d->W > 0 && d->hid > 0 && d->zdim >= 0, "coord_latent: bad dims");
  AB_CHECK(d->hid <= 512, "coord_latent: hid=%d > 512 unsupported", d->hid);
  AB_CHECK(d->wc && (d->zdim == 0 || (d->z && d->wz)), "coord_latent: null weights");
  o->B = d->B; o->H = d->H; o->W = d->W; o->zdim = d->zdim; o->hid = d->hid;
  o->tanh_act = d->tanh_act; o->z = d->z; o->phi = d->phi; o->dx = d->dx; o->wc = d->wc;
  o->bc = d->bc; o->wz = d->wz;
  return 0;
}

}  // namespace

int ab_colsum(const float* dy, int B, int O, float* db, cudaStream_t st);  // db[o] = sum_b dy[b][o]

extern "C" {

int atomai_b200_gemm(const float* A, int64_t a_sm, int64_t a_sk, const float* B, int64_t b_sk,
                     int64_t b_sn, float* C, int64_t c_sm, int M, int N, int K, const float* bias,
                     int act, float slope, int accumulate, int split_k, void* stream) {
  AB_CHECK(C && (K == 0 || (A && B)), "gemm: null pointer");   // K = 0: C (+)= act(bias)
  AB_CHECK(M >= 0 && N >= 0 && K >= 0, "gemm: negative dims");
  if (M == 0 || N == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (split_k < 1) split_k = 1;
  GemmParams p{A, a_sm, a_sk, B, b_sk, b_sn, C, c_sm, M, N, K, bias, act, slope, accumulate,
               split_k, 0};
  int kps = (K + split_k - 1) / split_k;
  kps = (kps + TK - 1) / TK * TK;
  if (kps < TK) kps = TK;
  p.k_per_split = kps;
  p.split_k = (K + kps - 1) / kps;
  if (p.split_k < 1) p.split_k = 1;
  if (p.split_k > 1) {
    AB_CHECK(act == AB_ACT_LRELU && slope == 1.f, "gemm: split-K needs an identity epilogue");
    if (!accumulate) {
      bias_fill_kernel<<<ab_num_sms(), 256, 0, st>>>(C, c_sm, M, N, bias);
      AB_LAUNCH_CHECK();
    }
  }
  dim3 grid((N + TN - 1) / TN, (M + TM - 1) / TM, p.split_k);
  AB_CHECK(grid.y <= 65535 && grid.z <= 65535, "gemm: grid too large");
  gemm_kernel<<<grid, GT, 0, st>>>(p);
  AB_LAUNCH_CHECK();
  return 0;
}

// y[B][O] = x[B][K] W[O][K]^T + b   — nn.Linear forward
int atomai_b200_linear_fwd(const float* x, const float* w, const float* b, float* y, int B, int K,
                           int O, void* stream) {
  if (skinny_ok(x, w, nullptr, B, K, O)) {
    // y = bias, then every k-slice CTA adds its partial sums
    bias_fill_kernel<<<(B * O + 255) / 256, 256, 0, (cudaStream_t)stream>>>(y, O, B, O, b);
    AB_LAUNCH_CHECK();
    const int slices = (K + SK_KS - 1) / SK_KS;
    int rows = (4 * ab_num_sms() + slices - 1) / slices;      // row groups: >= 4 CTAs per SM
    if (rows > B) rows = B;
    if (rows < 1) rows = 1;
    skinny_fwd_kernel<<<dim3(slices, rows), SK_T, 0, (cudaStream_t)stream>>>(x, w, y, B, K, O);
    AB_LAUNCH_CHECK();
    return 0;
  }
  // split K so that roughly 2 waves of CTAs exist even for a 100 x 5 output
  const int tiles = ((B + TM - 1) / TM) * ((O + TN - 1) / TN);
  int split = (2 * ab_num_sms() + tiles - 1) / tiles;
  const int max_split = (K + 4 * TK - 1) / (4 * TK);
  if (split > max_split) split = max_split;
  if (split < 1) split = 1;
  return atomai_b200_gemm(x, K, 1, w, 1, K, y, O, B, O, K, b, AB_ACT_LRELU, 1.f, 0, split, stream);
}

// dx[B][K] = dy[B][O] W[O][K];  dW[O][K] = dy^T x;  db[O] = sum_b dy   (all overwrite)
int atomai_b200_linear_bwd(const float* x, const float* w, const float* dy, float* dx, float* dw,
                           float* db, int B, int K, int O, void* stream) {
  if (skinny_ok(x, w, dx, B, K, O) && ((uintptr_t)dw & 15) == 0 && (size_t)B * O * 4 <= 48 * 1024 &&
      (dx || dw)) {
    const int slices = (K + SK_KSB - 1) / SK_KSB;
    if (O <= 8)
      skinny_bwd_kernel<8><<<slices, SK_TB, (size_t)B * O * 4, (cudaStream_t)stream>>>(x, w, dy, dx, dw,
                                                                                      B, K, O);
    else
      skinny_bwd_kernel<16><<<slices, SK_TB, (size_t)B * O * 4, (cudaStream_t)stream>>>(x, w, dy, dx, dw,
                                                                                       B, K, O);
    AB_LAUNCH_CHECK();
    if (db && ab_colsum(dy, B, O, db, (cudaStream_t)stream)) return 1;
    return 0;
  }
  if (dx) {
    if (atomai_b200_gemm(dy, O, 1, w, K, 1, dx, K, B, K, O, nullptr, AB_ACT_LRELU, 1.f, 0, 1, stream))
      return 1;
  }
  if (dw) {
    if (atomai_b200_gemm(dy, 1, O, x, K, 1, dw, K, O, K, B, nullptr, AB_ACT_LRELU, 1.f, 0, 1, stream))
      return 1;
  }
  if (db) {
    if (ab_colsum(dy, B, O, db, (cudaStream_t)stream)) return 1;
  }
  return 0;
}

int atomai_b200_coord_latent_fwd(const ab_coordlat_t* d, float* h0, void* stream) {
  CoordDev dev;
  if (to_dev(d, &dev)) return 1;
  AB_CHECK(h0, "coord_latent_fwd: null output");
  const int HW = d->H * d->W;
  int chunks = (4 * ab_num_sms() + d->B - 1) / d->B;
  if (chunks > HW) chunks = HW;
  if (chunks < 1) chunks = 1;
  const int ppc = (HW + chunks - 1) / chunks;
  dim3 grid((HW + ppc - 1) / ppc, d->B);
  coord_latent_fwd_kernel<<<grid, 128, d->hid * sizeof(float), (cudaStream_t)stream>>>(dev, h0, ppc);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_coord_latent_bwd(const ab_coordlat_t* d, const float* dpre0, float* dwc, float* dbc,
                                 float* sb, float* dphi, float* ddx, void* stream) {
  CoordDev dev;
  if (to_dev(d, &dev)) return 1;
  AB_CHECK(dpre0 && dwc && dbc && sb, "coord_latent_bwd: null pointer");
  const int HW = d->H * d->W;
  int chunks = (4 * ab_num_sms() + d->B - 1) / d->B;
  if (chunks > HW) chunks = HW;
  if (chunks < 1) chunks = 1;
  const int ppc = (HW + chunks - 1) / chunks;
  dim3 grid((HW + ppc - 1) / ppc, d->B);
  coord_latent_bwd_kernel<<<grid, 128, 3 * 128 * sizeof(float), (cudaStream_t)stream>>>(
      dev, dpre0, dwc, dbc, sb, dphi, ddx, ppc);
  AB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"

namespace {
__global__ void colsum_kernel(const float* __restrict__ dy, int B, int O, float* __restrict__ db) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= O) return;
  float acc = 0.f;
  for (int b = 0; b < B; ++b) acc += dy[(int64_t)b * O + o];
  db[o] = acc;
}
}  // namespace
int ab_colsum(const float* dy, int B, int O, float* db, cudaStream_t st) {
  colsum_kernel<<<(O + 127) / 128, 128, 0, st>>>(dy, B, O, db);
  AB_LAUNCH_CHECK();
  return 0;
}
