// jlatent.cu — the joint (continuous + Gumbel-softmax) latent block of jVAE / jrVAE between the
// encoder heads and the decoder (atomai/models/dgm/jvae.py:103-131, jrvae.py:117-151,
// trainers/vitrainer.py:223-248, losses_metrics/vi_losses.py:40-84,140-221): head softmax,
// reparameterisation, Gumbel-softmax sample, decoder input and the KL batch means in one forward
// launch, every gradient in one backward launch.  The tensors are (B, <= 64): these kernels replace
// a few dozen tiny torch launches per step, not a bandwidth problem.
//
// Layout: one warp per row.  A lane owns continuous column `lane` and discrete columns lane and
// lane + 32; a row's values sit in shared memory so that each lane reduces over its own head
// (max, sum) in column order — every lane of a head gets bit-identical head sums.
#include <math.h>
#include "common.cuh"

namespace {

constexpr int JT = 1024;          // threads per CTA
constexpr int JW = JT / 32;       // rows in flight per CTA
constexpr float kEps = 1e-12f;    // the reference's guard in log(alpha + eps) and the Gumbel noise

struct JDev {
  int B, Dc, coord, D, Dz;        // Dz = Dc - coord + D: width of the decoder input
  float tau, phi_prior, dx_prior;
  double log_phi_prior;
  double h2[AB_JLAT_MAX_DISC];                           // log(1/D_h + 1e-12) of column j's head
  uint8_t hb[AB_JLAT_MAX_DISC], he[AB_JLAT_MAX_DISC];   // [begin, end) of column j's head
};

__device__ __forceinline__ float head_max(const float* s, int b0, int b1) {
  float m = s[b0];
  for (int k = b0 + 1; k < b1; ++k) m = fmaxf(m, s[k]);
  return m;
}
__device__ __forceinline__ float head_expsum(const float* s, int b0, int b1, float m) {
  float t = 0.f;
  for (int k = b0; k < b1; ++k) t += expf(s[k] - m);
  return t;
}
__device__ __forceinline__ float head_sum(const float* s, int b0, int b1) {
  float t = 0.f;
  for (int k = b0; k < b1; ++k) t += s[k];
  return t;
}
// Gumbel noise of column j of row b (vitrainer.py:242-244)
__device__ __forceinline__ float gumbel(const JDev& p, const float* u, uint64_t seed, int b, int j) {
  const int64_t idx = (int64_t)b * p.D + j;
  const float uu = u ? __ldg(u + idx) : hash_uniform((uint64_t)idx, seed);
  return -logf(-logf(uu + kEps) + kEps);
}

// s_l (this warp's row of logits) -> the two alphas of this lane (columns lane, lane + 32)
__device__ __forceinline__ void row_alpha(const JDev& p, const float* __restrict__ logits, int b,
                                          float* s_l, int lane, float a[2]) {
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int j = lane + 32 * r;
    if (j < p.D) s_l[j] = __ldg(logits + (int64_t)b * p.D + j);
  }
  __syncwarp();
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int j = lane + 32 * r;
    a[r] = 0.f;
    if (j < p.D) {
      const int b0 = p.hb[j], b1 = p.he[j];
      const float m = head_max(s_l, b0, b1);
      a[r] = expf(s_l[j] - m) / head_expsum(s_l, b0, b1, m);
    }
  }
  __syncwarp();
}

__global__ void __launch_bounds__(JT) jlatent_fwd_kernel(
    const JDev p, int mode, const float* __restrict__ mu, const float* __restrict__ logsd,
    const float* __restrict__ logits, const float* __restrict__ eps, const float* __restrict__ u,
    uint64_t seed, float* __restrict__ alpha, float* __restrict__ zdec, float* __restrict__ phi,
    float* __restrict__ dx, float* __restrict__ kl) {
  __shared__ float s_l[JW][AB_JLAT_MAX_DISC];
  __shared__ float s_y[JW][AB_JLAT_MAX_DISC];
  __shared__ double s_kl[JW][2];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int Dcc = p.Dc - p.coord;
  double kc = 0.0, kd = 0.0;      // this lane's KL partials over its rows (fixed order)
  for (int b = blockIdx.x * JW + warp; b < p.B; b += gridDim.x * JW) {
    float a[2];
    row_alpha(p, logits, b, s_l[warp], lane, a);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int j = lane + 32 * r;
      if (j < p.D) alpha[(int64_t)b * p.D + j] = a[r];
    }
    if (mode == AB_JLAT_ALPHAS) continue;
    float y[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int j = lane + 32 * r;
      if (j < p.D) {
        const float la = logf(a[r] + kEps);
        y[r] = (la + gumbel(p, u, seed, b, j)) / p.tau;
        s_y[warp][j] = y[r];
        kd += (double)a[r] * ((double)la - p.h2[j]);
      }
    }
    __syncwarp();
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int j = lane + 32 * r;
      if (j < p.D) {
        const int b0 = p.hb[j], b1 = p.he[j];
        const float m = head_max(s_y[warp], b0, b1);
        zdec[(int64_t)b * p.Dz + Dcc + j] = expf(y[r] - m) / head_expsum(s_y[warp], b0, b1, m);
      }
    }
    __syncwarp();
    if (lane < p.Dc) {
      const int64_t i = (int64_t)b * p.Dc + lane;
      const float m = __ldg(mu + i), ls = __ldg(logsd + i);
      const float sd = expf(ls);
      const float z = m + sd * __ldg(eps + i);
      if (lane >= p.coord) zdec[(int64_t)b * p.Dz + lane - p.coord] = z;
      else if (lane == 0) phi[b] = z;
      else dx[b * 2 + lane - 1] = z * p.dx_prior;
      const double dls = ls, dsd = sd;
      if (p.coord && lane == 0)   // kld_rot (vi_losses.py:77-84)
        kc += -dls + p.log_phi_prior + dsd * dsd / (2.0 * (double)p.phi_prior * p.phi_prior) - 0.5;
      else                        // kld_normal (vi_losses.py:40-57)
        kc += -dls + 0.5 * dsd * dsd + 0.5 * (double)m * m - 0.5;
    }
  }
  if (kl == nullptr) return;      // (launched as a single CTA whenever kl is requested)
  kc = warp_sum_d(kc);
  kd = warp_sum_d(kd);
  if (lane == 0) { s_kl[warp][0] = kc; s_kl[warp][1] = kd; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double tc = 0.0, td = 0.0;
    for (int w = 0; w < JW; ++w) { tc += s_kl[w][0]; td += s_kl[w][1]; }
    kl[0] = (float)(tc / p.B);
    kl[1] = (float)(td / p.B);
  }
}

__global__ void __launch_bounds__(JT) jlatent_bwd_kernel(
    const JDev p, int mode, const float* __restrict__ mu, const float* __restrict__ logsd,
    const float* __restrict__ logits, const float* __restrict__ eps, const float* __restrict__ u,
    uint64_t seed, const float* __restrict__ dzdec, const float* __restrict__ dphi,
    const float* __restrict__ ddx, const float* __restrict__ dalpha, const float* __restrict__ gkl,
    float* __restrict__ dmu, float* __restrict__ dlogsd, float* __restrict__ dlogits) {
  __shared__ float s_l[JW][AB_JLAT_MAX_DISC];
  __shared__ float s_t[JW][AB_JLAT_MAX_DISC];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int Dcc = p.Dc - p.coord;
  const float gc = gkl ? __ldg(gkl) / p.B : 0.f;       // d loss / d (per-row KL terms)
  const float gd = gkl ? __ldg(gkl + 1) / p.B : 0.f;
  for (int b = blockIdx.x * JW + warp; b < p.B; b += gridDim.x * JW) {
    float a[2], da[2] = {0.f, 0.f};
    row_alpha(p, logits, b, s_l[warp], lane, a);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int j = lane + 32 * r;
      if (j < p.D && dalpha) da[r] = __ldg(dalpha + (int64_t)b * p.D + j);
    }
    if (mode == AB_JLAT_SAMPLE) {
      // tau-softmax: recompute y (into s_l, free again) and the sample zd
      float la[2], y[2], zd[2], gz[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int j = lane + 32 * r;
        la[r] = y[r] = 0.f;
        if (j < p.D) {
          la[r] = logf(a[r] + kEps);
          y[r] = (la[r] + gumbel(p, u, seed, b, j)) / p.tau;
          s_l[warp][j] = y[r];
        }
      }
      __syncwarp();
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int j = lane + 32 * r;
        zd[r] = gz[r] = 0.f;
        if (j < p.D) {
          const int b0 = p.hb[j], b1 = p.he[j];
          const float m = head_max(s_l[warp], b0, b1);
          zd[r] = expf(y[r] - m) / head_expsum(s_l[warp], b0, b1, m);
          gz[r] = dzdec ? __ldg(dzdec + (int64_t)b * p.Dz + Dcc + j) : 0.f;
          s_t[warp][j] = zd[r] * gz[r];
        }
      }
      __syncwarp();
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int j = lane + 32 * r;
        if (j < p.D) {
          const float sdz = head_sum(s_t[warp], p.hb[j], p.he[j]);
          const float dla = (zd[r] * gz[r] - zd[r] * sdz) / p.tau;       // through softmax(y)
          const float h2 = (float)p.h2[j];
          da[r] += dla / (a[r] + kEps)                                     // through log(alpha+eps)
                   + gd * ((la[r] - h2) + a[r] / (a[r] + kEps));           // kld_discrete
        }
      }
      __syncwarp();
    }
    // head softmax: dl = alpha (da - sum_head alpha da)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int j = lane + 32 * r;
      if (j < p.D) s_t[warp][j] = a[r] * da[r];
    }
    __syncwarp();
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int j = lane + 32 * r;
      if (j < p.D)
        dlogits[(int64_t)b * p.D + j] = a[r] * da[r] - a[r] * head_sum(s_t[warp], p.hb[j], p.he[j]);
    }
    __syncwarp();
    if (mode == AB_JLAT_SAMPLE && lane < p.Dc) {
      const int64_t i = (int64_t)b * p.Dc + lane;
      const float m = __ldg(mu + i), ls = __ldg(logsd + i);
      const float sd = expf(ls);
      float gzc;
      if (lane >= p.coord) gzc = dzdec ? __ldg(dzdec + (int64_t)b * p.Dz + lane - p.coord) : 0.f;
      else if (lane == 0) gzc = dphi ? __ldg(dphi + b) : 0.f;
      else gzc = ddx ? __ldg(ddx + b * 2 + lane - 1) * p.dx_prior : 0.f;
      float gm = gzc, gl = gzc * sd * __ldg(eps + i);
      if (p.coord && lane == 0) {
        gl += gc * (sd * sd / (p.phi_prior * p.phi_prior) - 1.f);
      } else {
        gm += gc * m;
        gl += gc * (sd * sd - 1.f);
      }
      dmu[i] = gm;
      dlogsd[i] = gl;
    }
  }
}

int to_dev(const ab_jlat_t* d, int mode, JDev* o) {
  AB_CHECK(d, "jlatent: null descriptor");
  AB_CHECK(mode == AB_JLAT_ALPHAS || mode == AB_JLAT_SAMPLE, "jlatent: mode=%d", mode);
  AB_CHECK(d->B >= 0, "jlatent: B=%d", d->B);
  AB_CHECK(d->nheads >= 1 && d->nheads <= AB_JLAT_MAX_DISC, "jlatent: %d discrete heads (1..%d)",
           d->nheads, AB_JLAT_MAX_DISC);
  int D = 0;
  for (int h = 0; h < d->nheads; ++h) {
    AB_CHECK(d->heads[h] >= 1, "jlatent: head %d has size %d", h, d->heads[h]);
    AB_CHECK(D + d->heads[h] <= AB_JLAT_MAX_DISC, "jlatent: sum of discrete dims > %d",
             AB_JLAT_MAX_DISC);
    for (int k = 0; k < d->heads[h]; ++k) {
      o->h2[D + k] = log(1.0 / d->heads[h] + 1e-12);     // np.log(1. / cat_dim + eps)
      o->hb[D + k] = (uint8_t)D;
      o->he[D + k] = (uint8_t)(D + d->heads[h]);
    }
    D += d->heads[h];
  }
  o->B = d->B; o->D = D; o->Dc = d->Dc; o->coord = d->coord;
  o->tau = d->tau; o->phi_prior = d->phi_prior; o->dx_prior = d->dx_prior;
  o->log_phi_prior = d->phi_prior > 0.f ? log((double)d->phi_prior) : 0.0;
  if (mode == AB_JLAT_SAMPLE) {
    AB_CHECK(d->Dc >= 1 && d->Dc <= AB_JLAT_MAX_CONT, "jlatent: %d continuous dims (1..%d)", d->Dc,
             AB_JLAT_MAX_CONT);
    AB_CHECK((d->coord == 0 || d->coord == 1 || d->coord == 3) && d->coord < d->Dc,
             "jlatent: coord=%d with %d continuous dims", d->coord, d->Dc);
    AB_CHECK(d->tau > 0.f && d->tau < 3.0e38f, "jlatent: temperature %f", d->tau);
    AB_CHECK(d->coord == 0 || d->phi_prior > 0.f, "jlatent: rotation prior %f", d->phi_prior);
  }
  o->Dz = d->Dc - d->coord + D;
  return 0;
}

int grid_rows(int B, bool single) {
  if (single) return 1;
  int g = (B + JW - 1) / JW;
  const int cap = 2 * ab_num_sms();
  return g < 1 ? 1 : (g > cap ? cap : g);
}

}  // namespace

extern "C" {

int atomai_b200_jlatent_fwd(const ab_jlat_t* d, int mode, const float* mu, const float* logsd,
                            const float* logits, const float* eps, const float* u, uint64_t seed,
                            float* alpha, float* zdec, float* phi, float* dx, float* kl,
                            void* stream) {
  JDev p;
  if (to_dev(d, mode, &p)) return 1;
  AB_CHECK(logits && alpha, "jlatent_fwd: null logits / alpha");
  if (mode == AB_JLAT_SAMPLE) {
    AB_CHECK(mu && logsd && eps && zdec, "jlatent_fwd: null mu / logsd / eps / zdec");
    AB_CHECK(p.coord == 0 || (phi && (p.coord == 1 || dx)), "jlatent_fwd: null phi / dx");
  } else {
    kl = nullptr;
  }
  if (p.B == 0) return 0;
  jlatent_fwd_kernel<<<grid_rows(p.B, kl != nullptr), JT, 0, (cudaStream_t)stream>>>(
      p, mode, mu, logsd, logits, eps, u, seed, alpha, zdec, phi, dx, kl);
  AB_LAUNCH_CHECK();
  return 0;
}

int atomai_b200_jlatent_bwd(const ab_jlat_t* d, int mode, const float* mu, const float* logsd,
                            const float* logits, const float* eps, const float* u, uint64_t seed,
                            const float* dzdec, const float* dphi, const float* ddx,
                            const float* dalpha, const float* gkl, float* dmu, float* dlogsd,
                            float* dlogits, void* stream) {
  JDev p;
  if (to_dev(d, mode, &p)) return 1;
  AB_CHECK(logits && dlogits, "jlatent_bwd: null logits / dlogits");
  if (mode == AB_JLAT_SAMPLE)
    AB_CHECK(mu && logsd && eps && dmu && dlogsd, "jlatent_bwd: null mu / logsd / eps / dmu / dlogsd");
  if (p.B == 0) return 0;
  jlatent_bwd_kernel<<<grid_rows(p.B, false), JT, 0, (cudaStream_t)stream>>>(
      p, mode, mu, logsd, logits, eps, u, seed, dzdec, dphi, ddx, dalpha, gkl, dmu, dlogsd, dlogits);
  AB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
