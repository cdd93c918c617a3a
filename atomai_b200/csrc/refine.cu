// refine.cu — 2-D Gaussian peak refinement of atom positions (atomai/utils/coords.py:152-231).
// Every atom gets one unconstrained least-squares fit of a rotated Gaussian to the (2d)^2 pixels
// around it, with the iteration scipy.optimize.curve_fit runs: MINPACK's lmdif (forward-difference
// Jacobian, QR with column pivoting, Levenberg-Marquardt parameter, trust-region update, Moré 1978)
// with ftol = xtol = 1.49012e-8, gtol = 0, factor = 100, mode 1 and maxfev = 200 (n + 1).
// Many of these fits are ill-posed (theta is free while sigma_x = sigma_y), and only the same
// iteration lands on the same answer for them, so the routines below follow MINPACK step by step,
// in fp64, and form products without fused multiply-adds where MINPACK's Fortran rounds twice.
//
// Layout: one warp per atom.  The m = (2d)^2 residual rows are spread over the lanes; the m x 7
// Jacobian, the residuals and the trial residuals sit in the warp's slice of shared memory
// (57 KB of Jacobian at d = 16).  Column norms and dot products are warp reductions in a fixed
// order (a butterfly gives every lane the same bits).  The 7 x 7 work of lmpar / qrsolv runs in
// lane 0 on shared memory; every lane then reads the same values, so the control flow stays
// warp-uniform.  No atomics: two launches on the same inputs give identical outputs.
//
// lmdif, fdjac2, qrfac, lmpar and qrsolv are translated from MINPACK-1, which carries this notice:
//
//   Minpack Copyright Notice (1999) University of Chicago.  All rights reserved
//
//   Redistribution and use in source and binary forms, with or without modification, are
//   permitted provided that the following conditions are met:
//   1. Redistributions of source code must retain the above copyright notice, this list of
//      conditions and the following disclaimer.
//   2. Redistributions in binary form must reproduce the above copyright notice, this list of
//      conditions and the following disclaimer in the documentation and/or other materials
//      provided with the distribution.
//   3. The end-user documentation included with the redistribution, if any, must include the
//      following acknowledgment:
//         "This product includes software developed by the University of Chicago, as Operator
//         of Argonne National Laboratory.
//      Alternately, this acknowledgment may appear in the software itself, if and wherever such
//      third-party acknowledgments normally appear.
//   4. WARRANTY DISCLAIMER. THE SOFTWARE IS SUPPLIED "AS IS" WITHOUT WARRANTY OF ANY KIND. THE
//      COPYRIGHT HOLDER, THE UNITED STATES, THE UNITED STATES DEPARTMENT OF ENERGY, AND THEIR
//      EMPLOYEES: (1) DISCLAIM ANY WARRANTIES, EXPRESS OR IMPLIED, INCLUDING BUT NOT LIMITED TO
//      ANY IMPLIED WARRANTIES OF MERCHANTABILITY, FITNESS FOR A PARTICULAR PURPOSE, TITLE OR
//      NON-INFRINGEMENT, (2) DO NOT ASSUME ANY LEGAL LIABILITY OR RESPONSIBILITY FOR THE
//      ACCURACY, COMPLETENESS, OR USEFULNESS OF THE SOFTWARE, (3) DO NOT REPRESENT THAT USE OF
//      THE SOFTWARE WOULD NOT INFRINGE PRIVATELY OWNED RIGHTS, (4) DO NOT WARRANT THAT THE
//      SOFTWARE WILL FUNCTION UNINTERRUPTED, THAT IT IS ERROR-FREE OR THAT ANY ERRORS WILL BE
//      CORRECTED.
//   5. LIMITATION OF LIABILITY. IN NO EVENT WILL THE COPYRIGHT HOLDER, THE UNITED STATES, THE
//      UNITED STATES DEPARTMENT OF ENERGY, OR THEIR EMPLOYEES: BE LIABLE FOR ANY INDIRECT,
//      INCIDENTAL, CONSEQUENTIAL, SPECIAL OR PUNITIVE DAMAGES OF ANY KIND OR NATURE, INCLUDING
//      BUT NOT LIMITED TO LOSS OF PROFITS OR LOSS OF DATA, FOR ANY REASON WHATSOEVER, WHETHER
//      SUCH LIABILITY IS ASSERTED ON THE BASIS OF CONTRACT, TORT (INCLUDING NEGLIGENCE OR STRICT
//      LIABILITY), OR OTHERWISE, EVEN IF ANY OF SAID PARTIES HAS BEEN WARNED OF THE POSSIBILITY
//      OF SUCH LOSS OR DAMAGES.
#include <float.h>

#include "common.cuh"

namespace {

constexpr int kN = 7;            // amp, xo, yo, sigma_x, sigma_y, theta, offset
constexpr int kMaxWarps = 4;     // warps (atoms) per CTA
constexpr int kSmemCap = 227 * 1024;
constexpr double kEpsmch = DBL_EPSILON;
constexpr double kDwarf = DBL_MIN;
constexpr double kSqrtEps = 1.4901161193847656e-08;  // sqrt(max(epsfcn, epsmch)), epsfcn = eps
constexpr double kTol = 1.49012e-8;                   // curve_fit / leastsq ftol = xtol
constexpr double kFactor = 100.0;
constexpr int kMaxfev = 200 * (kN + 1);
constexpr double p1 = 0.1, p5 = 0.5, p25 = 0.25, p75 = 0.75, p05 = 0.05, p001 = 1.0e-3,
                 p0001 = 1.0e-4;

// per-warp small work area (doubles): n-vectors, R (7 x 7, column-major), pivots
enum : int {
  kX = 0, kDiag = 8, kQtf = 16, kWa1 = 24, kWa2 = 32, kWa3 = 40, kRdiag = 48, kAcn = 56, kWq = 64,
  kSdiag = 72, kWb = 80, kWc = 88, kR = 96, kPar = 145, kIpvt = 146, kSmall = 152
};
static_assert(kR + kN * kN <= kPar && kIpvt * 2 + kN <= kSmall * 2, "small area layout");

// a product that is rounded before it is added (nvcc would otherwise fuse it into an FMA)
__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }

__device__ __forceinline__ double norm7(const double* v) {
  double s = 0.0;
#pragma unroll
  for (int j = 0; j < kN; ++j) s += mul(v[j], v[j]);
  return sqrt(s);
}

// sum over rows i >= j0 of a[i] * b[i]
__device__ __forceinline__ double wdot(const double* a, const double* b, int j0, int m, int lane) {
  double s = 0.0;
  for (int i = j0 + lane; i < m; i += 32) s += mul(a[i], b[i]);
  return warp_sum_d(s);
}

struct Window {
  const float* img;  // pixel (0, 0) of the window
  int W;             // row pitch of the frame
  int e;             // side 2d
  int m;             // e * e residual rows
};

// f[i] = model(p; row i) - data[i], or (that - f0[i]) / h when f0 is given (a Jacobian column).
// The Gaussian follows atomai/utils/coords.py:171-176 operation by operation.
__device__ __forceinline__ void residuals(const Window& w, const double* p, double* f,
                                          const double* f0, double h, int lane) {
  const double amp = p[0], xo = p[1], yo = p[2], sx = p[3], sy = p[4], th = p[5], off = p[6];
  const double ct = cos(th), st = sin(th), s2t = sin(2.0 * th);
  const double sx2 = mul(sx, sx), sy2 = mul(sy, sy);
  const double a = mul(ct, ct) / (2.0 * sx2) + mul(st, st) / (2.0 * sy2);
  const double b = (-s2t) / (4.0 * sx2) + s2t / (4.0 * sy2);
  const double c = mul(st, st) / (2.0 * sx2) + mul(ct, ct) / (2.0 * sy2);
  const double b2 = 2.0 * b;
  for (int i = lane; i < w.m; i += 32) {
    const int r = i / w.e, col = i - r * w.e;
    const double dx = (double)r - xo, dy = (double)col - yo;
    const double q = mul(a, mul(dx, dx)) + mul(mul(b2, dx), dy) + mul(c, mul(dy, dy));
    const double g = off + mul(amp, exp(-q));
    const double v = g - (double)__ldg(w.img + (size_t)r * w.W + col);
    f[i] = f0 ? (v - f0[i]) / h : v;
  }
}

// qrfac with column pivoting on the m x 7 matrix held column by column in A: Householder vectors
// below the diagonal, R above it, rdiag = diag(R), acnorm = initial column norms, ipvt = pivots.
// Columns stay where they are; position j of the factorisation is column ipvt[j] of A.
__device__ __forceinline__ void qrfac(double* A, int m, double* s, int lane) {
  double* rdiag = s + kRdiag;
  double* acn = s + kAcn;
  double* wq = s + kWq;
  int* ipvt = reinterpret_cast<int*>(s + kIpvt);
  for (int j = 0; j < kN; ++j) {
    const double nrm = sqrt(wdot(A + j * m, A + j * m, 0, m, lane));
    if (lane == 0) acn[j] = rdiag[j] = wq[j] = nrm, ipvt[j] = j;
  }
  __syncwarp();
  for (int j = 0; j < kN; ++j) {
    if (lane == 0) {
      int kmax = j;
      for (int k = j; k < kN; ++k)
        if (rdiag[k] > rdiag[kmax]) kmax = k;
      if (kmax != j) {
        const int t = ipvt[j];
        ipvt[j] = ipvt[kmax];
        ipvt[kmax] = t;
        rdiag[kmax] = rdiag[j];
        wq[kmax] = wq[j];
      }
    }
    __syncwarp();
    double* aj = A + ipvt[j] * m;
    double ajnorm = sqrt(wdot(aj, aj, j, m, lane));
    if (ajnorm != 0.0) {
      if (aj[j] < 0.0) ajnorm = -ajnorm;
      __syncwarp();
      for (int i = j + lane; i < m; i += 32) aj[i] /= ajnorm;
      if (lane == 0) aj[j] += 1.0;
      __syncwarp();
      const double ajj = aj[j];
      for (int k = j + 1; k < kN; ++k) {
        double* ak = A + ipvt[k] * m;
        const double temp = wdot(aj, ak, j, m, lane) / ajj;
        for (int i = j + lane; i < m; i += 32) ak[i] -= mul(temp, aj[i]);
        __syncwarp();
        double rk = rdiag[k];
        if (rk != 0.0) {
          const double t = ak[j] / rk;
          rk *= sqrt(fmax(0.0, 1.0 - mul(t, t)));
          const double u = rk / wq[k];
          if (mul(p05, mul(u, u)) <= kEpsmch) {  // same values in every lane: a uniform branch
            rk = sqrt(wdot(ak, ak, j + 1, m, lane));
            if (lane == 0) wq[k] = rk;
          }
          if (lane == 0) rdiag[k] = rk;
        }
        __syncwarp();
      }
    }
    if (lane == 0) rdiag[j] = -ajnorm;
    __syncwarp();
  }
}

// qrsolv: least-squares solution of [R; D P^T] x = [Q^T b; 0] given the QR factors of A P.
// r(i, j) = r[i + 7 j]; its strict lower triangle is work space.
__device__ void qrsolv(double* r, const int* ipvt, const double* diag, const double* qtb,
                       double* x, double* sdiag, double* wa) {
  for (int j = 0; j < kN; ++j) {
    for (int i = j; i < kN; ++i) r[i + kN * j] = r[j + kN * i];
    x[j] = r[j + kN * j];
    wa[j] = qtb[j];
  }
  for (int j = 0; j < kN; ++j) {
    const int l = ipvt[j];
    if (diag[l] != 0.0) {
      for (int k = j; k < kN; ++k) sdiag[k] = 0.0;
      sdiag[j] = diag[l];
      double qtbpj = 0.0;
      for (int k = j; k < kN; ++k) {
        if (sdiag[k] == 0.0) continue;
        double sn, cs;
        const double rkk = r[k + kN * k];
        if (fabs(rkk) < fabs(sdiag[k])) {
          const double cotan = rkk / sdiag[k];
          sn = p5 / sqrt(p25 + mul(p25, mul(cotan, cotan)));
          cs = sn * cotan;
        } else {
          const double tn = sdiag[k] / rkk;
          cs = p5 / sqrt(p25 + mul(p25, mul(tn, tn)));
          sn = cs * tn;
        }
        r[k + kN * k] = mul(cs, rkk) + mul(sn, sdiag[k]);
        const double temp = mul(cs, wa[k]) + mul(sn, qtbpj);
        qtbpj = mul(-sn, wa[k]) + mul(cs, qtbpj);
        wa[k] = temp;
        for (int i = k + 1; i < kN; ++i) {
          const double t = mul(cs, r[i + kN * k]) + mul(sn, sdiag[i]);
          sdiag[i] = mul(-sn, r[i + kN * k]) + mul(cs, sdiag[i]);
          r[i + kN * k] = t;
        }
      }
    }
    sdiag[j] = r[j + kN * j];
    r[j + kN * j] = x[j];
  }
  int nsing = kN;
  for (int j = 0; j < kN; ++j) {
    if (sdiag[j] == 0.0 && nsing == kN) nsing = j;
    if (nsing < kN) wa[j] = 0.0;
  }
  for (int j = nsing - 1; j >= 0; --j) {
    double sum = 0.0;
    for (int i = j + 1; i < nsing; ++i) sum += mul(r[i + kN * j], wa[i]);
    wa[j] = (wa[j] - sum) / sdiag[j];
  }
  for (int j = 0; j < kN; ++j) x[ipvt[j]] = wa[j];
}

// lmpar: the Levenberg-Marquardt parameter par for the trust region delta and the step x
// (diag-scaled norm within 10 % of delta, or the Gauss-Newton step if that is inside)
__device__ double lmpar(double* r, const int* ipvt, const double* diag, const double* qtb,
                        double delta, double par, double* x, double* sdiag, double* wa1,
                        double* wa2) {
  int nsing = kN;
  for (int j = 0; j < kN; ++j) {
    wa1[j] = qtb[j];
    if (r[j + kN * j] == 0.0 && nsing == kN) nsing = j;
    if (nsing < kN) wa1[j] = 0.0;
  }
  for (int j = nsing - 1; j >= 0; --j) {
    wa1[j] /= r[j + kN * j];
    const double temp = wa1[j];
    for (int i = 0; i < j; ++i) wa1[i] -= mul(r[i + kN * j], temp);
  }
  for (int j = 0; j < kN; ++j) x[ipvt[j]] = wa1[j];
  int iter = 0;
  for (int j = 0; j < kN; ++j) wa2[j] = diag[j] * x[j];
  double dxnorm = norm7(wa2);
  double fp = dxnorm - delta;
  if (fp <= p1 * delta) return 0.0;
  double parl = 0.0;
  if (nsing >= kN) {
    for (int j = 0; j < kN; ++j) {
      const int l = ipvt[j];
      wa1[j] = diag[l] * (wa2[l] / dxnorm);
    }
    for (int j = 0; j < kN; ++j) {
      double sum = 0.0;
      for (int i = 0; i < j; ++i) sum += mul(r[i + kN * j], wa1[i]);
      wa1[j] = (wa1[j] - sum) / r[j + kN * j];
    }
    const double temp = norm7(wa1);
    parl = ((fp / delta) / temp) / temp;
  }
  for (int j = 0; j < kN; ++j) {
    double sum = 0.0;
    for (int i = 0; i <= j; ++i) sum += mul(r[i + kN * j], qtb[i]);
    wa1[j] = sum / diag[ipvt[j]];
  }
  const double gnorm = norm7(wa1);
  double paru = gnorm / delta;
  if (paru == 0.0) paru = kDwarf / fmin(delta, p1);
  par = fmax(par, parl);
  par = fmin(par, paru);
  if (par == 0.0) par = gnorm / dxnorm;
  for (;;) {
    ++iter;
    if (par == 0.0) par = fmax(kDwarf, p001 * paru);
    const double sp = sqrt(par);
    for (int j = 0; j < kN; ++j) wa1[j] = sp * diag[j];
    qrsolv(r, ipvt, wa1, qtb, x, sdiag, wa2);
    for (int j = 0; j < kN; ++j) wa2[j] = diag[j] * x[j];
    dxnorm = norm7(wa2);
    const double fp_old = fp;
    fp = dxnorm - delta;
    if (fabs(fp) <= p1 * delta || (parl == 0.0 && fp <= fp_old && fp_old < 0.0) || iter == 10)
      break;
    for (int j = 0; j < kN; ++j) {
      const int l = ipvt[j];
      wa1[j] = diag[l] * (wa2[l] / dxnorm);
    }
    for (int j = 0; j < kN; ++j) {
      wa1[j] /= sdiag[j];
      const double temp = wa1[j];
      for (int i = j + 1; i < kN; ++i) wa1[i] -= mul(r[i + kN * j], temp);
    }
    const double temp = norm7(wa1);
    const double parc = ((fp / delta) / temp) / temp;
    if (fp > 0.0) parl = fmax(parl, par);
    if (fp < 0.0) paru = fmin(paru, par);
    par = fmax(parl, par + parc);
  }
  return par;
}

// lmdif on one window; x (in s) holds the start point on entry and the solution on exit.
// Returns MINPACK's info (1..8); *nfev_out = function evaluations, Jacobian columns included.
__device__ __forceinline__ int lmdif(const Window& w, double* A, double* fv, double* wf, double* s,
                                     int lane, int* nfev_out) {
  const int m = w.m;
  double* x = s + kX;
  double* diag = s + kDiag;
  double* qtf = s + kQtf;
  double* wa1 = s + kWa1;
  double* wa2 = s + kWa2;
  double* wa3 = s + kWa3;
  const double* rdiag = s + kRdiag;
  const double* acn = s + kAcn;
  double* R = s + kR;
  const int* ipvt = reinterpret_cast<const int*>(s + kIpvt);

  residuals(w, x, fv, nullptr, 0.0, lane);
  int nfev = 1;
  __syncwarp();
  double fnorm = sqrt(wdot(fv, fv, 0, m, lane));
  double par = 0.0, delta = 0.0, xnorm = 0.0;
  int iter = 1, info = 0;
  for (;;) {
    // forward-difference Jacobian (fdjac2)
    for (int j = 0; j < kN; ++j) {
      const double temp = x[j];
      double h = kSqrtEps * fabs(temp);
      if (h == 0.0) h = kSqrtEps;
      __syncwarp();
      if (lane == 0) x[j] = temp + h;
      __syncwarp();
      residuals(w, x, A + j * m, fv, h, lane);
      __syncwarp();
      if (lane == 0) x[j] = temp;
    }
    nfev += kN;
    __syncwarp();
    qrfac(A, m, s, lane);
    if (iter == 1) {
      if (lane == 0)
        for (int j = 0; j < kN; ++j) diag[j] = acn[j] == 0.0 ? 1.0 : acn[j];
      __syncwarp();
      double t[kN];
#pragma unroll
      for (int j = 0; j < kN; ++j) t[j] = diag[j] * x[j];
      xnorm = norm7(t);
      delta = kFactor * xnorm;
      if (delta == 0.0) delta = kFactor;
    }
    // Q^T fvec -> qtf, R's diagonal back in place
    for (int i = lane; i < m; i += 32) wf[i] = fv[i];
    __syncwarp();
    for (int j = 0; j < kN; ++j) {
      double* aj = A + ipvt[j] * m;
      if (aj[j] != 0.0) {
        const double temp = -wdot(aj, wf, j, m, lane) / aj[j];
        for (int i = j + lane; i < m; i += 32) wf[i] += mul(aj[i], temp);
      }
      __syncwarp();
      if (lane == 0) {
        aj[j] = rdiag[j];
        qtf[j] = wf[j];
      }
      __syncwarp();
    }
    for (int t = lane; t < kN * kN; t += 32) {
      const int i = t % kN, j = t / kN;
      if (i <= j) R[t] = A[ipvt[j] * m + i];
    }
    __syncwarp();
    // norm of the scaled gradient
    double gnorm = 0.0;
    if (fnorm != 0.0) {
      for (int j = 0; j < kN; ++j) {
        const int l = ipvt[j];
        if (acn[l] == 0.0) continue;
        double sum = 0.0;
        for (int i = 0; i <= j; ++i) sum += mul(R[i + kN * j], qtf[i] / fnorm);
        gnorm = fmax(gnorm, fabs(sum / acn[l]));
      }
    }
    if (gnorm <= 0.0) {  // gtol = 0
      info = 4;
      break;
    }
    if (lane == 0)
      for (int j = 0; j < kN; ++j) diag[j] = fmax(diag[j], acn[j]);
    __syncwarp();
    double ratio;
    do {
      if (lane == 0) {
        s[kPar] = lmpar(R, ipvt, diag, qtf, delta, par, wa1, s + kSdiag, s + kWb, s + kWc);
        for (int j = 0; j < kN; ++j) {
          wa1[j] = -wa1[j];
          wa2[j] = x[j] + wa1[j];
          wa3[j] = diag[j] * wa1[j];
        }
      }
      __syncwarp();
      par = s[kPar];
      const double pnorm = norm7(wa3);
      if (iter == 1) delta = fmin(delta, pnorm);
      residuals(w, wa2, wf, nullptr, 0.0, lane);
      ++nfev;
      const double fnorm1 = sqrt(wdot(wf, wf, 0, m, lane));
      double actred = -1.0;
      if (p1 * fnorm1 < fnorm) {
        const double t = fnorm1 / fnorm;
        actred = 1.0 - mul(t, t);
      }
      // predicted reduction: |R P^T p| / fnorm, row by row in MINPACK's order
      double s2 = 0.0;
      for (int i = 0; i < kN; ++i) {
        double acc = 0.0;
        for (int j = i; j < kN; ++j) acc += mul(R[i + kN * j], wa1[ipvt[j]]);
        s2 += mul(acc, acc);
      }
      const double temp1 = sqrt(s2) / fnorm;
      const double temp2 = (sqrt(par) * pnorm) / fnorm;
      const double prered = mul(temp1, temp1) + mul(temp2, temp2) / p5;
      const double dirder = -(mul(temp1, temp1) + mul(temp2, temp2));
      ratio = prered != 0.0 ? actred / prered : 0.0;
      if (ratio <= p25) {
        double temp = p5;
        if (actred < 0.0) temp = p5 * dirder / (dirder + mul(p5, actred));
        if (p1 * fnorm1 >= fnorm || temp < p1) temp = p1;
        delta = temp * fmin(delta, pnorm / p1);
        par = par / temp;
      } else if (par == 0.0 || ratio >= p75) {
        delta = pnorm / p5;
        par = p5 * par;
      }
      if (ratio >= p0001) {  // successful iteration
        __syncwarp();
        if (lane == 0)
          for (int j = 0; j < kN; ++j) x[j] = wa2[j];
        for (int i = lane; i < m; i += 32) fv[i] = wf[i];
        __syncwarp();
        double t[kN];
#pragma unroll
        for (int j = 0; j < kN; ++j) t[j] = diag[j] * x[j];
        xnorm = norm7(t);
        fnorm = fnorm1;
        ++iter;
      }
      if (fabs(actred) <= kTol && prered <= kTol && p5 * ratio <= 1.0) info = 1;
      if (delta <= kTol * xnorm) info = info == 1 ? 3 : 2;
      if (info == 0) {
        if (nfev >= kMaxfev) info = 5;
        if (fabs(actred) <= kEpsmch && prered <= kEpsmch && p5 * ratio <= 1.0) info = 6;
        if (delta <= kEpsmch * xnorm) info = 7;
        if (gnorm <= kEpsmch) info = 8;
      }
      __syncwarp();
    } while (info == 0 && ratio < p0001);
    if (info != 0) break;
  }
  *nfev_out = nfev;
  return info;
}

__global__ void __launch_bounds__(kMaxWarps * 32)
    peak_refine_kernel(const float* __restrict__ img, int n, int H, int W,
                       const int32_t* __restrict__ atoms, int K, int warp_doubles,
                       double* __restrict__ popt, int32_t* __restrict__ info,
                       int32_t* __restrict__ nfev) {
  extern __shared__ double smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int k = blockIdx.x * (blockDim.x >> 5) + warp;
  if (k >= K) return;
  const int f = atoms[4 * k], r0 = atoms[4 * k + 1], c0 = atoms[4 * k + 2], d = atoms[4 * k + 3];
  const int e = 2 * d, m = e * e;
  double* base = smem + (size_t)warp * warp_doubles;
  double* s = base + (size_t)(kN + 2) * m;
  int code = AB_REFINE_SKIPPED, evals = 0;
  if (r0 >= 0) {
    if (f < 0 || f >= n || d < 1 || (kN + 2) * m + kSmall > warp_doubles || c0 < 0 ||
        r0 + e > H || c0 + e > W) {
      code = AB_REFINE_BAD_ATOM;
    } else {
      const Window w{img + ((size_t)f * H + r0) * W + c0, W, e, m};
      bool bad = false;
      for (int i = lane; i < m; i += 32) bad |= !isfinite(__ldg(w.img + (size_t)(i / e) * W + i % e));
      if (__any_sync(0xffffffffu, bad)) {
        code = AB_REFINE_NONFINITE;
      } else {
        if (lane == 0) {
          s[kX + 0] = (double)__ldg(w.img + (size_t)d * W + d);   // p0 = (img[d, d], d, d, 1, 1, 0, 0)
          s[kX + 1] = s[kX + 2] = (double)d;
          s[kX + 3] = s[kX + 4] = 1.0;
          s[kX + 5] = s[kX + 6] = 0.0;
        }
        __syncwarp();
        // MINPACK rejects m < n before evaluating anything (info 0)
        code = m < kN ? 0 : lmdif(w, base, base + kN * m, base + (kN + 1) * m, s, lane, &evals);
      }
    }
  }
  __syncwarp();
  if (lane < kN) popt[(size_t)k * kN + lane] = code >= 0 ? s[kX + lane] : __longlong_as_double(0x7ff8000000000000ll);
  if (lane == 0) {
    info[k] = code;
    if (nfev) nfev[k] = evals;
  }
}

unsigned char g_optin[64];

}  // namespace

extern "C" int atomai_b200_peak_refine(const float* img, int n, int H, int W, const int32_t* atoms,
                                       int K, int dmax, double* popt, int32_t* info, int32_t* nfev,
                                       void* stream) {
  AB_CHECK(img && atoms && popt && info, "peak_refine: null pointer argument");
  AB_CHECK(n > 0 && H > 0 && W > 0 && K >= 0, "peak_refine: bad sizes n=%d H=%d W=%d K=%d", n, H,
           W, K);
  AB_CHECK(dmax >= 1 && dmax <= 16, "peak_refine: d=%d outside the supported range 1..16", dmax);
  if (K == 0) return 0;
  const int warp_doubles = (kN + 2) * 4 * dmax * dmax + kSmall;
  int warps = kSmemCap / (warp_doubles * (int)sizeof(double));
  warps = warps > kMaxWarps ? kMaxWarps : warps;
  const int smem = warps * warp_doubles * (int)sizeof(double);
  if (smem > 48 * 1024 && ab_optin_smem((const void*)peak_refine_kernel, kSmemCap, g_optin)) return 1;
  const int grid = (K + warps - 1) / warps;
  peak_refine_kernel<<<grid, warps * 32, smem, (cudaStream_t)stream>>>(img, n, H, W, atoms, K,
                                                                      warp_doubles, popt, info, nfev);
  AB_LAUNCH_CHECK();
  return 0;
}
