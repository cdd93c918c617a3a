// cellgrid.cuh — the cell list shared by the neighbour searches of graph.cu and coords.cu.
//
// Atoms are binned into cubic cells of side `side` from the origin lo; the int64 key of a cell is
// ((frame * nz + cz) * ny + cy) * nx + cx, so the frames of one batch never share a cell and the
// cells x0 ... x1 of one row are contiguous in key order.  graph_cell_keys_kernel (graph.cu) writes
// the keys; the caller sorts them stably, and a search finds a row of cells by binary search in
// the sorted keys, so the grid is never materialised.
#pragma once
#include <math.h>
#include <stdint.h>

struct Grid {
  double lo[3];
  double side;
  int64_t n[3];
};

__device__ __forceinline__ int64_t cell_of(double p, double lo, double side, int64_t n) {
  int64_t c = (int64_t)floor((p - lo) / side);
  return c < 0 ? 0 : (c >= n ? n - 1 : c);
}

// first index t of the sorted keys with keys[t] >= k
__device__ __forceinline__ int lower_key(const int64_t* __restrict__ keys, int N, int64_t k) {
  int a = 0, b = N;
  while (a < b) {
    const int m = (a + b) >> 1;
    if (keys[m] < k) a = m + 1;
    else b = m;
  }
  return a;
}

// Correctly rounded square root of a finite s >= 0, equal to sqrt(s), inline: the library's sqrt
// branches to an out-of-line slow path, and that call makes a kernel that keeps state in registers
// save them to a stack frame.  The operand is scaled by an even power of two into the range where
// the reciprocal-square-root estimate and two Newton steps are accurate, and the final step rounds
// through the exact residual s - g * g.
__device__ __forceinline__ double sqrt_rn(double s) {
  if (s == 0.0) return s;
  double scale = 1.0;
  if (s < 0x1p-900) {
    s *= 0x1p+1000;
    scale = 0x1p-500;
  } else if (s > 0x1p+900) {
    s *= 0x1p-1000;
    scale = 0x1p+500;
  }
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(s));
  double g = __dmul_rn(s, y), h = __dmul_rn(0.5, y);
  for (int it = 0; it < 2; ++it) {
    const double r = __fma_rn(-g, h, 0.5);
    g = __fma_rn(g, r, g);
    h = __fma_rn(h, r, h);
  }
  return __dmul_rn(__fma_rn(__fma_rn(-g, g, s), h, g), scale);
}

__device__ __forceinline__ double sq_dist3(const double* a, const double* b) {
  const double dx = __dsub_rn(a[0], b[0]), dy = __dsub_rn(a[1], b[1]), dz = __dsub_rn(a[2], b[2]);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// |a - b| in float64 with every operation rounded on its own (no FMA), in column order: the value
// scipy's k-d tree and a numpy expression give.  dist3_inline is the same value through sqrt_rn,
// for the searches that keep a top-k list in registers (coords.cu); the bond search of graph.cu
// keeps the library's sqrt, with which ptxas allocates it fewer spill slots.
__device__ __forceinline__ double dist3(const double* a, const double* b) {
  return sqrt(sq_dist3(a, b));
}
__device__ __forceinline__ double dist3_inline(const double* a, const double* b) {
  return sqrt_rn(sq_dist3(a, b));
}

// host: a Grid from host arrays of the origin and the cell counts
inline Grid make_grid(const double* lo_host, double side, const int64_t* dims_host) {
  Grid g;
  for (int a = 0; a < 3; ++a) {
    g.lo[a] = lo_host[a];
    g.n[a] = dims_host[a];
  }
  g.side = side;
  return g;
}
