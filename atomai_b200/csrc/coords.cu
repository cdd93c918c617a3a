// coords.cu — neighbour searches of utils.coords: k nearest atoms, balls, trajectories through a
// movie and DBSCAN labels.  The atoms live in the cell list of cellgrid.cuh (keys written by
// graph_cell_keys, sorted stably by the caller); `foff` holds the first sorted key of every frame,
// which is the frame's first atom because the keys are frame-major and the atoms frame-ordered.
//
//   knn      one thread per query: the K least (distance, index) pairs of its frame in registers
//            (K a compile-time bucket, so the list is never spilled).  Rings of cells are visited
//            outward from the query's cell; the search stops once no atom outside the rings seen
//            can come closer than the k-th pair, when no atom can be within the upper bound, or
//            when every atom of the frame or every cell of its grid has been visited.
//   ball     count pass: atoms with d < rmax of every query; fill pass: their indices and
//            distances in scan order (the caller orders each row by distance, then index).
//   walk     one thread per start position: in every frame, the nearest atom with d < rmax; when
//            numpy's slice of the r x r window around its rounded centre is r x r, the step is
//            recorded and the walk moves to that atom, else the frame is skipped.
//   dbscan   core points (neighbours + 1 >= min_samples) are joined by atomicMin hooking of roots
//            and pointer jumping until every component points to its lowest core index; the final
//            roots do not depend on the order of the atomics.  A border point takes the lowest
//            root among its core neighbours; the caller's rank of the roots renumbers them.
//
// Distances are float64 and unfused (dist3_inline); a tie in distance goes to the lower index.  Output
// positions come from counts, never from atomics, and a repeated call gives identical results.
#include <math.h>
#include "cellgrid.cuh"
#include "common.cuh"

namespace {

constexpr int kThreads = 128;
constexpr int kNone = 0x7fffffff;

__device__ __forceinline__ bool before(double d, int j, double e, int k) {
  return d < e || (d == e && j < k);
}

// The k least (distance, index) pairs seen, ascending, in the last k of K slots; the first K - k
// slots hold (-inf, -1), which no pair displaces.  Every slot index is a constant after
// unrolling, so the list stays in registers.
template <int K>
struct TopK {
  double d[K];
  int j[K];

  __device__ __forceinline__ void init(int k) {
#pragma unroll
    for (int a = 0; a < K; ++a) {
      d[a] = a < K - k ? -INFINITY : INFINITY;
      j[a] = a < K - k ? -1 : kNone;
    }
  }
  __device__ __forceinline__ double kth() const { return d[K - 1]; }
  __device__ __forceinline__ void push(double dd, int jj) {
    if (!before(dd, jj, d[K - 1], j[K - 1])) return;
#pragma unroll
    for (int a = K - 1; a > 0; --a) {
      if (before(dd, jj, d[a - 1], j[a - 1])) {
        d[a] = d[a - 1];
        j[a] = j[a - 1];
      } else if (before(dd, jj, d[a], j[a])) {
        d[a] = dd;
        j[a] = jj;
      }
    }
    if (before(dd, jj, d[0], j[0])) {
      d[0] = dd;
      j[0] = jj;
    }
  }
};

// The k nearest atoms of frame f (sorted keys [t0, t1)) to q, in cell c, with d < ub, into top.
//
// An atom binned c cells from the query's cell along an axis is at least (c - 1) * side away,
// and rounding of a cell index moves an atom or the query by at most one cell near a cell face, so
// an atom outside the rings 0 ... r - 1 is at least (r - 2) * side away.  A query outside the grid
// is clamped to an edge cell, which only makes the bound more conservative.
template <int K>
__device__ __forceinline__ void knn_search(const double* q, const int64_t* c, int64_t f,
                                           const double* __restrict__ pos,
                                           const int64_t* __restrict__ keys,
                                           const int64_t* __restrict__ perm, int t0, int t1,
                                           const Grid& g, double ub, TopK<K>& top) {
  const int64_t cx = c[0], cy = c[1], cz = c[2];
  const int64_t last = max(max(max(cx, g.n[0] - 1 - cx), max(cy, g.n[1] - 1 - cy)),
                           max(cz, g.n[2] - 1 - cz));
  const int64_t* fk = keys + t0;
  const int nf = t1 - t0;
  int seen = 0;  // atoms of the frame visited so far
  for (int64_t r = 0; r <= last && seen < nf; ++r) {
    if (r >= 2) {
      const double lb = (double)(r - 2) * g.side;
      if (lb >= ub || top.kth() < lb) break;
    }
    for (int64_t z = max(cz - r, (int64_t)0); z <= min(cz + r, g.n[2] - 1); ++z) {
      for (int64_t y = max(cy - r, (int64_t)0); y <= min(cy + r, g.n[1] - 1); ++y) {
        const int64_t base = ((f * g.n[2] + z) * g.n[1] + y) * g.n[0];
        const bool face = z == cz - r || z == cz + r || y == cy - r || y == cy + r;
        // a face row of the ring is a run of cells; any other row holds its two end cells
        for (int end = 0; end < (face ? 1 : 2); ++end) {
          int64_t x0, x1;
          if (face) {
            x0 = max(cx - r, (int64_t)0);
            x1 = min(cx + r, g.n[0] - 1);
          } else {
            x0 = x1 = end ? cx + r : cx - r;
            if (x0 < 0 || x0 >= g.n[0]) continue;
          }
          const int e = lower_key(fk, nf, base + x1 + 1);
          const int b = lower_key(fk, nf, base + x0);
          seen += e - b;
          for (int t = b; t < e; ++t) {
            const int j = (int)perm[t0 + t];
            const double d = dist3_inline(q, pos + 3 * (int64_t)j);
            if (d < ub) top.push(d, j);
          }
        }
      }
    }
  }
}

template <int K>
__global__ void __launch_bounds__(kThreads)
    coords_knn_kernel(const double* __restrict__ qpos, const int64_t* __restrict__ qcell,
                      const int* __restrict__ qframe, int Q,
                      const double* __restrict__ pos, const int64_t* __restrict__ keys,
                      const int64_t* __restrict__ perm, const int64_t* __restrict__ foff, int N,
                      Grid g, int k, double ub, int* __restrict__ oidx,
                      double* __restrict__ odist) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= Q) return;
  const int f = qframe ? qframe[i] : 0;
  const int t0 = foff ? (int)foff[f] : 0, t1 = foff ? (int)foff[f + 1] : N;
  const double q[3] = {qpos[3 * (int64_t)i], qpos[3 * (int64_t)i + 1], qpos[3 * (int64_t)i + 2]};
  TopK<K> top;
  top.init(k);
  knn_search<K>(q, qcell + 3 * (int64_t)i, f, pos, keys, perm, t0, t1, g, ub, top);
  int* oi = oidx + (int64_t)i * k - (K - k);
  double* od = odist + (int64_t)i * k - (K - k);
#pragma unroll
  for (int a = 0; a < K; ++a) {
    if (a >= K - k) {
      oi[a] = top.j[a] == kNone ? -1 : top.j[a];
      od[a] = top.d[a];
    }
  }
}

// the cell of every point, as graph_cell_keys bins it.  The searches read cells from here: the
// division of cell_of has an out-of-line slow path, which in a search would cost a stack frame.
__global__ void __launch_bounds__(kThreads)
    coords_cells_kernel(const double* __restrict__ pos, int N, Grid g,
                        int64_t* __restrict__ cell) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= N) return;
  for (int a = 0; a < 3; ++a) cell[3 * (int64_t)i + a] = cell_of(pos[3 * (int64_t)i + a], g.lo[a], g.side, g.n[a]);
}

// kFill false: cnt[i] = atoms with d < rmax of query i; true: oidx / odist[rowptr[i] ...] = those
// atoms and distances, in scan order.  The cell side is >= rmax.  (Without the occupancy hint of the
// launch bounds, ptxas parks one value of the count instance in a stack slot over the loops.)
template <bool kFill>
__global__ void __launch_bounds__(kThreads, 4)
    coords_ball_kernel(const double* __restrict__ qpos, const int64_t* __restrict__ qcell, int Q,
                       const double* __restrict__ pos, const int64_t* __restrict__ keys,
                       const int64_t* __restrict__ perm, int N, Grid g, double rmax,
                       const int64_t* __restrict__ rowptr, int* __restrict__ oidx,
                       double* __restrict__ odist, int64_t* __restrict__ cnt) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= Q) return;
  const double q[3] = {qpos[3 * (int64_t)i], qpos[3 * (int64_t)i + 1], qpos[3 * (int64_t)i + 2]};
  const int64_t* c = qcell + 3 * (int64_t)i;
  const int64_t cx = c[0], cy = c[1], cz = c[2];
  const int64_t x0 = max(cx - 1, (int64_t)0), x1 = min(cx + 1, g.n[0] - 1);
  const int64_t y0 = max(cy - 1, (int64_t)0), y1 = min(cy + 1, g.n[1] - 1);
  const int64_t z0 = max(cz - 1, (int64_t)0), z1 = min(cz + 1, g.n[2] - 1);
  int64_t o = kFill ? rowptr[i] : 0;
  for (int64_t z = z0; z <= z1; ++z) {
    for (int64_t y = y0; y <= y1; ++y) {
      const int64_t base = (z * g.n[1] + y) * g.n[0];
      const int e = lower_key(keys, N, base + x1 + 1);
      for (int t = lower_key(keys, N, base + x0); t < e; ++t) {
        const int j = (int)perm[t];
        const double d = dist3_inline(q, pos + 3 * (int64_t)j);
        if (d < rmax) {
          if (kFill) {
            oidx[o] = j;
            odist[o] = d;
          }
          ++o;
        }
      }
    }
  }
  if (!kFill) cnt[i] = o;
}

// numpy's bound of a slice start or stop i on an axis of `len` (positive step)
__device__ __forceinline__ int64_t slice_bound(int64_t i, int64_t len) {
  if (i < 0) i += len;
  return i < 0 ? 0 : (i > len ? len : i);
}

// out[(s * F + f) * 4 ...] = (f, atom, row0, col0) of walk s in frame f, or (f, -1, -1, -1)
__global__ void __launch_bounds__(kThreads)
    coords_walk_kernel(const double* __restrict__ start, const int64_t* __restrict__ scell, int S,
                       const double* __restrict__ pos, const int64_t* __restrict__ pcell,
                       const int64_t* __restrict__ keys, const int64_t* __restrict__ perm,
                       const int64_t* __restrict__ foff, int F, Grid g, double rmax, int64_t H,
                       int64_t W, int64_t half, int64_t r, int* __restrict__ out) {
  const int s = blockIdx.x * kThreads + threadIdx.x;
  if (s >= S) return;
  double q[3] = {start[3 * (int64_t)s], start[3 * (int64_t)s + 1], 0.0};
  const int64_t* c = scell + 3 * (int64_t)s;
  for (int f = 0; f < F; ++f) {
    TopK<1> top;
    top.init(1);
    knn_search<1>(q, c, f, pos, keys, perm, (int)foff[f], (int)foff[f + 1], g, rmax, top);
    int* o = out + ((int64_t)s * F + f) * 4;
    o[0] = f;
    o[1] = o[2] = o[3] = -1;
    if (top.j[0] == kNone) continue;
    const double* p = pos + 3 * (int64_t)top.j[0];
    const int64_t cx = (int64_t)rint(p[0]), cy = (int64_t)rint(p[1]);  // np.around: half to even
    const int64_t x0 = slice_bound(cx - half, H), x1 = slice_bound(cx + half, H);
    const int64_t y0 = slice_bound(cy - half, W), y1 = slice_bound(cy + half, W);
    if (max(x1 - x0, (int64_t)0) != r || max(y1 - y0, (int64_t)0) != r) continue;
    o[1] = top.j[0];
    o[2] = (int)x0;
    o[3] = (int)y0;
    q[0] = p[0];
    q[1] = p[1];
    c = pcell + 3 * (int64_t)top.j[0];
  }
}

// parent[i] = i for a core point, -1 for the others
__global__ void __launch_bounds__(kThreads)
    dbscan_init_kernel(const int64_t* __restrict__ rowptr, int N, int min_samples,
                       int* __restrict__ parent) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= N) return;
  parent[i] = rowptr[i + 1] - rowptr[i] + 1 >= min_samples ? i : -1;
}

// the root of core point i; parents only decrease and stay inside i's component, so a stale read
// still names an atom of it
__device__ __forceinline__ int find_root(const int* parent, int i) {
  int p = __ldcg(parent + i);
  while (p != i) {
    i = p;
    p = __ldcg(parent + i);
  }
  return i;
}

__global__ void __launch_bounds__(kThreads)
    dbscan_hook_kernel(const int64_t* __restrict__ rowptr, const int* __restrict__ cols, int N,
                       int* parent, int* __restrict__ changed) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= N || __ldcg(parent + i) < 0) return;
  for (int64_t e = rowptr[i]; e < rowptr[i + 1]; ++e) {
    const int j = cols[e];
    if (j <= i || __ldcg(parent + j) < 0) continue;
    const int ri = find_root(parent, i), rj = find_root(parent, j);
    if (ri != rj) {
      atomicMin(parent + max(ri, rj), min(ri, rj));
      *changed = 1;
    }
  }
}

__global__ void __launch_bounds__(kThreads) dbscan_compress_kernel(int N, int* parent) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= N || parent[i] < 0) return;
  parent[i] = find_root(parent, i);
}

// labels[i] = rank of i's root (core) or of the lowest root among its core neighbours (border),
// else -1
__global__ void __launch_bounds__(kThreads)
    dbscan_label_kernel(const int64_t* __restrict__ rowptr, const int* __restrict__ cols, int N,
                        const int* __restrict__ parent, const int64_t* __restrict__ rank,
                        int64_t* __restrict__ labels) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= N) return;
  int root = parent[i];
  if (root < 0) {
    root = kNone;
    for (int64_t e = rowptr[i]; e < rowptr[i + 1]; ++e) {
      const int p = parent[cols[e]];
      if (p >= 0 && p < root) root = p;
    }
  }
  labels[i] = root == kNone ? -1 : rank[root];
}

unsigned blocks(int64_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }

template <int K>
void launch_knn(const double* qpos, const int64_t* qcell, const int* qframe, int Q, const double* pos,
                const int64_t* keys, const int64_t* perm, const int64_t* foff, int N, Grid g,
                int k, double ub, int* oidx, double* odist, cudaStream_t st) {
  coords_knn_kernel<K><<<blocks(Q), kThreads, 0, st>>>(qpos, qcell, qframe, Q, pos, keys, perm, foff, N,
                                                       g, k, ub, oidx, odist);
}

int check_grid(const char* what, const double* lo_host, double side, const int64_t* dims_host) {
  AB_CHECK(lo_host && dims_host && side > 0, "%s: side=%g", what, side);
  for (int a = 0; a < 3; ++a)
    AB_CHECK(dims_host[a] >= 1, "%s: dims[%d]=%lld", what, a, (long long)dims_host[a]);
  return 0;
}

}  // namespace

extern "C" int atomai_b200_coords_cells(const double* pos, int N, const double* lo_host,
                                        double side, const int64_t* dims_host, int64_t* cells,
                                        void* stream) {
  AB_CHECK(N >= 1 && pos && cells, "coords_cells: N=%d or null pointer", N);
  if (check_grid("coords_cells", lo_host, side, dims_host)) return 1;
  coords_cells_kernel<<<blocks(N), kThreads, 0, (cudaStream_t)stream>>>(
      pos, N, make_grid(lo_host, side, dims_host), cells);
  AB_LAUNCH_CHECK();
  return 0;
}

extern "C" int atomai_b200_coords_knn(const double* qpos, const int64_t* qcell, const int* qframe,
                                      int Q,
                                      const double* pos, int N, const int64_t* keys,
                                      const int64_t* perm, const int64_t* foff,
                                      const double* lo_host, double side,
                                      const int64_t* dims_host, int k, double ub, int* oidx,
                                      double* odist, void* stream) {
  AB_CHECK(Q >= 1 && N >= 1, "coords_knn: Q=%d N=%d", Q, N);
  AB_CHECK(k >= 1 && k <= AB_COORDS_MAX_K, "coords_knn: k=%d (1 ... %d)", k, AB_COORDS_MAX_K);
  AB_CHECK(qpos && qcell && pos && keys && perm && oidx && odist &&
               (qframe == nullptr || foff != nullptr),
           "coords_knn: null pointer");
  if (check_grid("coords_knn", lo_host, side, dims_host)) return 1;
  const Grid g = make_grid(lo_host, side, dims_host);
  cudaStream_t st = (cudaStream_t)stream;
  if (k <= 1) launch_knn<1>(qpos, qcell, qframe, Q, pos, keys, perm, foff, N, g, k, ub, oidx, odist, st);
  else if (k <= 4) launch_knn<4>(qpos, qcell, qframe, Q, pos, keys, perm, foff, N, g, k, ub, oidx, odist, st);
  else if (k <= 8) launch_knn<8>(qpos, qcell, qframe, Q, pos, keys, perm, foff, N, g, k, ub, oidx, odist, st);
  else if (k <= 16) launch_knn<16>(qpos, qcell, qframe, Q, pos, keys, perm, foff, N, g, k, ub, oidx, odist, st);
  else launch_knn<32>(qpos, qcell, qframe, Q, pos, keys, perm, foff, N, g, k, ub, oidx, odist, st);
  AB_LAUNCH_CHECK();
  return 0;
}

extern "C" int atomai_b200_coords_ball(const double* qpos, const int64_t* qcell, int Q, const double* pos, int N,
                                       const int64_t* keys, const int64_t* perm,
                                       const double* lo_host, double side,
                                       const int64_t* dims_host, double rmax,
                                       const int64_t* rowptr, int* oidx, double* odist,
                                       int64_t* cnt, void* stream) {
  AB_CHECK(Q >= 1 && N >= 1 && rmax <= side, "coords_ball: Q=%d N=%d rmax=%g side=%g", Q, N, rmax,
           side);
  AB_CHECK(qpos && qcell && pos && keys && perm && (rowptr ? (oidx && odist) != 0 : cnt != nullptr),
           "coords_ball: null pointer");
  if (check_grid("coords_ball", lo_host, side, dims_host)) return 1;
  const Grid g = make_grid(lo_host, side, dims_host);
  if (rowptr)
    coords_ball_kernel<true><<<blocks(Q), kThreads, 0, (cudaStream_t)stream>>>(
        qpos, qcell, Q, pos, keys, perm, N, g, rmax, rowptr, oidx, odist, cnt);
  else
    coords_ball_kernel<false><<<blocks(Q), kThreads, 0, (cudaStream_t)stream>>>(
        qpos, qcell, Q, pos, keys, perm, N, g, rmax, rowptr, oidx, odist, cnt);
  AB_LAUNCH_CHECK();
  return 0;
}

extern "C" int atomai_b200_coords_walk(const double* start, const int64_t* scell, int S,
                                       const double* pos, const int64_t* pcell,
                                       const int64_t* keys, const int64_t* perm,
                                       const int64_t* foff, int F, const double* lo_host,
                                       double side, const int64_t* dims_host, double rmax,
                                       int64_t H, int64_t W, int64_t half, int64_t r, int* out,
                                       void* stream) {
  AB_CHECK(S >= 1 && F >= 1 && H >= 0 && W >= 0 && H < (1ll << 31) && W < (1ll << 31),
           "coords_walk: S=%d F=%d H=%lld W=%lld", S, F, (long long)H, (long long)W);
  AB_CHECK(start && scell && pos && pcell && keys && perm && foff && out,
           "coords_walk: null pointer");
  if (check_grid("coords_walk", lo_host, side, dims_host)) return 1;
  coords_walk_kernel<<<blocks(S), kThreads, 0, (cudaStream_t)stream>>>(
      start, scell, S, pos, pcell, keys, perm, foff, F, make_grid(lo_host, side, dims_host), rmax, H, W, half, r,
      out);
  AB_LAUNCH_CHECK();
  return 0;
}

extern "C" int atomai_b200_coords_dbscan_roots(const int64_t* rowptr, const int* cols, int N,
                                               int min_samples, int* parent, int* flag,
                                               void* stream) {
  AB_CHECK(N >= 1, "coords_dbscan_roots: N=%d", N);
  AB_CHECK(rowptr && parent && flag, "coords_dbscan_roots: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  dbscan_init_kernel<<<blocks(N), kThreads, 0, st>>>(rowptr, N, min_samples, parent);
  AB_LAUNCH_CHECK();
  // every round with a change lowers some parent, so the loop ends; in practice after a few rounds
  for (int64_t round = 0;; ++round) {
    AB_CHECK(round <= (int64_t)N, "coords_dbscan_roots: no convergence after %lld rounds",
             (long long)round);
    AB_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), st));
    dbscan_hook_kernel<<<blocks(N), kThreads, 0, st>>>(rowptr, cols, N, parent, flag);
    AB_LAUNCH_CHECK();
    dbscan_compress_kernel<<<blocks(N), kThreads, 0, st>>>(N, parent);
    AB_LAUNCH_CHECK();
    int h = 0;
    AB_CUDA(cudaMemcpyAsync(&h, flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    AB_CUDA(cudaStreamSynchronize(st));
    if (!h) break;
  }
  return 0;
}

extern "C" int atomai_b200_coords_dbscan_labels(const int64_t* rowptr, const int* cols, int N,
                                                const int* parent, const int64_t* rank,
                                                int64_t* labels, void* stream) {
  AB_CHECK(N >= 1, "coords_dbscan_labels: N=%d", N);
  AB_CHECK(rowptr && parent && rank && labels, "coords_dbscan_labels: null pointer");
  dbscan_label_kernel<<<blocks(N), kThreads, 0, (cudaStream_t)stream>>>(rowptr, cols, N, parent,
                                                                        rank, labels);
  AB_LAUNCH_CHECK();
  return 0;
}
