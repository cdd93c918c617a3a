// graph.cu — bond graphs, shortest-path rings and hop tables of atomic lattices (utils.graphx).
//
//   cell_keys   int64 key of each atom's cell (side >= the largest bond cutoff), frame-major, so the
//               frames of one batch never share a cell.  The caller sorts the keys (stably).
//   bonds       count pass: degree of every atom; fill pass: its CSR row, sorted ascending.  Atoms
//               i != j bond when |p_i - p_j| (float64, unfused) <= cut[c_i][c_j]; the candidates
//               come from the 3 x 3 (x 3) cells around the atom, found by binary search in the
//               sorted keys, so the grid is never materialised (cellgrid.cuh).
//   hops        one level of the bounded hop table: ball_k(u) = ball_{k-1}(u) U ball_{k-1}(w) + 1
//               over the bonded w, as sorted rows of packed (id << 5 | hops) words.  Count pass and
//               fill pass, like bonds.
//   rings       one thread per root: an explicit depth-first search over atoms > root, which emits
//               every simple cycle of 3 ... max_depth atoms whose lowest atom is the root, once, in
//               the order of a recursive search over ascending neighbour lists (the ring is emitted
//               when its last atom is pushed, and only when that atom is above the root's first
//               step).  A step to n is taken only when hops(root, n) <= max_depth - depth: every
//               atom of a closing ring meets that bound, so the pruning does not change the set.
//   ring_filter one thread per ring: the ring is dropped when two of its atoms j < k are joined in
//               the bond graph by fewer hops than min(k - j, l - k + j).
//
// Determinism: every output position comes from a count pass and a prefix sum of the caller; no
// atomics decide any order, and a repeated call gives identical results.
#include <math.h>
#include "cellgrid.cuh"
#include "common.cuh"

namespace {

constexpr int kThreads = 128;
constexpr int kHopBits = 5;  // hops <= 16 in the low bits of a packed hop-table word
constexpr uint32_t kHopMask = (1u << kHopBits) - 1;

__global__ void __launch_bounds__(kThreads)
    graph_cell_keys_kernel(const double* __restrict__ pos, const int* __restrict__ frame, int N,
                           Grid g, int64_t* __restrict__ keys) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= N) return;
  const int64_t f = frame ? frame[i] : 0;
  const int64_t cx = cell_of(pos[3 * i], g.lo[0], g.side, g.n[0]);
  const int64_t cy = cell_of(pos[3 * i + 1], g.lo[1], g.side, g.n[1]);
  const int64_t cz = cell_of(pos[3 * i + 2], g.lo[2], g.side, g.n[2]);
  keys[i] = ((f * g.n[2] + cz) * g.n[1] + cy) * g.n[0] + cx;
}

// rowptr == nullptr: deg[i] = number of bonds of i; else cols[rowptr[i] ...] = the bonded atoms,
// ascending
__global__ void __launch_bounds__(kThreads)
    graph_bonds_kernel(const double* __restrict__ pos, const int* __restrict__ cls,
                       const int* __restrict__ frame, int N, const int64_t* __restrict__ keys,
                       const int64_t* __restrict__ perm, const double* __restrict__ cut, int C,
                       Grid g, const int64_t* __restrict__ rowptr, int* __restrict__ out) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= N) return;
  const double* pi = pos + 3 * i;
  const double* ci = cut + (int64_t)(cls ? cls[i] : 0) * C;
  const int64_t f = frame ? frame[i] : 0;
  const int64_t cx = cell_of(pi[0], g.lo[0], g.side, g.n[0]);
  const int64_t cy = cell_of(pi[1], g.lo[1], g.side, g.n[1]);
  const int64_t cz = cell_of(pi[2], g.lo[2], g.side, g.n[2]);
  int* row = rowptr ? out + rowptr[i] : nullptr;
  int cnt = 0;
  for (int64_t z = cz - 1; z <= cz + 1; ++z) {
    if (z < 0 || z >= g.n[2]) continue;
    for (int64_t y = cy - 1; y <= cy + 1; ++y) {
      if (y < 0 || y >= g.n[1]) continue;
      const int64_t base = ((f * g.n[2] + z) * g.n[1] + y) * g.n[0];
      const int64_t x0 = cx > 0 ? cx - 1 : 0, x1 = cx + 1 < g.n[0] ? cx + 1 : g.n[0] - 1;
      // cells x0 ... x1 of one row are contiguous in key order
      const int t1 = lower_key(keys, N, base + x1 + 1);
      for (int t = lower_key(keys, N, base + x0); t < t1; ++t) {
        const int j = (int)perm[t];
        if (j == i) continue;
        if (dist3(pi, pos + 3 * j) <= ci[cls ? cls[j] : 0]) {
          if (row) row[cnt] = j;
          ++cnt;
        }
      }
    }
  }
  if (!row) {
    out[i] = cnt;
    return;
  }
  for (int a = 1; a < cnt; ++a) {  // insertion sort: the rows are short and any length is allowed
    const int v = row[a];
    int b = a - 1;
    while (b >= 0 && row[b] > v) {
      row[b + 1] = row[b];
      --b;
    }
    row[b + 1] = v;
  }
}

// next packed word of `row` (length n) with id > c, or UINT32_MAX
__device__ __forceinline__ uint32_t next_after(const uint32_t* __restrict__ row, int64_t n,
                                               uint32_t key) {
  int64_t a = 0, b = n;
  while (a < b) {
    const int64_t m = (a + b) >> 1;
    if (row[m] < key) a = m + 1;
    else b = m;
  }
  return a < n ? row[a] : 0xffffffffu;
}

// ball_k(u) from ball_{k-1}: a merge of the sorted rows of u and of its bonded atoms (+1 hop),
// keeping the least hop count of each id.  optr == nullptr: cnt[u] = its length.
__global__ void __launch_bounds__(kThreads)
    graph_hops_kernel(const int64_t* __restrict__ rowptr, const int* __restrict__ cols, int N,
                      const int64_t* __restrict__ bptr, const uint32_t* __restrict__ ball,
                      const int64_t* __restrict__ optr, uint32_t* __restrict__ out,
                      int64_t* __restrict__ cnt) {
  const int u = blockIdx.x * kThreads + threadIdx.x;
  if (u >= N) return;
  const int64_t r0 = rowptr[u], r1 = rowptr[u + 1];
  uint32_t* dst = optr ? out + optr[u] : nullptr;
  int64_t n = 0;
  uint32_t key = 0;  // search for ids >= key >> kHopBits
  for (;;) {
    uint32_t best = 0xffffffffu;
    for (int64_t e = r0 - 1; e < r1; ++e) {
      const int w = e < r0 ? u : cols[e];
      uint32_t x = next_after(ball + bptr[w], bptr[w + 1] - bptr[w], key);
      if (x == 0xffffffffu) continue;
      if (e >= r0) ++x;
      if (x < best) best = x;  // least id, then least hops
    }
    if (best == 0xffffffffu) break;
    if (dst) dst[n] = best;
    ++n;
    key = ((best >> kHopBits) + 1) << kHopBits;
    if (key == 0) break;
  }
  if (!dst) cnt[u] = n;
}

// hops from the row's owner to v, or -1 when v is not within the table's radius
__device__ __forceinline__ int hops_to(const uint32_t* __restrict__ row, int64_t n, int v) {
  const uint32_t x = next_after(row, n, (uint32_t)v << kHopBits);
  return (x != 0xffffffffu && (int)(x >> kHopBits) == v) ? (int)(x & kHopMask) : -1;
}

// ring_base == nullptr: cnt[3 r] = rings of root r, cnt[3 r + 1] = their atoms, cnt[3 r + 2] = DFS
// paths (steps taken); else the rings of root r go to lens[ring_base[r] ...] and
// atoms[atom_base[r] ...], in discovery order.
__global__ void __launch_bounds__(kThreads)
    graph_rings_kernel(const int64_t* __restrict__ rowptr, const int* __restrict__ cols, int N,
                       const int64_t* __restrict__ bptr, const uint32_t* __restrict__ ball,
                       int max_depth, const int64_t* __restrict__ ring_base,
                       const int64_t* __restrict__ atom_base, int* __restrict__ lens,
                       int* __restrict__ atoms, int64_t* __restrict__ cnt) {
  const int root = blockIdx.x * kThreads + threadIdx.x;
  if (root >= N) return;
  int path[AB_GRAPH_MAX_RING];
  int64_t cur[AB_GRAPH_MAX_RING];
  const uint32_t* B = ball + bptr[root];
  const int64_t nb = bptr[root + 1] - bptr[root];
  int64_t nr = 0, na = 0, np = 0;
  int64_t rb = ring_base ? ring_base[root] : 0, ab = ring_base ? atom_base[root] : 0;
  path[0] = root;
  cur[0] = rowptr[root];
  int d = 0;
  while (d >= 0) {
    const int64_t end = d + 1 < max_depth ? rowptr[path[d] + 1] : cur[d];
    if (cur[d] >= end) {
      --d;
      continue;
    }
    const int n = cols[cur[d]++];
    if (n <= root) continue;
    bool on = false;
    for (int a = 1; a <= d; ++a) on |= path[a] == n;
    if (on) continue;
    const int h = hops_to(B, nb, n);
    if (h < 0 || h > max_depth - (d + 1)) continue;
    ++d;
    path[d] = n;
    cur[d] = rowptr[n];
    ++np;
    if (d >= 2 && h == 1 && n > path[1]) {
      if (ring_base) {
        lens[rb++] = d + 1;
        for (int a = 0; a <= d; ++a) atoms[ab++] = path[a];
      }
      ++nr;
      na += d + 1;
    }
  }
  if (!ring_base) {
    cnt[3 * root] = nr;
    cnt[3 * root + 1] = na;
    cnt[3 * root + 2] = np;
  }
}

__global__ void __launch_bounds__(kThreads)
    graph_ring_filter_kernel(const int64_t* __restrict__ off, const int* __restrict__ lens,
                             const int* __restrict__ atoms, int64_t R,
                             const int64_t* __restrict__ bptr, const uint32_t* __restrict__ ball,
                             unsigned char* __restrict__ keep) {
  const int64_t r = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (r >= R) return;
  const int* a = atoms + off[r];
  const int l = lens[r];
  bool k_ = true;
  for (int j = 0; j < l && k_; ++j) {
    const uint32_t* B = ball + bptr[a[j]];
    const int64_t nb = bptr[a[j] + 1] - bptr[a[j]];
    for (int k = j + 2; k < l && k_; ++k) {
      const int h = hops_to(B, nb, a[k]);
      if (h >= 0 && h < min(k - j, l - k + j)) k_ = false;
    }
  }
  keep[r] = k_;
}

unsigned blocks(int64_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }

}  // namespace

extern "C" int atomai_b200_graph_cell_keys(const double* pos, const int* frame, int N,
                                           const double* lo_host, double side,
                                           const int64_t* dims_host, int64_t* keys, void* stream) {
  AB_CHECK(N >= 1 && side > 0 && lo_host && dims_host, "graph_cell_keys: N=%d side=%g", N, side);
  AB_CHECK(pos && keys, "graph_cell_keys: null pointer");
  Grid g;
  for (int a = 0; a < 3; ++a) {
    g.lo[a] = lo_host[a];
    g.n[a] = dims_host[a];
    AB_CHECK(g.n[a] >= 1, "graph_cell_keys: dims[%d]=%lld", a, (long long)g.n[a]);
  }
  g.side = side;
  graph_cell_keys_kernel<<<blocks(N), kThreads, 0, (cudaStream_t)stream>>>(pos, frame, N, g, keys);
  AB_LAUNCH_CHECK();
  return 0;
}

extern "C" int atomai_b200_graph_bonds(const double* pos, const int* cls, const int* frame, int N,
                                       const int64_t* keys, const int64_t* perm, const double* cut,
                                       int C, const double* lo_host, double side,
                                       const int64_t* dims_host, const int64_t* rowptr, int* out,
                                       void* stream) {
  AB_CHECK(N >= 1 && C >= 1 && side > 0 && lo_host && dims_host, "graph_bonds: N=%d C=%d side=%g",
           N, C, side);
  AB_CHECK(pos && keys && perm && cut && out, "graph_bonds: null pointer");
  Grid g;
  for (int a = 0; a < 3; ++a) {
    g.lo[a] = lo_host[a];
    g.n[a] = dims_host[a];
    AB_CHECK(g.n[a] >= 1, "graph_bonds: dims[%d]=%lld", a, (long long)g.n[a]);
  }
  g.side = side;
  graph_bonds_kernel<<<blocks(N), kThreads, 0, (cudaStream_t)stream>>>(
      pos, cls, frame, N, keys, perm, cut, C, g, rowptr, out);
  AB_LAUNCH_CHECK();
  return 0;
}

extern "C" int atomai_b200_graph_hops(const int64_t* rowptr, const int* cols, int N,
                                      const int64_t* bptr, const uint32_t* ball,
                                      const int64_t* optr, uint32_t* out, int64_t* cnt,
                                      void* stream) {
  AB_CHECK(N >= 1 && N < (1 << (31 - kHopBits)), "graph_hops: N=%d (< %d)", N,
           1 << (31 - kHopBits));
  AB_CHECK(rowptr && bptr && ball && (optr ? out != nullptr : cnt != nullptr),
           "graph_hops: null pointer");
  graph_hops_kernel<<<blocks(N), kThreads, 0, (cudaStream_t)stream>>>(rowptr, cols, N, bptr, ball,
                                                                      optr, out, cnt);
  AB_LAUNCH_CHECK();
  return 0;
}

extern "C" int atomai_b200_graph_rings(const int64_t* rowptr, const int* cols, int N,
                                       const int64_t* bptr, const uint32_t* ball, int max_depth,
                                       const int64_t* ring_base, const int64_t* atom_base,
                                       int* lens, int* atoms, int64_t* cnt, void* stream) {
  AB_CHECK(N >= 1 && max_depth >= 3 && max_depth <= AB_GRAPH_MAX_RING,
           "graph_rings: N=%d max_depth=%d (3 ... %d)", N, max_depth, AB_GRAPH_MAX_RING);
  AB_CHECK(rowptr && bptr && ball &&
               (ring_base ? (atom_base && lens && atoms) != 0 : cnt != nullptr),
           "graph_rings: null pointer");
  graph_rings_kernel<<<blocks(N), kThreads, 0, (cudaStream_t)stream>>>(
      rowptr, cols, N, bptr, ball, max_depth, ring_base, atom_base, lens, atoms, cnt);
  AB_LAUNCH_CHECK();
  return 0;
}

extern "C" int atomai_b200_graph_ring_filter(const int64_t* off, const int* lens, const int* atoms,
                                             int64_t R, const int64_t* bptr, const uint32_t* ball,
                                             unsigned char* keep, void* stream) {
  AB_CHECK(R >= 1, "graph_ring_filter: R=%lld", (long long)R);
  AB_CHECK(off && lens && atoms && bptr && ball && keep, "graph_ring_filter: null pointer");
  graph_ring_filter_kernel<<<blocks(R), kThreads, 0, (cudaStream_t)stream>>>(off, lens, atoms, R,
                                                                              bptr, ball, keep);
  AB_LAUNCH_CHECK();
  return 0;
}
