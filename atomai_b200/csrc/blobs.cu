// blobs.cu — blob filtering of utils.filter_cells[_]: threshold every frame of an (n, h, w) stack,
// label the 4-connected components of its foreground, and keep the pixels of the components whose
// size passes the test.  Every pass covers all frames of the stack in one launch.
//
// The labelling is union-find over frame-local linear indices in which a set's root is always its
// smallest index: a root is hooked under a smaller root by a CAS that only succeeds on a root, and
// every other write replaces a parent with one of its ancestors.  So each component ends with its
// smallest index (scipy's raster order of first pixels) as its label, whatever order the atomics
// run in.
//
//   local   one CTA per 32 x 32 tile of a frame, a warp per tile row: threshold, start every pixel
//           in the set of the first pixel of its run in the row (a ballot, no atomics), link the
//           vertical neighbours in shared memory (only where a run of vertical pairs starts), and
//           find each pixel's tile root.  labels = the tile root, counts = the tile component's
//           size at its root and 0 elsewhere.
//   merge   a warp per tile edge: pixels on the top and left edges are linked with their neighbour
//           across the edge in global memory, again only where a run of such pairs starts.
//   roots   every tile root climbs to its final root, stores it as its label and adds its tile
//           size to the final root's count: one atomic per tile component, not per pixel, so a
//           component that spans a 4096^2 frame costs one add per tile.
//   write   every other pixel points at its tile root, whose label is now final: labels = that
//           root, out = 1 on the pixels of kept components.
#include "common.cuh"

namespace {

constexpr int kTile = 32;                 // tile side; one warp covers one tile row
constexpr int kRows = 8;                  // warps per tile CTA, each taking every 8th row
constexpr int kThreads = kTile * kRows;
constexpr int kPer = kTile / kRows;       // tile rows per thread
constexpr int kMergeThreads = 64;         // warp 0: the top edge, warp 1: the left edge

struct Stack {
  int h, w;
  int tx, ty;        // tiles per frame along the columns and the rows
  int64_t tiles;     // n * tx * ty
};

struct Tile {
  int64_t base;      // the frame's first element
  int row0, col0;
};

__device__ __forceinline__ Tile tile_at(const Stack& s, int64_t t) {
  const int64_t per = (int64_t)s.tx * s.ty;
  const int64_t f = t / per;
  const int r = (int)(t - f * per);
  const int ty = r / s.tx;
  return {f * s.h * s.w, ty * kTile, (r - ty * s.tx) * kTile};
}

// foreground: cv2.threshold(THRESH_BINARY)'s x > thresh, float32 pixels against thresh rounded to
// float32; NaN compares false
template <typename T>
__device__ __forceinline__ bool is_fg(T x, double thresh) {
  if constexpr (std::is_same<T, float>::value) return x > __double2float_rn(thresh);
  else return (double)x > thresh;
}

// The root of x.  On the way up every visited node is pointed at its grandparent; only non-roots
// are written, and only with an ancestor, so concurrent finds and hooks stay consistent.
__device__ __forceinline__ int find_root(volatile int* L, int x) {
  int cur = L[x];
  if (cur != x) {
    int prev = x, next;
    while (cur > (next = L[cur])) {
      L[prev] = next;
      prev = cur;
      cur = next;
    }
  }
  return cur;
}

// Joins the sets of a and b: the larger root goes under the smaller one by a CAS that succeeds only
// on a root; when it fails the node has gained a parent, and the walk goes on from there.
__device__ __forceinline__ void unite(volatile int* L, int a, int b) {
  a = find_root(L, a);
  b = find_root(L, b);
  while (a != b) {
    if (a > b) {
      const int t = a;
      a = b;
      b = t;
    }
    const int old = atomicCAS(const_cast<int*>(L + b), b, a);
    if (old == b) return;
    b = old;
  }
}

// lanes where a run of set bits starts
__device__ __forceinline__ unsigned run_starts(unsigned bits) { return bits & ~(bits << 1); }

template <typename T>
__global__ void __launch_bounds__(kThreads) blob_local_kernel(const T* __restrict__ img, Stack s,
                                                              double thresh,
                                                              int32_t* __restrict__ labels,
                                                              int32_t* __restrict__ counts) {
  __shared__ int s_lab[kTile * kTile];
  __shared__ int s_size[kTile * kTile];
  __shared__ unsigned s_bits[kTile];
  const int lane = threadIdx.x, wy = threadIdx.y;
  for (int64_t t = blockIdx.x; t < s.tiles; t += gridDim.x) {
    const Tile tl = tile_at(s, t);
    const int col = tl.col0 + lane;
    for (int k = 0; k < kPer; ++k) {
      const int r = wy + k * kRows, row = tl.row0 + r;
      const bool fg = row < s.h && col < s.w &&
                      is_fg(img[tl.base + (int64_t)row * s.w + col], thresh);
      const unsigned bits = __ballot_sync(~0u, fg);
      const unsigned bg_below = ~bits & ((1u << lane) - 1u);
      s_lab[r * kTile + lane] = fg ? r * kTile + (bg_below ? 32 - __clz(bg_below) : 0) : -1;
      s_size[r * kTile + lane] = 0;
      if (lane == 0) s_bits[r] = bits;
    }
    __syncthreads();
    for (int k = 0; k < kPer; ++k) {
      const int r = wy + k * kRows;
      if (r == 0) continue;
      const unsigned pairs = s_bits[r] & s_bits[r - 1];
      if (run_starts(pairs) >> lane & 1u) unite(s_lab, r * kTile + lane, (r - 1) * kTile + lane);
    }
    __syncthreads();
    int root[kPer];
    for (int k = 0; k < kPer; ++k) {
      const int r = wy + k * kRows;
      const unsigned bits = s_bits[r];
      root[k] = bits >> lane & 1u ? find_root(s_lab, r * kTile + lane) : -1;
      if (run_starts(bits) >> lane & 1u) {
        // the run's length: up to the next background lane
        const unsigned after = ~bits & ~((2u << lane) - 1u);
        const int end = after ? __ffs(after) - 1 : kTile;
        atomicAdd(&s_size[root[k]], end - lane);
      }
    }
    __syncthreads();
    for (int k = 0; k < kPer; ++k) {
      const int r = wy + k * kRows, row = tl.row0 + r;
      if (row < s.h && col < s.w) {
        const int64_t p = tl.base + (int64_t)row * s.w + col;
        const int q = root[k];
        labels[p] = q < 0 ? -1 : (tl.row0 + q / kTile) * s.w + tl.col0 + q % kTile;
        counts[p] = s_size[r * kTile + lane];
      }
    }
    __syncthreads();   // the next tile reuses the shared arrays
  }
}

__global__ void __launch_bounds__(kMergeThreads) blob_merge_kernel(Stack s,
                                                                   int32_t* __restrict__ labels) {
  const int lane = threadIdx.x & 31;
  const bool left_edge = threadIdx.x >= 32;
  for (int64_t t = blockIdx.x; t < s.tiles; t += gridDim.x) {
    const Tile tl = tile_at(s, t);
    volatile int* L = labels + tl.base;
    int a = -1, b = -1;   // an edge pixel and its neighbour across the edge
    if (!left_edge && tl.row0 > 0 && tl.col0 + lane < s.w) {
      a = tl.row0 * s.w + tl.col0 + lane;
      b = a - s.w;
    } else if (left_edge && tl.col0 > 0 && tl.row0 + lane < s.h) {
      a = (tl.row0 + lane) * s.w + tl.col0;
      b = a - 1;
    }
    const bool pair = a >= 0 && L[a] >= 0 && L[b] >= 0;
    // the previous lane's pair is already joined through the tiles on both sides of the edge
    if (run_starts(__ballot_sync(~0u, pair)) >> lane & 1u) unite(L, a, b);
  }
}

__global__ void __launch_bounds__(kThreads) blob_roots_kernel(Stack s,
                                                              int32_t* __restrict__ labels,
                                                              int32_t* __restrict__ counts) {
  const int lane = threadIdx.x, wy = threadIdx.y;
  for (int64_t t = blockIdx.x; t < s.tiles; t += gridDim.x) {
    const Tile tl = tile_at(s, t);
    const int col = tl.col0 + lane;
    if (col >= s.w) continue;
    volatile int* L = labels + tl.base;
    for (int k = 0; k < kPer; ++k) {
      const int row = tl.row0 + wy + k * kRows;
      if (row >= s.h) break;
      const int q = row * s.w + col;
      const int size = counts[tl.base + q];
      if (size == 0) continue;   // not a tile root
      // No writes on the way up: the owner of every tile root stores only its final root, so a
      // label read here is that root or an ancestor of it.
      int r = q;
      for (int nx; (nx = L[r]) != r;) r = nx;
      if (r != q) {
        L[q] = r;
        atomicAdd(counts + tl.base + r, size);
      }
    }
  }
}

template <typename O>
__global__ void __launch_bounds__(kThreads) blob_write_kernel(Stack s, int32_t* __restrict__ labels,
                                                              const int32_t* __restrict__ counts,
                                                              double blob_thresh, int above,
                                                              O* __restrict__ out) {
  const int lane = threadIdx.x, wy = threadIdx.y;
  for (int64_t t = blockIdx.x; t < s.tiles; t += gridDim.x) {
    const Tile tl = tile_at(s, t);
    const int col = tl.col0 + lane;
    if (col >= s.w) continue;
    int32_t* L = labels + tl.base;
    for (int k = 0; k < kPer; ++k) {
      const int row = tl.row0 + wy + k * kRows;
      if (row >= s.h) break;
      const int q = row * s.w + col;
      const int tr = L[q];
      bool keep = false;
      if (tr >= 0) {
        // tr is a tile root, final since the roots pass; only pixels that are not tile roots
        // change here, and no pixel's label points at those
        const int r = L[tr];
        if (r != tr) L[q] = r;
        const double c = (double)counts[tl.base + r];
        keep = !(above ? c > blob_thresh : c < blob_thresh);
      }
      out[tl.base + q] = keep ? (O)1 : (O)0;
    }
  }
}

template <typename T>
void launch_local(const void* img, const Stack& s, double thresh, int32_t* labels, int32_t* counts,
                  cudaStream_t st) {
  blob_local_kernel<T><<<ab_grid(s.tiles, 1, 8), dim3(kTile, kRows), 0, st>>>(
      (const T*)img, s, thresh, labels, counts);
}

template <typename O>
void launch_write(const Stack& s, int32_t* labels, const int32_t* counts, double blob_thresh,
                  int above, void* out, cudaStream_t st) {
  blob_write_kernel<O><<<ab_grid(s.tiles, 1, 8), dim3(kTile, kRows), 0, st>>>(
      s, labels, counts, blob_thresh, above, (O*)out);
}

}  // namespace

extern "C" {

int atomai_b200_blob_filter(const void* img, int dtype, int64_t n, int h, int w, double im_thresh,
                            double blob_thresh, int above, int32_t* labels, int32_t* counts,
                            void* out, int out_dtype, void* stream) {
  AB_CHECK(n >= 0 && h >= 0 && w >= 0 && (int64_t)h * w < ((int64_t)1 << 31),
           "blob_filter: bad shape (n=%lld, h=%d, w=%d)", (long long)n, h, w);
  AB_CHECK(dtype >= AB_BLOB_U8 && dtype <= AB_BLOB_F64, "blob_filter: input dtype code %d", dtype);
  AB_CHECK(out_dtype >= AB_BLOB_U8 && out_dtype <= AB_BLOB_I32,
           "blob_filter: output dtype code %d", out_dtype);
  if (n == 0 || h == 0 || w == 0) return 0;
  AB_CHECK(img && labels && counts && out, "blob_filter: null pointer");
  Stack s{h, w, (w + kTile - 1) / kTile, (h + kTile - 1) / kTile, 0};
  s.tiles = n * s.tx * s.ty;
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case AB_BLOB_U8: launch_local<uint8_t>(img, s, im_thresh, labels, counts, st); break;
    case AB_BLOB_I16: launch_local<int16_t>(img, s, im_thresh, labels, counts, st); break;
    case AB_BLOB_U16: launch_local<uint16_t>(img, s, im_thresh, labels, counts, st); break;
    case AB_BLOB_F32: launch_local<float>(img, s, im_thresh, labels, counts, st); break;
    default: launch_local<double>(img, s, im_thresh, labels, counts, st); break;
  }
  blob_merge_kernel<<<ab_grid(s.tiles, 1, 32), kMergeThreads, 0, st>>>(s, labels);
  blob_roots_kernel<<<ab_grid(s.tiles, 1, 8), dim3(kTile, kRows), 0, st>>>(s, labels, counts);
  // 1 has the same bits in int16 and uint16
  switch (out_dtype) {
    case AB_BLOB_U8: launch_write<uint8_t>(s, labels, counts, blob_thresh, above, out, st); break;
    case AB_BLOB_I16:
    case AB_BLOB_U16: launch_write<uint16_t>(s, labels, counts, blob_thresh, above, out, st); break;
    case AB_BLOB_F32: launch_write<float>(s, labels, counts, blob_thresh, above, out, st); break;
    case AB_BLOB_F64: launch_write<double>(s, labels, counts, blob_thresh, above, out, st); break;
    default: launch_write<int32_t>(s, labels, counts, blob_thresh, above, out, st); break;
  }
  AB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
