// knn_tree.cuh -- the Morton-ordered 32-ary box tree of DESIGN section 4.5, generic over the coordinate type.  knn.cu builds it
// over float points (simple_knn's distCUDA2), dtu_eval.cu over double points (the DTU evaluation's radius and 1-NN searches).
//
//   bbox     order-free min / max of the finite points (ordered-integer atomics) into scratch
//   keys     96-bit Morton code of each point over that box (32 bits per axis, quantised in double; positions outside the box
//            clamp to its faces, so query points of another set can be keyed against a tree's box); non-finite points get the
//            all-ones key, which no finite point can have, so they sort last
//   sort     the library's multi-word sort, the key as three u32 words
//   gather   sorted coordinates into three planes, padded with NaN to whole leaves of 32
//   boxes    one AABB per leaf of 32 consecutive points (finite points only), then an implicit 32-ary tree of unions
//
// Every step is a comparison, a min / max or an exact copy, except the key quantisation, which only decides the order.  The
// box of a node therefore holds the exact coordinates of its points, and a bound computed from it with rounded operations
// that are monotone in each gap never exceeds the same formula for a point inside.
#pragma once
#include <math.h>

#include "gof_common.cuh"

namespace gof_tree {

constexpr int THREADS = 256;
constexpr int LEAF = 32;
constexpr int MAX_LEVELS = 8;                // 2^31 points: 2^26 leaves, 32-ary -> 7 levels
constexpr int LEVEL_SHIFT = 26;              // stack entry of a walk: level << 26 | node (node < 2^26)

template <class T> struct Coord;
template <> struct Coord<float> {
  using U = uint32_t;                        // ordered-integer image of a value
  using V4 = float4;                         // box corner
  static constexpr U SIGN = 0x80000000u;
  __device__ static U bits(float f) { return __float_as_uint(f); }
  __device__ static float value(U u) { return __uint_as_float(u); }
  __device__ static float nan() { return __int_as_float(0x7fc00000); }
  __device__ static float vmin(float a, float b) { return fminf(a, b); }
  __device__ static float vmax(float a, float b) { return fmaxf(a, b); }
  __device__ static V4 corner(float x, float y, float z) { return make_float4(x, y, z, 0.f); }
};
template <> struct Coord<double> {
  using U = unsigned long long;
  using V4 = double4;
  static constexpr U SIGN = 0x8000000000000000ull;
  __device__ static U bits(double f) { return (U)__double_as_longlong(f); }
  __device__ static double value(U u) { return __longlong_as_double((long long)u); }
  __device__ static double nan() { return __longlong_as_double(0x7ff8000000000000ll); }
  __device__ static double vmin(double a, double b) { return fmin(a, b); }
  __device__ static double vmax(double a, double b) { return fmax(a, b); }
  __device__ static V4 corner(double x, double y, double z) { return make_double4(x, y, z, 0.0); }
};

struct Tree {
  int levels;                                // level 0 = leaves, levels-1 = the root (one node)
  int count[MAX_LEVELS];                     // nodes per level
  long long offset[MAX_LEVELS];              // first box of each level in the box array
  long long nodes;                           // boxes in all levels
};

static inline Tree make_tree(int P) {
  Tree t{};
  int n = (P + LEAF - 1) / LEAF;
  long long off = 0;
  t.levels = 0;
  while (true) {
    t.count[t.levels] = n;
    t.offset[t.levels] = off;
    off += n;
    ++t.levels;
    if (n <= 1) break;
    n = (n + LEAF - 1) / LEAF;
  }
  t.nodes = off;
  return t;
}

// Scratch of one tree over P points of type T, carved from `take` (256-byte aligned offsets)
struct Layout { size_t bbox, hi1, hi2, ka, kb, va, vb, hist, xs, ys, zs, boxes; };

template <class T, class Take>
Layout tree_layout(int P, Take&& take) {
  const Tree t = make_tree(P);
  const size_t padded = (size_t)t.count[0] * LEAF;
  Layout L;
  L.bbox = take(256);
  L.hi1 = take((size_t)P * 4); L.hi2 = take((size_t)P * 4);
  L.ka = take((size_t)P * 4); L.kb = take((size_t)P * 4); L.va = take((size_t)P * 4); L.vb = take((size_t)P * 4);
  L.hist = take(gof_sort_scratch_bytes((size_t)P));
  L.xs = take(padded * sizeof(T)); L.ys = take(padded * sizeof(T)); L.zs = take(padded * sizeof(T));
  L.boxes = take((size_t)t.nodes * 2 * sizeof(typename Coord<T>::V4));
  return L;
}

// T <-> unsigned with the same order (finite values)
template <class T>
__device__ __forceinline__ typename Coord<T>::U ord_of(T f) {
  using C = Coord<T>;
  const typename C::U u = C::bits(f);
  return (u & C::SIGN) ? ~u : (u | C::SIGN);
}
template <class T>
__device__ __forceinline__ T value_of(typename Coord<T>::U o) {
  using C = Coord<T>;
  return C::value((o & C::SIGN) ? (o & ~C::SIGN) : ~o);
}
template <class T>
__device__ __forceinline__ bool finite3(T x, T y, T z) { return isfinite(x) && isfinite(y) && isfinite(z); }

__device__ __forceinline__ uint32_t warp_min_u(uint32_t v) { return __reduce_min_sync(0xffffffffu, v); }
__device__ __forceinline__ uint32_t warp_max_u(uint32_t v) { return __reduce_max_sync(0xffffffffu, v); }
__device__ __forceinline__ unsigned long long warp_min_u(unsigned long long v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) { const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o); v = w < v ? w : v; }
  return v;
}
__device__ __forceinline__ unsigned long long warp_max_u(unsigned long long v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) { const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o); v = w > v ? w : v; }
  return v;
}

// bbox[0..2] = ordered min, bbox[3..5] = ordered max (initialised to all-ones / 0 by init_bbox)
template <class T>
__global__ void __launch_bounds__(THREADS) k_tree_bbox(int P, const T* __restrict__ pts, typename Coord<T>::U* __restrict__ bbox) {
  using U = typename Coord<T>::U;
  U mn[3] = {~(U)0, ~(U)0, ~(U)0}, mx[3] = {0, 0, 0};
  for (int i = blockIdx.x * THREADS + threadIdx.x; i < P; i += gridDim.x * THREADS) {
    const T x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
    if (!finite3(x, y, z)) continue;
    const U o[3] = {ord_of(x), ord_of(y), ord_of(z)};
#pragma unroll
    for (int a = 0; a < 3; ++a) { mn[a] = min(mn[a], o[a]); mx[a] = max(mx[a], o[a]); }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    mn[a] = warp_min_u(mn[a]);
    mx[a] = warp_max_u(mx[a]);
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (mn[a] != ~(U)0) atomicMin(bbox + a, mn[a]);
      if (mx[a] != 0) atomicMax(bbox + 3 + a, mx[a]);
    }
  }
}

// the low 21 bits of v at every third bit of a 64-bit word
__device__ __forceinline__ uint64_t spread21(uint32_t v) {
  uint64_t x = v & 0x1fffffu;
  x = (x | x << 32) & 0x001f00000000ffffull;
  x = (x | x << 16) & 0x001f0000ff0000ffull;
  x = (x | x << 8) & 0x100f00f00f00f00full;
  x = (x | x << 4) & 0x10c30c30c30c30c3ull;
  x = (x | x << 2) & 0x1249249249249249ull;
  return x;
}

// position -> [0, 2^32 - 2] over [lo, hi], clamped outside it; a zero extent maps to 0.  The subtraction and the quotient are
// monotone in v, so the key order follows the position order on each axis.  For v in [lo, hi] the clamps change nothing.
template <class T>
__device__ __forceinline__ uint32_t quantise(T v, T lo, T hi) {
  const double ext = (double)hi - (double)lo;
  if (!(ext > 0.0)) return 0u;
  const double t = ((double)v - (double)lo) / ext;
  if (!(t > 0.0)) return 0u;
  if (t >= 1.0) return 4294967294u;
  return (uint32_t)(t * 4294967294.0);
}

// 96-bit key over the box `bbox`, bit 3k + a = bit k of axis a: word 0 -> w0 (the sort's first key buffer), words 1, 2 -> hi1, hi2
template <class T>
__global__ void __launch_bounds__(THREADS) k_tree_keys(int P, const T* __restrict__ pts, const typename Coord<T>::U* __restrict__ bbox,
                                                       uint32_t* __restrict__ w0, uint32_t* __restrict__ hi1, uint32_t* __restrict__ hi2) {
  const int i = blockIdx.x * THREADS + threadIdx.x;
  if (i >= P) return;
  const T x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
  uint32_t k0 = 0xffffffffu, k1 = 0xffffffffu, k2 = 0xffffffffu;
  if (finite3(x, y, z)) {
    const uint32_t qx = quantise<T>(x, value_of<T>(bbox[0]), value_of<T>(bbox[3]));
    const uint32_t qy = quantise<T>(y, value_of<T>(bbox[1]), value_of<T>(bbox[4]));
    const uint32_t qz = quantise<T>(z, value_of<T>(bbox[2]), value_of<T>(bbox[5]));
    const uint64_t lo = spread21(qx) | spread21(qy) << 1 | spread21(qz) << 2;                    // key bits 0..62
    const uint64_t hi = spread21(qx >> 21) | spread21(qy >> 21) << 1 | spread21(qz >> 21) << 2;  // key bits 63..95
    k0 = (uint32_t)lo;
    k1 = (uint32_t)(lo >> 32) | (uint32_t)(hi << 31);
    k2 = (uint32_t)(hi >> 1);
  }
  w0[i] = k0; hi1[i] = k1; hi2[i] = k2;
}

// sorted coordinates into planes; slots P .. padded-1 hold NaN (never accepted, never in a box)
template <class T>
__global__ void __launch_bounds__(THREADS) k_tree_gather(int P, int padded, const T* __restrict__ pts, const uint32_t* __restrict__ order,
                                                         T* __restrict__ xs, T* __restrict__ ys, T* __restrict__ zs) {
  const int s = blockIdx.x * THREADS + threadIdx.x;
  if (s >= padded) return;
  T x = Coord<T>::nan(), y = x, z = x;
  if (s < P) {
    const size_t i = order[s];
    x = pts[3 * i]; y = pts[3 * i + 1]; z = pts[3 * i + 2];
  }
  xs[s] = x; ys[s] = y; zs[s] = z;
}

template <class T>
__device__ __forceinline__ T warp_vmin(T v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v = Coord<T>::vmin(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
template <class T>
__device__ __forceinline__ T warp_vmax(T v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v = Coord<T>::vmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// one warp per leaf: AABB of its finite points (empty: lo = +inf, hi = -inf, which every bound turns into +inf)
template <class T>
__global__ void __launch_bounds__(THREADS) k_tree_leaf_boxes(int leaves, const T* __restrict__ xs, const T* __restrict__ ys,
                                                             const T* __restrict__ zs, typename Coord<T>::V4* __restrict__ boxes) {
  const int leaf = (blockIdx.x * THREADS + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (leaf >= leaves) return;
  const size_t s = (size_t)leaf * LEAF + lane;
  const T x = xs[s], y = ys[s], z = zs[s];
  const bool ok = finite3(x, y, z);
  const T inf = (T)INFINITY;
  const T lx = warp_vmin(ok ? x : inf), ly = warp_vmin(ok ? y : inf), lz = warp_vmin(ok ? z : inf);
  const T hx = warp_vmax(ok ? x : -inf), hy = warp_vmax(ok ? y : -inf), hz = warp_vmax(ok ? z : -inf);
  if (lane == 0) {
    boxes[2 * (size_t)leaf] = Coord<T>::corner(lx, ly, lz);
    boxes[2 * (size_t)leaf + 1] = Coord<T>::corner(hx, hy, hz);
  }
}

// one warp per node of a level: union of its (up to) 32 children's boxes
template <class T>
__global__ void __launch_bounds__(THREADS) k_tree_node_boxes(int nodes, int children, const typename Coord<T>::V4* __restrict__ child,
                                                             typename Coord<T>::V4* __restrict__ boxes) {
  using V4 = typename Coord<T>::V4;
  const int node = (blockIdx.x * THREADS + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (node >= nodes) return;
  const int c = node * LEAF + lane;
  const T inf = (T)INFINITY;
  V4 lo = Coord<T>::corner(inf, inf, inf), hi = Coord<T>::corner(-inf, -inf, -inf);
  if (c < children) { lo = child[2 * (size_t)c]; hi = child[2 * (size_t)c + 1]; }
  lo.x = warp_vmin(lo.x); lo.y = warp_vmin(lo.y); lo.z = warp_vmin(lo.z);
  hi.x = warp_vmax(hi.x); hi.y = warp_vmax(hi.y); hi.z = warp_vmax(hi.z);
  if (lane == 0) { boxes[2 * (size_t)node] = lo; boxes[2 * (size_t)node + 1] = hi; }
}

static inline int blocks_for(size_t n, int per_block) { return (int)((n + per_block - 1) / per_block); }

// Device buffers of one tree, carved from a scratch block by a Layout
template <class T>
struct Bufs {
  typename Coord<T>::U* bbox;
  uint32_t *hi1, *hi2, *ka, *kb, *va, *vb, *hist;
  T *xs, *ys, *zs;
  typename Coord<T>::V4* boxes;
};

template <class T>
Bufs<T> carve(char* S, const Layout& L) {
  return Bufs<T>{(typename Coord<T>::U*)(S + L.bbox), (uint32_t*)(S + L.hi1), (uint32_t*)(S + L.hi2), (uint32_t*)(S + L.ka),
                 (uint32_t*)(S + L.kb), (uint32_t*)(S + L.va), (uint32_t*)(S + L.vb), (uint32_t*)(S + L.hist),
                 (T*)(S + L.xs), (T*)(S + L.ys), (T*)(S + L.zs), (typename Coord<T>::V4*)(S + L.boxes)};
}

// Builds the tree over pts[P,3] (P >= 1): afterwards b.va[s] = the point at sorted slot s, b.xs/ys/zs its coordinates and b.boxes
// the level boxes.  Enqueued on st; no host synchronisation.
template <class T>
int build_tree(int P, const T* pts, const Bufs<T>& b, const Tree& tree, cudaStream_t st) {
  using U = typename Coord<T>::U;
  const int padded = tree.count[0] * LEAF;
  const int gp = blocks_for((size_t)P, THREADS);
  int rc;
  GOF_CUDA_OK(cudaMemsetAsync(b.bbox, 0xff, 3 * sizeof(U), st));
  GOF_CUDA_OK(cudaMemsetAsync(b.bbox + 3, 0, 3 * sizeof(U), st));
  const int gb = gp < 1056 ? gp : 1056;
  GOF_LAUNCH("tree_bbox", st, k_tree_bbox<T><<<gb, THREADS, 0, st>>>(P, pts, b.bbox));
  GOF_LAUNCH_CHECK(false, st);
  GOF_LAUNCH("tree_keys", st, k_tree_keys<T><<<gp, THREADS, 0, st>>>(P, pts, b.bbox, b.ka, b.hi1, b.hi2));
  GOF_LAUNCH_CHECK(false, st);
  const GofKeyWords key{{b.ka, b.hi1, b.hi2}, {32, 32, 32}, 3};
  if ((rc = gof_sort_words_u32(key, (size_t)P, GofSortBufs{b.ka, b.kb, b.va, b.vb, b.hist}, b.va, false, st)) != GOF_OK) return rc;
  GOF_LAUNCH("tree_gather", st, k_tree_gather<T><<<blocks_for((size_t)padded, THREADS), THREADS, 0, st>>>(P, padded, pts, b.va, b.xs,
                                                                                                          b.ys, b.zs));
  GOF_LAUNCH_CHECK(false, st);
  GOF_LAUNCH("tree_leaf_boxes", st, k_tree_leaf_boxes<T><<<blocks_for((size_t)tree.count[0] * 32, THREADS), THREADS, 0, st>>>(
                                        tree.count[0], b.xs, b.ys, b.zs, b.boxes));
  GOF_LAUNCH_CHECK(false, st);
  for (int l = 1; l < tree.levels; ++l) {
    GOF_LAUNCH("tree_node_boxes", st, k_tree_node_boxes<T><<<blocks_for((size_t)tree.count[l] * 32, THREADS), THREADS, 0, st>>>(
                                          tree.count[l], tree.count[l - 1], b.boxes + 2 * tree.offset[l - 1], b.boxes + 2 * tree.offset[l]));
    GOF_LAUNCH_CHECK(false, st);
  }
  return GOF_OK;
}

}  // namespace gof_tree
