// knn.cu -- mean squared distance to the three nearest neighbours of every point: simple_knn's distCUDA2
// (submodules/simple-knn/spatial.cu:15-25, simple_knn.cu:147-183), which GaussianModel.create_from_pcd uses to initialise
// the scales.  The contract is DESIGN section 4.5: out_i = ((b0 + b1) + b2) / 3 over the three smallest accepted
// d(i,j) = fmaf(dz, dz, fmaf(dx, dx, dy*dy)), j != i by index, accepted iff d < FLT_MAX, padded with FLT_MAX.  Every float
// step below is one explicit IEEE operation, so the result is bit-identical to the reference whatever order the search
// takes (the reference's own pruning is exact, so its output does not depend on its search order either).
//
//   bbox     order-free min / max of the finite points (ordered-integer atomics) into scratch
//   keys     96-bit Morton code of each point over that box (32 bits per axis, quantised in double); non-finite points
//            get the all-ones key, which no finite point can have, so they sort last
//   sort     the library's multi-word sort, the key as three u32 words
//   gather   sorted coordinates into three planes, padded with NaN to whole leaves of 32
//   boxes    one AABB per leaf of 32 consecutive points (finite points only), then an implicit 32-ary tree of unions
//   search   one warp per leaf: seed from the leaf itself, then a depth-first walk from the root, nearest child first.  A
//            node is entered while some lane's point-to-box bound is below that lane's best[2]; a child is pushed while
//            its box-to-box bound against the leaf's query box is below the warp's largest best[2]
//
// Bounds have the shape of d: per axis the rounded gap to the box (0 inside), then fmaf(gz,gz,fmaf(gx,gx,gy*gy)).
// Rounding is monotone, so a bound never exceeds d for any point in the box, and pruning at bound >= best[2] never drops
// a distance that could change the three values (an equal one cannot).  No host synchronisation, no allocation: every size
// follows from P, so a call can be captured in a CUDA graph.
#include <float.h>
#include <math.h>

#include "gof_common.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int SEARCH_WARPS = 4;              // warps per CTA of the search kernel
constexpr int LEAF = 32;
constexpr int MAX_LEVELS = 8;                // 2^31 points: 2^26 leaves, 32-ary -> 7 levels
constexpr int STACK = 256;                   // per warp; a walk holds at most 31 entries per level + 1
constexpr int LEVEL_SHIFT = 26;              // stack entry: level << 26 | node (node < 2^26)

struct KnnTree {
  int levels;                                // level 0 = leaves, levels-1 = the root (one node)
  int count[MAX_LEVELS];                     // nodes per level
  long long offset[MAX_LEVELS];              // first box of each level in the box array
  long long nodes;                           // boxes in all levels
};

KnnTree knn_tree(int P) {
  KnnTree t{};
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

struct KnnLayout { size_t bbox, hi1, hi2, ka, kb, va, vb, hist, xs, ys, zs, boxes, bytes; };

KnnLayout knn_layout(int P) {
  const KnnTree t = knn_tree(P);
  const size_t padded = (size_t)t.count[0] * LEAF;
  KnnLayout L; size_t o = 0;
  auto take = [&](size_t b) { size_t r = o; o = gof_align_up(o + b, 256); return r; };
  L.bbox = take(256);
  L.hi1 = take((size_t)P * 4); L.hi2 = take((size_t)P * 4);
  L.ka = take((size_t)P * 4); L.kb = take((size_t)P * 4); L.va = take((size_t)P * 4); L.vb = take((size_t)P * 4);
  L.hist = take(gof_sort_scratch_bytes((size_t)P));
  L.xs = take(padded * 4); L.ys = take(padded * 4); L.zs = take(padded * 4);
  L.boxes = take((size_t)t.nodes * 2 * sizeof(float4));
  L.bytes = o;
  return L;
}

// float <-> unsigned with the same order (finite values)
__device__ __forceinline__ uint32_t ord_of(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float float_of(uint32_t o) {
  return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}
__device__ __forceinline__ bool finite3(float x, float y, float z) { return isfinite(x) && isfinite(y) && isfinite(z); }

// bbox[0..2] = ordered min, bbox[3..5] = ordered max (initialised to 0xFFFFFFFF / 0 by the caller)
__global__ void __launch_bounds__(THREADS) k_knn_bbox(int P, const float* __restrict__ pts, uint32_t* __restrict__ bbox) {
  uint32_t mn[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, mx[3] = {0u, 0u, 0u};
  for (int i = blockIdx.x * THREADS + threadIdx.x; i < P; i += gridDim.x * THREADS) {
    const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
    if (!finite3(x, y, z)) continue;
    const uint32_t o[3] = {ord_of(x), ord_of(y), ord_of(z)};
#pragma unroll
    for (int a = 0; a < 3; ++a) { mn[a] = min(mn[a], o[a]); mx[a] = max(mx[a], o[a]); }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    mn[a] = __reduce_min_sync(0xffffffffu, mn[a]);
    mx[a] = __reduce_max_sync(0xffffffffu, mx[a]);
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (mn[a] != 0xffffffffu) atomicMin(bbox + a, mn[a]);
      if (mx[a] != 0u) atomicMax(bbox + 3 + a, mx[a]);
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

// position in [min, max] -> [0, 2^32 - 2]; a zero extent maps to 0.  Double keeps the difference of two floats monotone
// and the quotient at most 1.
__device__ __forceinline__ uint32_t quantise(float v, float lo, float hi) {
  const double ext = (double)hi - (double)lo;
  if (!(ext > 0.0)) return 0u;
  const double t = ((double)v - (double)lo) / ext;
  return (uint32_t)(t * 4294967294.0);
}

// 96-bit key, bit 3k + a = bit k of axis a: word 0 -> ka (the sort's first key buffer), words 1, 2 -> hi1, hi2
__global__ void __launch_bounds__(THREADS) k_knn_keys(int P, const float* __restrict__ pts, const uint32_t* __restrict__ bbox,
                                                      uint32_t* __restrict__ w0, uint32_t* __restrict__ hi1,
                                                      uint32_t* __restrict__ hi2) {
  const int i = blockIdx.x * THREADS + threadIdx.x;
  if (i >= P) return;
  const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
  uint32_t k0 = 0xffffffffu, k1 = 0xffffffffu, k2 = 0xffffffffu;
  if (finite3(x, y, z)) {
    const uint32_t qx = quantise(x, float_of(bbox[0]), float_of(bbox[3]));
    const uint32_t qy = quantise(y, float_of(bbox[1]), float_of(bbox[4]));
    const uint32_t qz = quantise(z, float_of(bbox[2]), float_of(bbox[5]));
    const uint64_t lo = spread21(qx) | spread21(qy) << 1 | spread21(qz) << 2;                    // key bits 0..62
    const uint64_t hi = spread21(qx >> 21) | spread21(qy >> 21) << 1 | spread21(qz >> 21) << 2;  // key bits 63..95
    k0 = (uint32_t)lo;
    k1 = (uint32_t)(lo >> 32) | (uint32_t)(hi << 31);
    k2 = (uint32_t)(hi >> 1);
  }
  w0[i] = k0; hi1[i] = k1; hi2[i] = k2;
}

// sorted coordinates into planes; slots P .. padded-1 hold NaN (never accepted, never in a box)
__global__ void __launch_bounds__(THREADS) k_knn_gather_points(int P, int padded, const float* __restrict__ pts,
                                                               const uint32_t* __restrict__ order, float* __restrict__ xs,
                                                               float* __restrict__ ys, float* __restrict__ zs) {
  const int s = blockIdx.x * THREADS + threadIdx.x;
  if (s >= padded) return;
  float x = __int_as_float(0x7fc00000), y = x, z = x;
  if (s < P) {
    const size_t i = order[s];
    x = pts[3 * i]; y = pts[3 * i + 1]; z = pts[3 * i + 2];
  }
  xs[s] = x; ys[s] = y; zs[s] = z;
}

__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// one warp per leaf: AABB of its finite points (empty: lo = +inf, hi = -inf, which every bound turns into +inf)
__global__ void __launch_bounds__(THREADS) k_knn_leaf_boxes(int leaves, const float* __restrict__ xs, const float* __restrict__ ys,
                                                            const float* __restrict__ zs, float4* __restrict__ boxes) {
  const int leaf = (blockIdx.x * THREADS + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (leaf >= leaves) return;
  const size_t s = (size_t)leaf * LEAF + lane;
  const float x = xs[s], y = ys[s], z = zs[s];
  const bool ok = finite3(x, y, z);
  const float lx = warp_min(ok ? x : INFINITY), ly = warp_min(ok ? y : INFINITY), lz = warp_min(ok ? z : INFINITY);
  const float hx = warp_max(ok ? x : -INFINITY), hy = warp_max(ok ? y : -INFINITY), hz = warp_max(ok ? z : -INFINITY);
  if (lane == 0) {
    boxes[2 * (size_t)leaf] = make_float4(lx, ly, lz, 0.f);
    boxes[2 * (size_t)leaf + 1] = make_float4(hx, hy, hz, 0.f);
  }
}

// one warp per node of a level: union of its (up to) 32 children's boxes
__global__ void __launch_bounds__(THREADS) k_knn_node_boxes(int nodes, int children, const float4* __restrict__ child,
                                                            float4* __restrict__ boxes) {
  const int node = (blockIdx.x * THREADS + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (node >= nodes) return;
  const int c = node * LEAF + lane;
  float4 lo = make_float4(INFINITY, INFINITY, INFINITY, 0.f), hi = make_float4(-INFINITY, -INFINITY, -INFINITY, 0.f);
  if (c < children) { lo = child[2 * (size_t)c]; hi = child[2 * (size_t)c + 1]; }
  lo.x = warp_min(lo.x); lo.y = warp_min(lo.y); lo.z = warp_min(lo.z);
  hi.x = warp_max(hi.x); hi.y = warp_max(hi.y); hi.z = warp_max(hi.z);
  if (lane == 0) { boxes[2 * (size_t)node] = lo; boxes[2 * (size_t)node + 1] = hi; }
}

// rounded gap between [qlo, qhi] and [lo, hi] on one axis (a point is qlo == qhi); 0 where they overlap
__device__ __forceinline__ float gap(float qlo, float qhi, float lo, float hi) {
  if (qhi < lo) return __fsub_rn(lo, qhi);
  if (qlo > hi) return __fsub_rn(qlo, hi);
  return 0.f;
}
// the reference's d.x*d.x + d.y*d.y + d.z*d.z as nvcc contracts it (SASS of updateKBest: FMUL y, FFMA x, FFMA z)
__device__ __forceinline__ float sq3(float gx, float gy, float gz) {
  return __fmaf_rn(gz, gz, __fmaf_rn(gx, gx, __fmul_rn(gy, gy)));
}

// the reference's insertion rule (updateKBest<3>, simple_knn.cu:132-145): NaN and values >= FLT_MAX never enter
__device__ __forceinline__ void insert(float d, float& b0, float& b1, float& b2) {
  if (b0 > d) { const float t = b0; b0 = d; d = t; }
  if (b1 > d) { const float t = b1; b1 = d; d = t; }
  if (b2 > d) b2 = d;
}

// every lane offers its query all 32 points of leaf `leaf` (except itself, by sorted position == index)
__device__ __forceinline__ void visit_leaf(int leaf, int lane, int self, float qx, float qy, float qz, const float* __restrict__ xs,
                                           const float* __restrict__ ys, const float* __restrict__ zs, float& b0, float& b1,
                                           float& b2) {
  const size_t base = (size_t)leaf * LEAF;
  const float cx = xs[base + lane], cy = ys[base + lane], cz = zs[base + lane];
  const int skip = self - leaf * LEAF;   // in 0..31 only for the query's own leaf
#pragma unroll 8
  for (int k = 0; k < LEAF; ++k) {
    const float px = __shfl_sync(0xffffffffu, cx, k), py = __shfl_sync(0xffffffffu, cy, k), pz = __shfl_sync(0xffffffffu, cz, k);
    const float d = sq3(__fsub_rn(px, qx), __fsub_rn(py, qy), __fsub_rn(pz, qz));
    if (k != skip) insert(d, b0, b1, b2);
  }
}

__global__ void __launch_bounds__(SEARCH_WARPS * 32) k_knn_search(int P, KnnTree tree, const float* __restrict__ xs,
                                                                  const float* __restrict__ ys, const float* __restrict__ zs,
                                                                  const uint32_t* __restrict__ order,
                                                                  const float4* __restrict__ boxes, float* __restrict__ out) {
  __shared__ uint32_t s_stack[SEARCH_WARPS][STACK];
  __shared__ int s_count[MAX_LEVELS];          // the level tables, indexed at run time: in shared memory, not a stack frame
  __shared__ long long s_offset[MAX_LEVELS];
  if (threadIdx.x == 0) {
#pragma unroll
    for (int l = 0; l < MAX_LEVELS; ++l) { s_count[l] = tree.count[l]; s_offset[l] = tree.offset[l]; }
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int leaf = blockIdx.x * SEARCH_WARPS + warp;
  if (leaf >= tree.count[0]) return;
  uint32_t* stack = s_stack[warp];
  const int self = leaf * LEAF + lane;
  const float qx = xs[self], qy = ys[self], qz = zs[self];
  const bool valid = finite3(qx, qy, qz);
  float b0 = FLT_MAX, b1 = FLT_MAX, b2 = FLT_MAX;
  if (__any_sync(0xffffffffu, valid)) {
    visit_leaf(leaf, lane, self, qx, qy, qz, xs, ys, zs, b0, b1, b2);
    const float qlx = warp_min(valid ? qx : INFINITY), qly = warp_min(valid ? qy : INFINITY), qlz = warp_min(valid ? qz : INFINITY);
    const float qhx = warp_max(valid ? qx : -INFINITY), qhy = warp_max(valid ? qy : -INFINITY), qhz = warp_max(valid ? qz : -INFINITY);
    int sp = 0;
    if (tree.levels > 1) {
      if (lane == 0) stack[0] = (uint32_t)(tree.levels - 1) << LEVEL_SHIFT;
      sp = 1;
    }
    __syncwarp();
    while (sp > 0) {
      const uint32_t e = stack[--sp];
      const int lvl = (int)(e >> LEVEL_SHIFT), node = (int)(e & ((1u << LEVEL_SHIFT) - 1));
      if (lvl == 0 && node == leaf) continue;
      const float4* nb = boxes + 2 * (s_offset[lvl] + node);
      const float4 lo = nb[0], hi = nb[1];
      const bool need = valid && sq3(gap(qx, qx, lo.x, hi.x), gap(qy, qy, lo.y, hi.y), gap(qz, qz, lo.z, hi.z)) < b2;
      if (!__any_sync(0xffffffffu, need)) continue;
      if (lvl == 0) {
        visit_leaf(node, lane, self, qx, qy, qz, xs, ys, zs, b0, b1, b2);
        continue;
      }
      // children: one per lane, pushed farthest first so that the nearest is popped next
      const float thr = __uint_as_float(__reduce_max_sync(0xffffffffu, valid ? __float_as_uint(b2) : 0u));   // b2 >= 0
      const int c = node * LEAF + lane;
      float cb = INFINITY;
      if (c < s_count[lvl - 1]) {
        const float4* cbx = boxes + 2 * (s_offset[lvl - 1] + c);
        const float4 clo = cbx[0], chi = cbx[1];
        cb = sq3(gap(qlx, qhx, clo.x, chi.x), gap(qly, qhy, clo.y, chi.y), gap(qlz, qhz, clo.z, chi.z));
      }
      const bool push = cb < thr;
      const uint32_t mask = __ballot_sync(0xffffffffu, push);
      int rank = 0;
#pragma unroll 8
      for (int k = 0; k < 32; ++k) {
        const float o = __shfl_sync(0xffffffffu, cb, k);
        rank += ((mask >> k) & 1u) && (o < cb || (o == cb && k < lane));
      }
      const int n = __popc(mask);
      __syncwarp();
      if (push) stack[sp + n - 1 - rank] = ((uint32_t)(lvl - 1) << LEVEL_SHIFT) | (uint32_t)c;
      sp += n;
      __syncwarp();
    }
  }
  if (self < P) out[order[self]] = __fdiv_rn(__fadd_rn(__fadd_rn(b0, b1), b2), 3.0f);
}

int blocks_for(size_t n, int per_block) { return (int)((n + per_block - 1) / per_block); }

}  // namespace

extern "C" GOF_API size_t gof_knn_scratch_bytes(int P) {
  if (P <= 0) return 0;
  return knn_layout(P).bytes;
}

extern "C" GOF_API int gof_knn_mean_dist(int P, const float* points, float* mean_dists, void* scratch, size_t scratch_bytes,
                                         void* stream) {
  if (P < 0) { gof_set_error("knn_mean_dist: P = %d < 0", P); return GOF_E_INVALID; }
  if (P == 0) return GOF_OK;
  if (!points || !mean_dists || !scratch) { gof_set_error("knn_mean_dist: NULL argument"); return GOF_E_INVALID; }
  const KnnLayout L = knn_layout(P);
  if (scratch_bytes < L.bytes) {
    gof_set_error("knn_mean_dist: scratch of %zu bytes, %zu needed (gof_knn_scratch_bytes)", scratch_bytes, L.bytes);
    return GOF_E_INVALID;
  }
  const KnnTree tree = knn_tree(P);
  cudaStream_t st = (cudaStream_t)stream;
  char* S = static_cast<char*>(scratch);
  uint32_t* bbox = (uint32_t*)(S + L.bbox);
  uint32_t *hi1 = (uint32_t*)(S + L.hi1), *hi2 = (uint32_t*)(S + L.hi2);
  uint32_t *ka = (uint32_t*)(S + L.ka), *kb = (uint32_t*)(S + L.kb), *va = (uint32_t*)(S + L.va), *vb = (uint32_t*)(S + L.vb);
  uint32_t* hist = (uint32_t*)(S + L.hist);
  float *xs = (float*)(S + L.xs), *ys = (float*)(S + L.ys), *zs = (float*)(S + L.zs);
  float4* boxes = (float4*)(S + L.boxes);
  const int padded = tree.count[0] * LEAF;
  const int gp = blocks_for((size_t)P, THREADS);
  int rc;

  GOF_CUDA_OK(cudaMemsetAsync(bbox, 0xff, 12, st));
  GOF_CUDA_OK(cudaMemsetAsync(bbox + 3, 0, 12, st));
  const int gb = gp < 1056 ? gp : 1056;
  GOF_LAUNCH("knn_bbox", st, k_knn_bbox<<<gb, THREADS, 0, st>>>(P, points, bbox));
  GOF_LAUNCH_CHECK(false, st);
  GOF_LAUNCH("knn_keys", st, k_knn_keys<<<gp, THREADS, 0, st>>>(P, points, bbox, ka, hi1, hi2));
  GOF_LAUNCH_CHECK(false, st);
  const GofKeyWords key{{ka, hi1, hi2}, {32, 32, 32}, 3};
  if ((rc = gof_sort_words_u32(key, (size_t)P, GofSortBufs{ka, kb, va, vb, hist}, va, false, st)) != GOF_OK) return rc;
  GOF_LAUNCH("knn_gather_points", st, k_knn_gather_points<<<blocks_for((size_t)padded, THREADS), THREADS, 0, st>>>(
                                          P, padded, points, va, xs, ys, zs));
  GOF_LAUNCH_CHECK(false, st);
  GOF_LAUNCH("knn_leaf_boxes", st, k_knn_leaf_boxes<<<blocks_for((size_t)tree.count[0] * 32, THREADS), THREADS, 0, st>>>(
                                       tree.count[0], xs, ys, zs, boxes));
  GOF_LAUNCH_CHECK(false, st);
  for (int l = 1; l < tree.levels; ++l) {
    GOF_LAUNCH("knn_node_boxes", st, k_knn_node_boxes<<<blocks_for((size_t)tree.count[l] * 32, THREADS), THREADS, 0, st>>>(
                                         tree.count[l], tree.count[l - 1], boxes + 2 * tree.offset[l - 1], boxes + 2 * tree.offset[l]));
    GOF_LAUNCH_CHECK(false, st);
  }
  GOF_LAUNCH("knn_search", st, k_knn_search<<<blocks_for((size_t)tree.count[0], SEARCH_WARPS), SEARCH_WARPS * 32, 0, st>>>(
                                   P, tree, xs, ys, zs, va, boxes, mean_dists));
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}
