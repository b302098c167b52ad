// dtu_eval.cu -- the DTU mesh evaluation of dtu_eval/eval.py on the GPU (DESIGN section 4.6): sampling a mesh at a density,
// the order-dependent greedy downsample, and the nearest-neighbour distances between two clouds.  Coordinates are double;
// every arithmetic step is one IEEE double operation written out (__dmul_rn / __dadd_rn / __dsub_rn / __ddiv_rn / __dsqrt_rn),
// so nvcc cannot contract it and a numpy restatement of the same steps reproduces each value bit for bit.
//
//   sample     per face: v1 = p1 - p0, v2 = p2 - p0, l = |v| as sqrt((x*x + y*y) + z*z), area2 = |v1 x v2|, faces with
//              area2 > 0 only; thr = r * sqrt((l1*l2) / area2), n1 = floor(l1 / thr), n2 = floor(l2 / thr); sample (i, j),
//              0 <= i <= n1, 0 <= j <= n2, exists iff fl(c0 + c1) < 1, c0 = (i + 0.5) / max(n1, 1e-7), c1 likewise; it sits
//              at (v1*c0 + v2*c1) + p0.  Rows (face, i) are flattened: one thread per row counts its samples by a binary search
//              on j (the predicate is monotone in j), one thread per sample finds its row and face by binary searches in the
//              scanned offsets, so a face with millions of samples does not serialise on a thread.
//   downsample in a given order, a point is kept iff no earlier kept point lies within ((dx*dx + dy*dy) + dz*dz) <= r*r.  The
//              earlier neighbours of every point are listed in CSR form (count, scan, emit over the box tree of knn_tree.cuh),
//              then rounds decide points: one whose listed neighbours are all removed is kept, one with a kept neighbour is
//              removed.  Each round reads the previous round's states only, so the number of rounds is deterministic; each
//              decides at least the earliest undecided point, and a random order needs polylogarithmically many.
//   nn_dist    min over the reference points of ((dx*dx + dy*dy) + dz*dz) for every query (and its sqrt): the queries are
//              Morton-keyed against the reference tree's box (clamped), sorted, and searched one warp per 32 of them, nearest
//              child first, with the pruning of DESIGN section 4.5 on double bounds.
//
// A bound is the same formula over the per-axis rounded gaps to a box (0 inside); rounding is monotone, so it never exceeds the
// value for a point in the box.  The radius search enters a node while some lane's bound is <= r*r, the 1-NN search while it
// is < that lane's best; neither can drop a point that decides the result.
#include <float.h>
#include <math.h>

#include "knn_tree.cuh"

namespace {

using gof_tree::LEAF;
using gof_tree::LEVEL_SHIFT;
using gof_tree::MAX_LEVELS;
using gof_tree::THREADS;
using gof_tree::blocks_for;
using gof_tree::finite3;
using gof_tree::warp_vmax;
using gof_tree::warp_vmin;

constexpr int SEARCH_WARPS = 4;              // warps per CTA of the search kernels
constexpr int STACK = 256;                   // per warp; a walk holds at most 31 entries per level + 1
constexpr size_t SORT_LIMIT = (size_t)1 << 30;   // the radix passes' item limit (DESIGN section 4.4)
constexpr int ROUND_BATCH = 8;               // downsample rounds enqueued between two reads of the undecided counts

auto layout_taker(size_t& o) {
  return [&o](size_t b) { size_t r = o; o = gof_align_up(o + b, 256); return r; };
}

__device__ __forceinline__ double sq3(double x, double y, double z) {
  return __dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z));
}
// rounded gap between [qlo, qhi] and [lo, hi] on one axis (a point is qlo == qhi); 0 where they overlap
__device__ __forceinline__ double gap(double qlo, double qhi, double lo, double hi) {
  if (qhi < lo) return __dsub_rn(lo, qhi);
  if (qlo > hi) return __dsub_rn(qlo, hi);
  return 0.0;
}

__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// first index in a[0, n) whose value exceeds v (a non-decreasing)
__device__ __forceinline__ size_t upper_bound_u32(const uint32_t* __restrict__ a, size_t n, uint32_t v) {
  size_t lo = 0, hi = n;
  while (lo < hi) {
    const size_t mid = (lo + hi) >> 1;
    if (a[mid] <= v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// ---- sample -----------------------------------------------------------------------------------------------------

struct Face {
  double p0[3], v1[3], v2[3];
  double n1, n2;
  bool ok;                                   // area2 > 0
};

__device__ __forceinline__ Face face_geom(const double* __restrict__ V, const int64_t* __restrict__ F, size_t f, double r) {
  Face g;
  const int64_t a = F[3 * f], b = F[3 * f + 1], c = F[3 * f + 2];
  double p1[3], p2[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    g.p0[k] = V[3 * a + k]; p1[k] = V[3 * b + k]; p2[k] = V[3 * c + k];
    g.v1[k] = __dsub_rn(p1[k], g.p0[k]);
    g.v2[k] = __dsub_rn(p2[k], g.p0[k]);
  }
  const double* u = g.v1;
  const double* w = g.v2;
  const double cx = __dsub_rn(__dmul_rn(u[1], w[2]), __dmul_rn(u[2], w[1]));   // numpy.cross: two rounded products, then the difference
  const double cy = __dsub_rn(__dmul_rn(u[2], w[0]), __dmul_rn(u[0], w[2]));
  const double cz = __dsub_rn(__dmul_rn(u[0], w[1]), __dmul_rn(u[1], w[0]));
  const double l1 = __dsqrt_rn(sq3(u[0], u[1], u[2]));
  const double l2 = __dsqrt_rn(sq3(w[0], w[1], w[2]));
  const double area2 = __dsqrt_rn(sq3(cx, cy, cz));
  g.ok = area2 > 0.0;
  const double thr = __dmul_rn(r, __dsqrt_rn(__ddiv_rn(__dmul_rn(l1, l2), area2)));
  g.n1 = floor(__ddiv_rn(l1, thr));
  g.n2 = floor(__ddiv_rn(l2, thr));
  return g;
}

// Python's max(n, 1e-7)
__device__ __forceinline__ double denom(double n) { return 1e-7 > n ? 1e-7 : n; }
__device__ __forceinline__ double coef(double i, double n) { return __ddiv_rn(__dadd_rn(i, 0.5), denom(n)); }

// a face's rows are 0..n1; more than 2^31 rows or columns in one face is refused
constexpr double MAX_SPAN = 2147483647.0;

struct FaceHeader { uint32_t err, rows32; unsigned long long rows64; };
struct RowHeader { uint32_t samples32, pad; unsigned long long samples64; unsigned long long rows; };

__global__ void __launch_bounds__(THREADS) k_face_rows(size_t nv, const double* __restrict__ V, size_t nf, const int64_t* __restrict__ F,
                                                       double r, uint32_t* __restrict__ rows, FaceHeader* __restrict__ hd) {
  const size_t f = (size_t)blockIdx.x * THREADS + threadIdx.x;
  unsigned long long n = 0;
  if (f < nf) {
    bool in_range = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) { const int64_t v = F[3 * f + k]; in_range &= v >= 0 && (uint64_t)v < nv; }
    if (!in_range) {
      atomicOr(&hd->err, 1u);
    } else {
      const Face g = face_geom(V, F, f, r);
      if (g.ok) {
        if (!(g.n1 < MAX_SPAN && g.n2 < MAX_SPAN)) atomicOr(&hd->err, 2u);
        else n = (unsigned long long)g.n1 + 1;
      }
    }
    rows[f] = (uint32_t)n;
  }
  n = warp_sum_u64(n);
  if ((threadIdx.x & 31) == 0 && n) atomicAdd(&hd->rows64, n);
}

// row -> (face, i): the last face whose first row is <= row (faces without rows share their successor's offset)
__device__ __forceinline__ void row_of(size_t row, const uint32_t* __restrict__ row_start, size_t nf, size_t* f, double* i) {
  const size_t face = upper_bound_u32(row_start, nf, (uint32_t)row) - 1;
  *f = face;
  *i = (double)(row - row_start[face]);
}

__global__ void __launch_bounds__(THREADS) k_row_count(size_t R, const double* __restrict__ V, size_t nf, const int64_t* __restrict__ F,
                                                       double r, const uint32_t* __restrict__ row_start, uint32_t* __restrict__ cnt,
                                                       RowHeader* __restrict__ hd) {
  const size_t row = (size_t)blockIdx.x * THREADS + threadIdx.x;
  unsigned long long n = 0;
  if (row < R) {
    size_t f; double i;
    row_of(row, row_start, nf, &f, &i);
    const Face g = face_geom(V, F, f, r);
    const double c0 = coef(i, g.n1);
    // samples of the row: the first j in [0, n2 + 1) whose c0 + c1 is not below 1 (monotone in j)
    long long lo = 0, hi = (long long)g.n2 + 1;
    while (lo < hi) {
      const long long mid = (lo + hi) >> 1;
      if (__dadd_rn(c0, coef((double)mid, g.n2)) < 1.0) lo = mid + 1; else hi = mid;
    }
    n = (unsigned long long)lo;
    cnt[row] = (uint32_t)lo;
  }
  n = warp_sum_u64(n);
  if ((threadIdx.x & 31) == 0 && n) atomicAdd(&hd->samples64, n);
}

__global__ void __launch_bounds__(THREADS) k_sample_emit(size_t S, size_t R, const double* __restrict__ V, size_t nf,
                                                         const int64_t* __restrict__ F, double r, const uint32_t* __restrict__ row_start,
                                                         const uint32_t* __restrict__ sample_off, double* __restrict__ out) {
  const size_t s = (size_t)blockIdx.x * THREADS + threadIdx.x;
  if (s >= S) return;
  const size_t row = upper_bound_u32(sample_off, R, (uint32_t)s) - 1;
  size_t f; double i;
  row_of(row, row_start, nf, &f, &i);
  const Face g = face_geom(V, F, f, r);
  const double c0 = coef(i, g.n1), c1 = coef((double)(s - sample_off[row]), g.n2);
#pragma unroll
  for (int k = 0; k < 3; ++k) out[3 * s + k] = __dadd_rn(__dadd_rn(__dmul_rn(g.v1[k], c0), __dmul_rn(g.v2[k], c1)), g.p0[k]);
}

struct FaceLayout { size_t header, rows, row_start, scan_tmp, bytes; };
FaceLayout face_layout(size_t nf) {
  FaceLayout L; size_t o = 0;
  auto take = layout_taker(o);
  L.header = take(sizeof(FaceHeader));
  L.rows = take(nf * 4); L.row_start = take(nf * 4); L.scan_tmp = take(gof_scan_scratch_bytes(nf));
  L.bytes = o;
  return L;
}
struct RowLayout { size_t header, cnt, off, scan_tmp, bytes; };
RowLayout row_layout(size_t R) {
  RowLayout L; size_t o = 0;
  auto take = layout_taker(o);
  L.header = take(sizeof(RowHeader));
  L.cnt = take(R * 4); L.off = take(R * 4); L.scan_tmp = take(gof_scan_scratch_bytes(R));
  L.bytes = o;
  return L;
}

// ---- downsample -------------------------------------------------------------------------------------------------

struct DownHeader { unsigned long long pairs64; uint32_t pairs32, err; uint32_t undecided[ROUND_BATCH]; };

// pts in the given order; seen[p] counts how often p occurs in perm
__global__ void __launch_bounds__(THREADS) k_perm_gather(size_t n, const double* __restrict__ pts, const uint32_t* __restrict__ perm,
                                                         double* __restrict__ out, uint32_t* __restrict__ seen, DownHeader* __restrict__ hd) {
  const size_t k = (size_t)blockIdx.x * THREADS + threadIdx.x;
  if (k >= n) return;
  const uint32_t p = perm[k];
  if (p >= n) {
    atomicOr(&hd->err, 1u);
    out[3 * k] = out[3 * k + 1] = out[3 * k + 2] = __longlong_as_double(0x7ff8000000000000ll);
    return;
  }
  atomicAdd(seen + p, 1u);
  out[3 * k] = pts[3 * (size_t)p]; out[3 * k + 1] = pts[3 * (size_t)p + 1]; out[3 * k + 2] = pts[3 * (size_t)p + 2];
}

__global__ void __launch_bounds__(THREADS) k_perm_check(size_t n, const uint32_t* __restrict__ seen, DownHeader* __restrict__ hd) {
  const size_t k = (size_t)blockIdx.x * THREADS + threadIdx.x;
  if (k < n && seen[k] != 1u) atomicOr(&hd->err, 1u);
}

// One warp per leaf of the tree over the ordered points; lane = one point q (its position in the order: qidx).  Lists every
// point p with ((dx*dx + dy*dy) + dz*dz) <= r2 and an earlier position: EMIT = false counts them into cnt[qidx] (and the total),
// EMIT = true writes their positions to nbr[off[qidx] ...] in the walk's order.
template <bool EMIT>
__global__ void __launch_bounds__(SEARCH_WARPS * 32) k_radius_pairs(int n, gof_tree::Tree tree, const double* __restrict__ xs,
                                                                    const double* __restrict__ ys, const double* __restrict__ zs,
                                                                    const uint32_t* __restrict__ order, const double4* __restrict__ boxes,
                                                                    double r2, uint32_t* __restrict__ cnt, const uint32_t* __restrict__ off,
                                                                    uint32_t* __restrict__ nbr, DownHeader* __restrict__ hd) {
  __shared__ uint32_t s_stack[SEARCH_WARPS][STACK];
  __shared__ int s_count[MAX_LEVELS];
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
  const double qx = xs[self], qy = ys[self], qz = zs[self];
  const bool valid = self < n && finite3(qx, qy, qz);
  const uint32_t qidx = self < n ? order[self] : 0u;
  uint32_t c = 0;
  const uint32_t base = (EMIT && valid) ? off[qidx] : 0u;
  if (__any_sync(0xffffffffu, valid)) {
    const double inf = INFINITY;
    const double qlx = warp_vmin(valid ? qx : inf), qly = warp_vmin(valid ? qy : inf), qlz = warp_vmin(valid ? qz : inf);
    const double qhx = warp_vmax(valid ? qx : -inf), qhy = warp_vmax(valid ? qy : -inf), qhz = warp_vmax(valid ? qz : -inf);
    if (lane == 0) stack[0] = (uint32_t)(tree.levels - 1) << LEVEL_SHIFT;
    int sp = 1;
    __syncwarp();
    while (sp > 0) {
      const uint32_t e = stack[--sp];
      const int lvl = (int)(e >> LEVEL_SHIFT), node = (int)(e & ((1u << LEVEL_SHIFT) - 1));
      const double4* nb = boxes + 2 * (s_offset[lvl] + node);
      const double4 lo = nb[0], hi = nb[1];
      const bool need = valid && sq3(gap(qx, qx, lo.x, hi.x), gap(qy, qy, lo.y, hi.y), gap(qz, qz, lo.z, hi.z)) <= r2;
      if (!__any_sync(0xffffffffu, need)) continue;
      if (lvl == 0) {
        const int ps = node * LEAF + lane;
        const double cx = xs[ps], cy = ys[ps], cz = zs[ps];
        const uint32_t ci = ps < n ? order[ps] : 0xffffffffu;
#pragma unroll 4
        for (int k = 0; k < LEAF; ++k) {
          const double px = __shfl_sync(0xffffffffu, cx, k), py = __shfl_sync(0xffffffffu, cy, k), pz = __shfl_sync(0xffffffffu, cz, k);
          const uint32_t pi = __shfl_sync(0xffffffffu, ci, k);
          if (need && pi < qidx && sq3(__dsub_rn(px, qx), __dsub_rn(py, qy), __dsub_rn(pz, qz)) <= r2) {
            if (EMIT) nbr[(size_t)base + c] = pi;
            ++c;
          }
        }
        continue;
      }
      const int ch = node * LEAF + lane;
      bool push = false;
      if (ch < s_count[lvl - 1]) {
        const double4* cbx = boxes + 2 * (s_offset[lvl - 1] + ch);
        const double4 clo = cbx[0], chi = cbx[1];
        push = sq3(gap(qlx, qhx, clo.x, chi.x), gap(qly, qhy, clo.y, chi.y), gap(qlz, qhz, clo.z, chi.z)) <= r2;
      }
      const uint32_t mask = __ballot_sync(0xffffffffu, push);
      __syncwarp();
      if (push) stack[sp + __popc(mask & ((1u << lane) - 1u))] = ((uint32_t)(lvl - 1) << LEVEL_SHIFT) | (uint32_t)ch;
      sp += __popc(mask);
      __syncwarp();
    }
  }
  if (!EMIT) {
    if (valid) cnt[qidx] = c;
    const unsigned long long t = warp_sum_u64(c);
    if (lane == 0 && t) atomicAdd(&hd->pairs64, t);
  }
}

// states: 0 undecided, 1 kept, 2 removed.  One round: a point with a kept earlier neighbour is removed, one whose earlier
// neighbours are all removed is kept.  Reads `in` only, so the result of a round does not depend on scheduling.
__global__ void __launch_bounds__(THREADS) k_round(size_t n, const uint32_t* __restrict__ off, const uint32_t* __restrict__ cnt,
                                                   const uint32_t* __restrict__ nbr, const uint8_t* __restrict__ in,
                                                   uint8_t* __restrict__ out, uint32_t* __restrict__ undecided) {
  const size_t i = (size_t)blockIdx.x * THREADS + threadIdx.x;
  uint8_t s = 1;
  if (i < n) {
    s = in[i];
    if (s == 0) {
      bool open = false, hit = false;
      const size_t b = off[i], e = b + cnt[i];
      for (size_t k = b; k < e; ++k) {
        const uint8_t t = in[nbr[k]];
        if (t == 1) { hit = true; break; }
        open |= t == 0;
      }
      s = hit ? 2 : (open ? 0 : 1);
    }
    out[i] = s;
  }
  const uint32_t u = __popc(__ballot_sync(0xffffffffu, s == 0));
  if ((threadIdx.x & 31) == 0 && u) atomicAdd(undecided, u);
}

__global__ void __launch_bounds__(THREADS) k_kept(size_t n, const uint8_t* __restrict__ state, uint8_t* __restrict__ kept) {
  const size_t i = (size_t)blockIdx.x * THREADS + threadIdx.x;
  if (i < n) kept[i] = state[i] == 1;
}

struct DownLayout { size_t header, pts, cnt, off, scan_tmp, sa, sb, bytes; gof_tree::Layout t; };
DownLayout down_layout(int n) {
  DownLayout L; size_t o = 0;
  auto take = layout_taker(o);
  L.header = take(sizeof(DownHeader));
  L.pts = take((size_t)n * 24);
  L.cnt = take((size_t)n * 4); L.off = take((size_t)n * 4);
  L.scan_tmp = take(gof_scan_scratch_bytes((size_t)n));
  L.sa = take((size_t)n); L.sb = take((size_t)n);
  L.t = gof_tree::tree_layout<double>(n, take);
  L.bytes = o;
  return L;
}

// ---- nearest-neighbour distances --------------------------------------------------------------------------------

// One warp per 32 Morton-sorted queries (sorted slot s -> query order[s]); best = the smallest squared distance to any point of
// the reference tree.  INDEXED: the search starts from best = r2 and accepts a point only below it, ids[slot] is the original
// index of the tree point at a slot, and among points at the same smallest distance the lowest original index wins; nodes and
// children are entered while their bound is <= best (not <), so a tied point is never pruned.  out = best (INFINITY when no
// point lies below r2) and out_idx = its index or -1.
template <bool INDEXED>
__global__ void __launch_bounds__(SEARCH_WARPS * 32) k_nn_search(int nq, gof_tree::Tree tree, const double* __restrict__ xs,
                                                                 const double* __restrict__ ys, const double* __restrict__ zs,
                                                                 const double4* __restrict__ boxes, const double* __restrict__ qxs,
                                                                 const double* __restrict__ qys, const double* __restrict__ qzs,
                                                                 const uint32_t* __restrict__ qorder, int take_sqrt, double* __restrict__ out,
                                                                 int n_ref, const uint32_t* __restrict__ ids, double r2,
                                                                 int32_t* __restrict__ out_idx) {
  __shared__ uint32_t s_stack[SEARCH_WARPS][STACK];
  __shared__ int s_count[MAX_LEVELS];
  __shared__ long long s_offset[MAX_LEVELS];
  if (threadIdx.x == 0) {
#pragma unroll
    for (int l = 0; l < MAX_LEVELS; ++l) { s_count[l] = tree.count[l]; s_offset[l] = tree.offset[l]; }
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int group = blockIdx.x * SEARCH_WARPS + warp;
  if ((long long)group * LEAF >= nq) return;
  uint32_t* stack = s_stack[warp];
  const int self = group * LEAF + lane;
  const double qx = qxs[self], qy = qys[self], qz = qzs[self];
  const bool valid = self < nq && finite3(qx, qy, qz);
  double best = INDEXED ? r2 : INFINITY;
  int bi = -1;
  const double inf = INFINITY;
  const double qlx = warp_vmin(valid ? qx : inf), qly = warp_vmin(valid ? qy : inf), qlz = warp_vmin(valid ? qz : inf);
  const double qhx = warp_vmax(valid ? qx : -inf), qhy = warp_vmax(valid ? qy : -inf), qhz = warp_vmax(valid ? qz : -inf);
  if (lane == 0) stack[0] = (uint32_t)(tree.levels - 1) << LEVEL_SHIFT;
  int sp = 1;
  __syncwarp();
  while (sp > 0) {
    const uint32_t e = stack[--sp];
    const int lvl = (int)(e >> LEVEL_SHIFT), node = (int)(e & ((1u << LEVEL_SHIFT) - 1));
    const double4* nb = boxes + 2 * (s_offset[lvl] + node);
    const double4 lo = nb[0], hi = nb[1];
    const double bound = sq3(gap(qx, qx, lo.x, hi.x), gap(qy, qy, lo.y, hi.y), gap(qz, qz, lo.z, hi.z));
    const bool need = valid && (INDEXED ? bound <= best : bound < best);
    if (!__any_sync(0xffffffffu, need)) continue;
    if (lvl == 0) {
      const size_t ps = (size_t)node * LEAF + lane;
      const double cx = xs[ps], cy = ys[ps], cz = zs[ps];
      const int ci = INDEXED && (long long)ps < n_ref ? (int)ids[ps] : 0;
#pragma unroll 4
      for (int k = 0; k < LEAF; ++k) {
        const double px = __shfl_sync(0xffffffffu, cx, k), py = __shfl_sync(0xffffffffu, cy, k), pz = __shfl_sync(0xffffffffu, cz, k);
        const double d = sq3(__dsub_rn(px, qx), __dsub_rn(py, qy), __dsub_rn(pz, qz));
        if (INDEXED) {
          const int pi = __shfl_sync(0xffffffffu, ci, k);
          if (d < best || (d == best && bi >= 0 && pi < bi)) { best = d; bi = pi; }   // NaN padding never enters
        } else if (d < best) {
          best = d;                            // NaN padding never enters
        }
      }
      continue;
    }
    // children: one per lane, pushed farthest first so that the nearest is popped next
    const double thr = warp_vmax(valid ? best : 0.0);
    const int c = node * LEAF + lane;
    double cb = INFINITY;
    const bool exists = c < s_count[lvl - 1];
    if (exists) {
      const double4* cbx = boxes + 2 * (s_offset[lvl - 1] + c);
      const double4 clo = cbx[0], chi = cbx[1];
      cb = sq3(gap(qlx, qhx, clo.x, chi.x), gap(qly, qhy, clo.y, chi.y), gap(qlz, qhz, clo.z, chi.z));
    }
    // INDEXED with r2 = inf: thr may be inf, so a missing child (cb = inf) must be excluded explicitly
    const bool push = INDEXED ? exists && cb <= thr : cb < thr;
    const uint32_t mask = __ballot_sync(0xffffffffu, push);
    int rank = 0;
#pragma unroll 8
    for (int k = 0; k < 32; ++k) {
      const double o = __shfl_sync(0xffffffffu, cb, k);
      rank += ((mask >> k) & 1u) && (o < cb || (o == cb && k < lane));
    }
    const int n = __popc(mask);
    __syncwarp();
    if (push) stack[sp + n - 1 - rank] = ((uint32_t)(lvl - 1) << LEVEL_SHIFT) | (uint32_t)c;
    sp += n;
    __syncwarp();
  }
  if (self < nq) {
    if (INDEXED) {
      out[qorder[self]] = bi >= 0 ? best : INFINITY;
      out_idx[qorder[self]] = bi;
    } else {
      out[qorder[self]] = take_sqrt ? __dsqrt_rn(best) : best;
    }
  }
}

// The queries' half of a 1-NN search: keys, sort buffers and the gathered planes padded to whole groups of 32
struct QueryLayout { size_t qhi1, qhi2, qka, qkb, qva, qvb, qhist, qxs, qys, qzs; };
template <class Take>
QueryLayout query_layout(int n_query, Take&& take) {
  QueryLayout L;
  const size_t q = (size_t)n_query, padded = (q + LEAF - 1) / LEAF * LEAF;
  L.qhi1 = take(q * 4); L.qhi2 = take(q * 4);
  L.qka = take(q * 4); L.qkb = take(q * 4); L.qva = take(q * 4); L.qvb = take(q * 4);
  L.qhist = take(gof_sort_scratch_bytes(q));
  L.qxs = take(padded * 8); L.qys = take(padded * 8); L.qzs = take(padded * 8);
  return L;
}

struct NnLayout { gof_tree::Layout t; QueryLayout q; size_t bytes; };
NnLayout nn_layout(int n_ref, int n_query) {
  NnLayout L; size_t o = 0;
  auto take = layout_taker(o);
  L.t = gof_tree::tree_layout<double>(n_ref, take);
  L.q = query_layout(n_query, take);
  L.bytes = o;
  return L;
}

// A query scratch of gof_nn_query is stamped after its queries are sorted, so that a later call may reuse the order; the stamp
// names the query count, and an order is only a permutation of 0 .. nq-1 when the stamp says nq.
__host__ __device__ constexpr unsigned long long order_stamp(int nq) { return 0x6e6e5f6f72646572ull ^ (unsigned long long)nq; }

__global__ void k_order_stamp(unsigned long long* stamp, int nq) { *stamp = order_stamp(nq); }

// Before an order is reused: if the scratch holds no order for nq queries (fresh, or sorted for another count), the identity
// order is used instead.  The order changes the speed of the search only, never its results.
__global__ void __launch_bounds__(THREADS) k_order_guard(int nq, const unsigned long long* __restrict__ stamp, uint32_t* __restrict__ va) {
  const int s = blockIdx.x * THREADS + threadIdx.x;
  if (s < nq && *stamp != order_stamp(nq)) va[s] = (uint32_t)s;
}

// The queries against a built tree: keyed against the tree's box (clamped), sorted unless `sort` is false (then the order left
// in the query scratch by an earlier call with the same n_query is reused, checked against `stamp`), gathered and searched.
// stamp: NULL (gof_nn_dist, always sorting) or the query scratch's stamp word.  No host synchronisation.
template <bool INDEXED>
int nn_query(int n_ref, const gof_tree::Bufs<double>& b, int nq, const double* query, char* S, const QueryLayout& L, bool sort,
             unsigned long long* stamp, int take_sqrt, double* out, double r2, int32_t* out_idx, cudaStream_t st) {
  int rc;
  const gof_tree::Tree tree = gof_tree::make_tree(n_ref);
  const int padded = (nq + LEAF - 1) / LEAF * LEAF;
  uint32_t *hi1 = (uint32_t*)(S + L.qhi1), *hi2 = (uint32_t*)(S + L.qhi2), *ka = (uint32_t*)(S + L.qka), *kb = (uint32_t*)(S + L.qkb);
  uint32_t *va = (uint32_t*)(S + L.qva), *vb = (uint32_t*)(S + L.qvb), *hist = (uint32_t*)(S + L.qhist);
  double *qxs = (double*)(S + L.qxs), *qys = (double*)(S + L.qys), *qzs = (double*)(S + L.qzs);
  if (sort) {
    GOF_LAUNCH("dtu_query_keys", st, gof_tree::k_tree_keys<double><<<blocks_for((size_t)nq, THREADS), THREADS, 0, st>>>(nq, query, b.bbox,
                                                                                                                       ka, hi1, hi2));
    GOF_LAUNCH_CHECK(false, st);
    const GofKeyWords key{{ka, hi1, hi2}, {32, 32, 32}, 3};
    if ((rc = gof_sort_words_u32(key, (size_t)nq, GofSortBufs{ka, kb, va, vb, hist}, va, false, st)) != GOF_OK) return rc;
    if (stamp) {
      GOF_LAUNCH("dtu_order_stamp", st, k_order_stamp<<<1, 1, 0, st>>>(stamp, nq));
      GOF_LAUNCH_CHECK(false, st);
    }
  } else {
    GOF_LAUNCH("dtu_order_guard", st, k_order_guard<<<blocks_for((size_t)nq, THREADS), THREADS, 0, st>>>(nq, stamp, va));
    GOF_LAUNCH_CHECK(false, st);
  }
  GOF_LAUNCH("dtu_query_gather", st, gof_tree::k_tree_gather<double><<<blocks_for((size_t)padded, THREADS), THREADS, 0, st>>>(
                                         nq, padded, query, va, qxs, qys, qzs));
  GOF_LAUNCH_CHECK(false, st);
  GOF_LAUNCH("dtu_nn_search", st, k_nn_search<INDEXED><<<blocks_for((size_t)padded / LEAF, SEARCH_WARPS), SEARCH_WARPS * 32, 0, st>>>(
                                      nq, tree, b.xs, b.ys, b.zs, b.boxes, qxs, qys, qzs, va, take_sqrt, out, n_ref, b.va, r2, out_idx));
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}

int check_count(int64_t n, const char* what, const char* fn) {
  if (n < 0) { gof_set_error("%s: %s = %lld < 0", fn, what, (long long)n); return GOF_E_INVALID; }
  if ((uint64_t)n >= SORT_LIMIT) {
    gof_set_error("%s: %lld %s; at most 2^30 - 1 are supported (the limit of the library's radix sort)", fn, (long long)n, what);
    return GOF_E_INVALID;
  }
  return GOF_OK;
}

}  // namespace

// ---- C ABI -------------------------------------------------------------------------------------------------------

extern "C" GOF_API size_t gof_mesh_sample_scratch_bytes(int64_t num_faces) {
  return num_faces <= 0 ? 0 : face_layout((size_t)num_faces).bytes;
}

extern "C" GOF_API int gof_mesh_sample_count(int64_t num_vertices, const double* vertices, int64_t num_faces, const int64_t* faces,
                                             double density, void* scratch, size_t scratch_bytes, gof_alloc_fn row_alloc,
                                             void* row_user, int64_t* num_samples_out, void* stream) {
  if (!num_samples_out || !row_alloc) { gof_set_error("mesh_sample_count: NULL argument"); return GOF_E_INVALID; }
  *num_samples_out = 0;
  int rc;
  if ((rc = check_count(num_vertices, "vertices", "mesh_sample_count")) != GOF_OK) return rc;
  if (num_faces < 0 || num_faces >= ((int64_t)1 << 31)) { gof_set_error("mesh_sample_count: %lld faces", (long long)num_faces); return GOF_E_INVALID; }
  if (!(density > 0.0) || !isfinite(density)) { gof_set_error("mesh_sample_count: density %g must be positive and finite", density); return GOF_E_INVALID; }
  if (num_faces == 0) return GOF_OK;
  if (!vertices || !faces || !scratch) { gof_set_error("mesh_sample_count: NULL input"); return GOF_E_INVALID; }
  const size_t nf = (size_t)num_faces;
  const FaceLayout L = face_layout(nf);
  if (scratch_bytes < L.bytes) {
    gof_set_error("mesh_sample_count: scratch of %zu bytes, %zu needed (gof_mesh_sample_scratch_bytes)", scratch_bytes, L.bytes);
    return GOF_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  char* S = static_cast<char*>(scratch);
  FaceHeader* fh = (FaceHeader*)(S + L.header);
  uint32_t *rows = (uint32_t*)(S + L.rows), *row_start = (uint32_t*)(S + L.row_start), *tmp = (uint32_t*)(S + L.scan_tmp);
  GOF_CUDA_OK(cudaMemsetAsync(fh, 0, sizeof(FaceHeader), st));
  GOF_LAUNCH("dtu_face_rows", st, k_face_rows<<<blocks_for(nf, THREADS), THREADS, 0, st>>>((size_t)num_vertices, vertices, nf, faces,
                                                                                           density, rows, fh));
  GOF_LAUNCH_CHECK(false, st);
  if ((rc = gof_exclusive_scan_u32(rows, row_start, tmp, &fh->rows32, nf, false, st)) != GOF_OK) return rc;
  FaceHeader h;
  if ((rc = gof_read_back(&h, fh, sizeof(h), st)) != GOF_OK) return rc;
  if (h.err & 1u) { gof_set_error("mesh_sample_count: a face index is outside [0, %lld)", (long long)num_vertices); return GOF_E_INVALID; }
  if (h.err) { gof_set_error("mesh_sample_count: a face spans 2^31 or more samples per edge at density %g", density); return GOF_E_INVALID; }
  if (h.rows64 >= (1ull << 32)) { gof_set_error("mesh_sample_count: %llu sample rows; at most 2^32 - 1 are supported", h.rows64); return GOF_E_INVALID; }
  const size_t R = (size_t)h.rows64;
  const RowLayout RL = row_layout(R);
  char* RS = (char*)row_alloc(row_user, RL.bytes);
  if (!RS) { gof_set_error("scratch allocator returned NULL"); return GOF_E_ALLOC; }
  RowHeader* rh = (RowHeader*)(RS + RL.header);
  GOF_CUDA_OK(cudaMemsetAsync(rh, 0, sizeof(RowHeader), st));
  RowHeader r{};
  if (R) {
    uint32_t *cnt = (uint32_t*)(RS + RL.cnt), *off = (uint32_t*)(RS + RL.off), *rtmp = (uint32_t*)(RS + RL.scan_tmp);
    GOF_LAUNCH("dtu_row_count", st, k_row_count<<<blocks_for(R, THREADS), THREADS, 0, st>>>(R, vertices, nf, faces, density, row_start,
                                                                                           cnt, rh));
    GOF_LAUNCH_CHECK(false, st);
    if ((rc = gof_exclusive_scan_u32(cnt, off, rtmp, &rh->samples32, R, false, st)) != GOF_OK) return rc;
    if ((rc = gof_read_back(&r, rh, sizeof(r), st)) != GOF_OK) return rc;
  }
  if (r.samples64 + (unsigned long long)num_vertices >= SORT_LIMIT) {
    gof_set_error("mesh_sample_count: %lld vertices + %llu samples; at most 2^30 - 1 points are supported (the limit of the "
                  "library's radix sort)", (long long)num_vertices, r.samples64);
    return GOF_E_INVALID;
  }
  r.rows = R;
  GOF_CUDA_OK(cudaMemcpyAsync(rh, &r, sizeof(r), cudaMemcpyHostToDevice, st));
  GOF_CUDA_OK(cudaStreamSynchronize(st));      // r lives on this frame
  *num_samples_out = (int64_t)r.samples64;
  return GOF_OK;
}

extern "C" GOF_API int gof_mesh_sample_emit(int64_t num_vertices, const double* vertices, int64_t num_faces, const int64_t* faces,
                                            double density, const void* scratch, const void* row_scratch, int64_t num_samples,
                                            double* out, void* stream) {
  if (num_vertices < 0 || num_faces < 0 || num_samples < 0) { gof_set_error("mesh_sample_emit: negative size"); return GOF_E_INVALID; }
  if (num_vertices + num_samples == 0) return GOF_OK;
  if (!out || (num_vertices && !vertices)) { gof_set_error("mesh_sample_emit: NULL argument"); return GOF_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if (num_vertices) GOF_CUDA_OK(cudaMemcpyAsync(out, vertices, (size_t)num_vertices * 24, cudaMemcpyDeviceToDevice, st));
  if (num_samples == 0) return GOF_OK;
  if (!faces || !scratch || !row_scratch) { gof_set_error("mesh_sample_emit: NULL scratch"); return GOF_E_INVALID; }
  const size_t nf = (size_t)num_faces;
  const FaceLayout L = face_layout(nf);
  RowHeader r;
  if ((rc = gof_read_back(&r, (const char*)row_scratch, sizeof(r), st)) != GOF_OK) return rc;
  if ((int64_t)r.samples64 != num_samples) { gof_set_error("mesh_sample_emit: size does not match the count phase"); return GOF_E_INVALID; }
  const RowLayout RL = row_layout((size_t)r.rows);
  const uint32_t* row_start = (const uint32_t*)((const char*)scratch + L.row_start);
  const uint32_t* off = (const uint32_t*)((const char*)row_scratch + RL.off);
  const size_t S = (size_t)num_samples;
  GOF_LAUNCH("dtu_sample_emit", st, k_sample_emit<<<blocks_for(S, THREADS), THREADS, 0, st>>>(S, (size_t)r.rows, vertices, nf, faces,
                                                                                             density, row_start, off,
                                                                                             out + 3 * (size_t)num_vertices));
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}

extern "C" GOF_API size_t gof_ordered_downsample_scratch_bytes(int64_t n) {
  return (n <= 0 || (uint64_t)n >= SORT_LIMIT) ? 0 : down_layout((int)n).bytes;
}

extern "C" GOF_API int gof_ordered_downsample(int64_t n, const double* points, const uint32_t* perm, double radius, uint8_t* kept,
                                              int64_t* num_rounds_out, int64_t* num_pairs_out, void* scratch, size_t scratch_bytes,
                                              gof_alloc_fn pair_alloc, void* pair_user, void* stream) {
  if (!num_rounds_out || !pair_alloc) { gof_set_error("ordered_downsample: NULL argument"); return GOF_E_INVALID; }
  *num_rounds_out = 0;
  if (num_pairs_out) *num_pairs_out = 0;
  int rc;
  if ((rc = check_count(n, "points", "ordered_downsample")) != GOF_OK) return rc;
  if (!(radius >= 0.0) || !isfinite(radius)) { gof_set_error("ordered_downsample: radius %g must be finite and >= 0", radius); return GOF_E_INVALID; }
  if (n == 0) return GOF_OK;
  if (!points || !perm || !kept || !scratch) { gof_set_error("ordered_downsample: NULL input"); return GOF_E_INVALID; }
  const DownLayout L = down_layout((int)n);
  if (scratch_bytes < L.bytes) {
    gof_set_error("ordered_downsample: scratch of %zu bytes, %zu needed (gof_ordered_downsample_scratch_bytes)", scratch_bytes, L.bytes);
    return GOF_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const size_t N = (size_t)n;
  char* S = static_cast<char*>(scratch);
  DownHeader* hd = (DownHeader*)(S + L.header);
  double* pts = (double*)(S + L.pts);
  uint32_t *cnt = (uint32_t*)(S + L.cnt), *off = (uint32_t*)(S + L.off), *tmp = (uint32_t*)(S + L.scan_tmp);
  uint8_t *sa = (uint8_t*)(S + L.sa), *sb = (uint8_t*)(S + L.sb);
  const gof_tree::Bufs<double> b = gof_tree::carve<double>(S, L.t);
  const gof_tree::Tree tree = gof_tree::make_tree((int)n);
  const double r2 = radius * radius;
  const int gn = blocks_for(N, THREADS);

  GOF_CUDA_OK(cudaMemsetAsync(hd, 0, sizeof(DownHeader), st));
  GOF_CUDA_OK(cudaMemsetAsync(cnt, 0, N * 4, st));
  GOF_LAUNCH("dtu_perm_gather", st, k_perm_gather<<<gn, THREADS, 0, st>>>(N, points, perm, pts, cnt, hd));
  GOF_LAUNCH_CHECK(false, st);
  GOF_LAUNCH("dtu_perm_check", st, k_perm_check<<<gn, THREADS, 0, st>>>(N, cnt, hd));
  GOF_LAUNCH_CHECK(false, st);
  if ((rc = gof_tree::build_tree<double>((int)n, pts, b, tree, st)) != GOF_OK) return rc;
  const int gs = blocks_for((size_t)tree.count[0], SEARCH_WARPS);
  GOF_LAUNCH("dtu_radius_count", st, k_radius_pairs<false><<<gs, SEARCH_WARPS * 32, 0, st>>>((int)n, tree, b.xs, b.ys, b.zs, b.va, b.boxes,
                                                                                           r2, cnt, nullptr, nullptr, hd));
  GOF_LAUNCH_CHECK(false, st);
  if ((rc = gof_exclusive_scan_u32(cnt, off, tmp, &hd->pairs32, N, false, st)) != GOF_OK) return rc;
  DownHeader h;
  if ((rc = gof_read_back(&h, hd, sizeof(h), st)) != GOF_OK) return rc;
  if (h.err) { gof_set_error("ordered_downsample: perm is not a permutation of 0 .. %lld", (long long)n - 1); return GOF_E_INVALID; }
  if (h.pairs64 > 0xffffffffull) {
    gof_set_error("ordered_downsample: %llu neighbour pairs within the radius; at most 2^32 - 1 are supported", h.pairs64);
    return GOF_E_INVALID;
  }
  if (num_pairs_out) *num_pairs_out = (int64_t)h.pairs64;
  uint32_t* nbr = nullptr;
  if (h.pairs64) {
    nbr = (uint32_t*)pair_alloc(pair_user, (size_t)h.pairs64 * 4);
    if (!nbr) { gof_set_error("scratch allocator returned NULL"); return GOF_E_ALLOC; }
    GOF_LAUNCH("dtu_radius_emit", st, k_radius_pairs<true><<<gs, SEARCH_WARPS * 32, 0, st>>>((int)n, tree, b.xs, b.ys, b.zs, b.va, b.boxes,
                                                                                            r2, nullptr, off, nbr, hd));
    GOF_LAUNCH_CHECK(false, st);
  }
  GOF_CUDA_OK(cudaMemsetAsync(sa, 0, N, st));
  // rounds in batches: undecided[k] counts the points still open after round k of the batch; a finished batch runs no-op rounds
  int64_t rounds = 0;
  uint8_t *in = sa, *out = sb;
  while (true) {
    GOF_CUDA_OK(cudaMemsetAsync(hd->undecided, 0, sizeof(hd->undecided), st));
    for (int k = 0; k < ROUND_BATCH; ++k) {
      GOF_LAUNCH("dtu_round", st, k_round<<<gn, THREADS, 0, st>>>(N, off, cnt, nbr, in, out, hd->undecided + k));
      GOF_LAUNCH_CHECK(false, st);
      uint8_t* t = in; in = out; out = t;
    }
    uint32_t u[ROUND_BATCH];
    if ((rc = gof_read_back(u, hd->undecided, sizeof(u), st)) != GOF_OK) return rc;
    int k = 0;
    while (k < ROUND_BATCH && u[k] != 0) ++k;
    if (k < ROUND_BATCH) { rounds += k + 1; break; }
    rounds += ROUND_BATCH;
  }
  GOF_LAUNCH("dtu_kept", st, k_kept<<<gn, THREADS, 0, st>>>(N, in, kept));
  GOF_LAUNCH_CHECK(false, st);
  *num_rounds_out = rounds;
  return GOF_OK;
}

extern "C" GOF_API size_t gof_nn_dist_scratch_bytes(int64_t n_ref, int64_t n_query) {
  if (n_ref <= 0 || n_query <= 0 || (uint64_t)n_ref >= SORT_LIMIT || (uint64_t)n_query >= SORT_LIMIT) return 0;
  return nn_layout((int)n_ref, (int)n_query).bytes;
}

extern "C" GOF_API int gof_nn_dist(int64_t n_ref, const double* ref, int64_t n_query, const double* query, double* out, int take_sqrt,
                                   void* scratch, size_t scratch_bytes, void* stream) {
  int rc;
  if ((rc = check_count(n_ref, "reference points", "nn_dist")) != GOF_OK) return rc;
  if ((rc = check_count(n_query, "query points", "nn_dist")) != GOF_OK) return rc;
  if (n_query == 0) return GOF_OK;
  if (n_ref == 0) { gof_set_error("nn_dist: no reference points for %lld queries", (long long)n_query); return GOF_E_INVALID; }
  if (!ref || !query || !out || !scratch) { gof_set_error("nn_dist: NULL argument"); return GOF_E_INVALID; }
  const NnLayout L = nn_layout((int)n_ref, (int)n_query);
  if (scratch_bytes < L.bytes) {
    gof_set_error("nn_dist: scratch of %zu bytes, %zu needed (gof_nn_dist_scratch_bytes)", scratch_bytes, L.bytes);
    return GOF_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  char* S = static_cast<char*>(scratch);
  const gof_tree::Bufs<double> b = gof_tree::carve<double>(S, L.t);
  const gof_tree::Tree tree = gof_tree::make_tree((int)n_ref);
  if ((rc = gof_tree::build_tree<double>((int)n_ref, ref, b, tree, st)) != GOF_OK) return rc;
  return nn_query<false>((int)n_ref, b, (int)n_query, query, S, L.q, true, nullptr, take_sqrt, out, 0.0, nullptr, st);
}

// ---- the same search split into a persistent tree and repeated queries (Tanks and Temples ICP, DESIGN section 4.7) ----------

namespace {
gof_tree::Layout tree_only_layout(int n_ref, size_t* bytes) {
  size_t o = 0;
  auto take = layout_taker(o);
  const gof_tree::Layout L = gof_tree::tree_layout<double>(n_ref, take);
  *bytes = o;
  return L;
}
// gof_nn_query's scratch: the order stamp, then the queries' buffers
QueryLayout query_only_layout(int n_query, size_t* stamp, size_t* bytes) {
  size_t o = 0;
  auto take = layout_taker(o);
  *stamp = take(8);
  const QueryLayout L = query_layout(n_query, take);
  *bytes = o;
  return L;
}
}  // namespace

extern "C" GOF_API size_t gof_nn_tree_scratch_bytes(int64_t n_ref) {
  if (n_ref <= 0 || (uint64_t)n_ref >= SORT_LIMIT) return 0;
  size_t bytes;
  tree_only_layout((int)n_ref, &bytes);
  return bytes;
}

extern "C" GOF_API int gof_nn_tree_build(int64_t n_ref, const double* ref, void* tree_scratch, size_t scratch_bytes, void* stream) {
  int rc;
  if ((rc = check_count(n_ref, "reference points", "nn_tree_build")) != GOF_OK) return rc;
  if (n_ref == 0) { gof_set_error("nn_tree_build: no reference points"); return GOF_E_INVALID; }
  if (!ref || !tree_scratch) { gof_set_error("nn_tree_build: NULL argument"); return GOF_E_INVALID; }
  size_t need;
  const gof_tree::Layout L = tree_only_layout((int)n_ref, &need);
  if (scratch_bytes < need) {
    gof_set_error("nn_tree_build: scratch of %zu bytes, %zu needed (gof_nn_tree_scratch_bytes)", scratch_bytes, need);
    return GOF_E_INVALID;
  }
  const gof_tree::Bufs<double> b = gof_tree::carve<double>(static_cast<char*>(tree_scratch), L);
  return gof_tree::build_tree<double>((int)n_ref, ref, b, gof_tree::make_tree((int)n_ref), (cudaStream_t)stream);
}

extern "C" GOF_API size_t gof_nn_query_scratch_bytes(int64_t n_query) {
  if (n_query <= 0 || (uint64_t)n_query >= SORT_LIMIT) return 0;
  size_t stamp, bytes;
  query_only_layout((int)n_query, &stamp, &bytes);
  return bytes;
}

extern "C" GOF_API int gof_nn_query(int64_t n_ref, void* tree_scratch, size_t tree_scratch_bytes, int64_t n_query, const double* query,
                                    double r2, int reuse_order, int32_t* out_index, double* out_d2, void* query_scratch,
                                    size_t scratch_bytes, void* stream) {
  int rc;
  if ((rc = check_count(n_ref, "reference points", "nn_query")) != GOF_OK) return rc;
  if ((rc = check_count(n_query, "query points", "nn_query")) != GOF_OK) return rc;
  if (!(r2 >= 0.0)) { gof_set_error("nn_query: r2 = %g must be >= 0", r2); return GOF_E_INVALID; }
  if (n_query == 0) return GOF_OK;
  if (n_ref == 0) { gof_set_error("nn_query: no reference points for %lld queries", (long long)n_query); return GOF_E_INVALID; }
  if (!tree_scratch || !query || !out_index || !out_d2 || !query_scratch) { gof_set_error("nn_query: NULL argument"); return GOF_E_INVALID; }
  size_t tree_need;
  const gof_tree::Layout TL = tree_only_layout((int)n_ref, &tree_need);
  if (tree_scratch_bytes < tree_need) {
    gof_set_error("nn_query: tree scratch of %zu bytes, %zu needed for %lld reference points (gof_nn_tree_scratch_bytes)",
                  tree_scratch_bytes, tree_need, (long long)n_ref);
    return GOF_E_INVALID;
  }
  size_t stamp, need;
  const QueryLayout L = query_only_layout((int)n_query, &stamp, &need);
  if (scratch_bytes < need) {
    gof_set_error("nn_query: scratch of %zu bytes, %zu needed (gof_nn_query_scratch_bytes)", scratch_bytes, need);
    return GOF_E_INVALID;
  }
  char* QS = static_cast<char*>(query_scratch);
  const gof_tree::Bufs<double> b = gof_tree::carve<double>(static_cast<char*>(tree_scratch), TL);
  return nn_query<true>((int)n_ref, b, (int)n_query, query, QS, L, reuse_order == 0, (unsigned long long*)(QS + stamp), 0, out_d2, r2,
                        out_index, (cudaStream_t)stream);
}
