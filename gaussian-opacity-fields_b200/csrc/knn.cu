// knn.cu -- mean squared distance to the three nearest neighbours of every point: simple_knn's distCUDA2
// (submodules/simple-knn/spatial.cu:15-25, simple_knn.cu:147-183), which GaussianModel.create_from_pcd uses to initialise
// the scales.  The contract is DESIGN section 4.5: out_i = ((b0 + b1) + b2) / 3 over the three smallest accepted
// d(i,j) = fmaf(dz, dz, fmaf(dx, dx, dy*dy)), j != i by index, accepted iff d < FLT_MAX, padded with FLT_MAX.  Every float
// step below is one explicit IEEE operation, so the result is bit-identical to the reference whatever order the search
// takes (the reference's own pruning is exact, so its output does not depend on its search order either).
//
//   tree     the Morton-ordered 32-ary box tree of knn_tree.cuh over the float points
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

#include "knn_tree.cuh"

namespace {

using gof_tree::LEAF;
using gof_tree::LEVEL_SHIFT;
using gof_tree::MAX_LEVELS;
using gof_tree::finite3;
using gof_tree::warp_vmax;
using gof_tree::warp_vmin;
using KnnTree = gof_tree::Tree;

constexpr int SEARCH_WARPS = 4;              // warps per CTA of the search kernel
constexpr int STACK = 256;                   // per warp; a walk holds at most 31 entries per level + 1

struct KnnLayout { gof_tree::Layout t; size_t bytes; };

KnnLayout knn_layout(int P) {
  KnnLayout L; size_t o = 0;
  auto take = [&](size_t b) { size_t r = o; o = gof_align_up(o + b, 256); return r; };
  L.t = gof_tree::tree_layout<float>(P, take);
  L.bytes = o;
  return L;
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
    const float qlx = warp_vmin(valid ? qx : INFINITY), qly = warp_vmin(valid ? qy : INFINITY), qlz = warp_vmin(valid ? qz : INFINITY);
    const float qhx = warp_vmax(valid ? qx : -INFINITY), qhy = warp_vmax(valid ? qy : -INFINITY), qhz = warp_vmax(valid ? qz : -INFINITY);
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
  const KnnTree tree = gof_tree::make_tree(P);
  cudaStream_t st = (cudaStream_t)stream;
  const gof_tree::Bufs<float> b = gof_tree::carve<float>(static_cast<char*>(scratch), L.t);
  int rc;
  if ((rc = gof_tree::build_tree<float>(P, points, b, tree, st)) != GOF_OK) return rc;
  GOF_LAUNCH("knn_search", st, k_knn_search<<<gof_tree::blocks_for((size_t)tree.count[0], SEARCH_WARPS), SEARCH_WARPS * 32, 0, st>>>(
                                   P, tree, b.xs, b.ys, b.zs, b.va, b.boxes, mean_dists));
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}
