// tnt_eval.cu -- the point-cloud steps of the Tanks and Temples evaluation (eval_tnt/run.py, DESIGN section 4.7) on the GPU:
// transform + polygon-volume crop, Open3D's voxel down-sample, the moments of a point-to-point ICP update and the in-place
// transform of the moving cloud.  The 1-NN search with index and radius is gof_nn_tree_build / gof_nn_query in dtu_eval.cu.
// Coordinates are double; every arithmetic step the specification fixes is one IEEE double operation written out, so a numpy
// restatement of the same steps reproduces each value bit for bit.
//
//   transform  ((m00*x + m01*y) + m02*z) + m03 per row, then each of the three divided by the fourth row's value w
//   crop       w = the orthogonal axis, (u, v) the other two ascending.  Dropped if p_w < axis_min or p_w > axis_max; else the
//              edges (a, b) of the polygon with (a_v < p_v && b_v >= p_v) || (b_v < p_v && a_v >= p_v) give the nodes
//              a_u + ((p_v - a_v) / (b_v - a_v)) * (b_u - a_u), and the point is kept iff an odd number of them are < p_u.
//              Flags, a scan, then a stable scatter: the kept points stay in input order.
//   voxel      lo = min - voxel*0.5 per axis (exact min by ordered-integer atomics); key = int(floor((p - lo) / voxel)); a stable
//              sort by (x, y, z) key keeps each voxel's members in input order; one thread per voxel sums them from the first
//              member on and divides by double(count).  Output in ascending (x, y, z) voxel order.
//   moments    over the pairs (i, idx[i]) with idx[i] >= 0: count, sum d2, sum src, sum tgt (pass 1), then with the means
//              m = sum * (1 / count): sum (t - mt)(s - ms)^T and sum |s - ms|^2 (pass 2).  Each pass reduces fixed chunks of
//              2048 pairs in a fixed order, then the chunk partials in a fixed order, so two runs are bit-identical.
#include <float.h>
#include <limits.h>
#include <math.h>
#include <string.h>

#include "knn_tree.cuh"

namespace {

using gof_tree::THREADS;
using gof_tree::blocks_for;

constexpr size_t SORT_LIMIT = (size_t)1 << 30;   // the radix passes' item limit (DESIGN section 4.4)
constexpr int MAX_POLYGON = 3072;               // polygon vertices (u, v) staged in 48 KB of shared memory
constexpr int CHUNK_ITEMS = 8;                  // pairs per thread of a moments chunk
constexpr int CHUNK = THREADS * CHUNK_ITEMS;    // pairs per moments chunk (one block)
constexpr int M1 = 8;                           // pass-1 sums: count, d2, src xyz, tgt xyz
constexpr int M2 = 10;                          // pass-2 sums: cov 3x3 (row = target axis), src variance

auto layout_taker(size_t& o) {
  return [&o](size_t b) { size_t r = o; o = gof_align_up(o + b, 256); return r; };
}

struct Mat4 { double m[16]; };

__device__ __forceinline__ void transform_point(const Mat4& T, double x, double y, double z, double* o) {
  double r[4];
#pragma unroll
  for (int k = 0; k < 4; ++k)
    r[k] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T.m[4 * k], x), __dmul_rn(T.m[4 * k + 1], y)), __dmul_rn(T.m[4 * k + 2], z)),
                     T.m[4 * k + 3]);
#pragma unroll
  for (int k = 0; k < 3; ++k) o[k] = __ddiv_rn(r[k], r[3]);
}

int check_count(int64_t n, const char* what, const char* fn) {
  if (n < 0) { gof_set_error("%s: %s = %lld < 0", fn, what, (long long)n); return GOF_E_INVALID; }
  if ((uint64_t)n >= SORT_LIMIT) {
    gof_set_error("%s: %lld %s; at most 2^30 - 1 are supported (the limit of the library's radix sort)", fn, (long long)n, what);
    return GOF_E_INVALID;
  }
  return GOF_OK;
}

bool finite16(const double* m) {
  for (int k = 0; k < 16; ++k) if (!isfinite(m[k])) return false;
  return true;
}

// ---- crop -------------------------------------------------------------------------------------------------------

struct CropArgs { Mat4 T; int has_T, w, u, v, nv; double axis_min, axis_max; };

__device__ __forceinline__ void crop_point(const CropArgs& a, const double* __restrict__ pts, size_t i, double* p) {
  const double x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
  if (a.has_T) { transform_point(a.T, x, y, z, p); } else { p[0] = x; p[1] = y; p[2] = z; }
}

__global__ void __launch_bounds__(THREADS) k_crop_flags(size_t n, const double* __restrict__ pts, CropArgs a,
                                                        const double2* __restrict__ poly, uint32_t* __restrict__ flags) {
  extern __shared__ double2 s_poly[];
  for (int k = threadIdx.x; k < a.nv; k += THREADS) s_poly[k] = poly[k];
  __syncthreads();
  const size_t i = (size_t)blockIdx.x * THREADS + threadIdx.x;
  if (i >= n) return;
  double p[3];
  crop_point(a, pts, i, p);
  // selects, not p[a.w]: a dynamic index would put p in a local-memory frame
  const double pw = a.w == 0 ? p[0] : (a.w == 1 ? p[1] : p[2]);
  const double pu = a.u == 0 ? p[0] : p[1];
  const double pv = a.v == 1 ? p[1] : p[2];
  uint32_t keep = 0;
  if (!(pw < a.axis_min || pw > a.axis_max)) {
    uint32_t below = 0;
    double2 A = s_poly[a.nv - 1];
    for (int k = 0; k < a.nv; ++k) {            // edge (k - 1, k) = (i, i + 1 mod n) of the specification, visited from i = n - 1
      const double2 B = s_poly[k];
      if ((A.y < pv && B.y >= pv) || (B.y < pv && A.y >= pv))
        below += __dadd_rn(A.x, __dmul_rn(__ddiv_rn(__dsub_rn(pv, A.y), __dsub_rn(B.y, A.y)), __dsub_rn(B.x, A.x))) < pu;
      A = B;
    }
    keep = below & 1u;
  }
  flags[i] = keep;
}

__global__ void __launch_bounds__(THREADS) k_crop_emit(size_t n, const double* __restrict__ pts, CropArgs a,
                                                       const uint32_t* __restrict__ flags, const uint32_t* __restrict__ off,
                                                       double* __restrict__ out, uint32_t* __restrict__ out_index) {
  const size_t i = (size_t)blockIdx.x * THREADS + threadIdx.x;
  if (i >= n || !flags[i]) return;
  double p[3];
  crop_point(a, pts, i, p);
  const size_t o = off[i];
  out[3 * o] = p[0]; out[3 * o + 1] = p[1]; out[3 * o + 2] = p[2];
  if (out_index) out_index[o] = (uint32_t)i;
}

struct CropLayout { size_t poly, flags, off, scan_tmp, total, bytes; };
CropLayout crop_layout(size_t n) {
  CropLayout L; size_t o = 0;
  auto take = layout_taker(o);
  L.poly = take(MAX_POLYGON * sizeof(double2));
  L.flags = take(n * 4); L.off = take(n * 4); L.scan_tmp = take(gof_scan_scratch_bytes(n)); L.total = take(8);
  L.bytes = o;
  return L;
}

// ---- voxel down-sample --------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(THREADS) k_voxel_keys(size_t n, const double* __restrict__ pts, double lx, double ly, double lz,
                                                        double voxel, uint32_t* __restrict__ kx, uint32_t* __restrict__ ky,
                                                        uint32_t* __restrict__ kz) {
  const size_t i = (size_t)blockIdx.x * THREADS + threadIdx.x;
  if (i >= n) return;
  kx[i] = (uint32_t)(int)floor(__ddiv_rn(__dsub_rn(pts[3 * i], lx), voxel));
  ky[i] = (uint32_t)(int)floor(__ddiv_rn(__dsub_rn(pts[3 * i + 1], ly), voxel));
  kz[i] = (uint32_t)(int)floor(__ddiv_rn(__dsub_rn(pts[3 * i + 2], lz), voxel));
}

// start[run of a head] = its sorted position; start[runs] = n
__global__ void __launch_bounds__(THREADS) k_voxel_starts(size_t n, const uint32_t* __restrict__ head, const uint32_t* __restrict__ run,
                                                          const uint32_t* __restrict__ num_runs, uint32_t* __restrict__ start) {
  const size_t j = (size_t)blockIdx.x * THREADS + threadIdx.x;
  if (j == 0) start[*num_runs] = (uint32_t)n;
  if (j < n && head[j]) start[run[j]] = (uint32_t)j;
}

__global__ void __launch_bounds__(THREADS) k_voxel_mean(size_t voxels, const double* __restrict__ pts, const uint32_t* __restrict__ ord,
                                                        const uint32_t* __restrict__ start, double* __restrict__ out) {
  const size_t v = (size_t)blockIdx.x * THREADS + threadIdx.x;
  if (v >= voxels) return;
  const uint32_t b = start[v], e = start[v + 1];
  const size_t f = ord[b];
  double sx = pts[3 * f], sy = pts[3 * f + 1], sz = pts[3 * f + 2];
  for (uint32_t j = b + 1; j < e; ++j) {
    const size_t p = ord[j];
    sx = __dadd_rn(sx, pts[3 * p]); sy = __dadd_rn(sy, pts[3 * p + 1]); sz = __dadd_rn(sz, pts[3 * p + 2]);
  }
  const double c = (double)(e - b);
  out[3 * v] = __ddiv_rn(sx, c); out[3 * v + 1] = __ddiv_rn(sy, c); out[3 * v + 2] = __ddiv_rn(sz, c);
}

// bad[0] = 1 when some point has a non-finite coordinate
__global__ void __launch_bounds__(THREADS) k_nonfinite(size_t n, const double* __restrict__ pts, unsigned long long* __restrict__ bad) {
  const size_t i = (size_t)blockIdx.x * THREADS + threadIdx.x;
  if (i < n && !gof_tree::finite3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2])) *bad = 1ull;
}

struct VoxelLayout { size_t bbox, kx, ky, kz, ka, kb, va, vb, hist, head, run, scan_tmp, runs, start, bytes; };
VoxelLayout voxel_layout(size_t n) {
  VoxelLayout L; size_t o = 0;
  auto take = layout_taker(o);
  L.bbox = take(7 * 8);                        // ordered min[3], max[3], the non-finite flag
  L.kx = take(n * 4); L.ky = take(n * 4); L.kz = take(n * 4);
  L.ka = take(n * 4); L.kb = take(n * 4); L.va = take(n * 4); L.vb = take(n * 4);
  L.hist = take(gof_sort_scratch_bytes(n));
  L.head = take(n * 4); L.run = take(n * 4); L.scan_tmp = take(gof_scan_scratch_bytes(n)); L.runs = take(8);
  L.start = take((n + 1) * 4);
  L.bytes = o;
  return L;
}

// host image of gof_tree::value_of<double>
double host_value_of(unsigned long long o) {
  const unsigned long long u = (o & 0x8000000000000000ull) ? (o & ~0x8000000000000000ull) : ~o;
  double d;
  memcpy(&d, &u, 8);
  return d;
}

int bit_width(double kmax) {
  int b = 1;
  while (b < 32 && (double)(1ull << b) <= kmax) ++b;
  return b;
}

// ---- ICP moments ----------------------------------------------------------------------------------------------------

// block-wide sum of M values per thread in a fixed tree order; result in s[0..M) of thread 0's row
template <int M>
__device__ __forceinline__ void block_sum(double (&v)[M], double (*s)[M]) {
#pragma unroll
  for (int k = 0; k < M; ++k) s[threadIdx.x][k] = v[k];
  __syncthreads();
  for (int h = THREADS / 2; h >= 1; h >>= 1) {
    if ((int)threadIdx.x < h) {
#pragma unroll
      for (int k = 0; k < M; ++k) s[threadIdx.x][k] = __dadd_rn(s[threadIdx.x][k], s[threadIdx.x + h][k]);
    }
    __syncthreads();
  }
}

// the values of pair i for a pass (false when i has no correspondence)
template <int PASS>
__device__ __forceinline__ bool pair_values(size_t i, const double* __restrict__ src, const double* __restrict__ tgt,
                                            const int32_t* __restrict__ idx, const double* __restrict__ d2,
                                            const double* __restrict__ mean, double* v) {
  const int t = idx[i];
  if (t < 0) return false;
  const double s0 = src[3 * i], s1 = src[3 * i + 1], s2 = src[3 * i + 2];
  const double t0 = tgt[3 * (size_t)t], t1 = tgt[3 * (size_t)t + 1], t2 = tgt[3 * (size_t)t + 2];
  if (PASS == 1) {
    v[0] = 1.0; v[1] = d2[i]; v[2] = s0; v[3] = s1; v[4] = s2; v[5] = t0; v[6] = t1; v[7] = t2;
  } else {
    const double ds[3] = {__dsub_rn(s0, mean[0]), __dsub_rn(s1, mean[1]), __dsub_rn(s2, mean[2])};
    const double dt[3] = {__dsub_rn(t0, mean[3]), __dsub_rn(t1, mean[4]), __dsub_rn(t2, mean[5])};
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) v[3 * r + c] = __dmul_rn(dt[r], ds[c]);
    v[9] = __dadd_rn(__dadd_rn(__dmul_rn(ds[0], ds[0]), __dmul_rn(ds[1], ds[1])), __dmul_rn(ds[2], ds[2]));
  }
  return true;
}

// one block per chunk of CHUNK pairs: thread t sums pairs chunk*CHUNK + t + THREADS*k, k = 0..7, in order; then the block tree
template <int PASS, int M>
__global__ void __launch_bounds__(THREADS) k_moments_chunk(size_t n, const double* __restrict__ src, const double* __restrict__ tgt,
                                                           const int32_t* __restrict__ idx, const double* __restrict__ d2,
                                                           const double* __restrict__ mean, double* __restrict__ part) {
  __shared__ double s[THREADS][M];
  double acc[M];
#pragma unroll
  for (int k = 0; k < M; ++k) acc[k] = 0.0;
#pragma unroll
  for (int j = 0; j < CHUNK_ITEMS; ++j) {
    const size_t i = (size_t)blockIdx.x * CHUNK + (size_t)j * THREADS + threadIdx.x;
    double v[M];
    if (i < n && pair_values<PASS>(i, src, tgt, idx, d2, mean, v)) {
#pragma unroll
      for (int k = 0; k < M; ++k) acc[k] = __dadd_rn(acc[k], v[k]);
    }
  }
  block_sum<M>(acc, s);
  if (threadIdx.x < M) part[(size_t)blockIdx.x * M + threadIdx.x] = s[0][threadIdx.x];
}

// one block: thread t sums the partials t, t + THREADS, ... in order, then the block tree.  Pass 1 also writes the means
// (sum * (1 / count), 0 for an empty set) to mean[0..6) for pass 2.
template <int PASS, int M>
__global__ void __launch_bounds__(THREADS) k_moments_total(size_t chunks, const double* __restrict__ part, double* __restrict__ total,
                                                           double* __restrict__ mean) {
  __shared__ double s[THREADS][M];
  double acc[M];
#pragma unroll
  for (int k = 0; k < M; ++k) acc[k] = 0.0;
  for (size_t c = threadIdx.x; c < chunks; c += THREADS)
#pragma unroll
    for (int k = 0; k < M; ++k) acc[k] = __dadd_rn(acc[k], part[c * M + k]);
  block_sum<M>(acc, s);
  if (threadIdx.x < M) total[threadIdx.x] = s[0][threadIdx.x];
  if (PASS == 1 && threadIdx.x < 6) {
    const double cnt = s[0][0];
    mean[threadIdx.x] = cnt > 0.0 ? __dmul_rn(s[0][2 + threadIdx.x], __ddiv_rn(1.0, cnt)) : 0.0;
  }
}

// result: the totals of both passes (M1 + M2 doubles) followed by the six means, read back with one copy
struct MomLayout { size_t part, result, bytes; };
MomLayout moments_layout(size_t n) {
  MomLayout L; size_t o = 0;
  auto take = layout_taker(o);
  const size_t chunks = (n + CHUNK - 1) / CHUNK;
  L.part = take(chunks * M2 * 8); L.result = take((M1 + M2 + 6) * 8);
  L.bytes = o;
  return L;
}

// ---- in-place transform ---------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(THREADS) k_transform(size_t n, double* __restrict__ pts, Mat4 T) {
  const size_t i = (size_t)blockIdx.x * THREADS + threadIdx.x;
  if (i >= n) return;
  double p[3];
  transform_point(T, pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], p);
  pts[3 * i] = p[0]; pts[3 * i + 1] = p[1]; pts[3 * i + 2] = p[2];
}

}  // namespace

// ---- C ABI -------------------------------------------------------------------------------------------------------

extern "C" GOF_API size_t gof_crop_scratch_bytes(int64_t n) {
  return (n <= 0 || (uint64_t)n >= SORT_LIMIT) ? 0 : crop_layout((size_t)n).bytes;
}

extern "C" GOF_API int gof_crop_polygon(int64_t n, const double* points, const double* transform, int axis, double axis_min, double axis_max,
                                        int num_vertices, const double* polygon_uv, double* out, uint32_t* out_index, int64_t* num_out,
                                        void* scratch, size_t scratch_bytes, void* stream) {
  if (!num_out) { gof_set_error("crop_polygon: NULL argument"); return GOF_E_INVALID; }
  *num_out = 0;
  int rc;
  if ((rc = check_count(n, "points", "crop_polygon")) != GOF_OK) return rc;
  if (axis < 0 || axis > 2) { gof_set_error("crop_polygon: orthogonal axis %d is not 0, 1 or 2", axis); return GOF_E_INVALID; }
  if (num_vertices < 3 || num_vertices > MAX_POLYGON) {
    gof_set_error("crop_polygon: %d polygon vertices; 3 to %d are supported (the polygon is staged in shared memory)", num_vertices,
                  MAX_POLYGON);
    return GOF_E_INVALID;
  }
  if (!polygon_uv) { gof_set_error("crop_polygon: NULL polygon"); return GOF_E_INVALID; }
  for (int k = 0; k < 2 * num_vertices; ++k)
    if (!isfinite(polygon_uv[k])) { gof_set_error("crop_polygon: non-finite polygon vertex"); return GOF_E_INVALID; }
  if (isnan(axis_min) || isnan(axis_max)) { gof_set_error("crop_polygon: NaN axis bound"); return GOF_E_INVALID; }
  if (transform && !finite16(transform)) { gof_set_error("crop_polygon: non-finite transformation"); return GOF_E_INVALID; }
  if (n == 0) return GOF_OK;
  if (!points || !out || !scratch) { gof_set_error("crop_polygon: NULL input"); return GOF_E_INVALID; }
  const size_t N = (size_t)n;
  const CropLayout L = crop_layout(N);
  if (scratch_bytes < L.bytes) {
    gof_set_error("crop_polygon: scratch of %zu bytes, %zu needed (gof_crop_scratch_bytes)", scratch_bytes, L.bytes);
    return GOF_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  char* S = static_cast<char*>(scratch);
  double2* poly = (double2*)(S + L.poly);
  uint32_t *flags = (uint32_t*)(S + L.flags), *off = (uint32_t*)(S + L.off), *tmp = (uint32_t*)(S + L.scan_tmp);
  uint32_t* total = (uint32_t*)(S + L.total);
  CropArgs a{};
  a.has_T = transform != nullptr;
  if (transform) memcpy(a.T.m, transform, sizeof(a.T.m));
  a.w = axis; a.u = axis == 0 ? 1 : 0; a.v = axis == 2 ? 1 : 2;
  a.nv = num_vertices; a.axis_min = axis_min; a.axis_max = axis_max;
  GOF_CUDA_OK(cudaMemcpyAsync(poly, polygon_uv, (size_t)num_vertices * sizeof(double2), cudaMemcpyHostToDevice, st));
  const int g = blocks_for(N, THREADS);
  GOF_LAUNCH("tnt_crop_flags", st, k_crop_flags<<<g, THREADS, (size_t)num_vertices * sizeof(double2), st>>>(N, points, a, poly, flags));
  GOF_LAUNCH_CHECK(false, st);
  if ((rc = gof_exclusive_scan_u32(flags, off, tmp, total, N, false, st)) != GOF_OK) return rc;
  GOF_LAUNCH("tnt_crop_emit", st, k_crop_emit<<<g, THREADS, 0, st>>>(N, points, a, flags, off, out, out_index));
  GOF_LAUNCH_CHECK(false, st);
  uint32_t kept;
  if ((rc = gof_read_back(&kept, total, 4, st)) != GOF_OK) return rc;
  *num_out = kept;
  return GOF_OK;
}

extern "C" GOF_API size_t gof_voxel_down_sample_scratch_bytes(int64_t n) {
  return (n <= 0 || (uint64_t)n >= SORT_LIMIT) ? 0 : voxel_layout((size_t)n).bytes;
}

extern "C" GOF_API int gof_voxel_down_sample(int64_t n, const double* points, double voxel, double* out, int64_t* num_out, void* scratch,
                                             size_t scratch_bytes, void* stream) {
  if (!num_out) { gof_set_error("voxel_down_sample: NULL argument"); return GOF_E_INVALID; }
  *num_out = 0;
  int rc;
  if ((rc = check_count(n, "points", "voxel_down_sample")) != GOF_OK) return rc;
  if (!(voxel > 0.0) || !isfinite(voxel)) { gof_set_error("voxel_down_sample: voxel_size %g must be positive and finite", voxel); return GOF_E_INVALID; }
  if (n == 0) return GOF_OK;
  if (!points || !out || !scratch) { gof_set_error("voxel_down_sample: NULL input"); return GOF_E_INVALID; }
  const size_t N = (size_t)n;
  const VoxelLayout L = voxel_layout(N);
  if (scratch_bytes < L.bytes) {
    gof_set_error("voxel_down_sample: scratch of %zu bytes, %zu needed (gof_voxel_down_sample_scratch_bytes)", scratch_bytes, L.bytes);
    return GOF_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  char* S = static_cast<char*>(scratch);
  unsigned long long* bbox = (unsigned long long*)(S + L.bbox);
  GOF_CUDA_OK(cudaMemsetAsync(bbox, 0xff, 24, st));
  GOF_CUDA_OK(cudaMemsetAsync(bbox + 3, 0, 32, st));
  const int g = blocks_for(N, THREADS);
  GOF_LAUNCH("tnt_voxel_bbox", st, gof_tree::k_tree_bbox<double><<<g < 1056 ? g : 1056, THREADS, 0, st>>>((int)n, points, bbox));
  GOF_LAUNCH_CHECK(false, st);
  GOF_LAUNCH("tnt_voxel_nonfinite", st, k_nonfinite<<<g, THREADS, 0, st>>>(N, points, bbox + 6));
  GOF_LAUNCH_CHECK(false, st);
  unsigned long long hb[7];
  if ((rc = gof_read_back(hb, bbox, sizeof(hb), st)) != GOF_OK) return rc;
  if (hb[6]) { gof_set_error("voxel_down_sample: non-finite coordinates"); return GOF_E_INVALID; }
  double lo[3], hi[3], kmax = 0.0, ext = 0.0;
  for (int a = 0; a < 3; ++a) {
    const double mn = host_value_of(hb[a]), mx = host_value_of(hb[3 + a]);
    lo[a] = mn - voxel * 0.5;
    hi[a] = mx + voxel * 0.5;
    ext = fmax(ext, hi[a] - lo[a]);
    kmax = fmax(kmax, floor((mx - lo[a]) / voxel));
  }
  if (voxel * (double)INT_MAX < ext) {
    gof_set_error("voxel_down_sample: voxel_size is too small (%g for an extent of %g)", voxel, ext);
    return GOF_E_INVALID;
  }
  uint32_t *kx = (uint32_t*)(S + L.kx), *ky = (uint32_t*)(S + L.ky), *kz = (uint32_t*)(S + L.kz);
  uint32_t *ka = (uint32_t*)(S + L.ka), *kb = (uint32_t*)(S + L.kb), *va = (uint32_t*)(S + L.va), *vb = (uint32_t*)(S + L.vb);
  uint32_t *hist = (uint32_t*)(S + L.hist), *head = (uint32_t*)(S + L.head), *run = (uint32_t*)(S + L.run);
  uint32_t *tmp = (uint32_t*)(S + L.scan_tmp), *runs = (uint32_t*)(S + L.runs), *start = (uint32_t*)(S + L.start);
  GOF_LAUNCH("tnt_voxel_keys", st, k_voxel_keys<<<g, THREADS, 0, st>>>(N, points, lo[0], lo[1], lo[2], voxel, kx, ky, kz));
  GOF_LAUNCH_CHECK(false, st);
  const int bits = bit_width(kmax);              // every key is <= kmax: the quotient is monotone in p
  const GofKeyWords key{{kz, ky, kx}, {bits, bits, bits}, 3};
  if ((rc = gof_sort_words_u32(key, N, GofSortBufs{ka, kb, va, vb, hist}, va, false, st)) != GOF_OK) return rc;
  if ((rc = gof_key_runs_u32(key, va, N, head, run, tmp, runs, false, st)) != GOF_OK) return rc;
  GOF_LAUNCH("tnt_voxel_starts", st, k_voxel_starts<<<g, THREADS, 0, st>>>(N, head, run, runs, start));
  GOF_LAUNCH_CHECK(false, st);
  uint32_t voxels;
  if ((rc = gof_read_back(&voxels, runs, 4, st)) != GOF_OK) return rc;
  GOF_LAUNCH("tnt_voxel_mean", st, k_voxel_mean<<<blocks_for(voxels, THREADS), THREADS, 0, st>>>(voxels, points, va, start, out));
  GOF_LAUNCH_CHECK(false, st);
  *num_out = voxels;
  return GOF_OK;
}

extern "C" GOF_API size_t gof_icp_moments_scratch_bytes(int64_t n) {
  return (n <= 0 || (uint64_t)n >= SORT_LIMIT) ? 0 : moments_layout((size_t)n).bytes;
}

extern "C" GOF_API int gof_icp_moments(int64_t n, const double* src, const double* tgt, const int32_t* index, const double* d2,
                                       double* moments, void* scratch, size_t scratch_bytes, void* stream) {
  int rc;
  if (!moments) { gof_set_error("icp_moments: NULL argument"); return GOF_E_INVALID; }
  if ((rc = check_count(n, "source points", "icp_moments")) != GOF_OK) return rc;
  for (int k = 0; k < M1 + M2; ++k) moments[k] = 0.0;
  if (n == 0) return GOF_OK;
  if (!src || !tgt || !index || !d2 || !scratch) { gof_set_error("icp_moments: NULL input"); return GOF_E_INVALID; }
  const size_t N = (size_t)n;
  const MomLayout L = moments_layout(N);
  if (scratch_bytes < L.bytes) {
    gof_set_error("icp_moments: scratch of %zu bytes, %zu needed (gof_icp_moments_scratch_bytes)", scratch_bytes, L.bytes);
    return GOF_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  char* S = static_cast<char*>(scratch);
  double *part = (double*)(S + L.part), *total = (double*)(S + L.result), *mean = total + M1 + M2;
  const size_t chunks = (N + CHUNK - 1) / CHUNK;
  GOF_LAUNCH("tnt_moments1", st, (k_moments_chunk<1, M1><<<(int)chunks, THREADS, 0, st>>>(N, src, tgt, index, d2, nullptr, part)));
  GOF_LAUNCH_CHECK(false, st);
  GOF_LAUNCH("tnt_moments1_total", st, (k_moments_total<1, M1><<<1, THREADS, 0, st>>>(chunks, part, total, mean)));
  GOF_LAUNCH_CHECK(false, st);
  GOF_LAUNCH("tnt_moments2", st, (k_moments_chunk<2, M2><<<(int)chunks, THREADS, 0, st>>>(N, src, tgt, index, d2, mean, part)));
  GOF_LAUNCH_CHECK(false, st);
  GOF_LAUNCH("tnt_moments2_total", st, (k_moments_total<2, M2><<<1, THREADS, 0, st>>>(chunks, part, total + M1, nullptr)));
  GOF_LAUNCH_CHECK(false, st);
  double h[M1 + M2 + 6];
  if ((rc = gof_read_back(h, total, sizeof(h), st)) != GOF_OK) return rc;
  // out: count, sum d2, mean src[3], mean tgt[3], cov[9] (row = target axis), src variance sum
  moments[0] = h[0]; moments[1] = h[1];
  for (int k = 0; k < 6; ++k) moments[2 + k] = h[M1 + M2 + k];
  for (int k = 0; k < M2; ++k) moments[M1 + k] = h[M1 + k];
  return GOF_OK;
}

extern "C" GOF_API int gof_transform_points(int64_t n, double* points, const double* transform, void* stream) {
  int rc;
  if ((rc = check_count(n, "points", "transform_points")) != GOF_OK) return rc;
  if (!transform) { gof_set_error("transform_points: NULL transformation"); return GOF_E_INVALID; }
  if (!finite16(transform)) { gof_set_error("transform_points: non-finite transformation"); return GOF_E_INVALID; }
  if (n == 0) return GOF_OK;
  if (!points) { gof_set_error("transform_points: NULL points"); return GOF_E_INVALID; }
  Mat4 T;
  memcpy(T.m, transform, sizeof(T.m));
  cudaStream_t st = (cudaStream_t)stream;
  GOF_LAUNCH("tnt_transform", st, k_transform<<<blocks_for((size_t)n, THREADS), THREADS, 0, st>>>((size_t)n, points, T));
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}
