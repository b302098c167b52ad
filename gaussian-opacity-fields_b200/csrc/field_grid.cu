// field_grid.cu -- the sparse voxel-block lattice of the opacity field (DESIGN section 4.15): the blocks the Gaussians touch and
// the lattice points of those blocks.  Marching cubes of the field on the lattice is tsdf.cu's extraction, instantiated for
// one value plane (gof_field_grid_extract_*).
//
//   count   one thread per Gaussian: the frustum test of its centre and the block box of its dilated 3-sigma box
//           (tetra_points.cuh, so the corners are gof_tetra_points' bit for bit); its block count, its box origin and
//           extents; a scan of the counts
//   emit    one thread per (Gaussian, block) instance, its Gaussian found by binary search of the scanned counts, so a
//           Gaussian touching many blocks spreads over many threads; the 63-bit keys as (lo, hi) u32 words -> the library's
//           multi-word sort -> one key per run of equal keys (voxel_blocks.cuh)
//   points  one thread per lattice point, in pool order
#include "gof_common.cuh"
#include "tetra_points.cuh"
#include "voxel_blocks.cuh"

namespace {

constexpr uint64_t MAX_INSTANCES = 1ull << 30;   // the sort's limit

struct GridPar { float s, bs; int B; };

static GridPar make_grid_par(const gof_field_grid_params_t* p) {
  GridPar q;
  q.s = p->voxel_size; q.B = p->block_resolution;
  q.bs = (float)q.B * q.s;   // fl(B * s): B is exact in float
  return q;
}

struct GaussHeader { unsigned long long n_inst64; uint32_t err, n_inst, n_unique, pad; };
struct GaussLayout { size_t header, cnt, off, lo, ext, scan_tmp, bytes; };
static GaussLayout gauss_layout(size_t P) {
  GaussLayout L; size_t o = 0;
  auto take = [&](size_t b) { size_t r = o; o = gof_align_up(o + b, 256); return r; };
  L.header = take(256);
  L.cnt = take(P * 4); L.off = take(P * 4);
  L.lo = take(P * 12); L.ext = take(P * 8);
  L.scan_tmp = take(gof_scan_scratch_bytes(P));
  L.bytes = o;
  return L;
}
struct InstLayout { size_t lo, hi, val_a, val_b, hist, head, uid, scan_tmp, bytes; };
static InstLayout inst_layout(size_t I) {
  InstLayout L; size_t o = 0;
  auto take = [&](size_t b) { size_t r = o; o = gof_align_up(o + b, 256); return r; };
  L.lo = take(I * 4); L.hi = take(I * 4);
  L.val_a = take(I * 4); L.val_b = take(I * 4);
  L.hist = take(gof_sort_scratch_bytes(I));
  L.head = take(I * 4); L.uid = take(I * 4);
  L.scan_tmp = take(gof_scan_scratch_bytes(I));
  L.bytes = o;
  return L;
}

// NaN-propagating min / max, so that a non-finite corner reaches the range check instead of being dropped
__device__ __forceinline__ float min_nan(float a, float b) { return (b != b || b < a) ? b : a; }
__device__ __forceinline__ float max_nan(float a, float b) { return (b != b || b > a) ? b : a; }

// Block range [lo, hi] per axis (as floats) of Gaussian g; false when no view's frustum holds its centre
__device__ __forceinline__ bool gaussian_blocks(int g, const float* __restrict__ xyz, const float* __restrict__ scales,
                                                const float4* __restrict__ rotations, int n_views, const float* __restrict__ views,
                                                float near, float far, const GridPar& p, float* lo, float* hi) {
  const float c[3] = {xyz[3 * (size_t)g], xyz[3 * (size_t)g + 1], xyz[3 * (size_t)g + 2]};
  if (tp_first_view(c, views, n_views, 0, near, far) < 0) return false;
  const float4 q = rotations[g];
  const float r[4] = {q.x, q.y, q.z, q.w};
  const float s[3] = {scales[3 * (size_t)g], scales[3 * (size_t)g + 1], scales[3 * (size_t)g + 2]};
  float R[9], s3[3], ps;
  tp_gaussian_frame(r, s, R, s3, &ps);
  float mn[3], mx[3];
  tp_corner(R, s3, c, 0, mn);
#pragma unroll
  for (int a = 0; a < 3; ++a) mx[a] = mn[a];
#pragma unroll 1
  for (int k = 1; k < 8; ++k) {
    float v[3];
    tp_corner(R, s3, c, k, v);
#pragma unroll
    for (int a = 0; a < 3; ++a) { mn[a] = min_nan(mn[a], v[a]); mx[a] = max_nan(mx[a], v[a]); }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    lo[a] = floorf(__fdiv_rn(__fsub_rn(mn[a], p.s), p.bs));
    hi[a] = floorf(__fdiv_rn(__fadd_rn(mx[a], p.s), p.bs));
  }
  return true;
}

__global__ void __launch_bounds__(THREADS) k_grid_count(int P, const float* __restrict__ xyz, const float* __restrict__ scales,
                                                       const float4* __restrict__ rotations, int n_views, const float* __restrict__ views,
                                                       float near, float far, const GridPar p, uint32_t* __restrict__ cnt,
                                                       int3* __restrict__ blo, uint2* __restrict__ ext, GaussHeader* __restrict__ hd) {
  const int g = blockIdx.x * THREADS + threadIdx.x;
  unsigned long long n = 0;
  if (g < P) {
    float lo[3], hi[3];
    if (gaussian_blocks(g, xyz, scales, rotations, n_views, views, near, far, p, lo, hi)) {
      bool in_range = true;
#pragma unroll
      for (int a = 0; a < 3; ++a) in_range = in_range && lo[a] >= -(float)KEY_BIAS && hi[a] < (float)KEY_BIAS;
      if (!in_range) {
        atomicOr(&hd->err, 1u);
      } else {
        const int l[3] = {(int)lo[0], (int)lo[1], (int)lo[2]};
        const unsigned long long e[3] = {(unsigned long long)((int)hi[0] - l[0] + 1), (unsigned long long)((int)hi[1] - l[1] + 1),
                                         (unsigned long long)((int)hi[2] - l[2] + 1)};
        n = e[0] * e[1] * e[2];   // < 2^63: each extent is at most 2^21
        blo[g] = make_int3(l[0], l[1], l[2]);
        ext[g] = make_uint2((uint32_t)e[0], (uint32_t)e[1]);
      }
    }
    // a Gaussian's own count beyond the instance limit is recorded, and summed, as the limit: the total then reaches it as
    // well, and cannot wrap (at most 2^32 / 9 Gaussians of at most 2^30 each)
    n = n < MAX_INSTANCES ? n : MAX_INSTANCES;
    cnt[g] = (uint32_t)n;
  }
  // the total in 64 bits, checked against the sort's limit before the u32 offsets are used
  for (int o = 16; o > 0; o >>= 1) n += __shfl_down_sync(0xffffffffu, n, o);
  if ((threadIdx.x & 31) == 0 && n) atomicAdd(&hd->n_inst64, n);
}

// instance i: the Gaussian whose scanned range holds it (the last g with off[g] <= i), then its block in x-fastest order
__global__ void __launch_bounds__(THREADS) k_grid_emit(int P, size_t I, const uint32_t* __restrict__ off, const int3* __restrict__ blo,
                                                      const uint2* __restrict__ ext, uint32_t* __restrict__ lo_w,
                                                      uint32_t* __restrict__ hi_w) {
  const size_t i = (size_t)blockIdx.x * THREADS + threadIdx.x;
  if (i >= I) return;
  int a = 0, b = P;   // upper bound of i in off, minus one
  while (a < b) {
    const int m = (a + b) >> 1;
    if (off[m] <= (uint32_t)i) a = m + 1; else b = m;
  }
  const int g = a - 1;
  const uint32_t j = (uint32_t)i - off[g];
  const int3 l = blo[g];
  const uint2 e = ext[g];
  const uint32_t x = j % e.x, yz = j / e.x;
  const uint64_t k = (uint64_t)pack_key(l.x + (int)x, l.y + (int)(yz % e.y), l.z + (int)(yz / e.y));
  lo_w[i] = (uint32_t)k;
  hi_w[i] = (uint32_t)(k >> 32);
}

__global__ void __launch_bounds__(THREADS) k_grid_points(size_t N, int B, float s, const int64_t* __restrict__ keys,
                                                        float* __restrict__ points) {
  const size_t idx = (size_t)blockIdx.x * THREADS + threadIdx.x;
  if (idx >= N) return;
  const int n3 = B * B * B;
  const int lin = (int)(idx % n3);
  int b[3];
  unpack_key(keys[idx / n3], b);
  const int li[3] = {lin % B, (lin / B) % B, lin / (B * B)};
#pragma unroll
  for (int a = 0; a < 3; ++a) points[3 * idx + a] = __fmul_rn(__int2float_rn(b[a] * B + li[a]), s);
}

}  // namespace

extern "C" GOF_API int gof_field_grid_blocks_count(const gof_field_grid_params_t* params, int P, const float* xyz, const float* scales,
                                                   const float* rotations, int n_views, const float* views, float near, float far,
                                                   gof_alloc_fn gauss_alloc, void* gauss_user, gof_alloc_fn inst_alloc, void* inst_user,
                                                   int64_t* num_blocks_out, void* stream) {
  if (!num_blocks_out || !gauss_alloc || !inst_alloc) { gof_set_error("field_grid_blocks_count: NULL argument"); return GOF_E_INVALID; }
  *num_blocks_out = 0;
  int rc;
  if ((rc = field_grid_check_params(params, "field_grid_blocks_count")) != GOF_OK) return rc;
  if (P < 0 || 9ull * (unsigned long long)P > 0xFFFFFFFFull || n_views < 1) {
    gof_set_error("field_grid_blocks_count: bad sizes (P = %d, n_views = %d; need 0 <= 9 P < 2^32 and at least one view)", P, n_views);
    return GOF_E_INVALID;
  }
  if (P == 0) return GOF_OK;
  if (!xyz || !scales || !rotations || !views) { gof_set_error("field_grid_blocks_count: NULL pointer"); return GOF_E_INVALID; }
  if (reinterpret_cast<uintptr_t>(rotations) & 15) {
    gof_set_error("field_grid_blocks_count: rotations must be 16-byte aligned (they are read as float4)");
    return GOF_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const GridPar p = make_grid_par(params);
  const GaussLayout L = gauss_layout((size_t)P);
  char* S = (char*)gauss_alloc(gauss_user, L.bytes);
  if (!S) { gof_set_error("scratch allocator returned NULL"); return GOF_E_ALLOC; }
  GaussHeader* hd = (GaussHeader*)(S + L.header);
  uint32_t *cnt = (uint32_t*)(S + L.cnt), *off = (uint32_t*)(S + L.off), *tmp = (uint32_t*)(S + L.scan_tmp);
  int3* blo = (int3*)(S + L.lo);
  uint2* ext = (uint2*)(S + L.ext);
  GOF_CUDA_OK(cudaMemsetAsync(hd, 0, sizeof(GaussHeader), st));
  const unsigned gp = (unsigned)((P + THREADS - 1) / THREADS);
  GOF_LAUNCH("field_grid_count", st, k_grid_count<<<gp, THREADS, 0, st>>>(P, xyz, scales, reinterpret_cast<const float4*>(rotations),
                                                                           n_views, views, near, far, p, cnt, blo, ext, hd));
  GOF_LAUNCH_CHECK(false, st);
  if ((rc = gof_exclusive_scan_u32(cnt, off, tmp, &hd->n_inst, (size_t)P, false, st)) != GOF_OK) return rc;
  GaussHeader h;
  if ((rc = gof_read_back(&h, hd, sizeof(h), st)) != GOF_OK) return rc;
  if (h.err) { gof_set_error("field_grid_blocks_count: a touched block lies outside [-2^20, 2^20) per axis"); return GOF_E_INVALID; }
  if (h.n_inst64 >= MAX_INSTANCES) {
    gof_set_error("field_grid_blocks_count: 2^30 or more (Gaussian, block) instances; fewer than 2^30 are supported (a larger "
                  "voxel_size or block_resolution touches fewer blocks)");
    return GOF_E_INVALID;
  }
  const size_t I = (size_t)h.n_inst64;
  if (I == 0) return GOF_OK;
  const InstLayout IL = inst_layout(I);
  char* T = (char*)inst_alloc(inst_user, IL.bytes);
  if (!T) { gof_set_error("scratch allocator returned NULL"); return GOF_E_ALLOC; }
  uint32_t *lo = (uint32_t*)(T + IL.lo), *hi = (uint32_t*)(T + IL.hi);
  uint32_t *va = (uint32_t*)(T + IL.val_a), *vb = (uint32_t*)(T + IL.val_b), *hist = (uint32_t*)(T + IL.hist);
  uint32_t *head = (uint32_t*)(T + IL.head), *uid = (uint32_t*)(T + IL.uid), *itmp = (uint32_t*)(T + IL.scan_tmp);
  GOF_LAUNCH("field_grid_emit", st, k_grid_emit<<<(unsigned)((I + THREADS - 1) / THREADS), THREADS, 0, st>>>(P, I, off, blo, ext, lo, hi));
  GOF_LAUNCH_CHECK(false, st);
  // ascending 63-bit keys (the high word has 31 bits); head / uid are written only after the sort, so they are its key
  // buffers; the order lands in val_a
  const GofKeyWords key{{lo, hi, nullptr}, {32, 31, 0}, 2};
  if ((rc = gof_sort_words_u32(key, I, GofSortBufs{head, uid, va, vb, hist}, va, false, st)) != GOF_OK) return rc;
  if ((rc = gof_key_runs_u32(key, va, I, head, uid, itmp, &hd->n_unique, false, st)) != GOF_OK) return rc;
  if ((rc = gof_read_back(&h, hd, sizeof(h), st)) != GOF_OK) return rc;
  *num_blocks_out = (int64_t)h.n_unique;
  return GOF_OK;
}

extern "C" GOF_API int gof_field_grid_blocks_emit(const gof_field_grid_params_t* params, int P, void* gauss_scratch, void* inst_scratch,
                                                  int64_t num_blocks, int64_t* keys_out, void* stream) {
  if (num_blocks == 0) return GOF_OK;
  if (!gauss_scratch || !inst_scratch || !keys_out || P <= 0) { gof_set_error("field_grid_blocks_emit: NULL argument"); return GOF_E_INVALID; }
  int rc;
  if ((rc = field_grid_check_params(params, "field_grid_blocks_emit")) != GOF_OK) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const GaussLayout L = gauss_layout((size_t)P);
  GaussHeader h;
  if ((rc = gof_read_back(&h, (char*)gauss_scratch + L.header, sizeof(h), st)) != GOF_OK) return rc;
  if ((int64_t)h.n_unique != num_blocks) { gof_set_error("field_grid_blocks_emit: size does not match the count phase"); return GOF_E_INVALID; }
  const size_t I = (size_t)h.n_inst64;
  const InstLayout IL = inst_layout(I);
  const char* T = (const char*)inst_scratch;
  GOF_LAUNCH("field_grid_keys", st, k_key_emit<<<(unsigned)((I + THREADS - 1) / THREADS), THREADS, 0, st>>>(
      I, (const uint32_t*)(T + IL.lo), (const uint32_t*)(T + IL.hi), (const uint32_t*)(T + IL.val_a), (const uint32_t*)(T + IL.head),
      (const uint32_t*)(T + IL.uid), keys_out));
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}

extern "C" GOF_API int gof_field_grid_points(const gof_field_grid_params_t* params, int64_t num_blocks, const int64_t* keys, float* points,
                                             void* stream) {
  int rc;
  if ((rc = field_grid_check_params(params, "field_grid_points")) != GOF_OK) return rc;
  if ((rc = field_grid_check_points(params, num_blocks, "field_grid_points")) != GOF_OK) return rc;
  const int64_t n3 = (int64_t)params->block_resolution * params->block_resolution * params->block_resolution;
  if (num_blocks == 0) return GOF_OK;
  if (!keys || !points) { gof_set_error("field_grid_points: NULL pointer"); return GOF_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const size_t N = (size_t)num_blocks * (size_t)n3;
  GOF_LAUNCH("field_grid_points", st, k_grid_points<<<(unsigned)((N + THREADS - 1) / THREADS), THREADS, 0, st>>>(
      N, params->block_resolution, params->voxel_size, keys, points));
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}
