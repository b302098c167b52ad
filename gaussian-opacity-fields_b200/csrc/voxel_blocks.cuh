// voxel_blocks.cuh -- the sparse voxel-block keys shared by the TSDF volume (tsdf.cu, DESIGN section 4.4) and the opacity
// field's lattice (field_grid.cu, DESIGN section 4.15): the 63-bit key packing, the binary search of a sorted key list and
// the emission of one key per run of equal keys after the library's multi-word sort; and the lattice's parameter checks.
#pragma once
#include "gof_common.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int KEY_BITS = 21;
constexpr int64_t KEY_BIAS = (int64_t)1 << 20;

__device__ __forceinline__ int64_t pack_key(int bx, int by, int bz) {
  return (((int64_t)bz + KEY_BIAS) << (2 * KEY_BITS)) | (((int64_t)by + KEY_BIAS) << KEY_BITS) | ((int64_t)bx + KEY_BIAS);
}
__device__ __forceinline__ void unpack_key(int64_t k, int* b) {
  const int64_t m = ((int64_t)1 << KEY_BITS) - 1;
  b[0] = (int)((k & m) - KEY_BIAS);
  b[1] = (int)(((k >> KEY_BITS) & m) - KEY_BIAS);
  b[2] = (int)((k >> (2 * KEY_BITS)) - KEY_BIAS);
}

// position of the first key >= k in the sorted list
__device__ __forceinline__ int64_t lower_bound(const int64_t* __restrict__ keys, int64_t n, int64_t k) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (keys[mid] < k) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// ord: the instances in key order; head / uid: the runs of equal keys along it (gof_key_runs_u32)
__global__ void __launch_bounds__(THREADS) k_key_emit(size_t n, const uint32_t* __restrict__ lo_w, const uint32_t* __restrict__ hi_w,
                                                     const uint32_t* __restrict__ ord, const uint32_t* __restrict__ head,
                                                     const uint32_t* __restrict__ uid, int64_t* __restrict__ keys) {
  const size_t j = (size_t)blockIdx.x * THREADS + threadIdx.x;
  if (j >= n || !head[j]) return;
  const uint32_t i = ord[j];
  keys[uid[j]] = (int64_t)(((uint64_t)hi_w[i] << 32) | lo_w[i]);
}

// The opacity field's lattice (field_grid.cu, tsdf.cu's field marching cubes): voxel_size > 0 and block_resolution in 1..64
static int field_grid_check_params(const gof_field_grid_params_t* p, const char* who) {
  if (!p || !(p->voxel_size > 0.f) || p->block_resolution < 1 || p->block_resolution > 64) {
    gof_set_error("%s: voxel_size > 0 and block_resolution in 1..64 required", who);
    return GOF_E_INVALID;
  }
  return GOF_OK;
}

// ... and fewer than 2^31 lattice points (the query's point count is an int), hence fewer than 2^31 blocks
static int field_grid_check_points(const gof_field_grid_params_t* p, int64_t num_blocks, const char* who) {
  const int64_t n3 = (int64_t)p->block_resolution * p->block_resolution * p->block_resolution;
  if (num_blocks < 0 || num_blocks > (((int64_t)1 << 31) - 1) / n3) {
    gof_set_error("%s: %lld blocks of %lld voxels; the lattice must have fewer than 2^31 points", who, (long long)num_blocks,
                  (long long)n3);
    return GOF_E_INVALID;
  }
  return GOF_OK;
}

}  // namespace
