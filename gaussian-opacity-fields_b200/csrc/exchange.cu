// exchange.cu -- the reduction of the one exchange step of view-parallel training (SURVEY.md 8(e)): the sum over ranks of the flat
// per-Gaussian gradient bucket -- 59 gradient + 5 statistics floats per Gaussian, or 11 + 5 when the SH gradient travels as
// per-view dL_dRGB records (gof_dp.GradBucket(factor_sh=True), csrc/sh_views.cu) -- done by ONE kernel over NVLink peer memory
// or through the NVSwitch instead of a library all-reduce.  No reference counterpart (the reference is single-GPU).
//
// Every rank's bucket is mapped into every process (CUDA IPC).  Rank r owns the r-th 1/N slice of the index space:
// it loads that slice from all N buckets (N-1 of them over NVLink), adds them in rank order 0..N-1 -- so every rank
// ends with bit-identical sums -- and stores the result into all N buckets.  Slices are disjoint, so inside the
// kernel no location is touched by two ranks; the caller brackets the launch with two cross-rank barriers
// (all buckets complete before / all slices written after).  Per GPU: (N-1)/N of the bucket in and the same out.
#include <stdint.h>

#include "gof_common.cuh"

namespace {

constexpr int GOF_MAX_PEERS = 8;
struct PeerPtrs { float4* p[GOF_MAX_PEERS]; };

__device__ __forceinline__ float4 ld_cg(const float4* p) { return __ldcg(p); }   // L2 only: peer data is never L1-cached

// elements [begin, end) of this rank's slice; float4 index < sum_end: SUM over ranks, otherwise MAX (the densification
// statistics max_radii2D / xyz_gradient_accum_abs_max ride in the tail of the same bucket)
__device__ __forceinline__ float4 combine(const float4 s, const float4 v, bool is_sum) {
  return is_sum ? make_float4(s.x + v.x, s.y + v.y, s.z + v.z, s.w + v.w)
                : make_float4(fmaxf(s.x, v.x), fmaxf(s.y, v.y), fmaxf(s.z, v.z), fmaxf(s.w, v.w));
}

template <int W>
__global__ void __launch_bounds__(512) k_p2p_allreduce(const PeerPtrs a, size_t begin, size_t end, size_t sum_end) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = begin + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < end; i += stride) {
    float4 v[W];
#pragma unroll
    for (int r = 0; r < W; ++r) v[r] = ld_cg(a.p[r] + i);
    float4 s = v[0];
    const bool is_sum = i < sum_end;
#pragma unroll
    for (int r = 1; r < W; ++r) s = combine(s, v[r], is_sum);
#pragma unroll
    for (int r = 0; r < W; ++r) __stcg(a.p[r] + i, s);
  }
}

// generic world size (3, 5, 6, 7): same scheme, runtime loop
__global__ void __launch_bounds__(512) k_p2p_allreduce_any(const PeerPtrs a, int world, size_t begin, size_t end, size_t sum_end) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = begin + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < end; i += stride) {
    float4 s = ld_cg(a.p[0] + i);
    const bool is_sum = i < sum_end;
    for (int r = 1; r < world; ++r) s = combine(s, ld_cg(a.p[r] + i), is_sum);
    for (int r = 0; r < world; ++r) __stcg(a.p[r] + i, s);
  }
}

// ---- the same exchange through the NVSwitch (NVLS): `mc` is the MULTICAST address of the bucket (every rank's copy bound to
// one multicast object at the same offset).  multimem.ld_reduce pulls the 16 bytes at that offset from ALL ranks and hands
// back their sum -- reduced inside the switch -- and multimem.st pushes the result to all of them: per GPU one bucket's worth of
// NVLink traffic in each direction instead of 2 (N-1)/N buckets over peer loads/stores.  Rank r handles the r-th 1/N slice; the
// MAX tail holds non-negative floats, whose bit patterns order like unsigned integers (f32 has no multimem max).
__device__ __forceinline__ float4 mm_ld_add(const float4* p) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void mm_st(float4* p, const float4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

__global__ void __launch_bounds__(512) k_nvls_allreduce(float4* mc, size_t begin, size_t end, size_t sum_end) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  size_t i = begin + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  // SUM part, four independent 16-byte reductions in flight per thread (a switch round trip is microseconds)
  const size_t s_end = sum_end < end ? sum_end : end;
  for (; i + 3 * stride < s_end; i += 4 * stride) {
    const float4 a = mm_ld_add(mc + i), b = mm_ld_add(mc + i + stride), c = mm_ld_add(mc + i + 2 * stride), d = mm_ld_add(mc + i + 3 * stride);
    mm_st(mc + i, a); mm_st(mc + i + stride, b); mm_st(mc + i + 2 * stride, c); mm_st(mc + i + 3 * stride, d);
  }
  for (; i < s_end; i += stride) mm_st(mc + i, mm_ld_add(mc + i));
  // MAX tail (continues on the same index lattice)
  for (; i < end; i += stride) {
    uint32_t* q = reinterpret_cast<uint32_t*>(mc + i);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      uint32_t u;
      asm volatile("multimem.ld_reduce.relaxed.sys.global.max.u32 %0, [%1];" : "=r"(u) : "l"(q + k) : "memory");
      asm volatile("multimem.st.relaxed.sys.global.u32 [%0], %1;" ::"l"(q + k), "r"(u) : "memory");
    }
  }
}

}  // namespace

// A bucket that other processes can map: plain cudaMalloc (its own allocation, so the IPC handle addresses it at offset
// 0), zero-filled.  handle64 receives the 64-byte cudaIpcMemHandle_t to send to the peers.
extern "C" GOF_API int gof_peer_alloc(size_t bytes, void** ptr, unsigned char* handle64) {
  if (!ptr || !handle64 || bytes == 0) { gof_set_error("peer_alloc: bad arguments"); return GOF_E_INVALID; }
  void* p = nullptr;
  GOF_CUDA_OK(cudaMalloc(&p, bytes));
  GOF_CUDA_OK(cudaMemset(p, 0, bytes));
  cudaIpcMemHandle_t h;
  GOF_CUDA_OK(cudaIpcGetMemHandle(&h, p));
  static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(handle64, &h, 64);
  *ptr = p;
  return GOF_OK;
}
// Maps a peer's bucket into this process FOR THE CURRENT DEVICE (peer access to the exporting device is enabled by
// the driver as part of the mapping -- the way NCCL's P2P transport opens its buffers).
extern "C" GOF_API int gof_peer_open(const unsigned char* handle64, void** ptr) {
  if (!ptr || !handle64) { gof_set_error("peer_open: bad arguments"); return GOF_E_INVALID; }
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  void* p = nullptr;
  GOF_CUDA_OK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  *ptr = p;
  return GOF_OK;
}
extern "C" GOF_API int gof_peer_close(void* ptr) { if (ptr) GOF_CUDA_OK(cudaIpcCloseMemHandle(ptr)); return GOF_OK; }
extern "C" GOF_API int gof_peer_free(void* ptr) { if (ptr) GOF_CUDA_OK(cudaFree(ptr)); return GOF_OK; }

static unsigned exchange_grid(size_t items) {
  const size_t want = (items + 511) / 512;
  return (unsigned)(want < (size_t)gof_sm_count() * 4 ? want : (size_t)gof_sm_count() * 4);
}

// mc: multicast address of the bucket (valid in THIS process); n floats, the first n_sum summed, the rest max-reduced as
// non-negative floats; n and n_sum multiples of 4.  The caller brackets the call with two cross-rank barriers on `stream`.
extern "C" GOF_API int gof_nvls_allreduce_f32(float* mc, int world, int rank, size_t n_sum, size_t n, void* stream) {
  if (!mc || world < 1 || rank < 0 || rank >= world || (n & 3u) || (n_sum & 3u) || n_sum > n || (reinterpret_cast<uintptr_t>(mc) & 15u)) {
    gof_set_error("nvls_allreduce: bad arguments");
    return GOF_E_INVALID;
  }
  if (world == 1 || n == 0) return GOF_OK;
  const size_t n4 = n / 4;
  const size_t begin = n4 * (size_t)rank / (size_t)world, end = n4 * (size_t)(rank + 1) / (size_t)world;
  if (end <= begin) return GOF_OK;
  cudaStream_t st = (cudaStream_t)stream;
  GOF_LAUNCH("nvls_allreduce", st, k_nvls_allreduce<<<exchange_grid(end - begin), 512, 0, st>>>(reinterpret_cast<float4*>(mc), begin, end, n_sum / 4));
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}

// the first n_sum floats are summed over the ranks, the remaining n - n_sum max-reduced (n_sum == n: plain sum)
extern "C" GOF_API int gof_p2p_allreduce_f32(float* const* peers, int world, int rank, size_t n_sum, size_t n, void* stream) {
  if (!peers || world < 1 || world > GOF_MAX_PEERS || rank < 0 || rank >= world || (n & 3u) || (n_sum & 3u) || n_sum > n) {
    gof_set_error("p2p_allreduce: bad arguments (world 1..8, n and n_sum multiples of 4, n_sum <= n)");
    return GOF_E_INVALID;
  }
  if (world == 1 || n == 0) return GOF_OK;
  PeerPtrs a;
  for (int r = 0; r < GOF_MAX_PEERS; ++r) a.p[r] = reinterpret_cast<float4*>(r < world ? peers[r] : nullptr);
  for (int r = 0; r < world; ++r)
    if (!a.p[r] || (reinterpret_cast<uintptr_t>(a.p[r]) & 15u)) { gof_set_error("p2p_allreduce: peer pointer NULL or unaligned"); return GOF_E_INVALID; }
  const size_t n4 = n / 4;
  const size_t begin = n4 * (size_t)rank / (size_t)world, end = n4 * (size_t)(rank + 1) / (size_t)world;
  if (end <= begin) return GOF_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned grid = exchange_grid(end - begin);
  const size_t sum_end = n_sum / 4;
  switch (world) {
    case 2: GOF_LAUNCH("p2p_allreduce", st, k_p2p_allreduce<2><<<grid, 512, 0, st>>>(a, begin, end, sum_end)); break;
    case 4: GOF_LAUNCH("p2p_allreduce", st, k_p2p_allreduce<4><<<grid, 512, 0, st>>>(a, begin, end, sum_end)); break;
    case 8: GOF_LAUNCH("p2p_allreduce", st, k_p2p_allreduce<8><<<grid, 512, 0, st>>>(a, begin, end, sum_end)); break;
    default: GOF_LAUNCH("p2p_allreduce", st, k_p2p_allreduce_any<<<grid, 512, 0, st>>>(a, world, begin, end, sum_end)); break;
  }
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}
