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


// ---- tuning probes (tools/exchange_sweep.py): the SUM exchange with every launch parameter exposed.
// layout 0: grid-stride lattice (consecutive warps of the whole grid touch consecutive 512 bytes); layout 1: each CTA walks
// contiguous chunks of threads*U float4.  mode bit 0: reduce (ld_reduce / peer loads), bit 1: broadcast (st / peer stores).
template <int U>
__global__ void k_nvls_probe(float4* mc, size_t begin, size_t end, int layout, int mode, float4* sink) {
  const size_t T = blockDim.x, G = gridDim.x;
  const size_t inner = layout ? T : G * T;                      // distance between a thread's U elements
  const size_t outer = G * T * U;                               // distance between a thread's rounds
  size_t i = begin + (layout ? (size_t)blockIdx.x * T * U + threadIdx.x : (size_t)blockIdx.x * T + threadIdx.x);
  float4 keep = make_float4(0.f, 0.f, 0.f, 0.f);
  for (; i < end; i += outer) {
    float4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const size_t j = i + u * inner;
      v[u] = (j < end && (mode & 1)) ? mm_ld_add(mc + j) : make_float4(1.f, 1.f, 1.f, 1.f);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const size_t j = i + u * inner;
      if (j < end) { if (mode & 2) mm_st(mc + j, v[u]); else keep.x += v[u].x + v[u].w; }
    }
  }
  if (!(mode & 2) && keep.x == 123.456f) sink[0] = keep;
}

template <int W, int U>
__global__ void k_p2p_probe(const PeerPtrs a, size_t begin, size_t end, int layout) {
  const size_t T = blockDim.x, G = gridDim.x;
  const size_t inner = layout ? T : G * T, outer = G * T * U;
  size_t i = begin + (layout ? (size_t)blockIdx.x * T * U + threadIdx.x : (size_t)blockIdx.x * T + threadIdx.x);
  for (; i < end; i += outer) {
    float4 v[U][W];
#pragma unroll
    for (int u = 0; u < U; ++u)
#pragma unroll
      for (int r = 0; r < W; ++r) { const size_t j = i + u * inner; v[u][r] = j < end ? ld_cg(a.p[r] + j) : make_float4(0.f, 0.f, 0.f, 0.f); }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const size_t j = i + u * inner;
      float4 s = v[u][0];
#pragma unroll
      for (int r = 1; r < W; ++r) s = combine(s, v[u][r], true);
      if (j < end) {
#pragma unroll
        for (int r = 0; r < W; ++r) __stcg(a.p[r] + j, s);
      }
    }
  }
}

}  // namespace

// Peer access from the current device to `peer_device` (the device index, in THIS process, on which a peer bucket was
// mapped).  CUDA IPC mappings opened under the exporting device's context are not reachable from kernels of another
// device until this has been called once.  Idempotent.
extern "C" GOF_API int gof_enable_peer_access(int peer_device) {
  int cur = 0;
  GOF_CUDA_OK(cudaGetDevice(&cur));
  if (peer_device == cur) return GOF_OK;
  int can = 0;
  GOF_CUDA_OK(cudaDeviceCanAccessPeer(&can, cur, peer_device));
  if (!can) { gof_set_error("device %d cannot access device %d (no NVLink/PCIe peer path)", cur, peer_device); return GOF_E_INVALID; }
  const cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) { (void)cudaGetLastError(); return GOF_OK; }
  if (e != cudaSuccess) { gof_set_error("cudaDeviceEnablePeerAccess(%d): %s", peer_device, cudaGetErrorString(e)); return GOF_E_CUDA; }
  return GOF_OK;
}

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

// peers[r] = address (in THIS process) of rank r's bucket, r = 0..world-1; n = floats per bucket (multiple of 4,
// 16-byte aligned buffers).  Reduces this rank's slice; the caller provides the two cross-rank barriers.
extern "C" GOF_API int gof_p2p_allreduce_sum_f32(float* const* peers, int world, int rank, size_t n, void* stream) {
  return gof_p2p_allreduce_f32(peers, world, rank, n, n, stream);
}

static unsigned exchange_grid(size_t items) {
  static int sms = 0;
  if (!sms) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); if (sms <= 0) sms = 132; }
  const size_t want = (items + 511) / 512;
  return (unsigned)(want < (size_t)sms * 4 ? want : (size_t)sms * 4);
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

// Tuning probes (developer tools only; SUM over [n*rank/world, n*(rank+1)/world) of an n-float bucket).
extern "C" GOF_API int gof_nvls_probe(float* mc, int world, int rank, size_t n, int grid, int threads, int unroll, int layout, int mode, float* sink,
                                      void* stream) {
  if (!mc || world < 1 || (n & 3u) || grid < 1 || threads < 32 || threads > 1024) { gof_set_error("nvls_probe: bad arguments"); return GOF_E_INVALID; }
  const size_t n4 = n / 4, begin = n4 * (size_t)rank / (size_t)world, end = n4 * (size_t)(rank + 1) / (size_t)world;
  cudaStream_t st = (cudaStream_t)stream;
  float4* m = reinterpret_cast<float4*>(mc);
  float4* sk = reinterpret_cast<float4*>(sink);
  switch (unroll) {
    case 1: k_nvls_probe<1><<<grid, threads, 0, st>>>(m, begin, end, layout, mode, sk); break;
    case 2: k_nvls_probe<2><<<grid, threads, 0, st>>>(m, begin, end, layout, mode, sk); break;
    case 4: k_nvls_probe<4><<<grid, threads, 0, st>>>(m, begin, end, layout, mode, sk); break;
    case 8: k_nvls_probe<8><<<grid, threads, 0, st>>>(m, begin, end, layout, mode, sk); break;
    default: gof_set_error("nvls_probe: unroll 1, 2, 4 or 8"); return GOF_E_INVALID;
  }
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}
extern "C" GOF_API int gof_p2p_probe(float* const* peers, int world, int rank, size_t n, int grid, int threads, int unroll, int layout, void* stream) {
  if (!peers || (world != 2 && world != 4 && world != 8) || (n & 3u) || grid < 1 || threads < 32 || threads > 1024) {
    gof_set_error("p2p_probe: bad arguments"); return GOF_E_INVALID; }
  PeerPtrs a;
  for (int r = 0; r < GOF_MAX_PEERS; ++r) a.p[r] = reinterpret_cast<float4*>(r < world ? peers[r] : nullptr);
  const size_t n4 = n / 4, begin = n4 * (size_t)rank / (size_t)world, end = n4 * (size_t)(rank + 1) / (size_t)world;
  cudaStream_t st = (cudaStream_t)stream;
#define GOF_P2P_PROBE(W, U) k_p2p_probe<W, U><<<grid, threads, 0, st>>>(a, begin, end, layout)
  if (world == 2) { if (unroll == 1) GOF_P2P_PROBE(2, 1); else if (unroll == 2) GOF_P2P_PROBE(2, 2); else if (unroll == 4) GOF_P2P_PROBE(2, 4); else GOF_P2P_PROBE(2, 8); }
  else if (world == 4) { if (unroll == 1) GOF_P2P_PROBE(4, 1); else if (unroll == 2) GOF_P2P_PROBE(4, 2); else GOF_P2P_PROBE(4, 4); }
  else { if (unroll == 1) GOF_P2P_PROBE(8, 1); else GOF_P2P_PROBE(8, 2); }
#undef GOF_P2P_PROBE
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}
