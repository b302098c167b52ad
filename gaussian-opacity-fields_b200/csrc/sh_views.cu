// sh_views.cu -- the SH-gradient half of the view-parallel exchange (SURVEY.md 8(e); no reference counterpart).
//
// Of the 64 floats per Gaussian a view-parallel step has to combine across GPUs, 48 are dL_dsh -- and one view's dL_dsh is an
// outer product: dL_dsh[k][c] = w_k(dir) * dL_dRGB[c] (backward.cu:45-139), dir = normalize(mean - camera centre).  Every
// rank holds all means and can learn every rank's camera centre, so the ranks only need each other's dL_dRGB: 3 floats per
// Gaussian and view instead of an all-reduce over 48.  This kernel forms sum_v w(dir_v) (x) rgb_v for all views v, in rank
// order and with the products rounded before the additions -- bit-identical to adding the per-view dL_dsh tensors that
// k_preprocess_backward would have written (it evaluates the same gof_sh_grad_weights).  The view records are read through
// a pointer per view: local memory after an NCCL all-gather, or the peers' buckets themselves over NVLink.
#include "gof_common.cuh"
#include "gof_math.cuh"

namespace {

constexpr int SHV_THREADS = 128;
constexpr int SHV_ROW = 49;      // 48 floats per Gaussian + 1 pad
constexpr int SHV_MAX_VIEWS = 16;

struct ShvArgs {
  int P, M, n_views;
  const float* means3D;
  const float* slot[SHV_MAX_VIEWS];
  float* dL_dsh;
};

// NV: compile-time bound of the view loop (2, 4, 8 or 16 >= n_views).  ALL views' dL_dRGB of a Gaussian are requested before the
// first one is used: the records may sit in peer memory, and a loop that loads, computes, loads ... pays an NVLink round trip per
// view (measured at 8 GPUs: 0.55 ms for the expansion alone, against 0.13 ms of link time for its 84 MB).
template <int NV>
__global__ void __launch_bounds__(SHV_THREADS) k_sh_grad_from_views(const ShvArgs a) {
  __shared__ float s_out[SHV_THREADS / 32][32 * SHV_ROW];
  __shared__ float s_cam[SHV_MAX_VIEWS][4];
  if (threadIdx.x < a.n_views * 4) s_cam[threadIdx.x >> 2][threadIdx.x & 3] = __ldcg(a.slot[threadIdx.x >> 2] + (threadIdx.x & 3));
  __syncthreads();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float acc[48];
#pragma unroll
  for (int k = 0; k < 48; ++k) acc[k] = 0.f;
  const size_t plane = GOF_SH_PLANE(a.P);
  if (idx < a.P) {
    float rgb[NV][3];
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      rgb[v][0] = rgb[v][1] = rgb[v][2] = 0.f;
      if (v < a.n_views) {
        // three colour PLANES: a warp's load is one contiguous 128 bytes.  (Interleaved [P][3] records made every scalar load
        // touch all twelve sectors of the warp's 384 bytes -- three times the NVLink traffic when the record is a peer's.)
        const float* p = a.slot[v] + GOF_SH_SLOT_HEADER + idx;
        rgb[v][0] = __ldcg(p); rgb[v][1] = __ldcg(p + plane); rgb[v][2] = __ldcg(p + 2 * plane);   // L2 only: may be a peer's memory
      }
    }
    const float mx = a.means3D[3 * (size_t)idx], my = a.means3D[3 * (size_t)idx + 1], mz = a.means3D[3 * (size_t)idx + 2];
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      const float r = rgb[v][0], g = rgb[v][1], b = rgb[v][2];
      if (v >= a.n_views || (r == 0.f && g == 0.f && b == 0.f)) continue;   // not seen by view v (or clamped in all channels): adds +0
      const int D = (int)s_cam[v][3];
      float x, y, z;   // the direction exactly as k_preprocess_backward forms it
      gof_sh_view_dir(mx, my, mz, s_cam[v][0], s_cam[v][1], s_cam[v][2], &x, &y, &z);
      float w[16];
      gof_sh_grad_weights(D, x, y, z, w);
      const int nk = (D + 1) * (D + 1);
#pragma unroll
      for (int k = 0; k < 16; ++k)
        if (k < nk) {
          acc[3 * k] = __fadd_rn(acc[3 * k], __fmul_rn(w[k], r));
          acc[3 * k + 1] = __fadd_rn(acc[3 * k + 1], __fmul_rn(w[k], g));
          acc[3 * k + 2] = __fadd_rn(acc[3 * k + 2], __fmul_rn(w[k], b));
        }
    }
  }
  float* mine = &s_out[warp][lane * SHV_ROW];
#pragma unroll
  for (int k = 0; k < 48; ++k) mine[k] = acc[k];
  __syncwarp();
  // the warp's 32 consecutive Gaussians leave as one contiguous block
  const int row = a.M * 3;
  const size_t g0 = (size_t)blockIdx.x * blockDim.x + (size_t)warp * 32;
  const int in_range = (int)min((size_t)32, (size_t)a.P > g0 ? (size_t)a.P - g0 : (size_t)0);
  if (a.M == 16) {
    float4* dst = reinterpret_cast<float4*>(a.dL_dsh + g0 * 48);
#pragma unroll 4
    for (int i = lane; i < in_range * 12; i += 32) {
      const int g = i / 12, j = (i - g * 12) * 4;
      const float* r = &s_out[warp][g * SHV_ROW + j];
      dst[i] = make_float4(r[0], r[1], r[2], r[3]);
    }
  } else {
    for (int i = lane; i < in_range * row; i += 32) {
      const int g = i / row, j = i - g * row;
      a.dL_dsh[(g0 + g) * (size_t)row + j] = j < 48 ? s_out[warp][g * SHV_ROW + j] : 0.f;
    }
  }
}

}  // namespace

extern "C" GOF_API int gof_sh_grad_from_views(int P, int M, int n_views, const float* means3D, const float* const* slots, float* dL_dsh,
                                              void* stream) {
  if (P < 0 || M < 1 || M > 16 || n_views < 1 || n_views > SHV_MAX_VIEWS || !slots) {
    gof_set_error("sh_grad_from_views: bad arguments (1 <= M <= 16, 1 <= n_views <= %d)", SHV_MAX_VIEWS);
    return GOF_E_INVALID;
  }
  if (P == 0) return GOF_OK;
  if (!means3D || !dL_dsh || (reinterpret_cast<uintptr_t>(dL_dsh) & 15u)) { gof_set_error("sh_grad_from_views: NULL or unaligned argument"); return GOF_E_INVALID; }
  ShvArgs a{};
  a.P = P; a.M = M; a.n_views = n_views; a.means3D = means3D; a.dL_dsh = dL_dsh;
  for (int v = 0; v < SHV_MAX_VIEWS; ++v) a.slot[v] = v < n_views ? slots[v] : nullptr;
  for (int v = 0; v < n_views; ++v)
    if (!a.slot[v]) { gof_set_error("sh_grad_from_views: NULL view record"); return GOF_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = (P + SHV_THREADS - 1) / SHV_THREADS;
  if (n_views <= 2) { GOF_LAUNCH("sh_grad_from_views", st, k_sh_grad_from_views<2><<<grid, SHV_THREADS, 0, st>>>(a)); }
  else if (n_views <= 4) { GOF_LAUNCH("sh_grad_from_views", st, k_sh_grad_from_views<4><<<grid, SHV_THREADS, 0, st>>>(a)); }
  else if (n_views <= 8) { GOF_LAUNCH("sh_grad_from_views", st, k_sh_grad_from_views<8><<<grid, SHV_THREADS, 0, st>>>(a)); }
  else { GOF_LAUNCH("sh_grad_from_views", st, k_sh_grad_from_views<16><<<grid, SHV_THREADS, 0, st>>>(a)); }
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}
