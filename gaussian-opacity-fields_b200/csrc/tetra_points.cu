// tetra_points.cu -- kernels and C ABI of GaussianModel.get_tetra_points and get_frustum_mask (see tetra_points.cuh;
// DESIGN §4.8).  One thread per Gaussian generates its 8 box corners and its centre, with their scales and frustum flags, in
// one pass: 153 bytes written per Gaussian whatever the number of views, where the reference materialises ~40 bytes per
// (view, point).  The compaction (`points[mask]`) is left to the caller, as the reference does it.
#include "gof_common.cuh"
#include "tetra_points.cuh"

namespace {

__global__ void __launch_bounds__(256) k_tetra_points(int P, const float* __restrict__ xyz, const float* __restrict__ scales,
                                                      const float4* __restrict__ rotations, int n_views,
                                                      const float* __restrict__ views, float near, float far,
                                                      float* __restrict__ out_points, float* __restrict__ out_scale,
                                                      uint8_t* __restrict__ out_mask) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= P) return;
  const float4 q = rotations[g];
  const float r[4] = {q.x, q.y, q.z, q.w};
  const float s[3] = {scales[3 * (size_t)g], scales[3 * (size_t)g + 1], scales[3 * (size_t)g + 2]};
  const float c[3] = {xyz[3 * (size_t)g], xyz[3 * (size_t)g + 1], xyz[3 * (size_t)g + 2]};
  float R[9], s3[3], ps;
  tp_gaussian_frame(r, s, R, s3, &ps);

  // the centre first: its view is where the corners' search starts (a Gaussian's corners are usually seen by the same view)
  const size_t ci = 8 * (size_t)P + g;
  out_points[3 * ci] = c[0];
  out_points[3 * ci + 1] = c[1];
  out_points[3 * ci + 2] = c[2];
  out_scale[ci] = ps;
  int hit = tp_first_view(c, views, n_views, 0, near, far);
  out_mask[ci] = hit >= 0;
  int start = hit >= 0 ? hit : 0;
#pragma unroll 1
  for (int k = 0; k < 8; ++k) {
    float p[3];
    tp_corner(R, s3, c, k, p);
    const size_t pi = 8 * (size_t)g + k;
    out_points[3 * pi] = p[0];
    out_points[3 * pi + 1] = p[1];
    out_points[3 * pi + 2] = p[2];
    out_scale[pi] = ps;
    hit = tp_first_view(p, views, n_views, start, near, far);
    out_mask[pi] = hit >= 0;
    if (hit >= 0) start = hit;
  }
}

__global__ void __launch_bounds__(256) k_frustum_mask(int64_t N, const float* __restrict__ points, int n_views,
                                                      const float* __restrict__ views, float near, float far,
                                                      uint8_t* __restrict__ out_mask) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const float p[3] = {points[3 * i], points[3 * i + 1], points[3 * i + 2]};
  out_mask[i] = tp_first_view(p, views, n_views, 0, near, far) >= 0;
}

}  // namespace

extern "C" GOF_API int gof_tetra_points(int P, const float* xyz, const float* scales, const float* rotations, int n_views,
                                        const float* views, float near, float far, float* out_points, float* out_scale,
                                        unsigned char* out_mask, void* stream) {
  if (P < 0 || 9ull * (unsigned long long)P > 0xFFFFFFFFull || n_views < 1) {
    gof_set_error("tetra_points: bad sizes (P = %d, n_views = %d; need 0 <= 9 P < 2^32 and at least one view)", P, n_views);
    return GOF_E_INVALID;
  }
  if (P == 0) return GOF_OK;
  if (!xyz || !scales || !rotations || !views || !out_points || !out_scale || !out_mask) {
    gof_set_error("tetra_points: NULL pointer");
    return GOF_E_INVALID;
  }
  if (reinterpret_cast<uintptr_t>(rotations) & 15) {
    gof_set_error("tetra_points: rotations must be 16-byte aligned (they are read as float4)");
    return GOF_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned blocks = (unsigned)((P + 255) / 256);
  GOF_LAUNCH("tetra_points", st,
             k_tetra_points<<<blocks, 256, 0, st>>>(P, xyz, scales, reinterpret_cast<const float4*>(rotations), n_views, views, near,
                                                    far, out_points, out_scale, out_mask));
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}

extern "C" GOF_API int gof_frustum_mask(int64_t N, const float* points, int n_views, const float* views, float near, float far,
                                        unsigned char* out_mask, void* stream) {
  if (N < 0 || n_views < 1) {
    gof_set_error("frustum_mask: bad sizes (N = %lld, n_views = %d; need N >= 0 and at least one view)", (long long)N, n_views);
    return GOF_E_INVALID;
  }
  if (N == 0) return GOF_OK;
  if (!points || !views || !out_mask) {
    gof_set_error("frustum_mask: NULL pointer");
    return GOF_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned long long blocks = ((unsigned long long)N + 255) / 256;
  if (blocks > 0x7FFFFFFFull) {
    gof_set_error("frustum_mask: N = %lld exceeds the grid", (long long)N);
    return GOF_E_INVALID;
  }
  GOF_LAUNCH("frustum_mask", st,
             k_frustum_mask<<<(unsigned)blocks, 256, 0, st>>>(N, points, n_views, views, near, far, out_mask));
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}
