// tests/hostmath/tetra_points_host.cpp -- TEST INFRASTRUCTURE: csrc/tetra_points.cuh compiled for the host (-ffp-contract=off),
// walked in the same order as the CUDA kernels (the centre first, each corner's view search starting where the last hit was).
#include <stddef.h>

#include "../../gaussian-opacity-fields_b200/csrc/tetra_points.cuh"

extern "C" void hm_tp_frame(int P, const float* rotations, const float* scales, float* R, float* s3, float* point_scale) {
  for (int g = 0; g < P; ++g) tp_gaussian_frame(rotations + 4 * (size_t)g, scales + 3 * (size_t)g, R + 9 * (size_t)g, s3 + 3 * (size_t)g, point_scale + g);
}

extern "C" void hm_tp_points(int P, const float* xyz, const float* scales, const float* rotations, int n_views, const float* views,
                             float near, float far, float* out_points, float* out_scale, unsigned char* out_mask) {
  for (int g = 0; g < P; ++g) {
    float R[9], s3[3], ps;
    tp_gaussian_frame(rotations + 4 * (size_t)g, scales + 3 * (size_t)g, R, s3, &ps);
    const float* c = xyz + 3 * (size_t)g;
    const size_t ci = 8 * (size_t)P + g;
    for (int i = 0; i < 3; ++i) out_points[3 * ci + i] = c[i];
    out_scale[ci] = ps;
    int hit = tp_first_view(c, views, n_views, 0, near, far);
    out_mask[ci] = hit >= 0;
    int start = hit >= 0 ? hit : 0;
    for (int k = 0; k < 8; ++k) {
      const size_t pi = 8 * (size_t)g + k;
      tp_corner(R, s3, c, k, out_points + 3 * pi);
      out_scale[pi] = ps;
      hit = tp_first_view(out_points + 3 * pi, views, n_views, start, near, far);
      out_mask[pi] = hit >= 0;
      if (hit >= 0) start = hit;
    }
  }
}

extern "C" void hm_tp_mask(long long N, const float* points, int n_views, const float* views, float near, float far, unsigned char* out_mask) {
  for (long long i = 0; i < N; ++i) out_mask[i] = tp_first_view(points + 3 * i, views, n_views, 0, near, far) >= 0;
}

extern "C" float hm_tp_corner_sign(int k, int axis) { return tp_corner_sign(k, axis); }
