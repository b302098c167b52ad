// tetra_points.cuh -- GaussianModel.get_tetra_points (scene/gaussian_model.py:433-463) and the module-level get_frustum_mask
// (:31-72) for one Gaussian / one point, host/device so that tests/hostmath can run it on the CPU (DESIGN §4.8).
//
// Every product, sum, difference and quotient of the reference's elementwise torch ops is rounded on its own (the tp_*
// helpers: __fmul_rn & co. on the device, plain operators on a host compiled with -ffp-contract=off), so that nvcc cannot
// contract them into FMAs.  The two matrix products the reference runs through cuBLAS (the box corners' bmm and the view
// transform's einsum) are FMA chains from zero in ascending inner index, what a GEMM inner loop does.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define TP_HD __host__ __device__ __forceinline__
#else
#define TP_HD static inline
#endif

// one view: world_view_transform (16 floats, row-major as stored), focal_x, focal_y, width, height
#define TP_VIEW_FLOATS 20

TP_HD float tp_mul(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
TP_HD float tp_add(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
TP_HD float tp_sub(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
TP_HD float tp_div(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}
TP_HD float tp_sqrt(float a) {
#if defined(__CUDA_ARCH__)
  return __fsqrt_rn(a);
#else
  return sqrtf(a);
#endif
}
// torch.max: a NaN operand wins (fmaxf would drop it)
TP_HD float tp_max_nan(float a, float b) { return (a != a || a > b) ? a : b; }

// Box corner k (0..7) of trimesh.creation.box() after `vertices *= 2`: signs (sx, sy, sz), sz fastest (DESIGN §4.8).
TP_HD float tp_corner_sign(int k, int axis) { return ((k >> (2 - axis)) & 1) ? 1.0f : -1.0f; }

// build_rotation (utils/general_utils.py:78-99) of the raw quaternion r, and s3 = scales * 3 with its NaN-propagating max.
TP_HD void tp_gaussian_frame(const float r[4], const float s[3], float R[9], float s3[3], float* point_scale) {
  const float norm = tp_sqrt(tp_add(tp_add(tp_add(tp_mul(r[0], r[0]), tp_mul(r[1], r[1])), tp_mul(r[2], r[2])), tp_mul(r[3], r[3])));
  const float w = tp_div(r[0], norm), x = tp_div(r[1], norm), y = tp_div(r[2], norm), z = tp_div(r[3], norm);
  R[0] = tp_sub(1.0f, tp_mul(2.0f, tp_add(tp_mul(y, y), tp_mul(z, z))));
  R[1] = tp_mul(2.0f, tp_sub(tp_mul(x, y), tp_mul(w, z)));
  R[2] = tp_mul(2.0f, tp_add(tp_mul(x, z), tp_mul(w, y)));
  R[3] = tp_mul(2.0f, tp_add(tp_mul(x, y), tp_mul(w, z)));
  R[4] = tp_sub(1.0f, tp_mul(2.0f, tp_add(tp_mul(x, x), tp_mul(z, z))));
  R[5] = tp_mul(2.0f, tp_sub(tp_mul(y, z), tp_mul(w, x)));
  R[6] = tp_mul(2.0f, tp_sub(tp_mul(x, z), tp_mul(w, y)));
  R[7] = tp_mul(2.0f, tp_add(tp_mul(y, z), tp_mul(w, x)));
  R[8] = tp_sub(1.0f, tp_mul(2.0f, tp_add(tp_mul(x, x), tp_mul(y, y))));
  for (int j = 0; j < 3; ++j) s3[j] = tp_mul(s[j], 3.0f);
  *point_scale = tp_max_nan(tp_max_nan(s3[0], s3[1]), s3[2]);
}

// corner k = bmm(R, signs * s3) + xyz: the 3-term product as an FMA chain from zero, then a separately rounded add
TP_HD void tp_corner(const float R[9], const float s3[3], const float xyz[3], int k, float out[3]) {
  float v[3];
  for (int j = 0; j < 3; ++j) v[j] = tp_corner_sign(k, j) * s3[j];   // exact: a sign flip
  for (int i = 0; i < 3; ++i) {
    float acc = 0.0f;
    for (int j = 0; j < 3; ++j) acc = fmaf(R[3 * i + j], v[j], acc);
    out[i] = tp_add(acc, xyz[i]);
  }
}

// Is p in view `vw`'s frustum?  W, H are those of views[0] (the reference's quirk), near/far already rounded to float32.
// The intrinsics product keeps its zero terms: a non-finite view coordinate makes z' NaN, so the point is never in.
TP_HD bool tp_in_view(const float p[3], const float* vw, float W, float H, float near, float far) {
  float vp[3];
  for (int b = 0; b < 3; ++b) {   // world_view_transform^T (x, y, z, 1): element [c][b] of the stored matrix is vw[4c + b]
    float acc = 0.0f;
    acc = fmaf(vw[b], p[0], acc);
    acc = fmaf(vw[4 + b], p[1], acc);
    acc = fmaf(vw[8 + b], p[2], acc);
    acc = fmaf(vw[12 + b], 1.0f, acc);
    vp[b] = acc;
  }
  const float fx = vw[16], fy = vw[17], cx = tp_mul(W, 0.5f), cy = tp_mul(H, 0.5f);
  const float un = fmaf(cx, vp[2], fmaf(0.0f, vp[1], fmaf(fx, vp[0], 0.0f)));
  const float vn = fmaf(cy, vp[2], fmaf(fy, vp[1], fmaf(0.0f, vp[0], 0.0f)));
  const float zp = fmaf(1.0f, vp[2], fmaf(0.0f, vp[1], fmaf(0.0f, vp[0], 0.0f)));
  const float u = tp_div(un, zp), v = tp_div(vn, zp), depth = vp[2];
  return depth >= near && depth <= far && u >= 0.0f && u <= tp_sub(W, 1.0f) && v >= 0.0f && v <= tp_sub(H, 1.0f);
}

// The first view, starting at `start` and wrapping around, whose frustum holds p; -1 when none does.
TP_HD int tp_first_view(const float p[3], const float* views, int n_views, int start, float near, float far) {
  const float W = views[18], H = views[19];
  for (int t = 0; t < n_views; ++t) {
    int c = start + t;
    if (c >= n_views) c -= n_views;
    if (tp_in_view(p, views + (size_t)c * TP_VIEW_FLOATS, W, H, near, far)) return c;
  }
  return -1;
}
