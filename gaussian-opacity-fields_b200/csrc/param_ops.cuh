// param_ops.cuh -- the parameter prologue / epilogue around the rasterizer (SURVEY.md 8(f) rank 2; reference:
// scene/gaussian_model.py:152-194 activations with the 3D filter, :360 torch.optim.Adam(eps=1e-15)).
// A caller of the rasterizer.  Per-Gaussian functions are host/device so that tests/hostmath can run this very source on the
// CPU against golden vectors generated from the reference's own Python; tests/test_gpu_train_step.py checks the CUDA kernels
// against fp64 restatements of the formulas below.
//
//   activate:           raw (log-scale[3], quaternion[4], opacity logit, filter_3D, f_dc[3], f_rest[15*3])
//                       -> scales = sqrt(exp(s)^2 + f^2), rotations = q / max(|q|, 1e-12),
//                          opacity = sigmoid(o) * sqrt(prod exp(s)^2 / prod (exp(s)^2 + f^2)), shs = cat(f_dc, f_rest)
//   activate_backward:  gradients w.r.t. those four outputs (what the rasterizer's backward returns) -> raw gradients
//   adam:               one element of torch.optim.Adam's step (no weight decay, no amsgrad)
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define PO_HD __host__ __device__ __forceinline__
#else
#define PO_HD static inline
#endif

struct PoActivated { float scales[3]; float rot[4]; float opacity; };

PO_HD PoActivated po_activate(const float* s_raw, const float* q, float o_raw, float f) {
  PoActivated a;
  const float f2 = f * f;
  float coef2 = 1.0f, det1 = 1.0f, det2 = 1.0f;
  (void)coef2;
  for (int k = 0; k < 3; ++k) {
    const float e = expf(s_raw[k]);                    // scaling_activation = torch.exp
    const float e2 = e * e, S2 = e2 + f2;
    a.scales[k] = sqrtf(S2);                           // get_scaling_with_3D_filter
    det1 *= e2; det2 *= S2;
  }
  const float coef = sqrtf(det1 / det2);               // get_opacity_with_3D_filter
  a.opacity = (1.0f / (1.0f + expf(-o_raw))) * coef;
  const float len = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  const float d = len > 1e-12f ? len : 1e-12f;         // F.normalize eps
  for (int k = 0; k < 4; ++k) a.rot[k] = q[k] / d;
  return a;
}

// gradients w.r.t. the raw parameters from gradients w.r.t. scales[3], rot[4], opacity
PO_HD void po_activate_backward(const float* s_raw, const float* q, float o_raw, float f, const float* g_scales, const float* g_rot,
                                float g_opacity, float* d_s_raw, float* d_q, float* d_o_raw) {
  const float f2 = f * f;
  float e2[3], S2[3], det1 = 1.0f, det2 = 1.0f;
  for (int k = 0; k < 3; ++k) {
    const float e = expf(s_raw[k]);
    e2[k] = e * e; S2[k] = e2[k] + f2;
    det1 *= e2[k]; det2 *= S2[k];
  }
  const float coef = sqrtf(det1 / det2);
  const float sg = 1.0f / (1.0f + expf(-o_raw));
  *d_o_raw = g_opacity * coef * sg * (1.0f - sg);
  for (int k = 0; k < 3; ++k) {
    // d sqrt(e^2 + f^2) / d s_raw = e^2 / S ;   d ln coef / d s_raw = 1 - e^2 / S^2
    d_s_raw[k] = g_scales[k] * e2[k] / sqrtf(S2[k]) + g_opacity * sg * coef * (1.0f - e2[k] / S2[k]);
  }
  const float len = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  if (len > 1e-12f) {
    float u[4], ug = 0.f;
    for (int k = 0; k < 4; ++k) { u[k] = q[k] / len; ug += u[k] * g_rot[k]; }
    for (int k = 0; k < 4; ++k) d_q[k] = (g_rot[k] - u[k] * ug) / len;
  } else {
    for (int k = 0; k < 4; ++k) d_q[k] = g_rot[k] / 1e-12f;
  }
}

// torch.optim.Adam, one element.  The scalars are formed by the HOST in double like torch does (Python floats) and
// rounded once: omb1 = 1-beta1, omb2 = 1-beta2, step_size = lr / (1 - beta1^t), bias2_sqrt = sqrt(1 - beta2^t), t = step count
// after the increment.  m <- lerp(m, g, 1-beta1);  v <- beta2 v + (1-beta2) g^2;  p <- p - step_size * m / (sqrt(v)/bias2_sqrt + eps)
PO_HD void po_adam(float* p, float* m, float* v, float g, float beta2, float omb1, float omb2, float eps, float step_size, float bias2_sqrt) {
  const float mm = *m + omb1 * (g - *m);
  const float vv = beta2 * (*v) + omb2 * g * g;
  const float denom = sqrtf(vv) / bias2_sqrt + eps;
  *p = *p - step_size * (mm / denom);
  *m = mm; *v = vv;
}
