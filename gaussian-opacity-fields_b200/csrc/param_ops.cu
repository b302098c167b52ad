// param_ops.cu -- kernels and C ABI of the parameter prologue / epilogue (see param_ops.cuh).  The per-Gaussian arithmetic
// is verified on the CPU (tests/test_param_ops_host.py); these kernels against fp64 restatements on the GPU at up to 10^6
// Gaussians and 59 M Adam elements (tests/test_gpu_train_step.py).
#include <math.h>
#include <stdint.h>

#include "gof_common.cuh"
#include "param_ops.cuh"

namespace {

// the activation kernels move rotations as float4
inline bool misaligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) != 0; }

__global__ void __launch_bounds__(256) k_activate(int P, const float* __restrict__ s_raw, const float* __restrict__ q,
                                                  const float* __restrict__ o_raw, const float* __restrict__ filt,
                                                  float* __restrict__ scales, float* __restrict__ rot, float* __restrict__ op) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const float s[3] = {s_raw[3 * i], s_raw[3 * i + 1], s_raw[3 * i + 2]};
  const float4 qq = reinterpret_cast<const float4*>(q)[i];
  const float qa[4] = {qq.x, qq.y, qq.z, qq.w};
  const PoActivated a = po_activate(s, qa, o_raw[i], filt[i]);
  scales[3 * i] = a.scales[0]; scales[3 * i + 1] = a.scales[1]; scales[3 * i + 2] = a.scales[2];
  reinterpret_cast<float4*>(rot)[i] = make_float4(a.rot[0], a.rot[1], a.rot[2], a.rot[3]);
  op[i] = a.opacity;
}

// shs[i] = cat(f_dc[i] (3 floats), f_rest[i] (3*Mr floats)); backward splits the same way
__global__ void __launch_bounds__(256) k_cat_sh(size_t n, int Mr, const float* __restrict__ f_dc, const float* __restrict__ f_rest,
                                                float* __restrict__ shs) {
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int row = 3 * (Mr + 1);
  const size_t i = e / row;
  const int j = (int)(e - i * row);
  shs[e] = j < 3 ? f_dc[3 * i + j] : f_rest[(size_t)3 * Mr * i + (j - 3)];
}
__global__ void __launch_bounds__(256) k_split_sh(size_t n, int Mr, const float* __restrict__ g_shs, float* __restrict__ d_dc,
                                                  float* __restrict__ d_rest) {
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int row = 3 * (Mr + 1);
  const size_t i = e / row;
  const int j = (int)(e - i * row);
  if (j < 3) d_dc[3 * i + j] = g_shs[e];
  else d_rest[(size_t)3 * Mr * i + (j - 3)] = g_shs[e];
}

__global__ void __launch_bounds__(256) k_activate_backward(int P, const float* __restrict__ s_raw, const float* __restrict__ q,
                                                           const float* __restrict__ o_raw, const float* __restrict__ filt,
                                                           const float* __restrict__ g_scales, const float* __restrict__ g_rot,
                                                           const float* __restrict__ g_op, float* __restrict__ d_s,
                                                           float* __restrict__ d_q, float* __restrict__ d_o) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const float s[3] = {s_raw[3 * i], s_raw[3 * i + 1], s_raw[3 * i + 2]};
  const float gs[3] = {g_scales[3 * i], g_scales[3 * i + 1], g_scales[3 * i + 2]};
  const float4 qq = reinterpret_cast<const float4*>(q)[i], gq = reinterpret_cast<const float4*>(g_rot)[i];
  const float qa[4] = {qq.x, qq.y, qq.z, qq.w}, gr[4] = {gq.x, gq.y, gq.z, gq.w};
  float ds[3], dq[4], dop;
  po_activate_backward(s, qa, o_raw[i], filt[i], gs, gr, g_op[i], ds, dq, &dop);
  d_s[3 * i] = ds[0]; d_s[3 * i + 1] = ds[1]; d_s[3 * i + 2] = ds[2];
  reinterpret_cast<float4*>(d_q)[i] = make_float4(dq[0], dq[1], dq[2], dq[3]);
  d_o[i] = dop;
}

__global__ void __launch_bounds__(256) k_adam(size_t n, float* __restrict__ p, float* __restrict__ m, float* __restrict__ v,
                                              const float* __restrict__ g, float beta2, float omb1, float omb2, float eps,
                                              float step_size, float bias2_sqrt) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  po_adam(p + i, m + i, v + i, g[i], beta2, omb1, omb2, eps, step_size, bias2_sqrt);
}

inline unsigned blocks_for(size_t n) { return (unsigned)((n + 255) / 256); }

}  // namespace

// scene/gaussian_model.py:152-194.  All pointers device, fp32; rotations 16-byte aligned.  M_rest = SH coefficients in f_rest (15).
extern "C" GOF_API int gof_activate_params(int P, int M_rest, const float* scaling_raw, const float* rotation_raw, const float* opacity_raw,
                                           const float* filter_3D, const float* features_dc, const float* features_rest, float* scales,
                                           float* rotations, float* opacities, float* shs, void* stream) {
  if (P < 0 || M_rest < 0) { gof_set_error("activate_params: bad sizes"); return GOF_E_INVALID; }
  if (P == 0) return GOF_OK;
  if (!scaling_raw || !rotation_raw || !opacity_raw || !filter_3D || !scales || !rotations || !opacities) {
    gof_set_error("activate_params: NULL argument");
    return GOF_E_INVALID;
  }
  if (misaligned16(rotation_raw) || misaligned16(rotations)) {
    gof_set_error("activate_params: rotations must be 16-byte aligned");
    return GOF_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  GOF_LAUNCH("activate_params", st, k_activate<<<blocks_for((size_t)P), 256, 0, st>>>(P, scaling_raw, rotation_raw, opacity_raw, filter_3D,
                                                                                        scales, rotations, opacities));
  GOF_LAUNCH_CHECK(false, st);
  if (shs) {
    if (!features_dc || (M_rest > 0 && !features_rest)) { gof_set_error("activate_params: features missing"); return GOF_E_INVALID; }
    const size_t n = (size_t)P * 3 * (M_rest + 1);
    GOF_LAUNCH("cat_sh", st, k_cat_sh<<<blocks_for(n), 256, 0, st>>>(n, M_rest, features_dc, features_rest, shs));
    GOF_LAUNCH_CHECK(false, st);
  }
  return GOF_OK;
}

extern "C" GOF_API int gof_activate_params_backward(int P, int M_rest, const float* scaling_raw, const float* rotation_raw,
                                                    const float* opacity_raw, const float* filter_3D, const float* g_scales,
                                                    const float* g_rotations, const float* g_opacities, const float* g_shs,
                                                    float* d_scaling_raw, float* d_rotation_raw, float* d_opacity_raw,
                                                    float* d_features_dc, float* d_features_rest, void* stream) {
  if (P < 0 || M_rest < 0) { gof_set_error("activate_params_backward: bad sizes"); return GOF_E_INVALID; }
  if (P == 0) return GOF_OK;
  if (!scaling_raw || !rotation_raw || !opacity_raw || !filter_3D || !g_scales || !g_rotations || !g_opacities || !d_scaling_raw ||
      !d_rotation_raw || !d_opacity_raw) {
    gof_set_error("activate_params_backward: NULL argument");
    return GOF_E_INVALID;
  }
  if (misaligned16(rotation_raw) || misaligned16(g_rotations) || misaligned16(d_rotation_raw)) {
    gof_set_error("activate_params_backward: rotations must be 16-byte aligned");
    return GOF_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  GOF_LAUNCH("activate_params_bwd", st, k_activate_backward<<<blocks_for((size_t)P), 256, 0, st>>>(
      P, scaling_raw, rotation_raw, opacity_raw, filter_3D, g_scales, g_rotations, g_opacities, d_scaling_raw, d_rotation_raw, d_opacity_raw));
  GOF_LAUNCH_CHECK(false, st);
  if (g_shs) {
    if (!d_features_dc || (M_rest > 0 && !d_features_rest)) { gof_set_error("activate_params_backward: feature outputs missing"); return GOF_E_INVALID; }
    const size_t n = (size_t)P * 3 * (M_rest + 1);
    GOF_LAUNCH("split_sh", st, k_split_sh<<<blocks_for(n), 256, 0, st>>>(n, M_rest, g_shs, d_features_dc, d_features_rest));
    GOF_LAUNCH_CHECK(false, st);
  }
  return GOF_OK;
}

// One torch.optim.Adam step (gaussian_model.py:360 uses eps = 1e-15) on n floats; `step` = step count after the increment (>= 1).
extern "C" GOF_API int gof_adam_step(size_t n, float* param, float* exp_avg, float* exp_avg_sq, const float* grad, double lr, double beta1,
                                     double beta2, double eps, int step, void* stream) {
  if (step < 1 || !(beta1 >= 0.0 && beta1 < 1.0) || !(beta2 >= 0.0 && beta2 < 1.0)) { gof_set_error("adam_step: bad hyper-parameters"); return GOF_E_INVALID; }
  if (n == 0) return GOF_OK;
  if (!param || !exp_avg || !exp_avg_sq || !grad) { gof_set_error("adam_step: NULL argument"); return GOF_E_INVALID; }
  const double bias1 = 1.0 - pow(beta1, (double)step), bias2 = 1.0 - pow(beta2, (double)step);
  cudaStream_t st = (cudaStream_t)stream;
  GOF_LAUNCH("adam_step", st, k_adam<<<blocks_for(n), 256, 0, st>>>(n, param, exp_avg, exp_avg_sq, grad, (float)beta2, (float)(1.0 - beta1),
                                                                      (float)(1.0 - beta2), (float)eps, (float)(lr / bias1), (float)sqrt(bias2)));
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}
