// densify.cu -- GaussianModel.densify_and_prune (scene/gaussian_model.py:631-707 with its helpers :549-629) as three kernels
// (SURVEY.md 8(f) rank 4; a caller of the rasterizer: it consumes the densification statistics the backward accumulates).
//
// The reference runs clone -> split -> prune as ~60 torch ops with three rounds of boolean-mask re-allocation of every parameter
// and optimizer-state tensor.  Their NET effect on Gaussian i is a function of i alone:
//   sel    = grad_i >= max_grad  or  grad_abs_i >= Q                         (grads = accumulators / denom, NaN -> 0)
//   clone  = sel and max(exp(scaling_i)) <= percent_dense * extent           -> one new Gaussian, position re-sampled
//   split  = sel and max(exp(scaling_i)) >  percent_dense * extent           -> two new Gaussians (scale / 1.6), the original removed
//   prune  = sigmoid(opacity) < min_opacity  or  (max_screen_size and max scale > 0.1 * extent)     applied to EVERYTHING,
//            new Gaussians included (max_radii2D has just been reset to zero, so the screen-size term never fires)
// and the surviving rows end up in the order  [kept originals | clones | first split children | second split children],
// each block in ascending source index.  So: one kernel decides the four keep-flags of every Gaussian, four scans turn them
// into output rows, one kernel builds (source index, kind) per output row and the new positions / scales, and every parameter and
// Adam-state tensor is rebuilt by ONE row gather (new rows of the Adam states are zero, like cat_tensors_to_optimizer's).
#include <math.h>

#include "gof_common.cuh"

namespace {

struct PlanArgs {
  int P;
  const float* accum;       // xyz_gradient_accum [P]
  const float* accum_abs;   // xyz_gradient_accum_abs [P]
  const float* denom;       // [P]
  const float* scaling;     // raw (log) scaling [P,3]
  const float* opacity;     // raw (logit) opacity [P]
  float max_grad, abs_threshold, dense_extent, min_opacity, prune_scale;   // prune_scale <= 0: no world-size pruning
  uint32_t* flags;          // [4][P]: kept original | clone | split child 1 | split child 2
};

// A split child's raw scaling, scaling_inverse_activation(get_scaling / (0.8 * N)) with N = 2 (gaussian_model.py:649): torch
// divides a CUDA tensor by a Python scalar as a product with the scalar's float reciprocal, and 1 / 1.6f rounds to 0.625f.
__device__ __forceinline__ float child_raw_scaling(float s) { return logf(s * 0.625f); }

__global__ void __launch_bounds__(256) k_densify_plan(const PlanArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.P) return;
  float g = a.accum[i] / a.denom[i], ga = a.accum_abs[i] / a.denom[i];
  if (g != g) g = 0.f;                                   // grads[grads.isnan()] = 0.0
  if (ga != ga) ga = 0.f;
  const bool sel = (g >= a.max_grad) || (ga >= a.abs_threshold);
  const float s0 = expf(a.scaling[3 * i]), s1 = expf(a.scaling[3 * i + 1]), s2 = expf(a.scaling[3 * i + 2]);
  const float smax = fmaxf(fmaxf(s0, s1), s2);
  const bool clone = sel && smax <= a.dense_extent;
  const bool split = sel && smax > a.dense_extent;
  const float op = 1.0f / (1.0f + expf(-a.opacity[i]));
  const bool low = op < a.min_opacity;
  const bool prune_self = low || (a.prune_scale > 0.f && smax > a.prune_scale);
  // a child is pruned on the scale it is stored with, read back: exp(log(s * 0.625f)), which can differ from s / 1.6f
  const bool prune_child = low || (split && a.prune_scale > 0.f &&
                                   fmaxf(fmaxf(expf(child_raw_scaling(s0)), expf(child_raw_scaling(s1))), expf(child_raw_scaling(s2))) > a.prune_scale);
  a.flags[i] = (!split && !prune_self) ? 1u : 0u;
  a.flags[(size_t)a.P + i] = (clone && !prune_self) ? 1u : 0u;
  const uint32_t c = (split && !prune_child) ? 1u : 0u;
  a.flags[2 * (size_t)a.P + i] = c;
  a.flags[3 * (size_t)a.P + i] = c;
}

// Philox-4x32-10 keyed by (seed, Gaussian, copy): the library's own counter-based generator (torch.normal's stream cannot be
// reproduced outside torch; the sampling is statistical in the reference as well)
__device__ __forceinline__ void philox(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t* out) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t h0 = __umulhi(0xD2511F53u, c0), l0 = 0xD2511F53u * c0;
    const uint32_t h1 = __umulhi(0xCD9E8D57u, c2), l1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = h1 ^ c1 ^ k0, n1 = l1, n2 = h0 ^ c3 ^ k1, n3 = l0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
__device__ __forceinline__ float u01(uint32_t x) { return ((float)(x >> 8) + 0.5f) * (1.0f / 16777216.0f); }   // (0,1)

struct EmitArgs {
  int P;
  const uint32_t* flags;     // [4][P]
  const uint32_t* offsets;   // [4][P] exclusive scans of the four flag rows
  uint32_t base[4];          // first output row of each block
  const float* xyz;          // [P,3]
  const float* scaling;      // raw [P,3]
  const float* rotation;     // raw [P,4]
  const float* noise;        // optional [3][P][3] standard-normal samples (clone, child 1, child 2); NULL: Philox(seed)
  unsigned long long seed;
  int32_t* src;              // [N] source Gaussian of every output row
  unsigned char* kind;       // [N] 0 kept original, 1 clone, 2 / 3 split children
  float* new_xyz;            // [N,3]
  float* new_scaling;        // [N,3] raw
};

__global__ void __launch_bounds__(256) k_densify_emit(const EmitArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.P) return;
  const float px = a.xyz[3 * i], py = a.xyz[3 * i + 1], pz = a.xyz[3 * i + 2];
  const float l0 = a.scaling[3 * i], l1 = a.scaling[3 * i + 1], l2 = a.scaling[3 * i + 2];
  bool any_new = false;
#pragma unroll
  for (int k = 1; k < 4; ++k) any_new |= a.flags[(size_t)k * a.P + i] != 0u;
  float R[9] = {1.f, 0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f, 1.f};
  float s0 = 0.f, s1 = 0.f, s2 = 0.f;
  if (any_new) {   // build_rotation (utils/general_utils.py:78-99) normalises the raw quaternion
    float r = a.rotation[4 * i], x = a.rotation[4 * i + 1], y = a.rotation[4 * i + 2], z = a.rotation[4 * i + 3];
    const float inv = 1.0f / sqrtf(r * r + x * x + y * y + z * z);
    r *= inv; x *= inv; y *= inv; z *= inv;
    R[0] = 1.f - 2.f * (y * y + z * z); R[1] = 2.f * (x * y - r * z); R[2] = 2.f * (x * z + r * y);
    R[3] = 2.f * (x * y + r * z); R[4] = 1.f - 2.f * (x * x + z * z); R[5] = 2.f * (y * z - r * x);
    R[6] = 2.f * (x * z - r * y); R[7] = 2.f * (y * z + r * x); R[8] = 1.f - 2.f * (x * x + y * y);
    s0 = expf(l0); s1 = expf(l1); s2 = expf(l2);
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (a.flags[(size_t)k * a.P + i] == 0u) continue;
    const uint32_t o = a.base[k] + a.offsets[(size_t)k * a.P + i];
    a.src[o] = i;
    a.kind[o] = (unsigned char)k;
    float nx = px, ny = py, nz = pz, ns0 = l0, ns1 = l1, ns2 = l2;
    if (k > 0) {
      float e0, e1, e2;   // standard-normal samples
      if (a.noise != nullptr) {
        const float* n = a.noise + ((size_t)(k - 1) * a.P + i) * 3;
        e0 = n[0]; e1 = n[1]; e2 = n[2];
      } else {
        uint32_t rnd[4];
        philox((uint32_t)a.seed, (uint32_t)(a.seed >> 32), (uint32_t)i, (uint32_t)k, 0x243F6A88u, 0x85A308D3u, rnd);
        const float ra = sqrtf(-2.0f * logf(u01(rnd[0]))), rb = sqrtf(-2.0f * logf(u01(rnd[2])));
        float sn, cs;
        sincosf(6.28318530717958647692f * u01(rnd[1]), &sn, &cs);
        e0 = ra * cs; e1 = ra * sn;
        e2 = rb * cosf(6.28318530717958647692f * u01(rnd[3]));
      }
      // samples = normal(0, std = get_scaling); new_xyz = R * samples + xyz  (gaussian_model.py:649-653 / :674-679)
      const float v0 = e0 * s0, v1 = e1 * s1, v2 = e2 * s2;
      nx = px + R[0] * v0 + R[1] * v1 + R[2] * v2;
      ny = py + R[3] * v0 + R[4] * v1 + R[5] * v2;
      nz = pz + R[6] * v0 + R[7] * v1 + R[8] * v2;
      if (k >= 2) {
        ns0 = child_raw_scaling(s0); ns1 = child_raw_scaling(s1); ns2 = child_raw_scaling(s2);
      }
    }
    a.new_xyz[3 * (size_t)o] = nx; a.new_xyz[3 * (size_t)o + 1] = ny; a.new_xyz[3 * (size_t)o + 2] = nz;
    a.new_scaling[3 * (size_t)o] = ns0; a.new_scaling[3 * (size_t)o + 1] = ns1; a.new_scaling[3 * (size_t)o + 2] = ns2;
  }
}

__global__ void __launch_bounds__(256) k_gather_rows(const float* __restrict__ src, int row, const int32_t* __restrict__ idx,
                                                    const unsigned char* __restrict__ kind, size_t n_out, int zero_new,
                                                    float* __restrict__ dst) {
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_out * (size_t)row) return;
  const size_t o = e / (size_t)row;
  const int c = (int)(e - o * (size_t)row);
  dst[e] = (zero_new && kind[o] != 0) ? 0.f : src[(size_t)idx[o] * row + c];
}

}  // namespace

// Step 1: the four keep-flags of every Gaussian and their exclusive scans.  flags / offsets: [4][P] u32 (device), totals: [4] u32
// (device; read them back to size the outputs), scan_tmp: gof_densify_scratch_bytes(P).
extern "C" GOF_API size_t gof_densify_scratch_bytes(int P) {
  if (P <= 0) return 0;
  return gof_scan_scratch_bytes((size_t)P);
}

extern "C" GOF_API int gof_densify_plan(int P, const float* accum, const float* accum_abs, const float* denom, const float* scaling_raw,
                                        const float* opacity_raw, float max_grad, float abs_threshold, float dense_extent,
                                        float min_opacity, float prune_scale, uint32_t* flags, uint32_t* offsets, uint32_t* totals,
                                        uint32_t* scan_tmp, void* stream) {
  if (P < 0) { gof_set_error("densify_plan: P < 0"); return GOF_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  if (P == 0) { if (totals) GOF_CUDA_OK(cudaMemsetAsync(totals, 0, 16, st)); return GOF_OK; }
  if (!accum || !accum_abs || !denom || !scaling_raw || !opacity_raw || !flags || !offsets || !totals || !scan_tmp) {
    gof_set_error("densify_plan: NULL argument");
    return GOF_E_INVALID;
  }
  PlanArgs a{};
  a.P = P; a.accum = accum; a.accum_abs = accum_abs; a.denom = denom; a.scaling = scaling_raw; a.opacity = opacity_raw;
  a.max_grad = max_grad; a.abs_threshold = abs_threshold; a.dense_extent = dense_extent; a.min_opacity = min_opacity;
  a.prune_scale = prune_scale; a.flags = flags;
  GOF_LAUNCH("densify_plan", st, k_densify_plan<<<(P + 255) / 256, 256, 0, st>>>(a));
  GOF_LAUNCH_CHECK(false, st);
  for (int k = 0; k < 4; ++k) {
    const int rc = gof_exclusive_scan_u32(flags + (size_t)k * P, offsets + (size_t)k * P, scan_tmp, totals + k, (size_t)P, false, st);
    if (rc != GOF_OK) return rc;
  }
  return GOF_OK;
}

// Step 2: per output row its source Gaussian and kind, the new positions and raw scalings.  totals_host: the four block sizes
// read back from step 1 (N = their sum).  noise: optional [3][P][3] standard-normal samples (tests); otherwise Philox(seed).
extern "C" GOF_API int gof_densify_emit(int P, const uint32_t* flags, const uint32_t* offsets, const uint32_t* totals_host,
                                        const float* xyz, const float* scaling_raw, const float* rotation_raw, const float* noise,
                                        unsigned long long seed, int32_t* src_index, unsigned char* kind, float* new_xyz,
                                        float* new_scaling_raw, void* stream) {
  if (P <= 0) return GOF_OK;
  if (!flags || !offsets || !totals_host || !xyz || !scaling_raw || !rotation_raw || !src_index || !kind || !new_xyz || !new_scaling_raw) {
    gof_set_error("densify_emit: NULL argument");
    return GOF_E_INVALID;
  }
  EmitArgs a{};
  a.P = P; a.flags = flags; a.offsets = offsets;
  uint32_t b = 0;
  for (int k = 0; k < 4; ++k) { a.base[k] = b; b += totals_host[k]; }
  a.xyz = xyz; a.scaling = scaling_raw; a.rotation = rotation_raw; a.noise = noise; a.seed = seed;
  a.src = src_index; a.kind = kind; a.new_xyz = new_xyz; a.new_scaling = new_scaling_raw;
  cudaStream_t st = (cudaStream_t)stream;
  GOF_LAUNCH("densify_emit", st, k_densify_emit<<<(P + 255) / 256, 256, 0, st>>>(a));
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}

// Step 3, once per tensor: dst[o, :] = src[src_index[o], :], or zeros for rows of new Gaussians when zero_new (Adam states).
extern "C" GOF_API int gof_gather_rows_f32(const float* src, int row_floats, const int32_t* src_index, const unsigned char* kind,
                                           size_t n_out, int zero_new, float* dst, void* stream) {
  if (n_out == 0 || row_floats <= 0) return GOF_OK;
  if (!src || !src_index || !kind || !dst) { gof_set_error("gather_rows: NULL argument"); return GOF_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const size_t total = n_out * (size_t)row_floats;
  GOF_LAUNCH("gather_rows", st, k_gather_rows<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(src, row_floats, src_index, kind, n_out, zero_new, dst));
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}
