// preprocess.cu -- per-Gaussian kernels: forward preprocess (K1), backward preprocess (K8), frustum mask (K9).
//
// Restates forward.cu:283-404 (preprocessCUDA), backward.cu:593-631 (+ :381-587, :20-139) and
// rasterizer_impl.cu:54-66 (checkFrustum) of the reference.  One thread per Gaussian, 128-bit loads of the
// SH rows, one 64-byte GofSplat record out (see gof_common.cuh).
#include <stdlib.h>

#include "gof_common.cuh"
#include "gof_math.cuh"

namespace {

struct PreArgs {
  int P, D, M, W, H, grid_x, grid_y;
  float tan_fovx, tan_fovy, focal_x, focal_y, kernel_size, scale_modifier;
  const float* means3D;
  const float* shs;
  const float* colors_precomp;
  const float* opacities;
  const float* scales;
  const float* rotations;
  const float* cov3D_precomp;
  const float* v2g_precomp;
  const float* viewmatrix;
  const float* projmatrix;
  const float* cam_pos;
  int prefiltered;
  // outputs
  int* radii;
  GofSplat* splat;
  GofSplatBwd* splat_bwd;
  uint2* rect;          // packed (xmin | ymin<<16, xmax | ymax<<16)
  uint32_t* tiles;
  unsigned char* clamped;
  uint32_t* depth_key;  // depth bits for visible Gaussians, 0xFFFFFFFF otherwise (sorts last)
  uint32_t* order;      // identity permutation, the value array of the depth sort
  float* depth;         // view-space z of visible Gaussians (parity export)
  uint32_t* total;      // sum of tiles_touched = num_rendered (zeroed by the launcher)
  float* reject_k;      // see GofGeomLayout::reject_k
  int cull;             // 1: store the conservative alpha-support box, 0: store the whole plane
  float box_margin;     // pixels the box reaches beyond the centre rays (gof_cull_bbox): 0 blend, 0.5 opacity-field query
};

__global__ void __launch_bounds__(256) k_preprocess(const PreArgs a) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= a.P) return;

  const float* __restrict__ vm = a.viewmatrix;
  const float* __restrict__ pm = a.projmatrix;

  // forward.cu:319-320
  int radius_out = 0;
  uint32_t tiles_out = 0;
  uint32_t key_out = 0xFFFFFFFFu;
  uint2 rect_out = make_uint2(0u, 0u);

  const float px = a.means3D[3 * idx + 0], py = a.means3D[3 * idx + 1], pz = a.means3D[3 * idx + 2];
  // in_frustum (auxiliary.h:177-202): only the near-plane test survives
  const float tz = gof_affine(px, py, pz, __ldg(vm + 2), __ldg(vm + 6), __ldg(vm + 10), __ldg(vm + 14));
  bool alive = !(tz <= 0.2f);
  if (!alive && a.prefiltered) {
    printf("Point is filtered although prefiltered is set. This shouldn't happen!");
    __trap();
  }

  GofCov2D cov;
  float cov3D[6];
  float pix_x = 0.f, pix_y = 0.f;
  uint32_t x0 = 0, y0 = 0, x1 = 0, y1 = 0;
  int my_radius = 0;
  if (alive) {
    // forward.cu:328-331
    const float hx = gof_affine(px, py, pz, __ldg(pm + 0), __ldg(pm + 4), __ldg(pm + 8), __ldg(pm + 12));
    const float hy = gof_affine(px, py, pz, __ldg(pm + 1), __ldg(pm + 5), __ldg(pm + 9), __ldg(pm + 13));
    const float hw = gof_affine(px, py, pz, __ldg(pm + 3), __ldg(pm + 7), __ldg(pm + 11), __ldg(pm + 15));
    const float p_w = F_RCP(F_ADD(hw, 0.0000001f));
    const float proj_x = F_MUL(hx, p_w), proj_y = F_MUL(hy, p_w);

    // forward.cu:339-348
    if (a.cov3D_precomp != nullptr) {
#pragma unroll
      for (int k = 0; k < 6; ++k) cov3D[k] = a.cov3D_precomp[6 * idx + k];
    } else {
      const float4 q = reinterpret_cast<const float4*>(a.rotations)[idx];
      const GofRot R = gof_quat_to_rot(q.x, q.y, q.z, q.w);
      gof_cov3d(R, a.scales[3 * idx + 0], a.scales[3 * idx + 1], a.scales[3 * idx + 2], a.scale_modifier, cov3D);
    }
    // forward.cu:351 (view-space x,y re-derived inside computeCov2D)
    float vmat[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) vmat[k] = __ldg(vm + k);
    const float tx = gof_affine(px, py, pz, vmat[0], vmat[4], vmat[8], vmat[12]);
    const float ty = gof_affine(px, py, pz, vmat[1], vmat[5], vmat[9], vmat[13]);
    cov = gof_cov2d(tx, ty, tz, a.focal_x, a.focal_y, a.tan_fovx, a.tan_fovy, a.kernel_size, cov3D, vmat);
    // forward.cu:354-356
    if (cov.det == 0.0f) alive = false;
    if (alive) {
      // forward.cu:364-372
      const float mid = F_MUL(F_ADD(cov.a, cov.c), 0.5f);
      const float sq = F_SQRT(fmaxf(F_FMA(mid, mid, -cov.det), 0.1f));
      const float lambda1 = F_ADD(mid, sq), lambda2 = F_SUB(mid, sq);
      const float rad_f = ceilf(F_MUL(F_SQRT(fmaxf(lambda1, lambda2)), 3.0f));
      my_radius = gof_f2i_rz(rad_f);
      pix_x = gof_ndc2pix(proj_x, a.W);
      pix_y = gof_ndc2pix(proj_y, a.H);
      gof_get_rect(pix_x, pix_y, my_radius, a.grid_x, a.grid_y, &x0, &y0, &x1, &y1);
      if ((x1 - x0) * (y1 - y0) == 0) alive = false;
    }
  }

  if (alive) {
    GofSplat rec;
    unsigned char clamp_bits = 0;
    // forward.cu:376-382
    if (a.colors_precomp == nullptr) {
      // Every sh[] index is a compile-time constant (the loops are unrolled, the degree only predicates the loads), so the row
      // lives in registers: one runtime index would put all 48 floats in local memory, 192 B per thread through L1/L2.
      float sh[48];
      const int nf = 3 * (a.D + 1) * (a.D + 1);   // floats the degree reads; <= 3 M (checked by the API)
      if (a.M == 16) {
        const float4* src = reinterpret_cast<const float4*>(a.shs + (size_t)idx * 48);
#pragma unroll
        for (int k = 0; k < 12; ++k) {
          const float4 v = (4 * k < nf) ? __ldg(src + k) : make_float4(0.f, 0.f, 0.f, 0.f);
          sh[4 * k + 0] = v.x; sh[4 * k + 1] = v.y; sh[4 * k + 2] = v.z; sh[4 * k + 3] = v.w;
        }
      } else {
        const float* s = a.shs + (size_t)idx * a.M * 3;
#pragma unroll
        for (int k = 0; k < 48; ++k) sh[k] = (k < nf) ? s[k] : 0.f;
      }
      gof_sh_to_rgb(a.D, px, py, pz, a.cam_pos, sh, rec.rgb, &clamp_bits);
    } else {
      rec.rgb[0] = a.colors_precomp[3 * idx + 0];
      rec.rgb[1] = a.colors_precomp[3 * idx + 1];
      rec.rgb[2] = a.colors_precomp[3 * idx + 2];
    }
    // forward.cu:385-390
    const float det_inv = F_RCP(cov.det);
    GofSplatBwd rb;
    rb.mx = pix_x; rb.my = pix_y;
    rb.cx = F_MUL(cov.c, det_inv);
    rb.cy = F_MUL(det_inv, -cov.b);
    rb.cz = F_MUL(cov.a, det_inv);
    rb.self = (uint32_t)idx;
    rb.pad[0] = rb.pad[1] = 0.f;
    rec.opacity = F_MUL(cov.coef, a.opacities[idx]);
    double lambda_min = 0.0;   // smallest eigenvalue of Sigma = min S^-2; unknown for a precomputed record
    // forward.cu:395-403 (the precomputed record is used with stride 10, rasterizer_impl.cu:379)
    if (a.v2g_precomp == nullptr) {
      float vmat[16];
#pragma unroll
      for (int k = 0; k < 16; ++k) vmat[k] = __ldg(vm + k);
      const float4 q = reinterpret_cast<const float4*>(a.rotations)[idx];
      const GofRot R = gof_quat_to_rot(q.x, q.y, q.z, q.w);
      const float sx = a.scales[3 * idx + 0], sy = a.scales[3 * idx + 1], sz = a.scales[3 * idx + 2];
      gof_view2gaussian(R, sx, sy, sz, px, py, pz, vmat, rec.v2g);
      const double smax = fmax(fmax(fabs((double)sx), fabs((double)sy)), fabs((double)sz));
      lambda_min = 1.0 / (smax * smax + 1e-7);
    } else {
#pragma unroll
      for (int k = 0; k < 10; ++k) rec.v2g[k] = a.v2g_precomp[10 * idx + k];
    }
    const GofBox box = a.cull ? gof_cull_bbox(rec.v2g, rec.opacity, lambda_min, a.W, a.H, a.focal_x, a.focal_y, a.tan_fovx, a.tan_fovy,
                                                a.box_margin)
                              : gof_full_box();
    rec.box_lo = ((uint32_t)box.x0 & 0xffffu) | ((uint32_t)box.y0 << 16);
    rec.box_hi = ((uint32_t)box.x1 & 0xffffu) | ((uint32_t)box.y1 << 16);
    a.depth[idx] = tz;
    // Constant of the blend kernel's conservative pair reject (render_fwd.cu): with thr = -ln(255 op) - 2e-3 (the margin
    // covers expf and the float rounding of power) a pair is provably below alpha = 1/255 when
    // -1/2 (C - (B/2)^2 / A) < thr  <=>  (B/2)^2 < A (C + 2 thr)  for A > 0.  K' carries a 4e-7 relative margin: the
    // two float products of the test are each within 2^-24 and K' itself is rounded once (6e-8); K <= 0 (camera inside the iso-surface) or op <= 0 can never reject / always reject.
    {
      float kp;
      if (!(rec.opacity > 0.f)) kp = __int_as_float(0x7f800000);            // +inf: every pair rejected (alpha <= 0)
      else {
        const double K = (double)rec.v2g[9] + 2.0 * (-(double)logf(255.0f * rec.opacity) - 2e-3);
        kp = K > 0.0 ? (float)(K * (1.0 - 4e-7)) : __int_as_float(0xff800000);   // -inf: never rejected
      }
      a.reject_k[idx] = kp;
    }
    float4* dst = reinterpret_cast<float4*>(a.splat + idx);
    const float4* srcr = reinterpret_cast<const float4*>(&rec);
    dst[0] = srcr[0]; dst[1] = srcr[1]; dst[2] = srcr[2]; dst[3] = srcr[3];
    float4* dstb = reinterpret_cast<float4*>(a.splat_bwd + idx);
    const float4* srcb = reinterpret_cast<const float4*>(&rb);
    dstb[0] = srcb[0]; dstb[1] = srcb[1];
    a.clamped[idx] = clamp_bits;
    radius_out = my_radius;
    tiles_out = (y1 - y0) * (x1 - x0);
    rect_out = make_uint2(x0 | (y0 << 16), x1 | (y1 << 16));
    key_out = __float_as_uint(tz);
  }
  a.radii[idx] = radius_out;
  a.tiles[idx] = tiles_out;
  a.rect[idx] = rect_out;
  a.depth_key[idx] = key_out;
  a.order[idx] = (uint32_t)idx;
  // num_rendered = sum of tiles_touched (the reference reads the last element of its inclusive scan, rasterizer_impl.cu:334-336).
  // Summed here so that the host can read it while the depth sort runs; order-independent (integer adds).
  {
    const uint32_t active = __activemask();
    const uint32_t wsum = __reduce_add_sync(active, tiles_out);
    if ((int)(threadIdx.x & 31) == __ffs(active) - 1 && wsum) atomicAdd(a.total, wsum);
  }
}

__global__ void k_mark_visible(int P, const float* __restrict__ means3D, const float* __restrict__ vm,
                               unsigned char* __restrict__ present) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= P) return;
  const float tz = gof_affine(means3D[3 * idx], means3D[3 * idx + 1], means3D[3 * idx + 2], __ldg(vm + 2),
                              __ldg(vm + 6), __ldg(vm + 10), __ldg(vm + 14));
  present[idx] = !(tz <= 0.2f) ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------------
// K8: backward.cu:593-631.  Gradient arithmetic is stated naturally (tolerance 1e-4 relative; the
// reference itself is only reproducible to ~1e-6 because of its float atomics).
struct PreBwdArgs {
  int P, D, M;
  const float* means3D;
  const int* radii;
  const float* shs;
  const unsigned char* clamped;
  const float* scales;
  const float* rotations;
  const float* viewmatrix;
  const float* cam_pos;
  const double2* grad_acc;  // [P][8] double2: the blend kernel's accumulator rows (dv2g[10] | dcolor[3] | dmean2D[3])
  const GofSplat* splat;    // for the effective opacity (dL_dopacity = -2/opacity * dL_dC)
  float* dL_dmean2D;        // outputs unpacked from the accumulator row
  float* dL_dopacity;
  float* dL_dcolor;
  float* dL_dv2g;
  float* dL_dmean3D;
  float* dL_dsh;
  float* dL_dscale;
  float* dL_drot;
  float* dL_dcov3D;         // optional [P][6]: written as zeros
  float* dens_sum;          // optional [P][3]: |dL_dmean2D.xy|, |dL_dmean2D.z|, 1 for visible Gaussians (gof_backward_out_t::dens_sum)
  float* dens_max;          // optional [P][2]: |dL_dmean2D.z|, radius
  float* sh_rgb;            // optional [3][GOF_SH_PLANE(P)] planes: the clamp-masked dL_dRGB the SH gradient is the outer product of
  float* sh_hdr;            //   (view-parallel exchange, csrc/sh_views.cu); sh_hdr[0..3] = camera centre, active degree.  dL_dsh may be NULL.
  size_t sh_plane;
  // camera gradient (k_preprocess_backward<true> only)
  double* cam_partial;      // [gridDim.x][K8_CAM_ROW]: the CTA's sum of its Gaussians' camera terms
  int cam_vm;               // 0: view2gaussian was precomputed, so the view matrix receives no gradient
};

// m[c][r] column-major helpers mirroring the glm products used by backward.cu:381-587.  The chain rule through
// view2gaussian multiplies rounding errors by ~1/scale^2 (the reference's own float results scatter by 1e-3..1e-1
// between runs), so it is evaluated in double here: the result is the well-conditioned value the reference's
// float evaluation samples with noise.
struct M3 { double m[3][3]; };

__device__ __forceinline__ M3 m3_mul(const M3& A, const M3& B) {   // (A*B)[c][r] = sum_k A[k][r]*B[c][k]
  M3 o;
#pragma unroll
  for (int c = 0; c < 3; ++c)
#pragma unroll
    for (int r = 0; r < 3; ++r) o.m[c][r] = A.m[0][r] * B.m[c][0] + A.m[1][r] * B.m[c][1] + A.m[2][r] * B.m[c][2];
  return o;
}
__device__ __forceinline__ M3 m3_t(const M3& A) {
  M3 o;
#pragma unroll
  for (int c = 0; c < 3; ++c)
#pragma unroll
    for (int r = 0; r < 3; ++r) o.m[c][r] = A.m[r][c];
  return o;
}

constexpr int K8_THREADS = 128;
constexpr int K8_ROW = 49;   // 48 SH-gradient floats per Gaussian + 1 pad: lanes of a warp hit distinct banks
// Camera terms of one Gaussian (DESIGN.md 4.9): dL_dviewmatrix[4k+i] for k < 4, i < 3 at 3k+i, dL_dcampos at 12..14; a partial
// row holds them plus one pad double.
constexpr int K8_CAM_TERMS = 15, K8_CAM_ROW = 16;

// The outputs with rows of 2..10 floats, staged per warp in shared memory: each field holds the warp's 32 rows back to back, i.e.
// exactly the layout of the warp's block of the global tensor.  Every field starts on a multiple of 32 floats, so the copy-out
// reads it with 128-bit shared loads.
constexpr int K8_V2G = 0, K8_COLOR = K8_V2G + 32 * 10, K8_MEAN2D = K8_COLOR + 32 * 3, K8_MEAN3D = K8_MEAN2D + 32 * 3,
              K8_SCALE = K8_MEAN3D + 32 * 3, K8_DSUM = K8_SCALE + 32 * 3, K8_DMAX = K8_DSUM + 32 * 3, K8_STAGED = K8_DMAX + 32 * 2;

// n staged floats (src, 16-byte aligned shared memory) -> dst with lane-consecutive stores, 128-bit wherever dst is 16-byte
// aligned (the bucket's and the binding's tensors are; a caller's other tensor may be 4-byte aligned only)
__device__ __forceinline__ void k8_copy_out(float* __restrict__ dst, const float* src, int n, int lane) {
  int i = lane;
  if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
    for (; i < (n >> 2); i += 32) reinterpret_cast<float4*>(dst)[i] = reinterpret_cast<const float4*>(src)[i];
    i = 4 * (n >> 2) + lane;
  }
  for (; i < n; i += 32) dst[i] = src[i];
}

// CAMERA: also form this Gaussian's camera terms and leave the CTA's fp64 sum of them in a.cam_partial (the instantiation
// without it is the plain backward, instruction for instruction).
template <bool CAMERA>
__global__ void __launch_bounds__(K8_THREADS) k_preprocess_backward(const PreBwdArgs a) {
  // Every output leaves through shared memory: a thread produces its Gaussian's row (for dL_dsh one coefficient at a time), the
  // warp then writes its 32 consecutive Gaussians as one contiguous block with 128-bit stores.  Per-thread stores at the rows'
  // 8..192-byte strides touch scattered sectors (ncu showed the dL_dsh stores waiting on the LSU queue, lg_throttle 14 /
  // long_scoreboard 17 warps per issue).
  __shared__ float s_dsh[K8_THREADS / 32][32 * K8_ROW];
  __shared__ __align__(16) float s_out[K8_THREADS / 32][K8_STAGED];
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool active = idx < a.P && a.radii[idx] > 0;
  const unsigned active_mask = __ballot_sync(0xffffffffu, active);
  float* my_dsh = &s_dsh[warp][lane * K8_ROW];
  float* out = s_out[warp];
  const size_t g0 = (size_t)blockIdx.x * blockDim.x + (size_t)warp * 32;   // first Gaussian of this warp
  const int in_range = (int)min((size_t)32, (size_t)a.P > g0 ? (size_t)a.P - g0 : (size_t)0);
  if (idx == 0 && a.sh_hdr != nullptr) {
    a.sh_hdr[0] = a.cam_pos[0]; a.sh_hdr[1] = a.cam_pos[1]; a.sh_hdr[2] = a.cam_pos[2]; a.sh_hdr[3] = (float)a.D;
  }

  // EVERY output element of every Gaussian is written by this kernel (zeros for Gaussians this view does not see): callers may
  // hand in uninitialised tensors -- the reference zero-fills ten tensors per backward (rasterize_points.cu:161-170), which at
  // 1 M Gaussians is 324 MB of memset in front of the kernels.  So every output starts as zero here.
  float accv[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) accv[k] = 0.f;
  float dopacity = 0.f, dscale[3] = {0.f, 0.f, 0.f}, dmean[3] = {0.f, 0.f, 0.f}, dens[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
  float4 drot = make_float4(0.f, 0.f, 0.f, 0.f);
  float dRGB[3] = {0.f, 0.f, 0.f};
  double cam[K8_CAM_TERMS];
  if constexpr (CAMERA) {
#pragma unroll
    for (int k = 0; k < K8_CAM_TERMS; ++k) cam[k] = 0.0;
  }

  if (active) {
  // the blend kernel's accumulator row -> the public gradient tensors (the double sums rounded once to float)
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const double2 g = a.grad_acc[8 * (size_t)idx + k];
    accv[2 * k] = (float)g.x;
    accv[2 * k + 1] = (float)g.y;
  }
  {
    // alpha = opacity * G, dL_dC = dL_dG * G * -1/2  =>  sum(G * dL_dalpha) = -2/opacity * sum(dL_dC)   (backward.cu:912)
    const float op = a.splat[idx].opacity;
    dopacity = (accv[9] != 0.f) ? accv[9] * (-2.0f / op) : 0.f;
    // this view's densification statistics (GaussianModel.add_densification_stats, scene/gaussian_model.py:709-714, and the
    // max_radii2D update of train.py:255), written next to the gradients so that a view-parallel step reduces them in the
    // same exchange instead of deriving them with a dozen elementwise kernels
    const float gz = fabsf(accv[15]);
    dens[0] = sqrtf(accv[13] * accv[13] + accv[14] * accv[14]);
    dens[1] = gz;
    dens[2] = 1.0f;
    dens[3] = gz;
    dens[4] = (float)a.radii[idx];
  }
  }   // active
  // the accumulator row and the statistics go to the staging area now, so that their registers are free for the chain rule
#pragma unroll
  for (int k = 0; k < 10; ++k) out[K8_V2G + 10 * lane + k] = accv[k];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    out[K8_COLOR + 3 * lane + c] = accv[10 + c];
    out[K8_MEAN2D + 3 * lane + c] = accv[13 + c];
    out[K8_DSUM + 3 * lane + c] = dens[c];
  }
  out[K8_DMAX + 2 * lane] = dens[3];
  out[K8_DMAX + 2 * lane + 1] = dens[4];

  if (active) {

  const float mx = a.means3D[3 * idx], my = a.means3D[3 * idx + 1], mz = a.means3D[3 * idx + 2];

  if (a.scales != nullptr && a.rotations != nullptr) {
    // ---- computeView2Gaussian_backward, backward.cu:381-587 ----
    double vm[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) vm[k] = (double)__ldg(a.viewmatrix + k);
    const float4 q = reinterpret_cast<const float4*>(a.rotations)[idx];
    const double r = q.x, x = q.y, y = q.z, z = q.w;
    const double sx = a.scales[3 * idx], sy = a.scales[3 * idx + 1], sz = a.scales[3 * idx + 2];
    double dv[10];
#pragma unroll
    for (int k = 0; k < 10; ++k) dv[k] = (double)accv[k];

    M3 R;   // glm::mat3 R(...), column-major constructor
    R.m[0][0] = 1. - 2. * (y * y + z * z); R.m[0][1] = 2. * (x * y - r * z); R.m[0][2] = 2. * (x * z + r * y);
    R.m[1][0] = 2. * (x * y + r * z); R.m[1][1] = 1. - 2. * (x * x + z * z); R.m[1][2] = 2. * (y * z - r * x);
    R.m[2][0] = 2. * (x * z - r * y); R.m[2][1] = 2. * (y * z + r * x); R.m[2][2] = 1. - 2. * (x * x + y * y);

    // G2V = W2V * G2W; G2W[c] = (R[0][c], R[1][c], R[2][c], 0), G2W[3] = (mean, 1)
    double G2V[4][3];
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int i = 0; i < 3; ++i)
        G2V[c][i] = vm[i] * R.m[0][c] + vm[4 + i] * R.m[1][c] + vm[8 + i] * R.m[2][c];
#pragma unroll
    for (int i = 0; i < 3; ++i) G2V[3][i] = vm[i] * (double)mx + vm[4 + i] * (double)my + vm[8 + i] * (double)mz + vm[12 + i];

    M3 Rt;   // R_transpose[c][r] = G2V[r][c]
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int rr = 0; rr < 3; ++rr) Rt.m[c][rr] = G2V[rr][c];
    const double t[3] = {G2V[3][0], G2V[3][1], G2V[3][2]};
    double t2[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) t2[i] = -Rt.m[0][i] * t[0] - Rt.m[1][i] * t[1] - Rt.m[2][i] * t[2];

    const double si[3] = {1.0 / (sx * sx + 1e-7), 1.0 / (sy * sy + 1e-7), 1.0 / (sz * sz + 1e-7)};
    M3 SR;   // S_inv_square_R[c][r] = si[r] * Rt[c][r]
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int rr = 0; rr < 3; ++rr) SR.m[c][rr] = si[rr] * Rt.m[c][rr];

    M3 dS;   // symmetric
    dS.m[0][0] = dv[0]; dS.m[0][1] = 0.5 * dv[1]; dS.m[0][2] = 0.5 * dv[2];
    dS.m[1][0] = 0.5 * dv[1]; dS.m[1][1] = dv[3]; dS.m[1][2] = 0.5 * dv[4];
    dS.m[2][0] = 0.5 * dv[2]; dS.m[2][1] = 0.5 * dv[4]; dS.m[2][2] = dv[5];
    const double dB[3] = {dv[6], dv[7], dv[8]};
    const double dC = dv[9];

    // dL_dS_inv_square_R = R_transpose * dL_dSigma + outerProduct(t2, dL_dB)   (backward.cu:458)
    M3 dSR = m3_mul(Rt, dS);
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int rr = 0; rr < 3; ++rr) dSR.m[c][rr] += t2[rr] * dB[c];
    // dL_dR_transpose = transpose(dL_dSigma * transpose(S_inv_square_R)) + diag(si) scaling (:459-470)
    M3 dRt = m3_t(m3_mul(dS, m3_t(SR)));
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int rr = 0; rr < 3; ++rr) dRt.m[c][rr] += si[rr] * dSR.m[c][rr];
    // :471-484
    double dSi[3], dt2[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      dSi[i] = dSR.m[0][i] * Rt.m[0][i] + dSR.m[1][i] * Rt.m[1][i] + dSR.m[2][i] * Rt.m[2][i];
      dt2[i] = 2 * t2[i] * si[i] * dC + dB[0] * SR.m[0][i] + dB[1] * SR.m[1][i] + dB[2] * SR.m[2][i];
      dSi[i] += dC * t2[i] * t2[i];
    }
    const double sc[3] = {sx, sy, sz};
#pragma unroll
    for (int i = 0; i < 3; ++i) dscale[i] = (float)(-2 / sc[i] * si[i] * dSi[i]);   // :486-497

    // :523-535  dL_dG2V_R[c][r] = dL_dRt[r][c] - dt2[c]*t[r];  dL_dG2V_t[c] = sum_r (-dt2[r]) * Rt[c][r]
    double dG2V[4][3];
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int rr = 0; rr < 3; ++rr) dG2V[c][rr] = dRt.m[rr][c] + (-dt2[c] * t[rr]);
#pragma unroll
    for (int c = 0; c < 3; ++c)
      dG2V[3][c] = Rt.m[c][0] * (-dt2[0]) + Rt.m[c][1] * (-dt2[1]) + Rt.m[c][2] * (-dt2[2]);
    // dL_dG2W = transpose(W2V) * dL_dG2V  (:547): [c][r] = sum_k vm[4r+k] * dG2V[c][k], k<3 (4th row is 0)
    double dG2W[4][3];
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
      for (int rr = 0; rr < 3; ++rr)
        dG2W[c][rr] = vm[4 * rr + 0] * dG2V[c][0] + vm[4 * rr + 1] * dG2V[c][1] + vm[4 * rr + 2] * dG2V[c][2];
    dmean[0] = (float)dG2W[3][0]; dmean[1] = (float)dG2W[3][1]; dmean[2] = (float)dG2W[3][2];   // :570-573
    if constexpr (CAMERA) {
      // G2V[c][i] = sum_k vm[4k+i] R[k][c] (c < 3) and G2V[3][i] = sum_k vm[4k+i] h_k, h = (mean, 1)
      if (a.cam_vm) {
        const double h[3] = {mx, my, mz};
#pragma unroll
        for (int k = 0; k < 3; ++k)
#pragma unroll
          for (int i = 0; i < 3; ++i)
            cam[3 * k + i] = dG2V[0][i] * R.m[k][0] + dG2V[1][i] * R.m[k][1] + dG2V[2][i] * R.m[k][2] + dG2V[3][i] * h[k];
#pragma unroll
        for (int i = 0; i < 3; ++i) cam[9 + i] = dG2V[3][i];
      }
    }

    // :575-586 quaternion gradient from dL_dMt = dL_dG2W_R
#define MT(c, r) dG2W[c][r]
    drot.x = (float)(2 * z * (MT(0, 1) - MT(1, 0)) + 2 * y * (MT(2, 0) - MT(0, 2)) + 2 * x * (MT(1, 2) - MT(2, 1)));
    drot.y = (float)(2 * y * (MT(1, 0) + MT(0, 1)) + 2 * z * (MT(2, 0) + MT(0, 2)) + 2 * r * (MT(1, 2) - MT(2, 1)) -
                     4 * x * (MT(2, 2) + MT(1, 1)));
    drot.z = (float)(2 * x * (MT(1, 0) + MT(0, 1)) + 2 * r * (MT(2, 0) - MT(0, 2)) + 2 * z * (MT(1, 2) + MT(2, 1)) -
                     4 * y * (MT(2, 2) + MT(0, 0)));
    drot.w = (float)(2 * r * (MT(0, 1) - MT(1, 0)) + 2 * x * (MT(2, 0) + MT(0, 2)) + 2 * y * (MT(1, 2) + MT(2, 1)) -
                     4 * z * (MT(1, 1) + MT(0, 0)));
#undef MT
  }

  // ---- computeColorFromSH backward, backward.cu:20-139 ----
  if (a.shs != nullptr) {
    const float dox = mx - a.cam_pos[0], doy = my - a.cam_pos[1], doz = mz - a.cam_pos[2];
    float x, y, z;
    gof_sh_view_dir(mx, my, mz, a.cam_pos[0], a.cam_pos[1], a.cam_pos[2], &x, &y, &z);
    float sh[48];
    if (a.M == 16) {   // 192-byte rows: 12 x LDG.128
      const float4* src = reinterpret_cast<const float4*>(a.shs + (size_t)idx * 48);
#pragma unroll
      for (int k = 0; k < 12; ++k) {
        const float4 t4 = __ldg(src + k);
        sh[4 * k] = t4.x; sh[4 * k + 1] = t4.y; sh[4 * k + 2] = t4.z; sh[4 * k + 3] = t4.w;
      }
    } else {
      const float* src = a.shs + (size_t)idx * a.M * 3;
#pragma unroll
      for (int k = 0; k < 48; ++k) sh[k] = (k < 3 * a.M) ? src[k] : 0.f;
    }
    const unsigned char cb = a.clamped[idx];
#pragma unroll
    for (int c = 0; c < 3; ++c) dRGB[c] = accv[10 + c] * ((cb >> c) & 1 ? 0.f : 1.f);

    float dRGBdx[3] = {0, 0, 0}, dRGBdy[3] = {0, 0, 0}, dRGBdz[3] = {0, 0, 0};
#define SH(k, c) sh[3 * (k) + (c)]
    if (a.dL_dsh != nullptr) {
      float w[16];
      gof_sh_grad_weights(a.D, x, y, z, w);
      const int nk = (a.D + 1) * (a.D + 1);
#pragma unroll
      for (int k = 0; k < 16; ++k)
        if (k < nk) { my_dsh[3 * k] = __fmul_rn(w[k], dRGB[0]); my_dsh[3 * k + 1] = __fmul_rn(w[k], dRGB[1]); my_dsh[3 * k + 2] = __fmul_rn(w[k], dRGB[2]); }
    }
    if (a.D > 0) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        dRGBdx[c] = -GOF_SH_C1 * SH(3, c);
        dRGBdy[c] = -GOF_SH_C1 * SH(1, c);
        dRGBdz[c] = GOF_SH_C1 * SH(2, c);
      }
      if (a.D > 1) {
        const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          dRGBdx[c] += GOF_SH_C2_0 * y * SH(4, c) + GOF_SH_C2_2 * 2.f * -x * SH(6, c) + GOF_SH_C2_3 * z * SH(7, c) +
                       GOF_SH_C2_4 * 2.f * x * SH(8, c);
          dRGBdy[c] += GOF_SH_C2_0 * x * SH(4, c) + GOF_SH_C2_1 * z * SH(5, c) + GOF_SH_C2_2 * 2.f * -y * SH(6, c) +
                       GOF_SH_C2_4 * 2.f * -y * SH(8, c);
          dRGBdz[c] += GOF_SH_C2_1 * y * SH(5, c) + GOF_SH_C2_2 * 2.f * 2.f * z * SH(6, c) + GOF_SH_C2_3 * x * SH(7, c);
        }
        if (a.D > 2) {
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            dRGBdx[c] += (GOF_SH_C3_0 * SH(9, c) * 3.f * 2.f * xy + GOF_SH_C3_1 * SH(10, c) * yz +
                          GOF_SH_C3_2 * SH(11, c) * -2.f * xy + GOF_SH_C3_3 * SH(12, c) * -3.f * 2.f * xz +
                          GOF_SH_C3_4 * SH(13, c) * (-3.f * xx + 4.f * zz - yy) + GOF_SH_C3_5 * SH(14, c) * 2.f * xz +
                          GOF_SH_C3_6 * SH(15, c) * 3.f * (xx - yy));
            dRGBdy[c] += (GOF_SH_C3_0 * SH(9, c) * 3.f * (xx - yy) + GOF_SH_C3_1 * SH(10, c) * xz +
                          GOF_SH_C3_2 * SH(11, c) * (-3.f * yy + 4.f * zz - xx) +
                          GOF_SH_C3_3 * SH(12, c) * -3.f * 2.f * yz + GOF_SH_C3_4 * SH(13, c) * -2.f * xy +
                          GOF_SH_C3_5 * SH(14, c) * -2.f * yz + GOF_SH_C3_6 * SH(15, c) * -3.f * 2.f * xy);
            dRGBdz[c] += (GOF_SH_C3_1 * SH(10, c) * xy + GOF_SH_C3_2 * SH(11, c) * 4.f * 2.f * yz +
                          GOF_SH_C3_3 * SH(12, c) * 3.f * (2.f * zz - xx - yy) +
                          GOF_SH_C3_4 * SH(13, c) * 4.f * 2.f * xz + GOF_SH_C3_5 * SH(14, c) * (xx - yy));
          }
        }
      }
    }
#undef SH
    const float ddx = dRGBdx[0] * dRGB[0] + dRGBdx[1] * dRGB[1] + dRGBdx[2] * dRGB[2];
    const float ddy = dRGBdy[0] * dRGB[0] + dRGBdy[1] * dRGB[1] + dRGBdy[2] * dRGB[2];
    const float ddz = dRGBdz[0] * dRGB[0] + dRGBdz[1] * dRGB[1] + dRGBdz[2] * dRGB[2];
    // dnormvdv (auxiliary.h:145-155)
    const float sum2 = dox * dox + doy * doy + doz * doz;
    const float invsum32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
    dmean[0] += ((+sum2 - dox * dox) * ddx - doy * dox * ddy - doz * dox * ddz) * invsum32;
    dmean[1] += (-dox * doy * ddx + (sum2 - doy * doy) * ddy - doz * doy * ddz) * invsum32;
    dmean[2] += (-dox * doz * ddx - doy * doz * ddy + (sum2 - doz * doz) * ddz) * invsum32;
    if constexpr (CAMERA) {
      // the direction is mean - campos: minus the SH term of dL_dmean3D, evaluated again in double from the same float
      // ddx, ddy, ddz (the float expressions above keep their own rounding, so dL_dmean3D is the plain backward's)
      const double ex = dox, ey = doy, ez = doz;
      const double s2 = ex * ex + ey * ey + ez * ez, inv = 1.0 / (s2 * sqrt(s2));
      const double gx = ddx, gy = ddy, gz = ddz;
      cam[12] = -(((s2 - ex * ex) * gx - ey * ex * gy - ez * ex * gz) * inv);
      cam[13] = -((-ex * ey * gx + (s2 - ey * ey) * gy - ez * ey * gz) * inv);
      cam[14] = -((-ex * ez * gx - ey * ez * gy + (s2 - ez * ez) * gz) * inv);
    }
  }
  }   // active

  // ---- the outputs with one float per Gaussian, or one 16-byte row: already contiguous per warp ----
  if (idx < a.P) {
    a.dL_dopacity[idx] = dopacity;
    if (a.dL_drot != nullptr) reinterpret_cast<float4*>(a.dL_drot)[idx] = drot;
    if (a.sh_rgb != nullptr) { a.sh_rgb[idx] = dRGB[0]; a.sh_rgb[a.sh_plane + idx] = dRGB[1]; a.sh_rgb[2 * a.sh_plane + idx] = dRGB[2]; }
  }
  if (a.dL_dcov3D != nullptr) {   // never receives a gradient (backward.cu:991-1007: EWA backward disabled)
    for (int i = lane; i < 6 * in_range; i += 32) a.dL_dcov3D[6 * g0 + i] = 0.f;
  }

  // ---- the rows of 2..10 floats: written one field at a time as the warp's contiguous block ----
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    out[K8_MEAN3D + 3 * lane + c] = dmean[c];
    out[K8_SCALE + 3 * lane + c] = dscale[c];
  }
  __syncwarp();
  k8_copy_out(a.dL_dv2g + 10 * g0, out + K8_V2G, 10 * in_range, lane);
  k8_copy_out(a.dL_dcolor + 3 * g0, out + K8_COLOR, 3 * in_range, lane);
  k8_copy_out(a.dL_dmean2D + 3 * g0, out + K8_MEAN2D, 3 * in_range, lane);
  k8_copy_out(a.dL_dmean3D + 3 * g0, out + K8_MEAN3D, 3 * in_range, lane);
  if (a.dL_dscale != nullptr) k8_copy_out(a.dL_dscale + 3 * g0, out + K8_SCALE, 3 * in_range, lane);
  if (a.dens_sum != nullptr) {
    k8_copy_out(a.dens_sum + 3 * g0, out + K8_DSUM, 3 * in_range, lane);
    k8_copy_out(a.dens_max + 2 * g0, out + K8_DMAX, 2 * in_range, lane);
  }

  // ---- the warp's dL_dsh rows: shared memory -> global, contiguous; rows of invisible Gaussians and the coefficients above
  // the active degree (backward.cu:20-139 writes degree <= D only) are written as zeros ----
  if (a.shs != nullptr && a.dL_dsh != nullptr) {
    __syncwarp();
    const int nw = 3 * (a.D + 1) * (a.D + 1);             // floats carrying a gradient per Gaussian
    const int row = a.M * 3;                              // floats per Gaussian in dL_dsh
    if (a.M == 16 && nw == 48) {
      float4* dst = reinterpret_cast<float4*>(a.dL_dsh + g0 * 48);
#pragma unroll 4
      for (int i = lane; i < in_range * 12; i += 32) {
        const int g = i / 12, j = (i - g * 12) * 4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if ((active_mask >> g) & 1u) {
          const float* r = &s_dsh[warp][g * K8_ROW + j];
          v = make_float4(r[0], r[1], r[2], r[3]);
        }
        dst[i] = v;
      }
    } else {
      for (int i = lane; i < in_range * row; i += 32) {
        const int g = i / row, j = i - g * row;
        a.dL_dsh[(g0 + g) * (size_t)row + j] = (((active_mask >> g) & 1u) && j < nw) ? s_dsh[warp][g * K8_ROW + j] : 0.f;
      }
    }
  }

  // ---- the CTA's camera row: a fixed shuffle tree per warp, then the warps in order (no atomics: bit-reproducible) ----
  if constexpr (CAMERA) {
    __shared__ double s_cam[K8_THREADS / 32][K8_CAM_TERMS];
#pragma unroll
    for (int k = 0; k < K8_CAM_TERMS; ++k) {
      double t = cam[k];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) t += __shfl_down_sync(0xffffffffu, t, o);
      if (lane == 0) s_cam[warp][k] = t;
    }
    __syncthreads();
    if (threadIdx.x < K8_CAM_ROW) {
      double t = 0.0;
      if (threadIdx.x < K8_CAM_TERMS) {
        t = s_cam[0][threadIdx.x];
#pragma unroll
        for (int w = 1; w < K8_THREADS / 32; ++w) t += s_cam[w][threadIdx.x];
      }
      a.cam_partial[(size_t)blockIdx.x * K8_CAM_ROW + threadIdx.x] = t;
    }
  }
}

// The camera gradient from the partial rows of k_preprocess_backward<true>: group g of 16 threads sums rows g, g + 64, ... in
// index order, a fixed tree joins the 64 groups, and the sums are rounded to float once.  dL_dviewmatrix[4k+3] (the
// coefficients of the view matrix's fourth row, which view2gaussian does not read) are written as zeros.
constexpr int CAM_SUM_THREADS = 1024, CAM_SUM_GROUPS = CAM_SUM_THREADS / K8_CAM_ROW;
__global__ void __launch_bounds__(CAM_SUM_THREADS) k_camera_grad_sum(int rows, const double* __restrict__ partial,
                                                                       float* __restrict__ dL_dviewmatrix, float* __restrict__ dL_dcampos) {
  __shared__ double s[CAM_SUM_GROUPS][K8_CAM_ROW];
  const int j = threadIdx.x % K8_CAM_ROW, g = threadIdx.x / K8_CAM_ROW;
  double t = 0.0;
#pragma unroll 4
  for (int r = g; r < rows; r += CAM_SUM_GROUPS) t += partial[(size_t)r * K8_CAM_ROW + j];
  s[g][j] = t;
  __syncthreads();
#pragma unroll
  for (int n = CAM_SUM_GROUPS / 2; n > 0; n >>= 1) {
    if (g < n) s[g][j] += s[g + n][j];
    __syncthreads();
  }
  if (threadIdx.x < 16) {
    const int k = threadIdx.x >> 2, i = threadIdx.x & 3;
    dL_dviewmatrix[threadIdx.x] = i < 3 ? (float)s[0][3 * k + i] : 0.f;
  }
  if (threadIdx.x < 3) dL_dcampos[threadIdx.x] = (float)s[0][12 + threadIdx.x];
}

}  // namespace

size_t gof_camera_grad_scratch_bytes(int P) {
  return P > 0 ? (size_t)((P + K8_THREADS - 1) / K8_THREADS) * K8_CAM_ROW * sizeof(double) : 0;
}

int gof_launch_preprocess(const gof_scene_t* s, const GofView& v, char* geom, const GofGeomLayout& L,
                          int* radii, float box_margin, cudaStream_t st) {
  PreArgs a{};
  a.P = s->P; a.D = s->D; a.M = s->M; a.W = v.W; a.H = v.H; a.grid_x = v.grid_x; a.grid_y = v.grid_y;
  a.tan_fovx = s->tan_fovx; a.tan_fovy = s->tan_fovy; a.focal_x = v.focal_x; a.focal_y = v.focal_y;
  a.kernel_size = s->kernel_size; a.scale_modifier = s->scale_modifier;
  a.means3D = s->means3D; a.shs = s->shs; a.colors_precomp = s->colors_precomp; a.opacities = s->opacities;
  a.scales = s->scales; a.rotations = s->rotations; a.cov3D_precomp = s->cov3D_precomp;
  a.v2g_precomp = s->view2gaussian_precomp; a.viewmatrix = s->viewmatrix; a.projmatrix = s->projmatrix;
  a.cam_pos = s->cam_pos; a.prefiltered = s->prefiltered;
  a.radii = radii;
  a.splat = reinterpret_cast<GofSplat*>(geom + L.splat);
  a.splat_bwd = reinterpret_cast<GofSplatBwd*>(geom + L.splat_bwd);
  a.rect = reinterpret_cast<uint2*>(geom + L.rect);
  a.tiles = reinterpret_cast<uint32_t*>(geom + L.tiles);
  a.clamped = reinterpret_cast<unsigned char*>(geom + L.clamped);
  a.depth_key = reinterpret_cast<uint32_t*>(geom + L.key_a);
  a.order = reinterpret_cast<uint32_t*>(geom + L.val_a);
  a.depth = reinterpret_cast<float*>(geom + L.depth);
  a.total = reinterpret_cast<uint32_t*>(geom + L.total);
  a.reject_k = reinterpret_cast<float*>(geom + L.reject_k);
  GOF_CUDA_OK(cudaMemsetAsync(a.total, 0, 4, st));
  {
    // GOF_CULL=0 stores the whole plane instead of the alpha-support boxes (A/B testing).  Results are identical as long as
    // the box covers every ray its consumer casts: the centre ray for the blend, centre and corner rays for the query.
    static int cull = -1;
    if (cull < 0) { const char* e = getenv("GOF_CULL"); cull = (e && e[0] == '0') ? 0 : 1; }
    a.cull = cull;
    a.box_margin = box_margin;
  }
  GOF_LAUNCH("preprocess_fwd", st, k_preprocess<<<(s->P + 255) / 256, 256, 0, st>>>(a));
  GOF_LAUNCH_CHECK(s->debug, st);
  return GOF_OK;
}

int gof_launch_preprocess_backward(const gof_scene_t* s, const char* geom, const GofGeomLayout& L, const int* radii,
                                   const gof_backward_out_t& o, cudaStream_t st) {
  PreBwdArgs a{};
  a.P = s->P; a.D = s->D; a.M = s->M;
  a.means3D = s->means3D; a.radii = radii; a.shs = s->shs;
  a.clamped = reinterpret_cast<const unsigned char*>(geom + L.clamped);
  a.scales = s->scales; a.rotations = s->rotations; a.viewmatrix = s->viewmatrix; a.cam_pos = s->cam_pos;
  a.grad_acc = reinterpret_cast<const double2*>(geom + L.grad_acc);
  a.splat = reinterpret_cast<const GofSplat*>(geom + L.splat);
  a.dL_dmean2D = o.dL_dmean2D; a.dL_dopacity = o.dL_dopacity;
  a.dL_dcolor = o.dL_dcolor; a.dL_dv2g = o.dL_dview2gaussian; a.dL_dmean3D = o.dL_dmean3D; a.dL_dsh = o.dL_dsh;
  a.dL_dscale = o.dL_dscale; a.dL_drot = o.dL_drot; a.dL_dcov3D = o.dL_dcov3D;
  a.dens_sum = (o.dens_sum && o.dens_max) ? o.dens_sum : nullptr; a.dens_max = a.dens_sum ? o.dens_max : nullptr;
  a.sh_rgb = s->shs ? o.sh_rgb : nullptr; a.sh_hdr = a.sh_rgb ? o.sh_hdr : nullptr; a.sh_plane = GOF_SH_PLANE(s->P);
  const int blocks = (s->P + K8_THREADS - 1) / K8_THREADS;
  if (o.dL_dviewmatrix == nullptr) {
    GOF_LAUNCH("preprocess_bwd", st, k_preprocess_backward<false><<<blocks, K8_THREADS, 0, st>>>(a));
    GOF_LAUNCH_CHECK(s->debug, st);
    return GOF_OK;
  }
  a.cam_partial = static_cast<double*>(o.scratch);
  a.cam_vm = s->view2gaussian_precomp == nullptr;
  GOF_LAUNCH("preprocess_bwd_camera", st, k_preprocess_backward<true><<<blocks, K8_THREADS, 0, st>>>(a));
  GOF_LAUNCH_CHECK(s->debug, st);
  GOF_LAUNCH("camera_grad_sum", st, k_camera_grad_sum<<<1, CAM_SUM_THREADS, 0, st>>>(blocks, a.cam_partial, o.dL_dviewmatrix,
                                                                                       o.dL_dcampos));
  GOF_LAUNCH_CHECK(s->debug, st);
  return GOF_OK;
}

int gof_launch_mark_visible(int P, const float* means3D, const float* vm, unsigned char* present,
                            cudaStream_t st) {
  GOF_LAUNCH("mark_visible", st, k_mark_visible<<<(P + 255) / 256, 256, 0, st>>>(P, means3D, vm, present));
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}
