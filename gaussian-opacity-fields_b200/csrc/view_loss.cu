// view_loss.cu -- CUDA kernels and C ABI of the per-view training loss (see view_loss.cuh for the algorithm and the
// reference lines).  Each kernel is the sequence of phases of view_loss.cuh with a block barrier between them; the host
// twin in tests/hostmath runs the same phases in the same order.
#include <math.h>

#include "gof_common.cuh"
#include "view_loss.cuh"

namespace {

// APPEARANCE = false pins p.mapping to NULL, so that the plain kernels compile without the appearance branches of the phases
template <bool APPEARANCE>
__global__ void __launch_bounds__(VL_THREADS) k_view_loss_a(const VlParams params) {
  VlParams p = params;
  if (!APPEARANCE) p.mapping = nullptr;
  __shared__ VlShared s;
  const int tile = blockIdx.x, tx = tile % p.tiles_x, ty = tile / p.tiles_x, tid = threadIdx.x;
  vl_a_zero(s, tid);
  for (int ch = 0; ch < 3; ++ch) {
    __syncthreads();
    vl_a_load(p, s, tx, ty, ch, tid);
    __syncthreads();
    vl_a_hblur(p, s, tid);
    __syncthreads();
    vl_a_ssim(p, s, tx, ty, ch, tid);
  }
  __syncthreads();
  vl_a_points(p, s, tx, ty, tid);
  __syncthreads();
  vl_a_normals(p, s, tx, ty, tid);
  __syncthreads();
  vl_a_pixel(p, s, tx, ty, tid);
  for (int stride = VL_THREADS / 2; stride >= 1; stride >>= 1) {
    __syncthreads();
    vl_a_reduce(p, s, tile, stride, tid);
  }
}

template <bool APPEARANCE>
__global__ void __launch_bounds__(VL_THREADS) k_view_loss_b(const VlParams params) {
  VlParams p = params;
  if (!APPEARANCE) p.mapping = nullptr;
  __shared__ VlShared s;
  const int tile = blockIdx.x, tx = tile % p.tiles_x, ty = tile / p.tiles_x, tid = threadIdx.x;
  for (int ch = 0; ch < 3; ++ch) {
    __syncthreads();
    vl_b_load(p, s, tx, ty, ch, tid);
    __syncthreads();
    vl_b_hblur(p, s, tid);
    __syncthreads();
    vl_b_grad(p, s, tx, ty, ch, tid);
  }
}

// fixed-order sum of the per-tile partials in double: thread t adds tiles t, t+256, ...; then a tree over the threads
// N_l1 = the number of terms of the L1 mean: 3 H W, or 3 Hc Wc in appearance mode
__global__ void __launch_bounds__(VL_THREADS) k_view_loss_c(const float* __restrict__ partial, int tiles, double N, double N_l1,
                                                           float lam, float lam_dn, float lam_dist, float* __restrict__ terms) {
  __shared__ double acc[4][VL_THREADS];
  const int tid = threadIdx.x;
  double a[4] = {0.0, 0.0, 0.0, 0.0};
  for (int t = tid; t < tiles; t += VL_THREADS)
    for (int q = 0; q < 4; ++q) a[q] += (double)partial[(size_t)t * 4 + q];
  for (int q = 0; q < 4; ++q) acc[q][tid] = a[q];
  for (int stride = VL_THREADS / 2; stride >= 1; stride >>= 1) {
    __syncthreads();
    if (tid < stride)
      for (int q = 0; q < 4; ++q) acc[q][tid] += acc[q][tid + stride];
  }
  if (tid == 0) {
    const double ssim = acc[0][0] / (3.0 * N), l1 = acc[1][0] / N_l1, dnl = acc[2][0] / N, dist = acc[3][0] / N;
    terms[0] = (float)l1; terms[1] = (float)ssim; terms[2] = (float)dnl; terms[3] = (float)dist;
    terms[4] = (float)((1.0 - (double)lam) * l1 + (double)lam * (1.0 - ssim) + (double)lam_dn * dnl + (double)lam_dist * dist);
  }
}

}  // namespace

extern "C" GOF_API size_t gof_view_loss_scratch_bytes(int W, int H) {
  if (W <= 0 || H <= 0) return 0;
  const size_t tiles = (size_t)((W + VL_TILE - 1) / VL_TILE) * ((H + VL_TILE - 1) / VL_TILE);
  return gof_align_up((size_t)9 * W * H * sizeof(float), 256) + tiles * 4 * sizeof(float);
}

namespace {

int view_loss_checked(int W, int H, const float* render, const float* gt, const float* c2w_R9, float fx, float fy, float* terms,
                      void* scratch) {
  if (W <= 0 || H <= 0 || !render || !gt || !c2w_R9 || !terms || !scratch || !(fx > 0.f) || !(fy > 0.f)) {
    gof_set_error("view_loss: bad arguments");
    return GOF_E_INVALID;
  }
  return GOF_OK;
}

// the three launches over a VlParams whose pointers and crop the caller has set and checked
int view_loss_run(VlParams& p, const float* c2w_R9, float fx, float fy, float lambda_dssim, float lambda_depth_normal,
                  float lambda_distortion, float* terms, void* scratch, void* stream) {
  const int W = p.W, H = p.H;
  p.tiles_x = (W + VL_TILE - 1) / VL_TILE; p.tiles_y = (H + VL_TILE - 1) / VL_TILE;
  for (int k = 0; k < 9; ++k) p.R[k] = c2w_R9[k];
  p.fx = fx; p.fy = fy;
  {   // utils/loss_utils.py:23-25, evaluated in float like torch.Tensor([...]) / sum
    float sum = 0.f;
    for (int k = 0; k < 11; ++k) { p.g[k] = (float)exp(-(double)((k - 5) * (k - 5)) / (2.0 * 1.5 * 1.5)); sum += p.g[k]; }
    for (int k = 0; k < 11; ++k) p.g[k] /= sum;
  }
  p.lam = lambda_dssim; p.lam_dn = lambda_depth_normal; p.lam_dist = lambda_distortion;
  p.inv_N = 1.0f / ((float)W * (float)H); p.inv_N3 = 1.0f / (3.0f * (float)W * (float)H);
  p.dmap = static_cast<float*>(scratch);
  p.partial = reinterpret_cast<float*>(static_cast<char*>(scratch) + gof_align_up((size_t)9 * W * H * sizeof(float), 256));
  const double N_l1 = p.mapping ? 3.0 * ((double)p.Hc * (double)p.Wc) : 3.0 * ((double)W * (double)H);
  cudaStream_t st = (cudaStream_t)stream;
  const int tiles = p.tiles_x * p.tiles_y;
  if (p.mapping) GOF_LAUNCH("view_loss_a", st, k_view_loss_a<true><<<tiles, VL_THREADS, 0, st>>>(p));
  else GOF_LAUNCH("view_loss_a", st, k_view_loss_a<false><<<tiles, VL_THREADS, 0, st>>>(p));
  GOF_LAUNCH_CHECK(false, st);
  if (p.grad) {
    if (p.mapping) GOF_LAUNCH("view_loss_b", st, k_view_loss_b<true><<<tiles, VL_THREADS, 0, st>>>(p));
    else GOF_LAUNCH("view_loss_b", st, k_view_loss_b<false><<<tiles, VL_THREADS, 0, st>>>(p));
    GOF_LAUNCH_CHECK(false, st);
  }
  GOF_LAUNCH("view_loss_c", st, k_view_loss_c<<<1, VL_THREADS, 0, st>>>(p.partial, tiles, (double)W * (double)H, N_l1, p.lam,
                                                                          p.lam_dn, p.lam_dist, terms));
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}

}  // namespace

// render [9,H,W], gt [3,H,W], terms [5] = (L1, SSIM, normal-consistency loss, distortion loss, total), grad [9,H,W] or NULL:
// device pointers.  c2w_R9: HOST pointer to the 3x3 camera-to-world rotation, row-major.
extern "C" GOF_API int gof_view_loss(int W, int H, const float* render, const float* gt, const float* c2w_R9, float fx, float fy,
                                     float lambda_dssim, float lambda_depth_normal, float lambda_distortion, float* terms,
                                     float* grad, void* scratch, void* stream) {
  if (view_loss_checked(W, H, render, gt, c2w_R9, fx, fy, terms, scratch) != GOF_OK) return GOF_E_INVALID;
  VlParams p;
  p.W = W; p.H = H; p.render = render; p.gt = gt; p.grad = grad;
  return view_loss_run(p, c2w_R9, fx, fy, lambda_dssim, lambda_depth_normal, lambda_distortion, terms, scratch, stream);
}

// gof_view_loss with the decoupled-appearance L1 (train.py:67-88): mapping [3,Hc,Wc] on the crop at (top, left) of the image,
// grad_mapping [3,Hc,Wc] = d total / d mapping, NULL exactly when grad is.  Device pointers.
extern "C" GOF_API int gof_view_loss_appearance(int W, int H, const float* render, const float* gt, const float* c2w_R9, float fx,
                                                float fy, float lambda_dssim, float lambda_depth_normal, float lambda_distortion,
                                                const float* mapping, int top, int left, int Hc, int Wc, float* terms, float* grad,
                                                float* grad_mapping, void* scratch, void* stream) {
  if (view_loss_checked(W, H, render, gt, c2w_R9, fx, fy, terms, scratch) != GOF_OK) return GOF_E_INVALID;
  if (!mapping) {
    gof_set_error("view_loss_appearance: mapping is NULL");
    return GOF_E_INVALID;
  }
  if (Hc < 1 || Wc < 1 || top < 0 || left < 0 || top > H - Hc || left > W - Wc) {
    gof_set_error("view_loss_appearance: the crop is empty or not inside the image");
    return GOF_E_INVALID;
  }
  if ((grad == nullptr) != (grad_mapping == nullptr)) {
    gof_set_error("view_loss_appearance: grad and grad_mapping must both be given or both be NULL");
    return GOF_E_INVALID;
  }
  VlParams p;
  p.W = W; p.H = H; p.render = render; p.gt = gt; p.grad = grad;
  p.mapping = mapping; p.grad_mapping = grad_mapping;
  p.top = top; p.left = left; p.Hc = Hc; p.Wc = Wc;
  p.inv_Na3 = 1.0f / (3.0f * (float)Hc * (float)Wc);
  return view_loss_run(p, c2w_R9, fx, fy, lambda_dssim, lambda_depth_normal, lambda_distortion, terms, scratch, stream);
}
