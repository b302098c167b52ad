// tests/hostmath/view_loss_app_host.cpp -- TEST INFRASTRUCTURE.  The per-view loss phases of
// gaussian-opacity-fields_b200/csrc/view_loss.cuh in their decoupled-appearance mode, compiled for the HOST and run the way
// the CUDA kernels do -- tile by tile, phase by phase, "thread" by thread -- with kernel C's fixed-order double sum and
// its division of the L1 sum by 3 Hc Wc.  Never loaded by the product.
#include <cstring>
#include <vector>

#include "../../gaussian-opacity-fields_b200/csrc/view_loss.cuh"

extern "C" int hm_view_loss_app(int W, int H, const float* render, const float* gt, const float* R9, float fx, float fy,
                                const float* g11, float lam, float lam_dn, float lam_dist, const float* mapping, int top, int left,
                                int Hc, int Wc, float* terms5, float* grad, float* grad_mapping) {
  VlParams p;
  p.W = W; p.H = H; p.tiles_x = (W + VL_TILE - 1) / VL_TILE; p.tiles_y = (H + VL_TILE - 1) / VL_TILE;
  p.render = render; p.gt = gt;
  memcpy(p.R, R9, sizeof(p.R)); memcpy(p.g, g11, sizeof(p.g));
  p.fx = fx; p.fy = fy; p.lam = lam; p.lam_dn = lam_dn; p.lam_dist = lam_dist;
  p.inv_N = 1.0f / ((float)W * (float)H); p.inv_N3 = 1.0f / (3.0f * (float)W * (float)H);
  p.mapping = mapping; p.grad_mapping = grad_mapping;
  p.top = top; p.left = left; p.Hc = Hc; p.Wc = Wc;
  p.inv_Na3 = 1.0f / (3.0f * (float)Hc * (float)Wc);
  std::vector<float> dmap((size_t)9 * W * H, 0.f), partial((size_t)p.tiles_x * p.tiles_y * 4, 0.f);
  p.dmap = dmap.data(); p.grad = grad; p.partial = partial.data();
  VlShared* s = new VlShared;
#define PHASE(call) for (int tid = 0; tid < VL_THREADS; ++tid) { call; }
  for (int ty = 0; ty < p.tiles_y; ++ty)
    for (int tx = 0; tx < p.tiles_x; ++tx) {           // kernel A, one block per tile
      PHASE(vl_a_zero(*s, tid));
      for (int ch = 0; ch < 3; ++ch) {
        PHASE(vl_a_load(p, *s, tx, ty, ch, tid));
        PHASE(vl_a_hblur(p, *s, tid));
        PHASE(vl_a_ssim(p, *s, tx, ty, ch, tid));
      }
      PHASE(vl_a_points(p, *s, tx, ty, tid));
      PHASE(vl_a_normals(p, *s, tx, ty, tid));
      PHASE(vl_a_pixel(p, *s, tx, ty, tid));
      for (int stride = VL_THREADS / 2; stride >= 1; stride >>= 1) PHASE(vl_a_reduce(p, *s, ty * p.tiles_x + tx, stride, tid));
    }
  if (grad)
    for (int ty = 0; ty < p.tiles_y; ++ty)
      for (int tx = 0; tx < p.tiles_x; ++tx)           // kernel B
        for (int ch = 0; ch < 3; ++ch) {
          PHASE(vl_b_load(p, *s, tx, ty, ch, tid));
          PHASE(vl_b_hblur(p, *s, tid));
          PHASE(vl_b_grad(p, *s, tx, ty, ch, tid));
        }
#undef PHASE
  delete s;
  double acc[4] = {0, 0, 0, 0};                        // kernel C: fixed-order sum in double
  for (size_t t = 0; t < (size_t)p.tiles_x * p.tiles_y; ++t)
    for (int q = 0; q < 4; ++q) acc[q] += (double)partial[t * 4 + q];
  const double N = (double)W * H, N_l1 = 3.0 * ((double)Hc * (double)Wc);
  const double ssim = acc[0] / (3 * N), l1 = acc[1] / N_l1, dnl = acc[2] / N, dist = acc[3] / N;
  terms5[0] = (float)l1; terms5[1] = (float)ssim; terms5[2] = (float)dnl; terms5[3] = (float)dist;
  terms5[4] = (float)((1.0 - lam) * l1 + lam * (1.0 - ssim) + lam_dn * dnl + lam_dist * dist);
  return 0;
}
