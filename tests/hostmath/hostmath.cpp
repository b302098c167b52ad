// tests/hostmath/hostmath.cpp -- TEST INFRASTRUCTURE.  Compiles the product's arithmetic header
// (gaussian-opacity-fields_b200/csrc/gof_math.cuh) for the HOST so that the `-m "not gpu"` suite can check the
// exact-rounding restatement against the CPU oracle without a GPU.  Never loaded by the product.
#include <cstring>

#include "../../gaussian-opacity-fields_b200/csrc/gof_math.cuh"

extern "C" {

// one Gaussian through the forward-preprocess arithmetic; returns 0 if culled
int hm_preprocess_one(const float* mean, const float* scale, const float* rot, float opacity, float mod,
                      const float* vm, const float* pm, int W, int H, float tan_fovx, float tan_fovy,
                      float kernel_size, float* out_cov3D, float* out_conic_opacity, float* out_means2D,
                      float* out_depth, int* out_radius, unsigned* out_tiles, float* out_v2g) {
  const float focal_y = H / (2.0f * tan_fovy), focal_x = W / (2.0f * tan_fovx);
  const int gx = (W + 15) / 16, gy = (H + 15) / 16;
  const float px = mean[0], py = mean[1], pz = mean[2];
  const float tz = gof_affine(px, py, pz, vm[2], vm[6], vm[10], vm[14]);
  if (tz <= 0.2f) return 0;
  const float hx = gof_affine(px, py, pz, pm[0], pm[4], pm[8], pm[12]);
  const float hy = gof_affine(px, py, pz, pm[1], pm[5], pm[9], pm[13]);
  const float hw = gof_affine(px, py, pz, pm[3], pm[7], pm[11], pm[15]);
  const float p_w = F_RCP(F_ADD(hw, 0.0000001f));
  const GofRot R = gof_quat_to_rot(rot[0], rot[1], rot[2], rot[3]);
  gof_cov3d(R, scale[0], scale[1], scale[2], mod, out_cov3D);
  const float tx = gof_affine(px, py, pz, vm[0], vm[4], vm[8], vm[12]);
  const float ty = gof_affine(px, py, pz, vm[1], vm[5], vm[9], vm[13]);
  const GofCov2D cov = gof_cov2d(tx, ty, tz, focal_x, focal_y, tan_fovx, tan_fovy, kernel_size, out_cov3D, vm);
  if (cov.det == 0.0f) return 0;
  const float mid = F_MUL(F_ADD(cov.a, cov.c), 0.5f);
  const float sq = F_SQRT(fmaxf(F_FMA(mid, mid, -cov.det), 0.1f));
  const float rad_f = ceilf(F_MUL(F_SQRT(fmaxf(F_ADD(mid, sq), F_SUB(mid, sq))), 3.0f));
  const int radius = gof_f2i_rz(rad_f);
  const float pix_x = gof_ndc2pix(F_MUL(hx, p_w), W), pix_y = gof_ndc2pix(F_MUL(hy, p_w), H);
  uint32_t x0, y0, x1, y1;
  gof_get_rect(pix_x, pix_y, radius, gx, gy, &x0, &y0, &x1, &y1);
  if ((x1 - x0) * (y1 - y0) == 0) return 0;
  const float det_inv = F_RCP(cov.det);
  out_conic_opacity[0] = F_MUL(cov.c, det_inv);
  out_conic_opacity[1] = F_MUL(det_inv, -cov.b);
  out_conic_opacity[2] = F_MUL(cov.a, det_inv);
  out_conic_opacity[3] = F_MUL(cov.coef, opacity);
  out_means2D[0] = pix_x; out_means2D[1] = pix_y;
  *out_depth = tz;
  *out_radius = radius;
  *out_tiles = (y1 - y0) * (x1 - x0);
  gof_view2gaussian(R, scale[0], scale[1], scale[2], px, py, pz, vm, out_v2g);
  return 1;
}

// one (pixel, Gaussian) pair: out = (AA, BB, t, power, mapped_t, normal_length, n0, n1, n2)
void hm_pair(const float* v2g, unsigned pix_x, unsigned pix_y, int W, int H, float focal_x, float focal_y, float* out) {
  const float rx = gof_ray(pix_x, W, focal_x), ry = gof_ray(pix_y, H, focal_y);
  const GofPair p = gof_pair_geom(v2g, rx, ry);
  out[0] = p.AA; out[1] = p.BB; out[2] = gof_pair_t(p); out[3] = gof_pair_power(p, v2g[9]);
  out[4] = gof_mapped_t(out[2]); out[5] = gof_normal_length(p); out[6] = p.n0; out[7] = p.n1; out[8] = p.n2;
}

// conservative cull box of one Gaussian (gof_cull_bbox); scale may be NULL (then no box: full plane); margin_px is 0 for
// the blend's centre rays and 0.5 for the five rays of the opacity-field query
void hm_bbox_margin(const float* v2g, float opacity, const float* scale, int W, int H, float tan_fovx, float tan_fovy,
                    float margin_px, int* out) {
  const float focal_y = H / (2.0f * tan_fovy), focal_x = W / (2.0f * tan_fovx);
  double lam = 0.0;
  if (scale) {
    lam = 1e300;
    for (int k = 0; k < 3; ++k) { const double si = 1.0 / ((double)scale[k] * scale[k] + 1e-7); lam = si < lam ? si : lam; }
  }
  const GofBox b = gof_cull_bbox(v2g, opacity, lam, W, H, focal_x, focal_y, tan_fovx, tan_fovy, margin_px);
  out[0] = b.x0; out[1] = b.y0; out[2] = b.x1; out[3] = b.y1;
}

// the blend's box (margin 0)
void hm_bbox(const float* v2g, float opacity, const float* scale, int W, int H, float tan_fovx, float tan_fovy, int* out) {
  hm_bbox_margin(v2g, opacity, scale, W, H, tan_fovx, tan_fovy, 0.0f, out);
}

void hm_sh(int deg, const float* mean, const float* campos, const float* sh, float* rgb, unsigned char* clamped) {
  gof_sh_to_rgb(deg, mean[0], mean[1], mean[2], campos, sh, rgb, clamped);
}

// the pixel of thread (warp, lane) in tile (tile_x, tile_y): out = (wx0, wy0, pix_x, pix_y)
void hm_warp_block(int tile_x, int tile_y, int warp, int lane, int* out) {
  const GofWarpBlock b = gof_warp_block(tile_x, tile_y, warp, lane);
  out[0] = b.wx0; out[1] = b.wy0; out[2] = (int)b.pix_x; out[3] = (int)b.pix_y;
}

int hm_pixel_slot(int lx, int ly) { return gof_pixel_slot(lx, ly); }

// n points: slot[i] = gof_point_slot(xy[2i], xy[2i+1], tile[2i], tile[2i+1])
void hm_point_slots(int n, const float* xy, const int* tile, int* slot) {
  for (int i = 0; i < n; ++i) slot[i] = gof_point_slot(xy[2 * i], xy[2 * i + 1], tile[2 * i], tile[2 * i + 1]);
}

// n boxes (x0, y0, x1, y1) packed into the record's words, each tested against the 8x4 block at rect (wx0, wy0):
// words[2i..2i+1] = (lo, hi), hit[i] = gof_box_hits
void hm_box_hits(int n, const int* box, const int* rect, unsigned* words, int* hit) {
  for (int i = 0; i < n; ++i) {
    GofBox b;
    b.x0 = box[4 * i]; b.y0 = box[4 * i + 1]; b.x1 = box[4 * i + 2]; b.y1 = box[4 * i + 3];
    uint32_t lo, hi;
    gof_box_pack(b, &lo, &hi);
    words[2 * i] = lo; words[2 * i + 1] = hi;
    const int wx0 = rect[2 * i], wy0 = rect[2 * i + 1];
    hit[i] = gof_box_hits(lo, hi, wx0, wy0, wx0 + 7, wy0 + 3);
  }
}
}
