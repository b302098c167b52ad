/* Float64 oracle of the opacity-field query's colour backward (DESIGN.md 4.13).  TEST INFRASTRUCTURE.
 *
 * It builds on integrate_grad_oracle.c (the alpha backward's oracle, included as it is): that file's restatement of pass 1 --
 * the five rays' fusion pattern (geom_k) and the marginal / transmittance flags (pass1) -- is the one used here. */
#include "integrate_grad_oracle.c"

/* ---- the colour of the query (DESIGN.md 4.13) ----
 * color_integrated of a point is its pixel's C + T bg on pass 1's centre ray r = (rx0, ry0, 1): over the pairs j the centre ray
 * blended, in list order, C_c = sum_j T_j alpha_j c_jc + T bg_c with T_j = prod_{i<j} (1 - alpha_i), each pair at its stationary
 * point t* = -BB / (2 AA), alpha_j = min(0.99, op exp(min(0, power_j))), power_j = -1/2 (CC - BB^2 / (4 AA)).  With the blended
 * set, the rejects and both clamps held fixed:
 *   dC_c / dc_jc = T_j alpha_j,   dC_c / dalpha_j = T_j c_jc - (sum_{i>j} T_i alpha_i c_ic + T bg_c) / (1 - alpha_j),
 *   dalpha_j / dpower_j = alpha_j (0 where alpha or power is clamped),  dpower / d(AA, BB, CC) = -1/2 (t*^2, t*, 1).
 * Error scale of each output component: the term's magnitude times (1 + K), K = sum_j 1 / (1 - alpha_j), as for the alpha. */

/* The centre ray of pass 1 at pixel (px, py): the Gaussians it blended, in order (true ids: no uint16 wrap, the cap of
 * pass 1's five rays included), their float alphas and stationary points; returns their number.  *near_c = 1 if one of the
 * centre ray's own decisions that rest on expf (alpha against 1/255 and 0.99, T against 1e-4) lies near its threshold; t and
 * power are formed by the same IEEE operations on host and device.  *capped = 1 if pass 1 reached its 1 024 contributors. */
static int centre_ray(int W, int H, float fx, float fy, int px, int py, const uint32_t* range, const uint32_t* point_list,
                      const float* v2g, const float* conic_opacity, uint32_t* cg, float* cal, float* ct, int* near_c, int* capped) {
  const float pfx = (float)px + 0.5f, pfy = (float)py + 0.5f;
  float rxk[5], ryk[5], Ts[5] = {1, 1, 1, 1, 1};
  for (int k = 0; k < 5; ++k) {
    rxk[k] = (float)(((double)(pfx + OFFX[k]) - W * 0.5) / fx);
    ryk[k] = (float)(((double)(pfy + OFFY[k]) - H * 0.5) / fy);
  }
  int n = 0, nc = 0;
  float terr = 0.f;   /* the centre T's accumulated error, as in pass1 */
  for (uint32_t kk = range[0]; kk < range[1] && n < MAX_CONTRIB; ++kk) {
    const uint32_t g = point_list[kk];
    const float* v = v2g + 10 * (size_t)g;
    const float op = conic_opacity[4 * (size_t)g + 3];
    int used = 0;
    for (int k = 0; k < 5; ++k) {
      float AA, BB;
      geom_k(k, v, rxk[k], ryk[k], &AA, &BB);
      const float t = -BB / (AA + AA);
      if (t < 0.2f) continue;
      float power = (float)(-0.5 * fma((double)(-BB / AA), (double)BB * 0.25, (double)v[9]));
      if (power > 0.0f) power = 0.0f;
      const float raw = op * expf(power);
      const float al = fminf(raw, ALPHA_MAX);
      if (k == 0 && (near(al, ALPHA_MIN, 8.f) || near(raw, ALPHA_MAX, 8.f))) *near_c = 1;
      if (al < ALPHA_MIN) continue;
      const float tt = Ts[k] * (1.0f - al);
      const float te = terr + (8.f * al / (1 - al) + 2.f) * 5.9604645e-8f;
      if (k == 0 && fabsf(tt - 0.0001f) <= 2.f * te * 0.0001f) *near_c = 1;
      if (tt < 0.0001f) continue;
      if (k == 0) terr = te;
      Ts[k] = tt;
      used = 1;
      if (k == 0) { cg[nc] = g; cal[nc] = al; ct[nc] = t; ++nc; }
    }
    if (used) ++n;
  }
  *capped = n >= MAX_CONTRIB;
  return nc;
}

/* One pixel over its centre ray's blended Gaussians g[0..n) (alphas al, stationary points t), dL/dC [3]: accumulates dL/dcolor
 * into dcol / mag_c ([P][3]) and dL/dview2gaussian into dv2g / mag_g ([P][10]); returns C in double in C_out [3]. */
void igc_pixel(int n, const uint32_t* g, const float* al, const float* tst, const float* v2g, const float* opac, const float* rgb,
               float rx, float ry, const float* bg, const double* dLdC, double* dcol, double* mag_c, double* dv2g, double* mag_g,
               double* C_out) {
  double T = 1.0, K = 0.0, tot[3] = {0, 0, 0};
  for (int j = 0; j < n; ++j) {
    const double a = al[j];
    for (int c = 0; c < 3; ++c) tot[c] += T * a * rgb[3 * (size_t)g[j] + c];
    T *= 1.0 - a;
    K += 1.0 / (1.0 - a);
  }
  for (int c = 0; c < 3; ++c) { tot[c] += T * bg[c]; if (C_out) C_out[c] = tot[c]; }
  double Tj = 1.0, pre[3] = {0, 0, 0};
  for (int j = 0; j < n; ++j) {
    const uint32_t gj = g[j];
    const double a = al[j], w = Tj * a, om = 1.0 - a;
    double dal = 0.0, mal = 0.0;
    for (int c = 0; c < 3; ++c) {
      const double cc = rgb[3 * (size_t)gj + c];
      pre[c] += w * cc;
      const double S = tot[c] - pre[c];
      dcol[3 * (size_t)gj + c] += w * dLdC[c];
      mag_c[3 * (size_t)gj + c] += fabs(w * dLdC[c]) * (1.0 + K);
      dal += dLdC[c] * (Tj * cc - S / om);
      mal += fabs(dLdC[c]) * (Tj * fabs(cc) + fabs(S) / om);
    }
    Tj *= om;
    /* the derivative exists where neither alpha (0.99) nor power (0) was clamped */
    const float* v = v2g + 10 * (size_t)gj;
    float AA, BB;
    geom_k(0, v, rx, ry, &AA, &BB);
    const float power = (float)(-0.5 * fma((double)(-BB / AA), (double)BB * 0.25, (double)v[9]));
    if (power > 0.0f || opac[gj] * expf(power) > ALPHA_MAX) continue;
    const double x = rx, y = ry, t = tst[j];
    const double jv[10] = {t * t * x * x, 2 * t * t * x * y, 2 * t * t * x, t * t * y * y, 2 * t * t * y, t * t, 2 * t * x, 2 * t * y,
                           2 * t, 1.0};
    const double f = -0.5 * dal * a, mf = 0.5 * mal * a;
    for (int k = 0; k < 10; ++k) {
      dv2g[10 * (size_t)gj + k] += f * jv[k];
      mag_g[10 * (size_t)gj + k] += mf * fabs(jv[k]) * (1.0 + K);
    }
  }
}

/* The whole view: every pixel with a non-zero dL/dC (dLdC [H][W][3], the sum of its points' dL/dcolor_integrated).  Outputs
 * dcol / mag_c [P][3], dv2g / mag_g [P][10], marg_g [P], C [H][W][3] (the oracle's colour).  Left out (marg_g): the Gaussians of a
 * pixel where a decision of its centre ray lies near its threshold; where pass 1 reached the cap, the decisions of the other
 * rays move the cap too, so there pass 1's marginal flags count (its transmittance flag: every Gaussian of the tile). */
void igc_view(int W, int H, float tan_fovx, float tan_fovy, int P, const uint32_t* ranges, const uint32_t* point_list,
              const float* v2g, const float* conic_opacity, const float* rgb, const float* bg, const double* dLdC, double* dcol,
              double* mag_c, double* dv2g, double* mag_g, unsigned char* marg_g, double* C) {
  const float fy = H / (2.0f * tan_fovy), fx = W / (2.0f * tan_fovx);
  const int gx = (W + 15) / 16;
  float* opac = (float*)malloc(((size_t)P + 1) * sizeof(float));
  for (int i = 0; i < P; ++i) opac[i] = conic_opacity[4 * (size_t)i + 3];
  uint32_t* list = (uint32_t*)malloc(MAX_CONTRIB * sizeof(uint32_t));
  uint32_t* unc = (uint32_t*)malloc(MAX_CONTRIB * sizeof(uint32_t));
  uint32_t* cg = (uint32_t*)malloc(MAX_CONTRIB * sizeof(uint32_t));
  float* cal = (float*)malloc(MAX_CONTRIB * sizeof(float));
  float* ct = (float*)malloc(MAX_CONTRIB * sizeof(float));
  for (int py = 0; py < H; ++py)
    for (int px = 0; px < W; ++px) {
      const double* d = dLdC + 3 * ((size_t)py * W + px);
      if (d[0] == 0.0 && d[1] == 0.0 && d[2] == 0.0) continue;
      const uint32_t* range = ranges + 2 * ((size_t)(py / 16) * gx + (px / 16));
      int marg = 0, hard = 0, nu = 0, near_c = 0, capped = 0;
      const int n = centre_ray(W, H, fx, fy, px, py, range, point_list, v2g, conic_opacity, cg, cal, ct, &near_c, &capped);
      if (capped) pass1(W, H, fx, fy, px, py, range, point_list, v2g, conic_opacity, list, &marg, unc, &nu, &hard);
      const float rx = (float)(((double)((float)px + 0.5f) - W * 0.5) / fx);
      const float ry = (float)(((double)((float)py + 0.5f) - H * 0.5) / fy);
      igc_pixel(n, cg, cal, ct, v2g, opac, rgb, rx, ry, bg, d, dcol, mag_c, dv2g, mag_g, C + 3 * ((size_t)py * W + px));
      if (hard) {
        for (uint32_t kk = range[0]; kk < range[1]; ++kk) marg_g[point_list[kk]] = 1;
      } else if (marg || near_c) {
        for (int j = 0; j < n; ++j) marg_g[cg[j]] = 1;
        for (int u = 0; u < nu; ++u) marg_g[unc[u]] = 1;
      }
    }
  free(opac); free(list); free(unc); free(cg); free(cal); free(ct);
}
