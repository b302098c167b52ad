/* Float64 oracle of the opacity-field query's backward (DESIGN.md 4.11).  TEST INFRASTRUCTURE.
 *
 * For one point with ray (rx, ry), depth d and a fixed contributor list, the query integrates
 *   A = sum_j alpha_j T_j = 1 - prod_j (1 - alpha_j),   alpha_j = min(0.99, op_j exp(power_j)),  alpha_j >= 1/255 kept,
 *   power_j = -1/2 (AA t^2 + BB t + CC),  t = min(-BB / (2 AA), d),  AA = r^T Sigma r,  BB = 2 b.r,  r = (rx, ry, 1).
 * With the list, the rejects and both clamps held fixed, dA/dalpha_j = T / (1 - alpha_j) (T = prod_i (1 - alpha_i)) and
 * dalpha_j/dpower_j = alpha_j where alpha_j is not clamped (0 where it is); power_j is differentiated with t held fixed (t is
 * stationary where it is not clamped), plus d power / d d = -(AA t + BB / 2) where it is clamped to the depth.  The ray is
 * rx = tx / (tz + 1e-7), ry = ty / (tz + 1e-7) and d = tz, (tx, ty, tz) = the view matrix applied to the point.
 *
 * The alphas are evaluated in float with the forward's operations (host expf); everything after them in double.  Error
 * scales, per output component: mag = sum over the point's pairs of |term| * (1 + K), K = sum_i 1 / (1 - alpha_i) -- an alpha
 * that is a few ulp off moves T by alpha / (1 - alpha) of that, and each term by as much.  A point is `marginal` when one of the
 * decisions it depends on (pass 1 at its pixel: t against 0.2, alpha against 1/255, T against 1e-4; its own pass: alpha
 * against 1/255 and against 0.99) lies within 8 ulp of its threshold (for T, the accumulated error of oracle_integrate).  What
 * such a decision can change if it flips is returned as an allowance (see igo_point_checked and igo_view). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define MAX_CONTRIB 1024
#define ALPHA_MIN (1.0f / 255.0f)
#define ALPHA_MAX 0.99f

static int near(float x, float thr, float ulps) { return fabsf(x - thr) <= ulps * 5.9604645e-8f * 2.f * fabsf(thr); }

/* pass 1's pair geometry of ray k: the forward's fusion pattern of each unrolled ray (integrate.cu pair_geom_k) */
static void geom_k(int k, const float* v, float rx, float ry, float* AA, float* BB) {
  float n0, n1, n2, bh;
  if (k == 0) {
    n0 = fmaf(rx, v[0], ry * v[1]) + v[2];
    n1 = fmaf(rx, v[1], ry * v[3]) + v[4];
    n2 = fmaf(ry, v[4], rx * v[2]) + v[5];
    bh = fmaf(rx, v[6], ry * v[7]) + v[8];
  } else {
    n0 = (rx * v[0] + ry * v[1]) + v[2];
    n1 = (k == 1 || k == 3) ? fmaf(rx, v[1], ry * v[3]) + v[4] : (ry * v[3] + rx * v[1]) + v[4];
    n2 = fmaf(rx, v[2], ry * v[4]) + v[5];
    bh = (rx * v[6] + ry * v[7]) + v[8];
  }
  *AA = fmaf(rx, n0, ry * n1) + n2;
  *BB = bh + bh;
}

static const float OFFX[5] = {0.0f, -0.5f, 0.5f, -0.5f, 0.5f};
static const float OFFY[5] = {0.0f, -0.5f, -0.5f, 0.5f, 0.5f};

/* pass 1 at pixel (px, py): the contributor list as the query reads it (tile-list positions, uint16 semantics of the forward:
 * the list ends at the first id that does not increase), returns its length; *marg = 1 if a decision lies near its threshold */
static int pass1(int W, int H, float fx, float fy, int px, int py, const uint32_t* range, const uint32_t* point_list,
                 const float* v2g, const float* conic_opacity, uint32_t* list, int* marg, uint32_t* unc, int* n_unc, int* hard) {
  const float pfx = (float)px + 0.5f, pfy = (float)py + 0.5f;
  float rxk[5], ryk[5], Ts[5] = {1, 1, 1, 1, 1}, Terr[5] = {0, 0, 0, 0, 0};
  for (int k = 0; k < 5; ++k) {
    rxk[k] = (float)(((double)(pfx + OFFX[k]) - W * 0.5) / fx);
    ryk[k] = (float)(((double)(pfy + OFFY[k]) - H * 0.5) / fy);
  }
  int n = 0;
  uint32_t contributor = 0;
  for (uint32_t kk = range[0]; kk < range[1] && n < MAX_CONTRIB; ++kk) {
    contributor++;
    const uint32_t g = point_list[kk];
    const float* v = v2g + 10 * (size_t)g;
    const float op = conic_opacity[4 * (size_t)g + 3];
    int used = 0, cm = 0;
    for (int k = 0; k < 5; ++k) {
      float AA, BB;
      geom_k(k, v, rxk[k], ryk[k], &AA, &BB);
      const float t = -BB / (AA + AA);
      if (near(t, 0.2f, 8.f)) cm = 1;
      if (t < 0.2f) continue;
      float power = (float)(-0.5 * fma((double)(-BB / AA), (double)BB * 0.25, (double)v[9]));
      if (power > 0.0f) power = 0.0f;
      const float al = fminf(op * expf(power), ALPHA_MAX);
      if (near(al, ALPHA_MIN, 8.f)) cm = 1;
      if (al < ALPHA_MIN) continue;
      const float tt = Ts[k] * (1.0f - al);
      const float terr = Terr[k] + (8.f * al / (1 - al) + 2.f) * 5.9604645e-8f;
      /* a T decision that may flip changes every later decision of the ray: no allowance covers that */
      if (fabsf(tt - 0.0001f) <= 2.f * terr * 0.0001f) { *marg = 1; *hard = 1; }
      if (tt < 0.0001f) continue;
      Terr[k] = terr;
      Ts[k] = tt;
      used = 1;
    }
    if (cm) {   /* this Gaussian may be in the forward's list or not, whichever way the oracle decided */
      *marg = 1;
      if (*n_unc < MAX_CONTRIB) unc[(*n_unc)++] = g;
      else *hard = 1;
    }
    if (used) list[n++] = kk;
  }
  /* the forward reads the recorded uint16 ids up to the first one that does not increase, and gathers the Gaussian at the
   * TRUNCATED id: past 65 535 list entries that is another Gaussian of the tile list than the one recorded */
  uint32_t prev = 0;
  int m = 0;
  for (; m < n; ++m) {
    const uint32_t id16 = (list[m] - range[0] + 1) & 0xffffu;
    if (id16 <= prev) break;
    prev = id16;
    list[m] = range[0] + id16 - 1;
  }
  return m;
}

/* The float alpha of Gaussian v at the point's ray, as the forward evaluates it, and the derivative pieces of its term. */
typedef struct {
  float al, raw;
  int clamped;
  double jv[10];   /* d power / d v2g times -2 */
  double drx, dry, dd, mrx, mry, md;   /* d power / d(rx, ry, depth) and their magnitudes */
} pair_t;

static pair_t pair_eval(const float* v, float op, float rx, float ry, float depth) {
  pair_t e;
  const float n0 = v[2] + fmaf(v[0], rx, v[1] * ry), n1 = v[4] + fmaf(v[1], rx, v[3] * ry), n2 = v[5] + fmaf(v[4], ry, v[2] * rx);
  const float AA = fmaf(n0, rx, n1 * ry) + n2, bh = v[8] + fmaf(v[6], rx, v[7] * ry), BB = bh + bh;
  float t = -BB / (AA + AA);
  e.clamped = t > depth;
  if (e.clamped) t = depth;
  const float power = (v[9] + fmaf(BB, t, t * (AA * t))) * -0.5f;
  e.raw = op * expf(power);
  e.al = fminf(e.raw, ALPHA_MAX);
  const double x = rx, y = ry, tt = t;
  const double jv[10] = {tt * tt * x * x, 2 * tt * tt * x * y, 2 * tt * tt * x, tt * tt * y * y, 2 * tt * tt * y, tt * tt,
                         2 * tt * x, 2 * tt * y, 2 * tt, 1.0};
  memcpy(e.jv, jv, sizeof jv);
  const double N0 = (double)v[0] * x + (double)v[1] * y + v[2], N1 = (double)v[1] * x + (double)v[3] * y + v[4];
  e.drx = -(tt * tt * N0 + tt * v[6]);
  e.dry = -(tt * tt * N1 + tt * v[7]);
  e.mrx = tt * tt * fabs(N0) + fabs(tt * v[6]);
  e.mry = tt * tt * fabs(N1) + fabs(tt * v[7]);
  e.dd = e.md = 0.0;
  if (e.clamped) {
    const double AAd = (double)v[0] * x * x + 2.0 * v[1] * x * y + 2.0 * v[2] * x + (double)v[3] * y * y + 2.0 * v[4] * y + v[5];
    const double bhd = (double)v[6] * x + (double)v[7] * y + v[8];
    e.dd = -(AAd * tt + bhd);
    e.md = fabs(AAd * tt) + fabs(bhd);
  }
  return e;
}

/* d(rx, ry, depth) -> d points3D, and the same map on magnitudes */
static void point_chain(const float* p3, const float* vm, double s, double grx, double gry, double gd, double mrx, double mry, double md,
                        double* dpts, double* mag) {
  const double px = p3[0], py = p3[1], pz = p3[2];
  const double tx = vm[0] * px + vm[4] * py + vm[8] * pz + vm[12];
  const double ty = vm[1] * px + vm[5] * py + vm[9] * pz + vm[13];
  const double tz = vm[2] * px + vm[6] * py + vm[10] * pz + vm[14];
  const double den = tz + 1e-7, a = fabs(s);
  const double dtx = s * grx / den, dty = s * gry / den, dtz = s * gd - s * (grx * tx + gry * ty) / (den * den);
  const double mtx = a * mrx / fabs(den), mty = a * mry / fabs(den), mtz = a * md + a * (mrx * fabs(tx) + mry * fabs(ty)) / (den * den);
  for (int i = 0; i < 3; ++i) {
    if (dpts) dpts[i] = vm[4 * i] * dtx + vm[4 * i + 1] * dty + vm[4 * i + 2] * dtz;
    mag[i] = fabs(vm[4 * i]) * mtx + fabs(vm[4 * i + 1]) * mty + fabs(vm[4 * i + 2]) * mtz;
  }
}

/* One point over a fixed list of Gaussians g[0..n): see the header.  dv2g / mag_g ([P][10]) are accumulated; returns A in float
 * as the forward computes it.  Marginal decisions: gu[0..nu) are Gaussians that pass 1 may have recorded or not (NULL: none);
 * with allow_g ([P][10]) / allow_pts ([3]) non-NULL and the point marginal, they receive what a flip of any such decision, or of
 * one of the point's own near-threshold alphas, can change: the flipped Gaussian's whole term, and every other term scaled by
 * T's change, at most prod_u (1 + alpha_u / (1 - alpha_u)) - 1. */
float igo_point_checked(int n, const uint32_t* g, int nu, const uint32_t* gu, const float* v2g, const float* opac, float rx, float ry,
                        float depth, const float* p3, const float* vm, double dLdA, double* dpts, double* mag_pts, double* dv2g,
                        double* mag_g, double* allow_g, double* allow_pts, int* marginal) {
  double T = 1.0, K = 0.0, F = 1.0;   /* F: prod over the uncertain Gaussians of 1 + alpha / (1 - alpha) */
  float A = 0.f, Tf = 1.f;
  for (int j = 0; j < n; ++j) {   /* walk 1: T and K */
    const pair_t e = pair_eval(v2g + 10 * (size_t)g[j], opac[g[j]], rx, ry, depth);
    if (near(e.al, ALPHA_MIN, 8.f) || near(e.raw, ALPHA_MAX, 8.f)) {
      *marginal = 1;
      F *= 1.0 + (double)e.al / (1.0 - (double)e.al);
    }
    if (e.al < ALPHA_MIN) continue;
    A = fmaf(e.al, Tf, A);
    Tf = Tf * (1.0f - e.al);
    T *= 1.0 - (double)e.al;
    K += 1.0 / (1.0 - (double)e.al);
  }
  for (int u = 0; u < nu; ++u) {
    const pair_t e = pair_eval(v2g + 10 * (size_t)gu[u], opac[gu[u]], rx, ry, depth);
    F *= 1.0 + (double)e.al / (1.0 - (double)e.al);
  }
  const int allow = *marginal && allow_g;
  const double s = dLdA * T, dF = F - 1.0;
  double grx = 0, gry = 0, gd = 0, mrx = 0, mry = 0, md = 0, arx = 0, ary = 0, ad = 0;
  for (int j = 0; j < n + (allow ? nu : 0); ++j) {   /* walk 2: the terms (then, for the allowance, the uncertain Gaussians) */
    const int extra = j >= n;
    const uint32_t gj = extra ? gu[j - n] : g[j];
    const pair_t e = pair_eval(v2g + 10 * (size_t)gj, opac[gj], rx, ry, depth);
    const int own = extra || near(e.al, ALPHA_MIN, 8.f) || near(e.raw, ALPHA_MAX, 8.f);   /* a term that may appear or vanish */
    if (!own && (e.al < ALPHA_MIN || e.raw > ALPHA_MAX)) continue;
    const double w = (double)e.al / (1.0 - (double)e.al);
    const double f = -0.5 * s * w;   /* dL/dpower times -1/2 */
    const double scale = own ? F : dF;   /* the allowance: the whole term, or its change with T */
    if (allow)
      for (int k = 0; k < 10; ++k) allow_g[10 * (size_t)gj + k] += fabs(f * e.jv[k]) * scale * 1.01;
    if (allow) { arx += w * e.mrx * scale * 1.01; ary += w * e.mry * scale * 1.01; ad += w * e.md * scale * 1.01; }
    if (extra || e.al < ALPHA_MIN || e.raw > ALPHA_MAX) continue;
    for (int k = 0; k < 10; ++k) {
      dv2g[10 * (size_t)gj + k] += f * e.jv[k];
      mag_g[10 * (size_t)gj + k] += fabs(f * e.jv[k]) * (1.0 + K);
    }
    grx += w * e.drx; gry += w * e.dry; gd += w * e.dd;
    mrx += w * e.mrx * (1.0 + K); mry += w * e.mry * (1.0 + K); md += w * e.md * (1.0 + K);
  }
  point_chain(p3, vm, s, grx, gry, gd, mrx, mry, md, dpts, mag_pts);
  if (allow_pts) {
    if (allow) point_chain(p3, vm, s, 0, 0, 0, arx, ary, ad, NULL, allow_pts);
    else allow_pts[0] = allow_pts[1] = allow_pts[2] = 0.0;
  }
  return A;
}

float igo_point(int n, const uint32_t* g, const float* v2g, const float* opac, float rx, float ry, float depth, const float* p3,
                const float* vm, double dLdA, double* dpts, double* mag_pts, double* dv2g, double* mag_g, int* marginal) {
  return igo_point_checked(n, g, 0, NULL, v2g, opac, rx, ry, depth, p3, vm, dLdA, dpts, mag_pts, dv2g, mag_g, NULL, NULL, marginal);
}

/* The whole view: every point that projects (ok[i]; xy / depth as the forward computes them) against its pixel's pass-1 list.
 * Outputs: alpha [PN] (float, the forward's value), dpts / mag_pts / allow_pts [PN][3], marg_pt [PN] (0, 1 marginal, 2 with a
 * transmittance decision that may flip), n_list [PN] (list length);
 * dv2g / mag_g / allow_g [P][10].  A marginal point's terms are kept, and what its uncertain decisions can change goes to
 * allow_g / allow_pts; only where a transmittance decision of pass 1 may flip (every later decision of that ray with it) are its
 * terms left out instead, and marg_g [P] = 1 for every Gaussian of its tile. */
void igo_view(int W, int H, float tan_fovx, float tan_fovy, const float* vm, int P, int PN, const float* points3D, const float* xy,
              const float* depth, const unsigned char* ok, const uint32_t* ranges, const uint32_t* point_list, const float* v2g,
              const float* conic_opacity, const float* dL_dalpha, float* alpha, double* dpts, double* mag_pts, double* allow_pts,
              unsigned char* marg_pt, uint32_t* n_list, double* dv2g, double* mag_g, double* allow_g, unsigned char* marg_g) {
  const float fy = H / (2.0f * tan_fovy), fx = W / (2.0f * tan_fovx);
  const int gx = (W + 15) / 16;
  float* opac = (float*)malloc(((size_t)P + 1) * sizeof(float));
  for (int i = 0; i < P; ++i) opac[i] = conic_opacity[4 * (size_t)i + 3];
  uint32_t* list = (uint32_t*)malloc(MAX_CONTRIB * sizeof(uint32_t));
  uint32_t* gl = (uint32_t*)malloc(MAX_CONTRIB * sizeof(uint32_t));
  uint32_t* unc = (uint32_t*)malloc(MAX_CONTRIB * sizeof(uint32_t));
  double* hd = (double*)calloc((size_t)P * 10 + 1, sizeof(double));   /* terms of a hard-marginal point, dropped */
  double* hm = (double*)calloc((size_t)P * 10 + 1, sizeof(double));
  int last_pix = -1, n = 0, nu = 0, pmarg = 0, phard = 0;
  /* the caller passes the points sorted by pixel, so each pixel's list is computed once */
  for (int i = 0; i < PN; ++i) {
    if (!ok[i]) continue;
    const int px = (int)xy[2 * (size_t)i], py = (int)xy[2 * (size_t)i + 1];
    const int pix = py * W + px;
    if (pix != last_pix) {
      last_pix = pix;
      pmarg = phard = nu = 0;
      const uint32_t* range = ranges + 2 * ((size_t)(py / 16) * gx + (px / 16));
      n = pass1(W, H, fx, fy, px, py, range, point_list, v2g, conic_opacity, list, &pmarg, unc, &nu, &phard);
      for (int j = 0; j < n; ++j) gl[j] = point_list[list[j]];
    }
    const float rx = (float)(((double)xy[2 * (size_t)i] - W * 0.5) / fx);
    const float ry = (float)(((double)xy[2 * (size_t)i + 1] - H * 0.5) / fy);
    int marg = pmarg;
    const int hard = phard;
    alpha[i] = igo_point_checked(n, gl, nu, unc, v2g, opac, rx, ry, depth[i], points3D + 3 * (size_t)i, vm, (double)dL_dalpha[i],
                                 dpts + 3 * (size_t)i, mag_pts + 3 * (size_t)i, hard ? hd : dv2g, hard ? hm : mag_g,
                                 hard ? NULL : allow_g, allow_pts + 3 * (size_t)i, &marg);
    marg_pt[i] = (unsigned char)(hard ? 2 : marg);
    n_list[i] = (uint32_t)n;
    if (hard) {   /* the forward's list may hold any Gaussian of the tile */
      const uint32_t* range = ranges + 2 * ((size_t)(py / 16) * gx + (px / 16));
      for (uint32_t kk = range[0]; kk < range[1]; ++kk) marg_g[point_list[kk]] = 1;
    }
  }
  free(opac); free(list); free(gl); free(unc); free(hd); free(hm);
}
