/* Float64 oracle of the per-pixel ray gradient dL/drx, dL/dry of the blend backward (DESIGN.md 4.10).  TEST INFRASTRUCTURE.
 *
 * It walks every pixel like the blend backward (backward.cu:634-955): the pixel's blended pairs are the entries of its tile list
 * before n_contrib[0] that pass the forward's float tests (t > 0.2, alpha >= 1/255), and its gradient terms are formed back to
 * front.  Unlike the C oracle of the parameter gradients, every per-pair quantity after the pair geometry is evaluated in double
 * from scratch: T is the forward product of (1 - alpha) in double, not recovered from the float final T.  For each pair
 *
 *   dL/drx += dnrm . (v0, v1, v2) + dA n0 + dB2 v6,   dL/dry += dnrm . (v1, v3, v4) + dA n1 + dB2 v7,
 *
 * with dnrm the total dL/dnormal (including AA's dependence on the normal), dA = dL/dAA and dB2 = 2 dL/dBB, following the
 * backward's conventions: dL/dG = opacity * dL/dalpha also where alpha is clamped to 0.99 and where power is clamped to 0,
 * channel 7 (alpha) receives no gradient, and the distortion channel keeps only its depth path (the weights T alpha and the
 * pixel's final A and D are constants).
 *
 * float_geometry: 1 evaluates n = M r, AA and BB in float with the forward's operation sequence (the values the GPU kernel
 * differentiates at), 0 in double (the exact function a complex-step derivative sees).
 *
 * Error scales, per pixel and component ([2,H,W] each; NULL to skip), in the model of tests/_grad_bounds.py:
 *   mag       the sum over the pixel's pairs of the term's magnitude, every sum and difference replaced by the sum of the
 *             absolute values of its operands, down to the pair's inputs;
 *   marginal  the same sum over the pairs whose value depends on a blend decision that a last-ulp difference in expf can flip:
 *             a pair whose alpha lies within 8 ulp of 1/255 or whose t lies within 8 ulp of the near plane, every pair in
 *             front of it, and such a pair that this walk rejects, evaluated as if it blended. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define NEAR_PLANE 0.2
#define ALPHA_MAX 0.99f
#define MAX_LIST 65536

typedef struct { float n0, n1, n2, AA, BB; } pairf_t;

static pairf_t pair_geom_f(const float* v, float rx, float ry) { /* forward.cu:504-512, as oracle/gof_oracle.c */
  pairf_t p;
  p.n0 = fmaf(v[0], rx, v[1] * ry) + v[2];
  p.n1 = fmaf(v[1], rx, v[3] * ry) + v[4];
  p.n2 = fmaf(v[4], ry, v[2] * rx) + v[5];
  p.AA = fmaf(p.n0, rx, p.n1 * ry) + p.n2;
  const float bh = fmaf(v[6], rx, v[7] * ry) + v[8];
  p.BB = bh + bh;
  return p;
}

static int near_ulp(float x, float ref, int n) { return fabsf(x - ref) <= n * (nextafterf(ref, INFINITY) - ref); }

/* the forward's float blend test of one pair */
static void test_f(const float* v, float opac, float rx, float ry, float* t_out, float* alpha_out) {
  const pairf_t p = pair_geom_f(v, rx, ry);
  const double AA = p.AA, BB = p.BB;
  *t_out = (float)(-BB / (2 * AA));
  float power = (float)(-0.5 * fma(-BB / AA, BB / 4., (double)v[9]));
  if (power > 0.0f) power = 0.0f;
  *alpha_out = fminf(ALPHA_MAX, opac * expf(power));
}

typedef struct {
  double n[3], AA, BB, t, G, alpha;
} pair_t;

static pair_t pair_eval(const float* v, float opac, float rxf, float ryf, int float_geometry) {
  pair_t q;
  if (float_geometry) {
    const pairf_t p = pair_geom_f(v, rxf, ryf);
    q.n[0] = p.n0; q.n[1] = p.n1; q.n[2] = p.n2; q.AA = p.AA; q.BB = p.BB;
  } else {
    const double rx = rxf, ry = ryf;
    q.n[0] = v[0] * rx + v[1] * ry + v[2];
    q.n[1] = v[1] * rx + v[3] * ry + v[4];
    q.n[2] = v[2] * rx + v[4] * ry + v[5];
    q.AA = q.n[0] * rx + q.n[1] * ry + q.n[2];
    q.BB = 2.0 * (v[6] * rx + v[7] * ry + v[8]);
  }
  q.t = -q.BB / (2 * q.AA);
  double power = -0.5 * ((-q.BB / q.AA) * (q.BB / 4.) + (double)v[9]);
  if (power > 0.0) power = 0.0;
  q.G = exp(power);
  q.alpha = fmin((double)ALPHA_MAX, (double)opac * q.G);
  return q;
}

/* the walk's state behind the current pair (back to front) */
typedef struct {
  double last_alpha, last_c[3], acc_c[3], last_n[3], acc_n[3];
  double acc_c_abs[3], acc_n_abs[3];
} walk_t;

typedef struct {
  const float *dpix, *dn, *bg;
  double ddepth, dreg, T_final, final_A, final_D;
  double rx, ry;
} pixel_t;

/* One pair's ray terms (out[0..1]) and their magnitudes (mag[0..1]); T is the transmittance in front of the pair.  Advances
 * the walk's state w. */
static void pair_term(const pixel_t* px, walk_t* w, const float* v, float opac, const float* col, const pair_t* q, double T,
                      int median, double out[2], double mag[2]) {
  const double alpha = q->alpha, wT = alpha * T;
  const double len = sqrt(q->n[0] * q->n[0] + q->n[1] * q->n[1] + q->n[2] * q->n[2] + 1e-7);
  double nn[3], dL_dalpha = 0, mA = 0, mbg = 0;
  for (int k = 0; k < 3; ++k) nn[k] = -q->n[k] / len;
  for (int ch = 0; ch < 3; ++ch) {
    w->acc_c_abs[ch] = w->last_alpha * fabs(w->last_c[ch]) + (1 - w->last_alpha) * w->acc_c_abs[ch];
    w->acc_c[ch] = w->last_alpha * w->last_c[ch] + (1 - w->last_alpha) * w->acc_c[ch];
    w->last_c[ch] = col[ch];
    dL_dalpha += (col[ch] - w->acc_c[ch]) * px->dpix[ch];
    mA += (fabs((double)col[ch]) + w->acc_c_abs[ch]) * fabs((double)px->dpix[ch]);
    mbg += fabs((double)px->bg[ch]) * fabs((double)px->dpix[ch]);
  }
  for (int ch = 0; ch < 3; ++ch) {
    w->acc_n_abs[ch] = w->last_alpha * fabs(w->last_n[ch]) + (1 - w->last_alpha) * w->acc_n_abs[ch];
    w->acc_n[ch] = w->last_alpha * w->last_n[ch] + (1 - w->last_alpha) * w->acc_n[ch];
    w->last_n[ch] = nn[ch];
    dL_dalpha += (nn[ch] - w->acc_n[ch]) * px->dn[ch];
    mA += (fabs(nn[ch]) + w->acc_n_abs[ch]) * fabs((double)px->dn[ch]);
  }
  w->last_alpha = alpha;
  double bg_dot = 0;
  for (int ch = 0; ch < 3; ++ch) bg_dot += (double)px->bg[ch] * px->dpix[ch];
  dL_dalpha = dL_dalpha * T - px->T_final / (1 - alpha) * bg_dot;
  mA = mA * T + px->T_final / (1 - alpha) * mbg;
  /* depth: the mapped depth m = (100 t - 20) / (99.8 t) of the distortion channel, weights held fixed; the median depth */
  const double t = q->t, m = (100 * t - 20) / (99.8 * t), dm_dt = 20 / (99.8 * t * t);
  double dL_dt = 2 * wT * (m * px->final_A - px->final_D) * px->dreg * dm_dt;
  double mDt = 2 * wT * (fabs(m) * fabs(px->final_A) + fabs(px->final_D)) * fabs(px->dreg) * dm_dt;
  if (median) { dL_dt += px->ddepth; mDt += fabs(px->ddepth); }
  const double dL_dG = opac * dL_dalpha, mG = opac * mA;
  const double dL_dmin = -0.5 * dL_dG * q->G, mMin = 0.5 * mG * q->G;
  const double qd = -q->BB / q->AA, aq = fabs(qd), aA = fabs(q->AA);
  const double dA = dL_dmin * qd * qd / 4 - dL_dt * qd / (2 * q->AA);
  const double dB2 = dL_dmin * qd - dL_dt / q->AA;
  const double mdA = mMin * aq * aq / 4 + mDt * aq / (2 * aA), mdB2 = mMin * aq + mDt / aA;
  /* normal: nn = -n / len */
  double dnn[3], mdnn[3], dlen = 0, mlen = 0;
  for (int k = 0; k < 3; ++k) {
    dnn[k] = wT * px->dn[k];
    mdnn[k] = wT * fabs((double)px->dn[k]);
    dlen += dnn[k] * q->n[k];
    mlen += mdnn[k] * fabs(q->n[k]);
  }
  dlen /= len * len;
  mlen /= len * len;
  const double r[3] = {px->rx, px->ry, 1.0};
  double dnrm[3], mN[3];
  for (int k = 0; k < 3; ++k) {
    dnrm[k] = (dlen * q->n[k] - dnn[k]) / len + dA * r[k];
    mN[k] = (mdnn[k] + mlen * fabs(q->n[k])) / len + mdA * fabs(r[k]);
  }
  /* |n_k| as the sum of its operands' magnitudes */
  const double arx = fabs(px->rx), ary = fabs(px->ry);
  const double an0 = fabs((double)v[0]) * arx + fabs((double)v[1]) * ary + fabs((double)v[2]);
  const double an1 = fabs((double)v[1]) * arx + fabs((double)v[3]) * ary + fabs((double)v[4]);
  out[0] = dnrm[0] * v[0] + dnrm[1] * v[1] + dnrm[2] * v[2] + dA * q->n[0] + dB2 * v[6];
  out[1] = dnrm[0] * v[1] + dnrm[1] * v[3] + dnrm[2] * v[4] + dA * q->n[1] + dB2 * v[7];
  mag[0] = mN[0] * fabs((double)v[0]) + mN[1] * fabs((double)v[1]) + mN[2] * fabs((double)v[2]) + mdA * an0 + mdB2 * fabs((double)v[6]);
  mag[1] = mN[0] * fabs((double)v[1]) + mN[1] * fabs((double)v[3]) + mN[2] * fabs((double)v[4]) + mdA * an1 + mdB2 * fabs((double)v[7]);
}

void focal_oracle_rays(int W, int H, float tan_fovx, float tan_fovy, const uint32_t* ranges, const uint32_t* point_list,
                       const float* bg, const float* conic_opacity, const float* colors, const float* view2gaussian,
                       const float* final_Ts, const uint32_t* n_contrib, const float* dL_dpixels, int float_geometry,
                       double* drays, double* mag, double* marginal) {
  const float focal_y = H / (2.0f * tan_fovy), focal_x = W / (2.0f * tan_fovx);
  const int gx = (W + 15) / 16;
  const size_t HW = (size_t)H * W;
#pragma omp parallel for schedule(dynamic, 4)
  for (int py = 0; py < H; ++py) {
    uint32_t* list = (uint32_t*)malloc(MAX_LIST * sizeof(uint32_t));
    unsigned char* ghost = (unsigned char*)malloc(MAX_LIST);
    double* Tin = (double*)malloc(MAX_LIST * sizeof(double));
    for (int pxi = 0; pxi < W; ++pxi) {
      const size_t pid = (size_t)W * py + pxi;
      const float pixfx = (float)pxi + 0.5f, pixfy = (float)py + 0.5f;
      const float rx = (float)((pixfx - W / 2.) / focal_x), ry = (float)((pixfy - H / 2.) / focal_y);
      const uint32_t* range = ranges + 2 * ((py / 16) * gx + (pxi / 16));
      const int last = (int)n_contrib[pid];
      const int median = (int)n_contrib[pid + HW] - 1;   /* -2 (none) when n_contrib[1] is 0xffffffff */
      /* front to back: the blended pairs, the ghosts, the transmittance in front of each; the deepest marginal decision */
      int n = 0, marginal_upto = -1;
      double T = 1.0;
      for (int c = 0; c < last && range[0] + (uint32_t)c < range[1] && n < MAX_LIST; ++c) {
        const uint32_t gid = point_list[range[0] + c];
        const float* v = view2gaussian + 10 * (size_t)gid;
        const float opac = conic_opacity[4 * (size_t)gid + 3];
        float tf, af;
        test_f(v, opac, rx, ry, &tf, &af);
        const int marg = near_ulp(af, 1.0f / 255.0f, 8) || near_ulp(tf, (float)NEAR_PLANE, 8);
        if (marg) marginal_upto = c;
        const int blends = tf > NEAR_PLANE && af >= 1.0f / 255.0f;
        if (!blends && !(marg && mag)) continue;
        list[n] = (uint32_t)c;
        ghost[n] = (unsigned char)!blends;
        Tin[n] = T;
        if (blends) T *= 1 - pair_eval(v, opac, rx, ry, float_geometry).alpha;
        ++n;
      }
      pixel_t px;
      float dpix[3], dn[3];
      for (int ch = 0; ch < 3; ++ch) { dpix[ch] = dL_dpixels[ch * HW + pid]; dn[ch] = dL_dpixels[(3 + ch) * HW + pid]; }
      px.dpix = dpix; px.dn = dn; px.bg = bg;
      px.ddepth = dL_dpixels[6 * HW + pid];
      px.dreg = dL_dpixels[8 * HW + pid];
      px.T_final = T;
      px.final_A = 1.0 - (double)final_Ts[pid];
      px.final_D = final_Ts[pid + HW];
      px.rx = rx; px.ry = ry;
      walk_t w;
      memset(&w, 0, sizeof w);
      double acc[2] = {0, 0}, amag[2] = {0, 0}, amarg[2] = {0, 0};
      for (int i = n; i-- > 0;) {
        const int c = (int)list[i];
        const uint32_t gid = point_list[range[0] + c];
        const float* v = view2gaussian + 10 * (size_t)gid;
        const float opac = conic_opacity[4 * (size_t)gid + 3];
        pair_t q = pair_eval(v, opac, rx, ry, float_geometry);
        double o[2], m[2];
        if (ghost[i]) {   /* as if it blended; the walk's state stays as without it */
          walk_t w2 = w;
          if (q.alpha < 1.0 / 255.0) q.alpha = 1.0 / 255.0;
          pair_term(&px, &w2, v, opac, colors + 3 * (size_t)gid, &q, Tin[i], c == median, o, m);
          amarg[0] += m[0]; amarg[1] += m[1];
          continue;
        }
        pair_term(&px, &w, v, opac, colors + 3 * (size_t)gid, &q, Tin[i], c == median, o, m);
        acc[0] += o[0]; acc[1] += o[1];
        amag[0] += m[0]; amag[1] += m[1];
        if (c <= marginal_upto) { amarg[0] += m[0]; amarg[1] += m[1]; }
      }
      drays[pid] = acc[0]; drays[HW + pid] = acc[1];
      if (mag) { mag[pid] = amag[0]; mag[HW + pid] = amag[1]; }
      if (marginal) { marginal[pid] = amarg[0]; marginal[HW + pid] = amarg[1]; }
    }
    free(list); free(ghost); free(Tin);
  }
}
