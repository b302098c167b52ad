/*
 * gof_oracle.c -- TEST INFRASTRUCTURE ONLY (never linked, imported or executed by the product path).
 *
 * CPU restatement, in plain C, of the reference Gaussian-opacity-field rasterizer
 *   <original project>/submodules/diff-gaussian-rasterization/cuda_rasterizer/{forward.cu,backward.cu,
 *   rasterizer_impl.cu,auxiliary.h}
 * function by function; every block cites the reference lines it follows.  Only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may call it.
 *
 * Floating point: the reference is ill-conditioned by design (power = -1/2 (C - B^2/4A) with C ~ 1e5..1e6),
 * so its results are defined by the exact IEEE operation sequence nvcc produced for it (default -fmad=true).
 * Where that matters (quaternion->R, view2gaussian, covariance chain, A/B/normal of the ray-Gaussian
 * intersection) this file states the fused operations of the reference's sm_100a SASS explicitly with
 * fmaf(); everything else is written as in the CUDA source.  Build with -ffp-contract=off so the compiler
 * adds no fusion of its own (oracle/Makefile).
 *
 * Parity pinning: the reference ships no golden vectors (SURVEY.md section 4), so this oracle is pinned
 * against outputs of the reference extension itself, generated on a B200 by tests/golden/make_golden.py
 * and committed under tests/golden/ (tests/test_oracle_golden.py).
 *
 * Backward accumulations are carried in double and rounded once: the reference accumulates float
 * atomics in a non-deterministic order, so its own run-to-run noise is the comparison floor.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define BLOCK_X 16
#define BLOCK_Y 16
#define BLOCK_SIZE 256
#define NEAR_PLANE 0.2
#define FAR_PLANE 100.0

static const float SH_C0 = 0.28209479177387814f;
static const float SH_C1 = 0.4886025119029199f;
static const float SH_C2[] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                              -1.0925484305920792f, 0.5462742152960396f};
static const float SH_C3[] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f, 0.3731763325901154f,
                              -0.4570457994644658f, 1.445305721320277f, -0.5900435899266435f};

typedef struct {
  int P, D, M, W, H;
  float tan_fovx, tan_fovy, kernel_size, scale_modifier;
  const float* background;
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
} oracle_scene_t;

/* per-Gaussian state in the reference's GeometryState layout (rasterizer_impl.cu:188-204) */
typedef struct {
  int* radii;               /* [P] */
  float* means2D;           /* [P,2] */
  float* depths;            /* [P] */
  float* cov3D;             /* [P,6] */
  float* view2gaussian;     /* [P,10] */
  float* rgb;               /* [P,3] */
  float* conic_opacity;     /* [P,4] */
  uint32_t* tiles_touched;  /* [P] */
  unsigned char* clamped;   /* [P,3] */
} oracle_geom_t;

int oracle_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

static int f2i(float v) { /* cvt.rzi.s32.f32: NaN -> 0, saturating */
  if (!(v == v)) return 0;
  if (v >= 2147483648.0f) return 2147483647;
  if (v <= -2147483648.0f) return (-2147483647 - 1);
  return (int)v;
}

static float dot3f(float a0, float b0, float a1, float b1, float a2, float b2) {
  /* the reference's SASS evaluates every 3-term glm product sum as fma(a2,b2, fma(a0,b0, a1*b1)) */
  return fmaf(a2, b2, fmaf(a0, b0, a1 * b1));
}

/* auxiliary.h:86-94,106-115: m[a]*x + m[b]*y + m[c]*z + m[d] */
static float affine(float x, float y, float z, float ma, float mb, float mc, float md) {
  return fmaf(z, mc, fmaf(x, ma, y * mb)) + md;
}

/* forward.cu:138-149: rotation matrix from the (unnormalised) quaternion; R[c][r] column-major like glm */
static void quat_to_R(const float* q, float R[3][3]) {
  const float r = q[0], x = q[1], y = q[2], z = q[3];
  const float yy = y * y, zz = z * z, xz = x * z, rz = r * z, rx = r * x;
  float s;
  s = yy + zz;            R[0][0] = 1.f - (s + s);
  s = fmaf(x, y, -rz);    R[0][1] = s + s;
  s = fmaf(r, y, xz);     R[0][2] = s + s;
  s = fmaf(x, y, rz);     R[1][0] = s + s;
  s = fmaf(x, x, zz);     R[1][1] = 1.f - (s + s);
  s = fmaf(y, z, -rx);    R[1][2] = s + s;
  s = fmaf(-r, y, xz);    R[2][0] = s + s;
  s = fmaf(y, z, rx);     R[2][1] = s + s;
  s = fmaf(x, x, yy);     R[2][2] = 1.f - (s + s);
}

/* forward.cu:129-163 computeCov3D */
static void compute_cov3D(const float* scale, float mod, float R[3][3], float* cov3D) {
  float M[3][3];
  for (int c = 0; c < 3; ++c)
    for (int r = 0; r < 3; ++r) M[c][r] = (mod * scale[r]) * R[c][r]; /* S * R, S diagonal */
  /* Sigma = transpose(M) * M */
  cov3D[0] = dot3f(M[0][0], M[0][0], M[0][1], M[0][1], M[0][2], M[0][2]);
  cov3D[1] = dot3f(M[1][0], M[0][0], M[1][1], M[0][1], M[1][2], M[0][2]);
  cov3D[2] = dot3f(M[2][0], M[0][0], M[2][1], M[0][1], M[2][2], M[0][2]);
  cov3D[3] = dot3f(M[1][0], M[1][0], M[1][1], M[1][1], M[1][2], M[1][2]);
  cov3D[4] = dot3f(M[2][0], M[1][0], M[2][1], M[1][1], M[2][2], M[1][2]);
  cov3D[5] = dot3f(M[2][0], M[2][0], M[2][1], M[2][1], M[2][2], M[2][2]);
}

/* forward.cu:74-124 computeCov2D; out = (cov.x, cov.y, cov.z, coef), *det = cov.x*cov.z - cov.y^2 */
static void compute_cov2D(const float* mean, float focal_x, float focal_y, float tan_fovx, float tan_fovy,
                          float kernel_size, const float* cov3D, const float* vm, float out[4], float* det) {
  float tx = affine(mean[0], mean[1], mean[2], vm[0], vm[4], vm[8], vm[12]);
  float ty = affine(mean[0], mean[1], mean[2], vm[1], vm[5], vm[9], vm[13]);
  const float tz = affine(mean[0], mean[1], mean[2], vm[2], vm[6], vm[10], vm[14]);
  const float limx = 1.3f * tan_fovx, limy = 1.3f * tan_fovy;
  const float txtz = tx / tz, tytz = ty / tz;
  tx = fminf(limx, fmaxf(-limx, txtz)) * tz;
  ty = fminf(limy, fmaxf(-limy, tytz)) * tz;
  const float J00 = focal_x / tz, J11 = focal_y / tz;
  const float jx = -(focal_x * tx) / (tz * tz), jy = -(focal_y * ty) / (tz * tz);
  /* T = W * J (columns of T; third column is zero) */
  const float T00 = fmaf(vm[2], jx, vm[0] * J00), T01 = fmaf(vm[6], jx, vm[4] * J00), T02 = fmaf(jx, vm[10], vm[8] * J00);
  const float T10 = fmaf(vm[2], jy, J11 * vm[1]), T11 = fmaf(vm[6], jy, J11 * vm[5]), T12 = fmaf(jy, vm[10], J11 * vm[9]);
  const float c0 = cov3D[0], c1 = cov3D[1], c2 = cov3D[2], c3 = cov3D[3], c4 = cov3D[4], c5 = cov3D[5];
  /* cov = transpose(T) * transpose(Vrk) * T */
  const float a00 = dot3f(T00, c0, T01, c1, T02, c2), a01 = dot3f(T00, c1, T01, c3, T02, c4), a02 = dot3f(T00, c2, T01, c4, T02, c5);
  const float b00 = dot3f(T10, c0, T11, c1, T12, c2), b01 = dot3f(T10, c1, T11, c3, T12, c4), b02 = dot3f(T10, c2, T11, c4, T12, c5);
  const float cov00 = dot3f(T00, a00, T01, a01, T02, a02);
  const float cov11 = dot3f(T10, b00, T11, b01, T12, b02);
  const float cov01 = dot3f(T00, b00, T01, b01, T02, b02);
  const float b2 = cov01 * cov01;
  /* forward.cu:112-118 */
  const float det_0 = (float)fmax(1e-6, (double)fmaf(cov00, cov11, -b2));
  const float ca = cov00 + kernel_size, cc = cov11 + kernel_size;
  const float det1_raw = fmaf(ca, cc, -b2);
  const float det_1 = (float)fmax(1e-6, (double)det1_raw);
  float coef = (float)sqrt((double)det_0 / ((double)det_1 + 1e-6) + 1e-6);
  if ((double)det_0 <= 1e-6 || (double)det_1 <= 1e-6) coef = 0.0f;
  out[0] = ca; out[1] = cov01; out[2] = cc; out[3] = coef;
  *det = det1_raw;
}

/* forward.cu:168-279 computeView2Gaussian */
static void compute_view2gaussian(const float* scale, const float* mean, float R[3][3], const float* vm, float* v2g) {
  /* G2V = W2V * G2W (rotation part): G2V[j][i] = sum_k vm[4k+i] * R[k][j] */
  float g[3][3];
  for (int j = 0; j < 3; ++j)
    for (int i = 0; i < 3; ++i) g[j][i] = fmaf(R[2][j], vm[8 + i], fmaf(R[0][j], vm[i], R[1][j] * vm[4 + i]));
  const float tx = fmaf(mean[2], vm[8], fmaf(mean[0], vm[0], mean[1] * vm[4])) + vm[12];
  const float ty = fmaf(mean[2], vm[9], fmaf(mean[0], vm[1], mean[1] * vm[5])) + vm[13];
  const float tz = fmaf(mean[2], vm[10], fmaf(mean[0], vm[2], mean[1] * vm[6])) + vm[14];
  /* R_transpose[c][r] = G2V[r][c]; t2 = -R_transpose * t */
  float t2[3];
  for (int i = 0; i < 3; ++i) t2[i] = fmaf(g[i][2], -tz, fmaf(-g[i][1], ty, -(g[i][0] * tx)));
  double si[3];
  for (int k = 0; k < 3; ++k) si[k] = 1.0 / fma((double)scale[k], (double)scale[k], 1e-7);
  /* S_inv_square_R[c][r] = si[r] * R_transpose[c][r] = si[r] * g[r][c] */
  float q[3][3];
  for (int c = 0; c < 3; ++c)
    for (int r = 0; r < 3; ++r) q[c][r] = (float)(si[r] * (double)g[r][c]);
  /* Sigma = transpose(R_transpose) * S_inv_square_R : Sigma[c][r] = sum_k g[k][r] * q[c][k] */
  v2g[0] = dot3f(g[0][0], q[0][0], g[1][0], q[0][1], g[2][0], q[0][2]);
  v2g[1] = dot3f(g[0][1], q[0][0], g[1][1], q[0][1], g[2][1], q[0][2]);
  v2g[2] = dot3f(g[0][2], q[0][0], g[1][2], q[0][1], g[2][2], q[0][2]);
  v2g[3] = dot3f(g[0][1], q[1][0], g[1][1], q[1][1], g[2][1], q[1][2]);
  v2g[4] = dot3f(g[0][2], q[1][0], g[1][2], q[1][1], g[2][2], q[1][2]);
  v2g[5] = dot3f(g[0][2], q[2][0], g[1][2], q[2][1], g[2][2], q[2][2]);
  /* B = t2 * S_inv_square_R */
  for (int c = 0; c < 3; ++c) v2g[6 + c] = dot3f(t2[0], q[c][0], t2[1], q[c][1], t2[2], q[c][2]);
  const double cx = (double)(t2[0] * t2[0]), cy = (double)(t2[1] * t2[1]), cz = (double)(t2[2] * t2[2]);
  v2g[9] = (float)fma(si[2], cz, fma(si[0], cx, si[1] * cy));
}

/* forward.cu:20-71 computeColorFromSH */
static void color_from_sh(int deg, int M, const float* mean, const float* campos, const float* sh, float* rgb,
                          unsigned char* clamped) {
  (void)M;
  float dx = mean[0] - campos[0], dy = mean[1] - campos[1], dz = mean[2] - campos[2];
  const float len = sqrtf(dx * dx + dy * dy + dz * dz);
  const float x = dx / len, y = dy / len, z = dz / len;
  for (int c = 0; c < 3; ++c) {
#define S(k) sh[3 * (k) + c]
    float result = SH_C0 * S(0);
    if (deg > 0) {
      result = result - SH_C1 * y * S(1) + SH_C1 * z * S(2) - SH_C1 * x * S(3);
      if (deg > 1) {
        const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
        result = result + SH_C2[0] * xy * S(4) + SH_C2[1] * yz * S(5) + SH_C2[2] * (2.0f * zz - xx - yy) * S(6) +
                 SH_C2[3] * xz * S(7) + SH_C2[4] * (xx - yy) * S(8);
        if (deg > 2) {
          result = result + SH_C3[0] * y * (3.0f * xx - yy) * S(9) + SH_C3[1] * xy * z * S(10) +
                   SH_C3[2] * y * (4.0f * zz - xx - yy) * S(11) + SH_C3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * S(12) +
                   SH_C3[4] * x * (4.0f * zz - xx - yy) * S(13) + SH_C3[5] * z * (xx - yy) * S(14) +
                   SH_C3[6] * x * (xx - 3.0f * yy) * S(15);
        }
      }
    }
#undef S
    result += 0.5f;
    clamped[c] = (result < 0);
    rgb[c] = (result < 0.0f) ? 0.0f : result;
  }
}

static float ndc2Pix(float v, int S) { return (float)(fma((double)v + 1.0, (double)S, -1.0) * 0.5); } /* auxiliary.h:59-62 */

static void get_rect(float px, float py, int max_radius, uint32_t rmin[2], uint32_t rmax[2], int gx, int gy) {
  /* auxiliary.h:64-74 */
  const float r = (float)max_radius;
  int x0 = f2i((px - r) / BLOCK_X), y0 = f2i((py - r) / BLOCK_Y);
  int x1 = f2i((px + r + BLOCK_X - 1) / BLOCK_X), y1 = f2i((py + r + BLOCK_Y - 1) / BLOCK_Y);
  if (x0 < 0) x0 = 0; if (y0 < 0) y0 = 0; if (x1 < 0) x1 = 0; if (y1 < 0) y1 = 0;
  rmin[0] = (uint32_t)x0 < (uint32_t)gx ? (uint32_t)x0 : (uint32_t)gx;
  rmin[1] = (uint32_t)y0 < (uint32_t)gy ? (uint32_t)y0 : (uint32_t)gy;
  rmax[0] = (uint32_t)x1 < (uint32_t)gx ? (uint32_t)x1 : (uint32_t)gx;
  rmax[1] = (uint32_t)y1 < (uint32_t)gy ? (uint32_t)y1 : (uint32_t)gy;
}

/* forward.cu:283-404 preprocessCUDA.  Fields of culled Gaussians are left untouched except radii and
 * tiles_touched (= 0), exactly like the reference. */
void oracle_preprocess(const oracle_scene_t* s, oracle_geom_t* g) {
  const float focal_y = s->H / (2.0f * s->tan_fovy), focal_x = s->W / (2.0f * s->tan_fovx); /* rasterizer_impl.cu:274-275 */
  const int gx = (s->W + BLOCK_X - 1) / BLOCK_X, gy = (s->H + BLOCK_Y - 1) / BLOCK_Y;
  const float* vm = s->viewmatrix;
  const float* pm = s->projmatrix;
#pragma omp parallel for schedule(static)
  for (int idx = 0; idx < s->P; ++idx) {
    g->radii[idx] = 0;
    g->tiles_touched[idx] = 0;
    const float* p = s->means3D + 3 * idx;
    const float pvz = affine(p[0], p[1], p[2], vm[2], vm[6], vm[10], vm[14]);
    if (pvz <= 0.2f) continue; /* in_frustum, auxiliary.h:192 */
    const float hx = affine(p[0], p[1], p[2], pm[0], pm[4], pm[8], pm[12]);
    const float hy = affine(p[0], p[1], p[2], pm[1], pm[5], pm[9], pm[13]);
    const float hw = affine(p[0], p[1], p[2], pm[3], pm[7], pm[11], pm[15]);
    const float p_w = 1.0f / (hw + 0.0000001f);
    const float projx = hx * p_w, projy = hy * p_w;
    float R[3][3];
    float cov3D_local[6];
    const float* cov3D;
    if (s->rotations) quat_to_R(s->rotations + 4 * idx, R);
    if (s->cov3D_precomp) {
      cov3D = s->cov3D_precomp + 6 * idx;
    } else {
      compute_cov3D(s->scales + 3 * idx, s->scale_modifier, R, cov3D_local);
      memcpy(g->cov3D + 6 * idx, cov3D_local, sizeof(cov3D_local));
      cov3D = cov3D_local;
    }
    float cov[4], det;
    compute_cov2D(p, focal_x, focal_y, s->tan_fovx, s->tan_fovy, s->kernel_size, cov3D, vm, cov, &det);
    if (det == 0.0f) continue;
    const float det_inv = 1.f / det;
    const float conic[3] = {cov[2] * det_inv, -cov[1] * det_inv, cov[0] * det_inv};
    const float mid = 0.5f * (cov[0] + cov[2]);
    const float disc = fmaxf(0.1f, fmaf(mid, mid, -det));
    const float lambda1 = mid + sqrtf(disc), lambda2 = mid - sqrtf(disc);
    const float my_radius = ceilf(3.f * sqrtf(fmaxf(lambda1, lambda2)));
    const float pix[2] = {ndc2Pix(projx, s->W), ndc2Pix(projy, s->H)};
    uint32_t rmin[2], rmax[2];
    get_rect(pix[0], pix[1], f2i(my_radius), rmin, rmax, gx, gy);
    if ((rmax[0] - rmin[0]) * (rmax[1] - rmin[1]) == 0) continue;
    if (s->colors_precomp == NULL) color_from_sh(s->D, s->M, p, s->cam_pos, s->shs + (size_t)idx * s->M * 3, g->rgb + 3 * idx, g->clamped + 3 * idx);
    g->depths[idx] = pvz;
    g->radii[idx] = f2i(my_radius);
    g->means2D[2 * idx] = pix[0];
    g->means2D[2 * idx + 1] = pix[1];
    g->conic_opacity[4 * idx + 0] = conic[0];
    g->conic_opacity[4 * idx + 1] = conic[1];
    g->conic_opacity[4 * idx + 2] = conic[2];
    g->conic_opacity[4 * idx + 3] = s->opacities[idx] * cov[3];
    g->tiles_touched[idx] = (rmax[1] - rmin[1]) * (rmax[0] - rmin[0]);
    if (s->v2g_precomp == NULL) compute_view2gaussian(s->scales + 3 * idx, p, R, vm, g->view2gaussian + 10 * idx);
  }
}

/* rasterizer_impl.cu:330-372: scan, duplicateWithKeys, stable sort by (tile, depth bits), identifyTileRanges.
 * point_list must hold sum(tiles_touched) entries; returns that count.  ranges: [tiles][2]. */
typedef struct { uint64_t key; uint32_t val; } kv_t;

static void radix_sort_kv(kv_t* a, kv_t* tmp, size_t n, int bits) {
  for (int shift = 0; shift < bits; shift += 8) {
    size_t cnt[257] = {0};
    for (size_t i = 0; i < n; ++i) cnt[((a[i].key >> shift) & 0xff) + 1]++;
    for (int d = 0; d < 256; ++d) cnt[d + 1] += cnt[d];
    for (size_t i = 0; i < n; ++i) tmp[cnt[(a[i].key >> shift) & 0xff]++] = a[i];
    kv_t* t = a; a = tmp; tmp = t;
  }
  if ((bits + 7) / 8 % 2 == 1) memcpy(tmp, a, n * sizeof(kv_t)); /* result back in the caller's array */
}

long long oracle_bin(int P, int W, int H, const int* radii, const float* means2D, const float* depths,
                     const uint32_t* tiles_touched, uint32_t* point_list, uint32_t* ranges, uint64_t* keys_out) {
  const int gx = (W + BLOCK_X - 1) / BLOCK_X, gy = (H + BLOCK_Y - 1) / BLOCK_Y;
  size_t R = 0;
  for (int i = 0; i < P; ++i) R += tiles_touched[i];
  memset(ranges, 0, (size_t)gx * gy * 2 * sizeof(uint32_t));
  if (R == 0) return 0;
  kv_t* kv = (kv_t*)malloc(R * sizeof(kv_t));
  kv_t* tmp = (kv_t*)malloc(R * sizeof(kv_t));
  size_t off = 0;
  for (int idx = 0; idx < P; ++idx) { /* duplicateWithKeys, :70-111 */
    if (radii[idx] > 0) {
      uint32_t rmin[2], rmax[2];
      get_rect(means2D[2 * idx], means2D[2 * idx + 1], radii[idx], rmin, rmax, gx, gy);
      uint32_t dbits;
      memcpy(&dbits, depths + idx, 4);
      for (uint32_t y = rmin[1]; y < rmax[1]; ++y)
        for (uint32_t x = rmin[0]; x < rmax[0]; ++x) {
          kv[off].key = ((uint64_t)(y * gx + x) << 32) | dbits;
          kv[off].val = (uint32_t)idx;
          off++;
        }
    }
  }
  /* getHigherMsb, :35-50 */
  uint32_t n = (uint32_t)(gx * gy), msb = 16, step = 16;
  while (step > 1) { step /= 2; if (n >> msb) msb += step; else msb -= step; }
  if (n >> msb) msb++;
  const int bits = 32 + (int)msb;
  /* stable LSD radix sort over the same key bits as cub::DeviceRadixSort::SortPairs(..., 0, 32 + bit) */
  {
    kv_t* a = kv; kv_t* b = tmp;
    for (int shift = 0; shift < bits; shift += 8) {
      size_t cnt[257];
      memset(cnt, 0, sizeof(cnt));
      const int w = (bits - shift) < 8 ? (bits - shift) : 8;
      const uint64_t mask = ((uint64_t)1 << w) - 1;
      for (size_t i = 0; i < off; ++i) cnt[((a[i].key >> shift) & mask) + 1]++;
      for (int d = 0; d < 256; ++d) cnt[d + 1] += cnt[d];
      for (size_t i = 0; i < off; ++i) b[cnt[(a[i].key >> shift) & mask]++] = a[i];
      kv_t* t = a; a = b; b = t;
    }
    if (a != kv) memcpy(kv, a, off * sizeof(kv_t));
  }
  for (size_t i = 0; i < off; ++i) {
    point_list[i] = kv[i].val;
    if (keys_out) keys_out[i] = kv[i].key;
  }
  for (size_t idx = 0; idx < off; ++idx) { /* identifyTileRanges, :149-171 */
    const uint32_t cur = (uint32_t)(kv[idx].key >> 32);
    if (idx == 0) ranges[2 * cur] = 0;
    else {
      const uint32_t prev = (uint32_t)(kv[idx - 1].key >> 32);
      if (cur != prev) { ranges[2 * prev + 1] = (uint32_t)idx; ranges[2 * cur] = (uint32_t)idx; }
    }
    if (idx == off - 1) ranges[2 * cur + 1] = (uint32_t)off;
  }
  free(kv); free(tmp);
  (void)radix_sort_kv;
  return (long long)off;
}

/* the five float expressions whose fusion pattern defines the reference's alpha (forward.cu:504-512) */
typedef struct { float n0, n1, n2, AA, BB; } pair_t;
static pair_t pair_geom(const float* v, float rx, float ry) {
  pair_t p;
  p.n0 = fmaf(v[0], rx, v[1] * ry) + v[2];
  p.n1 = fmaf(v[1], rx, v[3] * ry) + v[4];
  p.n2 = fmaf(v[4], ry, v[2] * rx) + v[5];
  p.AA = fmaf(p.n0, rx, p.n1 * ry) + p.n2;
  const float bh = fmaf(v[6], rx, v[7] * ry) + v[8];
  p.BB = bh + bh;
  return p;
}

/* forward.cu:409-612 renderCUDA.  out_color [9,H,W], final_T [4,H,W], n_contrib [2,H,W]. */
void oracle_render_forward(int W, int H, float tan_fovx, float tan_fovy, const uint32_t* ranges,
                           const uint32_t* point_list, const float* features, const float* view2gaussian,
                           const float* conic_opacity, const float* bg, float* out_color, float* final_T,
                           uint32_t* n_contrib) {
  const float focal_y = H / (2.0f * tan_fovy), focal_x = W / (2.0f * tan_fovx);
  const int gx = (W + BLOCK_X - 1) / BLOCK_X;
  const size_t HW = (size_t)H * W;
#pragma omp parallel for schedule(dynamic, 8)
  for (int py = 0; py < H; ++py) {
    for (int px = 0; px < W; ++px) {
      const size_t pix_id = (size_t)W * py + px;
      const float pixfx = (float)px + 0.5f, pixfy = (float)py + 0.5f;
      const float rx = (float)((pixfx - W / 2.) / focal_x), ry = (float)((pixfy - H / 2.) / focal_y);
      const uint32_t* range = ranges + 2 * ((py / BLOCK_Y) * gx + (px / BLOCK_X));
      float T = 1.0f;
      uint32_t contributor = 0, last_contributor = 0, max_contributor = (uint32_t)-1;
      float C[8] = {0};
      float dist1 = 0, dist2 = 0, distortion = 0;
      for (uint32_t k = range[0]; k < range[1]; ++k) {
        contributor++;
        const uint32_t gid = point_list[k];
        const float* v = view2gaussian + 10 * (size_t)gid;
        const float opac = conic_opacity[4 * (size_t)gid + 3];
        const pair_t p = pair_geom(v, rx, ry);
        const double AA = p.AA, BB = p.BB;
        const float CC = v[9];
        const float t = (float)(-BB / (2 * AA));
        if (t <= NEAR_PLANE) continue;
        const double min_value = fma(-BB / AA, BB / 4., (double)CC); /* -(BB/AA)*(BB/4.) + CC, dfma in SASS */
        float power = (float)(-0.5 * min_value);
        if (power > 0.0f) power = 0.0f;
        const float alpha = fminf(0.99f, opac * expf(power));
        if (alpha < 1.0f / 255.0f) continue;
        const float test_T = T * (1 - alpha);
        if (test_T < 0.0001f) break; /* done = true */
        const float max_t = t;
        const float mapped_max_t = (float)((FAR_PLANE * max_t - FAR_PLANE * NEAR_PLANE) / ((FAR_PLANE - NEAR_PLANE) * max_t));
        const float length = (float)sqrt((double)fmaf(p.n2, p.n2, fmaf(p.n0, p.n0, p.n1 * p.n1)) + 1e-7);
        const float nn[3] = {-p.n0 / length, -p.n1 / length, -p.n2 / length};
        const float A = 1 - T;
        /* forward.cu:552-565 in the fused form of the reference's SASS (fma accumulation onto T) */
        const float m2 = mapped_max_t * mapped_max_t;
        const float error = fmaf(-dist1, mapped_max_t + mapped_max_t, fmaf(A, m2, dist2));
        distortion = fmaf(T, error * alpha, distortion);
        dist1 = fmaf(T, alpha * mapped_max_t, dist1);
        dist2 = fmaf(T, m2 * alpha, dist2);
        for (int ch = 0; ch < 3; ++ch) C[ch] = fmaf(T, alpha * features[3 * (size_t)gid + ch], C[ch]);
        for (int ch = 0; ch < 3; ++ch) C[3 + ch] = fmaf(T, alpha * nn[ch], C[3 + ch]);
        if (T > 0.5) { C[6] = t; max_contributor = contributor; }
        C[7] = fmaf(T, alpha, C[7]);
        T = test_T;
        last_contributor = contributor;
      }
      const float dbn = distortion;
      distortion = (float)(distortion / ((double)((1 - T) * (1 - T)) + 1e-7));
      final_T[pix_id] = T; final_T[pix_id + HW] = dist1; final_T[pix_id + 2 * HW] = dist2; final_T[pix_id + 3 * HW] = dbn;
      n_contrib[pix_id] = last_contributor; n_contrib[pix_id + HW] = max_contributor;
      for (int ch = 0; ch < 3; ++ch) out_color[ch * HW + pix_id] = fmaf(T, bg[ch], C[ch]);
      for (int ch = 0; ch < 3; ++ch) out_color[(3 + ch) * HW + pix_id] = C[3 + ch];
      out_color[6 * HW + pix_id] = C[6];
      out_color[7 * HW + pix_id] = C[7];
      out_color[8 * HW + pix_id] = distortion;
    }
  }
}

/* |x - ref| within n float ulp of ref */
static int near_ulp(float x, float ref, int n) { return fabsf(x - ref) <= n * (nextafterf(ref, INFINITY) - ref); }

/* The t and alpha of the forward's blend test (forward.cu:499-535) for the pair (v, opacity, ray). */
static void pair_t_alpha(const float* v, float opac, float rx, float ry, float* t_out, float* alpha_out) {
  const pair_t p = pair_geom(v, rx, ry);
  const double AA = p.AA, BB = p.BB;
  *t_out = (float)(-BB / (2 * AA));
  const double min_value = fma(-BB / AA, BB / 4., (double)v[9]);
  float power = (float)(-0.5 * min_value);
  if (power > 0.0f) power = 0.0f;
  *alpha_out = fminf(0.99f, opac * expf(power));
}

/* backward.cu:634-955 renderCUDA.  Gradients are accumulated in per-thread double buffers, then reduced.
 * dL_dmean2D [P,3], dL_dopacity [P], dL_dcolors [P,3], dL_dview2gaussian [P,10] (float outputs).
 *
 * Optional error scales, [P,17] doubles each (NULL: not computed; the gradients do not depend on it), in the order of the
 * accumulator (dL_dcolors 0-2 | dL_dmean2D 3-5 | dL_dopacity 6 | dL_dview2gaussian 7-16):
 *   mag       for every Gaussian and component, the sum over its pairs of the pair term's magnitude: the term with every sum
 *             and difference replaced by the sum of the absolute values of its operands, down to the pair's inputs (T,
 *             accum_rec, colours, dL_dpix, G, conic, AA, BB, rx, ry, normal).  A rounding of any intermediate moves a
 *             component by a multiple of 2^-24 of this, whatever cancels inside the term or across terms.
 *   marginal  the same sum over the pairs whose value depends on a blend decision that a last-ulp difference in expf can
 *             flip: a pair whose alpha lies within 8 ulp of 1/255 or whose t lies within 8 ulp of the near plane
 *             (alpha < 1/255 and t <= 0.2 reject a pair), and every pair in front of it at that pixel, whose T and
 *             accum_rec the decision changes.  Pairs behind it do not depend on it (the walk runs back to front). */
void oracle_render_backward(int P, int W, int H, float tan_fovx, float tan_fovy, const uint32_t* ranges,
                            const uint32_t* point_list, const float* bg, const float* means2D,
                            const float* conic_opacity, const float* colors, const float* view2gaussian,
                            const float* final_Ts, const uint32_t* n_contrib, const float* dL_dpixels,
                            float* dL_dmean2D, float* dL_dopacity, float* dL_dcolors, float* dL_dview2gaussian,
                            double* mag, double* marginal) {
  const float focal_y = H / (2.0f * tan_fovy), focal_x = W / (2.0f * tan_fovx);
  const int gx = (W + BLOCK_X - 1) / BLOCK_X;
  const size_t HW = (size_t)H * W;
  const int NG = 17;
  const int bounds = mag != NULL && marginal != NULL;
  const int NS = bounds ? 3 * NG : NG;   /* per Gaussian and thread: the sums, then mag, then marginal */
  int nthreads = 1;
#ifdef _OPENMP
  nthreads = omp_get_max_threads();
  if (nthreads > 8 && (size_t)P * NS * 8 * nthreads > ((size_t)4 << 30)) nthreads = 8;
#endif
  double* acc = (double*)calloc((size_t)nthreads * P * NS, sizeof(double));
#pragma omp parallel for schedule(dynamic, 8) num_threads(nthreads)
  for (int py = 0; py < H; ++py) {
    int tid = 0;
#ifdef _OPENMP
    tid = omp_get_thread_num();
#endif
    double* my = acc + (size_t)tid * P * NS;
    for (int px = 0; px < W; ++px) {
      const size_t pix_id = (size_t)W * py + px;
      const float pixfx = (float)px + 0.5f, pixfy = (float)py + 0.5f;
      const float rx = (float)((pixfx - W / 2.) / focal_x), ry = (float)((pixfy - H / 2.) / focal_y);
      const uint32_t* range = ranges + 2 * ((py / BLOCK_Y) * gx + (px / BLOCK_X));
      const float T_final = final_Ts[pix_id];
      float T = T_final;
      const float final_D = final_Ts[pix_id + HW];
      const float final_A = 1 - T_final;
      const float dL_dreg = dL_dpixels[8 * HW + pix_id];
      uint32_t contributor = range[1] - range[0];
      const int last_contributor = (int)n_contrib[pix_id];
      const int max_contributor = (int)n_contrib[pix_id + HW];
      float accum_rec[3] = {0}, dL_dpixel[3], dL_dnormal2D[3];
      for (int i = 0; i < 3; ++i) dL_dpixel[i] = dL_dpixels[i * HW + pix_id];
      for (int i = 0; i < 3; ++i) dL_dnormal2D[i] = dL_dpixels[(3 + i) * HW + pix_id];
      const float dL_dmax_depth = dL_dpixels[6 * HW + pix_id];
      float last_alpha = 0, last_color[3] = {0}, last_normal[3] = {0}, accum_normal_rec[3] = {0};
      const float ddelx_dx = 0.5f * W, ddely_dy = 0.5f * H;
      /* error scales: the magnitudes of accum_rec / accum_normal_rec, and the deepest pair of the walk whose blend decision
       * is marginal (-1: none) */
      double accum_abs[3] = {0, 0, 0}, accum_normal_abs[3] = {0, 0, 0};
      long marginal_upto = -1;
      if (bounds) {
        for (int c = 0; c < last_contributor && range[0] + (uint32_t)c < range[1]; ++c) {
          const uint32_t gid = point_list[range[0] + c];
          float t, alpha;
          pair_t_alpha(view2gaussian + 10 * (size_t)gid, conic_opacity[4 * (size_t)gid + 3], rx, ry, &t, &alpha);
          if (near_ulp(alpha, 1.0f / 255.0f, 8) || near_ulp(t, (float)NEAR_PLANE, 8)) marginal_upto = c;
        }
      }
      for (uint32_t k = range[1]; k-- > range[0];) {
        contributor--;
        if (contributor >= (uint32_t)last_contributor) continue;
        const uint32_t gid = point_list[k];
        const float* v = view2gaussian + 10 * (size_t)gid;
        const float* con_o = conic_opacity + 4 * (size_t)gid;
        const float dx = (float)(means2D[2 * (size_t)gid] - (pixfx - 0.5)), dy = (float)(means2D[2 * (size_t)gid + 1] - (pixfy - 0.5));
        const pair_t p = pair_geom(v, rx, ry);
        const double AA = p.AA, BB = p.BB;
        const float CC = v[9];
        const float t = (float)(-BB / (2 * AA));
        const int near_t = bounds && near_ulp(t, (float)NEAR_PLANE, 8);
        if (t <= NEAR_PLANE && !near_t) continue;
        const double min_value = fma(-BB / AA, BB / 4., (double)CC);
        float power = (float)(-0.5 * min_value);
        if (power > 0.0f) power = 0.0f;
        const float G = expf(power);
        const float alpha0 = fminf(0.99f, con_o[3] * G);
        const int near_a = bounds && near_ulp(alpha0, 1.0f / 255.0f, 8);
        if (alpha0 < 1.0f / 255.0f && !near_a) continue;
        /* a "ghost": a pair this walk rejects by a marginal decision, which a 2-ulp expf may have blended.  Its term, evaluated
         * as if it blended, goes to `marginal` only; the gradients and the walk's state stay as without it */
        const int ghost = t <= NEAR_PLANE || alpha0 < 1.0f / 255.0f;
        const float alpha = ghost ? fmaxf(alpha0, 1.0f / 255.0f) : alpha0;
        float saved_f[14];
        double saved_d[6], ghost_acc[3 * 17];
        if (ghost) {
          memset(ghost_acc, 0, sizeof ghost_acc);
          saved_f[0] = T; saved_f[1] = last_alpha;
          memcpy(saved_f + 2, accum_rec, sizeof accum_rec); memcpy(saved_f + 5, last_color, sizeof last_color);
          memcpy(saved_f + 8, accum_normal_rec, sizeof accum_normal_rec); memcpy(saved_f + 11, last_normal, sizeof last_normal);
          memcpy(saved_d, accum_abs, sizeof accum_abs); memcpy(saved_d + 3, accum_normal_abs, sizeof accum_normal_abs);
        }
        const float max_t = t;
        const float mapped_max_t = (float)((FAR_PLANE * max_t - FAR_PLANE * NEAR_PLANE) / ((FAR_PLANE - NEAR_PLANE) * max_t));
        const float dmax_t_dd = (float)((FAR_PLANE * NEAR_PLANE) / ((FAR_PLANE - NEAR_PLANE) * max_t * max_t));
        const float normal[3] = {p.n0, p.n1, p.n2};
        const float length = (float)sqrt((double)fmaf(p.n2, p.n2, fmaf(p.n0, p.n0, p.n1 * p.n1)) + 1e-7);
        const float nn[3] = {-normal[0] / length, -normal[1] / length, -normal[2] / length};
        T = T / (1.f - alpha);
        const float dchannel_dcolor = alpha * T;
        float dL_dalpha = 0.0f;
        double* gacc = ghost ? ghost_acc : my + (size_t)gid * NS;
        for (int ch = 0; ch < 3; ++ch) {
          const float c = colors[3 * (size_t)gid + ch];
          accum_abs[ch] = last_alpha * fabs((double)last_color[ch]) + (1. - last_alpha) * accum_abs[ch];
          accum_rec[ch] = last_alpha * last_color[ch] + (1.f - last_alpha) * accum_rec[ch];
          last_color[ch] = c;
          dL_dalpha += (c - accum_rec[ch]) * dL_dpixel[ch];
          gacc[ch] += (double)(dchannel_dcolor * dL_dpixel[ch]);
        }
        const float dL_dmax_t = 2.0f * (T * alpha) * (mapped_max_t * final_A - final_D) * dL_dreg * dmax_t_dd;
        float dL_dnn[3];
        for (int ch = 0; ch < 3; ++ch) {
          accum_normal_abs[ch] = last_alpha * fabs((double)last_normal[ch]) + (1. - last_alpha) * accum_normal_abs[ch];
          accum_normal_rec[ch] = last_alpha * last_normal[ch] + (1.f - last_alpha) * accum_normal_rec[ch];
          last_normal[ch] = nn[ch];
          dL_dalpha += (nn[ch] - accum_normal_rec[ch]) * dL_dnormal2D[ch];
          dL_dnn[ch] = alpha * T * dL_dnormal2D[ch];
        }
        float dL_dlength = dL_dnn[0] * normal[0] + dL_dnn[1] * normal[1] + dL_dnn[2] * normal[2];
        dL_dlength *= 1.f / (length * length);
        float dL_dnormal[3] = {(-dL_dnn[0] + dL_dlength * normal[0]) / length, (-dL_dnn[1] + dL_dlength * normal[1]) / length,
                               (-dL_dnn[2] + dL_dlength * normal[2]) / length};
        float dL_dt = dL_dmax_t;
        if (contributor == (uint32_t)(max_contributor - 1)) dL_dt += dL_dmax_depth;
        dL_dalpha *= T;
        last_alpha = alpha;
        float bg_dot_dpixel = 0;
        for (int i = 0; i < 3; ++i) bg_dot_dpixel += bg[i] * dL_dpixel[i];
        dL_dalpha += (-T_final / (1.f - alpha)) * bg_dot_dpixel;
        const float dL_dG = con_o[3] * dL_dalpha;
        const float gdx = G * dx, gdy = G * dy;
        const float dG_ddelx = -gdx * con_o[0] - gdy * con_o[1];
        const float dG_ddely = -gdy * con_o[2] - gdx * con_o[1];
        const float gx_ = dL_dG * dG_ddelx * ddelx_dx, gy_ = dL_dG * dG_ddely * ddely_dy;
        gacc[3] += (double)gx_;
        gacc[4] += (double)gy_;
        gacc[5] += (double)(fabsf(gx_) + fabsf(gy_));
        gacc[6] += (double)(G * dL_dalpha);
        const float dL_dpower = dL_dG * G;
        const float dL_dmin_value = dL_dpower * -0.5f;
        double dL_dA = dL_dmin_value * (BB / AA) * (BB / AA) / 4.f;
        double dL_dB = dL_dmin_value * -BB / (2 * AA);
        const double dL_dC = dL_dmin_value * 1.0f;
        dL_dA += dL_dt * BB / (2 * AA * AA);
        dL_dB += dL_dt * -1.f / (2 * AA);
        dL_dnormal[0] = (float)(dL_dnormal[0] + dL_dA * rx);
        dL_dnormal[1] = (float)(dL_dnormal[1] + dL_dA * ry);
        dL_dnormal[2] = (float)(dL_dnormal[2] + dL_dA);
        gacc[7] += (double)(dL_dnormal[0] * rx);
        gacc[8] += (double)(dL_dnormal[0] * ry + dL_dnormal[1] * rx);
        gacc[9] += (double)(dL_dnormal[0] + dL_dnormal[2] * rx);
        gacc[10] += (double)(dL_dnormal[1] * ry);
        gacc[11] += (double)(dL_dnormal[1] + dL_dnormal[2] * ry);
        gacc[12] += (double)(dL_dnormal[2]);
        gacc[13] += (double)(float)(dL_dB * 2 * rx);
        gacc[14] += (double)(float)(dL_dB * 2 * ry);
        gacc[15] += (double)(float)(dL_dB * 2);
        gacc[16] += (double)(float)dL_dC;
        if (bounds) {
          /* the magnitude of every term above, operand by operand */
          const double Td = T, wT = (double)alpha * T, Gd = G, op = con_o[3];
          double m[17];
          double mA = 0, mbg = 0;
          for (int ch = 0; ch < 3; ++ch) {
            m[ch] = wT * fabs((double)dL_dpixel[ch]);
            mA += (fabs((double)colors[3 * (size_t)gid + ch]) + accum_abs[ch]) * fabs((double)dL_dpixel[ch]);
            mA += (fabs((double)nn[ch]) + accum_normal_abs[ch]) * fabs((double)dL_dnormal2D[ch]);
            mbg += fabs((double)bg[ch]) * fabs((double)dL_dpixel[ch]);
          }
          mA = mA * Td + T_final / (1. - alpha) * mbg;                 /* dL_dalpha */
          const double mG = op * mA;                                    /* dL_dG */
          m[3] = mG * Gd * (fabs((double)dx) * fabs((double)con_o[0]) + fabs((double)dy) * fabs((double)con_o[1])) * ddelx_dx;
          m[4] = mG * Gd * (fabs((double)dy) * fabs((double)con_o[2]) + fabs((double)dx) * fabs((double)con_o[1])) * ddely_dy;
          m[5] = m[3] + m[4];
          m[6] = Gd * mA;
          const double mMin = 0.5 * mG * Gd;                            /* dL_dmin_value */
          double mDt = 2.0 * wT * (fabs((double)mapped_max_t) * fabs((double)final_A) + fabs((double)final_D)) *
                       fabs((double)dL_dreg) * fabs((double)dmax_t_dd);
          if (contributor == (uint32_t)(max_contributor - 1)) mDt += fabs((double)dL_dmax_depth);
          const double q = fabs(BB / AA);
          const double mdA = mMin * q * q / 4. + mDt * fabs(BB) / (2 * AA * AA);
          const double mdB = mMin * q / 2. + mDt / (2 * fabs(AA));
          const double il = 1.0 / length;
          double mdnn[3], mlen = 0;
          for (int ch = 0; ch < 3; ++ch) { mdnn[ch] = wT * fabs((double)dL_dnormal2D[ch]); mlen += mdnn[ch] * fabs((double)normal[ch]); }
          mlen *= il * il;
          const double arx = fabs((double)rx), ary = fabs((double)ry);
          const double mN0 = (mdnn[0] + mlen * fabs((double)normal[0])) * il + mdA * arx;
          const double mN1 = (mdnn[1] + mlen * fabs((double)normal[1])) * il + mdA * ary;
          const double mN2 = (mdnn[2] + mlen * fabs((double)normal[2])) * il + mdA;
          m[7] = mN0 * arx;
          m[8] = mN0 * ary + mN1 * arx;
          m[9] = mN0 + mN2 * arx;
          m[10] = mN1 * ary;
          m[11] = mN1 + mN2 * ary;
          m[12] = mN2;
          m[13] = 2 * mdB * arx;
          m[14] = 2 * mdB * ary;
          m[15] = 2 * mdB;
          m[16] = mMin;
          for (int i = 0; i < NG; ++i) gacc[NG + i] += m[i];
          double* gmarg = my + (size_t)gid * NS + 2 * NG;
          if (ghost || (long)contributor <= marginal_upto)
            for (int i = 0; i < NG; ++i) gmarg[i] += m[i];
        }
        if (ghost) {
          T = saved_f[0]; last_alpha = saved_f[1];
          memcpy(accum_rec, saved_f + 2, sizeof accum_rec); memcpy(last_color, saved_f + 5, sizeof last_color);
          memcpy(accum_normal_rec, saved_f + 8, sizeof accum_normal_rec); memcpy(last_normal, saved_f + 11, sizeof last_normal);
          memcpy(accum_abs, saved_d, sizeof accum_abs); memcpy(accum_normal_abs, saved_d + 3, sizeof accum_normal_abs);
        }
      }
    }
  }
#pragma omp parallel for schedule(static)
  for (int g = 0; g < P; ++g) {
    double s[3 * 17] = {0};
    for (int t = 0; t < nthreads; ++t) {
      const double* a = acc + ((size_t)t * P + g) * NS;
      for (int k = 0; k < NS; ++k) s[k] += a[k];
    }
    if (bounds)
      for (int k = 0; k < NG; ++k) { mag[(size_t)NG * g + k] = s[NG + k]; marginal[(size_t)NG * g + k] = s[2 * NG + k]; }
    for (int k = 0; k < 3; ++k) dL_dcolors[3 * (size_t)g + k] = (float)s[k];
    for (int k = 0; k < 3; ++k) dL_dmean2D[3 * (size_t)g + k] = (float)s[3 + k];
    dL_dopacity[g] = (float)s[6];
    for (int k = 0; k < 10; ++k) dL_dview2gaussian[10 * (size_t)g + k] = (float)s[7 + k];
  }
  free(acc);
}

/* ---- 3x3 column-major helpers mirroring the glm operators used by backward.cu:381-587 ---- */
typedef struct { float m[3][3]; } m3;
static m3 m3_mul(m3 A, m3 B) { /* (A*B)[c][r] = sum_k A[k][r] * B[c][k] */
  m3 o;
  for (int c = 0; c < 3; ++c)
    for (int r = 0; r < 3; ++r) o.m[c][r] = A.m[0][r] * B.m[c][0] + A.m[1][r] * B.m[c][1] + A.m[2][r] * B.m[c][2];
  return o;
}
static m3 m3_t(m3 A) {
  m3 o;
  for (int c = 0; c < 3; ++c)
    for (int r = 0; r < 3; ++r) o.m[c][r] = A.m[r][c];
  return o;
}

/* backward.cu:593-631 preprocessCUDA (+ :381-587 computeView2Gaussian_backward, :20-139 SH backward).
 * Intermediate arithmetic in double (a well-conditioned evaluation of the same formulas: the formulas
 * themselves amplify rounding by ~S^-2, so the float reference is only a noisy sample of this value). */
void oracle_preprocess_backward(const oracle_scene_t* s, const int* radii, const unsigned char* clamped,
                                const float* dL_dcolor, const float* dL_dv2g, float* dL_dmean3D, float* dL_dsh,
                                float* dL_dscale, float* dL_drot) {
  const float* vm = s->viewmatrix;
#pragma omp parallel for schedule(static)
  for (int idx = 0; idx < s->P; ++idx) {
    if (!(radii[idx] > 0)) continue;
    const float* mean = s->means3D + 3 * idx;
    double dmean[3] = {0, 0, 0};
    if (s->scales && s->rotations) {
      const float* q = s->rotations + 4 * idx;
      const double r = q[0], x = q[1], y = q[2], z = q[3];
      const float* sc = s->scales + 3 * idx;
      const float* dv = dL_dv2g + 10 * (size_t)idx;
      double R[3][3];
      R[0][0] = 1. - 2. * (y * y + z * z); R[0][1] = 2. * (x * y - r * z); R[0][2] = 2. * (x * z + r * y);
      R[1][0] = 2. * (x * y + r * z); R[1][1] = 1. - 2. * (x * x + z * z); R[1][2] = 2. * (y * z - r * x);
      R[2][0] = 2. * (x * z - r * y); R[2][1] = 2. * (y * z + r * x); R[2][2] = 1. - 2. * (x * x + y * y);
      double G2V[4][3];
      for (int c = 0; c < 3; ++c)
        for (int i = 0; i < 3; ++i) G2V[c][i] = vm[i] * R[0][c] + vm[4 + i] * R[1][c] + vm[8 + i] * R[2][c];
      for (int i = 0; i < 3; ++i) G2V[3][i] = vm[i] * (double)mean[0] + vm[4 + i] * (double)mean[1] + vm[8 + i] * (double)mean[2] + vm[12 + i];
      double Rt[3][3];
      for (int c = 0; c < 3; ++c)
        for (int rr = 0; rr < 3; ++rr) Rt[c][rr] = G2V[rr][c];
      const double t[3] = {G2V[3][0], G2V[3][1], G2V[3][2]};
      double t2[3];
      for (int i = 0; i < 3; ++i) t2[i] = -Rt[0][i] * t[0] - Rt[1][i] * t[1] - Rt[2][i] * t[2];
      double si[3];
      for (int k = 0; k < 3; ++k) si[k] = 1.0 / ((double)sc[k] * sc[k] + 1e-7);
      double SR[3][3];
      for (int c = 0; c < 3; ++c)
        for (int rr = 0; rr < 3; ++rr) SR[c][rr] = si[rr] * Rt[c][rr];
      double dS[3][3] = {{dv[0], 0.5 * dv[1], 0.5 * dv[2]}, {0.5 * dv[1], dv[3], 0.5 * dv[4]}, {0.5 * dv[2], 0.5 * dv[4], dv[5]}};
      const double dB[3] = {dv[6], dv[7], dv[8]};
      const double dC = dv[9];
      double dSR[3][3], dRt[3][3];
      for (int c = 0; c < 3; ++c)
        for (int rr = 0; rr < 3; ++rr) {
          dSR[c][rr] = Rt[0][rr] * dS[c][0] + Rt[1][rr] * dS[c][1] + Rt[2][rr] * dS[c][2] + t2[rr] * dB[c];
        }
      for (int c = 0; c < 3; ++c)
        for (int rr = 0; rr < 3; ++rr) {
          /* transpose(dL_dSigma * transpose(S_inv_square_R))[c][r] = sum_k dS[k][c] * SR[k][r] */
          dRt[c][rr] = dS[0][c] * SR[0][rr] + dS[1][c] * SR[1][rr] + dS[2][c] * SR[2][rr] + si[rr] * dSR[c][rr];
        }
      double dSi[3], dt2[3];
      for (int i = 0; i < 3; ++i) {
        dSi[i] = dSR[0][i] * Rt[0][i] + dSR[1][i] * Rt[1][i] + dSR[2][i] * Rt[2][i] + dC * t2[i] * t2[i];
        dt2[i] = 2 * t2[i] * si[i] * dC + dB[0] * SR[0][i] + dB[1] * SR[1][i] + dB[2] * SR[2][i];
      }
      for (int i = 0; i < 3; ++i) dL_dscale[3 * idx + i] = (float)(-2 / (double)sc[i] * si[i] * dSi[i]);
      double dG2V[4][3], dG2W[4][3];
      for (int c = 0; c < 3; ++c)
        for (int rr = 0; rr < 3; ++rr) dG2V[c][rr] = dRt[rr][c] - dt2[c] * t[rr];
      for (int c = 0; c < 3; ++c) dG2V[3][c] = -(Rt[c][0] * dt2[0] + Rt[c][1] * dt2[1] + Rt[c][2] * dt2[2]);
      for (int c = 0; c < 4; ++c)
        for (int rr = 0; rr < 3; ++rr) dG2W[c][rr] = vm[4 * rr + 0] * dG2V[c][0] + vm[4 * rr + 1] * dG2V[c][1] + vm[4 * rr + 2] * dG2V[c][2];
      dmean[0] = dG2W[3][0]; dmean[1] = dG2W[3][1]; dmean[2] = dG2W[3][2];
#define MT(c, r) dG2W[c][r]
      dL_drot[4 * idx + 0] = (float)(2 * z * (MT(0, 1) - MT(1, 0)) + 2 * y * (MT(2, 0) - MT(0, 2)) + 2 * x * (MT(1, 2) - MT(2, 1)));
      dL_drot[4 * idx + 1] = (float)(2 * y * (MT(1, 0) + MT(0, 1)) + 2 * z * (MT(2, 0) + MT(0, 2)) + 2 * r * (MT(1, 2) - MT(2, 1)) - 4 * x * (MT(2, 2) + MT(1, 1)));
      dL_drot[4 * idx + 2] = (float)(2 * x * (MT(1, 0) + MT(0, 1)) + 2 * r * (MT(2, 0) - MT(0, 2)) + 2 * z * (MT(1, 2) + MT(2, 1)) - 4 * y * (MT(2, 2) + MT(0, 0)));
      dL_drot[4 * idx + 3] = (float)(2 * r * (MT(0, 1) - MT(1, 0)) + 2 * x * (MT(2, 0) + MT(0, 2)) + 2 * y * (MT(1, 2) + MT(2, 1)) - 4 * z * (MT(1, 1) + MT(0, 0)));
#undef MT
    }
    if (s->shs) {
      const double dox = (double)mean[0] - s->cam_pos[0], doy = (double)mean[1] - s->cam_pos[1], doz = (double)mean[2] - s->cam_pos[2];
      const double len = sqrt(dox * dox + doy * doy + doz * doz);
      const double x = dox / len, y = doy / len, z = doz / len;
      const float* sh = s->shs + (size_t)idx * s->M * 3;
      float* dsh = dL_dsh + (size_t)idx * s->M * 3;
      double dRGB[3];
      for (int c = 0; c < 3; ++c) dRGB[c] = clamped[3 * idx + c] ? 0.0 : (double)dL_dcolor[3 * idx + c];
      double dRGBdx[3] = {0}, dRGBdy[3] = {0}, dRGBdz[3] = {0};
#define SHV(k, c) ((double)sh[3 * (k) + (c)])
#define DSH(k, w) { for (int c = 0; c < 3; ++c) dsh[3 * (k) + c] = (float)((w) * dRGB[c]); }
      DSH(0, SH_C0);
      if (s->D > 0) {
        DSH(1, -SH_C1 * y); DSH(2, SH_C1 * z); DSH(3, -SH_C1 * x);
        for (int c = 0; c < 3; ++c) { dRGBdx[c] = -SH_C1 * SHV(3, c); dRGBdy[c] = -SH_C1 * SHV(1, c); dRGBdz[c] = SH_C1 * SHV(2, c); }
        if (s->D > 1) {
          const double xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
          DSH(4, SH_C2[0] * xy); DSH(5, SH_C2[1] * yz); DSH(6, SH_C2[2] * (2. * zz - xx - yy)); DSH(7, SH_C2[3] * xz); DSH(8, SH_C2[4] * (xx - yy));
          for (int c = 0; c < 3; ++c) {
            dRGBdx[c] += SH_C2[0] * y * SHV(4, c) + SH_C2[2] * 2. * -x * SHV(6, c) + SH_C2[3] * z * SHV(7, c) + SH_C2[4] * 2. * x * SHV(8, c);
            dRGBdy[c] += SH_C2[0] * x * SHV(4, c) + SH_C2[1] * z * SHV(5, c) + SH_C2[2] * 2. * -y * SHV(6, c) + SH_C2[4] * 2. * -y * SHV(8, c);
            dRGBdz[c] += SH_C2[1] * y * SHV(5, c) + SH_C2[2] * 2. * 2. * z * SHV(6, c) + SH_C2[3] * x * SHV(7, c);
          }
          if (s->D > 2) {
            DSH(9, SH_C3[0] * y * (3. * xx - yy)); DSH(10, SH_C3[1] * xy * z); DSH(11, SH_C3[2] * y * (4. * zz - xx - yy));
            DSH(12, SH_C3[3] * z * (2. * zz - 3. * xx - 3. * yy)); DSH(13, SH_C3[4] * x * (4. * zz - xx - yy));
            DSH(14, SH_C3[5] * z * (xx - yy)); DSH(15, SH_C3[6] * x * (xx - 3. * yy));
            for (int c = 0; c < 3; ++c) {
              dRGBdx[c] += SH_C3[0] * SHV(9, c) * 3. * 2. * xy + SH_C3[1] * SHV(10, c) * yz + SH_C3[2] * SHV(11, c) * -2. * xy +
                           SH_C3[3] * SHV(12, c) * -3. * 2. * xz + SH_C3[4] * SHV(13, c) * (-3. * xx + 4. * zz - yy) +
                           SH_C3[5] * SHV(14, c) * 2. * xz + SH_C3[6] * SHV(15, c) * 3. * (xx - yy);
              dRGBdy[c] += SH_C3[0] * SHV(9, c) * 3. * (xx - yy) + SH_C3[1] * SHV(10, c) * xz + SH_C3[2] * SHV(11, c) * (-3. * yy + 4. * zz - xx) +
                           SH_C3[3] * SHV(12, c) * -3. * 2. * yz + SH_C3[4] * SHV(13, c) * -2. * xy + SH_C3[5] * SHV(14, c) * -2. * yz +
                           SH_C3[6] * SHV(15, c) * -3. * 2. * xy;
              dRGBdz[c] += SH_C3[1] * SHV(10, c) * xy + SH_C3[2] * SHV(11, c) * 4. * 2. * yz + SH_C3[3] * SHV(12, c) * 3. * (2. * zz - xx - yy) +
                           SH_C3[4] * SHV(13, c) * 4. * 2. * xz + SH_C3[5] * SHV(14, c) * (xx - yy);
            }
          }
        }
      }
#undef SHV
#undef DSH
      const double ddx = dRGBdx[0] * dRGB[0] + dRGBdx[1] * dRGB[1] + dRGBdx[2] * dRGB[2];
      const double ddy = dRGBdy[0] * dRGB[0] + dRGBdy[1] * dRGB[1] + dRGBdy[2] * dRGB[2];
      const double ddz = dRGBdz[0] * dRGB[0] + dRGBdz[1] * dRGB[1] + dRGBdz[2] * dRGB[2];
      const double sum2 = dox * dox + doy * doy + doz * doz;
      const double inv = 1.0 / sqrt(sum2 * sum2 * sum2);
      dmean[0] += ((sum2 - dox * dox) * ddx - doy * dox * ddy - doz * dox * ddz) * inv;
      dmean[1] += (-dox * doy * ddx + (sum2 - doy * doy) * ddy - doz * doy * ddz) * inv;
      dmean[2] += (-dox * doz * ddx - doy * doz * ddy + (sum2 - doz * doz) * ddz) * inv;
    }
    for (int i = 0; i < 3; ++i) dL_dmean3D[3 * idx + i] = (float)dmean[i];
  }
  (void)m3_mul; (void)m3_t;
}

/* rasterizer_impl.cu:54-66 checkFrustum */
void oracle_mark_visible(int P, const float* means3D, const float* vm, unsigned char* present) {
  for (int i = 0; i < P; ++i) {
    const float z = affine(means3D[3 * i], means3D[3 * i + 1], means3D[3 * i + 2], vm[2], vm[6], vm[10], vm[14]);
    present[i] = !(z <= 0.2f);
  }
}

/* Test helper: the reference's per-pixel alpha of ONE Gaussian over the whole image (0 where the pair is rejected by
 * t <= 0.2 or alpha < 1/255), forward.cu:499-535.  Used to check conservative culling bounds. */
void oracle_alpha_map(int W, int H, float tan_fovx, float tan_fovy, const float* v2g, float opacity, float* out) {
  const float focal_y = H / (2.0f * tan_fovy), focal_x = W / (2.0f * tan_fovx);
  for (int py = 0; py < H; ++py)
    for (int px = 0; px < W; ++px) {
      const float pixfx = (float)px + 0.5f, pixfy = (float)py + 0.5f;
      const float rx = (float)((pixfx - W / 2.) / focal_x), ry = (float)((pixfy - H / 2.) / focal_y);
      const pair_t p = pair_geom(v2g, rx, ry);
      const double AA = p.AA, BB = p.BB;
      float a = 0.f;
      const float t = (float)(-BB / (2 * AA));
      if (!(t <= NEAR_PLANE)) {
        const double min_value = fma(-BB / AA, BB / 4., (double)v2g[9]);
        float power = (float)(-0.5 * min_value);
        if (power > 0.0f) power = 0.0f;
        const float alpha = fminf(0.99f, opacity * expf(power));
        if (!(alpha < 1.0f / 255.0f)) a = alpha;
      }
      out[(size_t)py * W + px] = a;
    }
}

/* =====================================================================================================
 * Opacity-field query ("integrate"): forward.cu:722-766 preprocessPointsCUDA, rasterizer_impl.cu:113-144
 * createWithKeys, forward.cu:803-1218 integrateCUDA.
 *
 * The five sub-pixel rays of pass 1 are unrolled by nvcc and share products between rays, so each ray ends up
 * with its own fusion pattern in the reference's SASS; pass 2 evaluates  -1/2 (A t^2 + B t + C)  entirely in
 * float (C ~ 1e5..1e6), so its value is defined by that exact sequence.  Both are restated below.
 * ===================================================================================================== */

/* forward.cu:722-766: returns 1 and fills xy/depth when the point projects inside the image */
static int point_project(const float* p, const float* vm, int W, int H, float focal_x, float focal_y, float* xy, float* depth) {
  const float tz = affine(p[0], p[1], p[2], vm[2], vm[6], vm[10], vm[14]);
  if (tz <= 0.2f) return 0;
  const float tx = affine(p[0], p[1], p[2], vm[0], vm[4], vm[8], vm[12]);
  const float ty = affine(p[0], p[1], p[2], vm[1], vm[5], vm[9], vm[13]);
  const float x = (float)((double)((focal_x * tx) / (tz + 0.0000001f)) + W / 2.);
  const float y = (float)((double)((focal_y * ty) / (tz + 0.0000001f)) + H / 2.);
  if (x < 0 || x >= W || y < 0 || y >= H) return 0;
  xy[0] = x; xy[1] = y; *depth = tz;
  return 1;
}

/* the five rays of forward.cu:919-930 with the reference's per-ray fusion (k = 0: centre, 1..4: corners) */
static void pair_geom_k(int k, const float* v, float rx, float ry, float* n, float* AA, float* BB) {
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
  n[0] = n0; n[1] = n1; n[2] = n2;
  *AA = fmaf(rx, n0, ry * n1) + n2;
  *BB = bh + bh;
}

#define MAX_CONTRIB 1024 /* MAX_NUM_CONTRIBUTORS * 4, forward.cu:879,986 */

/* Whole integrate for one view.  Inputs: Gaussian state + tile lists from oracle_preprocess / oracle_bin.
 * out_color [9,H,W] (channels 0-2, 6, 7, 8 written), final_T [H,W], n_contrib [H,W],
 * out_alpha_integrated [PN] (caller-initialised to 1), out_color_integrated [PN,3] (caller-initialised to 0). */
void oracle_integrate(int W, int H, float tan_fovx, float tan_fovy, const float* viewmatrix, int PN, const float* points3D,
                      const uint32_t* ranges, const uint32_t* point_list, const float* features, const float* view2gaussian,
                      const float* conic_opacity, const float* bg, float* out_color, float* final_T, uint32_t* n_contrib,
                      float* out_alpha_integrated, float* out_color_integrated) {
  const float focal_y = H / (2.0f * tan_fovy), focal_x = W / (2.0f * tan_fovx);
  const int gx = (W + BLOCK_X - 1) / BLOCK_X;
  const size_t HW = (size_t)H * W;
  /* bucket the projected points per pixel (which pixel handles a point: forward.cu:1071-1072) */
  float* pxy = (float*)malloc((size_t)PN * 2 * sizeof(float));
  float* pdepth = (float*)malloc((size_t)PN * sizeof(float));
  int* ppix = (int*)malloc((size_t)PN * sizeof(int));
  uint32_t* cnt = (uint32_t*)calloc(HW + 1, sizeof(uint32_t));
  for (int i = 0; i < PN; ++i) {
    ppix[i] = -1;
    if (point_project(points3D + 3 * (size_t)i, viewmatrix, W, H, focal_x, focal_y, pxy + 2 * (size_t)i, pdepth + i)) {
      const int px = (int)pxy[2 * (size_t)i], py = (int)pxy[2 * (size_t)i + 1];
      ppix[i] = py * W + px;
      cnt[ppix[i] + 1]++;
    }
  }
  for (size_t i = 0; i < HW; ++i) cnt[i + 1] += cnt[i];
  uint32_t* order = (uint32_t*)malloc(((size_t)cnt[HW] + 1) * sizeof(uint32_t));
  uint32_t* cur = (uint32_t*)malloc(HW * sizeof(uint32_t));
  memcpy(cur, cnt, HW * sizeof(uint32_t));
  for (int i = 0; i < PN; ++i)
    if (ppix[i] >= 0) order[cur[ppix[i]]++] = (uint32_t)i;

  static const float offx[5] = {0.0f, -0.5f, 0.5f, -0.5f, 0.5f};
  static const float offy[5] = {0.0f, -0.5f, -0.5f, 0.5f, 0.5f};
#pragma omp parallel for schedule(dynamic, 4)
  for (int py = 0; py < H; ++py) {
    uint16_t* ids = (uint16_t*)malloc(MAX_CONTRIB * sizeof(uint16_t));
    for (int px = 0; px < W; ++px) {
      const size_t pix_id = (size_t)W * py + px;
      const float pixfx = (float)px + 0.5f, pixfy = (float)py + 0.5f;
      const uint32_t* range = ranges + 2 * ((py / BLOCK_Y) * gx + (px / BLOCK_X));
      float rxk[5], ryk[5];
      for (int k = 0; k < 5; ++k) {
        rxk[k] = (float)((pixfx + offx[k] - W / 2.) / focal_x);
        ryk[k] = (float)((pixfy + offy[k] - H / 2.) / focal_y);
      }
      float Ts[5] = {1, 1, 1, 1, 1};
      float C[8] = {0};
      uint32_t contributor = 0, last_contributor = 0, n_local = 0;
      /* pass 1, forward.cu:886-993 */
      for (uint32_t kk = range[0]; kk < range[1]; ++kk) {
        contributor++;
        const uint32_t gid = point_list[kk];
        const float* v = view2gaussian + 10 * (size_t)gid;
        const float opac = conic_opacity[4 * (size_t)gid + 3];
        int used = 0;
        for (int k = 0; k < 5; ++k) {
          float nrm[3], AA, BB;
          pair_geom_k(k, v, rxk[k], ryk[k], nrm, &AA, &BB);
          const float CC = v[9];
          const float t = -BB / (2 * AA);
          if (t <= NEAR_PLANE) continue;
          const double min_value = fma((double)(-BB / AA), (double)BB / 4., (double)CC);
          float power = (float)(-0.5 * min_value);
          if (power > 0.0f) power = 0.0f;
          const float alpha = fminf(0.99f, opac * expf(power));
          if (alpha < 1.0f / 255.0f) continue;
          const float test_T = Ts[k] * (1 - alpha);
          if (test_T < 0.0001f) continue;
          if (k == 0)
            for (int ch = 0; ch < 3; ++ch) C[ch] = fmaf(Ts[0], alpha * features[3 * (size_t)gid + ch], C[ch]);
          if (t > C[6]) C[6] = t;
          if (k == 0) C[7] = fmaf(Ts[0], alpha, C[7]);
          Ts[k] = test_T;
          used = 1;
        }
        if (used) {
          last_contributor = contributor;
          ids[n_local++] = (uint16_t)contributor;
          if (n_local >= MAX_CONTRIB) break;
        }
      }
      final_T[pix_id] = Ts[0];
      n_contrib[pix_id] = last_contributor;
      float col[3];
      for (int ch = 0; ch < 3; ++ch) { col[ch] = fmaf(Ts[0], bg[ch], C[ch]); out_color[ch * HW + pix_id] = col[ch]; }
      out_color[6 * HW + pix_id] = C[6];
      out_color[7 * HW + pix_id] = C[7];
      /* pass 2, forward.cu:1116-1210: every point of this pixel against the recorded contributors */
      const uint32_t p0 = cnt[pix_id], p1 = cnt[pix_id + 1];
      for (uint32_t q = p0; q < p1; ++q) {
        const uint32_t id = order[q];
        const float rx = (float)(((double)pxy[2 * (size_t)id] - W / 2.) / focal_x);
        const float ry = (float)(((double)pxy[2 * (size_t)id + 1] - H / 2.) / focal_y);
        const float ray_depth = pdepth[id];
        float point_alpha = 0.f, point_T = 1.f;
        uint32_t num_iterated = 0, second = 0;
        for (uint32_t kk = range[0]; kk < range[1]; ++kk) {
          num_iterated++;
          if (num_iterated > last_contributor) break;
          if (second >= n_local || num_iterated != (uint32_t)ids[second]) continue;
          second++;
          const uint32_t gid = point_list[kk];
          const float* v = view2gaussian + 10 * (size_t)gid;
          const pair_t p = pair_geom(v, rx, ry);
          float t = -p.BB / (2 * p.AA);
          if (t > ray_depth) t = ray_depth;
          const float power = -0.5f * (v[9] + fmaf(p.BB, t, (p.AA * t) * t));
          const float alpha = fminf(0.99f, conic_opacity[4 * (size_t)gid + 3] * expf(power));
          if (alpha < 1.0f / 255.0f) continue;
          point_alpha = fmaf(alpha, point_T, point_alpha);
          point_T = point_T * (1 - alpha);
        }
        out_alpha_integrated[id] = point_alpha;
        for (int ch = 0; ch < 3; ++ch) out_color_integrated[3 * (size_t)id + ch] = col[ch];
      }
      out_color[8 * HW + pix_id] = (float)(p1 - p0);
    }
    free(ids);
  }
  free(pxy); free(pdepth); free(ppix); free(cnt); free(order); free(cur);
}
