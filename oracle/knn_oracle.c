/* knn_oracle.c -- TEST INFRASTRUCTURE ONLY.  Brute-force CPU restatement of simple_knn's distCUDA2
 * (submodules/simple-knn/spatial.cu:15-25, simple_knn.cu:132-183), the contract of gof_knn_mean_dist (DESIGN section 4.5):
 *
 *   d(i,j) = fmaf(dz, dz, fmaf(dx, dx, dy*dy)), dx = x_j - x_i, ...  over every j != i (by index) -- the reference's
 *   d.x*d.x + d.y*d.y + d.z*d.z as nvcc contracts it (its SASS: FMUL of dy, FFMA of dx, FFMA of dz);
 *   accepted only if d < FLT_MAX (the reference's `knn[j] > dist` with knn[] starting at FLT_MAX);
 *   b0 <= b1 <= b2 the three smallest accepted, padded with FLT_MAX;  out_i = ((b0 + b1) + b2) / 3.0f.
 *
 * Built with -ffp-contract=off -fno-fast-math, so every operation is the one written.  The insertion is the reference's
 * (updateKBest<3>); with an explicit fmaf both the plain and the FMA-instruction builds compute the same bits.
 */
#include <float.h>
#include <math.h>
#include <stddef.h>

static inline void knn_insert(float d, float* b) {
  for (int k = 0; k < 3; ++k)
    if (b[k] > d) { const float t = b[k]; b[k] = d; d = t; }
}

#define KNN_QUERY_BODY                                                        \
  const float qx = pts[3 * (size_t)i], qy = pts[3 * (size_t)i + 1], qz = pts[3 * (size_t)i + 2]; \
  b[0] = b[1] = b[2] = FLT_MAX;                                               \
  for (long long j = 0; j < P; ++j) {                                         \
    if (j == i) continue;                                                     \
    const float dx = pts[3 * (size_t)j] - qx, dy = pts[3 * (size_t)j + 1] - qy, dz = pts[3 * (size_t)j + 2] - qz; \
    knn_insert(fmaf(dz, dz, fmaf(dx, dx, dy * dy)), b);                       \
  }

static void query_plain(long long P, const float* pts, long long i, float* b) { KNN_QUERY_BODY }

#if defined(__x86_64__) && defined(__GNUC__)
/* the same source compiled to use the FMA instruction instead of a libm call (identical results: fmaf is exact-then-round) */
__attribute__((target("fma"))) static void query_fma(long long P, const float* pts, long long i, float* b) { KNN_QUERY_BODY }
#endif

/* queries: NULL = all P points (out [P]), else the nq point indices to evaluate (out [nq]).  best: [n,3] or NULL. */
void gof_oracle_knn_mean_dist(int P, const float* pts, int nq, const int* queries, float* out, float* best) {
  const long long n = queries ? nq : P;
  int use_fma = 0;
#if defined(__x86_64__) && defined(__GNUC__)
  __builtin_cpu_init();
  use_fma = __builtin_cpu_supports("fma");
#endif
#pragma omp parallel for schedule(dynamic, 16)
  for (long long q = 0; q < n; ++q) {
    const long long i = queries ? queries[q] : q;
    float b[3];
#if defined(__x86_64__) && defined(__GNUC__)
    if (use_fma) query_fma(P, pts, i, b); else
#endif
    query_plain(P, pts, i, b);
    out[q] = ((b[0] + b[1]) + b[2]) / 3.0f;
    if (best) { best[3 * q] = b[0]; best[3 * q + 1] = b[1]; best[3 * q + 2] = b[2]; }
  }
  (void)use_fma;
}
