// view_loss.cuh -- the per-view training loss on the rasterizer's 9-channel output and its gradient, in one pass
// over the image (reference: train.py:151-188 with utils/loss_utils.py:17-63 and utils/depth_utils.py:6-35):
//
//   loss = (1-l) * mean|rgb - gt| + l * (1 - SSIM(rgb, gt)) + l_dn * mean(1 - n_world . n_depth) + l_dist * mean(distortion)
//
// STAGED COMPONENT (SURVEY.md 8(f) rank 1): not on the rasterizer's drop-in path.  The work of one 16x16 pixel tile is
// written as PHASES -- device functions of (tile, thread id, shared block) separated by block barriers -- so that
// tests/hostmath can compile this very file for the host, run the phases thread by thread, and check the result against
// an independent CPU restatement pinned to the reference's own Python, without a GPU.
//
//   kernel A (vl_a_*):  SSIM statistics of the tile (11x11 window, zero padding) -> SSIM map sum, L1 sum, and the three
//                       derivative maps d map/d(mu1, E11, E12) for kernel B; depth -> normal on a 2-pixel halo, normal
//                       consistency error and its gradient w.r.t. the rendered normal (ch 3-5) and the depth (ch 6);
//                       distortion mean and its constant gradient (ch 8); per-tile partial sums.
//   kernel B (vl_b_*):  blurs the derivative maps back (the window is symmetric) and writes the rgb gradient (ch 0-2).
//   kernel C:           fixed-order sum of the per-tile partials in double -> the four terms and the loss.
//
// Appearance mode (mapping != NULL; train.py:67-88, 157-159 with --use_decoupled_appearance): the L1 term becomes
// mean over the crop (top, left, Hc, Wc) of |fl(m * rgb) - gt|, m = mapping[c][y-top][x-left] the appearance network's
// output; SSIM, the normal and the distortion terms stay on the whole image.  Kernel A sums that L1 over the crop only,
// kernel B adds its rgb gradient inside the crop and writes d loss / d mapping, kernel C divides by 3 Hc Wc.  With
// mapping == NULL every phase does exactly what it did before the mode existed.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define VL_HD __host__ __device__ __forceinline__
#else
#define VL_HD static inline
#endif

#define VL_TILE 16
#define VL_R 5                       // window radius (11 taps)
#define VL_HT (VL_TILE + 2 * VL_R)   // 26: tile + SSIM halo
#define VL_DT (VL_TILE + 4)          // 20: tile + 2-pixel halo for depth -> normal -> depth gradient
#define VL_NT (VL_TILE + 2)          // 18: tile + 1-pixel halo (pixels whose normal a tile pixel's depth feeds)
#define VL_THREADS 256

struct VlParams {
  int W, H, tiles_x, tiles_y;
  const float* render;   // [9][H][W]
  const float* gt;       // [3][H][W]
  float R[9];            // camera-to-world rotation, row-major: (world_view_transform^T)^-1 [:3,:3]  (train.py:178)
  float fx, fy;          // W / (2 tan(FoVx/2)), H / (2 tan(FoVy/2))                                 (depth_utils.py:9-10)
  float g[11];           // normalised 1-D Gaussian window, sigma 1.5                                (loss_utils.py:23-25)
  float lam, lam_dn, lam_dist;
  float inv_N, inv_N3;   // 1/(H W), 1/(3 H W)
  float* dmap;           // [9][H][W] scratch: d map/d mu1 [3], d map/d E11 [3], d map/d E12 [3]
  float* grad;           // [9][H][W] out (may be NULL: values only)
  float* partial;        // [tiles][4]: sum of SSIM map, sum |rgb-gt|, sum normal error, sum distortion
  // appearance mode; the defaults are the plain L1
  const float* mapping = nullptr;   // [3][Hc][Wc] appearance mapping, or NULL
  float* grad_mapping = nullptr;    // [3][Hc][Wc] out: d loss / d mapping (NULL exactly when grad is)
  int top = 0, left = 0, Hc = 0, Wc = 0;
  float inv_Na3 = 0.f;              // 1/(3 Hc Wc)
};

struct VlShared {
  float a[VL_HT * VL_HT], b[VL_HT * VL_HT];      // image / ground-truth halo tile (kernel B: derivative maps 0 and 1)
  float c[VL_HT * VL_HT];                        // kernel B: derivative map 2
  float h[5][VL_HT * VL_TILE];                   // horizontally blurred rows
  float red[4][VL_THREADS];                      // per-thread partial sums
  float P[VL_DT * VL_DT][3];                     // depth * ray direction (the camera origin cancels in the differences)
  float dn[VL_NT * VL_NT][3];                    // depth normal (zero on the image border)
  float ga[VL_NT * VL_NT][3], gb[VL_NT * VL_NT][3];   // gradient w.r.t. the two central differences
};

VL_HD float vl_load(const float* plane, int W, int H, int x, int y) {
  return (x >= 0 && x < W && y >= 0 && y < H) ? plane[(size_t)y * W + x] : 0.0f;
}

// m * v rounded to float before anything else touches it (torch's `mapping_image * crop_image`): no fused multiply-add
VL_HD float vl_mul_rn(float m, float v) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(m, v);
#else
  return m * v;
#endif
}

// appearance mode: is image pixel (x, y) inside the crop, and the offset of its mapping value in channel 0
VL_HD bool vl_in_crop(const VlParams& p, int x, int y) {
  return x >= p.left && x < p.left + p.Wc && y >= p.top && y < p.top + p.Hc;
}
VL_HD size_t vl_crop_offset(const VlParams& p, int x, int y) { return (size_t)(y - p.top) * p.Wc + (x - p.left); }

VL_HD void vl_cross(const float* a, const float* b, float* o) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}

VL_HD void vl_ray(const VlParams& p, int x, int y, float* rd) {   // depth_utils.py:16-18: R K^-1 (x+0.5, y+0.5, 1)
  const float kx = ((float)x + 0.5f - 0.5f * (float)p.W) / p.fx, ky = ((float)y + 0.5f - 0.5f * (float)p.H) / p.fy;
  rd[0] = p.R[0] * kx + p.R[1] * ky + p.R[2];
  rd[1] = p.R[3] * kx + p.R[4] * ky + p.R[5];
  rd[2] = p.R[6] * kx + p.R[7] * ky + p.R[8];
}

// ------------------------------------------------------------------------------------------------ kernel A
VL_HD void vl_a_zero(VlShared& s, int tid) {
  for (int q = 0; q < 4; ++q) s.red[q][tid] = 0.0f;
}

// phase A1(ch): halo tiles of render[ch] and gt[ch]
VL_HD void vl_a_load(const VlParams& p, VlShared& s, int tile_x, int tile_y, int ch, int tid) {
  const size_t plane = (size_t)p.W * p.H;
  for (int i = tid; i < VL_HT * VL_HT; i += VL_THREADS) {
    const int r = i / VL_HT, c = i - r * VL_HT;
    const int x = tile_x * VL_TILE + c - VL_R, y = tile_y * VL_TILE + r - VL_R;
    s.a[i] = vl_load(p.render + ch * plane, p.W, p.H, x, y);
    s.b[i] = vl_load(p.gt + ch * plane, p.W, p.H, x, y);
  }
}

// phase A2: horizontal pass of the five blurs (mu1, mu2, E11, E22, E12)
VL_HD void vl_a_hblur(const VlParams& p, VlShared& s, int tid) {
  for (int i = tid; i < VL_HT * VL_TILE; i += VL_THREADS) {
    const int r = i / VL_TILE, c = i - r * VL_TILE;
    float m1 = 0.f, m2 = 0.f, e11 = 0.f, e22 = 0.f, e12 = 0.f;
    for (int k = 0; k < 2 * VL_R + 1; ++k) {
      const float w = p.g[k], va = s.a[r * VL_HT + c + k], vb = s.b[r * VL_HT + c + k];
      m1 += w * va; m2 += w * vb; e11 += w * va * va; e22 += w * vb * vb; e12 += w * va * vb;
    }
    s.h[0][i] = m1; s.h[1][i] = m2; s.h[2][i] = e11; s.h[3][i] = e22; s.h[4][i] = e12;
  }
}

// phase A3(ch): vertical pass, SSIM map and its derivatives at this thread's pixel (loss_utils.py:42-58)
VL_HD void vl_a_ssim(const VlParams& p, VlShared& s, int tile_x, int tile_y, int ch, int tid) {
  const int lx = tid % VL_TILE, ly = tid / VL_TILE;
  const int x = tile_x * VL_TILE + lx, y = tile_y * VL_TILE + ly;
  if (x >= p.W || y >= p.H) return;
  float v[5];
  for (int q = 0; q < 5; ++q) {
    float acc = 0.f;
    for (int k = 0; k < 2 * VL_R + 1; ++k) acc += p.g[k] * s.h[q][(ly + k) * VL_TILE + lx];
    v[q] = acc;
  }
  const float mu1 = v[0], mu2 = v[1];
  const float s11 = v[2] - mu1 * mu1, s22 = v[3] - mu2 * mu2, s12 = v[4] - mu1 * mu2;
  const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
  const float A1 = 2.f * mu1 * mu2 + C1, A2 = 2.f * s12 + C2, B1 = mu1 * mu1 + mu2 * mu2 + C1, B2 = s11 + s22 + C2;
  const float iB = 1.0f / (B1 * B2);
  const float map = A1 * A2 * iB;
  // map as a function of (mu1, E11, E12), E11 = blur(img^2), E12 = blur(img*gt)
  const float dm_dmu1 = (2.f * mu2 * (A2 - A1)) * iB - map * (2.f * mu1 * (B2 - B1)) * iB;
  const float dm_de11 = -map / B2;
  const float dm_de12 = 2.f * A1 * iB;
  const size_t plane = (size_t)p.W * p.H, o = (size_t)y * p.W + x;
  p.dmap[(0 + ch) * plane + o] = dm_dmu1;
  p.dmap[(3 + ch) * plane + o] = dm_de11;
  p.dmap[(6 + ch) * plane + o] = dm_de12;
  const float va = s.a[(ly + VL_R) * VL_HT + lx + VL_R], vb = s.b[(ly + VL_R) * VL_HT + lx + VL_R];
  s.red[0][tid] += map;
  if (p.mapping == nullptr) {
    s.red[1][tid] += fabsf(va - vb);
  } else if (vl_in_crop(p, x, y)) {
    const float m = p.mapping[(size_t)ch * p.Hc * p.Wc + vl_crop_offset(p, x, y)];
    s.red[1][tid] += fabsf(vl_mul_rn(m, va) - vb);
  }
}

// phase N1: depth * ray direction on the 20x20 halo tile (outside the image: zero, never used)
VL_HD void vl_a_points(const VlParams& p, VlShared& s, int tile_x, int tile_y, int tid) {
  const size_t plane = (size_t)p.W * p.H;
  for (int i = tid; i < VL_DT * VL_DT; i += VL_THREADS) {
    const int r = i / VL_DT, c = i - r * VL_DT;
    const int x = tile_x * VL_TILE + c - 2, y = tile_y * VL_TILE + r - 2;
    float rd[3] = {0.f, 0.f, 0.f};
    float d = 0.f;
    if (x >= 0 && x < p.W && y >= 0 && y < p.H) { d = p.render[6 * plane + (size_t)y * p.W + x]; vl_ray(p, x, y, rd); }
    s.P[i][0] = d * rd[0]; s.P[i][1] = d * rd[1]; s.P[i][2] = d * rd[2];
  }
}

// world-space unit normal of the render at (x, y): normalize(render[3:6]) rotated by R (train.py:175-180)
VL_HD void vl_world_normal(const VlParams& p, int x, int y, float* n, float* nl, float* u, float* nw) {
  const size_t plane = (size_t)p.W * p.H, o = (size_t)y * p.W + x;
  n[0] = p.render[3 * plane + o]; n[1] = p.render[4 * plane + o]; n[2] = p.render[5 * plane + o];
  const float len = sqrtf(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
  *nl = len > 1e-12f ? len : 1e-12f;                               // F.normalize eps
  u[0] = n[0] / *nl; u[1] = n[1] / *nl; u[2] = n[2] / *nl;
  nw[0] = p.R[0] * u[0] + p.R[1] * u[1] + p.R[2] * u[2];
  nw[1] = p.R[3] * u[0] + p.R[4] * u[1] + p.R[5] * u[2];
  nw[2] = p.R[6] * u[0] + p.R[7] * u[1] + p.R[8] * u[2];
}

// phase N2: depth normal and the gradient w.r.t. its two central differences on the 18x18 halo tile
// (depth_utils.py:29-34; only interior image pixels have a normal)
VL_HD void vl_a_normals(const VlParams& p, VlShared& s, int tile_x, int tile_y, int tid) {
  for (int i = tid; i < VL_NT * VL_NT; i += VL_THREADS) {
    const int r = i / VL_NT, c = i - r * VL_NT;
    const int x = tile_x * VL_TILE + c - 1, y = tile_y * VL_TILE + r - 1;
    for (int k = 0; k < 3; ++k) { s.dn[i][k] = 0.f; s.ga[i][k] = 0.f; s.gb[i][k] = 0.f; }
    if (x < 1 || x > p.W - 2 || y < 1 || y > p.H - 2) continue;
    const int pc = (r + 1) * VL_DT + (c + 1);                        // this pixel in the 20x20 tile
    float dxv[3], dyv[3], cr[3];
    for (int k = 0; k < 3; ++k) {
      dxv[k] = s.P[pc + VL_DT][k] - s.P[pc - VL_DT][k];              // points[2:, 1:-1] - points[:-2, 1:-1]
      dyv[k] = s.P[pc + 1][k] - s.P[pc - 1][k];                      // points[1:-1, 2:] - points[1:-1, :-2]
    }
    vl_cross(dxv, dyv, cr);
    const float len = sqrtf(cr[0] * cr[0] + cr[1] * cr[1] + cr[2] * cr[2]);
    const float cl = len > 1e-12f ? len : 1e-12f;
    float d[3] = {cr[0] / cl, cr[1] / cl, cr[2] / cl};
    for (int k = 0; k < 3; ++k) s.dn[i][k] = d[k];
    if (p.grad == nullptr || p.lam_dn == 0.0f) continue;
    float n[3], nl, u[3], nw[3];
    vl_world_normal(p, x, y, n, &nl, u, nw);
    const float sc = -p.lam_dn * p.inv_N;
    float gd[3] = {sc * nw[0], sc * nw[1], sc * nw[2]};              // dL/d(depth normal)
    float gc[3];
    if (len > 1e-12f) {
      const float dg = d[0] * gd[0] + d[1] * gd[1] + d[2] * gd[2];
      for (int k = 0; k < 3; ++k) gc[k] = (gd[k] - d[k] * dg) / cl;
    } else {
      for (int k = 0; k < 3; ++k) gc[k] = gd[k] / 1e-12f;
    }
    float ga[3], gb[3];
    vl_cross(dyv, gc, ga);                                           // c = a x b:  dc.g = da.(b x g) + db.(g x a)
    vl_cross(gc, dxv, gb);
    for (int k = 0; k < 3; ++k) { s.ga[i][k] = ga[k]; s.gb[i][k] = gb[k]; }
  }
}

// phase N3: this thread's pixel: normal-consistency error, gradients of channels 3-8
VL_HD void vl_a_pixel(const VlParams& p, VlShared& s, int tile_x, int tile_y, int tid) {
  const int lx = tid % VL_TILE, ly = tid / VL_TILE;
  const int x = tile_x * VL_TILE + lx, y = tile_y * VL_TILE + ly;
  if (x >= p.W || y >= p.H) return;
  const size_t plane = (size_t)p.W * p.H, o = (size_t)y * p.W + x;
  const int ic = (ly + 1) * VL_NT + (lx + 1);                        // this pixel in the 18x18 tile
  float n[3], nl, u[3], nw[3];
  vl_world_normal(p, x, y, n, &nl, u, nw);
  const float* d = s.dn[ic];
  s.red[2][tid] += 1.0f - (nw[0] * d[0] + nw[1] * d[1] + nw[2] * d[2]);
  s.red[3][tid] += p.render[8 * plane + o];
  if (p.grad == nullptr) return;
  // d/d(render normal): dL/du = -R^T dn * l_dn / N, through u = n / max(|n|, eps)
  const float sc = -p.lam_dn * p.inv_N;
  float gu[3] = {sc * (p.R[0] * d[0] + p.R[3] * d[1] + p.R[6] * d[2]), sc * (p.R[1] * d[0] + p.R[4] * d[1] + p.R[7] * d[2]),
                 sc * (p.R[2] * d[0] + p.R[5] * d[1] + p.R[8] * d[2])};
  const float len = sqrtf(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
  float gn[3];
  if (len > 1e-12f) {
    const float ug = u[0] * gu[0] + u[1] * gu[1] + u[2] * gu[2];
    for (int k = 0; k < 3; ++k) gn[k] = (gu[k] - u[k] * ug) / nl;
  } else {
    for (int k = 0; k < 3; ++k) gn[k] = gu[k] / 1e-12f;
  }
  p.grad[3 * plane + o] = gn[0]; p.grad[4 * plane + o] = gn[1]; p.grad[5 * plane + o] = gn[2];
  // d/d(depth): this pixel's point enters the differences of its four neighbours
  float gP[3], rd[3];
  for (int k = 0; k < 3; ++k) gP[k] = s.ga[ic - VL_NT][k] - s.ga[ic + VL_NT][k] + s.gb[ic - 1][k] - s.gb[ic + 1][k];
  vl_ray(p, x, y, rd);
  p.grad[6 * plane + o] = gP[0] * rd[0] + gP[1] * rd[1] + gP[2] * rd[2];
  p.grad[7 * plane + o] = 0.0f;                                      // the alpha channel does not enter the loss
  p.grad[8 * plane + o] = p.lam_dist * p.inv_N;
}

// phase R(stride): tree reduction of the per-thread partial sums; after stride 1 thread 0 writes the tile's partials
VL_HD void vl_a_reduce(const VlParams& p, VlShared& s, int tile, int stride, int tid) {
  if (tid < stride)
    for (int q = 0; q < 4; ++q) s.red[q][tid] += s.red[q][tid + stride];
  if (stride == 1 && tid == 0)
    for (int q = 0; q < 4; ++q) p.partial[(size_t)tile * 4 + q] = s.red[q][0];
}

// ------------------------------------------------------------------------------------------------ kernel B
VL_HD void vl_b_load(const VlParams& p, VlShared& s, int tile_x, int tile_y, int ch, int tid) {
  const size_t plane = (size_t)p.W * p.H;
  for (int i = tid; i < VL_HT * VL_HT; i += VL_THREADS) {
    const int r = i / VL_HT, c = i - r * VL_HT;
    const int x = tile_x * VL_TILE + c - VL_R, y = tile_y * VL_TILE + r - VL_R;
    s.a[i] = vl_load(p.dmap + (0 + ch) * plane, p.W, p.H, x, y);
    s.b[i] = vl_load(p.dmap + (3 + ch) * plane, p.W, p.H, x, y);
    s.c[i] = vl_load(p.dmap + (6 + ch) * plane, p.W, p.H, x, y);
  }
}

VL_HD void vl_b_hblur(const VlParams& p, VlShared& s, int tid) {
  for (int i = tid; i < VL_HT * VL_TILE; i += VL_THREADS) {
    const int r = i / VL_TILE, c = i - r * VL_TILE;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    for (int k = 0; k < 2 * VL_R + 1; ++k) {
      const float w = p.g[k];
      s0 += w * s.a[r * VL_HT + c + k]; s1 += w * s.b[r * VL_HT + c + k]; s2 += w * s.c[r * VL_HT + c + k];
    }
    s.h[0][i] = s0; s.h[1][i] = s1; s.h[2][i] = s2;
  }
}

// d(loss)/d(rgb) = (1-l) sign(rgb-gt)/N3 - l/N3 * (blur(dm_dmu1) + 2 rgb blur(dm_dE11) + gt blur(dm_dE12))
VL_HD void vl_b_grad(const VlParams& p, VlShared& s, int tile_x, int tile_y, int ch, int tid) {
  const int lx = tid % VL_TILE, ly = tid / VL_TILE;
  const int x = tile_x * VL_TILE + lx, y = tile_y * VL_TILE + ly;
  if (x >= p.W || y >= p.H) return;
  float v[3];
  for (int q = 0; q < 3; ++q) {
    float acc = 0.f;
    for (int k = 0; k < 2 * VL_R + 1; ++k) acc += p.g[k] * s.h[q][(ly + k) * VL_TILE + lx];
    v[q] = acc;
  }
  const size_t plane = (size_t)p.W * p.H, o = (size_t)y * p.W + x;
  const float va = p.render[ch * plane + o], vb = p.gt[ch * plane + o];
  if (p.mapping == nullptr) {
    const float df = va - vb;
    const float sgn = df > 0.f ? 1.f : (df < 0.f ? -1.f : 0.f);
    p.grad[ch * plane + o] = (1.0f - p.lam) * sgn * p.inv_N3 - p.lam * p.inv_N3 * (v[0] + 2.f * va * v[1] + vb * v[2]);
    return;
  }
  // appearance mode: the L1 term lives on the crop only; its sign is that of fl(m rgb) - gt (sgn(0) = 0, torch's abs)
  float l1 = 0.f;
  if (vl_in_crop(p, x, y)) {
    const size_t oc = (size_t)ch * p.Hc * p.Wc + vl_crop_offset(p, x, y);
    const float m = p.mapping[oc];
    const float df = vl_mul_rn(m, va) - vb;
    const float c = df > 0.f ? (1.0f - p.lam) * p.inv_Na3 : (df < 0.f ? -(1.0f - p.lam) * p.inv_Na3 : 0.f);
    l1 = c * m;
    p.grad_mapping[oc] = c * va;
  }
  p.grad[ch * plane + o] = l1 - p.lam * p.inv_N3 * (v[0] + 2.f * va * v[1] + vb * v[2]);
}
