// integrate.cu -- the opacity-field query of mesh extraction: K10/K11/K13 of the reference
// (forward.cu:722-766 preprocessPointsCUDA, rasterizer_impl.cu:113-144 createWithKeys, forward.cu:803-1218
// integrateCUDA), restructured:
//  * points are binned per tile with one stable radix sort on the tile id (their depth order inside a tile cannot
//    influence any output, SURVEY.md A.6), no second host round-trip for the point count;
//  * pass 1 (per pixel, five sub-pixel rays, records which Gaussians contribute) keeps the reference's arithmetic --
//    including the different FMA fusion nvcc gave each of the five unrolled rays -- but only visits Gaussians whose
//    alpha-support box holds one of the warp's pixels (preprocess builds that box for all five rays, gof_cull_bbox with
//    margin 0.5);
//  * pass 2 is POINT-parallel: one thread per query point walks the contributor list of the pixel the point falls in
//    and gathers the records directly, instead of every pixel thread rescanning all points of the tile and keeping
//    8 KB of per-thread arrays (forward.cu:879,1015-1017,1104-1105);
//  * persistent CTAs (3 per SM) with a private 512 KB contributor-list slab each.
// Results are identical to the reference's: same contributor selection, uint16 id semantics, 1024-contributor cap.
#include <stdlib.h>

#include <algorithm>
#include <type_traits>

#include "gof_common.cuh"
#include "gof_math.cuh"

namespace {

constexpr int PT_KEY_SHIFT = 8;   // point key = tile << 8 | pixel slot inside the tile (points of one pixel become neighbours)
// bits of that key, the sentinel tile (not projected) included
inline int pt_key_bits(int tiles) { return gof_bits_for(((uint32_t)tiles + 1u) << PT_KEY_SHIFT); }

struct PtArgs {
  int PN, W, H, grid_x, grid_y, tiles;
  float focal_x, focal_y;
  const float* points3D;
  const float* vm;
  float2* xy;
  float* depth;
  uint32_t* key;
  uint32_t* val;
};

// forward.cu:722-766 + rasterizer_impl.cu:113-144
__global__ void __launch_bounds__(256) k_preprocess_points(const PtArgs a) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= a.PN) return;
  const float px = a.points3D[3 * (size_t)idx], py = a.points3D[3 * (size_t)idx + 1], pz = a.points3D[3 * (size_t)idx + 2];
  const float* vm = a.vm;
  uint32_t key = (uint32_t)a.tiles << PT_KEY_SHIFT;   // sentinel: not projected
  const float tz = gof_affine(px, py, pz, __ldg(vm + 2), __ldg(vm + 6), __ldg(vm + 10), __ldg(vm + 14));
  if (!(tz <= 0.2f)) {
    const float tx = gof_affine(px, py, pz, __ldg(vm + 0), __ldg(vm + 4), __ldg(vm + 8), __ldg(vm + 12));
    const float ty = gof_affine(px, py, pz, __ldg(vm + 1), __ldg(vm + 5), __ldg(vm + 9), __ldg(vm + 13));
    const float den = F_ADD(tz, 0.0000001f);
    const float x = (float)D_FMA((double)a.W, 0.5, (double)F_DIV(F_MUL(a.focal_x, tx), den));
    const float y = (float)D_FMA((double)a.H, 0.5, (double)F_DIV(F_MUL(a.focal_y, ty), den));
    if (!(x < 0 || x >= a.W || y < 0 || y >= a.H)) {
      a.xy[idx] = make_float2(x, y);
      a.depth[idx] = tz;
      int cx = gof_f2i_rz(x * 0.0625f), cy = gof_f2i_rz(y * 0.0625f);
      cx = min(a.grid_x - 1, max(0, cx));
      cy = min(a.grid_y - 1, max(0, cy));
      // the thread slot of the pixel the point falls in, as pass 2 finds it: sorting on it makes the points of one pixel --
      // which replay the SAME contributor list -- neighbours, so a warp's record gathers coincide
      key = ((uint32_t)(cy * a.grid_x + cx) << PT_KEY_SHIFT) | (uint32_t)gof_point_slot(x, y, cx, cy);
    }
  }
  a.key[idx] = key;
  a.val[idx] = (uint32_t)idx;
}

// One view's query state, read by the forward and the backward alike (int_query fills it)
struct IntQuery {
  int W, H, grid_x, tiles;
  float focal_x, focal_y;
  const uint2* ranges;          // per tile: its Gaussian list in point_list
  const uint32_t* point_list;
  const GofSplat* splat;
  const uint2* pranges;         // per tile: its points in pt_list
  const uint32_t* pt_list;      // point ids sorted by tile and pixel slot
  const float2* pt_xy;
  const float* pt_depth;
  uint16_t* ids;                // [gridDim][256][1024] contributor slab
};

struct IntArgs : IntQuery {
  const float* bg;
  float* final_T;       // tile-major plane 0 of the image state
  uint32_t* ncontrib;   // tile-major planes 0 (last contributor) and 1 (contributors recorded, for export_state)
  float* out_color;     // [9][H][W]
  float* out_alpha;     // [PN]
  float* out_color_int; // [PN][3]
  // k_integrate<true> (the running minimum over views, DESIGN.md 4.12): writes only these two
  float* alpha_min;     // [PN]
  int* argmin;          // [PN]
  int view;
  float* color_min;     // [PN][3], k_integrate<true, true>: the winning view's pixel colour (DESIGN.md 4.13)
  // k_integrate<true, *, true> (DESIGN.md 4.14): the winning view's d alpha_integrated / d point, world space
  float* grad_min;      // [PN][3]
  const float* points3D;
  const float* vm;
};

constexpr int BATCH = GOF_BLOCK_SIZE;

// forward.cu:919-930: the five rays (k = 0 centre, 1..4 corners) with the reference's per-ray fusion pattern
template <int K>
__device__ __forceinline__ void pair_geom_k(const float* v, float rx, float ry, float* AA, float* BB) {
  float n0, n1, n2, bh;
  if (K == 0) {
    n0 = F_ADD(F_FMA(rx, v[0], F_MUL(ry, v[1])), v[2]);
    n1 = F_ADD(F_FMA(rx, v[1], F_MUL(ry, v[3])), v[4]);
    n2 = F_ADD(F_FMA(ry, v[4], F_MUL(rx, v[2])), v[5]);
    bh = F_ADD(F_FMA(rx, v[6], F_MUL(ry, v[7])), v[8]);
  } else {
    n0 = F_ADD(F_ADD(F_MUL(rx, v[0]), F_MUL(ry, v[1])), v[2]);
    n1 = (K == 1 || K == 3) ? F_ADD(F_FMA(rx, v[1], F_MUL(ry, v[3])), v[4]) : F_ADD(F_ADD(F_MUL(ry, v[3]), F_MUL(rx, v[1])), v[4]);
    n2 = F_ADD(F_FMA(rx, v[2], F_MUL(ry, v[4])), v[5]);
    bh = F_ADD(F_ADD(F_MUL(rx, v[6]), F_MUL(ry, v[7])), v[8]);
  }
  *AA = F_ADD(F_FMA(rx, n0, F_MUL(ry, n1)), n2);
  *BB = F_ADD(bh, bh);
}

struct RayHit {
  float alpha, test_T;   // the blend weight and the transmittance after it
  float t;               // the stationary point -BB / (2 AA), where the ray meets the Gaussian
  bool free;             // power <= 0 and op * exp(power) <= GOF_ALPHA_MAX: alpha carries a derivative
};

// one ray of pass 1 (forward.cu:931-975): true when the Gaussian is blended on this ray; then *h holds the hit, and tmax has
// been raised to t (forward.cu:965-967)
template <int K>
__device__ __forceinline__ bool ray_step(const float* v, float op, float thr, float rx, float ry, float Tk, float& tmax, RayHit* h) {
  float AA, BB;
  pair_geom_k<K>(v, rx, ry, &AA, &BB);
  {
    // conservative single-precision reject of alpha < 1/255 (both early-outs below return false as well): the exact
    // power is -1/2 (CC - q) with q = fl32(-BB/AA) * BB/4 = BB^2/(4AA) (1 +- 6e-8); qf below carries <= 2.4e-7 (see
    // render_fwd.cu), thr = -ln(255 op) - 2e-3 absorbs the remaining roundings
    const float bh = 0.5f * BB;
    const float qf = bh * bh * gof_rcp_approx(AA);
    const float pw = -0.5f * (v[9] - qf);
    if (fmaf(fabsf(qf), 5e-7f, pw) < thr && fabsf(AA) < 1e30f) return false;
  }
  const float t = F_DIV(-BB, F_ADD(AA, AA));
  if (GOF_T_BEHIND_NEAR(t)) return false;
  const double mv = D_FMA((double)F_DIV(-BB, AA), D_MUL((double)BB, 0.25), (double)v[9]);
  float power = (float)D_MUL(mv, -0.5);
  const bool unclamped = power <= 0.0f;
  if (power > 0.0f) power = 0.0f;
  const float raw = F_MUL(op, F_EXP(power));
  const float al = fminf(raw, GOF_ALPHA_MAX);
  if (al < GOF_ALPHA_MIN) return false;
  const float tt = F_MUL(Tk, F_SUB(1.0f, al));
  if (tt < GOF_T_EPS) return false;
  if (t > tmax) tmax = t;
  *h = RayHit{al, tt, t, unclamped && raw <= GOF_ALPHA_MAX};
  return true;
}

// Pass 1 of one pixel (forward.cu:886-993): the five rays, the contributor list (uint16 ids in my_ids, at most
// GOF_INT_MAX_CONTRIB), and the centre ray's colour, depth and alpha.  k_integrate and k_integrate_backward both run it, so the
// backward's lists are the forward's, bit for bit.  Ends with the CTA in step (every thread calls it once per tile).
struct Pass1 {
  uint2 range;   // the tile's Gaussian list
  float T0, C0, C1, C2, tmax, Aacc;
  uint32_t last_contributor, n_local;
};

// One batch of the tile list into shared memory: the record and the reject threshold of ray_step (pass 1 and the colour walk)
__device__ __forceinline__ void int_load_batch(const IntQuery& q, float4 (*s_rec)[5], uint2 range, int progress, int total) {
  if (progress < total) {
    const uint32_t g = q.point_list[range.x + progress];
    const float4* src = reinterpret_cast<const float4*>(q.splat + g);
    const float4 r2 = __ldg(src + 2);
    s_rec[threadIdx.x][0] = __ldg(src); s_rec[threadIdx.x][1] = __ldg(src + 1);
    s_rec[threadIdx.x][2] = r2; s_rec[threadIdx.x][3] = __ldg(src + 3);
    const float op = r2.z;
    s_rec[threadIdx.x][4].x = (op > 0.f) ? (-logf(255.0f * op) - 2e-3f) : __int_as_float(0x7f800000);
  }
}

// CTOT: also sum the centre ray's blend in double, ctot = (T, C_0, C_1, C_2) with C = sum_j T_j alpha_j c_j (the colour walk's
// totals, DESIGN.md 4.13); the float state is the same either way
template <bool CTOT = false>
__device__ __forceinline__ Pass1 int_pass1(const IntQuery& q, float4 (*s_rec)[5], uint32_t s_base, int tile, const GofWarpBlock& blk,
                                           bool inside, uint16_t* my_ids, double* ctot = nullptr) {
  const int lane = threadIdx.x & 31;
  bool done = !inside;

  // forward.cu:920: ((pixf + offset) - S/2.) / focal, offsets 0 / -0.5 / +0.5
  const float pfx = F_ADD((float)blk.pix_x, 0.5f), pfy = F_ADD((float)blk.pix_y, 0.5f);
  const float rx0 = gof_ray_at(pfx, q.W, q.focal_x), ry0 = gof_ray_at(pfy, q.H, q.focal_y);
  const float rxm = gof_ray_at(F_ADD(pfx, -0.5f), q.W, q.focal_x), rxp = gof_ray_at(F_ADD(pfx, 0.5f), q.W, q.focal_x);
  const float rym = gof_ray_at(F_ADD(pfy, -0.5f), q.H, q.focal_y), ryp = gof_ray_at(F_ADD(pfy, 0.5f), q.H, q.focal_y);

  const uint2 range = q.ranges[tile];
  const int total = (int)(range.y - range.x);
  const int rounds = (total + BATCH - 1) / BATCH;

  float T0 = 1.f, T1 = 1.f, T2 = 1.f, T3 = 1.f, T4 = 1.f;
  float C0 = 0.f, C1 = 0.f, C2 = 0.f, tmax = 0.f, Aacc = 0.f;
  uint32_t last_contributor = 0, n_local = 0;

  for (int i = 0; i < rounds; ++i) {
    __syncthreads();
    int_load_batch(q, s_rec, range, i * BATCH + (int)threadIdx.x, total);
    __syncthreads();
    const int nb = min(BATCH, total - i * BATCH);
#pragma unroll 1
    for (int k = 0; k < BATCH / 32; ++k) {
      if (k * 32 >= nb) break;
      const int idx = k * 32 + lane;
      const float4 qb = s_rec[idx][3];
      // The box holds every pixel at which one of the five rays can pass the alpha test (the half pixel of the corner
      // rays is inside it, added before the rounding to integers), so it is tested against the warp's 8x4 pixels as they
      // are: a Gaussian skipped here would be rejected by all five ray_step calls of all 32 lanes.
      uint32_t m = __ballot_sync(0xffffffffu, idx < nb && gof_box_hits(__float_as_uint(qb.z), __float_as_uint(qb.w), blk.wx0, blk.wy0,
                                                                      blk.wx0 + 7, blk.wy0 + 3));
      while (m) {
        const int j = k * 32 + __ffs(m) - 1;
        m &= m - 1;
        if (done) continue;
        const uint32_t contributor = (uint32_t)(i * BATCH + j + 1);
        const uint32_t row = s_base + (uint32_t)j * 80u;
        const float4 q0 = gof_lds128<0>(row), q1 = gof_lds128<16>(row), q2 = gof_lds128<32>(row);
        const float v[10] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y};
        const float op = q2.z;
        const float thr = gof_lds32<64>(row);
        RayHit h;
        bool used = false;
        if (ray_step<0>(v, op, thr, rx0, ry0, T0, tmax, &h)) {
          const float2 q3 = gof_lds64<48>(row);
          C0 = F_FMA(T0, F_MUL(h.alpha, q2.w), C0);
          C1 = F_FMA(T0, F_MUL(h.alpha, q3.x), C1);
          C2 = F_FMA(T0, F_MUL(h.alpha, q3.y), C2);
          Aacc = F_FMA(T0, h.alpha, Aacc);
          if constexpr (CTOT) {
            const double w = ctot[0] * (double)h.alpha;
            ctot[1] += w * (double)q2.w; ctot[2] += w * (double)q3.x; ctot[3] += w * (double)q3.y;
            ctot[0] *= 1.0 - (double)h.alpha;
          }
          T0 = h.test_T; used = true;
        }
        if (ray_step<1>(v, op, thr, rxm, rym, T1, tmax, &h)) { T1 = h.test_T; used = true; }
        if (ray_step<2>(v, op, thr, rxp, rym, T2, tmax, &h)) { T2 = h.test_T; used = true; }
        if (ray_step<3>(v, op, thr, rxm, ryp, T3, tmax, &h)) { T3 = h.test_T; used = true; }
        if (ray_step<4>(v, op, thr, rxp, ryp, T4, tmax, &h)) { T4 = h.test_T; used = true; }
        if (used) {
          last_contributor = contributor;
          my_ids[n_local] = (uint16_t)contributor;    // uint16 truncation as in forward.cu:983
          n_local += 1;
          if (n_local >= GOF_INT_MAX_CONTRIB) done = true;   // forward.cu:986-990
        }
      }
    }
  }
  return Pass1{range, T0, C0, C1, C2, tmax, Aacc, last_contributor, n_local};
}

// The quadric v[10] and the opacity of record g, read from global memory (pass 2 and the backward's walks)
__device__ __forceinline__ float load_rec(const GofSplat* __restrict__ splat, uint32_t g, float* v) {
  const float4* src = reinterpret_cast<const float4*>(splat + g);
  const float4 q0 = __ldg(src), q1 = __ldg(src + 1), q2 = __ldg(src + 2);
  v[0] = q0.x; v[1] = q0.y; v[2] = q0.z; v[3] = q0.w; v[4] = q1.x; v[5] = q1.y; v[6] = q1.z; v[7] = q1.w; v[8] = q2.x; v[9] = q2.y;
  return q2.z;
}

// One pair of pass 2 and of the backward's walks 1 and 2 (forward.cu:1158-1190): the float alpha and what its derivative needs
struct PairEval {
  float al;       // alpha after the clamp; < GOF_ALPHA_MIN: rejected
  bool free;      // op * exp(power) <= GOF_ALPHA_MAX: alpha carries a derivative
  bool clamped;   // t was clamped to the point's depth
  float t;
};
__device__ __forceinline__ PairEval pair_eval(const float* v, float op, float rx, float ry, float ray_depth) {
  const GofPair p = gof_pair_geom(v, rx, ry);
  PairEval e;
  float t = F_DIV(-p.BB, F_ADD(p.AA, p.AA));
  e.clamped = t > ray_depth;
  if (e.clamped) t = ray_depth;
  const float power = F_MUL(F_ADD(v[9], F_FMA(p.BB, t, F_MUL(t, F_MUL(p.AA, t)))), -0.5f);
  const float raw = F_MUL(op, F_EXP(power));
  e.al = fminf(raw, GOF_ALPHA_MAX);
  e.free = raw <= GOF_ALPHA_MAX;
  e.t = t;
  return e;
}

// Walk 1's step for one pair that passed the alpha reject (k_integrate_backward, and pass 2 of k_integrate<true, *, true>): T and
// sum_j alpha_j / (1 - alpha_j) * d power_j / d(rx, ry, depth) over the free pairs
__device__ __forceinline__ void walk1_step(const float* v, const PairEval& e, float rx, float ry, double& T, double& grx, double& gry,
                                           double& gdep) {
  const double om = 1.0 - (double)e.al;
  T *= om;
  if (!e.free) return;
  const double w = (double)e.al / om, t = e.t;
  // power = -1/2 (AA t^2 + BB t + CC): AA = r^T Sigma r, BB = 2 b.r, r = (rx, ry, 1)
  const double n0 = (double)v[0] * rx + (double)v[1] * ry + v[2];
  const double n1 = (double)v[1] * rx + (double)v[3] * ry + v[4];
  grx -= w * (t * t * n0 + t * v[6]);
  gry -= w * (t * t * n1 + t * v[7]);
  if (e.clamped) {
    const double AA = ((double)v[0] * rx + 2.0 * v[1] * ry + 2.0 * v[2]) * rx + ((double)v[3] * ry + 2.0 * v[4]) * ry + v[5];
    const double bh = (double)v[6] * rx + (double)v[7] * ry + v[8];
    gdep -= w * (AA * t + bh);
  }
}

// Walk 1's totals (T, grx, gry, gdep) of point id -> dL/dA * d A / d point in world space, rounded to float once into out[3].
// rx = tx / (tz + 1e-7), ry = ty / (tz + 1e-7), depth = tz; (tx, ty, tz) = the view matrix applied to the point
__device__ __forceinline__ void walk1_point_grad(const float* points3D, const float* vm_, uint32_t id, float dLdA, double T, double grx,
                                                 double gry, double gdep, float* out) {
  const double px = points3D[3 * (size_t)id], py = points3D[3 * (size_t)id + 1], pz = points3D[3 * (size_t)id + 2];
  double vm[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) vm[k] = (double)__ldg(vm_ + k);
  const double tx = vm[0] * px + vm[4] * py + vm[8] * pz + vm[12];
  const double ty = vm[1] * px + vm[5] * py + vm[9] * pz + vm[13];
  const double tz = vm[2] * px + vm[6] * py + vm[10] * pz + vm[14];
  const double s = (double)dLdA * T, den = tz + 1e-7;
  const double drx = s * grx, dry = s * gry;
  const double dtx = drx / den, dty = dry / den, dtz = s * gdep - (drx * tx + dry * ty) / (den * den);
#pragma unroll
  for (int i = 0; i < 3; ++i) out[i] = (float)(vm[4 * i] * dtx + vm[4 * i + 1] * dty + vm[4 * i + 2] * dtz);
}

// k_integrate<true, *, true> carries walk 1's four doubles: two CTAs per SM, and a grid of that many (see the launcher)
constexpr int INT_GRAD_CTAS_PER_SM = 2;

// MIN_UPDATE: the query of one view of the multi-view opacity field (DESIGN.md 4.12).  Each point that projects folds its alpha
// into alpha_min / argmin with the strict `<` of evaluate_alpha; views run in stream order and a point is one thread of one call,
// so no atomics are needed.  Nothing else is written: no image, no point colour, no pixel state.  MIN_COLOR (DESIGN.md 4.13):
// the same update also writes the point's colour of this view, C + T*bg as k_integrate<false> forms it, to color_min.  MIN_GRAD
// (DESIGN.md 4.14): pass 2 also runs walk 1 beside the float alpha, over the same pairs, and the update writes walk 1's
// d alpha_integrated / d point (dL/dA = 1) to grad_min.
template <bool MIN_UPDATE, bool MIN_COLOR = false, bool MIN_GRAD = false>
__global__ void __launch_bounds__(GOF_BLOCK_SIZE, MIN_GRAD ? INT_GRAD_CTAS_PER_SM : 3) k_integrate(const IntArgs a) {
  __shared__ float4 s_rec[BATCH][5];   // 80-byte rows: GofSplat | (thr, -, -, -), see render_fwd.cu
  __shared__ uint32_t s_cnt[256];      // contributors recorded per pixel (slot = thread of that pixel)
  __shared__ float s_col[256][3];      // pixel colour (C + T*bg)
  __shared__ uint32_t s_proj[256];     // points that fell into each pixel

  const uint32_t s_base = gof_smem_base(&s_rec[0][0]);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint16_t* slab = a.ids + (size_t)blockIdx.x * 256 * GOF_INT_MAX_CONTRIB;
  uint16_t* my_ids = slab + (size_t)threadIdx.x * GOF_INT_MAX_CONTRIB;
  const size_t HW = (size_t)a.H * a.W;

  for (int tile = blockIdx.x; tile < a.tiles; tile += gridDim.x) {
    const int tile_x = tile % a.grid_x, tile_y = tile / a.grid_x;
    const GofWarpBlock blk = gof_warp_block(tile_x, tile_y, warp, lane);
    const bool inside = blk.pix_x < (uint32_t)a.W && blk.pix_y < (uint32_t)a.H;

    // ---------------- pass 1 (forward.cu:886-993) ----------------
    const Pass1 p1 = int_pass1(a, s_rec, s_base, tile, blk, inside, my_ids);
    const uint2 range = p1.range;
    const float T0 = p1.T0, C0 = p1.C0, C1 = p1.C1, C2 = p1.C2, tmax = p1.tmax, Aacc = p1.Aacc;
    const uint32_t last_contributor = p1.last_contributor, n_local = p1.n_local;

    // forward.cu:997-1008
    if constexpr (!MIN_UPDATE) {
      const size_t slot = (size_t)tile * 256 + threadIdx.x;
      a.final_T[slot] = T0;
      a.ncontrib[slot] = last_contributor;
      a.ncontrib[(size_t)a.tiles * 256 + slot] = n_local;
    }
    float col0 = 0.f, col1 = 0.f, col2 = 0.f;   // the pixel colour C + T*bg
    if constexpr (!MIN_UPDATE || MIN_COLOR) {
      col0 = F_FMA(T0, a.bg[0], C0); col1 = F_FMA(T0, a.bg[1], C1); col2 = F_FMA(T0, a.bg[2], C2);
      s_col[threadIdx.x][0] = col0; s_col[threadIdx.x][1] = col1; s_col[threadIdx.x][2] = col2;
    }
    s_cnt[threadIdx.x] = n_local;
    if constexpr (!MIN_UPDATE) s_proj[threadIdx.x] = 0u;
    __threadfence_block();
    __syncthreads();

    // ---------------- pass 2 (forward.cu:1116-1210), one thread per query point ----------------
    const uint2 pr = a.pranges[tile];
    for (uint32_t base = pr.x; base < pr.y; base += BATCH) {
      const uint32_t q = base + threadIdx.x;
      if (q < pr.y) {
        const uint32_t id = a.pt_list[q];
        const float2 xy = a.pt_xy[id];
        const float ray_depth = a.pt_depth[id];
        const int pslot = gof_point_slot(xy.x, xy.y, tile_x, tile_y);
        if constexpr (!MIN_UPDATE) atomicAdd(&s_proj[pslot], 1u);
        const float rx = gof_point_ray(xy.x, a.W, a.focal_x), ry = gof_point_ray(xy.y, a.H, a.focal_y);
        const uint32_t cnt = s_cnt[pslot];
        const uint16_t* ids = slab + (size_t)pslot * GOF_INT_MAX_CONTRIB;
        float point_alpha = 0.f, point_T = 1.f;
        double T = 1.0, grx = 0.0, gry = 0.0, gdep = 0.0;   // walk 1 (MIN_GRAD)
        uint32_t prev = 0;
        for (uint32_t c = 0; c < cnt; ++c) {
          const uint32_t cid = (uint32_t)ids[c];
          if (cid <= prev) break;     // a wrapped uint16 id can never be matched again by the running index (:1141-1149)
          prev = cid;
          float v[10];
          const float op = load_rec(a.splat, a.point_list[range.x + cid - 1], v);
          const PairEval e = pair_eval(v, op, rx, ry, ray_depth);
          const float al = e.al;
          if (al < GOF_ALPHA_MIN) continue;
          point_alpha = F_FMA(al, point_T, point_alpha);
          point_T = F_MUL(point_T, F_SUB(1.0f, al));
          if constexpr (MIN_GRAD) walk1_step(v, e, rx, ry, T, grx, gry, gdep);
        }
        if constexpr (MIN_UPDATE) {
          if (point_alpha < a.alpha_min[id]) {   // evaluate_alpha's update, in view order
            a.alpha_min[id] = point_alpha;
            a.argmin[id] = a.view;
            if constexpr (MIN_COLOR) {
              a.color_min[3 * (size_t)id + 0] = s_col[pslot][0];
              a.color_min[3 * (size_t)id + 1] = s_col[pslot][1];
              a.color_min[3 * (size_t)id + 2] = s_col[pslot][2];
            }
            if constexpr (MIN_GRAD) walk1_point_grad(a.points3D, a.vm, id, 1.f, T, grx, gry, gdep, a.grad_min + 3 * (size_t)id);
          }
        } else {
          a.out_alpha[id] = point_alpha;
          a.out_color_int[3 * (size_t)id + 0] = s_col[pslot][0];
          a.out_color_int[3 * (size_t)id + 1] = s_col[pslot][1];
          a.out_color_int[3 * (size_t)id + 2] = s_col[pslot][2];
        }
      }
    }
    __syncthreads();
    if (!MIN_UPDATE && inside) {
      const size_t pid = (size_t)blk.pix_y * a.W + blk.pix_x;
      a.out_color[0 * HW + pid] = col0;
      a.out_color[1 * HW + pid] = col1;
      a.out_color[2 * HW + pid] = col2;
      a.out_color[6 * HW + pid] = tmax;
      a.out_color[7 * HW + pid] = Aacc;
      a.out_color[8 * HW + pid] = (float)s_proj[threadIdx.x];   // forward.cu:1216
    }
    __syncthreads();
  }
}

// ---------------- backward of the query (DESIGN.md 4.11) ----------------
// A = sum_j alpha_j T_j over the point's contributors is 1 - prod_j (1 - alpha_j), so with the list, the rejects and the clamps
// held fixed dA/dalpha_j = T / (1 - alpha_j), T = prod_i (1 - alpha_i) the point's final transmittance.  Walk 1 forms T and the
// point's own gradient; walk 2 (which needs T) hands each pair's dL/dview2gaussian to its Gaussian's accumulator row.
struct IntBwdArgs : IntQuery {   // ids: the forward's slab, rewritten
  const float* points3D;
  const float* vm;
  const float* dL_dalpha;   // [PN]
  double* grad_acc;         // [P][16]: dL_dview2gaussian[10] of every pair lands in 0..9 (zeroed by the launcher)
  float* dL_dpoints3D;      // [PN][3] or NULL (zeroed by the launcher: points that do not project keep the zeros)
};
// k_integrate_backward<true> (DESIGN.md 4.13); dL_dalpha may then be NULL (no alpha walk).  A type of its own, so that the
// alpha-only instantiation keeps its parameter block.
struct IntBwdColorArgs : IntBwdArgs {
  const float* dL_dcolor;   // [PN][3], the gradient of color_integrated: dL/dcolor lands in rows 10..12 of grad_acc
  const float* bg;          // [3]
};

// A pair's dL/dview2gaussian rows from f = dL/dCC, at depth t on the ray (x, y, 1): power = -1/2 (AA t^2 + BB t + CC) with t held
// fixed, AA = r^T Sigma r and BB = 2 b.r, the off-diagonal entries of Sigma counted twice (walk 2 and the colour walk)
__device__ __forceinline__ void v2g_rows(double f, double t, double x, double y, double* d) {
  const double ft2 = f * t * t, ft = f * t;
  d[0] = ft2 * x * x; d[1] = 2.0 * ft2 * x * y; d[2] = 2.0 * ft2 * x;
  d[3] = ft2 * y * y; d[4] = 2.0 * ft2 * y; d[5] = ft2;
  d[6] = 2.0 * ft * x; d[7] = 2.0 * ft * y; d[8] = 2.0 * ft; d[9] = f;
}

// 94 registers: two CTAs per SM (the query's three do not fit), and the grid is that many, so no CTA waits for a second wave
constexpr int INT_BWD_CTAS_PER_SM = 2;

// The colour walk of one tile (DESIGN.md 4.13).  color_integrated of a point is its pixel's C + T*bg on the centre ray, so
// dL/dC of a pixel is the sum of dL/dcolor_integrated over its points.  The walk replays pass 1's centre ray over the tile list
// -- the same batches, the same box test, the same ray_step<0> with the same float T -- up to the pixel's last contributor (the
// forward's cap ends every ray there), so it visits exactly the Gaussians the forward blended, with their true list positions
// (the recorded uint16 ids wrap past 65 535).  With T_j, the suffix S_j = tot - sum_{i<=j} T_i alpha_i c_i (tot from pass 1, in
// double):  dL/dc_j = T_j alpha_j dL/dC  and  dL/dalpha_j = dL/dC . (T_j c_j - S_j / (1 - alpha_j)).  A warp visits its candidate
// Gaussians in step, so each pair's 13 rows are summed over the warp and sent by one lane.
__device__ __forceinline__ void int_color_walk(const IntBwdColorArgs& a, float4 (*s_rec)[5], uint32_t s_base, uint2 range,
                                               const GofWarpBlock& blk, const double* dC, const double* tot, uint32_t last,
                                               uint32_t* s_last) {
  const int lane = threadIdx.x & 31;
  const bool want = last > 0 && (dC[0] != 0.0 || dC[1] != 0.0 || dC[2] != 0.0);
  if (threadIdx.x == 0) *s_last = 0u;
  __syncthreads();
  if (want) atomicMax(s_last, last);
  __syncthreads();
  const int total = (int)*s_last;   // no wanting pixel of the CTA blended anything past it
  if (total == 0) return;           // uniform
  const bool warp_wants = __any_sync(0xffffffffu, want);
  const uint32_t warp_last = __reduce_max_sync(0xffffffffu, want ? last : 0u);

  const float rx0 = gof_ray(blk.pix_x, a.W, a.focal_x), ry0 = gof_ray(blk.pix_y, a.H, a.focal_y);
  float T0 = 1.f, tmax = 0.f;
  double T = 1.0, pre0 = 0.0, pre1 = 0.0, pre2 = 0.0;
  const int rounds = (total + BATCH - 1) / BATCH;
  for (int i = 0; i < rounds; ++i) {
    __syncthreads();
    int_load_batch(a, s_rec, range, i * BATCH + (int)threadIdx.x, total);
    __syncthreads();
    if (!warp_wants) continue;
    const int nb = min(BATCH, total - i * BATCH);
#pragma unroll 1
    for (int k = 0; k < BATCH / 32; ++k) {
      if (k * 32 >= nb || (uint32_t)(i * BATCH + k * 32) >= warp_last) break;
      const int idx = k * 32 + lane;
      const float4 qb = s_rec[idx][3];
      uint32_t m = __ballot_sync(0xffffffffu, idx < nb && gof_box_hits(__float_as_uint(qb.z), __float_as_uint(qb.w), blk.wx0, blk.wy0,
                                                                      blk.wx0 + 7, blk.wy0 + 3));
      while (m) {
        const int j = k * 32 + __ffs(m) - 1;
        m &= m - 1;
        const uint32_t contributor = (uint32_t)(i * BATCH + j + 1);
        double d[13];
#pragma unroll
        for (int r = 0; r < 13; ++r) d[r] = 0.0;
        bool has = false;
        if (want && contributor <= last) {
          const uint32_t row = s_base + (uint32_t)j * 80u;
          const float4 q0 = gof_lds128<0>(row), q1 = gof_lds128<16>(row), q2 = gof_lds128<32>(row);
          const float v[10] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y};
          const float op = q2.z;
          RayHit h;
          if (ray_step<0>(v, op, gof_lds32<64>(row), rx0, ry0, T0, tmax, &h)) {
            T0 = h.test_T; has = true;
            const float2 q3 = gof_lds64<48>(row);
            const double c[3] = {(double)q2.w, (double)q3.x, (double)q3.y};
            const double alpha = h.alpha, w = T * alpha, om = 1.0 - alpha;
            pre0 += w * c[0]; pre1 += w * c[1]; pre2 += w * c[2];
            const double S[3] = {tot[1] - pre0, tot[2] - pre1, tot[3] - pre2};
            double dLdal = 0.0;
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
              d[10 + ch] = w * dC[ch];
              dLdal += dC[ch] * (T * c[ch] - S[ch] / om);
            }
            T *= om;
            // power = -1/2 (CC - BB^2 / (4 AA)) is stationary in t = -BB / (2 AA), so its derivative is -1/2 (t^2, t, 1)
            if (h.free) v2g_rows(-0.5 * dLdal * alpha, h.t, rx0, ry0, d);
          }
        }
        const uint32_t with = __ballot_sync(0xffffffffu, has);
        if (!with) continue;
        const int src = __ffs(with) - 1;
        if (__popc(with) > 1) {
#pragma unroll
          for (int off = 16; off > 0; off >>= 1)
#pragma unroll
            for (int r = 0; r < 13; ++r) d[r] += __shfl_xor_sync(0xffffffffu, d[r], off);
        }
        if (lane == src) {
          double* acc = a.grad_acc + (size_t)a.point_list[range.x + contributor - 1] * 16;
#pragma unroll
          for (int r = 0; r < 13; ++r) atomicAdd(acc + r, d[r]);
        }
      }
    }
  }
}

template <bool COLOR>
__global__ void __launch_bounds__(GOF_BLOCK_SIZE, INT_BWD_CTAS_PER_SM)
    k_integrate_backward(const std::conditional_t<COLOR, IntBwdColorArgs, IntBwdArgs> a) {
  __shared__ float4 s_rec[BATCH][5];
  __shared__ uint32_t s_cnt[256];

  const uint32_t s_base = gof_smem_base(&s_rec[0][0]);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint16_t* slab = a.ids + (size_t)blockIdx.x * 256 * GOF_INT_MAX_CONTRIB;
  uint16_t* my_ids = slab + (size_t)threadIdx.x * GOF_INT_MAX_CONTRIB;

  for (int tile = blockIdx.x; tile < a.tiles; tile += gridDim.x) {
    const uint2 pr = a.pranges[tile];
    if (pr.x == pr.y) continue;   // uniform over the CTA: no point here, no list needed
    const int tile_x = tile % a.grid_x, tile_y = tile / a.grid_x;
    const GofWarpBlock blk = gof_warp_block(tile_x, tile_y, warp, lane);
    const bool inside = blk.pix_x < (uint32_t)a.W && blk.pix_y < (uint32_t)a.H;

    double tot[4] = {1.0, 0.0, 0.0, 0.0};
    const Pass1 p1 = int_pass1<COLOR>(a, s_rec, s_base, tile, blk, inside, my_ids, COLOR ? tot : nullptr);
    const uint2 range = p1.range;
    s_cnt[threadIdx.x] = p1.n_local;
    __threadfence_block();
    __syncthreads();

    for (uint32_t base = pr.x; base < (COLOR && a.dL_dalpha == nullptr ? pr.x : pr.y); base += BATCH) {
      const uint32_t q = base + threadIdx.x;
      const bool valid = q < pr.y;
      uint32_t id = 0;
      float rx = 0.f, ry = 0.f, ray_depth = 0.f;
      int pslot = 256 + lane;   // lanes without a point form runs of their own
      if (valid) {
        id = a.pt_list[q];
        const float2 xy = a.pt_xy[id];
        ray_depth = a.pt_depth[id];
        pslot = gof_point_slot(xy.x, xy.y, tile_x, tile_y);
        rx = gof_point_ray(xy.x, a.W, a.focal_x); ry = gof_point_ray(xy.y, a.H, a.focal_y);
      }
      const float dLdA = valid ? a.dL_dalpha[id] : 0.f;
      const uint16_t* ids = slab + (size_t)(pslot & 255) * GOF_INT_MAX_CONTRIB;
      const uint32_t cnt = valid ? s_cnt[pslot] : 0u;

      // walk 1: T and sum_j alpha_j / (1 - alpha_j) * d power_j / d(rx, ry, depth) over the free pairs
      double T = 1.0, grx = 0.0, gry = 0.0, gdep = 0.0;
      uint32_t n_eff = 0, prev = 0;
      for (uint32_t c = 0; c < cnt; ++c) {
        const uint32_t cid = (uint32_t)ids[c];
        if (cid <= prev) break;   // a wrapped uint16 id ends the list, as in the forward
        prev = cid;
        n_eff = c + 1;
        float v[10];
        const float op = load_rec(a.splat, a.point_list[range.x + cid - 1], v);
        const PairEval e = pair_eval(v, op, rx, ry, ray_depth);
        if (e.al < GOF_ALPHA_MIN) continue;
        walk1_step(v, e, rx, ry, T, grx, gry, gdep);
      }
      if (valid && a.dL_dpoints3D != nullptr)
        walk1_point_grad(a.points3D, a.vm, id, dLdA, T, grx, gry, gdep, a.dL_dpoints3D + 3 * (size_t)id);

      // walk 2: pair j of the point adds dL/dA * T / (1 - alpha_j) * alpha_j * d power_j / d view2gaussian to Gaussian j.  Lanes of
      // one pixel (neighbours: the points are sorted by pixel) walk the same list in step, so each run of them sums its rows with
      // shuffles and its first lane issues the atomics.
      const uint32_t nxt = __shfl_down_sync(0xffffffffu, (uint32_t)pslot, 1);
      const uint32_t prv = __shfl_up_sync(0xffffffffu, (uint32_t)pslot, 1);
      const uint32_t ends = __ballot_sync(0xffffffffu, lane == 31 || nxt != (uint32_t)pslot);
      const bool head = lane == 0 || prv != (uint32_t)pslot;
      const int run_end = __ffs(ends & (0xffffffffu << lane)) - 1;
      const int longest = __reduce_max_sync(0xffffffffu, (uint32_t)(run_end - lane + 1));
      const uint32_t steps = __reduce_max_sync(0xffffffffu, dLdA != 0.f ? n_eff : 0u);
      const double s = (double)dLdA * T;
      for (uint32_t c = 0; c < steps; ++c) {
        double d[10];
#pragma unroll
        for (int k = 0; k < 10; ++k) d[k] = 0.0;
        uint32_t g = 0;
        bool has = false;
        if (c < n_eff) {
          g = a.point_list[range.x + (uint32_t)ids[c] - 1];
          if (dLdA != 0.f) {
            float v[10];
            const float op = load_rec(a.splat, g, v);
            const PairEval e = pair_eval(v, op, rx, ry, ray_depth);
            if (e.al >= GOF_ALPHA_MIN && e.free) {
              has = true;
              v2g_rows(-0.5 * s * (double)e.al / (1.0 - (double)e.al), e.t, rx, ry, d);
            }
          }
        }
        const uint32_t with = __ballot_sync(0xffffffffu, has);
        if (!with) continue;
        for (int off = 1; off < longest; off <<= 1) {
#pragma unroll
          for (int k = 0; k < 10; ++k) {
            const double o = __shfl_down_sync(0xffffffffu, d[k], off);
            if (lane + off <= run_end) d[k] += o;
          }
        }
        const uint32_t mine = (run_end == 31 ? 0xffffffffu : ((1u << (run_end + 1)) - 1u)) & (0xffffffffu << lane);
        if (head && (with & mine)) {
          double* row = a.grad_acc + (size_t)g * 16;
#pragma unroll
          for (int k = 0; k < 10; ++k) atomicAdd(row + k, d[k]);
        }
      }
    }
    if constexpr (COLOR) {
      // dL/dC of each pixel: its points' dL/dcolor_integrated summed in double in the point sort's order (a pixel's points are
      // neighbours there, a run may cross batches), by the first point of the run in each batch
      __shared__ double s_dC[256][3];
      __shared__ uint32_t s_slot[BATCH + 1];
      __shared__ float s_g[BATCH][3];
      __shared__ uint32_t s_last;
      s_dC[threadIdx.x][0] = s_dC[threadIdx.x][1] = s_dC[threadIdx.x][2] = 0.0;
      for (uint32_t base = pr.x; base < pr.y; base += BATCH) {
        const uint32_t q = base + threadIdx.x;
        uint32_t pslot = 256;
        float g[3] = {0.f, 0.f, 0.f};
        if (q < pr.y) {
          const uint32_t id = a.pt_list[q];
          const float2 xy = a.pt_xy[id];
          pslot = gof_point_slot(xy.x, xy.y, tile_x, tile_y);
#pragma unroll
          for (int ch = 0; ch < 3; ++ch) g[ch] = a.dL_dcolor[3 * (size_t)id + ch];
        }
        __syncthreads();   // s_slot / s_g of the previous batch are read
        s_slot[threadIdx.x] = pslot;
        s_g[threadIdx.x][0] = g[0]; s_g[threadIdx.x][1] = g[1]; s_g[threadIdx.x][2] = g[2];
        if (threadIdx.x == 0) s_slot[BATCH] = 256;
        __syncthreads();
        if (pslot < 256 && (threadIdx.x == 0 || s_slot[threadIdx.x - 1] != pslot)) {
          double acc[3] = {s_dC[pslot][0], s_dC[pslot][1], s_dC[pslot][2]};
          for (int k = threadIdx.x; s_slot[k] == pslot; ++k)
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) acc[ch] += (double)s_g[k][ch];
          s_dC[pslot][0] = acc[0]; s_dC[pslot][1] = acc[1]; s_dC[pslot][2] = acc[2];
        }
      }
      __syncthreads();
      const double dC[3] = {s_dC[threadIdx.x][0], s_dC[threadIdx.x][1], s_dC[threadIdx.x][2]};
      tot[1] += tot[0] * (double)a.bg[0]; tot[2] += tot[0] * (double)a.bg[1]; tot[3] += tot[0] * (double)a.bg[2];
      int_color_walk(a, s_rec, s_base, range, blk, dC, tot, p1.last_contributor, &s_last);
    }
    __syncthreads();
  }
}

// The query's state in the caller's buffers.  The point sort of gof_launch_integrate (PN > 0 pairs over pt_key_bits) leaves
// the sorted ids in val_a or val_b by the parity of its passes.
IntQuery int_query(const GofView& v, const GofSplat* splat, const uint32_t* point_list, const uint2* ranges, const char* pts,
                   const GofPointLayout& PL, char* pbin, const GofPointBinLayout& PBL) {
  IntQuery q;
  q.W = v.W; q.H = v.H; q.grid_x = v.grid_x; q.tiles = v.tiles; q.focal_x = v.focal_x; q.focal_y = v.focal_y;
  q.ranges = ranges; q.point_list = point_list; q.splat = splat;
  q.pranges = reinterpret_cast<const uint2*>(pbin + PBL.pranges);
  q.pt_list = reinterpret_cast<const uint32_t*>(pbin + (gof_radix_result_in_b(pt_key_bits(v.tiles)) ? PBL.val_b : PBL.val_a));
  q.pt_xy = reinterpret_cast<const float2*>(pts + PL.xy); q.pt_depth = reinterpret_cast<const float*>(pts + PL.depth);
  q.ids = reinterpret_cast<uint16_t*>(pbin + PBL.ids);
  return q;
}

}  // namespace

int gof_launch_integrate(const gof_scene_t* s, const GofView& v, int PN, const float* points3D, const GofSplat* splat,
                         const uint32_t* point_list, const uint2* ranges, char* img, char* pts, char* pbin,
                         const gof_integrate_out_t& out, cudaStream_t st) {
  const bool debug = s->debug != 0;
  const GofImageLayout IL = gof_image_layout(s->width, s->height);
  const GofPointLayout PL = gof_point_layout((size_t)PN);
  const GofPointBinLayout PBL = gof_point_bin_layout((size_t)PN, v.tiles, gof_sm_count());
  PtArgs pa{};
  pa.PN = PN; pa.W = v.W; pa.H = v.H; pa.grid_x = v.grid_x; pa.grid_y = v.grid_y; pa.tiles = v.tiles;
  pa.focal_x = v.focal_x; pa.focal_y = v.focal_y; pa.points3D = points3D; pa.vm = s->viewmatrix;
  pa.xy = reinterpret_cast<float2*>(pts + PL.xy); pa.depth = reinterpret_cast<float*>(pts + PL.depth);
  uint32_t* ka = reinterpret_cast<uint32_t*>(pbin + PBL.key_a);
  uint32_t* kb = reinterpret_cast<uint32_t*>(pbin + PBL.key_b);
  uint32_t* va = reinterpret_cast<uint32_t*>(pbin + PBL.val_a);
  uint32_t* vb = reinterpret_cast<uint32_t*>(pbin + PBL.val_b);
  pa.key = ka; pa.val = va;
  GOF_LAUNCH("preprocess_points", st, k_preprocess_points<<<(PN + 255) / 256, 256, 0, st>>>(pa));
  GOF_LAUNCH_CHECK(debug, st);
  int rc = gof_sort_points_by_tile((size_t)PN, pt_key_bits(v.tiles), PT_KEY_SHIFT, ka, kb, va, vb,
                                   reinterpret_cast<uint32_t*>(pbin + PBL.hist), reinterpret_cast<uint2*>(pbin + PBL.pranges),
                                   v.tiles, debug, st);
  if (rc != GOF_OK) return rc;

  IntArgs a{};
  static_cast<IntQuery&>(a) = int_query(v, splat, point_list, ranges, pts, PL, pbin, PBL);
  a.bg = s->background;
  a.final_T = reinterpret_cast<float*>(img + IL.accum);
  a.ncontrib = reinterpret_cast<uint32_t*>(img + IL.ncontrib);
  a.out_color = out.out_color; a.out_alpha = out.out_alpha_integrated; a.out_color_int = out.out_color_integrated;
  if (out.alpha_min) {
    a.alpha_min = out.alpha_min; a.argmin = out.argmin; a.view = out.view; a.color_min = out.color_min;
    a.grad_min = out.grad_min; a.points3D = points3D; a.vm = s->viewmatrix;
    // persistent CTAs stride over the tiles, each with the slab of its blockIdx.x (PBL.nblk slabs exist)
    const int grad_grid = std::min(PBL.nblk, INT_GRAD_CTAS_PER_SM * gof_sm_count());
    if (out.grad_min && out.color_min)
      GOF_LAUNCH("integrate_min_color_grad", st, k_integrate<true, true, true><<<grad_grid, GOF_BLOCK_SIZE, 0, st>>>(a));
    else if (out.grad_min)
      GOF_LAUNCH("integrate_min_grad", st, k_integrate<true, false, true><<<grad_grid, GOF_BLOCK_SIZE, 0, st>>>(a));
    else if (out.color_min)
      GOF_LAUNCH("integrate_min_color", st, k_integrate<true, true><<<PBL.nblk, GOF_BLOCK_SIZE, 0, st>>>(a));
    else
      GOF_LAUNCH("integrate_min", st, k_integrate<true><<<PBL.nblk, GOF_BLOCK_SIZE, 0, st>>>(a));
  } else {
    GOF_LAUNCH("integrate", st, k_integrate<false><<<PBL.nblk, GOF_BLOCK_SIZE, 0, st>>>(a));
  }
  GOF_LAUNCH_CHECK(debug, st);
  return GOF_OK;
}

size_t gof_integrate_backward_scratch(int P) { return P > 0 ? 2 * gof_align_up((size_t)P * 12, 256) : 0; }

int gof_launch_integrate_backward(const gof_scene_t* s, const GofView& v, int PN, const float* points3D, const int* radii,
                                  char* geom, const GofGeomLayout& GL, const uint32_t* point_list, const uint2* ranges, const char* pts,
                                  char* pbin, const float* dL_dalpha, const float* dL_dcolor_int, float* dL_dpoints3D,
                                  const gof_backward_out_t& o, cudaStream_t st) {
  const bool debug = s->debug != 0;
  const GofPointBinLayout PBL = gof_point_bin_layout((size_t)PN, v.tiles, gof_sm_count());
  IntBwdColorArgs a{};
  static_cast<IntQuery&>(a) = int_query(v, reinterpret_cast<const GofSplat*>(geom + GL.splat), point_list, ranges, pts,
                                        gof_point_layout((size_t)PN), pbin, PBL);
  a.points3D = points3D; a.vm = s->viewmatrix; a.dL_dalpha = dL_dalpha;
  a.grad_acc = reinterpret_cast<double*>(geom + GL.grad_acc);
  a.dL_dpoints3D = dL_dpoints3D;
  a.dL_dcolor = dL_dcolor_int; a.bg = s->background;
  GOF_CUDA_OK(cudaMemsetAsync(a.grad_acc, 0, (size_t)s->P * 128, st));
  if (dL_dpoints3D) GOF_CUDA_OK(cudaMemsetAsync(dL_dpoints3D, 0, (size_t)PN * 12, st));
  // persistent CTAs: each strides over the tiles and uses the slab of its blockIdx.x (PBL.nblk slabs exist)
  const int grid = std::min(PBL.nblk, INT_BWD_CTAS_PER_SM * gof_sm_count());
  if (dL_dcolor_int)
    GOF_LAUNCH("integrate_bwd_color", st, k_integrate_backward<true><<<grid, GOF_BLOCK_SIZE, 0, st>>>(a));
  else
    GOF_LAUNCH("integrate_bwd", st, k_integrate_backward<false><<<grid, GOF_BLOCK_SIZE, 0, st>>>(static_cast<const IntBwdArgs&>(a)));
  GOF_LAUNCH_CHECK(debug, st);
  // the accumulator rows -> the Gaussian parameters, exactly as after the blend backward.  dL_dmean2D (zero rows) lands in the
  // scratch.  Without o.dL_dcolor (alpha mode) the scene goes in without SHs, and dL_dcolor lands in the scratch too; with it,
  // rows 10..12 go through the SH (or colors_precomp) backward as after the blend.
  gof_scene_t sg = *s;
  gof_backward_out_t po = o;
  po.dL_dmean2D = reinterpret_cast<float*>(static_cast<char*>(o.scratch) + gof_align_up((size_t)s->P * 12, 256));
  if (!o.dL_dcolor) { sg.shs = nullptr; po.dL_dcolor = static_cast<float*>(o.scratch); po.dL_dsh = nullptr; }
  return gof_launch_preprocess_backward(&sg, geom, GL, radii, po, st);
}
