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

#include "gof_common.cuh"
#include "gof_math.cuh"

namespace {

constexpr int PT_KEY_SHIFT = 8;   // point key = tile << 8 | pixel slot inside the tile (points of one pixel become neighbours)

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
      // the thread slot of the pixel the point falls in (same mapping as k_integrate's pass 2): sorting on it makes the points
      // of one pixel -- which replay the SAME contributor list -- neighbours, so a warp's record gathers coincide
      int lx = gof_f2i_rz(x) - cx * 16, ly = gof_f2i_rz(y) - cy * 16;
      lx = min(15, max(0, lx)); ly = min(15, max(0, ly));
      key = ((uint32_t)(cy * a.grid_x + cx) << PT_KEY_SHIFT) | (uint32_t)(((ly >> 2) * 2 + (lx >> 3)) * 32 + (ly & 3) * 8 + (lx & 7));
    }
  }
  a.key[idx] = key;
  a.val[idx] = (uint32_t)idx;
}

struct IntArgs {
  int W, H, grid_x, tiles;
  float focal_x, focal_y;
  const uint2* ranges;
  const uint32_t* point_list;
  const GofSplat* splat;
  const uint2* pranges;
  const uint32_t* pt_list;
  const float2* pt_xy;
  const float* pt_depth;
  const float* bg;
  uint16_t* ids;        // [gridDim][256][1024]
  float* final_T;       // tile-major plane 0 of the image state
  uint32_t* ncontrib;   // tile-major planes 0 (last contributor) and 1 (contributors recorded, for export_state)
  float* out_color;     // [9][H][W]
  float* out_alpha;     // [PN]
  float* out_color_int; // [PN][3]
};

constexpr int BATCH = GOF_BLOCK_SIZE;

__device__ __forceinline__ bool box_hits(uint32_t lo, uint32_t hi, int wx0, int wy0, int wx1, int wy1) {
  const int x0 = (int)(short)(lo & 0xffffu), y0 = (int)(short)(lo >> 16);
  const int x1 = (int)(short)(hi & 0xffffu), y1 = (int)(short)(hi >> 16);
  return x0 <= wx1 && x1 >= wx0 && y0 <= wy1 && y1 >= wy0;
}

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

// one ray of pass 1 (forward.cu:931-975): true when the Gaussian is blended on this ray; then *alpha / *test_T hold the
// blend weight and the transmittance after it, and tmax has been raised to t (forward.cu:965-967)
template <int K>
__device__ __forceinline__ bool ray_step(const float* v, float op, float thr, float rx, float ry, float Tk, float& tmax,
                                         float* alpha, float* test_T) {
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
  if (power > 0.0f) power = 0.0f;
  const float al = fminf(F_MUL(op, F_EXP(power)), GOF_ALPHA_MAX);
  if (al < GOF_ALPHA_MIN) return false;
  const float tt = F_MUL(Tk, F_SUB(1.0f, al));
  if (tt < GOF_T_EPS) return false;
  if (t > tmax) tmax = t;
  *alpha = al;
  *test_T = tt;
  return true;
}

__global__ void __launch_bounds__(GOF_BLOCK_SIZE, 3) k_integrate(const IntArgs a) {
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
    const int wx0 = tile_x * 16 + (warp & 1) * 8, wy0 = tile_y * 16 + (warp >> 1) * 4;
    const uint32_t pix_x = wx0 + (lane & 7), pix_y = wy0 + (lane >> 3);
    const bool inside = pix_x < (uint32_t)a.W && pix_y < (uint32_t)a.H;
    bool done = !inside;

    // forward.cu:920: ((pixf + offset) - S/2.) / focal, offsets 0 / -0.5 / +0.5
    const float pfx = F_ADD((float)pix_x, 0.5f), pfy = F_ADD((float)pix_y, 0.5f);
    const double hw = D_MUL((double)a.W, 0.5), hh = D_MUL((double)a.H, 0.5);
    const float rx0 = (float)D_DIV(D_SUB((double)pfx, hw), (double)a.focal_x);
    const float ry0 = (float)D_DIV(D_SUB((double)pfy, hh), (double)a.focal_y);
    const float rxm = (float)D_DIV(D_SUB((double)F_ADD(pfx, -0.5f), hw), (double)a.focal_x);
    const float rxp = (float)D_DIV(D_SUB((double)F_ADD(pfx, 0.5f), hw), (double)a.focal_x);
    const float rym = (float)D_DIV(D_SUB((double)F_ADD(pfy, -0.5f), hh), (double)a.focal_y);
    const float ryp = (float)D_DIV(D_SUB((double)F_ADD(pfy, 0.5f), hh), (double)a.focal_y);

    const uint2 range = a.ranges[tile];
    const int total = (int)(range.y - range.x);
    const int rounds = (total + BATCH - 1) / BATCH;

    float T0 = 1.f, T1 = 1.f, T2 = 1.f, T3 = 1.f, T4 = 1.f;
    float C0 = 0.f, C1 = 0.f, C2 = 0.f, tmax = 0.f, Aacc = 0.f;
    uint32_t last_contributor = 0, n_local = 0;

    // ---------------- pass 1 (forward.cu:886-993) ----------------
    for (int i = 0; i < rounds; ++i) {
      __syncthreads();
      const int progress = i * BATCH + (int)threadIdx.x;
      if (progress < total) {
        const uint32_t g = a.point_list[range.x + progress];
        const float4* src = reinterpret_cast<const float4*>(a.splat + g);
        const float4 r2 = __ldg(src + 2);
        s_rec[threadIdx.x][0] = __ldg(src); s_rec[threadIdx.x][1] = __ldg(src + 1);
        s_rec[threadIdx.x][2] = r2; s_rec[threadIdx.x][3] = __ldg(src + 3);
        const float op = r2.z;
        s_rec[threadIdx.x][4].x = (op > 0.f) ? (-logf(255.0f * op) - 2e-3f) : __int_as_float(0x7f800000);
      }
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
        uint32_t m = __ballot_sync(0xffffffffu, idx < nb && box_hits(__float_as_uint(qb.z), __float_as_uint(qb.w), wx0, wy0, wx0 + 7, wy0 + 3));
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
          float al, tt;
          bool used = false;
          if (ray_step<0>(v, op, thr, rx0, ry0, T0, tmax, &al, &tt)) {
            const float2 q3 = gof_lds64<48>(row);
            C0 = F_FMA(T0, F_MUL(al, q2.w), C0);
            C1 = F_FMA(T0, F_MUL(al, q3.x), C1);
            C2 = F_FMA(T0, F_MUL(al, q3.y), C2);
            Aacc = F_FMA(T0, al, Aacc);
            T0 = tt; used = true;
          }
          if (ray_step<1>(v, op, thr, rxm, rym, T1, tmax, &al, &tt)) { T1 = tt; used = true; }
          if (ray_step<2>(v, op, thr, rxp, rym, T2, tmax, &al, &tt)) { T2 = tt; used = true; }
          if (ray_step<3>(v, op, thr, rxm, ryp, T3, tmax, &al, &tt)) { T3 = tt; used = true; }
          if (ray_step<4>(v, op, thr, rxp, ryp, T4, tmax, &al, &tt)) { T4 = tt; used = true; }
          if (used) {
            last_contributor = contributor;
            my_ids[n_local] = (uint16_t)contributor;    // uint16 truncation as in forward.cu:983
            n_local += 1;
            if (n_local >= GOF_INT_MAX_CONTRIB) done = true;   // forward.cu:986-990
          }
        }
      }
    }

    // forward.cu:997-1008
    const size_t slot = (size_t)tile * 256 + threadIdx.x;
    a.final_T[slot] = T0;
    a.ncontrib[slot] = last_contributor;
    a.ncontrib[(size_t)a.tiles * 256 + slot] = n_local;
    const float col0 = F_FMA(T0, a.bg[0], C0), col1 = F_FMA(T0, a.bg[1], C1), col2 = F_FMA(T0, a.bg[2], C2);
    s_cnt[threadIdx.x] = n_local;
    s_col[threadIdx.x][0] = col0; s_col[threadIdx.x][1] = col1; s_col[threadIdx.x][2] = col2;
    s_proj[threadIdx.x] = 0u;
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
        // the pixel (thread slot) this point belongs to: pix <= xy < pix + 1 (forward.cu:1071-1072)
        int lx = gof_f2i_rz(xy.x) - tile_x * 16, ly = gof_f2i_rz(xy.y) - tile_y * 16;
        lx = min(15, max(0, lx)); ly = min(15, max(0, ly));
        const int pslot = ((ly >> 2) * 2 + (lx >> 3)) * 32 + (ly & 3) * 8 + (lx & 7);
        atomicAdd(&s_proj[pslot], 1u);
        const float rx = (float)D_DIV(D_FMA((double)a.W, -0.5, (double)xy.x), (double)a.focal_x);
        const float ry = (float)D_DIV(D_FMA((double)a.H, -0.5, (double)xy.y), (double)a.focal_y);
        const uint32_t cnt = s_cnt[pslot];
        const uint16_t* ids = slab + (size_t)pslot * GOF_INT_MAX_CONTRIB;
        float point_alpha = 0.f, point_T = 1.f;
        uint32_t prev = 0;
        for (uint32_t c = 0; c < cnt; ++c) {
          const uint32_t cid = (uint32_t)ids[c];
          if (cid <= prev) break;     // a wrapped uint16 id can never be matched again by the running index (:1141-1149)
          prev = cid;
          const uint32_t g = a.point_list[range.x + cid - 1];
          const float4* src = reinterpret_cast<const float4*>(a.splat + g);
          const float4 q0 = __ldg(src), q1 = __ldg(src + 1), q2 = __ldg(src + 2);
          const float v[10] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y};
          const GofPair p = gof_pair_geom(v, rx, ry);
          float t = F_DIV(-p.BB, F_ADD(p.AA, p.AA));
          if (t > ray_depth) t = ray_depth;
          const float power = F_MUL(F_ADD(v[9], F_FMA(p.BB, t, F_MUL(t, F_MUL(p.AA, t)))), -0.5f);
          const float al = fminf(F_MUL(q2.z, F_EXP(power)), GOF_ALPHA_MAX);
          if (al < GOF_ALPHA_MIN) continue;
          point_alpha = F_FMA(al, point_T, point_alpha);
          point_T = F_MUL(point_T, F_SUB(1.0f, al));
        }
        a.out_alpha[id] = point_alpha;
        a.out_color_int[3 * (size_t)id + 0] = s_col[pslot][0];
        a.out_color_int[3 * (size_t)id + 1] = s_col[pslot][1];
        a.out_color_int[3 * (size_t)id + 2] = s_col[pslot][2];
      }
    }
    __syncthreads();
    if (inside) {
      const size_t pid = (size_t)pix_y * a.W + pix_x;
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

}  // namespace

int gof_launch_integrate(const gof_scene_t* s, const GofView& v, int PN, const float* points3D, const GofSplat* splat,
                         const uint32_t* point_list, const uint2* ranges, char* img, const GofImageLayout& IL, char* pts,
                         const GofPointLayout& PL, char* pbin, const GofPointBinLayout& PBL, float* out_color, float* out_alpha,
                         float* out_color_int, cudaStream_t st) {
  const bool debug = s->debug != 0;
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
  int in_b = 0;
  uint2* pranges = reinterpret_cast<uint2*>(pbin + PBL.pranges);
  int rc = gof_sort_points_by_tile((size_t)PN, gof_bits_for(((uint32_t)v.tiles + 1u) << PT_KEY_SHIFT), PT_KEY_SHIFT, ka, kb, va, vb,
                                   reinterpret_cast<uint32_t*>(pbin + PBL.hist), pranges, v.tiles, debug, st, &in_b);
  if (rc != GOF_OK) return rc;

  IntArgs a{};
  a.W = v.W; a.H = v.H; a.grid_x = v.grid_x; a.tiles = v.tiles; a.focal_x = v.focal_x; a.focal_y = v.focal_y;
  a.ranges = ranges;
  a.point_list = point_list;
  a.splat = splat;
  a.pranges = pranges; a.pt_list = in_b ? vb : va; a.pt_xy = pa.xy; a.pt_depth = pa.depth; a.bg = s->background;
  a.ids = reinterpret_cast<uint16_t*>(pbin + PBL.ids);
  a.final_T = reinterpret_cast<float*>(img + IL.accum);
  a.ncontrib = reinterpret_cast<uint32_t*>(img + IL.ncontrib);
  a.out_color = out_color; a.out_alpha = out_alpha; a.out_color_int = out_color_int;
  GOF_LAUNCH("integrate", st, k_integrate<<<PBL.nblk, GOF_BLOCK_SIZE, 0, st>>>(a));
  GOF_LAUNCH_CHECK(debug, st);
  return GOF_OK;
}
