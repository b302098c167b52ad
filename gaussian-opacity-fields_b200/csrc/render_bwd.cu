// render_bwd.cu -- K7: per-tile back-to-front gradient pass (backward.cu:634-955).
//
// The reference issues 17 global float atomics per contributing (pixel,Gaussian) pair
// (backward.cu:836,905-912,943-952).  Here a warp owns an 8x4 pixel block; the partial gradients of its 32
// pixels are summed with a 16-shuffle butterfly (dL_dopacity is -2/opacity * dL_dC, so 16 values carry all
// 17 outputs) and leave the SM as 16 atomics per (warp,Gaussian) into that Gaussian's accumulator row (16 doubles).
// The forward leaves, per (warp, tile-list entry), the mask of pixels that blended it (GofBinLayout::vmask): the
// backward visits exactly those (no box test, no reject arithmetic -- 44 % of the forward's visits blend nothing),
// re-evaluating t, G and alpha with the forward's operation sequence (gof_math.cuh) so that they are bit-identical.
// The traversal starts at the last Gaussian any pixel of the tile blended.
// Staging of the per-tile slab (64-byte record + 32-byte backward record per list entry) as in render_fwd.cu: bulk copies
// completing on an mbarrier, cp.async, or the round-1 load/store staging (GOF_STAGE_BWD=bulk|cpasync|regs; regs is the default
// -- see the launcher for the measurements), the first two double buffered in 2 x 24 KB of dynamic shared memory.
#include <stdlib.h>

#include "gof_common.cuh"
#include "gof_math.cuh"

namespace {

struct BwdArgs {
  int W, H, grid_x;
  float focal_x, focal_y;
  const uint2* ranges;
  const uint32_t* point_list;
  const GofSplat* splat;
  const GofSplatBwd* splat_bwd;
  const float* bg;
  const float* accum;        // [4][tiles*256]
  const uint32_t* ncontrib;  // [2][tiles*256]
  const float* dL_dpix;      // [9][H][W]
  size_t plane;
  const uint32_t* vmask;   // blend masks left by the forward (GofBinLayout::vmask)
  size_t vstride;
  double* grad_acc;    // [P][16]: dL_dview2gaussian[10] | dL_dcolor[3] | dL_dmean2D[3] (128-byte rows, zeroed per call).  Double:
                       // the float partials arrive in scheduling order.  A float sum differs from run to run by ulps, which
                       // the view2gaussian chain rule amplifies to percents in dL_dscale / dL_drot; the order moves a double
                       // sum only in its last bits, so after k_preprocess_backward's one rounding to float the gradients
                       // agree from run to run unless a sum lies that close to a float rounding boundary
  unsigned long long* stats;   // optional [8] counters (GOF_STATS=1), else nullptr
};

constexpr int BATCH = GOF_BLOCK_SIZE;

// Sum 16 per-lane values over the warp with 16 shuffles (instead of 16 x 5): at every step each lane keeps half of
// its values and trades the other half with its partner.  On return `r` holds, in BOTH lanes of each even/odd
// pair, the warp-wide sum of value number (lane >> 1).
__device__ __forceinline__ float warp_reduce16(const float (&a)[16], int lane) {
  float b[8], c[4], d[2], e;
  const bool h16 = lane & 16, h8 = lane & 8, h4 = lane & 4, h2 = lane & 2;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float send = h16 ? a[i] : a[i + 8], keep = h16 ? a[i + 8] : a[i];
    b[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float send = h8 ? b[i] : b[i + 4], keep = h8 ? b[i + 4] : b[i];
    c[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const float send = h4 ? c[i] : c[i + 2], keep = h4 ? c[i + 2] : c[i];
    d[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
  }
  {
    const float send = h2 ? d[0] : d[1], keep = h2 ? d[1] : d[0];
    e = keep + __shfl_xor_sync(0xffffffffu, send, 2);
  }
  e += __shfl_xor_sync(0xffffffffu, e, 1);
  return e;
}

// STAGE: 0 = registers + st.shared (round 1), 1 = cp.async.bulk + mbarrier, 2 = cp.async (LDGSTS)
// The same over a QUARTER of the warp -- the 8 lanes of a 4x2 pixel block: lanes that differ in bits 0, 1 (x) and 3 (y) only --
// with 14 shuffles.  On return r0 / r1 hold the quarter-wide sums of values number `base` and `base + 1`,
// base = (lane & 8 ? 8 : 0) + (lane & 2 ? 4 : 0) + (lane & 1 ? 2 : 0).
__device__ __forceinline__ void quarter_reduce16(const float (&a)[16], int lane, float* r0, float* r1) {
  float b[8], c[4];
  const bool h3 = lane & 8, h1 = lane & 2, h0 = lane & 1;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float send = h3 ? a[i] : a[i + 8], keep = h3 ? a[i + 8] : a[i];
    b[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float send = h1 ? b[i] : b[i + 4], keep = h1 ? b[i + 4] : b[i];
    c[i] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
  }
  {
    const float send0 = h0 ? c[0] : c[2], keep0 = h0 ? c[2] : c[0];
    const float send1 = h0 ? c[1] : c[3], keep1 = h0 ? c[3] : c[1];
    *r0 = keep0 + __shfl_xor_sync(0xffffffffu, send0, 1);
    *r1 = keep1 + __shfl_xor_sync(0xffffffffu, send1, 1);
  }
}

// SUB: the four 4x2 pixel blocks of a warp walk their OWN lists (see the loop); otherwise the warp walks one list (round 1)
template <bool STATS, int MINB, int STAGE, bool SUB>
__global__ void __launch_bounds__(GOF_BLOCK_SIZE, MINB) k_render_backward(const BwdArgs a) {
  constexpr bool BULK = STAGE == 1, CPA = STAGE == 2;
  unsigned long long st_visit = 0, st_eval = 0, st_pass = 0, st_contrib = 0, st_anyhit = 0;
  // rows of 96 bytes per staged Gaussian = GofSplat (64 B) | GofSplatBwd (32 B: means2D, 2D conic, own index); one row base
  // register serves every load of a visit (see gof_smem_base).  One buffer (24 KB) for STAGE 0, two otherwise.
  extern __shared__ __align__(128) float4 s_dyn[];
  __shared__ __align__(8) unsigned long long s_bar[2];
  __shared__ uint32_t s_max;
  const uint32_t s_base = gof_smem_base(s_dyn);
  const uint32_t bar0 = (uint32_t)__cvta_generic_to_shared(&s_bar[0]);

  const int tile = blockIdx.x;
  const int tile_x = tile % a.grid_x, tile_y = tile / a.grid_x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int wx0 = tile_x * 16 + (warp & 1) * 8, wy0 = tile_y * 16 + (warp >> 1) * 4;
  const uint32_t pix_x = wx0 + (lane & 7);
  const uint32_t pix_y = wy0 + (lane >> 3);
  const bool inside = pix_x < (uint32_t)a.W && pix_y < (uint32_t)a.H;
  const float rx = gof_ray(pix_x, a.W, a.focal_x);
  const float ry = gof_ray(pix_y, a.H, a.focal_y);

  const uint2 range = a.ranges[tile];
  const uint32_t* vm_row = a.vmask + (size_t)warp * a.vstride + range.x + 32u * (uint32_t)tile + lane;   // + 32*group
  const size_t slot = (size_t)tile * 256 + threadIdx.x;
  const size_t HW = (size_t)a.H * a.W;
  const size_t pid = (size_t)pix_y * a.W + pix_x;

  // backward.cu:692-723
  const float T_final = inside ? a.accum[slot] : 0.f;
  float T = T_final;
  const float final_D = inside ? a.accum[a.plane + slot] : 0.f;
  const float final_A = 1.f - T_final;
  const uint32_t last_contributor = inside ? a.ncontrib[slot] : 0u;
  const uint32_t max_contributor = inside ? a.ncontrib[a.plane + slot] : 0u;
  float dpix0 = 0.f, dpix1 = 0.f, dpix2 = 0.f, dn0 = 0.f, dn1 = 0.f, dn2 = 0.f, ddepth = 0.f, dreg = 0.f;
  if (inside) {
    dpix0 = a.dL_dpix[0 * HW + pid]; dpix1 = a.dL_dpix[1 * HW + pid]; dpix2 = a.dL_dpix[2 * HW + pid];
    dn0 = a.dL_dpix[3 * HW + pid]; dn1 = a.dL_dpix[4 * HW + pid]; dn2 = a.dL_dpix[5 * HW + pid];
    ddepth = a.dL_dpix[6 * HW + pid];
    dreg = a.dL_dpix[8 * HW + pid];   // channel 7 (alpha) receives no gradient, backward.cu:697,717-723
  }
  const float bg_dot_dpixel = a.bg[0] * dpix0 + a.bg[1] * dpix1 + a.bg[2] * dpix2;

  // traversal starts at the deepest Gaussian any pixel of this tile blended; each warp additionally skips
  // everything behind the deepest Gaussian ITS 32 pixels blended
  uint32_t warp_last = last_contributor;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) warp_last = max(warp_last, __shfl_xor_sync(0xffffffffu, warp_last, d));
  if (threadIdx.x == 0) {
    s_max = 0u;
    if (BULK) {
      gof_mbar_init(bar0, GOF_BLOCK_SIZE);
      gof_mbar_init(bar0 + 8u, GOF_BLOCK_SIZE);
      gof_mbar_init_fence();
    }
  }
  __syncthreads();
  if (lane == 0) atomicMax(&s_max, warp_last);
  __syncthreads();
  const int used = (int)min(s_max, range.y - range.x);
  const int rounds = (used + BATCH - 1) / BATCH;

  float last_alpha = 0.f;
  float last_c0 = 0.f, last_c1 = 0.f, last_c2 = 0.f, acc_c0 = 0.f, acc_c1 = 0.f, acc_c2 = 0.f;
  float last_n0 = 0.f, last_n1 = 0.f, last_n2 = 0.f, acc_n0 = 0.f, acc_n1 = 0.f, acc_n2 = 0.f;
  const float ddelx_dx = 0.5f * a.W, ddely_dy = 0.5f * a.H;

  // which output the even lanes of the butterfly feed: value index v = lane >> 1
  //   v 0..9 -> dL_dview2gaussian[0..9] (v 9 = dL_dC also yields dL_dopacity = -2/opacity * that sum: both are
  //   G*dL_dalpha up to a per-Gaussian constant; dL_dC is the one carried through the reduction because the
  //   view2gaussian chain rule cancels it against the other nine to ~1e-5 and needs them rounded consistently),
  //   v 10..12 -> dL_dcolor, v 13..15 -> dL_dmean2D
  const int vidx = lane >> 1;

  // ---- staging: step s of the walk handles batch ib = rounds-1-s (entries [256*ib, 256*ib+256) of the tile list) out of
  // buffer s & 1; its copies are issued one step earlier -------------------------------------------------------
  uint32_t meta_id = 0;
  auto load_meta = [&](int step) {
    const int e = (rounds - 1 - step) * BATCH + (int)threadIdx.x;
    if (step < rounds && e < used) meta_id = a.point_list[range.x + (uint32_t)e];
  };
  auto issue = [&](int step) {
    const bool has = (rounds - 1 - step) * BATCH + (int)threadIdx.x < used;
    const uint32_t row = s_base + (uint32_t)((step & 1) * BATCH + (int)threadIdx.x) * 96u;
    if (BULK) {   // every thread arrives once per step on the buffer's mbarrier; threads with an entry add 96 bytes
      const uint32_t bar = bar0 + 8u * (uint32_t)(step & 1);
      if (has) {
        gof_mbar_arrive_expect_tx(bar, 96u);
        gof_bulk_g2s(row, a.splat + meta_id, 64u, bar);
        gof_bulk_g2s(row + 64u, a.splat_bwd + meta_id, 32u, bar);
      } else {
        gof_mbar_arrive(bar);
      }
    } else if (has) {
      const char* src = reinterpret_cast<const char*>(a.splat + meta_id);
      const char* srcb = reinterpret_cast<const char*>(a.splat_bwd + meta_id);
      gof_cp_async16(row, src); gof_cp_async16(row + 16u, src + 16);
      gof_cp_async16(row + 32u, src + 32); gof_cp_async16(row + 48u, src + 48);
      gof_cp_async16(row + 64u, srcb); gof_cp_async16(row + 80u, srcb + 16);
    }
  };
  if (STAGE) {
    load_meta(0);
    if (rounds > 0) issue(0);
    load_meta(1);
  }

  // Batches are the forward's, taken from the deepest one the tile used down to 0; inside a batch the groups of 32 and the
  // bits inside a group are walked from high to low: back to front.
  for (int i = 0; i < rounds; ++i) {
    const int ib = rounds - 1 - i;
    const int base = ib * BATCH;
    uint32_t buf_base = s_base;
    if (STAGE) {
      if (CPA) gof_cp_async_wait_all();   // this thread's copies of step i have landed; the barrier publishes everybody's
      __syncthreads();                    // every warp has finished step i-1: its buffer may be refilled
      buf_base = s_base + (uint32_t)(i & 1) * (uint32_t)(BATCH * 96);
      if (i + 1 < rounds) {
        issue(i + 1);                     // lands while this batch is walked
        load_meta(i + 2);
      }
      if (BULK) gof_mbar_wait(bar0 + 8u * (uint32_t)(i & 1), (uint32_t)(i >> 1) & 1u);
    } else {
      __syncthreads();
      if (base + (int)threadIdx.x < used) {
        const uint32_t g = a.point_list[range.x + (uint32_t)(base + (int)threadIdx.x)];
        const float4* src = reinterpret_cast<const float4*>(a.splat + g);
        const float4 r0 = __ldg(src), r1 = __ldg(src + 1), r2 = __ldg(src + 2), r3 = __ldg(src + 3);
        float4* dst = s_dyn + (size_t)threadIdx.x * 6;
        dst[0] = r0; dst[1] = r1; dst[2] = r2; dst[3] = r3;
        const float4* srcb = reinterpret_cast<const float4*>(a.splat_bwd + g);
        dst[4] = __ldg(srcb); dst[5] = __ldg(srcb + 1);
      }
      __syncthreads();
    }

    // the loop is NOT unrolled (one copy of the body, see render_fwd.cu)
#pragma unroll 1
    for (int k = BATCH / 32 - 1; k >= 0; --k) {
      const int gstart = base + k * 32;
      // the forward wrote the masks of every group up to this warp's deepest contributor; nothing behind it blended
      if ((uint32_t)gstart >= warp_last) continue;
      const uint32_t mybits = __ldg(vm_row + gstart);        // bit b: this pixel blended entry gstart+b

      // the 16 partial gradients of ONE (pixel, Gaussian) pair: row = the staged record, contributor = its zero-based index in the
      // tile list (the reference's `contributor` after its decrement, backward.cu:763), contrib = this pixel blended it
      auto pair_grad = [&](const uint32_t row, const uint32_t contributor, const bool contrib, float (&g)[16]) {
        if (STATS) { st_eval += contrib; st_pass += contrib; }
        const float4 q0 = gof_lds128<0>(row), q1 = gof_lds128<16>(row), q2 = gof_lds128<32>(row);
        const float v[10] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y};
        GofPair p;
        float t = 0.f, G = 0.f, alpha = 0.f;
        double qd = 0.0, rA = 0.0;
        if (contrib) {
          // re-evaluated with the forward's operation sequence: bit-identical t, G, alpha
          p = gof_pair_geom(v, rx, ry);
          float power;
          gof_pair_t_power(p, v[9], &t, &power, &qd, &rA);
          G = F_EXP(power);
          alpha = fminf(F_MUL(q2.z, G), GOF_ALPHA_MAX);
        }
        if (STATS) st_contrib += contrib;

#pragma unroll
        for (int q = 0; q < 16; ++q) g[q] = 0.f;
        if (contrib) {
          // backward.cu:806-817
          float rt;
          const float mt = gof_mapped_t_fast(t, &rt);
          const float dm_dt = ((20.0f / 99.8f) * rt) * rt;   // d/dt of 100/99.8 - (20/99.8)/t
          // 1/|n| to ~1 ulp (Newton-refined rsqrt; as accurate as an IEEE sqrt followed by an IEEE reciprocal -- the
          // plain 2-ulp rsqrt is not: this feeds dL_dview2gaussian, whose chain rule amplifies every ulp by ~1/scale^2)
          const float rlen = gof_rsqrt_newton(F_FMA(p.n2, p.n2, F_FMA(p.n0, p.n0, F_MUL(p.n1, p.n1))) + 1e-7f);
          const float nn0 = -p.n0 * rlen, nn1 = -p.n1 * rlen, nn2 = -p.n2 * rlen;
          const float r1a = gof_rcp_newton(1.f - alpha);   // 1 - alpha in [0.01, 1]
          T = T * r1a;
          const float w = alpha * T;
          float dL_dalpha = 0.f;
          // colour, :824-837
          const float2 q3 = gof_lds64<48>(row);
          const float c0 = q2.w, c1 = q3.x, c2 = q3.y;
          acc_c0 = last_alpha * last_c0 + (1.f - last_alpha) * acc_c0; last_c0 = c0;
          acc_c1 = last_alpha * last_c1 + (1.f - last_alpha) * acc_c1; last_c1 = c1;
          acc_c2 = last_alpha * last_c2 + (1.f - last_alpha) * acc_c2; last_c2 = c2;
          dL_dalpha += (c0 - acc_c0) * dpix0;
          dL_dalpha += (c1 - acc_c1) * dpix1;
          dL_dalpha += (c2 - acc_c2) * dpix2;
          g[10] = w * dpix0; g[11] = w * dpix1; g[12] = w * dpix2;
          // distortion: only the depth path survives ("detach weight", :848-858)
          const float dL_dmax_t = 2.0f * (T * alpha) * (mt * final_A - final_D) * dreg * dm_dt;
          // normal, :860-877
          acc_n0 = last_alpha * last_n0 + (1.f - last_alpha) * acc_n0; last_n0 = nn0;
          acc_n1 = last_alpha * last_n1 + (1.f - last_alpha) * acc_n1; last_n1 = nn1;
          acc_n2 = last_alpha * last_n2 + (1.f - last_alpha) * acc_n2; last_n2 = nn2;
          dL_dalpha += (nn0 - acc_n0) * dn0;
          dL_dalpha += (nn1 - acc_n1) * dn1;
          dL_dalpha += (nn2 - acc_n2) * dn2;
          const float dnn0 = w * dn0, dnn1 = w * dn1, dnn2 = w * dn2;
          const float dL_dlength = (dnn0 * p.n0 + dnn1 * p.n1 + dnn2 * p.n2) * (rlen * rlen);
          float dnrm0 = (-dnn0 + dL_dlength * p.n0) * rlen;
          float dnrm1 = (-dnn1 + dL_dlength * p.n1) * rlen;
          float dnrm2 = (-dnn2 + dL_dlength * p.n2) * rlen;
          // :879-893
          float dL_dt = dL_dmax_t;
          if (contributor == max_contributor - 1u) dL_dt += ddepth;
          dL_dalpha *= T;
          last_alpha = alpha;
          dL_dalpha += (-T_final * r1a) * bg_dot_dpixel;
          // :896-912  2D-mean statistic and opacity
          const float4 b0 = gof_lds128<64>(row);   // (mx, my, cx, cy)
          const float b1x = gof_lds32<80>(row);    // cz
          const float dx = b0.x - (float)pix_x, dy = b0.y - (float)pix_y;
          const float dL_dG = q2.z * dL_dalpha;
          const float gdx = G * dx, gdy = G * dy;
          const float dG_ddelx = -gdx * b0.z - gdy * b0.w;
          const float dG_ddely = -gdy * b1x - gdx * b0.w;
          g[13] = dL_dG * dG_ddelx * ddelx_dx;
          g[14] = dL_dG * dG_ddely * ddely_dy;
          g[15] = fabsf(g[13]) + fabsf(g[14]);
          // :914-928 in double like the reference; BB/AA = -qd is reused from the forward evaluation
          const float dL_dmin = dL_dG * G * -0.5f;
          g[9] = dL_dmin;   // dL_dC; dL_dopacity = G*dL_dalpha = dL_dC * (-2/opacity) is derived from its sum below
          // A and B enter in double like the reference; 1/AA comes from the forward division (rA), -BB/AA = qd.
          // The sums below are formed by single float FMAs on the rounded dL_dA / dL_dB: one rounding each, like
          // the reference's double expression stored to float.
          const double inv2A = 0.5 * rA;
          const float dA = (float)((double)dL_dmin * qd * qd * 0.25 - (double)dL_dt * qd * inv2A);
          const float dB2 = (float)((double)dL_dmin * qd - (double)dL_dt * rA);   // 2 * dL_dB
          // :938-952
          dnrm0 = fmaf(dA, rx, dnrm0);
          dnrm1 = fmaf(dA, ry, dnrm1);
          dnrm2 = dnrm2 + dA;
          g[0] = dnrm0 * rx;
          g[1] = dnrm0 * ry + dnrm1 * rx;
          g[2] = dnrm0 + dnrm2 * rx;
          g[3] = dnrm1 * ry;
          g[4] = dnrm1 + dnrm2 * ry;
          g[5] = dnrm2;
          g[6] = dB2 * rx;
          g[7] = dB2 * ry;
          g[8] = dB2;
        }
      };

      if (!SUB) {
        uint32_t m = __reduce_or_sync(0xffffffffu, mybits);
        while (m) {
          const int b = 31 - __clz(m);
          m &= ~(1u << b);
          const uint32_t row = buf_base + (uint32_t)(k * 32 + b) * 96u;
          const bool contrib = ((mybits >> b) & 1u) != 0u;   // implies inside && contributor < last_contributor
          if (STATS) { st_visit += (lane == 0); st_anyhit += (lane == 0); }
          float g[16];
          pair_grad(row, (uint32_t)(gstart + b), contrib, g);
          const float sum = warp_reduce16(g, lane);
          // one red per even lane into the Gaussian's accumulator row: 16 global atomics per (warp, Gaussian) instead of
          // 17 per (pixel, Gaussian); dL_dopacity = -2/opacity * sum(dL_dC) is formed by k_preprocess_backward
          const uint32_t gid = __float_as_uint(gof_lds32<84>(row));   // GofSplatBwd::self
          if (!(lane & 1) && sum != 0.f) atomicAdd(a.grad_acc + ((size_t)gid * 16 + vidx), (double)sum);
        }
      } else {
        // Each 4x2 pixel block (a quarter of the warp: the lanes that differ in bits 0, 1, 3) walks ITS OWN list -- the entries one
        // of its 8 pixels blended -- in lockstep with the other three: an iteration handles up to four different Gaussians, one per
        // quarter.  A Gaussian of pixel-scale footprint touches 16 of a warp's 32 pixels on average, so the warp-wide walk leaves
        // half of the lanes idle; quarter-wide, 4.9 M instead of 5.9 M iterations cover the same 93 M pairs at the benchmark
        // workload.  The partial gradients are reduced over the quarter (14 shuffles) and leave
        // as two reds per lane.
        uint32_t qb = mybits;
        qb |= __shfl_xor_sync(0xffffffffu, qb, 1);
        qb |= __shfl_xor_sync(0xffffffffu, qb, 2);
        qb |= __shfl_xor_sync(0xffffffffu, qb, 8);
        while (__any_sync(0xffffffffu, qb != 0u)) {
          const bool act = qb != 0u;
          const int b = act ? 31 - __clz(qb) : 0;
          if (act) qb &= ~(1u << b);
          const uint32_t row = buf_base + (uint32_t)(k * 32 + b) * 96u;
          const bool contrib = act && ((mybits >> b) & 1u) != 0u;
          if (STATS) { st_visit += (lane == 0); st_anyhit += act && !(lane & 11); }
          float g[16];
          pair_grad(row, (uint32_t)(gstart + b), contrib, g);
          float r0, r1;
          quarter_reduce16(g, lane, &r0, &r1);
          if (act) {
            const uint32_t gid = __float_as_uint(gof_lds32<84>(row));   // GofSplatBwd::self
            double* dst = a.grad_acc + ((size_t)gid * 16 + ((lane & 8) ? 8 : 0) + ((lane & 2) ? 4 : 0) + ((lane & 1) ? 2 : 0));
            if (r0 != 0.f) atomicAdd(dst, (double)r0);
            if (r1 != 0.f) atomicAdd(dst + 1, (double)r1);
          }
        }
      }
    }
  }
  if (STATS && a.stats) {
    atomicAdd(a.stats + 0, st_visit); atomicAdd(a.stats + 1, st_eval); atomicAdd(a.stats + 2, st_pass);
    atomicAdd(a.stats + 3, st_contrib); atomicAdd(a.stats + 4, st_anyhit);
    if (threadIdx.x == 0) { atomicAdd(a.stats + 5, (unsigned long long)used); atomicAdd(a.stats + 6, (unsigned long long)(range.y - range.x)); }
  }
}

}  // namespace

int gof_launch_render_backward(const gof_scene_t* s, const GofView& v, char* geom, const GofGeomLayout& GL,
                               const char* bin, const GofBinLayout& BL, const char* img, const GofImageLayout& IL,
                               const float* dL_dpix, cudaStream_t st) {
  BwdArgs a{};
  a.W = v.W; a.H = v.H; a.grid_x = v.grid_x; a.focal_x = v.focal_x; a.focal_y = v.focal_y;
  a.ranges = reinterpret_cast<const uint2*>(img + IL.ranges);
  a.point_list = reinterpret_cast<const uint32_t*>(bin + BL.point_list);
  a.splat = reinterpret_cast<const GofSplat*>(geom + GL.splat);
  a.splat_bwd = reinterpret_cast<const GofSplatBwd*>(geom + GL.splat_bwd);
  a.bg = s->background;
  a.accum = reinterpret_cast<const float*>(img + IL.accum);
  a.ncontrib = reinterpret_cast<const uint32_t*>(img + IL.ncontrib);
  a.dL_dpix = dL_dpix;
  a.plane = (size_t)v.tiles * 256;
  a.vmask = reinterpret_cast<const uint32_t*>(bin + BL.vmask);
  a.vstride = BL.vmask_stride;
  a.grad_acc = reinterpret_cast<double*>(geom + GL.grad_acc);
  GOF_CUDA_OK(cudaMemsetAsync(a.grad_acc, 0, (size_t)s->P * 128, st));
  a.stats = gof_stats_buffer();
  static int occ = -1, stage = -1;   // GOF_BWD_OCC=2|3|4 (tuning knob); GOF_STAGE: staging variant (see render_fwd.cu)
  if (occ < 0) { const char* e = getenv("GOF_BWD_OCC"); occ = e ? atoi(e) : 4; }
  if (stage < 0) {
    const char* e = getenv("GOF_STAGE_BWD");
    if (!e) e = getenv("GOF_STAGE");
    // default: the round-1 staging, which was not slower than cp.async or bulk copies at the benchmark workload with right-sized
    // carveouts -- the backward walks each batch once and four CTAs per SM already cover the gather latency, while the two
    // per-thread bulk copies cost ~18 issue slots per record (ELECT loop) and the double buffer takes 96 KB of L1 away from the
    // mask / spill traffic.
    stage = !e ? 0 : (e[0] == 'r' ? 0 : (e[0] == 'c' ? 2 : 1));
  }
  // GOF_SUBWARP_BWD=0: one list per warp (round 1); default: one list per 4x2 pixel block
  static int sub = -1;
  if (sub < 0) { const char* e = getenv("GOF_SUBWARP_BWD"); sub = (e && e[0] == '0') ? 0 : 1; }
  const size_t smem = (size_t)(stage ? 2 : 1) * BATCH * 96;
#define GOF_BWD_LAUNCH(STATS, MINB, STG, SUBW)                                                                                      \
  do {                                                                                                                        \
    static bool attr_set = false;                                                                                             \
    if (!attr_set) {                                                                                                          \
      GOF_CUDA_OK(cudaFuncSetAttribute(k_render_backward<STATS, MINB, STG, SUBW>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * BATCH * 96)); \
      const int need = MINB * ((STG ? 2 : 1) * BATCH * 96 + 1024 + 128);   /* only what MINB CTAs need: the rest stays L1 */             \
      GOF_CUDA_OK(cudaFuncSetAttribute(k_render_backward<STATS, MINB, STG, SUBW>, cudaFuncAttributePreferredSharedMemoryCarveout,                \
                                       (need * 100 + 233471) / 233472 > 100 ? 100 : (need * 100 + 233471) / 233472));                     \
      attr_set = true;                                                                                                        \
    }                                                                                                                         \
    GOF_LAUNCH("render_bwd", st, k_render_backward<STATS, MINB, STG, SUBW><<<v.tiles, GOF_BLOCK_SIZE, smem, st>>>(a));       \
  } while (0)
#define GOF_BWD_STAGES(STATS, MINB)                                                                   \
  do {                                                                                                \
    if (sub) {                                                                                         \
      if (stage == 1) GOF_BWD_LAUNCH(STATS, MINB, 1, true); else if (stage == 2) GOF_BWD_LAUNCH(STATS, MINB, 2, true); \
      else GOF_BWD_LAUNCH(STATS, MINB, 0, true);                                                       \
    } else {                                                                                           \
      if (stage == 1) GOF_BWD_LAUNCH(STATS, MINB, 1, false); else if (stage == 2) GOF_BWD_LAUNCH(STATS, MINB, 2, false); \
      else GOF_BWD_LAUNCH(STATS, MINB, 0, false);                                                      \
    }                                                                                                  \
  } while (0)
  if (a.stats) GOF_BWD_STAGES(true, 3);
  else if (occ >= 4) GOF_BWD_STAGES(false, 4);
  else if (occ <= 2) GOF_BWD_STAGES(false, 2);
  else GOF_BWD_STAGES(false, 3);
#undef GOF_BWD_STAGES
#undef GOF_BWD_LAUNCH
  GOF_LAUNCH_CHECK(s->debug, st);
  return GOF_OK;
}
