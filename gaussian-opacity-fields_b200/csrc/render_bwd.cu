// render_bwd.cu -- K7: per-tile back-to-front gradient pass (backward.cu:634-955).
//
// The reference issues 17 global float atomics per contributing (pixel,Gaussian) pair
// (backward.cu:836,905-912,943-952).  Here a warp owns an 8x4 pixel block and each of its four 4x2 pixel blocks (a
// quarter of the warp) walks its own list; the partial gradients of a quarter's 8 pixels are summed with 14 shuffles
// (dL_dopacity is -2/opacity * dL_dC, so 16 values carry all 17 outputs) and leave the SM as 16 atomics per
// (quarter,Gaussian) into that Gaussian's accumulator row (16 doubles).
// The forward leaves, per (warp, tile-list entry), the mask of pixels that blended it (GofBinLayout::vmask): the
// backward visits exactly those (no box test, no reject arithmetic -- 44 % of the forward's visits blend nothing),
// re-evaluating t, G and alpha with the forward's operation sequence (gof_math.cuh) so that they are bit-identical.
// The traversal starts at the last Gaussian any pixel of the tile blended.
// The per-tile slab (64-byte record + 32-byte backward record per list entry) is staged through registers into one 24 KB
// buffer of dynamic shared memory, and each warp's masks of the batch into an 8 KB slab next to it.  The bulk-copy double
// buffer of render_fwd.cu does not pay here: the backward walks each batch once, four resident CTAs already cover the gather
// latency, the two per-thread bulk copies cost ~18 issue slots per record (ELECT loop) and the second buffer takes 96 KB per
// SM away from L1, which carries the gather / spill traffic.
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
  double* drays;       // RAYS only: [2][H][W] dL/drx, dL/dry of every pixel | [tiles][2] the tile's sums of rx dL/drx, ry dL/dry
};

constexpr int BATCH = GOF_BLOCK_SIZE;
constexpr int GROUPS = BATCH / 32;   // groups of 32 list entries per batch: one mask word per (warp, group, lane)
constexpr int WARPS = GOF_BLOCK_SIZE / 32;
// dynamic shared memory: [BATCH] records of 96 bytes | [WARPS][GROUPS][32] u32 blend masks of the batch.  32 KB in all, so that
// four CTAs (plus 1 KB reserved per CTA) fill the 132 KB shared-memory carveout exactly and L1 keeps the rest of the SM's 256 KB
constexpr int SMEM_RECORDS = BATCH * 96;
constexpr int SMEM_BYTES = SMEM_RECORDS + WARPS * GROUPS * 32 * 4;

// Sum 16 per-lane values over a QUARTER of the warp -- the 8 lanes of a 4x2 pixel block: lanes that differ in bits 0, 1 (x)
// and 3 (y) only -- with 14 shuffles: at every step each lane keeps half of its values and trades the other half with its
// partner.  On return r0 / r1 hold the quarter-wide sums of values number `v` and `v + 8`,
// v = (lane & 8 ? 1 : 0) + (lane & 2 ? 2 : 0) + (lane & 1 ? 4 : 0): the quarter's eight r0 cover values 0..7 of the Gaussian's
// accumulator row, 64 contiguous bytes (two 32-byte sectors), and its r1 values 8..15, so that each of the two reds per lane
// touches half of the row instead of all of it.  Each stage splits on one bit of the value index; which bit does not change
// the sums, since every value is added over the same lane pairs (xor 8, then 2, then 1).
__device__ __forceinline__ void quarter_reduce16(const float (&a)[16], int lane, float* r0, float* r1) {
  float b[8], c[4];
  const bool h3 = lane & 8, h1 = lane & 2, h0 = lane & 1;
#pragma unroll
  for (int i = 0; i < 8; ++i) {   // b[i] = value 2i + h3
    const float send = h3 ? a[2 * i] : a[2 * i + 1], keep = h3 ? a[2 * i + 1] : a[2 * i];
    b[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {   // c[i] = value 4i + 2 h1 + h3
    const float send = h1 ? b[2 * i] : b[2 * i + 1], keep = h1 ? b[2 * i + 1] : b[2 * i];
    c[i] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
  }
  {
    const float send0 = h0 ? c[0] : c[1], keep0 = h0 ? c[1] : c[0];
    const float send1 = h0 ? c[2] : c[3], keep1 = h0 ? c[3] : c[2];
    *r0 = keep0 + __shfl_xor_sync(0xffffffffu, send0, 1);
    *r1 = keep1 + __shfl_xor_sync(0xffffffffu, send1, 1);
  }
}

// RAYS (DESIGN.md 4.10): also differentiate the loss with respect to the pixel's ray r = (rx, ry, 1).  Each pair adds, in
// float, what the gradients it already holds give through n = M r, AA = r.n and BB; each lane sums its pixel's terms in double
// in the walk's own back-to-front order, so the per-pixel values and the tile sums involve no atomics.  RAYS = false is the
// plain backward, compiled to the same instructions as before the template.
template <bool RAYS>
__global__ void __launch_bounds__(GOF_BLOCK_SIZE, 4) k_render_backward(const BwdArgs a) {
  // rows of 96 bytes per staged Gaussian = GofSplat (64 B) | GofSplatBwd (32 B: means2D, 2D conic, own index); one row base
  // register serves every load of a visit (see gof_smem_base)
  extern __shared__ __align__(128) float4 s_dyn[];
  const uint32_t s_base = gof_smem_base(s_dyn);

  const int tile = blockIdx.x;
  const int tile_x = tile % a.grid_x, tile_y = tile / a.grid_x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // this warp's mask slab [GROUPS][32]; its first word also carries the tile's deepest contributor before the first batch
  uint32_t* const s_mask = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(s_dyn) + SMEM_RECORDS) + warp * GROUPS * 32;
  uint32_t* const s_max = s_mask - warp * GROUPS * 32;
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
  if (threadIdx.x == 0) *s_max = 0u;
  __syncthreads();
  if (lane == 0) atomicMax(s_max, warp_last);
  __syncthreads();
  const int used = (int)min(*s_max, range.y - range.x);
  const int rounds = (used + BATCH - 1) / BATCH;

  float last_alpha = 0.f;
  float last_c0 = 0.f, last_c1 = 0.f, last_c2 = 0.f, acc_c0 = 0.f, acc_c1 = 0.f, acc_c2 = 0.f;
  float last_n0 = 0.f, last_n1 = 0.f, last_n2 = 0.f, acc_n0 = 0.f, acc_n1 = 0.f, acc_n2 = 0.f;
  const float ddelx_dx = 0.5f * a.W, ddely_dy = 0.5f * a.H;
  double ray_x = 0.0, ray_y = 0.0;   // RAYS: this pixel's dL/drx, dL/dry

  // The 16 values of a pair's partial gradient g[] and of the accumulator row:
  //   0..9 -> dL_dview2gaussian[0..9] (9 = dL_dC also yields dL_dopacity = -2/opacity * that sum: both are
  //   G*dL_dalpha up to a per-Gaussian constant; dL_dC is the one carried through the reduction because the
  //   view2gaussian chain rule cancels it against the other nine to ~1e-5 and needs them rounded consistently),
  //   10..12 -> dL_dcolor, 13..15 -> dL_dmean2D

  // Batches are the forward's, taken from the deepest one the tile used down to 0; inside a batch the groups of 32 and the
  // bits inside a group are walked from high to low: back to front.
  for (int i = 0; i < rounds; ++i) {
    const int ib = rounds - 1 - i;
    const int base = ib * BATCH;
    __syncthreads();   // every warp has finished the previous batch: the buffer may be refilled
    if (base + (int)threadIdx.x < used) {
      const uint32_t g = a.point_list[range.x + (uint32_t)(base + (int)threadIdx.x)];
      const float4* src = reinterpret_cast<const float4*>(a.splat + g);
      const float4 r0 = __ldg(src), r1 = __ldg(src + 1), r2 = __ldg(src + 2), r3 = __ldg(src + 3);
      float4* dst = s_dyn + (size_t)threadIdx.x * 6;
      dst[0] = r0; dst[1] = r1; dst[2] = r2; dst[3] = r3;
      const float4* srcb = reinterpret_cast<const float4*>(a.splat_bwd + g);
      dst[4] = __ldg(srcb); dst[5] = __ldg(srcb + 1);
    }
    // the batch's masks, one coalesced 128-byte row per group as the forward wrote them.  The forward wrote the rows of every
    // group up to this warp's deepest contributor; nothing behind it blended, and the rows past it read as empty.
#pragma unroll
    for (int k = 0; k < GROUPS; ++k) {
      const int gstart = base + k * 32;
      s_mask[k * 32 + lane] = (uint32_t)gstart < warp_last ? __ldg(vm_row + gstart) : 0u;
    }
    __syncthreads();

    // the 16 partial gradients of ONE (pixel, Gaussian) pair: row = the staged record, contributor = its zero-based index in the
    // tile list (the reference's `contributor` after its decrement, backward.cu:763), contrib = this pixel blended it
    auto pair_grad = [&](const uint32_t row, const uint32_t contributor, const bool contrib, float (&g)[16]) {
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
        // Every sum of two products below names the product that is fused (F_FMA) and the one that is rounded (F_MUL), as
        // gof_math.cuh does for the forward: left to ptxas, the choice can change with any edit of this kernel, and the
        // view2gaussian chain rule turns the last-ulp difference into percents in dL_dscale / dL_drot.
        // colour, :824-837
        const float2 q3 = gof_lds64<48>(row);
        const float c0 = q2.w, c1 = q3.x, c2 = q3.y;
        const float one_m_last = 1.f - last_alpha;
        acc_c0 = F_FMA(last_alpha, last_c0, F_MUL(one_m_last, acc_c0)); last_c0 = c0;
        acc_c1 = F_FMA(last_alpha, last_c1, F_MUL(one_m_last, acc_c1)); last_c1 = c1;
        acc_c2 = F_FMA(last_alpha, last_c2, F_MUL(one_m_last, acc_c2)); last_c2 = c2;
        float dL_dalpha = F_FMA(c0 - acc_c0, dpix0, 0.f);
        dL_dalpha = F_FMA(c1 - acc_c1, dpix1, dL_dalpha);
        dL_dalpha = F_FMA(c2 - acc_c2, dpix2, dL_dalpha);
        g[10] = w * dpix0; g[11] = w * dpix1; g[12] = w * dpix2;
        // distortion: only the depth path survives ("detach weight", :848-858)
        const float dL_dmax_t = 2.0f * (T * alpha) * F_FMA(mt, final_A, -final_D) * dreg * dm_dt;
        // normal, :860-877
        acc_n0 = F_FMA(last_alpha, last_n0, F_MUL(one_m_last, acc_n0)); last_n0 = nn0;
        acc_n1 = F_FMA(last_alpha, last_n1, F_MUL(one_m_last, acc_n1)); last_n1 = nn1;
        acc_n2 = F_FMA(last_alpha, last_n2, F_MUL(one_m_last, acc_n2)); last_n2 = nn2;
        dL_dalpha = F_FMA(nn0 - acc_n0, dn0, dL_dalpha);
        dL_dalpha = F_FMA(nn1 - acc_n1, dn1, dL_dalpha);
        dL_dalpha = F_FMA(nn2 - acc_n2, dn2, dL_dalpha);
        const float dnn0 = w * dn0, dnn1 = w * dn1, dnn2 = w * dn2;
        const float dL_dlength = F_MUL(F_FMA(dnn2, p.n2, F_FMA(dnn0, p.n0, F_MUL(dnn1, p.n1))), F_MUL(rlen, rlen));
        const float dnrm0_l = F_FMA(dL_dlength, p.n0, -dnn0);   // before the factor rlen
        const float dnrm1_l = F_FMA(dL_dlength, p.n1, -dnn1);
        const float dnrm2_l = F_FMA(dL_dlength, p.n2, -dnn2);
        // :879-893
        float dL_dt = dL_dmax_t;
        if (contributor == max_contributor - 1u) dL_dt += ddepth;
        last_alpha = alpha;
        dL_dalpha = F_FMA(dL_dalpha, T, F_MUL(F_MUL(-T_final, r1a), bg_dot_dpixel));
        // :896-912  2D-mean statistic and opacity
        const float4 b0 = gof_lds128<64>(row);   // (mx, my, cx, cy)
        const float b1x = gof_lds32<80>(row);    // cz
        const float dx = b0.x - (float)pix_x, dy = b0.y - (float)pix_y;
        const float dL_dG = q2.z * dL_dalpha;
        const float gdx = G * dx, gdy = G * dy;
        const float dG_ddelx = F_FMA(-gdx, b0.z, -F_MUL(gdy, b0.w));
        const float dG_ddely = F_FMA(-gdy, b1x, -F_MUL(gdx, b0.w));
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
        const float dA = (float)D_FMA(D_MUL(D_MUL((double)dL_dmin, qd), qd), 0.25, -D_MUL(D_MUL((double)dL_dt, qd), inv2A));
        const float dB2 = (float)D_FMA((double)dL_dt, -rA, D_MUL((double)dL_dmin, qd));   // 2 * dL_dB
        // :938-952
        const float dnrm0 = F_FMA(dA, rx, F_MUL(dnrm0_l, rlen));
        const float dnrm1 = F_FMA(dA, ry, F_MUL(dnrm1_l, rlen));
        const float dnrm2 = F_FMA(dnrm2_l, rlen, dA);
        g[0] = dnrm0 * rx;
        g[1] = F_FMA(dnrm0, ry, F_MUL(dnrm1, rx));
        g[2] = F_FMA(dnrm2, rx, dnrm0);
        g[3] = dnrm1 * ry;
        g[4] = F_FMA(dnrm2, ry, dnrm1);
        g[5] = dnrm2;
        g[6] = dB2 * rx;
        g[7] = dB2 * ry;
        g[8] = dB2;
        if constexpr (RAYS) {
          // dL/drx = dnrm . dn/drx (n = M r, first column of M) + dA n0 (AA = r.n at fixed n) + dB2 v6 (BB), likewise for ry
          const float tx = F_FMA(dB2, v[6], F_FMA(dA, p.n0, F_FMA(dnrm2, v[2], F_FMA(dnrm1, v[1], F_MUL(dnrm0, v[0])))));
          const float ty = F_FMA(dB2, v[7], F_FMA(dA, p.n1, F_FMA(dnrm2, v[4], F_FMA(dnrm1, v[3], F_MUL(dnrm0, v[1])))));
          ray_x = D_ADD(ray_x, (double)tx);
          ray_y = D_ADD(ray_y, (double)ty);
        }
      }
    };

    // Each 4x2 pixel block (a quarter of the warp: the lanes that differ in bits 0, 1, 3) walks ITS OWN list -- the entries one
    // of its 8 pixels blended -- in lockstep with the other three: an iteration handles up to four different Gaussians, one per
    // quarter.  A Gaussian of pixel-scale footprint touches 16 of a warp's 32 pixels on average, so a warp-wide walk leaves
    // half of the lanes idle.  The lockstep spans the whole batch: a quarter whose group runs out moves on to its next
    // non-empty group while the others are still in theirs, so an iteration waits only for the quarter with the most entries
    // in the batch, not in each group of 32 (4.4 M instead of 4.9 M iterations for the same 93 M pairs at the benchmark
    // workload).  The partial gradients are reduced over the quarter (14 shuffles) and leave as two reds per lane; no red
    // carries dL_dopacity, which k_preprocess_backward forms as -2/opacity * sum(dL_dC).
    const uint32_t* const s_quarter = s_mask + (lane & 20);   // the words of this lane's quarter: + {0..3, 8..11} + 32*group
    // bit 4*group + quarter of `nonempty`: that quarter blended something in that group; lane l forms the bit of group l/4
    // and of the quarter whose first lane is ((l & 1) << 2) | ((l & 2) << 3)
    auto quarter_word = [](const uint32_t* w) {
      const uint4 x = *reinterpret_cast<const uint4*>(w), y = *reinterpret_cast<const uint4*>(w + 8);
      return x.x | x.y | x.z | x.w | y.x | y.y | y.z | y.w;
    };
    const uint32_t nonempty = __ballot_sync(0xffffffffu,
                                            quarter_word(s_mask + (lane >> 2) * 32 + ((lane & 1) << 2) + ((lane & 2) << 3)) != 0u);
    // the cursor: the groups still to visit (bit 4*group), the current group's first entry, the quarter's entries left in it
    // and this pixel's own mask of it
    uint32_t left = (nonempty >> (((lane >> 2) & 1) | ((lane >> 3) & 2))) & 0x11111111u;
    uint32_t first = 0u, qb = 0u, mybits = 0u;
    auto next_group = [&]() {
      if (left == 0u) return;
      const int hb = 31 - __clz(left);   // 4 * group
      left ^= 1u << hb;
      first = (uint32_t)hb * 8u;
      qb = quarter_word(s_quarter + first);
      mybits = s_mask[first + lane];
    };
    next_group();
    while (__any_sync(0xffffffffu, qb != 0u)) {
      const bool act = qb != 0u;
      const int b = act ? 31 - __clz(qb) : 0;
      if (act) qb &= ~(1u << b);
      const uint32_t row = s_base + (first + (uint32_t)b) * 96u;
      const bool contrib = act && ((mybits >> b) & 1u) != 0u;
      float g[16];
      pair_grad(row, (uint32_t)base + first + (uint32_t)b, contrib, g);
      float r0, r1;
      quarter_reduce16(g, lane, &r0, &r1);
      if (act) {
        const uint32_t gid = __float_as_uint(gof_lds32<84>(row));   // GofSplatBwd::self
        double* dst = a.grad_acc + ((size_t)gid * 16 + ((lane & 8) ? 1 : 0) + ((lane & 2) ? 2 : 0) + ((lane & 1) ? 4 : 0));
        if (r0 != 0.f) atomicAdd(dst, (double)r0);
        if (r1 != 0.f) atomicAdd(dst + 8, (double)r1);
      }
      if (qb == 0u) next_group();
    }
  }

  if constexpr (RAYS) {
    if (inside) { a.drays[pid] = ray_x; a.drays[HW + pid] = ray_y; }
    // the tile's sums of rx dL/drx and ry dL/dry: a fixed shuffle tree per warp, then the eight warps in order
    double sx = D_MUL((double)rx, ray_x), sy = D_MUL((double)ry, ray_y);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      sx = D_ADD(sx, __shfl_down_sync(0xffffffffu, sx, o));
      sy = D_ADD(sy, __shfl_down_sync(0xffffffffu, sy, o));
    }
    __syncthreads();   // every warp is done with the staged records: their buffer takes the warp sums
    double* const s_sum = reinterpret_cast<double*>(s_dyn);
    if (lane == 0) { s_sum[2 * warp] = sx; s_sum[2 * warp + 1] = sy; }
    __syncthreads();
    if (threadIdx.x < 2) {
      double t = s_sum[threadIdx.x];
#pragma unroll
      for (int w = 1; w < WARPS; ++w) t = D_ADD(t, s_sum[2 * w + threadIdx.x]);
      a.drays[2 * HW + 2 * (size_t)tile + threadIdx.x] = t;
    }
  }
}

// dL/dtan_fov from the tile sums of k_render_backward<true>: thread j adds tiles j, j + 1024, ... in index order, a fixed tree
// joins the threads, and each sum is divided by tan_fov and rounded to float once.  rx = (px + 0.5 - W/2) 2 tan_fovx / W, so
// d rx / d tan_fovx = rx / tan_fovx.
constexpr int FOCAL_SUM_THREADS = 1024;
__global__ void __launch_bounds__(FOCAL_SUM_THREADS) k_focal_grad_sum(int tiles, const double* __restrict__ partial, float tan_fovx,
                                                                        float tan_fovy, float* __restrict__ dL_dtan_fov) {
  __shared__ double s[2][FOCAL_SUM_THREADS];
  double sx = 0.0, sy = 0.0;
  for (int t = threadIdx.x; t < tiles; t += FOCAL_SUM_THREADS) {
    sx = D_ADD(sx, partial[2 * (size_t)t]);
    sy = D_ADD(sy, partial[2 * (size_t)t + 1]);
  }
  s[0][threadIdx.x] = sx;
  s[1][threadIdx.x] = sy;
  __syncthreads();
#pragma unroll
  for (int n = FOCAL_SUM_THREADS / 2; n > 0; n >>= 1) {
    if ((int)threadIdx.x < n) {
      s[0][threadIdx.x] = D_ADD(s[0][threadIdx.x], s[0][threadIdx.x + n]);
      s[1][threadIdx.x] = D_ADD(s[1][threadIdx.x], s[1][threadIdx.x + n]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    dL_dtan_fov[0] = (float)(s[0][0] / (double)tan_fovx);
    dL_dtan_fov[1] = (float)(s[1][0] / (double)tan_fovy);
  }
}

template <bool RAYS>
int carveout_once() {
  return gof_device_once((const void*)k_render_backward<RAYS>, [](int, int*) -> int {
    const int need = 4 * (SMEM_BYTES + 1024);   // only what the resident CTAs need: the rest stays L1
    GOF_CUDA_OK(cudaFuncSetAttribute(k_render_backward<RAYS>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                     (need * 100 + 233471) / 233472 > 100 ? 100 : (need * 100 + 233471) / 233472));
    return GOF_OK;
  }, nullptr);
}

}  // namespace

size_t gof_ray_grad_scratch_bytes(int W, int H) {
  if (W <= 0 || H <= 0) return 0;
  const size_t tiles = (size_t)((W + 15) / 16) * ((H + 15) / 16);
  return (2 * (size_t)W * H + 2 * tiles) * sizeof(double);
}

int gof_launch_render_backward(const gof_scene_t* s, const GofView& v, char* geom, const GofGeomLayout& GL,
                               const char* bin, const GofBinLayout& BL, const char* img, const GofImageLayout& IL,
                               const float* dL_dpix, double* rays, float* dL_dtan_fov, cudaStream_t st) {
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
  if (rays == nullptr) {
    const int rc = carveout_once<false>();
    if (rc != GOF_OK) return rc;
    GOF_LAUNCH("render_bwd", st, k_render_backward<false><<<v.tiles, GOF_BLOCK_SIZE, SMEM_BYTES, st>>>(a));
    GOF_LAUNCH_CHECK(s->debug, st);
    return GOF_OK;
  }
  a.drays = rays;
  const int rc = carveout_once<true>();
  if (rc != GOF_OK) return rc;
  GOF_LAUNCH("render_bwd_rays", st, k_render_backward<true><<<v.tiles, GOF_BLOCK_SIZE, SMEM_BYTES, st>>>(a));
  GOF_LAUNCH_CHECK(s->debug, st);
  GOF_LAUNCH("focal_grad_sum", st, k_focal_grad_sum<<<1, FOCAL_SUM_THREADS, 0, st>>>(v.tiles, rays + 2 * (size_t)v.W * v.H, s->tan_fovx,
                                                                                     s->tan_fovy, dL_dtan_fov));
  GOF_LAUNCH_CHECK(s->debug, st);
  return GOF_OK;
}
