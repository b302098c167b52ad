// render_fwd.cu -- K6: per-tile front-to-back ray-Gaussian compositing (forward.cu:409-612).
//
// One 256-thread CTA per 16x16 tile.  Differences from the reference that do not change results:
//  * a warp covers an 8x4 pixel block (not a 16x2 strip) so the 32 rays of a warp are spatially compact;
//  * each (tile,Gaussian) instance is gathered as ONE 64-byte record (two sectors).  The per-tile slab is staged by the
//    copy engine: every thread issues one 64-byte cp.async.bulk (global -> shared, completing on the mbarrier of the
//    staging buffer) for its entry of batch i+1 while batch i is blended out of the other buffer (forward.cu:472-491 is a
//    load/store/__syncthreads loop).  No registers hold records in flight (a register double buffer costs 16 registers and
//    spills at 4 CTAs/SM) and a batch needs ONE CTA barrier instead of two.  ptxas issues a per-thread bulk copy from the
//    uniform datapath, one elected lane at a time (UBLKCP inside an ELECT loop, ~9 issue slots per record);
//  * every record carries a conservative pixel box of the region where its alpha can reach 1/255
//    (gof_cull_bbox); each warp ballots the 256 staged boxes against its own 8x4 pixel block and only visits
//    the Gaussians that can touch it;
//  * a conservative single-precision pre-test discards pairs whose alpha is provably < 1/255 before the
//    reference's double-precision evaluation; every pair that survives is evaluated with exactly the
//    reference's operation sequence (gof_math.cuh), so t, power, alpha, T -- everything a threshold or a
//    per-pixel counter depends on -- are bit-identical;
//  * the quantities that only feed float outputs (mapped depth of the distortion term, the normalised normal)
//    use cheaper evaluations accurate to ~1e-16 / 2e-7 instead of a double division, a double sqrt and three
//    IEEE float divisions per blended pair.
#include "gof_common.cuh"
#include "gof_math.cuh"

namespace {

struct FwdArgs {
  int W, H, grid_x;
  float focal_x, focal_y;
  const uint2* ranges;
  const uint32_t* point_list;
  const GofSplat* splat;
  const float* reject_k;   // GofGeomLayout::reject_k
  const float* bg;
  float* accum;        // [4][tiles*256] tile-major
  uint32_t* ncontrib;  // [2][tiles*256]
  float* out_color;    // [9][H][W]
  size_t plane;        // tiles*256
  uint32_t* vmask;     // blend masks for the backward (GofBinLayout::vmask)
  size_t vstride;
};

constexpr int BATCH = GOF_BLOCK_SIZE;

__global__ void __launch_bounds__(GOF_BLOCK_SIZE, 4) k_render_forward(const FwdArgs a) {
  // Rows of 80 bytes = the 64-byte record of a staged Gaussian + (K', -, -, -), K' = the reject constant (see
  // GofGeomLayout::reject_k).  One row base serves every load of a visit.  Two buffers (40 KB), filled by bulk copies.
  __shared__ __align__(128) float4 s_rec[2][BATCH][5];
  __shared__ __align__(8) unsigned long long s_bar[2];
  const uint32_t s_base = gof_smem_base(&s_rec[0][0][0]);
  const uint32_t bar0 = (uint32_t)__cvta_generic_to_shared(&s_bar[0]);

  const int tile = blockIdx.x;
  const int tile_x = tile % a.grid_x, tile_y = tile / a.grid_x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const GofWarpBlock blk = gof_warp_block(tile_x, tile_y, warp, lane);   // this warp's 8x4 pixel block and the lane's pixel
  const uint32_t pix_x = blk.pix_x, pix_y = blk.pix_y;
  const bool inside = pix_x < (uint32_t)a.W && pix_y < (uint32_t)a.H;
  bool done = !inside;

  const float rx = gof_ray(pix_x, a.W, a.focal_x);
  const float ry = gof_ray(pix_y, a.H, a.focal_y);

  const uint2 range = a.ranges[tile];
  const int total = (int)(range.y - range.x);
  uint32_t* vm_row = a.vmask + (size_t)warp * a.vstride + range.x + 32u * (uint32_t)tile + lane;   // + 32*group
  const int rounds = (total + BATCH - 1) / BATCH;

  float T = 1.0f;
  uint32_t last_contributor = 0, max_contributor = 0xFFFFFFFFu;
  float C0 = 0.f, C1 = 0.f, C2 = 0.f, N0 = 0.f, N1 = 0.f, N2 = 0.f, Dm = 0.f, Aacc = 0.f;
  float dist1 = 0.f, dist2 = 0.f, distortion = 0.f;

  // ---- staging ------------------------------------------------------------------------------------------------
  // meta_id / meta_k hold this thread's list entry of the batch that is issued NEXT.
  uint32_t meta_id = 0;
  float meta_k = 0.f;
  auto load_meta = [&](int batch) {
    const int e = batch * BATCH + (int)threadIdx.x;
    if (e < total) {
      meta_id = a.point_list[range.x + e];
      meta_k = __ldg(a.reject_k + meta_id);
    }
  };
  auto issue = [&](int batch) {
    const bool has = batch * BATCH + (int)threadIdx.x < total;
    const uint32_t row = s_base + (uint32_t)((batch & 1) * BATCH + (int)threadIdx.x) * 80u;
    // every thread arrives once per batch on the buffer's mbarrier; threads with an entry add 64 bytes
    const uint32_t bar = bar0 + 8u * (uint32_t)(batch & 1);
    if (has) {
      gof_mbar_arrive_expect_tx(bar, 64u);
      gof_bulk_g2s(row, a.splat + meta_id, 64u, bar);
      gof_sts32(row + 64u, meta_k);
    } else {
      gof_mbar_arrive(bar);
    }
  };
  if (threadIdx.x == 0) {
    gof_mbar_init(bar0, GOF_BLOCK_SIZE);
    gof_mbar_init(bar0 + 8u, GOF_BLOCK_SIZE);
    gof_mbar_init_fence();
  }
  __syncthreads();
  load_meta(0);
  issue(0);
  load_meta(1);

  int toDo = total;
  int i = 0;
  for (; i < rounds; ++i, toDo -= BATCH) {
    // forward.cu:475-477: stop when every pixel of the tile is saturated.  The barrier also says: every warp has finished
    // with the buffer of batch i-1, and the K' values of batch i (plain stores) are visible.
    if (__syncthreads_and(done)) break;
    const uint32_t buf_base = s_base + (uint32_t)(i & 1) * (uint32_t)(BATCH * 80);
    if (i + 1 < rounds) {
      issue(i + 1);        // lands while this batch is blended
      load_meta(i + 2);
    }

    const int nb = toDo < BATCH ? toDo : BATCH;
    if (__all_sync(0xffffffffu, done)) continue;   // this warp's 32 pixels are saturated (it still takes part in the staging)
    gof_mbar_wait(bar0 + 8u * (uint32_t)(i & 1), (uint32_t)(i >> 1) & 1u);   // batch i has landed

    // Sub-batches of 32: ballot which of these 32 staged Gaussians can reach this warp's 8x4 pixels at all, then
    // visit only those.  (The loop is deliberately NOT unrolled: the body is ~10 KB of SASS and eight copies
    // of it thrash the instruction cache -- ncu: 65 % of stall samples were "no instruction".)
#pragma unroll 1
    for (int k = 0; k < BATCH / 32; ++k) {
      if (k * 32 >= nb) break;
      const int idx = k * 32 + lane;
      const float4 qb = gof_lds128<48>(buf_base + (uint32_t)idx * 80u);
      uint32_t m = __ballot_sync(0xffffffffu, idx < nb && gof_box_hits(__float_as_uint(qb.z), __float_as_uint(qb.w), blk.wx0, blk.wy0, blk.wx0 + 7, blk.wy0 + 3));
      uint32_t mybits = 0u;   // bit b: this pixel blended entry k*32+b of the batch
      while (m != 0u) {
        const int b = __ffs(m) - 1;
        const int j = k * 32 + b;
        m &= m - 1;
        bool blended = false;
        if (!done) {
          const uint32_t contributor = (uint32_t)(i * BATCH + j + 1);   // 1-based position in the tile list
          const uint32_t row = buf_base + (uint32_t)j * 80u;
          const float4 q0 = gof_lds128<0>(row), q1 = gof_lds128<16>(row), q2 = gof_lds128<32>(row);
          const float v[10] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y};
          const GofPair p = gof_pair_geom(v, rx, ry);

          // ---- conservative reject (single precision, division-free): alpha < 1/255 is certain when
          // (B/2)^2 < A * K' with A > 0 (derivation and margins at GofGeomLayout::reject_k / k_preprocess) ----
          const float bh = 0.5f * p.BB;
          if (!(F_MUL(bh, bh) < F_MUL(p.AA, gof_lds32<64>(row)) && p.AA > 0.f)) {
            // ---- exact path: forward.cu:516-541 ----
            float t, power;
            gof_pair_t_power(p, v[9], &t, &power);
            if (!GOF_T_BEHIND_NEAR(t)) {
              const float alpha = fminf(F_MUL(q2.z, F_EXP(power)), GOF_ALPHA_MAX);
              if (!(alpha < GOF_ALPHA_MIN)) {
                const float test_T = F_MUL(T, F_SUB(1.0f, alpha));
                if (test_T < GOF_T_EPS) {
                  done = true;
                } else {
                  // forward.cu:543-578 (accumulation order = the reference's SASS: fma onto T)
                  const float mt = gof_mapped_t_fast(t);
                  const float rlen = gof_normal_rlen_fast(p);
                  const float nn0 = p.n0 * rlen, nn1 = p.n1 * rlen, nn2 = p.n2 * rlen;
                  const float A = F_SUB(1.0f, T);
                  const float m2 = F_MUL(mt, mt);
                  const float err = F_FMA(-dist1, F_ADD(mt, mt), F_FMA(A, m2, dist2));
                  distortion = F_FMA(T, F_MUL(err, alpha), distortion);
                  dist1 = F_FMA(T, F_MUL(alpha, mt), dist1);
                  dist2 = F_FMA(T, F_MUL(m2, alpha), dist2);
                  const float2 q3 = gof_lds64<48>(row);   // rgb1, rgb2
                  C0 = F_FMA(T, F_MUL(alpha, q2.w), C0);
                  C1 = F_FMA(T, F_MUL(alpha, q3.x), C1);
                  C2 = F_FMA(T, F_MUL(alpha, q3.y), C2);
                  N0 = F_FMA(-T, F_MUL(alpha, nn0), N0);
                  N1 = F_FMA(-T, F_MUL(alpha, nn1), N1);
                  N2 = F_FMA(-T, F_MUL(alpha, nn2), N2);
                  if (T > 0.5f) {
                    Dm = t;
                    max_contributor = contributor;
                  }
                  Aacc = F_FMA(T, alpha, Aacc);
                  T = test_T;
                  last_contributor = contributor;
                  blended = true;
                }
              }
            }
          }
        }
        if (blended) mybits |= 1u << b;
      }
      vm_row[i * BATCH + k * 32] = mybits;   // one coalesced 128-byte store per (warp, group): the backward's work list
    }
  }

  // a CTA must not exit with copies in flight towards its shared memory: after an early break batch i may still be landing
  if (i < rounds) gof_mbar_wait(bar0 + 8u * (uint32_t)(i & 1), (uint32_t)(i >> 1) & 1u);

  // forward.cu:584-611
  const size_t slot = (size_t)tile * 256 + threadIdx.x;
  a.accum[slot] = T;
  a.accum[a.plane + slot] = dist1;
  a.accum[2 * a.plane + slot] = dist2;
  a.accum[3 * a.plane + slot] = distortion;
  a.ncontrib[slot] = last_contributor;
  a.ncontrib[a.plane + slot] = max_contributor;
  if (inside) {
    const size_t HW = (size_t)a.H * a.W;
    const size_t pid = (size_t)pix_y * a.W + pix_x;
    const float omt = F_SUB(1.0f, T);
    const float dnorm = (float)D_DIV((double)distortion, D_ADD((double)F_MUL(omt, omt), 1e-7));
    a.out_color[0 * HW + pid] = F_FMA(T, a.bg[0], C0);
    a.out_color[1 * HW + pid] = F_FMA(T, a.bg[1], C1);
    a.out_color[2 * HW + pid] = F_FMA(T, a.bg[2], C2);
    a.out_color[3 * HW + pid] = N0;
    a.out_color[4 * HW + pid] = N1;
    a.out_color[5 * HW + pid] = N2;
    a.out_color[6 * HW + pid] = Dm;
    a.out_color[7 * HW + pid] = Aacc;
    a.out_color[8 * HW + pid] = dnorm;
  }
}

}  // namespace

int gof_launch_render_forward(const gof_scene_t* s, const GofView& v, const char* geom, const GofGeomLayout& GL,
                              char* bin, const GofBinLayout& BL, char* img, const GofImageLayout& IL,
                              float* out_color, cudaStream_t st) {
  FwdArgs a{};
  a.W = v.W; a.H = v.H; a.grid_x = v.grid_x; a.focal_x = v.focal_x; a.focal_y = v.focal_y;
  a.ranges = reinterpret_cast<const uint2*>(img + IL.ranges);
  a.point_list = reinterpret_cast<const uint32_t*>(bin + BL.point_list);
  a.splat = reinterpret_cast<const GofSplat*>(geom + GL.splat);
  a.reject_k = reinterpret_cast<const float*>(geom + GL.reject_k);
  a.bg = s->background;
  a.accum = reinterpret_cast<float*>(img + IL.accum);
  a.ncontrib = reinterpret_cast<uint32_t*>(img + IL.ncontrib);
  a.out_color = out_color;
  a.plane = (size_t)v.tiles * 256;
  a.vmask = reinterpret_cast<uint32_t*>(bin + BL.vmask);
  a.vstride = BL.vmask_stride;
  // 4 CTAs x (40 KB + 1 KB) per SM: ask for just that much shared memory -- the rest stays L1 (local-memory spills and the
  // mask / output traffic go through it)
  const int rc = gof_device_once((const void*)k_render_forward, [](int, int*) -> int {
    const int need = 4 * (2 * BATCH * 80 + 1024 + 64);
    GOF_CUDA_OK(cudaFuncSetAttribute(k_render_forward, cudaFuncAttributePreferredSharedMemoryCarveout,
                                     (need * 100 + 233471) / 233472 > 100 ? 100 : (need * 100 + 233471) / 233472));
    return GOF_OK;
  }, nullptr);
  if (rc != GOF_OK) return rc;
  GOF_LAUNCH("render_fwd", st, k_render_forward<<<v.tiles, GOF_BLOCK_SIZE, 0, st>>>(a));
  GOF_LAUNCH_CHECK(s->debug, st);
  return GOF_OK;
}
