// conv_wgrad.cu -- weight and bias gradient of a 3x3, stride-1, pad-1 convolution with few channels at full image resolution:
// the two convolutions at the tail of the reference's AppearanceNetwork (scene/appearance_network.py:28-29, 16 -> 16 and 16 -> 3
// channels at 1056x1920 in BASELINE config C4) and its last upsample block (8 -> 16 at half resolution).  Why hand-written:
// cuDNN answers these shapes with its generic fp32 `wgrad_alg0_engine`, which takes longer than the whole forward of the
// network.
//
// dW[co][ci][ky][kx] = sum_p gy[co][p] * x[ci][p + (ky-1, kx-1)] is a reduction over two million pixels into at most 2304
// numbers.  One thread owns COPT (co, ci) pairs and keeps their nine sums each in registers; persistent CTAs sweep 32x8 pixel
// tiles staged in shared memory; a 3x3 window of x slides along the row (3 + COPT shared loads per 9 COPT FMAs).  fp32
// accumulation (cuDNN's TF32 path rounds the products to 10 bits).
//
// The tile pipeline is what the time depends on (ncu of the first versions: 11 % issue utilisation, 23 warps per issue waiting on
// global loads -- a thread filled the tile through ~40 serialised DRAM round trips, and ptxas re-pairs every load with its store
// whatever the source order).  Now: two tile buffers, filled by cp.async (16-byte copies for the aligned 32-float interior of a
// row, 4-byte copies for the two halo columns, zero-filled outside the image) for tile t+1 while tile t is consumed; per-CTA
// partial sums are combined in shared memory before ONE global atomic per weight and CTA.
#include "gof_common.cuh"

namespace {

constexpr int TW = 32, TH = 8;   // pixel tile

__device__ __forceinline__ void cp16_zfill(uint32_t dst, const float* src, bool ok) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(ok ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp4_zfill(uint32_t dst, const float* src, bool ok) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(ok ? 4 : 0) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// Shared layout of one tile buffer.  PIPE (cp.async, 16-byte destinations): x rows of 40 floats -- element xx = 0..33 (image
// column x0 - 1 + xx) at row[3 + xx], so that the interior starts 16-byte aligned -- planes 404 floats apart; g rows of 36, planes
// 292 apart.  All pitches are multiples of 4, so the CI planes share 8 banks (two-way conflicts on the x loads; the odd pitches of
// the scalar layout are conflict-free but cannot take 16-byte copies).
template <int CO, int CI, bool PIPE>
struct TileLayout {
  static constexpr int XOFF = PIPE ? 3 : 0;
  static constexpr int XROW = PIPE ? 40 : TW + 3;
  static constexpr int XP = PIPE ? (TH + 2) * 40 + 4 : (TH + 2) * (TW + 3);
  static constexpr int GROW = PIPE ? 36 : TW + 1;
  static constexpr int GP = PIPE ? TH * 36 + 4 : TH * (TW + 1) + 1;
  static constexpr int FLOATS = CI * XP + CO * GP;
};

// the products of one tile: thread (ci, cog, rg) adds rows [rg*ROWS, rg*ROWS + ROWS) to its COPT x 9 sums
template <int CO, int CI, int COPT, int RG, bool PIPE>
__device__ __forceinline__ void tile_products(const float* s_x, const float* s_g, int ci, int cog, int rg, float (&acc)[COPT][9], float (&accb)[COPT]) {
  using L = TileLayout<CO, CI, PIPE>;
  constexpr int ROWS = TH / RG;
  const float* xs = s_x + ci * L::XP + L::XOFF;
  const float* gs = s_g + cog * COPT * L::GP;
#pragma unroll 1
  for (int yy = rg * ROWS; yy < rg * ROWS + ROWS; ++yy) {
    const float* r0 = xs + yy * L::XROW;
    const float* r1 = r0 + L::XROW;
    const float* r2 = r1 + L::XROW;
    float a0 = r0[0], a1 = r0[1], b0 = r1[0], b1 = r1[1], c0 = r2[0], c1 = r2[1];
#pragma unroll 8
    for (int xx = 0; xx < TW; ++xx) {
      const float a2 = r0[xx + 2], b2 = r1[xx + 2], c2 = r2[xx + 2];
#pragma unroll
      for (int j = 0; j < COPT; ++j) {
        const float g = gs[j * L::GP + yy * L::GROW + xx];
        acc[j][0] = fmaf(g, a0, acc[j][0]); acc[j][1] = fmaf(g, a1, acc[j][1]); acc[j][2] = fmaf(g, a2, acc[j][2]);
        acc[j][3] = fmaf(g, b0, acc[j][3]); acc[j][4] = fmaf(g, b1, acc[j][4]); acc[j][5] = fmaf(g, b2, acc[j][5]);
        acc[j][6] = fmaf(g, c0, acc[j][6]); acc[j][7] = fmaf(g, c1, acc[j][7]); acc[j][8] = fmaf(g, c2, acc[j][8]);
        if (ci == 0) accb[j] += g;
      }
      a0 = a1; a1 = a2; b0 = b1; b1 = b2; c0 = c1; c1 = c2;
    }
  }
}

// COPT output channels per thread, RG row groups per tile (so that small channel pairs still fill a CTA):
// THREADS = CO/COPT * CI * RG.  PIPE: W % 4 == 0 and 16-byte aligned planes (cp.async double buffer); otherwise one buffer, scalar loads.
template <int CO, int CI, int COPT, int RG, bool PIPE>
__global__ void __launch_bounds__((CO / COPT) * CI * RG) k_conv3x3_wgrad(const float* __restrict__ x, const float* __restrict__ gy, int H, int W,
                                                                          int tiles_x, int tiles, float* __restrict__ dW, float* __restrict__ db) {
  using L = TileLayout<CO, CI, PIPE>;
  constexpr int THREADS = (CO / COPT) * CI * RG;
  static_assert(CO % COPT == 0 && TH % RG == 0 && THREADS >= 64 && THREADS <= 1024 && TW == 32, "tile shape");
  static_assert(CO * CI * 9 + CO <= L::FLOATS, "the final partial sums reuse a tile buffer");
  extern __shared__ __align__(16) float s_tiles[];   // PIPE: two buffers of L::FLOATS, else one
  const int tid = threadIdx.x;
  const int ci = tid % CI, cog = (tid / CI) % (CO / COPT), rg = tid / (CI * (CO / COPT));
  float acc[COPT][9], accb[COPT];
#pragma unroll
  for (int j = 0; j < COPT; ++j) {
    accb[j] = 0.f;
#pragma unroll
    for (int k = 0; k < 9; ++k) acc[j][k] = 0.f;
  }
  const size_t HW = (size_t)H * W;

  if (PIPE) {
    const uint32_t s_base = (uint32_t)__cvta_generic_to_shared(s_tiles);
    auto fill = [&](int tile, int buf) {
      const int ty = tile / tiles_x, tx = tile - ty * tiles_x;
      const int y0 = ty * TH, x0 = tx * TW;
      const uint32_t sx = s_base + 4u * (uint32_t)(buf * L::FLOATS), sg = sx + 4u * (uint32_t)(CI * L::XP);
      constexpr int XG = CI * (TH + 2) * (TW / 4), XH = CI * (TH + 2) * 2, GG = CO * TH * (TW / 4);
      for (int g = tid; g < XG; g += THREADS) {   // interior: 8 x 16 bytes per row
        const int c = g / ((TH + 2) * (TW / 4)), r = g - c * ((TH + 2) * (TW / 4));
        const int yy = r / (TW / 4), k = r - yy * (TW / 4);
        const int iy = y0 + yy - 1, ix = x0 + 4 * k;
        const bool ok = iy >= 0 && iy < H && ix < W;
        cp16_zfill(sx + 4u * (uint32_t)(c * L::XP + yy * L::XROW + 4 + 4 * k), ok ? x + (size_t)c * HW + (size_t)iy * W + ix : x, ok);
      }
      for (int h = tid; h < XH; h += THREADS) {   // the two halo columns
        const int c = h / ((TH + 2) * 2), r = h - c * ((TH + 2) * 2);
        const int yy = r >> 1, side = r & 1;
        const int iy = y0 + yy - 1, ix = side ? x0 + TW : x0 - 1;
        const bool ok = iy >= 0 && iy < H && ix >= 0 && ix < W;
        cp4_zfill(sx + 4u * (uint32_t)(c * L::XP + yy * L::XROW + (side ? 4 + TW : 3)), ok ? x + (size_t)c * HW + (size_t)iy * W + ix : x, ok);
      }
      for (int g = tid; g < GG; g += THREADS) {
        const int c = g / (TH * (TW / 4)), r = g - c * (TH * (TW / 4));
        const int yy = r / (TW / 4), k = r - yy * (TW / 4);
        const int iy = y0 + yy, ix = x0 + 4 * k;
        const bool ok = iy < H && ix < W;
        cp16_zfill(sg + 4u * (uint32_t)(c * L::GP + yy * L::GROW + 4 * k), ok ? gy + (size_t)c * HW + (size_t)iy * W + ix : gy, ok);
      }
      cp_commit();
    };
    int tile = blockIdx.x, buf = 0;
    if (tile < tiles) fill(tile, 0);
    for (; tile < tiles; tile += gridDim.x, buf ^= 1) {
      const int next = tile + gridDim.x;
      if (next < tiles) { fill(next, buf ^ 1); cp_wait<1>(); } else { cp_wait<0>(); }   // this thread's copies of `tile` have landed
      __syncthreads();                                                                  // ... and everybody else's
      const float* sb = s_tiles + buf * L::FLOATS;
      tile_products<CO, CI, COPT, RG, true>(sb, sb + CI * L::XP, ci, cog, rg, acc, accb);
      __syncthreads();                                                                  // `buf` may be refilled (two iterations ahead)
    }
  } else {
    float* s_x = s_tiles;
    float* s_g = s_tiles + CI * L::XP;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
      const int ty = tile / tiles_x, tx = tile - ty * tiles_x;
      const int y0 = ty * TH, x0 = tx * TW;
      __syncthreads();
      constexpr int NX = CI * (TH + 2) * (TW + 2), NG = CO * TH * TW;
      for (int e = tid; e < NX; e += THREADS) {
        const int c = e / ((TH + 2) * (TW + 2)), r = e - c * ((TH + 2) * (TW + 2));
        const int yy = r / (TW + 2), xx = r - yy * (TW + 2);
        const int iy = y0 + yy - 1, ix = x0 + xx - 1;
        s_x[c * L::XP + yy * L::XROW + xx] = (iy >= 0 && iy < H && ix >= 0 && ix < W) ? __ldg(x + (size_t)c * HW + (size_t)iy * W + ix) : 0.f;
      }
      for (int e = tid; e < NG; e += THREADS) {
        const int c = e / (TH * TW), r = e - c * (TH * TW);
        const int iy = y0 + r / TW, ix = x0 + (r & (TW - 1));
        s_g[c * L::GP + (r / TW) * L::GROW + (r & (TW - 1))] = (iy < H && ix < W) ? __ldg(gy + (size_t)c * HW + (size_t)iy * W + ix) : 0.f;
      }
      __syncthreads();
      tile_products<CO, CI, COPT, RG, false>(s_x, s_g, ci, cog, rg, acc, accb);
    }
    __syncthreads();
  }

  // ---- the CTA's partial sums: row groups combined in shared memory, then one global atomic per weight ----
  float* s_sum = s_tiles;   // [CO*CI*9 | CO]; every thread is past the last tile barrier
  for (int i = tid; i < CO * CI * 9 + CO; i += THREADS) s_sum[i] = 0.f;
  __syncthreads();
#pragma unroll
  for (int j = 0; j < COPT; ++j) {
    const int co = cog * COPT + j;
#pragma unroll
    for (int k = 0; k < 9; ++k) atomicAdd(&s_sum[(co * CI + ci) * 9 + k], acc[j][k]);
    if (ci == 0) atomicAdd(&s_sum[CO * CI * 9 + co], accb[j]);
  }
  __syncthreads();
  for (int i = tid; i < CO * CI * 9; i += THREADS) atomicAdd(dW + i, s_sum[i]);
  if (db != nullptr)
    for (int i = tid; i < CO; i += THREADS) atomicAdd(db + i, s_sum[CO * CI * 9 + i]);
}

template <int CO, int CI, int COPT, int RG, bool PIPE>
int launch_v(const float* x, const float* gy, int H, int W, float* dW, float* db, cudaStream_t st) {
  constexpr int THREADS = (CO / COPT) * CI * RG;
  constexpr int SMEM = 4 * TileLayout<CO, CI, PIPE>::FLOATS * (PIPE ? 2 : 1);
  const int tiles_x = (W + TW - 1) / TW, tiles_y = (H + TH - 1) / TH, tiles = tiles_x * tiles_y;
  static int sms = 0, per_sm = 0;   // resident CTAs per SM of this instantiation: the persistent grid is exactly one wave
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
    GOF_CUDA_OK(cudaFuncSetAttribute(k_conv3x3_wgrad<CO, CI, COPT, RG, PIPE>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_conv3x3_wgrad<CO, CI, COPT, RG, PIPE>, THREADS, SMEM) != cudaSuccess || per_sm < 1)
      per_sm = 1;
  }
  const int grid = tiles < sms * per_sm ? tiles : sms * per_sm;
  GOF_LAUNCH("conv3x3_wgrad", st, (k_conv3x3_wgrad<CO, CI, COPT, RG, PIPE><<<grid, THREADS, SMEM, st>>>(x, gy, H, W, tiles_x, tiles, dW, db)));
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}

template <int CO, int CI, int COPT, int RG>
int launch(const float* x, const float* gy, int H, int W, float* dW, float* db, cudaStream_t st) {
  const bool pipe = (W & 3) == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(gy)) & 15u) == 0;
  return pipe ? launch_v<CO, CI, COPT, RG, true>(x, gy, H, W, dW, db, st) : launch_v<CO, CI, COPT, RG, false>(x, gy, H, W, dW, db, st);
}

}  // namespace

// x [CI,H,W], gy [CO,H,W] (contiguous fp32, batch 1) -> dW [CO,CI,3,3] and db [CO] (may be NULL), both ACCUMULATED INTO (zero them
// first).  Supported shapes: the channel pairs of the reference's AppearanceNetwork tail and its last upsample block.
extern "C" GOF_API int gof_conv3x3_wgrad(int CO, int CI, int H, int W, const float* x, const float* gy, float* dW, float* db, void* stream) {
  if (H <= 0 || W <= 0 || !x || !gy || !dW) { gof_set_error("conv3x3_wgrad: bad arguments"); return GOF_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  if (CO == 16 && CI == 16) return launch<16, 16, 4, 4>(x, gy, H, W, dW, db, st);
  if (CO == 3 && CI == 16) return launch<3, 16, 3, 8>(x, gy, H, W, dW, db, st);
  if (CO == 16 && CI == 8) return launch<16, 8, 4, 8>(x, gy, H, W, dW, db, st);
  gof_set_error("conv3x3_wgrad: unsupported channel pair %d -> %d", CI, CO);
  return GOF_E_INVALID;
}
