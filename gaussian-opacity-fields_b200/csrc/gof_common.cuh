// gof_common.cuh -- private layouts, launch helpers and error plumbing shared by the .cu files.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/gof_rasterizer.h"

#define GOF_BLOCK_X 16
#define GOF_BLOCK_Y 16
#define GOF_BLOCK_SIZE 256

// ---- error plumbing -------------------------------------------------------------------------
void gof_set_error(const char* fmt, ...);

#define GOF_CUDA_OK(expr)                                                                      \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      gof_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e));     \
      return GOF_E_CUDA;                                                                       \
    }                                                                                          \
  } while (0)

// after every launch: always catch launch-configuration errors; with debug also synchronise and
// surface execution errors (reference: CHECK_CUDA, auxiliary.h:204-211)
#define GOF_LAUNCH_CHECK(debug, stream)                                                        \
  do {                                                                                         \
    cudaError_t _e = cudaGetLastError();                                                       \
    if (_e == cudaSuccess && (debug)) _e = cudaStreamSynchronize(stream);                      \
    if (_e != cudaSuccess) {                                                                   \
      gof_set_error("%s:%d: kernel failed -> %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return GOF_E_CUDA;                                                                       \
    }                                                                                          \
  } while (0)

// ---- launch accounting / per-kernel timing (gof_profile_* in the C ABI) ------------------------------------
// Every kernel launch goes through GOF_LAUNCH: it bumps the global launch counter and, when profiling is
// enabled, brackets the launch with CUDA events on the launching stream so bench.py can report per-kernel
// durations measured live (not under a profiler).
void gof_prof_begin(const char* name, cudaStream_t st);
void gof_prof_end(cudaStream_t st);
#define GOF_LAUNCH(name, st, ...)   \
  do {                              \
    gof_prof_begin(name, st);       \
    __VA_ARGS__;                    \
    gof_prof_end(st);               \
  } while (0)

// Small device->host readbacks (num_rendered, tet-mesh counters) land in a per-thread PINNED slot: a pageable
// destination turns cudaMemcpyAsync into a staged, driver-synchronised copy.  Returns nullptr if pinning failed.
void* gof_pinned_slot();   // 64 bytes
int gof_read_back(void* dst, const void* src_dev, size_t bytes, cudaStream_t st);   // copy + stream sync; GOF_OK / GOF_E_CUDA

// ---- per-device launch state (api.cu; safe to call from several host threads) ----------------------------------------
// SM count of the current device (132 if the query fails).
int gof_sm_count();
// Runs setup(device, &value) once per (current device, key) -- e.g. key = a kernel whose function attributes it sets -- and
// returns the value it left in *value (may be NULL).  A setup that does not return GOF_OK runs again on the next call.
// setup runs under the state's mutex and must not call these functions itself.
int gof_device_once(const void* key, int (*setup)(int dev, int* value), int* value);

// ---- shared-memory access with an explicit base register ----------------------------------------------
// On sm_90 and later a shared address carries the CTA's rank in its cluster; ptxas re-derives that window base
// (S2UR SR_CgaCtaId + UMOV + ULEA) next to every dynamically indexed access when registers are tight, which was
// 5-8 issue slots per visited Gaussian in the blend kernels.  gof_smem_base() turns the base into an opaque
// register value once; gof_lds* then compile to a bare LDS [R + imm].
#if defined(__CUDACC__)
__device__ __forceinline__ uint32_t gof_smem_base(const void* p) {
  uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("mov.u32 %0, %0;" : "+r"(a));
  return a;
}
template <int OFF>
__device__ __forceinline__ float4 gof_lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4+%5];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr), "n"(OFF) : "memory");
  return v;
}
template <int OFF>
__device__ __forceinline__ float2 gof_lds64(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0,%1}, [%2+%3];" : "=f"(v.x), "=f"(v.y) : "r"(addr), "n"(OFF) : "memory");
  return v;
}
template <int OFF>
__device__ __forceinline__ float gof_lds32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1+%2];" : "=f"(v) : "r"(addr), "n"(OFF) : "memory");
  return v;
}
// ---- bulk asynchronous copies (cp.async.bulk, the 1-D form of TMA) completing on an mbarrier -----------------------
// A tile's slab is an INDIRECT gather of 64-byte records, which a tensor-map copy cannot express; one 1-D bulk copy per
// record can: the copy engine moves the record global -> shared while the issuing thread carries on, and signals the
// mbarrier of the staging buffer with the bytes it delivered (complete_tx).  `bar` / `dst` are shared-window addresses.
__device__ __forceinline__ void gof_mbar_init(uint32_t bar, uint32_t arrivals) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(arrivals) : "memory");
}
__device__ __forceinline__ void gof_mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void gof_mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void gof_mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void gof_mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "GOF_MBAR_WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra GOF_MBAR_DONE_%=;\n"
      "bra GOF_MBAR_WAIT_%=;\n"
      "GOF_MBAR_DONE_%=:\n"
      "}\n" ::"r"(bar), "r"(parity) : "memory");
}
// orders this thread's earlier generic-proxy accesses to shared memory before later async-proxy (bulk copy) accesses
__device__ __forceinline__ void gof_fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void gof_bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
               "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void gof_sts32(uint32_t addr, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory"); }
__device__ __forceinline__ void gof_sts32u(uint32_t addr, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }

// 1/x, <= 1 ulp, no range guard (MUFU.RCP): for x known to be a normal number, or where inf/NaN are acceptable
__device__ __forceinline__ float gof_rcp_approx(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
// 1/x refined by one Newton step (error < 1 ulp for normal x)
__device__ __forceinline__ float gof_rcp_newton(float x) {
  const float r = gof_rcp_approx(x);
  return fmaf(r, fmaf(-x, r, 1.0f), r);
}
// 1/sqrt(x) refined by one Newton step (error ~1 ulp, like an IEEE sqrt followed by an IEEE reciprocal)
__device__ __forceinline__ float gof_rsqrt_newton(float x) {
  float y;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  const float e = fmaf(-x * y, y, 1.0f);
  return fmaf(0.5f * y, e, y);
}

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t n = __shfl_up_sync(0xffffffffu, v, d);
    if ((threadIdx.x & 31) >= d) v += n;
  }
  return v;
}

// block-wide exclusive scan of one value per thread (GOF_BLOCK_SIZE threads); total in *total.  Ends with a barrier.
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t* total) {
  constexpr int WARPS = GOF_BLOCK_SIZE / 32;
  __shared__ uint32_t s_warp[WARPS];
  __shared__ uint32_t s_total;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t incl = warp_incl_scan(v);
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    const uint32_t w = lane < WARPS ? s_warp[lane] : 0u;
    const uint32_t wi = warp_incl_scan(w);
    if (lane < WARPS) s_warp[lane] = wi - w;
    if (lane == WARPS - 1) s_total = wi;
  }
  __syncthreads();
  const uint32_t r = s_warp[warp] + incl - v;
  *total = s_total;
  __syncthreads();
  return r;
}
#endif

// ---- per-Gaussian records ---------------------------------------------------------------------
// One 64-byte, 64-byte-aligned record per Gaussian holds everything the forward blend gathers per
// (tile,Gaussian) instance: two 32-byte sectors instead of the reference's three unaligned gathers
// (conic_opacity 16 B + view2gaussian 40 B + rgb 12 B, forward.cu:483-489,561).
struct __align__(16) GofSplat {
  float v2g[10];   // view2gaussian quadric: Sigma(6) B(3) C(1)
  float opacity;   // conic_opacity.w = opacity * coef
  float rgb[3];    // SH colour (clamped) or colors_precomp
  uint32_t box_lo; // conservative pixel box of the alpha >= 1/255 region: int16 x0 | int16 y0 << 16
  uint32_t box_hi; //                                                       int16 x1 | int16 y1 << 16
};
static_assert(sizeof(GofSplat) == 64, "GofSplat must be 64 bytes");

// extra per-Gaussian data only the backward blend needs (backward.cu:748-749)
struct __align__(16) GofSplatBwd {
  float mx, my;          // means2D
  float cx, cy, cz;      // 2D conic (used for the densification statistic only)
  uint32_t self;         // this Gaussian's index (the backward blend reads it from the staged row: accumulator row address)
  float pad[2];
};
static_assert(sizeof(GofSplatBwd) == 32, "GofSplatBwd must be 32 bytes");

// ---- scratch layouts ----------------------------------------------------------------------------
static inline size_t gof_align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

#define GOF_SORT_ITEMS 16                              // keys per thread in a radix pass
#define GOF_SORT_CHUNK (GOF_BLOCK_SIZE * GOF_SORT_ITEMS) // keys per block in a radix pass
#define GOF_RADIX 256

static constexpr inline int gof_sort_blocks(size_t n) { return (int)((n + GOF_SORT_CHUNK - 1) / GOF_SORT_CHUNK); }

// Scratch of one radix sort of n pairs (binning.cu) in c = gof_sort_blocks(n) chunks of GOF_SORT_CHUNK keys: global digit
// histograms of up to 4 passes [4][256], 64 ticket/flag words, and per pass one decoupled-look-back status word per
// (chunk, digit), padded to whole groups of four chunks: at most 4 * (c + 7) * 256 words.
#define GOF_SORT_HEAD_BYTES (4 * GOF_RADIX * 4 + 256)
static constexpr inline size_t gof_sort_scratch_bytes(size_t n) {
  return (size_t)GOF_SORT_HEAD_BYTES + (size_t)4 * ((size_t)gof_sort_blocks(n) + 8) * GOF_RADIX * 4;
}

#define GOF_SCAN_ITEMS 8                               // values per thread of the single-launch exclusive scan
#define GOF_SCAN_CHUNK (GOF_BLOCK_SIZE * GOF_SCAN_ITEMS) // values per block of that scan

// Scratch (`tmp`, 8-byte aligned) of gof_exclusive_scan_u32 over n values: one 8-byte look-back status word per chunk of
// GOF_SCAN_CHUNK values and a ticket word, with slack.
static constexpr inline size_t gof_scan_scratch_bytes(size_t n) { return (n / GOF_SCAN_CHUNK + 4) * 8 + 4096; }

struct GofGeomLayout {      // "geomBuffer": everything sized by P
  size_t splat, splat_bwd, rect, tiles, clamped, depth;
  size_t key_a, key_b, val_a, val_b;   // depth radix sort ping-pong
  size_t hist;                         // radix sort scratch (gof_sort_scratch_bytes)
  size_t scan_tmp;                     // scan block sums / look-back status words
  size_t total;                        // u32 num_rendered (device copy)
  size_t grad_acc;                     // double[P][16]: backward accumulators of the blend kernel (dv2g[10], dcolor[3], dmean2D[3])
  size_t reject_k;                     // float[P]: K' = (C + 2 thr)(1 - 4e-7), thr = -ln(255 opacity) - 2e-3: a pair with (B/2)^2 < A K' has alpha < 1/255
  size_t bytes;
};

static inline GofGeomLayout gof_geom_layout(size_t P) {
  GofGeomLayout L;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o = gof_align_up(o + bytes, 256); return r; };
  L.splat = take(P * sizeof(GofSplat));
  L.splat_bwd = take(P * sizeof(GofSplatBwd));
  L.rect = take(P * 8);
  L.tiles = take(P * 4);
  L.clamped = take(P);
  L.depth = take(P * 4);
  L.key_a = take(P * 4);
  L.key_b = take(P * 4);
  L.val_a = take(P * 4);
  L.val_b = take(P * 4);
  L.hist = take(gof_sort_scratch_bytes(P));
  L.scan_tmp = take((P / 256 + 8) * 4 + 4096);      // look-back status words of the fused scan+emit kernel (one per 256 Gaussians) + ticket
  L.total = take(256);
  L.grad_acc = take(P * 128);
  L.reject_k = take(P * 4);
  L.bytes = o;
  return L;
}

struct GofImageLayout {     // "imgBuffer": per pixel + per tile
  size_t accum;      // float[4][tiles*256]  tile-major: T, dist1, dist2, raw distortion
  size_t ncontrib;   // u32  [2][tiles*256]  tile-major: last contributor, median contributor (integrate: contributors recorded)
  size_t ranges;     // uint2[tiles]
  size_t bytes;
};

static inline GofImageLayout gof_image_layout(int W, int H) {
  const size_t tiles = (size_t)((W + 15) / 16) * ((H + 15) / 16);
  GofImageLayout L;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o = gof_align_up(o + bytes, 256); return r; };
  L.accum = take(tiles * 256 * 4 * 4);
  L.ncontrib = take(tiles * 256 * 2 * 4);
  L.ranges = take(tiles * 8);
  L.bytes = o;
  return L;
}

struct GofBinLayout {       // "binningBuffer": everything sized by R = num_rendered
  size_t key_a, key_b;      // tile ids (u16 when tiles <= 65536, else u32)
  size_t val_a, val_b;      // Gaussian ids
  size_t hist;
  int key_bytes;
  int passes;               // number of radix passes over the tile id
  int bits[4];              // digit widths, low digit first
  size_t point_list;        // offset of the final sorted Gaussian-id list (val_a or val_b)
  size_t sorted_keys;       // offset of the final sorted tile-id list
  size_t vmask_stride;      // = R + 32 * tiles (u32 elements per warp plane)
  size_t vmask;             // u32[8][R + 32*tiles]: blend masks left by k_render_forward for the backward.  A tile's list is
                            // cut into groups of 32 entries; for warp w, group g of tile t, lane l the word at
                            // w*stride + ranges[t].x + 32*t + 32*g + l holds, bit b, "pixel l blended entry 32*g+b".
                            // (32 words of slack per tile: its last group may be partial)
  size_t bytes;
};

static inline int gof_bits_for(uint32_t n) {   // bits needed to represent values < n
  int b = 0;
  while ((1ull << b) < (unsigned long long)n) ++b;
  return b < 1 ? 1 : b;
}

// with_masks = false: the opacity-field query's binning buffer carries no blend masks (its backward recomputes its
// contributor lists instead)
static inline GofBinLayout gof_bin_layout(size_t R, int W, int H, bool with_masks = true) {
  const uint32_t tiles = (uint32_t)((W + 15) / 16) * (uint32_t)((H + 15) / 16);
  GofBinLayout L;
  const int nbits = gof_bits_for(tiles);
  L.key_bytes = tiles <= 65536u ? 2 : 4;
  L.passes = (nbits + 7) / 8;
  int rem = nbits;
  for (int p = 0; p < 4; ++p) L.bits[p] = 0;
  for (int p = 0; p < L.passes; ++p) {   // split as evenly as possible (e.g. 13 -> 7 + 6)
    int b = (rem + (L.passes - p) - 1) / (L.passes - p);
    L.bits[p] = b;
    rem -= b;
  }
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o = gof_align_up(o + bytes, 256); return r; };
  L.key_a = take(R * L.key_bytes);
  L.key_b = take(R * L.key_bytes);
  L.val_a = take(R * 4);
  L.val_b = take(R * 4);
  L.hist = take(gof_sort_scratch_bytes(R));
  L.point_list = (L.passes % 2 == 0) ? L.val_a : L.val_b;
  L.sorted_keys = (L.passes % 2 == 0) ? L.key_a : L.key_b;
  L.vmask_stride = R + 32 * (size_t)tiles;
  L.vmask = with_masks ? take(L.vmask_stride * 32) : o;
  L.bytes = o;
  return L;
}

// ---- launch prototypes (one per .cu) ----------------------------------------------------------------
struct GofView {           // host-side derived constants
  int W, H, grid_x, grid_y, tiles;
  float focal_x, focal_y;
};

static inline GofView gof_make_view(const gof_scene_t* s) {
  GofView v;
  v.W = s->width; v.H = s->height;
  v.grid_x = (s->width + 15) / 16; v.grid_y = (s->height + 15) / 16;
  v.tiles = v.grid_x * v.grid_y;
  v.focal_y = s->height / (2.0f * s->tan_fovy);   // rasterizer_impl.cu:274-275
  v.focal_x = s->width / (2.0f * s->tan_fovx);
  return v;
}

// preprocess.cu
// box_margin: see gof_cull_bbox (0 when the records feed the blend kernels, 0.5 when they feed k_integrate)
int gof_launch_preprocess(const gof_scene_t* s, const GofView& v, char* geom, const GofGeomLayout& L,
                          int* radii, float box_margin, cudaStream_t st);
// The accumulator rows in geom -> the outputs in o (checked by the caller)
int gof_launch_preprocess_backward(const gof_scene_t* s, const char* geom, const GofGeomLayout& L, const int* radii,
                                   const gof_backward_out_t& o, cudaStream_t st);
// bytes of o.scratch for the camera-gradient pass (o.dL_dviewmatrix non-NULL): it leaves one partial row per CTA there
size_t gof_camera_grad_scratch_bytes(int P);
int gof_launch_mark_visible(int P, const float* means3D, const float* vm, unsigned char* present,
                            cudaStream_t st);

// binning.cu
// A sort key of 1-3 u32 words per item: w[0] is the least significant word, and only the low bits[k] (1..32) bits of w[k]
// count.
struct GofKeyWords {
  const uint32_t* w[3];
  int bits[3];
  int nw;
};
// Buffers of gof_sort_words_u32 over n items, carved by the caller: ka, kb, va, vb n u32 each, hist gof_sort_scratch_bytes(n).
// The sort never writes the key words, except w[0] when the caller made it ka; no other word may be one of these buffers.
struct GofSortBufs { uint32_t *ka, *kb, *va, *vb, *hist; };
// Stable sort of the items 0..n-1 by `key`: leaves ord[j] = the item at sorted position j in `ord`, which is va or vb.
// n < 2^30 (the radix passes count items in 30-bit fields); a larger n fails with GOF_E_INVALID before any work is enqueued.
int gof_sort_words_u32(const GofKeyWords& key, size_t n, const GofSortBufs& b, uint32_t* ord, bool debug, cudaStream_t st);
// Runs of equal keys along ord: head[j] = 1 where the key of ord[j] differs from that of ord[j - 1] (head[0] = 1), run[j] = the
// exclusive scan of head, *num_runs (device) = the number of runs.  scan_tmp: gof_scan_scratch_bytes(n).
int gof_key_runs_u32(const GofKeyWords& key, const uint32_t* ord, size_t n, uint32_t* head, uint32_t* run, uint32_t* scan_tmp,
                     uint32_t* num_runs, bool debug, cudaStream_t st);
// exclusive scan of n u32 (in != out allowed); total (if non-NULL, device) receives the sum; tmp: gof_scan_scratch_bytes(n),
// 8-byte aligned.  Offsets and total are exact while the sum stays below 2^32 and wrap mod 2^32 beyond.
int gof_exclusive_scan_u32(const uint32_t* in, uint32_t* out, uint32_t* tmp, uint32_t* total, size_t n, bool debug, cudaStream_t st);
// The depth sort, the tile binning (R = the number of (tile, Gaussian) instances) and the point sort share the radix passes'
// limit: P, R and n below 2^30, or GOF_E_INVALID.
int gof_depth_sort(int P, char* geom, const GofGeomLayout& L, bool debug, cudaStream_t st);
int gof_bin_tiles(int P, size_t R, const GofView& v, char* geom, const GofGeomLayout& GL, char* bin,
                  const GofBinLayout& BL, char* img, const GofImageLayout& IL, bool debug, cudaStream_t st);
int gof_sort_points_by_tile(size_t n, int nbits, int key_shift, uint32_t* ka, uint32_t* kb, uint32_t* va, uint32_t* vb, uint32_t* hist,
                            uint2* ranges, int num_tiles, bool debug, cudaStream_t st);
// *result_in_b of a radix sort of n > 0 pairs over nbits key bits (gof_sort_points_by_tile, gof_bin_tiles): 1 when the sorted pairs
// end in the b buffers
int gof_radix_result_in_b(int nbits);

// integrate.cu
struct GofPointLayout { size_t xy, depth, bytes; };
struct GofPointBinLayout { size_t key_a, key_b, val_a, val_b, hist, pranges, ids, bytes; int nblk; };
static inline GofPointLayout gof_point_layout(size_t PN) {
  GofPointLayout L; size_t o = 0;
  auto take = [&](size_t b) { size_t r = o; o = gof_align_up(o + b, 256); return r; };
  L.xy = take(PN * 8); L.depth = take(PN * 4); L.bytes = o; return L;
}
#define GOF_INT_MAX_CONTRIB 1024   // MAX_NUM_CONTRIBUTORS * 4 (auxiliary.h:26, forward.cu:879)
static inline GofPointBinLayout gof_point_bin_layout(size_t PN, int tiles, int sm_count) {
  GofPointBinLayout L; size_t o = 0;
  auto take = [&](size_t b) { size_t r = o; o = gof_align_up(o + b, 256); return r; };
  L.key_a = take(PN * 4); L.key_b = take(PN * 4); L.val_a = take(PN * 4); L.val_b = take(PN * 4);
  L.hist = take(gof_sort_scratch_bytes(PN));
  L.pranges = take((size_t)(tiles + 1) * 8);
  L.nblk = tiles < sm_count * 3 ? tiles : sm_count * 3;
  if (L.nblk < 1) L.nblk = 1;
  L.ids = take((size_t)L.nblk * 256 * GOF_INT_MAX_CONTRIB * 2);
  L.bytes = o; return L;
}
// mn != NULL: the running minimum over views (gof_integrate_min, DESIGN.md 4.12) instead of the query's outputs, which are not read
struct GofIntMin {
  float* alpha_min;   // [PN]
  int* argmin;        // [PN]
  int view;
  float* color_min;   // [PN][3] or NULL: also the winning view's colour (gof_integrate_min's color_min, DESIGN.md 4.13)
};
int gof_launch_integrate(const gof_scene_t* s, const GofView& v, int PN, const float* points3D, const GofSplat* splat,
                         const uint32_t* point_list, const uint2* ranges, char* img, char* pts, char* pbin, float* out_color,
                         float* out_alpha, float* out_color_int, const GofIntMin* mn, cudaStream_t st);
// The backward of the query (DESIGN.md 4.11) from the state gof_launch_integrate left in geom / pts / pbin: dL_dalpha [PN] ->
// dL_dpoints3D [PN][3] (optional) and, through the accumulator rows and k_preprocess_backward, the Gaussian gradients.  The
// contributor slab in pbin and the accumulator rows in geom are rewritten.  o.scratch: gof_integrate_backward_scratch(P) bytes.
// o.dL_dcolor NULL: the alpha-only backward (no SH chain).  Otherwise (DESIGN.md 4.13) dL_dcolor_int [PN][3] (NULL: no colour
// loss) also goes through the colour walk, dL_dalpha may be NULL, and o.dL_dcolor [P][3] / o.dL_dsh receive the colour's chain.
size_t gof_integrate_backward_scratch(int P);
int gof_launch_integrate_backward(const gof_scene_t* s, const GofView& v, int PN, const float* points3D, const int* radii,
                                  char* geom, const GofGeomLayout& GL, const uint32_t* point_list, const uint2* ranges, const char* pts,
                                  char* pbin, const float* dL_dalpha, const float* dL_dcolor_int, float* dL_dpoints3D,
                                  const gof_backward_out_t& o, cudaStream_t st);

// Per-view cache of the Gaussian side of the opacity-field query (gof_integrate_prepare / gof_integrate_cached): the records,
// the tile ranges and the per-tile Gaussian lists are all a query needs, and they do not depend on the query points.
struct GofIntCacheLayout { size_t splat, ranges, point_list, bytes; };
static inline GofIntCacheLayout gof_int_cache_layout(size_t P, int W, int H, size_t R) {
  const size_t tiles = (size_t)((W + 15) / 16) * ((H + 15) / 16);
  GofIntCacheLayout L; size_t o = 0;
  auto take = [&](size_t b) { size_t r = o; o = gof_align_up(o + b, 256); return r; };
  L.splat = take(P * sizeof(GofSplat)); L.ranges = take(tiles * 8); L.point_list = take(R * 4); L.bytes = o;
  return L;
}

// render_fwd.cu / render_bwd.cu
int gof_launch_render_forward(const gof_scene_t* s, const GofView& v, const char* geom,
                              const GofGeomLayout& GL, char* bin, const GofBinLayout& BL, char* img,
                              const GofImageLayout& IL, float* out_color, cudaStream_t st);
int gof_launch_render_backward(const gof_scene_t* s, const GofView& v, char* geom,
                               const GofGeomLayout& GL, const char* bin, const GofBinLayout& BL,
                               const char* img, const GofImageLayout& IL, const float* dL_dpix, double* rays,
                               float* dL_dtan_fov, cudaStream_t st);
// bytes of `rays` above: the ray-gradient pass (rays non-NULL) leaves [2][H][W] per-pixel dL/dr and [tiles][2] tile sums there,
// and writes dL_dtan_fov [2]
size_t gof_ray_grad_scratch_bytes(int W, int H);
