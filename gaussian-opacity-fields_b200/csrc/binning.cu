// binning.cu -- tile binning without the reference's 64-bit global sort, one launch per radix pass.
//
// The reference emits one (tile<<32 | depth_bits, gaussian) pair per (Gaussian,tile) instance and runs
// cub::DeviceRadixSort over 32+log2(tiles) bits of R instances (rasterizer_impl.cu:70-111, 355-363:
// 6 passes x 24 B x R at 1080p), plus cub::DeviceScan and identifyTileRanges.  The order it defines is
// (tile, depth bits, Gaussian index) because the radix sort is stable and instances are emitted in ascending
// Gaussian index.  The SAME order (bit-exact point_list / ranges) is produced here by splitting the key LSD-style:
//   1. stable radix sort of the P Gaussians by depth bits (4 x 8-bit passes over P pairs),
//   2. ONE kernel scans tiles_touched in that order (decoupled look-back across CTAs) and emits the instances
//      (tile id, gaussian) -- flattened so that every thread writes one instance -- and counts the tile-sort digits,
//   3. stable radix sort of the R instances by tile id only (13 bits at 1080p -> 2 passes, u16 keys),
//   4. tile ranges from the sorted tile ids (rasterizer_impl.cu:149-171).
// Every radix pass is ONE kernel ("onesweep"): a CTA ranks its 4096 keys (per-warp __match_any_sync ranks -> stable),
// obtains the number of keys with the same digit in all earlier chunks by decoupled look-back over single-word
// (flag | count) status entries, reorders the chunk in shared memory and writes digit runs coalesced.  Positions are a
// pure function of the input (no atomic decides an output position; the only atomic hands out chunk numbers in launch
// order so that a chunk never waits for one that has not started).  This replaced a design with histogram + row scan +
// scatter launches per pass and a three-kernel scan: 26 launches and 0.44 ms at the benchmark workload, against 10 launches
// and 0.25 ms (DESIGN §4.1); that code is in the repository history.
// The same passes sort the wider keys of the extraction paths (tetmesh, TSDF, kNN): gof_sort_words_u32 sorts by a key of up
// to three u32 words, one stable sort per word on the previous word's order, and gof_key_runs_u32 numbers the runs of equal
// keys in that order.
#include "gof_common.cuh"

namespace {

constexpr int THREADS = GOF_BLOCK_SIZE;              // 256
constexpr int WARPS = THREADS / 32;
constexpr uint32_t LB_AGG = 1u << 30;                // status word = flag (2 bits) | count (30 bits): written and read as ONE word
constexpr uint32_t LB_INC = 2u << 30;
constexpr uint32_t LB_VAL = (1u << 30) - 1u;
// The radix passes and the scan + emit kernel count at most n items per status word: their sizes stay below 2^30.
constexpr size_t LB_MAX_ITEMS = (size_t)1 << 30;

__device__ __forceinline__ uint32_t ld_volatile(const uint32_t* p) { return *reinterpret_cast<const volatile uint32_t*>(p); }
__device__ __forceinline__ void st_volatile(uint32_t* p, uint32_t v) { *reinterpret_cast<volatile uint32_t*>(p) = v; }
__device__ __forceinline__ uint64_t ld_volatile(const uint64_t* p) { return *reinterpret_cast<const volatile uint64_t*>(p); }
__device__ __forceinline__ void st_volatile(uint64_t* p, uint64_t v) { *reinterpret_cast<volatile uint64_t*>(p) = v; }

// Look-back status words.  u32: flag in bits 30-31, a 30-bit count (the radix passes and the scan + emit kernel, whose
// counts stay below 2^30).  u64: flag in the high half, the full u32 running total in the low half (the general scan, whose
// totals may reach 2^32 - 1); 8-byte aligned, so one load or store moves flag and value together.
template <typename W> struct LbWord;
template <> struct LbWord<uint32_t> {
  static constexpr int SHIFT = 30;
  static constexpr uint32_t VAL = LB_VAL;
};
template <> struct LbWord<uint64_t> {
  static constexpr int SHIFT = 32;
  static constexpr uint64_t VAL = 0xffffffffull;
};

// Decoupled look-back: a chunk publishes its aggregate in a status word (flag | count, written and read as ONE word), walks
// back over its predecessors' words until one carries an inclusive prefix, then publishes its own inclusive prefix.
// Warp-wide variant for the scans (one running quantity per chunk, thousands of chunks in flight): the 32 lanes of a warp
// fetch 32 consecutive predecessors in one coalesced request, so a walk over k predecessors costs k/32 dependent round
// trips.  Called by ALL lanes of one warp; every lane returns the exclusive prefix.
template <typename W>
__device__ __forceinline__ uint32_t lookback_warp(W* status, uint32_t chunk, uint32_t aggregate) {
  constexpr int S = LbWord<W>::SHIFT;
  constexpr W AGG = (W)1 << S, INC = (W)2 << S;
  const int lane = threadIdx.x & 31;
  if (lane == 0) st_volatile(status + chunk, (chunk == 0 ? INC : AGG) | (W)aggregate);
  uint32_t excl = 0u;
  int64_t pos = (int64_t)chunk;   // entries [0, pos) still to be examined; lane 0 takes the nearest
  while (pos > 0) {
    const int64_t idx = pos - 1 - lane;
    W w;
    do {
      w = idx >= 0 ? ld_volatile(status + idx) : INC;   // in front of chunk 0: an inclusive prefix of zero
    } while (__any_sync(0xffffffffu, (w >> S) == 0u));
    const uint32_t inc = __ballot_sync(0xffffffffu, (w >> S) == 2u);
    const int first = inc ? __ffs(inc) - 1 : 31;       // nearest predecessor carrying an inclusive prefix
    uint32_t v = lane <= first ? (uint32_t)(w & LbWord<W>::VAL) : 0u;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    excl += v;
    if (inc) break;
    pos -= 32;
  }
  if (lane == 0 && chunk != 0) st_volatile(status + chunk, INC | (W)(excl + aggregate));
  return excl;
}

// The same for the radix passes, where 256 digits look back at once: one 128-bit volatile load fetches the status words of four
// consecutive predecessors.  With all chunks of a pass resident at the same time a chunk has to walk back over about half of
// its predecessors before it meets an inclusive prefix; four at a time quarters the number of dependent L2 round trips.
__device__ __forceinline__ uint4 ld_volatile_v4(const uint32_t* p) {
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
// Status words of the radix passes: word (chunk c, digit d) lives at ((c >> 2) * 256 + d) * 4 + (c & 3) -- the four chunks of
// a group are the four lanes of ONE 128-bit word per digit, and the 256 digits of a group are contiguous, so the 32 threads of
// a warp (32 digits) poll 512 contiguous bytes per round trip.
__device__ __forceinline__ void lookback_digit_publish(uint32_t* status, uint32_t digit, uint32_t chunk, uint32_t aggregate) {
  st_volatile(status + ((size_t)(chunk >> 2) * GOF_RADIX + digit) * 4 + (chunk & 3u), (chunk == 0 ? LB_INC : LB_AGG) | aggregate);
}
__device__ __forceinline__ uint32_t lookback_digit_walk(uint32_t* status, uint32_t digit, uint32_t chunk, uint32_t aggregate) {
  uint32_t* own = status + ((size_t)(chunk >> 2) * GOF_RADIX + digit) * 4 + (chunk & 3u);
  if (chunk == 0) return 0u;
  uint32_t excl = 0u;
  uint32_t pos = chunk;   // chunks [0, pos) are still to be examined, from the top
  while (pos > 0) {
    const uint32_t g = (pos - 1u) >> 2;
    const uint32_t need = pos - 4u * g;   // lanes 0 .. need-1 of this group
    const uint32_t* word = status + ((size_t)g * GOF_RADIX + digit) * 4;
    uint4 w;
    bool ready;
    do {
      w = ld_volatile_v4(word);
      ready = (w.x >> 30) != 0u && (need < 2u || (w.y >> 30) != 0u) && (need < 3u || (w.z >> 30) != 0u) && (need < 4u || (w.w >> 30) != 0u);
    } while (!ready);
    const uint32_t e[4] = {w.x, w.y, w.z, w.w};
    bool done = false;
#pragma unroll
    for (int i = 3; i >= 0; --i) {
      if (!done && (uint32_t)i < need) {
        excl += e[i] & LB_VAL;
        if ((e[i] >> 30) == 2u) done = true;
      }
    }
    if (done) break;
    pos = 4u * g;
  }
  st_volatile(own, LB_INC | (excl + aggregate));
  return excl;
}

// ------------------------------------------------------------------------------------------------
// global digit histograms of up to 4 passes in one sweep over the keys (the depth sort and the generic sorts; the tile
// sort's digits are counted by the emit kernel)
struct Digits { int shift[4]; uint32_t mask[4]; int passes; };

template <typename KeyT>
__global__ void __launch_bounds__(THREADS) k_digit_hist(const KeyT* __restrict__ keys, size_t n, Digits dg, uint32_t* __restrict__ ghist) {
  __shared__ uint32_t s_h[4][GOF_RADIX];
#pragma unroll
  for (int p = 0; p < 4; ++p) s_h[p][threadIdx.x] = 0;
  __syncthreads();
  const size_t stride = (size_t)gridDim.x * THREADS;
  for (size_t i = (size_t)blockIdx.x * THREADS + threadIdx.x; i < n; i += stride) {
    const uint32_t k = (uint32_t)keys[i];
#pragma unroll
    for (int p = 0; p < 4; ++p)
      if (p < dg.passes) atomicAdd(&s_h[p][(k >> dg.shift[p]) & dg.mask[p]], 1u);
  }
  __syncthreads();
#pragma unroll
  for (int p = 0; p < 4; ++p)
    if (p < dg.passes && s_h[p][threadIdx.x]) atomicAdd(ghist + p * GOF_RADIX + threadIdx.x, s_h[p][threadIdx.x]);
}

// ------------------------------------------------------------------------------------------------
// One stable LSD radix pass in one launch.  Chunk c = keys [c*4096, (c+1)*4096); warp w of the CTA owns a contiguous
// 1/8 of it, 32 keys per round: (chunk, warp, round, lane) order == input order, ranks within a digit follow it.
template <typename KeyT>
__global__ void __launch_bounds__(THREADS, 3) k_onesweep(const KeyT* __restrict__ keys_in, const uint32_t* __restrict__ vals_in,
                                                        KeyT* __restrict__ keys_out, uint32_t* __restrict__ vals_out, size_t n,
                                                        int shift, uint32_t mask, const uint32_t* __restrict__ ghist,
                                                        uint32_t* __restrict__ status /* see lookback_digit */,
                                                        uint32_t* __restrict__ ticket) {
  __shared__ uint32_t s_cnt[WARPS][GOF_RADIX];   // per-warp digit counters -> exclusive offsets over the warps
  __shared__ uint32_t s_gbase[GOF_RADIX];        // global position of this chunk's first key of each digit
  __shared__ uint32_t s_lbase[GOF_RADIX];        // chunk-local position of the first key of each digit
  __shared__ KeyT s_keys[GOF_SORT_CHUNK];
  __shared__ uint32_t s_vals[GOF_SORT_CHUNK];
  __shared__ uint32_t s_chunk;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_chunk = atomicAdd(ticket, 1u);   // chunk numbers follow launch order: predecessors are running
#pragma unroll
  for (int w = 0; w < WARPS; ++w) s_cnt[w][threadIdx.x] = 0;
  uint32_t dig_total;
  const uint32_t gstart = block_excl_scan(threadIdx.x <= mask ? ghist[threadIdx.x] : 0u, &dig_total);   // barrier inside
  const uint32_t chunk = s_chunk;
  const size_t cbase = (size_t)chunk * GOF_SORT_CHUNK;
  const size_t wbase = cbase + (size_t)warp * (GOF_SORT_ITEMS * 32);

  KeyT key[GOF_SORT_ITEMS];
  uint32_t rank[GOF_SORT_ITEMS];
  // all 16 key loads of the thread are issued before the first one is used
#pragma unroll
  for (int r = 0; r < GOF_SORT_ITEMS; ++r) {
    const size_t i = wbase + (size_t)r * 32 + lane;
    key[r] = i < n ? keys_in[i] : (KeyT)0;
  }
  const uint32_t lt = (1u << lane) - 1u;
#pragma unroll
  for (int r = 0; r < GOF_SORT_ITEMS; ++r) {
    const size_t i = wbase + (size_t)r * 32 + lane;
    const bool valid = i < n;
    const uint32_t d = valid ? (((uint32_t)key[r] >> shift) & mask) : (uint32_t)GOF_RADIX;   // sentinel digit for the ragged tail
    const uint32_t peers = __match_any_sync(0xffffffffu, d);
    const int leader = __ffs(peers) - 1;
    uint32_t old = 0;
    if (lane == leader && valid) {
      old = s_cnt[warp][d];
      s_cnt[warp][d] = old + __popc(peers);
    }
    old = __shfl_sync(0xffffffffu, old, leader);
    rank[r] = old + __popc(peers & lt);
    __syncwarp();   // the leaders' counter updates are ordered before the next round's reads (same warp, different lanes)
  }
  __syncthreads();
  // per digit: exclusive offsets over the 8 warps, the chunk's count, its global base by look-back
  uint32_t count = 0;
  if (threadIdx.x <= mask) {
#pragma unroll
    for (int w = 0; w < WARPS; ++w) {
      const uint32_t c = s_cnt[w][threadIdx.x];
      s_cnt[w][threadIdx.x] = count;
      count += c;
    }
    lookback_digit_publish(status, threadIdx.x, chunk, count);   // successors can start adding this chunk's counts at once
  }
  uint32_t chunk_n;
  const uint32_t lstart = block_excl_scan(count, &chunk_n);   // barrier inside
  s_lbase[threadIdx.x] = lstart;
  __syncthreads();
  // reorder the chunk in shared memory (digit runs become contiguous); the values are fetched only now -- they are not
  // needed for ranking and 16 more live registers would cost a resident CTA per SM
#pragma unroll
  for (int r = 0; r < GOF_SORT_ITEMS; ++r) {
    const size_t i = wbase + (size_t)r * 32 + lane;
    if (i < n) {
      const uint32_t d = ((uint32_t)key[r] >> shift) & mask;
      const uint32_t lp = s_lbase[d] + s_cnt[warp][d] + rank[r];
      s_keys[lp] = key[r];
      s_vals[lp] = vals_in[i];
    }
  }
  // the look-back (dependent L2 round trips) overlaps the value loads above
  if (threadIdx.x <= mask) s_gbase[threadIdx.x] = gstart + lookback_digit_walk(status, threadIdx.x, chunk, count);
  __syncthreads();
#pragma unroll
  for (int r = 0; r < GOF_SORT_ITEMS; ++r) {
    const uint32_t i = (uint32_t)r * THREADS + threadIdx.x;
    if (i < chunk_n) {
      const KeyT k = s_keys[i];
      const uint32_t d = ((uint32_t)k >> shift) & mask;
      const uint32_t pos = s_gbase[d] + (i - s_lbase[d]);
      keys_out[pos] = k;
      vals_out[pos] = s_vals[i];
    }
  }
}

struct SortScratch {
  uint32_t* ghist;     // [4][256]
  uint32_t* tickets;   // [64]: [0..3] chunk tickets of the passes
  uint32_t* status;    // [4][chunk groups][256][4]: look-back status words (lookback_digit)
  size_t pass_words;   // words per pass in status
};

SortScratch carve_sort_scratch(uint32_t* scratch, size_t n) {
  SortScratch s;
  s.ghist = scratch;
  s.tickets = scratch + 4 * GOF_RADIX;
  s.status = scratch + GOF_SORT_HEAD_BYTES / 4;
  s.pass_words = (size_t)((gof_sort_blocks(n) + 3) / 4 + 1) * GOF_RADIX * 4;
  return s;
}

void split_digits(int nbits, Digits* dg) {   // as evenly as possible, low digit first (e.g. 13 -> 7 + 6)
  dg->passes = (nbits + 7) / 8;
  int rem = nbits, shift = 0;
  for (int p = 0; p < 4; ++p) { dg->shift[p] = 0; dg->mask[p] = 0; }
  for (int p = 0; p < dg->passes; ++p) {
    const int b = (rem + (dg->passes - p) - 1) / (dg->passes - p);
    dg->shift[p] = shift; dg->mask[p] = (1u << b) - 1u;
    shift += b; rem -= b;
  }
}

// Runs dg.passes one-sweep passes a -> b -> a ...; ghist must hold the digit counts, tickets/status must be zero.
template <typename KeyT>
int onesweep_passes(KeyT* ka, KeyT* kb, uint32_t* va, uint32_t* vb, size_t n, const Digits& dg, const SortScratch& sc, bool debug,
                    cudaStream_t st) {
  const unsigned nb = (unsigned)gof_sort_blocks(n);
  for (int p = 0; p < dg.passes; ++p) {
    const bool a2b = (p % 2 == 0);
    GOF_LAUNCH("radix_onesweep", st, (k_onesweep<KeyT><<<nb, THREADS, 0, st>>>(
        a2b ? ka : kb, a2b ? va : vb, a2b ? kb : ka, a2b ? vb : va, n, dg.shift[p], dg.mask[p], sc.ghist + p * GOF_RADIX,
        sc.status + (size_t)p * sc.pass_words, sc.tickets + p)));
    GOF_LAUNCH_CHECK(debug, st);
  }
  return GOF_OK;
}

// complete sort of n (key, value) pairs on the low nbits of the key: memset of the scratch, digit histograms, passes
template <typename KeyT>
int sort_pairs(KeyT* ka, KeyT* kb, uint32_t* va, uint32_t* vb, uint32_t* scratch, size_t n, int nbits, bool debug, cudaStream_t st,
               int* result_in_b) {
  *result_in_b = 0;
  if (n == 0 || nbits <= 0) return GOF_OK;
  if (n >= LB_MAX_ITEMS) { gof_set_error("radix sort of %zu items: fewer than 2^30 supported", n); return GOF_E_INVALID; }
  Digits dg;
  split_digits(nbits, &dg);
  const SortScratch sc = carve_sort_scratch(scratch, n);
  GOF_CUDA_OK(cudaMemsetAsync(scratch, 0, GOF_SORT_HEAD_BYTES + (size_t)dg.passes * sc.pass_words * 4, st));
  const size_t want = (n + (size_t)THREADS * 8 - 1) / ((size_t)THREADS * 8);
  const unsigned grid = (unsigned)(want < (size_t)gof_sm_count() * 4 ? want : (size_t)gof_sm_count() * 4);
  GOF_LAUNCH("radix_hist", st, k_digit_hist<KeyT><<<grid, THREADS, 0, st>>>(ka, n, dg, sc.ghist));
  GOF_LAUNCH_CHECK(debug, st);
  const int rc = onesweep_passes<KeyT>(ka, kb, va, vb, n, dg, sc, debug, st);
  *result_in_b = gof_radix_result_in_b(nbits);
  return rc;
}

// ------------------------------------------------------------------------------------------------
// single-launch exclusive scan of u32 (decoupled look-back over 64-bit status words: running totals up to 2^32 - 1 are exact,
// larger ones wrap like any u32 sum); chunk = GOF_SCAN_CHUNK values per CTA
__global__ void __launch_bounds__(THREADS) k_scan_excl(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, size_t n,
                                                      uint64_t* __restrict__ status, uint32_t* __restrict__ ticket,
                                                      uint32_t* __restrict__ total_out, uint32_t nchunks) {
  __shared__ uint32_t s_chunk, s_prefix;
  if (threadIdx.x == 0) s_chunk = atomicAdd(ticket, 1u);
  __syncthreads();
  const uint32_t chunk = s_chunk;
  const size_t base = (size_t)chunk * GOF_SCAN_CHUNK + (size_t)threadIdx.x * GOF_SCAN_ITEMS;
  uint32_t v[GOF_SCAN_ITEMS];
  uint32_t s = 0;
#pragma unroll
  for (int k = 0; k < GOF_SCAN_ITEMS; ++k) {
    v[k] = (base + k < n) ? in[base + k] : 0u;
    s += v[k];
  }
  uint32_t total;
  uint32_t run = block_excl_scan(s, &total);
  if (threadIdx.x < 32) {
    const uint32_t excl = lookback_warp(status, chunk, total);
    if (threadIdx.x == 0) {
      s_prefix = excl;
      if (chunk == nchunks - 1 && total_out) *total_out = excl + total;
    }
  }
  __syncthreads();
  run += s_prefix;
#pragma unroll
  for (int k = 0; k < GOF_SCAN_ITEMS; ++k) {
    if (base + k < n) out[base + k] = run;
    run += v[k];
  }
}

// ------------------------------------------------------------------------------------------------
// Scan + instance emission in one launch (duplicateWithKeys, rasterizer_impl.cu:70-111, and the InclusiveSum in front of
// it, :332).  A CTA owns 256 consecutive depth-ordered Gaussians: block scan of their tiles_touched, look-back for the
// number of instances in front of the CTA, then the CTA's instances are FLATTENED -- slot j belongs to the Gaussian found
// by binary search in the CTA's offsets -- so every thread writes one (tile id, Gaussian) pair per iteration, coalesced,
// whatever the footprints are.  The digits of the tile sort are counted on the way.
template <typename KeyT>
__global__ void __launch_bounds__(THREADS) k_scan_emit(int P, const uint32_t* __restrict__ order, const uint2* __restrict__ rect,
                                                      const uint32_t* __restrict__ tiles, int grid_x, KeyT* __restrict__ keys,
                                                      uint32_t* __restrict__ vals, uint32_t* __restrict__ status,
                                                      uint32_t* __restrict__ ticket, Digits dg, uint32_t* __restrict__ ghist,
                                                      uint32_t capacity) {
  __shared__ uint32_t s_off[THREADS + 1];
  __shared__ uint32_t s_g[THREADS];
  __shared__ uint2 s_rect[THREADS];
  __shared__ uint32_t s_h[2][GOF_RADIX];
  __shared__ uint32_t s_chunk, s_prefix;
  if (threadIdx.x == 0) s_chunk = atomicAdd(ticket, 1u);
  s_h[0][threadIdx.x] = 0; s_h[1][threadIdx.x] = 0;
  __syncthreads();
  const uint32_t chunk = s_chunk;
  const int k = (int)(chunk * THREADS + threadIdx.x);   // position in depth order
  uint32_t g = 0, n = 0;
  uint2 rc = make_uint2(0u, 0u);
  if (k < P) {
    g = order[k];
    n = tiles[g];
    if (n) rc = rect[g];
  }
  uint32_t total;
  const uint32_t lo = block_excl_scan(n, &total);
  s_off[threadIdx.x] = lo; s_g[threadIdx.x] = g; s_rect[threadIdx.x] = rc;
  if (threadIdx.x < 32) {
    const uint32_t excl = lookback_warp(status, chunk, total);
    if (threadIdx.x == 0) { s_off[THREADS] = total; s_prefix = excl; }
  }
  __syncthreads();
  const uint32_t prefix = s_prefix;
  for (uint32_t j = threadIdx.x; j < total; j += THREADS) {
    // largest i with s_off[i] <= j (Gaussians without tiles repeat their successor's offset and are skipped)
    int lo_i = 0, hi_i = THREADS;
    while (hi_i - lo_i > 1) {
      const int mid = (lo_i + hi_i) >> 1;
      if (s_off[mid] <= j) lo_i = mid; else hi_i = mid;
    }
    const uint32_t t = j - s_off[lo_i];
    const uint2 r = s_rect[lo_i];
    const uint32_t xmin = r.x & 0xffffu, ymin = r.x >> 16;
    const uint32_t w = (r.y & 0xffffu) - xmin;
    const uint32_t dy = t / w, dx = t - dy * w;
    const uint32_t tile = (ymin + dy) * (uint32_t)grid_x + xmin + dx;
    const uint32_t pos = prefix + j;
    if (pos < capacity) {   // capacity == num_rendered: always true; guards the buffer should the two ever disagree
      keys[pos] = (KeyT)tile;
      vals[pos] = s_g[lo_i];
    }
    atomicAdd(&s_h[0][(tile >> dg.shift[0]) & dg.mask[0]], 1u);
    if (dg.passes > 1) atomicAdd(&s_h[1][(tile >> dg.shift[1]) & dg.mask[1]], 1u);
  }
  __syncthreads();
  if (s_h[0][threadIdx.x]) atomicAdd(ghist + threadIdx.x, s_h[0][threadIdx.x]);
  if (dg.passes > 1 && s_h[1][threadIdx.x]) atomicAdd(ghist + GOF_RADIX + threadIdx.x, s_h[1][threadIdx.x]);
}

// rasterizer_impl.cu:149-171 identifyTileRanges on the sorted tile ids (ranges pre-zeroed, :365)
template <typename KeyT>
__global__ void __launch_bounds__(256) k_tile_ranges(size_t L, const KeyT* __restrict__ keys, uint2* __restrict__ ranges, int key_shift) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= L) return;
  const uint32_t cur = (uint32_t)keys[idx] >> key_shift;   // tile id = key >> key_shift (the query points' keys carry the pixel below it)
  if (idx == 0)
    ranges[cur].x = 0;
  else {
    const uint32_t prev = (uint32_t)keys[idx - 1] >> key_shift;
    if (cur != prev) {
      ranges[prev].y = (uint32_t)idx;
      ranges[cur].x = (uint32_t)idx;
    }
  }
  if (idx == L - 1) ranges[cur].y = (uint32_t)L;
}

template <typename KeyT>
int bin_tiles_t(int P, size_t R, const GofView& v, char* geom, const GofGeomLayout& GL, char* bin, const GofBinLayout& BL, char* img,
                const GofImageLayout& IL, bool debug, cudaStream_t st) {
  if (R >= LB_MAX_ITEMS) { gof_set_error("binning: %zu (tile, Gaussian) instances, fewer than 2^30 supported", R); return GOF_E_INVALID; }
  uint2* ranges = reinterpret_cast<uint2*>(img + IL.ranges);
  GOF_CUDA_OK(cudaMemsetAsync(ranges, 0, (size_t)v.tiles * sizeof(uint2), st));
  if (R == 0) return GOF_OK;
  KeyT* ka = reinterpret_cast<KeyT*>(bin + BL.key_a);
  KeyT* kb = reinterpret_cast<KeyT*>(bin + BL.key_b);
  uint32_t* va = reinterpret_cast<uint32_t*>(bin + BL.val_a);
  uint32_t* vb = reinterpret_cast<uint32_t*>(bin + BL.val_b);
  uint32_t* scratch = reinterpret_cast<uint32_t*>(bin + BL.hist);
  Digits dg;
  dg.passes = BL.passes;
  int shift = 0;
  for (int p = 0; p < 4; ++p) {
    dg.shift[p] = shift; dg.mask[p] = p < BL.passes ? (1u << BL.bits[p]) - 1u : 0u;
    shift += BL.bits[p];
  }
  if (BL.passes > 2) { gof_set_error("tile ids need more than two radix digits"); return GOF_E_INVALID; }   // > 65536 tiles
  const SortScratch sc = carve_sort_scratch(scratch, R);
  GOF_CUDA_OK(cudaMemsetAsync(scratch, 0, GOF_SORT_HEAD_BYTES + (size_t)dg.passes * sc.pass_words * 4, st));
  uint32_t* scan_status = reinterpret_cast<uint32_t*>(geom + GL.scan_tmp);
  const int nchunks = (P + THREADS - 1) / THREADS;
  GOF_CUDA_OK(cudaMemsetAsync(scan_status, 0, ((size_t)nchunks + 8) * 4, st));
  // the depth sort always runs 4 passes: its result is back in the *_a buffers of the geometry state
  const uint32_t* order = reinterpret_cast<const uint32_t*>(geom + GL.val_a);
  GOF_LAUNCH("scan_emit", st, k_scan_emit<KeyT><<<nchunks, THREADS, 0, st>>>(
      P, order, reinterpret_cast<const uint2*>(geom + GL.rect), reinterpret_cast<const uint32_t*>(geom + GL.tiles), v.grid_x, ka, va,
      scan_status, scan_status + nchunks + 4, dg, sc.ghist, (uint32_t)R));
  GOF_LAUNCH_CHECK(debug, st);
  const int rc = onesweep_passes<KeyT>(ka, kb, va, vb, R, dg, sc, debug, st);
  if (rc != GOF_OK) return rc;
  const KeyT* sorted = reinterpret_cast<const KeyT*>(bin + BL.sorted_keys);
  GOF_LAUNCH("tile_ranges", st, k_tile_ranges<KeyT><<<(unsigned)((R + 255) / 256), 256, 0, st>>>(R, sorted, ranges, 0));
  GOF_LAUNCH_CHECK(debug, st);
  return GOF_OK;
}

// ------------------------------------------------------------------------------------------------
// Multi-word keys: one stable sort per word, least significant first, each on the previous word's order

// values = identity; ka = w0 (nullptr: w0 is ka already)
__global__ void __launch_bounds__(THREADS) k_sort_init(size_t n, const uint32_t* __restrict__ w0, uint32_t* __restrict__ ka,
                                                      uint32_t* __restrict__ vals) {
  const size_t i = (size_t)blockIdx.x * THREADS + threadIdx.x;
  if (i >= n) return;
  vals[i] = (uint32_t)i;
  if (w0) ka[i] = w0[i];
}

// the next word in the current order: keys[j] = word[ord[j]]
__global__ void __launch_bounds__(THREADS) k_gather_word(size_t n, const uint32_t* __restrict__ word, const uint32_t* __restrict__ ord,
                                                        uint32_t* __restrict__ keys) {
  const size_t j = (size_t)blockIdx.x * THREADS + threadIdx.x;
  if (j < n) keys[j] = word[ord[j]];
}

__global__ void __launch_bounds__(THREADS) k_run_heads(size_t n, const GofKeyWords key, const uint32_t* __restrict__ ord,
                                                      uint32_t* __restrict__ head) {
  const size_t j = (size_t)blockIdx.x * THREADS + threadIdx.x;
  if (j >= n) return;
  if (j == 0) { head[0] = 1; return; }
  const uint32_t a = ord[j], b = ord[j - 1];
  uint32_t diff = 0;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    if (k >= key.nw) break;
    const uint32_t mask = key.bits[k] >= 32 ? 0xffffffffu : (1u << key.bits[k]) - 1u;
    diff |= (key.w[k][a] ^ key.w[k][b]) & mask;
  }
  head[j] = diff ? 1u : 0u;
}

}  // namespace

// every pass moves the pairs to the other buffers
int gof_radix_result_in_b(int nbits) {
  Digits dg;
  split_digits(nbits, &dg);
  return dg.passes % 2;
}

// Stable sort of the P (depth bits, gaussian id) pairs written by the preprocess kernel into key_a/val_a; 4 passes ->
// result back in *_a.  (The scan of tiles_touched in that order happens inside the emit kernel, gof_bin_tiles.)
int gof_depth_sort(int P, char* geom, const GofGeomLayout& L, bool debug, cudaStream_t st) {
  int in_b = 0;
  return sort_pairs<uint32_t>(reinterpret_cast<uint32_t*>(geom + L.key_a), reinterpret_cast<uint32_t*>(geom + L.key_b),
                              reinterpret_cast<uint32_t*>(geom + L.val_a), reinterpret_cast<uint32_t*>(geom + L.val_b),
                              reinterpret_cast<uint32_t*>(geom + L.hist), (size_t)P, 32, debug, st, &in_b);
}

// Stable sort of `n` (key, index) pairs on the low nbits of the key for the integrate path's query points (tile id = key >>
// key_shift; the bits below it order the points of a tile by pixel), then the per-tile ranges of the first ids < num_tiles (ranges must hold num_tiles + 1 uint2; the last slot absorbs the
// sentinel id given to points outside the image).  Buffers: keys/vals ping-pong (u32), scratch as in gof_sort_scratch_bytes.
int gof_sort_points_by_tile(size_t n, int nbits, int key_shift, uint32_t* ka, uint32_t* kb, uint32_t* va, uint32_t* vb, uint32_t* hist,
                            uint2* ranges, int num_tiles, bool debug, cudaStream_t st) {
  GOF_CUDA_OK(cudaMemsetAsync(ranges, 0, (size_t)(num_tiles + 1) * sizeof(uint2), st));
  if (n == 0) return GOF_OK;
  int in_b = 0;
  const int rc = sort_pairs<uint32_t>(ka, kb, va, vb, hist, n, nbits, debug, st, &in_b);
  if (rc != GOF_OK) return rc;
  const uint32_t* sorted = in_b ? kb : ka;
  GOF_LAUNCH("tile_ranges", st, k_tile_ranges<uint32_t><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(n, sorted, ranges, key_shift));
  GOF_LAUNCH_CHECK(debug, st);
  return GOF_OK;
}

int gof_exclusive_scan_u32(const uint32_t* in, uint32_t* out, uint32_t* tmp, uint32_t* total, size_t n, bool debug, cudaStream_t st) {
  if (n == 0) {
    if (total) GOF_CUDA_OK(cudaMemsetAsync(total, 0, 4, st));
    return GOF_OK;
  }
  if (reinterpret_cast<uintptr_t>(tmp) % 8u) { gof_set_error("exclusive_scan: tmp must be 8-byte aligned"); return GOF_E_INVALID; }
  // tmp: nchunks u64 status words, then the chunk ticket
  const uint32_t nchunks = (uint32_t)((n + GOF_SCAN_CHUNK - 1) / GOF_SCAN_CHUNK);
  GOF_CUDA_OK(cudaMemsetAsync(tmp, 0, ((size_t)nchunks * 2 + 1) * 4, st));
  GOF_LAUNCH("scan", st, k_scan_excl<<<nchunks, THREADS, 0, st>>>(in, out, n, reinterpret_cast<uint64_t*>(tmp), tmp + (size_t)nchunks * 2,
                                                                  total, nchunks));
  GOF_LAUNCH_CHECK(debug, st);
  return GOF_OK;
}

int gof_sort_words_u32(const GofKeyWords& key, size_t n, const GofSortBufs& b, uint32_t* ord, bool debug, cudaStream_t st) {
  if (key.nw < 1 || key.nw > 3 || (ord != b.va && ord != b.vb)) { gof_set_error("sort_words: 1-3 words, ord = va or vb"); return GOF_E_INVALID; }
  int passes = 0;
  for (int k = 0; k < key.nw; ++k) {
    if (key.bits[k] < 1 || key.bits[k] > 32) { gof_set_error("sort_words: %d bits in word %d", key.bits[k], k); return GOF_E_INVALID; }
    passes += (key.bits[k] + 7) / 8;
  }
  if (n == 0) return GOF_OK;
  if (n >= LB_MAX_ITEMS) { gof_set_error("sort_words: %zu items, the radix sort takes fewer than 2^30", n); return GOF_E_INVALID; }
  // every radix pass moves the values to the other buffer: start in the one from which the last pass ends in ord
  uint32_t* vals = passes % 2 == 0 ? ord : (ord == b.va ? b.vb : b.va);
  uint32_t* spare = vals == b.va ? b.vb : b.va;
  const unsigned grid = (unsigned)((n + THREADS - 1) / THREADS);
  GOF_LAUNCH("sort_init", st, k_sort_init<<<grid, THREADS, 0, st>>>(n, key.w[0] == b.ka ? nullptr : key.w[0], b.ka, vals));
  GOF_LAUNCH_CHECK(debug, st);
  for (int k = 0; k < key.nw; ++k) {
    if (k > 0) {
      GOF_LAUNCH("sort_gather", st, k_gather_word<<<grid, THREADS, 0, st>>>(n, key.w[k], vals, b.ka));
      GOF_LAUNCH_CHECK(debug, st);
    }
    int in_b = 0;
    const int rc = sort_pairs<uint32_t>(b.ka, b.kb, vals, spare, b.hist, n, key.bits[k], debug, st, &in_b);
    if (rc != GOF_OK) return rc;
    if (in_b) { uint32_t* t = vals; vals = spare; spare = t; }
  }
  return GOF_OK;
}

int gof_key_runs_u32(const GofKeyWords& key, const uint32_t* ord, size_t n, uint32_t* head, uint32_t* run, uint32_t* scan_tmp,
                     uint32_t* num_runs, bool debug, cudaStream_t st) {
  if (key.nw < 1 || key.nw > 3) { gof_set_error("key_runs: 1-3 words"); return GOF_E_INVALID; }
  if (n > 0) {
    GOF_LAUNCH("run_heads", st, k_run_heads<<<(unsigned)((n + THREADS - 1) / THREADS), THREADS, 0, st>>>(n, key, ord, head));
    GOF_LAUNCH_CHECK(debug, st);
  }
  return gof_exclusive_scan_u32(head, run, scan_tmp, num_runs, n, debug, st);
}

int gof_bin_tiles(int P, size_t R, const GofView& v, char* geom, const GofGeomLayout& GL, char* bin, const GofBinLayout& BL,
                  char* img, const GofImageLayout& IL, bool debug, cudaStream_t st) {
  if (BL.key_bytes == 2) return bin_tiles_t<uint16_t>(P, R, v, geom, GL, bin, BL, img, IL, debug, st);
  return bin_tiles_t<uint32_t>(P, R, v, geom, GL, bin, BL, img, IL, debug, st);
}

// ------------------------------------------------------------------------------------------------
// Test entry points (tests/test_gpu_sort_primitives.py, tools/sanitize_run.py): the sort, run and scan primitives above over
// plain pointers, so that they can be checked against an exact reference on their own.  Not part of the public header.
// All pointers are device pointers except `words` and `bits` (host arrays of nw entries).
namespace {
GofKeyWords probe_key(int nw, const uint32_t* const* words, const int* bits) {
  GofKeyWords key{};
  key.nw = nw;
  for (int k = 0; k < nw && k < 3; ++k) { key.w[k] = words[k]; key.bits[k] = bits[k]; }
  return key;
}
}  // namespace

extern "C" GOF_API int gof_probe_sort_words_u32(int nw, const uint32_t* const* words, const int* bits, size_t n, uint32_t* ka,
                                                uint32_t* kb, uint32_t* va, uint32_t* vb, uint32_t* hist, int ord_is_vb, void* stream) {
  return gof_sort_words_u32(probe_key(nw, words, bits), n, GofSortBufs{ka, kb, va, vb, hist}, ord_is_vb ? vb : va, false,
                            (cudaStream_t)stream);
}

extern "C" GOF_API int gof_probe_key_runs_u32(int nw, const uint32_t* const* words, const int* bits, const uint32_t* ord, size_t n,
                                              uint32_t* head, uint32_t* run, uint32_t* scan_tmp, uint32_t* num_runs, void* stream) {
  return gof_key_runs_u32(probe_key(nw, words, bits), ord, n, head, run, scan_tmp, num_runs, false, (cudaStream_t)stream);
}

extern "C" GOF_API int gof_probe_exclusive_scan_u32(const uint32_t* in, uint32_t* out, uint32_t* tmp, uint32_t* total, size_t n,
                                                    void* stream) {
  return gof_exclusive_scan_u32(in, out, tmp, total, n, false, (cudaStream_t)stream);
}

// which = 0: the `hist` scratch of a sort of n items (gof_sort_scratch_bytes); 1: the `tmp` of a scan of n values
// (gof_scan_scratch_bytes)
extern "C" GOF_API size_t gof_probe_scratch_bytes(int which, size_t n) {
  return which == 0 ? gof_sort_scratch_bytes(n) : which == 1 ? gof_scan_scratch_bytes(n) : 0;
}
