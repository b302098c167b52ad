// tsdf.cu -- TSDF fusion of rendered depth into a sparse voxel-block volume, and marching-cubes extraction.
//
// Reference: extract_mesh_tsdf.py:16-83, which fuses median depth and colour into Open3D's VoxelBlockGrid
// (compute_unique_block_coordinates, integrate, extract_triangle_mesh).  The contract is DESIGN section 4.4: every float
// step is one IEEE operation in the written order (__fmul_rn / __fadd_rn / __fdiv_rn, no contraction), so that the numpy
// float32 oracle reproduces it bit for bit.  The library keeps no state: the block table (sorted keys + pool slots) and
// the voxel pool belong to the caller.
//
//   touch     one thread per sampled pixel: count its blocks -> scan -> emit 63-bit keys as (lo, hi) u32 words -> the
//             library's multi-word sort -> one unique key per run of equal keys
//   activate  binary search of the view's keys in the table, scan of the "new" flags, merge by binary search
//   integrate one CTA per block of the view's list; voxel data is structure-of-arrays per block, read coalesced, and
//             only updated voxels are written; the depth and colour images are gathers that stay in L2
//   extract   one CTA per table block: its +1 neighbour blocks are found once by binary search; meshed cubes mark the
//             edges they use at the edges' owner voxels; per-block vertex and face counts are scanned; the emit kernels
//             re-derive each voxel's offset with a block scan and write vertices and faces in canonical order; the same
//             kernels, instantiated for one value plane without weights, mesh the opacity field's lattice (DESIGN 4.15)
#include "gof_common.cuh"
#include "mc_table.cuh"
#include "voxel_blocks.cuh"

namespace {

constexpr int TOUCH_STRIDE = 4;
constexpr int PLANES = 5;   // tsdf, weight, r, g, b

struct Cam {
  int W, H;
  float fx, fy, cx, cy;
  float R[9], t[3];
};

static Cam make_cam(const gof_tsdf_camera_t* c) {
  Cam k;
  k.W = c->width; k.H = c->height; k.fx = c->fx; k.fy = c->fy; k.cx = c->cx; k.cy = c->cy;
  for (int r = 0; r < 3; ++r) {
    for (int q = 0; q < 3; ++q) k.R[3 * r + q] = c->extrinsic[4 * r + q];
    k.t[r] = c->extrinsic[4 * r + 3];
  }
  return k;
}

struct Par {
  float s, tau, bs, dmax;
  int B;
  int span;   // most blocks per axis one pixel can touch: floor((x + tau) / bs) - floor((x - tau) / bs) + 1 <= 2 tau / bs + 2
};

static Par make_par(const gof_tsdf_params_t* p) {
  Par q;
  q.s = p->voxel_size; q.tau = p->trunc; q.dmax = p->depth_max; q.B = p->block_resolution;
  q.bs = (float)q.B * q.s;   // fl(B * s): B is exact in float
  const double r = 2.0 * (double)q.tau / (double)q.bs;
  q.span = r < 1e6 ? (int)r + 2 : 1 << 20;
  return q;
}

static int check_params(const gof_tsdf_params_t* p, const char* who) {
  if (!p || !(p->voxel_size > 0.f) || p->block_resolution < 1 || p->block_resolution > 64 || !(p->trunc > 0.f)) {
    gof_set_error("%s: voxel_size > 0, trunc > 0 and block_resolution in 1..64 required", who);
    return GOF_E_INVALID;
  }
  return GOF_OK;
}

// ---- touch -------------------------------------------------------------------------------------------------------

struct TouchLayout {
  size_t header, cnt, off, scan_tmp, lo, hi, val_a, val_b, hist, head, uid, bytes;
  size_t npix, cap;
};
struct TouchHeader { uint32_t n_inst, err, n_unique, pad; };

static TouchLayout touch_layout(int W, int H, const Par& p) {
  TouchLayout L; size_t o = 0;
  auto take = [&](size_t b) { size_t r = o; o = gof_align_up(o + b, 256); return r; };
  L.npix = (size_t)((W + TOUCH_STRIDE - 1) / TOUCH_STRIDE) * (size_t)((H + TOUCH_STRIDE - 1) / TOUCH_STRIDE);
  const size_t span = (size_t)p.span;
  L.cap = L.npix * span * span * span;
  const size_t I = L.cap > L.npix ? L.cap : L.npix;
  L.header = take(256);
  L.cnt = take(L.npix * 4); L.off = take(L.npix * 4);
  L.scan_tmp = take(gof_scan_scratch_bytes(I));
  L.lo = take(L.cap * 4); L.hi = take(L.cap * 4);
  L.val_a = take(L.cap * 4); L.val_b = take(L.cap * 4);
  L.hist = take(gof_sort_scratch_bytes(L.cap));
  L.head = take(L.cap * 4); L.uid = take(L.cap * 4);
  L.bytes = o;
  return L;
}

// block range [lo, hi] per axis of the sampled pixel `pix`; false if the pixel has no valid depth
__device__ __forceinline__ bool pixel_blocks(int pix, const float* __restrict__ depth, const Cam& c, const Par& p, float* lo, float* hi) {
  const int sw = (c.W + TOUCH_STRIDE - 1) / TOUCH_STRIDE;
  const int u = (pix % sw) * TOUCH_STRIDE, v = (pix / sw) * TOUCH_STRIDE;
  const float d = depth[(size_t)v * c.W + u];
  if (!(d > 0.f && d < p.dmax)) return false;
  float pc[3];
  pc[0] = __fdiv_rn(__fmul_rn(__fsub_rn((float)u, c.cx), d), c.fx);
  pc[1] = __fdiv_rn(__fmul_rn(__fsub_rn((float)v, c.cy), d), c.fy);
  pc[2] = d;
  float q[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) q[i] = __fsub_rn(pc[i], c.t[i]);
#pragma unroll
  for (int i = 0; i < 3; ++i) {   // pw = R^T q
    const float pw = __fadd_rn(__fadd_rn(__fmul_rn(c.R[i], q[0]), __fmul_rn(c.R[3 + i], q[1])), __fmul_rn(c.R[6 + i], q[2]));
    lo[i] = floorf(__fdiv_rn(__fsub_rn(pw, p.tau), p.bs));
    hi[i] = floorf(__fdiv_rn(__fadd_rn(pw, p.tau), p.bs));
  }
  return true;
}

__global__ void __launch_bounds__(THREADS) k_touch_count(int npix, const float* __restrict__ depth, const Cam c, const Par p,
                                                        uint32_t* __restrict__ cnt, TouchHeader* __restrict__ hd) {
  const int pix = blockIdx.x * THREADS + threadIdx.x;
  if (pix >= npix) return;
  float lo[3], hi[3];
  uint32_t n = 0;
  if (pixel_blocks(pix, depth, c, p, lo, hi)) {
    bool in_range = true, in_span = true;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      in_range = in_range && lo[i] >= -(float)KEY_BIAS && hi[i] < (float)KEY_BIAS;
      in_span = in_span && hi[i] - lo[i] < (float)p.span;
    }
    if (!in_range) atomicOr(&hd->err, 1u);
    else if (!in_span) atomicOr(&hd->err, 2u);   // more blocks than the scratch was sized for (rounding beyond the bound)
    else n = (uint32_t)((hi[0] - lo[0] + 1.f) * (hi[1] - lo[1] + 1.f) * (hi[2] - lo[2] + 1.f));
  }
  cnt[pix] = n;
}

__global__ void __launch_bounds__(THREADS) k_touch_emit(int npix, const float* __restrict__ depth, const Cam c, const Par p,
                                                       const uint32_t* __restrict__ cnt, const uint32_t* __restrict__ off,
                                                       uint32_t* __restrict__ lo_w, uint32_t* __restrict__ hi_w) {
  const int pix = blockIdx.x * THREADS + threadIdx.x;
  if (pix >= npix || !cnt[pix]) return;
  float lo[3], hi[3];
  pixel_blocks(pix, depth, c, p, lo, hi);
  uint32_t o = off[pix];
  for (int z = (int)lo[2]; z <= (int)hi[2]; ++z)
    for (int y = (int)lo[1]; y <= (int)hi[1]; ++y)
      for (int x = (int)lo[0]; x <= (int)hi[0]; ++x) {
        const uint64_t k = (uint64_t)pack_key(x, y, z);
        lo_w[o] = (uint32_t)k; hi_w[o] = (uint32_t)(k >> 32);
        ++o;
      }
}

// ---- activate ----------------------------------------------------------------------------------------------------

struct ActLayout { size_t header, pos, flag, off, scan_tmp, bytes; };
static ActLayout act_layout(size_t nv) {
  ActLayout L; size_t o = 0;
  auto take = [&](size_t b) { size_t r = o; o = gof_align_up(o + b, 256); return r; };
  L.header = take(256); L.pos = take(nv * 8); L.flag = take(nv * 4); L.off = take(nv * 4);
  L.scan_tmp = take(gof_scan_scratch_bytes(nv));
  L.bytes = o;
  return L;
}

__global__ void __launch_bounds__(THREADS) k_act_find(int64_t nt, const int64_t* __restrict__ tkeys, int64_t nv,
                                                     const int64_t* __restrict__ vkeys, int64_t* __restrict__ pos,
                                                     uint32_t* __restrict__ flag) {
  const int64_t j = (int64_t)blockIdx.x * THREADS + threadIdx.x;
  if (j >= nv) return;
  const int64_t k = vkeys[j];
  const int64_t p = lower_bound(tkeys, nt, k);
  pos[j] = p;
  flag[j] = (p < nt && tkeys[p] == k) ? 0u : 1u;
}

// old entry i moves up by the number of new keys below it: the new-flag scan at the first view key >= its key
__global__ void __launch_bounds__(THREADS) k_act_merge_old(int64_t nt, const int64_t* __restrict__ tkeys, const int32_t* __restrict__ tslots,
                                                          int64_t nv, const int64_t* __restrict__ vkeys, const uint32_t* __restrict__ off,
                                                          uint32_t n_new, int64_t* __restrict__ okeys, int32_t* __restrict__ oslots) {
  const int64_t i = (int64_t)blockIdx.x * THREADS + threadIdx.x;
  if (i >= nt) return;
  const int64_t k = tkeys[i];
  const int64_t j = lower_bound(vkeys, nv, k);
  const int64_t o = i + (j < nv ? off[j] : n_new);
  okeys[o] = k;
  oslots[o] = tslots[i];
}

__global__ void __launch_bounds__(THREADS) k_act_merge_new(int64_t nt, const int32_t* __restrict__ tslots, int64_t nv,
                                                          const int64_t* __restrict__ vkeys, const int64_t* __restrict__ pos,
                                                          const uint32_t* __restrict__ flag, const uint32_t* __restrict__ off,
                                                          int64_t* __restrict__ okeys, int32_t* __restrict__ oslots,
                                                          int32_t* __restrict__ vslots) {
  const int64_t j = (int64_t)blockIdx.x * THREADS + threadIdx.x;
  if (j >= nv) return;
  if (flag[j]) {
    const int32_t slot = (int32_t)(nt + off[j]);
    const int64_t o = pos[j] + off[j];
    okeys[o] = vkeys[j];
    oslots[o] = slot;
    vslots[j] = slot;
  } else {
    vslots[j] = tslots[pos[j]];
  }
}

// ---- integrate ---------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(THREADS) k_integrate(const float* __restrict__ depth, const float* __restrict__ color, const Cam c,
                                                      const Par p, const int64_t* __restrict__ vkeys, const int32_t* __restrict__ vslots,
                                                      float* __restrict__ pool, unsigned long long* __restrict__ num_updates) {
  const int B = p.B;
  const int n3 = B * B * B;
  int b[3];
  unpack_key(vkeys[blockIdx.x], b);
  float* blk = pool + (size_t)vslots[blockIdx.x] * PLANES * n3;
  const size_t HW = (size_t)c.W * c.H;
  const float wm1 = (float)(c.W - 1), hm1 = (float)(c.H - 1), ntau = -p.tau;
  uint32_t updates = 0;
  for (int lin = threadIdx.x; lin < n3; lin += THREADS) {
    const int li[3] = {lin % B, (lin / B) % B, lin / (B * B)};
    float pw[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) pw[a] = __fmul_rn(__int2float_rn(b[a] * B + li[a]), p.s);
    float pc[3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
      pc[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(c.R[3 * r], pw[0]), __fmul_rn(c.R[3 * r + 1], pw[1])), __fmul_rn(c.R[3 * r + 2], pw[2])),
                        c.t[r]);
    if (!(pc[2] > 0.f)) continue;
    const float u = __fadd_rn(__fdiv_rn(__fmul_rn(c.fx, pc[0]), pc[2]), c.cx);
    const float v = __fadd_rn(__fdiv_rn(__fmul_rn(c.fy, pc[1]), pc[2]), c.cy);
    if (!(u >= 0.f && u <= wm1 && v >= 0.f && v <= hm1)) continue;
    const size_t px = (size_t)__float2int_rz(v) * c.W + __float2int_rz(u);
    const float d = __ldg(depth + px);
    const float sdf = __fsub_rn(d, pc[2]);
    if (!(d > 0.f && d <= p.dmax && sdf >= ntau)) continue;
    const float sd = __fdiv_rn(fminf(sdf, p.tau), p.tau);
    const float w = blk[n3 + lin];
    const float w1 = __fadd_rn(w, 1.f);
    blk[lin] = __fdiv_rn(__fadd_rn(__fmul_rn(w, blk[lin]), sd), w1);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      float* cp = blk + (size_t)(2 + ch) * n3 + lin;
      *cp = __fdiv_rn(__fadd_rn(__fmul_rn(w, *cp), __ldg(color + ch * HW + px)), w1);
    }
    blk[n3 + lin] = w1;
    ++updates;
  }
  if (num_updates) {
    uint32_t total;
    block_excl_scan(updates, &total);
    if (threadIdx.x == 0 && total) atomicAdd(num_updates, (unsigned long long)total);
  }
}

// ---- extract -----------------------------------------------------------------------------------------------------
//
// One set of kernels serves two value layouts, chosen at compile time:
//   FIELD = false  the TSDF pool [slot][tsdf, weight, r, g, b][B^3] behind the table's slots; a cube is meshed iff its eight
//                  corners exist with weight > theta; vertices are interpolated on their edge, with colours
//   FIELD = true   the opacity field's lattice (field_grid.cu, DESIGN section 4.15): one value plane [n][B^3] in table order
//                  (slot = table position), every voxel of a listed block present with weight 1 and theta 0, so a cube is
//                  meshed iff its eight corners exist; each vertex is returned as its edge -- the two lattice points and
//                  their values -- for the bisection

struct MeshLayout { size_t header, nbr, marks, vid, bv, bf, bv_off, bf_off, scan_tmp, bytes; };
// totals of the per-block counts in 64 bits (checked against the 32-bit ids) and as the scans report them
struct MeshHeader { unsigned long long nv64, nf64; uint32_t nv, nf; };

static MeshLayout mesh_layout(size_t n, int B) {
  const size_t n3 = (size_t)B * B * B;
  MeshLayout L; size_t o = 0;
  auto take = [&](size_t b) { size_t r = o; o = gof_align_up(o + b, 256); return r; };
  L.header = take(256);
  L.nbr = take(n * 8 * 4);
  L.marks = take(n * n3);
  L.vid = take(n * n3 * 4);
  L.bv = take(n * 4); L.bf = take(n * 4); L.bv_off = take(n * 4); L.bf_off = take(n * 4);
  L.scan_tmp = take(gof_scan_scratch_bytes(n));
  L.bytes = o;
  return L;
}

struct MeshArgs {
  int64_t n;
  const int64_t* keys;
  const int32_t* slots;  // FIELD: unused (slot = table position)
  const float* pool;
  int B;
  float s;
  float theta;
  int32_t* nbr;          // [n][8] table position of the block at corner offset c (c = 0: itself), -1 if absent
  uint8_t* marks;        // [n][B^3] bit a: the voxel's edge along axis a carries a vertex
  uint32_t* vid;         // [n][B^3] id of the voxel's first vertex
  uint32_t *bv, *bf;     // per block vertex / face counts
  uint32_t *bv_off, *bf_off;   // their exclusive scans: the block's first vertex / face
  unsigned long long* totals;  // [2] vertex and face totals
  float *vertices, *colors;    // !FIELD
  float *edge_points, *edge_values;   // FIELD: [V][2][3] the owner's and the far end's lattice points, [V][2] their values
  int64_t* faces;
};

template <bool FIELD>
__device__ __forceinline__ const float* block_values(const MeshArgs& a, int slot, size_t n3) {
  return a.pool + (size_t)slot * (FIELD ? 1 : PLANES) * n3;
}

// voxel (x, y, z) in 0..B of this block (the +1 layer lies in a neighbour): returns which neighbour (its corner offset c,
// 0 = this block) and its lin index there
__device__ __forceinline__ int locate(int B, int x, int y, int z, int* lin) {
  const int c = (x >= B ? 1 : 0) | (y >= B ? 2 : 0) | (z >= B ? 4 : 0);
  *lin = (x - (x >= B ? B : 0)) + B * (y - (y >= B ? B : 0)) + B * B * (z - (z >= B ? B : 0));
  return c;
}

template <bool FIELD>
__device__ __forceinline__ void load_neighbours(const MeshArgs& a, int* s_nbr, int* s_slot, bool find) {
  const int64_t p = blockIdx.x;
  if (threadIdx.x < 8) {
    const int c = threadIdx.x;
    int q;
    if (find) {
      int b[3];
      unpack_key(a.keys[p], b);
      const int nb[3] = {b[0] + (c & 1), b[1] + ((c >> 1) & 1), b[2] + ((c >> 2) & 1)};
      q = -1;
      if (c == 0) q = (int)p;
      else if (nb[0] < KEY_BIAS && nb[1] < KEY_BIAS && nb[2] < KEY_BIAS) {
        const int64_t k = pack_key(nb[0], nb[1], nb[2]);
        const int64_t i = lower_bound(a.keys, a.n, k);
        if (i < a.n && a.keys[i] == k) q = (int)i;
      }
      a.nbr[8 * p + c] = q;
    } else {
      q = a.nbr[8 * p + c];
    }
    s_nbr[c] = q;
    s_slot[c] = q >= 0 ? (FIELD ? q : a.slots[q]) : -1;
  }
  __syncthreads();
}

// cube at voxel (x, y, z) of this block: true if meshed (all 8 corners exist, with weight > theta in the TSDF layout);
// *code: bit c = corner c negative
template <bool FIELD>
__device__ __forceinline__ bool cube_code(const MeshArgs& a, const int* s_nbr, const int* s_slot, int x, int y, int z, uint32_t* code) {
  const int B = a.B;
  const size_t n3 = (size_t)B * B * B;
  uint32_t cd = 0;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    int lin;
    const int nb = locate(B, x + (c & 1), y + ((c >> 1) & 1), z + ((c >> 2) & 1), &lin);
    if (s_nbr[nb] < 0) return false;
    const float* blk = block_values<FIELD>(a, s_slot[nb], n3);
    if (!FIELD && !(__ldg(blk + n3 + lin) > a.theta)) return false;
    cd |= (__ldg(blk + lin) < 0.f ? 1u : 0u) << c;
  }
  *code = cd;
  return true;
}

template <bool FIELD>
__global__ void __launch_bounds__(THREADS) k_mc_mark(const MeshArgs a) {
  __shared__ int s_nbr[8], s_slot[8];
  load_neighbours<FIELD>(a, s_nbr, s_slot, true);
  const int B = a.B;
  const int n3 = B * B * B;
  uint32_t nf = 0;
  for (int lin = threadIdx.x; lin < n3; lin += THREADS) {
    const int x = lin % B, y = (lin / B) % B, z = lin / (B * B);
    uint32_t code;
    if (!cube_code<FIELD>(a, s_nbr, s_slot, x, y, z, &code)) continue;
    nf += c_mc_ntri[code];
#pragma unroll
    for (int e = 0; e < 12; ++e) {
      const int o = c_mc_edge_owner[e], f = o | (1 << (e >> 2));
      if (!(((code >> o) ^ (code >> f)) & 1u)) continue;
      int ol;
      const int q = s_nbr[locate(B, x + (o & 1), y + ((o >> 1) & 1), z + ((o >> 2) & 1), &ol)];
      const size_t idx = (size_t)q * n3 + ol;
      atomicOr(reinterpret_cast<unsigned int*>(a.marks + (idx & ~(size_t)3)), (1u << (e >> 2)) << (8 * (idx & 3)));
    }
  }
  uint32_t total;
  block_excl_scan(nf, &total);
  if (threadIdx.x == 0) {
    a.bf[blockIdx.x] = total;
    if (total) atomicAdd(a.totals + 1, (unsigned long long)total);
  }
}

__global__ void __launch_bounds__(THREADS) k_mc_vcount(const MeshArgs a) {
  const int B = a.B;
  const int n3 = B * B * B;
  const uint8_t* m = a.marks + (size_t)blockIdx.x * n3;
  uint32_t nv = 0;
  for (int lin = threadIdx.x; lin < n3; lin += THREADS) nv += __popc(m[lin]);
  uint32_t total;
  block_excl_scan(nv, &total);
  if (threadIdx.x == 0) {
    a.bv[blockIdx.x] = total;
    if (total) atomicAdd(a.totals, (unsigned long long)total);
  }
}

// voxels of a block in consecutive runs per thread (voxel order = vertex / face order)
__device__ __forceinline__ void thread_run(int n3, int* l0, int* l1) {
  const int per = (n3 + THREADS - 1) / THREADS;
  *l0 = min((int)threadIdx.x * per, n3);
  *l1 = min(*l0 + per, n3);
}

template <bool FIELD>
__global__ void __launch_bounds__(THREADS) k_mc_emit_vertices(const MeshArgs a) {
  __shared__ int s_nbr[8], s_slot[8];
  load_neighbours<FIELD>(a, s_nbr, s_slot, false);
  const int B = a.B;
  const int n3 = B * B * B;
  const size_t p = blockIdx.x;
  const uint8_t* m = a.marks + p * n3;
  int l0, l1;
  thread_run(n3, &l0, &l1);
  uint32_t cnt = 0;
  for (int lin = l0; lin < l1; ++lin) cnt += __popc(m[lin]);
  uint32_t total;
  uint32_t id = a.bv_off[p] + block_excl_scan(cnt, &total);
  int b[3];
  unpack_key(a.keys[p], b);
  for (int lin = l0; lin < l1; ++lin) {
    const uint32_t mk = m[lin];
    a.vid[p * n3 + lin] = id;
    if (!mk) continue;
    const int li[3] = {lin % B, (lin / B) % B, lin / (B * B)};
    const float* bo = block_values<FIELD>(a, s_slot[0], n3);
    const float to = bo[lin];
    for (int ax = 0; ax < 3; ++ax) {
      if (!((mk >> ax) & 1u)) continue;
      int el;
      const int ec = locate(B, li[0] + (ax == 0), li[1] + (ax == 1), li[2] + (ax == 2), &el);
      const float* be = block_values<FIELD>(a, s_slot[ec], n3);
      const float te = be[el];
      if (FIELD) {
        // the two lattice points exactly as gof_field_grid_points computes them, and their values
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const int g = b[k] * B + li[k];
          a.edge_points[6 * (size_t)id + k] = __fmul_rn(__int2float_rn(g), a.s);
          a.edge_points[6 * (size_t)id + 3 + k] = __fmul_rn(__int2float_rn(k == ax ? g + 1 : g), a.s);
        }
        a.edge_values[2 * (size_t)id] = to;
        a.edge_values[2 * (size_t)id + 1] = te;
      } else {
        const float r = __fdiv_rn(__fsub_rn(0.f, to), __fsub_rn(te, to));
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const float g = __int2float_rn(b[k] * B + li[k]);
          a.vertices[3 * (size_t)id + k] = __fmul_rn(k == ax ? __fadd_rn(g, r) : g, a.s);
        }
        const float one_r = __fsub_rn(1.f, r);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch)
          a.colors[3 * (size_t)id + ch] = __fadd_rn(__fmul_rn(one_r, bo[(size_t)(2 + ch) * n3 + lin]), __fmul_rn(r, be[(size_t)(2 + ch) * n3 + el]));
      }
      ++id;
    }
  }
}

template <bool FIELD>
__global__ void __launch_bounds__(THREADS) k_mc_emit_faces(const MeshArgs a) {
  __shared__ int s_nbr[8], s_slot[8];
  load_neighbours<FIELD>(a, s_nbr, s_slot, false);
  const int B = a.B;
  const int n3 = B * B * B;
  const size_t p = blockIdx.x;
  int l0, l1;
  thread_run(n3, &l0, &l1);
  uint32_t cnt = 0;
  for (int lin = l0; lin < l1; ++lin) {
    uint32_t code;
    if (cube_code<FIELD>(a, s_nbr, s_slot, lin % B, (lin / B) % B, lin / (B * B), &code)) cnt += c_mc_ntri[code];
  }
  uint32_t total;
  size_t f = a.bf_off[p] + block_excl_scan(cnt, &total);
  for (int lin = l0; lin < l1; ++lin) {
    const int x = lin % B, y = (lin / B) % B, z = lin / (B * B);
    uint32_t code;
    if (!cube_code<FIELD>(a, s_nbr, s_slot, x, y, z, &code)) continue;
    const int nt = c_mc_ntri[code];
    for (int k = 0; k < 3 * nt; ++k) {
      const int e = c_mc_tri[code][k];
      const int o = c_mc_edge_owner[e];
      int ol;
      const int q = s_nbr[locate(B, x + (o & 1), y + ((o >> 1) & 1), z + ((o >> 2) & 1), &ol)];
      const size_t idx = (size_t)q * n3 + ol;
      const uint32_t below = a.marks[idx] & ((1u << (e >> 2)) - 1u);
      a.faces[3 * f + k] = (int64_t)(a.vid[idx] + __popc(below));
    }
    f += nt;
  }
}

static void mesh_args(int64_t n, const int64_t* keys, const int32_t* slots, const float* pool, int B, float s, float theta, char* S,
                      const MeshLayout& L, MeshArgs* a) {
  a->n = n; a->keys = keys; a->slots = slots; a->pool = pool; a->B = B; a->s = s; a->theta = theta;
  a->nbr = (int32_t*)(S + L.nbr); a->marks = (uint8_t*)(S + L.marks); a->vid = (uint32_t*)(S + L.vid);
  a->bv = (uint32_t*)(S + L.bv); a->bf = (uint32_t*)(S + L.bf);
  a->bv_off = (uint32_t*)(S + L.bv_off); a->bf_off = (uint32_t*)(S + L.bf_off);
  a->totals = (unsigned long long*)(S + L.header);
  a->vertices = nullptr; a->colors = nullptr; a->edge_points = nullptr; a->edge_values = nullptr; a->faces = nullptr;
}

// The count phase of either layout: marks, per-block counts and their scans; the totals, checked against the u32 ids.
template <bool FIELD>
static int mc_count(int64_t num_table, const int64_t* keys, const int32_t* slots, const float* pool, int B, float s, float theta,
                    gof_alloc_fn scratch_alloc, void* scratch_user, int64_t* num_vertices_out, int64_t* num_faces_out, const char* who,
                    cudaStream_t st) {
  const size_t n3 = (size_t)B * B * B;
  const MeshLayout L = mesh_layout((size_t)num_table, B);
  char* S = (char*)scratch_alloc(scratch_user, L.bytes);
  if (!S) { gof_set_error("scratch allocator returned NULL"); return GOF_E_ALLOC; }
  MeshArgs a;
  mesh_args(num_table, keys, slots, pool, B, s, theta, S, L, &a);
  MeshHeader* hd = (MeshHeader*)(S + L.header);
  GOF_CUDA_OK(cudaMemsetAsync(hd, 0, sizeof(MeshHeader), st));
  GOF_CUDA_OK(cudaMemsetAsync(a.marks, 0, (size_t)num_table * n3, st));
  const unsigned g = (unsigned)num_table;
  GOF_LAUNCH(FIELD ? "field_mc_mark" : "tsdf_mc_mark", st, k_mc_mark<FIELD><<<g, THREADS, 0, st>>>(a));
  GOF_LAUNCH_CHECK(false, st);
  GOF_LAUNCH(FIELD ? "field_mc_vcount" : "tsdf_mc_vcount", st, k_mc_vcount<<<g, THREADS, 0, st>>>(a));
  GOF_LAUNCH_CHECK(false, st);
  uint32_t* tmp = (uint32_t*)(S + L.scan_tmp);
  int rc;
  if ((rc = gof_exclusive_scan_u32(a.bv, a.bv_off, tmp, &hd->nv, (size_t)num_table, false, st)) != GOF_OK) return rc;
  if ((rc = gof_exclusive_scan_u32(a.bf, a.bf_off, tmp, &hd->nf, (size_t)num_table, false, st)) != GOF_OK) return rc;
  MeshHeader h;
  if ((rc = gof_read_back(&h, hd, sizeof(h), st)) != GOF_OK) return rc;
  // vertex ids live in u32 (per-voxel first ids, scanned offsets): the mesh must have fewer than 2^32 vertices and faces
  if (h.nv64 >= (1ull << 32) || h.nf64 >= (1ull << 32)) {
    gof_set_error("%s: %llu vertices / %llu faces; at most 2^32 - 1 of each are supported", who, h.nv64, h.nf64);
    return GOF_E_INVALID;
  }
  *num_vertices_out = (int64_t)h.nv64; *num_faces_out = (int64_t)h.nf64;
  return GOF_OK;
}

// The emit phase: `out` carries the caller's output pointers (vertices / colors or edge_points / edge_values, and faces).
template <bool FIELD>
static int mc_emit(int64_t num_table, const int64_t* keys, const int32_t* slots, const float* pool, int B, float s, float theta,
                   void* scratch, int64_t num_vertices, int64_t num_faces, const MeshArgs& out, const char* who, cudaStream_t st) {
  const MeshLayout L = mesh_layout((size_t)num_table, B);
  char* S = (char*)scratch;
  MeshHeader h;
  int rc;
  if ((rc = gof_read_back(&h, S + L.header, sizeof(h), st)) != GOF_OK) return rc;
  if ((int64_t)h.nv64 != num_vertices || (int64_t)h.nf64 != num_faces) {
    gof_set_error("%s: sizes do not match the count phase", who);
    return GOF_E_INVALID;
  }
  MeshArgs a;
  mesh_args(num_table, keys, slots, pool, B, s, theta, S, L, &a);
  a.vertices = out.vertices; a.colors = out.colors; a.edge_points = out.edge_points; a.edge_values = out.edge_values;
  a.faces = out.faces;
  const unsigned g = (unsigned)num_table;
  GOF_LAUNCH(FIELD ? "field_mc_vertices" : "tsdf_mc_vertices", st, k_mc_emit_vertices<FIELD><<<g, THREADS, 0, st>>>(a));
  GOF_LAUNCH_CHECK(false, st);
  if (num_faces > 0) {
    GOF_LAUNCH(FIELD ? "field_mc_faces" : "tsdf_mc_faces", st, k_mc_emit_faces<FIELD><<<g, THREADS, 0, st>>>(a));
    GOF_LAUNCH_CHECK(false, st);
  }
  return GOF_OK;
}

}  // namespace

// ---- C ABI -------------------------------------------------------------------------------------------------------

extern "C" __attribute__((visibility("default")))
int gof_tsdf_touch_count(const gof_tsdf_params_t* params, const gof_tsdf_camera_t* cam, const float* depth, gof_alloc_fn scratch_alloc,
                         void* scratch_user, int64_t* num_blocks_out, void* stream) {
  if (!num_blocks_out || !scratch_alloc || !cam || !depth) { gof_set_error("tsdf_touch_count: NULL argument"); return GOF_E_INVALID; }
  *num_blocks_out = 0;
  int rc;
  if ((rc = check_params(params, "tsdf_touch_count")) != GOF_OK) return rc;
  if (cam->width <= 0 || cam->height <= 0) { gof_set_error("tsdf_touch_count: empty image"); return GOF_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const Cam c = make_cam(cam);
  const Par p = make_par(params);
  const TouchLayout L = touch_layout(c.W, c.H, p);
  if (L.cap >= ((size_t)1 << 31)) { gof_set_error("tsdf_touch_count: image too large for the truncation / block size"); return GOF_E_INVALID; }
  char* S = (char*)scratch_alloc(scratch_user, L.bytes);
  if (!S) { gof_set_error("scratch allocator returned NULL"); return GOF_E_ALLOC; }
  TouchHeader* hd = (TouchHeader*)(S + L.header);
  uint32_t *cnt = (uint32_t*)(S + L.cnt), *off = (uint32_t*)(S + L.off), *tmp = (uint32_t*)(S + L.scan_tmp);
  GOF_CUDA_OK(cudaMemsetAsync(hd, 0, sizeof(TouchHeader), st));
  const int npix = (int)L.npix;
  const unsigned gp = (unsigned)((npix + THREADS - 1) / THREADS);
  GOF_LAUNCH("tsdf_touch_count", st, k_touch_count<<<gp, THREADS, 0, st>>>(npix, depth, c, p, cnt, hd));
  GOF_LAUNCH_CHECK(false, st);
  if ((rc = gof_exclusive_scan_u32(cnt, off, tmp, &hd->n_inst, L.npix, false, st)) != GOF_OK) return rc;
  TouchHeader h;
  if ((rc = gof_read_back(&h, hd, sizeof(h), st)) != GOF_OK) return rc;
  if (h.err & 1u) { gof_set_error("tsdf_touch_count: a touched block lies outside [-2^20, 2^20) per axis"); return GOF_E_INVALID; }
  if (h.err) { gof_set_error("tsdf_touch_count: a pixel touches more blocks per axis than 2 tau / (B s) + 2"); return GOF_E_INVALID; }
  const size_t I = h.n_inst;
  if (I == 0) return GOF_OK;
  uint32_t *lo = (uint32_t*)(S + L.lo), *hi = (uint32_t*)(S + L.hi);
  uint32_t *va = (uint32_t*)(S + L.val_a), *vb = (uint32_t*)(S + L.val_b), *hist = (uint32_t*)(S + L.hist);
  uint32_t *head = (uint32_t*)(S + L.head), *uid = (uint32_t*)(S + L.uid);
  GOF_LAUNCH("tsdf_touch_emit", st, k_touch_emit<<<gp, THREADS, 0, st>>>(npix, depth, c, p, cnt, off, lo, hi));
  GOF_LAUNCH_CHECK(false, st);
  // ascending 63-bit keys (the high word has 31 bits); head / uid are written only after the sort, so they are its key
  // buffers; the order lands in val_a
  const GofKeyWords key{{lo, hi, nullptr}, {32, 31, 0}, 2};
  if ((rc = gof_sort_words_u32(key, I, GofSortBufs{head, uid, va, vb, hist}, va, false, st)) != GOF_OK) return rc;
  if ((rc = gof_key_runs_u32(key, va, I, head, uid, tmp, &hd->n_unique, false, st)) != GOF_OK) return rc;
  if ((rc = gof_read_back(&h, hd, sizeof(h), st)) != GOF_OK) return rc;
  *num_blocks_out = (int64_t)h.n_unique;
  return GOF_OK;
}

extern "C" __attribute__((visibility("default")))
int gof_tsdf_touch_emit(const gof_tsdf_params_t* params, const gof_tsdf_camera_t* cam, void* scratch, int64_t num_blocks,
                        int64_t* keys_out, void* stream) {
  if (num_blocks == 0) return GOF_OK;
  if (!scratch || !cam || !keys_out) { gof_set_error("tsdf_touch_emit: NULL argument"); return GOF_E_INVALID; }
  int rc;
  if ((rc = check_params(params, "tsdf_touch_emit")) != GOF_OK) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const TouchLayout L = touch_layout(cam->width, cam->height, make_par(params));
  char* S = (char*)scratch;
  TouchHeader h;
  if ((rc = gof_read_back(&h, S + L.header, sizeof(h), st)) != GOF_OK) return rc;
  if ((int64_t)h.n_unique != num_blocks) { gof_set_error("tsdf_touch_emit: size does not match the count phase"); return GOF_E_INVALID; }
  const size_t I = h.n_inst;
  GOF_LAUNCH("tsdf_touch_keys", st, k_key_emit<<<(unsigned)((I + THREADS - 1) / THREADS), THREADS, 0, st>>>(
      I, (const uint32_t*)(S + L.lo), (const uint32_t*)(S + L.hi), (const uint32_t*)(S + L.val_a), (const uint32_t*)(S + L.head),
      (const uint32_t*)(S + L.uid), keys_out));
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}

extern "C" __attribute__((visibility("default")))
int gof_tsdf_activate_count(int64_t num_table, const int64_t* table_keys, int64_t num_view, const int64_t* view_keys,
                            gof_alloc_fn scratch_alloc, void* scratch_user, int64_t* num_new_out, void* stream) {
  if (!num_new_out || !scratch_alloc) { gof_set_error("tsdf_activate_count: NULL argument"); return GOF_E_INVALID; }
  *num_new_out = 0;
  if (num_view <= 0) return GOF_OK;
  if (!view_keys || num_table < 0 || (num_table > 0 && !table_keys)) { gof_set_error("tsdf_activate_count: NULL input"); return GOF_E_INVALID; }
  if (num_table + num_view >= ((int64_t)1 << 31)) { gof_set_error("tsdf_activate_count: more than 2^31 blocks"); return GOF_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const ActLayout L = act_layout((size_t)num_view);
  char* S = (char*)scratch_alloc(scratch_user, L.bytes);
  if (!S) { gof_set_error("scratch allocator returned NULL"); return GOF_E_ALLOC; }
  uint32_t* total = (uint32_t*)(S + L.header);
  GOF_LAUNCH("tsdf_activate_find", st, k_act_find<<<(unsigned)((num_view + THREADS - 1) / THREADS), THREADS, 0, st>>>(
      num_table, table_keys, num_view, view_keys, (int64_t*)(S + L.pos), (uint32_t*)(S + L.flag)));
  GOF_LAUNCH_CHECK(false, st);
  int rc;
  if ((rc = gof_exclusive_scan_u32((uint32_t*)(S + L.flag), (uint32_t*)(S + L.off), (uint32_t*)(S + L.scan_tmp), total,
                                   (size_t)num_view, false, st)) != GOF_OK)
    return rc;
  uint32_t n_new;
  if ((rc = gof_read_back(&n_new, total, 4, st)) != GOF_OK) return rc;
  *num_new_out = n_new;
  return GOF_OK;
}

extern "C" __attribute__((visibility("default")))
int gof_tsdf_activate_emit(int64_t num_table, const int64_t* table_keys, const int32_t* table_slots, int64_t num_view,
                           const int64_t* view_keys, void* scratch, int64_t num_new, int64_t* out_keys, int32_t* out_slots,
                           int32_t* view_slots, void* stream) {
  if (num_view <= 0) return GOF_OK;
  if (!scratch || !view_keys || !out_keys || !out_slots || !view_slots || (num_table > 0 && (!table_keys || !table_slots))) {
    gof_set_error("tsdf_activate_emit: NULL argument");
    return GOF_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const ActLayout L = act_layout((size_t)num_view);
  char* S = (char*)scratch;
  uint32_t n_new;
  int rc;
  if ((rc = gof_read_back(&n_new, S + L.header, 4, st)) != GOF_OK) return rc;
  if ((int64_t)n_new != num_new) { gof_set_error("tsdf_activate_emit: size does not match the count phase"); return GOF_E_INVALID; }
  const uint32_t* off = (const uint32_t*)(S + L.off);
  if (num_table > 0) {
    GOF_LAUNCH("tsdf_activate_old", st, k_act_merge_old<<<(unsigned)((num_table + THREADS - 1) / THREADS), THREADS, 0, st>>>(
        num_table, table_keys, table_slots, num_view, view_keys, off, n_new, out_keys, out_slots));
    GOF_LAUNCH_CHECK(false, st);
  }
  GOF_LAUNCH("tsdf_activate_new", st, k_act_merge_new<<<(unsigned)((num_view + THREADS - 1) / THREADS), THREADS, 0, st>>>(
      num_table, table_slots, num_view, view_keys, (const int64_t*)(S + L.pos), (const uint32_t*)(S + L.flag), off, out_keys, out_slots,
      view_slots));
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}

extern "C" __attribute__((visibility("default")))
int gof_tsdf_integrate(const gof_tsdf_params_t* params, const gof_tsdf_camera_t* cam, const float* depth, const float* color,
                       int64_t num_view, const int64_t* view_keys, const int32_t* view_slots, float* pool,
                       unsigned long long* num_updates, void* stream) {
  int rc;
  if ((rc = check_params(params, "tsdf_integrate")) != GOF_OK) return rc;
  if (num_view <= 0) return GOF_OK;
  if (!cam || !depth || !color || !view_keys || !view_slots || !pool) { gof_set_error("tsdf_integrate: NULL argument"); return GOF_E_INVALID; }
  if (cam->width <= 0 || cam->height <= 0) { gof_set_error("tsdf_integrate: empty image"); return GOF_E_INVALID; }
  if (num_view >= ((int64_t)1 << 31)) { gof_set_error("tsdf_integrate: too many blocks"); return GOF_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  GOF_LAUNCH("tsdf_integrate", st, k_integrate<<<(unsigned)num_view, THREADS, 0, st>>>(depth, color, make_cam(cam), make_par(params),
                                                                                      view_keys, view_slots, pool, num_updates));
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}

extern "C" __attribute__((visibility("default")))
int gof_tsdf_extract_count(const gof_tsdf_params_t* params, int64_t num_table, const int64_t* table_keys, const int32_t* table_slots,
                           const float* pool, float weight_threshold, gof_alloc_fn scratch_alloc, void* scratch_user,
                           int64_t* num_vertices_out, int64_t* num_faces_out, void* stream) {
  if (!num_vertices_out || !num_faces_out || !scratch_alloc) { gof_set_error("tsdf_extract_count: NULL argument"); return GOF_E_INVALID; }
  *num_vertices_out = 0; *num_faces_out = 0;
  int rc;
  if ((rc = check_params(params, "tsdf_extract_count")) != GOF_OK) return rc;
  if (num_table <= 0) return GOF_OK;
  if (!table_keys || !table_slots || !pool) { gof_set_error("tsdf_extract_count: NULL input"); return GOF_E_INVALID; }
  const Par p = make_par(params);
  return mc_count<false>(num_table, table_keys, table_slots, pool, p.B, p.s, weight_threshold, scratch_alloc, scratch_user,
                         num_vertices_out, num_faces_out, "tsdf_extract_count", (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default")))
int gof_tsdf_extract_emit(const gof_tsdf_params_t* params, int64_t num_table, const int64_t* table_keys, const int32_t* table_slots,
                          const float* pool, float weight_threshold, void* scratch, int64_t num_vertices, int64_t num_faces,
                          float* vertices, float* colors, int64_t* faces, void* stream) {
  int rc;
  if ((rc = check_params(params, "tsdf_extract_emit")) != GOF_OK) return rc;
  if (num_table <= 0 || (num_vertices == 0 && num_faces == 0)) return GOF_OK;
  if (!scratch || !table_keys || !table_slots || !pool || (num_vertices > 0 && (!vertices || !colors)) || (num_faces > 0 && !faces)) {
    gof_set_error("tsdf_extract_emit: NULL argument");
    return GOF_E_INVALID;
  }
  const Par p = make_par(params);
  MeshArgs out{};
  out.vertices = vertices; out.colors = colors; out.faces = faces;
  return mc_emit<false>(num_table, table_keys, table_slots, pool, p.B, p.s, weight_threshold, scratch, num_vertices, num_faces, out,
                        "tsdf_extract_emit", (cudaStream_t)stream);
}

// ---- marching cubes of the opacity field's lattice (DESIGN section 4.15; the lattice itself is field_grid.cu's) ---------

extern "C" __attribute__((visibility("default")))
int gof_field_grid_extract_count(const gof_field_grid_params_t* params, int64_t num_blocks, const int64_t* keys, const float* values,
                                 gof_alloc_fn scratch_alloc, void* scratch_user, int64_t* num_vertices_out, int64_t* num_faces_out,
                                 void* stream) {
  if (!num_vertices_out || !num_faces_out || !scratch_alloc) { gof_set_error("field_grid_extract_count: NULL argument"); return GOF_E_INVALID; }
  *num_vertices_out = 0; *num_faces_out = 0;
  int rc;
  if ((rc = field_grid_check_params(params, "field_grid_extract_count")) != GOF_OK) return rc;
  if ((rc = field_grid_check_points(params, num_blocks, "field_grid_extract_count")) != GOF_OK) return rc;
  if (num_blocks == 0) return GOF_OK;
  if (!keys || !values) { gof_set_error("field_grid_extract_count: NULL input"); return GOF_E_INVALID; }
  return mc_count<true>(num_blocks, keys, nullptr, values, params->block_resolution, params->voxel_size, 0.f, scratch_alloc, scratch_user,
                        num_vertices_out, num_faces_out, "field_grid_extract_count", (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default")))
int gof_field_grid_extract_emit(const gof_field_grid_params_t* params, int64_t num_blocks, const int64_t* keys, const float* values,
                                void* scratch, int64_t num_vertices, int64_t num_faces, float* edge_points, float* edge_values,
                                int64_t* faces, void* stream) {
  int rc;
  if ((rc = field_grid_check_params(params, "field_grid_extract_emit")) != GOF_OK) return rc;
  if ((rc = field_grid_check_points(params, num_blocks, "field_grid_extract_emit")) != GOF_OK) return rc;
  if (num_blocks == 0 || (num_vertices == 0 && num_faces == 0)) return GOF_OK;
  if (!scratch || !keys || !values || (num_vertices > 0 && (!edge_points || !edge_values)) || (num_faces > 0 && !faces)) {
    gof_set_error("field_grid_extract_emit: NULL argument");
    return GOF_E_INVALID;
  }
  MeshArgs out{};
  out.edge_points = edge_points; out.edge_values = edge_values; out.faces = faces;
  return mc_emit<true>(num_blocks, keys, nullptr, values, params->block_resolution, params->voxel_size, 0.f, scratch, num_vertices,
                       num_faces, out, "field_grid_extract_emit", (cudaStream_t)stream);
}
