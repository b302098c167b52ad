// tetmesh.cu -- marching tetrahedra on the GPU without torch.unique.
//
// Reference: utils/tetmesh.py:47-138.  It builds all 6 edges of every valid tet, torch.unique(dim=0)s them (a sort of
// int64 pairs plus an inverse map), keeps the edges with exactly one occupied endpoint and renumbers them, then
// gathers faces through the triangle table, all 1-triangle tets before all 2-triangle tets (per chunk of 32 Mi tets).
// Here only the CROSSING edges are ever materialised (3 or 4 per valid tet; the others are never referenced by the
// triangle table), as (lo, hi) u32 pairs sorted with two rounds of the library's stable u32 radix sort; unique ids come
// from head flags + a scan, so interp_v is the same lexicographically sorted list the reference produces, and faces
// are written at offsets given by scans of the 1-/2-triangle flags, reproducing the reference's face order exactly.
#include "gof_common.cuh"

namespace {

__constant__ int8_t c_tri[16][6] = {   // utils/tetmesh.py:23-40
    {-1, -1, -1, -1, -1, -1}, {1, 0, 2, -1, -1, -1}, {4, 0, 3, -1, -1, -1}, {1, 4, 2, 1, 3, 4},
    {3, 1, 5, -1, -1, -1},    {2, 3, 0, 2, 5, 3},    {1, 4, 0, 1, 5, 4},    {4, 2, 5, -1, -1, -1},
    {4, 5, 2, -1, -1, -1},    {4, 1, 0, 4, 5, 1},    {3, 2, 0, 3, 5, 2},    {1, 3, 5, -1, -1, -1},
    {4, 1, 2, 4, 3, 1},       {3, 0, 4, -1, -1, -1}, {2, 0, 1, -1, -1, -1}, {-1, -1, -1, -1, -1, -1}};
__constant__ int8_t c_ntri[16] = {0, 1, 1, 2, 1, 2, 2, 1, 1, 2, 2, 1, 2, 1, 1, 0};   // :42
// base_tet_edges (:43): slot s joins local vertices (EA[s], EB[s])
__device__ __constant__ int8_t c_ea[6] = {0, 0, 0, 1, 1, 2};
__device__ __constant__ int8_t c_eb[6] = {1, 2, 3, 2, 3, 3};

struct TetLayout {   // scratch layout, a function of (T, capacity of edge instances = 4T)
  size_t header, code, cross, f1, f2, cross_off, f1_off, f2_off, scan_tmp;
  size_t lo_a, lo_b, hi, val_a, val_b, hist, head, uid_sorted, inst_uid, bytes;
};

static TetLayout tet_layout(size_t T) {
  TetLayout L; size_t o = 0;
  auto take = [&](size_t b) { size_t r = o; o = gof_align_up(o + b, 256); return r; };
  const size_t I = 4 * T;   // upper bound on crossing-edge instances
  L.header = take(256);
  L.code = take(T);
  L.cross = take(T * 4); L.f1 = take(T * 4); L.f2 = take(T * 4);
  L.cross_off = take(T * 4); L.f1_off = take(T * 4); L.f2_off = take(T * 4);
  L.scan_tmp = take((I / 2048 + 4) * 4 + 4096);
  L.lo_a = take(I * 4); L.lo_b = take(I * 4); L.hi = take(I * 4);
  L.val_a = take(I * 4); L.val_b = take(I * 4);
  L.hist = take(gof_sort_scratch_bytes(I));
  L.head = take(I * 4); L.uid_sorted = take(I * 4); L.inst_uid = take(I * 4);
  L.bytes = o;
  return L;
}

struct Header { uint32_t n_inst, n1, n2, n_edges; };

__device__ __forceinline__ uint32_t occ_code(const float* __restrict__ sdf, const int64_t* __restrict__ tet, uint32_t* v) {
  uint32_t code = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    v[k] = (uint32_t)tet[k];
    code |= (sdf[v[k]] > 0.f ? 1u : 0u) << k;
  }
  return code;
}

__global__ void __launch_bounds__(256) k_tet_classify(int64_t T, const float* __restrict__ sdf, const int64_t* __restrict__ tets,
                                                     unsigned char* __restrict__ code_out, uint32_t* __restrict__ cross,
                                                     uint32_t* __restrict__ f1, uint32_t* __restrict__ f2) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  uint32_t v[4];
  const uint32_t code = occ_code(sdf, tets + 4 * t, v);
  const int k = __popc(code);
  const bool valid = k > 0 && k < 4;
  code_out[t] = valid ? (unsigned char)code : 0;
  cross[t] = valid ? (uint32_t)(k * (4 - k)) : 0u;       // 3 or 4 edges join an occupied and a free vertex
  const int nt = c_ntri[code];
  f1[t] = nt == 1; f2[t] = nt == 2;
}

// one thread per tet: write its crossing edges (sorted endpoints) in base-edge order at cross_off[t]
__global__ void __launch_bounds__(256) k_tet_edges(int64_t T, const int64_t* __restrict__ tets, const unsigned char* __restrict__ code,
                                                  const uint32_t* __restrict__ cross_off, uint32_t* __restrict__ lo,
                                                  uint32_t* __restrict__ hi, uint32_t* __restrict__ val) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const uint32_t c = code[t];
  if (!c) return;
  uint32_t v[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = (uint32_t)tets[4 * t + k];
  uint32_t o = cross_off[t];
#pragma unroll
  for (int s = 0; s < 6; ++s) {
    const int a = c_ea[s], b = c_eb[s];
    if (((c >> a) ^ (c >> b)) & 1u) {
      const uint32_t x = v[a], y = v[b];
      lo[o] = x < y ? x : y;      // first column of the sorted pair
      hi[o] = x < y ? y : x;      // second column
      val[o] = o;
      ++o;
    }
  }
}

__global__ void __launch_bounds__(256) k_gather_u32(size_t n, const uint32_t* __restrict__ src, const uint32_t* __restrict__ idx,
                                                   uint32_t* __restrict__ dst) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[idx[i]];
}

// sorted order `ord`: head[j] = 1 when (lo,hi)[ord[j]] differs from its predecessor
__global__ void __launch_bounds__(256) k_heads(size_t n, const uint32_t* __restrict__ lo, const uint32_t* __restrict__ hi,
                                              const uint32_t* __restrict__ ord, uint32_t* __restrict__ head) {
  const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  if (j == 0) { head[0] = 1; return; }
  const uint32_t a = ord[j], b = ord[j - 1];
  head[j] = (lo[a] != lo[b] || hi[a] != hi[b]) ? 1u : 0u;
}

// uid_sorted = exclusive scan of head; unique id of sorted position j is uid_sorted[j] + head[j] - 1
__global__ void __launch_bounds__(256) k_scatter_uid(size_t n, const uint32_t* __restrict__ ord, const uint32_t* __restrict__ head,
                                                    const uint32_t* __restrict__ uid_sorted, uint32_t* __restrict__ inst_uid) {
  const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) inst_uid[ord[j]] = uid_sorted[j] + head[j] - 1u;
}

struct EmitArgs {
  int64_t T, chunk;
  const int64_t* tets;
  const unsigned char* code;
  const uint32_t *cross_off, *f1_off, *f2_off, *inst_uid;
  const uint32_t *lo, *hi, *ord, *head, *uid_sorted;
  size_t n_inst;
  int64_t* interp_v;
  int64_t* faces;
  const float *vertices, *sdf, *scales;
  float *edge_pos, *edge_sdf, *edge_scales;
};

__global__ void __launch_bounds__(256) k_emit_edges(const EmitArgs a) {
  const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= a.n_inst || !a.head[j]) return;
  const uint32_t e = a.uid_sorted[j];
  const uint32_t i = a.ord[j];
  const uint32_t v0 = a.lo[i], v1 = a.hi[i];
  a.interp_v[2 * (size_t)e] = (int64_t)v0;
  a.interp_v[2 * (size_t)e + 1] = (int64_t)v1;
  if (a.edge_pos) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      a.edge_pos[6 * (size_t)e + k] = a.vertices[3 * (size_t)v0 + k];
      a.edge_pos[6 * (size_t)e + 3 + k] = a.vertices[3 * (size_t)v1 + k];
    }
  }
  if (a.edge_sdf) { a.edge_sdf[2 * (size_t)e] = a.sdf[v0]; a.edge_sdf[2 * (size_t)e + 1] = a.sdf[v1]; }
  if (a.edge_scales) { a.edge_scales[2 * (size_t)e] = a.scales[v0]; a.edge_scales[2 * (size_t)e + 1] = a.scales[v1]; }
}

// faces of tet t: in chunk c = t / chunk the 1-triangle tets come first, then the 2-triangle tets (tetmesh.py:131-136)
__global__ void __launch_bounds__(256) k_emit_faces(const EmitArgs a) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= a.T) return;
  const uint32_t c = a.code[t];
  if (!c) return;
  const int nt = c_ntri[c];
  const int64_t c0 = (t / a.chunk) * a.chunk;                      // first tet of this chunk
  const int64_t c1 = min(c0 + a.chunk, a.T);                       // one past its last tet
  const uint64_t f1_before = a.f1_off[c0], f2_before = a.f2_off[c0];
  // faces of all earlier chunks + this chunk's 1-triangle block (+ earlier 2-triangle tets of this chunk)
  const uint64_t f1_chunk_end = (c1 < a.T) ? a.f1_off[c1] : (uint64_t)a.f1_off[a.T - 1] + (c_ntri[a.code[a.T - 1]] == 1);
  uint64_t face;
  if (nt == 1) face = f1_before + 2 * f2_before + (a.f1_off[t] - f1_before);
  else face = f1_chunk_end + 2 * f2_before + 2 * (uint64_t)(a.f2_off[t] - f2_before);
  // crossing-edge slot -> instance index: rank of the slot among this tet's crossing slots
  int rank[6];
  int r = 0;
#pragma unroll
  for (int s = 0; s < 6; ++s) {
    const bool crossing = ((c >> c_ea[s]) ^ (c >> c_eb[s])) & 1u;
    rank[s] = crossing ? r : -1;
    r += crossing;
  }
  const uint32_t base = a.cross_off[t];
  for (int k = 0; k < 3 * nt; ++k) {
    const int slot = c_tri[c][k];
    a.faces[3 * face + k] = (int64_t)a.inst_uid[base + rank[slot]];
  }
}

}  // namespace

extern "C" __attribute__((visibility("default")))
int gof_marching_tets_count(int num_verts, const float* sdf, int64_t num_tets, const int64_t* tets, int64_t chunk_tets,
                            gof_alloc_fn scratch_alloc, void* scratch_user, int64_t* num_edges_out, int64_t* num_faces_out,
                            void* stream) {
  (void)chunk_tets;
  if (!num_edges_out || !num_faces_out || !scratch_alloc) { gof_set_error("marching_tets_count: NULL argument"); return GOF_E_INVALID; }
  *num_edges_out = 0; *num_faces_out = 0;
  if (num_tets <= 0) return GOF_OK;
  if (!sdf || !tets || num_verts <= 0) { gof_set_error("marching_tets_count: NULL input"); return GOF_E_INVALID; }
  if (num_tets > (int64_t)1 << 30) { gof_set_error("marching_tets_count: more than 2^30 tets unsupported"); return GOF_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const size_t T = (size_t)num_tets;
  const TetLayout L = tet_layout(T);
  char* S = (char*)scratch_alloc(scratch_user, L.bytes);
  if (!S) { gof_set_error("scratch allocator returned NULL"); return GOF_E_ALLOC; }
  unsigned char* code = (unsigned char*)(S + L.code);
  uint32_t *cross = (uint32_t*)(S + L.cross), *f1 = (uint32_t*)(S + L.f1), *f2 = (uint32_t*)(S + L.f2);
  uint32_t *cross_off = (uint32_t*)(S + L.cross_off), *f1_off = (uint32_t*)(S + L.f1_off), *f2_off = (uint32_t*)(S + L.f2_off);
  uint32_t* tmp = (uint32_t*)(S + L.scan_tmp);
  Header* hd = (Header*)(S + L.header);
  GOF_CUDA_OK(cudaMemsetAsync(hd, 0, sizeof(Header), st));   // n_edges is read back (with the rest) before it is written
  const unsigned grid = (unsigned)((T + 255) / 256);
  GOF_LAUNCH("tet_classify", st, k_tet_classify<<<grid, 256, 0, st>>>(num_tets, sdf, tets, code, cross, f1, f2));
  GOF_LAUNCH_CHECK(false, st);
  int rc;
  if ((rc = gof_exclusive_scan_u32(cross, cross_off, tmp, &hd->n_inst, T, false, st)) != GOF_OK) return rc;
  if ((rc = gof_exclusive_scan_u32(f1, f1_off, tmp, &hd->n1, T, false, st)) != GOF_OK) return rc;
  if ((rc = gof_exclusive_scan_u32(f2, f2_off, tmp, &hd->n2, T, false, st)) != GOF_OK) return rc;
  Header h;
  { const int rb = gof_read_back(&h, hd, sizeof(Header), st); if (rb != GOF_OK) return rb; }
  *num_faces_out = (int64_t)h.n1 + 2 * (int64_t)h.n2;
  const size_t I = h.n_inst;
  if (I == 0) return GOF_OK;
  uint32_t *lo_a = (uint32_t*)(S + L.lo_a), *lo_b = (uint32_t*)(S + L.lo_b), *hi = (uint32_t*)(S + L.hi);
  uint32_t *va = (uint32_t*)(S + L.val_a), *vb = (uint32_t*)(S + L.val_b), *hist = (uint32_t*)(S + L.hist);
  uint32_t *head = (uint32_t*)(S + L.head), *uid_sorted = (uint32_t*)(S + L.uid_sorted), *inst_uid = (uint32_t*)(S + L.inst_uid);
  // lo_b doubles as the unsorted copy of the first column: edges are written to (lo_b, hi), sorted through (lo_a, ...)
  GOF_LAUNCH("tet_edges", st, k_tet_edges<<<grid, 256, 0, st>>>(num_tets, tets, code, cross_off, lo_b, hi, va));
  GOF_LAUNCH_CHECK(false, st);
  const int vbits = gof_bits_for((uint32_t)num_verts);
  const unsigned gi = (unsigned)((I + 255) / 256);
  // round 1: stable sort of instance ids by the SECOND column
  uint32_t* k1a = head;          // reuse head / uid_sorted as key ping-pong for the two rounds
  uint32_t* k1b = uid_sorted;
  GOF_CUDA_OK(cudaMemcpyAsync(k1a, hi, I * 4, cudaMemcpyDeviceToDevice, st));
  int in_b = 0;
  if ((rc = gof_sort_pairs_u32(k1a, k1b, va, vb, hist, I, vbits, false, st, &in_b)) != GOF_OK) return rc;
  uint32_t* ord1 = in_b ? vb : va;
  uint32_t* ord1_other = in_b ? va : vb;
  // round 2: stable sort of that order by the FIRST column -> lexicographic (first, second) order
  GOF_LAUNCH("tet_gather", st, k_gather_u32<<<gi, 256, 0, st>>>(I, lo_b, ord1, k1a));
  GOF_LAUNCH_CHECK(false, st);
  if (ord1 != va) GOF_CUDA_OK(cudaMemcpyAsync(va, ord1, I * 4, cudaMemcpyDeviceToDevice, st));
  (void)ord1_other;
  if ((rc = gof_sort_pairs_u32(k1a, k1b, va, vb, hist, I, vbits, false, st, &in_b)) != GOF_OK) return rc;
  uint32_t* ord = in_b ? vb : va;
  if (ord != lo_a) GOF_CUDA_OK(cudaMemcpyAsync(lo_a, ord, I * 4, cudaMemcpyDeviceToDevice, st));   // final order lives in lo_a
  GOF_LAUNCH("tet_heads", st, k_heads<<<gi, 256, 0, st>>>(I, lo_b, hi, lo_a, head));
  GOF_LAUNCH_CHECK(false, st);
  if ((rc = gof_exclusive_scan_u32(head, uid_sorted, tmp, &hd->n_edges, I, false, st)) != GOF_OK) return rc;
  GOF_LAUNCH("tet_uid", st, k_scatter_uid<<<gi, 256, 0, st>>>(I, lo_a, head, uid_sorted, inst_uid));
  GOF_LAUNCH_CHECK(false, st);
  { const int rb = gof_read_back(&h, hd, sizeof(Header), st); if (rb != GOF_OK) return rb; }
  *num_edges_out = (int64_t)h.n_edges;
  return GOF_OK;
}

extern "C" __attribute__((visibility("default")))
int gof_marching_tets_emit(int num_verts, const float* sdf, int64_t num_tets, const int64_t* tets, int64_t chunk_tets, void* scratch,
                           int64_t num_edges, int64_t num_faces, int64_t* interp_v, int64_t* faces, const float* vertices,
                           const float* scales, float* edge_pos, float* edge_sdf, float* edge_scales, void* stream) {
  (void)num_verts;
  if (num_tets <= 0 || (num_edges == 0 && num_faces == 0)) return GOF_OK;
  if (!scratch || !tets || !sdf || (num_edges > 0 && !interp_v) || (num_faces > 0 && !faces)) {
    gof_set_error("marching_tets_emit: NULL argument");
    return GOF_E_INVALID;
  }
  if ((edge_pos && !vertices) || (edge_scales && !scales)) { gof_set_error("marching_tets_emit: gather source missing"); return GOF_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const size_t T = (size_t)num_tets;
  const TetLayout L = tet_layout(T);
  char* S = (char*)scratch;
  Header h;
  { const int rb = gof_read_back(&h, S + L.header, sizeof(Header), st); if (rb != GOF_OK) return rb; }
  if ((int64_t)h.n_edges != num_edges || (int64_t)h.n1 + 2 * (int64_t)h.n2 != num_faces) {
    gof_set_error("marching_tets_emit: sizes do not match the count phase");
    return GOF_E_INVALID;
  }
  EmitArgs a{};
  // rows per chunk: the reference splits with torch.chunk(tets, T // chunk_size + 1) (utils/tetmesh.py:56-58), i.e. ceil(T / n)
  // rows; a NEGATIVE chunk_tets states the rows per chunk directly (tet-sharded extraction: every shard must cut where the
  // unsharded call cuts)
  a.T = num_tets;
  if (chunk_tets < 0) a.chunk = -chunk_tets;
  else a.chunk = (chunk_tets > 0 && num_tets > chunk_tets) ? (num_tets + (num_tets / chunk_tets + 1) - 1) / (num_tets / chunk_tets + 1) : num_tets;
  a.tets = tets; a.code = (unsigned char*)(S + L.code);
  a.cross_off = (uint32_t*)(S + L.cross_off); a.f1_off = (uint32_t*)(S + L.f1_off); a.f2_off = (uint32_t*)(S + L.f2_off);
  a.inst_uid = (uint32_t*)(S + L.inst_uid); a.lo = (uint32_t*)(S + L.lo_b); a.hi = (uint32_t*)(S + L.hi);
  a.ord = (uint32_t*)(S + L.lo_a); a.head = (uint32_t*)(S + L.head); a.uid_sorted = (uint32_t*)(S + L.uid_sorted);
  a.n_inst = h.n_inst; a.interp_v = interp_v; a.faces = faces; a.vertices = vertices; a.sdf = sdf; a.scales = scales;
  a.edge_pos = edge_pos; a.edge_sdf = edge_sdf; a.edge_scales = edge_scales;
  if (h.n_inst) {
    GOF_LAUNCH("tet_emit_edges", st, k_emit_edges<<<(unsigned)((h.n_inst + 255) / 256), 256, 0, st>>>(a));
    GOF_LAUNCH_CHECK(false, st);
  }
  GOF_LAUNCH("tet_emit_faces", st, k_emit_faces<<<(unsigned)((T + 255) / 256), 256, 0, st>>>(a));
  GOF_LAUNCH_CHECK(false, st);
  return GOF_OK;
}
