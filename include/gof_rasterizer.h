/*
 * gof_rasterizer.h -- C ABI of the H100-native Gaussian-opacity-field rasterizer (libgof_b200.so).
 *
 * Drop-in boundary for the reference's `CudaRasterizer::Rasterizer` static interface
 * (reference: submodules/diff-gaussian-rasterization/cuda_rasterizer/rasterizer.h:20-124) and for the
 * four pybind entry points built on it (rasterize_points.h:18-98, ext.cpp:16-19).  Plain pointers and
 * sizes only; no torch / C++ types.  All pointers are DEVICE pointers unless stated otherwise; "absent"
 * optional inputs are NULL (the reference receives empty CPU tensors whose data_ptr() is nullptr,
 * rasterize_points.cu:98-115).  All functions return 0 on success, a negative GOF_E_* code on failure;
 * gof_last_error() gives the message.  Kernels are enqueued on `stream` (a cudaStream_t passed as void*,
 * NULL = legacy default stream as in the reference, forward.cu:637).
 *
 * Scratch memory follows the reference's convention (rasterizer.h:31-56: std::function<char*(size_t)>):
 * the library calls a caller-provided allocator once per buffer with the exact byte count and the
 * caller keeps the three opaque buffers alive until backward has run.  Layouts are private to this
 * library (gof_export_state() converts to the reference's field layout for parity tests).
 */
#ifndef GOF_RASTERIZER_H_INCLUDED
#define GOF_RASTERIZER_H_INCLUDED

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define GOF_API __attribute__((visibility("default")))
#else
#define GOF_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define GOF_OUTPUT_CHANNELS 9   /* auxiliary.h:24 : rgb(3) normal(3) depth alpha distortion */
#define GOF_TILE 16             /* config.h:16-17 BLOCK_X = BLOCK_Y = 16 */

enum {
  GOF_OK = 0,
  GOF_E_INVALID = -1,   /* bad argument combination (mirrors AT_ERROR / std::runtime_error sites) */
  GOF_E_CUDA = -2,      /* a CUDA call or (with debug=1) a kernel failed */
  GOF_E_ALLOC = -3      /* the allocator callback returned NULL */
};

/* rasterizer.h:31-33 : std::function<char*(size_t N)> geometryBuffer / binningBuffer / imageBuffer.
 * Must return a device pointer aligned to >= 256 bytes valid for `bytes` bytes (bytes may be 0). */
typedef void* (*gof_alloc_fn)(void* user, size_t bytes);

/* One view + one Gaussian set: the argument list shared by Rasterizer::forward / backward / integrate
 * (rasterizer_impl.cu:247-272, 409-442, 530-560). */
typedef struct gof_scene {
  int P;                /* number of Gaussians                                   (means3D.size(0)) */
  int D;                /* active SH degree 0..3                                 (raster_settings.sh_degree) */
  int M;                /* SH coefficients stored per Gaussian, 0 if shs absent  (sh.size(1)) */
  int width, height;    /* image size in pixels */
  float tan_fovx, tan_fovy;
  float kernel_size;    /* 2D mip filter added to the screen-space covariance diagonal */
  float scale_modifier;
  const float* background;            /* [3] */
  const float* means3D;               /* [P,3] */
  const float* shs;                   /* [P,M,3] or NULL */
  const float* colors_precomp;        /* [P,3]   or NULL (exactly one of shs / colors_precomp) */
  const float* opacities;             /* [P] */
  const float* scales;                /* [P,3]   or NULL */
  const float* rotations;             /* [P,4] (r,x,y,z), used as given (not re-normalised) or NULL */
  const float* cov3D_precomp;         /* [P,6]   or NULL */
  const float* view2gaussian_precomp; /* [P,10]  or NULL */
  const float* viewmatrix;            /* [16] column-major world->view  */
  const float* projmatrix;            /* [16] column-major full projection */
  const float* cam_pos;               /* [3] */
  const float* subpixel_offset;       /* [H,W,2]; accepted for signature parity, never read by forward */
  int prefiltered;
  int debug;                          /* 1: synchronise + check after every launch (auxiliary.h:204-211) */
} gof_scene_t;

/* Rasterizer::forward (rasterizer_impl.cu:247-405) == _C.rasterize_gaussians.
 * out_color [9,H,W] and radii [P] must be zero-initialised by the caller (rasterize_points.cu:72-73).
 * *num_rendered (HOST int) receives the number of (Gaussian,tile) instances. */
GOF_API int gof_rasterize_forward(const gof_scene_t* scene,
                          gof_alloc_fn geom_alloc, void* geom_user,
                          gof_alloc_fn binning_alloc, void* binning_user,
                          gof_alloc_fn image_alloc, void* image_user,
                          float* out_color, int* radii, int* num_rendered, void* stream);

/* Rasterizer::backward (rasterizer_impl.cu:409-526) == _C.rasterize_gaussians_backward.
 * All dL_d* outputs must be zero-initialised by the caller (rasterize_points.cu:161-170).
 * dL_dconic [P,4] and dL_dcov3D [P,6] are accepted and left untouched (the reference's EWA backward
 * is disabled, backward.cu:991-1007, 627-630).  dL_dsh may be NULL when M == 0.
 * geom_buffer is the forward's geometry scratch: the backward reads the forward state in it and uses its last
 * section (64 bytes per Gaussian) as accumulator rows, re-zeroed by every call -- hence not const. */
GOF_API int gof_rasterize_backward(const gof_scene_t* scene, int num_rendered, const int* radii,
                           void* geom_buffer, const void* binning_buffer, const void* image_buffer,
                           const float* dL_dpix,        /* [9,H,W] */
                           float* dL_dmean2D,           /* [P,3] */
                           float* dL_dconic,            /* [P,4]  untouched */
                           float* dL_dopacity,          /* [P] */
                           float* dL_dcolor,            /* [P,3] */
                           float* dL_dmean3D,           /* [P,3] */
                           float* dL_dcov3D,            /* [P,6]  untouched */
                           float* dL_dsh,               /* [P,M,3] */
                           float* dL_dscale,            /* [P,3] */
                           float* dL_drot,              /* [P,4] */
                           float* dL_dview2gaussian,    /* [P,10] */
                           void* stream);

/* gof_rasterize_backward that also leaves this view's densification statistics next to the gradients (view-parallel training
 * reduces them in the same exchange): dens_sum [P,3] = (|dL_dmean2D.xy|, |dL_dmean2D.z|, 1) and dens_max [P,2] =
 * (|dL_dmean2D.z|, radius) for visible Gaussians -- what GaussianModel.add_densification_stats (scene/gaussian_model.py:709-714)
 * and train.py:255 accumulate per view with SUM resp. MAX.  Rows of invisible Gaussians are written as zeros (like every
 * gradient output: no pre-zeroing needed).  Both NULL: plain gof_rasterize_backward. */
GOF_API int gof_rasterize_backward_stats(const gof_scene_t* scene, int num_rendered, const int* radii, void* geom_buffer,
                           const void* binning_buffer, const void* image_buffer, const float* dL_dpix, float* dL_dmean2D,
                           float* dL_dconic, float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D,
                           float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dview2gaussian, float* dens_sum,
                           float* dens_max, void* stream);

/* View-parallel training (one view per GPU, gradients summed over the GPUs; no reference counterpart -- the reference is
 * single-GPU).  The SH gradient of ONE view is an outer product: dL_dsh[g][k][c] = w_k(dir(mean_g, camera)) * dL_dRGB[g][c]
 * (backward.cu:45-139), so the ranks exchange the 3 floats of the clamp-masked dL_dRGB per Gaussian and view instead of the
 * 48 of dL_dsh and every rank expands the sum over the views itself (gof_sh_grad_from_views).
 * gof_rasterize_backward_dp = gof_rasterize_backward_stats that additionally writes sh_rgb -- three colour planes
 * [3][GOF_SH_PLANE(P)], zeros for invisible Gaussians -- and sh_hdr[0..3] = camera centre, active SH degree; with both given
 * dL_dsh may be NULL (it is then not computed). */
#define GOF_SH_PLANE(P) ((((size_t)(P)) + 63u) / 64u * 64u)
GOF_API int gof_rasterize_backward_dp(const gof_scene_t* scene, int num_rendered, const int* radii, void* geom_buffer,
                           const void* binning_buffer, const void* image_buffer, const float* dL_dpix, float* dL_dmean2D,
                           float* dL_dconic, float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D,
                           float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dview2gaussian, float* dens_sum,
                           float* dens_max, float* sh_rgb, float* sh_hdr, void* stream);
/* dL_dsh [P,M,3] = sum over v = 0..n_views-1, in that order, of w(dir(means3D, camera_v)) (x) rgb_v, bit-identical to adding the
 * views' own dL_dsh in that order; coefficients above the active degree are written as zeros.  slots[v] points to view v's
 * record: 64 floats of header (sh_hdr as written by gof_rasterize_backward_dp) followed by the planes [3][GOF_SH_PLANE(P)]; the pointers may address
 * peer GPUs' memory (NVLink): the records are then read where the ranks left them, without a gather step. */
#define GOF_SH_SLOT_HEADER 64
GOF_API int gof_sh_grad_from_views(int P, int M, int n_views, const float* means3D, const float* const* slots, float* dL_dsh,
                           void* stream);

/* Rasterizer::integrate (rasterizer_impl.cu:530-792) == _C.integrate_gaussians_to_points.
 * out_alpha_integrated [PN] must be initialised to 1 and out_color_integrated [PN,3] to 0 by the
 * caller (rasterize_points.cu:277-278); out_color / radii zero-initialised. */
GOF_API int gof_integrate(const gof_scene_t* scene, int PN, const float* points3D,
                  gof_alloc_fn geom_alloc, void* geom_user,
                  gof_alloc_fn binning_alloc, void* binning_user,
                  gof_alloc_fn image_alloc, void* image_user,
                  gof_alloc_fn point_alloc, void* point_user,
                  gof_alloc_fn point_binning_alloc, void* point_binning_user,
                  float* out_color, int* radii,
                  float* out_alpha_integrated, float* out_color_integrated,
                  int* num_rendered, void* stream);

/* The same query with the Gaussian side cached per view.  extract_mesh.py:56,92,107 calls integrate for the SAME views ten
 * times (tetrahedra vertices, 8 bisection steps, colours) -- only points3D changes, so preprocess / depth sort / instance
 * emission / tile sort of the Gaussians (rasterizer_impl.cu:566-660) are identical in every pass.
 *   gof_integrate_prepare: runs them once; `cache_alloc` is called once with gof_integrate_cache_bytes(P, W, H, *num_rendered)
 *                          and receives records, tile ranges and per-tile lists (64 B/Gaussian + 4 B/instance + 8 B/tile);
 *                          geom / binning / image buffers are scratch that may be released after the call; radii [P] out.
 *   gof_integrate_cached:  the point side alone (rasterizer_impl.cu:662-792) against such a cache; of `scene` only P, width,
 *                          height, tan_fovx/y, viewmatrix, background and debug are read.  Outputs as gof_integrate. */
GOF_API size_t gof_integrate_cache_bytes(int P, int width, int height, int num_rendered);
GOF_API int gof_integrate_prepare(const gof_scene_t* scene, gof_alloc_fn geom_alloc, void* geom_user,
                  gof_alloc_fn binning_alloc, void* binning_user, gof_alloc_fn image_alloc, void* image_user,
                  gof_alloc_fn cache_alloc, void* cache_user, int* radii, int* num_rendered, void* stream);
GOF_API int gof_integrate_cached(const gof_scene_t* scene, int PN, const float* points3D, const void* cache, int num_rendered,
                  gof_alloc_fn image_alloc, void* image_user, gof_alloc_fn point_alloc, void* point_user,
                  gof_alloc_fn point_binning_alloc, void* point_binning_user, float* out_color,
                  float* out_alpha_integrated, float* out_color_integrated, void* stream);

/* Rasterizer::markVisible (rasterizer_impl.cu:174-186) == _C.mark_visible.  present: [P] bytes (bool). */
GOF_API int gof_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                     unsigned char* present, void* stream);

/* Parity-test helper: converts this library's private scratch layout into the reference's field
 * layout (rasterizer_impl.h:30-77).  Any output pointer may be NULL.  Per-Gaussian fields of culled
 * Gaussians (radii == 0) are written as 0. */
typedef struct gof_state_view {
  float* depths;            /* [P]     GeometryState::depths */
  float* means2D;           /* [P,2]   GeometryState::means2D */
  float* conic_opacity;     /* [P,4]   GeometryState::conic_opacity */
  float* rgb;               /* [P,3]   GeometryState::rgb */
  float* view2gaussian;     /* [P,10]  GeometryState::view2gaussian */
  unsigned char* clamped;   /* [P,3]   GeometryState::clamped */
  uint32_t* tiles_touched;  /* [P]     GeometryState::tiles_touched */
  uint32_t* point_list;     /* [R]     BinningState::point_list (sorted Gaussian ids) */
  uint32_t* ranges;         /* [tiles,2] ImageState::ranges */
  float* accum_alpha;       /* [4,H,W] ImageState::accum_alpha (T, dist1, dist2, raw distortion) */
  uint32_t* n_contrib;      /* [2,H,W] ImageState::n_contrib (last, median) */
  uint32_t* blend_masks;    /* [8, R + 32*tiles] a raw copy of the blend masks the forward leaves for the backward; word
                               layout: GofBinLayout::vmask in csrc/gof_common.cuh.  Only the words of group g of (tile, warp)
                               with 32 g < the largest n_contrib[0] of the warp's 32 pixels are defined.  No reference
                               counterpart; binning buffers of gof_integrate carry no masks. */
} gof_state_view_t;

GOF_API int gof_export_state(int P, int width, int height, int num_rendered,
                     const void* geom_buffer, const void* binning_buffer, const void* image_buffer,
                     const int* radii, const gof_state_view_t* out, void* stream);

/* Marching tetrahedra, utils/tetmesh.py:47-138 (_unbatched_marching_tetrahedra), as CUDA.
 * Two phases because the output sizes are data dependent: `count` classifies the tets, emits and sorts the crossing
 * edges and returns the number of unique crossing edges E and of faces F on the host; `emit` then fills
 * caller-allocated outputs.  `chunk_tets` reproduces the reference's chunked face order (its chunk_size of
 * 32*1024*1024, tetmesh.py:55: the tets are cut into T / chunk_tets + 1 pieces of ceil(T / pieces) rows); pass 0 for "one
 * chunk", or a NEGATIVE value -r to state r rows per chunk directly (used when the tets are sharded over ranks: every shard
 * must cut where the unsharded call cuts).  tets: [T,4] int64 vertex ids < 2^32.  Outputs:
 * interp_v [E,2] int64 (sorted unique crossing edges), faces [F,3] int64; optional gathers of the edge endpoints:
 * edge_pos [E,2,3] from vertices [V,3], edge_sdf [E,2], edge_scales [E,2] from scales [V] (any may be NULL). */
GOF_API int gof_marching_tets_count(int num_verts, const float* sdf, int64_t num_tets, const int64_t* tets, int64_t chunk_tets,
                                    gof_alloc_fn scratch_alloc, void* scratch_user,
                                    int64_t* num_edges_out, int64_t* num_faces_out, void* stream);
GOF_API int gof_marching_tets_emit(int num_verts, const float* sdf, int64_t num_tets, const int64_t* tets, int64_t chunk_tets,
                                   void* scratch, int64_t num_edges, int64_t num_faces,
                                   int64_t* interp_v /* [E,2] */, int64_t* faces /* [F,3] */,
                                   const float* vertices, const float* scales,
                                   float* edge_pos, float* edge_sdf, float* edge_scales, void* stream);

/* TSDF fusion of rendered depth into a sparse voxel-block volume and marching-cubes extraction (extract_mesh_tsdf.py:16-83,
 * which uses Open3D's VoxelBlockGrid; the specification is DESIGN section 4.4).  Stateless: the caller owns the block table
 * (block keys sorted ascending + the pool slot of each block) and the voxel pool [slots][5][B^3] float32 (tsdf, weight,
 * colour r, g, b planes per block, voxel i + B j + B^2 k).  A block key packs block coordinates (bx, by, bz), each in
 * [-2^20, 2^20), as (bz + 2^20) << 42 | (by + 2^20) << 21 | (bx + 2^20); a touched block outside that range fails with
 * GOF_E_INVALID.  Sizes that depend on the data come from a count call, then the caller allocates and calls emit with the
 * count call's scratch. */
typedef struct {
  float voxel_size;       /* s */
  int block_resolution;   /* B, 1..64 */
  float trunc;            /* tau = fl(trunc_voxel_multiplier * s) */
  float depth_max;
} gof_tsdf_params_t;
typedef struct {
  int width, height;
  float fx, fy, cx, cy;
  float extrinsic[12];    /* world -> camera [R | t], row-major 3x4 */
} gof_tsdf_camera_t;
/* Touch: the sorted unique keys of the blocks within tau of the unprojected depth of every 4th pixel in x and y with
 * 0 < depth < depth_max.  depth: [H,W] float32 (0 = none). */
GOF_API int gof_tsdf_touch_count(const gof_tsdf_params_t* params, const gof_tsdf_camera_t* cam, const float* depth,
                                 gof_alloc_fn scratch_alloc, void* scratch_user, int64_t* num_blocks_out, void* stream);
GOF_API int gof_tsdf_touch_emit(const gof_tsdf_params_t* params, const gof_tsdf_camera_t* cam, void* scratch, int64_t num_blocks,
                                int64_t* keys_out, void* stream);
/* Activate: merge a view's sorted unique keys into the table.  count returns how many are new; emit writes the merged table
 * (out_keys / out_slots, num_table + num_new entries, must not alias the inputs; new blocks take slots num_table,
 * num_table + 1, ... in key order, which the caller must have zeroed) and the pool slot of every view block. */
GOF_API int gof_tsdf_activate_count(int64_t num_table, const int64_t* table_keys, int64_t num_view, const int64_t* view_keys,
                                    gof_alloc_fn scratch_alloc, void* scratch_user, int64_t* num_new_out, void* stream);
GOF_API int gof_tsdf_activate_emit(int64_t num_table, const int64_t* table_keys, const int32_t* table_slots, int64_t num_view,
                                   const int64_t* view_keys, void* scratch, int64_t num_new, int64_t* out_keys, int32_t* out_slots,
                                   int32_t* view_slots, void* stream);
/* Integrate one view into the voxels of its blocks (view_keys / view_slots from touch + activate).  depth [H,W],
 * color [3,H,W] float32.  num_updates (optional, device uint64) accumulates the number of voxels updated. */
GOF_API int gof_tsdf_integrate(const gof_tsdf_params_t* params, const gof_tsdf_camera_t* cam, const float* depth, const float* color,
                               int64_t num_view, const int64_t* view_keys, const int32_t* view_slots, float* pool,
                               unsigned long long* num_updates, void* stream);
/* Marching cubes over the whole table (cubes whose 8 corners exist with weight > weight_threshold).  count returns the
 * vertex and face counts; emit writes vertices [V,3], colors [V,3] float32 and faces [F,3] int64 in canonical order. */
GOF_API int gof_tsdf_extract_count(const gof_tsdf_params_t* params, int64_t num_table, const int64_t* table_keys,
                                   const int32_t* table_slots, const float* pool, float weight_threshold, gof_alloc_fn scratch_alloc,
                                   void* scratch_user, int64_t* num_vertices_out, int64_t* num_faces_out, void* stream);
GOF_API int gof_tsdf_extract_emit(const gof_tsdf_params_t* params, int64_t num_table, const int64_t* table_keys,
                                  const int32_t* table_slots, const float* pool, float weight_threshold, void* scratch,
                                  int64_t num_vertices, int64_t num_faces, float* vertices, float* colors, int64_t* faces,
                                  void* stream);

/* Launch accounting and live per-kernel timing (CUDA events on the launching stream; not a profiler).
 * gof_launch_count(): kernels launched by this library so far.  gof_profile_report(): lines of
 * "<kernel> <launches> <total_ms>" accumulated while profiling was enabled. */
GOF_API unsigned long long gof_launch_count(void);
GOF_API void gof_profile_enable(int on);
GOF_API void gof_profile_reset(void);
GOF_API int gof_profile_report(char* buf, int cap);
/* "<kernel> <start_ms> <end_ms>" per bracketed launch since the last reset (origin: the first of them): shows idle
 * gaps between launches.  Returns the bytes needed. */
GOF_API int gof_profile_timeline(char* buf, int cap);
/* GOF_STATS=1 only: copies the 8 counters of the backward blend to `out` (host) and clears them; 0 if disabled.
 * [0] walk iterations, [1..3] pairs evaluated / passed / contributing, [4] (quarter-)warp visits, [5] list entries walked,
 * [6] list entries, [7] double atomics issued into the accumulator rows. */
GOF_API int gof_stats_read(unsigned long long* out);

/* The exchange step of view-parallel training (no reference counterpart: the reference is single-GPU): sum over
 * ranks of a flat f32 buffer over NVLink peer memory.  peers[r] = address, valid in THIS process, of rank r's buffer
 * (CUDA IPC mapping; peers[rank] is the local one); n = floats per buffer (multiple of 4, 16-byte aligned).  This
 * rank reduces its 1/world slice from all buffers (rank order 0..world-1: bit-identical results everywhere) and
 * stores it into all of them.  The caller brackets the call with two cross-rank barriers on `stream`. */
GOF_API int gof_p2p_allreduce_sum_f32(float* const* peers, int world, int rank, size_t n, void* stream);
/* The same with a MAX tail: floats [0, n_sum) are summed over the ranks, [n_sum, n) max-reduced (the densification statistics
 * max_radii2D / xyz_gradient_accum_abs_max travel in the same bucket); n_sum, n multiples of 4. */
GOF_API int gof_p2p_allreduce_f32(float* const* peers, int world, int rank, size_t n_sum, size_t n, void* stream);
/* The same exchange reduced INSIDE the NVSwitch (NVLS): `mc` is the multicast address, valid in this process, of a buffer that
 * every rank has bound to one multicast object at the same offset (e.g. a torch symmetric-memory allocation).  One kernel:
 * multimem.ld_reduce of this rank's 1/world slice (sum, or unsigned max for the non-negative MAX tail) + multimem.st of the
 * result to all ranks.  The caller brackets the call with two cross-rank barriers on `stream`. */
GOF_API int gof_nvls_allreduce_f32(float* mc, int world, int rank, size_t n_sum, size_t n, void* stream);
/* Enables peer access from the current device to `peer_device` (needed once per peer before kernels of this device
 * may dereference that peer's IPC-mapped memory).  Idempotent. */
GOF_API int gof_enable_peer_access(int peer_device);
/* Buffers for that exchange: gof_peer_alloc = cudaMalloc'ed, zero-filled buffer + its 64-byte CUDA IPC handle;
 * gof_peer_open maps a peer's buffer (handle received from that process) for the CURRENT device. */
GOF_API int gof_peer_alloc(size_t bytes, void** ptr, unsigned char* handle64);
GOF_API int gof_peer_open(const unsigned char* handle64, void** ptr);
GOF_API int gof_peer_close(void* ptr);
GOF_API int gof_peer_free(void* ptr);

/* The per-view training loss on the 9-channel render and its gradient (reference: train.py:151-188,
 * utils/loss_utils.py:17-63, utils/depth_utils.py:6-35; SURVEY.md 8(f) rank 1 -- a caller of the rasterizer, not part
 * of its drop-in surface):  loss = (1-l)*L1(rgb,gt) + l*(1-SSIM(rgb,gt)) + l_dn*mean(1 - n_world.n_depth) + l_dist*mean(ch 8).
 * Device pointers: render [9,H,W], gt [3,H,W], terms [5] = (L1, SSIM, normal loss, distortion loss, total),
 * grad [9,H,W] = d total / d render (NULL: values only), scratch of gof_view_loss_scratch_bytes(W,H) bytes.
 * c2w_R9 is a HOST pointer to the row-major camera-to-world rotation ((world_view_transform^T)^-1 [:3,:3]). */
GOF_API size_t gof_view_loss_scratch_bytes(int W, int H);
GOF_API int gof_view_loss(int W, int H, const float* render, const float* gt, const float* c2w_R9, float fx, float fy,
                          float lambda_dssim, float lambda_depth_normal, float lambda_distortion, float* terms,
                          float* grad, void* scratch, void* stream);

/* Parameter prologue / epilogue around the rasterizer (SURVEY.md 8(f) rank 2; callers of the rasterizer, staged):
 * activations with the 3D filter (scene/gaussian_model.py:152-194: scales = sqrt(exp(s)^2 + f^2), rotations = normalize(q),
 * opacity = sigmoid(o) * sqrt(prod exp(s)^2 / prod(exp(s)^2 + f^2)), shs = cat(f_dc, f_rest)), their backward (raw-parameter
 * gradients from the rasterizer's output gradients), and one torch.optim.Adam step (:360, eps 1e-15).  Device pointers, fp32.
 * Rotation arrays (input, output and their gradients) must be 16-byte aligned; otherwise the call returns GOF_E_INVALID. */
GOF_API int gof_activate_params(int P, int M_rest, const float* scaling_raw, const float* rotation_raw, const float* opacity_raw,
                                const float* filter_3D, const float* features_dc, const float* features_rest, float* scales,
                                float* rotations, float* opacities, float* shs, void* stream);
GOF_API int gof_activate_params_backward(int P, int M_rest, const float* scaling_raw, const float* rotation_raw,
                                         const float* opacity_raw, const float* filter_3D, const float* g_scales,
                                         const float* g_rotations, const float* g_opacities, const float* g_shs,
                                         float* d_scaling_raw, float* d_rotation_raw, float* d_opacity_raw,
                                         float* d_features_dc, float* d_features_rest, void* stream);
/* GaussianModel.compute_3D_filter (scene/gaussian_model.py:262-311; staged): per point the smallest camera-space depth over the
 * cameras that see it (depth > 0.2, projection inside the image enlarged by 15 %), unseen points take the largest seen
 * depth; filter = depth / max_focal * sqrt(0.2).  cams [n_cams,16] = R (3x3 as the reference stores it, used as xyz @ R),
 * T, focal_x, focal_y, width, height.  scratch4: 4 device bytes. */
GOF_API int gof_compute_3d_filter(int P, const float* xyz, int n_cams, const float* cams, float max_focal, float* filter_3D,
                                  void* scratch4, void* stream);
/* GaussianModel.get_tetra_points (scene/gaussian_model.py:433-463) before its compaction, and get_frustum_mask (:31-72)
 * (csrc/tetra_points.cu, DESIGN §4.8).  views [n_views,20] float32 = world_view_transform (16, row-major as the reference
 * stores it), focal_x, focal_y, width, height; width and height are read from views[0] only, for every view, as the
 * reference does.  near / far are the reference's Python scalars rounded to float32.
 * gof_tetra_points: xyz, scales (get_scaling_with_3D_filter) [P,3], rotations [P,4] the RAW quaternions (_rotation, 16-byte
 *   aligned) -> out_points [9P,3] (corner k of Gaussian g at 8g + k, sz fastest in the signs (sx, sy, sz); the centres at
 *   8P + g), out_scale [9P] (max of 3 * scales, NaN-propagating), out_mask [9P] bytes 0/1 (inside the frustum of a view).
 * gof_frustum_mask: points [N,3] -> out_mask [N] bytes 0/1.
 * No allocation, no host synchronisation.  GOF_E_INVALID when P < 0, 9P > 2^32 - 1, N < 0, n_views < 1, or the rotations
 * are misaligned. */
GOF_API int gof_tetra_points(int P, const float* xyz, const float* scales, const float* rotations, int n_views, const float* views,
                             float near, float far, float* out_points, float* out_scale, unsigned char* out_mask, void* stream);
GOF_API int gof_frustum_mask(int64_t N, const float* points, int n_views, const float* views, float near, float far,
                             unsigned char* out_mask, void* stream);
/* GaussianModel.densify_and_prune (scene/gaussian_model.py:631-707) in three steps (csrc/densify.cu; SURVEY.md 8(f) rank 4):
 * plan   -- the four keep-flags of every Gaussian (kept original | clone | split child 1 | split child 2) from the accumulated
 *           statistics and their exclusive scans; flags / offsets [4][P] u32, totals [4] u32 on the device, scan_tmp
 *           gof_densify_scratch_bytes(P) device bytes, 8-byte aligned, contents irrelevant;
 * emit   -- per output row (blocks in that order, ascending source index) its source Gaussian and kind, the re-sampled
 *           positions and the raw scalings; totals_host = the four block sizes read back; noise = optional [3][P][3] standard
 *           normal samples, otherwise Philox(seed);
 * gather -- dst[o,:] = src[src_index[o],:] for one parameter / optimizer-state tensor (zero_new: rows of new Gaussians are 0). */
GOF_API size_t gof_densify_scratch_bytes(int P);
GOF_API int gof_densify_plan(int P, const float* accum, const float* accum_abs, const float* denom, const float* scaling_raw,
                             const float* opacity_raw, float max_grad, float abs_threshold, float dense_extent, float min_opacity,
                             float prune_scale, uint32_t* flags, uint32_t* offsets, uint32_t* totals, uint32_t* scan_tmp, void* stream);
GOF_API int gof_densify_emit(int P, const uint32_t* flags, const uint32_t* offsets, const uint32_t* totals_host, const float* xyz,
                             const float* scaling_raw, const float* rotation_raw, const float* noise, unsigned long long seed,
                             int32_t* src_index, unsigned char* kind, float* new_xyz, float* new_scaling_raw, void* stream);
GOF_API int gof_gather_rows_f32(const float* src, int row_floats, const int32_t* src_index, const unsigned char* kind, size_t n_out,
                                int zero_new, float* dst, void* stream);
/* Weight / bias gradient of a 3x3, stride-1, pad-1 convolution with few channels at full image resolution (the tail of the
 * reference's AppearanceNetwork, scene/appearance_network.py:28-29): x [CI,H,W], gy [CO,H,W] -> dW [CO,CI,3,3], db [CO] or NULL,
 * ACCUMULATED into (zero first).  Channel pairs CI->CO: 16->16, 16->3, 8->16. */
GOF_API int gof_conv3x3_wgrad(int CO, int CI, int H, int W, const float* x, const float* gy, float* dW, float* db, void* stream);
GOF_API int gof_adam_step(size_t n, float* param, float* exp_avg, float* exp_avg_sq, const float* grad, double lr, double beta1,
                          double beta2, double eps, int step, void* stream);

/* simple_knn's distCUDA2 (submodules/simple-knn/spatial.cu:15-25, simple_knn.cu:147-183), which GaussianModel.create_from_pcd
 * (scene/gaussian_model.py:327) uses to initialise the scales: for every point i of points [P,3] (device, float32) the mean
 * squared distance to its three nearest neighbours, bit-identical to the reference (DESIGN section 4.5):
 *   d(i,j) = fmaf(dz, dz, fmaf(dx, dx, dy*dy)), dx = x_j - x_i, ...  (updateKBest, simple_knn.cu:132-145: nvcc contracts
 *   d.x*d.x + d.y*d.y + d.z*d.z to FMUL of dy, FFMA of dx, FFMA of dz)
 *   over all j != i BY INDEX (coincident points count, at distance 0); d is accepted only if d < FLT_MAX, so NaN and inf
 *   never enter; b0 <= b1 <= b2 = the three smallest accepted distances, padded with FLT_MAX;
 *   mean_dists[i] = ((b0 + b1) + b2) / 3.0f, IEEE adds and a correctly rounded divide (simple_knn.cu:182).
 * Hence P = 1, 2 and points with a non-finite coordinate give +inf, and such points are nobody's neighbour.  The reference's
 * pruning is exact, so its output does not depend on its search order; this library searches a Morton-ordered 32-ary box
 * tree instead of testing every 1024-point box (simple_knn.cu:168-181).  Scratch: gof_knn_scratch_bytes(P) device bytes,
 * 256-byte aligned, contents irrelevant.  No allocation and no host synchronisation (the call can be captured in a CUDA
 * graph); kernels run on `stream`.  P = 0 launches nothing; P < 0 and P >= 2^30 (the limit of the library's radix sort) fail
 * with GOF_E_INVALID. */
GOF_API size_t gof_knn_scratch_bytes(int P);
GOF_API int gof_knn_mean_dist(int P, const float* points /*[P,3]*/, float* mean_dists /*[P]*/, void* scratch, size_t scratch_bytes,
                              void* stream);

/* The DTU mesh evaluation of dtu_eval/eval.py (DESIGN section 4.6).  Points are device double [n,3]; every step is a
 * sequence of single IEEE double operations in the order written in DESIGN, so oracle/dtu_eval_oracle.py reproduces it bit for
 * bit.  Coordinates must be finite (the Python layer refuses others); any point count of 2^30 or more is refused.
 *
 * Mesh sampling (eval.py:48-71) at `density` = r: out [num_vertices + num_samples, 3] = the vertices in order, then per face
 * with area2 > 0, per row i, per column j, the samples of the face.  Count first, with scratch of
 * gof_mesh_sample_scratch_bytes(num_faces) bytes (256-byte aligned) and a second, row-sized scratch taken through row_alloc;
 * then emit with both.  A face index outside [0, num_vertices) fails with GOF_E_INVALID. */
GOF_API size_t gof_mesh_sample_scratch_bytes(int64_t num_faces);
GOF_API int gof_mesh_sample_count(int64_t num_vertices, const double* vertices, int64_t num_faces, const int64_t* faces /*[F,3]*/,
                                  double density, void* scratch, size_t scratch_bytes, gof_alloc_fn row_alloc, void* row_user,
                                  int64_t* num_samples_out, void* stream);
GOF_API int gof_mesh_sample_emit(int64_t num_vertices, const double* vertices, int64_t num_faces, const int64_t* faces, double density,
                                 const void* scratch, const void* row_scratch, int64_t num_samples, double* out, void* stream);
/* Greedy downsample (eval.py:86-94) in the order perm (a permutation of 0..n-1, else GOF_E_INVALID): position k holds point
 * perm[k]; kept[k] = 1 iff no kept position k' < k has ((dx*dx + dy*dy) + dz*dz) <= radius*radius.  Scratch of
 * gof_ordered_downsample_scratch_bytes(n) bytes; the neighbour list (4 bytes per pair) through pair_alloc.  More than
 * 2^32 - 1 pairs fail with GOF_E_INVALID.  *num_rounds_out: the rounds the parallel decision took. */
GOF_API size_t gof_ordered_downsample_scratch_bytes(int64_t n);
GOF_API int gof_ordered_downsample(int64_t n, const double* points, const uint32_t* perm, double radius, uint8_t* kept,
                                   int64_t* num_rounds_out, int64_t* num_pairs_out, void* scratch, size_t scratch_bytes,
                                   gof_alloc_fn pair_alloc, void* pair_user, void* stream);
/* out[i] = min over the n_ref reference points of ((dx*dx + dy*dy) + dz*dz) to query i, or its sqrt if take_sqrt (eval.py:119-133).
 * n_ref = 0 with queries fails with GOF_E_INVALID.  Scratch of gof_nn_dist_scratch_bytes(n_ref, n_query) bytes; no allocation
 * and no host synchronisation. */
GOF_API size_t gof_nn_dist_scratch_bytes(int64_t n_ref, int64_t n_query);
GOF_API int gof_nn_dist(int64_t n_ref, const double* ref, int64_t n_query, const double* query, double* out, int take_sqrt,
                        void* scratch, size_t scratch_bytes, void* stream);

/* The same 1-NN search split in two, for repeated queries against one cloud (the Tanks and Temples ICP, DESIGN section 4.7):
 * gof_nn_tree_build keeps the tree over ref in tree_scratch (gof_nn_tree_scratch_bytes(n_ref) bytes, kept intact between
 * queries); gof_nn_query writes, for every query, out_index = the reference point with the smallest ((dx*dx + dy*dy) + dz*dz)
 * strictly below r2, the lowest index among equals, or -1, and out_d2 = that value (INFINITY for -1).  Query scratch of
 * gof_nn_query_scratch_bytes(n_query) bytes.  tree_scratch_bytes is the size of tree_scratch, checked against n_ref.
 * reuse_order != 0 skips the Morton sort of the queries and reuses the order that an earlier call with this query scratch and
 * the same n_query stamped into it; a scratch without such a stamp (fresh, or sorted for another count) is searched in input
 * order instead.  Results never depend on the order.  No allocation and no host synchronisation. */
GOF_API size_t gof_nn_tree_scratch_bytes(int64_t n_ref);
GOF_API int gof_nn_tree_build(int64_t n_ref, const double* ref, void* tree_scratch, size_t scratch_bytes, void* stream);
GOF_API size_t gof_nn_query_scratch_bytes(int64_t n_query);
GOF_API int gof_nn_query(int64_t n_ref, void* tree_scratch, size_t tree_scratch_bytes, int64_t n_query, const double* query, double r2,
                         int reuse_order, int32_t* out_index, double* out_d2, void* query_scratch, size_t scratch_bytes, void* stream);

/* The Tanks and Temples evaluation of eval_tnt/run.py (DESIGN section 4.7).  Points are device double [n,3], finite; any count
 * of 2^30 or more is refused with GOF_E_INVALID.  A transformation is a host double[16], row-major; a point maps to
 * (((m00*x + m01*y) + m02*z) + m03) / w per row, w the fourth row's value.
 *
 * Polygon-volume crop (SelectionPolygonVolume.crop_point_cloud), optionally after `transform` (NULL: none): axis = the
 * orthogonal axis (0, 1, 2), polygon_uv = host [num_vertices, 2] of the polygon's two other coordinates in ascending axis order,
 * 3 <= num_vertices <= 3072.  out [*num_out, 3] = the kept points in input order (capacity n), out_index (or NULL) their
 * input indices.  Scratch of gof_crop_scratch_bytes(n) bytes; reads back the kept count. */
GOF_API size_t gof_crop_scratch_bytes(int64_t n);
GOF_API int gof_crop_polygon(int64_t n, const double* points, const double* transform, int axis, double axis_min, double axis_max,
                             int num_vertices, const double* polygon_uv, double* out, uint32_t* out_index, int64_t* num_out,
                             void* scratch, size_t scratch_bytes, void* stream);
/* Voxel down-sample (PointCloud.voxel_down_sample): out [*num_out, 3] (capacity n) = per occupied voxel the mean of its points,
 * summed in input order, in ascending (x, y, z) voxel index order.  voxel * INT_MAX below the extent of the box grown by
 * voxel / 2 fails with GOF_E_INVALID ("voxel_size is too small"), and so does a point with a non-finite coordinate.  Scratch of gof_voxel_down_sample_scratch_bytes(n) bytes. */
GOF_API size_t gof_voxel_down_sample_scratch_bytes(int64_t n);
GOF_API int gof_voxel_down_sample(int64_t n, const double* points, double voxel, double* out, int64_t* num_out, void* scratch,
                                  size_t scratch_bytes, void* stream);
/* Point-to-point ICP moments over the pairs (i, index[i]), index[i] >= 0, with d2[i] their squared distances.  Host
 * moments[18] = count, sum d2, mean src[3], mean tgt[3] (sum * (1 / count)), sum (t - mt)(s - ms)^T [3][3] row-major by target
 * axis, sum |s - ms|^2.  Fixed summation order, independent of the launch: two runs are bit-identical.  Scratch of
 * gof_icp_moments_scratch_bytes(n) bytes; one read-back. */
GOF_API size_t gof_icp_moments_scratch_bytes(int64_t n);
GOF_API int gof_icp_moments(int64_t n, const double* src, const double* tgt, const int32_t* index, const double* d2, double* moments,
                            void* scratch, size_t scratch_bytes, void* stream);
/* points <- transform(points), in place. */
GOF_API int gof_transform_points(int64_t n, double* points, const double* transform, void* stream);

GOF_API const char* gof_last_error(void);
GOF_API int gof_version(void);

#ifdef __cplusplus
}
#endif
#endif /* GOF_RASTERIZER_H_INCLUDED */
