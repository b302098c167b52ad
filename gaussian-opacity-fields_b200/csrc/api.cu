// api.cu -- the extern "C" boundary (include/gof_rasterizer.h): host orchestration of the kernels,
// replacing CudaRasterizer::Rasterizer::{forward,backward,markVisible} (rasterizer_impl.cu:174-526).
#include <stdarg.h>
#include <stdlib.h>

#include "gof_common.cuh"
#include "gof_math.cuh"

// ---- launch counter + optional per-kernel event timing ----------------------------------------------------
#include <map>
#include <mutex>
#include <string>
#include <vector>
namespace {
struct ProfEntry { const char* name; cudaEvent_t a, b; };
std::mutex g_prof_mu;
bool g_prof_on = false;
unsigned long long g_launches = 0;
std::vector<ProfEntry> g_prof_pending;
std::vector<cudaEvent_t> g_prof_pool;
std::map<std::string, std::pair<unsigned long long, double>> g_prof_acc;   // name -> (count, ms)
cudaEvent_t g_prof_base = nullptr;      // first bracket's start: origin of the timeline
std::string g_prof_timeline;            // "name start_ms end_ms\n" per launch since the last reset
thread_local ProfEntry g_prof_cur = {nullptr, nullptr, nullptr};
cudaEvent_t prof_get_event() {
  if (!g_prof_pool.empty()) { cudaEvent_t e = g_prof_pool.back(); g_prof_pool.pop_back(); return e; }
  cudaEvent_t e; cudaEventCreate(&e); return e;
}
void prof_drain_locked() {
  for (auto& e : g_prof_pending) {
    cudaEventSynchronize(e.b);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e.a, e.b);
    auto& acc = g_prof_acc[e.name];
    acc.first += 1; acc.second += ms;
    if (g_prof_base && g_prof_timeline.size() < (1u << 22)) {
      float t0 = 0.f;
      cudaEventElapsedTime(&t0, g_prof_base, e.a);
      char line[160];
      snprintf(line, sizeof(line), "%s %.4f %.4f\n", e.name, t0, t0 + ms);
      g_prof_timeline += line;
    }
    g_prof_pool.push_back(e.a); g_prof_pool.push_back(e.b);
  }
  g_prof_pending.clear();
}
}  // namespace

void gof_prof_begin(const char* name, cudaStream_t st) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_launches++;
  if (!g_prof_on) return;
  g_prof_cur.name = name; g_prof_cur.a = prof_get_event(); g_prof_cur.b = prof_get_event();
  if (!g_prof_base) { cudaEventCreate(&g_prof_base); cudaEventRecord(g_prof_base, st); }
  cudaEventRecord(g_prof_cur.a, st);
}
void gof_prof_end(cudaStream_t st) {
  if (!g_prof_on || !g_prof_cur.name) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  cudaEventRecord(g_prof_cur.b, st);
  g_prof_pending.push_back(g_prof_cur);
  g_prof_cur.name = nullptr;
  if (g_prof_pending.size() > 4096) prof_drain_locked();
}
extern "C" unsigned long long gof_launch_count(void) { return g_launches; }
extern "C" void gof_profile_enable(int on) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (!on) prof_drain_locked();
  g_prof_on = on != 0;
}
extern "C" void gof_profile_reset(void) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  prof_drain_locked();
  g_prof_acc.clear();
  g_prof_timeline.clear();
  if (g_prof_base) { cudaEventDestroy(g_prof_base); g_prof_base = nullptr; }
}
// writes "name count total_ms\n" lines; returns the number of bytes needed (excluding the terminator)
extern "C" int gof_profile_report(char* buf, int cap) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  prof_drain_locked();
  std::string out;
  for (auto& kv : g_prof_acc) {
    char line[256];
    snprintf(line, sizeof(line), "%s %llu %.6f\n", kv.first.c_str(), kv.second.first, kv.second.second);
    out += line;
  }
  if (buf && cap > 0) { strncpy(buf, out.c_str(), (size_t)cap - 1); buf[cap - 1] = 0; }
  return (int)out.size();
}

// writes "name start_ms end_ms\n" per bracketed launch (origin: the first launch after the last reset)
extern "C" int gof_profile_timeline(char* buf, int cap) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  prof_drain_locked();
  if (buf && cap > 0) { strncpy(buf, g_prof_timeline.c_str(), (size_t)cap - 1); buf[cap - 1] = 0; }
  return (int)g_prof_timeline.size();
}

void* gof_pinned_slot() {
  static thread_local void* slot = nullptr;
  static thread_local bool tried = false;
  if (!tried) {
    tried = true;
    if (cudaHostAlloc(&slot, 64, cudaHostAllocDefault) != cudaSuccess) { slot = nullptr; (void)cudaGetLastError(); }
  }
  return slot;
}
int gof_read_back(void* dst, const void* src_dev, size_t bytes, cudaStream_t st) {
  void* pin = bytes <= 64 ? gof_pinned_slot() : nullptr;
  GOF_CUDA_OK(cudaMemcpyAsync(pin ? pin : dst, src_dev, bytes, cudaMemcpyDeviceToHost, st));
  GOF_CUDA_OK(cudaStreamSynchronize(st));
  if (pin) memcpy(dst, pin, bytes);
  return GOF_OK;
}

// The instance count (num_rendered) sizes the binning buffer, so the host needs it in the middle of the forward
// (rasterizer_impl.cu:334-340 does a blocking cudaMemcpy there, idling the GPU for the round trip).  Here the preprocess kernel
// itself sums tiles_touched; the 4-byte copy runs on a side stream as soon as that kernel has finished, while the launching
// stream carries on with the depth sort, and the host waits for the copy only: by the time it has sized the buffer and queued
// the emit kernel the GPU is still busy sorting.
namespace {
struct SideCopy { cudaStream_t st = nullptr; cudaEvent_t after_kernel = nullptr, copied = nullptr; uint32_t* pin = nullptr; bool ok = false, tried = false; };
SideCopy* side_copy_for_current_device() {
  static thread_local SideCopy table[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  SideCopy& s = table[dev];
  if (!s.tried) {
    s.tried = true;
    s.ok = cudaStreamCreateWithFlags(&s.st, cudaStreamNonBlocking) == cudaSuccess &&
           cudaEventCreateWithFlags(&s.after_kernel, cudaEventDisableTiming) == cudaSuccess &&
           cudaEventCreateWithFlags(&s.copied, cudaEventDisableTiming) == cudaSuccess &&
           cudaHostAlloc((void**)&s.pin, 64, cudaHostAllocDefault) == cudaSuccess;
    if (!s.ok) (void)cudaGetLastError();
  }
  return s.ok ? &s : nullptr;
}
}  // namespace

// Queues "copy *src_dev (u32) to the host once everything queued on `st` so far has finished" on the side stream.
// Returns nullptr when side-stream resources are unavailable (the caller then reads back synchronously).
static SideCopy* begin_async_read_u32(const void* src_dev, cudaStream_t st) {
  SideCopy* sc = side_copy_for_current_device();
  if (!sc) return nullptr;
  if (cudaEventRecord(sc->after_kernel, st) != cudaSuccess || cudaStreamWaitEvent(sc->st, sc->after_kernel, 0) != cudaSuccess ||
      cudaMemcpyAsync(sc->pin, src_dev, 4, cudaMemcpyDeviceToHost, sc->st) != cudaSuccess ||
      cudaEventRecord(sc->copied, sc->st) != cudaSuccess) {
    (void)cudaGetLastError();
    return nullptr;
  }
  return sc;
}
static int finish_async_read_u32(SideCopy* sc, uint32_t* out) {
  GOF_CUDA_OK(cudaEventSynchronize(sc->copied));
  *out = *sc->pin;
  return GOF_OK;
}

// ---- per-device launch state ---------------------------------------------------------------------------------
// Function attributes and SM counts belong to one device; a process may drive several, from several host threads
// (autograd runs the backward on its own thread).  One mutex guards all of it.
static std::mutex g_dev_mu;
static std::map<std::pair<int, const void*>, int> g_dev_once;   // (device, key) -> the value its setup left

int gof_device_once(const void* key, int (*setup)(int dev, int* value), int* value) {
  int dev = 0;
  GOF_CUDA_OK(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lk(g_dev_mu);
  auto it = g_dev_once.find({dev, key});
  if (it == g_dev_once.end()) {
    int v = 0;
    const int rc = setup(dev, &v);
    if (rc != GOF_OK) return rc;
    it = g_dev_once.emplace(std::make_pair(dev, key), v).first;
  }
  if (value) *value = it->second;
  return GOF_OK;
}

int gof_sm_count() {
  int n = 132;
  gof_device_once((const void*)&gof_sm_count, [](int dev, int* v) -> int {
    if (cudaDeviceGetAttribute(v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || *v <= 0) { (void)cudaGetLastError(); *v = 132; }
    return GOF_OK;
  }, &n);
  return n;
}

static thread_local char g_err[1024] = "";

void gof_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

extern "C" const char* gof_last_error(void) { return g_err; }
extern "C" int gof_version(void) { return 104; }

static int validate_scene(const gof_scene_t* s) {
  if (!s) { gof_set_error("scene is NULL"); return GOF_E_INVALID; }
  if (s->P < 0 || s->width <= 0 || s->height <= 0) { gof_set_error("bad sizes P=%d W=%d H=%d", s->P, s->width, s->height); return GOF_E_INVALID; }
  if (s->P == 0) return GOF_OK;
  if (!s->means3D || !s->opacities || !s->viewmatrix || !s->projmatrix || !s->background) {
    gof_set_error("means3D/opacities/viewmatrix/projmatrix/background must be non-NULL");
    return GOF_E_INVALID;
  }
  // diff_gaussian_rasterization/__init__.py:203-207
  if ((s->shs == nullptr) == (s->colors_precomp == nullptr)) {
    gof_set_error("Please provide excatly one of either SHs or precomputed colors!");
    return GOF_E_INVALID;
  }
  if (s->shs) {
    if (!s->cam_pos) { gof_set_error("cam_pos required with SHs"); return GOF_E_INVALID; }
    if (s->D < 0 || s->D > 3 || (s->D + 1) * (s->D + 1) > s->M) {
      gof_set_error("SH degree %d needs %d coefficients, got M=%d", s->D, (s->D + 1) * (s->D + 1), s->M);
      return GOF_E_INVALID;
    }
    if (s->M > 16) { gof_set_error("M=%d SH coefficients unsupported (max 16)", s->M); return GOF_E_INVALID; }
  }
  const bool has_sr = s->scales && s->rotations;
  if (!has_sr && !s->cov3D_precomp) {
    gof_set_error("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!");
    return GOF_E_INVALID;
  }
  // the reference dereferences scales/rotations unconditionally for view2gaussian (forward.cu:334-335,399);
  // without them a precomputed view2gaussian is the only defined input
  if (!has_sr && !s->view2gaussian_precomp) {
    gof_set_error("scales/rotations absent: view2gaussian_precomp is required");
    return GOF_E_INVALID;
  }
  if (s->width > 16 * 65535 || s->height > 16 * 65535) { gof_set_error("image too large"); return GOF_E_INVALID; }
  return GOF_OK;
}

// The Gaussian side of the forward and of the opacity-field query: geometry and image scratch, preprocess, depth sort, the
// instance count (it sizes the binning buffer, rasterizer_impl.cu:334-340, and is read while the depth sort runs) and the tile
// binning.  box_margin (gof_cull_bbox) is 0 for the forward and 0.5 for the query, whose corner rays reach half a pixel beyond
// the centre ray; only the forward's binning buffer carries the blend masks its backward reads.
struct GaussianSide {
  GofGeomLayout GL;
  GofImageLayout IL;
  GofBinLayout BL;
  char *geom, *img, *bin;
  uint32_t R;
};
static int gaussian_side(const gof_scene_t* s, const GofView& v, gof_alloc_fn geom_alloc, void* geom_user, gof_alloc_fn binning_alloc,
                         void* binning_user, gof_alloc_fn image_alloc, void* image_user, int* radii, float box_margin, bool with_masks,
                         int* num_rendered, cudaStream_t st, GaussianSide& g) {
  int rc;
  g.GL = gof_geom_layout((size_t)s->P);
  g.geom = (char*)geom_alloc(geom_user, g.GL.bytes);
  g.IL = gof_image_layout(s->width, s->height);
  g.img = (char*)image_alloc(image_user, g.IL.bytes);
  if (!g.geom || !g.img) { gof_set_error("scratch allocator returned NULL"); return GOF_E_ALLOC; }

  if ((rc = gof_launch_preprocess(s, v, g.geom, g.GL, radii, box_margin, st)) != GOF_OK) return rc;
  SideCopy* sc = s->debug ? nullptr : begin_async_read_u32(g.geom + g.GL.total, st);
  if ((rc = gof_depth_sort(s->P, g.geom, g.GL, s->debug != 0, st)) != GOF_OK) return rc;
  rc = sc ? finish_async_read_u32(sc, &g.R) : gof_read_back(&g.R, g.geom + g.GL.total, sizeof(uint32_t), st);
  if (rc != GOF_OK) return rc;
  *num_rendered = (int)g.R;

  g.BL = gof_bin_layout((size_t)g.R, s->width, s->height, with_masks);
  g.bin = (char*)binning_alloc(binning_user, g.BL.bytes);
  if (!g.bin && g.BL.bytes) { gof_set_error("binning allocator returned NULL"); return GOF_E_ALLOC; }
  return gof_bin_tiles(s->P, (size_t)g.R, v, g.geom, g.GL, g.bin, g.BL, g.img, g.IL, s->debug != 0, st);
}

// The point side of the query, against the Gaussian side of gaussian_side or of a gof_integrate_prepare cache (img: the
// image scratch, NULL if its allocator failed).
static int point_side(const gof_scene_t* s, const GofView& v, int PN, const float* points3D, const GofSplat* splat,
                      const uint32_t* point_list, const uint2* ranges, char* img, gof_alloc_fn point_alloc, void* point_user,
                      gof_alloc_fn point_binning_alloc, void* point_binning_user, const gof_integrate_out_t& out, cudaStream_t st) {
  char* pts = (char*)point_alloc(point_user, gof_point_layout((size_t)PN).bytes);
  char* pbin = (char*)point_binning_alloc(point_binning_user, gof_point_bin_layout((size_t)PN, v.tiles, gof_sm_count()).bytes);
  if (!img || !pts || !pbin) { gof_set_error("scratch allocator returned NULL"); return GOF_E_ALLOC; }
  return gof_launch_integrate(s, v, PN, points3D, splat, point_list, ranges, img, pts, pbin, out, st);
}

// The checks of both queries' outputs (gof_integrate_out_t) and allocators, in one order: out given, no field of the other mode,
// the view, the allocators.  Then, with something to do, each query checks its buffers and integrate_outputs_given.
static int check_integrate_out(const char* who, const gof_integrate_out_t* out, bool grad_min_offered, bool allocators) {
  const char* err = nullptr;
  const bool min = out && (out->alpha_min || out->argmin);
  if (!out) err = "out is NULL";
  else if (min && (out->out_color || out->out_alpha_integrated || out->out_color_integrated))
    err = "out_color / out_alpha_integrated / out_color_integrated must be NULL with alpha_min / argmin";
  else if (!min && (out->color_min || out->grad_min)) err = "color_min / grad_min need alpha_min and argmin";
  else if (out->grad_min && !grad_min_offered) err = "grad_min is an output of gof_integrate_cached only";
  else if (min && (out->view < 0 || out->view >= (1 << 30))) err = "view outside [0, 2^30)";   // 2^30 is argmin's "no view" value
  else if (!allocators) err = "allocators must be non-NULL";
  if (err) gof_set_error("%s: %s", who, err);
  return err ? GOF_E_INVALID : GOF_OK;
}
static bool integrate_outputs_given(const gof_integrate_out_t& o) {
  return o.alpha_min || o.argmin ? o.alpha_min && o.argmin : o.out_color && o.out_alpha_integrated && o.out_color_integrated;
}

extern "C" int gof_rasterize_forward(const gof_scene_t* s, gof_alloc_fn geom_alloc, void* geom_user,
                                     gof_alloc_fn binning_alloc, void* binning_user, gof_alloc_fn image_alloc,
                                     void* image_user, float* out_color, int* radii, int* num_rendered,
                                     void* stream) {
  int rc = validate_scene(s);
  if (rc != GOF_OK) return rc;
  if (!geom_alloc || !binning_alloc || !image_alloc || !num_rendered) {
    gof_set_error("allocators / num_rendered must be non-NULL");
    return GOF_E_INVALID;
  }
  *num_rendered = 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (s->P == 0) return GOF_OK;   // rasterize_points.cu:85
  if (!out_color || !radii) { gof_set_error("out_color / radii must be non-NULL"); return GOF_E_INVALID; }
  const GofView v = gof_make_view(s);
  GaussianSide g;
  if ((rc = gaussian_side(s, v, geom_alloc, geom_user, binning_alloc, binning_user, image_alloc, image_user, radii, 0.0f, true,
                          num_rendered, st, g)) != GOF_OK)
    return rc;
  return gof_launch_render_forward(s, v, g.geom, g.GL, g.bin, g.BL, g.img, g.IL, out_color, st);
}

// Where the focal-length scratch keeps the camera pass's rows (first) and the ray pass's per-pixel values (256-byte aligned after them)
static size_t intrinsics_camera_bytes(int P) { return (gof_camera_grad_scratch_bytes(P) + 255) / 256 * 256; }

extern "C" size_t gof_rasterize_backward_scratch_bytes(int P, int width, int height, int camera, int intrinsics) {
  if (P <= 0) return 0;
  if (intrinsics) return width > 0 && height > 0 ? intrinsics_camera_bytes(P) + gof_ray_grad_scratch_bytes(width, height) : 0;
  return camera ? gof_camera_grad_scratch_bytes(P) : 0;
}

// The checks of the Gaussian gradients that both backwards hand to k_preprocess_backward, which stores dL_drot as float4, and
// dL_dsh too at M == 16 and degree 3.
static int check_gaussian_grads(const char* who, const gof_scene_t* s, const gof_backward_out_t& o) {
  const char* err = nullptr;
  if (s->P > 0 && s->scales && s->rotations && (!o.dL_dscale || !o.dL_drot)) err = "dL_dscale / dL_drot required";
  else if (reinterpret_cast<uintptr_t>(o.dL_drot) & 15) err = "dL_drot must be 16-byte aligned";
  else if (s->shs && s->M == 16 && s->D == 3 && (reinterpret_cast<uintptr_t>(o.dL_dsh) & 15)) err = "dL_dsh must be 16-byte aligned";
  if (err) gof_set_error("%s: %s", who, err);
  return err ? GOF_E_INVALID : GOF_OK;
}

extern "C" int gof_rasterize_backward_ex(const gof_scene_t* s, int num_rendered, const int* radii, void* geom_buffer,
                                         const void* binning_buffer, const void* image_buffer, const float* dL_dpix,
                                         const gof_backward_out_t* out, void* stream) {
  if (!out) { gof_set_error("backward: out is NULL"); return GOF_E_INVALID; }
  int rc = validate_scene(s);
  if (rc != GOF_OK) return rc;
  const gof_backward_out_t& o = *out;
  const bool camera = o.dL_dviewmatrix != nullptr;
  const bool intrinsics = o.dL_dtan_fov != nullptr;
  if (camera != (o.dL_dcampos != nullptr)) {
    gof_set_error("backward: dL_dviewmatrix and dL_dcampos come together");
    return GOF_E_INVALID;
  }
  if ((o.sh_rgb || o.sh_hdr) && (camera || intrinsics)) {
    gof_set_error("backward: sh_rgb / sh_hdr do not combine with the camera or focal-length gradient");
    return GOF_E_INVALID;
  }
  const size_t need = gof_rasterize_backward_scratch_bytes(s->P, s->width, s->height, camera, intrinsics);
  if ((camera || intrinsics) && o.scratch_bytes < need) {
    gof_set_error("backward: %s scratch of %zu bytes, %zu needed (gof_rasterize_backward_scratch_bytes)",
                  intrinsics ? "intrinsics" : "camera", o.scratch_bytes, need);
    return GOF_E_INVALID;
  }
  if ((camera || intrinsics) && s->P > 0 && !o.scratch) {
    gof_set_error("backward: %s scratch is NULL", intrinsics ? "intrinsics" : "camera");
    return GOF_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (s->P == 0) {   // rasterize_points.cu:172; the camera and focal-length gradients of no Gaussians are zero
    if (camera) {
      GOF_CUDA_OK(cudaMemsetAsync(o.dL_dviewmatrix, 0, 16 * sizeof(float), st));
      GOF_CUDA_OK(cudaMemsetAsync(o.dL_dcampos, 0, 3 * sizeof(float), st));
    }
    if (intrinsics) GOF_CUDA_OK(cudaMemsetAsync(o.dL_dtan_fov, 0, 2 * sizeof(float), st));
    return GOF_OK;
  }
  if (!radii || !geom_buffer || !image_buffer || !dL_dpix || !o.dL_dmean2D || !o.dL_dopacity || !o.dL_dcolor ||
      !o.dL_dmean3D || !o.dL_dview2gaussian || (num_rendered > 0 && !binning_buffer)) {
    gof_set_error("backward: NULL argument");
    return GOF_E_INVALID;
  }
  if (s->shs && !o.dL_dsh && !(o.sh_rgb && o.sh_hdr)) {
    gof_set_error("backward: dL_dsh (or sh_rgb + sh_hdr) required with SHs");
    return GOF_E_INVALID;
  }
  if ((o.sh_rgb != nullptr) != (o.sh_hdr != nullptr) || (o.sh_rgb && !s->shs)) {
    gof_set_error("backward: sh_rgb and sh_hdr come together and need SHs");
    return GOF_E_INVALID;
  }
  if ((rc = check_gaussian_grads("backward", s, o)) != GOF_OK) return rc;
  const GofView v = gof_make_view(s);
  const GofGeomLayout GL = gof_geom_layout((size_t)s->P);
  const GofImageLayout IL = gof_image_layout(s->width, s->height);
  const GofBinLayout BL = gof_bin_layout((size_t)num_rendered, s->width, s->height);
  // The geometry buffer is the caller's scratch for this view: its last section holds the blend kernel's 64-byte
  // per-Gaussian accumulator rows, zeroed and filled by every backward call (the forward state in it is only read).
  char* geom = static_cast<char*>(geom_buffer);
  double* rays = intrinsics ? reinterpret_cast<double*>(static_cast<char*>(o.scratch) + intrinsics_camera_bytes(s->P)) : nullptr;
  if ((rc = gof_launch_render_backward(s, v, geom, GL, (const char*)binning_buffer, BL, (const char*)image_buffer, IL, dL_dpix,
                                       rays, o.dL_dtan_fov, st)) != GOF_OK)
    return rc;
  return gof_launch_preprocess_backward(s, geom, GL, radii, o, st);
}

extern "C" int gof_rasterize_backward(const gof_scene_t* s, int num_rendered, const int* radii, void* geom_buffer,
                                      const void* binning_buffer, const void* image_buffer, const float* dL_dpix, float* dL_dmean2D,
                                      float* dL_dconic, float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D,
                                      float* dL_dsh, float* dL_dscale, float* dL_drot, float* dL_dview2gaussian, void* stream) {
  (void)dL_dconic;
  gof_backward_out_t o{};
  o.dL_dmean2D = dL_dmean2D;
  o.dL_dopacity = dL_dopacity;
  o.dL_dcolor = dL_dcolor;
  o.dL_dmean3D = dL_dmean3D;
  o.dL_dcov3D = dL_dcov3D;
  o.dL_dsh = dL_dsh;
  o.dL_dscale = dL_dscale;
  o.dL_drot = dL_drot;
  o.dL_dview2gaussian = dL_dview2gaussian;
  return gof_rasterize_backward_ex(s, num_rendered, radii, geom_buffer, binning_buffer, image_buffer, dL_dpix, &o, stream);
}

extern "C" int gof_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                                unsigned char* present, void* stream) {
  (void)projmatrix;
  if (P < 0) { gof_set_error("P < 0"); return GOF_E_INVALID; }
  if (P == 0) return GOF_OK;
  if (!means3D || !viewmatrix || !present) { gof_set_error("mark_visible: NULL argument"); return GOF_E_INVALID; }
  return gof_launch_mark_visible(P, means3D, viewmatrix, present, (cudaStream_t)stream);
}

// ---- parity-test export ------------------------------------------------------------------------------
namespace {
__global__ void k_export_geom(int P, const int* __restrict__ radii, const GofSplat* __restrict__ splat,
                              const GofSplatBwd* __restrict__ sb, const unsigned char* __restrict__ clamped,
                              const uint32_t* __restrict__ tiles, const float* __restrict__ depth, gof_state_view_t o) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const bool vis = radii[i] > 0;
  GofSplat s;
  GofSplatBwd b;
  if (vis) { s = splat[i]; b = sb[i]; }
  if (o.depths) o.depths[i] = vis ? depth[i] : 0.f;
  if (o.means2D) { o.means2D[2 * i] = vis ? b.mx : 0.f; o.means2D[2 * i + 1] = vis ? b.my : 0.f; }
  if (o.conic_opacity) {
    o.conic_opacity[4 * i + 0] = vis ? b.cx : 0.f; o.conic_opacity[4 * i + 1] = vis ? b.cy : 0.f;
    o.conic_opacity[4 * i + 2] = vis ? b.cz : 0.f; o.conic_opacity[4 * i + 3] = vis ? s.opacity : 0.f;
  }
  if (o.rgb) for (int k = 0; k < 3; ++k) o.rgb[3 * i + k] = vis ? s.rgb[k] : 0.f;
  if (o.view2gaussian) for (int k = 0; k < 10; ++k) o.view2gaussian[10 * i + k] = vis ? s.v2g[k] : 0.f;
  if (o.clamped) for (int k = 0; k < 3; ++k) o.clamped[3 * i + k] = vis ? ((clamped[i] >> k) & 1) : 0;
  if (o.tiles_touched) o.tiles_touched[i] = tiles[i];
}

__global__ void k_export_image(int W, int H, int grid_x, size_t plane, const float* __restrict__ accum,
                               const uint32_t* __restrict__ nc, gof_state_view_t o) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  const int tile = (y / 16) * grid_x + (x / 16);
  const size_t slot = (size_t)tile * 256 + gof_pixel_slot(x & 15, y & 15);
  const size_t HW = (size_t)W * H, pid = (size_t)y * W + x;
  if (o.accum_alpha) for (int k = 0; k < 4; ++k) o.accum_alpha[k * HW + pid] = accum[k * plane + slot];
  if (o.n_contrib) for (int k = 0; k < 2; ++k) o.n_contrib[k * HW + pid] = nc[k * plane + slot];
}
}  // namespace

extern "C" int gof_export_state(int P, int width, int height, int num_rendered, const void* geom_buffer,
                                const void* binning_buffer, const void* image_buffer, const int* radii,
                                const gof_state_view_t* out, void* stream) {
  if (!out || P <= 0) { gof_set_error("export_state: bad arguments"); return GOF_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const char* geom = (const char*)geom_buffer;
  const char* img = (const char*)image_buffer;
  const char* bin = (const char*)binning_buffer;
  const GofGeomLayout GL = gof_geom_layout((size_t)P);
  const GofImageLayout IL = gof_image_layout(width, height);
  const GofBinLayout BL = gof_bin_layout((size_t)num_rendered, width, height);
  const int grid_x = (width + 15) / 16, grid_y = (height + 15) / 16;
  k_export_geom<<<(P + 255) / 256, 256, 0, st>>>(P, radii, (const GofSplat*)(geom + GL.splat),
                                                 (const GofSplatBwd*)(geom + GL.splat_bwd),
                                                 (const unsigned char*)(geom + GL.clamped),
                                                 (const uint32_t*)(geom + GL.tiles), (const float*)(geom + GL.depth), *out);
  GOF_LAUNCH_CHECK(true, st);
  if (out->point_list && num_rendered > 0)
    GOF_CUDA_OK(cudaMemcpyAsync(out->point_list, bin + BL.point_list, (size_t)num_rendered * 4,
                                cudaMemcpyDeviceToDevice, st));
  if (out->ranges)
    GOF_CUDA_OK(cudaMemcpyAsync(out->ranges, img + IL.ranges, (size_t)grid_x * grid_y * 8, cudaMemcpyDeviceToDevice, st));
  if (out->blend_masks && num_rendered > 0)
    GOF_CUDA_OK(cudaMemcpyAsync(out->blend_masks, bin + BL.vmask, BL.vmask_stride * 8 * 4, cudaMemcpyDeviceToDevice, st));
  if (out->accum_alpha || out->n_contrib) {
    dim3 b(16, 16), g((width + 15) / 16, (height + 15) / 16);
    k_export_image<<<g, b, 0, st>>>(width, height, grid_x, (size_t)grid_x * grid_y * 256,
                                    (const float*)(img + IL.accum), (const uint32_t*)(img + IL.ncontrib), *out);
    GOF_LAUNCH_CHECK(true, st);
  }
  return GOF_OK;
}

// Rasterizer::integrate (rasterizer_impl.cu:530-792): Gaussian side exactly as the forward (preprocess, depth sort,
// binning), then the point side and the query kernel.
extern "C" int gof_integrate(const gof_scene_t* s, int PN, const float* points3D, gof_alloc_fn geom_alloc, void* geom_user,
                             gof_alloc_fn binning_alloc, void* binning_user, gof_alloc_fn image_alloc, void* image_user,
                             gof_alloc_fn point_alloc, void* point_user, gof_alloc_fn point_binning_alloc,
                             void* point_binning_user, int* radii, int* num_rendered, const gof_integrate_out_t* out, void* stream) {
  int rc = validate_scene(s);
  if (rc != GOF_OK) return rc;
  if ((rc = check_integrate_out("integrate", out, false, geom_alloc && binning_alloc && image_alloc && point_alloc &&
                                point_binning_alloc)) != GOF_OK)
    return rc;
  if (!num_rendered) { gof_set_error("integrate: num_rendered is NULL"); return GOF_E_INVALID; }
  *num_rendered = 0;
  if (s->P == 0 || PN <= 0) return GOF_OK;   // rasterize_points.cu:305
  if (!points3D || !radii || !integrate_outputs_given(*out)) {
    gof_set_error("integrate: NULL argument");
    return GOF_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const GofView v = gof_make_view(s);
  GaussianSide g;
  if ((rc = gaussian_side(s, v, geom_alloc, geom_user, binning_alloc, binning_user, image_alloc, image_user, radii, 0.5f, false,
                          num_rendered, st, g)) != GOF_OK)
    return rc;
  return point_side(s, v, PN, points3D, reinterpret_cast<const GofSplat*>(g.geom + g.GL.splat),
                    reinterpret_cast<const uint32_t*>(g.bin + g.BL.point_list), reinterpret_cast<const uint2*>(g.img + g.IL.ranges), g.img,
                    point_alloc, point_user, point_binning_alloc, point_binning_user, *out, st);
}

extern "C" size_t gof_integrate_backward_scratch_bytes(int P) { return gof_integrate_backward_scratch(P); }

extern "C" int gof_integrate_backward(const gof_scene_t* s, int PN, const float* points3D, int num_rendered, const int* radii,
                                      void* geom_buffer, const void* binning_buffer, const void* image_buffer, const void* point_buffer,
                                      void* point_binning_buffer, const float* dL_dalpha, const float* dL_dcolor_int, float* dL_dpoints3D,
                                      const gof_backward_out_t* out, void* stream) {
  if (!out) { gof_set_error("integrate_backward: out is NULL"); return GOF_E_INVALID; }
  const struct { const void* p; const char* name; } not_produced[] = {
      {out->dL_dmean2D, "dL_dmean2D"}, {out->dens_sum, "dens_sum"}, {out->dens_max, "dens_max"}, {out->sh_rgb, "sh_rgb"},
      {out->sh_hdr, "sh_hdr"}, {out->dL_dviewmatrix, "dL_dviewmatrix"}, {out->dL_dcampos, "dL_dcampos"}, {out->dL_dtan_fov, "dL_dtan_fov"}};
  for (const auto& f : not_produced)
    if (f.p) { gof_set_error("integrate_backward: out->%s must be NULL (not an output of this backward)", f.name); return GOF_E_INVALID; }
  gof_backward_out_t o = *out;
  const bool with_color = dL_dcolor_int || o.dL_dcolor;   // colour mode (DESIGN.md 4.13)
  if (!with_color) o.dL_dsh = nullptr;                    // alpha mode does not read it
  int rc = validate_scene(s);
  if (rc != GOF_OK) return rc;
  if (PN < 0) { gof_set_error("integrate_backward: PN < 0"); return GOF_E_INVALID; }
  const size_t need = gof_integrate_backward_scratch(s->P);
  if (o.scratch_bytes < need) {
    gof_set_error("integrate_backward: scratch of %zu bytes, %zu needed (gof_integrate_backward_scratch_bytes)", o.scratch_bytes, need);
    return GOF_E_INVALID;
  }
  if (s->P > 0 && !o.scratch) { gof_set_error("integrate_backward: scratch is NULL"); return GOF_E_INVALID; }
  const size_t P = (size_t)s->P;
  if ((PN > 0 && !dL_dalpha && !with_color) || (P > 0 && (!o.dL_dopacity || !o.dL_dmean3D || !o.dL_dview2gaussian)) ||
      (with_color && P > 0 && !o.dL_dcolor)) {
    gof_set_error("integrate_backward: NULL argument");
    return GOF_E_INVALID;
  }
  if (with_color && s->shs && P > 0 && !o.dL_dsh) { gof_set_error("integrate_backward: dL_dsh required with SHs"); return GOF_E_INVALID; }
  if ((rc = check_gaussian_grads("integrate_backward", s, o)) != GOF_OK) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  // P == 0 or PN == 0: gof_integrate ran nothing, no output depends on anything; likewise with no loss at all
  if (P == 0 || PN == 0 || (!dL_dalpha && !dL_dcolor_int)) {
    if (dL_dpoints3D && PN > 0) GOF_CUDA_OK(cudaMemsetAsync(dL_dpoints3D, 0, (size_t)PN * 12, st));
    if (P > 0) {
      if (with_color) GOF_CUDA_OK(cudaMemsetAsync(o.dL_dcolor, 0, P * 12, st));
      if (with_color && s->shs) GOF_CUDA_OK(cudaMemsetAsync(o.dL_dsh, 0, P * (size_t)s->M * 12, st));
      GOF_CUDA_OK(cudaMemsetAsync(o.dL_dopacity, 0, P * 4, st));
      GOF_CUDA_OK(cudaMemsetAsync(o.dL_dmean3D, 0, P * 12, st));
      GOF_CUDA_OK(cudaMemsetAsync(o.dL_dview2gaussian, 0, P * 40, st));
      if (o.dL_dscale) GOF_CUDA_OK(cudaMemsetAsync(o.dL_dscale, 0, P * 12, st));
      if (o.dL_drot) GOF_CUDA_OK(cudaMemsetAsync(o.dL_drot, 0, P * 16, st));
      if (o.dL_dcov3D) GOF_CUDA_OK(cudaMemsetAsync(o.dL_dcov3D, 0, P * 24, st));
    }
    return GOF_OK;
  }
  if (!points3D || !radii || !geom_buffer || !image_buffer || !point_buffer || !point_binning_buffer ||
      (num_rendered > 0 && !binning_buffer) || num_rendered < 0) {
    gof_set_error("integrate_backward: NULL forward state");
    return GOF_E_INVALID;
  }
  const GofView v = gof_make_view(s);
  const GofGeomLayout GL = gof_geom_layout(P);
  const GofImageLayout IL = gof_image_layout(s->width, s->height);
  const GofBinLayout BL = gof_bin_layout((size_t)num_rendered, s->width, s->height, false);
  char* geom = static_cast<char*>(geom_buffer);
  return gof_launch_integrate_backward(s, v, PN, points3D, radii, geom, GL,
                                       reinterpret_cast<const uint32_t*>(static_cast<const char*>(binning_buffer) + BL.point_list),
                                       reinterpret_cast<const uint2*>(static_cast<const char*>(image_buffer) + IL.ranges),
                                       static_cast<const char*>(point_buffer), static_cast<char*>(point_binning_buffer), dL_dalpha,
                                       dL_dcolor_int, dL_dpoints3D, o, st);
}

// ---- the Gaussian side of the query, once per view --------------------------------------------------------------
// extract_mesh.py calls integrate for the same 64 views 10 times (evaluage_alpha on the tetrahedra vertices, 8 bisection
// steps, optionally the colours: extract_mesh.py:56,92,107) and only the query points change: preprocess, depth sort,
// instance emission and tile sort of the Gaussians are identical in every pass.  gof_integrate_prepare runs them once and
// leaves what the query kernel reads -- records, tile ranges, per-tile lists -- in ONE compact cache buffer
// (64 B/Gaussian + 4 B/instance); gof_integrate_cached is the point side alone.
extern "C" size_t gof_integrate_cache_bytes(int P, int width, int height, int num_rendered) {
  if (P < 0 || width <= 0 || height <= 0 || num_rendered < 0) return 0;
  return gof_int_cache_layout((size_t)P, width, height, (size_t)num_rendered).bytes;
}

extern "C" int gof_integrate_prepare(const gof_scene_t* s, gof_alloc_fn geom_alloc, void* geom_user, gof_alloc_fn binning_alloc,
                                     void* binning_user, gof_alloc_fn image_alloc, void* image_user, gof_alloc_fn cache_alloc,
                                     void* cache_user, int* radii, int* num_rendered, void* stream) {
  int rc = validate_scene(s);
  if (rc != GOF_OK) return rc;
  if (!geom_alloc || !binning_alloc || !image_alloc || !cache_alloc || !num_rendered || (!radii && s->P > 0)) {
    gof_set_error("integrate_prepare: NULL argument");
    return GOF_E_INVALID;
  }
  *num_rendered = 0;
  cudaStream_t st = (cudaStream_t)stream;
  const GofView v = gof_make_view(s);
  GaussianSide g{};
  if (s->P > 0 && (rc = gaussian_side(s, v, geom_alloc, geom_user, binning_alloc, binning_user, image_alloc, image_user, radii, 0.5f,
                                      false, num_rendered, st, g)) != GOF_OK)
    return rc;
  const GofIntCacheLayout CL = gof_int_cache_layout((size_t)s->P, s->width, s->height, (size_t)g.R);
  char* cache = (char*)cache_alloc(cache_user, CL.bytes);
  if (!cache) { gof_set_error("cache allocator returned NULL"); return GOF_E_ALLOC; }
  if (s->P == 0) { GOF_CUDA_OK(cudaMemsetAsync(cache + CL.ranges, 0, (size_t)v.tiles * 8, st)); return GOF_OK; }
  GOF_CUDA_OK(cudaMemcpyAsync(cache + CL.splat, g.geom + g.GL.splat, (size_t)s->P * sizeof(GofSplat), cudaMemcpyDeviceToDevice, st));
  GOF_CUDA_OK(cudaMemcpyAsync(cache + CL.ranges, g.img + g.IL.ranges, (size_t)v.tiles * 8, cudaMemcpyDeviceToDevice, st));
  if (g.R) GOF_CUDA_OK(cudaMemcpyAsync(cache + CL.point_list, g.bin + g.BL.point_list, (size_t)g.R * 4, cudaMemcpyDeviceToDevice, st));
  return GOF_OK;
}

extern "C" int gof_integrate_cached(const gof_scene_t* s, int PN, const float* points3D, const void* cache, int num_rendered,
                                    gof_alloc_fn image_alloc, void* image_user, gof_alloc_fn point_alloc, void* point_user,
                                    gof_alloc_fn point_binning_alloc, void* point_binning_user, const gof_integrate_out_t* out,
                                    void* stream) {
  if (!s || s->P < 0 || s->width <= 0 || s->height <= 0 || !s->viewmatrix || !s->background) {
    gof_set_error("integrate_cached: scene needs P, width, height, tan_fov, viewmatrix, background");
    return GOF_E_INVALID;
  }
  int rc = check_integrate_out("integrate_cached", out, true, image_alloc && point_alloc && point_binning_alloc);
  if (rc != GOF_OK) return rc;
  if (s->P == 0 || PN <= 0) return GOF_OK;
  if (!cache || !points3D || num_rendered < 0 || !integrate_outputs_given(*out)) {
    gof_set_error("integrate_cached: NULL argument");
    return GOF_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const GofView v = gof_make_view(s);
  const GofIntCacheLayout CL = gof_int_cache_layout((size_t)s->P, s->width, s->height, (size_t)num_rendered);
  char* img = (char*)image_alloc(image_user, gof_image_layout(s->width, s->height).bytes);
  const char* c = (const char*)cache;
  return point_side(s, v, PN, points3D, reinterpret_cast<const GofSplat*>(c + CL.splat), reinterpret_cast<const uint32_t*>(c + CL.point_list),
                    reinterpret_cast<const uint2*>(c + CL.ranges), img, point_alloc, point_user, point_binning_alloc,
                    point_binning_user, *out, st);
}
