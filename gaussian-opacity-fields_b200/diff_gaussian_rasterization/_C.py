"""`_C` -- the four native entry points of the reference's pybind module, bound over the C ABI.

Same names, argument order and return tuples as `diff_gaussian_rasterization._C` of the reference
(submodules/diff-gaussian-rasterization/ext.cpp:16-19, rasterize_points.cu:36-122, 124-211, 213-232,
234-343), implemented by ctypes calls into libgof_b200.so (include/gof_rasterizer.h).  torch is used
only for device memory and the current stream.  There is NO fallback: if the CUDA library cannot be
loaded the import fails, and CPU tensors are rejected.
"""
import ctypes
import os
import sys
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libgof_b200.so")
if not os.path.exists(_LIB_PATH):
    raise ImportError(
        f"{_LIB_PATH} is missing: build it with `python gaussian-opacity-fields_b200/build.py` "
        "(or __graft_entry__.build()). The rasterizer has no CPU / PyTorch fallback."
    )
_lib = ctypes.CDLL(_LIB_PATH)

_TRACE = os.environ.get("GOF_TRACE") == "1"
_ALLOC_FN = ctypes.CFUNCTYPE(ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t)
_fp = ctypes.c_void_p  # device pointers travel as integers


class _Scene(ctypes.Structure):
    _fields_ = [
        ("P", ctypes.c_int), ("D", ctypes.c_int), ("M", ctypes.c_int),
        ("width", ctypes.c_int), ("height", ctypes.c_int),
        ("tan_fovx", ctypes.c_float), ("tan_fovy", ctypes.c_float),
        ("kernel_size", ctypes.c_float), ("scale_modifier", ctypes.c_float),
        ("background", _fp), ("means3D", _fp), ("shs", _fp), ("colors_precomp", _fp),
        ("opacities", _fp), ("scales", _fp), ("rotations", _fp), ("cov3D_precomp", _fp),
        ("view2gaussian_precomp", _fp), ("viewmatrix", _fp), ("projmatrix", _fp),
        ("cam_pos", _fp), ("subpixel_offset", _fp),
        ("prefiltered", ctypes.c_int), ("debug", ctypes.c_int),
    ]


class _StateView(ctypes.Structure):
    _fields_ = [(n, _fp) for n in (
        "depths", "means2D", "conic_opacity", "rgb", "view2gaussian", "clamped", "tiles_touched",
        "point_list", "ranges", "accum_alpha", "n_contrib", "blend_masks")]


_lib.gof_last_error.restype = ctypes.c_char_p
_lib.gof_rasterize_forward.restype = ctypes.c_int
_lib.gof_rasterize_forward.argtypes = [
    ctypes.POINTER(_Scene), _ALLOC_FN, ctypes.c_void_p, _ALLOC_FN, ctypes.c_void_p, _ALLOC_FN, ctypes.c_void_p,
    _fp, _fp, ctypes.POINTER(ctypes.c_int), ctypes.c_void_p]
_lib.gof_rasterize_backward.restype = ctypes.c_int
_lib.gof_rasterize_backward.argtypes = [ctypes.POINTER(_Scene), ctypes.c_int] + [_fp] * 15 + [ctypes.c_void_p]
_lib.gof_rasterize_backward_stats.restype = ctypes.c_int
_lib.gof_rasterize_backward_stats.argtypes = [ctypes.POINTER(_Scene), ctypes.c_int] + [_fp] * 17 + [ctypes.c_void_p]
_lib.gof_rasterize_backward_dp.restype = ctypes.c_int
_lib.gof_rasterize_backward_dp.argtypes = [ctypes.POINTER(_Scene), ctypes.c_int] + [_fp] * 19 + [ctypes.c_void_p]
_lib.gof_sh_grad_from_views.restype = ctypes.c_int
_lib.gof_sh_grad_from_views.argtypes = [ctypes.c_int] * 3 + [_fp, ctypes.c_void_p, _fp, ctypes.c_void_p]
_lib.gof_mark_visible.restype = ctypes.c_int
_lib.gof_mark_visible.argtypes = [ctypes.c_int, _fp, _fp, _fp, _fp, ctypes.c_void_p]
_lib.gof_integrate.restype = ctypes.c_int
_lib.gof_integrate.argtypes = [ctypes.POINTER(_Scene), ctypes.c_int, _fp] + [_ALLOC_FN, ctypes.c_void_p] * 5 + \
    [_fp, _fp, _fp, _fp, ctypes.POINTER(ctypes.c_int), ctypes.c_void_p]
_lib.gof_export_state.restype = ctypes.c_int
_lib.gof_export_state.argtypes = [ctypes.c_int] * 4 + [_fp] * 4 + [ctypes.POINTER(_StateView), ctypes.c_void_p]


_ALLOC_ERROR = threading.local()   # per thread: what a scratch allocation raised inside the ctypes callback (see _Scratch)


def _check(rc):
    err = getattr(_ALLOC_ERROR, "exc", None)
    _ALLOC_ERROR.exc = None
    if rc != 0:
        if err is not None:
            raise err
        raise RuntimeError(f"gof_b200 (code {rc}): {_lib.gof_last_error().decode()}")


def _ptr(t, dtype=torch.float32, device=None):
    """Device pointer of a tensor, or None for the reference's "absent" encoding (empty tensor whose
    data_ptr() is null, rasterize_points.cu:98-115)."""
    if t is None or t.numel() == 0:
        return None
    if not t.is_cuda:
        raise RuntimeError("gof_b200: all non-empty tensor arguments must live on a CUDA device (no CPU path)")
    if device is not None and t.device != device:
        raise RuntimeError(f"gof_b200: tensor on {t.device}, expected {device}")
    if t.dtype != dtype:
        raise RuntimeError(f"gof_b200: expected dtype {dtype}, got {t.dtype}")
    return t.data_ptr()


def _c(t, dtype=torch.float32):
    """contiguous and 16-byte aligned (keeps a reference alive in the caller's frame).  The kernels read rotations as float4
    and SH rows with 128-bit loads; the reference accepts any 4-byte aligned tensor, so a contiguous view with an odd storage
    offset (a parameter sliced out of a flat buffer) is copied to a fresh allocation instead of faulting."""
    if t is None:
        return None
    t = t.contiguous()
    if t.is_cuda and t.numel() and (t.data_ptr() & 15):
        t = t.clone(memory_format=torch.contiguous_format)
    return t


class _Pool:
    """Recycles the opaque scratch tensors between calls.

    The reference allocates three fresh byte tensors per forward (rasterize_points.cu:75-79) and lets torch's
    caching allocator recycle them.  At 1080p / 1M Gaussians those are 130 + 50 + 35 MB blocks whose
    allocation showed up as 0.1-2 ms of host time per call in front of the first kernel launch, so the shim
    keeps them: a buffer handed out earlier is reused once nothing else references it any more (neither a
    Python variable nor an autograd saved-tensor slot), which is exactly when the caching allocator could have
    recycled it.  Keyed by (device, stream, role) so that reuse is ordered on one stream."""

    def __init__(self, keep=4):
        self.items, self.keep = {}, keep

    def take(self, key, nbytes, device, slack=1.0):
        lst = self.items.setdefault(key, [])
        for t in lst:
            # references: the list, the loop variable and getrefcount's argument; _use_count()==1: no C++ holder
            if t.numel() >= nbytes and t._use_count() == 1 and sys.getrefcount(t) <= 3:
                return t
        cap = ((int(nbytes * slack) + (1 << 20) - 1) >> 20) << 20
        t = torch.empty(max(cap, 1 << 20), dtype=torch.uint8, device=device)
        # drop surplus idle buffers (identity-based: list.remove would compare tensors element-wise)
        surplus = len(lst) + 1 - self.keep
        if surplus > 0:
            kept = []
            for x in lst:
                if surplus > 0 and x._use_count() == 1 and sys.getrefcount(x) <= 3:
                    surplus -= 1
                else:
                    kept.append(x)
            lst[:] = kept
        lst.append(t)
        return t


_POOL = _Pool()
_USE_POOL = os.environ.get("GOF_POOL", "1") != "0"


class _Scratch:
    """One opaque uint8 CUDA tensor sized by the library through the allocator callback
    (resizeFunctional, rasterize_points.cu:28-34).

    The callback is a closure over a one-element list, NOT a bound method: a ctypes thunk that references its
    owner forms a reference cycle, the buffer then lives until Python's cyclic collector happens to run, and
    both the pool and torch's caching allocator see it as busy (measured: +5 cudaMalloc and ~500 MB of extra
    reserved memory per integrate call, 14 ms spikes in the training loop)."""

    def __init__(self, device, role="", slack=1.0):
        holder = [torch.empty(0, dtype=torch.uint8, device=device)]
        self._holder = holder
        pooled = bool(_USE_POOL and role)

        def alloc(_user, nbytes):
            try:
                return _alloc(nbytes)
            except BaseException as e:      # noqa: BLE001 -- an exception cannot cross the C frame (ctypes would hand the
                _ALLOC_ERROR.exc = e        # library an undefined pointer): NULL makes the call fail, and _check raises e
                return 0

        def _alloc(nbytes):
            if not nbytes:
                return 0
            if pooled:
                idx = device.index if device.index is not None else torch.cuda.current_device()
                key = (idx, torch.cuda.current_stream().cuda_stream, role)
                holder[0] = None                      # drop our reference before asking: the old buffer may be reusable
                holder[0] = _POOL.take(key, int(nbytes), device, slack)
            else:
                if _TRACE:
                    import time
                    t0 = time.perf_counter()
                holder[0] = torch.empty(int(nbytes), dtype=torch.uint8, device=device)   # >= 512-byte aligned
                if _TRACE:
                    print(f"[gof trace py] alloc {int(nbytes)} bytes took {1e6 * (time.perf_counter() - t0):.1f} us",
                          file=sys.stderr, flush=True)
            return holder[0].data_ptr()

        self.cb = _ALLOC_FN(alloc)

    @property
    def tensor(self):
        return self._holder[0]


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _scene(keep, bg, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, v2g_precomp,
           viewmatrix, projmatrix, tan_fovx, tan_fovy, kernel_size, subpixel_offset, H, W, sh, degree, campos,
           prefiltered, debug):
    if means3D.ndimension() != 2 or means3D.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")   # rasterize_points.cu:61-63
    dev = means3D.device
    s = _Scene()
    s.P = means3D.size(0)
    s.D = int(degree)
    s.M = int(sh.size(1)) if (sh is not None and sh.numel() != 0 and sh.size(0) != 0) else 0
    s.width, s.height = int(W), int(H)
    s.tan_fovx, s.tan_fovy = float(tan_fovx), float(tan_fovy)
    s.kernel_size, s.scale_modifier = float(kernel_size), float(scale_modifier)
    for name, t in (("background", bg), ("means3D", means3D), ("shs", sh), ("colors_precomp", colors),
                    ("opacities", opacity), ("scales", scales), ("rotations", rotations),
                    ("cov3D_precomp", cov3D_precomp), ("view2gaussian_precomp", v2g_precomp),
                    ("viewmatrix", viewmatrix), ("projmatrix", projmatrix), ("cam_pos", campos),
                    ("subpixel_offset", subpixel_offset)):
        tc = _c(t)
        keep.append(tc)
        setattr(s, name, _ptr(tc, device=dev if s.P else None) if s.P else None)
    s.prefiltered, s.debug = int(bool(prefiltered)), int(bool(debug))
    return s


def rasterize_gaussians(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                        view2gaussian_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, kernel_size,
                        subpixel_offset, image_height, image_width, sh, degree, campos, prefiltered, debug):
    """RasterizeGaussiansCUDA (rasterize_points.cu:36-122).
    Returns (num_rendered, out_color[9,H,W], radii[P], geomBuffer, binningBuffer, imgBuffer)."""
    keep = []
    s = _scene(keep, background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
               view2gaussian_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, kernel_size, subpixel_offset,
               image_height, image_width, sh, degree, campos, prefiltered, debug)
    dev = means3D.device
    if s.P and not means3D.is_cuda:
        raise RuntimeError("gof_b200: means3D must be a CUDA tensor (no CPU path)")
    with torch.cuda.device(dev if means3D.is_cuda else torch.cuda.current_device()):
        # the forward writes every pixel of the 9 channels and every radius (the reference zero-fills both, rasterize_points.cu:70-72)
        alloc = torch.empty if s.P != 0 else torch.zeros
        out_color = alloc((9, int(image_height), int(image_width)), dtype=torch.float32, device=dev)
        radii = alloc((s.P,), dtype=torch.int32, device=dev)
        sdev = dev if means3D.is_cuda else torch.device("cuda")
        geom, binning, img = _Scratch(sdev, "geom"), _Scratch(sdev, "binning", 1.25), _Scratch(sdev, "image")
        rendered = ctypes.c_int(0)
        if s.P != 0:
            _check(_lib.gof_rasterize_forward(ctypes.byref(s), geom.cb, None, binning.cb, None, img.cb, None,
                                              out_color.data_ptr(), radii.data_ptr(), ctypes.byref(rendered),
                                              _stream()))
    return rendered.value, out_color, radii, geom.tensor, binning.tensor, img.tensor


def rasterize_gaussians_backward(background, means3D, radii, colors, scales, rotations, scale_modifier,
                                 cov3D_precomp, view2gaussian_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy,
                                 kernel_size, subpixel_offset, dL_dout_color, sh, degree, campos, geomBuffer, R,
                                 binningBuffer, imageBuffer, debug, _out=None):
    """RasterizeGaussiansBackwardCUDA (rasterize_points.cu:124-211).  Returns, in the reference's order
    (:210): (dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales,
    dL_drotations, dL_dview2gaussian)."""
    P = means3D.size(0)
    H, W = dL_dout_color.size(1), dL_dout_color.size(2)
    keep = []
    opac_dummy = means3D  # backward never reads opacities; any non-null pointer satisfies validation
    s = _scene(keep, background, means3D, colors, opac_dummy, scales, rotations, scale_modifier, cov3D_precomp,
               view2gaussian_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, kernel_size, subpixel_offset,
               H, W, sh, degree, campos, False, debug)
    M = s.M
    o = dict(dtype=means3D.dtype, device=means3D.device)

    # One UNINITIALISED block for all gradient tensors (the reference zero-fills ten tensors, rasterize_points.cu:161-170: 324 MB
    # of memset per backward at 1 M Gaussians): the library's backward writes every element of every output itself -- zeros for
    # Gaussians the view does not see, for dL_dcov3D and for SH coefficients above the active degree.  Every tensor is a
    # contiguous, 256-byte aligned view of the block.
    shapes = dict(dmeans3D=(P, 3), dmeans2D=(P, 3), dcolors=(P, 3), dopacity=(P, 1), dcov3D=(P, 6), dsh=(P, M, 3),
                  dscales=(P, 3), drot=(P, 4), dv2g=(P, 10))
    # `_out` with "dsh_rgb" (3, GOF_SH_PLANE(P)) + "sh_hdr" (>= 4 floats): the factored SH gradient of view-parallel training (gof_dp.GradBucket,
    # csrc/sh_views.cu) -- the backward leaves the clamp-masked dL_dRGB and the camera centre instead of dL_dsh, which only exists
    # after the bucket's exchange (the returned dL_dsh is then _out.get("dsh"): the tensor the exchange fills)
    factored = _out is not None and "dsh_rgb" in _out
    if factored:
        rgb_t, hdr_t = _out["dsh_rgb"], _out.get("sh_hdr")
        if sh is None or sh.numel() == 0:
            raise RuntimeError("gof_b200: the factored SH gradient (_out['dsh_rgb']) needs SH input")
        plane = (P + 63) // 64 * 64          # GOF_SH_PLANE(P)
        if hdr_t is None or not (rgb_t.is_contiguous() and hdr_t.is_contiguous() and tuple(rgb_t.shape) == (3, plane) and hdr_t.numel() >= 4
                                 and rgb_t.dtype == torch.float32 and hdr_t.dtype == torch.float32):
            raise RuntimeError(f"gof_b200: _out['dsh_rgb'] must be a contiguous float32 (3, {plane}) tensor (three colour planes of "
                               "GOF_SH_PLANE(P) floats) and _out['sh_hdr'] hold >= 4 floats")
        _out["_means3D"] = means3D if means3D.is_contiguous() else means3D.contiguous()
        full_t = _out.get("_dsh_full")      # checks only: ALSO write this view's own dL_dsh (P,M,3), from the same dL_dRGB
        if full_t is not None and not (full_t.is_contiguous() and tuple(full_t.shape) == (P, M, 3) and full_t.dtype == torch.float32
                                       and not (full_t.data_ptr() & 15)):
            raise RuntimeError("gof_b200: _out['_dsh_full'] must be a contiguous, 16-byte aligned float32 (P,M,3) tensor")
    need = {k: v for k, v in shapes.items() if not (_out is not None and k in _out) and not (factored and k == "dsh")}
    offs, total = {}, 0
    for k, shp in need.items():
        offs[k] = total
        n = 1
        for d in shp:
            n *= d
        total += (n + 63) // 64 * 64
    block = torch.empty(max(total, 1), **o) if P else torch.zeros(max(total, 1), **o)

    def _z(name, shape):
        # `_out` (extension, used by gof_dp.GradBucket): pre-zeroed, contiguous destination tensors, e.g. views
        # of one flat all-reduce buffer, so the backward writes straight into the communication buffer
        if _out is not None and name in _out:
            t = _out[name]
            if not (t.is_contiguous() and tuple(t.shape) == tuple(shape) and t.dtype == means3D.dtype):
                raise RuntimeError(f"gof_b200: _out[{name!r}] must be a contiguous {means3D.dtype} tensor of shape {tuple(shape)}")
            if t.numel() and (t.data_ptr() & 15):
                raise RuntimeError(f"gof_b200: _out[{name!r}] must be 16-byte aligned (128-bit stores)")
            return t
        n = 1
        for d in shape:
            n *= d
        return block[offs[name]:offs[name] + n].view(shape)

    dL_dmeans3D = _z("dmeans3D", (P, 3))
    dL_dmeans2D = _z("dmeans2D", (P, 3))
    dL_dcolors = _z("dcolors", (P, 3))
    dL_dconic = None       # the reference allocates (P,2,2) zeros that nothing writes or returns
    dL_dopacity = _z("dopacity", (P, 1))
    dL_dcov3D = _z("dcov3D", (P, 6))
    dL_dsh = _out.get("dsh") if factored else _z("dsh", (P, M, 3))
    dL_dscales = _z("dscales", (P, 3))
    dL_drotations = _z("drot", (P, 4))
    dL_dv2g = _z("dv2g", (P, 10))
    if P != 0:
        g = dL_dout_color.contiguous()
        rad = radii.contiguous()
        with torch.cuda.device(means3D.device):
            # `_out` may carry "dens_sum" (P,3) / "dens_max" (P,2): this view's densification statistics (gof_dp.GradBucket)
            ds = _out.get("dens_sum") if _out is not None else None
            dm = _out.get("dens_max") if _out is not None else None
            if (ds is None) != (dm is None):
                raise RuntimeError("gof_b200: _out needs both dens_sum and dens_max, or neither")
            if ds is not None and not (ds.is_contiguous() and dm.is_contiguous() and tuple(ds.shape) == (P, 3) and tuple(dm.shape) == (P, 2)
                                       and ds.dtype == torch.float32 and dm.dtype == torch.float32):
                raise RuntimeError("gof_b200: dens_sum must be a contiguous float32 (P,3) and dens_max (P,2) tensor")
            _check(_lib.gof_rasterize_backward_dp(
                ctypes.byref(s), int(R), _ptr(rad, torch.int32), _ptr(geomBuffer, torch.uint8),
                _ptr(binningBuffer, torch.uint8), _ptr(imageBuffer, torch.uint8), _ptr(g),
                dL_dmeans2D.data_ptr(), None, dL_dopacity.data_ptr(), dL_dcolors.data_ptr(),
                dL_dmeans3D.data_ptr(), dL_dcov3D.data_ptr(), (_ptr(full_t) if full_t is not None else None) if factored else _ptr(dL_dsh),
                dL_dscales.data_ptr(),
                dL_drotations.data_ptr(), dL_dv2g.data_ptr(), ds.data_ptr() if ds is not None else None,
                dm.data_ptr() if dm is not None else None, rgb_t.data_ptr() if factored else None,
                hdr_t.data_ptr() if factored else None, _stream()))
    return (dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales, dL_drotations,
            dL_dv2g)


def mark_visible(means3D, viewmatrix, projmatrix):
    """markVisible (rasterize_points.cu:213-232)."""
    P = means3D.size(0)
    present = torch.zeros((P,), dtype=torch.bool, device=means3D.device)
    if P != 0:
        m, v, p = means3D.contiguous(), viewmatrix.contiguous(), projmatrix.contiguous()
        with torch.cuda.device(means3D.device):
            _check(_lib.gof_mark_visible(P, _ptr(m), _ptr(v), _ptr(p), present.data_ptr(), _stream()))
    return present


def integrate_gaussians_to_points(background, points3D, means3D, colors, opacity, scales, rotations,
                                  scale_modifier, cov3D_precomp, view2gaussian_precomp, viewmatrix, projmatrix,
                                  tan_fovx, tan_fovy, kernel_size, subpixel_offset, image_height, image_width, sh,
                                  degree, campos, prefiltered, debug):
    """IntegrateGaussiansToPointsCUDA (rasterize_points.cu:234-343).  Returns (num_rendered, out_color,
    out_alpha_integrated, out_color_integrated, radii, geomBuffer, binningBuffer, imgBuffer)."""
    if points3D.ndimension() != 2 or points3D.size(1) != 3:
        raise RuntimeError("points3D must have dimensions (num_points, 3)")
    keep = []
    s = _scene(keep, background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
               view2gaussian_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, kernel_size, subpixel_offset,
               image_height, image_width, sh, degree, campos, prefiltered, debug)
    dev = means3D.device
    PN = points3D.size(0)
    out_color = torch.zeros((9, int(image_height), int(image_width)), dtype=torch.float32, device=dev)
    radii = torch.zeros((s.P,), dtype=torch.int32, device=dev)
    alpha_int = torch.ones((PN,), dtype=torch.float32, device=dev)
    color_int = torch.zeros((PN, 3), dtype=torch.float32, device=dev)
    sdev = dev if means3D.is_cuda else torch.device("cuda")
    geom, binning, img = _Scratch(sdev, "geom"), _Scratch(sdev, "binning", 1.25), _Scratch(sdev, "image")
    pts, pbin = _Scratch(sdev, "points"), _Scratch(sdev, "point_binning")
    rendered = ctypes.c_int(0)
    if s.P != 0 and PN != 0:
        p3 = points3D.contiguous()
        with torch.cuda.device(dev):
            _check(_lib.gof_integrate(ctypes.byref(s), PN, _ptr(p3), geom.cb, None, binning.cb, None, img.cb, None,
                                      pts.cb, None, pbin.cb, None, out_color.data_ptr(), radii.data_ptr(),
                                      alpha_int.data_ptr(), color_int.data_ptr(), ctypes.byref(rendered), _stream()))
    return rendered.value, out_color, alpha_int, color_int, radii, geom.tensor, binning.tensor, img.tensor


_lib.gof_integrate_cache_bytes.restype = ctypes.c_size_t
_lib.gof_integrate_cache_bytes.argtypes = [ctypes.c_int] * 4
_lib.gof_integrate_prepare.restype = ctypes.c_int
_lib.gof_integrate_prepare.argtypes = [ctypes.POINTER(_Scene)] + [_ALLOC_FN, ctypes.c_void_p] * 4 + [_fp, ctypes.POINTER(ctypes.c_int), ctypes.c_void_p]
_lib.gof_integrate_cached.restype = ctypes.c_int
_lib.gof_integrate_cached.argtypes = [ctypes.POINTER(_Scene), ctypes.c_int, _fp, _fp, ctypes.c_int] + [_ALLOC_FN, ctypes.c_void_p] * 3 + \
    [_fp, _fp, _fp, ctypes.c_void_p]


class IntegrateCache:
    """Gaussian side of one view of the opacity-field query (gof_integrate_prepare): records + tile ranges + tile lists in one
    uint8 CUDA tensor.  Opaque; pass it to integrate_points_cached."""

    def __init__(self, buffer, num_rendered, radii, P, H, W):
        self.buffer, self.num_rendered, self.radii, self.P, self.H, self.W = buffer, num_rendered, radii, P, H, W

    @property
    def nbytes(self):
        return self.buffer.numel()


def integrate_prepare(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, view2gaussian_precomp,
                      viewmatrix, projmatrix, tan_fovx, tan_fovy, kernel_size, subpixel_offset, image_height, image_width, sh, degree,
                      campos, prefiltered, debug):
    """Gaussian side of integrate_gaussians_to_points for one view (same arguments minus points3D) -> IntegrateCache."""
    keep = []
    s = _scene(keep, background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, view2gaussian_precomp,
               viewmatrix, projmatrix, tan_fovx, tan_fovy, kernel_size, subpixel_offset, image_height, image_width, sh, degree, campos,
               prefiltered, debug)
    dev = means3D.device
    radii = torch.zeros((s.P,), dtype=torch.int32, device=dev)
    geom, binning, img = _Scratch(dev, "geom"), _Scratch(dev, "binning", 1.25), _Scratch(dev, "image")
    cache = _Scratch(dev)          # not pooled: the cache outlives the call
    rendered = ctypes.c_int(0)
    with torch.cuda.device(dev):
        _check(_lib.gof_integrate_prepare(ctypes.byref(s), geom.cb, None, binning.cb, None, img.cb, None, cache.cb, None,
                                          radii.data_ptr(), ctypes.byref(rendered), _stream()))
    return IntegrateCache(cache.tensor, rendered.value, radii, s.P, int(image_height), int(image_width))


def integrate_points_cached(cache, background, points3D, viewmatrix, tan_fovx, tan_fovy, debug=False):
    """Point side of integrate_gaussians_to_points against an IntegrateCache of the same view.
    Returns (out_color[9,H,W], out_alpha_integrated[PN], out_color_integrated[PN,3])."""
    if points3D.ndimension() != 2 or points3D.size(1) != 3:
        raise RuntimeError("points3D must have dimensions (num_points, 3)")
    dev = cache.buffer.device
    s = _Scene()
    s.P, s.width, s.height = cache.P, cache.W, cache.H
    s.tan_fovx, s.tan_fovy = float(tan_fovx), float(tan_fovy)
    bg, vm, p3 = _c(background), _c(viewmatrix), _c(points3D)
    s.background, s.viewmatrix, s.debug = _ptr(bg, device=dev), _ptr(vm, device=dev), int(bool(debug))
    PN = p3.size(0)
    out_color = torch.zeros((9, cache.H, cache.W), dtype=torch.float32, device=dev)
    alpha_int = torch.ones((PN,), dtype=torch.float32, device=dev)
    color_int = torch.zeros((PN, 3), dtype=torch.float32, device=dev)
    img, pts, pbin = _Scratch(dev, "image"), _Scratch(dev, "points"), _Scratch(dev, "point_binning")
    if cache.P != 0 and PN != 0:
        with torch.cuda.device(dev):
            _check(_lib.gof_integrate_cached(ctypes.byref(s), PN, _ptr(p3, device=dev), cache.buffer.data_ptr(), cache.num_rendered, img.cb,
                                             None, pts.cb, None, pbin.cb, None, out_color.data_ptr(), alpha_int.data_ptr(),
                                             color_int.data_ptr(), _stream()))
    return out_color, alpha_int, color_int


def export_state(P, W, H, num_rendered, geomBuffer, binningBuffer, imgBuffer, radii, masks=False):
    """Parity-test helper (gof_export_state): this library's scratch buffers in the reference's field layout.  masks=True
    (buffers of a forward only) adds "blend_masks", int32 [8, num_rendered + 32 * tiles]: the masks the forward leaves for the
    backward, laid out as GofBinLayout::vmask (csrc/gof_common.cuh); opt-in, as they take 32 bytes per rendered pair."""
    dev = radii.device
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    out = {
        "depths": torch.zeros(P, device=dev), "means2D": torch.zeros(P, 2, device=dev),
        "conic_opacity": torch.zeros(P, 4, device=dev), "rgb": torch.zeros(P, 3, device=dev),
        "view2gaussian": torch.zeros(P, 10, device=dev),
        "clamped": torch.zeros(P, 3, dtype=torch.uint8, device=dev),
        "tiles_touched": torch.zeros(P, dtype=torch.int32, device=dev),
        "point_list": torch.zeros(max(num_rendered, 1), dtype=torch.int32, device=dev),
        "ranges": torch.zeros(tiles, 2, dtype=torch.int32, device=dev),
        "accum_alpha": torch.zeros(4, H, W, device=dev),
        "n_contrib": torch.zeros(2, H, W, dtype=torch.int32, device=dev),
    }
    if masks:
        out["blend_masks"] = torch.zeros(8, num_rendered + 32 * tiles, dtype=torch.int32, device=dev)
    sv = _StateView()
    for k, t in out.items():
        setattr(sv, k, t.data_ptr())
    with torch.cuda.device(dev):
        _check(_lib.gof_export_state(P, W, H, num_rendered, geomBuffer.data_ptr(),
                                     binningBuffer.data_ptr() if binningBuffer.numel() else None,
                                     imgBuffer.data_ptr(), radii.data_ptr(), ctypes.byref(sv), _stream()))
    out["point_list"] = out["point_list"][:num_rendered]
    return out


_lib.gof_launch_count.restype = ctypes.c_ulonglong
_lib.gof_profile_report.restype = ctypes.c_int
_lib.gof_profile_report.argtypes = [ctypes.c_char_p, ctypes.c_int]
_lib.gof_profile_enable.argtypes = [ctypes.c_int]
_lib.gof_profile_timeline.restype = ctypes.c_int
_lib.gof_profile_timeline.argtypes = [ctypes.c_char_p, ctypes.c_int]


def launch_count():
    """Number of CUDA kernels this library has launched so far (process-wide)."""
    return int(_lib.gof_launch_count())


def profile_enable(on=True):
    _lib.gof_profile_enable(1 if on else 0)


def profile_reset():
    _lib.gof_profile_reset()


def profile_timeline():
    """[(kernel, start_ms, end_ms)] for every bracketed launch since profile_reset()."""
    n = _lib.gof_profile_timeline(None, 0)
    buf = ctypes.create_string_buffer(n + 1)
    _lib.gof_profile_timeline(buf, n + 1)
    return [(a, float(b), float(c)) for a, b, c in (ln.split() for ln in buf.value.decode().splitlines())]


def profile_report():
    """{kernel: (launches, total_ms)} measured with CUDA events on the launching stream while enabled."""
    n = _lib.gof_profile_report(None, 0)
    buf = ctypes.create_string_buffer(n + 1)
    _lib.gof_profile_report(buf, n + 1)
    out = {}
    for line in buf.value.decode().splitlines():
        name, cnt, ms = line.split()
        out[name] = (int(cnt), float(ms))
    return out
