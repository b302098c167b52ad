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


class _BackwardOut(ctypes.Structure):
    """gof_backward_out_t: the outputs of gof_rasterize_backward_ex and of gof_integrate_backward."""
    _fields_ = [(n, _fp) for n in (
        "dL_dmean2D", "dL_dopacity", "dL_dcolor", "dL_dmean3D", "dL_dcov3D", "dL_dsh", "dL_dscale", "dL_drot", "dL_dview2gaussian",
        "dens_sum", "dens_max", "sh_rgb", "sh_hdr", "dL_dviewmatrix", "dL_dcampos", "dL_dtan_fov", "scratch")] + \
        [("scratch_bytes", ctypes.c_size_t)]


class _IntegrateOut(ctypes.Structure):
    """gof_integrate_out_t: the outputs of gof_integrate and gof_integrate_cached, the query's or the running minimum's."""
    _fields_ = [(n, _fp) for n in ("out_color", "out_alpha_integrated", "out_color_integrated", "alpha_min", "argmin")] + \
        [("view", ctypes.c_int), ("color_min", _fp), ("grad_min", _fp)]


class _StateView(ctypes.Structure):
    _fields_ = [(n, _fp) for n in (
        "depths", "means2D", "conic_opacity", "rgb", "view2gaussian", "clamped", "tiles_touched",
        "point_list", "ranges", "accum_alpha", "n_contrib", "blend_masks")]


_lib.gof_last_error.restype = ctypes.c_char_p
_lib.gof_rasterize_forward.restype = ctypes.c_int
_lib.gof_rasterize_forward.argtypes = [
    ctypes.POINTER(_Scene), _ALLOC_FN, ctypes.c_void_p, _ALLOC_FN, ctypes.c_void_p, _ALLOC_FN, ctypes.c_void_p,
    _fp, _fp, ctypes.POINTER(ctypes.c_int), ctypes.c_void_p]
_lib.gof_rasterize_backward_scratch_bytes.restype = ctypes.c_size_t
_lib.gof_rasterize_backward_scratch_bytes.argtypes = [ctypes.c_int] * 5
_lib.gof_rasterize_backward_ex.restype = ctypes.c_int
_lib.gof_rasterize_backward_ex.argtypes = [ctypes.POINTER(_Scene), ctypes.c_int, _fp, _fp, _fp, _fp, _fp, ctypes.POINTER(_BackwardOut),
                                           ctypes.c_void_p]
_lib.gof_sh_grad_from_views.restype = ctypes.c_int
_lib.gof_sh_grad_from_views.argtypes = [ctypes.c_int] * 3 + [_fp, ctypes.c_void_p, _fp, ctypes.c_void_p]
_lib.gof_mark_visible.restype = ctypes.c_int
_lib.gof_mark_visible.argtypes = [ctypes.c_int, _fp, _fp, _fp, _fp, ctypes.c_void_p]
_lib.gof_integrate.restype = ctypes.c_int
_lib.gof_integrate.argtypes = [ctypes.POINTER(_Scene), ctypes.c_int, _fp] + [_ALLOC_FN, ctypes.c_void_p] * 5 + \
    [_fp, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(_IntegrateOut), ctypes.c_void_p]
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


def _check_out(name, t, shape, dtype, aligned=False):
    """Checks an output tensor the caller supplies: contiguous, of `dtype` and of `shape` -- or, with `shape` an int, of at least
    that many elements in any shape -- and, with `aligned`, 16-byte aligned for the library's 128-bit stores.  Returns t."""
    fits = t is not None and (t.numel() >= shape if isinstance(shape, int) else tuple(t.shape) == tuple(shape))
    if not (fits and t.is_contiguous() and t.dtype == dtype):
        size = f"at least {shape} elements" if isinstance(shape, int) else f"shape {tuple(shape)}"
        raise RuntimeError(f"gof_b200: {name} must be a contiguous {dtype} tensor of {size}")
    if aligned and t.numel() and (t.data_ptr() & 15):
        raise RuntimeError(f"gof_b200: {name} must be 16-byte aligned (128-bit stores)")
    return t


def _pad64(n):
    return (int(n) + 63) // 64 * 64


def _sh_plane(P):
    """GOF_SH_PLANE(P) (include/gof_rasterizer.h): the floats of one colour plane of a factored SH gradient record."""
    return _pad64(P)


def _layout(shapes):
    """Lays the named shapes out, in order, in one flat fp32 buffer: ({name: (offset, shape)}, total floats).  Every view starts
    on a multiple of 64 floats, 256 bytes: k_preprocess_backward stores dL_drot as float4 and dL_dsh in 128-bit rows, so the views
    must be 16-byte aligned for any P (after densification P is arbitrary)."""
    offsets, total = {}, 0
    for name, shape in shapes.items():
        offsets[name] = (total, tuple(shape))
        total += _pad64(torch.Size(shape).numel())
    return offsets, total


def _views(flat, offsets):
    """The contiguous views of `flat` at the offsets of _layout, by name."""
    return {name: flat[off:off + torch.Size(shape).numel()].view(shape) for name, (off, shape) in offsets.items()}


def _backward_out(scratch_bytes=0, **tensors):
    """The _BackwardOut of the given output tensors by field name; a tensor that is None or empty is NULL (_ptr)."""
    return _BackwardOut(scratch_bytes=scratch_bytes, **{k: None if t is None else _ptr(t, t.dtype) for k, t in tensors.items()})


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
        pooled = bool(role)

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
                holder[0] = torch.empty(int(nbytes), dtype=torch.uint8, device=device)   # >= 512-byte aligned
            return holder[0].data_ptr()

        self.cb = _ALLOC_FN(alloc)

    @property
    def tensor(self):
        return self._holder[0]


def _gaussian_scratch(device):
    """The pooled geom / binning / image _Scratch of a view's Gaussian side, on `device`, or on the current CUDA device when
    `device` is not a CUDA device (a call without Gaussians).  The binning buffer is sized by the number of rendered instances,
    which changes from view to view: it is allocated with 25% slack so that the pooled buffer can be reused."""
    dev = device if device.type == "cuda" else torch.device("cuda")
    return _Scratch(dev, "geom"), _Scratch(dev, "binning", 1.25), _Scratch(dev, "image")


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _scalar(x):
    return float(x.detach()) if isinstance(x, torch.Tensor) else float(x)


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
    # tan_fovx / tan_fovy: Python floats or one-element tensors (a tensor that requires grad carries the focal-length gradient,
    # DESIGN.md 4.10).  Reading a CUDA tensor's value costs one synchronisation of the current stream per call.
    s.tan_fovx, s.tan_fovy = _scalar(tan_fovx), _scalar(tan_fovy)
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
        geom, binning, img = _gaussian_scratch(dev)
        rendered = ctypes.c_int(0)
        if s.P != 0:
            _check(_lib.gof_rasterize_forward(ctypes.byref(s), geom.cb, None, binning.cb, None, img.cb, None,
                                              out_color.data_ptr(), radii.data_ptr(), ctypes.byref(rendered),
                                              _stream()))
    return rendered.value, out_color, radii, geom.tensor, binning.tensor, img.tensor


def rasterize_gaussians_backward(background, means3D, radii, colors, scales, rotations, scale_modifier,
                                 cov3D_precomp, view2gaussian_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy,
                                 kernel_size, subpixel_offset, dL_dout_color, sh, degree, campos, geomBuffer, R,
                                 binningBuffer, imageBuffer, debug, _out=None, _camera=False, _intrinsics=False, _ray_map=False):
    """RasterizeGaussiansBackwardCUDA (rasterize_points.cu:124-211).  Returns, in the reference's order
    (:210): (dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales,
    dL_drotations, dL_dview2gaussian).  `_camera=True` (extension, gof_backward_out_t.dL_dviewmatrix / dL_dcampos) appends
    dL_dviewmatrix and dL_dcampos, shaped like viewmatrix and campos.  `_intrinsics=True` (extension,
    gof_backward_out_t.dL_dtan_fov) then appends dL_dtanfovx and dL_dtanfovy, 0-dim float32 tensors on the device.
    `_ray_map=True` (tests only; needs _intrinsics) appends the per-pixel float64 [2,H,W] dL/drx, dL/dry of the call."""
    P = means3D.size(0)
    H, W = dL_dout_color.size(1), dL_dout_color.size(2)
    keep = []
    opac_dummy = means3D  # backward never reads opacities; any non-null pointer satisfies validation
    s = _scene(keep, background, means3D, colors, opac_dummy, scales, rotations, scale_modifier, cov3D_precomp,
               view2gaussian_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, kernel_size, subpixel_offset,
               H, W, sh, degree, campos, False, debug)
    M, dev = s.M, means3D.device
    # `_out` (extension, used by gof_dp.GradBucket): pre-zeroed, contiguous destination tensors, e.g. views of one flat all-reduce
    # buffer, so the backward writes straight into the communication buffer
    out = {} if _out is None else _out
    # `_out` with "dsh_rgb" (3, GOF_SH_PLANE(P)) + "sh_hdr" (>= 4 floats): the factored SH gradient of view-parallel training (gof_dp.GradBucket,
    # csrc/sh_views.cu) -- the backward leaves the clamp-masked dL_dRGB and the camera centre instead of dL_dsh, which only exists
    # after the bucket's exchange (the returned dL_dsh is then _out.get("dsh"): the tensor the exchange fills)
    factored = "dsh_rgb" in out
    if factored and _camera:
        raise NotImplementedError("gof_b200: camera gradients are not available with the factored SH gradient (_out['dsh_rgb'])")
    if factored and _intrinsics:
        raise NotImplementedError("gof_b200: focal-length gradients are not available with the factored SH gradient (_out['dsh_rgb'])")
    if _ray_map and not _intrinsics:
        raise RuntimeError("gof_b200: _ray_map needs _intrinsics=True")
    rgb_t = hdr_t = full_t = None
    if factored:
        if sh is None or sh.numel() == 0:
            raise RuntimeError("gof_b200: the factored SH gradient (_out['dsh_rgb']) needs SH input")
        rgb_t = _check_out("_out['dsh_rgb']", out["dsh_rgb"], (3, _sh_plane(P)), torch.float32)
        hdr_t = _check_out("_out['sh_hdr']", out.get("sh_hdr"), 4, torch.float32)
        out["_means3D"] = means3D if means3D.is_contiguous() else means3D.contiguous()
        full_t = out.get("_dsh_full")      # checks only: ALSO write this view's own dL_dsh (P,M,3), from the same dL_dRGB
        if full_t is not None:
            _check_out("_out['_dsh_full']", full_t, (P, M, 3), torch.float32, aligned=True)

    # One UNINITIALISED block for the gradient tensors `_out` does not supply (the reference zero-fills ten tensors,
    # rasterize_points.cu:161-170: 324 MB of memset per backward at 1 M Gaussians): the library's backward writes every element of
    # every output itself -- zeros for Gaussians the view does not see, for dL_dcov3D and for SH coefficients above the active degree.
    # (The reference also allocates dL_dconic, (P,2,2) zeros that nothing writes or returns.)
    shapes = dict(dmeans3D=(P, 3), dmeans2D=(P, 3), dcolors=(P, 3), dopacity=(P, 1), dcov3D=(P, 6), dsh=(P, M, 3),
                  dscales=(P, 3), drot=(P, 4), dv2g=(P, 10))
    if factored:
        del shapes["dsh"]
    offsets, total = _layout({k: shp for k, shp in shapes.items() if k not in out})
    dL = _views((torch.empty if P else torch.zeros)(max(total, 1), dtype=means3D.dtype, device=dev), offsets)
    for k, shp in shapes.items():
        if k in out:
            dL[k] = _check_out(f"_out[{k!r}]", out[k], shp, means3D.dtype, aligned=True)
    dL_dsh = out.get("dsh") if factored else dL["dsh"]
    dL_dviewmatrix = dL_dcampos = fov_out = None
    if _camera:
        if viewmatrix.numel() != 16 or campos.numel() != 3:
            raise RuntimeError("gof_b200: camera gradients need a 16-element viewmatrix and a 3-element campos")
        cam_out = torch.empty(19, dtype=torch.float32, device=dev)
        dL_dviewmatrix, dL_dcampos = cam_out[:16], cam_out[16:]
    if _intrinsics:
        fov_out = torch.empty(2, dtype=torch.float32, device=dev)
    if P != 0 or _camera or _intrinsics:   # with P == 0 the library writes the camera and focal-length gradients as zeros
        g = dL_dout_color.contiguous()
        rad = radii.contiguous()
        with torch.cuda.device(dev):
            # `_out` may carry "dens_sum" (P,3) / "dens_max" (P,2): this view's densification statistics (gof_dp.GradBucket)
            ds, dm = out.get("dens_sum"), out.get("dens_max")
            if (ds is None) != (dm is None):
                raise RuntimeError("gof_b200: _out needs both dens_sum and dens_max, or neither")
            if ds is not None:
                _check_out("dens_sum", ds, (P, 3), torch.float32)
                _check_out("dens_max", dm, (P, 2), torch.float32)
            nbytes = int(_lib.gof_rasterize_backward_scratch_bytes(P, W, H, int(_camera), int(_intrinsics)))
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev) if nbytes else None
            o = _backward_out(nbytes, dL_dmean2D=dL["dmeans2D"], dL_dopacity=dL["dopacity"], dL_dcolor=dL["dcolors"],
                              dL_dmean3D=dL["dmeans3D"], dL_dcov3D=dL["dcov3D"], dL_dsh=full_t if factored else dL_dsh,
                              dL_dscale=dL["dscales"], dL_drot=dL["drot"], dL_dview2gaussian=dL["dv2g"], dens_sum=ds, dens_max=dm,
                              sh_rgb=rgb_t, sh_hdr=hdr_t, dL_dviewmatrix=dL_dviewmatrix, dL_dcampos=dL_dcampos,
                              dL_dtan_fov=fov_out, scratch=scratch)
            _check(_lib.gof_rasterize_backward_ex(ctypes.byref(s), int(R), _ptr(rad, torch.int32), _ptr(geomBuffer, torch.uint8),
                                                  _ptr(binningBuffer, torch.uint8), _ptr(imageBuffer, torch.uint8), _ptr(g),
                                                  ctypes.byref(o), _stream()))
    grads = (dL["dmeans2D"], dL["dcolors"], dL["dopacity"], dL["dmeans3D"], dL["dcov3D"], dL_dsh, dL["dscales"], dL["drot"], dL["dv2g"])
    if _camera:
        grads += (dL_dviewmatrix.view(viewmatrix.shape), dL_dcampos.view(campos.shape))
    if _intrinsics:
        grads += (fov_out[0], fov_out[1])
    if _ray_map:
        # the per-pixel [2][H][W] doubles follow the camera pass's rows in the scratch (gof_backward_out_t.scratch)
        if P == 0:
            grads += (torch.zeros((2, H, W), dtype=torch.float64, device=dev),)
        else:
            off = nbytes - 16 * (W * H + ((W + 15) // 16) * ((H + 15) // 16))
            grads += (scratch[off:off + 16 * W * H].view(torch.float64).view(2, H, W),)
    return grads


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
    return _integrate(background, points3D, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                      view2gaussian_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, kernel_size, subpixel_offset,
                      image_height, image_width, sh, degree, campos, prefiltered, debug)[:8]


def integrate_gaussians_to_points_state(*args):
    """integrate_gaussians_to_points (same arguments) that also returns the point-side buffers the backward reads:
    (num_rendered, out_color, out_alpha_integrated, out_color_integrated, radii, geomBuffer, binningBuffer, imgBuffer,
    pointBuffer, pointBinningBuffer) -- together the forward state of integrate_gaussians_to_points_backward."""
    return _integrate(*args)


def _running_min(PN, alpha_min, argmin, color_min=None, grad_min=None):
    """Checks the running minimum's tensors: alpha_min float32 [PN], argmin int32 [PN], color_min and grad_min float32 [PN,3] or
    None, all contiguous.  Returns those given, by name."""
    given = {"alpha_min": (alpha_min, (PN,), torch.float32), "argmin": (argmin, (PN,), torch.int32),
             "color_min": (color_min, (PN, 3), torch.float32), "grad_min": (grad_min, (PN, 3), torch.float32)}
    return {name: _check_out(name, t, shape, dt) for name, (t, shape, dt) in given.items() if t is not None}


def _query_outputs(PN, H, W, dev, minimum):
    """The outputs of one query by gof_integrate_out_t's field names: the running minimum's tensors `minimum` (from _running_min)
    or, with `minimum` None, the query's three, initialised as the library expects (it leaves the points that do not project,
    and channels 3-5 of out_color, alone)."""
    if minimum is not None:
        return minimum
    return {"out_color": torch.zeros((9, H, W), dtype=torch.float32, device=dev),
            "out_alpha_integrated": torch.ones((PN,), dtype=torch.float32, device=dev),
            "out_color_integrated": torch.zeros((PN, 3), dtype=torch.float32, device=dev)}


def _integrate_out(outs, view, dev):
    """The _IntegrateOut of _query_outputs' tensors."""
    return _IntegrateOut(view=int(view), **{k: _ptr(t, t.dtype, device=dev) for k, t in outs.items()})


def _integrate(background, points3D, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
               view2gaussian_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, kernel_size, subpixel_offset, image_height,
               image_width, sh, degree, campos, prefiltered, debug, view=0, **running_min):
    """gof_integrate, the query's outputs or, with `running_min` (the tensors of _running_min), a view's step of the running
    minimum.  Returns integrate_gaussians_to_points_state's tuple; its three outputs are None with `running_min`."""
    if points3D.ndimension() != 2 or points3D.size(1) != 3:
        raise RuntimeError("points3D must have dimensions (num_points, 3)")
    PN = points3D.size(0)
    minimum = _running_min(PN, **running_min) if running_min else None
    keep = []
    s = _scene(keep, background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
               view2gaussian_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, kernel_size, subpixel_offset,
               image_height, image_width, sh, degree, campos, prefiltered, debug)
    dev = means3D.device
    outs = _query_outputs(PN, int(image_height), int(image_width), dev, minimum)
    radii = torch.zeros((s.P,), dtype=torch.int32, device=dev)
    geom, binning, img = _gaussian_scratch(dev)
    sdev = geom.tensor.device
    pts, pbin = _Scratch(sdev, "points"), _Scratch(sdev, "point_binning")
    rendered = ctypes.c_int(0)
    if s.P != 0 and PN != 0:
        p3 = points3D.contiguous()
        with torch.cuda.device(dev):
            _check(_lib.gof_integrate(ctypes.byref(s), PN, _ptr(p3, device=dev), geom.cb, None, binning.cb, None, img.cb, None,
                                      pts.cb, None, pbin.cb, None, radii.data_ptr(), ctypes.byref(rendered),
                                      ctypes.byref(_integrate_out(outs, view, dev)), _stream()))
    return (rendered.value, outs.get("out_color"), outs.get("out_alpha_integrated"), outs.get("out_color_integrated"), radii,
            geom.tensor, binning.tensor, img.tensor, pts.tensor, pbin.tensor)


def integrate_gaussians_to_points_min(background, points3D, means3D, colors, opacity, scales, rotations, scale_modifier,
                                      cov3D_precomp, view2gaussian_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, kernel_size,
                                      subpixel_offset, image_height, image_width, sh, degree, campos, prefiltered, debug, view,
                                      alpha_min, argmin, color_min=None):
    """gof_integrate's running minimum (extension, DESIGN.md 4.12): integrate_gaussians_to_points for view index `view`, folded
    into the running minimum over views in place: where a point's alpha_integrated < alpha_min, alpha_min takes it and argmin
    takes `view`.  alpha_min (float32 [PN], start at 1) and argmin (int32 [PN], start at 2^30) must be contiguous.  With
    color_min (float32 [PN,3], contiguous; DESIGN.md 4.13) the same update also stores the point's color_integrated of that
    view.  Returns radii [P]."""
    return _integrate(background, points3D, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                      view2gaussian_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, kernel_size, subpixel_offset, image_height,
                      image_width, sh, degree, campos, prefiltered, debug, view, alpha_min=alpha_min, argmin=argmin,
                      color_min=color_min)[4]


_lib.gof_integrate_backward_scratch_bytes.restype = ctypes.c_size_t
_lib.gof_integrate_backward_scratch_bytes.argtypes = [ctypes.c_int]
_lib.gof_integrate_backward.restype = ctypes.c_int
_lib.gof_integrate_backward.argtypes = [ctypes.POINTER(_Scene), ctypes.c_int, _fp, ctypes.c_int] + [_fp] * 9 + \
    [ctypes.POINTER(_BackwardOut), ctypes.c_void_p]


def integrate_gaussians_to_points_backward(background, points3D, means3D, radii, colors, scales, rotations, scale_modifier,
                                           cov3D_precomp, view2gaussian_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy,
                                           kernel_size, subpixel_offset, image_height, image_width, sh, degree, campos,
                                           dL_dalpha, num_rendered, geomBuffer, binningBuffer, imgBuffer, pointBuffer,
                                           pointBinningBuffer, debug, points_grad=True, dL_dcolor=None):
    """gof_integrate_backward (extension, DESIGN.md 4.11): the gradient dL_dalpha [PN] of out_alpha_integrated ->
    (dL_dpoints3D [PN,3] or None, dL_dopacity [P,1], dL_dmeans3D [P,3], dL_dscales [P,3], dL_drotations [P,4],
    dL_dcov3D [P,6], dL_dview2gaussian [P,10], dL_dcolors, dL_dsh).  The state is what integrate_gaussians_to_points_state
    returned.  With dL_dcolor [PN,3], the gradient of out_color_integrated (colour mode, DESIGN.md 4.13), dL_dalpha may be
    None, and dL_dcolors [P,3] and dL_dsh [P,M,3] (None without SHs) are computed; without it both are None."""
    P, PN = means3D.size(0), points3D.size(0)
    keep = []
    s = _scene(keep, background, means3D, colors, means3D, scales, rotations, scale_modifier, cov3D_precomp,
               view2gaussian_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, kernel_size, subpixel_offset, image_height,
               image_width, sh, degree, campos, False, debug)
    dev = means3D.device
    # one block for the six outputs, laid out as rasterize_gaussians_backward's: the rotation gradient is written with 16-byte stores
    offsets, total = _layout(dict(dopacity=(P, 1), dmeans3D=(P, 3), dscales=(P, 3), drot=(P, 4), dcov3D=(P, 6), dv2g=(P, 10)))
    out = _views(torch.empty(max(total, 1), dtype=torch.float32, device=dev), offsets)
    dpts = torch.empty((PN, 3), dtype=torch.float32, device=dev) if points_grad else None
    nbytes = int(_lib.gof_integrate_backward_scratch_bytes(P))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev) if nbytes else None
    p3 = _c(points3D)
    color = dL_dcolor is not None
    g = None if color and dL_dalpha is None else _c(dL_dalpha)
    if g is not None and g.numel() != PN:
        raise RuntimeError(f"gof_b200: dL_dalpha has {g.numel()} elements, expected {PN}")
    has_sr = s.scales is not None and s.rotations is not None
    gc = dcolors = dsh = None
    if color:
        gc = _c(dL_dcolor)
        if gc.numel() != 3 * PN:
            raise RuntimeError(f"gof_b200: dL_dcolor has {gc.numel()} elements, expected {3 * PN}")
        dcolors = torch.empty((P, 3), dtype=torch.float32, device=dev)
        dsh = torch.empty((P, s.M, 3), dtype=torch.float32, device=dev) if s.M > 0 else None
    o = _backward_out(nbytes, dL_dopacity=out["dopacity"], dL_dmean3D=out["dmeans3D"], dL_dscale=out["dscales"] if has_sr else None,
                      dL_drot=out["drot"] if has_sr else None, dL_dview2gaussian=out["dv2g"], dL_dcov3D=out["dcov3D"], dL_dcolor=dcolors,
                      dL_dsh=dsh, scratch=scratch)
    u8 = torch.uint8
    with torch.cuda.device(dev):
        _check(_lib.gof_integrate_backward(
            ctypes.byref(s), PN, _ptr(p3, device=dev), int(num_rendered), _ptr(radii.contiguous(), torch.int32), _ptr(geomBuffer, u8),
            _ptr(binningBuffer, u8), _ptr(imgBuffer, u8), _ptr(pointBuffer, u8), _ptr(pointBinningBuffer, u8), _ptr(g, device=dev),
            _ptr(gc, device=dev), _ptr(dpts), ctypes.byref(o), _stream()))
    if P and not has_sr:
        out["dscales"].zero_()
        out["drot"].zero_()
    return dpts, out["dopacity"], out["dmeans3D"], out["dscales"], out["drot"], out["dcov3D"], out["dv2g"], dcolors, dsh


_lib.gof_integrate_cache_bytes.restype = ctypes.c_size_t
_lib.gof_integrate_cache_bytes.argtypes = [ctypes.c_int] * 4
_lib.gof_integrate_prepare.restype = ctypes.c_int
_lib.gof_integrate_prepare.argtypes = [ctypes.POINTER(_Scene)] + [_ALLOC_FN, ctypes.c_void_p] * 4 + [_fp, ctypes.POINTER(ctypes.c_int), ctypes.c_void_p]
_lib.gof_integrate_cached.restype = ctypes.c_int
_lib.gof_integrate_cached.argtypes = [ctypes.POINTER(_Scene), ctypes.c_int, _fp, _fp, ctypes.c_int] + [_ALLOC_FN, ctypes.c_void_p] * 3 + \
    [ctypes.POINTER(_IntegrateOut), ctypes.c_void_p]


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
    geom, binning, img = _gaussian_scratch(dev)
    cache = _Scratch(dev)          # not pooled: the cache outlives the call
    rendered = ctypes.c_int(0)
    with torch.cuda.device(dev):
        _check(_lib.gof_integrate_prepare(ctypes.byref(s), geom.cb, None, binning.cb, None, img.cb, None, cache.cb, None,
                                          radii.data_ptr(), ctypes.byref(rendered), _stream()))
    return IntegrateCache(cache.tensor, rendered.value, radii, s.P, int(image_height), int(image_width))


def _integrate_cached(cache, background, points3D, viewmatrix, tan_fovx, tan_fovy, debug, view=0, **running_min):
    """gof_integrate_cached, the query's outputs or, with `running_min` (the tensors of _running_min), a view's step of the
    running minimum.  Returns the three outputs, None with `running_min`."""
    if points3D.ndimension() != 2 or points3D.size(1) != 3:
        raise RuntimeError("points3D must have dimensions (num_points, 3)")
    PN = points3D.size(0)
    minimum = _running_min(PN, **running_min) if running_min else None
    dev = cache.buffer.device
    s = _Scene()
    s.P, s.width, s.height = cache.P, cache.W, cache.H
    s.tan_fovx, s.tan_fovy = _scalar(tan_fovx), _scalar(tan_fovy)
    bg, vm, p3 = _c(background), _c(viewmatrix), _c(points3D)
    s.background, s.viewmatrix, s.debug = _ptr(bg, device=dev), _ptr(vm, device=dev), int(bool(debug))
    outs = _query_outputs(PN, cache.H, cache.W, dev, minimum)
    img, pts, pbin = _Scratch(dev, "image"), _Scratch(dev, "points"), _Scratch(dev, "point_binning")
    if cache.P != 0 and PN != 0:
        with torch.cuda.device(dev):
            _check(_lib.gof_integrate_cached(ctypes.byref(s), PN, _ptr(p3, device=dev), cache.buffer.data_ptr(), cache.num_rendered,
                                             img.cb, None, pts.cb, None, pbin.cb, None, ctypes.byref(_integrate_out(outs, view, dev)),
                                             _stream()))
    return outs.get("out_color"), outs.get("out_alpha_integrated"), outs.get("out_color_integrated")


def integrate_points_cached(cache, background, points3D, viewmatrix, tan_fovx, tan_fovy, debug=False):
    """Point side of integrate_gaussians_to_points against an IntegrateCache of the same view.
    Returns (out_color[9,H,W], out_alpha_integrated[PN], out_color_integrated[PN,3])."""
    return _integrate_cached(cache, background, points3D, viewmatrix, tan_fovx, tan_fovy, debug)


def integrate_points_cached_min(cache, background, points3D, viewmatrix, tan_fovx, tan_fovy, view, alpha_min, argmin,
                                color_min=None, grad_min=None, debug=False):
    """gof_integrate_cached's running minimum (extension, DESIGN.md 4.14): integrate_points_cached for view index `view`, folded
    into the running minimum over views in place, as integrate_gaussians_to_points_min folds it (alpha_min float32 [PN] from 1,
    argmin int32 [PN] from 2^30, color_min float32 [PN,3] or None).  With grad_min (float32 [PN,3]) the same update also stores
    the winning view's d alpha_integrated / d point in world space; points that no view updates keep what the caller put there."""
    _integrate_cached(cache, background, points3D, viewmatrix, tan_fovx, tan_fovy, debug, view, alpha_min=alpha_min, argmin=argmin,
                      color_min=color_min, grad_min=grad_min)


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
