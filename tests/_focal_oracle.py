"""ctypes binding of the float64 ray-gradient oracle (tests/focal_oracle/focal_oracle.c, DESIGN.md 4.10).  TEST INFRASTRUCTURE.

The library is compiled on first use into a per-user temporary directory keyed by the source's hash, so that a read-only tree
works too."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "focal_oracle", "focal_oracle.c")
_FLAGS = ["-O2", "-std=gnu99", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-shared"]
_lib = None


def _load():
    global _lib
    if _lib is None:
        src = open(_SRC, "rb").read()
        key = hashlib.sha256(src + " ".join(_FLAGS).encode()).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), f"gof_focal_oracle_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        lib = os.path.join(d, f"libfocal_oracle_{key}.so")
        if not os.path.exists(lib):
            tmp = f"{lib}.{os.getpid()}"
            cc = "/usr/bin/gcc" if os.access("/usr/bin/gcc", os.X_OK) else "gcc"
            try:   # OpenMP when the toolchain has libgomp, serial otherwise (same results: the pixels are independent)
                subprocess.check_call([cc] + _FLAGS + ["-fopenmp", "-o", tmp, _SRC, "-lm"], stderr=subprocess.DEVNULL)
            except subprocess.CalledProcessError:
                subprocess.check_call([cc] + _FLAGS + ["-o", tmp, _SRC, "-lm"])
            os.replace(tmp, lib)
        _lib = ctypes.CDLL(lib)
        _lib.focal_oracle_rays.restype = None
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def rays(W, H, tan_fovx, tan_fovy, st, bg, dL_dpix, float_geometry=True, bounds=True):
    """Per-pixel dL/drx, dL/dry [2,H,W] float64 of the blend backward from the forward state `st` (the keys of
    gof_oracle.forward's state or _C.export_state: ranges, point_list, conic_opacity, rgb, view2gaussian, accum_alpha,
    n_contrib).  bounds=True also returns the error scales `mag` and `marginal` [2,H,W] (see focal_oracle.c)."""
    lib = _load()
    c = lambda a, dt: np.ascontiguousarray(a, dt)   # noqa: E731
    d = dict(drays=np.zeros((2, H, W), np.float64))
    if bounds:
        d.update(mag=np.zeros((2, H, W), np.float64), marginal=np.zeros((2, H, W), np.float64))
    keep = [c(st["ranges"], np.uint32), c(st["point_list"], np.uint32), c(bg, np.float32), c(st["conic_opacity"], np.float32),
            c(st["rgb"], np.float32), c(st["view2gaussian"], np.float32), c(st["accum_alpha"], np.float32),
            c(st["n_contrib"], np.uint32), c(dL_dpix, np.float32)]
    lib.focal_oracle_rays(int(W), int(H), ctypes.c_float(tan_fovx), ctypes.c_float(tan_fovy), *[_p(a) for a in keep],
                          int(bool(float_geometry)), _p(d["drays"]), _p(d.get("mag")), _p(d.get("marginal")))
    return d


def pixel_rays(W, H, tan_fovx, tan_fovy):
    """The float rays (rx [W], ry [H]) of the blend kernels: ((p + 0.5) - S/2) / focal, focal = S / (2 tan_fov) in float."""
    fx = np.float32(W) / (np.float32(2.0) * np.float32(tan_fovx))
    fy = np.float32(H) / (np.float32(2.0) * np.float32(tan_fovy))
    px = (np.arange(W, dtype=np.float32) + np.float32(0.5)).astype(np.float64)
    py = (np.arange(H, dtype=np.float32) + np.float32(0.5)).astype(np.float64)
    return ((px - W / 2.0) / np.float64(fx)).astype(np.float32), ((py - H / 2.0) / np.float64(fy)).astype(np.float32)


def tan_fov_grad(drays, tan_fovx, tan_fovy):
    """(dL/dtan_fovx, dL/dtan_fovy) in float64 from a [2,H,W] ray gradient: sum rx dL/drx / tan_fovx (and y)."""
    _, H, W = drays.shape
    rx, ry = pixel_rays(W, H, tan_fovx, tan_fovy)
    gx = float((rx.astype(np.float64)[None, :] * drays[0]).sum()) / float(np.float32(tan_fovx))
    gy = float((ry.astype(np.float64)[:, None] * drays[1]).sum()) / float(np.float32(tan_fovy))
    return gx, gy
