"""ctypes binding of the float64 oracle of the query's colour backward (tests/integrate_grad_oracle/integrate_color_oracle.c,
DESIGN.md 4.13).  TEST INFRASTRUCTURE.

That source includes the alpha backward's oracle (integrate_grad_oracle.c) for its restatement of pass 1.  The library is compiled
on first use into a per-user temporary directory keyed by the hash of both sources and the flags, so that a read-only tree works
too."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import _integrate_grad_oracle as igo

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "integrate_grad_oracle")
_SRC = os.path.join(_DIR, "integrate_color_oracle.c")
_lib_handle = None


def _lib():
    global _lib_handle
    if _lib_handle is None:
        h = hashlib.sha256()
        for f in (_SRC, os.path.join(_DIR, "integrate_grad_oracle.c")):
            h.update(open(f, "rb").read())
        h.update(" ".join(igo._FLAGS).encode())
        d = os.path.join(tempfile.gettempdir(), f"gof_integrate_color_oracle_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        path = os.path.join(d, f"libintegrate_color_oracle_{h.hexdigest()[:16]}.so")
        if not os.path.exists(path):
            tmp = f"{path}.{os.getpid()}"
            cc = "/usr/bin/gcc" if os.access("/usr/bin/gcc", os.X_OK) else "gcc"
            subprocess.check_call([cc] + igo._FLAGS + ["-o", tmp, _SRC, "-lm"])
            os.replace(tmp, path)
        lib = ctypes.CDLL(path)
        lib.igc_pixel.restype = None
        lib.igc_pixel.argtypes = [ctypes.c_int] + [ctypes.c_void_p] * 6 + [ctypes.c_float, ctypes.c_float] + [ctypes.c_void_p] * 7
        lib.igc_view.restype = None
        lib.igc_view.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int] + [ctypes.c_void_p] * 13
        _lib_handle = lib
    return _lib_handle


def pixel_dC(xy, ok, dL_dcolor, W, H):
    """dL/dC [H,W,3] of every pixel: the sum of dL/dcolor_integrated over the projected points that fall into it."""
    d = np.zeros((H * W, 3))
    pix = (np.floor(xy[ok, 1]).astype(np.int64) * W + np.floor(xy[ok, 0]).astype(np.int64))
    np.add.at(d, pix, np.asarray(dL_dcolor, np.float64)[ok])
    return d.reshape(H, W, 3)


def view(W, H, tan_fovx, tan_fovy, st, bg, dLdC):
    """The colour backward of one view from the forward state `st` (_C.export_state: ranges, point_list, view2gaussian,
    conic_opacity, rgb) and the per-pixel dL/dC [H,W,3].  Returns dict(dcol / mag_c [P,3], dv2g / mag_g [P,10], marg_g [P] (left
    out), C [H,W,3] (the oracle's pixel colours, where dL/dC != 0))."""
    lib = _lib()
    P = st["view2gaussian"].shape[0]
    c = lambda a, dt: np.ascontiguousarray(a, dt)   # noqa: E731
    d = dict(dcol=np.zeros((P, 3)), mag_c=np.zeros((P, 3)), dv2g=np.zeros((P, 10)), mag_g=np.zeros((P, 10)),
             marg_g=np.zeros(P, np.uint8), C=np.zeros((H, W, 3)))
    keep = [c(st["ranges"], np.uint32), c(st["point_list"], np.uint32), c(st["view2gaussian"], np.float32),
            c(st["conic_opacity"], np.float32), c(st["rgb"], np.float32), c(bg, np.float32), c(dLdC, np.float64)]
    lib.igc_view(int(W), int(H), ctypes.c_float(tan_fovx), ctypes.c_float(tan_fovy), int(P), *[igo._p(a) for a in keep],
                 *[igo._p(d[k]) for k in ("dcol", "mag_c", "dv2g", "mag_g", "marg_g", "C")])
    d["marg_g"] = d["marg_g"].astype(bool)
    return d
