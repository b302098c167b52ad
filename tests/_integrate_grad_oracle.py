"""ctypes binding of the float64 oracle of the opacity-field query's backward (tests/integrate_grad_oracle, DESIGN.md 4.11).
TEST INFRASTRUCTURE.

The library is compiled on first use into a per-user temporary directory keyed by the source's hash, so that a read-only tree
works too."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "integrate_grad_oracle", "integrate_grad_oracle.c")
_FLAGS = ["-O2", "-std=gnu99", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-shared"]
_lib = None


def _load():
    global _lib
    if _lib is None:
        src = open(_SRC, "rb").read()
        key = hashlib.sha256(src + " ".join(_FLAGS).encode()).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), f"gof_integrate_grad_oracle_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        lib = os.path.join(d, f"libintegrate_grad_oracle_{key}.so")
        if not os.path.exists(lib):
            tmp = f"{lib}.{os.getpid()}"
            cc = "/usr/bin/gcc" if os.access("/usr/bin/gcc", os.X_OK) else "gcc"
            subprocess.check_call([cc] + _FLAGS + ["-o", tmp, _SRC, "-lm"])
            os.replace(tmp, lib)
        _lib = ctypes.CDLL(lib)
        _lib.igo_point.restype = ctypes.c_float
        _lib.igo_point.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_float, ctypes.c_float,
                                   ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_double] + [ctypes.c_void_p] * 5
        _lib.igo_view.restype = None
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def point(v2g, opacity, rx, ry, depth, p3, viewmatrix, dL_dA=1.0):
    """One point over the fixed list of Gaussians 0..n-1 (v2g [n,10], effective opacity [n]).  Returns dict(A, dpts [3],
    mag_pts [3], dv2g [n,10], mag_g [n,10], marginal)."""
    lib = _load()
    v = np.ascontiguousarray(v2g, np.float32)
    n = v.shape[0]
    op = np.ascontiguousarray(opacity, np.float32)
    g = np.arange(n, dtype=np.uint32)
    p = np.ascontiguousarray(p3, np.float32)
    vm = np.ascontiguousarray(np.asarray(viewmatrix, np.float64).reshape(16))
    d = dict(dpts=np.zeros(3), mag_pts=np.zeros(3), dv2g=np.zeros((n, 10)), mag_g=np.zeros((n, 10)))
    marg = ctypes.c_int(0)
    vmf = np.ascontiguousarray(vm, np.float32)
    A = lib.igo_point(n, _p(g), _p(v), _p(op), float(rx), float(ry), float(depth), _p(p), _p(vmf), float(dL_dA), _p(d["dpts"]),
                      _p(d["mag_pts"]), _p(d["dv2g"]), _p(d["mag_g"]), ctypes.byref(marg))
    d.update(A=float(A), marginal=bool(marg.value))
    return d


def view(W, H, tan_fovx, tan_fovy, viewmatrix, points3D, xy, depth, ok, st, dL_dalpha):
    """Every point of one view against its pixel's pass-1 list, from the forward state `st` (_C.export_state of an integrate:
    ranges, point_list, view2gaussian, conic_opacity).  xy / depth / ok: the query's projection (gof_oracle.project_points).
    The points must come sorted by pixel (see view_order).  Returns dict(alpha [PN], dpts / mag_pts / allow_pts [PN,3],
    marg_pt [PN] (0; 1 marginal, covered by allow_*; 2 left out), n_list [PN], dv2g / mag_g / allow_g [P,10], marg_g [P] (left
    out))."""
    lib = _load()
    P = st["view2gaussian"].shape[0]
    PN = points3D.shape[0]
    c = lambda a, dt: np.ascontiguousarray(a, dt)   # noqa: E731
    d = dict(alpha=np.ones(PN, np.float32), dpts=np.zeros((PN, 3)), mag_pts=np.zeros((PN, 3)), allow_pts=np.zeros((PN, 3)),
             marg_pt=np.zeros(PN, np.uint8), n_list=np.zeros(PN, np.uint32), dv2g=np.zeros((P, 10)), mag_g=np.zeros((P, 10)),
             allow_g=np.zeros((P, 10)), marg_g=np.zeros(P, np.uint8))
    keep = [c(viewmatrix, np.float32).reshape(16), c(points3D, np.float32), c(np.nan_to_num(xy), np.float32),
            c(np.nan_to_num(depth), np.float32), c(ok, np.uint8), c(st["ranges"], np.uint32), c(st["point_list"], np.uint32),
            c(st["view2gaussian"], np.float32), c(st["conic_opacity"], np.float32), c(dL_dalpha, np.float32)]
    lib.igo_view(int(W), int(H), ctypes.c_float(tan_fovx), ctypes.c_float(tan_fovy), _p(keep[0]), int(P), int(PN),
                 *[_p(a) for a in keep[1:]], *[_p(d[k]) for k in ("alpha", "dpts", "mag_pts", "allow_pts", "marg_pt", "n_list", "dv2g",
                                                                   "mag_g", "allow_g", "marg_g")])
    d["marg_g"] = d["marg_g"].astype(bool)
    return d


def view_order(xy, ok, W):
    """A permutation that sorts the projected points by pixel (the others last)."""
    pix = np.where(ok, np.floor(np.nan_to_num(xy[:, 1])) * W + np.floor(np.nan_to_num(xy[:, 0])), np.inf)
    return np.argsort(pix, kind="stable")
