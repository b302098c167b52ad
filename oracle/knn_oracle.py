"""ctypes binding of the brute-force CPU oracle of distCUDA2 (oracle/knn_oracle.c).  TEST INFRASTRUCTURE ONLY.

    mean = knn_mean_dist(points)                         # float32 [P]
    mean, best = knn_mean_dist(points, return_best=True) # + the three chosen distances [P,3]
    mean = knn_mean_dist(points, queries=idx)            # only the points idx (spot checks of large clouds)

Compiled with the same flags as libgof_oracle.so (oracle/Makefile: -ffp-contract=off -fno-fast-math, OpenMP when the
toolchain has it).
"""
import ctypes
import os
import shutil
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "knn_oracle.c")
_LIB = os.path.join(_HERE, "libknn_oracle.so")
_CFLAGS = ["-O2", "-std=gnu99", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-shared"]


def build():
    cc = "/usr/bin/gcc" if os.access("/usr/bin/gcc", os.X_OK) else (shutil.which("gcc") or "cc")
    tmp = _LIB + f".{os.getpid()}.tmp"
    try:
        subprocess.check_call([cc] + _CFLAGS + ["-fopenmp", "-o", tmp, _SRC, "-lm"], stderr=subprocess.DEVNULL)
    except subprocess.CalledProcessError:
        subprocess.check_call([cc] + _CFLAGS + ["-o", tmp, _SRC, "-lm"])
    os.replace(tmp, _LIB)
    return _LIB


def _load():
    if not os.path.exists(_LIB) or os.path.getmtime(_LIB) < os.path.getmtime(_SRC):
        build()
    lib = ctypes.CDLL(_LIB)
    lib.gof_oracle_knn_mean_dist.restype = None
    lib.gof_oracle_knn_mean_dist.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                             ctypes.c_void_p]
    return lib


_lib = None


def knn_mean_dist(points, queries=None, return_best=False):
    global _lib
    if _lib is None:
        _lib = _load()
    pts = np.ascontiguousarray(np.asarray(points, dtype=np.float32).reshape(-1, 3))
    P = pts.shape[0]
    q = None if queries is None else np.ascontiguousarray(np.asarray(queries, dtype=np.int32))
    n = P if q is None else q.size
    out = np.empty(n, np.float32)
    best = np.empty((n, 3), np.float32) if return_best else None
    if n:
        _lib.gof_oracle_knn_mean_dist(P, pts.ctypes.data, n, None if q is None else q.ctypes.data, out.ctypes.data,
                                      None if best is None else best.ctypes.data)
    return (out, best) if return_best else out
