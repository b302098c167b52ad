"""Builds libgof_b200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

No torch headers, no pybind: plain `nvcc -shared`.  The .so lands next to the Python package
(gaussian-opacity-fields_b200/diff_gaussian_rasterization/libgof_b200.so), is git-ignored.
"""
import os
import subprocess
import sys
import hashlib

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT_DIR = os.path.join(HERE, "diff_gaussian_rasterization")
LIB = os.path.join(OUT_DIR, "libgof_b200.so")
SOURCES = ["api.cu", "preprocess.cu", "binning.cu", "render_fwd.cu", "render_bwd.cu", "integrate.cu", "tetmesh.cu", "tsdf.cu", "knn.cu", "dtu_eval.cu", "tnt_eval.cu", "exchange.cu", "view_loss.cu", "param_ops.cu", "filter3d.cu", "tetra_points.cu", "field_grid.cu", "densify.cu", "conv_wgrad.cu", "sh_views.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr",
]


def _digest():
    h = hashlib.sha256()
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for name in sorted(os.listdir(root)):
            if name.endswith((".cu", ".cuh", ".h")):
                with open(os.path.join(root, name), "rb") as f:
                    h.update(name.encode())
                    h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=True):
    stamp = LIB + ".stamp"
    digest = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == digest:
        return LIB
    nvcc = os.environ.get("NVCC", "nvcc")
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    procs = []
    objs = []
    for src in SOURCES:
        path = os.path.join(CSRC, src)
        if not os.path.exists(path):
            continue
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [nvcc] + NVCC_FLAGS + ["-Xptxas", "-v", "-c", path, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        log.append(f"==== {src}\n{out}")
        failed |= p.returncode != 0
    with open(os.path.join(objdir, "ptxas.log"), "w") as f:
        f.write("\n".join(log))
    if failed:
        sys.stderr.write("\n".join(log))
        raise RuntimeError("nvcc failed building libgof_b200.so")
    cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"]
    subprocess.check_call(cmd)
    with open(stamp, "w") as f:
        f.write(digest)
    if verbose:
        print(f"[gof_b200] built {LIB}")
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv)
