"""Regenerates tests/golden/densify_*.npz and tests/golden/extract_ref.npz: the reference's own Python (GaussianModel's
densification methods, extract_mesh.evaluage_alpha over gaussian_renderer.integrate), staged unmodified by
baseline/stage_ref.sh, on a CUDA device -- the latter on the reference's compiled rasterizer (oracle/_ref).

  python tests/golden/make_golden_ref_python.py [OUT_DIR]      (default: tests/golden)"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle")]
import _util  # noqa: E402,F401  (puts the package on sys.path)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import _refpy  # noqa: E402
import test_gpu_densify  # noqa: E402
import test_gpu_extract  # noqa: E402


def densify_methods():
    """The reference's densification methods with torch.normal replaced by a queue of given samples."""
    gu = _refpy.ref_utils("general_utils")
    assert gu is not None and _refpy.staged("text", "gaussian_model.py") is not None, "run baseline/stage_ref.sh first"
    feed = {"queue": []}

    class TorchProxy:
        def __getattr__(self, k):
            return getattr(torch, k)

        @staticmethod
        def normal(mean, std):
            return std * feed["queue"].pop(0)

    glb = {"torch": TorchProxy(), "nn": torch.nn, "build_rotation": gu.build_rotation}
    ns = {}
    for m in test_gpu_densify.METHODS:
        exec(_refpy.ref_method_source("gaussian_model.py", "GaussianModel", m), glb, ns)
    return ns, feed


def extract_eval():
    pkg = _refpy.ref_rasterizer_package()
    assert pkg is not None and _refpy.staged("text", "extract_mesh.py") is not None, "needs oracle/_ref and baseline/stage_ref.sh"
    gr = _refpy.ref_gaussian_renderer(pkg, "gof_gr_on_ref_extract")
    glb = {"torch": torch, "integrate": gr.integrate, "tqdm": lambda it, **kw: it}
    return _refpy.ref_function("extract_mesh.py", "evaluage_alpha", glb)


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    os.makedirs(out_dir, exist_ok=True)
    dev = torch.device("cuda")
    methods, feed = densify_methods()
    recs = {f"densify_{P}": test_gpu_densify.record(P, ms, dev, methods, feed) for P, ms in test_gpu_densify.CASES}
    recs["extract_ref"] = test_gpu_extract.record(extract_eval())
    for name, rec in recs.items():
        path = os.path.join(out_dir, f"{name}.npz")
        np.savez_compressed(path, **rec)
        print(f"[make_golden_ref_python] {path}: {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
