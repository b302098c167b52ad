"""Regenerates tests/golden/live_knn.npz: the unmodified reference simple-knn extension (oracle/_ref/simple_knn_ref_C*.so,
built by oracle/build_ref_knn.sh from the original project) run on a CUDA device on the point clouds of CASES.  Per case
it stores the SHA-256 of the full float32 output and the values at 4096 seeded sample positions.

  python tests/golden/make_golden_knn.py [OUT_DIR]      (default: tests/golden)"""
import glob
import hashlib
import importlib.machinery
import importlib.util
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(ROOT, "gaussian-opacity-fields_b200")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import gof_synth  # noqa: E402

# (name, kind, P, seed)
CASES = [
    ("uniform_65537", "uniform", 65537, 11),
    ("uniform_1m", "uniform", 1 << 20, 12),
    ("uniform_4m", "uniform", 1 << 22, 13),
    ("colmap_65537", "colmap", 65537, 21),
    ("colmap_1m", "colmap", 1 << 20, 22),
    ("colmap_4m", "colmap", 1 << 22, 23),
    ("lattice_262144", "lattice", 1 << 18, 31),
    ("nonfinite_65537", "nonfinite", 65537, 41),
]
SAMPLES = 4096


def load_reference():
    paths = glob.glob(os.path.join(ROOT, "oracle", "_ref", "simple_knn_ref_C*.so"))
    if not paths:
        raise RuntimeError("oracle/_ref/simple_knn_ref_C*.so missing: run oracle/build_ref_knn.sh where the original project is")
    loader = importlib.machinery.ExtensionFileLoader("simple_knn_ref_C", paths[0])
    spec = importlib.util.spec_from_file_location("simple_knn_ref_C", paths[0], loader=loader)
    mod = importlib.util.module_from_spec(spec)
    loader.exec_module(mod)
    return mod


def sample_positions(P, seed):
    return np.sort(np.random.default_rng([seed, 7]).choice(P, min(P, SAMPLES), replace=False)).astype(np.int64)


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float32).tobytes()).hexdigest()


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    os.makedirs(out_dir, exist_ok=True)
    ref = load_reference()
    dev = torch.device("cuda:0")
    rec = {}
    for name, kind, P, seed in CASES:
        pts = torch.from_numpy(gof_synth.make_point_cloud(kind, P, seed)).to(dev)
        out = ref.distCUDA2(pts)
        torch.cuda.synchronize()
        o = out.cpu().numpy()
        idx = sample_positions(P, seed)
        rec[f"{name}/spec"] = np.array([kind, str(P), str(seed)])
        rec[f"{name}/sha256"] = np.array(digest(o))
        rec[f"{name}/idx"] = idx
        rec[f"{name}/val"] = o[idx]
        print(f"[make_golden_knn] {name}: {digest(o)[:16]}  inf={int(np.isinf(o).sum())} nan={int(np.isnan(o).sum())}")
    path = os.path.join(out_dir, "live_knn.npz")
    np.savez_compressed(path, **rec)
    print(f"[make_golden_knn] wrote {path}")


if __name__ == "__main__":
    main()
