"""Times the Tanks and Temples evaluation (gof_tnt_eval.evaluate, DESIGN section 4.7) on a seeded TnT-sized synthetic scene:
a height-field surface sampled by --gt GT points, a noisy grid mesh of about --verts vertices (twice as many faces, so
vertices + face centroids ~ 3 x --verts source points) moved by a known similarity, a ring of --cams cameras, tau = 0.01
(Barn).  Prints the GPU name and power limit, then CUDA-event times per stage from the second of two runs, with the ICP
iteration counts.  --cpu also times the float64 oracle (oracle/tnt_eval_oracle.py, scipy cKDTree with workers=-1) on the same
inputs.

    python tools/tnt_eval_bench.py [--gt 10000000] [--verts 5000000] [--cams 300] [--cpu]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "gaussian-opacity-fields_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]


def scene(n_gt, n_verts, n_cams, seed=0):
    import _tnt_scenes as S
    import tnt_eval_oracle as O
    rng = np.random.default_rng(seed)
    g = rng.uniform(-1.0, 1.0, (n_gt, 2))
    gt = np.stack([g[:, 0], g[:, 1], S._surface(g[:, 0], g[:, 1])], 1)
    k = int(round(np.sqrt(n_verts)))
    u = np.linspace(-1.0, 1.0, k)
    X, Y = np.meshgrid(u, u, indexing="ij")
    V = np.stack([X.ravel(), Y.ravel(), S._surface(X.ravel(), Y.ravel())], 1) + rng.normal(0, 0.002, (k * k, 3))
    S_true = S._similarity(1.7, 25.0, [0.2, 0.3, 1.0], [0.4, -0.2, 0.1])
    V = O.transform(V, np.linalg.inv(S_true))
    i, j = np.meshgrid(np.arange(k - 1), np.arange(k - 1), indexing="ij")
    a, b, c, d = (i * k + j).ravel(), (i * k + j + 1).ravel(), ((i + 1) * k + j).ravel(), ((i + 1) * k + j + 1).ravel()
    F = np.concatenate([np.stack([a, c, b], 1), np.stack([b, c, d], 1)])
    traj = S._ring(n_cams, 1.2, 0.8, rng)
    traj[:, :3, 3] = O.transform(traj[:, :3, 3], np.linalg.inv(S_true))
    S_gt = S_true @ S._similarity(1.0, 0.4, [1.0, 0.0, 0.2], [0.004, -0.003, 0.002])
    poly = np.array([[-0.75, -0.75, 0.0], [0.75, -0.75, 0.0], [0.75, 0.0, 0.0], [0.0, 0.0, 0.0], [0.0, 0.75, 0.0], [-0.75, 0.75, 0.0]])
    return V, F, gt, traj, S_gt, poly


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gt", type=int, default=10_000_000)
    ap.add_argument("--verts", type=int, default=5_000_000)
    ap.add_argument("--cams", type=int, default=300)
    ap.add_argument("--cpu", action="store_true")
    a = ap.parse_args()
    import torch
    import gof_tnt_eval as G
    V, F, gt, traj, S_gt, poly = scene(a.gt, a.verts, a.cams)
    tau = G.SCENES_TAU["Barn"]
    vol = G.crop_volume("z", -0.25, 0.25, poly)
    print(json.dumps({"gpu": gpu_info() or torch.cuda.get_device_name(), "gt": gt.shape[0], "vertices": V.shape[0], "faces": F.shape[0],
                      "source_points": V.shape[0] + F.shape[0], "cameras": a.cams}), flush=True)
    for run in range(2):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        o = G.evaluate(V, F, gt, traj, traj, S_gt, vol, tau, timing=True)
        wall = time.perf_counter() - t0
    res = {"wall_s": round(wall, 3), "stage_ms": {k: round(v, 2) for k, v in o["stage_ms"].items()},
           "iterations": [o["iterations_r2"], o["iterations_r3"], o["iterations_r"]], "source_down": int(o["source_down"].shape[0]),
           "target_down": int(o["target_down"].shape[0]), "precision": o["precision"], "recall": o["recall"], "fscore": o["fscore"]}
    print(json.dumps(res), flush=True)
    if a.cpu:
        import tnt_eval_oracle as O
        t0 = time.perf_counter()
        w = O.evaluate(V, F, gt, traj, traj, S_gt, O.crop_volume(2, -0.25, 0.25, poly), tau)
        print(json.dumps({"cpu_oracle_s": round(time.perf_counter() - t0, 2),
                          "same_iterations": [w["iterations_r2"], w["iterations_r3"], w["iterations_r"]] == res["iterations"],
                          "precision": w["precision"], "recall": w["recall"]}), flush=True)


if __name__ == "__main__":
    main()
