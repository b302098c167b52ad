"""DTU evaluation timings: gof_dtu_eval.evaluate on the GPU against the CPU path of the reference's dtu_eval/eval.py (numpy
sampling, scikit-learn k-d tree queries on all cores, the Python downsample loop) on one DTU-sized synthetic scene, with a check
that both give the same outputs.

  python tools/dtu_eval_bench.py [--faces 4000000] [--stl 3000000] [--density 0.2] [--skip-cpu]

The scene: a perturbed UV sphere of radius 100 mm with about --faces triangles, --stl points on the unperturbed sphere, an
ObsMask grid at 2 mm over the box, a ground plane.  Reported: per-stage CUDA-event times of `evaluate` (second of two runs),
its wall time including the host permutation and the copies, the number of downsample rounds, the CPU stage times, and the
card name with its power limit.  Prints one JSON line at the end."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "gaussian-opacity-fields_b200"), os.path.join(ROOT, "oracle")]

import numpy as np  # noqa: E402
import torch  # noqa: E402


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def scene(faces, n_stl, seed=0):
    rng = np.random.default_rng(seed)
    nu = int(np.sqrt(faces))
    nv = max(faces // (2 * nu), 3)
    th = np.linspace(0, np.pi, nv + 1)[1:-1]
    ph = np.linspace(0, 2 * np.pi, nu, endpoint=False)
    T, P = np.meshgrid(th, ph, indexing="ij")
    v = np.stack([np.sin(T) * np.cos(P), np.sin(T) * np.sin(P), np.cos(T)], -1).reshape(-1, 3) * 100.0
    v = v + rng.normal(0, 0.05, v.shape)
    a, b = np.meshgrid(np.arange(nv - 2), np.arange(nu), indexing="ij")
    i0, i1 = a * nu + b, a * nu + (b + 1) % nu
    j0, j1 = i0 + nu, i1 + nu
    f = np.concatenate([np.stack([i0, j0, i1], -1).reshape(-1, 3), np.stack([i1, j0, j1], -1).reshape(-1, 3)]).astype(np.int64)
    x = rng.normal(size=(n_stl, 3))
    stl = x / np.linalg.norm(x, axis=1, keepdims=True) * 100.0
    bb = np.array([[-90.0, -100.0, -80.0], [100.0, 95.0, 70.0]])
    shape = tuple(int(s) for s in np.ceil((bb[1] - bb[0]) / 2.0).astype(int) + 1)
    obs = (rng.random(shape) < 0.85).astype(np.uint8)
    return dict(data=v, faces=f, stl=stl, obs_mask=obs, bb=bb, res=np.array([[2.0]]), plane=np.array([0.05, 0.1, 1.0, 40.0]))


def cpu_path(sc, r, seed, args):
    """The reference's steps on the CPU (eval.py:54-134), sampling vectorised in numpy; returns outputs and stage seconds."""
    import sklearn.neighbors as skln
    import dtu_eval_oracle as O
    t = {}
    t0 = time.perf_counter()
    data_pcd = O.sample_mesh(sc["data"], sc["faces"], r)
    t["sample"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    data_pcd = data_pcd[np.random.default_rng(seed).permutation(data_pcd.shape[0])]
    nn_engine = skln.NearestNeighbors(n_neighbors=1, radius=r, algorithm='kd_tree', n_jobs=-1)
    nn_engine.fit(data_pcd)
    rnn_idxs = nn_engine.radius_neighbors(data_pcd, radius=r, return_distance=False)
    mask = np.ones(data_pcd.shape[0], dtype=np.bool_)
    for curr, idxs in enumerate(rnn_idxs):
        if mask[curr]:
            mask[idxs] = 0
            mask[curr] = 1
    data_down = data_pcd[mask]
    t["downsample"] = time.perf_counter() - t0
    inbound, grid_inbound, in_obs = O.masks(data_down, sc["obs_mask"], sc["bb"], sc["res"], args["patch_size"])
    data_in = data_down[inbound]
    data_in_obs = data_in[grid_inbound][in_obs]
    t0 = time.perf_counter()
    nn_engine.fit(sc["stl"])
    dist_d2s, _ = nn_engine.kneighbors(data_in_obs, n_neighbors=1, return_distance=True)
    t["data2stl"] = time.perf_counter() - t0
    stl_hom = np.concatenate([sc["stl"], np.ones_like(sc["stl"][:, :1])], -1)
    above = (sc["plane"].reshape((1, 4)) * stl_hom).sum(-1) > 0
    t0 = time.perf_counter()
    nn_engine.fit(data_in)
    dist_s2d, _ = nn_engine.kneighbors(sc["stl"][above], n_neighbors=1, return_distance=True)
    t["stl2data"] = time.perf_counter() - t0
    return dict(data_down=data_down, dist_d2s=dist_d2s, dist_s2d=dist_s2d), t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--faces", type=int, default=4_000_000)
    ap.add_argument("--stl", type=int, default=3_000_000)
    ap.add_argument("--density", type=float, default=0.2)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--skip-cpu", action="store_true")
    a = ap.parse_args()
    import gof_dtu_eval
    card = _card()
    sc = scene(a.faces, a.stl)
    args = dict(downsample_density=a.density, patch_size=60.0, max_dist=20.0, visualize_threshold=10.0)
    run = lambda: gof_dtu_eval.evaluate(sc["data"], sc["stl"], sc["obs_mask"], sc["bb"], sc["res"], sc["plane"], faces=sc["faces"],  # noqa: E731
                                        seed=a.seed, timing=True, **args)
    run()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    g = run()
    wall = time.perf_counter() - t0
    row = dict(card=card, faces=int(sc["faces"].shape[0]), vertices=int(sc["data"].shape[0]), stl=int(sc["stl"].shape[0]),
               samples=g["num_samples"], data_down=int(g["data_down"].shape[0]), rounds=g["rounds"],
               gpu_stage_ms={k: round(v, 2) for k, v in g["stage_ms"].items()}, gpu_wall_s=round(wall, 3),
               scores=[g["mean_d2s"], g["mean_s2d"], g["overall"]])
    print(f"[dtu_eval_bench] {card}: {row['samples']} points -> {row['data_down']} kept in {row['rounds']} rounds; "
          f"GPU wall {wall:.3f} s, stages {row['gpu_stage_ms']}")
    if not a.skip_cpu:
        c, t = cpu_path(sc, a.density, a.seed, args)
        row["cpu_stage_s"] = {k: round(v, 3) for k, v in t.items()}
        row["cpu_threads"] = os.cpu_count()
        row["same_outputs"] = bool(np.array_equal(c["data_down"], g["data_down"]) and np.array_equal(c["dist_d2s"], g["dist_d2s"])
                                   and np.array_equal(c["dist_s2d"], g["dist_s2d"]))
        print(f"[dtu_eval_bench] CPU ({os.cpu_count()} threads) stages {row['cpu_stage_s']} s; same outputs: {row['same_outputs']}")
    print(json.dumps(row))


if __name__ == "__main__":
    main()
