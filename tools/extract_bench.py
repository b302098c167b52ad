#!/usr/bin/env python
"""Developer timing (GPU box) of the extraction rows: GaussianRasterizer.integrate (ours vs the live reference
extension, CUDA events, median of n) and marching tetrahedra (ours vs the numpy oracle on the host)."""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import _util  # noqa: E402
import gof_synth  # noqa: E402
import gof_tetmesh  # noqa: E402
from diff_gaussian_rasterization import _C as ours  # noqa: E402
from quick_bench import time_it  # noqa: E402


def main():
    ref = _util.load_ref()
    dev = torch.device("cuda")
    out = {}
    for name, n_pts in (("C2", 900_000), ("C3", 2_000_000), ("C3", 9_000_000)):
        cam, gs = gof_synth.make_scene(name, view=3)
        P = gs["means3D"].shape[0]
        g = torch.Generator().manual_seed(4)
        # extract_mesh.py evaluates the 9 cell vertices of every Gaussian: points hug the Gaussians
        idx = torch.randint(0, P, (n_pts,), generator=g)
        pts = (gs["means3D"][idx] + gs["scales"][idx] * 3.0 * (torch.rand(n_pts, 3, generator=g) * 2 - 1)).contiguous().to(dev)
        fa = _util.fwd_args(cam, gs, dev)
        ia = (fa[0], pts) + tuple(fa[1:])
        res = {"points": n_pts, "P": P}
        for label, mod in (("ours", ours), ("ref", ref)):
            if mod is None:
                continue
            res[label + "_ms"] = time_it(lambda: mod.integrate_gaussians_to_points(*ia), n_warm=2, n=5)
        if "ref_ms" in res:
            res["speedup"] = res["ref_ms"] / res["ours_ms"]
        ours.profile_reset(); ours.profile_enable(True)
        ours.integrate_gaussians_to_points(*ia); torch.cuda.synchronize(); ours.profile_enable(False)
        res["kernels_ms"] = {k: round(v[1], 4) for k, v in sorted(ours.profile_report().items(), key=lambda kv: -kv[1][1])}
        out[f"integrate_{name}_{n_pts}"] = res
        print(name, n_pts, json.dumps(res), flush=True)
        del pts

    import tetmesh_oracle
    rng = np.random.default_rng(5)
    for V, T in ((400_000, 2_600_000), (4_000_000, 26_000_000)):
        v = rng.uniform(-1, 1, size=(V, 3)).astype(np.float32)
        a = rng.integers(0, V, size=T)
        tets = np.stack([a, (a + rng.integers(1, 50, size=T)) % V, (a + rng.integers(50, 400, size=T)) % V,
                         (a + rng.integers(400, 3000, size=T)) % V], axis=1).astype(np.int64)
        sdf = (0.8 - np.linalg.norm(v, axis=1) + 0.05 * rng.standard_normal(V)).astype(np.float32)
        sc = rng.uniform(0.01, 0.1, size=(V, 1)).astype(np.float32)
        t = lambda x: torch.from_numpy(x).to(dev)
        tv, tt, ts_, tsc = t(v), t(tets), t(sdf), t(sc)
        ms = time_it(lambda: gof_tetmesh._unbatched_marching_tetrahedra(tv, tt, ts_, tsc), n_warm=2, n=5)
        res = {"verts": V, "tets": T, "ours_ms": ms}
        if T <= 3_000_000:
            t0 = time.perf_counter(); tetmesh_oracle.marching_tetrahedra(v, tets, sdf, sc); res["numpy_oracle_ms"] = (time.perf_counter() - t0) * 1e3
        (_, _), _, faces, _ = gof_tetmesh._unbatched_marching_tetrahedra(tv, tt, ts_, tsc)
        res["faces"] = int(faces.shape[0])
        out[f"tetmesh_{T}"] = res
        print("tetmesh", json.dumps(res), flush=True)
    with open(os.path.join(ROOT, "tool_out", "extract_bench.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
