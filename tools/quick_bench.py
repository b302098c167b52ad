#!/usr/bin/env python
"""Developer timing (GPU box): fwd / bwd of ours and of the live reference extension, CUDA events."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _util  # noqa: E402
import gof_synth  # noqa: E402
from diff_gaussian_rasterization import _C as ours  # noqa: E402


def time_it(fn, n_warm=3, n=10):
    for _ in range(n_warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ref = _util.load_ref()
    dev = torch.device("cuda")
    names = sys.argv[1:] or ["C2", "C3"]
    out = {}
    for name in names:
        cam, gs = gof_synth.make_scene(name, view=1)
        fa = _util.fwd_args(cam, gs, dev)
        H, W = cam.image_height, cam.image_width
        grad = torch.randn(9, H, W, device=dev)
        res = {}
        for label, mod in (("ours", ours), ("ref", ref)):
            if mod is None:
                continue
            st = {}
            def fwd():
                st["o"] = mod.rasterize_gaussians(*fa)
            t_f = time_it(fwd)
            R, color, radii, geom, binning, img = st["o"]
            ba = _util.bwd_args(fa, radii, geom, R, binning, img, grad)
            t_b = time_it(lambda: mod.rasterize_gaussians_backward(*ba))
            res[label] = {"fwd_ms": t_f, "bwd_ms": t_b, "R": R, "visible": int((radii > 0).sum())}
            if label == "ours":
                ours.profile_reset(); ours.profile_enable(True)
                for _ in range(3):
                    o = mod.rasterize_gaussians(*fa)
                    mod.rasterize_gaussians_backward(*_util.bwd_args(fa, o[2], o[3], o[0], o[4], o[5], grad))
                torch.cuda.synchronize(); ours.profile_enable(False)
                res[label]["kernels_ms"] = {k: round(v[1] / 3, 4) for k, v in sorted(ours.profile_report().items(), key=lambda kv: -kv[1][1])}
        out[name] = res
        print(name, json.dumps(res), flush=True)
    os.makedirs(os.path.join(ROOT, "tool_out"), exist_ok=True)
    with open(os.path.join(ROOT, "tool_out", "quick_bench.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
