"""Cost of the opacity field's point gradient in the cached query's own pass (DESIGN.md 4.14) at C5's shape: 3 M Gaussians seen
from `--views` cached 1920x1080 cameras of the ring, queried at N points sampled around the Gaussians' centres.

Times, with CUDA events after a warm-up, alternating, `--reps` times each:
  * cached_alpha:   one evaluate_alpha pass over a CachedIntegrator (one gof_integrate_cached per view);
  * field_gradient: one field_gradient pass over the same cache (one gof_integrate_cached with grad_min per view);
  * autograd_fwd / autograd_bwd: opacity_field(points, ...) and its .sum().backward() for the points alone (the uncached
    query per view, then the Gaussian side rebuilt for every winning view).
Checks that field_gradient's alpha equals evaluate_alpha's and its gradient equals the autograd point gradient, bit for bit.

  python tools/field_gradient_bench.py [--config C5] [--views 64] [--points 2000000] [--reps 3]

Prints one JSON line with the medians, their spread, ms per view, and the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "gaussian-opacity-fields_b200")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import gof_extract  # noqa: E402
import gof_synth  # noqa: E402


def _card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=30).stdout.strip().splitlines()
    return out[torch.cuda.current_device()] if out else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C5")
    ap.add_argument("--views", type=int, default=64)
    ap.add_argument("--points", type=int, default=2_000_000)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("field_gradient_bench needs a GPU")
    dev = torch.device("cuda")
    cam0, gs = gof_synth.make_scene(a.config, view=0)
    W, H = cam0.image_width, cam0.image_height
    n_ring = gof_synth.CONFIGS[a.config]["n_views"] if a.config in gof_synth.CONFIGS else 64
    cams = [gof_synth.make_camera(W, H, view=(v * n_ring) // a.views, n_views=n_ring) for v in range(a.views)]
    settings = {id(c): gof_synth.raster_settings(c, gs["sh_degree"], dev) for c in cams}
    sf = lambda c: settings[id(c)]   # noqa: E731
    P = gs["means3D"].shape[0]
    rng = np.random.default_rng(1)
    ids = rng.integers(0, P, a.points)
    pts = torch.from_numpy((gs["means3D"].numpy()[ids] + rng.uniform(-0.01, 0.01, (a.points, 3))).astype(np.float32)).to(dev)
    g = {k: gs[k].to(dev) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    ci = gof_extract.CachedIntegrator(g["means3D"], g["opacities"], g["scales"], g["rotations"], g["shs"], gs["sh_degree"], sf)
    for c in cams:
        ci.prepare(c)

    def timed(fn):
        s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        s.record()
        out = fn()
        t.record()
        torch.cuda.synchronize()
        return s.elapsed_time(t), out

    def autograd_fwd():
        p = pts.clone().requires_grad_(True)
        return p, gof_extract.opacity_field(p, g["means3D"], g["opacities"], g["scales"], g["rotations"], g["shs"], gs["sh_degree"],
                                            cams, sf)

    cached = lambda: gof_extract.evaluate_alpha(pts, cams, ci)          # noqa: E731
    gradient = lambda: gof_extract.field_gradient(pts, cams, ci)        # noqa: E731
    cached()
    gradient()
    p, f = autograd_fwd()
    f.sum().backward()
    del p, f
    t = dict(cached_alpha=[], field_gradient=[], autograd_fwd=[], autograd_bwd=[])
    for _ in range(a.reps):
        ms, alpha0 = timed(cached)
        t["cached_alpha"].append(ms)
        ms, (alpha, grad) = timed(gradient)
        t["field_gradient"].append(ms)
        ms, (p, f) = timed(autograd_fwd)
        t["autograd_fwd"].append(ms)
        ms, _ = timed(lambda: f.sum().backward())
        t["autograd_bwd"].append(ms)
        assert torch.equal(alpha, alpha0), "field_gradient's alpha differs from evaluate_alpha"
        assert torch.equal(grad, p.grad), "field_gradient's gradient differs from opacity_field's backward"
        won = int((grad != 0).any(dim=1).sum())
        del alpha0, alpha, grad, p, f
    out = dict(config=a.config, P=P, width=W, height=H, views=a.views, points=a.points, points_with_gradient=won,
               cached_bytes=ci.cached_bytes, card=_card())
    for k, v in t.items():
        v = np.array(v)
        out[f"{k}_ms_median"] = round(float(np.median(v)), 3)
        out[f"{k}_ms_spread"] = [round(float(v.min()), 3), round(float(v.max()), 3)]
        out[f"{k}_ms_per_view"] = round(float(np.median(v)) / a.views, 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
