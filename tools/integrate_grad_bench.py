"""Cost of the opacity-field query's backward (DESIGN.md 4.11, 4.13): one view of a C5-sized scene (3 M Gaussians, 1920x1080)
queried at N points sampled around the Gaussians' centres.  Times, with CUDA events around single calls after warm-up: the plain
forward (`_C.integrate_gaussians_to_points`), the forward that keeps its state (`integrate_gaussians_to_points_state`) and the
backward (`integrate_gaussians_to_points_backward`) of an alpha loss, of a colour loss and of both, alternating; medians and
spreads, plus the per-kernel split of the library's event brackets (integrate vs integrate_bwd / integrate_bwd_color +
preprocess_bwd).  Checks that the point gradients of two backward calls are bit-identical.

  python tools/integrate_grad_bench.py [--config C5] [--view 5] [--points 2000000] [--reps 20]

Prints one line per timing and a JSON summary with the card name and its power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "gaussian-opacity-fields_b200"), os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import gof_synth  # noqa: E402


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else "unknown"
    except Exception:   # noqa: BLE001
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C5")
    ap.add_argument("--view", type=int, default=5)
    ap.add_argument("--points", type=int, default=2_000_000)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("integrate_grad_bench needs a GPU")
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda")
    cam, gs = gof_synth.make_scene(a.config, view=a.view)
    P = gs["means3D"].shape[0]
    rng = np.random.default_rng(1)
    ids = rng.integers(0, P, a.points)
    pts = (gs["means3D"].numpy()[ids] + rng.uniform(-0.01, 0.01, (a.points, 3))).astype(np.float32)
    pts = torch.from_numpy(pts).to(dev)
    e = torch.Tensor([])
    H, W = cam.image_height, cam.image_width
    g = {k: gs[k].to(dev) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    ia = (torch.zeros(3, device=dev), pts, g["means3D"], e, g["opacities"], g["scales"], g["rotations"], 1.0, e, e,
          cam.world_view_transform.to(dev), cam.full_proj_transform.to(dev), cam.tanfovx, cam.tanfovy, 0.0,
          torch.zeros((H, W, 2), device=dev), H, W, g["shs"], gs["sh_degree"], cam.camera_center.to(dev), False, False)
    dL = torch.randn(a.points, generator=torch.Generator().manual_seed(2)).to(dev)
    dC = torch.randn(a.points, 3, generator=torch.Generator().manual_seed(3)).to(dev)
    losses = dict(backward=(dL, None), backward_color=(None, dC), backward_both=(dL, dC))

    def bwd(state, mode="backward"):
        R, _c, _a, _ci, radii, geom, binning, img, pt, pbin = state
        (bg, p3, m3, col, op, sc, rot, sm, cov, v2g, vm, pm, tfx, tfy, ks, sub, H_, W_, sh, deg, cp, _pf, dbg) = ia
        da, dc = losses[mode]
        return _C.integrate_gaussians_to_points_backward(bg, p3, m3, radii, col, sc, rot, sm, cov, v2g, vm, pm, tfx, tfy, ks, sub, H_,
                                                         W_, sh, deg, cp, da, R, geom, binning, img, pt, pbin, dbg, dL_dcolor=dc)

    def timed(fn):
        s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        out = fn()
        t.record()
        torch.cuda.synchronize()
        return s.elapsed_time(t), out

    state = _C.integrate_gaussians_to_points_state(*ia)
    for _ in range(3):
        _C.integrate_gaussians_to_points(*ia)
        state = _C.integrate_gaussians_to_points_state(*ia)
        for mode in losses:
            bwd(state, mode)
    torch.cuda.synchronize()
    t = dict(forward=[], forward_state=[], backward=[], backward_color=[], backward_both=[])
    first = None
    for _ in range(a.reps):
        t["forward"].append(timed(lambda: _C.integrate_gaussians_to_points(*ia))[0])
        ms, state = timed(lambda: _C.integrate_gaussians_to_points_state(*ia))
        t["forward_state"].append(ms)
        for mode in losses:   # the backward reads the forward state and rewrites only its own scratch: one state serves all three
            ms, g_ = timed(lambda: bwd(state, mode))
            t[mode].append(ms)
            if mode == "backward_color":
                assert not bool(g_[0].any()), "a colour loss moved the points"
            elif first is None:
                first = g_[0].clone()
            else:
                assert torch.equal(first, g_[0]), "point gradients of two backward calls differ"
    _C.profile_reset()
    _C.profile_enable(True)
    state = _C.integrate_gaussians_to_points_state(*ia)
    for mode in losses:   # one bracketed call of each kernel
        bwd(state, mode)
    torch.cuda.synchronize()
    rep = _C.profile_report()
    _C.profile_enable(False)
    summary = dict(config=a.config, view=a.view, P=P, points=a.points, projected=int((state[2] < 1).sum()), card=_card())
    for k, v in t.items():
        v = np.array(v)
        summary[f"{k}_ms_median"] = round(float(np.median(v)), 3)
        summary[f"{k}_ms_spread"] = [round(float(v.min()), 3), round(float(v.max()), 3)]
        print(f"{k:14s} median {np.median(v):8.3f} ms  min {v.min():8.3f}  max {v.max():8.3f}")
    for k in ("integrate", "integrate_bwd", "integrate_bwd_color", "preprocess_bwd", "preprocess_points", "preprocess_fwd"):
        if k in rep:
            summary[f"kernel_{k}_ms"] = round(rep[k][1] / rep[k][0], 3)
            print(f"kernel {k:20s} {rep[k][1] / rep[k][0]:8.3f} ms  ({rep[k][0]} calls)")
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
