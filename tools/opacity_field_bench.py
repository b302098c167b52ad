"""Cost of the multi-view opacity field with gradients (DESIGN.md 4.12): a C5-sized scene (3 M Gaussians, 1920x1080) seen from
`--views` cameras of the ring, queried at N points sampled around the Gaussians' centres.

Times, with CUDA events after warm-up, alternating: the plain multi-view query (`evaluate_alpha` over
`GaussianRasterizer.integrate`, one call per view), the forward of `gof_extract.opacity_field` (one running-minimum `gof_integrate` per
view), the same forward with `return_color=True` (one with `color_min` per view, DESIGN.md 4.13) and the backward.  Reports ms per view for both forwards, the backward's ms in all and per winning view, and the
per-kernel split of the library's event brackets.  Then the peak `torch.cuda.max_memory_allocated` growth over forward and
backward of `opacity_field` against the naive composition (per-view `integrate_gaussians` kept by autograd, torch.min).  Checks
that the field equals evaluate_alpha bit for bit and that the point gradients of two backward calls are bit-identical.

  python tools/opacity_field_bench.py [--config C5] [--views 8] [--points 2000000] [--reps 3]

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

import gof_extract  # noqa: E402
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
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--points", type=int, default=2_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-memory", action="store_true", help="skip the peak-memory comparison")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("opacity_field_bench needs a GPU")
    from diff_gaussian_rasterization import _C, GaussianRasterizer, integrate_gaussians
    dev = torch.device("cuda")
    cam0, gs = gof_synth.make_scene(a.config, view=0)
    W, H = cam0.image_width, cam0.image_height
    n_ring = gof_synth.CONFIGS[a.config]["n_views"] if isinstance(a.config, str) and a.config in gof_synth.CONFIGS else 64
    cams = [gof_synth.make_camera(W, H, view=(v * n_ring) // a.views, n_views=n_ring) for v in range(a.views)]
    settings = {id(c): gof_synth.raster_settings(c, gs["sh_degree"], dev) for c in cams}
    sf = lambda c: settings[id(c)]   # noqa: E731
    P = gs["means3D"].shape[0]
    rng = np.random.default_rng(1)
    ids = rng.integers(0, P, a.points)
    pts = torch.from_numpy((gs["means3D"].numpy()[ids] + rng.uniform(-0.01, 0.01, (a.points, 3))).astype(np.float32)).to(dev)
    g = {k: gs[k].to(dev) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    dL = torch.randn(a.points, generator=torch.Generator().manual_seed(2)).to(dev)

    def plain():
        fn = gof_extract.make_integrate_fn(g["means3D"], g["opacities"], g["scales"], g["rotations"], g["shs"], gs["sh_degree"], sf)
        return gof_extract.evaluate_alpha(pts, cams, fn)

    def leaves():
        q = {k: v.clone().requires_grad_(k != "shs") for k, v in g.items()}
        return pts.clone().requires_grad_(True), q

    def field(p, q, return_color=False):
        return gof_extract.opacity_field(p, q["means3D"], q["opacities"], q["scales"], q["rotations"], q["shs"], gs["sh_degree"], cams, sf,
                                         return_color=return_color)

    def timed(fn):
        s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        out = fn()
        t.record()
        torch.cuda.synchronize()
        return s.elapsed_time(t), out

    for _ in range(2):
        plain()
        p, q = leaves()
        (field(p, q) * dL).sum().backward()
        with torch.no_grad():
            field(p, q, True)
    torch.cuda.synchronize()
    with torch.no_grad():
        fn = gof_extract.make_integrate_fn(g["means3D"], g["opacities"], g["scales"], g["rotations"], g["shs"], gs["sh_degree"], sf)
        ref_color = gof_extract.evaluate_alpha(pts, cams, fn, return_color=True)[1]
    t = dict(plain=[], forward=[], forward_color=[], backward=[])
    first = None
    for _ in range(a.reps):
        ms, ref = timed(plain)
        t["plain"].append(ms)
        p, q = leaves()
        ms, alpha = timed(lambda: field(p, q))
        t["forward"].append(ms)
        assert torch.equal(alpha.detach(), ref), "opacity_field differs from evaluate_alpha"
        with torch.no_grad():
            ms, (alpha_c, color) = timed(lambda: field(p, q, True))
        t["forward_color"].append(ms)
        assert torch.equal(alpha_c, ref) and torch.equal(color, ref_color), "return_color differs from evaluate_alpha"
        del alpha_c, color
        ms, _ = timed(lambda: (alpha * dL).sum().backward())
        t["backward"].append(ms)
        if first is None:
            first = p.grad.clone()
        else:
            assert torch.equal(first, p.grad), "point gradients of two backward calls differ"
    _C.profile_reset()
    _C.profile_enable(True)
    plain()
    p, q = leaves()
    (field(p, q) * dL).sum().backward()
    with torch.no_grad():
        field(p, q, True)
    torch.cuda.synchronize()
    rep = _C.profile_report()
    _C.profile_enable(False)
    with torch.no_grad():
        won = int((ref > 0).sum())
        alpha_int = [GaussianRasterizer(sf(c)).integrate(pts, g["means3D"], torch.zeros_like(g["means3D"]), g["opacities"],
                                                         shs=g["shs"], scales=g["scales"], rotations=g["rotations"])[1] for c in cams]
        winners = len(torch.unique(torch.argmin(torch.stack(alpha_int), 0)[ref > 0]))
        del alpha_int
    summary = dict(config=a.config, P=P, points=a.points, views=a.views, points_won=won, winning_views=winners, card=_card())
    for k, v in t.items():
        v = np.array(v)
        summary[f"{k}_ms_median"] = round(float(np.median(v)), 3)
        summary[f"{k}_ms_spread"] = [round(float(v.min()), 3), round(float(v.max()), 3)]
        print(f"{k:10s} median {np.median(v):9.3f} ms  min {v.min():9.3f}  max {v.max():9.3f}")
    summary["plain_ms_per_view"] = round(summary["plain_ms_median"] / a.views, 3)
    summary["forward_ms_per_view"] = round(summary["forward_ms_median"] / a.views, 3)
    summary["forward_color_ms_per_view"] = round(summary["forward_color_ms_median"] / a.views, 3)
    summary["backward_ms_per_winning_view"] = round(summary["backward_ms_median"] / max(winners, 1), 3)
    print(f"per view: plain {summary['plain_ms_per_view']} ms, opacity_field forward {summary['forward_ms_per_view']} ms, with "
          f"return_color {summary['forward_color_ms_per_view']} ms; backward "
          f"{summary['backward_ms_per_winning_view']} ms per winning view ({winners} of {a.views})")
    for k in ("integrate", "integrate_min", "integrate_min_color", "integrate_bwd", "preprocess_bwd", "preprocess_points", "preprocess_fwd"):
        if k in rep:
            summary[f"kernel_{k}_ms"] = round(rep[k][1] / rep[k][0], 3)
            print(f"kernel {k:18s} {rep[k][1] / rep[k][0]:8.3f} ms  ({rep[k][0]} launches)")

    if not a.no_memory:
        def peak(fn):
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            fn()
            torch.cuda.synchronize()
            return (torch.cuda.max_memory_allocated() - base) / 2 ** 20

        def naive():
            p, q = leaves()
            stack = torch.stack([integrate_gaussians(p, q["means3D"], torch.zeros_like(q["means3D"]), q["opacities"], q["shs"], None,
                                                     q["scales"], q["rotations"], None, None, sf(c))[1] for c in cams])
            (1 - stack.min(0).values).mul(dL).sum().backward()

        def ours():
            p, q = leaves()
            (field(p, q) * dL).sum().backward()

        summary["peak_mib_opacity_field"] = round(peak(ours), 1)
        summary["peak_mib_naive"] = round(peak(naive), 1)
        print(f"peak memory growth over forward + backward ({a.views} views): opacity_field {summary['peak_mib_opacity_field']} MiB, "
              f"naive composition {summary['peak_mib_naive']} MiB")
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
