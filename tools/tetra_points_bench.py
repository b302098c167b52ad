"""Times gof_extract.get_tetra_points (DESIGN §4.8) at C5 (3 M Gaussians, 64 views at 1920x1080) and, at --common Gaussians
(default 500 k, 64 views), against the reference's own GaussianModel.get_tetra_points run from its staged source on the same
inputs.  CUDA-event medians over --reps calls after one warm-up call; peak memory is the growth of
torch.cuda.max_memory_allocated over what the inputs hold.  Prints one JSON line with the card's name and power limit.

    python tools/tetra_points_bench.py [--reps 10] [--common 500000]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "gaussian-opacity-fields_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return ""


def timed(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
        del out
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    kept = int(out[0].shape[0])
    del out
    return sorted(times)[len(times) // 2], peak, kept


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--common", type=int, default=500_000)
    a = ap.parse_args()
    import torch
    import _tetra_scenes as ts
    import gof_extract
    import gof_synth
    dev = torch.device("cuda:0")
    res = {"gpu": gpu_info() or torch.cuda.get_device_name()}
    cfg = gof_synth.CONFIGS["C5"]
    for tag, P in (("c5", cfg["P"]), ("common", a.common)):
        xyz, s, r = (t.to(dev) for t in ts.gaussians(P, cfg["seed"]))
        views = ts.ring_views(cfg["n_views"], cfg["width"], cfg["height"], device=dev)
        ms, peak, kept = timed(lambda: gof_extract.get_tetra_points(xyz, s, r, views), a.reps)
        row = {"P": P, "views": len(views), "points_kept": kept, "ours_ms": round(ms, 3), "ours_peak_bytes": peak,
               "ours_peak_bytes_per_gaussian": round(peak / P, 1)}
        if tag == "common":
            if ts.ref_tetra_points(xyz[:8], s[:8], r[:8], views[:1]) is None:
                row["reference"] = "not measured: the reference's source is not staged"
            else:
                rms, rpeak, rkept = timed(lambda: ts.ref_tetra_points(xyz, s, r, views)[:2], a.reps)
                row.update({"reference_ms": round(rms, 3), "reference_peak_bytes": rpeak, "reference_points_kept": rkept})
        res[tag] = row
        del xyz, s, r
        torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
