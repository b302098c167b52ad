"""Opacity-field mesh on a sparse voxel-block lattice (gof_extract.extract_level_set_grid): stage times, counts, peak memory.

    python tools/field_grid_bench.py [--gaussians 1000000] [--views 64] [--width 1920] [--height 1080] [--points 27000000]
                                     [--block 8] [--voxel 0]

1 M surface Gaussians on a radius-1 sphere seen by 64 views; the voxel size is chosen (three rounds of the block pass alone)
so that the lattice has about --points points, as many as the tetrahedra points of the C5 extraction, unless --voxel is
given.  The Gaussian side of every view is prepared once (CachedIntegrator) before the timed run.  Prints one JSON line:
seconds per stage (blocks, lattice, field on the lattice, marching cubes, bisection, colours and normals in one
field_gradient pass), the counts, peak memory (in all, and above what was allocated after the warm-up run: the cached views
and the pooled scratch buffers), and the card's name and power limit read in the same run.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "gaussian-opacity-fields_b200"))

import torch  # noqa: E402


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0])
    except Exception:   # noqa: BLE001 -- the number is informative; its absence is reported as null
        power = None
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--views", type=int, default=64)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--points", type=float, default=27e6)
    ap.add_argument("--block", type=int, default=8)
    ap.add_argument("--voxel", type=float, default=0.0)
    args = ap.parse_args()

    import gof_extract
    import gof_synth

    if not torch.cuda.is_available():
        raise SystemExit("field_grid_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    name, power = _card()
    gs = gof_synth.make_surface_gaussians(args.gaussians, seed=0)
    g = {k: (v.to(dev).contiguous() if isinstance(v, torch.Tensor) else v) for k, v in gs.items()}
    views = gof_synth.make_surface_views(args.width, args.height, args.views)
    B = args.block
    xyz, sc, rot = g["means3D"], g["scales"], g["rotations"]

    s = args.voxel
    if s <= 0:
        s = 0.004
        for _ in range(3):
            n = gof_extract.field_grid_blocks(xyz, sc, rot, views, s, B).numel() * B ** 3
            s *= math.sqrt(n / args.points)
    ci = gof_extract.CachedIntegrator(g["means3D"], g["opacities"], g["scales"], g["rotations"], g["shs"], g["sh_degree"],
                                      lambda v: gof_synth.raster_settings(v, g["sh_degree"], dev))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for v in views:
        ci.prepare(v)
    torch.cuda.synchronize()
    t_prepare = time.perf_counter() - t0
    # warm-up at a coarse lattice: the library, the scratch pools and the allocator
    gof_extract.extract_level_set_grid(xyz, sc, rot, views, ci, 4 * s, B, return_color=True, return_normals=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    tm = {}
    t0 = time.perf_counter()
    mesh = gof_extract.extract_level_set_grid(xyz, sc, rot, views, ci, s, B, return_color=True, return_normals=True, timings=tm)
    torch.cuda.synchronize()
    total = time.perf_counter() - t0
    keys = gof_extract.field_grid_blocks(xyz, sc, rot, views, s, B)
    print(json.dumps({
        "workload": f"extract_level_set_grid: {args.gaussians} surface Gaussians on a radius-1 sphere, {args.views} views "
                    f"{args.width}x{args.height}, block {B}, voxel {s:.6g}, 8 bisection steps, colours and normals",
        "voxel_size": s,
        "blocks": int(keys.numel()),
        "lattice_points": int(keys.numel()) * B ** 3,
        "vertices": int(mesh["vertices"].shape[0]),
        "faces": int(mesh["faces"].shape[0]),
        "prepare_views_s": round(t_prepare, 4),
        "stage_s": {k: round(v, 4) for k, v in tm.items()},
        "total_s": round(total, 4),
        "cached_views_gb": round(ci.cached_bytes / 1e9, 3),
        "peak_memory_gb": round(torch.cuda.max_memory_allocated() / 1e9, 3),
        "peak_above_warm_baseline_gb": round((torch.cuda.max_memory_allocated() - base) / 1e9, 3),
        "gpu": name,
        "power_limit_w": power,
    }))


if __name__ == "__main__":
    main()
