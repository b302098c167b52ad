"""DTU-sized TSDF fusion benchmark: 1 M surface Gaussians on a radius-1 sphere, 49 views at 1600x1200, voxel 0.002.

    python tools/tsdf_bench.py [--gaussians 1000000] [--views 49] [--width 1600] [--height 1200] [--voxel 0.002]

Prints one JSON line: per-view milliseconds of render, touch + activate and integrate (median over the views, CUDA events),
extraction milliseconds, blocks, voxel updates, V and F, the integrate kernel's bytes / time as a share of HBM bandwidth,
peak memory, and the card's name and power limit read in the same run.  There is no reference arm: the reference path
needs Open3D, which this environment does not have.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "gaussian-opacity-fields_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM5 80 GB HBM3


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
    ap.add_argument("--views", type=int, default=49)
    ap.add_argument("--width", type=int, default=1600)
    ap.add_argument("--height", type=int, default=1200)
    ap.add_argument("--voxel", type=float, default=0.002)
    args = ap.parse_args()

    import gof_synth
    import gof_tsdf
    from diff_gaussian_rasterization import _C

    dev = torch.device("cuda:0")
    name, power = _card()
    gs = gof_synth.make_surface_gaussians(args.gaussians, seed=0)
    g = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in gs.items()}
    views = gof_synth.make_surface_views(args.width, args.height, args.views)
    render = gof_tsdf.make_render_fn(g["means3D"], g["opacities"], g["scales"], g["rotations"], g["shs"], g["sh_degree"],
                                      lambda v: gof_synth.raster_settings(v, g["sh_degree"], dev))
    render(views[0])                                  # warm-up: library, pools, allocator
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()

    vol = gof_tsdf.TSDFVolume(voxel_size=args.voxel, device=dev)
    ev = lambda: torch.cuda.Event(enable_timing=True)   # noqa: E731
    t_render, t_touch, t_int, int_kernel_ms = [], [], [], 0.0
    _C.profile_reset()
    for v in views:
        e = [ev() for _ in range(4)]
        e[0].record()
        img = render(v)
        depth = img[6].clone()
        depth[img[7] < 0.5] = 0
        color = img[:3].contiguous()
        e[1].record()
        fx, fy, cx, cy = gof_tsdf.intrinsics_from_view(v)
        cam = vol._camera(args.height, args.width, fx, fy, cx, cy, gof_tsdf.extrinsic_from_view(v))
        par = vol._params(6.0)
        keys = vol._touch(depth, cam, par)
        slots = vol._activate(keys) if keys.numel() else None
        e[2].record()
        if keys.numel():
            _C.profile_enable(True)
            _C._check(gof_tsdf._lib.gof_tsdf_integrate(
                ctypes.byref(par), ctypes.byref(cam), depth.data_ptr(), color.data_ptr(), int(keys.numel()),
                keys.data_ptr(), slots.data_ptr(), vol.pool.data_ptr(), vol.num_updates.data_ptr(), _C._stream()))
            _C.profile_enable(False)
        e[3].record()
        torch.cuda.synchronize()
        t_render.append(e[0].elapsed_time(e[1]))
        t_touch.append(e[1].elapsed_time(e[2]))
        t_int.append(e[2].elapsed_time(e[3]))
    rep = _C.profile_report()
    int_kernel_ms = rep.get("tsdf_integrate", (0, 0.0))[1]
    updates = int(vol.num_updates.item())
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mesh = vol.extract_triangle_mesh(3.0)
    torch.cuda.synchronize()
    t_ext = 1e3 * (time.perf_counter() - t0)
    # integrate traffic: every updated voxel reads and writes its five floats (tsdf, weight, rgb); plus one read of each view's
    # depth and colour images (gathers that stay in L2) -- a lower bound on the bytes moved
    img_bytes = args.views * args.width * args.height * 4 * 4
    int_bytes = updates * 5 * 4 * 2 + img_bytes
    med = lambda x: float(np.median(x))   # noqa: E731
    print(json.dumps({
        "workload": f"tsdf_fusion {args.gaussians} surface Gaussians, radius-1 sphere, {args.views} views {args.width}x{args.height}, "
                    f"voxel {args.voxel}, block 16, trunc 8 voxels, depth_max 6, weight_threshold 3",
        "reference_arm": None,
        "reference_note": "no reference arm: the reference path (extract_mesh_tsdf.py) needs Open3D, which is not installed",
        "render_ms_per_view": round(med(t_render), 3),
        "touch_activate_ms_per_view": round(med(t_touch), 3),
        "integrate_ms_per_view": round(med(t_int), 3),
        "integrate_kernel_ms_total": round(int_kernel_ms, 3),
        "extract_ms": round(t_ext, 3),
        "blocks": vol.num_blocks,
        "voxel_updates": updates,
        "vertices": int(mesh["vertices"].shape[0]),
        "faces": int(mesh["faces"].shape[0]),
        "integrate_bytes": int_bytes,
        "integrate_hbm_share": round(int_bytes / (int_kernel_ms * 1e-3) / HBM_BYTES_PER_S, 4) if int_kernel_ms else None,
        "peak_memory_gb": round(torch.cuda.max_memory_allocated() / 1e9, 3),
        "gpu": name,
        "power_limit_w": power,
    }))


if __name__ == "__main__":
    main()
