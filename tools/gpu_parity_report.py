#!/usr/bin/env python
"""Developer report (run on the GPU box): ours vs the live reference extension, field by field."""
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _util  # noqa: E402
import gof_synth  # noqa: E402
from diff_gaussian_rasterization import _C as ours  # noqa: E402


def bits_equal(a, b):
    return (a.view(torch.int32) == b.view(torch.int32))


def main():
    ref = _util.load_ref()
    dev = torch.device("cuda")
    report = {}
    cfgs = [("C1", 0), ("C1", 5), ("C2", 3)] + ([("C3", 1)] if "--big" in sys.argv else [])
    for name, view in cfgs:
        cam, gs = gof_synth.make_scene(name, view=view)
        fa = _util.fwd_args(cam, gs, dev)
        P, W, H = gs["means3D"].shape[0], cam.image_width, cam.image_height
        torch.cuda.synchronize(); t0 = time.time()
        Ro, co, rado, geo, bino, imo = ours.rasterize_gaussians(*fa)
        torch.cuda.synchronize(); t_ours = time.time() - t0
        so = ours.export_state(P, W, H, Ro, geo, bino, imo, rado)
        entry = {"P": P, "W": W, "H": H, "R_ours": Ro, "t_ours_first_call_s": t_ours}
        g = torch.Generator(device="cpu").manual_seed(123)
        grad = torch.randn(9, H, W, generator=g).to(dev)
        go = ours.rasterize_gaussians_backward(*_util.bwd_args(fa, rado, geo, Ro, bino, imo, grad))
        torch.cuda.synchronize()
        names = ["dmeans2D", "dcolors", "dopacity", "dmeans3D", "dcov3D", "dsh", "dscales", "drot", "dv2g"]
        entry["grad_norms_ours"] = {n: float(t.double().norm()) for n, t in zip(names, go)}
        if ref is not None:
            torch.cuda.synchronize(); t0 = time.time()
            Rr, cr, radr, ger, binr, imr = ref.rasterize_gaussians(*fa)
            torch.cuda.synchronize(); entry["t_ref_first_call_s"] = time.time() - t0
            entry["R_ref"] = Rr
            sr = _util.carve_ref_geom(ger, P)
            si = _util.carve_ref_image(imr, W, H)
            sb = _util.carve_ref_binning(binr, Rr)
            vis = radr > 0
            entry["radii_mismatch"] = int((rado != radr).sum())
            entry["visible"] = int(vis.sum())
            entry["tiles_touched_mismatch"] = int((so["tiles_touched"] != sr["tiles_touched"]).sum())
            for f in ["depths", "means2D", "conic_opacity", "rgb", "view2gaussian"]:
                a, b = so[f][vis], sr[f][vis]
                eq = bits_equal(a, b)
                entry[f + "_bit_mismatch_frac"] = float(1.0 - eq.float().mean()) if eq.numel() else 0.0
                if a.dim() == 2:
                    entry[f + "_bit_mismatch_per_col"] = [float(1.0 - eq[:, k].float().mean()) for k in range(a.shape[1])]
                entry[f + "_relerr"] = _util.rel_err(a, b)
            entry["clamped_mismatch"] = int((so["clamped"][vis] != sr["clamped"][vis]).sum())
            if Ro == Rr:
                entry["point_list_mismatch"] = int((so["point_list"] != sb["point_list"]).sum())
            entry["ranges_mismatch"] = int((so["ranges"] != si["ranges"]).sum())
            entry["n_contrib_mismatch"] = [int((so["n_contrib"][k] != si["n_contrib"][k]).sum()) for k in range(2)]
            entry["accum_alpha_relerr"] = [_util.rel_err(so["accum_alpha"][k], si["accum_alpha"][k]) for k in range(4)]
            entry["color_relerr"] = [_util.rel_err(co[k], cr[k]) for k in range(9)]
            entry["color_bit_mismatch"] = [int((~bits_equal(co[k], cr[k])).sum()) for k in range(9)]
            gr = ref.rasterize_gaussians_backward(*_util.bwd_args(fa, radr, ger, Rr, binr, imr, grad))
            gr2 = ref.rasterize_gaussians_backward(*_util.bwd_args(fa, radr, ger, Rr, binr, imr, grad))
            torch.cuda.synchronize()
            entry["grad_relerr"] = {n: _util.rel_err(a, b) for n, a, b in zip(names, go, gr)}
            entry["grad_ref_vs_ref_relerr"] = {n: _util.rel_err(a, b) for n, a, b in zip(names, gr2, gr)}
        report[f"{name}_view{view}"] = entry
        print(name, view, json.dumps(entry)[:3000], flush=True)
    os.makedirs(os.path.join(ROOT, "tool_out"), exist_ok=True)
    with open(os.path.join(ROOT, "tool_out", "parity_report.json"), "w") as f:
        json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
