#!/usr/bin/env python
"""Generates the golden fixtures under tests/golden/ by running the UNMODIFIED reference extension
(oracle/_ref/gof_ref_C*.so, built by oracle/build_ref.sh from /root/reference) on a CUDA device.

The reference ships no golden vectors or tests for this path (SURVEY.md section 4), so these fixtures --
inputs, every reachable forward intermediate, outputs and gradients of the reference itself -- are what
pins both the CPU oracle (tests/test_oracle_golden.py, no GPU needed) and the CUDA path
(tests/test_gpu_golden.py).

Run on the GPU box:  python tests/golden/make_golden.py   (writes gpurun_out/golden/*.npz; copy them to
tests/golden/).  Each fixture also records the reference's own run-to-run gradient noise (its float atomics
are unordered), which is the floor for gradient comparisons.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _util  # noqa: E402
import gof_synth  # noqa: E402

FIXTURES = {
    # name: (P, W, H, seed, view, sigma_px, sh_degree, kernel_size, scale_modifier, bg, colors_precomp, radius)
    "f0_sh3": dict(P=1000, W=88, H=60, seed=11, view=3, sigma_px=2.0, sh_degree=3, kernel_size=0.0, scale_modifier=1.0, bg=(0, 0, 0)),
    "f1_sh1_mip_bg": dict(P=1000, W=96, H=64, seed=12, view=17, sigma_px=1.5, sh_degree=1, kernel_size=0.1, scale_modifier=0.8, bg=(1, 1, 1)),
    "f2_precomp_big": dict(P=600, W=64, H=64, seed=13, view=40, sigma_px=14.0, sh_degree=0, kernel_size=0.0, scale_modifier=1.0, bg=(0.2, 0.4, 0.6), colors_precomp=True),
    "f3_sh0_inside": dict(P=1000, W=80, H=56, seed=14, view=9, sigma_px=3.0, sh_degree=0, kernel_size=0.0, scale_modifier=1.0, bg=(0, 0, 0), cam_radius=1.2),
}


def build_inputs(cfg):
    cam = gof_synth.make_camera(cfg["W"], cfg["H"], view=cfg["view"], radius=cfg.get("cam_radius", 4.0))
    gs = gof_synth.make_gaussians(cfg["P"], cfg["seed"], cam.focal_x, sh_degree=cfg["sh_degree"], sigma_px=cfg["sigma_px"])
    colors = None
    if cfg.get("colors_precomp"):
        g = torch.Generator().manual_seed(cfg["seed"] + 1000)
        colors = torch.rand(cfg["P"], 3, generator=g)
    return cam, gs, colors


def main():
    ref = _util.load_ref()
    assert ref is not None, "oracle/_ref/gof_ref_C*.so missing: run oracle/build_ref.sh where /root/reference exists"
    dev = torch.device("cuda")
    outdir = os.path.join(ROOT, "gpurun_out", "golden")
    os.makedirs(outdir, exist_ok=True)
    for name, cfg in FIXTURES.items():
        cam, gs, colors = build_inputs(cfg)
        fa = _util.fwd_args(cam, gs, dev, kernel_size=cfg["kernel_size"], scale_modifier=cfg["scale_modifier"], bg=cfg["bg"],
                            colors_precomp=colors)
        P, W, H = cfg["P"], cfg["W"], cfg["H"]
        R, color, radii, geom, binning, img = ref.rasterize_gaussians(*fa)
        sg = _util.carve_ref_geom(geom, P)
        si = _util.carve_ref_image(img, W, H)
        sb = _util.carve_ref_binning(binning, R)
        g = torch.Generator().manual_seed(cfg["seed"] + 7)
        grad = torch.randn(9, H, W, generator=g)
        names = ["dmeans2D", "dcolors", "dopacity", "dmeans3D", "dcov3D", "dsh", "dscales", "drot", "dv2g"]
        runs = []
        for _ in range(3):
            gr = ref.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, grad.to(dev)))
            runs.append([t.cpu().numpy() for t in gr])
        vis = (radii > 0).cpu().numpy()
        out = dict(
            cfg=np.array(repr(cfg)),
            # inputs
            viewmatrix=cam.world_view_transform.numpy(), projmatrix=cam.full_proj_transform.numpy(),
            campos=cam.camera_center.numpy(), tanfovx=np.float32(cam.tanfovx), tanfovy=np.float32(cam.tanfovy),
            means3D=gs["means3D"].numpy(), scales=gs["scales"].numpy(), rotations=gs["rotations"].numpy(),
            opacities=gs["opacities"].numpy(), shs=gs["shs"].numpy(),
            colors_precomp=(colors.numpy() if colors is not None else np.zeros((0, 3), np.float32)),
            dL_dout=grad.numpy(),
            # reference forward
            num_rendered=np.int64(R), color=color.cpu().numpy(), radii=radii.cpu().numpy(), visible=vis,
            depths=sg["depths"].cpu().numpy(), means2D=sg["means2D"].cpu().numpy(), cov3D=sg["cov3D"].cpu().numpy(),
            view2gaussian=sg["view2gaussian"].cpu().numpy(), conic_opacity=sg["conic_opacity"].cpu().numpy(),
            rgb=sg["rgb"].cpu().numpy(), clamped=sg["clamped"].cpu().numpy(), tiles_touched=sg["tiles_touched"].cpu().numpy(),
            point_list=sb["point_list"].cpu().numpy(), ranges=si["ranges"].cpu().numpy(),
            accum_alpha=si["accum_alpha"].cpu().numpy(), n_contrib=si["n_contrib"].cpu().numpy(),
        )
        # fields of culled Gaussians are uninitialised memory in the reference: zero them for a stable file
        for k in ("depths", "means2D", "cov3D", "view2gaussian", "conic_opacity", "rgb", "clamped"):
            out[k][~vis] = 0
        for i, n in enumerate(names):
            out["grad_" + n] = runs[0][i]
            a = np.stack([r[i] for r in runs]).astype(np.float64)
            out["gradnoise_" + n] = np.float64(np.abs(a - a[0]).max() / max(np.abs(a[0]).max(), 1e-30)) if a.size else np.float64(0)
        # ---- opacity-field query (GaussianRasterizer.integrate -> _C.integrate_gaussians_to_points) ----
        gp = torch.Generator().manual_seed(cfg["seed"] + 21)
        npts = 3000
        near = gs["means3D"][torch.randint(0, P, (npts // 2,), generator=gp)] + 0.02 * torch.randn(npts // 2, 3, generator=gp)
        pts = torch.cat([near, (torch.rand(npts - npts // 2, 3, generator=gp) * 2 - 1) * 1.5]).contiguous()
        ia = (fa[0], pts.to(dev)) + tuple(fa[1:])
        iR, icolor, ialpha, icol, iradii, igeom, ibin, iimg = ref.integrate_gaussians_to_points(*ia)
        ii = _util.carve_ref_image(iimg, W, H)
        out.update(int_points=pts.numpy(), int_color=icolor.cpu().numpy(), int_alpha=ialpha.cpu().numpy(),
                   int_color_integrated=icol.cpu().numpy(), int_n_contrib=ii["n_contrib"][0].cpu().numpy(),
                   int_final_T=ii["accum_alpha"][0].cpu().numpy())
        # backward and opacity-field query arrays in companion files (tests/_golden.load merges them): each file stays < 1 MB
        parts = {"": {k: v for k, v in out.items() if not k.startswith(("grad", "int_"))},
                 "bwd_": {k: v for k, v in out.items() if k.startswith("grad")},
                 "int_": {k: v for k, v in out.items() if k.startswith("int_")}}
        for prefix, arrays in parts.items():
            if arrays:
                np.savez_compressed(os.path.join(outdir, prefix + name + ".npz"), **arrays)
        print(name, "R", R, "visible", int(vis.sum()), "max tile list", int((si["ranges"][:, 1] - si["ranges"][:, 0]).max()),
              {n: float(out["gradnoise_" + n]) for n in names})


if __name__ == "__main__":
    main()
