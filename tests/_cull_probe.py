"""Helper for test_gpu_culling.py: renders the scenes stored in an .npz (written ONCE by the parent test, so that both
GOF_CULL modes see bit-identical inputs -- torch's vectorised CPU exp/sigmoid may differ by an ulp between processes)
and dumps the outputs.  Usage: _cull_probe.py <inputs.npz> <outputs.npz>, GOF_CULL=0/1 in the environment."""
import sys
import numpy as np
import torch
import _integrate_scenes
import _util
import gof_synth
from diff_gaussian_rasterization import _C

CASES = [("a", dict(P=40000, width=640, height=360, seed=3), 2, 2.0, (0.3, 1.0), 4.0),
         ("b", dict(P=20000, width=320, height=200, seed=4), 9, 6.0, (0.02, 1.0), 2.0),   # needles / pancakes
         ("c", dict(P=20000, width=320, height=200, seed=5), 5, 0.7, (0.3, 1.0), 4.0)]    # sub-pixel
KEYS = ("means3D", "scales", "rotations", "opacities", "shs")
NEEDLES = "n"   # _integrate_scenes.needle_scene: Gaussians that only the corner rays of the opacity-field query meet


def _built_scenes():
    """Scenes of the forward's edge tests: pixels saturating at batch and group boundaries, and alphas on and just above
    1/255 (the pre-reject's margin)."""
    return [("s", *_integrate_scenes.saturation_scene()), ("t", *_integrate_scenes.threshold_scene())]


def make_inputs(path):
    out = {}
    for tag, cfg, view, sigma, aniso, radius in CASES:
        cam = gof_synth.make_camera(cfg["width"], cfg["height"], view=view, radius=radius)
        gs = gof_synth.make_gaussians(cfg["P"], cfg["seed"], cam.focal_x, sigma_px=sigma)
        g = torch.Generator().manual_seed(cfg["seed"] + 50)
        an = torch.exp(torch.rand(cfg["P"], 3, generator=g) * np.log(aniso[1] / aniso[0]) + np.log(aniso[0]))
        gs["scales"] = (gs["scales"].max(dim=1, keepdim=True).values * an).contiguous()
        for k in KEYS:
            out[f"{tag}_{k}"] = gs[k].numpy()
    cam, gs = _integrate_scenes.needle_scene()
    for k in KEYS:
        out[f"{NEEDLES}_{k}"] = gs[k].numpy()
    for tag, cam, gs in _built_scenes():
        for k in KEYS:
            out[f"{tag}_{k}"] = gs[k].numpy()
    np.savez(path, **out)


def main(in_path, out_path):
    dev = torch.device("cuda")
    inp = np.load(in_path)
    res = {}
    views = [(tag, gof_synth.make_camera(cfg["width"], cfg["height"], view=view, radius=radius), cfg["P"]) for tag, cfg, view, _, _, radius in CASES]
    views.append((NEEDLES, _integrate_scenes.needle_scene()[0], _integrate_scenes.NEEDLE_CASE["P"]))
    views += [(tag, cam, int(gs["means3D"].shape[0])) for tag, cam, gs in _built_scenes()]
    degree = {tag: gs["sh_degree"] for tag, _, gs in _built_scenes()}
    for tag, cam, P in views:
        cfg = dict(P=P, width=cam.image_width, height=cam.image_height)
        gs = {k: torch.from_numpy(inp[f"{tag}_{k}"]) for k in KEYS}
        gs["sh_degree"] = degree.get(tag, 3)
        fa = _util.fwd_args(cam, gs, dev)
        # the opacity-field query of points around every Gaussian: its boxes must cover the corner rays as well
        g = torch.Generator().manual_seed(7)
        idx = torch.randint(0, P, (30000,), generator=g)
        pts = (gs["means3D"][idx] + 0.004 * (torch.rand(30000, 3, generator=g) * 2 - 1)).contiguous().to(dev)
        Ri, icolor, ialpha, icol, iradii, igeom, ibin, iimg = _C.integrate_gaussians_to_points(fa[0], pts, *fa[1:])
        ist = _C.export_state(P, cfg["width"], cfg["height"], Ri, igeom, ibin, iimg, iradii)
        res[tag + "_int_color"] = icolor.cpu().numpy()
        res[tag + "_int_alpha"] = ialpha.cpu().numpy()
        res[tag + "_int_colint"] = icol.cpu().numpy()
        res[tag + "_int_ncontrib"] = ist["n_contrib"].cpu().numpy()
        R, color, radii, geom, binning, img = _C.rasterize_gaussians(*fa)
        st = _C.export_state(cfg["P"], cfg["width"], cfg["height"], R, geom, binning, img, radii)
        grad = torch.randn(9, cfg["height"], cfg["width"], generator=torch.Generator().manual_seed(1)).to(dev)
        grads = _C.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, grad))
        res[tag + "_color"] = color.cpu().numpy()
        res[tag + "_ncontrib"] = st["n_contrib"].cpu().numpy()
        res[tag + "_accum"] = st["accum_alpha"].cpu().numpy()
        for n, t in zip(["dmeans2D", "dcolors", "dopacity", "dmeans3D", "dcov3D", "dsh", "dscales", "drot", "dv2g"], grads):
            res[tag + "_" + n] = t.cpu().numpy()
    np.savez(out_path, **res)


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
