"""GPU: deterministic gradient criterion at BASELINE config 2 size (200 k Gaussians, 800x800).

The reference accumulates 17 float atomics per (pixel, Gaussian) in scheduling order, and its view2gaussian chain rule
multiplies that noise by ~1/scale^2 -- two reference runs differ by percents in dL_dscales / dL_drot / dL_dmeans3D, so
"ours == reference within 1e-4" is not a usable criterion for those (DESIGN.md 2.2).  This test pins them against the fp64
evaluation of the SAME formulas instead (oracle/gof_oracle.c: double accumulation, double chain rule):

    err(ours, fp64)  <=  max(2 * err(reference, fp64), 1e-6)          for every gradient tensor, max-norm and relative L2

with err(reference, fp64) measured in the same run on the live reference extension, or, where that is not built, as stored by
tests/golden/make_golden_live_ref.py in tests/golden/live_grad_fp64_c2.npz."""
import numpy as np
import pytest
import torch

import _liveref
import _util
import gof_oracle
import gof_synth

pytestmark = pytest.mark.gpu
NAMES = ["dmeans2D", "dcolors", "dopacity", "dmeans3D", "dcov3D", "dsh", "dscales", "drot", "dv2g"]
OMAP = dict(dmeans2D="dL_dmean2D", dopacity="dL_dopacity", dmeans3D="dL_dmean3D", dsh="dL_dsh", dscales="dL_dscale", drot="dL_drot", dv2g="dL_dv2g")


def _err(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)), float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def c2_inputs(dev):
    cam, gs = gof_synth.make_scene("C2", view=3)
    dL = torch.randn(9, cam.image_height, cam.image_width, generator=torch.Generator().manual_seed(77))
    return cam, gs, _util.fwd_args(cam, gs, dev), dL


def fp64_gradients(cam, gs, dL):
    """The oracle's fp64 forward + backward of the C2 view: (radii, {name: gradient})."""
    sc = gof_oracle.scene_from_synth(cam, gs)
    _out, oradii, st = gof_oracle.forward(sc)
    return oradii, gof_oracle.backward(sc, st, dL.numpy())


def test_gradients_against_fp64_oracle_at_c2():
    from diff_gaussian_rasterization import _C as ours
    ref = _util.load_ref()
    dev = torch.device("cuda")
    cam, gs, fa, dL = c2_inputs(dev)
    R, color, radii, geom, binning, img = ours.rasterize_gaussians(*fa)
    go = ours.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, dL.to(dev)))
    gr = None
    stored = _liveref.load("grad_fp64_c2") if ref is None else None
    if ref is not None:
        Rr, cr, radr, ger, binr, imr = ref.rasterize_gaussians(*fa)
        gr = ref.rasterize_gaussians_backward(*_util.bwd_args(fa, radr, ger, Rr, binr, imr, dL.to(dev)))
        gr2 = ref.rasterize_gaussians_backward(*_util.bwd_args(fa, radr, ger, Rr, binr, imr, dL.to(dev)))
    torch.cuda.synchronize()
    oradii, od = fp64_gradients(cam, gs, dL)
    assert np.array_equal(radii.cpu().numpy(), oradii)
    report, failures = {"config": "C2 view 3: 200000 Gaussians, 800x800, sh_degree 3", "criterion": "err(ours,fp64) <= max(2*err(ref,fp64), 1e-6); (max-norm, relative L2)"}, []
    for i, n in enumerate(NAMES):
        if n not in OMAP:
            continue
        eo = _err(go[i].cpu().numpy(), od[OMAP[n]])
        row = {"ours_vs_fp64": eo}
        if gr is not None:
            er = _err(gr[i].cpu().numpy(), od[OMAP[n]])
            row.update(ref_vs_fp64=er, ref_vs_ref=_err(gr2[i].cpu().numpy(), gr[i].cpu().numpy()), ours_vs_ref=_err(go[i].cpu().numpy(), gr[i].cpu().numpy()))
        else:
            er = tuple(float(x) for x in stored[n])
            row.update(ref_vs_fp64=er)
        ok = eo[0] <= max(2 * er[0], 1e-6) and eo[1] <= max(2 * er[1], 1e-6)
        row["ok"] = bool(ok)
        report[n] = row
        if not ok:
            failures.append((n, row))
    assert not failures, (failures, report)
