"""Opacity-field query (GaussianRasterizer.integrate).  CPU: the oracle against the reference's golden outputs.
GPU: the CUDA path against the golden outputs, the oracle and (when built) the live reference."""
import numpy as np
import pytest
import torch

import _golden
import gof_oracle
import gof_synth

FIX = [p for p in _golden.fixture_paths() if "int_alpha" in _golden.load(p)]


def _check_vs_golden(fx, color, alpha, col_int, n_contrib, final_T, tol_alpha, exact_counts=True):
    nc = np.asarray(n_contrib).astype(np.int64)
    if exact_counts:
        np.testing.assert_array_equal(nc, fx["int_n_contrib"].astype(np.int64))
    else:   # CPU expf differs from CUDA's by an ulp: a blend weight sitting on the 1/255 threshold may flip
        assert (nc != fx["int_n_contrib"].astype(np.int64)).mean() < 5e-3
    np.testing.assert_array_equal(color[8], fx["int_color"][8])                       # projected points per pixel
    assert _golden.relerr(color[6], fx["int_color"][6])[0] < 1e-6                     # max t
    ftol = 1e-5 if exact_counts else 5e-4      # a flipped threshold on the CPU moves T by up to 1e-4
    for ch in (0, 1, 2, 7):
        assert _golden.relerr(color[ch], fx["int_color"][ch])[0] < ftol, f"channel {ch}"
    assert float(np.abs(color[3:6]).max()) == 0.0
    assert _golden.relerr(final_T, fx["int_final_T"])[0] < ftol
    assert np.abs(alpha.astype(np.float64) - fx["int_alpha"]).max() < tol_alpha
    assert _golden.relerr(col_int, fx["int_color_integrated"])[0] < ftol
    # points that never projected keep the initial 1.0 / 0.0 (rasterize_points.cu:277-278)
    untouched = (fx["int_alpha"] == 1.0) & (np.abs(fx["int_color_integrated"]).sum(1) == 0)
    assert np.all(alpha[untouched] == 1.0)


def test_integrate_fixtures_present():
    assert len(FIX) >= 2, "golden fixtures lack the integrate section: regenerate with tests/golden/make_golden.py"


@pytest.mark.parametrize("path", FIX, ids=[p.split("/")[-1] for p in FIX])
def test_oracle_integrate_matches_reference(path):
    fx = _golden.load(path)
    sc = _golden.oracle_scene(fx)
    color, alpha, col_int, radii, st = gof_oracle.integrate(sc, fx["int_points"])
    # the CPU expf differs from CUDA's by an ulp and pass 2 evaluates -(A t^2 + B t + C)/2 in float: 2e-4 absolute
    _check_vs_golden(fx, color, alpha, col_int, st["n_contrib"], st["final_T"], tol_alpha=2e-4, exact_counts=False)


@pytest.mark.gpu
@pytest.mark.parametrize("path", FIX, ids=[p.split("/")[-1] for p in FIX])
def test_cuda_integrate_matches_reference_golden(path):
    import test_gpu_golden as tg
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda")
    fx = _golden.load(path)
    cfg = fx["cfg"]
    fa = tg._fwd_args(fx, dev)
    ia = (fa[0], torch.from_numpy(fx["int_points"]).to(dev)) + tuple(fa[1:])
    R, color, alpha, col_int, radii, geom, binning, img = _C.integrate_gaussians_to_points(*ia)
    assert R == int(fx["num_rendered"])
    np.testing.assert_array_equal(radii.cpu().numpy(), fx["radii"])
    st = _C.export_state(cfg["P"], cfg["W"], cfg["H"], R, geom, binning, img, radii)
    _check_vs_golden(fx, color.cpu().numpy(), alpha.cpu().numpy(), col_int.cpu().numpy(), st["n_contrib"][0].cpu().numpy(),
                     st["accum_alpha"][0].cpu().numpy(), tol_alpha=2e-6)


@pytest.mark.gpu
def test_cuda_integrate_vs_oracle_and_module_api():
    """Through GaussianRasterizer.integrate (the call extract_mesh.py makes, gaussian_renderer/__init__.py:199-209)."""
    from diff_gaussian_rasterization import GaussianRasterizer
    dev = torch.device("cuda")
    cam, gs = gof_synth.make_scene(dict(P=8000, width=208, height=136, seed=33), view=12)
    g = torch.Generator().manual_seed(2)
    pts = torch.cat([gs["means3D"][torch.randint(0, 8000, (6000,), generator=g)] + 0.01 * torch.randn(6000, 3, generator=g),
                     (torch.rand(6000, 3, generator=g) * 2 - 1) * 1.6]).contiguous()
    rs = gof_synth.raster_settings(cam, 3, dev, bg=(0.2, 0.3, 0.4))
    with torch.no_grad():
        color, alpha, col_int, radii = GaussianRasterizer(rs).integrate(
            points3D=pts.to(dev), means3D=gs["means3D"].to(dev), means2D=torch.zeros_like(gs["means3D"]).to(dev),
            opacities=gs["opacities"].to(dev), shs=gs["shs"].to(dev), scales=gs["scales"].to(dev), rotations=gs["rotations"].to(dev))
    sc = gof_oracle.scene_from_synth(cam, gs, bg=(0.2, 0.3, 0.4))
    ocolor, oalpha, ocol, oradii, st = gof_oracle.integrate(sc, pts)
    np.testing.assert_array_equal(radii.cpu().numpy(), oradii)
    np.testing.assert_array_equal(color[8].cpu().numpy(), ocolor[8])
    for ch in (0, 1, 2, 6, 7):
        assert _golden.relerr(color[ch].cpu().numpy(), ocolor[ch])[0] < 1e-5
    assert np.abs(alpha.cpu().numpy().astype(np.float64) - oalpha).max() < 5e-4
    assert (oalpha < 1).sum() > 3000


@pytest.mark.gpu
def test_cuda_integrate_vs_live_reference_1080p():
    """Against the unmodified reference extension's outputs stored in tests/golden/live_integrate_1080p.npz (tests/_liveref.py).
    Colour, accumulated alpha, point counts and integrated colours are bit-exact.  The reference's integrateCUDA evaluates the
    five rays' quadrics with whatever fusion ptxas picks for the target: its sm_90a build rounds some ray depths differently
    from the sm_100a build this implementation restates (and the fixtures above pin), which moves the maximum depth of a few
    pixels (0.06 % beyond 1e-5 on an H100; at most 3.76 of a 6.34 maximum, where another Gaussian's depth becomes the largest)
    and the alpha of a few points (0.002 % beyond 2e-6, at most 0.0091) -- compared here as the share that agrees to 2e-6,
    with every sampled value bounded by about 1.3x (depth) and 2x (alpha) those measured maxima."""
    import _liveref
    from diff_gaussian_rasterization import _C as ours
    gold = _liveref.load("integrate_1080p")
    dev = torch.device("cuda")
    Ro, co, ao, cio, rado, *_ = ours.integrate_gaussians_to_points(*_liveref.integrate_inputs(dev))
    assert Ro == int(gold["R"]) and _liveref.digest(rado) == str(gold["radii"])
    for ch in (0, 1, 2, 3, 4, 5, 7, 8):
        assert _liveref.digest(co[ch]) == str(gold[f"color{ch}"]), f"channel {ch}"
    assert _liveref.digest(cio) == str(gold["color_integrated"])
    px, pt = torch.from_numpy(gold["pix"]).to(dev), torch.from_numpy(gold["pts"]).to(dev)
    tmax = co[6].flatten()[px].cpu().double().numpy()
    assert np.mean(np.abs(tmax - gold["tmax"]) <= 2e-6 * float(gold["tmax_absmax"])) > 0.995
    assert np.abs(tmax - gold["tmax"]).max() <= 0.75 * float(gold["tmax_absmax"])
    alpha = ao[pt].cpu().double().numpy()
    assert np.mean(np.abs(alpha - gold["alpha"]) <= 2e-6) > 0.995
    assert np.abs(alpha - gold["alpha"]).max() <= 0.02
