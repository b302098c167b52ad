"""GPU: differential test against the unmodified reference extension, through its outputs stored in tests/golden/live_*.npz
(tests/_liveref.py; regenerated on a GPU by tests/golden/make_golden_live_ref.py from oracle/_ref, the reference built by
oracle/build_ref.sh).  BASELINE configs 2 and 3 at full size: every integer / index buffer bit-exact, view2gaussian
bit-exact, images <= 2e-6 relative, gradients within max(1e-4, 6 x the reference's own run-to-run noise)."""
import pytest
import torch

import _liveref
import _util
import gof_synth

pytestmark = pytest.mark.gpu


def _run(name):
    from diff_gaussian_rasterization import _C as ours
    dev = torch.device("cuda")
    fa, P, W, H, grad = _liveref.inputs(name, dev)
    out = ours.rasterize_gaussians(*fa)
    R, _color, radii, geom, binning, img = out
    go = ours.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, grad))
    return fa, P, W, H, grad, out, go


@pytest.mark.parametrize("name,view", [("C2", 3), ("C3", 1)])
def test_full_size_against_live_reference(name, view):
    gold = _liveref.load(f"{name}_v{view}")
    fa, P, W, H, grad, out, go = _run(f"{name}_v{view}")
    _liveref.check_forward(gold, out, P, W, H, buffers=_liveref.BUFFERS,
                           vis_fields=("depths", "means2D", "conic_opacity", "view2gaussian"), depth_channels=True, rgb=True)
    _liveref.check_grads(gold, go)


@pytest.mark.parametrize("M,deg", [(4, 1), (9, 2), (16, 2)])
def test_sh_layouts_against_live_reference(M, deg):
    """SH tensors with M != 16 coefficients / degree below the maximum (scalar load path and partial dL_dsh rows of
    k_preprocess_backward), P not a multiple of the warp size, and backward called twice on the same saved buffers."""
    from diff_gaussian_rasterization import _C as ours
    gold = _liveref.load(f"sh{M}_deg{deg}")
    fa, P, W, H, grad, out, go = _run(f"sh{M}_deg{deg}")
    _liveref.check_forward(gold, out, P, W, H)
    _liveref.check_grads(gold, go, amp_floor=1e-3, amp_factor=6.0)
    R, _c, radii, geom, binning, img = out
    go2 = ours.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, grad))
    for n, a, a2 in zip(_liveref.NAMES, go, go2):
        assert a.shape == a2.shape, n
        if n in _liveref.AMPLIFIED:      # float atomics: the bulk, relative L2
            assert _util.rel_err(a2, a)[1] <= max(1e-3, 6.0 * float(gold[n + "_noise"])), f"{n}: second backward on the same buffers differs"
        else:
            assert _util.rel_err(a2, a)[0] <= max(1e-5, 2.0 * float(gold[n + "_noise"])), f"{n}: second backward on the same buffers differs"
    # coefficients above the active degree receive no gradient (backward.cu:20-139 writes degree <= D only)
    used = (deg + 1) ** 2
    assert float(go[5][:, used:, :].abs().max()) == 0.0 if used < M else True


def test_view2gaussian_precomp_against_live_reference():
    """`view2gaussian_precomp` supplied by the caller (gaussian_renderer/__init__.py: pipe.compute_view2gaussian_python):
    K1 must take the 10-float records as given, the backward must return dL_dview2gaussian and leave scale/rotation
    gradients to the caller's autograd."""
    from diff_gaussian_rasterization import _C as ours
    gold = _liveref.load("v2g_precomp")
    fa, P, W, H, grad, out, go = _run("v2g_precomp")
    _liveref.check_forward(gold, out, P, W, H)
    fa0 = list(fa)
    fa0[8] = torch.Tensor([])
    c0 = ours.rasterize_gaussians(*fa0)[1]
    assert torch.equal(out[1][6], c0[6]) and torch.equal(out[1][7], c0[7])          # same records -> same image as the computed path
    _liveref.check_grads(gold, go)


@pytest.mark.parametrize("with_v2g", [False, True])
def test_cov3d_precomp_against_live_reference(with_v2g):
    """`cov3D_precomp` (forward.cu:339-348): the EWA footprint (radii, tiles, 2D conic, coef) comes from the caller's 3D
    covariance -- here deliberately 1.7x the one scale/rotation would give, so a path that ignored it fails on radii --
    while view2gaussian comes from scale/rotation (with_v2g=False) or from the caller (with_v2g=True, forward.cu:395-403).
    The reference dereferences scales/rotations unconditionally (forward.cu:334-335), so they are always supplied here."""
    from diff_gaussian_rasterization import _C as ours
    name = "cov3d_v2g" if with_v2g else "cov3d"
    gold = _liveref.load(name)
    fa, P, W, H, grad, out, go = _run(name)
    base = list(fa)
    base[7], base[8] = torch.Tensor([]), torch.Tensor([])
    assert not torch.equal(ours.rasterize_gaussians(*base)[2], out[2]), "the inflated covariance must change the radii"
    _liveref.check_forward(gold, out, P, W, H, buffers=_liveref.BUFFERS, vis_fields=("depths", "means2D", "conic_opacity"))
    _liveref.check_grads(gold, go)
    assert float(go[4].abs().max()) == 0.0          # dL_dcov3D stays zero (backward.cu:991-1007: EWA backward disabled)


def test_precomp_through_public_api():
    """GaussianRasterizer.forward(cov3D_precomp=..., view2gaussian_precomp=...) without scales/rotations (the combination the
    Python surface asks for, dgr.py:206-207): same image and dL_dview2gaussian as the `_C`-level call that also passes
    scales/rotations.  (The reference itself faults here: it reads scales[idx] from a null pointer.)"""
    from diff_gaussian_rasterization import _C as ours, GaussianRasterizer
    dev = torch.device("cuda")
    cam, gs = gof_synth.make_scene(dict(P=20_000, width=320, height=240, seed=43), view=2)
    P, W, H = 20_000, 320, 240
    fa0 = _util.fwd_args(cam, gs, dev)
    R0, c0, rad0, geo0, bin0, im0 = ours.rasterize_gaussians(*fa0)
    v2g = ours.export_state(P, W, H, R0, geo0, bin0, im0, rad0)["view2gaussian"].contiguous().requires_grad_(True)
    cov = _liveref.cov3d_from(gs["scales"], gs["rotations"], 1.0).to(dev)
    rs = gof_synth.raster_settings(cam, gs["sh_degree"], dev)
    means3D = gs["means3D"].to(dev).requires_grad_(True)
    means2D = torch.zeros_like(means3D, requires_grad=True)
    color, radii = GaussianRasterizer(rs)(means3D=means3D, means2D=means2D, opacities=gs["opacities"].to(dev), shs=gs["shs"].to(dev),
                                          cov3D_precomp=cov, view2gaussian_precomp=v2g)
    assert torch.equal(color[6], c0[6]) and torch.equal(color[7], c0[7]) and torch.equal(radii, rad0)
    grad = torch.randn(9, H, W, generator=torch.Generator().manual_seed(8)).to(dev)
    (color * grad).sum().backward()
    g0 = ours.rasterize_gaussians_backward(*_util.bwd_args(fa0, rad0, geo0, R0, bin0, im0, grad))
    assert _util.rel_err(v2g.grad, g0[8])[0] < 1e-5


def test_error_in_debug_mode_dumps_snapshot(tmp_path, monkeypatch):
    """debug=True: a failing native call writes the CPU snapshot of its inputs and re-raises
    (diff_gaussian_rasterization/__init__.py:89-96 of the reference)."""
    from diff_gaussian_rasterization import GaussianRasterizer
    dev = torch.device("cuda")
    cam, gs = gof_synth.make_scene(dict(P=500, width=64, height=48, seed=3), view=0)
    rs = gof_synth.raster_settings(cam, 3, dev, debug=True)
    monkeypatch.chdir(tmp_path)
    bad_sh = gs["shs"][:, :4, :].contiguous().to(dev)            # degree 3 needs 16 coefficients: native validation fails
    m3 = gs["means3D"].to(dev)
    with pytest.raises(RuntimeError):
        GaussianRasterizer(rs)(means3D=m3, means2D=torch.zeros_like(m3), opacities=gs["opacities"].to(dev), shs=bad_sh,
                               scales=gs["scales"].to(dev), rotations=gs["rotations"].to(dev))
    snap = torch.load(tmp_path / "snapshot_fw.dump")
    assert isinstance(snap, tuple) and len(snap) == 22 and torch.equal(snap[1], gs["means3D"])   # the forward argument tuple
    # without debug the same error is raised and nothing is written
    (tmp_path / "snapshot_fw.dump").unlink()
    rs2 = gof_synth.raster_settings(cam, 3, dev, debug=False)
    with pytest.raises(RuntimeError):
        GaussianRasterizer(rs2)(means3D=m3, means2D=torch.zeros_like(m3), opacities=gs["opacities"].to(dev), shs=bad_sh,
                                scales=gs["scales"].to(dev), rotations=gs["rotations"].to(dev))
    assert not (tmp_path / "snapshot_fw.dump").exists()
