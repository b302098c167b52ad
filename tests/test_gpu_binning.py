"""GPU: the one-sweep binning (csrc/binning.cu: single-launch radix passes with decoupled look-back, fused scan + instance
emission, num_rendered summed by the preprocess kernel and read on a side stream) against the CPU oracle's restatement of
the reference's binning (oracle/gof_oracle.c, pinned to the reference's golden lists by test_oracle_golden.py) -- every
index buffer bit-exact, over sizes that exercise one / two tile digits, ragged tails, chunks with empty digits, a single
chunk, and tile lists of big splats.  Also: the query points' sort by tile and pixel (integrate) through the permutation
invariance of the integrate outputs, and the look-back scan through gof_densify_plan against numpy.  The pair sorts and
scans of marching tetrahedra are pinned to the reference's outputs by test_tetmesh.py::test_cuda_matches_reference_golden."""
import numpy as np
import pytest
import torch

import _golden
import _util
import gof_oracle
import gof_synth

pytestmark = pytest.mark.gpu

CASES = [
    dict(P=1, width=16, height=16, seed=1),                       # one Gaussian, one tile
    dict(P=257, width=64, height=48, seed=2),                     # a few chunks' worth of nothing: single-chunk sorts
    dict(P=5_000, width=256, height=256, seed=3),                 # 256 tiles: ONE tile digit
    dict(P=4_097, width=272, height=256, seed=4),                 # 272 tiles: two digits, P just over one sort chunk
    dict(P=70_001, width=800, height=608, seed=5),
    dict(P=3_000, width=320, height=240, seed=6, sigma_px=25.0),  # big splats: thousands of instances per CTA of the emit kernel
    dict(P=300_000, width=1920, height=1080, seed=7),
]


def _bits(t):
    return t.contiguous().view(torch.int32)


def _forward(fa, P, W, H):
    """One forward; returns host copies only, so the scratch buffers go back to the pool for the next call."""
    from diff_gaussian_rasterization import _C
    R, color, radii, geom, binning, img = _C.rasterize_gaussians(*fa)
    st = _C.export_state(P, W, H, R, geom, binning, img, radii)
    torch.cuda.synchronize()
    keep = ("means2D", "depths", "tiles_touched", "point_list", "ranges", "n_contrib")
    return R, radii.cpu(), {k: st[k].cpu() for k in keep}, color.cpu()


@pytest.mark.parametrize("cfg", CASES, ids=[f"P{c['P']}_{c['width']}x{c['height']}" for c in CASES])
def test_onesweep_binning_matches_oracle(cfg):
    dev = torch.device("cuda")
    cam, gs = gof_synth.make_scene(cfg, view=cfg["seed"])
    fa = _util.fwd_args(cam, gs, dev)
    P, W, H = cfg["P"], cfg["width"], cfg["height"]
    R, radii, st, color = _forward(fa, P, W, H)
    R2, radii2, st2, color2 = _forward(fa, P, W, H)              # again, over the pooled scratch the first call left behind
    assert R > 0
    assert R2 == R, "num_rendered"
    assert torch.equal(radii2, radii)
    for k in ("point_list", "ranges", "n_contrib"):
        assert torch.equal(st2[k], st[k]), k
    assert torch.equal(_bits(color2), _bits(color)), "same lists -> same image bits"

    # the oracle bins the Gaussians this call preprocessed: (tile, depth bits, index) order of the reference's stable sort
    oR, opoint_list, oranges = gof_oracle.bin_tiles(W, H, radii.numpy(), st["means2D"].numpy(), st["depths"].numpy(),
                                                    st["tiles_touched"].numpy().view(np.uint32))
    assert R == oR, "num_rendered"
    np.testing.assert_array_equal(st["point_list"].numpy().view(np.uint32), opoint_list)
    np.testing.assert_array_equal(st["ranges"].numpy().view(np.uint32), oranges)


def test_integrate_is_invariant_to_the_order_of_the_points():
    """The query points are sorted by (tile, pixel) before the point-parallel pass.  Every per-point result depends on that
    point alone, and the only per-pixel atomic is the integer point count, so shuffling the points must give bit-identical
    results once they are put back in order: a point sorted into the wrong tile or pixel, or a wrong per-tile point range,
    shows up here."""
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda")
    cam, gs = gof_synth.make_scene(dict(P=20_000, width=400, height=304, seed=9), view=3)
    fa = _util.fwd_args(cam, gs, dev)
    PN = 300_007
    pts = ((torch.rand(PN, 3, generator=torch.Generator().manual_seed(1)) * 2 - 1) * 1.6).to(dev)
    perm = torch.randperm(PN, generator=torch.Generator().manual_seed(2)).to(dev)
    R, color, alpha, col_int, radii = _C.integrate_gaussians_to_points(fa[0], pts, *fa[1:])[:5]
    Rp, color_p, alpha_p, col_int_p, radii_p = _C.integrate_gaussians_to_points(fa[0], pts[perm].contiguous(), *fa[1:])[:5]
    alpha_u, col_int_u = torch.empty_like(alpha_p), torch.empty_like(col_int_p)
    alpha_u[perm], col_int_u[perm] = alpha_p, col_int_p
    torch.cuda.synchronize()
    assert Rp == R and torch.equal(radii_p, radii)
    assert torch.equal(_bits(alpha_u), _bits(alpha))
    assert torch.equal(_bits(col_int_u), _bits(col_int))
    for ch in range(9):
        assert torch.equal(_bits(color_p[ch]), _bits(color[ch])), f"channel {ch}"

    # and the unshuffled call against the oracle, within test_integrate.py's tolerances
    ocolor, oalpha, _ocol, oradii, _st = gof_oracle.integrate(gof_oracle.scene_from_synth(cam, gs), pts.cpu())
    color, alpha = color.cpu().numpy(), alpha.cpu().numpy()
    np.testing.assert_array_equal(radii.cpu().numpy(), oradii)
    np.testing.assert_array_equal(color[8], ocolor[8])
    np.testing.assert_array_equal(color[3:6], ocolor[3:6])
    for ch in (0, 1, 2, 6, 7):
        assert _golden.relerr(color[ch], ocolor[ch])[0] < 1e-5, f"channel {ch}"
    assert np.abs(alpha.astype(np.float64) - oalpha).max() < 5e-4
    assert (oalpha < 1).sum() > PN // 2


@pytest.mark.parametrize("P", [1, 2047, 2048, 2049, 4097, 1_000_003])
def test_exclusive_scan_through_densify_plan(P):
    """gof_densify_plan scans its four keep-flag rows with the single-launch look-back scan (2048 values per CTA): sizes
    around one chunk and over hundreds of chunks, every offset and total against numpy."""
    import gof_densify
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(P)
    acc = (torch.rand(P, generator=g) * 6e-4).to(dev)
    acc_abs = (torch.rand(P, generator=g) * 9e-4).to(dev)
    den = torch.randint(0, 3, (P,), generator=g).float().to(dev)
    scaling = torch.log(torch.rand(P, 3, generator=g) * 0.04 + 1e-3).to(dev)
    opacity = (torch.randn(P, generator=g) * 2.0).to(dev)
    flags = torch.empty(4 * P, dtype=torch.int32, device=dev)
    offsets = torch.empty_like(flags)
    totals = torch.empty(4, dtype=torch.int32, device=dev)
    tmp = torch.empty(int(gof_densify._lib.gof_densify_scratch_bytes(P)), dtype=torch.uint8, device=dev)
    _C._check(gof_densify._lib.gof_densify_plan(P, acc.data_ptr(), acc_abs.data_ptr(), den.data_ptr(), scaling.data_ptr(),
                                                opacity.data_ptr(), 2e-4, 4e-4, 0.017, 0.05, 0.035, flags.data_ptr(),
                                                offsets.data_ptr(), totals.data_ptr(), tmp.data_ptr(), _C._stream()))
    f = flags.cpu().numpy().astype(np.int64).reshape(4, P)
    assert set(np.unique(f)) <= {0, 1}
    np.testing.assert_array_equal(offsets.cpu().numpy().astype(np.int64).reshape(4, P), np.cumsum(f, axis=1) - f)
    np.testing.assert_array_equal(totals.cpu().numpy().astype(np.int64), f.sum(axis=1))
    if P > 2048:
        assert np.all((f.sum(axis=1) > 0) & (f.sum(axis=1) < P)), "every row mixes kept and dropped Gaussians"
