"""The error scales of the oracle's blend backward (gof_oracle.render_backward(..., bounds=True)) and the per-Gaussian
comparator built on them (tests/_grad_bounds.py), on the CPU: the scales bound what they claim to bound, the marginal mass
marks exactly the pairs whose blend decision is marginal, and the comparator catches a wrong gradient."""
import numpy as np
import pytest

import _grad_bounds as gb
import gof_oracle
import gof_synth


@pytest.fixture(scope="module")
def scene():
    cam, gs = gof_synth.make_scene(dict(P=3000, width=96, height=64, seed=13), view=6)
    sc = gof_oracle.scene_from_synth(cam, gs, bg=(0.2, 0.5, 0.8))
    _out, radii, st = gof_oracle.forward(sc)
    dL = np.random.default_rng(4).standard_normal((9, cam.image_height, cam.image_width)).astype(np.float32)
    return sc, radii, st, dL


def _bwd(sc, st, dL):
    return gof_oracle.render_backward(sc, st, st["point_list"], st["ranges"], st["accum_alpha"], st["n_contrib"], dL, bounds=True)


def test_bounds_leave_the_gradients_unchanged(scene):
    sc, radii, st, dL = scene
    plain = gof_oracle.render_backward(sc, st, st["point_list"], st["ranges"], st["accum_alpha"], st["n_contrib"], dL)
    d = _bwd(sc, st, dL)
    for k, v in plain.items():
        np.testing.assert_array_equal(d[k], v, err_msg=k)


def test_mag_bounds_every_value(scene):
    sc, radii, st, dL = scene
    d = _bwd(sc, st, dL)
    val, mag = gb.oracle17(d), d["mag"]
    assert (mag >= 0).all() and (mag[radii > 0].sum(axis=1) > 0).mean() > 0.5
    assert (mag[radii == 0] == 0).all()
    # the float rounding of each pair term may exceed its exact magnitude by a few ulp
    assert (np.abs(val) <= mag * (1 + 2.0 ** -20)).all()
    # dL_dcolors is a sum of alpha * T * dL_dpix: for non-negative dL_dpix a sum of non-negative terms, equal to its magnitude
    d = _bwd(sc, st, np.abs(dL))
    val, mag = gb.oracle17(d), d["mag"]
    np.testing.assert_allclose(val[:, :3], mag[:, :3], rtol=2.0 ** -20, atol=0)


def _state(v2g, opacity, lists, W=48, H=16):
    """A hand-made forward state: Gaussian i has view2gaussian v2g[i] and opacity[i]; tile j's list is lists[j]."""
    P = len(v2g)
    sc = gof_oracle.Scene(W, H, 0.5, 0.5, np.eye(4), np.eye(4), np.zeros(3), np.zeros((P, 3)), np.asarray(opacity).reshape(P, 1),
                          bg=(0.3, 0.1, 0.6))
    g = dict(view2gaussian=np.asarray(v2g, np.float32), rgb=np.tile(np.float32([0.9, 0.4, 0.1]), (P, 1)),
             means2D=np.tile(np.float32([8.0, 8.0]), (P, 1)),
             conic_opacity=np.concatenate([np.tile(np.float32([0.05, 0.01, 0.04]), (P, 1)), np.float32(opacity).reshape(P, 1)], 1))
    point_list = np.asarray([i for lst in lists for i in lst], np.uint32)
    ranges, o = [], 0
    for lst in lists:
        ranges.append((o, o + len(lst)))
        o += len(lst)
    ranges = np.asarray(ranges, np.uint32)
    _out, final_T, n_contrib = gof_oracle.render_forward(sc, g, point_list, ranges)
    return sc, g, point_list, ranges, final_T, n_contrib


def test_marginal_mass_marks_threshold_pairs():
    """v2g (0,0,0,0,0,1, 0,0,-2, C): normal (0,0,1), AA = 1, BB = -4, t = 2 at every pixel, and power = min(0, 2 - C/2).  So
    C = 0 gives G = 1 and alpha = opacity exactly."""
    thr = np.float32(1.0) / np.float32(255.0)
    below = np.nextafter(thr, np.float32(0))
    flat = lambda c: [0, 0, 0, 0, 0, 1, 0.3, 0, -2, c]   # noqa: E731  (+0.3 rx: the ordinary ones vary over the tile)
    v2g = [flat(0.0), flat(4.5), flat(0.0), flat(4.5)]
    opacity = [thr, 0.5, below, 0.5]
    # tile 0: alpha exactly 1/255 (blended by the host); tile 1: an ordinary Gaussian; tile 2: alpha one ulp below 1/255
    # (rejected by the host, where a 2-ulp expf may blend it) in front of an ordinary one, which keeps it inside the walk
    sc, g, pl, ranges, final_T, n_contrib = _state(v2g, opacity, [[0], [1], [2, 3]])
    assert (n_contrib[0][:, :16] == 1).all() and (n_contrib[0][:, 32:] == 2).all()
    dL = np.random.default_rng(1).standard_normal((9, 16, 48)).astype(np.float32)
    d = gof_oracle.render_backward(sc, g, pl, ranges, final_T, n_contrib, dL, bounds=True)
    mag, marg = d["mag"], d["marginal"]
    assert marg[0].sum() > 0 and np.array_equal(marg[0], mag[0])   # every pair of Gaussian 0 is marginal
    assert (marg[1] == 0).all() and mag[1].sum() > 0
    assert (gb.oracle17(d)[2] == 0).all() and marg[2].sum() > 0     # not blended here: its would-be term is marginal
    assert (marg[3] == 0).all() and mag[3].sum() > 0                # behind the marginal pair: unaffected by its decision


def test_ordinary_scene_has_almost_no_marginal_mass(scene):
    sc, radii, st, dL = scene
    d = _bwd(sc, st, dL)
    vis = radii > 0
    share = float((d["marginal"][vis].sum(axis=1) > 0).mean())
    assert share <= 1e-3, share


def test_comparator_flags_a_perturbed_pixel(scene):
    """The oracle against itself with dL_dpix changed at one pixel: the comparator flags some Gaussians, and only ones that
    blend at that pixel.  With nothing changed it flags nothing."""
    sc, radii, st, dL = scene
    base = _bwd(sc, st, dL)
    L = int(st["n_contrib"][0].max())
    args = (base["mag"], base["marginal"], L, gb.blend_constant(L))
    assert gb.flagged(gb.oracle17(base), gb.oracle17(base), *args).size == 0
    py, px = np.unravel_index(np.argmax(st["n_contrib"][0]), st["n_contrib"][0].shape)
    one = np.zeros_like(dL)
    one[:, py, px] = 1.0
    blends_there = np.nonzero(_bwd(sc, st, one)["mag"].sum(axis=1) > 0)[0]
    assert blends_there.size > 10
    dL2 = dL.copy()
    dL2[:, py, px] += 0.05
    bad = gb.flagged(gb.oracle17(_bwd(sc, st, dL2)), gb.oracle17(base), *args)
    assert bad.size > 0
    assert np.isin(bad, blends_there).all()
