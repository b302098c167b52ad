"""CPU: the oracle (oracle/gof_oracle.c) against the golden fixtures generated from the UNMODIFIED reference
extension (tests/golden/*.npz, see tests/golden/make_golden.py).  This is what pins the oracle.

Tolerances: integer/index outputs bit-exact.  Per-Gaussian floats bit-exact except rgb (SH evaluation is not
written in the reference's fused order; <= 2e-7).  Image channels 1e-5 except distortion: the CPU expf
differs from CUDA's by an ulp, and the distortion numerator m^2 A + D2 - 2 m D1 cancels to ~1e-4 of its
terms, so that channel only agrees to ~1e-3 on the CPU (it is bit-exact GPU-vs-GPU, test_gpu_golden.py).
Gradients: within max(1e-4, 4 x the reference's own run-to-run noise recorded in the fixture)."""
import numpy as np
import pytest

import _golden
import gof_oracle

FIX = _golden.fixture_paths()
GRADS = dict(dL_dmean2D="dmeans2D", dL_dcolors="dcolors", dL_dopacity="dopacity", dL_dmean3D="dmeans3D", dL_dsh="dsh",
             dL_dscale="dscales", dL_drot="drot", dL_dv2g="dv2g")


def test_fixtures_present():
    assert len(FIX) >= 2, "golden fixtures missing (tests/golden/*.npz)"


@pytest.mark.parametrize("path", FIX, ids=[p.split("/")[-1] for p in FIX])
def test_forward_matches_reference(path):
    fx = _golden.load(path)
    sc = _golden.oracle_scene(fx)
    out, radii, st = gof_oracle.forward(sc)
    vis = fx["visible"]
    assert st["num_rendered"] == int(fx["num_rendered"])
    np.testing.assert_array_equal(radii, fx["radii"])
    np.testing.assert_array_equal(st["tiles_touched"], fx["tiles_touched"].view(np.uint32))
    np.testing.assert_array_equal(st["point_list"], fx["point_list"].view(np.uint32))
    np.testing.assert_array_equal(st["ranges"], fx["ranges"].view(np.uint32))
    np.testing.assert_array_equal(st["n_contrib"], fx["n_contrib"].view(np.uint32))
    for f in ("depths", "means2D", "conic_opacity", "view2gaussian"):
        np.testing.assert_array_equal(st[f][vis].view(np.int32), fx[f][vis].view(np.int32), err_msg=f)
    if fx["colors_precomp"].shape[0] == 0:
        np.testing.assert_array_equal(st["cov3D"][vis].view(np.int32), fx["cov3D"][vis].view(np.int32))
        np.testing.assert_array_equal(st["clamped"][vis], fx["clamped"][vis])
        assert _golden.relerr(st["rgb"][vis], fx["rgb"][vis])[0] < 5e-7
    for ch in range(8):
        assert _golden.relerr(out[ch], fx["color"][ch])[0] < 1e-5, f"channel {ch}"
    np.testing.assert_array_equal(out[6].view(np.int32), fx["color"][6].view(np.int32))   # median depth is exact
    assert _golden.relerr(out[8], fx["color"][8])[0] < 1e-2
    for k in range(3):
        assert _golden.relerr(st["accum_alpha"][k], fx["accum_alpha"][k])[0] < 1e-5


def _bits_popcount(b):
    return np.unpackbits(np.ascontiguousarray(b).view(np.uint8), axis=-1).sum(-1, dtype=np.int64)


def _highest_bit_plus_one(b):
    """[..., nwords] u32 bitsets -> 1 + the index of the highest set bit, 0 where none is set."""
    bits = np.unpackbits(np.ascontiguousarray(b).view(np.uint8), axis=-1, bitorder="little")
    has = bits.any(-1)
    return np.where(has, bits.shape[-1] - np.argmax(bits[..., ::-1], axis=-1), 0)


@pytest.mark.parametrize("path", FIX, ids=[p.split("/")[-1] for p in FIX])
def test_checked_forward_is_the_plain_forward(path):
    """oracle_render_forward_checked computes the plain oracle's outputs bit for bit; its blend bitset agrees with its own
    counters; and its accumulator error bounds hold against the reference extension's outputs (CUDA expf, a double mapped depth)
    at every pixel it does not flag marginal."""
    fx = _golden.load(path)
    sc = _golden.oracle_scene(fx)
    out, radii, st = gof_oracle.forward(sc)
    cout, cradii, cst = gof_oracle.forward(sc, checked=True)
    np.testing.assert_array_equal(cout.view(np.int32), out.view(np.int32))
    np.testing.assert_array_equal(cst["accum_alpha"].view(np.int32), st["accum_alpha"].view(np.int32))
    np.testing.assert_array_equal(cst["n_contrib"], st["n_contrib"])
    bits, last, med = cst["blended"], cst["n_contrib"][0], cst["n_contrib"][1]
    assert bits.shape[-1] * 32 >= int((st["ranges"][:, 1] - st["ranges"][:, 0]).max())
    np.testing.assert_array_equal(_bits_popcount(bits), cst["n_blended"])
    np.testing.assert_array_equal(_highest_bit_plus_one(bits), last)
    has = med != 0xFFFFFFFF
    ys, xs = np.nonzero(has)
    p = med[has].astype(np.int64) - 1
    assert ((bits[ys, xs, p >> 5] >> (p & 31).astype(np.uint32)) & 1).all(), "the median contributor is not in the bitset"
    assert (cst["n_blended"] > 0).mean() > 0.5 and cst["n_blended"].max() > 8
    good = ~cst["marginal_pix"]
    assert good.mean() > 0.99
    np.testing.assert_array_equal(last[good], fx["n_contrib"][0].view(np.uint32)[good])
    np.testing.assert_array_equal(med[good], fx["n_contrib"][1].view(np.uint32)[good])
    for k in range(4):
        d = np.abs(fx["accum_alpha"][k].astype(np.float64) - cst["accum_alpha"][k])
        assert (d[good] <= cst["accum_err"][k][good]).all(), f"accum_alpha[{k}]: {float((d / cst['accum_err'][k])[good].max())} x the bound"


@pytest.mark.parametrize("path", FIX, ids=[p.split("/")[-1] for p in FIX])
def test_backward_matches_reference(path):
    fx = _golden.load(path)
    sc = _golden.oracle_scene(fx)
    _, _, st = gof_oracle.forward(sc)
    d = gof_oracle.backward(sc, st, fx["dL_dout"])
    for k, v in GRADS.items():
        if v == "dsh" and fx["colors_precomp"].shape[0] > 0:
            continue
        err = _golden.relerr(d[k], fx["grad_" + v])[0]
        noise = float(fx["gradnoise_" + v])
        # the three gradients that pass through the view2gaussian chain rule are amplified by ~1/scale^2: the
        # reference's own runs differ by 1e-3..1e-2 there and the 3-run noise estimate in the fixture is itself rough
        tol = max(3e-2, 8.0 * noise) if v in ("dscales", "drot", "dmeans3D") else max(1e-4, 4.0 * noise)
        assert err <= tol, f"{v}: {err} > {tol} (reference noise {noise})"


def test_mark_visible():
    fx = _golden.load(FIX[0])
    vis = gof_oracle.mark_visible(fx["means3D"], fx["viewmatrix"])
    # every Gaussian the reference rasterized is in front of the near plane
    assert np.all(vis[fx["radii"] > 0])
