"""CPU: the float64 oracle of the query's colour backward (tests/integrate_grad_oracle/integrate_color_oracle.c, DESIGN.md 4.13) against central
differences of a float64 restatement of one pixel's compositing with its blended set held fixed, and the argument checks of
gof_integrate_backward with the colour through the built library (decided before any device work)."""
import ctypes

import numpy as np
import pytest

import _integrate_color_oracle as igc

W = H = 16
TAN = 0.5
PX, PY = 8, 8
FX = W / (2 * TAN)
RX, RY = float(np.float32((PX + 0.5 - W * 0.5) / FX)), float(np.float32((PY + 0.5 - H * 0.5) / FX))


def iso(m, s, dc=0.0):
    """view2gaussian of an isotropic Gaussian at camera-space m with inverse variance s: q(p) = s |p - m|^2 - dc."""
    m = np.asarray(m, np.float64)
    return np.array([s, 0, 0, s, 0, s, -s * m[0], -s * m[1], -s * m[2], s * m @ m - dc])


def composite(v2g, op, rgb, bg, keep=None):
    """Float64 restatement of the centre ray of pixel (PX, PY) over the list in order: returns (C [3], accepted mask).  With
    `keep`, the accepted set is held fixed to it."""
    x, y = RX, RY
    T, C, acc = 1.0, np.zeros(3), np.zeros(len(op), bool)
    for j, v in enumerate(v2g):
        AA = v[0] * x * x + 2 * v[1] * x * y + 2 * v[2] * x + v[3] * y * y + 2 * v[4] * y + v[5]
        BB = 2 * (v[6] * x + v[7] * y + v[8])
        t = -BB / (2 * AA)
        power = min(0.0, -0.5 * (v[9] - BB * BB / (4 * AA)))
        al = min(0.99, op[j] * np.exp(power))
        if keep is None:
            if t < 0.2 or al < 1 / 255 or T * (1 - al) < 1e-4:
                continue
        elif not keep[j]:
            continue
        acc[j] = True
        C += T * al * rgb[j]
        T *= 1 - al
    return C + T * np.asarray(bg), acc


def oracle(v2g, op, rgb, bg, dLdC):
    n = len(op)
    st = dict(ranges=np.array([[0, n]]), point_list=np.arange(n), view2gaussian=v2g.astype(np.float32),
              conic_opacity=np.stack([np.zeros(n), np.zeros(n), np.zeros(n), op], 1).astype(np.float32), rgb=rgb.astype(np.float32))
    d = np.zeros((H, W, 3))
    d[PY, PX] = dLdC
    return igc.view(W, H, TAN, TAN, st, np.asarray(bg, np.float32), d)


def fd(v2g, op, rgb, bg, dLdC, acc):
    """Central differences of dLdC . C with respect to every v2g and rgb entry, the accepted set fixed."""
    L = lambda v, c: float(np.dot(dLdC, composite(v, op, c, bg, acc)[0]))   # noqa: E731
    dv, dc = np.zeros_like(v2g), np.zeros_like(rgb)
    for j in range(len(op)):
        for k in range(10):
            h = 1e-6 * max(1.0, abs(v2g[j, k]))
            a, b = v2g.copy(), v2g.copy()
            a[j, k] += h
            b[j, k] -= h
            dv[j, k] = (L(a, rgb) - L(b, rgb)) / (2 * h)
        for c in range(3):
            a, b = rgb.copy(), rgb.copy()
            a[j, c] += 1e-6
            b[j, c] -= 1e-6
            dc[j, c] = (L(v2g, a) - L(v2g, b)) / 2e-6
    return dv, dc


def check(v2g, op, rgb, bg, dLdC, expect_accepted=None):
    v2g = v2g.astype(np.float32).astype(np.float64)   # the oracle sees the float records
    op, rgb = np.asarray(op, np.float32).astype(np.float64), np.asarray(rgb, np.float32).astype(np.float64)
    C, acc = composite(v2g, op, rgb, bg)
    if expect_accepted is not None:
        assert acc.tolist() == expect_accepted
    o = oracle(v2g, op, rgb, bg, np.asarray(dLdC))
    assert not o["marg_g"].any()   # the cases are built away from every threshold
    np.testing.assert_allclose(o["C"][PY, PX], C, rtol=1e-5, atol=1e-6)
    dv, dc = fd(v2g, op, rgb, bg, np.asarray(dLdC), acc)
    tol_c = 1e-5 * (o["mag_c"] + 1e-3)
    assert np.all(np.abs(o["dcol"] - dc) <= tol_c), np.abs(o["dcol"] - dc).max()
    tol_v = 1e-4 * (o["mag_g"] + 1e-4 * np.abs(o["mag_g"]).max(axis=1, keepdims=True) + 1e-6)
    assert np.all(np.abs(o["dv2g"] - dv) <= tol_v), np.abs(o["dv2g"] - dv).max()
    return o, acc


def test_random_pairs_and_background():
    rng = np.random.default_rng(1)
    n = 12
    m = np.stack([RX * 3 + rng.normal(0, 0.05, n), RY * 3 + rng.normal(0, 0.05, n), rng.uniform(2.5, 4.0, n)], 1)
    v2g = np.stack([iso(m[j], rng.uniform(20, 80)) for j in range(n)])
    o, acc = check(v2g, rng.uniform(0.1, 0.6, n), rng.uniform(0, 1, (n, 3)), (0.3, 0.6, 0.1), rng.normal(size=3))
    assert acc.sum() >= 8 and np.abs(o["dv2g"]).max() > 0


def test_alpha_clamp_and_power_clamp_have_zero_v2g_derivative():
    """Pair 1 sits at the 0.99 clamp (op 0.9995 just off the ray), pair 2 has its power clamped to 0 (a quadric whose minimum is
    below 0): both keep their colour derivative and have an exact zero view2gaussian derivative."""
    v2g = np.stack([iso((RX * 3 + 0.03, RY * 3, 3.0), 40), iso((RX * 3, RY * 3, 3.2), 40), iso((RX * 3.4, RY * 3.4, 3.4), 30, dc=0.5),
                    iso((RX * 3.6 - 0.02, RY * 3.6, 3.6), 30)])
    o, acc = check(v2g, [0.3, 0.9995, 0.4, 0.5], [[1, 0, 0], [0, 1, 0], [0, 0, 1], [0.5, 0.5, 0.5]], (0.2, 0.2, 0.2), [0.7, -0.4, 1.1])
    assert acc.all()
    assert np.all(o["dv2g"][1] == 0) and np.all(o["dv2g"][2] == 0)
    assert np.all(o["dcol"][1] != 0) and np.all(o["dcol"][2] != 0)


def test_transmittance_skip_is_followed_by_accepted_pairs():
    """T falls to 2.25e-4 after two pairs of alpha 0.985; a third of alpha 0.9 would take it below 1e-4 and is skipped without
    ending the ray, and a fourth of alpha 0.3 is still blended."""
    c = (RX * 3, RY * 3)
    v2g = np.stack([iso((c[0], c[1], 3.0), 40, dc=-0.004), iso((c[0], c[1], 3.1), 40, dc=-0.004), iso((c[0], c[1], 3.2), 40, dc=-0.004),
                    iso((c[0], c[1], 3.3), 40, dc=-0.004)])
    op = np.array([0.985, 0.985, 0.9, 0.3]) / np.exp(-0.002)
    o, acc = check(v2g, op, np.random.default_rng(2).uniform(0, 1, (4, 3)), (0.5, 0.1, 0.9), [1.0, -2.0, 0.5],
                   expect_accepted=[True, True, False, True])
    assert np.all(o["dcol"][2] == 0) and np.all(o["dv2g"][2] == 0) and np.all(o["dcol"][3] != 0)


# ---------------- argument checks of the colour backward and of the binding's color_min ----------------
FAKE = 0x1000


def _abi():
    try:
        from diff_gaussian_rasterization import _C
    except ImportError as e:   # the library is built by __graft_entry__.build()
        pytest.skip(str(e))
    return _C


def _scene(_C, P=10, shs=False):
    s = _C._Scene()
    s.P, s.width, s.height, s.tan_fovx, s.tan_fovy = P, 32, 32, 0.5, 0.5
    for name in ("means3D", "opacities", "viewmatrix", "projmatrix", "background", "scales", "rotations"):
        setattr(s, name, FAKE)
    if shs:
        s.shs, s.cam_pos, s.M, s.D = FAKE, FAKE, 16, 3
    else:
        s.colors_precomp = FAKE
    return s


def _bwd(_C, s, PN=4, scratch=FAKE, nbytes=10 ** 6, **kw):
    a = dict(points=FAKE, radii=FAKE, geom=FAKE, binning=FAKE, image=FAKE, pts=FAKE, pbin=FAKE, dalpha=FAKE, dcolor=FAKE,
             dpts=FAKE, dop=FAKE, dmean=FAKE, dscale=FAKE, drot=FAKE, dv2g=FAKE, dcov=FAKE, dcolors=FAKE, dsh=FAKE)
    a.update(kw)
    o = _C._BackwardOut(dL_dopacity=a["dop"], dL_dmean3D=a["dmean"], dL_dscale=a["dscale"], dL_drot=a["drot"],
                        dL_dview2gaussian=a["dv2g"], dL_dcov3D=a["dcov"], dL_dcolor=a["dcolors"], dL_dsh=a["dsh"], scratch=scratch,
                        scratch_bytes=nbytes)
    return _C._lib.gof_integrate_backward(ctypes.byref(s), PN, a["points"], 1, a["radii"], a["geom"], a["binning"], a["image"],
                                          a["pts"], a["pbin"], a["dalpha"], a["dcolor"], a["dpts"], ctypes.byref(o), None)


def test_backward_color_refusals_with_out():
    _C = _abi()
    err = _C._lib.gof_last_error
    s = _scene(_C)
    assert _bwd(_C, s, scratch=None) == -1 and b"scratch" in err()
    assert _bwd(_C, s, nbytes=16) == -1 and b"scratch" in err()
    for k in ("dop", "dmean", "dv2g", "dcolors"):
        assert _bwd(_C, s, **{k: None}) == -1 and b"NULL argument" in err(), k
    for k in ("dscale", "drot"):
        assert _bwd(_C, s, **{k: None}) == -1 and b"dL_dscale / dL_drot" in err(), k
    assert _bwd(_C, s, drot=FAKE + 4) == -1 and b"aligned" in err()
    assert _bwd(_C, _scene(_C, shs=True), dsh=None) == -1 and b"dL_dsh" in err()
    # M = 16 and degree 3: dL_dsh is written with 16-byte stores
    assert _bwd(_C, _scene(_C, shs=True), dsh=FAKE + 4) == -1 and b"dL_dsh must be 16-byte aligned" in err()
    assert _bwd(_C, s, PN=-1) == -1 and b"PN" in err()
    for k in ("points", "radii", "geom", "image", "pts", "pbin"):
        assert _bwd(_C, s, **{k: None}) == -1 and b"forward state" in err(), k
    bad = _scene(_C)
    bad.P = -1
    assert _bwd(_C, bad) == -1
    o = _C._BackwardOut(dL_dopacity=FAKE, dL_dmean3D=FAKE, dL_dview2gaussian=FAKE, dL_dcolor=FAKE, scratch=FAKE, scratch_bytes=10 ** 6)
    assert _C._lib.gof_integrate_backward(None, 4, FAKE, 1, *[FAKE] * 9, ctypes.byref(o), None) == -1


def test_binding_checks_color_min():
    import torch
    _C = _abi()
    pts = torch.zeros(5, 3)
    with pytest.raises(RuntimeError, match="color_min"):
        _C.integrate_gaussians_to_points_min(None, pts, None, None, None, None, None, 1.0, None, None, None, None, 0.5, 0.5, 0.0, None, 8,
                                             8, None, 0, None, False, False, 0, torch.ones(5), torch.zeros(5, dtype=torch.int32),
                                             torch.ones(5, 4))
