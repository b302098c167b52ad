"""CPU: the float64 camera-gradient oracle (tests/_camera_oracle.py) against central differences (the C ABI's checks are in
test_backward_abi.py).

The oracle's camera terms are Jacobian-vector products of the loss L = sum_g <dL_dv2g_g, view2gaussian_g(vm)> +
<dL_dRGB_g, rgb_g(campos)> (dL_dRGB masked by the clamp flags), so for any direction u, <dL_dvm, u> and <dL_dcampos, u>
must match (L(x + h u) - L(x - h u)) / 2h of a float64 evaluation of view2gaussian and of the SH colour."""
import numpy as np
import pytest

import _camera_oracle as co
import gof_oracle
import gof_synth


def _scene(D, precomp=None, seed=0, P=96):
    cam, gs = gof_synth.make_scene(dict(P=P, width=96, height=64, seed=60 + seed, sh_degree=D), view=7 * seed + 3)
    colors = np.random.default_rng(seed).random((P, 3)).astype(np.float32) if precomp == "colors" else None
    sc = gof_oracle.scene_from_synth(cam, gs)
    if colors is not None:
        sc = gof_oracle.Scene(cam.image_width, cam.image_height, cam.tanfovx, cam.tanfovy, cam.world_view_transform,
                              cam.full_proj_transform, cam.camera_center, gs["means3D"], gs["opacities"], scales=gs["scales"],
                              rotations=gs["rotations"], colors_precomp=colors, sh_degree=D)
    g = gof_oracle.preprocess(sc)
    if precomp == "v2g":   # the record the forward computed, handed back in as view2gaussian_precomp
        sc.arr["v2g_precomp"] = np.ascontiguousarray(g["view2gaussian"])
    return sc, g


def _upstream(P, seed):
    rng = np.random.default_rng(100 + seed)
    return rng.standard_normal((P, 3)).astype(np.float32), rng.standard_normal((P, 10)).astype(np.float32)


def _check_jvp(f, x0, grad, rng, n_dirs=4, free=None):
    """<grad, u> against central differences of f at x0 along random unit directions u (zero where `free` is False)."""
    for _ in range(n_dirs):
        u = rng.standard_normal(x0.shape)
        if free is not None:
            u = np.where(free, u, 0.0)
        u /= np.linalg.norm(u)
        h = 1e-6 * max(1.0, float(np.abs(x0).max()))
        fd = (f(x0 + h * u) - f(x0 - h * u)) / (2 * h)
        jvp = float(grad @ u)
        scale = max(abs(fd), abs(jvp), 1e-3 * float(np.abs(grad).sum()), 1e-12)
        assert abs(jvp - fd) <= 1e-5 * scale, (jvp, fd)


CASES = [(D, None) for D in range(4)] + [(3, "v2g"), (2, "colors"), (1, "v2g")]


@pytest.mark.parametrize("D,precomp", CASES)
def test_oracle_jvp_matches_central_differences(D, precomp):
    seed = 4 * D + (precomp is not None) * (2 if precomp == "v2g" else 3)
    sc, g = _scene(D, precomp, seed)
    P = sc.P
    vis = g["radii"] > 0
    assert vis.sum() > 10
    dcol, dv2g = _upstream(P, seed)
    t = co.terms(sc, g["radii"], g["clamped"], dcol, dv2g)
    assert (t[~vis] == 0).all()
    dvm, dcp = co.assemble(t.sum(axis=0))
    assert (dvm[3::4] == 0).all()
    rng = np.random.default_rng(7 + seed)
    a = sc.arr

    if precomp == "v2g":
        assert (dvm == 0).all()          # view2gaussian given: it does not depend on the view matrix
    else:
        m, s, q, dv = a["means3D"][vis], a["scales"][vis], a["rotations"][vis], dv2g[vis].astype(np.float64)
        f_vm = lambda vm: float((co.view2gaussian(vm, m, s, q) * dv).sum())   # noqa: E731
        free = np.ones(16, bool)
        free[3::4] = False
        _check_jvp(f_vm, a["viewmatrix"].astype(np.float64).ravel(), dvm, rng, free=free)
        # and the fourth row of the view matrix really is not read
        e = np.zeros(16)
        e[3::4] = 1.0
        vm0 = a["viewmatrix"].astype(np.float64).ravel()
        assert f_vm(vm0 + 0.1 * e) == f_vm(vm0)

    if precomp == "colors":
        assert (dcp == 0).all()
    else:
        keep = np.where(g["clamped"][vis].astype(bool), 0.0, dcol[vis].astype(np.float64))
        m, sh = a["means3D"][vis], a["shs"][vis]
        f_cp = lambda cp: float((co.sh_rgb(m, cp, sh, D) * keep).sum())   # noqa: E731
        if D == 0:
            assert (dcp == 0).all()      # a constant colour does not depend on the direction
        else:
            _check_jvp(f_cp, a["cam_pos"].astype(np.float64), dcp, rng)


def test_view2gaussian_restatement_matches_the_oracle_forward():
    """The float64 view2gaussian the differences are taken of is the record the oracle's forward computes (to float
    rounding, amplified by 1/scale^2 like every view2gaussian evaluation)."""
    sc, g = _scene(3, None, 1)
    vis = g["radii"] > 0
    a = sc.arr
    v = co.view2gaussian(a["viewmatrix"].ravel(), a["means3D"][vis], a["scales"][vis], a["rotations"][vis])
    ref = g["view2gaussian"][vis].astype(np.float64)
    scale = np.abs(ref).max(axis=1, keepdims=True)
    assert (np.abs(v - ref) <= 1e-4 * scale).all()


def test_sh_rgb_restatement_matches_the_oracle_forward():
    sc, g = _scene(3, None, 2)
    vis = g["radii"] > 0
    a = sc.arr
    rgb = np.maximum(co.sh_rgb(a["means3D"][vis], a["cam_pos"], a["shs"][vis], 3), 0.0)
    assert np.allclose(rgb, g["rgb"][vis], rtol=0, atol=1e-5)

