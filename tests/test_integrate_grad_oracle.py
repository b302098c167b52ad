"""CPU: the float64 oracle of the opacity-field query's backward (DESIGN.md 4.11) against central differences of a float64
restatement of one point's integration, and the argument checks of gof_integrate_backward in alpha mode.

The restatement holds the contributor list, the rejects and both clamps fixed, as the definition does; each case is built so
that no decision lies within the finite-difference step of its threshold."""
import ctypes

import numpy as np
import pytest

import _integrate_grad_oracle as igo

VM = np.array([[0.96, -0.05, 0.27, 0.0], [0.08, 0.99, -0.1, 0.0], [-0.26, 0.12, 0.95, 0.0], [0.1, -0.2, 0.3, 1.0]], np.float64)


def _A(v2g, op, p3, vm, depth_fixed=None, clamp_alpha=None, keep=None):
    """A = 1 - prod (1 - alpha_j) in float64 with rx = tx / (tz + 1e-7), ry = ty / (tz + 1e-7), depth = tz."""
    v = np.asarray(v2g, np.float64)
    t3 = np.asarray(p3, np.float64) @ vm[:3, :3] + vm[3, :3]
    den = t3[2] + 1e-7
    rx, ry, d = t3[0] / den, t3[1] / den, t3[2]
    T = 1.0
    for j in range(v.shape[0]):
        r = np.array([rx, ry, 1.0])
        S = np.array([[v[j, 0], v[j, 1], v[j, 2]], [v[j, 1], v[j, 3], v[j, 4]], [v[j, 2], v[j, 4], v[j, 5]]])
        AA, BB = r @ S @ r, 2.0 * (v[j, 6:9] @ r)
        t = -BB / (2 * AA)
        if depth_fixed[j]:
            t = d
        al = op[j] * np.exp(-0.5 * (AA * t * t + BB * t + v[j, 9]))
        if clamp_alpha[j]:
            al = 0.99
        if not keep[j]:
            continue
        T *= 1.0 - al
    return 1.0 - T


def _case(seed, n, depth_clamp=(), alpha_clamp=(), near_reject=()):
    """n Gaussians in front of a point; returns (v2g [n,10] float32, opacity [n] float32, p3 [3] float32)."""
    rng = np.random.default_rng(seed)
    p3 = np.array([0.05, -0.03, 3.0], np.float32)
    t3 = p3.astype(np.float64) @ VM[:3, :3] + VM[3, :3]
    v = np.zeros((n, 10), np.float32)
    op = np.zeros(n, np.float32)
    for j in range(n):
        # a Gaussian centred on the point's ray at depth zc: v2g of an axis-aligned ellipsoid seen from the camera
        # free pairs in front of the point; a depth-clamped one has its centre a little behind it (t* > depth)
        zc = float(t3[2]) + 0.15 if j in depth_clamp else float(t3[2]) * (0.4 + 0.1 * j)
        s = rng.uniform(0.2, 0.4, 3)
        c = np.array([t3[0] / t3[2] * zc, t3[1] / t3[2] * zc, zc]) + rng.normal(0, 0.02, 3)
        S = np.diag(1.0 / s ** 2)
        b = -S @ c
        C = c @ S @ c
        v[j] = [S[0, 0], S[0, 1], S[0, 2], S[1, 1], S[1, 2], S[2, 2], b[0], b[1], b[2], C]
        op[j] = 0.98 if j in alpha_clamp else rng.uniform(0.2, 0.7)
    return v, op, p3


def _check(v, op, p3, expect_zero=(), rtol=2e-6):
    den = float(np.float32(p3 @ VM[:3, 2].astype(np.float32) + np.float32(VM[3, 2]))) + 1e-7
    t3 = p3.astype(np.float64) @ VM[:3, :3] + VM[3, :3]
    rx = np.float32(t3[0] / den)
    ry = np.float32(t3[1] / den)
    dep = np.float32(t3[2])
    o = igo.point(v, op, rx, ry, dep, p3, VM.reshape(16), 1.0)
    assert not o["marginal"]
    n = v.shape[0]
    # the decisions of the oracle's own float evaluation, to hold fixed
    depth_fixed, clamp_alpha, keep = [], [], []
    for j in range(n):
        r = np.array([rx, ry, 1.0])
        S = np.array([[v[j, 0], v[j, 1], v[j, 2]], [v[j, 1], v[j, 3], v[j, 4]], [v[j, 2], v[j, 4], v[j, 5]]], np.float64)
        AA, BB = r @ S @ r, 2.0 * (v[j, 6:9].astype(np.float64) @ r)
        t = -BB / (2 * AA)
        depth_fixed.append(t > dep)
        t = min(t, dep)
        raw = op[j] * np.exp(-0.5 * (AA * t * t + BB * t + v[j, 9]))
        clamp_alpha.append(raw > 0.99)
        keep.append(min(raw, 0.99) >= 1 / 255)
    f = lambda vv, oo, pp: _A(vv, oo, pp, VM, depth_fixed, clamp_alpha, keep)   # noqa: E731
    v64, o64, p64 = v.astype(np.float64), op.astype(np.float64), p3.astype(np.float64)
    for j in range(n):
        for k in range(10):
            h = 1e-6 * max(1.0, abs(v64[j, k]))
            a, b = v64.copy(), v64.copy()
            a[j, k] += h
            b[j, k] -= h
            fd = (f(a, o64, p64) - f(b, o64, p64)) / (2 * h)
            scale = o["mag_g"][j].max() + 1e-12
            assert abs(o["dv2g"][j, k] - fd) <= 1e-5 * scale + rtol * abs(fd), (j, k, o["dv2g"][j, k], fd)
        if j in expect_zero:
            assert np.all(o["dv2g"][j] == 0.0)
    for i in range(3):
        h = 1e-6
        a, b = p64.copy(), p64.copy()
        a[i] += h
        b[i] -= h
        fd = (f(v64, o64, a) - f(v64, o64, b)) / (2 * h)
        assert abs(o["dpts"][i] - fd) <= 1e-5 * (o["mag_pts"].max() + 1e-12) + rtol * abs(fd), (i, o["dpts"][i], fd)
    return o


def test_free_pairs():
    v, op, p3 = _case(1, 5)
    o = _check(v, op, p3)
    assert o["A"] > 0.1


def test_depth_clamp():
    v, op, p3 = _case(2, 4, depth_clamp=(1, 3))
    _check(v, op, p3)


def test_alpha_clamp_has_exact_zero_derivative():
    v, op, p3 = _case(3, 3, alpha_clamp=(1,))
    v[1, 9] -= 0.5   # exp(power) > 1 / 0.98 near the centre: op exp(power) > 0.99
    _check(v, op, p3, expect_zero=(1,))


def test_near_reject_alpha_is_kept():
    v, op, p3 = _case(4, 3)
    op[2] = np.float32(1.0 / 255.0 * 1.5)   # alpha a little above the reject threshold where the power is ~0
    o = _check(v, op, p3)
    assert np.abs(o["dv2g"][2]).max() > 0.0


def test_dL_dA_scales_linearly():
    v, op, p3 = _case(5, 4)
    vm = VM.reshape(16)
    a = igo.point(v, op, 0.01, -0.01, 3.0, p3, vm, 1.0)
    b = igo.point(v, op, 0.01, -0.01, 3.0, p3, vm, -2.5)
    np.testing.assert_allclose(b["dv2g"], -2.5 * a["dv2g"], rtol=1e-12, atol=0)
    np.testing.assert_allclose(b["dpts"], -2.5 * a["dpts"], rtol=1e-12, atol=0)


# ---- the C ABI's argument checks ----
def _abi():
    try:
        from diff_gaussian_rasterization import _C
    except ImportError as e:   # the library is built by __graft_entry__.build()
        pytest.skip(str(e))
    return _C


def test_scratch_bytes():
    _C = _abi()
    f = _C._lib.gof_integrate_backward_scratch_bytes
    assert f(0) == 0
    assert f(1) == 512
    assert f(1000) == 2 * ((12000 + 255) // 256 * 256)


FAKE = 0x1000


def _alpha_call(_C, s, **out):
    """gof_integrate_backward in alpha mode (dL_dalpha, no dL_dcolor_integrated) with the forward state at FAKE and the Gaussian
    gradients and a large scratch at FAKE, updated by `out` (field name -> pointer or None)."""
    o = dict(dL_dopacity=FAKE, dL_dmean3D=FAKE, dL_dscale=FAKE, dL_drot=FAKE, dL_dview2gaussian=FAKE, dL_dcov3D=FAKE,
             scratch=FAKE, scratch_bytes=10 ** 6)
    o.update(out)
    o = _C._BackwardOut(**o)
    return _C._lib.gof_integrate_backward(ctypes.byref(s), 4, FAKE, 1, *[FAKE] * 6, FAKE, None, FAKE, ctypes.byref(o), None)


def _alpha_scene(_C):
    s = _C._Scene()
    s.P, s.width, s.height, s.tan_fovx, s.tan_fovy = 10, 32, 32, 0.5, 0.5
    for name in ("means3D", "opacities", "viewmatrix", "projmatrix", "background", "colors_precomp", "scales", "rotations"):
        setattr(s, name, FAKE)
    return s


def test_scratch_in_out_and_scene_are_checked():
    _C = _abi()
    s = _alpha_scene(_C)
    # a NULL or short scratch is refused before any work
    rc_null = _alpha_call(_C, s, scratch=None)
    rc_short = _alpha_call(_C, s, scratch_bytes=16)
    assert rc_null == rc_short == -1   # GOF_E_INVALID
    assert b"scratch" in _C._lib.gof_last_error()
    s.P = -1
    assert _alpha_call(_C, s) != 0


def test_misaligned_rotation_gradient_in_out_is_refused():
    """dL_drot is written with 16-byte stores: a pointer that is not 16-byte aligned fails with GOF_E_INVALID before any work."""
    _C = _abi()
    assert _alpha_call(_C, _alpha_scene(_C), dL_drot=FAKE + 4) == -1
    assert b"aligned" in _C._lib.gof_last_error()


def test_out_is_checked():
    """A NULL out, and any output this backward cannot produce, fail with GOF_E_INVALID and the field's name."""
    _C = _abi()
    s = _alpha_scene(_C)
    assert _C._lib.gof_integrate_backward(ctypes.byref(s), 4, FAKE, 1, *[FAKE] * 6, FAKE, None, FAKE, None, None) == -1
    assert b"out is NULL" in _C._lib.gof_last_error()
    for name in ("dL_dmean2D", "dens_sum", "dens_max", "sh_rgb", "sh_hdr", "dL_dviewmatrix", "dL_dcampos", "dL_dtan_fov"):
        assert _alpha_call(_C, s, **{name: FAKE}) == -1, name
        assert f"out->{name} must be NULL".encode() in _C._lib.gof_last_error(), name
