"""GPU: every Gaussian's gradient, stage by stage, against the fp64 oracle fed with this library's own intermediate values.

The view2gaussian chain rule multiplies an ulp of dL_dview2gaussian by ~1/scale^2 (DESIGN.md 4.1), so the gradients of the
whole backward can only be compared per tensor and loosely.  The two backward kernels split exactly there, and each is
compared here on its own, per Gaussian and per component, from inputs that are not ill-conditioned:

Stage A, the blend backward (render_bwd.cu).  The oracle's blend backward runs from THIS library's forward state
(_C.export_state: tile lists, ranges, 2D means, conics, colours, view2gaussian, accum_alpha, n_contrib) with the same
dL_dpix, and returns next to its gradients the error scales `mag` and `marginal` (tests/_grad_bounds.py).  For every Gaussian
and every component of dL_dcolors[3], dL_dmeans2D[3], dL_dopacity and dL_dview2gaussian[10]:

    |gpu - oracle|  <=  c * 2^-24 * (1 + L) * mag  +  marginal,      L = the view's longest walk, c = min(8, 2^12 / (1 + L))

and at most SHARE_MARGINAL of the visible Gaussians may carry marginal mass.  Observed on an H100 80GB HBM3 (700 W power limit):

  scene             L     largest |gpu - oracle - marginal| / (2^-24 (1 + L) mag)   share with marginal mass
  sh_deg0..3        319-357   0.034 - 0.057                                         0
  c1                350       0.060                                                 5.0e-4
  precomp_bg_mip    249       0.043                                                 1.1e-3
  screen_filling    150       0.019                                                 0
  camera_inside     281       0.019                                                 0
  stacked_interior  1005      0.021                                                 0
  stacked_border    888       0.039                                                 0
  stacked_bg        1019      0.036                                                 0
  c2_v3             816       0.068                                                 1.0e-3
  c3_v5             828       0.077                                                 1.7e-3
  bucket_1 / 33 / 4097  1 / 3 / 119   0.12 / 1.47 / 0.082                           0

A pair near a blend threshold exempts every pair in front of it at its pixel; at C2 / C3 each such pixel has a walk of hundreds
of entries, which is why the share there reaches 1.0e-3 / 1.7e-3.

Stage B, the per-Gaussian chain rule and SH backward (k_preprocess_backward, preprocess.cu).  The oracle's
preprocess backward runs from the GPU's own float dL_dview2gaussian and dL_dcolors (and clamp flags), so oracle and kernel start
from identical floats and both evaluate the view2gaussian part in double:
  - dL_dscales, dL_drotations and the view2gaussian part of dL_dmeans3D: within 2 ulp of the oracle value, plus 2^-30 of the
    largest |value| in the Gaussian's row, plus C_CHAIN * 2^-53 of the magnitude of the ten terms dL_dv2g_k * J_k that the
    double chain rule sums (chain_mag): the kernel's double FMAs and the oracle's separate multiplies and adds differ by a few
    2^-53 of those terms, and where they cancel by ~1e9 that is more than an ulp of the result.  Largest need for C_CHAIN
    observed: 44.8 (dL_drot, C3), 7.9 (dL_drot, C2), <= 2.8 elsewhere;
  - dL_dsh and the SH part of dL_dmeans3D, evaluated in float by the kernel: within C_SH * 2^-24 of their magnitude --
    |dL_dRGB_c| for dL_dsh, the SH expression with absolute values (float64, sh_dmean_mag) for dL_dmeans3D.  The oracle is
    linear in its inputs: one call with dL_dcolor = 0 and one with dL_dv2g = 0 separate the two parts of dL_dmeans3D.
    Largest error / (2^-24 magnitude) observed: 5.3 (dL_dsh), 0.96 (dL_dmeans3D);
  - Gaussians this view does not see: exact zeros in every gradient."""
import numpy as np
import pytest
import torch

import _grad_bounds as gb
import _util
import gof_dp
import gof_oracle
import gof_synth
from test_gpu_bwd_walk import stacked_scene

pytestmark = pytest.mark.gpu

C_CHAIN = 256.0          # 4x the largest need observed (44.8, dL_drot at C3), rounded up to a power of two
C_SH = 32.0              # 4x the largest need observed (5.3, dL_dsh at C2), rounded up to a power of two
SHARE_MARGINAL = 4e-3    # at most this share of the visible Gaussians may carry marginal mass (observed: <= 1.7e-3)

SH_C1 = 0.4886025119029199
SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
         1.445305721320277, -0.5900435899266435)


def _inside_scene():
    cam = gof_synth.make_camera(160, 96, view=9, radius=0.8)
    return cam, gof_synth.make_gaussians(6000, 51, cam.focal_x, sigma_px=3.0)


# name -> (scene factory, options).  The scenes of test_gpu_oracle and test_gpu_bwd_walk, a stacked scene with a background
# (the background term of the blend backward is applied per pair, across batches), C2 / C3, and P in {1, 33, 4097} through a
# GradBucket (partial warps of k_preprocess_backward's staged copy-out)
SCENES = {
    **{f"sh_deg{d}": (lambda d=d: gof_synth.make_scene(dict(P=6000, width=208, height=120, seed=20 + d, sh_degree=d), view=d * 5), {})
       for d in range(4)},
    "c1": (lambda: gof_synth.make_scene("C1", view=0), {}),
    "precomp_bg_mip": (lambda: gof_synth.make_scene(dict(P=5000, width=203, height=117, seed=31), view=11),
                       dict(kernel_size=0.1, scale_modifier=0.7, bg=(1.0, 1.0, 1.0), colors_seed=5)),
    "screen_filling": (lambda: gof_synth.make_scene(dict(P=3000, width=96, height=96, seed=41, sigma_px=20.0), view=3), {}),
    "camera_inside": (_inside_scene, {}),
    "stacked_interior": (lambda: stacked_scene(150, 90, 1500, 900, 7, (37, 21)), {}),
    "stacked_border": (lambda: stacked_scene(147, 83, 800, 900, 8, (145, 81)), {}),
    "stacked_bg": (lambda: stacked_scene(150, 90, 1500, 900, 9, (70, 40)), dict(bg=(0.3, 0.6, 0.9))),
    "c2_v3": (lambda: gof_synth.make_scene("C2", view=3), {}),
    "c3_v5": (lambda: gof_synth.make_scene("C3", view=5), {}),
    **{f"bucket_{P}": (lambda P=P: gof_synth.make_scene(dict(P=P, width=320, height=208, seed=17), view=4), dict(bucket=True))
       for P in (1, 33, 4097)},
}


def run(name):
    """GPU forward + backward of scene `name` with a seeded dL_dpix over all 9 channels; the exported forward state; the
    oracle scene.  numpy throughout."""
    from diff_gaussian_rasterization import _C
    make, opt = SCENES[name]
    cam, gs = make()
    dev = torch.device("cuda")
    P, W, H = gs["means3D"].shape[0], cam.image_width, cam.image_height
    colors = None
    if "colors_seed" in opt:
        colors = torch.rand(P, 3, generator=torch.Generator().manual_seed(opt["colors_seed"]))
    bg = opt.get("bg", (0.0, 0.0, 0.0))
    ks, sm = opt.get("kernel_size", 0.0), opt.get("scale_modifier", 1.0)
    fa = _util.fwd_args(cam, gs, dev, kernel_size=ks, scale_modifier=sm, bg=bg, colors_precomp=colors)
    R, _color, radii, geom, binning, img = _C.rasterize_gaussians(*fa)
    st = {k: v.cpu().numpy() for k, v in _C.export_state(P, W, H, R, geom, binning, img, radii).items()}
    dL = torch.randn(9, H, W, generator=torch.Generator().manual_seed(1000 + list(SCENES).index(name)))
    out = gof_dp.GradBucket(P, gs["shs"].shape[1], dev).views if opt.get("bucket") else None
    grads = _C.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, dL.to(dev)), _out=out)
    torch.cuda.synchronize()
    names = ["dmeans2D", "dcolors", "dopacity", "dmeans3D", "dcov3D", "dsh", "dscales", "drot", "dv2g"]
    got = {n: (None if g is None else g.detach().cpu().numpy()) for n, g in zip(names, grads)}
    sc = gof_oracle.Scene(W, H, cam.tanfovx, cam.tanfovy, cam.world_view_transform, cam.full_proj_transform, cam.camera_center,
                          gs["means3D"], gs["opacities"], scales=gs["scales"], rotations=gs["rotations"],
                          shs=None if colors is not None else gs["shs"], colors_precomp=colors, sh_degree=gs["sh_degree"],
                          kernel_size=ks, scale_modifier=sm, bg=bg)
    return dict(got=got, st=st, radii=radii.cpu().numpy(), dL=dL.numpy(), sc=sc)


def stage_a(r):
    """(ratio [P,17], L, share of visible Gaussians with marginal mass)."""
    st, sc = r["st"], r["sc"]
    d = gof_oracle.render_backward(sc, st, st["point_list"], st["ranges"], st["accum_alpha"], st["n_contrib"], r["dL"], bounds=True)
    g = r["got"]
    L = int(st["n_contrib"][0].max())
    ratio = gb.blend_ratio(gb.stack17(g["dcolors"], g["dmeans2D"], g["dopacity"], g["dv2g"]), gb.oracle17(d), d["mag"], d["marginal"], L)
    vis = r["radii"] > 0
    share = float((d["marginal"][vis].sum(axis=1) > 0).mean()) if vis.any() else 0.0
    return ratio, L, share


def _ulp(x):
    return np.spacing(np.abs(x).astype(np.float32)).astype(np.float64)


def chain_mag(sc, radii, clamped, dv2g):
    """{output: sum_k |J_k| |dL_dv2g_k|}: the magnitudes of the ten terms of the linear map dL_dv2g -> (dL_dscale, dL_drot, the
    view2gaussian part of dL_dmeans3D), one oracle call per column J_k of its Jacobian.  A double evaluation of the map is
    exact to a few 2^-53 of this, whatever the ten terms cancel to."""
    P = dv2g.shape[0]
    zc = np.zeros((P, 3), np.float32)
    mag = dict(dL_dscale=0.0, dL_drot=0.0, dL_dmean3D=0.0)
    for k in range(10):
        e = np.zeros((P, 10), np.float32)
        e[:, k] = 1.0
        col = gof_oracle.preprocess_backward(sc, radii, clamped, zc, e)
        w = np.abs(dv2g[:, k:k + 1].astype(np.float64))
        for n in mag:
            mag[n] = mag[n] + np.abs(col[n].astype(np.float64)) * w
    return mag


def _chain_ratio(gpu, ora, jmag, extra=0.0, need=None, key=None):
    """|gpu - ora| in units of the stage-B allowance 2 ulp(ora) + 2^-30 max|row| + C_CHAIN 2^-53 jmag (+ extra); passes iff
    <= 1.  `need[key]`, if given, receives the smallest C_CHAIN that would pass."""
    gpu, ora = np.asarray(gpu, np.float64), np.asarray(ora, np.float64)
    fixed = 2.0 * _ulp(ora) + 2.0 ** -30 * np.abs(ora).max(axis=1, keepdims=True) + extra
    err = np.abs(gpu - ora)
    with np.errstate(divide="ignore", invalid="ignore"):
        if need is not None:
            left = np.maximum(err - fixed, 0.0)
            need[key] = float(np.where(left > 0, left / (2.0 ** -53 * jmag), 0.0).max()) if left.size else 0.0
        return float(np.where(err > 0, err / (fixed + C_CHAIN * 2.0 ** -53 * jmag), 0.0).max()) if err.size else 0.0


def sh_dmean_mag(means, campos, shs, D, dRGB):
    """The SH part of dL_dmeans3D (backward.cu:45-139 + dnormvdv) with every sum and difference replaced by the sum of the
    absolute values of its operands, in float64: [P,3]."""
    m = np.asarray(means, np.float64)
    dvec = m - np.asarray(campos, np.float64).reshape(1, 3)
    dox, doy, doz = dvec[:, 0:1], dvec[:, 1:2], dvec[:, 2:3]
    nrm = np.sqrt((dvec ** 2).sum(axis=1, keepdims=True))
    x, y, z = np.abs(dox / nrm), np.abs(doy / nrm), np.abs(doz / nrm)
    sh = np.abs(np.asarray(shs, np.float64))
    S = lambda k: sh[:, k, :]   # noqa: E731  [P,3]
    a1, a2, a3 = abs(SH_C1), [abs(c) for c in SH_C2], [abs(c) for c in SH_C3]
    zero = np.zeros_like(S(0))
    mx, my, mz = zero.copy(), zero.copy(), zero.copy()
    if D > 0:
        mx, my, mz = a1 * S(3), a1 * S(1), a1 * S(2)
        if D > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            mx = mx + a2[0] * y * S(4) + a2[2] * 2 * x * S(6) + a2[3] * z * S(7) + a2[4] * 2 * x * S(8)
            my = my + a2[0] * x * S(4) + a2[1] * z * S(5) + a2[2] * 2 * y * S(6) + a2[4] * 2 * y * S(8)
            mz = mz + a2[1] * y * S(5) + a2[2] * 4 * z * S(6) + a2[3] * x * S(7)
            if D > 2:
                mx = mx + (a3[0] * S(9) * 6 * xy + a3[1] * S(10) * yz + a3[2] * S(11) * 2 * xy + a3[3] * S(12) * 6 * xz +
                           a3[4] * S(13) * (3 * xx + 4 * zz + yy) + a3[5] * S(14) * 2 * xz + a3[6] * S(15) * 3 * (xx + yy))
                my = my + (a3[0] * S(9) * 3 * (xx + yy) + a3[1] * S(10) * xz + a3[2] * S(11) * (3 * yy + 4 * zz + xx) +
                           a3[3] * S(12) * 6 * yz + a3[4] * S(13) * 2 * xy + a3[5] * S(14) * 2 * yz + a3[6] * S(15) * 6 * xy)
                mz = mz + (a3[1] * S(10) * xy + a3[2] * S(11) * 8 * yz + a3[3] * S(12) * 3 * (2 * zz + xx + yy) +
                           a3[4] * S(13) * 8 * xz + a3[5] * S(14) * (xx + yy))
    dr = np.abs(np.asarray(dRGB, np.float64))
    ddx, ddy, ddz = (mx * dr).sum(1, keepdims=True), (my * dr).sum(1, keepdims=True), (mz * dr).sum(1, keepdims=True)
    s2 = nrm ** 2
    ax, ay, az = np.abs(dox), np.abs(doy), np.abs(doz)
    inv = 1.0 / (s2 * nrm)
    return np.concatenate([((s2 + ax * ax) * ddx + ay * ax * ddy + az * ax * ddz) * inv,
                           (ax * ay * ddx + (s2 + ay * ay) * ddy + az * ay * ddz) * inv,
                           (ax * az * ddx + ay * az * ddy + (s2 + az * az) * ddz) * inv], axis=1)


def stage_b(r, need=None):
    """{output: largest ratio to its allowance (<= 1 passes)}, after asserting exact zeros for invisible Gaussians.  `need`, if
    given, receives the smallest C_CHAIN / C_SH that would pass."""
    g, st, sc, radii = r["got"], r["st"], r["sc"], r["radii"]
    inv = radii <= 0
    for n in ("dmeans2D", "dcolors", "dopacity", "dmeans3D", "dsh", "dscales", "drot", "dv2g"):
        if g[n] is not None and g[n].size:
            assert (g[n][inv] == 0).all(), n
    vis = ~inv
    if not vis.any():
        return {}
    dv2g, dcol = g["dv2g"], g["dcolors"]
    full = gof_oracle.preprocess_backward(sc, radii, st["clamped"], dcol, dv2g)
    v_only = gof_oracle.preprocess_backward(sc, radii, st["clamped"], np.zeros_like(dcol), dv2g)
    jm = {k: v[vis] for k, v in chain_mag(sc, radii, st["clamped"], dv2g).items()}
    out = {"dscales": _chain_ratio(g["dscales"][vis], full["dL_dscale"][vis], jm["dL_dscale"], need=need, key="dscales"),
           "drot": _chain_ratio(g["drot"][vis], full["dL_drot"][vis], jm["dL_drot"], need=need, key="drot")}
    V = v_only["dL_dmean3D"][vis].astype(np.float64)
    if sc.arr["shs"] is None:
        out["dmeans3D"] = _chain_ratio(g["dmeans3D"][vis], V, jm["dL_dmean3D"], need=need, key="dmeans3D")
        return out
    s_only = gof_oracle.preprocess_backward(sc, radii, st["clamped"], dcol, np.zeros_like(dv2g))
    dRGB = np.where(st["clamped"].astype(bool), 0.0, dcol.astype(np.float64))[vis]
    # dL_dsh: a product w_k(dir) * dL_dRGB_c per element, the weight evaluated in float
    err = np.abs(g["dsh"][vis].astype(np.float64) - s_only["dL_dsh"][vis])
    allow = gb.EPS * np.abs(dRGB)[:, None, :]
    with np.errstate(divide="ignore", invalid="ignore"):
        out["dsh"] = float(np.where(err > 0, err / (C_SH * allow), 0.0).max())
        if need is not None:
            need["dsh_C_SH"] = out["dsh"] * C_SH
    # dL_dmeans3D = float(view2gaussian part) + float SH part, rounded once more
    msh = sh_dmean_mag(sc.arr["means3D"][vis], sc.arr["cam_pos"], sc.arr["shs"][vis], sc.D, dRGB)
    gm = g["dmeans3D"][vis]
    S = s_only["dL_dmean3D"][vis].astype(np.float64)
    out["dmeans3D"] = _chain_ratio(gm, V + S, jm["dL_dmean3D"], extra=C_SH * gb.EPS * msh + _ulp(gm), need=need, key="dmeans3D")
    if need is not None:   # the SH part's own constant, with the view2gaussian part's allowance at C_CHAIN
        left = np.maximum(np.abs(gm - V - S) - 2.0 * _ulp(V) - 2.0 ** -30 * np.abs(V).max(axis=1, keepdims=True)
                          - C_CHAIN * 2.0 ** -53 * jm["dL_dmean3D"] - _ulp(gm), 0.0)
        with np.errstate(divide="ignore", invalid="ignore"):
            need["dmeans3D_C_SH"] = float(np.where(left > 0, left / (gb.EPS * msh), 0.0).max())
    return out


@pytest.mark.parametrize("name", list(SCENES))
def test_gradients_stage_by_stage_per_gaussian(name):
    r = run(name)
    failures = []
    # stage A
    ratio, L, share = stage_a(r)
    worst, c = (float(ratio.max()) if ratio.size else 0.0), gb.blend_constant(L)
    if not worst <= c:
        i, k = np.unravel_index(np.argmax(ratio), ratio.shape)
        failures.append(f"stage A: Gaussian {i} component {k}: ratio {worst:.3g} > c {c:.3g} (L = {L}); "
                        f"{int((ratio > c).any(axis=1).sum())} Gaussians out of bound")
    if not share <= SHARE_MARGINAL:
        failures.append(f"stage A: {share:.2e} of the visible Gaussians carry marginal mass")
    # stage B
    res = stage_b(r)
    bad = {k: v for k, v in res.items() if not v <= 1.0}
    if bad:
        failures.append(f"stage B: {bad}")
    assert not failures, (name, failures)
