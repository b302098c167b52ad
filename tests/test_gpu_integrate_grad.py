"""GPU: the backward of the opacity-field query (DESIGN.md 4.11) against the float64 oracle, fed with this library's own forward
state (_C.export_state of the query: tile lists, ranges, view2gaussian, effective opacity) and the query's own projection.

For every point that projects, each component of dL/dpoints3D, and for every visible Gaussian, each component of
dL/dview2gaussian and dL/dopacity:

    |gpu - oracle|  <=  C * 2^-24 * mag  +  2 ulp(oracle)  +  allow

mag (the oracle's) is the sum of the magnitudes of the terms, each times 1 + sum_i 1 / (1 - alpha_i) of its point.  allow is what
the decisions within 8 ulp of a threshold (tests/integrate_grad_oracle) can change if the device takes them the other way: the
term that may appear or vanish, and the other terms of that point scaled by the change of its T.  Only a point at which a
transmittance decision of pass 1 may flip (every later decision of that ray with it) is left out, with every Gaussian of its
tile.  The rest of the
chain (dL/dmeans3D, dL/dscales, dL/drotations) is k_preprocess_backward, run unchanged: it is compared as stage B of
test_gpu_grad_stagewise, from the GPU's own float dL/dview2gaussian.  At most SHARE_MARGINAL of the projected points may be
left out, and at most SHARE_MARGINAL_G of the visible Gaussians; the test prints the shares
it saw.  The forward's alpha of every point with no marginal decision is also compared with the oracle's float restatement of it, which
confirms that the oracle rebuilt the forward's contributor lists and decisions."""
import numpy as np
import pytest
import torch

import _integrate_grad_oracle as igo
import _integrate_scenes as isc
import gof_oracle
import gof_synth
from test_gpu_grad_stagewise import _chain_ratio, chain_mag

pytestmark = pytest.mark.gpu

C = 64.0
SHARE_MARGINAL = 0.05     # of the projected points
SHARE_MARGINAL_G = 0.1    # of the visible Gaussians (observed: <= 0.024), except in cap_1024, see SCENES


def _ulp(x):
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(np.float32)).astype(np.float64)


def _args(cam, gs, pts, dev, kernel_size=0.0, v2g_precomp=None):
    e = torch.Tensor([])
    H, W = cam.image_height, cam.image_width
    return (torch.zeros(3, device=dev), pts.to(dev), gs["means3D"].to(dev), e, gs["opacities"].to(dev), gs["scales"].to(dev),
            gs["rotations"].to(dev), 1.0, e, e if v2g_precomp is None else v2g_precomp.to(dev), cam.world_view_transform.to(dev),
            cam.full_proj_transform.to(dev), cam.tanfovx, cam.tanfovy, kernel_size, torch.zeros((H, W, 2), device=dev), H, W,
            gs["shs"].to(dev), gs["sh_degree"], cam.camera_center.to(dev), False, False)


def _backward(ia, state, dL):
    from diff_gaussian_rasterization import _C
    (bg, p3, m3, col, op, sc, rot, sm, cov, v2g, vm, pm, tfx, tfy, ks, sub, H, W, sh, deg, cp, _pf, dbg) = ia
    R, _color, _a, _c, radii, geom, binning, img, pts, pbin = state
    return _C.integrate_gaussians_to_points_backward(bg, p3, m3, radii, col, sc, rot, sm, cov, v2g, vm, pm, tfx, tfy, ks, sub, H, W,
                                                     sh, deg, cp, dL, R, geom, binning, img, pts, pbin, dbg)


def run(cam, gs, pts, seed=0, kernel_size=0.0):
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda")
    P, PN, W, H = gs["means3D"].shape[0], pts.shape[0], cam.image_width, cam.image_height
    ia = _args(cam, gs, pts, dev, kernel_size)
    state = _C.integrate_gaussians_to_points_state(*ia)
    dL = torch.randn(PN, generator=torch.Generator().manual_seed(seed))
    g = _backward(ia, state, dL.to(dev))
    torch.cuda.synchronize()
    assert g[7:] == (None, None)   # alpha mode: no dL_dcolors, no dL_dsh
    got = dict(zip(("dpts", "dopacity", "dmeans3D", "dscales", "drot", "dcov3D", "dv2g"), (t.cpu().numpy() for t in g[:7])))
    R, _color, alpha, _ci, radii, geom, binning, img, _pts, _pbin = state
    sc = gof_oracle.Scene(W, H, cam.tanfovx, cam.tanfovy, cam.world_view_transform, cam.full_proj_transform, cam.camera_center,
                          gs["means3D"], gs["opacities"], scales=gs["scales"], rotations=gs["rotations"], shs=gs["shs"],
                          sh_degree=gs["sh_degree"], kernel_size=kernel_size)
    st = {k: v.cpu().numpy() for k, v in _C.export_state(P, W, H, R, geom, binning, img, radii).items()}
    xy, depth, ok = gof_oracle.project_points(sc, pts)
    order = igo.view_order(xy, ok, W)
    o = igo.view(W, H, cam.tanfovx, cam.tanfovy, cam.world_view_transform.numpy(), pts.numpy()[order], xy[order], depth[order],
                 ok[order], st, dL.numpy()[order])
    inv = np.empty_like(order)
    inv[order] = np.arange(PN)
    for k in ("alpha", "dpts", "mag_pts", "allow_pts", "marg_pt", "n_list"):
        o[k] = o[k][inv]
    return dict(got=got, o=o, ok=ok, alpha=alpha.cpu().numpy(), radii=radii.cpu().numpy(), st=st, sc=sc, P=P, PN=PN,
                scales=gs["scales"].numpy())


def check(r, name, share_g_max=SHARE_MARGINAL_G):
    got, o, ok = r["got"], r["o"], r["ok"]
    out = {}
    # points that do not project: exact zeros
    assert np.all(got["dpts"][~ok] == 0.0), name
    cmp_pt = ok & (o["marg_pt"] != 2)       # points whose possible decision flips the allowance covers
    exact = ok & (o["marg_pt"] == 0)
    share_pt = float((o["marg_pt"][ok] == 2).mean()) if ok.any() else 0.0
    assert share_pt <= SHARE_MARGINAL, (name, share_pt)
    # the forward's alpha: same lists and decisions, alphas apart only by the host's and the device's expf (a few ulp each)
    da = np.abs(r["alpha"][exact].astype(np.float64) - o["alpha"][exact].astype(np.float64))
    assert np.all(da <= 8.0 * 2.0 ** -24 * (1.0 + o["n_list"][exact])), (name, "alpha", float(da.max()) if da.size else 0.0)
    # the point gradient
    err = np.abs(got["dpts"][cmp_pt] - o["dpts"][cmp_pt])
    left = np.maximum(err - o["allow_pts"][cmp_pt], 0.0)
    allow = C * 2.0 ** -24 * o["mag_pts"][cmp_pt] + 2 * _ulp(o["dpts"][cmp_pt]) + 1e-30
    out["point"] = float((left / allow).max()) * C if err.size else 0.0
    assert np.all(left <= allow), (name, "points3D", out["point"])
    # the Gaussian side: dL/dview2gaussian and dL/dopacity of every Gaussian not left out
    vis = r["radii"] > 0
    gsel = vis & ~o["marg_g"]
    share_g = float(o["marg_g"][vis].mean()) if vis.any() else 0.0
    share_allow = float((o["allow_g"][vis] > 0).any(axis=1).mean()) if vis.any() else 0.0
    assert share_g <= share_g_max, (name, "share of Gaussians left out", share_g)
    err = np.abs(got["dv2g"][gsel] - o["dv2g"][gsel])
    left = np.maximum(err - o["allow_g"][gsel], 0.0)
    allow = C * 2.0 ** -24 * o["mag_g"][gsel] + 2 * _ulp(o["dv2g"][gsel]) + 1e-30
    out["v2g"] = float((left / allow).max()) * C if err.size else 0.0
    assert np.all(left <= allow), (name, "view2gaussian", out["v2g"])
    op = r["st"]["conic_opacity"][:, 3].astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        ora_op = np.where(vis, o["dv2g"][:, 9] * (-2.0 / op), 0.0)
        mag_op = np.where(vis, o["mag_g"][:, 9] * (2.0 / np.abs(op)), 0.0)
        allow_op = np.where(vis, o["allow_g"][:, 9] * (2.0 / np.abs(op)), 0.0)
    err = np.abs(got["dopacity"][:, 0][gsel] - ora_op[gsel])
    left = np.maximum(err - allow_op[gsel], 0.0)
    allow = C * 2.0 ** -24 * mag_op[gsel] + 4 * _ulp(ora_op[gsel]) + 1e-30
    assert np.all(left <= allow), (name, "opacity")
    # invisible Gaussians: exact zeros everywhere
    for k in ("dv2g", "dopacity", "dmeans3D", "dscales", "drot"):
        assert np.all(got[k][~vis] == 0.0), (name, k)
    # stage B from the GPU's own float dL/dview2gaussian
    sc = r["sc"]
    P = r["P"]
    if vis.any():
        zc = np.zeros((P, 3), np.float32)
        ora = gof_oracle.preprocess_backward(sc, r["radii"], r["st"]["clamped"], zc, got["dv2g"])
        jm = chain_mag(sc, r["radii"], r["st"]["clamped"], got["dv2g"])
        # an isotropic Gaussian's rotation gradient is a cancellation to an exact zero: there is nothing to compare
        scl = r["scales"]
        aniso = vis & ~((scl[:, 0] == scl[:, 1]) & (scl[:, 1] == scl[:, 2]))
        for gk, ok_, sel in (("dscales", "dL_dscale", vis), ("drot", "dL_drot", aniso), ("dmeans3D", "dL_dmean3D", vis)):
            if not sel.any():
                continue
            ratio = _chain_ratio(got[gk][sel], ora[ok_][sel], jm[ok_][sel])
            assert ratio <= 1.0, (name, gk, ratio)
    print(f"[{name}] P={P} PN={r['PN']} projected={int(ok.sum())} longest list={int(o['n_list'].max()) if r['PN'] else 0} "
          f"point ratio={out['point']:.4f} v2g ratio={out['v2g']:.4f} (of C={C}) points left out={share_pt:.2e} "
          f"marginal points={float((o['marg_pt'][ok] == 1).mean()) if ok.any() else 0.0:.2e} Gaussians left out={share_g:.2e} "
          f"with an allowance={share_allow:.2e}")
    return out


def _surface_points(cam, gs, n, seed, jitter=0.02):
    rng = np.random.default_rng(seed)
    ids = rng.integers(0, gs["means3D"].shape[0], n)
    return isc.points_around(gs, ids, 1, jitter, seed)


def cap_clear_scene():
    """The 1 024-contributor cap with every transmittance well above 1e-4: 2 400 Gaussians 16 pixels wide of opacity 0.006 over
    48x32 pixels.  A Gaussian is recorded within 0.92 sigma of a pixel, about 1 300 of them near the middle (the cap is reached),
    and no ray's T falls below 0.994^1300 = 4e-4, so no decision of pass 1 sits at the T threshold and the Gaussian side of
    long lists is compared in full."""
    cam = gof_synth.make_camera(48, 32, view=3)
    rng = np.random.default_rng(17)
    n = 2400
    xy = np.stack([rng.normal(24, 14, n), rng.normal(16, 10, n)], 1)
    gs = isc.blobs(cam, xy, rng.uniform(3.0, 5.0, n), 16.0, 0.006, seed=18)
    pts = torch.from_numpy(isc.cam_to_world(cam, isc.pixel_to_cam(cam, rng.uniform(0, 48, 4000), rng.uniform(0, 32, 4000),
                                                                  rng.uniform(2.5, 5.5, 4000))).astype(np.float32))
    return cam, gs, pts


# name -> (scene, the largest share of marginal Gaussians allowed).  The Gaussian counts of ragged (4 001) and c_1080p (20 003)
# are not multiples of 4: the binding's output slices must keep dL_drotations 16-byte aligned for any P.  In cap_1024 the lists
# are long enough for T to reach 1e-4 at most pixels, so most Gaussians are left out; cap_clear covers the Gaussian side of the
# cap instead.
SCENES = {
    "c_1080p": (lambda: (lambda cg: (cg[0], cg[1], _surface_points(cg[0], cg[1], 200_000, 5)))(
        gof_synth.make_scene(dict(P=20_003, width=1920, height=1080, seed=3), view=2)), SHARE_MARGINAL_G),
    "ragged": (lambda: (lambda cg: (cg[0], cg[1], _surface_points(cg[0], cg[1], 30_000, 6, 0.05)))(
        gof_synth.make_scene(dict(P=4001, width=203, height=117, seed=31), view=11)), SHARE_MARGINAL_G),
    "cap_1024": (isc.cap_scene, 1.0),
    "cap_clear": (cap_clear_scene, SHARE_MARGINAL_G),
    "u16_wrap": (lambda: isc.u16_scene()[:3], SHARE_MARGINAL_G),
}


@pytest.mark.parametrize("name", list(SCENES))
def test_against_oracle(name):
    make, share_g = SCENES[name]
    cam, gs, pts = make()
    r = run(cam, gs, pts, seed=11)
    if name == "cap_clear":
        assert int(r["o"]["n_list"].max()) == 1024   # the cap is reached
    check(r, name, share_g)


def test_mip_filter():
    cam, gs = gof_synth.make_scene(dict(P=3001, width=160, height=96, seed=41), view=4)
    check(run(cam, gs, _surface_points(cam, gs, 20_000, 9, 0.05), seed=3, kernel_size=0.1), "mip")


def test_many_points_in_one_pixel_and_borders():
    """5 000 points in one pixel (one warp run walks the same list), points on tile and image borders."""
    cam, gs = gof_synth.make_scene(dict(P=3000, width=160, height=96, seed=42), view=5)
    W, H = cam.image_width, cam.image_height
    rng = np.random.default_rng(4)
    x = np.concatenate([80.0 + 0.999 * rng.random(5000), rng.choice([0.0, 15.999, 16.0, 31.999, 32.0, W - 1e-3], 3000)])
    y = np.concatenate([48.0 + 0.999 * rng.random(5000), rng.uniform(0, H - 1e-3, 3000)])
    z = rng.uniform(3.0, 5.0, x.size)
    pts = torch.from_numpy(isc.cam_to_world(cam, isc.pixel_to_cam(cam, x, y, z)).astype(np.float32))
    check(run(cam, gs, pts, seed=5), "one_pixel_borders")


def test_empty_cases_write_zeros():
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda")
    cam, gs = gof_synth.make_scene(dict(P=500, width=64, height=48, seed=2), view=1)
    pts = _surface_points(cam, gs, 1000, 3)
    # no Gaussian in view: every Gaussian behind the camera
    behind = dict(gs)
    c = torch.as_tensor(isc.cam_to_world(cam, np.array([[0.0, 0.0, -5.0]])), dtype=torch.float32)
    behind["means3D"] = (gs["means3D"] * 0.01 + c).contiguous()
    for g_, p_ in ((behind, pts), (gs, pts[:0]), ({k: (v[:0] if isinstance(v, torch.Tensor) else v) for k, v in gs.items()}, pts)):
        ia = _args(cam, g_, p_, dev)
        state = _C.integrate_gaussians_to_points_state(*ia)
        dL = torch.randn(p_.shape[0], device=dev)
        for t in _backward(ia, state, dL):
            assert t is None or bool((t == 0).all())


def test_bit_identity_reproducibility_and_pooled_scratch():
    from diff_gaussian_rasterization import GaussianRasterizer, integrate_gaussians
    dev = torch.device("cuda")
    cam, gs = gof_synth.make_scene(dict(P=4003, width=208, height=120, seed=20), view=3)   # P % 4 != 0: see SCENES
    rs = gof_synth.raster_settings(cam, gs["sh_degree"], dev)
    pts = _surface_points(cam, gs, 40_000, 8).to(dev)
    p = {k: gs[k].to(dev) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    ref = GaussianRasterizer(rs).integrate(pts, p["means3D"], torch.zeros_like(p["means3D"]), p["opacities"], shs=p["shs"],
                                           scales=p["scales"], rotations=p["rotations"])
    dL = torch.randn(pts.shape[0], device=dev)
    grads = []
    for _ in range(3):   # the pooled scratch buffers are handed out again on every call
        q = {k: v.clone().requires_grad_(True) for k, v in p.items()}
        pp = pts.clone().requires_grad_(True)
        out = integrate_gaussians(pp, q["means3D"], torch.zeros_like(q["means3D"]), q["opacities"], q["shs"], None, q["scales"],
                                  q["rotations"], None, None, rs)
        for a, b in zip(out, ref):
            assert torch.equal(a, b)
        (out[1] * dL).sum().backward()
        grads.append((pp.grad.clone(), q["opacities"].grad.clone(), q["means3D"].grad.clone()))
        assert q["shs"].grad is None
    assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][0], grads[2][0])   # no atomics on the point side
    torch.testing.assert_close(grads[0][1], grads[1][1], rtol=1e-5, atol=1e-7)
    # the public API returns what the ABI computes
    from diff_gaussian_rasterization import _C
    ia = _args(cam, gs, pts.cpu(), dev)
    g = _backward(ia, _C.integrate_gaussians_to_points_state(*ia), dL)
    assert torch.equal(g[0], grads[0][0])
    torch.testing.assert_close(g[1], grads[0][1], rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(g[2], grads[0][2], rtol=1e-4, atol=1e-6)
    # grad mode off: the plain query
    with torch.no_grad():
        out = integrate_gaussians(pts, p["means3D"], torch.zeros_like(p["means3D"]), p["opacities"], p["shs"], None, p["scales"],
                                  p["rotations"], None, None, rs)
    for a, b in zip(out, ref):
        assert torch.equal(a, b)


def test_view2gaussian_precomp_receives_the_gradient():
    from diff_gaussian_rasterization import integrate_gaussians, _C
    dev = torch.device("cuda")
    cam, gs = gof_synth.make_scene(dict(P=2000, width=128, height=96, seed=12), view=2)
    rs = gof_synth.raster_settings(cam, gs["sh_degree"], dev)
    pts = _surface_points(cam, gs, 10_000, 2).to(dev)
    P = gs["means3D"].shape[0]
    ia = _args(cam, gs, pts.cpu(), dev)
    st = _C.integrate_gaussians_to_points_state(*ia)
    v2g = _C.export_state(P, cam.image_width, cam.image_height, st[0], st[5], st[6], st[7], st[4])["view2gaussian"]
    v = v2g.clone().requires_grad_(True)
    p = {k: gs[k].to(dev) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    out = integrate_gaussians(pts, p["means3D"], torch.zeros_like(p["means3D"]), p["opacities"], p["shs"], None, p["scales"],
                              p["rotations"], None, v, rs)
    assert torch.equal(out[1], st[2])
    dL = torch.randn(pts.shape[0], device=dev)
    (out[1] * dL).sum().backward()
    g = _backward(ia, st, dL)
    torch.testing.assert_close(v.grad, g[6], rtol=1e-5, atol=1e-7)


def test_descent_to_half_alpha():
    """Adam on the Gaussians drives alpha_integrated at sampled surface points toward 0.5."""
    from diff_gaussian_rasterization import integrate_gaussians
    dev = torch.device("cuda")
    cam, gs = gof_synth.make_scene(dict(P=3000, width=160, height=120, seed=9), view=6)
    rs = gof_synth.raster_settings(cam, gs["sh_degree"], dev)
    pts = _surface_points(cam, gs, 20_000, 4, 0.01).to(dev)
    q = {k: gs[k].to(dev).clone().requires_grad_(k != "shs") for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    opt = torch.optim.Adam([q["means3D"], q["scales"], q["rotations"], q["opacities"]], lr=2e-3)

    def loss_fn():
        out = integrate_gaussians(pts, q["means3D"], torch.zeros_like(q["means3D"]), q["opacities"], q["shs"], None, q["scales"],
                                  q["rotations"], None, None, rs)
        a = out[1]
        keep = a < 1.0   # points that project (the others keep alpha = 1)
        return ((a[keep] - 0.5) ** 2).mean()

    first = float(loss_fn())
    for _ in range(60):
        opt.zero_grad()
        loss = loss_fn()
        loss.backward()
        opt.step()
        with torch.no_grad():
            q["opacities"].clamp_(1e-3, 1.0)
    last = float(loss_fn())
    print(f"[descent] loss {first:.5f} -> {last:.5f}")
    assert last < 0.5 * first
