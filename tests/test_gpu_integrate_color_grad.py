"""GPU: the colour backward of the opacity-field query (DESIGN.md 4.13) against the float64 colour oracle
(tests/integrate_grad_oracle/integrate_color_oracle.c), fed with this library's own forward state (_C.export_state: tile lists, ranges,
view2gaussian, effective opacity, colours) and the query's own projection of the points.

For every visible Gaussian not left out, each component of dL/dcolors and of dL/dview2gaussian:

    |gpu - oracle|  <=  C * 2^-24 * mag  +  2 ulp(oracle)

mag (the oracle's) is the sum of the magnitudes of the terms, each times 1 + sum_j 1 / (1 - alpha_j) of its pixel.  A Gaussian of a
pixel at which a decision of the centre ray that rests on expf lies within a few ulp of its threshold is left out (where pass 1
reaches the cap, so are those of pass 1's marginal decisions, which move the cap); at most SHARE_MARGINAL_G of the visible
Gaussians may be.  The rest of the chain (dL/dsh, dL/dmeans3D,
dL/dscales, dL/drotations) is k_preprocess_backward, run unchanged: it is compared as stage B of test_gpu_grad_stagewise, from the
GPU's own float dL/dcolors and dL/dview2gaussian.  The test prints the largest constant each scene needed."""
import numpy as np
import pytest
import torch

import _integrate_color_oracle as igc
import gof_oracle
import gof_synth
from test_gpu_grad_stagewise import _chain_ratio, chain_mag, stage_b
from test_gpu_integrate_grad import SCENES, _args, _surface_points

pytestmark = pytest.mark.gpu

C = 64.0
SHARE_MARGINAL_G = 0.1
BG = (0.2, 0.5, 0.7)


def _ulp(x):
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(np.float32)).astype(np.float64)


def _cargs(cam, gs, pts, dev, kernel_size=0.0, colors=None):
    ia = list(_args(cam, gs, pts, dev, kernel_size))
    ia[0] = torch.tensor(BG, device=dev)
    if colors is not None:   # colors_precomp in place of the SHs
        ia[3], ia[18] = colors.to(dev), torch.Tensor([])
    return tuple(ia)


def _backward(ia, state, dL_dalpha, dL_dcolor, points_grad=True):
    from diff_gaussian_rasterization import _C
    (bg, p3, m3, col, op, sc, rot, sm, cov, v2g, vm, pm, tfx, tfy, ks, sub, H, W, sh, deg, cp, _pf, dbg) = ia
    R, _color, _a, _c, radii, geom, binning, img, pts, pbin = state
    return _C.integrate_gaussians_to_points_backward(bg, p3, m3, radii, col, sc, rot, sm, cov, v2g, vm, pm, tfx, tfy, ks, sub, H, W,
                                                     sh, deg, cp, dL_dalpha, R, geom, binning, img, pts, pbin, dbg,
                                                     points_grad=points_grad, dL_dcolor=dL_dcolor)


def run(cam, gs, pts, seed=0, kernel_size=0.0):
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda")
    P, PN, W, H = gs["means3D"].shape[0], pts.shape[0], cam.image_width, cam.image_height
    ia = _cargs(cam, gs, pts, dev, kernel_size)
    state = _C.integrate_gaussians_to_points_state(*ia)
    dLc = torch.randn(PN, 3, generator=torch.Generator().manual_seed(seed))
    g = _backward(ia, state, None, dLc.to(dev))
    torch.cuda.synchronize()
    names = ("dpts", "dopacity", "dmeans3D", "dscales", "drot", "dcov3D", "dv2g", "dcolors", "dsh")
    got = dict(zip(names, (None if t is None else t.cpu().numpy() for t in g)))
    R, _color, _alpha, _ci, radii, geom, binning, img, _pts, _pbin = state
    sc = gof_oracle.Scene(W, H, cam.tanfovx, cam.tanfovy, cam.world_view_transform, cam.full_proj_transform, cam.camera_center,
                          gs["means3D"], gs["opacities"], scales=gs["scales"], rotations=gs["rotations"], shs=gs["shs"],
                          sh_degree=gs["sh_degree"], kernel_size=kernel_size)
    st = {k: v.cpu().numpy() for k, v in _C.export_state(P, W, H, R, geom, binning, img, radii).items()}
    xy, _depth, ok = gof_oracle.project_points(sc, pts)
    o = igc.view(W, H, cam.tanfovx, cam.tanfovy, st, np.asarray(BG, np.float32), igc.pixel_dC(xy, ok, dLc.numpy(), W, H))
    return dict(got=got, o=o, ok=ok, ci=_ci.cpu().numpy(), xy=xy, radii=radii.cpu().numpy(), st=st, sc=sc, P=P, PN=PN, W=W,
                scales=gs["scales"].numpy())


def check(r, name, share_g_max=SHARE_MARGINAL_G):
    got, o = r["got"], r["o"]
    out = {}
    # the colour is piecewise constant in the point: exactly no point gradient
    assert np.all(got["dpts"] == 0.0), name
    vis = r["radii"] > 0
    share_g = float(o["marg_g"][vis].mean()) if vis.any() else 0.0
    assert share_g <= share_g_max, (name, "share of Gaussians left out", share_g)
    gsel = vis & ~o["marg_g"]
    for key, ok_, mk in (("dcolors", "dcol", "mag_c"), ("dv2g", "dv2g", "mag_g")):
        err = np.abs(got[key][gsel].astype(np.float64) - o[ok_][gsel])
        allow = 2 * _ulp(o[ok_][gsel]) + 1e-30
        need = np.maximum(err - allow, 0.0) / (2.0 ** -24 * o[mk][gsel] + 1e-300)
        out[key] = float(need.max()) if need.size else 0.0
        assert out[key] <= C, (name, key, out[key])
    # the oracle's pixel colour is the forward's (the same blended set): every projected point of a pixel not left out
    ok = r["ok"]
    pix = np.floor(r["xy"][ok, 1]).astype(np.int64) * r["W"] + np.floor(r["xy"][ok, 0]).astype(np.int64)
    oc = o["C"].reshape(-1, 3)[pix]
    dc = np.abs(oc - r["ci"][ok])
    assert np.median(dc) <= 1e-5, (name, "colour", float(np.median(dc)))
    for k in ("dv2g", "dopacity", "dmeans3D", "dscales", "drot", "dcolors"):
        assert np.all(got[k][~vis] == 0.0), (name, k)
    if vis.any():
        b = stage_b(dict(got=dict(got, dmeans2D=None), st=r["st"], sc=r["sc"], radii=r["radii"]))
        # an isotropic Gaussian's rotation gradient is a cancellation to an exact zero: there is nothing to compare
        scl = r["scales"]
        aniso = vis & ~((scl[:, 0] == scl[:, 1]) & (scl[:, 1] == scl[:, 2]))
        if not aniso.all():
            b.pop("drot")
            if aniso.any():
                ora = gof_oracle.preprocess_backward(r["sc"], r["radii"], r["st"]["clamped"], got["dcolors"], got["dv2g"])
                jm = chain_mag(r["sc"], r["radii"], r["st"]["clamped"], got["dv2g"])
                b["drot"] = _chain_ratio(got["drot"][aniso], ora["dL_drot"][aniso], jm["dL_drot"][aniso])
        for k, v in b.items():
            assert v <= 1.0, (name, "stage B", k, v)
    print(f"[{name}] P={r['P']} PN={r['PN']} projected={int(ok.sum())} need C: dcolors={out['dcolors']:.3f} dv2g={out['dv2g']:.3f} "
          f"(of {C}) Gaussians left out={share_g:.2e}")
    return out


# In the cap scenes pass 1 reaches 1 024 contributors at most pixels, and there a marginal decision of any of the five rays
# can move the cap and with it the end of the centre ray's blend, which changes every suffix: those pixels are left out.
SHARE = dict({k: v[1] for k, v in SCENES.items()}, cap_clear=0.5)


@pytest.mark.parametrize("name", list(SCENES))
def test_against_oracle(name):
    make, _share = SCENES[name]
    cam, gs, pts = make()
    check(run(cam, gs, pts, seed=13), name, SHARE[name])


def test_mip_filter():
    cam, gs = gof_synth.make_scene(dict(P=3001, width=160, height=96, seed=41), view=4)
    check(run(cam, gs, _surface_points(cam, gs, 20_000, 9, 0.05), seed=3, kernel_size=0.1), "mip")


def test_many_points_in_one_pixel_and_borders():
    """5 000 points in one pixel (one pixel's run crosses warps and batches), points on tile and image borders."""
    import _integrate_scenes as isc
    cam, gs = gof_synth.make_scene(dict(P=3000, width=160, height=96, seed=42), view=5)
    W, H = cam.image_width, cam.image_height
    rng = np.random.default_rng(4)
    x = np.concatenate([80.0 + 0.999 * rng.random(5000), rng.choice([0.0, 15.999, 16.0, 31.999, 32.0, W - 1e-3], 3000)])
    y = np.concatenate([48.0 + 0.999 * rng.random(5000), rng.uniform(0, H - 1e-3, 3000)])
    z = rng.uniform(3.0, 5.0, x.size)
    pts = torch.from_numpy(isc.cam_to_world(cam, isc.pixel_to_cam(cam, x, y, z)).astype(np.float32))
    check(run(cam, gs, pts, seed=5), "one_pixel_borders")


def _scene_small(dev, seed=20, n=40_000):
    cam, gs = gof_synth.make_scene(dict(P=4003, width=208, height=120, seed=seed), view=3)
    pts = _surface_points(cam, gs, n, 8)
    return cam, gs, pts


def test_sum_of_losses_and_reproducibility():
    """Alpha and colour loss together = the two backwards apart (points bit for bit, Gaussians to summation order); the point
    gradient is reproducible bit for bit.  On the Gaussian side the sums are compared where they are formed: dL/dview2gaussian,
    dL/dcolors and dL/dopacity.  The map from there to dL/dmeans3D, dL/dscales and dL/drotations cancels heavily for small
    Gaussians, which magnifies the float rounding of its inputs; stage B of the oracle tests checks it with that taken into
    account."""
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda")
    cam, gs, pts = _scene_small(dev)
    ia = _cargs(cam, gs, pts, dev)
    gen = torch.Generator().manual_seed(2)
    dA, dCol = torch.randn(pts.shape[0], generator=gen).to(dev), torch.randn(pts.shape[0], 3, generator=gen).to(dev)
    both = _backward(ia, _C.integrate_gaussians_to_points_state(*ia), dA, dCol)
    both2 = _backward(ia, _C.integrate_gaussians_to_points_state(*ia), dA, dCol)
    alpha = _backward(ia, _C.integrate_gaussians_to_points_state(*ia), dA, None)
    color = _backward(ia, _C.integrate_gaussians_to_points_state(*ia), None, dCol)
    assert torch.equal(both[0], alpha[0]) and torch.equal(both[0], both2[0])
    assert bool((color[0] == 0).all())
    for i in (1, 6):   # dL/dopacity, dL/dview2gaussian
        w = alpha[i] + color[i]
        torch.testing.assert_close(both[i], w, rtol=1e-4, atol=1e-6 * float(w.abs().max()) + 1e-30)
    for i in (7, 8):
        torch.testing.assert_close(both[i], color[i], rtol=1e-4, atol=1e-6 * float(color[i].abs().max()) + 1e-30)
        assert float(color[i].abs().max()) > 0
    # the colour backward with no colour loss is the alpha backward, with zero colour gradients
    none = _backward(ia, _C.integrate_gaussians_to_points_state(*ia), dA, torch.zeros_like(dCol))
    assert torch.equal(none[0], alpha[0]) and bool((none[7] == 0).all()) and bool((none[8] == 0).all())


@pytest.mark.parametrize("kind", ["shs", "colors_precomp"])
def test_public_api_equals_abi(kind):
    """integrate_gaussians: the forward is bit-identical with and without colour gradients, and .grad of shs / colors_precomp and
    the other inputs is what the ABI computes."""
    from diff_gaussian_rasterization import GaussianRasterizer, integrate_gaussians, _C
    dev = torch.device("cuda")
    cam, gs, pts = _scene_small(dev, n=30_000)
    rs = gof_synth.raster_settings(cam, gs["sh_degree"], dev, bg=BG)
    pts = pts.to(dev)
    p = {k: gs[k].to(dev) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    colors = torch.rand(p["means3D"].shape[0], 3, generator=torch.Generator().manual_seed(1)).to(dev)
    kw = dict(shs=p["shs"]) if kind == "shs" else dict(colors_precomp=colors)
    ref = GaussianRasterizer(rs).integrate(pts, p["means3D"], torch.zeros_like(p["means3D"]), p["opacities"], scales=p["scales"],
                                           rotations=p["rotations"], **kw)
    q = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    qc = colors.clone().requires_grad_(True)
    out = integrate_gaussians(pts, q["means3D"], torch.zeros_like(q["means3D"]), q["opacities"], q["shs"] if kind == "shs" else None,
                              None if kind == "shs" else qc, q["scales"], q["rotations"], None, None, rs)
    for a, b in zip(out, ref):
        assert torch.equal(a, b)
    assert out[2].requires_grad
    dCol = torch.randn(pts.shape[0], 3, generator=torch.Generator().manual_seed(4)).to(dev)
    (out[2] * dCol).sum().backward()
    ia = _cargs(cam, gs, pts.cpu(), dev, colors=None if kind == "shs" else colors)
    g = _backward(ia, _C.integrate_gaussians_to_points_state(*ia), None, dCol)
    tc = lambda a, b: torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6 * float(b.abs().max()) + 1e-30)   # noqa: E731
    tc(q["opacities"].grad, g[1])
    tc(q["means3D"].grad, g[2])
    tc(q["scales"].grad, g[3])
    if kind == "shs":
        tc(q["shs"].grad, g[8])
    else:
        tc(qc.grad, g[7])
        assert g[8] is None
    # only the Gaussians that the colours require grad: a colour loss alone reaches them
    qc2 = colors.clone().requires_grad_(True)
    if kind == "colors_precomp":
        out = integrate_gaussians(pts, p["means3D"], torch.zeros_like(p["means3D"]), p["opacities"], None, qc2, p["scales"],
                                  p["rotations"], None, None, rs)
        (out[2] * dCol).sum().backward()
        tc(qc2.grad, g[7])


def test_empty_cases_write_zeros():
    from diff_gaussian_rasterization import _C
    import _integrate_scenes as isc
    dev = torch.device("cuda")
    cam, gs = gof_synth.make_scene(dict(P=500, width=64, height=48, seed=2), view=1)
    pts = _surface_points(cam, gs, 1000, 3)
    behind = dict(gs)
    c = torch.as_tensor(isc.cam_to_world(cam, np.array([[0.0, 0.0, -5.0]])), dtype=torch.float32)
    behind["means3D"] = (gs["means3D"] * 0.01 + c).contiguous()
    far = -pts * 0 + torch.as_tensor(isc.cam_to_world(cam, np.array([[0.0, 0.0, -3.0]])), dtype=torch.float32)   # no point projects
    empty_g = {k: (v[:0] if isinstance(v, torch.Tensor) else v) for k, v in gs.items()}
    for g_, p_ in ((behind, pts), (gs, pts[:0]), (empty_g, pts), (gs, far.contiguous())):
        ia = _cargs(cam, g_, p_, dev)
        state = _C.integrate_gaussians_to_points_state(*ia)
        n = p_.shape[0]
        for dA, dC in ((torch.randn(n, device=dev), torch.randn(n, 3, device=dev)), (None, torch.randn(n, 3, device=dev))):
            for t in _backward(ia, state, dA, dC):
                assert t is None or bool((t == 0).all())


def test_descent_fits_sh_dc_colours():
    """Adam on the SH DC coefficients of ~3 000 Gaussians fits color_integrated at surface points to target colours."""
    from diff_gaussian_rasterization import integrate_gaussians
    dev = torch.device("cuda")
    cam, gs = gof_synth.make_scene(dict(P=3000, width=160, height=120, seed=9), view=6)
    rs = gof_synth.raster_settings(cam, gs["sh_degree"], dev, bg=BG)
    pts = _surface_points(cam, gs, 20_000, 4, 0.01).to(dev)
    p = {k: gs[k].to(dev) for k in ("means3D", "scales", "rotations", "opacities")}
    shs = gs["shs"].to(dev).clone()
    dc = shs[:, :1, :].clone().requires_grad_(True)
    rest = shs[:, 1:, :]
    # the target: the query's colour with other DC coefficients (random colours 0.5 + C0 * dc in [0.2, 0.8])
    tshs = shs.clone()
    tshs[:, 0, :] = (torch.rand(shs.shape[0], 3, generator=torch.Generator().manual_seed(3)).to(dev) * 0.6 - 0.3) / 0.28209479177387814
    with torch.no_grad():
        tgt = integrate_gaussians(pts, p["means3D"], torch.zeros_like(p["means3D"]), p["opacities"], tshs, None, p["scales"],
                                  p["rotations"], None, None, rs)
        ci, ai = tgt[2], tgt[1]
    keep = ai < 0.999   # points that project and see something
    opt = torch.optim.Adam([dc], lr=0.05)

    def loss_fn():
        out = integrate_gaussians(pts, p["means3D"], torch.zeros_like(p["means3D"]), p["opacities"], torch.cat([dc, rest], 1), None,
                                  p["scales"], p["rotations"], None, None, rs)
        return ((out[2][keep] - ci[keep]) ** 2).mean()

    first = float(loss_fn())
    for _ in range(80):
        opt.zero_grad()
        loss = loss_fn()
        loss.backward()
        opt.step()
    last = float(loss_fn())
    print(f"[colour descent] {int(keep.sum())} points, loss {first:.5f} -> {last:.6f}")
    assert last < 0.1 * first
