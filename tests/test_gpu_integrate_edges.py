"""GPU: the opacity-field query (csrc/integrate.cu) per pixel and per point against the CPU oracle, at its edges.

The reference is gof_oracle.integrate: plain C, the float sequence of the original kernels, no culling box, no pre-reject,
no point sorting.  An fp64 evaluation is NOT a reference for pass 2: -(A t^2 + B t + C)/2 is computed in float with C of
1e5..1e6, so its value is defined by that float sequence (DESIGN 2.1, the comment above oracle_integrate) and an fp64 result
differs from every correct implementation by far more than any bound below.  Do not add one.

Criterion.  The host's expf and CUDA's differ in the last bits, so a decision can come out differently where a value sits on
its threshold (alpha on 1/255, T' on 1e-4, t on 0.2): the oracle flags those pixels and points `marginal`, every scene
asserts that they are under 1 %, and they are left out.  At all other pixels n_contrib, the number of recorded contributors,
channel 8 (points per pixel) and channel 6 (largest t, no expf involved) are exact.  Channels 0-2, 7, final_T and
alpha_integrated are sums  S = sum_j T_{j-1} a_j c_j,  T_j = T_{j-1} (1 - a_j),  |c_j| <= cmax, whose only differing input is
expf.  With u = 2^-24:
  * CUDA's expf is within 2 ulp, glibc's within 1, and the product op * exp rounds once on each side: |da_j| <= 8 u a_j = d a_j;
  * T_j picks up  T_{j-1} d a_j  from a_j and 2 u T_j from the two sides' roundings, both shrunk by the later factors
    (1 - a_k) <= 1:  |dT_j| <= sum_{i<=j} (d a_i / (1 - a_i) + 2 u) T_j;
  * S picks up, per term,  a_j |dT_{j-1}| cmax  +  T_{j-1} (d + 3 u) a_j cmax  +  2 u cmax (its own fma on both sides).
    Summed over j with  sum_{j>i} T_{j-1} a_j = T_i - T_n <= T_i  the first part is at most
    sum_i (d a_i T_{i-1} + 2 u T_i) cmax <= (d + 2 n u) cmax, the second at most (d + 3 u) cmax since sum_j T_{j-1} a_j <= 1.
  Total  |dS| <= (2 d + 3 u + 4 n u) cmax = (19 + 4 n) u cmax <= 19 u (1 + n) cmax,  so c = 19; n is the number of recorded
  contributors of the pixel (of the point's pixel), cmax = max(1, |colour|, |background|).  final_T obeys the smaller
  (8 + 2 n) u.  Each test prints the largest observed ratio to this bound and its marginal share.
color_integrated is a copy of the pixel's colour and is compared with it bit for bit; points that do not project keep
alpha 1 and colour 0."""
import numpy as np
import pytest
import torch

import _integrate_scenes as scenes
import _util
import gof_oracle
import gof_synth

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
C_BOUND = 19.0


def cuda_integrate(cam, gs, pts, bg=(0.0, 0.0, 0.0)):
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda")
    fa = _util.fwd_args(cam, gs, dev, bg=bg)
    R, color, alpha, col_int, radii, geom, binning, img = _C.integrate_gaussians_to_points(fa[0], pts.to(dev), *fa[1:])
    out = dict(R=R, color=color.cpu().numpy(), alpha=alpha.cpu().numpy(), col_int=col_int.cpu().numpy(), radii=radii.cpu().numpy())
    P = int(gs["means3D"].shape[0])
    if P and pts.shape[0]:
        st = _C.export_state(P, cam.image_width, cam.image_height, R, geom, binning, img, radii)
        nc = st["n_contrib"].cpu().numpy()
        out.update(n_contrib=nc[0], n_recorded=nc[1], final_T=st["accum_alpha"][0].cpu().numpy())
    return out


def check(name, cam, gs, pts, bg=(0.0, 0.0, 0.0), got=None):
    """Compares one CUDA call with the oracle by the criterion of the module docstring; returns (oracle outputs, CUDA outputs)."""
    sc = gof_oracle.scene_from_synth(cam, gs, bg=bg)
    ocolor, oalpha, ocol, oradii, st = gof_oracle.integrate(sc, pts)
    got = cuda_integrate(cam, gs, pts, bg) if got is None else got
    W, H = sc.W, sc.H
    np.testing.assert_array_equal(got["radii"], oradii)
    assert got["R"] == st["num_rendered"]
    xy, depth, ok = gof_oracle.project_points(sc, pts)
    ppix = np.where(ok, np.nan_to_num(xy[:, 1]).astype(np.int64) * W + np.nan_to_num(xy[:, 0]).astype(np.int64), 0)
    good, goodp = ~st["marginal_pix"], ok & ~st["marginal_pt"]
    mfrac = max(st["marginal_pix"].mean(), st["marginal_pt"].mean() if len(oalpha) else 0.0)
    assert mfrac < 0.01, f"{name}: {mfrac:.4f} of the pixels or points are marginal"
    # exact: point counts everywhere (no expf decides them); contributor ids, counts and the largest t at non-marginal pixels
    np.testing.assert_array_equal(got["color"][8], ocolor[8], err_msg=f"{name}: points per pixel")
    assert float(np.abs(got["color"][3:6]).max()) == 0.0
    for key, ref in (("n_contrib", st["n_contrib"]), ("n_recorded", st["n_recorded"])):
        np.testing.assert_array_equal(got[key][good], ref[good], err_msg=f"{name}: {key}")
    np.testing.assert_array_equal(got["color"][6][good].view(np.int32), ocolor[6][good].view(np.int32), err_msg=f"{name}: largest t")
    cmax = max(1.0, float(np.abs(st["rgb"][oradii > 0]).max(initial=0.0)), float(np.abs(np.asarray(bg)).max()))
    n = st["n_recorded"].astype(np.float64)
    bound = C_BOUND * U * (1.0 + n) * cmax
    ratio = 0.0
    for ch in (0, 1, 2, 7):
        r = np.abs(got["color"][ch].astype(np.float64) - ocolor[ch]) / bound
        ratio = max(ratio, float(r[good].max(initial=0.0)))
    rT = np.abs(got["final_T"].astype(np.float64) - st["final_T"]) / ((8.0 + 2.0 * n) * U)
    ratio = max(ratio, float(rT[good].max(initial=0.0)))
    pbound = C_BOUND * U * (1.0 + n.reshape(-1)[ppix])
    rp = np.abs(got["alpha"].astype(np.float64) - oalpha) / pbound
    pratio = float(rp[goodp].max(initial=0.0))
    print(f"[integrate-edges] {name}: pixel ratio {ratio:.3f}, point ratio {pratio:.3f} of the bound; marginal {mfrac:.5f}; "
          f"{int(ok.sum())}/{len(ok)} points project, max contributors {int(n.max(initial=0))}")
    assert ratio <= 1.0, f"{name}: a pixel is {ratio:.2f} x its bound away from the oracle"
    assert pratio <= 1.0, f"{name}: a point is {pratio:.2f} x its bound away from the oracle"
    # integrated colour: the colour of the pixel the oracle charges the point to, bit for bit; untouched points keep 1 / 0
    img = np.stack([got["color"][c].reshape(-1)[ppix] for c in range(3)], 1)
    np.testing.assert_array_equal(got["col_int"][ok].view(np.int32), img[ok].view(np.int32), err_msg=f"{name}: color_integrated")
    assert np.all(got["alpha"][~ok] == 1.0) and np.all(got["col_int"][~ok] == 0.0), f"{name}: a point that does not project was written"
    return dict(color=ocolor, alpha=oalpha, st=st, xy=xy, depth=depth, ok=ok, ppix=ppix), got


def corner_only_ids(cam, gs):
    """Gaussians that some corner ray of some pixel accepts and no centre ray does (oracle_ray_mask_map)."""
    sc = gof_oracle.scene_from_synth(cam, gs)
    st = gof_oracle.preprocess(sc)
    ids = []
    for gid in np.nonzero(st["radii"] > 0)[0]:
        m = gof_oracle.ray_mask_map(sc.W, sc.H, sc.tan_fovx, sc.tan_fovy, st["view2gaussian"][gid], float(st["conic_opacity"][gid, 3]))
        if m.any() and not (m & 1).any():
            ids.append(gid)
    return np.asarray(ids)


def needle_inputs():
    cam, gs = scenes.needle_scene()
    ids = corner_only_ids(cam, gs)
    return cam, gs, ids, scenes.points_around(gs, ids, 20, 0.002, seed=4)


def test_gaussians_that_only_corner_rays_hit():
    """Scene 1.  Gaussians thinner than a pixel lying between two pixel centres: no centre ray blends them, a corner ray
    records them, and pass 2 then evaluates them for every point of the pixel."""
    cam, gs, ids, pts = needle_inputs()
    assert len(ids) > 100
    only = scenes.subset(gs, ids)
    o, got = check("corner-only Gaussians alone", cam, only, pts)
    assert float(o["color"][7].max()) == 0.0, "a centre ray blends one of them"
    depends = o["ok"] & (o["alpha"] > 0) & (o["alpha"] < 1)
    assert depends.sum() >= 100 and (o["st"]["n_recorded"] > 0).sum() >= 100
    assert (got["alpha"][depends] > 0).all()
    check("needles and pancakes, all 3000", cam, gs, pts, bg=(0.3, 0.1, 0.7))


def test_contributor_cap():
    """Scene 3.  Pixels that reach 1 024 recorded contributors stop there, their neighbours go on."""
    cam, gs, pts = scenes.cap_scene()
    o, _ = check("1024-contributor cap", cam, gs, pts)
    n = o["st"]["n_recorded"]
    assert n.max() == 1024 and (n == 1024).sum() > 20 and (n < 1024).sum() > 20
    assert (o["st"]["n_contrib"][n == 1024] < len(gs["means3D"])).any(), "no capped pixel stopped before the end of its list"


def test_uint16_contributor_ids():
    """Scene 4.  A tile list longer than 65 536: recorded ids wrap, and pass 2 replays them as the original's running index
    does -- a wrapped id selects the early list entry of that number, and nothing after it can be matched."""
    cam, gs, pts, pix = scenes.u16_scene()
    o, got = check("uint16 ids", cam, gs, pts)
    st = o["st"]
    assert (st["ranges"][:, 1] - st["ranges"][:, 0]).min() > 65536 + 4000
    x, y = pix["first_wrapped"]
    assert st["n_recorded"][y, x] == 2 and st["n_contrib"][y, x] > 65536        # B (65 541 -> 5) and Z
    x, y = pix["wrapped_after"]
    assert st["n_recorded"][y, x] == 3                                           # A (65 000), B (-> 5), Z
    in_pix = o["ok"] & (o["ppix"] == y * cam.image_width + x)
    assert in_pix.sum() > 3 and ((o["alpha"][in_pix] > 0.01) & (o["alpha"][in_pix] < 0.7)).any(), "A alone must show in the points"
    x, y = pix["id_zero"]
    assert st["n_recorded"][y, x] == 2
    # the first contributor of this pixel sits at list position 65 536 exactly: id 0, which stops the replay at once
    tile1 = st["point_list"][st["ranges"][1, 0]:st["ranges"][1, 1]]
    assert tile1[65535] == scenes.U16_FILL + 2
    in_pix = o["ok"] & (o["ppix"] == y * cam.image_width + x)
    assert in_pix.sum() > 3 and (o["alpha"][in_pix] == 0).all() and (got["alpha"][in_pix] == 0).all()


def _landing(cam, sc, x_target, y, z, axis=0):
    """float32 points whose projected x (axis 0) or y (axis 1) is exactly `x_target`, exactly one float below it, and one above:
    candidates around the float64 pre-image, stepped by single float32 ulps, classified with the oracle's projection."""
    xy = (x_target, y) if axis == 0 else (y, x_target)
    base = scenes.cam_to_world(cam, scenes.pixel_to_cam(cam, xy[0], xy[1], z)).astype(np.float32).reshape(3)
    k = np.arange(-40, 41)
    cand = np.repeat(base[None], len(k) ** 2, 0)
    for col, steps in ((0, np.repeat(k, len(k))), (2, np.tile(k, len(k)))):
        v = cand[:, col].copy()
        for s in range(1, 41):
            v = np.where(steps >= s, np.nextafter(v, np.float32(np.inf)), np.where(steps <= -s, np.nextafter(v, np.float32(-np.inf)), v))
        cand[:, col] = v
    pxy, _, ok = gof_oracle.project_points(sc, cand)
    t, v = np.float32(x_target), pxy[:, axis]
    picks = [cand[i] for i in np.nonzero(ok & (v == t))[0][:1]]                       # exactly on the border, when one exists
    below, above = np.nonzero(ok & (v < t))[0], np.nonzero(ok & (v >= t))[0]
    picks += [cand[below[np.argmax(v[below])]]] if len(below) else []                  # the closest float below it
    picks += [cand[above[np.argmin(v[above])]]] if len(above) else []                  # the closest at or above it
    return picks + [cand[i] for i in np.nonzero(~ok)[0][:1]]                           # one the projection drops, at the image border


def test_point_placement():
    """Scene 5.  Points that land exactly on pixel borders, tile borders and the image border, one float either side of them,
    at depth 0.2 and either side of it: which pixel each is charged to, and which are dropped.  (Non-finite coordinates are
    not covered: the oracle's float-to-int conversion of a NaN position is undefined on the host.)"""
    W, H = 80, 48
    cam = gof_synth.make_camera(W, H, view=11)
    rng = np.random.default_rng(23)
    gs = scenes.blobs(cam, np.stack([rng.uniform(0, W, 600), rng.uniform(0, H, 600)], 1), rng.uniform(2.0, 5.0, 600), rng.uniform(1.0, 4.0, 600),
                      rng.uniform(0.05, 0.9, 600), seed=24)
    sc = gof_oracle.scene_from_synth(cam, gs)
    pts = []
    for xt in (0.0, 1.0, 7.0, 16.0, 32.0, 37.0, 64.0, float(W - 1), float(W)):
        pts += _landing(cam, sc, xt, 20.3, 3.1, axis=0)
    for yt in (0.0, 5.0, 16.0, 32.0, float(H - 1), float(H)):
        pts += _landing(cam, sc, yt, 33.6, 2.7, axis=1)
    pts = np.asarray(pts, np.float32)
    # depth 0.2 and its neighbours, along the optical axis
    zs = [np.float32(0.2), np.nextafter(np.float32(0.2), np.float32(0)), np.nextafter(np.float32(0.2), np.float32(1)), np.float32(0.21), np.float32(0.19)]
    near = scenes.cam_to_world(cam, scenes.pixel_to_cam(cam, W / 2.0 + 0.25, H / 2.0 + 0.25, np.asarray(zs, np.float64))).astype(np.float32)
    fill = scenes.cam_to_world(cam, scenes.pixel_to_cam(cam, rng.uniform(-4, W + 4, 3000), rng.uniform(-4, H + 4, 3000), rng.uniform(0.1, 6, 3000))).astype(np.float32)
    allp = torch.from_numpy(np.concatenate([pts, near, fill]))
    o, got = check("point placement", cam, gs, allp)
    xy, depth, ok = o["xy"], o["depth"], o["ok"]
    m = len(pts)
    x, y = xy[:m, 0], xy[:m, 1]
    # each class is present, by the oracle's projection: within 1e-4 px of the border on either side of it
    for t in (7.0, 16.0, 32.0, 37.0, 64.0):
        assert (ok[:m] & (x < t) & (x > t - 1e-4)).any() and (ok[:m] & (x >= t) & (x < t + 1e-4)).any(), f"no points either side of x = {t}"
    for t in (5.0, 16.0, 32.0):
        assert (ok[:m] & (y < t) & (y > t - 1e-4)).any() and (ok[:m] & (y >= t) & (y < t + 1e-4)).any(), f"no points either side of y = {t}"
    assert (ok[:m] & (x < 1e-4)).any() and (ok[:m] & (x > W - 1e-4)).any() and (ok[:m] & (y > H - 1e-4)).any()
    assert (~ok[:m]).sum() >= 3, "no point landed on x = W / y = H or below 0"
    pz = gof_oracle.project_points(sc, near)
    assert pz[2][3] and not pz[2][4], "depth 0.21 must project and depth 0.19 must not"


def test_point_counts():
    """Scene 6.  0, 1 and 255-257 points; 5 000 points in one pixel; no point that projects; points in every tile."""
    cam, gs = gof_synth.make_scene(dict(P=700, width=96, height=64, seed=41), view=3)   # sparse: few pixels saturate at T' = 1e-4
    rng = np.random.default_rng(5)
    spread = lambda n: torch.from_numpy(scenes.cam_to_world(cam, scenes.pixel_to_cam(   # noqa: E731
        cam, rng.uniform(0, 96, n), rng.uniform(0, 64, n), rng.uniform(2.0, 6.0, n))).astype(np.float32))
    for n in (1, 255, 256, 257):
        check(f"{n} points", cam, gs, spread(n))
    got = cuda_integrate(cam, gs, torch.zeros(0, 3))
    assert got["alpha"].shape == (0,) and got["col_int"].shape == (0, 3)
    hot = torch.from_numpy(scenes.cam_to_world(cam, scenes.pixel_to_cam(cam, rng.uniform(40.0, 41.0, 5000), rng.uniform(30.0, 31.0, 5000),
                                                                        rng.uniform(2.0, 6.0, 5000))).astype(np.float32))
    o, _ = check("5000 points in one pixel", cam, gs, hot)
    assert o["color"][8].max() >= 4990
    behind = torch.from_numpy(scenes.cam_to_world(cam, scenes.pixel_to_cam(cam, rng.uniform(0, 96, 500), rng.uniform(0, 64, 500), -2.0)).astype(np.float32))
    o, _ = check("no point projects", cam, gs, behind)
    assert not o["ok"].any()
    o, _ = check("points in every tile", cam, gs, spread(20000))
    assert (o["color"][8].reshape(4, 16, 6, 16).sum((1, 3)) > 0).all()
    left = spread(4000)
    o, _ = check("points in the left half only", cam, gs, left[gof_oracle.project_points(gof_oracle.scene_from_synth(cam, gs), left)[0][:, 0] < 48])
    assert o["color"][8][:, 48:].sum() == 0 and o["color"][8][:, :48].sum() > 1000


def test_point_depth_clamp():
    """Scene 7.  Points in front of, inside and behind the contributors of their ray: both branches of the depth clamp."""
    cam, gs = gof_synth.make_scene(dict(P=700, width=96, height=64, seed=43), view=8)
    pts = torch.cat([scenes.points_around(gs, np.arange(700), 12, 0.05, seed=6),
                     torch.from_numpy(scenes.cam_to_world(cam, scenes.pixel_to_cam(cam, np.random.default_rng(7).uniform(0, 96, 6000),
                                                                                   np.random.default_rng(8).uniform(0, 64, 6000),
                                                                                   np.random.default_rng(9).uniform(0.5, 8.0, 6000))).astype(np.float32))])
    o, _ = check("depth clamp", cam, gs, pts)
    clamped, free = o["st"]["pt_clamp"][:, 0], o["st"]["pt_clamp"][:, 1]
    assert (clamped > 0).sum() > 1000 and (free > 0).sum() > 1000 and ((clamped > 0) & (free > 0)).sum() > 1000


@pytest.mark.parametrize("W,H", [(203, 117), (16, 16), (7, 5)])
def test_image_shapes(W, H):
    """Scene 8.  Sizes that are not multiples of the tile, a single full tile, a single partial tile; non-zero background."""
    cam, gs = gof_synth.make_scene(dict(P=max(40, W * H // 10), width=W, height=H, seed=47), view=5)
    rng = np.random.default_rng(9)
    pts = torch.from_numpy(scenes.cam_to_world(cam, scenes.pixel_to_cam(cam, rng.uniform(-1, W + 1, 8000), rng.uniform(-1, H + 1, 8000),
                                                                        rng.uniform(1.5, 6.0, 8000))).astype(np.float32))
    o, _ = check(f"{W}x{H}", cam, gs, pts, bg=(0.2, 0.9, 0.4))
    assert o["ok"].sum() > 4000 and (o["alpha"][o["ok"]] > 0).sum() > 100 and (o["st"]["n_recorded"] > 0).mean() > 0.3


def test_more_tiles_than_resident_blocks():
    """Scene 8.  1920x1080 (8 160 tiles) under sparse Gaussians: every block of the persistent grid walks many tiles and reuses
    its contributor slab, most tiles without any Gaussian or any point."""
    cam, gs = gof_synth.make_scene(dict(P=6000, width=1920, height=1080, seed=49), view=2)
    props = torch.cuda.get_device_properties(0)
    assert 120 * 68 > 3 * props.multi_processor_count
    pts = torch.cat([scenes.points_around(gs, np.arange(6000), 4, 0.01, seed=3), (torch.rand(20000, 3, generator=torch.Generator().manual_seed(4)) * 2 - 1) * 1.5])
    o, _ = check("1920x1080", cam, gs, pts, bg=(0.5, 0.5, 0.5))
    assert (o["st"]["n_recorded"] > 0).sum() > 5000 and (o["alpha"][o["ok"]] > 0).sum() > 2000


def test_no_gaussian_in_view():
    """Scene 8.  No Gaussian at all, and every Gaussian behind the camera: the image is the background, every alpha 0."""
    cam, gs = gof_synth.make_scene(dict(P=500, width=64, height=48, seed=51), view=1)
    rng = np.random.default_rng(2)
    pts = torch.from_numpy(scenes.cam_to_world(cam, scenes.pixel_to_cam(cam, rng.uniform(0, 64, 900), rng.uniform(0, 48, 900), rng.uniform(1, 5, 900))).astype(np.float32))
    back = dict(gs)
    back["means3D"] = torch.from_numpy(scenes.cam_to_world(cam, scenes.pixel_to_cam(cam, rng.uniform(0, 64, 500), rng.uniform(0, 48, 500),
                                                                                   rng.uniform(-6, -1, 500))).astype(np.float32))
    o, got = check("all Gaussians behind the camera", cam, back, pts, bg=(0.1, 0.6, 0.3))
    assert (o["st"]["n_recorded"] == 0).all() and (got["alpha"] == 0).all()
    assert (got["color"][0] == np.float32(0.1)).all() and (got["color"][1] == np.float32(0.6)).all()
    got = cuda_integrate(cam, scenes.subset(gs, []), pts)   # P = 0: nothing runs, outputs keep their initial values
    assert (got["alpha"] == 1).all() and (got["col_int"] == 0).all() and (got["color"] == 0).all()


def test_scratch_reuse():
    """Scene 9.  The pooled scratch buffers carry whatever the previous call left: repeating a call after a different, larger
    one -- stale contributor slabs, point keys and tile ranges in the buffers -- gives the same bits."""
    cam, gs, ids, pts = needle_inputs()
    first = cuda_integrate(cam, gs, pts)
    capcam, capgs, cappts = scenes.cap_scene()
    cuda_integrate(capcam, capgs, cappts)            # fills the slabs up to 1 024 ids per pixel
    big = gof_synth.make_scene(dict(P=20000, width=320, height=200, seed=3), view=4)
    cuda_integrate(big[0], big[1], (torch.rand(50000, 3, generator=torch.Generator().manual_seed(1)) * 2 - 1) * 1.5)
    for k in range(2):
        again = cuda_integrate(cam, gs, pts)
        for key in ("color", "alpha", "col_int", "n_contrib", "n_recorded", "final_T"):
            np.testing.assert_array_equal(first[key].view(np.int32), again[key].view(np.int32), err_msg=f"run {k}: {key}")
