"""GPU: the forward blend (csrc/render_fwd.cu) per pixel, per counter and per blend mask against the CPU oracle, at its edges.

The reference is gof_oracle.forward(checked=True): plain C, the float sequence of the original kernel, no culling box, no
pre-reject, no staging.  An fp64 evaluation is not a reference here: power = -(C - B^2/(4A))/2 cancels C of 1e2..1e6 in float,
so the float sequence defines the value (see test_gpu_integrate_edges.py).

Criterion.  The host's expf and CUDA's differ in the last bits, so a decision can come out differently where a value sits on
its threshold: the oracle flags a pixel `marginal` when an alpha lies within 8 ulp of 1/255, a T' within twice its error bound
of 1e-4, or a T within twice its error bound of 0.5 at the median test.  Every scene asserts that under 1 % of its pixels are
marginal; they are left out of the comparisons below (the GPU's self-consistency checks still cover them).
  * Exact at the other pixels: radii, R, the tile ranges, n_contrib[0] (last contributor), n_contrib[1] (median contributor),
    channel 6 (median t) bit for bit, and the number of pairs blended (popcount of the pixel's blend-mask bits).
  * Bounded, with n the pixel's blended pairs and u = 2^-24.  Both sides run the same float sequence after expf, so alpha
    differs by at most 8u relative (expf within 3 ulp over both sides, op * exp rounded once on each) and every later rounding
    happens on both sides:
      - channels 0-2 and 7: sums S = sum_j T_{j-1} a_j c_j with |c_j| <= cmax; the bound of test_gpu_integrate_edges.py,
        19 u (1 + n) cmax, holds unchanged (cmax = max(1, |colour|, |background|); the background term adds (8 + 2n) u cmax,
        inside it for n >= 1, and n = 0 leaves T = 1 exact).
      - channels 3-5 (normals): c_j = the unit normal, |c_j| <= 1.  The GPU scales by rsqrtf(s + 1e-7f) (2 ulp, after one
        float add: 5u relative with the rounding of 1e-7 to float) and one product (u); the reference takes a double sqrt
        rounded to float (u) and divides (u).  So c_j differs by at most 8u, which adds sum_j T_{j-1} a_j 8u <= 8u:
        bound (19 (1 + n) + 8) u.
      - accum_alpha[0..3] (T, dist1, dist2, raw distortion): the oracle's running bounds accum_err (oracle_render_forward_checked
        states them), which take the GPU's mapped depth (gof_mapped_t_fast, within 1 ulp <= 2u m of the double quotient) into
        account.  The raw distortion cancels, so only a bound carried through its terms can hold it.
      - channel 8 = D / ((1 - T)^2 + 1e-7): with dT, dD the bounds above, d(1 - T) <= dT + u, the denominator moves by at
        most dden = 2 (1 - T) d(1 - T) + d(1 - T)^2 + 2u (1 - T)^2, so |dch8| <= (dD + |D| dden / den) / (den - dden) plus the
        final rounding on both sides.
  * Blend masks (GofBinLayout::vmask, exported by export_state(masks=True)): for every (tile, warp, group of 32 entries) with
    32 g < the warp's largest last contributor, the word of every lane at a non-marginal pixel equals the oracle's bits of that
    pixel for those entries, and lanes outside the image hold 0.  At every pixel inside the image, marginal ones included, the
    GPU agrees with itself: its highest set bit + 1 = n_contrib[0], and the entry n_contrib[1] has its bit set.
Each scene prints the largest ratio to each bound and the marginal share."""
import numpy as np
import pytest
import torch

import _integrate_scenes as scenes
import _util
import gof_oracle
import gof_synth

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
NONE = 0xFFFFFFFF


def cuda_forward(cam, gs, bg=(0.0, 0.0, 0.0), colors=None):
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda")
    fa = _util.fwd_args(cam, gs, dev, bg=bg, colors_precomp=colors)
    R, color, radii, geom, binning, img = _C.rasterize_gaussians(*fa)
    P, W, H = int(gs["means3D"].shape[0]), cam.image_width, cam.image_height
    st = _C.export_state(P, W, H, R, geom, binning, img, radii, masks=True)
    return dict(R=R, color=color.cpu().numpy(), radii=radii.cpu().numpy(), ranges=st["ranges"].cpu().numpy().view(np.uint32),
                n_contrib=st["n_contrib"].cpu().numpy().view(np.uint32), accum=st["accum_alpha"].cpu().numpy(),
                masks=st["blend_masks"].cpu().numpy().view(np.uint32), bufs=(fa, radii, geom, R, binning, img))


def to_lanes(a, fill, W, H):
    """[H,W,...] image array -> [tiles, 8 warps, 32 lanes, ...] in the forward's thread layout (warp = 8x4 block, lane =
    (y & 3) * 8 + (x & 7)); pixels outside the image get `fill`."""
    gx, gy = (W + 15) // 16, (H + 15) // 16
    rest = a.shape[2:]
    pad = np.full((gy * 16, gx * 16) + rest, fill, a.dtype)
    pad[:H, :W] = a
    pad = pad.reshape((gy, 4, 4, gx, 2, 8) + rest)
    return pad.transpose((0, 3, 1, 4, 2, 5) + tuple(range(6, 6 + len(rest)))).reshape((gx * gy, 8, 32) + rest)


def from_lanes(a, W, H):
    gx, gy = (W + 15) // 16, (H + 15) // 16
    return a.reshape(gy, gx, 4, 2, 4, 8).transpose(0, 2, 4, 1, 3, 5).reshape(gy * 16, gx * 16)[:H, :W]


def mask_words(W, H, ranges, masks, last):
    """The defined words of the exported masks: (words [8,G,32], valid [8,G], tile of each group [G], group index [G])."""
    tiles = len(ranges)
    r = ranges.astype(np.int64)
    lens = r[:, 1] - r[:, 0]
    ng = (lens + 31) // 32
    tog = np.repeat(np.arange(tiles), ng)
    gin = np.arange(int(ng.sum())) - np.repeat(np.cumsum(ng) - ng, ng)
    start = r[tog, 0] + 32 * tog + 32 * gin
    words = masks[:, start[:, None] + np.arange(32)[None, :]]
    warp_last = to_lanes(last.astype(np.int64), 0, W, H).max(2)                     # [tiles, 8]
    valid = (32 * gin)[None, :] < warp_last[tog].T
    return np.where(valid[:, :, None], words, 0).astype(np.uint32), valid, tog, gin


def check_masks(name, W, H, got, obits, good):
    """The criterion's blend-mask part; returns the GPU's blended-pair count per pixel [H,W]."""
    last, med = got["n_contrib"][0], got["n_contrib"][1]
    words, valid, tog, gin = mask_words(W, H, got["ranges"], got["masks"], last)
    tiles = len(got["ranges"])
    # the oracle's bits of each pixel, folded into the same layout
    ob = to_lanes(obits, 0, W, H)[tog, :, :, gin].transpose(1, 0, 2)                 # [8,G,32]
    gl = to_lanes(good, True, W, H)[tog].transpose(1, 0, 2)                          # outside the image: compared (must be 0)
    bad = valid[:, :, None] & gl & (words != ob)
    assert not bad.any(), f"{name}: {int(bad.sum())} mask words differ from the oracle, first (warp, group, lane) {np.argwhere(bad)[0].tolist()}"
    inside = to_lanes(np.ones((H, W), bool), False, W, H)
    assert not (words.transpose(1, 0, 2) * ~inside[tog]).any(), f"{name}: a lane outside the image has a mask bit"
    # self-consistency at every pixel
    cnt = np.zeros((tiles, 8, 32), np.int64)
    np.add.at(cnt, tog, np.bitwise_count(words).astype(np.int64).transpose(1, 0, 2))
    hb = np.zeros((tiles, 8, 32), np.int64)
    top = np.where(words != 0, 32 * gin[None, :, None] + np.frexp(words.astype(np.float64))[1], 0)
    np.maximum.at(hb, tog, top.transpose(1, 0, 2))
    hb_img = from_lanes(hb, W, H)
    np.testing.assert_array_equal(hb_img, last.astype(np.int64), err_msg=f"{name}: highest mask bit + 1 != n_contrib[0]")
    ys, xs = np.nonzero(med != NONE)
    p = med[ys, xs].astype(np.int64) - 1
    tile = (ys // 16) * ((W + 15) // 16) + xs // 16
    warp = ((ys % 16) // 4) * 2 + (xs % 16) // 8
    lane = (ys % 4) * 8 + xs % 8
    w = got["masks"][warp, got["ranges"][tile, 0].astype(np.int64) + 32 * tile + 32 * (p // 32) + lane]
    assert ((w >> (p % 32).astype(np.uint32)) & 1).all(), f"{name}: the median contributor's mask bit is not set"
    return from_lanes(cnt, W, H)


def _ratio(d, bound):
    return np.where(d == 0, 0.0, d / np.maximum(bound, 1e-300))


def check(name, cam, gs, bg=(0.0, 0.0, 0.0), colors=None, got=None):
    """One CUDA forward against the oracle by the criterion of the module docstring; returns (oracle state, CUDA outputs)."""
    sc = gof_oracle.scene_from_synth(cam, gs, bg=bg, colors_precomp=colors)
    out, oradii, st = gof_oracle.forward(sc, checked=True)
    got = cuda_forward(cam, gs, bg, colors) if got is None else got
    W, H = sc.W, sc.H
    np.testing.assert_array_equal(got["radii"], oradii, err_msg=f"{name}: radii")
    assert got["R"] == st["num_rendered"], name
    np.testing.assert_array_equal(got["ranges"], st["ranges"], err_msg=f"{name}: ranges")
    good = ~st["marginal_pix"]
    mfrac = float(st["marginal_pix"].mean())
    assert mfrac < 0.01, f"{name}: {mfrac:.4f} of the pixels are marginal"
    nb = check_masks(name, W, H, got, st["blended"], good)
    for k, what in ((0, "last contributor"), (1, "median contributor")):
        np.testing.assert_array_equal(got["n_contrib"][k][good], st["n_contrib"][k][good], err_msg=f"{name}: {what}")
    np.testing.assert_array_equal(nb[good], st["n_blended"][good], err_msg=f"{name}: blended pairs")
    np.testing.assert_array_equal(got["color"][6][good].view(np.int32), out[6][good].view(np.int32), err_msg=f"{name}: median t")
    n = st["n_blended"].astype(np.float64)
    vis = oradii > 0
    cmax = max(1.0, float(np.abs(st["rgb"][vis]).max(initial=0.0)), float(np.abs(np.asarray(bg)).max()))
    d = lambda a, b: np.abs(a.astype(np.float64) - b.astype(np.float64))   # noqa: E731
    ratios = {}
    ratios["colour"] = max(float(_ratio(d(got["color"][c], out[c]), 19 * U * (1 + n) * cmax)[good].max(initial=0)) for c in (0, 1, 2, 7))
    ratios["normal"] = max(float(_ratio(d(got["color"][c], out[c]), (19 * (1 + n) + 8) * U)[good].max(initial=0)) for c in (3, 4, 5))
    err = st["accum_err"]
    for k, key in enumerate(("T", "dist1", "dist2", "distortion")):
        ratios[key] = float(_ratio(d(got["accum"][k], st["accum_alpha"][k]), err[k])[good].max(initial=0))
    omt = 1.0 - st["accum_alpha"][0].astype(np.float64)
    domt = err[0] + U
    den = omt * omt + 1e-7
    dden = 2 * omt * domt + domt * domt + 2 * U * omt * omt
    D = np.abs(st["accum_alpha"][3].astype(np.float64))
    with np.errstate(divide="ignore", invalid="ignore"):
        b8 = np.where(den > dden, (err[3] + D * dden / den) / (den - dden), np.inf) * (1 + 2 * U) + 2 * U * np.abs(out[8].astype(np.float64))
    ratios["ch8"] = float(_ratio(d(got["color"][8], out[8]), b8)[good].max(initial=0))
    print(f"[forward-edges] {name}: " + ", ".join(f"{k} {v:.3f}" for k, v in ratios.items()) +
          f"; marginal {mfrac:.5f}; max blended {int(n.max(initial=0))}, R {got['R']}")
    for k, v in ratios.items():
        assert v <= 1.0, f"{name}: {k} is {v:.2f} x its bound away from the oracle"
    return st, got


# ---- scene builders ------------------------------------------------------------------------------------------------------

def pixel_walls(cam, pixels, depth, layers, seed, opacity=0.97):
    """`layers` tiny opaque Gaussians centred on each pixel centre of `pixels` [N,2] (a pixel saturates within them)."""
    px = np.repeat(np.asarray(pixels, np.float64), layers, 0) + 0.5
    rng = np.random.default_rng(seed)
    dep = depth + 0.01 * np.tile(np.arange(layers), len(pixels)) + rng.uniform(0, 1e-3, len(px))
    return scenes.blobs(cam, px, dep, 0.4, opacity, seed=seed)


def lens_of(st):
    return (st["ranges"][:, 1].astype(np.int64) - st["ranges"][:, 0]).tolist()


LENGTHS = [0, 1, 31, 32, 33, 255, 256, 257, 511, 512, 513, 3000]


def test_list_lengths_on_every_boundary():
    """Scene 1.  Twelve tiles whose lists hold 0, 1, 31-33, 255-257, 511-513 and 3 000 entries (faint stacks, one per tile)."""
    cam = gof_synth.make_camera(64, 48, view=4)
    parts = [scenes.tile_stack(cam, t % 4, t // 4, n, seed=100 + t) for t, n in enumerate(LENGTHS) if n]
    st, got = check("list lengths", cam, scenes.concat(parts))
    assert lens_of(st) == LENGTHS
    assert st["n_contrib"][0].max() > 2800 and st["n_blended"].max() > 100


def test_saturation_at_chosen_positions():
    """Scene 2a (_integrate_scenes.saturation_scene): tile k saturates its centre pixel at list position SAT_AT[k]."""
    st, got = check("saturation positions", *scenes.saturation_scene())
    for t, s in enumerate(scenes.SAT_AT):
        assert st["n_contrib"][0][8, 16 * t + 8] == s - 1 and st["accum_alpha"][0][8, 16 * t + 8] < 1e-3, (t, s)
        assert st["n_contrib"][1][8, 16 * t + 8] == s - 2, "T crosses 0.5 at the first layer"
        assert lens_of(st)[t] >= s + 60
    # scene 5's other median cases: pixels that never drop below 0.5 and pixels without any contributor
    last, med, T = st["n_contrib"][0], st["n_contrib"][1], st["accum_alpha"][0]
    assert (last == 0).sum() > 10 and ((med == last) & (last > 0) & (T > 0.5)).sum() > 10


def test_tile_saturates_within_its_first_batch():
    """Scene 2b.  Opaque layers in front of everything saturate every pixel of every tile within batch 0 while each list runs
    on for several batches: the CTA leaves its loop with the copy of batch 1 in flight."""
    cam = gof_synth.make_camera(48, 32, view=8)
    rng = np.random.default_rng(3)
    front = scenes.blobs(cam, np.tile([[24.0, 16.0]], (6, 1)), 1.5 + 0.05 * np.arange(6), 80.0, 0.97, seed=4)
    back = scenes.blobs(cam, np.stack([rng.uniform(0, 48, 1500), rng.uniform(0, 32, 1500)], 1), rng.uniform(3.0, 6.0, 1500), 12.0, 0.3, seed=5)
    st, got = check("saturated in batch 0", cam, scenes.concat([front, back]))
    # every pixel would blend the wide fillers behind the layers: stopping within the layers is saturation
    assert min(lens_of(st)) > 3 * 256 and st["n_contrib"][0].max() <= 6


def test_one_pixel_alive_for_ten_batches():
    """Scene 2c.  One 16x16 tile: every pixel but one is walled off by opaque layers at the front of the list; the remaining
    pixel blends a faint stack on its ray to the end of a 2 800-entry list.  Seven warps skip every later batch (no mbarrier
    wait, no mask store) while the eighth keeps the CTA going; the mbarrier parities stay in step across the skipped waits."""
    cam = gof_synth.make_camera(16, 16, view=9)
    q = (5, 13)
    pix = [(x, y) for y in range(16) for x in range(16) if (x, y) != q]
    walls = pixel_walls(cam, pix, 2.0, 4, seed=6)
    rng = np.random.default_rng(7)
    stack = scenes.blobs(cam, np.tile([[q[0] + 0.5, q[1] + 0.5]], (1800, 1)), rng.uniform(3.0, 6.0, 1800), 0.5, rng.uniform(0.0041, 0.0046, 1800), seed=8)
    st, got = check("one pixel alive", cam, scenes.concat([walls, stack]))
    last = st["n_contrib"][0]
    assert last[q[1], q[0]] > 10 * 256 and np.sort(last.reshape(-1))[-2] < 4 * 255, "the other pixels must stop in the first batches"


def test_warps_saturate_in_different_batches():
    """Scene 2d.  One tile: the pixels of warp w are walled off at list position ~300 w, behind faint fillers."""
    cam = gof_synth.make_camera(16, 16, view=10)
    parts = []
    for w in range(8):
        x0, y0 = (w & 1) * 8, (w >> 1) * 4
        parts.append(pixel_walls(cam, [(x0 + i, y0 + j) for j in range(4) for i in range(8)], 2.0 + 0.5 * w, 3, seed=30 + w))
    rng = np.random.default_rng(11)
    n = 2400
    parts.append(scenes.blobs(cam, np.stack([rng.uniform(2, 14, n), rng.uniform(2, 14, n)], 1), rng.uniform(1.9, 6.0, n), 0.6,
                              rng.uniform(0.004, 0.01, n), seed=12))
    st, got = check("warps saturate apart", cam, scenes.concat(parts))
    warp_last = to_lanes(st["n_contrib"][0].astype(np.int64), 0, 16, 16).max(2)[0]
    assert len(set((warp_last // 256).tolist())) >= 5, warp_last


def test_alpha_thresholds_and_pre_reject():
    """Scene 3 (_integrate_scenes.threshold_scene).  Every pair whose alpha lies in 1/255 (1 + [1e-5, 2e-3]) -- outside the
    marginal band, inside the pre-reject's margin -- is blended; opacity 0 and opacities below 1/255 blend nothing; the
    0.99 clamp holds."""
    cam, gs = scenes.threshold_scene()
    st, got = check("alpha thresholds", cam, gs)
    op = st["conic_opacity"][:, 3]
    vis = st["radii"] > 0
    a = np.float32(1.0 / 255.0)
    assert (vis & (op == a)).sum() >= 3 and (vis & (op == np.nextafter(a, np.float32(0)))).sum() >= 3
    assert (vis & (op >= 0.00392) & (op < a)).sum() >= 10 and (vis & (op == 0)).sum() >= 10 and (vis & (op >= 0.99)).sum() >= 30
    # pairs whose alpha lies in the pre-reject's margin but outside the marginal band, counted per Gaussian from the oracle
    sc = gof_oracle.scene_from_synth(cam, gs)
    lo, hi = float(a) * (1 + 1e-5), float(a) * (1 + 2e-3)
    inwin = 0
    for gid in np.nonzero(vis & (op >= a))[0]:
        am = gof_oracle.alpha_map(sc.W, sc.H, sc.tan_fovx, sc.tan_fovy, st["view2gaussian"][gid], float(op[gid]))
        inwin += int(((am >= lo) & (am <= hi)).sum())
    assert inwin > 500, inwin
    assert (st["accum_alpha"][0] > 1e-3).mean() > 0.99, "pixels must not saturate before the window pairs"
    assert got["color"][7].max() > 0.98, "the clamped opaque Gaussians must show"


def test_near_plane_and_camera_inside():
    """Scene 4.  The camera inside the cloud: pairs with t either side of 0.2, and Gaussians the camera sits inside the
    alpha >= 1/255 iso-surface of (K <= 0: K' = -inf, the whole plane as box)."""
    cam = gof_synth.make_camera(96, 64, view=9, radius=0.8)
    gs = gof_synth.make_gaussians(3000, 51, cam.focal_x, sigma_px=3.0)
    st, got = check("camera inside", cam, gs, bg=(0.2, 0.3, 0.9))
    vis = st["radii"] > 0
    op = st["conic_opacity"][:, 3].astype(np.float64)
    K = st["view2gaussian"][:, 9].astype(np.float64) - 2.0 * np.log(255.0 * np.maximum(op, 1e-30))
    assert (vis & (K <= 0)).sum() >= 3 and (vis & (st["depths"] < 0.4)).sum() >= 10


def test_median_depth_cases():
    """Scene 5.  The stacked scene of test_gpu_bwd_walk.py: T crosses 0.5 at many contributors, some pixels never drop below
    0.5, some have no contributor."""
    from test_gpu_bwd_walk import stacked_scene
    cam, gs = stacked_scene(150, 90, 1500, 900, 7, (37, 21))
    st, got = check("stacked", cam, gs)
    last, med, T = st["n_contrib"][0], st["n_contrib"][1], st["accum_alpha"][0]
    assert ((med != NONE) & (med < last) & (T < 0.5)).sum() > 100 and last[21, 37] > 256


def test_box_geometry():
    """Scene 6.  The `placed` scene of test_cull_bbox.py: sub-pixel needles between pixel centres (nothing may blend them),
    Gaussians centred on pixel corners, edges, tile borders and the image border, and screen-filling ones."""
    from test_cull_bbox import _placed_scene
    cam, gs = _placed_scene()
    rng = np.random.default_rng(19)
    big = scenes.blobs(cam, np.stack([rng.uniform(-30, 126, 12), rng.uniform(-30, 94, 12)], 1), rng.uniform(3.0, 6.0, 12), 40.0, 0.2, seed=20)
    off = scenes.blobs(cam, np.stack([np.r_[rng.uniform(-6, -0.5, 20), rng.uniform(96.5, 102, 20)], rng.uniform(0, 64, 40)], 1),
                       rng.uniform(3.0, 5.0, 40), 3.0, 0.8, seed=21)
    check("placed", cam, scenes.concat([gs, big, off]))
    cam, gs = scenes.needle_scene()
    check("needles", cam, gs, bg=(0.3, 0.1, 0.7))


@pytest.mark.parametrize("W,H", [(203, 117), (16, 16), (7, 5), (1, 1), (17, 1), (1, 17), (8, 4), (9, 5)])
def test_image_shapes(W, H):
    """Scene 7.  Warps partly or wholly outside the image; a non-zero background and precomputed colours outside [0, 1]."""
    P = max(40, W * H // 6)
    cam, gs = gof_synth.make_scene(dict(P=P, width=W, height=H, seed=47), view=5)
    colors = (torch.rand(P, 3, generator=torch.Generator().manual_seed(W * 100 + H)) * 3.0 - 1.0).contiguous()
    st, got = check(f"{W}x{H}", cam, gs, bg=(0.2, 0.9, 0.4), colors=colors)
    assert (st["n_blended"] > 0).any() and float(np.abs(st["rgb"]).max()) > 1.5


def test_more_tiles_than_resident_blocks():
    """Scene 7.  1920x1080 (8 160 tiles) under a sparse scene."""
    cam, gs = gof_synth.make_scene(dict(P=6000, width=1920, height=1080, seed=49), view=2)
    st, got = check("1920x1080", cam, gs, bg=(0.5, 0.5, 0.5))
    assert (st["n_blended"] > 0).sum() > 20000 and min(lens_of(st)) == 0


def test_stale_scratch():
    """Scene 8.  With the scratch pool on, a scene, a larger and denser one, then the first again: outputs, counters and every
    defined mask word are bit-identical, and a backward from the repeated forward agrees with the first."""
    from diff_gaussian_rasterization import _C
    cam, gs = scenes.threshold_scene()
    first = cuda_forward(cam, gs)
    grad = torch.randn(9, cam.image_height, cam.image_width, generator=torch.Generator().manual_seed(3)).cuda()
    g1 = [t.clone() for t in _C.rasterize_gaussians_backward(*_util.bwd_args(*first["bufs"], grad))]
    big = gof_synth.make_scene(dict(P=40000, width=320, height=200, seed=3, sigma_px=4.0), view=4)
    cuda_forward(*big)
    again = cuda_forward(cam, gs)
    for key in ("color", "n_contrib", "accum", "ranges"):
        np.testing.assert_array_equal(first[key].view(np.int32), again[key].view(np.int32), err_msg=key)
    W, H = cam.image_width, cam.image_height
    w1, v1, _, _ = mask_words(W, H, first["ranges"], first["masks"], first["n_contrib"][0])
    w2, v2, _, _ = mask_words(W, H, again["ranges"], again["masks"], again["n_contrib"][0])
    np.testing.assert_array_equal(v1, v2)
    np.testing.assert_array_equal(w1, w2, err_msg="defined mask words")
    check("repeated after a larger scene", cam, gs, got=again)
    g2 = _C.rasterize_gaussians_backward(*_util.bwd_args(*again["bufs"], grad))
    for a, b in zip(g2, g1):
        assert _util.same_up_to_summation_order(a, b)
