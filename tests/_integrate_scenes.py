"""Scene builders for the edge tests of the opacity-field query (test_gpu_integrate_edges.py, test_cull_bbox.py,
_cull_probe.py, test_gpu_extract.py).  Everything is drawn in float64 from a seed and rounded to float32 once."""
import math

import numpy as np
import torch

import gof_synth

NEEDLE_CASE = dict(P=3000, W=96, H=64, seed=2, sigma_px=0.5, radius=4.0, aniso=(0.05, 1.0))


def aniso_scene(case):
    """Random Gaussians whose three axes are scaled by independent log-uniform factors in `aniso` (needles and pancakes),
    seen by camera `7 * seed` of the ring.  The recipe of test_cull_bbox.py's cases."""
    cam = gof_synth.make_camera(case["W"], case["H"], view=case["seed"] * 7, radius=case["radius"])
    gs = gof_synth.make_gaussians(case["P"], case["seed"], cam.focal_x, sigma_px=case["sigma_px"])
    lo, hi = case["aniso"]
    g = torch.Generator().manual_seed(case["seed"] + 99)
    an = torch.exp(torch.rand(case["P"], 3, generator=g) * np.log(hi / lo) + np.log(lo))
    gs["scales"] = (gs["scales"].max(dim=1, keepdim=True).values * an).contiguous()
    return cam, gs


def needle_scene():
    """Sub-pixel needles and pancakes: about a tenth of the visible Gaussians have an alpha >= 1/255 ellipse that is thinner
    than a pixel and lies between two pixel centres, so only corner rays of the query meet them."""
    return aniso_scene(NEEDLE_CASE)


def subset(gs, ids):
    ids = torch.as_tensor(np.asarray(ids), dtype=torch.long)
    return {k: (v[ids].contiguous() if isinstance(v, torch.Tensor) else v) for k, v in gs.items()}


def points_around(gs, ids, per_gaussian, jitter, seed):
    """`per_gaussian` query points within `jitter` (uniform, per axis) of the centre of each Gaussian in `ids`."""
    rng = np.random.default_rng(seed)
    m = gs["means3D"].numpy().astype(np.float64)[np.asarray(ids)]
    p = np.repeat(m, per_gaussian, axis=0) + (rng.random((len(m) * per_gaussian, 3)) * 2 - 1) * jitter
    return torch.from_numpy(p.astype(np.float32))


def cam_to_world(cam, p_cam):
    """World coordinates (float64 [N,3]) of camera-space points: p_cam = R^T p_w + T with [R^T | T] the view matrix."""
    w2v = cam.world_view_transform.double().numpy().T
    return (np.asarray(p_cam, np.float64) - w2v[:3, 3]) @ w2v[:3, :3]


def pixel_to_cam(cam, x, y, z):
    """Camera-space point that projects to the continuous image position (x, y) at depth z."""
    W, H = cam.image_width, cam.image_height
    fx, fy = W / (2.0 * cam.tanfovx), H / (2.0 * cam.tanfovy)
    x, y, z = np.broadcast_arrays(np.asarray(x, np.float64), np.asarray(y, np.float64), np.asarray(z, np.float64))
    return np.stack([(x - W / 2.0) * z / fx, (y - H / 2.0) * z / fy, z], axis=-1)


def blobs(cam, xy, depth, sigma_px, opacity, seed=0, sh_degree=0):
    """Isotropic Gaussians centred on image positions `xy` [N,2] at `depth` [N], `sigma_px` pixels wide at that depth."""
    n = len(xy)
    rng = np.random.default_rng(seed)
    depth = np.broadcast_to(np.asarray(depth, np.float64), (n,))
    fx = cam.image_width / (2.0 * cam.tanfovx)
    means = cam_to_world(cam, pixel_to_cam(cam, np.asarray(xy)[:, 0], np.asarray(xy)[:, 1], depth))
    s = np.broadcast_to(np.asarray(sigma_px, np.float64), (n,)) * depth / fx
    shs = np.zeros((n, 16, 3))
    shs[:, 0, :] = (rng.random((n, 3)) * 2 - 1) * 1.77
    rot = np.zeros((n, 4))
    rot[:, 0] = 1.0
    f32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32))   # noqa: E731
    return {"means3D": f32(means), "scales": f32(np.repeat(s[:, None], 3, 1)), "rotations": f32(rot),
            "opacities": f32(np.broadcast_to(np.asarray(opacity, np.float64), (n,))[:, None]), "shs": f32(shs), "sh_degree": sh_degree}


def concat(parts):
    return {k: (torch.cat([p[k] for p in parts]).contiguous() if isinstance(parts[0][k], torch.Tensor) else parts[0][k]) for k in parts[0]}


def cap_scene():
    """48x32 pixels under 1 600 wide Gaussians of opacity 0.012: a pixel records every Gaussian whose centre is within
    1.5 sigma of it, so pixels near the middle reach the 1 024-contributor cap and stop while pixels near the rim do not."""
    cam = gof_synth.make_camera(48, 32, view=3)
    rng = np.random.default_rng(7)
    n = 1600
    xy = np.stack([rng.normal(24, 14, n), rng.normal(16, 10, n)], 1)
    gs = blobs(cam, xy, rng.uniform(3.0, 5.0, n), 16.0, 0.012, seed=8)
    pts = torch.from_numpy(cam_to_world(cam, pixel_to_cam(cam, rng.uniform(0, 48, 4000), rng.uniform(0, 32, 4000), rng.uniform(2.5, 5.5, 4000))).astype(np.float32))
    return cam, gs, pts


U16_FILL = 70_000


def u16_scene():
    """32x16 pixels (two tiles) under 70 000 Gaussians that are in both tile lists but too faint to be recorded, ordered by
    depth, plus five opaque ones placed at chosen positions of the lists:
      tile 0  A at 65 000 over pixels (2..5, 2..5), B at 65 541 over (2..5, 2..5) and (9..12, 9..12);
      tile 1  C at 65 536 over pixels (20..23, 4..7);
      both    Z last (70 00x), over the whole image.
    Pixel (10, 10): the first contributor is B, recorded as uint16 id 5.  Pixel (3, 3): ids 65 000, 5: the second can never be
    matched by the running index.  Pixel (21, 5): the first id is 65 536 -> 0.
    Returns (cam, gs, pts, pixels) with pixels = dict of the (x, y) named above."""
    cam = gof_synth.make_camera(32, 16, view=5)
    n = U16_FILL
    d = 3.0 + 2.0 * np.arange(n) / n                     # filler k (0-based) has k fillers in front of it
    between = lambda k: 3.0 + 2.0 * (k - 0.5) / n        # noqa: E731  a depth with exactly k fillers in front
    fill = blobs(cam, np.tile([[16.0, 8.0]], (n, 1)), d, 30.0, 0.001, seed=1)
    # list position (1-based) = fillers in front + opaque Gaussians of the same tile in front + 1
    A = blobs(cam, [[4.0, 4.0]], between(64_999), 1.2, 0.6, seed=2)     # tile 0: 64 999 fillers in front -> position 65 000
    B1 = blobs(cam, [[4.0, 4.0]], between(65_539), 1.2, 0.6, seed=3)    # tile 0: 65 539 fillers + A -> 65 541
    C = blobs(cam, [[22.0, 6.0]], between(65_535), 1.2, 0.6, seed=5)    # tile 1: 65 535 fillers -> 65 536
    Z = blobs(cam, [[16.0, 8.0]], 5.5, 60.0, 0.5, seed=6)
    # B must cover two separate pixel groups of tile 0 with one Gaussian: a needle along the diagonal through (4,4) and (11,11)
    B = dict(B1)
    fx = cam.image_width / (2.0 * cam.tanfovx)
    px = between(65_539) / fx
    B["means3D"] = torch.from_numpy(cam_to_world(cam, pixel_to_cam(cam, [7.5], [7.5], between(65_539))).astype(np.float32))
    B["scales"] = torch.tensor([[6.0 * px, 1.0 * px, 1.0 * px]], dtype=torch.float32)
    # rotate the long axis onto the image diagonal: camera-space direction (1, 1, 0) expressed in world space
    w2v = cam.world_view_transform.double().numpy().T
    Rc = w2v[:3, :3].T                                    # columns: camera axes in world coordinates
    e0 = (Rc[:, 0] + Rc[:, 1]) / math.sqrt(2.0)
    e1 = (Rc[:, 1] - Rc[:, 0]) / math.sqrt(2.0)
    e2 = np.cross(e0, e1)
    B["rotations"] = torch.from_numpy(_quat(np.stack([e0, e1, e2], 1)).astype(np.float32))[None]
    gs = concat([fill, A, B, C, Z])
    rng = np.random.default_rng(11)
    m = 6000
    pts = torch.from_numpy(cam_to_world(cam, pixel_to_cam(cam, rng.uniform(0, 32, m), rng.uniform(0, 16, m), rng.uniform(2.5, 6.0, m))).astype(np.float32))
    return cam, gs, pts, dict(first_wrapped=(10, 10), wrapped_after=(3, 3), id_zero=(21, 5))


def tile_stack(cam, tx, ty, n, seed, opacity=(0.005, 0.015), sigma=0.5, depth=(2.0, 6.0), spread=2.5, at=(8.0, 8.0)):
    """n Gaussians whose tile rectangle is tile (tx, ty) alone: centres within `spread` px of the tile position `at`,
    `sigma` px wide (the rectangle reaches radius ~ 3 sigma px beyond the centre)."""
    rng = np.random.default_rng(seed)
    xy = np.stack([16 * tx + at[0] + rng.uniform(-spread, spread, n), 16 * ty + at[1] + rng.uniform(-spread, spread, n)], 1)
    return blobs(cam, xy, rng.uniform(*depth, n), sigma, rng.uniform(*opacity, n), seed=seed)


SAT_AT = [3, 32, 33, 256, 257]


def saturation_scene():
    """One row of tiles; tile k saturates its centre pixel at list position SAT_AT[k]: faint fillers in a tile corner, then
    opaque layers on the centre, then more fillers; the centre pixel's last contributor is the entry before."""
    cam = gof_synth.make_camera(16 * len(SAT_AT), 16, view=6)
    parts = []
    for t, s in enumerate(SAT_AT):
        if s > 3:
            parts.append(tile_stack(cam, t, 0, s - 3, seed=200 + t, depth=(1.5, 2.0), spread=1.0, at=(4.5, 4.5)))
        layers = blobs(cam, np.tile([[16 * t + 8.5, 8.5]], (5, 1)), 2.5 + 0.05 * np.arange(5), 2.0, 0.97, seed=210 + t)
        parts += [layers, tile_stack(cam, t, 0, 60, seed=220 + t, depth=(3.0, 4.0), spread=1.0, at=(11.5, 11.5))]
    return cam, concat(parts)


def threshold_scene():
    """96x64 pixels under opacities on and around the blend's alpha thresholds: in 1/255 (1 + [1e-5, 2e-3]) (the window the
    pre-reject's 2e-3 margin must keep), exactly float(1/255) and a few ulp either side of it, in [0.00392, 1/255), 0, and
    0.99, 0.995 and 1.0 (the clamp); over wide faint Gaussians, a thin ring of each of which lies in that window, and under
    which no pixel saturates."""
    cam = gof_synth.make_camera(96, 64, view=12)
    rng = np.random.default_rng(13)
    xy = lambda n: np.stack([rng.uniform(-4, 100, n), rng.uniform(-4, 68, n)], 1)   # noqa: E731
    a = np.float64(np.float32(1.0 / 255.0))
    ulps = np.nextafter(np.float32(a), np.float32(1)) - np.float32(a)
    groups = [
        (300, a * (1 + rng.uniform(1e-5, 2e-3, 300)), rng.uniform(2.0, 8.0, 300)),
        # the stored opacity is op * coef, coef = sqrt(det0 / (det1 + 1e-6) + 1e-6) a few 1e-7 above 1: a spread of ulps below
        (200, a + ulps * rng.integers(-16, 2, 200), rng.uniform(1.0, 6.0, 200)),
        (30, rng.uniform(0.00392, a, 30), rng.uniform(1.0, 6.0, 30)),
        (30, np.zeros(30), rng.uniform(1.0, 6.0, 30)),
        (90, np.repeat([0.99, 0.995, 1.0], 30), rng.uniform(0.5, 2.0, 90)),
        (300, rng.uniform(0.01, 0.05, 300), rng.uniform(12.0, 25.0, 300)),
    ]
    parts = [blobs(cam, xy(n), rng.uniform(2.0, 6.0, n), s, np.asarray(op, np.float32), seed=40 + i) for i, (n, op, s) in enumerate(groups)]
    return cam, concat(parts)


def _quat(R):
    """(w, x, y, z) of a proper rotation matrix."""
    w = math.sqrt(max(0.0, 1.0 + R[0, 0] + R[1, 1] + R[2, 2])) / 2.0
    if w > 1e-6:
        return np.array([w, (R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w)])
    x = math.sqrt(max(0.0, 1.0 + R[0, 0] - R[1, 1] - R[2, 2])) / 2.0
    return np.array([(R[2, 1] - R[1, 2]) / (4 * x), x, (R[0, 1] + R[1, 0]) / (4 * x), (R[0, 2] + R[2, 0]) / (4 * x)])
