"""CPU: the culling box (gof_cull_bbox in csrc/gof_math.cuh, host twin) is conservative: every pixel at which the
reference's pair test accepts a Gaussian (oracle_alpha_map) lies inside that Gaussian's box -- including strongly
anisotropic Gaussians, large and tiny footprints, and a camera inside the cloud.  The opacity-field query casts four more
rays per pixel, through its corners: the box it is given (margin 0.5) holds every pixel at which ANY of the five rays
accepts (oracle_ray_mask_map), also for Gaussians thinner than a pixel and for Gaussians centred on pixel corners, pixel
edges, tile borders and the image border."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import _integrate_scenes as scenes
import gof_oracle
import gof_synth

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def hm():
    d = os.path.join(HERE, "hostmath")
    lib, src = os.path.join(d, "libhostmath.so"), os.path.join(d, "hostmath.cpp")
    hdr = os.path.join(HERE, "..", "gaussian-opacity-fields_b200", "csrc", "gof_math.cuh")
    if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-x", "c++", src, "-o", lib])
    return ctypes.CDLL(lib)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


CASES = [
    dict(P=500, W=96, H=64, seed=1, sigma_px=2.0, radius=4.0, aniso=(0.3, 1.0)),
    dict(P=300, W=80, H=60, seed=2, sigma_px=0.6, radius=4.0, aniso=(0.3, 1.0)),     # sub-pixel Gaussians, C ~ 1e6
    dict(P=200, W=64, H=48, seed=3, sigma_px=12.0, radius=4.0, aniso=(0.3, 1.0)),    # screen-filling
    dict(P=400, W=96, H=64, seed=4, sigma_px=3.0, radius=4.0, aniso=(0.01, 1.0)),    # needles / pancakes 100:1
    dict(P=400, W=96, H=64, seed=5, sigma_px=3.0, radius=1.0, aniso=(0.1, 1.0)),     # camera inside the cloud
]


@pytest.mark.parametrize("case", CASES + ["needles", "placed", "thresholds"],
                         ids=[f"case{i}" for i in range(len(CASES))] + ["needles", "placed", "thresholds"])
def test_box_contains_every_accepted_pixel(hm, case):
    """The blend's box (margin 0, centre rays), also for sub-pixel needles, Gaussians centred on pixel corners, edges and
    borders, and opacities on and around 1/255 (_integrate_scenes.threshold_scene)."""
    if case == "needles":
        cam, gs = scenes.needle_scene()
    elif case == "placed":
        cam, gs = _placed_scene()
    elif case == "thresholds":
        cam, gs = scenes.threshold_scene()
    else:
        cam = gof_synth.make_camera(case["W"], case["H"], view=case["seed"] * 7, radius=case["radius"])
        gs = gof_synth.make_gaussians(case["P"], case["seed"], cam.focal_x, sigma_px=case["sigma_px"])
        lo, hi = case["aniso"]
        g = torch.Generator().manual_seed(case["seed"] + 99)
        an = torch.exp(torch.rand(case["P"], 3, generator=g) * np.log(hi / lo) + np.log(lo))
        gs["scales"] = (gs["scales"].max(dim=1, keepdim=True).values * an).contiguous()
    sc = gof_oracle.scene_from_synth(cam, gs)
    st = gof_oracle.preprocess(sc)
    vis = np.nonzero(st["radii"] > 0)[0]
    assert len(vis) > 50
    W, H = sc.W, sc.H
    tight = nonempty = 0
    box = np.zeros(4, np.int32)
    for gid in vis:
        v = np.ascontiguousarray(st["view2gaussian"][gid])
        op = float(st["conic_opacity"][gid, 3])
        scale = np.ascontiguousarray(sc.arr["scales"][gid])
        hm.hm_bbox(_p(v), ctypes.c_float(op), _p(scale), W, H, ctypes.c_float(sc.tan_fovx), ctypes.c_float(sc.tan_fovy), _p(box))
        amap = gof_oracle.alpha_map(W, H, sc.tan_fovx, sc.tan_fovy, v, op)
        ys, xs = np.nonzero(amap > 0)
        if len(xs) == 0:
            continue
        nonempty += 1
        assert box[0] <= xs.min() and xs.max() <= box[2] and box[1] <= ys.min() and ys.max() <= box[3], \
            f"gaussian {gid}: accepted pixels x[{xs.min()},{xs.max()}] y[{ys.min()},{ys.max()}] outside box {box.tolist()}"
        if box[0] > -30000:
            tight += 1
    assert nonempty > 20
    if isinstance(case, str) or case["radius"] >= 4.0:
        assert tight > 0.5 * nonempty, "the box should be finite for most Gaussians in front of the camera"


def _placed_scene():
    """Sub-pixel needles and pancakes centred exactly on pixel corners, pixel edges, tile borders and the image border."""
    W, H = 96, 64
    cam = gof_synth.make_camera(W, H, view=21)
    rng = np.random.default_rng(17)
    xs = np.concatenate([rng.integers(0, W + 1, 150), rng.integers(0, W + 1, 150), rng.integers(0, W, 150) + 0.5,   # corners, x edges, y edges
                         16.0 * rng.integers(0, W // 16 + 1, 150), rng.choice([0.0, W], 75), rng.uniform(0, W, 75)])
    ys = np.concatenate([rng.integers(0, H + 1, 150), rng.integers(0, H, 150) + 0.5, rng.integers(0, H + 1, 150),
                         16.0 * rng.integers(0, H // 16 + 1, 150), rng.uniform(0, H, 75), rng.choice([0.0, H], 75)])
    n = len(xs)
    gs = scenes.blobs(cam, np.stack([xs, ys], 1), rng.uniform(3.0, 5.0, n), rng.uniform(0.3, 1.5, n), rng.uniform(0.05, 1.0, n), seed=18)
    an = np.exp(rng.uniform(np.log(0.05), 0.0, (n, 3)))
    gs["scales"] = (gs["scales"] * torch.from_numpy(an.astype(np.float32))).contiguous()
    q = rng.normal(size=(n, 4))
    gs["rotations"] = torch.from_numpy((q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32))
    return cam, gs


FIVE_RAY_CASES = CASES + [scenes.NEEDLE_CASE, "placed"]


@pytest.mark.parametrize("case", FIVE_RAY_CASES, ids=[f"case{i}" for i in range(len(CASES))] + ["needles", "placed"])
def test_query_box_contains_every_pixel_a_corner_or_centre_ray_accepts(hm, case):
    """k_integrate visits a Gaussian for a warp only when the box preprocess stored for the query (margin 0.5) holds one of the
    warp's pixels, with no further widening: so every pixel where one of the five rays accepts must be inside that box."""
    cam, gs = _placed_scene() if case == "placed" else scenes.aniso_scene(case)
    sc = gof_oracle.scene_from_synth(cam, gs)
    st = gof_oracle.preprocess(sc)
    vis = np.nonzero(st["radii"] > 0)[0]
    W, H = sc.W, sc.H
    box, box0 = np.zeros(4, np.int32), np.zeros(4, np.int32)
    nonempty = corner_only = slipped = 0
    for gid in vis:
        v = np.ascontiguousarray(st["view2gaussian"][gid])
        op = float(st["conic_opacity"][gid, 3])
        scale = np.ascontiguousarray(sc.arr["scales"][gid])
        args = (_p(v), ctypes.c_float(op), _p(scale), W, H, ctypes.c_float(sc.tan_fovx), ctypes.c_float(sc.tan_fovy))
        hm.hm_bbox_margin(*args, ctypes.c_float(0.5), _p(box))
        hm.hm_bbox(*args, _p(box0))
        mask = gof_oracle.ray_mask_map(W, H, sc.tan_fovx, sc.tan_fovy, v, op)
        ys, xs = np.nonzero(mask)
        if len(xs) == 0:
            continue
        nonempty += 1
        corner_only += not (mask & 1).any()
        slipped += box0[0] > box0[2] and op >= 1.0 / 255.0
        assert box[0] <= xs.min() and xs.max() <= box[2] and box[1] <= ys.min() and ys.max() <= box[3], \
            f"gaussian {gid}: pixels x[{xs.min()},{xs.max()}] y[{ys.min()},{ys.max()}] with an accepting ray outside box {box.tolist()}"
        # the blend's box never reaches beyond the query's
        assert box[0] <= box0[0] and box0[2] <= box[2] and box[1] <= box0[1] and box0[3] <= box[3] or box0[0] > box0[2]
    assert nonempty > 20
    if case is scenes.NEEDLE_CASE or case == "placed":
        # the scenes reach the case they are for: Gaussians no centre ray meets, whose centre-ray box is empty
        assert corner_only > 50 and slipped > 50, (corner_only, slipped)
