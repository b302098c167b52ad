"""CPU: the product's arithmetic header (csrc/gof_math.cuh), compiled for the host by tests/hostmath, against
the CPU oracle and the golden fixtures: the explicit-rounding restatement must be BIT-exact for everything
that feeds tile indices and the view2gaussian record, with no GPU in the loop."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import _golden
import gof_oracle
import gof_synth

HERE = os.path.dirname(os.path.abspath(__file__))
HM_DIR = os.path.join(HERE, "hostmath")


@pytest.fixture(scope="module")
def hm():
    lib = os.path.join(HM_DIR, "libhostmath.so")
    src = os.path.join(HM_DIR, "hostmath.cpp")
    hdr = os.path.join(HERE, "..", "gaussian-opacity-fields_b200", "csrc", "gof_math.cuh")
    if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math",
                               "-x", "c++", src, "-o", lib])
    return ctypes.CDLL(lib)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _run_preprocess(hm, sc):
    P = sc.P
    out = dict(cov3D=np.zeros((P, 6), np.float32), conic_opacity=np.zeros((P, 4), np.float32),
               means2D=np.zeros((P, 2), np.float32), depths=np.zeros(P, np.float32), radii=np.zeros(P, np.int32),
               tiles_touched=np.zeros(P, np.uint32), view2gaussian=np.zeros((P, 10), np.float32))
    a = sc.arr
    for i in range(P):
        r, t, d = ctypes.c_int(0), ctypes.c_uint(0), ctypes.c_float(0)
        ok = hm.hm_preprocess_one(_p(a["means3D"][i]), _p(a["scales"][i]), _p(a["rotations"][i]),
                                  ctypes.c_float(float(a["opacities"].reshape(-1)[i])), ctypes.c_float(sc.scale_modifier),
                                  _p(a["viewmatrix"]), _p(a["projmatrix"]), sc.W, sc.H, ctypes.c_float(sc.tan_fovx),
                                  ctypes.c_float(sc.tan_fovy), ctypes.c_float(sc.kernel_size), _p(out["cov3D"][i]),
                                  _p(out["conic_opacity"][i]), _p(out["means2D"][i]), ctypes.byref(d), ctypes.byref(r),
                                  ctypes.byref(t), _p(out["view2gaussian"][i]))
        if ok:
            out["radii"][i], out["tiles_touched"][i], out["depths"][i] = r.value, t.value, d.value
    return out


@pytest.mark.parametrize("path", _golden.fixture_paths(), ids=[p.split("/")[-1] for p in _golden.fixture_paths()])
def test_product_math_bit_exact_vs_reference_golden(hm, path):
    fx = _golden.load(path)
    sc = _golden.oracle_scene(fx)
    out = _run_preprocess(hm, sc)
    vis = fx["visible"]
    np.testing.assert_array_equal(out["radii"], fx["radii"])
    np.testing.assert_array_equal(out["tiles_touched"], fx["tiles_touched"].view(np.uint32))
    for f in ("depths", "means2D", "conic_opacity", "view2gaussian"):
        np.testing.assert_array_equal(out[f][vis].view(np.int32), fx[f][vis].view(np.int32), err_msg=f)


def test_product_math_bit_exact_vs_oracle_random_scene(hm):
    cam, gs = gof_synth.make_scene(dict(P=3000, width=200, height=120, seed=77), view=21)
    sc = gof_oracle.scene_from_synth(cam, gs, kernel_size=0.05, scale_modifier=1.3)
    g = gof_oracle.preprocess(sc)
    out = _run_preprocess(hm, sc)
    vis = g["radii"] > 0
    assert vis.sum() > 1000
    np.testing.assert_array_equal(out["radii"], g["radii"])
    np.testing.assert_array_equal(out["tiles_touched"], g["tiles_touched"])
    for f in ("depths", "means2D", "conic_opacity", "view2gaussian", "cov3D"):
        np.testing.assert_array_equal(out[f][vis].view(np.int32), g[f][vis].view(np.int32), err_msg=f)


def test_pair_math_matches_oracle_render(hm):
    """A/B/t/power of the ray-Gaussian intersection: product header vs an independent numpy float64 evaluation."""
    fx = _golden.load(_golden.fixture_paths()[0])
    cfg = fx["cfg"]
    W, H = cfg["W"], cfg["H"]
    fx_, fy_ = W / (2.0 * float(fx["tanfovx"])), H / (2.0 * float(fx["tanfovy"]))
    vis = np.nonzero(fx["visible"])[0][:200]
    rng = np.random.default_rng(0)
    out = np.zeros(9, np.float32)
    for gidx in vis:
        v = np.ascontiguousarray(fx["view2gaussian"][gidx])
        px, py = int(rng.integers(0, W)), int(rng.integers(0, H))
        hm.hm_pair(_p(v), px, py, W, H, ctypes.c_float(fx_), ctypes.c_float(fy_), _p(out))
        rx = np.float32((np.float64(np.float32(px) + np.float32(0.5)) - W / 2.0) / np.float64(np.float32(fx_)))
        ry = np.float32((np.float64(np.float32(py) + np.float32(0.5)) - H / 2.0) / np.float64(np.float32(fy_)))
        r = np.array([rx, ry, 1.0], np.float64)
        S = np.array([[v[0], v[1], v[2]], [v[1], v[3], v[4]], [v[2], v[4], v[5]]], np.float64)
        AA = r @ S @ r
        BB = 2.0 * (np.array(v[6:9], np.float64) @ r)
        scale = max(abs(S).max() * (r ** 2).max(), 1.0)
        assert abs(out[0] - AA) <= 1e-5 * scale
        assert abs(out[1] - BB) <= 1e-5 * max(abs(v[6:9]).max() * 2, 1.0)
        # t and power are evaluated in double FROM the float A/B (forward.cu:516-524)
        t = np.float32(-np.float64(out[1]) / (2 * np.float64(out[0])))
        assert out[2] == t
        pw = np.float32(-0.5 * (-(np.float64(out[1]) / np.float64(out[0])) * (np.float64(out[1]) / 4.0) + np.float64(v[9])))
        pw = min(pw, np.float32(0.0))
        assert abs(out[3] - pw) <= 1e-6 * max(abs(pw), 1.0)


def test_tile_slots_and_box_packing(hm):
    """The thread <-> pixel map of a 16x16 tile, the pixel slot of a projected point, and the 16-bit box packing with its overlap
    test against a warp's 8x4 block, checked against plain integer arithmetic."""
    i32 = ctypes.POINTER(ctypes.c_int)
    # every thread of a tile gets its own pixel, and gof_pixel_slot maps that pixel back to the thread
    for tile_x, tile_y in ((0, 0), (3, 1), (119, 67)):
        seen = set()
        out = np.zeros(4, np.int32)
        for t in range(256):
            warp, lane = t >> 5, t & 31
            hm.hm_warp_block(tile_x, tile_y, warp, lane, _p(out))
            wx0, wy0, px, py = (int(v) for v in out)
            assert (wx0, wy0) == (tile_x * 16 + (warp & 1) * 8, tile_y * 16 + (warp >> 1) * 4)
            assert wx0 <= px < wx0 + 8 and wy0 <= py < wy0 + 4
            lx, ly = px - tile_x * 16, py - tile_y * 16
            assert hm.hm_pixel_slot(lx, ly) == t
            seen.add((lx, ly))
        assert len(seen) == 256

    # a point falls in the pixel that contains it (pix <= xy < pix + 1), clamped to its tile
    rng = np.random.default_rng(5)
    W, H = 1920, 1080
    xy = np.concatenate([
        rng.uniform(0, [W, H], (4000, 2)),
        np.stack(np.meshgrid(np.arange(0, W + 1, 16.0), [0.0, 15.5, 16.0, H - 1e-3])).reshape(2, -1).T,   # tile edges
        [[np.nextafter(np.float32(16), 0), 0.0], [np.nextafter(np.float32(W), 0), np.nextafter(np.float32(H), 0)]],
    ]).astype(np.float32)
    tile = np.minimum((xy // 16).astype(np.int32), [(W + 15) // 16 - 1, (H + 15) // 16 - 1]).astype(np.int32)
    # and points the clamp takes to the tile's edge: left of / above it (trunc towards 0), and past its right / lower edge
    xy = np.concatenate([xy, [[-0.75, -0.25], [5.0, -3.0], [40.0, 3.0], [3.0, 47.9]]]).astype(np.float32)
    tile = np.concatenate([tile, [[0, 0], [0, 0], [1, 0], [0, 1]]]).astype(np.int32)
    slots = np.zeros(len(xy), np.int32)
    hm.hm_point_slots(len(xy), _p(xy), _p(tile), _p(slots))
    lxy = np.clip(np.trunc(xy).astype(np.int64) - tile * 16, 0, 15)
    lx, ly = lxy[:, 0], lxy[:, 1]
    expect = ((ly >> 2) * 2 + (lx >> 3)) * 32 + (ly & 3) * 8 + (lx & 7)
    np.testing.assert_array_equal(slots, expect)
    own = (xy >= tile * 16).all(1) & (xy < (tile + 1) * 16).all(1)   # the point lies in its tile: no clamp, the containing pixel
    assert (~own).sum() == 8   # x = W on the image's right edge (four rows), and the four points placed outside their tile
    np.testing.assert_array_equal(lxy[own], np.floor(xy[own]).astype(np.int64) - tile[own] * 16)

    # box packing: every bound in [-32768, 32767], the full and the empty box among them
    lo, hi = -32768, 32767
    edge = np.array([lo, lo + 1, -8, -1, 0, 1, 7, hi - 7, hi - 1, hi])
    n = 20000
    box = rng.integers(lo, hi + 1, (n, 4))
    pick = rng.random((n, 4)) < 0.3
    box[pick] = rng.choice(edge, pick.sum())
    small = rng.random(n) < 0.5   # boxes of a few pixels near the blocks, where the overlap test is decided at the edges
    box[small, 0:2] = rng.integers(-40, 40, (small.sum(), 2))
    box[small, 2:4] = box[small, 0:2] + rng.integers(-2, 12, (small.sum(), 2))
    box = np.concatenate([box, [[lo, lo, hi, hi], [hi, hi, lo, lo]] * 4]).astype(np.int32)
    rect = rng.integers(-48, 48, (len(box), 2))
    rect[:n][small] = box[:n][small, 0:2] + rng.integers(-10, 4, (small.sum(), 2))
    rect[-8:] = [[lo, lo], [lo, lo], [hi - 7, hi - 3], [hi - 7, hi - 3], [0, 0], [0, 0], [-8, -4], [-8, -4]]
    rect = rect.astype(np.int32)
    words = np.zeros((len(box), 2), np.uint32)
    hits = np.zeros(len(box), np.int32)
    hm.hm_box_hits(len(box), _p(box), _p(rect), _p(words), _p(hits))
    b = box.astype(np.int64)
    np.testing.assert_array_equal(words[:, 0], (b[:, 0] & 0xFFFF) | ((b[:, 1] & 0xFFFF) << 16))
    np.testing.assert_array_equal(words[:, 1], (b[:, 2] & 0xFFFF) | ((b[:, 3] & 0xFFFF) << 16))
    wx0, wy0 = rect[:, 0].astype(np.int64), rect[:, 1].astype(np.int64)
    expect = (b[:, 0] <= wx0 + 7) & (b[:, 2] >= wx0) & (b[:, 1] <= wy0 + 3) & (b[:, 3] >= wy0)
    np.testing.assert_array_equal(hits.astype(bool), expect)
    assert hits[-8::2].all() and not hits[-7::2].any()   # the full box hits every block, the empty box none
    assert 0.05 < expect[:n][small].mean() < 0.95
