"""CPU: the tetrahedra points and their frustum mask (csrc/tetra_points.cuh compiled for the host) against the numpy oracle
(oracle/tetra_points_oracle.py), and the oracle against the reference's own get_frustum_mask run on the CPU from its staged
source (scene/gaussian_model.py:31-72).  Parity rule (DESIGN §4.8): the Gaussian-side scalars and the centres are
bit-identical; corners lie within the rounding bound of the 3-term product; the mask agrees with the float64 decision
wherever that decision is outside the rounding bound ("decided"), and the undecided points are counted."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import _tetra_scenes as ts
import gof_synth
import tetra_points_oracle as tpo

HERE = os.path.dirname(os.path.abspath(__file__))
_p = lambda a: a.ctypes.data_as(ctypes.c_void_p)   # noqa: E731


@pytest.fixture(scope="module")
def hm():
    d = os.path.join(HERE, "hostmath")
    lib, src = os.path.join(d, "libtetra_points_host.so"), os.path.join(d, "tetra_points_host.cpp")
    hdr = os.path.join(HERE, "..", "gaussian-opacity-fields_b200", "csrc", "tetra_points.cuh")
    if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-x", "c++", src, "-o", lib])
    h = ctypes.CDLL(lib)
    h.hm_tp_points.argtypes = [ctypes.c_int] + [ctypes.c_void_p] * 3 + [ctypes.c_int, ctypes.c_void_p, ctypes.c_float, ctypes.c_float] + \
        [ctypes.c_void_p] * 3
    h.hm_tp_mask.argtypes = [ctypes.c_longlong, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_float, ctypes.c_float, ctypes.c_void_p]
    h.hm_tp_corner_sign.restype = ctypes.c_float
    return h


def _host_points(hm, xyz, scales, rot, table, near=0.02, far=1e6):
    P = xyz.shape[0]
    pts, sc, m = np.zeros((9 * P, 3), np.float32), np.zeros(9 * P, np.float32), np.zeros(9 * P, np.uint8)
    hm.hm_tp_points(P, _p(xyz), _p(scales), _p(rot), table.shape[0], _p(table), near, far, _p(pts), _p(sc), _p(m))
    return pts, sc, m.astype(bool)


def _scene(P, seed, kind, n_views, W, H):
    xyz, s, r = (t.numpy() for t in ts.gaussians(P, seed, kind))
    views = (ts.surface_views if kind == "surface" else ts.ring_views)(n_views, W, H)
    return np.ascontiguousarray(xyz), np.ascontiguousarray(s), np.ascontiguousarray(r), views


def _same_bits(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def test_box_order_matches_gof_synth_and_trimesh(hm):
    table = np.array([[hm.hm_tp_corner_sign(k, a) for a in range(3)] for k in range(8)], np.float32)
    assert np.array_equal(table, tpo.BOX_SIGNS)
    # gof_synth.make_tetra_points: identity rotation, unit 3-sigma half-extent, centre at the origin -> the corners are the signs
    gs = {"means3D": torch.zeros(1, 3), "scales": torch.full((1, 3), 1.0 / 3.0), "rotations": torch.tensor([[1.0, 0.0, 0.0, 0.0]])}
    pts, _sc = gof_synth.make_tetra_points(gs, 9, seed=0, device="cpu")
    assert np.array_equal(np.sign(pts[:8].numpy()), tpo.BOX_SIGNS)
    try:
        import trimesh
    except ImportError:
        return
    assert np.array_equal(trimesh.creation.box().vertices * 2, tpo.BOX_SIGNS)


@pytest.mark.parametrize("kind,P,n_views,W,H", [("random", 4000, 16, 320, 200), ("surface", 3000, 6, 256, 256)])
def test_host_twin_matches_oracle(hm, kind, P, n_views, W, H):
    xyz, s, r, views = _scene(P, 11 + P, kind, n_views, W, H)
    # a zero quaternion (NaN corners) and a NaN scale (NaN point scale) ride along
    r[5] = 0.0
    s[7, 1] = np.nan
    table = np.ascontiguousarray(tpo.pack_views(views))
    R = np.zeros((P, 9), np.float32)
    s3, ps = np.zeros((P, 3), np.float32), np.zeros(P, np.float32)
    hm.hm_tp_frame(P, _p(r), _p(s), _p(R), _p(s3), _p(ps))
    oR, os3, ops = tpo.frame(r, s)
    assert _same_bits(R, oR.reshape(P, 9)) and _same_bits(s3, os3) and _same_bits(ps, ops)

    pts, sc, m = _host_points(hm, xyz, s, r, table)
    opts, obnd, osc = tpo.tetra_points(xyz, s, r)
    assert _same_bits(pts[8 * P:], xyz) and _same_bits(sc, osc)
    fin = np.isfinite(opts).all(1)
    assert not np.isfinite(pts[:8 * P][~fin[:8 * P]]).all(1).any()       # the zero quaternion's corners are NaN
    assert (np.abs(pts[fin] - opts[fin]) <= obnd[fin]).all()
    assert not m[8 * 5:8 * 6].any() and m[8 * P + 5] == tpo.frustum_decision(xyz[5:6], table)[0][0]

    mask64, decided = tpo.frustum_decision(pts, table)
    bad = decided & (m != mask64)
    print(f"[tetra host {kind}] points {m.size}  in {int(m.sum())}  undecided {int((~decided).sum())}  disagreeing {int(bad.sum())}")
    assert not bad.any()
    assert m.sum() > 0.3 * m.size and (~m).sum() > 0


def test_edge_points_on_the_host(hm):
    view, pts, exp = ts.edge_scene()
    table = np.ascontiguousarray(tpo.pack_views([view]))
    m = np.zeros(len(pts), np.uint8)
    hm.hm_tp_mask(len(pts), _p(pts), 1, _p(table), 0.02, 1e6, _p(m))
    assert np.array_equal(m.astype(bool), exp)
    mask64, decided = tpo.frustum_decision(pts, table)
    assert np.array_equal(mask64, exp)


def test_reference_frustum_mask_on_cpu_agrees_with_oracle():
    ref = ts.ref_frustum_mask()
    if ref is None:
        pytest.skip("the reference's scene/gaussian_model.py is not staged (baseline/stage_ref.sh)")
    for kind, P, n, W, H in (("random", 3000, 12, 320, 200), ("surface", 3000, 5, 200, 150)):
        xyz, s, r, views = _scene(P, 5 + P, kind, n, W, H)
        # the quirk: the later views' sizes differ from views[0]'s, whose W and H the reference uses for every view
        views[1].image_width, views[1].image_height = 2 * W, 2 * H
        opts, obnd, _sc = tpo.tetra_points(xyz, s, r)
        pts = opts.astype(np.float32)
        got = ref(torch.from_numpy(pts), views).numpy()
        mask64, decided = tpo.frustum_decision(pts, tpo.pack_views(views))
        bad = decided & (got != mask64)
        print(f"[tetra ref-cpu {kind}] points {got.size}  in {int(got.sum())}  undecided {int((~decided).sum())}  disagreeing {int(bad.sum())}")
        assert not bad.any()
    view, pts, exp = ts.edge_scene()
    assert np.array_equal(ref(torch.from_numpy(pts), [view]).numpy(), exp)
