"""CPU: the brute-force oracle of distCUDA2 (oracle/knn_oracle.c) states the contract of DESIGN section 4.5 -- checked against
scipy's k-d tree and against hand-worked edge cases."""
from fractions import Fraction

import numpy as np
import pytest

import gof_synth
import knn_oracle

FMAX = np.float32(np.finfo(np.float32).max)


def _r32(x):
    """An exact rational rounded to the nearest float32 (ties to even)."""
    if x == 0:
        return np.float32(0)
    f = np.float32(float(x))
    cands = [np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))]
    return np.float32(min(cands, key=lambda v: (abs(Fraction(float(v)) - x), int(np.float32(v).view(np.uint32)) & 1)))


def _fma(a, b, c):
    return _r32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def _mean(b):
    return np.float32(np.float32(np.float32(b[0]) + np.float32(b[1])) + np.float32(b[2])) / np.float32(3)


def test_agrees_with_kdtree():
    from scipy.spatial import cKDTree
    for kind, P, seed in (("uniform", 3000, 1), ("colmap", 4000, 2), ("plane", 2000, 3)):
        pts = gof_synth.make_point_cloud(kind, P, seed)
        if kind == "colmap":   # the k-d tree cannot tell exact duplicates from the query itself
            pts = np.unique(pts, axis=0)
        mean, best = knn_oracle.knn_mean_dist(pts, return_best=True)
        d, _ = cKDTree(pts.astype(np.float64)).query(pts.astype(np.float64), k=4)
        want = d[:, 1:] ** 2
        assert np.all(np.diff(best, axis=1) >= 0)
        np.testing.assert_allclose(best, want, rtol=3e-6, atol=0)
        np.testing.assert_array_equal(mean, ((best[:, 0] + best[:, 1]) + best[:, 2]) / np.float32(3))


def test_small_counts():
    assert knn_oracle.knn_mean_dist(np.zeros((0, 3), np.float32)).shape == (0,)
    for P in (1, 2):
        assert np.isposinf(knn_oracle.knn_mean_dist(np.random.default_rng(P).random((P, 3), dtype=np.float32))).all()
    pts = np.array([[0, 0, 0], [1, 0, 0], [0, 2, 0]], np.float32)
    out = knn_oracle.knn_mean_dist(pts)
    assert out[0] == _mean([1, 4, FMAX]) and out[1] == _mean([1, 5, FMAX]) and out[2] == _mean([4, 5, FMAX])
    assert np.isfinite(out).all() and abs(float(out[0]) - 1.134e38) < 1e35
    pts = np.array([[0, 0, 0], [1, 0, 0], [0, 2, 0], [0, 0, 3], [5, 5, 5]], np.float32)
    for P in (4, 5):
        out = knn_oracle.knn_mean_dist(pts[:P])
        assert out[0] == _mean([1, 4, 9])
    assert knn_oracle.knn_mean_dist(pts)[4] == _mean([54, 59, 66])


def test_coincident_points_count_by_index():
    pts = np.array([[1, 1, 1]] * 3 + [[1, 1, 2]], np.float32)
    out = knn_oracle.knn_mean_dist(pts)
    assert out[0] == _mean([0, 0, 1]) and out[3] == np.float32(1)
    assert (knn_oracle.knn_mean_dist(np.full((7, 3), 2.5, np.float32)) == 0).all()


def test_non_finite_points_are_excluded():
    pts = np.array([[0, 0, 0], [np.nan, 0, 0], [1, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [0, 2, 0], [0, 0, 3]], np.float32)
    out = knn_oracle.knn_mean_dist(pts)
    assert np.isposinf(out[[1, 3, 4]]).all()
    assert out[0] == _mean([1, 4, 9])
    clean = pts[[0, 2, 5, 6]]
    np.testing.assert_array_equal(out[[0, 2, 5, 6]], knn_oracle.knn_mean_dist(clean))


def test_overflowing_distances_are_excluded():
    pts = np.array([[0, 0, 0], [1, 0, 0], [2e19, 0, 0], [-2e19, 0, 0]], np.float32)
    out, best = knn_oracle.knn_mean_dist(pts, return_best=True)
    assert best[0].tolist() == [1.0, float(FMAX), float(FMAX)]   # 4e38 overflows to inf: not accepted
    assert np.isposinf(out[0])   # 1 + FLT_MAX + FLT_MAX overflows in the mean
    assert (best[2:] == FMAX).all() and np.isposinf(out[2:]).all()   # every distance of the far points overflows
    assert np.isposinf(knn_oracle.knn_mean_dist(np.array([[0, 0, 0], [3e19, 0, 0]], np.float32))).all()


def test_subnormal_distances_are_kept():
    pts = np.array([[0, 0, 0], [1e-22, 0, 0], [0, 3e-22, 0], [0, 0, 5e-21]], np.float32)
    _, best = knn_oracle.knn_mean_dist(pts, return_best=True)
    tiny = np.finfo(np.float32).tiny
    assert 0 < best[0, 0] < tiny and best[0, 0] == _fma(0, 0, _fma(pts[1, 0], pts[1, 0], 0))
    assert (best[:3, :2] > 0).all() and (best[:3, :2] < tiny).all()
    pts = gof_synth.make_point_cloud("tiny", 2001, 4)
    _, best = knn_oracle.knn_mean_dist(pts, return_best=True)
    assert (best[:, 0] < tiny).mean() > 0.9 and (best[:, 0] > 0).all()


def test_fused_evaluation_order():
    """fmaf(dz, dz, fmaf(dx, dx, dy*dy)) -- the reference's contraction -- differs here from the unfused sum and from the
    other fused order, and the oracle returns it."""
    q = np.array([-0.38698557019233704, -0.5372548699378967, 0.30153265595436096], np.float32)
    p = np.array([-0.3916918635368347, -0.530009388923645, 0.29694563150405884], np.float32)
    dx, dy, dz = (p - q).astype(np.float32)
    ref = _fma(dz, dz, _fma(dx, dx, _r32(Fraction(float(dy)) ** 2)))
    other = _fma(dz, dz, _fma(dy, dy, _r32(Fraction(float(dx)) ** 2)))
    unfused = np.float32(np.float32(dx * dx + dy * dy) + dz * dz)
    assert len({float(ref), float(other), float(unfused)}) == 3
    far = np.float32(100)
    pts = np.stack([q, p, q + far, q - far])
    _, best = knn_oracle.knn_mean_dist(pts, queries=[0], return_best=True)
    assert best[0, 0] == ref


def test_permutation_and_query_subset():
    pts = gof_synth.make_point_cloud("lattice", 1500, 5)
    perm = np.random.default_rng(2).permutation(1500)
    full = knn_oracle.knn_mean_dist(pts)
    np.testing.assert_array_equal(knn_oracle.knn_mean_dist(pts[perm]), full[perm])
    q = np.array([7, 0, 1499, 300])
    np.testing.assert_array_equal(knn_oracle.knn_mean_dist(pts, queries=q), full[q])


@pytest.mark.parametrize("kind", gof_synth.POINT_CLOUD_KINDS)
def test_point_clouds_are_reproducible(kind):
    a = gof_synth.make_point_cloud(kind, 1000, 3)
    assert a.dtype == np.float32 and a.shape == (1000, 3) and a.flags.c_contiguous
    assert np.array_equal(a.view(np.uint32), gof_synth.make_point_cloud(kind, 1000, 3).view(np.uint32))
    assert gof_synth.make_point_cloud(kind, 0, 3).shape == (0, 3)
