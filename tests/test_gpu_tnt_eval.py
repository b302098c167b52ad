"""GPU tests of the Tanks and Temples evaluation (csrc/tnt_eval.cu and the indexed 1-NN of csrc/dtu_eval.cu through
gof_tnt_eval, DESIGN section 4.7): crop, voxel down-sample and the indexed 1-NN bit for bit against the float64 oracle
(oracle/tnt_eval_oracle.py), the ICP correspondences and moments, `evaluate` end to end against the reference's stored outputs
(tests/golden/tnt_eval_ref.npz), determinism, scratch independence, the refusals and the command line."""
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "gaussian-opacity-fields_b200")]
import _tnt_scenes  # noqa: E402
import tnt_eval_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(ROOT, "tests", "golden", "tnt_eval_ref.npz")
DEV = "cuda:0"


@pytest.fixture(scope="module")
def m():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import gof_tnt_eval
    return gof_tnt_eval


def _t(x):
    return torch.as_tensor(np.asarray(x, np.float64).reshape(-1, 3), device=DEV)


def _golden_scene(z, name):
    g = lambda k: z[f"{name}/{k}"]  # noqa: E731
    axis, amin, amax = g("crop")
    return dict(name=name, vertices=g("vertices"), faces=g("faces"), gt=g("gt"), traj=g("traj"), gt_trans=g("gt_trans"),
                axis=int(axis), axis_min=amin, axis_max=amax, polygon=g("polygon"), tau=O.SCENES_TAU[name])


def _similar(scale=1.3):
    T = _tnt_scenes._similarity(scale, 17.0, [0.3, -0.2, 1.0], [0.5, -1.0, 0.25])
    return T


# ---- crop --------------------------------------------------------------------------------------------------------------

def _crop_check(m, pts, vol, T=None):
    got, idx = m.crop(_t(pts), vol, T, return_index=True)
    want, widx = O.crop(pts, vol, T)
    assert np.array_equal(idx.cpu().numpy(), widx)
    assert np.array_equal(got.cpu().numpy(), want)
    return widx


@pytest.mark.parametrize("with_T", [False, True])
def test_crop_scene_ties(m, with_T):
    """GT points exactly on the polygon's vertices, on its (axis-aligned, some horizontal) edges and on axis_min / axis_max."""
    sc = _tnt_scenes.scenes()["Barn"]
    vol = _tnt_scenes.volume(sc)
    T = _similar() if with_T else None
    kept = _crop_check(m, sc["gt"], vol, T)
    assert 0 < kept.size < sc["gt"].shape[0]


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 2 ** 16 - 1, 2 ** 16 + 1])
def test_crop_sizes(m, n):
    rng = np.random.default_rng(n)
    pts = rng.uniform(-1, 1, (n, 3))
    ang = np.linspace(0, 2 * np.pi, 9, endpoint=False)
    r = np.where(np.arange(9) % 2, 0.4, 0.9)                 # a concave star
    poly = np.stack([r * np.cos(ang), np.zeros(9), r * np.sin(ang)], 1)
    vol = O.crop_volume(1, -0.5, 0.5, poly)
    _crop_check(m, pts, vol)
    _crop_check(m, pts, vol, _similar(0.9))


@pytest.mark.parametrize("nv", [3, 500])
def test_crop_polygon_sizes(m, nv):
    rng = np.random.default_rng(nv)
    ang = np.sort(rng.uniform(0, 2 * np.pi, nv))
    r = rng.uniform(0.3, 1.0, nv)
    poly = np.stack([r * np.cos(ang), r * np.sin(ang), np.zeros(nv)], 1)
    pts = rng.uniform(-1, 1, (50000, 3))
    pts[:nv, :2] = poly[:, :2]                                   # on every vertex
    for axis in (0, 1, 2):
        vol = O.crop_volume(axis, -0.7, 0.7, np.roll(poly, axis, 1))
        _crop_check(m, pts, vol)


# ---- voxel down-sample -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n,voxel", [(1, 0.1), (33, 0.5), (20000, 0.05), (2 ** 16 + 1, 0.013)])
def test_voxel_random(m, n, voxel):
    rng = np.random.default_rng(n)
    pts = rng.normal(size=(n, 3)) * 2 - 3                        # negative coordinates
    got = m.voxel_down_sample(_t(pts), voxel).cpu().numpy()
    assert np.array_equal(got, O.voxel_down_sample(pts, voxel))


def test_voxel_one_big_voxel(m):
    """10^6 points in one voxel: summed sequentially in input order."""
    rng = np.random.default_rng(3)
    pts = np.concatenate([rng.uniform(0.2, 0.3, (10 ** 6, 3)), rng.uniform(-5, 5, (1000, 3))])
    got = m.voxel_down_sample(_t(pts), 1.0).cpu().numpy()
    assert np.array_equal(got, O.voxel_down_sample(pts, 1.0))


def test_voxel_too_small(m):
    pts = np.array([[0.0, 0.0, 0.0], [1e3, 0.0, 0.0]])
    with pytest.raises(ValueError, match="too small"):
        O.voxel_down_sample(pts, 1e-7)
    with pytest.raises(RuntimeError, match="too small"):
        m.voxel_down_sample(_t(pts), 1e-7)


def test_uniform_down_sample(m):
    pts = np.random.default_rng(0).normal(size=(1001, 3))
    for mp in (100, 250, 1001, 2000):
        assert np.array_equal(m.uniform_down_sample(_t(pts), mp).cpu().numpy(), O.uniform_down_sample(pts, mp))


# ---- indexed 1-NN ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("nr,nq", [(1, 1), (31, 33), (33, 31), (2 ** 16 - 1, 2 ** 16 + 1)])
def test_nn_index_sizes(m, nr, nq):
    rng = np.random.default_rng(nr + nq)
    ref = rng.normal(size=(nr, 3))
    q = rng.normal(size=(nq, 3)) * 1.3
    tree = m.NNTree(_t(ref))
    for r2 in (math.inf, 0.01):
        idx, d2 = tree.query(_t(q), r2)
        wi, wd = O.nn(ref, q, r2)
        assert np.array_equal(idx.cpu().numpy(), wi)
        assert np.array_equal(d2.cpu().numpy(), wd)


def test_nn_index_ties_and_radius(m):
    """A lattice with duplicates: every query has exact ties (the lowest index wins); queries at exactly r are refused."""
    g = np.stack(np.meshgrid(*[np.arange(6) * 0.25] * 3, indexing="ij"), -1).reshape(-1, 3)
    ref = np.concatenate([g, g[::-1], g])                       # each position three times
    rng = np.random.default_rng(1)
    q = np.concatenate([g + 0.125, g, g + np.array([0.25, 0, 0]), rng.uniform(0, 1.25, (3000, 3))])
    tree = m.NNTree(_t(ref))
    for r2 in (math.inf, 0.0625, 0.046875):                     # 0.0625 = (0.25)^2: a query 0.25 from its nearest is refused
        idx, d2 = tree.query(_t(q), r2)
        wi, wd = O.nn(ref, q, r2)
        assert np.array_equal(idx.cpu().numpy(), wi)
        assert np.array_equal(d2.cpu().numpy(), wd)
    # reusing the order of a first query changes nothing
    idx2, d22 = tree.query(_t(q * 1.0001), 0.0625, reuse_order=True)
    wi, wd = O.nn(ref, q * 1.0001, 0.0625)
    assert np.array_equal(idx2.cpu().numpy(), wi) and np.array_equal(d22.cpu().numpy(), wd)


@pytest.mark.parametrize("fill", [0x00, 0xFF])
def test_nn_reuse_order_on_an_unsorted_scratch(m, fill):
    """reuse_order on a query scratch that holds no order for this query count (fresh, or sorted for another count) searches
    in input order: the same results, no read through stale indices."""
    lib = m._lib
    rng = np.random.default_rng(12)
    ref, q = rng.normal(size=(4000, 3)), rng.normal(size=(5000, 3))
    R, Q = _t(ref), _t(q)
    nt = int(lib.gof_nn_tree_scratch_bytes(4000))
    tb = torch.empty(nt, dtype=torch.uint8, device=DEV)
    m._C._check(lib.gof_nn_tree_build(4000, R.data_ptr(), tb.data_ptr(), nt, m._C._stream()))
    nq = int(lib.gof_nn_query_scratch_bytes(5000))
    qb = torch.full((nq,), fill, dtype=torch.uint8, device=DEV)
    idx = torch.empty(5000, dtype=torch.int32, device=DEV)
    d2 = torch.empty(5000, dtype=torch.float64, device=DEV)
    wi, wd = O.nn(ref, q, 0.05)

    def query(n, reuse):
        m._C._check(lib.gof_nn_query(4000, tb.data_ptr(), nt, n, Q.data_ptr(), 0.05, reuse, idx.data_ptr(), d2.data_ptr(),
                                     qb.data_ptr(), nq, m._C._stream()))
        return idx[:n].cpu().numpy(), d2[:n].cpu().numpy()

    got = query(5000, 1)                                        # fresh scratch
    assert np.array_equal(got[0], wi) and np.array_equal(got[1], wd)
    query(3000, 0)                                              # sorted for 3000 queries ...
    got = query(5000, 1)                                        # ... then reused for 5000
    assert np.array_equal(got[0], wi) and np.array_equal(got[1], wd)
    query(5000, 0)
    got = query(5000, 1)                                        # the stamped order
    assert np.array_equal(got[0], wi) and np.array_equal(got[1], wd)


# ---- ICP -----------------------------------------------------------------------------------------------------------------

def _scene_clouds(sc, voxel):
    pcd = O.reconstruction_cloud(sc["vertices"], sc["faces"])
    src_c = sc["traj"][:, :3, 3]
    T0 = O.ransac_alignment(src_c, O.transform(src_c, sc["gt_trans"]), 0, iterations=2000)
    vol = _tnt_scenes.volume(sc)
    s = O.voxel_down_sample(O.crop(pcd, vol, T0)[0], voxel)
    t = O.voxel_down_sample(O.crop(sc["gt"], vol)[0], voxel)
    return s, t


def test_icp_iterations_match_oracle(m):
    """Both fed the same moving points: identical correspondences and d2; moments within a summation bound."""
    sc = _tnt_scenes.scenes()["Barn"]
    s, t = _scene_clouds(sc, sc["tau"])
    trace = []
    O.registration_icp(s, t, 80 * sc["tau"], max_iteration=6, relative_fitness=0.0, relative_rmse=0.0, trace=trace)
    tree = m.NNTree(_t(t))
    r2 = O.icp_r2(80 * sc["tau"])
    tt = _t(t)
    for k, (pts, wi, wd) in enumerate(trace):
        idx, d2 = tree.query(_t(pts), r2, reuse_order=k > 0)
        assert np.array_equal(idx.cpu().numpy(), wi)
        assert np.array_equal(d2.cpu().numpy(), wd)
        n, sd2, ms, mt, cov, var = m.icp_moments(_t(pts), tt, idx, d2)
        wn, wsd2, wms, wmt, wcov, wvar = O.moments(pts, t, wi, wd)
        assert n == wn
        eps = np.finfo(np.float64).eps
        bound = 4 * n * eps                                  # relative to the sum of magnitudes, log2(n) + 1 levels of rounding
        sel = wi >= 0
        assert abs(sd2 - wsd2) <= bound * np.abs(wd[sel]).sum()
        np.testing.assert_allclose(ms, wms, rtol=0, atol=bound * np.abs(pts[sel]).max() * 2)
        np.testing.assert_allclose(mt, wmt, rtol=0, atol=bound * np.abs(t[wi[sel]]).max() * 2)
        ds, dt = pts[sel] - wms, t[wi[sel]] - wmt
        np.testing.assert_allclose(cov, wcov, rtol=0, atol=bound * (np.abs(dt).T @ np.abs(ds)).max() * 4 + 1e-300)
        assert abs(var - wvar) <= bound * (ds * ds).sum() * 4


@pytest.mark.parametrize("name", ["Barn", "Truck"])
def test_icp_full_registrations(m, name):
    sc = _tnt_scenes.scenes()[name]
    for voxel, thr in ((sc["tau"], 80 * sc["tau"]), (sc["tau"] / 2, 20 * sc["tau"])):
        s, t = _scene_clouds(sc, voxel)
        want = O.registration_icp(s, t, thr, **O.ICP_CRITERIA)
        got = m.registration_icp(_t(s), _t(t), thr, **m.ICP_CRITERIA)
        assert got["iterations"] == want["iterations"]
        scale = abs(np.linalg.det(want["transformation"][:3, :3])) ** (1 / 3)
        assert np.abs(got["transformation"] - want["transformation"]).max() <= 1e-12 * max(scale, 1.0)


def test_icp_empty_sides(m):
    s = np.random.default_rng(0).normal(size=(100, 3))
    r = m.registration_icp(_t(s), _t(np.zeros((0, 3))), 0.1, **m.ICP_CRITERIA)
    assert np.array_equal(r["transformation"], np.eye(4)) and r["fitness"] == 0.0


# ---- scoring -------------------------------------------------------------------------------------------------------------

def test_distances_and_histograms(m):
    sc = _tnt_scenes.scenes()["Barn"]
    s, t = _scene_clouds(sc, sc["tau"] / 2)
    d1 = m.distances(_t(s), _t(t)).cpu().numpy()
    d2 = m.distances(_t(t), _t(s)).cpu().numpy()
    assert np.array_equal(d1, O.distances(s, t)) and np.array_equal(d2, O.distances(t, s))
    got, want = m.evaluate_histo(d1, d2, sc["tau"]), O.f1_histo(sc["tau"], 5, d1, d2)
    for a, b in zip(got, want):
        assert np.array_equal(np.asarray(a), np.asarray(b))
    assert np.array_equal(m.distances(_t(s), _t(np.zeros((0, 3)))).cpu().numpy(), np.zeros(s.shape[0]))


# ---- end to end ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("scale", [1.0, 1e3, 1e-3])
def test_reconstruction_cloud_bit_exact(m, scale):
    """The face centroids ((v0 + v1) + v2) / 3, correctly rounded, equal the oracle's and numpy's mean bit for bit."""
    rng = np.random.default_rng(int(scale * 1000) % 97)
    V = rng.normal(size=(20000, 3)) * scale
    F = rng.integers(0, 20000, (60000, 3))
    got = m.reconstruction_cloud(_t(V), torch.as_tensor(F, device=DEV)).cpu().numpy()
    assert np.array_equal(got, O.reconstruction_cloud(V, F))
    assert np.array_equal(got[20000:], V[F].mean(axis=1))


def _evaluate(m, sc, **kw):
    return m.evaluate(sc["vertices"], sc["faces"], sc["gt"], sc["traj"], sc["traj"], sc["gt_trans"], _tnt_scenes.volume(sc), sc["tau"],
                      **kw)


@pytest.mark.parametrize("name", ["Barn", "Truck"])
def test_evaluate_equals_reference(m, name):
    z = np.load(GOLDEN)
    sc = _golden_scene(z, name)
    o = _evaluate(m, sc)
    g = lambda k: z[f"{name}/{k}"]  # noqa: E731
    T = g("transforms")
    for k, key in enumerate(("T_ransac", "T_r2", "T_r3", "T_r")):
        assert np.abs(o[key] - T[k]).max() <= 1e-9, key
    assert [o["iterations_r2"], o["iterations_r3"], o["iterations_r"]] == list(g("icp_iterations"))
    tau = sc["tau"]
    # precision and recall exactly; a mismatch is allowed only for distances within 1e-9 tau of tau
    near = int((np.abs(o["d1"] - tau) <= 1e-9 * tau).sum() + (np.abs(o["d2"] - tau) <= 1e-9 * tau).sum())
    prf = np.array([o["precision"], o["recall"], o["fscore"], tau, 5], np.float64)
    if near == 0:
        assert np.array_equal(prf, g("prf")), (prf, g("prf"))
        assert np.array_equal(o["cum_source"], np.atleast_1d(g("cum_source")))
        assert np.array_equal(o["cum_target"], np.atleast_1d(g("cum_target")))
    else:
        print(f"{name}: {near} distances within 1e-9 tau of tau")
        np.testing.assert_allclose(prf, g("prf"), rtol=0, atol=near / max(len(o["d1"]), len(o["d2"]), 1) * 2)
    assert o["source_down"].shape == g("source_down").shape and o["target_down"].shape == g("target_down").shape
    np.testing.assert_allclose(o["source_down"], g("source_down"), rtol=0, atol=1e-9)
    np.testing.assert_allclose(o["d1"], g("d1"), rtol=0, atol=1e-9)


def test_two_runs_identical(m):
    sc = _tnt_scenes.scenes()["Barn"]
    a, b = _evaluate(m, sc, seed=4), _evaluate(m, sc, seed=4)
    for k in ("T_ransac", "T_r2", "T_r3", "T_r", "source_down", "target_down", "d1", "d2", "cum_source", "cum_target"):
        assert np.array_equal(a[k], b[k]), k


def test_evaluate_uniform_branch(m):
    """max_points below the cropped sizes: the last registration takes the uniform down-sample."""
    sc = _tnt_scenes.scenes()["Barn"]
    o = _evaluate(m, sc, max_points=1000)
    want = O.evaluate(sc["vertices"], sc["faces"], sc["gt"], sc["traj"], sc["traj"], sc["gt_trans"], _tnt_scenes.volume(sc),
                      sc["tau"], max_points=1000)
    assert o["iterations_r"] == want["iterations_r"]
    assert np.abs(o["T_r"] - want["T_r"]).max() <= 1e-9


# ---- scratch -------------------------------------------------------------------------------------------------------------

GUARD = 64 * 1024


@pytest.mark.parametrize("fill", [0x00, 0xFF])
def test_scratch_contents_and_guard(m, fill):
    lib = m._lib
    rng = np.random.default_rng(9)
    pts = rng.normal(size=(7000, 3))

    def guarded(nb):
        return torch.full((nb + 2 * GUARD,), fill, dtype=torch.uint8, device=DEV)

    def intact(buf, nb):
        return bool((buf[:GUARD] == fill).all()) and bool((buf[GUARD + nb:] == fill).all())

    P = _t(pts)
    vol = O.crop_volume(2, -0.5, 0.5, [[-1, -1, 0], [1, -1, 0], [0, 0, 0], [1, 1, 0], [-1, 1, 0]])
    nb = int(lib.gof_crop_scratch_bytes(7000))
    buf = guarded(nb)
    out = torch.empty((7000, 3), dtype=torch.float64, device=DEV)
    k = ctypes.c_int64(0)
    poly = np.ascontiguousarray(vol["polygon_uv"])
    m._C._check(lib.gof_crop_polygon(7000, P.data_ptr(), None, 2, -0.5, 0.5, poly.shape[0], poly.ctypes.data_as(m._dp), out.data_ptr(),
                                     None, ctypes.byref(k), buf.data_ptr() + GUARD, nb, m._C._stream()))
    assert np.array_equal(out[:k.value].cpu().numpy(), O.crop(pts, vol)[0]) and intact(buf, nb)

    nb = int(lib.gof_voxel_down_sample_scratch_bytes(7000))
    buf = guarded(nb)
    m._C._check(lib.gof_voxel_down_sample(7000, P.data_ptr(), 0.3, out.data_ptr(), ctypes.byref(k), buf.data_ptr() + GUARD, nb,
                                          m._C._stream()))
    assert np.array_equal(out[:k.value].cpu().numpy(), O.voxel_down_sample(pts, 0.3)) and intact(buf, nb)

    ref = _t(pts[:3000])
    nt, nq = int(lib.gof_nn_tree_scratch_bytes(3000)), int(lib.gof_nn_query_scratch_bytes(7000))
    tb, qb = guarded(nt), guarded(nq)
    idx = torch.empty(7000, dtype=torch.int32, device=DEV)
    d2 = torch.empty(7000, dtype=torch.float64, device=DEV)
    m._C._check(lib.gof_nn_tree_build(3000, ref.data_ptr(), tb.data_ptr() + GUARD, nt, m._C._stream()))
    m._C._check(lib.gof_nn_query(3000, tb.data_ptr() + GUARD, nt, 7000, P.data_ptr(), 0.05, 0, idx.data_ptr(), d2.data_ptr(),
                                 qb.data_ptr() + GUARD, nq, m._C._stream()))
    wi, wd = O.nn(pts[:3000], pts, 0.05)
    assert np.array_equal(idx.cpu().numpy(), wi) and np.array_equal(d2.cpu().numpy(), wd)
    assert intact(tb, nt) and intact(qb, nq)

    nb = int(lib.gof_icp_moments_scratch_bytes(7000))
    buf = guarded(nb)
    mom = (ctypes.c_double * 18)()
    m._C._check(lib.gof_icp_moments(7000, P.data_ptr(), ref.data_ptr(), idx.data_ptr(), d2.data_ptr(), mom, buf.data_ptr() + GUARD, nb,
                                    m._C._stream()))
    assert mom[0] == float((wi >= 0).sum()) and intact(buf, nb)


# ---- refusals ------------------------------------------------------------------------------------------------------------

def test_refusals(m, tmp_path):
    bad = tmp_path / "bad.json"
    bad.write_text("{not json")
    with pytest.raises(ValueError, match="crop volume"):
        m.read_crop_volume(str(bad))
    with pytest.raises(ValueError, match="at least 3"):
        m.crop_volume("z", 0, 1, [[0, 0, 0], [1, 0, 0]])
    with pytest.raises(ValueError, match="at most"):
        m.crop_volume("z", 0, 1, np.zeros((m.MAX_POLYGON + 1, 3)))
    with pytest.raises(ValueError, match="not one of"):
        m.run_evaluation(str(tmp_path / "NotAScene"), "x.log", "x.ply", str(tmp_path))
    with pytest.raises(ValueError, match=r"\.json trajectories"):
        m.read_trajectory(str(tmp_path / "traj.json"))
    pts = np.zeros((4, 3))
    pts[2, 1] = np.nan
    vol = O.crop_volume(2, -1, 1, [[0, 0, 0], [1, 0, 0], [0, 1, 0]])
    with pytest.raises(ValueError, match="non-finite"):
        m.crop(_t(pts), vol)
    with pytest.raises(ValueError, match="non-finite"):
        m.voxel_down_sample(_t(pts), 0.1)
    with pytest.raises(ValueError, match="non-finite"):
        m.NNTree(_t(pts))
    lib = m._lib
    k = ctypes.c_int64(0)
    big = 2 ** 30
    poly = np.zeros((3, 2))
    assert lib.gof_crop_polygon(big, 1, None, 2, 0.0, 1.0, 3, poly.ctypes.data_as(m._dp), 1, None, ctypes.byref(k), 1, 1 << 40, None) != 0
    assert b"2^30" in lib.gof_last_error()
    assert lib.gof_voxel_down_sample(big, 1, 0.1, 1, ctypes.byref(k), 1, 1 << 40, None) != 0
    assert b"2^30" in lib.gof_last_error()
    assert lib.gof_nn_query(big, 1, 1 << 40, 1, 1, 1.0, 0, 1, 1, 1, 1 << 40, None) != 0
    # a tree scratch smaller than n_ref needs
    rc = lib.gof_nn_query(1000, 1, int(lib.gof_nn_tree_scratch_bytes(1000)) - 1, 10, 1, 1.0, 0, 1, 1, 1, 1 << 40, None)
    assert rc != 0 and b"tree scratch" in lib.gof_last_error()
    # non-finite points at the C ABI (the Python layer refuses them earlier)
    bad = _t([[0.0, 0.0, 0.0], [1.0, np.inf, 0.0], [2.0, 2.0, 2.0]])
    out = torch.empty((3, 3), dtype=torch.float64, device=DEV)
    nb = int(lib.gof_voxel_down_sample_scratch_bytes(3))
    buf = torch.empty(nb, dtype=torch.uint8, device=DEV)
    assert lib.gof_voxel_down_sample(3, bad.data_ptr(), 0.5, out.data_ptr(), ctypes.byref(k), buf.data_ptr(), nb, m._C._stream()) != 0
    assert b"non-finite" in lib.gof_last_error()
    assert lib.gof_crop_polygon(4, 1, None, 2, 0.0, 1.0, 2, poly.ctypes.data_as(m._dp), 1, None, ctypes.byref(k), 1, 1 << 40, None) != 0
    assert b"polygon vertices" in lib.gof_last_error()


# ---- command line --------------------------------------------------------------------------------------------------------

def test_cli_writes_reference_files(m, tmp_path):
    z = np.load(GOLDEN)
    sc = _golden_scene(z, "Barn")
    d, mesh = _tnt_scenes.write_dataset(str(tmp_path), sc)
    m.main(["--dataset-dir", d, "--traj-path", os.path.join(d, "Barn_COLMAP_SfM.log"), "--ply-path", mesh, "--view-crop", "1"])
    out = os.path.join(os.path.dirname(mesh), "evaluation")
    np.testing.assert_array_equal(np.loadtxt(os.path.join(out, "Barn.precision.txt")), z["Barn/cum_source"])
    np.testing.assert_array_equal(np.loadtxt(os.path.join(out, "Barn.recall.txt")), z["Barn/cum_target"])
    np.testing.assert_array_equal(np.loadtxt(os.path.join(out, "Barn.prf_tau_plotstr.txt")), z["Barn/prf"])
    for name, key in (("precision", "source_down"), ("recall", "target_down")):
        p = m.read_ply(os.path.join(out, f"Barn.{name}.ply"))["points"]
        np.testing.assert_allclose(p, z[f"Barn/{key}"], rtol=0, atol=1e-9)
