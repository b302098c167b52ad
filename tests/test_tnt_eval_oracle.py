"""CPU tests of the Tanks and Temples evaluation's oracle (oracle/tnt_eval_oracle.py, DESIGN section 4.7): against brute force
(crop, voxel averages, 1-NN ties, Umeyama), against the reference's own helpers where baseline/stage_ref.sh staged them
(trajectory_io.read_trajectory, config.scenes_tau_dict), the RANSAC host code of gof_tnt_eval against the oracle, and the
stubbed reference run.py against tests/golden/tnt_eval_ref.npz."""
import ast
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]
import _tnt_scenes  # noqa: E402
import tnt_eval_oracle as O  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "tnt_eval_ref.npz")


def _staged(name):
    p = os.path.join(_tnt_scenes.REF_DIR, name)
    if not os.path.exists(p):
        pytest.skip(f"the reference's eval_tnt/{name} is not staged (baseline/stage_ref.sh)")
    return p


def test_crop_against_brute_force():
    """Per point, per edge, the specification's rule written out in Python floats."""
    rng = np.random.default_rng(0)
    poly = np.array([[0, 0, 0], [2, 0, 0], [2, 1, 0], [1, 1, 0], [1, 2, 0], [0, 2, 0]], np.float64)
    pts = np.concatenate([rng.uniform(-0.5, 2.5, (3000, 3)) * [1, 1, 0.4], poly, (poly + np.roll(poly, -1, 0)) / 2,
                          [[0.5, 0.5, -0.5], [0.5, 0.5, 0.5], [0.5, 0.5, 0.50000001]]])
    vol = O.crop_volume(2, -0.5, 0.5, poly)
    _, idx = O.crop(pts, vol)
    want = []
    for i, p in enumerate(pts):
        if p[2] < -0.5 or p[2] > 0.5:
            continue
        nodes = 0
        for a in range(6):
            A, B = poly[a], poly[(a + 1) % 6]
            if (A[1] < p[1] and B[1] >= p[1]) or (B[1] < p[1] and A[1] >= p[1]):
                nodes += (A[0] + ((p[1] - A[1]) / (B[1] - A[1])) * (B[0] - A[0])) < p[0]
        if nodes % 2:
            want.append(i)
    assert np.array_equal(idx, want)


def test_voxel_against_brute_force():
    rng = np.random.default_rng(1)
    pts = rng.normal(size=(2000, 3)) - 4
    v = 0.7
    got = O.voxel_down_sample(pts, v)
    lo = pts.min(0) - v * 0.5
    groups = {}
    for p in pts:
        k = tuple(int(np.floor(c)) for c in (p - lo) / v)
        if k in groups:
            groups[k][0] = groups[k][0] + p
            groups[k][1] += 1
        else:
            groups[k] = [p.copy(), 1]
    want = np.array([groups[k][0] / float(groups[k][1]) for k in sorted(groups)])
    assert np.array_equal(got, want)


def test_nn_ties_against_brute_force():
    g = np.stack(np.meshgrid(*[np.arange(4) * 0.5] * 3, indexing="ij"), -1).reshape(-1, 3)
    ref = np.concatenate([g, g[::-1], g])
    q = np.concatenate([g + 0.25, g, np.random.default_rng(2).uniform(0, 1.5, (300, 3))])
    for r2 in (np.inf, 0.25, 0.1875):
        idx, d2 = O.nn(ref, q, r2)
        for i, p in enumerate(q):
            d = O._sq(ref - p)
            b = d.min()
            if b < r2:
                assert d2[i] == b and idx[i] == np.nonzero(d == b)[0].min()
            else:
                assert idx[i] == -1 and d2[i] == np.inf


def test_umeyama_recovers_similarity():
    rng = np.random.default_rng(3)
    src = rng.normal(size=(500, 3))
    T = _tnt_scenes._similarity(2.5, 40.0, [1, 2, 3], [0.3, -1.0, 2.0])
    tgt = O.transform(src, T)
    got = O.umeyama(*((500,) + O.moments(src, tgt, np.arange(500), np.zeros(500))[2:]))
    assert np.abs(got - T).max() < 1e-12
    assert np.array_equal(O.umeyama(0, np.zeros(3), np.zeros(3), np.zeros((3, 3)), 0.0), np.eye(4))


def test_centroids_equal_numpy_mean():
    rng = np.random.default_rng(4)
    V = rng.normal(size=(500, 3)) * 1e3
    F = rng.integers(0, 500, (2000, 3))
    assert np.array_equal(O.reconstruction_cloud(V, F)[500:], V[F].mean(axis=1))


def test_log_reader_against_reference(tmp_path):
    src = open(_staged("trajectory_io.py")).read()
    mod = ast.parse(src)
    ns = {"np": np}
    for node in mod.body:
        if isinstance(node, (ast.ClassDef, ast.FunctionDef)) and node.name in ("CameraPose", "read_trajectory"):
            exec(compile(ast.Module([node], []), "trajectory_io.py", "exec"), ns)
    P = np.random.default_rng(5).normal(size=(7, 4, 4))
    path = str(tmp_path / "t.log")
    _tnt_scenes.write_log(path, P)
    want = np.array([c.pose for c in ns["read_trajectory"](path)])
    assert np.array_equal(O.read_log(path), want) and np.array_equal(want, P)


def test_tau_table_against_reference():
    ns = {}
    exec(open(_staged("config.py")).read(), ns)
    assert ns["scenes_tau_dict"] == O.SCENES_TAU


def test_ransac_host_code_against_oracle():
    sys.path.insert(0, os.path.join(ROOT, "gaussian-opacity-fields_b200"))
    pytest.importorskip("torch")
    try:
        import gof_tnt_eval as G
    except OSError:
        pytest.skip("the library is not built")
    rng = np.random.default_rng(6)
    src = rng.normal(size=(60, 3))
    T = _tnt_scenes._similarity(0.8, 30.0, [0, 1, 1], [1.0, 0.0, 0.5])
    tgt = O.transform(src, T) + rng.normal(0, 0.05, (60, 3))
    tgt[:10] += 1.0                                            # outliers
    src[5] = src[6]                                            # a duplicate: some draws are degenerate
    for seed in (0, 1):
        got, want = G.align_trajectory(src, tgt, seed, iterations=3000), O.ransac_alignment(src, tgt, seed, iterations=3000)
        assert np.abs(got - want).max() < 1e-12             # batched and single 3x3 SVDs round differently


@pytest.mark.parametrize("name", ["Barn", "Truck"])
def test_stubbed_reference_equals_golden(name):
    _staged("run.py")
    z = np.load(GOLDEN)
    ref = _tnt_scenes.run_reference(_tnt_scenes.scenes()[name], 0)
    for k in ("transforms", "icp_iterations", "prf", "cum_source", "cum_target", "d1", "d2", "source_down", "target_down"):
        assert np.array_equal(np.asarray(ref[k]), z[f"{name}/{k}"]), k
    for k in ("vertices", "faces", "gt", "traj", "gt_trans", "polygon"):
        assert np.array_equal(np.asarray(_tnt_scenes.scenes()[name][k]), z[f"{name}/{k}"]), k


def test_oracle_evaluate_equals_golden():
    z = np.load(GOLDEN)
    sc = _tnt_scenes.scenes()["Barn"]
    o = O.evaluate(sc["vertices"], sc["faces"], sc["gt"], sc["traj"], sc["traj"], sc["gt_trans"], _tnt_scenes.volume(sc), sc["tau"])
    assert np.array_equal(np.stack([o["T_ransac"], o["T_r2"], o["T_r3"], o["T_r"]]), z["Barn/transforms"])
    assert np.array_equal(np.array([o["precision"], o["recall"], o["fscore"], sc["tau"], 5]), z["Barn/prf"])
    assert np.array_equal(o["cum_source"], z["Barn/cum_source"]) and np.array_equal(o["d2"], z["Barn/d2"])


def test_hot_r_lut_against_matplotlib():
    plt_cm = pytest.importorskip("matplotlib.cm")
    sys.path.insert(0, os.path.join(ROOT, "gaussian-opacity-fields_b200"))
    pytest.importorskip("torch")
    try:
        import gof_tnt_eval as G
    except OSError:
        pytest.skip("the library is not built")
    import matplotlib
    cmap = matplotlib.colormaps["hot_r"] if hasattr(matplotlib, "colormaps") else plt_cm.get_cmap("hot_r")
    x = np.concatenate([np.linspace(0, 1, 1001), [0.0, 1.0, 0.5, 255.5 / 256]])
    d = x * 0.03
    assert np.array_equal(G.distance_colors(d, 0.03), cmap(np.minimum(d, 0.03) / 0.03)[:, :3])
