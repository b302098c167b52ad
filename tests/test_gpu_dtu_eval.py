"""GPU tests of the DTU mesh evaluation (csrc/dtu_eval.cu through gof_dtu_eval, DESIGN section 4.6): every stage bit for bit
against the float64 oracle (oracle/dtu_eval_oracle.py), `evaluate` end to end against the reference's stored outputs
(tests/golden/dtu_eval_ref.npz), determinism, scratch independence and the refusals."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "gaussian-opacity-fields_b200")]
import _dtu_scenes  # noqa: E402
import dtu_eval_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(ROOT, "tests", "golden", "dtu_eval_ref.npz")
DEV = "cuda:0"


@pytest.fixture(scope="module")
def m():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import gof_dtu_eval
    return gof_dtu_eval


def _t(x):
    return torch.as_tensor(np.asarray(x, np.float64), device=DEV)


# ---- sampling ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["sphere", "soup"])
def test_sample_scene(m, name):
    sc = _dtu_scenes.scenes()[name]
    r = sc["args"]["downsample_density"]
    got = m.sample_mesh(_t(sc["data"]), torch.as_tensor(sc["faces"], device=DEV), r).cpu().numpy()
    assert np.array_equal(got, O.sample_mesh(sc["data"], sc["faces"], r))


@pytest.mark.parametrize("nf,r", [(0, 0.2), (1, 0.05), (33, 0.1), (2000, 0.3)])
def test_sample_random_soup(m, nf, r):
    rng = np.random.default_rng(nf)
    V = rng.uniform(-5, 5, (max(3 * nf, 4), 3))
    F = rng.integers(0, V.shape[0], (nf, 3))
    got = m.sample_mesh(_t(V), torch.as_tensor(F, device=DEV), r).cpu().numpy()
    assert np.array_equal(got, O.sample_mesh(V, F, r))


def test_sample_one_large_face(m):
    """~5 * 10^6 samples in one triangle: emitted one thread per sample."""
    V = np.array([[0, 0, 0], [640.0, 0, 0], [0, 640.0, 1.0]])
    F = np.array([[0, 1, 2]])
    got = m.sample_mesh(_t(V), torch.as_tensor(F, device=DEV), 0.2).cpu().numpy()
    assert got.shape[0] > 4_000_000
    want = O.sample_mesh(V, F, 0.2)
    assert np.array_equal(got, want)


# ---- downsample --------------------------------------------------------------------------------------------------------

def _down(m, pts, perm, r):
    kept, rounds = m.ordered_downsample(_t(pts), torch.as_tensor(np.asarray(perm, np.int64), device=DEV), r)
    return kept.cpu().numpy(), rounds


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_downsample_seeds(m, seed):
    sc = _dtu_scenes.scenes()["pcd"]
    perm = np.random.default_rng(seed).permutation(sc["data"].shape[0])
    kept, rounds = _down(m, sc["data"], perm, 0.5)
    assert np.array_equal(kept, O.ordered_downsample(sc["data"], perm, 0.5))
    assert 1 <= rounds < 64


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 2 ** 16 - 1, 2 ** 16 + 1])
def test_downsample_sizes(m, n):
    rng = np.random.default_rng(n)
    pts = rng.uniform(0, 10, (n, 3)) * np.array([1, 1, 0.1])
    perm = rng.permutation(n)
    kept, _ = _down(m, pts, perm, 0.2)
    assert np.array_equal(kept, O.ordered_downsample(pts, perm, 0.2))


def test_downsample_adversarial_line(m):
    """Points 0.6 r apart along a line, in order: every point's only earlier neighbour is its predecessor, so the rounds
    settle one point each."""
    n = 3000
    pts = np.stack([np.arange(n) * 0.3, np.zeros(n), np.zeros(n)], 1)
    kept, rounds = _down(m, pts, np.arange(n), 0.5)
    assert np.array_equal(kept, O.ordered_downsample(pts, np.arange(n), 0.5))
    assert rounds >= n - 1


def test_downsample_coincident(m):
    pts = np.tile([[1.5, -2.0, 3.25]], (10 ** 4, 1))
    perm = np.random.default_rng(0).permutation(10 ** 4)
    kept, _ = _down(m, pts, perm, 0.2)
    assert kept.sum() == 1 and kept[0]


def test_downsample_lattice_at_exactly_r(m):
    g = np.stack(np.meshgrid(*[np.arange(12) * 0.25] * 3, indexing="ij"), -1).reshape(-1, 3) - 1.0
    perm = np.random.default_rng(4).permutation(g.shape[0])
    kept, _ = _down(m, g, perm, 0.25)
    assert np.array_equal(kept, O.ordered_downsample(g, perm, 0.25))


# ---- distances ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("nr,nq", [(1, 1), (1, 33), (31, 32), (33, 31), (2 ** 16 - 1, 2 ** 16 + 1), (2 ** 16 + 1, 1000)])
def test_nn_dist_sizes(m, nr, nq):
    rng = np.random.default_rng(nr + nq)
    ref = rng.normal(size=(nr, 3)) * 50
    q = rng.normal(size=(nq, 3)) * 60          # some queries outside the reference box
    got = m.nn_dist(_t(ref), _t(q), sqrt=False).cpu().numpy()
    assert np.array_equal(got, O.nn_sqdist(ref, q))
    got = m.nn_dist(_t(ref), _t(q)).cpu().numpy()
    assert np.array_equal(got, np.sqrt(O.nn_sqdist(ref, q)))


def test_nn_dist_large_spot_check(m):
    from scipy.spatial import cKDTree
    rng = np.random.default_rng(7)
    ref = _dtu_scenes._on_sphere(100.0, 2 ** 21, rng) + rng.normal(0, 0.05, (2 ** 21, 3))
    nq = 2 ** 24
    q = _dtu_scenes._on_sphere(100.0, nq, rng) + rng.normal(0, 0.3, (nq, 3))
    got = m.nn_dist(_t(ref), _t(q), sqrt=False).cpu().numpy()
    idx = rng.choice(nq, 20000, replace=False)
    _, nb = cKDTree(ref).query(q[idx], k=8)
    d = ref[nb] - q[idx][:, None, :]
    want = ((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]).min(1)
    assert np.array_equal(got[idx], want)


# ---- end to end --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["sphere", "soup", "pcd"])
def test_evaluate_equals_reference(m, name):
    z = np.load(GOLDEN)
    sc = _dtu_scenes.scenes()[name]
    faces = z[f"{name}/faces"] if f"{name}/faces" in z.files else None
    o = m.evaluate(z[f"{name}/data"], z[f"{name}/stl"], z[f"{name}/obs_mask"], z[f"{name}/bb"], z[f"{name}/res"], z[f"{name}/plane"],
                   mode=sc["mode"], faces=faces, seed=0, **sc["args"])
    assert np.array_equal(o["data_down"], z[f"{name}/data_down"])
    assert np.array_equal(o["data_color"], z[f"{name}/data_color"])
    assert np.array_equal(o["stl_color"], z[f"{name}/stl_color"])
    np.testing.assert_allclose([o["mean_d2s"], o["mean_s2d"], o["overall"]], z[f"{name}/scores"], rtol=1e-12, atol=0)
    ref = O.evaluate(sc["data"], sc["stl"], sc["obs_mask"], sc["bb"], sc["res"], sc["plane"], mode=sc["mode"], faces=sc["faces"],
                     seed=0, **sc["args"])
    for k in ("inbound", "grid_inbound", "in_obs", "above", "dist_d2s", "dist_s2d"):
        assert np.array_equal(o[k], ref[k]), k


def test_cli_writes_reference_results(m, tmp_path):
    import json
    sc = _dtu_scenes.scenes()["sphere"]
    _dtu_scenes.write_dataset(str(tmp_path), sc, 24)
    os.makedirs(tmp_path / "Points" / "stl")
    zero = np.zeros((sc["data"].shape[0], 3))
    import gof_tsdf
    gof_tsdf.write_ply(str(tmp_path / "mesh.ply"), {"vertices": sc["data"].astype(np.float32), "faces": sc["faces"], "colors": zero})
    m.write_vis_ply(str(tmp_path / "Points" / "stl" / "stl024_total.ply"), sc["stl"], np.zeros_like(sc["stl"]))
    a = sc["args"]
    m.main(["--data", str(tmp_path / "mesh.ply"), "--scan", "24", "--dataset_dir", str(tmp_path), "--vis_out_dir", str(tmp_path),
            "--downsample_density", str(a["downsample_density"]), "--patch_size", str(a["patch_size"]), "--max_dist", str(a["max_dist"]),
            "--visualize_threshold", str(a["visualize_threshold"])])
    res = json.load(open(tmp_path / "results.json"))
    # the mesh went through float32 PLY vertices: compare with the oracle on those
    o = O.evaluate(sc["data"].astype(np.float32).astype(np.float64), sc["stl"], sc["obs_mask"], sc["bb"], sc["res"], sc["plane"],
                   faces=sc["faces"], seed=0, **a)
    np.testing.assert_allclose([res["mean_d2s"], res["mean_s2d"], res["overall"]], [o["mean_d2s"], o["mean_s2d"], o["overall"]],
                               rtol=1e-12, atol=0)
    d = m.read_ply(str(tmp_path / "vis_024_d2s.ply"))["points"]
    assert np.array_equal(d, o["data_down"])


def test_two_runs_identical(m):
    sc = _dtu_scenes.scenes()["sphere"]
    a, b = (m.evaluate(sc["data"], sc["stl"], sc["obs_mask"], sc["bb"], sc["res"], sc["plane"], faces=sc["faces"], seed=3, **sc["args"])
            for _ in range(2))
    for k in ("data_down", "dist_d2s", "dist_s2d", "data_color", "stl_color"):
        assert np.array_equal(a[k], b[k])
    assert a["rounds"] == b["rounds"]


# ---- scratch -----------------------------------------------------------------------------------------------------------

GUARD = 64 * 1024


@pytest.mark.parametrize("fill", [0x00, 0xFF])
def test_scratch_contents_and_guard(m, fill):
    lib = m._lib
    rng = np.random.default_rng(9)
    ref, q = _t(rng.normal(size=(5000, 3))), _t(rng.normal(size=(7000, 3)) * 1.2)
    nb = int(lib.gof_nn_dist_scratch_bytes(5000, 7000))
    buf = torch.full((nb + 2 * GUARD,), fill, dtype=torch.uint8, device=DEV)
    out = torch.empty(7000, dtype=torch.float64, device=DEV)
    m._C._check(lib.gof_nn_dist(5000, ref.data_ptr(), 7000, q.data_ptr(), out.data_ptr(), 0, buf.data_ptr() + GUARD, nb,
                                m._C._stream()))
    assert np.array_equal(out.cpu().numpy(), O.nn_sqdist(ref.cpu().numpy(), q.cpu().numpy()))
    assert bool((buf[:GUARD] == fill).all()) and bool((buf[GUARD + nb:] == fill).all())

    pts = rng.uniform(0, 3, (6000, 3))
    perm = rng.permutation(6000)
    nb = int(lib.gof_ordered_downsample_scratch_bytes(6000))
    buf = torch.full((nb + 2 * GUARD,), fill, dtype=torch.uint8, device=DEV)
    kept = torch.empty(6000, dtype=torch.uint8, device=DEV)
    P, perm_t = _t(pts), torch.as_tensor(perm.astype(np.int32), device=DEV)
    pairs = m._C._Scratch(torch.device(DEV))
    rounds, npairs = ctypes.c_int64(0), ctypes.c_int64(0)
    m._C._check(lib.gof_ordered_downsample(6000, P.data_ptr(), perm_t.data_ptr(), 0.2, kept.data_ptr(), ctypes.byref(rounds),
                                           ctypes.byref(npairs), buf.data_ptr() + GUARD, nb, pairs.cb, None, m._C._stream()))
    assert np.array_equal(kept.cpu().numpy().astype(bool), O.ordered_downsample(pts, perm, 0.2))
    assert npairs.value == O.radius_pairs(pts[perm], 0.2).shape[0]
    assert bool((buf[:GUARD] == fill).all()) and bool((buf[GUARD + nb:] == fill).all())


# ---- refusals ----------------------------------------------------------------------------------------------------------

def test_refusals(m):
    sc = _dtu_scenes.scenes()["soup"]
    args = (sc["stl"], sc["obs_mask"], sc["bb"], sc["res"], sc["plane"])
    bad = sc["data"].copy()
    bad[3, 1] = np.nan
    with pytest.raises(ValueError, match="non-finite"):
        m.evaluate(bad, *args, faces=sc["faces"])
    stl = sc["stl"].copy()
    stl[0, 0] = np.inf
    with pytest.raises(ValueError, match="non-finite"):
        m.evaluate(sc["data"], stl, *args[1:], faces=sc["faces"])
    F = sc["faces"].copy()
    F[2, 1] = sc["data"].shape[0]
    with pytest.raises(RuntimeError, match="face index"):
        m.evaluate(sc["data"], *args, faces=F)
    F[2, 1] = -1
    with pytest.raises(RuntimeError, match="face index"):
        m.evaluate(sc["data"], *args, faces=F)
    with pytest.raises(ValueError, match="empty"):
        m.evaluate(np.zeros((0, 3)), *args, mode="pcd")
    with pytest.raises(ValueError, match="empty"):
        m.evaluate(sc["data"], np.zeros((0, 3)), *args[1:], faces=sc["faces"])
    with pytest.raises(ValueError, match="permutation"):
        m.ordered_downsample(_t(np.zeros((4, 3))), torch.tensor([0, 1, 2, 4], device=DEV), 0.1)
    with pytest.raises(RuntimeError, match="permutation"):
        m.ordered_downsample(_t(np.arange(12.0).reshape(4, 3)), torch.tensor([0, 1, 1, 3], device=DEV), 0.1)
    lib = m._lib
    big = 2 ** 30
    rc = lib.gof_nn_dist(big, 1, 1, 1, 1, 0, 1, 1 << 40, None)
    assert rc != 0 and b"2^30" in lib.gof_last_error()
    r, p = ctypes.c_int64(0), ctypes.c_int64(0)
    rc = lib.gof_ordered_downsample(big, 1, 1, 0.1, 1, ctypes.byref(r), ctypes.byref(p), 1, 1 << 40, m._C._Scratch(torch.device(DEV)).cb,
                                    None, None)
    assert rc != 0 and b"2^30" in lib.gof_last_error()


def test_refuses_more_than_2_32_pairs(m):
    n = 93000                                    # n (n - 1) / 2 > 2^32 - 1 coincident pairs
    with pytest.raises(RuntimeError, match="2\\^32 - 1"):
        m.ordered_downsample(_t(np.zeros((n, 3))), torch.arange(n, device=DEV), 0.1)
