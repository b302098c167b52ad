"""CPU tests of the DTU evaluation's oracle (oracle/dtu_eval_oracle.py, DESIGN section 4.6) against the reference's own
dtu_eval/eval.py: the stored outputs of tests/golden/dtu_eval_ref.npz and, where baseline/stage_ref.sh staged the script, live
runs on fresh seeds; plus the PLY reader and writer of gof_dtu_eval and the permutation that stands for the shuffle."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]
import _dtu_scenes  # noqa: E402
import dtu_eval_oracle as O  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "dtu_eval_ref.npz")
SCENES = ("sphere", "soup", "pcd")


def _golden_scene(z, name):
    g = lambda k: z[f"{name}/{k}"]  # noqa: E731
    faces = g("faces") if f"{name}/faces" in z.files else None
    sc = _dtu_scenes.scenes()[name]
    return dict(mode=sc["mode"], data=g("data"), faces=faces, stl=g("stl"), obs_mask=g("obs_mask"), bb=g("bb"), res=g("res"),
                plane=g("plane"), args=sc["args"])


def _oracle(sc, seed):
    return O.evaluate(sc["data"], sc["stl"], sc["obs_mask"], sc["bb"], sc["res"], sc["plane"], mode=sc["mode"], faces=sc["faces"],
                      seed=seed, **sc["args"])


def _same(o, ref):
    assert np.array_equal(o["data_down"], ref["data_down"])
    assert np.array_equal(o["data_color"], ref["data_color"])
    assert np.array_equal(o["stl_color"], ref["stl_color"])
    got = np.array([o["mean_d2s"], o["mean_s2d"], o["overall"]])
    want = np.asarray(ref["scores"])
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)


@pytest.mark.parametrize("name", SCENES)
def test_oracle_equals_golden(name):
    z = np.load(GOLDEN)
    sc = _golden_scene(z, name)
    o = _oracle(sc, 0)
    _same(o, {k: z[f"{name}/{k}"] for k in ("data_down", "data_color", "stl_color", "scores")})


@pytest.mark.parametrize("name,seed", [("sphere", 5), ("soup", 17), ("pcd", 123)])
def test_oracle_equals_live_reference(name, seed):
    sc = _dtu_scenes.scenes()[name]
    ref = _dtu_scenes.run_reference(sc, seed)
    if ref is None:
        pytest.skip("the reference's dtu_eval/eval.py is not staged (baseline/stage_ref.sh)")
    ref["scores"] = [ref["mean_d2s"], ref["mean_s2d"], ref["overall"]]
    _same(_oracle(sc, seed), ref)


def test_sampling_edge_faces():
    """Zero-area faces give no samples, a face below the density (n1 = 0) gives none, the vertices come first unchanged."""
    V = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [0, 0.01, 0], [5, 5, 5]], np.float64)
    F = np.array([[0, 1, 2], [0, 0, 1], [0, 1, 3]])
    out = O.sample_mesh(V, F, 0.2)
    assert np.array_equal(out[:5], V)
    _, _, _, n1, n2, ok = O.face_params(V, F, 0.2)
    assert list(ok) == [False, False, True]
    assert n1[2] == 5 and n2[2] == 0 and out.shape[0] == 5


def test_perm_equals_shuffle():
    x = np.random.default_rng(3).normal(size=(1000, 3))
    for seed in (0, 1, 99):
        a = x.copy()
        np.random.default_rng(seed).shuffle(a, axis=0)
        assert np.array_equal(a, x[np.random.default_rng(seed).permutation(x.shape[0])])


def test_downsample_inclusive_radius():
    """Points exactly r apart are neighbours: of a lattice with spacing r only every other point along a line survives."""
    p = np.stack([np.arange(9) * 0.5, np.zeros(9), np.zeros(9)], 1)
    kept = O.ordered_downsample(p, np.arange(9), 0.5)
    assert kept.tolist() == [True, False] * 4 + [True]


def _gof_dtu_eval():
    pkg = os.path.join(ROOT, "gaussian-opacity-fields_b200")
    if pkg not in sys.path:
        sys.path.insert(0, pkg)
    try:
        import gof_dtu_eval
    except ImportError as e:
        pytest.skip(f"the package's library is not built: {e}")
    return gof_dtu_eval


def test_ply_reader_round_trips_vis_writer(tmp_path):
    m = _gof_dtu_eval()
    rng = np.random.default_rng(0)
    p, c = rng.normal(size=(100, 3)) * 1e3, rng.random((100, 3))
    m.write_vis_ply(str(tmp_path / "v.ply"), p, c)
    r = m.read_ply(str(tmp_path / "v.ply"))
    assert r["faces"] is None
    assert np.array_equal(r["points"], p)


def test_ply_reader_reads_tsdf_mesh(tmp_path):
    m = _gof_dtu_eval()
    import gof_tsdf
    rng = np.random.default_rng(1)
    mesh = {"vertices": rng.normal(size=(50, 3)).astype(np.float32), "faces": rng.integers(0, 50, (80, 3)),
            "colors": rng.random((50, 3)).astype(np.float32)}
    gof_tsdf.write_ply(str(tmp_path / "t.ply"), mesh)
    r = m.read_ply(str(tmp_path / "t.ply"))
    assert np.array_equal(r["points"], mesh["vertices"].astype(np.float64))
    assert np.array_equal(r["faces"], mesh["faces"])


def test_ply_reader_any_scalar_types_and_refusals(tmp_path):
    m = _gof_dtu_eval()
    vert = np.array([(1, 2.5, -3, 7), (4, 5.5, 6, 8)], dtype=[("x", "<i2"), ("y", "<f8"), ("z", "<i4"), ("q", "u1")])
    face = np.array([(3, [0, 1, 1])], dtype=[("n", "u1"), ("i", "<u4", (3,))])
    hdr = ("ply\nformat binary_little_endian 1.0\nelement vertex 2\nproperty short x\nproperty double y\nproperty int z\n"
           "property uchar q\nelement face 1\nproperty list uchar uint vertex_indices\nend_header\n")
    (tmp_path / "a.ply").write_bytes(hdr.encode() + vert.tobytes() + face.tobytes())
    r = m.read_ply(str(tmp_path / "a.ply"))
    assert np.array_equal(r["points"], [[1, 2.5, -3], [4, 5.5, 6]])
    assert np.array_equal(r["faces"], [[0, 1, 1]])
    (tmp_path / "b.ply").write_bytes(b"ply\nformat ascii 1.0\nelement vertex 0\nproperty float x\nend_header\n")
    with pytest.raises(ValueError, match="binary_little_endian"):
        m.read_ply(str(tmp_path / "b.ply"))
