"""GPU: simple_knn.distCUDA2 (csrc/knn.cu) bit for bit against the brute-force CPU oracle (oracle/knn_oracle.c) and against
the stored outputs of the unmodified reference extension (tests/golden/live_knn.npz, tests/golden/make_golden_knn.py)."""
import ctypes
import hashlib
import os

import numpy as np
import pytest
import torch

import gof_synth
import knn_oracle

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "live_knn.npz")


def _dist(pts_np, device=DEV):
    from simple_knn._C import distCUDA2
    out = distCUDA2(torch.from_numpy(pts_np).to(device))
    assert out.dtype == torch.float32 and out.device == torch.device(device) and out.shape == (pts_np.shape[0],)
    return out.cpu().numpy()


def _assert_bits(got, want):
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape
    bad = np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, f"{bad.size} differ, first at {bad[:5]}: {got[bad[:5]]} vs {want[bad[:5]]}"


@pytest.mark.parametrize("kind", gof_synth.POINT_CLOUD_KINDS)
@pytest.mark.parametrize("P", [0, 1, 2, 3, 4, 5, 31, 32, 33, 1023, 1024, 1025, 4097])
def test_small_clouds_match_oracle(kind, P):
    pts = gof_synth.make_point_cloud(kind, P, seed=P + 1)
    _assert_bits(_dist(pts), knn_oracle.knn_mean_dist(pts))


@pytest.mark.parametrize("kind", gof_synth.POINT_CLOUD_KINDS)
def test_65537_points_match_oracle(kind):
    pts = gof_synth.make_point_cloud(kind, 65537, seed=3)
    _assert_bits(_dist(pts), knn_oracle.knn_mean_dist(pts))


def test_edge_values():
    from simple_knn._C import distCUDA2
    assert distCUDA2(torch.zeros(0, 3, device=DEV)).shape == (0,)
    assert np.isposinf(distCUDA2(torch.ones(1, 3, device=DEV)).cpu().numpy()).all()
    assert np.isposinf(distCUDA2(torch.rand(2, 3, device=DEV)).cpu().numpy()).all()
    three = distCUDA2(torch.tensor([[0., 0, 0], [1, 0, 0], [0, 2, 0]], device=DEV)).cpu().numpy()
    fm = np.float32(np.finfo(np.float32).max)
    assert three[0] == np.float32((np.float32(1) + np.float32(4)) + fm) / np.float32(3)
    assert (distCUDA2(torch.zeros(10, 3, device=DEV)) == 0).all()   # coincident points count, at distance 0


@pytest.mark.skipif(not os.path.exists(GOLDEN), reason="tests/golden/live_knn.npz not recorded")
def test_reference_outputs():
    g = np.load(GOLDEN)
    names = sorted({k.split("/")[0] for k in g.files})
    assert len(names) >= 8
    for name in names:
        kind, P, seed = g[f"{name}/spec"]
        pts = gof_synth.make_point_cloud(str(kind), int(P), int(seed))
        out = _dist(pts)
        _assert_bits(out[g[f"{name}/idx"]], g[f"{name}/val"])
        assert hashlib.sha256(out.tobytes()).hexdigest() == str(g[f"{name}/sha256"]), name


@pytest.mark.parametrize("kind,P", [("colmap", 1 << 24), ("core", 1 << 20)])
def test_large_cloud_spot_check(kind, P):
    pts = gof_synth.make_point_cloud(kind, P, seed=5)
    out = _dist(pts)
    q = np.random.default_rng(9).choice(P, 256, replace=False)
    _assert_bits(out[q], knn_oracle.knn_mean_dist(pts, queries=q))


def test_permutation_equivariance():
    pts = gof_synth.make_point_cloud("colmap", 100003, seed=8)
    perm = np.random.default_rng(1).permutation(pts.shape[0])
    _assert_bits(_dist(pts[perm]), _dist(pts)[perm])


def test_rejects_bad_input():
    from simple_knn._C import distCUDA2
    with pytest.raises(RuntimeError):
        distCUDA2(torch.rand(10, 3))
    with pytest.raises(RuntimeError):
        distCUDA2(torch.rand(10, 3, device=DEV, dtype=torch.float64))
    for shape in [(10,), (10, 2), (10, 4), (2, 5, 3), (30,)]:
        with pytest.raises(RuntimeError):
            distCUDA2(torch.rand(*shape, device=DEV))


def test_odd_offset_and_non_contiguous_input():
    from simple_knn._C import distCUDA2
    pts = gof_synth.make_point_cloud("uniform", 5000, seed=4)
    want = knn_oracle.knn_mean_dist(pts)
    flat = torch.zeros(1 + pts.size, device=DEV)
    flat[1:] = torch.from_numpy(pts.reshape(-1)).to(DEV)
    _assert_bits(distCUDA2(flat[1:].view(-1, 3)).cpu().numpy(), want)
    wide = torch.zeros(pts.shape[0], 5, device=DEV)
    wide[:, 1:4] = torch.from_numpy(pts).to(DEV)
    _assert_bits(distCUDA2(wide[:, 1:4]).cpu().numpy(), want)
    _assert_bits(distCUDA2(torch.from_numpy(np.ascontiguousarray(pts.T)).to(DEV).t()).cpu().numpy(), want)


def test_other_device_and_side_stream():
    from simple_knn._C import distCUDA2
    pts = gof_synth.make_point_cloud("colmap", 20000, seed=6)
    want = knn_oracle.knn_mean_dist(pts)
    dev = torch.device(f"cuda:{torch.cuda.device_count() - 1}")
    _assert_bits(_dist(pts, dev), want)
    x = torch.from_numpy(pts).to(DEV)
    s = torch.cuda.Stream(DEV)
    s.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(s):
        out = distCUDA2(x)
    s.synchronize()
    _assert_bits(out.cpu().numpy(), want)


def test_graph_capture_replays_on_new_points():
    from simple_knn._C import distCUDA2
    a = gof_synth.make_point_cloud("uniform", 30000, seed=1)
    b = gof_synth.make_point_cloud("colmap", 30000, seed=2)
    static = torch.from_numpy(a).to(DEV)
    s = torch.cuda.Stream(DEV)
    s.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(s):
        distCUDA2(static)   # warm-up outside the capture
    torch.cuda.current_stream(DEV).wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = distCUDA2(static)
    static.copy_(torch.from_numpy(b).to(DEV))
    g.replay()
    torch.cuda.synchronize()
    _assert_bits(out.cpu().numpy(), _dist(b))
    _assert_bits(out.cpu().numpy(), knn_oracle.knn_mean_dist(b))


def test_scratch_bounds_and_initialisation():
    """The C ABI with scratch pre-filled with 0x00 and with 0xFF gives identical results, equal to the oracle, and a guard
    band after the scratch layout stays intact."""
    from diff_gaussian_rasterization import _C
    import simple_knn._C as K
    guard, canary = 64 * 1024, 0x5A
    for kind, P in [("colmap", 70001), ("nonfinite", 4097), ("lattice", 33)]:
        pts = gof_synth.make_point_cloud(kind, P, seed=7)
        x = torch.from_numpy(pts).to(DEV)
        nbytes = int(K._lib.gof_knn_scratch_bytes(P))
        results = []
        for fill in (0x00, 0xFF):
            buf = torch.full((nbytes + guard,), fill, dtype=torch.uint8, device=DEV)
            buf[nbytes:] = canary
            out = torch.full((P,), float("nan"), device=DEV)
            _C._check(K._lib.gof_knn_mean_dist(P, x.data_ptr(), out.data_ptr(), buf.data_ptr(), nbytes, _C._stream()))
            torch.cuda.synchronize()
            assert bool((buf[nbytes:] == canary).all()), "write past the end of the scratch layout"
            results.append(out.cpu().numpy())
        _assert_bits(results[0], results[1])
        _assert_bits(results[0], knn_oracle.knn_mean_dist(pts))
    assert K._lib.gof_knn_mean_dist(-1, None, None, None, 0, None) == -1
    x = torch.rand(100, 3, device=DEV)
    out = torch.empty(100, device=DEV)
    small = torch.empty(16, dtype=torch.uint8, device=DEV)
    assert K._lib.gof_knn_mean_dist(100, x.data_ptr(), out.data_ptr(), small.data_ptr(), 16, _C._stream()) == -1
    assert b"scratch" in _C._lib.gof_last_error()
