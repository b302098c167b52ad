"""Marching tetrahedra.  CPU: the numpy oracle (oracle/tetmesh_oracle.py) against golden vectors produced by importing
the reference's own utils/tetmesh.py (tests/golden/make_golden_tetmesh.py), including its chunked-merge path.
GPU: the CUDA implementation against the same vectors and, at a larger size, against the oracle -- faces and edge ids
bit-exact (int64)."""
import glob
import os

import numpy as np
import pytest
import torch

import tetmesh_oracle

HERE = os.path.dirname(os.path.abspath(__file__))
FIX = sorted(glob.glob(os.path.join(HERE, "golden", "tetmesh_*.npz")))


def test_fixtures_present():
    assert len(FIX) >= 4


@pytest.mark.parametrize("path", FIX, ids=[os.path.basename(p) for p in FIX])
def test_oracle_matches_reference(path):
    z = np.load(path)
    chunk = int(z["chunk_size"]) if "chunk_size" in z.files else 32 * 1024 * 1024
    (pos, esdf), esc, faces, iv = tetmesh_oracle.marching_tetrahedra(z["vertices"], z["tets"], z["sdf"], z["scales"], chunk_size=chunk)
    np.testing.assert_array_equal(iv, z["interp_v"])
    np.testing.assert_array_equal(faces, z["faces"])
    np.testing.assert_array_equal(pos, z["edge_pos"])
    np.testing.assert_array_equal(esdf, z["edge_sdf"])
    np.testing.assert_array_equal(esc, z["edge_scales"])


def test_chunk_rows_is_the_reference_split():
    """gof_tetmesh.chunk_rows, the rows per chunk that set the face order of the CUDA implementation, cuts the tets as
    utils/tetmesh.py:55-58 does: torch.chunk(tets, T // chunk_size + 1) when T > chunk_size, else one chunk.  chunk_tets = 0:
    one chunk."""
    import gof_tetmesh
    for chunk in (1, 7, 1000, gof_tetmesh.CHUNK_TETS):
        for T in sorted({k * chunk + d for k in (1, 2, 3, 10) for d in (-1, 0, 1)} - {0}):
            tets = torch.empty((T, 0))        # the split depends on the row count alone
            want = torch.chunk(tets, T // chunk + 1) if T > chunk else (tets,)
            got = torch.split(tets, gof_tetmesh.chunk_rows(T, chunk))
            assert [t.shape[0] for t in got] == [t.shape[0] for t in want], (T, chunk)
    for T in (1, 7, 1000, 3 * gof_tetmesh.CHUNK_TETS + 1):
        assert gof_tetmesh.chunk_rows(T, 0) == T


@pytest.mark.gpu
@pytest.mark.parametrize("path", FIX, ids=[os.path.basename(p) for p in FIX])
def test_cuda_matches_reference_golden(path):
    import gof_tetmesh
    dev = torch.device("cuda")
    z = np.load(path)
    chunk = int(z["chunk_size"]) if "chunk_size" in z.files else gof_tetmesh.CHUNK_TETS
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    (pos, esdf), esc, faces, iv = gof_tetmesh._unbatched_marching_tetrahedra(t(z["vertices"]), t(z["tets"]), t(z["sdf"]), t(z["scales"]),
                                                                             chunk_tets=chunk)
    np.testing.assert_array_equal(iv.cpu().numpy(), z["interp_v"].reshape(-1, 2))
    np.testing.assert_array_equal(faces.cpu().numpy(), z["faces"].reshape(-1, 3))
    np.testing.assert_array_equal(pos.cpu().numpy(), z["edge_pos"].reshape(-1, 2, 3))
    np.testing.assert_array_equal(esdf.cpu().numpy(), z["edge_sdf"].reshape(-1, 2, 1))
    np.testing.assert_array_equal(esc.cpu().numpy(), z["edge_scales"].reshape(-1, 2, 1))


@pytest.mark.gpu
def test_cuda_large_random_vs_oracle_and_batched_api():
    """400k points / ~2.6M tets (synthetic BCC-like connectivity from a Delaunay of a subset is too slow: random tets over a
    jittered grid exercise the same code), batched entry point, chunked face order with 1M-tet chunks."""
    import gof_tetmesh
    dev = torch.device("cuda")
    rng = np.random.default_rng(5)
    V = 400_000
    v = rng.uniform(-1, 1, size=(V, 3)).astype(np.float32)
    # locally connected random tets: vertex i with three of its index-neighbours
    T = 2_600_000
    a = rng.integers(0, V, size=T)
    tets = np.stack([a, (a + rng.integers(1, 50, size=T)) % V, (a + rng.integers(50, 400, size=T)) % V, (a + rng.integers(400, 3000, size=T)) % V], axis=1).astype(np.int64)
    sdf = (0.8 - np.linalg.norm(v, axis=1) + 0.05 * rng.standard_normal(V)).astype(np.float32)
    scales = rng.uniform(0.01, 0.1, size=(V, 1)).astype(np.float32)
    t = lambda x: torch.from_numpy(x).to(dev)
    verts_list, scale_list, faces_list, iv_list = gof_tetmesh.marching_tetrahedra(t(v)[None], t(tets), t(sdf)[None], t(scales)[None])
    (opos, osdf), osc, ofaces, oiv = tetmesh_oracle.marching_tetrahedra(v, tets, sdf, scales)
    np.testing.assert_array_equal(iv_list[0].cpu().numpy(), oiv)
    np.testing.assert_array_equal(faces_list[0].cpu().numpy(), ofaces)
    np.testing.assert_array_equal(verts_list[0][0].cpu().numpy(), opos)
    np.testing.assert_array_equal(scale_list[0].cpu().numpy(), osc)
    assert ofaces.shape[0] > 100_000
    # chunked order
    (_, _), _, cf, civ = gof_tetmesh._unbatched_marching_tetrahedra(t(v), t(tets), t(sdf), t(scales), chunk_tets=1_000_000)
    (_, _), _, of2, oiv2 = tetmesh_oracle.marching_tetrahedra(v, tets, sdf, scales, chunk_size=1_000_000)
    np.testing.assert_array_equal(civ.cpu().numpy(), oiv2)
    np.testing.assert_array_equal(cf.cpu().numpy(), of2)
