"""CPU: the opacity-field lattice oracle (oracle/field_grid_oracle.py) against brute force, the float64 corner and frustum
bounds of tetra_points_oracle and the TSDF extraction; and the C ABI's refusals, which return before any device work."""
import ctypes
import os
from fractions import Fraction

import numpy as np
import pytest

import _field_grid_scenes as FS
import field_grid_oracle as O
import tetra_points_oracle as tpo

f32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _round_f32(x):
    """Round-to-nearest-even of the exact rational x to float32 (finite, normal range)."""
    f = f32(float(x))
    lo, hi = (np.nextafter(f, f32(-np.inf)), f) if Fraction(float(f)) > x else (f, np.nextafter(f, f32(np.inf)))
    dl, dh = x - Fraction(float(lo)), Fraction(float(hi)) - x
    if dl != dh:
        return lo if dl < dh else hi
    return lo if (int(np.asarray(lo).view(np.uint32)) & 1) == 0 else hi


def test_fma32_is_correctly_rounded():
    rng = np.random.default_rng(0)
    a = (rng.standard_normal(3000) * np.exp(rng.uniform(-5, 5, 3000))).astype(f32)
    b = (rng.standard_normal(3000) * np.exp(rng.uniform(-5, 5, 3000))).astype(f32)
    c = (rng.standard_normal(3000) * np.exp(rng.uniform(-8, 8, 3000))).astype(f32)
    # a b on a float32 rounding midpoint: 1 + 2^-11 + 2^-24 between 1 + 2^-11 and its successor; c decides, or ties go to even
    m = f32(1 + 2.0 ** -12)
    a = np.concatenate([a, [m, m, m, m]]).astype(f32)
    b = np.concatenate([b, [m, m, m, -m]]).astype(f32)
    c = np.concatenate([c, [2.0 ** -60, -(2.0 ** -60), 0.0, 2.0 ** -60]]).astype(f32)
    got = O.fma32(a, b, c)
    for i in range(a.size):
        want = _round_f32(Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i])))
        assert got[i] == want, (i, a[i], b[i], c[i])
    assert got[-4] == np.nextafter(f32(1 + 2.0 ** -11), f32(2)) and got[-3] == f32(1 + 2.0 ** -11) and got[-2] == f32(1 + 2.0 ** -11)


def test_corners_and_frustum_agree_with_the_float64_bounds():
    xyz, sc, rot = FS.gaussians(400, 1)
    views = FS.views_around()
    c = O.corners(xyz, sc, rot)
    pts64, bnd, _ = tpo.tetra_points(xyz, sc, rot)
    P = xyz.shape[0]
    assert np.all(np.abs(c.reshape(-1, 3).astype(np.float64) - pts64[:8 * P]) <= bnd[:8 * P])
    seen = O.in_view(xyz, FS.table(views))
    mask, decided = tpo.frustum_decision(xyz, FS.table(views))
    assert decided.mean() > 0.99 and np.array_equal(seen[decided], mask[decided])
    assert seen.sum() > 100 and not seen[-2:].any()


@pytest.mark.parametrize("seed", [1, 2])
def test_blocks_equal_brute_force(seed):
    xyz, sc, rot = FS.gaussians(300, seed)
    tab = FS.table(FS.views_around())
    seen, lo, hi = O.boxes(xyz, sc, rot, tab, FS.S_EXACT)
    bs = f32(FS.B_EXACT * FS.S_EXACT)
    keys = O.blocks(xyz, sc, rot, tab, FS.S_EXACT, FS.B_EXACT)
    assert np.array_equal(keys, O.brute_force_blocks(lo[seen], hi[seen], bs))
    assert np.all(np.diff(keys) > 0) and np.any(O.T.unpack_keys(keys) < 0)
    # the zero-scale Gaussians whose dilated boxes end exactly on a block face touch the block beyond it
    face = xyz.shape[0] - 6 + np.arange(4)
    assert np.all(seen[face]) and np.all(sc[face] == 0)
    for g in face:
        for a in range(3):
            if hi[g, a] == np.floor(hi[g, a]):
                b = O.T.unpack_keys(keys)
                assert np.any(b[:, a] == int(hi[g, a]))


def test_blocks_at_a_general_voxel_size():
    """s = 0.03: the quotients round, so a Gaussian whose dilated bound lies within rounding of a block face may touch one block
    more or less than the exact intersection says.  Every other Gaussian's blocks equal the brute force's."""
    xyz, sc, rot = FS.gaussians(200, 3)
    tab = FS.table(FS.views_around())
    s, B = 0.03, 8
    seen, lo, hi = O.boxes(xyz, sc, rot, tab, s)
    bs = f32(B * f32(s))
    q = np.concatenate([lo, hi], 1).astype(np.float64) / float(bs)
    near_face = np.any(np.abs(q - np.round(q)) < 1e-5, axis=1)
    keep = ~near_face
    assert seen[keep].sum() > 150
    keys = O.blocks(xyz[keep], sc[keep], rot[keep], tab, s, B)
    assert np.array_equal(keys, O.brute_force_blocks(lo[keep & seen], hi[keep & seen], bs))
    assert keys.size > 50
    # the near-face Gaussians add blocks next to the ones the brute force gives for them
    full = O.blocks(xyz, sc, rot, tab, s, B)
    assert np.all(np.isin(keys, full))


def test_zero_scales_and_nothing_in_view():
    xyz, sc, rot = FS.gaussians(50, 4)
    tab = FS.table(FS.views_around())
    keys = O.blocks(xyz, np.zeros_like(sc), rot, tab, FS.S_EXACT, FS.B_EXACT)
    # a point dilated by s = 0.25 touches one block per axis unless it lies within s of a face
    seen = O.in_view(xyz, tab)
    assert 0 < keys.size <= 8 * seen.sum()
    far = FS.table([FS.view(np.eye(3), (0, 0, -100.0))])
    assert O.blocks(xyz, sc, rot, far, FS.S_EXACT, FS.B_EXACT).size == 0
    empty = O.blocks(np.zeros((0, 3), f32), np.zeros((0, 3), f32), np.zeros((0, 4), f32), tab, FS.S_EXACT, FS.B_EXACT)
    assert empty.dtype == np.int64 and empty.size == 0
    assert O.lattice_points(empty, FS.S_EXACT, FS.B_EXACT).shape == (0, 3)


def test_key_limit():
    top = (1 << 20) - 0.5                         # dilated box [2^20 - 0.75, 2^20 - 0.25]: the last block, 2^20 - 1
    x, s, r, v = FS.key_limit_case(top)
    k = O.blocks(x, s, r, FS.table(v), FS.S_EXACT, FS.B_EXACT)
    top_b = (1 << 20) - 1
    assert sorted(map(tuple, O.T.unpack_keys(k).tolist())) == sorted((top_b, y, z) for y in (-1, 0) for z in (-1, 0))
    for bad in ((1 << 20) - 0.125, -(1 << 20) + 0.125):      # hi = 2^20 + 0.125, lo = -2^20 - 0.125
        x, s, r, v = FS.key_limit_case(bad)
        with pytest.raises(O.BlockRangeError):
            O.blocks(x, s, r, FS.table(v), FS.S_EXACT, FS.B_EXACT)
    x, s, r, v = FS.key_limit_case(-(1 << 20) + 0.5, axis=1)
    k = O.blocks(x, s, r, FS.table(v), FS.S_EXACT, FS.B_EXACT)
    assert np.all(O.T.unpack_keys(k)[:, 1] == -(1 << 20))


def test_lattice_points_are_exact_multiples():
    xyz, sc, rot = FS.gaussians(100, 5)
    tab = FS.table(FS.views_around())
    for s, B in ((FS.S_EXACT, FS.B_EXACT), (0.03, 8)):
        keys = O.blocks(xyz, sc, rot, tab, s, B)
        pts = O.lattice_points(keys, s, B)
        g = O.voxels(keys, B)
        assert pts.dtype == np.float32 and pts.shape == (keys.size * B ** 3, 3)
        assert np.array_equal(pts, g.astype(f32) * f32(s))
        if s == FS.S_EXACT:
            assert np.array_equal(pts.astype(np.float64), g * 0.25)
        # pool order: block in key order, then voxel i + B j + B^2 k
        assert np.array_equal(g[:B ** 3][:, 0] - g[0, 0], np.arange(B ** 3) % B)


def test_marching_cubes_edges_match_the_tsdf_vertices():
    """The oracle's own edge list against tsdf_oracle's interpolated vertices: same count and order, each vertex on its edge."""
    rng = np.random.default_rng(6)
    s, B = 0.25, 4
    keys = O.T.pack_keys(np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0], [0, 0, 1], [-1, 0, 0], [3, 3, 3]]))
    keys = np.sort(keys)
    pts = O.lattice_points(keys, s, B).astype(np.float64)
    vals = (np.linalg.norm(pts - [0.3, 0.4, 0.2], axis=1) - 0.6 + 0.05 * rng.standard_normal(pts.shape[0])).astype(f32)
    m = O.marching_cubes(keys, vals, s, B)
    V = m["vertices"].shape[0]
    assert V > 20 and m["faces"].shape[0] > 20
    assert m["edge_points"].shape == (V, 2, 3) and m["edge_values"].shape == (V, 2)
    assert m["faces"].max() < V
    d = m["edge_points"][:, 1] - m["edge_points"][:, 0]
    assert np.all((d != 0).sum(1) == 1) and np.all(d[d != 0] == f32(s))
    on = d == 0
    assert np.array_equal(m["vertices"][on], m["edge_points"][:, 0][on])
    ax = ~on
    lo, hi = m["edge_points"][:, 0][ax], m["edge_points"][:, 1][ax]
    assert np.all((m["vertices"][ax] >= lo) & (m["vertices"][ax] <= hi))
    assert np.all((m["edge_values"][:, 0] < 0) != (m["edge_values"][:, 1] < 0))
    idx = {tuple(p): i for i, p in enumerate(O.lattice_points(keys, s, B).tolist())}
    for k in range(3):
        i0, i1 = idx[tuple(m["edge_points"][k, 0].tolist())], idx[tuple(m["edge_points"][k, 1].tolist())]
        assert m["edge_values"][k, 0] == vals[i0] and m["edge_values"][k, 1] == vals[i1]


# ---- the C ABI's refusals, before any device work ------------------------------------------------------------------------
class _Par(ctypes.Structure):
    _fields_ = [("voxel_size", ctypes.c_float), ("block_resolution", ctypes.c_int)]


@pytest.fixture(scope="module")
def lib():
    path = os.path.join(ROOT, "gaussian-opacity-fields_b200", "diff_gaussian_rasterization", "libgof_b200.so")
    if not os.path.exists(path):
        pytest.skip("libgof_b200.so not built")
    L = ctypes.CDLL(path)
    L.gof_last_error.restype = ctypes.c_char_p
    v, i64, P, f = ctypes.c_void_p, ctypes.c_int64, ctypes.POINTER(_Par), ctypes.c_float
    i64p = ctypes.POINTER(ctypes.c_int64)
    L.gof_field_grid_points.argtypes = [P, i64, v, v, v]
    L.gof_field_grid_blocks_count.argtypes = [P, ctypes.c_int, v, v, v, ctypes.c_int, v, f, f, v, v, v, v, i64p, v]
    L.gof_field_grid_blocks_emit.argtypes = [P, ctypes.c_int, v, v, i64, v, v]
    L.gof_field_grid_extract_count.argtypes = [P, i64, v, v, v, v, i64p, i64p, v]
    L.gof_field_grid_extract_emit.argtypes = [P, i64, v, v, v, i64, i64, v, v, v, v]
    return L


FAKE = 0x1000   # a non-NULL pointer the refusals never dereference


def test_abi_refuses_bad_parameters(lib):
    for s, B in ((0.0, 8), (-1.0, 8), (float("nan"), 8), (0.1, 0), (0.1, 65), (0.1, -3)):
        p = _Par(s, B)
        assert lib.gof_field_grid_points(ctypes.byref(p), 1, FAKE, FAKE, None) == -1
        assert b"block_resolution in 1..64" in lib.gof_last_error()
        n = ctypes.c_int64(7)
        assert lib.gof_field_grid_blocks_count(ctypes.byref(p), 1, FAKE, FAKE, FAKE, 1, FAKE, 0.02, 1e6, FAKE, None, FAKE, None,
                                               ctypes.byref(n), None) == -1
        assert n.value == 0
        nv, nf = ctypes.c_int64(1), ctypes.c_int64(1)
        assert lib.gof_field_grid_extract_count(ctypes.byref(p), 1, FAKE, FAKE, FAKE, None, ctypes.byref(nv), ctypes.byref(nf), None) == -1
        assert lib.gof_field_grid_extract_emit(ctypes.byref(p), 1, FAKE, FAKE, FAKE, 1, 1, FAKE, FAKE, FAKE, None) == -1
    assert lib.gof_field_grid_points(None, 1, FAKE, FAKE, None) == -1


def test_abi_refuses_null_pointers(lib):
    p = _Par(0.1, 8)
    n = ctypes.c_int64(0)
    assert lib.gof_field_grid_points(ctypes.byref(p), 3, None, FAKE, None) == -1
    assert lib.gof_field_grid_points(ctypes.byref(p), 3, FAKE, None, None) == -1
    assert b"NULL" in lib.gof_last_error()
    args = [FAKE, FAKE, FAKE, 1, FAKE, 0.02, 1e6, FAKE, None, FAKE, None, ctypes.byref(n), None]
    for i in (0, 1, 2, 4):
        a = list(args)
        a[i] = None
        assert lib.gof_field_grid_blocks_count(ctypes.byref(p), 5, *a) == -1, i
    for i in (7, 9, 11):   # the allocators and the output count
        a = list(args)
        a[i] = None
        assert lib.gof_field_grid_blocks_count(ctypes.byref(p), 5, *a) == -1, i
    assert lib.gof_field_grid_blocks_count(ctypes.byref(p), -1, *args) == -1
    assert lib.gof_field_grid_blocks_count(ctypes.byref(p), 5, FAKE, FAKE, FAKE, 0, FAKE, 0.02, 1e6, FAKE, None, FAKE, None,
                                           ctypes.byref(n), None) == -1
    assert lib.gof_field_grid_blocks_count(ctypes.byref(p), 5, FAKE, FAKE, FAKE + 4, 1, FAKE, 0.02, 1e6, FAKE, None, FAKE, None,
                                           ctypes.byref(n), None) == -1
    assert b"16-byte aligned" in lib.gof_last_error()
    assert lib.gof_field_grid_blocks_emit(ctypes.byref(p), 5, None, FAKE, 3, FAKE, None) == -1
    nv, nf = ctypes.c_int64(0), ctypes.c_int64(0)
    assert lib.gof_field_grid_extract_count(ctypes.byref(p), 2, None, FAKE, FAKE, None, ctypes.byref(nv), ctypes.byref(nf), None) == -1
    assert lib.gof_field_grid_extract_count(ctypes.byref(p), 2, FAKE, None, FAKE, None, ctypes.byref(nv), ctypes.byref(nf), None) == -1
    assert lib.gof_field_grid_extract_emit(ctypes.byref(p), 2, FAKE, FAKE, FAKE, 4, 2, None, FAKE, FAKE, None) == -1
    # nothing to do is not an error, and needs no pointer
    assert lib.gof_field_grid_points(ctypes.byref(p), 0, None, None, None) == 0
    assert lib.gof_field_grid_blocks_count(ctypes.byref(p), 0, None, None, None, 1, None, 0.02, 1e6, FAKE, None, FAKE, None,
                                           ctypes.byref(n), None) == 0 and n.value == 0
    assert lib.gof_field_grid_extract_count(ctypes.byref(p), 0, None, None, FAKE, None, ctypes.byref(nv), ctypes.byref(nf), None) == 0


@pytest.mark.parametrize("B", [1, 8, 64])
def test_abi_refuses_the_point_count_limit(lib, B):
    p = _Par(0.1, B)
    n3 = B ** 3
    last_ok = (2 ** 31 - 1) // n3
    assert lib.gof_field_grid_points(ctypes.byref(p), last_ok + 1, FAKE, FAKE, None) == -1
    assert b"2^31" in lib.gof_last_error()
    nv, nf = ctypes.c_int64(0), ctypes.c_int64(0)
    assert lib.gof_field_grid_extract_count(ctypes.byref(p), last_ok + 1, FAKE, FAKE, FAKE, None, ctypes.byref(nv), ctypes.byref(nf),
                                            None) == -1
    assert b"2^31" in lib.gof_last_error()
    assert lib.gof_field_grid_points(ctypes.byref(p), -1, FAKE, FAKE, None) == -1
    # the public function refuses the same limit with ValueError, before allocating
    import gof_extract
    import torch
    with pytest.raises(ValueError, match="2\\^31"):
        gof_extract.field_grid_points(torch.zeros(last_ok + 1, dtype=torch.int64, device="meta"), 0.1, B)


def test_public_functions_refuse_bad_tensors():
    """Keys must be 1-D int64 and on the GPU, values float32 of the lattice's size: refused before any launch."""
    import gof_extract
    import torch
    for bad in (torch.zeros(3, dtype=torch.int32), torch.zeros(3), torch.zeros(3, 1, dtype=torch.int64), [1, 2, 3]):
        with pytest.raises(ValueError, match="int64"):
            gof_extract.field_grid_points(bad, 0.1, 4)
        with pytest.raises(ValueError, match="int64"):
            gof_extract.field_grid_marching_cubes(bad, torch.zeros(192), 0.1, 4)
    keys = torch.zeros(3, dtype=torch.int64)
    with pytest.raises(RuntimeError, match="CUDA"):
        gof_extract.field_grid_points(keys, 0.1, 4)
    for bad in (torch.zeros(192, dtype=torch.float64), torch.zeros(191), torch.zeros(3, 64), None):
        with pytest.raises(ValueError, match="float32"):
            gof_extract.field_grid_marching_cubes(keys, bad, 0.1, 4)
    with pytest.raises(RuntimeError, match="CUDA"):
        gof_extract.field_grid_marching_cubes(keys, torch.zeros(192), 0.1, 4)


def test_public_function_refuses_bad_parameters():
    import gof_extract
    import torch
    x = torch.zeros(4, 3)
    for kw, msg in ((dict(voxel_size=0.0), "voxel_size"), (dict(voxel_size=-0.5), "voxel_size"), (dict(voxel_size=float("nan")), "voxel_size"),
                    (dict(voxel_size=0.1, block_resolution=0), "1..64"), (dict(voxel_size=0.1, block_resolution=65), "1..64")):
        with pytest.raises(ValueError, match=msg):
            gof_extract.extract_level_set_grid(x, x, torch.zeros(4, 4), [], None, **kw)
