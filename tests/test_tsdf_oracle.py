"""CPU: the TSDF fusion / marching-cubes oracle (oracle/tsdf_oracle.py) against brute force and geometry."""
import numpy as np
import pytest

import _tsdf_scenes as S
import gof_synth
import tsdf_oracle as O

f32 = np.float32
W, H = 64, 48
FX, FY, CX, CY = f32(40.0), f32(40.0), f32(31.5), f32(23.5)


def test_plane_touch_matches_brute_force_and_tsdf_formula():
    s, B = 0.05, 8
    vol = O.Volume(voxel_size=s, block_resolution=B)
    d = np.full((H, W), 2.0, np.float32)
    E = np.eye(4, dtype=np.float32)
    keys = vol.integrate(d, np.zeros((3, H, W), np.float32), FX, FY, CX, CY, E)
    # brute force: every sampled pixel, every block whose index range covers [p - tau, p + tau] on each axis
    tau, bs = vol.tau, vol.bs
    want = set()
    for v in range(0, H, 4):
        for u in range(0, W, 4):
            p = np.array([((f32(u) - CX) * f32(2.0)) / FX, ((f32(v) - CY) * f32(2.0)) / FY, f32(2.0)], np.float32)
            lo = np.floor((p - tau) / bs).astype(int)
            hi = np.floor((p + tau) / bs).astype(int)
            for bz in range(lo[2], hi[2] + 1):
                for by in range(lo[1], hi[1] + 1):
                    for bx in range(lo[0], hi[0] + 1):
                        want.add(int(O.pack_keys([[bx, by, bz]])[0]))
    assert keys.tolist() == sorted(want)
    assert np.array_equal(vol.keys, keys)
    # tsdf of an updated voxel of a fronto-parallel plane seen by an identity camera: min(d - z, tau) / tau, weight 1
    st = vol.state()
    lin = np.arange(B ** 3)
    z = (O.unpack_keys(st["keys"])[:, 2:3] * B + lin[None] // (B * B)).astype(np.float32) * f32(s)
    upd = st["weight"] > 0
    assert upd.any()
    assert np.array_equal(st["tsdf"][upd], (np.minimum(f32(2.0) - z, tau) / tau)[upd])
    assert np.all(f32(2.0) - z[upd] >= -tau)
    assert np.all(st["weight"][upd] == 1)


@pytest.fixture(scope="module")
def sphere():
    vol = O.Volume(voxel_size=0.02, block_resolution=8)
    views = gof_synth.make_surface_views(320, 240, 40)
    for v in views:
        fx, fy, cx, cy, E = S.view_params(v)
        vol.integrate(S.sphere_depth(v), S.sphere_color(v, (0.25, 0.5, 0.125)), fx, fy, cx, cy, E)
    return vol, vol.extract_triangle_mesh()


def test_sphere_mesh_is_closed_oriented_genus0(sphere):
    _, m = sphere
    closed, chi = S.mesh_topology(m["faces"])
    assert closed, "every undirected edge must lie in exactly two faces, in opposite directions"
    assert chi == 2
    assert S.signed_volume(m["vertices"], m["faces"]) > 0


def test_sphere_vertices_within_one_voxel(sphere):
    """A vertex lies on a voxel edge whose two ends have tsdf of opposite sign.  If those signs are right -- one end inside the
    sphere, one outside -- the vertex is within one edge length s of the sphere.  A sign can only be wrong where the depth
    read at the truncated pixel (a ray up to one pixel away) hits the sphere on the other side of the voxel: at 320x240 a
    pixel covers ~0.014 < s at the sphere, and the fusion of 40 views, each with its projective sdf clamped to tau = 8 s,
    leaves no such voxel next to a crossing."""
    vol, m = sphere
    r = np.linalg.norm(m["vertices"].astype(np.float64), axis=1)
    assert np.abs(r - 1.0).max() < float(vol.s)


def test_constant_colour_comes_back_exactly(sphere):
    _, m = sphere
    assert np.array_equal(np.unique(m["colors"], axis=0), np.array([[0.25, 0.5, 0.125]], np.float32))


def test_fewer_than_threshold_plus_one_observations_give_no_mesh():
    vol = O.Volume(voxel_size=0.05, block_resolution=8)
    d = np.full((H, W), 2.0, np.float32)
    for i in range(3):
        vol.integrate(d, np.zeros((3, H, W), np.float32), FX, FY, CX, CY, np.eye(4, dtype=np.float32))
    assert vol.weight.max() == 3
    assert vol.extract_triangle_mesh(3.0)["faces"].shape == (0, 3)
    vol.integrate(d, np.zeros((3, H, W), np.float32), FX, FY, CX, CY, np.eye(4, dtype=np.float32))
    assert vol.extract_triangle_mesh(3.0)["faces"].shape[0] > 0


def test_invalid_observations_leave_voxels_untouched():
    s, B = 0.25, 8                                  # powers of two: every value below is exact
    vol = O.Volume(voxel_size=s, block_resolution=B)
    d = np.full((H, W), 3.0, np.float32)
    E = np.eye(4, dtype=np.float32)
    vol.integrate(d, np.ones((3, H, W), np.float32), FX, FY, CX, CY, E)
    before = vol.state()
    lin = np.arange(B ** 3)
    vox = O.unpack_keys(before["keys"])[:, None, :] * B + np.stack([lin % B, (lin // B) % B, lin // (B * B)], 1)[None]
    z = vox[..., 2] * s
    # sdf < -tau: behind the plane by more than tau = 2
    assert np.all(before["weight"][z > 5.0] == 0) and np.any(before["weight"][z == 5.0] == 1)
    # out of the image: projections outside [0, W-1] x [0, H-1]
    with np.errstate(invalid="ignore", divide="ignore"):
        u = (FX * (vox[..., 0] * s).astype(np.float32)) / z.astype(np.float32) + CX
    out = (z > 0) & ((u < 0) | (u > W - 1))
    assert out.any() and np.all(before["weight"][out] == 0)
    # depth 0 and depth > depth_max: nothing changes, not even the block table
    for bad in (np.zeros((H, W), np.float32), np.full((H, W), 6.5, np.float32)):
        assert vol.integrate(bad, np.zeros((3, H, W), np.float32), FX, FY, CX, CY, E).size == 0
        after = vol.state()
        for k in before:
            assert np.array_equal(before[k], after[k])
    # depth exactly depth_max touches no block but still updates voxels of blocks other pixels touched
    d2 = d.copy()
    d2[:, : W // 2] = 6.0
    keys = vol.integrate(d2, np.zeros((3, H, W), np.float32), FX, FY, CX, CY, E, depth_max=6.0)
    assert keys.size and vol.last_updates > 0


def test_block_range_is_checked():
    far = np.eye(4, dtype=np.float32)
    far[0, 3] = -1.0e5
    with pytest.raises(O.BlockRangeError):
        O.Volume().integrate(np.full((H, W), 2.0, np.float32), np.zeros((3, H, W), np.float32), FX, FY, CX, CY, far)
    with pytest.raises(O.BlockRangeError):
        O.pack_keys([[1 << 20, 0, 0]])
    k = O.pack_keys([[-(1 << 20), (1 << 20) - 1, -5]])
    assert np.array_equal(O.unpack_keys(k), [[-(1 << 20), (1 << 20) - 1, -5]])
