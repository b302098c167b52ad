"""GPU: TSDF fusion and marching-cubes extraction (csrc/tsdf.cu via gof_tsdf) against the float32 oracle, bit for bit."""
import numpy as np
import pytest
import torch

import _tsdf_scenes as S
import gof_synth
import tsdf_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _bits(a):
    a = np.ascontiguousarray(np.asarray(a, np.float32))
    return a.view(np.uint32)


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _gpu_volume(**kw):
    import gof_tsdf
    return gof_tsdf.TSDFVolume(device=DEV, **kw)


def _assert_state_equal(vol, ref):
    st = {k: v.cpu().numpy() for k, v in vol.state().items()}
    rs = ref.state()
    assert np.array_equal(st["keys"], rs["keys"])
    for k in ("tsdf", "weight", "color"):
        assert np.array_equal(_bits(st[k]), _bits(rs[k])), k


def _assert_mesh_equal(mesh, ref_mesh):
    m = {k: v.cpu().numpy() for k, v in mesh.items()}
    assert m["faces"].dtype == np.int64 and m["vertices"].dtype == np.float32 and m["colors"].dtype == np.float32
    assert m["vertices"].shape == ref_mesh["vertices"].shape and m["faces"].shape == ref_mesh["faces"].shape
    assert np.array_equal(m["faces"], ref_mesh["faces"])
    assert np.array_equal(_bits(m["vertices"]), _bits(ref_mesh["vertices"]))
    assert np.array_equal(_bits(m["colors"]), _bits(ref_mesh["colors"]))


def _look(R_rows, t):
    E = np.eye(4, dtype=np.float32)
    E[:3, :3] = np.asarray(R_rows, np.float32)
    E[:3, 3] = np.asarray(t, np.float32)
    return E


W_EC, H_EC = 64, 48
K_EC = (np.float32(40.0), np.float32(40.0), np.float32(31.5), np.float32(23.5))
# fx = W - 1, fy = H - 1: a voxel with x / z = 0.5 projects to u = 63 * 0.5 + 31.5 = W - 1 exactly (y / z = 0.5: v = H - 1)
K_LAST = (np.float32(63.0), np.float32(47.0), np.float32(31.5), np.float32(23.5))
# voxels of the K_LAST view that are seen only through the inclusive bounds u <= W-1, v <= H-1: (x, y, z) with z = 3
LAST_ROW_COL_VOXELS = ((1.5, 0.0, 3.0), (0.0, 1.5, 3.0), (1.5, 1.5, 3.0))


def _edge_case_views(seed=0):
    """(depth, colour, extrinsic, intrinsics) of views on a coarse power-of-two grid (s = 0.25, tau = 2) where the edge cases
    are hit exactly:
    view 0: identity camera facing a plane at depth 3 (voxels at z = 5 have sdf exactly -tau), with pixels at exactly
            depth_max = 6, beyond it and with no depth; x, y < 0 give negative block coordinates;
    view 1: a camera inside the volume fused so far (at z = 2.5, turned to face -z);
    view 2: identity camera with fx = W - 1, fy = H - 1 facing a plane at depth 3: the voxels LAST_ROW_COL_VOXELS project
            exactly onto u = W - 1 and / or v = H - 1 and read valid depth in the last column and row;
    views 3..8: small random rotations and offsets of random depth maps (noisy surfaces)."""
    rng = np.random.default_rng(seed)
    views = []
    d0 = np.full((H_EC, W_EC), 3.0, np.float32)
    d0[5:9, 10:20] = 6.0
    d0[20:24, 30:40] = 7.0
    d0[30:34, 0:12] = 0.0
    c0 = rng.random((3, H_EC, W_EC), dtype=np.float32)
    views.append((d0, c0, _look(np.eye(3), (0, 0, 0)), K_EC))
    d1 = (1.5 + rng.random((H_EC, W_EC), dtype=np.float32)).astype(np.float32)
    views.append((d1, rng.random((3, H_EC, W_EC), dtype=np.float32), _look([[1, 0, 0], [0, -1, 0], [0, 0, -1]], (0, 0, 2.5)), K_EC))
    d2 = np.full((H_EC, W_EC), 3.0, np.float32)
    d2[:, W_EC - 1] = 2.75        # a different depth in the last column and row: the value read there shows in the tsdf
    d2[H_EC - 1, :] = 2.75
    views.append((d2, rng.random((3, H_EC, W_EC), dtype=np.float32), _look(np.eye(3), (0, 0, 0)), K_LAST))
    for _ in range(6):
        a = rng.normal(0, 0.08, 3)
        cx_, sx_ = np.cos(a), np.sin(a)
        Rx = np.array([[1, 0, 0], [0, cx_[0], -sx_[0]], [0, sx_[0], cx_[0]]])
        Ry = np.array([[cx_[1], 0, sx_[1]], [0, 1, 0], [-sx_[1], 0, cx_[1]]])
        Rz = np.array([[cx_[2], -sx_[2], 0], [sx_[2], cx_[2], 0], [0, 0, 1]])
        d = (3.0 + 0.6 * rng.random((H_EC, W_EC))).astype(np.float32)
        d[rng.random((H_EC, W_EC)) < 0.05] = 0
        views.append((d, rng.random((3, H_EC, W_EC), dtype=np.float32), _look(Rx @ Ry @ Rz, rng.normal(0, 0.3, 3)), K_EC))
    return views


def _voxel(st, p, s, B, field):
    """Value of `field` at the voxel at world position p (a multiple of s) in a state() dict; 0 if its block is absent."""
    g = [int(round(c / s)) for c in p]
    b = [c // B for c in g]
    k = int(O.pack_keys([b])[0])
    row = int(np.searchsorted(st["keys"], k))
    if row == st["keys"].size or st["keys"][row] != k:
        return 0.0
    lin = (g[0] - B * b[0]) + B * (g[1] - B * b[1]) + B * B * (g[2] - B * b[2])
    return st[field][row, lin]


def test_integrate_parity_edge_cases():
    kw = dict(voxel_size=0.25, block_resolution=8)
    ref = O.Volume(**kw)
    vol = _gpu_volume(block_count=4, **kw)
    views = _edge_case_views()
    for i, (d, c, E, (fx, fy, cx, cy)) in enumerate(views):
        rk = ref.integrate(d, c, fx, fy, cx, cy, E)
        gk = vol.integrate(_cuda(d), _cuda(c), fx, fy, cx, cy, E).cpu().numpy()
        assert np.array_equal(gk, rk), i
        if i + 1 in (1, 2, 8):
            _assert_state_equal(vol, ref)
        if i == 2:
            # the voxels that only the inclusive bounds u <= W-1 / v <= H-1 admit were updated by this view
            st = {k: v.cpu().numpy() for k, v in vol.state().items()}
            for p in LAST_ROW_COL_VOXELS:
                u = (fx * np.float32(p[0])) / np.float32(p[2]) + cx
                v = (fy * np.float32(p[1])) / np.float32(p[2]) + cy
                assert u == W_EC - 1 or v == H_EC - 1
                assert _voxel(st, p, 0.25, 8, "weight") == _voxel(before, p, 0.25, 8, "weight") + 1, p
        before = {k: v.cpu().numpy() for k, v in vol.state().items()}
    _assert_state_equal(vol, ref)
    assert np.any(O.unpack_keys(ref.keys) < 0)
    _assert_mesh_equal(vol.extract_triangle_mesh(), ref.extract_triangle_mesh())
    _assert_mesh_equal(vol.extract_triangle_mesh(1.0), ref.extract_triangle_mesh(1.0))


def test_exact_edge_values():
    """On a power-of-two grid: a voxel with sdf exactly -tau is updated (to tsdf -1), the next one behind it is not."""
    kw = dict(voxel_size=0.25, block_resolution=8)
    fx, fy, cx, cy = K_EC
    d = np.full((H_EC, W_EC), 3.0, np.float32)
    vol = _gpu_volume(**kw)
    vol.integrate(_cuda(d), _cuda(np.ones((3, H_EC, W_EC), np.float32)), fx, fy, cx, cy, np.eye(4, dtype=np.float32))
    st = {k: v.cpu().numpy() for k, v in vol.state().items()}
    ref = O.Volume(**kw)
    ref.integrate(d, np.ones((3, H_EC, W_EC), np.float32), fx, fy, cx, cy, np.eye(4, dtype=np.float32))
    B = 8
    lin = np.arange(B ** 3)
    z = (O.unpack_keys(st["keys"])[:, 2:3] * B + lin[None] // (B * B)) * 0.25          # voxel z of every voxel
    w = st["weight"]
    assert np.any((z == 5.0) & (w == 1)), "sdf == -tau must update"
    assert not np.any((z > 5.0) & (w > 0)), "sdf < -tau must not update"
    assert np.all(st["tsdf"][(z == 5.0) & (w == 1)] == -1.0)
    _assert_state_equal(vol, ref)


def test_mesh_parity_sphere():
    kw = dict(voxel_size=0.02, block_resolution=8)
    ref = O.Volume(**kw)
    vol = _gpu_volume(**kw)
    for v in gof_synth.make_surface_views(320, 240, 40):
        fx, fy, cx, cy, E = S.view_params(v)
        d, c = S.sphere_depth(v), S.sphere_color(v, (0.25, 0.5, 0.125))
        ref.integrate(d, c, fx, fy, cx, cy, E)
        vol.integrate(_cuda(d), _cuda(c), fx, fy, cx, cy, E)
    _assert_state_equal(vol, ref)
    mesh = vol.extract_triangle_mesh()
    rm = ref.extract_triangle_mesh()
    _assert_mesh_equal(mesh, rm)
    closed, chi = S.mesh_topology(rm["faces"])
    assert closed and chi == 2


def test_mesh_parity_noisy():
    """Fused from noisy random depth maps: many ambiguous cubes."""
    kw = dict(voxel_size=0.05, block_resolution=8)
    rng = np.random.default_rng(7)
    ref = O.Volume(**kw)
    vol = _gpu_volume(**kw)
    fx, fy, cx, cy = K_EC
    for i in range(10):
        d = (3.0 + 0.15 * rng.standard_normal((H_EC, W_EC))).astype(np.float32)
        c = rng.random((3, H_EC, W_EC), dtype=np.float32)
        E = _look(np.eye(3), rng.normal(0, 0.05, 3))
        ref.integrate(d, c, fx, fy, cx, cy, E)
        vol.integrate(_cuda(d), _cuda(c), fx, fy, cx, cy, E)
    _assert_state_equal(vol, ref)
    rm = ref.extract_triangle_mesh()
    assert rm["faces"].shape[0] > 1000
    _assert_mesh_equal(vol.extract_triangle_mesh(), rm)


def test_growth_from_one_block():
    views = _edge_case_views(seed=3)
    out = []
    for cap in (1, 100000):
        vol = _gpu_volume(voxel_size=0.25, block_resolution=8, block_count=cap)
        for d, c, E, (fx, fy, cx, cy) in views:
            vol.integrate(_cuda(d), _cuda(c), fx, fy, cx, cy, E)
        st = {k: v.cpu().numpy() for k, v in vol.state().items()}
        out.append((st, {k: v.cpu().numpy() for k, v in vol.extract_triangle_mesh().items()}))
    for k in out[0][0]:
        assert np.array_equal(out[0][0][k], out[1][0][k]), k
    for k in out[0][1]:
        assert np.array_equal(out[0][1][k], out[1][1][k]), k


def test_empty_inputs():
    fx, fy, cx, cy = K_EC
    vol = _gpu_volume(voxel_size=0.25, block_resolution=8)
    keys = vol.integrate(torch.zeros(H_EC, W_EC, device=DEV), torch.zeros(3, H_EC, W_EC, device=DEV), fx, fy, cx, cy, np.eye(4))
    assert keys.numel() == 0 and vol.num_blocks == 0
    m = vol.extract_triangle_mesh()
    assert tuple(m["vertices"].shape) == (0, 3) and m["vertices"].dtype == torch.float32
    assert tuple(m["colors"].shape) == (0, 3) and m["colors"].dtype == torch.float32
    assert tuple(m["faces"].shape) == (0, 3) and m["faces"].dtype == torch.int64
    d, c, E, _ = _edge_case_views()[0]
    vol.integrate(_cuda(d), _cuda(c), fx, fy, cx, cy, E)
    assert vol.num_blocks > 0
    m = vol.extract_triangle_mesh(weight_threshold=1e9)
    assert m["vertices"].shape[0] == 0 and m["faces"].shape[0] == 0


def test_rejection():
    fx, fy, cx, cy = K_EC
    vol = _gpu_volume(voxel_size=0.002, block_resolution=16)
    d = torch.full((H_EC, W_EC), 3.0, device=DEV)
    c = torch.zeros(3, H_EC, W_EC, device=DEV)
    with pytest.raises(RuntimeError):
        vol.integrate(d.cpu(), c, fx, fy, cx, cy, np.eye(4))
    with pytest.raises(RuntimeError):
        vol.integrate(d, c.cpu(), fx, fy, cx, cy, np.eye(4))
    with pytest.raises(ValueError):
        vol.integrate(d, torch.zeros(3, H_EC, W_EC + 1, device=DEV), fx, fy, cx, cy, np.eye(4))
    with pytest.raises(ValueError):
        vol.integrate(d.double(), c, fx, fy, cx, cy, np.eye(4))
    with pytest.raises(ValueError):
        vol.integrate(d, c, fx, fy, cx, cy, np.eye(3))
    with pytest.raises(RuntimeError):
        __import__("gof_tsdf").TSDFVolume(device="cpu")
    far = np.eye(4, dtype=np.float32)
    far[0, 3] = -1.0e5            # pw.x ~ 1e5 -> block x ~ 3e6 >= 2^20
    with pytest.raises(RuntimeError, match="2\\^20"):
        vol.integrate(d, c, fx, fy, cx, cy, far)
    with pytest.raises(O.BlockRangeError):
        O.Volume().integrate(d.cpu().numpy(), c.cpu().numpy(), fx, fy, cx, cy, far)
    assert vol.num_blocks == 0


def test_end_to_end_surface_gaussians(tmp_path):
    import gof_tsdf
    gs = gof_synth.make_surface_gaussians(100_000, seed=11)
    g = {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in gs.items()}
    views = gof_synth.make_surface_views(320, 240, 40)
    s = 0.01
    render = gof_tsdf.make_render_fn(g["means3D"], g["opacities"], g["scales"], g["rotations"], g["shs"], g["sh_degree"],
                                      lambda v: gof_synth.raster_settings(v, g["sh_degree"], DEV))
    meshes = [gof_tsdf.tsdf_fusion(views, render, voxel_size=s, block_resolution=8) for _ in range(2)]
    for k in meshes[0]:
        assert torch.equal(meshes[0][k], meshes[1][k]), k
    m = {k: v.cpu().numpy() for k, v in meshes[0].items()}
    closed, chi = S.mesh_topology(m["faces"])
    vol = S.signed_volume(m["vertices"], m["faces"])
    r = np.linalg.norm(m["vertices"].astype(np.float64), axis=1)
    print(f"[tsdf e2e] V={len(r)} F={len(m['faces'])} closed={closed} chi={chi} volume={vol:.4f} |r-1| max={np.abs(r - 1).max():.4f}")
    assert closed
    assert vol > 0 and abs(vol - 4.0 / 3.0 * np.pi) < 0.05 * 4.0 / 3.0 * np.pi
    # the splats are flat (normal extent 0.05 sigma, sigma ~ 0.011) and opaque, so the rendered median depth lies on the sphere
    # up to the splat thickness and the pixel footprint (~0.014 at the far side); a vertex lies within one voxel of a sign
    # change of the fused tsdf: three voxels bound both
    assert np.abs(r - 1).max() < 3 * s
    path = tmp_path / "tsdf.ply"
    gof_tsdf.write_ply(str(path), meshes[0])
    back = gof_tsdf.read_ply(str(path))
    assert np.array_equal(back["vertices"], m["vertices"]) and np.array_equal(back["faces"], m["faces"])
    assert np.array_equal(back["colors_u8"], np.clip(m["colors"] * np.float32(255), 0, 255).astype(np.uint8))


class _GuardedScratch:
    """Stand-in for _C._Scratch: every buffer the library asks for is pre-filled with `fill` and followed by a guard band of
    known bytes, so writes past a scratch layout's end and results that depend on scratch the library never wrote show up."""
    GUARD = 64 * 1024
    CANARY = 0x5A
    made = []

    def __init__(self, device, role="", slack=1.0, fill=0):
        holder = [torch.empty(0, dtype=torch.uint8, device=device)]
        self._holder = holder

        def alloc(_user, nbytes):
            buf = torch.full((int(nbytes) + self.GUARD,), fill, dtype=torch.uint8, device=device)
            buf[int(nbytes):] = self.CANARY
            holder[0] = buf
            _GuardedScratch.made.append((buf, int(nbytes)))
            return buf.data_ptr()
        self.cb = __import__("diff_gaussian_rasterization")._C._ALLOC_FN(alloc)

    @property
    def tensor(self):
        return self._holder[0]


def test_scratch_bounds_and_initialisation(monkeypatch):
    """Every scratch buffer of touch, activate and extraction stays inside its layout, no result depends on scratch contents
    the library did not write (scratch pre-filled with 0x00 and with 0xFF gives identical results, equal to the oracle),
    and pool slots beyond the table stay zero."""
    import gof_tsdf
    views = _edge_case_views(seed=5)
    ref = O.Volume(voxel_size=0.25, block_resolution=8)
    for d, c, E, (fx, fy, cx, cy) in views:
        ref.integrate(d, c, fx, fy, cx, cy, E)
    results = []
    for fill in (0x00, 0xFF):
        _GuardedScratch.made = []
        monkeypatch.setattr(gof_tsdf._C, "_Scratch", lambda device, role="", slack=1.0, f=fill: _GuardedScratch(device, role, slack, f))
        vol = _gpu_volume(voxel_size=0.25, block_resolution=8, block_count=3)
        for d, c, E, (fx, fy, cx, cy) in views:
            vol.integrate(_cuda(d), _cuda(c), fx, fy, cx, cy, E)
        mesh = vol.extract_triangle_mesh()
        torch.cuda.synchronize()
        assert len(_GuardedScratch.made) >= 2 * len(views)
        for buf, n in _GuardedScratch.made:
            assert bool((buf[n:] == _GuardedScratch.CANARY).all()), f"write past the end of a {n}-byte scratch buffer"
        assert not bool(vol.pool[vol.num_blocks:].any()), "pool slots beyond the table were written"
        _assert_state_equal(vol, ref)
        results.append({k: v.cpu().numpy() for k, v in mesh.items()})
        monkeypatch.undo()
    _assert_mesh_equal({k: torch.from_numpy(v) for k, v in results[0].items()}, ref.extract_triangle_mesh())
    for k in results[0]:
        assert np.array_equal(results[0][k], results[1][k]), k
