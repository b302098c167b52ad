"""GPU: the opacity field's level set on a sparse voxel-block lattice (csrc/field_grid.cu, tsdf.cu's field marching cubes,
gof_extract.extract_level_set_grid) against oracle/field_grid_oracle.py and the existing extraction pieces, bit for bit.

* blocks and lattice points equal the oracle on the CPU cases and on 200 k surface Gaussians over 64 views;
* the field values meshed are evaluate_alpha at the oracle's lattice points, minus 0.5;
* faces, vertex edges and their values equal the oracle's marching cubes; vertices are binary_search on those edges, colours
  evaluate_alpha's, normals field_gradient's, normalised;
* on a sphere the mesh is closed, of genus 0, oriented outward, and within a voxel of extract_level_set's mesh of the same lattice
  split into Kuhn tetrahedra;
* two ranks give the one-rank mesh; P = 0, no Gaussian in view, one block, open boundaries, refusals, scratch contents."""
import itertools
import os
import socket
import sys

import numpy as np
import pytest
import torch

import _field_grid_scenes as FS
import _tsdf_scenes as S
import field_grid_oracle as O
import gof_extract
import gof_synth

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, np.float32)).view(np.uint32)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _gpu_blocks(xyz, sc, rot, views, s, B, **kw):
    return gof_extract.field_grid_blocks(_t(xyz), _t(sc), _t(rot), views, s, B, **kw).cpu().numpy()


def _check_blocks_and_points(xyz, sc, rot, views, s, B):
    want = O.blocks(xyz, sc, rot, FS.table(views), s, B)
    got = _gpu_blocks(xyz, sc, rot, views, s, B)
    assert got.dtype == np.int64 and np.array_equal(got, want)
    pts = gof_extract.field_grid_points(torch.from_numpy(got).to(DEV), s, B).cpu().numpy()
    assert np.array_equal(_bits(pts), _bits(O.lattice_points(want, s, B)))
    return want


@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("s,B", [(FS.S_EXACT, FS.B_EXACT), (0.03, 8), (0.1, 1)])
def test_blocks_and_lattice_equal_the_oracle(seed, s, B):
    xyz, sc, rot = FS.gaussians(300, seed)
    keys = _check_blocks_and_points(xyz, sc, rot, FS.views_around(), s, B)
    assert keys.size > 10 and np.any(O.T.unpack_keys(keys) < 0)


def test_blocks_edge_cases():
    xyz, sc, rot = FS.gaussians(60, 4)
    views = FS.views_around()
    _check_blocks_and_points(xyz, np.zeros_like(sc), rot, views, FS.S_EXACT, FS.B_EXACT)          # zero scales
    assert _gpu_blocks(xyz, sc, rot, [FS.view(np.eye(3), (0, 0, -100.0))], 0.25, 4).size == 0     # nothing in view
    z3, z4 = np.zeros((0, 3), np.float32), np.zeros((0, 4), np.float32)
    assert _gpu_blocks(z3, z3, z4, views, 0.25, 4).size == 0                                       # P = 0
    x, s_, r, v = FS.key_limit_case((1 << 20) - 0.5)
    assert _check_blocks_and_points(x, s_, r, v, FS.S_EXACT, FS.B_EXACT).size == 4
    x, s_, r, v = FS.key_limit_case(-(1 << 20) + 0.5, axis=1)
    _check_blocks_and_points(x, s_, r, v, FS.S_EXACT, FS.B_EXACT)
    for bad in ((1 << 20) - 0.125, -(1 << 20) + 0.125):
        x, s_, r, v = FS.key_limit_case(bad)
        with pytest.raises(ValueError, match="2\\^20"):
            _gpu_blocks(x, s_, r, v, FS.S_EXACT, FS.B_EXACT)


def test_blocks_and_lattice_at_scale():
    """200 k surface Gaussians over 64 views: many Gaussians per block, so the sort and the run detection do real work."""
    gs = gof_synth.make_surface_gaussians(200_000, seed=21)
    views = gof_synth.make_surface_views(320, 240, 64)
    xyz, sc, rot = (gs[k].numpy() for k in ("means3D", "scales", "rotations"))
    keys = _check_blocks_and_points(xyz, sc, rot, views, 0.01, 8)
    assert keys.size > 3000


# ---- the whole extraction on a sphere of surface Gaussians ---------------------------------------------------------------
def _sphere(P=20_000, n_views=24, seed=3):
    gs = gof_synth.make_surface_gaussians(P, seed=seed)
    g = {k: (v.to(DEV).contiguous() if isinstance(v, torch.Tensor) else v) for k, v in gs.items()}
    views = gof_synth.make_surface_views(320, 240, n_views)
    ci = gof_extract.CachedIntegrator(g["means3D"], g["opacities"], g["scales"], g["rotations"], g["shs"], 0,
                                      lambda c: gof_synth.raster_settings(c, 0, DEV))
    return g, views, ci


S_SPHERE, B_SPHERE = 0.04, 8


def _run(g, views, ci, **kw):
    """extract_level_set_grid, with the keys and field values it meshes captured."""
    seen = {}
    mc = gof_extract.field_grid_marching_cubes

    def spy(keys, values, voxel_size, block_resolution=8):
        seen["keys"], seen["values"] = keys.clone(), values.clone()
        out = mc(keys, values, voxel_size, block_resolution)
        seen["mc"] = tuple(t.clone() for t in out)
        return out
    mp = pytest.MonkeyPatch()
    mp.setattr(gof_extract, "field_grid_marching_cubes", spy)
    try:
        out = gof_extract.extract_level_set_grid(g["means3D"], g["scales"], g["rotations"], views, ci, S_SPHERE, B_SPHERE, **kw)
    finally:
        mp.undo()
    return out, seen


@pytest.fixture(scope="module")
def sphere():
    g, views, ci = _sphere()
    tm = {}
    out, seen = _run(g, views, ci, return_color=True, return_normals=True, timings=tm)
    return g, views, ci, out, seen, tm


def test_field_values_are_evaluate_alpha_at_the_oracle_points(sphere):
    g, views, ci, out, seen, tm = sphere
    keys = seen["keys"].cpu().numpy()
    want = O.blocks(*(g[k].cpu().numpy() for k in ("means3D", "scales", "rotations")), FS.table(views), S_SPHERE, B_SPHERE)
    assert np.array_equal(keys, want)
    pts = _t(O.lattice_points(want, S_SPHERE, B_SPHERE))
    alpha = gof_extract.evaluate_alpha(pts, views, ci)
    assert torch.equal(seen["values"], alpha - 0.5)
    assert float((alpha < 0.5).float().mean()) > 0.01 and float((alpha > 0.5).float().mean()) > 0.01
    assert set(tm) >= {"blocks_s", "lattice_s", "evaluate_alpha_lattice_s", "marching_cubes_s", "binary_search_s", "field_gradient_s"}


def test_marching_cubes_equal_the_oracle(sphere):
    _g, _v, _ci, out, seen, _tm = sphere
    ep, ev, faces = (t.cpu().numpy() for t in seen["mc"])
    ref = O.marching_cubes(seen["keys"].cpu().numpy(), seen["values"].cpu().numpy(), S_SPHERE, B_SPHERE)
    assert faces.shape[0] > 1000
    assert np.array_equal(faces, ref["faces"])
    assert np.array_equal(_bits(ep), _bits(ref["edge_points"]))
    assert np.array_equal(_bits(ev), _bits(ref["edge_values"]))
    assert torch.equal(out["faces"].cpu(), torch.from_numpy(faces))


def test_bisection_colours_and_normals(sphere):
    g, views, ci, out, seen, _tm = sphere
    ep, ev, _f = seen["mc"]
    verts = gof_extract.binary_search(ep, ev.unsqueeze(-1), lambda p: gof_extract.evaluate_alpha(p, views, ci), n_steps=8)
    assert torch.equal(out["vertices"], verts)
    _a, colors = gof_extract.evaluate_alpha(verts, views, ci, return_color=True)
    assert torch.equal(out["colors"], colors)
    _a, grad = gof_extract.field_gradient(verts, views, ci)
    norm = grad.norm(dim=1, keepdim=True)
    want = torch.where(norm > 0, grad / torch.where(norm > 0, norm, torch.ones_like(norm)), torch.zeros_like(grad))
    assert torch.equal(out["normals"], want)
    # colours and normals alone: the same arrays
    plain, _ = _run(g, views, ci, return_color=True)
    assert torch.equal(plain["vertices"], out["vertices"]) and torch.equal(plain["colors"], colors) and "normals" not in plain
    bare, _ = _run(g, views, ci)
    assert bare["colors"] is None and torch.equal(bare["faces"], out["faces"])


def test_sphere_mesh_is_closed_genus0_and_outward(sphere):
    _g, _v, _ci, out, _seen, _tm = sphere
    v, f = out["vertices"].cpu().numpy(), out["faces"].cpu().numpy()
    closed, chi = S.mesh_topology(f)
    r = np.linalg.norm(v.astype(np.float64), axis=1)
    print(f"[field grid sphere] V={v.shape[0]} F={f.shape[0]} closed={closed} chi={chi} |r-1| max={np.abs(r - 1).max():.4f}")
    assert closed and chi == 2
    assert S.signed_volume(v, f) > 0
    a, b, c = v[f[:, 0]].astype(np.float64), v[f[:, 1]].astype(np.float64), v[f[:, 2]].astype(np.float64)
    n = np.cross(b - a, c - a)
    assert np.mean((n * (a + b + c)).sum(1) > 0) > 0.99
    assert np.abs(r - 1).max() < 2 * S_SPHERE
    n_out = out["normals"].cpu().numpy()
    ok = np.linalg.norm(n_out, axis=1) > 0
    assert ok.mean() > 0.9 and np.mean((n_out[ok] * v[ok]).sum(1) > 0) > 0.99


def _kuhn_tets(keys, B):
    """Six tetrahedra per cube whose eight corners are listed, split along the cube's main diagonal (Freudenthal / Kuhn)."""
    G = O.voxels(keys, B)
    idx = np.stack([O._lookup(keys, B, G + O.T.CORNER_OFF[c]) for c in range(8)], 1)
    idx = idx[np.all(idx >= 0, axis=1)]
    tets = []
    for p in itertools.permutations(range(3)):
        c1 = 1 << p[0]
        c2 = c1 | (1 << p[1])
        tets.append(idx[:, [0, c1, c2, 7]])
    return np.concatenate(tets)


def test_agrees_with_the_tetrahedra_path_on_the_same_lattice(sphere):
    from scipy.spatial import cKDTree
    _g, views, ci, out, seen, _tm = sphere
    keys = seen["keys"].cpu().numpy()
    pts = _t(O.lattice_points(keys, S_SPHERE, B_SPHERE))
    tets = _t(_kuhn_tets(keys, B_SPHERE))
    tet = gof_extract.extract_level_set(pts, torch.full((pts.shape[0], 1), 0.05, device=DEV), tets, views, ci)
    a, b = out["vertices"].cpu().numpy().astype(np.float64), tet["vertices"].cpu().numpy().astype(np.float64)
    d_ab, _ = cKDTree(b).query(a)
    d_ba, _ = cKDTree(a).query(b)
    print(f"[field grid vs tets] {a.shape[0]} / {b.shape[0]} vertices; max distance {d_ab.max():.5f} / {d_ba.max():.5f}, "
          f"voxel {S_SPHERE}")
    lim = S_SPHERE * np.sqrt(3) * (1 + 1e-5)
    assert d_ab.max() <= lim and d_ba.max() <= lim
    assert np.median(d_ab) < 0.25 * S_SPHERE


# ---- sharding ------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _dist_worker(rank, world, port, backend, q):
    here = os.path.dirname(os.path.abspath(__file__))
    for p in (here, os.path.join(here, "..", "gaussian-opacity-fields_b200"), os.path.join(here, "..", "oracle")):
        sys.path.insert(0, p)
    import torch.distributed as dist
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    kw = dict(device_id=dev) if backend == "nccl" else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    global DEV
    DEV = dev
    g, views, ci = _sphere(P=8_000, n_views=9)
    out = gof_extract.extract_level_set_grid(g["means3D"], g["scales"], g["rotations"], views, ci, 0.06, 8, return_color=True,
                                             group=dist.group.WORLD)
    q.put((rank, {k: v.cpu().numpy() for k, v in out.items()}))
    dist.barrier()
    dist.destroy_process_group()


def test_two_ranks_equal_one():
    """Over NCCL with a GPU per rank where there are two, otherwise over gloo with both ranks on one GPU."""
    import torch.multiprocessing as mp
    backend = "nccl" if torch.cuda.device_count() >= 2 else "gloo"
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_dist_worker, args=(r, world, port, backend, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=600) for _ in range(world)], key=lambda x: x[0])
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    g, views, ci = _sphere(P=8_000, n_views=9)
    one = gof_extract.extract_level_set_grid(g["means3D"], g["scales"], g["rotations"], views, ci, 0.06, 8, return_color=True)
    assert one["faces"].shape[0] > 500
    for _rank, r in res:
        for k in ("vertices", "faces", "colors"):
            assert np.array_equal(r[k], one[k].cpu().numpy()), k


# ---- edges and refusals --------------------------------------------------------------------------------------------------
def _sdf_values(keys, s, B, center=(0.3, 0.4, 0.2), radius=0.6, seed=0, noise=0.02):
    pts = O.lattice_points(keys, s, B).astype(np.float64)
    rng = np.random.default_rng(seed)
    return (np.linalg.norm(pts - center, axis=1) - radius + noise * rng.standard_normal(pts.shape[0])).astype(np.float32)


def _check_mc(keys, s, B, values):
    ep, ev, f = gof_extract.field_grid_marching_cubes(_t(keys), _t(values), s, B)
    ref = O.marching_cubes(keys, values, s, B)
    assert np.array_equal(f.cpu().numpy(), ref["faces"])
    assert np.array_equal(_bits(ep.cpu().numpy()), _bits(ref["edge_points"]))
    assert np.array_equal(_bits(ev.cpu().numpy()), _bits(ref["edge_values"]))
    return ref


def test_one_block_and_open_boundaries():
    s, B = 0.125, 8
    one = O.T.pack_keys([[0, 0, 0]])
    ref = _check_mc(one, s, B, _sdf_values(one, s, B, center=(0.5, 0.5, 0.5), radius=0.3, noise=0.0))
    closed, chi = S.mesh_topology(ref["faces"])
    assert ref["faces"].shape[0] > 50 and closed and chi == 2        # the sphere lies inside the block's own cubes
    # blocks with missing +1 neighbours: an open surface, cut where cubes are incomplete, with no crack inside
    keys = np.sort(O.T.pack_keys([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [-1, -1, 0], [-1, 0, 0], [2, 2, 2]]))
    ref = _check_mc(keys, s, B, _sdf_values(keys, s, B, center=(0.9, 0.9, 0.9), radius=0.7))
    f = ref["faces"]
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), axis=1)
    _u, cnt = np.unique(e, axis=0, return_counts=True)
    assert cnt.max() == 2 and (cnt == 1).any()
    # every boundary edge (one face) lies on a cube face with a meshed cube on one side only: the surface ends where the lattice
    # does, and nowhere inside it
    uniq = _u[cnt == 1]
    G = np.rint(ref["edge_points"].astype(np.float64) / s).astype(np.int64)          # [V, 2, 3] lattice coordinates
    for v1, v2 in uniq:
        ends = np.concatenate([G[v1], G[v2]])                                          # four lattice points on one cube face
        d = [a for a in range(3) if np.all(ends[:, a] == ends[0, a])]
        assert len(d) == 1, ends
        corner = ends.min(0)
        sides = []
        for off in (-1, 0):
            c = corner.copy()
            c[d[0]] += off
            idx = np.stack([O._lookup(keys, B, (c + O.T.CORNER_OFF[k])[None])[0] for k in range(8)])
            sides.append(bool(np.all(idx >= 0)))
        assert sides.count(True) == 1, (ends, sides)
    for B1 in (1, 2):
        k1 = np.sort(O.T.pack_keys([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 1]]))
        _check_mc(k1, 0.2, B1, _sdf_values(k1, 0.2, B1, center=(0.3, 0.3, 0.3), radius=0.35, seed=B1))


def test_empty_inputs():
    g, views, ci = _sphere(P=2_000, n_views=4)
    z = torch.zeros((0, 3), device=DEV)
    out = gof_extract.extract_level_set_grid(z, z, torch.zeros((0, 4), device=DEV), views, ci, 0.05, return_color=True,
                                             return_normals=True)
    assert out["vertices"].shape == (0, 3) and out["faces"].shape == (0, 3) and out["faces"].dtype == torch.int64
    assert out["colors"].shape == (0, 3) and out["normals"].shape == (0, 3)
    away = [FS.view(np.eye(3), (0, 0, -100.0))]
    keys = gof_extract.field_grid_blocks(g["means3D"], g["scales"], g["rotations"], away, 0.05)
    assert keys.numel() == 0
    ep, ev, f = gof_extract.field_grid_marching_cubes(keys, torch.zeros(0, device=DEV), 0.05)
    assert ep.shape == (0, 2, 3) and ev.shape == (0, 2) and f.shape == (0, 3)


def test_refusals():
    g, views, ci = _sphere(P=2_000, n_views=4)
    x, s, r = g["means3D"], g["scales"], g["rotations"]
    for kw, msg in ((dict(voxel_size=0.0), "voxel_size"), (dict(voxel_size=-1.0), "voxel_size"),
                    (dict(voxel_size=0.05, block_resolution=0), "1..64"), (dict(voxel_size=0.05, block_resolution=65), "1..64")):
        with pytest.raises(ValueError, match=msg):
            gof_extract.extract_level_set_grid(x, s, r, views, ci, **kw)
    one = lambda sc: (torch.zeros((1, 3), device=DEV), torch.full((1, 3), sc, device=DEV), torch.tensor([[1.0, 0, 0, 0]], device=DEV))  # noqa: E731
    with pytest.raises(ValueError, match="2\\^30"):
        gof_extract.extract_level_set_grid(*one(1.0), views, ci, 0.001, 1)             # (6 / 0.001)^3 blocks
    with pytest.raises(ValueError, match="2\\^31"):
        gof_extract.extract_level_set_grid(*one(3.0), views, ci, 0.01, 64)             # 29^3 blocks of 64^3 voxels
    x0, s0, r0, v0 = FS.key_limit_case((1 << 20) - 0.125)
    with pytest.raises(ValueError, match="2\\^20"):
        gof_extract.extract_level_set_grid(_t(x0), _t(s0), _t(r0), v0, ci, FS.S_EXACT, FS.B_EXACT)
    with pytest.raises(RuntimeError):
        gof_extract.field_grid_blocks(x.cpu(), s.cpu(), r.cpu(), views, 0.05)
    # the lattice's own inputs: int64 CUDA keys, float32 values on the keys' device, refused before any launch
    keys = gof_extract.field_grid_blocks(x, s, r, views, 0.05)
    vals = torch.zeros(keys.numel() * 512, device=DEV)
    for bad in (keys.int(), keys.float(), keys.reshape(-1, 1)):
        with pytest.raises(ValueError, match="int64"):
            gof_extract.field_grid_points(bad, 0.05)
        with pytest.raises(ValueError, match="int64"):
            gof_extract.field_grid_marching_cubes(bad, vals, 0.05)
    with pytest.raises(RuntimeError, match="CUDA"):
        gof_extract.field_grid_marching_cubes(keys, vals.cpu(), 0.05)
    with pytest.raises(ValueError, match="float32"):
        gof_extract.field_grid_marching_cubes(keys, vals.double(), 0.05)
    with pytest.raises(RuntimeError, match="CUDA"):
        gof_extract.field_grid_points(keys.cpu(), 0.05)


class _GuardedScratch:
    """Stand-in for _C._Scratch: every buffer is pre-filled with `fill` and followed by a guard band of known bytes."""
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
    """Blocks, lattice and marching cubes stay inside their scratch layouts and depend on no scratch contents they did not write:
    scratch pre-filled with 0x00 and with 0xFF gives the same mesh, with every guard band intact."""
    from diff_gaussian_rasterization import _C
    g, views, ci = _sphere(P=6_000, n_views=6)
    results = []
    for fill in (0x00, 0xFF):
        _GuardedScratch.made = []
        monkeypatch.setattr(_C, "_Scratch", lambda device, role="", slack=1.0, f=fill: _GuardedScratch(device, role, slack, f))
        keys = gof_extract.field_grid_blocks(g["means3D"], g["scales"], g["rotations"], views, 0.05, 8)
        vals = _t(_sdf_values(keys.cpu().numpy(), 0.05, 8, center=(0, 0, 0), radius=1.0))
        ep, ev, f = gof_extract.field_grid_marching_cubes(keys, vals, 0.05, 8)
        torch.cuda.synchronize()
        monkeypatch.undo()
        assert len(_GuardedScratch.made) >= 3
        for buf, n in _GuardedScratch.made:
            assert bool((buf[n:] == _GuardedScratch.CANARY).all()), f"write past the end of a {n}-byte scratch buffer"
        results.append([t.cpu().numpy() for t in (keys, ep, ev, f)])
    for a, b in zip(*results):
        assert np.array_equal(a, b)
    assert results[0][3].shape[0] > 1000
