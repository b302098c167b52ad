"""CPU: extraction-side host logic (gof_extract): view-sharded evaluate_alpha over gloo (world 2) equals the serial
loop of extract_mesh.py:17-34 including the colour arg-min rule; the bisection converges on an analytic level set."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import gof_extract


def _fake_integrate(points, view):
    g = torch.Generator().manual_seed(1000 + int(view))
    a = torch.rand(points.shape[0], generator=g)
    a = torch.where(a > 0.7, torch.ones_like(a), a)          # many points unseen by a view keep alpha 1
    a[::7] = 0.25                                            # exact ties between views
    c = torch.rand(points.shape[0], 3, generator=g)
    return a, c


def _serial(points, views, return_color):
    final_alpha = torch.ones(points.shape[0])
    final_color = torch.ones(points.shape[0], 3)
    for v in views:
        a, c = _fake_integrate(points, v)
        if return_color:
            final_color = torch.where((a < final_alpha).reshape(-1, 1), c, final_color)
        final_alpha = torch.min(final_alpha, a)
    return (1 - final_alpha, final_color) if return_color else 1 - final_alpha


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    pts = torch.zeros(500, 3)
    alpha, color = gof_extract.evaluate_alpha(pts, range(9), _fake_integrate, return_color=True)
    alpha2 = gof_extract.evaluate_alpha(pts, range(9), _fake_integrate)
    q.put((rank, alpha.numpy().copy(), color.numpy().copy(), alpha2.numpy().copy()))
    dist.destroy_process_group()


def test_view_sharded_evaluate_alpha_world2():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(2)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    want_a, want_c = _serial(torch.zeros(500, 3), range(9), True)
    for _, a, c, a2 in res:
        assert torch.equal(torch.from_numpy(a), want_a)
        assert torch.equal(torch.from_numpy(a2), want_a)
        assert torch.equal(torch.from_numpy(c), want_c)


def test_single_process_matches_serial():
    pts = torch.zeros(300, 3)
    a, c = gof_extract.evaluate_alpha(pts, range(5), _fake_integrate, return_color=True)
    wa, wc = _serial(pts, range(5), True)
    assert torch.equal(a, wa) and torch.equal(c, wc)


def test_binary_search_converges_on_sphere():
    g = torch.Generator().manual_seed(0)
    inner = torch.nn.functional.normalize(torch.randn(200, 3, generator=g), dim=1) * 0.3
    outer = torch.nn.functional.normalize(torch.randn(200, 3, generator=g), dim=1) * 1.2
    alpha = lambda p: (p.norm(dim=1) < 0.7).float()          # occupancy: 1 inside the sphere of radius 0.7
    end_points = torch.stack([inner, outer], dim=1)
    end_sdf = torch.stack([alpha(inner) - 0.5, alpha(outer) - 0.5], dim=1).reshape(-1, 2, 1)
    pts = gof_extract.binary_search(end_points, end_sdf, alpha, n_steps=8)
    # each step halves the bracket: |r - 0.7| <= |outer - inner| / 2^9
    assert float((pts.norm(dim=1) - 0.7).abs().max()) < 1.5 / 2 ** 8


# ---- tet-chunk sharded marching tetrahedra (SURVEY 8(e)) -----------------------------------------------------------------
def _oracle_extract(vertices, tets, sdf, scales, rows):
    """extract_fn for gof_extract.marching_tetrahedra_sharded backed by the numpy oracle (stated rows per chunk)."""
    import numpy as np
    import tetmesh_oracle
    t = tets.numpy()
    ids, faces = None, None
    for c0 in range(0, t.shape[0], rows):          # the oracle's chunk loop with the rows given directly
        i, f = tetmesh_oracle._one_chunk(t[c0:c0 + rows], sdf.numpy().reshape(-1))
        if ids is None:
            ids, faces = i, f
        else:
            allk = np.concatenate([ids, i], axis=0)
            uniq, inv = np.unique(allk, axis=0, return_inverse=True)
            inv = inv.reshape(-1)
            faces = np.concatenate([inv[faces.reshape(-1)].reshape(-1, 3), inv[f.reshape(-1) + ids.shape[0]].reshape(-1, 3)], axis=0)
            ids = uniq
    if ids is None:
        ids, faces = np.zeros((0, 2), np.int64), np.zeros((0, 3), np.int64)
    iv = torch.from_numpy(ids)
    v = vertices.reshape(-1, 3)
    return ((v[iv.reshape(-1)].reshape(-1, 2, 3), sdf.reshape(-1)[iv.reshape(-1)].reshape(-1, 2, 1)),
            scales.reshape(-1)[iv.reshape(-1)].reshape(-1, 2, 1), torch.from_numpy(faces), iv)


def _golden_chunked():
    import numpy as np
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tetmesh_chunked1000.npz"))
    return {k: torch.from_numpy(z[k]) for k in z.files if k != "chunk_size"}, int(z["chunk_size"])


def test_merge_of_tet_shards_equals_reference_chunked_output():
    """Shards cut at the chunk boundaries of the unsharded call, extracted independently and merged by
    gof_extract.merge_tet_shards, reproduce the reference's own chunked output (golden from utils/tetmesh.py) bit for bit."""
    import gof_tetmesh
    g, chunk = _golden_chunked()
    T = g["tets"].shape[0]
    rows = gof_tetmesh.chunk_rows(T, chunk)
    assert rows == -(-T // (T // chunk + 1))
    for world in (1, 2, 3, 4, 7):
        keys, faces = [], []
        for r in range(world):
            b, e = gof_extract.shard_tet_range(T, rows, r, world)
            (_p, _s), _sc, f, iv = _oracle_extract(g["vertices"], g["tets"][b:e], g["sdf"], g["scales"], rows)
            keys.append(gof_extract._edge_keys(iv)); faces.append(f)
        (pos, esdf), esc, f, iv = gof_extract.merge_tet_shards(g["vertices"], g["sdf"], g["scales"], keys, faces)
        assert torch.equal(iv, g["interp_v"]) and torch.equal(f, g["faces"]), world
        assert torch.equal(pos, g["edge_pos"]) and torch.equal(esdf, g["edge_sdf"]) and torch.equal(esc, g["edge_scales"])


def _tet_worker(rank, world, port, q):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    g, chunk = _golden_chunked()
    (pos, esdf), esc, f, iv = gof_extract.marching_tetrahedra_sharded(g["vertices"], g["tets"], g["sdf"], g["scales"], chunk_tets=chunk,
                                                                       extract_fn=_oracle_extract)
    q.put((rank, f.numpy().copy(), iv.numpy().copy(), pos.numpy().copy()))
    dist.destroy_process_group()


def test_tet_sharded_marching_tetrahedra_world2():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_tet_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(2)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    g, _ = _golden_chunked()
    for _, f, iv, pos in res:
        assert torch.equal(torch.from_numpy(f), g["faces"]) and torch.equal(torch.from_numpy(iv), g["interp_v"])
        assert torch.equal(torch.from_numpy(pos), g["edge_pos"])
