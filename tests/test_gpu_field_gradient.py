"""GPU: gof_extract.field_gradient, evaluate_alpha's field and its point gradient in one pass over cached views (DESIGN.md 4.14),
and the vertex normals extract_level_set derives from it.

* alpha, the winning view and the colour equal evaluate_alpha over the same CachedIntegrator bit for bit, and the gradient
  equals points.grad of opacity_field(...).sum().backward() bit for bit, on the extract scene, exact view ties with points
  outside every view, the 1 024-contributor cap, the uint16 id wrap, 5 000 points in one pixel and points on tile and image
  borders; points no view wins get zeros;
* no Gaussians, no points, no view;
* two ranks equal one bit for bit;
* on a sphere of surface Gaussians the normals at bisected vertices point outward (alpha rises from inside to outside);
* extract_level_set(return_normals=True) leaves the rest of the mesh as it is, and its normals survive a PLY round trip."""
import os
import socket
import sys

import numpy as np
import pytest
import torch

import _integrate_scenes as isc
import gof_extract
import gof_synth
import gof_tsdf
from test_gpu_extract import _points, _scene, _settings_for
from test_gpu_opacity_field import _outside_points

pytestmark = pytest.mark.gpu

NO_VIEW = 2 ** 30


def _dev_gs(gs, dev):
    return {k: (v.to(dev).contiguous() if isinstance(v, torch.Tensor) else v) for k, v in gs.items()}


def _cached(g, deg, sf):
    return gof_extract.CachedIntegrator(g["means3D"], g["opacities"], g["scales"], g["rotations"], g["shs"], deg, sf)


def _reference_argmin(pts, views, ci):
    """The lowest view index attaining the minimum over views of alpha_integrated, where it is below 1 (evaluate_alpha's winner)."""
    n = pts.shape[0]
    best = torch.ones(n, device=pts.device)
    arg = torch.full((n,), NO_VIEW, dtype=torch.int32, device=pts.device)
    for vi, v in enumerate(views):
        a, _c = ci(pts, v)
        better = a < best
        arg = torch.where(better, torch.full_like(arg, vi), arg)
        best = torch.where(better, a, best)
    return arg


def _argmin(pts, views, ci):
    """argmin as the cached running minimum leaves it (with the gradient formed, as field_gradient runs it)."""
    n = pts.shape[0]
    am = torch.ones(n, device=pts.device)
    arg = torch.full((n,), NO_VIEW, dtype=torch.int32, device=pts.device)
    gm = torch.zeros(n, 3, device=pts.device)
    for vi, v in enumerate(views):
        ci.min_update(pts, v, vi, am, arg, grad_min=gm)
    return arg


def _autograd_point_grad(pts, g, deg, views, sf):
    p = pts.clone().requires_grad_(True)
    a = gof_extract.opacity_field(p, g["means3D"], g["opacities"], g["scales"], g["rotations"], g["shs"], deg, views, sf)
    a.sum().backward()
    return a.detach(), p.grad


def check_case(name, pts, g, deg, views, sf, min_active=0.01):
    ci = _cached(g, deg, sf)
    alpha, grad, color = gof_extract.field_gradient(pts, views, ci, return_color=True)
    alpha0, color0 = gof_extract.evaluate_alpha(pts, views, ci, return_color=True)
    assert torch.equal(alpha, alpha0), name
    assert torch.equal(color, color0), name
    arg = _argmin(pts, views, ci)
    assert torch.equal(arg, _reference_argmin(pts, views, ci)), name
    # the alpha-only instantiation gives the same field and gradient
    alpha1, grad1 = gof_extract.field_gradient(pts, views, ci)
    assert torch.equal(alpha1, alpha0) and torch.equal(grad1, grad), name
    a_ag, grad_ag = _autograd_point_grad(pts, g, deg, views, sf)
    assert torch.equal(a_ag, alpha0), name
    assert torch.equal(grad, grad_ag), name
    assert bool((grad[arg == NO_VIEW] == 0).all()), name
    active = float((grad != 0).any(dim=1).float().mean())
    print(f"[field_gradient] {name}: {pts.shape[0]} points, {active:.3f} with a nonzero gradient")
    assert active >= min_active, (name, active)
    return alpha, grad, arg


def test_extract_scene():
    dev, cams, gs, g = _scene()
    pts = _points(gs, 200_000, 5, dev)
    check_case("extract", pts, g, 3, cams, _settings_for(dev), min_active=0.1)


def test_ties_and_points_outside_every_view():
    dev, cams, gs, g = _scene()
    pts = torch.cat([_outside_points(3000, 2).to(dev), _points(gs, 60_000, 6, dev)]).contiguous()
    views = [cams[1], cams[0], cams[1], cams[3], cams[1]]
    alpha, grad, arg = check_case("ties and outside", pts, g, 3, views, _settings_for(dev))
    assert bool((arg[:3000] == NO_VIEW).all()) and bool((grad[:3000] == 0).all()) and bool((alpha[:3000] == 0).all())
    assert not bool((arg == 2).any()) and not bool((arg == 4).any())   # a tie goes to the lowest view index


def _small_sf(dev, deg):
    return lambda c: gof_synth.raster_settings(c, deg, dev)   # noqa: E731


def test_contributor_cap_scene():
    cam, gs, pts = isc.cap_scene()
    dev = torch.device("cuda")
    views = [cam, gof_synth.make_camera(48, 32, view=4), gof_synth.make_camera(48, 32, view=2)]
    check_case("cap", pts.to(dev), _dev_gs(gs, dev), gs["sh_degree"], views, _small_sf(dev, gs["sh_degree"]), min_active=0.3)


def test_uint16_wrap_scene():
    cam, gs, pts, _pix = isc.u16_scene()
    dev = torch.device("cuda")
    views = [cam, gof_synth.make_camera(32, 16, view=6)]
    check_case("u16", pts.to(dev), _dev_gs(gs, dev), gs["sh_degree"], views, _small_sf(dev, gs["sh_degree"]))


def test_5000_points_in_one_pixel():
    cam, gs = gof_synth.make_scene(dict(P=700, width=96, height=64, seed=41), view=3)
    dev = torch.device("cuda")
    rng = np.random.default_rng(5)
    hot = isc.cam_to_world(cam, isc.pixel_to_cam(cam, rng.uniform(40.0, 41.0, 5000), rng.uniform(30.0, 31.0, 5000), rng.uniform(2.0, 6.0, 5000)))
    pts = torch.from_numpy(hot.astype(np.float32)).to(dev)
    views = [cam, gof_synth.make_camera(96, 64, view=5)]
    check_case("one pixel", pts, _dev_gs(gs, dev), gs["sh_degree"], views, _small_sf(dev, gs["sh_degree"]))


def _border_points(cam, W, H):
    """float32 points whose projection lies on pixel, tile and image borders: the float64 pre-image of each border and up to
    20 float32 steps either way in each coordinate."""
    out = []
    targets = [(x, 20.3) for x in (0.0, 1.0, 16.0, 32.0, 64.0, W - 1.0, float(W))] + \
              [(33.6, y) for y in (0.0, 16.0, 32.0, H - 1.0, float(H))] + [(0.0, 0.0), (float(W), float(H)), (16.0, 16.0)]
    for x, y in targets:
        base = isc.cam_to_world(cam, isc.pixel_to_cam(cam, x, y, 3.1)).astype(np.float32).reshape(3)
        for col in (0, 1, 2):
            v = np.float32(base[col])
            up, dn = v, v
            for _ in range(20):
                up, dn = np.nextafter(up, np.float32(np.inf)), np.nextafter(dn, np.float32(-np.inf))
                for val in (up, dn):
                    p = base.copy()
                    p[col] = val
                    out.append(p)
        out.append(base)
    return np.asarray(out, np.float32)


def test_points_on_tile_and_image_borders():
    W, H = 80, 48
    cam = gof_synth.make_camera(W, H, view=11)
    rng = np.random.default_rng(23)
    gs = isc.blobs(cam, np.stack([rng.uniform(0, W, 600), rng.uniform(0, H, 600)], 1), rng.uniform(2.0, 5.0, 600),
                   rng.uniform(1.0, 4.0, 600), rng.uniform(0.05, 0.9, 600), seed=24)
    dev = torch.device("cuda")
    pts = torch.from_numpy(_border_points(cam, W, H)).to(dev)
    views = [cam, gof_synth.make_camera(W, H, view=12)]
    check_case("borders", pts, _dev_gs(gs, dev), gs["sh_degree"], views, _small_sf(dev, gs["sh_degree"]))


def test_empty_inputs():
    dev, cams, gs, g = _scene(P=5000, W=160, H=120)
    sf = _settings_for(dev)
    pts = _points(gs, 4000, 3, dev)
    none = {k: (v[:0].contiguous() if isinstance(v, torch.Tensor) else v) for k, v in g.items()}
    for name, p, gg, views in (("no Gaussians", pts, none, cams), ("no points", pts[:0], g, cams), ("no view", pts, g, [])):
        ci = _cached(gg, 3, sf)
        alpha, grad, color = gof_extract.field_gradient(p, views, ci, return_color=True)
        alpha0, color0 = gof_extract.evaluate_alpha(p, views, ci, return_color=True)
        assert torch.equal(alpha, alpha0) and torch.equal(color, color0), name
        assert grad.shape == (p.shape[0], 3) and bool((grad == 0).all()), name
        assert bool((alpha == 0).all()), name


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _dist_case(dev):
    _d, cams, gs, g = _scene(P=20_000, W=320, H=240, seed=61, n_views=7)
    g = _dev_gs(gs, dev)
    pts = _points(gs, 40_000, 5, dev)
    return g, pts, cams + [cams[2]]   # a tie across ranks: view 2 (rank 0 of 2) and view 7 (rank 1)


def _dist_worker(rank, world, port, backend, q):
    here = os.path.dirname(os.path.abspath(__file__))
    for p in (here, os.path.join(here, "..", "gaussian-opacity-fields_b200")):
        sys.path.insert(0, p)
    import torch.distributed as dist
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    kw = dict(device_id=dev) if backend == "nccl" else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    g, pts, views = _dist_case(dev)
    ci = _cached(g, 3, _settings_for(dev))
    a, gr, c = gof_extract.field_gradient(pts, views, ci, return_color=True, group=dist.group.WORLD)
    a1, gr1 = gof_extract.field_gradient(pts, views, ci, group=dist.group.WORLD)
    q.put((rank, a.cpu().numpy(), gr.cpu().numpy(), c.cpu().numpy(), a1.cpu().numpy(), gr1.cpu().numpy()))
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
    dev = torch.device("cuda", 0)
    g, pts, views = _dist_case(dev)
    ci = _cached(g, 3, _settings_for(dev))
    a, gr, c = gof_extract.field_gradient(pts, views, ci, return_color=True)
    assert float((gr != 0).any(dim=1).float().mean()) > 0.1
    for _rank, ra, rgr, rc, ra1, rgr1 in res:
        assert np.array_equal(ra, a.cpu().numpy()) and np.array_equal(ra1, ra)
        assert np.array_equal(rgr, gr.cpu().numpy()) and np.array_equal(rgr1, rgr)
        assert np.array_equal(rc, c.cpu().numpy())


def _sphere(dev, P=20_000, n_views=24):
    gs = gof_synth.make_surface_gaussians(P, seed=3)
    views = gof_synth.make_surface_views(320, 240, n_views)
    sf = _small_sf(dev, 0)
    return _dev_gs(gs, dev), views, sf


def test_normals_point_outward_on_a_sphere():
    dev = torch.device("cuda")
    g, views, sf = _sphere(dev)
    ci = _cached(g, 0, sf)
    gen = torch.Generator().manual_seed(11)
    d = torch.randn(20_000, 3, generator=gen, dtype=torch.float64)
    d = (d / d.norm(dim=1, keepdim=True)).to(torch.float32).to(dev)
    ends = torch.stack([0.7 * d, 1.3 * d], dim=1).contiguous()                         # (E, 2, 3): inside, outside
    sdf = (gof_extract.evaluate_alpha(ends.reshape(-1, 3), views, ci) - 0.5).reshape(-1, 2, 1)
    # alpha = 1 - min over views of the opacity in front of the point: ~0 inside the sphere, ~1 outside it
    keep = (sdf[:, 0, 0] < 0) & (sdf[:, 1, 0] > 0)
    assert float(keep.float().mean()) > 0.9, float(keep.float().mean())
    ends, sdf, d = ends[keep], sdf[keep], d[keep]
    verts = gof_extract.binary_search(ends, sdf, lambda p: gof_extract.evaluate_alpha(p, views, ci), n_steps=8)
    _a, grad = gof_extract.field_gradient(verts, views, ci)
    norm = grad.norm(dim=1)
    ok = norm > 0
    n = grad[ok] / norm[ok, None]   # extract_level_set's normal
    cos = (n * d[ok]).sum(dim=1)
    deg = torch.rad2deg(torch.acos(cos.clamp(-1, 1))).cpu().numpy()
    q = np.percentile(deg, [50, 90, 99, 100])
    print(f"[normals] {int(ok.sum())} of {verts.shape[0]} vertices with a gradient; angle to the radial direction, degrees: "
          f"median {q[0]:.2f}, 90% {q[1]:.2f}, 99% {q[2]:.2f}, max {q[3]:.2f}; min dot {float(cos.min()):.4f}")
    assert float(ok.float().mean()) > 0.99
    assert bool((cos > 0).all())
    assert q[0] < 20.0 and q[1] < 45.0


def _sphere_tets(dev, n_points=40_000, n_tets=250_000):
    gen = torch.Generator().manual_seed(9)
    pts = (torch.rand(n_points, 3, generator=gen) * 2 - 1) * 1.5
    a = torch.randint(0, n_points, (n_tets,), generator=gen)
    tets = torch.stack([a, (a + 1) % n_points, (a + 7) % n_points, (a + 31) % n_points], dim=1)
    return pts.to(dev), torch.full((n_points, 1), 0.05, device=dev), tets.to(dev)


def test_extract_level_set_normals(tmp_path):
    dev = torch.device("cuda")
    g, views, sf = _sphere(dev)
    ci = _cached(g, 0, sf)
    pts, scales, tets = _sphere_tets(dev)
    base = gof_extract.extract_level_set(pts, scales, tets, views, ci, return_color=True, chunk_tets=100_000)
    tm = {}
    out = gof_extract.extract_level_set(pts, scales, tets, views, ci, return_color=True, chunk_tets=100_000, return_normals=True,
                                        timings=tm)
    assert "normals" not in base and "field_gradient_s" in tm
    for k in ("vertices", "faces", "mask", "colors"):
        assert torch.equal(out[k], base[k]), k
    n = out["normals"]
    assert n.shape == out["vertices"].shape and out["vertices"].shape[0] > 1000
    length = n.norm(dim=1)
    assert bool(((length - 1).abs() < 1e-5).logical_or(length == 0).all())
    # the random tets' long edges also cross jumps of the field (where a view stops seeing a point, its alpha_integrated is exactly
    # 0 or 1 with no gradient); bisection stops next to the jump, and such vertices get zero normals
    print(f"[extract normals] {n.shape[0]} vertices, {float((length > 0).float().mean()):.3f} with a normal")
    assert float((length > 0).float().mean()) > 0.5
    # without colours: the same normals
    plain = gof_extract.extract_level_set(pts, scales, tets, views, ci, chunk_tets=100_000, return_normals=True)
    assert plain["colors"] is None and torch.equal(plain["normals"], n)
    path = tmp_path / "mesh.ply"
    gof_tsdf.write_ply(str(path), out)
    back = gof_tsdf.read_ply(str(path))
    assert np.array_equal(back["normals"], n.cpu().numpy())
    assert np.array_equal(back["vertices"], out["vertices"].cpu().numpy())
    assert np.array_equal(back["faces"], out["faces"].cpu().numpy())
