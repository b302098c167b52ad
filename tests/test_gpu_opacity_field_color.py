"""GPU: gof_extract.opacity_field(..., return_color=True), the colour of the multi-view opacity field (DESIGN.md 4.13).

* (alpha, colour) equal evaluate_alpha(..., return_color=True) bit for bit, ties and points that no view lowers included;
* the gradients equal autograd through the explicit composition (per-view integrate_gaussians, the winner's colour gathered):
  the points bit for bit, the Gaussians and their SHs up to summation order;
* peak memory over forward and backward does not grow with the number of views;
* two ranks equal one under a colour loss;
* Adam on the SH DC coefficients fits the field's colour over 8 views."""
import os
import sys

import numpy as np
import pytest
import torch

import _integrate_scenes as isc
import gof_extract
import gof_synth
from test_gpu_extract import _points, _scene, _settings_for
from test_gpu_opacity_field import _free_port, _outside_points, _peak, assert_gaussian_grads_close, extract_scene

pytestmark = pytest.mark.gpu

KEYS = ("means3D", "opacities", "scales", "rotations", "shs")


def _gs(gs, dev, grad=False):
    return {k: gs[k].to(dev).clone().requires_grad_(grad) for k in KEYS}


def field(pts, g, views, sf, deg=3, group=None):
    return gof_extract.opacity_field(pts, g["means3D"], g["opacities"], g["scales"], g["rotations"], g["shs"], deg, views, sf,
                                     group=group, return_color=True)


def reference(pts, g, views, sf, deg=3):
    ci = gof_extract.make_integrate_fn(g["means3D"], g["opacities"], g["scales"], g["rotations"], g["shs"], deg, sf)
    return gof_extract.evaluate_alpha(pts, views, ci, return_color=True)


def composition(pts, g, views, sf):
    """The field and its colour through autograd's own bookkeeping: every view's integrate_gaussians kept until backward()."""
    from diff_gaussian_rasterization import integrate_gaussians
    outs = [integrate_gaussians(pts, g["means3D"], torch.zeros_like(g["means3D"]), g["opacities"], g["shs"], None, g["scales"],
                                g["rotations"], None, None, sf(v)) for v in views]
    a = torch.stack([o[1] for o in outs])
    c = torch.stack([o[2] for o in outs])
    win = torch.argmin(a.detach(), dim=0)   # the first (lowest-index) minimum
    amin = a.gather(0, win[None]).squeeze(0)
    col = c.gather(0, win[None, :, None].expand(1, -1, 3)).squeeze(0)
    col = torch.where((amin.detach() < 1.0)[:, None], col, torch.ones_like(col))
    return 1 - amin, col


def grads(fn, pts, gs, dev, dA, dC):
    p = pts.clone().requires_grad_(True)
    g = _gs(gs, dev, grad=True)
    a, c = fn(p, g)
    ((a * dA).sum() + (c * dC).sum()).backward()
    return a.detach(), c.detach(), p.grad, {k: g[k].grad for k in KEYS}


def _cap():
    cam, gs, pts = isc.cap_scene()
    dev = torch.device("cuda")
    views = [cam, gof_synth.make_camera(48, 32, view=4), gof_synth.make_camera(48, 32, view=2)]
    sf = lambda c: gof_synth.raster_settings(c, gs["sh_degree"], dev)   # noqa: E731
    return dev, views, gs, pts.to(dev), sf


def test_forward_equals_evaluate_alpha():
    dev, cams, gs, pts = extract_scene()
    sf = _settings_for(dev)
    g = _gs(gs, dev)
    pts = torch.cat([_outside_points(5000, 1).to(dev), pts])
    for views in (cams, [cams[1], cams[0], cams[1], cams[2], cams[1]]):   # the second with exact ties
        a, c = field(pts, g, views, sf)
        ra, rc = reference(pts, g, views, sf)
        assert torch.equal(a, ra) and torch.equal(c, rc)
        assert bool((c[:5000] == 1).all())   # no view lowered them
        assert float((c[5000:] != 1).any(dim=1).float().mean()) > 0.3
    dev, views, gs, pts, sf = _cap()
    g = _gs(gs, dev)
    a, c = field(pts, g, views, sf, gs["sh_degree"])
    ra, rc = reference(pts, g, views, sf, gs["sh_degree"])
    assert torch.equal(a, ra) and torch.equal(c, rc)


@pytest.mark.parametrize("case", ["extract", "ties_and_outside", "cap"])
def test_gradients_equal_the_composition(case):
    if case == "cap":
        dev, views, gs, pts, sf = _cap()
    else:
        dev, cams, gs, pts = extract_scene()
        pts = pts[:60_000].contiguous()
        sf = _settings_for(dev)
        views = cams
        if case == "ties_and_outside":
            views = [cams[1], cams[0], cams[1], cams[3], cams[1]]
            pts = torch.cat([_outside_points(2000, 2).to(dev), pts])
    gen = torch.Generator().manual_seed(7)
    dA, dC = torch.randn(pts.shape[0], generator=gen).to(dev), torch.randn(pts.shape[0], 3, generator=gen).to(dev)
    deg = gs["sh_degree"] if case == "cap" else 3
    a, c, gp, gg = grads(lambda p, g: field(p, g, views, sf, deg), pts, gs, dev, dA, dC)
    a0, c0, gp0, gg0 = grads(lambda p, g: composition(p, g, views, sf), pts, gs, dev, dA, dC)
    assert torch.equal(a, a0) and torch.equal(c, c0)
    assert torch.equal(gp, gp0)
    assert_gaussian_grads_close(gg, gg0, case)
    assert float(gg["shs"].abs().max()) > 0
    # a colour loss alone: zero point gradients
    _a, _c, gpc, _gg = grads(lambda p, g: field(p, g, views, sf, deg), pts, gs, dev, torch.zeros_like(dA), dC)
    assert bool((gpc == 0).all())


def test_memory_does_not_grow_with_views():
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda")
    P, W, H = 20_000, 320, 240
    gs = gof_synth.make_scene(dict(P=P, width=W, height=H, seed=61), view=0)[1]
    cams = [gof_synth.make_camera(W, H, view=2 * v) for v in range(32)]
    sf = _settings_for(dev)
    pts = _points(gs, 50_000, 3, dev)
    g = _gs(gs, dev)
    st = _C.integrate_gaussians_to_points_state(*gof_extract._field_args(sf(cams[0]), pts, g["means3D"], g["opacities"], g["scales"],
                                                                          g["rotations"], g["shs"]))
    state_bytes = sum(t.numel() for t in st[5:])
    del st

    def run(n):
        p = pts.clone().requires_grad_(True)
        q = _gs(gs, dev, grad=True)
        a, c = field(p, q, cams[:n], sf)
        (a.sum() + c.sum()).backward()

    run(4)
    peak = {n: _peak(lambda: run(n)) for n in (4, 32, 4)}
    print(f"[memory, colour] one view's state {state_bytes / 2**20:.1f} MiB; peak 4 views {peak[4] / 2**20:.1f} MiB, 32 views "
          f"{peak[32] / 2**20:.1f} MiB")
    assert abs(peak[32] - peak[4]) < state_bytes


def _dist_case(dev):
    _dev, cams, gs, _g = _scene(P=20_000, W=320, H=240, seed=61, n_views=7)
    pts = _points(gs, 40_000, 5, dev)
    views = cams + [cams[2]]   # a tie across ranks
    gen = torch.Generator().manual_seed(9)
    return gs, pts, views, torch.randn(pts.shape[0], 3, generator=gen).to(dev)


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
    gs, pts, views, dC = _dist_case(dev)
    half = pts.shape[0] // 2   # each rank supervises the colour of its own half of the points
    keep = ((torch.arange(pts.shape[0], device=dev) < half) == (rank == 0))[:, None]
    a, c, gp, gg = grads(lambda p, g: field(p, g, views, _settings_for(dev), group=dist.group.WORLD), pts, gs, dev,
                         torch.zeros(pts.shape[0], device=dev), torch.where(keep, dC, torch.zeros_like(dC)))
    q.put((rank, a.cpu().numpy(), c.cpu().numpy(), gp.cpu().numpy(), {k: v.cpu().numpy() for k, v in gg.items()}))
    dist.barrier()
    dist.destroy_process_group()


def test_two_ranks_equal_one():
    """Two ranks, each with a colour loss on half of the points: every rank's field and colour equal the single-GPU ones bit for
    bit, and every rank's gradients are the single-GPU gradients of the sum of the two losses.  NCCL with a GPU per rank where
    there are two, otherwise gloo with both ranks on one GPU."""
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
    gs, pts, views, dC = _dist_case(dev)
    a, c, gp, gg = grads(lambda p, g: field(p, g, views, _settings_for(dev)), pts, gs, dev, torch.zeros(pts.shape[0], device=dev), dC)
    assert float(gg["shs"].abs().max()) > 0
    for _rank, ra, rc, rgp, rgg in res:
        assert np.array_equal(ra, a.cpu().numpy()) and np.array_equal(rc, c.cpu().numpy())
        assert np.array_equal(rgp, gp.cpu().numpy()) and not rgp.any()
        assert_gaussian_grads_close({k: torch.from_numpy(v) for k, v in rgg.items()}, {k: v.cpu() for k, v in gg.items()},
                                    "2 ranks, colour")


def test_colour_descent_over_8_views():
    """Adam on the SH DC coefficients (geometry fixed) fits the field's colour at surface points to the colour of another set of
    DC coefficients, over 8 views."""
    from test_gpu_opacity_field import cloud_scene
    dev = torch.device("cuda")
    cams, gs = cloud_scene()
    sf = lambda c: gof_synth.raster_settings(c, 0, dev)   # noqa: E731
    g = _gs(gs, dev)
    gen = torch.Generator().manual_seed(9)
    cand = ((torch.rand(100_000, 3, generator=gen) * 2 - 1) * 1.3).to(dev)
    tg = dict(g)
    tg["shs"] = g["shs"].clone()
    tg["shs"][:, 0, :] = (torch.rand(g["shs"].shape[0], 3, generator=gen).to(dev) * 0.6 - 0.3) / 0.28209479177387814
    with torch.no_grad():
        a0, target = field(cand, tg, cams, sf, 0)
    pts = cand[(a0 > 0.3)][:20_000].contiguous()
    target = target[(a0 > 0.3)][:20_000]
    assert pts.shape[0] > 1000
    dc = g["shs"][:, :1, :].clone().requires_grad_(True)
    rest = g["shs"][:, 1:, :]
    opt = torch.optim.Adam([dc], lr=0.05)

    def loss_fn():
        q = dict(g, shs=torch.cat([dc, rest], 1))
        return ((field(pts, q, cams, sf, 0)[1] - target) ** 2).mean()

    first = float(loss_fn())
    for _ in range(60):
        opt.zero_grad()
        loss = loss_fn()
        loss.backward()
        opt.step()
    last = float(loss_fn())
    print(f"[colour descent, 8 views] {pts.shape[0]} points, loss {first:.5f} -> {last:.6f}")
    assert last < 0.1 * first
