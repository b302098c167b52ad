"""GPU: gof_extract.opacity_field, the multi-view opacity field alpha = 1 - min over views of alpha_integrated with gradients
(DESIGN.md 4.12).

* the forward equals gof_extract.evaluate_alpha bit for bit;
* a query of a subset of the points gives each point the alpha bits of the full query (the backward relies on it);
* the point gradients equal, bit for bit, autograd through the explicit composition: per-view integrate_gaussians, stacked,
  each point's lowest-index winner gathered; the Gaussian gradients match it up to summation order (ALLOW below);
* no points, or no view that wins a point, give zeros;
* peak memory over forward and backward does not grow with the number of views, where the composition's does;
* two ranks, each with its own loss, give the single-GPU field bit for bit and the single-GPU gradients of the sum of
  their losses (point gradients bit for bit);
* Adam on the points pulls them onto the 0.5 level set."""
import os
import socket
import sys

import numpy as np
import pytest
import torch

import _integrate_scenes as isc
import gof_extract
import gof_synth
from test_gpu_extract import _points, _scene, _settings_for

pytestmark = pytest.mark.gpu

# The Gaussian gradients of the field and of the composition are the same sums of the same per-(view, point) terms, formed in a
# different order: within a view the double atomics of k_integrate_backward (then rounded to float once, as in DESIGN.md 4.11),
# across views a float sum in view order here and in autograd's order there.  Allowance, as in test_gpu_integrate_grad.py's
# comparison of two such sums: rtol 1e-4 and atol 1e-6 relative to the largest entry of the tensor.
ALLOW = dict(rtol=1e-4, atol_rel=1e-6)


def _gs_from(gs, dev, grad=False):
    return {k: (gs[k].to(dev).clone().requires_grad_(grad and k != "shs")) for k in ("means3D", "opacities", "scales", "rotations", "shs")}


def field(pts, g, views, sf, group=None):
    return gof_extract.opacity_field(pts, g["means3D"], g["opacities"], g["scales"], g["rotations"], g["shs"], 3, views, sf, group=group)


def composition(pts, g, views, sf):
    """The field through autograd's own bookkeeping: every view's integrate_gaussians kept alive until backward()."""
    from diff_gaussian_rasterization import integrate_gaussians
    stack = torch.stack([integrate_gaussians(pts, g["means3D"], torch.zeros_like(g["means3D"]), g["opacities"], g["shs"], None,
                                             g["scales"], g["rotations"], None, None, sf(v))[1] for v in views])
    win = torch.argmin(stack.detach(), dim=0)   # the first (lowest-index) minimum
    return 1 - stack.gather(0, win[None]).squeeze(0)


def reference(pts, g, views, sf):
    ci = gof_extract.make_integrate_fn(g["means3D"], g["opacities"], g["scales"], g["rotations"], g["shs"], 3, sf)
    return gof_extract.evaluate_alpha(pts, views, ci)


def grads(fn, pts, gs, dev, dL):
    p = pts.clone().requires_grad_(True)
    g = _gs_from(gs, dev, grad=True)
    a = fn(p, g)
    (a * dL).sum().backward()
    return a.detach(), p.grad, {k: g[k].grad for k in ("means3D", "opacities", "scales", "rotations")}


def assert_gaussian_grads_close(got, want, name):
    for k in want:
        w = want[k]
        atol = ALLOW["atol_rel"] * float(w.abs().max()) + 1e-30
        torch.testing.assert_close(got[k], w, rtol=ALLOW["rtol"], atol=atol, msg=lambda m: f"{name} {k}: {m}")


def _outside_points(n, seed):
    """Points that project into no camera of the ring (gof_synth.make_camera: radius 4, 20 degrees below the origin, 60 degree
    horizontal field of view): 1 000 units straight above or below the origin, 70 degrees or more off every optical axis."""
    gen = torch.Generator().manual_seed(seed)
    p = (torch.rand(n, 3, generator=gen) * 2 - 1) * 50.0
    p[:, 1] = torch.where(torch.rand(n, generator=gen) < 0.5, -1e3, 1e3)
    return p.contiguous()


def extract_scene():
    dev, cams, gs, _g = _scene()
    pts = _points(gs, 200_000, 5, dev)
    return dev, cams, gs, pts


def test_forward_equals_evaluate_alpha():
    dev, cams, gs, pts = extract_scene()
    sf = _settings_for(dev)
    g = _gs_from(gs, dev)
    a = field(pts, g, cams, sf)
    want = reference(pts, g, cams, sf)
    assert torch.equal(a, want)
    assert float((a > 0).float().mean()) > 0.3   # the scene has an inside
    # points outside every view: the field is 0 and no view wins
    out = torch.cat([_outside_points(5000, 1).to(dev), pts[:5000]])
    a = field(out, g, cams, sf)
    assert torch.equal(a, reference(out, g, cams, sf))
    assert bool((a[:5000] == 0).all())
    # exact ties: the same camera three times, between others
    views = [cams[1], cams[0], cams[1], cams[2], cams[1]]
    assert torch.equal(field(pts, g, views, sf), reference(pts, g, views, sf))


def test_forward_cap_scene():
    """The 1 024-contributor cap (isc.cap_scene), seen from its own camera and two more of the ring."""
    cam, gs, pts = isc.cap_scene()
    dev = torch.device("cuda")
    views = [cam, gof_synth.make_camera(48, 32, view=4), gof_synth.make_camera(48, 32, view=2)]
    sf = lambda c: gof_synth.raster_settings(c, gs["sh_degree"], dev)   # noqa: E731
    g = _gs_from(gs, dev)
    p = pts.to(dev)
    a = gof_extract.opacity_field(p, g["means3D"], g["opacities"], g["scales"], g["rotations"], g["shs"], gs["sh_degree"], views, sf)
    ci = gof_extract.make_integrate_fn(g["means3D"], g["opacities"], g["scales"], g["rotations"], g["shs"], gs["sh_degree"], sf)
    assert torch.equal(a, gof_extract.evaluate_alpha(p, views, ci))
    assert float((a > 0).float().mean()) > 0.5


def test_subset_query_is_bit_identical():
    """alpha_integrated of a point does not depend on which other points are queried with it: pass 1's contributor lists depend
    on the pixel only."""
    from diff_gaussian_rasterization import GaussianRasterizer
    dev, cams, gs, pts = extract_scene()
    g = _gs_from(gs, dev)
    gen = torch.Generator().manual_seed(4)
    for cam in cams[:3]:
        rs = gof_synth.raster_settings(cam, 3, dev)
        q = lambda p: GaussianRasterizer(rs).integrate(points3D=p, means3D=g["means3D"], means2D=torch.zeros_like(g["means3D"]),  # noqa: E731
                                                       opacities=g["opacities"], shs=g["shs"], scales=g["scales"],
                                                       rotations=g["rotations"])[1]
        full = q(pts)
        for frac in (0.5, 0.01):
            sel = torch.nonzero(torch.rand(pts.shape[0], generator=gen) < frac).flatten().to(dev)
            assert torch.equal(q(pts[sel].contiguous()), full[sel])


@pytest.mark.parametrize("case", ["extract", "ties_and_outside", "cap"])
def test_gradients_equal_the_composition(case):
    if case == "cap":
        cam, gs, pts = isc.cap_scene()
        dev = torch.device("cuda")
        views = [cam, gof_synth.make_camera(48, 32, view=4), gof_synth.make_camera(48, 32, view=2)]
        sf = lambda c: gof_synth.raster_settings(c, gs["sh_degree"], dev)   # noqa: E731
        pts = pts.to(dev)
    else:
        dev, cams, gs, pts = extract_scene()
        pts = pts[:60_000].contiguous()
        sf = _settings_for(dev)
        views = cams
        if case == "ties_and_outside":
            views = [cams[1], cams[0], cams[1], cams[3], cams[1]]
            pts = torch.cat([_outside_points(2000, 2).to(dev), pts])
    dL = torch.randn(pts.shape[0], generator=torch.Generator().manual_seed(7)).to(dev)
    a, gp, gg = grads(lambda p, g: field(p, g, views, sf), pts, gs, dev, dL)
    a0, gp0, gg0 = grads(lambda p, g: composition(p, g, views, sf), pts, gs, dev, dL)
    assert torch.equal(a, a0)
    assert torch.equal(gp, gp0)
    assert float((gp != 0).any(dim=1).float().mean()) > 0.1
    assert_gaussian_grads_close(gg, gg0, case)
    if case == "ties_and_outside":
        assert bool((gp[:2000] == 0).all())
    # a second call gives the same point gradients (no atomics on the point side)
    _a, gp1, _gg = grads(lambda p, g: field(p, g, views, sf), pts, gs, dev, dL)
    assert torch.equal(gp, gp1)


def test_empty_inputs_give_zeros():
    dev, cams, gs, pts = extract_scene()
    sf = _settings_for(dev)
    for p in (pts[:0], _outside_points(3000, 3).to(dev)):
        pp = p.clone().requires_grad_(True)
        g = _gs_from(gs, dev, grad=True)
        a = field(pp, g, cams, sf)
        assert a.shape == (p.shape[0],) and bool((a == 0).all())
        (a * 1.5).sum().backward()
        assert pp.grad is not None and bool((pp.grad == 0).all())
        for k in ("means3D", "opacities", "scales", "rotations"):
            assert bool((g[k].grad == 0).all()), k


def _peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def test_memory_does_not_grow_with_views():
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda")
    P, W, H = 20_000, 320, 240
    gs = gof_synth.make_scene(dict(P=P, width=W, height=H, seed=61), view=0)[1]
    cams = [gof_synth.make_camera(W, H, view=2 * v) for v in range(32)]
    sf = _settings_for(dev)
    pts = _points(gs, 50_000, 3, dev)
    g = _gs_from(gs, dev)
    # one view's query state: the five scratch buffers of integrate_gaussians_to_points_state
    st = _C.integrate_gaussians_to_points_state(*gof_extract._field_args(sf(cams[0]), pts, g["means3D"], g["opacities"], g["scales"],
                                                                          g["rotations"], g["shs"]))
    state_bytes = sum(t.numel() for t in st[5:])
    del st

    def run(fn, n):
        p = pts.clone().requires_grad_(True)
        q = _gs_from(gs, dev, grad=True)
        fn(p, q, cams[:n]).sum().backward()

    f = lambda p, q, v: field(p, q, v, sf)         # noqa: E731
    c = lambda p, q, v: composition(p, q, v, sf)   # noqa: E731
    run(f, 4)   # the scratch pool holds the buffers a view needs from here on
    peak = {n: _peak(lambda: run(f, n)) for n in (4, 32, 4)}
    naive = {n: _peak(lambda: run(c, n)) for n in (4, 16)}
    print(f"[memory] one view's state {state_bytes / 2**20:.1f} MiB; field peak 4 views {peak[4] / 2**20:.1f} MiB, 32 views "
          f"{peak[32] / 2**20:.1f} MiB; composition 4 views {naive[4] / 2**20:.1f} MiB, 16 views {naive[16] / 2**20:.1f} MiB")
    assert abs(peak[32] - peak[4]) < state_bytes
    assert naive[16] - naive[4] > 6 * state_bytes


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _dist_case(dev):
    dev_, cams, gs, _g = _scene(P=20_000, W=320, H=240, seed=61, n_views=7)
    pts = _points(gs, 40_000, 5, dev)
    views = cams + [cams[2]]   # a tie across ranks: view 2 (rank 0 of 2) and view 7 (rank 1)
    dL = torch.randn(pts.shape[0], generator=torch.Generator().manual_seed(9)).to(dev)
    return gs, pts, views, dL


def _rank_loss(dL, loss, rank):
    """dL/dalpha of `rank` (of 2) in each case of test_two_ranks_equal_one."""
    if loss == "replicated":     # the same loss on every rank: it counts twice
        return dL
    if loss == "one_rank":       # only rank 0 has a loss
        return dL if rank == 0 else torch.zeros_like(dL)
    half = dL.shape[0] // 2      # "split": each rank supervises its own half of the points
    keep = (torch.arange(dL.shape[0], device=dL.device) < half) == (rank == 0)
    return torch.where(keep, dL, torch.zeros_like(dL))


def _dist_worker(rank, world, port, backend, loss, q):
    here = os.path.dirname(os.path.abspath(__file__))
    for p in (here, os.path.join(here, "..", "gaussian-opacity-fields_b200")):
        sys.path.insert(0, p)
    import torch.distributed as dist
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    kw = dict(device_id=dev) if backend == "nccl" else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    gs, pts, views, dL = _dist_case(dev)
    a, gp, gg = grads(lambda p, g: field(p, g, views, _settings_for(dev), group=dist.group.WORLD), pts, gs, dev,
                      _rank_loss(dL, loss, rank))
    q.put((rank, a.cpu().numpy(), gp.cpu().numpy(), {k: v.cpu().numpy() for k, v in gg.items()}))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("loss", ["replicated", "one_rank", "split"])
def test_two_ranks_equal_one(loss):
    """Two ranks, each with its own dL/dalpha: every rank's field equals the single-GPU field bit for bit, and every rank's
    gradients are the single-GPU gradients of the sum of the two losses, the point gradients bit for bit.  Over NCCL with a GPU
    per rank where there are two, otherwise over gloo with both ranks on one GPU."""
    import torch.multiprocessing as mp
    backend = "nccl" if torch.cuda.device_count() >= 2 else "gloo"
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_dist_worker, args=(r, world, port, backend, loss, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=600) for _ in range(world)], key=lambda x: x[0])
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    dev = torch.device("cuda", 0)
    gs, pts, views, dL = _dist_case(dev)
    total = _rank_loss(dL, loss, 0) + _rank_loss(dL, loss, 1)
    a, gp, gg = grads(lambda p, g: field(p, g, views, _settings_for(dev)), pts, gs, dev, total)
    assert float((gp != 0).any(dim=1).float().mean()) > 0.1
    for _rank, ra, rgp, rgg in res:
        assert np.array_equal(ra, a.cpu().numpy())
        assert np.array_equal(rgp, gp.cpu().numpy())
        assert_gaussian_grads_close({k: torch.from_numpy(v) for k, v in rgg.items()}, {k: v.cpu() for k, v in gg.items()},
                                    f"2 ranks, {loss}")


def cloud_scene(P=2000, seed=5):
    """A soft cloud: P isotropic Gaussians (sigma 0.25, opacity 0.02) uniform in the unit ball, seen by 8 cameras of the ring at
    160x120.  The field rises from 0 outside to 1 inside over about a tenth of the radius, smoothly enough for descent."""
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(P, 3, generator=g, dtype=torch.float64)
    m = d / d.norm(dim=1, keepdim=True) * torch.rand(P, 1, generator=g, dtype=torch.float64) ** (1.0 / 3.0)
    f32 = lambda t: t.to(torch.float32).contiguous()   # noqa: E731
    gs = {"means3D": f32(m), "scales": f32(torch.full((P, 3), 0.25, dtype=torch.float64)),
          "rotations": f32(torch.tensor([1.0, 0.0, 0.0, 0.0], dtype=torch.float64).expand(P, 4)),
          "opacities": f32(torch.full((P, 1), 0.02, dtype=torch.float64)), "shs": f32(torch.zeros(P, 16, 3, dtype=torch.float64)),
          "sh_degree": 0}
    cams = [gof_synth.make_camera(160, 120, view=8 * k) for k in range(8)]
    return cams, gs


def test_descent_onto_the_half_level_set():
    """Adam on the points alone (Gaussians fixed) drives the multi-view field at them toward 0.5."""
    dev = torch.device("cuda")
    cams, gs = cloud_scene()
    sf = lambda c: gof_synth.raster_settings(c, 0, dev)   # noqa: E731
    g = _gs_from(gs, dev)
    gen = torch.Generator().manual_seed(9)
    cand = ((torch.rand(100_000, 3, generator=gen) * 2 - 1) * 1.3).to(dev)
    with torch.no_grad():
        a0 = field(cand, g, cams, sf)
    pts = cand[(a0 > 0.05) & (a0 < 0.95)][:20_000].clone().requires_grad_(True)
    assert pts.shape[0] > 1000
    steps = 150
    opt = torch.optim.Adam([pts], lr=1e-2)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda i: 0.03 ** (i / steps))

    def loss_fn():
        return ((field(pts, g, cams, sf) - 0.5) ** 2).mean()

    first = float(loss_fn())
    for _ in range(steps):
        opt.zero_grad()
        loss = loss_fn()
        loss.backward()
        opt.step()
        sched.step()
    last = float(loss_fn())
    print(f"[descent] {pts.shape[0]} points, mean (alpha - 0.5)^2 {first:.5f} -> {last:.6f} ({first / max(last, 1e-30):.1f}x)")
    assert last * 10 <= first
