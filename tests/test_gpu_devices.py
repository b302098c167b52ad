"""GPU, needs >= 2 devices (skipped on a one-GPU box): one process drives cuda:0, then cuda:1, then cuda:0 again, and every
device computes what the first one computed.  The library keeps its launch state per device -- the blend kernels'
shared-memory carveout, conv3x3_wgrad's opt-in to ~89 KB of dynamic shared memory and its occupancy, the SM counts that size
grids and scratch -- so a device used second is set up like the first."""
import pytest
import torch

import _util
import gof_synth
from test_gpu_train_step import _ternary, _wgrad_call, conv_wgrad_ref

pytestmark = pytest.mark.gpu

ORDER = (0, 1, 0)
GRADS = ["dmeans2D", "dcolors", "dopacity", "dmeans3D", "dcov3D", "dsh", "dscales", "drotations", "dv2g"]


def _need_two():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs in one process")


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _views(cam, gs, pts, dL, d):
    """Forward + export_state, backward, integrate and prepare + cached query of one view on cuda:d."""
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda", d)
    fa = _util.fwd_args(cam, gs, dev)
    R, color, radii, geom, binning, img = _C.rasterize_gaussians(*fa)
    exact = dict(R=torch.tensor(R), color=color, radii=radii)
    exact.update(_C.export_state(gs["means3D"].shape[0], cam.image_width, cam.image_height, R, geom, binning, img, radii))
    grads = _C.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, dL.to(dev)))
    p = pts.to(dev)
    iR, icolor, ialpha, icol, iradii = _C.integrate_gaussians_to_points(fa[0], p, *fa[1:])[:5]
    exact.update(iR=torch.tensor(iR), icolor=icolor, ialpha=ialpha, icol=icol, iradii=iradii)
    cache = _C.integrate_prepare(*fa)
    ccolor, calpha, ccol = _C.integrate_points_cached(cache, fa[0], p, fa[9], fa[11], fa[12])
    exact.update(cR=torch.tensor(cache.num_rendered), cradii=cache.radii, ccolor=ccolor, calpha=calpha, ccol=ccol)
    torch.cuda.synchronize(dev)
    return {k: v.cpu() for k, v in exact.items()}, [g.cpu() for g in grads]


def test_rasterizer_computes_the_same_on_every_device():
    """Forward outputs, export_state fields and both opacity-field queries bit-identical; gradients within test_gpu_repro's
    bound (the backward's double atomics may land in another order)."""
    _need_two()
    cam, gs = gof_synth.make_scene("C2", view=3)
    pts, _ = gof_synth.make_tetra_points(gs, 9 * gs["means3D"].shape[0], seed=7, device="cpu")
    dL = torch.randn(9, cam.image_height, cam.image_width, generator=torch.Generator().manual_seed(11))
    first = None
    for d in ORDER:
        exact, grads = _views(cam, gs, pts, dL, d)
        if first is None:
            first = exact, grads
            assert int(exact["R"]) > 0 and float(exact["ialpha"].max()) > 0
            continue
        for k, v in first[0].items():
            assert torch.equal(_bits(exact[k]), _bits(v)), (d, k)
        for name, a, b in zip(GRADS, grads, first[1]):
            assert _util.same_up_to_summation_order(a, b), (d, name)


def test_queries_refuse_points_on_another_device():
    """The binding refuses query points on another device than the Gaussians or the cache, before the library sees the pointer."""
    _need_two()
    from diff_gaussian_rasterization import _C
    cam, gs = gof_synth.make_scene("C2", view=3)
    fa = _util.fwd_args(cam, gs, torch.device("cuda", 0))
    p = torch.rand(1000, 3, device="cuda:1")
    with pytest.raises(RuntimeError, match="expected cuda:0"):
        _C.integrate_gaussians_to_points(fa[0], p, *fa[1:])
    cache = _C.integrate_prepare(*fa)
    with pytest.raises(RuntimeError, match="expected cuda:0"):
        _C.integrate_points_cached(cache, fa[0], p, fa[9], fa[11], fa[12])


def test_conv_wgrad_on_every_device():
    """The 16 -> 16 instantiation needs its dynamic shared memory opt-in on each device; {-1, 0, 1} inputs make dW and db exact."""
    _need_two()
    co, ci, H, W = 16, 16, 1056, 1920
    gen = torch.Generator().manual_seed(5)
    x, gy = _ternary((ci, H, W), 0.6, gen, "cpu"), _ternary((co, H, W), 0.6, gen, "cpu")
    ref_w, ref_b = conv_wgrad_ref(x.double(), gy.double())
    for d in ORDER:
        dev = torch.device("cuda", d)
        xd, gd = x.to(dev), gy.to(dev)
        dW, db = torch.zeros(co, ci, 3, 3, device=dev), torch.zeros(co, device=dev)
        with torch.cuda.device(dev):
            _wgrad_call(co, ci, H, W, xd, gd, dW, db)
            torch.cuda.synchronize()
        assert torch.equal(dW.cpu().double(), ref_w) and torch.equal(db.cpu().double(), ref_b), d
