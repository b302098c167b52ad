"""GPU: the rasterizer backward writing straight into a gof_dp.GradBucket (the `_out=` extension of
`_C.rasterize_gaussians_backward`): every gradient view equals the plain call for a P that is NOT a multiple of 4 (the
bucket's fields are 256-byte aligned, k_preprocess_backward stores dL_drot / dL_dsh with 128-bit stores), and the
densification statistics the backward leaves in the bucket's tail equal GaussianModel.add_densification_stats' inputs
(scene/gaussian_model.py:709-714, train.py:255) derived from dL_dmeans2D and radii."""
import pytest
import torch

import _util
import gof_dp
import gof_synth

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("P", [30_011, 4_097, 1])
def test_backward_into_bucket_any_P(P):
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda")
    cam, gs = gof_synth.make_scene(dict(P=P, width=320, height=208, seed=17), view=4)
    fa = _util.fwd_args(cam, gs, dev)
    R, color, radii, geom, binning, img = _C.rasterize_gaussians(*fa)
    grad = torch.randn(9, 208, 320, generator=torch.Generator().manual_seed(2)).to(dev)
    plain = _C.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, grad))
    bucket = gof_dp.GradBucket(P, 16, dev)
    for v in bucket.views.values():
        assert v.data_ptr() % 256 == 0
    out = _C.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, grad), _out=bucket.views)
    torch.cuda.synchronize()
    names = ["dmeans2D", "dcolors", "dopacity", "dmeans3D", "dcov3D", "dsh", "dscales", "drot", "dv2g"]
    for n, a, b in zip(names, out, plain):
        assert _util.same_up_to_summation_order(a, b), (n, _util.rel_err(a, b))
        if n in bucket.views:
            assert a.data_ptr() == bucket.views[n].data_ptr()
    # densification statistics of this view
    dm2, vis = out[0], radii > 0
    want_sum = torch.zeros(P, 3, device=dev)
    want_sum[:, 0] = torch.where(vis, dm2[:, :2].norm(dim=-1), want_sum[:, 0])
    want_sum[:, 1] = torch.where(vis, dm2[:, 2].abs(), want_sum[:, 1])
    want_sum[:, 2] = vis.float()
    want_max = torch.stack([torch.where(vis, dm2[:, 2].abs(), torch.zeros_like(dm2[:, 2])), radii.float()], dim=1)
    assert _util.rel_err(bucket.views["dens_sum"], want_sum)[0] < 1e-6
    assert torch.equal(bucket.views["dens_max"], want_max)
    old = gof_dp.densification_stats(dm2, radii)          # the round-1 helper: same quantities, [P,4]
    assert _util.rel_err(bucket.views["dens_sum"], old[:, :3])[0] < 1e-6 and torch.equal(bucket.views["dens_max"][:, 1], old[:, 3])


def test_misaligned_inputs_are_accepted():
    """A parameter sliced out of a flat buffer at an odd offset (4-byte aligned only, like the reference accepts) must not fault:
    the binding copies it to an aligned allocation, and forward and backward compute what they compute from aligned inputs."""
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda")
    P = 5_003
    cam, gs = gof_synth.make_scene(dict(P=P, width=160, height=128, seed=19), view=1)
    fa = list(_util.fwd_args(cam, gs, dev))
    base = _C.rasterize_gaussians(*fa)
    flat = torch.zeros(1 + P * 4 + P * 48 + 8, device=dev)
    rot = flat[1:1 + 4 * P].view(P, 4); rot.copy_(gs["rotations"].to(dev))
    shs = flat[1 + 4 * P:1 + 4 * P + 48 * P].view(P, 16, 3); shs.copy_(gs["shs"].to(dev))
    assert rot.data_ptr() % 16 != 0 and shs.data_ptr() % 16 != 0
    fa[5], fa[17] = rot, shs
    out = _C.rasterize_gaussians(*fa)
    assert out[0] == base[0] and torch.equal(out[1], base[1]) and torch.equal(out[2], base[2])
    grad = torch.randn(9, 128, 160, generator=torch.Generator().manual_seed(7)).to(dev)
    g = _C.rasterize_gaussians_backward(*_util.bwd_args(tuple(fa), out[2], out[3], out[0], out[4], out[5], grad))
    g = [t.clone() for t in g]
    aligned = _C.rasterize_gaussians_backward(*_util.bwd_args(_util.fwd_args(cam, gs, dev), base[2], base[3], base[0], base[4],
                                                             base[5], grad))
    torch.cuda.synchronize()
    names = ["dmeans2D", "dcolors", "dopacity", "dmeans3D", "dcov3D", "dsh", "dscales", "drot", "dv2g"]
    assert float(aligned[5].abs().max()) > 0 and float(aligned[7].abs().max()) > 0
    for n, a, b in zip(names, g, aligned):
        assert _util.same_up_to_summation_order(a, b), (n, _util.rel_err(a, b))


def test_backward_fills_uninitialised_outputs():
    """The backward writes EVERY element of its outputs (zeros for unseen Gaussians, for dL_dcov3D, for SH coefficients above the
    active degree): garbage-filled `_out` tensors end up identical to the plain call's."""
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda")
    P = 20_001
    cam, gs = gof_synth.make_scene(dict(P=P, width=256, height=192, seed=23), view=40)      # many Gaussians outside this view
    gs = dict(gs)
    fa = _util.fwd_args(cam, gs, dev, sh_degree=1)                                          # degree 1 of 16 coefficients: tail columns
    R, color, radii, geom, binning, img = _C.rasterize_gaussians(*fa)
    assert int((radii == 0).sum()) > 100
    grad = torch.randn(9, 192, 256, generator=torch.Generator().manual_seed(5)).to(dev)
    shapes = dict(dmeans3D=(P, 3), dmeans2D=(P, 3), dcolors=(P, 3), dopacity=(P, 1), dcov3D=(P, 6), dsh=(P, 16, 3), dscales=(P, 3),
                  drot=(P, 4), dv2g=(P, 10), dens_sum=(P, 3), dens_max=(P, 2))
    out = {k: torch.full(s, float("nan"), device=dev) for k, s in shapes.items()}
    g = _C.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, grad), _out=out)
    torch.cuda.synchronize()
    for k, t in out.items():
        assert torch.isfinite(t).all(), k
    inv = radii == 0
    for k in ("dmeans3D", "dmeans2D", "dcolors", "dopacity", "dsh", "dscales", "drot", "dv2g", "dens_sum", "dens_max"):
        assert float(out[k][inv].abs().max()) == 0.0, k
    assert float(out["dcov3D"].abs().max()) == 0.0
    assert float(out["dsh"][:, 4:, :].abs().max()) == 0.0 and float(out["dsh"][:, :4, :].abs().max()) > 0.0
    plain = _C.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, grad))
    assert _util.rel_err(g[5], plain[5])[0] < 1e-5 and _util.rel_err(g[2], plain[2])[0] < 1e-5


def test_conv3x3_weight_gradient_kernel():
    """csrc/conv_wgrad.cu (the appearance network's tail) against a float64 evaluation of the same convolution's weight / bias
    gradient, for every instantiated channel pair, on image sizes that are not tile multiples."""
    import gof_appearance
    dev = torch.device("cuda")
    gen = torch.Generator().manual_seed(3)
    # (W % 4 == 0: the kernel's vector fill; otherwise its scalar fill)
    for (co, ci), (H, W) in (((16, 16), (203, 333)), ((16, 16), (130, 200)), ((3, 16), (130, 200)), ((3, 16), (131, 257)),
                             ((16, 8), (264, 129)), ((16, 8), (136, 264))):
        conv = torch.nn.Conv2d(ci, co, 3, padding=1).to(dev)
        x = torch.randn(1, ci, H, W, generator=gen).to(dev).requires_grad_(True)
        gy = torch.randn(1, co, H, W, generator=gen).to(dev)
        y = gof_appearance.conv3x3(x, conv)
        assert y.grad_fn is not None and "Conv3x3" in type(y.grad_fn).__name__
        y.backward(gy)
        conv64 = torch.nn.Conv2d(ci, co, 3, padding=1).to(dev).double()
        conv64.load_state_dict({k: v.double() for k, v in conv.state_dict().items()})
        x64 = x.detach().double().requires_grad_(True)
        conv64(x64).backward(gy.double())
        assert _util.rel_err(conv.weight.grad, conv64.weight.grad)[0] < 2e-5, (co, ci)
        assert _util.rel_err(conv.bias.grad, conv64.bias.grad)[0] < 2e-5
        assert _util.rel_err(x.grad, x64.grad)[0] < 5e-3          # cuDNN's TF32 data gradient


@pytest.mark.parametrize("P,degrees", [(30_011, (3, 3, 3)), (4_097, (3, 1, 2)), (4_097, (3,) * 7), (2_051, (3,) * 11), (1_027, (2, 3))])
def test_factored_sh_gradient_is_the_sum_of_the_views(P, degrees):
    """View-parallel exchange (csrc/sh_views.cu): the backward asked for the factored SH gradient leaves dL_dRGB + the camera
    centre (and every other output unchanged); gof_sh_grad_from_views over the views' records is BIT-identical to adding the
    views' dL_dsh tensors of the same backward runs in view order (backward.cu:45-139 is an outer product per view)."""
    import ctypes
    from diff_gaussian_rasterization import _C
    import gof_dp
    dev = torch.device("cuda")
    H, W = 208, 320
    plane = (P + 63) // 64 * 64                        # GOF_SH_PLANE(P)
    slot = gof_dp.SH_SLOT_HEADER + 3 * plane
    nv = len(degrees)                                  # 2 / 3 / 7 / 11 views: every instantiation of the expansion kernel
    records = torch.full((nv * slot,), float("nan"), device=dev)
    grad = torch.randn(9, H, W, generator=torch.Generator().manual_seed(2)).to(dev)
    want, means = None, None
    for i, (view, deg) in enumerate(zip([(4 + 7 * j) % 64 for j in range(nv)], degrees)):
        cam, gs = gof_synth.make_scene(dict(P=P, width=W, height=H, seed=17), view=view)
        fa = _util.fwd_args(cam, gs, dev, sh_degree=deg)
        R, color, radii, geom, binning, img = _C.rasterize_gaussians(*fa)
        plain = _C.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, grad))
        rec = records[i * slot:(i + 1) * slot]
        # ONE backward leaves both the record and (checks only: "_dsh_full") this view's own dL_dsh -- the order of the blend
        # kernel's double sums may move a last bit between two backward runs, so the bit-exact statement needs both from one run
        full = torch.full((P, 16, 3), float("nan"), device=dev)
        out = {"sh_hdr": rec[:gof_dp.SH_SLOT_HEADER], "dsh_rgb": rec[gof_dp.SH_SLOT_HEADER:].view(3, plane),
               "_dsh_full": full}
        fact = _C.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, grad), _out=out)
        torch.cuda.synchronize()
        assert fact[5] is None and out["_means3D"].data_ptr() == fa[1].data_ptr()
        for k in (0, 1, 2, 3, 4, 6, 7, 8):           # the other outputs: the plain backward's, up to the order of its double sums
            assert _util.same_up_to_summation_order(fact[k], plain[k]), (k, _util.rel_err(fact[k], plain[k]))
        assert _util.rel_err(full, plain[5])[1] < 1e-4
        assert torch.equal(rec[:3], fa[19]) and float(rec[3]) == deg
        assert not torch.isnan(out["dsh_rgb"][:, :P]).any() and not torch.isnan(full).any()
        assert float(out["dsh_rgb"][:, :P][:, radii == 0].abs().sum()) == 0.0
        want = full.clone() if want is None else want + full
        means = fa[1]
    got = torch.full((P, 16, 3), float("nan"), device=dev)
    ptrs = (ctypes.c_void_p * nv)(*[records.data_ptr() + 4 * i * slot for i in range(nv)])
    _C._check(_C._lib.gof_sh_grad_from_views(P, 16, nv, means.data_ptr(), ptrs, got.data_ptr(), _C._stream()))
    torch.cuda.synchronize()
    assert float(want.abs().max()) > 0
    assert torch.equal(got, want)
    # ... and the torch statement of the same sum (the CPU buckets of the gloo tests) agrees to rounding
    ref = gof_dp.sh_grad_from_views_torch(means, [records[i * slot:(i + 1) * slot] for i in range(nv)], P, 16)
    assert _util.rel_err(ref, want)[0] < 1e-5


def test_public_rasterizer_writes_into_grad_bucket():
    """`GaussianRasterizer(settings, grad_bucket=bucket)` (extension): loss.backward() through the public autograd wrapper leaves
    the parameter gradients and the densification statistics in the bucket -- the .grad tensors of the plain wrapper -- and hands
    nothing but dL_dmeans2D back to autograd."""
    from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    dev = torch.device("cuda")
    P, H, W = 20_003, 208, 320
    cam, gs = gof_synth.make_scene(dict(P=P, width=W, height=H, seed=17), view=4)
    rs = GaussianRasterizationSettings(
        image_height=H, image_width=W, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, kernel_size=0.0,
        subpixel_offset=torch.zeros(H, W, 2, device=dev), bg=torch.zeros(3, device=dev), scale_modifier=1.0,
        viewmatrix=cam.world_view_transform.to(dev), projmatrix=cam.full_proj_transform.to(dev), sh_degree=3,
        campos=cam.camera_center.to(dev), prefiltered=False, debug=False)
    wgt = torch.randn(9, H, W, generator=torch.Generator().manual_seed(3)).to(dev)

    def run(bucket):
        params = {k: gs[k].to(dev).clone().requires_grad_(True) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
        means2D = torch.zeros(P, 3, device=dev, requires_grad=True)
        r = GaussianRasterizer(rs) if bucket is None else GaussianRasterizer(rs, grad_bucket=bucket)
        img, radii = r(means3D=params["means3D"], means2D=means2D, opacities=params["opacities"], shs=params["shs"],
                       scales=params["scales"], rotations=params["rotations"])
        (img * wgt).sum().backward()
        return params, means2D, radii

    params, m2d, radii = run(None)
    bucket = gof_dp.GradBucket(P, 16, dev)
    params_b, m2d_b, _ = run(bucket)
    torch.cuda.synchronize()
    for name, key in (("means3D", "dmeans3D"), ("shs", "dsh"), ("opacities", "dopacity"), ("scales", "dscales"), ("rotations", "drot")):
        assert params_b[name].grad is None
        # (two backward runs: equal up to the order of the blend kernel's double sums)
        got = bucket.views[key].reshape(params[name].grad.shape)
        assert _util.same_up_to_summation_order(got, params[name].grad), (name, _util.rel_err(got, params[name].grad))
    assert _util.same_up_to_summation_order(m2d_b.grad, m2d.grad)
    assert torch.equal(bucket.views["dens_max"][:, 1], radii.float())
