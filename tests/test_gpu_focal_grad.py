"""GPU: the focal-length gradient of the backward (gof_backward_out_t.dL_dtan_fov, DESIGN.md 4.10).

(a) Every pixel's dL/drx, dL/dry (the [2,H,W] map the call leaves in its scratch) against the float64 oracle
    (tests/focal_oracle/focal_oracle.c) run from this library's own forward state with the same dL_dpix:

        |gpu - oracle|  <=  c * 2^-24 * (1 + L) * mag  +  marginal,      L = the view's longest walk, c = C_RAYS,

    the model of tests/_grad_bounds.py: T is recovered pair by pair on the GPU, which drifts by about one ulp per pair, and a
    pair near a blend threshold exempts every pair in front of it.  Both sums against the oracle's within the sum over the
    pixels of |rx| (|ry|) times the pixel's allowance, over tan_fov, plus half an ulp of the float result.  Observed on an
    H100 80GB HBM3 (700 W power limit): largest per-pixel ratio 0.0017 (c2_v3, L = 816) and 0.0055 (ragged_4097, L = 245);
    largest summed error / allowance 1.7e-6 and 3.1e-4.  The per-pixel values go through no atomics, so these are the same
    on every run.
(b) Two calls give identical bits; every other output, the pose gradient included, is bit-identical with and without the
    intrinsics outputs wherever the blend's outputs are identical (the blend backward sums with double atomics, see
    test_gpu_camera_grad (b)).
(c) Through the public API, .grad of tanfovx / tanfovy (CPU or CUDA 0-dim tensors) is the ABI output; joint use with the
    view matrix; float settings still run the plain kernels; P == 0; the refusal with a grad_bucket; integrate and
    markVisible accept tensor tan_fov values.
(d) Descent: Adam on the field of view recovers a perturbed focal length against the unperturbed render, alone and together
    with a pose perturbation.  Reached on an H100 80GB HBM3 (700 W power limit): largest relative field-of-view error
    0.040 -> 0.00003 alone, 0.040 -> 0.0071 together with the pose."""
import math

import numpy as np
import pytest
import torch

import _focal_oracle as fo
import _grad_bounds as gb
import _util
import gof_synth

pytestmark = pytest.mark.gpu

C_RAYS = 2.0 ** -5   # 4x the largest ratio observed (0.0055, ragged_4097), rounded up to a power of two
NAMES = ("dmeans2D", "dcolors", "dopacity", "dmeans3D", "dcov3D", "dsh", "dscales", "drot", "dv2g")
BLEND = ("dmeans2D", "dcolors", "dopacity", "dv2g")

SCENES = {
    "c2_v3": (lambda: gof_synth.make_scene("C2", view=3), (0.0, 0.0, 0.0)),
    # P not a multiple of the 128-Gaussian CTA, odd image size, a background
    "ragged_4097": (lambda: gof_synth.make_scene(dict(P=4097, width=203, height=117, seed=17), view=4), (0.3, 0.6, 0.9)),
}


def _forward(cam, gs, bg=(0.0, 0.0, 0.0)):
    from diff_gaussian_rasterization import _C
    fa = _util.fwd_args(cam, gs, torch.device("cuda"), bg=bg)
    R, _color, radii, geom, binning, img = _C.rasterize_gaussians(*fa)
    return fa, R, radii, geom, binning, img


def _backward(fwd, dL, camera=False, intrinsics=False, ray_map=False):
    from diff_gaussian_rasterization import _C
    fa, R, radii, geom, binning, img = fwd
    out = _C.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, dL), _camera=camera,
                                          _intrinsics=intrinsics, _ray_map=ray_map)
    torch.cuda.synchronize()
    return [t.detach().clone() for t in out]


def _ulp(x):
    return np.spacing(np.abs(np.float32(x))).astype(np.float64)


@pytest.mark.parametrize("name", list(SCENES))
def test_ray_gradient_against_the_fp64_oracle(name):
    from diff_gaussian_rasterization import _C
    make, bg = SCENES[name]
    cam, gs = make()
    P, W, H = gs["means3D"].shape[0], cam.image_width, cam.image_height
    fwd = _forward(cam, gs, bg)
    st = {k: v.cpu().numpy() for k, v in _C.export_state(P, W, H, fwd[1], fwd[3], fwd[4], fwd[5], fwd[2]).items()}
    dL = torch.randn(9, H, W, generator=torch.Generator().manual_seed(41))
    g = _backward(fwd, dL.cuda(), intrinsics=True, ray_map=True)
    gx, gy, rays = float(g[9]), float(g[10]), g[11].cpu().numpy()
    d = fo.rays(W, H, cam.tanfovx, cam.tanfovy, st, np.asarray(bg, np.float32), dL.numpy(), float_geometry=True)
    L = int(st["n_contrib"][0].max())
    allow = C_RAYS * gb.EPS * (1.0 + L) * d["mag"] + d["marginal"]
    err = np.abs(rays - d["drays"])
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(err > 0, np.maximum(err - d["marginal"], 0.0) / (gb.EPS * (1.0 + L) * d["mag"]), 0.0)
    print(f"{name}: L = {L}, largest per-pixel |gpu - oracle - marginal| / (2^-24 (1 + L) mag) = {float(ratio.max()):.3g}, "
          f"pixels with marginal mass {float((d['marginal'].sum(axis=0) > 0).mean()):.2e}")
    assert (err <= allow).all(), (float(ratio.max()), np.unravel_index(np.argmax(ratio), ratio.shape))
    assert np.abs(d["drays"]).max() > 0
    # the sums
    rx, ry = fo.pixel_rays(W, H, cam.tanfovx, cam.tanfovy)
    ox, oy = fo.tan_fov_grad(d["drays"], cam.tanfovx, cam.tanfovy)
    ax = float((np.abs(rx.astype(np.float64))[None, :] * allow[0]).sum()) / float(np.float32(cam.tanfovx))
    ay = float((np.abs(ry.astype(np.float64))[:, None] * allow[1]).sum()) / float(np.float32(cam.tanfovy))
    for what, got, ora, a in (("tanfovx", gx, ox, ax), ("tanfovy", gy, oy, ay)):
        bound = a + 0.5 * _ulp(ora)
        print(f"{name} {what}: gpu {got:.9g} oracle {ora:.9g}, |gpu - oracle| / allowance = {abs(got - ora) / bound:.3g}")
        assert abs(got - ora) <= bound, (what, got, ora, bound)
        assert ora != 0.0


def _bits(a):
    return a.contiguous().view(torch.int32)


@pytest.mark.parametrize("name", list(SCENES))
def test_reproducible_and_other_outputs_unchanged(name):
    make, bg = SCENES[name]
    cam, gs = make()
    fwd = _forward(cam, gs, bg)
    dL = torch.randn(9, cam.image_height, cam.image_width, generator=torch.Generator().manual_seed(5)).cuda()
    plain = _backward(fwd, dL, camera=True)
    both = _backward(fwd, dL, camera=True, intrinsics=True, ray_map=True)
    again = _backward(fwd, dL, camera=True, intrinsics=True, ray_map=True)
    fov_only = _backward(fwd, dL, intrinsics=True)
    assert len(plain) == 11 and len(both) == 14 and len(fov_only) == 11
    # the focal-length gradient does not go through the blend's atomics: bit-identical from call to call
    assert torch.equal(both[13].view(torch.int64), again[13].view(torch.int64))
    for i in (11, 12):
        assert torch.equal(_bits(both[i]), _bits(again[i])) and torch.equal(_bits(both[i]), _bits(fov_only[9 + i - 11]))
    P = gs["means3D"].shape[0]
    vis = fwd[2] > 0

    def same_blend(x, y):   # [P] bool: every blend-stage output of the Gaussian is bitwise equal in x and y
        m = torch.ones(P, dtype=torch.bool, device=vis.device)
        for n in BLEND:
            i = NAMES.index(n)
            m &= (_bits(x[i]).view(P, -1) == _bits(y[i]).view(P, -1)).all(dim=1)
        return m

    for other in (both, fov_only):
        same = same_blend(plain, other)
        assert float((~same & vis).sum()) <= 1e-3 * float(vis.sum())
        for i, n in enumerate(NAMES):
            a, b = plain[i], other[i]
            if n in BLEND:
                assert _util.same_up_to_summation_order(b, a), n
            elif a.numel():
                assert torch.equal(_bits(a).view(P, -1)[same], _bits(b).view(P, -1)[same]), n
    if bool(same_blend(plain, both).all()):
        assert torch.equal(_bits(plain[9]), _bits(both[9])) and torch.equal(_bits(plain[10]), _bits(both[10]))
    else:
        for i in (9, 10):
            assert _util.same_up_to_summation_order(both[i], plain[i])


# ---- the public API ----------------------------------------------------------------------------------------------------

def _small_scene(P=4000):
    return gof_synth.make_scene(dict(P=P, width=160, height=104, seed=5), view=7)


def _api(cam, gs, fov_device="cpu", fov_dtype=torch.float32, camera=False, fov=True, colors=False):
    """Render + backward through GaussianRasterizer with tanfovx / tanfovy as 0-dim tensors on `fov_device` (float settings
    when fov is False)."""
    from diff_gaussian_rasterization import GaussianRasterizer, _C
    dev = torch.device("cuda")
    rs = gof_synth.raster_settings(cam, gs["sh_degree"], dev)
    vm = rs.viewmatrix.clone().requires_grad_(camera)
    tx = torch.tensor(cam.tanfovx, dtype=fov_dtype, device=fov_device, requires_grad=True) if fov else cam.tanfovx
    ty = torch.tensor(cam.tanfovy, dtype=fov_dtype, device=fov_device, requires_grad=True) if fov else cam.tanfovy
    rs = rs._replace(viewmatrix=vm, tanfovx=tx, tanfovy=ty)
    p = {k: gs[k].to(dev).requires_grad_(True) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    kw = dict(colors_precomp=torch.rand(p["means3D"].shape[0], 3, generator=torch.Generator().manual_seed(2)).to(dev)) if colors \
        else dict(shs=p["shs"])
    _C.profile_reset()
    _C.profile_enable(True)
    color, _radii = GaussianRasterizer(rs)(means3D=p["means3D"], means2D=torch.zeros_like(p["means3D"], requires_grad=True),
                                           opacities=p["opacities"], scales=p["scales"], rotations=p["rotations"], **kw)
    dL = torch.randn(9, cam.image_height, cam.image_width, generator=torch.Generator().manual_seed(9))
    (color * dL.to(dev)).sum().backward()
    torch.cuda.synchronize()
    kernels = set(_C.profile_report())
    _C.profile_enable(False)
    return dict(tx=tx, ty=ty, vm=vm, p=p, dL=dL, kernels=kernels)


@pytest.mark.parametrize("fov_device,fov_dtype,camera", [("cpu", torch.float32, False), ("cuda", torch.float32, False),
                                                         ("cpu", torch.float64, True), ("cuda", torch.float32, True)])
def test_public_api_focal_grad_is_the_abi_output(fov_device, fov_dtype, camera):
    cam, gs = _small_scene()
    r = _api(cam, gs, fov_device, fov_dtype, camera)
    assert "render_bwd_rays" in r["kernels"] and "focal_grad_sum" in r["kernels"] and "render_bwd" not in r["kernels"]
    assert ("preprocess_bwd_camera" in r["kernels"]) == camera
    gx, gy = r["tx"].grad, r["ty"].grad
    for g, t in ((gx, r["tx"]), (gy, r["ty"])):
        assert g.shape == t.shape and g.dtype == t.dtype and g.device == t.device
    fwd = _forward(cam, gs)
    g = _backward(fwd, r["dL"].cuda(), camera=camera, intrinsics=True)
    # the focal-length gradient is bit-reproducible; the API's value is the ABI's float, converted to the input's dtype
    assert float(gx) == float(g[-2]) and float(gy) == float(g[-1])
    assert float(g[-2]) != 0.0 and float(g[-1]) != 0.0
    if camera:
        assert r["vm"].grad is not None and _util.same_up_to_summation_order(r["vm"].grad, g[9])


def test_public_api_float_settings_run_the_plain_backward():
    cam, gs = _small_scene()
    r = _api(cam, gs, fov=False, camera=True)
    assert "render_bwd" in r["kernels"] and "render_bwd_rays" not in r["kernels"] and "focal_grad_sum" not in r["kernels"]
    assert "preprocess_bwd_camera" in r["kernels"]


def test_public_api_zero_gaussians():
    cam, gs = _small_scene()
    gs = {k: (v[:0] if isinstance(v, torch.Tensor) else v) for k, v in gs.items()}
    r = _api(cam, gs, "cuda", colors=True)
    assert float(r["tx"].grad) == 0.0 and float(r["ty"].grad) == 0.0


def test_grad_bucket_refuses_focal_gradients():
    import gof_dp
    from diff_gaussian_rasterization import GaussianRasterizer
    cam, gs = _small_scene()
    dev = torch.device("cuda")
    rs = gof_synth.raster_settings(cam, gs["sh_degree"], dev)
    rs = rs._replace(tanfovx=torch.tensor(cam.tanfovx, requires_grad=True))
    P = gs["means3D"].shape[0]
    r = GaussianRasterizer(rs, grad_bucket=gof_dp.GradBucket(P, gs["shs"].shape[1], dev))
    p = {k: gs[k].to(dev) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    with pytest.raises(NotImplementedError):
        r(means3D=p["means3D"], means2D=torch.zeros_like(p["means3D"]), opacities=p["opacities"], shs=p["shs"], scales=p["scales"],
          rotations=p["rotations"])


def test_integrate_and_mark_visible_accept_tensor_tan_fov():
    from diff_gaussian_rasterization import GaussianRasterizer
    cam, gs = _small_scene(1500)
    dev = torch.device("cuda")
    rs = gof_synth.raster_settings(cam, gs["sh_degree"], dev)
    rs_t = rs._replace(tanfovx=torch.tensor(cam.tanfovx, device=dev, requires_grad=True),
                       tanfovy=torch.tensor(cam.tanfovy, dtype=torch.float64))
    p = {k: gs[k].to(dev) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    pts = p["means3D"][:300].contiguous()
    outs = []
    for s in (rs, rs_t):
        r = GaussianRasterizer(s)
        res = r.integrate(points3D=pts, means3D=p["means3D"], means2D=torch.zeros_like(p["means3D"]), opacities=p["opacities"],
                          shs=p["shs"], scales=p["scales"], rotations=p["rotations"])
        outs.append((res, r.markVisible(p["means3D"])))
    (a, va), (b, vb) = outs
    assert torch.equal(va, vb)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert not any(t.requires_grad for t in b)


# ---- descent -----------------------------------------------------------------------------------------------------------

def _skew(w):
    z = torch.zeros((), dtype=w.dtype, device=w.device)
    return torch.stack([torch.stack([z, -w[2], w[1]]), torch.stack([w[2], z, -w[0]]), torch.stack([-w[1], w[0], z])])


@pytest.mark.parametrize("with_pose", [False, True])
def test_focal_descent_recovers_a_perturbed_focal_length(with_pose):
    """The field of view of a ring camera, perturbed by +4 % in x and -3 % in y, is brought back by Adam on the two angles
    (tanfov = tan(fov / 2)) against the unperturbed render; the projection matrix follows without a gradient.  with_pose also
    turns the camera by 0.3 degree and moves it by 0.005, and refines a 6-dof pose delta in the same loop."""
    from diff_gaussian_rasterization import GaussianRasterizer
    dev = torch.device("cuda")
    cam, gs = gof_synth.make_scene(dict(P=20000, width=256, height=192, seed=8, sigma_px=4.0), view=2)
    p = {k: gs[k].to(dev) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    rs0 = gof_synth.raster_settings(cam, gs["sh_degree"], dev)
    proj0 = torch.linalg.inv(rs0.viewmatrix) @ rs0.projmatrix
    znear, zfar = 0.01, 100.0

    def render(vm, campos, tx, ty):
        value = lambda x: float(x.detach()) if torch.is_tensor(x) else float(x)   # noqa: E731
        proj = gof_synth._projection(znear, zfar, value(tx), value(ty)).t().to(dev)
        rs = rs0._replace(viewmatrix=vm, campos=campos, tanfovx=tx, tanfovy=ty, projmatrix=(vm.detach() @ proj).contiguous())
        color, _ = GaussianRasterizer(rs)(means3D=p["means3D"], means2D=torch.zeros_like(p["means3D"]), opacities=p["opacities"],
                                          shs=p["shs"], scales=p["scales"], rotations=p["rotations"])
        return color[:3]

    assert torch.allclose(gof_synth._projection(znear, zfar, cam.tanfovx, cam.tanfovy).t().to(dev), proj0, atol=1e-5)
    with torch.no_grad():
        target = render(rs0.viewmatrix, rs0.campos, cam.tanfovx, cam.tanfovy)
    fov_true = torch.tensor([2 * math.atan(cam.tanfovx), 2 * math.atan(cam.tanfovy)], dtype=torch.float64, device=dev)
    fov = (fov_true * torch.tensor([1.04, 0.97], dtype=torch.float64, device=dev)).requires_grad_(True)
    W2V = rs0.viewmatrix.t().double()
    start = W2V.clone()
    if with_pose:
        g = torch.Generator().manual_seed(4)
        axis, shift = torch.randn(3, generator=g, dtype=torch.float64), torch.randn(3, generator=g, dtype=torch.float64)
        Rp = torch.linalg.matrix_exp(_skew(math.radians(0.3) * axis / axis.norm())).to(dev)
        start[:3, :3] = Rp @ W2V[:3, :3]
        start[:3, 3] = Rp @ W2V[:3, 3] + 0.005 * (shift / shift.norm()).to(dev)
    w = torch.zeros(3, dtype=torch.float64, device=dev, requires_grad=with_pose)
    tau = torch.zeros(3, dtype=torch.float64, device=dev, requires_grad=with_pose)
    params = [{"params": [fov], "lr": 2e-3}] + ([{"params": [w, tau], "lr": 1e-3}] if with_pose else [])
    opt = torch.optim.Adam(params)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, 0.98)

    def fov_err():
        return float((fov.detach() / fov_true - 1).abs().max())

    e0 = fov_err()
    for _ in range(150):
        Rw = torch.linalg.matrix_exp(_skew(w))
        R, t = Rw @ start[:3, :3], Rw @ start[:3, 3] + tau
        M = torch.cat([torch.cat([R, t[:, None]], 1), torch.tensor([[0.0, 0.0, 0.0, 1.0]], dtype=R.dtype, device=dev)], 0)
        vm = M.t().float().contiguous()
        tan = torch.tan(0.5 * fov).float()
        loss = ((render(vm, (-R.t() @ t).float(), tan[0], tan[1]) - target) ** 2).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        sched.step()
    e1 = fov_err()
    print(f"focal error (with_pose={with_pose}): {e0:.4f} -> {e1:.5f} (relative, largest of x / y)")
    # thresholds: about 2x the measured residual with the pose, 30x alone (see the module docstring)
    assert e1 <= (0.015 if with_pose else 0.001), (e0, e1)
