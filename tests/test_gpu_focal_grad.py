"""GPU: the focal-length gradient of the backward (gof_backward_out_t.dL_dtan_fov, DESIGN.md 4.10).

(a) Every pixel's dL/drx, dL/dry (the [2,H,W] map the call leaves in its scratch) against the float64 oracle
    (tests/focal_oracle/focal_oracle.c) run from this library's own forward state with the same dL_dpix, over every scene of
    tests/_view_grad_scenes.py, from a call that also asks for the pose (the joint scratch layout):

        |gpu - oracle|  <=  (C_PAIR + C_RAYS (1 + L)) * 2^-24 * mag  +  marginal,      L = the view's longest walk,

    the model of tests/_grad_bounds.py: T is recovered pair by pair on the GPU, which drifts by about one ulp per pair, and a
    pair near a blend threshold exempts every pair in front of it; at most SHARE_MARGINAL of the pixels may carry marginal
    mass.  C_PAIR is the part that does not grow with the walk: each pair's dL/dr is a five-term float FMA chain of the float
    dA, dB2 and dnrm, about one ulp of its magnitude.  At walks of hundreds of pairs C_RAYS (1 + L) covers it; at walks of
    1-35 pairs (the scenes with P <= 129) it did not (need 0.92 at plain_33, L = 3).  Both sums against the oracle's within
    the sum over the pixels of |rx| (|ry|) times the pixel's allowance, over tan_fov, plus half an ulp; and, because that
    allowance is loose (a sum that missed half its tiles passed it at C2), against the float64 sum of the call's own ray map
    within half an ulp + 2^-46 of the sum of |rx dL/drx|: the tile sums and k_focal_grad_sum add in double and round once.
    Observed on an H100 80GB HBM3 (700 W power limit), largest |gpu - oracle - marginal| / (2^-24 (1 + L) mag), share of
    pixels with marginal mass:
      sh_deg0..3 (L 319-357) 0.003-0.005, 0;  c1 0.008, 1.5e-5;  precomp_bg_mip 0.005, 4.2e-5;  screen_filling 0.024, 0;
      camera_inside / near_plane 0.003 / 0.004, 0;  stacked_* (L 888-1019) 0.001, 0;  c2_v3 0.0017, 1.3e-5;
      c3_v5 0.0015, 2.7e-5;  plain_4097 0.010, 0;  saturation 0.009, 0;  threshold 0.010, 1.6e-4;  rows_8192..8321 <= 5e-4, 0;
      image_* 0.0013-0.017, <= 1.5e-5;  ragged_4097 0.0055, 0;  and C_PAIR needed at the short walks: plain_1 / 33 0.52 /
      0.92, rows_1 / 127 / 128 / 129 0.42 / 0.61 / <= 0.45.  Sums: largest error / oracle allowance 3e-4, largest error /
      own-sum bound 0.996 (the float rounding itself).  The per-pixel values go through no atomics: the same on every run.
(b) Two calls give identical bits; every other output, the pose gradient included, is bit-identical with and without the
    intrinsics outputs wherever the blend's outputs are identical (the blend backward sums with double atomics, see
    test_gpu_camera_grad (b)).
(c) Through the public API, .grad of tanfovx / tanfovy (CPU or CUDA 0-dim tensors) is the ABI output; joint use with the
    view matrix; float settings still run the plain kernels; P == 0; the refusal with a grad_bucket; integrate and
    markVisible accept tensor tan_fov values.
(d) Descent: Adam on the field of view recovers a perturbed focal length against the unperturbed render, alone and together
    with a pose perturbation.  Reached on an H100 80GB HBM3 (700 W power limit): largest relative field-of-view error
    0.040 -> 0.00003 alone, 0.040 -> 0.0071 together with the pose.
(e) The caller's scratch, through gof_rasterize_backward_ex directly: a guard band after exactly the size the library asks
    for stays intact, and outputs do not depend on the scratch's or the outputs' previous contents."""
import math

import numpy as np
import pytest
import torch

import _focal_oracle as fo
import _grad_bounds as gb
import _util
import _view_grad_scenes as vs
import gof_synth

pytestmark = pytest.mark.gpu

C_RAYS = 2.0 ** -5   # 4x the largest ratio observed (0.0055, ragged_4097), rounded up to a power of two
C_PAIR = 4.0         # 4x the largest need observed at short walks (0.92, plain_33, L = 3), rounded up to a power of two
SHARE_MARGINAL = 0.01   # at most this share of the pixels may carry marginal mass (as test_gpu_forward_edges)
NAMES = ("dmeans2D", "dcolors", "dopacity", "dmeans3D", "dcov3D", "dsh", "dscales", "drot", "dv2g")
BLEND = ("dmeans2D", "dcolors", "dopacity", "dv2g")


def _forward(cam, gs, **kw):
    from diff_gaussian_rasterization import _C
    fa = _util.fwd_args(cam, gs, torch.device("cuda"), **kw)
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


@pytest.mark.parametrize("name", list(vs.SCENES))
def test_ray_gradient_against_the_fp64_oracle(name):
    from diff_gaussian_rasterization import _C
    cam, gs, kw = vs.inputs(name)
    P, W, H = gs["means3D"].shape[0], cam.image_width, cam.image_height
    fwd = _forward(cam, gs, **kw)
    st = {k: v.cpu().numpy() for k, v in _C.export_state(P, W, H, fwd[1], fwd[3], fwd[4], fwd[5], fwd[2]).items()}
    dL = torch.randn(9, H, W, generator=torch.Generator().manual_seed(41))
    g = _backward(fwd, dL.cuda(), camera=True, intrinsics=True, ray_map=True)   # the pose outputs too: the joint scratch layout
    gx, gy, rays = float(g[11]), float(g[12]), g[13].cpu().numpy()
    d = fo.rays(W, H, cam.tanfovx, cam.tanfovy, st, np.asarray(kw["bg"], np.float32), dL.numpy(), float_geometry=True)
    L = int(st["n_contrib"][0].max())
    allow = (C_PAIR + C_RAYS * (1.0 + L)) * gb.EPS * d["mag"] + d["marginal"]
    err = np.abs(rays - d["drays"])
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(err > 0, np.maximum(err - d["marginal"], 0.0) / (gb.EPS * (1.0 + L) * d["mag"]), 0.0)
        need = np.where(err > 0, np.maximum(err - d["marginal"] - C_RAYS * gb.EPS * (1.0 + L) * d["mag"], 0.0) / (gb.EPS * d["mag"]), 0.0)
    share = float((d["marginal"].sum(axis=0) > 0).mean())
    print(f"{name}: L = {L}, largest per-pixel |gpu - oracle - marginal| / (2^-24 (1 + L) mag) = {float(ratio.max()):.3g}, "
          f"C_PAIR needed {float(need.max()):.3g}, pixels with marginal mass {share:.2e}")
    assert (err <= allow).all(), (float(need.max()), np.unravel_index(np.argmax(need), need.shape))
    assert share <= SHARE_MARGINAL, share
    assert np.abs(d["drays"]).max() > 0
    # the sums
    rx, ry = fo.pixel_rays(W, H, cam.tanfovx, cam.tanfovy)
    ox, oy = fo.tan_fov_grad(d["drays"], cam.tanfovx, cam.tanfovy)
    ax = float((np.abs(rx.astype(np.float64))[None, :] * allow[0]).sum()) / float(np.float32(cam.tanfovx))
    ay = float((np.abs(ry.astype(np.float64))[:, None] * allow[1]).sum()) / float(np.float32(cam.tanfovy))
    # the reduction alone: the fp64 sums of this call's own ray map, which k_render_backward<true>'s tile sums and
    # k_focal_grad_sum add in double (at most ~30 levels of double rounding) and round to float once
    tx, ty = float(np.float32(cam.tanfovx)), float(np.float32(cam.tanfovy))
    wx, wy = rx.astype(np.float64)[None, :] * rays[0], ry.astype(np.float64)[:, None] * rays[1]
    for what, got, ora, a, n, w, tan in (("tanfovx", gx, ox, ax, W, wx, tx), ("tanfovy", gy, oy, ay, H, wy, ty)):
        bound = a + 0.5 * _ulp(ora)
        own = float(w.sum()) / tan
        tight = 0.5 * _ulp(max(abs(own), abs(got))) + 2.0 ** -46 * float(np.abs(w).sum()) / tan
        print(f"{name} {what}: gpu {got:.9g} oracle {ora:.9g}, |gpu - oracle| / allowance = {abs(got - ora) / bound:.3g}, "
              f"|gpu - sum of its ray map| / (half an ulp + 2^-46 sum|r dL/dr|) = {abs(got - own) / tight if tight else 0.0:.3g}")
        if n == 1:   # the one pixel's ray is the optical axis: rx = 0 (ry = 0), and so is the sum
            assert got == 0.0 and ora == 0.0, (what, got, ora)
            continue
        assert abs(got - own) <= tight, (what, got, own, tight)
        assert abs(got - ora) <= bound, (what, got, ora, bound)
        assert ora != 0.0


def _bits(a):
    return a.contiguous().view(torch.int32)


def _same_blend(x, y, P):
    """[P] bool: every blend-stage output of the Gaussian is bitwise equal in the gradient lists x and y."""
    m = torch.ones(P, dtype=torch.bool, device=x[0].device)
    for n in BLEND:
        i = NAMES.index(n)
        m &= (_bits(x[i]).view(P, -1) == _bits(y[i]).view(P, -1)).all(dim=1)
    return m


@pytest.mark.parametrize("name", list(vs.SCENES))
def test_reproducible_and_other_outputs_unchanged(name):
    cam, gs, kw = vs.inputs(name)
    fwd = _forward(cam, gs, **kw)
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
    for other in (both, fov_only):
        same = _same_blend(plain, other, P)
        assert float((~same & vis).sum()) <= 1e-3 * float(vis.sum())
        for i, n in enumerate(NAMES):
            a, b = plain[i], other[i]
            if n in BLEND:
                assert _util.same_up_to_summation_order(b, a), n
            elif a.numel():
                assert torch.equal(_bits(a).view(P, -1)[same], _bits(b).view(P, -1)[same]), n
    if bool(_same_blend(plain, both, P).all()):
        assert torch.equal(_bits(plain[9]), _bits(both[9])) and torch.equal(_bits(plain[10]), _bits(both[10]))
    else:
        for i in (9, 10):
            assert _util.same_up_to_summation_order(both[i], plain[i])


# ---- the caller's scratch ----------------------------------------------------------------------------------------------

GUARD = 64 * 1024


def _backward_ex(fwd, dL, camera, intrinsics, fill):
    """gof_rasterize_backward_ex called directly, with every output and a scratch of exactly
    gof_rasterize_backward_scratch_bytes(P, W, H, camera, intrinsics) bytes followed by a GUARD-byte band, all pre-filled with
    the byte `fill`.  Returns (the nine gradients, the camera [19] or None, the focal sums [2] or None, the ray map [2,H,W] or
    None, the scratch buffer, its size)."""
    import ctypes
    from diff_gaussian_rasterization import _C
    fa, R, radii, geom, binning, img = fwd
    (bg, means3D, colors, _opacity, scales, rotations, sm, cov3D, v2g, vm, pm, tfx, tfy, ks, subpix, H, W, sh, deg, campos,
     _prefiltered, _debug) = fa
    keep = []
    s = _C._scene(keep, bg, means3D, colors, means3D, scales, rotations, sm, cov3D, v2g, vm, pm, tfx, tfy, ks, subpix, H, W, sh, deg,
                  campos, False, False)
    P, M, dev = means3D.shape[0], s.M, means3D.device
    filled = lambda n, dt=torch.float32: torch.full((n,), fill, dtype=torch.uint8, device=dev).view(dt)   # noqa: E731
    grads = [filled(4 * P * k) for k in (3, 3, 1, 3, 6, 3 * M, 3, 4, 10)]
    cam, fov = filled(4 * 19), filled(4 * 2)
    need = int(_C._lib.gof_rasterize_backward_scratch_bytes(P, W, H, int(camera), int(intrinsics)))
    scratch = filled(need + GUARD, torch.uint8)
    o = _C._BackwardOut(dL_dmean2D=grads[0].data_ptr(), dL_dcolor=grads[1].data_ptr(), dL_dopacity=grads[2].data_ptr(),
                        dL_dmean3D=grads[3].data_ptr(), dL_dcov3D=grads[4].data_ptr(), dL_dsh=grads[5].data_ptr() if M else None,
                        dL_dscale=grads[6].data_ptr(), dL_drot=grads[7].data_ptr(), dL_dview2gaussian=grads[8].data_ptr(),
                        dL_dviewmatrix=cam.data_ptr() if camera else None, dL_dcampos=cam.data_ptr() + 64 if camera else None,
                        dL_dtan_fov=fov.data_ptr() if intrinsics else None, scratch=scratch.data_ptr(), scratch_bytes=need)
    g = dL.contiguous()
    _C._check(_C._lib.gof_rasterize_backward_ex(ctypes.byref(s), int(R), radii.data_ptr(), geom.data_ptr(),
                                                 binning.data_ptr() if binning.numel() else None, img.data_ptr(), g.data_ptr(),
                                                 ctypes.byref(o), _C._stream()))
    torch.cuda.synchronize()
    rays = None
    if intrinsics:
        off = need - 16 * (W * H + ((W + 15) // 16) * ((H + 15) // 16))
        rays = scratch[off:off + 16 * W * H].view(torch.float64).view(2, H, W).clone()
    return grads, cam if camera else None, fov if intrinsics else None, rays, scratch, need


def _camera_rows(P):
    return (P + 127) // 128


@pytest.mark.parametrize("P", [1, 128, 129, 64 * 128 + 1])
@pytest.mark.parametrize("W,H", [(16, 16), (400, 656)])
def test_scratch_bounds_and_initialisation(P, W, H):
    """With the pose outputs, the focal-length outputs, both or neither: nothing is written past the scratch size the library
    asks for (the guard band keeps its fill), and no output depends on what the scratch or the outputs held before the call
    (pre-filled with 0x00 and with 0xFF, the pose, focal and ray outputs are bit-identical wherever the blend's outputs are;
    the ray map and the focal sums always).  P = 1 and 128 have one camera row, which the joint layout pads from 128 to 256
    bytes, and 8 193 has 65; W x H = 16 x 16 is one tile, 400 x 656 is 1 025.  The pose outputs are also the fp64
    sum of the camera rows left in the scratch, rounded to float."""
    cam, gs = gof_synth.make_scene(dict(P=P, width=W, height=H, seed=90 + P), view=3)
    fwd = _forward(cam, gs)
    assert int((fwd[2] > 0).sum()) > 0
    dL = torch.randn(9, H, W, generator=torch.Generator().manual_seed(6)).cuda()
    for camera in (False, True):
        for intrinsics in (False, True):
            runs = []
            for fill in (0x00, 0xFF):
                r = _backward_ex(fwd, dL, camera, intrinsics, fill)
                scratch, need = r[4], r[5]
                assert bool((scratch[need:] == fill).all()), (camera, intrinsics, fill, "write past the end of the scratch")
                runs.append(r)
            (g0, c0, f0, r0, _, _), (g1, c1, f1, r1, _, _) = runs
            for t in g0 + g1:   # every gradient element was written
                assert not bool(torch.isnan(t).any())
            same = bool(_same_blend(g0, g1, P).all())
            if camera:   # k_camera_grad_sum against the fp64 sum of the rows it read (at the front of the scratch)
                rows = runs[0][4][:_camera_rows(P) * 128].view(torch.float64).view(-1, 16).cpu().numpy()
                tot, mag = rows.sum(axis=0), np.abs(rows).sum(axis=0)
                want = np.concatenate([np.stack([tot[3 * k:3 * k + 3] for k in range(4)], 0), np.zeros((4, 1))], 1).ravel()
                want = np.concatenate([want, tot[12:15]])
                wmag = np.concatenate([np.concatenate([np.stack([mag[3 * k:3 * k + 3] for k in range(4)], 0), np.zeros((4, 1))], 1).ravel(),
                                       mag[12:15]])
                got = c0.cpu().numpy().astype(np.float64)
                assert (np.abs(got - want) <= 0.5 * _ulp(want) + 2.0 ** -46 * wmag).all(), (got, want)
            if camera and same:
                assert torch.equal(_bits(c0), _bits(c1)), (camera, intrinsics)
            elif camera:   # the blend's double atomics rounded some Gaussian differently (test (b))
                assert _util.same_up_to_summation_order(c0, c1), (camera, intrinsics)
            if intrinsics:
                assert torch.equal(_bits(f0), _bits(f1)) and torch.equal(r0.view(torch.int64), r1.view(torch.int64))
                assert bool(torch.isfinite(r0).all())


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
