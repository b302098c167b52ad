"""GPU: the camera gradient of the backward (gof_backward_out_t.dL_dviewmatrix / dL_dcampos, DESIGN.md 4.9).

(a) The 19 values against the float64 oracle (tests/_camera_oracle.py) fed with this backward's own dL_dview2gaussian and
    dL_dcolors, as test_gpu_grad_stagewise feeds the preprocess backward, over every scene of tests/_view_grad_scenes.py.  The
    backward is called with the pose, focal-length and ray outputs together (the joint scratch layout).  The allowance of each
    value is the sum over the visible Gaussians of the per-Gaussian allowance test_gpu_grad_stagewise gives dL_dmeans3D -- 2
    ulp of the Gaussian's term + 2^-30 of the largest term of its row + C_CHAIN 2^-53 of the magnitude of the ten dL_dv2g
    terms (view matrix), or C_SH 2^-24 of the SH magnitude (campos) -- plus half an ulp of the float result.  The oracle starts
    from the GPU's own per-Gaussian inputs, so no blend decision is exempted here (the marginal share is test (a) of
    test_gpu_focal_grad).  At SH degree 0, and with precomputed colours, dL_dcampos is exactly zero.  Largest error /
    allowance observed on an H100 80GB HBM3 (700 W power limit), view matrix / campos:
      sh_deg0..3 0.009-0.021 / 0-0.001, c1 0.012 / 3e-4, precomp_bg_mip 0.014 / 0, screen_filling 0.197 / 0.023,
      camera_inside 0.037 / 0.0015, near_plane 0.022 / 6e-4, stacked_* 0.006-0.026 / 5e-4, c2_v3 0.004 / 2e-4,
      c3_v5 0.001 / 4e-5, plain_1 / 33 / 4097 0.195 / 0.183 / 0.006 and 0.002 / 0.002 / 3e-4, saturation 0.077 / 0,
      threshold 0.038 / 0, rows_1..129 0.037-0.166 / 7e-4-0.0023, rows_8192 / 8193 / 8321 0.017 / 0.009 / 0.013 and
      <= 1e-3, image_* 0.003-0.168 / 8e-5-0.0074, ragged_4097 0.019 / 6e-4.
(b) Asking for the camera changes no other gradient, and the camera reduction is bit-reproducible.  The blend backward sums
    with double atomics, so two backward calls may round a Gaussian's accumulated gradient differently (test_gpu_repro);
    bit-identity is asserted wherever the blend stage's outputs are identical between the calls.
(c) Through the public API, .grad of viewmatrix / campos is what the ABI returns; projmatrix gets none; the precomputed
    colour / view2gaussian variants, P == 0 and the refusal with a grad_bucket.
(d) Descent: Adam on a 6-dof pose delta recovers a perturbed ring camera against the unperturbed render."""
import math

import numpy as np
import pytest
import torch

import _camera_oracle as co
import _grad_bounds as gb
import _util
import _view_grad_scenes as vs
import gof_synth
from test_gpu_grad_stagewise import C_CHAIN, C_SH, _ulp, sh_dmean_mag

pytestmark = pytest.mark.gpu

BLEND = ("dmeans2D", "dcolors", "dopacity", "dv2g")
NAMES = ("dmeans2D", "dcolors", "dopacity", "dmeans3D", "dcov3D", "dsh", "dscales", "drot", "dv2g")


def _forward(cam, gs, v2g=None, **kw):
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda")
    fa = list(_util.fwd_args(cam, gs, dev, **kw))
    if v2g is not None:
        fa[8] = v2g.to(dev)
    R, _color, radii, geom, binning, img = _C.rasterize_gaussians(*fa)
    return fa, R, radii, geom, binning, img


def _backward(fwd, dL, camera, intrinsics=False):
    from diff_gaussian_rasterization import _C
    fa, R, radii, geom, binning, img = fwd
    out = _C.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, dL), _camera=camera,
                                          _intrinsics=intrinsics, _ray_map=intrinsics)
    torch.cuda.synchronize()
    return [t.detach().clone() for t in out]


def _run(name, precomp=None):
    """Forward of scene `name` (precomp: None, "colors" or "v2g"), one backward with the pose, focal-length and ray outputs
    together; numpy results."""
    from diff_gaussian_rasterization import _C
    cam, gs, kw = vs.inputs(name, colors=precomp == "colors")
    P, W, H = gs["means3D"].shape[0], cam.image_width, cam.image_height
    v2g = None
    if precomp == "v2g":   # the records the forward computes, handed back in as view2gaussian_precomp
        f0 = _forward(cam, gs, **kw)
        v2g = _C.export_state(P, W, H, f0[1], f0[3], f0[4], f0[5], f0[2])["view2gaussian"].cpu()
    fwd = _forward(cam, gs, v2g, **kw)
    st = {k: v.cpu().numpy() for k, v in _C.export_state(P, W, H, fwd[1], fwd[3], fwd[4], fwd[5], fwd[2]).items()}
    dL = torch.randn(9, H, W, generator=torch.Generator().manual_seed(77)).cuda()
    g = [t.cpu().numpy() for t in _backward(fwd, dL, True, intrinsics=True)]
    return dict(got=dict(zip(NAMES, g[:9])), dvm=g[9].ravel(), dcp=g[10].ravel(), radii=fwd[2].cpu().numpy(), st=st,
                sc=vs.oracle_scene(cam, gs, kw, v2g), sh_degree=gs["sh_degree"])


def _allowance(r, t):
    """[15] summed per-Gaussian allowance of the camera terms t [P,15] (see the module docstring)."""
    sc, radii, st, g = r["sc"], r["radii"], r["st"], r["got"]
    vis = radii > 0
    tv = t[vis]
    allow = np.zeros(15)
    a = sc.arr
    if a["v2g_precomp"] is None:
        dv = g["dv2g"][vis].astype(np.float64)
        jmag = np.zeros((int(vis.sum()), 12))
        for k in range(10):
            e = np.zeros_like(dv)
            e[:, k] = 1.0
            jmag += np.abs(co.vm_terms(a["viewmatrix"], a["means3D"][vis], a["scales"][vis], a["rotations"][vis], e)) * np.abs(dv[:, k:k + 1])
        row = np.abs(tv[:, :12]).max(axis=1, keepdims=True)
        allow[:12] = (2.0 * _ulp(tv[:, :12]) + 2.0 ** -30 * row + C_CHAIN * 2.0 ** -53 * jmag).sum(axis=0)
    if a["shs"] is not None:
        dRGB = np.where(st["clamped"].astype(bool), 0.0, g["dcolors"].astype(np.float64))[vis]
        msh = sh_dmean_mag(a["means3D"][vis], a["cam_pos"], a["shs"][vis], sc.D, dRGB)
        row = np.abs(tv[:, 12:]).max(axis=1, keepdims=True)
        allow[12:] = (2.0 * _ulp(tv[:, 12:]) + 2.0 ** -30 * row + C_SH * gb.EPS * msh).sum(axis=0)
    return allow


def _pose_ratio(r):
    """(largest |gpu - oracle| / bound over the 19 values, {what: (gpu, oracle, bound)}) of one run, checking nothing."""
    t = co.terms(r["sc"], r["radii"], r["st"]["clamped"], r["got"]["dcolors"], r["got"]["dv2g"])
    ovm, ocp = co.assemble(t.sum(axis=0))
    allow_vm, allow_cp = co.assemble(_allowance(r, t))
    out, worst = {}, {}
    for what, got, ora, allow in (("viewmatrix", r["dvm"], ovm, allow_vm), ("campos", r["dcp"], ocp, allow_cp)):
        bound = allow + 0.5 * _ulp(ora)
        err = np.abs(got.astype(np.float64) - ora)
        worst[what] = float(np.where(err > 0, err / np.where(bound > 0, bound, 1), 0.0).max())
        out[what] = (got, ora, bound)
    return worst, out


@pytest.mark.parametrize("name", list(vs.SCENES))
def test_camera_gradient_against_the_fp64_oracle(name):
    r = _run(name)
    worst, out = _pose_ratio(r)
    print(f"{name}: largest |gpu - oracle| / allowance: view matrix {worst['viewmatrix']:.3g}, campos {worst['campos']:.3g} "
          f"(SH degree {r['sh_degree']}, {int((r['radii'] > 0).sum())} visible Gaussians)")
    assert (r["dvm"][3::4] == 0).all()
    gvm, ovm, bvm = out["viewmatrix"]
    assert (np.abs(gvm - ovm) <= bvm).all(), ("viewmatrix", gvm, ovm, bvm)
    assert np.abs(ovm).max() > 0 and np.abs(gvm).max() > 0
    gcp, ocp, bcp = out["campos"]
    if r["sh_degree"] == 0 or r["sc"].arr["shs"] is None:   # the colour does not depend on the view direction: exact zeros
        assert (ocp == 0).all() and (gcp == 0).all(), gcp
    else:
        assert (np.abs(gcp - ocp) <= bcp).all(), ("campos", gcp, ocp, bcp)
        assert np.abs(ocp).max() > 0


@pytest.mark.parametrize("precomp", ["colors", "v2g"])
def test_precomputed_inputs_zero_their_part(precomp):
    r = _run("ragged_4097", precomp)
    t = co.terms(r["sc"], r["radii"], r["st"]["clamped"], r["got"]["dcolors"], r["got"]["dv2g"])
    ovm, ocp = co.assemble(t.sum(axis=0))
    allow_vm, allow_cp = co.assemble(_allowance(r, t))
    if precomp == "colors":
        assert (r["dcp"] == 0).all() and np.abs(r["dvm"]).max() > 0
        assert (np.abs(r["dvm"] - ovm) <= allow_vm + 0.5 * _ulp(ovm)).all()
    else:
        assert (r["dvm"] == 0).all() and np.abs(r["dcp"]).max() > 0
        assert (np.abs(r["dcp"] - ocp) <= allow_cp + 0.5 * _ulp(ocp)).all()


def _bits(a):
    return a.contiguous().view(torch.int32)


@pytest.mark.parametrize("name", list(vs.SCENES))
def test_other_gradients_unchanged_and_camera_reproducible(name):
    cam, gs, kw = vs.inputs(name)
    fwd = _forward(cam, gs, **kw)
    dL = torch.randn(9, cam.image_height, cam.image_width, generator=torch.Generator().manual_seed(3)).cuda()
    plain, with_cam, again = _backward(fwd, dL, False), _backward(fwd, dL, True), _backward(fwd, dL, True)
    assert len(plain) == 9 and len(with_cam) == 11
    P = gs["means3D"].shape[0]
    vis = fwd[2] > 0

    def same_blend(x, y):   # [P] bool: every blend-stage output of the Gaussian is bitwise equal in x and y
        m = torch.ones(P, dtype=torch.bool, device=vis.device)
        for n in BLEND:
            i = NAMES.index(n)
            m &= (_bits(x[i]).view(P, -1) == _bits(y[i]).view(P, -1)).all(dim=1)
        return m

    same = same_blend(plain, with_cam)
    assert float((~same & vis).sum()) <= 1e-3 * float(vis.sum())
    for i, n in enumerate(NAMES):
        a, b = plain[i], with_cam[i]
        if n in BLEND:
            assert _util.same_up_to_summation_order(b, a), n
        elif a.numel():
            assert torch.equal(_bits(a).view(P, -1)[same], _bits(b).view(P, -1)[same]), n
    if bool(same_blend(with_cam, again).all()):
        assert torch.equal(_bits(with_cam[9]), _bits(again[9])) and torch.equal(_bits(with_cam[10]), _bits(again[10]))
    else:   # the two calls' blend stages rounded some Gaussian differently: the camera sums then differ by as little
        for i in (9, 10):
            assert _util.same_up_to_summation_order(again[i], with_cam[i])


# ---- the public API ----------------------------------------------------------------------------------------------------

def _api(cam, gs, precomp=None, camera=True, P=None):
    """Render + backward through GaussianRasterizer; returns (settings tensors, parameter tensors, launched kernel names)."""
    from diff_gaussian_rasterization import GaussianRasterizer, _C
    dev = torch.device("cuda")
    rs = gof_synth.raster_settings(cam, gs["sh_degree"], dev)
    vm, cp, pm = (t.clone().requires_grad_(camera) for t in (rs.viewmatrix, rs.campos, rs.projmatrix))
    rs = rs._replace(viewmatrix=vm, campos=cp, projmatrix=pm)
    p = {k: gs[k].to(dev).requires_grad_(True) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    means2D = torch.zeros_like(p["means3D"], requires_grad=True)
    kw = dict(shs=p["shs"])
    if precomp == "colors":
        kw = dict(colors_precomp=gs["colors"].to(dev))
    elif precomp == "v2g":
        kw["view2gaussian_precomp"] = gs["v2g"].to(dev)
    _C.profile_reset()
    _C.profile_enable(True)
    color, _radii = GaussianRasterizer(rs)(means3D=p["means3D"], means2D=means2D, opacities=p["opacities"], scales=p["scales"],
                                           rotations=p["rotations"], **kw)
    dL = torch.randn(9, cam.image_height, cam.image_width, generator=torch.Generator().manual_seed(9))
    (color * dL.to(dev)).sum().backward()
    torch.cuda.synchronize()
    kernels = set(_C.profile_report())
    _C.profile_enable(False)
    return dict(vm=vm, cp=cp, pm=pm, p=p, means2D=means2D, dL=dL, kernels=kernels)


def _small_scene(precomp=None, P=4000):
    from diff_gaussian_rasterization import _C
    cam, gs = gof_synth.make_scene(dict(P=P, width=160, height=104, seed=5), view=7)
    if precomp == "colors":
        gs["colors"] = torch.rand(P, 3, generator=torch.Generator().manual_seed(2))
    elif precomp == "v2g":
        fwd = _forward(cam, gs)
        gs["v2g"] = _C.export_state(P, cam.image_width, cam.image_height, fwd[1], fwd[3], fwd[4], fwd[5], fwd[2])["view2gaussian"].cpu()
    return cam, gs


@pytest.mark.parametrize("precomp", [None, "colors", "v2g"])
def test_public_api_camera_grad_is_the_abi_output(precomp):
    cam, gs = _small_scene(precomp)
    r = _api(cam, gs, precomp)
    assert "preprocess_bwd_camera" in r["kernels"] and "camera_grad_sum" in r["kernels"] and "preprocess_bwd" not in r["kernels"]
    assert r["pm"].grad is None
    vmg, cpg = r["vm"].grad, r["cp"].grad
    assert vmg.shape == (4, 4) and cpg.shape == (3,)
    # the same render and backward through the ABI
    fwd = _forward(cam, gs, gs.get("v2g"), colors_precomp=gs.get("colors"))
    g = _backward(fwd, r["dL"].cuda(), True)
    api = {"dmeans2D": r["means2D"].grad, "dopacity": r["p"]["opacities"].grad, "dmeans3D": r["p"]["means3D"].grad,
           "dscales": r["p"]["scales"].grad, "drot": r["p"]["rotations"].grad}
    if precomp != "colors":
        api["dsh"] = r["p"]["shs"].grad
    if all(torch.equal(_bits(api[n]), _bits(g[NAMES.index(n)])) for n in api):
        assert torch.equal(_bits(vmg), _bits(g[9])) and torch.equal(_bits(cpg), _bits(g[10]))
    else:   # the blend stage rounded some Gaussian differently in the two calls (see the module docstring)
        assert _util.same_up_to_summation_order(vmg, g[9]) and _util.same_up_to_summation_order(cpg, g[10])
    if precomp == "colors":
        assert (cpg == 0).all() and vmg.abs().max() > 0
    elif precomp == "v2g":
        assert (vmg == 0).all() and cpg.abs().max() > 0
    else:
        assert vmg.abs().max() > 0 and cpg.abs().max() > 0
    assert (vmg[:, 3] == 0).all()


def test_public_api_without_camera_grad_runs_the_plain_backward():
    cam, gs = _small_scene()
    r = _api(cam, gs, camera=False)
    assert "preprocess_bwd" in r["kernels"] and "preprocess_bwd_camera" not in r["kernels"]
    assert r["vm"].grad is None and r["cp"].grad is None


def test_public_api_zero_gaussians():
    # precomputed colours: with P == 0 the binding sizes dL_dsh (P, 0, 3), which autograd refuses for a (0, 16, 3) input
    cam, gs = _small_scene("colors")
    gs = {k: (v[:0] if isinstance(v, torch.Tensor) else v) for k, v in gs.items()}
    r = _api(cam, gs, "colors")
    assert torch.equal(r["vm"].grad, torch.zeros(4, 4, device="cuda")) and torch.equal(r["cp"].grad, torch.zeros(3, device="cuda"))


def test_grad_bucket_refuses_camera_gradients():
    import gof_dp
    from diff_gaussian_rasterization import GaussianRasterizer
    cam, gs = _small_scene()
    dev = torch.device("cuda")
    rs = gof_synth.raster_settings(cam, gs["sh_degree"], dev)
    rs = rs._replace(viewmatrix=rs.viewmatrix.clone().requires_grad_(True))
    P = gs["means3D"].shape[0]
    r = GaussianRasterizer(rs, grad_bucket=gof_dp.GradBucket(P, gs["shs"].shape[1], dev))
    p = {k: gs[k].to(dev) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    with pytest.raises(NotImplementedError):
        r(means3D=p["means3D"], means2D=torch.zeros_like(p["means3D"]), opacities=p["opacities"], shs=p["shs"], scales=p["scales"],
          rotations=p["rotations"])


# ---- descent -----------------------------------------------------------------------------------------------------------

def _skew(w):
    z = torch.zeros((), dtype=w.dtype, device=w.device)
    return torch.stack([torch.stack([z, -w[2], w[1]]), torch.stack([w[2], z, -w[0]]), torch.stack([-w[1], w[0], z])])


def test_pose_descent_recovers_a_perturbed_camera():
    """A ring camera turned by 0.5 degree and moved by 0.01 (the ring's radius is 4) is brought back by Adam on a 6-dof
    delta (rotation vector w, translation tau: W2V = [exp(w) R | exp(w) t + tau]) against the unperturbed render; the
    projection matrix follows the pose without a gradient.  Reached on an H100 80GB HBM3 (700 W power limit): rotation
    0.500 -> 0.072 degree, camera centre 0.0100 -> 0.0033."""
    from diff_gaussian_rasterization import GaussianRasterizer
    dev = torch.device("cuda")
    cam, gs = gof_synth.make_scene(dict(P=20000, width=256, height=192, seed=8, sigma_px=4.0), view=2)
    p = {k: gs[k].to(dev) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    rs0 = gof_synth.raster_settings(cam, gs["sh_degree"], dev)
    proj = torch.linalg.inv(rs0.viewmatrix) @ rs0.projmatrix          # the projection part of full_proj_transform

    def render(vm, campos):
        rs = rs0._replace(viewmatrix=vm, campos=campos, projmatrix=(vm.detach() @ proj).contiguous())
        color, _ = GaussianRasterizer(rs)(means3D=p["means3D"], means2D=torch.zeros_like(p["means3D"]), opacities=p["opacities"],
                                          shs=p["shs"], scales=p["scales"], rotations=p["rotations"])
        return color[:3]

    with torch.no_grad():
        target = render(rs0.viewmatrix, rs0.campos)
    W2V = rs0.viewmatrix.t().double()                                  # column-vector world -> view
    g = torch.Generator().manual_seed(4)
    axis = torch.randn(3, generator=g, dtype=torch.float64)
    shift = torch.randn(3, generator=g, dtype=torch.float64)
    Rp = torch.linalg.matrix_exp(_skew(math.radians(0.5) * axis / axis.norm()))
    start = torch.eye(4, dtype=torch.float64)
    start[:3, :3] = Rp @ W2V[:3, :3].cpu()
    start[:3, 3] = Rp @ W2V[:3, 3].cpu() + 0.01 * shift / shift.norm()
    start = start.to(dev)

    def pose(w, tau):
        R = torch.linalg.matrix_exp(_skew(w)) @ start[:3, :3]
        t = torch.linalg.matrix_exp(_skew(w)) @ start[:3, 3] + tau
        return R, t

    def error(R, t):
        Rg, tg = W2V[:3, :3], W2V[:3, 3]
        ang = float(torch.arccos(((torch.trace(R @ Rg.t()) - 1) / 2).clamp(-1, 1)))
        centre = float(((-R.t() @ t) - (-Rg.t() @ tg)).norm())
        return math.degrees(ang), centre

    w = torch.zeros(3, dtype=torch.float64, device=dev, requires_grad=True)
    tau = torch.zeros(3, dtype=torch.float64, device=dev, requires_grad=True)
    opt = torch.optim.Adam([w, tau], lr=1e-3)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, 0.98)
    e0 = error(*pose(w.detach(), tau.detach()))
    for _ in range(150):
        R, t = pose(w, tau)
        M = torch.cat([torch.cat([R, t[:, None]], 1), torch.tensor([[0.0, 0.0, 0.0, 1.0]], dtype=R.dtype, device=dev)], 0)
        vm = M.t().float().contiguous()
        campos = (-R.t() @ t).float()
        loss = ((render(vm, campos) - target) ** 2).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        sched.step()
    e1 = error(*pose(w.detach(), tau.detach()))
    print(f"pose error: rotation {e0[0]:.4f} -> {e1[0]:.4f} deg, camera centre {e0[1]:.5f} -> {e1[1]:.5f}")
    assert e1[0] <= 0.5 * e0[0] and e1[1] <= 0.5 * e0[1], (e0, e1)
