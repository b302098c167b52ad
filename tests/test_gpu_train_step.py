"""The kernels a training step runs around the rasterizer, at the shapes the step runs them, against plain fp64 references:

  conv_wgrad  (csrc/conv_wgrad.cu)  the appearance network's weight / bias gradient: 9 shifted matmuls in fp64.  With inputs in
              {-1, 0, 1} every partial sum the kernel forms is an integer below 2^24, so dW and db must be EXACT whatever the
              summation order; at production shapes every CTA of the persistent grid walks >= 3 tiles, so the cp.async
              prefetch, the buffer swap and the refill barrier all run.
  view_loss   (csrc/view_loss.cu)   the fused per-view loss against oracle/loss_oracle.py (numpy fp64), ragged and 1080p.
  param_ops   (csrc/param_ops.cu)   activate / its backward / Adam against fp64 torch restatements of param_ops.cuh, up to
              10^6 Gaussians and 59 M Adam elements; misaligned rotations.
  filter3d    (csrc/filter3d.cu)    compute_3D_filter against an fp64 restatement, 10^6 points and 200 cameras.

Tests without the gpu mark check the fp64 helpers themselves (against torch's own conv2d_weight and against the goldens the
reference's Python wrote) and the C ABI's refusal of misaligned rotations; they run without a device.

Rounding bounds are stated as |gpu - fp64| <= c * 2^-24 * scale, scale = the sum of the magnitudes of the operation's terms
(so that cancellation does not shrink the allowance below what one rounding of an operand can move); each c is given where
it is used, with how it was chosen."""
import ctypes
import json
import math
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB_PATH = os.path.join(ROOT, "gaussian-opacity-fields_b200", "diff_gaussian_rasterization", "libgof_b200.so")
EPS = 2.0 ** -24
GOF_OK, GOF_E_INVALID, GOF_E_CUDA = 0, -1, -2
gpu = pytest.mark.gpu


def _ulp32(x):
    """fp32 ulp at |x| (x float64 tensor); 2^-149 at zero."""
    m, e = torch.frexp(x.abs())
    return torch.where(x == 0, torch.full_like(x, 2.0 ** -149), torch.ldexp(torch.ones_like(x), (e - 24).clamp(min=-149)))


def _ratio(got, ref, scale):
    """max |got - ref| / (2^-24 * scale) over the elements (0 where both agree, inf where scale is 0 and they differ)."""
    d = (got.detach().double() - ref).abs()
    s = EPS * scale
    r = torch.where(d > 0, d / torch.where(s > 0, s, torch.ones_like(s)), torch.zeros_like(d))
    r = torch.where((d > 0) & (s == 0), torch.full_like(d, math.inf), r)
    return float(r.max()) if r.numel() else 0.0


# ========================================================================================================================
# 1. conv_wgrad
# ========================================================================================================================

def conv_wgrad_ref(x, gy):
    """dW[co, ci, ky, kx] = sum_p gy[co, p] * x[ci, p + (ky-1, kx-1)] (zero outside the image), db[co] = sum_p gy[co, p]:
    nine shifted matmuls in the inputs' dtype (float64 here).  x [CI,H,W], gy [CO,H,W]."""
    CI, H, W = x.shape
    CO = gy.shape[0]
    xp = torch.nn.functional.pad(x, (1, 1, 1, 1))
    g = gy.reshape(CO, H * W)
    dW = torch.empty((CO, CI, 3, 3), dtype=x.dtype, device=x.device)
    for ky in range(3):
        for kx in range(3):
            dW[:, :, ky, kx] = g @ xp[:, ky:ky + H, kx:kx + W].reshape(CI, H * W).t()
    return dW, g.sum(1)


# Mirror of conv_wgrad.cu: TW x TH pixel tiles, the instantiation (COPT, RG) of each channel pair, TileLayout's floats per buffer.
TW, TH = 32, 8
_INST = {(16, 16): (4, 4), (3, 16): (3, 8), (16, 8): (4, 8)}       # (CO, CI) -> (COPT, RG)
_SMEM_RESERVED = 1024       # shared memory the driver reserves per CTA on sm_90 (cudaDevAttrReservedSharedMemoryPerBlock)


def _tile_floats(co, ci, pipe):
    xp = (TH + 2) * 40 + 4 if pipe else (TH + 2) * (TW + 3)
    gp = TH * 36 + 4 if pipe else TH * (TW + 1) + 1
    return ci * xp + co * gp


def conv_geometry(co, ci, H, W, pipe, sms=132, smem_per_sm=233472, threads_per_sm=2048):
    """(tiles, grid upper bound, threads, RG) of one launch.  The grid is min(tiles, SMs x resident CTAs per SM); resident CTAs
    are bounded by shared memory and threads (registers can only lower it), so SMs x min(those two) bounds the grid from above.
    On an H100 (132 SMs, 228 KB per SM) that is 2 / 3 / 3 CTAs per SM pipelined and 5 / 8 / 8 scalar for 16->16 / 16->3 / 8->16;
    the grids measured there (torch.profiler, C4 shapes) are 2 / 3 / 2 pipelined and 3 / 7 / 2 scalar: registers bind below."""
    copt, rg = _INST[(co, ci)]
    threads = (co // copt) * ci * rg
    smem = 4 * _tile_floats(co, ci, pipe) * (2 if pipe else 1)
    per_sm = min(smem_per_sm // (smem + _SMEM_RESERVED), threads_per_sm // threads)
    tiles = ((W + TW - 1) // TW) * ((H + TH - 1) // TH)
    return tiles, sms * per_sm, threads, rg


def _device_geometry(co, ci, H, W, pipe):
    p = torch.cuda.get_device_properties(torch.cuda.current_device())
    return conv_geometry(co, ci, H, W, pipe, p.multi_processor_count, p.shared_memory_per_multiprocessor, p.max_threads_per_multi_processor)


def _wgrad_call(co, ci, H, W, x, gy, dW, db):
    import gof_appearance
    from diff_gaussian_rasterization import _C
    _C._check(gof_appearance._wgrad_lib().gof_conv3x3_wgrad(co, ci, H, W, x.data_ptr(), gy.data_ptr(), dW.data_ptr(),
                                                            db.data_ptr() if db is not None else None, _C._stream()))


def _ternary(shape, density, gen, dev):
    """entries in {-1, 0, 1}, nonzero with probability `density`"""
    v = torch.randint(-1, 2, shape, generator=gen, device=dev, dtype=torch.int8)
    keep = torch.rand(shape, generator=gen, device=dev) < density
    return (v * keep).float()


def test_conv_wgrad_reference_matches_torch_conv2d_weight():
    """CPU: the nine-matmul reference equals torch.nn.grad.conv2d_weight (double) at small shapes, borders included."""
    g = torch.Generator().manual_seed(1)
    for (co, ci), (H, W) in (((16, 16), (5, 7)), ((3, 16), (9, 33)), ((16, 8), (1, 1)), ((16, 8), (12, 4))):
        x = torch.randn(ci, H, W, generator=g, dtype=torch.float64)
        gy = torch.randn(co, H, W, generator=g, dtype=torch.float64)
        dW, db = conv_wgrad_ref(x, gy)
        want = torch.nn.grad.conv2d_weight(x[None], (co, ci, 3, 3), gy[None], padding=1)
        assert torch.allclose(dW, want, rtol=1e-12, atol=1e-12), (co, ci, H, W)
        assert torch.allclose(db, gy.sum((1, 2)), rtol=1e-12, atol=1e-12)


def test_conv_geometry_at_the_production_shapes():
    """CPU: the mirrored launch geometry gives every CTA at least three tiles at the appearance network's C4 shapes (1056 x 1920
    for conv2 / conv3, 528 x 960 for up4) on a 132-SM H100, so the pipelined cases below do exercise the prefetch."""
    for (co, ci), (H, W) in (((16, 16), (1056, 1920)), ((3, 16), (1056, 1920)), ((16, 8), (528, 960))):
        tiles, bound, _, _ = conv_geometry(co, ci, H, W, True)
        assert tiles >= 3 * bound, (co, ci, tiles, bound)
    assert conv_geometry(16, 16, 1056, 1920, True)[1] == 264 and conv_geometry(3, 16, 1056, 1920, True)[1] == 396


# (co, ci), (H, W), pipelined fill expected, x offset in floats; the first three are the C4 shapes (gof_appearance.py conv2,
# conv3 at 1056 x 1920, up4.conv at 528 x 960), then ragged shapes with many tiles per CTA on both fills, the alignment fallback
# (W % 4 == 0 but x 4 bytes into its storage) and images smaller than one tile
_EXACT_CASES = [
    ((16, 16), (1056, 1920), True, 0), ((3, 16), (1056, 1920), True, 0), ((16, 8), (528, 960), True, 0),
    ((16, 16), (1003, 1924), True, 0), ((3, 16), (1001, 1924), True, 0), ((16, 8), (517, 964), True, 0),
    ((16, 16), (1001, 1921), False, 0), ((3, 16), (1003, 1923), False, 0), ((16, 8), (1003, 963), False, 0),
    ((16, 16), (1056, 1920), False, 1), ((16, 8), (1040, 1924), False, 1),
    ((16, 16), (5, 20), True, 0), ((3, 16), (7, 31), False, 0), ((16, 8), (1, 1), False, 0), ((16, 16), (8, 32), True, 0),
    ((3, 16), (12, 4), True, 0),
]


@gpu
@pytest.mark.parametrize("pair,hw,pipe,xoff", _EXACT_CASES, ids=[f"{p[0]}x{p[1]}-{h[0]}x{h[1]}-{'pipe' if q else 'scalar'}{'-off' if o else ''}"
                                                                   for p, h, q, o in _EXACT_CASES])
def test_conv_wgrad_exact(pair, hw, pipe, xoff):
    """Exact-integer inputs: dW (accumulated onto a nonzero prefill) and db equal the fp64 reference bit for bit; db = NULL
    leaves dW the same.  Every partial sum is bounded by H*W < 2^24 in magnitude, so any summation order is exact."""
    (co, ci), (H, W) = pair, hw
    dev = torch.device("cuda")
    gen = torch.Generator(device=dev).manual_seed(H * 7919 + W * 31 + co + ci)
    assert H * W < 2 ** 24
    buf = torch.empty(ci * H * W + xoff, device=dev)
    x = buf[xoff:].view(ci, H, W)
    x.copy_(_ternary((ci, H, W), 0.6, gen, dev))
    gy = _ternary((co, H, W), 0.6, gen, dev)
    assert ((x.data_ptr() % 16) == 0) == (xoff == 0)
    assert ((W % 4 == 0) and xoff == 0) == pipe
    tiles, bound, _, _ = _device_geometry(co, ci, H, W, pipe)
    if H * W >= 400_000:                         # the large cases, on both fills: every CTA walks >= 3 tiles
        assert tiles >= 3 * bound, (tiles, bound)
    ref_w, ref_b = conv_wgrad_ref(x.double(), gy.double())
    prefill = torch.randint(-1000, 1001, (co, ci, 3, 3), generator=gen, device=dev).float()
    prefill_b = torch.randint(-1000, 1001, (co,), generator=gen, device=dev).float()
    dW, db = prefill.clone(), prefill_b.clone()
    _wgrad_call(co, ci, H, W, x, gy, dW, db)
    dW2 = torch.zeros_like(dW)
    _wgrad_call(co, ci, H, W, x, gy, dW2, None)
    torch.cuda.synchronize()
    assert torch.equal(dW.double(), prefill.double() + ref_w), float((dW.double() - prefill - ref_w).abs().max())
    assert torch.equal(db.double(), prefill_b.double() + ref_b)
    assert torch.equal(dW2.double(), ref_w)
    assert float(ref_w.abs().max()) > 0


# c of the random-valued bound:  |dW - fp64| <= C_WGRAD * 2^-24 * n_chain * sum_p |gy * x|  per weight, where n_chain is the
# longest chain of dependent fp32 additions a weight's partial sums pass through: the per-thread register sum over its CTA's
# tiles (tiles per CTA x TH / RG rows x 32 columns), the shared-memory combine over the RG row groups, the global atomics over
# the grid.  With c = 1 this is the classical worst-case bound of recursive summation; random rounding errors mostly cancel,
# so C_WGRAD is 4x the largest ratio measured on an H100 (8.1e-5, at the 8->16 C4 shape; 1.5e-5 and 1.6e-5 for the other two),
# rounded up to a power of two.
C_WGRAD = 2.0 ** -11


def conv_wgrad_random_ratio(co, ci, H, W, seed, dev):
    gen = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(ci, H, W, generator=gen, device=dev)
    gy = torch.randn(co, H, W, generator=gen, device=dev)
    pipe = W % 4 == 0
    tiles, bound, _, rg = _device_geometry(co, ci, H, W, pipe)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    n_chain = -(-tiles // min(tiles, sms)) * (TH // rg) * TW + rg + min(tiles, bound)
    ref_w, ref_b = conv_wgrad_ref(x.double(), gy.double())
    mag_w, mag_b = conv_wgrad_ref(x.double().abs(), gy.double().abs())
    dW, db = torch.zeros(co, ci, 3, 3, device=dev), torch.zeros(co, device=dev)
    _wgrad_call(co, ci, H, W, x, gy, dW, db)
    torch.cuda.synchronize()
    return max(_ratio(dW, ref_w, n_chain * mag_w), _ratio(db, ref_b, n_chain * mag_b))


@gpu
@pytest.mark.parametrize("pair,hw", [((16, 16), (1056, 1920)), ((3, 16), (1003, 1923)), ((16, 8), (528, 960))])
def test_conv_wgrad_random_values(pair, hw):
    (co, ci), (H, W) = pair, hw
    r = conv_wgrad_random_ratio(co, ci, H, W, 11 + H, torch.device("cuda"))
    assert r <= C_WGRAD, r


@gpu
def test_conv3x3_end_to_end_weight_gradient():
    """gof_appearance.conv3x3 at the C4 shape routes its backward through _Conv3x3, and conv.weight.grad / bias.grad equal the
    fp64 reference exactly on exact-integer inputs."""
    import gof_appearance
    dev = torch.device("cuda")
    gen = torch.Generator(device=dev).manual_seed(5)
    for (co, ci), (H, W) in (((16, 16), (1056, 1920)), ((16, 8), (528, 960))):
        conv = torch.nn.Conv2d(ci, co, 3, padding=1).to(dev)
        x = _ternary((1, ci, H, W), 0.5, gen, dev).requires_grad_(True)
        gy = _ternary((1, co, H, W), 0.5, gen, dev)
        y = gof_appearance.conv3x3(x, conv)
        assert y.grad_fn is not None and "Conv3x3" in type(y.grad_fn).__name__
        y.backward(gy)
        ref_w, ref_b = conv_wgrad_ref(x.detach()[0].double(), gy[0].double())
        assert torch.equal(conv.weight.grad.double(), ref_w) and torch.equal(conv.bias.grad.double(), ref_b)


# ========================================================================================================================
# 2. view_loss against oracle/loss_oracle.py
# ========================================================================================================================

def _loss_case(render, gt, cam, lambdas, need_grad=True):
    import gof_loss
    dev = torch.device("cuda")
    r = torch.from_numpy(render).to(dev).requires_grad_(need_grad)
    loss, terms = gof_loss.view_loss(r, torch.from_numpy(gt).to(dev), cam.world_view_transform, cam.tanfovx, cam.tanfovy, *lambdas)
    grad = None
    if need_grad:
        loss.backward()
        grad = r.grad.cpu().numpy()
    return terms.cpu().numpy(), grad


def _check_loss(render, gt, cam, lambdas, normal_tol=1e-4):
    """terms within 1e-5 relative; each gradient channel within 1e-4 (channel 6: 2e-3) of its largest magnitude, computed
    separately over the pixels where F.normalize's eps branch makes the gradient ~10^12 larger (rendered normal of length
    <= 1e-12 for channels 3-5; neighbours of an interior pixel whose depth normal is degenerate for channel 6) and the rest;
    channel 7 exactly 0, channel 8 exactly lam_dist / N.  `normal_tol` replaces 1e-4 for channels 3-5: their gradient is
    linear in the depth normal, which the kernel forms in fp32 from central differences of depth x ray; on a smooth surface
    those differences cancel (an fp32 restatement of depth_to_normal on a smooth 1920 x 1080 depth map is off by up to 2.1e-4
    from fp64), so a rendered scene needs a looser bound there than noise does."""
    import loss_oracle
    H, W = render.shape[1:]
    terms, grad = _loss_case(render, gt, cam, lambdas)
    o = loss_oracle.view_loss(render, gt, cam.world_view_transform.numpy(), cam.tanfovx, cam.tanfovy, lambdas)
    for i, k in enumerate(("Ll1", "ssim", "depth_normal_loss", "distortion_loss", "loss")):
        assert abs(float(terms[i]) - o[k]) <= 1e-5 * max(abs(o[k]), 1e-30) + 1e-30, (k, float(terms[i]), o[k])
    ref = o["grad"]
    small_n = np.linalg.norm(render[3:6].astype(np.float64), axis=0) <= 1e-12
    degen = np.zeros((H, W), bool)
    degen[1:-1, 1:-1] = np.linalg.norm(o["depth_normal"][:, 1:-1, 1:-1], axis=0) < 0.5
    feeds = np.zeros_like(degen)                       # pixels whose depth enters a degenerate pixel's central differences
    feeds[:-1] |= degen[1:]; feeds[1:] |= degen[:-1]; feeds[:, :-1] |= degen[:, 1:]; feeds[:, 1:] |= degen[:, :-1]
    for ch in range(7):
        special = small_n if 3 <= ch <= 5 else feeds if ch == 6 else np.zeros((H, W), bool)
        for m in (special, ~special):
            if not m.any():
                continue
            den = max(np.abs(ref[ch][m]).max(), 1e-30)
            err = np.abs(grad[ch][m] - ref[ch][m]).max() / den
            tol = 2e-3 if ch == 6 else normal_tol if ch >= 3 else 1e-4
            assert err < tol, (ch, "special" if m is special else "ordinary", err)
    assert (grad[7] == 0).all()
    lam_dist = np.float32(lambdas[2])
    assert (grad[8] == lam_dist * (np.float32(1.0) / (np.float32(W) * np.float32(H)))).all()
    assert np.isclose(float(grad[8][0, 0]), lambdas[2] / (W * H), rtol=1e-6)
    return terms, grad


def _noise_render(W, H, seed):
    rng = np.random.default_rng(seed)
    render = rng.uniform(0, 1, size=(9, H, W)).astype(np.float32)
    render[3:6] -= 0.5
    render[6] += 2.0
    # a ground truth correlated with the render, so that SSIM is well away from 0 and its relative tolerance means something
    return render, np.clip(render[:3] + rng.normal(0, 0.1, size=(3, H, W)), 0, 1).astype(np.float32)


@gpu
@pytest.mark.parametrize("W,H", [(37, 9), (16, 16), (50, 35), (49, 32), (48, 33), (17, 17), (331, 203)])
def test_view_loss_ragged_vs_oracle(W, H):
    """The host test's ragged shapes, one odd tile column (49 x 32), one odd tile row (48 x 33), both, and several tiles."""
    import gof_synth
    render, gt = _noise_render(W, H, W * 1000 + H)
    _check_loss(render, gt, gof_synth.make_camera(W, H, view=12), (0.2, 0.05, 100.0))


@gpu
def test_view_loss_branches_vs_oracle():
    """Exactly-zero rendered normals (F.normalize's eps branch), zero depth (degenerate depth normals), lambda_depth_normal = 0
    (channels 3-6 of the gradient exactly zero), and need_grad=False (terms bit-equal to the need_grad=True run)."""
    import gof_synth
    W, H = 203, 131
    cam = gof_synth.make_camera(W, H, view=21)
    render, gt = _noise_render(W, H, 77)
    render[3:6, 10:30, 40:75] = 0.0
    render[6, 60:90, 100:140] = 0.0
    render[6, :, 190:] = 0.0
    terms, grad = _check_loss(render, gt, cam, (0.2, 0.05, 100.0))
    big = np.abs(grad[3:6, 10:30, 40:75]).max()
    assert big > 1e3 * np.abs(grad[3:6, 50:, :40]).max()          # the eps branch did run
    t2, _ = _loss_case(render, gt, cam, (0.2, 0.05, 100.0), need_grad=False)
    assert np.array_equal(t2, terms)
    terms0, grad0 = _check_loss(render, gt, cam, (0.3, 0.0, 10.0))
    assert (grad0[3:7] == 0).all() and terms0[2] > 0


@gpu
def test_view_loss_1080p_rendered_vs_oracle():
    """1920 x 1080, the render taken from the rasterizer on a synthetic scene (P = 200 000; consistent depth and normal
    channels, background pixels with zero depth and zero normal), and the uniform-noise render (channels 3-5 within 1e-4)."""
    import _util
    import gof_synth
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda")
    cam, gs = gof_synth.make_scene(dict(P=200_000, width=1920, height=1080, seed=2), view=5)
    out = _C.rasterize_gaussians(*_util.fwd_args(cam, gs, dev))[1].cpu().numpy()
    assert (out[6] == 0).mean() > 0.01 and (out[6] > 0).mean() > 0.3, ((out[6] == 0).mean(), (out[6] > 0).mean())
    gt = np.clip(out[:3] + np.random.default_rng(3).normal(0, 0.05, size=out[:3].shape), 0, 1).astype(np.float32)
    _check_loss(out, gt, cam, (0.2, 0.05, 100.0), normal_tol=1e-3)       # measured on an H100: 1.2e-4
    render, gt = _noise_render(1920, 1080, 5)
    _check_loss(render, gt, gof_synth.make_camera(1920, 1080, view=7), (0.2, 0.05, 100.0))


# ========================================================================================================================
# 3. activate / activate_backward / adam_step
# ========================================================================================================================

def activate_ref(s, q, o, f, g_s, g_q, g_o):
    """fp64 restatement of param_ops.cuh:6-9 (values) and torch autograd of it (raw gradients), plus per-output error scales.
    s [P,3], q [P,4], o [P,1], f [P,1]; g_* the upstream gradients of scales, rotations, opacities."""
    s, q, o, f = (t.double().detach().requires_grad_(True) for t in (s, q, o, f))
    e = torch.exp(s)
    S2 = e * e + f * f
    scales = torch.sqrt(S2)
    coef = torch.sqrt((e * e).prod(1, keepdim=True) / S2.prod(1, keepdim=True))
    sg = torch.sigmoid(o)
    op = sg * coef
    n2 = (q * q).sum(1, keepdim=True)
    big = n2 > 1e-24                                     # |q| > 1e-12; below, F.normalize divides by the constant eps
    d = torch.where(big, torch.sqrt(torch.where(big, n2, torch.ones_like(n2))), torch.full_like(n2, 1e-12))
    rot = q / d
    torch.autograd.backward([scales, rot, op], [g_s.double(), g_q.double(), g_o.double()])
    with torch.no_grad():
        gs, gq, go = g_s.double(), g_q.double(), g_o.double()
        e2 = e * e
        u = rot
        scale = dict(
            scales=scales, rot=torch.ones_like(rot), op=op,
            d_s=(gs * e2 / scales).abs() + (go * sg * coef).abs(),
            d_q=(gq.abs() + u.abs() * (u * gq).abs().sum(1, keepdim=True)) / d,
            d_o=(go * coef * sg).abs())
    return dict(scales=scales.detach(), rot=rot.detach(), op=op.detach(), d_s=s.grad, d_q=q.grad, d_o=o.grad), scale


def test_activate_reference_matches_reference_goldens():
    """CPU: the fp64 restatement against the goldens the reference's own Python produced (fp32, so 1e-5 relative)."""
    import glob
    for path in sorted(glob.glob(os.path.join(HERE, "golden", "params_*.npz"))):
        fx = np.load(path)
        t = lambda k: torch.from_numpy(fx[k])   # noqa: E731
        out, _ = activate_ref(t("raw_scaling"), t("raw_rotation"), t("raw_opacity"), t("filter_3D"), t("up_scales"),
                              t("up_rotations"), t("up_opacities"))
        for k, g in (("scales", "out_scales"), ("rot", "out_rotations"), ("op", "out_opacities"), ("d_s", "grad_scaling"),
                     ("d_o", "grad_opacity")):
            ref = fx[g].astype(np.float64)
            assert np.abs(out[k].numpy() - ref).max() <= 1e-5 * np.abs(ref).max(), (path, k)
        ok = np.linalg.norm(fx["raw_rotation"], axis=1) > 1e-6
        r, a = fx["grad_rotation"].astype(np.float64), out["d_q"].numpy()
        assert np.abs(a[ok] - r[ok]).max() <= 2e-5 * np.abs(r[ok]).max()


def _raw_params(P, Mr, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    s = torch.rand(P, 3, generator=g, device=dev) * 14.0 - 12.0              # raw log-scales -12 .. +2
    q = torch.randn(P, 4, generator=g, device=dev)
    q[::17] = 0.0                                                            # zero quaternions
    o = torch.randn(P, 1, generator=g, device=dev) * 3.0
    f = torch.rand(P, 1, generator=g, device=dev) * 0.05
    f[::5] = 0.0                                                             # filter_3D = 0 rows
    s[1::7] = torch.tensor([-12.0, 2.0, -5.0], device=dev)                  # the ends of the range
    dc, rest = torch.randn(P, 1, 3, generator=g, device=dev), torch.randn(P, Mr, 3, generator=g, device=dev)
    ups = [torch.randn(P, 3, generator=g, device=dev), torch.randn(P, 4, generator=g, device=dev),
           torch.randn(P, 1, generator=g, device=dev), torch.randn(P, Mr + 1, 3, generator=g, device=dev)]
    return [s, q, o, f, dc, rest], ups


# c of the activation bounds (|gpu - fp64| <= c * 2^-24 * scale): expf / sqrtf / divisions of the kernel round within a few
# ulps each and the opacity's coefficient chains about a dozen of them.  C_ACT is 4x the largest ratio measured on an H100
# over every case below (7.97, the opacity and its raw gradient; 7.8 the scale gradient, 3.8 the scales), rounded up to a
# power of two.
C_ACT = 32.0


def activate_ratios(P, Mr, seed, dev):
    import gof_params
    raw, ups = _raw_params(P, Mr, seed, dev)
    s, q, o, f, dc, rest = raw
    leaves = [t.clone().requires_grad_(i != 3) for i, t in enumerate(raw)]
    outs = gof_params.activate(*leaves)
    torch.autograd.backward(list(outs), ups)
    torch.cuda.synchronize()
    ref, scale = activate_ref(s, q, o, f, ups[0], ups[1], ups[2])
    shs = outs[3]
    assert torch.equal(shs[:, :1], dc) and torch.equal(shs[:, 1:], rest)
    assert torch.equal(leaves[4].grad, ups[3][:, :1]) and torch.equal(leaves[5].grad, ups[3][:, 1:])
    got = dict(scales=outs[0], rot=outs[1], op=outs[2], d_s=leaves[0].grad, d_q=leaves[1].grad, d_o=leaves[2].grad)
    for k, v in got.items():
        assert torch.isfinite(v).all(), k
    return {k: _ratio(got[k], ref[k], scale[k]) for k in got}


@gpu
@pytest.mark.parametrize("Mr", [0, 3, 8, 15])
@pytest.mark.parametrize("P", [1, 255, 257, 1_000_003])
def test_activate_vs_fp64(P, Mr):
    r = activate_ratios(P, Mr, P + 100 * Mr, torch.device("cuda"))
    assert max(r.values()) <= C_ACT, r


@gpu
def test_activate_accepts_misaligned_views():
    """Raw parameters, and the rotations' upstream gradient, as views 4 bytes into one flat buffer (like a parameter sliced out
    of a flat tensor): forward and backward equal the aligned call bit for bit."""
    import gof_params
    dev = torch.device("cuda")
    P, Mr = 5003, 15
    raw, ups = _raw_params(P, Mr, 3, dev)
    shapes = [t.shape for t in raw] + [ups[1].shape]
    flat = torch.zeros(1 + sum(math.prod(sh) + 4 for sh in shapes) + 8, device=dev)
    views, off = [], 1
    for t in raw + [ups[1]]:
        off += (1 - off) % 4                                                 # 4 bytes past a 16-byte boundary
        v = flat[off:off + t.numel()].view(t.shape)
        v.copy_(t)
        off += t.numel()
        views.append(v)
    assert views[1].data_ptr() % 16 != 0 and views[-1].data_ptr() % 16 != 0

    def run(ins, g_rot):
        leaves = [t.detach().requires_grad_(i != 3) for i, t in enumerate(ins)]
        outs = gof_params.activate(*leaves)
        torch.autograd.backward(list(outs), [ups[0], g_rot, ups[2], ups[3]])
        return [t.detach().clone() for t in outs] + [leaves[i].grad.clone() for i in (0, 1, 2, 4, 5)]

    a = run(raw, ups[1])
    b = run(views[:-1], views[-1])
    torch.cuda.synchronize()
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), i


_REFUSAL_SCRIPT = textwrap.dedent("""
    import ctypes, json, sys
    lib = ctypes.CDLL(sys.argv[1])
    lib.gof_last_error.restype = ctypes.c_char_p
    v = ctypes.c_void_p
    lib.gof_activate_params.argtypes = [ctypes.c_int, ctypes.c_int] + [v] * 11
    lib.gof_activate_params_backward.argtypes = [ctypes.c_int, ctypes.c_int] + [v] * 14
    A = 1 << 20                                  # stand-in device addresses: the checks must refuse before any CUDA call
    ptrs = [A + 4096 * k for k in range(16)]
    out = {}
    def fwd(name, bad):                          # 10 arrays, then the stream; rotation_raw is #1, rotations #7
        p = list(ptrs[:10])
        if bad is not None:
            p[bad] += 4
        out[name] = [lib.gof_activate_params(1000, 15, *p, None), lib.gof_last_error().decode()]
    def bwd(name, bad):                          # 13 arrays; rotation_raw #1, g_rotations #5, d_rotation_raw #9
        p = list(ptrs[:13])
        if bad is not None:
            p[bad] += 8
        out[name] = [lib.gof_activate_params_backward(1000, 15, *p, None), lib.gof_last_error().decode()]
    fwd("fwd_rotation_in", 1); fwd("fwd_rotation_out", 7); fwd("fwd_aligned", None)
    bwd("bwd_rotation_in", 1); bwd("bwd_g_rotation", 5); bwd("bwd_d_rotation", 9); bwd("bwd_aligned", None)
    print(json.dumps(out))
""")


def test_activate_refuses_misaligned_rotations_without_a_device():
    """CPU: the C ABI refuses a rotation pointer (input, output, upstream or raw gradient) that is not 16-byte aligned with
    GOF_E_INVALID, on the host; the same call with aligned pointers gets past the checks to its first launch (which fails:
    no device is visible)."""
    assert os.path.exists(LIB_PATH), "build the library first: python gaussian-opacity-fields_b200/build.py"
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, "-c", _REFUSAL_SCRIPT, LIB_PATH], env=env, capture_output=True, text=True, timeout=120)
    assert res.returncode == 0, res.stderr
    out = json.loads(res.stdout.strip().splitlines()[-1])
    for name in ("fwd_rotation_in", "fwd_rotation_out", "bwd_rotation_in", "bwd_g_rotation", "bwd_d_rotation"):
        assert out[name][0] == GOF_E_INVALID and "aligned" in out[name][1], (name, out[name])
    assert out["fwd_aligned"][0] == GOF_E_CUDA and out["bwd_aligned"][0] == GOF_E_CUDA, out


def adam_ref_step(p, m, v, g, lr, step, beta1=0.9, beta2=0.999, eps=1e-15):
    """One torch.optim.Adam step (no weight decay, no amsgrad) in fp64 from the given state; returns (p, m, v) and their error
    scales (the magnitudes of the terms each new value is formed from)."""
    p, m, v, g = (t.double() for t in (p, m, v, g))
    mm = m + (1.0 - beta1) * (g - m)
    vv = beta2 * v + (1.0 - beta2) * g * g
    bias1, bias2 = 1.0 - beta1 ** step, 1.0 - beta2 ** step
    upd = (lr / bias1) * mm / (torch.sqrt(vv) / math.sqrt(bias2) + eps)
    sc_m = m.abs() + (1.0 - beta1) * (g.abs() + m.abs())
    return (p - upd, mm, vv), (p.abs() + upd.abs() * (1.0 + sc_m / mm.abs().clamp(min=1e-300)), sc_m, vv)


def test_adam_reference_matches_reference_goldens():
    """CPU: three fp64 steps from zero moments against the reference's torch.optim.Adam run (fp32 goldens)."""
    import glob
    for path in sorted(glob.glob(os.path.join(HERE, "golden", "params_*.npz"))):
        fx = np.load(path)
        p = torch.from_numpy(fx["adam_p0"]).double()
        m, v = torch.zeros_like(p), torch.zeros_like(p)
        for step, g in enumerate(fx["adam_grads"], start=1):
            (p, m, v), _ = adam_ref_step(p, m, v, torch.from_numpy(g), float(fx["adam_lr"]), step)
        assert np.abs(m.numpy() - fx["adam_m"]).max() <= 1e-6 * np.abs(fx["adam_m"]).max()
        assert np.abs(v.numpy() - fx["adam_v"]).max() <= 1e-6 * np.abs(fx["adam_v"]).max()
        assert np.abs(p.numpy() - fx["adam_p"]).max() <= 1e-6


# c of the Adam bound, in fp32 ulps of each new value's term scale (adam_ref_step): m and v take 2-3 roundings, p's update a
# division, a square root and the bias corrections rounded to float once by the host.  C_ADAM is 4x the largest ratio measured
# on an H100 over 59 M elements x 5 steps (2.27), rounded up to a power of two.
C_ADAM = 16.0


def adam_ratios(n, steps, dev, torch_check=True):
    """Per step, from the kernel's own state: the kernel's new (p, m, v) against one fp64 step, and against one step of
    torch.optim.Adam(eps=1e-15, foreach=False) started from the same state; both in ulps of the fp64 term scale."""
    import gof_params
    gen = torch.Generator(device=dev).manual_seed(n % 1000 + 1)
    p = torch.randn(n, generator=gen, device=dev)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    tp = p.clone().requires_grad_(True)
    opt = torch.optim.Adam([tp], lr=1.6e-4, eps=1e-15, foreach=False) if torch_check else None
    worst, worst_torch = 0.0, 0.0
    for step in range(1, steps + 1):
        g = torch.randn(n, generator=gen, device=dev) * 10.0 ** (step % 3 - 1)
        g[(step * 48) % 4096::4096] = 0.0                                # elements without gradient this step
        if step == 1:
            g[: 48 * 1000] = 0.0                                        # elements without gradient at the first step
        (rp, rm, rv), (sp, sm, sv) = adam_ref_step(p, m, v, g, 1.6e-4, step)
        if opt is not None:
            with torch.no_grad():
                tp.copy_(p)
                if step > 1:
                    opt.state[tp]["exp_avg"].copy_(m)
                    opt.state[tp]["exp_avg_sq"].copy_(v)
            tp.grad = g.clone()
            opt.step()
        gof_params.adam_step(p, m, v, g, 1.6e-4, step)
        torch.cuda.synchronize()
        for got, ref, sc in ((p, rp, sp), (m, rm, sm), (v, rv, sv)):
            worst = max(worst, _ratio(got, ref, _ulp32(sc) / EPS))
        if opt is not None:
            st = opt.state[tp]
            for got, ref, sc in ((p, tp.detach(), sp), (m, st["exp_avg"], sm), (v, st["exp_avg_sq"], sv)):
                worst_torch = max(worst_torch, _ratio(got, ref.double(), _ulp32(sc) / EPS))
        del rp, rm, rv, sp, sm, sv
    return worst, worst_torch


@gpu
@pytest.mark.parametrize("n", [257, 1_000_003, 59_000_011])
def test_adam_vs_fp64_and_torch(n):
    worst, worst_torch = adam_ratios(n, 5, torch.device("cuda"))
    assert worst <= C_ADAM, worst
    assert worst_torch <= 4.0, worst_torch        # "a few ulp"; measured on an H100: 2


# ========================================================================================================================
# 4. compute_3d_filter
# ========================================================================================================================

def filter3d_ref(xyz, cams, margin=1e-6):
    """fp64 restatement of compute_3D_filter (scene/gaussian_model.py:262-311): filter [P] (NaN if no point is seen) and, per
    point, whether an fp32 evaluation may legitimately differ: some camera's decision lies within `margin` of a cut -- depth
    0.2, or the frame enlarged by 15 % -- relative to the magnitude of the terms the compared value is formed from, and that
    camera's depth is below the smallest depth of the cameras whose decisions are clear."""
    x = xyz.double()
    c = cams.double()
    P = x.shape[0]
    dist = torch.full((P,), 100000.0, dtype=torch.float64, device=x.device)
    seen = torch.zeros(P, dtype=torch.bool, device=x.device)
    clear_min = torch.full((P,), math.inf, dtype=torch.float64, device=x.device)
    near_min = torch.full((P,), math.inf, dtype=torch.float64, device=x.device)
    for k in c:
        R, T = k[:9].view(3, 3), k[9:12]
        fx, fy, W, H = (float(k[i]) for i in range(12, 16))
        xc = x @ R + T
        sc = x.abs() @ R.abs() + T.abs()                               # term scale of each camera coordinate
        z = xc[:, 2].clamp(min=0.001)
        u = xc[:, 0] / z * fx + W / 2.0
        w = xc[:, 1] / z * fy + H / 2.0
        su = fx * (sc[:, 0] + xc[:, 0].abs() * sc[:, 2] / z) / z + W
        sw = fy * (sc[:, 1] + xc[:, 1].abs() * sc[:, 2] / z) / z + H
        valid = (xc[:, 2] > 0.2) & (u >= -0.15 * W) & (u <= 1.15 * W) & (w >= -0.15 * H) & (w <= 1.15 * H)
        near = (xc[:, 2] - 0.2).abs() <= margin * sc[:, 2]
        for val, cut, s in ((u, -0.15 * W, su), (u, 1.15 * W, su), (w, -0.15 * H, sw), (w, 1.15 * H, sw)):
            near |= (xc[:, 2] > 0.2) & ((val - cut).abs() <= margin * s)
        dist = torch.where(valid, torch.minimum(dist, z), dist)
        seen |= valid
        clear_min = torch.where(valid & ~near, torch.minimum(clear_min, z), clear_min)
        near_min = torch.where(near, torch.minimum(near_min, z), near_min)
    if not seen.any():
        return torch.full((P,), math.nan, dtype=torch.float64, device=x.device), seen, near_min < clear_min
    dist = torch.where(seen, dist, dist[seen].max())
    max_focal = float(c[:, 12].max())
    return dist / max_focal * math.sqrt(0.2), seen, near_min < clear_min


def test_filter3d_reference_matches_reference_golden():
    """CPU: the fp64 restatement against the reference's own output on 5 000 points and 5 cameras (tests/golden/filter3d_a.npz,
    fp32: the criterion of test_gpu_param_ops.py)."""
    fx = np.load(os.path.join(HERE, "golden", "filter3d_a.npz"))
    out, seen, _ = filter3d_ref(torch.from_numpy(fx["xyz"]), torch.from_numpy(fx["cams"]))
    ref = fx["filter_3D"][:, 0].astype(np.float64)
    rel = np.abs(out.numpy() - ref) / ref
    assert np.quantile(rel, 0.999) < 1e-5 and (rel > 1e-5).sum() <= 3
    assert 0 < int((~seen).sum()) < len(ref)


def _filter_cameras(n):
    import gof_synth
    sizes = [(640, 480), (800, 600), (1920, 1080), (1600, 1200), (320, 200), (1280, 720), (1000, 1000)]
    rows = []
    for v in range(n):
        W, H = sizes[v % len(sizes)]
        c = gof_synth.make_camera(W, H, view=v, n_views=n, radius=3.5 + 0.4 * (v % 7), fovx_deg=(40.0, 60.0, 75.0, 90.0)[v % 4],
                                  elevation=0.2 * ((v % 5) - 2))
        w2v = c.world_view_transform.t()
        R, T = w2v[:3, :3].t().contiguous().numpy(), w2v[:3, 3].contiguous().numpy()
        rows.append(np.concatenate([R.reshape(-1), T, [W / (2 * c.tanfovx), H / (2 * c.tanfovy), W, H]]).astype(np.float32))
    return torch.from_numpy(np.stack(rows))


def _filter_points(P, n_unseen, seed):
    g = torch.Generator().manual_seed(seed)
    xyz = (torch.rand(P, 3, generator=g) * 2 - 1) * 1.2
    xyz[:n_unseen, 1] = torch.where(torch.arange(n_unseen) % 2 == 0, 50.0, -50.0)     # straight above / below every camera
    return xyz


@gpu
def test_filter3d_at_scale():
    """10^6 + 3 points, 200 cameras of seven image sizes and four fields of view, 1 000 points no camera sees: each point's
    filter within 1e-5 relative of fp64 unless its fp64 decision for the camera that decides lies within 1e-6 of a cut."""
    import gof_params
    dev = torch.device("cuda")
    P, n_unseen = 1_000_003, 1000
    cams = _filter_cameras(200).to(dev)
    xyz = _filter_points(P, n_unseen, 9).to(dev)
    ref, seen, marginal = filter3d_ref(xyz, cams)
    assert not seen[:n_unseen].any() and bool(seen[n_unseen:].all())
    out = gof_params.compute_3d_filter(xyz, cams, float(cams[:, 12].max()))[:, 0].double()
    rel = (out - ref).abs() / ref
    n_marginal = int(marginal.sum())
    assert n_marginal <= 100, n_marginal                  # 0 of the 10^6 points in this scene
    bad = (rel > 1e-5) & ~marginal
    assert not bad.any(), (int(bad.sum()), float(rel[~marginal].max()))
    assert torch.equal(out[:n_unseen], torch.full_like(out[:n_unseen], float(out[:n_unseen][0])))


@gpu
def test_filter3d_raises_when_no_point_is_seen():
    import gof_params
    dev = torch.device("cuda")
    cams = _filter_cameras(20).to(dev)
    xyz = _filter_points(4097, 4097, 4).to(dev)
    assert not filter3d_ref(xyz, cams)[1].any()
    with pytest.raises(RuntimeError, match="no point is seen"):
        gof_params.compute_3d_filter(xyz, cams, float(cams[:, 12].max()))
