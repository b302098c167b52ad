"""GPU: the fused per-view loss with the decoupled-appearance L1 (gof_loss.view_loss(..., appearance=mapping) ->
gof_view_loss_appearance, csrc/view_loss.cu) against the goldens the reference's own Python produced
(tests/golden/make_golden_loss_appearance.py) and the fp64 oracle (tests/_loss_app_oracle.py), at the training shape
1920 x 1080 and ragged ones, at its edges (exact ties, mapping 0 and 1, lambda_dssim 0 and 1, lambda_depth_normal 0), against
the plain call on the same inputs, and end to end through the appearance network against the reference's loss lines in
torch.  The same kernel source is checked phase by phase on the CPU in test_view_loss_appearance_host.py.

Tolerances follow _check_loss of test_gpu_train_step.py: terms within 1e-5 relative, gradients within 1e-4 of their largest
magnitude (channel 6: 2e-3), over the pixels whose L1 sign the oracle decides (see _loss_app_oracle.view_loss's `marginal`)."""
import glob
import hashlib
import math
import os
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
FIX = sorted(glob.glob(os.path.join(HERE, "golden", "loss_app_*.npz")))
TERMS = ("Ll1", "ssim", "depth_normal_loss", "distortion_loss", "loss")
LAM = (0.2, 0.05, 100.0)
C4 = (1080, 1920)                 # H x W; crop_window: 1056 x 1920 at top 12, left 0 (12 is not on the 16-pixel tile grid)
# SHA-256 of the plain gof_view_loss's terms and gradient on c4_plain_inputs(), computed by the build of the commit before
# gof_view_loss_appearance existed, on an H100: the plain mode is bit-identical to it.
C4_PLAIN_SHA256 = "39bb1d9ec7b699b76fc7ed45b2e1e4bf200169f371b5a4ff8d5a96f1937adcbe"


def noise_inputs(H, W, seed, Hc, Wc):
    rng = np.random.default_rng(seed)
    render = rng.uniform(0, 1, size=(9, H, W)).astype(np.float32)
    render[3:6] -= 0.5
    render[6] += 2.0
    gt = np.clip(render[:3] + rng.normal(0, 0.1, size=(3, H, W)), 0, 1).astype(np.float32)
    mapping = rng.uniform(0.6, 1.4, size=(3, Hc, Wc)).astype(np.float32)
    return render, gt, mapping


def c4_plain_inputs():
    """The render, gt and camera of the plain call whose outputs C4_PLAIN_SHA256 pins."""
    import gof_synth
    render, gt, _ = noise_inputs(*C4, 2024, 1, 1)
    return render, gt, gof_synth.make_camera(C4[1], C4[0], view=7)


def outputs_sha256(terms, grad):
    h = hashlib.sha256()
    for a in (terms, grad):
        h.update(np.ascontiguousarray(a, np.float32).tobytes())
    return h.hexdigest()


def run(render, gt, cam, lambdas, mapping=None, need_grad=True, batch_dim=False):
    """gof_loss.view_loss through autograd; returns numpy (terms, d loss / d render, d loss / d mapping)."""
    import gof_loss
    dev = torch.device("cuda")
    r = torch.from_numpy(render).to(dev).requires_grad_(need_grad)
    m = None
    if mapping is not None:
        m = torch.from_numpy(mapping).to(dev)
        m = (m[None] if batch_dim else m).requires_grad_(need_grad)
    loss, terms = gof_loss.view_loss(r, torch.from_numpy(gt).to(dev), cam.world_view_transform, cam.tanfovx, cam.tanfovy, *lambdas,
                                     appearance=m)
    assert float(loss.detach()) == float(terms[4])
    if not need_grad:
        return terms.cpu().numpy(), None, None
    loss.backward()
    gm = None
    if m is not None:
        assert m.grad.shape == m.shape
        gm = m.grad.reshape(mapping.shape).cpu().numpy()
    return terms.cpu().numpy(), r.grad.cpu().numpy(), gm


def oracle(render, gt, cam, lambdas, mapping):
    import _loss_app_oracle
    import gof_appearance
    top, left, _, _ = gof_appearance.crop_window(*render.shape[1:])
    o = _loss_app_oracle.view_loss(render, gt, cam.world_view_transform.numpy(), cam.tanfovx, cam.tanfovy, lambdas, mapping,
                                   top, left)
    o.update(top=top, left=left)
    return o


def check(terms, grad, grad_m, exp, keep=None):
    """`exp` = oracle or golden values (TERMS, grad [9,H,W], grad_mapping, top, left); `keep` [3,Hc,Wc] = crop pixels whose
    L1 sign is decided (None: all)."""
    for i, k in enumerate(TERMS):
        assert abs(float(terms[i]) - exp[k]) <= 1e-5 * max(abs(exp[k]), 1e-30) + 1e-30, (k, float(terms[i]), exp[k])
    top, left = exp["top"], exp["left"]
    Hc, Wc = exp["grad_mapping"].shape[1:]
    mask = np.ones(grad.shape, bool)
    if keep is not None:
        mask[:3, top:top + Hc, left:left + Wc] = keep
    for ch in range(9):
        den = max(np.abs(exp["grad"][ch]).max(), 1e-30)
        err = np.abs(grad[ch] - exp["grad"][ch])[mask[ch]].max() / den
        assert err < (2e-3 if ch == 6 else 1e-4), (ch, err)
    mk = np.ones(grad_m.shape, bool) if keep is None else keep
    if np.abs(exp["grad_mapping"]).max() == 0:
        assert (grad_m[mk] == 0).all()
    else:
        assert np.abs(grad_m - exp["grad_mapping"])[mk].max() / np.abs(exp["grad_mapping"]).max() < 1e-4


def check_vs_oracle(render, gt, cam, lambdas, mapping):
    out = run(render, gt, cam, lambdas, mapping)
    o = oracle(render, gt, cam, lambdas, mapping)
    check(*out, o, keep=~o["marginal"])
    return out, o


@pytest.mark.parametrize("path", FIX, ids=[os.path.basename(p)[:-4] for p in FIX])
def test_matches_reference_goldens_and_oracle(path):
    """48x72 (32x64 crop at top 8, left 4), 70x101 (64x96 at 3, 2), 96x160 (the crop is the whole image); the mapping passed
    as [3,Hc,Wc] and as the network's [1,3,Hc,Wc]."""
    fx = np.load(path)
    render, gt, mapping = fx["render"], fx["gt"], fx["mapping"]
    lam = [float(x) for x in fx["lambdas"]]
    cam = types.SimpleNamespace(world_view_transform=torch.from_numpy(fx["world_view_transform"]), tanfovx=float(fx["tanfovx"]),
                                tanfovy=float(fx["tanfovy"]))
    grad = fx["grad"].astype(np.float64).copy()
    grad[:3] = fx["app_grad_rgb"]
    exp = dict(Ll1=float(fx["app_Ll1"]), ssim=float(fx["ssim"]), depth_normal_loss=float(fx["depth_normal_loss"]),
               distortion_loss=float(fx["distortion_loss"]), loss=float(fx["app_loss"]), grad=grad,
               grad_mapping=fx["grad_mapping"].astype(np.float64), top=int(fx["top"]), left=int(fx["left"]))
    out = run(render, gt, cam, lam, mapping)
    check(*out, exp)
    o = oracle(render, gt, cam, lam, mapping)
    assert (o["top"], o["left"]) == (exp["top"], exp["left"])
    check(*out, o, keep=~o["marginal"])
    out4 = run(render, gt, cam, lam, mapping, batch_dim=True)
    for a, b in zip(out, out4):
        assert np.array_equal(a, b)


def test_c4_vs_oracle_and_plain_call():
    """1920 x 1080: against the oracle; terms[1..3] and gradient channels 3-8 bit-equal to the plain call on the same inputs;
    values-only terms bit-equal to the gradient run; two runs bit-identical."""
    import gof_synth
    H, W = C4
    cam = gof_synth.make_camera(W, H, view=7)
    render, gt, mapping = noise_inputs(H, W, 11, 1056, 1920)
    out, o = check_vs_oracle(render, gt, cam, LAM, mapping)
    assert (o["top"], o["left"]) == (12, 0)
    plain = run(render, gt, cam, LAM)
    assert np.array_equal(out[0][1:4], plain[0][1:4])
    assert np.array_equal(out[1][3:], plain[1][3:])
    assert out[0][0] != plain[0][0]
    t_values, _, _ = run(render, gt, cam, LAM, mapping, need_grad=False)
    assert np.array_equal(t_values, out[0])
    again = run(render, gt, cam, LAM, mapping)
    for a, b in zip(out, again):
        assert np.array_equal(a, b)


def test_plain_call_is_bit_identical_to_before_the_appearance_mode():
    render, gt, cam = c4_plain_inputs()
    terms, grad, _ = run(render, gt, cam, LAM)
    assert outputs_sha256(terms, grad) == C4_PLAIN_SHA256


@pytest.mark.parametrize("lambdas", [(0.0, 0.05, 100.0), (1.0, 0.05, 100.0), (0.2, 0.0, 100.0), (0.35, 0.3, 10.0)],
                         ids=["dssim0", "dssim1", "dn0", "other"])
def test_lambdas_vs_oracle(lambdas):
    """lambda_dssim 0 (the rgb gradient is the L1 part alone: exactly 0 outside the crop) and 1 (no L1 part: the mapping
    gradient is exactly 0), lambda_depth_normal 0 (channels 3-6 exactly 0), on a 203 x 331 image (192 x 320 crop at 5, 5)."""
    import gof_synth
    H, W = 203, 331
    cam = gof_synth.make_camera(W, H, view=21)
    render, gt, mapping = noise_inputs(H, W, 5, 192, 320)
    (terms, grad, grad_m), o = check_vs_oracle(render, gt, cam, lambdas, mapping)
    assert (o["top"], o["left"]) == (5, 5)
    outside = np.ones((H, W), bool)
    outside[5:197, 5:325] = False
    if lambdas[0] == 0.0:
        assert (grad[:3][:, outside] == 0).all() and (grad[:3][:, ~outside] != 0).any()
    if lambdas[0] == 1.0:
        assert (grad_m == 0).all()
    if lambdas[1] == 0.0:
        assert (grad[3:7] == 0).all() and terms[2] > 0


def dyadic_inputs(H, W, Hc, Wc, top, left, seed):
    """Render and mapping on coarse dyadic grids, so that mapping * rgb is exact in float; gt equals that product on the
    even pixels of the crop (exact ties) and differs from it elsewhere."""
    rng = np.random.default_rng(seed)
    render, gt, _ = noise_inputs(H, W, seed, Hc, Wc)
    render[:3] = rng.integers(1, 64, size=(3, H, W)) / 64.0
    mapping = (rng.integers(8, 24, size=(3, Hc, Wc)) / 16.0).astype(np.float32)
    crop = (slice(0, 3), slice(top, top + Hc), slice(left, left + Wc))
    prod = (mapping.astype(np.float64) * render[crop]).astype(np.float32)
    assert np.array_equal(prod.astype(np.float64), mapping.astype(np.float64) * render[crop])
    tie = (np.add.outer(np.arange(Hc), np.arange(Wc)) % 2 == 0)[None].repeat(3, 0)
    gt[crop] = np.where(tie, prod, np.clip(prod + rng.choice([-1, 1], size=prod.shape) * 0.125, 0, 2)).astype(np.float32)
    return render, gt.astype(np.float32), mapping, tie


def test_exact_ties():
    """fl(m * rgb) == gt exactly: the L1 part of both gradients is exactly 0 there (torch's abs backward, sgn(0) = 0)."""
    import gof_synth
    H, W = 100, 140                  # crop 96 x 128 at top 2, left 6
    cam = gof_synth.make_camera(W, H, view=3)
    render, gt, mapping, tie = dyadic_inputs(H, W, 96, 128, 2, 6, 9)
    (terms, grad, grad_m), o = check_vs_oracle(render, gt, cam, LAM, mapping)
    assert not o["marginal"].any()
    assert (grad_m[tie] == 0).all() and (grad_m[~tie] != 0).all()
    _, g0, gm0 = run(render, gt, cam, (0.0, 0.05, 100.0), mapping)       # no SSIM term: the rgb gradient is the L1 part
    rgb = g0[:3, 2:98, 6:134]
    assert (rgb[tie] == 0).all() and (rgb[~tie] != 0).all() and (gm0[tie] == 0).all()


@pytest.mark.parametrize("value", [0.0, 1.0])
def test_constant_mapping(value):
    """mapping 0 (the L1 of gt alone: no L1 part in the rgb gradient) and mapping 1 (the plain L1 on the crop; with the crop
    equal to the image the terms are bit-equal to the plain call's)."""
    import gof_synth
    for (H, W) in ((70, 101), (96, 160)):
        cam = gof_synth.make_camera(W, H, view=4)
        render, gt, _ = noise_inputs(H, W, 17, 1, 1)
        mapping = np.full((3, H // 32 * 32, W // 32 * 32), value, np.float32)
        (terms, grad, grad_m), o = check_vs_oracle(render, gt, cam, LAM, mapping)
        if value == 0.0:
            _, g0, _ = run(render, gt, cam, (0.0, 0.05, 100.0), mapping)
            assert (g0[:3] == 0).all() and (grad_m != 0).any()
        elif (H, W) == (96, 160):
            plain = run(render, gt, cam, LAM)
            assert np.array_equal(terms, plain[0])


# ---------------------------------------------------------------------------------------------------- end to end
def torch_train_loss(rendering, gt, cam, lambdas, network, embedding):
    """The reference's loss lines (train.py:151-188 with 157-159) in torch: gof_appearance.l1_loss_appearance,
    ssim (utils/loss_utils.py:20-63), depth_to_normal (utils/depth_utils.py:6-35) and the distortion mean."""
    import gof_appearance
    lam, lam_dn, lam_dist = lambdas
    image = rendering[:3]
    Ll1 = gof_appearance.l1_loss_appearance(image, gt, network, embedding)
    g = torch.tensor([math.exp(-(x - 5) ** 2 / float(2 * 1.5 ** 2)) for x in range(11)])
    g = g / g.sum()
    window = (g[:, None] @ g[None, :]).float()[None, None].expand(3, 1, 11, 11).contiguous().to(rendering.device)
    conv = lambda x: F.conv2d(x[None], window, padding=5, groups=3)[0]
    mu1, mu2 = conv(image), conv(gt)
    s11, s22, s12 = conv(image * image) - mu1 * mu1, conv(gt * gt) - mu2 * mu2, conv(image * gt) - mu1 * mu2
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    ssim = (((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 * mu1 + mu2 * mu2 + C1) * (s11 + s22 + C2))).mean()
    H, W = rendering.shape[1:]
    c2w = cam.world_view_transform.to(rendering.device).T.inverse()
    fx, fy = W / (2 * cam.tanfovx), H / (2 * cam.tanfovy)
    intrins_inv = torch.tensor([[1 / fx, 0., -W / (2 * fx)], [0., 1 / fy, -H / (2 * fy)], [0., 0., 1.0]]).float().to(rendering.device)
    gx, gy = torch.meshgrid(torch.arange(W, device=rendering.device).float() + 0.5,
                            torch.arange(H, device=rendering.device).float() + 0.5, indexing="xy")
    points = torch.stack([gx, gy, torch.ones_like(gx)], dim=-1).reshape(-1, 3)
    rays_d = points @ intrins_inv.T @ c2w[:3, :3].T
    pts = (rendering[6].reshape(-1, 1) * rays_d + c2w[:3, 3]).reshape(H, W, 3)
    dn = torch.zeros_like(pts)
    dx = torch.cat([pts[2:, 1:-1] - pts[:-2, 1:-1]], dim=0)
    dy = torch.cat([pts[1:-1, 2:] - pts[1:-1, :-2]], dim=1)
    dn[1:-1, 1:-1, :] = F.normalize(torch.cross(dx, dy, dim=-1), dim=-1)
    rn = F.normalize(rendering[3:6], p=2, dim=0)
    rnw = (c2w[:3, :3] @ rn.reshape(3, -1)).reshape(3, H, W)
    dnl = (1 - (rnw * dn.permute(2, 0, 1)).sum(dim=0)).mean()
    return (1.0 - lam) * Ll1 + lam * (1.0 - ssim) + dnl * lam_dn + rendering[8].mean() * lam_dist


@pytest.mark.parametrize("H,W", [(200, 300), (540, 960)])
def test_end_to_end_through_the_network(H, W):
    """appearance_mapping + view_loss(appearance=...) against the torch loss lines: .grad of the rendering, of every network
    parameter and of the embedding row.  TF32 off in both arms."""
    import gof_appearance
    import gof_loss
    import gof_synth
    dev = torch.device("cuda")
    saved = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.deterministic)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.deterministic = True
    try:
        cam = gof_synth.make_camera(W, H, view=9)
        render, gt, _ = noise_inputs(H, W, H + W, 1, 1)
        torch.manual_seed(0)
        net = gof_appearance.AppearanceNetwork(67, 3).to(dev)
        emb_table = (torch.randn(4, 64, generator=torch.Generator().manual_seed(1)) * 1e-2).to(dev)
        gt_d = torch.from_numpy(gt).to(dev)
        res = []
        for fused in (True, False):
            rendering = torch.from_numpy(render).to(dev).requires_grad_(True)
            table = emb_table.clone().requires_grad_(True)
            for p in net.parameters():
                p.grad = None
            if fused:
                mapping = gof_appearance.appearance_mapping(rendering[:3], net, table[2])
                loss, _ = gof_loss.view_loss(rendering, gt_d, cam.world_view_transform, cam.tanfovx, cam.tanfovy, *LAM,
                                             appearance=mapping)
            else:
                loss = torch_train_loss(rendering, gt_d, cam, LAM, net, table[2])
            loss.backward()
            res.append([float(loss.detach()), rendering.grad.cpu().double(), table.grad[2].cpu().double()]
                       + [p.grad.cpu().double() for p in net.parameters()])
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.deterministic = saved
    (lf, *gf), (lt, *gt_) = res
    assert abs(lf - lt) <= 1e-5 * abs(lt), (lf, lt)
    names = ["rendering", "embedding"] + [n for n, _ in net.named_parameters()]
    for name, a, b in zip(names, gf, gt_):
        if name == "rendering":
            for ch in range(9):
                err = float((a[ch] - b[ch]).abs().max() / b[ch].abs().max().clamp_min(1e-30))
                assert err < (2e-3 if ch == 6 else 1e-4), (name, ch, err)
        else:
            err = float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))
            assert err < 1e-4, (name, err)
