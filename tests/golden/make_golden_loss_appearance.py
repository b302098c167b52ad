#!/usr/bin/env python
"""Golden vectors for the per-view training loss with decoupled appearance (train.py:151-188 with 157-159 of the reference):
generated HERE by executing the reference's own Python on the CPU -- L1_loss_appearance (train.py:67-88, staged by
baseline/stage_ref.sh), l1_loss / ssim (utils/loss_utils.py) and depth_to_normal (utils/depth_utils.py), the latter two
loaded as make_golden_loss.py does.  The `gaussians` handed to L1_loss_appearance is a stub whose appearance_network
returns a fixed leaf `mapping`, so that the stored image gradient is the loss's direct one and mapping.grad is
d loss / d mapping.

Each tests/golden/loss_app_<H>x<W>.npz holds the inputs, every term and the gradient of the PLAIN loss under the keys of
make_golden_loss.py (the same lines with the plain l1_loss), and the appearance loss under app_*: mapping [3,Hc,Wc], its
crop (top, left), app_Ll1, app_loss, app_grad_rgb = d loss / d rendering[:3] (channels 3-8 equal the plain `grad`) and
grad_mapping.

  python tests/golden/make_golden_loss_appearance.py"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden_loss as mgl  # noqa: E402  (puts the package on sys.path)
import _refpy  # noqa: E402
import gof_appearance  # noqa: E402
import gof_synth  # noqa: E402

CASES = {   # (H, W): crop = (top, left, Hc, Wc) of train.py:70-75, stated for the reader and checked against crop_window
    (48, 72): dict(seed=11, view=5, lambdas=(0.2, 0.05, 100.0), crop=(8, 4, 32, 64)),
    (70, 101): dict(seed=12, view=23, lambdas=(0.35, 0.3, 10.0), crop=(3, 2, 64, 96)),
    # the crop is the whole image; the geometry terms are off (before iteration 15000) and the depth is zero, which keeps
    # the file small (no depth normals to store) and pins the zero-depth branch of depth_to_normal
    (96, 160): dict(seed=13, view=40, lambdas=(0.2, 0.0, 0.0), crop=(0, 0, 96, 160), zero_depth=True),
}


def on_grid(x, step):
    """x rounded to a multiple of the power of two `step`: short mantissas keep the stored files small."""
    return torch.round(x / step) * step


def make_inputs(H, W, seed, Hc, Wc):
    """make_golden_loss.py's render and gt on coarse dyadic grids (rgb, gt and the mapping in steps of 2^-8, so exact ties
    fl(mapping * rgb) == gt occur too), and a mapping in [0.6, 1.4] so that both signs of mapping * rgb - gt occur."""
    render, gt = mgl.make_inputs(dict(H=H, W=W, seed=seed))
    for ch, step in ((slice(0, 3), 2.0 ** -8), (slice(3, 6), 2.0 ** -6), (6, 2.0 ** -10), (7, 2.0 ** -4), (8, 2.0 ** -16)):
        render[ch] = on_grid(render[ch], step)
    g = torch.Generator().manual_seed(seed + 100)
    mapping = on_grid(0.6 + 0.8 * torch.rand(1, 3, Hc, Wc, generator=g), 2.0 ** -8)
    return render.contiguous(), on_grid(gt, 2.0 ** -8).contiguous(), mapping


def train_loss(lu, du, ref_app, view, rendering, gt, lambdas, mapping=None):
    """train.py:151-188, line by line; with `mapping` the decoupled-appearance branch (157-159) through a stub model."""
    lam_dssim, lam_dn, lam_dist = lambdas
    image = rendering[:3, :, :]
    Ll1 = lu.l1_loss(image, gt)
    if mapping is not None:
        def network(x):
            assert x.shape == (1, 67, mapping.shape[2] // 32, mapping.shape[3] // 32), x.shape
            return mapping
        gaussians = types.SimpleNamespace(get_apperance_embedding=lambda idx: torch.zeros(64), appearance_network=network)
        Ll1 = ref_app(image, gt, gaussians, 0)
    rgb_loss = (1.0 - lam_dssim) * Ll1 + lam_dssim * (1.0 - lu.ssim(image, gt))
    distortion_loss = rendering[8, :, :].mean()
    depth = rendering[6, :, :]
    depth_normal, _ = du.depth_to_normal(view, depth[None, ...])
    depth_normal = depth_normal.permute(2, 0, 1)
    render_normal = torch.nn.functional.normalize(rendering[3:6, :, :], p=2, dim=0)
    c2w = (view.world_view_transform.T).inverse()
    normal2 = c2w[:3, :3] @ render_normal.reshape(3, -1)
    render_normal_world = normal2.reshape(3, *render_normal.shape[1:])
    normal_error = 1 - (render_normal_world * depth_normal).sum(dim=0)
    depth_normal_loss = normal_error.mean()
    loss = rgb_loss + depth_normal_loss * lam_dn + distortion_loss * lam_dist
    return loss, Ll1, lu.ssim(image, gt), distortion_loss, depth_normal_loss, depth_normal


def main():
    lu, du = mgl.load_ref_module("utils/loss_utils.py"), mgl.load_ref_module("utils/depth_utils.py")
    assert _refpy.staged("text", "train.py") is not None, "run baseline/stage_ref.sh first"
    ref_app = _refpy.ref_function("train.py", "L1_loss_appearance", {"torch": torch, "l1_loss": lu.l1_loss})
    for (H, W), cfg in CASES.items():
        top, left, Hc, Wc = cfg["crop"]
        assert gof_appearance.crop_window(H, W) == (top, left, Hc, Wc)
        cam = gof_synth.make_camera(W, H, view=cfg["view"])
        view = mgl.View(cam)
        render0, gt, mapping0 = make_inputs(H, W, cfg["seed"], Hc, Wc)
        if cfg.get("zero_depth"):
            render0[6] = 0.0
        rec = dict(render=render0.numpy(), gt=gt.numpy(), world_view_transform=cam.world_view_transform.numpy(),
                   tanfovx=np.float64(cam.tanfovx), tanfovy=np.float64(cam.tanfovy), lambdas=np.array(cfg["lambdas"], np.float64))
        # the plain loss, under make_golden_loss.py's keys
        rendering = render0.clone().requires_grad_(True)
        loss, Ll1, ssim_v, dist, dnl, dn = train_loss(lu, du, ref_app, view, rendering, gt, cfg["lambdas"])
        loss.backward()
        rec.update(Ll1=Ll1.detach().numpy(), ssim=ssim_v.detach().numpy(), distortion_loss=dist.detach().numpy(),
                   depth_normal_loss=dnl.detach().numpy(), depth_normal=dn.detach().numpy(), loss=loss.detach().numpy(),
                   grad=rendering.grad.numpy())
        # the appearance loss
        rendering = render0.clone().requires_grad_(True)
        mapping = mapping0.clone().requires_grad_(True)
        aloss, aLl1, *_ = train_loss(lu, du, ref_app, view, rendering, gt, cfg["lambdas"], mapping)
        aloss.backward()
        assert torch.equal(rendering.grad[3:], torch.from_numpy(rec["grad"][3:]))
        rec.update(mapping=mapping0[0].numpy(), top=np.int64(top), left=np.int64(left), app_Ll1=aLl1.detach().numpy(),
                   app_loss=aloss.detach().numpy(), app_grad_rgb=rendering.grad[:3].numpy(), grad_mapping=mapping.grad[0].numpy())
        out = os.path.join(HERE, f"loss_app_{H}x{W}.npz")
        np.savez_compressed(out, **rec)
        print(out, os.path.getsize(out), loss.item(), aloss.item(), aLl1.item())


if __name__ == "__main__":
    main()
