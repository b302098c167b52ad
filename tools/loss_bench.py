#!/usr/bin/env python
"""Developer timing (GPU box): the fused per-view loss (gof_loss.view_loss, forward + backward) against the same loss
written with torch ops the way train.py:151-188 does it (depthwise conv2d SSIM, depth_to_normal with torch.cross, ...).
The torch version below is a restatement for TIMING and a cross-check only; parity is pinned elsewhere
(tests/test_gpu_view_loss.py against reference-generated goldens)."""
import json
import math
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "gaussian-opacity-fields_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gof_loss  # noqa: E402
import gof_synth  # noqa: E402
from quick_bench import time_it  # noqa: E402


def torch_loss(rendering, gt, wvt, tanfovx, tanfovy, lam, lam_dn, lam_dist, window):
    image = rendering[:3]
    Ll1 = (image - gt).abs().mean()
    conv = lambda x: F.conv2d(x[None], window, padding=5, groups=3)[0]
    mu1, mu2 = conv(image), conv(gt)
    s11, s22, s12 = conv(image * image) - mu1 * mu1, conv(gt * gt) - mu2 * mu2, conv(image * gt) - mu1 * mu2
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    ssim = (((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 * mu1 + mu2 * mu2 + C1) * (s11 + s22 + C2))).mean()
    H, W = rendering.shape[1:]
    c2w = torch.linalg.inv(wvt.t())
    fx, fy = W / (2 * tanfovx), H / (2 * tanfovy)
    gx, gy = torch.meshgrid(torch.arange(W, device=rendering.device).float() + 0.5, torch.arange(H, device=rendering.device).float() + 0.5, indexing="xy")
    k = torch.stack([(gx - W / 2) / fx, (gy - H / 2) / fy, torch.ones_like(gx)], dim=-1)
    rays_d = k @ c2w[:3, :3].t()
    pts = rendering[6][..., None] * rays_d + c2w[:3, 3]
    dn = torch.zeros_like(pts)
    dx, dy = pts[2:, 1:-1] - pts[:-2, 1:-1], pts[1:-1, 2:] - pts[1:-1, :-2]
    dn[1:-1, 1:-1] = F.normalize(torch.cross(dx, dy, dim=-1), dim=-1)
    rn = F.normalize(rendering[3:6], p=2, dim=0)
    rnw = (c2w[:3, :3] @ rn.reshape(3, -1)).reshape(3, H, W)
    dnl = (1 - (rnw * dn.permute(2, 0, 1)).sum(0)).mean()
    return (1 - lam) * Ll1 + lam * (1 - ssim) + lam_dn * dnl + lam_dist * rendering[8].mean()


def main():
    dev = torch.device("cuda")
    out = {}
    for (W, H) in ((800, 800), (1920, 1080)):
        cam = gof_synth.make_camera(W, H, view=7)
        g = torch.Generator().manual_seed(5)
        rendering = torch.rand(9, H, W, generator=g).to(dev).requires_grad_(True)
        gt = torch.rand(3, H, W, generator=g).to(dev)
        wvt = cam.world_view_transform.to(dev)
        rot = gof_loss.camera_rotation(cam.world_view_transform)
        gw = torch.tensor([math.exp(-(x - 5) ** 2 / (2 * 1.5 ** 2)) for x in range(11)])
        gw = gw / gw.sum()
        window = (gw[:, None] @ gw[None, :]).float()[None, None].expand(3, 1, 11, 11).contiguous().to(dev)
        lam = (0.2, 0.05, 100.0)

        def fused():
            rendering.grad = None
            loss, _ = gof_loss.view_loss(rendering, gt, cam.world_view_transform, cam.tanfovx, cam.tanfovy, *lam, rotation=rot)
            loss.backward()
            return loss

        def stock():
            rendering.grad = None
            loss = torch_loss(rendering, gt, wvt, cam.tanfovx, cam.tanfovy, *lam, window)
            loss.backward()
            return loss

        lf = fused(); gf = rendering.grad.clone()
        ls = stock(); gs_ = rendering.grad.clone()
        res = {"fused_ms": time_it(fused), "torch_ms": time_it(stock), "loss_rel_diff": float((lf - ls).abs() / ls.abs()),
               "grad_rel_diff": float((gf - gs_).abs().max() / gs_.abs().max())}
        res["speedup"] = res["torch_ms"] / res["fused_ms"]
        out[f"{W}x{H}"] = res
        print(W, H, json.dumps(res), flush=True)
    os.makedirs(os.path.join(ROOT, "tool_out"), exist_ok=True)
    json.dump(out, open(os.path.join(ROOT, "tool_out", "loss_bench.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
