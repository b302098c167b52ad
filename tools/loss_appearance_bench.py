#!/usr/bin/env python
"""Developer timing (GPU box): the per-view loss with decoupled appearance (train.py:151-188 with 157-159), forward +
backward at 1920 x 1080, in two arms that both run the appearance network:

  torch:  gof_appearance.l1_loss_appearance + SSIM (depthwise conv2d) + depth_to_normal + distortion, in torch ops
  fused:  gof_appearance.appearance_mapping + gof_loss.view_loss(..., appearance=mapping)

and the network's own share (appearance_mapping forward + backward from a fixed upstream gradient), which is common to
both.  The torch arm is a restatement for TIMING and a cross-check only; parity is pinned by
tests/test_gpu_view_loss_appearance.py.  cuDNN runs with torch's defaults (TF32 convolutions), as training does.
Writes tool_out/loss_appearance_bench.json."""
import json
import math
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "gaussian-opacity-fields_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gof_appearance  # noqa: E402
import gof_loss  # noqa: E402
import gof_synth  # noqa: E402
from quick_bench import time_it  # noqa: E402


def torch_loss(rendering, gt, wvt, tanfovx, tanfovy, lam, lam_dn, lam_dist, window, network, embedding):
    image = rendering[:3]
    Ll1 = gof_appearance.l1_loss_appearance(image, gt, network, embedding)
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


def gpu_info():
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return info


def main():
    dev = torch.device("cuda")
    W, H = 1920, 1080
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
    torch.manual_seed(0)
    net = gof_appearance.AppearanceNetwork(67, 3).to(dev)
    table = (torch.randn(8, 64, generator=g) * 1e-2).to(dev).requires_grad_(True)
    _, _, Hc, Wc = gof_appearance.crop_window(H, W)
    g_mapping = torch.rand(3, Hc, Wc, generator=g).to(dev)

    def zero():
        rendering.grad = table.grad = None
        for p in net.parameters():
            p.grad = None

    def fused():
        zero()
        mapping = gof_appearance.appearance_mapping(rendering[:3], net, table[2])
        loss, _ = gof_loss.view_loss(rendering, gt, cam.world_view_transform, cam.tanfovx, cam.tanfovy, *lam, rotation=rot,
                                     appearance=mapping)
        loss.backward()
        return loss

    def stock():
        zero()
        loss = torch_loss(rendering, gt, wvt, cam.tanfovx, cam.tanfovy, *lam, window, net, table[2])
        loss.backward()
        return loss

    def network():
        zero()
        mapping = gof_appearance.appearance_mapping(rendering[:3], net, table[2])
        (mapping * g_mapping).sum().backward()

    lf = fused(); gf = rendering.grad.clone()
    ls = stock(); gs_ = rendering.grad.clone()
    res = {"shape": f"{W}x{H}", "crop": f"{Wc}x{Hc}"}
    for _ in range(2):          # alternate the arms; the second round is reported
        res.update(fused_ms=time_it(fused, n_warm=5, n=30), torch_ms=time_it(stock, n_warm=5, n=30),
                   network_ms=time_it(network, n_warm=5, n=30))
    res["loss_rel_diff"] = float((lf - ls).detach().abs() / ls.detach().abs())
    # rgb: the channels the appearance L1 changes; all nine include the depth channel, whose gradient on a uniform-noise
    # depth map (near-degenerate depth normals) differs between any two fp32 formulations
    res["grad_rel_diff_rgb"] = float((gf[:3] - gs_[:3]).abs().max() / gs_[:3].abs().max())
    res["grad_rel_diff"] = float((gf - gs_).abs().max() / gs_.abs().max())
    res["speedup"] = res["torch_ms"] / res["fused_ms"]
    res["loss_only_torch_ms"] = res["torch_ms"] - res["network_ms"]
    res["loss_only_fused_ms"] = res["fused_ms"] - res["network_ms"]
    res.update(gpu_info())
    print(json.dumps(res), flush=True)
    os.makedirs(os.path.join(ROOT, "tool_out"), exist_ok=True)
    json.dump(res, open(os.path.join(ROOT, "tool_out", "loss_appearance_bench.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
