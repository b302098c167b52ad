#!/usr/bin/env python
"""Developer timing (GPU box, next round): one full training iteration around the rasterizer, two ways --

  ours:       gof_params.activate -> GaussianRasterizer (this repo) -> gof_loss.view_loss -> backward -> gof_params.adam_step
  stock:      torch activations (scene/gaussian_model.py:152-194 restated) -> the same rasterizer module given on the command
              line (ours | ref) -> torch loss (tools/loss_bench.torch_loss) -> backward -> torch.optim.Adam(eps=1e-15)

python tools/train_step_bench.py [C2|C3] [ours|ref]     (ref = oracle/_ref reference extension for the stock arm)
Needs GOF_STAGED components; numbers only, parity is pinned by the tests."""
import json
import math
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in ("gaussian-opacity-fields_b200", "tests", "tools"):
    sys.path.insert(0, os.path.join(ROOT, p))
import _util  # noqa: E402
import gof_loss  # noqa: E402
import gof_params  # noqa: E402
import gof_synth  # noqa: E402
from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer  # noqa: E402
from loss_bench import torch_loss  # noqa: E402
from quick_bench import time_it  # noqa: E402

LRS = {"_xyz": 1.6e-4, "_features_dc": 2.5e-3, "_features_rest": 2.5e-3 / 20, "_opacity": 0.05, "_scaling": 0.005, "_rotation": 0.001}


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "C3"
    dev = torch.device("cuda")
    cam, gs = gof_synth.make_scene(name, view=3)
    H, W = cam.image_height, cam.image_width
    P = gs["means3D"].shape[0]
    filt = (torch.rand(P, 1) * 0.002).to(dev)
    raw0 = {"_xyz": gs["means3D"], "_scaling": torch.log(gs["scales"]), "_rotation": gs["rotations"],
            "_opacity": torch.logit(gs["opacities"].clamp(1e-4, 1 - 1e-4)), "_features_dc": gs["shs"][:, :1].contiguous(),
            "_features_rest": gs["shs"][:, 1:].contiguous()}
    gt = torch.rand(3, H, W).to(dev)
    rs = GaussianRasterizationSettings(
        image_height=H, image_width=W, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, kernel_size=0.0,
        subpixel_offset=torch.zeros((H, W, 2), device=dev), bg=torch.zeros(3, device=dev), scale_modifier=1.0,
        viewmatrix=cam.world_view_transform.to(dev), projmatrix=cam.full_proj_transform.to(dev), sh_degree=3,
        campos=cam.camera_center.to(dev), prefiltered=False, debug=False)
    rot = gof_loss.camera_rotation(cam.world_view_transform)
    gw = torch.tensor([math.exp(-(x - 5) ** 2 / (2 * 1.5 ** 2)) for x in range(11)])
    gw = gw / gw.sum()
    window = (gw[:, None] @ gw[None, :]).float()[None, None].expand(3, 1, 11, 11).contiguous().to(dev)
    lam = (0.2, 0.05, 100.0)
    out = {}

    # ---------------- ours ----------------
    raw = {k: v.clone().to(dev).requires_grad_(True) for k, v in raw0.items()}
    state = {k: (torch.zeros_like(v), torch.zeros_like(v)) for k, v in raw.items()}
    step = [0]

    def ours():
        step[0] += 1
        for v in raw.values():
            v.grad = None
        scales, rots, ops, shs = gof_params.activate(raw["_scaling"], raw["_rotation"], raw["_opacity"], filt, raw["_features_dc"], raw["_features_rest"])
        means2D = torch.zeros_like(raw["_xyz"], requires_grad=True)
        img, radii = GaussianRasterizer(rs)(means3D=raw["_xyz"], means2D=means2D, opacities=ops, shs=shs, scales=scales, rotations=rots)
        loss, _ = gof_loss.view_loss(img, gt, cam.world_view_transform, cam.tanfovx, cam.tanfovy, *lam, rotation=rot)
        loss.backward()
        with torch.no_grad():
            for k, v in raw.items():
                gof_params.adam_step(v.data, state[k][0], state[k][1], v.grad.contiguous(), LRS[k], step[0])
        return loss

    out["ours_ms"] = time_it(ours, n_warm=3, n=10)

    # ---------------- stock torch around the same rasterizer ----------------
    raw2 = {k: v.clone().to(dev).requires_grad_(True) for k, v in raw0.items()}
    opt = torch.optim.Adam([{"params": [v], "lr": LRS[k]} for k, v in raw2.items()], lr=0.0, eps=1e-15)

    def stock():
        opt.zero_grad(set_to_none=True)
        s = torch.exp(raw2["_scaling"])
        s2 = torch.square(s)
        scales = torch.sqrt(s2 + torch.square(filt))
        coef = torch.sqrt(s2.prod(dim=1) / (s2 + torch.square(filt)).prod(dim=1))
        ops = torch.sigmoid(raw2["_opacity"]) * coef[..., None]
        rots = F.normalize(raw2["_rotation"])
        shs = torch.cat((raw2["_features_dc"], raw2["_features_rest"]), dim=1)
        means2D = torch.zeros_like(raw2["_xyz"], requires_grad=True)
        img, radii = GaussianRasterizer(rs)(means3D=raw2["_xyz"], means2D=means2D, opacities=ops, shs=shs, scales=scales, rotations=rots)
        loss = torch_loss(img, gt, rs.viewmatrix, cam.tanfovx, cam.tanfovy, *lam, window)
        loss.backward()
        opt.step()
        return loss

    out["torch_around_our_rasterizer_ms"] = time_it(stock, n_warm=3, n=10)
    out["speedup"] = out["torch_around_our_rasterizer_ms"] / out["ours_ms"]
    print(name, json.dumps(out), flush=True)
    os.makedirs(os.path.join(ROOT, "tool_out"), exist_ok=True)
    json.dump(out, open(os.path.join(ROOT, "tool_out", "train_step_bench.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
