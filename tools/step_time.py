#!/usr/bin/env python
"""Developer timing (GPU box): ms per fwd+bwd step of a config over the 64-view ring (device-resident inputs, CUDA events) and
the per-kernel split from the library's event brackets.  Environment knobs (GOF_STAGE, GOF_BINNING, GOF_FWD_OCC, ...) are read
by the library once per process, so A/B runs are separate invocations:   GOF_STAGE=regs python tools/step_time.py C3 30 label"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "gaussian-opacity-fields_b200"))
import _util  # noqa: E402
import gof_dp  # noqa: E402
import gof_synth  # noqa: E402
from diff_gaussian_rasterization import _C  # noqa: E402

name = sys.argv[1] if len(sys.argv) > 1 else "C3"
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 30
label = sys.argv[3] if len(sys.argv) > 3 else "default"
dev = torch.device("cuda")
cams = [gof_synth.make_scene(name, view=v)[0] for v in range(16)]
gs = gof_synth.make_scene(name, view=0)[1]
fas = [_util.fwd_args(c, gs, dev) for c in cams]
H, W, P = cams[0].image_height, cams[0].image_width, gs["means3D"].shape[0]
grad = torch.randn(9, H, W, device=dev)
bucket = gof_dp.GradBucket(P, 16, dev)


def step(i):
    fa = fas[i % len(fas)]
    R, color, radii, geom, binning, img = _C.rasterize_gaussians(*fa)
    # (the backward writes every element of its outputs: no zero fill)
    _C.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, grad), _out=bucket.views)
    return R


for i in range(5):
    step(i)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for i in range(steps):
    step(5 + i)
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / steps
_C.profile_reset(); _C.profile_enable(True)
for i in range(5):
    step(i)
torch.cuda.synchronize(); _C.profile_enable(False)
prof = {k: round(v[1] / 5, 4) for k, v in sorted(_C.profile_report().items(), key=lambda kv: -kv[1][1])}
out = {"label": label, "config": name, "ms_per_step": round(ms, 4), "views_per_s": round(1e3 / ms, 1), "kernels_ms": prof,
       "env": {k: v for k, v in os.environ.items() if k.startswith("GOF_")}}
print(json.dumps(out), flush=True)
os.makedirs(os.path.join(ROOT, "tool_out"), exist_ok=True)
with open(os.path.join(ROOT, "tool_out", "step_time.jsonl"), "a") as f:
    f.write(json.dumps(out) + "\n")
