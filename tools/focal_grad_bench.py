"""Cost of the focal-length gradient: the backward of one C3 view (1 M Gaussians, 1920x1080) with and without the intrinsics
outputs (`_C.rasterize_gaussians_backward(..., _intrinsics=True)`, gof_rasterize_backward_ex with dL_dtan_fov), alternating calls over
one forward state after warm-up.  CUDA events around single calls; medians and spreads are reported, plus the per-kernel split
of the library's event brackets (render_bwd vs render_bwd_rays + focal_grad_sum).

Checks that the focal-length outputs of two calls are bit-identical, and that the parameter gradients of the two variants are
bit-identical wherever the blend stage (whose double atomics may round a Gaussian's sum differently from call to call) produced
identical values.

  python tools/focal_grad_bench.py [--config C3] [--view 5] [--reps 30]

Prints one line per variant and a JSON summary with the card name and its power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "gaussian-opacity-fields_b200"), os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import _util  # noqa: E402
import gof_synth  # noqa: E402

BLEND = (0, 1, 2, 8)


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def _bits(t):
    return t.contiguous().view(torch.int32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C3")
    ap.add_argument("--view", type=int, default=5)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    from diff_gaussian_rasterization import _C
    dev = torch.device("cuda")
    cam, gs = gof_synth.make_scene(a.config, view=a.view)
    fa = _util.fwd_args(cam, gs, dev)
    R, _color, radii, geom, binning, img = _C.rasterize_gaussians(*fa)
    dL = torch.randn(9, cam.image_height, cam.image_width, generator=torch.Generator().manual_seed(1)).to(dev)
    args = _util.bwd_args(fa, radii, geom, R, binning, img, dL)
    P = gs["means3D"].shape[0]

    def call(fov):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = _C.rasterize_gaussians_backward(*args, _intrinsics=fov)
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1), out

    for _ in range(a.warmup):
        call(False)
        call(True)
    ms = {False: [], True: []}
    for i in range(a.reps):
        for fov in ((False, True) if i % 2 == 0 else (True, False)):
            ms[fov].append(call(fov)[0])

    # per-kernel split, one bracketed call of each variant
    _C.profile_reset()
    _C.profile_enable(True)
    call(False)
    call(True)
    kernels = {k: v[1] for k, v in _C.profile_report().items() if k.startswith(("preprocess_bwd", "focal_grad", "render_bwd"))}
    _C.profile_enable(False)

    _t, plain = call(False)
    plain = [t.clone() for t in plain]
    _t, fa_ = call(True)
    fa_ = [t.clone() for t in fa_]
    _t, fb_ = call(True)
    same = torch.ones(P, dtype=torch.bool, device=dev)
    for i in BLEND:
        same &= (_bits(plain[i]).view(P, -1) == _bits(fa_[i]).view(P, -1)).all(dim=1)
    identical = all(torch.equal(_bits(plain[i]).view(P, -1)[same], _bits(fa_[i]).view(P, -1)[same])
                    for i in range(9) if plain[i].numel() and i not in BLEND)
    fov_repro = all(torch.equal(_bits(fa_[i]), _bits(fb_[i])) for i in (9, 10))

    med = {k: float(np.median(v)) for k, v in ms.items()}
    for fov in (False, True):
        v = np.array(ms[fov])
        print(f"backward {'with' if fov else 'without'} intrinsics: median {med[fov]:.3f} ms  (min {v.min():.3f}, max {v.max():.3f}, n={len(v)})")
    print(f"kernel ms (one call each): {kernels}")
    summary = dict(config=a.config, view=a.view, P=P, W=cam.image_width, H=cam.image_height, card=_card(), reps=a.reps,
                   backward_ms=med[False], backward_intrinsics_ms=med[True], overhead_ms=med[True] - med[False],
                   overhead_pct=100.0 * (med[True] - med[False]) / med[False], kernels_ms=kernels,
                   gaussians_with_identical_blend_outputs=int(same.sum()), parameter_gradients_bit_identical=bool(identical),
                   focal_outputs_bit_identical=bool(fov_repro), dL_dtanfov=[float(fa_[9]), float(fa_[10])])
    print(json.dumps(summary))
    if not identical or not fov_repro:
        sys.exit(1)


if __name__ == "__main__":
    main()
