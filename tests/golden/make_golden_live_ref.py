"""Regenerates tests/golden/live_*.npz: the unmodified reference extension (oracle/_ref/gof_ref_C*.so, built by
oracle/build_ref.sh from the original project) run on a CUDA device on every case of tests/_liveref.py.

  python tests/golden/make_golden_live_ref.py [OUT_DIR]      (default: tests/golden)"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle")]
import _util  # noqa: E402  (puts the package on sys.path)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import _liveref  # noqa: E402


def record_grad_fp64(ref, dev):
    """err(reference, fp64) per gradient (max-norm, relative L2) at the C2 view of test_gpu_grad_fp64.py."""
    import test_gpu_grad_fp64 as t
    cam, gs, fa, dL = t.c2_inputs(dev)
    R, _color, radii, geom, binning, img = ref.rasterize_gaussians(*fa)
    gr = ref.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, dL.to(dev)))
    _oradii, od = t.fp64_gradients(cam, gs, dL)
    return {n: np.array(t._err(gr[i].cpu().numpy(), od[t.OMAP[n]])) for i, n in enumerate(t.NAMES) if n in t.OMAP}


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    os.makedirs(out_dir, exist_ok=True)
    ref = _util.load_ref()
    assert ref is not None, "oracle/_ref/gof_ref_C*.so missing: run oracle/build_ref.sh where the original project exists"
    dev = torch.device("cuda")
    recs = {name: _liveref.record(ref, name, dev) for name in _liveref.CASES}
    recs["integrate_1080p"] = _liveref.record_integrate(ref, dev)
    recs["grad_fp64_c2"] = record_grad_fp64(ref, dev)
    for name, rec in recs.items():
        path = os.path.join(out_dir, f"live_{name}.npz")
        np.savez_compressed(path, **rec)
        print(f"[make_golden_live_ref] {path}: {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
