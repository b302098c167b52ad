"""GPU: the alpha-support boxes only skip work.  Rendering with GOF_CULL=0 (every staged Gaussian visited by every
warp, like the reference) and GOF_CULL=1 must give BIT-identical images and per-pixel counters, and gradients that
differ only by float summation order -- on ordinary, needle-shaped and sub-pixel Gaussians, on pixels that saturate at
batch and group boundaries, and on alphas just above 1/255.  The same holds bit for bit for the
opacity-field query (image, per-point alpha and colour, last contributor and contributor count), also on Gaussians thinner
than a pixel that only its corner rays meet."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _run(cull, inputs, path):
    env = dict(os.environ, GOF_CULL=cull)
    env["PYTHONPATH"] = os.pathsep.join([HERE, os.path.join(HERE, "..", "gaussian-opacity-fields_b200"), env.get("PYTHONPATH", "")])
    subprocess.check_call([sys.executable, os.path.join(HERE, "_cull_probe.py"), inputs, path], env=env)
    return np.load(path)


def test_culling_never_changes_results():
    import _cull_probe
    with tempfile.TemporaryDirectory() as d:
        inputs = os.path.join(d, "inputs.npz")
        _cull_probe.make_inputs(inputs)      # once: both modes must see bit-identical Gaussians
        a = _run("0", inputs, os.path.join(d, "a.npz"))
        b = _run("1", inputs, os.path.join(d, "b.npz"))
        for k in a.files:
            if k.endswith(("_color", "_ncontrib", "_accum", "_int_alpha", "_int_colint")):
                np.testing.assert_array_equal(a[k].view(np.int32), b[k].view(np.int32), err_msg=k)
            else:
                den = max(np.abs(a[k]).max(), 1e-30)
                diff = np.abs(a[k].astype(np.float64) - b[k]) / den
                if k.endswith(("dscales", "drot", "dmeans3D")):
                    # K8 multiplies the summation-order noise of dv2g (checked to 1e-5 below) by ~1/scale^2, up to 1e5 for
                    # the needles of scene b: single elements are noise-dominated, so bound the bulk of the distribution
                    assert np.quantile(diff, 0.99) < 1e-2, f"{k}: q99 {np.quantile(diff, 0.99)}"
                else:
                    assert diff.max() < 1e-5, f"{k}: {diff.max()}"
        assert sum(k.endswith("_int_alpha") for k in a.files) == 6 and (a["n_int_alpha"] < 1).sum() > 1000
