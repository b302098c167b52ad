"""Regenerates tests/golden/appearance_*.npz: the reference's own AppearanceNetwork (scene/appearance_network.py) and
L1_loss_appearance (train.py), staged unmodified by baseline/stage_ref.sh, on the inputs of tests/test_appearance.py.  CPU only.

  python tests/golden/make_golden_appearance.py [OUT_DIR]      (default: tests/golden)"""
import importlib.util
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import _util  # noqa: E402,F401  (puts the package on sys.path)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import _refpy  # noqa: E402
import test_appearance as t  # noqa: E402


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    path = _refpy.staged("scene", "appearance_network.py")
    assert path is not None and _refpy.ref_utils("loss_utils") is not None, "run baseline/stage_ref.sh first"
    spec = importlib.util.spec_from_file_location("gof_ref_appearance_network", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    ref_loss = _refpy.ref_function("train.py", "L1_loss_appearance", {"torch": torch, "l1_loss": _refpy.ref_utils("loss_utils").l1_loss})
    for H, W in t.SHAPES:
        seed, emb_table, image, gt = t.inputs(H, W)
        torch.manual_seed(seed)
        net = mod.AppearanceNetwork(67, 3)
        loss, gi, gtab, gp = t.run(ref_loss, net, image, gt, emb_table, True)
        rec = {"loss": float(loss), "grad_image": t.flat_sample(gi, 1), "grad_table": gtab.double().numpy(),
               "param_names": np.array([k for k, _ in net.named_parameters()])}
        rec.update({f"grad_param{i}": t.flat_sample(g, 10 + i) for i, g in enumerate(gp)})
        g = t.types.SimpleNamespace(get_apperance_embedding=lambda idx: emb_table[idx], appearance_network=net)
        with torch.no_grad():
            rec["transformed"] = t.flat_sample(ref_loss(image, gt, g, 2, return_transformed_image=True), 2)
        out = os.path.join(out_dir, f"appearance_{H}x{W}.npz")
        np.savez_compressed(out, **rec)
        print(f"[make_golden_appearance] {out}: {os.path.getsize(out)} bytes")


if __name__ == "__main__":
    main()
