"""TEST INFRASTRUCTURE -- fp64 restatement of the per-view training loss with the decoupled-appearance L1 (train.py:67-88,
157-159 of the reference) and of its gradients with respect to the 9-channel render and the appearance mapping.

The SSIM, depth-normal and distortion terms are those of oracle/loss_oracle.py, on the whole image; only the L1 term
changes: mean over the crop (top, left, Hc, Wc) of |mapping * rgb - gt|.  So this takes loss_oracle.view_loss's result and
swaps its L1 term and the L1 part of its rgb gradient for the appearance ones.  Pinned by tests/golden/loss_app_*.npz
(tests/golden/make_golden_loss_appearance.py, the reference's own Python)."""
import numpy as np

import loss_oracle


def view_loss(render, gt, world_view_transform, tanfovx, tanfovy, lambdas, mapping, top, left, need_grad=True):
    """loss_oracle.view_loss's dict with Ll1 and loss of the appearance L1, plus marginal [3,Hc,Wc]: the crop pixels whose
    float32 product fl(mapping * rgb) could round onto gt (|mapping * rgb - gt| within half an ulp of the product, not equal),
    where the sign of the L1 term is not decided; with need_grad, grad [9,H,W] and grad_mapping [3,Hc,Wc]."""
    out = loss_oracle.view_loss(render, gt, world_view_transform, tanfovx, tanfovy, lambdas, need_grad)
    render, gt = np.asarray(render, np.float64), np.asarray(gt, np.float64)
    mapping = np.asarray(mapping, np.float64).reshape(3, *np.shape(mapping)[-2:])
    lam = float(lambdas[0])
    img = render[:3]
    Hc, Wc = mapping.shape[1:]
    crop = (slice(0, 3), slice(top, top + Hc), slice(left, left + Wc))
    prod = mapping * img[crop]
    diff = prod - gt[crop]
    Ll1 = np.abs(diff).mean()
    out["loss"] += (1.0 - lam) * (Ll1 - out["Ll1"])
    out["Ll1"] = Ll1
    out["marginal"] = (np.abs(diff) <= 2.0 ** -24 * np.abs(prod)) & (diff != 0)
    if not need_grad:
        return out
    grad = out["grad"]
    grad[:3] -= (1.0 - lam) * np.sign(img - gt) / img.size        # the plain L1 part
    k1 = (1.0 - lam) * np.sign(diff) / mapping.size
    grad[crop] += k1 * mapping
    out["grad_mapping"] = k1 * img[crop]
    return out
