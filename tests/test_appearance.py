"""CPU: gof_appearance (AppearanceNetwork, l1_loss_appearance) against the reference's OWN code: its AppearanceNetwork class
(scene/appearance_network.py) with the same weights, and its L1_loss_appearance (train.py) -- values and gradients w.r.t. the
image, the embedding and every network parameter.  The reference's results are stored in tests/golden/appearance_*.npz
(tests/golden/make_golden_appearance.py; a seeded sample of the larger arrays); both networks are initialised from the same
seed, which gives identical weights (same modules, same construction order)."""
import os
import types

import numpy as np
import pytest
import torch

import gof_appearance

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SHAPES = [(96, 160), (70, 101)]
SAMPLE = 256


def inputs(H, W):
    """(network seed, embedding table, image, ground truth) of one case."""
    g = torch.Generator().manual_seed(H * 1000 + W)
    return 0, torch.randn(8, 64, generator=g) * 1e-2, torch.rand(3, H, W, generator=g), torch.rand(3, H, W, generator=g)


def sample_idx(n, seed):
    return np.sort(np.random.default_rng(seed).choice(n, min(n, SAMPLE), replace=False))


def run(loss_fn, network, image, gt, emb_table, via_stub):
    """Loss at embedding row 5 and its gradients; with via_stub the loss takes the reference's (gaussians, idx) signature."""
    img = image.clone().requires_grad_(True)
    table = emb_table.clone().requires_grad_(True)
    for p in network.parameters():
        p.grad = None
    if via_stub:
        g = types.SimpleNamespace(get_apperance_embedding=lambda idx: table[idx], appearance_network=network)
        loss = loss_fn(img, gt, g, 5)
    else:
        loss = loss_fn(img, gt, network, table[5])
    loss.backward()
    return loss.detach(), img.grad, table.grad, [p.grad.clone() for p in network.parameters()]


def flat_sample(t, seed):
    f = t.detach().flatten()
    return f[torch.from_numpy(sample_idx(f.numel(), seed))].double().numpy()


@pytest.mark.parametrize("H,W", SHAPES)
def test_network_and_loss_equal_reference(H, W):
    z = np.load(os.path.join(GOLDEN, f"appearance_{H}x{W}.npz"))
    seed, emb_table, image, gt = inputs(H, W)
    torch.manual_seed(seed)
    net = gof_appearance.AppearanceNetwork(67, 3)
    assert [k for k, _ in net.named_parameters()] == [str(k) for k in z["param_names"]]     # same parameter names / shapes
    lo, gio, gto, gpo = run(gof_appearance.l1_loss_appearance, net, image, gt, emb_table, False)

    def close(a, b, rtol, atol):
        return np.all(np.abs(a - b) <= atol + rtol * np.abs(b))

    assert close(float(lo), float(z["loss"]), 1e-6, 1e-7)
    assert close(flat_sample(gio, 1), z["grad_image"], 1e-5, 1e-8) and close(gto.double().numpy(), z["grad_table"], 1e-5, 1e-8)
    for i, a in enumerate(gpo):
        assert close(flat_sample(a, 10 + i), z[f"grad_param{i}"], 1e-4, 1e-7), str(z["param_names"][i])
    # the transformed image (evaluation path, train.py:200)
    with torch.no_grad():
        to = gof_appearance.l1_loss_appearance(image, gt, net, emb_table[2], return_transformed_image=True)
    assert close(flat_sample(to, 2), z["transformed"], 1e-6, 1e-7)


def test_flat_gradient_packing_round_trip():
    net = gof_appearance.AppearanceNetwork(67, 3)
    n = gof_appearance.appearance_numel(net)
    assert n == sum(p.numel() for p in net.parameters()) + 64
    for i, p in enumerate(net.parameters()):
        p.grad = torch.full_like(p, float(i + 1))
    flat = torch.zeros(n)
    gof_appearance.appearance_grads_flat(net, torch.arange(64.0), flat)
    want = [p.grad.clone() for p in net.parameters()]
    emb = gof_appearance.load_flat_grads_(net, flat * 2)
    for p, w in zip(net.parameters(), want):
        assert torch.equal(p.grad, 2 * w)
    assert torch.equal(emb, 2 * torch.arange(64.0))
