"""GPU: gof_densify.densify_and_prune against the reference's OWN methods (scene/gaussian_model.py: densify_and_prune,
densify_and_clone, densify_and_split, densification_postfix, cat_tensors_to_optimizer, prune_points, _prune_optimizer --
compiled from the unmodified source text into a stub class around a real torch.optim.Adam), through their results stored in
tests/golden/densify_*.npz.  torch.normal is the only thing replaced on the reference side: it returns std * the same
standard-normal samples our kernel is given, so every surviving parameter row, both Adam moments and the row order can be
compared exactly (positions / scalings to float rounding)."""

import numpy as np
import pytest
import torch

import _liveref

pytestmark = pytest.mark.gpu
METHODS = ["densify_and_prune", "densify_and_clone", "densify_and_split", "densification_postfix", "cat_tensors_to_optimizer",
           "prune_points", "_prune_optimizer"]
NAMES = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity", "scaling": "_scaling", "rotation": "_rotation"}
CASES = [(20_003, 20), (5_000, None), (257, 20)]
EXTENT, MAX_GRAD, MIN_OP = 1.7, 2e-4, 0.05


def _model(P, dev, gen, methods=None):
    """The state GaussianModel.densify_and_prune reads, in a stub class around a real torch.optim.Adam (one step taken, so that
    every group has Adam state).  `methods`: the reference's own methods to bind (tests/golden/make_golden_ref_python.py)."""
    Stub = type("GaussianModelStub", (), dict(methods or {}))
    Stub.get_xyz = property(lambda s: s._xyz)
    Stub.get_scaling = property(lambda s: torch.exp(s._scaling))
    Stub.get_opacity = property(lambda s: torch.sigmoid(s._opacity))
    g = Stub()
    g.scaling_inverse_activation = torch.log
    g.percent_dense = 0.01
    r = lambda *shape: torch.randn(*shape, generator=gen).to(dev)
    g._xyz = torch.nn.Parameter(r(P, 3))
    g._features_dc = torch.nn.Parameter(r(P, 1, 3))
    g._features_rest = torch.nn.Parameter(r(P, 15, 3))
    g._opacity = torch.nn.Parameter(r(P, 1) * 2.0)
    g._scaling = torch.nn.Parameter(torch.log(torch.rand(P, 3, generator=gen) * 0.04 + 1e-3).to(dev))
    g._rotation = torch.nn.Parameter(r(P, 4))
    groups = [{"params": [getattr(g, a)], "lr": 1e-3, "name": n} for n, a in NAMES.items()]
    groups.append({"params": [torch.nn.Parameter(r(4, 4))], "lr": 1e-3, "name": "appearance_network"})      # skipped by the reference's loops
    g.optimizer = torch.optim.Adam(groups, lr=0.0, eps=1e-15)
    for grp in g.optimizer.param_groups:
        grp["params"][0].grad = torch.randn(grp["params"][0].shape, generator=gen).to(dev)
    g.optimizer.step()
    g.xyz_gradient_accum = (torch.rand(P, 1, generator=gen) * 6e-4).to(dev)
    g.xyz_gradient_accum_abs = (torch.rand(P, 1, generator=gen) * 9e-4).to(dev)
    g.xyz_gradient_accum_abs_max = torch.zeros(P, 1, device=dev)
    g.denom = torch.randint(0, 3, (P, 1), generator=gen).float().to(dev)              # zeros: the NaN -> 0 path
    g.max_radii2D = (torch.rand(P, generator=gen) * 40).to(dev)
    return g


def inputs(P, dev, methods=None):
    """(model, parameters, Adam moments, statistics, the standard-normal samples of the split / clone positions)."""
    gen = torch.Generator().manual_seed(P)
    g = _model(P, dev, gen, methods)
    params = {n: getattr(g, a).detach().clone() for n, a in NAMES.items()}
    m = {n: g.optimizer.state[getattr(g, a)]["exp_avg"].clone() for n, a in NAMES.items()}
    v = {n: g.optimizer.state[getattr(g, a)]["exp_avg_sq"].clone() for n, a in NAMES.items()}
    stats = (g.xyz_gradient_accum.clone(), g.xyz_gradient_accum_abs.clone(), g.denom.clone())
    noise = torch.randn(3, P, 3, generator=gen).to(dev)
    return g, params, m, v, stats, noise


def record(P, max_screen, dev, methods, feed):
    """The reference's densify_and_prune (its methods in `methods`, torch.normal replaced by `feed`) on case P: the stored
    result of test_densify_and_prune_equals_reference."""
    g, params, m, v, (acc, acc_abs, den), noise = inputs(P, dev, methods)
    # the samples the reference's two torch.normal calls will consume: rows of the selected Gaussians, in order
    grads_abs = (acc_abs / den).reshape(-1); grads_abs[grads_abs.isnan()] = 0.0
    grads = (acc / den).reshape(-1); grads[grads.isnan()] = 0.0
    ratio = (grads >= MAX_GRAD).float().mean()
    Q = torch.quantile(grads_abs, 1 - ratio)
    sel = (grads >= MAX_GRAD) | (grads_abs >= Q)
    smax = torch.exp(params["scaling"]).max(dim=1).values
    clone, split = sel & (smax <= 0.01 * EXTENT), sel & (smax > 0.01 * EXTENT)
    feed["queue"] = [noise[0][clone], torch.cat([noise[1][split], noise[2][split]])]
    g.densify_and_prune(MAX_GRAD, MIN_OP, EXTENT, max_screen)
    assert not feed["queue"]
    n = g._xyz.shape[0]
    rows = np.sort(np.random.default_rng(n).choice(n, min(n, 256), replace=False))
    out = {"rows": rows.astype(np.int32)}
    for k, a in NAMES.items():
        p, st = getattr(g, a).detach(), g.optimizer.state[getattr(g, a)]
        if k in ("xyz", "scaling"):
            out[k] = p[torch.from_numpy(rows).to(dev)].cpu().numpy()
        else:
            out[k] = _liveref.digest(p)
        out["exp_avg_" + k], out["exp_avg_sq_" + k] = _liveref.digest(st["exp_avg"]), _liveref.digest(st["exp_avg_sq"])
    return out


@pytest.mark.parametrize("P,max_screen", CASES)
def test_densify_and_prune_equals_reference(P, max_screen):
    """Against the reference's own GaussianModel methods (scene/gaussian_model.py: densify_and_prune, densify_and_clone,
    densify_and_split, densification_postfix, cat_tensors_to_optimizer, prune_points, _prune_optimizer) on the same state, as
    stored in tests/golden/densify_<P>.npz: every surviving parameter row, both Adam moments and the row order exactly, positions
    and scalings to float rounding."""
    import gof_densify
    dev = torch.device("cuda")
    z = _liveref.load_npz(f"densify_{P}.npz")
    _g, params, m, v, (acc, acc_abs, den), noise = inputs(P, dev)
    ours = gof_densify.densify_and_prune(params, m, v, acc, acc_abs, den, MAX_GRAD, MIN_OP, EXTENT, max_screen, noise=noise)
    n = ours.params["xyz"].shape[0]
    assert n == sum(ours.counts) and np.array_equal(np.sort(np.random.default_rng(n).choice(n, min(n, 256), replace=False)), z["rows"])
    rows = torch.from_numpy(z["rows"]).to(dev)
    for k in NAMES:
        if k in ("xyz", "scaling"):
            assert torch.allclose(ours.params[k][rows].cpu(), torch.from_numpy(z[k]), rtol=1e-5, atol=1e-6), k
        else:
            assert _liveref.digest(ours.params[k]) == str(z[k]), k
        assert _liveref.digest(ours.exp_avg[k]) == str(z["exp_avg_" + k]), k
        assert _liveref.digest(ours.exp_avg_sq[k]) == str(z["exp_avg_sq_" + k]), k
    assert ours.counts[1] > 0 and ours.counts[2] > 0 and ours.counts[2] == ours.counts[3]
    # the library's own sampler: same decisions, positions within a few sigma of the parents
    own = gof_densify.densify_and_prune(params, m, v, acc, acc_abs, den, MAX_GRAD, MIN_OP, EXTENT, max_screen, seed=7)
    assert own.counts == ours.counts and torch.equal(own.src_index, ours.src_index)
    new = own.kind > 0
    parent = params["xyz"][own.src_index.long()]
    dist = (own.params["xyz"] - parent).norm(dim=1)
    assert float(dist[~new].max()) == 0.0
    sig = torch.exp(params["scaling"])[own.src_index.long()].max(dim=1).values
    assert float((dist[new] / sig[new]).max()) < 8.0 and float((dist[new] / sig[new]).mean()) > 0.3
