"""gof_densify.densify_and_prune (csrc/densify.cu) against a plain restatement of the reference's densify_and_prune
(tests/_densify_ref.py), at every threshold it compares against, on degenerate populations and at training sizes; the row
gather on its own; the library's own position sampler against N(0, 1).

What is compared, and how:
  * every decision, src_index / kind, the row order, every gathered parameter and Adam-moment tensor and every raw scaling
    (split children included): BIT FOR BIT against the float32 restatement on the same device, which issues the
    reference's own torch operations;
  * the new positions against the fp64 restatement: |gpu - fp64| <= C_XYZ * 2^-24 * (|x| + sum_j (|R_ij| + 1) |e_j s_j|),
    x the parent's position, R its rotation, s = exp(raw scaling), e the standard-normal sample.  C_XYZ = 16 counts the
    roundings: s = expf(raw) (<= 2 ulp, 4 * 2^-24 relative), e * s and R_ij * (e s) (one each), the three additions into
    x (one each, relative to the running magnitude), and R's entries, which come out of a normalised quaternion with an
    ABSOLUTE error of <= ~11 * 2^-24 (the "+ 1" beside |R_ij|: an entry near zero is not relatively accurate) -- 11 * 2^-24
    on the largest term in all, rounded up to 16;
  * the children's raw scalings, besides the bits, against fp64 log(exp(raw) / 1.6):
    |gpu - fp64| <= 2^-24 * (C_S_ARG + C_S_LOG * |fp64|), C_S_ARG = 6 for the argument of the log (expf's 2 ulp = 4 * 2^-24
    relative, the product with 0.625f one more, one spare; a relative error of the argument is an absolute one of the log)
    and C_S_LOG = 3 for logf's own 1 ulp (<= 2 * 2^-24 relative) and one spare.

Each threshold case builds Gaussians exactly on the comparison and on its float neighbours, asserts that the construction
landed (evaluated with torch on the device, the way the reference evaluates it), and prints which side every one of them
fell on.  Scale and opacity thresholds are reached through exp / sigmoid of a raw float, whose consecutive values are a few
float steps apart, so there the THRESHOLD is moved instead (extent, percent_dense, min_opacity) to the realised value and to
its float neighbours.

The one test without the gpu mark holds the restatement itself against the reference's stored results
(tests/golden/densify_*.npz)."""
import math

import numpy as np
import pytest
import torch

import _densify_ref as ref
import _liveref
import test_gpu_densify as golden_case

GROUPS = ref.GROUPS
EPS = 2.0 ** -24
C_XYZ = 16
C_S_ARG, C_S_LOG = 6, 3
MAX_GRAD, MIN_OP, EXTENT = 2e-4, 0.05, 1.7
gpu = pytest.mark.gpu
FATE = {(): "pruned", (0,): "kept", (0, 1): "cloned", (2, 3): "split"}


# ---- float helpers ---------------------------------------------------------------------------------------------------
def consecutive(x, lo, hi, dev):
    """The float32 values lo..hi steps away from float32(x) (steps in the bit pattern), on dev."""
    b = int(np.float32(x).view(np.int32))
    return (torch.arange(b + lo, b + hi + 1, dtype=torch.int64).to(torch.int32)).view(torch.float32).to(dev)


def step(x, k):
    """float32(x) moved k steps in its bit pattern (x > 0: k > 0 is up)."""
    return float((np.float32(x).view(np.int32) + np.int32(k)).view(np.float32))


def scalar_for(target, factor):
    """A double d with float32(factor * d) == target: how a Python threshold reaches the float32 comparison."""
    d = float(target) / factor
    for _ in range(64):
        v = np.float32(factor * d)
        if v == np.float32(target):
            return d
        d = float(np.nextafter(d, math.inf if v < np.float32(target) else -math.inf))
    raise AssertionError(f"no double d with float32({factor} * d) == {target}")


def accum_for(x, d, dev):
    """A float32 accumulator a with a / d == x in float32 on the device (the quotient the kernel and torch both take)."""
    c = consecutive(x * d, -8, 8, dev)
    hit = (c / torch.full_like(c, d) == x).nonzero()
    assert len(hit), (x, d)
    return float(c[hit[0, 0]])


# ---- states ----------------------------------------------------------------------------------------------------------
SHAPES = {"xyz": (3,), "f_dc": (1, 3), "f_rest": (15, 3), "opacity": (1,), "scaling": (3,), "rotation": (4,)}


def state(P, dev, seed):
    """P Gaussians with statistics shaped like a training step's: denom a small integer (10 % zero, accum zero with it),
    accum and accum_abs denom times a heavy-tailed (log-normal) integer multiple of 2^-18 -- so the mean gradients take
    exact repeated values, as on a real step; 3 % of the Gaussians above the world-size prune, the rest around the
    clone / split boundary; opacities from 0.0003 to 0.9997."""
    g = torch.Generator(device=dev).manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device=dev)
    ru = lambda *s: torch.rand(*s, generator=g, device=dev)
    params = {k: rn(P, *s) for k, s in SHAPES.items()}
    params["opacity"] = params["opacity"] * 2.0
    big = ru(P) < 0.03
    params["scaling"] = torch.log(torch.where(big[:, None], 0.1 + 0.4 * ru(P, 3), 1e-3 + 0.03 * ru(P, 3)))
    den = torch.randint(1, 8, (P,), generator=g, device=dev).float()
    den[ru(P) < 0.1] = 0.0
    level = lambda median: torch.floor(median * torch.exp(1.2 * rn(P))).clamp(max=4095.0)
    return dict(params=params, m={k: rn(P, *s) * 1e-3 for k, s in SHAPES.items()},
                v={k: ru(P, *s) * 1e-6 for k, s in SHAPES.items()},
                acc=den * level(15) * 2.0 ** -18, acc_abs=den * level(30) * 2.0 ** -18, den=den, noise=rn(3, P, 3))


def append(st, n, seed=1, scale=None, opacity=3.0, acc=0.0, acc_abs=0.0, den=1.0):
    """st with n more Gaussians (returned with their indices): scale 2e-3 unless `scale` (the raw value of component
    i % 3, the others log(1e-3)), raw opacity `opacity`, the given statistics (scalars or per-row lists)."""
    dev = st["den"].device
    P = st["den"].shape[0]
    add = state(n, dev, seed)
    col = lambda v: torch.as_tensor(v, dtype=torch.float32, device=dev).expand(n).clone()
    raw = torch.full((n, 3), math.log(2e-3), device=dev)
    if scale is not None:
        raw = torch.full((n, 3), math.log(1e-3), device=dev)
        raw[torch.arange(n, device=dev), torch.arange(n, device=dev) % 3] = col(scale)
    add["params"]["scaling"] = raw
    add["params"]["opacity"] = col(opacity)[:, None]
    add["acc"], add["acc_abs"], add["den"] = col(acc), col(acc_abs), col(den)
    cat = lambda a, b: {k: torch.cat([a[k], b[k]]) for k in a}
    out = dict(params=cat(st["params"], add["params"]), m=cat(st["m"], add["m"]), v=cat(st["v"], add["v"]),
               noise=torch.cat([st["noise"], add["noise"]], 1))
    for k in ("acc", "acc_abs", "den"):
        out[k] = torch.cat([st[k], add[k]])
    return out, torch.arange(P, P + n, device=dev)


# ---- running and comparing -------------------------------------------------------------------------------------------
def run(st, max_grad=MAX_GRAD, min_opacity=MIN_OP, extent=EXTENT, max_screen=20, percent_dense=0.01):
    """gof_densify on st (with st's noise), checked against the restatement (check()); returns gof_densify's result."""
    import gof_densify
    args = (st["params"], st["m"], st["v"], st["acc"], st["acc_abs"], st["den"], max_grad, min_opacity, extent, max_screen)
    ours = gof_densify.densify_and_prune(*args, percent_dense=percent_dense, noise=st["noise"])
    check(ours, ref.densify_and_prune(*args, st["noise"], percent_dense=percent_dense, fp64=True), st)
    return ours


def check(ours, want, st):
    assert ours.counts == want["counts"], (ours.counts, want["counts"])
    assert torch.equal(ours.src_index.long(), want["src_index"]) and torch.equal(ours.kind, want["kind"])
    for k in GROUPS:
        if k != "xyz":
            assert torch.equal(ours.params[k], want["params"][k]), k
        assert torch.equal(ours.exp_avg[k], want["exp_avg"][k]), k
        assert torch.equal(ours.exp_avg_sq[k], want["exp_avg_sq"][k]), k
    new = ours.kind > 0
    assert torch.equal(ours.params["xyz"][~new], want["params"]["xyz"][~new])
    if bool(new.any()):
        src = ours.src_index.long()[new]
        es = st["noise"][ours.kind[new].long() - 1, src].double() * torch.exp(st["params"]["scaling"][src].double())
        R = ref.build_rotation(st["params"]["rotation"][src].double())
        scale = st["params"]["xyz"][src].double().abs() + ((R.abs() + 1.0) * es.abs()[:, None, :]).sum(2)
        err = (ours.params["xyz"][new].double() - want["xyz64"][new]).abs()
        assert bool((err <= C_XYZ * EPS * scale).all()), f"xyz: {float((err / (EPS * scale)).max())} x 2^-24 of the scale"
    child = ours.kind >= 2
    if bool(child.any()):
        s64 = want["scaling64"][child]
        err = (ours.params["scaling"][child].double() - s64).abs()
        assert bool((err <= EPS * (C_S_ARG + C_S_LOG * s64.abs())).all()), float((err / EPS).max())


def fates(out, idx):
    """The sorted kinds of the output rows of each source Gaussian in idx: () pruned, (0,) kept, (0, 1) cloned, (2, 3) split."""
    src = out.src_index.long()
    sel = torch.isin(src, idx)
    d = {i: () for i in idx.tolist()}
    for i, k in sorted(zip(src[sel].tolist(), out.kind[sel].tolist())):
        d[i] += (k,)
    return [d[i] for i in idx.tolist()]


def report(name, values, thr, got):
    for x, f in zip(values, got):
        side = "on" if x == thr else ("below" if x < thr else "above")
        print(f"[{name}] {x!r} {side} threshold {thr!r}: {FATE.get(f, f)}")


def selected(st, max_grad):
    """The reference's selection (either gradient at its threshold) of every Gaussian, and Q."""
    g, ga, Q = ref.grads_and_threshold(st["acc"], st["acc_abs"], st["den"], max_grad)
    return (g.reshape(-1) >= max_grad) | (ga.reshape(-1) >= Q), Q


# ======================================================================================================================
# 1. the restatement against the reference's stored results (no device)
# ======================================================================================================================
def golden_inputs(P):
    """test_gpu_densify.inputs(P, cuda) made on the CPU.  The parameters and moments there come out of one step of
    torch.optim.Adam on CUDA (the multi-tensor path); it is restated here in float64 with the float32 roundings it makes,
    the fused multiply-adds of its addcmul and addcdiv included, so that the CPU sees the device's bits."""
    _g, _p, _m, _v, stats, noise = golden_case.inputs(P, torch.device("cpu"))
    gen = torch.Generator().manual_seed(P)
    r = lambda *shape: torch.randn(*shape, generator=gen)
    raw = {"xyz": r(P, 3), "f_dc": r(P, 1, 3), "f_rest": r(P, 15, 3), "opacity": r(P, 1) * 2.0,
           "scaling": torch.log(torch.rand(P, 3, generator=gen) * 0.04 + 1e-3), "rotation": r(P, 4)}
    r(4, 4)                                                   # the appearance group's parameter
    grads = {k: torch.randn(raw[k].shape, generator=gen) for k in raw}
    f32 = lambda x: x.float().double()
    c = lambda x: f32(torch.tensor(x, dtype=torch.float64))
    params, m, v = {}, {}, {}
    for k in raw:
        gr, p = grads[k].double(), raw[k].double()
        m_ = f32(c(1 - 0.9) * gr)                                                  # lerp from 0
        v_ = f32(c(1 - 0.999) * f32(gr * gr))                                      # addcmul onto 0
        d = f32(f32(f32(v_.sqrt()) / c((1 - 0.999) ** 0.5)) + c(1e-15))
        params[k] = f32(c((1e-3 / (1 - 0.9)) * -1) * f32(m_ / d) + p).float()     # addcdiv, one rounding
        m[k], v[k] = m_.float(), v_.float()
    return params, m, v, stats, noise


@pytest.mark.parametrize("P,max_screen", golden_case.CASES)
def test_restatement_equals_stored_reference(P, max_screen):
    """The float32 restatement on the CPU against the reference's own methods run on the device (tests/golden/densify_*.npz):
    the row count and sample, every gathered tensor's digest exactly, the sampled positions and scalings within float
    rounding (the CPU's exp / log / division and the device's differ in the last bits: 2 * C_XYZ and 4 ulp)."""
    z = _liveref.load_npz(f"densify_{P}.npz")
    params, m, v, (acc, acc_abs, den), noise = golden_inputs(P)
    out = ref.densify_and_prune(params, m, v, acc, acc_abs, den, golden_case.MAX_GRAD, golden_case.MIN_OP, golden_case.EXTENT,
                                max_screen, noise)
    n = out["params"]["xyz"].shape[0]
    assert n == sum(out["counts"]) and np.array_equal(np.sort(np.random.default_rng(n).choice(n, min(n, 256), replace=False)), z["rows"])
    rows = torch.from_numpy(z["rows"])
    for k in GROUPS:
        if k not in ("xyz", "scaling"):
            assert _liveref.digest(out["params"][k]) == str(z[k]), k
        assert _liveref.digest(out["exp_avg"][k]) == str(z["exp_avg_" + k]), k
        assert _liveref.digest(out["exp_avg_sq"][k]) == str(z["exp_avg_sq_" + k]), k
    src, kind = out["src_index"][rows], out["kind"][rows].long()
    es = noise[(kind - 1).clamp(min=0), src].double() * torch.exp(params["scaling"][src].double()) * (kind > 0)[:, None]
    R = ref.build_rotation(params["rotation"][src].double())
    scale = params["xyz"][src].double().abs() + ((R.abs() + 1.0) * es.abs()[:, None, :]).sum(2)
    assert bool(((out["params"]["xyz"][rows].double() - torch.from_numpy(z["xyz"]).double()).abs() <= 2 * C_XYZ * EPS * scale).all())
    s = out["params"]["scaling"][rows].double()
    assert bool(((s - torch.from_numpy(z["scaling"]).double()).abs() <= 4 * EPS * 2 * s.abs()).all())


# ======================================================================================================================
# 2. thresholds
# ======================================================================================================================
@gpu
def test_grad_threshold():
    """accum / denom == max_grad (>=: selected), and the float neighbours, through denom 1 and through denom 9 (a rounded
    quotient; 9 * max_grad lies low enough in its binade that every float near max_grad is some a / 9)."""
    dev = torch.device("cuda")
    t = float(np.float32(MAX_GRAD))
    vals = [step(t, -1), t, step(t, 1)]
    acc = vals + [accum_for(x, 9.0, dev) for x in vals]
    st, idx = append(state(1000, dev, 11), 6, acc=acc, den=[1.0] * 3 + [9.0] * 3)
    assert (st["acc"] / st["den"])[idx].tolist() == vals * 2                     # landed
    assert float(selected(st, MAX_GRAD)[1]) > 0.0                               # grad_abs = 0 does not select them
    got = fates(run(st), idx)
    report("grad", vals * 2, t, got)
    assert got == [(0,), (0, 1), (0, 1)] * 2


@gpu
def test_grad_abs_quantile_threshold():
    """grad_abs == Q on a run of 200 equal values that holds the quantile's position, and the float neighbours of Q."""
    dev = torch.device("cuda")
    V = float(np.float32(6e-4))
    g = torch.Generator(device=dev).manual_seed(5)
    low = (1e-5 + 4.9e-4 * torch.rand(800, generator=g, device=dev)).tolist()
    acc_abs = low + [step(V, -1)] + [V] * 196 + [2 * V] * 4 + [step(V, 1)] + [1e-3, 2e-3]
    den = [1.0] * 997 + [2.0] * 4 + [1.0] * 3
    acc = [1e-3] * 10 + [0.0] * 994                                                # ratio = 10 / 1004
    st, idx = append(state(0, dev, 12), 1004, acc=acc, acc_abs=acc_abs, den=den)
    sel, Q = selected(st, MAX_GRAD)
    ga = (st["acc_abs"] / st["den"])
    assert float(Q) == V and int((ga == Q).sum()) == 200                         # landed on the run
    probe = idx[800:1002]
    got = fates(run(st), probe)
    vals = ga[probe].tolist()
    report("grad_abs", [vals[0], vals[1], vals[-1]], V, [got[0], got[1], got[-1]])
    assert got == [(0,)] + [(0, 1)] * 201


@gpu
@pytest.mark.parametrize("shift", [-1, 0, 1])
def test_clone_split_boundary(shift):
    """max exp(scaling) == percent_dense * extent (<=: clone, >: split) for seven consecutive raw scalings, with the threshold
    on the middle one's scale (shift 0) or one float below / above it; the max in each of the three components."""
    dev = torch.device("cuda")
    raws = consecutive(math.log(0.01 * EXTENT), -3, 3, dev)
    s = torch.exp(raws)
    thr = step(float(s[3]), shift)
    extent = scalar_for(thr, 0.01)
    assert float(np.float32(0.01 * extent)) == thr and bool((s[3] == 0.01 * extent) == (shift == 0))   # landed
    st, idx = append(state(1000, dev, 13), 7, scale=raws.tolist(), acc=1e-3)
    got = fates(run(st, extent=extent, max_screen=None), idx)
    report(f"dense{shift:+d}", s.tolist(), thr, got)
    assert got == [(0, 1) if x <= thr else (2, 3) for x in s.tolist()]


@gpu
@pytest.mark.parametrize("shift", [-1, 0, 1])
def test_min_opacity_boundary(shift):
    """sigmoid(opacity) == min_opacity (<: pruned) for seven consecutive raw opacities, the threshold on the middle one's
    opacity or one float below / above it; unselected, cloned and split Gaussians (the children inherit the opacity)."""
    dev = torch.device("cuda")
    raws = consecutive(math.log(0.05 / 0.95), -3, 3, dev)
    o = torch.sigmoid(raws)
    thr = step(float(o[3]), shift)
    assert bool((o[3] == thr) == (shift == 0)) and float(np.float32(thr)) == thr                  # landed
    st = state(1000, dev, 14)
    idx = []
    for scale, acc in ((math.log(2e-3), 0.0), (math.log(2e-3), 1e-3), (math.log(0.03), 1e-3)):
        st, i = append(st, 7, scale=[scale] * 7, opacity=raws.tolist(), acc=acc)
        idx.append(i)
    out = run(st, min_opacity=thr)
    for name, i, alive in (("kept", idx[0], (0,)), ("cloned", idx[1], (0, 1)), ("split", idx[2], (2, 3))):
        got = fates(out, i)
        report(f"opacity{shift:+d} {name}", o.tolist(), thr, got)
        assert got == [() if x < thr else alive for x in o.tolist()]


@gpu
@pytest.mark.parametrize("shift", [-1, 0, 1])
def test_world_size_prune_boundary(shift):
    """max exp(scaling) == 0.1 * extent (>: pruned, when max_screen_size is given) for seven consecutive raw scalings of
    unselected Gaussians, the threshold on the middle one's scale or one float below / above it; with max_screen_size
    None all are kept."""
    dev = torch.device("cuda")
    raws = consecutive(math.log(0.1 * EXTENT), -3, 3, dev)
    s = torch.exp(raws)
    thr = step(float(s[3]), shift)
    extent = scalar_for(thr, 0.1)
    assert float(np.float32(0.1 * extent)) == thr and bool((s[3] == 0.1 * extent) == (shift == 0))     # landed
    st, idx = append(state(1000, dev, 15), 7, scale=raws.tolist())
    got = fates(run(st, extent=extent), idx)
    report(f"world{shift:+d}", s.tolist(), thr, got)
    assert got == [(0,) if x <= thr else () for x in s.tolist()]
    assert fates(run(st, extent=extent, max_screen=None), idx) == [(0,)] * 7


def child_sweep(dev, n=1 << 20):
    """Raw scalings of 2^20 consecutive floats from log(1.6 * 0.1 * EXTENT) down, their scale s = exp(raw), the children's
    scale by s / 1.6f (the kernel's former rule) and as the reference reads it back, exp(log(s / 1.6)) in torch."""
    raws = consecutive(math.log(1.6 * 0.1 * EXTENT), 0, n - 1, dev)
    s = torch.exp(raws)
    return raws, s, (s.double() / float(np.float32(1.6))).float(), torch.exp(torch.log(s / 1.6))


@gpu
def test_split_child_prune():
    """A split child is pruned by world size on the scale the reference stores and reads back, exp(log(s / 1.6)), not on
    s / 1.6f.  Over the 2^20 raw scalings of child_sweep (children from 0.17 = 0.1 * 1.7 down to 0.15), observed on an H100:
    the two differ for 416 044.  Two causes: torch divides a CUDA tensor by a Python scalar as a product with the float
    reciprocal, so the stored child is log(s * 0.625f), and s * 0.625f != s / 1.6f for 152 514 of them; and
    expf(logf(c)) != c for 334 812.  With the threshold on the lower of the two values the rules fall on different sides;
    eight such cases spread over the sweep, each with the threshold exactly there (three of the eight are pruned by the reference)."""
    dev = torch.device("cuda")
    raws, s, old, back = child_sweep(dev)
    cand = (old != back).nonzero().flatten()
    recip = int(((s / 1.6) != old).sum())
    as_product = bool(torch.equal(s / 1.6, s * 0.625))
    trip = int((back != s / 1.6).sum())
    print(f"[child] {len(cand)} of {len(raws)} raw scalings: exp(log(s / 1.6)) != s / 1.6f; torch's s / 1.6 != s / 1.6f: "
          f"{recip} (torch's s / 1.6 == s * 0.625f everywhere: {as_product}); exp(log(c)) != c: {trip}")
    assert len(cand) > 0
    for j in cand[torch.linspace(0, len(cand) - 1, 8).long()].tolist():
        thr = min(float(old[j]), float(back[j]))
        extent = scalar_for(thr, 0.1)
        assert float(np.float32(0.1 * extent)) == thr and (float(old[j]) > thr) != (float(back[j]) > thr)   # landed
        st, idx = append(state(300, dev, 16), 1, scale=[float(raws[j])], acc=1e-3)
        got = fates(run(st, extent=extent), idx)
        print(f"[child] s {float(s[j])!r}: s / 1.6f = {float(old[j])!r}, read back {float(back[j])!r}, threshold {thr!r}: "
              f"{FATE.get(got[0], got[0])}")
        assert got == [(2, 3) if float(back[j]) <= thr else ()]


@gpu
def test_zero_denominator():
    """denom == 0 with accum == accum_abs == 0: NaN -> 0 in both gradients, not selected; with accum > 0: +inf, selected."""
    dev = torch.device("cuda")
    st, idx = append(state(1000, dev, 17), 2, acc=[0.0, 1e-4], den=0.0)
    got = fates(run(st), idx)
    print(f"[denom 0] accum 0: {FATE[got[0]]}, accum 1e-4: {FATE[got[1]]}")
    assert got == [(0,), (0, 1)]


# ======================================================================================================================
# 3. degenerate populations
# ======================================================================================================================
@gpu
def test_empty_population():
    out = run(state(0, torch.device("cuda"), 18))
    assert out.counts == (0, 0, 0, 0) and out.params["f_rest"].shape == (0, 15, 3)


@gpu
@pytest.mark.parametrize("big", [False, True])
@pytest.mark.parametrize("max_screen", [None, 20])
@pytest.mark.parametrize("opacity", [-4.0, 3.0])
@pytest.mark.parametrize("scale", [2e-3, 0.05, 0.3])
def test_single_gaussian(scale, opacity, max_screen, big):
    """P = 1: the quantile of one value is that value, so the Gaussian is always selected; clone, split and world-size
    prune sizes, pruned by opacity or not, with and without max_screen_size, and with a large or a zero gradient."""
    st, _ = append(state(0, torch.device("cuda"), 19), 1, scale=[math.log(scale)], opacity=opacity, acc=1e-3 if big else 0.0)
    out = run(st, max_screen=max_screen)
    pruned = opacity < 0 or (scale * 0.625 > 0.1 * EXTENT and max_screen)       # by opacity; split children by world size
    assert sum(out.counts) == (0 if pruned else 2) and out.counts[1] == (0 if pruned or scale > 0.01 * EXTENT else 1)


@gpu
def test_nearly_nothing_selected():
    """No gradient reaches max_grad: ratio = 0, and Q, the quantile at 1, is the largest grad_abs -- so the reference always
    selects its arg-max and nothing else; an empty selection does not exist."""
    st = state(3000, torch.device("cuda"), 20)
    st["acc_abs"][7], st["den"][7], st["params"]["opacity"][7], st["params"]["scaling"][7] = 1.0, 1.0, 3.0, math.log(2e-3)
    out = run(st, max_grad=1.0)
    assert out.counts[1] + out.counts[2] == 1 and int(out.src_index[out.kind > 0][0]) == 7


@gpu
def test_everything_selected():
    """max_grad = 0: ratio = 1, Q is the minimum, every Gaussian is cloned or split (or pruned)."""
    st = state(3000, torch.device("cuda"), 21)
    sel, Q = selected(st, 0.0)
    assert bool(sel.all()) and float(Q) == float((st["acc_abs"] / st["den"]).nan_to_num(0.0).min())
    out = run(st, max_grad=0.0, max_screen=None)
    assert out.counts[0] == out.counts[1] and out.counts[1] + out.counts[2] > 0


@gpu
def test_everything_pruned():
    """min_opacity = 1: every row pruned, N = 0: empty outputs of the right shapes, no launch."""
    out = run(state(3000, torch.device("cuda"), 22), min_opacity=1.0)
    assert out.counts == (0, 0, 0, 0)
    assert out.params["f_rest"].shape == (0, 15, 3) and out.exp_avg_sq["rotation"].shape == (0, 4)


@gpu
@pytest.mark.parametrize("scale,want", [(5e-3, "clone"), (0.05, "split")])
def test_only_clones_or_only_splits(scale, want):
    dev = torch.device("cuda")
    st = state(3000, dev, 23)
    st["params"]["scaling"] = math.log(scale) + 0.1 * (torch.arange(9000, device=dev) % 7 / 7.0).reshape(3000, 3)
    out = run(st, max_grad=0.0)
    assert (out.counts[1] > 0 and out.counts[2] == 0) if want == "clone" else (out.counts[:2] == (0, 0) and out.counts[2] > 0)


@gpu
@pytest.mark.parametrize("max_screen", [None, 0, 20])
def test_max_screen_size(max_screen):
    """None and 0 switch the world-size prune off (the reference's `if max_screen_size:`), 20 on."""
    st = state(5000, torch.device("cuda"), 24)
    out = run(st, max_screen=max_screen)
    big = torch.exp(st["params"]["scaling"]).max(1).values > 0.1 * EXTENT
    assert bool(big[out.src_index.long()[out.kind == 0]].any()) == (not max_screen)


@gpu
@pytest.mark.parametrize("P", [255, 256, 257, 2047, 2048, 2049])
def test_sizes_at_block_edges(P):
    """The decision grid's 256-thread blocks and the exclusive scan's 2048-value chunks, just below, at and above."""
    run(state(P, torch.device("cuda"), P))


# ======================================================================================================================
# 4. training sizes
# ======================================================================================================================
@gpu
def test_training_size():
    """P ~ 4 * 10^6 with a training step's statistics, and the threshold Gaussians of section 2 in it, every threshold
    exactly on a realised value at once: max_grad; Q on a data value of the step's own repeated gradients; percent_dense
    * extent through percent_dense; 0.1 * extent on a split child where s / 1.6f and exp(log(s / 1.6)) disagree, and
    on an original; min_opacity.  Everything compared as in section 2, and the counts."""
    dev = torch.device("cuda")
    _raws, s, old, back = child_sweep(dev, 1 << 16)
    hit = None
    for j in (old != back).nonzero().flatten().tolist():       # a disagreeing child whose threshold is also some exp(raw)
        thr = min(float(old[j]), float(back[j]))
        near = consecutive(math.log(thr), -64, 64, dev)
        w = (torch.exp(near) == thr).nonzero()
        if len(w):
            hit = (j, thr, near[w[0, 0]].item())
            break
    assert hit is not None
    j, thr_w, raw_w = hit
    extent = scalar_for(thr_w, 0.1)
    raws_d = consecutive(math.log(0.01 * extent), -2, 2, dev)
    thr_d = float(torch.exp(raws_d[2]))
    pd = scalar_for(thr_d, extent)
    raws_o = consecutive(math.log(0.05 / 0.95), -2, 2, dev)
    min_op = float(torch.sigmoid(raws_o[2]))
    t = float(np.float32(MAX_GRAD))
    st = state(4_000_000, dev, 25)
    st, i_g = append(st, 3, seed=2, acc=[step(t, -1), t, step(t, 1)])
    st, i_d = append(st, 5, seed=3, scale=raws_d.tolist(), acc=1e-3)
    st, i_w = append(st, 3, seed=4, scale=consecutive(raw_w, -1, 1, dev).tolist())
    st, i_c = append(st, 1, seed=5, scale=[float(_raws[j])], acc=1e-3)
    st, i_o = append(st, 5, seed=6, opacity=raws_o.tolist())
    Q = float(selected(st, MAX_GRAD)[1])
    st, i_q = append(st, 3, seed=7, acc_abs=[step(Q, -1), Q, step(Q, 1)])
    ga = st["acc_abs"] / st["den"]
    assert float(selected(st, MAX_GRAD)[1]) == Q and int((ga == Q).sum()) > 100                     # Q on a data value
    assert float(np.float32(0.1 * extent)) == thr_w and float(np.float32(pd * extent)) == thr_d       # landed
    assert float(torch.exp(torch.tensor(raw_w, device=dev))) == thr_w and float(torch.sigmoid(raws_o[2])) == min_op
    assert (float(old[j]) > thr_w) != (float(back[j]) > thr_w)
    import gof_densify
    args = (st["params"], st["m"], st["v"], st["acc"], st["acc_abs"], st["den"], MAX_GRAD, min_op, extent, 20)
    ours = gof_densify.densify_and_prune(*args, percent_dense=pd, noise=st["noise"])
    want = ref.densify_and_prune(*args, st["noise"], percent_dense=pd, fp64=True)
    check(ours, want, st)
    print(f"[training size] P = {st['den'].shape[0]}, counts {ours.counts}")
    got = {k: fates(ours, i) for k, i in (("g", i_g), ("d", i_d), ("w", i_w), ("c", i_c), ("o", i_o), ("q", i_q))}
    report("4M grad", [step(t, -1), t, step(t, 1)], t, got["g"])
    report("4M grad_abs", [step(Q, -1), Q, step(Q, 1)], Q, got["q"])
    report("4M dense", torch.exp(raws_d).tolist(), thr_d, got["d"])
    report("4M world", torch.exp(consecutive(raw_w, -1, 1, dev)).tolist(), thr_w, got["w"])
    report("4M child (read back)", [float(back[j])], thr_w, got["c"])
    report("4M opacity", torch.sigmoid(raws_o).tolist(), min_op, got["o"])
    assert got["g"] == [(0,), (0, 1), (0, 1)] and got["q"] == [(0,), (0, 1), (0, 1)]
    assert got["d"] == [(0, 1) if x <= thr_d else (2, 3) for x in torch.exp(raws_d).tolist()]
    assert got["w"] == [(0,) if x <= thr_w else () for x in torch.exp(consecutive(raw_w, -1, 1, dev)).tolist()]
    assert got["c"] == [(2, 3) if float(back[j]) <= thr_w else ()]
    assert got["o"] == [() if x < min_op else (0,) for x in torch.sigmoid(raws_o).tolist()]


# ======================================================================================================================
# 5. the row gather on its own
# ======================================================================================================================
def gather(src, idx, kind, n_out, zero_new):
    import gof_densify
    from diff_gaussian_rasterization import _C
    row = int(src[0].numel())
    dst = torch.full((n_out,) + tuple(src.shape[1:]), float("nan"), device=src.device)
    _C._check(gof_densify._lib.gof_gather_rows_f32(src.data_ptr(), row, idx.data_ptr(), kind.data_ptr(), n_out, zero_new,
                                                   dst.data_ptr(), _C._stream()))
    return dst


@gpu
@pytest.mark.parametrize("zero_new", [0, 1])
@pytest.mark.parametrize("shape", [(1,), (3,), (4,), (15, 3)])
def test_gather_rows(shape, zero_new):
    """dst[o] = src[idx[o]], zero where zero_new and kind[o] != 0, for every kind, n_out = 1001 (not a multiple of 256)."""
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(sum(shape) + 10 * zero_new)
    src = torch.randn((777,) + shape, generator=g, device=dev)
    idx = torch.randint(0, 777, (1001,), generator=g, device=dev, dtype=torch.int32)
    kind = (torch.arange(1001, device=dev) % 4).to(torch.uint8)
    want = src[idx.long()].clone()
    if zero_new:
        want[kind != 0] = 0.0
    assert torch.equal(gather(src, idx, kind, 1001, zero_new), want)


@gpu
def test_gather_rows_large():
    """3.4 * 10^6 rows of 45 floats (1.53 * 10^8 floats) from 10^6."""
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(3)
    src = torch.randn((1_000_000, 15, 3), generator=g, device=dev)
    n = 3_400_000
    idx = torch.randint(0, 1_000_000, (n,), generator=g, device=dev, dtype=torch.int32)
    kind = torch.randint(0, 4, (n,), generator=g, device=dev, dtype=torch.int32).to(torch.uint8)
    want = src[idx.long()]
    want[kind != 0] = 0.0
    assert want.numel() >= 1.5e8 and torch.equal(gather(src, idx, kind, n, 1), want)


# ======================================================================================================================
# 6. the library's own sampler (noise=None)
# ======================================================================================================================
def sampler_state(P, dev):
    """P selected Gaussians (max_grad 0 selects all), opaque, at the origin; the first half clone-sized, the second
    split-sized; random rotations."""
    g = torch.Generator(device=dev).manual_seed(26)
    params = {k: torch.randn((P,) + s, generator=g, device=dev) for k, s in SHAPES.items()}
    params["xyz"].zero_()
    params["opacity"].fill_(3.0)
    u = torch.rand(P, 3, generator=g, device=dev)
    params["scaling"] = torch.log(torch.where(torch.arange(P, device=dev)[:, None] < P // 2, 1e-3 + 0.014 * u, 0.02 + 0.1 * u))
    zeros = {k: torch.zeros_like(t) for k, t in params.items()}
    return params, zeros, torch.rand(P, generator=g, device=dev), torch.rand(P, generator=g, device=dev), torch.ones(P, device=dev)


@gpu
def test_philox_sampler():
    """Whitened offsets e = diag(1/s) R^T (x_new - x) in fp64, >= 10^6 per kind: finite; per component mean and variance
    within 6 sigma of N(0, 1); Kolmogorov-Smirnov statistic below its 10^-6 critical value (sqrt(ln(2 / 10^-6) / 2n));
    correlations between the components and between the two children within 6 sigma of zero.  The same seed gives the
    same bits, another seed other rows, and Gaussian i's samples do not depend on P (the key is (seed, i, kind))."""
    import gof_densify
    dev = torch.device("cuda")
    P = 2_000_000
    params, zeros, acc, acc_abs, den = sampler_state(P, dev)
    run_ = lambda p, seed, n=P: gof_densify.densify_and_prune({k: t[:n] for k, t in p.items()}, {k: t[:n] for k, t in zeros.items()},
                                                              {k: t[:n] for k, t in zeros.items()}, acc[:n], acc_abs[:n], den[:n], 0.0,
                                                              MIN_OP, EXTENT, None, seed=seed)
    out = run_(params, 7)
    assert out.counts == (P // 2, P // 2, P // 2, P // 2)
    src = out.src_index.long()
    e_of = {}
    for k in (1, 2, 3):
        rows = out.kind == k
        i = src[rows]
        R = ref.build_rotation(params["rotation"][i].double())
        d = out.params["xyz"][rows].double() - params["xyz"][i].double()
        e = torch.bmm(R.transpose(1, 2), d[:, :, None])[:, :, 0] / torch.exp(params["scaling"][i].double())
        n = e.shape[0]
        assert n >= 1_000_000 and bool(torch.isfinite(e).all())
        mean, var = e.mean(0), e.var(0)
        assert bool((mean.abs() <= 6 / math.sqrt(n)).all()), (k, mean)
        assert bool(((var - 1).abs() <= 6 * math.sqrt(2 / n)).all()), (k, var)
        ks_crit = math.sqrt(math.log(2 / 1e-6) / 2) / math.sqrt(n)
        for c in range(3):
            x, _ = torch.sort(e[:, c])
            F = torch.special.ndtr(x)
            i = torch.arange(0, n + 1, device=dev, dtype=torch.float64) / n
            ks = float(torch.maximum(i[1:] - F, F - i[:-1]).max())
            assert ks < ks_crit, (k, c, ks, ks_crit)
        cor = torch.corrcoef(e.T)
        assert float((cor - torch.eye(3, device=dev, dtype=torch.float64)).abs().max()) <= 6 / math.sqrt(n), (k, cor)
        e_of[k] = e
        print(f"[philox] kind {k}: n {n}, mean {mean.tolist()}, var {var.tolist()}")
    for c in range(3):
        r = float(torch.corrcoef(torch.stack([e_of[2][:, c], e_of[3][:, c]]))[0, 1])
        assert abs(r) <= 6 / math.sqrt(P // 2), (c, r)
    again, other = run_(params, 7), run_(params, 8)
    assert torch.equal(again.params["xyz"], out.params["xyz"])
    new = out.kind > 0
    assert torch.equal(other.src_index, out.src_index)
    assert torch.equal(other.params["xyz"][~new], out.params["xyz"][~new])
    assert bool((other.params["xyz"][new] != out.params["xyz"][new]).any(1).all())
    small = run_(params, 7, P // 2 + 1000)                                       # the first P / 2 + 1000 Gaussians alone
    for k in (1, 2, 3):
        a = out.params["xyz"][(out.kind == k) & (src < P // 2 + 1000)]
        b = small.params["xyz"][small.kind == k]
        assert torch.equal(a, b), k
