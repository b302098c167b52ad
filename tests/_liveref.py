"""Stored comparisons with the unmodified reference extension (test infrastructure, not product code).

tests/golden/make_golden_live_ref.py runs the reference (oracle/_ref, built by oracle/build_ref.sh) once on a GPU for every
case below and stores what test_gpu_live_ref.py and test_integrate.py compare against in tests/golden/live_*.npz:
  * buffers the implementation reproduces bit for bit (radii, tile lists, per-Gaussian records of the visible Gaussians,
    the median-depth channels) as SHA-256 digests of their bytes;
  * every float image channel and every gradient as a CountSketch of the whole array (sketch()), from which the full-array
    relative L2 difference is estimated to ~2 %, next to the reference's run-to-run noise measured against a second backward
    of its own (the tolerance scale of the atomically accumulated gradients);
  * besides, the image channels and the gradients other than the AMPLIFIED ones as a seeded sample of pixels / rows, checked
    element by element in max-norm relative to the reference's full-array maximum.
The inputs are regenerated from the seeds in CASES, so the files hold reference outputs only."""
import hashlib
import os

import numpy as np
import torch

import _util
import gof_synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAMES = ["dmeans2D", "dcolors", "dopacity", "dmeans3D", "dcov3D", "dsh", "dscales", "drot", "dv2g"]
AMPLIFIED = ("dmeans3D", "dscales", "drot")      # view2gaussian chain rule: summation noise x ~1/scale^2 (DESIGN.md 2.2)
PIX, ROWS, SKETCH = 1024, 128, 512

CASES = {
    "C2_v3": dict(scene="C2", view=3, gseed=9),
    "C3_v1": dict(scene="C3", view=1, gseed=9),
    "sh4_deg1": dict(scene=dict(P=30_011, width=400, height=300, seed=21), view=11, gseed=3, M=4, deg=1),
    "sh9_deg2": dict(scene=dict(P=30_011, width=400, height=300, seed=21), view=11, gseed=3, M=9, deg=2),
    "sh16_deg2": dict(scene=dict(P=30_011, width=400, height=300, seed=21), view=11, gseed=3, M=16, deg=2),
    "v2g_precomp": dict(scene=dict(P=50_000, width=640, height=400, seed=31), view=5, gseed=4, v2g=True),
    "cov3d": dict(scene=dict(P=40_000, width=512, height=384, seed=41), view=9, gseed=6, cov=True, ks=0.1),
    "cov3d_v2g": dict(scene=dict(P=40_000, width=512, height=384, seed=41), view=9, gseed=6, cov=True, ks=0.1, v2g=True),
}
BUFFERS = ("tiles_touched", "point_list", "ranges", "n_contrib")


def digest(t):
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def cov3d_from(scales, rotations, mod):
    """computeCov3D (forward.cu:129-163) in torch float64 -> float32: Sigma = (S R)^T (S R), upper triangle."""
    s = scales.double() * mod
    r, x, y, z = rotations.double().unbind(1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).view(-1, 3, 3)
    M = R * s[:, None, :]
    S = M @ M.transpose(1, 2)
    return torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1).float().contiguous()


def inputs(name, dev):
    """(forward argument tuple, P, W, H, upstream gradient) of case `name`.  Precomputed view2gaussian records come from this
    package's own forward (bit-identical to the reference's, checked by the cases without them)."""
    from diff_gaussian_rasterization import _C as ours
    c = CASES[name]
    cam, gs = gof_synth.make_scene(c["scene"], view=c["view"])
    P, W, H = gs["means3D"].shape[0], cam.image_width, cam.image_height
    if "M" in c:
        gs = dict(gs)
        gs["shs"] = gs["shs"][:, :c["M"], :].contiguous()
    ks = c.get("ks", 0.0)
    fa = list(_util.fwd_args(cam, gs, dev, kernel_size=ks, sh_degree=c.get("deg")))
    if c.get("v2g"):
        R0, _c0, rad0, geo0, bin0, im0 = ours.rasterize_gaussians(*fa)
        v2g = ours.export_state(P, W, H, R0, geo0, bin0, im0, rad0)["view2gaussian"].contiguous()
        if c.get("cov"):
            # the inflated covariance below makes a few more Gaussians visible: give those a well-formed record (an isotropic
            # sigma = 0.01 Gaussian 5 units in front of the camera) rather than zeros (A = B = 0 -> NaN depth in both)
            filler = torch.tensor([1e4, 0.0, 0.0, 1e4, 0.0, 1e4, 0.0, 0.0, -5e4, 25e4], device=dev)
            v2g = torch.where((rad0 > 0)[:, None], v2g, filler[None, :]).contiguous()
        fa[8] = v2g
    if c.get("cov"):
        fa[7] = cov3d_from(gs["scales"], gs["rotations"], 1.7).to(dev)       # 1.7x the covariance scale/rotation would give
    grad = torch.randn(9, H, W, generator=torch.Generator().manual_seed(c["gseed"])).to(dev)
    return tuple(fa), P, W, H, grad


def _sample(n, k, seed):
    k = min(n, k)
    return np.sort(np.random.default_rng(seed).choice(n, k, replace=False)) if n else np.zeros(0, np.int64)


def _rows(vis_idx):
    return vis_idx[_sample(len(vis_idx), ROWS, 5)]


def sketch(t):
    """CountSketch of a tensor into SKETCH buckets: element i goes to bucket h(i) mod SKETCH with sign bit 63 of h(i), h a
    splitmix64-style hash of i.  The squared norm of the sketch of a difference estimates the difference's squared L2 norm
    without bias, with a relative standard deviation of at most sqrt(2 / SKETCH)."""
    x = t.detach().double().flatten().cpu().numpy()
    h = np.arange(x.size, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    h ^= h >> np.uint64(29)
    h *= np.uint64(0xBF58476D1CE4E5B9)
    h ^= h >> np.uint64(32)
    sign = 1.0 - 2.0 * (h >> np.uint64(63)).astype(np.float64)
    return np.bincount((h % np.uint64(SKETCH)).astype(np.int64), weights=sign * x, minlength=SKETCH)


def _l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def _maxrel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)) if b.numel() else 0.0


def record(ref, name, dev):
    """Runs the reference on case `name` and returns the dictionary stored as live_<name>.npz."""
    fa, P, W, H, grad = inputs(name, dev)
    R, color, radii, geom, binning, img = ref.rasterize_gaussians(*fa)
    sg, si, sb = _util.carve_ref_geom(geom, P), _util.carve_ref_image(img, W, H), _util.carve_ref_binning(binning, R)
    vis = radii > 0
    out = {"R": np.int64(R), "radii": digest(radii), "tiles_touched": digest(sg["tiles_touched"]),
           "point_list": digest(sb["point_list"]), "ranges": digest(si["ranges"]), "n_contrib": digest(si["n_contrib"]),
           "color6": digest(color[6]), "color7": digest(color[7])}
    for f in ("depths", "means2D", "conic_opacity", "view2gaussian"):
        out["bits_" + f] = digest(sg[f][vis])
    vis_idx = vis.nonzero().flatten().cpu().numpy()
    rgb_rows = _rows(vis_idx)
    out["rgb_rows"], out["rgb"] = rgb_rows, sg["rgb"][torch.from_numpy(rgb_rows).to(dev)].cpu().numpy()
    out["rgb_absmax"] = float(sg["rgb"][vis].abs().max())
    px = _sample(W * H, PIX, 11)
    flat = color.reshape(9, -1)
    out["pix"], out["color"], out["color_absmax"] = px, flat[:, torch.from_numpy(px).to(dev)].cpu().numpy(), flat.abs().amax(1).cpu().numpy()
    out["color_sketch"] = np.stack([sketch(flat[ch]) for ch in range(9)]).astype(np.float32)
    out["color_norm"] = flat.double().norm(dim=1).cpu().numpy()
    g1 = ref.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, grad))
    g2 = ref.rasterize_gaussians_backward(*_util.bwd_args(fa, radii, geom, R, binning, img, grad))
    for n, a, b in zip(NAMES, g1, g2):
        if n in AMPLIFIED:
            out[n + "_sketch"], out[n + "_norm"], out[n + "_noise"] = sketch(a).astype(np.float32), float(a.double().norm()), _l2(b, a)
            continue
        rows = _rows(vis_idx)
        out[n + "_rows"], out[n] = rows, a[torch.from_numpy(rows).to(dev)].cpu().numpy()
        out[n + "_absmax"] = float(a.abs().max()) if a.numel() else 0.0
        out[n + "_noise"] = _maxrel(b, a)
        out[n + "_sketch"], out[n + "_norm"], out[n + "_noise_l2"] = sketch(a).astype(np.float32), float(a.double().norm()), _l2(b, a)
    return _compact(out)


def _compact(rec):
    """Row indices are stored as int32 (load() widens them again)."""
    return {k: (v.astype(np.int32) if isinstance(v, np.ndarray) and v.dtype == np.int64 else v) for k, v in rec.items()}


def load_npz(fname):
    z = np.load(os.path.join(GOLDEN, fname))
    return {k: (z[k].astype(np.int64) if z[k].dtype == np.int32 else z[k]) for k in z.files}


def load(name):
    return load_npz(f"live_{name}.npz")


def check_forward(gold, ours_out, P, W, H, buffers=(), vis_fields=(), depth_channels=False, rgb=False):
    """The forward of this package against the stored reference forward: R and radii always, the named integer buffers and
    per-Gaussian records of the visible Gaussians bit for bit, the median-depth channels 6 and 7 bit for bit if asked, every
    colour channel within 2e-6 (distortion, channel 8: 2e-5): on the sampled pixels relative to the reference's maximum, over
    the whole channel in relative L2."""
    from diff_gaussian_rasterization import _C as ours
    R, color, radii, geom, binning, img = ours_out
    dev = color.device
    assert R == int(gold["R"])
    assert digest(radii) == str(gold["radii"])
    so = ours.export_state(P, W, H, R, geom, binning, img, radii)
    for f in buffers:
        assert digest(so[f]) == str(gold[f]), f
    vis = radii > 0
    for f in vis_fields:
        assert digest(so[f][vis]) == str(gold["bits_" + f]), f
    if depth_channels:
        assert digest(color[6]) == str(gold["color6"]) and digest(color[7]) == str(gold["color7"])
    if rgb:
        got = so["rgb"][torch.from_numpy(gold["rgb_rows"]).to(dev)].cpu().double().numpy()
        assert np.abs(got - gold["rgb"]).max(initial=0.0) / max(float(gold["rgb_absmax"]), 1e-30) < 5e-7
    got = color.reshape(9, -1)[:, torch.from_numpy(gold["pix"]).to(dev)].cpu().double().numpy()
    flat = color.reshape(9, -1)
    for ch in range(9):
        tol = 2e-5 if ch == 8 else 2e-6
        err = np.abs(got[ch] - gold["color"][ch]).max() / max(float(gold["color_absmax"][ch]), 1e-30)
        assert err < tol, f"channel {ch}: {err}"
        l2 = float(np.linalg.norm(sketch(flat[ch]) - gold["color_sketch"][ch])) / max(float(gold["color_norm"][ch]), 1e-30)
        assert l2 < tol, f"channel {ch}: relative L2 {l2}"


def check_grads(gold, grads, amp_floor=1e-4, amp_factor=3.0):
    """Gradients against the stored reference gradients.  Every gradient: the full-array relative L2 difference (estimated from
    the sketches) within max(1e-4, 6 x the reference's own relative L2 noise), for AMPLIFIED max(amp_floor, amp_factor x it).
    The others also element by element: max-norm over the sampled rows relative to the reference's full-array maximum, within
    max(1e-4, 6 x its own max-norm noise)."""
    for n, a in zip(NAMES, grads):
        noise = float(gold[n + "_noise"])
        if n in AMPLIFIED:
            err = float(np.linalg.norm(sketch(a) - gold[n + "_sketch"])) / max(float(gold[n + "_norm"]), 1e-30)
            assert err <= max(amp_floor, amp_factor * noise), f"{n}: ours-vs-ref L2 {err}, ref-vs-ref {noise}"
        else:
            l2 = float(np.linalg.norm(sketch(a) - gold[n + "_sketch"])) / max(float(gold[n + "_norm"]), 1e-30) if a.numel() else 0.0
            noise_l2 = float(gold[n + "_noise_l2"])
            assert l2 <= max(1e-4, 6.0 * noise_l2), f"{n}: ours-vs-ref L2 {l2}, ref-vs-ref {noise_l2}"
            got = a[torch.from_numpy(gold[n + "_rows"]).to(a.device)].cpu().double()
            want = torch.from_numpy(gold[n]).double()
            err = float((got - want).abs().max()) / max(float(gold[n + "_absmax"]), 1e-30) if want.numel() else 0.0
            assert err <= max(1e-4, 6.0 * noise), f"{n}: ours-vs-ref {err}, ref-vs-ref {noise}"


# ---- the opacity-field query at 1080p -----------------------------------------------------------------------------
def integrate_inputs(dev):
    cam, gs = gof_synth.make_scene(dict(P=150_000, width=1920, height=1080, seed=6), view=20)
    g = torch.Generator().manual_seed(4)
    n = 400_000
    pts = torch.cat([gs["means3D"][torch.randint(0, 150_000, (n // 2,), generator=g)] + 0.01 * torch.randn(n // 2, 3, generator=g),
                     (torch.rand(n // 2, 3, generator=g) * 2 - 1) * 1.6]).contiguous().to(dev)
    fa = _util.fwd_args(cam, gs, dev)
    return (fa[0], pts) + tuple(fa[1:])


def record_integrate(ref, dev):
    R, color, alpha, col_int, radii, *_ = ref.integrate_gaussians_to_points(*integrate_inputs(dev))
    px, pt = _sample(color[0].numel(), 4096, 13), _sample(alpha.shape[0], 4096, 17)
    out = {"R": np.int64(R), "radii": digest(radii), "color_integrated": digest(col_int), "pix": px, "pts": pt,
           "tmax": color[6].flatten()[torch.from_numpy(px).to(dev)].cpu().numpy(), "tmax_absmax": float(color[6].abs().max()),
           "alpha": alpha[torch.from_numpy(pt).to(dev)].cpu().numpy()}
    out.update({f"color{ch}": digest(color[ch]) for ch in (0, 1, 2, 3, 4, 5, 7, 8)})
    return _compact(out)
