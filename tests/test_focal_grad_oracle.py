"""CPU: the float64 ray-gradient oracle (tests/focal_oracle/focal_oracle.c) against a complex-step derivative (the C ABI's checks
are in test_backward_abi.py).

The oracle's per-pixel dL/drx, dL/dry (DESIGN.md 4.10) is checked against an independent float64 restatement of one pixel's
compositing, differentiated by the complex step Im L(rx + ih) / h, which has no cancellation.  The restatement keeps the pixel's
contributor list fixed (the oracle forward's blend decisions) and follows the backward's conventions: the 0.99 alpha clamp and
the power <= 0 clamp subtract a real constant (the backward differentiates opacity * G through both), the distortion weights
T alpha and the pixel's final A and D are constants, and channel 7 is ignored.  Branches (the clamps, and through the fixed
list the 1/255 and near-plane gates) are taken on the real part."""
import cmath

import numpy as np
import pytest

import _focal_oracle as fo
import gof_oracle
import gof_synth

ALPHA_MAX = float(np.float32(0.99))
H_STEP = 1e-30


def _scene(seed, view, P=160, W=64, H=48, bg=(0.2, 0.5, 0.8)):
    """A small scene with a non-zero background, a few nearly opaque Gaussians (their alpha reaches the 0.99 clamp near their
    centres) and one wide Gaussian 0.22 in front of the camera, whose t crosses the 0.2 near plane inside the image."""
    cam, gs = gof_synth.make_scene(dict(P=P, width=W, height=H, seed=seed, sigma_px=5.0), view=view)
    op = gs["opacities"].clone()
    op[: P // 8] = 0.9995
    gs["opacities"] = op
    C = cam.camera_center.double()
    fwd = -C / C.norm()
    m, s = gs["means3D"].clone(), gs["scales"].clone()
    m[P - 1] = (C + 0.22 * fwd).float()
    s[P - 1] = 0.06
    gs["means3D"], gs["scales"] = m, s
    sc = gof_oracle.Scene(W, H, cam.tanfovx, cam.tanfovy, cam.world_view_transform, cam.full_proj_transform, cam.camera_center,
                          gs["means3D"], gs["opacities"], scales=gs["scales"], rotations=gs["rotations"], shs=gs["shs"],
                          sh_degree=gs["sh_degree"], bg=bg)
    return sc


def _pixel_loss(rx, ry, pairs, dpix, bg, fA, fD, median):
    """The float64 (complex) restatement of one pixel's loss; `pairs` = [(list index, v[10], opacity, colour[3])] front to back."""
    T = 1.0
    C = [0j, 0j, 0j]
    N = [0j, 0j, 0j]
    dist, tmed = 0j, 0j
    for c, v, op, col in pairs:
        n0 = v[0] * rx + v[1] * ry + v[2]
        n1 = v[1] * rx + v[3] * ry + v[4]
        n2 = v[2] * rx + v[4] * ry + v[5]
        AA = n0 * rx + n1 * ry + n2
        BB = 2.0 * (v[6] * rx + v[7] * ry + v[8])
        t = -BB / (2.0 * AA)
        power = -0.5 * ((-BB / AA) * (BB / 4.0) + v[9])
        if power.real > 0.0:
            power -= power.real
        a = op * cmath.exp(power)
        if a.real > ALPHA_MAX:
            a -= a.real - ALPHA_MAX
        w = T * a
        ln = cmath.sqrt(n0 * n0 + n1 * n1 + n2 * n2 + 1e-7)
        for ch in range(3):
            C[ch] += w * col[ch]
        for ch, nk in enumerate((n0, n1, n2)):
            N[ch] += w * (-nk / ln)
        m = (100.0 * t - 20.0) / (99.8 * t)
        dist += w.real * (fA * m * m - 2.0 * fD * m)
        if c == median:
            tmed = t
        T = T * (1.0 - a)
    L = sum(dpix[ch] * (C[ch] + T * bg[ch]) for ch in range(3)) + sum(dpix[3 + ch] * N[ch] for ch in range(3))
    return L + dpix[6] * tmed + dpix[8] * dist


def _complex_step(sc, st, dL):
    """[2,H,W] complex-step dL/drx, dL/dry of every pixel, and how often the clamp and the near plane were met."""
    W, H = sc.W, sc.H
    rxs, rys = fo.pixel_rays(W, H, sc.tan_fovx, sc.tan_fovy)
    gx = (W + 15) // 16
    out = np.zeros((2, H, W))
    v2g, co, rgb, bg = st["view2gaussian"].astype(np.float64), st["conic_opacity"].astype(np.float64), st["rgb"].astype(np.float64), \
        sc.arr["background"].astype(np.float64)
    seen = dict(clamped=0, near_rejected=0, near_blended=0)
    straddler = sc.P - 1
    for py in range(H):
        for px in range(W):
            r0, r1 = st["ranges"][(py // 16) * gx + px // 16]
            bits = st["blended"][py, px]
            pairs = []
            for c in range(int(r1 - r0)):
                gid = int(st["point_list"][r0 + c])
                blended = (bits[c >> 5] >> (c & 31)) & 1
                if gid == straddler and c < st["n_contrib"][0, py, px]:
                    seen["near_blended" if blended else "near_rejected"] += 1
                if blended:
                    pairs.append((c, v2g[gid], co[gid, 3], rgb[gid]))
            rx, ry = float(rxs[px]), float(rys[py])
            dpix = [float(dL[k, py, px]) for k in range(9)]
            fA = 1.0 - float(st["accum_alpha"][0, py, px])
            fD = float(st["accum_alpha"][1, py, px])
            median = int(st["n_contrib"][1, py, px]) - 1 if st["n_contrib"][1, py, px] != 0xFFFFFFFF else -2
            for c, v, op, _col in pairs:
                n = (v[0] * rx + v[1] * ry + v[2], v[1] * rx + v[3] * ry + v[4], v[2] * rx + v[4] * ry + v[5])
                AA = n[0] * rx + n[1] * ry + n[2]
                BB = 2.0 * (v[6] * rx + v[7] * ry + v[8])
                pw = min(-0.5 * ((-BB / AA) * (BB / 4.0) + v[9]), 0.0)
                seen["clamped"] += op * np.exp(pw) > ALPHA_MAX
            out[0, py, px] = _pixel_loss(complex(rx, H_STEP), ry, pairs, dpix, bg, fA, fD, median).imag / H_STEP
            out[1, py, px] = _pixel_loss(rx, complex(ry, H_STEP), pairs, dpix, bg, fA, fD, median).imag / H_STEP
    return out, seen


@pytest.mark.parametrize("seed,view", [(3, 5), (11, 21), (29, 40)])
def test_oracle_matches_the_complex_step(seed, view):
    sc = _scene(seed, view)
    _out, _radii, st = gof_oracle.forward(sc, checked=True)
    dL = np.random.default_rng(seed).standard_normal((9, sc.H, sc.W)).astype(np.float32)
    d = fo.rays(sc.W, sc.H, sc.tan_fovx, sc.tan_fovy, st, sc.arr["background"], dL, float_geometry=False)
    cs, seen = _complex_step(sc, st, dL)
    assert seen["clamped"] > 0 and seen["near_rejected"] > 0 and seen["near_blended"] > 0, seen
    err = np.abs(d["drays"] - cs)
    assert np.abs(cs).max() > 0
    assert (err <= 1e-9 * d["mag"] + 1e-300).all(), float((err / np.maximum(d["mag"], 1e-300)).max())
    # the float-geometry mode differs only by the float rounding of n, AA and BB
    f = fo.rays(sc.W, sc.H, sc.tan_fovx, sc.tan_fovy, st, sc.arr["background"], dL, float_geometry=True)
    assert np.allclose(f["drays"], d["drays"], rtol=0, atol=float(1e-3 * d["mag"].max()))

