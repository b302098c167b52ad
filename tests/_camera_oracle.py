"""The camera gradient of the backward (DESIGN.md 4.9) in float64 (test infrastructure).

The view-matrix part differentiates view2gaussian written as matrices -- Sigma = G^T diag(si) G, B = G^T diag(si) t2,
C = t2^T diag(si) t2 with G the rotation rows of G2V = W2V G2W, t its translation, t2 = -G t and si = 1 / (s^2 + 1e-7) --
instead of restating the kernel's chain rule step by step.  The campos part is minus the SH-direction part of dL_dmean3D,
taken from the CPU oracle (oracle/gof_oracle.c) called with dL_dview2gaussian = 0.

Layouts: vm is the 16 floats of the viewmatrix tensor, vm[4k+i] the coefficient of W2V[i][k]; the per-Gaussian terms are
[P,15] = dL_dvm[4k+i] (k < 4, i < 3) at 3k+i, then dL_dcampos."""
import numpy as np

import gof_oracle

SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
         1.445305721320277, -0.5900435899266435)


def rotation(q):
    """[P,4] (r,x,y,z) -> Rm [P,3,3] with Rm[:,k,c] the rotation entry that multiplies vm[4k+i] in G2V[c][i] (the glm
    column-major constructor of backward.cu, not re-normalised)."""
    q = np.asarray(q, np.float64)
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = np.empty((q.shape[0], 3, 3))
    R[:, 0, 0] = 1 - 2 * (y * y + z * z); R[:, 0, 1] = 2 * (x * y - r * z); R[:, 0, 2] = 2 * (x * z + r * y)
    R[:, 1, 0] = 2 * (x * y + r * z); R[:, 1, 1] = 1 - 2 * (x * x + z * z); R[:, 1, 2] = 2 * (y * z - r * x)
    R[:, 2, 0] = 2 * (x * z - r * y); R[:, 2, 1] = 2 * (y * z + r * x); R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def _g2v(vm, Rm, means):
    W = np.asarray(vm, np.float64).reshape(4, 4)            # W[k, i] = vm[4k+i]
    G = np.einsum("pkc,ki->pci", Rm, W[:3, :3])             # G[p, c, i] = G2V[c][i]
    t = np.asarray(means, np.float64) @ W[:3, :3] + W[3, :3]
    return G, t


def _si(scales):
    s = np.asarray(scales, np.float64)
    return 1.0 / (s * s + 1e-7)


def view2gaussian(vm, means, scales, rotations):
    """[P,10] view2gaussian records (Sigma upper triangle, B, C) in float64."""
    G, t = _g2v(vm, rotation(rotations), means)
    si = _si(scales)
    t2 = -np.einsum("pci,pi->pc", G, t)
    S = np.einsum("pc,pci,pcj->pij", si, G, G)
    B = np.einsum("pc,pci->pi", si * t2, G)
    C = (si * t2 * t2).sum(axis=1)
    return np.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2], B[:, 0], B[:, 1], B[:, 2], C], axis=1)


def vm_terms(vm, means, scales, rotations, dL_dv2g):
    """[P,12] per-Gaussian dL_dvm[4k+i] (k < 4, i < 3) at 3k+i for the given dL_dview2gaussian [P,10]."""
    Rm = rotation(rotations)
    G, t = _g2v(vm, Rm, means)
    si = _si(scales)
    dv = np.asarray(dL_dv2g, np.float64)
    D = np.empty((dv.shape[0], 3, 3))
    D[:, 0, 0], D[:, 1, 1], D[:, 2, 2] = dv[:, 0], dv[:, 3], dv[:, 5]
    D[:, 0, 1] = D[:, 1, 0] = 0.5 * dv[:, 1]
    D[:, 0, 2] = D[:, 2, 0] = 0.5 * dv[:, 2]
    D[:, 1, 2] = D[:, 2, 1] = 0.5 * dv[:, 4]
    b, dC = dv[:, 6:9], dv[:, 9]
    Gt = np.einsum("pci,pi->pc", G, t)
    Gb = np.einsum("pci,pi->pc", G, b)
    dG = (2.0 * si[:, :, None] * np.einsum("pci,pij->pcj", G, D)
          - si[:, :, None] * (Gb[:, :, None] * t[:, None, :] + Gt[:, :, None] * b[:, None, :])
          + 2.0 * (dC[:, None] * si * Gt)[:, :, None] * t[:, None, :])
    dt = np.einsum("pc,pci->pi", -si * Gb + 2.0 * dC[:, None] * si * Gt, G)
    h = np.asarray(means, np.float64)
    out = np.empty((dv.shape[0], 12))
    for k in range(3):
        out[:, 3 * k:3 * k + 3] = np.einsum("pci,pc->pi", dG, Rm[:, k, :]) + dt * h[:, k:k + 1]
    out[:, 9:12] = dt
    return out


def terms(sc, radii, clamped, dL_dcolor, dL_dv2g):
    """[P,15] per-Gaussian camera terms of oracle scene `sc` (gof_oracle.Scene); zero rows for Gaussians with radii <= 0."""
    P = sc.P
    out = np.zeros((P, 15))
    vis = np.asarray(radii) > 0
    a = sc.arr
    if a["v2g_precomp"] is None and a["scales"] is not None and a["rotations"] is not None and vis.any():
        out[vis, :12] = vm_terms(a["viewmatrix"], a["means3D"][vis], a["scales"][vis], a["rotations"][vis],
                                 np.asarray(dL_dv2g)[vis])
    if a["shs"] is not None:
        sh_part = gof_oracle.preprocess_backward(sc, radii, clamped, dL_dcolor, np.zeros((P, 10), np.float32))["dL_dmean3D"]
        out[:, 12:] = -sh_part.astype(np.float64)
    return out


def assemble(t):
    """Summed terms [15] -> (dL_dviewmatrix [16], dL_dcampos [3]), float64."""
    vm = np.zeros(16)
    for k in range(4):
        vm[4 * k:4 * k + 3] = t[3 * k:3 * k + 3]
    return vm, np.asarray(t[12:15], np.float64)


def sh_rgb(means, campos, shs, D):
    """[P,3] unclamped SH colour (computeColorFromSH before the clamp) in float64."""
    d = np.asarray(means, np.float64) - np.asarray(campos, np.float64).reshape(1, 3)
    d = d / np.linalg.norm(d, axis=1, keepdims=True)
    x, y, z = d[:, 0:1], d[:, 1:2], d[:, 2:3]
    sh = np.asarray(shs, np.float64)
    S = lambda k: sh[:, k, :]   # noqa: E731
    r = SH_C0 * S(0)
    if D > 0:
        r = r - SH_C1 * y * S(1) + SH_C1 * z * S(2) - SH_C1 * x * S(3)
        if D > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            r = (r + SH_C2[0] * xy * S(4) + SH_C2[1] * yz * S(5) + SH_C2[2] * (2 * zz - xx - yy) * S(6) + SH_C2[3] * xz * S(7)
                 + SH_C2[4] * (xx - yy) * S(8))
            if D > 2:
                r = (r + SH_C3[0] * y * (3 * xx - yy) * S(9) + SH_C3[1] * xy * z * S(10) + SH_C3[2] * y * (4 * zz - xx - yy) * S(11)
                     + SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * S(12) + SH_C3[4] * x * (4 * zz - xx - yy) * S(13)
                     + SH_C3[5] * z * (xx - yy) * S(14) + SH_C3[6] * x * (xx - 3 * yy) * S(15))
    return r + 0.5
