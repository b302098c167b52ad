"""numpy float32 restatement of csrc/sh_views.cu (the SH-gradient expansion of the view-parallel exchange) -- TEST
INFRASTRUCTURE ONLY.

Every operation of gof_sh_view_dir, gof_sh_grad_weights (csrc/gof_math.cuh) and k_sh_grad_from_views is an explicitly rounded
fp32 operation, and numpy's float32 add, subtract, multiply, divide and sqrt round the same way; the fused multiply-adds go
through field_grid_oracle.fma32.  So this is bit for bit what the kernel computes:

  dir_v = (mean - cam_v) / |mean - cam_v|           (differences, squares by fma, sqrt, three divisions)
  dL_dsh[g, k, c] = sum over v in view order of fl(w_k(dir_v) * rgb_v[c])   (each product rounded, then added; acc starts at +0)

with a view skipped for a Gaussian whose three rgb are all zero, the degree of view v taken as (int)header[3], and the
coefficients k < min(M, 16, (D_v + 1)^2) written (the others stay +0)."""
import numpy as np

from field_grid_oracle import fma32

f32 = np.float32
SLOT_HEADER = 64     # GOF_SH_SLOT_HEADER (include/gof_rasterizer.h)

C0 = f32(0.28209479177387814)
C1 = f32(0.4886025119029199)
C2 = tuple(f32(c) for c in (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396))
C3 = tuple(f32(c) for c in (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
                            1.445305721320277, -0.5900435899266435))


def sh_plane(P):
    """GOF_SH_PLANE(P): floats of one colour plane of a view record."""
    return (int(P) + 63) // 64 * 64


def view_dir(means, cam):
    """gof_sh_view_dir: the unit direction camera centre -> mean, [P,3] float32."""
    m = np.asarray(means, f32)
    cam = np.asarray(cam, f32)
    d = [m[:, i] - cam[i] for i in range(3)]
    with np.errstate(all="ignore"):
        ln = np.sqrt(fma32(d[2], d[2], fma32(d[1], d[1], d[0] * d[0])))
        return np.stack([d[i] / ln for i in range(3)], axis=1)


def grad_weights(D, dirs):
    """gof_sh_grad_weights: [P, (D+1)^2] float32 for directions [P,3]."""
    x, y, z = (np.asarray(dirs, f32)[:, i] for i in range(3))
    w = [np.full_like(x, C0)]
    with np.errstate(all="ignore"):
        if D > 0:
            w += [-C1 * y, C1 * z, -C1 * x]
        if D > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            xx_yy = xx - yy
            w += [C2[0] * xy, C2[1] * yz, C2[2] * (fma32(f32(2), zz, -xx) - yy), C2[3] * xz, C2[4] * xx_yy]
        if D > 2:
            f4 = fma32(f32(4), zz, -xx) - yy
            w += [(C3[0] * y) * fma32(f32(3), xx, -yy),
                  (C3[1] * xy) * z,
                  (C3[2] * y) * f4,
                  (C3[3] * z) * fma32(f32(-3), yy, fma32(f32(-3), xx, f32(2) * zz)),
                  (C3[4] * x) * f4,
                  (C3[5] * z) * xx_yy,
                  (C3[6] * x) * fma32(f32(-3), yy, xx)]
    return np.stack(w, axis=1).astype(f32)


def sh_grad_from_views(means, records, P, M):
    """dL_dsh [P,M,3] float32 from view records (each: 64-float header -- camera centre, degree -- then rgb planes [3][plane])."""
    plane = sh_plane(P)
    out = np.zeros((P, M, 3), f32)
    for rec in records:
        rec = np.asarray(rec, f32)
        D = int(rec[3])
        rgb = rec[SLOT_HEADER:SLOT_HEADER + 3 * plane].reshape(3, plane)[:, :P].T
        seen = np.any(rgb != 0, axis=1)
        if not seen.any():
            continue
        nk = min(M, 16, (D + 1) * (D + 1))
        if nk == 0:
            continue
        w = grad_weights(D, view_dir(np.asarray(means, f32)[seen], rec[:3]))
        # ordinary float32 ops: one rounding for the product, one for the sum
        out[seen, :nk, :] = out[seen, :nk, :] + w[:, :nk, None] * rgb[seen][:, None, :]
    return out
