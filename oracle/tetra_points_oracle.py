"""numpy restatement of GaussianModel.get_tetra_points (scene/gaussian_model.py:433-463) and get_frustum_mask (:31-72) for the
tests (DESIGN §4.8).

The parts the reference computes with elementwise torch ops -- the quaternion norm, q, R, 3 * scales and their max -- are
reproduced in float32, one rounding per operation, so they are bit-exact.  The two matrix products the reference leaves to
cuBLAS (the box corners and the view transform) have no specified rounding order; they are computed in float64 from the
float32 inputs, with a bound on how far any float32 evaluation can be from them:

  a dot product of n terms plus nothing else, in any order, fused or not, is within gamma_n * sum|terms| of the exact value,
  gamma_n = n u / (1 - n u), u = 2^-24.

A corner is sum_j R_ij v_j + xyz_i: gamma_4 * (sum_j |R_ij v_j| + |xyz_i|) per evaluation.  A frustum comparison is decided
when its float64 margin exceeds the bound of the float32 quantity compared (depth, u or v), widened by how far the point itself
may lie from the one evaluated (`pos_err`, per coordinate).  The bounds are first order; SLACK doubles them to cover the rest.
"""
import numpy as np

U32 = 2.0 ** -24
SLACK = 2.0
# box corners of trimesh.creation.box() after `vertices *= 2`, as rows of signs (sx, sy, sz), sz fastest
BOX_SIGNS = np.array([[sx, sy, sz] for sx in (-1.0, 1.0) for sy in (-1.0, 1.0) for sz in (-1.0, 1.0)], np.float32)


def gamma(n):
    return n * U32 / (1.0 - n * U32)


def frame(rotation, scales):
    """float32, bit-exact: (R [P,3,3], s3 [P,3], point_scale [P]) of build_rotation(rotation) and scales * 3."""
    r = np.asarray(rotation, np.float32)
    s = np.asarray(scales, np.float32)
    with np.errstate(all="ignore"):
        norm = np.sqrt(((r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1]) + r[:, 2] * r[:, 2]) + r[:, 3] * r[:, 3])
        q = r / norm[:, None]
        w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
        one, two = np.float32(1), np.float32(2)
        R = np.stack([one - two * (y * y + z * z), two * (x * y - w * z), two * (x * z + w * y),
                      two * (x * y + w * z), one - two * (x * x + z * z), two * (y * z - w * x),
                      two * (x * z - w * y), two * (y * z + w * x), one - two * (x * x + y * y)], 1).reshape(-1, 3, 3)
        s3 = s * np.float32(3)
        ps = np.maximum(np.maximum(s3[:, 0], s3[:, 1]), s3[:, 2])   # np.maximum propagates NaN, as torch.max does
    return R.astype(np.float32), s3.astype(np.float32), ps.astype(np.float32)


def tetra_points(xyz, scales, rotation):
    """Unmasked points in the reference's order (corner k of g at 8g + k, centres at 8P + g), float64 [9P,3]; their bound
    per coordinate for ONE float32 evaluation [9P,3] (0 for the centres, which are copies); point scales float32 [9P]."""
    xyz32 = np.asarray(xyz, np.float32)
    R, s3, ps = frame(rotation, scales)
    P = xyz32.shape[0]
    R64, xyz64 = R.astype(np.float64), xyz32.astype(np.float64)
    v = BOX_SIGNS.astype(np.float64)[None, :, :] * s3.astype(np.float64)[:, None, :]          # [P,8,3], exact
    with np.errstate(all="ignore"):
        terms = R64[:, None, :, :] * v[:, :, None, :]                                          # [P,8,i,j]
        corners = terms.sum(-1) + xyz64[:, None, :]
        mag = np.abs(terms).sum(-1) + np.abs(xyz64)[:, None, :]
    err = gamma(4) * mag * (1.0 + 1e-12)
    pts = np.concatenate([corners.reshape(-1, 3), xyz64])
    bnd = np.concatenate([err.reshape(-1, 3), np.zeros((P, 3))])
    scale = np.concatenate([np.repeat(ps, 8), ps])
    return pts, bnd, scale


def pack_views(views):
    """[n,20] float32: world_view_transform (row-major), focal_x, focal_y, width, height of each view."""
    rows = []
    for v in views:
        wvt = np.asarray(v.world_view_transform.detach().cpu() if hasattr(v.world_view_transform, "detach") else v.world_view_transform,
                         np.float32).reshape(16)
        rows.append(np.concatenate([wvt, np.array([v.focal_x, v.focal_y, v.image_width, v.image_height], np.float32)]))
    return np.stack(rows)


def frustum_decision(points, views, near=0.02, far=1e6, pos_err=None):
    """(mask, decided) [N] bool: mask = the float64 evaluation of get_frustum_mask at `points`, decided = every float32
    evaluation of the reference's arithmetic at any point within `pos_err` of `points` gives the same answer."""
    p = np.asarray(points, np.float64)
    N = p.shape[0]
    e = np.zeros((N, 3)) if pos_err is None else np.asarray(pos_err, np.float64)
    vt = np.asarray(views, np.float32)
    W, H = float(vt[0, 18]), float(vt[0, 19])
    near32, far32 = float(np.float32(near)), float(np.float32(far))
    finite = np.isfinite(p).all(1)
    p = np.where(finite[:, None], p, 0.0)
    sure_in = np.zeros(N, bool)
    all_out = np.ones(N, bool)
    mask = np.zeros(N, bool)
    big = 1e37
    for row in vt.astype(np.float64):
        M = row[:16].reshape(4, 4)                       # M[c, b]: view coordinate b = sum_c M[c, b] h_c
        fx, fy = row[16], row[17]
        vp = p @ M[:3, :3] + M[3, :3]
        vmag = np.abs(p) @ np.abs(M[:3, :3]) + np.abs(M[3, :3])
        ev = SLACK * gamma(4) * vmag + e @ np.abs(M[:3, :3])              # [N,3] bound on a float32 view coordinate
        x, y, z = vp[:, 0], vp[:, 1], vp[:, 2]
        ex, ey, ez = ev[:, 0], ev[:, 1], ev[:, 2]
        with np.errstate(all="ignore"):
            un, vn = fx * x + (W / 2) * z, fy * y + (H / 2) * z
            eun = fx * ex + (W / 2) * ez + SLACK * gamma(3) * (np.abs(fx * x) + (W / 2) * np.abs(z) + fx * ex + (W / 2) * ez)
            evn = fy * ey + (H / 2) * ez + SLACK * gamma(3) * (np.abs(fy * y) + (H / 2) * np.abs(z) + fy * ey + (H / 2) * ez)
            u, v = un / z, vn / z
            den = np.abs(z) - ez
            ok = den > 0
            eu = np.where(ok, (eun + np.abs(u) * ez) / np.where(ok, den, 1.0), np.inf)
            ev_ = np.where(ok, (evn + np.abs(v) * ez) / np.where(ok, den, 1.0), np.inf)
            eu = eu + SLACK * U32 * (np.abs(u) + eu)
            ev_ = ev_ + SLACK * U32 * (np.abs(v) + ev_)
        # each comparison as (float64 value, its float32 bound)
        cmps = [(z - near32, ez), (far32 - z, ez), (u, eu), ((W - 1) - u, eu), (v, ev_), ((H - 1) - v, ev_)]
        with np.errstate(invalid="ignore"):
            truth = np.ones(N, bool)
            surely_true = np.ones(N, bool)
            surely_false = np.zeros(N, bool)
            for m, b in cmps:
                m = np.where(np.isfinite(m), m, np.nan)
                truth &= m >= 0
                surely_true &= m > b
                surely_false |= -m > b
        overflow = (vmag > big).any(1)
        truth &= finite & ~overflow
        surely_true &= finite & ~overflow
        surely_false |= ~finite
        mask |= truth
        sure_in |= surely_true
        all_out &= surely_false
    return mask, sure_in | all_out
