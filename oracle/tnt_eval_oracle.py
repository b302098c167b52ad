"""CPU oracle of the Tanks and Temples evaluation (DESIGN section 4.7): a float64 numpy / scipy restatement of the specification
of the Open3D 0.10 operations that eval_tnt/run.py calls, with the operation order of csrc/tnt_eval.cu wherever the
specification fixes one.  No Open3D.

    read_log(path)                          -> [k, 4, 4] (trajectory_io.read_trajectory)
    read_crop_volume(path)                  -> volume dict (read_selection_polygon_volume)
    transform(points, T)                    -> (((m00*x + m01*y) + m02*z) + m03) / w per row
    crop(points, volume, T=None)            -> (kept points in input order, their indices)
    voxel_down_sample(points, voxel)        -> per voxel mean, ascending (x, y, z) voxel order
    uniform_down_sample(points, max_points) -> every k-th point, k = round(n / max_points), when n > max_points
    nn(ref, query, r2)                      -> (index or -1, d2): the nearest ref point with d2 < r2, lowest index on ties
    registration_icp(src, tgt, threshold)   -> dict(transformation, iterations, fitness, inlier_rmse)
    ransac_alignment(src, tgt, seed)        -> 4x4 (registration_ransac_based_on_correspondence, seeded)
    evaluate(...)                           -> dict like gof_tnt_eval.evaluate
"""
import json
import math

import numpy as np
from scipy.spatial import cKDTree

SCENES_TAU = {"Barn": 0.01, "Caterpillar": 0.005, "Church": 0.025, "Courthouse": 0.025, "Ignatius": 0.003, "Meetingroom": 0.01,
              "Truck": 0.005}
MAX_POINT_NUMBER = 4e6
INT_MAX = 2147483647
# ICPConvergenceCriteria(1e-6, max_itr) as Open3D 0.10 binds it: (relative_fitness, relative_rmse, max_iteration = default 30)
ICP_CRITERIA = {"relative_fitness": 1e-6, "relative_rmse": 20.0, "max_iteration": 30}


def read_log(path):
    mats = []
    with open(path) as fh:
        lines = [ln for ln in fh.read().splitlines()]
    k = 0
    while k < len(lines) and lines[k].strip():
        mats.append(np.array([[float(x) for x in lines[k + 1 + r].split()] for r in range(4)], np.float64))
        k += 5
    return np.asarray(mats, np.float64).reshape(-1, 4, 4)


def crop_volume(axis, axis_min, axis_max, polygon):
    """volume dict from the JSON fields: axis 0-2, bounds, the polygon's [m, 3] vertices"""
    P = np.asarray(polygon, np.float64).reshape(-1, 3)
    u, v = [a for a in range(3) if a != axis]
    return {"axis": int(axis), "axis_min": float(axis_min), "axis_max": float(axis_max), "polygon_uv": P[:, [u, v]].copy()}


def read_crop_volume(path):
    with open(path) as fh:
        d = json.load(fh)
    axis = {"x": 0, "y": 1, "z": 2}[str(d["orthogonal_axis"]).lower()]
    return crop_volume(axis, d["axis_min"], d["axis_max"], d["bounding_polygon"])


def transform(points, T):
    P = np.asarray(points, np.float64).reshape(-1, 3)
    T = np.asarray(T, np.float64)
    x, y, z = P[:, 0], P[:, 1], P[:, 2]
    r = [((T[k, 0] * x + T[k, 1] * y) + T[k, 2] * z) + T[k, 3] for k in range(4)]
    return np.stack([r[0] / r[3], r[1] / r[3], r[2] / r[3]], 1)


def crop(points, volume, T=None):
    P = np.asarray(points, np.float64).reshape(-1, 3)
    if T is not None:
        P = transform(P, T)
    w = volume["axis"]
    u, v = [a for a in range(3) if a != w]
    pw, pu, pv = P[:, w], P[:, u], P[:, v]
    inside = ~((pw < volume["axis_min"]) | (pw > volume["axis_max"]))
    poly = volume["polygon_uv"]
    m = poly.shape[0]
    below = np.zeros(P.shape[0], np.int64)
    with np.errstate(divide="ignore", invalid="ignore"):
        for i in range(m):
            (au, av), (bu, bv) = poly[i], poly[(i + 1) % m]
            cross = ((av < pv) & (bv >= pv)) | ((bv < pv) & (av >= pv))
            node = au + ((pv - av) / (bv - av)) * (bu - au)
            below += cross & (node < pu)
    idx = np.nonzero(inside & (below % 2 == 1))[0]
    return P[idx], idx


def voxel_down_sample(points, voxel):
    P = np.asarray(points, np.float64).reshape(-1, 3)
    if P.shape[0] == 0:
        return P.copy()
    lo = P.min(0) - voxel * 0.5
    hi = P.max(0) + voxel * 0.5
    if voxel * INT_MAX < (hi - lo).max():
        raise ValueError("voxel_size is too small")
    key = np.floor((P - lo) / voxel).astype(np.int64)
    order = np.lexsort((key[:, 2], key[:, 1], key[:, 0]))          # stable: members stay in input order
    k = key[order]
    head = np.ones(len(order), bool)
    head[1:] = (k[1:] != k[:-1]).any(1)
    group = np.cumsum(head) - 1
    first = order[head]
    acc = P[first].copy()
    rest = ~head
    np.add.at(acc, group[rest], P[order[rest]])                     # sequential, in sorted (= input) order per voxel
    count = np.bincount(group).astype(np.float64)
    return acc / count[:, None]


def uniform_down_sample(points, max_points=MAX_POINT_NUMBER):
    P = np.asarray(points, np.float64).reshape(-1, 3)
    n = P.shape[0]
    if n > max_points:
        return P[::int(round(n / float(max_points)))]
    return P


def _sq(d):
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def nn(ref, query, r2=np.inf, k=16):
    """(idx [m] int64, d2 [m]): over every candidate at the exact minimum the lowest index; -1 / inf unless d2 < r2."""
    R = np.asarray(ref, np.float64).reshape(-1, 3)
    Q = np.asarray(query, np.float64).reshape(-1, 3)
    m = Q.shape[0]
    if m == 0:
        return np.zeros(0, np.int64), np.zeros(0)
    tree = cKDTree(R)
    k = min(k, R.shape[0])
    _, cand = tree.query(Q, k=k, workers=-1)
    cand = cand.reshape(m, k)
    d2 = _sq(R[cand] - Q[:, None, :])
    best = d2.min(1)
    idx = np.where(d2 == best[:, None], cand, np.iinfo(np.int64).max).min(1)
    if k < R.shape[0]:
        # the k-th candidate ties the minimum (or the k-d tree's rounding could hide one): every point within reach
        redo = np.nonzero(d2[:, -1] <= best * (1 + 1e-9) + 1e-300)[0]
        for q in redo:
            c = np.asarray(tree.query_ball_point(Q[q], math.sqrt(best[q]) * (1 + 1e-9) + 1e-300), np.int64)
            dd = _sq(R[c] - Q[q])
            best[q] = dd.min()
            idx[q] = c[dd == best[q]].min()
    ok = best < r2
    return np.where(ok, idx, -1), np.where(ok, best, np.inf)


def icp_r2(threshold):
    """the squared radius as Open3D 0.10 hands it to FLANN: (threshold * threshold) rounded to float32"""
    return float(np.float32(threshold * threshold))


def moments(src, tgt, idx, d2):
    """count, sum d2, means (fsum * (1 / count)), sum (t - mt)(s - ms)^T, sum |s - ms|^2 -- every sum exactly rounded"""
    sel = np.nonzero(idx >= 0)[0]
    n = sel.size
    if n == 0:
        return 0, 0.0, np.zeros(3), np.zeros(3), np.zeros((3, 3)), 0.0
    s, t = src[sel], tgt[idx[sel]]
    inv = 1.0 / n
    ms = np.array([math.fsum(s[:, a]) * inv for a in range(3)])
    mt = np.array([math.fsum(t[:, a]) * inv for a in range(3)])
    ds, dt = s - ms, t - mt
    cov = np.array([[math.fsum(dt[:, r] * ds[:, c]) for c in range(3)] for r in range(3)])
    var = math.fsum(_sq(ds))
    return n, math.fsum(d2[sel]), ms, mt, cov, var


def umeyama(n, ms, mt, cov, var):
    """Eigen::umeyama with scaling from the moments; the identity for an empty set"""
    T = np.eye(4)
    if n == 0:
        return T
    inv = 1.0 / n
    sigma = cov * inv
    U, sv, Vt = np.linalg.svd(sigma)
    S = np.ones(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2] = -1.0
    R = U @ np.diag(S) @ Vt
    with np.errstate(divide="ignore", invalid="ignore"):
        c = (1.0 / (var * inv)) * float(sv @ S)
    T[:3, 3] = mt - c * (R @ ms)
    T[:3, :3] = R * c
    return T


def registration_icp(src, tgt, threshold, max_iteration=30, relative_fitness=1e-6, relative_rmse=1e-6, trace=None):
    """Open3D 0.10 registration_icp with TransformationEstimationPointToPoint(True), from the identity.  trace (a list) gets
    (moving points, idx, d2) of every evaluation."""
    src = np.asarray(src, np.float64).reshape(-1, 3)
    tgt = np.asarray(tgt, np.float64).reshape(-1, 3)
    r2 = icp_r2(threshold)
    T = np.eye(4)
    moving = src.copy()

    def evaluate(pts):
        if tgt.shape[0] == 0 or pts.shape[0] == 0:
            idx, d2 = np.full(pts.shape[0], -1, np.int64), np.full(pts.shape[0], np.inf)
        else:
            idx, d2 = nn(tgt, pts, r2)
        if trace is not None:
            trace.append((pts.copy(), idx, d2))
        mom = moments(pts, tgt, idx, d2)
        n = mom[0]
        fitness = n / pts.shape[0] if pts.shape[0] else 0.0
        rmse = math.sqrt(mom[1] / n) if n else 0.0
        return mom, fitness, rmse

    mom, fitness, rmse = evaluate(moving)
    it = 0
    for it in range(1, max_iteration + 1):
        update = umeyama(*((mom[0],) + mom[2:]))
        T = update @ T
        moving = transform(moving, update)
        prev = (fitness, rmse)
        mom, fitness, rmse = evaluate(moving)
        if abs(prev[0] - fitness) < relative_fitness and abs(prev[1] - rmse) < relative_rmse:
            break
    return {"transformation": T, "iterations": it, "fitness": fitness, "inlier_rmse": rmse}


def ransac_draws(n, seed, iterations=100000, ransac_n=6):
    return np.random.default_rng(seed).integers(0, n, (iterations, ransac_n))


def _lsum(a, axis):
    """left-to-right sum along axis"""
    a = np.moveaxis(a, axis, 0)
    acc = a[0]
    for x in a[1:]:
        acc = acc + x
    return acc


def ransac_hypotheses(src, tgt, draws):
    """[H, 4, 4]: umeyama with scaling on each draw's pairs, every sum over the draw left to right"""
    s, t = src[draws], tgt[draws]
    n = draws.shape[1]
    inv = 1.0 / n
    ms = _lsum(s, 1) * inv
    mt = _lsum(t, 1) * inv
    ds, dt = s - ms[:, None], t - mt[:, None]
    cov = _lsum(dt[:, :, :, None] * ds[:, :, None, :], 1)
    var = _lsum(_sq(ds), 1)
    out = np.empty((draws.shape[0], 4, 4))
    for h in range(draws.shape[0]):
        with np.errstate(all="ignore"):
            try:
                out[h] = umeyama(n, ms[h], mt[h], cov[h], var[h])
            except np.linalg.LinAlgError:
                out[h] = np.nan
    return out


def ransac_alignment(src, tgt, seed=0, max_distance=0.2, ransac_n=6, iterations=100000, chunk=2048):
    """One hypothesis per draw, scored over every correspondence i <-> i (inlier iff d2 < max_distance^2, rmse from the inliers'
    d2 summed left to right); the best by fitness, then rmse, then draw; the identity unless some draw has an inlier."""
    src = np.asarray(src, np.float64).reshape(-1, 3)
    tgt = np.asarray(tgt, np.float64).reshape(-1, 3)
    N = src.shape[0]
    if N < ransac_n or ransac_n < 3:
        return np.eye(4)
    draws = ransac_draws(N, seed, iterations, ransac_n)
    best = (0.0, 0.0, np.eye(4))
    md2 = max_distance * max_distance
    for c0 in range(0, iterations, chunk):
        Ts = ransac_hypotheses(src, tgt, draws[c0:c0 + chunk])
        for h, T in enumerate(Ts):
            with np.errstate(all="ignore"):
                d2 = _sq(transform(src, T) - tgt)
            inl = d2 < md2
            good = int(inl.sum())
            if good == 0:
                continue
            fit = good / N
            rmse = math.sqrt(float(_lsum(np.where(inl, d2, 0.0), 0)) / good)
            if fit > best[0] or (fit == best[0] and rmse < best[1]):
                best = (fit, rmse, T)
    return best[2]


# ---- scoring (evaluation.py:173-215, verbatim on arrays) -------------------------------------------------------------------

def f1_histo(threshold, plot_stretch, distance1, distance2):
    if len(distance1) and len(distance2):
        recall = float(np.count_nonzero(distance2 < threshold)) / float(len(distance2))
        precision = float(np.count_nonzero(distance1 < threshold)) / float(len(distance1))
        fscore = 2 * recall * precision / (recall + precision)
        num = len(distance1)
        bins = np.arange(0, threshold * plot_stretch, threshold / 100)
        hist, edges_source = np.histogram(distance1, bins)
        cum_source = np.cumsum(hist).astype(float) / num
        num = len(distance2)
        bins = np.arange(0, threshold * plot_stretch, threshold / 100)
        hist, edges_target = np.histogram(distance2, bins)
        cum_target = np.cumsum(hist).astype(float) / num
    else:
        precision = recall = fscore = 0
        edges_source = cum_source = edges_target = cum_target = np.array([0])
    return precision, recall, fscore, edges_source, cum_source, edges_target, cum_target


def distances(s, t):
    """compute_point_cloud_distance: sqrt of the exact 1-NN d2; 0 per point when t is empty"""
    if s.shape[0] == 0:
        return np.zeros(0)
    if t.shape[0] == 0:
        return np.zeros(s.shape[0])
    return np.sqrt(nn(t, s)[1])


def reconstruction_cloud(vertices, faces):
    V = np.asarray(vertices, np.float64).reshape(-1, 3)
    F = np.asarray(faces, np.int64).reshape(-1, 3)
    c = ((V[F[:, 0]] + V[F[:, 1]]) + V[F[:, 2]]) / 3
    return np.concatenate([V, c], 0)


def evaluate(vertices, faces, gt, traj, colmap_traj, gt_trans, volume, dTau, seed=0, max_points=MAX_POINT_NUMBER):
    pcd = reconstruction_cloud(vertices, faces)
    gt = np.asarray(gt, np.float64).reshape(-1, 3)
    src_c = np.asarray(traj, np.float64)[:, :3, 3]
    tgt_c = transform(np.asarray(colmap_traj, np.float64)[:, :3, 3], gt_trans)
    T0 = ransac_alignment(src_c, tgt_c, seed)
    out = {"T_ransac": T0}
    init = T0
    for name, mode, voxel, thr in (("r2", "voxel", dTau, 80 * dTau), ("r3", "voxel", dTau / 2.0, 20 * dTau),
                                   ("r", "uniform", None, 2 * dTau)):
        s, _ = crop(pcd, volume, init)
        t, _ = crop(gt, volume)
        if mode == "voxel":
            s, t = voxel_down_sample(s, voxel), voxel_down_sample(t, voxel)
        else:
            s, t = uniform_down_sample(s, max_points), uniform_down_sample(t, max_points)
        reg = registration_icp(s, t, thr, **ICP_CRITERIA)
        init = reg["transformation"] @ init
        out[f"T_{name}"] = init
        out[f"iterations_{name}"] = reg["iterations"]
    s = voxel_down_sample(crop(pcd, volume, init)[0], dTau / 2.0)
    t = voxel_down_sample(crop(gt, volume)[0], dTau / 2.0)
    d1, d2 = distances(s, t), distances(t, s)
    p, r, f, es, cs, et, ct = f1_histo(dTau, 5, d1, d2)
    out.update(source_down=s, target_down=t, d1=d1, d2=d2, precision=p, recall=r, fscore=f, edges_source=es, cum_source=cs,
               edges_target=et, cum_target=ct)
    return out
