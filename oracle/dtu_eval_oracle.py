"""CPU oracle of the DTU mesh evaluation (DESIGN section 4.6): numpy / scipy restatement of dtu_eval/eval.py's steps with the
exact operation order of csrc/dtu_eval.cu, so that every array compares bit for bit.

    sample_mesh(vertices, faces, r)           -> [V + S, 3]
    ordered_downsample(points, perm, r)       -> kept [n] bool (over positions of the order)
    nn_sqdist(ref, query)                     -> [m] smallest ((dx*dx + dy*dy) + dz*dz)
    evaluate(data, stl, obs_mask, bb, res, plane, mode, faces, ...) -> dict like gof_dtu_eval.evaluate
"""
import warnings

import numpy as np
from scipy.spatial import cKDTree


def _norm(v):
    return np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])


def face_params(vertices, faces, r):
    """Per face (v1, v2, p0, n1, n2, ok) with numpy's norm and cross (eval.py:54-65)."""
    V = np.asarray(vertices, np.float64)
    F = np.asarray(faces, np.int64).reshape(-1, 3)
    p0, p1, p2 = V[F[:, 0]], V[F[:, 1]], V[F[:, 2]]
    v1, v2 = p1 - p0, p2 - p0
    l1, l2 = _norm(v1), _norm(v2)
    c = np.stack([v1[:, 1] * v2[:, 2] - v1[:, 2] * v2[:, 1], v1[:, 2] * v2[:, 0] - v1[:, 0] * v2[:, 2],
                  v1[:, 0] * v2[:, 1] - v1[:, 1] * v2[:, 0]], 1)
    area2 = _norm(c)
    ok = area2 > 0
    with np.errstate(divide="ignore", invalid="ignore"):
        thr = r * np.sqrt(l1 * l2 / area2)
        n1, n2 = np.floor(l1 / thr), np.floor(l2 / thr)
    return v1, v2, p0, n1, n2, ok


def sample_mesh(vertices, faces, r):
    V = np.asarray(vertices, np.float64).reshape(-1, 3)
    F = np.asarray(faces, np.int64).reshape(-1, 3)
    if F.shape[0] == 0:
        return V.copy()
    v1, v2, p0, n1, n2, ok = face_params(V, F, r)
    idx = np.nonzero(ok)[0]
    n1, n2 = n1[idx], n2[idx]
    rows = (n1 + 1).astype(np.int64)
    face_of_row = np.repeat(np.arange(idx.size), rows)
    i = (np.arange(face_of_row.size) - np.repeat(np.cumsum(rows) - rows, rows)).astype(np.float64)
    d1 = np.where(1e-7 > n1, 1e-7, n1)
    d2 = np.where(1e-7 > n2, 1e-7, n2)
    c0_row = (i + 0.5) / d1[face_of_row]
    # candidate columns: all j <= n2 of every row, then the predicate of eval.py:17
    cols = (n2[face_of_row] + 1).astype(np.int64)
    row_of = np.repeat(np.arange(face_of_row.size), cols)
    j = (np.arange(row_of.size) - np.repeat(np.cumsum(cols) - cols, cols)).astype(np.float64)
    f = face_of_row[row_of]
    c0 = c0_row[row_of]
    c1 = (j + 0.5) / d2[f]
    keep = (c0 + c1) < 1
    f, c0, c1 = idx[f[keep]], c0[keep][:, None], c1[keep][:, None]
    q = (v1[f] * c0 + v2[f] * c1) + p0[f]
    return np.concatenate([V, q], 0)


def radius_pairs(points, r):
    """All pairs (a < b) with ((dx*dx + dy*dy) + dz*dz) <= r*r, exact formula over cKDTree candidates."""
    P = np.asarray(points, np.float64)
    if P.shape[0] < 2:
        return np.zeros((0, 2), np.int64)
    cand = cKDTree(P).query_pairs(r * (1 + 1e-9) + 1e-300, output_type="ndarray")
    if cand.size == 0:
        return np.zeros((0, 2), np.int64)
    d = P[cand[:, 0]] - P[cand[:, 1]]
    d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    cand = np.sort(cand[d2 <= r * r], axis=1)
    return cand


def ordered_downsample(points, perm, r):
    """kept[k] for position k of the order (points[perm[k]]): the sequential loop of eval.py:89-93."""
    Q = np.asarray(points, np.float64)[np.asarray(perm)]
    n = Q.shape[0]
    pairs = radius_pairs(Q, r)
    order = np.argsort(pairs[:, 0], kind="stable")
    a, b = pairs[order, 0], pairs[order, 1]
    start = np.searchsorted(a, np.arange(n + 1))
    mask = np.ones(n, dtype=np.bool_)
    for cur in range(n):
        if mask[cur] and start[cur] < start[cur + 1]:
            mask[b[start[cur]:start[cur + 1]]] = False
    return mask


def nn_sqdist(ref, query, k=8):
    R = np.asarray(ref, np.float64)
    Q = np.asarray(query, np.float64).reshape(-1, 3)
    if Q.shape[0] == 0:
        return np.zeros(0)
    k = min(k, R.shape[0])
    _, idx = cKDTree(R).query(Q, k=k)
    idx = idx.reshape(Q.shape[0], k)
    d = R[idx] - Q[:, None, :]
    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    return d2.min(1)


def masks(data_down, obs_mask, bb, res, patch):
    """eval.py:100-110: (inbound, grid_inbound, in_obs)."""
    BB = np.asarray(bb).astype(np.float32)
    inbound = ((data_down >= BB[:1] - patch) & (data_down < BB[1:] + patch * 2)).sum(axis=-1) == 3
    data_in = data_down[inbound]
    data_grid = np.around((data_in - BB[:1]) / res).astype(np.int32)
    grid_inbound = ((data_grid >= 0) & (data_grid < np.expand_dims(obs_mask.shape, 0))).sum(axis=-1) == 3
    g = data_grid[grid_inbound]
    in_obs = obs_mask[g[:, 0], g[:, 1], g[:, 2]].astype(np.bool_)
    return inbound, grid_inbound, in_obs


def evaluate(data, stl, obs_mask, bb, res, plane, mode="mesh", faces=None, downsample_density=0.2, patch_size=60.0, max_dist=20.0,
             visualize_threshold=10.0, seed=0, perm=None):
    r = downsample_density
    data_pcd = sample_mesh(data, faces if faces is not None else np.zeros((0, 3), np.int64), r) if mode == "mesh" \
        else np.asarray(data, np.float64)
    if perm is None:
        perm = np.random.default_rng(seed).permutation(data_pcd.shape[0])
    kept = ordered_downsample(data_pcd, perm, r)
    data_down = data_pcd[np.asarray(perm)][kept]
    obs_mask = np.asarray(obs_mask)
    inbound, grid_inbound, in_obs = masks(data_down, obs_mask, bb, res, patch_size)
    data_in = data_down[inbound]
    data_in_obs = data_in[grid_inbound][in_obs]
    stl = np.asarray(stl, np.float64)
    dist_d2s = np.sqrt(nn_sqdist(stl, data_in_obs))[:, None]
    stl_hom = np.concatenate([stl, np.ones_like(stl[:, :1])], -1)
    above = (np.asarray(plane, np.float64).reshape((1, 4)) * stl_hom).sum(-1) > 0
    dist_s2d = np.sqrt(nn_sqdist(data_in, stl[above]))[:, None]
    with warnings.catch_warnings(), np.errstate(invalid="ignore", divide="ignore"):
        warnings.simplefilter("ignore", RuntimeWarning)
        mean_d2s = dist_d2s[dist_d2s < max_dist].mean()
        mean_s2d = dist_s2d[dist_s2d < max_dist].mean()
    vis = visualize_threshold
    R, G, B, W = (np.array([c], dtype=np.float64) for c in ([1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 1]))
    data_color = np.tile(B, (data_down.shape[0], 1))
    a = dist_d2s.clip(max=vis) / vis
    sel = np.where(inbound)[0][grid_inbound][in_obs]
    data_color[sel] = R * a + W * (1 - a)
    data_color[sel[dist_d2s[:, 0] >= max_dist]] = G
    stl_color = np.tile(B, (stl.shape[0], 1))
    a = dist_s2d.clip(max=vis) / vis
    data_sel = np.where(above)[0]
    stl_color[data_sel] = R * a + W * (1 - a)
    stl_color[data_sel[dist_s2d[:, 0] >= max_dist]] = G
    return {"data_pcd": data_pcd, "kept": kept, "data_down": data_down, "inbound": inbound, "grid_inbound": grid_inbound,
            "in_obs": in_obs, "above": above, "dist_d2s": dist_d2s, "dist_s2d": dist_s2d, "mean_d2s": float(mean_d2s),
            "mean_s2d": float(mean_s2d), "overall": float((mean_d2s + mean_s2d) / 2), "data_color": data_color,
            "stl_color": stl_color}
