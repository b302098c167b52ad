"""Tanks and Temples evaluation on the GPU -- the reference's eval_tnt/run.py without Open3D, trimesh or matplotlib.

    python -m gof_tnt_eval --dataset-dir DIR/Barn --traj-path DIR/Barn/Barn_COLMAP_SfM.log --ply-path mesh.ply [--out-dir OUT]
                           [--view-crop 0] [--seed 0]

takes run.py's flags and default out_dir (`evaluation/` beside the mesh) and writes the same {scene}.precision.txt,
{scene}.recall.txt and {scene}.prf_tau_plotstr.txt, the colour-coded {scene}.precision.ply / {scene}.recall.ply and, when
matplotlib imports, the PR plot.  `evaluate(...)` runs the same steps on arrays and returns every intermediate.  The contract is
DESIGN section 4.7: crop, voxel down-sample, the ICP correspondences and moments and the distances run in csrc/tnt_eval.cu and
csrc/dtu_eval.cu in double precision; the Umeyama fits (3x3 SVD), the convergence tests and the seeded RANSAC run on the host
in numpy; the scores and histograms are the reference's own numpy expressions on the copied-back distances.
"""
import argparse
import ctypes
import json
import math
import os

import numpy as np
import torch

from diff_gaussian_rasterization import _C
from gof_dtu_eval import read_ply, write_vis_ply

_lib = _C._lib
_fp = ctypes.c_void_p
_i64 = ctypes.c_int64
_i64p = ctypes.POINTER(ctypes.c_int64)
_dp = ctypes.POINTER(ctypes.c_double)

for _name, _res, _args in (
        ("gof_nn_tree_scratch_bytes", ctypes.c_size_t, [_i64]),
        ("gof_nn_tree_build", ctypes.c_int, [_i64, _fp, _fp, ctypes.c_size_t, _fp]),
        ("gof_nn_query_scratch_bytes", ctypes.c_size_t, [_i64]),
        ("gof_nn_query", ctypes.c_int, [_i64, _fp, ctypes.c_size_t, _i64, _fp, ctypes.c_double, ctypes.c_int, _fp, _fp, _fp,
                                         ctypes.c_size_t, _fp]),
        ("gof_crop_scratch_bytes", ctypes.c_size_t, [_i64]),
        ("gof_crop_polygon", ctypes.c_int, [_i64, _fp, _dp, ctypes.c_int, ctypes.c_double, ctypes.c_double, ctypes.c_int, _dp, _fp, _fp,
                                            _i64p, _fp, ctypes.c_size_t, _fp]),
        ("gof_voxel_down_sample_scratch_bytes", ctypes.c_size_t, [_i64]),
        ("gof_voxel_down_sample", ctypes.c_int, [_i64, _fp, ctypes.c_double, _fp, _i64p, _fp, ctypes.c_size_t, _fp]),
        ("gof_icp_moments_scratch_bytes", ctypes.c_size_t, [_i64]),
        ("gof_icp_moments", ctypes.c_int, [_i64, _fp, _fp, _fp, _fp, _dp, _fp, ctypes.c_size_t, _fp]),
        ("gof_transform_points", ctypes.c_int, [_i64, _fp, _dp, _fp])):
    getattr(_lib, _name).restype = _res
    getattr(_lib, _name).argtypes = _args

SORT_LIMIT = 2 ** 30   # points in any one sort (the library's radix passes)
MAX_POINT_NUMBER = 4e6                       # registration.py:41
MAX_POLYGON = 3072                           # polygon vertices the crop kernel stages in shared memory
# config.py: scenes_tau_dict
SCENES_TAU = {"Barn": 0.01, "Caterpillar": 0.005, "Church": 0.025, "Courthouse": 0.025, "Ignatius": 0.003, "Meetingroom": 0.01,
              "Truck": 0.005}
# ICPConvergenceCriteria(1e-6, max_itr) binds positionally in Open3D 0.10 to (relative_fitness, relative_rmse); max_iteration
# keeps its default of 30 (DESIGN section 4.7)
ICP_CRITERIA = {"relative_fitness": 1e-6, "relative_rmse": 20.0, "max_iteration": 30}


def _device(device):
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    if dev.type != "cuda":
        raise RuntimeError("gof_tnt_eval: a CUDA device is required (no CPU path)")
    return dev if dev.index is not None else torch.device("cuda", torch.cuda.current_device())


def _points(x, name, dev):
    t = torch.as_tensor(x).to(dev, torch.float64)
    if t.dim() != 2 or t.shape[1] != 3:
        raise ValueError(f"{name}: expected [n, 3] coordinates, got shape {tuple(t.shape)}")
    if t.shape[0] >= SORT_LIMIT:
        raise ValueError(f"{name}: {t.shape[0]} points; at most 2^30 - 1 are supported (the limit of the library's radix sort)")
    if t.numel() and not bool(torch.isfinite(t).all()):
        raise ValueError(f"{name}: non-finite coordinates")
    return t.contiguous()


def _scratch(nbytes, dev):
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=dev)


def _mat(T):
    T = np.ascontiguousarray(np.asarray(T, np.float64).reshape(4, 4))
    if not np.isfinite(T).all():
        raise ValueError("non-finite transformation")
    return T, T.ctypes.data_as(_dp)


# ---- crop volume -------------------------------------------------------------------------------------------------------

def crop_volume(axis, axis_min, axis_max, polygon):
    """The polygon volume of read_selection_polygon_volume: axis 'x' / 'y' / 'z' (either case) or 0-2, the bounds along it and the
    polygon's [m, 3] vertices, of which the two other coordinates (ascending axis order) are kept."""
    if isinstance(axis, str):
        if axis.lower() not in ("x", "y", "z"):
            raise ValueError(f"crop volume: orthogonal_axis {axis!r} is not x, y or z")
        axis = "xyz".index(axis.lower())
    P = np.asarray(polygon, np.float64)
    if P.ndim != 2 or P.shape[1] != 3 or P.shape[0] < 3:
        raise ValueError(f"crop volume: bounding_polygon must hold at least 3 vertices of 3 coordinates, got shape {P.shape}")
    if P.shape[0] > MAX_POLYGON:
        raise ValueError(f"crop volume: {P.shape[0]} polygon vertices; at most {MAX_POLYGON} are supported")
    if not np.isfinite(P).all() or math.isnan(axis_min) or math.isnan(axis_max):
        raise ValueError("crop volume: non-finite polygon or bounds")
    u, v = [a for a in range(3) if a != axis]
    return {"axis": int(axis), "axis_min": float(axis_min), "axis_max": float(axis_max),
            "polygon_uv": np.ascontiguousarray(P[:, [u, v]])}


def read_crop_volume(path):
    """A SelectionPolygonVolume JSON file (class_name, orthogonal_axis, axis_min, axis_max, bounding_polygon)."""
    try:
        with open(path) as fh:
            d = json.load(fh)
    except (OSError, ValueError) as e:
        raise ValueError(f"crop volume {path}: {e}") from None
    if not isinstance(d, dict) or d.get("class_name", "SelectionPolygonVolume") != "SelectionPolygonVolume":
        raise ValueError(f"crop volume {path}: not a SelectionPolygonVolume")
    missing = [k for k in ("orthogonal_axis", "axis_min", "axis_max", "bounding_polygon") if k not in d]
    if missing:
        raise ValueError(f"crop volume {path}: missing {', '.join(missing)}")
    return crop_volume(d["orthogonal_axis"], float(d["axis_min"]), float(d["axis_max"]), d["bounding_polygon"])


# ---- stages on tensors ---------------------------------------------------------------------------------------------------

def crop(points, volume, transform=None, return_index=False):
    """SelectionPolygonVolume.crop_point_cloud, after `transform` (4x4) when given: the kept points in input order [k, 3]
    (and their input indices, int64)."""
    dev = points.device
    P = _points(points, "crop points", dev)
    n = int(P.shape[0])
    poly = np.ascontiguousarray(volume["polygon_uv"], np.float64)
    out = torch.empty((n, 3), dtype=torch.float64, device=dev)
    idx = torch.empty(n, dtype=torch.int32, device=dev) if return_index else None
    k = ctypes.c_int64(0)
    Tp = _mat(transform) if transform is not None else (None, None)
    with torch.cuda.device(dev):
        scratch = _scratch(_lib.gof_crop_scratch_bytes(n), dev)
        _C._check(_lib.gof_crop_polygon(n, P.data_ptr() if n else None, Tp[1], int(volume["axis"]), float(volume["axis_min"]),
                                        float(volume["axis_max"]), int(poly.shape[0]), poly.ctypes.data_as(_dp),
                                        out.data_ptr() if n else None, idx.data_ptr() if (n and idx is not None) else None,
                                        ctypes.byref(k), scratch.data_ptr(), scratch.numel(), _C._stream()))
    out = out[:k.value]
    return (out, idx[:k.value].long()) if return_index else out


def voxel_down_sample(points, voxel):
    """PointCloud.voxel_down_sample: per occupied voxel the mean of its points (summed in input order), in ascending (x, y, z)
    voxel order."""
    dev = points.device
    P = _points(points, "voxel_down_sample points", dev)
    n = int(P.shape[0])
    out = torch.empty((n, 3), dtype=torch.float64, device=dev)
    k = ctypes.c_int64(0)
    with torch.cuda.device(dev):
        scratch = _scratch(_lib.gof_voxel_down_sample_scratch_bytes(n), dev)
        _C._check(_lib.gof_voxel_down_sample(n, P.data_ptr() if n else None, float(voxel), out.data_ptr() if n else None,
                                             ctypes.byref(k), scratch.data_ptr(), scratch.numel(), _C._stream()))
    return out[:k.value]


def uniform_down_sample(points, max_points=MAX_POINT_NUMBER):
    """registration.py:125-129: every k-th point, k = round(n / max_points), when there are more than max_points."""
    n = int(points.shape[0])
    if n > max_points:
        return points[::int(round(n / float(max_points)))].contiguous()
    return points


class NNTree:
    """A 1-NN tree over ref kept on the device for repeated queries: query(q, r2) -> (index int32 or -1, d2) with the lowest
    index among equal distances and only d2 < r2 accepted."""

    def __init__(self, ref):
        self.dev = ref.device
        self.ref = _points(ref, "nn reference", self.dev)
        self.n = int(self.ref.shape[0])
        if self.n == 0:
            raise ValueError("nn reference: the cloud is empty")
        with torch.cuda.device(self.dev):
            self.scratch = _scratch(_lib.gof_nn_tree_scratch_bytes(self.n), self.dev)
            _C._check(_lib.gof_nn_tree_build(self.n, self.ref.data_ptr(), self.scratch.data_ptr(), self.scratch.numel(), _C._stream()))
        self._qscratch, self._qn = None, -1

    def query(self, q, r2=math.inf, reuse_order=False):
        Q = _points(q, "nn query", self.dev)
        m = int(Q.shape[0])
        idx = torch.empty(m, dtype=torch.int32, device=self.dev)
        d2 = torch.empty(m, dtype=torch.float64, device=self.dev)
        if m == 0:
            return idx, d2
        reuse = bool(reuse_order) and self._qn == m
        with torch.cuda.device(self.dev):
            if self._qn != m:
                self._qscratch, self._qn = _scratch(_lib.gof_nn_query_scratch_bytes(m), self.dev), m
            _C._check(_lib.gof_nn_query(self.n, self.scratch.data_ptr(), self.scratch.numel(), m, Q.data_ptr(), float(r2), int(reuse), idx.data_ptr(),
                                        d2.data_ptr(), self._qscratch.data_ptr(), self._qscratch.numel(), _C._stream()))
        return idx, d2


def icp_moments(src, tgt, idx, d2):
    """(count, sum d2, mean src, mean tgt, sum (t - mt)(s - ms)^T, sum |s - ms|^2) over the pairs (i, idx[i] >= 0)."""
    n = int(src.shape[0])
    if tgt.shape[0] == 0:                                # an empty target: no pairs
        return 0, 0.0, np.zeros(3), np.zeros(3), np.zeros((3, 3)), 0.0
    m = (ctypes.c_double * 18)()
    with torch.cuda.device(src.device):
        scratch = _scratch(_lib.gof_icp_moments_scratch_bytes(n), src.device)
        _C._check(_lib.gof_icp_moments(n, src.data_ptr() if n else None, tgt.data_ptr(),
                                       idx.data_ptr() if n else None, d2.data_ptr() if n else None, m, scratch.data_ptr(),
                                       scratch.numel(), _C._stream()))
    a = np.frombuffer(m, np.float64).copy()
    return int(a[0]), float(a[1]), a[2:5], a[5:8], a[8:17].reshape(3, 3), float(a[17])


def umeyama(n, ms, mt, cov, var):
    """Eigen::umeyama with scaling, from the moments of n pairs (the identity when n = 0), in float64 on the host."""
    T = np.eye(4)
    if n == 0:
        return T
    inv = 1.0 / n
    U, sv, Vt = np.linalg.svd(cov * inv)
    S = np.ones(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2] = -1.0
    R = U @ np.diag(S) @ Vt
    with np.errstate(divide="ignore", invalid="ignore"):
        c = (1.0 / (var * inv)) * float(sv @ S)
    T[:3, 3] = mt - c * (R @ ms)
    T[:3, :3] = R * c
    return T


def transform_points(points, T):
    """points <- T(points) in place on the device."""
    T, Tp = _mat(T)
    with torch.cuda.device(points.device):
        _C._check(_lib.gof_transform_points(int(points.shape[0]), points.data_ptr() if points.numel() else None, Tp, _C._stream()))
    return points


def registration_icp(source, target, threshold, relative_fitness=1e-6, relative_rmse=1e-6, max_iteration=30, trace=None):
    """registration_icp with TransformationEstimationPointToPoint(True) from the identity (Open3D 0.10's loop): correspondences
    = the nearest target point with d2 < float32(threshold^2); per iteration the update T = umeyama @ T is applied to the moving
    points in place; stops when |d fitness| < relative_fitness and |d rmse| < relative_rmse, or after max_iteration updates.
    Returns dict(transformation, iterations, fitness, inlier_rmse).  trace (a list) gets (moving, idx, d2) of every
    evaluation, as device tensors."""
    dev = source.device
    moving = _points(source, "icp source", dev).clone()
    tgt = _points(target, "icp target", dev)
    n = int(moving.shape[0])
    r2 = float(np.float32(threshold * threshold))
    tree = NNTree(tgt) if tgt.shape[0] and n else None
    first = [True]

    def evaluate():
        if tree is None:
            idx = torch.full((n,), -1, dtype=torch.int32, device=dev)
            d2 = torch.full((n,), math.inf, dtype=torch.float64, device=dev)
        else:
            idx, d2 = tree.query(moving, r2, reuse_order=not first[0])
            first[0] = False
        if trace is not None:
            trace.append((moving.clone(), idx, d2))
        mom = icp_moments(moving, tgt, idx, d2)
        fitness = mom[0] / n if n else 0.0
        rmse = math.sqrt(mom[1] / mom[0]) if mom[0] else 0.0
        return mom, fitness, rmse

    T = np.eye(4)
    mom, fitness, rmse = evaluate()
    it = 0
    for it in range(1, max_iteration + 1):
        update = umeyama(mom[0], *mom[2:])
        T = update @ T
        transform_points(moving, update)
        prev = (fitness, rmse)
        mom, fitness, rmse = evaluate()
        if abs(prev[0] - fitness) < relative_fitness and abs(prev[1] - rmse) < relative_rmse:
            break
    return {"transformation": T, "iterations": it, "fitness": fitness, "inlier_rmse": rmse}


# ---- trajectory alignment (host) -----------------------------------------------------------------------------------------

def _lsum(a, axis):
    a = np.moveaxis(a, axis, 0)
    acc = a[0]
    for x in a[1:]:
        acc = acc + x
    return acc


def _sq(d):
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def _transform_np(P, T):
    """[..., n, 3] by [..., 4, 4]: (((m00*x + m01*y) + m02*z) + m03) / w per row"""
    x, y, z = P[..., 0], P[..., 1], P[..., 2]
    r = [((T[..., k, 0, None] * x + T[..., k, 1, None] * y) + T[..., k, 2, None] * z) + T[..., k, 3, None] for k in range(4)]
    return np.stack([r[0] / r[3], r[1] / r[3], r[2] / r[3]], -1)


def align_trajectory(source, target, seed=0, max_distance=0.2, ransac_n=6, iterations=100000, chunk=2048):
    """registration_ransac_based_on_correspondence(source, target, i <-> i, max_distance, PointToPoint(True), ransac_n,
    iterations), seeded: the draws are np.random.default_rng(seed).integers(0, N, (iterations, ransac_n)); each is fitted by
    Umeyama with scaling (sums over the draw left to right); a pair is an inlier iff d2 < max_distance^2; the best hypothesis by
    fitness, then rmse, then draw index replaces the identity when it has an inlier.  Host numpy, in chunks of draws."""
    src = np.asarray(source, np.float64).reshape(-1, 3)
    tgt = np.asarray(target, np.float64).reshape(-1, 3)
    N = src.shape[0]
    if tgt.shape[0] != N:
        raise ValueError(f"align_trajectory: {N} source and {tgt.shape[0]} target cameras")
    if N < ransac_n or ransac_n < 3:
        return np.eye(4)
    draws = np.random.default_rng(seed).integers(0, N, (iterations, ransac_n))
    md2 = max_distance * max_distance
    best_fit, best_rmse, best_T = 0.0, 0.0, np.eye(4)
    inv = 1.0 / ransac_n
    for c0 in range(0, iterations, chunk):
        d = draws[c0:c0 + chunk]
        s, t = src[d], tgt[d]
        ms, mt = _lsum(s, 1) * inv, _lsum(t, 1) * inv
        ds, dt = s - ms[:, None], t - mt[:, None]
        cov = _lsum(dt[:, :, :, None] * ds[:, :, None, :], 1)
        var = _lsum(_sq(ds), 1)
        H = d.shape[0]
        Ts = np.full((H, 4, 4), np.nan)
        ok = np.isfinite(cov).all((1, 2))
        with np.errstate(all="ignore"):
            U, sv, Vt = np.linalg.svd(cov[ok] * inv)
            S = np.ones((U.shape[0], 3))
            S[np.linalg.det(U) * np.linalg.det(Vt) < 0, 2] = -1.0
            R = U @ (S[:, :, None] * Vt)
            c = (1.0 / (var[ok] * inv)) * np.einsum("hk,hk->h", sv, S)
            Th = np.zeros((U.shape[0], 4, 4))
            Th[:, 3, 3] = 1.0
            Th[:, :3, 3] = mt[ok] - c[:, None] * np.einsum("hij,hj->hi", R, ms[ok])
            Th[:, :3, :3] = R * c[:, None, None]
            Ts[ok] = Th
            d2 = _sq(_transform_np(src[None], Ts) - tgt[None])
        inl = d2 < md2
        good = inl.sum(1)
        fit = good / N
        rmse = np.sqrt(_lsum(np.where(inl, d2, 0.0), 1) / np.maximum(good, 1))
        for h in np.nonzero(good)[0]:
            if fit[h] > best_fit or (fit[h] == best_fit and rmse[h] < best_rmse):
                best_fit, best_rmse, best_T = fit[h], rmse[h], Ts[h].copy()
    return best_T


# ---- scoring -------------------------------------------------------------------------------------------------------------

def distances(s, t):
    """compute_point_cloud_distance: [len(s)] sqrt of the exact 1-NN d2 from s to t (0 per point when t is empty)."""
    if s.shape[0] == 0:
        return torch.zeros(0, dtype=torch.float64, device=s.device)
    if t.shape[0] == 0:
        return torch.zeros(s.shape[0], dtype=torch.float64, device=s.device)
    import gof_dtu_eval
    return gof_dtu_eval.nn_dist(t, s, sqrt=True)


def evaluate_histo(distance1, distance2, threshold, plot_stretch=5):
    """evaluation.py:173-215 on host arrays: (precision, recall, fscore, edges_source, cum_source, edges_target, cum_target)."""
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


def reconstruction_cloud(vertices, faces):
    """run.py:95-108: the mesh vertices in file order, then per face ((v0 + v1) + v2) / 3 (numpy's mean over the corners)."""
    V = vertices
    F = faces.long()
    if F.numel() and (int(F.min()) < 0 or int(F.max()) >= V.shape[0]):
        raise ValueError(f"mesh: a face index is outside [0, {V.shape[0]})")
    # the divisor as a device tensor: a Python-scalar divisor lets the CUDA kernel multiply by the rounded 1/3 instead, which
    # is not the correctly rounded quotient
    three = torch.full((1, 1), 3.0, dtype=torch.float64, device=V.device)
    return torch.cat([V, ((V[F[:, 0]] + V[F[:, 1]]) + V[F[:, 2]]) / three], 0)


def _timer(enabled):
    marks = []

    def mark(name):
        if enabled:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            marks.append((name, ev))
    return marks, mark


def evaluate(vertices, faces, gt, traj, colmap_traj, gt_trans, volume, dTau, seed=0, max_points=MAX_POINT_NUMBER, device=None,
             timing=False):
    """run.py:58-184 on arrays.  vertices [V,3] / faces [F,3] of the mesh; gt [m,3]; traj and colmap_traj [k,4,4] poses; gt_trans
    4x4; volume from crop_volume / read_crop_volume; dTau the scene's tau.  Returns a dict: T_ransac, T_r2, T_r3, T_r (the
    composed transformations after each step), iterations_r2/_r3/_r, source_down / target_down, d1, d2 (numpy), precision,
    recall, fscore, the edges and cumulative histograms and, with timing=True, per-stage milliseconds (CUDA events; the
    RANSAC is host time between two events)."""
    dev = _device(device)
    marks, mark = _timer(timing)
    out = {}
    with torch.cuda.device(dev):
        mark("start")
        V = _points(vertices, "mesh vertices", dev)
        F = torch.as_tensor(np.asarray(faces, np.int64) if not torch.is_tensor(faces) else faces).to(dev).reshape(-1, 3)
        pcd = reconstruction_cloud(V, F)
        gt_t = _points(gt, "gt", dev)
        mark("upload")
        traj = np.asarray(traj, np.float64).reshape(-1, 4, 4)
        col = np.asarray(colmap_traj, np.float64).reshape(-1, 4, 4)
        T0 = align_trajectory(traj[:, :3, 3], _transform_np(col[:, :3, 3], np.asarray(gt_trans, np.float64)), seed=seed)
        out["T_ransac"] = T0
        mark("ransac")
        init = T0
        for name, mode, voxel, thr in (("r2", "voxel", dTau, dTau * 80), ("r3", "voxel", dTau / 2.0, dTau * 20),
                                       ("r", "uniform", None, 2 * dTau)):
            s, t = crop(pcd, volume, init), crop(gt_t, volume)
            mark(f"{name}_crop")
            if mode == "voxel":
                s, t = voxel_down_sample(s, voxel), voxel_down_sample(t, voxel)
            else:
                s, t = uniform_down_sample(s, max_points), uniform_down_sample(t, max_points)
            mark(f"{name}_down")
            reg = registration_icp(s, t, thr, **ICP_CRITERIA)
            init = reg["transformation"] @ init
            out[f"T_{name}"] = init
            out[f"iterations_{name}"] = reg["iterations"]
            mark(f"{name}_icp")
        s = crop(pcd, volume, init)
        t = crop(gt_t, volume)
        mark("score_crop")
        s, t = voxel_down_sample(s, dTau / 2.0), voxel_down_sample(t, dTau / 2.0)
        mark("score_down")
        d1 = distances(s, t)
        mark("d1")
        d2 = distances(t, s)
        mark("d2")
        out.update(source_down=s.cpu().numpy(), target_down=t.cpu().numpy(), d1=d1.cpu().numpy(), d2=d2.cpu().numpy())
        mark("copy")
    p, r, f, es, cs, et, ct = evaluate_histo(out["d1"], out["d2"], dTau, 5)
    out.update(precision=p, recall=r, fscore=f, edges_source=es, cum_source=cs, edges_target=et, cum_target=ct)
    if timing:
        torch.cuda.synchronize(dev)
        out["stage_ms"] = {b[0]: a[1].elapsed_time(b[1]) for a, b in zip(marks[:-1], marks[1:])}
    return out


# ---- files ---------------------------------------------------------------------------------------------------------------

def read_trajectory(path):
    """trajectory_io.read_trajectory: [k, 4, 4] from a .log file (a metadata line, then four rows per pose); .npy loads
    directly; .json is refused (the reference's .json branch calls torch without importing it and raises NameError)."""
    if path.endswith(".npy"):
        return np.asarray(np.load(path), np.float64).reshape(-1, 4, 4)
    if path.endswith(".json"):
        raise ValueError(f"{path}: .json trajectories are not supported (run.py's .json branch does not run); "
                         "convert it to a .log or .npy file")
    mats = []
    with open(path) as fh:
        lines = fh.read().splitlines()
    k = 0
    while k < len(lines) and lines[k].strip():
        try:
            mats.append([[float(x) for x in lines[k + 1 + r].split()] for r in range(4)])
        except (IndexError, ValueError):
            raise ValueError(f"{path}: pose {len(mats)} is not four rows of four numbers") from None
        k += 5
    M = np.asarray(mats, np.float64).reshape(-1, 4, 4)
    if M.shape[0] == 0:
        raise ValueError(f"{path}: no poses")
    return M


def hot_r_lut(N=256):
    """matplotlib's 'hot_r' at N entries: LinearSegmentedColormap's lookup table built from the reversed segment data of
    'hot' ((1 - x, y1, y0) per point, last first), as matplotlib builds a reversed colormap."""
    seg = {"red": ((0., 0.0416, 0.0416), (0.365079, 1.0, 1.0), (1.0, 1.0, 1.0)),
           "green": ((0., 0., 0.), (0.365079, 0.0, 0.0), (0.746032, 1.0, 1.0), (1.0, 1.0, 1.0)),
           "blue": ((0., 0., 0.), (0.746032, 0.0, 0.0), (1.0, 1.0, 1.0))}
    lut = np.empty((N, 3))
    for c, name in enumerate(("red", "green", "blue")):
        a = np.asarray([(1.0 - x, y1, y0) for x, y0, y1 in reversed(seg[name])], np.float64)
        x, y0, y1 = a[:, 0], a[:, 1], a[:, 2]
        xind = np.linspace(0, 1, N)
        ind = np.searchsorted(x, xind)[1:-1]
        dist = (xind[1:-1] - x[ind - 1]) / (x[ind] - x[ind - 1])
        lut[:, c] = np.clip(np.concatenate([[y1[0]], dist * (y0[ind] - y1[ind - 1]) + y1[ind - 1], [y0[-1]]]), 0, 1)
    return lut


def distance_colors(distances, max_distance, N=256):
    """write_color_distances: hot_r(min(d, max) / max) with matplotlib's lookup (int(x * N), x = 1 -> N - 1)."""
    x = np.minimum(np.asarray(distances, np.float64), max_distance) / max_distance
    i = (x * N).astype(np.int64)
    i[i == N] = N - 1
    return hot_r_lut(N)[np.clip(i, 0, N - 1)]


def _mesh_report(points, faces):
    """exact-duplicate positions and unreferenced vertices: what trimesh's processing could merge or drop"""
    dup = points.shape[0] - np.unique(points, axis=0).shape[0] if points.shape[0] else 0
    used = np.zeros(points.shape[0], bool)
    if faces is not None and faces.size:
        used[faces.reshape(-1)] = True
    return int(dup), int((~used).sum())


def run_evaluation(dataset_dir, traj_path, ply_path, out_dir, seed=0):
    scene = os.path.basename(os.path.normpath(dataset_dir))
    if scene not in SCENES_TAU:
        raise ValueError(f"invalid dataset-dir {dataset_dir}: scene {scene!r} is not one of {sorted(SCENES_TAU)}")
    dTau = SCENES_TAU[scene]
    print(f"Evaluating {scene} (tau {dTau})")
    os.makedirs(out_dir, exist_ok=True)
    mesh = read_ply(ply_path)
    faces = mesh["faces"] if mesh["faces"] is not None else np.zeros((0, 3), np.int64)
    dup, unref = _mesh_report(mesh["points"], faces)
    print(f"{ply_path}: {mesh['points'].shape[0]} vertices, {faces.shape[0]} faces; {dup} exact-duplicate vertex positions, "
          f"{unref} unreferenced vertices (read as stored, not merged or dropped)")
    gt = read_ply(os.path.join(dataset_dir, scene + ".ply"))["points"]
    gt_trans = np.loadtxt(os.path.join(dataset_dir, scene + "_trans.txt"))
    traj = read_trajectory(traj_path)
    col = read_trajectory(os.path.join(dataset_dir, scene + "_COLMAP_SfM.log"))
    volume = read_crop_volume(os.path.join(dataset_dir, scene + ".json"))
    o = evaluate(mesh["points"], faces, gt, traj, col, gt_trans, volume, dTau, seed=seed)
    prefix = os.path.join(out_dir, scene)
    write_vis_ply(prefix + ".precision.ply", o["source_down"], distance_colors(o["d1"], 3 * dTau))
    write_vis_ply(prefix + ".recall.ply", o["target_down"], distance_colors(o["d2"], 3 * dTau))
    np.savetxt(prefix + ".recall.txt", o["cum_target"])
    np.savetxt(prefix + ".precision.txt", o["cum_source"])
    np.savetxt(prefix + ".prf_tau_plotstr.txt", np.array([o["precision"], o["recall"], o["fscore"], dTau, 5]))
    print(f"precision : {o['precision']:.4f}\nrecall : {o['recall']:.4f}\nf-score : {o['fscore']:.4f}")
    _plot(scene, o, dTau, out_dir)
    return o


def _plot(scene, o, dTau, out_dir, plot_stretch=5):
    try:
        import matplotlib
        matplotlib.use("Agg")
        import matplotlib.pyplot as plt
    except ImportError:
        print("matplotlib is not importable: the PR plot was skipped")
        return
    f = plt.figure()
    ax = plt.subplot(111)
    ax.plot(o["edges_source"][1::], o["cum_source"] * 100, c="red", label="precision", linewidth=2.0)
    ax.plot(o["edges_target"][1::], o["cum_target"] * 100, c="blue", label="recall", linewidth=2.0)
    ax.grid(True)
    plt.title("Precision and Recall: " + scene + ", " + "%02.2f f-score" % (o["fscore"] * 100))
    plt.axvline(x=dTau, c="black", ls="dashed", linewidth=2.0)
    plt.ylabel("# of points (%)", fontsize=15)
    plt.xlabel("Meters", fontsize=15)
    plt.axis([0, dTau * plot_stretch, 0, 100])
    ax.legend(loc="center left", bbox_to_anchor=(1, 0.5))
    name = os.path.join(out_dir, "PR_{0}_@d_th_0_{1}".format(scene, "%04d" % (dTau * 10000)))
    f.savefig(name + ".png", format="png", bbox_inches="tight")
    f.savefig(name + ".pdf", format="pdf", bbox_inches="tight")
    plt.close(f)


def parse_args(argv=None):
    parser = argparse.ArgumentParser(description="Tanks and Temples evaluation (eval_tnt/run.py) on the GPU")
    parser.add_argument("--dataset-dir", type=str, required=True, help="scene directory holding X.json, X.ply, X_trans.txt, ...")
    parser.add_argument("--traj-path", type=str, required=True, help="trajectory .log or .npy")
    parser.add_argument("--ply-path", type=str, required=True, help="reconstruction mesh (binary PLY)")
    parser.add_argument("--out-dir", type=str, default="", help="default: an `evaluation` directory beside the ply file")
    parser.add_argument("--view-crop", type=int, default=0, help="accepted and ignored, as run.py does")
    parser.add_argument("--seed", type=int, default=0, help="seed of the RANSAC trajectory alignment")
    args = parser.parse_args(argv)
    if args.out_dir.strip() == "":
        args.out_dir = os.path.join(os.path.dirname(args.ply_path), "evaluation")
    return args


def main(argv=None):
    args = parse_args(argv)
    return run_evaluation(args.dataset_dir, args.traj_path, args.ply_path, args.out_dir, seed=args.seed)


if __name__ == "__main__":
    main()
