"""DTU mesh evaluation on the GPU -- the reference's dtu_eval/eval.py without Open3D or scikit-learn.

    python -m gof_dtu_eval --data mesh.ply --scan 24 --mode mesh --dataset_dir DTU --vis_out_dir out [--seed 0]

takes the reference's arguments and defaults and writes the same results.json (mean_d2s, mean_s2d, overall) and the two
vis_{scan:03}_d2s.ply / vis_{scan:03}_s2d.ply clouds.  `evaluate(...)` runs the same steps on arrays and returns every
intermediate.  The contract is DESIGN section 4.6: sampling, downsampling and the nearest-neighbour distances run in
csrc/dtu_eval.cu in double precision, one IEEE operation at a time; the masks are element-wise torch ops on the device; the
scores and colours are the reference's own numpy expressions on the copied-back distances.  The reference shuffles with an
unseeded generator; here the order is np.random.default_rng(seed).permutation(n), which equals that generator's
shuffle(data, axis=0) for the same seed.
"""
import argparse
import ctypes
import json
import os
import warnings

import numpy as np
import torch

from diff_gaussian_rasterization import _C

_lib = _C._lib
_fp = ctypes.c_void_p
_i64 = ctypes.c_int64
_i64p = ctypes.POINTER(ctypes.c_int64)

for _name, _res, _args in (
        ("gof_mesh_sample_scratch_bytes", ctypes.c_size_t, [_i64]),
        ("gof_mesh_sample_count", ctypes.c_int, [_i64, _fp, _i64, _fp, ctypes.c_double, _fp, ctypes.c_size_t, _C._ALLOC_FN, _fp,
                                                 _i64p, _fp]),
        ("gof_mesh_sample_emit", ctypes.c_int, [_i64, _fp, _i64, _fp, ctypes.c_double, _fp, _fp, _i64, _fp, _fp]),
        ("gof_ordered_downsample_scratch_bytes", ctypes.c_size_t, [_i64]),
        ("gof_ordered_downsample", ctypes.c_int, [_i64, _fp, _fp, ctypes.c_double, _fp, _i64p, _i64p, _fp, ctypes.c_size_t,
                                                  _C._ALLOC_FN, _fp, _fp]),
        ("gof_nn_dist_scratch_bytes", ctypes.c_size_t, [_i64, _i64]),
        ("gof_nn_dist", ctypes.c_int, [_i64, _fp, _i64, _fp, _fp, ctypes.c_int, _fp, ctypes.c_size_t, _fp])):
    getattr(_lib, _name).restype = _res
    getattr(_lib, _name).argtypes = _args

SORT_LIMIT = 2 ** 30   # points in any one sort (the library's radix passes)


def _device(device):
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    if dev.type != "cuda":
        raise RuntimeError("gof_b200 evaluation: a CUDA device is required (no CPU path)")
    return dev if dev.index is not None else torch.device("cuda", torch.cuda.current_device())


def _points(x, name, dev, allow_empty=False):
    t = torch.as_tensor(x).to(dev, torch.float64).contiguous()
    if t.dim() != 2 or t.shape[1] != 3:
        raise ValueError(f"{name}: expected [n, 3] coordinates, got shape {tuple(t.shape)}")
    if t.shape[0] == 0 and not allow_empty:
        raise ValueError(f"{name}: the cloud is empty")
    if t.shape[0] >= SORT_LIMIT:
        raise ValueError(f"{name}: {t.shape[0]} points; at most 2^30 - 1 are supported (the limit of the library's radix sort)")
    if t.numel() and not bool(torch.isfinite(t).all()):
        raise ValueError(f"{name}: non-finite coordinates")
    return t


def _scratch(nbytes, dev):
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=dev)


def sample_mesh(vertices, faces, density):
    """eval.py:48-71 on the device: [V + S, 3] float64 = the vertices in file order, then each face's samples by row and
    column.  vertices [V,3] and faces [F,3] (int) tensors on one CUDA device."""
    dev = vertices.device
    V = _points(vertices, "sample_mesh vertices", dev, allow_empty=True)
    F = torch.as_tensor(faces).to(dev, torch.int64).reshape(-1, 3).contiguous()
    nv, nf = int(V.shape[0]), int(F.shape[0])
    with torch.cuda.device(dev):
        scratch = _scratch(_lib.gof_mesh_sample_scratch_bytes(nf), dev)
        rows = _C._Scratch(dev)
        ns = ctypes.c_int64(0)
        _C._check(_lib.gof_mesh_sample_count(nv, V.data_ptr() if nv else None, nf, F.data_ptr() if nf else None, float(density),
                                             scratch.data_ptr(), scratch.numel(), rows.cb, None, ctypes.byref(ns), _C._stream()))
        out = torch.empty((nv + ns.value, 3), dtype=torch.float64, device=dev)
        if out.numel():
            _C._check(_lib.gof_mesh_sample_emit(nv, V.data_ptr() if nv else None, nf, F.data_ptr() if nf else None, float(density),
                                                scratch.data_ptr(), rows.tensor.data_ptr() if rows.tensor.numel() else None,
                                                ns.value, out.data_ptr(), _C._stream()))
    return out


def ordered_downsample(points, perm, radius):
    """eval.py:86-94 on the device: kept [n] bool over the order perm (position k holds points[perm[k]]): a position is kept iff
    no kept earlier position lies within ((dx*dx + dy*dy) + dz*dz) <= radius*radius.  Returns (kept, rounds)."""
    dev = points.device
    P = _points(points, "ordered_downsample points", dev, allow_empty=True)
    n = int(P.shape[0])
    perm = torch.as_tensor(perm)
    if perm.shape != (n,):
        raise ValueError(f"ordered_downsample: perm must have shape ({n},), got {tuple(perm.shape)}")
    perm = perm.to(dev).to(torch.int64)
    if n and (int(perm.min()) < 0 or int(perm.max()) >= n):
        raise ValueError("ordered_downsample: perm is not a permutation of 0 .. n-1")
    perm32 = perm.to(torch.int32).contiguous()
    kept = torch.zeros(n, dtype=torch.uint8, device=dev)
    rounds, pairs = ctypes.c_int64(0), ctypes.c_int64(0)
    with torch.cuda.device(dev):
        scratch = _scratch(_lib.gof_ordered_downsample_scratch_bytes(n), dev)
        nbr = _C._Scratch(dev)
        _C._check(_lib.gof_ordered_downsample(n, P.data_ptr() if n else None, perm32.data_ptr() if n else None, float(radius),
                                              kept.data_ptr() if n else None, ctypes.byref(rounds), ctypes.byref(pairs),
                                              scratch.data_ptr(), scratch.numel(), nbr.cb, None, _C._stream()))
    return kept.bool(), int(rounds.value)


def nn_dist(ref, query, sqrt=True):
    """eval.py:119-133 on the device: [m] float64, for every query the smallest ((dx*dx + dy*dy) + dz*dz) to any reference
    point, or its square root."""
    dev = ref.device
    R = _points(ref, "nn_dist reference", dev)
    Q = _points(query, "nn_dist query", dev, allow_empty=True)
    out = torch.empty(int(Q.shape[0]), dtype=torch.float64, device=dev)
    if out.numel() == 0:
        return out
    with torch.cuda.device(dev):
        scratch = _scratch(_lib.gof_nn_dist_scratch_bytes(R.shape[0], Q.shape[0]), dev)
        _C._check(_lib.gof_nn_dist(R.shape[0], R.data_ptr(), Q.shape[0], Q.data_ptr(), out.data_ptr(), int(bool(sqrt)),
                                   scratch.data_ptr(), scratch.numel(), _C._stream()))
    return out


def _timer(enabled):
    marks = []

    def mark(name):
        if enabled:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            marks.append((name, ev))
    return marks, mark


def evaluate(data, stl, obs_mask, bb, res, plane, mode="mesh", faces=None, downsample_density=0.2, patch_size=60.0, max_dist=20.0,
             visualize_threshold=10.0, seed=0, perm=None, device=None, timing=False):
    """eval.py:42-166 on arrays.  data: mesh vertices [V,3] (mode 'mesh', with faces [F,3]) or a point cloud [n,3] (mode 'pcd');
    stl [m,3]; obs_mask: the ObsMask grid; bb: BB [2,3]; res: Res; plane: P (4 values).  perm: the order of the downsample
    (default np.random.default_rng(seed).permutation(n)).  Returns a dict of the scores (mean_d2s, mean_s2d, overall), the
    per-point arrays as numpy (data_down, dist_d2s [k,1], dist_s2d [j,1], data_color, stl_color, masks), the number of
    downsample rounds and, with timing=True, per-stage milliseconds (CUDA events)."""
    if mode not in ("mesh", "pcd"):
        raise ValueError(f"evaluate: mode must be 'mesh' or 'pcd', got {mode!r}")
    dev = _device(device)
    marks, mark = _timer(timing)
    with torch.cuda.device(dev):
        mark("start")
        pts = _points(data, "data", dev, allow_empty=(mode == "mesh"))
        stl_t = _points(stl, "stl", dev)
        if mode == "mesh":
            data_pcd = sample_mesh(pts, torch.zeros((0, 3), dtype=torch.int64) if faces is None else faces, downsample_density)
        else:
            data_pcd = pts
        n = int(data_pcd.shape[0])
        if n == 0:
            raise ValueError("data: the cloud is empty")
        mark("sample")
        if perm is None:
            perm = np.random.default_rng(seed).permutation(n)
        perm_t = torch.as_tensor(np.asarray(perm)).to(dev)
        kept, rounds = ordered_downsample(data_pcd, perm_t, downsample_density)
        data_down = data_pcd[perm_t.long()][kept]
        mark("downsample")

        # masking (eval.py:97-110): the bounds are float32 as numpy computes them, compared in float64
        BB = np.asarray(bb).astype(np.float32)
        patch = patch_size
        lo = torch.as_tensor((BB[:1] - patch).astype(np.float64), device=dev)
        hi = torch.as_tensor((BB[1:] + patch * 2).astype(np.float64), device=dev)
        inbound = ((data_down >= lo) & (data_down < hi)).all(-1)
        data_in = data_down[inbound]
        bb0 = torch.as_tensor(BB[:1].astype(np.float64), device=dev)
        res_t = torch.as_tensor(np.asarray(res, dtype=np.float64), device=dev)
        data_grid = torch.round((data_in - bb0) / res_t).to(torch.int32)      # np.around: half to even
        obs = np.asarray(obs_mask)
        shape = torch.as_tensor(np.asarray(obs.shape, dtype=np.int64), device=dev)
        grid_inbound = ((data_grid >= 0) & (data_grid < shape)).all(-1)
        g = data_grid[grid_inbound].long()
        obs_t = torch.as_tensor(obs.astype(np.bool_).reshape(-1), device=dev)
        in_obs = obs_t[(g[:, 0] * obs.shape[1] + g[:, 1]) * obs.shape[2] + g[:, 2]]
        data_in_obs = data_in[grid_inbound][in_obs]
        if data_in.shape[0] == 0:
            raise ValueError("evaluate: no downsampled data point lies inside the bounding box (nothing to measure stl2data against)")
        mark("mask")

        dist_d2s = nn_dist(stl_t, data_in_obs)
        mark("data2stl")
        P = torch.as_tensor(np.asarray(plane, dtype=np.float64).reshape(4), device=dev)
        above = (((stl_t[:, 0] * P[0] + stl_t[:, 1] * P[1]) + stl_t[:, 2] * P[2]) + P[3]) > 0
        dist_s2d = nn_dist(data_in, stl_t[above])
        mark("stl2data")
        out = {k: v.cpu().numpy() for k, v in (("data_down", data_down), ("inbound", inbound), ("grid_inbound", grid_inbound),
                                               ("in_obs", in_obs), ("above", above))}
        out["dist_d2s"] = dist_d2s.cpu().numpy().reshape(-1, 1)
        out["dist_s2d"] = dist_s2d.cpu().numpy().reshape(-1, 1)
        mark("copy")
    out.update(_scores(out, stl_t.shape[0], max_dist, visualize_threshold))
    out["rounds"] = rounds
    out["num_samples"] = n
    if timing:
        torch.cuda.synchronize(dev)
        out["stage_ms"] = {b[0]: a[1].elapsed_time(b[1]) for a, b in zip(marks[:-1], marks[1:])}
    return out


def _scores(o, n_stl, max_dist, vis_dist):
    """eval.py:122, 134, 138-157 verbatim on the copied-back arrays."""
    dist_d2s, dist_s2d = o["dist_d2s"], o["dist_s2d"]
    inbound, grid_inbound, in_obs, above = o["inbound"], o["grid_inbound"], o["in_obs"], o["above"]
    with warnings.catch_warnings(), np.errstate(invalid="ignore", divide="ignore"):
        warnings.simplefilter("ignore", RuntimeWarning)
        mean_d2s = dist_d2s[dist_d2s < max_dist].mean()
        mean_s2d = dist_s2d[dist_s2d < max_dist].mean()
    R = np.array([[1, 0, 0]], dtype=np.float64)
    G = np.array([[0, 1, 0]], dtype=np.float64)
    B = np.array([[0, 0, 1]], dtype=np.float64)
    W = np.array([[1, 1, 1]], dtype=np.float64)
    data_color = np.tile(B, (o["data_down"].shape[0], 1))
    data_alpha = dist_d2s.clip(max=vis_dist) / vis_dist
    data_color[np.where(inbound)[0][grid_inbound][in_obs]] = R * data_alpha + W * (1 - data_alpha)
    data_color[np.where(inbound)[0][grid_inbound][in_obs][dist_d2s[:, 0] >= max_dist]] = G
    stl_color = np.tile(B, (n_stl, 1))
    stl_alpha = dist_s2d.clip(max=vis_dist) / vis_dist
    stl_color[np.where(above)[0]] = R * stl_alpha + W * (1 - stl_alpha)
    stl_color[np.where(above)[0][dist_s2d[:, 0] >= max_dist]] = G
    over_all = (mean_d2s + mean_s2d) / 2
    return {"mean_d2s": float(mean_d2s), "mean_s2d": float(mean_s2d), "overall": float(over_all),
            "data_color": data_color, "stl_color": stl_color}


# ---- PLY -----------------------------------------------------------------------------------------------------------

_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "<i2", "int16": "<i2", "ushort": "<u2",
              "uint16": "<u2", "int": "<i4", "int32": "<i4", "uint": "<u4", "uint32": "<u4", "float": "<f4", "float32": "<f4",
              "double": "<f8", "float64": "<f8"}


def read_ply(path):
    """Binary little-endian PLY: dict(points [V,3] float64 from the vertex x, y, z, faces [F,3] int64 or None).  Any scalar
    property type; the face element's index list must hold triangles.  Other elements are skipped when all their properties
    are scalar.  ASCII and big-endian files are refused."""
    with open(path, "rb") as fh:
        data = fh.read()
    marker = b"end_header"
    k = data.find(marker)
    if not data.startswith(b"ply") or k < 0:
        raise ValueError(f"read_ply: {path} is not a PLY file")
    end = data.index(b"\n", k) + 1
    lines = [ln.strip() for ln in data[:end].decode("ascii", "replace").splitlines()]
    fmt = next((ln.split()[1] for ln in lines if ln.startswith("format")), None)
    if fmt != "binary_little_endian":
        raise ValueError(f"read_ply: {path}: format {fmt}; only binary_little_endian is supported")
    elements = []
    for ln in lines:
        w = ln.split()
        if not w:
            continue
        if w[0] == "element":
            elements.append((w[1], int(w[2]), []))
        elif w[0] == "property":
            if w[1] == "list":
                elements[-1][2].append((w[4], "list", _PLY_TYPES[w[2]], _PLY_TYPES[w[3]]))
            else:
                if w[1] not in _PLY_TYPES:
                    raise ValueError(f"read_ply: {path}: unknown property type {w[1]}")
                elements[-1][2].append((w[2], _PLY_TYPES[w[1]]))
    off, points, faces = end, None, None
    for name, count, props in elements:
        lists = [p for p in props if len(p) == 4]
        if not lists:
            dt = np.dtype([(p[0], p[1]) for p in props])
            arr = np.frombuffer(data, dt, count, off)
            off += count * dt.itemsize
            if name == "vertex":
                points = np.stack([arr["x"], arr["y"], arr["z"]], 1).astype(np.float64)
            continue
        if name != "face" or len(props) != 1:
            raise ValueError(f"read_ply: {path}: list properties are supported only as the face element's single index list")
        _, _, ct, it = props[0]
        dt = np.dtype([("n", ct), ("i", it, (3,))])
        arr = np.frombuffer(data, dt, count, off)
        if count and not np.all(arr["n"] == 3):
            raise ValueError(f"read_ply: {path}: only triangle faces are supported")
        faces = arr["i"].astype(np.int64).reshape(-1, 3)
        off += count * dt.itemsize
    if points is None:
        raise ValueError(f"read_ply: {path} has no vertex element")
    return {"points": points, "faces": faces}


def write_vis_ply(path, points, colors):
    """Binary little-endian PLY: double x y z, uchar red green blue = round(clip(colour, 0, 1) * 255) (half away from zero)."""
    p = np.ascontiguousarray(points, np.float64).reshape(-1, 3)
    c = np.floor(np.clip(np.asarray(colors, np.float64), 0.0, 1.0) * 255.0 + 0.5).astype(np.uint8).reshape(-1, 3)
    vert = np.empty(p.shape[0], dtype=[("x", "<f8"), ("y", "<f8"), ("z", "<f8"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    vert["x"], vert["y"], vert["z"] = p[:, 0], p[:, 1], p[:, 2]
    vert["red"], vert["green"], vert["blue"] = c[:, 0], c[:, 1], c[:, 2]
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {p.shape[0]}\nproperty double x\nproperty double y\nproperty double z\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n")
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        fh.write(vert.tobytes())


# ---- command line ----------------------------------------------------------------------------------------------------

def parse_args(argv=None):
    parser = argparse.ArgumentParser(description="DTU Chamfer evaluation (dtu_eval/eval.py) on the GPU")
    parser.add_argument('--data', type=str, default='data_in.ply')
    parser.add_argument('--scan', type=int, default=1)
    parser.add_argument('--mode', type=str, default='mesh', choices=['mesh', 'pcd'])
    parser.add_argument('--dataset_dir', type=str, default='.')
    parser.add_argument('--vis_out_dir', type=str, default='.')
    parser.add_argument('--downsample_density', type=float, default=0.2)
    parser.add_argument('--patch_size', type=float, default=60)
    parser.add_argument('--max_dist', type=float, default=20)
    parser.add_argument('--visualize_threshold', type=float, default=10)
    parser.add_argument('--seed', type=int, default=0, help="seed of the shuffle before the downsample")
    return parser.parse_args(argv)


def main(argv=None):
    from scipy.io import loadmat
    args = parse_args(argv)
    ply = read_ply(args.data)
    obs_mask_file = loadmat(f'{args.dataset_dir}/ObsMask/ObsMask{args.scan}_10.mat')
    ObsMask, BB, Res = [obs_mask_file[attr] for attr in ['ObsMask', 'BB', 'Res']]
    plane = loadmat(f'{args.dataset_dir}/ObsMask/Plane{args.scan}.mat')['P']
    stl = read_ply(f'{args.dataset_dir}/Points/stl/stl{args.scan:03}_total.ply')["points"]
    out = evaluate(ply["points"], stl, ObsMask, BB, Res, plane, mode=args.mode,
                   faces=ply["faces"] if args.mode == "mesh" else None, downsample_density=args.downsample_density,
                   patch_size=args.patch_size, max_dist=args.max_dist, visualize_threshold=args.visualize_threshold, seed=args.seed)
    write_vis_ply(f'{args.vis_out_dir}/vis_{args.scan:03}_d2s.ply', out["data_down"], out["data_color"])
    write_vis_ply(f'{args.vis_out_dir}/vis_{args.scan:03}_s2d.ply', stl, out["stl_color"])
    print(out["mean_d2s"], out["mean_s2d"], out["overall"])
    with open(os.path.join(args.vis_out_dir, "results.json"), "w") as fp:
        json.dump({'mean_d2s': out["mean_d2s"], 'mean_s2d': out["mean_s2d"], 'overall': out["overall"]}, fp, indent=True)
    return out


if __name__ == "__main__":
    main()
