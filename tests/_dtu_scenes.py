"""TEST INFRASTRUCTURE of the DTU evaluation: three synthetic scenes and a runner of the reference's own dtu_eval/eval.py
(staged unmodified as text by baseline/stage_ref.sh).  The runner executes the script as __main__ with an `open3d` stub that
serves the scene's arrays and captures write_point_cloud, np.random.default_rng bound to a seed, a serial multiprocessing.Pool,
and the .mat inputs written with scipy.io.savemat into a temporary dataset directory."""
import contextlib
import json
import os
import runpy
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_EVAL = os.path.join(ROOT, "baseline", "_ref", "gof_ref_py", "text", "dtu_eval.py")


def _uv_sphere(radius, nu, nv, rng, noise):
    th = np.linspace(0, np.pi, nv + 1)[1:-1]
    ph = np.linspace(0, 2 * np.pi, nu, endpoint=False)
    T, Pp = np.meshgrid(th, ph, indexing="ij")
    v = np.stack([np.sin(T) * np.cos(Pp), np.sin(T) * np.sin(Pp), np.cos(T)], -1).reshape(-1, 3)
    v = np.concatenate([v, [[0, 0, 1], [0, 0, -1]]]) * radius
    v = v + rng.normal(0, noise, v.shape)
    top, bot = len(v) - 2, len(v) - 1
    f = []
    for a in range(nv - 2):
        for b in range(nu):
            i0, i1 = a * nu + b, a * nu + (b + 1) % nu
            j0, j1 = i0 + nu, i1 + nu
            f += [[i0, j0, i1], [i1, j0, j1]]
    for b in range(nu):
        f += [[top, b, (b + 1) % nu], [bot, (nv - 2) * nu + (b + 1) % nu, (nv - 2) * nu + b]]
    return v, np.asarray(f, np.int64)


def _on_sphere(radius, n, rng):
    x = rng.normal(size=(n, 3))
    return x / np.linalg.norm(x, axis=1, keepdims=True) * radius


def _grid(bb, res, rng, fill):
    shape = tuple(int(s) for s in np.ceil((bb[1] - bb[0]) / res).astype(int) + 1)
    return (rng.random(shape) < fill).astype(np.uint8)


def scenes():
    """name -> dict(mode, data, faces, stl, obs_mask, bb, res, plane, args)"""
    out = {}
    rng = np.random.default_rng(11)
    v, f = _uv_sphere(20.0, 48, 34, rng, 0.25)
    bb = np.array([[-18.0, -22.0, -22.0], [22.0, 21.0, 15.0]])
    stl = np.concatenate([_on_sphere(20.0, 3000, rng), rng.uniform(-40, 40, (200, 3))])
    out["sphere"] = dict(mode="mesh", data=v, faces=f, stl=stl, obs_mask=_grid(bb, 2.0, rng, 0.8), bb=bb, res=np.array([[2.0]]),
                         plane=np.array([[0.1], [0.2], [1.0], [3.0]]),
                         args=dict(downsample_density=0.5, patch_size=1.5, max_dist=1.0, visualize_threshold=0.5))
    rng = np.random.default_rng(12)
    base = rng.uniform(-10, 10, (40, 3))
    tris = [[0, 1, 2], [3, 4, 5], [6, 7, 8], [9, 10, 11]]
    # degenerate: collinear and repeated vertices
    base[14] = base[12] + 0.5 * (base[13] - base[12])
    tris += [[12, 13, 14], [15, 15, 16], [17, 17, 17]]
    # sliver: a long, thin triangle
    base[20] = base[18] + np.array([0.0, 1e-3, 0.0])
    base[19] = base[18] + np.array([15.0, 0.0, 0.0])
    tris += [[18, 19, 20]]
    # tiny: well below the density (n1 = 0)
    base[22] = base[21] + np.array([0.01, 0.0, 0.0])
    base[23] = base[21] + np.array([0.0, 0.02, 0.0])
    tris += [[21, 22, 23]]
    # large: an 18 x 18 right triangle
    base[25] = base[24] + np.array([18.0, 0.0, 0.0])
    base[26] = base[24] + np.array([0.0, 0.0, 18.0])
    tris += [[24, 25, 26], [26, 25, 24], [27, 28, 29]]
    bb = np.array([[-12.0, -12.0, -12.0], [12.0, 12.0, 12.0]])
    stl = rng.uniform(-12, 12, (2500, 3))
    out["soup"] = dict(mode="mesh", data=base, faces=np.asarray(tris, np.int64), stl=stl, obs_mask=_grid(bb, 1.0, rng, 0.7), bb=bb,
                       res=np.array([[1.0]]), plane=np.array([[0.0], [0.3], [-1.0], [2.0]]),
                       args=dict(downsample_density=0.5, patch_size=3.0, max_dist=2.0, visualize_threshold=1.0))
    rng = np.random.default_rng(13)
    clusters = rng.uniform(-8, 8, (30, 3))
    pts = clusters[rng.integers(0, 30, 4000)] + rng.normal(0, 0.6, (4000, 3))
    lattice = np.stack(np.meshgrid(*[np.arange(8) * 0.5] * 3, indexing="ij"), -1).reshape(-1, 3) + 20.0   # spacing exactly r
    pts = np.concatenate([pts, lattice])
    bb = np.array([[-9.0, -9.0, -9.0], [9.0, 9.0, 9.0]])
    stl = np.concatenate([clusters[rng.integers(0, 30, 3000)] + rng.normal(0, 0.5, (3000, 3)), rng.uniform(-10, 25, (200, 3))])
    out["pcd"] = dict(mode="pcd", data=pts, faces=None, stl=stl, obs_mask=_grid(bb, 1.5, rng, 0.75), bb=bb, res=np.array([[1.5]]),
                      plane=np.array([[0.2], [-0.1], [0.5], [1.0]]),
                      args=dict(downsample_density=0.5, patch_size=12.0, max_dist=1.5, visualize_threshold=0.8))
    return out


def _open3d_stub(files, written):
    o3d = types.ModuleType("open3d")

    class PointCloud:
        def __init__(self):
            self.points, self.colors = None, None

    class Mesh:
        pass

    def read_triangle_mesh(path):
        m = Mesh()
        m.vertices, m.triangles = files[path]["vertices"], files[path]["triangles"]
        return m

    def read_point_cloud(path):
        pc = PointCloud()
        pc.points = files[path]["points"]
        return pc

    def write_point_cloud(path, pcd):
        written[os.path.basename(path)] = (np.array(pcd.points), np.array(pcd.colors))
        return True

    o3d.geometry = types.SimpleNamespace(PointCloud=PointCloud)
    o3d.utility = types.SimpleNamespace(Vector3dVector=lambda a: np.array(a, dtype=np.float64))
    o3d.io = types.SimpleNamespace(read_triangle_mesh=read_triangle_mesh, read_point_cloud=read_point_cloud,
                                   write_point_cloud=write_point_cloud)
    return o3d


class _SerialPool:
    def __init__(self, *a, **k):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False

    def map(self, fn, it, chunksize=None):
        return list(map(fn, it))


def write_dataset(d, sc, scan):
    from scipy.io import savemat
    os.makedirs(os.path.join(d, "ObsMask"), exist_ok=True)
    savemat(os.path.join(d, "ObsMask", f"ObsMask{scan}_10.mat"), {"ObsMask": sc["obs_mask"], "BB": sc["bb"], "Res": sc["res"]})
    savemat(os.path.join(d, "ObsMask", f"Plane{scan}.mat"), {"P": sc["plane"]})


def run_reference(sc, seed, scan=1):
    """Runs the staged eval.py on scene `sc`; returns dict(data_down, data_color, stl_color, mean_d2s, mean_s2d, overall) or None
    when the script is not staged."""
    if not os.path.exists(REF_EVAL):
        return None
    import multiprocessing
    files, written = {}, {}
    with tempfile.TemporaryDirectory() as d:
        write_dataset(d, sc, scan)
        data_path = os.path.join(d, "data.ply")
        if sc["mode"] == "mesh":
            files[data_path] = {"vertices": np.array(sc["data"], np.float64), "triangles": np.asarray(sc["faces"], np.int32)}
        else:
            files[data_path] = {"points": np.array(sc["data"], np.float64)}   # a copy: the script shuffles it in place
        files[f"{d}/Points/stl/stl{scan:03}_total.ply"] = {"points": np.array(sc["stl"], np.float64)}
        a = sc["args"]
        argv = [REF_EVAL, "--data", data_path, "--scan", str(scan), "--mode", sc["mode"], "--dataset_dir", d, "--vis_out_dir", d,
                "--downsample_density", repr(a["downsample_density"]), "--patch_size", repr(a["patch_size"]),
                "--max_dist", repr(a["max_dist"]), "--visualize_threshold", repr(a["visualize_threshold"])]
        orig_rng, orig_pool, orig_argv = np.random.default_rng, multiprocessing.Pool, sys.argv
        saved = sys.modules.get("open3d")
        sys.modules["open3d"] = _open3d_stub(files, written)
        np.random.default_rng = lambda *args, **kw: orig_rng(seed)
        multiprocessing.Pool = _SerialPool
        sys.argv = argv
        try:
            with contextlib.redirect_stdout(open(os.devnull, "w")), contextlib.redirect_stderr(open(os.devnull, "w")):
                runpy.run_path(REF_EVAL, run_name="__main__")
        finally:
            np.random.default_rng, multiprocessing.Pool, sys.argv = orig_rng, orig_pool, orig_argv
            if saved is None:
                sys.modules.pop("open3d", None)
            else:
                sys.modules["open3d"] = saved
        with open(os.path.join(d, "results.json")) as fh:
            res = json.load(fh)
    down, dcol = written[f"vis_{scan:03}_d2s.ply"]
    _, scol = written[f"vis_{scan:03}_s2d.ply"]
    return dict(data_down=down, data_color=dcol, stl_color=scol, **res)
