"""TEST INFRASTRUCTURE of the Tanks and Temples evaluation: two seeded synthetic scenes, writers of a scene directory in the
layout run.py reads, and a runner of the reference's own eval_tnt/run.py (staged unmodified as text by baseline/stage_ref.sh).
The runner executes the script as __main__ with stub modules built on the float64 oracle (oracle/tnt_eval_oracle.py):
`open3d` with only the 0.10 surface the scripts touch, in 0.10's positional signatures (ICPConvergenceCriteria(relative_fitness,
relative_rmse, max_iteration) included), `trimesh.load_mesh` without processing, and a no-op `matplotlib` / `cycler`."""
import contextlib
import os
import runpy
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "baseline", "_ref", "gof_ref_py", "eval_tnt")
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import tnt_eval_oracle as O  # noqa: E402


def _similarity(scale, angle_deg, axis, t):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    a = np.deg2rad(angle_deg)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    R = np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K
    T = np.eye(4)
    T[:3, :3] = scale * R
    T[:3, 3] = t
    return T


def _surface(x, y):
    return 0.3 * np.sin(2.0 * x) * np.cos(1.5 * y)


def _ring(n, radius, height, rng):
    """camera poses (camera-to-world) on a ring, looking at the origin; [n, 4, 4]"""
    P = np.tile(np.eye(4), (n, 1, 1))
    ang = np.linspace(0, 2 * np.pi, n, endpoint=False) + rng.uniform(0, 0.05, n)
    P[:, 0, 3] = radius * np.cos(ang)
    P[:, 1, 3] = radius * np.sin(ang)
    P[:, 2, 3] = height + rng.uniform(-0.2, 0.2, n)
    return P


def _scene(name, seed, gt_offset):
    rng = np.random.default_rng(seed)
    # the GT: samples of a height field in the GT frame, plus points exactly on the crop polygon's vertices and edges and on
    # axis_min / axis_max
    g = rng.uniform(-1.0, 1.0, (12000, 2))
    gt = np.stack([g[:, 0], g[:, 1], _surface(g[:, 0], g[:, 1])], 1)
    # a concave (L-shaped) polygon with axis-aligned edges, and a horizontal edge at v = -0.75
    poly = np.array([[-0.75, -0.75, 0.0], [0.75, -0.75, 0.0], [0.75, 0.0, 0.0], [0.0, 0.0, 0.0], [0.0, 0.75, 0.0], [-0.75, 0.75, 0.0]])
    axis_min, axis_max = -0.25, 0.25
    ties = [poly, (poly + np.roll(poly, -1, 0)) / 2,
            np.array([[-0.5, -0.5, axis_min], [-0.5, -0.4, axis_max], [0.5, -0.5, axis_min], [-0.3, 0.5, axis_max]])]
    gt = np.concatenate([gt] + ties) + gt_offset
    # the reconstruction: a noisy triangulated grid of the same surface, moved by the inverse of a similarity (scale != 1);
    # gt_trans maps the COLMAP frame (= the reconstruction's frame) to the GT frame, slightly off so ICP has work to do
    S_true = _similarity(1.7, 25.0, [0.2, 0.3, 1.0], [0.4, -0.2, 0.1])
    S_gt = S_true @ _similarity(1.0, 0.4, [1.0, 0.0, 0.2], [0.004, -0.003, 0.002])
    k = 40
    u = np.linspace(-1.0, 1.0, k)
    X, Y = np.meshgrid(u, u, indexing="ij")
    V = np.stack([X.ravel(), Y.ravel(), _surface(X.ravel(), Y.ravel())], 1) + rng.normal(0, 0.002, (k * k, 3))
    V = O.transform(V, np.linalg.inv(S_true))
    F = []
    for i in range(k - 1):
        for j in range(k - 1):
            a, b, c, d = i * k + j, i * k + j + 1, (i + 1) * k + j, (i + 1) * k + j + 1
            F += [[a, c, b], [b, c, d]]
    traj = _ring(48, 1.2, 0.8, rng)
    traj[:, :3, 3] = O.transform(traj[:, :3, 3], np.linalg.inv(S_true))
    return dict(name=name, vertices=V, faces=np.asarray(F, np.int64), gt=gt, traj=traj, gt_trans=S_gt, axis=2, axis_min=axis_min,
                axis_max=axis_max, polygon=poly, tau=O.SCENES_TAU[name])


def scenes():
    """name -> scene dict.  Barn: the full chain.  Truck: the GT lies outside the crop volume (the zeros branch)."""
    return {"Barn": _scene("Barn", 21, np.zeros(3)), "Truck": _scene("Truck", 22, np.array([0.0, 0.0, 5.0]))}


def volume(sc):
    return O.crop_volume(sc["axis"], sc["axis_min"], sc["axis_max"], sc["polygon"])


# ---- files -----------------------------------------------------------------------------------------------------------------

def write_log(path, poses):
    with open(path, "w") as fh:
        for i, P in enumerate(np.asarray(poses, np.float64).reshape(-1, 4, 4)):
            fh.write(f"{i} {i} {len(poses)}\n")
            for r in range(4):
                fh.write(" ".join(repr(float(x)) for x in P[r]) + "\n")


def write_mesh_ply(path, vertices, faces):
    V = np.ascontiguousarray(vertices, "<f8")
    F = np.asarray(faces, np.int64)
    face = np.empty(F.shape[0], dtype=[("n", "u1"), ("i", "<i4", (3,))])
    face["n"], face["i"] = 3, F
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {V.shape[0]}\nproperty double x\nproperty double y\nproperty double z\n"
              f"element face {F.shape[0]}\nproperty list uchar int vertex_indices\nend_header\n")
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        fh.write(V.tobytes())
        fh.write(face.tobytes())


def write_dataset(root, sc):
    """root/<name>/{name}_COLMAP_SfM.log, _trans.txt, .json, .ply (GT) and root/mesh.ply; returns (scene dir, mesh path)."""
    import json
    d = os.path.join(root, sc["name"])
    os.makedirs(d, exist_ok=True)
    write_log(os.path.join(d, sc["name"] + "_COLMAP_SfM.log"), sc["traj"])
    np.savetxt(os.path.join(d, sc["name"] + "_trans.txt"), sc["gt_trans"], fmt="%.17g")
    with open(os.path.join(d, sc["name"] + ".json"), "w") as fh:
        json.dump({"class_name": "SelectionPolygonVolume", "version_major": 1, "version_minor": 0,
                   "orthogonal_axis": "XYZ"[sc["axis"]], "axis_min": sc["axis_min"], "axis_max": sc["axis_max"],
                   "bounding_polygon": np.asarray(sc["polygon"]).tolist()}, fh)
    write_mesh_ply(os.path.join(d, sc["name"] + ".ply"), sc["gt"], np.zeros((0, 3), np.int64))
    mesh = os.path.join(root, "mesh.ply")
    write_mesh_ply(mesh, sc["vertices"], sc["faces"])
    return d, mesh


# ---- the stubbed reference run ---------------------------------------------------------------------------------------------

class _Nop:
    """matplotlib / cycler stand-in: every attribute, call, item and arithmetic gives itself"""

    def __getattr__(self, name):
        return self

    def __call__(self, *a, **k):
        return self

    def __setitem__(self, k, v):
        pass

    def __mul__(self, o):
        return self

    __rmul__ = __add__ = __radd__ = __mul__

    def __iter__(self):
        return iter(())


class _Pyplot(_Nop):
    """a no-op pyplot whose colour maps give black (the colours of the written clouds are not compared)"""

    def get_cmap(self, name):
        return lambda x: np.zeros((len(x), 4))


def _open3d_stub(files, log):
    o3d = types.ModuleType("open3d")

    class Points(list):
        pass

    def vec3(a):
        return Points([np.asarray(p, np.float64) for p in np.asarray(a, np.float64).reshape(-1, 3)])

    class PointCloud:
        def __init__(self):
            self.points = Points()

        def _arr(self):
            return np.asarray(self.points, np.float64).reshape(-1, 3)

        def _make(self, a):
            pc = PointCloud()
            pc.points = vec3(a)
            return pc

        def transform(self, T):
            log["transforms"].append((len(self.points), np.array(T, np.float64)))
            self.points = vec3(O.transform(self._arr(), T))
            return self

        def voxel_down_sample(self, voxel_size):
            return self._make(O.voxel_down_sample(self._arr(), voxel_size))

        def uniform_down_sample(self, every_k_points):
            return self._make(self._arr()[::every_k_points])

        def estimate_normals(self, search_param=None):
            return True

        def compute_point_cloud_distance(self, target):
            d = O.distances(self._arr(), target._arr())
            log["distances"].append(d)
            return Points(list(d))

    class Volume:
        def __init__(self, vol):
            self.vol = vol

        def crop_point_cloud(self, pcd):
            return pcd._make(O.crop(pcd._arr(), self.vol)[0])

    class Result:
        def __init__(self, T):
            self.transformation = T

    class RANSACConvergenceCriteria:
        def __init__(self, max_iteration=1000, max_validation=1000):
            self.max_iteration, self.max_validation = max_iteration, max_validation

    class ICPConvergenceCriteria:                # 0.10's positional order
        def __init__(self, relative_fitness=1e-6, relative_rmse=1e-6, max_iteration=30):
            self.relative_fitness, self.relative_rmse, self.max_iteration = relative_fitness, relative_rmse, max_iteration

    class TransformationEstimationPointToPoint:
        def __init__(self, with_scaling=False):
            assert with_scaling is True
            self.with_scaling = with_scaling

    def registration_ransac_based_on_correspondence(source, target, corres, max_dist, estimation, ransac_n, criteria):
        c = np.asarray(corres)
        assert np.array_equal(c[:, 0], np.arange(len(c))) and np.array_equal(c[:, 1], c[:, 0])
        T = O.ransac_alignment(source._arr(), target._arr(), log["seed"], max_dist, ransac_n,
                               min(criteria.max_iteration, criteria.max_validation))
        return Result(T)

    def registration_icp(source, target, max_dist, init, estimation, criteria):
        assert np.array_equal(init, np.eye(4))
        r = O.registration_icp(source._arr(), target._arr(), max_dist, max_iteration=criteria.max_iteration,
                               relative_fitness=criteria.relative_fitness, relative_rmse=criteria.relative_rmse)
        log["icp"].append(r["iterations"])
        return Result(r["transformation"])

    def read_point_cloud(path):
        pc = PointCloud()
        f = files[path]
        pc.points = vec3(f["vertices"] if isinstance(f, dict) else f)     # a mesh file reads as its vertices
        return pc

    def write_point_cloud(path, pcd):
        log["written"][os.path.basename(path)] = (pcd._arr(), np.asarray(getattr(pcd, "colors", np.zeros((0, 3)))))
        return True

    def read_selection_polygon_volume(path):
        return Volume(O.read_crop_volume(path))

    o3d.geometry = types.SimpleNamespace(PointCloud=PointCloud, KDTreeSearchParamKNN=lambda knn=30: None)
    o3d.utility = types.SimpleNamespace(Vector3dVector=vec3, Vector2iVector=lambda a: np.asarray(a, np.int64),
                                        set_verbosity_level=lambda level: None, VerbosityLevel=types.SimpleNamespace(Debug=0))
    o3d.io = types.SimpleNamespace(read_point_cloud=read_point_cloud, write_point_cloud=write_point_cloud)
    o3d.registration = types.SimpleNamespace(
        RANSACConvergenceCriteria=RANSACConvergenceCriteria, ICPConvergenceCriteria=ICPConvergenceCriteria,
        TransformationEstimationPointToPoint=TransformationEstimationPointToPoint,
        registration_ransac_based_on_correspondence=registration_ransac_based_on_correspondence, registration_icp=registration_icp)
    o3d.visualization = types.SimpleNamespace(read_selection_polygon_volume=read_selection_polygon_volume,
                                              draw_geometries=lambda *a, **k: None)
    return o3d


def _trimesh_stub(files):
    tm = types.ModuleType("trimesh")
    tm.load_mesh = lambda path, **k: types.SimpleNamespace(vertices=files[path]["vertices"], faces=files[path]["faces"])
    return tm


def run_reference(sc, seed=0):
    """Runs the staged run.py on scene sc; returns dict(transforms [4,4,4] (RANSAC, r2, r3, final), icp_iterations [3],
    prf [5], cum_source, cum_target, d1, d2, source_down, target_down, colors_source, colors_target), or None when the script
    is not staged."""
    if not os.path.exists(os.path.join(REF_DIR, "run.py")):
        return None
    files = {}
    log = {"seed": seed, "transforms": [], "icp": [], "distances": [], "written": {}}
    mpl = _Pyplot()
    stubs = {"open3d": _open3d_stub(files, log), "trimesh": _trimesh_stub(files), "matplotlib": mpl, "matplotlib.pyplot": mpl,
             "cycler": types.SimpleNamespace(cycler=mpl)}
    names = ("run", "config", "registration", "evaluation", "trajectory_io", "util", "plot")
    with tempfile.TemporaryDirectory() as root:
        d, mesh = write_dataset(root, sc)
        name = sc["name"]
        files[mesh] = {"vertices": np.array(sc["vertices"], np.float64), "faces": np.asarray(sc["faces"], np.int64)}
        files[os.path.join(d, name + ".ply")] = np.array(sc["gt"], np.float64)
        out = os.path.join(root, "out")
        argv = [os.path.join(REF_DIR, "run.py"), "--dataset-dir", d, "--traj-path", os.path.join(d, name + "_COLMAP_SfM.log"),
                "--ply-path", mesh, "--out-dir", out]
        saved = {k: sys.modules.get(k) for k in list(stubs) + list(names)}
        orig_argv, orig_path = sys.argv, list(sys.path)
        sys.modules.update(stubs)
        for k in names:
            sys.modules.pop(k, None)
        sys.argv = argv
        sys.path.insert(0, REF_DIR)
        try:
            with contextlib.redirect_stdout(open(os.devnull, "w")), contextlib.redirect_stderr(open(os.devnull, "w")):
                runpy.run_path(argv[0], run_name="__main__")
        finally:
            sys.argv, sys.path[:] = orig_argv, orig_path
            for k, v in saved.items():
                if v is None:
                    sys.modules.pop(k, None)
                else:
                    sys.modules[k] = v
        res = {k: np.loadtxt(os.path.join(out, f"{name}.{k}.txt"), ndmin=1)
               for k in ("precision", "recall", "prf_tau_plotstr")}
    n_src = sc["vertices"].shape[0] + sc["faces"].shape[0]
    T = [t for n, t in log["transforms"] if n == n_src]
    ps, pc = log["written"][f"{name}.precision.ply"]
    ts, tc = log["written"][f"{name}.recall.ply"]
    return {"transforms": np.stack(T), "icp_iterations": np.array(log["icp"]), "prf": res["prf_tau_plotstr"],
            "cum_source": res["precision"], "cum_target": res["recall"], "d1": np.asarray(log["distances"][0]),
            "d2": np.asarray(log["distances"][1]), "source_down": ps, "target_down": ts}

