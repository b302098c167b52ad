"""Loading of the golden fixtures (tests/golden/*.npz, produced from the reference by make_golden.py)."""
import ast
import glob
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def fixture_paths():
    return sorted(glob.glob(os.path.join(HERE, "golden", "f[0-9]_*.npz")))


def load(path):
    """One fixture as a dict.  A fixture too large for one file keeps its backward (grad*) and opacity-field query (int_*)
    arrays in bwd_<name>.npz / int_<name>.npz next to it; they are merged in here."""
    d = {}
    head, base = os.path.split(path)
    for part in (path, os.path.join(head, "bwd_" + base), os.path.join(head, "int_" + base)):
        if os.path.exists(part):
            z = np.load(part, allow_pickle=False)
            d.update({k: z[k] for k in z.files})
    d["cfg"] = ast.literal_eval(str(d["cfg"]))
    d["name"] = os.path.splitext(os.path.basename(path))[0]
    return d


def oracle_scene(fx):
    import gof_oracle
    cfg = fx["cfg"]
    has_colors = fx["colors_precomp"].shape[0] > 0
    return gof_oracle.Scene(cfg["W"], cfg["H"], float(fx["tanfovx"]), float(fx["tanfovy"]), fx["viewmatrix"], fx["projmatrix"],
                            fx["campos"], fx["means3D"], fx["opacities"], scales=fx["scales"], rotations=fx["rotations"],
                            shs=None if has_colors else fx["shs"], colors_precomp=fx["colors_precomp"] if has_colors else None,
                            sh_degree=cfg["sh_degree"], kernel_size=cfg["kernel_size"], scale_modifier=cfg["scale_modifier"],
                            bg=cfg["bg"])


def relerr(a, b):
    a = np.asarray(a, np.float64).ravel()
    b = np.asarray(b, np.float64).ravel()
    if a.size == 0:
        return 0.0, 0.0
    den = max(np.abs(b).max(), 1e-30)
    return float(np.abs(a - b).max() / den), float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))
