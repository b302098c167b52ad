"""Writes tests/golden/tnt_eval_ref.npz: the reference's own eval_tnt/run.py (staged unmodified by baseline/stage_ref.sh, run as a
script by tests/_tnt_scenes.run_reference with stub open3d / trimesh / matplotlib modules built on oracle/tnt_eval_oracle.py) on
the two synthetic scenes of tests/_tnt_scenes.py, RANSAC seed 0.  Stored per scene: the inputs, the transformations after the
RANSAC and each registration, the ICP iteration counts, d1 / d2, the down-sampled clouds and the three .txt outputs.  CPU only."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import _tnt_scenes  # noqa: E402

SEED = 0


def main():
    out = {}
    for name, sc in _tnt_scenes.scenes().items():
        ref = _tnt_scenes.run_reference(sc, SEED)
        assert ref is not None, "run baseline/stage_ref.sh first"
        for k in ("vertices", "faces", "gt", "traj", "gt_trans", "polygon"):
            out[f"{name}/{k}"] = np.asarray(sc[k])
        out[f"{name}/crop"] = np.array([sc["axis"], sc["axis_min"], sc["axis_max"]], np.float64)
        for k in ("transforms", "icp_iterations", "prf", "cum_source", "cum_target", "d1", "d2", "source_down", "target_down"):
            out[f"{name}/{k}"] = np.asarray(ref[k])
        print(name, ref["icp_iterations"], ref["prf"])
    np.savez_compressed(os.path.join(HERE, "tnt_eval_ref.npz"), **out)


if __name__ == "__main__":
    main()
