"""Writes tests/golden/dtu_eval_ref.npz: the reference's own dtu_eval/eval.py (staged unmodified by baseline/stage_ref.sh, run as
a script by tests/_dtu_scenes.run_reference) on the three synthetic scenes of tests/_dtu_scenes.py, shuffle seed 0.  Stored per
scene: the inputs, data_down, both colour arrays and the three scores.  CPU only (scikit-learn, scipy)."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import _dtu_scenes  # noqa: E402

SEED = 0


def main():
    out = {}
    for name, sc in _dtu_scenes.scenes().items():
        ref = _dtu_scenes.run_reference(sc, SEED)
        assert ref is not None, "run baseline/stage_ref.sh first"
        for k in ("data", "stl", "obs_mask", "bb", "res", "plane"):
            out[f"{name}/{k}"] = np.asarray(sc[k])
        if sc["faces"] is not None:
            out[f"{name}/faces"] = np.asarray(sc["faces"], np.int64)
        for k in ("data_down", "data_color", "stl_color"):
            out[f"{name}/{k}"] = ref[k]
        out[f"{name}/scores"] = np.array([ref["mean_d2s"], ref["mean_s2d"], ref["overall"]])
        print(name, ref["data_down"].shape, ref["mean_d2s"], ref["mean_s2d"], ref["overall"])
    np.savez_compressed(os.path.join(HERE, "dtu_eval_ref.npz"), **out)


if __name__ == "__main__":
    main()
