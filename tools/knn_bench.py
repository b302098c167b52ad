"""distCUDA2 timings: this package's simple_knn (csrc/knn.cu) against the unmodified reference extension
(oracle/_ref/simple_knn_ref_C*.so, oracle/build_ref_knn.sh), alternating calls in one process, with a bit-identity check of
the two outputs at every size both ran.  CUDA events around single calls after warm-up; the median is reported.

  python tools/knn_bench.py [--reps 5] [--ref-max 4194304] [--cases uniform:1048576,core:1048576]

The reference is quadratic (every point tests every 1024-point box), so it is only run up to --ref-max points.
Prints one line per case and a JSON summary with the card name and its power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "gaussian-opacity-fields_b200"), os.path.join(ROOT, "tests", "golden")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import gof_synth  # noqa: E402

M = 1 << 20
DEFAULT = [("uniform", M), ("uniform", 4 * M), ("uniform", 16 * M), ("colmap", M), ("colmap", 4 * M), ("colmap", 16 * M),
           ("core", M), ("lattice", M)]


def _time(fn, x, reps):
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn(x)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), out


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return q
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-max", type=int, default=4 * M)
    ap.add_argument("--cases", default="")
    a = ap.parse_args()
    cases = [(c.split(":")[0], int(c.split(":")[1])) for c in a.cases.split(",")] if a.cases else DEFAULT
    from simple_knn._C import distCUDA2
    ref = None
    try:
        import make_golden_knn
        ref = make_golden_knn.load_reference().distCUDA2
    except Exception as e:  # the reference is optional: without it only our times are reported
        print(f"[knn_bench] reference not available ({e})")
    card = _card()
    print(f"[knn_bench] {card}")
    rows = []
    for kind, P in cases:
        x = torch.from_numpy(gof_synth.make_point_cloud(kind, P, seed=1)).cuda()
        distCUDA2(x)
        run_ref = ref is not None and P <= a.ref_max
        if run_ref:
            ref(x)
        ours, rmed = [], []
        out_o = out_r = None
        for _ in range(a.reps):   # alternate single calls so both see the same clocks
            t, out_o = _time(distCUDA2, x, 1)
            ours.append(t)
            if run_ref:
                t, out_r = _time(ref, x, 1)
                rmed.append(t)
        row = dict(kind=kind, P=P, ours_ms=round(float(np.median(ours)), 3))
        if run_ref:
            row["ref_ms"] = round(float(np.median(rmed)), 3)
            row["speedup"] = round(row["ref_ms"] / row["ours_ms"], 1)
            row["bit_identical"] = bool(torch.equal(out_o.view(torch.int32), out_r.view(torch.int32)))
            assert row["bit_identical"], f"outputs differ at {kind} {P}"
        print(f"[knn_bench] {kind:8s} P={P:>9d}  ours {row['ours_ms']:9.3f} ms" +
              (f"  reference {row['ref_ms']:10.3f} ms  x{row['speedup']}  bit-identical" if run_ref else ""))
        rows.append(row)
        del x
        torch.cuda.empty_cache()
    print(json.dumps(dict(card=card, reps=a.reps, cases=rows)))


if __name__ == "__main__":
    main()
