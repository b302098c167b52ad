#!/usr/bin/env python
"""Achieved HBM bandwidth of the two per-Gaussian kernels from a bench.py result line.

The bytes each kernel must move are counted from the code (csrc/preprocess.cu) for P Gaussians of which V are visible, with
D = 3 and M = 16 (192-byte SH rows):
  k_preprocess           36 P + 329 V   reads means 12, scales 12, rotation 16, opacity 4, SH 192; writes splat 64, splat_bwd
                                        32, radii/tiles/rect/key/order 24, depth 4, reject_k 4, clamped 1
  k_preprocess_backward  324 P + 365 V  writes every gradient element of every Gaussian (dL_dsh 192, dens_sum/max 20, ...); reads
                                        the 128-byte accumulator row, SH 192, means/scales/rotation 40 and one 32-byte sector of
                                        the splat record for the opacity

    python bench.py --gpus 1 --steps 30 --warmup 5 --no-cpu-baseline | tail -n 1 | python tools/preprocess_bytes.py
    python tools/preprocess_bytes.py result.json [--peak-gbs 3350]
"""
import argparse
import json
import sys

FWD_P, FWD_V = 36, 329     # bytes per Gaussian / per visible Gaussian, k_preprocess
BWD_P, BWD_V = 324, 365    # bytes per Gaussian / per visible Gaussian, k_preprocess_backward


def report(line, peak_gbs):
    P = int(line["config"]["workload"].split(": ")[1].split(" Gaussians")[0])   # "C3: 1000000 Gaussians, ..."
    V = int(line["config"]["visible"])
    kms = line["kernels_ms_per_step"]
    rows = []
    for name, bp, bv in (("preprocess_fwd", FWD_P, FWD_V), ("preprocess_bwd", BWD_P, BWD_V)):
        nbytes = bp * P + bv * V
        ms = kms[name]
        gbs = nbytes / (ms * 1e-3) / 1e9
        rows.append({"kernel": name, "P": P, "V": V, "bytes": nbytes, "ms": round(ms, 4), "GB/s": round(gbs, 1),
                     "floor_ms": round(nbytes / (peak_gbs * 1e9) * 1e3, 4), "frac_of_peak": round(gbs / peak_gbs, 3)})
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("result", nargs="?", help="file holding bench.py's JSON result line (default: stdin)")
    ap.add_argument("--peak-gbs", type=float, default=3350.0, help="HBM bandwidth to compare with (H100 SXM data sheet: 3350)")
    args = ap.parse_args()
    text = open(args.result).read() if args.result else sys.stdin.read()
    line = json.loads([ln for ln in text.splitlines() if ln.strip().startswith("{")][-1])
    for row in report(line, args.peak_gbs):
        print(json.dumps(row))


if __name__ == "__main__":
    main()
