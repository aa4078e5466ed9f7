"""Line hypotheses in the absolute pose: recall and cost of `estimate_absolute_poses(..., n_line_hypotheses)`.

    python tools/line_localization_bench.py [--queries 64] [--db 4] [--lines 300] [--outliers 0.5] [--hypotheses 1024]
                                            [--line-hypotheses 0,256,1024] [--reps 5]

Point-poor scenes from `localization_bench.make_groups`: per query 2 k point matches at --outliers outliers (about k
point inliers, k = 0, 2, 4) and --lines line matches (30 % outliers), seen by --db database images.  Per count of line
hypotheses (per solver) it prints the recall of `localization_recall` (InLoc bins), the median call time (CUDA events
around the whole call after a warm-up) and the kernel time (ltr_profile_*), then the same times on the
`localization_bench` scene (1000 point and 300 line matches per pair), the cost the line hypotheses add there.  Prints
the GPU model and power limit read in the same run, then one JSON line.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from linetr_b200 import _native as N, localization as L, synthetic as syn   # noqa: E402
from tools.localization_bench import gpu_info, make_groups, time_cuda   # noqa: E402


def measure(scene, n_hyp, n_line, reps):
    res, X1, L1, groups, truth = scene
    call = lambda: L.estimate_absolute_poses(res, syn.DEFAULT_K, X1, L1, groups=groups, n_hypotheses=n_hyp,
                                             n_line_hypotheses=n_line)
    med, _, _ = time_cuda(call, reps)
    N.profile_begin()
    r = call()
    kern = N.profile_end().get("absolute_pose", (float("nan"), 0))[0]
    Rg, tg = np.stack([c["R"] for c in truth]), np.stack([c["t"] for c in truth])
    return med, kern, L.localization_recall(L.absolute_pose_errors(r.R, r.t, Rg, tg))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=64)
    ap.add_argument("--unique", type=int, default=64)
    ap.add_argument("--db", type=int, default=4)
    ap.add_argument("--lines", type=int, default=300)
    ap.add_argument("--outliers", type=float, default=0.5)
    ap.add_argument("--hypotheses", type=int, default=1024)
    ap.add_argument("--line-hypotheses", default="0,256,1024")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("line_localization_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    counts = [int(c) for c in args.line_hypotheses.split(",")]
    gpu = gpu_info()
    print(f"{gpu}: {args.queries} queries x {args.db} database images, {args.lines} line matches per pair, "
          f"{args.hypotheses} P3P hypotheses")
    rows = []
    for k in (0, 2, 4):
        scene = make_groups(args.queries, min(args.unique, args.queries), args.db, 2 * k, args.lines, args.outliers,
                            dev)
        for n_line in counts:
            med, kern, rec = measure(scene, args.hypotheses, n_line, args.reps)
            print(f"  ~{k} point inliers ({2 * k} matches), {n_line:5d} line hypotheses: recall "
                  f"{' / '.join(f'{r:.3f}' for r in rec)}; call {med:8.3f} ms, kernels {kern:8.3f} ms")
            rows.append({"point_matches": 2 * k, "line_hypotheses": n_line, "recall": rec, "call_ms": med,
                         "kernel_ms": kern})
    scene = make_groups(args.queries, 8, args.db, 1000, args.lines, args.outliers, dev)
    for n_line in counts:
        med, kern, rec = measure(scene, args.hypotheses, n_line, args.reps)
        print(f"  localization_bench scene, {n_line:5d} line hypotheses: recall "
              f"{' / '.join(f'{r:.3f}' for r in rec)}; call {med:8.3f} ms, kernels {kern:8.3f} ms")
        rows.append({"point_matches": 1000, "line_hypotheses": n_line, "recall": rec, "call_ms": med,
                     "kernel_ms": kern})
    print(json.dumps({"gpu": gpu, "rows": rows}))


if __name__ == "__main__":
    main()
