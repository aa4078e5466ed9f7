"""Fundamental matrices of many uncalibrated pairs: `estimate_fundamentals` (`ltr_fundamental`) against
cv2.findFundamentalMat(FM_RANSAC) per pair.

    python tools/fundamental_bench.py [--pairs 496] [--points 1000] [--lines 300] [--outliers 0.5] [--hypotheses 2048]
                                      [--reps 5]

Data: --pairs uncalibrated pairs (different random intrinsics per view, 640 x 480, rotations up to 15 degrees) from
`synthetic.make_fundamental_correspondences`: --points point matches with 0.5 px of noise and --outliers of them moved
10 to 60 px off their epipolar lines, plus --lines line matches of projected 3D segments, 30 % of them moved off their
epipolar bands.  --unique distinct pairs are generated and repeated (each batch position still draws its own samples).
Device times are CUDA-event medians of --reps calls after a warm-up (the whole call: host pools, one pinned copy, the
two kernels), and the kernel time from ltr_profile_*.  The baseline is cv2.findFundamentalMat(FM_RANSAC, 3 px, prob
0.99999) on --host-pairs pairs when cv2 is importable.  Prints the accuracy, the GPU model and power limit (read in the
same run), then one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from linetr_b200 import _native as N, engine, geometry as G, synthetic as syn   # noqa: E402


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:   # pragma: no cover
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"


def make_matches(n_pairs, n_unique, n_points, n_lines, outliers, dev):
    cases = [syn.make_fundamental_correspondences(100 + u, n_points, n_lines, noise_px=0.5, outlier_frac=outliers)
             for u in range(n_unique)]
    k0 = [torch.from_numpy(d["kpts0"]).to(dev) for d in cases]
    k1 = [torch.from_numpy(d["kpts1"]).to(dev) for d in cases]
    order = [p % n_unique for p in range(n_pairs)]
    cat = lambda key: torch.from_numpy(np.concatenate([cases[u][key] for u in order]).astype(np.int32)).to(dev)
    off = lambda key: np.concatenate([[0], np.cumsum([len(cases[u][key]) for u in order])]).astype(np.int32)
    mp, ml = cat("matches_p"), cat("matches_l")
    z = torch.zeros(n_pairs, dtype=torch.int32, device=dev)
    res = engine.ImagePairMatches(ml, ml.float(), z, off("matches_l"), mp, mp.float(), z, off("matches_p"),
                                  [cases[u]["klines0"] for u in order], [cases[u]["klines1"] for u in order],
                                  [k0[u] for u in order], [k1[u] for u in order])
    return res, [cases[u] for u in order]


def time_cuda(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(np.min(ts)), float(np.max(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=496)
    ap.add_argument("--unique", type=int, default=16)
    ap.add_argument("--points", type=int, default=1000)
    ap.add_argument("--lines", type=int, default=300)
    ap.add_argument("--outliers", type=float, default=0.5)
    ap.add_argument("--hypotheses", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-pairs", type=int, default=16)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fundamental_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    res, cases = make_matches(args.pairs, min(args.unique, args.pairs), args.points, args.lines, args.outliers, dev)
    P = res.n_pairs
    call = lambda: G.estimate_fundamentals(res, n_hypotheses=args.hypotheses)
    med, lo, hi = time_cuda(call, args.reps)
    N.profile_begin()
    r = call()
    prof = N.profile_end()
    kern = prof.get("fundamental", (float("nan"), 0))
    true_p = np.concatenate([d["true_p"] for d in cases])
    true_l = np.concatenate([d["true_l"] for d in cases])
    mp, ml = r.inliers_p.cpu().numpy().astype(bool), r.lines_consistent.cpu().numpy().astype(bool)
    recall = float((mp & true_p).sum() / true_p.sum())
    false_in = int((mp & ~true_p).sum())
    line_acc = float(np.mean(ml == true_l)) if len(ml) else float("nan")
    host = None
    try:
        import cv2
        k = min(args.host_pairs, P)
        t0 = time.perf_counter()
        for p in range(k):
            cv2.findFundamentalMat(cases[p]["kpts0"], cases[p]["kpts1"], cv2.FM_RANSAC, 3.0, 0.99999)
        host = (time.perf_counter() - t0) / k * 1e3
    except ImportError:
        pass
    gpu = gpu_info()
    print(f"{gpu}: {P} pairs, {args.points} point and {args.lines} line matches per pair, {args.outliers:.0%} point "
          f"outliers, {args.hypotheses} hypotheses")
    print(f"  estimate_fundamentals call median {med:8.3f} ms (min {lo:.3f}, max {hi:.3f}); kernels {kern[0]:.3f} ms "
          f"in {kern[1]} launches; {med / P * 1e3:.1f} us per pair")
    print(f"  valid {int(r.valid.sum())}/{P}, refitted {int(r.refit.sum())}; true inliers kept {recall:.4f}, outliers "
          f"accepted {false_in}; line check agrees with the truth on {line_acc:.4f} of the line matches")
    if host is not None:
        print(f"  cv2.findFundamentalMat(FM_RANSAC): {host:.2f} ms/pair -> {host * P / 1e3:.2f} s for {P} pairs")
    else:
        print("  cv2 not importable: no host comparison")
    print(json.dumps({"gpu": gpu, "pairs": P, "call_ms": med, "kernel_ms": kern[0], "inlier_recall": recall,
                      "outliers_accepted": false_in, "line_accuracy": line_acc, "cv2_ms_per_pair": host}))


if __name__ == "__main__":
    main()
