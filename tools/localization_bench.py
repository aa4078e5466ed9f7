"""Absolute pose of many queries: `estimate_absolute_poses` (`ltr_absolute_pose`) against cv2.solvePnPRansac per query.

    python tools/localization_bench.py [--queries 64] [--db 4] [--points 1000] [--lines 300] [--outliers 0.5]
                                       [--hypotheses 1024] [--reps 5]

Data: --queries queries, each matched against --db database images that hold its 3D points and segments in their own
row order (one group of --db pairs per query) from
`synthetic.make_localization_correspondences`: per pair --points 2D-3D point matches with 0.5 px of noise and
--outliers of them moved 10 to 60 px off their projection, plus --lines line matches of projected 3D segments, 30 % of
them moved off their projected lines.  --unique distinct groups are generated and repeated (each group still draws its
own samples).  Device times are CUDA-event medians of --reps calls after a warm-up (the whole call: host pools, one
pinned copy, the two kernels), and the kernel time from ltr_profile_*.  The baseline is cv2.solvePnPRansac (points
only, 8 px, 1024 iterations) on --host-queries queries when cv2 is importable.  Prints the accuracy, the GPU model and
power limit (read in the same run), then one JSON line.
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
from linetr_b200 import _native as N, engine, localization as L, synthetic as syn   # noqa: E402


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:   # pragma: no cover
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"


def make_groups(n_queries, n_unique, n_db, n_points, n_lines, outliers, dev):
    """Per query, one set of correspondences of one camera, seen by each of its n_db database images: image i holds
    the 3D points / segments in its own row order, and every query row matches its row there."""
    rng = np.random.default_rng(0)
    uniq = []
    for u in range(n_unique):
        c = syn.make_localization_correspondences(100 + u, n_points, n_lines, noise_px=0.5, outlier_frac=outliers)
        db = []
        for _ in range(n_db):
            pp, pl = rng.permutation(n_points), rng.permutation(len(c["klines0"]))
            db.append((c["points3d1"][pp], c["lines3d1"][pl], np.argsort(pp).astype(np.int32),
                       np.argsort(pl).astype(np.int32), torch.from_numpy(c["kpts0"][pp]).to(dev), c["klines0"][pl]))
        uniq.append((c, torch.from_numpy(c["kpts0"]).to(dev), db))
    k0, l0, k1, l1, X1, L1, mp, ml, truth = [], [], [], [], [], [], [], [], []
    for q in range(n_queries):
        c, kq, db = uniq[q % n_unique]
        for X, E, m, n, kd, ld in db:
            k0.append(kq)
            l0.append(c["klines0"])
            k1.append(kd)
            l1.append(ld)
            X1.append(X)
            L1.append(E)
            mp.append(m)
            ml.append(n)
        truth.append(c)
    P = len(mp)
    off = lambda x: np.concatenate([[0], np.cumsum([len(v) for v in x])]).astype(np.int32)
    cat = lambda x: torch.from_numpy(np.concatenate(x)).to(dev)
    mpt, mlt = cat(mp), cat(ml)
    z = torch.zeros(P, dtype=torch.int32, device=dev)
    res = engine.ImagePairMatches(mlt, mlt.float(), z, off(ml), mpt, mpt.float(), z, off(mp), l0, l1, k0, k1)
    return res, X1, L1, np.arange(0, P + 1, n_db), truth


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
    ap.add_argument("--queries", type=int, default=64)
    ap.add_argument("--unique", type=int, default=8)
    ap.add_argument("--db", type=int, default=4)
    ap.add_argument("--points", type=int, default=1000)
    ap.add_argument("--lines", type=int, default=300)
    ap.add_argument("--outliers", type=float, default=0.5)
    ap.add_argument("--hypotheses", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-queries", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("localization_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    res, X1, L1, groups, truth = make_groups(args.queries, min(args.unique, args.queries), args.db, args.points,
                                             args.lines, args.outliers, dev)
    G = len(groups) - 1
    K = syn.DEFAULT_K
    call = lambda: L.estimate_absolute_poses(res, K, X1, L1, groups=groups, n_hypotheses=args.hypotheses)
    med, lo, hi = time_cuda(call, args.reps)
    N.profile_begin()
    r = call()
    prof = N.profile_end()
    kern = prof.get("absolute_pose", (float("nan"), 0))
    Rg = np.stack([c["R"] for c in truth])
    tg = np.stack([c["t"] for c in truth])
    et, eR = L.absolute_pose_errors(r.R, r.t, Rg, tg)
    true_p = np.concatenate([np.tile(c["true_p"], args.db) for c in truth])
    mp = r.inliers_p.cpu().numpy().astype(bool)
    recall = float((mp & true_p).sum() / true_p.sum())
    false_in = int((mp & ~true_p).sum())
    host = None
    try:
        import cv2
        k = min(args.host_queries, G)
        t0 = time.perf_counter()
        for q in range(k):
            c = truth[q]
            cv2.solvePnPRansac(c["points3d1"], c["kpts0"].astype(np.float64), K, None, iterationsCount=args.hypotheses, reprojectionError=8.0,
                               confidence=0.99999)
        host = (time.perf_counter() - t0) / k * 1e3
    except ImportError:
        pass
    gpu = gpu_info()
    print(f"{gpu}: {G} queries x {args.db} database images, {args.points} point and {args.lines} line matches per pair, "
          f"{args.outliers:.0%} point outliers, {args.hypotheses} hypotheses")
    print(f"  estimate_absolute_poses call median {med:8.3f} ms (min {lo:.3f}, max {hi:.3f}); kernels {kern[0]:.3f} ms "
          f"in {kern[1]} launches; {med / G * 1e3:.1f} us per query")
    print(f"  valid {int(r.valid.sum())}/{G}, refitted {int(r.refit.sum())}; true inliers kept {recall:.4f}, outliers "
          f"accepted {false_in}; median centre error {np.median(et):.2e}, rotation {np.median(eR):.2e} deg")
    if host is not None:
        print(f"  cv2.solvePnPRansac (points only): {host:.2f} ms/query -> {host * G / 1e3:.2f} s for {G} queries")
    else:
        print("  cv2 not importable: no host comparison")
    print(json.dumps({"gpu": gpu, "queries": G, "pairs": res.n_pairs, "call_ms": med, "kernel_ms": kern[0],
                      "inlier_recall": recall, "outliers_accepted": false_in, "median_centre_error": float(np.median(et)),
                      "median_rotation_deg": float(np.median(eR)), "cv2_ms_per_query": host}))


if __name__ == "__main__":
    main()
