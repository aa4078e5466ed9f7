"""Relative pose of many pairs: `estimate_poses` (`ltr_essential`) against cv2.findEssentialMat + cv2.recoverPose per pair.

    python tools/pose_bench.py [--views 32] [--points 1000] [--outliers 0.5] [--hypotheses 1024] [--reps 5]

Data: one cloud of --points 3D points seen by --views calibrated cameras (f = 500 px, 640 x 480, rotations up to 4
degrees, centres within 0.8 of the origin, points 4 to 8 units away) with 0.5 px of noise; all exhaustive pairs of views
(496 for 32), matched row to row, with --outliers of the matches replaced by a random other row.  This measures the
estimator alone.  Device times are CUDA-event medians of --reps calls after a warm-up (the whole call: host pools, one
pinned copy, the two kernels), and the per-kernel time from ltr_profile_*.  The same pairs and hypotheses with 8
matches per pair split the kernel time: with 8 rows the scoring is negligible, so what remains is the solver.  The baseline is the reference's
estimate_pose (cv2.findEssentialMat(RANSAC, prob 0.99999) + cv2.recoverPose) on --host-pairs pairs when cv2 is
importable.  Prints the pose errors, the GPU model and power limit, then one JSON line.
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

W, H = 640, 480
K = syn.DEFAULT_K


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:   # pragma: no cover
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"


def make_matches(n_views, n_points, outliers, dev, seed=0):
    rng = np.random.default_rng(seed)
    _, Ts = syn.make_pose_set(seed, n_views, 0, 0)   # camera poses only
    X = np.c_[rng.uniform(-1.5, 1.5, (n_points, 2)), rng.uniform(4.0, 8.0, n_points)]
    kps = []
    for T in Ts:
        q = (X @ T[:3, :3].T + T[:3, 3]) @ K.T
        kps.append(torch.from_numpy((q[:, :2] / q[:, 2:] + rng.normal(0, 0.5, (n_points, 2))).astype(np.float32)).to(dev))
    pairs = engine.exhaustive_pairs(n_views)
    P = len(pairs)
    m = np.tile(np.arange(n_points, dtype=np.int32), P)
    bad = rng.random(m.shape) < outliers
    m[bad] = (m[bad] + rng.integers(1, n_points, int(bad.sum()))) % n_points
    mp, op = torch.from_numpy(m).to(dev), np.arange(P + 1, dtype=np.int32) * n_points
    ml = torch.zeros(0, dtype=torch.int32, device=dev)
    z = torch.zeros(P, dtype=torch.int32, device=dev)
    res = engine.ImagePairMatches(ml, ml.float(), z, np.zeros(P + 1, np.int32), mp, mp.float(), z, op,
                                  [np.zeros((0, 2, 2))] * P, [np.zeros((0, 2, 2))] * P,
                                  [kps[i] for i, _ in pairs], [kps[j] for _, j in pairs])
    Tgt = np.stack([Ts[j] @ np.linalg.inv(Ts[i]) for i, j in pairs])
    return res, Tgt


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
    ap.add_argument("--views", type=int, default=32)
    ap.add_argument("--points", type=int, default=1000)
    ap.add_argument("--outliers", type=float, default=0.5)
    ap.add_argument("--hypotheses", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-pairs", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pose_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    res, Tgt = make_matches(args.views, args.points, args.outliers, dev)
    P = res.n_pairs
    call = lambda: G.estimate_poses(res, K, K, n_hypotheses=args.hypotheses)
    med, lo, hi = time_cuda(call, args.reps)
    N.profile_begin()
    r = call()
    prof = N.profile_end()
    # the solver alone: the same pairs and hypotheses with 8 matches each, where scoring is negligible
    few, _ = make_matches(args.views, 8, 0.0, dev)
    G.estimate_poses(few, K, K, n_hypotheses=args.hypotheses)
    N.profile_begin()
    G.estimate_poses(few, K, K, n_hypotheses=args.hypotheses)
    solver = N.profile_end().get("essential", (float("nan"), 0))[0]
    et, eR = G.pose_errors(r.R, r.t, Tgt)
    err = np.maximum(et, eR)
    auc = G.pose_auc(err, [5, 10, 20])
    host = host_err = None
    try:
        import cv2
        k = min(args.host_pairs, P)
        tn = 1.0 / G._f_mean(K, K)
        Rs, ts = np.full((k, 3, 3), np.nan), np.full((k, 3), np.nan)
        t0 = time.perf_counter()
        for p in range(k):
            a, b = res.offsets_p[p:p + 2]
            x0 = G._normalised(res.keypoints0[p].cpu().numpy(), K)
            x1 = G._normalised(res.keypoints1[p].cpu().numpy()[res.matches_p[a:b].cpu().numpy()], K)
            E, mask = cv2.findEssentialMat(x0, x1, np.eye(3), threshold=tn, prob=0.99999, method=cv2.RANSAC)
            if E is None:
                continue
            # findEssentialMat may return several stacked solutions; keep the pose of the one recoverPose likes best
            poses = [cv2.recoverPose(E[i:i + 3], x0, x1, np.eye(3), 1e9, mask=mask.copy()) for i in range(0, len(E), 3)]
            n, R, t, _ = max(poses, key=lambda r: r[0])
            if n > 0:
                Rs[p], ts[p] = R, t[:, 0]
        host = (time.perf_counter() - t0) / k * 1e3
        errs = np.maximum(*G.pose_errors(Rs, ts, Tgt[:k]))
        host_err = float(np.median(errs))
    except ImportError:
        pass
    gpu = gpu_info()
    kern = prof.get("essential", (float("nan"), 0))
    print(f"{gpu}: {P} pairs, {args.points} point matches per pair, {args.outliers:.0%} outliers, "
          f"{args.hypotheses} hypotheses")
    print(f"  estimate_poses call median {med:8.3f} ms (min {lo:.3f}, max {hi:.3f}); kernels {kern[0]:.3f} ms in "
          f"{kern[1]} launches; {med / P * 1e3:.1f} us per pair")
    print(f"  kernels with 8 matches per pair (solver, staging and the pose kernel; scoring negligible): {solver:.3f} ms "
          f"-> scoring about {kern[0] - solver:.3f} ms")
    print(f"  valid {int(r.valid.sum())}/{P}; pose error max(t, R): median {np.median(err):.3f} deg, max "
          f"{err.max():.3f} deg; AUC @5/10/20 deg {auc[0]:.3f} / {auc[1]:.3f} / {auc[2]:.3f}")
    if host is not None:
        print(f"  cv2.findEssentialMat + recoverPose: {host:.2f} ms/pair -> {host * P / 1e3:.2f} s for {P} pairs; "
              f"median pose error {host_err:.3f} deg")
    else:
        print("  cv2 not importable: no host comparison")
    print(json.dumps({"gpu": gpu, "pairs": P, "call_ms": med, "kernel_ms": kern[0], "kernel_8_matches_ms": solver, "median_err_deg": float(np.median(err)),
                      "auc": auc, "cv2_ms_per_pair": host, "cv2_median_err_deg": host_err}))


if __name__ == "__main__":
    main()
