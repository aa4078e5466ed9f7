"""RANSAC homographies of many pairs: `estimate_homographies` (`ltr_homography`) against cv2.findHomography per pair.

    python tools/homography_bench.py [--views 32] [--points 1000] [--lines 300] [--outliers 0.5] [--reps 10]

Data: one scene of --points keypoints and --lines segments seen by --views views, each view related to the scene by a
random homography (corners moved by up to 6 % of the image) plus 0.5 px of noise; all exhaustive pairs of views (496
for 32), matched row to row, with --outliers of the matches replaced by a random other row.  This measures the
estimator alone, on the match counts `match_set` produces for SuperPoint-sized inputs.  Device times are CUDA-event
medians of --reps calls after a warm-up (the whole call: host pools, one pinned copy, the two kernels), the per-class
kernel time from ltr_profile_*.  cv2.findHomography(RANSAC, 3.0) runs on the points of --host-pairs pairs when cv2 is
importable.  Prints corner accuracy for lines only, points only and both, the GPU model and power limit, then one JSON
line.
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


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:   # pragma: no cover
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"


def make_matches(n_views, n_points, n_lines, outliers, dev, seed=0):
    rng = np.random.default_rng(seed)
    lo, hi = np.array([0.2 * W, 0.2 * H]), np.array([0.8 * W, 0.8 * H])
    kp = rng.uniform(lo, hi, (n_points, 2))
    a = rng.uniform(lo, hi, (n_lines, 2))
    t = rng.uniform(0, 2 * np.pi, n_lines)
    b = np.clip(a + rng.uniform(30, 150, n_lines)[:, None] * np.stack([np.cos(t), np.sin(t)], 1), lo, hi)
    Hs, kps, lines = [], [], []
    for _ in range(n_views):
        Hv = syn.random_homography(rng, W, H, 0.06)
        Hs.append(Hv)
        kps.append(torch.from_numpy((syn.warp_points(Hv, kp) + rng.normal(0, 0.5, kp.shape)).astype(np.float32)).to(dev))
        seg = np.stack([syn.warp_points(Hv, a), syn.warp_points(Hv, b)], 1) + rng.normal(0, 0.5, (n_lines, 2, 2))
        lines.append(seg)
    pairs = engine.exhaustive_pairs(n_views)
    P = len(pairs)

    def rows(n):
        m = np.tile(np.arange(n, dtype=np.int32), P)
        bad = rng.random(m.shape) < outliers
        m[bad] = (m[bad] + rng.integers(1, max(n, 2), int(bad.sum()))) % max(n, 1)
        return torch.from_numpy(m).to(dev), np.arange(P + 1, dtype=np.int32) * n

    ml, ol = rows(n_lines)
    mp, op = rows(n_points)
    z = torch.zeros(P, dtype=torch.int32, device=dev)
    res = engine.ImagePairMatches(ml, ml.float(), z, ol, mp, mp.float(), z, op,
                                  [lines[i] for i, _ in pairs], [lines[j] for _, j in pairs],
                                  [kps[i] for i, _ in pairs], [kps[j] for _, j in pairs])
    Hgt = np.stack([Hs[j] @ np.linalg.inv(Hs[i]) for i, j in pairs])
    return res, Hgt


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
    ap.add_argument("--lines", type=int, default=300)
    ap.add_argument("--outliers", type=float, default=0.5)
    ap.add_argument("--hypotheses", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--host-pairs", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("homography_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    res, Hgt = make_matches(args.views, args.points, args.lines, args.outliers, dev)
    P = res.n_pairs
    out, acc = {}, {}
    for name, kw in (("both", {}), ("points", {"use_lines": False}), ("lines", {"use_points": False})):
        call = lambda: G.estimate_homographies(res, n_hypotheses=args.hypotheses, **kw)
        out[f"call_{name}_ms"] = time_cuda(call, args.reps)
        N.profile_begin()
        r = call()
        prof = N.profile_end()
        out[f"kernel_{name}_ms"] = prof.get("homography", (float("nan"), 0))[0]
        m = G.homography_corner_error(r.H, Hgt, (H, W))
        acc[name] = {k: m[k] for k in ("mean_error", "accuracy_1", "accuracy_3", "accuracy_5")}
        acc[name]["valid"] = int(r.valid.sum())
    host = None
    try:
        import cv2
        k = min(args.host_pairs, P)
        t0 = time.perf_counter()
        for p in range(k):
            a, b = res.offsets_p[p:p + 2]
            m = res.matches_p[a:b].cpu().numpy()
            cv2.findHomography(res.keypoints0[p].cpu().numpy(), res.keypoints1[p].cpu().numpy()[m], cv2.RANSAC, 3.0)
        host = (time.perf_counter() - t0) / k * 1e3
    except ImportError:
        pass
    gpu = gpu_info()
    print(f"{gpu}: {P} pairs, {args.points} point and {args.lines} line matches per pair, "
          f"{args.outliers:.0%} outliers, {args.hypotheses} hypotheses")
    for name in ("both", "points", "lines"):
        med, lo, hi = out[f"call_{name}_ms"]
        a = acc[name]
        print(f"  {name:6s} call median {med:8.3f} ms (min {lo:.3f}, max {hi:.3f}), kernels {out[f'kernel_{name}_ms']:.3f} ms;"
              f" valid {a['valid']}/{P}, mean corner error {a['mean_error']:.3f} px, accuracy @1/3/5 px "
              f"{a['accuracy_1']:.3f} / {a['accuracy_3']:.3f} / {a['accuracy_5']:.3f}")
    if host is not None:
        print(f"  cv2.findHomography(RANSAC, 3.0), points only: {host:.2f} ms/pair -> {host * P / 1e3:.2f} s for {P} pairs")
    else:
        print("  cv2 not importable: no host comparison")
    print(json.dumps({"gpu": gpu, "pairs": P, **{k: (v[0] if isinstance(v, tuple) else v) for k, v in out.items()},
                      "accuracy": acc, "cv2_ms_per_pair": host}))


if __name__ == "__main__":
    main()
