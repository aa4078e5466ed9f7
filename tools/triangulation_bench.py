"""Triangulation of a posed image set: `triangulate` (`ltr_triangulate`) against cv2.triangulatePoints per pair.

    python tools/triangulation_bench.py [--images 64] [--neighbours 4] [--points 2000] [--lines 300] [--outliers 0.3]
                                        [--reps 20]

Data: `synthetic.make_line_map_set` with --images posed views of one scene (every view sees every point and segment,
0.5 px of noise, --outliers of the observations moved 10 to 60 px), each image paired with its --neighbours next
images in a ring, so each image takes part in 2 --neighbours pairs (64 images: 256 pairs, 8 per image).  Matches are
the ground truth (outliers included).  Device times are CUDA-event medians of --reps calls after a warm-up (the whole
call: host checks and tables, one pinned copy, the two kernels), and the kernel time from ltr_profile_*.  Accuracy is
against the true 3D points and each view's true segment end points, over the rows whose anchor observation was not
moved.  The host reference is cv2.triangulatePoints per pair on the point matches only: two-view, no outlier
rejection.  Prints the GPU model and power limit read in the same run, then one JSON line.
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
from linetr_b200 import _native as N, engine, synthetic as syn, triangulation as T   # noqa: E402


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:   # pragma: no cover
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"


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
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def ring_matches(d, pairs, dev):
    n, m = len(d["points3d"]), len(d["segments3d"])
    P = len(pairs)
    mp = torch.arange(n, dtype=torch.int32, device=dev).repeat(P)
    ml = torch.arange(m, dtype=torch.int32, device=dev).repeat(P)
    z = torch.zeros(P, dtype=torch.int32, device=dev)
    kp, kl = d["keypoints"], d["klines"]
    return engine.ImagePairMatches(ml, ml.float(), z, np.arange(P + 1, dtype=np.int32) * m, mp, mp.float(), z,
                                   np.arange(P + 1, dtype=np.int32) * n, [kl[i] for i, _ in pairs],
                                   [kl[j] for _, j in pairs], [kp[i] for i, _ in pairs], [kp[j] for _, j in pairs])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--neighbours", type=int, default=4)
    ap.add_argument("--points", type=int, default=2000)
    ap.add_argument("--lines", type=int, default=300)
    ap.add_argument("--outliers", type=float, default=0.3)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("triangulation_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    V = args.images
    d = syn.make_line_map_set(0, V, args.points, args.lines, jitter_px=0.5, outlier_frac=args.outliers)
    pairs = np.array([(i, (i + k) % V) for i in range(V) for k in range(1, args.neighbours + 1)], dtype=np.int32)
    res = ring_matches(d, pairs, dev)
    call = lambda: T.triangulate(d["keypoints"], d["klines"], pairs, res, d["K"], d["R"], d["t"])
    med, lo, hi = time_cuda(call, args.reps)
    N.profile_begin()
    r = call()
    prof = N.profile_end()
    kern = prof.get("triangulate", (float("nan"), 0))
    n, m = len(d["points3d"]), len(d["segments3d"])
    X = r.points3d.cpu().numpy().reshape(V, n, 3)
    E = r.lines3d.cpu().numpy().reshape(V, m, 2, 3)
    nvp, nvl = r.n_views_p.cpu().numpy().reshape(V, n), r.n_views_l.cpu().numpy().reshape(V, m)
    cp, cl = ~d["outlier_p"], ~d["outlier_l"]
    centres = np.einsum("vji,vj->vi", -d["R"], d["t"])
    dist_p = np.linalg.norm(d["points3d"][None] - centres[:, None], axis=-1)
    err_p = np.linalg.norm(X - d["points3d"][None], axis=-1) / dist_p
    dist_l = np.linalg.norm(d["lines3d"] - centres[:, None, None], axis=-1)
    err_l = (np.linalg.norm(E - d["lines3d"], axis=-1) / dist_l).max(-1)
    vp, vl = cp & (nvp > 0), cl & (nvl > 0)
    host = None
    try:
        import cv2
        Pm = [syn.DEFAULT_K @ np.c_[d["R"][v], d["t"][v]] for v in range(V)]
        kp = [k.T.astype(np.float64) for k in d["keypoints"]]
        t0 = time.perf_counter()
        for i, j in pairs:
            cv2.triangulatePoints(Pm[i], Pm[j], kp[i], kp[j])
        host = (time.perf_counter() - t0) * 1e3
    except ImportError:
        pass
    gpu = gpu_info()
    print(f"{gpu}: {V} posed images, {len(pairs)} pairs ({2 * args.neighbours} per image), {n} keypoints and {m} key "
          f"lines per image, {args.outliers:.0%} of the observations moved 10-60 px, 0.5 px noise")
    print(f"  triangulate call median {med:8.3f} ms (min {lo:.3f}, max {hi:.3f}); kernels {kern[0]:.3f} ms in "
          f"{kern[1]} launches")
    print(f"  unmoved rows valid: points {vp.sum() / cp.sum():.4f}, lines {vl.sum() / cl.sum():.4f}; moved rows valid: "
          f"points {(~cp & (nvp > 0)).sum() / max((~cp).sum(), 1):.4f}; median n_views points {np.median(nvp[vp]):.0f}, "
          f"lines {np.median(nvl[vl]):.0f}")
    print(f"  error / distance to the camera over valid unmoved rows: points median {np.median(err_p[vp]):.2e}, "
          f"99th pct {np.percentile(err_p[vp], 99):.2e}; line end points median {np.median(err_l[vl]):.2e}, 99th pct "
          f"{np.percentile(err_l[vl], 99):.2e}")
    if host is not None:
        print(f"  cv2.triangulatePoints per pair (points only, two-view, no outlier rejection): {host:.1f} ms for "
              f"{len(pairs)} pairs")
    else:
        print("  cv2 not importable: no host comparison")
    print(json.dumps({"gpu": gpu, "images": V, "pairs": len(pairs), "call_ms": med, "kernel_ms": kern[0],
                      "kernel_launches": kern[1], "valid_points": float(vp.sum() / cp.sum()),
                      "valid_lines": float(vl.sum() / cl.sum()), "median_rel_error_points": float(np.median(err_p[vp])),
                      "median_rel_error_lines": float(np.median(err_l[vl])), "cv2_ms_all_pairs": host}))


if __name__ == "__main__":
    main()
