"""Tracks of a posed image set: `triangulate_tracks` (`ltr_tracks`) against `triangulate` on the same scene.

    python tools/tracks_bench.py [--images 64] [--neighbours 4] [--points 2000] [--lines 300] [--outliers 0.3]
                                 [--reps 20]

Data: the scene and pair ring of tools/triangulation_bench.py (`synthetic.make_line_map_set`, 0.5 px of noise,
--outliers of the observations moved 10 to 60 px, each image paired with its --neighbours next images, ground-truth
matches).  Device times are CUDA-event medians of --reps calls after a warm-up (the whole call: host checks, the pairs'
fundamental matrices, one pinned copy, the kernels), and the kernel time from ltr_profile_*.  Accuracy is per row,
against the true 3D points and each view's true segment end points, over the unmoved rows with a valid estimate, as
error / distance to the row's camera.  Prints the GPU model and power limit read in the same run, then one JSON line.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from linetr_b200 import _native as N, synthetic as syn, tracks as TR, triangulation as T   # noqa: E402
from triangulation_bench import gpu_info, ring_matches, time_cuda   # noqa: E402


def accuracy(d, X, E, cp, cl):
    """Median error / camera distance of valid unmoved rows: (points, line end points, valid point rows, valid line
    rows)."""
    V = len(d["keypoints"])
    n, m = len(d["points3d"]), len(d["segments3d"])
    X, E = X.reshape(V, n, 3), E.reshape(V, m, 2, 3)
    centres = np.einsum("vji,vj->vi", -d["R"], d["t"])
    err_p = np.linalg.norm(X - d["points3d"][None], axis=-1) / np.linalg.norm(d["points3d"][None] - centres[:, None],
                                                                              axis=-1)
    err_l = (np.linalg.norm(E - d["lines3d"], axis=-1) /
             np.linalg.norm(d["lines3d"] - centres[:, None, None], axis=-1)).max(-1)
    vp, vl = np.isfinite(X).all(-1), np.isfinite(E).all((-1, -2))
    return (float(np.median(err_p[vp & cp])), float(np.median(err_l[vl & cl])), vp, vl)


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
        raise SystemExit("tracks_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    V = args.images
    d = syn.make_line_map_set(0, V, args.points, args.lines, jitter_px=0.5, outlier_frac=args.outliers)
    pairs = np.array([(i, (i + k) % V) for i in range(V) for k in range(1, args.neighbours + 1)], dtype=np.int32)
    res = ring_matches(d, pairs, dev)
    cam = (d["keypoints"], d["klines"], pairs, res, d["K"], d["R"], d["t"])
    call = lambda: TR.triangulate_tracks(*cam)
    med, lo, hi = time_cuda(call, args.reps)
    tri_med, _, _ = time_cuda(lambda: T.triangulate(*cam), args.reps)
    N.profile_begin()
    r = call()
    prof = N.profile_end()
    kern = prof.get("tracks", (float("nan"), 0))
    N.profile_begin()
    tri = T.triangulate(*cam)
    tri_kern = N.profile_end().get("triangulate", (float("nan"), 0))
    ntp, ntl = r.n_tracks()
    status = {k: np.bincount(getattr(r, f"status_{k}")[:n].cpu().numpy(), minlength=4).tolist()
              for k, n in (("p", ntp), ("l", ntl))}
    op, ol = d["outlier_p"].reshape(-1), d["outlier_l"].reshape(-1)
    track_p, inl_p = r.track_p.cpu().numpy(), r.inlier_p.cpu().numpy().astype(bool)
    track_l, inl_l = r.track_l.cpu().numpy(), r.inlier_l.cpu().numpy().astype(bool)
    rows = r.rows()
    cp, cl = ~d["outlier_p"], ~d["outlier_l"]
    ep, el, vp, vl = accuracy(d, rows.points3d.cpu().numpy(), rows.lines3d.cpu().numpy(), cp, cl)
    tp, tl, tvp, tvl = accuracy(d, tri.points3d.cpu().numpy(), tri.lines3d.cpu().numpy(), cp, cl)
    moved = {"joined_p": float((track_p >= 0)[op].mean()), "inlier_p": float(inl_p[op].mean()),
             "valid_p": float(vp.reshape(-1)[op].mean()), "joined_l": float((track_l >= 0)[ol].mean()),
             "inlier_l": float(inl_l[ol].mean()), "valid_l": float(vl.reshape(-1)[ol].mean())}
    tri_moved = {"valid_p": float(tvp.reshape(-1)[op].mean()), "valid_l": float(tvl.reshape(-1)[ol].mean())}
    gpu = gpu_info()
    print(f"{gpu}: {V} posed images, {len(pairs)} pairs ({2 * args.neighbours} per image), {args.points} keypoints and "
          f"{args.lines} key lines per image, {args.outliers:.0%} of the observations moved 10-60 px, 0.5 px noise")
    print(f"  triangulate_tracks call median {med:8.3f} ms (min {lo:.3f}, max {hi:.3f}); kernels {kern[0]:.3f} ms in "
          f"{kern[1]} launches; triangulate {tri_med:.3f} ms (kernels {tri_kern[0]:.3f} ms)")
    print(f"  tracks: {ntp} point tracks (ok, too long, no candidate, too few: {status['p']}), {ntl} line tracks "
          f"({status['l']})")
    print(f"  moved observations: points {moved['joined_p']:.4f} joined a track, {moved['inlier_p']:.4f} inliers, "
          f"{moved['valid_p']:.4f} valid (triangulate {tri_moved['valid_p']:.4f}); key lines {moved['joined_l']:.4f} "
          f"joined, {moved['inlier_l']:.4f} inliers, {moved['valid_l']:.4f} valid (triangulate {tri_moved['valid_l']:.4f})")
    print(f"  error / distance over valid unmoved rows: points {ep:.2e} (triangulate {tp:.2e}), line end points "
          f"{el:.2e} ({tl:.2e}); unmoved rows valid: points {vp[cp].mean():.4f} ({tvp[cp].mean():.4f}), lines "
          f"{vl[cl].mean():.4f} ({tvl[cl].mean():.4f})")
    print(json.dumps({"gpu": gpu, "images": V, "pairs": len(pairs), "call_ms": med, "kernel_ms": kern[0],
                      "kernel_launches": kern[1], "n_tracks_p": ntp, "n_tracks_l": ntl, "status_p": status["p"],
                      "status_l": status["l"], "moved": moved, "median_rel_error_points": ep,
                      "median_rel_error_lines": el, "valid_unmoved_points": float(vp[cp].mean()),
                      "valid_unmoved_lines": float(vl[cl].mean()),
                      "triangulate": {"call_ms": tri_med, "kernel_ms": tri_kern[0], "moved": tri_moved,
                                      "median_rel_error_points": tp, "median_rel_error_lines": tl,
                                      "valid_unmoved_points": float(tvp[cp].mean()),
                                      "valid_unmoved_lines": float(tvl[cl].mean())}}))


if __name__ == "__main__":
    main()
