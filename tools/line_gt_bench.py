"""Homography ground truth for line matches: `ltr_line_gt` (dense and counts-only) against the numpy restatement.

    python tools/line_gt_bench.py [--pairs 1000] [--lines 250] [--reps 20] [--host-pairs 20]

1000 pairs of 250 x 250 segments (synthetic lines mapped by a homography plus noise, so there are many true
matches, plus distractors) with predictions.  Device times are CUDA-event medians over --reps launches after a
warm-up: the kernel alone (`ltr_line_gt` on staged inputs) and the whole `homography_ground_truth` call (host
checks, np.linalg.inv, one pinned copy).  The host number is `line_assignment` + `calc_tfpn` per pair, timed on
--host-pairs pairs.  Prints the GPU model and power limit with the numbers, then one JSON line.
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
from linetr_b200 import _ops, eval_homography as EH   # noqa: E402


def make_pairs(n_pairs, n, seed=0):
    rng = np.random.default_rng(seed)
    l0s, l1s, hs, preds = [], [], [], []
    for _ in range(n_pairs):
        h = np.eye(3)
        h[:2, :2] += rng.normal(0, 0.05, (2, 2))
        h[:2, 2] = rng.normal(0, 15, 2)
        h[2, :2] = rng.normal(0, 1e-4, 2)
        sp = rng.random((n, 2)) * [620, 460] + 10
        l0 = np.stack([sp, sp + rng.normal(0, 60, (n, 2))], 1).astype(np.float32)
        m = n * 3 // 4
        mapped = EH.project_lines(l0[:m], h) + rng.normal(0, 0.3, (m, 2, 2)).astype(np.float32)
        perm = rng.permutation(n)
        l1 = np.concatenate([mapped, (rng.random((n - m, 2, 2)) * [640, 480]).astype(np.float32)])[perm]
        inv = np.argsort(perm)
        pred = np.where(rng.random(n) < 0.8, np.concatenate([inv[:m], rng.integers(0, n, n - m)]), -1)
        l0s.append(l0); l1s.append(l1.astype(np.float32)); hs.append(h); preds.append(pred.astype(np.int32))
    return l0s, l1s, np.stack(hs), preds


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:   # pragma: no cover
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"


def time_cuda(fn, reps):
    dev = torch.device("cuda", 0)
    fn()
    torch.cuda.synchronize(dev)
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
    ap.add_argument("--pairs", type=int, default=1000)
    ap.add_argument("--lines", type=int, default=250)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-pairs", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("line_gt_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    P, n = args.pairs, args.lines
    l0s, l1s, hs, preds = make_pairs(P, n)
    cu = np.arange(P + 1, dtype=np.int32) * n
    s0 = torch.from_numpy(np.concatenate(l0s)).to(dev)
    s1 = torch.from_numpy(np.concatenate(l1s)).to(dev)
    pred = torch.from_numpy(np.concatenate(preds)).to(dev)
    i32 = dict(dtype=torch.int32, device=dev)
    cu_d = torch.from_numpy(cu).to(dev)
    h_d = torch.from_numpy(hs).to(dev)
    hi_d = torch.from_numpy(np.linalg.inv(hs)).to(dev)
    counts, tfpn = torch.zeros(P, **i32), torch.zeros((P, 4), **i32)
    assign = torch.zeros(P * n * n, dtype=torch.float32, device=dev)

    def kernel(dense):
        _ops.call_struct("ltr_line_gt",
                         dict(segs0=s0, segs1=s1, cu0=cu_d, cu1=cu_d, homography=h_d, homography_inv=hi_d, pred0=pred,
                              n_pairs=P, max_n0=n, max_n1=n, thres_reprojected=3.0, thres_angdiff=2.0,
                              min_overlap_ratio=0.3),
                         dict(assign=assign if dense else None, assign_stride=n * n, n_gt=counts, tfpn=tfpn))

    res = {}
    res["kernel_dense_ms"] = time_cuda(lambda: kernel(True), args.reps)
    dense_counts, dense_tfpn = counts.clone(), tfpn.clone()
    res["kernel_counts_ms"] = time_cuda(lambda: kernel(False), args.reps)
    assert torch.equal(counts, dense_counts) and torch.equal(tfpn, dense_tfpn), "counts-only differs from dense"
    res["call_dense_ms"] = time_cuda(lambda: EH.homography_ground_truth(s0, s1, cu, cu, hs, pred0=pred), args.reps)
    res["call_counts_ms"] = time_cuda(lambda: EH.homography_ground_truth(s0, s1, cu, cu, hs, pred0=pred,
                                                                         want_assign=False), args.reps)
    # host restatement on a subset, also a spot check of the device results
    k = min(args.host_pairs, P)
    t0 = time.perf_counter()
    host_tfpn = []
    for p in range(k):
        a, _ = EH.line_assignment(l0s[p], l1s[p], hs[p])
        score = np.zeros((n, n))
        r = np.nonzero(preds[p] >= 0)[0]
        score[r, preds[p][r]] = 1
        host_tfpn.append(EH.calc_tfpn(score, a))
        assert np.array_equal(assign[p * n * n:(p + 1) * n * n].view(n, n).cpu().numpy(), a.astype(np.float32)), p
    host_s = (time.perf_counter() - t0) / k
    assert [tuple(x) for x in tfpn[:k].cpu().numpy()] == host_tfpn
    gpu = gpu_info()
    print(f"{gpu}: {P} pairs of {n} x {n} segments, {int(counts.sum())} ground-truth matches")
    for key in ("kernel_dense_ms", "kernel_counts_ms", "call_dense_ms", "call_counts_ms"):
        med, lo, hi = res[key]
        print(f"  {key:18s} median {med:8.3f} ms  (min {lo:.3f}, max {hi:.3f})  = {med / P * 1e3:.2f} us/pair")
    print(f"  host numpy restatement: {host_s * 1e3:.1f} ms/pair (single thread, {k} pairs) "
          f"-> {host_s * P:.1f} s for {P} pairs")
    print(json.dumps({"gpu": gpu, "pairs": P, "lines": n, **{k: v[0] for k, v in res.items()},
                      "host_ms_per_pair": host_s * 1e3}))


if __name__ == "__main__":
    main()
