"""The validation step's loss and metrics on the GPU: `validation_metrics` over a validation set.

    python tools/triplet_bench.py [--batches 100] [--pairs 32] [--lines 250] [--reps 10]

A validation set of --batches batches of --pairs pairs of --lines sublines, shaped like train.py's: unit descriptors
channel-first [P, 256, n], side 1 a permuted copy of side 0 with per-line noise, and the [P, n+1, n+1] 0/1
mat_assign_sublines from lmatches (about half of the lines matched), read in place.  It is timed as one grouped
`validation_metrics` call (one group per batch) and as one call per batch.  Call times are CUDA-event medians over
--reps repetitions after a warm-up; per-class kernel times come from `ltr_profile_*` in a separate pass.  Prints the GPU
model and power limit with the numbers, then one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from linetr_b200 import _native as N, eval_criteria as EC   # noqa: E402


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:   # pragma: no cover
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"


def make_set(P, n, dev, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(P, 256, n, device=dev, generator=g)
    x = x / x.norm(dim=1, keepdim=True)
    perm = torch.stack([torch.randperm(n, device=dev, generator=g) for _ in range(P)])
    sigma = 0.02 + 0.33 * torch.rand(P, 1, n, device=dev, generator=g)
    y = torch.gather(x, 2, perm[:, None, :].expand(P, 256, n)) + sigma * torch.randn(P, 256, n, device=dev, generator=g)
    y = y / y.norm(dim=1, keepdim=True)
    assign = torch.zeros(P, n + 1, n + 1, device=dev)
    matched = torch.rand(P, n, device=dev, generator=g) < 0.5
    p_idx, j = torch.nonzero(matched, as_tuple=True)
    assign[p_idx, perm[p_idx, j], j] = 1   # side-1 line j is side-0 line perm[j]
    return x.contiguous(), y.contiguous(), assign


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
    ap.add_argument("--batches", type=int, default=100)
    ap.add_argument("--pairs", type=int, default=32)
    ap.add_argument("--lines", type=int, default=250)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("triplet_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    B, Pb, n = args.batches, args.pairs, args.lines
    P = B * Pb
    x, y, assign = make_set(P, n, dev)
    groups = np.arange(B + 1, dtype=np.int32) * Pb
    kw = dict(layout=N.LAYOUT_CHANNEL_FIRST, match_thr=EC.MATCH_THR_F32)

    def grouped():
        return EC.validation_metrics(x, y, assign, groups=groups, **kw)

    def per_batch():
        return [EC.validation_metrics(x[b * Pb:(b + 1) * Pb], y[b * Pb:(b + 1) * Pb], assign[b * Pb:(b + 1) * Pb], **kw)
                for b in range(B)]

    res = {"grouped_ms": time_cuda(grouped, args.reps), "per_batch_ms": time_cuda(per_batch, args.reps)}
    one, many = grouped(), per_batch()
    for b, r in enumerate(many):   # one call per batch gives the grouped call's bits
        for k in ("loss", "hardest_pos", "hardest_neg", "n_valid"):
            assert getattr(r, k)[0].view(torch.int32) == getattr(one, k)[b].view(torch.int32), (b, k)
    torch.cuda.synchronize()
    N.profile_begin()
    grouped()
    prof = N.profile_end()
    nv = one.n_valid.cpu().numpy()
    pr = one.precision_recall()
    gpu = gpu_info()
    print(f"{gpu}: {B} batches x {Pb} pairs x {n} sublines = {P * 2 * n} anchors")
    for k, (med, lo, hi) in res.items():
        print(f"  {k:14s} median {med:8.3f} ms  (min {lo:.3f}, max {hi:.3f})  = {med / B * 1e3:.1f} us/batch")
    for k, (ms, cnt) in sorted(prof.items()):
        print(f"  kernel {k:12s} {ms:8.3f} ms in {cnt} launches")
    print(f"  valid anchors per batch: mean {nv.mean():.0f} of {Pb * 2 * n}; mean loss {float(one.loss.mean()):.4f}; "
          f"mean precision {pr[0].mean():.2f} recall {pr[1].mean():.2f}")
    print(json.dumps({"gpu": gpu, "batches": B, "pairs_per_batch": Pb, "lines": n,
                      **{k: v[0] for k, v in res.items()}, "kernels_ms": {k: v[0] for k, v in prof.items()},
                      "valid_anchors_per_batch": float(nv.mean())}))


if __name__ == "__main__":
    main()
