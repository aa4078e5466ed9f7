"""Global poses on one GPU: 128-image sets with ring +-5 (640 pairs) and exhaustive (8128 pairs) view graphs, relative
poses from `synthetic.make_relative_poses` with 0.5 deg noise and 20 % planted outlier pairs.  Prints one JSON line
per graph: the CUDA-event time of a `global_poses` call over --iters calls after warm-ups (median, min, max), the
numpy model's host time, the accuracy after a similarity alignment, the GPU's name and power limit, and (from a
separate torch.profiler run) the device time of each of the three kernels."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from linetr_b200 import synthetic as syn  # noqa: E402
from linetr_b200.global_poses import global_poses, global_poses_host  # noqa: E402


def align(R, C, Rt, Ct):
    U, _, Vt = np.linalg.svd(sum(Rt[k].T @ R[k] for k in range(len(R))))
    G = U @ Vt
    rdeg = [np.degrees(np.linalg.norm(Rt[k] @ G - R[k]) / np.sqrt(2)) for k in range(len(R))]
    A = Ct @ G
    am, cm = A.mean(0), C.mean(0)
    s = ((A - am) * (C - cm)).sum() / ((A - am) ** 2).sum()
    base = np.mean([np.linalg.norm(C[i] - C[j]) for i in range(len(C)) for j in range(i)])
    return float(np.median(rdeg)), float(np.median(np.linalg.norm(s * (A - am) + cm - C, axis=1)) / base)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    dev = torch.device("cuda", 0)
    n = 128
    d = syn.make_line_map_set(0, n, 8, 2, max_angle_deg=30)
    Ct = -np.einsum("nji,nj->ni", d["R"], d["t"])
    graphs = {"ring5": np.array([(i, (i + k) % n) for i in range(n) for k in range(1, 6)]),
              "exhaustive": np.array([(i, j) for i in range(n) for j in range(i + 1, n)])}
    for name, pairs in graphs.items():
        rp = syn.make_relative_poses(d["R"], d["t"], pairs, 0.5, 0.2, 1)
        dp = {k: torch.as_tensor(v).to(dev) for k, v in rp.items() if k != "outlier"}
        for _ in range(args.warmup):
            o = global_poses(pairs, dp, n)
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.iters):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            o = global_poses(pairs, dp, n)
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b))
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                global_poses(pairs, dp, n)
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA and "gp_" in ev.name:
                nm = ev.name.split("gp_")[1].split("_kernel")[0]
                kern[nm] = kern.get(nm, 0.0) + ev.device_time / 1000.0 / 5
        t0 = time.perf_counter()
        h = global_poses_host(pairs, rp, n)
        host_s = time.perf_counter() - t0
        same = all(np.array_equal(getattr(o, k).cpu().numpy(), h[k], equal_nan=True)
                   for k in ("R", "t", "edge_status", "support"))
        st = o.stats_dict()
        reg = o.registered.cpu().numpy()
        R, t = o.R.cpu().numpy()[reg], o.t.cpu().numpy()[reg]
        rerr, cerr = align(R, -np.einsum("nji,nj->ni", R, t), d["R"][reg], Ct[reg])
        status = o.edge_status.cpu().numpy()
        print(json.dumps(dict(graph=name, pairs=len(pairs), gpu=gpu, call_ms_median=float(np.median(ms)),
                              call_ms_min=float(min(ms)), call_ms_max=float(max(ms)), calls=args.iters,
                              kernel_ms=kern,
                              host_model_s=host_s, matches_model=bool(same), stats=st,
                              planted_flagged=bool((status[rp["outlier"]] == 2).all()),
                              clean_inliers=bool((status[~rp["outlier"]] == 4).all()),
                              median_rot_err_deg=rerr, median_centre_err_rel=cerr)))


if __name__ == "__main__":
    main()
