"""Homography image pairs: `ltr_warp_pairs` (warped grey image + eroded valid mask) against the builder's per-pair
cv2 calls.

    python tools/homography_pairs_bench.py [--images 64] [--pairs 256 1024] [--launches 50] [--windows 5]

Data: --images seeded synthetic 640 x 480 colour images and their grey images, and for every --pairs count that many
homographies sampled with the reference's default parameters, the sources cycling through the images (so several
homographies share a source, as the builder's n_iters loop does).  Kernel time: CUDA events around --launches
back-to-back launches of the native entry on pre-staged inputs, after a warm-up; the median of --windows windows.  Call
time: the whole `warp_pairs` call (host inversion, one pinned copy, the launch) timed the same way.  Bytes per pair are
what the contract needs: the colour and grey source read once (h*w*(C+1)) and the grey image and mask written
(2*h*w); bytes/s is that over the kernel time, beside HBM3's 3.35 TB/s.  When cv2 is importable, the reference's
per-pair host work (cv2.warpPerspective of the grey and of the float32 colour image, the == 0 mask and cv2.erode 5 x 5)
is timed on --host-pairs pairs.  Prints the GPU model and power limit, then one JSON line.
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
from linetr_b200 import _ops, synthetic as syn   # noqa: E402
from linetr_b200._ops import stage   # noqa: E402
from linetr_b200.homography_pairs import sample_homographies, warp_pairs   # noqa: E402

W, H = 640, 480
HBM_TBPS = 3.35


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:   # pragma: no cover
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"


def time_windows(fn, launches, windows):
    """Median (and min, max) ms per call over `windows` event-timed windows of `launches` calls, after a warm-up."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(windows):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(launches):
            fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) / launches)
    return float(np.median(ts)), float(np.min(ts)), float(np.max(ts))


def host_reference(gray, colour, Hs, src):
    import cv2
    kernel = np.ones((5, 5), np.uint8)
    colour_f = colour.astype(np.float32)
    t0 = time.perf_counter()
    for Hp, s in zip(Hs, src):
        cv2.warpPerspective(gray[s], Hp, (W, H))
        wc = cv2.warpPerspective(colour_f[s], Hp, (W, H))
        m = np.ones((H, W), np.uint8)
        m[(wc == 0).all(-1)] = 0
        cv2.erode(m, kernel)
    return (time.perf_counter() - t0) / len(Hs) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--pairs", type=int, nargs="+", default=[256, 1024])
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--host-pairs", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("homography_pairs_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    gray, colour = syn.make_warp_images(0, args.images, H, W)
    g, c = (torch.from_numpy(a).to(dev) for a in (gray, colour))
    C = colour.shape[-1]
    bytes_per_pair = H * W * (C + 1) + 2 * H * W
    rng = np.random.default_rng(0)
    gpu = gpu_info()
    rows = []
    for P in args.pairs:
        Hs, _ = sample_homographies(P, (H, W), rng)
        src = np.arange(P, dtype=np.int32) % args.images
        dv = stage({"src_index": src, "inv_maps": np.linalg.inv(Hs).reshape(P, 9)}, dev)
        warped = torch.empty((P, H, W), dtype=torch.uint8, device=dev)
        mask = torch.empty_like(warped)
        kern = time_windows(lambda: _ops.warp_pairs(g, c, src, dv["src_index"], dv["inv_maps"], warped, mask),
                            args.launches, args.windows)
        call = time_windows(lambda: warp_pairs(g, c, src, Hs), args.launches, args.windows)
        tbps = bytes_per_pair * P / (kern[0] * 1e-3) / 1e12
        rows.append({"pairs": P, "kernel_ms": kern[0], "kernel_ms_min": kern[1], "kernel_ms_max": kern[2],
                     "call_ms": call[0], "pairs_per_s": P / (kern[0] * 1e-3), "tb_per_s": tbps,
                     "hbm_fraction": tbps / HBM_TBPS})
    host = None
    try:
        import cv2  # noqa: F401
        k = min(args.host_pairs, args.pairs[0])
        Hs, _ = sample_homographies(k, (H, W), np.random.default_rng(1))
        host = host_reference(gray, colour, Hs, np.arange(k) % args.images)
    except ImportError:
        pass
    print(f"{gpu}: {W} x {H}, {args.images} source images (colour C = {C}), {bytes_per_pair / 1e6:.2f} MB per pair")
    for r in rows:
        print(f"  {r['pairs']:5d} pairs: kernel {r['kernel_ms']:.3f} ms (min {r['kernel_ms_min']:.3f}, max "
              f"{r['kernel_ms_max']:.3f}), call {r['call_ms']:.3f} ms; {r['pairs_per_s']:,.0f} pairs/s, "
              f"{r['tb_per_s']:.2f} TB/s = {r['hbm_fraction']:.0%} of {HBM_TBPS} TB/s")
    if host is not None:
        print(f"  host cv2 (warp grey + warp float32 colour + mask + erode): {host:.2f} ms/pair -> "
              f"{1e3 / host:.0f} pairs/s on the host CPU")
    else:
        print("  cv2 not importable: no host comparison")
    print(json.dumps({"gpu": gpu, "width": W, "height": H, "images": args.images, "bytes_per_pair": bytes_per_pair,
                      "runs": rows, "cv2_ms_per_pair": host}))


if __name__ == "__main__":
    main()
