"""Photometric augmentation: `ltr_photometric` and `photometric_homography_pairs` against the host path.

    python tools/photometric_bench.py [--batches 64 256] [--launches 20] [--windows 5] [--host-images 4]

Data: seeded synthetic 640 x 480 grey and colour images, augmented with the homography yaml's parameters
(HOMOGRAPHY_PHOTOMETRIC; motion blur on for about half the images, the shade on for all).  Kernel time: CUDA events
around --launches back-to-back `ltr_photometric` calls on pre-staged parameters (four kernels and a memset each), after
a warm-up; the median of --windows windows.  Augment time: the whole `photometric_augment` call on a sampled record
(parameter staging, workspace, launches), timed the same way.  Pairs time: `photometric_homography_pairs` with one pair
per image, including the host sampling of homographies and photometric draws, ending in a device synchronise.  Host
path: per image, the numpy model of stage 1 (brightness, contrast, noise, motion blur) and cv2 for the shade
(cv2.ellipse x 20, cv2.GaussianBlur of the float32 mask, the float chain), as the builder runs it on the CPU.  Prints
the GPU model and power limit, then one JSON line.
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
from linetr_b200 import _native as N, _ops, synthetic as syn   # noqa: E402
from linetr_b200 import photometric as PH   # noqa: E402
from linetr_b200._ops import stage   # noqa: E402

W, H = 640, 480


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


def host_path(gray, rec):
    """ms per image of the builder's host path: the numpy model of stage 1, cv2 for the shade."""
    import cv2
    t0 = time.perf_counter()
    for i in range(len(gray)):
        v = PH._pointwise(gray[i], rec, i, rec["key"][i]).astype(np.uint8)
        a = cv2.filter2D(v, -1, rec["blur_kernel"][i]) if rec["blur"][i] else v
        mask = np.zeros((H, W), np.uint8)
        for ax, ay, x, y, ang in rec["ellipses"][i]:
            cv2.ellipse(mask, (int(x), int(y)), (int(ax), int(ay)), float(ang), 0, 360, 255, -1)
        k = int(rec["ksize"][i])
        m = cv2.GaussianBlur(mask.astype(np.float32), (k, k), 0)
        PH.shade_pre_truncation(a, m, rec["transparency"][i]).astype(np.uint8)
    return (time.perf_counter() - t0) / len(gray) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--host-images", type=int, default=4)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("photometric_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    gpu = gpu_info()
    rows = []
    for n in args.batches:
        gray, colour = syn.make_warp_images(n, n, H, W)
        g, c = (torch.from_numpy(a).to(dev) for a in (gray, colour))
        rec = PH.sample_photometric(n, (H, W), np.random.default_rng(n), **PH.HOMOGRAPHY_PHOTOMETRIC)
        ph = PH.params_array(rec)
        dv = stage({"params": ph, "ellipses": rec["ellipses"], "taps": rec["taps"]}, dev)
        out = torch.empty_like(g)
        ws = torch.empty(N.photometric_workspace_bytes(n, H, W), dtype=torch.uint8, device=dev)
        kern = time_windows(lambda: _ops.photometric(g, out, ph, dv["params"], dv["ellipses"], dv["taps"], ws),
                            args.launches, args.windows)
        call = time_windows(lambda: PH.photometric_augment(g, rec), args.launches, args.windows)
        rng = np.random.default_rng(0)
        PH.photometric_homography_pairs(g, c, 1, rng)
        torch.cuda.synchronize()
        ts = []
        for _ in range(args.windows):
            t0 = time.perf_counter()
            PH.photometric_homography_pairs(g, c, 1, rng)
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
        pairs = float(np.median(ts))
        rows.append({"images": n, "kernel_ms": kern[0], "kernel_ms_min": kern[1], "kernel_ms_max": kern[2],
                     "augment_ms": call[0], "pairs_ms": pairs, "kernel_images_per_s": n / (kern[0] * 1e-3),
                     "augment_images_per_s": n / (call[0] * 1e-3), "pairs_per_s": n / (pairs * 1e-3)})
    host = None
    try:
        import cv2  # noqa: F401
        k = args.host_images
        gray, _ = syn.make_warp_images(1, k, H, W)
        host = host_path(gray, PH.sample_photometric(k, (H, W), np.random.default_rng(1), **PH.HOMOGRAPHY_PHOTOMETRIC))
    except ImportError:
        pass
    print(f"{gpu}: {W} x {H}, the homography yaml's photometric parameters")
    for r in rows:
        print(f"  {r['images']:4d} images: kernels {r['kernel_ms']:.3f} ms (min {r['kernel_ms_min']:.3f}, max "
              f"{r['kernel_ms_max']:.3f}) = {r['kernel_images_per_s']:,.0f} images/s; photometric_augment "
              f"{r['augment_ms']:.3f} ms = {r['augment_images_per_s']:,.0f} images/s; photometric_homography_pairs "
              f"{r['pairs_ms']:.2f} ms = {r['pairs_per_s']:,.0f} pairs/s")
    if host is not None:
        print(f"  host path (numpy stage 1 + cv2 shade): {host:.2f} ms/image -> {1e3 / host:.0f} images/s")
    else:
        print("  cv2 not importable: no host comparison")
    print(json.dumps({"gpu": gpu, "width": W, "height": H, "runs": rows, "host_ms_per_image": host}))


if __name__ == "__main__":
    main()
