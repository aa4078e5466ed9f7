"""One signature layer's row-local GEMMs (mlp1 ReLU -> mlp2 + x -> qkv) as one chained launch against three launches
of gemm_img_kernel, at the row counts of bench.py cfg1 (64 pairs x 2 x 128 lines) and cfg2 (x 256 lines) and a few
batch sizes around the chaining threshold (run on the GPU box).

Per arm: `ms/layer` = CUDA events around back-to-back layers (the profiler off), `linear ms/layer` = the sum of the
per-launch CUDA events of the library's profiler (kernel class `linear`, the figure bench.py's kernel_time_shares are
built from) per layer, and useful TFLOP/s = 2 M (512*512 + 256*512 + 768*256) over each."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from linetr_b200 import _native as N  # noqa: E402

FLOP_PER_ROW = 2 * (512 * 512 + 256 * 512 + 768 * 256)
WARM = 3   # untimed layers ltr_gemm_chain_bench runs first (the profiler sees them too)


def gpu_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                      text=True, timeout=30)
        return out.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001 - informational only
        return f"unknown ({e})"


def arm(lib, rows, chained, iters):
    ms = lib.ltr_gemm_chain_bench(rows, chained, iters, 0)
    N.profile_begin()
    ms_prof = lib.ltr_gemm_chain_bench(rows, chained, iters, 0)
    prof = N.profile_end()
    if ms < 0 or ms_prof < 0:
        raise N.LtrError(f"ltr_gemm_chain_bench failed at {rows} rows (chained={chained})")
    lin_ms, launches = prof["linear"]
    layers = iters + WARM
    lin = lin_ms / layers
    return dict(ms_per_layer=round(ms, 5), linear_ms_per_layer=round(lin, 5), launches_per_layer=launches / layers,
                tflops_useful=round(FLOP_PER_ROW * rows / ms / 1e9, 1),
                tflops_useful_linear=round(FLOP_PER_ROW * rows / lin / 1e9, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=3, help="alternating runs of both arms per row count")
    ap.add_argument("--tiles", type=int, nargs="*", default=[64, 88, 96, 112, 128, 256],
                    help="128-row tiles per batch (128 = cfg1, 256 = cfg2)")
    args = ap.parse_args()
    lib = N.load()
    print(f"# {gpu_info()}")
    print(f"{'tiles':>5s} {'rows':>6s} {'arm':>8s} {'ms/layer':>9s} {'linear ms':>10s} {'launches':>8s} {'TFLOP/s':>8s} {'TFLOP/s lin':>11s}")
    results = []
    for t in args.tiles:
        rows = 128 * t
        for rep in range(args.repeats):
            for chained in (0, 1):
                r = arm(lib, rows, chained, args.iters)
                r.update(tiles=t, rows=rows, chained=chained, rep=rep)
                results.append(r)
                print(f"{t:5d} {rows:6d} {'chain' if chained else '3 launch':>8s} {r['ms_per_layer']:9.4f} "
                      f"{r['linear_ms_per_layer']:10.4f} {r['launches_per_layer']:8.1f} {r['tflops_useful']:8.1f} "
                      f"{r['tflops_useful_linear']:11.1f}", flush=True)
    print(json.dumps({"gpu": gpu_info(), "results": results}))


if __name__ == "__main__":
    main()
