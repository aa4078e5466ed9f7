"""k-block timeline of gemm_chain_kernel's CTA 0 on one signature layer (mlp1 ReLU -> mlp2 + x -> qkv) at cfg1's
row count (128 m-tiles, so CTA 0 owns one m-tile: 6 tiles, 36 k-blocks), from the clock64 stamps the kernel leaves
when ltr_debug_trace_arm is on (slot layout: CHAIN_TRACE_* in csrc/gemm_img.cuh).  Run on the GPU box.

Per k-block, in microseconds at the card's max SM clock (read from nvidia-smi in the same run) or --mhz:
  issue   producer has issued the k-block's loads (its last empty-wait ended), from the consumers' start
  land    consumers see all of its operands landed (their last full-wait returned)
  i->l    land - issue: how long the k-block's operands took from request to use
  wait    land - (previous k-block's MMAs done, or the previous tile's epilogue end): time the consumers spent
          waiting on `full`
  mma     MMAs done - land: issue to wgmma.wait_group 0
Per tile: the epilogue time (epilogue done - last k-block's MMAs done).  The stamps are those of the last of a few
back-to-back layer launches (steady state); only the consumers' first thread and the producer thread stamp.
The summary gives the median k-block period inside a tile (MMAs done to MMAs done) in SM cycles, which does not
depend on the clock, next to the tensor pipe's bound: a k-block is 128 x 256 x 64 x 3 split products = 12.6 MFLOP,
and an H100 SM does 4096 dense bf16 FLOP per cycle (989.4 TFLOP/s over 132 SMs at 1830 MHz), so 3072 cycles."""
import argparse
import ctypes as C
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from linetr_b200 import _native as N  # noqa: E402

TRACE_KB = 36                      # CHAIN_TRACE_KB
EPI = 3 * TRACE_KB                 # CHAIN_TRACE_EPI
T0 = EPI + 4 * 4                   # CHAIN_TRACE_T0
TILES = [("mlp1", 0, 2, 8), ("mlp2", 1, 1, 8), ("qkv", 2, 3, 4)]   # (name, op, n-blocks, k-blocks per tile)
MMA_BOUND_CYCLES = 128 * 256 * 64 * 2 * 3 // 4096


def sm_clock_mhz():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                                       "--format=csv,noheader"], text=True, timeout=30).strip().splitlines()[0]
        return out, float(out.split(",")[-1].split()[0])
    except Exception as e:  # noqa: BLE001 - informational only
        return f"unknown ({e})", None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tiles", type=int, default=128, help="128-row m-tiles (128 = cfg1)")
    ap.add_argument("--mhz", type=float, default=None, help="SM clock for cycles -> us (default: max SM clock)")
    args = ap.parse_args()
    lib = N.load()
    info, mhz = sm_clock_mhz()
    mhz = args.mhz or mhz or 1980.0
    print(f"# {info}; cycles -> us at {mhz:.0f} MHz")
    rows = 128 * args.tiles
    if lib.ltr_gemm_chain_bench(rows, 1, 5, 0) < 0:   # warm
        raise N.LtrError("ltr_gemm_chain_bench failed")
    lib.ltr_debug_trace_arm(1)
    ms = lib.ltr_gemm_chain_bench(rows, 1, 1, 0)
    buf = (C.c_uint64 * 128)()
    rc = lib.ltr_debug_trace_read(buf)
    lib.ltr_debug_trace_arm(0)
    if ms < 0 or rc != 0:
        raise N.LtrError("chain trace failed")
    t = [int(v) for v in buf]
    c0 = t[T0 + 1]
    us = lambda cyc: (cyc - c0) / mhz   # noqa: E731

    print(f"{'kb':>3s} {'op':>5s} {'nb':>2s} {'k':>2s} {'issue':>8s} {'land':>8s} {'i->l':>6s} {'wait':>6s} {'mma':>6s}")
    it, prev_done = 0, c0
    sums = dict(il=0.0, wait=0.0, mma=0.0, epi=0.0, n=0)
    periods = []
    for name, o, nbl, nk in TILES:
        for nb in range(nbl):
            for k in range(nk):
                iss, land, done = t[3 * it], t[3 * it + 1], t[3 * it + 2]
                if k > 0:
                    periods.append(done - prev_done)
                il, wait, mma = (land - iss) / mhz, (land - prev_done) / mhz, (done - land) / mhz
                print(f"{it:3d} {name:>5s} {nb:2d} {k:2d} {us(iss):8.2f} {us(land):8.2f} {il:6.2f} {wait:6.2f} {mma:6.2f}")
                sums["il"] += il; sums["wait"] += wait; sums["mma"] += mma; sums["n"] += 1
                prev_done = done
                it += 1
            epi_end = t[EPI + o * 4 + nb]
            epi = (epi_end - prev_done) / mhz
            sums["epi"] += epi
            print(f"    {name:>5s} {nb:2d} epilogue {epi:6.2f} us (ends at {us(epi_end):8.2f})")
            prev_done = epi_end
    n = sums["n"]
    total = (prev_done - c0) / mhz
    print(f"# {n} k-blocks, {total:.2f} us from consumer start to last epilogue end ({ms * 1e3:.1f} us per layer launch); "
          f"mean per k-block: issue->land {sums['il'] / n:.2f}, wait on full {sums['wait'] / n:.2f}, "
          f"MMA {sums['mma'] / n:.2f} us; epilogues {sums['epi']:.2f} us in all")
    periods.sort()
    print(f"# k-block period inside a tile: median {periods[len(periods) // 2]} cycles (min {periods[0]}, "
          f"max {periods[-1]}); tensor-pipe bound {MMA_BOUND_CYCLES} cycles")


if __name__ == "__main__":
    main()
