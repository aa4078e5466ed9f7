"""Signature attention on its own at bench.py cfg1's shape (128 images x 128 lines, 4 heads of 64): CUDA events around
back-to-back launches on a staged qkv image, sig_attention_pipe_kernel (LTR_ATTN_PIPE=1) against sig_attention_tc_kernel
(LTR_ATTN_PIPE=0) in the same process, alternated (run on the GPU box).

Per arm: us per layer (one launch), against two floors of one layer:
  tensor: the MMAs issued, 3 split products for S (128 x 128 x 64) and for PV (128 x 64 x 128) per image and head,
          at the dense BF16 data-sheet rate of the H100 SXM (989 TFLOP/s);
  bytes:  the qkv image read once (hi + lo, 768 columns) and the output written once (hi + lo, 256 columns), at the
          HBM3 data-sheet rate (3.35 TB/s) - an upper bound on that floor, since the qkv image the previous kernel just
          wrote can still be in L2.
Both arms must give the same bits."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from linetr_b200 import _native as N  # noqa: E402

PEAK_TFLOPS = 989.0
PEAK_GBS = 3350.0


def gpu_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                      text=True, timeout=30)
        return out.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001 - informational only
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=128, help="128-line images (128 = bench.py cfg1)")
    ap.add_argument("--layers", type=int, default=7 * 20, help="timed launches per run (7 signature layers x 20 steps)")
    ap.add_argument("--repeats", type=int, default=3, help="alternating runs of both arms")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sig_attention_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    lib = N.load()
    n = args.images
    g = torch.Generator(device=dev).manual_seed(0)
    # a qkv image of split-bf16 values: hi ~ N(0, 0.5), lo ~ 2^-9 of it (the layout does not change the work)
    hi = (0.5 * torch.randn(n * 128 * 768, generator=g, device=dev)).to(torch.bfloat16)
    lo = (torch.randn(n * 128 * 768, generator=g, device=dev) * 2.0 ** -10).to(torch.bfloat16)
    outs = {p: torch.zeros(2, n * 128 * 512, dtype=torch.bfloat16, device=dev) for p in (0, 1)}
    stream = torch.cuda.current_stream().cuda_stream

    def launch(pipe, k):
        os.environ["LTR_ATTN_PIPE"] = str(pipe)
        o = outs[pipe]
        N.check(lib.ltr_debug_sig_attention(hi.data_ptr(), lo.data_ptr(), o[0].data_ptr(), o[1].data_ptr(), n, k, stream),
                "ltr_debug_sig_attention")

    flop = n * 4 * 3 * 2 * (128 * 128 * 64 + 128 * 64 * 128)
    nbytes = n * 128 * (768 + 256) * 2 * 2
    floor_t, floor_b = flop / (PEAK_TFLOPS * 1e12) * 1e6, nbytes / (PEAK_GBS * 1e9) * 1e6
    print(f"# {gpu_info()}")
    print(f"# {n} images x 128 lines; per layer {flop / 1e9:.2f} GFLOP issued (tensor floor {floor_t:.1f} us), "
          f"{nbytes / 1e6:.1f} MB (HBM floor {floor_b:.1f} us)")
    for p in (0, 1):
        launch(p, 20)
    torch.cuda.synchronize()
    same = torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    res = {0: [], 1: []}
    for _ in range(args.repeats):
        for p in (0, 1):
            launch(p, 5)
            e0.record()
            launch(p, args.layers)
            e1.record()
            e1.synchronize()
            res[p].append(e0.elapsed_time(e1) * 1e3 / args.layers)
    os.environ.pop("LTR_ATTN_PIPE", None)
    names = {0: "sig_attention_tc_kernel", 1: "sig_attention_pipe_kernel"}
    summary = {}
    for p in (0, 1):
        us = sorted(res[p])
        med = us[len(us) // 2]
        summary[names[p]] = dict(us_per_layer=[round(x, 2) for x in res[p]], median_us=round(med, 2),
                                 x_tensor_floor=round(med / floor_t, 2), x_hbm_floor=round(med / floor_b, 2))
        print(f"{names[p]:>26s}: us/layer {' '.join(f'{x:6.2f}' for x in res[p])}  median {med:6.2f}  "
              f"= {med / floor_t:4.1f}x tensor floor, {med / floor_b:4.2f}x HBM floor")
    print(f"# outputs bit-identical: {same}")
    print(json.dumps(dict(gpu=gpu_info(), images=n, layers=args.layers, floors_us=dict(tensor=round(floor_t, 2), hbm=round(floor_b, 2)),
                          arms=summary, bit_identical=same)))
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
