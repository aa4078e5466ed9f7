"""How much of the tensor-core matcher's work goes to the exact fp32 re-check, on bench.py's cfg1 descriptors.

  * flagged lines per pair, counted on the host from numpy fp32 distances of the encoded descriptors (side 0: top-2
    gap or distance to the 0.8 threshold below MATCH_EPS; side 1: top-2 gap of the column below MATCH_EPS).  The GPU
    flags from its own tensor-core values, so its counts differ slightly; these explain the re-check's load;
  * CUDA-event times per call of the matcher's kernel classes (`_native.profile_begin/end`) for `ltr_match` on those
    descriptors (64 pairs x 128 x 128, rows layout, mutual);
  * the same on a stress case where every line of both sides is flagged: 1024 x 1024 lines made of duplicated and
    1-ulp-nudged copies.

Prints one JSON line with the GPU's name and power limit.

    python tools/match_exact_bench.py [--iters 50] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import load_weights, make_pairs  # noqa: E402
from linetr_b200 import LineBatch, LineTransformer, PairEngine, _native as N, _ops  # noqa: E402

EPS, THR = 1e-4, 0.8
MATCHER = ("desc_tiles", "match_tc", "match_exact", "match_tail")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [x.strip() for x in out.split(",")]
    except (OSError, subprocess.SubprocessError, IndexError):
        return ["unknown"]


def flagged_counts(d0, d1, P, L):
    """-> (side-0 flags per pair, side-1 flags per pair) from fp32 distances 2 - 2 a b^T."""
    f0, f1 = [], []
    for p in range(P):
        a, b = d0[p * L:(p + 1) * L], d1[p * L:(p + 1) * L]
        dist = np.maximum(np.float32(2) - np.float32(2) * (a @ b.T), np.float32(0))
        r = np.sort(dist, axis=1)
        c = np.sort(dist, axis=0)
        f0.append(int(((r[:, 1] - r[:, 0] < EPS) | (np.abs(r[:, 0] - THR) < EPS)).sum()))
        f1.append(int((c[1] - c[0] < EPS).sum()))
    return f0, f1


def time_classes(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    N.profile_begin()
    for _ in range(iters):
        fn()
    prof = N.profile_end()
    return {k: round(prof[k][0] / iters * 1e3, 2) for k in MATCHER if k in prof}   # us per call


def stress_descriptors(n, seed):
    """n lines per side, every line with exact ties or 1-ulp near-ties among its candidates on the other side."""
    rng = np.random.default_rng(seed)
    unit = lambda x: (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)
    base = unit(rng.standard_normal((n // 4, 256)))
    noisy = unit(base + 0.1 * rng.standard_normal(base.shape))

    def copies(x):
        out = x[np.arange(n) % len(x)].copy()
        for i in range(len(x), n, 2):
            k = rng.integers(0, 256, 3)
            out[i, k] = np.nextafter(out[i, k], np.float32(1))
        return out
    return copies(noisy), copies(base)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "match_exact_bench.py needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.set_grad_enabled(False)

    P, L = 64, 128
    sd, wnote = load_weights()
    model = LineTransformer({"mode": "train", "max_tokens": 21})
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    eng = PairEngine(model.eval().to(dev), dev)
    pairs = make_pairs("cfg1", 10_000, P)
    batch = LineBatch.from_images([a for a, _ in pairs] + [b for _, b in pairs]).to(dev)
    res = eng.match_packed(batch, P, THR, keep_desc=True)
    d0, d1 = res.desc0.contiguous(), res.desc1.contiguous()
    f0, f1 = flagged_counts(d0.cpu().numpy(), d1.cpu().numpy(), P, L)
    cfg1 = lambda: _ops.match_descriptors(d0, d1, N.LAYOUT_ROWS, P, THR, True, n0=L, n1=L, want_dist=False)

    s0, s1 = stress_descriptors(1024, 3)
    s0, s1 = torch.from_numpy(s0).to(dev), torch.from_numpy(s1).to(dev)
    stress = lambda: _ops.match_descriptors(s0, s1, N.LAYOUT_ROWS, 1, THR, True, n0=1024, n1=1024, want_dist=False)

    out = {
        "gpu": gpu_info(), "weights": wnote,
        "cfg1_flagged_per_pair": {"side0_mean": float(np.mean(f0)), "side0_range": [min(f0), max(f0)],
                                  "side1_mean": float(np.mean(f1)), "side1_range": [min(f1), max(f1)]},
        "cfg1_us_per_call": time_classes(cfg1, args.iters, args.warmup),
        "stress_1024_us_per_call": time_classes(stress, args.iters, args.warmup),
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
