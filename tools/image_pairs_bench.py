"""Image-pair matching, two ways, on seeded synthetic pairs (P 640x480 pairs, ~150 key lines and ~1000 keypoints
per image; side 1 a jittered copy of side 0):

  (a) per image / per pair: `LineTransformer.preprocess` per image (GPU tokeniser, one call each), the tokenised
      dicts batched with `LineBatch.from_images`, `PairEngine.match_pairs` for the lines and `nn_matcher` per pair
      for the points - what a user of the batched engine had to do before `match_images`;
  (b) `PairEngine.match_images`: one batched tokeniser call, one encode + line match, one point match.

Times are CUDA-event times of whole calls (host preparation included) after warm-up, each ending in a device
synchronise.  Both paths must produce equal line and point matches.  Prints one JSON line with the GPU's name
and power limit.

    python tools/image_pairs_bench.py [--pairs 64] [--iters 10] [--warmup 3]
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

from linetr_b200 import LineBatch, LineTransformer, PairEngine, _native as N, synthetic as syn  # noqa: E402
from linetr_b200.nn_matcher import nn_matcher  # noqa: E402
from linetr_b200.match_io import dense_to_indices  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def per_image_path(model, eng, dev, pairs):
    sides = []
    for s in (0, 1):
        dicts = []
        for pr in pairs:
            im = pr[s]
            shape = im["image_shape"]
            model.config["min_length"] = max(16, max(shape) / 40)        # models/matching.py:29-32
            model.config["token_distance"] = max(8, max(shape) / 80)
            dicts.append(model.preprocess(im["klines"], shape, im, None))
        sides.append(LineBatch.from_images(dicts).to(dev))
    lines = eng.match_pairs(sides[0], sides[1], model.config["nn_threshold"])
    points = [nn_matcher(a["descriptors"].cpu().numpy(), b["descriptors"].cpu().numpy(), 0.7, True)[0] for a, b in pairs]
    torch.cuda.synchronize()
    return lines, points


def batched_path(eng, pairs):
    res = eng.match_images([a for a, _ in pairs], [b for _, b in pairs])
    torch.cuda.synchronize()
    return res


def timed(fn, iters):
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return ts


def launches(fn):
    torch.cuda.synchronize()
    N.reset_launch_count()
    fn()
    torch.cuda.synchronize()
    return N.launch_count()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--lines", type=int, default=150)
    ap.add_argument("--points", type=int, default=1000)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("image_pairs_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    model = LineTransformer({"mode": "train", "nn_threshold": 0.8})
    model.load_state_dict({k: torch.from_numpy(v) for k, v in syn.make_state_dict(0, 1).items()})
    model = model.eval().to(dev)
    eng = PairEngine(model, dev)
    pairs = [tuple(syn.image_to(im, dev) for im in syn.make_image_pair(5000 + p, args.lines, args.points))
             for p in range(args.pairs)]

    for _ in range(args.warmup):
        per_image_path(model, eng, dev, pairs)
        batched_path(eng, pairs)
    lines_a, points_a = per_image_path(model, eng, dev, pairs)
    res = batched_path(eng, pairs)
    equal_l = all(np.array_equal(lines_a.pair(p).cpu().numpy(), res.pair_lines(p).cpu().numpy()) for p in range(args.pairs))
    equal_p = all(np.array_equal(dense_to_indices(points_a[p]), res.pair_points(p).cpu().numpy()) for p in range(args.pairs))

    ta, tb = [], []
    for _ in range(2):    # alternate the two paths: drift of the shared host hits both
        ta += timed(lambda: per_image_path(model, eng, dev, pairs), args.iters // 2 or 1)
        tb += timed(lambda: batched_path(eng, pairs), args.iters // 2 or 1)
    name, power = gpu_info()
    ma, mb = float(np.median(ta)), float(np.median(tb))
    out = {
        "workload": f"{args.pairs} synthetic 640x480 pairs, {args.lines} key lines and {args.points} keypoints per image",
        "gpu": name, "power_limit": power,
        "per_image_ms": {"median": ma, "min": float(np.min(ta)), "max": float(np.max(ta))},
        "match_images_ms": {"median": mb, "min": float(np.min(tb)), "max": float(np.max(tb))},
        "speedup_median": ma / mb,
        "launches_per_image_path": launches(lambda: per_image_path(model, eng, dev, pairs)),
        "launches_match_images": launches(lambda: batched_path(eng, pairs)),
        "equal_line_matches": bool(equal_l), "equal_point_matches": bool(equal_p),
        "line_matches": int(res.counts_l.sum()), "point_matches": int(res.counts_p.sum()),
    }
    print(json.dumps(out))
    if not (equal_l and equal_p):
        raise SystemExit("the two paths disagree")


if __name__ == "__main__":
    main()
