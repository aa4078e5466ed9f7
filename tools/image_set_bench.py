"""Exhaustive matching of an image set, four ways, on seeded synthetic views (`synthetic.make_image_set`: N 640x480
views of one scene, 150 key lines and 1000 keypoints per view, all N(N-1)/2 pairs):

  (a) `PairEngine.match_images` over the pair list: every image is tokenised and encoded once per pair it is in;
  (b) `PairEngine.encode_images` + `match_set`: every image encoded once, one indexed line and point match;
  (c) `match_set` alone on a set encoded beforehand;
  (d) the same encoded set, descriptors gathered per pair into packed copies, then the pair-batched `ltr_match`
      (what a caller can do without the indexed matcher; kept here as a comparison arm only).

Times are CUDA-event times of whole calls (host preparation included) after warm-up, each ending in a device
synchronise, the arms alternated so that drift hits all of them.  All arms must produce equal line and point matches
(exit status 1 otherwise).  Prints one JSON line with the GPU's name and power limit.

    python tools/image_set_bench.py [--views 32] [--iters 10] [--warmup 2]
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

from linetr_b200 import LineTransformer, PairEngine, _native as N, _ops, exhaustive_pairs, synthetic as syn  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def gathered_match(eng, s, pairs, line_thresh, point_thresh=0.7):
    """Arm (d): per-pair packed copies of the set's descriptors, then `ltr_match` (lines with key-line merging when an
    image splits a key line, as match_images does) and a channel-first `ltr_match` for the points."""
    dev = eng.device
    i0, i1 = pairs[:, 0], pairs[:, 1]
    cu, cuk, so, cup = (s.cu_lines.astype(np.int64), s.cuk.astype(np.int64), s.sub_off.astype(np.int64),
                        s.cu_points.astype(np.int64))
    pref = lambda c: np.concatenate([[0], np.cumsum(c)]).astype(np.int64)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(dev)
    out = []
    for idx in (i0, i1):
        rows = torch.cat([s.desc_l[cu[i]:cu[i + 1]] for i in idx])
        pts = torch.cat([s.desc_p[256 * cup[i]:256 * cup[i + 1]] for i in idx])
        gcu, gcuk, gcup = pref(np.diff(cu)[idx]), pref(np.diff(cuk)[idx]), pref(np.diff(cup)[idx])
        gso = np.concatenate([so[cuk[i]:cuk[i + 1]] - cu[i] + b for i, b in zip(idx, gcu[:-1])] + [gcu[-1:]])
        out.append((rows, pts, gcu, gcuk, gcup, gso))
    (r0, p0, cu0, ck0, cp0, so0), (r1, p1, cu1, ck1, cp1, so1) = out
    mx = lambda a: int(np.diff(a).max(initial=0))
    kw = dict(cu0=t(cu0), cu1=t(cu1), max_n0=mx(cu0), max_n1=mx(cu1), total_k0=int(ck0[-1]), total_k1=int(ck1[-1]))
    if (np.diff(cu0) != np.diff(ck0)).any() or (np.diff(cu1) != np.diff(ck1)).any():
        kw.update(sub_off0=t(so0), sub_off1=t(so1), cuk0=t(ck0), cuk1=t(ck1), max_k0=mx(ck0), max_k1=mx(ck1))
    lines = _ops.match_descriptors(r0, r1, N.LAYOUT_ROWS, len(pairs), float(line_thresh), True, want_dist=False, **kw)
    points = _ops.match_descriptors(p0, p1, N.LAYOUT_CHANNEL_FIRST, len(pairs), float(point_thresh), True, d=256,
                                    want_dist=False, cu0=t(cp0), cu1=t(cp1), max_n0=mx(cp0), max_n1=mx(cp1))
    return lines["matches0"], points["matches0"]


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
    ap.add_argument("--views", type=int, default=32)
    ap.add_argument("--lines", type=int, default=150)
    ap.add_argument("--points", type=int, default=1000)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("image_set_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    model = LineTransformer({"mode": "train", "nn_threshold": 0.8})
    model.load_state_dict({k: torch.from_numpy(v) for k, v in syn.make_state_dict(0, 1).items()})
    model = model.eval().to(dev)
    eng = PairEngine(model, dev)
    views = [syn.image_to(im, dev) for im in syn.make_image_set(6000, args.views, args.lines, args.points)]
    pairs = exhaustive_pairs(args.views)
    thr = model.config["nn_threshold"]
    pre = eng.encode_images(views)

    def arm_a():
        r = eng.match_images([views[i] for i, _ in pairs], [views[j] for _, j in pairs], line_thresh=thr)
        torch.cuda.synchronize()
        return r.matches_l, r.matches_p

    def arm_b():
        r = eng.match_set(eng.encode_images(views), pairs, line_thresh=thr)
        torch.cuda.synchronize()
        return r.matches_l, r.matches_p

    def arm_c():
        r = eng.match_set(pre, pairs, line_thresh=thr)
        torch.cuda.synchronize()
        return r.matches_l, r.matches_p

    def arm_d():
        r = gathered_match(eng, pre, pairs, thr)
        torch.cuda.synchronize()
        return r

    arms = {"match_images": arm_a, "encode_images+match_set": arm_b, "match_set": arm_c, "gather+ltr_match": arm_d}
    for _ in range(args.warmup):
        for fn in arms.values():
            fn()
    results = {k: fn() for k, fn in arms.items()}
    ref_l, ref_p = results["match_images"]
    equal = {k: bool(torch.equal(l, ref_l) and torch.equal(p, ref_p)) for k, (l, p) in results.items()}
    times = {k: [] for k in arms}
    for _ in range(2):
        for k, fn in arms.items():
            times[k] += timed(fn, args.iters // 2 or 1)
    name, power = gpu_info()
    out = {
        "workload": f"{args.views} synthetic 640x480 views of one scene, {args.lines} key lines and {args.points} keypoints "
                    f"per view, all {len(pairs)} pairs",
        "gpu": name, "power_limit": power,
        "ms": {k: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))} for k, v in times.items()},
        "launches": {k: launches(fn) for k, fn in arms.items()},
        "equal_to_match_images": equal,
        "line_matches": int((ref_l >= 0).sum()), "point_matches": int((ref_p >= 0).sum()),
    }
    print(json.dumps(out))
    if not all(equal.values()):
        raise SystemExit("the arms disagree")


if __name__ == "__main__":
    main()
