"""Single-pair latency through the reference-shaped API (the way `Matching.forward` drives the hot path:
models/matching.py:41,59,77-81): two LineTransformer.forward calls of ONE image each + get_dist_matrix +
subline2keyline + nn_matcher_distmat with host numpy in between, eager launches vs the CUDA-graph option,
next to the CPU port on the host cores.  Prints one JSON object."""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from bench import load_weights, run_cpu_leg
from linetr_b200 import LineTransformer, PairEngine, LineBatch, get_dist_matrix, nn_matcher_distmat, synthetic as syn

dev = torch.device("cuda", 0)
sd, wnote = load_weights()
out = {"weights": wnote, "shape": "1 pair x 128 lines x 21 tokens"}
a, b, _ = syn.make_pair_inputs(5, 128, 21)
da = {k: torch.from_numpy(v).to(dev) for k, v in a.items()}
db = {k: torch.from_numpy(v).to(dev) for k, v in b.items()}


def timeit(fn, n=200, warm=20):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(n):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    ts = np.asarray(ts) * 1e3
    return {"median_ms": float(np.median(ts)), "p10_ms": float(np.percentile(ts, 10)), "p90_ms": float(np.percentile(ts, 90))}


for mode in ("eager", "cuda_graph"):
    m = LineTransformer({"mode": "train", "cuda_graph": mode == "cuda_graph"})
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    m = m.eval().to(dev)

    def forward_one():
        return m(dict(da))["line_desc"]

    def pair_reference_sequence():
        d0 = m(dict(da))["line_desc"].cpu().numpy()          # matching.py:77-78
        d1 = m(dict(db))["line_desc"].cpu().numpy()
        dist = get_dist_matrix(d0, d1)[0]                      # :79
        dk = m.subline2keyline(dist, da["mat_klines2sublines"][0], db["mat_klines2sublines"][0])   # :80
        return nn_matcher_distmat(dk, 0.8, True)               # :81

    want = pair_reference_sequence()
    out[mode] = {"forward_1_image": timeit(forward_one), "pair_reference_call_sequence": timeit(pair_reference_sequence, n=100)}
    if mode == "eager":
        ref = want
    else:
        out["graph_equals_eager"] = bool(np.array_equal(ref, want))
    # batched front-end, one pair, everything on the device
    eng = PairEngine(m, dev)
    ba, bb = LineBatch.from_images([a]).to(dev), LineBatch.from_images([b]).to(dev)
    if mode == "eager":
        out["engine_match_pairs_1_pair"] = timeit(lambda: eng.match_pairs(ba, bb, 0.8).counts)
# ---- the same pair starting where `Matching` starts the plugin: SuperPoint's dense maps already on the device + detected key
#      lines (host objects) -> GPU tokeniser (LineTransformer.preprocess -> ltr_tokenize_batch) -> forward x2 -> matcher calls
try:
    from tests.test_tokenizer import fake_lines, fake_superpoint
    m = LineTransformer({"mode": "test"})
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    m = m.eval().to(dev)
    sp = [{k: v.to(dev) for k, v in fake_superpoint(s).items()} for s in (7, 8)]
    kl = [fake_lines(7, 120), fake_lines(8, 120)]

    def pair_from_maps():
        p0 = m.preprocess(kl[0], (1, 1, 480, 640), sp[0], None)
        p1 = m.preprocess(kl[1], (1, 1, 480, 640), sp[1], None)
        d0 = m(p0)["line_desc"].cpu().numpy()
        d1 = m(p1)["line_desc"].cpu().numpy()
        dist = get_dist_matrix(d0, d1)[0]
        dk = m.subline2keyline(dist, p0["mat_klines2sublines"][0], p1["mat_klines2sublines"][0])
        return nn_matcher_distmat(dk, 0.8, True), int(p0["sublines"].shape[1]), int(p1["sublines"].shape[1])

    _, s0, s1 = pair_from_maps()
    out["pair_from_superpoint_maps_on_device"] = {**timeit(lambda: pair_from_maps(), n=60, warm=10),
                                                  "sublines": [s0, s1], "note": "2 x (host line filtering + GPU tokeniser) + "
                                                  "2 x forward + get_dist_matrix + subline2keyline + nn_matcher_distmat"}
except Exception as e:   # the tool must not fail on the optional leg
    out["pair_from_superpoint_maps_on_device"] = {"error": f"{type(e).__name__}: {e}"}
leg = run_cpu_leg("cfg1", 8, 10, 3)
out["cpu_port_8_threads"] = {"ms_per_pair_median": 1e3 * leg["s_per_pair_median"]}
leg = run_cpu_leg("cfg1", 1, 10, 3)
out["cpu_port_1_thread"] = {"ms_per_pair_median": 1e3 * leg["s_per_pair_median"]}
print(json.dumps(out))
