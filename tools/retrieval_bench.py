"""Image retrieval timings on one GPU, printed as one JSON line:
- an encoded set of 256 images (16 scenes of 16 views, `encode_images` with seeded weights): vocabulary training,
  VLAD, and `retrieval_pairs(k = 10)` + `match_set` against `match_set` on all 32,640 pairs;
- vocabulary training and VLAD of a larger synthetic descriptor set;
- `retrieve` for 1024 queries against 8192 database images at D = 32768, with torch.profiler kernel times, the
  screening kernel's share of its lower bound, and torch.topk(q @ d.T) in fp32 (TF32 off) for comparison."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from linetr_b200 import retrieval as RT
from linetr_b200 import synthetic as syn


def gpu_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"]).decode()
        return out.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def timed(fn, reps):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def kernel_times(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            out[e.key] = round(e.device_time_total / 1e3 / max(e.count, 1), 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=1024)
    ap.add_argument("--database", type=int, default=8192)
    ap.add_argument("--dim", type=int, default=32768)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--places", type=int, default=512)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    res = {"gpu": gpu_info()}

    # an encoded set: retrieval pairs + match_set against exhaustive match_set
    from linetr_b200 import LineTransformer, PairEngine
    from linetr_b200.engine import exhaustive_pairs
    model = LineTransformer({"mode": "train"})
    model.load_state_dict({k: torch.from_numpy(v) for k, v in syn.make_state_dict(0, 1).items()})
    eng = PairEngine(model.eval().to(dev), dev)
    views = [syn.image_to(v, dev) for sc in range(16) for v in syn.make_image_set(200 + sc, 16, 60, 400)]
    es = eng.encode_images(views)
    res["encoded_train_ms"] = timed(lambda: RT.train_vocabulary(es, 64, 64, iters=20, seed=0), 2)
    evoc = RT.train_vocabulary(es, 64, 64, iters=20, seed=0)
    res["encoded_vlad_ms"] = timed(lambda: RT.global_descriptors(es, evoc), a.reps)
    eg = RT.global_descriptors(es, evoc)
    rp = RT.retrieval_pairs(eg, 10)
    ex = exhaustive_pairs(len(views))
    res["encoded_pairs"] = {"retrieved": len(rp), "exhaustive": len(ex),
                            "retrieved_within_scene": float((rp[:, 0] // 16 == rp[:, 1] // 16).mean())}
    res["encoded_retrieval_pairs_plus_match_set_ms"] = timed(lambda: eng.match_set(es, RT.retrieval_pairs(eg, 10)), 3)
    res["encoded_exhaustive_match_set_ms"] = timed(lambda: eng.match_set(es, ex), 2)

    # vocabulary and VLAD of a synthetic set (256 views of a corridor, 24 observations per landmark part)
    s = syn.make_covisibility_set(0, n_views=256, n_distractors=0, per_landmark=24)
    ds = RT.descriptor_set(s["points"], s["lines"], dev)
    res["set_rows"] = [int(ds.cu_points[-1]), int(ds.cu_lines[-1])]
    res["train_ms"] = timed(lambda: RT.train_vocabulary(ds, 64, 64, iters=20, seed=0), 2)
    voc = RT.train_vocabulary(ds, 64, 64, iters=20, seed=0)
    res["vlad_ms"] = timed(lambda: RT.global_descriptors(ds, voc), a.reps)

    # retrieval: database images drawn around `places` place vectors, queries near database images
    g = torch.Generator(device=dev).manual_seed(0)
    Q, Nn, D = a.queries, a.database, a.dim
    place = torch.nn.functional.normalize(torch.randn(a.places, D, device=dev, generator=g), dim=1)
    member = torch.randint(0, a.places, (Nn,), device=dev, generator=g)
    db = torch.nn.functional.normalize(place[member] + 0.8 * torch.randn(Nn, D, device=dev, generator=g) / D ** 0.5, dim=1)
    pick = torch.randint(0, Nn, (Q,), device=dev, generator=g)
    q = torch.nn.functional.normalize(db[pick] + 0.8 * torch.randn(Q, D, device=dev, generator=g) / D ** 0.5, dim=1)
    gq, gd = RT.GlobalDescriptors.from_rows(q.contiguous()), RT.GlobalDescriptors.from_rows(db.contiguous())
    r = RT.retrieve(gq, gd, a.k)
    res["retrieve_ms"] = timed(lambda: RT.retrieve(gq, gd, a.k), a.reps)
    res["full_pass_queries"] = int(r.n_full.item())
    res["retrieve_kernels_ms"] = kernel_times(lambda: RT.retrieve(gq, gd, a.k))
    screen = next((v for k, v in res["retrieve_kernels_ms"].items() if "rt_screen" in k), None)
    flop_s = 3 * 2 * Q * Nn * D / 989e12
    byte_s = (Q + Nn) * D * 4 / 3.35e12    # the two tile images (hi + lo bf16), each read at least once
    res["screen_bound_ms"] = {"tensor": flop_s * 1e3, "bytes": byte_s * 1e3}
    if screen:
        res["screen_share_of_bound"] = max(flop_s, byte_s) * 1e3 / screen
        res["screen_bound_by"] = "tensor FLOP" if flop_s > byte_s else "bytes"
    torch.backends.cuda.matmul.allow_tf32 = False
    tk = lambda: torch.topk(q @ db.T, a.k, dim=1)   # noqa: E731
    res["torch_topk_fp32_ms"] = timed(tk, a.reps)
    ti = tk().indices.int()
    res["torch_topk_rows_differing"] = int((ti != r.idx).any(1).sum().item())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
