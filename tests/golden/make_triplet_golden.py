"""Triplet-loss fixtures (`triplet_outputs.npz`): the UNMODIFIED reference descriptor_loss
(evaluations/criteria.py:35-192, `compute_distances` and `forward`) and Result('val', args).evaluate
(evaluations/metric.py:16-46: nn_matcher_batches at nn_thresh 0.7, mutual, then Evaluate_PR) on CPU torch, called as
train.py:198-240 calls them.  Build container only:

    python tests/golden/make_triplet_golden.py

Cases (inputs [b, 256, n] float32 descriptors and [b, n+1, n+1] float32 mat_assign_sublines, dustbin included):
  trainlike  one pair (train.py's batch size) of n = 250: unit descriptors, side 1 a permuted and noised copy of side 0,
             0/1 assignments from lmatches with about half of the lines matched (train.py's gt_matches_sublines);
  overlap    overlap-valued assignments: entries in (0, 0.3], entries exactly 0.3f, many-to-many matches;
  far        descriptors far from unit norm with pos just above 9999.5, so the literal 10000 entries enter the window;
  duplicate  half of side 1 exact copies of side-0 lines (matched: distances within an ulp of 0, where `pos > 0`
             decides), the other half noisy unmatched copies of the same lines (their negatives);
  nopos      no entry above 0.3: the reference raises;
  nowindow   every entry matched, so no candidate is a negative: the reference raises.
Descriptors are rounded to bfloat16 values (stored as float32), so that the file stays small; `far` and `duplicate` are not,
because their edges (pos near 9999.5, unit norms that put pos within an ulp of 0) need the exact values.  Per case the file holds the inputs, the reference's outputs (dists_pos, dists_neg,
t_loss, hardest_positive, hardest_negative; or the exception's type), Result.evaluate's precision / recall / F1, the
per-anchor terms the reference computed (`ref_pos`, `ref_neg`, `ref_state`: the restatement on the reference's own
distances, checked here to reproduce its outputs bit for bit) and, up to SMALL lines, the reference's distance
matrices `2 - 2 einsum('bdn,bdm->bnm')`.
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("LINETR_REFERENCE", "/root/reference")
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)

from evaluations.criteria import descriptor_loss   # noqa: E402
from evaluations.metric import Result   # noqa: E402

from linetr_b200 import eval_criteria as EC   # noqa: E402

ARGS = types.SimpleNamespace(dataset_type="homography", nn_thresh=0.7, mutual_nn=True)   # train_manager.yaml
SMALL = 64   # distance matrices are stored up to this many lines


def unit(x):
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def bf16(x):
    """Round to the nearest bfloat16 value, kept as float32 (half of every value's bytes are then zero)."""
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).bfloat16().float().numpy()


def trainlike(rng, b=1, n=250):
    d0, d1, a = [], [], []
    for _ in range(b):
        x = unit(rng.normal(size=(256, n)).astype(np.float32).T).T
        perm = rng.permutation(n)
        sigma = rng.uniform(0.02, 0.35, n)   # close matches (the matcher finds them) to far ones (semi-hard windows)
        y = unit((x[:, perm] + rng.normal(0, 1, (256, n)) * sigma).T).T
        g = np.zeros((n + 1, n + 1), np.float32)
        m = rng.random(n) < 0.5                       # lmatches: about half of the lines
        cols = np.argsort(perm)                       # line i of side 0 is column cols[i] of side 1
        g[np.nonzero(m)[0], cols[m]] = 1
        d0.append(x); d1.append(y); a.append(g)
    return np.stack(d0), np.stack(d1), np.stack(a)


def overlap(rng, b=2, n=48):
    d0, d1, a = [], [], []
    for _ in range(b):
        x = unit(rng.normal(size=(n, 256))).T
        sigma = rng.uniform(0.02, 0.35, (n, 1))
        y = unit(x.T[rng.permutation(n)] + rng.normal(0, 1, (n, 256)) * sigma).T
        g = np.zeros((n + 1, n + 1), np.float32)
        r = rng.random((n, n))
        g[:n, :n] = np.where(r < 0.08, rng.uniform(0.31, 1.0, (n, n)), 0).astype(np.float32)        # many-to-many
        g[:n, :n] = np.where((r >= 0.08) & (r < 0.2), rng.uniform(1e-4, 0.3, (n, n)), g[:n, :n])   # (0, 0.3]
        g[:n, :n] = np.where((r >= 0.2) & (r < 0.25), np.float32(0.3), g[:n, :n])                  # exactly 0.3f
        g[:n, :n] = np.where((r >= 0.25) & (r < 0.27), np.nextafter(np.float32(0.3), np.float32(1)), g[:n, :n])
        g[n, :] = rng.random(n + 1) < 0.5   # dustbin entries are never read
        d0.append(x); d1.append(y); a.append(g.astype(np.float32))
    return np.stack(d0), np.stack(d1), np.stack(a)


def far(rng, b=1, n=32):
    """a_i = 70 u_i, the matched b_j = -(s_i / 70) u_i with <a_i, b_j> = -s_i: d = 2 + 2 s_i just above 9999.5."""
    d0, d1, a = [], [], []
    for _ in range(b):
        u = unit(rng.normal(size=(n, 256)))
        s = rng.uniform(4998.8, 4998.99, n)
        x = (70.0 * u).astype(np.float32)
        perm = rng.permutation(n)
        y = np.empty_like(x)
        y[perm] = (-(s / 70.0)[:, None] * u).astype(np.float32)
        y[perm[n // 2:]] = (70.0 * unit(rng.normal(size=(n - n // 2, 256)))).astype(np.float32)   # unrelated lines
        g = np.zeros((n + 1, n + 1), np.float32)
        g[np.arange(n // 2), perm[:n // 2]] = 1
        g[np.arange(n // 2, n), perm[np.arange(n // 2, n)]] = 0.2   # in-between entries: neither match nor unmatch
        d0.append(x.T); d1.append(y.T); a.append(g)
    return np.stack(d0), np.stack(d1), np.stack(a)


def duplicate(rng, b=1, n=40):
    d0, d1, a = [], [], []
    for _ in range(b):
        x = unit(rng.normal(size=(n, 256)))
        perm = rng.permutation(n)
        h = n // 2
        # side-1 line j < h is side-0 line perm[j] (matched); line j + h is a noisy, unmatched copy of the same line,
        # the negative of the semi-hard window (0, 0.5)
        y = np.concatenate([x[perm[:h]], unit(x[perm[:h]] + rng.normal(0, 0.015, (h, 256)))])
        g = np.zeros((n + 1, n + 1), np.float32)
        g[perm[:h], np.arange(h)] = 1
        d0.append(x.T); d1.append(y.T); a.append(g)
    return np.stack(d0), np.stack(d1), np.stack(a)


def nopos(rng, b=1, n=16):
    x = unit(rng.normal(size=(n, 256))).T[None]
    y = unit(rng.normal(size=(n, 256))).T[None]
    g = np.zeros((1, n + 1, n + 1), np.float32)
    g[0, :n, :n] = np.float32(0.3)   # exactly 0.3f: not a match in float32
    return x, y, g


def nowindow(rng, b=1, n=16):
    x = unit(rng.normal(size=(n, 256))).T[None]
    y = unit(rng.normal(size=(n, 256))).T[None]
    return x, y, np.ones((1, n + 1, n + 1), np.float32)


CASES = [("trainlike", trainlike), ("overlap", overlap), ("far", far), ("duplicate", duplicate), ("nopos", nopos),
         ("nowindow", nowindow)]
EXACT = {"far", "duplicate"}   # descriptors kept as generated: their norms decide the edge they test


def main():
    out = {"names": np.array([c for c, _ in CASES])}
    crit = descriptor_loss()
    for k, (name, make) in enumerate(CASES):
        rng = np.random.default_rng(100 + k)
        x, y, g = make(rng)
        if name not in EXACT:
            x, y = bf16(x), bf16(y)
        x, y, g = (np.ascontiguousarray(v, np.float32) for v in (x, y, g))
        pred = {"line_desc0": torch.from_numpy(x), "line_desc1": torch.from_numpy(y)}
        target = {"mat_assign_sublines": torch.from_numpy(g)}
        c = {"desc0": x, "desc1": y, "assign": g}
        with torch.no_grad():
            dist = (2 - 2 * torch.einsum("bdn,bdm->bnm", pred["line_desc0"], pred["line_desc1"])).numpy()
            try:
                dp, dn = crit.compute_distances(pred, target)
                t_loss, hp, hn = crit.forward(pred, target)
                c.update(dists_pos=dp.numpy(), dists_neg=dn.numpy(), loss=np.float32(t_loss.item()),
                         hardest_pos=np.float32(hp.item()), hardest_neg=np.float32(hn.item()), raised=np.array(""))
            except Exception as e:   # the reference's own failure on this input
                c["raised"] = np.array(type(e).__name__)
        if x.shape[2] <= SMALL:
            c["dist"] = dist
        # the restatement on the reference's distances must reproduce its outputs bit for bit
        t = EC.triplet_terms(list(dist), [a[:-1, :-1] for a in g])
        c.update(ref_pos=t["pos"], ref_neg=t["neg"], ref_state=t["state"].astype(np.int8))
        if str(c["raised"]) == "":
            v = t["state"] == EC.STATE_VALID
            assert np.array_equal(t["pos"][v], c["dists_pos"]) and np.array_equal(t["neg"][v], c["dists_neg"]), name
        else:
            assert t["n_valid"] == 0, name
        if str(c["raised"]) == "":
            res = Result("val", ARGS)
            res.evaluate(pred, target)
            c["pr"] = np.array([res.precision, res.recall, res.f1_score], np.float64).T
        for key, v in c.items():
            out[f"c{k}_{key}"] = v
        print(name, x.shape, "raised " + str(c["raised"]) if str(c["raised"]) else
              f"valid {len(c['dists_pos'])} loss {float(c['loss']):.6f} pr {c['pr'][:, 0]}")
    path = os.path.join(HERE, "triplet_outputs.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
