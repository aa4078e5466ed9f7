"""Homography ground-truth fixtures (`line_gt_outputs.npz`): the UNMODIFIED reference functions
find_line_matches / calculate_line_overlaps (dataloaders/utils/util_lines.py:67-171), called the way the dataset
builder calls them (dataloaders/build_homography_dataset.py:210-234, with cv2.perspectiveTransform), and
Evaluate_PR (evaluations/evaluate_pr.py) on predictions from nn_matcher_batches (evaluations/matcher.py) and on
hand-made predictions.  Build container only:

    python tests/golden/make_line_gt_golden.py

Cases: (a) the sublines of the four bundled real pairs (plumbing_pairs.npz) under seeded homographies sampled by the
reference's sample_homography_np with the parameters of dataloaders/confs/homography.yaml; (b) synthetic lines
mapped by a homography plus sub-pixel noise (many true matches); (c) adversarial pairs: zero-length segments, nested /
touching / disjoint collinear segments, anti-parallel lines and lines at ~179 degrees, one end point within the
reprojection threshold, points with |w| <= FLT_EPSILON, a non-square pair for calc_TFPN's TN rule.

Per pair the file holds the inputs, the cv2 projections the reference used, both find_line_matches matrices (the
second transposed), both overlap matrices (the second transposed), mat_assign_sublines, lmatches, the Evaluate_PR
counts and outputs for both kinds of predictions, and two sparse sets of entries where a computation that differs
from the reference's on purpose could change the result:
  - `ang_flag`: entries where the reference's float32 angle decision (numpy scalar arctan2 / degrees, as the
    reference evaluates them) differs from the fp64 one, or the fp64 margin to a decision boundary (the threshold,
    or |a1 - a0| at 180 / 360) is below 1e-9; `ang_margin` is the fp64 margin of every entry below 1e-2 degrees;
  - `pow_flag`: entries whose result changes when squares are numpy float32 scalar `x**2` (libm powf, which is not
    correctly rounded) instead of correctly rounded products.
The generator checks that linetr_b200.eval_homography with the reference's squares reproduces every matrix outside
ang_flag exactly.
"""
import os
import sys

import cv2
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("LINETR_REFERENCE", "/root/reference")
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(REF, "dataloaders"))   # the reference's own `utils.*` imports

from utils.util_lines import find_line_matches, calculate_line_overlaps   # noqa: E402
from utils.homographies import sample_homography_np   # noqa: E402
from evaluations.evaluate_pr import Evaluate_PR   # noqa: E402
from evaluations.matcher import nn_matcher_batches   # noqa: E402

from linetr_b200 import eval_homography as EH   # noqa: E402

THR_R, THR_A, MIN_OV = 3, 2, 0.3           # dataloaders/confs/homography.yaml
HOMOGRAPHY_PARAMS = dict(perspective=True, scaling=True, translation=True, rotation=True, patch_ratio=0.85,
                         perspective_amplitude_x=0.2, perspective_amplitude_y=0.2, scaling_amplitude=0.2,
                         max_angle=1.0472, allow_artifacts=True)
W, H = 640, 480


def pixel_homography(rng_seed):
    """A homography image 0 -> image 1 in pixels, as the builder derives `htrans`: the inverse of a sampled
    normalised-coordinate homography, conjugated into pixel coordinates."""
    np.random.seed(rng_seed)
    h = sample_homography_np(np.array([2, 2]), shift=-1, **HOMOGRAPHY_PARAMS)
    t = np.array([[2. / W, 0., -1.], [0., 2. / H, -1.], [0., 0., 1.]])
    return np.linalg.inv(t) @ np.linalg.inv(h) @ t


def cv2_project(lines, h):
    if len(lines) == 0:
        return np.zeros((0, 2, 2), np.float32)
    return cv2.perspectiveTransform(lines.reshape(1, -1, 2), h)[0].reshape(-1, 2, 2)


def reference_assignment(l0, l1, htrans):
    """The builder's calls, lines 214-234."""
    p0 = cv2_project(l0, htrans)
    p1 = cv2_project(l1, np.linalg.inv(htrans))
    m0 = find_line_matches(l0, p1, THR_R, THR_A)
    m1 = find_line_matches(l1, p0, THR_R, THR_A).T
    b = np.logical_and(m0 > 0, m1 > 0)
    lm0 = np.array(np.where(b)).T
    lm1 = np.zeros_like(lm0)
    lm1[:, 0], lm1[:, 1] = lm0[:, 1], lm0[:, 0]
    ov0, _ = calculate_line_overlaps(l0, p1, lm0)
    ov1, _ = calculate_line_overlaps(l1, p0, lm1)
    ov1 = ov1.T
    assign = np.where(ov0 > ov1, ov0, ov1)
    lmatches = np.array(np.where(assign > MIN_OV)).T
    return p0, p1, m0, m1, ov0, ov1, assign, lmatches


def scalar_angles(lines):
    """The reference's per-line float32 angle, evaluated as it does: numpy scalars."""
    return np.array([np.degrees(np.arctan2((l[1, 0] - l[0, 0]), (l[1, 1] - l[0, 1]))) for l in lines], np.float32)


def angle_flags(l0, l1, p0, p1):
    """(flag [n0,n1] bool, fp64 margin [n0,n1]) over both directions of find_line_matches."""
    flag = np.zeros((len(l0), len(l1)), bool)
    margin = np.full((len(l0), len(l1)), np.inf)
    for a, b, tr in ((l0, p1, False), (l1, p0, True)):
        ra, rb = scalar_angles(a), scalar_angles(b)
        ref_pass = ~((np.abs(rb[None, :] - ra[:, None]) % np.float32(180)) > THR_A)
        a64 = EH._line_terms(a)[9]
        b64 = EH._line_terms(b)[9]
        diff = np.abs(b64[None, :] - a64[:, None])
        pass64 = ~(np.fmod(diff, 180.0) > THR_A)
        m = np.minimum(np.abs(np.fmod(diff, 180.0) - THR_A), np.minimum(np.abs(diff - 180.0), np.abs(diff - 360.0)))
        f = (ref_pass != pass64) | (m < 1e-9)
        flag |= f.T if tr else f
        margin = np.minimum(margin, m.T if tr else m)
    return flag, margin


def powf_square(x):
    x = np.asarray(x, dtype=np.float32)
    return np.array([v ** 2 for v in x.ravel()], dtype=np.float32).reshape(x.shape)


def oracle(l0, l1, p0, p1, square=None):
    if square is not None:
        EH._sq = square
    try:
        return EH.assignment_terms(l0, l1, p0, p1, THR_R, THR_A)
    finally:
        EH._sq = lambda v: v * v


def predictions(rng, assign, n1):
    """nn_matcher_batches on descriptors that follow the ground truth, and hand-made predictions: int32 [n0]."""
    n0 = assign.shape[0]
    d0 = rng.standard_normal((256, n0)).astype(np.float32)
    d1 = rng.standard_normal((256, n1)).astype(np.float32)
    for i in range(n0):
        j = int(np.argmax(assign[i])) if n1 else 0
        if n1 and assign[i, j] > 0:
            d1[:, j] = d0[:, i] + 0.6 * rng.standard_normal(256).astype(np.float32)
    if n1:
        nn = nn_matcher_batches(d0[None] / 16, d1[None] / 16, 1.0, is_mutual_NN=True)[0, :-1, :-1]
        pred_nn = np.where(nn.any(1), nn.argmax(1), -1).astype(np.int32)
    else:
        pred_nn = np.full(n0, -1, np.int32)
    u = rng.random(n0)
    gtj = assign.argmax(1) if n1 else np.zeros(n0, np.int64)
    rand = rng.integers(0, max(n1, 1), n0)
    pred_hand = np.where(u < 0.5, gtj, np.where(u < 0.75, rand, -1)).astype(np.int32) if n1 else np.full(n0, -1, np.int32)
    return pred_nn, pred_hand


def dense(pred, n1):
    m = np.zeros((len(pred), n1))
    r = np.nonzero(pred >= 0)[0]
    m[r, pred[r]] = 1
    return m


def seg(x0, y0, x1, y1):
    return [[x0, y0], [x1, y1]]


def polar(x, y, deg, length):
    """A segment from (x, y) whose reference angle degrees(atan2(dx, dy)) is `deg`."""
    r = np.radians(deg)
    return seg(x, y, x + length * np.sin(r), y + length * np.cos(r))


def adversarial():
    ident = np.eye(3)
    a0 = float(np.degrees(np.arctan2(30.0, 40.0)))
    l0 = [seg(10, 50, 50, 50),                  # collinear family on y = 50
          seg(100, 100, 100, 100),              # zero length
          seg(200, 200, 230, 240),              # dx 30, dy 40
          seg(300, 300, 300, 360),              # vertical, for the end-point-threshold cases
          seg(400, 100, 460, 100),
          seg(500, 300, 500, 300)]              # zero length, no partner
    l1 = [seg(20, 50, 40, 50),                  # nested in l0[0]
          seg(50, 50, 80, 50),                  # touching at an end point
          seg(90, 50, 120, 50),                 # disjoint, collinear
          seg(30, 50, 70, 50),                  # overlapping
          seg(50, 50, 10, 50),                  # identical, reversed (anti-parallel, exactly 180)
          seg(95, 100, 105, 100),               # through the zero-length l0[1]
          seg(100, 100, 100, 100),              # zero length on the zero-length l0[1]
          seg(230, 240, 200, 200),              # anti-parallel to l0[2]
          polar(201, 201, a0 - 180.5, 50),      # |a1 - a0| = 180.5: passes
          polar(201, 201, a0 - 179.0, 50),      # 179 degrees: fails
          polar(201, 201, a0 + 1.5, 50),        # 1.5 degrees: passes
          polar(201, 201, a0 + 2.5, 50),        # 2.5 degrees: fails
          seg(302, 310, 310, 350),              # start within 3 px of l0[3], end far
          seg(310, 310, 320, 350),              # both far
          seg(302.5, 320, 302.9, 340),          # both within, nearly parallel
          seg(400, 102, 430, 102),              # parallel, 2 px off, inside
          seg(450, 99, 500, 99),                # parallel, one end inside
          seg(380, 100, 480, 100)]              # contains l0[4]
    cases = [("adv_lines", np.array(l0, np.float32), np.array(l1, np.float32), ident)]
    # |w| <= FLT_EPSILON: w = 1e-3 x - 0.1 vanishes at x = 100
    hw = np.array([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [1e-3, 0.0, -0.1]])
    lw0 = np.array([seg(100, 10, 100, 60), seg(100, 10, 160, 10), seg(150, 40, 170, 90), seg(0, 0, 0, 0)], np.float32)
    lw1 = np.array([seg(0, 0, 0, 0), seg(0, 0, 600, 0), seg(-1000, 100, -1000, 600), seg(100, 5, 100, 400)], np.float32)
    cases.append(("adv_w_eps", lw0, lw1, hw))
    # non-square (n1 = n0 + 1) and (n1 = n0 - 2) pairs: TN counts rows with shape[0] "neither" columns
    rng = np.random.default_rng(5)
    base = (rng.random((6, 2, 2)) * np.array([600, 440]) + 20).astype(np.float32)
    cases.append(("adv_nonsquare_wide", base, np.concatenate([base[::-1], base[:1] + 200]).astype(np.float32), ident))
    cases.append(("adv_nonsquare_tall", base, base[[1, 3, 0, 5]].copy(), ident))
    cases.append(("adv_empty_side", base, np.zeros((0, 2, 2), np.float32), ident))
    return cases


def synthetic(seed, n, noise):
    rng = np.random.default_rng(seed)
    sp = rng.random((n, 2)) * np.array([W - 40, H - 40]) + 20
    ang = rng.random(n) * 2 * np.pi
    ln = rng.uniform(20, 150, n)
    l0 = np.stack([sp, sp + np.stack([np.cos(ang), np.sin(ang)], 1) * ln[:, None]], 1).astype(np.float32)
    h = pixel_homography(100 + seed)
    keep = rng.permutation(n)[: int(n * 0.8)]
    mapped = cv2_project(l0[keep], h) + rng.normal(0, noise, (len(keep), 2, 2)).astype(np.float32)
    extra = (rng.random((n - len(keep), 2, 2)) * np.array([W, H])).astype(np.float32)
    l1 = np.concatenate([mapped, extra])[rng.permutation(n)].astype(np.float32)
    return l0, l1, h


def real_pairs():
    z = np.load(os.path.join(HERE, "plumbing_pairs.npz"))
    out = []
    for p in range(4):
        l0 = z[f"p{p}_0_sublines"][0].astype(np.float32)
        other = z[f"p{p}_1_sublines"][0].astype(np.float32)
        h = pixel_homography(10 + p)
        rng = np.random.default_rng(20 + p)
        keep = rng.permutation(len(l0))[: len(l0) * 2 // 3]
        mapped = cv2_project(l0[keep], h) + rng.normal(0, 0.2, (len(keep), 2, 2)).astype(np.float32)
        l1 = np.concatenate([mapped, other[: len(other) // 2]])
        out.append((f"real_{p}", l0, l1[rng.permutation(len(l1))].astype(np.float32), h))
    return out


def main():
    cases = real_pairs()
    for s, (n, noise) in enumerate(((250, 0.3), (250, 0.8))):
        l0, l1, h = synthetic(s, n, noise)
        cases.append((f"synthetic_{s}", l0, l1, h))
    cases += adversarial()
    ev = Evaluate_PR(None)
    rng = np.random.default_rng(7)
    out = {"names": np.array([c[0] for c in cases]), "thresholds": np.array([THR_R, THR_A, MIN_OV], np.float64)}
    tot_flag = tot_pow = 0
    for k, (name, l0, l1, h) in enumerate(cases):
        p0, p1, m0, m1, ov0, ov1, assign, lmatches = reference_assignment(l0, l1, h)
        # the restatement with the reference's squares must reproduce everything outside the angle flags
        ang_flag, ang_margin = angle_flags(l0, l1, p0, p1)
        mine_ref_sq = oracle(l0, l1, p0, p1, powf_square)
        mine = oracle(l0, l1, p0, p1)
        for nm, want, a, b in zip(("m0", "m1", "ov0", "ov1", "assign"), (m0, m1, ov0, ov1, assign), mine_ref_sq, mine):
            bad = (a != want) & ~ang_flag
            assert not bad.any(), (name, nm, np.argwhere(bad)[:5])
        pow_flag = np.zeros_like(ang_flag)
        for a, b in zip(mine_ref_sq, mine):
            pow_flag |= a != b
        pred_nn, pred_hand = predictions(rng, assign, len(l1))
        g = f"c{k}_"
        out.update({g + "lines0": l0, g + "lines1": l1, g + "H": h, g + "proj0": p0, g + "proj1": p1,
                    g + "m0": m0.astype(np.uint8), g + "m1": m1.astype(np.uint8), g + "ov0": ov0.astype(np.float32),
                    g + "ov1": ov1.astype(np.float32), g + "assign": assign.astype(np.float32),
                    g + "lmatches": lmatches.astype(np.int64), g + "pred_nn": pred_nn, g + "pred_hand": pred_hand,
                    g + "ang_flag": np.argwhere(ang_flag).astype(np.int32),
                    g + "ang_near": np.argwhere(ang_margin < 1e-2).astype(np.int32),
                    g + "ang_margin": ang_margin[ang_margin < 1e-2],
                    g + "pow_flag": np.argwhere(pow_flag).astype(np.int32)})
        assert np.array_equal(assign.astype(np.float32).astype(np.float64), assign)   # fp32 storage is lossless
        for tag, pred in (("nn", pred_nn), ("hand", pred_hand)):
            score = dense(pred, len(l1))
            out[g + f"tfpn_{tag}"] = np.array(ev.calc_TFPN(score, assign), np.int64)
            out[g + f"pr_{tag}"] = np.array([v[0] for v in ev.get_precision_recall(score[None], assign[None])], np.float64)
        tot_flag += int(ang_flag.sum())
        tot_pow += int(pow_flag.sum())
        print(f"{name}: {len(l0)} x {len(l1)}, {int((m0 * m1).sum())} mutual, {len(lmatches)} lmatches, "
              f"angle-flagged {int(ang_flag.sum())}, pow-flagged {int(pow_flag.sum())}, tfpn nn {out[g + 'tfpn_nn']}, "
              f"hand {out[g + 'tfpn_hand']}")
    path = os.path.join(HERE, "line_gt_outputs.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path)} bytes); angle-flagged {tot_flag}, pow-flagged {tot_pow}")


if __name__ == "__main__":
    torch.set_grad_enabled(False)
    main()
