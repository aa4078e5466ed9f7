"""Homography ground truth for line matches and precision / recall of predicted matches.

Host drop-ins, numpy in and numpy out like the reference:

    line_assignment(lines0 [n0,2,2], lines1 [n1,2,2], homography [3,3], thres_reprojected=3, thres_angdiff=2,
                    min_overlap_ratio=0.3) -> (mat_assign_sublines [n0,n1] float64, lmatches [M,2] int64)
        the homography dataset builder's ground truth (dataloaders/build_homography_dataset.py:210-234: both
        find_line_matches, the mutual AND, both calculate_line_overlaps, their max, the min_overlap_ratio cut;
        dataloaders/utils/util_lines.py:67-171), including the np.linalg.inv of the homography; defaults of
        dataloaders/confs/homography.yaml
    get_precision_recall(score [B,n0,n1], score_gt [B,n0,n1]) -> (precisions, recalls, fscores)   (Evaluate_PR,
        evaluations/evaluate_pr.py:10-35)

`line_assignment` is a vectorised float32 restatement of the reference's scalar loops in the same operation order,
so its distances, lengths and ratios are the reference's bit for bit.  Two deliberate differences: squares are
correctly rounded products (numpy's float32 scalar `x**2` goes through libm powf, which is not correctly rounded and
differs from x*x in about 1 of 1000 values), and the angle is computed in fp64 (numpy's float32 arctan2 / degrees are
not correctly rounded either).  Both follow the CUDA kernel exactly.

Batched on the GPU (`ltr_line_gt`):

    homography_ground_truth(segs0, segs1, cu0, cu1, homographies, pred0=None, want_assign=True) -> LineGroundTruth
    score_line_matches(res: ImagePairMatches, homographies) -> per-pair and mean precision / recall / F1 of the
        line matches of `match_images` / `match_sets` against key-line ground truth
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from . import _native as N
from . import _ops

FLT_EPSILON = float(np.finfo(np.float32).eps)
EPS_PR = 1e-5   # Evaluate_PR.eps


# ------------------------------------------------------------------ host restatement
def _sq(x):
    return x * x


def project_lines(lines, homography) -> np.ndarray:
    """cv2.perspectiveTransform of [n,2,2] end points: fp64, times 1/w, rounded to fp32; (0, 0) where
    |w| <= FLT_EPSILON."""
    m = np.asarray(homography, dtype=np.float64).reshape(9)
    p = np.asarray(lines, dtype=np.float32).reshape(-1, 2).astype(np.float64)
    x, y = p[:, 0], p[:, 1]
    w = x * m[6] + y * m[7] + m[8]
    ok = np.abs(w) > FLT_EPSILON
    r = 1.0 / np.where(ok, w, 1.0)
    out = np.stack([(x * m[0] + y * m[1] + m[2]) * r, (x * m[3] + y * m[4] + m[5]) * r], 1)
    out[~ok] = 0.0
    return out.astype(np.float32).reshape(-1, 2, 2)


def _line_terms(l):
    sx, sy, ex, ey = l[:, 0, 0], l[:, 0, 1], l[:, 1, 0], l[:, 1, 1]
    a, b = ey - sy, ex - sx
    length = np.sqrt(_sq(a) + _sq(b))
    ang = np.degrees(np.arctan2(b.astype(np.float64), a.astype(np.float64)))   # atan2(dx, dy): x and y swapped
    return sx, sy, ex, ey, a, b, ex * sy, ey * sx, length, ang


def _match_overlap(l0, l1, thr_r, thr_a):
    """find_line_matches(l0, l1) and calc_overlap on the same entries: [n0, n1] float32 ratio where l1[j] matches
    l0[i], else -1."""
    sx0, sy0, ex0, ey0, a, b, c, d, len0, ang0 = (t[:, None] for t in _line_terms(l0))
    sx1, sy1, ex1, ey1, _, _, _, _, len1, ang1 = (t[None, :] for t in _line_terms(l1))

    def pl(x0, y0):   # |(y2-y1)*x0 - (x2-x1)*y0 + x2*y1 - y2*x1| / sqrt((y2-y1)^2 + (x2-x1)^2)
        return np.abs(((a * x0 - b * y0) + c) - d) / len0

    def pp(x0, y0, x1, y1):
        return np.sqrt(_sq(x1 - x0) + _sq(y1 - y0))

    ok = ~((pl(sx1, sy1) > thr_r) & (pl(ex1, ey1) > thr_r))
    ok &= ~(np.fmod(np.abs(ang1 - ang0), 180.0) > thr_a)
    s0s1, e0s1 = pp(sx0, sy0, sx1, sy1), pp(ex0, ey0, sx1, sy1)
    s0e1, e0e1 = pp(sx0, sy0, ex1, ey1), pp(ex0, ey0, ex1, ey1)
    sp_in = (s0s1 < len0) & (e0s1 < len0)
    ep_in = (s0e1 < len0) & (e0e1 < len0)
    mx = np.maximum(np.maximum(s0s1, e0s1), np.maximum(s0e1, e0e1))
    neither = np.where(mx > len0 + len1, np.float32(-1), np.float32(1))
    ratio = np.select([sp_in & ep_in, sp_in, ep_in],
                      [len1 / len0, np.where(s0e1 > e0e1, e0s1, s0s1) / len0, np.where(s0s1 > e0s1, e0e1, s0e1) / len0],
                      neither)
    return np.where(ok, ratio, np.float32(-1)).astype(np.float32)


def assignment_terms(lines0, lines1, proj0, proj1, thres_reprojected=3, thres_angdiff=2):
    """The builder's intermediate matrices from given projections (proj0 = lines0 mapped into image 1, proj1 = lines1
    mapped into image 0): find_line_matches(lines0, proj1), find_line_matches(lines1, proj0)^T, both
    calculate_line_overlaps on the mutual entries (the second transposed) and mat_assign_sublines, all float64
    [n0, n1]."""
    f32 = lambda v: np.asarray(v, dtype=np.float32).reshape(-1, 2, 2)
    lines0, lines1, proj0, proj1 = map(f32, (lines0, lines1, proj0, proj1))
    n0, n1 = len(lines0), len(lines1)
    if n0 == 0 or n1 == 0:
        z = np.zeros((n0, n1))
        return z, z.copy(), z.copy(), z.copy(), z.copy()
    thr_r, thr_a = np.float32(thres_reprojected), float(thres_angdiff)
    with np.errstate(all="ignore"):
        o0 = _match_overlap(lines0, proj1, thr_r, thr_a)
        o1 = _match_overlap(lines1, proj0, thr_r, thr_a).T
    m0, m1 = o0 >= 0, o1 >= 0
    mutual = m0 & m1
    ov0 = np.where(mutual, o0, 0).astype(np.float64)
    ov1 = np.where(mutual, o1, 0).astype(np.float64)
    return m0.astype(np.float64), m1.astype(np.float64), ov0, ov1, np.where(ov0 > ov1, ov0, ov1)


def line_assignment(lines0, lines1, homography, thres_reprojected=3, thres_angdiff=2, min_overlap_ratio=0.3):
    """-> (mat_assign_sublines [n0,n1] float64, lmatches [M,2] int64); homography maps image 0 to image 1 (the
    builder's `htrans`)."""
    h = np.asarray(homography, dtype=np.float64)
    proj0 = project_lines(lines0, h)
    proj1 = project_lines(lines1, np.linalg.inv(h))
    assign = assignment_terms(lines0, lines1, proj0, proj1, thres_reprojected, thres_angdiff)[4]
    return assign, np.array(np.where(assign > min_overlap_ratio), dtype=np.int64).T


def calc_tfpn(score, score_gt):
    """Evaluate_PR.calc_TFPN: (TP, FP, FN, TN) of one pair; TN counts rows whose number of columns with neither a
    prediction nor ground truth equals the number of rows."""
    score = np.asarray(score)
    g = np.where(np.asarray(score_gt) > 0, 1, 0)
    rows = g.sum(axis=1)
    n_pos, n_neg = int(np.count_nonzero(rows > 0)), int(np.count_nonzero(rows == 0))
    tp = int(np.count_nonzero(np.sum(score * g, axis=1) > 0))
    tn = int(np.count_nonzero(np.sum((1 - score) * (1 - g), axis=1) == g.shape[0]))
    return tp, n_neg - tn, n_pos - tp, tn


def precision_recall_from_counts(tfpn):
    """Per-pair precision, recall and F1 (float64 [P], percent) from TP/FP/FN/TN counts [P,4], with Evaluate_PR's
    formulas."""
    c = np.asarray(tfpn, dtype=np.int64).reshape(-1, 4)
    tp, fp, fn = c[:, 0], c[:, 1], c[:, 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        precision = np.nan_to_num(tp / (tp + fp + EPS_PR)) * 100.
        recall = np.nan_to_num(tp / (tp + fn + EPS_PR)) * 100.
        f1 = np.nan_to_num(2 * precision * recall / (precision + recall))
    return precision, recall, f1


def get_precision_recall(score, score_gt):
    """Evaluate_PR.get_precision_recall: per-pair lists (precisions, recalls, fscores) of score[i] against
    score_gt[i]."""
    counts = [calc_tfpn(score[i], score_gt[i]) for i in range(np.shape(score)[0])]
    p, r, f = precision_recall_from_counts(np.array(counts, dtype=np.int64).reshape(-1, 4))
    return list(p), list(r), list(f)


# ------------------------------------------------------------------ batched on the GPU
def _check_offsets(cu, n_pairs, n_segs, name) -> np.ndarray:
    cu = np.asarray(cu)
    if cu.ndim != 1 or len(cu) != n_pairs + 1 or not np.issubdtype(cu.dtype, np.integer):
        raise N.LtrError(f"homography_ground_truth: {name} must be integers [{n_pairs + 1}]")
    if n_pairs >= 0 and (cu[0] != 0 or cu[-1] != n_segs or np.any(np.diff(cu) < 0)):
        raise N.LtrError(f"homography_ground_truth: {name} must rise from 0 to the number of segments ({n_segs})")
    return np.ascontiguousarray(cu, dtype=np.int32)


@dataclass
class LineGroundTruth:
    """Result of `homography_ground_truth` (device outputs; nothing has been waited for).

    counts int32 [P]: entries > min_overlap_ratio per pair (the length of the builder's lmatches); tfpn int32 [P,4]
    (TP, FP, FN, TN) when predictions were given; assign_flat: the dense assignments, pair p at p * stride, row-major
    [n0[p], n1[p]] (want_assign only)."""
    counts: torch.Tensor
    tfpn: Optional[torch.Tensor]
    assign_flat: Optional[torch.Tensor]
    stride: int
    n0: np.ndarray
    n1: np.ndarray
    min_overlap_ratio: float

    @property
    def n_pairs(self) -> int:
        return len(self.n0)

    def assign(self, p: int) -> np.ndarray:
        """mat_assign_sublines of pair p, float64 [n0, n1] (host copy)."""
        if self.assign_flat is None:
            raise N.LtrError("assign() needs homography_ground_truth(..., want_assign=True)")
        n0, n1 = int(self.n0[p]), int(self.n1[p])
        return self.assign_flat[p * self.stride:p * self.stride + n0 * n1].view(n0, n1).cpu().numpy().astype(np.float64)

    def lmatches(self, p: int) -> np.ndarray:
        """The builder's lmatches of pair p: int64 [M, 2] row-major indices of entries > min_overlap_ratio."""
        return np.array(np.where(self.assign(p) > self.min_overlap_ratio), dtype=np.int64).T

    def precision_recall(self):
        """Per-pair (precision, recall, f1) float64 [P] from the counts, Evaluate_PR's formulas (host copy)."""
        if self.tfpn is None:
            raise N.LtrError("precision_recall() needs homography_ground_truth(..., pred0=...)")
        return precision_recall_from_counts(self.tfpn.cpu().numpy())


def homography_ground_truth(segs0, segs1, cu0, cu1, homographies, pred0=None, want_assign=True,
                            thres_reprojected=3.0, thres_angdiff=2.0, min_overlap_ratio=0.3, proj0=None, proj1=None,
                            device=None) -> LineGroundTruth:
    """`line_assignment` (and, with pred0, Evaluate_PR's counts) for P pairs in one `ltr_line_gt` launch.

    segs0 / segs1: [S,2,2] float32 segments of all pairs back to back, CUDA tensors or host arrays; cu0 / cu1: host
    int [P+1] offsets (side s of pair p = [cu_s[p], cu_s[p+1])); homographies: host [P,3,3] image 0 -> image 1, inverted
    on the host with np.linalg.inv as the builder does.  pred0: CUDA int32 [S0], predicted side-1 index (local to the
    pair) of every side-0 segment or -1.  want_assign=False writes no dense matrix (counts only).  proj0 / proj1:
    optional CUDA [S,2,2] projections to use instead of the kernel's own (segs0 by H, segs1 by H^-1).  Host arrays
    go up in one pinned copy; the call never waits for the device."""
    hs = np.asarray(homographies, dtype=np.float64)
    if hs.ndim != 3 or hs.shape[1:] != (3, 3):
        raise N.LtrError("homography_ground_truth: homographies must be [P, 3, 3]")
    if not np.all(np.isfinite(hs)):
        raise N.LtrError("homography_ground_truth: homographies must be finite")
    P = hs.shape[0]
    host, devs = {}, {}
    for nm, s in (("segs0", segs0), ("segs1", segs1)):
        if isinstance(s, torch.Tensor) and s.is_cuda:
            if s.dtype != torch.float32 or s.dim() != 3 or tuple(s.shape[1:]) != (2, 2):
                raise N.LtrError(f"homography_ground_truth: {nm} must be float32 [S, 2, 2]")
            devs[nm] = s.contiguous()
        else:
            a = np.ascontiguousarray(np.asarray(s, dtype=np.float32))
            if a.ndim != 3 or a.shape[1:] != (2, 2):
                raise N.LtrError(f"homography_ground_truth: {nm} must be [S, 2, 2]")
            host[nm] = a
    S0 = int((devs.get("segs0") if "segs0" in devs else host["segs0"]).shape[0])
    S1 = int((devs.get("segs1") if "segs1" in devs else host["segs1"]).shape[0])
    c0, c1 = _check_offsets(cu0, P, S0, "cu0"), _check_offsets(cu1, P, S1, "cu1")
    if pred0 is not None and (not isinstance(pred0, torch.Tensor) or pred0.dim() != 1 or pred0.shape[0] != S0):
        raise N.LtrError(f"homography_ground_truth: pred0 must be a CUDA tensor [{S0}]")
    hinv = np.linalg.inv(hs) if P else hs.copy()
    if device is None:
        device = next((t.device for t in devs.values()), None) or _ops.current_cuda_device()
    device = torch.device(device)
    dv = _ops.stage({**host, "cu0": c0, "cu1": c1, "homography": hs, "homography_inv": np.ascontiguousarray(hinv)},
                    device)
    dv.update(devs)
    n0, n1 = np.diff(c0), np.diff(c1)
    mx0, mx1 = int(n0.max(initial=0)), int(n1.max(initial=0))
    i32 = dict(dtype=torch.int32, device=device)
    counts = torch.zeros(P, **i32)
    tfpn = torch.zeros((P, 4), **i32) if pred0 is not None else None
    stride = mx0 * mx1
    assign = torch.zeros(max(P * stride, 1), dtype=torch.float32, device=device) if want_assign else None
    if pred0 is not None:
        pred0 = pred0.to(device=device, dtype=torch.int32).contiguous()
    if proj0 is not None:
        proj0 = proj0.float().contiguous()
    if proj1 is not None:
        proj1 = proj1.float().contiguous()
    _ops.call_struct("ltr_line_gt", {**dv, "proj0": proj0, "proj1": proj1, "pred0": pred0, "n_pairs": P,
                                     "max_n0": mx0, "max_n1": mx1, "thres_reprojected": thres_reprojected,
                                     "thres_angdiff": thres_angdiff, "min_overlap_ratio": min_overlap_ratio},
                     dict(assign=assign, assign_stride=stride, n_gt=counts, tfpn=tfpn))
    return LineGroundTruth(counts, tfpn, assign, stride, n0, n1, float(min_overlap_ratio))


def score_line_matches(res, homographies, thres_reprojected=3.0, thres_angdiff=2.0, min_overlap_ratio=0.3) -> dict:
    """Precision / recall / F1 of the line matches of an `ImagePairMatches` (`match_images`, `match_sets`) against
    homography ground truth between its key lines (res.klines0 / res.klines1, as float32 segments); homographies
    [P,3,3] map image 0 to image 1 of every pair.  Returns per-pair float64 arrays 'precision', 'recall', 'f1' (percent,
    Evaluate_PR) and their means over the pairs 'mean_precision', 'mean_recall', 'mean_f1' (AverageMeter); copies the
    P x 4 counts to the host."""
    P = res.n_pairs
    segs = lambda ks: (np.concatenate([np.asarray(k, dtype=np.float32).reshape(-1, 2, 2) for k in ks])
                       if len(ks) else np.zeros((0, 2, 2), dtype=np.float32))
    cu = lambda ks: np.concatenate([[0], np.cumsum([len(k) for k in ks])]).astype(np.int32)
    cu0, cu1 = cu(res.klines0), cu(res.klines1)
    if not np.array_equal(cu0, np.asarray(res.offsets_l)):
        raise N.LtrError("score_line_matches: key lines and line-match offsets disagree")
    gt = homography_ground_truth(segs(res.klines0), segs(res.klines1), cu0, cu1, homographies, pred0=res.matches_l,
                                 want_assign=False, thres_reprojected=thres_reprojected, thres_angdiff=thres_angdiff,
                                 min_overlap_ratio=min_overlap_ratio, device=res.matches_l.device)
    p, r, f = gt.precision_recall()
    mean = lambda v: float(np.sum(v) / P) if P else 0.0
    return {"precision": p, "recall": r, "f1": f, "mean_precision": mean(p), "mean_recall": mean(r), "mean_f1": mean(f)}
