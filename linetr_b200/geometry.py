"""Geometric verification of matches: RANSAC homographies from line and point matches, the corner-error metric, and
the relative pose of calibrated pairs with the reference's pose metrics.

    estimate_homographies(res: ImagePairMatches, thresh=3.0, n_hypotheses=2048, seed=0, use_lines=True,
                          use_points=True) -> HomographyResult
        one `ltr_homography` call for every pair of a `match_images` / `match_sets` result; device outputs, no
        synchronisation
    ransac_homography_host(kpts0, kpts1, matches_p, klines0, klines1, matches_l, pair=0, ...) -> dict
        the same model for one pair in numpy: the normalisation, the hash, the solve and the residuals are the
        kernels' operations in the kernels' order (so the winning hypothesis and its inlier count are the same bits);
        the refit uses np.linalg.eigh instead of the kernels' Jacobi solve
    homography_corner_error(H_est, H_gt, shapes) -> mean distance of the four mapped image corners per pair and the
        accuracy at 1 / 3 / 5 px (host numpy)

The model (DESIGN.md "Homography estimation", include/linetr_b200.h `ltr_homography`): H maps image 0 to image 1.  The
correspondences of a pair are its matched side-0 keypoints in row order, then its matched side-0 key lines (segments
s0 = (a0, b0) with partner s1) in row order.  Per side, coordinates are normalised by the midpoint c of their
bounding box and s = half its larger extent (1 when 0).  A point gives the two DLT rows, a line l1^T H p = 0 for both
end points p of s0, with l1 the line through s1 scaled to l1x^2 + l1y^2 = 1.  Hypothesis k of pair p draws 4 distinct
correspondences (`draw_samples`) and solves them with h33 = 1 by Gaussian elimination with partial pivoting in fp64.
Residuals are in pixels of image 1: a point's |pi(H x0) - x1|^2 (OpenCV's reprojection error), a line's larger squared
distance of pi(H a0), pi(H b0) to the line through s1; |w| <= FLT_EPSILON makes an outlier; inlier iff < thresh^2.
The winner has the most inliers (lowest k on a tie) and is refitted by least squares over its inliers, kept iff the
refit has at least as many inliers.

    estimate_poses(res, K0, K1, thresh=1.0, n_hypotheses=1024, seed=0, dist_thresh=1e9) -> PoseResult
        one `ltr_essential` call for every pair of a `match_images` / `match_sets` result; device outputs, no
        synchronisation
    ransac_essential_host(kpts0, kpts1, matches_p, K0, K1, pair=0, ...) -> dict
        the same model for one pair in numpy: everything up to the winner is the kernels' operations in the kernels'
        order (the winning sample, root and inlier count are the same bits); the decomposition uses np.linalg.svd
    compute_epipolar_error, compute_pose_error, pose_auc: the reference's metrics (models/utils.py:358-412);
    pose_errors(R, t, T_0to1): compute_pose_error over a batch of pairs

The relative-pose model (DESIGN.md "Relative pose", include/linetr_b200.h `ltr_essential`): the correspondences of a
pair are its matched side-0 keypoints in row order with their partners, in normalised coordinates (k - c) / f.
t_n = thresh / f_mean with the reference's f_mean = mean(K0[0,0], K1[1,1], K0[0,0], K1[1,1]); an inlier has Sampson
error < t_n^2, evaluated as (x1^T E x0)^2 < t_n^2 * den.  Hypothesis k draws 5 distinct correspondences
(`draw_samples(..., size=5)`) and solves them with Nister's five-point method: the null basis of the 5 epipolar rows
from a Householder QR, the 10 x 20 cubic constraints, Gauss-Jordan with partial pivoting, the degree-10 determinant
of the hidden-variable matrix, its real roots by a Sturm chain and bisection (`sturm_roots`), (x, y) from the null
vector; solution j is real root j.  Every operation is one explicitly rounded fp64 operation (no FMA).  The winner has
the most inliers, then the lowest k, then the lowest j.  E is scaled to unit Frobenius norm (largest |entry| positive);
of its four (R, t) candidates the one with the most inliers in front of both cameras wins (depths from the 2 x 2 normal
equations of d1 x1 = d0 R x0 + t in (0, dist_thresh)).  No refit.  Fewer than 5 correspondences or no finite E makes
the pair invalid.

    estimate_fundamentals(res, thresh=3.0, n_hypotheses=2048, seed=0, min_overlap=0.5) -> FundamentalResult
        one `ltr_fundamental` call for every pair of a `match_images` / `match_sets` result, for pairs without
        intrinsics; device outputs, no synchronisation
    ransac_fundamental_host(kpts0, kpts1, matches_p, klines0, klines1, matches_l, pair=0, ...) -> dict
        the same model for one pair in numpy: everything up to the winner is the kernels' operations in the kernels'
        order; the refit uses np.linalg.eigh / svd

The fundamental-matrix model (DESIGN.md "Fundamental matrices", include/linetr_b200.h `ltr_fundamental`): x1^T F x0 = 0
in pixels.  The correspondences are the pair's matched side-0 keypoints in row order with their partners, normalised
per side as the homography's points.  Hypothesis k draws 7 distinct correspondences (`draw_samples(..., size=7)`) and
solves them with the seven-point method: the null basis F1, F2 of the 7 epipolar rows (the essential solver's QR), the
cubic det(F2 + a (F1 - F2)), its real roots by `sturm_roots`; solution j is real root j, denormalised and scaled to
unit Frobenius norm (largest |entry| positive).  A row is an inlier iff cv2's FM error (the larger squared distance to
the two epipolar lines) is below thresh^2.  The winner has the most inliers, then the lowest k, then the lowest j; with
at least 8 inliers it is refitted by the normalised eight-point method (rank 2 through the SVD), kept iff the refit has
at least as many inliers.  Matched key lines are then checked against the kept F (`lines_consistent`): the epipolar
band of each segment must overlap its partner by at least min_overlap of the shorter extent, on both sides.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

from . import _native as N
from . import _ops

FLT_EPSILON = float(np.finfo(np.float32).eps)
MAX_DRAWS = 64          # draws per hypothesis before it is rejected (HG_MAX_DRAWS)
PIVOT_MIN = 1e-12
# One pair's staging in shared memory (ltr_homography's capacity): bytes per keypoint / segment row and the limit.
SMEM_PER_POINT, SMEM_PER_LINE, SMEM_MAX = 18, 58, 200 * 1024
_U64 = np.uint64


# ------------------------------------------------------------------ the model in numpy
def splitmix64(x) -> np.ndarray:
    """splitmix64 of a uint64 array (wrapping arithmetic)."""
    z = np.asarray(x, dtype=_U64) + _U64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> _U64(30))) * _U64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> _U64(27))) * _U64(0x94D049BB133111EB)
    return z ^ (z >> _U64(31))


def draw_samples(seed: int, pair: int, n_hypotheses: int, n: int, size: int = 4):
    """The `size` correspondence indices of hypotheses 0..n_hypotheses-1 of `pair` among n (4 for a homography, 5 for
    an essential matrix): s = splitmix64(seed + splitmix64(pair << 32 | k)), draw j = splitmix64(s + j) mod n for
    j = 0, 1, ..., a duplicate redrawn with the next j.  -> (idx int64 [K, size], ok [K]); ok is False where MAX_DRAWS
    draws did not give `size` distinct indices."""
    k = np.arange(n_hypotheses, dtype=_U64)
    s = splitmix64(_U64(int(seed) & 0xFFFFFFFFFFFFFFFF) + splitmix64((_U64(pair) << _U64(32)) | k))
    idx = np.full((n_hypotheses, size), -1, dtype=np.int64)
    got = np.zeros(n_hypotheses, dtype=np.int64)
    rows = np.arange(n_hypotheses)
    for j in range(MAX_DRAWS):
        active = got < size
        if not active.any():
            break
        v = (splitmix64(s + _U64(j)) % _U64(n)).astype(np.int64)
        take = active & ~(idx == v[:, None]).any(1)
        idx[rows[take], got[take]] = v[take]
        got += take
    return idx, got == size


@dataclass
class _Norm:
    c0x: float
    c0y: float
    i0: float
    s0: float
    c1x: float
    c1y: float
    i1: float
    s1: float


def _side_norm(xy):
    """Centre, 1/scale and scale of one side's fp32 coordinates [m, 2] (m >= 1)."""
    lo, hi = xy.min(0).astype(np.float64), xy.max(0).astype(np.float64)
    c = (lo + hi) * 0.5
    w = hi - lo
    s = (w[0] if w[0] > w[1] else w[1]) * 0.5
    s = s if s > 0 else 1.0
    return float(c[0]), float(c[1]), 1.0 / s, s


def _normalisation(pts, seg0, seg1) -> _Norm:
    side0 = np.concatenate([pts[:, :2], seg0.reshape(-1, 2)])
    side1 = np.concatenate([pts[:, 2:], seg1.reshape(-1, 2)])
    c0x, c0y, i0, s0 = _side_norm(side0)
    c1x, c1y, i1, s1 = _side_norm(side1)
    return _Norm(c0x, c0y, i0, s0, c1x, c1y, i1, s1)


def _rows(pts, seg0, seg1, nm: _Norm) -> np.ndarray:
    """The two equation rows of every correspondence (points, then lines), normalised coordinates: [n, 2, 9]."""
    f = lambda a: np.asarray(a, dtype=np.float64)
    x, y = (f(pts[:, 0]) - nm.c0x) * nm.i0, (f(pts[:, 1]) - nm.c0y) * nm.i0
    u, v = (f(pts[:, 2]) - nm.c1x) * nm.i1, (f(pts[:, 3]) - nm.c1y) * nm.i1
    one, zero = np.ones_like(x), np.zeros_like(x)
    rp = np.stack([np.stack([x, y, one, zero, zero, zero, -(u * x), -(u * y), -u], 1),
                   np.stack([zero, zero, zero, x, y, one, -(v * x), -(v * y), -v], 1)], 1)
    ua, va = (f(seg1[:, 0, 0]) - nm.c1x) * nm.i1, (f(seg1[:, 0, 1]) - nm.c1y) * nm.i1
    ub, vb = (f(seg1[:, 1, 0]) - nm.c1x) * nm.i1, (f(seg1[:, 1, 1]) - nm.c1y) * nm.i1
    la, lb, lc = va - vb, ub - ua, ua * vb - ub * va
    r = 1.0 / np.sqrt(la * la + lb * lb)
    A, B, C = la * r, lb * r, lc * r
    rl = []
    for e in range(2):
        xe, ye = (f(seg0[:, e, 0]) - nm.c0x) * nm.i0, (f(seg0[:, e, 1]) - nm.c0y) * nm.i0
        rl.append(np.stack([A * xe, A * ye, A, B * xe, B * ye, B, C * xe, C * ye, C], 1))
    rl = np.stack(rl, 1) if len(seg0) else np.zeros((0, 2, 9))
    return np.concatenate([rp.reshape(-1, 2, 9), rl])


def _solve_minimal(rows8):
    """h (h33 = 1) of each [8, 9] system by Gaussian elimination with partial pivoting (first largest |pivot|):
    -> (h [K, 9], ok [K]); ok is False for a pivot below PIVOT_MIN or a non-finite result."""
    K = rows8.shape[0]
    A = np.concatenate([rows8[:, :, :8], -rows8[:, :, 8:]], 2)
    ok = np.ones(K, dtype=bool)
    ar = np.arange(K)
    for c in range(8):
        piv = np.full(K, c)
        best = np.abs(A[:, c, c])
        for r in range(c + 1, 8):
            v = np.abs(A[:, r, c])
            upd = v > best
            best, piv = np.where(upd, v, best), np.where(upd, r, piv)
        ok &= best >= PIVOT_MIN
        rc, rp = A[ar, c].copy(), A[ar, piv].copy()
        A[ar, c], A[ar, piv] = rp, rc
        for r in range(c + 1, 8):
            f = A[:, r, c] / A[:, c, c]
            A[:, r, c + 1:] = A[:, r, c + 1:] - f[:, None] * A[:, c, c + 1:]
    h = np.zeros((K, 9))
    h[:, 8] = 1.0
    for i in range(7, -1, -1):
        acc = A[:, i, 8].copy()
        for j in range(i + 1, 8):
            acc = acc - A[:, i, j] * h[:, j]
        h[:, i] = acc / A[:, i, i]
    return h, ok & np.isfinite(h).all(1)


def _to_pixels(h, nm: _Norm):
    """Normalised h [K, 9] -> pixel H = T1^-1 H^ T0 / H33 [K, 9] and ok (|H33| >= 1e-12 before the division, finite)."""
    t0x, t0y = -(nm.c0x * nm.i0), -(nm.c0y * nm.i0)
    M = np.empty_like(h)
    for i in range(3):
        M[:, 3 * i] = h[:, 3 * i] * nm.i0
        M[:, 3 * i + 1] = h[:, 3 * i + 1] * nm.i0
        M[:, 3 * i + 2] = (h[:, 3 * i] * t0x + h[:, 3 * i + 1] * t0y) + h[:, 3 * i + 2]
    G = np.empty_like(h)
    for j in range(3):
        G[:, j] = nm.s1 * M[:, j] + nm.c1x * M[:, 6 + j]
        G[:, 3 + j] = nm.s1 * M[:, 3 + j] + nm.c1y * M[:, 6 + j]
        G[:, 6 + j] = M[:, 6 + j]
    ok = np.abs(G[:, 8]) >= PIVOT_MIN
    H = G / np.where(ok, G[:, 8], 1.0)[:, None]
    return H, ok & np.isfinite(H).all(1)


def _project(H, x, y):
    w = H[:, 6:7] * x + H[:, 7:8] * y + H[:, 8:9]
    ok = np.abs(w) > FLT_EPSILON
    r = 1.0 / np.where(ok, w, 1.0)
    return (H[:, 0:1] * x + H[:, 1:2] * y + H[:, 2:3]) * r, (H[:, 3:4] * x + H[:, 4:5] * y + H[:, 5:6]) * r, ok


def pixel_lines(seg1) -> np.ndarray:
    """The line through every segment s1 [m, 2, 2] in pixels, scaled so that a^2 + b^2 = 1: [m, 3] fp64."""
    f = lambda a: np.asarray(a, dtype=np.float64)
    ax, ay, bx, by = f(seg1[:, 0, 0]), f(seg1[:, 0, 1]), f(seg1[:, 1, 0]), f(seg1[:, 1, 1])
    la, lb, lc = ay - by, bx - ax, ax * by - bx * ay
    r = 1.0 / np.sqrt(la * la + lb * lb)
    return np.stack([la * r, lb * r, lc * r], 1)


def residuals(H, pts, seg0, lines1):
    """Residuals [K, n] (squared pixels, points then lines) of pixel homographies H [K, 9]; inf where a projected
    |w| <= FLT_EPSILON."""
    f = lambda a: np.asarray(a, dtype=np.float64)[None, :]
    px, py, okp = _project(H, f(pts[:, 0]), f(pts[:, 1]))
    dx, dy = px - f(pts[:, 2]), py - f(pts[:, 3])
    ep = np.where(okp, dx * dx + dy * dy, np.inf)
    ax, ay, oka = _project(H, f(seg0[:, 0, 0]), f(seg0[:, 0, 1]))
    bx, by, okb = _project(H, f(seg0[:, 1, 0]), f(seg0[:, 1, 1]))
    la, lb, lc = (f(lines1[:, i]) for i in range(3))
    da, db = la * ax + lb * ay + lc, la * bx + lb * by + lc
    ea, eb = da * da, db * db
    el = np.where(oka & okb, np.where(ea > eb, ea, eb), np.inf)
    return np.concatenate([ep, el], 1)


def _inliers(H, pts, seg0, lines1, t2, chunk=256):
    out = np.empty((H.shape[0], len(pts) + len(seg0)), dtype=bool)
    for a in range(0, H.shape[0], chunk):
        with np.errstate(all="ignore"):
            out[a:a + chunk] = residuals(H[a:a + chunk], pts, seg0, lines1) < t2
    return out


def _correspondences(kpts0, kpts1, matches_p, klines0, klines1, matches_l, use_points, use_lines):
    """Compacted correspondences in the kernels' order: (pts [np, 4] fp32, seg0 [nl, 2, 2], seg1 [nl, 2, 2], row
    indices of the matched keypoint rows, of the matched segment rows)."""
    k0 = np.asarray(kpts0, dtype=np.float32).reshape(-1, 2)
    k1 = np.asarray(kpts1, dtype=np.float32).reshape(-1, 2)
    l0 = np.asarray(klines0, dtype=np.float32).reshape(-1, 2, 2)
    l1 = np.asarray(klines1, dtype=np.float32).reshape(-1, 2, 2)
    mp = np.asarray(matches_p, dtype=np.int64).reshape(-1)
    ml = np.asarray(matches_l, dtype=np.int64).reshape(-1)
    rp = np.flatnonzero((mp >= 0) & (mp < len(k1))) if use_points else np.zeros(0, dtype=np.int64)
    rl = np.flatnonzero((ml >= 0) & (ml < len(l1))) if use_lines else np.zeros(0, dtype=np.int64)
    pts = np.concatenate([k0[rp], k1[mp[rp]]], 1)
    return pts, l0[rl], l1[ml[rl]], rp, rl


def ransac_homography_host(kpts0, kpts1, matches_p, klines0, klines1, matches_l, pair=0, thresh=3.0,
                           n_hypotheses=2048, seed=0, use_lines=True, use_points=True) -> dict:
    """The estimator's model for one pair in numpy (see the module docstring).  kpts [N, 2], klines [K, 2, 2] (used as
    float32), matches_p [N0] / matches_l [K0]: local side-1 index or -1 per side-0 row; `pair` is the pair's index in
    the batch (it seeds the samples).  Returns H [3, 3] (NaN when invalid), valid, inliers_p uint8 [N0] / inliers_l
    uint8 [K0] aligned with the match rows, n_inliers_p / n_inliers_l, hypothesis (winning index or -1),
    hypothesis_inliers, H_hypothesis (the winner before the refit) and refit (whether the refit was kept)."""
    pts, seg0, seg1, rp, rl = _correspondences(kpts0, kpts1, matches_p, klines0, klines1, matches_l, use_points,
                                               use_lines)
    n_p, n = len(pts), len(pts) + len(seg0)
    out = dict(H=np.full((3, 3), np.nan), valid=False, inliers_p=np.zeros(len(np.ravel(matches_p)), dtype=np.uint8),
               inliers_l=np.zeros(len(np.ravel(matches_l)), dtype=np.uint8), n_inliers_p=0, n_inliers_l=0,
               hypothesis=-1, hypothesis_inliers=0, H_hypothesis=np.full((3, 3), np.nan), refit=False)
    if n < 4:
        return out
    t2 = float(thresh) * float(thresh)
    nm = _normalisation(pts, seg0, seg1)
    with np.errstate(all="ignore"):
        rows = _rows(pts, seg0, seg1, nm)
        lines1 = pixel_lines(seg1) if len(seg1) else np.zeros((0, 3))
        idx, ok = draw_samples(seed, pair, n_hypotheses, n)
        h, oks = _solve_minimal(rows[np.maximum(idx, 0)].reshape(n_hypotheses, 8, 9))
        Hk, okp = _to_pixels(h, nm)
    ok &= oks & okp
    cnt = np.where(ok, _inliers(np.where(ok[:, None], Hk, 0.0), pts, seg0, lines1, t2).sum(1), -1)
    k = int(np.argmax(cnt))
    if cnt[k] < 0:
        return out
    H, fl = Hk[k], _inliers(Hk[k:k + 1], pts, seg0, lines1, t2)[0]
    out.update(hypothesis=k, hypothesis_inliers=int(cnt[k]), H_hypothesis=H.reshape(3, 3).copy())
    if fl.sum() >= 4:
        A = rows[fl].reshape(-1, 9)
        _, V = np.linalg.eigh(A.T @ A)
        with np.errstate(all="ignore"):
            Hr, okr = _to_pixels(V[:, 0][None], nm)
        if okr[0]:
            flr = _inliers(Hr, pts, seg0, lines1, t2)[0]
            if flr.sum() >= fl.sum():
                H, fl = Hr[0], flr
                out["refit"] = True
    out["inliers_p"][rp] = fl[:n_p]
    out["inliers_l"][rl] = fl[n_p:]
    out.update(H=H.reshape(3, 3).copy(), valid=True, n_inliers_p=int(fl[:n_p].sum()), n_inliers_l=int(fl[n_p:].sum()))
    return out


# ------------------------------------------------------------------ batched on the GPU
@dataclass
class HomographyResult:
    """Result of `estimate_homographies` (device tensors; nothing has been waited for).

    H float64 [P, 3, 3] image 0 -> image 1 (NaN where not valid), valid bool [P], inliers_l / inliers_p uint8 aligned
    with the result's matches_l / matches_p (0 for unmatched rows), n_inliers_l / n_inliers_p int32 [P], hypothesis
    int32 [P] (index of the winning RANSAC hypothesis, -1 when not valid) and hypothesis_inliers int32 [P] (its inlier
    count before the refit)."""
    H: torch.Tensor
    valid: torch.Tensor
    inliers_l: torch.Tensor
    inliers_p: torch.Tensor
    n_inliers_l: torch.Tensor
    n_inliers_p: torch.Tensor
    hypothesis: torch.Tensor
    hypothesis_inliers: torch.Tensor


def _pool(items, P, to_rows):
    """Each distinct image once (by identity: `match_sets` results repeat the set's objects): -> (rows of the pool,
    first row of pair p's image [P], rows of pair p's image [P])."""
    first, parts, off, cnt, total = {}, [], np.zeros(P, dtype=np.int32), np.zeros(P, dtype=np.int32), 0
    for p, it in enumerate(items):
        if id(it) not in first:
            rows = to_rows(it)
            first[id(it)] = (total, len(rows))
            parts.append(rows)
            total += len(rows)
        off[p], cnt[p] = first[id(it)]
    return parts, off, cnt


def _stage_pairs(res, dev, who, lines, extra=None) -> dict:
    """The pair estimators' inputs of `res`: its side-0 / side-1 keypoints and, with `lines`, key lines (float32
    segments) pooled by `_pool`, their pool offsets and side-1 counts, the match offsets and the `extra` host arrays in
    one pinned copy.  -> device tensors and row bounds by input-struct field name (pts0 / pts1, pts_off0 / pts_off1,
    n_pts1, matches_p, cu_p, max_rows_p, with lines the same for segs, and the `extra` names)."""
    P = res.n_pairs
    op = np.asarray(res.offsets_p, dtype=np.int64)
    pt_rows = lambda k: torch.as_tensor(k).to(device=dev, dtype=torch.float32).reshape(-1, 2)
    p0, poff0, pn0 = _pool(res.keypoints0, P, pt_rows)
    p1, poff1, pn1 = _pool(res.keypoints1, P, pt_rows)
    arrays = {**(extra or {}), "pts_off0": poff0, "pts_off1": poff1, "n_pts1": pn1,
              "cu_p": np.ascontiguousarray(op, dtype=np.int32)}
    agree = np.array_equal(pn0, np.diff(op))
    if lines:
        ol = np.asarray(res.offsets_l, dtype=np.int64)
        seg_rows = lambda k: np.asarray(k, dtype=np.float32).reshape(-1, 4)
        s0, soff0, sn0 = _pool(res.klines0, P, seg_rows)
        s1, soff1, sn1 = _pool(res.klines1, P, seg_rows)
        agree &= np.array_equal(sn0, np.diff(ol))
        cat_np = lambda parts: np.concatenate(parts) if parts else np.zeros((0, 4), dtype=np.float32)
        arrays.update(segs0=cat_np(s0), segs1=cat_np(s1), seg_off0=soff0, seg_off1=soff1, n_segs1=sn1,
                      cu_l=np.ascontiguousarray(ol, dtype=np.int32))
    if not agree:
        raise N.LtrError(f"{who}: side-0 {'key lines / ' if lines else ''}keypoints and the match offsets disagree")
    dv = _ops.stage(arrays, dev)
    cat_t = lambda parts: torch.cat(parts) if parts else torch.zeros((0, 2), dtype=torch.float32, device=dev)
    dv.update(pts0=cat_t(p0).contiguous(), pts1=cat_t(p1).contiguous(), matches_p=res.matches_p.contiguous(),
              max_rows_p=int(np.diff(op).max(initial=0)))
    if lines:
        dv.update(matches_l=res.matches_l.contiguous(), max_rows_l=int(np.diff(ol).max(initial=0)))
    return dv


def estimate_homographies(res, thresh=3.0, n_hypotheses=2048, seed=0, use_lines=True, use_points=True) -> HomographyResult:
    """RANSAC homographies (image 0 -> image 1) of every pair of an `ImagePairMatches` (`match_images`, `match_sets`)
    from its line matches (res.klines0 / klines1 as float32 segments) and point matches (res.keypoints0 / keypoints1),
    in one `ltr_homography` call.  use_lines / use_points select the kinds of correspondence.  Host arrays go up in one
    pinned copy; the call never waits for the device.  Raises LtrError (LTR_E_UNSUPPORTED) when a pair has more match
    rows than one CTA can stage (SMEM_PER_POINT / SMEM_PER_LINE bytes per row, SMEM_MAX in all)."""
    P = res.n_pairs
    dev = res.matches_l.device
    if int(n_hypotheses) < 1:
        raise N.LtrError("estimate_homographies: n_hypotheses must be >= 1")
    dv = _stage_pairs(res, dev, "estimate_homographies", lines=True)
    u8, i32d = dict(dtype=torch.uint8, device=dev), dict(dtype=torch.int32, device=dev)
    out = HomographyResult(torch.empty((P, 3, 3), dtype=torch.float64, device=dev), torch.empty(P, **u8),
                           torch.empty(res.matches_l.shape[0], **u8), torch.empty(res.matches_p.shape[0], **u8),
                           torch.empty(P, **i32d), torch.empty(P, **i32d), torch.empty(P, **i32d),
                           torch.empty(P, **i32d))
    _ops.call_struct("ltr_homography", {**dv, "n_pairs": P, "thresh": thresh, "n_hypotheses": n_hypotheses,
                                        "seed": seed, "use_points": use_points, "use_lines": use_lines},
                     {**vars(out), "key": torch.empty(P, dtype=torch.int64, device=dev)})
    out.valid = out.valid.view(torch.bool)
    return out


# ------------------------------------------------------------------ metric
def homography_corner_error(H_est, H_gt, shapes) -> dict:
    """The homography-estimation metric: per pair, the mean distance between the four image corners (0, 0),
    (0, h-1), (w-1, 0), (w-1, h-1) mapped by H_est and by H_gt ([P, 3, 3] or [3, 3]; shapes: (h, w) or [P, 2]).
    Returns 'error' float64 [P] (inf where H_est is not finite or maps a corner to infinity), 'mean_error' over the
    pairs with a finite error, and 'accuracy_1' / 'accuracy_3' / 'accuracy_5': the fraction of all pairs with error
    <= 1 / 3 / 5 px."""
    He = np.asarray(H_est.cpu() if isinstance(H_est, torch.Tensor) else H_est, dtype=np.float64).reshape(-1, 3, 3)
    Hg = np.asarray(H_gt, dtype=np.float64).reshape(-1, 3, 3)
    P = max(len(He), len(Hg))
    hw = np.broadcast_to(np.asarray(shapes, dtype=np.float64).reshape(-1, 2), (P, 2))
    h, w = hw[:, 0] - 1, hw[:, 1] - 1
    z = np.zeros(P)
    c = np.stack([np.stack([z, z], 1), np.stack([z, h], 1), np.stack([w, z], 1), np.stack([w, h], 1)], 1)   # [P,4,2]
    ch = np.concatenate([c, np.ones((P, 4, 1))], 2)

    def warp(Hs):
        q = np.einsum("pij,pcj->pci", np.broadcast_to(Hs, (P, 3, 3)), ch)
        return q[..., :2] / q[..., 2:]

    with np.errstate(all="ignore"):
        err = np.linalg.norm(warp(He) - warp(Hg), axis=2).mean(1)
    err = np.where(np.isfinite(err), err, np.inf)
    fin = np.isfinite(err)
    out = {"error": err, "mean_error": float(err[fin].mean()) if fin.any() else float("inf")}
    for t in (1, 3, 5):
        out[f"accuracy_{t}"] = float(np.mean(err <= t)) if P else 0.0
    return out


# ------------------------------------------------------------------ relative pose: the model in numpy
# DESIGN.md "Relative pose"; the kernels are csrc/essential.cuh.  Every step up to the winner is one IEEE fp64 operation
# per numpy elementwise operation (no FMA, no reductions whose order numpy chooses), in the kernels' order.
ESS_SAMPLE = 5
ESS_MAX_ROOTS = 10
ESS_RANK_EPS = 1e-10      # a sample whose QR column norm falls below this times the first one's is rejected
ESS_ROOT_BOUND = 1e8      # real roots are searched in [-B, B], B = min(Cauchy bound, ESS_ROOT_BOUND)
ESS_BISECT_STEPS = 100
# One pair's staging in shared memory (ltr_essential's capacity): 32 bytes of normalised fp64 coordinates plus one
# inlier flag byte per keypoint row.
SMEM_PER_ROW_E = 33

# Products of the monomials in (x, y, z): degree 1 [x, y, z, 1], degree 2 [x^2, xy, xz, x, y^2, yz, y, z^2, z, 1],
# degree 3 in the elimination order [x^3, y^3, x^2y, xy^2, x^2z, x^2, y^2z, y^2, xyz, xy | xz^2, xz, x, yz^2, yz, y,
# z^3, z^2, z, 1] (csrc/essential.cuh ESS_MUL11 / ESS_MUL21).
_MUL11 = ((0, 1, 2, 3), (1, 4, 5, 6), (2, 5, 7, 8), (3, 6, 8, 9))
_MUL21 = ((0, 2, 4, 5), (2, 3, 8, 9), (4, 8, 10, 11), (5, 9, 11, 12), (3, 1, 6, 7), (8, 6, 13, 14), (9, 7, 14, 15),
          (10, 13, 16, 17), (11, 14, 17, 18), (12, 15, 18, 19))


def _normalised(kpts, K):
    """Pixel keypoints (used as float32) -> normalised fp64 coordinates (k - c) / f per axis."""
    k = np.asarray(kpts, dtype=np.float32).astype(np.float64).reshape(-1, 2)
    K = np.asarray(K, dtype=np.float64)
    return np.stack([(k[:, 0] - K[0, 2]) / K[0, 0], (k[:, 1] - K[1, 2]) / K[1, 1]], 1)


def _f_mean(K0, K1):
    """The reference's mean focal length (models/utils.py:295: K0[0,0], K1[1,1] twice each), summed in order."""
    return (((K0[0, 0] + K1[1, 1]) + K0[0, 0]) + K1[1, 1]) / 4.0


def _mul(a, b, table, n_out):
    """Product of polynomials in (x, y, z) given as coefficient arrays [K, len] in the monomial orders above."""
    out = np.zeros((a.shape[0], n_out))
    for i in range(a.shape[1]):
        for j in range(b.shape[1]):
            m = table[i][j]
            out[:, m] = out[:, m] + a[:, i] * b[:, j]
    return out


def _pmul(a, b):
    """Product of polynomials in z, ascending coefficients [K, la] x [K, lb] -> [K, la + lb - 1]."""
    out = np.zeros((a.shape[0], a.shape[1] + b.shape[1] - 1))
    for i in range(a.shape[1]):
        for j in range(b.shape[1]):
            out[:, i + j] = out[:, i + j] + a[:, i] * b[:, j]
    return out


def _null_basis(q):
    """Null-space basis of the S epipolar rows of each sample (S = 5 for an essential matrix, 7 for a fundamental
    matrix): q [K, S, 4] normalised (a0, b0, a1, b1) -> (basis [K, 9 - S, 9] = Q e_S .. Q e_8 of the Householder QR of
    the 9 x S transpose, ok [K]) (csrc/ransac_common.cuh rc_null_basis)."""
    K, S = q.shape[0], q.shape[1]
    a0, b0, a1, b1 = (q[:, :, i] for i in range(4))
    M = np.stack([a1 * a0, a1 * b0, a1, b1 * a0, b1 * b0, b1, a0, b0, np.ones_like(a0)], 1)   # [K, 9, S]
    ok = np.ones(K, dtype=bool)
    vs, betas, nrm0 = [], [], None
    for c in range(S):
        acc = np.zeros(K)
        for i in range(c, 9):
            acc = acc + M[:, i, c] * M[:, i, c]
        nrm = np.sqrt(acc)
        if c == 0:
            nrm0 = nrm
            ok &= nrm > 0
        else:
            ok &= nrm > ESS_RANK_EPS * nrm0
        alpha = np.where(M[:, c, c] >= 0, -nrm, nrm)
        v = M[:, c:, c].copy()
        v[:, 0] = M[:, c, c] - alpha
        vtv = np.zeros(K)
        for i in range(9 - c):
            vtv = vtv + v[:, i] * v[:, i]
        beta = np.where(vtv > 0, 2.0 / np.where(vtv > 0, vtv, 1.0), 0.0)
        for j in range(c + 1, S):
            s = np.zeros(K)
            for i in range(9 - c):
                s = s + v[:, i] * M[:, c + i, j]
            g = s * beta
            for i in range(9 - c):
                M[:, c + i, j] = M[:, c + i, j] - g * v[:, i]
        vs.append(v)
        betas.append(beta)
    basis = np.zeros((K, 9 - S, 9))
    for b in range(9 - S):
        y = np.zeros((K, 9))
        y[:, S + b] = 1.0
        for c in range(S - 1, -1, -1):
            v = vs[c]
            s = np.zeros(K)
            for i in range(9 - c):
                s = s + v[:, i] * y[:, c + i]
            g = s * betas[c]
            for i in range(9 - c):
                y[:, c + i] = y[:, c + i] - g * v[:, i]
        basis[:, b] = y
    return basis, ok


def _constraints(basis):
    """The 10 x 20 cubic constraints (det E = 0, then 2 E E^T E - tr(E E^T) E = 0 row-major) of E = x X + y Y + z Z + W
    in the degree-3 monomial order: [K, 10, 20]."""
    e = [basis[:, :, i] for i in range(9)]          # entry i of E as a polynomial [x, y, z, 1]: [K, 4]
    m11 = lambda a, b: _mul(a, b, _MUL11, 10)
    m21 = lambda a, b: _mul(a, b, _MUL21, 20)
    det = (m21(m11(e[4], e[8]) - m11(e[5], e[7]), e[0]) - m21(m11(e[3], e[8]) - m11(e[5], e[6]), e[1])) \
        + m21(m11(e[3], e[7]) - m11(e[4], e[6]), e[2])
    eet = {}
    for i in range(3):
        for k in range(i, 3):
            eet[i, k] = eet[k, i] = (m11(e[3 * i], e[3 * k]) + m11(e[3 * i + 1], e[3 * k + 1])) \
                + m11(e[3 * i + 2], e[3 * k + 2])
    tr = (eet[0, 0] + eet[1, 1]) + eet[2, 2]
    L = {(i, k): eet[i, k] * 2.0 - tr if i == k else eet[i, k] * 2.0 for i in range(3) for k in range(3)}
    rows = [det]
    for i in range(3):
        for j in range(3):
            rows.append((m21(L[i, 0], e[j]) + m21(L[i, 1], e[3 + j])) + m21(L[i, 2], e[6 + j]))
    return np.stack(rows, 1)


def _gauss_jordan(C):
    """Gauss-Jordan elimination of the first 10 columns with partial pivoting (first largest |pivot|): -> (the last 10
    columns of the reduced rows [K, 10, 10], ok [K]: every pivot > 0)."""
    C = C.copy()
    K = C.shape[0]
    ok = np.ones(K, dtype=bool)
    ar = np.arange(K)
    for c in range(10):
        piv = np.full(K, c)
        best = np.abs(C[:, c, c])
        for r in range(c + 1, 10):
            v = np.abs(C[:, r, c])
            upd = v > best
            best, piv = np.where(upd, v, best), np.where(upd, r, piv)
        ok &= best > 0
        rc, rp = C[ar, c].copy(), C[ar, piv].copy()
        C[ar, c], C[ar, piv] = rp, rc
        p = C[:, c, c].copy()
        C[:, c, c + 1:] = C[:, c, c + 1:] / p[:, None]
        for r in range(10):
            if r != c:
                f = C[:, r, c].copy()
                C[:, r, c + 1:] = C[:, r, c + 1:] - f[:, None] * C[:, c, c + 1:]
    return C[:, :, 10:], ok


def _hidden_matrix(R):
    """The 3 x 3 matrix of polynomials in z (ascending coefficients) whose null vector is (x, y, 1): rows from
    x^2z - z x^2, y^2z - z y^2, xyz - z xy.  -> [[bx, by, b1] per row] with bx, by [K, 4] and b1 [K, 5]."""
    B = []
    for u, l in ((4, 5), (6, 7), (8, 9)):
        ru, rl = R[:, u], R[:, l]
        bx = np.stack([-ru[:, 2], rl[:, 2] - ru[:, 1], rl[:, 1] - ru[:, 0], rl[:, 0]], 1)
        by = np.stack([-ru[:, 5], rl[:, 5] - ru[:, 4], rl[:, 4] - ru[:, 3], rl[:, 3]], 1)
        b1 = np.stack([-ru[:, 9], rl[:, 9] - ru[:, 8], rl[:, 8] - ru[:, 7], rl[:, 7] - ru[:, 6], rl[:, 6]], 1)
        B.append([bx, by, b1])
    return B


def _det_poly(B):
    """det B(z), degree 10, ascending coefficients [K, 11]."""
    t0 = _pmul(B[0][0], _pmul(B[1][1], B[2][2]) - _pmul(B[1][2], B[2][1]))
    t1 = _pmul(B[0][1], _pmul(B[1][0], B[2][2]) - _pmul(B[1][2], B[2][0]))
    t2 = _pmul(B[0][2], _pmul(B[1][0], B[2][1]) - _pmul(B[1][1], B[2][0]))
    return (t0 - t1) + t2


def _maxabs(p):
    m = np.zeros(p.shape[0])
    for i in range(p.shape[1]):
        a = np.abs(p[:, i])
        m = np.where(a > m, a, m)
    return m


def _horner(c, x):
    """Polynomial with ascending coefficients c [K, n] at x [K, ...] (one multiply, then one add, per step)."""
    sh = (-1,) + (1,) * (x.ndim - 1)
    v = np.broadcast_to(c[:, -1].reshape(sh), x.shape).copy()
    for i in range(c.shape[1] - 2, -1, -1):
        v = v * x + c[:, i].reshape(sh)
    return v


def _sign_changes(chain, length, x):
    """Sign changes of the Sturm chain at x [K, m] (zeros and NaNs skipped), over its first length[K] members."""
    K = x.shape[0]
    prev = np.zeros(x.shape, dtype=np.int8)
    n = np.zeros(x.shape, dtype=np.int64)
    for k, c in enumerate(chain):
        v = _horner(c, x)
        s = (v > 0).astype(np.int8) - (v < 0).astype(np.int8)
        live = (s != 0) & (k < length.reshape(K, *([1] * (x.ndim - 1))))
        n += live & (prev != 0) & (s != prev)
        prev = np.where(live, s, prev)
    return n


def _degree(c):
    """Degree of each polynomial c [K, n] (ascending): the highest index with a non-zero coefficient, 0 for a
    constant."""
    nz = c != 0
    return np.where(nz.any(1), c.shape[1] - 1 - np.argmax(nz[:, ::-1], 1), 0)


def sturm_roots(p):
    """The real roots of polynomials of degree 1 to 10 (ascending coefficients p [K, 11], exact-zero leading
    coefficients stripped) in [-B, B], B = min(Cauchy bound, ESS_ROOT_BOUND), with the kernels' operation sequence:
    the Sturm chain of p (each member's remainder by long division, stripped of exact-zero leading coefficients and
    divided by its largest |coefficient|; the chain ends at a constant or before a zero remainder), then per root
    index i < (number of distinct real roots) ESS_BISECT_STEPS bisection steps on "roots below mid > i".  A constant
    or a non-finite coefficient has no roots.  -> (roots [K, 10] ascending, NaN past the count, count [K])."""
    p = np.asarray(p, dtype=np.float64)
    K = p.shape[0]
    ar = np.arange(K)
    with np.errstate(all="ignore"):
        m = _maxabs(p)
        ok = (m > 0) & np.isfinite(p).all(1)
        s0 = p / np.where(ok, m, 1.0)[:, None]
        n = _degree(s0)
        ok &= n > 0
        lead = s0[ar, n]
        bound = np.ones(K)
        for i in range(10):
            a = np.abs(s0[:, i] / lead)
            bound = np.where((i < n) & (a + 1.0 > bound), a + 1.0, bound)
        bound = np.where(bound < ESS_ROOT_BOUND, bound, ESS_ROOT_BOUND)
        ok &= bound == bound
        d = np.stack([s0[:, i + 1] * float(i + 1) for i in range(10)], 1)
        md = _maxabs(d)
        chain = [s0, d / np.where(md > 0, md, 1.0)[:, None]]
        length = np.where(ok, 2, 0)
        # members k - 1 (degree da) and k (degree db < da) give member k + 1 (csrc/essential.cuh ess_roots)
        da, db = n, _degree(chain[1])
        for k in range(1, 10):
            A, Bp = chain[k - 1], chain[k]
            go = (length == k + 1) & (db > 0)
            lead = Bp[ar, np.minimum(db, 10 - k)]      # (rows whose chain has ended read any coefficient)
            T = np.zeros((K, 11))
            T[:, :A.shape[1]] = A
            for j in range(10, 0, -1):
                act = go & (j <= da) & (j >= db)
                q = T[ar, j] / lead
                for i in range(10 - k):
                    col = np.where(act & (i < db), j - db + i, 0)
                    upd = T[ar, col] - q * Bp[:, i]
                    T[ar, col] = np.where(act & (i < db), upd, T[ar, col])
            r = np.stack([np.where(i < db, -T[:, i], 0.0) for i in range(10 - k)], 1)
            mr = _maxabs(r)
            go &= mr > 0
            chain.append(r / np.where(go, mr, 1.0)[:, None])
            length = np.where(go, k + 2, length)
            da, db = np.where(go, db, da), np.where(go, _degree(chain[-1]), db)
        lo0 = -bound
        v_lo = _sign_changes(chain, length, lo0[:, None])[:, 0]
        v_hi = _sign_changes(chain, length, bound[:, None])[:, 0]
        count = np.clip(v_lo - v_hi, 0, 10)
        count = np.where(ok, count, 0)
        idx = np.arange(10)[None, :]
        lo = np.broadcast_to(lo0[:, None], (K, 10)).copy()
        hi = np.broadcast_to(bound[:, None], (K, 10)).copy()
        live = idx < count[:, None]
        for _ in range(ESS_BISECT_STEPS):
            mid = (lo + hi) * 0.5
            act = live & (mid > lo) & (mid < hi)
            if not act.any():
                break
            below = v_lo[:, None] - _sign_changes(chain, length, mid)
            up = below > idx
            hi = np.where(act & up, mid, hi)
            lo = np.where(act & ~up, mid, lo)
        roots = np.where(live, (lo + hi) * 0.5, np.nan)
    return roots, count


def _back_substitute(B, basis, z):
    """E of every root z [K, 10]: (x, y, 1) from the cross product of two rows of B(z) (the pair whose third component
    is largest in magnitude, first on a tie), E = ((x X + y Y) + z Z) + W.  -> (E [K, 10, 9], ok [K, 10])."""
    rows = [[_horner(B[r][c], z) for c in range(3)] for r in range(3)]

    def cross(a, b):
        return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])

    best = cross(rows[0], rows[1])
    for a, b in ((0, 2), (1, 2)):
        c = cross(rows[a], rows[b])
        upd = np.abs(c[2]) > np.abs(best[2])
        best = tuple(np.where(upd, c[i], best[i]) for i in range(3))
    ok = np.abs(best[2]) > 0
    x, y = best[0] / best[2], best[1] / best[2]
    X, Y, Z, W = (basis[:, b, None, :] for b in range(4))
    E = ((x[..., None] * X + y[..., None] * Y) + z[..., None] * Z) + W
    return E, ok & np.isfinite(E).all(-1)


def essential_solutions(q):
    """The five-point solver (DESIGN.md "Relative pose") on samples q [K, 5, 4] of normalised correspondences
    (a0, b0, a1, b1): -> (E [K, 10, 9] row-major, ok [K, 10]); solution j of sample k is real root j of det B(z)."""
    q = np.asarray(q, dtype=np.float64)
    with np.errstate(all="ignore"):
        basis, ok = _null_basis(q)
        R, okg = _gauss_jordan(_constraints(basis))
        B = _hidden_matrix(R)
        roots, count = sturm_roots(_det_poly(B))
        E, oke = _back_substitute(B, basis, np.where(np.isnan(roots), 0.0, roots))
    return E, oke & (ok & okg)[:, None] & ~np.isnan(roots)


def sampson_inliers(E, q, t2, chunk=512):
    """Inlier flags [M, n] of essential matrices E [M, 9] on normalised correspondences q [n, 4]: (x1^T E x0)^2 <
    t2 * ((E x0)_0^2 + (E x0)_1^2 + (E^T x1)_0^2 + (E^T x1)_1^2), i.e. Sampson error < t2 without the division."""
    a0, b0, a1, b1 = (q[None, :, i] for i in range(4))
    out = np.empty((E.shape[0], q.shape[0]), dtype=bool)
    with np.errstate(all="ignore"):
        for s in range(0, E.shape[0], chunk):
            e = [E[s:s + chunk, i:i + 1] for i in range(9)]
            u0 = (e[0] * a0 + e[1] * b0) + e[2]
            u1 = (e[3] * a0 + e[4] * b0) + e[5]
            u2 = (e[6] * a0 + e[7] * b0) + e[8]
            w0 = (e[0] * a1 + e[3] * b1) + e[6]
            w1 = (e[1] * a1 + e[4] * b1) + e[7]
            num = (a1 * u0 + b1 * u1) + u2
            den = ((u0 * u0 + u1 * u1) + w0 * w0) + w1 * w1
            out[s:s + chunk] = num * num < t2 * den
    return out


def sampson_error(E, q):
    """Sampson error [n] of one essential matrix E [9] on normalised correspondences q [n, 4] (fp64)."""
    E = np.asarray(E, dtype=np.float64).reshape(3, 3)
    x0 = np.concatenate([q[:, :2], np.ones((len(q), 1))], 1)
    x1 = np.concatenate([q[:, 2:], np.ones((len(q), 1))], 1)
    Ex0, Etx1 = x0 @ E.T, x1 @ E
    num = np.sum(x1 * Ex0, 1)
    return num * num / (Ex0[:, 0] ** 2 + Ex0[:, 1] ** 2 + Etx1[:, 0] ** 2 + Etx1[:, 1] ** 2)


def decompose_essential(E):
    """The four (R, t) candidates of E [3, 3] in OpenCV's order (R1, t), (R2, t), (R1, -t), (R2, -t)."""
    U, _, Vt = np.linalg.svd(np.asarray(E, dtype=np.float64).reshape(3, 3))
    if np.linalg.det(U) < 0:
        U = -U
    if np.linalg.det(Vt) < 0:
        Vt = -Vt
    W = np.array([[0.0, 1.0, 0.0], [-1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    R1, R2, t = U @ W @ Vt, U @ W.T @ Vt, U[:, 2]
    return [(R1, t), (R2, t), (R1, -t), (R2, -t)]


def cheirality(R, t, q, dist_thresh=1e9):
    """Rows of q [n, 4] in front of both cameras: depths (d0, d1) of d1 x1 = d0 R x0 + t from the 2 x 2 normal
    equations, 0 < d0 < dist_thresh and 0 < d1 < dist_thresh."""
    x0 = np.concatenate([q[:, :2], np.ones((len(q), 1))], 1)
    x1 = np.concatenate([q[:, 2:], np.ones((len(q), 1))], 1)
    a, b = x0 @ np.asarray(R).T, x1
    aa, ab, bb = (a * a).sum(1), (a * b).sum(1), (b * b).sum(1)
    at, bt = a @ t, b @ t
    with np.errstate(all="ignore"):
        det = ab * ab - aa * bb
        d0, d1 = (at * bb - ab * bt) / det, (ab * at - aa * bt) / det
    return (d0 > 0) & (d0 < dist_thresh) & (d1 > 0) & (d1 < dist_thresh)


def unit_essential(E):
    """E [9] scaled to unit Frobenius norm, the sign making its largest-magnitude entry (the first on a tie) positive."""
    E = np.asarray(E, dtype=np.float64).reshape(9)
    E = E / np.sqrt(np.sum(E * E))
    return E if E[int(np.argmax(np.abs(E)))] > 0 else -E


def ransac_essential_host(kpts0, kpts1, matches_p, K0, K1, pair=0, thresh=1.0, n_hypotheses=1024, seed=0,
                          dist_thresh=1e9) -> dict:
    """The relative-pose estimator's model for one pair in numpy (DESIGN.md "Relative pose").  kpts [N, 2] (used as
    float32), matches_p [N0]: local side-1 index or -1 per side-0 row, K0 / K1 [3, 3] fp64; `pair` is the pair's index
    in the batch (it seeds the samples).  Returns E [3, 3] (unit Frobenius norm), R [3, 3], t [3] (unit; all NaN when
    invalid), valid, inliers_p uint8 [N0] aligned with the match rows, n_inliers, n_cheirality (inliers in front of
    both cameras under the chosen (R, t)), hypothesis (10 k + j of the winning sample k and root j, or -1),
    hypothesis_inliers and E_hypothesis (the winning solution before scaling)."""
    k0 = np.asarray(kpts0, dtype=np.float32).reshape(-1, 2)
    k1 = np.asarray(kpts1, dtype=np.float32).reshape(-1, 2)
    mp = np.asarray(matches_p, dtype=np.int64).reshape(-1)
    K0, K1 = np.asarray(K0, dtype=np.float64), np.asarray(K1, dtype=np.float64)
    rp = np.flatnonzero((mp >= 0) & (mp < len(k1)))
    out = dict(E=np.full((3, 3), np.nan), R=np.full((3, 3), np.nan), t=np.full(3, np.nan), valid=False,
               inliers_p=np.zeros(len(mp), dtype=np.uint8), n_inliers=0, n_cheirality=0, hypothesis=-1,
               hypothesis_inliers=0, E_hypothesis=np.full((3, 3), np.nan))
    n = len(rp)
    if n < ESS_SAMPLE:
        return out
    q = np.concatenate([_normalised(k0[rp], K0), _normalised(k1[mp[rp]], K1)], 1)
    tn = float(thresh) / _f_mean(K0, K1)
    t2 = tn * tn
    idx, ok = draw_samples(seed, pair, n_hypotheses, n, ESS_SAMPLE)
    E, oke = essential_solutions(q[np.maximum(idx, 0)])
    oke &= ok[:, None]
    flat = np.flatnonzero(oke.reshape(-1))
    if not len(flat):
        return out
    cnt = sampson_inliers(E.reshape(-1, 9)[flat], q, t2).sum(1)
    # the kernels' key: (count << 32) | ~(10 k + j); flat = 10 k + j
    w = int(flat[np.lexsort((flat, -cnt))[0]])
    Ew = E.reshape(-1, 9)[w]
    fl = sampson_inliers(Ew[None], q, t2)[0]
    Eu = unit_essential(Ew)
    best, R, t = -1, None, None
    for Rc, tc in decompose_essential(Eu):
        c = int(cheirality(Rc, tc, q[fl], dist_thresh).sum())
        if c > best:
            best, R, t = c, Rc, tc
    out["inliers_p"][rp] = fl
    out.update(E=Eu.reshape(3, 3), R=R, t=t / np.linalg.norm(t), valid=True, n_inliers=int(fl.sum()),
               n_cheirality=best, hypothesis=w, hypothesis_inliers=int(fl.sum()), E_hypothesis=Ew.reshape(3, 3).copy())
    return out


# ------------------------------------------------------------------ relative pose, batched on the GPU
@dataclass
class PoseResult:
    """Result of `estimate_poses` (device tensors; nothing has been waited for).

    E float64 [P, 3, 3] (x1^T E x0 = 0 in normalised coordinates, unit Frobenius norm), R float64 [P, 3, 3] and t
    float64 [P, 3] (unit) with X1 = R X0 + t (all NaN where not valid), valid bool [P], inliers uint8 aligned with the
    result's matches_p (0 for unmatched rows), n_inliers int32 [P], n_cheirality int32 [P] (inliers in front of both
    cameras under (R, t)), hypothesis int32 [P] (10 k + j of the winning sample k and root j, -1 when not valid) and
    hypothesis_inliers int32 [P]."""
    E: torch.Tensor
    R: torch.Tensor
    t: torch.Tensor
    valid: torch.Tensor
    inliers: torch.Tensor
    n_inliers: torch.Tensor
    n_cheirality: torch.Tensor
    hypothesis: torch.Tensor
    hypothesis_inliers: torch.Tensor


def _intrinsics(K, P, name):
    K = np.asarray(K.cpu() if isinstance(K, torch.Tensor) else K, dtype=np.float64)
    if K.shape not in ((3, 3), (P, 3, 3)):
        raise N.LtrError(f"estimate_poses: {name} must be [3, 3] or [{P}, 3, 3], got {list(K.shape)}")
    K = np.ascontiguousarray(np.broadcast_to(K, (P, 3, 3)))
    if not np.isfinite(K).all() or not ((K[:, 0, 0] > 0) & (K[:, 1, 1] > 0)).all():
        raise N.LtrError(f"estimate_poses: {name} must be finite with fx, fy > 0")
    return K


def estimate_poses(res, K0, K1, thresh=1.0, n_hypotheses=1024, seed=0, dist_thresh=1e9) -> PoseResult:
    """Relative pose of every pair of an `ImagePairMatches` (`match_images`, `match_sets`) from its point matches
    (res.keypoints0 / keypoints1 in pixels): five-point RANSAC essential matrices and the pose, in one `ltr_essential`
    call (the batched form of the reference's estimate_pose, models/utils.py:291-315).  K0 / K1: intrinsics of side 0
    / side 1, [3, 3] for every pair or [P, 3, 3]; thresh in pixels, scaled by the reference's mean focal length.  Host
    arrays go up in one pinned copy; the call never waits for the device.  Raises LtrError for non-finite K or K with
    fx / fy <= 0, and (LTR_E_UNSUPPORTED) when a pair has more match rows than one CTA can stage (SMEM_PER_ROW_E bytes
    per row, SMEM_MAX in all)."""
    P = res.n_pairs
    dev = res.matches_p.device
    if int(n_hypotheses) < 1:
        raise N.LtrError("estimate_poses: n_hypotheses must be >= 1")
    k0, k1 = _intrinsics(K0, P, "K0"), _intrinsics(K1, P, "K1")
    dv = _stage_pairs(res, dev, "estimate_poses", lines=False, extra={"K0": k0, "K1": k1})
    f64, i32 = dict(dtype=torch.float64, device=dev), dict(dtype=torch.int32, device=dev)
    out = PoseResult(torch.empty((P, 3, 3), **f64), torch.empty((P, 3, 3), **f64), torch.empty((P, 3), **f64),
                     torch.empty(P, dtype=torch.uint8, device=dev),
                     torch.empty(res.matches_p.shape[0], dtype=torch.uint8, device=dev),
                     torch.empty(P, **i32), torch.empty(P, **i32), torch.empty(P, **i32), torch.empty(P, **i32))
    outputs = {**vars(out), "inliers_p": out.inliers, "key": torch.empty(P, dtype=torch.int64, device=dev)}
    del outputs["inliers"]
    _ops.call_struct("ltr_essential", {**dv, "n_pairs": P, "thresh": thresh, "dist_thresh": dist_thresh,
                                       "n_hypotheses": n_hypotheses, "seed": seed}, outputs)
    out.valid = out.valid.view(torch.bool)
    return out


# ------------------------------------------------------------------ fundamental matrices: the model in numpy
# DESIGN.md "Fundamental matrices"; the kernels are csrc/fundamental.cuh.  As for the essential model, every step up to
# the winner is one IEEE fp64 operation per numpy elementwise operation, in the kernels' order.
FM_SAMPLE = 7
FM_MAX_SOLUTIONS = 3
FM_MIN_REFIT = 8          # winner inliers needed for the eight-point refit
# One pair's staging in shared memory (ltr_fundamental's capacity): 16 bytes of fp32 pixel coordinates plus two inlier
# flag bytes per keypoint row.
SMEM_PER_ROW_F = 18


def fundamental_cubic(basis):
    """det(F2 + a (F1 - F2)) of null bases [K, 2, 9] (F1, F2 row-major) as ascending coefficients [K, 4], expanded
    along the first row: (c0 (c4 c8 - c5 c7) - c1 (c3 c8 - c5 c6)) + c2 (c3 c7 - c4 c6), with c_i = [F2_i, F1_i - F2_i]
    the entries as polynomials in a.  -> (coefficients, F2 [K, 9], F1 - F2 [K, 9])."""
    F1, F2 = basis[:, 0], basis[:, 1]
    D = F1 - F2
    c = [np.stack([F2[:, i], D[:, i]], 1) for i in range(9)]
    t0 = _pmul(c[0], _pmul(c[4], c[8]) - _pmul(c[5], c[7]))
    t1 = _pmul(c[1], _pmul(c[3], c[8]) - _pmul(c[5], c[6]))
    t2 = _pmul(c[2], _pmul(c[3], c[7]) - _pmul(c[4], c[6]))
    return (t0 - t1) + t2, F2, D


def fundamental_solutions(q):
    """The seven-point solver (DESIGN.md "Fundamental matrices") on samples q [K, 7, 4] of normalised correspondences
    (x0, y0, x1, y1): -> (F^ [K, 3, 9] row-major in normalised coordinates, ok [K, 3]); solution j of sample k is
    F2 + a_j (F1 - F2) for real root a_j (ascending) of the cubic.  The solution at a = infinity (F1 - F2 singular on
    its own) is not returned."""
    q = np.asarray(q, dtype=np.float64)
    K = q.shape[0]
    with np.errstate(all="ignore"):
        basis, ok = _null_basis(q)
        cubic, F2, D = fundamental_cubic(basis)
        p = np.zeros((K, 11))
        p[:, :4] = cubic
        roots, _ = sturm_roots(p)
        a = roots[:, :FM_MAX_SOLUTIONS]
        F = F2[:, None, :] + np.where(np.isnan(a), 0.0, a)[..., None] * D[:, None, :]
    return F, ok[:, None] & ~np.isnan(a) & np.isfinite(F).all(-1)


def _fundamental_to_pixels(f, nm: _Norm):
    """Normalised F^ [..., 9] -> pixel F = T1^T F^ T0 scaled to unit Frobenius norm, its largest |entry| (the first on a
    tie) positive; ok is False for a zero or non-finite norm."""
    t0x, t0y = -(nm.c0x * nm.i0), -(nm.c0y * nm.i0)
    t1x, t1y = -(nm.c1x * nm.i1), -(nm.c1y * nm.i1)
    M, G = np.empty_like(f), np.empty_like(f)
    for i in range(3):
        M[..., 3 * i] = f[..., 3 * i] * nm.i0
        M[..., 3 * i + 1] = f[..., 3 * i + 1] * nm.i0
        M[..., 3 * i + 2] = (f[..., 3 * i] * t0x + f[..., 3 * i + 1] * t0y) + f[..., 3 * i + 2]
    for j in range(3):
        G[..., j] = M[..., j] * nm.i1
        G[..., 3 + j] = M[..., 3 + j] * nm.i1
        G[..., 6 + j] = (t1x * M[..., j] + t1y * M[..., 3 + j]) + M[..., 6 + j]
    s = np.zeros(f.shape[:-1])
    for j in range(9):
        s = s + G[..., j] * G[..., j]
    with np.errstate(all="ignore"):
        nrm = np.sqrt(s)
        ok = (nrm > 0) & np.isfinite(nrm)
        F = G / np.where(ok, nrm, 1.0)[..., None]
    neg = np.take_along_axis(G, np.argmax(np.abs(G), -1)[..., None], -1) < 0
    return np.where(neg, -F, F), ok


def _fm_terms(F, pts):
    """x1^T F x0, |(F x0)_xy|^2 and |(F^T x1)_xy|^2 of pixel F [M, 9] on correspondences pts [n, 4]: [M, n] each."""
    x0, y0, x1, y1 = (np.asarray(pts[:, i], dtype=np.float64)[None, :] for i in range(4))
    f = [F[:, i:i + 1] for i in range(9)]
    u0 = (f[0] * x0 + f[1] * y0) + f[2]
    u1 = (f[3] * x0 + f[4] * y0) + f[5]
    u2 = (f[6] * x0 + f[7] * y0) + f[8]
    w0 = (f[0] * x1 + f[3] * y1) + f[6]
    w1 = (f[1] * x1 + f[4] * y1) + f[7]
    return (x1 * u0 + y1 * u1) + u2, u0 * u0 + u1 * u1, w0 * w0 + w1 * w1


def fundamental_inliers(F, pts, t2, chunk=512):
    """Inlier flags [M, n] of pixel F [M, 9] on correspondences pts [n, 4] (x0, y0, x1, y1): cv2's FM error below t2,
    evaluated as (x1^T F x0)^2 < t2 min(|(F x0)_xy|^2, |(F^T x1)_xy|^2); a zero line normal is an outlier."""
    F = np.asarray(F, dtype=np.float64).reshape(-1, 9)
    out = np.empty((F.shape[0], len(pts)), dtype=bool)
    with np.errstate(all="ignore"):
        for s in range(0, F.shape[0], chunk):
            num, a, b = _fm_terms(F[s:s + chunk], pts)
            m = np.where(a < b, a, b)
            out[s:s + chunk] = (m > 0) & (num * num < t2 * m)
    return out


def fundamental_error(F, pts):
    """cv2's FM error [n] of one pixel F [3, 3] on correspondences pts [n, 4]: the larger squared distance of x1 to the
    epipolar line F x0 and of x0 to F^T x1, in pixels^2."""
    num, a, b = _fm_terms(np.asarray(F, dtype=np.float64).reshape(1, 9), pts)
    with np.errstate(all="ignore"):
        return np.maximum(num * num / a, num * num / b)[0]


def _side_ratio(la, lb, px, py, qx, qy):
    """Overlap ratio of one side: the lines la, lb (3 arrays each) cut the line through (p, q) at positions ta, tb (p at
    0, q at 1) -> |[min, max] n [0, 1]| / min(max - min, 1), NaN where the side cannot reject (an intersection with
    |w| <= FLT_EPSILON |X|, or ta == tb)."""
    l0, l1, l2 = py - qy, qx - px, px * qy - qx * py
    dx, dy = qx - px, qy - py
    len2 = dx * dx + dy * dy
    ok, t = np.ones(px.shape, dtype=bool), []
    for m in (la, lb):
        X0, X1, X2 = m[1] * l2 - m[2] * l1, m[2] * l0 - m[0] * l2, m[0] * l1 - m[1] * l0
        nrm = np.sqrt((X0 * X0 + X1 * X1) + X2 * X2)
        ok &= np.abs(X2) > FLT_EPSILON * nrm
        x, y = X0 / X2, X1 / X2
        t.append(((x - px) * dx + (y - py) * dy) / len2)
    lo, hi = np.where(t[0] < t[1], t[0], t[1]), np.where(t[0] < t[1], t[1], t[0])
    ok &= hi > lo
    a, b = np.where(lo > 0, lo, 0.0), np.where(hi < 1, hi, 1.0)
    ov = np.where(b > a, b - a, 0.0)
    span = hi - lo
    return np.where(ok, ov / np.where(span < 1, span, 1.0), np.nan)


def line_overlap_ratios(F, seg0, seg1):
    """The epipolar overlap ratios of matched key-line pairs under pixel F [3, 3] (x1^T F x0 = 0): seg0 / seg1 [m, 2, 2]
    (start xy, end xy; used as float32).  -> (ratio in image 1 of F a0, F b0 against s1, ratio in image 0 of F^T a1,
    F^T b1 against s0), [m] each, NaN where that side cannot reject (DESIGN.md "Fundamental matrices")."""
    F = np.asarray(F, dtype=np.float64).reshape(9)
    s0 = np.asarray(seg0, dtype=np.float32).reshape(-1, 4).astype(np.float64)
    s1 = np.asarray(seg1, dtype=np.float32).reshape(-1, 4).astype(np.float64)
    a0x, a0y, b0x, b0y = (s0[:, i] for i in range(4))
    a1x, a1y, b1x, b1y = (s1[:, i] for i in range(4))
    with np.errstate(all="ignore"):
        img1 = [[(F[3 * r] * x + F[3 * r + 1] * y) + F[3 * r + 2] for r in range(3)] for x, y in ((a0x, a0y), (b0x, b0y))]
        r1 = _side_ratio(img1[0], img1[1], a1x, a1y, b1x, b1y)
        img0 = [[(F[c] * x + F[3 + c] * y) + F[6 + c] for c in range(3)] for x, y in ((a1x, a1y), (b1x, b1y))]
        r0 = _side_ratio(img0[0], img0[1], a0x, a0y, b0x, b0y)
    return r1, r0


def lines_consistent(F, seg0, seg1, min_overlap=0.5):
    """The epipolar check of matched key-line pairs [m]: True iff no side's overlap ratio (`line_overlap_ratios`) is
    below min_overlap."""
    r1, r0 = line_overlap_ratios(F, seg0, seg1)
    return ~(r1 < min_overlap) & ~(r0 < min_overlap)


def _epipolar_rows(q):
    """The normalised epipolar rows (x1 x0, x1 y0, x1, y1 x0, y1 y0, y1, x0, y0, 1) of q [n, 4]: [n, 9]."""
    x0, y0, x1, y1 = (q[:, i] for i in range(4))
    return np.stack([x1 * x0, x1 * y0, x1, y1 * x0, y1 * y0, y1, x0, y0, np.ones_like(x0)], 1)


def ransac_fundamental_host(kpts0, kpts1, matches_p, klines0=None, klines1=None, matches_l=None, pair=0, thresh=3.0,
                            n_hypotheses=2048, seed=0, min_overlap=0.5) -> dict:
    """The fundamental-matrix estimator's model for one pair in numpy (DESIGN.md "Fundamental matrices").  kpts [N, 2]
    and klines [K, 2, 2] are used as float32; matches_p [N0] / matches_l [K0]: local side-1 index or -1 per side-0 row;
    `pair` is the pair's index in the batch (it seeds the samples).  Everything up to the winner is the kernels'
    operations in the kernels' order (the winning sample, root and inlier count are the same bits); the refit uses
    np.linalg.eigh / svd instead of the kernels' Jacobi solves.  Returns F [3, 3] (pixels, unit Frobenius norm, NaN when
    invalid), valid, inliers_p uint8 [N0], lines_consistent uint8 [K0] (aligned with the match rows), n_inliers,
    n_lines_consistent, hypothesis (3 k + j of the winning sample k and root j, or -1), hypothesis_inliers,
    F_hypothesis (the winning solution) and refit (whether the eight-point refit was kept)."""
    l0 = np.zeros((0, 2, 2), np.float32) if klines0 is None else klines0
    l1 = np.zeros((0, 2, 2), np.float32) if klines1 is None else klines1
    ml = np.zeros(0, np.int64) if matches_l is None else matches_l
    pts, _, _, rp, _ = _correspondences(kpts0, kpts1, matches_p, l0, l1, ml, True, False)
    ml = np.asarray(ml, dtype=np.int64).reshape(-1)
    out = dict(F=np.full((3, 3), np.nan), valid=False, inliers_p=np.zeros(len(np.ravel(matches_p)), dtype=np.uint8),
               lines_consistent=np.zeros(len(ml), dtype=np.uint8), n_inliers=0, n_lines_consistent=0, hypothesis=-1,
               hypothesis_inliers=0, F_hypothesis=np.full((3, 3), np.nan), refit=False)
    n = len(pts)
    if n < FM_SAMPLE:
        return out
    t2 = float(thresh) * float(thresh)
    e = np.zeros((0, 2, 2), np.float32)
    nm = _normalisation(pts, e, e)
    f = lambda a: np.asarray(a, dtype=np.float64)
    q = np.stack([(f(pts[:, 0]) - nm.c0x) * nm.i0, (f(pts[:, 1]) - nm.c0y) * nm.i0,
                  (f(pts[:, 2]) - nm.c1x) * nm.i1, (f(pts[:, 3]) - nm.c1y) * nm.i1], 1)
    idx, ok = draw_samples(seed, pair, n_hypotheses, n, FM_SAMPLE)
    Fh, okf = fundamental_solutions(q[np.maximum(idx, 0)])
    Fp, okp = _fundamental_to_pixels(Fh, nm)
    flat = np.flatnonzero((okf & okp & ok[:, None]).reshape(-1))
    if not len(flat):
        return out
    cnt = fundamental_inliers(Fp.reshape(-1, 9)[flat], pts, t2).sum(1)
    # the kernels' key: (count << 32) | ~(3 k + j); flat = 3 k + j
    w = int(flat[np.lexsort((flat, -cnt))[0]])
    F = Fp.reshape(-1, 9)[w]
    fl = fundamental_inliers(F, pts, t2)[0]
    out.update(hypothesis=w, hypothesis_inliers=int(fl.sum()), F_hypothesis=F.reshape(3, 3).copy())
    if fl.sum() >= FM_MIN_REFIT:
        A = _epipolar_rows(q[fl])
        _, V = np.linalg.eigh(A.T @ A)
        U, S, Vt = np.linalg.svd(V[:, 0].reshape(3, 3))
        S[2] = 0.0
        Fr, okr = _fundamental_to_pixels(((U * S) @ Vt).reshape(1, 9), nm)
        if okr[0]:
            flr = fundamental_inliers(Fr[0], pts, t2)[0]
            if flr.sum() >= fl.sum():
                F, fl = Fr[0], flr
                out["refit"] = True
    out["inliers_p"][rp] = fl
    k1 = np.asarray(l1, dtype=np.float32).reshape(-1, 2, 2)
    rl = np.flatnonzero((ml >= 0) & (ml < len(k1)))
    if len(rl):
        k0 = np.asarray(l0, dtype=np.float32).reshape(-1, 2, 2)
        out["lines_consistent"][rl] = lines_consistent(F, k0[rl], k1[ml[rl]], min_overlap)
    out.update(F=F.reshape(3, 3).copy(), valid=True, n_inliers=int(fl.sum()),
               n_lines_consistent=int(out["lines_consistent"].sum()))
    return out


# ------------------------------------------------------------------ fundamental matrices, batched on the GPU
@dataclass
class FundamentalResult:
    """Result of `estimate_fundamentals` (device tensors; nothing has been waited for).

    F float64 [P, 3, 3] (x1^T F x0 = 0 in pixels, unit Frobenius norm, NaN where not valid), valid bool [P], inliers_p
    uint8 aligned with the result's matches_p (0 for unmatched rows), n_inliers int32 [P], hypothesis int32 [P] (3 k + j
    of the winning sample k and root j, -1 when not valid), hypothesis_inliers int32 [P], refit bool [P] (F is the
    eight-point refit), lines_consistent uint8 aligned with matches_l (1 where the line match passes the epipolar
    check, 0 for unmatched rows and invalid pairs) and n_lines_consistent int32 [P]."""
    F: torch.Tensor
    valid: torch.Tensor
    inliers_p: torch.Tensor
    n_inliers: torch.Tensor
    hypothesis: torch.Tensor
    hypothesis_inliers: torch.Tensor
    refit: torch.Tensor
    lines_consistent: torch.Tensor
    n_lines_consistent: torch.Tensor


def estimate_fundamentals(res, thresh=3.0, n_hypotheses=2048, seed=0, min_overlap=0.5) -> FundamentalResult:
    """Fundamental matrices (x1^T F x0 = 0 in pixels) of every pair of an `ImagePairMatches` (`match_images`,
    `match_sets`) from its point matches (res.keypoints0 / keypoints1), for pairs without intrinsics: seven-point RANSAC
    with an eight-point refit, and the epipolar check of its line matches (res.klines0 / klines1 as float32 segments),
    in one `ltr_fundamental` call.  thresh in pixels (cv2's default 3); 2048 hypotheses leave about e^-16 chance of no
    all-inlier sample at 50 % outliers; min_overlap is the line check's bound.  A planar scene is degenerate for F:
    `estimate_homographies` is the tool there.  Host arrays go up in one pinned copy; the call never waits for the
    device.  Raises LtrError (LTR_E_UNSUPPORTED) when a pair has more point match rows than one CTA can stage
    (SMEM_PER_ROW_F bytes per row, SMEM_MAX in all)."""
    P = res.n_pairs
    dev = res.matches_p.device
    if int(n_hypotheses) < 1:
        raise N.LtrError("estimate_fundamentals: n_hypotheses must be >= 1")
    dv = _stage_pairs(res, dev, "estimate_fundamentals", lines=True)
    u8, i32d = dict(dtype=torch.uint8, device=dev), dict(dtype=torch.int32, device=dev)
    out = FundamentalResult(torch.empty((P, 3, 3), dtype=torch.float64, device=dev), torch.empty(P, **u8),
                            torch.empty(res.matches_p.shape[0], **u8), torch.empty(P, **i32d), torch.empty(P, **i32d),
                            torch.empty(P, **i32d), torch.empty(P, **u8), torch.empty(res.matches_l.shape[0], **u8),
                            torch.empty(P, **i32d))
    _ops.call_struct("ltr_fundamental", {**dv, "n_pairs": P, "thresh": thresh, "min_overlap": min_overlap,
                                         "n_hypotheses": n_hypotheses, "seed": seed},
                     {**vars(out), "key": torch.empty(P, dtype=torch.int64, device=dev)})
    out.valid = out.valid.view(torch.bool)
    out.refit = out.refit.view(torch.bool)
    return out


# ------------------------------------------------------------------ pose metrics
# The reference's evaluation metrics (models/utils.py:358-412), with its signatures and results.  pose_errors is the
# batched form; compute_pose_error is its one-pair case.
def _host64(a):
    return np.asarray(a.cpu() if isinstance(a, torch.Tensor) else a, dtype=np.float64)


def _pixels_to_rays(kpts, K):
    """Pixel keypoints [n, 2] -> homogeneous normalised coordinates [n, 3] ((u - cx) / fx, (v - cy) / fy, 1)."""
    K = _host64(K)
    xy = (_host64(kpts).reshape(-1, 2) - np.array([K[0, 2], K[1, 2]])) / np.array([K[0, 0], K[1, 1]])
    return np.concatenate([xy, np.ones((len(xy), 1))], 1)


def compute_epipolar_error(kpts0, kpts1, T_0to1, K0, K1):
    """Symmetric epipolar error [n] of matched keypoints under the true relative pose T_0to1 [4, 4] (X1 = R X0 + t):
    with E = [t]x R and normalised rays x0, x1, the squared residual x1^T E x0 divided by the squared normal length of
    each epipolar line, E x0 in image 1 and E^T x1 in image 0, summed over both images."""
    T = _host64(T_0to1)
    E = np.cross(T[:3, 3], T[:3, :3].T).T            # column j of [t]x R is t x R[:, j]
    x0, x1 = _pixels_to_rays(kpts0, K0), _pixels_to_rays(kpts1, K1)
    line1, line0 = x0 @ E.T, x1 @ E                   # epipolar lines in image 1 and image 0
    r2 = np.einsum("ni,ni->n", x1, line1) ** 2
    return r2 / (line1[:, 0] ** 2 + line1[:, 1] ** 2) + r2 / (line0[:, 0] ** 2 + line0[:, 1] ** 2)


def pose_errors(R, t, T_0to1):
    """Pose errors of P estimates in degrees: R [P, 3, 3] and t [P, 3] (tensors or arrays) against T_0to1 [P, 4, 4]
    or [4, 4] -> (error_t [P], error_R [P]).  error_R is the angle of the rotation R_gt^T R; error_t is the angle
    between t and t_gt folded to [0, 90] (E fixes t only up to sign).  A pair whose R or t is not finite (an invalid
    estimate) gets inf in both, as the reference's evaluation scores a failed estimate_pose."""
    R, t = _host64(R).reshape(-1, 3, 3), _host64(t).reshape(-1, 3)
    T = np.broadcast_to(_host64(T_0to1).reshape(-1, 4, 4), (len(R), 4, 4))
    ok = np.isfinite(R).all((1, 2)) & np.isfinite(t).all(1)
    with np.errstate(all="ignore"):
        cos_r = ((T[:, :3, :3] * R).sum((1, 2)) - 1.0) / 2.0        # trace(R_gt^T R) = sum of the elementwise product
        err_R = np.degrees(np.arccos(np.clip(cos_r, -1.0, 1.0)))
        t_gt = T[:, :3, 3]
        cos_t = (t * t_gt).sum(1) / (np.linalg.norm(t, axis=1) * np.linalg.norm(t_gt, axis=1))
        ang = np.degrees(np.arccos(np.clip(cos_t, -1.0, 1.0)))
    err_t = np.minimum(ang, 180.0 - ang)
    return np.where(ok, err_t, np.inf), np.where(ok, err_R, np.inf)


def compute_pose_error(T_0to1, R, t):
    """(translation error, rotation error) in degrees of one estimate: `pose_errors` for one pair."""
    et, eR = pose_errors(np.asarray(R)[None], np.asarray(t).reshape(1, 3), T_0to1)
    return et[0], eR[0]


def pose_auc(errors, thresholds):
    """Normalised area under the cumulative error curve, one value per threshold: the curve rises linearly from (0, 0)
    through (e_i, i / n) for the sorted errors e_1 <= ... <= e_n and stays flat after the last error below the
    threshold; its area up to the threshold is divided by the threshold."""
    e = np.sort(_host64(errors).reshape(-1))
    x = np.concatenate([[0.0], e])
    y = np.arange(len(x)) / max(len(e), 1)
    seg = np.diff(x) * (y[1:] + y[:-1]) / 2.0           # trapezoid between consecutive curve points
    out = []
    for thr in thresholds:
        k = int(np.searchsorted(x, thr))                  # curve points strictly below thr (x[0] = 0 included)
        out.append(float((seg[:k - 1].sum() + (thr - x[k - 1]) * y[k - 1]) / thr))
    return out
