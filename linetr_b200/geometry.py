"""Geometric verification of matches: RANSAC homographies from line and point matches, and the corner-error metric.

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
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

from . import _native as N
from . import _ops
from .eval_homography import _stage

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


def draw_samples(seed: int, pair: int, n_hypotheses: int, n: int):
    """The 4 correspondence indices of hypotheses 0..n_hypotheses-1 of `pair` among n: s = splitmix64(seed +
    splitmix64(pair << 32 | k)), draw j = splitmix64(s + j) mod n for j = 0, 1, ..., a duplicate redrawn with the next
    j.  -> (idx int64 [K, 4], ok [K]); ok is False where MAX_DRAWS draws did not give 4 distinct indices."""
    k = np.arange(n_hypotheses, dtype=_U64)
    s = splitmix64(_U64(int(seed) & 0xFFFFFFFFFFFFFFFF) + splitmix64((_U64(pair) << _U64(32)) | k))
    idx = np.full((n_hypotheses, 4), -1, dtype=np.int64)
    got = np.zeros(n_hypotheses, dtype=np.int64)
    rows = np.arange(n_hypotheses)
    for j in range(MAX_DRAWS):
        active = got < 4
        if not active.any():
            break
        v = (splitmix64(s + _U64(j)) % _U64(n)).astype(np.int64)
        take = active & ~(idx == v[:, None]).any(1)
        idx[rows[take], got[take]] = v[take]
        got += take
    return idx, got == 4


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


def estimate_homographies(res, thresh=3.0, n_hypotheses=2048, seed=0, use_lines=True, use_points=True) -> HomographyResult:
    """RANSAC homographies (image 0 -> image 1) of every pair of an `ImagePairMatches` (`match_images`, `match_sets`)
    from its line matches (res.klines0 / klines1 as float32 segments) and point matches (res.keypoints0 / keypoints1),
    in one `ltr_homography` call.  use_lines / use_points select the kinds of correspondence.  Host arrays go up in one
    pinned copy; the call never waits for the device.  Raises LtrError (LTR_E_UNSUPPORTED) when a pair has more match
    rows than one CTA can stage (SMEM_PER_POINT / SMEM_PER_LINE bytes per row, SMEM_MAX in all)."""
    P = res.n_pairs
    dev = res.matches_l.device
    op, ol = np.asarray(res.offsets_p, dtype=np.int64), np.asarray(res.offsets_l, dtype=np.int64)
    if int(n_hypotheses) < 1:
        raise N.LtrError("estimate_homographies: n_hypotheses must be >= 1")
    seg_rows = lambda k: np.asarray(k, dtype=np.float32).reshape(-1, 4)
    pt_rows = lambda k: torch.as_tensor(k).to(device=dev, dtype=torch.float32).reshape(-1, 2)
    s0, soff0, sn0 = _pool(res.klines0, P, seg_rows)
    s1, soff1, sn1 = _pool(res.klines1, P, seg_rows)
    p0, poff0, pn0 = _pool(res.keypoints0, P, pt_rows)
    p1, poff1, pn1 = _pool(res.keypoints1, P, pt_rows)
    if not (np.array_equal(sn0, np.diff(ol)) and np.array_equal(pn0, np.diff(op))):
        raise N.LtrError("estimate_homographies: side-0 key lines / keypoints and the match offsets disagree")
    cat_np = lambda parts: np.concatenate(parts) if parts else np.zeros((0, 4), dtype=np.float32)
    cat_t = lambda parts: torch.cat(parts) if parts else torch.zeros((0, 2), dtype=torch.float32, device=dev)
    i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)
    dv = _stage({"segs0": cat_np(s0), "segs1": cat_np(s1), "seg_off0": soff0, "seg_off1": soff1, "n_segs1": sn1,
                 "pts_off0": poff0, "pts_off1": poff1, "n_pts1": pn1, "cu_p": i32(op), "cu_l": i32(ol)}, dev)
    u8, i32d = dict(dtype=torch.uint8, device=dev), dict(dtype=torch.int32, device=dev)
    out = HomographyResult(torch.empty((P, 3, 3), dtype=torch.float64, device=dev), torch.empty(P, **u8),
                           torch.empty(res.matches_l.shape[0], **u8), torch.empty(res.matches_p.shape[0], **u8),
                           torch.empty(P, **i32d), torch.empty(P, **i32d), torch.empty(P, **i32d),
                           torch.empty(P, **i32d))
    key = torch.empty(P, dtype=torch.int64, device=dev)
    mx = lambda a: int(np.diff(a).max(initial=0))
    _ops.homography(P, pts0=cat_t(p0).contiguous(), pts1=cat_t(p1).contiguous(), pts_off0=dv["pts_off0"],
                    pts_off1=dv["pts_off1"], n_pts1=dv["n_pts1"], matches_p=res.matches_p.contiguous(), cu_p=dv["cu_p"],
                    max_rows_p=mx(op), segs0=dv["segs0"], segs1=dv["segs1"], seg_off0=dv["seg_off0"],
                    seg_off1=dv["seg_off1"], n_segs1=dv["n_segs1"], matches_l=res.matches_l.contiguous(),
                    cu_l=dv["cu_l"], max_rows_l=mx(ol), H=out.H, valid=out.valid, inliers_p=out.inliers_p,
                    inliers_l=out.inliers_l, n_inliers_p=out.n_inliers_p, n_inliers_l=out.n_inliers_l,
                    hypothesis=out.hypothesis, hypothesis_inliers=out.hypothesis_inliers, key=key, thresh=thresh,
                    n_hypotheses=n_hypotheses, seed=seed, use_points=use_points, use_lines=use_lines)
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
