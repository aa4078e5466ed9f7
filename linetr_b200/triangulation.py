"""Triangulation of posed images: a world point for every keypoint and two world end points for every key line of
every image of a set, from the pair matches between them, batched on the GPU.

    triangulate(keypoints, klines, pairs, res, K, R, t, thresh=4.0, min_angle=1.5, min_views=2) -> TriangulationResult
        one `ltr_triangulate` call (two kernel launches) for the whole set; device outputs, no synchronisation
    triangulate_host(...)
        the same model in numpy, vectorised over each image's rows: every operation is the kernels' operation in the
        kernels' order, so the outputs are the same bits

The model (DESIGN.md "Triangulation", include/linetr_b200.h `ltr_triangulate`): image i has intrinsics K[i] (zero
skew) and the world -> camera pose X_cam = R[i] X + t[i] (the convention of `AbsolutePoseResult`), centre C = -R^T t.
A row of image a (the anchor) is lifted along its own ray by its depth s, X = C_a + s R_a^T K_a^-1 (x, y, 1); a key
line's end points each along their own ray.  Every pair that contains a gives at most one partner observation, in
pair order: matches[k] when a is side 0, the lowest side-0 row that matched k when a is side 1.  Residuals are pixels
of the form (alpha + s beta) / (gamma + s delta): a point's reprojection errors in x and y, an end point's signed
distance to the line through the partner segment.  Each observation gives a candidate depth (a point's least-squares
root of its two numerators, an end point's plane intersection), kept iff it is > 0 and the triangulation angle is at
least min_angle degrees.  An observation supports a depth iff its own depth is > 0 and its residual is <= thresh (a
key line at both end points); the winner has the most supporters, ties to the lowest observation, and is refined by
TRI_GN_ITERS Gauss-Newton steps over its supporters, kept iff it stays > 0 with at least as many supporters.  A row is
valid iff 1 + supporters >= min_views: n_views = 1 + supporters, else NaN and n_views = 0.  Explicitly rounded fp64.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

from . import _native as N
from . import _ops
from ._posed import (PosedSet, centre, check_set, dot3, host, line_normal, mv3, offsets, pool64, ray,
                     stage_with_pools)

TRI_THREADS = 128          # rows per block of the triangulation kernel
TRI_GN_ITERS = 5           # Gauss-Newton steps of the refit (fixed budget)
TRI_MAX_VIEWS = N.TRI_MAX_VIEWS


# ------------------------------------------------------------------ arguments
def _check(keypoints, klines, pairs, res, K, R, t, who="triangulate") -> PosedSet:
    """The posed-set checks (`_posed.check_set`) with `triangulate`'s messages unless `who` is given."""
    return check_set(keypoints, klines, pairs, res, K, R, t, who)


def _check_views(S: PosedSet):
    """`triangulate`'s capacity: at most LTR_TRI_MAX_VIEWS pairs per image (tracks have no such limit)."""
    cnt = np.diff(S.view_off)
    if len(cnt) and cnt.max(initial=0) > TRI_MAX_VIEWS:
        bad = int(np.argmax(cnt))
        raise N.LtrError(f"triangulate: image {bad} takes part in {int(cnt[bad])} pairs, more than LTR_TRI_MAX_VIEWS "
                         f"({TRI_MAX_VIEWS})")


# ------------------------------------------------------------------ the model in numpy
def _cameras(S: PosedSet, a):
    """The anchor a's centre and, per observation, (fx, fy, cx, cy, R_v, A = R_v C_a + t_v, pair, side, partner)."""
    C = centre(S.R[a].reshape(9), S.t[a])
    out = []
    for code in S.views[S.view_off[a]:S.view_off[a + 1]]:
        p, side = int(code) >> 1, int(code) & 1
        v = int(S.pairs[p, 1 - side])
        Rv = S.R[v].reshape(9)
        A = [x + S.t[v, i] for i, x in enumerate(mv3(Rv, C))]
        out.append((S.K[v, 0, 0], S.K[v, 1, 1], S.K[v, 0, 2], S.K[v, 1, 2], Rv, A, p, side, v))
    return C, out


def _partner_rows(S: PosedSet, matches, cu, counts, a, cams):
    """Per observation of anchor a: its partner row for each of a's rows, or -1."""
    na = int(counts[a])
    out = []
    for *_, p, side, v in cams:
        nv = int(counts[v])
        if side == 0:
            j = matches[cu[p]:cu[p + 1]].astype(np.int64)
        else:
            m = matches[cu[p]:cu[p + 1]].astype(np.int64)
            rows = np.flatnonzero((m >= 0) & (m < na))
            j = np.full(na, np.iinfo(np.int64).max)
            np.minimum.at(j, m[rows], rows)
        out.append(np.where((j >= 0) & (j < nv), j, -1))
    return out


def _gather(pool, off, v, j, width):
    out = np.full((len(j), width), np.nan)
    ok = j >= 0
    out[ok] = pool[off[v] + j[ok]]
    return out


def _point_terms(cam, r, px):
    fx, fy, cx, cy, Rv, A = cam[:6]
    B = mv3(Rv, r)
    dx, dy = px[:, 0] - cx, px[:, 1] - cy
    return dict(ax=fx * A[0] - dx * A[2], bx=fx * B[0] - dx * B[2], ay=fy * A[1] - dy * A[2], by=fy * B[1] - dy * B[2],
                g=A[2], d=B[2], B=B, A=A)


def _point_support(o, s, t2):
    pz = o["g"] + s * o["d"]
    ex, ey = o["ax"] + s * o["bx"], o["ay"] + s * o["by"]
    return (pz > 0) & ((ex * ex + ey * ey) <= t2 * (pz * pz))


def _end_terms(cam, n, r):
    B = mv3(cam[4], r)
    return dict(alpha=dot3(n, cam[5]), beta=dot3(n, B), g=cam[5][2], d=B[2], BB=dot3(B, B))


def _end_support(e, s, t2):
    pz = e["g"] + s * e["d"]
    v = e["alpha"] + s * e["beta"]
    return (pz > 0) & ((v * v) <= t2 * (pz * pz))


def _gn(terms_of, mask, s, active):
    """TRI_GN_ITERS Gauss-Newton steps from s over the observations in mask (uint64 [rows]); terms_of(q) -> the list
    of (alpha, beta, gamma, delta) residual terms of observation q, summed in that order."""
    V = len(terms_of)
    s = s.copy()
    for _ in range(TRI_GN_ITERS):
        jj, jr = np.zeros_like(s), np.zeros_like(s)
        for q in range(V):
            sel = ((mask >> np.uint64(q)) & np.uint64(1)).astype(bool)
            for a, b, g, d in terms_of[q]:
                den = g + s * d
                r = (a + s * b) / den
                J = (b - r * d) / den
                jj = np.where(sel, jj + J * J, jj)
                jr = np.where(sel, jr + J * r, jr)
        sn = s - jr / jj
        active = active & (jj > 0) & np.isfinite(sn)
        s = np.where(active, sn, s)
    return s


def _select(cand, supports, V, rows):
    """The winner over the observations: cand(o) -> (ok [rows], depths); supports(o, depths) -> bool [rows] per
    observation q.  -> (best count, -1 without a candidate; the winner's depths; its support mask uint64)."""
    best = np.full(rows, -1, dtype=np.int64)
    win, mask = None, np.zeros(rows, dtype=np.uint64)
    for o in range(V):
        ok, s = cand(o)
        cnt = np.zeros(rows, dtype=np.int64)
        m = np.zeros(rows, dtype=np.uint64)
        for q, sup in enumerate(supports(s)):
            cnt += sup
            m |= sup.astype(np.uint64) << np.uint64(q)
        up = ok & (cnt > best)
        best = np.where(up, cnt, best)
        win = [np.where(up, x, y) for x, y in zip(s, win)] if win is not None else [np.where(up, x, 0.0) for x in s]
        mask = np.where(up, m, mask)
    return best, win, mask


def triangulate_host(keypoints, klines, pairs, res, K, R, t, thresh=4.0, min_angle=1.5, min_views=2) -> dict:
    """The triangulation model in numpy (DESIGN.md "Triangulation"), same arguments as `triangulate` (keypoints and key
    lines used as float32).  -> dict points3d [sum n_i, 3], lines3d [sum m_i, 2, 3], n_views_p, n_views_l (int32),
    offsets_p / offsets_l [n + 1], and per row the winner's depth (winner_p [sum n_i], winner_l [sum m_i, 2]), its
    supporters (support_p / support_l uint64, bit o = observation o of the row's image), the kept depth (depth_p /
    depth_l, NaN where not valid) and refit_p / refit_l (the Gauss-Newton refit was kept); views / view_off list each
    image's observations (pair << 1 | side) in order."""
    S = _check(keypoints, klines, pairs, res, K, R, t)
    _check_views(S)
    if not (float(thresh) > 0 and math.isfinite(float(thresh))) or not (0 <= float(min_angle) < 90) or int(min_views) < 1:
        raise N.LtrError("triangulate: thresh must be finite and > 0, min_angle in [0, 90) and min_views >= 1")
    n = len(keypoints)
    kp_off, kl_off = offsets(S.n_kp).astype(np.int64), offsets(S.n_kl).astype(np.int64)
    kp_pool, kl_pool = pool64(keypoints, 2), pool64(klines, 4)
    mp, ml = host(res.matches_p, np.int64).reshape(-1), host(res.matches_l, np.int64).reshape(-1)
    cu_p, cu_l = np.asarray(res.offsets_p, dtype=np.int64), np.asarray(res.offsets_l, dtype=np.int64)
    t2 = float(thresh) * float(thresh)
    rad = float(min_angle) * (math.pi / 180.0)
    cmin, sn = math.cos(rad), math.sin(rad)
    s2min = sn * sn
    Np, Nl = int(kp_off[-1]), int(kl_off[-1])
    out = dict(points3d=np.full((Np, 3), np.nan), lines3d=np.full((Nl, 2, 3), np.nan),
               n_views_p=np.zeros(Np, np.int32), n_views_l=np.zeros(Nl, np.int32), offsets_p=kp_off, offsets_l=kl_off,
               winner_p=np.full(Np, np.nan), winner_l=np.full((Nl, 2), np.nan), support_p=np.zeros(Np, np.uint64),
               support_l=np.zeros(Nl, np.uint64), depth_p=np.full(Np, np.nan), depth_l=np.full((Nl, 2), np.nan),
               refit_p=np.zeros(Np, bool), refit_l=np.zeros(Nl, bool), views=S.views, view_off=S.view_off)
    with np.errstate(all="ignore"):
        for a in range(n):
            C, cams = _cameras(S, a)
            V = len(cams)
            # points
            rows = int(S.n_kp[a])
            if rows:
                Ra, fx, fy, cx, cy = S.R[a].reshape(9), S.K[a, 0, 0], S.K[a, 1, 1], S.K[a, 0, 2], S.K[a, 1, 2]
                kp = kp_pool[kp_off[a]:kp_off[a + 1]]
                r = ray(Ra, fx, fy, cx, cy, kp[:, 0], kp[:, 1])
                js = _partner_rows(S, mp, cu_p, S.n_kp, a, cams)
                T = [_point_terms(c, r, _gather(kp_pool, kp_off, c[8], j, 2)) for c, j in zip(cams, js)]

                def cand(o):
                    o_ = T[o]
                    s = -((o_["ax"] * o_["bx"] + o_["ay"] * o_["by"]) / (o_["bx"] * o_["bx"] + o_["by"] * o_["by"]))
                    P = [A + s * B for A, B in zip(o_["A"], o_["B"])]
                    ang = dot3(o_["B"], P) <= cmin * np.sqrt(dot3(o_["B"], o_["B"]) * dot3(P, P))
                    return (s > 0) & ang, [s]

                best, win, mask = _select(cand, lambda s: [_point_support(o_, s[0], t2) for o_ in T], V, rows)
                have = best >= 0
                s_w = win[0] if V else np.zeros(rows)
                s = _gn([[(o_["ax"], o_["bx"], o_["g"], o_["d"]), (o_["ay"], o_["by"], o_["g"], o_["d"])] for o_ in T],
                        mask, s_w, have)
                cnt = sum((_point_support(o_, s, t2).astype(np.int64) for o_ in T), np.zeros(rows, np.int64))
                keep = have & (s > 0) & (cnt >= best)
                best = np.where(keep, cnt, best)
                s_k = np.where(keep, s, s_w)
                ok = have & (1 + best >= int(min_views))
                sl = slice(kp_off[a], kp_off[a + 1])
                X = np.stack([C[e] + s_k * r[e] for e in range(3)], 1)
                out["points3d"][sl] = np.where(ok[:, None], X, np.nan)
                out["n_views_p"][sl] = np.where(ok, 1 + best, 0)
                out["winner_p"][sl] = np.where(have, s_w, np.nan)
                out["support_p"][sl] = mask
                out["depth_p"][sl] = np.where(ok, s_k, np.nan)
                out["refit_p"][sl] = keep
            # key lines
            rows = int(S.n_kl[a])
            if rows:
                Ra, fx, fy, cx, cy = S.R[a].reshape(9), S.K[a, 0, 0], S.K[a, 1, 1], S.K[a, 0, 2], S.K[a, 1, 2]
                kl = kl_pool[kl_off[a]:kl_off[a + 1]]
                r0 = ray(Ra, fx, fy, cx, cy, kl[:, 0], kl[:, 1])
                r1 = ray(Ra, fx, fy, cx, cy, kl[:, 2], kl[:, 3])
                js = _partner_rows(S, ml, cu_l, S.n_kl, a, cams)
                T = []
                for c, j in zip(cams, js):
                    nrm = line_normal(*c[:4], _gather(kl_pool, kl_off, c[8], j, 4))
                    T.append((_end_terms(c, nrm, r0), _end_terms(c, nrm, r1), dot3(nrm, nrm)))

                def cand(o):
                    e0, e1, nn = T[o]
                    s0, s1 = -(e0["alpha"] / e0["beta"]), -(e1["alpha"] / e1["beta"])
                    ok = (s0 > 0) & (s1 > 0) & (e0["beta"] * e0["beta"] >= s2min * (nn * e0["BB"])) \
                        & (e1["beta"] * e1["beta"] >= s2min * (nn * e1["BB"]))
                    return ok, [s0, s1]

                sup = lambda s: [_end_support(e0, s[0], t2) & _end_support(e1, s[1], t2) for e0, e1, _ in T]
                best, win, mask = _select(cand, sup, V, rows)
                have = best >= 0
                w = win if V else [np.zeros(rows), np.zeros(rows)]
                s = [_gn([[(T[q][e]["alpha"], T[q][e]["beta"], T[q][e]["g"], T[q][e]["d"])] for q in range(V)],
                         mask, w[e], have) for e in range(2)]
                cnt = sum((x.astype(np.int64) for x in sup(s)), np.zeros(rows, np.int64))
                keep = have & (s[0] > 0) & (s[1] > 0) & (cnt >= best)
                best = np.where(keep, cnt, best)
                s_k = [np.where(keep, s[e], w[e]) for e in range(2)]
                ok = have & (1 + best >= int(min_views))
                sl = slice(kl_off[a], kl_off[a + 1])
                X = np.stack([np.stack([C[e] + s_k[i] * (r0, r1)[i][e] for e in range(3)], 1) for i in range(2)], 1)
                out["lines3d"][sl] = np.where(ok[:, None, None], X, np.nan)
                out["n_views_l"][sl] = np.where(ok, 1 + best, 0)
                out["winner_l"][sl] = np.where(have[:, None], np.stack(w, 1), np.nan)
                out["support_l"][sl] = mask
                out["depth_l"][sl] = np.where(ok[:, None], np.stack(s_k, 1), np.nan)
                out["refit_l"][sl] = keep
    return out


# ------------------------------------------------------------------ batched on the GPU
@dataclass
class TriangulationResult:
    """Result of `triangulate` (device tensors; nothing has been waited for).

    points3d float64 [sum n_i, 3] (image i's keypoints are rows offsets_p[i] to offsets_p[i + 1]), lines3d float64
    [sum m_i, 2, 3] (start and end point of each key line, rows offsets_l[i] to offsets_l[i + 1]); NaN where a row has
    no valid estimate.  n_views_p / n_views_l int32: 1 + the supporting observations of each valid row, else 0.
    offsets_p / offsets_l: host int64 [n + 1]."""
    points3d: torch.Tensor
    lines3d: torch.Tensor
    n_views_p: torch.Tensor
    n_views_l: torch.Tensor
    offsets_p: np.ndarray
    offsets_l: np.ndarray

    def per_image(self):
        """Host copies, one array per image: (points [n_i, 3] list, lines [m_i, 2, 3] list) fp64.  They are what
        `estimate_absolute_poses` reads as points3d1 / lines3d1: pass pts[j] for every pair whose side 1 is image j,
        the same object each time, so it goes up once."""
        P, L = self.points3d.cpu().numpy(), self.lines3d.cpu().numpy()
        op, ol = self.offsets_p, self.offsets_l
        return ([P[op[i]:op[i + 1]] for i in range(len(op) - 1)], [L[ol[i]:ol[i + 1]] for i in range(len(ol) - 1)])


def triangulate(keypoints, klines, pairs, res, K, R, t, thresh=4.0, min_angle=1.5, min_views=2) -> TriangulationResult:
    """World points of every keypoint and world end points of every key line of n posed images, from the matches `res`
    (an `ImagePairMatches`, as `match_set(images, pairs)` returns) of the host pair list pairs [P, 2], in one
    `ltr_triangulate` call (two kernel launches, no synchronisation).  keypoints[i] [n_i, 2] and klines[i] [m_i, 2, 2]
    (or [m_i, 4]) are image i's, as `ImageSet.keypoints` / `ImageSet.klines` hold them; K [3, 3] or [n, 3, 3] (zero
    skew), R [n, 3, 3] and t [n, 3] the world -> camera poses (X_cam = R X + t).  thresh in pixels, min_angle in
    degrees (COLMAP's minimum triangulation angle), min_views the views a valid row needs, the anchor included.
    Raises LtrError before any device work for bad K, R or t, a pair list that disagrees with res, self or duplicate
    pairs, and an image in more than LTR_TRI_MAX_VIEWS pairs."""
    S = _check(keypoints, klines, pairs, res, K, R, t)
    _check_views(S)
    n, P = len(keypoints), len(S.pairs)
    dev = res.matches_p.device
    op, ol = offsets(S.n_kp), offsets(S.n_kl)
    f64, i32 = dict(dtype=torch.float64, device=dev), dict(dtype=torch.int32, device=dev)
    # at least one row each, so a set without keypoints or without key lines hands ltr_triangulate no null output
    Np, Nl = int(op[-1]), int(ol[-1])
    rp, rl = max(Np, 1), max(Nl, 1)
    buf = dict(points3d=torch.empty((rp, 3), **f64), lines3d=torch.empty((rl, 2, 3), **f64),
               n_views_p=torch.empty(rp, **i32), n_views_l=torch.empty(rl, **i32))
    out = TriangulationResult(buf["points3d"][:Np], buf["lines3d"][:Nl], buf["n_views_p"][:Np], buf["n_views_l"][:Nl],
                              op.astype(np.int64), ol.astype(np.int64))
    if n == 0:
        return out
    blocks = np.concatenate([(S.n_kp + TRI_THREADS - 1) // TRI_THREADS, (S.n_kl + TRI_THREADS - 1) // TRI_THREADS])
    block_off = offsets(blocks)
    inv_off_p = offsets(S.n_kp[S.pairs[:, 1]] if P else [])
    inv_off_l = offsets(S.n_kl[S.pairs[:, 1]] if P else [])
    arrays = {"K": S.K, "R": S.R, "t": S.t, "pairs": S.pairs.reshape(-1, 2),
              "cu_p": np.asarray(res.offsets_p, dtype=np.int32), "cu_l": np.asarray(res.offsets_l, dtype=np.int32),
              "views": S.views, "view_off": S.view_off, "block_off": block_off, "inv_off_p": inv_off_p,
              "inv_off_l": inv_off_l, "kp_off": op, "seg_off": ol}
    dv = stage_with_pools(arrays, keypoints, klines, dev)
    inv_p = torch.empty(max(int(inv_off_p[-1]), 1), **i32)
    inv_l = torch.empty(max(int(inv_off_l[-1]), 1), **i32)
    _ops.call_struct("ltr_triangulate",
                     {**dv, "matches_p": res.matches_p.contiguous(), "matches_l": res.matches_l.contiguous(),
                      "n_images": n, "n_pairs": P, "total_p": int(res.offsets_p[-1]), "total_l": int(res.offsets_l[-1]),
                      "n_inv_p": int(inv_off_p[-1]), "n_inv_l": int(inv_off_l[-1]), "n_blocks": int(block_off[-1]),
                      "max_views": int(np.diff(S.view_off).max(initial=0)), "thresh": thresh,
                      "min_angle": min_angle, "min_views": min_views},
                     dict(**buf, inv_p=inv_p, inv_l=inv_l))
    return out
