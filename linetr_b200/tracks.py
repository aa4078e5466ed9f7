"""Tracks of posed image sets: the pair matches that agree with the known poses join the keypoints and key lines of all
images into point and line tracks, and each track gets one robust multi-view world point or world line, on the GPU.

    triangulate_tracks(keypoints, klines, pairs, res, K, R, t, thresh=4.0, min_angle=1.5, min_views=2, epi_thresh=4.0,
                       min_overlap=0.5) -> TrackResult
        one `ltr_tracks` call (six kernel launches) for the whole set; device outputs, no synchronisation
    triangulate_tracks_host(...) -> dict
        the same model in numpy (scipy's connected_components for the components), vectorised over the tracks of one
        length: every operation of the estimate is the kernels' operation in the kernels' order, so the outputs are
        the same bits

The model (DESIGN.md "Tracks", include/linetr_b200.h `ltr_tracks`): image i has intrinsics K[i] (zero skew) and the
world -> camera pose X_cam = R[i] X + t[i].  A match row of pair (i, j) is an edge iff its match lies in the rows of j
and agrees with the pair's pixel fundamental matrix F = K_j^-T [t]x R K_i^-1 (R = R_j R_i^T, t = t_j - R t_i): a point
under cv2's FM error below epi_thresh (`geometry.fundamental_inliers`), a key line under the epipolar overlap check
(`geometry.lines_consistent`).  A track is a connected component of >= 2 rows of one kind (ids in ascending order of
their minimum pooled row, observations in ascending row order).  A track of at most LTR_TRK_MAX_OBS observations takes
the two-view estimate of `triangulate` of every observation pair (i, j), i < j, with the most supporters (ties to the
lowest i * LTR_TRK_MAX_OBS + j), refines it by Gauss-Newton on the world point (a key line: each of the anchor's end
points) over its supporters, and keeps the refit iff every supporter stays in front and the supporter count does not
fall.  It is valid iff its inliers (the supporters of the kept estimate) number at least min_views.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

from . import _native as N
from . import _ops
from .geometry import fundamental_inliers, lines_consistent
from ._posed import (centre, check_set, closest_on_line, dot3, host, line_normal, mv3, offsets, pool64, ray,
                     stage_with_pools)
from .triangulation import TriangulationResult

TRK_MAX_OBS = N.TRK_MAX_OBS
TRK_GN_ITERS = 5           # Gauss-Newton steps of the refits (fixed budget)
TRK_OK, TRK_TOO_LONG, TRK_NO_CANDIDATE, TRK_TOO_FEW = N.TRK_OK, N.TRK_TOO_LONG, N.TRK_NO_CANDIDATE, N.TRK_TOO_FEW
_WHO = "triangulate_tracks"


def _check_params(thresh, min_angle, min_views, epi_thresh, min_overlap):
    ok = lambda x: float(x) > 0 and math.isfinite(float(x))
    if not ok(thresh) or not ok(epi_thresh) or not (0 <= float(min_angle) < 90) or int(min_views) < 1 \
            or not math.isfinite(float(min_overlap)):
        raise N.LtrError(f"{_WHO}: thresh and epi_thresh must be finite and > 0, min_angle in [0, 90), min_views >= 1 "
                         "and min_overlap finite")


def pair_fundamentals(S) -> np.ndarray:
    """The pixel fundamental matrix of every pair (i, j) of the checked set S from the poses: F = K_j^-T [t]x R K_i^-1
    with R = R_j R_i^T and t = t_j - R t_i, scaled to unit Frobenius norm with its largest |entry| positive; fp64 in a
    fixed order, vectorised over the pairs.  -> [P, 3, 3]."""
    P = len(S.pairs)
    i, j = S.pairs[:, 0], S.pairs[:, 1]
    Ri, Rj, ti, tj, Ki, Kj = S.R[i], S.R[j], S.t[i], S.t[j], S.K[i], S.K[j]
    R = np.empty((P, 3, 3))
    for a in range(3):
        for b in range(3):
            R[:, a, b] = (Rj[:, a, 0] * Ri[:, b, 0] + Rj[:, a, 1] * Ri[:, b, 1]) + Rj[:, a, 2] * Ri[:, b, 2]
    t = np.stack([tj[:, a] - ((R[:, a, 0] * ti[:, 0] + R[:, a, 1] * ti[:, 1]) + R[:, a, 2] * ti[:, 2])
                  for a in range(3)], 1)
    z = np.zeros(P)
    tx = [[z, -t[:, 2], t[:, 1]], [t[:, 2], z, -t[:, 0]], [-t[:, 1], t[:, 0], z]]
    E = [[(tx[a][0] * R[:, 0, b] + tx[a][1] * R[:, 1, b]) + tx[a][2] * R[:, 2, b] for b in range(3)] for a in range(3)]

    def kinv(K):
        return [[1.0 / K[:, 0, 0], z, -(K[:, 0, 2] / K[:, 0, 0])], [z, 1.0 / K[:, 1, 1], -(K[:, 1, 2] / K[:, 1, 1])],
                [z, z, z + 1.0]]
    A, B = kinv(Ki), kinv(Kj)
    M = [[(E[a][0] * A[0][b] + E[a][1] * A[1][b]) + E[a][2] * A[2][b] for b in range(3)] for a in range(3)]
    F = np.stack([np.stack([(B[0][a] * M[0][b] + B[1][a] * M[1][b]) + B[2][a] * M[2][b] for b in range(3)], -1)
                  for a in range(3)], -2)
    f = F.reshape(P, 9)
    nrm = np.sqrt((f * f).sum(1))
    with np.errstate(all="ignore"):
        f = f / nrm[:, None]
    big = np.take_along_axis(f, np.argmax(np.abs(f), 1)[:, None], 1)
    return np.where(big < 0, -f, f).reshape(P, 3, 3)


# ------------------------------------------------------------------ the model in numpy
class _Obs:
    """The staged observations of a group of tracks of V observations each: every field [T, V] (vectors: lists)."""

    def __init__(self, S, nodes, off, pool, lines):
        img = np.searchsorted(off, nodes, side="right") - 1
        K = S.K[img]
        self.fx, self.fy, self.cx, self.cy = K[..., 0, 0], K[..., 1, 1], K[..., 0, 2], K[..., 1, 2]
        self.R = S.R[img].reshape(*nodes.shape, 9)
        self.t = [S.t[img][..., e] for e in range(3)]
        self.C = centre(self.R, self.t)
        px = pool[nodes]
        self.px = px
        cam = (self.R, self.fx, self.fy, self.cx, self.cy)
        self.r0 = ray(*cam, px[..., 0], px[..., 1])
        if lines:
            self.r1 = ray(*cam, px[..., 2], px[..., 3])
            self.n = line_normal(self.fx, self.fy, self.cx, self.cy, px)

    def at(self, field, q):
        v = getattr(self, field)
        return [x[:, q] for x in v] if isinstance(v, list) else v[:, q]

    def camera_P(self, X):
        """P = R_q X + t_q of world points X (3 arrays [T]) in every observation: 3 arrays [T, V]."""
        P = mv3(self.R, [x[:, None] for x in X])
        return [P[e] + self.t[e] for e in range(3)]

    def A(self, i, q):
        """R_q C_i + t_q of anchor column i for observation column q: 3 arrays [T]."""
        Ci = self.at("C", i)
        Rq = self.R[:, q]
        return [x + self.t[e][:, q] for e, x in enumerate(mv3(Rq, Ci))]


def _point_support(o: _Obs, X, t2):
    P = o.camera_P(X)
    dx, dy = o.px[..., 0] - o.cx, o.px[..., 1] - o.cy
    ex, ey = o.fx * P[0] - dx * P[2], o.fy * P[1] - dy * P[2]
    return (P[2] > 0) & ((ex * ex + ey * ey) <= t2 * (P[2] * P[2]))


def _end_support(o: _Obs, X, t2):
    P = o.camera_P(X)
    v = dot3(o.n, P)
    return (P[2] > 0) & ((v * v) <= t2 * (P[2] * P[2]))


def _depth(o: _Obs, X):
    return o.camera_P(X)[2]


def _point_candidate(o: _Obs, i, j, cos_min):
    A = o.A(i, j)
    r = o.at("r0", i)
    Rj = o.R[:, j]
    B = mv3(Rj, r)
    dx, dy = o.px[:, j, 0] - o.cx[:, j], o.px[:, j, 1] - o.cy[:, j]
    fx, fy = o.fx[:, j], o.fy[:, j]
    ax, bx = fx * A[0] - dx * A[2], fx * B[0] - dx * B[2]
    ay, by = fy * A[1] - dy * A[2], fy * B[1] - dy * B[2]
    s = -((ax * bx + ay * by) / (bx * bx + by * by))
    P = [A[e] + s * B[e] for e in range(3)]
    ok = (s > 0) & (dot3(B, P) <= cos_min * np.sqrt(dot3(B, B) * dot3(P, P)))
    Ci = o.at("C", i)
    return ok, [Ci[e] + s * r[e] for e in range(3)]


def _line_candidate(o: _Obs, i, j, sin2_min):
    A = o.A(i, j)
    n = o.at("n", j)
    Rj = o.R[:, j]
    alpha, nn = dot3(n, A), dot3(n, n)
    Ci = o.at("C", i)
    ok, X = None, []
    for r in (o.at("r0", i), o.at("r1", i)):
        B = mv3(Rj, r)
        beta, BB = dot3(n, B), dot3(B, B)
        s = -(alpha / beta)
        okr = (s > 0, beta * beta >= sin2_min * (nn * BB))
        ok = okr if ok is None else (ok[0] & okr[0], ok[1] & okr[1])
        X += [Ci[e] + s * r[e] for e in range(3)]
    return ok[0] & ok[1], X


def _gn_term(num, den, b, d, h, g, sel):
    r = num / den
    J = [(b[k] - r * d[k]) / den for k in range(3)]
    for m, (u, v) in enumerate(((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))):
        h[m] = np.where(sel, h[m] + J[u] * J[v], h[m])
    for k in range(3):
        g[k] = np.where(sel, g[k] + J[k] * r, g[k])


def _pixel_terms(o: _Obs, q, A, px, Y, h, g, sel):
    """The two pixel residuals of observation column q, or per track of column q[track] (the anchor's)."""
    col = lambda a: a[np.arange(len(sel)), q]
    R = col(o.R)
    P = [x + A[e] for e, x in enumerate(mv3(R, Y))]
    fx, fy, cx, cy = col(o.fx), col(o.fy), col(o.cx), col(o.cy)
    dx, dy = px[0] - cx, px[1] - cy
    d = [R[:, 6], R[:, 7], R[:, 8]]
    _gn_term(fx * P[0] - dx * P[2], P[2], [fx * R[:, k] - dx * R[:, 6 + k] for k in range(3)], d, h, g, sel)
    _gn_term(fy * P[1] - dy * P[2], P[2], [fy * R[:, 3 + k] - dy * R[:, 6 + k] for k in range(3)], d, h, g, sel)


def _line_term(o: _Obs, q, A, Y, h, g, sel):
    R = o.R[:, q]
    n = o.at("n", q)
    P = [x + A[e] for e, x in enumerate(mv3(R, Y))]
    b = [(n[0] * R[:, k] + n[1] * R[:, 3 + k]) + n[2] * R[:, 6 + k] for k in range(3)]
    _gn_term(dot3(n, P), P[2], b, [R[:, 6], R[:, 7], R[:, 8]], h, g, sel)


def _solve_step(h, g, Y, active):
    """Gaussian elimination with first-largest partial pivoting of the 3 x 3 normal equations, per track; -> (Y - step
    where active and the step exists and is finite, the updated active flags)."""
    T = len(Y[0])
    M = np.stack([np.stack([h[0], h[1], h[2], g[0]], 1), np.stack([h[1], h[3], h[4], g[1]], 1),
                  np.stack([h[2], h[4], h[5], g[2]], 1)], 1)
    ok = np.ones(T, bool)
    ar = np.arange(T)
    for c in range(3):
        p = np.full(T, c)
        for r in range(c + 1, 3):
            p = np.where(np.abs(M[:, r, c]) > np.abs(M[ar, p, c]), r, p)
        ok &= np.abs(M[ar, p, c]) > 0
        rc, rp = M[ar, c].copy(), M[ar, p].copy()
        M[ar, c], M[ar, p] = rp, rc
        for r in range(c + 1, 3):
            f = M[:, r, c] / M[:, c, c]
            for k in range(c + 1, 4):
                M[:, r, k] = M[:, r, k] - f * M[:, c, k]
    d2 = M[:, 2, 3] / M[:, 2, 2]
    d1 = (M[:, 1, 3] - M[:, 1, 2] * d2) / M[:, 1, 1]
    d0 = ((M[:, 0, 3] - M[:, 0, 1] * d1) - M[:, 0, 2] * d2) / M[:, 0, 0]
    Yn = [Y[0] - d0, Y[1] - d1, Y[2] - d2]
    active = active & ok & np.isfinite(Yn[0]) & np.isfinite(Yn[1]) & np.isfinite(Yn[2])
    return [np.where(active, Yn[k], Y[k]) for k in range(3)], active


def _bits(mask, V):
    return [((mask >> np.uint64(q)) & np.uint64(1)).astype(bool) for q in range(V)]


def _popcount(m):
    return np.array([bin(int(x)).count("1") for x in m], dtype=np.int64)


def _estimate(o: _Obs, V, T, lines, t2, cos_min, sin2_min):
    """Candidates, winner, refit of T tracks of V observations -> dict of per-track results."""
    key = np.zeros(T, np.uint64)
    sup = (lambda X: _end_support(o, X[:3], t2) & _end_support(o, X[3:], t2)) if lines else \
        (lambda X: _point_support(o, X, t2))
    for i in range(V):
        for j in range(i + 1, V):
            ok, X = _line_candidate(o, i, j, sin2_min) if lines else _point_candidate(o, i, j, cos_min)
            cnt = sup(X).sum(1).astype(np.uint64)
            k = (cnt << np.uint64(32)) | np.uint64(~np.uint32(i * TRK_MAX_OBS + j))
            key = np.where(ok & (k > key), k, key)
    have = key > 0
    idx = (~(key & np.uint64(0xFFFFFFFF)).astype(np.uint32)).astype(np.int64)
    ai, aj = np.where(have, idx // TRK_MAX_OBS, 0), np.where(have, idx % TRK_MAX_OBS, 1)
    best = (key >> np.uint64(32)).astype(np.int64)
    # the winner again, per track (its anchor column varies)
    width = 6 if lines else 3
    X = [np.full(T, np.nan) for _ in range(width)]
    for i in range(V):
        for j in range(i + 1, V):
            sel = have & (ai == i) & (aj == j)
            if sel.any():
                _, Xc = _line_candidate(o, i, j, sin2_min) if lines else _point_candidate(o, i, j, cos_min)
                X = [np.where(sel, a, b) for a, b in zip(Xc, X)]
    s = sup(X)
    mask = np.zeros(T, np.uint64)
    for q in range(V):
        mask |= s[:, q].astype(np.uint64) << np.uint64(q)
    bits = _bits(mask, V)
    # columns of the anchor as [T] arrays
    pick = lambda a: np.take_along_axis(a, ai[:, None], 1)[:, 0]
    Ci = [pick(c) for c in o.C]
    Ra, ta = o.R[np.arange(T), ai], [pick(x) for x in o.t]
    Aa = [x + ta[e] for e, x in enumerate(mv3(Ra, Ci))]
    Aq = [[x + o.t[e][:, q] for e, x in enumerate(mv3(o.R[:, q], Ci))] for q in range(V)]
    ends = 2 if lines else 1
    Xr = []
    for e in range(ends):
        Y = [X[3 * e + k] - Ci[k] for k in range(3)]
        active = have.copy()
        if lines:
            pe = [pick(o.px[..., 2 * e]), pick(o.px[..., 2 * e + 1])]
        for _ in range(TRK_GN_ITERS):
            h, g = [np.zeros(T) for _ in range(6)], [np.zeros(T) for _ in range(3)]
            if lines:
                _pixel_terms(o, ai, Aa, pe, Y, h, g, np.ones(T, bool))
                for q in range(V):
                    _line_term(o, q, Aq[q], Y, h, g, bits[q] & (ai != q))
            else:
                for q in range(V):
                    _pixel_terms(o, q, Aq[q], [o.px[:, q, 0], o.px[:, q, 1]], Y, h, g, bits[q])
            Y, active = _solve_step(h, g, Y, active)
        Xr += [Ci[k] + Y[k] for k in range(3)]
    front = np.ones(T, bool)
    for e in range(ends):
        dz = _depth(o, Xr[3 * e:3 * e + 3])
        for q in range(V):
            front &= ~bits[q] | (dz[:, q] > 0)
    sr = sup(Xr)
    mr = np.zeros(T, np.uint64)
    for q in range(V):
        mr |= sr[:, q].astype(np.uint64) << np.uint64(q)
    keep = have & front & (_popcount(mr) >= best)
    Xf = [np.where(keep, a, b) for a, b in zip(Xr, X)]
    mask_f = np.where(keep, mr, np.where(have, mask, np.uint64(0)))
    return dict(have=have, anchor=np.where(have, ai, -1), partner=np.where(have, aj, -1), winner=np.stack(X, 1),
                support=np.where(have, mask, np.uint64(0)), refit=keep, X=np.stack(Xf, 1), mask=mask_f)


def _components(n_nodes, u, v):
    """Labels of the connected components of the graph (u, v edges): each component's minimum node."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    if n_nodes == 0:
        return np.zeros(0, np.int64)
    A = coo_matrix((np.ones(len(u)), (u, v)), shape=(n_nodes, n_nodes)).tocsr()
    nc, lab = connected_components(A, directed=False)
    mn = np.full(nc, n_nodes, np.int64)
    np.minimum.at(mn, lab, np.arange(n_nodes))
    return mn[lab]


def triangulate_tracks_host(keypoints, klines, pairs, res, K, R, t, thresh=4.0, min_angle=1.5, min_views=2,
                            epi_thresh=4.0, min_overlap=0.5) -> dict:
    """The track model in numpy (DESIGN.md "Tracks"), same arguments as `triangulate_tracks` (keypoints and key lines
    used as float32).  -> dict, per kind k in (p, l): track_k (per row, -1 for none), n_tracks_k, track_off_k, obs_k,
    points3d [T_p, 3] / lines3d [T_l, 2, 3], n_obs_k, n_inliers_k, n_images_k, status_k, inlier_k, n_views_k,
    row_points3d / row_lines3d, edges_k (per match row), label_k (each row's component: its minimum row), and per track
    the winner (anchor_k / partner_k observation index, winner_k its coordinates, support_k its supporter mask, bit o =
    observation o) and refit_k (the refit was kept); F [P, 3, 3] and offsets_p / offsets_l [n + 1]."""
    S = check_set(keypoints, klines, pairs, res, K, R, t, _WHO)
    _check_params(thresh, min_angle, min_views, epi_thresh, min_overlap)
    n, P = len(keypoints), len(S.pairs)
    kp_off, kl_off = offsets(S.n_kp).astype(np.int64), offsets(S.n_kl).astype(np.int64)
    kp_pool, kl_pool = pool64(keypoints, 2), pool64(klines, 4)
    F = pair_fundamentals(S) if P else np.zeros((0, 3, 3))
    t2, epi2 = float(thresh) * float(thresh), float(epi_thresh) * float(epi_thresh)
    rad = float(min_angle) * (math.pi / 180.0)
    cos_min, sn = math.cos(rad), math.sin(rad)
    sin2_min = sn * sn
    out = dict(F=F, offsets_p=kp_off, offsets_l=kl_off)
    for kind, off, pool, mt, cu, width in (
            ("p", kp_off, kp_pool, res.matches_p, res.offsets_p, 2), ("l", kl_off, kl_pool, res.matches_l, res.offsets_l, 4)):
        lines = kind == "l"
        m = host(mt, np.int64).reshape(-1)
        cu = np.asarray(cu, dtype=np.int64)
        Nn = int(off[-1])
        edges = np.zeros(len(m), bool)
        us, vs = [], []
        for p in range(P):
            i, j = int(S.pairs[p, 0]), int(S.pairs[p, 1])
            mm = m[cu[p]:cu[p + 1]]
            ok = (mm >= 0) & (mm < off[j + 1] - off[j])
            k = np.flatnonzero(ok)
            a, b = off[i] + k, off[j] + mm[k]
            if lines:
                e = lines_consistent(F[p], pool[a].reshape(-1, 2, 2), pool[b].reshape(-1, 2, 2), min_overlap)
            else:
                e = fundamental_inliers(F[p], np.concatenate([pool[a], pool[b]], 1), epi2)[0]
            edges[cu[p] + k[e]] = True
            us.append(a[e])
            vs.append(b[e])
        u = np.concatenate(us) if us else np.zeros(0, np.int64)
        v = np.concatenate(vs) if vs else np.zeros(0, np.int64)
        label = _components(Nn, u, v)
        size = np.bincount(label, minlength=Nn)
        roots = np.flatnonzero((label == np.arange(Nn)) & (size >= 2))
        T = len(roots)
        tid = np.full(Nn, -1, np.int64)
        tid[roots] = np.arange(T)
        track = np.where(size[label] >= 2, tid[label], -1) if Nn else np.zeros(0, np.int64)
        n_obs = size[roots]
        track_off = np.concatenate([[0], np.cumsum(n_obs)]).astype(np.int64)
        inn = np.flatnonzero(track >= 0)
        obs = inn[np.argsort(track[inn], kind="stable")]
        img = np.searchsorted(off, obs, side="right") - 1
        first = np.ones(len(obs), bool)
        first[1:] = (img[1:] != img[:-1]) | (track[obs][1:] != track[obs][:-1])
        n_images = np.add.reduceat(first.astype(np.int64), track_off[:-1]) if T else np.zeros(0, np.int64)
        X = np.full((T, 6 if lines else 3), np.nan)
        status = np.full(T, TRK_TOO_LONG, np.int32)
        n_inl = np.zeros(T, np.int32)
        anchor, partner = np.full(T, -1), np.full(T, -1)
        winner, support, refit = np.full((T, 6 if lines else 3), np.nan), np.zeros(T, np.uint64), np.zeros(T, bool)
        inlier = np.zeros(Nn, np.uint8)
        n_views = np.zeros(Nn, np.int32)
        row_X = np.full((Nn, 6 if lines else 3), np.nan)
        with np.errstate(all="ignore"):
            for V in np.unique(n_obs):
                if V > TRK_MAX_OBS:
                    continue
                V = int(V)
                sel = np.flatnonzero(n_obs == V)
                nodes = obs[track_off[sel][:, None] + np.arange(V)[None, :]]
                o = _Obs(S, nodes, off, pool, lines)
                r = _estimate(o, V, len(sel), lines, t2, cos_min, sin2_min)
                ninl = _popcount(r["mask"])
                st = np.where(~r["have"], TRK_NO_CANDIDATE, np.where(ninl >= int(min_views), TRK_OK, TRK_TOO_FEW))
                valid = st == TRK_OK
                status[sel], n_inl[sel] = st, ninl
                X[sel] = np.where(valid[:, None], r["X"], np.nan)
                anchor[sel], partner[sel], winner[sel] = r["anchor"], r["partner"], r["winner"]
                support[sel], refit[sel] = r["support"], r["refit"]
                for q, b in enumerate(_bits(r["mask"], V)):
                    rows = nodes[b, q]
                    inlier[rows] = 1
                    vq = b & valid
                    rows = nodes[vq, q]
                    n_views[rows] = ninl[vq]
                    if not lines:
                        row_X[rows] = r["X"][vq]
                        continue
                    Xa, Xb = r["X"][vq, :3].T, r["X"][vq, 3:].T
                    d = [Xb[k] - Xa[k] for k in range(3)]
                    Cq = [c[vq, q] for c in o.C]
                    w = [Xa[k] - Cq[k] for k in range(3)]
                    for e, r_e in enumerate((o.r0, o.r1)):
                        row_X[rows, 3 * e:3 * e + 3] = np.stack(closest_on_line(Xa, d, w, [x[vq, q] for x in r_e]), 1)
        out.update({f"track_{kind}": track.astype(np.int32), f"n_tracks_{kind}": T,
                    f"track_off_{kind}": track_off.astype(np.int32), f"obs_{kind}": obs.astype(np.int32),
                    f"n_obs_{kind}": n_obs.astype(np.int32), f"n_inliers_{kind}": n_inl,
                    f"n_images_{kind}": n_images.astype(np.int32), f"status_{kind}": status,
                    f"inlier_{kind}": inlier, f"n_views_{kind}": n_views, f"edges_{kind}": edges,
                    f"label_{kind}": label, f"anchor_{kind}": anchor, f"partner_{kind}": partner,
                    f"winner_{kind}": winner if not lines else winner.reshape(T, 2, 3), f"support_{kind}": support,
                    f"refit_{kind}": refit})
        if lines:
            out["lines3d"], out["row_lines3d"] = X.reshape(T, 2, 3), row_X.reshape(Nn, 2, 3)
        else:
            out["points3d"], out["row_points3d"] = X, row_X
    return out


# ------------------------------------------------------------------ batched on the GPU
@dataclass
class TrackResult:
    """Result of `triangulate_tracks` (device tensors; nothing has been waited for).

    Per keypoint row (image i's from offsets_p[i]) / key-line row: track_p / track_l int32 (-1: in no track),
    inlier_p / inlier_l uint8 (a supporter of its track's kept estimate).  n_tracks_p / n_tracks_l: device int32 [1].
    Per track t < n_tracks (the tensors are sized by the bound of half the rows; later entries are not written):
    track_off_* [T + 1] and obs_* (its rows, ascending, at obs[track_off[t]:track_off[t + 1]]), points3d [T, 3] /
    lines3d [T, 2, 3] fp64 (NaN unless status is TRK_OK; a line's end points are those of its anchor observation),
    n_obs_*, n_inliers_*, n_images_* (distinct images among the observations: fewer than n_obs flags a merged track)
    and status_* (TRK_OK, TRK_TOO_LONG, TRK_NO_CANDIDATE, TRK_TOO_FEW).  row_points3d / row_lines3d and n_views_p /
    n_views_l hold the per-row coordinates `rows()` returns.  offsets_p / offsets_l: host int64 [n + 1]."""
    track_p: torch.Tensor
    track_l: torch.Tensor
    n_tracks_p: torch.Tensor
    n_tracks_l: torch.Tensor
    track_off_p: torch.Tensor
    track_off_l: torch.Tensor
    obs_p: torch.Tensor
    obs_l: torch.Tensor
    points3d: torch.Tensor
    lines3d: torch.Tensor
    n_obs_p: torch.Tensor
    n_obs_l: torch.Tensor
    n_inliers_p: torch.Tensor
    n_inliers_l: torch.Tensor
    n_images_p: torch.Tensor
    n_images_l: torch.Tensor
    status_p: torch.Tensor
    status_l: torch.Tensor
    inlier_p: torch.Tensor
    inlier_l: torch.Tensor
    row_points3d: torch.Tensor
    row_lines3d: torch.Tensor
    n_views_p: torch.Tensor
    n_views_l: torch.Tensor
    offsets_p: np.ndarray
    offsets_l: np.ndarray

    def n_tracks(self):
        """(point tracks, line tracks) on the host (waits for the call)."""
        return int(self.n_tracks_p.item()), int(self.n_tracks_l.item())

    def rows(self) -> TriangulationResult:
        """Per row: the track's point (a key line: the points of its track's line closest to the row's own two end-point
        rays) for the inlier rows of valid tracks, NaN elsewhere; n_views = the track's inlier count, else 0.  Its
        `per_image()` feeds `estimate_absolute_poses` as `triangulate`'s does."""
        Np, Nl = int(self.offsets_p[-1]), int(self.offsets_l[-1])
        return TriangulationResult(self.row_points3d[:Np], self.row_lines3d[:Nl], self.n_views_p[:Np],
                                   self.n_views_l[:Nl], self.offsets_p, self.offsets_l)


def triangulate_tracks(keypoints, klines, pairs, res, K, R, t, thresh=4.0, min_angle=1.5, min_views=2, epi_thresh=4.0,
                       min_overlap=0.5) -> TrackResult:
    """Point and line tracks of n posed images and one world point or world line per track, from the matches `res` (an
    `ImagePairMatches`, as `match_set(images, pairs)` returns) of the host pair list pairs [P, 2], in one `ltr_tracks`
    call (six kernel launches, no synchronisation).  Arguments as `triangulation.triangulate`; epi_thresh (pixels) and
    min_overlap decide which matches agree with the poses.  Raises LtrError before any device work on the arguments
    `triangulate` refuses, except that an image may take part in any number of pairs."""
    S = check_set(keypoints, klines, pairs, res, K, R, t, _WHO)
    _check_params(thresh, min_angle, min_views, epi_thresh, min_overlap)
    n, P = len(keypoints), len(S.pairs)
    dev = res.matches_p.device
    op, ol = offsets(S.n_kp), offsets(S.n_kl)
    Np, Nl = int(op[-1]), int(ol[-1])
    Tp, Tl = max(Np // 2, 1), max(Nl // 2, 1)
    f64, i32 = dict(dtype=torch.float64, device=dev), dict(dtype=torch.int32, device=dev)
    rp, rl = max(Np, 1), max(Nl, 1)
    o = dict(track_p=torch.empty(rp, **i32), track_l=torch.empty(rl, **i32), n_tracks_p=torch.zeros(1, **i32),
             n_tracks_l=torch.zeros(1, **i32), track_off_p=torch.zeros(Tp + 1, **i32),
             track_off_l=torch.zeros(Tl + 1, **i32), obs_p=torch.empty(rp, **i32), obs_l=torch.empty(rl, **i32),
             points3d=torch.empty((Tp, 3), **f64), lines3d=torch.empty((Tl, 2, 3), **f64),
             n_obs_p=torch.empty(Tp, **i32), n_obs_l=torch.empty(Tl, **i32), n_inliers_p=torch.empty(Tp, **i32),
             n_inliers_l=torch.empty(Tl, **i32), n_images_p=torch.empty(Tp, **i32), n_images_l=torch.empty(Tl, **i32),
             status_p=torch.empty(Tp, **i32), status_l=torch.empty(Tl, **i32),
             inlier_p=torch.empty(rp, dtype=torch.uint8, device=dev),
             inlier_l=torch.empty(rl, dtype=torch.uint8, device=dev), row_points3d=torch.empty((rp, 3), **f64),
             row_lines3d=torch.empty((rl, 2, 3), **f64), n_views_p=torch.empty(rp, **i32),
             n_views_l=torch.empty(rl, **i32), workspace=torch.empty(max(5 * (Np + Nl), 1), **i32))
    if n == 0 or Np + Nl == 0:
        o["track_p"].fill_(-1)
        o["track_l"].fill_(-1)
    else:
        arrays = {"K": S.K, "R": S.R, "t": S.t, "F": pair_fundamentals(S).reshape(-1, 9) if P else np.zeros((1, 9)),
                  "pairs": S.pairs.reshape(-1, 2) if P else np.zeros((1, 2), np.int32),
                  "cu_p": np.asarray(res.offsets_p, dtype=np.int32), "cu_l": np.asarray(res.offsets_l, dtype=np.int32),
                  "kp_off": op, "seg_off": ol}
        dv = stage_with_pools(arrays, keypoints, klines, dev)
        _ops.call_struct("ltr_tracks",
                         {**dv, "matches_p": res.matches_p.contiguous(), "matches_l": res.matches_l.contiguous(),
                          "n_images": n, "n_pairs": P, "total_p": int(res.offsets_p[-1]),
                          "total_l": int(res.offsets_l[-1]), "n_kp": Np, "n_kl": Nl, "thresh": thresh,
                          "min_angle": min_angle, "min_views": min_views, "epi_thresh": epi_thresh,
                          "min_overlap": min_overlap},
                         o, workspace_bytes=4 * 5 * (Np + Nl))
    del o["workspace"]     # the caching allocator reuses it only behind this stream's kernels
    return TrackResult(**o, offsets_p=op.astype(np.int64), offsets_l=ol.astype(np.int64))
