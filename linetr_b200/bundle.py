"""Bundle adjustment of posed image sets: the camera poses, the world points of the point tracks and the world lines of
the line tracks of `tracks.triangulate_tracks` refined together, on the GPU.

    bundle_adjust(keypoints, klines, K, R, t, tracks, fixed=(0,), max_iters=50, ftol=1e-10) -> BundleResult
        one `ltr_bundle_adjust` call; device outputs, no synchronisation
    bundle_adjust_host(...) -> dict
        the same model in numpy: every operation is the kernels' operation in the kernels' order, so the outputs are
        the same bits

The model (DESIGN.md "Bundle adjustment", include/linetr_b200.h `ltr_bundle_adjust`): a track takes part iff its
tracks status is TRK_OK and its inlier rows lie in distinct images, and its undamped initial normal block is not
degenerate.  A point row gives its two reprojection errors (x, y), a key-line row the signed pixel distances n . P / P_z
of the track's two world end points to the row's infinite line; the cost is their sum of squares.  A camera moves as
R <- cay(w) R, C <- C + dC (t = -R C); a point has 3 DoF; a line's end points each move in the plane orthogonal to its
direction d = X_b - X_a (basis u1 = normalize(d x e_k), e_k the first-smallest |d_k|, u2 = normalize(d x u1)).  Images
in `fixed` keep their pose; with exactly one fixed image f, the lowest free image k with a participating row also holds
the first-largest coordinate of its input C_k - C_f.  Levenberg-Marquardt (A + lambda diag A, lambda from 1e-3, x0.1 on
an accepted step, x10 on a rejected one) with a Schur complement onto the cameras: per-track Cholesky of the landmark
blocks, the reduced camera matrix assembled in ascending track order, a dense right-looking Cholesky and two triangular
solves, then the landmark steps.  A step is accepted iff every factorization succeeds, every participating depth stays
> 0 and the cost falls.  Everything is explicitly rounded fp64 in a fixed order.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

from . import _native as N
from . import _ops
from ._posed import (block_sum, cayley, centre, check_poses, cholesky_solve, closest_on_line, cross3, dot3,
                     line_normal, offsets, pool64, ray, row_counts, stage_with_pools)
from .triangulation import TriangulationResult

BA_MAX_IMAGES, BA_MAX_ITERS = N.BA_MAX_IMAGES, N.BA_MAX_ITERS
BA_IN, BA_NOT_VALID, BA_SAME_IMAGE, BA_DEGENERATE = N.BA_IN, N.BA_NOT_VALID, N.BA_SAME_IMAGE, N.BA_DEGENERATE
BA_STOP_ITERS, BA_STOP_FTOL, BA_STOP_LAMBDA = N.BA_STOP_ITERS, N.BA_STOP_FTOL, N.BA_STOP_LAMBDA
BA_LAMBDA0, BA_ACCEPT, BA_REJECT, BA_LAMBDA_MAX = 1e-3, 0.1, 10.0, 1e32
BA_DEGENERATE_PIVOT = 1e-12   # relative pivot of the undamped initial landmark block below which a track is left out
BA_COST_THREADS = 256         # the cost reduction's thread count (_posed.block_sum)
STATS = ("initial_cost", "final_cost", "lambda", "iterations", "accepted", "stop_reason", "n_obs", "n_tracks")
_WHO = "bundle_adjust"


# ------------------------------------------------------------------ arguments
def _get(tr, name):
    v = tr[name] if isinstance(tr, dict) else getattr(tr, name)
    return v.cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)


def _check(keypoints, klines, K, R, t, tracks, fixed, max_iters, ftol):
    """The host checks of `bundle_adjust` (before any device work) -> (n, K, R, t, sorted fixed images)."""
    n = len(keypoints)
    if len(klines) != n:
        raise N.LtrError(f"{_WHO}: {n} keypoint arrays but {len(klines)} key-line arrays")
    if n > BA_MAX_IMAGES:
        raise N.LtrError(f"{_WHO}: {n} images exceed LTR_BA_MAX_IMAGES = {BA_MAX_IMAGES}")
    n_kp, n_kl = row_counts(keypoints, 2, "keypoints", _WHO), row_counts(klines, 4, "klines", _WHO)
    for nm, cnt in (("offsets_p", n_kp), ("offsets_l", n_kl)):
        off = np.asarray(tracks[nm] if isinstance(tracks, dict) else getattr(tracks, nm), dtype=np.int64)
        if off.shape != (n + 1,) or not np.array_equal(np.diff(off), cnt):
            raise N.LtrError(f"{_WHO}: the tracks' {nm} disagree with the rows of keypoints / klines")
    Kn, Rn, tn = check_poses(K, R, t, n, _WHO)
    fx = sorted({int(f) for f in fixed})
    if not fx:
        raise N.LtrError(f"{_WHO}: at least one image must be fixed")
    if fx[0] < 0 or fx[-1] >= n:
        raise N.LtrError(f"{_WHO}: fixed image indices must lie in [0, {n})")
    if not 0 <= int(max_iters) <= BA_MAX_ITERS:
        raise N.LtrError(f"{_WHO}: max_iters must lie in [0, LTR_BA_MAX_ITERS = {BA_MAX_ITERS}]")
    if not (math.isfinite(float(ftol)) and float(ftol) >= 0):
        raise N.LtrError(f"{_WHO}: ftol must be finite and >= 0")
    return n, Kn, Rn, tn, fx


def _centres(R, t):
    """C = -R^T t per image in the tracks' order: [n, 3]."""
    return np.stack(centre(R.reshape(-1, 9), t.T), 1)


def _hold(R, t, fixed):
    """The held centre coordinate of every image (the first-largest |C_i - C_f|; only used for the one image k) when
    exactly one image f is fixed, else -1 everywhere."""
    n = len(R)
    if len(fixed) != 1:
        return np.full(n, -1, np.int32)
    C = _centres(R, t)
    d = np.abs(C - C[fixed[0]])
    return np.argmax(d, 1).astype(np.int32)


# ------------------------------------------------------------------ the model in numpy
def _basis(X):
    """u1, u2 (3 arrays each) of lines X (6 arrays)."""
    d = [X[3 + k] - X[k] for k in range(3)]
    ad = [np.abs(x) for x in d]
    k = np.where(ad[1] < ad[0], 1, 0)
    k = np.where(ad[2] < np.where(k == 1, ad[1], ad[0]), 2, k)
    e = [np.where(k == j, 1.0, 0.0) for j in range(3)]
    v = cross3(d, e)
    nv = np.sqrt(dot3(v, v))
    u1 = [x / nv for x in v]
    w = cross3(d, u1)
    nw = np.sqrt(dot3(w, w))
    return u1, [x / nw for x in w]


def _residual(R, C, X, cam, ob, line):
    """One residual of a row at world point X: R [..., 9], C / X 3 arrays; cam (fx, fy, cx, cy); ob (dx, dy) for the
    two point residuals, or the line normal n (3 arrays).  -> list of (r, dr/dP) per residual, P."""
    D = [X[k] - C[k] for k in range(3)]
    P = [(R[..., 3 * e] * D[0] + R[..., 3 * e + 1] * D[1]) + R[..., 3 * e + 2] * D[2] for e in range(3)]
    fx, fy = cam[0], cam[1]
    z = np.zeros_like(P[2])
    if line:
        n = ob
        r = ((n[0] * P[0] + n[1] * P[1]) + n[2] * P[2]) / P[2]
        return [(r, [n[0] / P[2], n[1] / P[2], (n[2] - r) / P[2]])], P
    dx, dy = ob
    rx = (fx * P[0] - dx * P[2]) / P[2]
    ry = (fy * P[1] - dy * P[2]) / P[2]
    return [(rx, [fx / P[2], z, -(dx + rx) / P[2]]), (ry, [z, fy / P[2], -(dy + ry) / P[2]])], P


def _jac(R, P, g):
    """Camera Jacobian [6] (w, C) and world Jacobian [3] of a residual with dr/dP = g."""
    gX = [(R[..., k] * g[0] + R[..., 3 + k] * g[1]) + R[..., 6 + k] * g[2] for k in range(3)]
    c = cross3(P, g)
    return [2.0 * c[0], 2.0 * c[1], 2.0 * c[2], -gX[0], -gX[1], -gX[2]], gX


class _Kind:
    """The participating rows of one kind, padded per track: [T, Vm] arrays."""

    def __init__(self, line, rows, cnt, img, K, pool):
        self.line, self.rows, self.cnt, self.img = line, rows, cnt, img
        T, Vm = rows.shape
        self.mask = np.arange(Vm)[None, :] < cnt[:, None]
        Ki = K[img]
        self.cam = (Ki[..., 0, 0], Ki[..., 1, 1], Ki[..., 0, 2], Ki[..., 1, 2])
        px = pool[np.where(self.mask, rows, 0)]
        if line:
            self.ob = line_normal(*self.cam, px)
        else:
            self.ob = (px[..., 0] - self.cam[2], px[..., 1] - self.cam[3])
        self.k = 4 if line else 3

    def terms(self, Rs, Cs, X):
        """-> r [2], Jc [2][6], Jl [2][k] (each [T, Vm]), front [T, Vm] at cameras (Rs [n, 9], Cs [n, 3]) and
        landmarks X (list of 3 or 6 arrays [T])."""
        R = Rs[self.img]
        C = [Cs[self.img][..., e] for e in range(3)]
        Xb = [x[:, None] for x in X]
        if not self.line:
            res, P = _residual(R, C, Xb, self.cam, self.ob, False)
            r, Jc, Jl = [], [], []
            for rq, g in res:
                jc, gX = _jac(R, P, g)
                r.append(rq)
                Jc.append(jc)
                Jl.append(gX)
            return r, Jc, Jl, P[2] > 0
        u1, u2 = _basis(X)
        u1, u2 = [x[:, None] for x in u1], [x[:, None] for x in u2]
        r, Jc, Jl, front = [], [], [], None
        for e in range(2):
            res, P = _residual(R, C, Xb[3 * e:3 * e + 3], self.cam, self.ob, True)
            rq, g = res[0]
            jc, gX = _jac(R, P, g)
            a, b = dot3(gX, u1), dot3(gX, u2)
            z = np.zeros_like(a)
            r.append(rq)
            Jc.append(jc)
            Jl.append([a, b, z, z] if e == 0 else [z, z, a, b])
            front = P[2] > 0 if front is None else front & (P[2] > 0)
        return r, Jc, Jl, front

    def step(self, X, dl):
        """Landmarks X moved by the steps dl (k arrays)."""
        if not self.line:
            return [X[k] + dl[k] for k in range(3)]
        u1, u2 = _basis(X)
        return [X[k] + (u1[k] * dl[0] + u2[k] * dl[1]) for k in range(3)] + \
               [X[3 + k] + (u1[k] * dl[2] + u2[k] * dl[3]) for k in range(3)]


def _normal(kd: _Kind, Jl, r):
    """Per-track landmark block (full k x k, symmetric) and gradient: fixed-order sums over the rows."""
    T, Vm = kd.rows.shape
    k = kd.k
    V = [[np.zeros(T) for _ in range(k)] for _ in range(k)]
    g = [np.zeros(T) for _ in range(k)]
    for o in range(Vm):
        m = kd.mask[:, o]
        for q in range(2):
            for a in range(k):
                for b in range(a, k):
                    V[a][b] = np.where(m, V[a][b] + Jl[q][a][:, o] * Jl[q][b][:, o], V[a][b])
                g[a] = np.where(m, g[a] + Jl[q][a][:, o] * r[q][:, o], g[a])
    for a in range(k):
        for b in range(a):
            V[a][b] = V[b][a]
    return V, g


def _chol(V, rel=None):
    """Cholesky L of k x k blocks V (lists of arrays): -> (L lower, ok).  With rel, ok also needs every pivot
    d_c > rel * V_cc."""
    k = len(V)
    L = [[None] * k for _ in range(k)]
    ok = np.ones(V[0][0].shape, bool)
    for c in range(k):
        d = V[c][c]
        for p in range(c):
            d = d - L[c][p] * L[c][p]
        ok &= (d > (rel * V[c][c])) if rel is not None else (d > 0)
        L[c][c] = np.sqrt(np.where(d > 0, d, np.nan))
        for r_ in range(c + 1, k):
            s = V[r_][c]
            for p in range(c):
                s = s - L[r_][p] * L[c][p]
            L[r_][c] = s / L[c][c]
    return L, ok


def _cholsolve(L, b):
    k = len(L)
    y = [None] * k
    for c in range(k):
        s = b[c]
        for p in range(c):
            s = s - L[c][p] * y[p]
        y[c] = s / L[c][c]
    x = [None] * k
    for c in range(k - 1, -1, -1):
        s = y[c]
        for p in range(c + 1, k):
            s = s - L[p][c] * x[p]
        x[c] = s / L[c][c]
    return x


def _seq_sum(acc, group, key, vals, sign):
    """acc[group] += sign * vals, each group's values added one at a time in ascending key order."""
    order = np.lexsort((key, group))
    group, vals = group[order], vals[order]
    first = np.searchsorted(group, group, side="left")
    rank = np.arange(len(group)) - first
    acc = acc.copy()
    for k in range(int(rank.max()) + 1 if len(rank) else 0):
        sel = rank == k
        acc[group[sel]] = acc[group[sel]] + vals[sel] if sign > 0 else acc[group[sel]] - vals[sel]
    return acc


def _tracks_of(tr, line, n, off):
    """Participating-row layout of one kind of a TrackResult / triangulate_tracks_host dict -> (T bound, T, status,
    rows [T, Vm], cnt [T], img [T, Vm], X [T, 3|6], trk_status)."""
    s = "l" if line else "p"
    T = int(_get(tr, f"n_tracks_{s}").reshape(-1)[0]) if not isinstance(tr, dict) else int(tr[f"n_tracks_{s}"])
    Xall = _get(tr, "lines3d" if line else "points3d").reshape(-1, 6 if line else 3).astype(np.float64)
    Tb = len(Xall)
    toff = _get(tr, f"track_off_{s}").astype(np.int64)[:T + 1]
    obs = _get(tr, f"obs_{s}").astype(np.int64)
    st = _get(tr, f"status_{s}").astype(np.int32)[:T]
    inl = _get(tr, f"inlier_{s}").astype(bool)
    rows_l, cnt = [], np.zeros(T, np.int64)
    status = np.full(T, BA_NOT_VALID, np.int32)
    for t_ in range(T):
        if st[t_] != N.TRK_OK:
            continue
        o = obs[toff[t_]:toff[t_ + 1]]
        o = o[inl[o]]
        im = np.searchsorted(off, o, side="right") - 1
        if len(o) > 1 and (np.diff(im) == 0).any():
            status[t_] = BA_SAME_IMAGE
            continue
        status[t_] = BA_IN
        cnt[t_] = len(o)
        rows_l.append((t_, o))
    Vm = max(1, int(cnt.max()) if T else 1)
    rows = np.zeros((T, Vm), np.int64)
    for t_, o in rows_l:
        rows[t_, :len(o)] = o
    img = np.searchsorted(off, rows, side="right") - 1
    img = np.clip(img, 0, max(n - 1, 0))
    return Tb, T, status, rows, cnt, img, Xall[:T].copy(), st


def bundle_adjust_host(keypoints, klines, K, R, t, tracks, fixed=(0,), max_iters=50, ftol=1e-10) -> dict:
    """The bundle adjustment model in numpy (DESIGN.md "Bundle adjustment"), same arguments as `bundle_adjust` (the
    tracks a TrackResult or a `triangulate_tracks_host` dict).  -> dict of host arrays: R [n, 3, 3], t [n, 3],
    points3d [T_p, 3], lines3d [T_l, 2, 3] (the first n_tracks rows), status_p / status_l, residual_p / residual_l (per
    row), row_points3d / row_lines3d / n_views_p / n_views_l (`rows()`), stats (dict of STATS) and history (the cost
    of every accepted state, the initial one first) and C [n, 3] (the camera centres the adjustment holds, before t = -R C)."""
    n, Kn, R0, t0, fixed = _check(keypoints, klines, K, R, t, tracks, fixed, max_iters, ftol)
    op = np.asarray(_get(tracks, "offsets_p"), dtype=np.int64)
    ol = np.asarray(_get(tracks, "offsets_l"), dtype=np.int64)
    kp_pool, kl_pool = pool64(keypoints, 2), pool64(klines, 4)
    hold = _hold(R0, t0, fixed)
    Rs, Cs = R0.reshape(n, 9).copy(), _centres(R0, t0)
    free = np.ones(n, bool)
    free[fixed] = False
    kinds, Xs, info = [], [], []
    with np.errstate(all="ignore"):
        for line, off, pool in ((False, op, kp_pool), (True, ol, kl_pool)):
            Tb, T, status, rows, cnt, img, X, st = _tracks_of(tracks, line, n, off)
            kd = _Kind(line, rows, cnt, img, Kn, pool if len(pool) else np.zeros((1, pool.shape[1])))
            X = [X[:, k] for k in range(X.shape[1])]
            r, Jc, Jl, front = kd.terms(Rs, Cs, X)
            V, g = _normal(kd, Jl, r)
            _, okd = _chol(V, BA_DEGENERATE_PIVOT)
            status = np.where((status == BA_IN) & ~okd, BA_DEGENERATE, status).astype(np.int32)
            kd.cnt = np.where(status == BA_IN, kd.cnt, 0)
            kd.mask = np.arange(kd.rows.shape[1])[None, :] < kd.cnt[:, None]
            kinds.append(kd)
            Xs.append(X)
            info.append((Tb, T, status, st))
        # the system: free images with a participating row, ascending; image k holds one centre coordinate
        part = np.zeros(n, bool)
        for kd in kinds:
            part[kd.img[kd.mask]] = True
        sysimg = free & part
        kimg = int(np.flatnonzero(sysimg)[0]) if (len(fixed) == 1 and sysimg.any()) else -1
        col = np.full((n, 6), -1, np.int64)
        m = 0
        for i in range(n):
            if not sysimg[i]:
                continue
            for a in range(6):
                if i == kimg and a == 3 + hold[i]:
                    continue
                col[i, a] = m
                m += 1
        Tp = info[0][1]

        def cost_of(Rs_, Cs_, X_):
            costs, fr = [], True
            for kd, X in zip(kinds, X_):
                r, _, _, front = kd.terms(Rs_, Cs_, X)
                c = np.zeros(kd.rows.shape[0])
                for o in range(kd.rows.shape[1]):
                    mk = kd.mask[:, o]
                    for q in range(2):
                        c = np.where(mk, c + r[q][:, o] * r[q][:, o], c)
                    fr = fr and bool((front[:, o] | ~mk).all())
                costs.append(c)
            cc = np.concatenate(costs)
            return (block_sum(cc[:, None], BA_COST_THREADS)[0] if len(cc) else 0.0), fr

        cost, _ = cost_of(Rs, Cs, Xs)
        init_cost = cost
        lam, it, acc, stop = BA_LAMBDA0, 0, 0, BA_STOP_ITERS
        history = [cost]
        while it < int(max_iters):
            # per-track blocks
            per = []
            for kd, X in zip(kinds, Xs):
                r, Jc, Jl, _ = kd.terms(Rs, Cs, X)
                V, g = _normal(kd, Jl, r)
                Vd = [[V[a][b] if a != b else V[a][a] + lam * V[a][a] for b in range(kd.k)] for a in range(kd.k)]
                L, okl = _chol(Vd)
                W = [[Jc[0][a] * Jl[0][b] + Jc[1][a] * Jl[1][b] for b in range(kd.k)] for a in range(6)]
                Lb = [[None if x is None else x[:, None] for x in row] for row in L]
                Y = [_cholsolve(Lb, W[a]) for a in range(6)]
                per.append((r, Jc, W, Y, g, L, okl))
            ok = all(bool(p[6][kd.cnt > 0].all()) for p, kd in zip(per, kinds))
            # reduced camera system: every sum in ascending track order per image (pair)
            A = np.zeros((m, m))
            rhs = np.zeros(m)
            Ug, Uk, Uv, Gv, Sg, Sk, Sv, Rv = [], [], [], [], [], [], [], []
            for ki, (kd, (r, Jc, W, Y, g, L, okl)) in enumerate(zip(kinds, per)):
                cbase = Tp if ki else 0
                tt, oo = np.nonzero(kd.mask & sysimg[kd.img])
                Ug.append(kd.img[tt, oo])
                Uk.append(tt + cbase)
                Uv.append(np.stack([Jc[0][a][tt, oo] * Jc[0][b][tt, oo] + Jc[1][a][tt, oo] * Jc[1][b][tt, oo]
                                    for a in range(6) for b in range(6)], 1))
                Gv.append(np.stack([Jc[0][a][tt, oo] * r[0][tt, oo] + Jc[1][a][tt, oo] * r[1][tt, oo]
                                    for a in range(6)], 1))

                def dot(u, v):
                    d = u[0] * v[0]
                    for q in range(1, kd.k):
                        d = d + u[q] * v[q]
                    return d
                Rv.append(np.stack([dot([Y[a][q][tt, oo] for q in range(kd.k)], [g[q][tt] for q in range(kd.k)])
                                    for a in range(6)], 1))
                Vm = kd.rows.shape[1]
                for oi in range(Vm):
                    for oj in range(Vm):
                        sel = kd.mask[:, oi] & kd.mask[:, oj] & sysimg[kd.img[:, oi]] & sysimg[kd.img[:, oj]] & \
                            (kd.img[:, oi] >= kd.img[:, oj])
                        t2 = np.flatnonzero(sel)
                        if not len(t2):
                            continue
                        Sg.append(kd.img[t2, oi] * n + kd.img[t2, oj])
                        Sk.append(t2 + cbase)
                        Sv.append(np.stack([dot([Y[a][q][t2, oi] for q in range(kd.k)],
                                                [W[b][q][t2, oj] for q in range(kd.k)])
                                            for a in range(6) for b in range(6)], 1))
            cat = lambda xs, w: np.concatenate(xs) if xs else np.zeros((0, w) if w else 0, np.int64 if not w else None)
            U = _seq_sum(np.zeros((n, 36)), cat(Ug, 0).astype(np.int64), cat(Uk, 0), cat(Uv, 36), 1.0)
            gc = _seq_sum(np.zeros((n, 6)), cat(Ug, 0).astype(np.int64), cat(Uk, 0), cat(Gv, 6), 1.0)
            for a in range(6):
                U[:, 7 * a] = U[:, 7 * a] + lam * U[:, 7 * a]
            S0 = np.zeros((n * n, 36))
            S0[np.arange(n) * (n + 1)] = U
            S = _seq_sum(S0, cat(Sg, 0).astype(np.int64), cat(Sk, 0), cat(Sv, 36), -1.0)
            gs = _seq_sum(gc, cat(Ug, 0).astype(np.int64), cat(Uk, 0), cat(Rv, 6), -1.0)
            for i in np.flatnonzero(sysimg):
                for j in np.flatnonzero(sysimg[:i + 1]):
                    for a in range(6):
                        for b in range(6):
                            if col[i, a] >= 0 and col[j, b] >= 0 and col[i, a] >= col[j, b]:
                                A[col[i, a], col[j, b]] = S[i * n + j, 6 * a + b]
                for a in range(6):
                    if col[i, a] >= 0:
                        rhs[col[i, a]] = -gs[i, a]
            # the dense solver (skipped, with a zero camera step, once a landmark factorization has failed: the step is
            # rejected either way)
            x = rhs.copy()
            ok = ok and cholesky_solve(A, x)
            if not ok:
                x = np.zeros(m)
            dcam = np.zeros((n, 6))
            for i in range(n):
                for a in range(6):
                    if col[i, a] >= 0:
                        dcam[i, a] = x[col[i, a]]
            Rn, Cn = Rs.copy(), Cs.copy()
            si = np.flatnonzero(sysimg)
            if len(si):
                Q, Rc = cayley([dcam[si, 0], dcam[si, 1], dcam[si, 2]]), Rs[si]
                Rn[si] = np.stack([dot3(Q[i], Rc[:, k::3].T) for i in range(3) for k in range(3)], 1)
                Cn[si] = Cs[si] + dcam[si, 3:]
            Xn = []
            for (r, Jc, W, Y, g, L, okl), kd, X in zip(per, kinds, Xs):
                s = list(g)
                for o in range(kd.rows.shape[1]):
                    mk = kd.mask[:, o]
                    dc = dcam[kd.img[:, o]]
                    for q in range(kd.k):
                        dd = W[0][q][:, o] * dc[:, 0]
                        for a in range(1, 6):
                            dd = dd + W[a][q][:, o] * dc[:, a]
                        s[q] = np.where(mk, s[q] + dd, s[q])
                dl = [-v for v in _cholsolve(L, s)]
                Xc = kd.step(X, dl)
                Xn.append([np.where(kd.cnt > 0, a, b) for a, b in zip(Xc, X)])
            cnew, front = cost_of(Rn, Cn, Xn)
            it += 1
            if ok and front and cnew < cost:
                rel = (cost - cnew) / cost
                Rs, Cs, Xs, cost = Rn, Cn, Xn, cnew
                lam, acc = lam * BA_ACCEPT, acc + 1
                history.append(cost)
                if rel <= float(ftol):
                    stop = BA_STOP_FTOL
                    break
            else:
                lam = lam * BA_REJECT
                if lam > BA_LAMBDA_MAX:
                    stop = BA_STOP_LAMBDA
                    break
        # outputs
        moved = sysimg & (acc > 0)
        Ro, to = R0.copy(), t0.copy()
        for i in np.flatnonzero(moved):
            Ri = Rs[i]
            Ro[i] = Ri.reshape(3, 3)
            to[i] = [-((Ri[3 * e] * Cs[i, 0] + Ri[3 * e + 1] * Cs[i, 1]) + Ri[3 * e + 2] * Cs[i, 2]) for e in range(3)]
        Cf = _centres(Ro, to)
        out = dict(R=Ro, t=to, C=Cs.copy(), history=np.array(history))
        n_obs_used = 0
        n_trk_used = 0
        for ki, (kd, X, (Tb, T, status, st)) in enumerate(zip(kinds, Xs, info)):
            s = "l" if kd.line else "p"
            off = ol if kd.line else op
            Nr = int(off[-1])
            r, _, _, _ = kd.terms(Rs, Cs, X)
            res = np.full(Nr, np.nan)
            rr = kd.rows[kd.mask]
            if kd.line:
                res[rr] = np.maximum(np.abs(r[0]), np.abs(r[1]))[kd.mask]
            else:
                res[rr] = np.sqrt(r[0] * r[0] + r[1] * r[1])[kd.mask]
            out[f"residual_{s}"] = res
            out[f"status_{s}"] = status
            Xa = np.stack(X, 1) if T else np.zeros((0, 6 if kd.line else 3))
            out["lines3d" if kd.line else "points3d"] = Xa.reshape(T, 2, 3) if kd.line else Xa
            n_obs_used += int(kd.cnt.sum())
            n_trk_used += int((status == BA_IN).sum())
            # rows(): every inlier row of a TRK_OK track
            trk = _get(tracks, f"track_{s}").astype(np.int64)[:Nr]
            inl = _get(tracks, f"inlier_{s}").astype(bool)[:Nr]
            nv = _get(tracks, f"n_views_{s}").astype(np.int32)[:Nr]
            rowsel = np.flatnonzero((trk >= 0) & inl)
            rowsel = rowsel[st[trk[rowsel]] == N.TRK_OK]
            rowX = np.full((Nr, 6 if kd.line else 3), np.nan)
            tt = trk[rowsel]
            if not kd.line:
                rowX[rowsel] = Xa[tt]
            else:
                im = np.searchsorted(off, rowsel, side="right") - 1
                Ri = Ro[im].reshape(-1, 9)
                Kr = Kn[im]
                fx, fy, cx, cy = Kr[:, 0, 0], Kr[:, 1, 1], Kr[:, 0, 2], Kr[:, 1, 2]
                seg = kl_pool[rowsel]
                Xa_, Xb_ = Xa[tt, :3].T, Xa[tt, 3:].T
                d = [Xb_[k] - Xa_[k] for k in range(3)]
                w = [Xa_[k] - Cf[im, k] for k in range(3)]
                for e in range(2):
                    r_e = ray(Ri, fx, fy, cx, cy, seg[:, 2 * e], seg[:, 2 * e + 1])
                    rowX[rowsel, 3 * e:3 * e + 3] = np.stack(closest_on_line(Xa_, d, w, r_e), 1)
            out["row_lines3d" if kd.line else "row_points3d"] = rowX.reshape(Nr, 2, 3) if kd.line else rowX
            out[f"n_views_{s}"] = nv
    out["stats"] = dict(initial_cost=float(init_cost), final_cost=float(cost), **{"lambda": float(lam)},
                        iterations=it, accepted=acc, stop_reason=stop, n_obs=n_obs_used, n_tracks=n_trk_used)
    return out


# ------------------------------------------------------------------ batched on the GPU
@dataclass
class BundleResult:
    """Result of `bundle_adjust` (device tensors; nothing has been waited for).

    R [n, 3, 3], t [n, 3] fp64 (the input bits for an image whose pose did not move); points3d [T_p, 3] / lines3d
    [T_l, 2, 3] (refined for BA_IN tracks, passed through otherwise) and status_p / status_l int32 (BA_IN,
    BA_NOT_VALID, BA_SAME_IMAGE, BA_DEGENERATE) per track, entries past the track counts not written; residual_p /
    residual_l fp64 per row (a participating point row's reprojection error, a participating key-line row's larger
    end-point distance, NaN elsewhere); stats fp64 [8] in the order of STATS.  row_points3d / row_lines3d and n_views_p
    / n_views_l hold what `rows()` returns.  offsets_p / offsets_l: host int64 [n + 1]."""
    R: torch.Tensor
    t: torch.Tensor
    points3d: torch.Tensor
    lines3d: torch.Tensor
    status_p: torch.Tensor
    status_l: torch.Tensor
    residual_p: torch.Tensor
    residual_l: torch.Tensor
    row_points3d: torch.Tensor
    row_lines3d: torch.Tensor
    n_views_p: torch.Tensor
    n_views_l: torch.Tensor
    stats: torch.Tensor
    offsets_p: np.ndarray
    offsets_l: np.ndarray

    def stats_dict(self) -> dict:
        """The stats on the host (waits for the call)."""
        s = self.stats.cpu().numpy()
        return {k: (float(v) if i < 3 else int(v)) for i, (k, v) in enumerate(zip(STATS, s))}

    def rows(self) -> TriangulationResult:
        """Per row, as `TrackResult.rows()` but under the refined poses: the track's point (a key line: the points of
        its track's line closest to the row's own two end-point rays) for the inlier rows of valid tracks, NaN
        elsewhere.  Its `per_image()` feeds `estimate_absolute_poses`."""
        Np, Nl = int(self.offsets_p[-1]), int(self.offsets_l[-1])
        return TriangulationResult(self.row_points3d[:Np], self.row_lines3d[:Nl], self.n_views_p[:Np],
                                   self.n_views_l[:Nl], self.offsets_p, self.offsets_l)


def bundle_adjust(keypoints, klines, K, R, t, tracks, fixed=(0,), max_iters=50, ftol=1e-10) -> BundleResult:
    """Refine the poses R [n, 3, 3], t [n, 3] of n images and the world points and lines of `tracks` (the TrackResult
    of `triangulate_tracks(keypoints, klines, pairs, res, K, R, t, ...)`) together, in one `ltr_bundle_adjust` call
    with no synchronisation.  Images in `fixed` keep their pose.  Raises LtrError before any device work on bad
    arguments: no fixed image or one out of range, offsets that disagree with keypoints / klines, more than
    BA_MAX_IMAGES images, max_iters < 0, or a non-finite or negative ftol."""
    n, Kn, Rn, tn, fixed = _check(keypoints, klines, K, R, t, tracks, fixed, max_iters, ftol)
    dev = tracks.points3d.device
    _ops._req_cuda(tracks.points3d, "tracks")
    op, ol = np.asarray(tracks.offsets_p, np.int64), np.asarray(tracks.offsets_l, np.int64)
    Np, Nl = int(op[-1]), int(ol[-1])
    Tp, Tl = len(tracks.points3d), len(tracks.lines3d)
    fx = np.zeros(n, np.int32)
    fx[fixed] = 1
    f64, i32 = dict(dtype=torch.float64, device=dev), dict(dtype=torch.int32, device=dev)
    rp, rl = max(Np, 1), max(Nl, 1)
    ws = N.ba_workspace_bytes(n, Np, Nl, Tp, Tl)
    o = dict(R=torch.empty((n, 3, 3), **f64), t=torch.empty((n, 3), **f64), points3d=torch.empty((Tp, 3), **f64),
             lines3d=torch.empty((Tl, 2, 3), **f64), status_p=torch.empty(Tp, **i32), status_l=torch.empty(Tl, **i32),
             residual_p=torch.empty(rp, **f64), residual_l=torch.empty(rl, **f64),
             row_points3d=torch.empty((rp, 3), **f64), row_lines3d=torch.empty((rl, 2, 3), **f64),
             n_views_p=torch.empty(rp, **i32), n_views_l=torch.empty(rl, **i32), stats=torch.empty(8, **f64),
             workspace=torch.empty(-(-ws // 8), **f64))
    arrays = {"K": Kn, "R": Rn, "t": tn, "kp_off": offsets(np.diff(op)), "seg_off": offsets(np.diff(ol)),
              "hold": np.maximum(_hold(Rn, tn, fixed), 0).astype(np.int32), "fixed": fx}
    dv = stage_with_pools(arrays, keypoints, klines, dev)
    for nm in ("n_tracks_p", "n_tracks_l", "track_off_p", "track_off_l", "obs_p", "obs_l", "status_p", "status_l",
               "inlier_p", "inlier_l", "track_p", "track_l", "n_views_p", "n_views_l", "points3d", "lines3d"):
        dv[nm] = getattr(tracks, nm).contiguous()
    dv["segs"] = dv["segs"].reshape(-1, 4)
    _ops.call_struct("ltr_bundle_adjust", {**dv, "n_images": n, "n_fixed": len(fixed), "n_kp": Np, "n_kl": Nl,
                                           "t_p": Tp, "t_l": Tl, "max_iters": max_iters, "ftol": ftol},
                     o, workspace_bytes=ws)
    del o["workspace"]     # the caching allocator reuses it only behind this stream's kernels
    return BundleResult(**o, offsets_p=op, offsets_l=ol)
