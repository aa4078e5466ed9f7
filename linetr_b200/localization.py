"""Visual localization: the absolute pose of query images from their point and line matches to database images with
3D coordinates (PL-Loc's last step), batched on the GPU, and the localization metrics.

    estimate_absolute_poses(res, K0, points3d1, lines3d1=None, groups=None, thresh=8.0, n_hypotheses=1024, seed=0,
                            use_lines=True, n_line_hypotheses=0) -> AbsolutePoseResult
        one `ltr_absolute_pose_lines` call for every query (group of pairs) of a `match_images` / `match_sets` result;
        device outputs, no synchronisation
    ransac_absolute_pose_host(kpts0, matches_p, points3d1, K0, klines0=None, matches_l=None, lines3d1=None, ...)
        the same model for one group in numpy: every operation is the kernels' operation in the kernels' order, the
        refit included, so the winner, its inlier count and the refitted pose are the same bits
    p3p_solutions(bearings, X): the point solver; p2p1l_solutions, p1p2l_solutions, p3l_solutions: the line solvers
        (line_pose_solutions), all three through trig_pair_roots; refine_pose_host: the refit
    absolute_pose_errors, localization_recall: rotation / camera-centre errors and the InLoc recall bins
    lift_to_3d: 3D coordinates of database keypoints / segment end points from a depth map

The model (DESIGN.md "Absolute pose", include/linetr_b200.h `ltr_absolute_pose`): side 0 is the query, side 1 a
database image whose keypoints (and key-line end points) have world coordinates; the pose maps world to query camera,
X_cam = R X + t.  A group of pairs (one query against several database images) gives one pose from its pairs' point
rows in pair and row order (a matched side-0 keypoint whose partner has finite 3D), then its line rows (a matched side-0
segment whose partner has two finite 3D end points).  World coordinates are shifted by the midpoint c of the bounding
box of the group's staged 3D coordinates.  Hypothesis k draws 3 distinct point rows (`draw_samples(..., size=3)`) and
solves them with Grunert's P3P (Haralick et al. 1994, section 2.1): the quartic in v = s3 / s1, its real roots by
`sturm_roots`, positive distances only, the rotation from the triads of the camera and world points; solution j is
real root j.  Every operation is one explicitly rounded fp64 operation.  A point is an inlier iff its depth is > 0 and
its reprojection error in pixels is below thresh; a line iff both end points have depth > 0 and lie within thresh of
the line through its query segment.  The winner has the most inliers (points and lines), then the lowest k, then the
lowest j, and is refined by Levenberg-Marquardt over its inliers, kept iff the refit has at least as many inliers.
With n_line_hypotheses, three line solvers (P2P1L: 2 points and 1 line; P1P2L: 1 point and 2 lines; P3L: 3 lines)
add hypotheses that compete for the same winner at indices after the P3P ones.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

from . import _native as N
from . import _ops
from . import _posed
from ._posed import block_sum
from .geometry import SMEM_MAX, _intrinsics, _pool, draw_samples, sturm_roots

AP_SAMPLE = 3
AP_MAX_SOLUTIONS = 4
AP_COLLINEAR_EPS = 1e-10   # a sample whose world cross-product norm is at most this times the edge lengths is rejected
AP_MIN_REFIT = 3           # winner inliers needed for the refit
AP_LINE_MAX_SOLUTIONS = 8  # line solvers: solutions per sample (the real roots of a degree-8 polynomial)
AP_LINE_NP, AP_LINE_NL = (2, 1, 0), (1, 2, 3)   # point and line rows of a sample of P2P1L, P1P2L, P3L
AP_BEARING_EPS = 1e-10     # P2P1L: |j1 x j2| of the unit bearings at most this rejects the sample
AP_POINT_LINE_EPS = 1e-10  # P1P2L: |n1 . j1| / |n1| at most this (the query point on query line 1) rejects it
AP_CONCURRENT_EPS = 1e-10  # P3L: |n1 . (n2 x n3)| at most this times |n1| |n2| |n3| (concurrent query lines) rejects it
AP_LM_ITERS = 20           # Levenberg-Marquardt iterations (fixed budget)
AP_LM_LAMBDA0 = 1e-3       # initial damping (Marquardt: A_ii + lambda A_ii)
AP_LM_ACCEPT = 0.1         # damping factor after a step that lowers the cost
AP_LM_REJECT = 10.0        # damping factor after a step that does not
AP_FIT_THREADS = 256       # rows t, t + 256, ... are summed by thread t of the refit
# One group's staging in shared memory (ltr_absolute_pose's capacity): a point row is its fp32 query pixel and fp64
# world point, a line row its fp32 query segment and two fp64 world end points.
SMEM_PER_POINT_A, SMEM_PER_LINE_A = 32, 64


# ------------------------------------------------------------------ the model in numpy
def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def bearings(q):
    """Unit bearing vectors [..., 3] of normalised query coordinates q [..., 2]: (x, y, 1) / sqrt((x^2 + y^2) + 1)."""
    q = np.asarray(q, dtype=np.float64)
    x, y = q[..., 0], q[..., 1]
    nb = np.sqrt((x * x + y * y) + 1.0)
    return np.stack([x / nb, y / nb, 1.0 / nb], -1)


def grunert_quartic(j, X):
    """Grunert's quartic in v = s3 / s1 of samples j [K, 3, 3] (unit bearings of the three points) and X [K, 3, 3]
    (their world points): -> (ascending coefficients [K, 5], and the terms the back-substitution reuses)."""
    j1, j2, j3 = j[:, 0], j[:, 1], j[:, 2]
    X1, X2, X3 = X[:, 0], X[:, 1], X[:, 2]
    d1, d2, d3 = X2 - X1, X3 - X1, X3 - X2
    c2, b2, a2 = _dot(d1, d1), _dot(d2, d2), _dot(d3, d3)
    ca, cb, cg = _dot(j2, j3), _dot(j1, j3), _dot(j1, j2)
    p, q = (a2 - c2) / b2, (a2 + c2) / b2
    rc, ra, rbc, rba = c2 / b2, a2 / b2, (b2 - c2) / b2, (b2 - a2) / b2
    ca2, cb2, cg2 = ca * ca, cb * cb, cg * cg
    pm1, pp1, omq = p - 1.0, p + 1.0, 1.0 - q
    A4 = pm1 * pm1 - (4.0 * rc) * ca2
    A3 = 4.0 * (((p * (1.0 - p)) * cb - (omq * ca) * cg) + ((2.0 * rc) * ca2) * cb)
    A2 = 2.0 * (((((p * p - 1.0) + ((2.0 * (p * p)) * cb2)) + (2.0 * rbc) * ca2) - (((4.0 * q) * ca) * cb) * cg)
                + (2.0 * rba) * cg2)
    A1 = 4.0 * ((-((p * pp1) * cb) + ((2.0 * ra) * cg2) * cb) - (omq * ca) * cg)
    A0 = pp1 * pp1 - (4.0 * ra) * cg2
    return np.stack([A0, A1, A2, A3, A4], 1), dict(b2=b2, p=p, pm1=pm1, pp1=pp1, ca=ca, cb=cb, cg=cg, d1=d1, d2=d2, c2=c2)


def p3p_solutions(j, X):
    """Grunert's P3P (DESIGN.md "Absolute pose") on samples of unit bearings j [K, 3, 3] and world points X [K, 3, 3]:
    -> (R [K, 4, 3, 3], t [K, 4, 3], ok [K, 4]) with X_cam = R X + t; solution j is real root j (ascending) of the
    quartic.  A root is kept iff its back-substitution divisors are non-zero, both distance ratios u, v are > 0 and
    the pose is finite; a sample whose world points are collinear has none."""
    j, X = np.asarray(j, dtype=np.float64), np.asarray(X, dtype=np.float64)
    K = j.shape[0]
    with np.errstate(all="ignore"):
        A, w = grunert_quartic(j, X)
        d1, d2 = w["d1"], w["d2"]
        cr = _cross(d1, d2)
        n1, n2, ncr = np.sqrt(w["c2"]), np.sqrt(w["b2"]), np.sqrt(_dot(cr, cr))
        ok_s = ncr > (AP_COLLINEAR_EPS * n1) * n2
        poly = np.zeros((K, 11))
        poly[:, :5] = A
        roots, _ = sturm_roots(poly)
        v = roots[:, :AP_MAX_SOLUTIONS]
        live = ~np.isnan(v) & ok_s[:, None]
        v = np.where(live, v, 1.0)
        c = lambda a: a[:, None]
        v2 = v * v
        num = (c(w["pm1"]) * v2 - ((2.0 * c(w["p"])) * c(w["cb"])) * v) + c(w["pp1"])
        den = 2.0 * (c(w["cg"]) - v * c(w["ca"]))
        u = num / den
        den1 = (1.0 + v2) - (2.0 * v) * c(w["cb"])
        s1 = np.sqrt(c(w["b2"]) / den1)
        live &= (den != 0) & (den1 > 0) & (u > 0) & (v > 0)
        P1, P2, P3 = s1[..., None] * j[:, None, 0], (u * s1)[..., None] * j[:, None, 1], (v * s1)[..., None] * j[:, None, 2]
        f1, f2 = P2 - P1, P3 - P1
        m1 = np.sqrt(_dot(f1, f1))
        cc = _cross(f1, f2)
        mc = np.sqrt(_dot(cc, cc))
        g1, g3 = f1 / m1[..., None], cc / mc[..., None]
        g2 = _cross(g3, g1)
        e1, e3 = d1 / n1[:, None], cr / ncr[:, None]
        e2 = _cross(e3, e1)
        e1, e2, e3 = e1[:, None], e2[:, None], e3[:, None]
        R = np.empty((K, AP_MAX_SOLUTIONS, 3, 3))
        for i in range(3):
            for k in range(3):
                R[..., i, k] = (g1[..., i] * e1[..., k] + g2[..., i] * e2[..., k]) + g3[..., i] * e3[..., k]
        X1 = X[:, None, 0]
        t = P1 - ((R[..., 0] * X1[..., 0:1] + R[..., 1] * X1[..., 1:2]) + R[..., 2] * X1[..., 2:3])
        live &= np.isfinite(R).all((-1, -2)) & np.isfinite(t).all(-1)
    return R, t, live


# ------------------------------------------------------------------ line solvers (P2P1L, P1P2L, P3L)
def _unit(v):
    """(v / |v|, |v|) of vectors v [..., 3]."""
    n = np.sqrt(_dot(v, v))
    return v / n[..., None], n


def _mv(M, v):
    """M v for row-major M [..., 9] (or [..., 3, 3]) and v [..., 3]."""
    M = M.reshape(M.shape[:-2] + (9,)) if M.shape[-2:] == (3, 3) else M
    return np.stack([_dot(M[..., 3 * i:3 * i + 3], v) for i in range(3)], -1)


def trig_terms(n, E):
    """The coefficients [..., 9] of n' . Rz(a) Rx(b) E' (row-major; rows cos a, sin a, 1; columns cos b, sin b, 1)."""
    z = np.zeros(np.broadcast_shapes(n.shape, E.shape)[:-1])
    return np.stack([n[..., 1] * E[..., 1], -(n[..., 1] * E[..., 2]), n[..., 0] * E[..., 0],
                     -(n[..., 0] * E[..., 1]), n[..., 0] * E[..., 2], n[..., 1] * E[..., 0],
                     n[..., 2] * E[..., 2], n[..., 2] * E[..., 1], z], -1)


def _pmul(a, b):
    """a b over the last axis (ascending coefficients), each coefficient summed over a's index ascending from 0."""
    na, nb = a.shape[-1], b.shape[-1]
    out = []
    for k in range(na + nb - 1):
        acc = np.zeros(a.shape[:-1])
        for i in range(na):
            if 0 <= k - i < nb:
                acc = acc + a[..., i] * b[..., k - i]
        out.append(acc)
    return np.stack(out, -1)


def trig_pair_poly(M1, M2):
    """The core's polynomials of the equations [cos a, sin a, 1] M_i [cos b, sin b, 1]^T = 0, M1, M2 [K, 9] (row-major
    3 x 3): with tau = tan(b / 2), row r of M_i is the quadratic M_i[r,0] (1 - tau^2) + 2 M_i[r,1] tau + M_i[r,2]
    (1 + tau^2); A_i, B_i, C_i its rows 0, 1, 2.  -> (D = A1 B2 - A2 B1, X = B1 C2 - B2 C1, Y = A2 C1 - A1 C2 [K, 5],
    p = (X^2 + Y^2) - D^2 [K, 9]), ascending coefficients."""
    M1, M2 = np.asarray(M1, dtype=np.float64), np.asarray(M2, dtype=np.float64)
    q = [[np.stack([M[..., 3 * r] + M[..., 3 * r + 2], 2.0 * M[..., 3 * r + 1], M[..., 3 * r + 2] - M[..., 3 * r]], -1)
          for r in range(3)] for M in (M1, M2)]
    (A1, B1, C1), (A2, B2, C2) = q
    D = _pmul(A1, B2) - _pmul(A2, B1)
    X = _pmul(B1, C2) - _pmul(B2, C1)
    Y = _pmul(A2, C1) - _pmul(A1, C2)
    return D, X, Y, (_pmul(X, X) + _pmul(Y, Y)) - _pmul(D, D)


def _horner4(c, x):
    v = c[..., 4]
    for k in range(3, -1, -1):
        v = v * x + c[..., k]
    return v


def trig_pair_roots(M1, M2):
    """The two bilinear trigonometric equations' solutions (DESIGN.md "Absolute pose"): the real roots tau of p by
    `sturm_roots`, then at each (cos a, sin a) = (X, Y) / D normalised by their norm and (cos b, sin b) = (1 - tau^2,
    2 tau) / (1 + tau^2); a root with D == 0 is dropped.  Solution j is real root j (ascending).  -> (cs [K, 8, 4] of
    (cos a, sin a, cos b, sin b), ok [K, 8], p [K, 9])."""
    D, X, Y, p = trig_pair_poly(M1, M2)
    K = len(p)
    poly = np.zeros((K, 11))
    poly[:, :9] = p
    with np.errstate(all="ignore"):
        roots, _ = sturm_roots(poly)
        tau = roots[:, :AP_LINE_MAX_SOLUTIONS]
        ok = ~np.isnan(tau)
        tau = np.where(ok, tau, 0.0)
        c = lambda a: a[:, None, :]
        d = _horner4(c(D), tau)
        ok &= d != 0
        ca, sa = _horner4(c(X), tau) / d, _horner4(c(Y), tau) / d
        nr = np.sqrt(ca * ca + sa * sa)
        t2 = tau * tau
        den = 1.0 + t2
        cs = np.stack([ca / nr, sa / nr, (1.0 - t2) / den, (2.0 * tau) / den], -1)
    return cs, ok, p


def _triad(f):
    """Rows (f, u, v) [K, 3, 3] of unit f [K, 3]: u = f x e / |f x e| for the coordinate axis e least aligned with f
    (the first of the smallest |f_k|), v = f x u."""
    a = np.abs(f)
    k = np.where(a[:, 1] < a[:, 0], 1, 0)
    k = np.where(a[:, 2] < a[np.arange(len(f)), k], 2, k)
    e = np.zeros_like(f)
    e[np.arange(len(f)), k] = 1.0
    u, _ = _unit(_cross(f, e))
    return np.stack([f, u, _cross(f, u)], 1)


def line_pose_solutions(solver, j, X, n, E):
    """Line solver `solver` (0 P2P1L, 1 P1P2L, 2 P3L; DESIGN.md "Absolute pose") on K samples: unit bearings j and
    world points X [K, 2 - solver, 3] of the sample's points, camera-ray normals n [K, solver + 1, 3] of its query
    lines and world end points E [K, solver + 1, 2, 3] of its lines.  -> (R [K, 8, 3, 3], t [K, 8, 3], ok [K, 8]) with
    X_cam = R X + t; solution j is real root j of the degree-8 polynomial."""
    j, X = np.asarray(j, dtype=np.float64), np.asarray(X, dtype=np.float64)
    n, E = np.asarray(n, dtype=np.float64), np.asarray(E, dtype=np.float64)
    K = len(n)
    with np.errstate(all="ignore"):
        if solver == 0:
            w = X[:, 1] - X[:, 0]
            h1, _ = _unit(w)
            L = np.sqrt(_dot(w, w))
            H = _triad(h1)
            c = _cross(j[:, 0], j[:, 1])
            sg = np.sqrt(_dot(c, c))
            ok_s = sg > AP_BEARING_EPS
            gs = _dot(j[:, 0], j[:, 1]) / sg
            g3 = c / sg[:, None]
            G = np.stack([j[:, 0], _cross(g3, j[:, 0]), g3], 1)
            npr = _mv(G, n[:, 0])
            Ln = L * npr[:, 0]
            Ms = []
            for e in range(2):
                M = trig_terms(npr, _mv(H, E[:, 0, e] - X[:, 0]))
                M[:, 2] = M[:, 2] - Ln
                M[:, 5] = M[:, 5] + Ln * gs
                Ms.append(M)
        else:
            T = _triad(_unit(n[:, 0])[0])
            G = np.stack([T[:, 1], T[:, 2], T[:, 0]], 1)
            H = _triad(_unit(E[:, 0, 1] - E[:, 0, 0])[0])
            if solver == 1:
                m1, m2 = _dot(G[:, 2], j[:, 0]), _dot(n[:, 1], j[:, 0])
                ok_s = np.abs(m1) > AP_POINT_LINE_EPS
                npr = _mv(G, n[:, 1])
                M1 = trig_terms(npr, _mv(H, E[:, 1, 1] - E[:, 1, 0]))
                M2 = trig_terms(m1[:, None] * npr, _mv(H, E[:, 1, 0] - X[:, 0]))
                E1 = _mv(H, E[:, 0, 0] - X[:, 0])
                M2[:, 6] = M2[:, 6] - m2 * E1[:, 2]
                M2[:, 7] = M2[:, 7] - m2 * E1[:, 1]
                Ms = [M1, M2]
            else:
                det = _dot(n[:, 0], _cross(n[:, 1], n[:, 2]))
                nn = [np.sqrt(_dot(n[:, i], n[:, i])) for i in range(3)]
                ok_s = np.abs(det) > ((AP_CONCURRENT_EPS * nn[0]) * nn[1]) * nn[2]
                Ms = [trig_terms(_mv(G, n[:, e]), _mv(H, E[:, e, 1] - E[:, e, 0])) for e in (1, 2)]
        cs, ok, _ = trig_pair_roots(Ms[0], Ms[1])
        ok &= ok_s[:, None]
        ca, sa, cb, sb = (cs[..., i] for i in range(4))
        c = lambda a: a[:, None]
        if solver == 0:
            s2 = (c(L) * sa) / c(sg)
            s1 = c(L) * (c(gs) * sa - ca)
            ok &= (s1 > 0) & (s2 > 0)
        elif solver == 1:
            s1 = -(sb * c(E1[:, 1]) + cb * c(E1[:, 2])) / c(m1)
            ok &= s1 > 0
        z = np.zeros_like(ca)
        Rp = np.stack([ca, -(sa * cb), sa * sb, sa, ca * cb, -(ca * sb), z, sb, cb], -1).reshape(K, -1, 3, 3)
        Hb, Gb = H[:, None], G[:, None]
        W = np.empty_like(Rp)
        R = np.empty_like(Rp)
        for i in range(3):
            for k in range(3):
                W[..., i, k] = (Rp[..., i, 0] * Hb[..., 0, k] + Rp[..., i, 1] * Hb[..., 1, k]) + Rp[..., i, 2] * Hb[..., 2, k]
        for i in range(3):
            for k in range(3):
                R[..., i, k] = (Gb[..., 0, i] * W[..., 0, k] + Gb[..., 1, i] * W[..., 1, k]) + Gb[..., 2, i] * W[..., 2, k]
        if solver < 2:
            X1 = X[:, None, 0]
            t = np.stack([s1 * c(j[:, 0, i]) - _dot(R[..., i, :], X1) for i in range(3)], -1)
        else:
            t = _solve3(R, n, E)
        ok &= np.isfinite(R).all((-1, -2)) & np.isfinite(t).all(-1)
    return R, t, ok


def _solve3(R, n, E):
    """P3L's translations [K, S, 3]: n_i . t = -n_i . R A_i (A_i line i's first end point) by Gaussian elimination with
    partial pivoting (first largest |pivot|) and back substitution, as the kernels do."""
    K, S = R.shape[:2]
    A = np.empty((K, S, 3, 4))
    for i in range(3):
        RA = np.stack([_dot(R[..., r, :], E[:, None, i, 0]) for r in range(3)], -1)
        A[..., i, :3] = n[:, None, i]
        A[..., i, 3] = -_dot(n[:, None, i], RA)
    A = A.reshape(K * S, 3, 4)
    rows = np.arange(K * S)
    for cc in range(3):
        piv, best = np.full(K * S, cc), np.abs(A[:, cc, cc])
        for q in range(cc + 1, 3):
            m = np.abs(A[:, q, cc]) > best
            best, piv = np.where(m, np.abs(A[:, q, cc]), best), np.where(m, q, piv)
        top, pr = A[rows, cc].copy(), A[rows, piv].copy()
        A[rows, cc], A[rows, piv] = pr, top
        for q in range(cc + 1, 3):
            f = A[:, q, cc] / A[:, cc, cc]
            for k in range(cc + 1, 4):
                A[:, q, k] = A[:, q, k] - f * A[:, cc, k]
    t = np.zeros((K * S, 3))
    for i in range(2, -1, -1):
        acc = A[:, i, 3]
        for k in range(i + 1, 3):
            acc = acc - A[:, i, k] * t[:, k]
        t[:, i] = acc / A[:, i, i]
    return t.reshape(K, S, 3)


def p2p1l_solutions(j, X, n, E):
    """P2P1L: two points (unit bearings j [K, 2, 3], world points X [K, 2, 3]) and one line (normal n [K, 3], world
    end points E [K, 2, 3]).  -> `line_pose_solutions`' (R, t, ok)."""
    return line_pose_solutions(0, j, X, np.asarray(n)[:, None], np.asarray(E)[:, None])


def p1p2l_solutions(j, X, n, E):
    """P1P2L: one point (j [K, 3], X [K, 3]) and two lines (n [K, 2, 3], E [K, 2, 2, 3])."""
    return line_pose_solutions(1, np.asarray(j)[:, None], np.asarray(X)[:, None], n, E)


def p3l_solutions(n, E):
    """P3L: three lines (n [K, 3, 3], E [K, 3, 2, 3])."""
    K = len(n)
    return line_pose_solutions(2, np.zeros((K, 0, 3)), np.zeros((K, 0, 3)), n, E)


def _cam(R, t, X):
    """Camera coordinates (Px, Py, Pz) [M, n] of world points X [n, 3] under poses R [M, 3, 3], t [M, 3]."""
    R, t = R.reshape(-1, 9), t.reshape(-1, 3)
    return [((R[:, 3 * i:3 * i + 1] * X[None, :, 0] + R[:, 3 * i + 1:3 * i + 2] * X[None, :, 1])
             + R[:, 3 * i + 2:3 * i + 3] * X[None, :, 2]) + t[:, i:i + 1] for i in range(3)]


def line_normals(seg0, K):
    """The query line of every segment s0 [m, 2, 2] (used as float32) in camera-ray form [m, 3]: the pixel line
    (a, b, c) through s0 scaled to a^2 + b^2 = 1, then n = (a fx, b fy, (a cx + b cy) + c), so that n . P / Pz is the
    signed pixel distance of the projection of the camera point P to the line."""
    s = np.asarray(seg0, dtype=np.float32).reshape(-1, 4).astype(np.float64)
    with np.errstate(all="ignore"):
        return np.stack(_posed.line_normal(K[0, 0], K[1, 1], K[0, 2], K[1, 2], s), 1)


@dataclass
class _Group:
    K: np.ndarray        # [3, 3]
    d: np.ndarray        # [np, 2] query pixel minus the principal point
    X: np.ndarray        # [np, 3] shifted world points
    n: np.ndarray        # [nl, 3] camera-ray line normals
    E: np.ndarray        # [nl, 2, 3] shifted world end points
    c: np.ndarray        # [3] the shift


def _inliers(g: _Group, R, t, t2, chunk=256):
    """Inlier flags [M, np + nl] of poses R [M, 3, 3], t [M, 3]: points, then lines."""
    R, t = R.reshape(-1, 3, 3), t.reshape(-1, 3)
    fx, fy = g.K[0, 0], g.K[1, 1]
    out = np.empty((len(R), len(g.X) + len(g.E)), dtype=bool)
    with np.errstate(all="ignore"):
        for s in range(0, len(R), chunk):
            Rc, tc = R[s:s + chunk], t[s:s + chunk]
            Px, Py, Pz = _cam(Rc, tc, g.X)
            ex, ey = fx * Px - g.d[None, :, 0] * Pz, fy * Py - g.d[None, :, 1] * Pz
            fp = (Pz > 0) & ((ex * ex + ey * ey) < t2 * (Pz * Pz))
            fl = np.ones((len(Rc), len(g.E)), dtype=bool)
            for e in range(2):
                Qx, Qy, Qz = _cam(Rc, tc, g.E[:, e])
                dd = (g.n[None, :, 0] * Qx + g.n[None, :, 1] * Qy) + g.n[None, :, 2] * Qz
                fl &= (Qz > 0) & ((dd * dd) < t2 * (Qz * Qz))
            out[s:s + chunk] = np.concatenate([fp, fl], 1)
    return out


_TRI = [(a, b) for a in range(6) for b in range(a, 6)]   # the 21 entries of J^T J, row-major upper triangle


def _row_terms(g: _Group, R, t, rows):
    """Per-row terms [n, 28] of the refit at pose (R, t): J^T J (upper triangle), J^T r and r^T r of each row's two
    residual components (a point's pixel x / y residuals, a line's two signed end-point distances); rows outside
    `rows` (bool [np + nl]) are 0."""
    npt = len(g.X)
    fx, fy = g.K[0, 0], g.K[1, 1]
    out = np.zeros((npt + len(g.E), 28))
    with np.errstate(all="ignore"):
        def jac(Xw, gx, gy, gz):   # (2 (R X) x g, g)
            Y = np.stack([(R[i, 0] * Xw[:, 0] + R[i, 1] * Xw[:, 1]) + R[i, 2] * Xw[:, 2] for i in range(3)], 1)
            gg = np.stack([gx, gy, gz], 1)
            return np.concatenate([2.0 * _cross(Y, gg), gg], 1)

        def terms(J0, r0, J1, r1):
            o = np.empty((len(r0), 28))
            for e, (a, b) in enumerate(_TRI):
                o[:, e] = J0[:, a] * J0[:, b] + J1[:, a] * J1[:, b]
            for a in range(6):
                o[:, 21 + a] = J0[:, a] * r0 + J1[:, a] * r1
            o[:, 27] = r0 * r0 + r1 * r1
            return o

        if npt:
            Px, Py, Pz = [((R[i, 0] * g.X[:, 0] + R[i, 1] * g.X[:, 1]) + R[i, 2] * g.X[:, 2]) + t[i] for i in range(3)]
            iz = 1.0 / Pz
            xn, yn = Px * iz, Py * iz
            r0, r1 = fx * xn - g.d[:, 0], fy * yn - g.d[:, 1]
            z = np.zeros(npt)
            J0 = jac(g.X, fx * iz, z, -((fx * xn) * iz))
            J1 = jac(g.X, z, fy * iz, -((fy * yn) * iz))
            out[:npt] = terms(J0, r0, J1, r1)
        if len(g.E):
            Js, rs = [], []
            for e in range(2):
                Xe = g.E[:, e]
                Qx, Qy, Qz = [((R[i, 0] * Xe[:, 0] + R[i, 1] * Xe[:, 1]) + R[i, 2] * Xe[:, 2]) + t[i] for i in range(3)]
                iz = 1.0 / Qz
                r = ((g.n[:, 0] * Qx + g.n[:, 1] * Qy) + g.n[:, 2] * Qz) * iz
                J = jac(Xe, g.n[:, 0] * iz, g.n[:, 1] * iz, -((r - g.n[:, 2]) * iz))
                Js.append(J)
                rs.append(r)
            out[npt:] = terms(Js[0], rs[0], Js[1], rs[1])
    out[~rows] = 0.0
    return out


def cayley(w):
    """The Cayley map ((1 - w.w) I + 2 [w]x + 2 w w^T) / (1 + w.w) of w [3], explicitly rounded: [3, 3]."""
    return np.array(_posed.cayley(np.asarray(w, dtype=np.float64)), dtype=np.float64)


def _lm_step(S, lam, R, t):
    """One damped Gauss-Newton step from the reduced terms S [28]: (A + lam diag A) x = -J^T r by Gaussian
    elimination with partial pivoting (first largest |pivot|), then R <- cay(w) R, t <- t + dt.  -> (R, t, ok)."""
    A = np.zeros((6, 7))
    for e, (a, b) in enumerate(_TRI):
        A[a, b] = A[b, a] = S[e]
    for a in range(6):
        A[a, a] = A[a, a] + lam * A[a, a]
        A[a, 6] = -S[21 + a]
    with np.errstate(all="ignore"):
        for c in range(6):
            piv, best = c, abs(A[c, c])
            for r in range(c + 1, 6):
                if abs(A[r, c]) > best:
                    best, piv = abs(A[r, c]), r
            if not best > 0:
                return R, t, False
            A[[c, piv]] = A[[piv, c]]
            for r in range(c + 1, 6):
                f = A[r, c] / A[c, c]
                for k in range(c + 1, 7):
                    A[r, k] = A[r, k] - f * A[c, k]
        x = np.zeros(6)
        for i in range(5, -1, -1):
            acc = A[i, 6]
            for k in range(i + 1, 6):
                acc = acc - A[i, k] * x[k]
            x[i] = acc / A[i, i]
        if not np.isfinite(x).all():
            return R, t, False
        C = cayley(x[:3])
        Rn = np.empty((3, 3))
        for i in range(3):
            for k in range(3):
                Rn[i, k] = (C[i, 0] * R[0, k] + C[i, 1] * R[1, k]) + C[i, 2] * R[2, k]
        tn = t + x[3:]
    return Rn, tn, bool(np.isfinite(Rn).all() and np.isfinite(tn).all())


def refine_pose_host(g: _Group, R, t, rows):
    """The refit (Levenberg-Marquardt over the rows `rows`, bool [np + nl]) from pose (R, t) in the group's shifted
    frame: AP_LM_ITERS steps with damping AP_LM_LAMBDA0, multiplied by AP_LM_ACCEPT after a step that lowers the cost
    and by AP_LM_REJECT otherwise.  -> (R, t, cost, number of accepted steps)."""
    R, t = np.array(R, dtype=np.float64), np.array(t, dtype=np.float64)
    S = block_sum(_row_terms(g, R, t, rows), AP_FIT_THREADS)
    lam, acc = AP_LM_LAMBDA0, 0
    for _ in range(AP_LM_ITERS):
        Rn, tn, ok = _lm_step(S, lam, R, t)
        cost = block_sum(_row_terms(g, Rn, tn, rows)[:, 27:], AP_FIT_THREADS)[0] if ok else np.nan
        if ok and cost < S[27]:
            R, t, lam, acc = Rn, tn, lam * AP_LM_ACCEPT, acc + 1
            S = block_sum(_row_terms(g, R, t, rows), AP_FIT_THREADS)
        else:
            lam = lam * AP_LM_REJECT
    return R, t, float(S[27]), acc


def _as_list(a, n):
    return list(a) if isinstance(a, (list, tuple)) else [a] * n if n else []


def stage_group(kpts0, matches_p, points3d1, K0, klines0=None, matches_l=None, lines3d1=None, use_lines=True):
    """The group's correspondences in the kernels' order and frame: -> (_Group, [per pair: matched point rows], [per
    pair: matched line rows]).  matches_* / *3d1 are lists with one entry per pair of the group (or one array for a
    single pair)."""
    single = not isinstance(matches_p, (list, tuple))
    mps = [matches_p] if single else list(matches_p)
    X1s = [points3d1] if single else list(points3d1)
    k0 = np.asarray(kpts0, dtype=np.float32).reshape(-1, 2).astype(np.float64)
    K = np.asarray(K0, dtype=np.float64).reshape(3, 3)
    rows_p, Xs, ds = [], [], []
    for mp, X1 in zip(mps, X1s):
        mp = np.asarray(mp, dtype=np.int64).reshape(-1)
        X1 = np.asarray(X1, dtype=np.float64).reshape(-1, 3)
        ok = (mp >= 0) & (mp < len(X1))
        ok[ok] = np.isfinite(X1[mp[ok]]).all(1)
        r = np.flatnonzero(ok)
        rows_p.append(r)
        Xs.append(X1[mp[r]])
        ds.append(k0[r])
    rows_l, Es, ss = [], [], []
    lines = use_lines and lines3d1 is not None and matches_l is not None
    if lines:
        mls = [matches_l] if single else list(matches_l)
        L1s = [lines3d1] if single else list(lines3d1)
        s0 = np.asarray(klines0, dtype=np.float32).reshape(-1, 2, 2)
        for ml, L1 in zip(mls, L1s):
            ml = np.asarray(ml, dtype=np.int64).reshape(-1)
            L1 = np.asarray(L1, dtype=np.float64).reshape(-1, 2, 3)
            ok = (ml >= 0) & (ml < len(L1))
            ok[ok] = np.isfinite(L1[ml[ok]]).all((1, 2))
            r = np.flatnonzero(ok)
            rows_l.append(r)
            Es.append(L1[ml[r]])
            ss.append(s0[r])
    else:
        rows_l = [np.zeros(0, np.int64) for _ in mps]
    X = np.concatenate(Xs) if Xs else np.zeros((0, 3))
    E = np.concatenate(Es) if Es else np.zeros((0, 2, 3))
    allw = np.concatenate([X, E.reshape(-1, 3)])
    c = (allw.min(0) + allw.max(0)) * 0.5 if len(allw) else np.zeros(3)
    d = (np.concatenate(ds) if ds else np.zeros((0, 2))) - np.array([K[0, 2], K[1, 2]])
    s0 = np.concatenate(ss) if ss else np.zeros((0, 2, 2), np.float32)
    g = _Group(K, d, X - c, line_normals(s0, K) if len(s0) else np.zeros((0, 3)), E - c, c)
    return g, rows_p, rows_l


def ransac_absolute_pose_host(kpts0, matches_p, points3d1, K0, klines0=None, matches_l=None, lines3d1=None, group=0,
                              thresh=8.0, n_hypotheses=1024, seed=0, use_lines=True, n_line_hypotheses=0) -> dict:
    """The absolute-pose estimator's model for one group in numpy (DESIGN.md "Absolute pose").  kpts0 [N0, 2] /
    klines0 [K0, 2, 2] are the query's (used as float32); matches_p / points3d1 (and matches_l / lines3d1) are one
    array per pair of the group in a list (or one array for a single pair): matches_p [N0] the local side-1 index or -1
    per query keypoint, points3d1 [n1, 3] fp64 (NaN rows: no 3D), lines3d1 [m1, 2, 3].  `group` seeds the samples.
    Returns R [3, 3], t [3] (X_cam = R X + t; NaN when invalid), valid, refit, inliers_p / inliers_l uint8 (the pairs'
    match rows concatenated), n_inliers_p, n_inliers_l, hypothesis (the winner's index: 4 k + j of P3P sample k and root
    j, 4 n_hypotheses + 8 (s n_line_hypotheses + k) + j of line solver s's sample k, or -1), hypothesis_inliers,
    R_hypothesis / t_hypothesis (the winner before the refit) and cost (the refit's final sum of squared residuals, NaN
    without a refit).  n_line_hypotheses samples of each line solver s (`line_pose_solutions`) join the P3P ones: the
    point rows drawn with seed + 2 s + 1, the line rows with seed + 2 s + 2, in groups with the rows the solver
    needs."""
    single = not isinstance(matches_p, (list, tuple))
    mps = [matches_p] if single else list(matches_p)
    mls = ([matches_l] if single else list(matches_l)) if matches_l is not None else [np.zeros(0)] * len(mps)
    n_rows_p = [len(np.ravel(m)) for m in mps]
    n_rows_l = [len(np.ravel(m)) for m in mls]
    g, rows_p, rows_l = stage_group(kpts0, matches_p, points3d1, K0, klines0, matches_l, lines3d1, use_lines)
    out = dict(R=np.full((3, 3), np.nan), t=np.full(3, np.nan), valid=False, refit=False,
               inliers_p=np.zeros(sum(n_rows_p), np.uint8), inliers_l=np.zeros(sum(n_rows_l), np.uint8),
               n_inliers_p=0, n_inliers_l=0, hypothesis=-1, hypothesis_inliers=0, R_hypothesis=np.full((3, 3), np.nan),
               t_hypothesis=np.full(3, np.nan), cost=np.nan)
    t2 = float(thresh) * float(thresh)
    fx, fy = g.K[0, 0], g.K[1, 1]
    q = np.stack([g.d[:, 0] / fx, g.d[:, 1] / fy], 1)
    cands = []   # (winner index, R, t, ok) per hypothesis kind
    if len(g.X) >= AP_SAMPLE and n_hypotheses > 0:
        idx, ok = draw_samples(seed, group, n_hypotheses, len(g.X), AP_SAMPLE)
        idx = np.maximum(idx, 0)
        R, t, oks = p3p_solutions(bearings(q[idx]), g.X[idx])
        cands.append((np.arange(AP_MAX_SOLUTIONS * n_hypotheses), R, t, oks & ok[:, None]))
    for s in range(3) if n_line_hypotheses > 0 else ():
        mp, ml = AP_LINE_NP[s], AP_LINE_NL[s]
        if len(g.X) < mp or len(g.E) < ml:
            continue
        il, ok = draw_samples(seed + 2 * s + 2, group, n_line_hypotheses, len(g.E), ml)
        ip = np.zeros((n_line_hypotheses, 0), np.int64)
        if mp:
            ip, okp = draw_samples(seed + 2 * s + 1, group, n_line_hypotheses, len(g.X), mp)
            ok &= okp
        ip, il = np.maximum(ip, 0), np.maximum(il, 0)
        R, t, oks = line_pose_solutions(s, bearings(q[ip]), g.X[ip], g.n[il], g.E[il])
        base = AP_MAX_SOLUTIONS * n_hypotheses + AP_LINE_MAX_SOLUTIONS * s * n_line_hypotheses
        cands.append((base + np.arange(AP_LINE_MAX_SOLUTIONS * n_line_hypotheses), R, t, oks & ok[:, None]))
    if not cands:
        return out
    okf = np.concatenate([c[3].reshape(-1) for c in cands])
    flat = np.concatenate([c[0] for c in cands])[okf]
    R = np.concatenate([c[1].reshape(-1, 3, 3) for c in cands])[okf]
    t = np.concatenate([c[2].reshape(-1, 3) for c in cands])[okf]
    if not len(flat):
        return out
    Rf, tf = R, t
    cnt = np.concatenate([_inliers(g, Rf[s:s + 256], tf[s:s + 256], t2).sum(1) for s in range(0, len(flat), 256)])
    order = np.lexsort((flat, -cnt))[0]
    w = int(flat[order])
    Rw, tw = Rf[order], tf[order]
    fl = _inliers(g, Rw, tw, t2)[0]
    out.update(hypothesis=w, hypothesis_inliers=int(fl.sum()), R_hypothesis=Rw.copy(), t_hypothesis=tw - Rw @ g.c)
    Rk, tk = Rw, tw
    if fl.sum() >= AP_MIN_REFIT:
        Rr, tr, cost, _ = refine_pose_host(g, Rw, tw, fl)
        flr = _inliers(g, Rr, tr, t2)[0]
        if flr.sum() >= fl.sum():
            Rk, tk, fl = Rr, tr, flr
            out.update(refit=True, cost=cost)
    npt = len(g.X)
    bp = np.concatenate([[0], np.cumsum(n_rows_p)])
    bl = np.concatenate([[0], np.cumsum(n_rows_l)])
    cp = np.concatenate([[0], np.cumsum([len(r) for r in rows_p])])
    cl = np.concatenate([[0], np.cumsum([len(r) for r in rows_l])])
    for i in range(len(mps)):
        out["inliers_p"][bp[i] + rows_p[i]] = fl[cp[i]:cp[i + 1]]
        out["inliers_l"][bl[i] + rows_l[i]] = fl[npt + cl[i]:npt + cl[i + 1]]
    c = g.c
    tc = np.array([tk[i] - ((Rk[i, 0] * c[0] + Rk[i, 1] * c[1]) + Rk[i, 2] * c[2]) for i in range(3)])
    out.update(R=Rk.copy(), t=tc, valid=True, n_inliers_p=int(fl[:npt].sum()), n_inliers_l=int(fl[npt:].sum()))
    return out


# ------------------------------------------------------------------ batched on the GPU
@dataclass
class AbsolutePoseResult:
    """Result of `estimate_absolute_poses` (device tensors; nothing has been waited for).

    R float64 [G, 3, 3] and t float64 [G, 3] with X_cam = R X_world + t (NaN where not valid), valid bool [G], refit
    bool [G] (the pose is the Levenberg-Marquardt refit), inliers_p / inliers_l uint8 aligned with the result's
    matches_p / matches_l (0 for unmatched rows, rows without 3D and invalid groups), n_inliers_p / n_inliers_l int32
    [G], hypothesis int32 [G] (the winner's index, -1 when not valid: 4 k + j of P3P sample k and root j, or
    4 n_hypotheses + 8 (s n_line_hypotheses + k) + j of sample k of line solver s = 0 P2P1L, 1 P1P2L, 2 P3L) and
    hypothesis_inliers int32 [G] (its inlier count, points and lines)."""
    R: torch.Tensor
    t: torch.Tensor
    valid: torch.Tensor
    refit: torch.Tensor
    inliers_p: torch.Tensor
    inliers_l: torch.Tensor
    n_inliers_p: torch.Tensor
    n_inliers_l: torch.Tensor
    hypothesis: torch.Tensor
    hypothesis_inliers: torch.Tensor


def _f64_rows(a, width):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else a
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(-1, width))


def estimate_absolute_poses(res, K0, points3d1, lines3d1=None, groups=None, thresh=8.0, n_hypotheses=1024, seed=0,
                            use_lines=True, n_line_hypotheses=0) -> AbsolutePoseResult:
    """Absolute pose of every query of an `ImagePairMatches` (`match_images`, `match_sets`) whose side 1 are database
    images with 3D: P3P RANSAC over the point matches, scored and refined with the line matches too, in one
    `ltr_absolute_pose_lines` call (two kernel launches, three with line hypotheses).  points3d1[p] fp64 [n1, 3] is aligned with res.keypoints1[p] and
    lines3d1[p] fp64 [m1, 2, 3] with res.klines1[p] (NaN rows: no 3D); both are pooled by identity, so a database
    image repeated by `match_sets` goes up once.  groups int [G + 1]: offsets over the pairs, group g is the query of
    pairs [groups[g], groups[g + 1]), which must share one side-0 image (None: one group per pair).  K0: the query
    intrinsics, [3, 3] or [G, 3, 3] (zero skew).  thresh in pixels (cv2.solvePnPRansac's default 8); use_lines=False
    scores points only.  n_line_hypotheses > 0 adds that many hypotheses of each line solver (P2P1L, P1P2L, P3L;
    DESIGN.md "Absolute pose") next to the n_hypotheses P3P ones, which may then be 0: queries with fewer than 3
    point matches, or few point inliers, are localized from their line matches too (one more kernel launch); it needs
    lines3d1 and use_lines.  Host arrays go up in one pinned copy; the call never waits for the device.  Raises LtrError
    for bad K0, misaligned 3D arrays, bad groups or groups that mix query images, and (LTR_E_UNSUPPORTED) when a group
    has more match rows than one CTA can stage (SMEM_PER_POINT_A / SMEM_PER_LINE_A bytes per row, SMEM_MAX in all)."""
    P = res.n_pairs
    dev = res.matches_p.device
    op, ol = np.asarray(res.offsets_p, dtype=np.int64), np.asarray(res.offsets_l, dtype=np.int64)
    n_line_hypotheses = int(n_line_hypotheses)
    if n_line_hypotheses < 0:
        raise N.LtrError("estimate_absolute_poses: n_line_hypotheses must be >= 0")
    if int(n_hypotheses) < (0 if n_line_hypotheses else 1):
        raise N.LtrError("estimate_absolute_poses: n_hypotheses must be >= 1 (>= 0 with line hypotheses)")
    if n_line_hypotheses and not (use_lines and lines3d1 is not None):
        raise N.LtrError("estimate_absolute_poses: line hypotheses need lines3d1 and use_lines")
    gr = np.arange(P + 1, dtype=np.int64) if groups is None else np.asarray(groups, dtype=np.int64).reshape(-1)
    if len(gr) < 1 or gr[0] != 0 or gr[-1] != P or (np.diff(gr) < 0).any():
        raise N.LtrError(f"estimate_absolute_poses: groups must be non-decreasing offsets from 0 to {P}")
    G_ = len(gr) - 1
    k0 = _intrinsics(K0, G_, "K0")
    if len(points3d1) != P or (lines3d1 is not None and len(lines3d1) != P):
        raise N.LtrError(f"estimate_absolute_poses: points3d1 / lines3d1 need one array per pair ({P})")
    lines = bool(use_lines) and lines3d1 is not None
    for g in range(G_):
        for p in range(gr[g] + 1, gr[g + 1]):
            if res.keypoints0[p] is not res.keypoints0[gr[g]] or (lines and res.klines0[p] is not res.klines0[gr[g]]):
                raise N.LtrError(f"estimate_absolute_poses: group {g} mixes query images (pair {p})")
    x_rows = lambda a: _f64_rows(a, 3)
    X1, xoff, xn = _pool(points3d1, P, x_rows)
    kn1 = np.array([len(k) for k in res.keypoints1], dtype=np.int32)
    if not np.array_equal(xn, kn1):
        bad = int(np.flatnonzero(xn != kn1)[0])
        raise N.LtrError(f"estimate_absolute_poses: points3d1[{bad}] has {xn[bad]} rows for {kn1[bad]} keypoints")
    pt_rows = lambda k: torch.as_tensor(k).to(device=dev, dtype=torch.float32).reshape(-1, 2)
    p0, poff0, pn0 = _pool(res.keypoints0, P, pt_rows)
    if not np.array_equal(pn0, np.diff(op)):
        raise N.LtrError("estimate_absolute_poses: side-0 keypoints and the match offsets disagree")
    arrays = {"X1": np.concatenate(X1) if X1 else np.zeros((0, 3)), "K0": k0, "x_off1": xoff, "n_x1": xn,
              "pts_off0": poff0, "cu_p": np.ascontiguousarray(op, dtype=np.int32),
              "cu_l": np.ascontiguousarray(ol, dtype=np.int32), "groups": np.ascontiguousarray(gr, dtype=np.int32)}
    rows_l = 0
    if lines:
        L1, loff, ln = _pool(lines3d1, P, lambda a: _f64_rows(a, 6))
        sn1 = np.array([len(np.asarray(k).reshape(-1, 4)) for k in res.klines1], dtype=np.int32)
        if not np.array_equal(ln, sn1):
            bad = int(np.flatnonzero(ln != sn1)[0])
            raise N.LtrError(f"estimate_absolute_poses: lines3d1[{bad}] has {ln[bad]} rows for {sn1[bad]} key lines")
        s0, soff0, sn0 = _pool(res.klines0, P, lambda k: np.asarray(k, dtype=np.float32).reshape(-1, 4))
        if not np.array_equal(sn0, np.diff(ol)):
            raise N.LtrError("estimate_absolute_poses: side-0 key lines and the match offsets disagree")
        arrays.update(L1=np.concatenate(L1) if L1 else np.zeros((0, 6)), l_off1=loff, n_l1=ln,
                      segs0=np.concatenate(s0) if s0 else np.zeros((0, 4), np.float32), seg_off0=soff0)
        rows_l = int((ol[gr[1:]] - ol[gr[:-1]]).max(initial=0))
    dv = _ops.stage(arrays, dev)
    u8, i32 = dict(dtype=torch.uint8, device=dev), dict(dtype=torch.int32, device=dev)
    # the entry takes a mask buffer even for a batch without point (or line) match rows, as line-only queries give
    n_mp, n_ml = res.matches_p.shape[0], res.matches_l.shape[0]
    masks = {"inliers_p": torch.empty(max(n_mp, 1), **u8), "inliers_l": torch.empty(max(n_ml, 1), **u8)}
    out = AbsolutePoseResult(torch.empty((G_, 3, 3), dtype=torch.float64, device=dev),
                             torch.empty((G_, 3), dtype=torch.float64, device=dev), torch.empty(G_, **u8),
                             torch.empty(G_, **u8), masks["inliers_p"][:n_mp], masks["inliers_l"][:n_ml],
                             torch.empty(G_, **i32), torch.empty(G_, **i32), torch.empty(G_, **i32),
                             torch.empty(G_, **i32))
    pts0 = torch.cat(p0) if p0 else torch.zeros((0, 2), dtype=torch.float32, device=dev)
    _ops.call_struct("ltr_absolute_pose_lines",
                     {**dv, "pts0": pts0.contiguous(), "matches_p": res.matches_p.contiguous(),
                      "matches_l": res.matches_l.contiguous(), "n_pairs": P, "n_groups": G_,
                      "max_rows_p": int((op[gr[1:]] - op[gr[:-1]]).max(initial=0)), "max_rows_l": rows_l,
                      "thresh": thresh, "n_hypotheses": n_hypotheses, "seed": seed, "use_lines": lines},
                     {**vars(out), **masks, "key": torch.empty(G_, dtype=torch.int64, device=dev)},
                     scalars=(n_line_hypotheses,))
    out.valid = out.valid.view(torch.bool)
    out.refit = out.refit.view(torch.bool)
    return out


# ------------------------------------------------------------------ metrics and 3D from depth
def _host64(a):
    return np.asarray(a.cpu() if isinstance(a, torch.Tensor) else a, dtype=np.float64)


def absolute_pose_errors(R, t, R_gt, t_gt):
    """Errors of G absolute poses (X_cam = R X + t) against the truth: -> (camera-centre distance [G] in world units,
    rotation angle of R_gt^T R [G] in degrees); inf in both where R or t is not finite."""
    R, t = _host64(R).reshape(-1, 3, 3), _host64(t).reshape(-1, 3)
    Rg = np.broadcast_to(_host64(R_gt).reshape(-1, 3, 3), R.shape)
    tg = np.broadcast_to(_host64(t_gt).reshape(-1, 3), t.shape)
    ok = np.isfinite(R).all((1, 2)) & np.isfinite(t).all(1)
    with np.errstate(all="ignore"):
        cos_r = ((Rg * R).sum((1, 2)) - 1.0) / 2.0
        err_R = np.degrees(np.arccos(np.clip(cos_r, -1.0, 1.0)))
        c, cg = -np.einsum("gji,gj->gi", R, t), -np.einsum("gji,gj->gi", Rg, tg)
        err_t = np.linalg.norm(c - cg, axis=1)
    return np.where(ok, err_t, np.inf), np.where(ok, err_R, np.inf)


def localization_recall(errors, thresholds=((0.25, 2), (0.5, 5), (5, 10))):
    """The fraction of queries localized within each (distance, degrees) bin, as InLoc / visuallocalization.net
    report it: errors = (centre distance [G], rotation degrees [G]) from `absolute_pose_errors`.  -> [len(thresholds)]."""
    et, eR = (np.asarray(e, dtype=np.float64).reshape(-1) for e in errors)
    return [float(np.mean((et <= d) & (eR <= a))) if len(et) else 0.0 for d, a in thresholds]


def lift_to_3d(xy, depth, K, cam_to_world):
    """World coordinates of database pixels xy [..., 2] from the image's depth map depth [H, W] (z along the optical
    axis), intrinsics K [3, 3] and pose cam_to_world [4, 4]: the depth of the nearest pixel (floor(x + 0.5), floor(y +
    0.5)), X_cam = depth K^-1 (x, y, 1), X = R X_cam + t.  NaN where that pixel is outside the map or its depth is not
    finite or not > 0.  Keypoints [n, 2] give points3d1 [n, 3]; segments [m, 2, 2] give lines3d1 [m, 2, 3]."""
    xy = _host64(xy)
    D = _host64(depth)
    K, T = _host64(K).reshape(3, 3), _host64(cam_to_world).reshape(4, 4)
    flat = xy.reshape(-1, 2)
    with np.errstate(all="ignore"):
        c, r = np.floor(flat[:, 0] + 0.5), np.floor(flat[:, 1] + 0.5)
        inside = (c >= 0) & (c < D.shape[1]) & (r >= 0) & (r < D.shape[0]) & np.isfinite(flat).all(1)
        ci, ri = np.where(inside, c, 0).astype(np.int64), np.where(inside, r, 0).astype(np.int64)
        z = np.where(inside, D[ri, ci], np.nan)
        ok = inside & np.isfinite(z) & (z > 0)
        ray = np.c_[flat, np.ones(len(flat))] @ np.linalg.inv(K).T
        Xc = ray * z[:, None]
        X = Xc @ T[:3, :3].T + T[:3, 3]
    X[~ok] = np.nan
    return X.reshape(xy.shape[:-1] + (3,))
