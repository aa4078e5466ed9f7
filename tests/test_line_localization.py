"""Line hypotheses in the absolute-pose RANSAC (`ltr_absolute_pose_lines`, `estimate_absolute_poses(...,
n_line_hypotheses)`): the P2P1L, P1P2L and P3L solvers of `localization.line_pose_solutions` on exact scenes, their
polynomial against 60 digits, their degenerate samples, what they add to localization on the host model, and the
kernels against that model bit for bit."""
import ctypes as C
import math

import mpmath
import numpy as np
import pytest
import torch

from linetr_b200 import _native as N, localization as L, synthetic as syn
from tests.test_estimator_edges import _Mag, _within
from tests.test_localization import FIELDS, _host_group, _matches

DEV = torch.device("cuda", 0)
K = syn.DEFAULT_K
LTR_E_INVALID = -1


# ------------------------------------------------------------------ exact samples
def _exact(seed, solver):
    """An exact fp64 sample of `solver` from a random pose: (j, X [2 - s, 3], n [s + 1, 3], E [s + 1, 2, 3], R, t).
    Bearings are the unit camera points; a line's normal is the cross product of its two camera end points."""
    rng = np.random.default_rng(seed)
    R = syn.random_rotation(rng)
    t = rng.normal(size=3) * 3
    P = np.c_[rng.uniform(-1, 1, (2, 2)), np.ones(2)] * rng.uniform(2, 8, (2, 1))
    Q = np.concatenate([rng.uniform(-1, 1, (3, 2, 2)), np.ones((3, 2, 1))], -1) * rng.uniform(2, 8, (3, 2, 1))
    npt, nl = L.AP_LINE_NP[solver], L.AP_LINE_NL[solver]
    j = P / np.linalg.norm(P, axis=1, keepdims=True)
    n = np.cross(Q[:, 0], Q[:, 1]) * rng.uniform(100, 1000)
    return j[:npt], ((P - t) @ R)[:npt], n[:nl], ((Q - t) @ R)[:nl], R, t


def _stack(samples):
    return [np.stack([s[i] for s in samples]) for i in range(6)]


def _residuals(R, t, j, X, n, E):
    """The six constraints of a pose, relative: each point's bearing against its camera point (the cross product's
    two largest components), each line end point's distance to its plane over its camera distance."""
    out = []
    for a, b in zip(j, X):
        P = R @ b + t
        out += sorted(np.abs(np.cross(a, P / np.linalg.norm(P))))[1:]
    for m, ab in zip(n, E):
        for e in ab:
            P = R @ e + t
            out.append(abs(m @ P) / (np.linalg.norm(m) * np.linalg.norm(P)))
    return np.array(out)


@pytest.mark.parametrize("solver", [0, 1, 2])
def test_solvers_recover_the_true_pose_and_satisfy_their_constraints(solver):
    """On exact samples from 200 random poses the true pose is among the solutions to 1e-9 in at least 90 % of cases,
    and every returned solution satisfies its six constraints to 1e-9 relative."""
    j, X, n, E, Rt, tt = _stack([_exact(s, solver) for s in range(200)])
    R, t, ok = L.line_pose_solutions(solver, j, X, n, E)
    errs, worst = [], 0.0
    for k in range(200):
        e = [max(np.abs(R[k, i] - Rt[k]).max(), np.abs(t[k, i] - tt[k]).max()) for i in np.flatnonzero(ok[k])]
        errs.append(min(e, default=np.inf))
        for i in np.flatnonzero(ok[k]):
            worst = max(worst, _residuals(R[k, i], t[k, i], j[k], X[k], n[k], E[k]).max())
            assert np.abs(R[k, i] @ R[k, i].T - np.eye(3)).max() < 1e-9
    errs = np.array(errs)
    print(f"solver {solver}: true pose within 1e-9 in {(errs < 1e-9).sum()} of 200 (median {np.median(errs):.1e}), "
          f"{ok.sum() / 200:.2f} solutions per sample, worst constraint residual {worst:.1e}")
    assert (errs < 1e-9).mean() >= 0.9
    assert worst < 1e-9
    # the public wrappers are the same solver
    R2, t2, ok2 = (lambda: L.p2p1l_solutions(j, X, n[:, 0], E[:, 0]), lambda: L.p1p2l_solutions(j[:, 0], X[:, 0], n, E),
                   lambda: L.p3l_solutions(n, E))[solver]()
    assert np.array_equal(ok2, ok) and np.array_equal(R2[ok], R[ok]) and np.array_equal(t2[ok], t[ok])


# ------------------------------------------------------------------ the polynomial against 60 digits
def _poly_mags(M1, M2):
    """trig_pair_poly's operations in its order with their running error bounds: p [9] as _Mag."""
    with mpmath.workdps(60):
        def quads(M):
            M = [_Mag.of(v) for v in M]
            return [[M[3 * r] + M[3 * r + 2], 2.0 * M[3 * r + 1], M[3 * r + 2] - M[3 * r]] for r in range(3)]

        def mul(a, b):
            out = []
            for k in range(len(a) + len(b) - 1):
                acc = _Mag(0)
                for i in range(len(a)):
                    if 0 <= k - i < len(b):
                        acc = acc + a[i] * b[k - i]
                out.append(acc)
            return out

        (A1, B1, C1), (A2, B2, C2) = quads(M1), quads(M2)
        sub = lambda u, v: [x - y for x, y in zip(u, v)]
        D, X, Y = sub(mul(A1, B2), mul(A2, B1)), sub(mul(B1, C2), mul(B2, C1)), sub(mul(A2, C1), mul(A1, C2))
        XX, YY, DD = mul(X, X), mul(Y, Y), mul(D, D)
        return [(XX[k] + YY[k]) - DD[k] for k in range(9)]


def _poly_mp(M1, M2):
    """X^2 + Y^2 - D^2 at 60 digits from the fp64 M_i, by exact polynomial arithmetic in tau."""
    with mpmath.workdps(60):
        def quads(M):
            M = [mpmath.mpf(float(v)) for v in M]
            return [[M[3 * r] + M[3 * r + 2], 2 * M[3 * r + 1], M[3 * r + 2] - M[3 * r]] for r in range(3)]

        def mul(a, b):
            out = [mpmath.mpf(0)] * (len(a) + len(b) - 1)
            for i, x in enumerate(a):
                for k, y in enumerate(b):
                    out[i + k] += x * y
            return out

        (A1, B1, C1), (A2, B2, C2) = quads(M1), quads(M2)
        sub = lambda u, v: [x - y for x, y in zip(u, v)]
        D, X, Y = sub(mul(A1, B2), mul(A2, B1)), sub(mul(B1, C2), mul(B2, C1)), sub(mul(A2, C1), mul(A1, C2))
        XX, YY, DD = mul(X, X), mul(Y, Y), mul(D, D)
        return [XX[k] + YY[k] - DD[k] for k in range(9)]


def _solver_Ms(n_random=40):
    """The M1, M2 each solver builds (the host's operations up to trig_pair_roots), on exact samples."""
    Ms = []
    orig = L.trig_pair_roots

    def grab(M1, M2):
        Ms.append((M1.copy(), M2.copy()))
        return orig(M1, M2)

    L.trig_pair_roots = grab
    try:
        for solver in range(3):
            j, X, n, E, _, _ = _stack([_exact(100 + s, solver) for s in range(n_random)])
            L.line_pose_solutions(solver, j, X, n, E)
    finally:
        L.trig_pair_roots = orig
    return np.concatenate([m[0] for m in Ms]), np.concatenate([m[1] for m in Ms])


def test_polynomial_within_the_running_error_bound_and_its_roots():
    M1, M2 = _solver_Ms()
    _, _, _, p = L.trig_pair_poly(M1, M2)
    cs, ok, _ = L.trig_pair_roots(M1, M2)
    worst = worst_root = 0.0
    for k in range(len(M1)):
        ref = _poly_mp(M1[k], M2[k])
        r = _within(p[k], ref, _poly_mags(M1[k], M2[k]))
        assert r <= 1.0, (k, r)
        worst = max(worst, r)
        # each host root is a root of the 60-digit polynomial: one Newton step from it moves it by < 1e-9 relative
        poly = np.zeros((1, 11))
        poly[0, :9] = p[k]
        roots, cnt = L.sturm_roots(poly)
        with mpmath.workdps(60):
            for tau in roots[0, :cnt[0]]:
                v = mpmath.polyval(ref[::-1], tau)
                dv = mpmath.polyval([i * c for i, c in enumerate(ref)][1:][::-1], tau)
                step = float(abs(v / dv)) if dv != 0 else math.inf
                worst_root = max(worst_root, step / max(1.0, abs(tau)))
    print(f"{len(M1)} polynomials: worst |p_host - p_60| / running bound {worst:.3f}; worst Newton step of a host root "
          f"{worst_root:.1e}")
    assert worst_root < 1e-9


# ------------------------------------------------------------------ degenerate samples
def _bisect(ok, lo=0.0, hi=1e-6):
    """The adjacent doubles lo < hi of the parameter where the rule ok() flips from rejecting to accepting."""
    assert not ok(lo) and ok(hi)
    while True:
        mid = (lo + hi) / 2
        if mid in (lo, hi):
            return lo, hi
        lo, hi = (lo, mid) if ok(mid) else (mid, hi)


def _unit(v):
    return v / np.linalg.norm(v)


def _rule_samples():
    """(name, solver, j, X, n, E, rule accepts) of each AP_*_EPS rule at its threshold and 1 ulp either side."""
    out = []
    # P2P1L: j2 moved off j1 by e
    j, X, n, E, _, _ = _exact(7, 0)
    v = _unit(np.cross(j[0], [0.3, -0.5, 0.8]))

    def p2(e):
        jj = j.copy()
        jj[1] = _unit(j[0] + e * v)
        return jj

    def ok0(e):
        c = L._cross(p2(e)[0], p2(e)[1])
        return math.sqrt(L._dot(c, c)) > L.AP_BEARING_EPS

    lo, hi = _bisect(ok0)
    for name, e in (("below", lo), ("at", hi), ("above", math.nextafter(hi, 1))):
        out.append((f"bearing_{name}", 0, p2(e), X, n, E, ok0(e)))
    out.append(("coincident_bearings", 0, p2(0.0), X, n, E, False))
    # P1P2L: the query point moved off query line 1 by e
    j, X, n, E, _, _ = _exact(8, 1)
    u = _unit(n[0])
    base = _unit(j[0] - (j[0] @ u) * u)

    def p1(e):
        return _unit(base + e * u)[None]

    def ok1(e):
        G = L._triad(L._unit(n[None, 0])[0])
        return abs(L._dot(G[0, 0], p1(e)[0])) > L.AP_POINT_LINE_EPS

    lo, hi = _bisect(ok1)
    for name, e in (("below", lo), ("at", hi), ("above", math.nextafter(hi, 1))):
        out.append((f"point_line_{name}", 1, p1(e), X, n, E, ok1(e)))
    out.append(("point_on_line_1", 1, p1(0.0), X, n, E, bool(ok1(0.0))))
    # P3L: n3 moved out of the plane of n1, n2 by e (the three query lines through one image point at e = 0)
    j, X, n, E, _, _ = _exact(9, 2)
    w = _unit(np.cross(n[0], n[1]))
    n3 = 0.4 * n[0] - 0.7 * n[1]

    def p3(e):
        nn = n.copy()
        nn[2] = n3 + e * np.linalg.norm(n3) * w
        return nn

    def ok2(e):
        nn = p3(e)
        det = L._dot(nn[0], L._cross(nn[1], nn[2]))
        m = [math.sqrt(L._dot(a, a)) for a in nn]
        return abs(det) > ((L.AP_CONCURRENT_EPS * m[0]) * m[1]) * m[2]

    lo, hi = _bisect(ok2)
    for name, e in (("below", lo), ("at", hi), ("above", math.nextafter(hi, 1))):
        out.append((f"concurrent_{name}", 2, j, X, p3(e), E, ok2(e)))
    out.append(("concurrent_lines", 2, j, X, p3(0.0), E, bool(ok2(0.0))))
    return out


def _structured():
    """(name, solver, j, X, n, E) of the structured samples: the rules' samples, parallel world lines (P3L), and a
    sample planted at b = pi for each solver."""
    out = [s[:6] for s in _rule_samples()]
    rng = np.random.default_rng(11)
    # three parallel world lines and their exact query lines
    R, t = syn.random_rotation(rng), rng.normal(size=3)
    d = _unit(rng.normal(size=3))
    A = rng.normal(size=(3, 3)) + (R.T @ ([0, 0, 6] - t))
    E = np.stack([A, A + d], 1)
    Pc = E @ R.T + t
    out.append(("parallel_world_lines", 2, np.zeros((0, 3)), np.zeros((0, 3)), np.cross(Pc[:, 0], Pc[:, 1]), E))
    for solver in range(3):
        out.append((f"planted_b_pi_{solver}",) + (solver,) + _planted_b_pi(solver, rng))
    return out


def _planted_b_pi(solver, rng):
    """An exact sample of `solver` whose true rotation has b = pi in R' = Rz(a) Rx(b) between its triads."""
    for _ in range(100):
        j, X, n, E, _, _ = _exact(int(rng.integers(1 << 30)), solver)
        # the triads depend on the sample only through its first line's normal and direction (P1P2L, P3L) or its
        # bearings and points (P2P1L); keep those, plant R, then rebuild the rest of the scene under it
        a = rng.uniform(-np.pi, np.pi)
        Rp = np.array([[np.cos(a), np.sin(a), 0], [np.sin(a), -np.cos(a), 0], [0, 0, -1.0]])   # Rz(a) Rx(pi)
        if solver == 0:
            H = L._triad(_unit(X[1] - X[0])[None])[0]
            g3 = _unit(np.cross(j[0], j[1]))
            G = np.stack([j[0], np.cross(g3, j[0]), g3])
            R = G.T @ Rp @ H
            # depths from R' e_x: s2 = L sin a / sigma, s1 = L (gamma sin a / sigma - cos a)
            Ln, ga, sg = np.linalg.norm(X[1] - X[0]), j[0] @ j[1], np.linalg.norm(np.cross(j[0], j[1]))
            s1, s2 = Ln * (ga * np.sin(a) / sg - np.cos(a)), Ln * np.sin(a) / sg
            if not (s1 > 0 and s2 > 0):
                continue
            t = s1 * j[0] - R @ X[0]
        else:
            G = L._triad(_unit(n[0])[None])[0][[1, 2, 0]]
            H = L._triad(_unit(E[0, 1] - E[0, 0])[None])[0]
            R = G.T @ Rp @ H
            P = rng.uniform(-1, 1, 3) + [0, 0, 5]
            P -= (P @ G[2]) * G[2]                    # a camera point on plane 1
            t = P - R @ E[0, 0]
            if solver == 1:
                Q = R @ X[0] + t
                if Q[2] <= 0:
                    continue
                j = (Q / np.linalg.norm(Q))[None]
        Pc = E @ R.T + t
        n = n.copy()
        n[1:] = np.cross(Pc[1:, 0], Pc[1:, 1])
        if solver == 0:
            n[0] = np.cross(Pc[0, 0], Pc[0, 1])
        Pp = X @ R.T + t
        if solver == 0 and (Pp[:, 2] <= 0).any():
            continue
        return j, X, n, E
    raise AssertionError("no planted sample")


def test_degenerate_samples_follow_their_rules_without_a_nan_pose():
    for name, solver, j, X, n, E, accepts in _rule_samples():
        R, t, ok = L.line_pose_solutions(solver, j[None], X[None], n[None], E[None])
        assert np.isfinite(R[ok]).all() and np.isfinite(t[ok]).all(), name
        if not accepts:
            assert not ok.any(), name
    names = {s[0]: s[-1] for s in _rule_samples()}
    for rule in ("bearing", "point_line", "concurrent"):
        assert not names[f"{rule}_below"] and names[f"{rule}_at"] and names[f"{rule}_above"], rule
    for name, solver, j, X, n, E in _structured():
        R, t, ok = L.line_pose_solutions(solver, j[None], X[None], n[None], E[None])
        assert np.isfinite(R[ok]).all() and np.isfinite(t[ok]).all(), name
        print(f"{name}: {int(ok.sum())} solutions")


# ------------------------------------------------------------------ capability on the host model
def _pose_err(R, t, d):
    et, eR = L.absolute_pose_errors(R, t, d["R"], d["t"])
    return float(eR[0])


@pytest.mark.parametrize("n_points", [0, 1, 2])
def test_queries_with_few_points_are_localized_from_lines(n_points):
    """Queries with 0, 1 or 2 point matches and 40 line matches (30 % line outliers, 1 px noise) are valid with 256
    line hypotheses, median rotation error below 0.5 degrees, and invalid without them."""
    errs = []
    for seed in range(8):
        d = syn.make_localization_correspondences(700 + seed, n_points, 40, noise_px=1.0, outlier_frac=0.0,
                                                  line_outlier_frac=0.3)
        args = (d["kpts0"], d["matches_p"], d["points3d1"], d["K"], d["klines0"], d["matches_l"], d["lines3d1"])
        h0 = L.ransac_absolute_pose_host(*args, n_hypotheses=64, group=seed)
        assert not h0["valid"]
        h = L.ransac_absolute_pose_host(*args, n_hypotheses=64, n_line_hypotheses=256, group=seed)
        assert h["valid"]
        errs.append(_pose_err(h["R"], h["t"], d))
    print(f"{n_points} points: rotation errors {np.round(errs, 3)}")
    assert np.median(errs) < 0.5


def test_line_hypotheses_raise_recall_with_few_point_inliers():
    """4 point inliers among 40 points and 40 line matches (30 % outliers): with 1024 P3P hypotheses alone a query is
    localized (rotation within 2 degrees) less often than with 256 line hypotheses per solver too, at the same seed."""
    ok_p = ok_l = 0
    n = 12
    for seed in range(n):
        d = syn.make_localization_correspondences(900 + seed, 80, 40, noise_px=1.0, outlier_frac=0.5,
                                                  line_outlier_frac=0.3)
        keep = np.flatnonzero(d["true_p"])[:4]
        out = np.flatnonzero(~d["true_p"])[:36]
        rows = np.concatenate([keep, out])
        args = (d["kpts0"][rows], np.arange(40, dtype=np.int32), d["points3d1"][rows], d["K"],
                d["klines0"], d["matches_l"], d["lines3d1"])
        hp = L.ransac_absolute_pose_host(*args, n_hypotheses=1024, group=seed)
        hl = L.ransac_absolute_pose_host(*args, n_hypotheses=1024, n_line_hypotheses=256, group=seed)
        ok_p += hp["valid"] and _pose_err(hp["R"], hp["t"], d) < 2.0
        ok_l += hl["valid"] and _pose_err(hl["R"], hl["t"], d) < 2.0
    print(f"recall: P3P alone {ok_p}/{n}, with line hypotheses {ok_l}/{n}")
    assert ok_l > ok_p


# ------------------------------------------------------------------ argument errors (no launch)
def _structs(**kw):
    i, o = N.LtrAbsPoseInput(), N.LtrAbsPoseOutput()
    i.thresh, i.n_hypotheses, i.use_lines, i.n_groups = 8.0, 16, 1, 1
    for k, v in kw.items():
        setattr(i, k, v)
    return i, o


def test_absolute_pose_lines_refuses_bad_arguments():
    lib = N.load()
    call = lambda i, o, m: lib.ltr_absolute_pose_lines(C.byref(i), C.byref(o), m, 0, None)
    assert lib.ltr_absolute_pose_lines(None, None, 4, 0, None) == LTR_E_INVALID
    for kw, m, msg in ((dict(), -1, b"n_line_hypotheses"), (dict(), (1 << 21) + 1, b"n_line_hypotheses"),
                       (dict(use_lines=0), 4, b"use_lines"), (dict(n_hypotheses=0), 0, b"n_hypotheses"),
                       (dict(n_hypotheses=-1), 4, b"n_hypotheses"), (dict(thresh=0.0), 4, b"thresh"),
                       (dict(n_groups=-1), 4, b"negative"), (dict(), 4, b"null output"),
                       (dict(max_rows_l=4), 4, b"null output")):
        i, o = _structs(**kw)
        assert call(i, o, m) == LTR_E_INVALID, (kw, m)
        assert msg in lib.ltr_last_error(), (kw, m, lib.ltr_last_error())
    assert lib.ltr_last_error().startswith(b"ltr_absolute_pose_lines")
    i, o = _structs(n_groups=0, n_hypotheses=0)
    assert call(i, o, 4) == 0                     # nothing to do, nothing launched
    for s, cnt in ((3, 1), (-1, 1), (0, -1)):
        assert lib.ltr_debug_line_pose(s, None, None, None, None, cnt, None, None, None, None, 0, None) == LTR_E_INVALID


# ------------------------------------------------------------------ GPU
def _bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).view(np.int64)


def _debug_line_pose(solver, j, X, n, E):
    cnt = len(n)
    t_ = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(DEV)
    jd, Xd, nd, Ed = t_(j), t_(X), t_(n), t_(E)
    R = torch.empty((cnt, 8, 9), dtype=torch.float64, device=DEV)
    t = torch.empty((cnt, 8, 3), dtype=torch.float64, device=DEV)
    jr = torch.empty((cnt, 8), dtype=torch.int32, device=DEV)
    ns = torch.empty(cnt, dtype=torch.int32, device=DEV)
    with torch.cuda.device(DEV):
        rc = N.load().ltr_debug_line_pose(solver, jd.data_ptr() or None, Xd.data_ptr() or None, nd.data_ptr(),
                                          Ed.data_ptr(), cnt, R.data_ptr(), t.data_ptr(), jr.data_ptr(), ns.data_ptr(),
                                          0, None)
    N.check(rc, "ltr_debug_line_pose")
    return R.cpu().numpy(), t.cpu().numpy(), jr.cpu().numpy(), ns.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("solver", [0, 1, 2])
def test_debug_line_pose_bit_for_bit(solver):
    """`ltr_debug_line_pose` against `line_pose_solutions`, every output bit: exact samples, random inconsistent ones
    and the structured set."""
    rng = np.random.default_rng(20 + solver)
    items = [_exact(300 + s, solver)[:4] for s in range(300)]
    npt, nl = L.AP_LINE_NP[solver], L.AP_LINE_NL[solver]
    for _ in range(300):
        jr_ = rng.normal(size=(npt, 3)) + [0, 0, 2]
        items.append((jr_ / np.linalg.norm(jr_, axis=1, keepdims=True), rng.normal(size=(npt, 3)) * 3,
                      rng.normal(size=(nl, 3)) * 500, rng.normal(size=(nl, 2, 3)) * 3))
    items += [s[2:6] for s in _structured() if s[1] == solver]
    j, X, n, E = (np.stack([it[i] for it in items]) for i in range(4))
    R, t, ok = L.line_pose_solutions(solver, j, X, n, E)
    gR, gt, gjr, gns = _debug_line_pose(solver, j, X, n, E)
    for k in range(len(items)):
        idx = np.flatnonzero(ok[k])
        assert gns[k] == len(idx), k
        assert np.array_equal(gjr[k, :len(idx)], idx) and (gjr[k, len(idx):] == -1).all(), k
        assert np.array_equal(_bits(gR[k, :len(idx)]), _bits(R[k, idx].reshape(-1, 9))), k
        assert np.array_equal(_bits(gt[k, :len(idx)]), _bits(t[k, idx])), k
        assert np.isnan(gR[k, len(idx):]).all()
    print(f"solver {solver}: {len(items)} samples, {int(gns.sum())} solutions, every bit equal")


def _ragged(n_groups, seed):
    """Ragged groups of 1 to 4 pairs: groups with 0, 1, 2 and many point rows, 0 to 40 line rows, some all outliers."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n_groups):
        kind = i % 8
        cases = []
        for j in range(int(rng.integers(1, 5))):
            n = (0, 1, 2)[kind] if kind < 3 else int(rng.integers(0, 120))
            m = int(rng.integers(0, 3)) if kind == 3 else int(rng.integers(0, 40))
            cases.append(syn.make_localization_correspondences(8000 + 10 * i + j, n if j == 0 or kind >= 3 else 0, m,
                                                               noise_px=float(rng.uniform(0.1, 1.0)),
                                                               outlier_frac=1.0 if kind == 4 else
                                                               float(rng.uniform(0.1, 0.9))))
        out.append(cases)
    return out


def _compare(res, X1, L1, groups, Ks, out, **kw):
    got = {f: getattr(out, f).cpu().numpy() for f in FIELDS}
    n_valid = n_line = 0
    for g in range(len(groups) - 1):
        h = _host_group(res, X1, L1, groups, Ks, g, **kw)
        assert bool(got["valid"][g]) == h["valid"], g
        assert got["hypothesis"][g] == h["hypothesis"] and got["hypothesis_inliers"][g] == h["hypothesis_inliers"], g
        a, b = res.offsets_p[groups[g]], res.offsets_p[groups[g + 1]]
        c, e = res.offsets_l[groups[g]], res.offsets_l[groups[g + 1]]
        assert np.array_equal(got["inliers_p"][a:b], h["inliers_p"]) and np.array_equal(got["inliers_l"][c:e],
                                                                                         h["inliers_l"]), g
        assert got["n_inliers_p"][g] == h["n_inliers_p"] and got["n_inliers_l"][g] == h["n_inliers_l"], g
        if not h["valid"]:
            assert np.isnan(got["R"][g]).all() and np.isnan(got["t"][g]).all()
            continue
        n_valid += 1
        n_line += h["hypothesis"] >= 4 * kw["n_hypotheses"]
        assert bool(got["refit"][g]) == h["refit"], g
        for f in ("R", "t"):
            assert np.array_equal(_bits(got[f][g]), _bits(h[f])), (g, f)
    return n_valid, n_line


@pytest.mark.gpu
def test_kernels_match_host_model_with_line_hypotheses():
    """About 200 ragged groups, every output bit against `ransac_absolute_pose_host`."""
    res, X1, L1, groups, Ks = _matches(_ragged(200, 0))
    kw = dict(n_hypotheses=128, n_line_hypotheses=129, seed=3)
    out = L.estimate_absolute_poses(res, Ks, X1, L1, groups=groups, **kw)
    n_valid, n_line = _compare(res, X1, L1, groups, Ks, out, **kw)
    print(f"{len(groups) - 1} groups, {n_valid} valid, {n_line} won by a line hypothesis")
    assert n_line > 0 and n_valid > n_line


@pytest.mark.gpu
@pytest.mark.parametrize("n_hyp", [0, 1, 1024])
@pytest.mark.parametrize("n_line", [1, 127, 128, 129, 1024])
def test_hypothesis_counts_around_the_cta(n_hyp, n_line):
    res, X1, L1, groups, Ks = _matches(_ragged(16, 100 + n_line + n_hyp))
    kw = dict(n_hypotheses=n_hyp, n_line_hypotheses=n_line, seed=n_line)
    out = L.estimate_absolute_poses(res, Ks, X1, L1, groups=groups, **kw)
    _compare(res, X1, L1, groups, Ks, out, **kw)


@pytest.mark.gpu
def test_batch_without_point_matches():
    """A batch whose queries have line matches only is localized from them alone, as the host model does."""
    cases = [[syn.make_localization_correspondences(40 + i, 0, 40, noise_px=0.5, line_outlier_frac=0.3)]
             for i in range(6)]
    res, X1, L1, groups, Ks = _matches(cases, shuffle_rows=False)
    assert res.matches_p.shape[0] == 0
    kw = dict(n_hypotheses=0, n_line_hypotheses=128, seed=1)
    out = L.estimate_absolute_poses(res, Ks, X1, L1, groups=groups, **kw)
    n_valid, n_line = _compare(res, X1, L1, groups, Ks, out, **kw)
    assert n_valid == n_line == 6
    with pytest.raises(N.LtrError, match="n_hypotheses"):
        L.estimate_absolute_poses(res, Ks, X1, L1, groups=groups, n_hypotheses=0)
    with pytest.raises(N.LtrError, match="use_lines"):
        L.estimate_absolute_poses(res, Ks, X1, L1, groups=groups, n_line_hypotheses=8, use_lines=False)


def _call_raw(entry, res, X1, L1, groups, Ks, n_line):
    """estimate_absolute_poses' call through `entry` (ltr_absolute_pose, or ltr_absolute_pose_lines with n_line)."""
    from linetr_b200 import _ops
    captured = {}
    orig = _ops.call_struct

    def capture(e, inputs, outputs, *a, **k):
        captured.update(inputs=inputs, outputs=outputs)
        return orig(e, inputs, outputs, *a, **k)

    _ops.call_struct = capture
    try:
        L.estimate_absolute_poses(res, Ks, X1, L1, groups=groups, n_hypotheses=256, seed=9)
    finally:
        _ops.call_struct = orig
    outs = {k: torch.full_like(v, 0x5A) if v.dtype != torch.float64 else torch.full_like(v, 1.5)
            for k, v in captured["outputs"].items()}
    orig(entry, captured["inputs"], outs, scalars=(n_line,) if entry.endswith("lines") else ())
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in outs.items() if k != "key"}


@pytest.mark.gpu
def test_absolute_pose_and_lines_entry_with_zero_give_the_same_bits():
    res, X1, L1, groups, Ks = _matches(_ragged(60, 7))
    a = _call_raw("ltr_absolute_pose", res, X1, L1, groups, Ks, 0)
    b = _call_raw("ltr_absolute_pose_lines", res, X1, L1, groups, Ks, 0)
    for k in a:
        assert np.array_equal(np.ascontiguousarray(a[k]).view(np.uint8), np.ascontiguousarray(b[k]).view(np.uint8)), k


@pytest.mark.gpu
@pytest.mark.parametrize("n_hyp,launches", [(64, 3), (0, 2)])
def test_launch_accounting(n_hyp, launches):
    from tests.test_launch_accounting import _accounted, _counts
    res, X1, L1, groups, Ks = _matches(_ragged(8, 3))
    calls, classes = _accounted(lambda: L.estimate_absolute_poses(res, Ks, X1, L1, groups=groups, n_hypotheses=n_hyp,
                                                                  n_line_hypotheses=32))
    assert _counts(calls, "ltr_absolute_pose_lines") == [launches]
    assert classes == {"absolute_pose": launches}
