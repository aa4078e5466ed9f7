"""The fundamental-matrix (`ltr_fundamental`) and absolute-pose (`ltr_absolute_pose`) estimators at their edges.

- 60-digit references (mpmath) of the seven-point cubic and Grunert's quartic on the same fp64 inputs, bounding the
  host models' coefficients by a running-error bound, and their roots against the exact rational Sturm reference of
  test_ransac_edges.  The comparators are shown to catch a 1-ulp coefficient change and a wrong sign.
- The epipolar line check on exact hand-built cases, its NaN-cannot-reject rule included.
- On the GPU: the two minimal solvers (`fm_solve`, `ap_p3p`) and the line check through their debug hooks against
  `geometry.fundamental_solutions`, `localization.p3p_solutions` and `geometry.line_overlap_ratios` bit for bit; every
  hypothesis end to end (P copies of one set with n_hypotheses=1 evaluate P hypotheses, the sample hash mixes in the
  pair / group index), with lines planted 5e-10 px either side of the threshold of each hypothesis' pose; the depth
  rule on an exact scene; and degenerate, minimal, capacity, scale and intrinsics edges through the public API, each
  compared with the host model.

Not covered here: a 60-digit reference of the solutions themselves (P3P's back-substitution and triads, F from the
roots; their accuracy is checked against exact scenes in test_fundamental / test_localization), seven-point samples
with a root near ESS_ROOT_BOUND (the parametrisation comes from the QR basis of the sample, so a root cannot be placed),
and a pose winner with 2 inliers (P3P reprojects its own three sample points, so a winner has at least 3)."""
import ctypes as C
import math
from fractions import Fraction

import mpmath
import numpy as np
import pytest
import torch

from linetr_b200 import _native as N, geometry as G, localization as L, synthetic as syn
from tests.test_fundamental import FIELDS as FM_FIELDS, _matches as _fm_matches, _ragged_cases as _fm_ragged, check_pair
from tests.test_localization import FIELDS as AP_FIELDS, _host_group, _matches as _ap_matches, _ragged_groups
from tests.test_ransac_edges import SEPARATION, U, _band, _bits, _cauchy, exact_roots

DEV = torch.device("cuda", 0)
E22 = np.zeros((0, 2, 2), np.float32)
LTR_E_INVALID = -1


def _gamma(n):
    return n * U / (1 - n * U)


# ------------------------------------------------------------------ running-error magnitudes
class _Mag:
    """A value computed in fp64 with its first-order running error bound (Wilkinson; Higham, Accuracy and Stability,
    sec. 3.3): v is the exact value of the expression on the fp64 inputs (60 digits) and e bounds |fl(x) - x|.  Each
    operation adds the propagated errors of its operands and one rounding of its result:
        a +- b: e_a + e_b + u |a +- b|,    a b: |b| e_a + |a| e_b + u |a b|,    a / b: (e_a + |a / b| e_b) / |b| + u |a / b|
    (a product by a power of two and a negation are exact).  The bound is first order in u: terms of order u^2 are
    dropped, which `_within` covers with a factor 1.01."""

    def __init__(self, v, e=0):
        self.v, self.e = mpmath.mpf(v), mpmath.mpf(e)

    @staticmethod
    def of(x):
        return x if isinstance(x, _Mag) else _Mag(mpmath.mpf(float(x)), 0)

    @staticmethod
    def _pow2(x):
        return not isinstance(x, _Mag) and float(x) != 0 and math.frexp(abs(float(x)))[0] == 0.5

    def __add__(self, o):
        o = _Mag.of(o)
        v = self.v + o.v
        return _Mag(v, self.e + o.e + U * abs(v))

    __radd__ = __add__

    def __sub__(self, o):
        o = _Mag.of(o)
        v = self.v - o.v
        return _Mag(v, self.e + o.e + U * abs(v))

    def __rsub__(self, o):
        return _Mag.of(o) - self

    def __mul__(self, o):
        if _Mag._pow2(o):
            return _Mag(self.v * float(o), self.e * abs(float(o)))
        o = _Mag.of(o)
        v = self.v * o.v
        return _Mag(v, abs(o.v) * self.e + abs(self.v) * o.e + U * abs(v))

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = _Mag.of(o)
        v = self.v / o.v
        return _Mag(v, (self.e + abs(v) * o.e) / abs(o.v) + U * abs(v))

    def __neg__(self):
        return _Mag(-self.v, self.e)


def _dot3(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def _grunert_mags(j, X):
    """localization.grunert_quartic's operations, in its order, with their running error bounds: [A0 .. A4]."""
    with mpmath.workdps(60):
        j = [[_Mag.of(v) for v in r] for r in j]
        X = [[_Mag.of(v) for v in r] for r in X]
        d1 = [X[1][e] - X[0][e] for e in range(3)]
        d2 = [X[2][e] - X[0][e] for e in range(3)]
        d3 = [X[2][e] - X[1][e] for e in range(3)]
        c2, b2, a2 = _dot3(d1, d1), _dot3(d2, d2), _dot3(d3, d3)
        ca, cb, cg = _dot3(j[1], j[2]), _dot3(j[0], j[2]), _dot3(j[0], j[1])
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
        return [A0, A1, A2, A3, A4]


def _grunert_mp(j, X):
    """Grunert's quartic in v = s3 / s1 (Haralick et al. 1994, section 2.1) at 60 digits from the fp64 inputs, written
    from the paper rather than from the model: [A0 .. A4] as mpf."""
    with mpmath.workdps(60):
        j = [[mpmath.mpf(float(v)) for v in r] for r in j]
        X = [[mpmath.mpf(float(v)) for v in r] for r in X]
        sq = lambda a, b: sum((a[e] - b[e]) ** 2 for e in range(3))
        a2, b2, c2 = sq(X[2], X[1]), sq(X[2], X[0]), sq(X[1], X[0])
        dot = lambda a, b: sum(a[e] * b[e] for e in range(3))
        ca, cb, cg = dot(j[1], j[2]), dot(j[0], j[2]), dot(j[0], j[1])
        s, t = (a2 - c2) / b2, (a2 + c2) / b2
        A4 = (s - 1) ** 2 - 4 * c2 / b2 * ca ** 2
        A3 = 4 * (s * (1 - s) * cb - (1 - t) * ca * cg + 2 * c2 / b2 * ca ** 2 * cb)
        A2 = 2 * (s ** 2 - 1 + 2 * s ** 2 * cb ** 2 + 2 * (b2 - c2) / b2 * ca ** 2 - 4 * t * ca * cb * cg
                  + 2 * (b2 - a2) / b2 * cg ** 2)
        A1 = 4 * (-s * (1 + s) * cb + 2 * a2 / b2 * cg ** 2 * cb - (1 - t) * ca * cg)
        A0 = (1 + s) ** 2 - 4 * a2 / b2 * cg ** 2
        return [A0, A1, A2, A3, A4]


def _cubic_mp(basis):
    """det(F2 + a (F1 - F2)) at 60 digits from the fp64 null basis [2, 9], by the Leibniz formula over the six
    permutations (not the model's first-row expansion): ascending [c0 .. c3] as mpf."""
    with mpmath.workdps(60):
        F1 = [mpmath.mpf(float(v)) for v in basis[0]]
        F2 = [mpmath.mpf(float(v)) for v in basis[1]]
        ent = [(F2[i], F1[i] - F2[i]) for i in range(9)]
        out = [mpmath.mpf(0)] * 4
        for perm, sgn in (((0, 1, 2), 1), ((1, 2, 0), 1), ((2, 0, 1), 1), ((0, 2, 1), -1), ((2, 1, 0), -1),
                          ((1, 0, 2), -1)):
            poly = [mpmath.mpf(sgn)]
            for r in range(3):
                e = ent[3 * r + perm[r]]
                poly = [(poly[k] if k < len(poly) else 0) * e[0] + (poly[k - 1] * e[1] if k >= 1 else 0)
                        for k in range(len(poly) + 1)]
            out = [out[k] + poly[k] for k in range(4)]
        return out


def _cubic_mags(basis):
    """geometry.fundamental_cubic's operations on magnitudes: D = F1 - F2 (1 rounding); each 2 x 2 minor's coefficients
    are a product-sum (2) of entries carrying up to 1, then one subtraction (depth 4); times an entry (1 + 4 + 1) and a
    product-sum's add (7); then (t0 - t1) + t2 (9).  So every coefficient's error is below gamma_9 times its magnitude
    expansion, which is the Leibniz sum of |F2|, |D| products."""
    F1, F2 = np.abs(basis[0]).astype(object), np.abs(basis[1]).astype(object)
    D = [abs(mpmath.mpf(float(basis[0][i])) - mpmath.mpf(float(basis[1][i]))) for i in range(9)]
    ent = [(mpmath.mpf(float(F2[i])), D[i]) for i in range(9)]
    out = [mpmath.mpf(0)] * 4
    for perm in ((0, 1, 2), (1, 2, 0), (2, 0, 1), (0, 2, 1), (2, 1, 0), (1, 0, 2)):
        poly = [mpmath.mpf(1)]
        for r in range(3):
            e = ent[3 * r + perm[r]]
            poly = [(poly[k] if k < len(poly) else 0) * e[0] + (poly[k - 1] * e[1] if k >= 1 else 0)
                    for k in range(len(poly) + 1)]
        out = [out[k] + poly[k] for k in range(4)]
    return [(m, 9) for m in out]


def _within(host, ref, bounds):
    """|host_k - ref_k| <= bound_k for every coefficient k, the bound a _Mag's running error (times 1.01 for the
    dropped second-order terms) or (m, d) for gamma_d m; -> the worst ratio."""
    worst = 0.0
    for h, r, g in zip(host, ref, bounds):
        b = g.e * 1.01 if isinstance(g, _Mag) else _gamma(g[1]) * g[0]
        e = abs(mpmath.mpf(float(h)) - r)
        worst = max(worst, float(e / b) if b > 0 else (0.0 if e == 0 else math.inf))
    return worst


# ------------------------------------------------------------------ samples
def _fm_exact_sample(s):
    from tests.test_fundamental import _exact_sample
    return _exact_sample(s)[0]


def _ap_exact_sample(s):
    from tests.test_localization import _exact_sample
    j, X, _, _ = _exact_sample(s)
    return j, X


def _unit(v):
    v = np.asarray(v, dtype=np.float64)
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def _ap_structured():
    """Structured P3P samples (name, j [3, 3], X [3, 3])."""
    rng = np.random.default_rng(41)
    out = []
    # isosceles right triangle: p = (a2 - c2) / b2 = 1 exactly and cos alpha = 0 exactly, so A4 == 0 (a degree drop)
    out.append(("isosceles_A4_0", np.array([[0.1, 0.2, 0.97], [0.6, 0.0, 0.8], [-0.8, 0.0, 0.6]]),
                np.array([[0.0, 0.0, 5.0], [3.0, 0.0, 5.0], [0.0, 3.0, 5.0]])))
    # j2 orthogonal to j1 and j3: cos gamma = cos alpha = 0, so den = 2 (cos gamma - v cos alpha) == 0 at every root
    out.append(("den_0", np.array([[0.6, 0.0, 0.8], [0.0, 1.0, 0.0], [-0.8, 0.0, 0.6]]),
                np.array([[1.0, 0.5, 4.0], [-1.0, 2.0, 6.0], [0.5, -1.0, 5.0]])))
    for s in range(4):
        R = syn.random_rotation(rng)
        # the danger cylinder: the camera centre on the cylinder through the triangle's circumcircle, perpendicular to
        # its plane (a double root of the quartic)
        ang = rng.uniform(0, 2 * np.pi, 3)
        Xw = np.c_[np.cos(ang), np.sin(ang), np.zeros(3)] * 2.0
        phi = rng.uniform(0, 2 * np.pi)
        Cc = np.array([2 * np.cos(phi), 2 * np.sin(phi), rng.uniform(3, 6)])
        out.append(("danger_cylinder", _unit((Xw - Cc) @ R.T), Xw))
        # identical bearings of two points
        j, X = _ap_exact_sample(1000 + s)
        j2 = j.copy()
        j2[1] = j2[0]
        out.append(("identical_bearings", j2, X))
        # bearings at 60 degrees off the axis (a 120-degree field of view)
        a = rng.uniform(0, 2 * np.pi, 3)
        jb = np.c_[np.sin(np.pi / 3) * np.cos(a), np.sin(np.pi / 3) * np.sin(a), np.full(3, np.cos(np.pi / 3))]
        Rw = syn.random_rotation(rng)
        Xc = jb * rng.uniform(3, 8, (3, 1))
        out.append(("fov_120", jb, (Xc - 1.0) @ Rw))
        # a triangle of millimetres 100 m away
        Xc = np.array([0.0, 0.0, 100.0]) + rng.uniform(-1e-3, 1e-3, (3, 3))
        Rw = syn.random_rotation(rng)
        out.append(("mm_at_100m", _unit(Xc), (Xc - [0.3, -0.2, 1.0]) @ Rw))
        # inconsistent bearings and points: roots with v <= 0 and u <= 0 are common
        out.append(("random", _unit(rng.normal(size=(3, 3)) + [0, 0, 2]), rng.normal(size=(3, 3)) * 3))
    # world points at AP_COLLINEAR_EPS: X3 moved off the line X1 X2 by e, e bisected to where the rule flips
    j, X = _ap_exact_sample(77)
    n = _unit(np.cross(X[1] - X[0], rng.normal(size=3)))

    def sample(e):
        Xe = X.copy()
        Xe[2] = X[0] + 0.7 * (X[1] - X[0]) + e * n
        return Xe

    lo, hi = 0.0, 1e-6
    assert not _collinear_ok(sample(lo)) and _collinear_ok(sample(hi))
    for _ in range(300):
        mid = (lo + hi) / 2
        if mid in (lo, hi):
            break
        lo, hi = (lo, mid) if _collinear_ok(sample(mid)) else (mid, hi)
    # then the component of X3 along which n is largest, stepped by single ulps of that world coordinate from the
    # last sample the rule rejects (k = 0): k < 0 moves it towards the line, k > 0 away from it
    ax = int(np.argmax(np.abs(n)))
    up = math.inf if n[ax] > 0 else -math.inf
    for k in range(-3, 4):
        Xk = sample(lo)
        for _ in range(abs(k)):
            Xk[2, ax] = math.nextafter(Xk[2, ax], up if k > 0 else -up)
        out.append((f"collinear_ulp{k:+d}", j, Xk))
    return out


def _collinear_ok(X):
    """The P3P's collinearity rule on world points X [3, 3]: ncr > (AP_COLLINEAR_EPS n1) n2."""
    d1, d2 = X[1] - X[0], X[2] - X[0]
    cr = L._cross(d1[None], d2[None])[0]
    n1, n2, ncr = math.sqrt(L._dot(d1, d1)), math.sqrt(L._dot(d2, d2)), math.sqrt(L._dot(cr, cr))
    return ncr > (L.AP_COLLINEAR_EPS * n1) * n2


def _fm_scene(rng, n=7, plane=None, t=None, K0=None, K1=None):
    """n normalised-looking correspondences of a random two-view scene (points optionally on a plane n . X = 1; t = 0
    for a pure rotation), scaled to about [-1, 1]."""
    K0 = syn.DEFAULT_K if K0 is None else K0
    K1 = syn.DEFAULT_K if K1 is None else K1
    R, tt = syn.random_pose(rng)
    tt = tt if t is None else np.asarray(t, dtype=np.float64)
    ray = np.c_[rng.uniform(-0.5, 0.5, (n, 2)), np.ones(n)]
    X = ray * rng.uniform(2, 8, (n, 1)) if plane is None else ray / (ray @ plane)[:, None]
    x0, x1 = syn._project(K0, X), syn._project(K1, X @ R.T + tt)
    return np.concatenate([(x0 - 320) / 320, (x1 - 320) / 320], 1)


def _fm_structured():
    """Structured seven-point samples (name, q [7, 4])."""
    rng = np.random.default_rng(43)
    out = []
    for s in range(4):
        q = _fm_scene(rng)
        q[4] = q[2]
        out.append(("duplicated_rows", q))
        out.append(("coplanar7", _fm_scene(rng, plane=np.array([0.05, -0.1, 0.25]))))
        q = _fm_scene(rng, plane=np.array([0.02, 0.1, 0.2]))
        q[6] = _fm_scene(rng)[6]
        out.append(("coplanar6", q))
        out.append(("rotation", _fm_scene(rng, t=np.zeros(3))))
        # a repeated root: the pencil F2 + a D with D = diag(-1, -1, 0.5) has det(I + a D) = (1 - a)^2 (1 + a / 2);
        # seven x0 and their x1 on both epipolar lines of F1 = I + D and F2 = I, mixed by random invertible P, Q
        P, Q = rng.normal(size=(3, 3)), rng.normal(size=(3, 3))
        A, B = P.T @ np.diag([0.0, 0.0, 1.5]) @ Q, P.T @ np.eye(3) @ Q
        x0 = np.c_[rng.uniform(-1, 1, (7, 2)), np.ones(7)]
        x1 = np.cross(x0 @ A.T, x0 @ B.T)
        out.append(("repeated_root", np.concatenate([x0[:, :2], x1[:, :2] / x1[:, 2:]], 1)))
    # the rank rule: the seventh row moved off the sixth by delta, bisected to where the host's rule flips
    base = _fm_scene(rng)
    d = rng.normal(size=4)

    def sample(delta):
        q = base.copy()
        q[6] = q[5] + delta * d
        return q

    rank_ok = lambda delta: bool(G._null_basis(sample(delta)[None])[1][0])
    lo, hi = 0.0, 1e-6
    assert not rank_ok(lo) and rank_ok(hi)
    for _ in range(300):
        mid = (lo + hi) / 2
        if mid in (lo, hi):
            break
        lo, hi = (lo, mid) if rank_ok(mid) else (mid, hi)
    out += [("rank_below", sample(lo)), ("rank_above", sample(hi))]
    return out


# ------------------------------------------------------------------ CPU: the host models against 60 digits
def _quartics(n_random=150):
    """Host quartics with their inputs: exact scenes, random inconsistent samples and the structured set."""
    rng = np.random.default_rng(3)
    items = [_ap_exact_sample(s) for s in range(n_random)]
    items += [(_unit(rng.normal(size=(3, 3)) + [0, 0, 1.5]), rng.normal(size=(3, 3)) * 4) for _ in range(n_random)]
    items += [(j, X) for _, j, X in _ap_structured()]
    j = np.stack([a for a, _ in items])
    X = np.stack([b for _, b in items])
    A, _ = L.grunert_quartic(j, X)
    return j, X, A


def _cubics(n_random=150):
    rng = np.random.default_rng(4)
    q = [_fm_exact_sample(s) for s in range(n_random)]
    q += [rng.uniform(-1, 1, (7, 4)) for _ in range(n_random)]
    q += [x for _, x in _fm_structured()]
    q = np.stack(q)
    basis, ok = G._null_basis(q)
    c, _, _ = G.fundamental_cubic(basis)
    return q, basis, ok, c


def test_quartic_coefficients_within_the_running_error_bound():
    j, X, A = _quartics()
    worst = 0.0
    for k in range(len(j)):
        ref, mags = _grunert_mp(j[k], X[k]), _grunert_mags(j[k], X[k])
        if not np.isfinite(A[k]).all():
            continue
        r = _within(A[k], ref, mags)
        assert r <= 1.0, (k, r, A[k])
        worst = max(worst, r)
    print(f"{len(j)} quartics: worst |A_host - A_60| / running bound {worst:.3f}")
    assert A[len(j) - len(_ap_structured())][4] == 0.0     # the isosceles sample's degree drop is exact


def test_cubic_coefficients_within_the_running_error_bound():
    q, basis, ok, c = _cubics()
    worst = 0.0
    for k in np.flatnonzero(ok):
        r = _within(c[k], _cubic_mp(basis[k]), _cubic_mags(basis[k]))
        assert r <= 1.0, (k, r)
        worst = max(worst, r)
    print(f"{int(ok.sum())} cubics: worst |c_host - c_60| / (gamma_9 m) {worst:.3f}")


def test_null_basis_is_a_null_basis_to_householder_accuracy():
    """The Householder null basis of the 7 epipolar rows: orthonormal to 20 u, and |M b| <= 100 u |M|_F (Householder
    QR is backward stable with a backward error of a small multiple of 9 * 7 u |M|_F, Higham Thm 19.4)."""
    q, basis, ok, _ = _cubics()
    worst = 0.0
    for k in np.flatnonzero(ok):
        a0, b0, a1, b1 = (q[k, :, i] for i in range(4))
        M = np.stack([a1 * a0, a1 * b0, a1, b1 * a0, b1 * b0, b1, a0, b0, np.ones(7)], 1)
        with mpmath.workdps(60):
            Mm = mpmath.matrix(M.tolist())
            for b in basis[k]:
                r = Mm * mpmath.matrix(b.tolist())
                res = float(mpmath.norm(r))
                worst = max(worst, res / (U * np.linalg.norm(M)))
                assert res <= 100 * U * np.linalg.norm(M), (k, res)
        G2 = basis[k] @ basis[k].T
        assert np.abs(G2 - np.eye(2)).max() <= 20 * U, k
    print(f"worst |M b| / (u |M|_F) {worst:.2f}")


def _check_roots(c, roots, count, what):
    """The host's roots of polynomial c (ascending) against the exact reference: the count always, each root inside
    its Horner band when the roots are separated by SEPARATION.  -> False only when skipped as clustered."""
    p = np.zeros(11)
    p[:len(c)] = c
    ex = exact_roots(p)
    if ex is None:
        assert count == 0, what
        return True
    n, br = ex
    rs = [(lo + hi) / 2 for lo, hi in br]
    if any(abs(b - a) <= SEPARATION * max(abs(a), abs(b)) for a, b in zip(rs, rs[1:])):
        return False                  # clustered / multiple roots: the count is within rounding (test_ransac_edges)
    assert count == n, (what, count, n)
    B = _cauchy(p)
    for i, r in enumerate(rs):
        err = abs(Fraction(float(roots[i])) - r)
        assert float(err) <= _band(p, r, B), (what, i, float(roots[i]), float(r))
    return True


def test_cubic_and_quartic_roots_against_exact_roots():
    _, _, ok, c = _cubics()
    P = np.zeros((len(c), 11))
    P[:, :4] = c
    roots, count = G.sturm_roots(P)
    n_c = sum(_check_roots(c[k], roots[k], int(count[k]), ("cubic", k)) for k in np.flatnonzero(ok))
    _, _, A = _quartics()
    P = np.zeros((len(A), 11))
    P[:, :5] = A
    roots, count = G.sturm_roots(P)
    live = np.isfinite(A).all(1)
    n_q = sum(_check_roots(A[k], roots[k], int(count[k]), ("quartic", k)) for k in np.flatnonzero(live))
    print(f"roots checked inside their Horner band: {n_c} of {int(ok.sum())} cubics, {n_q} of {int(live.sum())} quartics")
    # every polynomial with separated roots had its count and roots checked above; the rest are the clustered ones
    # (the structured double roots and danger cylinders)
    skipped_c = int(ok.sum()) - n_c
    skipped_q = int(live.sum()) - n_q
    print(f"skipped as clustered: {skipped_c} cubics, {skipped_q} quartics")
    assert skipped_c <= 8 and skipped_q <= 8


def _host_layout_mismatch(a, oka, b, okb):
    """The bit-for-bit comparator of two solution sets in the host layout ([K, S, ...] with ok [K, S]): per sample,
    True if they keep different roots or any bit of a kept solution differs."""
    K, S = oka.shape
    ab = np.where(oka[..., None], _bits(a.reshape(K, S, -1)), 0)
    bb = np.where(okb[..., None], _bits(b.reshape(K, S, -1)), 0)
    return (oka != okb).any(1) | (ab != bb).any((1, 2))


def test_comparators_catch_one_ulp_and_a_wrong_sign(monkeypatch):
    """Moving one coefficient of the host cubic / quartic by 1 ulp changes the solutions' bits on a large fraction of
    the samples (the bit-for-bit comparator flags them), while the 60-digit bound still holds (it is not slack enough
    to hide a wrong formula: a wrong sign in one coefficient fails it)."""
    q, basis, ok, c = _cubics()
    F0, ok0 = G.fundamental_solutions(q)
    cubic = G.fundamental_cubic

    def ulp_cubic(b):
        cc, F2, D = cubic(b)
        cc = cc.copy()
        cc[:, 1] = np.nextafter(cc[:, 1], np.inf)
        return cc, F2, D

    monkeypatch.setattr(G, "fundamental_cubic", ulp_cubic)
    F1, ok1 = G.fundamental_solutions(q)
    frac_c = float(_host_layout_mismatch(F0, ok0, F1, ok1)[ok].mean())
    monkeypatch.undo()
    c_ulp = ulp_cubic(basis)[0]
    for k in np.flatnonzero(ok)[:60]:
        assert _within(c_ulp[k], _cubic_mp(basis[k]), _cubic_mags(basis[k])) <= 1.0, k
    sign_fail = np.mean([_within(np.r_[c[k][:2], -c[k][2], c[k][3]], _cubic_mp(basis[k]), _cubic_mags(basis[k])) > 1
                         for k in np.flatnonzero(ok)[:60]])

    j, X, A = _quartics()
    R0, t0, l0 = L.p3p_solutions(j, X)
    quartic = L.grunert_quartic

    def ulp_quartic(jj, XX):
        AA, w = quartic(jj, XX)
        AA = AA.copy()
        AA[:, 2] = np.nextafter(AA[:, 2], np.inf)
        return AA, w

    monkeypatch.setattr(L, "grunert_quartic", ulp_quartic)
    R1, t1, l1 = L.p3p_solutions(j, X)
    monkeypatch.undo()
    sols0 = np.concatenate([R0.reshape(len(j), 4, 9), t0], 2)
    sols1 = np.concatenate([R1.reshape(len(j), 4, 9), t1], 2)
    frac_q = float(_host_layout_mismatch(sols0, l0, sols1, l1).mean())
    A_ulp = ulp_quartic(j, X)[0]
    live = np.flatnonzero(np.isfinite(A).all(1))[:60]
    for k in live:
        assert _within(A_ulp[k], _grunert_mp(j[k], X[k]), _grunert_mags(j[k], X[k])) <= 1.0, k
    sign_fail_q = np.mean([_within(np.r_[A[k][:3], -A[k][3], A[k][4]], _grunert_mp(j[k], X[k]),
                                   _grunert_mags(j[k], X[k])) > 1 for k in live])
    print(f"1-ulp change flags {frac_c:.2f} of cubic samples and {frac_q:.2f} of quartic samples; a wrong sign fails "
          f"the bound on {sign_fail:.2f} / {sign_fail_q:.2f}")
    assert frac_c >= 0.5 and frac_q >= 0.5
    assert sign_fail >= 0.95 and sign_fail_q >= 0.95


# ------------------------------------------------------------------ CPU: the line check on exact cases
# F = [t]x with t = (1, 0, 0): the epipolar line of (x, y) is y' = y in the other image (a rectified pair).
F_RECT = np.array([[0.0, 0, 0], [0, 0, -1], [0, 1, 0]])
# F = [t]x with t = (0, 0, 1): both epipoles at the origin.
F_EPI = np.array([[0.0, -1, 0], [1, 0, 0], [0, 0, 0]])
EPS32 = float(np.finfo(np.float32).eps)


def _line_cases():
    """(name, F, s0, s1, min_overlap, expected r1, expected r0 (NaN: cannot reject), expected decision)."""
    v = [[0, 0], [0, 4]]                                            # vertical segment y in [0, 4]
    nan = np.nan
    return [
        ("ratio_equal", F_RECT, [[1, 2], [1, 6]], v, 0.5, 0.5, 0.5, True),
        ("ratio_ulp_below", F_RECT, [[1, 2], [1, 6]], v, math.nextafter(0.5, 1), 0.5, 0.5, False),
        ("ta_eq_tb", F_RECT, [[1, 2], [7, 2]], v, 0.5, nan, nan, True),     # s0 along the epipolar direction
        ("eps_rule_nan", F_RECT, [[0, 0], [0, 1]], [[0, 0], [1, EPS32]], 0.5, nan, None, None),
        ("eps_rule_finite", F_RECT, [[0, 0], [0, 1]], [[0, 0], [1, float(np.nextafter(np.float32(EPS32),
                                                                                         np.float32(1)))]],
         0.5, None, None, None),
        ("through_epipole", F_EPI, [[-1, -1], [2, 2]], [[10, 0], [10, 8]], 0.5, nan, nan, True),
        ("zero_length_s0", F_RECT, [[3, 3], [3, 3]], v, 0.5, nan, nan, True),
        ("zero_length_s1", F_RECT, [[1, 2], [1, 6]], [[5, 5], [5, 5]], 0.5, nan, nan, True),
        ("zero_length_both", F_RECT, [[3, 3], [3, 3]], [[5, 5], [5, 5]], 0.5, nan, nan, True),
        ("disjoint_min0", F_RECT, [[1, 10], [1, 14]], v, 0.0, 0.0, 0.0, True),
        ("disjoint_min05", F_RECT, [[1, 10], [1, 14]], v, 0.5, 0.0, 0.0, False),
        ("inside_min1", F_RECT, [[1, 1], [1, 3]], v, 1.0, 1.0, 1.0, True),
        ("partial_min1", F_RECT, [[1, 2], [1, 6]], v, 1.0, 0.5, 0.5, False),
    ]


def _line_arrays(cases):
    F = np.stack([np.asarray(c[1], np.float64).reshape(9) for c in cases])
    s0 = np.stack([np.asarray(c[2], np.float32).reshape(4) for c in cases])
    s1 = np.stack([np.asarray(c[3], np.float32).reshape(4) for c in cases])
    mo = np.array([c[4] for c in cases])
    return F, s0, s1, mo


def _host_lines(F, s0, s1, mo):
    r1 = np.empty(len(F))
    r0 = np.empty(len(F))
    ok = np.empty(len(F), bool)
    for i in range(len(F)):
        a, b = G.line_overlap_ratios(F[i], s0[i:i + 1].reshape(1, 2, 2), s1[i:i + 1].reshape(1, 2, 2))
        r1[i], r0[i] = a[0], b[0]
        ok[i] = G.lines_consistent(F[i], s0[i:i + 1].reshape(1, 2, 2), s1[i:i + 1].reshape(1, 2, 2), mo[i])[0]
    return r1, r0, ok


def test_line_check_exact_cases():
    """The hand-built cases' ratios and decisions.  A zero-length segment on either side (or a segment along the
    epipolar direction, or through the epipole) gives NaN ratios, and NaN cannot reject: such a match is consistent."""
    cases = _line_cases()
    r1, r0, ok = _host_lines(*_line_arrays(cases))
    for i, (name, _, _, _, _, e1, e0, eok) in enumerate(cases):
        for got, want in ((r1[i], e1), (r0[i], e0)):
            if want is not None:
                assert (np.isnan(got) and np.isnan(want)) or got == want, (name, got, want)
        if eok is not None:
            assert ok[i] == eok, name
    # the FLT_EPSILON rule flips between the two float32 slopes
    idx = {c[0]: i for i, c in enumerate(cases)}
    assert np.isnan(r1[idx["eps_rule_nan"]]) and np.isfinite(r1[idx["eps_rule_finite"]])


# ------------------------------------------------------------------ GPU hooks
def _stream():
    return C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)


def _dev(a, dtype=np.float64):
    return torch.as_tensor(np.ascontiguousarray(a, dtype=dtype), device=DEV)


def _fm_solve_gpu(q):
    qd = _dev(q)
    n = qd.shape[0]
    F = torch.empty((n, 3, 9), dtype=torch.float64, device=DEV)
    jr = torch.empty((n, 3), dtype=torch.int32, device=DEV)
    ns = torch.empty(n, dtype=torch.int32, device=DEV)
    with torch.cuda.device(DEV):
        rc = N.load().ltr_debug_fundamental_solve(qd.data_ptr(), n, F.data_ptr(), jr.data_ptr(), ns.data_ptr(),
                                                  DEV.index, _stream())
    N.check(rc, "ltr_debug_fundamental_solve")
    return F.cpu().numpy(), jr.cpu().numpy(), ns.cpu().numpy()


def _p3p_gpu(j, X):
    jd, Xd = _dev(j), _dev(X)
    n = jd.shape[0]
    R = torch.empty((n, 4, 9), dtype=torch.float64, device=DEV)
    t = torch.empty((n, 4, 3), dtype=torch.float64, device=DEV)
    jr = torch.empty((n, 4), dtype=torch.int32, device=DEV)
    ns = torch.empty(n, dtype=torch.int32, device=DEV)
    with torch.cuda.device(DEV):
        rc = N.load().ltr_debug_p3p(jd.data_ptr(), Xd.data_ptr(), n, R.data_ptr(), t.data_ptr(), jr.data_ptr(),
                                    ns.data_ptr(), DEV.index, _stream())
    N.check(rc, "ltr_debug_p3p")
    return R.cpu().numpy(), t.cpu().numpy(), jr.cpu().numpy(), ns.cpu().numpy()


def _lines_gpu(F, s0, s1, min_overlap):
    Fd, a, b = _dev(F), _dev(s0, np.float32), _dev(s1, np.float32)
    n = Fd.shape[0]
    r1 = torch.empty(n, dtype=torch.float64, device=DEV)
    r0 = torch.empty(n, dtype=torch.float64, device=DEV)
    ok = torch.empty(n, dtype=torch.uint8, device=DEV)
    with torch.cuda.device(DEV):
        rc = N.load().ltr_debug_fundamental_lines(Fd.data_ptr(), a.data_ptr(), b.data_ptr(), n, float(min_overlap),
                                                  r1.data_ptr(), r0.data_ptr(), ok.data_ptr(), DEV.index, _stream())
    N.check(rc, "ltr_debug_fundamental_lines")
    return r1.cpu().numpy(), r0.cpu().numpy(), ok.cpu().numpy()


def _to_host_layout(vals, jr, ns, S):
    """Kernel solutions [K, S, ...] in solution order with root indices -> the host layout (slot = root index)."""
    K = len(ns)
    out = np.full(vals.shape, np.nan)
    ok = np.zeros((K, S), bool)
    for s in range(S):
        live = np.flatnonzero(jr[:, s] >= 0)
        out[live, jr[live, s]] = vals[live, s]
        ok[live, jr[live, s]] = True
    assert np.array_equal(ok.sum(1), ns)
    # the kernel emits solutions in ascending root order and NaN / -1 past the count
    assert all(np.all(np.diff(jr[k, :ns[k]]) > 0) and (jr[k, ns[k]:] == -1).all() for k in range(K))
    return out, ok


def _fm_compare(q):
    Fg, jg, ng = _fm_solve_gpu(q)
    Fh, okh = G.fundamental_solutions(q)
    for k in range(len(q)):
        assert np.isnan(Fg[k, ng[k]:]).all(), k
    Fgh, okg = _to_host_layout(Fg, jg, ng, 3)
    bad = _host_layout_mismatch(Fgh, okg, Fh, okh)
    assert not bad.any(), (int(bad.sum()), np.flatnonzero(bad)[:10])
    return ng


def _ap_compare(j, X):
    Rg, tg, jg, ng = _p3p_gpu(j, X)
    Rh, th, okh = L.p3p_solutions(j, X)
    for k in range(len(j)):
        assert np.isnan(Rg[k, ng[k]:]).all() and np.isnan(tg[k, ng[k]:]).all(), k
    sg = np.concatenate([Rg, tg], 2)
    sh = np.concatenate([Rh.reshape(len(j), 4, 9), th], 2)
    sgh, okg = _to_host_layout(sg, jg, ng, 4)
    bad = _host_layout_mismatch(sgh, okg, sh, okh)
    assert not bad.any(), (int(bad.sum()), np.flatnonzero(bad)[:10])
    return ng


def _fm_ragged_samples(per_pair=700):
    """The seven-point samples the estimator draws on the ragged pairs of test_fundamental (normalised as it does)."""
    out = []
    for p, d in enumerate(_fm_ragged()):
        pts, _, _, _, _ = G._correspondences(d["kpts0"], d["kpts1"], d["matches_p"], E22, E22, np.zeros(0, np.int64),
                                             True, False)
        if len(pts) < 7:
            continue
        nm = G._normalisation(pts, E22, E22)
        f = lambda v: np.asarray(v, dtype=np.float64)
        q = np.stack([(f(pts[:, 0]) - nm.c0x) * nm.i0, (f(pts[:, 1]) - nm.c0y) * nm.i0,
                      (f(pts[:, 2]) - nm.c1x) * nm.i1, (f(pts[:, 3]) - nm.c1y) * nm.i1], 1)
        idx, ok = G.draw_samples(9, p, per_pair, len(q), 7)
        out.append(q[idx[ok]])
    return np.concatenate(out)


def _ap_ragged_samples(per_group=700):
    """The P3P samples the estimator draws on the ragged groups of test_localization (bearings and shifted points)."""
    js, Xs = [], []
    for g, cases in enumerate(_ragged_groups()):
        for d in cases:
            grp, _, _ = L.stage_group(d["kpts0"], d["matches_p"], d["points3d1"], d["K"])
            if len(grp.X) < 3:
                continue
            idx, ok = G.draw_samples(9, g, per_group, len(grp.X), 3)
            qn = np.stack([grp.d[:, 0] / grp.K[0, 0], grp.d[:, 1] / grp.K[1, 1]], 1)
            js.append(L.bearings(qn[idx[ok]]))
            Xs.append(grp.X[idx[ok]])
    return np.concatenate(js), np.concatenate(Xs)


@pytest.mark.gpu
def test_seven_point_solver_bit_for_bit():
    q = _fm_ragged_samples()
    assert len(q) >= 100_000
    ng = _fm_compare(q)
    names, qs = zip(*_fm_structured())
    ns = _fm_compare(np.stack(qs))
    got = dict(zip(names, ns))
    print(f"{len(q)} ragged samples, {int(ng.sum())} solutions, {np.bincount(ng, minlength=4).tolist()} per count; "
          f"structured {list(zip(names, ns.tolist()))}")
    assert got["rank_below"] == 0 and got["rank_above"] > 0
    assert all(n == 0 for name, n in zip(names, ns) if name == "duplicated_rows")


@pytest.mark.gpu
def test_p3p_bit_for_bit():
    j, X = _ap_ragged_samples()
    assert len(j) >= 100_000
    ng = _ap_compare(j, X)
    names, js, Xs = zip(*_ap_structured())
    ns = _ap_compare(np.stack(js), np.stack(Xs))
    got = dict(zip(names, ns))
    print(f"{len(j)} ragged samples, {int(ng.sum())} solutions, {np.bincount(ng, minlength=5).tolist()} per count; "
          f"structured {list(zip(names, ns.tolist()))}")
    assert got["den_0"] == 0
    # the collinearity rule rejects k <= 0 and accepts from some k > 0 on (the solver then returns what the quartic
    # allows); each k is a distinct world point
    eps = [n for name, n in zip(names, ns) if name.startswith("collinear_ulp")]
    Xs_eps = [X for name, _, X in _ap_structured() if name.startswith("collinear_ulp")]
    rule = [_collinear_ok(X) for X in Xs_eps]
    assert rule[:4] == [False] * 4 and rule[-1] and rule == sorted(rule) and eps[:4] == [0] * 4, rule
    assert len({X.tobytes() for X in Xs_eps}) == 7


@pytest.mark.gpu
def test_line_check_bit_for_bit():
    cases = _line_cases()
    F, s0, s1, mo = _line_arrays(cases)
    r1h, r0h, okh = _host_lines(F, s0, s1, mo)
    for i in range(len(cases)):
        r1, r0, ok = _lines_gpu(F[i:i + 1], s0[i:i + 1], s1[i:i + 1], mo[i])
        assert _bits(r1)[0] == _bits(r1h)[i] and _bits(r0)[0] == _bits(r0h)[i] and bool(ok[0]) == okh[i], cases[i][0]
    # 100 random F (over 6 decades of scale), each the F of 1000 random segment pairs, so that the host model itself
    # (one F per call) is the reference
    rng = np.random.default_rng(8)
    n_f, per = 100, 1000
    n = n_f * per
    Fs = rng.normal(size=(n_f, 9)) * 10.0 ** rng.uniform(-6, 0, (n_f, 1))
    Fr = np.repeat(Fs, per, 0)
    a = rng.uniform(0, 640, (n, 4)).astype(np.float32)
    b = rng.uniform(0, 640, (n, 4)).astype(np.float32)
    zero0 = rng.random(n) < 0.005
    zero1 = rng.random(n) < 0.005
    horiz = rng.random(n) < 0.005
    a[zero0, 2:] = a[zero0, :2]                                  # zero-length segments on side 0
    b[zero1, 2:] = b[zero1, :2]                                  # and on side 1
    a[horiz, 3] = a[horiz, 1]                                    # axis-aligned
    h1, h0 = np.empty(n), np.empty(n)
    for f in range(n_f):
        sl = slice(f * per, (f + 1) * per)
        h1[sl], h0[sl] = G.line_overlap_ratios(Fs[f], a[sl].reshape(-1, 2, 2), b[sl].reshape(-1, 2, 2))
    assert np.isnan(h1[zero0 | zero1]).all() and np.isnan(h0[zero0 | zero1]).all()
    for mo_ in (0.0, 0.5, 1.0):
        r1, r0, ok = _lines_gpu(Fr, a, b, mo_)
        hok = np.concatenate([G.lines_consistent(Fs[f], a[f * per:(f + 1) * per].reshape(-1, 2, 2),
                                                 b[f * per:(f + 1) * per].reshape(-1, 2, 2), mo_) for f in range(n_f)])
        assert np.array_equal(_bits(r1), _bits(h1)) and np.array_equal(_bits(r0), _bits(h0))
        assert np.array_equal(ok.astype(bool), hok)
    print(f"{n} random pairs: {int(np.isnan(r1).sum())} / {int(np.isnan(r0).sum())} NaN sides, "
          f"{int((zero0 | zero1).sum())} zero-length, {int(horiz.sum())} axis-aligned")


@pytest.mark.gpu
def test_hooks_refuse_bad_arguments():
    lib = N.load()
    assert lib.ltr_debug_fundamental_solve(None, 1, None, None, None, 0, None) == LTR_E_INVALID
    assert lib.ltr_debug_p3p(None, None, -1, None, None, None, None, 0, None) == LTR_E_INVALID
    z = _dev(np.zeros((1, 9)))
    s = _dev(np.zeros((1, 4)), np.float32)
    o = torch.empty(1, dtype=torch.float64, device=DEV)
    u8 = torch.empty(1, dtype=torch.uint8, device=DEV)
    for mo in (-0.1, 1.5, float("nan")):
        assert lib.ltr_debug_fundamental_lines(z.data_ptr(), s.data_ptr(), s.data_ptr(), 1, mo, o.data_ptr(),
                                               o.data_ptr(), u8.data_ptr(), 0, None) == LTR_E_INVALID
    assert lib.ltr_debug_fundamental_solve(None, 0, None, None, None, 0, None) == 0


# ------------------------------------------------------------------ every hypothesis end to end
P_COPIES = 1000


def _fm_run(res, **kw):
    out = G.estimate_fundamentals(res, **kw)
    return {f: getattr(out, f).cpu().numpy() for f in FM_FIELDS}


def _ap_run(res, Ks, X1, L1, groups, **kw):
    out = L.estimate_absolute_poses(res, Ks, X1, L1, groups=groups, **kw)
    return {f: getattr(out, f).cpu().numpy() for f in AP_FIELDS}


def check_group(res, X1, L1, groups, Ks, got, g, **kw):
    """Group g of an estimate_absolute_poses result against the host model, every output bit for bit."""
    h = _host_group(res, X1, L1, groups, Ks, g, **kw)
    a, b = res.offsets_p[groups[g]], res.offsets_p[groups[g + 1]]
    c, e = res.offsets_l[groups[g]], res.offsets_l[groups[g + 1]]
    assert bool(got["valid"][g]) == h["valid"] and bool(got["refit"][g]) == h["refit"], g
    assert got["hypothesis"][g] == h["hypothesis"] and got["hypothesis_inliers"][g] == h["hypothesis_inliers"], g
    assert np.array_equal(got["inliers_p"][a:b], h["inliers_p"]) and np.array_equal(got["inliers_l"][c:e],
                                                                                     h["inliers_l"]), g
    assert got["n_inliers_p"][g] == h["n_inliers_p"] and got["n_inliers_l"][g] == h["n_inliers_l"], g
    assert np.array_equal(_bits(got["R"][g]), _bits(h["R"])) and np.array_equal(_bits(got["t"][g]), _bits(h["t"])), \
        (g, got["R"][g], h["R"], got["t"][g], h["t"])
    return h


FM_RATIOS = []


@pytest.mark.gpu
@pytest.mark.parametrize("outlier_frac", [0.0, 0.5])
def test_fundamental_every_hypothesis_end_to_end(outlier_frac):
    d = syn.make_fundamental_correspondences(61, 60, 20, noise_px=0.3, outlier_frac=outlier_frac)
    res = _fm_matches([d] * P_COPIES, shuffle_rows=False)
    got = _fm_run(res, n_hypotheses=1, seed=2)
    hyp = set()
    for p in range(P_COPIES):
        h = check_pair(res, got, p, stats=FM_RATIOS, n_hypotheses=1, seed=2)
        hyp.add(h["F_hypothesis"].tobytes())
    print(f"{P_COPIES} hypotheses, {len(hyp)} distinct, {int(got['refit'].sum())} refits kept; worst refit "
          f"|dF| / (u cond) so far {max(FM_RATIOS, default=0.0):.3g}")
    assert len(hyp) > P_COPIES // 2


@pytest.mark.gpu
@pytest.mark.parametrize("use_lines", [True, False])
@pytest.mark.parametrize("outlier_frac", [0.0, 0.5])
def test_absolute_pose_every_hypothesis_end_to_end(outlier_frac, use_lines):
    d = syn.make_localization_correspondences(62, 60, 20, noise_px=0.3, outlier_frac=outlier_frac)
    res, X1, L1, groups, Ks = _ap_matches([[d]] * P_COPIES, shuffle_rows=False)
    got = _ap_run(res, Ks, X1, L1, groups, n_hypotheses=1, seed=2, use_lines=use_lines)
    hyp = set()
    for g in range(P_COPIES):
        h = check_group(res, X1, L1, groups, Ks, got, g, n_hypotheses=1, seed=2, use_lines=use_lines)
        hyp.add(h["R_hypothesis"].tobytes())
    print(f"{P_COPIES} hypotheses, {len(hyp)} distinct, {int(got['valid'].sum())} valid, {int(got['refit'].sum())} "
          f"refits kept")
    assert len(hyp) > P_COPIES // 2


def _plant_lines(d, R, t, thresh, deltas, depth=5.0):
    """Line rows whose two world end points lie at pixel distance thresh + delta from their query line under the pose
    (R, t) (world frame), one row per delta: the query segment is the exact float32 segment (100, 100)-(500, 150), each
    end point's pixel is moved along the line's unit normal and lifted to the given depth, and the fp64 world point is
    R^T (P - t), whose rounding moves the distance by about 1e-13 px."""
    a, b = np.array([100.0, 100.0]), np.array([500.0, 150.0])
    nrm = np.array([-(b - a)[1], (b - a)[0]]) / np.linalg.norm(b - a)
    Ki = np.linalg.inv(d["K"])
    segs, ends = [], []
    for dl in deltas:
        E = []
        for x in (a, b):
            px = x + (thresh + dl) * nrm
            Pc = (Ki @ np.r_[px, 1.0]) * depth
            E.append(R.T @ (Pc - t))
        segs.append([a, b])
        ends.append(E)
    e = dict(d)
    e["klines0"] = np.concatenate([d["klines0"], np.asarray(segs, np.float32)])
    e["lines3d1"] = np.concatenate([d["lines3d1"], np.asarray(ends)])
    e["matches_l"] = np.arange(len(e["klines0"]), dtype=np.int32)
    return e


@pytest.mark.gpu
def test_absolute_pose_lines_planted_at_the_threshold():
    """Every hypothesis with two lines planted 5e-10 px inside and outside the 8 px threshold of that hypothesis' pose:
    the hypothesis' inlier count takes in the inside one and not the outside one (lines take no part in sampling, so
    the hypothesis is the same), in the kernels as in the host model, every output bit equal."""
    d = syn.make_localization_correspondences(63, 60, 10, noise_px=0.3, outlier_frac=0.5)
    P, th = 300, 8.0
    groups_of_cases, base = [], []
    for g in range(P):
        h = L.ransac_absolute_pose_host(d["kpts0"], d["matches_p"], d["points3d1"], d["K"], d["klines0"],
                                        d["matches_l"], d["lines3d1"], group=g, thresh=th, n_hypotheses=1, seed=2)
        base.append(h)
        if h["valid"]:
            groups_of_cases.append([_plant_lines(d, h["R_hypothesis"], h["t_hypothesis"], th, (-5e-10, 5e-10))])
        else:
            groups_of_cases.append([d])
    res, X1, L1, groups, Ks = _ap_matches(groups_of_cases, shuffle_rows=False)
    got = _ap_run(res, Ks, X1, L1, groups, thresh=th, n_hypotheses=1, seed=2)
    plus_one = n_valid = 0
    for g in range(P):
        h = check_group(res, X1, L1, groups, Ks, got, g, thresh=th, n_hypotheses=1, seed=2)
        if base[g]["valid"]:
            n_valid += 1
            plus_one += h["hypothesis"] == base[g]["hypothesis"] and \
                h["hypothesis_inliers"] == base[g]["hypothesis_inliers"] + 1
    print(f"{P} hypotheses, {n_valid} valid; the inside plant alone counted in {plus_one}")
    assert n_valid > P // 2 and plus_one >= 0.95 * n_valid


# ------------------------------------------------------------------ edges through the public API
def _fm_case(kp0, kp1, mp, l0=E22, l1=E22, ml=()):
    f = lambda a, s: np.asarray(a, np.float32).reshape(s)
    return {"kpts0": f(kp0, (-1, 2)), "kpts1": f(kp1, (-1, 2)), "matches_p": np.asarray(mp, np.int32).reshape(-1),
            "klines0": f(l0, (-1, 2, 2)), "klines1": f(l1, (-1, 2, 2)), "matches_l": np.asarray(ml, np.int32).reshape(-1)}


@pytest.mark.gpu
def test_fundamental_minimal_refit_and_inlier_edges():
    """Exactly 7 correspondences (no refit), 8 (the refit runs), degenerate sets, a keypoint at the epipole (a zero
    epipolar normal: an outlier), zero-length and axis-aligned segments, and unusual intrinsics."""
    cases = []
    for n in (7, 8):
        cases.append(syn.make_fundamental_correspondences(70 + n, n, 0, noise_px=0.0, outlier_frac=0.0))
    six = np.array([[1, 2], [30, 4], [5, 60], [70, 80], [9, 9], [40, 41]], np.float32)
    same = np.tile(np.float32([[100, 100]]), (10, 1))
    cases += [_fm_case(six, six + 1, np.arange(6)), _fm_case(same, same + 5, np.arange(10)), _fm_case(E22[:, 0], E22[:, 0], [])]
    d = syn.make_fundamental_correspondences(75, 80, 30, noise_px=0.3, outlier_frac=0.3)
    e0 = np.linalg.svd(d["F"])[2][-1]
    d["kpts0"][0] = (e0[:2] / e0[2]).astype(np.float32)          # (nearly) the epipole: F x0 ~ 0
    d["klines0"][:5, 1] = d["klines0"][:5, 0]                      # zero-length segments
    d["klines1"][5:10, 1] = d["klines1"][5:10, 0]
    d["klines0"][10:15, 1, 1] = d["klines0"][10:15, 0, 1]         # axis-aligned
    cases.append(d)
    rng = np.random.default_rng(76)
    for K0, K1 in ((np.array([[50.0, 0, 320], [0, 60, 240], [0, 0, 1]]), syn.random_intrinsics(rng)),
                   (np.array([[1e4, 0, 320], [0, 0.9e4, 240], [0, 0, 1]]), np.array([[1.2e4, 0, 300], [0, 1e4, 250],
                                                                                   [0, 0, 1]])),
                   (np.array([[500.0, 0, 2000], [0, 450, -1500], [0, 0, 1]]), syn.random_intrinsics(rng))):
        cases.append(syn.make_fundamental_correspondences(int(rng.integers(1e6)), 200, 20, noise_px=0.3,
                                                          outlier_frac=0.3, K0=K0, K1=K1))
    res = _fm_matches(cases, shuffle_rows=False)
    got = _fm_run(res, n_hypotheses=256, seed=3)
    for p in range(len(cases)):
        check_pair(res, got, p, n_hypotheses=256, seed=3)
    assert got["valid"][:2].all() and got["n_inliers"][:2].tolist() == [7, 8]
    assert not got["refit"][0] and not got["valid"][2:5].any()
    assert got["refit"][1] and got["hypothesis_inliers"][1] == 8          # the refit is kept on the equal count


@pytest.mark.gpu
@pytest.mark.parametrize("n_hyp", [1, 127, 128, 129, 4097])
def test_hypothesis_counts_around_the_cta(n_hyp):
    res = _fm_matches(_fm_ragged(16, seed=2))
    got = _fm_run(res, n_hypotheses=n_hyp, seed=4)
    for p in range(res.n_pairs):
        check_pair(res, got, p, n_hypotheses=n_hyp, seed=4)
    res, X1, L1, groups, Ks = _ap_matches(_ragged_groups(12, seed=3))
    got = _ap_run(res, Ks, X1, L1, groups, n_hypotheses=n_hyp, seed=4)
    for g in range(len(groups) - 1):
        check_group(res, X1, L1, groups, Ks, got, g, n_hypotheses=n_hyp, seed=4)


@pytest.mark.gpu
def test_fundamental_staging_filled_exactly():
    """11 377 keypoint rows stage within SMEM_MAX (18 bytes a row): accepted and compared; 11 378 are refused (code
    -4) before any launch."""
    n = G.SMEM_MAX // G.SMEM_PER_ROW_F
    assert n == 11377
    d = syn.make_fundamental_correspondences(80, n, 10, noise_px=0.3, outlier_frac=0.4)
    small = syn.make_fundamental_correspondences(81, 50, 3, noise_px=0.3, outlier_frac=0.4)
    res = _fm_matches([small, d], shuffle_rows=False)
    got = _fm_run(res, n_hypotheses=128, seed=6)
    for p in range(2):
        check_pair(res, got, p, n_hypotheses=128, seed=6)
    assert got["valid"].all()
    N.reset_launch_count()
    with pytest.raises(N.LtrError, match=r"code -4"):
        G.estimate_fundamentals(_fm_matches([syn.make_fundamental_correspondences(82, n + 1, 0)], shuffle_rows=False))
    assert N.launch_count() == 0


@pytest.mark.gpu
def test_absolute_pose_staging_filled_exactly_and_struct_row_bounds(monkeypatch):
    """A group of 4 pairs with 1000 point and 300 line rows each stages exactly SMEM_MAX bytes: accepted and compared;
    one more point row is refused (code -4) before any launch.  A caller's max_rows_p / max_rows_l below a multi-pair
    group's rows leaves that group invalid and the others as they were."""
    assert 4 * (1000 * L.SMEM_PER_POINT_A + 300 * L.SMEM_PER_LINE_A) == L.SMEM_MAX
    big = syn.make_localization_correspondences(90, 1000, 300, noise_px=0.3, outlier_frac=0.3)
    assert len(big["klines0"]) == 300
    res, X1, L1, groups, Ks = _shared_query(big, 4)
    got = _ap_run(res, Ks, X1, L1, groups, n_hypotheses=64, seed=6)
    check_group(res, X1, L1, groups, Ks, got, 0, n_hypotheses=64, seed=6)
    assert got["valid"].all()
    over = syn.make_localization_correspondences(90, 1001, 300, noise_px=0.3, outlier_frac=0.3)
    r2, X2, L2, g2, K2 = _shared_query(over, 4)
    N.reset_launch_count()
    with pytest.raises(N.LtrError, match=r"code -4"):
        L.estimate_absolute_poses(r2, K2, X2, L2, groups=g2)
    assert N.launch_count() == 0
    small = [syn.make_localization_correspondences(95, 40, 10, noise_px=0.3, outlier_frac=0.3)]
    # caller bounds on a batch: group 0 single-pair (40 / 10 rows), group 1 two pairs of 60 / 15 rows each
    two = [syn.make_localization_correspondences(96 + i, 60, 15, noise_px=0.3, outlier_frac=0.3) for i in range(2)]
    res, X1, L1, groups, Ks = _ap_matches([small, two, small], shuffle_rows=False)
    ref = _ap_run(res, Ks, X1, L1, groups, n_hypotheses=64, seed=6)
    call = L._ops.call_struct
    for bound in ({"max_rows_p": 100}, {"max_rows_l": 20}):
        monkeypatch.setattr(L._ops, "call_struct",
                            lambda entry, inputs, *a, **kw: call(entry, {**inputs, **bound}, *a, **kw))
        got = _ap_run(res, Ks, X1, L1, groups, n_hypotheses=64, seed=6)
        monkeypatch.undo()
        assert got["valid"].tolist() == [True, False, True], bound
        a, b = res.offsets_p[groups[1]], res.offsets_p[groups[2]]
        assert not got["inliers_p"][a:b].any() and got["hypothesis"][1] == -1 and np.isnan(got["R"][1]).all()
        for g in (0, 2):
            for f in AP_FIELDS:
                assert np.array_equal(_bits(got[f][g]) if got[f].dtype == np.float64 else got[f][g],
                                      _bits(ref[f][g]) if ref[f].dtype == np.float64 else ref[f][g]), (bound, g, f)


def _shared_query(d, n_pairs):
    """One group of n_pairs pairs that all match the whole query of correspondence set d (every pair n point and m line
    match rows, as a query image matched against several database images), with its 3D arrays."""
    from linetr_b200 import engine
    kq = torch.from_numpy(d["kpts0"]).to(DEV)
    lq = d["klines0"]
    mp = torch.from_numpy(np.tile(d["matches_p"], n_pairs)).to(DEV)
    ml = torch.from_numpy(np.tile(d["matches_l"], n_pairs)).to(DEV)
    offp = np.arange(n_pairs + 1, dtype=np.int32) * len(d["matches_p"])
    offl = np.arange(n_pairs + 1, dtype=np.int32) * len(d["matches_l"])
    z = torch.zeros(n_pairs, dtype=torch.int32, device=DEV)
    res = engine.ImagePairMatches(ml, ml.float(), z, offl, mp, mp.float(), z, offp, [lq] * n_pairs, [lq] * n_pairs,
                                  [kq] * n_pairs, [kq] * n_pairs)
    return res, [d["points3d1"]] * n_pairs, [d["lines3d1"]] * n_pairs, np.array([0, n_pairs]), d["K"][None]


EXACT_K = np.array([[512.0, 0.0, 320.0], [0.0, 512.0, 240.0], [0.0, 0.0, 1.0]])


def _exact_depth_query():
    """A query whose true pose is the identity and whose correspondences are exact: integer pixels, depths 2, 4, 8 and
    f = 512, so X = ((u - cx) z / 512, (v - cy) z / 512, z) is exact in fp64 and the estimated pose is the identity to
    rounding.  Rows 0 to 3 test the depth rule: the camera centre (depth exactly 0), points on the optical axis at depth
    +1e-6 and -1e-6 with the principal point as their keypoint, and inlier 4's point mirrored through the camera centre
    with inlier 4's keypoint.  It is run at a 1e-3 px threshold, so that only samples of exact rows win and the pose is
    the identity to about 1e-15: rows 1 to 3 then reproject to within 1e-6 px of their keypoints, and without the depth
    > 0 rule rows 2 and 3 would be inliers too.  Line 0 has one end point mirrored behind the camera
    (also on its query line); the other lines join two exact points."""
    rng = np.random.default_rng(110)
    n = 60
    uv = np.c_[rng.integers(0, 640, n), rng.integers(0, 480, n)].astype(np.float64)
    z = rng.choice([2.0, 4.0, 8.0], n)
    X = np.c_[(uv[:, 0] - 320.0) * z / 512.0, (uv[:, 1] - 240.0) * z / 512.0, z]
    kp, X = np.r_[np.tile([[320.0, 240.0]], (3, 1)), uv[4:5], uv], np.r_[[[0.0, 0.0, 0.0], [0.0, 0.0, 1e-6],
                                                                         [0.0, 0.0, -1e-6]], -X[4:5], X]
    ends = rng.integers(4, 4 + n, (12, 2))
    ends = ends[ends[:, 0] != ends[:, 1]][:10]
    segs = kp[ends]
    L3 = X[ends].copy()
    L3[0, 1] = -L3[0, 1]
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    return {"kpts0": f32(kp), "points3d1": X, "matches_p": np.arange(len(kp), dtype=np.int32), "klines0": f32(segs),
            "lines3d1": L3, "matches_l": np.arange(len(segs), dtype=np.int32), "R": np.eye(3), "t": np.zeros(3),
            "K": EXACT_K}


def test_depth_rule_at_the_exact_pose():
    """The host model's inlier rule at the true pose (the identity, exact): depth exactly 0 and -1e-6 are outliers,
    +1e-6 is an inlier, the mirrored point and the line with an end point behind the camera are outliers."""
    d = _exact_depth_query()
    g, _, _ = L.stage_group(d["kpts0"], d["matches_p"], d["points3d1"], d["K"], d["klines0"], d["matches_l"],
                            d["lines3d1"])
    f = L._inliers(g, np.eye(3), g.c.copy(), 1e-6)[0]             # X_cam = X = (X - c) + c
    npt = len(g.X)
    assert f[:4].tolist() == [False, True, False, False] and f[4:npt].all()
    assert not f[npt] and f[npt + 1:].all()


@pytest.mark.gpu
def test_absolute_pose_depth_rule():
    """The exact query through the public API: every output bit equal to the host model's, and the depth rule's
    decisions under the estimated pose: +1e-6 an inlier, -1e-6, the mirrored point and the line with an end point
    behind the camera outliers (depth exactly 0 under the true pose is a rounding-sized depth under the estimate: its
    decision is only compared with the host's)."""
    d = _exact_depth_query()
    res, X1, L1, groups, Ks = _ap_matches([[d]] * 4, shuffle_rows=False)
    got = _ap_run(res, Ks, X1, L1, groups, thresh=1e-3, n_hypotheses=128, seed=9)
    for g in range(4):
        check_group(res, X1, L1, groups, Ks, got, g, thresh=1e-3, n_hypotheses=128, seed=9)
        a, c = res.offsets_p[g], res.offsets_l[g]
        n = len(d["kpts0"])
        assert got["valid"][g] and got["inliers_p"][a + 1] and not got["inliers_p"][a + 2:a + 4].any(), g
        assert got["inliers_p"][a + 4:a + n].all(), g
        assert not got["inliers_l"][c] and got["inliers_l"][c + 1:c + len(d["matches_l"])].all(), g
        et, eR = L.absolute_pose_errors(got["R"][g], got["t"][g], np.eye(3), np.zeros(3))
        assert et[0] < 1e-6 and eR[0] < 1e-5, (g, et, eR)


def _shift_world(d, offset=0.0, scale=1.0):
    """The same query with its world scaled by `scale` and moved by `offset` (the projections are unchanged)."""
    e = dict(d)
    e["points3d1"] = d["points3d1"] * scale + offset
    e["lines3d1"] = d["lines3d1"] * scale + offset
    e["t"] = d["t"] * scale - d["R"] @ (np.full(3, offset) if np.ndim(offset) == 0 else offset)
    return e


@pytest.mark.gpu
def test_absolute_pose_edges():
    """Exactly 3 point rows (the refit runs on 3 inliers and is kept on the equal count), 3 points and one outlier
    line, zero-length and axis-aligned query segments, world coordinates offset by 1e6 with a 10-unit scene and a 1e-3-unit scene, and unusual intrinsics: every
    output bit equal to the host model's, and the scaled scenes' poses close to the truth relative to the scene."""
    groups_of_cases = []
    three = syn.make_localization_correspondences(100, 3, 0, noise_px=0.0, outlier_frac=0.0)
    groups_of_cases.append([three])
    tl = syn.make_localization_correspondences(101, 3, 1, noise_px=0.0, outlier_frac=0.0, line_outlier_frac=1.0)
    groups_of_cases.append([tl])
    d = syn.make_localization_correspondences(102, 80, 30, noise_px=0.3, outlier_frac=0.3)
    d["klines0"][1:4, 1] = d["klines0"][1:4, 0]                     # zero-length query segments
    d["klines0"][4:8, 1, 1] = d["klines0"][4:8, 0, 1]               # horizontal
    d["klines0"][8:12, 1, 0] = d["klines0"][8:12, 0, 0]             # vertical
    groups_of_cases.append([d])
    far = _shift_world(syn.make_localization_correspondences(103, 200, 40, noise_px=0.3, outlier_frac=0.3,
                                                             origin_scale=5.0), offset=1e6)
    tiny = _shift_world(syn.make_localization_correspondences(104, 200, 40, noise_px=0.3, outlier_frac=0.3), scale=1e-3)
    groups_of_cases += [[far], [tiny]]
    for Kx in (np.array([[50.0, 0, 320], [0, 65, 240], [0, 0, 1]]), np.array([[1e4, 0, 320], [0, 1.1e4, 240],
                                                                              [0, 0, 1]]),
               np.array([[500.0, 0, 2500], [0, 420, -1800], [0, 0, 1]])):
        groups_of_cases.append([syn.make_localization_correspondences(105, 150, 30, noise_px=0.3, outlier_frac=0.3,
                                                                      K=Kx)])
    res, X1, L1, groups, Ks = _ap_matches(groups_of_cases, shuffle_rows=False)
    got = _ap_run(res, Ks, X1, L1, groups, n_hypotheses=256, seed=7)
    for g in range(len(groups_of_cases)):
        check_group(res, X1, L1, groups, Ks, got, g, n_hypotheses=256, seed=7)
    assert got["valid"].all()
    assert got["hypothesis_inliers"][0] == 3 and got["n_inliers_p"][0] == 3 and got["refit"][0]   # kept on 3 == 3
    assert got["n_inliers_l"][1] == 0
    for g, sd, size in ((3, far, 10.0), (4, tiny, 1e-3 * 20)):
        et, eR = L.absolute_pose_errors(got["R"][g], got["t"][g], sd["R"], sd["t"])
        assert et[0] < 0.01 * size and eR[0] < 0.5, (g, et, eR)
