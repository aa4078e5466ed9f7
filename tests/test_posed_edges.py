"""The pose stages' shared dense solver and their stop and failure paths, at their edges.

- `_posed.cholesky_solve` (the numpy twin of rn_fp64.cuh `rc_cholesky_solve`) against exact arithmetic: Higham's
  componentwise backward error bounds (Thm 10.3 for the factor, 10.4 for the solve) evaluated exactly, and the forward
  error bound they imply, on random, graded and ill-conditioned SPD matrices and on the normal matrices
  `global_poses_host` and `bundle_adjust_host` factorize.  Three broken solvers (the pivot race's result, a dropped
  trailing-update term, a back substitution through L instead of L^T) must fall outside the bound.  Failed pivots
  (0, -0.0, negative, NaN; first, middle, last column) return False with x untouched and a pinned A.
- The bundle adjustment's stop reasons and rejected steps, and the global poses' half-turn pairs (an infinite Cayley
  residual), pinned in the numpy models.
- Triangulation: the min-angle rule at its boundary and one ulp either side, candidate depths of exactly 0 and one
  float32 ulp either side (a partner keypoint on the epipole), points at 1e6 depth, and the refit's guards (J^T J not
  > 0, a non-finite step), against 50-digit mpmath angles and least-squares depths.
- On the GPU: `ltr_debug_cholesky_solve` (the stages' own rc_cholesky_solve<1024>, in shared and in global memory)
  gives the twin's bits, and the edge scenes give their model's bits through `bundle_adjust`, `global_poses` and
  `triangulate`.
"""
import dataclasses
from fractions import Fraction

import mpmath
import numpy as np
import pytest
import torch

from linetr_b200 import _native as N
from linetr_b200 import _posed
from linetr_b200 import bundle as BA
from linetr_b200 import global_poses as GPm
from linetr_b200 import synthetic as syn
from linetr_b200 import tracks as TR
from linetr_b200 import triangulation as TRI
from tests.test_bundle import _assert_same as _ba_same, ring_matches, scene
from tests.test_global_poses import _same as _gp_same, ring, truth

U = Fraction(1, 2 ** 53)
LTR_E_INVALID = -1
S = 1100          # every double is an integer multiple of 2^-1074: x * 2^S is an exact Python int


def gamma(n):
    return n * U / (1 - n * U)


def _int(a):
    """Exact Python ints a * 2^S of a float64 array (object array, same shape)."""
    a = np.asarray(a, np.float64)
    out = np.empty(a.shape, object)
    for i, v in np.ndenumerate(a):
        p, q = float(v).as_integer_ratio()
        out[i] = p * ((1 << S) // q)
    return out


def _sym(A):
    """The symmetric matrix of A's lower triangle (what the solver reads)."""
    L = np.tril(A)
    return L + np.tril(A, -1).T


def backward_ratios(A0, b, L, x):
    """Exact componentwise backward error ratios of a solve: max_i |A0 x - b|_i / (g_{3m+1} (|L||L^T||x|)_i) (Thm
    10.4), and max_ij |A0 - L L^T|_ij / (g_{m+1} (|L||L^T|)_ij) over the lower triangle (Thm 10.3).  <= 1 passes."""
    m = len(A0)
    Ai, Li, xi, bi = _int(_sym(A0)), _int(np.tril(L)), _int(x.reshape(m, -1)), _int(b.reshape(m, -1))
    aL = np.abs(Li)
    r = np.abs(Ai.dot(xi) - bi * (1 << S))                         # scale 2^2S
    w = aL.dot(aL.T.dot(np.abs(xi)))                                  # scale 2^3S
    g = gamma(3 * m + 1)
    rs = max((Fraction(int(r[i, j]) << S, 1) / (g * int(w[i, j])) if w[i, j] else
              (Fraction(0) if r[i, j] == 0 else Fraction(10 ** 9))) for i in range(m) for j in range(r.shape[1]))
    F = np.abs(Ai * (1 << S) - Li.dot(Li.T))                         # scale 2^2S
    G = aL.dot(aL.T)
    g1 = gamma(m + 1)
    fs = max((Fraction(int(F[i, j]), 1) / (g1 * int(G[i, j])) if G[i, j] else
              (Fraction(0) if F[i, j] == 0 else Fraction(10 ** 9))) for i in range(m) for j in range(i + 1))
    return float(rs), float(fs)


def exact_solution(A0, b):
    """x = A0^-1 b: Fractions for m <= 16, else mpmath at 50 digits, as mpmath matrices."""
    m = len(A0)
    As = _sym(A0)
    B = b.reshape(m, -1)
    if m <= 16:
        M = [[Fraction(float(v)) for v in row] + [Fraction(float(v)) for v in B[i]] for i, row in enumerate(As)]
        k = B.shape[1]
        for c in range(m):
            for i in range(c + 1, m):
                f = M[i][c] / M[c][c]
                M[i] = [a - f * p for a, p in zip(M[i], M[c])]
        X = [[Fraction(0)] * k for _ in range(m)]
        for c in range(m - 1, -1, -1):
            for e in range(k):
                s = M[c][m + e] - sum(M[c][j] * X[j][e] for j in range(c + 1, m))
                X[c][e] = s / M[c][c]
        with mpmath.workdps(50):
            return mpmath.matrix([[mpmath.mpf(v.numerator) / v.denominator for v in row] for row in X])
    with mpmath.workdps(50):
        M = mpmath.matrix(As.tolist())
        X = mpmath.matrix(m, B.shape[1])
        for e in range(B.shape[1]):
            col = mpmath.lu_solve(M, mpmath.matrix(B[:, e].tolist()))
            for i in range(m):
                X[i, e] = col[i]
        return X


def forward_ratio(A0, b, L, x):
    """max |x - x^| / (g_{3m+1} |A^-1| |L||L^T||x^|): the forward bound the backward one implies (at 50 digits)."""
    m = len(A0)
    xs = x.reshape(m, -1)
    with mpmath.workdps(50):
        X = exact_solution(A0, b)
        Ai = mpmath.inverse(mpmath.matrix(_sym(A0).tolist()))
        aL = np.abs(np.tril(L))
        w = aL @ (aL.T @ np.abs(xs))            # rounding here is far below the bound's slack
        g = mpmath.mpf(float(gamma(3 * m + 1))) * (1 + mpmath.mpf(2) ** -40)
        worst = mpmath.mpf(0)
        for i in range(m):
            for e in range(xs.shape[1]):
                bound = g * mpmath.fsum(abs(Ai[i, j]) * mpmath.mpf(float(w[j, e])) * (1 + mpmath.mpf(2) ** -40)
                                        for j in range(m))
                err = abs(X[i, e] - mpmath.mpf(float(xs[i, e])))
                if err:
                    worst = max(worst, err / bound)
        return float(worst)


# ------------------------------------------------------------------ the matrices
def random_spd(rng, m, scale=1.0):
    G = rng.normal(size=(m, m))
    return scale * ((G @ G.T) / m + 0.1 * np.eye(m))


def graded(rng, m):
    d = np.logspace(-8, 8, m)
    B = random_spd(rng, m)
    s = np.sqrt(d)
    return (s[:, None] * B) * s[None, :]


def conditioned(rng, m, cond):
    Q, _ = np.linalg.qr(rng.normal(size=(m, m)))
    A = (Q * np.logspace(0, -np.log10(cond), m)) @ Q.T
    return 0.5 * (A + A.T)


def _capture(module, run):
    """The (A, x) of every cholesky_solve call `run()` makes through `module`, copied before the solve."""
    seen = []
    real = module.cholesky_solve

    def spy(A, x):
        seen.append((A.copy(), x.copy()))
        return real(A, x)
    module.cholesky_solve = spy
    try:
        run()
    finally:
        module.cholesky_solve = real
    return seen


def gp_systems():
    """The anchored Laplacians of a noisy 12-image ring with planted outliers (rotation k = 3, positions k = 6)."""
    n = 12
    Rt, tt, _ = truth(21, n)
    pairs = ring(n, 3)
    rp = syn.make_relative_poses(Rt, tt, pairs, noise_deg=0.5, outlier_frac=0.15, seed=22)
    seen = _capture(GPm, lambda: GPm.global_poses_host(pairs, rp, n, rot_iters=8, pos_iters=6))
    rot = [s for s in seen if s[1].shape[1] == 3]
    pos = [s for s in seen if s[1].shape[1] == 6]
    return [rot[0], rot[-1], pos[0], pos[-1]]


def ba_systems():
    """The reduced camera matrices of a point-and-line scene (first and last iteration)."""
    d, pairs, R, t = scene(31, V=9, n_pts=60, n_lines=12, ring=2)
    tr = TR.triangulate_tracks_host(d["keypoints"], d["klines"], pairs, ring_matches(d, pairs, torch.device("cpu")),
                                    d["K"], R, t, thresh=8, epi_thresh=8)
    seen = _capture(BA, lambda: BA.bundle_adjust_host(d["keypoints"], d["klines"], d["K"], R, t, tr, max_iters=4))
    return [(A, x[:, None]) for A, x in (seen[0], seen[-1])]


def cpu_cases():
    """(name, A, b) of the CPU matrices; b [m, k]."""
    rng = np.random.default_rng(5)
    out = []
    for m, k in ((1, 1), (2, 3), (5, 1), (16, 6), (33, 3), (64, 1)):
        out.append((f"spd{m}", random_spd(rng, m), rng.normal(size=(m, k))))
    for m in (8, 40, 127):
        out.append((f"graded{m}", graded(rng, m), rng.normal(size=(m, 1))))
    out.append(("spd127", random_spd(rng, 127), rng.normal(size=(127, 3))))
    for c in (1e10, 1e12, 1e14, 1e15):
        out.append((f"cond{c:.0e}", conditioned(rng, 12, c), rng.normal(size=(12, 3))))
    out.append(("cond1e13_m48", conditioned(rng, 48, 1e13), rng.normal(size=(48, 1))))
    for i, (A, x) in enumerate(gp_systems()):
        out.append((f"gp{i}", A, x))
    for i, (A, x) in enumerate(ba_systems()):
        out.append((f"ba{i}", A, x))
    return out


CASES = cpu_cases()


def twin(A, b):
    A1, x1 = A.copy(), b.copy()
    ok = _posed.cholesky_solve(A1, x1)
    return ok, A1, x1


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_solver_within_the_backward_bound(case):
    name, A, b = case
    ok, L, x = twin(A, b)
    assert ok, name
    rs, fs = backward_ratios(A, b, L, x)
    assert rs <= 1.0 and fs <= 1.0, (name, rs, fs)


FORWARD = [c for c in CASES if len(c[1]) <= 48 or c[0] == "spd127"]      # |A^-1| at 50 digits: 20 s at m = 127


@pytest.mark.parametrize("case", FORWARD, ids=[c[0] for c in FORWARD])
def test_solver_within_the_forward_bound(case):
    name, A, b = case
    ok, L, x = twin(A, b)
    assert ok
    assert forward_ratio(A, b, L, x) <= 1.0, name


def test_graph_systems_are_what_the_stages_solve():
    """The captured systems are the stages' own: GP's are Laplacians with the anchor removed (rows of a weighted
    Laplacian: diagonal >= the sum of the off-diagonal magnitudes), BA's carry the camera blocks."""
    for name, A, b in CASES:
        if name.startswith("gp"):
            S_ = _sym(A)
            off = np.abs(S_).sum(1) - np.abs(np.diag(S_))
            assert (np.diag(S_) >= off * (1 - 1e-12)).all() and (S_ - np.diag(np.diag(S_)) <= 0).all(), name
        if name.startswith("ba"):
            assert len(A) % 6 in (0, 5) and len(A) >= 6, name


# ------------------------------------------------------------------ teeth: broken solvers leave the bound
def broken_solve(A, x, bug):
    """The twin with one fault: 'race' divides the rows of column 0 that the warps after the first scale (rows >= 33)
    by sqrt(l) in place of l, as warps that read A[0][0] after thread 0's store would; 'update' drops the last trailing-update term
    of every column; 'back' substitutes back reading A[i][c] in place of L[c][i] for i < c, i.e. the input's upper
    triangle, which the device never writes."""
    m = len(A)
    upper = np.triu(A, 1).copy()       # what the device leaves above the diagonal: the input, never written
    for c in range(m):
        if not A[c, c] > 0:
            return False
        piv = A[c, c]
        l_ = np.sqrt(piv)
        A[c + 1:, c] = A[c + 1:, c] / l_
        if bug == "race" and c == 0:
            A[c + 33:, c] = A[c + 33:, c] * l_ / np.sqrt(l_)
        A[c, c] = l_
        upd = np.outer(A[c + 1:, c], A[c + 1:, c])
        if bug == "update" and c + 1 < m:
            upd[-1, -1] = 0.0
        A[c + 1:, c + 1:] = A[c + 1:, c + 1:] - upd
    xs = x.reshape(m, -1)
    for c in range(m):
        xs[c] = xs[c] / A[c, c]
        xs[c + 1:] = xs[c + 1:] - A[c + 1:, c, None] * xs[c]
    for c in range(m - 1, -1, -1):
        xs[c] = xs[c] / A[c, c]
        col = upper[:c, c] if bug == "back" else A[c, :c]
        xs[:c] = xs[:c] - col[:, None] * xs[c]
    return True


@pytest.mark.parametrize("bug", ["race", "update", "back"])
def test_broken_solvers_fail_the_bound(bug):
    rng = np.random.default_rng(9)
    A = random_spd(rng, 48, scale=3.0)          # pivots near 3, so sqrt(l) != l
    b = rng.normal(size=(48, 1))
    if bug == "race":     # at scale 50 the race's larger column makes a later pivot negative: a false failure
        Ab, xb = 50.0 * A, b.copy()
        assert twin(Ab, b)[0] and not broken_solve(Ab, xb, bug)
    A1, x1 = A.copy(), b.copy()
    assert broken_solve(A1, x1, bug)
    rs, fs = backward_ratios(A, b, A1, x1)
    if bug == "back":        # the factor is right: only the solve leaves its bound
        assert fs <= 1.0 and rs > 1e3, (rs, fs)
    else:
        assert max(rs, fs) > 1e3, (bug, rs, fs)
    # and the unbroken twin passes on the same system
    ok, L, x = twin(A, b)
    assert ok and max(backward_ratios(A, b, L, x)) <= 1.0


# ------------------------------------------------------------------ failure semantics
def failing_system(m, c, bad):
    """A = G G^T (G lower, powers of two on the diagonal, small integers below, so every step up to column c is
    exact) whose pivot at column c is `bad`; row c is uncoupled for -0.0 and NaN (those only survive uncoupled).
    -> (A, expected lower triangle after the failed call)."""
    rng = np.random.default_rng(100 * m + c)
    G = np.tril(rng.integers(-3, 4, size=(m, m)).astype(np.float64), -1) + np.diag(2.0 ** rng.integers(0, 3, m))
    couple = not (np.isnan(bad) or (bad == 0 and np.signbit(bad)))
    if not couple:
        G[c, :c] = 0.0
    A = G @ G.T
    A[c, c] = float(G[c, :c] @ G[c, :c]) + bad if couple else bad
    # the exact state after columns 0 .. c-1: L's columns, then the Schur complement of the trailing block
    want = np.tril(A).copy()
    want[:, :c] = np.tril(G)[:, :c]
    Sc = A[c:, c:] - G[c:, :c] @ G[c:, :c].T
    want[c:, c:] = np.tril(Sc)
    if not couple:
        want[c, c] = bad
    return A, want


BADS = [0.0, -0.0, -1.0, float("nan")]


@pytest.mark.parametrize("bad", BADS, ids=["zero", "negzero", "negative", "nan"])
@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_failed_pivot_returns_false_and_leaves_x(bad, where):
    m = 7
    c = {"first": 0, "middle": 3, "last": m - 1}[where]
    A, want = failing_system(m, c, bad)
    b = np.arange(1.0, 2 * m + 1).reshape(m, 2)
    A1, x1 = A.copy(), b.copy()
    assert _posed.cholesky_solve(A1, x1) is False
    assert np.array_equal(x1.view(np.uint64), b.view(np.uint64))
    got = np.tril(A1)
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), (got, want)


def test_empty_and_scalar_systems():
    A, x = np.zeros((0, 0)), np.zeros((0, 3))
    assert _posed.cholesky_solve(A, x) is True
    A, x = np.array([[4.0]]), np.array([[2.0, -6.0]])
    assert _posed.cholesky_solve(A, x) is True
    assert np.array_equal(A, [[2.0]]) and np.array_equal(x, [[0.5, -1.5]])
    for bad in BADS:
        A, x = np.array([[bad]]), np.array([[1.0]])
        assert _posed.cholesky_solve(A, x) is False and x[0, 0] == 1.0
        assert A[0, 0] == bad or (np.isnan(bad) and np.isnan(A[0, 0]))


# ------------------------------------------------------------------ the bundle adjustment's stop and failure paths
def _ba_scene(seed=41):
    d, pairs, R, t = scene(seed, V=6, n_pts=40, n_lines=8, ring=2)
    tr = TR.triangulate_tracks_host(d["keypoints"], d["klines"], pairs, ring_matches(d, pairs, torch.device("cpu")),
                                    d["K"], R, t, thresh=8, epi_thresh=8)
    return d, pairs, R, t, tr


def _ba_host(d, R, t, tr, **kw):
    return BA.bundle_adjust_host(d["keypoints"], d["klines"], d["K"], R, t, tr, **kw)


BA_STOPS = {"iters": dict(max_iters=3), "ftol": dict(max_iters=200, ftol=1e-3),
            "ftol0": dict(max_iters=400, ftol=0.0), "iters0": dict(max_iters=0)}


@pytest.mark.parametrize("case", list(BA_STOPS))
def test_ba_stop_reasons(case):
    d, pairs, R, t, tr = _ba_scene()
    o = _ba_host(d, R, t, tr, **BA_STOPS[case])
    s = o["stats"]
    h = o["history"]
    assert (np.diff(h) < 0).all()                      # every accepted step lowers the cost
    assert s["final_cost"] == h[-1] and s["accepted"] == len(h) - 1
    if case == "iters":
        assert s["stop_reason"] == BA.BA_STOP_ITERS and s["iterations"] == 3
    if case == "iters0":
        assert s["stop_reason"] == BA.BA_STOP_ITERS and s["iterations"] == 0 and s["lambda"] == BA.BA_LAMBDA0
    if case == "ftol":
        assert s["stop_reason"] == BA.BA_STOP_FTOL and s["iterations"] < 200
        assert (h[-2] - h[-1]) / h[-2] <= 1e-3
    if case == "ftol0":
        # a relative decrease is never <= 0, so the run ends when lambda passes 1e32 after the cost stops falling
        assert s["stop_reason"] == BA.BA_STOP_LAMBDA and s["lambda"] > BA.BA_LAMBDA_MAX
        assert s["lambda"] / BA.BA_REJECT <= BA.BA_LAMBDA_MAX and s["iterations"] < 400


def _behind_scene():
    """Point track k moved to 1e-3 in front of the camera of its first row, on that camera's axis: its residuals are
    huge, and the first LM steps take it behind the camera."""
    d, pairs, R, t, tr = _ba_scene(43)
    tr = dict(tr)
    P = tr["points3d"].copy()
    k = int(np.flatnonzero(tr["status_p"] == N.TRK_OK)[0])
    obs = tr["obs_p"][tr["track_off_p"][k]:tr["track_off_p"][k + 1]]
    img = int(np.searchsorted(tr["offsets_p"], obs[0], side="right") - 1)
    C = -R[img].T @ t[img]
    P[k] = C + 1e-3 * R[img][2] + 3e-4 * R[img][0]
    tr["points3d"] = P
    return d, pairs, R, t, tr


def _spy_ba(monkeypatch):
    """Record the model's cost reductions ('cost', value) and dense solves ('solve', ok) in call order."""
    calls = []
    real_bs, real_cs = BA.block_sum, BA.cholesky_solve

    def bs(terms, nt):
        out = real_bs(terms, nt)
        calls.append(("cost", float(out[0])))
        return out

    def cs(A, x):
        ok = real_cs(A, x)
        calls.append(("solve", ok))
        return ok
    monkeypatch.setattr(BA, "block_sum", bs)
    monkeypatch.setattr(BA, "cholesky_solve", cs)
    return calls


def test_ba_rejects_a_step_behind_a_camera(monkeypatch):
    """Every factorization succeeds and the candidate cost falls, yet the step is rejected: only the depth test can
    have rejected it.  lambda x 10 per rejection, nothing moves."""
    d, pairs, R, t, tr = _behind_scene()
    calls = _spy_ba(monkeypatch)
    o = _ba_host(d, R, t, tr, max_iters=3)
    s = o["stats"]
    assert calls[0][0] == "cost" and calls[1] == ("solve", True) and calls[2][0] == "cost"
    assert calls[2][1] < calls[0][1]                              # the candidate's cost fell ...
    assert s["accepted"] == 0 and s["iterations"] == 3            # ... and every step was rejected
    assert s["lambda"] == BA.BA_LAMBDA0 * BA.BA_REJECT * BA.BA_REJECT * BA.BA_REJECT
    assert s["final_cost"] == s["initial_cost"] and np.array_equal(o["R"], R) and np.array_equal(o["t"], t)


def test_ba_failed_reduced_factorization_rejects_the_step(monkeypatch):
    """A reduced camera matrix whose factorization fails (the model's solver made to fail on the second iteration):
    the camera step is zero, the step is rejected with lambda x 10, and the next iteration continues from the same
    state."""
    d, pairs, R, t, tr = _ba_scene()
    ref = _ba_host(d, R, t, tr, max_iters=1)
    real = BA.cholesky_solve
    n = [0]

    def failing(A, x):
        n[0] += 1
        return False if n[0] == 2 else real(A, x)
    monkeypatch.setattr(BA, "cholesky_solve", failing)
    o2 = _ba_host(d, R, t, tr, max_iters=2)
    s1, s2 = ref["stats"], o2["stats"]
    assert s1["accepted"] == 1 and s2["accepted"] == 1 and s2["iterations"] == 2
    assert s2["lambda"] == s1["lambda"] * BA.BA_REJECT
    assert s2["final_cost"] == s1["final_cost"]
    assert np.array_equal(o2["R"], ref["R"]) and np.array_equal(o2["points3d"], ref["points3d"])


# ------------------------------------------------------------------ the global poses' half-turn pairs
def _axis_set(flip):
    """Seven images with R = I, centres on a helix; pairs 0..9 join images 0..5 (a ring with chords), pair 10 joins
    the leaf 6 to image 0 only.  The pairs in `flip` carry the half turn diag(1, -1, -1) in place of I, so a loop
    through one of them gives Q = diag(1, -1, -1) exactly: 1 + tr Q = 0 and |cayinv| = +inf."""
    n = 7
    a = np.arange(n) * 2 * np.pi / n
    C = np.stack([4 * np.cos(a), 4 * np.sin(a), 0.5 * np.arange(n)], 1)
    pairs = np.array([(i, i + 1) for i in range(5)] + [(i, i + 2) for i in range(4)] + [(0, 5), (0, 6)], np.int64)
    P = len(pairs)
    Rp = np.tile(np.eye(3), (P, 1, 1))
    tp = np.zeros((P, 3))
    for p, (i, j) in enumerate(pairs):
        tp[p] = -(C[j] - C[i]) / np.linalg.norm(C[j] - C[i])
        if p in flip:
            Rp[p] = np.diag([1.0, -1.0, -1.0])
    return pairs, dict(R=Rp, t=tp, valid=np.ones(P, bool), n_cheirality=np.full(P, 50, np.int32)), n


def test_gp_half_turn_pair_has_an_infinite_residual():
    """A half-turn pair inside the ring: loops through it have |cayinv| = +inf exactly, its L1 weight is 1/inf = 0,
    and the IRLS still ends with finite poses: every image keeps its spanning-tree pair, whose residual is finite, so
    no Laplacian row is empty.  Infinite residuals are rotation outliers, with Geman-McClure cost 1 each."""
    pairs, rp, n = _axis_set([1])
    H = np.diag([1.0, -1.0, -1.0]).reshape(9)
    with np.errstate(invalid="ignore"):
        _, r = GPm._loop(np.eye(3).reshape(9), H, np.eye(3).reshape(9))
    assert np.isinf(r)
    o = GPm.global_poses_host(pairs, rp, n)
    reg, res, st = o["registered"], o["rot_residual"], o["edge_status"]
    assert np.isfinite(o["R"][reg]).all() and np.isfinite(o["t"][reg]).all()
    assert np.isinf(res).any()
    tan = np.tan(np.radians(5.0) / 2)
    ce = np.isfinite(res) | np.isinf(res)
    assert (st[ce & ~(res <= tan)] == GPm.GP_EDGE_ROT_OUTLIER).all()
    assert o["stats"]["rot_cost"] == float(np.isinf(res).sum())      # the finite residuals are exactly 0
    # the rotation stage ended at a rejected Geman-McClure step after the five L1 steps, not at rot_iters
    assert GPm.GP_L1_ITERS < o["stats"]["rot_iterations"] < 100


def test_gp_half_turn_leaf_takes_the_half_turn():
    """A leaf joined only by a half-turn pair: the spanning tree chains its rotation through that pair, so its residual
    is 0 (not +inf) and its Laplacian row keeps the L1 weight 1 / 1e-9; rigidity then drops it (one pair)."""
    pairs, rp, n = _axis_set([10])
    o = GPm.global_poses_host(pairs, rp, n)
    assert o["rot_residual"][10] == 0.0
    assert not o["registered"][6] and o["registered"][:6].all()
    assert o["edge_status"][10] == GPm.GP_EDGE_OUTSIDE
    assert (o["edge_status"][:10] == GPm.GP_EDGE_INLIER).all()


# ------------------------------------------------------------------ on the GPU
DEV = torch.device("cuda", 0)


def hook(A, b, shared, ld=None):
    """ltr_debug_cholesky_solve on systems A [n, m, m] (embedded at leading dimension ld), b [n, m, k] -> (L [n, m, m],
    x, ok) as host arrays."""
    n, m = A.shape[:2]
    k = b.shape[2]
    ld = m if ld is None else ld
    Ad = np.zeros((n, m, ld))
    Ad[:, :, :m] = A
    Ad[:, :, m:] = 7.0              # past the matrix: must stay as it is
    At = torch.from_numpy(Ad).to(DEV)
    xt = torch.from_numpy(np.ascontiguousarray(b)).to(DEV)
    ok = torch.zeros(max(n, 1), dtype=torch.uint8, device=DEV)
    rc = N.load().ltr_debug_cholesky_solve(At.data_ptr(), n, m, ld, xt.data_ptr(), k, int(shared), ok.data_ptr(),
                                           DEV.index, None)
    N.check(rc, "ltr_debug_cholesky_solve")
    torch.cuda.synchronize()
    Ah = At.cpu().numpy()
    assert (Ah[:, :, m:] == 7.0).all()
    return Ah[:, :, :m], xt.cpu().numpy(), ok.cpu().numpy()[:n].astype(bool)


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def assert_hook_matches_twin(A, b, shared, ld=None):
    L, x, ok = hook(A, b, shared, ld)
    for s in range(len(A)):
        ok_t, Lt, xt = twin(A[s], b[s])
        assert ok[s] == ok_t, s
        # the device never writes the upper triangle; the twin's square trailing update does
        assert np.array_equal(_bits(np.tril(L[s])), _bits(np.tril(Lt))), s
        assert np.array_equal(_bits(np.triu(L[s], 1)), _bits(np.triu(A[s], 1))), s
        assert np.array_equal(_bits(x[s]), _bits(xt)), s
    return L, x, ok


@pytest.mark.gpu
def test_gpu_hook_matches_twin_on_the_cpu_matrices():
    worst = 0.0
    for name, A, b in CASES:
        m = len(A)
        for shared in ((0, 1) if m <= 127 else (0,)):
            L, x, ok = assert_hook_matches_twin(A[None], b[None], shared)
            assert ok[0], name
        worst = max(worst, *backward_ratios(A, b, L[0], x[0]))
    assert worst <= 1.0
    print(f"worst backward-error ratio on the device: {worst:.3g}")


SHARED_M = [1, 2, 31, 32, 33, 63, 64, 65, 126, 127]
GLOBAL_M = [128, 255, 256, 381, 511, 512, 762, 1023, 1024]


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 3, 6])
def test_gpu_hook_shared(k):
    rng = np.random.default_rng(k)
    for m in SHARED_M:
        A = np.stack([random_spd(rng, m, 30.0), graded(rng, m)])
        b = rng.normal(size=(2, m, k))
        assert assert_hook_matches_twin(A, b, 1)[2].all(), m


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 3, 6])
def test_gpu_hook_global(k):
    rng = np.random.default_rng(10 + k)
    for m in GLOBAL_M:
        A = random_spd(rng, m, 30.0)[None]
        b = rng.normal(size=(1, m, k))
        for ld in sorted({m, 6 * 128} - {x for x in (6 * 128,) if x < m}):
            assert assert_hook_matches_twin(A, b, 0, ld)[2].all(), (m, ld)


@pytest.mark.gpu
def test_gpu_hook_failures_and_refusals():
    for shared in (0, 1):
        for where in ("first", "middle", "last"):
            for bad in BADS:
                c = {"first": 0, "middle": 3, "last": 6}[where]
                A, want = failing_system(7, c, bad)
                b = np.arange(1.0, 15.0).reshape(1, 7, 2)
                L, x, ok = assert_hook_matches_twin(A[None], b, shared)
                assert not ok[0] and np.array_equal(_bits(x), _bits(b))
                assert np.array_equal(_bits(np.tril(L[0])), _bits(want))
        for bad in BADS:
            assert_hook_matches_twin(np.array([[[bad]]]), np.ones((1, 1, 1)), shared)
        assert assert_hook_matches_twin(np.array([[[4.0]]]), np.ones((1, 1, 3)), shared)[2].all()
        L, x, ok = hook(np.zeros((1, 0, 0)), np.zeros((1, 0, 1)), shared)
        assert ok.all()
    lib = N.load()
    z = torch.zeros(1024 * 1024, dtype=torch.float64, device=DEV)
    o = torch.zeros(1, dtype=torch.uint8, device=DEV)
    for m, ld, k, sh in ((-1, 4, 1, 0), (1025, 1025, 1, 0), (4, 4, 0, 0), (4, 4, 7, 0), (4, 3, 1, 0), (128, 128, 1, 1),
                         (4, 4, 1, 2)):
        assert lib.ltr_debug_cholesky_solve(z.data_ptr(), 1, m, ld, z.data_ptr(), k, sh, o.data_ptr(), 0,
                                            None) == LTR_E_INVALID, (m, ld, k, sh)
    assert lib.ltr_debug_cholesky_solve(None, 1, 4, 4, z.data_ptr(), 1, 0, o.data_ptr(), 0, None) == LTR_E_INVALID


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["iters", "ftol", "ftol0", "behind"])
def test_gpu_ba_edge_scenes_match_the_model(case):
    if case == "behind":
        d, pairs, R, t, tr = _behind_scene()
        kw = dict(max_iters=6)
    else:
        d, pairs, R, t, tr = _ba_scene()
        kw = BA_STOPS[case]
    res = ring_matches(d, pairs, DEV)
    trk = TR.triangulate_tracks(d["keypoints"], d["klines"], pairs, res, d["K"], R, t, thresh=8, epi_thresh=8)
    if case == "behind":
        trk = dataclasses.replace(trk, points3d=torch.from_numpy(tr["points3d"]).to(DEV))
    out = BA.bundle_adjust(d["keypoints"], d["klines"], d["K"], R, t, trk, **kw)
    host = BA.bundle_adjust_host(d["keypoints"], d["klines"], d["K"], R, t, trk, **kw)
    _ba_same(out, host)
    want = {"iters": BA.BA_STOP_ITERS, "ftol": BA.BA_STOP_FTOL, "ftol0": BA.BA_STOP_LAMBDA}.get(case)
    st = out.stats_dict()
    if want is not None:
        assert st["stop_reason"] == want
    if case == "behind":     # the device rejected every step on the depth test, as the model does
        lam = BA.BA_LAMBDA0
        for _ in range(6):
            lam = lam * BA.BA_REJECT
        assert st["accepted"] == 0 and st["iterations"] == 6 and st["lambda"] == lam
        assert st["final_cost"] == st["initial_cost"]
        assert torch.equal(out.R.cpu(), torch.from_numpy(R)) and torch.equal(out.t.cpu(), torch.from_numpy(t))


@pytest.mark.gpu
@pytest.mark.parametrize("flip", [[1], [10], [1, 10]])
def test_gpu_gp_half_turn_scenes_match_the_model(flip):
    pairs, rp, n = _axis_set(flip)
    want = GPm.global_poses_host(pairs, rp, n)
    dp = {k: torch.as_tensor(v).to(DEV) for k, v in rp.items()}
    got = GPm.global_poses(pairs, dp, n)
    torch.cuda.synchronize()
    for k in ("R", "t", "edge_status", "support", "rot_residual", "dir_cos"):
        g = getattr(got, k).cpu().numpy()
        assert _gp_same(g, want[k].astype(g.dtype)), k
    assert np.array_equal(got.registered.cpu().numpy(), want["registered"])
    s = got.stats_dict()
    for k in GPm.STATS:
        assert s[k] == want["stats"][k] or (np.isinf(s[k]) and np.isinf(want["stats"][k])), (k, s[k], want["stats"][k])


# ------------------------------------------------------------------ triangulation: the angle rule and the 1-D refit
TRI_K = syn.DEFAULT_K


def _tri_scene(X, c1, R1=np.eye(3), nudge=None):
    """Two views of the world points X [n, 3] (camera 0 at the origin looking down +z, camera 1 with rotation R1 and
    centre c1), points only, every row matched to itself; nudge(kps) may edit the float32 keypoints."""
    Rs = np.stack([np.eye(3), R1])
    ts = np.stack([np.zeros(3), -R1 @ np.asarray(c1, np.float64)])
    kps = []
    for R, t in zip(Rs, ts):
        q = X @ R.T + t
        kps.append((q[:, :2] / q[:, 2:] * TRI_K[0, 0] + TRI_K[:2, 2]).astype(np.float32))
    if nudge is not None:
        nudge(kps)
    kls = [np.zeros((0, 2, 2), np.float32)] * 2
    pairs = np.array([[0, 1]])
    return kps, kls, pairs, Rs, ts


def _tri_res(kps, kls, pairs, device="cpu"):
    n = len(kps[0])
    mp = [np.arange(n, dtype=np.int32)]
    ml = [np.zeros(0, np.int32)]
    off = np.array([0, n], np.int32)
    mpt = torch.from_numpy(mp[0]).to(device)
    mlt = torch.from_numpy(ml[0]).to(device)
    z = torch.zeros(1, dtype=torch.int32, device=device)
    from linetr_b200.engine import ImagePairMatches
    return ImagePairMatches(mlt, mlt.float(), z, np.array([0, 0], np.int32), mpt, mpt.float(), z, off,
                            [kls[0]], [kls[1]], [kps[0]], [kps[1]])


def _tri_host(scene_, **kw):
    kps, kls, pairs, Rs, ts = scene_
    return TRI.triangulate_host(kps, kls, pairs, _tri_res(kps, kls, pairs), TRI_K, Rs, ts, **kw)


def _mp_depth(scene_, row, s0):
    """The least-squares depth of anchor 0's keypoint `row` over its one observation, at 50 digits from the float
    inputs: the root of d/ds (ex^2 + ey^2) nearest the model's depth s0."""
    kps, _, _, Rs, ts = scene_
    with mpmath.workdps(50):
        mpf = mpmath.mpf
        fx, fy, cx, cy = (mpf(float(v)) for v in (TRI_K[0, 0], TRI_K[1, 1], TRI_K[0, 2], TRI_K[1, 2]))
        x, y = (mpf(float(v)) for v in kps[0][row])
        u, v = (mpf(float(w)) for w in kps[1][row])
        r = mpmath.matrix([(x - cx) / fx, (y - cy) / fy, 1])           # R_0 = I, C_0 = 0
        R1 = mpmath.matrix(Rs[1].tolist())
        t1 = mpmath.matrix(ts[1].tolist())
        B = R1 * r

        def cost(s):
            P = t1 + s * B
            return (fx * P[0] / P[2] + cx - u) ** 2 + (fy * P[1] / P[2] + cy - v) ** 2
        return mpmath.findroot(lambda s: mpmath.diff(cost, s), mpf(float(s0)))


def _angle_scene():
    return _tri_scene(np.array([[0.3, -0.2, 6.0]]), [0.2, 0.05, 0.0])


def _angle_boundary(sc):
    """The largest min_angle (in float64 steps) at which the row's candidate passes the angle rule."""
    kept = lambda a: _tri_host(sc, min_angle=a, thresh=50.0)["n_views_p"][0] == 2
    lo, hi = 0.0, 10.0
    assert kept(lo) and not kept(hi)
    while np.nextafter(lo, np.inf) < hi:
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if kept(mid) else (lo, mid)
    return lo, kept


def test_tri_min_angle_boundary():
    """The angle rule at its boundary: kept at the boundary min_angle and one ulp below, rejected one ulp above; the
    boundary lies at the row's true triangulation angle (50 digits, from the scene's exact points) to the float32
    keypoints' 1e-6."""
    sc = _angle_scene()
    lo, kept = _angle_boundary(sc)
    assert kept(lo) and kept(np.nextafter(lo, -np.inf)) and not kept(np.nextafter(lo, np.inf))
    with mpmath.workdps(50):
        C1 = mpmath.matrix([0.2, 0.05, 0.0])
        P = mpmath.matrix([0.3, -0.2, 6.0])
        b = P - C1
        ang = mpmath.degrees(mpmath.acos(sum(P[i] * b[i] for i in range(3)) / (mpmath.norm(P) * mpmath.norm(b))))
    assert abs(float(ang) - lo) <= 1e-6 * lo, (float(ang), lo)


def test_tri_far_points_against_mpmath():
    """Points at 1e6 depth (baseline 1, angles of 6e-5 degrees): with min_angle 0 every row is kept and its refit
    depth is the 50-digit least-squares depth of its own float inputs to 1e-6."""
    rng = np.random.default_rng(3)
    X = np.c_[rng.uniform(-2e5, 2e5, (6, 2)), rng.uniform(0.9e6, 1.1e6, 6)]
    sc = _tri_scene(X, [1.0, 0.0, 0.0])
    h = _tri_host(sc, min_angle=0.0, thresh=1e3)
    assert (h["n_views_p"][:6] == 2).all()
    for k in range(6):
        s = h["depth_p"][k]
        want = _mp_depth(sc, k, s)
        assert abs(s - float(want)) <= 1e-6 * float(want), (k, s, float(want))


def _epipole_scene(step):
    """Camera 1 directly behind camera 0 on its axis (centre (0, 0, -2)), so camera 0's centre projects to camera 1's
    principal point.  Row 0's partner keypoint is put exactly on that epipole and then moved `step` float32 ulps in x:
    its candidate depth is exactly 0 at step 0 and a tiny depth of either sign one ulp away."""
    X = np.array([[0.4, 0.1, 5.0], [0.5, -0.3, 7.0]])

    def nudge(kps):
        e = np.float32(TRI_K[0, 2])
        kps[1][0] = [e, np.float32(TRI_K[1, 2])]
        for _ in range(abs(step)):
            kps[1][0, 0] = np.nextafter(kps[1][0, 0], np.float32(np.inf if step > 0 else -np.inf))
    return _tri_scene(X, [0.0, 0.0, -2.0], nudge=nudge)


@pytest.mark.parametrize("step", [-1, 0, 1])
def test_tri_depth_zero_at_the_epipole(step):
    sc = _epipole_scene(step)
    h = _tri_host(sc, min_angle=0.0, thresh=4.0)
    o = TRI._point_terms
    # the candidate depth itself, as the model computes it
    kps, _, _, Rs, ts = sc
    C, cams = TRI._cameras(_posed.check_set(kps, [np.zeros((0, 2, 2), np.float32)] * 2, np.array([[0, 1]]),
                                            _tri_res(kps, sc[1], sc[2]), TRI_K, Rs, ts, "t"), 0)
    r = _posed.ray(Rs[0].reshape(9), TRI_K[0, 0], TRI_K[1, 1], TRI_K[0, 2], TRI_K[1, 2],
                   kps[0][:, 0].astype(np.float64), kps[0][:, 1].astype(np.float64))
    T_ = o(cams[0], r, kps[1].astype(np.float64))
    s = -((T_["ax"] * T_["bx"] + T_["ay"] * T_["by"]) / (T_["bx"] * T_["bx"] + T_["by"] * T_["by"]))
    if step == 0:
        assert s[0] == 0.0
    else:
        assert s[0] != 0.0 and abs(s[0]) < 1e-3
    # a depth that is not > 0 is no candidate, so the row has no estimate; one ulp to the other side gives a tiny
    # positive depth, which min_angle 0 keeps, refitted to the 50-digit least-squares depth
    if step <= 0:
        assert not s[0] > 0 and h["n_views_p"][0] == 0 and np.isnan(h["winner_p"][0]) and np.isnan(h["points3d"][0]).all()
    else:
        assert 0 < s[0] < 1e-5 and h["n_views_p"][0] == 2 and h["refit_p"][0]
        want = float(_mp_depth(sc, 0, h["depth_p"][0]))
        assert abs(h["depth_p"][0] - want) <= 1e-6 * want, (h["depth_p"][0], want)
    assert h["n_views_p"][1] == 2


def test_tri_refit_guards():
    """The refit's two guards, on its own terms (alpha, beta, gamma, delta): a step where J^T J is not > 0 (every
    supporter's J = (beta - r delta) / den is 0) and a step that is not finite (den = 0) leave the depth as it was and
    stop the refit; an ordinary system converges to the 50-digit least-squares depth."""
    one = np.uint64(1)
    s0 = np.array([2.0, 2.0, 3.0])
    act = np.ones(3, bool)
    # row 0: r = (a + s b) / (g + s d) with b = r d for every s: a = 2, b = 1, g = 2, d = 1 -> r = 1, J = 0
    # row 1: den = g + s d = 0 at s = 2: g = -2, d = 1
    # row 2: two ordinary terms
    terms = [[(np.array([2.0, 1.0, 0.3]), np.array([1.0, 1.0, -0.2]), np.array([2.0, -2.0, 1.0]),
               np.array([1.0, 1.0, 0.05])),
              (np.array([2.0, 1.0, -0.1]), np.array([1.0, 1.0, 0.1]), np.array([2.0, -2.0, 1.0]),
               np.array([1.0, 1.0, 0.02]))]]
    with np.errstate(all="ignore"):      # as triangulate_host runs it: the guarded rows divide by 0
        s = TRI._gn(terms, np.array([one, one, one]), s0, act)
    assert s[0] == 2.0 and s[1] == 2.0
    with mpmath.workdps(50):
        mpf = mpmath.mpf
        f = lambda z: sum(((mpf(a[2]) + z * mpf(b[2])) / (mpf(g[2]) + z * mpf(d[2]))) ** 2 for a, b, g, d in terms[0])
        want = mpmath.findroot(lambda z: mpmath.diff(f, z), mpf(3.0))
    assert abs(s[2] - float(want)) <= 1e-9 * abs(float(want)), (s[2], float(want))


@pytest.mark.gpu
def test_gpu_triangulation_edge_scenes_match_the_model():
    """The angle boundary (at it and one ulp either side), points at 1e6 depth and the epipole rows (depth 0 and one
    float32 ulp either side) through `triangulate`, bit for bit against `triangulate_host`."""
    sc = _angle_scene()
    lo, _ = _angle_boundary(sc)
    runs = [(sc, dict(min_angle=a, thresh=50.0)) for a in (np.nextafter(lo, -np.inf), lo, np.nextafter(lo, np.inf))]
    rng = np.random.default_rng(3)
    X = np.c_[rng.uniform(-2e5, 2e5, (6, 2)), rng.uniform(0.9e6, 1.1e6, 6)]
    runs.append((_tri_scene(X, [1.0, 0.0, 0.0]), dict(min_angle=0.0, thresh=1e3)))
    runs += [(_epipole_scene(step), dict(min_angle=0.0, thresh=4.0)) for step in (-1, 0, 1)]
    for i, (sc_, kw) in enumerate(runs):
        kps, kls, pairs, Rs, ts = sc_
        h = _tri_host(sc_, **kw)
        g = TRI.triangulate(kps, kls, pairs, _tri_res(kps, kls, pairs, DEV), TRI_K, Rs, ts, **kw)
        for f in ("points3d", "lines3d", "n_views_p", "n_views_l"):
            a, b = getattr(g, f).cpu().numpy(), h[f]
            assert a.shape == b.shape and a.tobytes() == b.astype(a.dtype).tobytes(), (i, f)
    assert [h_["n_views_p"][0] for h_ in (_tri_host(r[0], **r[1]) for r in runs[:3])] == [2, 2, 0]
