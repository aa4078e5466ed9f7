"""The two RANSAC estimators (`ltr_homography`, `ltr_essential`) at their edges, against exact and host references.

- The relative-pose estimator's fp64 root finder (`ess_roots` through `ltr_debug_sturm_roots`) and its host model
  `geometry.sturm_roots` against an exact Sturm count and exact bisection in rational arithmetic (`fractions`), on
  dense, sparse, degree-dropping, multiple-root, out-of-bound, badly scaled and non-finite polynomials.
- The five-point solver (`ess_solve` through `ltr_debug_essential_solve`) against `geometry.essential_solutions` bit
  for bit, on >= 100 000 samples and on structured ones, and against exact synthetic scenes.
- Every hypothesis end to end: the sample hash mixes in the pair index, so P copies of one correspondence set run with
  n_hypotheses=1 evaluate P different hypotheses, each compared with the host model run with pair=p.
- Degenerate inputs, minimal sets, hypothesis counts around the 128-thread CTA, staging filled exactly, a residual
  exactly at thresh^2, projections with |w| <= FLT_EPSILON, large and tiny coordinates and unusual intrinsics, each
  compared with the host model on the GPU."""
import ctypes as C
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

from linetr_b200 import _native as N, geometry as G, synthetic as syn
from tests.test_homography import _host_pair as _hg_host_pair, _matches as _hg_matches
from tests.test_pose import _host_pair as _es_host_pair, _matches as _es_matches, _ragged_cases as _es_ragged_cases

DEV = torch.device("cuda", 0)
K = syn.DEFAULT_K
U = 2.0 ** -53                        # unit roundoff of fp64
# Horner's rule of degree n <= 10 on the normalised coefficients c_i / m: each c_i / m carries one rounding (u), the
# evaluation 2n more (Higham, Accuracy and Stability, eq. 5.7: |fl(p(x)) - p(x)| <= gamma_2n sum |c_i||x|^i).  So the
# computed sign of p(x) can be wrong only where |p(x)| <= gamma sum |c_i||x|^i with gamma = gamma_21 = 21u / (1 - 21u),
# which near a simple root r is |x - r| <= gamma sum |c_i||r|^i / |p'(r)| to first order.
GAMMA = 21 * U / (1 - 21 * U)
SEPARATION = 1e-3                     # relative gap between adjacent simple roots for count and roots to be required


# ------------------------------------------------------------------ exact reference (rational arithmetic)
def _exact(c):
    """fp64 coefficients (ascending) -> exact rationals without leading zeros."""
    p = [Fraction(float(x)) for x in c]
    while len(p) > 1 and p[-1] == 0:
        p.pop()
    return p


def _ev(p, x):
    v = Fraction(0)
    for a in reversed(p):
        v = v * x + a
    return v


def _rem(a, b):
    a = list(a)
    while len(a) >= len(b) and any(a):
        q = a[-1] / b[-1]
        off = len(a) - len(b)
        for i, bi in enumerate(b):
            a[off + i] -= q * bi
        a.pop()
    while len(a) > 1 and a[-1] == 0:
        a.pop()
    return a


def _quo(a, b):
    """Quotient of the exact division a / b."""
    a, q = list(a), [Fraction(0)] * max(len(a) - len(b) + 1, 1)
    while len(a) >= len(b):
        c = a[-1] / b[-1]
        off = len(a) - len(b)
        q[off] = c
        for i, bi in enumerate(b):
            a[off + i] -= c * bi
        a.pop()
    assert not any(a)
    return q


def _sturm(p):
    """The exact Sturm chain of p (degree >= 1), divided by its last member (the gcd of p and p') so that it also
    counts correctly at a multiple root."""
    chain = [p, [i * a for i, a in enumerate(p)][1:]]
    while len(chain[-1]) > 1:
        r = _rem(chain[-2], chain[-1])
        if not any(r):
            break
        chain.append([-a for a in r])
    g = chain[-1]
    return [_quo(c, g) for c in chain] if len(g) > 1 else chain


def _var(chain, x):
    s = [v for v in (_ev(c, x) for c in chain) if v != 0]
    return sum((a > 0) != (b > 0) for a, b in zip(s, s[1:]))


def exact_roots(c, B=G.ESS_ROOT_BOUND):
    """Distinct real roots of the fp64 polynomial c in (-B, B]: (count, [(lo, hi)] brackets of each root, ascending,
    narrower than 1/8 ulp of the root or exactly the root as (r, r)).  None for a constant or non-finite c."""
    if not all(math.isfinite(x) for x in c):
        return None
    p = _exact(c)
    if len(p) < 2:
        return None
    chain = _sturm(p)
    lo0, hi0 = Fraction(-B), Fraction(B)
    v_lo = _var(chain, lo0)
    count = v_lo - _var(chain, hi0)
    brackets = []
    stack = [(lo0, hi0, count)]
    while stack:                      # isolate: (lo, hi] with one root each
        lo, hi, n = stack.pop()
        if n == 1:
            brackets.append((lo, hi))
        elif n > 1:
            mid = (lo + hi) / 2
            nl = _var(chain, lo) - _var(chain, mid)
            stack += [(lo, mid, nl), (mid, hi, n - nl)]
    out = []
    for lo, hi in sorted(brackets):
        if _ev(p, hi) == 0:
            out.append((hi, hi))
            continue
        # refine on the sign of the square-free part's Sturm count (works for multiple roots too)
        while hi - lo > abs(hi) * Fraction(2) ** -56 and hi - lo > Fraction(2) ** -1100:
            mid = (lo + hi) / 2
            if _var(chain, lo) - _var(chain, mid) == 1:
                hi = mid
            else:
                lo = mid
            if _ev(p, hi) == 0:
                lo = hi
                break
        out.append((lo, hi))
    return count, out


def _count_with_multiplicity(c, B=G.ESS_ROOT_BOUND):
    """Real roots of c in (-B, B] counted with multiplicity: distinct roots of p, of gcd(p, p'), of its gcd, ..."""
    p, total = _exact(c), 0
    while len(p) > 1:
        chain = [p, [i * a for i, a in enumerate(p)][1:]]
        while len(chain[-1]) > 1:
            r = _rem(chain[-2], chain[-1])
            if not any(r):
                break
            chain.append([-a for a in r])
        sq = _sturm(p)
        total += _var(sq, Fraction(-B)) - _var(sq, Fraction(B))
        p = chain[-1]
    return total


def _band(c, r, B):
    """Where the computed root of a simple root r may lie: the Horner band, one ulp and the width of the bisection's
    bracket after ESS_BISECT_STEPS steps from [-B, B]."""
    p = _exact(c)
    dp = [i * a for i, a in enumerate(p)][1:]
    rf = float(r)
    s = sum(abs(float(a)) * abs(rf) ** i for i, a in enumerate(p))
    return GAMMA * s / abs(float(_ev(dp, r))) + math.ulp(rf) + 2 * B * 2.0 ** -G.ESS_BISECT_STEPS


def _cauchy(c):
    """The kernels' search bound B for c (ascending fp64, finite, degree >= 1)."""
    c = np.asarray(c, dtype=np.float64)
    s = c / np.abs(c).max()
    n = int(np.flatnonzero(s)[-1])
    return min(max([1.0] + [abs(s[i] / s[n]) + 1.0 for i in range(n)]), G.ESS_ROOT_BOUND)


# ------------------------------------------------------------------ the polynomial cases
def _from_roots(real, pairs=(), scale=1.0, degree=10):
    """Ascending fp64 coefficients [11] of scale * prod (z - r) * prod (z^2 - 2 a z + a^2 + b^2), zero-padded."""
    poly = np.array([1.0])
    for r in real:
        poly = np.convolve(poly, [1.0, -r])
    for a, b in pairs:
        poly = np.convolve(poly, [1.0, -2 * a, a * a + b * b])
    assert len(poly) == degree + 1
    out = np.zeros(11)
    out[:degree + 1] = poly[::-1] * scale
    return out


def _asc(desc):
    """Descending coefficients -> ascending [11]."""
    out = np.zeros(11)
    out[:len(desc)] = np.asarray(desc, dtype=np.float64)[::-1]
    return out


def _dense_cases():
    """Dense polynomials with 0 to 10 well-separated real roots, the rest in complex pairs: degree 10 for an even
    number of real roots, degree 9 (p[10] = 0) for an odd one."""
    cases = []
    for n_real in range(11):
        for s in range(3):
            rng = np.random.default_rng(100 * n_real + s)
            while True:
                real = np.sort(rng.uniform(-3, 3, n_real))
                if n_real < 2 or np.diff(real).min() > 0.2:
                    break
            pairs = [(rng.uniform(-2, 2), rng.uniform(0.3, 2)) for _ in range((10 - n_real) // 2)]
            deg = 10 - n_real % 2
            cases.append((f"dense{deg}_{n_real}_{s}", _from_roots(real, pairs, rng.uniform(0.5, 2.0) * (-1) ** s, deg)))
    return cases


def _sparse_cases():
    """Sparse, even, odd and two-term polynomials: their Sturm chains drop degree by more than one."""
    return [("z10-5z2+1", _asc([1, 0, 0, 0, 0, 0, 0, 0, -5, 0, 1])),
            ("z10-3z+0.5", _asc([1, 0, 0, 0, 0, 0, 0, 0, 0, -3, 0.5])),
            ("z10-1", _asc([1, 0, 0, 0, 0, 0, 0, 0, 0, 0, -1])),
            ("even", _asc([1, 0, -3, 0, 0, 0, 2, 0, 0, 0, -0.25])),
            ("odd", _asc([1, 0, 0, 0, -4, 0, 0, 0, 1, 0])),
            ("z10-2", _asc([1, 0, 0, 0, 0, 0, 0, 0, 0, 0, -2])),
            ("z7+3", _asc([1, 0, 0, 0, 0, 0, 0, 3])),
            ("2z9-z2-1", _asc([2, 0, 0, 0, 0, 0, 0, -1, 0, -1]))]


def _degree_drop_cases():
    """p[10] = 0: degree 9, 5 and 1."""
    rng = np.random.default_rng(7)
    return [("deg9", _from_roots(np.linspace(-2.5, 2.2, 9), (), 1.5, degree=9)),
            ("deg5", _from_roots([-1.5, 0.25, 2.0], [(0.5, 1.0)], -0.75, degree=5)),
            ("deg1", _asc([3.0, -1.5])),
            ("deg9_dense", _from_roots(np.sort(rng.uniform(-3, 3, 5)) + np.arange(5) * 0.3, [(0.1, 1.2), (-1, 0.5)],
                                       degree=9))]


CPLX = [(0.0, 1.0), (0.5, 1.5), (1.0, 2.0)]     # three distinct complex pairs


def _edge_cases():
    """Roots at 0 and on the first bisection midpoints, near the search bound, and badly scaled coefficients."""
    B = G.ESS_ROOT_BOUND
    return [("root0", _from_roots([0.0, -1.25, 0.5, 2.0], [(0.3, 0.7), (-1, 1), (2, 0.5)])),
            ("z3-z", _asc([1, 0, -1, 0])),                     # B = 2: roots 0, -1, 1 are midpoints
            ("z3-2z2-3z", _asc([1, -2, -3, 0])),               # B = 4: roots -1 (-4 .. 0), 0, 3 (2 .. 4)
            ("bound_in", _from_roots([B * (1 - 1e-6), 1.0, -2.0, 0.5], CPLX, 1e-30)),
            ("bound_out", _from_roots([B * (1 + 1e-6), 1.0, -2.0, 0.5], CPLX, 1e-30)),
            ("bound_both", _from_roots([-B * (1 + 1e-6), B * (1 - 1e-6), 3.0, -0.5], CPLX, 1e-40)),
            ("scale_1e200", _from_roots([-1.0, 0.5, 2.0, -2.5], CPLX, 1e200)),
            ("scale_1e-200", _from_roots([-1.0, 0.5, 2.0, -2.5], CPLX, 1e-200)),
            ("span_1e200", _asc([1e-200, 0, 0, 0, 0, 0, 0, 0, 0, 1, -1])),
            ("span_underflow", _asc([1e-200, 0, 0, 0, 0, 0, 0, 0, 0, 1e200, -1e200])),   # p[10] / max|p| underflows
            ("span_1e-200", _asc([1, 0, 0, 0, 0, 0, 0, 0, 0, 1e-200, -1e-200]))]


def _multiple_root_cases():
    """Double and triple roots and clusters 1e-6 apart: only the count is checked (see _check_counts_and_roots), not
    the roots.  A root of multiplicity k moves by about (Horner error)^(1/k) under rounding, and roots 1e-6 apart are
    closer than SEPARATION, so the first-order band around a simple root does not bound where the bisection ends."""
    return [("double", _from_roots([1.0, 1.0, -2.0, 0.5], [(0, 1), (1, 1), (-1, 2)])),
            ("double_z10-2z9+z8", _asc([1, -2, 1, 0, 0, 0, 0, 0, 0, 0, 0])),
            ("triple", _from_roots([0.5, 0.5, 0.5, -1.0, 3.0], [(0, 1)], degree=7)),
            ("two_doubles", _from_roots([-1.5, -1.5, 2.0, 2.0], [(0, 1), (1, 2), (-1, 1)])),
            ("cluster", _from_roots([1.0, 1.0 + 1e-6, -0.5, 2.5], [(0, 1), (1, 1), (-2, 1)])),
            ("cluster3", _from_roots([0.25, 0.25 + 1e-6, 0.25 + 2e-6, -3.0], [(0, 1), (2, 1), (-1, 1)]))]


def _nonfinite_cases():
    out = []
    for name, v in (("nan", np.nan), ("inf", np.inf), ("-inf", -np.inf)):
        for i in (0, 4, 10):
            c = _from_roots([1.0, -1.0], [(0, 1)] * 4)
            c[i] = v
            out.append((f"{name}@{i}", c))
    return out


SIMPLE = _dense_cases() + _sparse_cases() + _degree_drop_cases() + _edge_cases()
MULTIPLE = _multiple_root_cases()
EXACT_IN_FP64 = {"double_z10-2z9+z8"}
NONFINITE = _nonfinite_cases()
ALL_POLYS = SIMPLE + MULTIPLE + NONFINITE


def _check_counts_and_roots(name, c, roots, count, exact):
    """The root finder's output for c against the exact reference."""
    if exact is None:
        assert count == 0 and np.isnan(roots).all(), name
        return
    n, brackets = exact
    if any(name == m for m, _ in MULTIPLE):
        # A multiple root makes the remainder at the gcd step zero only in exact arithmetic.  In fp64 that remainder
        # is a rounding residue unless every division on the way is exact, the chain goes on, and it counts the
        # distinct real roots of a polynomial within rounding of p: a root of multiplicity m then counts from 1 to m
        # times (m when it splits into m nearby simple roots).  Dyadic chains (z^8 (z - 1)^2) keep the exact count.
        assert n <= count <= _count_with_multiplicity(c), (name, count, n)
        if name in EXACT_IN_FP64:
            assert count == n, (name, count, n)
        assert np.isnan(roots[count:]).all() and not np.isnan(roots[:count]).any(), name
        return
    assert count == n, (name, count, n)
    assert np.isnan(roots[n:]).all(), name
    B = _cauchy(c)
    rs = [(lo + hi) / 2 for lo, hi in brackets]
    assert all(abs(b - a) > SEPARATION * max(abs(a), abs(b)) for a, b in zip(rs, rs[1:])), name   # precondition
    for i, r in enumerate(rs):
        err = abs(Fraction(float(roots[i])) - r)
        assert float(err) <= _band(c, r, B), (name, i, float(roots[i]), float(r), float(err), _band(c, r, B))


_EXACT = {}


def _exact_of(name, c):
    if name not in _EXACT:
        _EXACT[name] = exact_roots(c)
    return _EXACT[name]


# ------------------------------------------------------------------ CPU: the host model against the exact reference
def test_exact_reference_on_known_roots():
    """The exact reference itself: roots known in closed form."""
    n, br = exact_roots(_asc([1, 0, -1, 0]))               # z^3 - z
    assert n == 3 and all(lo <= r <= hi and hi - lo < Fraction(2) ** -50 for (lo, hi), r in zip(br, (-1, 0, 1)))
    n, br = exact_roots(_asc([1, 0, 0, 0, 0, 0, 0, 0, 0, 0, -2]))
    assert n == 2 and abs(float(br[1][0]) - 2 ** 0.1) <= math.ulp(2 ** 0.1)
    assert exact_roots(_asc([1, -2, 1]))[0] == 1           # (z - 1)^2: distinct roots
    assert exact_roots(_asc([1, 0, 1]))[0] == 0
    assert exact_roots(_asc([1, -2e8]))[0] == 0 and exact_roots(_asc([1, -1e8]))[0] == 1   # (-B, B]
    assert exact_roots([np.nan] + [1.0] * 10) is None and exact_roots(_asc([3.0])) is None


@pytest.mark.parametrize("name,c", ALL_POLYS, ids=[n for n, _ in ALL_POLYS])
def test_host_sturm_roots_against_exact(name, c):
    roots, count = G.sturm_roots(c[None])
    _check_counts_and_roots(name, c, roots[0], int(count[0]), _exact_of(name, c))


def test_host_sturm_roots_on_sparse_examples():
    """The polynomials a chain that assumed one degree less per member got wrong: z^10 - 5z^2 + 1 has 4 real roots
    (+-0.447, +-1.200), z^10 - 3z + 0.5 has 2 (0.167, 1.110)."""
    roots, count = G.sturm_roots(np.stack([_asc([1, 0, 0, 0, 0, 0, 0, 0, -5, 0, 1]),
                                           _asc([1, 0, 0, 0, 0, 0, 0, 0, 0, -3, 0.5])]))
    assert count.tolist() == [4, 2]
    assert np.allclose(roots[0, :4], [-1.2002, -0.4473, 0.4473, 1.2002], atol=1e-4)
    assert np.allclose(roots[1, :2], [0.1667, 1.1096], atol=1e-4)


def test_host_sturm_roots_batch_equals_single():
    """Rows of one batch do not interact: the batched model gives each row's single-row bits."""
    P = np.stack([c for _, c in ALL_POLYS])
    rb, cb = G.sturm_roots(P)
    for i, c in enumerate(P):
        r1, c1 = G.sturm_roots(c[None])
        assert c1[0] == cb[i] and np.array_equal(r1[0], rb[i], equal_nan=True), ALL_POLYS[i][0]


# ------------------------------------------------------------------ GPU hooks
def _bits(a):
    """fp64 bit patterns, every NaN as one pattern."""
    a = np.asarray(a, dtype=np.float64)
    return np.where(np.isnan(a), -1, a.view(np.int64))


def _sturm_gpu(P):
    P = torch.as_tensor(np.ascontiguousarray(P, dtype=np.float64), device=DEV)
    n = P.shape[0]
    roots = torch.empty((n, 10), dtype=torch.float64, device=DEV)
    count = torch.empty(n, dtype=torch.int32, device=DEV)
    with torch.cuda.device(DEV):
        rc = N.load().ltr_debug_sturm_roots(P.data_ptr(), n, roots.data_ptr(), count.data_ptr(), DEV.index,
                                            C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream))
    N.check(rc, "ltr_debug_sturm_roots")
    return roots.cpu().numpy(), count.cpu().numpy()


def _solve_gpu(q):
    q = torch.as_tensor(np.ascontiguousarray(q, dtype=np.float64), device=DEV)
    n = q.shape[0]
    E = torch.empty((n, 10, 9), dtype=torch.float64, device=DEV)
    jr = torch.empty((n, 10), dtype=torch.int32, device=DEV)
    ns = torch.empty(n, dtype=torch.int32, device=DEV)
    with torch.cuda.device(DEV):
        rc = N.load().ltr_debug_essential_solve(q.data_ptr(), n, E.data_ptr(), jr.data_ptr(), ns.data_ptr(), DEV.index,
                                                C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream))
    N.check(rc, "ltr_debug_essential_solve")
    return E.cpu().numpy(), jr.cpu().numpy(), ns.cpu().numpy()


@pytest.mark.gpu
def test_kernel_sturm_roots_against_exact_and_host():
    """ess_roots against the exact reference on every case, and bit for bit against geometry.sturm_roots."""
    P = np.stack([c for _, c in ALL_POLYS])
    rg, cg = _sturm_gpu(P)
    rh, ch = G.sturm_roots(P)
    failed = []
    for i, (name, c) in enumerate(ALL_POLYS):
        assert cg[i] == ch[i] and np.array_equal(_bits(rg[i]), _bits(rh[i])), (name, rg[i], rh[i])
        try:
            _check_counts_and_roots(name, c, rg[i], int(cg[i]), _exact_of(name, c))
        except AssertionError as e:
            failed.append((name, str(e)))
    assert not failed, failed


@pytest.mark.gpu
def test_kernel_sturm_roots_on_random_dense_polynomials():
    """20 000 random dense polynomials (normal coefficients over 6 decades of scale): kernel and host bit for bit."""
    rng = np.random.default_rng(11)
    P = rng.normal(size=(20000, 11)) * 10.0 ** rng.uniform(-3, 3, (20000, 1))
    rg, cg = _sturm_gpu(P)
    rh, ch = G.sturm_roots(P)
    assert np.array_equal(cg, ch) and np.array_equal(_bits(rg), _bits(rh))


# ------------------------------------------------------------------ the five-point solver
def _compare_solutions(q, what):
    """ess_solve against geometry.essential_solutions bit for bit: solution count, root indices and E."""
    Eg, jg, ng = _solve_gpu(q)
    Eh, ok = G.essential_solutions(q)
    for k in range(len(q)):
        js = np.flatnonzero(ok[k])
        assert ng[k] == len(js) and np.array_equal(jg[k, :ng[k]], js), (what, k, jg[k], js)
        assert np.array_equal(Eg[k, :ng[k]].view(np.int64), Eh[k, js].view(np.int64)), (what, k)
        assert np.isnan(Eg[k, ng[k]:]).all() and (jg[k, ng[k]:] == -1).all()
    return Eg, jg, ng


def _ragged_samples(min_samples=100_000):
    """Samples of the ragged pose cases of test_pose: each pair's normalised correspondences and its hypotheses'
    sample indices (as the estimator draws them)."""
    cases, K0, K1, _ = _es_ragged_cases()
    out, total, p = [], 0, 0
    per_pair = 640
    for p, d in enumerate(cases):
        n = len(d["matches_p"])
        if n < 5:
            continue
        q = np.concatenate([G._normalised(d["kpts0"], K0[p]), G._normalised(d["kpts1"], K1[p])], 1)
        idx, ok = G.draw_samples(9, p, per_pair, n, 5)
        out.append(q[idx[ok]])
        total += int(ok.sum())
    assert total >= min_samples
    return np.concatenate(out)


@pytest.mark.gpu
def test_five_point_solver_bit_for_bit_on_ragged_samples():
    q = _ragged_samples()
    Eg, jg, ng = _solve_gpu(q)
    Eh, ok = G.essential_solutions(q)
    assert np.array_equal(ng, ok.sum(1))
    jh = np.where(ok, np.arange(10)[None], 99)
    jh.sort(1)
    jh = np.where(jh == 99, -1, jh)
    assert np.array_equal(jg, jh.astype(np.int32))
    # solution s of sample k is root jg[k, s]; gather the host's E in that order
    sel = np.where(jg >= 0, jg, 0)
    Ehs = np.take_along_axis(Eh, sel[:, :, None], 1)
    live = jg >= 0
    assert np.array_equal(Eg[live].view(np.int64), Ehs[live].view(np.int64))
    assert np.isnan(Eg[~live]).all()
    print(f"{len(q)} samples, {int(ng.sum())} solutions, {np.bincount(ng, minlength=11).tolist()} per count")


def _scene(rng, R, t, n=5, plane=None, depth=(3.0, 6.0)):
    """Exact normalised correspondences of n points (X1 = R X0 + t), optionally on the plane n . X = 1."""
    xy = rng.uniform(-1, 1, (n, 2))
    if plane is None:
        X = np.c_[xy, np.ones(n)] * rng.uniform(*depth, (n, 1))
    else:
        ray = np.c_[xy, np.ones(n)]
        X = ray / (ray @ plane)[:, None]
    X1 = X @ R.T + t
    return np.concatenate([X[:, :2] / X[:, 2:], X1[:, :2] / X1[:, 2:]], 1)


def _rank_eps_samples():
    """Samples whose QR column-norm ratio is just above and just below ESS_RANK_EPS: the fifth correspondence is the
    fourth moved by delta, and delta is bisected to where the host model's rank test flips."""
    rng = np.random.default_rng(21)
    R, t = syn.random_pose(rng)
    base = _scene(rng, R, t)
    d = rng.normal(size=4)

    def sample(delta):
        q = base.copy()
        q[4] = q[3] + delta * d
        return q

    rank_ok = lambda delta: bool(G._null_basis(sample(delta)[None])[1][0])
    lo, hi = 0.0, 1e-6
    assert not rank_ok(lo) and rank_ok(hi)
    for _ in range(200):
        mid = (lo + hi) / 2
        if mid in (lo, hi):
            break
        lo, hi = (lo, mid) if rank_ok(mid) else (mid, hi)
    return np.stack([sample(lo), sample(hi)])


@pytest.mark.gpu
def test_five_point_solver_bit_for_bit_on_structured_samples():
    rng = np.random.default_rng(5)
    qs, names = [], []
    for s in range(8):
        R, t = syn.random_pose(rng)
        q = _scene(rng, R, t)
        q[s % 5, :2] = 0.0                          # a keypoint exactly at the principal point (side 0)
        X0 = np.array([0.0, 0.0, 4.0])
        X1 = R @ X0 + t
        q[s % 5, 2:] = X1[:2] / X1[2]
        qs.append(q)
        names.append("principal_point")
        qs.append(_scene(rng, R, t, plane=np.array([0.05, -0.1, 0.25])))
        names.append("planar")
        qs.append(_scene(rng, *syn.random_pose(rng, translation=[0.0, 0.0, 1.0])))
        names.append("forward")
        qs.append(_scene(rng, R, np.zeros(3)))
        names.append("rotation")
        q = _scene(rng, R, t)
        q[3] = q[1]
        qs.append(q)
        names.append("identical")
        q = _scene(rng, R, t)
        a, b = rng.uniform(-1, 1, 2), rng.uniform(-1, 1, 2)
        q[:, :2] = a + np.linspace(0, 1, 5)[:, None] * (b - a)
        q[:, 2:] = a + 0.3 + np.linspace(0.1, 0.9, 5)[:, None] * (b - a)
        qs.append(q)
        names.append("collinear")
    qe = _rank_eps_samples()
    qs += list(qe)
    names += ["rank_below", "rank_above"]
    q = np.stack(qs)
    _, _, ng = _compare_solutions(q, "structured")
    got = dict(zip(names, ng))
    assert all(ng[i] == 0 for i, n in enumerate(names) if n in ("identical", "collinear")), list(zip(names, ng))
    assert got["rank_below"] == 0 and got["rank_above"] > 0
    assert all(ng[i] > 0 for i, n in enumerate(names) if n in ("principal_point", "planar", "forward"))


@pytest.mark.gpu
def test_five_point_solver_on_exact_scenes():
    """The kernel's solutions on 200 exact synthetic scenes, built as test_pose's CPU test builds its 60.  The true E is
    among them (to that test's bound).  Every
    returned E (unit norm) satisfies the 5 epipolar equations to 1e-12, det E = 0 and the trace constraint
    2 E E^T E - tr(E E^T) E = 0 to 1e-4, and 98 % of them to 1e-7.  The looser bound is for spurious roots of det B(z)
    near a double root: such a root is fixed only to about sqrt(u), and the cubic constraints lose as many digits."""
    scenes, qs = [], []
    for s in range(200):
        rng = np.random.default_rng(s)
        R, t = syn.random_pose(rng, 20.0)
        X = np.c_[rng.uniform(-1, 1, (5, 2)), rng.uniform(3, 6, 5)]
        X1 = X @ R.T + t
        scenes.append((R, t))
        qs.append(np.concatenate([X[:, :2] / X[:, 2:], X1[:, :2] / X1[:, 2:]], 1))
    q = np.stack(qs)
    Eg, jg, ng = _solve_gpu(q)
    errs, cubic = [], []
    for k, (R, t) in enumerate(scenes):
        assert 1 <= ng[k] <= 10
        Et = (np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]]) @ R).reshape(9)
        Et /= np.linalg.norm(Et)
        x0, x1 = np.c_[q[k, :, :2], np.ones(5)], np.c_[q[k, :, 2:], np.ones(5)]
        best = np.inf
        for s in range(ng[k]):
            e = Eg[k, s] / np.linalg.norm(Eg[k, s])
            best = min(best, np.abs(e - Et).max(), np.abs(e + Et).max())
            M = e.reshape(3, 3)
            assert np.abs(np.einsum("ni,ij,nj->n", x1, M, x0)).max() < 1e-12, k
            cubic.append(max(abs(np.linalg.det(M)), np.abs(2 * M @ M.T @ M - np.trace(M @ M.T) * M).max()))
        errs.append(best)
    errs, cubic = np.array(errs), np.array(cubic)
    assert np.mean(errs < 1e-9) >= 0.9 and errs.max() < 1e-6, (np.median(errs), errs.max())
    assert cubic.max() < 1e-4 and np.mean(cubic < 1e-7) >= 0.98, (cubic.max(), np.mean(cubic < 1e-7))


# ------------------------------------------------------------------ every hypothesis through the public API
HG_FIELDS = ("H", "valid", "inliers_p", "inliers_l", "n_inliers_p", "n_inliers_l", "hypothesis", "hypothesis_inliers")
ES_FIELDS = ("E", "R", "t", "valid", "inliers", "n_inliers", "n_cheirality", "hypothesis", "hypothesis_inliers")


def _rel_h(a, b):
    a, b = np.asarray(a) / np.asarray(a)[2, 2], np.asarray(b) / np.asarray(b)[2, 2]
    return float(np.abs(a - b).max() / np.abs(b).max())


def _refit_condition(res, p, h, thresh, use_points=True, use_lines=True):
    """lambda_max / (lambda_2 - lambda_1) of A^T A over the hypothesis' inliers (the refit's normal matrix): how much a
    perturbation of A^T A, relative to its norm, can turn the refit's eigenvector (Davis-Kahan)."""
    a, b = res.offsets_p[p:p + 2]
    c, e = res.offsets_l[p:p + 2]
    pts, s0, s1, _, _ = G._correspondences(res.keypoints0[p].cpu().numpy(), res.keypoints1[p].cpu().numpy(),
                                           res.matches_p[a:b].cpu().numpy(), res.klines0[p], res.klines1[p],
                                           res.matches_l[c:e].cpu().numpy(), use_points, use_lines)
    lines1 = G.pixel_lines(s1) if len(s1) else np.zeros((0, 3))
    with np.errstate(all="ignore"):
        rows = G._rows(pts, s0, s1, G._normalisation(pts, s0, s1))
    fl = G._inliers(h["H_hypothesis"].reshape(1, 9), pts, s0, lines1, thresh * thresh)[0]
    A = rows[fl].reshape(-1, 9)
    w = np.linalg.eigvalsh(A.T @ A)
    return float(w[-1] / (w[1] - w[0]))


# The kernels sum A^T A in another order than numpy and solve it by Jacobi instead of eigh, so the refitted H differs
# by about (rows summed) * u * cond relative.  Measured on an H100 SXM (700 W limit) over 4000 single-hypothesis refits
# (some over exactly 4 inliers, cond up to 1e9): at most 250 u cond.  REFIT_C leaves a factor 4 above that.
REFIT_C = 1e3


def _check_homography(res, out, p, thresh=3.0, **kw):
    """Pair p of a homography result against the host model: hypothesis and its inlier count exactly; H to 1e-9
    relative, plus REFIT_C u cond when the refit was kept (see _refit_condition); masks exactly except rows within
    1e-6 px of the threshold; counts equal to the masks."""
    h = _hg_host_pair(res, p, thresh=thresh, **kw)
    assert bool(out["valid"][p]) == h["valid"], p
    assert out["hypothesis"][p] == h["hypothesis"] and out["hypothesis_inliers"][p] == h["hypothesis_inliers"], p
    a, b = res.offsets_p[p:p + 2]
    c, e = res.offsets_l[p:p + 2]
    gp, gl = out["inliers_p"][a:b], out["inliers_l"][c:e]
    if not h["valid"]:
        assert np.isnan(out["H"][p]).all() and not gp.any() and not gl.any(), p
        assert out["n_inliers_p"][p] == 0 and out["n_inliers_l"][p] == 0
        return h
    tol = 1e-9
    if h["refit"]:
        tol += REFIT_C * U * _refit_condition(res, p, h, thresh, kw.get("use_points", True), kw.get("use_lines", True))
    assert np.isfinite(out["H"][p]).all() and _rel_h(out["H"][p], h["H"]) < tol, (p, out["H"][p], h["H"], tol)
    dp, dl = np.flatnonzero(gp != h["inliers_p"]), np.flatnonzero(gl != h["inliers_l"])
    if len(dp) or len(dl):
        kp0 = res.keypoints0[p].cpu().numpy()[dp]
        m = res.matches_p[a:b].cpu().numpy()[dp]
        pts = np.concatenate([kp0, res.keypoints1[p].cpu().numpy()[m]], 1)
        s0 = np.asarray(res.klines0[p], np.float32)[dl]
        s1 = np.asarray(res.klines1[p], np.float32)[res.matches_l[c:e].cpu().numpy()[dl]]
        r = np.sqrt(G.residuals(h["H"].reshape(1, 9), pts, s0, G.pixel_lines(s1) if len(s1) else np.zeros((0, 3)))[0])
        assert np.all(np.abs(r - thresh) < 1e-6), (p, r)
    assert out["n_inliers_p"][p] == gp.sum() and out["n_inliers_l"][p] == gl.sum(), p
    return h


def _check_pose(res, out, p, K0, K1, **kw):
    """Pair p of a pose result against the host model: hypothesis, its inlier count, masks and counts exactly, E to
    1e-12 (the unit scaling's sums differ), (R, t) the host's or another candidate with the same cheirality count,
    finite when valid."""
    h = _es_host_pair(res, p, K0, K1, **kw)
    assert bool(out["valid"][p]) == h["valid"], p
    assert out["hypothesis"][p] == h["hypothesis"] and out["hypothesis_inliers"][p] == h["hypothesis_inliers"], p
    a, b = res.offsets_p[p:p + 2]
    gm = out["inliers"][a:b]
    if not h["valid"]:
        assert np.isnan(out["E"][p]).all() and np.isnan(out["R"][p]).all() and np.isnan(out["t"][p]).all(), p
        assert not gm.any() and out["n_inliers"][p] == 0 and out["n_cheirality"][p] == 0, p
        return h
    for f in ("E", "R", "t"):
        assert np.isfinite(out[f][p]).all(), (p, f)
    assert np.abs(out["E"][p] - h["E"]).max() < 1e-12, (p, out["E"][p], h["E"])
    assert np.array_equal(gm, h["inliers_p"]), p
    assert out["n_inliers"][p] == h["n_inliers"] == gm.sum(), p
    rows = np.flatnonzero(h["inliers_p"])
    m = res.matches_p[a:b].cpu().numpy()[rows]
    q = np.concatenate([G._normalised(res.keypoints0[p].cpu().numpy()[rows], K0),
                        G._normalised(res.keypoints1[p].cpu().numpy()[m], K1)], 1)
    cand = G.decompose_essential(h["E"])
    cnt = [int(G.cheirality(Rc, tc, q, kw.get("dist_thresh", 1e9)).sum()) for Rc, tc in cand]
    assert out["n_cheirality"][p] == h["n_cheirality"] == max(cnt), p
    assert any(c == h["n_cheirality"] and np.abs(out["R"][p] - Rc).max() < 1e-9
               and np.abs(out["t"][p] - tc).max() < 1e-9
               for c, (Rc, tc) in zip(cnt, cand)), p
    return h


def _hg_run(res, **kw):
    out = G.estimate_homographies(res, **kw)
    return {f: getattr(out, f).cpu().numpy() for f in HG_FIELDS}


def _es_run(res, K0, K1, **kw):
    out = G.estimate_poses(res, K0, K1, **kw)
    return {f: getattr(out, f).cpu().numpy() for f in ES_FIELDS}


P_COPIES = 2000


@pytest.mark.gpu
@pytest.mark.parametrize("outlier_frac", [0.0, 0.5])
def test_homography_every_hypothesis_end_to_end(outlier_frac):
    Ht = syn.random_homography(np.random.default_rng(3), strength=0.15)
    d = syn.make_homography_correspondences(31, 60, 20, Ht, noise_px=0.3, outlier_frac=outlier_frac)
    res = _hg_matches([d] * P_COPIES, shuffle_rows=False)
    out = _hg_run(res, n_hypotheses=1, seed=2)
    hyp = set()
    for p in range(P_COPIES):
        h = _check_homography(res, out, p, n_hypotheses=1, seed=2)
        hyp.add(h["H_hypothesis"].tobytes())
    assert len(hyp) > P_COPIES // 2         # the copies did evaluate different hypotheses


@pytest.mark.gpu
@pytest.mark.parametrize("outlier_frac", [0.0, 0.5])
def test_pose_every_hypothesis_end_to_end(outlier_frac):
    R, t = syn.random_pose(np.random.default_rng(6))
    d = syn.make_pose_correspondences(32, 80, R, t, noise_px=0.3, outlier_frac=outlier_frac)
    res = _es_matches([d] * P_COPIES, shuffle_rows=False)
    out = _es_run(res, K, K, n_hypotheses=1, seed=2)
    hyp = set()
    for p in range(P_COPIES):
        h = _check_pose(res, out, p, K, K, n_hypotheses=1, seed=2)
        hyp.add(h["E_hypothesis"].tobytes())
    assert len(hyp) > P_COPIES // 2


# ------------------------------------------------------------------ edges on the GPU
E2, E4 = np.zeros((0, 2), np.float32), np.zeros((0, 2, 2), np.float32)


def _hg_case(kp0, kp1, mp, l0, l1, ml):
    f = lambda a, s: np.asarray(a, np.float32).reshape(s)
    return {"kpts0": f(kp0, (-1, 2)), "kpts1": f(kp1, (-1, 2)), "matches_p": np.asarray(mp, np.int32).reshape(-1),
            "klines0": f(l0, (-1, 2, 2)), "klines1": f(l1, (-1, 2, 2)),
            "matches_l": np.asarray(ml, np.int32).reshape(-1)}


def _hg_degenerate_cases():
    """test_homography's degenerate inputs, and exactly 4 correspondences in each point / line mix."""
    three = np.array([[1, 2], [30, 4], [5, 60]], np.float32)
    same = np.tile(np.float32([[100, 100]]), (10, 1))
    line = np.stack([np.arange(10, 210, 20), np.full(10, 100)], 1).astype(np.float32)
    dot = np.tile(np.float32([[[5, 5], [5, 5]]]), (6, 1, 1))
    segs = np.random.default_rng(0).uniform(0, 400, (6, 2, 2)).astype(np.float32)
    cases = [_hg_case(three, three + 1, np.arange(3), E4, E4, []), _hg_case(same, same + 5, np.arange(10), E4, E4, []),
             _hg_case(line, line * 2, np.arange(10), E4, E4, []), _hg_case(E2, E2, [], segs, dot, np.arange(6)),
             _hg_case(E2, E2, [], E4, E4, []), _hg_case(three, three, [-1, 7, 2], E4, E4, [])]
    Ht = syn.random_homography(np.random.default_rng(4), strength=0.15)
    for n_p in range(5):
        d = syn.make_homography_correspondences(40 + n_p, n_p, 4 - n_p, Ht, noise_px=0.0, outlier_frac=0.0)
        cases.append(d)
    return cases


@pytest.mark.gpu
def test_homography_degenerate_and_minimal_inputs():
    cases = _hg_degenerate_cases()
    res = _hg_matches(cases, shuffle_rows=False)
    out = _hg_run(res, n_hypotheses=64, seed=1)
    for p in range(len(cases)):
        _check_homography(res, out, p, n_hypotheses=64, seed=1)
    assert not out["valid"][:6].any()
    # 4p, 3p1l, 1p3l and 4l fix H; 2p2l has a second null vector (test_two_points_two_lines_are_degenerate)
    assert out["valid"][[6, 7, 9, 10]].all()


@pytest.mark.gpu
def test_pose_degenerate_and_minimal_inputs():
    four = np.array([[1, 2], [30, 4], [5, 60], [70, 80]], np.float32)
    same = np.tile(np.float32([[100, 100]]), (10, 1))
    R, t = syn.random_pose(np.random.default_rng(5))
    d = syn.make_pose_correspondences(4, 8, R, t, noise_px=0.0, outlier_frac=0.0)
    c = lambda k0, k1, m: {"kpts0": np.asarray(k0, np.float32), "kpts1": np.asarray(k1, np.float32),
                           "matches_p": np.asarray(m, np.int32)}
    cases = [c(four, four + 1, np.arange(4)), c(same, same + 5, np.arange(10)), c(E2, E2, []),
             c(d["kpts0"], d["kpts1"], [-1, 9, 2, 3, 4, -5, 6, 7]),
             c(d["kpts0"], d["kpts1"], [-1, 9, 2, 3, 4, -5, 6, 100]),
             c(d["kpts0"][:5], d["kpts1"][:5], np.arange(5))]
    res = _es_matches(cases, shuffle_rows=False)
    out = _es_run(res, K, K, n_hypotheses=64, seed=1)
    for p in range(len(cases)):
        _check_pose(res, out, p, K, K, n_hypotheses=64, seed=1)
    assert out["valid"].tolist() == [False, False, False, True, False, True]
    assert out["n_inliers"][[3, 5]].tolist() == [5, 5]


@pytest.mark.gpu
@pytest.mark.parametrize("n_hyp", [1, 127, 128, 129, 4097])
def test_hypothesis_counts_around_the_cta(n_hyp):
    """n_hypotheses off the 128-thread CTA: the last CTA's idle threads must neither win nor be skipped."""
    from tests.test_homography import _ragged_cases as hg_ragged
    cases, _ = hg_ragged(16, seed=2)
    res = _hg_matches(cases)
    out = _hg_run(res, n_hypotheses=n_hyp, seed=4)
    for p in range(res.n_pairs):
        _check_homography(res, out, p, n_hypotheses=n_hyp, seed=4)
    cases, K0, K1, _ = _es_ragged_cases(12, seed=3)
    res = _es_matches(cases)
    out = _es_run(res, K0, K1, n_hypotheses=n_hyp, seed=4)
    for p in range(res.n_pairs):
        _check_pose(res, out, p, K0[p], K1[p], n_hypotheses=n_hyp, seed=4)


@pytest.mark.gpu
def test_homography_staging_filled_exactly():
    """11 352 point rows and 8 line rows stage exactly SMEM_MAX bytes: accepted and compared; one more row of either
    kind is refused (code -4) before any launch."""
    n_p = (G.SMEM_MAX - 8 * G.SMEM_PER_LINE) // G.SMEM_PER_POINT
    assert n_p == 11352 and n_p * G.SMEM_PER_POINT + 8 * G.SMEM_PER_LINE == G.SMEM_MAX
    Ht = syn.random_homography(np.random.default_rng(9), strength=0.1)
    d = syn.make_homography_correspondences(9, n_p, 8, Ht, noise_px=0.3, outlier_frac=0.4)
    small = syn.make_homography_correspondences(10, 50, 3, Ht, noise_px=0.3, outlier_frac=0.4)
    res = _hg_matches([small, d], shuffle_rows=False)
    out = _hg_run(res, n_hypotheses=200, seed=6)
    for p in range(2):
        _check_homography(res, out, p, n_hypotheses=200, seed=6)
    assert out["valid"].all()
    for extra_p, extra_l in ((1, 0), (0, 1)):
        e = syn.make_homography_correspondences(11, n_p + extra_p, 8 + extra_l, Ht)
        N.reset_launch_count()
        with pytest.raises(N.LtrError, match=r"code -4"):
            G.estimate_homographies(_hg_matches([e], shuffle_rows=False))
        assert N.launch_count() == 0


@pytest.mark.gpu
def test_pose_staging_filled_exactly():
    """6206 rows fit the pose kernel's staging (33 bytes a row): accepted and compared; 6207 are refused (code -4)
    before any launch."""
    n = G.SMEM_MAX // G.SMEM_PER_ROW_E
    assert n == 6206
    R, t = syn.random_pose(np.random.default_rng(12))
    d = syn.make_pose_correspondences(12, n, R, t, noise_px=0.3, outlier_frac=0.4)
    small = syn.make_pose_correspondences(13, 40, R, t, noise_px=0.3, outlier_frac=0.4)
    res = _es_matches([small, d], shuffle_rows=False)
    out = _es_run(res, K, K, n_hypotheses=128, seed=6)
    for p in range(2):
        _check_pose(res, out, p, K, K, n_hypotheses=128, seed=6)
    assert out["valid"].all()
    N.reset_launch_count()
    with pytest.raises(N.LtrError, match=r"code -4"):
        G.estimate_poses(_es_matches([syn.make_pose_correspondences(14, n + 1, R, t)], shuffle_rows=False), K, K)
    assert N.launch_count() == 0


def _threshold_at_residual():
    """A correspondence set whose row 0 has residual exactly thresh^2 under the single hypothesis (n_hypotheses=1,
    pair 0) and the thresh: row 0's partner is moved until the residual r is the square of a double."""
    Ht = syn.random_homography(np.random.default_rng(13), strength=0.1)
    d = syn.make_homography_correspondences(13, 40, 0, Ht, noise_px=0.2, outlier_frac=0.0)
    rng = np.random.default_rng(14)
    for _ in range(200):
        d["kpts1"][0] = (syn.warp_points(Ht, d["kpts0"][:1].astype(np.float64))[0]
                         + rng.uniform(-2.5, 2.5, 2)).astype(np.float32)
        h = _hg_host_pair(_FakeRes(d), 0, n_hypotheses=1, thresh=3.0)
        if not h["valid"] or h["hypothesis"] != 0:
            continue
        pts = np.concatenate([d["kpts0"][:1], d["kpts1"][:1]], 1)
        r = float(G.residuals(h["H_hypothesis"].reshape(1, 9), pts, E4, np.zeros((0, 3)))[0, 0])
        t0 = math.sqrt(r)
        for th in (t0, math.nextafter(t0, 0), math.nextafter(t0, math.inf), math.nextafter(math.nextafter(t0, 0), 0),
                   math.nextafter(math.nextafter(t0, math.inf), math.inf)):
            if th * th == r:
                return d, th, r
    raise AssertionError("no residual with an exact square root found")


class _FakeRes:
    """Just enough of an ImagePairMatches for _hg_host_pair on one host-side correspondence set."""

    def __init__(self, d):
        self.offsets_p, self.offsets_l = [0, len(d["matches_p"])], [0, len(d["matches_l"])]
        t = lambda a: torch.from_numpy(np.asarray(a))
        self.keypoints0, self.keypoints1 = [t(d["kpts0"])], [t(d["kpts1"])]
        self.matches_p, self.matches_l = t(d["matches_p"]), t(d["matches_l"])
        self.klines0, self.klines1 = [d["klines0"]], [d["klines1"]]


def test_threshold_case_is_exact_on_the_host():
    """The host model's side of the thresh^2 case: the row is not an inlier of the hypothesis at thresh, and is one
    at the next larger double."""
    d, th, r = _threshold_at_residual()
    h = _hg_host_pair(_FakeRes(d), 0, n_hypotheses=1, thresh=th)
    h_up = _hg_host_pair(_FakeRes(d), 0, n_hypotheses=1, thresh=math.nextafter(th, math.inf))
    assert h["hypothesis_inliers"] + 1 == h_up["hypothesis_inliers"]
    pts = np.concatenate([d["kpts0"], d["kpts1"]], 1)
    res = G.residuals(h["H_hypothesis"].reshape(1, 9), pts, E4, np.zeros((0, 3)))[0]
    assert res[0] == th * th and h["hypothesis_inliers"] == int((res < th * th).sum())


@pytest.mark.gpu
def test_homography_residual_exactly_at_threshold():
    """A point whose residual under the hypothesis is exactly thresh^2 is an outlier (the rule is strict <) in the
    kernels as in the host model: the hypothesis' inlier count leaves it out."""
    d, th, r = _threshold_at_residual()
    res = _hg_matches([d], shuffle_rows=False)
    out = _hg_run(res, n_hypotheses=1, thresh=th)
    h = _check_homography(res, out, 0, n_hypotheses=1, thresh=th)
    pts = np.concatenate([d["kpts0"], d["kpts1"]], 1)
    resid = G.residuals(h["H_hypothesis"].reshape(1, 9), pts, E4, np.zeros((0, 3)))[0]
    assert resid[0] == th * th
    assert out["hypothesis_inliers"][0] == int((resid < th * th).sum())
    if not h["refit"]:
        assert out["inliers_p"][0] == 0


@pytest.mark.gpu
def test_homography_projection_at_infinity():
    """A strong perspective whose horizon crosses the image: H = [[1, 0, 0], [0, 1, 0], [-1/512, 0, 1]] sends x = 512
    to infinity.  The inlier points sit on columns where w = 1, 1/2, ..., 1/16, so their images are exact in fp32 and
    the estimate is H to rounding; points on the horizon (random partners) and segments with one end point on it
    then project with |w| <= FLT_EPSILON and are outliers, in the kernels as in the host model."""
    rng = np.random.default_rng(15)
    cols = np.array([0.0, 256.0, 384.0, 448.0, 480.0])
    x0 = np.c_[rng.choice(cols, 150), rng.integers(0, 480, 150)].astype(np.float64)
    w = 1.0 - x0[:, 0] / 512.0
    x1 = x0 / w[:, None]
    horizon = np.c_[np.full(20, 512.0), rng.integers(0, 480, 20)]
    kp0 = np.concatenate([x0, horizon]).astype(np.float32)
    kp1 = np.concatenate([x1, rng.uniform(0, 600, (20, 2))]).astype(np.float32)
    c = rng.integers(0, 4, 30)                     # a0 and m0 on adjacent columns: b0 = 2 m0 - a0 is on the horizon
    a0 = np.c_[cols[c], rng.integers(100, 380, 30)]
    m0 = np.c_[cols[c + 1], rng.integers(100, 380, 30)]
    b0 = 2.0 * m0 - a0
    a1 = a0 / (1.0 - a0[:, :1] / 512.0)
    m1 = m0 / (1.0 - m0[:, :1] / 512.0)
    d = _hg_case(kp0, kp1, np.arange(170), np.stack([a0, b0], 1), np.stack([a1, m1], 1), np.arange(30))
    res = _hg_matches([d] * 8, shuffle_rows=False)
    out = _hg_run(res, n_hypotheses=256, seed=3)
    n_at_inf = 0
    for p in range(8):
        h = _check_homography(res, out, p, n_hypotheses=256, seed=3)
        assert h["valid"] and h["n_inliers_p"] == 150
        Hh = h["H_hypothesis"].reshape(9)
        ends = np.concatenate([kp0[150:], b0.astype(np.float32)]).astype(np.float64)
        n_at_inf += int((np.abs(Hh[6] * ends[:, 0] + Hh[7] * ends[:, 1] + Hh[8]) <= G.FLT_EPSILON).sum())
        assert not out["inliers_p"][res.offsets_p[p] + 150:res.offsets_p[p + 1]].any()
        assert not out["inliers_l"][res.offsets_l[p]:res.offsets_l[p + 1]].any()
    assert n_at_inf == 8 * 50


@pytest.mark.gpu
def test_homography_large_and_tiny_coordinates():
    """Coordinates up to 16 000 px, and point clouds less than 1e-3 px across."""
    rng = np.random.default_rng(16)
    big = syn.make_homography_correspondences(16, 400, 60, syn.random_homography(rng, 16000, 12000, 0.1),
                                              w=16000, h=12000, noise_px=0.5, outlier_frac=0.3)
    tiny = []
    for s in range(3):
        x0 = 3.0 + rng.uniform(0, 1e-3, (60, 2))
        A = np.array([[1.1, 0.1, 0.5], [-0.05, 0.9, 2.0], [1e-3, -2e-3, 1.0]])
        x1 = syn.warp_points(A, x0) + rng.normal(0, 1e-6, (60, 2)) * s
        tiny.append(_hg_case(x0, x1, np.arange(60), E4, E4, []))
    cases = [big] + tiny
    res = _hg_matches(cases, shuffle_rows=False)
    out = _hg_run(res, n_hypotheses=256, seed=8)
    for p in range(len(cases)):
        _check_homography(res, out, p, n_hypotheses=256, seed=8)
    assert out["valid"][0]


@pytest.mark.gpu
def test_pose_large_and_tiny_coordinates_and_intrinsics():
    """Coordinates up to 16 000 px, point clouds less than 1e-3 px across, and per-pair intrinsics with fx != fy and
    focal lengths near 1e5."""
    rng = np.random.default_rng(17)
    Kbig = np.array([[9000.0, 0.0, 8000.0], [0.0, 8500.0, 6000.0], [0.0, 0.0, 1.0]])
    Kfar0 = np.array([[1.0e5, 0.0, 320.0], [0.0, 0.93e5, 240.0], [0.0, 0.0, 1.0]])
    Kfar1 = np.array([[0.97e5, 0.0, 300.0], [0.0, 1.04e5, 250.0], [0.0, 0.0, 1.0]])
    Kx = np.array([[450.0, 0.0, 319.5], [0.0, 620.0, 239.5], [0.0, 0.0, 1.0]])
    cases, K0s, K1s = [], [], []
    Ky = np.array([[700.0, 0.0, 300.0], [0.0, 540.0, 260.0], [0.0, 0.0, 1.0]])
    for Ka, Kb, w, h in ((Kbig, Kbig, 16000, 12000), (Kfar0, Kfar1, 640, 480), (Kx, Kfar0, 640, 480),
                         (Kx, Ky, 640, 480)):
        R, t = syn.random_pose(rng)
        cases.append(syn.make_pose_correspondences(int(rng.integers(1e6)), 300, R, t, Ka, Kb, noise_px=0.3,
                                                   outlier_frac=0.4, w=w, h=h))
        K0s.append(Ka)
        K1s.append(Kb)
    for s in range(2):                                          # a cloud < 1e-3 px across on both sides
        x0 = 100.0 + rng.uniform(0, 1e-3, (40, 2))
        x1 = 120.0 + rng.uniform(0, 1e-3, (40, 2))
        cases.append({"kpts0": x0.astype(np.float32), "kpts1": x1.astype(np.float32),
                      "matches_p": np.arange(40, dtype=np.int32)})
        K0s.append(K)
        K1s.append(K)
    K0s, K1s = np.stack(K0s), np.stack(K1s)
    res = _es_matches(cases, shuffle_rows=False)
    out = _es_run(res, K0s, K1s, n_hypotheses=256, seed=9)
    for p in range(len(cases)):
        _check_pose(res, out, p, K0s[p], K1s[p], n_hypotheses=256, seed=9)
    assert out["valid"][:4].all()
