"""The descriptor matcher against float64 and against the fp32 arithmetic it promises, at the edges of its contract:
descriptor scale (distance mode 1), descriptor dimension, the strict threshold, exact ties at 0 and ragged batches
with an empty side.

Two host references:
- `dist64`: float64 distances of the fp32 descriptors.
- `dist32_model`: what the exact path promises (match_tc.cuh, match_kernels.cuh): squared norms and dot products as
  ascending-k fp32 fused multiply-add chains, then `2 - 2 acc` or `(sqa + sqb) - 2 acc`, clipped at 0.  It is a small
  C program calling `fmaf`, because emulating an FMA in float64 rounds twice.

Match indices must equal the decisions of `dist32_model` on every row.  On rows whose float64 margins are far above
the fp32 rounding (`decisive`), they must also equal the decisions of `dist64`."""
import ctypes
import os
import re
import shutil
import subprocess
from fractions import Fraction

import numpy as np
import pytest
import torch

from linetr_b200 import _native as N
from linetr_b200 import _ops, eval_matcher as em, nn_matcher as nnm
from oracle import linetr_oracle as orc
from tests.test_gpu_parity import DIST_TOL

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda", 0)
ROWS, CF = N.LAYOUT_ROWS, N.LAYOUT_CHANNEL_FIRST

_MODEL_SRC = r"""
#include <math.h>
/* squared norms: one ascending-k fmaf chain per row */
void model_sq(const float* x, long n, int d, float* out) {
  for (long i = 0; i < n; ++i) {
    float s = 0.f;
    for (int k = 0; k < d; ++k) s = fmaf(x[i * d + k], x[i * d + k], s);
    out[i] = s;
  }
}
/* mode 0: max(0, 2 - 2 acc); mode 1: max(0, (sqa + sqb) - 2 acc); acc an ascending-k fmaf chain */
void model_dist(const float* a, const float* b, long n0, long n1, int d, int mode, const float* sqa, const float* sqb,
                float* out) {
  for (long i = 0; i < n0; ++i)
    for (long j = 0; j < n1; ++j) {
      float acc = 0.f;
      for (int k = 0; k < d; ++k) acc = fmaf(a[i * d + k], b[j * d + k], acc);
      const float v = mode ? (sqa[i] + sqb[j]) - 2.f * acc : 2.f - 2.f * acc;
      out[i * n1 + j] = fmaxf(v, 0.f);
    }
}
"""


@pytest.fixture(scope="module")
def model32(tmp_path_factory):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler for the fp32 FMA model")
    td = tmp_path_factory.mktemp("fp32_model")
    src, so = str(td / "model.c"), str(td / "model.so")
    with open(src, "w") as f:
        f.write(_MODEL_SRC)
    # no contraction, no fast-math: every operation rounds exactly as written
    subprocess.check_call([cc, "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", "-o", so, src, "-lm"])
    lib = ctypes.CDLL(so)
    f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
    lib.model_sq.argtypes = [f32p, ctypes.c_long, ctypes.c_int, f32p]
    lib.model_dist.argtypes = [f32p, f32p, ctypes.c_long, ctypes.c_long, ctypes.c_int, ctypes.c_int, f32p, f32p, f32p]
    return lib


def sq32(lib, x):
    x = np.ascontiguousarray(x, np.float32)
    out = np.empty(len(x), np.float32)
    lib.model_sq(x, len(x), x.shape[1] if x.ndim == 2 else 0, out)
    return out


def dist32_model(lib, a, b, mode):
    """a [n0, d], b [n1, d] fp32 rows -> fp32 [n0, n1]."""
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    out = np.empty((len(a), len(b)), np.float32)
    if out.size:
        lib.model_dist(a, b, len(a), len(b), a.shape[1], int(mode), sq32(lib, a), sq32(lib, b), out)
    return out


def dist64(a, b, mode):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    s = a @ b.T
    if mode == 0:
        return np.maximum(2.0 - 2.0 * s, 0.0)
    return np.maximum((a * a).sum(1)[:, None] + (b * b).sum(1)[None, :] - 2.0 * s, 0.0)


def decisions(dist, thr, mutual):
    """orc.nn_matcher_distmat semantics on a [n0, n1] distance matrix: first-minimum argmin, strict `< thr`,
    optional mutual check.  Returns (matches0, row argmin, column argmin)."""
    n0, n1 = dist.shape
    if n0 == 0 or n1 == 0:
        return np.full(n0, -1, np.int32), np.zeros(n0, np.int64), np.zeros(n1, np.int64)
    idx = np.argmin(dist, axis=1)
    nn1 = np.argmin(dist, axis=0)
    keep = dist[np.arange(n0), idx] < thr
    if mutual:
        keep &= nn1[idx] == np.arange(n0)
    return np.where(keep, idx, -1).astype(np.int32), idx, nn1


def _top2_gap(x, axis):
    if x.shape[axis] < 2:
        return np.full(x.shape[1 - axis], np.inf)
    s = np.sort(x, axis=axis)
    return s[1] - s[0] if axis == 0 else s[:, 1] - s[:, 0]


def decisive(d64, d32, thr, mutual):
    """Rows whose decision no fp32 rounding can change: every float64 margin (top-2 gap, |best - thr|, and with the
    mutual check the top-2 gap of the partner column) exceeds 4x the largest |d32 - d64| among the entries involved."""
    n0, n1 = d64.shape
    if n0 == 0 or n1 == 0:
        return np.ones(n0, bool)
    err = np.abs(d32.astype(np.float64) - d64)
    idx = np.argmin(d64, axis=1)
    margin = np.minimum(_top2_gap(d64, 1), np.abs(d64[np.arange(n0), idx] - float(thr)))
    bound = err.max(axis=1)
    if mutual:
        margin = np.minimum(margin, _top2_gap(d64, 0)[idx])
        bound = np.maximum(bound, err.max(axis=0)[idx])
    return margin > 4.0 * bound


# ------------------------------------------------------------------ self-tests of the references (CPU)
def _round_f32(q: Fraction) -> Fraction:
    """Round an exact rational to the nearest float32, ties to even (normal and subnormal range)."""
    if q == 0:
        return Fraction(0)
    m = abs(q)
    e = m.numerator.bit_length() - m.denominator.bit_length()
    if m < Fraction(2) ** e:
        e -= 1
    e = max(e - 23, -149)
    scaled = m / Fraction(2) ** e
    n = scaled.numerator // scaled.denominator
    r = scaled - n
    if r > Fraction(1, 2) or (r == Fraction(1, 2) and n % 2):
        n += 1
    return (n * Fraction(2) ** e) * (1 if q > 0 else -1)


def _exact_model(a, b, mode):
    F = [[Fraction(float(v)) for v in row] for row in a], [[Fraction(float(v)) for v in row] for row in b]

    def chain(x, y):
        acc = Fraction(0)
        for u, v in zip(x, y):
            acc = _round_f32(u * v + acc)
        return acc

    out = np.empty((len(a), len(b)), np.float32)
    for i, x in enumerate(F[0]):
        for j, y in enumerate(F[1]):
            acc = chain(x, y)
            v = _round_f32(2 - 2 * acc) if mode == 0 else _round_f32(_round_f32(chain(x, x) + chain(y, y)) - 2 * acc)
            out[i, j] = max(float(v), 0.0)
    return out


def test_model_equals_exact_rational_evaluation(model32):
    rng = np.random.default_rng(5)
    for d, scale in ((16, 1.0), (48, 16.0), (32, 1e-3)):
        # mixed magnitudes make the products' low bits matter to every rounding of the chain
        a = (rng.standard_normal((3, d)) * scale * 2.0 ** rng.integers(-6, 7, (3, d))).astype(np.float32)
        b = (rng.standard_normal((4, d)) * scale * 2.0 ** rng.integers(-6, 7, (4, d))).astype(np.float32)
        b[0] = a[0]                                           # a self-distance: mode 1 cancels to ~0
        for mode in (0, 1):
            got = dist32_model(model32, a, b, mode)
            assert np.array_equal(got, _exact_model(a, b, mode)), (d, mode)
        want_sq = [float(_exact_model(a[i:i + 1], np.zeros((1, d), np.float32), 1)[0, 0]) for i in range(3)]
        assert np.array_equal(sq32(model32, a), np.float32(want_sq))


def test_model_fma_is_not_a_double_rounding(model32):
    """acc = fmaf(a, b, c) whose exact value lies just below a float32 midpoint: float64 lands on the midpoint and
    rounds to even, the other way.  The model must give the correctly rounded chain."""
    x = np.array([[0.25 * (1 + 2 ** -23), 2 ** -13 * (1 + 2 ** -23)]], np.float32)
    y = np.array([[1.0, 2 ** -13 * (1 - 2 ** -23)]], np.float32)
    acc = np.float32(0)
    for u, v in zip(x[0], y[0]):                         # float64 product and sum, then one rounding to float32
        acc = np.float32(np.float64(acc) + np.float64(u) * np.float64(v))
    emulated = np.maximum(np.float32(2) - np.float32(2) * acc, np.float32(0))
    exact = _exact_model(x, y, 0)
    assert exact[0, 0] != emulated
    assert np.array_equal(dist32_model(model32, x, y, 0), exact)


def test_decisions_equal_oracle():
    rng = np.random.default_rng(11)
    for n0, n1 in ((1, 1), (1, 9), (9, 1), (40, 33)):
        d = (rng.integers(0, 12, (n0, n1)) / 8.0).astype(np.float32)   # many exact ties
        for thr in (0.0, 0.5, 2.0):
            for mutual in (True, False):
                want = orc.match_indices(orc.nn_matcher_distmat(d[None], np.float32(thr), mutual))
                assert np.array_equal(decisions(d, np.float32(thr), mutual)[0], want)


def test_decisive_rule_rejects_planted_ties():
    thr = 0.5
    d64 = np.array([[0.10, 0.10, 0.90],                 # exact tie in the row
                    [0.50, 0.80, 0.90],                 # best exactly at the threshold
                    [0.20, 0.60, 0.95],                 # clear
                    [0.70, 0.30, 0.30 + 1e-9],          # gap far below the rounding bound
                    [0.90, 0.85, 0.15]], np.float64)    # clear
    d32 = (d64 + 1e-8).astype(np.float32)               # every entry carries >= ~1e-8 of rounding
    got = decisive(d64, d32, thr, mutual=False)
    assert got.tolist() == [False, False, True, False, True]
    # mutual: the partner column of row 2 (column 0) gets a near-tie between rows 0 and 4
    d64m = d64.copy()
    d64m[4, 0] = 0.10 + 1e-9
    assert decisive(d64m, d64m.astype(np.float32), thr, mutual=True).tolist()[2] is False
    assert decisive(d64m, d64m.astype(np.float32), thr, mutual=False).tolist()[2] is True
    # single column / single row: no second-best, the threshold margin alone decides
    assert decisive(np.array([[0.1]]), np.array([[0.1]], np.float32), thr, True).tolist() == [True]
    assert decisive(np.array([[0.5]]), np.array([[0.5]], np.float32), thr, True).tolist() == [False]


# ------------------------------------------------------------------ data
def _unit(rng, n, d):
    x = rng.standard_normal((n, d))
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def _sweep_data(c, n0, n1, seed, d=256):
    """Rows near a 'true' column (distance sigma^2 c^2 around thr = c^2 / 2), a few unrelated rows, columns planted
    at geometric gaps 1e-7 c^2 .. 1e-2 c^2 from a row's true column, and rows planted at the same gaps from the
    threshold.  Norms vary in 0.8 c .. 1.25 c.  Returns fp32 rows a [n0, d], b [n1, d] and the fp32 threshold."""
    rng = np.random.default_rng(seed)
    b = _unit(rng, n1, d) * (c * rng.uniform(0.8, 1.25, (n1, 1)))
    true = rng.integers(0, n1, n0)
    sigma = rng.uniform(0.2, 0.9, (n0, 1))
    a = b[true] + _unit(rng, n0, d) * sigma * c
    far = rng.random(n0) < 0.125
    a[far] = _unit(rng, int(far.sum()), d) * c
    thr = 0.5 * c * c
    gaps = c * c * 10.0 ** np.linspace(-7, -2, 11)
    used = set()
    rows = rng.permutation(n0)
    k = 0
    for g in gaps:                                   # rows at thr +- g
        if k >= n0:
            break
        i = rows[k]; k += 1
        r = a[i] - b[true[i]]
        a[i] = b[true[i]] + r * np.sqrt((thr + g * rng.choice([-1, 1])) / (r @ r))
        used.add(int(true[i]))
    for g in np.concatenate([gaps, gaps]):           # near-tie columns at +- g from a row's true column
        if k >= n0:
            break
        i = rows[k]; k += 1
        free = [j for j in range(n1) if j not in used and j != true[i]]
        if not free:
            break
        j = int(rng.choice(free))
        used.update((j, int(true[i])))
        r = b[true[i]] - a[i]
        v = rng.standard_normal(d)
        v -= (v @ r) / (r @ r) * r
        v *= np.linalg.norm(r) / np.linalg.norm(v)
        th = rng.uniform(0.3, 1.0)
        rr = r * np.cos(th) + v * np.sin(th)         # |rr| = |r|
        s = np.sqrt(max(r @ r + g * rng.choice([-1, 1]), 0.0) / (r @ r))
        b[j] = a[i] + rr * s                         # |a_i - b_j|^2 = |r|^2 +- g
    return a.astype(np.float32), b.astype(np.float32), np.float32(thr)


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _match(a, b, layout, thr, mutual, mode):
    """One pair through ltr_match (tensor-core path for d == 256); a, b fp32 rows [n, d]."""
    n0, n1, d = len(a), len(b), a.shape[1]
    x, y = (a, b) if layout == ROWS else (a.T, b.T)
    out = _ops.match_descriptors(_t(x), _t(y), layout, 1, float(thr), mutual, n0=n0, n1=n1, d=d, want_dist=d != 256,
                                 dist_mode=mode)
    return {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in out.items()}


def _check_contract(got, d32, d64, thr, mutual, tol_rows, what):
    """Indices equal the fp32 model on every row and fp64 on decisive rows; counts; returned best distances."""
    want32, idx32, nn32 = decisions(d32, thr, mutual)
    want64 = decisions(d64, float(thr), mutual)[0]
    ok = decisive(d64, d32, thr, mutual)
    m0 = got["matches0"]
    bad = np.nonzero(m0 != want32)[0]
    assert bad.size == 0, f"{what}: rows {bad[:8].tolist()} differ from the fp32 model ({bad.size} of {len(m0)})"
    assert np.array_equal(m0[ok], want64[ok]), what
    assert int(got["counts"][0]) == int((m0 >= 0).sum()), what
    if d64.shape[1]:
        err = np.abs(got["scores0"].astype(np.float64) - d64.min(axis=1))
        assert (err <= tol_rows).all(), f"{what}: score error {float((err / tol_rows).max()):.2f} x tolerance"
    if mutual and d64.shape[0]:
        assert np.array_equal(got["nn1"], nn32), what   # the column argmin is an output too
    return ok


# ------------------------------------------------------------------ distance mode 1: descriptor scale
SWEEP_C = [2.0 ** -4, 1.0, 4.0, 16.0, 64.0]
SWEEP_SIZES = [(1, 257), (127, 129), (129, 127), (300, 257)]


def _mode1_tol(a, b):
    na, nb = np.linalg.norm(a.astype(np.float64), axis=1), np.linalg.norm(b.astype(np.float64), axis=1)
    return DIST_TOL * np.maximum(1.0, na * (nb.max() if len(nb) else 0.0))


@pytest.mark.gpu
@pytest.mark.parametrize("n0,n1", SWEEP_SIZES)
@pytest.mark.parametrize("c", SWEEP_C)
def test_mode1_scale_sweep(model32, c, n0, n1):
    a, b, thr = _sweep_data(c, n0, n1, seed=int(c * 1024) * 1000 + n0 + 7 * n1)
    d32 = dist32_model(model32, a, b, 1)
    d64 = dist64(a, b, 1)
    tol = _mode1_tol(a, b)
    n_decisive = 0
    for mutual in (True, False):
        res = {}
        for layout in (ROWS, CF):
            got = res[layout] = _match(a, b, layout, thr, mutual, 1)
            ok = _check_contract(got, d32, d64, thr, mutual, tol, f"c={c} layout={layout} mutual={mutual}")
            n_decisive = max(n_decisive, int(ok.sum()))
        # the same descriptors in either layout give the same bits
        for k in ("matches0", "scores0", "counts"):
            assert np.array_equal(res[ROWS][k], res[CF][k]), (k, mutual)
        mat = em.nn_matcher_batches(a.T[None], b.T[None], thr, mutual)
        assert mat.shape == (1, n0 + 1, n1 + 1)
        idx = orc.match_indices(mat[:, :n0, :n1])
        assert np.array_equal(idx, res[CF]["matches0"]), mutual
    assert n_decisive >= n0 // 2                      # the data is mostly decidable in float64


def test_sweep_plants_gaps_between_eps_and_product_error():
    """The sweep's near-ties reach below the fp32 resolution and straddle MATCH_EPS = 1e-4 at large scales."""
    a, b, thr = _sweep_data(16.0, 300, 257, seed=1)
    d64 = dist64(a, b, 1)
    g = _top2_gap(d64, 1)
    assert (g < 1e-5 * 256).sum() >= 3 and ((g > 1e-4) & (g < 1e-2)).sum() >= 3
    assert (np.abs(d64.min(axis=1) - thr) < 1e-2 * 256).sum() >= 5


# ------------------------------------------------------------------ strict threshold on the tensor-core path
@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1])
def test_threshold_equality(model32, mode):
    rng = np.random.default_rng(31 + mode)
    n0, n1 = 150, 140
    if mode == 0:
        b = _unit(rng, n1, 256)
        a = _unit(rng, n0, 256) * 0.6 + b[rng.integers(0, n1, n0)]
        a /= np.linalg.norm(a, axis=1, keepdims=True)
        a, b = a.astype(np.float32), b.astype(np.float32)
    else:
        a, b, _ = _sweep_data(4.0, n0, n1, seed=77)
    d32 = dist32_model(model32, a, b, mode)
    d64 = dist64(a, b, mode)
    tol = np.full(n0, DIST_TOL) if mode == 0 else _mode1_tol(a, b)
    _, idx, nn1 = decisions(d32, np.float32(np.inf), False)
    best = d32[np.arange(n0), idx]
    mutual_rows = np.nonzero(nn1[idx] == np.arange(n0))[0]
    i = int(mutual_rows[np.argmin(np.abs(best[mutual_rows] - np.median(best)))])   # a mutual row mid-range
    v = best[i]
    for thr in (v, np.nextafter(v, np.float32(np.inf)), np.nextafter(v, np.float32(0))):
        for layout in (ROWS, CF):
            for mutual in (True, False):
                got = _match(a, b, layout, thr, mutual, mode)
                _check_contract(got, d32, d64, thr, mutual, tol, f"thr={thr!r} layout={layout} mutual={mutual}")
                assert got["matches0"][i] == (idx[i] if thr > v else -1), (thr, layout, mutual)


# ------------------------------------------------------------------ exact ties at 0 (clip) in both directions
@pytest.mark.gpu
@pytest.mark.parametrize("layout", [ROWS, CF])
def test_clip_and_exact_ties_at_zero(model32, layout):
    rng = np.random.default_rng(3)
    cand = _unit(rng, 400, 256).astype(np.float32)
    self_d = np.array([dist32_model(model32, x[None], x[None], 0)[0, 0] for x in cand])
    zero = cand[self_d == 0.0]                       # fp32 |x|^2 >= 1: 2 - 2s rounds to <= 0 and clips to 0
    assert len(zero) >= 3
    n1 = 200
    b = _unit(rng, n1, 256).astype(np.float32)
    b[5], b[70], b[199] = zero[0], zero[0], zero[0]  # exact duplicate columns
    b[6] = zero[0]
    ch = rng.integers(0, 256, 3)
    b[6, ch] = np.nextafter(b[6, ch], np.float32(0))  # a near-duplicate one ulp off in three channels
    b[130], b[131] = zero[1], zero[1]
    b[129] = zero[2]
    n0 = 130
    a = _unit(rng, n0, 256).astype(np.float32)
    a[3], a[64], a[128] = zero[0], zero[0], zero[0]  # duplicate rows: ties in the column direction
    a[10], a[129] = zero[1], zero[1]
    a[100] = b[6]
    a[11] = zero[2]
    d32 = dist32_model(model32, a, b, 0)
    assert (d32[[3, 10, 11], [5, 130, 129]] == 0).all()
    d64 = dist64(a, b, 0)
    for thr in (np.float32(0.8), np.float32(0.0)):
        for mutual in (True, False):
            got = _match(a, b, layout, thr, mutual, 0)
            _check_contract(got, d32, d64, thr, mutual, DIST_TOL, f"thr={thr} mutual={mutual}")
            if thr > 0:
                assert got["matches0"][3] == 5 and got["matches0"][10] == 130
                assert (got["matches0"][[64, 128, 129]] == (-1 if mutual else [5, 5, 130])).all()
            else:
                assert (got["matches0"] == -1).all()    # a distance of exactly 0 is not < 0


# ------------------------------------------------------------------ descriptor dimension other than 256
def _with_ties(rng, n, d, dup_from=None):
    x = _unit(rng, n, d).astype(np.float32)
    for _ in range(max(1, n // 5)):
        p, q = rng.integers(0, n, 2)
        x[p] = x[q] if dup_from is None else dup_from[rng.integers(0, len(dup_from))]
    return x


def _pack(blocks, layout):
    """Per-pair fp32 rows [n_p, d] -> one buffer: rows back to back, or channel-first [d, n_p] back to back."""
    return np.concatenate([(x if layout == ROWS else x.T).reshape(-1) for x in blocks]) if blocks else np.zeros(0, np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("d", [16, 48, 128, 240, 272, 512])
def test_generic_dimension(model32, d):
    rng = np.random.default_rng(d)
    cases = {"uniform": [(65, 70)] * 3, "ragged": [(1, 37), (70, 1), (129, 65), (33, 200)]}
    for name, sizes in cases.items():
        side1 = [_with_ties(rng, n1, d) for _, n1 in sizes]
        side0 = [_with_ties(rng, n0, d, dup_from=s1) for (n0, _), s1 in zip(sizes, side1)]
        for p in range(len(sizes)):                  # near-ties: a row nudged off a column by 1 ulp in 2 channels
            ch = rng.integers(0, d, 2)
            side0[p][0] = side1[p][-1]
            side0[p][0, ch] = np.nextafter(side0[p][0, ch], np.float32(2))
        d32 = [dist32_model(model32, x, y, 0) for x, y in zip(side0, side1)]
        d64 = [dist64(x, y, 0) for x, y in zip(side0, side1)]
        n0s, n1s = [n for n, _ in sizes], [n for _, n in sizes]
        cu0 = np.concatenate([[0], np.cumsum(n0s)]).astype(np.int32)
        cu1 = np.concatenate([[0], np.cumsum(n1s)]).astype(np.int32)
        for layout in (ROWS, CF):
            x, y = _t(_pack(side0, layout)), _t(_pack(side1, layout))
            for mutual in (True, False):
                for thr in (np.float32(0.8), np.float32(0.3)):
                    kw = dict(n0=sizes[0][0], n1=sizes[0][1]) if name == "uniform" else dict(
                        cu0=_t(cu0), cu1=_t(cu1), max_n0=max(n0s), max_n1=max(n1s))
                    out = _ops.match_descriptors(x, y, layout, len(sizes), float(thr), mutual, d=d, **kw)
                    got = {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in out.items()}
                    for p, (n0, n1) in enumerate(sizes):
                        what = f"{name} pair {p} layout={layout} mutual={mutual} thr={thr}"
                        dk = got["dist_key"][p * got["stride"]:p * got["stride"] + n0 * n1].reshape(n0, n1)
                        assert np.array_equal(dk, d32[p]), what          # fp32 FMA path: bit for bit
                        one = {"matches0": got["matches0"][cu0[p]:cu0[p + 1]], "scores0": got["scores0"][cu0[p]:cu0[p + 1]],
                               "nn1": got["nn1"][cu1[p]:cu1[p + 1]], "counts": got["counts"][p:p + 1]}
                        _check_contract(one, d32[p], d64[p], thr, mutual, DIST_TOL, what)
                        assert np.array_equal(one["scores0"], d32[p].min(axis=1)), what
        # the nn_matcher drop-in, channel-first [d, n], one pair
        for mutual in (True, False):
            mat, dist = nnm.nn_matcher(side0[2].T.copy(), side1[2].T.copy(), 0.8, mutual)
            assert np.array_equal(dist[0], d32[2])
            assert np.array_equal(orc.match_indices(mat), decisions(d32[2], np.float32(0.8), mutual)[0])


@pytest.mark.gpu
@pytest.mark.parametrize("d", [100, 250])
def test_unsupported_dimension(d):
    """The reference accepts any descriptor dimension; the kernels need d % 16 == 0 and refuse the rest."""
    rng = np.random.default_rng(d)
    a, b = _unit(rng, 20, d).astype(np.float32), _unit(rng, 30, d).astype(np.float32)
    hdr = open(os.path.join(ROOT, "include", "linetr_b200.h")).read()
    code = int(re.search(r"#define\s+LTR_E_UNSUPPORTED\s+\((-?\d+)\)", hdr).group(1))
    pattern = f"code {code}\\)"
    with pytest.raises(N.LtrError, match=pattern):
        nnm.nn_matcher(a.T.copy(), b.T.copy(), 0.8, True)
    for layout in (ROWS, CF):
        x, y = (a, b) if layout == ROWS else (a.T, b.T)
        with pytest.raises(N.LtrError, match=pattern):
            _ops.match_descriptors(_t(x), _t(y), layout, 1, 0.8, True, n0=20, n1=30, d=d)


# ------------------------------------------------------------------ empty side in a ragged tensor-core batch
@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1])
def test_empty_side_in_ragged_batch(model32, mode):
    rng = np.random.default_rng(50 + mode)
    sizes = [(1, 128), (0, 129), (257, 0), (128, 257), (129, 1), (0, 0), (257, 128)]
    c = 1.0 if mode == 0 else 16.0
    side1 = [(_unit(rng, n1, 256) * (c if mode else 1.0)).astype(np.float32) for _, n1 in sizes]
    side0 = []
    for (n0, _), s1 in zip(sizes, side1):
        x = _unit(rng, n0, 256) * (0.5 * c)
        if len(s1):
            x += s1[rng.integers(0, len(s1), n0)]
        if mode == 0:
            x /= np.linalg.norm(x, axis=1, keepdims=True)
        side0.append(x.astype(np.float32))
    n0s, n1s = [n for n, _ in sizes], [n for _, n in sizes]
    cu0 = np.concatenate([[0], np.cumsum(n0s)]).astype(np.int32)
    cu1 = np.concatenate([[0], np.cumsum(n1s)]).astype(np.int32)
    thr = np.float32(0.8 if mode == 0 else 0.5 * c * c)
    for layout in (ROWS, CF):
        for mutual in (True, False):
            out = _ops.match_descriptors(_t(_pack(side0, layout)), _t(_pack(side1, layout)), layout, len(sizes),
                                         float(thr), mutual, cu0=_t(cu0), cu1=_t(cu1), max_n0=max(n0s),
                                         max_n1=max(n1s), want_dist=False, dist_mode=mode)
            got = {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in out.items()}
            for p, (n0, n1) in enumerate(sizes):
                what = f"pair {p} ({n0} x {n1}) layout={layout} mutual={mutual}"
                m0, s0 = got["matches0"][cu0[p]:cu0[p + 1]], got["scores0"][cu0[p]:cu0[p + 1]]
                nn1 = got["nn1"][cu1[p]:cu1[p + 1]]
                if n0 == 0 or n1 == 0:
                    assert (m0 == -1).all() and np.isinf(s0).all() and got["counts"][p] == 0, what
                    if mutual:
                        assert (nn1 == -1).all(), what
                    continue
                one = _match(side0[p], side1[p], layout, thr, mutual, mode)
                assert np.array_equal(m0, one["matches0"]) and np.array_equal(s0, one["scores0"]), what
                assert got["counts"][p] == one["counts"][0], what
                if mutual:
                    assert np.array_equal(nn1, one["nn1"]), what
                d32 = dist32_model(model32, side0[p], side1[p], mode)
                assert np.array_equal(m0, decisions(d32, thr, mutual)[0]), what
