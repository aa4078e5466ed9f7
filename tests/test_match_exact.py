"""The exact re-check of the tensor-core matcher (match_exact_kernel) when every line needs it.

Descriptors are built so that every line of both sides has exact ties or 1-ulp near-ties among its candidates: each
side is made of small groups of duplicated or nudged copies.  Every decision then comes from the ascending-k fp32
FMA chains, and indices, scores, counts and nn1 must equal the host model of that arithmetic bit for bit."""
import numpy as np
import pytest
import torch

from linetr_b200 import _native as N
from linetr_b200 import _ops, eval_matcher as em
from tests.test_matcher_edges import decisions, dist32_model, model32  # noqa: F401  (model32 is a fixture)

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ROWS, CF = N.LAYOUT_ROWS, N.LAYOUT_CHANNEL_FIRST


def _unit(x):
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def _copies(rng, base, n):
    """n lines cycling through `base` rows, every second copy nudged by 1 ulp in 3 channels."""
    out = base[np.arange(n) % len(base)].copy()
    for i in range(len(base), n, 2):
        k = rng.integers(0, 256, 3)
        out[i, k] = np.nextafter(out[i, k], np.float32(1.0))
    return out


def flagged_pair(seed, n0, n1, scale=1.0):
    """Side 1: copies of max(1, n1 // 3) unit vectors; side 0: copies of noisy versions of them.  Rows [n, 256]."""
    rng = np.random.default_rng(seed)
    k1, k0 = max(1, n1 // 3), max(1, n0 // 3)
    base = _unit(rng.standard_normal((k1, 256)))
    noisy = _unit(base[np.arange(k0) % k1] + 0.1 * rng.standard_normal((k0, 256)))
    s = np.float32(scale)
    return _copies(rng, noisy, n0) * s, _copies(rng, base, n1) * s


def _thresholds(dist):
    """A threshold inside the rows' best distances, 3e-5 (well within MATCH_EPS) above an exact one, and a loose one."""
    best = np.sort(dist.min(axis=1))
    return [float(np.nextafter(best[len(best) // 2], np.float32(np.inf)) + np.float32(3e-5) * max(1.0, float(best[-1]))),
            float(best[-1]) * 1.5 + 0.1]


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(DEV)


def _check_scores(scores, dist, idx, thr):
    """Bit-exact where the line took the exact path.  With a single column a row has no near-tie and keeps its
    tensor-core distance unless it lies next to the threshold."""
    exact = dist[np.arange(len(dist)), idx]
    if dist.shape[1] > 1:
        assert np.array_equal(scores.view(np.uint32), exact.view(np.uint32)), thr
    else:
        assert np.abs(scores - exact).max() < 2e-5, thr


def _check(out, dist, thr, mutual):
    want, idx, nn1 = decisions(dist, thr, mutual)
    n0 = dist.shape[0]
    assert np.array_equal(out["matches0"].cpu().numpy(), want), (thr, mutual)
    _check_scores(out["scores0"].cpu().numpy(), dist, idx, thr)
    assert int(out["counts"][0]) == int((want >= 0).sum())
    if mutual:
        assert np.array_equal(out["nn1"].cpu().numpy(), nn1), (thr, mutual)


@pytest.mark.parametrize("n0,n1", [(1, 1), (127, 129), (128, 128), (300, 700), (1030, 1030)])
@pytest.mark.parametrize("layout", [ROWS, CF])
def test_every_line_flagged_mode0(model32, n0, n1, layout):
    a, b = flagged_pair(31 * n0 + n1, n0, n1)
    dist = dist32_model(model32, a, b, 0)
    x, y = (a, b) if layout == ROWS else (a.T, b.T)
    for thr in _thresholds(dist):
        for mutual in (True, False):
            out = _ops.match_descriptors(_dev(x), _dev(y), layout, 1, thr, mutual, n0=n0, n1=n1, want_dist=False)
            _check(out, dist, thr, mutual)


@pytest.mark.parametrize("scale", [1 / 16, 1.0, 4.0, 16.0])
@pytest.mark.parametrize("layout", [ROWS, CF])
def test_every_line_flagged_mode1(model32, scale, layout):
    n0, n1 = 200, 131
    a, b = flagged_pair(int(scale * 64) + layout, n0, n1, scale)
    dist = dist32_model(model32, a, b, 1)
    x, y = (a, b) if layout == ROWS else (a.T, b.T)
    for thr in _thresholds(dist):
        for mutual in (True, False):
            out = _ops.match_descriptors(_dev(x), _dev(y), layout, 1, thr, mutual, n0=n0, n1=n1, want_dist=False,
                                         dist_mode=1)
            _check(out, dist, thr, mutual)


@pytest.mark.parametrize("scale", [1 / 16, 16.0])
def test_every_line_flagged_eval_matcher(model32, scale):
    a, b = flagged_pair(5, 90, 140, scale)
    dist = dist32_model(model32, a, b, 1)
    for thr in _thresholds(dist):
        for mutual in (True, False):
            mat = em.nn_matcher(a.T.copy(), b.T.copy(), thr, mutual)
            got = np.where(mat.any(axis=1), mat.argmax(axis=1), -1)
            assert np.array_equal(got, decisions(dist, thr, mutual)[0]), (scale, thr, mutual)


def test_every_line_flagged_indexed(model32):
    """A pair list over two image pools with repeated images: equal to the gathered batch, and to the host model."""
    counts0, counts1 = [130, 7, 300], [129, 260, 1]
    pool0, pool1 = [], []
    for i, (n0, n1) in enumerate(zip(counts0, counts1)):
        a, b = flagged_pair(100 + i, n0, n1)
        pool0.append(a)
        pool1.append(b)
    pairs = np.array([[0, 0], [0, 1], [2, 1], [1, 0], [0, 0], [2, 2]], dtype=np.int32)
    P = len(pairs)
    i32 = lambda v: torch.from_numpy(np.ascontiguousarray(v, dtype=np.int32)).to(DEV)
    pref = lambda c: np.concatenate([[0], np.cumsum(c)]).astype(np.int64)
    cu0, cu1 = pref(counts0), pref(counts1)
    to0, to1 = _ops.tile_offsets(cu0), _ops.tile_offsets(cu1)
    f0, f1 = _dev(np.concatenate(pool0)), _dev(np.concatenate(pool1))
    t0 = _ops.image_tiles(f0, ROWS, cu0, i32(cu0), i32(to0), int(to0[-1]))
    t1 = _ops.image_tiles(f1, ROWS, cu1, i32(cu1), i32(to1), int(to1[-1]))
    k0, k1 = np.array(counts0)[pairs[:, 0]], np.array(counts1)[pairs[:, 1]]
    ol0, ol1 = pref(k0), pref(k1)
    g0, g1 = [pool0[i] for i, _ in pairs], [pool1[j] for _, j in pairs]
    dists = [dist32_model(model32, x, y, 0) for x, y in zip(g0, g1)]
    thr = _thresholds(dists[0])[0]
    for mutual in (True, False):
        out = dict(matches0=torch.empty(int(ol0[-1]), dtype=torch.int32, device=DEV),
                   scores0=torch.empty(int(ol0[-1]), device=DEV),
                   nn1=torch.full((int(ol1[-1]),), -7, dtype=torch.int32, device=DEV),
                   counts=torch.empty(P, dtype=torch.int32, device=DEV))
        _ops.match_indexed(f0, f1, ROWS, P, thr, cu0=i32(cu0), cu1=i32(cu1), max_n0=max(counts0), max_n1=max(counts1),
                           img0=i32(pairs[:, 0]), img1=i32(pairs[:, 1]), tiles0=t0, tiles1=t1, tile_off0=i32(to0),
                           tile_off1=i32(to1), n_tiles0=int(to0[-1]), n_tiles1=int(to1[-1]), out_off0=i32(ol0),
                           out_off1=i32(ol1), total_out0=int(ol0[-1]), total_out1=int(ol1[-1]), mutual=mutual, **out)
        want = _ops.match_descriptors(_dev(np.concatenate(g0)), _dev(np.concatenate(g1)), ROWS, P, thr, mutual,
                                      cu0=i32(ol0), cu1=i32(ol1), max_n0=int(k0.max()), max_n1=int(k1.max()),
                                      total_k0=int(ol0[-1]), total_k1=int(ol1[-1]), want_dist=False)
        for k in ("matches0", "scores0", "counts") + (("nn1",) if mutual else ()):
            assert torch.equal(out[k], want[k]), (k, mutual)
        m, s = out["matches0"].cpu().numpy(), out["scores0"].cpu().numpy()
        for p, dist in enumerate(dists):
            w, idx, _ = decisions(dist, thr, mutual)
            assert np.array_equal(m[ol0[p]:ol0[p + 1]], w), (p, mutual)
            _check_scores(s[ol0[p]:ol0[p + 1]], dist, idx, thr)
