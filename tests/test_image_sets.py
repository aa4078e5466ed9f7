"""Image sets: `PairEngine.encode_images` encodes every image once and `match_sets` matches any list of image pairs
between two encoded sets (`ltr_image_tiles` + `ltr_match_indexed`), against `match_images`, the numpy oracle and
`ltr_match` on descriptors gathered per pair."""
import ctypes
import os

import numpy as np
import pytest
import torch

from linetr_b200 import _native as N, _ops, engine, line_process as LP, synthetic as syn
from linetr_b200.match_io import dense_to_indices
from tests import helpers as H
from tests.test_image_pairs import DIST_TOL, _glue, _model, _reference_superpoint

DEV = torch.device("cuda", 0)


# ------------------------------------------------------------------ CPU
def test_exhaustive_pairs():
    for n in range(6):
        got = engine.exhaustive_pairs(n)
        assert got.dtype == np.int32 and got.shape == (n * (n - 1) // 2, 2)
        assert [tuple(r) for r in got] == [(i, j) for i in range(n) for j in range(i + 1, n)]


def test_pair_validation():
    ok = engine.check_pairs(np.array([[0, 2], [3, 0]], dtype=np.int64), 4, 3)
    assert ok.dtype == np.int32 and ok.tolist() == [[0, 2], [3, 0]]
    assert engine.check_pairs([], 2, 2).shape == (0, 2)
    assert engine.check_pairs(np.zeros((0, 2), dtype=np.int32), 0, 0).shape == (0, 2)
    for bad, what in [(np.zeros((3,), dtype=np.int32), "shape"), (np.zeros((2, 3), dtype=np.int32), "shape"),
                      (np.zeros((1, 2, 2), dtype=np.int32), "shape"), (np.zeros((2, 2), dtype=np.float32), "integers"),
                      (np.array([[0, -1]]), "negative"), (np.array([[-1, 0]]), "negative"),
                      (np.array([[4, 0]]), r"pairs\[:, 0\]"), (np.array([[0, 3]]), r"pairs\[:, 1\]")]:
        with pytest.raises(N.LtrError, match=what):
            engine.check_pairs(bad, 4, 3)


def _chunk_cost(n0, n1, a, b):
    return (b - a) * int(np.max(n0[a:b])) * int(np.max(n1[a:b])) * 4


def test_chunk_planning():
    rng = np.random.default_rng(3)
    n0, n1 = rng.integers(0, 300, 500), rng.integers(0, 300, 500)
    n0[123], n1[123] = 5000, 5000                       # one pair alone over the cap
    cap = 40 << 20
    chunks = engine.plan_chunks(n0, n1, cap)
    assert chunks[0][0] == 0 and chunks[-1][1] == len(n0)
    assert all(a < b for a, b in chunks) and all(chunks[i][1] == chunks[i + 1][0] for i in range(len(chunks) - 1))
    assert (123, 124) in chunks
    for a, b in chunks:
        assert b - a == 1 or _chunk_cost(n0, n1, a, b) <= cap
        if b < len(n0) and (a, b) != (123, 124) and b != 123:   # greedy: the next pair would not have fitted
            assert _chunk_cost(n0, n1, a, b + 1) > cap
    assert engine.plan_chunks(n0, n1, 1 << 40) == [(0, 500)]
    assert engine.plan_chunks(n0, n1, 1 << 40, max_pairs=200) == [(0, 200), (200, 400), (400, 500)]
    assert engine.plan_chunks(np.zeros(0), np.zeros(0)) == []


def test_make_image_set_deterministic():
    a, b = syn.make_image_set(5, 3, 20, 30), syn.make_image_set(5, 3, 20, 30)
    c = syn.make_image_set(6, 3, 20, 30)
    assert len(a) == 3
    for x, y in zip(a, b):
        for k in ("keypoints", "descriptors", "dense_descriptor", "dense_score", "scores"):
            assert torch.equal(x[k], y[k]), k
        assert [vars(l) for l in x["klines"]] == [vars(l) for l in y["klines"]]
    assert not torch.equal(a[0]["descriptors"], c[0]["descriptors"])
    assert not torch.equal(a[0]["descriptors"], a[1]["descriptors"])   # the views differ from each other


# ------------------------------------------------------------------ GPU helpers
def _dev(im):
    return syn.image_to(im, DEV)


def _length(kl):
    return float(np.hypot(kl.endPointX - kl.startPointX, kl.endPointY - kl.startPointY))


def _ragged_set():
    """Seven views of one scene: 0 without key lines, 1 without keypoints, 2 with long (split) lines, 3 with exactly
    128 lines, 4 with more than 128 lines (two tiles), 5 and 6 ordinary; only view 2 splits a key line."""
    views = syn.make_image_set(41, 7, 420, 300)
    short = [i for i, kl in enumerate(views[2]["klines"]) if _length(kl) < 140]
    assert len(short) > 200
    views[0]["klines"] = []
    views[1]["keypoints"] = torch.zeros(0, 2)
    views[1]["descriptors"] = torch.zeros(256, 0)
    for v, n in ((1, 60), (3, 129), (4, len(short)), (5, 90), (6, 150)):   # max_keylines -1 drops the shortest line
        views[v]["klines"] = [views[v]["klines"][i] for i in short[:n]]
    return [_dev(v) for v in views]


def _prep_counts(model, images):
    specs = [(im["klines"], tuple(im["image_shape"]), None) for im in images]
    host = LP.prepare_tokenizer_batch(specs, [LP.tokenizer_config(model.config, sh, True) for _, sh, _ in specs])
    return np.diff(host.cu_lines), np.diff(host.cuk)


def _dist_blocks(dist, stride, n0, n1):
    """The written part of per-pair distance matrices (pair p at p * stride, [n0[p], n1[p]])."""
    return [dist[p * stride:p * stride + int(a) * int(b)] for p, (a, b) in enumerate(zip(n0, n1))]


def _assert_pair_equal(res, p, want, q, scores=True):
    assert torch.equal(res.pair_lines(p).cpu(), want.pair_lines(q).cpu()), p
    assert torch.equal(res.pair_points(p).cpu(), want.pair_points(q).cpu()), p
    assert int(res.counts_l[p]) == int(want.counts_l[q]) and int(res.counts_p[p]) == int(want.counts_p[q]), p
    if scores:
        a, b = res.reference_dict(p), want.reference_dict(q)
        for k in a:
            assert a[k].shape == b[k].shape, (p, k)
            if a[k].numel():
                assert np.abs(a[k].numpy() - b[k].numpy()).max() <= DIST_TOL, (p, k)
                assert torch.equal(a[k], b[k]), (p, k)   # the same kernels on the same operands: bit-equal


# ------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_match_sets_equal_match_images_and_oracle():
    from oracle import linetr_oracle as orc
    model, sd = _model()
    eng = engine.PairEngine(model, DEV)
    images = _ragged_set()
    sub, key = _prep_counts(model, images)
    assert sub[0] == 0 and sub[3] == 128 and sub[4] > 128 and sub[2] > key[2] > 128
    assert all(sub[i] == key[i] for i in range(7) if i != 2)
    iset = eng.encode_images(images)
    assert len(iset) == 7 and iset.tile_off_l.tolist()[:5] == [0, 0, 1, 1 + int(-(-sub[2] // 128)), 2 + int(-(-sub[2] // 128))]
    ex = engine.exhaustive_pairs(7)
    pairs_a = np.concatenate([ex, [[i, i] for i in range(7)], ex[::5, ::-1], [[3, 4], [3, 4]]]).astype(np.int32)
    pairs_b = pairs_a[(pairs_a != 2).all(axis=1)]      # no image with split lines: no key-line merging
    checked_oracle = 0
    for pairs, merged in ((pairs_a, True), (pairs_b, False)):
        res = eng.match_set(iset, pairs, want_scores=True)
        for p, (i, j) in enumerate(pairs):   # image 0 has no key lines, image 1 no keypoints
            if 0 in (i, j):
                assert int(res.counts_l[p]) == 0 and (res.pair_lines(p) == -1).all()
            if 1 in (i, j):
                assert int(res.counts_p[p]) == 0 and (res.pair_points(p) == -1).all()
        assert res.n_pairs == len(pairs)
        batched = eng.match_images([images[i] for i, _ in pairs], [images[j] for _, j in pairs], want_scores=True)
        for p, (i, j) in enumerate(pairs):
            _assert_pair_equal(res, p, batched, p)
            # one pair alone merges key lines iff one of its images splits one: where that agrees with the call
            single = eng.match_images([images[i]], [images[j]], want_scores=True)
            if ((i == 2) or (j == 2)) == merged:
                _assert_pair_equal(res, p, single, 0)
            else:
                assert torch.equal(res.pair_points(p).cpu(), single.pair_points(0).cpu()), p
            if checked_oracle < 6 and len(res.klines0[p]) and len(res.klines1[p]) and i != j:
                sides = []
                for im in (images[i], images[j]):
                    shape = im["image_shape"]
                    c = LP.tokenizer_config(model.config, shape, True)
                    d = _glue(im["klines"], shape, {k: im[k].cpu() for k in ("dense_descriptor", "dense_score")},
                              {k: c[k] for k in ("min_length", "token_distance")})
                    sides.append({k: v.numpy() for k, v in d.items()})
                omat, odk, _, _ = orc.match_pair(sd, sides[0], sides[1], 0.8)
                dec = H.decisive_rows(odk[0], 0.8, 2e-3)
                assert np.array_equal(res.pair_lines(p).cpu().numpy()[dec], orc.match_indices(omat)[dec]), p
                checked_oracle += 1
        assert int(res.counts_l.sum()) > 0 and int(res.counts_p.sum()) > 0
    empty = eng.match_set(iset, [])
    assert empty.n_pairs == 0 and empty.matches_l.numel() == 0
    none = eng.encode_images([])
    assert len(none) == 0 and eng.match_set(none, np.zeros((0, 2), np.int32)).n_pairs == 0


@pytest.mark.gpu
def test_anchor_set_against_frames():
    model, _ = _model()
    eng = engine.PairEngine(model, DEV)
    views = [_dev(v) for v in syn.make_image_set(52, 6, 120, 400)]
    anchor, frames = eng.encode_images(views[:1]), eng.encode_images(views[1:])
    pairs = np.array([[0, j] for j in range(5)], dtype=np.int32)
    res = eng.match_sets(anchor, frames, pairs, want_scores=True)
    want = eng.match_images([views[0]] * 5, views[1:], want_scores=True)
    for p in range(5):
        _assert_pair_equal(res, p, want, p)
    assert all(int(res.counts_l[p]) > 0 and int(res.counts_p[p]) > 0 for p in range(5))
    with pytest.raises(N.LtrError, match="out of range"):
        eng.match_sets(anchor, frames, [[1, 0]])


def _near_tie_points(seed, n=200):
    """Point descriptors [256, n] of two images whose nearest neighbours include exact duplicates (both images) and
    near ties (distance gaps of 2e-5 .. 8e-5): every such row goes through the matcher's fp32 re-check."""
    rng = np.random.default_rng(seed)
    unit = lambda v: v / np.linalg.norm(v, axis=-1, keepdims=True)
    a = unit(rng.standard_normal((n, 256)))
    b = unit(a + 0.05 * rng.standard_normal((n, 256)))
    b[10:20] = b[0:10]                      # duplicated columns of image 1: exact ties
    a[30:35] = a[40:45]                     # duplicated rows of image 0: exact column ties
    for r in range(50, 60):                 # near ties: a second partner slightly farther than the first
        v = unit(rng.standard_normal(256))
        for dl in np.geomspace(1e-4, 1e-1, 200):
            c = unit(b[r] + dl * v)
            gap = (2 - 2 * a[r] @ c) - (2 - 2 * a[r] @ b[r])
            if 2e-5 <= gap <= 8e-5:
                b[r + 100] = c
                break
    return (torch.from_numpy(np.ascontiguousarray(a.T, dtype=np.float32)),
            torch.from_numpy(np.ascontiguousarray(b.T, dtype=np.float32)))


@pytest.mark.gpu
def test_exact_path_under_indexing():
    from oracle import linetr_oracle as orc
    model, _ = _model()
    eng = engine.PairEngine(model, DEV)
    views = syn.make_image_set(63, 2, 60, 200)
    da, db = _near_tie_points(7)
    views[0]["descriptors"], views[1]["descriptors"] = da, db
    views = [_dev(v) for v in views]
    pairs = np.array([[0, 1], [1, 0], [0, 0], [0, 1]], dtype=np.int32)
    res = eng.match_set(eng.encode_images(views), pairs)
    want = eng.match_images([views[i] for i, _ in pairs], [views[j] for _, j in pairs])
    for p, (i, j) in enumerate(pairs):
        _assert_pair_equal(res, p, want, p, scores=False)
        a, b = views[i]["descriptors"].cpu().numpy(), views[j]["descriptors"].cpu().numpy()
        omat = orc.nn_matcher(a.astype(np.float64), b.astype(np.float64), 0.7, True)[0]
        assert np.array_equal(res.pair_points(p).cpu().numpy(), dense_to_indices(omat)), p
    assert int(res.counts_p[0]) > 100


def _pool(rng, counts):
    descs = [rng.standard_normal((n, 256)).astype(np.float32) for n in counts]
    descs = [d / np.linalg.norm(d, axis=1, keepdims=True) for d in descs]
    return descs


def _flat(descs, layout):
    if layout == N.LAYOUT_ROWS:
        return torch.from_numpy(np.concatenate(descs or [np.zeros((0, 256), np.float32)]).reshape(-1, 256)).to(DEV)
    return torch.from_numpy(np.concatenate([d.T.reshape(-1) for d in descs] or [np.zeros(0, np.float32)])).to(DEV)


def _csr(rng, n):
    """Key lines of n sublines: groups of 1..3 consecutive sublines -> local offsets."""
    o = [0]
    while o[-1] < n:
        o.append(min(n, o[-1] + int(rng.integers(1, 4))))
    return np.array(o, dtype=np.int64)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", [N.LAYOUT_ROWS, N.LAYOUT_CHANNEL_FIRST])
@pytest.mark.parametrize("merge", [False, True])
def test_match_indexed_equals_gathered_match(layout, merge):
    rng = np.random.default_rng(11 + 2 * layout + merge)
    counts0, counts1 = [0, 37, 128, 200, 5, 129], [64, 0, 250, 17, 128]
    d0 = _pool(rng, counts0)
    d1 = []   # noisy copies of image 3 of pool 0 (then random rows): true matches exist
    for n in counts1:
        x = d0[3][:min(n, 200)] + 0.04 * rng.standard_normal((min(n, 200), 256)).astype(np.float32)
        x = np.concatenate([x, rng.standard_normal((n - len(x), 256)).astype(np.float32)])
        d1.append((x / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), 1e-12)).astype(np.float32))
    pairs = np.array([[i, j] for i in range(6) for j in range(5)] + [[3, 2], [2, 4], [3, 2]], dtype=np.int32)
    P = len(pairs)
    i32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(DEV)
    pref = lambda c: np.concatenate([[0], np.cumsum(c)]).astype(np.int64)
    cu0, cu1 = pref(counts0), pref(counts1)
    csr0 = [_csr(rng, n) for n in counts0] if merge else [np.arange(n + 1) for n in counts0]
    csr1 = [_csr(rng, n) for n in counts1] if merge else [np.arange(n + 1) for n in counts1]
    nk0, nk1 = np.array([len(c) - 1 for c in csr0]), np.array([len(c) - 1 for c in csr1])
    cuk0, cuk1 = pref(nk0), pref(nk1)
    so = lambda csr, cu: np.concatenate([c[:-1] + b for c, b in zip(csr, cu[:-1])] + [[cu[-1]]])
    # indexed
    to0, to1 = _ops.tile_offsets(cu0), _ops.tile_offsets(cu1)
    f0, f1 = _flat(d0, layout), _flat(d1, layout)
    t0 = _ops.image_tiles(f0, layout, cu0, i32(cu0), i32(to0), int(to0[-1]))
    t1 = _ops.image_tiles(f1, layout, cu1, i32(cu1), i32(to1), int(to1[-1]))
    k0, k1 = nk0[pairs[:, 0]], nk1[pairs[:, 1]]
    ol0, ol1 = pref(k0), pref(k1)
    mk0, mk1 = int(k0.max()), int(k1.max())
    out = dict(matches0=torch.empty(int(ol0[-1]), dtype=torch.int32, device=DEV),
               scores0=torch.empty(int(ol0[-1]), device=DEV), nn1=torch.empty(int(ol1[-1]), dtype=torch.int32, device=DEV),
               counts=torch.empty(P, dtype=torch.int32, device=DEV), dist_key=torch.empty(P * mk0 * mk1, device=DEV))
    kw = dict(cu0=i32(cu0), cu1=i32(cu1), max_n0=max(counts0), max_n1=max(counts1), img0=i32(pairs[:, 0]),
              img1=i32(pairs[:, 1]), tiles0=t0, tiles1=t1, tile_off0=i32(to0), tile_off1=i32(to1),
              n_tiles0=int(to0[-1]), n_tiles1=int(to1[-1]), out_off0=i32(ol0), out_off1=i32(ol1),
              total_out0=int(ol0[-1]), total_out1=int(ol1[-1]), dist_stride=mk0 * mk1, **out)
    if merge:
        kw.update(sub_off0=i32(so(csr0, cu0)), sub_off1=i32(so(csr1, cu1)), cuk0=i32(cuk0), cuk1=i32(cuk1),
                  max_k0=int(nk0.max()), max_k1=int(nk1.max()))
    _ops.match_indexed(f0, f1, layout, P, 0.8, **kw)
    # gathered per pair
    g0, g1 = [d0[i] for i, _ in pairs], [d1[j] for _, j in pairs]
    gc0, gc1 = pref([len(x) for x in g0]), pref([len(x) for x in g1])
    gkw = dict(cu0=i32(gc0), cu1=i32(gc1), max_n0=int(np.diff(gc0).max()), max_n1=int(np.diff(gc1).max()),
               total_k0=int(ol0[-1]), total_k1=int(ol1[-1]))
    if merge:
        gcs0, gcs1 = [csr0[i] for i, _ in pairs], [csr1[j] for _, j in pairs]
        gkw.update(sub_off0=i32(so(gcs0, gc0)), sub_off1=i32(so(gcs1, gc1)), cuk0=i32(ol0), cuk1=i32(ol1),
                   max_k0=mk0, max_k1=mk1)
    want = _ops.match_descriptors(_flat(g0, layout), _flat(g1, layout), layout, P, 0.8, True, d=256, want_dist=True, **gkw)
    assert torch.equal(out["matches0"], want["matches0"])
    assert torch.equal(out["scores0"], want["scores0"])
    assert torch.equal(out["counts"], want["counts"])
    assert want["stride"] == mk0 * mk1
    for a, b in zip(_dist_blocks(out["dist_key"], mk0 * mk1, k0, k1), _dist_blocks(want["dist_key"], mk0 * mk1, k0, k1)):
        assert torch.equal(a, b)
    assert int(out["counts"].sum()) > 0


@pytest.mark.gpu
def test_match_indexed_rejects_unsupported_modes():
    t = torch.zeros(64, device=DEV)
    z = torch.zeros(4, dtype=torch.int32, device=DEV)
    lib = N.load()
    inp = N.LtrMatchInput(t.data_ptr(), t.data_ptr(), 0, 256, 1, 0, 0, z.data_ptr(), z.data_ptr(), None, None, None, None,
                          1, 1, 0, 0, 0, 0.8, 1, 1, 1, 1, None, None, 0, 0, 0, 0)
    idx = N.LtrPairIndex(z.data_ptr(), z.data_ptr(), t.data_ptr(), t.data_ptr(), z.data_ptr(), z.data_ptr(), 1, 1,
                         z.data_ptr(), z.data_ptr(), 1, 1)
    o = N.LtrMatchOutput(z.data_ptr(), t.data_ptr(), z.data_ptr(), z.data_ptr(), None, None, t.data_ptr(), 256, None)
    assert lib.ltr_match_indexed(ctypes.byref(inp), ctypes.byref(idx), ctypes.byref(o), 0, None) == -4   # dist_mode 1
    gather = N.LtrPeerGather(None, None, 0, 2, 0, 1)
    inp.dist_mode = 0
    o.gather = ctypes.pointer(gather)
    assert lib.ltr_match_indexed(ctypes.byref(inp), ctypes.byref(idx), ctypes.byref(o), 0, None) == -4


@pytest.mark.gpu
def test_match_sets_chunking_is_invisible(monkeypatch):
    model, _ = _model()
    eng = engine.PairEngine(model, DEV)
    views = [_dev(v) for v in syn.make_image_set(71, 6, 150, 300)]
    iset = eng.encode_images(views)
    pairs = np.concatenate([engine.exhaustive_pairs(6), [[2, 2], [5, 1]]]).astype(np.int32)
    one = eng.match_set(iset, pairs, want_scores=True)
    n = np.diff(iset.cu_lines)[pairs]
    cap = 3 * int(n.max()) ** 2 * 4
    assert len(engine.plan_chunks(n[:, 0], n[:, 1], cap)) > 3
    monkeypatch.setattr(engine, "DIST_SUB_CAP", cap)
    chunked = eng.match_set(iset, pairs, want_scores=True)
    for k in ("matches_l", "scores_l", "counts_l", "matches_p", "scores_p", "counts_p"):
        assert torch.equal(getattr(one, k), getattr(chunked, k)), k
    assert np.array_equal(one.offsets_l, chunked.offsets_l) and np.array_equal(one.offsets_p, chunked.offsets_p)
    assert one.stride_l == chunked.stride_l and one.stride_p == chunked.stride_p
    k, q = np.diff(iset.cuk)[pairs], np.diff(iset.cu_points)[pairs]
    for dist, stride, c in (("dist_l", one.stride_l, k), ("dist_p", one.stride_p, q)):
        for a, b in zip(_dist_blocks(getattr(one, dist), stride, c[:, 0], c[:, 1]),
                        _dist_blocks(getattr(chunked, dist), stride, c[:, 0], c[:, 1])):
            assert torch.equal(a, b), dist


def _launches(fn):
    fn()                                       # warm-up: weight packing, workspaces
    torch.cuda.synchronize()
    N.reset_launch_count()
    fn()
    torch.cuda.synchronize()
    return N.launch_count()


@pytest.mark.gpu
def test_launch_counts():
    model, _ = _model()
    eng = engine.PairEngine(model, DEV)
    views = [_dev(v) for v in syn.make_image_set(81, 16, 80, 200)]
    enc = [_launches(lambda: eng.encode_images(views[:n])) for n in (4, 16)]
    assert enc[0] == enc[1] > 0, enc
    s4, s16 = eng.encode_images(views[:4]), eng.encode_images(views)
    pairs = engine.exhaustive_pairs(4)
    by_p = [_launches(lambda: eng.match_set(s16, np.tile(pairs, (r, 1)))) for r in (1, 5)]
    assert by_p[0] == by_p[1] > 0, by_p
    assert _launches(lambda: eng.match_set(s4, pairs)) == by_p[0]


@pytest.mark.gpu
def test_encode_and_match_never_synchronise():
    model, _ = _model()
    eng = engine.PairEngine(model, DEV)
    images = _ragged_set()
    pairs = np.concatenate([engine.exhaustive_pairs(7), [[4, 4]]]).astype(np.int32)
    want = eng.match_set(eng.encode_images(images), pairs)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = eng.match_set(eng.encode_images(images), pairs)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for k in ("matches_l", "scores_l", "counts_l", "matches_p", "scores_p", "counts_p"):
        assert torch.equal(getattr(got, k), getattr(want, k)), k


@pytest.mark.gpu
def test_real_images_as_one_set():
    """The eight bundled images as one set, pairs (2k, 2k+1), against match_images on the four bundled pairs."""
    pytest.importorskip("cv2")
    from tests.golden.make_plumbing_golden import ShimLSD, read_image
    model, _ = _model("shipped")
    sp = _reference_superpoint()
    lsd = ShimLSD({"n_octave": 2})
    _, meta = H.plumbing()
    images = []
    with torch.no_grad():
        for info in meta["pairs"]:
            for name in info["names"]:
                im = read_image(os.path.join(H.REF_DIR, "assets", name))
                images.append({"klines": lsd.detect_torch(im), "image_shape": tuple(im.shape), **sp({"image": im.to(DEV)})})
    eng = engine.PairEngine(model, DEV)
    res = eng.match_set(eng.encode_images(images), np.array([[2 * k, 2 * k + 1] for k in range(4)], dtype=np.int32),
                        want_scores=True)
    want = eng.match_images(images[0::2], images[1::2], want_scores=True)
    for p in range(4):
        _assert_pair_equal(res, p, want, p)
        assert int(res.counts_l[p]) > 0 and int(res.counts_p[p]) > 0
