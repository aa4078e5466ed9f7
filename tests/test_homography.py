"""RANSAC homographies from line and point matches (`ltr_homography`, `geometry.estimate_homographies`) against the
numpy model `geometry.ransac_homography_host`, OpenCV and known homographies."""
import numpy as np
import pytest
import torch

from linetr_b200 import _native as N, engine, geometry as G, synthetic as syn

DEV = torch.device("cuda", 0)
SHAPE = (480, 640)


def _host(d, **kw):
    return G.ransac_homography_host(d["kpts0"], d["kpts1"], d["matches_p"], d["klines0"], d["klines1"], d["matches_l"],
                                    **kw)


def _rel(a, b):
    a, b = np.asarray(a) / np.asarray(a)[2, 2], np.asarray(b) / np.asarray(b)[2, 2]
    return float(np.abs(a - b).max() / np.abs(b).max())


# ------------------------------------------------------------------ CPU
def test_splitmix64_and_samples():
    assert int(G.splitmix64(np.zeros(1, dtype=np.uint64))[0]) == 0xE220A8397B1DCDAF   # splitmix64's first output, seed 0
    for n in (4, 5, 37, 1000):
        idx, ok = G.draw_samples(7, 3, 512, n)
        assert ok.all() and idx.min() >= 0 and idx.max() < n
        assert all(len(set(r)) == 4 for r in idx.tolist())
    a, _ = G.draw_samples(7, 3, 64, 100)
    assert not np.array_equal(a, G.draw_samples(8, 3, 64, 100)[0])
    assert not np.array_equal(a, G.draw_samples(7, 4, 64, 100)[0])
    assert np.array_equal(a[:16], G.draw_samples(7, 3, 16, 100)[0])   # counter-based: no state across hypotheses


def _pixel_rows(pts, s0, s1):
    """Unnormalised equations of the same correspondences (independent of the model's normalisation)."""
    rows = []
    for x, y, u, v in np.asarray(pts, dtype=np.float64):
        rows += [[x, y, 1, 0, 0, 0, -u * x, -u * y, -u], [0, 0, 0, x, y, 1, -v * x, -v * y, -v]]
    for a, b in zip(np.asarray(s0, dtype=np.float64), np.asarray(s1, dtype=np.float64)):
        l = np.cross([*b[0], 1.0], [*b[1], 1.0])
        for x, y in a:
            rows.append([l[0] * x, l[0] * y, l[0], l[1] * x, l[1] * y, l[1], l[2] * x, l[2] * y, l[2]])
    return np.array(rows)


@pytest.mark.parametrize("n_p,n_l", [(4, 0), (0, 4), (3, 1), (1, 3)])
def test_minimal_solver_recovers_homography(n_p, n_l):
    rng = np.random.default_rng(n_p)
    Ht = syn.random_homography(rng, strength=0.15)
    d = syn.make_homography_correspondences(11 + n_l, n_p, n_l, Ht, noise_px=0.0, outlier_frac=0.0)
    r = _host(d, n_hypotheses=16)
    assert r["valid"] and r["hypothesis"] == 0 and r["hypothesis_inliers"] == 4
    # the exact homography through the float32 correspondences, from the unnormalised equations
    pts = np.concatenate([d["kpts0"], d["kpts1"]], 1)
    A = _pixel_rows(pts, d["klines0"], d["klines1"])
    exact = np.append(np.linalg.solve(A[:, :8], -A[:, 8]), 1.0).reshape(3, 3)
    assert _rel(r["H_hypothesis"], exact) < 1e-9
    assert _rel(r["H"], exact) < 1e-9
    assert _rel(r["H"], Ht) < 1e-4


def test_two_points_two_lines_are_degenerate():
    """Two points and two lines do not fix H in the linear equations: the rank-one H = (l1 x l2)(x1 x x2)^T sends both
    points to (0, 0, 0) and both lines' end points onto l1 and l2, so it satisfies all 8 rows, and the 8 x 9 system
    has a second null vector besides the true H.  Such samples give a spurious hypothesis; other samples win."""
    Ht = syn.random_homography(np.random.default_rng(2), strength=0.15)
    d = syn.make_homography_correspondences(13, 2, 2, Ht, noise_px=0.0, outlier_frac=0.0)
    pts = np.concatenate([d["kpts0"], d["kpts1"]], 1)
    sv = np.linalg.svd(_pixel_rows(pts, d["klines0"], d["klines1"]), compute_uv=False)
    assert sv[-1] < 1e-9 * sv[0]
    x = [np.array([*p, 1.0]) for p in d["kpts0"].astype(np.float64)]
    l = [np.cross([*s[0], 1.0], [*s[1], 1.0]) for s in d["klines1"].astype(np.float64)]
    R = np.outer(np.cross(l[0], l[1]), np.cross(x[0], x[1]))
    A = _pixel_rows(pts, d["klines0"], d["klines1"])
    assert np.abs(A @ R.reshape(9)).max() < 1e-9 * np.abs(A).max() * np.abs(R).max()


@pytest.mark.parametrize("use_lines,use_points", [(True, True), (False, True), (True, False)])
def test_host_model_finds_true_inliers(use_lines, use_points):
    Ht = syn.random_homography(np.random.default_rng(1))
    d = syn.make_homography_correspondences(3, 300, 80, Ht, noise_px=0.3, outlier_frac=0.5)
    r = _host(d, use_lines=use_lines, use_points=use_points)
    assert r["valid"]
    assert np.array_equal(r["inliers_p"].astype(bool), d["true_p"] & use_points)
    assert np.array_equal(r["inliers_l"].astype(bool), d["true_l"] & use_lines)
    assert r["n_inliers_p"] == int((d["true_p"] & use_points).sum()) and r["n_inliers_l"] == int((d["true_l"] & use_lines).sum())
    assert G.homography_corner_error(r["H"], Ht, SHAPE)["error"][0] < 0.5


def test_host_model_against_opencv():
    cv2 = pytest.importorskip("cv2")
    Ht = syn.random_homography(np.random.default_rng(5))
    d = syn.make_homography_correspondences(9, 300, 0, Ht, noise_px=0.3, outlier_frac=0.5)
    r = _host(d, use_lines=False)
    Hc, mask = cv2.findHomography(d["kpts0"], d["kpts1"], cv2.RANSAC, 3.0)
    ours, theirs = r["inliers_p"].astype(bool), mask.ravel().astype(bool)
    pts = np.concatenate([d["kpts0"], d["kpts1"]], 1)
    res = np.sqrt(G.residuals(r["H"].reshape(1, 9), pts, np.zeros((0, 2, 2)), np.zeros((0, 3)))[0])
    near = np.abs(res - 3.0) < 0.05
    differ = ours != theirs
    print(f"OpenCV: {int(differ.sum())} masks differ, {int(near.sum())} points within 0.05 px of the threshold")
    assert not (differ & ~near).any()
    assert G.homography_corner_error(r["H"], Hc, SHAPE)["error"][0] < 0.5


def test_degenerate_inputs():
    e2 = np.zeros((0, 2), np.float32)
    e4 = np.zeros((0, 2, 2), np.float32)
    three = np.array([[1, 2], [30, 4], [5, 60]], np.float32)
    r = G.ransac_homography_host(three, three + 1, np.arange(3), e4, e4, [])
    assert not r["valid"] and np.isnan(r["H"]).all() and r["hypothesis"] == -1 and not r["inliers_p"].any()
    same = np.tile(np.float32([[100, 100]]), (10, 1))
    assert not G.ransac_homography_host(same, same + 5, np.arange(10), e4, e4, [])["valid"]
    line = np.stack([np.arange(10, 210, 20), np.full(10, 100)], 1).astype(np.float32)   # exactly collinear
    assert not G.ransac_homography_host(line, line * 2, np.arange(10), e4, e4, [])["valid"]
    dot = np.tile(np.float32([[[5, 5], [5, 5]]]), (6, 1, 1))                            # zero-length partner segments
    segs = np.random.default_rng(0).uniform(0, 400, (6, 2, 2)).astype(np.float32)
    assert not G.ransac_homography_host(e2, e2, [], segs, dot, np.arange(6))["valid"]
    none = G.ransac_homography_host(e2, e2, [], e4, e4, [])
    assert not none["valid"] and none["inliers_p"].shape == (0,)
    unmatched = G.ransac_homography_host(three, three, [-1, 7, 2], e4, e4, [])   # only one match in range
    assert not unmatched["valid"] and unmatched["inliers_p"].tolist() == [0, 0, 0]


def test_corner_error_metric():
    Ht = syn.random_homography(np.random.default_rng(2))
    shift = np.eye(3)
    shift[0, 2] = 2.0
    m = G.homography_corner_error(np.stack([Ht, shift @ Ht, np.full((3, 3), np.nan)]), Ht, SHAPE)
    assert np.allclose(m["error"][:2], [0.0, 2.0]) and np.isinf(m["error"][2])
    assert m["accuracy_1"] == pytest.approx(1 / 3) and m["accuracy_3"] == pytest.approx(2 / 3)
    assert m["mean_error"] == pytest.approx(1.0)


# ------------------------------------------------------------------ GPU
def _matches(cases, shuffle_rows=True, seed=0):
    """An ImagePairMatches of synthetic correspondence sets (dicts of make_homography_correspondences), with some
    unmatched and out-of-range rows and extra side-1 rows."""
    rng = np.random.default_rng(seed)
    k0, k1, l0, l1, mp, ml = [], [], [], [], [], []
    for d in cases:
        mpp, mll = d["matches_p"].copy(), d["matches_l"].copy()
        if shuffle_rows and len(mpp):
            mpp[rng.random(len(mpp)) < 0.05] = -1
            mpp[rng.random(len(mpp)) < 0.01] = len(d["kpts1"]) + 3
        if shuffle_rows and len(mll):
            mll[rng.random(len(mll)) < 0.05] = -1
        extra = rng.uniform(0, 600, (int(rng.integers(0, 5)), 2)).astype(np.float32)
        k0.append(torch.from_numpy(d["kpts0"]).to(DEV))
        k1.append(torch.from_numpy(np.concatenate([d["kpts1"], extra])).to(DEV))
        l0.append(d["klines0"].astype(np.float64))
        l1.append(d["klines1"].astype(np.float64))
        mp.append(mpp)
        ml.append(mll)
    off = lambda xs: np.concatenate([[0], np.cumsum([len(x) for x in xs])]).astype(np.int32)
    cat = lambda xs: torch.from_numpy(np.concatenate(xs).astype(np.int32) if xs else np.zeros(0, np.int32)).to(DEV)
    P = len(cases)
    z = torch.zeros(P, dtype=torch.int32, device=DEV)
    return engine.ImagePairMatches(cat(ml), cat(ml).float(), z, off(ml), cat(mp), cat(mp).float(), z, off(mp),
                                   l0, l1, k0, k1)


def _host_pair(res, p, **kw):
    a, b = res.offsets_p[p:p + 2]
    c, e = res.offsets_l[p:p + 2]
    return G.ransac_homography_host(res.keypoints0[p].cpu().numpy(), res.keypoints1[p].cpu().numpy(),
                                    res.matches_p[a:b].cpu().numpy(), res.klines0[p], res.klines1[p],
                                    res.matches_l[c:e].cpu().numpy(), pair=p, **kw)


def _ragged_cases(n_pairs=200, seed=0):
    rng = np.random.default_rng(seed)
    cases, Hs = [], []
    for i in range(n_pairs):
        Ht = syn.random_homography(rng, strength=0.12)
        kind = i % 10
        n_p, n_l = int(rng.integers(0, 1001)), int(rng.integers(0, 301))
        frac = float(rng.uniform(0.1, 0.7))
        if kind == 0:
            n_p, n_l = int(rng.integers(0, 3)), int(rng.integers(0, 2))     # below 4 correspondences
        elif kind == 1:
            frac = 1.0                                                       # all outliers
        elif kind == 2:
            n_l = 0
        elif kind == 3:
            n_p = 0
        cases.append(syn.make_homography_correspondences(1000 + i, n_p, n_l, Ht, noise_px=float(rng.uniform(0.1, 1.0)),
                                                         outlier_frac=frac))
        Hs.append(Ht)
    return cases, np.stack(Hs)


@pytest.mark.gpu
def test_kernels_match_host_model():
    cases, _ = _ragged_cases()
    res = _matches(cases)
    K = 1024
    out = G.estimate_homographies(res, n_hypotheses=K, seed=5)
    got = {k: getattr(out, k).cpu().numpy() for k in ("H", "valid", "inliers_p", "inliers_l", "n_inliers_p",
                                                      "n_inliers_l", "hypothesis", "hypothesis_inliers")}
    near = total = refit_ok = 0
    for p in range(res.n_pairs):
        h = _host_pair(res, p, n_hypotheses=K, seed=5)
        assert bool(got["valid"][p]) == h["valid"], p
        assert got["hypothesis"][p] == h["hypothesis"] and got["hypothesis_inliers"][p] == h["hypothesis_inliers"], p
        a, b = res.offsets_p[p:p + 2]
        c, e = res.offsets_l[p:p + 2]
        gp, gl = got["inliers_p"][a:b], got["inliers_l"][c:e]
        total += (b - a) + (e - c)
        if not h["valid"]:
            assert np.isnan(got["H"][p]).all() and not gp.any() and not gl.any()
            continue
        assert _rel(got["H"][p], h["H"]) < 1e-9, (p, got["H"][p], h["H"])
        refit_ok += h["refit"]
        dp, dl = np.flatnonzero(gp != h["inliers_p"]), np.flatnonzero(gl != h["inliers_l"])
        if len(dp) or len(dl):   # only correspondences within 1e-6 px of the threshold may differ
            kp0 = res.keypoints0[p].cpu().numpy()[dp]
            m = res.matches_p[a:b].cpu().numpy()[dp]
            pts = np.concatenate([kp0, res.keypoints1[p].cpu().numpy()[m]], 1)
            s0 = np.asarray(res.klines0[p], np.float32)[dl]
            s1 = np.asarray(res.klines1[p], np.float32)[res.matches_l[c:e].cpu().numpy()[dl]]
            r = np.sqrt(G.residuals(h["H"].reshape(1, 9), pts, s0, G.pixel_lines(s1) if len(s1) else np.zeros((0, 3)))[0])
            assert np.all(np.abs(r - 3.0) < 1e-6), (p, r)
            near += len(dp) + len(dl)
        assert got["n_inliers_p"][p] == gp.sum() and got["n_inliers_l"][p] == gl.sum()
    print(f"{res.n_pairs} pairs, {int(got['valid'].sum())} valid, {refit_ok} refits kept, {near} of {total} rows differ")
    assert near * 10000 < total
    assert not got["valid"][::10].any()                                      # the pairs below 4 correspondences


@pytest.mark.gpu
def test_kinds_alone_match_host_model():
    cases, _ = _ragged_cases(24, seed=1)
    res = _matches(cases)
    for ul, up in ((True, False), (False, True)):
        out = G.estimate_homographies(res, n_hypotheses=256, seed=1, use_lines=ul, use_points=up)
        for p in range(res.n_pairs):
            h = _host_pair(res, p, n_hypotheses=256, seed=1, use_lines=ul, use_points=up)
            assert int(out.hypothesis[p]) == h["hypothesis"] and int(out.hypothesis_inliers[p]) == h["hypothesis_inliers"]
            assert bool(out.valid[p]) == h["valid"]
        assert (not ul or not out.inliers_p.any()) and (not up or not out.inliers_l.any())


@pytest.mark.gpu
def test_deterministic_and_seed_independent_on_clean_data():
    rng = np.random.default_rng(4)
    Hs = [syn.random_homography(rng) for _ in range(16)]
    cases = [syn.make_homography_correspondences(50 + i, 400, 100, H, noise_px=0.3, outlier_frac=0.5)
             for i, H in enumerate(Hs)]
    res = _matches(cases, shuffle_rows=False)
    fields = ("H", "valid", "inliers_p", "inliers_l", "n_inliers_p", "n_inliers_l", "hypothesis", "hypothesis_inliers")
    a, b = G.estimate_homographies(res, seed=3), G.estimate_homographies(res, seed=3)
    for f in fields:
        assert torch.equal(getattr(a, f), getattr(b, f)), f
    c = G.estimate_homographies(res, seed=4)
    assert not torch.equal(a.hypothesis, c.hypothesis)
    assert torch.equal(a.inliers_p, c.inliers_p) and torch.equal(a.inliers_l, c.inliers_l)
    true_p = torch.from_numpy(np.concatenate([d["true_p"] for d in cases]).astype(np.uint8)).to(DEV)
    true_l = torch.from_numpy(np.concatenate([d["true_l"] for d in cases]).astype(np.uint8)).to(DEV)
    assert torch.equal(a.inliers_p, true_p) and torch.equal(a.inliers_l, true_l)
    assert G.homography_corner_error(a.H, np.stack(Hs), SHAPE)["error"].max() < 0.5


@pytest.mark.gpu
def test_end_to_end_match_images_and_match_sets():
    from tests.test_image_pairs import _model
    model, _ = _model()
    eng = engine.PairEngine(model, DEV)
    views, Hv = syn.make_homography_set(21, 6, 60, 400, jitter_px=0.1, map_noise=0.02)
    views = [syn.image_to(v, DEV) for v in views]
    pairs = engine.exhaustive_pairs(len(views))
    Hgt = np.stack([Hv[j] @ np.linalg.inv(Hv[i]) for i, j in pairs])
    r_img = eng.match_images([views[i] for i, _ in pairs], [views[j] for _, j in pairs])
    r_set = eng.match_set(eng.encode_images(views), pairs)
    a, b = G.estimate_homographies(r_img), G.estimate_homographies(r_set)
    err = G.homography_corner_error(a.H, Hgt, SHAPE)["error"]
    # how many line matches are consistent with the true homography (both end points within 3 px of the partner line)
    good = 0
    for p in range(len(pairs)):
        c, e = r_img.offsets_l[p:p + 2]
        m = r_img.matches_l[c:e].cpu().numpy()
        r = np.flatnonzero(m >= 0)
        s0 = np.asarray(r_img.klines0[p], np.float32)[r]
        s1 = np.asarray(r_img.klines1[p], np.float32)[m[r]]
        res = G.residuals(Hgt[p].reshape(1, 9), np.zeros((0, 4)), s0, G.pixel_lines(s1))[0]
        good += int((res < 9.0).sum())
    n_l = int((r_img.matches_l >= 0).sum())
    print(f"corner error over {len(pairs)} pairs: max {err.max():.3f} px, mean {err.mean():.3f} px; "
          f"{good} of {n_l} line matches consistent with the true homography; inliers {a.n_inliers_p.tolist()}, "
          f"{a.n_inliers_l.tolist()}")
    assert good >= 0.9 * n_l
    assert a.valid.all() and err.max() < 1.0
    for f in ("H", "valid", "inliers_p", "inliers_l", "n_inliers_p", "n_inliers_l", "hypothesis", "hypothesis_inliers"):
        assert torch.equal(getattr(a, f), getattr(b, f)), f


@pytest.mark.gpu
def test_over_capacity_is_unsupported_before_any_launch():
    Ht = syn.random_homography(np.random.default_rng(0))
    big = syn.make_homography_correspondences(1, G.SMEM_MAX // G.SMEM_PER_POINT + 1, 0, Ht)
    res = _matches([big], shuffle_rows=False)
    N.reset_launch_count()
    with pytest.raises(N.LtrError, match=r"code -4"):
        G.estimate_homographies(res)
    assert N.launch_count() == 0
    # the same rows are within capacity when only the lines are used
    out = G.estimate_homographies(res, use_points=False)
    assert not out.valid.any()


@pytest.mark.gpu
def test_pair_over_the_struct_row_bound_is_invalid(monkeypatch):
    """A C-ABI caller's max_rows_p sizes the shared-memory staging; a pair with more rows is invalid, not staged."""
    Ht = syn.random_homography(np.random.default_rng(0))
    res = _matches([syn.make_homography_correspondences(2, n, 20, Ht, outlier_frac=0.3) for n in (300, 100)],
                   shuffle_rows=False)
    call = G._ops.call_struct
    monkeypatch.setattr(G._ops, "call_struct",
                        lambda entry, inputs, *a, **kw: call(entry, {**inputs, "max_rows_p": 200}, *a, **kw))
    out = G.estimate_homographies(res, n_hypotheses=256)
    assert out.valid.tolist() == [False, True]
    assert not out.inliers_p[:300].any() and not out.inliers_l[:20].any() and int(out.hypothesis[0]) == -1
    assert int(out.hypothesis[1]) == _host_pair(res, 1, n_hypotheses=256)["hypothesis"]
