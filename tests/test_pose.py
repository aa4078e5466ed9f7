"""Relative pose from point matches (`ltr_essential`, `geometry.estimate_poses`) against the numpy model
`geometry.ransac_essential_host`, OpenCV and known poses, and the reference's pose metrics."""
import numpy as np
import pytest
import torch

from linetr_b200 import _native as N, engine, geometry as G, synthetic as syn

DEV = torch.device("cuda", 0)
K = syn.DEFAULT_K


def _T(R, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def _skew(t):
    return np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])


def _unit_E(R, t):
    E = (_skew(t) @ R).reshape(9)
    return E / np.linalg.norm(E)


def _host(d, **kw):
    return G.ransac_essential_host(d["kpts0"], d["kpts1"], d["matches_p"], kw.pop("K0", K), kw.pop("K1", K), **kw)


# ------------------------------------------------------------------ CPU
def test_draw_samples_of_four_are_unchanged():
    """size=4 (the homography's samples) is the generalised function's default and gives the same bits as the
    four-sample draw it replaced, restated here."""
    def old(seed, pair, K, n):
        U = np.uint64
        k = np.arange(K, dtype=U)
        s = G.splitmix64(U(seed) + G.splitmix64((U(pair) << U(32)) | k))
        idx = np.full((K, 4), -1, dtype=np.int64)
        got = np.zeros(K, dtype=np.int64)
        for j in range(G.MAX_DRAWS):
            active = got < 4
            if not active.any():
                break
            v = (G.splitmix64(s + U(j)) % U(n)).astype(np.int64)
            take = active & ~(idx == v[:, None]).any(1)
            idx[np.arange(K)[take], got[take]] = v[take]
            got += take
        return idx, got == 4
    for seed, pair, n in ((0, 0, 4), (7, 3, 5), (123, 40, 1000), (2 ** 40 + 1, 7, 37)):
        a, b = G.draw_samples(seed, pair, 300, n), old(seed, pair, 300, n)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        assert np.array_equal(a[0], G.draw_samples(seed, pair, 300, n, 4)[0])
    idx, ok = G.draw_samples(5, 2, 512, 6, 5)
    assert ok.all() and all(len(set(r)) == 5 for r in idx.tolist()) and idx.max() < 6
    assert np.array_equal(idx[:, :4], G.draw_samples(5, 2, 512, 6)[0])   # the same stream, one more draw


def test_minimal_solver_recovers_true_essential():
    errs, n_sol = [], []
    for s in range(60):
        rng = np.random.default_rng(s)
        R, t = syn.random_pose(rng, 20.0)
        X = np.c_[rng.uniform(-1, 1, (5, 2)), rng.uniform(3, 6, 5)]
        X1 = X @ R.T + t
        q = np.concatenate([X[:, :2] / X[:, 2:], X1[:, :2] / X1[:, 2:]], 1)
        E, ok = G.essential_solutions(q[None])
        assert 1 <= ok.sum() <= G.ESS_MAX_ROOTS
        Et = _unit_E(R, t)
        best = np.inf
        for j in np.flatnonzero(ok[0]):
            e = E[0, j] / np.linalg.norm(E[0, j])
            best = min(best, np.abs(e - Et).max(), np.abs(e + Et).max())
            M = e.reshape(3, 3)
            assert abs(np.linalg.det(M)) < 1e-7
            assert np.abs(2 * M @ M.T @ M - np.trace(M @ M.T) * M).max() < 1e-7
            x0 = np.c_[q[:, :2], np.ones(5)]
            x1 = np.c_[q[:, 2:], np.ones(5)]
            assert np.abs(np.einsum("ni,ij,nj->n", x1, M, x0)).max() < 1e-7
        errs.append(best)
        n_sol.append(int(ok.sum()))
    errs = np.array(errs)
    print(f"solutions per sample: mean {np.mean(n_sol):.2f}; distance to the true E: median {np.median(errs):.1e}, "
          f"max {errs.max():.1e}")
    # the fp64 solver loses a few digits on the worse-conditioned configurations
    assert np.mean(errs < 1e-9) >= 0.9 and errs.max() < 1e-6


@pytest.mark.parametrize("seed", range(6))
def test_sturm_roots_against_np_roots(seed):
    rng = np.random.default_rng(seed)
    n_real = [10, 8, 6, 4, 2, 0][seed]
    real = np.sort(rng.uniform(-3, 3, n_real))
    if n_real >= 2:
        real[1] = real[0] + 1e-4 * (seed + 1)   # a close pair
        real = np.sort(real)
    poly = np.array([1.0])
    for r in real:
        poly = np.convolve(poly, [1.0, -r])
    for _ in range((10 - n_real) // 2):
        re, im = rng.uniform(-2, 2), rng.uniform(0.3, 2)
        poly = np.convolve(poly, [1.0, -2 * re, re * re + im * im])
    poly *= rng.uniform(0.5, 2.0)
    roots, count = G.sturm_roots(poly[::-1][None].copy())
    ref = np.sort(np.roots(poly)[np.abs(np.roots(poly).imag) < 1e-6].real)
    assert count[0] == n_real == len(ref)
    assert np.allclose(roots[0, :n_real], real, rtol=0, atol=1e-8)
    assert np.allclose(roots[0, :n_real], ref, rtol=0, atol=1e-6)   # np.roots loses digits on the close pair
    assert np.isnan(roots[0, n_real:]).all()


def test_host_model_finds_true_inliers_on_clean_data():
    R, t = syn.random_pose(np.random.default_rng(1))
    d = syn.make_pose_correspondences(3, 300, R, t, noise_px=0.0, outlier_frac=0.5)
    r = _host(d, n_hypotheses=256)
    assert r["valid"] and np.array_equal(r["inliers_p"].astype(bool), d["true_p"])
    assert r["n_inliers"] == r["hypothesis_inliers"] == r["n_cheirality"] == int(d["true_p"].sum())
    et, eR = G.compute_pose_error(_T(R, t), r["R"], r["t"])
    assert et < 1e-3 and eR < 1e-3
    assert abs(np.linalg.norm(r["E"]) - 1) < 1e-12 and abs(np.linalg.norm(r["t"]) - 1) < 1e-12
    assert np.abs(r["E"]).max() == r["E"].max()


def test_host_model_against_opencv():
    """The model against the reference's estimate_pose calls (cv2.findEssentialMat + cv2.recoverPose) on 300 points,
    0.5 px noise, 50 % outliers, 1 px threshold.

    Weaker than the bar "pose within 0.5 deg of cv2's, masks differing only within 5 % of the threshold": both
    estimators return an unrefined minimal-sample winner, and two different minimal samples from 0.5 px noise differ
    by about as much as each differs from the truth (here ours vs cv2 0.9 deg, cv2 vs truth 0.8 deg).  Their masks then
    differ on rows anywhere in the noise band under the 1 px threshold, not only near it.  So the test checks each pose
    against the truth (ours within 0.5 deg), ours against cv2's within 1 deg, that neither mask accepts an outlier (all
    are >= 10 px off their epipolar line) and that both keep >= 80 % of the true inliers, and that our mask is exactly
    our E's Sampson error below the threshold."""
    cv2 = pytest.importorskip("cv2")
    R, t = syn.random_pose(np.random.default_rng(3))
    d = syn.make_pose_correspondences(7, 300, R, t, noise_px=0.5, outlier_frac=0.5)
    r = _host(d, thresh=1.0)
    k0, k1 = G._normalised(d["kpts0"], K), G._normalised(d["kpts1"], K)
    f_mean = G._f_mean(K, K)
    E, mask = cv2.findEssentialMat(k0, k1, np.eye(3), threshold=1.0 / f_mean, prob=0.99999, method=cv2.RANSAC)
    _, Rc, tc, _ = cv2.recoverPose(E[:3], k0, k1, np.eye(3), 1e9, mask=mask)
    T = _T(R, t)
    ours, theirs = G.compute_pose_error(T, r["R"], r["t"]), G.compute_pose_error(T, Rc, tc[:, 0])
    vs = G.compute_pose_error(_T(Rc, tc[:, 0]), r["R"], r["t"])
    m_ours, m_cv = r["inliers_p"].astype(bool), mask.ravel().astype(bool)
    print(f"pose error (t, R) in degrees: ours {ours}, cv2 {theirs}, ours vs cv2 {vs}; inliers {m_ours.sum()} / "
          f"{m_cv.sum()} of {d['true_p'].sum()} true")
    assert max(ours) < 0.5 and max(vs) < 1.0
    for m in (m_ours, m_cv):
        assert not (m & ~d["true_p"]).any() and m.sum() >= 0.8 * d["true_p"].sum()
    err = G.sampson_error(r["E"], np.concatenate([k0, k1], 1)) / (1.0 / f_mean) ** 2
    assert np.array_equal(m_ours, err < 1)


def test_degenerate_inputs():
    e2 = np.zeros((0, 2), np.float32)
    four = np.array([[1, 2], [30, 4], [5, 60], [70, 80]], np.float32)
    r = G.ransac_essential_host(four, four + 1, np.arange(4), K, K)
    assert not r["valid"] and np.isnan(r["E"]).all() and np.isnan(r["R"]).all() and r["hypothesis"] == -1
    assert r["inliers_p"].tolist() == [0, 0, 0, 0]
    same = np.tile(np.float32([[100, 100]]), (10, 1))
    assert not G.ransac_essential_host(same, same + 5, np.arange(10), K, K)["valid"]
    none = G.ransac_essential_host(e2, e2, [], K, K)
    assert not none["valid"] and none["inliers_p"].shape == (0,)
    # exact correspondences of a random pose; unmatched (-1, -5) and out-of-range (9, 100) rows are not correspondences
    R, t = syn.random_pose(np.random.default_rng(5))
    d = syn.make_pose_correspondences(4, 8, R, t, noise_px=0.0, outlier_frac=0.0)
    five = G.ransac_essential_host(d["kpts0"], d["kpts1"], [-1, 9, 2, 3, 4, -5, 6, 7], K, K)   # 5 rows in range
    assert five["valid"] and five["n_inliers"] == 5
    assert five["inliers_p"].tolist() == [0, 0, 1, 1, 1, 0, 1, 1]
    # (every real solution of the only possible sample fits all five rows, so the winner need not be the true pose)
    few = G.ransac_essential_host(d["kpts0"], d["kpts1"], [-1, 9, 2, 3, 4, -5, 6, 100], K, K)   # 4 rows in range
    assert not few["valid"] and few["hypothesis"] == -1 and few["inliers_p"].tolist() == [0] * 8


def test_metrics_are_the_reference_formulas():
    R, t = syn.random_pose(np.random.default_rng(2), 10.0)
    T = _T(R, t)
    assert G.compute_pose_error(T, R, t) == pytest.approx((0.0, 0.0), abs=1e-5)
    assert G.compute_pose_error(T, R, -t) == pytest.approx((0.0, 0.0), abs=1e-5)   # the sign of t is not observable
    Rz = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])            # 90 degrees about z
    et, eR = G.compute_pose_error(_T(np.eye(3), [1.0, 0, 0]), Rz, np.array([0.0, 1.0, 0.0]))
    assert et == pytest.approx(90.0) and eR == pytest.approx(90.0)
    # pose_auc: errors 1, 2, 4 give the recall curve (0, 0), (1, 1/3), (2, 2/3), (4, 1), held flat after the last error
    # below the threshold.  Threshold 1: an error equal to it is not below it, so the area is 0.  Threshold 2:
    # 1/6 + (1/3 + 1/3) / 2 = 1/2, over 2.  Threshold 5: 1/6 + 1/2 + 2 (2/3 + 1) / 2 + 1 = 10/3, over 5.
    auc = G.pose_auc(np.array([4.0, 1.0, 2.0]), [1, 2, 5])
    assert auc == pytest.approx([0.0, 0.25, 10 / 3 / 5])
    # epipolar error: zero for exact correspondences, the reference's symmetric expression otherwise
    X = np.array([[0.3, -0.2, 4.0], [-0.5, 0.4, 6.0], [0.1, 0.1, 5.0]])
    k0 = syn._project(K, X)
    k1 = syn._project(K, X @ R.T + t)
    assert np.abs(G.compute_epipolar_error(k0, k1, T, K, K)).max() < 1e-20
    k1b = k1 + [0.0, 2.0]
    x0 = np.c_[(k0 - K[:2, 2]) / 500.0, np.ones(3)]
    x1 = np.c_[(k1b - K[:2, 2]) / 500.0, np.ones(3)]
    E = _skew(t) @ R
    Ex0, Etx1 = x0 @ E.T, x1 @ E
    num = np.sum(x1 * Ex0, 1) ** 2
    want = num / (Ex0[:, 0] ** 2 + Ex0[:, 1] ** 2) + num / (Etx1[:, 0] ** 2 + Etx1[:, 1] ** 2)
    assert np.allclose(G.compute_epipolar_error(k0, k1b, T, K, K), want, rtol=1e-12)
    et, eR = G.pose_errors(np.stack([R, np.full((3, 3), np.nan)]), np.stack([-t, t]), T)
    assert et[0] == pytest.approx(0.0, abs=1e-5) and eR[0] == pytest.approx(0.0, abs=1e-5)
    assert np.isinf(et[1]) and np.isinf(eR[1])


# ------------------------------------------------------------------ GPU
def _matches(cases, shuffle_rows=True, seed=0):
    """An ImagePairMatches of point-correspondence sets (dicts of make_pose_correspondences), with some unmatched and
    out-of-range rows and extra side-1 rows; no line matches."""
    rng = np.random.default_rng(seed)
    k0, k1, mp = [], [], []
    for d in cases:
        m = d["matches_p"].copy()
        if shuffle_rows and len(m):
            m[rng.random(len(m)) < 0.05] = -1
            m[rng.random(len(m)) < 0.01] = len(d["kpts1"]) + 3
        extra = rng.uniform(0, 600, (int(rng.integers(0, 5)), 2)).astype(np.float32)
        k0.append(torch.from_numpy(d["kpts0"]).to(DEV))
        k1.append(torch.from_numpy(np.concatenate([d["kpts1"], extra])).to(DEV))
        mp.append(m)
    P = len(cases)
    off = np.concatenate([[0], np.cumsum([len(x) for x in mp])]).astype(np.int32)
    mpt = torch.from_numpy(np.concatenate(mp).astype(np.int32) if mp else np.zeros(0, np.int32)).to(DEV)
    ml = torch.zeros(0, dtype=torch.int32, device=DEV)
    z = torch.zeros(P, dtype=torch.int32, device=DEV)
    return engine.ImagePairMatches(ml, ml.float(), z, np.zeros(P + 1, np.int32), mpt, mpt.float(), z, off,
                                   [np.zeros((0, 2, 2))] * P, [np.zeros((0, 2, 2))] * P, k0, k1)


def _host_pair(res, p, K0, K1, **kw):
    a, b = res.offsets_p[p:p + 2]
    return G.ransac_essential_host(res.keypoints0[p].cpu().numpy(), res.keypoints1[p].cpu().numpy(),
                                   res.matches_p[a:b].cpu().numpy(), K0, K1, pair=p, **kw)


def _ragged_cases(n_pairs=200, seed=0):
    rng = np.random.default_rng(seed)
    cases, K0s, K1s, poses = [], [], [], []
    for i in range(n_pairs):
        kind = i % 10
        R, t = syn.random_pose(rng, translation=[0.0, 0.0, 1.0] if kind == 2 else None)   # 2: pure forward motion
        n, frac = int(rng.integers(0, 1001)), float(rng.uniform(0.1, 0.7))
        if kind == 0:
            n = int(rng.integers(0, 5))        # below 5 correspondences
        elif kind == 1:
            frac = 1.0                          # all outliers
        Ka, Kb = K.copy(), K.copy()
        Ka[[0, 1], [0, 1]] *= rng.uniform(0.8, 1.25, 2)
        Kb[[0, 1], [0, 1]] *= rng.uniform(0.8, 1.25, 2)
        cases.append(syn.make_pose_correspondences(2000 + i, n, R, t, Ka, Kb, noise_px=float(rng.uniform(0.1, 1.0)),
                                                   outlier_frac=frac))
        K0s.append(Ka)
        K1s.append(Kb)
        poses.append(_T(R, t))
    return cases, np.stack(K0s), np.stack(K1s), np.stack(poses)


def _rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max())


@pytest.mark.gpu
def test_kernels_match_host_model():
    cases, K0, K1, _ = _ragged_cases()
    res = _matches(cases)
    Kh, seed = 256, 5
    out = G.estimate_poses(res, K0, K1, n_hypotheses=Kh, seed=seed)
    got = {f: getattr(out, f).cpu().numpy() for f in ("E", "R", "t", "valid", "inliers", "n_inliers", "n_cheirality",
                                                      "hypothesis", "hypothesis_inliers")}
    near = total = 0
    for p in range(res.n_pairs):
        h = _host_pair(res, p, K0[p], K1[p], n_hypotheses=Kh, seed=seed)
        assert bool(got["valid"][p]) == h["valid"], p
        assert got["hypothesis"][p] == h["hypothesis"] and got["hypothesis_inliers"][p] == h["hypothesis_inliers"], p
        a, b = res.offsets_p[p:p + 2]
        gm = got["inliers"][a:b]
        total += b - a
        if not h["valid"]:
            assert np.isnan(got["E"][p]).all() and np.isnan(got["R"][p]).all() and not gm.any()
            continue
        assert _rel(got["E"][p], h["E"]) < 1e-9, (p, got["E"][p], h["E"])
        # (R, t) is the host's, or on a tie of cheirality counts another of the tied candidates
        rows = np.flatnonzero(h["inliers_p"])
        m = res.matches_p[a:b].cpu().numpy()[rows]
        q = np.concatenate([G._normalised(res.keypoints0[p].cpu().numpy()[rows], K0[p]),
                            G._normalised(res.keypoints1[p].cpu().numpy()[m], K1[p])], 1)
        cand = G.decompose_essential(h["E"])
        cnt = [int(G.cheirality(Rc, tc, q).sum()) for Rc, tc in cand]
        assert cnt[int(np.argmax(cnt))] == h["n_cheirality"]
        assert any(c == h["n_cheirality"] and _rel(got["R"][p], Rc) < 1e-9 and _rel(got["t"][p], tc) < 1e-9
                   for c, (Rc, tc) in zip(cnt, cand)), p
        assert got["n_cheirality"][p] == h["n_cheirality"], p
        dp = np.flatnonzero(gm != h["inliers_p"])
        if len(dp):   # only rows within 1e-6 relative of the threshold may differ
            m = res.matches_p[a:b].cpu().numpy()[dp]
            q = np.concatenate([G._normalised(res.keypoints0[p].cpu().numpy()[dp], K0[p]),
                                G._normalised(res.keypoints1[p].cpu().numpy()[m], K1[p])], 1)
            tn = 1.0 / G._f_mean(K0[p], K1[p])
            r = G.sampson_error(h["E"], q) / (tn * tn)
            assert np.all(np.abs(r - 1) < 1e-6), (p, r)
            near += len(dp)
        assert got["n_inliers"][p] == gm.sum()
    print(f"{res.n_pairs} pairs, {int(got['valid'].sum())} valid, {near} of {total} mask rows differ")
    assert near * 10000 < total
    assert not got["valid"][::10].any()                       # the pairs below 5 correspondences


@pytest.mark.gpu
def test_deterministic_and_seed_independent_on_clean_data():
    rng = np.random.default_rng(4)
    poses = [syn.random_pose(rng) for _ in range(16)]
    cases = [syn.make_pose_correspondences(50 + i, 400, R, t, noise_px=0.0, outlier_frac=0.5)
             for i, (R, t) in enumerate(poses)]
    res = _matches(cases, shuffle_rows=False)
    fields = ("E", "R", "t", "valid", "inliers", "n_inliers", "n_cheirality", "hypothesis", "hypothesis_inliers")
    a, b = G.estimate_poses(res, K, K, seed=3), G.estimate_poses(res, K, K, seed=3)
    for f in fields:
        assert torch.equal(getattr(a, f), getattr(b, f)), f
    c = G.estimate_poses(res, K, K, seed=4)
    assert not torch.equal(a.hypothesis, c.hypothesis)
    assert torch.equal(a.inliers, c.inliers)
    true_p = torch.from_numpy(np.concatenate([d["true_p"] for d in cases]).astype(np.uint8)).to(DEV)
    assert torch.equal(a.inliers, true_p)
    et, eR = G.pose_errors(a.R, a.t, np.stack([_T(R, t) for R, t in poses]))
    assert et.max() < 0.5 and eR.max() < 0.5


@pytest.mark.gpu
def test_end_to_end_match_images_and_match_sets():
    from tests.test_image_pairs import _model
    model, _ = _model()
    eng = engine.PairEngine(model, DEV)
    views, Tv = syn.make_pose_set(31, 6, 60, 400, jitter_px=0.1)
    views = [syn.image_to(v, DEV) for v in views]
    pairs = engine.exhaustive_pairs(len(views))
    Tgt = np.stack([Tv[j] @ np.linalg.inv(Tv[i]) for i, j in pairs])
    r_img = eng.match_images([views[i] for i, _ in pairs], [views[j] for _, j in pairs])
    r_set = eng.match_set(eng.encode_images(views), pairs)
    # without a refit the pose is one minimal sample's: a threshold near the keypoint noise keeps it within 1 degree
    a, b = G.estimate_poses(r_img, K, K, thresh=0.3), G.estimate_poses(r_set, K, K, thresh=0.3)
    for f in ("E", "R", "t", "valid", "inliers", "n_inliers", "n_cheirality", "hypothesis", "hypothesis_inliers"):
        assert torch.equal(getattr(a, f), getattr(b, f)), f
    et, eR = G.pose_errors(a.R, a.t, Tgt)
    print(f"pose error over {len(pairs)} pairs: t max {et.max():.3f} deg, R max {eR.max():.3f} deg; point matches "
          f"{r_img.counts_p.tolist()}, inliers {a.n_inliers.tolist()}")
    assert a.valid.all() and et.max() < 1.0 and eR.max() < 1.0


@pytest.mark.gpu
def test_capacity_and_struct_row_bounds_and_empty_batches(monkeypatch):
    R, t = syn.random_pose(np.random.default_rng(0))
    big = syn.make_pose_correspondences(1, G.SMEM_MAX // G.SMEM_PER_ROW_E + 1, R, t)
    N.reset_launch_count()
    with pytest.raises(N.LtrError, match=r"code -4"):
        G.estimate_poses(_matches([big], shuffle_rows=False), K, K)
    assert N.launch_count() == 0
    # a C-ABI caller's max_rows_p sizes the staging; a pair with more rows is invalid, not staged
    res = _matches([syn.make_pose_correspondences(2, n, R, t, outlier_frac=0.3) for n in (300, 100)], shuffle_rows=False)
    call = G._ops.call_struct
    monkeypatch.setattr(G._ops, "call_struct",
                        lambda entry, inputs, *a, **kw: call(entry, {**inputs, "max_rows_p": 200}, *a, **kw))
    out = G.estimate_poses(res, K, K, n_hypotheses=256)
    assert out.valid.tolist() == [False, True]
    assert not out.inliers[:300].any() and int(out.hypothesis[0]) == -1 and np.isnan(out.E[0].cpu().numpy()).all()
    assert int(out.hypothesis[1]) == _host_pair(res, 1, K, K, n_hypotheses=256)["hypothesis"]
    monkeypatch.undo()
    N.reset_launch_count()
    empty = G.estimate_poses(_matches([]), K, K)
    assert N.launch_count() == 0 and empty.E.shape == (0, 3, 3)
    bad = K.copy()
    bad[0, 0] = 0.0
    for Kb in (bad, np.full((3, 3), np.nan)):
        with pytest.raises(N.LtrError, match="fx, fy > 0"):
            G.estimate_poses(res, Kb, K)
