"""Fundamental matrices of uncalibrated pairs (`ltr_fundamental`, `geometry.estimate_fundamentals`) against the numpy
model `geometry.ransac_fundamental_host`, OpenCV and known two-view geometry, and the epipolar check of line matches."""
import numpy as np
import pytest
import torch

from linetr_b200 import _native as N, engine, geometry as G, synthetic as syn

DEV = torch.device("cuda", 0)
E22 = np.zeros((0, 2, 2), np.float32)


def _host(d, **kw):
    return G.ransac_fundamental_host(d["kpts0"], d["kpts1"], d["matches_p"], d.get("klines0"), d.get("klines1"),
                                     d.get("matches_l"), **kw)


def _sign_free(a, b):
    a, b = np.asarray(a).reshape(9), np.asarray(b).reshape(9)
    return min(np.abs(a - b).max(), np.abs(a + b).max())


def _sym_dist(F, pts):
    """Symmetric epipolar distance [n] in pixels: distance of x1 to F x0 plus distance of x0 to F^T x1."""
    num, a, b = G._fm_terms(np.asarray(F, dtype=np.float64).reshape(1, 9), pts)
    return (np.abs(num) / np.sqrt(a) + np.abs(num) / np.sqrt(b))[0]


# ------------------------------------------------------------------ CPU
def test_draw_samples_of_seven():
    idx, ok = G.draw_samples(5, 2, 512, 9, 7)
    assert ok.all() and all(len(set(r)) == 7 for r in idx.tolist()) and idx.max() < 9
    assert np.array_equal(idx[:, :5], G.draw_samples(5, 2, 512, 9, 5)[0])   # the same stream, two more draws
    _, ok = G.draw_samples(0, 0, 64, 6, 7)
    assert not ok.any()                                                   # 7 distinct of 6 never succeed


def _exact_sample(s):
    """7 exact fp64 correspondences of a random uncalibrated pair, normalised by a per-side similarity, and the true
    normalised F^ (unit norm, largest |entry| positive)."""
    rng = np.random.default_rng(s)
    K0, K1 = syn.random_intrinsics(rng), syn.random_intrinsics(rng)
    R, t = syn.random_pose(rng)
    X = (np.c_[rng.uniform(0, 639, 7), rng.uniform(0, 479, 7), np.ones(7)] @ np.linalg.inv(K0).T) \
        * rng.uniform(2, 8, (7, 1))
    x0, x1 = syn._project(K0, X), syn._project(K1, X @ R.T + t)
    T = []
    for x in (x0, x1):
        c, sc = x.mean(0), 1.0 / np.abs(x - x.mean(0)).max()
        T.append(np.array([[sc, 0, -c[0] * sc], [0, sc, -c[1] * sc], [0, 0, 1.0]]))
    h = lambda x, T: (np.c_[x, np.ones(len(x))] @ T.T)[:, :2]
    q = np.concatenate([h(x0, T[0]), h(x1, T[1])], 1)
    Fn = np.linalg.inv(T[1]).T @ syn.fundamental_from_pose(K0, K1, R, t) @ np.linalg.inv(T[0])
    Fn /= np.linalg.norm(Fn)
    return q, (Fn if Fn.flat[int(np.argmax(np.abs(Fn)))] > 0 else -Fn).reshape(9)


def test_seven_point_solver_recovers_true_fundamental():
    errs, n_sol = [], []
    for s in range(100):
        q, Ft = _exact_sample(s)
        F, ok = G.fundamental_solutions(q[None])
        assert 1 <= ok.sum() <= G.FM_MAX_SOLUTIONS
        best = np.inf
        x0, x1 = np.c_[q[:, :2], np.ones(7)], np.c_[q[:, 2:], np.ones(7)]
        for j in np.flatnonzero(ok[0]):
            f = F[0, j] / np.linalg.norm(F[0, j])
            best = min(best, _sign_free(f, Ft))
            assert abs(np.linalg.det(f.reshape(3, 3))) < 1e-9
            assert np.abs(np.einsum("ni,ij,nj->n", x1, f.reshape(3, 3), x0)).max() < 1e-9
        errs.append(best)
        n_sol.append(int(ok.sum()))
    errs = np.array(errs)
    print(f"solutions per sample: {np.bincount(n_sol).tolist()}; distance to the true F: median {np.median(errs):.1e}, "
          f"max {errs.max():.1e}; found to 1e-9: {np.mean(errs < 1e-9):.2f}, to 1e-6: {np.mean(errs < 1e-6):.2f}")
    assert np.mean(errs < 1e-9) >= 0.9 and errs.max() < 1e-6


def test_cubic_roots_against_np_roots():
    for s in range(40):
        q, _ = _exact_sample(s)
        basis, ok = G._null_basis(q[None])
        cubic, _, _ = G.fundamental_cubic(basis)
        p = np.zeros((1, 11))
        p[0, :4] = cubic[0]
        roots, count = G.sturm_roots(p)
        r = np.roots(cubic[0, ::-1])
        ref = np.sort(r[np.abs(r.imag) < 1e-9 * np.maximum(1, np.abs(r))].real)
        assert count[0] == len(ref), (s, r)
        assert np.allclose(roots[0, :count[0]], ref, rtol=1e-9, atol=1e-9), s


def test_host_model_finds_true_inliers_on_clean_data():
    d = syn.make_fundamental_correspondences(1, 400, 60, noise_px=0.0, outlier_frac=0.5)
    r = _host(d, n_hypotheses=512)
    assert r["valid"] and r["refit"]
    assert np.array_equal(r["inliers_p"].astype(bool), d["true_p"])
    assert r["n_inliers"] == r["hypothesis_inliers"] == int(d["true_p"].sum())
    assert _sign_free(r["F"], d["F"]) < 1e-6
    assert np.array_equal(r["lines_consistent"].astype(bool), d["true_l"])
    assert abs(np.linalg.norm(r["F"]) - 1) < 1e-12 and np.abs(r["F"]).max() == r["F"].max()
    assert abs(np.linalg.det(r["F"])) < 1e-12


def test_host_model_against_opencv():
    """The model against cv2.findFundamentalMat(FM_RANSAC) on 1000 points, 0.5 px noise, 50 % outliers, 3 px threshold.
    Neither mask accepts an outlier (all are >= 10 px off their epipolar line) and both keep >= 80 % of the true
    inliers.  On the noise-free true correspondences our refitted F's median symmetric epipolar distance is below 1 px
    and at most cv2's plus 0.1 px: cv2 returns its best seven-point sample unrefined (about 1 px here, measured 0.8 to
    2.0 px over five seeds), ours is the least-squares fit over all inliers (0.15 to 0.37 px), so ours is normally the
    better of the two; the margin only absorbs the case where a lucky minimal sample comes close."""
    cv2 = pytest.importorskip("cv2")
    for seed in range(3):
        d = syn.make_fundamental_correspondences(7 + seed, 1000, 0, noise_px=0.5, outlier_frac=0.5)
        clean = syn.make_fundamental_correspondences(7 + seed, 1000, 0, noise_px=0.0, outlier_frac=0.5)
        r = _host(d, thresh=3.0)
        Fc, mask = cv2.findFundamentalMat(d["kpts0"], d["kpts1"], cv2.FM_RANSAC, 3.0, 0.99999)
        tp = d["true_p"]
        pts = np.concatenate([clean["kpts0"], clean["kpts1"]], 1)[clean["true_p"]]
        ours, theirs = np.median(_sym_dist(r["F"], pts)), np.median(_sym_dist(Fc[:3], pts))
        m_ours, m_cv = r["inliers_p"].astype(bool), mask.ravel().astype(bool)
        print(f"seed {seed}: median symmetric epipolar distance ours {ours:.3f} px, cv2 {theirs:.3f} px; inliers "
              f"{m_ours.sum()} / {m_cv.sum()} of {tp.sum()} true; refit {r['refit']}")
        assert r["refit"] and ours < 1.0 and ours <= theirs + 0.1
        for m in (m_ours, m_cv):
            assert not (m & ~tp).any() and m.sum() >= 0.8 * tp.sum()
        err = G.fundamental_error(r["F"], np.concatenate([d["kpts0"], d["kpts1"]], 1))
        assert np.array_equal(m_ours, err < 9.0)


def test_degenerate_inputs():
    six = np.array([[1, 2], [30, 4], [5, 60], [70, 80], [9, 9], [40, 41]], np.float32)
    r = G.ransac_fundamental_host(six, six + 1, np.arange(6))
    assert not r["valid"] and np.isnan(r["F"]).all() and r["hypothesis"] == -1 and r["inliers_p"].tolist() == [0] * 6
    same = np.tile(np.float32([[100, 100]]), (10, 1))
    r = G.ransac_fundamental_host(same, same + 5, np.arange(10))   # every sample is rank-deficient
    assert not r["valid"] and r["hypothesis"] == -1 and not r["inliers_p"].any()
    none = G.ransac_fundamental_host(np.zeros((0, 2), np.float32), np.zeros((0, 2), np.float32), [])
    assert not none["valid"] and none["inliers_p"].shape == (0,) and none["lines_consistent"].shape == (0,)
    d = syn.make_fundamental_correspondences(4, 10, 3, noise_px=0.0, outlier_frac=0.0, line_outlier_frac=0.0)
    unmatched = G.ransac_fundamental_host(d["kpts0"], d["kpts1"], np.full(10, -1), d["klines0"], d["klines1"],
                                          d["matches_l"])
    assert not unmatched["valid"] and unmatched["lines_consistent"].tolist() == [0, 0, 0]
    # unmatched (-1, -5) and out-of-range (10, 99) rows are not correspondences: 6 in range is too few, 7 suffice
    mp = np.array([-1, 10, 2, 3, 4, -5, 6, 7, 8, 99])
    assert not G.ransac_fundamental_host(d["kpts0"], d["kpts1"], mp)["valid"]
    mp[0] = 0
    seven = G.ransac_fundamental_host(d["kpts0"], d["kpts1"], mp, d["klines0"], d["klines1"], [2, -1, 7])
    assert seven["valid"] and seven["n_inliers"] == 7 and not seven["refit"]
    assert seven["inliers_p"].tolist() == [1, 0, 1, 1, 1, 0, 1, 1, 1, 0]
    assert seven["lines_consistent"][1:].tolist() == [0, 0]


def test_line_check_hand_built():
    """Exact cases under F = [t]x: t = (1, 0, 0) gives horizontal epipolar lines y = const in both images (a
    rectified pair); t = (0, 0, 1) puts both epipoles at the origin."""
    F = np.array([[0.0, 0, 0], [0, 0, -1], [0, 1, 0]])
    s1 = [[15, 20], [55, 60]]                 # a 45-degree segment spanning y in [20, 60] in image 1
    seg0 = np.float32([[[10, 20], [50, 60]],   # full overlap (shifted by 5 px of disparity)
                       [[20, 30], [30, 40]],   # a fragment inside its partner: ratio 1 on both sides
                       [[10, 100], [50, 140]], # disjoint along the band
                       [[10, 50], [50, 90]],   # half inside: ratio 0.25 in image 1
                       [[10, 20], [90, 20]]])  # along the epipolar direction: both sides undefined
    seg1 = np.float32([s1, s1, s1, s1, [[15, 20], [95, 20]]])
    r1, r0 = G.line_overlap_ratios(F, seg0, seg1)
    assert r1[:4].tolist() == [1.0, 1.0, 0.0, 0.25] and np.isnan(r1[4])
    assert r0[:3].tolist() == [1.0, 1.0, 0.0] and np.isnan(r0[4])
    assert G.lines_consistent(F, seg0, seg1).tolist() == [True, True, False, False, True]
    assert G.lines_consistent(F, seg0, seg1, min_overlap=0.0).tolist() == [True] * 5
    # segments through the epipole (0, 0): every epipolar line of their end points is the same line, so no side rejects,
    # whether or not the partner lies on it
    Fe = np.array([[0.0, -1, 0], [1, 0, 0], [0, 0, 0]])
    seg0 = np.float32([[[-1, -1], [2, 2]], [[0, 0], [3, 3]], [[-1, -1], [2, 2]]])
    seg1 = np.float32([[[2, 2], [4, 4]], [[1, 1], [5, 5]], [[10, 0], [10, 8]]])
    r1, r0 = G.line_overlap_ratios(Fe, seg0, seg1)
    assert np.isnan(r1).all() and np.isnan(r0).all()
    assert G.lines_consistent(Fe, seg0, seg1).all()


def test_line_check_on_synthetic_segments():
    for seed in range(4):
        d = syn.make_fundamental_correspondences(20 + seed, 300, 200, noise_px=0.5, outlier_frac=0.3,
                                                 line_outlier_frac=0.4)
        ok = G.lines_consistent(d["F"], d["klines0"], d["klines1"])
        assert np.array_equal(ok, d["true_l"]), seed
        r = _host(d, n_hypotheses=512)
        assert np.array_equal(r["lines_consistent"].astype(bool), d["true_l"])
        assert r["n_lines_consistent"] == int(d["true_l"].sum())


# ------------------------------------------------------------------ GPU
def _matches(cases, shuffle_rows=True, seed=0):
    """An ImagePairMatches of point and line correspondence sets (dicts of make_fundamental_correspondences), with some
    unmatched and out-of-range rows and extra side-1 rows."""
    rng = np.random.default_rng(seed)
    k0, k1, mp, l0, l1, ml = [], [], [], [], [], []
    for d in cases:
        m, n = d["matches_p"].copy(), d["matches_l"].copy()
        if shuffle_rows:
            m[rng.random(len(m)) < 0.05] = -1
            m[rng.random(len(m)) < 0.01] = len(d["kpts1"]) + 3
            n[rng.random(len(n)) < 0.05] = -1
            n[rng.random(len(n)) < 0.02] = len(d["klines1"]) + 2
        extra = rng.uniform(0, 600, (int(rng.integers(0, 5)), 2)).astype(np.float32)
        k0.append(torch.from_numpy(d["kpts0"]).to(DEV))
        k1.append(torch.from_numpy(np.concatenate([d["kpts1"], extra])).to(DEV))
        l0.append(d["klines0"])
        l1.append(np.concatenate([d["klines1"], extra[:2].reshape(-1, 2, 2) if len(extra) >= 2 else E22]))
        mp.append(m)
        ml.append(n)
    P = len(cases)
    offp = np.concatenate([[0], np.cumsum([len(x) for x in mp])]).astype(np.int32)
    offl = np.concatenate([[0], np.cumsum([len(x) for x in ml])]).astype(np.int32)
    cat = lambda x: torch.from_numpy(np.concatenate(x).astype(np.int32) if x else np.zeros(0, np.int32)).to(DEV)
    mpt, mlt = cat(mp), cat(ml)
    z = torch.zeros(P, dtype=torch.int32, device=DEV)
    return engine.ImagePairMatches(mlt, mlt.float(), z, offl, mpt, mpt.float(), z, offp, l0, l1, k0, k1)


def _host_pair(res, p, **kw):
    a, b = res.offsets_p[p:p + 2]
    c, e = res.offsets_l[p:p + 2]
    return G.ransac_fundamental_host(res.keypoints0[p].cpu().numpy(), res.keypoints1[p].cpu().numpy(),
                                     res.matches_p[a:b].cpu().numpy(), res.klines0[p], res.klines1[p],
                                     res.matches_l[c:e].cpu().numpy(), pair=p, **kw)


def _ragged_cases(n_pairs=200, seed=0):
    rng = np.random.default_rng(seed)
    cases = []
    for i in range(n_pairs):
        kind = i % 10
        n, frac = int(rng.integers(0, 601)), float(rng.uniform(0.1, 0.6))
        if kind == 0:
            n = int(rng.integers(0, 7))         # below 7 correspondences
        elif kind == 1:
            frac = 1.0                           # all outliers
        cases.append(syn.make_fundamental_correspondences(3000 + i, n, int(rng.integers(0, 40)),
                                                          noise_px=float(rng.uniform(0.1, 1.0)), outlier_frac=frac))
    return cases


FIELDS = ("F", "valid", "inliers_p", "n_inliers", "hypothesis", "hypothesis_inliers", "refit", "lines_consistent",
          "n_lines_consistent")
U = 2.0 ** -53
# The refit's A^T A is summed in another order than numpy's (and nvcc may contract its products to FMA), its smallest
# eigenvector comes from Jacobi instead of eigh, and the rank-2 step from Jacobi on F^T F instead of an SVD.  So the
# refitted F^ differs from the host's by about u times the conditioning of both steps: lambda_max / (lambda_2 -
# lambda_1) of A^T A (Davis-Kahan) plus sigma_1 / (sigma_2 - sigma_3) of F^ (the rank-2 direction).  Denormalising and
# the unit scaling keep that relative size.  Measured on an H100 80GB HBM3 (700 W limit) over the 162 kept refits of
# test_kernels_match_host_model and the 1290 of test_estimator_edges' every-hypothesis runs: at most 29.8 u cond.
# FM_REFIT_C leaves a factor 4 above that.
FM_REFIT_C = 120.0


def refit_condition(res, p, h, t2):
    """lambda_max / (lambda_2 - lambda_1) of the refit's A^T A plus sigma_1 / (sigma_2 - sigma_3) of its F^."""
    a, b = res.offsets_p[p:p + 2]
    pts, _, _, _, _ = G._correspondences(res.keypoints0[p].cpu().numpy(), res.keypoints1[p].cpu().numpy(),
                                         res.matches_p[a:b].cpu().numpy(), E22, E22, np.zeros(0, np.int64), True, False)
    nm = G._normalisation(pts, E22, E22)
    f = lambda v: np.asarray(v, dtype=np.float64)
    q = np.stack([(f(pts[:, 0]) - nm.c0x) * nm.i0, (f(pts[:, 1]) - nm.c0y) * nm.i0,
                  (f(pts[:, 2]) - nm.c1x) * nm.i1, (f(pts[:, 3]) - nm.c1y) * nm.i1], 1)
    fl = G.fundamental_inliers(h["F_hypothesis"].reshape(1, 9), pts, t2)[0]
    A = G._epipolar_rows(q[fl])
    w, V = np.linalg.eigh(A.T @ A)
    s = np.linalg.svd(V[:, 0].reshape(3, 3), compute_uv=False)
    return float(w[-1] / (w[1] - w[0]) + s[0] / (s[1] - s[2]))


def _masks_at(res, p, F, thresh, min_overlap):
    """The host model's point mask and line decisions of pair p under a given pixel F: -> (inliers_p, lines, pts, rp)
    with pts the correspondences and rp their match rows."""
    a, b = res.offsets_p[p:p + 2]
    c, e = res.offsets_l[p:p + 2]
    pts, _, _, rp, _ = G._correspondences(res.keypoints0[p].cpu().numpy(), res.keypoints1[p].cpu().numpy(),
                                          res.matches_p[a:b].cpu().numpy(), E22, E22, np.zeros(0, np.int64), True,
                                          False)
    mp = np.zeros(b - a, np.uint8)
    mp[rp] = G.fundamental_inliers(F.reshape(1, 9), pts, thresh * thresh)[0]
    ml = res.matches_l[c:e].cpu().numpy().astype(np.int64)
    k1 = np.asarray(res.klines1[p], np.float32).reshape(-1, 2, 2)
    rl = np.flatnonzero((ml >= 0) & (ml < len(k1)))
    lines = np.zeros(e - c, np.uint8)
    if len(rl):
        k0 = np.asarray(res.klines0[p], np.float32).reshape(-1, 2, 2)
        lines[rl] = G.lines_consistent(F, k0[rl], k1[ml[rl]], min_overlap)
    return mp, lines, pts, rp


def _residual_band(F, pts, tol):
    """How far a relative F error of tol (entrywise, relative to max |F|) can move the FM residual r = |x1^T F x0| /
    |n| of each correspondence (n the smaller epipolar line normal, (F x0)_xy or (F^T x1)_xy).  With |dF_ij| <= eps =
    tol max |F|: |d(x1^T F x0)| <= eps |x1|_1 |x0|_1 and |d|n|| <= sqrt(2) eps |x|_1 (x the point the normal is taken
    at, homogeneous), so to first order |dr| <= (eps |x1|_1 |x0|_1 + r sqrt(2) eps |x|_1) / |n|, taking the larger of the
    two normals' bounds.  Twice that covers the second-order terms and r being taken at one of the two F."""
    F = np.asarray(F, dtype=np.float64).reshape(1, 9)
    num, na, nb = (v[0] for v in G._fm_terms(F, pts))
    eps = tol * np.abs(F).max()
    h0 = np.abs(pts[:, 0]) + np.abs(pts[:, 1]) + 1.0
    h1 = np.abs(pts[:, 2]) + np.abs(pts[:, 3]) + 1.0
    with np.errstate(all="ignore"):
        r = np.abs(num) / np.sqrt(np.minimum(na, nb))
        band = np.maximum((eps * h1 * h0 + r * np.sqrt(2.0) * eps * h0) / np.sqrt(na),
                          (eps * h1 * h0 + r * np.sqrt(2.0) * eps * h1) / np.sqrt(nb))
    return r, 2.0 * band


def check_pair(res, got, p, thresh=3.0, stats=None, **kw):
    """Pair p of an estimate_fundamentals result (numpy fields) against the host model: validity, the hypothesis and
    its inlier count exactly; F bit for bit unless the refit was kept, else within FM_REFIT_C u refit_condition of the
    host's (relative to its largest entry).  The masks: bit for bit without a kept refit; with one, the point mask and
    line decisions must be exactly the host model's at the kernel's F (the inlier test and the line check are
    explicitly rounded, so no band is needed there), and a point row may differ from the host's own mask only where
    its residual lies within `_residual_band` of the threshold.  Counts equal to the masks."""
    h = _host_pair(res, p, thresh=thresh, **kw)
    assert bool(got["valid"][p]) == h["valid"], p
    assert got["hypothesis"][p] == h["hypothesis"] and got["hypothesis_inliers"][p] == h["hypothesis_inliers"], p
    a, b = res.offsets_p[p:p + 2]
    c, e = res.offsets_l[p:p + 2]
    gm, gl = got["inliers_p"][a:b], got["lines_consistent"][c:e]
    if not h["valid"]:
        assert np.isnan(got["F"][p]).all() and not gm.any() and not gl.any() and got["n_lines_consistent"][p] == 0
        assert got["n_inliers"][p] == 0 and not got["refit"][p], p
        return h
    assert bool(got["refit"][p]) == h["refit"], p
    assert got["n_inliers"][p] == gm.sum() and got["n_lines_consistent"][p] == gl.sum(), p
    if not h["refit"]:
        assert np.array_equal(got["F"][p].reshape(9).view(np.int64), h["F"].reshape(9).view(np.int64)), p
        assert np.array_equal(gm, h["inliers_p"]) and np.array_equal(gl, h["lines_consistent"]), p
        return h
    cond = refit_condition(res, p, h, thresh * thresh)
    err = float(np.abs(got["F"][p] - h["F"]).max() / np.abs(h["F"]).max())
    if stats is not None:
        stats.append(err / (U * cond))
    tol = FM_REFIT_C * U * cond
    assert err <= tol, (p, err, cond, tol)
    mp, ml, pts, rp = _masks_at(res, p, got["F"][p], thresh, kw.get("min_overlap", 0.5))
    assert np.array_equal(gm, mp) and np.array_equal(gl, ml), p
    diff = np.flatnonzero(gm[rp] != h["inliers_p"][rp])
    if len(diff):
        r, band = _residual_band(h["F"], pts[diff].astype(np.float64), tol)
        assert np.all(np.abs(r - thresh) <= band), (p, r, band)
    return h


@pytest.mark.gpu
def test_kernels_match_host_model():
    cases = _ragged_cases()
    res = _matches(cases)
    Kh, seed = 256, 5
    out = G.estimate_fundamentals(res, n_hypotheses=Kh, seed=seed)
    got = {f: getattr(out, f).cpu().numpy() for f in FIELDS}
    ratios = []
    for p in range(res.n_pairs):
        check_pair(res, got, p, stats=ratios, n_hypotheses=Kh, seed=seed)
    print(f"{res.n_pairs} pairs, {int(got['valid'].sum())} valid, {int(got['refit'].sum())} refitted; worst refit "
          f"|dF| / (u cond) {max(ratios, default=0.0):.3g}")
    assert not got["valid"][::10].any()                       # the pairs below 7 correspondences


@pytest.mark.gpu
def test_deterministic_and_seed_independent_on_clean_data():
    cases = [syn.make_fundamental_correspondences(50 + i, 400, 40, noise_px=0.0, outlier_frac=0.5) for i in range(16)]
    res = _matches(cases, shuffle_rows=False)
    a, b = G.estimate_fundamentals(res, seed=3), G.estimate_fundamentals(res, seed=3)
    for f in FIELDS:
        assert torch.equal(getattr(a, f), getattr(b, f)), f
    c = G.estimate_fundamentals(res, seed=4)
    assert not torch.equal(a.hypothesis, c.hypothesis)
    assert torch.equal(a.inliers_p, c.inliers_p) and torch.equal(a.lines_consistent, c.lines_consistent)
    true_p = torch.from_numpy(np.concatenate([d["true_p"] for d in cases]).astype(np.uint8)).to(DEV)
    true_l = torch.from_numpy(np.concatenate([d["true_l"] for d in cases]).astype(np.uint8)).to(DEV)
    assert torch.equal(a.inliers_p, true_p) and torch.equal(a.lines_consistent, true_l)
    assert a.refit.all()
    for p, d in enumerate(cases):
        assert _sign_free(a.F[p].cpu().numpy(), d["F"]) < 1e-6, p


@pytest.mark.gpu
def test_end_to_end_match_images_and_match_sets():
    """`make_pose_set` views, their intrinsics ignored: F from match_images and match_set agree, and the noise-free
    projections of the scene's points lie within 0.5 px (median 0.2 px) of their epipolar lines under it, with 0.1 px
    keypoint noise and the 3 px default threshold."""
    from tests.test_image_pairs import _model
    model, _ = _model()
    eng = engine.PairEngine(model, DEV)
    views, Tv = syn.make_pose_set(31, 6, 60, 400, jitter_px=0.1)
    views = [syn.image_to(v, DEV) for v in views]
    pairs = engine.exhaustive_pairs(len(views))
    r_img = eng.match_images([views[i] for i, _ in pairs], [views[j] for _, j in pairs])
    r_set = eng.match_set(eng.encode_images(views), pairs)
    a, b = G.estimate_fundamentals(r_img), G.estimate_fundamentals(r_set)
    for f in FIELDS:
        assert torch.equal(getattr(a, f), getattr(b, f)), f
    K = syn.DEFAULT_K
    worst, med = [], []
    for p, (i, j) in enumerate(pairs):
        T = Tv[j] @ np.linalg.inv(Tv[i])
        Ft = syn.fundamental_from_pose(K, K, T[:3, :3], T[:3, 3])
        # points on the true epipolar geometry: the matched keypoints moved onto their true epipolar lines
        pa, pb = r_img.offsets_p[p:p + 2]
        m = r_img.matches_p[pa:pb].cpu().numpy()
        rows = np.flatnonzero(a.inliers_p[pa:pb].cpu().numpy())
        x0 = r_img.keypoints0[p].cpu().numpy()[rows]
        x1 = r_img.keypoints1[p].cpu().numpy()[m[rows]]
        l = np.c_[x0, np.ones(len(x0))] @ Ft.T
        x1 = x1 - ((np.c_[x1, np.ones(len(x1))] * l).sum(1) / (l[:, 0] ** 2 + l[:, 1] ** 2))[:, None] * l[:, :2]
        dist = _sym_dist(a.F[p].cpu().numpy(), np.concatenate([x0, x1], 1).astype(np.float64)) / 2
        worst.append(float(np.percentile(dist, 90)))
        med.append(float(np.median(dist)))
    print(f"{len(pairs)} pairs: median epipolar distance of true correspondences per pair {np.round(med, 3).tolist()}; "
          f"90th percentile max {max(worst):.3f} px; inliers {a.n_inliers.tolist()}")
    assert a.valid.all() and a.refit.all() and max(med) < 0.2 and max(worst) < 0.5


@pytest.mark.gpu
def test_capacity_and_struct_row_bounds_and_empty_batches(monkeypatch):
    big = syn.make_fundamental_correspondences(1, G.SMEM_MAX // G.SMEM_PER_ROW_F + 1, 0)
    N.reset_launch_count()
    with pytest.raises(N.LtrError, match=r"code -4"):
        G.estimate_fundamentals(_matches([big], shuffle_rows=False))
    assert N.launch_count() == 0
    # a C-ABI caller's max_rows_p sizes the staging; a pair with more rows is invalid, not staged
    res = _matches([syn.make_fundamental_correspondences(2, n, 10, outlier_frac=0.3) for n in (300, 100)],
                   shuffle_rows=False)
    call = G._ops.call_struct
    monkeypatch.setattr(G._ops, "call_struct",
                        lambda entry, inputs, *a, **kw: call(entry, {**inputs, "max_rows_p": 200}, *a, **kw))
    out = G.estimate_fundamentals(res, n_hypotheses=256)
    assert out.valid.tolist() == [False, True]
    assert not out.inliers_p[:300].any() and not out.lines_consistent[:10].any() and int(out.hypothesis[0]) == -1
    assert np.isnan(out.F[0].cpu().numpy()).all()
    assert int(out.hypothesis[1]) == _host_pair(res, 1, n_hypotheses=256)["hypothesis"]
    monkeypatch.undo()
    N.reset_launch_count()
    empty = G.estimate_fundamentals(_matches([]))
    assert N.launch_count() == 0 and empty.F.shape == (0, 3, 3)
    for kw in ({"thresh": 0.0}, {"min_overlap": 1.5}, {"n_hypotheses": 65535 * 128 + 1}):
        N.reset_launch_count()
        with pytest.raises(N.LtrError, match=r"code -1"):
            G.estimate_fundamentals(res, **kw)
        assert N.launch_count() == 0
