"""Triangulation of posed images (`ltr_triangulate`, `triangulation.triangulate`) against the numpy model
`triangulation.triangulate_host`, known scene geometry, scipy and OpenCV, and end to end into `estimate_absolute_poses`."""
import numpy as np
import pytest
import torch

from linetr_b200 import _native as N, engine, localization as L, synthetic as syn, triangulation as T

DEV = torch.device("cuda", 0)
K = syn.DEFAULT_K


def _matches(d, pairs, drop_p=None, drop_l=None, device="cpu"):
    """The ground-truth ImagePairMatches of a `make_line_map_set` scene (row i of every view is point / segment i)
    for pairs [P, 2]; drop_p(i, j) / drop_l(i, j) -> bool rows of pair (i, j) to leave unmatched."""
    mp, ml = [], []
    for i, j in pairs:
        a = np.arange(len(d["keypoints"][i]), dtype=np.int32)
        b = np.arange(len(d["klines"][i]), dtype=np.int32)
        if drop_p is not None:
            a[drop_p(i, j)] = -1
        if drop_l is not None:
            b[drop_l(i, j)] = -1
        mp.append(a)
        ml.append(b)
    return _res(d["keypoints"], d["klines"], pairs, mp, ml, device)


def _res(kps, kls, pairs, mp, ml, device="cpu"):
    offp = np.concatenate([[0], np.cumsum([len(x) for x in mp])]).astype(np.int32)
    offl = np.concatenate([[0], np.cumsum([len(x) for x in ml])]).astype(np.int32)
    cat = lambda x: torch.from_numpy(np.concatenate(x).astype(np.int32) if len(x) else np.zeros(0, np.int32)).to(device)
    mpt, mlt = cat(mp), cat(ml)
    z = torch.zeros(len(pairs), dtype=torch.int32, device=device)
    return engine.ImagePairMatches(mlt, mlt.float(), z, offl, mpt, mpt.float(), z, offp,
                                   [kls[i] for i, _ in pairs], [kls[j] for _, j in pairs],
                                   [kps[i] for i, _ in pairs], [kps[j] for _, j in pairs])


def _host(d, pairs, res=None, **kw):
    res = _matches(d, pairs) if res is None else res
    return T.triangulate_host(d["keypoints"], d["klines"], pairs, res, d["K"], d["R"], d["t"], **kw)


def _rel(a, b):
    return np.abs(a - b).max(-1) / np.abs(b).max(-1)


# ------------------------------------------------------------------ CPU
def test_noise_free_scene_matches_ground_truth():
    """Keypoints and segment end points are stored as float32 (an error of up to 3e-5 px), which bounds how close the
    3D estimates get: 1e-6 of the distance.  What does not depend on that storage holds to 1e-9: every end point
    projects onto its own anchor end point."""
    V, pairs = 5, engine.exhaustive_pairs(5)
    d = syn.make_line_map_set(1, V, 300, 60)
    h = _host(d, pairs)
    X = h["points3d"].reshape(V, -1, 3)
    assert (h["n_views_p"] == V).all() and (h["n_views_l"] >= 2).all()
    assert _rel(X, d["points3d"][None]).max() < 1e-6
    Lw = h["lines3d"].reshape(V, -1, 2, 3)
    assert _rel(Lw, d["lines3d"]).max() < 1e-6
    S = d["segments3d"]
    u = (S[:, 1] - S[:, 0]) / np.linalg.norm(S[:, 1] - S[:, 0], axis=1, keepdims=True)
    w = Lw - S[None, :, None, 0]
    off_line = np.linalg.norm(w - (w * u[None, :, None]).sum(-1, keepdims=True) * u[None, :, None], axis=-1)
    assert off_line.max() < 1e-6 * np.abs(S).max()
    for v in range(V):
        q = Lw[v].reshape(-1, 3) @ d["R"][v].T + d["t"][v]
        px = syn._project(K, q).reshape(-1, 2, 2)
        assert np.abs(px - d["klines"][v].astype(np.float64)).max() < 1e-9 * 640
    print(f"points: max relative error {_rel(X, d['points3d'][None]).max():.1e}; lines {_rel(Lw, d['lines3d']).max():.1e}")


def _point_residuals(d, a, k, views, pairs, mask, s):
    """The reprojection errors of the supporters (bits of mask) of anchor a's keypoint k at depth s, computed directly."""
    Ra, ta = d["R"][a], d["t"][a]
    x = d["keypoints"][a][k].astype(np.float64)
    r = Ra.T @ np.linalg.solve(K, [x[0], x[1], 1.0])
    X = -Ra.T @ ta + s * r
    out = []
    for o, code in enumerate(views):
        if (int(mask) >> o) & 1:
            v = pairs[code >> 1][1 - (code & 1)]
            q = d["R"][v] @ X + d["t"][v]
            out += list(K[:2, :2] @ (q[:2] / q[2]) + K[:2, 2] - d["keypoints"][v][k])
    return np.array(out)


def _end_residuals(d, a, k, e, views, pairs, mask, s):
    Ra, ta = d["R"][a], d["t"][a]
    x = d["klines"][a][k, e].astype(np.float64)
    X = -Ra.T @ ta + s * (Ra.T @ np.linalg.solve(K, [x[0], x[1], 1.0]))
    out = []
    for o, code in enumerate(views):
        if (int(mask) >> o) & 1:
            v = pairs[code >> 1][1 - (code & 1)]
            q = d["R"][v] @ X + d["t"][v]
            p = K[:2, :2] @ (q[:2] / q[2]) + K[:2, 2]
            s0, s1 = d["klines"][v][k].astype(np.float64)
            dd = s1 - s0
            out.append((dd[0] * (p[1] - s0[1]) - dd[1] * (p[0] - s0[0])) / np.linalg.norm(dd))
    return np.array(out)


def test_refit_agrees_with_scipy_least_squares():
    """With 0.5 px noise every kept refit depth is the least-squares depth of its supporters' pixel residuals (each
    residual computed here from the projection itself) to 1e-6 relative."""
    from scipy.optimize import least_squares
    V, pairs = 5, engine.exhaustive_pairs(5)
    d = syn.make_line_map_set(2, V, 120, 30, jitter_px=0.5)
    h = _host(d, pairs)
    worst, n = 0.0, 0
    for a in range(V):
        views = h["view_off"][a], h["view_off"][a + 1]
        views = h["views"][views[0]:views[1]]
        for k in range(0, 120, 3):
            row = h["offsets_p"][a] + k
            if not h["refit_p"][row]:
                continue
            f = lambda s: _point_residuals(d, a, k, views, pairs, h["support_p"][row], s[0])
            s = least_squares(f, [h["winner_p"][row]], xtol=1e-15, ftol=1e-15, gtol=1e-15).x[0]
            worst, n = max(worst, abs(s - h["depth_p"][row]) / s), n + 1
        for k in range(30):
            row = h["offsets_l"][a] + k
            if not h["refit_l"][row]:
                continue
            for e in range(2):
                f = lambda s: _end_residuals(d, a, k, e, views, pairs, h["support_l"][row], s[0])
                s = least_squares(f, [h["winner_l"][row, e]], xtol=1e-15, ftol=1e-15, gtol=1e-15).x[0]
                worst, n = max(worst, abs(s - h["depth_l"][row, e]) / s), n + 1
    print(f"{n} refit depths, worst relative difference to scipy {worst:.1e}")
    assert n > 300 and worst < 1e-6


def test_two_view_points_against_opencv():
    cv2 = pytest.importorskip("cv2")
    d = syn.make_line_map_set(3, 2, 400, 0, jitter_px=0.5)
    pairs = np.array([[0, 1]])
    h = _host(d, pairs, min_angle=0.0, thresh=1e3)
    P = [K @ np.c_[d["R"][v], d["t"][v]] for v in range(2)]
    Xh = cv2.triangulatePoints(P[0], P[1], d["keypoints"][0].T.astype(np.float64), d["keypoints"][1].T.astype(np.float64))
    Xc = (Xh[:3] / Xh[3]).T
    ours = h["points3d"][:400]
    depth = np.linalg.norm(d["points3d"] + d["R"][0].T @ d["t"][0], axis=1)
    diff = np.linalg.norm(ours - Xc, axis=1) / depth
    err_ours = np.linalg.norm(ours - d["points3d"], axis=1) / depth
    err_cv = np.linalg.norm(Xc - d["points3d"], axis=1) / depth
    print(f"relative distance to cv2 median {np.median(diff):.1e}, max {diff.max():.1e}; to the truth ours "
          f"{np.median(err_ours):.1e}, cv2 {np.median(err_cv):.1e}")
    assert (h["n_views_p"][:400] == 2).all()
    assert np.median(diff) < 0.5 * np.median(err_cv) and diff.max() < 3 * err_cv.max()
    assert np.median(err_ours) < 1.5 * np.median(err_cv)


def test_outliers_are_excluded():
    """30 % of the observations moved 10 to 60 px: for every anchor row that was not moved itself, n_views and the
    result equal those computed with the moved observations unmatched, and n_views counts every unmoved partner.  Of
    the key lines at least 97 % of the rows pass both: a line's support is decided at both end points of a noisy segment,
    so a clean partner now and then falls outside the threshold."""
    V, pairs = 7, engine.exhaustive_pairs(7)
    d = syn.make_line_map_set(4, V, 300, 60, jitter_px=0.3, outlier_frac=0.3)
    h = _host(d, pairs)
    op, ol = d["outlier_p"], d["outlier_l"]
    clean = _host(d, pairs, _matches(d, pairs, lambda i, j: op[i] | op[j], lambda i, j: ol[i] | ol[j]))
    for kind, out, n in (("p", op, 300), ("l", ol, 60)):
        nv, nvc = h["n_views_" + kind].reshape(V, n), clean["n_views_" + kind].reshape(V, n)
        want = np.broadcast_to(V - out.sum(0), out.shape)     # the anchor and its unmoved partners
        rows = ~out & (want >= 3)
        print(f"{kind}: {rows.sum()} rows, n_views == unmoved views in {np.mean((nv == want)[rows]):.4f}")
        assert np.mean((nv == want)[rows]) >= (1.0 if kind == "p" else 0.97)
        X = (h["points3d"] if kind == "p" else h["lines3d"]).reshape(V, n, -1)
        Xc = (clean["points3d"] if kind == "p" else clean["lines3d"]).reshape(V, n, -1)
        same = (nv == nvc)[rows] & (_rel(X[rows], Xc[rows]) < 1e-9)
        print(f"{kind}: equal to the result without the moved observations in {same.mean():.4f}")
        assert same.mean() >= (1.0 if kind == "p" else 0.97)


def _two_views(X, c1, R1=np.eye(3)):
    """Two views of the world points X [n, 3]: camera 0 at the origin, camera 1 with rotation R1 and centre c1."""
    Rs, ts = np.stack([np.eye(3), R1]), np.stack([np.zeros(3), -R1 @ np.asarray(c1, dtype=np.float64)])
    kps = []
    for R, t in zip(Rs, ts):
        q = X @ R.T + t
        kps.append((q[:, :2] / q[:, 2:] * 500.0 + [319.5, 239.5]).astype(np.float32))
    return kps, Rs, ts


def _lines_of(E, Rs, ts):
    return [np.stack([(q[..., :2] / q[..., 2:] * 500.0 + [319.5, 239.5]) for q in (E @ R.T + t,)], 0)[0]
            .astype(np.float32) for R, t in zip(Rs, ts)]


def test_degenerate_rows_give_nan():
    rng = np.random.default_rng(5)
    X = np.c_[rng.uniform(-1, 1, (40, 2)), rng.uniform(4, 8, 40)]
    pairs = np.array([[0, 1]])

    def run(kps, kls, Rs, ts, res=None, **kw):
        res = _res(kps, kls, pairs, [np.arange(len(kps[0]), dtype=np.int32)],
                   [np.arange(len(kls[0]), dtype=np.int32)]) if res is None else res
        return T.triangulate_host(kps, kls, pairs, res, K, Rs, ts, **kw)

    # a baseline of 0.01 units at depth 4 to 8: below 1.5 degrees, above 0
    kps, Rs, ts = _two_views(X, [0.01, 0, 0])
    E = np.stack([X[:10], X[:10] + [0, 0.5, 0.2]], 1)
    kls = _lines_of(E, Rs, ts)
    h = run(kps, kls, Rs, ts)
    assert np.isnan(h["points3d"]).all() and np.isnan(h["lines3d"]).all()
    assert not h["n_views_p"].any() and not h["n_views_l"].any()
    h0 = run(kps, kls, Rs, ts, min_angle=0.0)
    assert (h0["n_views_p"] == 2).all() and np.isfinite(h0["points3d"]).all()
    # a wide baseline along x: lines parallel to it lie in an epipolar plane, lines along y do not
    kps, Rs, ts = _two_views(X, [1.0, 0, 0])
    E = np.concatenate([np.stack([X[:10], X[:10] + [0.8, 0, 0]], 1), np.stack([X[10:20], X[10:20] + [0, 0.8, 0]], 1)])
    h = run(kps, _lines_of(E, Rs, ts), Rs, ts)
    assert np.isnan(h["lines3d"][:10]).all() and not h["n_views_l"][:10].any()
    assert (h["n_views_l"][10:20] == 2).all() and _rel(h["lines3d"][10:20], E[10:20]).max() < 1e-6
    assert (h["n_views_p"] == 2).all()
    # every point behind camera 1 (it looks the other way)
    Rb = np.diag([-1.0, 1.0, -1.0])
    kps, Rs, ts = _two_views(X, [0.5, 0, -3.0], Rb)
    h = run(kps, _lines_of(E, Rs, ts), Rs, ts)
    assert np.isnan(h["points3d"]).all() and not h["n_views_p"].any() and not h["n_views_l"].any()
    # rows with no partner: an image in no pair, unmatched rows; and non-finite keypoints
    kps, Rs, ts = _two_views(X, [1.0, 0, 0])
    kls = _lines_of(E, Rs, ts)
    kps = [kps[0].copy(), kps[1].copy(), kps[0]]
    kps[0][3] = np.nan
    kps[1][5, 0] = np.inf
    kls = [kls[0], kls[1], kls[0]]
    m = np.arange(40, dtype=np.int32)
    m[7] = -1
    res = _res(kps, kls, pairs, [m], [np.arange(20, dtype=np.int32)])
    h = T.triangulate_host(kps, kls, pairs, res, K, np.concatenate([Rs, Rs[:1]]), np.concatenate([ts, ts[:1]]))
    nv = h["n_views_p"]
    assert (nv[:40][[3, 5, 7]] == 0).all() and (nv[40:80][[3, 5, 7]] == 0).all() and not nv[80:].any()
    assert np.isnan(h["points3d"][80:]).all() and np.isnan(h["lines3d"][40:]).all()
    keep = np.setdiff1d(np.arange(40), [3, 5, 7])
    assert (nv[keep] == 2).all() and (nv[40 + keep] == 2).all()


def test_argument_errors_before_device_work():
    """Every check runs on the host before anything touches a device (these pass on a machine without one)."""
    d = syn.make_line_map_set(6, 3, 20, 5)
    pairs = engine.exhaustive_pairs(3)
    res = _matches(d, pairs)
    args = lambda **kw: {**dict(keypoints=d["keypoints"], klines=d["klines"], pairs=pairs, res=res, K=d["K"],
                                R=d["R"], t=d["t"]), **kw}
    for kw, msg in ((dict(K=np.diag([-500.0, 500.0, 1.0])), "fx, fy > 0"), (dict(K=np.eye(4)), "K must be"),
                    (dict(R=d["R"][:2]), "R must be"), (dict(t=d["t"][:, :2]), "t \\["),
                    (dict(t=d["t"] * np.array([[np.nan, 1, 1]] * 3)), "finite"),
                    (dict(pairs=pairs[:2]), "2 pairs but"), (dict(pairs=np.array([[0, 1], [2, 2], [1, 2]])), "self pair"),
                    (dict(pairs=np.array([[0, 1], [1, 0], [0, 2]])), "listed twice"),
                    (dict(pairs=np.array([[0, 1], [0, 5], [1, 2]])), "in \\[0, 3\\)"),
                    (dict(keypoints=[d["keypoints"][0][:-1], d["keypoints"][1], d["keypoints"][2]]), "match rows"),
                    (dict(keypoints=[d["keypoints"][0], d["keypoints"][1], d["keypoints"][2][:-1]]), "side 1")):
        for f in (T.triangulate, T.triangulate_host):
            with pytest.raises(N.LtrError, match=msg):
                f(**args(**kw))
    n = N.TRI_MAX_VIEWS + 2
    kps, kls = [np.zeros((2, 2), np.float32)] * n, [np.zeros((0, 2, 2), np.float32)] * n
    star = np.array([[0, j] for j in range(1, n)])
    res = _res(kps, kls, star, [np.arange(2, dtype=np.int32)] * len(star), [np.zeros(0, np.int32)] * len(star))
    Rn, tn = np.broadcast_to(np.eye(3), (n, 3, 3)), np.zeros((n, 3))
    with pytest.raises(N.LtrError, match="more than LTR_TRI_MAX_VIEWS"):
        T.triangulate(kps, kls, star, res, K, Rn, tn)
    h = T.triangulate_host(kps, kls, star[:-1], _res(kps, kls, star[:-1], [np.arange(2, dtype=np.int32)] * (n - 2),
                                                     [np.zeros(0, np.int32)] * (n - 2)), K, Rn, tn)
    assert h["points3d"].shape == (2 * n, 3)


# ------------------------------------------------------------------ GPU
def _ragged(seed=0):
    """Nine images of one scene with ragged contents: images without keypoints or key lines, images in no pair, pairs
    in both directions, unmatched and wrongly matched rows, several side-0 rows matched to one side-1 row, non-finite
    keypoints, outliers and noise."""
    rng = np.random.default_rng(seed)
    d = syn.make_line_map_set(100 + seed, 9, 400, 80, jitter_px=0.7, outlier_frac=0.2)
    kps, kls = [k.copy() for k in d["keypoints"]], [k.copy() for k in d["klines"]]
    cut_p = [400, 0, 400, 250, 400, 400, 400, 13, 400]
    cut_l = [80, 80, 0, 80, 40, 80, 80, 80, 1]
    kps = [k[:c] for k, c in zip(kps, cut_p)]
    kls = [k[:c] for k, c in zip(kls, cut_l)]
    kps[0][::37] = np.nan
    kls[3][5, 1, 0] = np.inf
    pairs = np.array([[0, 1], [2, 0], [0, 3], [3, 4], [5, 3], [4, 0], [5, 6], [6, 0], [3, 2], [4, 7], [8, 3], [6, 4]])
    mp, ml = [], []
    for i, j in pairs:
        for src, dst, n0, n1 in ((mp, None, len(kps[i]), len(kps[j])), (ml, None, len(kls[i]), len(kls[j]))):
            m = np.where(np.arange(n0) < n1, np.arange(n0), -1).astype(np.int32)
            m[rng.random(n0) < 0.1] = -1
            wrong = rng.random(n0) < 0.05
            m[wrong] = rng.integers(-2, max(n1, 1) + 3, wrong.sum())
            src.append(m)
    d.update(keypoints=kps, klines=kls)
    return d, pairs, mp, ml


@pytest.mark.gpu
def test_kernels_match_host_model_bit_for_bit():
    for seed in range(3):
        d, pairs, mp, ml = _ragged(seed)
        kw = dict(thresh=[4.0, 2.0, 6.0][seed], min_angle=[1.5, 0.5, 3.0][seed], min_views=[2, 3, 1][seed])
        h = T.triangulate_host(d["keypoints"], d["klines"], pairs, _res(d["keypoints"], d["klines"], pairs, mp, ml),
                               d["K"], d["R"], d["t"], **kw)
        kps = [torch.from_numpy(k).to(DEV) for k in d["keypoints"]] if seed == 1 else d["keypoints"]
        res = _res(kps, d["klines"], pairs, mp, ml, DEV)
        g = T.triangulate(kps, d["klines"], pairs, res, d["K"], d["R"], d["t"], **kw)
        diff = 0
        for f in ("points3d", "lines3d", "n_views_p", "n_views_l"):
            a, b = getattr(g, f).cpu().numpy(), h[f]
            assert a.shape == b.shape, f
            diff += int((np.ascontiguousarray(a).view(np.int64 if a.dtype == np.float64 else np.int32)
                         != np.ascontiguousarray(b).view(np.int64 if b.dtype == np.float64 else np.int32)).sum())
        print(f"seed {seed}: {int((h['n_views_p'] > 0).sum())} of {len(h['n_views_p'])} points and "
              f"{int((h['n_views_l'] > 0).sum())} of {len(h['n_views_l'])} lines valid; {diff} differing words")
        assert diff == 0
        assert (h["n_views_p"] > 0).sum() > 500 and (h["n_views_l"] > 0).sum() > 100


@pytest.mark.gpu
def test_deterministic():
    d, pairs, mp, ml = _ragged(7)
    res = _res(d["keypoints"], d["klines"], pairs, mp, ml, DEV)
    a, b = (T.triangulate(d["keypoints"], d["klines"], pairs, res, d["K"], d["R"], d["t"]) for _ in range(2))
    for f in ("points3d", "lines3d", "n_views_p", "n_views_l"):
        x, y = getattr(a, f), getattr(b, f)
        assert torch.equal(x.view(torch.int64) if x.dtype == torch.float64 else x,
                           y.view(torch.int64) if y.dtype == torch.float64 else y), f
    N.reset_launch_count()
    T.triangulate(d["keypoints"], d["klines"], pairs, res, d["K"], d["R"], d["t"])
    assert N.launch_count() == 2


@pytest.mark.gpu
def test_end_to_end_points_localize_against_the_triangulated_map():
    """make_pose_set views 1 to 5 are matched with `match_set` and triangulated with their true poses; view 0 is then
    localized against that map as well as against the true 3D points."""
    from tests.test_image_pairs import _model
    model, _ = _model()
    eng = engine.PairEngine(model, DEV)
    views, Tv, X = syn.make_pose_set(41, 6, 60, 400, return_points=True)
    images = eng.encode_images([syn.image_to(v, DEV) for v in views])
    db = [(i, j) for i in range(1, 6) for j in range(i + 1, 6)]
    res = eng.match_set(images, db)
    tri = T.triangulate(images.keypoints, images.klines, db, res, K, Tv[:, :3, :3], Tv[:, :3, 3])
    pts, _ = tri.per_image()
    nv = tri.n_views_p.cpu().numpy()
    ok = np.isfinite(np.concatenate(pts[1:])).all(1)
    err = np.linalg.norm(np.concatenate(pts[1:])[ok] - np.tile(X, (5, 1))[ok], axis=1)
    print(f"{ok.mean():.3f} of the database keypoints triangulated, n_views {np.bincount(nv).tolist()}, 3D error "
          f"median {np.median(err):.1e}")
    assert ok.mean() > 0.9 and np.median(err) < 0.02
    assert np.isnan(pts[0]).all()
    q = [(0, j) for j in range(1, 6)]
    rq = eng.match_set(images, q)
    est = L.estimate_absolute_poses(rq, K, [pts[j] for _, j in q], groups=[0, 5])
    ref = L.estimate_absolute_poses(rq, K, [X] * 5, groups=[0, 5])
    e_tri = L.absolute_pose_errors(est.R, est.t, Tv[0, :3, :3], Tv[0, :3, 3])
    e_ref = L.absolute_pose_errors(ref.R, ref.t, Tv[0, :3, :3], Tv[0, :3, 3])
    print(f"query against the triangulated map: centre {e_tri[0][0]:.4f}, rotation {e_tri[1][0]:.4f} deg; against the "
          f"true points: {e_ref[0][0]:.4f}, {e_ref[1][0]:.4f} deg")
    assert est.valid.all() and e_tri[0][0] < max(3 * e_ref[0][0], 0.05) and e_tri[1][0] < max(3 * e_ref[1][0], 0.2)


@pytest.mark.gpu
def test_end_to_end_lines_localize_a_view_with_three_points():
    """A line map triangulated from five posed views (ground-truth matches, 0.5 px noise, 20 % outliers) localizes a
    sixth view that has only three point matches, the fewest P3P can sample: most of its line matches are inliers and
    its pose is within 0.2 units and 2 degrees (scene depth 4 to 9 units)."""
    d = syn.make_line_map_set(8, 6, 200, 120, jitter_px=0.5, outlier_frac=0.2)
    db = np.array([(i, j) for i in range(1, 6) for j in range(i + 1, 6)])
    res = _matches(d, db, device=DEV)
    tri = T.triangulate(d["keypoints"], d["klines"], db, res, d["K"], d["R"], d["t"])
    pts, lns = tri.per_image()
    valid_l = np.isfinite(np.concatenate(lns[1:])).all((1, 2)).mean()
    print(f"{valid_l:.3f} of the database key lines triangulated")
    assert valid_l > 0.7
    q = np.array([(0, j) for j in range(1, 6)])
    three = np.flatnonzero(~d["outlier_p"].any(0))[:3]            # points no view moved
    few = lambda i, j: ~np.isin(np.arange(len(d["keypoints"][i])), three)
    rq = _matches(d, q, drop_p=few, device=DEV)
    args = (rq, d["K"], [pts[j] for _, j in q], [lns[j] for _, j in q])
    with_l = L.estimate_absolute_poses(*args, groups=[0, 5])
    no_l = L.estimate_absolute_poses(*args, groups=[0, 5], use_lines=False)
    R0, t0 = d["R"][0], d["t"][0]
    e_l = L.absolute_pose_errors(with_l.R, with_l.t, R0, t0)
    e_p = L.absolute_pose_errors(no_l.R, no_l.t, R0, t0)
    print(f"with lines: centre {e_l[0][0]:.4f}, rotation {e_l[1][0]:.4f} deg ({int(with_l.n_inliers_l[0])} line "
          f"inliers); three points alone: {e_p[0][0]:.4f}, {e_p[1][0]:.4f} deg")
    assert with_l.valid.all() and e_l[0][0] < 0.2 and e_l[1][0] < 2.0
    assert int(with_l.n_inliers_l[0]) > 0.5 * len(rq.matches_l)
