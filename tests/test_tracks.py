"""Tracks of posed image sets (`ltr_tracks`, `tracks.triangulate_tracks`) against the numpy model
`tracks.triangulate_tracks_host`, scipy, known scene geometry and `triangulate`, and end to end into
`estimate_absolute_poses`."""
import numpy as np
import pytest
import torch

from linetr_b200 import _native as N, engine, geometry as G, localization as L, synthetic as syn, tracks as TR
from linetr_b200 import triangulation as T
from tests.test_triangulation import _lines_of, _matches, _ragged, _res, _two_views

DEV = torch.device("cuda", 0)
K = syn.DEFAULT_K


def _ring(V, k=2):
    """Each image paired with its next k neighbours around a ring: [P, 2] distinct unordered pairs."""
    return np.array(sorted({tuple(sorted((i, (i + s) % V))) for i in range(V) for s in range(1, k + 1)}))


def _host(d, pairs, res=None, **kw):
    res = _matches(d, pairs) if res is None else res
    return TR.triangulate_tracks_host(d["keypoints"], d["klines"], pairs, res, d["K"], d["R"], d["t"], **kw)


def _rel(a, b):
    return np.abs(a - b).max(-1) / np.abs(b).max(-1)


def _track_rows(h, kind, t):
    o = h[f"track_off_{kind}"]
    return h[f"obs_{kind}"][o[t]:o[t + 1]]


# ------------------------------------------------------------------ CPU
def test_structure_of_a_noise_free_ring():
    """One track per 3D point and per segment, holding every view's row in ascending order, ids ordered by the minimum
    row, and labels equal to scipy's components over edges rebuilt here from the geometry module."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    V, n, m = 8, 40, 9
    pairs = _ring(V)
    d = syn.make_line_map_set(11, V, n, m)
    res = _matches(d, pairs)
    h = _host(d, pairs, res)
    for kind, cnt, pool, mt, off in (("p", n, d["keypoints"], res.matches_p, res.offsets_p),
                                     ("l", m, d["klines"], res.matches_l, res.offsets_l)):
        assert h[f"n_tracks_{kind}"] == cnt
        for t in range(cnt):
            rows = _track_rows(h, kind, t)
            assert np.array_equal(rows, t + cnt * np.arange(V))      # row t of every view, ascending
        assert (h[f"n_obs_{kind}"] == V).all() and (h[f"n_images_{kind}"] == V).all()
        assert (h[f"status_{kind}"] == TR.TRK_OK).all() and (h[f"n_inliers_{kind}"] == V).all()
        # independent components over the edges
        F, u, v, e_all = h["F"], [], [], []
        mt = mt.numpy()
        for p, (i, j) in enumerate(pairs):
            mm = mt[off[p]:off[p + 1]]
            if kind == "p":
                e = G.fundamental_inliers(F[p], np.concatenate([pool[i], pool[j][mm]], 1).astype(np.float64), 16.0)[0]
            else:
                e = G.lines_consistent(F[p], pool[i], pool[j][mm], 0.5)
            e_all.append(e)
            u.append(cnt * i + np.flatnonzero(e))
            v.append(cnt * j + mm[e])
        assert np.array_equal(np.concatenate(e_all), h[f"edges_{kind}"])
        A = coo_matrix((np.ones(sum(map(len, u))), (np.concatenate(u), np.concatenate(v))), shape=(V * cnt,) * 2)
        _, lab = connected_components(A, directed=False)
        mn = np.full(lab.max() + 1, V * cnt)
        np.minimum.at(mn, lab, np.arange(V * cnt))
        assert np.array_equal(mn[lab], h[f"label_{kind}"])
        assert np.array_equal(h[f"track_{kind}"], np.tile(np.arange(cnt), V))


def test_noise_free_geometry():
    V = 8
    pairs = _ring(V)
    d = syn.make_line_map_set(12, V, 60, 15)
    h = _host(d, pairs)
    assert _rel(h["points3d"], d["points3d"]).max() < 1e-6
    rp = h["row_points3d"].reshape(V, 60, 3)
    assert _rel(rp, d["points3d"][None]).max() < 1e-6 and (h["n_views_p"] == V).all()
    S = d["segments3d"]
    u = (S[:, 1] - S[:, 0]) / np.linalg.norm(S[:, 1] - S[:, 0], axis=1, keepdims=True)
    Lw = h["row_lines3d"].reshape(V, 15, 2, 3)
    assert h["inlier_l"].all()
    w = Lw - S[None, :, None, 0]
    off_line = np.linalg.norm(w - (w * u[None, :, None]).sum(-1, keepdims=True) * u[None, :, None], axis=-1)
    assert off_line.max() < 1e-6 * np.abs(S).max()
    for v in range(V):
        q = Lw[v].reshape(-1, 3) @ d["R"][v].T + d["t"][v]
        px = syn._project(K, q).reshape(-1, 2, 2)
        assert np.abs(px - d["klines"][v].astype(np.float64)).max() < 1e-6 * 640
    print(f"points {_rel(h['points3d'], d['points3d']).max():.1e}, lines off the true line {off_line.max():.1e}")


def test_epipolar_filter_matches_the_geometry_module():
    """F of every pair agrees with `fundamental_from_pose`; the edges are `fundamental_inliers` / `lines_consistent` of
    the match rows, row for row, on a scene with noise, moved observations and unmatched rows."""
    V = 7
    pairs = _ring(V, 3)
    d = syn.make_line_map_set(13, V, 120, 30, jitter_px=0.5, outlier_frac=0.3)
    res = _matches(d, pairs, lambda i, j: np.arange(120) % 9 == 0)
    h = _host(d, pairs, res, epi_thresh=3.0, min_overlap=0.6)
    for p, (i, j) in enumerate(pairs):
        R = d["R"][j] @ d["R"][i].T
        Fr = syn.fundamental_from_pose(K, K, R, d["t"][j] - R @ d["t"][i])
        assert np.abs(h["F"][p] - Fr).max() < 1e-12 * np.abs(Fr).max()
        mp = res.matches_p.numpy()[res.offsets_p[p]:res.offsets_p[p + 1]]
        ok = mp >= 0
        want = np.zeros(len(mp), bool)
        want[ok] = G.fundamental_inliers(h["F"][p], np.concatenate([d["keypoints"][i][ok], d["keypoints"][j][mp[ok]]],
                                                                   1).astype(np.float64), 9.0)[0]
        assert np.array_equal(h["edges_p"][res.offsets_p[p]:res.offsets_p[p + 1]], want)
        want_l = G.lines_consistent(h["F"][p], d["klines"][i], d["klines"][j], 0.6)
        assert np.array_equal(h["edges_l"][res.offsets_l[p]:res.offsets_l[p + 1]], want_l)
    print(f"point edges {h['edges_p'].mean():.3f}, line edges {h['edges_l'].mean():.3f}")


def _project(d, v, X):
    q = X @ d["R"][v].T + d["t"][v]
    return syn._project(K, q)


def test_refits_agree_with_scipy_least_squares():
    """At 0.5 px noise every kept refit is the least-squares solution over its supporters' residuals, computed here
    from the projections themselves: points to 1e-6 relative, and each line end point from the anchor's own pixel and
    the supporters' distances to their lines."""
    from scipy.optimize import least_squares
    V = 6
    pairs = _ring(V)
    d = syn.make_line_map_set(14, V, 80, 25, jitter_px=0.5)
    h = _host(d, pairs)
    img = lambda kind, r: int(np.searchsorted(h[f"offsets_{kind}"], r, side="right") - 1)
    worst, n = 0.0, 0
    pool_p = np.concatenate(d["keypoints"]).astype(np.float64)
    for t in np.flatnonzero(h["refit_p"]):
        rows = _track_rows(h, "p", t)
        sup = [rows[q] for q in range(len(rows)) if (int(h["support_p"][t]) >> q) & 1]

        def f(X):
            return np.concatenate([_project(d, img("p", r), X[None])[0] - pool_p[r] for r in sup])
        X = least_squares(f, h["winner_p"][t], xtol=1e-15, ftol=1e-15, gtol=1e-15).x
        worst, n = max(worst, _rel(X, h["points3d"][t])), n + 1
    pool_l = np.concatenate(d["klines"]).astype(np.float64)
    for t in np.flatnonzero(h["refit_l"]):
        rows = _track_rows(h, "l", t)
        a = int(h["anchor_l"][t])
        sup = [rows[q] for q in range(len(rows)) if (int(h["support_l"][t]) >> q) & 1 and q != a]
        for e in range(2):
            def f(X):
                out = list(_project(d, img("l", rows[a]), X[None])[0] - pool_l[rows[a], e])
                for r in sup:
                    s0, s1 = pool_l[r]
                    p = _project(d, img("l", r), X[None])[0]
                    dd = s1 - s0
                    out.append((dd[0] * (p[1] - s0[1]) - dd[1] * (p[0] - s0[0])) / np.linalg.norm(dd))
                return np.array(out)
            X = least_squares(f, h["winner_l"][t, e], xtol=1e-15, ftol=1e-15, gtol=1e-15).x
            worst, n = max(worst, _rel(X, h["lines3d"][t, e])), n + 1
    print(f"{n} refits, worst relative difference to scipy {worst:.1e}")
    assert n > 100 and worst < 1e-6


def _errors(d, pts, lns, mask_p, mask_l):
    V = len(d["keypoints"])
    ep = np.linalg.norm(pts.reshape(V, -1, 3) - d["points3d"][None], axis=-1)[mask_p]
    S = d["segments3d"]
    u = (S[:, 1] - S[:, 0]) / np.linalg.norm(S[:, 1] - S[:, 0], axis=1, keepdims=True)
    w = lns.reshape(V, -1, 2, 3) - S[None, :, None, 0]
    dl = np.linalg.norm(w - (w * u[None, :, None]).sum(-1, keepdims=True) * u[None, :, None], axis=-1).max(-1)
    return ep[np.isfinite(ep)], dl[mask_l][np.isfinite(dl[mask_l])]


def test_outliers():
    """30 % of the observations moved 10 to 60 px, the ring of `tools/tracks_bench.py` at a smaller size: a moved
    observation that joins a track is not its inlier unless the move kept it within thresh of the track's point; the
    unmoved rows are closer to the truth than `triangulate`'s, and far fewer moved rows get a valid 3D point."""
    V = 16
    pairs = _ring(V, 4)
    d = syn.make_line_map_set(15, V, 150, 30, jitter_px=0.5, outlier_frac=0.3)
    res = _matches(d, pairs)
    h = _host(d, pairs, res)
    tri = T.triangulate_host(d["keypoints"], d["klines"], pairs, res, d["K"], d["R"], d["t"])
    op, ol = d["outlier_p"].reshape(-1), d["outlier_l"].reshape(-1)
    joined = op & (h["track_p"] >= 0)
    inl = joined & (h["inlier_p"] == 1)
    pool = np.concatenate(d["keypoints"]).astype(np.float64)
    for r in np.flatnonzero(inl):
        v = int(np.searchsorted(h["offsets_p"], r, side="right") - 1)
        X = h["points3d"][h["track_p"][r]]
        if np.isfinite(X).all():
            assert np.linalg.norm(_project(d, v, X[None])[0] - pool[r]) <= 4.0 + 1e-9
    valid_p = np.isfinite(h["row_points3d"]).all(1)
    valid_t = np.isfinite(tri["points3d"]).all(1)
    ours, theirs = valid_p[op].mean(), valid_t[op].mean()
    e_ours, l_ours = _errors(d, h["row_points3d"], h["row_lines3d"], ~d["outlier_p"], ~d["outlier_l"])
    e_tri, l_tri = _errors(d, tri["points3d"], tri["lines3d"], ~d["outlier_p"], ~d["outlier_l"])
    print(f"moved rows: {joined.mean() / op.mean():.3f} joined a track, {inl.sum() / op.sum():.3f} inliers; valid 3D "
          f"points {ours:.3f} (triangulate {theirs:.3f}); unmoved median error {np.median(e_ours):.2e} "
          f"(triangulate {np.median(e_tri):.2e}), line distance {np.median(l_ours):.2e} ({np.median(l_tri):.2e}); "
          f"moved key lines valid {np.isfinite(h['row_lines3d']).all((1, 2))[ol].mean():.3f}")
    assert ours < 0.25 * theirs
    assert np.median(e_ours) < np.median(e_tri) and np.median(l_ours) < np.median(l_tri)
    assert valid_p[~op].mean() > 0.95


def _merge_scene(V, drop_views, n=12, seed=16):
    """A noise-free ring of V views; point 1 left unmatched in every pair that touches an image of drop_views (those
    rows are isolated), and a planted side-0 match of point 0 in pair 0 to point 1, with epi_thresh set just above its
    epipolar error so that it joins the two tracks."""
    pairs = _ring(V)
    d = syn.make_line_map_set(seed, V, n, 2)
    drop = lambda i, j: (np.arange(n) == 1) & (i in drop_views or j in drop_views)
    res = _matches(d, pairs, drop)
    i, j = pairs[0]
    F = TR.pair_fundamentals(T._check(d["keypoints"], d["klines"], pairs, res, d["K"], d["R"], d["t"]))[0]
    err = G.fundamental_error(F, np.concatenate([d["keypoints"][i][:1], d["keypoints"][j][1:2]], 1).astype(np.float64))
    mp = res.matches_p.clone()
    mp[0] = 1
    planted = _res(d["keypoints"], d["klines"], pairs, [mp.numpy()[res.offsets_p[p]:res.offsets_p[p + 1]]
                                                        for p in range(len(pairs))],
                   [res.matches_l.numpy()[res.offsets_l[p]:res.offsets_l[p + 1]] for p in range(len(pairs))])
    return d, pairs, res, planted, float(np.sqrt(err[0])) * 1.01 + 1e-3


def test_planted_false_merge_keeps_the_larger_track():
    d, pairs, res, planted, eth = _merge_scene(10, {4, 5, 6, 7})
    h0 = _host(d, pairs, res, epi_thresh=eth)
    h = _host(d, pairs, planted, epi_thresh=eth)
    t = h["track_p"][0]
    rows = _track_rows(h, "p", t)
    n = len(d["keypoints"][0])
    assert h["n_obs_p"][t] == 10 + 6 and h["n_images_p"][t] == 10 < h["n_obs_p"][t]
    assert h["status_p"][t] == TR.TRK_OK and h["n_inliers_p"][t] == 10
    point0, point1 = rows[rows % n == 0], rows[rows % n == 1]
    assert h["inlier_p"][point0].all() and not h["inlier_p"][point1].any()
    assert _rel(h["points3d"][t], d["points3d"][0]) < 1e-6
    assert h0["n_tracks_p"] == h["n_tracks_p"] + 1


def test_planted_false_merge_of_65_is_too_long():
    d, pairs, res, planted, eth = _merge_scene(33, {0}, n=6)
    h0 = _host(d, pairs, res, epi_thresh=eth)
    h = _host(d, pairs, planted, epi_thresh=eth)
    t = h["track_p"][0]
    assert h["n_obs_p"][t] == 65 and h["status_p"][t] == TR.TRK_TOO_LONG and h["n_inliers_p"][t] == 0
    assert np.isnan(h["points3d"][t]).all()
    rows = _track_rows(h, "p", t)
    assert not h["inlier_p"][rows].any() and np.isnan(h["row_points3d"][rows]).all()
    other = np.setdiff1d(np.arange(len(h["track_p"])), rows)
    assert np.array_equal(h["row_points3d"][other].view(np.int64), h0["row_points3d"][other].view(np.int64))
    assert np.array_equal(h["row_lines3d"].view(np.int64), h0["row_lines3d"].view(np.int64))


def test_degenerate_cases():
    rng = np.random.default_rng(5)
    X = np.c_[rng.uniform(-1, 1, (40, 2)), rng.uniform(4, 8, 40)]
    pairs = np.array([[0, 1]])

    def run(kps, kls, Rs, ts, mp=None, **kw):
        mp = np.arange(len(kps[0]), dtype=np.int32) if mp is None else mp
        res = _res(kps, kls, pairs, [mp], [np.arange(len(kls[0]), dtype=np.int32)])
        return TR.triangulate_tracks_host(kps, kls, pairs, res, K, Rs, ts, **kw)

    # a baseline below min_angle: tracks, but no candidate
    kps, Rs, ts = _two_views(X, [0.01, 0, 0])
    kls = _lines_of(np.stack([X[:10], X[:10] + [0, 0.5, 0.2]], 1), Rs, ts)
    h = run(kps, kls, Rs, ts)
    assert h["n_tracks_p"] == 40 and (h["status_p"] == TR.TRK_NO_CANDIDATE).all() and np.isnan(h["points3d"]).all()
    assert (h["status_l"] == TR.TRK_NO_CANDIDATE).all() and np.isnan(h["row_lines3d"]).all()
    h0 = run(kps, kls, Rs, ts, min_angle=0.0)
    assert (h0["status_p"] == TR.TRK_OK).all()
    # points behind camera 1
    kps, Rs, ts = _two_views(X, [0.5, 0, -3.0], np.diag([-1.0, 1.0, -1.0]))
    h = run(kps, kls, Rs, ts)
    assert np.isnan(h["points3d"]).all() and np.isnan(h["row_points3d"]).all() and not h["n_views_p"].any()
    # two rows of image 0 joined through image 1 (rows 0 and 1 both match row 0): their own pair gives no candidate
    kps, Rs, ts = _two_views(X, [1.0, 0, 0])
    kps[0][1] = kps[0][0] + [0.3, -0.2]
    mp = np.arange(40, dtype=np.int32)
    mp[1] = 0
    mp[7] = -1
    h = run(kps, kls, Rs, ts, mp)
    t = h["track_p"][0]
    assert h["n_obs_p"][t] == 3 and h["n_images_p"][t] == 2 and h["track_p"][1] == t
    assert (h["anchor_p"][t], h["partner_p"][t]) != (0, 1) and h["status_p"][t] == TR.TRK_OK
    # rows in no edge
    assert h["track_p"][7] == -1 and h["track_p"][47] == -1 and h["track_p"][41] == -1


def test_argument_errors_before_device_work():
    """The errors of `triangulate`, raised on the host (these pass on a machine without a GPU); an image in more
    than LTR_TRI_MAX_VIEWS pairs is accepted."""
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
                    (dict(keypoints=[d["keypoints"][0], d["keypoints"][1], d["keypoints"][2][:-1]]), "side 1"),
                    (dict(thresh=0.0), "thresh"), (dict(epi_thresh=np.inf), "epi_thresh"),
                    (dict(min_angle=90.0), "min_angle"), (dict(min_views=0), "min_views")):
        for f in (TR.triangulate_tracks, TR.triangulate_tracks_host):
            with pytest.raises(N.LtrError, match=msg):
                f(**args(**kw))
    n = N.TRI_MAX_VIEWS + 2
    kps, kls = [np.zeros((2, 2), np.float32)] * n, [np.zeros((0, 2, 2), np.float32)] * n
    star = np.array([[0, j] for j in range(1, n)])
    res = _res(kps, kls, star, [np.arange(2, dtype=np.int32)] * len(star), [np.zeros(0, np.int32)] * len(star))
    Rn, tn = np.broadcast_to(np.eye(3), (n, 3, 3)), np.zeros((n, 3))
    with pytest.raises(N.LtrError, match="more than LTR_TRI_MAX_VIEWS"):
        T.triangulate(kps, kls, star, res, K, Rn, tn)
    h = TR.triangulate_tracks_host(kps, kls, star, res, K, Rn, tn)
    assert h["row_points3d"].shape == (2 * n, 3)


# ------------------------------------------------------------------ GPU
_FIELDS = ("track", "track_off", "obs", "n_obs", "n_inliers", "n_images", "status", "inlier", "n_views")


def _compare(g, h):
    """Differing words between the device result and the host model over everything the call writes."""
    diff = 0
    nt = g.n_tracks()
    assert nt == (h["n_tracks_p"], h["n_tracks_l"])
    for kind, T_ in zip("pl", nt):
        rows = int(h[f"offsets_{kind}"][-1])
        n_obs = int(h[f"track_off_{kind}"][-1])
        for f in _FIELDS:
            a = getattr(g, f"{f}_{kind}").cpu().numpy()
            b = h[f"{f}_{kind}"]
            size = {"track_off": T_ + 1, "obs": n_obs, "track": rows, "inlier": rows, "n_views": rows}.get(f, T_)
            a, b = a[:size], b[:size]
            assert a.shape == b.shape, (f, kind)
            diff += int((a.astype(np.int64) != b.astype(np.int64)).sum())
    for f, kind in (("points3d", "p"), ("lines3d", "l"), ("row_points3d", "p"), ("row_lines3d", "l")):
        n = (h[f"n_tracks_{kind}"] if not f.startswith("row") else int(h[f"offsets_{kind}"][-1]))
        a, b = getattr(g, f).cpu().numpy()[:n], h[f]
        assert a.shape == b.shape, f
        diff += int((np.ascontiguousarray(a).view(np.int64) != np.ascontiguousarray(b).view(np.int64)).sum())
    return diff


@pytest.mark.gpu
def test_kernels_match_host_model_bit_for_bit():
    """Ragged sets (empty images, images in no pair, both pair orientations, unmatched, out-of-range and many-to-one
    matches, non-finite pixels) and merged tracks of exactly 64 and 65 observations."""
    cases = []
    for seed in range(3):
        d, pairs, mp, ml = _ragged(seed)
        kw = dict(thresh=[4.0, 2.0, 6.0][seed], min_angle=[1.5, 0.5, 3.0][seed], min_views=[2, 3, 1][seed],
                  epi_thresh=[4.0, 2.0, 8.0][seed], min_overlap=[0.5, 0.3, 0.7][seed])
        cases.append((d, pairs, _res(d["keypoints"], d["klines"], pairs, mp, ml), kw, seed == 1))
    for drop in ({0, 5}, {0}):
        d, pairs, _, planted, eth = _merge_scene(33, drop, n=6)
        cases.append((d, pairs, planted, dict(epi_thresh=eth), False))
    for d, pairs, res, kw, on_dev in cases:
        h = TR.triangulate_tracks_host(d["keypoints"], d["klines"], pairs, res, d["K"], d["R"], d["t"], **kw)
        kps = [torch.from_numpy(k).to(DEV) for k in d["keypoints"]] if on_dev else d["keypoints"]
        rd = _res(kps, d["klines"], pairs, [res.matches_p.numpy()[res.offsets_p[p]:res.offsets_p[p + 1]]
                                            for p in range(len(pairs))],
                  [res.matches_l.numpy()[res.offsets_l[p]:res.offsets_l[p + 1]] for p in range(len(pairs))], DEV)
        g = TR.triangulate_tracks(kps, d["klines"], pairs, rd, d["K"], d["R"], d["t"], **kw)
        diff = _compare(g, h)
        print(f"{h['n_tracks_p']} point tracks (statuses {np.bincount(h['status_p'], minlength=4).tolist()}), "
              f"{h['n_tracks_l']} line tracks ({np.bincount(h['status_l'], minlength=4).tolist()}), longest "
              f"{max(h['n_obs_p'].max(initial=0), h['n_obs_l'].max(initial=0))}; {diff} differing words")
        assert diff == 0
    assert {64, 65} <= {int(x) for c in cases[3:] for x in
                        TR.triangulate_tracks_host(c[0]["keypoints"], c[0]["klines"], c[1], c[2], K, c[0]["R"],
                                                   c[0]["t"], **c[3])["n_obs_p"]}


@pytest.mark.gpu
def test_deterministic():
    d, pairs, mp, ml = _ragged(7)
    res = _res(d["keypoints"], d["klines"], pairs, mp, ml, DEV)
    a, b = (TR.triangulate_tracks(d["keypoints"], d["klines"], pairs, res, d["K"], d["R"], d["t"]) for _ in range(2))
    for f in TR.TrackResult.__dataclass_fields__:
        x, y = getattr(a, f), getattr(b, f)
        if not isinstance(x, torch.Tensor) or f in ("track_off_p", "track_off_l"):
            continue
        if f in ("track_p", "track_l", "inlier_p", "inlier_l", "row_points3d", "row_lines3d",
                 "n_views_p", "n_views_l", "n_tracks_p", "n_tracks_l"):
            assert torch.equal(x.view(torch.int64) if x.dtype == torch.float64 else x,
                               y.view(torch.int64) if y.dtype == torch.float64 else y), f
    nt = a.n_tracks()
    for kind, n in zip("pl", nt):
        for f in ("track_off", "n_obs", "n_inliers", "n_images", "status"):
            m = n + 1 if f == "track_off" else n
            assert torch.equal(getattr(a, f"{f}_{kind}")[:m], getattr(b, f"{f}_{kind}")[:m]), f
        n_obs = int(getattr(a, f"track_off_{kind}")[n])
        assert torch.equal(getattr(a, f"obs_{kind}")[:n_obs], getattr(b, f"obs_{kind}")[:n_obs])
    assert torch.equal(a.points3d[:nt[0]].view(torch.int64), b.points3d[:nt[0]].view(torch.int64))
    assert torch.equal(a.lines3d[:nt[1]].view(torch.int64), b.lines3d[:nt[1]].view(torch.int64))
    N.reset_launch_count()
    TR.triangulate_tracks(d["keypoints"], d["klines"], pairs, res, d["K"], d["R"], d["t"])
    assert N.launch_count() == 6


@pytest.mark.gpu
def test_end_to_end_points_localize_against_the_track_map():
    """make_pose_set views 1 to 5 are matched with `match_set` and joined into tracks with their true poses; view 0 is
    then localized against the rows' track points as well as against the true 3D points."""
    from tests.test_image_pairs import _model
    model, _ = _model()
    eng = engine.PairEngine(model, DEV)
    views, Tv, X = syn.make_pose_set(41, 6, 60, 400, return_points=True)
    images = eng.encode_images([syn.image_to(v, DEV) for v in views])
    db = [(i, j) for i in range(1, 6) for j in range(i + 1, 6)]
    res = eng.match_set(images, db)
    tr = TR.triangulate_tracks(images.keypoints, images.klines, db, res, K, Tv[:, :3, :3], Tv[:, :3, 3])
    pts, _ = tr.rows().per_image()
    ok = np.isfinite(np.concatenate(pts[1:])).all(1)
    err = np.linalg.norm(np.concatenate(pts[1:])[ok] - np.tile(X, (5, 1))[ok], axis=1)
    print(f"{ok.mean():.3f} of the database keypoints on a valid track ({tr.n_tracks()[0]} point tracks), 3D error "
          f"median {np.median(err):.1e}")
    assert ok.mean() > 0.8 and np.median(err) < 0.02
    q = [(0, j) for j in range(1, 6)]
    rq = eng.match_set(images, q)
    est = L.estimate_absolute_poses(rq, K, [pts[j] for _, j in q], groups=[0, 5])
    ref = L.estimate_absolute_poses(rq, K, [X] * 5, groups=[0, 5])
    e_tr = L.absolute_pose_errors(est.R, est.t, Tv[0, :3, :3], Tv[0, :3, 3])
    e_ref = L.absolute_pose_errors(ref.R, ref.t, Tv[0, :3, :3], Tv[0, :3, 3])
    print(f"query against the track map: centre {e_tr[0][0]:.4f}, rotation {e_tr[1][0]:.4f} deg; against the true "
          f"points: {e_ref[0][0]:.4f}, {e_ref[1][0]:.4f} deg")
    assert est.valid.all() and e_tr[0][0] < max(3 * e_ref[0][0], 0.05) and e_tr[1][0] < max(3 * e_ref[1][0], 0.2)


@pytest.mark.gpu
def test_end_to_end_lines_localize_a_view_with_three_points():
    """A line-track map of five posed views (ground-truth matches, 0.5 px noise, 20 % outliers) localizes a sixth view
    that has only three point matches."""
    d = syn.make_line_map_set(8, 6, 200, 120, jitter_px=0.5, outlier_frac=0.2)
    db = np.array([(i, j) for i in range(1, 6) for j in range(i + 1, 6)])
    res = _matches(d, db, device=DEV)
    tr = TR.triangulate_tracks(d["keypoints"], d["klines"], db, res, d["K"], d["R"], d["t"])
    pts, lns = tr.rows().per_image()
    valid_l = np.isfinite(np.concatenate(lns[1:])).all((1, 2)).mean()
    print(f"{valid_l:.3f} of the database key lines on a valid track")
    assert valid_l > 0.6
    q = np.array([(0, j) for j in range(1, 6)])
    three = np.flatnonzero(~d["outlier_p"].any(0))[:3]
    few = lambda i, j: ~np.isin(np.arange(len(d["keypoints"][i])), three)
    rq = _matches(d, q, drop_p=few, device=DEV)
    est = L.estimate_absolute_poses(rq, d["K"], [pts[j] for _, j in q], [lns[j] for _, j in q], groups=[0, 5])
    e = L.absolute_pose_errors(est.R, est.t, d["R"][0], d["t"][0])
    print(f"with lines: centre {e[0][0]:.4f}, rotation {e[1][0]:.4f} deg ({int(est.n_inliers_l[0])} line inliers)")
    assert est.valid.all() and e[0][0] < 0.2 and e[1][0] < 2.0
    assert int(est.n_inliers_l[0]) > 0.5 * len(rq.matches_l)
