"""Bundle adjustment (linetr_b200.bundle): the GPU kernels bit for bit against the numpy model, the model against
scipy.optimize.least_squares on the same residuals, its accuracy on synthetic scenes, and the argument checks."""
import dataclasses

import numpy as np
import pytest
import torch
from scipy.optimize import least_squares
from scipy.spatial.transform import Rotation as Rot

from linetr_b200 import _native as N
from linetr_b200 import bundle as BA
from linetr_b200 import synthetic as syn
from linetr_b200 import tracks as TR
from linetr_b200.engine import ImagePairMatches
from linetr_b200.localization import cayley


def ring_matches(d, pairs, dev):
    n, m = len(d["points3d"]), len(d["segments3d"])
    P = len(pairs)
    mp = torch.arange(n, dtype=torch.int32, device=dev).repeat(P)
    ml = torch.arange(m, dtype=torch.int32, device=dev).repeat(P)
    z = torch.zeros(P, dtype=torch.int32, device=dev)
    kp, kl = d["keypoints"], d["klines"]
    return ImagePairMatches(ml, ml.float(), z, np.arange(P + 1, dtype=np.int32) * m, mp, mp.float(), z,
                            np.arange(P + 1, dtype=np.int32) * n, [kl[i] for i, _ in pairs], [kl[j] for _, j in pairs],
                            [kp[i] for i, _ in pairs], [kp[j] for _, j in pairs])


def perturb(d, seed, deg=0.3, shift=0.03, skip=(0,)):
    rng = np.random.default_rng(seed)
    R, t = d["R"].copy(), d["t"].copy()
    for v in range(len(R)):
        if v in skip:
            continue
        dR = Rot.from_rotvec(rng.normal(size=3) / np.sqrt(3) * np.deg2rad(deg)).as_matrix()
        C = -R[v].T @ t[v] + rng.normal(size=3) / np.sqrt(3) * shift
        R[v] = dR @ R[v]
        t[v] = -R[v] @ C
    return R, t


def scene(seed=0, V=12, n_pts=120, n_lines=24, jitter=0.5, ring=3, deg=0.3, shift=0.03, skip=(0,)):
    d = syn.make_line_map_set(seed, V, n_pts, n_lines, jitter_px=jitter)
    pairs = np.array([(i, (i + k) % V) for i in range(V) for k in range(1, ring + 1)], dtype=np.int32)
    R, t = perturb(d, seed + 100, deg, shift, skip)
    return d, pairs, R, t


def host_tracks(d, pairs, R, t):
    res = ring_matches(d, pairs, torch.device("cpu"))
    return TR.triangulate_tracks_host(d["keypoints"], d["klines"], pairs, res, d["K"], R, t, thresh=8, epi_thresh=8)


def centres(R, t):
    return np.einsum("nji,nj->ni", R, -t)


def rot_err_deg(Ra, Rb):
    c = (np.einsum("nij,nij->n", Ra, Rb) - 1) / 2
    return np.degrees(np.arccos(np.clip(c, -1, 1)))


# ------------------------------------------------------------------ the independent solver
def scipy_ba(d, tr, out, R0, t0, fixed):
    """scipy.optimize.least_squares on the model's residuals, parametrization and gauge, started from the input."""
    n = len(R0)
    st_p, st_l = out["status_p"], out["status_l"]
    op, ol = tr["offsets_p"], tr["offsets_l"]
    kp = np.concatenate(d["keypoints"]).astype(np.float64)
    kl = np.concatenate([k.reshape(-1, 4) for k in d["klines"]]).astype(np.float64)
    K = d["K"]
    C0 = centres(R0, t0)
    obs = []
    part = np.zeros(n, bool)
    for kind, st, off in (("p", st_p, op), ("l", st_l, ol)):
        for tt in np.flatnonzero(st == BA.BA_IN):
            o = tr[f"obs_{kind}"][tr[f"track_off_{kind}"][tt]:tr[f"track_off_{kind}"][tt + 1]]
            o = o[tr[f"inlier_{kind}"][o].astype(bool)]
            im = np.searchsorted(off, o, side="right") - 1
            obs.append((kind, tt, o, im))
            part[im] = True
    free = [i for i in range(n) if i not in fixed and part[i]]
    held = None
    if len(fixed) == 1 and free:
        k = free[0]
        held = (k, int(np.argmax(np.abs(C0[k] - C0[fixed[0]]))))
    cam_idx = []
    for i in free:
        for a in range(6):
            if held and i == held[0] and a == 3 + held[1]:
                continue
            cam_idx.append((i, a))
    P0 = tr["points3d"][st_p == BA.BA_IN]
    L0 = tr["lines3d"].reshape(-1, 6)[st_l == BA.BA_IN]
    basis = []
    for X in L0:
        dd = X[3:] - X[:3]
        e = np.zeros(3)
        e[np.argmin(np.abs(dd))] = 1
        u1 = np.cross(dd, e)
        u1 /= np.linalg.norm(u1)
        u2 = np.cross(dd, u1)
        basis.append((u1, u2 / np.linalg.norm(u2)))
    pidx = {tt: j for j, tt in enumerate(np.flatnonzero(st_p == BA.BA_IN))}
    lidx = {tt: j for j, tt in enumerate(np.flatnonzero(st_l == BA.BA_IN))}
    nc, npn = len(cam_idx), 3 * len(P0)

    def unpack(x):
        dc = np.zeros((n, 6))
        for (i, a), v in zip(cam_idx, x[:nc]):
            dc[i, a] = v
        R = np.stack([cayley(dc[i, :3]) @ R0[i] for i in range(n)])
        C = C0 + dc[:, 3:]
        P = P0 + x[nc:nc + npn].reshape(-1, 3)
        dl = x[nc + npn:].reshape(-1, 4)
        L = np.stack([np.concatenate([X[:3] + b[0] * q[0] + b[1] * q[1], X[3:] + b[0] * q[2] + b[1] * q[3]])
                      for X, b, q in zip(L0, basis, dl)]) if len(L0) else np.zeros((0, 6))
        return R, C, P, L

    def fun(x):
        R, C, P, L = unpack(x)
        r = []
        for kind, tt, o, im in obs:
            Rr, Cr, Kr = R[im], C[im], K[im] if K.ndim == 3 else np.broadcast_to(K, (len(im), 3, 3))
            if kind == "p":
                Q = np.einsum("nij,nj->ni", Rr, P[pidx[tt]] - Cr)
                px = kp[o]
                r += [(Kr[:, 0, 0] * Q[:, 0] - (px[:, 0] - Kr[:, 0, 2]) * Q[:, 2]) / Q[:, 2],
                      (Kr[:, 1, 1] * Q[:, 1] - (px[:, 1] - Kr[:, 1, 2]) * Q[:, 2]) / Q[:, 2]]
            else:
                s = kl[o]
                a, b, c = s[:, 1] - s[:, 3], s[:, 2] - s[:, 0], s[:, 0] * s[:, 3] - s[:, 2] * s[:, 1]
                nn = np.hypot(a, b)
                la, lb, lc = a / nn, b / nn, c / nn
                nv = np.stack([la * Kr[:, 0, 0], lb * Kr[:, 1, 1], la * Kr[:, 0, 2] + lb * Kr[:, 1, 2] + lc], 1)
                for e in range(2):
                    Q = np.einsum("nij,nj->ni", Rr, L[lidx[tt], 3 * e:3 * e + 3] - Cr)
                    r.append((nv * Q).sum(1) / Q[:, 2])
        return np.concatenate(r)

    x0 = np.zeros(nc + npn + 4 * len(L0))
    sol = least_squares(fun, x0, method="trf", x_scale="jac", ftol=1e-15, xtol=1e-15, gtol=1e-15, max_nfev=200)
    R, C, P, L = unpack(sol.x)
    return dict(cost=float((sol.fun ** 2).sum()), R=R, C=C, P=P, L=L, held=held)


def line_dist(La, Lb):
    """Largest distance of Lb's end points to the infinite lines of La: [T]."""
    d = La[:, 3:] - La[:, :3]
    d = d / np.linalg.norm(d, axis=1, keepdims=True)
    out = []
    for e in range(2):
        w = Lb[:, 3 * e:3 * e + 3] - La[:, :3]
        out.append(np.linalg.norm(w - (w * d).sum(1, keepdims=True) * d, axis=1))
    return np.maximum(*out)


def points_only(d):
    return dict(d, klines=[k[:0] for k in d["klines"]], segments3d=d["segments3d"][:0])


@pytest.mark.parametrize("fixed", [(0,), (0, 3)])
def test_host_model_matches_scipy(fixed):
    # points only: a line's end points move in the plane orthogonal to its current direction, so the reachable end
    # points depend on the path; lines are checked from the model's own minimum below
    d, pairs, R, t = scene(0, V=12)
    d = points_only(d)
    tr = host_tracks(d, pairs, R, t)
    out = BA.bundle_adjust_host(d["keypoints"], d["klines"], d["K"], R, t, tr, fixed=fixed, max_iters=50,
                                ftol=1e-14)
    ref = scipy_ba(d, tr, out, R, t, list(fixed))
    s = out["stats"]
    assert s["accepted"] >= 1 and s["final_cost"] < s["initial_cost"]
    assert abs(s["final_cost"] - ref["cost"]) <= 1e-8 * ref["cost"]
    assert np.all(np.diff(out["history"]) < 0)
    np.testing.assert_allclose(out["R"], ref["R"], rtol=0, atol=1e-6)
    np.testing.assert_allclose(centres(out["R"], out["t"]), ref["C"], rtol=1e-6, atol=1e-6)
    P = out["points3d"][out["status_p"] == BA.BA_IN]
    np.testing.assert_allclose(P, ref["P"], rtol=1e-6, atol=1e-6)
    for f in fixed:
        assert np.array_equal(out["R"][f].view(np.uint64), R[f].view(np.uint64))
        assert np.array_equal(out["t"][f].view(np.uint64), t[f].view(np.uint64))
    if ref["held"]:
        # the held coordinate of the adjusted centre keeps its input bits (t = -R C then rounds it once more)
        k, e = ref["held"]
        assert out["C"][k, e].view(np.uint64) == BA._centres(R, t)[k, e].view(np.uint64)
        assert not np.array_equal(out["C"][k], BA._centres(R, t)[k])


def test_host_model_lines_at_scipy_minimum():
    """From the model's result, scipy on the same residuals, parametrization and gauge finds no lower cost."""
    d, pairs, R, t = scene(0, V=12)
    tr = host_tracks(d, pairs, R, t)
    out = BA.bundle_adjust_host(d["keypoints"], d["klines"], d["K"], R, t, tr, fixed=(0, 3), max_iters=50,
                                ftol=1e-14)
    assert np.all(np.diff(out["history"]) < 0) and (out["status_l"] == BA.BA_IN).sum() > 10
    at = dict(tr, points3d=out["points3d"], lines3d=out["lines3d"])
    ref = scipy_ba(d, at, out, out["R"], out["t"], [0, 3])
    assert ref["cost"] >= out["stats"]["final_cost"] * (1 - 1e-8)
    L = out["lines3d"].reshape(-1, 6)[out["status_l"] == BA.BA_IN]
    assert line_dist(ref["L"], L).max() < 1e-6 * np.abs(L).max()
    np.testing.assert_allclose(out["R"], ref["R"], rtol=0, atol=1e-6)


def similarity(A, B):
    """(s, Q, c) minimising |s Q A_i + c - B_i| (Umeyama)."""
    ma, mb = A.mean(0), B.mean(0)
    U, S, Vt = np.linalg.svd((B - mb).T @ (A - ma))
    D = np.diag([1, 1, np.sign(np.linalg.det(U @ Vt))])
    Q = U @ D @ Vt
    s = np.trace(np.diag(S) @ D) / ((A - ma) ** 2).sum()
    return s, Q, mb - s * Q @ ma


def test_noise_free_poses_return_to_truth():
    # one fixed image: the scale comes from the perturbed input, so compare after a similarity alignment
    d, pairs, R, t = scene(1, V=12, jitter=0.0)
    tr = host_tracks(d, pairs, R, t)
    out = BA.bundle_adjust_host(d["keypoints"], d["klines"], d["K"], R, t, tr, fixed=(0,), max_iters=50)
    C, Cg = centres(out["R"], out["t"]), centres(d["R"], d["t"])
    s, Q, c = similarity(C, Cg)
    scale = np.linalg.norm(Cg - Cg.mean(0), axis=1).max()
    assert np.abs(s * C @ Q.T + c - Cg).max() < 1e-6 * scale * 10
    assert rot_err_deg(out["R"] @ Q.T, d["R"]).max() < 1e-4
    s0, Q0, c0 = similarity(centres(R, t), Cg)
    assert np.abs(s0 * centres(R, t) @ Q0.T + c0 - Cg).max() > 1e3 * np.abs(s * C @ Q.T + c - Cg).max()
    assert out["stats"]["final_cost"] < 1e-6 * out["stats"]["initial_cost"]


def test_noise_reduces_errors():
    for seed in (2, 3):
        d, pairs, R, t = scene(seed, V=12, jitter=0.5, skip=(0, 1))
        tr = host_tracks(d, pairs, R, t)
        out = BA.bundle_adjust_host(d["keypoints"], d["klines"], d["K"], R, t, tr, fixed=(0, 1), max_iters=50)
        Cg = centres(d["R"], d["t"])
        assert np.median(np.linalg.norm(centres(out["R"], out["t"]) - Cg, axis=1)[2:]) < \
            np.median(np.linalg.norm(centres(R, t) - Cg, axis=1)[2:])
        assert np.median(rot_err_deg(out["R"], d["R"])[2:]) < np.median(rot_err_deg(R, d["R"])[2:])
        sel = out["status_p"] == BA.BA_IN
        gt = d["points3d"]
        assert np.median(np.linalg.norm(out["points3d"][sel] - gt[sel], axis=1)) < \
            np.median(np.linalg.norm(tr["points3d"][sel] - gt[sel], axis=1))
        rp = out["residual_p"][np.isfinite(out["residual_p"])]
        assert 0.3 < np.sqrt(np.mean(rp ** 2)) < 1.0
        sl = out["status_l"] == BA.BA_IN
        seg = true_segments(d, tr)
        assert np.median(line_to_segment(out["lines3d"], seg)[sl]) < \
            np.median(line_to_segment(tr["lines3d"], seg)[sl])


def true_segments(d, tr):
    """The true 3D segment of every line track (its first row's: row l of every view is segment l)."""
    ol = np.asarray(tr["offsets_l"])
    first = np.asarray(tr["obs_l"])[np.asarray(tr["track_off_l"])[:int(tr["n_tracks_l"])]]
    return d["segments3d"][first - ol[np.searchsorted(ol, first, side="right") - 1]]


def line_to_segment(L, seg):
    """Larger distance of the end points L [T, 2, 3] to the true segments' lines [T]."""
    u = seg[:, 1] - seg[:, 0]
    u = u / np.linalg.norm(u, axis=1, keepdims=True)
    w = L.reshape(-1, 2, 3) - seg[:, :1]
    return np.linalg.norm(w - (w * u[:, None]).sum(-1, keepdims=True) * u[:, None], axis=-1).max(1)


def make_degenerate(d, R, t, tr):
    """A 2-view line track in the epipolar plane, hand-built from the first valid line track of `tr` (a
    TrackResult or a host dict): its first two inlier rows stay inliers, its line becomes X_a + s (C_j - C_i) and both
    rows' key lines become that line's projections.  -> (klines, inlier_l, lines3d, track)."""
    obs, off = BA._get(tr, "obs_l").astype(np.int64), BA._get(tr, "track_off_l").astype(np.int64)
    st, inl = BA._get(tr, "status_l"), BA._get(tr, "inlier_l").copy()
    L = BA._get(tr, "lines3d").reshape(-1, 2, 3).copy()
    ol = np.asarray(tr["offsets_l"] if isinstance(tr, dict) else tr.offsets_l)
    K = np.broadcast_to(d["K"], (len(R), 3, 3)) if np.ndim(d["K"]) == 2 else d["K"]
    for k in range(len(off) - 1):
        rows = obs[off[k]:off[k + 1]]
        rows = rows[inl[rows] == 1]
        if st[k] != N.TRK_OK or len(rows) < 2:
            continue
        inl[rows[2:]] = 0
        img = np.searchsorted(ol, rows[:2], side="right") - 1
        C = centres(R, t)
        Xa = L[k, 0]
        Xb = Xa + (C[img[1]] - C[img[0]])
        L[k, 1] = Xb
        kl = [x.copy() for x in d["klines"]]
        for r, v in zip(rows[:2], img):
            p = [K[v] @ (R[v] @ X + t[v]) for X in (Xa, Xb)]
            kl[v].reshape(-1, 4)[r - ol[v]] = [p[0][0] / p[0][2], p[0][1] / p[0][2], p[1][0] / p[1][2], p[1][1] / p[1][2]]
        return kl, inl, L, k
    raise AssertionError("no valid line track")


def test_degenerate_line_is_left_out():
    d, pairs, R, t = scene(8, V=8, n_pts=30, n_lines=8, ring=2)
    tr = host_tracks(d, pairs, R, t)
    kl, inl, L, k = make_degenerate(d, R, t, tr)
    trd = dict(tr, inlier_l=inl, lines3d=L)
    out = BA.bundle_adjust_host(d["keypoints"], kl, d["K"], R, t, trd)
    assert out["status_l"][k] == BA.BA_DEGENERATE
    assert (out["status_l"] == BA.BA_IN).sum() == (tr["status_l"] == N.TRK_OK).sum() - 1
    assert np.array_equal(out["lines3d"][k], L[k])
    assert np.isnan(out["residual_l"][inl == 1][np.isin(np.flatnonzero(inl == 1),
                                                        tr["obs_l"][tr["track_off_l"][k]:tr["track_off_l"][k + 1]])]).all()
    assert out["stats"]["accepted"] >= 1


def test_structure_only_is_per_track_minimum():
    d, pairs, R, t = scene(4, V=12, n_pts=40, n_lines=8)
    d = points_only(d)
    tr = host_tracks(d, pairs, R, t)
    out = BA.bundle_adjust_host(d["keypoints"], d["klines"], d["K"], R, t, tr, fixed=tuple(range(12)),
                                max_iters=50, ftol=1e-14)
    ref = scipy_ba(d, tr, out, R, t, list(range(12)))
    assert np.array_equal(out["R"], R) and np.array_equal(out["t"], t)
    np.testing.assert_allclose(out["points3d"][out["status_p"] == BA.BA_IN], ref["P"], rtol=1e-6, atol=1e-6)
    assert abs(out["stats"]["final_cost"] - ref["cost"]) <= 1e-8 * ref["cost"]


def test_zero_iterations_pass_through():
    d, pairs, R, t = scene(5, V=8, ring=2)
    tr = host_tracks(d, pairs, R, t)
    out = BA.bundle_adjust_host(d["keypoints"], d["klines"], d["K"], R, t, tr, max_iters=0)
    assert np.array_equal(out["R"], R) and np.array_equal(out["t"], t)
    assert np.array_equal(out["row_points3d"], tr["row_points3d"], equal_nan=True)
    assert np.array_equal(out["row_lines3d"], tr["row_lines3d"], equal_nan=True)
    assert out["stats"]["iterations"] == 0 and out["stats"]["stop_reason"] == BA.BA_STOP_ITERS


def test_refusals_before_device_work():
    d, pairs, R, t = scene(6, V=6, n_pts=20, n_lines=4, ring=2)
    tr = host_tracks(d, pairs, R, t)
    args = (d["keypoints"], d["klines"], d["K"], R, t, tr)
    for fn in (BA.bundle_adjust, BA.bundle_adjust_host):
        with pytest.raises(N.LtrError, match="fixed"):
            fn(*args, fixed=())
        with pytest.raises(N.LtrError, match="fixed"):
            fn(*args, fixed=(6,))
        for bad in (-1, BA.BA_MAX_ITERS + 1):
            with pytest.raises(N.LtrError, match="max_iters"):
                fn(*args, max_iters=bad)
        for bad in (float("nan"), float("inf"), -1.0):
            with pytest.raises(N.LtrError, match="ftol"):
                fn(*args, ftol=bad)
        with pytest.raises(N.LtrError, match="disagree"):
            fn(d["keypoints"][:5] + [d["keypoints"][5][:3]], d["klines"], d["K"], R, t, tr)
    n = BA.BA_MAX_IMAGES + 1
    big = dict(offsets_p=np.zeros(n + 1, np.int64), offsets_l=np.zeros(n + 1, np.int64))
    z = [np.zeros((0, 2), np.float32)] * n
    with pytest.raises(N.LtrError, match="LTR_BA_MAX_IMAGES"):
        BA.bundle_adjust(z, z, np.eye(3), np.tile(np.eye(3), (n, 1, 1)), np.zeros((n, 3)), big)


# ------------------------------------------------------------------ on the GPU
def _gpu_case(d, pairs, R, t, **kw):
    dev = torch.device("cuda", 0)
    res = ring_matches(d, pairs, dev)
    trk = TR.triangulate_tracks(d["keypoints"], d["klines"], pairs, res, d["K"], R, t, thresh=8, epi_thresh=8)
    return trk


def _assert_same(out, host):
    for k in ("R", "t", "status_p", "status_l", "residual_p", "residual_l", "row_points3d", "row_lines3d",
              "n_views_p", "n_views_l"):
        a, b = getattr(out, k).cpu().numpy(), np.asarray(host[k])
        a = a[:len(b)]
        assert a.shape == b.shape, k
        assert np.array_equal(a.view(np.uint8), b.astype(a.dtype).view(np.uint8)), k
    for k in ("points3d", "lines3d"):
        b = host[k]
        a = getattr(out, k).cpu().numpy()[:len(b)]
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), k
    s = out.stats_dict()
    for k in BA.STATS:
        assert s[k] == host["stats"][k] or (np.isnan(s[k]) and np.isnan(host["stats"][k])), k


def _ragged():
    """Images without tracks and a merged track with two inlier rows of one image (the degenerate 2-view line is
    make_degenerate's case)."""
    d = syn.make_line_map_set(7, 10, 60, 12, jitter_px=0.5)
    d["keypoints"][8] = d["keypoints"][8][:0]
    d["klines"][8] = d["klines"][8][:0]
    d["keypoints"][9] = d["keypoints"][9][:0]
    kp1 = d["keypoints"][1].copy()
    kp1[5] = kp1[6]                           # rows 5 and 6 of image 1 merge points 5 and 6
    d["keypoints"][1] = kp1
    pairs = np.array([(i, i + 1) for i in range(7)] + [(i, i + 2) for i in range(6)] + [(0, 9)], dtype=np.int32)
    R, t = perturb(d, 8, skip=(0,))
    return d, pairs, R, t


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["ragged", "degenerate", "points", "lines", "fixed03", "allfixed", "it0", "it1",
                                  "max_images"])
def test_gpu_matches_host_model(case):
    fixed, iters = (0,), 50
    if case == "ragged":
        d, pairs, R, t = _ragged()
    elif case == "max_images":
        V = BA.BA_MAX_IMAGES
        d = syn.make_line_map_set(9, V, 30, 6, jitter_px=0.5)
        pairs = np.array([(i, (i + 1) % V) for i in range(V)], dtype=np.int32)
        R, t = perturb(d, 10)
        iters = 8
    else:
        d, pairs, R, t = scene(11, V=10, n_pts=80, n_lines=16)
        if case == "points":
            d["klines"] = [k[:0] for k in d["klines"]]
        if case == "lines":
            d["keypoints"] = [k[:0] for k in d["keypoints"]]
        fixed = {"fixed03": (0, 3), "allfixed": tuple(range(10))}.get(case, fixed)
        iters = {"it0": 0, "it1": 1}.get(case, iters)
    if case in ("points", "lines"):
        res = ring_matches(dict(d, points3d=d["points3d"][:len(d["keypoints"][0])],
                                segments3d=d["segments3d"][:len(d["klines"][0])]), pairs, torch.device("cuda", 0))
        trk = TR.triangulate_tracks(d["keypoints"], d["klines"], pairs, res, d["K"], R, t, thresh=8, epi_thresh=8)
    elif case == "ragged":
        res = _ragged_matches(d, pairs)
        trk = TR.triangulate_tracks(d["keypoints"], d["klines"], pairs, res, d["K"], R, t, thresh=8, epi_thresh=8)
    else:
        trk = _gpu_case(d, pairs, R, t)
    if case == "degenerate":
        kl, inl, L, k = make_degenerate(d, R, t, trk)
        dev = torch.device("cuda", 0)
        trk = dataclasses.replace(trk, inlier_l=torch.from_numpy(inl).to(dev), lines3d=torch.from_numpy(L).to(dev))
        d = dict(d, klines=kl)
    out = BA.bundle_adjust(d["keypoints"], d["klines"], d["K"], R, t, trk, fixed=fixed, max_iters=iters)
    host = BA.bundle_adjust_host(d["keypoints"], d["klines"], d["K"], R, t, trk, fixed=fixed, max_iters=iters)
    _assert_same(out, host)
    again = BA.bundle_adjust(d["keypoints"], d["klines"], d["K"], R, t, trk, fixed=fixed, max_iters=iters)
    _assert_same(again, host)
    if case == "ragged":
        st = host["status_p"]
        assert (st == BA.BA_SAME_IMAGE).any() and (st == BA.BA_IN).any()
    if case == "degenerate":
        assert out.status_l[k].item() == BA.BA_DEGENERATE and host["stats"]["accepted"] >= 1
        assert torch.equal(out.lines3d[k], trk.lines3d[k])
    if case == "it0":
        ref = trk.rows()
        assert torch.equal(out.rows().points3d.nan_to_num(7.0), ref.points3d.nan_to_num(7.0))
        assert torch.equal(out.rows().lines3d.nan_to_num(7.0), ref.lines3d.nan_to_num(7.0))


def _ragged_matches(d, pairs, dev=torch.device("cuda", 0)):
    kp, kl = d["keypoints"], d["klines"]
    mp, ml, cp, cl = [], [], [0], [0]
    for i, j in pairs:
        a, b = len(kp[i]), len(kp[j])
        m = np.where(np.arange(a) < b, np.arange(a), -1)
        if i == 1:
            m[5] = 6                                 # rows 5 and 6 of image 1 (both point 6) join one track
        mp.append(m)
        la, lb = len(kl[i]), len(kl[j])
        ml.append(np.where(np.arange(la) < lb, np.arange(la), -1))
        cp.append(cp[-1] + a)
        cl.append(cl[-1] + la)
    mp = torch.from_numpy(np.concatenate(mp).astype(np.int32)).to(dev)
    ml = torch.from_numpy(np.concatenate(ml).astype(np.int32)).to(dev)
    zp, zl = torch.zeros(len(pairs), dtype=torch.int32, device=dev), torch.zeros(len(pairs), dtype=torch.int32,
                                                                               device=dev)
    return ImagePairMatches(ml, ml.float(), zl, np.array(cl, np.int32), mp, mp.float(), zp, np.array(cp, np.int32),
                            [kl[i] for i, _ in pairs], [kl[j] for _, j in pairs], [kp[i] for i, _ in pairs],
                            [kp[j] for _, j in pairs])


@pytest.mark.gpu
def test_gpu_end_to_end_localization():
    from linetr_b200.localization import absolute_pose_errors, estimate_absolute_poses
    V, Q = 14, 4
    d = syn.make_line_map_set(12, V + Q, 300, 40, jitter_px=0.5)
    db = list(range(V))
    dd = dict(d, keypoints=d["keypoints"][:V], klines=d["klines"][:V], R=d["R"][:V], t=d["t"][:V])
    pairs = np.array([(i, (i + k) % V) for i in range(V) for k in range(1, 4)], dtype=np.int32)
    R, t = perturb(dd, 13, deg=0.5, shift=0.05, skip=(0, 1))
    dev = torch.device("cuda", 0)
    res = ring_matches(dd, pairs, dev)
    trk = TR.triangulate_tracks(dd["keypoints"], dd["klines"], pairs, res, dd["K"], R, t, thresh=8, epi_thresh=8)
    ba = BA.bundle_adjust(dd["keypoints"], dd["klines"], dd["K"], R, t, trk, fixed=(0, 1))
    errs = {}
    for name, rows in (("tracks", trk.rows()), ("ba", ba.rows())):
        pts, lns = rows.per_image()
        qpairs = [(V + q, j) for q in range(Q) for j in db[:4]]
        qres = ring_matches(dict(d, keypoints=d["keypoints"], klines=d["klines"]), np.array(qpairs, np.int32), dev)
        out = estimate_absolute_poses(qres, d["K"], [pts[j] for _, j in qpairs], [lns[j] for _, j in qpairs],
                                      groups=np.arange(Q + 1) * 4)
        Rq, tq = out.R.cpu().numpy(), out.t.cpu().numpy()
        errs[name] = absolute_pose_errors(Rq, tq, d["R"][V:], d["t"][V:])
    assert np.median(errs["ba"][0]) < np.median(errs["tracks"][0])
