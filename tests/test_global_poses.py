"""Global poses (`global_poses`): the numpy model's geometry, graph and robustness on the host, and the GPU's bits
against the model."""
import numpy as np
import pytest
import torch
from scipy.sparse import csr_matrix
from scipy.optimize import least_squares
from scipy.sparse.csgraph import connected_components, minimum_spanning_tree

from linetr_b200 import _native as N
from linetr_b200 import synthetic as syn
from linetr_b200.engine import ImagePairMatches
from linetr_b200.global_poses import (GP_EDGE_DIR_OUTLIER, GP_EDGE_INLIER, GP_EDGE_OUTSIDE, GP_EDGE_ROT_OUTLIER,
                                      GP_EDGE_UNUSED, GP_SIGMA_POS, GP_SIGMA_ROT, STATS, _loop, _rel, _spanning_tree,
                                      _tree_keys, global_poses, global_poses_host, registered_set)


def ring(n, k):
    return np.array([(i, (i + d) % n) for i in range(n) for d in range(1, k + 1) if (i + d) % n != i and
                     (k < n / 2 or i < (i + d) % n)], np.int64)


def exhaustive(n):
    return np.array([(i, j) for i in range(n) for j in range(i + 1, n)], np.int64).reshape(-1, 2)


def truth(seed, n, max_angle=20.0):
    d = syn.make_line_map_set(seed, n, 8, 2, max_angle_deg=max_angle)
    return d["R"], d["t"], -np.einsum("nji,nj->ni", d["R"], d["t"])


def align(R, C, Rt, Ct, mask=None):
    """Errors after the 7-DoF similarity that best maps the truth onto the estimate: (max rotation error as |dR|_F,
    max centre error relative to the mean baseline)."""
    mask = np.ones(len(R), bool) if mask is None else mask
    R, C, Rt, Ct = R[mask], C[mask], Rt[mask], Ct[mask]
    U, _, Vt = np.linalg.svd(sum(Rt[k].T @ R[k] for k in range(len(R))))
    G = U @ Vt                                  # R_k ~ Rt_k G
    rerr = max(np.linalg.norm(Rt[k] @ G - R[k]) for k in range(len(R)))
    A = Ct @ G
    am, cm = A.mean(0), C.mean(0)
    s = ((A - am) * (C - cm)).sum() / ((A - am) ** 2).sum()
    base = np.mean([np.linalg.norm(C[i] - C[j]) for i in range(len(C)) for j in range(i)])
    return rerr, np.linalg.norm(s * (A - am) + cm - C, axis=1).max() / base


def centres(o):
    return -np.einsum("nji,nj->ni", o["R"], o["t"])


# ------------------------------------------------------------------ host: geometry
@pytest.mark.parametrize("graph", ["ring4", "ring5", "exhaustive"])
def test_noise_free_recovers_the_truth(graph):
    n = 16
    Rt, tt, Ct = truth(1, n)
    pairs = {"ring4": ring(n, 4), "ring5": ring(n, 5), "exhaustive": exhaustive(n)}[graph]
    rp = syn.make_relative_poses(Rt, tt, pairs, seed=2)
    o = global_poses_host(pairs, rp, n, pos_iters=5000)
    assert o["registered"].all()
    assert (o["edge_status"] == GP_EDGE_INLIER).all()
    rerr, cerr = align(o["R"], centres(o), Rt, Ct)
    assert rerr < 1e-9
    # BATA converges linearly, and its cost stops falling in its last bits 0.9 - 1.5e-8 of the baseline from the truth
    assert cerr < 2e-8


def test_gauge_and_explicit_anchor():
    n = 8
    Rt, tt, _ = truth(3, n)
    pairs = ring(n, 3)
    rp = syn.make_relative_poses(Rt, tt, pairs, noise_deg=0.3, seed=4)
    for anchor, want in ((None, 0), (5, 5)):
        o = global_poses_host(pairs, rp, n, anchor=anchor)
        assert o["stats"]["anchor"] == want
        assert np.array_equal(o["R"][want], np.eye(3)) and np.array_equal(o["t"][want], np.zeros(3))
        assert not np.signbit(o["t"][want]).any()


# ------------------------------------------------------------------ host: graph
def test_components_and_unused_edges():
    n = 9
    Rt, tt, _ = truth(5, n)
    # two triangles-with-chords {0..3} and {4..8}, plus an invalid and a weak edge joining them
    pairs = np.array([(0, 1), (1, 2), (2, 3), (0, 2), (1, 3), (4, 5), (5, 6), (6, 7), (7, 8), (4, 6), (5, 7), (6, 8),
                      (3, 4), (2, 5)])
    rp = syn.make_relative_poses(Rt, tt, pairs, seed=6)
    rp["valid"][12] = False
    rp["n_cheirality"][13] = 5
    o = global_poses_host(pairs, rp, n)
    assert o["edge_status"][12] == GP_EDGE_UNUSED and o["edge_status"][13] == GP_EDGE_UNUSED
    usable = np.ones(len(pairs), bool)
    usable[12:] = False
    g = csr_matrix((np.ones(usable.sum()), (pairs[usable, 0], pairs[usable, 1])), shape=(n, n))
    _, lab = connected_components(g, directed=False)
    big = np.bincount(lab).argmax()
    assert np.array_equal(o["registered"], lab == big)
    assert (o["edge_status"][:5] == GP_EDGE_OUTSIDE).all()
    assert o["stats"]["anchor"] == 4
    # a tie: the component of the lowest image wins
    pt = pairs[[0, 1, 3, 5, 6, 9]]
    o = global_poses_host(pt, {k: v[[0, 1, 3, 5, 6, 9]] for k, v in rp.items()}, n)
    assert np.array_equal(np.flatnonzero(o["registered"]), [0, 1, 2])


def test_loop_support_counts_every_triangle():
    n = 9
    Rt, tt, _ = truth(7, n)
    pairs = exhaustive(n)
    rng = np.random.default_rng(0)
    pairs = pairs[rng.random(len(pairs)) < 0.7]
    rp = syn.make_relative_poses(Rt, tt, pairs, noise_deg=1.0, outlier_frac=0.2, seed=8)
    o = global_poses_host(pairs, rp, n)
    tan = np.tan(np.radians(5.0) / 2)
    E = {}
    for p, (i, j) in enumerate(pairs):
        E[(i, j)] = E[(j, i)] = p
    want = []
    for p, (i, j) in enumerate(pairs):
        c = 0
        for k in range(n):
            if k in (i, j) or (i, k) not in E or (k, j) not in E:
                continue
            Rik = _rel(rp["R"].reshape(-1, 9), pairs, np.array(E[(i, k)]), i)
            Rkj = _rel(rp["R"].reshape(-1, 9), pairs, np.array(E[(k, j)]), k)
            Q = rp["R"][p].T @ Rkj.reshape(3, 3) @ Rik.reshape(3, 3)
            ang = np.arccos(np.clip((np.trace(Q) - 1) / 2, -1, 1))
            c += abs(np.tan(ang / 2) - tan) > 1e-12 and np.tan(ang / 2) < tan
        want.append(c)
    assert np.array_equal(o["support"], want)


def test_spanning_tree_is_scipys():
    rng = np.random.default_rng(3)
    for n in (6, 17, 40):
        pairs = exhaustive(n)
        pairs = pairs[rng.random(len(pairs)) < 0.35]
        pairs = np.concatenate([np.stack([np.arange(n - 1), np.arange(1, n)], 1), pairs])   # connected
        pairs = np.unique(pairs, axis=0)
        P = len(pairs)
        E = np.full((n, n), -1, np.int64)
        E[pairs[:, 0], pairs[:, 1]] = E[pairs[:, 1], pairs[:, 0]] = np.arange(P)
        key = _tree_keys(rng.integers(0, 30, P), rng.integers(20, 200, P))
        anchor = int(rng.integers(n))
        tree = _spanning_tree(E, key, anchor, n)
        assert sorted(u for u, _ in tree) == sorted(set(range(n)) - {anchor})
        # scipy's minimum spanning tree of the key ranks, largest key cheapest (keys are distinct: the tree is unique)
        rank = np.empty(P)
        rank[np.argsort(-key)] = np.arange(1, P + 1)
        mst = minimum_spanning_tree(csr_matrix((rank, (pairs[:, 0], pairs[:, 1])), shape=(n, n))).tocoo()
        want = {int(E[i, j]) for i, j in zip(mst.row, mst.col)}
        assert {e for _, e in tree} == want


# ------------------------------------------------------------------ host: robustness
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_planted_outliers_are_flagged(seed):
    n = 24
    Rt, tt, Ct = truth(10 + seed, n)
    pairs = ring(n, 5)
    rp = syn.make_relative_poses(Rt, tt, pairs, noise_deg=0.5, outlier_frac=0.2, seed=seed)
    o = global_poses_host(pairs, rp, n)
    out = rp["outlier"]
    assert (o["edge_status"][out] == GP_EDGE_ROT_OUTLIER).all()
    assert (o["edge_status"][~out] == GP_EDGE_INLIER).all()
    clean = {k: v[~out] for k, v in rp.items()}
    oc = global_poses_host(pairs[~out], clean, n)
    ang = max(np.degrees(np.linalg.norm(o["R"][k] - oc["R"][k]) / np.sqrt(2)) for k in range(n))
    assert ang < 0.05
    Cc = centres(oc)
    base = np.mean([np.linalg.norm(Cc[i] - Cc[j]) for i in range(n) for j in range(i)])
    assert np.abs(centres(o) - Cc).max() / base < 0.01


def _cay(w):
    w = np.asarray(w, float)
    ww = w @ w
    S = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    return ((1 - ww) * np.eye(3) + 2 * S + 2 * np.outer(w, w)) / (1 + ww)


def _cayinv_norm(Q):
    v = np.array([Q[2, 1] - Q[1, 2], Q[0, 2] - Q[2, 0], Q[1, 0] - Q[0, 1]])
    den = 1 + np.trace(Q)
    return np.linalg.norm(v / den) if den > 0 else np.inf


def test_model_is_a_local_optimum_of_its_costs():
    """scipy's least_squares, started from the model's result, finds no lower robust rotation cost and no lower BATA
    position cost (the constraint eliminated through one coordinate, the scales at their optimum)."""
    n = 24
    Rt, tt, _ = truth(11, n)
    pairs = ring(n, 5)
    rp = syn.make_relative_poses(Rt, tt, pairs, noise_deg=0.5, outlier_frac=0.2, seed=1)
    o = global_poses_host(pairs, rp, n)
    anchor = o["stats"]["anchor"]
    free = [k for k in range(n) if k != anchor]
    Rm = o["R"]
    s2 = GP_SIGMA_ROT ** 2

    def rot_res(w):
        R = Rm.copy()
        for q, k in enumerate(free):
            R[k] = Rm[k] @ _cay(w[3 * q:3 * q + 3])
        r = np.array([_cayinv_norm(R[j].T @ rp["R"][p] @ R[i]) for p, (i, j) in enumerate(pairs)])
        return np.where(np.isinf(r), 1.0, r / np.sqrt(s2 + r * r))

    c0 = np.sum(rot_res(np.zeros(3 * len(free))) ** 2)
    assert np.isclose(c0, o["stats"]["rot_cost"], rtol=1e-12)
    ls = least_squares(rot_res, np.zeros(3 * len(free)), xtol=1e-15, ftol=1e-15, gtol=1e-15)
    assert 2 * ls.cost >= c0 * (1 - 1e-9)

    # positions: the edges of the solve, v_p = -R_j^T t_p, C_anchor = 0 and sum <dC_p, v_p> = E
    pe = np.isin(o["edge_status"], [GP_EDGE_INLIER, GP_EDGE_DIR_OUTLIER])
    ep = pairs[pe]
    v = np.stack([-Rm[j].T @ rp["t"][p] for p, (i, j) in zip(np.flatnonzero(pe), ep)])
    Cm = centres(o)
    a = np.zeros((n, 3))
    np.add.at(a, ep[:, 1], v)
    np.subtract.at(a, ep[:, 0], v)
    a[anchor] = 0
    assert np.isclose((a * Cm).sum(), len(ep), rtol=1e-10)
    k, c = np.unravel_index(np.argmax(np.abs(a)), a.shape)
    mask = np.ones((n, 3), bool)
    mask[anchor] = False
    mask[k, c] = False
    s2p = GP_SIGMA_POS ** 2

    def pos_res(x):
        C = np.zeros((n, 3))
        C[mask] = x
        C[k, c] = (len(ep) - (a * C).sum()) / a[k, c]
        dC = C[ep[:, 1]] - C[ep[:, 0]]
        dv, dd = (dC * v).sum(1), (dC * dC).sum(1)
        s = np.where(dd > 0, np.maximum(dv, 0) / np.where(dd > 0, dd, 1), 0)
        e = np.linalg.norm(s[:, None] * dC - v, axis=1)
        return e / np.sqrt(s2p + e * e)

    c0 = np.sum(pos_res(Cm[mask]) ** 2)
    assert np.isclose(c0, o["stats"]["pos_cost"], rtol=1e-9)
    ls = least_squares(pos_res, Cm[mask], xtol=1e-15, ftol=1e-15, gtol=1e-15)
    assert 2 * ls.cost >= c0 * (1 - 1e-9)


def _cpu_matches(d, pairs):
    n, m = len(d["keypoints"][0]), len(d["klines"][0])
    P = len(pairs)
    mp = torch.arange(n, dtype=torch.int32).repeat(P)
    ml = torch.arange(m, dtype=torch.int32).repeat(P)
    kp, kl = d["keypoints"], d["klines"]
    return ImagePairMatches(ml, ml.float() + 0.5, torch.arange(P, dtype=torch.int32), np.arange(P + 1, dtype=np.int32) * m,
                            mp, mp.float() + 0.25, torch.arange(P, dtype=torch.int32) + 100,
                            np.arange(P + 1, dtype=np.int32) * n, [kl[i] for i, _ in pairs],
                            [kl[j] for _, j in pairs], [kp[i] for i, _ in pairs], [kp[j] for _, j in pairs])


def test_registered_set_selects_and_renumbers():
    n = 8
    d = syn.make_line_map_set(6, n, 12, 3)
    pairs = np.concatenate([ring(6, 2), [(2, 6), (6, 7), (7, 3)]])      # 6 - 7 hang off the ring once (7, 3) is invalid
    rp = syn.make_relative_poses(d["R"], d["t"], pairs, seed=3)
    rp["valid"][-1] = False
    o = global_poses_host(pairs, rp, n)
    assert np.array_equal(np.flatnonzero(o["registered"]), np.arange(6))
    res = _cpu_matches(d, pairs)
    s = registered_set(d["keypoints"], d["klines"], pairs, res, o)
    keep = np.flatnonzero((pairs < 6).all(1))
    assert np.array_equal(s["images"], np.arange(6))
    assert np.array_equal(s["pairs"], pairs[keep])
    assert len(s["keypoints"]) == 6 and all(s["keypoints"][i] is d["keypoints"][i] for i in range(6))
    r = s["res"]
    assert r.n_pairs == len(keep)
    for q, p in enumerate(keep):
        assert torch.equal(r.pair_points(q), res.pair_points(p)) and torch.equal(r.pair_lines(q), res.pair_lines(p))
        sl = slice(int(r.offsets_p[q]), int(r.offsets_p[q + 1]))
        assert torch.equal(r.scores_p[sl], res.scores_p[int(res.offsets_p[p]):int(res.offsets_p[p + 1])])
        assert r.keypoints1[q] is res.keypoints1[p] and r.klines0[q] is res.klines0[p]
    assert torch.equal(r.counts_p, res.counts_p[keep]) and torch.equal(r.counts_l, res.counts_l[keep])
    assert np.array_equal(s["R"].numpy(), o["R"][:6]) and np.array_equal(s["t"].numpy(), o["t"][:6])
    # renumbering: registered images need not be a prefix
    o2 = dict(o, registered=np.isin(np.arange(n), [1, 2, 3, 4]))
    s2 = registered_set(d["keypoints"], d["klines"], pairs, res, o2)
    keep2 = np.flatnonzero(np.isin(pairs, [1, 2, 3, 4]).all(1))
    assert np.array_equal(s2["pairs"], pairs[keep2] - 1)


# ------------------------------------------------------------------ host: rigidity
def test_rigidity_drops_leaves_and_parallel_images():
    n = 7
    Rt, tt, _ = truth(20, n)
    pairs = np.concatenate([exhaustive(5), [(4, 5)]])       # image 5 is a leaf, image 6 has no edge
    rp = syn.make_relative_poses(Rt, tt, pairs, seed=1)
    o = global_poses_host(pairs, rp, n)
    assert np.array_equal(np.flatnonzero(o["registered"]), [0, 1, 2, 3, 4])
    assert o["edge_status"][-1] == GP_EDGE_OUTSIDE
    # image 3 on the line through the centres of images 1 and 2, linked to those two only
    C = -np.einsum("nji,nj->ni", Rt, tt)
    C[3] = C[1] + 2.0 * (C[2] - C[1])
    t2 = tt.copy()
    t2[3] = -Rt[3] @ C[3]
    pairs = np.array([(0, 1), (1, 2), (0, 2), (0, 4), (1, 4), (2, 4), (1, 3), (2, 3)])
    rp = syn.make_relative_poses(Rt, t2, pairs, seed=1)
    o = global_poses_host(pairs, rp, 5)
    assert np.array_equal(np.flatnonzero(o["registered"]), [0, 1, 2, 4])
    # two images
    rp = syn.make_relative_poses(Rt, tt, np.array([(0, 1)]), seed=1)
    o = global_poses_host(np.array([(0, 1)]), rp, 2)
    assert o["registered"].all() and o["edge_status"][0] == GP_EDGE_INLIER


# ------------------------------------------------------------------ host: refusals
def test_refusals():
    n = 4
    Rt, tt, _ = truth(30, n)
    pairs = ring(n, 1)
    rp = syn.make_relative_poses(Rt, tt, pairs, seed=1)
    bad = [
        dict(n_images=129),
        dict(poses={**rp, "t": rp["t"][:-1]}),
        dict(pairs=np.concatenate([pairs, [[1, 0]]]), poses={k: np.concatenate([v, v[:1]]) for k, v in rp.items()}),
        dict(pairs=np.concatenate([pairs, [[2, 2]]]), poses={k: np.concatenate([v, v[:1]]) for k, v in rp.items()}),
        dict(rot_thresh=float("nan")), dict(dir_thresh=float("inf")), dict(ftol=float("nan")),
        dict(anchor=4), dict(anchor=-1), dict(rot_iters=-1), dict(pos_iters=-1),
    ]
    for kw in bad:
        args = dict(pairs=pairs, poses=rp, n_images=n)
        args.update(kw)
        with pytest.raises(N.LtrError):
            global_poses_host(**args)
    # an anchor outside the registered component
    rp2 = dict(rp, valid=np.array([True, True, False, False]))
    with pytest.raises(N.LtrError, match="component"):
        global_poses_host(pairs, rp2, n, anchor=3)


# ------------------------------------------------------------------ GPU: bits
def _cases():
    out = []
    n = 12
    Rt, tt, _ = truth(40, n)
    # a leaf (11) inside the registered ring, a second component {9, 10} joined to it by a weak pair (8, 9)
    p = np.concatenate([ring(9, 3), [(9, 10), (3, 11), (8, 9)]])
    rp = syn.make_relative_poses(Rt, tt, p, noise_deg=0.5, outlier_frac=0.15, seed=1)
    rp["valid"][3] = False
    rp["n_cheirality"][-1] = 3
    out.append(("ragged", p, rp, n, {}))
    out.append(("one", np.zeros((0, 2), np.int64), {k: v[:0] for k, v in rp.items()}, 1, {}))
    rp2 = syn.make_relative_poses(Rt, tt, np.array([(1, 0)]), noise_deg=0.5, seed=2)
    out.append(("two", np.array([(1, 0)]), rp2, 2, {}))
    R1, t1, _ = truth(41, 128, 30.0)
    pe = exhaustive(128)
    out.append(("128", pe, syn.make_relative_poses(R1, t1, pe, noise_deg=0.5, outlier_frac=0.2, seed=3), 128,
                dict(pos_iters=60)))
    pr = ring(40, 5)
    R2, t2, _ = truth(42, 40)
    rp3 = syn.make_relative_poses(R2, t2, pr, noise_deg=0.5, outlier_frac=0.2, seed=4)
    for it in (0, 1):
        out.append((f"iters{it}", pr, rp3, 40, dict(rot_iters=it, pos_iters=it)))
    out.append(("full", pr, rp3, 40, dict(anchor=7)))
    return out


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("case", _cases(), ids=lambda c: c[0])
def test_gpu_matches_the_model(case):
    name, pairs, rp, n, kw = case
    dev = torch.device("cuda", 0)
    want = global_poses_host(pairs, rp, n, **kw)
    if name == "ragged":     # the leaf is pruned from the registered component
        assert want["registered"][:9].all() and not want["registered"][9:].any()
        assert want["edge_status"][-2] == GP_EDGE_OUTSIDE
    dp = {k: torch.as_tensor(v).to(dev) for k, v in rp.items() if k != "outlier"}
    got = global_poses(pairs, dp, n, **kw)
    again = global_poses(pairs, dp, n, **kw)
    torch.cuda.synchronize()
    for k in ("R", "t", "edge_status", "support", "rot_residual", "dir_cos"):
        g = getattr(got, k).cpu().numpy()
        w = want[k].astype(g.dtype)
        assert _same(g, w), (k, np.flatnonzero(g.reshape(-1).view(np.uint8) != w.reshape(-1).view(np.uint8))[:8])
        assert _same(g, getattr(again, k).cpu().numpy()), k
    assert np.array_equal(got.registered.cpu().numpy(), want["registered"])
    s = got.stats_dict()
    for k in STATS:
        assert s[k] == want["stats"][k] or (np.isinf(s[k]) and np.isinf(want["stats"][k])), (k, s[k], want["stats"][k])


def _similarity(R, t, Rt, tt):
    """The similarity (G, s, b) with R ~ Rt G and C ~ s Ct G + b over the images, fitted to the truth."""
    U, _, Vt = np.linalg.svd(sum(Rt[k].T @ R[k] for k in range(len(R))))
    G = U @ Vt
    C, Ct = -np.einsum("nji,nj->ni", R, t), -np.einsum("nji,nj->ni", Rt, tt)
    A = Ct @ G
    am, cm = A.mean(0), C.mean(0)
    s = ((A - am) * (C - cm)).sum() / ((A - am) ** 2).sum()
    return G, s, cm - s * am


def _errors(R, t, Rt, tt, sim):
    """Median rotation error (degrees) and median centre error (truth units) of poses mapped by sim to the truth."""
    G, s, b = sim
    Rm = R @ G.T
    Cm = ((-np.einsum("nji,nj->ni", R, t) - b) / s) @ G.T
    ang = [np.degrees(np.arccos(np.clip((np.trace(Rt[k].T @ Rm[k]) - 1) / 2, -1, 1))) for k in range(len(R))]
    Ct = -np.einsum("nji,nj->ni", Rt, tt)
    return float(np.median(ang)), float(np.median(np.linalg.norm(Cm - Ct, axis=1)))


@pytest.mark.gpu
def test_gpu_end_to_end_from_an_unposed_set():
    """estimate_poses -> global_poses -> registered_set -> triangulate_tracks -> bundle_adjust(fixed=(anchor,)) on an
    unposed set, then held-out queries localized against the adjusted map."""
    from linetr_b200 import bundle as BA
    from linetr_b200 import tracks as TR
    from linetr_b200.geometry import estimate_poses
    from linetr_b200.localization import estimate_absolute_poses
    from tests.test_bundle import ring_matches
    V, Q = 14, 4
    d = syn.make_line_map_set(12, V + Q, 300, 40, jitter_px=0.5, max_angle_deg=20)
    dd = dict(d, keypoints=d["keypoints"][:V], klines=d["klines"][:V])
    pairs = np.array([(i, (i + k) % V) for i in range(V) for k in range(1, 4)], dtype=np.int32)
    dev = torch.device("cuda", 0)
    res = ring_matches(dd, pairs, dev)
    poses = estimate_poses(res, d["K"], d["K"])
    gp = global_poses(pairs, poses, V)
    st = gp.stats_dict()
    s = registered_set(dd["keypoints"], dd["klines"], pairs, res, gp)
    img = s["images"]
    assert len(img) == V, st
    trk = TR.triangulate_tracks(s["keypoints"], s["klines"], s["pairs"], s["res"], d["K"], s["R"], s["t"], thresh=8,
                                epi_thresh=8)
    fixed = int(np.flatnonzero(img == st["anchor"])[0])
    ba = BA.bundle_adjust(s["keypoints"], s["klines"], d["K"], s["R"], s["t"], trk, fixed=(fixed,))
    Rt, tt = d["R"][img], d["t"][img]
    Rg, tg = s["R"].cpu().numpy(), s["t"].cpu().numpy()
    Rb, tb = ba.R.cpu().numpy(), ba.t.cpu().numpy()
    e_gp = _errors(Rg, tg, Rt, tt, _similarity(Rg, tg, Rt, tt))
    sim = _similarity(Rb, tb, Rt, tt)
    e_ba = _errors(Rb, tb, Rt, tt, sim)
    assert e_ba[0] < e_gp[0] and e_ba[1] < e_gp[1], (e_gp, e_ba, st, ba.stats_dict())
    # held-out queries against the adjusted map, mapped to the truth by the same similarity
    pts, lns = ba.rows().per_image()
    qpairs = [(V + q, j) for q in range(Q) for j in range(4)]
    qres = ring_matches(d, np.array(qpairs, np.int32), dev)
    out = estimate_absolute_poses(qres, d["K"], [pts[j] for _, j in qpairs], [lns[j] for _, j in qpairs],
                                  groups=np.arange(Q + 1) * 4)
    e_q = _errors(out.R.cpu().numpy(), out.t.cpu().numpy(), d["R"][V:], d["t"][V:], sim)
    assert e_q[0] < 0.5 and e_q[1] < 0.05, (e_q, e_gp, e_ba)
