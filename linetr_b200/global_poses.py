"""Global poses of an unposed image set from the relative poses of its pairs: rotation averaging and camera positions,
on the GPU.

    global_poses(pairs, poses, n_images, ...) -> GlobalPoseResult
        one `ltr_global_poses` call; device outputs, no synchronisation (an explicit `anchor` reads the edge flags
        back once, to check it lies in the registered component)
    global_poses_host(...) -> dict
        the same model in numpy: every operation is the kernels' operation in the kernels' order, so the outputs are
        the same bits
    registered_set(keypoints, klines, pairs, res, gp) -> dict
        the registered images as `triangulate_tracks`' arguments (waits for the call)

The model (DESIGN.md "Global poses", include/linetr_b200.h `ltr_global_poses`), with cayinv(Q) = vee(Q - Q^T) /
(1 + tr Q) the inverse of `_posed.cayley` (|cayinv| = tan(theta / 2), +inf where 1 + tr Q <= 0):
  1. view graph: edge p is usable iff poses.valid[p] and n_cheirality[p] >= min_inliers; the component of usable
     edges with the most images (ties: the one holding the lowest image) is registered; the anchor defaults to its
     lowest image;
  2. loop support of a usable edge (i, j): the third images k whose triangle R_ij^T R_kj R_ik through usable edges
     closes within rot_thresh;
  3. rotations (world -> camera R_k, R_k <- R_k cay(w_k)): Prim's maximum spanning tree from the anchor on the key
     (support, n_cheirality, -p), rotations chained along it; then IRLS on r_p = cayinv(R_j^T R_p R_i) - (w_j - w_i):
     GP_L1_ITERS L1 iterations, then Geman-McClure ones, until an accepted step decreases the cost by <= ftol
     relatively, a step is rejected or rot_iters; an edge is a rotation outlier iff its final |cayinv| > tan(rot_thresh
     / 2);
  4. rigidity: images with fewer than two rotation-inlier edges to kept images, or whose edge directions are all
     parallel to the first within GP_PARALLEL_SIN, are dropped until none is (the anchor is never dropped, and a set of
     two images keeps both); then only the images connected to the anchor stay;
  5. positions (BATA): min sum w_p |s_p dC_p - v_p|^2 with v_p = -R_j^T t_p, C_anchor = 0, sum <dC_p, v_p> = E;
     alternating C (one factorization, six right-hand sides), s_p = max(<dC_p, v_p>, 0) / |dC_p|^2 and Geman-McClure
     weights; stops as step 3 with pos_iters; an edge is a direction outlier iff not <dC_p, v_p> > cos(dir_thresh)
     |dC_p|; t_k = -R_k C_k.
Every operation is explicitly rounded fp64 and every sum has a fixed order.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

from . import _native as N
from . import _ops
from ._posed import block_sum, cayley, centre, cholesky_solve, cross3, dot3, host

GP_MAX_IMAGES = N.GP_MAX_IMAGES
GP_EDGE_UNUSED, GP_EDGE_OUTSIDE, GP_EDGE_ROT_OUTLIER, GP_EDGE_DIR_OUTLIER, GP_EDGE_INLIER = (
    N.GP_EDGE_UNUSED, N.GP_EDGE_OUTSIDE, N.GP_EDGE_ROT_OUTLIER, N.GP_EDGE_DIR_OUTLIER, N.GP_EDGE_INLIER)
GP_L1_ITERS = 5                        # LTR_GP_L1_ITERS: L1 iterations before the Geman-McClure ones
GP_L1_EPS = 1e-9                       # LTR_GP_L1_EPS: the L1 weight is 1 / max(|r|, eps)
GP_SIGMA_ROT = 0.04366094290851206     # LTR_GP_SIGMA_ROT: tan(2.5 deg), the rotation Geman-McClure scale
GP_SIGMA_POS = 0.1                     # LTR_GP_SIGMA_POS: the direction Geman-McClure scale (a sine)
GP_PARALLEL_SIN = 0.03489949670250097  # sin(LTR_GP_MIN_ANGLE = 2 deg), the rigidity test's parallel bound
GP_MAX_ITERS = 100000                  # LTR_GP_MAX_ITERS
GP_THREADS = 1024                      # the one-CTA stages (block sums: _posed.block_sum)
STATS = ("rot_iterations", "rot_cost", "pos_iterations", "pos_cost", "n_registered", "n_inliers", "anchor")
_WHO = "global_poses"
_T = [0, 3, 6, 1, 4, 7, 2, 5, 8]


# ------------------------------------------------------------------ arguments
def _pose_arrays(poses, P):
    get = (lambda k: poses[k]) if isinstance(poses, dict) else (lambda k: getattr(poses, k))
    return {k: get(k) for k in ("R", "t", "valid", "n_cheirality")}


def _check(pairs, poses, n_images, min_inliers, rot_thresh, dir_thresh, rot_iters, pos_iters, ftol, anchor):
    """The host checks of `global_poses` (before any device work) -> (n, pairs int64 [P, 2], pose arrays, anchor or
    None).  An explicit anchor is checked against the registered component (the edge flags are read to the host)."""
    n = int(n_images)
    if n < 1:
        raise N.LtrError(f"{_WHO}: n_images must be >= 1")
    if n > GP_MAX_IMAGES:
        raise N.LtrError(f"{_WHO}: {n} images exceed LTR_GP_MAX_IMAGES = {GP_MAX_IMAGES}")
    pr = host(pairs, np.int64)
    if pr.size == 0:
        pr = pr.reshape(0, 2)
    if pr.ndim != 2 or pr.shape[1] != 2:
        raise N.LtrError(f"{_WHO}: pairs must be [P, 2], got {list(pr.shape)}")
    P = len(pr)
    ps = _pose_arrays(poses, P)
    for k, shape in (("R", (P, 3, 3)), ("t", (P, 3)), ("valid", (P,)), ("n_cheirality", (P,))):
        if tuple(ps[k].shape) != shape:
            raise N.LtrError(f"{_WHO}: poses.{k} must be {list(shape)} for {P} pairs, got {list(ps[k].shape)}")
    if P and (pr.min() < 0 or pr.max() >= n):
        raise N.LtrError(f"{_WHO}: pair indices must lie in [0, {n})")
    if (pr[:, 0] == pr[:, 1]).any():
        raise N.LtrError(f"{_WHO}: pair {int(np.flatnonzero(pr[:, 0] == pr[:, 1])[0])} is a self pair")
    key = np.sort(pr, 1)
    if len(np.unique(key[:, 0] * n + key[:, 1])) != P:
        raise N.LtrError(f"{_WHO}: an unordered pair is listed twice")
    for nm, v in (("rot_thresh", rot_thresh), ("dir_thresh", dir_thresh), ("ftol", ftol)):
        if not math.isfinite(float(v)):
            raise N.LtrError(f"{_WHO}: {nm} must be finite")
    if not 0.0 < float(rot_thresh) < 180.0:
        raise N.LtrError(f"{_WHO}: rot_thresh must lie in (0, 180) degrees")
    if not 0.0 <= float(dir_thresh) <= 180.0:
        raise N.LtrError(f"{_WHO}: dir_thresh must lie in [0, 180] degrees")
    if float(ftol) < 0:
        raise N.LtrError(f"{_WHO}: ftol must be >= 0")
    for nm, v in (("rot_iters", rot_iters), ("pos_iters", pos_iters)):
        if not 0 <= int(v) <= GP_MAX_ITERS:
            raise N.LtrError(f"{_WHO}: {nm} must lie in [0, LTR_GP_MAX_ITERS = {GP_MAX_ITERS}]")
    if anchor is not None:
        a = int(anchor)
        if not 0 <= a < n:
            raise N.LtrError(f"{_WHO}: anchor must lie in [0, {n})")
        usable = host(ps["valid"], bool) & (host(ps["n_cheirality"], np.int64) >= int(min_inliers))
        if not _component(pr, usable, n)[a]:
            raise N.LtrError(f"{_WHO}: anchor {a} is not in the registered component")
        anchor = a
    return n, pr, ps, anchor


def _thresholds(rot_thresh, dir_thresh):
    """The degree thresholds as the tangent and cosine the kernels compare against (converted once, here)."""
    return math.tan(math.radians(float(rot_thresh)) / 2.0), math.cos(math.radians(float(dir_thresh)))


# ------------------------------------------------------------------ the model in numpy
def _component(pr, usable, n):
    """The registered component: bool [n]."""
    label = np.arange(n)
    e = pr[usable]
    while True:
        nl = label.copy()
        if len(e):
            np.minimum.at(nl, e[:, 0], label[e[:, 1]])
            np.minimum.at(nl, e[:, 1], label[e[:, 0]])
        nl = nl[nl]
        if np.array_equal(nl, label):
            break
        label = nl
    size = np.bincount(label, minlength=n)
    best = int(np.argmax(size))          # first maximum: the lowest label, i.e. the component of the lowest image
    return label == best


def _mm(A, B):
    """A B of rotations [..., 9] row-major, each entry rc_dot3 of a row and a column."""
    return np.stack([(A[..., 3 * r] * B[..., c] + A[..., 3 * r + 1] * B[..., 3 + c]) + A[..., 3 * r + 2] * B[..., 6 + c]
                     for r in range(3) for c in range(3)], -1)


def _loop(A, B, C):
    """cayinv(A^T (B C)) -> (c [..., 3], |c|): c = 0 and |c| = +inf where 1 + tr <= 0."""
    Q = _mm(A[..., _T], _mm(B, C))
    v = [Q[..., 7] - Q[..., 5], Q[..., 2] - Q[..., 6], Q[..., 3] - Q[..., 1]]
    den = ((1.0 + Q[..., 0]) + Q[..., 4]) + Q[..., 8]
    ok = den > 0
    c = [np.where(ok, x / den, 0.0) for x in v]
    return np.stack(c, -1), np.where(ok, np.sqrt(dot3(c, c)), np.inf)


def _rel(Rp, pr, e, a):
    """The rotation of edge e from image a to its other image: R_e, or R_e^T when a is its side 1."""
    return np.where((pr[e, 0] == a)[..., None], Rp[e], Rp[e][..., _T])


def _gm(q, s2):
    """Geman-McClure cost q / (s2 + q) and IRLS weight s2 / (s2 + q)^2 of squared residuals q (+inf: 1 and 0)."""
    inf = np.isinf(q)
    d = s2 + q
    return np.where(inf, 1.0, q / d), np.where(inf, 0.0, s2 / (d * d))


def _assemble(inc, col, m, pr, act, wt, rhs_terms):
    """The anchor-free weighted Laplacian (m x m) and the right-hand sides [m, k]: per image, a diagonal and k sums
    over its incident active edges in ascending pair index, + for side 1, - for side 0; off-diagonals -wt."""
    n, D = inc.shape
    k = rhs_terms.shape[1]
    diag, b = np.zeros(n), np.zeros((n, k))
    ids = np.arange(n)
    for r in range(D):
        e = inc[:, r]
        ok = (e >= 0) & act[np.maximum(e, 0)] & (col >= 0)
        es = np.maximum(e, 0)
        diag = np.where(ok, diag + wt[es], diag)
        side1 = (pr[es, 1] == ids)[:, None]
        b = np.where(ok[:, None], np.where(side1, b + rhs_terms[es], b - rhs_terms[es]), b)
    A = np.zeros((m, m))
    u = np.flatnonzero(col >= 0)
    A[col[u], col[u]] = diag[u]
    e = np.flatnonzero(act)
    ci, cj = col[pr[e, 0]], col[pr[e, 1]]
    both = (ci >= 0) & (cj >= 0)
    A[ci[both], cj[both]] = -wt[e[both]]
    A[cj[both], ci[both]] = -wt[e[both]]
    x = np.zeros((m, k))
    x[col[u]] = b[u]
    return A, x


def _esum(terms, mask):
    return float(block_sum(np.where(mask, terms, 0.0)[:, None], GP_THREADS)[0]) if len(terms) else 0.0


def global_poses_host(pairs, poses, n_images, min_inliers=20, rot_thresh=5.0, dir_thresh=10.0, rot_iters=100,
                      pos_iters=500, ftol=1e-12, anchor=None) -> dict:
    """The global-pose model in numpy (DESIGN.md "Global poses"), same arguments as `global_poses` (poses a
    PoseResult or a dict of R, t, valid, n_cheirality).  -> dict of host arrays: R [n, 3, 3], t [n, 3], registered,
    edge_status, support, rot_residual, dir_cos, stats (dict of STATS) and C [n, 3] (the centres)."""
    n, pr, ps, anchor = _check(pairs, poses, n_images, min_inliers, rot_thresh, dir_thresh, rot_iters, pos_iters,
                               ftol, anchor)
    P = len(pr)
    tan_rot, cos_dir = _thresholds(rot_thresh, dir_thresh)
    Rp = host(ps["R"], np.float64).reshape(P, 9)
    tp = host(ps["t"], np.float64).reshape(P, 3)
    usable = host(ps["valid"], bool) & (host(ps["n_cheirality"], np.int64) >= int(min_inliers))
    ncheir = host(ps["n_cheirality"], np.int64)
    with np.errstate(all="ignore"):
        comp = _component(pr, usable, n)
        if anchor is None:
            anchor = int(np.flatnonzero(comp)[0])
        E = np.full((n, n), -1, np.int64)
        for p in np.flatnonzero(usable):
            E[pr[p, 0], pr[p, 1]] = E[pr[p, 1], pr[p, 0]] = p
        # 2. loop support
        support = np.full(P, -1, np.int64)
        up = np.flatnonzero(usable)
        for s0 in range(0, len(up), 256):
            p = up[s0:s0 + 256]
            i, j = pr[p, 0][:, None], pr[p, 1][:, None]
            k = np.arange(n)[None, :]
            a, b = E[i, k], E[k, j]
            ok = (a >= 0) & (b >= 0) & (k != i) & (k != j)
            a, b = np.maximum(a, 0), np.maximum(b, 0)
            _, res = _loop(np.broadcast_to(Rp[p][:, None], (len(p), n, 9)), _rel(Rp, pr, b, k), _rel(Rp, pr, a, i))
            support[p] = (ok & (res <= tan_rot)).sum(1)
        # 3. rotations: the tree, then IRLS
        ce = usable & comp[pr[:, 0]]
        R = np.tile(np.eye(3).reshape(9), (n, 1))
        for u, e in _spanning_tree(E, _tree_keys(support, ncheir), anchor, int(comp.sum())):
            par = int(pr[e, 0] + pr[e, 1] - u)
            R[u] = _mm(_rel(Rp, pr, np.array(e), par), R[par])
        inc = _incidence(pr, ce, n)
        col = np.full(n, -1, np.int64)
        unk = np.flatnonzero(comp & (np.arange(n) != anchor))
        col[unk] = np.arange(len(unk))
        m = len(unk)
        s2r = GP_SIGMA_ROT * GP_SIGMA_ROT
        ii, jj = pr[:, 0], pr[:, 1]

        def rot_state(R_):
            c, res = _loop(R_[jj], Rp, R_[ii])
            return c, res, _esum(_gm(res * res, s2r)[0], ce)

        c, res, cost = rot_state(R)
        it_r = 0
        while m and it_r < int(rot_iters):
            if it_r < GP_L1_ITERS:
                wt = 1.0 / np.maximum(res, GP_L1_EPS)
            else:
                wt = _gm(res * res, s2r)[1]
            wt = np.where(ce, wt, 0.0)
            # Geman-McClure steps take the gradient's exact J^T r = +-(1 + |r|^2) r (the normal matrix keeps the
            # Laplacian of J's leading term [-I, +I]); L1 steps take the leading term there too
            gw = wt if it_r < GP_L1_ITERS else np.where(np.isinf(res), 0.0, wt * (1.0 + res * res))
            A, x = _assemble(inc, col, m, pr, ce, wt, gw[:, None] * c)
            if not cholesky_solve(A, x):
                break
            Q = cayley([x[:, 0], x[:, 1], x[:, 2]])
            Rc = R.copy()
            Rc[unk] = _mm(R[unk], np.stack([Q[a][b] for a in range(3) for b in range(3)], -1))
            cc, rc, cnew = rot_state(Rc)
            it_r += 1
            if it_r <= GP_L1_ITERS:
                R, c, res, cost = Rc, cc, rc, cnew
                continue
            if not cnew < cost:
                break
            rel = (cost - cnew) / cost
            R, c, res, cost = Rc, cc, rc, cnew
            if rel <= float(ftol):
                break
        # 4. rigidity
        ie = ce & (res <= tan_rot)
        v = np.stack(centre(R[jj], [tp[:, 0], tp[:, 1], tp[:, 2]]), 1)
        sin2 = GP_PARALLEL_SIN * GP_PARALLEL_SIN
        kept = comp.copy()
        while kept.sum() > 2:
            drop = np.zeros(n, bool)
            for a in np.flatnonzero(kept):
                if a == anchor:
                    continue
                es = [e for e in inc[a] if e >= 0 and ie[e] and kept[pr[e, 0] + pr[e, 1] - a]]
                allpar = True
                for e in es[1:]:
                    cr = cross3(list(v[es[0]]), list(v[e]))
                    allpar = allpar and bool(dot3(cr, cr) <= sin2 * (dot3(list(v[es[0]]), list(v[es[0]])) *
                                                                     dot3(list(v[e]), list(v[e]))))
                drop[a] = len(es) < 2 or allpar
            if not drop.any():
                break
            kept &= ~drop
        reg = np.zeros(n, bool)
        reg[anchor] = True
        ke = ie & kept[ii] & kept[jj]
        while True:
            nr = reg.copy()
            nr[ii[ke & reg[jj]]] = True
            nr[jj[ke & reg[ii]]] = True
            if np.array_equal(nr, reg):
                break
            reg = nr
        # 5. positions
        pe = ie & reg[ii] & reg[jj]
        Ecount = int(pe.sum())
        col2 = np.full(n, -1, np.int64)
        unk2 = np.flatnonzero(reg & (np.arange(n) != anchor))
        col2[unk2] = np.arange(len(unk2))
        m2 = len(unk2)
        C = np.zeros((n, 3))
        s, w = np.ones(P), np.ones(P)
        pcost = np.inf if Ecount else 0.0
        s2p = GP_SIGMA_POS * GP_SIGMA_POS
        it_p = 0
        while Ecount and it_p < int(pos_iters):
            q, ws = (w * s) * s, w * s
            A, x = _assemble(inc, col2, m2, pr, pe, q, np.concatenate([ws[:, None] * v, v], 1))
            av = x[:, 3:].copy()
            if not cholesky_solve(A, x):
                break
            xb, xa = x[:, :3], x[:, 3:]
            ab = block_sum(dot3(av.T, xb.T)[:, None], GP_THREADS)[0]
            aa = block_sum(dot3(av.T, xa.T)[:, None], GP_THREADS)[0]
            lam = (ab - float(Ecount)) / aa
            Cc = np.zeros((n, 3))
            Cc[unk2] = xb - lam * xa
            dC = Cc[jj] - Cc[ii]
            dd, dv = dot3(dC.T, dC.T), dot3(dC.T, v.T)
            sc = np.where(dd > 0, np.where(dv > 0, dv, 0.0) / dd, 0.0)
            e = sc[:, None] * dC - v
            rho, wc = _gm(dot3(e.T, e.T), s2p)
            cnew = _esum(rho, pe)
            it_p += 1
            if not cnew < pcost:
                break
            rel = (pcost - cnew) / pcost
            C, s, w, pcost = Cc, sc, wc, cnew
            if rel <= float(ftol):
                break
        # outputs
        dC = C[jj] - C[ii]
        dv, nrm = dot3(dC.T, v.T), np.sqrt(dot3(dC.T, dC.T))
        status = np.full(P, GP_EDGE_UNUSED, np.int32)
        status[usable] = GP_EDGE_OUTSIDE
        status[ce & ~ie] = GP_EDGE_ROT_OUTLIER
        status[pe] = np.where(dv[pe] > cos_dir * nrm[pe], GP_EDGE_INLIER, GP_EDGE_DIR_OUTLIER)
        Ro = np.full((n, 9), np.nan)
        to = np.full((n, 3), np.nan)
        Ro[reg] = R[reg]
        to[reg] = -np.stack([dot3([R[reg, 3 * e_], R[reg, 3 * e_ + 1], R[reg, 3 * e_ + 2]], list(C[reg].T))
                             for e_ in range(3)], 1)
        Ro[anchor] = np.eye(3).reshape(9)
        to[anchor] = 0.0
        dcos = np.where(pe, dv / nrm, np.nan)
    stats = dict(rot_iterations=it_r, rot_cost=float(cost), pos_iterations=it_p, pos_cost=float(pcost),
                 n_registered=int(reg.sum()), n_inliers=int((status == GP_EDGE_INLIER).sum()), anchor=anchor)
    return dict(R=Ro.reshape(n, 3, 3), t=to, registered=reg, edge_status=status, support=support.astype(np.int32),
                rot_residual=np.where(ce, res, np.nan), dir_cos=dcos, stats=stats,
                C=np.where(reg[:, None], C, np.nan))


def _tree_keys(support, ncheir):
    """The spanning tree's edge keys (support, n_cheirality, -p) packed into one int64 each, compared as integers."""
    return (np.maximum(support, 0) << 45) | (np.clip(ncheir, 0, None) << 13) | (8191 - np.arange(len(support)))


def _spanning_tree(E, key, anchor, size):
    """Prim's maximum spanning tree from the anchor over the edge table E [n, n] (pair index or -1): -> the (image,
    edge) of every image added, in the order of addition (size - 1 of them)."""
    n = len(E)
    intree = np.zeros(n, bool)
    intree[anchor] = True
    best, bedge = np.full(n, -1, np.int64), np.full(n, -1, np.int64)
    order, u = [], anchor
    for _ in range(size - 1):
        e = E[u]
        kk = np.where((e >= 0) & ~intree, key[np.maximum(e, 0)], -1)
        upd = kk > best
        best[upd], bedge[upd] = kk[upd], e[upd]
        u = int(np.argmax(np.where(intree, -1, best)))
        intree[u] = True
        order.append((u, int(bedge[u])))
    return order


def _incidence(pr, mask, n):
    """[n, n - 1] the pair indices of every image's masked edges, ascending, -1 padded."""
    inc = np.full((n, max(n - 1, 1)), -1, np.int64)
    cnt = np.zeros(n, np.int64)
    for p in np.flatnonzero(mask):
        for a in pr[p]:
            inc[a, cnt[a]] = p
            cnt[a] += 1
    return inc


# ------------------------------------------------------------------ batched on the GPU
@dataclass
class GlobalPoseResult:
    """Result of `global_poses` (device tensors; nothing has been waited for).

    R [n, 3, 3], t [n, 3] fp64 world -> camera (X_cam = R X + t; NaN for images not registered; the anchor exactly I
    and 0); registered bool [n]; per pair: edge_status int32 (GP_EDGE_*), support int32 (-1 for edges not usable),
    rot_residual fp64 (the final |cayinv(R_j^T R_p R_i)| of the registered component's edges, NaN elsewhere), dir_cos
    fp64 (<dC_p, v_p> / |dC_p| of the edges of the position solve, NaN elsewhere); stats fp64 [7] in the order of
    STATS."""
    R: torch.Tensor
    t: torch.Tensor
    registered: torch.Tensor
    edge_status: torch.Tensor
    support: torch.Tensor
    rot_residual: torch.Tensor
    dir_cos: torch.Tensor
    stats: torch.Tensor

    def stats_dict(self) -> dict:
        """The stats on the host (waits for the call)."""
        s = self.stats.cpu().numpy()
        return {k: (float(v) if k.endswith("cost") else int(v)) for k, v in zip(STATS, s)}


def global_poses(pairs, poses, n_images, min_inliers=20, rot_thresh=5.0, dir_thresh=10.0, rot_iters=100,
                 pos_iters=500, ftol=1e-12, anchor=None) -> GlobalPoseResult:
    """One world -> camera pose per image of an unposed set from the relative poses of its pairs: `pairs` int [P, 2]
    (image i side 0, image j side 1) and `poses` the PoseResult of `estimate_poses` on them (X_j = R_p X_i + t_p),
    in one `ltr_global_poses` call with no synchronisation.  Thresholds in degrees.  Raises LtrError before any device
    work on bad arguments: more than GP_MAX_IMAGES images, pairs and poses of different shapes, self or duplicate
    pairs, non-finite thresholds or ftol, negative iteration counts, an anchor out of range or outside the registered
    component."""
    n, pr, ps, anchor = _check(pairs, poses, n_images, min_inliers, rot_thresh, dir_thresh, rot_iters, pos_iters,
                               ftol, anchor)
    P = len(pr)
    tan_rot, cos_dir = _thresholds(rot_thresh, dir_thresh)
    dev = next((v.device for v in ps.values() if isinstance(v, torch.Tensor) and v.is_cuda), None)
    if dev is None:
        dev = _ops.current_cuda_device()
    arrays = {"pairs": pr.astype(np.int32).reshape(-1, 2) if P else np.zeros((1, 2), np.int32)}
    dv = {}
    for k, dt, npdt, w in (("R", torch.float64, np.float64, 9), ("t", torch.float64, np.float64, 3),
                           ("valid", torch.uint8, np.uint8, 1), ("n_cheirality", torch.int32, np.int32, 1)):
        v = ps[k]
        if isinstance(v, torch.Tensor) and v.is_cuda and P:
            dv[k] = (v.view(torch.uint8) if v.dtype == torch.bool else v).to(dev, dt).contiguous()
        else:
            a = host(v, npdt).reshape(P, w) if P else np.zeros((1, w), npdt)
            arrays[k] = a.astype(npdt)
    dv.update(_ops.stage(arrays, dev))
    f64, i32 = dict(dtype=torch.float64, device=dev), dict(dtype=torch.int32, device=dev)
    pb = max(P, 1)
    ws = N.gp_workspace_bytes(n, P)
    o = dict(R=torch.empty((n, 3, 3), **f64), t=torch.empty((n, 3), **f64),
             registered=torch.empty(n, dtype=torch.bool, device=dev), edge_status=torch.empty(pb, **i32),
             support=torch.empty(pb, **i32), rot_residual=torch.empty(pb, **f64), dir_cos=torch.empty(pb, **f64),
             stats=torch.empty(N.GP_STATS, **f64),
             workspace=torch.empty(-(-ws // 8), **f64))
    _ops.call_struct("ltr_global_poses", {**dv, "n_images": n, "n_pairs": P, "min_inliers": min_inliers,
                                          "anchor": -1 if anchor is None else anchor, "rot_iters": rot_iters,
                                          "pos_iters": pos_iters, "rot_tan": tan_rot, "dir_cos": cos_dir, "ftol": ftol},
                     o, workspace_bytes=ws)
    del o["workspace"]     # the caching allocator reuses it only behind this stream's kernels
    for k in ("edge_status", "support", "rot_residual", "dir_cos"):
        o[k] = o[k][:P]
    return GlobalPoseResult(**o)


def registered_set(keypoints, klines, pairs, res, gp) -> dict:
    """The registered images of a `global_poses` result as `triangulate_tracks`' arguments (waits for `registered`):
    -> dict images (int64 indices, ascending), keypoints, klines (theirs), pairs (the pairs between two registered
    images, renumbered), res (the matches restricted to those pairs) and R, t (theirs).  K is the caller's to index
    with `images`."""
    reg = gp.registered.cpu().numpy() if isinstance(gp, GlobalPoseResult) else np.asarray(gp["registered"])
    img = np.flatnonzero(reg)
    new = np.full(len(reg), -1, np.int64)
    new[img] = np.arange(len(img))
    pr = host(pairs, np.int64).reshape(-1, 2)
    keep = np.flatnonzero(reg[pr[:, 0]] & reg[pr[:, 1]]) if len(pr) else np.zeros(0, np.int64)
    R = gp.R if isinstance(gp, GlobalPoseResult) else torch.as_tensor(gp["R"])
    t = gp.t if isinstance(gp, GlobalPoseResult) else torch.as_tensor(gp["t"])
    it = torch.as_tensor(img, device=R.device)
    return dict(images=img, keypoints=[keypoints[i] for i in img], klines=[klines[i] for i in img],
                pairs=new[pr[keep]].astype(np.int32).reshape(-1, 2), res=_select_pairs(res, keep),
                R=R.index_select(0, it), t=t.index_select(0, it))


def _select_pairs(res, keep):
    """The ImagePairMatches of the pairs `keep` (ascending), selected on the device over the existing offsets."""
    out = {}
    for s in ("l", "p"):
        off = np.asarray(getattr(res, f"offsets_{s}"), np.int64)
        rows = np.concatenate([np.arange(off[p], off[p + 1]) for p in keep]) if len(keep) else np.zeros(0, np.int64)
        m = getattr(res, f"matches_{s}")
        idx = torch.as_tensor(rows, device=m.device)
        out[f"matches_{s}"] = m.index_select(0, idx)
        out[f"scores_{s}"] = getattr(res, f"scores_{s}").index_select(0, idx)
        out[f"counts_{s}"] = getattr(res, f"counts_{s}").index_select(0, torch.as_tensor(keep, device=m.device))
        out[f"offsets_{s}"] = np.concatenate([[0], np.cumsum(np.diff(off)[keep])]).astype(off.dtype)
    return type(res)(out["matches_l"], out["scores_l"], out["counts_l"], out["offsets_l"], out["matches_p"],
                     out["scores_p"], out["counts_p"], out["offsets_p"], [res.klines0[p] for p in keep],
                     [res.klines1[p] for p in keep], [res.keypoints0[p] for p in keep],
                     [res.keypoints1[p] for p in keep])
