"""What the posed-set stages (`triangulation`, `tracks`, `bundle`, and `localization`'s absolute pose) share on the
host: the numpy twins of the device camera primitives in csrc/rn_fp64.cuh, and the checks and staging of a posed
image set.

Each primitive does the device function's operations in its order, so a numpy model built from them gives the kernels'
bits.  Vectors are lists of three component arrays (or scalars) and a rotation R is row-major and flat, [..., 9].  A
new parity-bound stage takes its camera math from here.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

from . import _native as N
from . import _ops
from .geometry import _intrinsics


# ------------------------------------------------------------------ camera primitives (rn_fp64.cuh rc_*)
def dot3(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def mv3(R, v):
    """R v for R [..., 9] row-major."""
    return [(R[..., 3 * e] * v[0] + R[..., 3 * e + 1] * v[1]) + R[..., 3 * e + 2] * v[2] for e in range(3)]


def cross3(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def centre(R, t):
    """The camera centre C = -R^T t of the world -> camera pose X_cam = R X + t."""
    return [-((R[..., j] * t[0] + R[..., 3 + j] * t[1]) + R[..., 6 + j] * t[2]) for j in range(3)]


def ray(R, fx, fy, cx, cy, x, y):
    """The world ray R^T ((x - cx) / fx, (y - cy) / fy, 1) of pixel (x, y): X(s) = C + s r has depth s."""
    nx, ny = (x - cx) / fx, (y - cy) / fy
    return [(R[..., k] * nx + R[..., 3 + k] * ny) + R[..., 6 + k] for k in range(3)]


def line_normal(fx, fy, cx, cy, seg):
    """The segments seg [..., 4] (x0, y0, x1, y1) as unit pixel lines in camera-ray form: the line (a, b, c) scaled
    to a^2 + b^2 = 1, then (a fx, b fy, (a cx + b cy) + c), so n . P / P_z is the signed pixel distance of the
    projection of the camera point P."""
    x0, y0, x1, y1 = seg[..., 0], seg[..., 1], seg[..., 2], seg[..., 3]
    a, b, c = y0 - y1, x1 - x0, x0 * y1 - x1 * y0
    rn = 1.0 / np.sqrt(a * a + b * b)
    la, lb, lc = a * rn, b * rn, c * rn
    return [la * fx, lb * fy, (la * cx + lb * cy) + lc]


def closest_on_line(X, d, w, r):
    """The point X + u d of the world line through X with direction d closest to the ray C + s r, w = X - C."""
    aa, bb, cc, dd, ee = dot3(d, d), dot3(d, r), dot3(r, r), dot3(d, w), dot3(r, w)
    uu = (bb * ee - cc * dd) / (aa * cc - bb * bb)
    return [X[k] + uu * d[k] for k in range(3)]


def cayley(w):
    """The Cayley map ((1 - w.w) I + 2 [w]x + 2 w w^T) / (1 + w.w) of w: rows Q[i][k]; R <- Q R is the update."""
    ww = (w[0] * w[0] + w[1] * w[1]) + w[2] * w[2]
    den, s = 1.0 + ww, 1.0 - ww
    z = np.zeros_like(ww)
    wx = [[z, -w[2], w[1]], [w[2], z, -w[0]], [-w[1], w[0], z]]
    return [[(((s if i == k else z) + 2.0 * (w[i] * w[k])) + 2.0 * wx[i][k]) / den for k in range(3)] for i in range(3)]


def block_sum(terms, nt):
    """A one-CTA reduction of per-row terms [n, m] over nt threads: thread t sums rows t, t + nt, ... in order, each
    warp folds its 32 lanes with the xor butterfly (16, 8, 4, 2, 1), then lane 0 of every warp is added in warp
    order."""
    n, m = terms.shape
    R = -(-n // nt)
    pad = np.zeros((R * nt, m))
    pad[:n] = terms
    pad = pad.reshape(R, nt, m)
    acc = np.zeros((nt, m))
    for r in range(R):
        acc = acc + pad[r]
    acc = acc.reshape(nt // 32, 32, m)
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[:, lanes ^ o]
    out = np.zeros(m)
    for w in range(nt // 32):
        out = out + acc[w, 0]
    return out


def cholesky_solve(A, x) -> bool:
    """The dense solver of rn_fp64.cuh rc_cholesky_solve: a right-looking Cholesky of the m x m matrix A (its lower
    triangle read, L written over it), then the forward and back substitutions of the right-hand sides x [m] or
    [m, k], in place.  -> False (x untouched) at the first pivot that is not > 0."""
    m = len(A)
    if m == 0:
        return True
    for c in range(m):
        if not A[c, c] > 0:
            return False
        A[c, c] = np.sqrt(A[c, c])
        A[c + 1:, c] = A[c + 1:, c] / A[c, c]
        A[c + 1:, c + 1:] = A[c + 1:, c + 1:] - np.outer(A[c + 1:, c], A[c + 1:, c])
    xs = x.reshape(m, -1)
    for c in range(m):
        xs[c] = xs[c] / A[c, c]
        xs[c + 1:] = xs[c + 1:] - A[c + 1:, c, None] * xs[c]
    for c in range(m - 1, -1, -1):
        xs[c] = xs[c] / A[c, c]
        xs[:c] = xs[:c] - A[c, :c, None] * xs[c]
    return True


# ------------------------------------------------------------------ arguments
def host(a, dtype):
    return np.asarray(a.cpu() if isinstance(a, torch.Tensor) else a, dtype=dtype)


def row_counts(items, width, what, who):
    """The row count of every image's array in items, each holding `width` coordinates per row."""
    n = []
    for i, k in enumerate(items):
        shape = tuple(k.shape) if hasattr(k, "shape") else np.shape(k)
        m = shape[0] if len(shape) else 0
        if int(np.prod(shape)) != m * width:
            raise N.LtrError(f"{who}: {what}[{i}] must hold {width} coordinates per row, got shape {list(shape)}")
        n.append(m)
    return np.array(n, dtype=np.int64)


def check_poses(K, R, t, n, who):
    """The intrinsics K [3, 3] or [n, 3, 3] and the poses R [n, 3, 3], t [n, 3] -> (K [n, 3, 3], R, t) fp64."""
    Kn = _intrinsics(K, n, "K")
    Rn, tn = host(R, np.float64), host(t, np.float64)
    if Rn.shape != (n, 3, 3) or tn.shape != (n, 3):
        raise N.LtrError(f"{who}: R must be [{n}, 3, 3] and t [{n}, 3], got {list(Rn.shape)} and {list(tn.shape)}")
    if not (np.isfinite(Rn).all() and np.isfinite(tn).all()):
        raise N.LtrError(f"{who}: R and t must be finite")
    return Kn, np.ascontiguousarray(Rn), np.ascontiguousarray(tn)


@dataclass
class PosedSet:
    pairs: np.ndarray        # int32 [P, 2]
    K: np.ndarray            # [n, 3, 3]
    R: np.ndarray            # [n, 3, 3]
    t: np.ndarray            # [n, 3]
    n_kp: np.ndarray         # int64 [n]
    n_kl: np.ndarray         # int64 [n]
    views: np.ndarray        # int32: image i's observations [view_off[i], view_off[i + 1]), pair << 1 | side
    view_off: np.ndarray     # int32 [n + 1]


def check_set(keypoints, klines, pairs, res, K, R, t, who) -> PosedSet:
    """The argument checks of a posed image set with its pair matches, shared by `triangulate` and
    `tracks.triangulate_tracks` (all on the host, before any device work; messages start with `who`) -> the set's host
    tables."""
    n = len(keypoints)
    if len(klines) != n:
        raise N.LtrError(f"{who}: {n} keypoint arrays but {len(klines)} key-line arrays")
    n_kp, n_kl = row_counts(keypoints, 2, "keypoints", who), row_counts(klines, 4, "klines", who)
    pr = host(pairs, np.int64)
    if pr.size == 0:
        pr = pr.reshape(0, 2)
    if pr.ndim != 2 or pr.shape[1] != 2:
        raise N.LtrError(f"{who}: pairs must be [P, 2], got {list(pr.shape)}")
    P = len(pr)
    if P != res.n_pairs:
        raise N.LtrError(f"{who}: {P} pairs but the matches hold {res.n_pairs}")
    if P and (pr.min() < 0 or pr.max() >= n):
        raise N.LtrError(f"{who}: pair indices must lie in [0, {n})")
    if (pr[:, 0] == pr[:, 1]).any():
        raise N.LtrError(f"{who}: pair {int(np.flatnonzero(pr[:, 0] == pr[:, 1])[0])} is a self pair")
    key = np.sort(pr, 1)
    if len(np.unique(key[:, 0] * max(n, 1) + key[:, 1])) != P:
        raise N.LtrError(f"{who}: an unordered pair is listed twice")
    op, ol = np.asarray(res.offsets_p, dtype=np.int64), np.asarray(res.offsets_l, dtype=np.int64)
    for nm, off, cnt0, side1, cnt1 in (("keypoint", op, n_kp, res.keypoints1, n_kp), ("key-line", ol, n_kl, res.klines1, n_kl)):
        bad = np.flatnonzero(np.diff(off) != cnt0[pr[:, 0]])
        if len(bad):
            raise N.LtrError(f"{who}: pair {int(bad[0])} has {int(np.diff(off)[bad[0]])} {nm} match rows for "
                             f"{int(cnt0[pr[bad[0], 0]])} {nm}s of image {int(pr[bad[0], 0])}")
        for p in range(P):
            if len(side1[p]) != cnt1[pr[p, 1]]:
                raise N.LtrError(f"{who}: side 1 of pair {p} has {len(side1[p])} {nm}s, image {int(pr[p, 1])} "
                                 f"{int(cnt1[pr[p, 1]])}")
    Kn, Rn, tn = check_poses(K, R, t, n, who)
    img = np.concatenate([pr[:, 0], pr[:, 1]])
    code = np.concatenate([2 * np.arange(P), 2 * np.arange(P) + 1])
    order = np.lexsort((code, img))
    cnt = np.bincount(img, minlength=n)
    view_off = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32)
    return PosedSet(pr.astype(np.int32), Kn, Rn, tn, n_kp, n_kl, code[order].astype(np.int32), view_off)


def offsets(counts):
    return np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)


# ------------------------------------------------------------------ row pools
def _host_pool(items, width):
    parts = [host(k, np.float32).reshape(-1, width) for k in items]
    return np.concatenate(parts) if parts else np.zeros((0, width), np.float32)


def pool64(items, width):
    """The images' rows back to back, used as float32, as float64 [*, width] (the host models' pool)."""
    return _host_pool(items, width).astype(np.float64)


def _pool_rows(items, width, dev):
    """The images' rows back to back as float32 [*, width]: one device concatenation when every item is a CUDA
    tensor, else a host array for the staging copy."""
    if items and all(isinstance(k, torch.Tensor) and k.is_cuda for k in items):
        return torch.cat([k.to(device=dev, dtype=torch.float32).reshape(-1, width) for k in items]).contiguous()
    return _host_pool(items, width)


def stage_with_pools(arrays, keypoints, klines, dev) -> dict:
    """`_ops.stage` of the host arrays plus the keypoint pool "kpts" [*, 2] and the key-line pool "segs" [*, 4]: a
    host pool goes up with the one staging copy (an empty one as one row of zeros, which no kernel reads), a pool of
    CUDA tensors is concatenated on the device.  -> the device tensors by name."""
    pools = {"kpts": _pool_rows(keypoints, 2, dev), "segs": _pool_rows(klines, 4, dev)}
    for nm, a in pools.items():
        if isinstance(a, np.ndarray):
            arrays[nm] = a if len(a) else np.zeros((1, a.shape[1]), np.float32)
    dv = _ops.stage(arrays, dev)
    for nm, a in pools.items():
        if isinstance(a, torch.Tensor):
            dv[nm] = a
    return dv
