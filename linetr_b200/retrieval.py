"""Image retrieval on the GPU (DESIGN.md "Image retrieval"): a spherical k-means vocabulary trained on an encoded
image set's point and line descriptors, intra-normalised VLAD global descriptors over both, and the exact top-k
database images of every query, as pair lists for `match_sets`, `estimate_absolute_poses`, `match_set`,
`triangulate_tracks` and `global_poses`.

The host models (`train_vocabulary_host`, `vlad_host`, `retrieve_host`) do the device's fp64 operations in its order
and give every output bit; they take the nearest-centroid assignment as an input (on the device it is the descriptor
matcher's).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

from . import _native as N
from . import _ops
from ._posed import block_sum
from .engine import ImageSet, exhaustive_pairs

_DL = 256
_THRESH = 16.0   # above every distance 2 - 2s of unit rows: every row is matched to its nearest centroid


# ------------------------------------------------------------------ host models
def _normalized_sum(s):
    """fl32(s / sqrt(|s|^2)) with |s|^2 the rt_block_sum256 of s_k^2, or None for |s| = 0."""
    n2 = block_sum((s * s).reshape(_DL, 1), _DL)[0]
    return (s / np.sqrt(n2)).astype(np.float32) if n2 > 0 else None


def _ordered_sum(x):
    """The fp64 sum over the rows of x [m, 256] in ascending row order."""
    return np.cumsum(np.vstack([np.zeros((1, _DL)), x]), axis=0)[-1]   # from +0.0, as the device


def init_rows(seed, n_rows, K):
    """The K distinct row indices of the initial centroids of a part (a seeded np.random.Generator)."""
    if n_rows < K:
        raise N.LtrError(f"train_vocabulary: {n_rows} rows for {K} clusters")
    return np.random.default_rng(seed).choice(n_rows, K, replace=False).astype(np.int32)


def kmeans_update_host(rows, assign, cent):
    """One centroid update: centroid c <- the normalised fp64 sum of its rows in ascending row order; a cluster
    without rows (or whose sum has norm 0) keeps its centroid.  rows fp32 [R, 256], assign [R], cent fp32 [K, 256]."""
    x = np.asarray(rows, np.float32).astype(np.float64)
    out = np.array(cent, np.float32, copy=True)
    for c in range(len(out)):
        sel = x[np.asarray(assign) == c]
        if len(sel):
            v = _normalized_sum(_ordered_sum(sel))
            if v is not None:
                out[c] = v
    return out


def train_vocabulary_host(rows, K, iters, seed, assign_fn):
    """Spherical k-means of one part: rows fp32 [R, 256], initial centroids the rows `init_rows(seed, R, K)`, then
    `iters` steps of assign_fn(rows, centroids) -> nearest centroid [R] and `kmeans_update_host`.  -> (centroids fp32
    [K, 256], [assignment of every step])."""
    rows = np.asarray(rows, np.float32)
    cent = rows[init_rows(seed, len(rows), K)].copy()
    history = []
    for _ in range(iters):
        a = np.asarray(assign_fn(rows, cent))
        history.append(a)
        cent = kmeans_update_host(rows, a, cent)
    return cent, history


def vlad_part_host(rows, assign, cent, w):
    """The VLAD part of one image: rows fp32 [m, 256] in ascending row order, assign [m], cent fp32 [K, 256] -> fp32
    [K * 256]: v_c = sum (x - c) in fp64, v_c / |v_c| (0 when empty or of norm 0), the part / |part| * sqrt(w)."""
    return vlad_part64(rows, assign, cent, w).astype(np.float32)


def vlad_part64(rows, assign, cent, w):
    """`vlad_part_host` before its rounding to fp32."""
    cent = np.asarray(cent, np.float32)
    K = len(cent)
    x = np.asarray(rows, np.float32).astype(np.float64).reshape(-1, _DL)
    a = np.asarray(assign).reshape(-1)
    u = np.zeros((K, _DL))
    for c in range(K):
        sel = x[a == c]
        if len(sel):
            v = _ordered_sum(sel - cent[c].astype(np.float64))
            n2 = block_sum((v * v).reshape(_DL, 1), _DL)[0]
            if n2 > 0:
                u[c] = v / np.sqrt(n2)
    # per component the squares in ascending cluster order, then rt_block_sum256
    pn = np.sqrt(block_sum((u * u).reshape(K * _DL, 1), _DL)[0])
    if not pn > 0:
        return np.zeros(K * _DL)
    return ((u / pn) * np.sqrt(np.float64(w))).reshape(-1)


def vlad_host(parts):
    """Global descriptors of n images: parts = [(rows_i per image, assign_i per image, centroids, w)] for points then
    lines -> fp32 [n, D]."""
    cols = [np.stack([vlad_part_host(r, a, c, w) for r, a in zip(rows, assign)]) for rows, assign, c, w in parts]
    return np.concatenate(cols, axis=1)


def exact_scores(q, db):
    """The exact score of every query and database row: fp64 products of the fp32 components, summed as one warp's
    block_sum(products, 32).  -> [Q, N] fp64."""
    q, db = np.asarray(q, np.float32).astype(np.float64), np.asarray(db, np.float32).astype(np.float64)
    Q, D = q.shape
    R = -(-D // 32)
    qp, dp = np.zeros((Q, R * 32)), np.zeros((len(db), R * 32))
    qp[:, :D], dp[:, :D] = q, db
    acc = np.zeros((Q, len(db), 32))
    for r in range(R):
        acc = acc + qp[:, None, r * 32:(r + 1) * 32] * dp[None, :, r * 32:(r + 1) * 32]
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[..., lanes ^ o]
    return 0.0 + acc[..., 0]


def retrieve_host(q, db, k, exclude_self=False):
    """The model of `retrieve`: per query the k database rows of highest exact score, ties to the lower index; -1 and
    NaN past the candidates.  -> (idx int32 [Q, k], score fp64 [Q, k])."""
    s = exact_scores(q, db)
    Q, Nn = s.shape
    idx = np.full((Q, k), -1, np.int32)
    score = np.full((Q, k), np.nan)
    for i in range(Q):
        j = np.arange(Nn)
        if exclude_self:
            j = j[j != i]
        order = j[np.lexsort((j, -s[i, j]))][:k]
        idx[i, :len(order)] = order
        score[i, :len(order)] = s[i, order]
    return idx, score


# ------------------------------------------------------------------ the vocabulary
@dataclass
class Vocabulary:
    """fp32 centroids [K_p, 256] of the point part and [K_l, 256] of the line part, and the part weights."""
    points: torch.Tensor
    lines: torch.Tensor
    w_points: float = 0.5
    w_lines: float = 0.5

    @property
    def dim(self) -> int:
        return _DL * (len(self.points) + len(self.lines))

    def save(self, path):
        np.savez(path, points=self.points.cpu().numpy(), lines=self.lines.cpu().numpy(),
                 weights=np.array([self.w_points, self.w_lines]))

    @staticmethod
    def load(path) -> "Vocabulary":
        with np.load(path) as z:
            w = z["weights"]
            return Vocabulary(torch.from_numpy(z["points"].copy()), torch.from_numpy(z["lines"].copy()), float(w[0]),
                              float(w[1]))


def _parts(s: ImageSet):
    """(name, descriptors, layout, host offsets, device offsets, tiles, host / device tile offsets) of both parts."""
    return (("points", s.desc_p, N.LAYOUT_CHANNEL_FIRST, s.cu_points, s.dev["cu_points"], s.tiles_p, s.tile_off_p,
             s.dev["tile_off_p"]),
            ("lines", s.desc_l, N.LAYOUT_ROWS, s.cu_lines, s.dev["cu_lines"], s.tiles_l, s.tile_off_l,
             s.dev["tile_off_l"]))


class _Centroids:
    """A part's centroids on the device in the forms the matcher reads: rows, channel-first and the tile image."""

    def __init__(self, K, dev):
        f32 = dict(dtype=torch.float32, device=dev)
        self.K = K
        self.rows = torch.empty((K, _DL), **f32)
        self.cf = torch.empty((_DL, K), **f32)
        self.tiles = torch.zeros(2 * -(-K // 128) * 4 * 128 * 64 * 2, dtype=torch.uint8, device=dev)
        self.counts = torch.empty(K, dtype=torch.int32, device=dev)
        i32 = dict(dtype=torch.int32, device=dev)
        self.cu = torch.tensor([0, K], **i32)
        self.tile_off = torch.tensor([0, -(-K // 128)], **i32)

    def update(self, desc, cu, layout, n_images, n_rows, *, assign=None, scores=None, cost=None, init=None):
        dev = self.rows.device
        ws = torch.empty(N.rt_kmeans_workspace_bytes(n_rows, self.K), dtype=torch.uint8, device=dev)
        _ops.call_struct("ltr_kmeans_update",
                         dict(desc=desc, cu=cu, layout=layout, n_images=n_images, n_rows=n_rows, K=self.K,
                              centroids_in=self.rows, assign=assign, scores=scores, init_rows=init),
                         dict(centroids=self.rows, centroids_cf=self.cf, tiles=self.tiles, counts=self.counts,
                              cost=cost, workspace=ws, workspace_bytes=ws.numel()))

    @staticmethod
    def of(cent: torch.Tensor, dev) -> "_Centroids":
        """The device forms of given centroids [K, 256] (ltr_kmeans_update's gather of every row)."""
        c = _Centroids(len(cent), dev)
        x = cent.to(dev, torch.float32).contiguous()
        c.update(x, c.cu, N.LAYOUT_ROWS, 1, c.K, init=torch.arange(c.K, dtype=torch.int32, device=dev))
        return c

    def assign(self, s: ImageSet, part):
        """The nearest centroid and its distance for every row of one part of s: ltr_match_indexed with the centroids as
        a one-image pool, mutual off and a threshold above every distance.  -> (assign int32 [R], scores fp32 [R])."""
        _, desc, layout, cu_h, cu_d, tiles, to_h, to_d = part
        dev, n, R = s.device, len(s), int(cu_h[-1])
        i32 = dict(dtype=torch.int32, device=dev)
        m0 = torch.empty(max(R, 1), **i32)[:R]
        sc = torch.empty(max(R, 1), dtype=torch.float32, device=dev)[:R]
        if R == 0:
            return m0, sc
        nn1 = torch.empty(n * self.K, **i32)
        _ops.match_indexed(desc, self.cf if layout == N.LAYOUT_CHANNEL_FIRST else self.rows, layout, n, _THRESH,
                           cu0=cu_d, cu1=self.cu, max_n0=int(np.diff(cu_h).max()), max_n1=self.K,
                           img0=torch.arange(n, **i32), img1=torch.zeros(n, **i32), tiles0=tiles, tiles1=self.tiles,
                           tile_off0=to_d, tile_off1=self.tile_off, n_tiles0=int(to_h[-1]), n_tiles1=-(-self.K // 128),
                           out_off0=cu_d, out_off1=torch.arange(0, (n + 1) * self.K, self.K, **i32), total_out0=R,
                           total_out1=n * self.K, matches0=m0, scores0=sc, nn1=nn1, counts=torch.empty(n, **i32),
                           mutual=False)
        return m0, sc


def train_vocabulary(image_set: ImageSet, k_points=64, k_lines=64, iters=20, seed=0, w_points=0.5, w_lines=0.5,
                     stats=None) -> Vocabulary:
    """Spherical k-means vocabularies of the set's point descriptors and of its line rows (one per subline): the
    initial centroids are the rows `init_rows(seed, ...)` of the points and `init_rows(seed + 1, ...)` of the lines,
    then `iters` steps of nearest-centroid assignment (the descriptor matcher) and centroid update.  No host
    synchronise.  stats, a dict, receives the k-means cost (sum of the assignment distances) of every step per part."""
    K = (int(k_points), int(k_lines))
    for kk in K:
        if not 1 <= kk <= N.RT_MAX_CLUSTERS:
            raise N.LtrError(f"train_vocabulary: clusters per part must lie in [1, {N.RT_MAX_CLUSTERS}], got {kk}")
    if int(iters) < 0:
        raise N.LtrError("train_vocabulary: iters must be >= 0")
    _check_weights(w_points, w_lines)
    parts = _parts(image_set)
    draws = []
    for i, (part, kk) in enumerate(zip(parts, K)):
        rows = int(part[3][-1])
        if rows < kk:
            raise N.LtrError(f"train_vocabulary: the {part[0]} part has {rows} rows for {kk} clusters")
        draws.append(init_rows(seed + i, rows, kk))
    dev, n = image_set.device, len(image_set)
    out = []
    for part, kk, d in zip(parts, K, draws):
        name, desc, layout, cu_h, cu_d = part[:5]
        c = _Centroids(kk, dev)
        c.update(desc, cu_d, layout, n, int(cu_h[-1]), init=torch.from_numpy(d).to(dev))
        cost = torch.zeros(max(int(iters), 1), dtype=torch.float64, device=dev)
        for it in range(int(iters)):
            a, sc = c.assign(image_set, part)
            c.update(desc, cu_d, layout, n, int(cu_h[-1]), assign=a, scores=sc, cost=cost[it:it + 1])
        if stats is not None:
            stats[name + "_cost"] = cost[:int(iters)]
            stats[name + "_counts"] = c.counts
        out.append(c.rows)
    return Vocabulary(out[0], out[1], float(w_points), float(w_lines))


def _check_weights(wp, wl):
    """The part weights: finite, >= 0 and w_p + w_l <= 1, so every global descriptor has norm <= 1 (the screening
    bound LTR_RT_EPS holds for descriptors of norm <= 1)."""
    if not (np.isfinite(wp) and np.isfinite(wl) and wp >= 0 and wl >= 0 and wp + wl <= 1.0):
        raise N.LtrError("retrieval: the part weights must be finite, >= 0 and sum to at most 1")


# ------------------------------------------------------------------ global descriptors
@dataclass
class GlobalDescriptors:
    """fp32 [n, D] global descriptors on the device and their split-bf16 tile image."""
    desc: torch.Tensor
    tiles: torch.Tensor

    def __len__(self) -> int:
        return int(self.desc.shape[0])

    @property
    def device(self):
        return self.desc.device

    @staticmethod
    def from_rows(x: torch.Tensor, max_norm: float = 1.0 + 1e-6) -> "GlobalDescriptors":
        """Given fp32 rows [n, D] (CUDA, D a multiple of 64), with the tile image built on the device.  The rows must
        have norm <= 1: `retrieve`'s margin LTR_RT_EPS bounds the screened score of such rows only, so `max_norm`
        (default 1 + 1e-6) is checked here, which reads one value back to the host."""
        if not isinstance(x, torch.Tensor) or not x.is_cuda or x.dim() != 2 or x.dtype != torch.float32:
            raise N.LtrError("GlobalDescriptors.from_rows: x must be a CUDA float32 tensor [n, D]")
        n, D = (int(v) for v in x.shape)
        if n < 1 or D < 64 or D % 64:
            raise N.LtrError(f"GlobalDescriptors.from_rows: need n >= 1 and D a positive multiple of 64, got {[n, D]}")
        x = x.contiguous()
        if float(torch.linalg.vector_norm(x.double(), dim=1).max()) > max_norm:
            raise N.LtrError(f"GlobalDescriptors.from_rows: rows of norm above {max_norm}; retrieval's screening bound "
                             "holds for rows of norm <= 1")
        tiles = torch.empty(4 * -(-n // 128) * 128 * D, dtype=torch.uint8, device=x.device)
        _ops._call("ltr_rt_tiles", x.device, _ops._ptr(x), n, D, _ops._ptr(tiles))
        return GlobalDescriptors(x, tiles)


def global_descriptors(image_set: ImageSet, vocab: Vocabulary) -> GlobalDescriptors:
    """The intra-normalised VLAD of every image of the set over the vocabulary's point and line parts (ltr_vlad),
    assignments by the descriptor matcher.  No host synchronise."""
    if not isinstance(vocab, Vocabulary):
        raise N.LtrError("global_descriptors: vocab must be a Vocabulary")
    for nm, c in (("points", vocab.points), ("lines", vocab.lines)):
        if c.dim() != 2 or c.shape[1] != _DL or not 1 <= c.shape[0] <= N.RT_MAX_CLUSTERS:
            raise N.LtrError(f"global_descriptors: the vocabulary's {nm} must be [K, 256] with K in "
                             f"[1, {N.RT_MAX_CLUSTERS}], got {list(c.shape)}")
    _check_weights(vocab.w_points, vocab.w_lines)
    dev, n = image_set.device, len(image_set)
    if n < 1:
        raise N.LtrError("global_descriptors: empty image set")
    fields = {}
    keep = []
    for part, cent, w, sfx in zip(_parts(image_set), (vocab.points, vocab.lines), (vocab.w_points, vocab.w_lines),
                                  ("p", "l")):
        c = _Centroids.of(cent, dev)
        a, _ = c.assign(image_set, part)
        keep += [c, a]
        fields.update({f"desc_{sfx}": part[1], f"cu_{sfx}": part[4], f"layout_{sfx}": part[2],
                       f"rows_{sfx}": int(part[3][-1]), f"assign_{sfx}": a if len(a) else None,
                       f"centroids_{sfx}": c.rows, f"k_{sfx}": c.K, f"w_{sfx}": float(w)})
    D = vocab.dim
    desc = torch.empty((n, D), dtype=torch.float32, device=dev)
    tiles = torch.empty(4 * -(-n // 128) * 128 * D, dtype=torch.uint8, device=dev)
    ws_bytes = N.rt_vlad_workspace_bytes(n, fields["rows_p"], fields["rows_l"], fields["k_p"], fields["k_l"])
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    _ops.call_struct("ltr_vlad", dict(n_images=n, **fields),
                     dict(desc=desc, tiles=tiles, workspace=ws, workspace_bytes=ws.numel()))
    return GlobalDescriptors(desc, tiles)


# ------------------------------------------------------------------ top-k retrieval
@dataclass
class Retrieval:
    """idx int32 [Q, k] (-1 past the candidates), score fp64 [Q, k] (NaN there), n_full: queries that took the full
    exact pass (int32 [1] on the device)."""
    idx: torch.Tensor
    score: torch.Tensor
    n_full: torch.Tensor

    def pairs(self):
        """(pairs int32 [P, 2] of (query, database image) in query-major order without the -1 slots, groups int32
        [Q + 1]): the pair list and groups `match_sets` and `estimate_absolute_poses` take."""
        idx = self.idx.cpu().numpy()
        keep = idx >= 0
        q = np.repeat(np.arange(len(idx)), keep.sum(1))
        pairs = np.stack([q, idx[keep]], 1).astype(np.int32).reshape(-1, 2)
        groups = np.zeros(len(idx) + 1, np.int32)
        groups[1:] = np.cumsum(keep.sum(1))
        return pairs, groups


def _as_descriptors(x, who, what) -> GlobalDescriptors:
    if isinstance(x, GlobalDescriptors):
        return x
    raise N.LtrError(f"{who}: {what} must be GlobalDescriptors")


def retrieve(queries, database, k, exclude_self=False) -> Retrieval:
    """The k database images of highest exact score for every query, for descriptors of norm <= 1 (those of
    `global_descriptors` and of `GlobalDescriptors.from_rows`) (ltr_retrieve: a tensor-core screen, then exact
    fp64 rescoring, DESIGN.md "Image retrieval"); ties go to the lower index; exclude_self skips database index q for
    query q.  No host synchronise."""
    q = _as_descriptors(queries, "retrieve", "queries")
    db = _as_descriptors(database, "retrieve", "database")
    k = int(k)
    if not 1 <= k <= N.RT_MAX_K:
        raise N.LtrError(f"retrieve: k must lie in [1, {N.RT_MAX_K}], got {k}")
    if len(db) < 1 or len(q) < 1:
        raise N.LtrError("retrieve: empty query set or database")
    if q.desc.shape[1] != db.desc.shape[1]:
        raise N.LtrError(f"retrieve: queries of dimension {q.desc.shape[1]}, database of {db.desc.shape[1]}")
    if q.device != db.device:
        raise N.LtrError(f"retrieve: queries on {q.device}, database on {db.device}")
    Q, Nn, D = len(q), len(db), int(q.desc.shape[1])
    if D > 2 * _DL * N.RT_MAX_CLUSTERS:
        raise N.LtrError(f"retrieve: D = {D} is larger than {2 * _DL * N.RT_MAX_CLUSTERS}")
    dev = q.device
    idx = torch.empty((Q, k), dtype=torch.int32, device=dev)
    score = torch.empty((Q, k), dtype=torch.float64, device=dev)
    n_full = torch.empty(1, dtype=torch.int32, device=dev)
    ws = torch.empty(N.rt_workspace_bytes(Q, Nn, k), dtype=torch.uint8, device=dev)
    _ops.call_struct("ltr_retrieve",
                     dict(q=q.desc, q_tiles=q.tiles, db=db.desc, db_tiles=db.tiles, Q=Q, N=Nn, D=D, k=k,
                          exclude_self=int(bool(exclude_self))),
                     dict(idx=idx, score=score, n_full=n_full, workspace=ws, workspace_bytes=ws.numel()))
    return Retrieval(idx, score, n_full)


def pairs_from_topk(idx) -> np.ndarray:
    """Retrieval within one set -> int32 [P, 2]: each (query, result) as (min, max), deduplicated and sorted."""
    idx = np.asarray(idx)
    q = np.repeat(np.arange(len(idx)), idx.shape[1])
    j = idx.reshape(-1)
    keep = j >= 0
    a, b = np.minimum(q[keep], j[keep]), np.maximum(q[keep], j[keep])
    return np.unique(np.stack([a, b], 1).astype(np.int32).reshape(-1, 2), axis=0).astype(np.int32).reshape(-1, 2)


def retrieval_pairs(descriptors: GlobalDescriptors, k) -> np.ndarray:
    """The image pairs of one set for `match_set`, `triangulate_tracks` and `global_poses`: every image with its k
    best other images (`retrieve(..., exclude_self=True)`), as (min, max), deduplicated and sorted.  With k >= n - 1
    this is `exhaustive_pairs(n)`.  Reads the result back to the host."""
    d = _as_descriptors(descriptors, "retrieval_pairs", "descriptors")
    k = int(k)
    if k < 1:
        raise N.LtrError(f"retrieval_pairs: k must be >= 1, got {k}")
    n = len(d)
    if n < 2:
        return np.zeros((0, 2), np.int32)
    if k >= n - 1:
        return exhaustive_pairs(n)
    return pairs_from_topk(retrieve(d, d, k, exclude_self=True).idx.cpu().numpy())


def descriptor_set(points, lines, device) -> ImageSet:
    """An ImageSet of given local descriptors, without the encoder: points[i] fp32 [m_i, 256] and lines[i] fp32
    [l_i, 256] unit rows of image i (each key line one subline), for `train_vocabulary` and `global_descriptors`."""
    if len(points) != len(lines):
        raise N.LtrError("descriptor_set: points and lines must list the same images")
    dev = torch.device(device)
    n = len(points)
    cnt = lambda xs: np.concatenate([[0], np.cumsum([len(x) for x in xs])]).astype(np.int32)   # noqa: E731
    cup, cul = cnt(points), cnt(lines)
    cat = lambda xs: (np.concatenate([np.asarray(x, np.float32).reshape(-1) for x in xs]) if n else  # noqa: E731
                      np.zeros(0, np.float32))
    pool = torch.from_numpy(cat([np.asarray(p, np.float32).reshape(-1, _DL).T for p in points])).to(dev)
    rows = torch.from_numpy(cat(lines)).to(dev).reshape(-1, _DL)
    to_l, to_p = _ops.tile_offsets(cul), _ops.tile_offsets(cup)
    dv = _ops.stage({"cu_lines": cul, "cuk": cul, "tile_off_l": to_l, "cu_points": cup, "tile_off_p": to_p,
                     "sub_off": np.arange(cul[-1] + 1, dtype=np.int32)}, dev)
    tiles_l = _ops.image_tiles(rows, N.LAYOUT_ROWS, cul, dv["cu_lines"], dv["tile_off_l"], int(to_l[-1]))
    tiles_p = _ops.image_tiles(pool, N.LAYOUT_CHANNEL_FIRST, cup, dv["cu_points"], dv["tile_off_p"], int(to_p[-1]))
    return ImageSet(rows, tiles_l, pool, tiles_p, cul, cul.copy(), np.arange(cul[-1] + 1, dtype=np.int32), to_l, cup,
                    to_p, dv, [np.zeros((len(x), 4), np.float32) for x in lines],
                    [np.zeros((len(x), 2), np.float32) for x in points], dev)
