"""Batched front-end of the hot path: many image pairs per call, everything on the device.

The reference's `Matching.forward` (models/matching.py:18-86) handles ONE pair per call and
round-trips through host numpy between descriptor forward, distance matrix, subline merge
and matcher (matching.py:69-84).  `PairEngine.match_pairs` runs the same line branch
(matching.py:77-81) for a whole batch of independent pairs: two `ltr_encode` calls (side 0,
side 1; images of different line counts are handled with `cu_lines`, never by padding - the
signature attention has no mask, SURVEY.md §0 fact 6) and one `ltr_match`.

Pairs are independent, so multi-GPU use is plain sharding (`shard_range`) plus one
all-gather of the per-pair match counts (`gather_counts`); see DESIGN.md §multi-GPU.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _native as N
from . import _ops
from . import line_process as LP

_KEYS = ("sublines", "resp_sublines", "angle_sublines", "pnt_sublines", "desc_sublines", "score_sublines")


def _uniform(cu) -> Optional[int]:
    """The line count of every image of line offsets `cu` when they all have the same, else None."""
    d = np.diff(cu)
    return int(d[0]) if len(d) and bool((d == d[0]).all()) else None


@dataclass
class LineBatch:
    """Tokenised lines of a batch of images, rows of all images concatenated.

    sublines [R,2,2], resp [R,1], angle [R,2], pnt [R,T,2], desc [R,T,256], score [R,T,1];
    cu_lines: np.int32 [n_images+1] line offsets.  Optional key-line structure for
    subline->keyline merging: sub_off np.int32 [n_keylines+1] (CSR, global subline numbering)
    and cuk np.int32 [n_images+1]; None means every subline is its own key line.
    """
    sublines: torch.Tensor
    resp: torch.Tensor
    angle: torch.Tensor
    pnt: torch.Tensor
    desc: torch.Tensor
    score: torch.Tensor
    cu_lines: np.ndarray
    sub_off: Optional[np.ndarray] = None
    cuk: Optional[np.ndarray] = None
    _dev_cache: dict = field(default_factory=dict, repr=False)

    @property
    def n_images(self) -> int:
        return len(self.cu_lines) - 1

    @property
    def n_lines(self) -> int:
        return int(self.cu_lines[-1])

    @property
    def n_tokens(self) -> int:
        return int(self.desc.shape[1])

    @property
    def uniform_lines(self) -> Optional[int]:
        return _uniform(self.cu_lines)

    def nbytes(self) -> int:
        return sum(t.numel() * t.element_size() for t in self.tensors())

    def tensors(self):
        return (self.sublines, self.resp, self.angle, self.pnt, self.desc, self.score)

    @staticmethod
    def from_stacked(data: dict) -> "LineBatch":
        """From the reference's stacked dict layout [B,L,...] (line_process.py:182-193)."""
        B, L = int(data["desc_sublines"].shape[0]), int(data["desc_sublines"].shape[1])
        T = int(data["desc_sublines"].shape[2])
        f = lambda k, *s: torch.as_tensor(data[k]).float().reshape(B * L, *s).contiguous()
        return LineBatch(f("sublines", 2, 2), f("resp_sublines", 1), f("angle_sublines", 2), f("pnt_sublines", T, 2),
                         f("desc_sublines", T, 256), f("score_sublines", T, 1),
                         (np.arange(B + 1, dtype=np.int64) * L).astype(np.int32))

    @staticmethod
    def from_images(images: Sequence[dict]) -> "LineBatch":
        """From per-image tokenizer dicts (batch dim 1 each); line counts may differ.  Uses
        'mat_klines2sublines' (if present and not the identity) to build the key-line CSR."""
        from .nn_matcher import adjacency_to_csr
        T = int(images[0]["desc_sublines"].shape[2])
        cat = lambda k, *s: torch.cat([torch.as_tensor(im[k])[0].float().reshape(-1, *s) for im in images], 0).contiguous()
        counts = [int(im["desc_sublines"].shape[1]) for im in images]
        cu = np.zeros(len(images) + 1, dtype=np.int32)
        cu[1:] = np.cumsum(counts)
        sub_off = cuk = None
        if all("mat_klines2sublines" in im for im in images):
            offs, nk, merged = [], [], False
            for im, base in zip(images, cu[:-1]):
                A = im["mat_klines2sublines"]
                A = A.detach().cpu().numpy() if isinstance(A, torch.Tensor) else np.asarray(A)
                o = adjacency_to_csr(A[0])
                merged |= len(o) - 1 != o[-1]
                offs.append(o[:-1].astype(np.int64) + int(base))
                nk.append(len(o) - 1)
            if merged:
                sub_off = np.concatenate(offs + [np.array([cu[-1]], dtype=np.int64)]).astype(np.int32)
                cuk = np.zeros(len(images) + 1, dtype=np.int32)
                cuk[1:] = np.cumsum(nk)
        return LineBatch(cat("sublines", 2, 2), cat("resp_sublines", 1), cat("angle_sublines", 2),
                         cat("pnt_sublines", T, 2), cat("desc_sublines", T, 256), cat("score_sublines", T, 1),
                         cu, sub_off, cuk)

    def pin(self) -> "LineBatch":
        return LineBatch(*[t.pin_memory() for t in self.tensors()], self.cu_lines, self.sub_off, self.cuk)

    def to(self, device, non_blocking=True) -> "LineBatch":
        return LineBatch(*[t.to(device, non_blocking=non_blocking) for t in self.tensors()], self.cu_lines,
                         self.sub_off, self.cuk)

    def dev_i32(self, name: str, device) -> torch.Tensor:
        return self._dev_i32((name,), getattr(self, name), device)

    def _dev_i32(self, key: tuple, a: np.ndarray, device) -> torch.Tensor:
        """Device int32 copy of a host array of this batch, made once per key and device."""
        key = key + (str(device),)
        if key not in self._dev_cache:
            self._dev_cache[key] = torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(device)
        return self._dev_cache[key]


def merge_sublines(dist_sub: torch.Tensor, sub_off0: torch.Tensor, sub_off1: torch.Tensor, K0: int, K1: int):
    """A0 @ D @ A1^T for ONE pair on the GPU (ltr_merge_sublines); dist_sub [S0,S1] CUDA."""
    dev = dist_sub.device
    dist_sub = dist_sub.float().contiguous()
    cuk0 = torch.tensor([0, K0], dtype=torch.int32, device=dev)
    cuk1 = torch.tensor([0, K1], dtype=torch.int32, device=dev)
    out = torch.empty((K0, K1), dtype=torch.float32, device=dev)
    p = lambda t: C.c_void_p(t.data_ptr())
    _ops._call("ltr_merge_sublines", dev, p(dist_sub), 0, 1, p(cuk0), p(cuk1), p(sub_off0.int().contiguous()),
               p(sub_off1.int().contiguous()), K0, K1, p(out), 0)
    return out


@dataclass
class PairMatches:
    matches0: torch.Tensor     # int32 [total key lines side 0]: index in side 1 (local to the pair) or -1
    scores0: torch.Tensor      # float32, distance to the nearest neighbour
    counts: torch.Tensor       # int32 [n_pairs]
    offsets0: np.ndarray       # int32 [n_pairs+1] key-line offsets of side 0 into matches0
    dist: Optional[torch.Tensor]   # float32 flat, pair p at p*stride, row-major [K0_p, K1_p]; None unless requested
    stride: int                    # (want_dist=True) or needed for key-line merging
    desc0: Optional[torch.Tensor] = None   # [R0,256] unit descriptors (rows)
    desc1: Optional[torch.Tensor] = None

    def pair(self, p: int) -> torch.Tensor:
        return self.matches0[int(self.offsets0[p]):int(self.offsets0[p + 1])]


def _first(x):
    """SuperPoint returns per-image lists (or a batch of one): the first entry."""
    return x[0] if isinstance(x, (list, tuple)) or (isinstance(x, torch.Tensor) and x.dim() == 3 and x.shape[0] == 1) else x


def _dense_scores(dist: Optional[torch.Tensor], stride: int, p: int, n0: int, n1: int) -> np.ndarray:
    if dist is None or n0 == 0 or n1 == 0:
        return np.zeros((1, n0, n1), dtype=np.float32)
    return dist[p * stride:p * stride + n0 * n1].view(1, n0, n1).cpu().numpy()


@dataclass
class ImagePairMatches:
    """Line and point matches of a batch of image pairs (`PairEngine.match_images`).

    matches_l int32 [total side-0 key lines] (index local to the pair or -1), scores_l float32 (distance to the
    nearest neighbour), counts_l int32 [P], offsets_l np.int32 [P+1] (side-0 key lines of pair p); the same
    four fields for the SuperPoint keypoints (matches_p, scores_p, counts_p, offsets_p).  With want_scores the
    distance matrices: pair p at p * stride, row-major [K0_p, K1_p] / [N0_p, N1_p].  klines0/1: each image's
    tokenised key lines (after the reference's in-place clip), keypoints0/1: each image's keypoints."""
    matches_l: torch.Tensor
    scores_l: torch.Tensor
    counts_l: torch.Tensor
    offsets_l: np.ndarray
    matches_p: torch.Tensor
    scores_p: torch.Tensor
    counts_p: torch.Tensor
    offsets_p: np.ndarray
    klines0: List[np.ndarray]
    klines1: List[np.ndarray]
    keypoints0: list
    keypoints1: list
    dist_l: Optional[torch.Tensor] = None
    stride_l: int = 0
    dist_p: Optional[torch.Tensor] = None
    stride_p: int = 0

    @property
    def n_pairs(self) -> int:
        return len(self.offsets_l) - 1

    def pair_lines(self, p: int) -> torch.Tensor:
        return self.matches_l[int(self.offsets_l[p]):int(self.offsets_l[p + 1])]

    def pair_points(self, p: int) -> torch.Tensor:
        return self.matches_p[int(self.offsets_p[p]):int(self.offsets_p[p + 1])]

    def reference_dict(self, p: int) -> dict:
        """The match keys `Matching.forward` returns for pair p (models/matching.py:69-84): matches_l float64
        [1,K0,K1], matching_scores_l float32 [1,K0,K1], matches_p float64 [1,N0,N1], matching_scores_p float32
        [1,N0,N1].  Needs want_scores=True; copies to the host."""
        if self.dist_l is None or self.dist_p is None:
            raise N.LtrError("reference_dict needs match_images(..., want_scores=True)")
        from .match_io import indices_to_dense
        K0, K1 = len(self.klines0[p]), len(self.klines1[p])
        N0, N1 = len(self.keypoints0[p]), len(self.keypoints1[p])
        ml, mp = self.pair_lines(p).cpu().numpy(), self.pair_points(p).cpu().numpy()
        return {"matches_l": torch.from_numpy(indices_to_dense(ml, K1)[None]),
                "matching_scores_l": torch.from_numpy(_dense_scores(self.dist_l, self.stride_l, p, K0, K1)),
                "matches_p": torch.from_numpy(indices_to_dense(mp, N1)[None]),
                "matching_scores_p": torch.from_numpy(_dense_scores(self.dist_p, self.stride_p, p, N0, N1))}


@dataclass
class ImageSet:
    """Images encoded once (`PairEngine.encode_images`) for any number of `PairEngine.match_sets` calls.

    desc_l [R,256] unit line descriptors (rows; image i owns sublines [cu_lines[i], cu_lines[i+1])), tiles_l their
    image-aligned tile image (image i from tile tile_off_l[i]); the key-line CSR cuk [n+1] / sub_off [K+1] (global
    subline numbering, the identity for images without split lines); desc_p the SuperPoint point descriptors of all
    images, channel-first [256, N_i] blocks back to back (image i at 256 * cu_points[i]), tiles_p their tile image.
    Host int32 offset arrays, their device copies in `dev`.  klines / keypoints: each image's tokenised key lines
    (after the reference's in-place clip) and keypoints.  The tokenised token descriptors are not kept."""
    desc_l: torch.Tensor
    tiles_l: torch.Tensor
    desc_p: torch.Tensor
    tiles_p: torch.Tensor
    cu_lines: np.ndarray
    cuk: np.ndarray
    sub_off: np.ndarray
    tile_off_l: np.ndarray
    cu_points: np.ndarray
    tile_off_p: np.ndarray
    dev: dict
    klines: List[np.ndarray]
    keypoints: list
    device: torch.device

    def __len__(self) -> int:
        return len(self.cu_lines) - 1


# Cap on the subline distance scratch of one line match with key-line merging (n_pairs * max_n0 * max_n1 fp32):
# match_sets cuts longer pair lists into consecutive chunks that stay under it.
DIST_SUB_CAP = 512 << 20
# Pairs per matcher launch: the pair index is the grid's y dimension.
MAX_PAIRS_PER_CALL = 65535


def exhaustive_pairs(n: int) -> np.ndarray:
    """All pairs (i, j) with i < j of n images, row-major order: int32 [n(n-1)/2, 2]."""
    i, j = np.triu_indices(int(n), k=1)
    return np.ascontiguousarray(np.stack([i, j], 1), dtype=np.int32).reshape(-1, 2)


def check_pairs(pairs, n0: int, n1: int) -> np.ndarray:
    """A host pair list [P, 2] of image indices, column 0 into a set of n0 images and column 1 into one of n1 ->
    int32 [P, 2]; raises LtrError on a wrong shape or dtype or an index out of range."""
    if isinstance(pairs, torch.Tensor):
        if pairs.is_cuda:
            raise N.LtrError("match_sets: pairs must be a host array")
        pairs = pairs.numpy()
    a = np.asarray(pairs)
    if a.ndim == 1 and a.size == 0:   # an empty list
        a = a.reshape(0, 2)
    if a.ndim != 2 or a.shape[1] != 2:
        raise N.LtrError(f"match_sets: pairs must have shape [P, 2], got {list(a.shape)}")
    if a.size == 0:
        return np.zeros((0, 2), dtype=np.int32)
    if not np.issubdtype(a.dtype, np.integer):
        raise N.LtrError(f"match_sets: pairs must be integers, got {a.dtype}")
    if (a < 0).any():
        raise N.LtrError("match_sets: negative image index in pairs")
    if (a[:, 0] >= n0).any():
        raise N.LtrError(f"match_sets: pairs[:, 0] out of range for a set of {n0} images")
    if (a[:, 1] >= n1).any():
        raise N.LtrError(f"match_sets: pairs[:, 1] out of range for a set of {n1} images")
    return np.ascontiguousarray(a, dtype=np.int32)


def plan_chunks(n0, n1, cap_bytes: Optional[int] = None, max_pairs: int = MAX_PAIRS_PER_CALL):
    """Consecutive chunks [(begin, end)] of a pair list with per-pair subline counts n0 / n1 such that each chunk's
    distance scratch, len * max n0 * max n1 * 4 bytes, stays within cap_bytes (default DIST_SUB_CAP) and a chunk
    holds at most max_pairs pairs.  A pair that alone exceeds the cap gets a chunk of its own."""
    cap = DIST_SUB_CAP if cap_bytes is None else int(cap_bytes)
    chunks, a, m0, m1 = [], 0, 0, 0
    for p in range(len(n0)):
        c0, c1 = max(m0, int(n0[p])), max(m1, int(n1[p]))
        if p > a and ((p - a + 1) * c0 * c1 * 4 > cap or p - a >= max_pairs):
            chunks.append((a, p))
            a, c0, c1 = p, int(n0[p]), int(n1[p])
        m0, m1 = c0, c1
    if len(n0):
        chunks.append((a, len(n0)))
    return chunks


def _side(batch: LineBatch, a: int, b: int, split: bool) -> dict:
    """Images [a, b) of `batch` as one side of a batch of pairs, in the side's own line numbering (host arrays): line
    offsets 'cu' and, when `split` (some key line of the match is cut into sublines), key-line offsets 'cuk' and the
    key-line CSR 'sub_off', the identity for a batch without split key lines."""
    cu = batch.cu_lines
    side = dict(cu=cu[a:b + 1] - cu[a])
    if split and batch.sub_off is None:
        side.update(cuk=side["cu"], sub_off=np.arange(cu[b] - cu[a] + 1))
    elif split:
        ck = batch.cuk
        side.update(cuk=ck[a:b + 1] - ck[a], sub_off=batch.sub_off[ck[a]:ck[b] + 1] - cu[a])
    return side


def _tiled(s0: dict, s1: dict) -> bool:
    """Whether the encoder's final GEMM can write the matcher's operand tiles itself: no key-line merging and, on each
    side, every image with the same positive multiple of 128 lines."""
    uniform = (_uniform(s0["cu"]), _uniform(s1["cu"]))
    return "sub_off" not in s0 and all(L is not None and L > 0 and L % 128 == 0 for L in uniform)


class PairEngine:
    """Batched line-descriptor forward + mutual-NN matching on one GPU."""

    def __init__(self, model, device=None):
        self.model = model
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if self.device.type != "cuda":
            raise N.LtrError("PairEngine needs a CUDA device (there is no CPU fallback)")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())

    def encode(self, batch: LineBatch, want_cf=False, want_tiles=False):
        """-> unit descriptors [R,256] (rows); with want_cf also the flat channel-first layout, with
        want_tiles also the descriptor tile image the tensor-core matcher contracts (`ltr_encode`
        writes it from the same epilogue as the rows)."""
        h = self.model._get_handle(self.device)
        L = batch.uniform_lines
        kw = dict(lines_per_image=L) if L is not None and L > 0 else dict(
            cu_lines_host=batch.cu_lines, cu_lines_dev=batch.dev_i32("cu_lines", self.device))
        res = _ops.encode(h, batch.sublines, batch.resp, batch.angle, batch.pnt, batch.desc, batch.score,
                          self.model._image_wh(), want_cf=want_cf, want_rows=True, want_tiles=want_tiles, **kw)
        if want_tiles:
            return res[1], res[2]
        return (res[1], res[0]) if want_cf else res[1]

    def match_pairs(self, side0: LineBatch, side1: LineBatch, nn_thresh: Optional[float] = None, mutual=True,
                    keep_desc=False, want_dist=False, gather=None) -> PairMatches:
        """want_dist=True also returns the key-line distance matrices (`Matching`'s
        'matching_scores_l'); by default they are never materialised (the row argmin lives in the
        epilogue of the tensor-core contraction) unless key-line merging needs them."""
        if side0.n_images != side1.n_images:
            raise ValueError("match_pairs: both sides need the same number of images")
        P = side0.n_images
        split = side0.sub_off is not None or side1.sub_off is not None
        s0, s1 = _side(side0, 0, P, split), _side(side1, 0, P, split)
        if _tiled(s0, s1):
            d0, t0 = self.encode(side0, want_tiles=True)
            d1, t1 = self.encode(side1, want_tiles=True)
            tiles = dict(tiles0=t0, tiles1=t1, tiles_lines=(side0.n_lines, side1.n_lines), tiles_row0=(0, 0))
        else:
            d0, d1, tiles = self.encode(side0), self.encode(side1), {}
        dev = lambda s, k: (side0, side1)[s]._dev_i32(("match_side", 0, P, k), (s0, s1)[s][k], self.device)
        return self._match_sides(d0, d1, s0, s1, dev, tiles, nn_thresh, mutual, keep_desc, want_dist, gather)

    def match_packed(self, batch: LineBatch, n_pairs: int, nn_thresh: Optional[float] = None, mutual=True,
                     keep_desc=False, want_dist=False, gather=None) -> PairMatches:
        """Same as match_pairs for a batch that holds BOTH sides: images [0, P) are the side-0
        images of the P pairs, images [P, 2P) their side-1 partners.  One `ltr_encode` over all
        2P images (twice the rows per GEMM launch) and one `ltr_match`."""
        return self._match_packed(batch, n_pairs, nn_thresh, mutual, keep_desc, want_dist, gather)

    def _match_packed(self, batch: LineBatch, n_pairs: int, nn_thresh, mutual=True, keep_desc=False, want_dist=False,
                      gather=None, staged: Optional[dict] = None) -> PairMatches:
        """match_packed.  staged: device copies the caller has already made of the sides' offsets, by matcher keyword
        (cu0, cu1 and, with split key lines, cuk0, cuk1, sub_off0, sub_off1)."""
        P = int(n_pairs)
        if batch.n_images != 2 * P:
            raise ValueError("match_packed: batch must hold 2 * n_pairs images")
        split = batch.sub_off is not None
        s0, s1 = _side(batch, 0, P, split), _side(batch, P, 2 * P, split)
        R0 = int(batch.cu_lines[P])
        if _tiled(s0, s1):
            rows, t = self.encode(batch, want_tiles=True)
            tiles = dict(tiles0=t, tiles1=t, tiles_lines=(batch.n_lines, batch.n_lines), tiles_row0=(0, R0))
        else:
            rows, tiles = self.encode(batch), {}
        if staged is not None:
            dev = lambda s, k: staged[f"{k}{s}"]
        else:
            dev = lambda s, k: batch._dev_i32(("match_side", s * P, s * P + P, k), (s0, s1)[s][k], self.device)
        return self._match_sides(rows[:R0], rows[R0:], s0, s1, dev, tiles, nn_thresh, mutual, keep_desc, want_dist,
                                 gather)

    def _match_sides(self, d0, d1, s0: dict, s1: dict, dev, tiles: dict, nn_thresh, mutual, keep_desc, want_dist,
                     gather) -> PairMatches:
        """One `ltr_match` of the pairs whose side 0 / side 1 are `s0` / `s1` (`_side`), descriptor rows d0 / d1.
        dev(s, name): the device copy of array `name` of side s, asked for only when a side is ragged or key lines
        are merged; tiles: the encoder's operand tiles (matcher keywords), used only when both sides are uniform."""
        if nn_thresh is None:
            nn_thresh = self.model.config.get("nn_threshold", 0.8)
        L0, L1 = _uniform(s0["cu"]), _uniform(s1["cu"])
        if "sub_off" not in s0 and L0 is not None and L1 is not None:
            kw = dict(n0=L0, n1=L1, **tiles)
        else:
            mx = lambda a: int(np.diff(a).max(initial=0))
            kw = {}
            for s, side in enumerate((s0, s1)):
                kw.update({f"{k}{s}": dev(s, k) for k in side})
                kw.update({f"max_n{s}": mx(side["cu"]), f"total_k{s}": int(side.get("cuk", side["cu"])[-1])})
                if "cuk" in side:
                    kw[f"max_k{s}"] = mx(side["cuk"])
        off0 = s0.get("cuk", s0["cu"])
        out = _ops.match_descriptors(d0, d1, N.LAYOUT_ROWS, len(off0) - 1, float(nn_thresh), mutual, want_dist=want_dist,
                                     gather=gather, **kw)
        return PairMatches(out["matches0"], out["scores0"], out["counts"], np.asarray(off0, dtype=np.int32),
                           out["dist_key"], out["stride"], d0 if keep_desc else None, d1 if keep_desc else None)

    # ------------------------------------------------------------------ image-level front-end
    def _image_specs(self, images, auto_min_length):
        specs = [(im["klines"], tuple(im["image_shape"]), im.get("valid_mask")) for im in images]
        return specs, [LP.tokenizer_config(self.model.config, sh, auto_min_length) for _, sh, _ in specs]

    def _tokenize(self, host: "LP.TokenizerBatch", images: Sequence[dict], dv: dict) -> LineBatch:
        """ltr_tokenize_batch of `host` (its per-key-line arrays already staged in `dv`) -> the packed LineBatch."""
        maps = []
        for i, im in enumerate(images[:host.n_images]):
            if host.cu_lines[i + 1] == host.cu_lines[i]:
                maps.append(None)
                continue
            dense = im["dense_descriptor"]
            if not dense.is_cuda or dense.device != self.device:
                raise N.LtrError(f"match_images: SuperPoint maps must be on {self.device} (there is no CPU fallback)")
            maps.append((dense, im["dense_score"], host.token_distance[i]))
        cu = np.ascontiguousarray(host.cu_lines, dtype=np.int32)
        slines, pnt, mask, resp, ang, desc, score = _ops.tokenize(dv, maps, cu, host.max_tokens, self.device)
        batch = LineBatch(slines, resp, ang, pnt, desc, score, cu, host.sub0 if host.split else None,
                          host.cuk if host.split else None)
        batch._dev_cache[("cu_lines", str(self.device))] = dv["cu_lines"]
        return batch

    @staticmethod
    def _tok_arrays(host: "LP.TokenizerBatch") -> dict:
        return {"sp": host.sp, "ep": host.ep, "epc": host.epc, "length": host.length, "angle": host.angle,
                "n_tok": host.n_tok, "sub0": host.sub0, "sub2line": host.sub2line, "line_image": host.line_image,
                "cu_lines": host.cu_lines}

    def tokenize_images(self, images: Sequence[dict], auto_min_length: bool = True) -> LineBatch:
        """Tokenise many images in one `ltr_tokenize_batch` call -> device LineBatch (rows of all images
        concatenated; sub_off / cuk set whenever some key line is split into sublines).

        Per image a dict: 'klines' (cv2 KeyLine list or `change_cv2_T_np` dict), 'image_shape' (1,1,H,W),
        the SuperPoint outputs on this engine's device ('dense_descriptor' [1,256,H/8,W/8], 'dense_score'
        [1,H,W], ...) and optionally 'valid_mask'.  Filters and settings follow `Matching.forward`
        (auto_min_length: min_length and token_distance from each image's size)."""
        specs, cfgs = self._image_specs(images, auto_min_length)
        return self.tokenize_prepared(LP.prepare_tokenizer_batch(specs, cfgs), images)

    def tokenize_prepared(self, host: "LP.TokenizerBatch", images: Sequence[dict]) -> LineBatch:
        """`tokenize_images` for a batch already prepared on the host (`line_process.prepare_tokenizer_batch`,
        whose per-image settings may differ except for max_tokens); `images` supply the SuperPoint maps."""
        return self._tokenize(host, images, _ops.stage(self._tok_arrays(host), self.device))

    def match_images(self, images0: Sequence[dict], images1: Sequence[dict], line_thresh: Optional[float] = None,
                     point_thresh: float = 0.7, want_scores: bool = False, auto_min_length: bool = True) -> ImagePairMatches:
        """`Matching.forward` (models/matching.py:18-86) for P image pairs at once, from detector + SuperPoint
        outputs (image dicts as for `tokenize_images`, plus 'keypoints' [N,2] and 'descriptors' [256,N]):
        one `ltr_tokenize_batch` over the 2P images, one encode and one line `ltr_match` with key-line merging
        (`match_packed`), one point `ltr_match` over all pairs (mutual NN, threshold point_thresh).
        line_thresh defaults to the model's nn_threshold.  Host sizes come from the inputs' shapes: the call
        never waits for the device."""
        if len(images0) != len(images1):
            raise N.LtrError(f"match_images: {len(images0)} side-0 images but {len(images1)} side-1 images")
        if line_thresh is None:
            line_thresh = self.model.config.get("nn_threshold", 0.8)
        P = len(images0)
        images = list(images0) + list(images1)
        specs, cfgs = self._image_specs(images, auto_min_length)
        host = LP.prepare_tokenizer_batch(specs, cfgs)
        kp = [_first(im["keypoints"]) for im in images]
        dp = [_first(im["descriptors"]) for im in images]
        npts = np.array([int(d.shape[1]) for d in dp], dtype=np.int64)
        cup = np.zeros(2 * P + 1, dtype=np.int64)
        cup[1:] = np.cumsum(npts)
        i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)
        cu, cuk, so = host.cu_lines, host.cuk, host.sub0
        R0, K0 = int(cu[P]), int(cuk[P])
        arrays = self._tok_arrays(host)
        # everything match_packed and the point match upload, in the same staging buffer
        arrays.update(cu0=i32(cu[:P + 1]), cu1=i32(cu[P:] - R0), p_cu0=i32(cup[:P + 1]), p_cu1=i32(cup[P:] - cup[P]))
        if host.split:
            arrays.update(cuk0=i32(cuk[:P + 1]), cuk1=i32(cuk[P:] - K0), sub_off0=i32(so[:K0 + 1]), sub_off1=i32(so[K0:] - R0))
        dv = _ops.stage(arrays, self.device)
        batch = self._tokenize(host, images, dv)
        mx = lambda a: int(np.diff(a).max(initial=0))
        i32d = dict(dtype=torch.int32, device=self.device)
        f32d = dict(dtype=torch.float32, device=self.device)

        def unmatched(n_rows):   # a side without any line / point in the whole batch: nothing to match
            return (torch.full((n_rows,), -1, **i32d), torch.full((n_rows,), float("inf"), **f32d),
                    torch.zeros(P, **i32d), torch.empty(0, **f32d) if want_scores else None, 0)

        if K0 > 0 and int(cuk[-1]) > K0:
            lm = self._match_packed(batch, P, line_thresh, want_dist=want_scores, staged=dv)
            lines = (lm.matches0, lm.scores0, lm.counts, lm.dist, lm.stride)
        else:
            lines = unmatched(K0)
        N0 = int(cup[P])
        if N0 > 0 and int(cup[-1]) > N0:
            cat = lambda ds: torch.cat([d.float().contiguous().reshape(-1) for d in ds])   # [256, N_i] blocks back to back
            pm = _ops.match_descriptors(cat(dp[:P]), cat(dp[P:]), N.LAYOUT_CHANNEL_FIRST, P, float(point_thresh), True,
                                        cu0=dv["p_cu0"], cu1=dv["p_cu1"], max_n0=mx(cup[:P + 1]), max_n1=mx(cup[P:]),
                                        d=256, want_dist=want_scores)
            points = (pm["matches0"], pm["scores0"], pm["counts"], pm["dist_key"], pm["stride"])
        else:
            points = unmatched(N0)
        return ImagePairMatches(*lines[:3], i32(cuk[:P + 1]), *points[:3], i32(cup[:P + 1]),
                                host.klines[:P], host.klines[P:], kp[:P], kp[P:],
                                lines[3], lines[4], points[3], points[4])

    # ------------------------------------------------------------------ image sets: encode once, match many pairs
    def encode_images(self, images: Sequence[dict], auto_min_length: bool = True) -> ImageSet:
        """Encode each image once for later `match_sets` calls (image dicts as for `match_images`): one
        `ltr_tokenize_batch`, one `ltr_encode`, one `ltr_image_tiles` for the line descriptors and one for the
        SuperPoint point descriptors (concatenated channel-first into one pool).  All index arrays go up in one
        pinned copy; the call never waits for the device."""
        specs, cfgs = self._image_specs(images, auto_min_length)
        host = LP.prepare_tokenizer_batch(specs, cfgs)
        kp = [_first(im["keypoints"]) for im in images]
        dp = [_first(im["descriptors"]) for im in images]
        cup = np.zeros(len(images) + 1, dtype=np.int64)
        cup[1:] = np.cumsum([int(d.shape[1]) for d in dp])
        i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)
        cu, cup = i32(host.cu_lines), i32(cup)
        to_l, to_p = _ops.tile_offsets(cu), _ops.tile_offsets(cup)
        arrays = self._tok_arrays(host)
        arrays.update(cuk=i32(host.cuk), tile_off_l=to_l, cu_points=cup, tile_off_p=to_p)
        dv = _ops.stage(arrays, self.device)
        batch = self._tokenize(host, images, dv)
        rows = self.encode(batch)
        tiles_l = _ops.image_tiles(rows, N.LAYOUT_ROWS, cu, dv["cu_lines"], dv["tile_off_l"], int(to_l[-1]))
        pool = (torch.cat([d.float().contiguous().reshape(-1) for d in dp]) if dp
                else torch.empty(0, dtype=torch.float32, device=self.device))
        tiles_p = _ops.image_tiles(pool, N.LAYOUT_CHANNEL_FIRST, cup, dv["cu_points"], dv["tile_off_p"], int(to_p[-1]))
        dev = {k: dv[k] for k in ("cu_lines", "cuk", "tile_off_l", "cu_points", "tile_off_p")}
        dev["sub_off"] = dv["sub0"]
        return ImageSet(rows, tiles_l, pool, tiles_p, cu, i32(host.cuk), i32(host.sub0), to_l, cup, to_p, dev,
                        list(host.klines), kp, self.device)

    def match_set(self, images: ImageSet, pairs, **kw) -> ImagePairMatches:
        """`match_sets(images, images, pairs, ...)`: pairs of images of one set."""
        return self.match_sets(images, images, pairs, **kw)

    def match_sets(self, set0: ImageSet, set1: ImageSet, pairs, line_thresh: Optional[float] = None,
                   point_thresh: float = 0.7, want_scores: bool = False) -> ImagePairMatches:
        """Line and point matches of a list of image pairs between two encoded sets: pair p = (i, j) is image i of
        set0 against image j of set1 (pairs: host integer array [P, 2], validated before any device work).  The
        result equals `match_images` over the same pairs, images passed again per pair.  One indexed line match
        and one indexed point match per chunk of pairs (see `plan_chunks`; with key-line merging a chunk's subline
        distance scratch stays under DIST_SUB_CAP); the call never waits for the device."""
        pr = check_pairs(pairs, len(set0), len(set1))
        for s in (set0, set1):
            if s.device != self.device:
                raise N.LtrError(f"match_sets: image set on {s.device}, engine on {self.device}")
        if line_thresh is None:
            line_thresh = self.model.config.get("nn_threshold", 0.8)
        P = len(pr)
        i0, i1 = pr[:, 0], pr[:, 1]
        cnt = lambda a, i: np.diff(np.asarray(a, dtype=np.int64))[i]
        n0, n1 = cnt(set0.cu_lines, i0), cnt(set1.cu_lines, i1)      # sublines
        k0, k1 = cnt(set0.cuk, i0), cnt(set1.cuk, i1)                # key lines
        q0, q1 = cnt(set0.cu_points, i0), cnt(set1.cu_points, i1)    # keypoints
        # key-line merging exactly when match_images would merge these pairs: some image has a split key line
        merge = bool((n0 != k0).any() or (n1 != k1).any())
        pref = lambda c: np.concatenate([[0], np.cumsum(c)]).astype(np.int32)
        ol0, ol1, op0, op1 = pref(k0), pref(k1), pref(q0), pref(q1)
        dv = _ops.stage({"img0": pr[:, 0].copy(), "img1": pr[:, 1].copy(), "ol0": ol0, "ol1": ol1, "op0": op0,
                         "op1": op1}, self.device)
        i32d = dict(dtype=torch.int32, device=self.device)
        f32d = dict(dtype=torch.float32, device=self.device)
        alloc = lambda n, kw: torch.empty(max(int(n), 1), **kw)[:int(n)]   # never a null pointer
        mx = lambda a: int(a.max(initial=0))
        ml, sl, nl, cl = alloc(ol0[-1], i32d), alloc(ol0[-1], f32d), alloc(ol1[-1], i32d), alloc(P, i32d)
        mp, spp, npp, cp = alloc(op0[-1], i32d), alloc(op0[-1], f32d), alloc(op1[-1], i32d), alloc(P, i32d)
        stride_l = mx(k0) * mx(k1) if want_scores else 0
        stride_p = mx(q0) * mx(q1) if want_scores else 0
        dist_l = alloc(P * stride_l, f32d) if want_scores else None
        dist_p = alloc(P * stride_p, f32d) if want_scores else None
        zero = np.zeros(P, dtype=np.int64)
        for a, b in plan_chunks(n0 if merge else zero, n1 if merge else zero):
            def pools(cu, tiles, tile_off):   # the two image pools (lines or points) and this chunk's pairs
                return dict(cu0=set0.dev[cu], cu1=set1.dev[cu], tiles0=getattr(set0, tiles), tiles1=getattr(set1, tiles),
                            tile_off0=set0.dev[tile_off], tile_off1=set1.dev[tile_off],
                            n_tiles0=int(getattr(set0, tile_off)[-1]), n_tiles1=int(getattr(set1, tile_off)[-1]),
                            img0=dv["img0"][a:b], img1=dv["img1"][a:b])
            kw = pools("cu_lines", "tiles_l", "tile_off_l")
            kw.update(max_n0=mx(n0[a:b]), max_n1=mx(n1[a:b]), out_off0=dv["ol0"][a:b + 1], out_off1=dv["ol1"][a:b + 1],
                      total_out0=int(ol0[-1]), total_out1=int(ol1[-1]), matches0=ml, scores0=sl, nn1=nl, counts=cl[a:b])
            if want_scores:
                kw.update(dist_key=dist_l[a * stride_l:], dist_stride=stride_l)
            if merge:
                kw.update(sub_off0=set0.dev["sub_off"], sub_off1=set1.dev["sub_off"], cuk0=set0.dev["cuk"],
                          cuk1=set1.dev["cuk"], max_k0=mx(k0[a:b]), max_k1=mx(k1[a:b]))
            _ops.match_indexed(set0.desc_l, set1.desc_l, N.LAYOUT_ROWS, b - a, float(line_thresh), **kw)
            kw = pools("cu_points", "tiles_p", "tile_off_p")
            kw.update(max_n0=mx(q0[a:b]), max_n1=mx(q1[a:b]), out_off0=dv["op0"][a:b + 1], out_off1=dv["op1"][a:b + 1],
                      total_out0=int(op0[-1]), total_out1=int(op1[-1]), matches0=mp, scores0=spp, nn1=npp, counts=cp[a:b])
            if want_scores:
                kw.update(dist_key=dist_p[a * stride_p:], dist_stride=stride_p)
            _ops.match_indexed(set0.desc_p, set1.desc_p, N.LAYOUT_CHANNEL_FIRST, b - a, float(point_thresh), **kw)
        return ImagePairMatches(ml, sl, cl, ol0, mp, spp, cp, op0,
                                [set0.klines[i] for i in i0], [set1.klines[j] for j in i1],
                                [set0.keypoints[i] for i in i0], [set1.keypoints[j] for j in i1],
                                dist_l, stride_l, dist_p, stride_p)

    def match_packed_host(self, host: LineBatch, n_pairs: int, nn_thresh: Optional[float] = None, mutual=True,
                          n_chunks: int = 4):
        """End-to-end entry for HOST (ideally pinned) inputs: the packed batch is cut into
        `n_chunks` groups of pairs; the H2D copy of group i+1 runs on a side stream while group i
        is encoded and matched, so the PCIe transfer (the e2e bound: ~5.6 MB of fp32 inputs per
        pair) overlaps the kernels.  Returns (matches0 int32 [total key lines side 0], counts
        int32 [n_pairs], offsets0) with matches0/counts still on the device.  Batches with key-line
        structure (sub_off / cuk) are cut along the same pair boundaries."""
        P = int(n_pairs)
        if host.n_images != 2 * P:
            raise ValueError("match_packed_host: batch must hold 2 * n_pairs images")
        n_chunks = max(1, min(int(n_chunks), P))
        if not hasattr(self, "_copy_stream"):
            self._copy_stream = torch.cuda.Stream(device=self.device)
        main = torch.cuda.current_stream(self.device)
        cu = host.cu_lines
        seg = host.sub_off is not None
        outs, cnts = [], []
        for c in range(n_chunks):
            p0, p1 = shard_range(P, c, n_chunks)
            a0, a1, b0, b1 = int(cu[p0]), int(cu[p1]), int(cu[P + p0]), int(cu[P + p1])
            n0, n1 = a1 - a0, b1 - b0
            with torch.cuda.stream(self._copy_stream):
                dev_t = []
                for t in host.tensors():
                    d = torch.empty((n0 + n1,) + tuple(t.shape[1:]), dtype=t.dtype, device=self.device)
                    d[:n0].copy_(t[a0:a1], non_blocking=True)
                    d[n0:].copy_(t[b0:b1], non_blocking=True)
                    dev_t.append(d)
                ready = torch.cuda.Event()
                ready.record(self._copy_stream)
            main.wait_event(ready)
            cu_c = np.concatenate([cu[p0:p1 + 1] - a0, cu[P + p0 + 1:P + p1 + 1] - b0 + n0]).astype(np.int32)
            sub_c = cuk_c = None
            if seg:   # key lines of the chunk's images, sublines renumbered to the chunk ([side 0 | side 1])
                ck, so = host.cuk, host.sub_off
                k0a, k0b, k1a, k1b = int(ck[p0]), int(ck[p1]), int(ck[P + p0]), int(ck[P + p1])
                cuk_c = np.concatenate([ck[p0:p1 + 1] - k0a, ck[P + p0 + 1:P + p1 + 1] - k1a + (k0b - k0a)]).astype(np.int32)
                sub_c = np.concatenate([so[k0a:k0b] - a0, so[k1a:k1b + 1] - b0 + n0]).astype(np.int32)
            chunk = LineBatch(*dev_t, cu_c, sub_c, cuk_c)
            res = self.match_packed(chunk, p1 - p0, nn_thresh, mutual)
            for d in dev_t:
                d.record_stream(main)
            outs.append(res.matches0)
            cnts.append(res.counts)
        return torch.cat(outs), torch.cat(cnts), (host.cuk if seg else cu)[:P + 1]


# ------------------------------------------------------------------------------- multi-GPU
def shard_range(n_items: int, rank: int, world: int):
    """Contiguous block of items owned by `rank` (sizes differ by at most one)."""
    base, rem = divmod(n_items, world)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def gather_counts(local_counts: torch.Tensor, n_total: int, group=None, async_op: bool = False):
    """The path's one collective: all-gather of per-pair match counts (int32) so that every
    rank knows the global result size.  Works with NCCL (CUDA tensors) and gloo (CPU).
    Equal shards (the usual case) take the single-kernel `all_gather_into_tensor` path; ragged
    shards are padded to the widest one.

    async_op=True (equal CUDA shards only) returns (tensor, work): the collective runs on NCCL's
    stream behind the matcher and the caller's stream is NOT made to wait for it, so the next
    batch's kernels overlap the gather; call work.wait() before reading the tensor."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return (local_counts.clone(), None) if async_op else local_counts.clone()
    world = dist.get_world_size(group)
    sizes = [shard_range(n_total, r, world) for r in range(world)]
    width = max(e - s for s, e in sizes)
    equal = all(e - s == width for s, e in sizes) and local_counts.numel() == width
    if equal and local_counts.is_cuda:
        out = torch.empty(width * world, dtype=local_counts.dtype, device=local_counts.device)   # no kernel
        work = dist.all_gather_into_tensor(out, local_counts.contiguous(), group=group, async_op=async_op)
        return (out, work) if async_op else out
    if async_op:
        raise ValueError("gather_counts(async_op=True) needs equal CUDA shards")
    buf = torch.zeros(width, dtype=local_counts.dtype, device=local_counts.device)
    buf[:local_counts.numel()] = local_counts
    gathered = [torch.empty_like(buf) for _ in range(world)]
    dist.all_gather(gathered, buf, group=group)
    return torch.cat([g[:e - s] for g, (s, e) in zip(gathered, sizes)])


class PeerCounts:
    """The path's one collective without a collective kernel: a symmetric int32 buffer (peer-mapped over
    NVLink with torch.distributed._symmetric_memory) into which the matcher's tail kernel of every rank
    stores its per-pair match counts for ALL ranks - `multimem.st` through the NVSwitch multicast address
    when the allocation supports it, plain peer stores otherwise (include/linetr_b200.h: LtrPeerGather).

        pc = PeerCounts(n_pairs_per_rank)                            # collective: allocation + rendezvous
        res = eng.match_packed(batch, P, 0.8, gather=pc.publish())   # counts published by the tail kernel
        ...                                                          # (at most GATHER_SLOTS - 2 publishes in flight)
        all_counts = pc.collect()                                    # [world * n_pairs] of the OLDEST uncollected publish
    """

    def __init__(self, n_pairs: int, group=None, device=None, multicast=True):
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm_mem
        if not (dist.is_available() and dist.is_initialized()):
            raise N.LtrError("PeerCounts needs an initialised torch.distributed process group (NCCL)")
        group = group if group is not None else dist.group.WORLD
        self.world, self.rank, self.n_pairs = dist.get_world_size(group), dist.get_rank(group), int(n_pairs)
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        n = N.GATHER_SLOTS * self.world * (self.n_pairs + 1)
        self.buf = symm_mem.empty(n, dtype=torch.int32, device=self.device)
        self.buf.zero_()
        self.hdl = symm_mem.rendezvous(self.buf, group)
        torch.cuda.synchronize(self.device)
        dist.barrier(group)                      # every rank's flags are zero before anybody publishes
        mc = 0
        try:
            if multicast and self.hdl.has_multicast_support:
                mc = int(self.hdl.multicast_ptr)
        except Exception:
            mc = 0
        self.multicast = mc != 0
        self._mc = mc
        self._peers = int(self.hdl.buffer_ptrs_dev)
        self._published = 0
        self._collected = 0

    def publish(self) -> "N.LtrPeerGather":
        """Descriptor for the next ltr_match call (pass as `gather=`)."""
        if self._published - self._collected >= N.GATHER_SLOTS - 2:
            raise N.LtrError("PeerCounts: collect() earlier publishes first (at most GATHER_SLOTS - 2 in flight)")
        e = self._published
        self._published += 1
        return N.LtrPeerGather(self._mc or None, self._peers, self.rank, self.world, e % N.GATHER_SLOTS, e // N.GATHER_SLOTS + 1)

    def collect(self) -> torch.Tensor:
        """Device-side consumer: counts of all ranks for the oldest publish not collected yet, int32 CUDA tensor
        [world * n_pairs]; enqueues one tiny kernel on the current stream that waits for the world's flags
        (no host synchronisation).  Note that it couples the compute stream to the slowest rank; throughput
        loops should prefer collect_async(), which involves no kernel at all."""
        if self._collected >= self._published:
            raise N.LtrError("PeerCounts.collect(): nothing published")
        e = self._collected
        self._collected += 1
        out = torch.empty(self.world * self.n_pairs, dtype=torch.int32, device=self.device)
        _ops._call("ltr_gather_wait", self.device, C.c_void_p(self.buf.data_ptr()), self.world, self.n_pairs,
                   e % N.GATHER_SLOTS, e // N.GATHER_SLOTS + 1, C.c_void_p(out.data_ptr()))
        return out

    def collect_async(self) -> "PeerCountsHandle":
        """Host-side consumer without any kernel: a copy-engine D2H of the oldest uncollected slot (counts + flags)
        on a side stream, ordered behind everything enqueued on the current stream so far (this rank's own publish).
        `handle.result()` synchronises that copy only, and re-polls in the (rare) case that a peer's flag had not
        arrived yet - the compute stream never waits for another rank."""
        if self._collected >= self._published:
            raise N.LtrError("PeerCounts.collect_async(): nothing published")
        e = self._collected
        self._collected += 1
        if not hasattr(self, "_side"):
            self._side = torch.cuda.Stream(device=self.device)
        h = PeerCountsHandle(self, e % N.GATHER_SLOTS, e // N.GATHER_SLOTS + 1)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))
        self._side.wait_event(ev)
        h._enqueue()
        return h


class PeerCountsHandle:
    def __init__(self, pc: "PeerCounts", slot: int, epoch: int):
        self.pc, self.slot, self.epoch = pc, slot, epoch
        W, P = pc.world, pc.n_pairs
        self._counts = pc.buf[slot * W * P:(slot + 1) * W * P]
        f0 = N.GATHER_SLOTS * W * P + slot * W
        self._flags = pc.buf[f0:f0 + W]
        self._host = torch.empty(W * P + W, dtype=torch.int32).pin_memory()
        self._done = torch.cuda.Event()

    def _enqueue(self):
        W, P = self.pc.world, self.pc.n_pairs
        with torch.cuda.stream(self.pc._side):
            self._host[W * P:].copy_(self._flags, non_blocking=True)   # flags FIRST: a flag that is set implies its counts are
            self._host[:W * P].copy_(self._counts, non_blocking=True)  # (the publisher fences between the two)
            self._done.record(self.pc._side)

    def wait(self):
        self.result()

    def result(self, timeout_s: float = 30.0) -> torch.Tensor:
        """-> int32 CPU tensor [world * n_pairs]."""
        import time
        W, P = self.pc.world, self.pc.n_pairs
        t0 = time.perf_counter()
        while True:
            self._done.synchronize()
            if bool((self._host[W * P:] >= self.epoch).all()):
                return self._host[:W * P]
            if time.perf_counter() - t0 > timeout_s:
                raise N.LtrError("PeerCounts: a peer did not publish within the timeout")
            self._enqueue()
