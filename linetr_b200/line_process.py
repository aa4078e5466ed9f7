"""`get_dist_matrix` (CUDA) and the line tokeniser that feeds the hot path.

`get_dist_matrix` is on the hot path (reference models/line_process.py:198-201) and runs on
the GPU through `ltr_match`.  The tokeniser (reference models/line_process.py:6-196; SURVEY.md
§8f row 1, the first "next" row) exists twice: `line_tokenizer_gpu` (CUDA, `ltr_tokenize_batch`; used by
`LineTransformer.preprocess` whenever the SuperPoint outputs live on a CUDA device) and
`line_tokenizer`, numpy/PyTorch glue that reproduces the reference bit for bit - including its
quirks (in-place end-point clipping, `index[:max_keylines]` dropping the shortest line when
max_keylines == -1, the torch-version dependent `align_corners`) - and is the pin the GPU
tokeniser is tested against.  The cheap per-image filters (`remove_borders`,
`filter_by_length`, cv2 KeyLine conversion) stay vectorised numpy.

One deliberate difference: the reference squares the slope and the token distance as scalars
(`m ** 2`, `dist_px ** 2`), which numpy and Python evaluate with libm's pow.  pow is not correctly
rounded (glibc's differs from m * m for about 1 in 1200 random slopes), so its result depends on the
platform.  The glue squares with one correctly rounded product (m * m, d * d), which the GPU
reproduces exactly; a token differs from the reference only where pow's last bit differs and that
bit moves the fp32 rounding of the position.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List, Tuple

import numpy as np
import torch


# --------------------------------------------------------------------------- hot path
def get_dist_matrix(desc0, desc1):
    """(2 - 2 * desc0^T desc1).clip(0) per batch element; numpy [B,d,n],[B,d,m] -> [B,n,m] float32."""
    from . import _ops, _native as N
    desc0 = np.ascontiguousarray(desc0, dtype=np.float32)
    desc1 = np.ascontiguousarray(desc1, dtype=np.float32)
    B, d, n = desc0.shape
    m = desc1.shape[2]
    if B == 0 or n == 0 or m == 0:
        return np.zeros((B, n, m), dtype=np.float32)
    dev = _ops.current_cuda_device()
    a = torch.from_numpy(desc0).to(dev, non_blocking=True)
    b = torch.from_numpy(desc1).to(dev, non_blocking=True)
    out = _ops.match_descriptors(a, b, N.LAYOUT_CHANNEL_FIRST, B, 0.0, False, n0=n, n1=m, d=d, want_matches=False)
    return out["dist_key"].view(B, n, m).cpu().numpy()


# --------------------------------------------------------------------------- tokeniser glue
def keyline_geometry(kl, length, token_distance, max_tokens, width, height):
    """Per-key-line geometry of the tokeniser (reference line_tokenizer, models/line_process.py:100-196),
    vectorised over the key lines of one image or of many images concatenated.  `kl` [K,2,2] float64
    has its end points clipped IN PLACE to (width-0.6, height-0.6), as the reference does; token_distance,
    width and height are scalars or per-key-line arrays.  -> dict of n_tok, n_sub [K] int64, sub0 [K+1]
    (first subline of every key line, the key-line CSR), sub2line [S], and the float64 start point sp,
    end point ep (before the clip) and epc (after it), each [K,2].

    Key lines must have finite, non-negative coordinates (`remove_borders` keeps only such lines) and run left
    to right (start x <= end x), as `change_cv2_T_np` orders them: tokens step from the start in +x, so on a
    reversed line they would move away from it, and a token left of or above the image would look up a score
    before the start of the map (the reference wraps the negative index).  Any other line raises LtrError."""
    from . import _native as N
    T = int(max_tokens)
    K = len(kl)
    ends = lambda i: f"(start {tuple(kl[i, 0].tolist())}, end {tuple(kl[i, 1].tolist())})"
    for bad, why in ((~np.isfinite(kl).all(axis=(1, 2)), "has a non-finite coordinate"),
                     ((kl < 0).any(axis=(1, 2)), "has a negative coordinate: key lines must lie in the image"),
                     (kl[:, 0, 0] > kl[:, 1, 0], "runs right to left: key lines must have start x <= end x")):
        if bad.any():
            i = int(np.flatnonzero(bad)[0])
            raise N.LtrError(f"key line {i} {why} {ends(i)}")
    length = np.asarray(length, dtype=np.float64)
    n_tok = np.ceil(length / token_distance).astype(np.int64)
    n_sub = -(-n_tok // T)
    geo = np.sqrt(((kl[:, 1] - kl[:, 0]) ** 2).sum(axis=1))
    assert bool((geo >= np.maximum(n_tok - 2, 0) * token_distance).all()), "distance should be smaller than line length!"
    sp = np.ascontiguousarray(kl[:, 0], dtype=np.float64)
    ep = np.ascontiguousarray(kl[:, 1], dtype=np.float64).copy()
    kl[:, 1, 0] = np.minimum(kl[:, 1, 0], np.asarray(width) - 0.6)      # in place, like the reference
    kl[:, 1, 1] = np.minimum(kl[:, 1, 1], np.asarray(height) - 0.6)
    epc = np.ascontiguousarray(kl[:, 1], dtype=np.float64)
    sub0 = np.zeros(K + 1, dtype=np.int64)
    sub0[1:] = np.cumsum(n_sub)
    sub2line = np.repeat(np.arange(K), n_sub)
    return {"n_tok": n_tok, "n_sub": n_sub, "sub0": sub0, "sub2line": sub2line, "sp": sp, "ep": ep, "epc": epc}


def tokenizer_config(config, image_shape, auto_min_length=True):
    """The tokeniser settings `Matching.forward` uses for an image of shape (1,1,H,W) (models/matching.py:29-32):
    with auto_min_length, min_length and token_distance follow the image size."""
    cfg = {k: config[k] for k in ("min_length", "token_distance", "max_tokens", "remove_borders", "max_keylines")}
    if auto_min_length:
        cfg["min_length"] = max(16, max(image_shape) / 40)
        cfg["token_distance"] = max(8, max(image_shape) / 80)
    return cfg


def filter_keylines(klines, image_shape, cfg, valid_mask=None):
    """`LineTransformer.preprocess` up to the tokeniser: cv2 KeyLine list (or a `change_cv2_T_np` dict, which is
    copied, not modified) -> the kept key lines.  valid_mask None means all valid; it is honoured only as a
    numpy array, like the reference."""
    if isinstance(klines, dict):
        klines = {k: np.array(v, copy=True) for k, v in klines.items()}
    else:
        klines = change_cv2_T_np(klines)
    height, width = int(image_shape[-2]), int(image_shape[-1])
    if valid_mask is None:
        valid_mask = np.ones((height, width))
    klines = remove_borders(klines, cfg["remove_borders"], height, width, valid_mask)
    klines = filter_by_length(klines, cfg["min_length"], cfg["max_keylines"])
    klines["klines"] = np.asarray(klines["klines"], dtype=np.float64).reshape(-1, 2, 2)
    klines["length_klines"] = np.asarray(klines["length_klines"], dtype=np.float64).reshape(-1)
    klines["angles"] = np.asarray(klines["angles"], dtype=np.float64).reshape(-1, 2)
    return klines


@dataclass
class TokenizerBatch:
    """Host side of one `ltr_tokenize_batch` call: the key lines of many images concatenated image by image.

    Per key line: sp, ep, epc [K,2] float64, length [K] float64, angle [K,2] float32, n_tok, line_image [K]
    int32; sub0 int32 [K+1] (global subline numbering: the key-line CSR of the packed LineBatch),
    sub2line int32 [S]; per image: cu_lines int32 [n+1] (subline offsets), cuk int32 [n+1] (key-line
    offsets), token_distance float64 [n], shapes (H, W), and its kept key lines after the in-place clip
    (klines, views into one [K,2,2] array) with their length_klines and angles."""
    sp: np.ndarray
    ep: np.ndarray
    epc: np.ndarray
    length: np.ndarray
    angle: np.ndarray
    n_tok: np.ndarray
    line_image: np.ndarray
    sub0: np.ndarray
    sub2line: np.ndarray
    cu_lines: np.ndarray
    cuk: np.ndarray
    token_distance: np.ndarray
    shapes: List[Tuple[int, int]]
    max_tokens: int
    klines: List[np.ndarray]
    length_klines: List[np.ndarray]
    angles: List[np.ndarray]

    @property
    def n_images(self) -> int:
        return len(self.shapes)

    @property
    def n_keylines(self) -> int:
        return int(self.cuk[-1])

    @property
    def n_sublines(self) -> int:
        return int(self.cu_lines[-1])

    @property
    def split(self) -> bool:
        """True when some key line is cut into several sublines (key-line merging is needed)."""
        return self.n_sublines != self.n_keylines


def prepare_tokenizer_batch(images, configs) -> TokenizerBatch:
    """images: per image (klines, image_shape (1,1,H,W), valid_mask or None), klines a cv2 KeyLine list or a
    `change_cv2_T_np` dict; configs: per-image tokeniser settings (`tokenizer_config`).  Every image must use
    the same max_tokens (one token-slot count per batch)."""
    from . import _native as N
    if len(images) != len(configs):
        raise N.LtrError("prepare_tokenizer_batch: one config per image required")
    Ts = {int(c["max_tokens"]) for c in configs}
    if len(Ts) > 1:
        raise N.LtrError(f"prepare_tokenizer_batch: all images of a batch need the same max_tokens, got {sorted(Ts)}")
    T = Ts.pop() if Ts else 21
    kept = [filter_keylines(kl, shape, cfg, vm) for (kl, shape, vm), cfg in zip(images, configs)]
    counts = np.array([len(k["klines"]) for k in kept], dtype=np.int64)
    n = len(kept)
    shapes = [(int(shape[-2]), int(shape[-1])) for _, shape, _ in images]
    td = np.array([float(c["token_distance"]) for c in configs], dtype=np.float64)
    cat = lambda key, shp, dt: (np.concatenate([k[key] for k in kept]).astype(dt, copy=False) if n
                                else np.zeros(shp, dtype=dt))
    kl = np.ascontiguousarray(cat("klines", (0, 2, 2), np.float64))
    length = np.ascontiguousarray(cat("length_klines", (0,), np.float64))
    angle = np.ascontiguousarray(cat("angles", (0, 2), np.float32))
    line_image = np.repeat(np.arange(n), counts)
    H = np.array([h for h, _ in shapes], dtype=np.int64)[line_image]
    W = np.array([w for _, w in shapes], dtype=np.int64)[line_image]
    g = keyline_geometry(kl, length, td[line_image], T, W, H)
    cuk = np.zeros(n + 1, dtype=np.int64)
    cuk[1:] = np.cumsum(counts)
    bounds = list(zip(cuk[:-1], cuk[1:]))
    i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)
    return TokenizerBatch(g["sp"], g["ep"], g["epc"], length, angle, i32(g["n_tok"]), i32(line_image), i32(g["sub0"]),
                          i32(g["sub2line"]), i32(g["sub0"][cuk]), i32(cuk), td, shapes, T,
                          [kl[a:b] for a, b in bounds], [length[a:b] for a, b in bounds],
                          [angle[a:b] for a, b in bounds])


def get_angles(lines):
    """Orientation code (cos 2a, sin 2a) with a = atan2(dx, dy) folded into [0, pi)."""
    if len(lines) == 0:
        return []
    delta = lines[:, 1] - lines[:, 0]
    ang = np.arctan2(delta[:, 0], delta[:, 1])
    ang = np.where(ang < 0, ang + np.pi, ang)
    return np.stack([np.cos(2 * ang), np.sin(2 * ang)], axis=1)


def change_cv2_T_np(klines_cv):
    """cv2 KeyLine list -> {'klines' [n,2,2] (left end point first), 'length_klines', 'angles'}."""
    n = len(klines_cv)
    pts = np.zeros((n, 2, 2), dtype=np.float64)
    length = np.zeros((n,), dtype=np.float64)
    for i, ln in enumerate(klines_cv):
        a = (ln.startPointX, ln.startPointY)
        b = (ln.endPointX, ln.endPointY)
        pts[i] = (a, b) if a[0] < b[0] else (b, a)
        length[i] = ln.lineLength * (2 ** ln.octave)
    return {"klines": pts, "length_klines": length, "angles": get_angles(pts)}


def remove_borders(lines, border: int, height: int, width: int, valid_mask_given=None):
    k = lines["klines"]
    inside = np.ones(len(k), dtype=bool)
    for e in (0, 1):
        inside &= (k[:, e, 0] >= border) & (k[:, e, 0] < (width - border))
        inside &= (k[:, e, 1] >= border) & (k[:, e, 1] < (height - border))
    eps = 0.001
    k[:, :, 0] = k[:, :, 0].clip(max=width - eps - border)
    k[:, :, 1] = k[:, :, 1].clip(max=height - eps - border)
    if isinstance(valid_mask_given, np.ndarray):
        a = np.floor(k[:, 0]).astype(int)
        b = np.floor(k[:, 1]).astype(int)
        inside &= (valid_mask_given[a[:, 1], a[:, 0]] + valid_mask_given[b[:, 1], b[:, 0]]).astype(bool)
    return {key: np.asarray(v)[inside] for key, v in lines.items()}


def filter_by_length(lines, min_length, max_sublines):
    keep = lines["length_klines"] > min_length
    k, ln = lines["klines"][keep], lines["length_klines"][keep]
    order = np.argsort(ln)[::-1][:max_sublines]   # NB: max_sublines == -1 drops the shortest line
    k, ln = k[order], ln[order]
    return {"klines": k, "length_klines": ln, "angles": get_angles(k)}


def _tokens_on_line(kline, n_tokens, token_distance, width, height):
    """n_tokens-1 points every token_distance px from the start, then the (clipped, in place) end."""
    sp, ep = kline[0], kline[1]
    seg_len = math.sqrt(float(((ep - sp) ** 2).sum()))
    dists = np.arange(n_tokens - 1, dtype=np.float64) * token_distance
    assert n_tokens <= 1 or seg_len >= dists[-1], "distance should be smaller than line length!"
    vec = ep - sp
    if vec[0] != 0:
        m = vec[1] / vec[0]
        dx = np.sqrt(dists * dists / (1 + m * m))   # correctly rounded squares, not pow (module docstring)
        dy = m * dx
    else:
        dx = np.zeros_like(dists)
        dy = dists if vec[1] > 0 else -dists
    pts = np.stack([dx, dy], axis=1) + sp
    ep[0] = min(ep[0], width - 0.6)      # in place: the stored key line end point is clipped too
    ep[1] = min(ep[1], height - 0.6)
    return np.concatenate([pts, ep[None]], axis=0)


def sample_descriptors(keypoints, descriptors, s: int = 8):
    """Bilinear sampling of the dense descriptor map at pixel positions, L2-normalised."""
    b, c, h, w = descriptors.shape
    kp = keypoints - s / 2 + 0.5
    kp = kp / torch.tensor([(w * s - s / 2 - 0.5), (h * s - s / 2 - 0.5)]).to(kp)[None]
    kp = kp * 2 - 1
    # the reference keys align_corners on the third character of torch.__version__
    kwargs = {"align_corners": True} if int(torch.__version__[2]) > 2 else {}
    out = torch.nn.functional.grid_sample(descriptors, kp.view(b, 1, -1, 2), mode="bilinear", **kwargs)
    return torch.nn.functional.normalize(out.reshape(b, c, -1), p=2, dim=1)


def line_tokenizer(klines, token_distance, max_tokens, pred_superpoint, image_shape):
    """Key lines -> sublines/tokens/masks/descriptors dict consumed by LineTransformer.forward."""
    height, width = image_shape
    K = len(klines["klines"])
    sub_l, tok_l, mask_l, resp_l, ang_l, nsub = [], [], [], [], [], []
    max_len = token_distance * max_tokens
    for i in range(K):
        kline = klines["klines"][i]
        n_tok = int(math.ceil(klines["length_klines"][i] / token_distance))
        toks = _tokens_on_line(kline, n_tok, token_distance, width, height)
        n_sub = int(math.ceil(n_tok / max_tokens))
        subs = np.zeros((n_sub, 2, 2))
        subs[0, 0] = kline[0]
        subs[-1, 1] = kline[1]
        for j in range(n_sub - 1):
            cut = toks[(j + 1) * max_tokens - 1]
            subs[j, 1] = cut
            subs[j + 1, 0] = cut
        t = np.zeros((n_sub, max_tokens, 2))
        m = np.zeros((n_sub, max_tokens + 1, 1))
        m[:, 0] = 1
        for j in range(n_sub):
            part = toks[j * max_tokens:(j + 1) * max_tokens]
            t[j, :len(part)] = part
            m[j, 1:len(part) + 1] = 1
        sub_l.append(subs)
        tok_l.append(t)
        mask_l.append(m)
        resp_l.append(np.sqrt(((subs[:, 1] - subs[:, 0]) ** 2).sum(axis=1, keepdims=True)) / max_len)
        ang_l.append(np.repeat(np.asarray(klines["angles"][i])[None], n_sub, axis=0))
        nsub.append(n_sub)
    device = pred_superpoint["dense_descriptor"].device
    f = lambda arrs, shape: torch.from_numpy(np.concatenate(arrs, axis=0).reshape(shape)).float().to(device)
    slines = f(sub_l, (-1, 2, 2))
    tokens = f(tok_l, (-1, max_tokens, 2))
    masks = f(mask_l, (-1, max_tokens + 1, 1))
    responses = f(resp_l, (-1, 1))
    angles = f(ang_l, (-1, 2))
    S = slines.shape[0]
    adj = torch.zeros((K, S)).to(device)
    st = 0
    for i, n in enumerate(nsub):
        adj[i, st:st + n] = 1 / n
        st += n
    dense = pred_superpoint["dense_descriptor"]
    desc = sample_descriptors(tokens[None], dense, 8)[0].reshape(256, S, max_tokens).permute(1, 2, 0)
    score_map = pred_superpoint["dense_score"].transpose(1, 2)
    pos = torch.round(tokens).long().reshape(-1, 2)
    pos[:, 0] = pos[:, 0].clip(max=score_map.shape[1] - 1)
    pos[:, 1] = pos[:, 1].clip(max=score_map.shape[2] - 1)
    scores = score_map[0][pos[:, 0], pos[:, 1]].reshape(S, max_tokens, 1)

    klines["klines"] = torch.from_numpy(klines["klines"]).float().to(device)[None]
    klines["length_klines"] = torch.from_numpy(klines["length_klines"]).float().to(device)[None]
    klines["angles"] = torch.from_numpy(np.asarray(klines["angles"])).float().to(device)[None]
    klines["sublines"] = slines[None]
    klines["pnt_sublines"] = tokens[None]
    klines["mask_sublines"] = masks[None]
    klines["resp_sublines"] = responses[None]
    klines["angle_sublines"] = angles[None]
    klines["desc_sublines"] = desc[None]
    klines["score_sublines"] = scores[None]
    klines["mat_klines2sublines"] = adj[None]
    return klines


def line_tokenizer_gpu(klines, token_distance, max_tokens, pred_superpoint, image_shape):
    """`line_tokenizer` on the GPU (`ltr_tokenize_batch` with one image): same inputs, same output dict, no Python
    loops.  Token positions, sublines, masks, responses, scores and the adjacency are bit-identical to the CPU
    version (float64 arithmetic in numpy's operation order, rounded once to fp32); sampled descriptors agree to fp32
    rounding.  Key lines must lie in the image and run left to right (see `keyline_geometry`), and max_tokens must
    be 1..128 (the encoder's limit)."""
    from . import _native as N, _ops
    dense = pred_superpoint["dense_descriptor"]
    if not dense.is_cuda:
        raise N.LtrError("line_tokenizer_gpu needs the SuperPoint outputs on a CUDA device")
    dev = dense.device
    height, width = image_shape
    K = len(klines["klines"])
    length = np.ascontiguousarray(klines["length_klines"], dtype=np.float64)
    g = keyline_geometry(klines["klines"], length, token_distance, max_tokens, width, height)
    n_sub, sub2line = g["n_sub"], g["sub2line"]
    S = int(g["sub0"][-1])
    i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)   # noqa: E731
    dv = _ops.stage({"sp": g["sp"], "ep": g["ep"], "epc": g["epc"], "length": length,
                     "angle": np.ascontiguousarray(klines["angles"], dtype=np.float32).reshape(K, 2),
                     "n_tok": i32(g["n_tok"]), "sub0": i32(g["sub0"]), "sub2line": i32(sub2line),
                     "line_image": np.zeros(K, dtype=np.int32)}, dev)
    maps = [(dense, pred_superpoint["dense_score"], token_distance)]
    slines, tokens, masks, responses, ang, desc, scores = _ops.tokenize(dv, maps, np.array([0, S]), max_tokens, dev)
    adj = np.zeros((K, S), dtype=np.float32)
    w = (1.0 / n_sub).astype(np.float64)
    adj[sub2line, np.arange(S)] = w[sub2line]
    klines["klines"] = torch.from_numpy(klines["klines"]).float().to(dev)[None]
    klines["length_klines"] = torch.from_numpy(klines["length_klines"]).float().to(dev)[None]
    klines["angles"] = torch.from_numpy(np.asarray(klines["angles"])).float().to(dev)[None]
    klines["sublines"] = slines[None]
    klines["pnt_sublines"] = tokens[None]
    klines["mask_sublines"] = masks[None]
    klines["resp_sublines"] = responses[None]
    klines["angle_sublines"] = ang[None]
    klines["desc_sublines"] = desc[None]
    klines["score_sublines"] = scores[None]
    klines["mat_klines2sublines"] = torch.from_numpy(adj).to(dev)[None]
    return klines
