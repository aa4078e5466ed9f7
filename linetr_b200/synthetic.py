"""Seeded synthetic weights and inputs for the LineTR hot path (numpy only).

Everything here is regenerable from an integer seed on any machine, so the GPU box
(which has no copy of the reference checkout or its checkpoint) can rebuild exactly
the weights and inputs the committed golden fixtures were produced with.

Shapes/keys follow the reference checkpoint contract (SURVEY.md §8a "State-dict
contract"; reference models/line_transformer.py:93-105,139-162,203-217 and
models/line_attention.py:23-40,77-84).  Input distributions follow SURVEY.md §8(d).
"""
from __future__ import annotations

import numpy as np

D_MODEL = 256
N_HEADS = 4
D_INNER = 1024
MLP_HIDDEN = (32, 64, 128, 256)
N_SIG_LAYERS = 7


def state_dict_spec(n_desc_layers: int = 1, d_model: int = D_MODEL, d_inner: int = D_INNER):
    """[(key, shape, kind)] in the reference checkpoint's key order.

    kind in {'w','b','bn_w','bn_b','bn_mean','bn_var','bn_count','ln_w','ln_b','cls'}.
    """
    spec = [("klenc.cls_token", (1, 1, 1, d_model), "cls")]

    def mlp(prefix, chans):
        idx = 0
        for i in range(1, len(chans)):
            spec.append((f"{prefix}.{idx}.weight", (chans[i], chans[i - 1], 1), "w"))
            spec.append((f"{prefix}.{idx}.bias", (chans[i],), "b"))
            idx += 1
            if i < len(chans) - 1:
                c = chans[i]
                spec.append((f"{prefix}.{idx}.weight", (c,), "bn_w"))
                spec.append((f"{prefix}.{idx}.bias", (c,), "bn_b"))
                spec.append((f"{prefix}.{idx}.running_mean", (c,), "bn_mean"))
                spec.append((f"{prefix}.{idx}.running_var", (c,), "bn_var"))
                spec.append((f"{prefix}.{idx}.num_batches_tracked", (), "bn_count"))
                idx += 2  # BatchNorm1d + ReLU slots

    mlp("klenc.line_position_enc.encoder", [5, *MLP_HIDDEN, d_model])
    mlp("klenc.word_position_enc.encoder", [3, *MLP_HIDDEN, d_model])
    for i in range(n_desc_layers):
        p = f"klenc.desc_layers.{i}"
        for nm in ("w_qs", "w_ks", "w_vs", "fc"):
            spec.append((f"{p}.slf_attn.{nm}.weight", (d_model, d_model), "w"))
            spec.append((f"{p}.slf_attn.{nm}.bias", (d_model,), "b"))
        spec.append((f"{p}.slf_attn.layer_norm.weight", (d_model,), "ln_w"))
        spec.append((f"{p}.slf_attn.layer_norm.bias", (d_model,), "ln_b"))
        spec.append((f"{p}.pos_ffn.w_1.weight", (d_inner, d_model), "w"))
        spec.append((f"{p}.pos_ffn.w_1.bias", (d_inner,), "b"))
        spec.append((f"{p}.pos_ffn.w_2.weight", (d_model, d_inner), "w"))
        spec.append((f"{p}.pos_ffn.w_2.bias", (d_model,), "b"))
        spec.append((f"{p}.pos_ffn.layer_norm.weight", (d_model,), "ln_w"))
        spec.append((f"{p}.pos_ffn.layer_norm.bias", (d_model,), "ln_b"))
    for i in range(N_SIG_LAYERS):
        p = f"selfattn.layers.{i}"
        for nm in ("merge", "proj.0", "proj.1", "proj.2"):
            spec.append((f"{p}.attn.{nm}.weight", (d_model, d_model, 1), "w"))
            spec.append((f"{p}.attn.{nm}.bias", (d_model,), "b"))
        mlp(f"{p}.mlp", [2 * d_model, 2 * d_model, d_model])
    spec.append(("final_proj.weight", (d_model, d_model, 1), "w"))
    spec.append(("final_proj.bias", (d_model,), "b"))
    return spec


def make_state_dict(seed: int = 0, n_desc_layers: int = 1, d_inner: int = D_INNER) -> dict:
    """Random-init checkpoint of the LineTR architecture, as {key: np.ndarray}.

    Magnitudes are chosen to resemble the shipped checkpoint (weights ~ 1/sqrt(fan_in),
    non-trivial BatchNorm running stats so that the BN fold is actually exercised).
    """
    rng = np.random.Generator(np.random.PCG64(seed))
    sd = {}
    for key, shape, kind in state_dict_spec(n_desc_layers, D_MODEL, d_inner):
        if kind == "w":
            fan_in = shape[1]
            v = rng.standard_normal(shape) * (1.0 / np.sqrt(fan_in))
        elif kind == "b":
            v = rng.standard_normal(shape) * 0.05
        elif kind in ("bn_w", "ln_w"):
            v = 1.0 + 0.1 * rng.standard_normal(shape)
        elif kind in ("bn_b", "ln_b"):
            v = 0.1 * rng.standard_normal(shape)
        elif kind == "bn_mean":
            v = 0.3 * rng.standard_normal(shape)
        elif kind == "bn_var":
            v = rng.uniform(0.5, 1.5, shape)
        elif kind == "bn_count":
            sd[key] = np.array(0, dtype=np.int64)
            continue
        elif kind == "cls":
            v = rng.standard_normal(shape)
        else:  # pragma: no cover
            raise ValueError(kind)
        sd[key] = np.ascontiguousarray(v, dtype=np.float32)
    return sd


def _unit(v, axis=-1):
    n = np.sqrt((v.astype(np.float64) ** 2).sum(axis=axis, keepdims=True))
    return (v / np.maximum(n, 1e-12)).astype(np.float32)


def make_image_inputs(seed: int, n_lines: int, n_tokens: int, n_real_tokens=None,
                      width: int = 640, height: int = 480) -> dict:
    """One image's tokenised lines in the layout the tokenizer emits
    (reference models/line_process.py:182-193), batch dim 1, float32 numpy.

    Padded token slots carry the same kind of data as real ones: the reference
    attends to them (SURVEY.md §0 fact 3), so parity must not depend on the mask.
    """
    rng = np.random.Generator(np.random.PCG64(seed))
    L, T = n_lines, n_tokens
    wh = np.array([width, height], dtype=np.float32)
    sub = (rng.random((L, 2, 2), dtype=np.float32) * wh).astype(np.float32)
    pnt = (rng.random((L, T, 2), dtype=np.float32) * wh).astype(np.float32)
    desc = _unit(rng.standard_normal((L, T, D_MODEL)).astype(np.float32))
    score = (rng.random((L, T, 1), dtype=np.float32) * 0.1).astype(np.float32)
    resp = rng.random((L, 1), dtype=np.float32)
    theta = rng.random(L, dtype=np.float32) * np.float32(np.pi)
    angle = np.stack([np.cos(2 * theta), np.sin(2 * theta)], axis=1).astype(np.float32)
    if n_real_tokens is None:
        ntok = np.full(L, T, dtype=np.int64)
    elif np.isscalar(n_real_tokens):
        ntok = np.full(L, int(n_real_tokens), dtype=np.int64)
    else:
        lo, hi = n_real_tokens
        ntok = rng.integers(lo, hi + 1, size=L)
    mask = np.zeros((L, T + 1, 1), dtype=np.float32)
    mask[:, 0] = 1
    for i in range(L):
        mask[i, 1:1 + int(min(ntok[i], T))] = 1
    return {
        "klines": sub[None].copy(),
        "sublines": sub[None],
        "pnt_sublines": pnt[None],
        "desc_sublines": desc[None],
        "score_sublines": score[None],
        "resp_sublines": resp[None],
        "angle_sublines": angle[None],
        "mask_sublines": mask[None],
        "mat_klines2sublines": np.eye(L, dtype=np.float32)[None],
    }


def make_pair_inputs(seed: int, n_lines: int, n_tokens: int, n_lines1=None,
                     n_real_tokens=None, jitter_px: float = 2.0, desc_noise: float = 0.05):
    """An image pair whose second side is a row-permuted, jittered copy of the first
    (SURVEY.md §8(d)), so that mutual-NN matches exist with top-2 gaps >> 1e-3.

    Returns (side0, side1, perm) with side1 line j == side0 line perm[j] (+noise).
    If n_lines1 < n_lines only the first n_lines1 permuted lines are kept.
    """
    a = make_image_inputs(2 * seed, n_lines, n_tokens, n_real_tokens)
    rng = np.random.Generator(np.random.PCG64(2 * seed + 1))
    L1 = n_lines if n_lines1 is None else int(n_lines1)
    perm = rng.permutation(n_lines)[:L1]
    b = {}
    for k in ("sublines", "pnt_sublines"):
        v = a[k][0][perm]
        b[k] = (v + rng.standard_normal(v.shape).astype(np.float32) * np.float32(jitter_px))[None]
    d = a["desc_sublines"][0][perm]
    d = _unit(d + np.float32(desc_noise) * rng.standard_normal(d.shape).astype(np.float32))
    b["desc_sublines"] = d[None]
    for k in ("score_sublines", "resp_sublines", "angle_sublines", "mask_sublines"):
        b[k] = a[k][0][perm][None].copy()
    b["klines"] = b["sublines"].copy()
    b["mat_klines2sublines"] = np.eye(L1, dtype=np.float32)[None]
    return a, b, perm


def make_descriptor_pair(seed: int, n0: int, n1: int = None, d: int = D_MODEL, noise: float = 0.05):
    """Unit-norm descriptor sets [d,n0], [d,n1] for the matcher-only workload (cfg[4])."""
    rng = np.random.Generator(np.random.PCG64(seed))
    n1 = n0 if n1 is None else n1
    d0 = _unit(rng.standard_normal((n0, d)).astype(np.float32))
    perm = rng.permutation(max(n0, n1))
    perm = perm[perm < n0][:n1] if n1 <= n0 else np.concatenate([rng.permutation(n0), rng.integers(0, n0, n1 - n0)])
    d1 = _unit(d0[perm] + np.float32(noise) * rng.standard_normal((n1, d)).astype(np.float32))
    return np.ascontiguousarray(d0.T), np.ascontiguousarray(d1.T), perm


# ------------------------------------------------------------------ image-level inputs (PairEngine.match_images)
class SyntheticKeyLine:
    """The fields of a cv2 line_descriptor KeyLine the tokeniser reads (reference models/line_process.py:6-20)."""

    def __init__(self, x0, y0, x1, y1, octave=0):
        self.startPointX, self.startPointY, self.endPointX, self.endPointY = float(x0), float(y0), float(x1), float(y1)
        self.lineLength = float(np.hypot(x1 - x0, y1 - y0)) / (2 ** octave)
        self.octave = int(octave)


def make_image_pair(seed: int, n_lines: int, n_points: int, w: int = 640, h: int = 480, jitter_px: float = 0.5,
                    map_noise: float = 0.05):
    """A synthetic image pair as detector + SuperPoint outputs (CPU torch tensors): image 1 is a jittered copy of
    image 0 (key lines, keypoints, dense maps and point descriptors), so lines and points have true matches.
    Each image dict holds 'klines' (SyntheticKeyLine list), 'image_shape' (1,1,h,w), 'keypoints' [N,2],
    'scores' [N], 'descriptors' [256,N], 'dense_descriptor' [1,256,h/8,w/8] and 'dense_score' [1,h,w]."""
    import torch
    rng = np.random.Generator(np.random.PCG64(seed))
    x0, y0 = rng.uniform(8, w - 9, n_lines), rng.uniform(8, h - 9, n_lines)
    ang, ln = rng.uniform(0, 2 * np.pi, n_lines), rng.uniform(20, 300, n_lines)
    x1 = np.clip(x0 + ln * np.cos(ang), 8, w - 9)
    y1 = np.clip(y0 + ln * np.sin(ang), 8, h - 9)
    ends0 = np.stack([x0, y0, x1, y1], 1)
    ends1 = np.clip(ends0 + rng.normal(0, jitter_px, ends0.shape), 8, [w - 9, h - 9, w - 9, h - 9])
    octave = rng.integers(0, 2, n_lines)
    kp0 = np.stack([rng.uniform(0, w - 1, n_points), rng.uniform(0, h - 1, n_points)], 1).astype(np.float32)
    kp1 = np.clip(kp0 + rng.normal(0, jitter_px, kp0.shape), 0, [w - 1, h - 1]).astype(np.float32)
    d0 = _unit(rng.standard_normal((n_points, D_MODEL)).astype(np.float32))
    d1 = _unit(d0 + map_noise * rng.standard_normal(d0.shape).astype(np.float32))
    dense0 = rng.standard_normal((1, D_MODEL, h // 8, w // 8)).astype(np.float32)
    dense1 = dense0 + map_noise * rng.standard_normal(dense0.shape).astype(np.float32)
    score0 = rng.uniform(0, 1, (1, h, w)).astype(np.float32)
    score1 = np.clip(score0 + map_noise * rng.standard_normal(score0.shape), 0, 1).astype(np.float32)

    def image(ends, kp, desc, dense, score):
        dn = torch.from_numpy(dense)
        return {"klines": [SyntheticKeyLine(*e, o) for e, o in zip(ends, octave)], "image_shape": (1, 1, h, w),
                "keypoints": torch.from_numpy(kp), "scores": torch.from_numpy(score.reshape(-1)[:len(kp)].copy()),
                "descriptors": torch.from_numpy(np.ascontiguousarray(desc.T)),
                "dense_descriptor": torch.nn.functional.normalize(dn, dim=1), "dense_score": torch.from_numpy(score)}
    return image(ends0, kp0, d0, dense0, score0), image(ends1, kp1, d1, dense1, score1)


def make_image_set(seed: int, n_views: int, n_lines: int, n_points: int, w: int = 640, h: int = 480,
                   jitter_px: float = 0.5, map_noise: float = 0.05):
    """n_views synthetic views of one scene (image dicts as `make_image_pair` returns): every view is a jittered copy of
    the scene's key lines, keypoints, dense maps and point descriptors, made the way `make_image_pair` makes its
    second image, so every pair of views has true line and point matches."""
    import torch
    rng = np.random.Generator(np.random.PCG64(seed))
    x0, y0 = rng.uniform(8, w - 9, n_lines), rng.uniform(8, h - 9, n_lines)
    ang, ln = rng.uniform(0, 2 * np.pi, n_lines), rng.uniform(20, 300, n_lines)
    x1 = np.clip(x0 + ln * np.cos(ang), 8, w - 9)
    y1 = np.clip(y0 + ln * np.sin(ang), 8, h - 9)
    ends = np.stack([x0, y0, x1, y1], 1)
    octave = rng.integers(0, 2, n_lines)
    kp = np.stack([rng.uniform(0, w - 1, n_points), rng.uniform(0, h - 1, n_points)], 1).astype(np.float32)
    desc = _unit(rng.standard_normal((n_points, D_MODEL)).astype(np.float32))
    dense = rng.standard_normal((1, D_MODEL, h // 8, w // 8)).astype(np.float32)
    score = rng.uniform(0, 1, (1, h, w)).astype(np.float32)
    views = []
    for _ in range(n_views):
        e = np.clip(ends + rng.normal(0, jitter_px, ends.shape), 8, [w - 9, h - 9, w - 9, h - 9])
        k = np.clip(kp + rng.normal(0, jitter_px, kp.shape), 0, [w - 1, h - 1]).astype(np.float32)
        d = _unit(desc + map_noise * rng.standard_normal(desc.shape).astype(np.float32))
        dn = torch.from_numpy(dense + map_noise * rng.standard_normal(dense.shape).astype(np.float32))
        s = np.clip(score + map_noise * rng.standard_normal(score.shape), 0, 1).astype(np.float32)
        views.append({"klines": [SyntheticKeyLine(*x, o) for x, o in zip(e, octave)], "image_shape": (1, 1, h, w),
                      "keypoints": torch.from_numpy(k), "scores": torch.from_numpy(s.reshape(-1)[:len(k)].copy()),
                      "descriptors": torch.from_numpy(np.ascontiguousarray(d.T)),
                      "dense_descriptor": torch.nn.functional.normalize(dn, dim=1), "dense_score": torch.from_numpy(s)})
    return views


def image_to(im: dict, device) -> dict:
    """Tensors of an image dict moved to `device` (klines and shapes untouched)."""
    import torch
    return {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in im.items()}


# ------------------------------------------------------------------ homography-related inputs (geometry)
def random_homography(rng, w: int = 640, h: int = 480, strength: float = 0.1) -> np.ndarray:
    """A homography (fp64 [3, 3], H[2, 2] = 1) that moves each image corner by up to strength * (w, h)."""
    src = np.array([[0, 0], [w - 1, 0], [w - 1, h - 1], [0, h - 1]], dtype=np.float64)
    dst = src + rng.uniform(-strength, strength, (4, 2)) * [w, h]
    A = []
    for (x, y), (u, v) in zip(src, dst):
        A.append([x, y, 1, 0, 0, 0, -u * x, -u * y, u])
        A.append([0, 0, 0, x, y, 1, -v * x, -v * y, v])
    A = np.array(A)
    hv = np.linalg.solve(A[:, :8], A[:, 8])
    return np.append(hv, 1.0).reshape(3, 3)


def warp_points(H, xy) -> np.ndarray:
    """xy [..., 2] mapped by H (fp64)."""
    p = np.asarray(xy, dtype=np.float64)
    q = p @ np.asarray(H, dtype=np.float64)[:, :2].T + np.asarray(H, dtype=np.float64)[:, 2]
    return q[..., :2] / q[..., 2:]


def make_homography_correspondences(seed: int, n_points: int, n_lines: int, H, w: int = 640, h: int = 480,
                                    noise_px: float = 0.3, outlier_frac: float = 0.5, min_outlier_px: float = 10.0):
    """Point and line matches of an image pair related by H (image 0 -> image 1), with a fraction of outliers.

    Row i of side 0 matches row i of side 1 (matches_p / matches_l are the identity).  Inlier keypoints are H(x0) plus
    N(0, noise_px) per coordinate; inlier segments s1 are H of s0's end points slid along s0 (the line is what counts),
    plus the same noise.  An outlier keypoint is moved 10 to 100 px (at least min_outlier_px) from H(x0); an outlier
    segment is moved min_outlier_px + 2 to 60 px along its normal, so no outlier is within min_outlier_px of the true
    model.  Returns dict kpts0, kpts1 [n, 2] / klines0, klines1 [n, 2, 2] float32, matches_p / matches_l int32 and the
    true inlier masks true_p / true_l."""
    rng = np.random.Generator(np.random.PCG64(seed))
    x0 = rng.uniform([0, 0], [w - 1, h - 1], (n_points, 2))
    x1 = warp_points(H, x0) + rng.normal(0, noise_px, (n_points, 2))
    out_p = rng.random(n_points) < outlier_frac
    ang = rng.uniform(0, 2 * np.pi, n_points)
    r = rng.uniform(max(10.0, min_outlier_px), max(100.0, min_outlier_px + 1), n_points)
    x1[out_p] = warp_points(H, x0[out_p]) + (r[:, None] * np.stack([np.cos(ang), np.sin(ang)], 1))[out_p]
    a0 = rng.uniform([20, 20], [w - 21, h - 21], (n_lines, 2))
    t = rng.uniform(0, 2 * np.pi, n_lines)
    b0 = a0 + rng.uniform(40, 200, n_lines)[:, None] * np.stack([np.cos(t), np.sin(t)], 1)
    slide = rng.uniform(-0.1, 0.1, (n_lines, 2))
    a1 = warp_points(H, a0 + slide[:, :1] * (b0 - a0))
    b1 = warp_points(H, b0 + slide[:, 1:] * (b0 - a0))
    out_l = rng.random(n_lines) < outlier_frac
    d = b1 - a1
    nrm = np.stack([-d[:, 1], d[:, 0]], 1) / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-9)
    shift = (rng.uniform(min_outlier_px + 2, max(60.0, min_outlier_px + 3), n_lines)
             * rng.choice([-1.0, 1.0], n_lines))[:, None] * nrm
    a1[out_l] += shift[out_l]
    b1[out_l] += shift[out_l]
    a1 += rng.normal(0, noise_px, a1.shape)
    b1 += rng.normal(0, noise_px, b1.shape)
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    return {"kpts0": f32(x0), "kpts1": f32(x1), "matches_p": np.arange(n_points, dtype=np.int32),
            "klines0": f32(np.stack([a0, b0], 1).reshape(-1, 2, 2)), "klines1": f32(np.stack([a1, b1], 1).reshape(-1, 2, 2)),
            "matches_l": np.arange(n_lines, dtype=np.int32), "true_p": ~out_p, "true_l": ~out_l}


def _warp_field(coarse, Hinv, xs, ys, w, h):
    """A smooth scene field (bilinear over the coarse grid `coarse` [1, C, gh, gw] spread over the w x h image) read
    at the scene positions Hinv(x, y) of the pixel positions xs [n], ys [m]: [1, C, m, n] float32."""
    import torch
    gx, gy = np.meshgrid(xs, ys)
    q = warp_points(Hinv, np.stack([gx, gy], -1))
    grid = np.stack([(q[..., 0] + 0.5) / w * 2 - 1, (q[..., 1] + 0.5) / h * 2 - 1], -1)[None]
    return torch.nn.functional.grid_sample(torch.from_numpy(coarse), torch.from_numpy(grid.astype(np.float32)),
                                           mode="bilinear", padding_mode="border", align_corners=False)


def make_homography_set(seed: int, n_views: int, n_lines: int, n_points: int, w: int = 640, h: int = 480,
                        strength: float = 0.06, jitter_px: float = 0.5, map_noise: float = 0.05, map_cell_px: int = 32):
    """n_views views of one scene (image dicts as `make_image_set` returns) related by known homographies Hs[v] (scene
    -> view): key lines and keypoints are the scene's mapped by Hs[v] plus N(0, jitter_px), point descriptors jittered
    copies of the scene's.  The dense descriptor and score maps are the scene's maps warped by Hs[v] (plus map_noise),
    so a scene line is sampled at the same scene positions in every view and its line descriptors correspond; the
    scene maps are smooth (bilinear over a grid of map_cell_px cells) so that resampling at 8 px cells keeps them.  The
    scene keeps a margin so no view clips it.  Returns (views, Hs [V, 3, 3]); view i -> view j is Hs[j] @ inv(Hs[i])."""
    import torch
    rng = np.random.Generator(np.random.PCG64(seed))
    lo, hi = np.array([0.2 * w, 0.2 * h]), np.array([0.8 * w, 0.8 * h])
    a = rng.uniform(lo, hi, (n_lines, 2))
    ang, ln = rng.uniform(0, 2 * np.pi, n_lines), rng.uniform(30, 150, n_lines)
    b = np.clip(a + ln[:, None] * np.stack([np.cos(ang), np.sin(ang)], 1), lo, hi)
    octave = rng.integers(0, 2, n_lines)
    kp = rng.uniform(lo, hi, (n_points, 2))
    desc = _unit(rng.standard_normal((n_points, D_MODEL)).astype(np.float32))
    gh, gw = -(-h // map_cell_px), -(-w // map_cell_px)
    dense = rng.standard_normal((1, D_MODEL, gh, gw)).astype(np.float32)
    score = rng.uniform(0, 1, (1, 1, gh, gw)).astype(np.float32)
    cx, cy = np.arange(w // 8) * 8 + 3.5, np.arange(h // 8) * 8 + 3.5   # the pixel of each 8 px descriptor cell
    views, Hs = [], []
    for _ in range(n_views):
        Hv = random_homography(rng, w, h, strength)
        Hinv = np.linalg.inv(Hv)
        e = np.concatenate([warp_points(Hv, a), warp_points(Hv, b)], 1) + rng.normal(0, jitter_px, (n_lines, 4))
        k = (warp_points(Hv, kp) + rng.normal(0, jitter_px, kp.shape)).astype(np.float32)
        d = _unit(desc + map_noise * rng.standard_normal(desc.shape).astype(np.float32))
        dn = _warp_field(dense, Hinv, cx, cy, w, h)
        dn = dn + map_noise * torch.from_numpy(rng.standard_normal(tuple(dn.shape)).astype(np.float32))
        sm = _warp_field(score, Hinv, np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64), w, h)[0].numpy()
        s = np.clip(sm + map_noise * rng.standard_normal(sm.shape), 0, 1).astype(np.float32)
        views.append({"klines": [SyntheticKeyLine(*x, o) for x, o in zip(e, octave)], "image_shape": (1, 1, h, w),
                      "keypoints": torch.from_numpy(k), "scores": torch.from_numpy(s.reshape(-1)[:len(k)].copy()),
                      "descriptors": torch.from_numpy(np.ascontiguousarray(d.T)),
                      "dense_descriptor": torch.nn.functional.normalize(dn, dim=1), "dense_score": torch.from_numpy(s)})
        Hs.append(Hv)
    return views, np.stack(Hs)


def make_warp_images(seed: int, n: int, h: int, w: int):
    """n seeded uint8 images for the homography warp: colour [n, h, w, 3] (gradients, rectangles with hard edges, noise
    and regions that are black in every channel) and grey [n, h, w] from it (BT.601 weights, rounded)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    colour = np.empty((n, h, w, 3), dtype=np.uint8)
    for i in range(n):
        img = np.stack([(xx * rng.uniform(0.2, 2) + yy * rng.uniform(-1, 1) + rng.uniform(0, 255)) % 256
                        for _ in range(3)], -1)
        for _ in range(6):
            y0, x0 = rng.integers(0, h), rng.integers(0, w)
            y1, x1 = y0 + rng.integers(1, h // 2 + 2), x0 + rng.integers(1, w // 2 + 2)
            img[y0:y1, x0:x1] = rng.uniform(0, 255, 3)
        img += rng.normal(0, 6, img.shape)
        img = np.clip(np.rint(img), 0, 255)
        for _ in range(2):
            y0, x0 = rng.integers(0, h), rng.integers(0, w)
            img[y0:y0 + rng.integers(1, h // 3 + 2), x0:x0 + rng.integers(1, w // 3 + 2)] = 0
        colour[i] = img
    gray = np.rint(colour.astype(np.float64) @ np.array([0.114, 0.587, 0.299])).astype(np.uint8)
    return gray, colour


# ------------------------------------------------------------------ calibrated two-view inputs (relative pose)
DEFAULT_K = np.array([[500.0, 0.0, 319.5], [0.0, 500.0, 239.5], [0.0, 0.0, 1.0]])


def random_pose(rng, max_angle_deg: float = 15.0, translation=None) -> tuple:
    """A random relative pose (R [3, 3], t [3] with |t| = 1; X1 = R X0 + t): a rotation about a random axis by up to
    max_angle_deg, and a random unit translation unless `translation` is given (normalised)."""
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    a = np.deg2rad(max_angle_deg) * rng.uniform(0.2, 1.0)
    S = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    R = np.eye(3) + np.sin(a) * S + (1 - np.cos(a)) * S @ S
    t = rng.normal(size=3) if translation is None else np.asarray(translation, dtype=np.float64)
    return R, t / np.linalg.norm(t)


def _project(K, X):
    x = X @ np.asarray(K, dtype=np.float64).T
    return x[:, :2] / x[:, 2:]


def make_pose_correspondences(seed: int, n: int, R, t, K0=DEFAULT_K, K1=DEFAULT_K, noise_px: float = 0.5,
                              outlier_frac: float = 0.5, w: int = 640, h: int = 480, min_outlier_px: float = 10.0):
    """Point matches of a calibrated pair with relative pose (R, t) (X1 = R X0 + t): 3D points in front of both cameras
    (depth 2 to 8 in camera 0, seen inside image 0, depth > 0.5 in camera 1), projected with K0 / K1, plus N(0,
    noise_px) per coordinate on both sides.  An outlier's side-1 keypoint is moved min_outlier_px to 60 px across its
    epipolar line (and up to 30 px along it), so no outlier is within min_outlier_px of the true model.  Row i of side
    0 matches row i of side 1.  Returns dict kpts0, kpts1 [n, 2] float32, matches_p int32 and the true inlier mask
    true_p."""
    rng = np.random.Generator(np.random.PCG64(seed))
    R, t = np.asarray(R, dtype=np.float64), np.asarray(t, dtype=np.float64)
    X = np.zeros((0, 3))
    while len(X) < n:
        m = 2 * (n - len(X)) + 8
        x = np.stack([rng.uniform(0, w - 1, m), rng.uniform(0, h - 1, m), np.ones(m)], 1)
        Xc = (x @ np.linalg.inv(K0).T) * rng.uniform(2.0, 8.0, (m, 1))
        X = np.concatenate([X, Xc[(Xc @ R.T + t)[:, 2] > 0.5]])
    X = X[:n]
    x0 = _project(K0, X) + rng.normal(0, noise_px, (n, 2))
    x1 = _project(K1, X @ R.T + t)
    out = rng.random(n) < outlier_frac
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    F = np.linalg.inv(K1).T @ tx @ R @ np.linalg.inv(K0)
    l = np.concatenate([_project(K0, X), np.ones((n, 1))], 1) @ F.T
    nrm = l[:, :2] / np.maximum(np.linalg.norm(l[:, :2], axis=1, keepdims=True), 1e-12)
    tan = np.stack([-nrm[:, 1], nrm[:, 0]], 1)
    shift = (rng.uniform(min_outlier_px, max(60.0, min_outlier_px + 1), n) * rng.choice([-1.0, 1.0], n))[:, None] * nrm \
        + rng.uniform(-30, 30, (n, 1)) * tan
    x1[out] += shift[out]
    x1 += rng.normal(0, noise_px, (n, 2))
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    return {"kpts0": f32(x0), "kpts1": f32(x1), "matches_p": np.arange(n, dtype=np.int32), "true_p": ~out}


def make_pose_set(seed: int, n_views: int, n_lines: int, n_points: int, K=DEFAULT_K, w: int = 640, h: int = 480,
                  max_angle_deg: float = 4.0, max_shift: float = 0.8, jitter_px: float = 0.3, map_noise: float = 0.02,
                  return_points: bool = False):
    """n_views calibrated views (intrinsics K) of one 3D point cloud (image dicts as `make_image_set` returns): camera v
    has pose T[v] (world -> camera, [4, 4]): a rotation of up to max_angle_deg and a centre within max_shift of the
    origin, looking down +z at n_points points 4 to 8 units away, chosen so every view sees all of them.  Keypoints are
    the projections plus N(0, jitter_px); point descriptors are per 3D point plus map_noise, as `make_image_set` makes
    them; key lines and dense maps are `make_image_set`'s (line matches carry no two-view constraint for the pose).
    Returns (views, T [V, 4, 4]); the pose of view i -> view j is T[j] @ inv(T[i]).  With return_points, also the
    world points X [n_points, 3] (fp64): row i of every view's keypoints is the projection of X[i]."""
    import torch
    rng = np.random.Generator(np.random.PCG64(seed))
    K = np.asarray(K, dtype=np.float64)
    Ts = []
    for _ in range(n_views):
        R, _ = random_pose(rng, max_angle_deg)
        c = rng.uniform(-max_shift, max_shift, 3)
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = R, -R @ c
        Ts.append(T)
    X = np.zeros((0, 3))
    while len(X) < n_points:
        m = 2 * n_points
        x = np.stack([rng.uniform(0.15 * w, 0.85 * w, m), rng.uniform(0.15 * h, 0.85 * h, m), np.ones(m)], 1)
        Xc = (x @ np.linalg.inv(K).T) * rng.uniform(4.0, 8.0, (m, 1))
        keep = np.ones(m, dtype=bool)
        for T in Ts:
            q = Xc @ T[:3, :3].T + T[:3, 3]
            p = _project(K, q)
            keep &= (q[:, 2] > 1.0) & (p[:, 0] >= 0) & (p[:, 0] <= w - 1) & (p[:, 1] >= 0) & (p[:, 1] <= h - 1)
        X = np.concatenate([X, Xc[keep]])
    X = X[:n_points]
    base = make_image_set(seed + 1, n_views, n_lines, n_points, w, h, jitter_px, map_noise)
    desc = _unit(rng.standard_normal((n_points, D_MODEL)).astype(np.float32))
    for v, T in zip(base, Ts):
        k = _project(K, X @ T[:3, :3].T + T[:3, 3]) + rng.normal(0, jitter_px, (n_points, 2))
        d = _unit(desc + map_noise * rng.standard_normal(desc.shape).astype(np.float32))
        v["keypoints"] = torch.from_numpy(np.clip(k, 0, [w - 1, h - 1]).astype(np.float32))
        v["descriptors"] = torch.from_numpy(np.ascontiguousarray(d.T))
    return (base, np.stack(Ts), X) if return_points else (base, np.stack(Ts))


# ------------------------------------------------------------------ uncalibrated two-view inputs (fundamental matrices)
def fundamental_from_pose(K0, K1, R, t) -> np.ndarray:
    """F = K1^-T [t]x R K0^-1 (x1^T F x0 = 0 in pixels) scaled to unit Frobenius norm, its largest |entry| positive."""
    t = np.asarray(t, dtype=np.float64)
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    F = np.linalg.inv(K1).T @ tx @ np.asarray(R, dtype=np.float64) @ np.linalg.inv(K0)
    F = F / np.linalg.norm(F)
    return F if F.flat[int(np.argmax(np.abs(F)))] > 0 else -F


def random_intrinsics(rng, w: int = 640, h: int = 480) -> np.ndarray:
    """A pinhole K with focal lengths 0.6 to 1.6 times the image width (fx, fy within 5 % of each other) and the
    principal point within 5 % of the image size of its centre."""
    f = w * rng.uniform(0.6, 1.6)
    c = np.array([(w - 1) / 2, (h - 1) / 2]) + rng.uniform(-0.05, 0.05, 2) * [w, h]
    return np.array([[f, 0.0, c[0]], [0.0, f * rng.uniform(0.95, 1.05), c[1]], [0.0, 0.0, 1.0]])


def make_fundamental_correspondences(seed: int, n_points: int, n_lines: int, noise_px: float = 0.5,
                                     outlier_frac: float = 0.5, line_outlier_frac: float = 0.3, K0=None, K1=None,
                                     w: int = 640, h: int = 480, min_outlier_px: float = 10.0,
                                     min_epipolar_angle_deg: float = 30.0, min_length_px: float = 40.0):
    """Point and line matches of an uncalibrated pair: two views with different intrinsics (random_intrinsics unless
    K0 / K1 are given) and a random relative pose (up to 15 degrees, unit translation).  Points are
    `make_pose_correspondences`': N(0, noise_px) on both sides, an outlier's side-1 keypoint moved min_outlier_px to
    60 px across its epipolar line.  Lines are 3D segments (one end point at depth 2 to 8 in camera 0, 0.3 to 1.5 units
    long) seen inside both images, at least min_length_px long and at least min_epipolar_angle_deg from the epipolar
    line through their midpoint in both images (so end-point noise moves the epipolar intersections little), with
    N(0, noise_px) per end point.  A line outlier's side-1 segment is moved along itself by 1.2 to 2.5 of its lengths,
    off its epipolar band.  Row i of side 0 matches row i of side 1.  Returns dict kpts0 / kpts1 [n, 2], klines0 /
    klines1 [m, 2, 2] float32, matches_p / matches_l int32, the true masks true_p / true_l, the true F (unit norm,
    largest |entry| positive), K0, K1, R, t."""
    rng = np.random.Generator(np.random.PCG64(seed))
    K0 = random_intrinsics(rng, w, h) if K0 is None else np.asarray(K0, dtype=np.float64)
    K1 = random_intrinsics(rng, w, h) if K1 is None else np.asarray(K1, dtype=np.float64)
    R, t = random_pose(rng)
    d = make_pose_correspondences(seed + 1, n_points, R, t, K0, K1, noise_px, outlier_frac, w, h, min_outlier_px)
    F = fundamental_from_pose(K0, K1, R, t)

    def angle_ok(F, a, b):   # the segments a -> b [m, 2] against the epipolar lines F^T / F of their partner images
        mid = np.concatenate([(a + b) / 2, np.ones((len(a), 1))], 1)
        l = mid @ F.T
        n = l[:, :2] / np.maximum(np.linalg.norm(l[:, :2], axis=1, keepdims=True), 1e-300)
        u = (b - a) / np.maximum(np.linalg.norm(b - a, axis=1, keepdims=True), 1e-300)
        return np.abs((u * n).sum(1)) > np.sin(np.deg2rad(min_epipolar_angle_deg))

    segs0, segs1 = np.zeros((0, 2, 2)), np.zeros((0, 2, 2))
    for _ in range(200):
        if len(segs0) >= n_lines:
            break
        m = 4 * (n_lines - len(segs0)) + 16
        x = np.stack([rng.uniform(0, w - 1, m), rng.uniform(0, h - 1, m), np.ones(m)], 1)
        Xa = (x @ np.linalg.inv(K0).T) * rng.uniform(2.0, 8.0, (m, 1))
        u = rng.normal(size=(m, 3))
        Xb = Xa + u / np.linalg.norm(u, axis=1, keepdims=True) * rng.uniform(0.3, 1.5, (m, 1))
        keep = np.ones(m, dtype=bool)
        ends = []
        for Kc, Rc, tc in ((K0, np.eye(3), np.zeros(3)), (K1, R, t)):
            e = []
            for X in (Xa, Xb):
                q = X @ Rc.T + tc
                p = _project(Kc, q)
                keep &= (q[:, 2] > 0.5) & (p[:, 0] >= 0) & (p[:, 0] <= w - 1) & (p[:, 1] >= 0) & (p[:, 1] <= h - 1)
                e.append(p)
            keep &= np.linalg.norm(e[1] - e[0], axis=1) >= min_length_px
            ends.append(e)
        with np.errstate(all="ignore"):
            # side 1 against F x0 (epipolar lines of image 1 are F x0; those of image 0 are F^T x1)
            keep &= angle_ok(F, ends[1][0], ends[1][1]) & angle_ok(F.T, ends[0][0], ends[0][1])
        segs0 = np.concatenate([segs0, np.stack(ends[0], 1)[keep]])
        segs1 = np.concatenate([segs1, np.stack(ends[1], 1)[keep]])
    segs0, segs1 = segs0[:n_lines], segs1[:n_lines]
    m = len(segs0)
    out_l = rng.random(m) < line_outlier_frac
    shift = (segs1[:, 1] - segs1[:, 0]) * (rng.uniform(1.2, 2.5, m) * rng.choice([-1.0, 1.0], m))[:, None]
    segs1[out_l] += shift[out_l][:, None, :]
    segs0 = segs0 + rng.normal(0, noise_px, segs0.shape)
    segs1 = segs1 + rng.normal(0, noise_px, segs1.shape)
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    d.update(klines0=f32(segs0), klines1=f32(segs1), matches_l=np.arange(m, dtype=np.int32), true_l=~out_l, F=F,
             K0=K0, K1=K1, R=R, t=t)
    return d


# ------------------------------------------------------------------ 2D-3D inputs (absolute pose)
def random_rotation(rng) -> np.ndarray:
    """A rotation drawn uniformly (QR of a Gaussian matrix, signs fixed, determinant +1)."""
    Q, Rr = np.linalg.qr(rng.normal(size=(3, 3)))
    Q = Q * np.sign(np.diag(Rr))
    if np.linalg.det(Q) < 0:
        Q[:, 0] = -Q[:, 0]
    return Q


def make_localization_correspondences(seed: int, n_points: int, n_lines: int, noise_px: float = 0.5,
                                      outlier_frac: float = 0.5, line_outlier_frac: float = 0.3, K=DEFAULT_K,
                                      w: int = 640, h: int = 480, min_outlier_px: float = 10.0,
                                      min_length_px: float = 40.0, origin_scale: float = 10.0):
    """2D-3D point and line matches of one query: a query camera with a uniformly random rotation and a centre within
    origin_scale of the world origin (X_cam = R X + t), 3D points at depth 2 to 8 seen inside the image, and 3D segments
    (0.3 to 1.5 units, both end points at depth > 0.5 and inside the image, at least min_length_px long in it).  Query
    keypoints / segment end points are the projections plus N(0, noise_px) per coordinate.  A point outlier's keypoint
    is moved min_outlier_px to 60 px off its projection in a random direction; a line outlier's query segment is moved
    min_outlier_px to 60 px along its normal (both end points, so both are that far from the projected line).  Row i of
    the query matches row i of the 3D arrays.  Returns dict kpts0 [n, 2] / klines0 [m, 2, 2] float32, points3d1 [n, 3]
    / lines3d1 [m, 2, 3] fp64, matches_p / matches_l int32, the true masks true_p / true_l, R, t and K."""
    rng = np.random.Generator(np.random.PCG64(seed))
    K = np.asarray(K, dtype=np.float64)
    Ki = np.linalg.inv(K)
    R = random_rotation(rng)
    centre = rng.uniform(-origin_scale, origin_scale, 3)
    t = -R @ centre
    to_world = lambda Xc: (Xc - t) @ R          # R^T (X_cam - t)
    x = np.stack([rng.uniform(0, w - 1, n_points), rng.uniform(0, h - 1, n_points), np.ones(n_points)], 1)
    Xc = (x @ Ki.T) * rng.uniform(2.0, 8.0, (n_points, 1))
    kp = _project(K, Xc)
    out_p = rng.random(n_points) < outlier_frac
    ang = rng.uniform(0, 2 * np.pi, n_points)
    mag = rng.uniform(min_outlier_px, max(60.0, min_outlier_px + 1), n_points)
    kp[out_p] += (mag[:, None] * np.stack([np.cos(ang), np.sin(ang)], 1))[out_p]
    kp += rng.normal(0, noise_px, kp.shape)
    segs, ends = np.zeros((0, 2, 2)), np.zeros((0, 2, 3))
    for _ in range(200):
        if len(segs) >= n_lines:
            break
        m = 4 * (n_lines - len(segs)) + 16
        xa = np.stack([rng.uniform(0, w - 1, m), rng.uniform(0, h - 1, m), np.ones(m)], 1)
        A = (xa @ Ki.T) * rng.uniform(2.0, 8.0, (m, 1))
        u = rng.normal(size=(m, 3))
        B = A + u / np.linalg.norm(u, axis=1, keepdims=True) * rng.uniform(0.3, 1.5, (m, 1))
        pa, pb = _project(K, A), _project(K, np.where(B[:, 2:] > 0, B, 1.0))
        keep = (B[:, 2] > 0.5) & (pb[:, 0] >= 0) & (pb[:, 0] <= w - 1) & (pb[:, 1] >= 0) & (pb[:, 1] <= h - 1)
        keep &= np.linalg.norm(pb - pa, axis=1) >= min_length_px
        segs = np.concatenate([segs, np.stack([pa, pb], 1)[keep]])
        ends = np.concatenate([ends, np.stack([A, B], 1)[keep]])
    segs, ends = segs[:n_lines], ends[:n_lines]
    m = len(segs)
    out_l = rng.random(m) < line_outlier_frac
    d = segs[:, 1] - segs[:, 0]
    nrm = np.stack([-d[:, 1], d[:, 0]], 1) / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-12)
    shift = nrm * (rng.uniform(min_outlier_px, max(60.0, min_outlier_px + 1), m) * rng.choice([-1.0, 1.0], m))[:, None]
    segs[out_l] += shift[out_l][:, None, :]
    segs = segs + rng.normal(0, noise_px, segs.shape)
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    return {"kpts0": f32(kp), "points3d1": to_world(Xc), "matches_p": np.arange(n_points, dtype=np.int32),
            "klines0": f32(segs.reshape(-1, 2, 2)), "lines3d1": to_world(ends.reshape(-1, 3)).reshape(-1, 2, 3),
            "matches_l": np.arange(m, dtype=np.int32), "true_p": ~out_p, "true_l": ~out_l, "R": R, "t": t, "K": K}


# ------------------------------------------------------------------ posed views of points and segments (triangulation)
def make_line_map_set(seed: int, n_views: int, n_points: int, n_lines: int, K=DEFAULT_K, w: int = 640, h: int = 480,
                      jitter_px: float = 0.0, outlier_frac: float = 0.0, max_angle_deg: float = 6.0,
                      max_shift: float = 1.2, min_length_px: float = 40.0, min_outlier_px: float = 10.0):
    """n_views posed views (intrinsics K, world -> camera R [V, 3, 3], t [V, 3] with X_cam = R X + t: a rotation of up
    to max_angle_deg and a centre within max_shift of the origin, looking down +z) of one scene of n_points 3D points
    and n_lines 3D segments, 4 to 9 units away, every one seen inside every view.  A segment is at least min_length_px
    long in every view.  Each view holds its own clipped part of every segment: the sub-segment between parameters
    a ~ U(0, 0.2) and b ~ U(0.8, 1) of the 3D segment, drawn per view, so partner extents differ.  Row i of every
    view's keypoints is point i and row l of its key lines is segment l: the ground-truth matches of any pair are the
    identity.  Keypoints and segment end points are the projections plus N(0, jitter_px); with probability
    outlier_frac an observation is moved min_outlier_px to 60 px (a keypoint in a random direction, a segment along its
    normal).  Returns dict keypoints (list of float32 [n_points, 2]), klines (list of float32 [n_lines, 2, 2]), K, R,
    t, points3d [n_points, 3], segments3d [n_lines, 2, 3], lines3d [V, n_lines, 2, 3] (each view's end points on the
    true segment), outlier_p [V, n_points] and outlier_l [V, n_lines] (bool)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    K = np.asarray(K, dtype=np.float64)
    Ki = np.linalg.inv(K)
    Rs, ts = [], []
    for _ in range(n_views):
        R, _ = random_pose(rng, max_angle_deg)
        c = rng.uniform(-max_shift, max_shift, 3)
        Rs.append(R)
        ts.append(-R @ c)
    Rs, ts = np.stack(Rs) if n_views else np.zeros((0, 3, 3)), np.stack(ts) if n_views else np.zeros((0, 3))

    def seen(X, margin=0.05):   # [m] inside every view with a margin, depth > 1
        keep = np.ones(len(X), dtype=bool)
        for R, t in zip(Rs, ts):
            q = X @ R.T + t
            p = _project(K, np.where(q[:, 2:] > 0, q, 1.0))
            keep &= (q[:, 2] > 1.0) & (p[:, 0] >= margin * w) & (p[:, 0] <= (1 - margin) * w - 1) \
                & (p[:, 1] >= margin * h) & (p[:, 1] <= (1 - margin) * h - 1)
        return keep

    def sample(m):
        x = np.stack([rng.uniform(0.1 * w, 0.9 * w, m), rng.uniform(0.1 * h, 0.9 * h, m), np.ones(m)], 1)
        return (x @ Ki.T) * rng.uniform(4.0, 9.0, (m, 1))

    X = np.zeros((0, 3))
    for _ in range(200):
        if len(X) >= n_points:
            break
        Xc = sample(2 * n_points + 8)
        X = np.concatenate([X, Xc[seen(Xc)]])
    X = X[:n_points]
    S = np.zeros((0, 2, 3))
    for _ in range(400):
        if len(S) >= n_lines:
            break
        m = 4 * (n_lines - len(S)) + 16
        A = sample(m)
        u = rng.normal(size=(m, 3))
        B = A + u / np.linalg.norm(u, axis=1, keepdims=True) * rng.uniform(0.8, 2.5, (m, 1))
        keep = seen(A) & seen(B)
        for R, t in zip(Rs, ts):
            pa, pb = _project(K, A @ R.T + t), _project(K, np.where((B @ R.T + t)[:, 2:] > 0, B @ R.T + t, 1.0))
            keep &= np.linalg.norm(pb - pa, axis=1) >= min_length_px
        S = np.concatenate([S, np.stack([A, B], 1)[keep]])
    S = S[:n_lines]
    kps, kls, L3 = [], [], []
    out_p = rng.random((n_views, len(X))) < outlier_frac
    out_l = rng.random((n_views, len(S))) < outlier_frac
    for v, (R, t) in enumerate(zip(Rs, ts)):
        k = _project(K, X @ R.T + t)
        ang = rng.uniform(0, 2 * np.pi, len(X))
        mag = rng.uniform(min_outlier_px, max(60.0, min_outlier_px + 1), len(X))
        k[out_p[v]] += (mag[:, None] * np.stack([np.cos(ang), np.sin(ang)], 1))[out_p[v]]
        k += rng.normal(0, jitter_px, k.shape) if jitter_px > 0 else 0.0
        ab = np.stack([rng.uniform(0.0, 0.2, len(S)), rng.uniform(0.8, 1.0, len(S))], 1)
        E = S[:, :1] + ab[:, :, None] * (S[:, 1:] - S[:, :1])        # [m, 2, 3] this view's end points
        seg = _project(K, E.reshape(-1, 3) @ R.T + t).reshape(-1, 2, 2)
        d = seg[:, 1] - seg[:, 0]
        nrm = np.stack([-d[:, 1], d[:, 0]], 1) / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-12)
        shift = nrm * (rng.uniform(min_outlier_px, max(60.0, min_outlier_px + 1), len(S))
                       * rng.choice([-1.0, 1.0], len(S)))[:, None]
        seg[out_l[v]] += shift[out_l[v]][:, None, :]
        seg += rng.normal(0, jitter_px, seg.shape) if jitter_px > 0 else 0.0
        kps.append(np.ascontiguousarray(k, dtype=np.float32))
        kls.append(np.ascontiguousarray(seg, dtype=np.float32))
        L3.append(E)
    return {"keypoints": kps, "klines": kls, "K": K, "R": Rs, "t": ts, "points3d": X, "segments3d": S,
            "lines3d": np.stack(L3) if n_views else np.zeros((0, len(S), 2, 3)), "outlier_p": out_p,
            "outlier_l": out_l}


def _axis_angle(ax, a):
    S = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    return np.eye(3) + np.sin(a) * S + (1 - np.cos(a)) * S @ S


def make_relative_poses(R, t, pairs, noise_deg: float = 0.0, outlier_frac: float = 0.0, seed: int = 0,
                        n_cheirality: int = 100) -> dict:
    """The relative poses of `pairs` (int [P, 2], image i side 0, image j side 1) of the world -> camera poses R [n, 3,
    3], t [n, 3], shaped as an `estimate_poses` PoseResult on the host: R [P, 3, 3] and unit t [P, 3] with X_j = R_p
    X_i + t_p, valid (all True) and n_cheirality (all n_cheirality).  Each clean pose is turned by N(0, noise_deg) about
    a random axis and its direction by N(0, noise_deg) about another; a random outlier_frac of the pairs (exactly
    round(outlier_frac P)) get a random rotation of 30 to 180 degrees and a random direction.  Also returns outlier
    bool [P]."""
    rng = np.random.Generator(np.random.PCG64(seed))
    R, t = np.asarray(R, np.float64), np.asarray(t, np.float64)
    pr = np.asarray(pairs, np.int64).reshape(-1, 2)
    P = len(pr)
    C = -np.einsum("nji,nj->ni", R, t)
    out = np.zeros(P, bool)
    out[rng.permutation(P)[:int(round(outlier_frac * P))]] = True
    Rp, tp = np.zeros((P, 3, 3)), np.zeros((P, 3))
    for p, (i, j) in enumerate(pr):
        if out[p]:
            Rp[p] = _axis_angle(_unit(rng.normal(size=3)), np.deg2rad(rng.uniform(30.0, 180.0)))
            tp[p] = _unit(rng.normal(size=3))
            continue
        Rr = R[j] @ R[i].T
        d = _unit(R[j] @ (C[i] - C[j]))
        Rp[p] = _axis_angle(_unit(rng.normal(size=3)), np.deg2rad(noise_deg * rng.normal())) @ Rr
        tp[p] = _axis_angle(_unit(rng.normal(size=3)), np.deg2rad(noise_deg * rng.normal())) @ d
    return dict(R=Rp, t=tp, valid=np.ones(P, bool), n_cheirality=np.full(P, n_cheirality, np.int32), outlier=out)


def make_covisibility_set(seed: int, n_views: int = 24, window: int = 8, step: int = 2, n_distractors: int = 6,
                          per_landmark: int = 3, noise: float = 0.25, d: int = D_MODEL):
    """Views moving along a corridor of landmarks, each seeing `window` consecutive landmarks (view v from landmark
    v * step), plus distractor views of unrelated scenes.  Every landmark has a point and a key-line descriptor, and a
    view holds `per_landmark` observations of each (unit fp32 rows, noise of norm about `noise`), so both parts carry the overlap.  -> dict
    points / lines: per view [m, d] rows; overlap bool [n, n]: views sharing a landmark (distractors share none, the
    diagonal is False); distractor bool [n]."""
    rng = np.random.default_rng(seed)
    n_lm = (n_views - 1) * step + window
    lm_p, lm_l = _unit(rng.standard_normal((n_lm, d))), _unit(rng.standard_normal((n_lm, d)))
    points, lines, seen = [], [], []

    def observe(lp, ll):
        rep = lambda x: _unit(np.repeat(x, per_landmark, 0) + noise / np.sqrt(d) * rng.standard_normal((len(x) * per_landmark, d)))  # noqa: E731
        return rep(lp).astype(np.float32), rep(ll).astype(np.float32)

    for v in range(n_views):
        ids = np.arange(v * step, v * step + window)
        p, l = observe(lm_p[ids], lm_l[ids])
        points.append(p)
        lines.append(l)
        seen.append(set(ids.tolist()))
    for _ in range(n_distractors):
        p, l = observe(_unit(rng.standard_normal((window, d))), _unit(rng.standard_normal((window, d))))
        points.append(p)
        lines.append(l)
        seen.append(set())
    n = n_views + n_distractors
    overlap = np.array([[i != j and bool(seen[i] & seen[j]) for j in range(n)] for i in range(n)])
    return dict(points=points, lines=lines, overlap=overlap, distractor=np.arange(n) >= n_views)
