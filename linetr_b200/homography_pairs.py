"""Homography image pairs: sampled homographies, warped images and valid masks for a whole batch.

    sample_homographies(n, shape, rng, **params) -> (H [n,3,3], H_inv [n,3,3])
        the homography builder's `sample_homography_np` + `scale_homography` for n samples (host numpy fp64)
    warp_pairs(gray, colour, src_index, H) -> (warped [P,H,W] uint8, mask [P,H,W] uint8)
        one `ltr_warp_pairs` call: image 1 of every pair and its eroded valid mask; CUDA tensors, no synchronisation
    homography_pairs(gray, colour, n_per_image, rng, **params) -> (warped, mask, H)
        n_per_image sampled homographies of every image, warped in one call
    apply_valid_masks(image_dicts, masks) -> image dicts whose keypoints lie in the mask, with 'valid_mask' attached
    warp_perspective_host(src, M) / valid_mask_host(colour, M)
        numpy models of the two contracts below; tests compare the kernel and OpenCV against them

The warp contract (DESIGN.md "Homography image pairs") is OpenCV's classic fixed-point `warpPerspective` with
`INTER_LINEAR` and `BORDER_CONSTANT` 0.  M = inv(H) maps a pixel of image 1 to image 0.  Columns go in blocks of
bw = min(1024 // min(16, height), width); for column x = xb + j of block xb and row y, X0 = M0*xb + M1*y + M2 (likewise
Y0, W0), w = W0 + M6*j, w = 32/w (0 when w == 0), X = rint((X0 + M0*j) * w) clamped to int (likewise Y).  The source
cell is (X >> 5, Y >> 5) and the sub-pixel position (X & 31, Y & 31) / 32; the four neighbours weigh
(32-fx)(32-fy)*32, fx(32-fy)*32, (32-fx)fy*32 and fx*fy*32 (they sum to 32768), neighbours outside the image count
as 0, and the pixel is (sum w_i p_i + 16384) >> 15.

The mask contract is the builder's: a pixel is invalid where the (float) warp of the colour image is 0 in every
channel, i.e. where no in-image neighbour with a nonzero weight has a nonzero channel; then a 5 x 5 erosion in which
pixels outside the image count as valid.  Mask values are 1 (valid) and 0.
"""
from __future__ import annotations

from math import pi

import numpy as np
import torch

from . import _native as N
from . import _ops

INT_MIN, INT_MAX = -2147483648.0, 2147483647.0
MAX_SIDE = 32767      # OpenCV's remap keeps source cells in int16
ERODE = 5


# ------------------------------------------------------------------ homography sampling (host, fp64)
def _solve8(A, b):
    """x of each [8, 8] system A x = b by Gaussian elimination with partial pivoting in fp64 (first largest |pivot|)."""
    A = np.concatenate([np.array(A, dtype=np.float64), np.asarray(b, dtype=np.float64)[..., None]], -1)
    K, ar = A.shape[0], np.arange(A.shape[0])
    for c in range(8):
        piv = c + np.argmax(np.abs(A[:, c:8, c]), axis=1)
        rc, rp = A[ar, c].copy(), A[ar, piv].copy()
        A[ar, c], A[ar, piv] = rp, rc
        for r in range(c + 1, 8):
            f = A[:, r, c] / A[:, c, c]
            A[:, r, c:] = A[:, r, c:] - f[:, None] * A[:, c, c:]
    x = np.zeros((K, 8))
    for i in range(7, -1, -1):
        acc = A[:, i, 8].copy()
        for j in range(i + 1, 8):
            acc = acc - A[:, i, j] * x[:, j]
        x[:, i] = acc / A[:, i, i]
    return x


def get_perspective_transform(src, dst) -> np.ndarray:
    """cv2.getPerspectiveTransform of each set of four float32 corners [n, 4, 2] -> [n, 3, 3] fp64 (h33 = 1).  As
    OpenCV does, the products src * dst are taken in float32 and the 8 x 8 system is solved in fp64."""
    s = np.asarray(src, dtype=np.float32).reshape(-1, 4, 2)
    d = np.asarray(dst, dtype=np.float32).reshape(-1, 4, 2)
    n = len(s)
    A, b = np.zeros((n, 8, 8)), np.zeros((n, 8))
    sx, sy, dx, dy = s[..., 0], s[..., 1], d[..., 0], d[..., 1]
    A[:, :4, 0] = A[:, 4:, 3] = sx
    A[:, :4, 1] = A[:, 4:, 4] = sy
    A[:, :4, 2] = A[:, 4:, 5] = 1.0
    A[:, :4, 6], A[:, :4, 7] = -sx * dx, -sy * dx
    A[:, 4:, 6], A[:, 4:, 7] = -sx * dy, -sy * dy
    b[:, :4], b[:, 4:] = dx, dy
    return np.concatenate([_solve8(A, b), np.ones((n, 1))], 1).reshape(n, 3, 3)


def scale_homography(H, shape) -> np.ndarray:
    """The builder's scale_homography with shift (-1, -1): a homography of [-1, 1] coordinates -> pixels of an image
    of shape (height, width)."""
    height, width = shape[0], shape[1]
    trans = np.array([[2. / width, 0., -1.], [0., 2. / height, -1.], [0., 0., 1.]])
    return np.linalg.inv(trans) @ np.asarray(H, dtype=np.float64) @ trans


def _pick(valid, rng) -> np.ndarray:
    """Per row, a uniformly drawn column among the True ones of valid [n, k]."""
    cnt = valid.sum(1)
    if np.any(cnt == 0):
        raise ValueError("sample_homographies: no valid candidate (the patch leaves [0, 1) before scaling)")
    k = rng.integers(0, cnt)
    return np.argmax(np.cumsum(valid, 1) > k[:, None], axis=1)


def sample_homographies(n, shape, rng, perspective=True, scaling=True, rotation=True, translation=True, n_scales=5,
                        n_angles=25, scaling_amplitude=0.1, perspective_amplitude_x=0.1, perspective_amplitude_y=0.1,
                        patch_ratio=0.5, max_angle=pi / 2, allow_artifacts=False, translation_overflow=0.):
    """n random homographies as the homography builder samples them (`sample_homography_np` with shape [2, 2] and
    shift -1, then `scale_homography` to pixels of an image of shape (height, width)), drawn from the
    np.random.Generator rng.  Parameters and defaults are the reference's; the truncated normals are
    scipy.stats.truncnorm(-2, 2).  Returns (H, H_inv) fp64 [n, 3, 3]: H maps image 0 to the warped image 1 (the
    builder's `htrans`, the convention of `homography_ground_truth` and `estimate_homographies`), H_inv the other way.

    As in the reference: the corners are rotated as row vectors, (pts - center) @ rot; the candidate scale 1 and the
    candidate angle 0 are always appended, and with allow_artifacts the valid candidates are the first n_scales
    scales (so the last sampled scale is never used) and the first n_angles angles; the corners are rounded to float32
    before the 4-point solve."""
    from scipy.stats import truncnorm

    n = int(n)
    tn = lambda scale, size, loc=0.: truncnorm(-2, 2, loc=loc, scale=scale).rvs(size, random_state=rng)
    ar = np.arange(n)
    pts1 = np.array([[0., 0.], [0., 1.], [1., 1.], [1., 0.]])
    margin = (1 - patch_ratio) / 2
    patch = margin + np.array([[0, 0], [0, patch_ratio], [patch_ratio, patch_ratio], [patch_ratio, 0]])
    pts2 = np.repeat(patch[None], n, 0)
    if perspective:
        if not allow_artifacts:
            perspective_amplitude_x = min(perspective_amplitude_x, margin)
            perspective_amplitude_y = min(perspective_amplitude_y, margin)
        pd = tn(perspective_amplitude_y / 2, n)
        hl = tn(perspective_amplitude_x / 2, n)
        hr = tn(perspective_amplitude_x / 2, n)
        pts2 = pts2 + np.stack([np.stack([hl, pd], 1), np.stack([hl, -pd], 1), np.stack([hr, pd], 1),
                                np.stack([hr, -pd], 1)], 1)
    if scaling:
        scales = np.concatenate([np.ones((n, 1)), tn(scaling_amplitude / 2, (n, n_scales), loc=1.)], 1)
        center = pts2.mean(1, keepdims=True)
        scaled = (pts2 - center)[:, None] * scales[:, :, None, None] + center[:, None]
        if allow_artifacts:
            valid = np.arange(n_scales + 1)[None].repeat(n, 0) < n_scales
        else:
            valid = ((scaled >= 0.) & (scaled < 1.)).all((2, 3))
        pts2 = scaled[ar, _pick(valid, rng)]
    if translation:
        t_min, t_max = pts2.min(1), (1 - pts2).min(1)
        if allow_artifacts:
            t_min = t_min + translation_overflow
            t_max = t_max + translation_overflow
        pts2 = pts2 + rng.uniform(-t_min, t_max)[:, None]
    if rotation:
        angles = np.concatenate([np.linspace(-max_angle, max_angle, num=n_angles), [0.]])
        center = pts2.mean(1, keepdims=True)
        rot = np.stack([np.cos(angles), -np.sin(angles), np.sin(angles), np.cos(angles)], 1).reshape(-1, 2, 2)
        rotated = np.matmul((pts2 - center)[:, None], rot[None]) + center[:, None]
        if allow_artifacts:
            valid = np.arange(n_angles + 1)[None].repeat(n, 0) < n_angles
        else:
            valid = ((rotated >= 0.) & (rotated < 1.)).all((2, 3))
        pts2 = rotated[ar, _pick(valid, rng)]
    # shape [2, 2] and shift -1: the corners in [-1, 1]
    Hs = get_perspective_transform(np.repeat((pts1 * 2 - 1)[None], n, 0), pts2 * 2 - 1)
    return scale_homography(np.linalg.inv(Hs), shape), scale_homography(Hs, shape)


# ------------------------------------------------------------------ numpy models of the warp and the mask
def _cells(M, h, w):
    """Source cells (sx, sy) int64 [h, w] and sub-pixel positions (fx, fy) of every output pixel under M [3, 3]."""
    m = np.asarray(M, dtype=np.float64).reshape(9)
    bw = min(1024 // min(16, h), w)
    x = np.arange(w)
    xb, j = (x - x % bw).astype(np.float64), (x % bw).astype(np.float64)
    y = np.arange(h, dtype=np.float64)[:, None]
    X0 = m[0] * xb + m[1] * y + m[2]
    Y0 = m[3] * xb + m[4] * y + m[5]
    W0 = m[6] * xb + m[7] * y + m[8]
    with np.errstate(all="ignore"):
        W = W0 + m[6] * j
        W = np.where(W != 0, 32.0 / np.where(W != 0, W, 1.0), 0.0)
        X = np.rint(np.clip((X0 + m[0] * j) * W, INT_MIN, INT_MAX)).astype(np.int64)
        Y = np.rint(np.clip((Y0 + m[3] * j) * W, INT_MIN, INT_MAX)).astype(np.int64)
    return X >> 5, Y >> 5, X & 31, Y & 31


def _neighbours(M, h, w):
    """Per output pixel and neighbour k = (0, 0), (0, 1), (1, 0), (1, 1) (dy, dx): source row, column, in-image flag
    and fixed-point weight, each [4, h, w]."""
    sx, sy, fx, fy = _cells(M, h, w)
    rows, cols, inside, wts = [], [], [], []
    for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1)):
        r, c = sy + dy, sx + dx
        rows.append(r)
        cols.append(c)
        inside.append((r >= 0) & (r < h) & (c >= 0) & (c < w))
        wts.append((fy if dy else 32 - fy) * (fx if dx else 32 - fx) * 32)
    return np.stack(rows), np.stack(cols), np.stack(inside), np.stack(wts)


def warp_perspective_host(src, M) -> np.ndarray:
    """The warp contract in numpy: cv2.warpPerspective(src, M, (w, h), flags=INTER_LINEAR | WARP_INVERSE_MAP,
    borderMode=BORDER_CONSTANT) of a uint8 [h, w] or [h, w, C] image, M mapping output pixels to source pixels."""
    src = np.asarray(src, dtype=np.uint8)
    h, w = src.shape[:2]
    rows, cols, inside, wts = _neighbours(M, h, w)
    acc = np.full(src.shape, 16384, dtype=np.int64)
    for k in range(4):
        v = src[np.clip(rows[k], 0, h - 1), np.clip(cols[k], 0, w - 1)].astype(np.int64)
        inw = np.where(inside[k], wts[k], 0)
        acc += v * (inw[..., None] if src.ndim == 3 else inw)
    return np.clip(acc >> 15, 0, 255).astype(np.uint8)


def valid_mask_host(colour, M) -> np.ndarray:
    """The mask contract in numpy: 1 where the builder's valid mask is valid, 0 elsewhere, uint8 [h, w], for a uint8
    colour image [h, w, C] or [h, w] and M mapping output pixels to source pixels."""
    c = np.asarray(colour)
    nz = (c != 0).any(-1) if c.ndim == 3 else c != 0
    h, w = nz.shape
    rows, cols, inside, wts = _neighbours(M, h, w)
    pre = np.zeros((h, w), dtype=bool)
    for k in range(4):
        pre |= inside[k] & (wts[k] > 0) & nz[np.clip(rows[k], 0, h - 1), np.clip(cols[k], 0, w - 1)]
    r = ERODE // 2
    pad = np.pad(pre, r, constant_values=True)
    out = np.ones((h, w), dtype=bool)
    for dy in range(ERODE):
        for dx in range(ERODE):
            out &= pad[dy:dy + h, dx:dx + w]
    return out.astype(np.uint8)


# ------------------------------------------------------------------ batched on the GPU
def _inverse_maps(H, P) -> np.ndarray:
    Hh = np.asarray(H.cpu() if isinstance(H, torch.Tensor) else H, dtype=np.float64)
    if Hh.shape != (P, 3, 3):
        raise N.LtrError(f"warp_pairs: H must be [{P}, 3, 3], got {list(Hh.shape)}")
    try:
        M = np.linalg.inv(Hh)
    except np.linalg.LinAlgError:
        M = np.full_like(Hh, np.nan)
    if not np.isfinite(M).all():
        raise N.LtrError("warp_pairs: a homography is not invertible")
    return np.ascontiguousarray(M.reshape(P, 9))


def warp_pairs(gray, colour, src_index, H):
    """Image 1 of P homography pairs and its valid mask, in one `ltr_warp_pairs` call.

    gray: uint8 CUDA [N, h, w]; colour: uint8 CUDA [N, h, w, C] with C in {1, 3} (for grey-only data pass gray[..., None]);
    src_index: host ints [P], the source image of every pair; H: host fp64 [P, 3, 3], image 0 -> image 1 (inverted here
    in fp64, as cv2.warpPerspective does).  Returns (warped uint8 [P, h, w], mask uint8 [P, h, w]): warped[p] is
    cv2.warpPerspective(gray[src_index[p]], H[p], (w, h)) and mask[p] the builder's eroded valid mask (module
    docstring).  The call never waits for the device."""
    for nm, t in (("gray", gray), ("colour", colour)):
        if not isinstance(t, torch.Tensor):
            raise N.LtrError(f"warp_pairs: '{nm}' must be a torch tensor")
        _ops._req_cuda(t, nm)
    idx = np.asarray(src_index.cpu() if isinstance(src_index, torch.Tensor) else src_index).reshape(-1)
    if idx.size and not np.issubdtype(idx.dtype, np.integer):
        raise N.LtrError("warp_pairs: src_index must be integers")
    if idx.size and (idx.min() < 0 or idx.max() >= gray.shape[0]):
        raise N.LtrError(f"warp_pairs: src_index must lie in [0, {gray.shape[0]})")
    P, dev = len(idx), gray.device
    idx = np.ascontiguousarray(idx, dtype=np.int32)
    dv = _ops.stage({"src_index": idx, "inv_maps": _inverse_maps(H, P)}, dev)
    warped = torch.empty((P, *gray.shape[1:]), dtype=torch.uint8, device=dev)
    mask = torch.empty_like(warped)
    _ops.warp_pairs(gray.contiguous(), colour.contiguous(), idx, dv["src_index"], dv["inv_maps"], warped, mask)
    return warped, mask


def homography_pairs(gray, colour, n_per_image, rng, **params):
    """n_per_image homography pairs of every source image: (warped uint8 [P, h, w], mask uint8 [P, h, w], H fp64
    [P, 3, 3] host), P = N * n_per_image.  Pair p = i * n_per_image + k has image 0 = gray[i] and image 1 = warped[p],
    with H[p] mapping image 0 to image 1, the order `homography_ground_truth`, `score_line_matches` and
    `homography_corner_error` take.  params are `sample_homographies`'."""
    n_img, h, w = (int(s) for s in gray.shape)
    P = n_img * int(n_per_image)
    H, _ = sample_homographies(P, (h, w), rng, **params)
    warped, mask = warp_pairs(gray, colour, np.arange(P) // int(n_per_image), H)
    return warped, mask, H


def apply_valid_masks(image_dicts, masks):
    """Image dicts (detector + SuperPoint outputs as `match_images` takes them) restricted to their valid masks, as the
    builder's remove_out_edge does: keypoint i stays iff mask[int(y_i), int(x_i)] > 0.99, with its score and
    descriptor column.  'valid_mask' (host uint8 [h, w]) is attached, so that `match_images` drops the key lines
    outside it as `preprocess(..., mask=valid_mask)` does.  masks: one [h, w] mask (tensor or array) or None (all
    valid) per dict.  Returns new dicts; the inputs are not modified."""
    from .engine import _first

    if len(image_dicts) != len(masks):
        raise N.LtrError(f"apply_valid_masks: {len(image_dicts)} images but {len(masks)} masks")
    out = []
    for im, m in zip(image_dicts, masks):
        im = dict(im)
        if m is None:
            out.append(im)
            continue
        mh = np.ascontiguousarray(m.cpu().numpy() if isinstance(m, torch.Tensor) else m, dtype=np.uint8)
        kp, sc, de = _first(im["keypoints"]), _first(im["scores"]), _first(im["descriptors"])
        k = np.asarray(kp.detach().cpu().numpy() if isinstance(kp, torch.Tensor) else kp)
        keep = np.flatnonzero(mh[k[:, 1].astype(int), k[:, 0].astype(int)] > 0.99)
        sel = lambda t, dim: (t.index_select(dim, torch.as_tensor(keep, device=t.device))
                              if isinstance(t, torch.Tensor) else np.take(t, keep, axis=dim))
        im.update(keypoints=sel(kp, 0), scores=sel(sc, 0), descriptors=sel(de, 1), valid_mask=mh)
        out.append(im)
    return out
