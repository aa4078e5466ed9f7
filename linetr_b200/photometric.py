"""Photometric augmentation of the homography dataset builder, batched on the GPU.

    sample_photometric(n, shape, rng, **params) -> record
        every per-image scalar of the builder's `imgPhotometric` (ImgAugTransform + customizedTransform.additive_shade),
        drawn from a caller np.random.Generator; params are the yaml's `photometric.params` keys
    photometric_host(gray, record) -> uint8 [N, h, w]
        the numpy model of the whole contract below (the executable statement of it)
    photometric_augment(gray, record) -> uint8 CUDA [N, h, w]
        one `ltr_photometric` call on uint8 CUDA images; no synchronisation
    photometric_homography_pairs(gray, colour, n_per_image, rng, photometric=..., **homography_params)
        -> (image0, warped, mask, H): the builder's order (augment, warp the augmented image, mask from the unaugmented
        colour image)

The contract (DESIGN.md "Photometric augmentation").  Per image, on uint8 values a:
  1. brightness, `reps` times: a = clip(a + delta, 0, 255), delta an integer in [-max_abs_change, max_abs_change].
  2. contrast, `reps` times: a = trunc(clip(fl32(127.5 + fl32(alpha * fl32(a - 127.5))), 0, 255)), alpha float32.
  3. Gaussian noise, `reps` times: a = clip(a + clip(rint(s * z), -255, 255), 0, 255), z a standard normal (fp64).
  4. impulse noise, `reps` times: with probability p, a = rint(255 * sin(pi/2 * u)^2) (a Beta(0.5, 0.5) draw).
  5. motion blur (per image on or off): rint(clip(3 x 3 correlation)) with BORDER_REFLECT_101, the 9 products
     accumulated with fp32 FMAs in row-major kernel order starting from 0 (cv2.filter2D's arithmetic).
  6. additive shade: a uint8 mask of filled ellipses drawn as cv2.ellipse draws them, blurred with the separable
     fp32 Gaussian (row pass, then column pass, each acc = fl32(acc + fl32(tap_k * v_k)) for k = 0..ksize-1 from 0,
     BORDER_REFLECT_101 reflected as often as needed); then the reference's float chain
     x = fl32(fl32(a / 255) * 255), s = fl32(x * fl32(1 - fl32(fl32(t * m) / 255))), c = clip(s, 0, 255),
     out = trunc(float64(fl32(c / 255)) * 255).  Without the shade, out = a (the chain is the identity on all 256
     values).
Per-pixel randomness comes from Philox4x64-10 (numpy.random.Philox's generator) with key (record key, 0) and counter
(y * w + x, r, 0, 0) for application r of the noise primitives: words 0 and 1 give the normal by Box-Muller
(u1 = ((w0 >> 11) + 1) * 2^-53, u2 = (w1 >> 11) * 2^-53, z = sqrt(-2 log u1) * cos(2 pi u2)), word 2 the impulse
test u < p and word 3 the impulse value, both with u = (w >> 11) * 2^-53.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _native as N
from . import _ops

# the homography builder's `augmentation.photometric.params` (dataloaders/confs/homography.yaml)
HOMOGRAPHY_PHOTOMETRIC = {
    "random_brightness": {"max_abs_change": 50},
    "random_contrast": {"strength_range": [0.3, 1.5]},
    "additive_gaussian_noise": {"stddev_range": [0, 10]},
    "additive_speckle_noise": {"prob_range": [0, 0.0035]},
    "additive_shade": {"transparency_range": [-0.5, 0.5], "kernel_size_range": [100, 150]},
    "motion_blur": {"max_kernel_size": 3},
}
PRIMITIVES = ("random_brightness", "random_contrast", "additive_gaussian_noise", "additive_speckle_noise")
MAX_KSIZE = 149          # the largest odd kernel size the blur kernels take (kernel_size_range up to 150)
MIN_KSIZE = 11           # cv2 takes smaller Gaussian kernels from fixed tables, which are not modelled
MAX_REPS = 2

# per-image parameter slots of ltr_photometric (include/linetr_b200.h, csrc/photometric.cuh)
P_BRIGHT, P_CONTRAST, P_NOISE, P_SPECKLE = 0, 3, 6, 9      # each: count, value of application 0, of application 1
P_BLUR, P_KERNEL = 12, 13                                  # on/off, 9 float32 taps row-major
P_SHADE, P_TRANSPARENCY, P_KSIZE = 22, 23, 24
P_KEY_LO, P_KEY_HI, P_N_ELLIPSES = 25, 26, 27
N_PARAMS = 28

XY_SHIFT, XY_ONE = 16, 1 << 16
# cv2's drawing sine table: sin of each integer degree 0..450 rounded to 7 decimals, as float32
SIN_TABLE = (np.round(np.sin(np.deg2rad(np.arange(451, dtype=np.float64))) * 1e7) / 1e7).astype(np.float32)


# ------------------------------------------------------------------ Philox4x64-10
_M0, _M1 = np.uint64(0xD2E7470EE14C6C93), np.uint64(0xCA5A826395121157)
_W0, _W1 = np.uint64(0x9E3779B97F4A7C15), np.uint64(0xBB67AE8584CAA73B)
_M32 = np.uint64(0xFFFFFFFF)


def _mulhilo(a, b):
    """(lo, hi) of the 128-bit product of uint64 arrays a * b."""
    s32 = np.uint64(32)
    al, ah, bl, bh = a & _M32, a >> s32, b & _M32, b >> s32
    p0, p1, p2, p3 = al * bl, al * bh, ah * bl, ah * bh
    mid = (p0 >> s32) + (p1 & _M32) + (p2 & _M32)
    return a * b, p3 + (p1 >> s32) + (p2 >> s32) + (mid >> s32)


def philox4x64(counter, key):
    """Philox4x64-10 of uint64 counters [..., 4] under keys [..., 2] (broadcast) -> uint64 [..., 4].  numpy's
    Philox(key=k, counter=c).random_raw(4) is philox4x64(c + 1, k): the bit generator steps its counter first."""
    c = [np.array(v, dtype=np.uint64) for v in np.moveaxis(np.asarray(counter, dtype=np.uint64), -1, 0)]
    k = [np.array(v, dtype=np.uint64) for v in np.moveaxis(np.asarray(key, dtype=np.uint64), -1, 0)]
    with np.errstate(over="ignore"):
        for r in range(10):
            if r:
                k = [k[0] + _W0, k[1] + _W1]
            lo0, hi0 = _mulhilo(_M0, c[0])
            lo1, hi1 = _mulhilo(_M1, c[2])
            c = [hi1 ^ c[1] ^ k[0], lo1, hi0 ^ c[3] ^ k[1], lo0]
    return np.stack(np.broadcast_arrays(*c), -1)


def _uniform(w):
    return (w >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def noise_words(key, h, w, r):
    """The four Philox words of every pixel [h, w, 4] of one image for application r of the noise primitives."""
    pix = np.arange(h * w, dtype=np.uint64)
    ctr = np.stack([pix, np.full_like(pix, r), np.zeros_like(pix), np.zeros_like(pix)], -1)
    return philox4x64(ctr, np.array([key, 0], dtype=np.uint64)).reshape(h, w, 4)


def gaussian_from_words(w0, w1):
    u1 = ((w0 >> np.uint64(11)).astype(np.float64) + 1.0) * 2.0 ** -53
    u2 = _uniform(w1)
    return np.sqrt(-2.0 * np.log(u1)) * np.cos((2.0 * np.pi) * u2)


# ------------------------------------------------------------------ sampling (host)
def gaussian_taps(ksize) -> np.ndarray:
    """cv2.getGaussianKernel(ksize, 0, CV_32F) for odd ksize >= 11: exp(-x^2 / (2 sigma^2)) in fp64 with
    sigma = 0.3 * ((ksize - 1) / 2 - 1) + 0.8, divided by its fp64 sum, rounded to float32."""
    ksize = int(ksize)
    if ksize < MIN_KSIZE or ksize % 2 == 0:
        raise N.LtrError(f"gaussian_taps: ksize must be odd and >= {MIN_KSIZE}, got {ksize}")
    sigma = ((ksize - 1) * 0.5 - 1) * 0.3 + 0.8
    x = np.arange(ksize) - (ksize - 1) * 0.5
    t = np.exp((-0.5 / (sigma * sigma)) * x * x)
    return (t / t.sum()).astype(np.float32)


def motion_blur_kernel(angle, direction) -> np.ndarray:
    """The 3 x 3 float32 motion-blur kernel of this project (DESIGN.md): the middle column linspace(d, 1 - d, 3) with
    d = (clip(direction, -1, 1) + 1) / 2, quantised as trunc(255 * .) to uint8, rotated by `angle` degrees about the
    centre with bilinear interpolation and zero fill (fp64), divided by 255, rounded to float32 and normalised by its
    float32 sum."""
    d = (float(np.clip(direction, -1.0, 1.0)) + 1.0) / 2.0
    m = np.zeros((3, 3), np.float32)
    m[:, 1] = np.linspace(d, 1.0 - d, num=3)
    q = (m * 255).astype(np.uint8).astype(np.float64)
    th = np.deg2rad(float(angle))
    c, s = np.cos(th), np.sin(th)
    yy, xx = np.mgrid[0:3, 0:3].astype(np.float64) - 1.0
    sx, sy = c * xx + s * yy + 1.0, -s * xx + c * yy + 1.0     # source position of each output tap
    x0, y0 = np.floor(sx).astype(int), np.floor(sy).astype(int)
    fx, fy = sx - x0, sy - y0
    out = np.zeros((3, 3))
    for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1)):
        xi, yi = x0 + dx, y0 + dy
        wgt = (fx if dx else 1 - fx) * (fy if dy else 1 - fy)
        ok = (xi >= 0) & (xi < 3) & (yi >= 0) & (yi < 3)
        out += np.where(ok, wgt * q[np.clip(yi, 0, 2), np.clip(xi, 0, 2)], 0.0)
    k = (out / 255.0).astype(np.float32)
    return (k / np.sum(k, dtype=np.float32)).astype(np.float32)


def _reps(params):
    """How often each of PRIMITIVES is applied, and whether a 3-tap motion blur follows (ImgAugTransform's list)."""
    reps = {p: int(bool(params.get(p))) for p in PRIMITIVES}
    mb = params.get("motion_blur")
    blur = False
    if mb:
        k = mb["max_kernel_size"]
        if k == 3:
            blur = True
        else:
            # the reference builds no MotionBlur for any other size: it appends the previous augmenter once more
            last = [p for p in PRIMITIVES if reps[p]]
            if not last:
                raise N.LtrError("sample_photometric: motion_blur with max_kernel_size != 3 repeats the previous "
                                 "augmenter, and no augmenter precedes it (the reference fails here)")
            reps[last[-1]] += 1
    return reps, blur


def sample_photometric(n, shape, rng, **params):
    """Every per-image draw of the builder's photometric augmentation for n images of shape (height, width), from the
    np.random.Generator rng.  params are the yaml's `photometric.params` (HOMOGRAPHY_PHOTOMETRIC); a missing key turns
    that primitive off.  Returns a dict of numpy arrays (see DESIGN.md "Photometric augmentation"):

        reps          {primitive: 0, 1 or 2}, the applications of random_brightness, random_contrast,
                      additive_gaussian_noise and additive_speckle_noise (2 only through the motion-blur quirk)
        brightness    int32 [n, 2]        contrast  float32 [n, 2]      noise_std  float64 [n, 2]
        speckle_p     float64 [n, 2]      blur  bool [n]                blur_kernel  float32 [n, 3, 3]
        shade         bool                ellipses  int32 [n, E, 5] (ax, ay, x, y, rounded angle)
        transparency  float64 [n]         ksize  int32 [n]              taps  float32 [n, 149] (zero-padded)
        key           uint64 [n]          shape  (height, width)

    As ImgAugTransform builds it, motion_blur with max_kernel_size 3 is a 3-tap MotionBlur applied with probability
    0.5; any other max_kernel_size builds no MotionBlur and applies the previous augmenter (the last enabled of
    PRIMITIVES) a second time, with its own draw.  The shade draws follow _py_additive_shade per image, one uniform
    per draw in its order (ax, ay, x, y, angle per ellipse, then transparency and kernel size), an integer in
    [lo, hi) being lo + floor(u * (hi - lo)); cv2.ellipse rounds the angle, so the record holds rint(angle)."""
    n = int(n)
    h, w = int(shape[0]), int(shape[1])
    unknown = set(params) - set(PRIMITIVES) - {"motion_blur", "additive_shade"}
    if unknown:
        raise N.LtrError(f"sample_photometric: unsupported primitives {sorted(unknown)}")
    if n < 0 or h < 1 or w < 1:
        raise N.LtrError(f"sample_photometric: bad batch {n} x {h} x {w}")
    reps, blur_on = _reps(params)
    rec = {"reps": reps, "shape": (h, w), "brightness": np.zeros((n, MAX_REPS), np.int32),
           "contrast": np.ones((n, MAX_REPS), np.float32), "noise_std": np.zeros((n, MAX_REPS)),
           "speckle_p": np.zeros((n, MAX_REPS)), "blur": np.zeros(n, bool),
           "blur_kernel": np.zeros((n, 3, 3), np.float32)}
    rec["blur_kernel"][:, 1, 1] = 1
    r = reps["random_brightness"]
    if r:
        c = int(params["random_brightness"]["max_abs_change"])
        rec["brightness"][:, :r] = rng.integers(-c, c + 1, size=(n, r))
    r = reps["random_contrast"]
    if r:
        lo, hi = params["random_contrast"]["strength_range"]
        rec["contrast"][:, :r] = rng.uniform(lo, hi, size=(n, r)).astype(np.float32)
    r = reps["additive_gaussian_noise"]
    if r:
        lo, hi = params["additive_gaussian_noise"]["stddev_range"]
        rec["noise_std"][:, :r] = rng.uniform(lo, hi, size=(n, r))
    r = reps["additive_speckle_noise"]
    if r:
        lo, hi = params["additive_speckle_noise"]["prob_range"]
        rec["speckle_p"][:, :r] = rng.uniform(lo, hi, size=(n, r))
    if blur_on:
        rec["blur"] = rng.random(n) < 0.5
        ang, dirn = rng.uniform(0.0, 360.0, n), rng.uniform(-1.0, 1.0, n)
        for i in np.flatnonzero(rec["blur"]):
            rec["blur_kernel"][i] = motion_blur_kernel(ang[i], dirn[i])

    sh = params.get("additive_shade")
    rec["shade"] = bool(sh)
    n_ell = int(sh.get("nb_ellipses", 20)) if sh else 0
    rec["ellipses"] = np.zeros((n, n_ell, 5), np.int32)
    rec["transparency"] = np.zeros(n)
    rec["ksize"] = np.zeros(n, np.int32)
    rec["taps"] = np.zeros((n, MAX_KSIZE), np.float32)
    if sh:
        t_lo, t_hi = sh.get("transparency_range", [-0.5, 0.8])
        k_lo, k_hi = (int(v) for v in sh.get("kernel_size_range", [250, 350]))
        if k_hi <= k_lo:
            raise N.LtrError(f"sample_photometric: empty kernel_size_range [{k_lo}, {k_hi})")
        if k_lo + (k_lo % 2 == 0) < MIN_KSIZE or (k_hi - 1) + ((k_hi - 1) % 2 == 0) > MAX_KSIZE:
            raise N.LtrError(f"sample_photometric: kernel_size_range [{k_lo}, {k_hi}) gives kernel sizes outside "
                             f"[{MIN_KSIZE}, {MAX_KSIZE}]")
        u = rng.random((n, n_ell * 5 + 2))
        min_dim = min(h, w) / 4
        e = u[:, :n_ell * 5].reshape(n, n_ell, 5)
        ax = np.maximum(e[..., 0] * min_dim, min_dim / 5).astype(np.int64)
        ay = np.maximum(e[..., 1] * min_dim, min_dim / 5).astype(np.int64)
        mr = np.maximum(ax, ay)
        if n and n_ell and (np.any(w - mr <= mr) or np.any(h - mr <= mr)):
            raise N.LtrError(f"sample_photometric: a {h} x {w} image is too small for the shade's ellipses "
                             "(randint(max_rad, size - max_rad) is empty, as in the reference)")
        x = mr + np.floor(e[..., 2] * (w - 2 * mr)).astype(np.int64)
        y = mr + np.floor(e[..., 3] * (h - 2 * mr)).astype(np.int64)
        rec["ellipses"] = np.stack([ax, ay, x, y, np.rint(e[..., 4] * 90).astype(np.int64)], -1).astype(np.int32)
        rec["transparency"] = t_lo + u[:, -2] * (t_hi - t_lo)
        k = k_lo + np.floor(u[:, -1] * (k_hi - k_lo)).astype(np.int64)
        rec["ksize"] = (k + (k % 2 == 0)).astype(np.int32)
        for i in range(n):
            rec["taps"][i, :rec["ksize"][i]] = gaussian_taps(rec["ksize"][i])
    rec["key"] = rng.integers(0, 2 ** 63, size=n, dtype=np.int64).astype(np.uint64) * np.uint64(2) + \
        rng.integers(0, 2, size=n, dtype=np.int64).astype(np.uint64)
    return rec


# ------------------------------------------------------------------ numpy model
def reflect101(i, n):
    """cv2.borderInterpolate(i, n, BORDER_REFLECT_101), reflected as often as needed (n == 1 maps everything to 0)."""
    i = np.asarray(i, dtype=np.int64)
    if n == 1:
        return np.zeros_like(i)
    p = 2 * (n - 1)
    i = np.mod(i, p)
    return np.where(i >= n, p - i, i)


def _pointwise(a, rec, i, key):
    """Steps 1-4 of the contract on one uint8 image a [h, w] -> int64 [h, w]."""
    h, w = a.shape
    v = a.astype(np.int64)
    reps = rec["reps"]
    for r in range(reps["random_brightness"]):
        v = np.clip(v + int(rec["brightness"][i, r]), 0, 255)
    for r in range(reps["random_contrast"]):
        al = np.float32(rec["contrast"][i, r])
        t = np.float32(127.5) + al * (v.astype(np.float32) - np.float32(127.5))
        v = np.clip(t, np.float32(0), np.float32(255)).astype(np.int64)
    n_rnd = max(reps["additive_gaussian_noise"], reps["additive_speckle_noise"])
    words = [noise_words(key, h, w, r) for r in range(n_rnd)]
    for r in range(reps["additive_gaussian_noise"]):
        z = gaussian_from_words(words[r][..., 0], words[r][..., 1])
        v = np.clip(v + np.clip(np.rint(rec["noise_std"][i, r] * z), -255, 255).astype(np.int64), 0, 255)
    for r in range(reps["additive_speckle_noise"]):
        hit = _uniform(words[r][..., 2]) < rec["speckle_p"][i, r]
        val = np.rint(255.0 * np.sin((np.pi / 2) * _uniform(words[r][..., 3])) ** 2).astype(np.int64)
        v = np.where(hit, np.clip(val, 0, 255), v)
    return v


def _fma32(a, b, c):
    """fl32(a * b + c) for float32 arrays, exactly: a * b + c is exact in fp64 for the motion blur's operands (uint8
    values, normalised float32 taps, sums below 2^9)."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def filter3x3(v, k) -> np.ndarray:
    """cv2.filter2D(v, -1, k) of a uint8 image with a 3 x 3 float32 kernel, BORDER_REFLECT_101: fp32 FMAs over the
    kernel in row-major order from 0, rounded half to even and saturated to uint8."""
    h, w = v.shape
    rows, cols = reflect101(np.arange(-1, h + 1), h), reflect101(np.arange(-1, w + 1), w)
    p = v.astype(np.float32)[rows][:, cols]
    acc = np.zeros((h, w), np.float32)
    for dy in range(3):
        for dx in range(3):
            acc = _fma32(p[dy:dy + h, dx:dx + w], np.float32(k[dy, dx]), acc)
    return np.clip(np.rint(acc), 0, 255).astype(np.uint8)


def ellipse_polygon(ax, ay, x, y, angle):
    """The fixed-point (1/65536 pixel) polygon cv2.ellipse fills for a full ellipse with integer centre, axes and
    angle: ellipse2Poly on the sine table at the angular step cv2 picks from the larger axis, rounded to 1/65536 and
    with consecutive duplicates dropped.  int64 [V, 2]."""
    cx, cy = float(int(x) << XY_SHIFT), float(int(y) << XY_SHIFT)
    aw, ah = float(abs(int(ax)) << XY_SHIFT), float(abs(int(ay)) << XY_SHIFT)
    big = max(abs(int(ax)), abs(int(ay)))
    step = 90 if big < 3 else 30 if big < 10 else 18 if big < 15 else 5
    ang = int(angle) % 360
    alpha, beta = np.float64(SIN_TABLE[450 - ang]), np.float64(SIN_TABLE[ang])
    a = np.minimum(np.arange(0, 360 + step, step), 360)
    px = aw * SIN_TABLE[450 - a].astype(np.float64)
    py = ah * SIN_TABLE[a].astype(np.float64)
    vx = cx + px * alpha - py * beta
    vy = cy + px * beta + py * alpha
    qx = np.rint(vx / XY_ONE).astype(np.int64) << XY_SHIFT
    qy = np.rint(vy / XY_ONE).astype(np.int64) << XY_SHIFT
    pts = np.stack([qx + np.rint(vx - qx).astype(np.int64), qy + np.rint(vy - qy).astype(np.int64)], -1)
    keep = np.ones(len(pts), bool)
    keep[1:] = (pts[1:] != pts[:-1]).any(1)
    pts = pts[keep]
    if len(pts) == 1:
        pts = np.array([[int(x) << XY_SHIFT, int(y) << XY_SHIFT]] * 2, dtype=np.int64)
    return pts


def _tdiv(a, b):
    """C integer division (truncation toward zero)."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def _line(mask, p1, p2):
    """cv2's 8-connected fixed-point line (XY_SHIFT fraction bits) from p1 to p2, value 255, clipped to the image."""
    h, w = mask.shape
    (x1, y1), (x2, y2) = (int(p1[0]), int(p1[1])), (int(p2[0]), int(p2[1]))
    dx, dy = x2 - x1, y2 - y1
    half = XY_ONE >> 1
    pts = [((x2 + half) >> XY_SHIFT, (y2 + half) >> XY_SHIFT)]
    if abs(dx) > abs(dy):
        if dx < 0:
            x1, x2, y1, y2, dy = x2, x1, y2, y1, -dy
        ystep = _tdiv(dy << XY_SHIFT, abs(dx) | 1)
        ecount = (x2 - x1) >> XY_SHIFT
        x, yy = (x1 + half) >> XY_SHIFT, y1 + half
        k = np.arange(ecount + 1, dtype=np.int64)
        xs, ys = x + k, (yy + k * ystep) >> XY_SHIFT
    else:
        if dy < 0:
            x1, x2, y1, y2, dx = x2, x1, y2, y1, -dx
        xstep = _tdiv(dx << XY_SHIFT, abs(dy) | 1)
        ecount = (y2 - y1) >> XY_SHIFT
        xx, y = x1 + half, (y1 + half) >> XY_SHIFT
        k = np.arange(ecount + 1, dtype=np.int64)
        xs, ys = (xx + k * xstep) >> XY_SHIFT, y + k
    xs = np.concatenate([xs, [pts[0][0]]])
    ys = np.concatenate([ys, [pts[0][1]]])
    ok = (xs >= 0) & (xs < w) & (ys >= 0) & (ys < h)
    mask[ys[ok], xs[ok]] = 255


def fill_spans(v, h):
    """The spans of cv2's convex-polygon scan fill of the fixed-point polygon v [V, 2]: a list of (y0, y1, xl, dxl,
    xr, dxr) row ranges [y0, y1) whose two edge positions at row y are x + (y - y0) * dx (in 1/65536 pixel)."""
    npts = len(v)
    half = XY_ONE >> 1
    if npts < 3:
        return []
    ys = v[:, 1]
    imin = int(np.argmin(ys))
    ymin, ymax = (int(ys.min()) + half) >> XY_SHIFT, (int(ys.max()) + half) >> XY_SHIFT
    ymax = min(ymax, h - 1)
    edges = npts
    idx, ye, ex, edx = [imin, imin], [ymin, ymin], [0, 0], [0, 0]
    di = (1, npts - 1)
    out, y = [], ymin
    while y <= ymax:
        for i in range(2):
            if y >= ye[i]:
                i0 = idx[i]
                i1 = (i0 + di[i]) % npts
                while True:
                    edges -= 1
                    if edges < 0:
                        break
                    ty = (int(v[i1, 1]) + half) >> XY_SHIFT
                    if ty > y:
                        xs, xe = int(v[i0, 0]), int(v[i1, 0])
                        ye[i], ex[i], idx[i] = ty, xs, i1
                        edx[i] = _tdiv((xe - xs) * 2 + (ty - y), 2 * (ty - y))
                        break
                    i0, i1 = i1, (i1 + di[i]) % npts
        if edges < 0:
            break
        y1 = min(ye[0], ye[1], ymax + 1)
        out.append((y, y1, ex[0], edx[0], ex[1], edx[1]))
        ex = [ex[0] + edx[0] * (y1 - y), ex[1] + edx[1] * (y1 - y)]
        y = y1
    return out


def ellipse_mask(shape, ellipses) -> np.ndarray:
    """The shade mask: cv2.ellipse(mask, (x, y), (ax, ay), angle, 0, 360, 255, -1) of every (ax, ay, x, y, angle) row
    of ellipses into a zero uint8 image of the given shape."""
    h, w = shape
    mask = np.zeros((h, w), np.uint8)
    half = XY_ONE >> 1
    for ax, ay, x, y, angle in np.asarray(ellipses).reshape(-1, 5):
        v = ellipse_polygon(ax, ay, x, y, angle)
        for j in range(len(v)):
            _line(mask, v[j - 1], v[j])
        if len(v) < 3 or ((int(v[:, 0].max()) + half) >> XY_SHIFT) < 0 or ((int(v[:, 0].min()) + half) >> XY_SHIFT) >= w:
            continue
        for y0, y1, xl, dxl, xr, dxr in fill_spans(v, h):
            for yy in range(max(y0, 0), y1):
                a, b = xl + (yy - y0) * dxl, xr + (yy - y0) * dxr
                if a > b:
                    a, b = b, a
                x1, x2 = (a + half) >> XY_SHIFT, (b + half) >> XY_SHIFT
                if x2 >= 0 and x1 < w:
                    mask[yy, max(x1, 0):min(x2, w - 1) + 1] = 255
    return mask


def gaussian_blur(img, taps) -> np.ndarray:
    """The shade's separable blur of a float32 [h, w] image with float32 taps (odd length), BORDER_REFLECT_101:
    rows, then columns, each output fl32(acc + fl32(tap_k * v_k)) accumulated for k = 0.. from 0."""
    img = np.asarray(img, dtype=np.float32)
    taps = np.asarray(taps, dtype=np.float32)
    h, w = img.shape
    r = len(taps) // 2
    p = img[:, reflect101(np.arange(-r, w + r), w)]
    acc = np.zeros((h, w), np.float32)
    for k in range(len(taps)):
        acc = acc + taps[k] * p[:, k:k + w]
    p = acc[reflect101(np.arange(-r, h + r), h)]
    acc = np.zeros((h, w), np.float32)
    for k in range(len(taps)):
        acc = acc + taps[k] * p[k:k + h]
    return acc


def shade_pre_truncation(a, m, transparency) -> np.ndarray:
    """The value the builder truncates to a byte, float64 [h, w], for stage-1 bytes a and the blurred mask m."""
    f32 = np.float32
    x = (np.asarray(a).astype(f32) / f32(255)) * f32(255)
    s = x * (f32(1) - (f32(transparency) * np.asarray(m, dtype=f32)) / f32(255))
    c = np.clip(s, f32(0), f32(255)) / f32(255)
    return c.astype(np.float64) * 255


def photometric_host(gray, record, return_stages=False):
    """The contract in numpy: uint8 [N, h, w] -> uint8 [N, h, w].  With return_stages, also returns the stage-1 bytes,
    the shade masks, the blurred masks and the pre-truncation values (None where the shade is off)."""
    g = np.asarray(gray, dtype=np.uint8)
    n, h, w = g.shape
    if tuple(record["shape"]) != (h, w) or len(record["key"]) != n:
        raise N.LtrError(f"photometric_host: the record is for {len(record['key'])} images of {record['shape']}")
    out = np.empty_like(g)
    st = {"stage1": np.empty_like(g), "mask": [], "blur": [], "pre": []}
    for i in range(n):
        v = _pointwise(g[i], record, i, record["key"][i])
        a = filter3x3(v.astype(np.uint8), record["blur_kernel"][i]) if record["blur"][i] else v.astype(np.uint8)
        st["stage1"][i] = a
        if record["shade"]:
            mk = ellipse_mask((h, w), record["ellipses"][i])
            m = gaussian_blur(mk.astype(np.float32), record["taps"][i, :record["ksize"][i]])
            pre = shade_pre_truncation(a, m, record["transparency"][i])
            out[i] = pre.astype(np.uint8)
            st["mask"].append(mk), st["blur"].append(m), st["pre"].append(pre)
        else:
            out[i] = a
    return (out, st) if return_stages else out


# ------------------------------------------------------------------ batched on the GPU
def params_array(record) -> np.ndarray:
    """The record as ltr_photometric's per-image parameter rows, fp64 [n, N_PARAMS]."""
    n = len(record["key"])
    p = np.zeros((n, N_PARAMS))
    reps = record["reps"]
    for slot, prim, name in ((P_BRIGHT, "random_brightness", "brightness"), (P_CONTRAST, "random_contrast", "contrast"),
                             (P_NOISE, "additive_gaussian_noise", "noise_std"),
                             (P_SPECKLE, "additive_speckle_noise", "speckle_p")):
        p[:, slot] = reps[prim]
        p[:, slot + 1:slot + 3] = np.asarray(record[name], dtype=np.float64)
    p[:, P_BLUR] = np.asarray(record["blur"], dtype=bool)
    p[:, P_KERNEL:P_KERNEL + 9] = np.asarray(record["blur_kernel"], dtype=np.float32).reshape(n, 9)
    p[:, P_SHADE] = bool(record["shade"])
    p[:, P_TRANSPARENCY] = record["transparency"]
    p[:, P_KSIZE] = record["ksize"]
    key = np.asarray(record["key"], dtype=np.uint64)
    p[:, P_KEY_LO], p[:, P_KEY_HI] = key & _M32, key >> np.uint64(32)
    p[:, P_N_ELLIPSES] = np.asarray(record["ellipses"]).shape[1]
    return p


def _check_ellipses(ell, h, w):
    if ell.size == 0:
        return
    ax, ay, x, y = ell[..., 0], ell[..., 1], ell[..., 2], ell[..., 3]
    mr = np.maximum(ax, ay)
    if np.any(ax < 0) or np.any(ay < 0) or np.any(x < mr) or np.any(x + mr >= w) or np.any(y < mr) or \
            np.any(y + mr >= h):
        raise N.LtrError("photometric_augment: an ellipse does not lie inside the image "
                         "(max(ax, ay) <= x < w - max(ax, ay), likewise y)")


def photometric_augment(gray, record):
    """The builder's photometric augmentation of every image of gray (uint8 CUDA [N, h, w]) with the draws of
    `record` (sample_photometric(N, (h, w), ...)), in one `ltr_photometric` call.  Returns a new uint8 CUDA tensor
    [N, h, w], equal to photometric_host(gray, record); the call never waits for the device."""
    if not isinstance(gray, torch.Tensor):
        raise N.LtrError("photometric_augment: 'gray' must be a torch tensor")
    _ops._req_cuda(gray, "gray")
    if gray.dim() != 3 or gray.dtype != torch.uint8:
        raise N.LtrError(f"photometric_augment: gray must be uint8 [N, h, w], got {gray.dtype} {list(gray.shape)}")
    n, h, w = (int(s) for s in gray.shape)
    if tuple(record["shape"]) != (h, w) or len(record["key"]) != n:
        raise N.LtrError(f"photometric_augment: the record is for {len(record['key'])} images of "
                         f"{tuple(record['shape'])}, the batch is {n} of {(h, w)}")
    ell = np.ascontiguousarray(record["ellipses"], dtype=np.int32)
    _check_ellipses(ell, h, w)
    ph = params_array(record)
    dev = gray.device
    dv = _ops.stage({"params": ph, "ellipses": ell.reshape(n, -1, 5),
                      "taps": np.ascontiguousarray(record["taps"], dtype=np.float32)}, dev)
    out = torch.empty_like(gray)
    ws = torch.empty(N.photometric_workspace_bytes(n, h, w), dtype=torch.uint8, device=dev)
    _ops.photometric(gray.contiguous(), out, ph, dv["params"], dv["ellipses"], dv["taps"], ws)
    return out


def photometric_homography_pairs(gray, colour, n_per_image, rng, photometric=None, **homography_params):
    """Homography pairs built the way the builder builds them with photometric augmentation on: n_per_image pairs of
    every source image, each with its own augmentation of the source (image 0), image 1 the warp of the augmented
    image, and the valid mask from the unaugmented colour image.  gray uint8 CUDA [N, h, w], colour uint8 CUDA
    [N, h, w, C]; photometric: the yaml's `photometric.params` (default HOMOGRAPHY_PHOTOMETRIC); homography_params:
    `sample_homographies`'.  The homographies are drawn from rng first, exactly as `homography_pairs` draws them, then
    the photometric record.  Returns (image0 uint8 [P, h, w], warped uint8 [P, h, w], mask uint8 [P, h, w], H fp64
    [P, 3, 3] host), P = N * n_per_image, pair p = i * n_per_image + k."""
    from .homography_pairs import sample_homographies, warp_pairs

    n_img, h, w = (int(s) for s in gray.shape)
    per = int(n_per_image)
    P = n_img * per
    H, _ = sample_homographies(P, (h, w), rng, **homography_params)
    params = HOMOGRAPHY_PHOTOMETRIC if photometric is None else photometric
    record = sample_photometric(P, (h, w), rng, **params)
    src = np.arange(P) // per
    image0 = photometric_augment(gray.index_select(0, torch.as_tensor(src, device=gray.device)), record)
    warped, _ = warp_pairs(image0, image0[..., None], np.arange(P), H)
    _, mask = warp_pairs(gray, colour, src, H)
    return image0, warped, mask, H
