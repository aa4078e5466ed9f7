"""A float64 model of the GPU line tokenizer's sampled outputs, with element-wise error bounds.

Geometry (token positions, sublines, masks, responses, angles, the adjacency) needs no model: the CPU glue
`line_process.line_tokenizer` computes it in numpy float64 and is pinned to the reference by
tests/golden/tokenizer_outputs.npz, so the GPU must equal it bit for bit.  The sampled outputs are modelled here:

- scores: the score map at round-half-to-even token positions, clipped to the score map's own last row / column
  (reference line_process.py:176-178);
- descriptors: the fp32 grid coordinate exactly as the reference computes it, (kp - s/2 + 0.5) / (w*s - s/2 - 0.5)
  * 2 - 1, then in fp64 grid_sample's unnormalisation (either align_corners mode), a bilinear sample with zero
  padding and an L2 normalisation with the 1e-12 floor.

`desc_bound` bounds |kernel - model| per element from the fp32 operations of tok_sample_kernel.  Every term is a
first-order rounding-error bound; the factor (1 + 2^-10) covers the second-order products, which are smaller by a
factor of the unit roundoff u = 2^-24 at the normalised magnitudes involved.
"""
from fractions import Fraction

import numpy as np
import torch

U = 2.0 ** -24            # fp32 unit roundoff
S = 8                     # SuperPoint cell size


def gamma(n):
    return n * U / (1 - n * U)


def grid_coords(pnt, hc, wc):
    """[N,2] fp32 token positions -> fp32 grid coordinates (gx, gy), computed as the reference's
    sample_descriptors computes them (torch fp32 on the CPU)."""
    kp = torch.from_numpy(np.ascontiguousarray(pnt, dtype=np.float32))
    kp = kp - S / 2 + 0.5
    kp = kp / torch.tensor([(wc * S - S / 2 - 0.5), (hc * S - S / 2 - 0.5)]).to(kp)[None]
    kp = kp * 2 - 1
    return kp.numpy()


def unnormalise(g, size, align_corners):
    """grid_sample's pixel coordinate, fp64."""
    g = np.asarray(g, dtype=np.float64)
    return (g + 1) / 2 * (size - 1) if align_corners else ((g + 1) * size - 1) / 2


def _ix_error(g, size, align_corners):
    """Bound on |fp32 ix of the kernel - exact ix| from its three fp32 roundings."""
    g = np.asarray(g, dtype=np.float64)
    if align_corners:     # fl(fl(fl(g + 1) / 2) * (size - 1)): the halving is exact
        return U * (np.abs(g + 1) / 2 * (size - 1) + np.abs(unnormalise(g, size, True)))
    # fl(fl(fl(g + 1) * size) - 1) / 2, the product and the difference possibly one fma
    return U * (np.abs(g + 1) * size * 2 + np.abs((g + 1) * size - 1)) / 2


def _taps(dense, x, y):
    """dense [C,H,W] at integer arrays x, y (same shape) with zero padding -> [..., C]."""
    C, Hc, Wc = dense.shape
    inside = (x >= 0) & (x < Wc) & (y >= 0) & (y < Hc)
    v = dense[:, np.clip(y, 0, Hc - 1), np.clip(x, 0, Wc - 1)]
    return np.moveaxis(np.where(inside[None], v, 0.0), 0, -1)


def bilinear(dense, ix, iy, clamp=False):
    """fp64 bilinear sample of dense [C,Hc,Wc] at pixel coordinates ix, iy [N] -> (values [N,C], sum of |tap| *
    weight [N,C]).  clamp=True replicates the border instead of zero padding (a mutation, for the tests)."""
    dense = np.asarray(dense, dtype=np.float64)
    C, Hc, Wc = dense.shape
    x0 = np.floor(ix).astype(np.int64)
    y0 = np.floor(iy).astype(np.int64)
    wx1, wy1 = ix - x0, iy - y0
    wx0, wy0 = 1 - wx1, 1 - wy1
    out = np.zeros((len(ix), C))
    mag = np.zeros((len(ix), C))
    for dx, dy, w in ((0, 0, wx0 * wy0), (1, 0, wx1 * wy0), (0, 1, wx0 * wy1), (1, 1, wx1 * wy1)):
        x, y = x0 + dx, y0 + dy
        if clamp:
            x, y = np.clip(x, 0, Wc - 1), np.clip(y, 0, Hc - 1)
        v = _taps(dense, x, y)
        out += v * w[:, None]
        mag += np.abs(v) * w[:, None]
    return out, mag


def _lipschitz(dense, ix, iy, e_ix, e_iy):
    """Per channel bounds on |d sample / d ix| and |d sample / d iy| over every cell that a position within
    (e_ix, e_iy) of (ix, iy) can fall in (floor may move by one), and on the mixed derivative."""
    dense = np.asarray(dense, dtype=np.float64)
    xlo = np.floor(ix - e_ix).astype(np.int64)
    xhi = np.floor(ix + e_ix).astype(np.int64) + 1
    ylo = np.floor(iy - e_iy).astype(np.int64)
    yhi = np.floor(iy + e_iy).astype(np.int64) + 1
    C = dense.shape[0]
    lx = np.zeros((len(ix), C))
    ly = np.zeros((len(ix), C))
    vmax = np.zeros((len(ix), C))
    # the cells span at most 2 columns / rows: offsets 0..2 from (xlo, ylo) cover them
    for oy in range(3):
        for ox in range(3):
            x, y = xlo + ox, ylo + oy
            ok = (x <= xhi) & (y <= yhi)
            v = _taps(dense, x, y)
            vmax = np.maximum(vmax, np.where(ok[:, None], np.abs(v), 0))
            if ox < 2:
                okx = ok & (x + 1 <= xhi)
                lx = np.maximum(lx, np.where(okx[:, None], np.abs(_taps(dense, x + 1, y) - v), 0))
            if oy < 2:
                oky = ok & (y + 1 <= yhi)
                ly = np.maximum(ly, np.where(oky[:, None], np.abs(_taps(dense, x, y + 1) - v), 0))
    return lx, ly, 4 * vmax


def sample_desc(pnt, dense, align_corners, offset=0.5, clamp=False, normalise=True):
    """The fp64 descriptor model: pnt [N,2] fp32 token positions, dense [C,Hc,Wc] -> [N,C].  offset, clamp and
    normalise select the mutations the tests check the bound against."""
    C, Hc, Wc = dense.shape
    if offset == 0.5:
        g = grid_coords(pnt, Hc, Wc)
    else:                  # the half-pixel offset changed: (kp - s/2 + offset)
        kp = torch.from_numpy(np.ascontiguousarray(pnt, dtype=np.float32)) - S / 2 + offset
        kp = kp / torch.tensor([(Wc * S - S / 2 - 0.5), (Hc * S - S / 2 - 0.5)]).to(kp)[None]
        g = (kp * 2 - 1).numpy()
    ix = unnormalise(g[:, 0], Wc, align_corners)
    iy = unnormalise(g[:, 1], Hc, align_corners)
    a, _ = bilinear(dense, ix, iy, clamp)
    if not normalise:
        return a
    n = np.maximum(np.sqrt((a * a).sum(axis=1, keepdims=True)), 1e-12)
    return a / n


def desc_bound(pnt, dense, align_corners):
    """Element-wise bound [N,C] on |tok_sample_kernel's descriptor - sample_desc| for pnt [N,2] fp32.

    Kernel, per token: gx, gy in fp32 as the reference (bit-identical, so no error); ix, iy in fp32 (_ix_error);
    weights (x1 - ix) * (y1 - iy) etc. in fp32, relative error <= 3u; the 4-tap sum a (fma or mul + add), <= gamma_4
    relative to sum |tap| * w; the sum of squares over 256 channels (8 fmas per lane, 5 warp-shuffle levels),
    <= gamma_13 relative; sqrtf, 1 / max(., 1e-12) and the product with a, one rounding each (<= 3u beyond half the
    sum's error).  A change of ix, iy by e moves the exact sample by at most Lx * e_ix + Ly * e_iy + Lxy * e_ix * e_iy
    (bilinear in each cell, continuous across cells, so a moved floor costs nothing more)."""
    dense = np.asarray(dense, dtype=np.float64)
    C, Hc, Wc = dense.shape
    g = grid_coords(pnt, Hc, Wc)
    ix = unnormalise(g[:, 0], Wc, align_corners)
    iy = unnormalise(g[:, 1], Hc, align_corners)
    e_ix = _ix_error(g[:, 0], Wc, align_corners)[:, None]
    e_iy = _ix_error(g[:, 1], Hc, align_corners)[:, None]
    a, mag = bilinear(dense, ix, iy)
    lx, ly, lxy = _lipschitz(dense, ix, iy, e_ix[:, 0] * 1.5, e_iy[:, 0] * 1.5)
    # |a_kernel - a| per channel: position error, plus the weights' and the 4-tap sum's rounding (taken at the
    # kernel's position, whose |tap| * w differs from mag by at most the position term)
    e_pos = lx * e_ix + ly * e_iy + lxy * e_ix * e_iy
    E = e_pos + (3 * U + gamma(4)) * (mag + e_pos)
    norm = np.sqrt((a * a).sum(axis=1, keepdims=True))
    N = np.maximum(norm, 1e-12)
    rE = np.sqrt((E * E).sum(axis=1, keepdims=True)) / N          # relative change of the norm from E
    r_norm = gamma(13) / 2 + 3 * U                                 # the norm's own rounding, sqrt, reciprocal, product
    with np.errstate(divide="ignore", invalid="ignore"):
        r = (rE + r_norm) / (1 - rE - r_norm)
        b = E / N + (np.abs(a) + E) / N * r
    b = np.where(r < 0, np.inf, b) * (1 + 2.0 ** -10)
    # an all-zero patch: every tap is zero, the kernel's sum is exactly 0 and so is its output
    return np.where(mag == 0, 0.0, b)


def scores(pnt, score_map, round_half_even=True):
    """score_map [Hs,Ws] at the tokens pnt [N,2] fp32: round half to even (torch.round), clip to the last
    column / row of the score map -> [N] (round_half_even=False rounds .5 up: a mutation, for the tests)."""
    smap = np.asarray(score_map)
    Hs, Ws = smap.shape
    p = np.asarray(pnt, dtype=np.float32).astype(np.float64)
    r = np.rint(p) if round_half_even else np.floor(p + 0.5)
    rx = np.minimum(r[:, 0].astype(np.int64), Ws - 1)
    ry = np.minimum(r[:, 1].astype(np.int64), Hs - 1)
    return smap[ry, rx]


# ------------------------------------------------------------------ the two fp64 evaluation orders of a token
def _f(x):
    return Fraction(x)


def fma(a, b, c):
    """a * b + c rounded once (an fma.rn.f64), exactly."""
    return float(_f(a) * _f(b) + _f(c))


def point_numpy(sp, ep, d):
    """Token at distance d from sp towards ep, every operation rounded as the glue's numpy code rounds it
    (line_process._tokens_on_line): m = vy / vx, dx = sqrt(d * d / (1 + m * m)), dy = m * dx, + sp.  The squares
    are correctly rounded products, not libm pow (see the line_process module docstring)."""
    vx, vy = ep[0] - sp[0], ep[1] - sp[1]
    if vx == 0:
        return sp[0], (d if vy > 0 else -d) + sp[1]
    m = vy / vx
    dx = float(np.sqrt(d * d / (1 + m * m)))
    return dx + sp[0], m * dx + sp[1]


def point_contracted(sp, ep, d):
    """The same with 1 + m * m contracted into one fma, as nvcc's default -fmad=true compiles it."""
    vx, vy = ep[0] - sp[0], ep[1] - sp[1]
    if vx == 0:
        return sp[0], (d if vy > 0 else -d) + sp[1]
    m = vy / vx
    dx = float(np.sqrt(d * d / fma(m, m, 1.0)))
    return dx + sp[0], m * dx + sp[1]


def response_numpy(a, b, max_len):
    dx, dy = b[0] - a[0], b[1] - a[1]
    return float(np.sqrt(dx * dx + dy * dy)) / max_len


def response_contracted(a, b, max_len):
    dx, dy = b[0] - a[0], b[1] - a[1]
    return float(np.sqrt(fma(dx, dx, dy * dy))) / max_len
