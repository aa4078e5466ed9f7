"""The GPU line tokenizer (tok_points_kernel, tok_sample_kernel) at its edges, against the CPU glue and a float64 model.

Every GPU case checks that token positions, sublines, masks, responses, angles and scores equal the CPU glue
(`line_process.line_tokenizer`, pinned to the reference by tests/golden/tokenizer_outputs.npz) bit for bit, that the
scores equal the model's (round half to even, clipped to the score map's own size), that every descriptor is within
the element-wise bound of tests/tokenizer_model.py, and that a one-image `ltr_tokenize_batch` equals the image's rows
of the batch bit for bit.  The maps are shaped as SuperPoint shapes them: descriptors [256, H//8, W//8], scores
[H//8*8, W//8*8], so at sizes that are not multiples of 8 tokens near the right and bottom edges take the score
clip and bilinear taps outside the descriptor grid.  Both align_corners modes are run through the C ABI.

The constructed lines were found by a search that evaluates a token both in the glue's numpy order and with
1 + m*m (position) or dx*dx + dy*dy (response) contracted into one fma, exactly (fractions.Fraction), and keeps
lines where the two round to different fp32 values: a position, a subline cut point, a y coordinate, a score pixel
(a position either side of 301.5) and a response.  A kernel compiled with nvcc's default contraction gets them wrong:
on the parent of this file's commit every one of those five failed on the H100 (the cut points in `sublines`, the
score case in `pnt`, the response in `resp`).  A sixth line has a slope whose square glibc's pow rounds one bit away
from m * m, which moves the fp32 position; the glue and the kernel both square with one product.

Measured worst descriptor err / bound on one H100 80GB HBM3 (700 W), align_corners off / on, printed by each GPU test
with -s: 640x480 0.27 / 0.38, 641x479 0.27 / 0.40, 647x483 0.29 / 0.36, 1600x1200 0.28 / 0.39, 23x17 0.11 / 0.15,
600x15 0.19 / 0.46, the 300-image batch 0.29 / 0.44; T = 1, 7, 21, 128 (off) 0.26 to 0.28; the constructed lines
(off) 0.19 to 0.27.  The file runs in about 25 s on the GPU.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from linetr_b200 import _native as N, line_process as LP
from linetr_b200.nn_matcher import adjacency_to_csr
from tests import tokenizer_model as M
from tests import helpers
from tests.test_tokenizer import fake_superpoint

DEV = torch.device("cuda", 0)
FIELDS = ("sublines", "pnt", "mask", "resp", "angle", "desc", "score")
GLUE = {"sublines": "sublines", "pnt": "pnt_sublines", "mask": "mask_sublines", "resp": "resp_sublines",
        "angle": "angle_sublines", "score": "score_sublines"}


# ------------------------------------------------------------------ inputs
def _line(sp, ep, length=None):
    sp, ep = np.asarray(sp, np.float64), np.asarray(ep, np.float64)
    return sp, ep, float(np.hypot(*(ep - sp))) if length is None else float(length)


def klines_dict(lines):
    """[(sp, ep, length_klines)] -> a `change_cv2_T_np`-style dict (angles as the glue computes them)."""
    kl = np.array([[sp, ep] for sp, ep, _ in lines], dtype=np.float64).reshape(-1, 2, 2)
    return {"klines": kl, "length_klines": np.array([ln for *_, ln in lines], dtype=np.float64),
            "angles": np.asarray(LP.get_angles(kl), dtype=np.float64).reshape(-1, 2)}


def superpoint_maps(seed, W, H, zero_patch=None):
    """SuperPoint-shaped maps of a W x H image: per-cell unit descriptors [256, H//8, W//8] (cells (cx0, cy0, cx1,
    cy1) of zero_patch all zero) and scores [H//8*8, W//8*8]."""
    g = torch.Generator().manual_seed(seed)
    dense = torch.nn.functional.normalize(torch.randn(256, max(H // 8, 1), max(W // 8, 1), generator=g), dim=0)
    if zero_patch is not None:
        cx0, cy0, cx1, cy1 = zero_patch
        dense[:, cy0:cy1, cx0:cx1] = 0
    score = torch.rand(max(H // 8 * 8, 1), max(W // 8 * 8, 1), generator=g)
    return dense, score


def edge_lines(W, H, td, T):
    """The lines where the tokenizer branches, for a W x H image with token distance td and T tokens per subline."""
    out = [
        _line((0.75, H * 0.5), (W - 0.6, H * 0.5)),                 # horizontal, ends at W - 0.6
        _line((W * 0.3, H * 0.3), (W - 0.2, H - 0.3)),              # end point clipped to (W - 0.6, H - 0.6)
        _line((W * 0.1, 0.4), (W * 0.6, H - 0.6)),                  # ends at H - 0.6
        _line((W * 0.5, 0.5), (W * 0.5, H - 0.6)),                  # vertical, down
        _line((W * 0.25, H - 1.25), (W * 0.25, 0.25)),              # vertical, up
        _line((W * 0.7, 0.75), (W * 0.7 + (H - 1.5) * 1e-6, H - 0.75)),   # near vertical, |m| = 1e6
        _line((W * 0.8, H - 0.75), (W * 0.8 + (H - 1.5) * 1e-6, 0.75)),   # near vertical, up
        _line((0.5, 0.5), (W - 0.6, H - 0.6)),                      # the diagonal, through the last pixel
        _line((W * 0.4, H * 0.6), (W * 0.4 + min(td, W * 0.5) * 0.9, H * 0.6)),   # n_tok = 1
    ]
    if float(td).is_integer():                                       # tokens on .5 coordinates: x = 1.5 + i*td ...
        y = np.floor(H * 0.75) + 0.5
        out += [_line((1.5, y), (W - 1.0, y)), _line((2.5, y - 1), (W - 1.0, y - 1)),
                _line((np.floor(W * 0.9) + 0.5, 0.5), (np.floor(W * 0.9) + 0.5, H - 1.0))]
    for k in range(4, 0, -1):                                        # n_tok an exact multiple of T
        n = k * T
        if (n - 0.25) * td <= W - 2:
            out.append(_line((0.5, H * 0.2), (0.5 + (n - 0.25) * td, H * 0.2)))
            break
    return out


SHAPES = [  # W, H, token distance, tokens per subline
    (640, 480, 8.0, 21), (641, 479, 8.0, 7), (647, 483, 8.0875, 128), (1600, 1200, 20.0, 7), (23, 17, 3.0, 1),
    (600, 15, 7.5, 7)]

# lines whose token geometry rounds differently to fp32 in numpy's order and in the contracted one
# (T, td, start, end): token (index) is a position / cut point / score pixel / response that flips
_h = float.fromhex
CONSTRUCTED = [
    # x of token 6 = the cut point of subline 0 (T = 7, td = 16)
    (7, 16.0, (_h("0x1.dee1fcdf13545p+7"), 200.0), (_h("0x1.73310eaabb40ap+8"), _h("0x1.6893bd81810a8p+8")), 6, "x"),
    # x of token 20 = the cut point of subline 0 (T = 21, td = 8)
    (21, 8.0, (_h("0x1.6389761850207p+7"), 200.0), (_h("0x1.58d796151fa44p+8"), _h("0x1.5431eb834f9d1p+8")), 20, "x"),
    # y of token 6 = a cut point (T = 7, td = 16)
    (7, 16.0, (150.0, _h("0x1.01ad0ad6b8d6dp+6")), (_h("0x1.0b2ac80cc2959p+8"), _h("0x1.2a4a5f13debcep+8")), 6, "y"),
    # x of token 5 either side of 301.5: rint picks pixel 301 or 302
    (21, 8.0, (_h("0x1.11b48813955e6p+8"), 200.0), (_h("0x1.4599028094dedp+8"), _h("0x1.24973448dd8a1p+7")), 5, "x"),
    # response of a one-subline line, sp -> ep
    (21, 8.0, (_h("0x1.2292c62958e86p+5"), 240.0), (_h("0x1.2aebe947ead45p+7"), _h("0x1.101531b73073dp+8")), -1, "r"),
    # x of token 14 where libm's pow(m, 2) differs from m * m in the last bit (glibc) and the two round to
    # different fp32 x: the glue and the kernel square with one product
    (21, 8.0, (_h("0x1.5c22ddbdf02b5p+6"), 200.0), (_h("0x1.7d099cc588b0ap+7"), _h("0x1.2d3bed82e0526p+8")), 14, "pow"),
]


# ------------------------------------------------------------------ CPU: the model and the constructed lines
def _some_tokens(W, H, td, T, seed=3):
    dense, score = superpoint_maps(seed, W, H)
    kd = klines_dict(edge_lines(W, H, td, T))
    out = LP.line_tokenizer(kd, td, T, {"dense_descriptor": dense[None], "dense_score": score[None]}, (H, W))
    mask = out["mask_sublines"][0, :, 1:, 0].numpy() > 0
    return out["pnt_sublines"][0].numpy()[mask], dense.numpy(), score.numpy(), out


@pytest.mark.parametrize("W,H", [(641, 479), (23, 17), (600, 15), (647, 483)])
@pytest.mark.parametrize("align", [0, 1])
def test_model_equals_float64_grid_sample(W, H, align):
    pnt, dense, _, _ = _some_tokens(W, H, 8.0 if W > 100 else 3.0, 7)
    Hc, Wc = dense.shape[1:]
    g = torch.from_numpy(M.grid_coords(pnt, Hc, Wc)).double().view(1, 1, -1, 2)
    ref = torch.nn.functional.grid_sample(torch.from_numpy(dense).double()[None], g, mode="bilinear",
                                          align_corners=bool(align))
    ref = torch.nn.functional.normalize(ref.reshape(256, -1), dim=0, eps=1e-12).T.numpy()
    assert np.abs(M.sample_desc(pnt, dense, align) - ref).max() < 1e-13


@pytest.mark.parametrize("ci", [0, 1, 2])
def test_model_reproduces_reference_descriptor_rows(ci):
    """The reference's descriptor rows of tokenizer_outputs.npz (align_corners off) lie within the model's bound."""
    want, (rows, real, _) = helpers.tokenizer_fixture(ci)
    dense = fake_superpoint(7)["dense_descriptor"][0].numpy()
    pnt = want["pnt_sublines"][0][want["mask_sublines"][0, :, 1:, 0] > 0][rows]
    err = np.abs(M.sample_desc(pnt, dense, 0) - real)
    assert (err <= M.desc_bound(pnt, dense, 0)).all()


@pytest.mark.parametrize("W,H", [(641, 479), (23, 17), (600, 15)])
def test_model_mutations_exceed_the_bound(W, H):
    """A flipped align_corners, a half-pixel offset of -0.5, a clamped out-of-grid tap and a skipped normalisation
    each land outside the bound; rounding .5 up instead of to even changes a score.

    A clamped tap shows only where every tap of a token is outside the grid: with one tap inside, the clamped and
    the zero-padded samples are proportional and normalise to the same descriptor.  That happens with align_corners
    off at the bottom rows of these sizes (e.g. y = 478.4 in a 479-row image samples at iy = 59.4 of a 59-cell
    grid); with it on, ix never leaves [0, size - 1] by more than a cell, so the clamp cannot change the output."""
    pnt, dense, score, _ = _some_tokens(W, H, 8.0 if W > 100 else 3.0, 7)
    for align in (0, 1):
        want = M.sample_desc(pnt, dense, align)
        b = M.desc_bound(pnt, dense, align)
        muts = [M.sample_desc(pnt, dense, 1 - align), M.sample_desc(pnt, dense, align, offset=-0.5),
                M.sample_desc(pnt, dense, align, normalise=False)]
        if align == 0:
            muts.append(M.sample_desc(pnt, dense, align, clamp=True))
        for mut in muts:
            assert (np.abs(mut - want) > b).any()
    half = np.array([[2.5, 0.0], [0.0, 4.5], [1.5, 0.0]], dtype=np.float32)   # even + .5 rounds down, odd + .5 up
    assert (M.scores(half, score) != M.scores(half, score, round_half_even=False)).any()
    assert np.array_equal(np.rint(half), np.array([[2, 0], [0, 4], [2, 0]]))


def test_constructed_lines_round_differently_in_the_two_orders():
    """The fma-contracted order rounds each constructed position / response to another fp32 value than the glue's
    order, and the glue (`line_tokenizer`) computes exactly the model's values (squares as products, not pow)."""
    for T, td, sp, ep, i, what in CONSTRUCTED:
        kd = klines_dict([_line(sp, ep)])
        out = LP.line_tokenizer(kd, td, T, {"dense_descriptor": torch.zeros(1, 256, 60, 80),
                                            "dense_score": torch.zeros(1, 480, 640)}, (480, 640))
        if what == "r":
            got = [np.float32(f(sp, ep, td * T)) for f in (M.response_numpy, M.response_contracted)]
            assert out["resp_sublines"][0, 0, 0].item() == got[0]
        else:
            c = 1 if what == "y" else 0
            got = [np.float32(f(sp, ep, i * td)[c]) for f in (M.point_numpy, M.point_contracted)]
            n_tok = int(np.ceil(np.hypot(ep[0] - sp[0], ep[1] - sp[1]) / td))
            assert i < n_tok - 1                           # a token of the line, not its end point
            assert out["pnt_sublines"][0].reshape(-1, 2)[i, c].item() == got[0]
        if what != "pow":                                  # the pow line pins the glue's squares (above)
            assert got[0] != got[1], (sp, ep, i, what)


@pytest.mark.parametrize("bad,match", [(((300, 10), (100, 200)), "runs right to left"),
                                       (((100, 10), (200, -1)), "has a negative coordinate"),
                                       (((-0.5, 10), (200, 100)), "has a negative coordinate"),
                                       (((np.nan, 10), (200, 100)), "has a non-finite"),
                                       (((100, 10), (np.inf, 100)), "has a non-finite")])
def test_key_lines_outside_the_contract_are_refused(bad, match):
    """Reversed key lines, negative coordinates (a score row or column before the map) and NaN / inf."""
    kd = klines_dict([_line((100, 100), (200, 150)), _line(*bad, 100.0)])
    with pytest.raises(N.LtrError, match="key line 1 " + match):
        LP.keyline_geometry(kd["klines"], kd["length_klines"], 8.0, 21, 640, 480)


# ------------------------------------------------------------------ GPU plumbing
def _i32(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(DEV)


def _f64(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(DEV)


def _outputs(S, T):
    f = dict(dtype=torch.float32, device=DEV)
    shapes = ((S, 2, 2), (S, T, 2), (S, T + 1, 1), (S, 1), (S, 2), (S, T, 256), (S, T, 1))
    return {k: torch.full(s, float("nan"), **f) for k, s in zip(FIELDS, shapes)}


def _ptrs(out):
    return [C.c_void_p(out[k].data_ptr()) for k in FIELDS]


def _stream():
    return C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)


class Batch:
    """Host geometry + device arrays of a list of images for ltr_tokenize_batch.  image: dict kd (klines dict),
    td, dense [256,Hc,Wc] and score [Hs,Ws] (CUDA), W, H."""

    def __init__(self, images, T):
        self.images, self.T = images, T
        counts = [len(im["kd"]["klines"]) for im in images]
        n = len(images)
        kl = np.concatenate([im["kd"]["klines"] for im in images]).reshape(-1, 2, 2).copy()
        length = np.concatenate([im["kd"]["length_klines"] for im in images])
        angle = np.concatenate([im["kd"]["angles"] for im in images]).reshape(-1, 2).astype(np.float32)
        li = np.repeat(np.arange(n), counts)
        per = lambda key: np.array([im[key] for im in images])[li]
        g = LP.keyline_geometry(kl, length, per("td").astype(np.float64), T, per("W"), per("H"))
        cuk = np.concatenate([[0], np.cumsum(counts)])
        self.cu = np.ascontiguousarray(g["sub0"][cuk], dtype=np.int32)
        self.sub0, self.K, self.S = g["sub0"], len(kl), int(g["sub0"][-1])
        self.dev = {"sp": _f64(g["sp"]), "ep": _f64(g["ep"]), "epc": _f64(g["epc"]), "len": _f64(length),
                    "ang": torch.from_numpy(angle).to(DEV), "ntok": _i32(g["n_tok"]), "sub0": _i32(g["sub0"]),
                    "s2l": _i32(g["sub2line"]), "li": _i32(li)}
        self.tab = (N.LtrTokenizeImage * max(n, 1))()
        for i, im in enumerate(images):
            if counts[i] or i % 2:     # an image without key lines may pass null maps
                self.tab[i] = N.LtrTokenizeImage(im["dense"].data_ptr(), im["score"].data_ptr(), float(im["td"]),
                                                 im["dense"].shape[1], im["dense"].shape[2], im["score"].shape[0],
                                                 im["score"].shape[1])

    def input(self, align, **override):
        d = self.dev
        kw = dict(n_images=len(self.images), n_keylines=self.K, n_sublines=self.S, n_tokens=self.T)
        kw.update(override)
        return N.LtrTokenizeBatchInput(d["sp"].data_ptr(), d["ep"].data_ptr(), d["epc"].data_ptr(), d["len"].data_ptr(),
                                       d["ang"].data_ptr(), d["ntok"].data_ptr(), d["sub0"].data_ptr(),
                                       d["s2l"].data_ptr(), d["li"].data_ptr(), kw["n_images"], kw["n_keylines"],
                                       kw["n_sublines"], kw["n_tokens"], 256, align, self.tab,
                                       self.cu.ctypes.data_as(N.c_int32_p))

    def run(self, align):
        out = _outputs(self.S, self.T)
        inp = self.input(align)
        N.check(N.load().ltr_tokenize_batch(C.byref(inp), *_ptrs(out), DEV.index, _stream()), "ltr_tokenize_batch")
        return out


def tokenize_one(im, T, align):
    """ltr_tokenize_batch of one image -> outputs."""
    return Batch([im], T).run(align)


def check_image(im, T, align, rows, tag):
    """One image's rows of a GPU run against the glue, the model and a one-image batch."""
    kd = {k: np.array(v, copy=True) for k, v in im["kd"].items()}
    dense, score = im["dense"].cpu(), im["score"].cpu()
    want = LP.line_tokenizer(kd, float(im["td"]), T, {"dense_descriptor": dense[None], "dense_score": score[None]},
                             (im["H"], im["W"]))
    got = {k: v.cpu() for k, v in rows.items()}
    for k, g in GLUE.items():
        assert torch.equal(got[k], want[g][0]), (tag, k)
    one = tokenize_one(im, T, align)
    for k in FIELDS:
        assert torch.equal(one[k].cpu(), got[k]), (tag, "one image", k)
    pnt = got["pnt"].numpy().reshape(-1, 2)
    assert np.array_equal(M.scores(pnt, score.numpy()), got["score"].numpy().reshape(-1)), tag
    d = got["desc"].numpy().reshape(-1, 256)
    err = np.abs(d - M.sample_desc(pnt, dense.numpy(), align))
    b = M.desc_bound(pnt, dense.numpy(), align)
    assert (err <= b).all(), (tag, float(np.max(err - b)))
    with np.errstate(divide="ignore", invalid="ignore"):
        return want, float(np.max(np.where(b > 0, err / b, 0.0)))


def _image(kd, td, W, H, seed, zero_patch=None):
    dense, score = superpoint_maps(seed, W, H, zero_patch)
    return {"kd": kd, "td": td, "W": W, "H": H, "dense": dense.to(DEV), "score": score.to(DEV)}


def _check_batch(images, T, align, tag):
    """Every image of one ltr_tokenize_batch run through check_image; prints the worst descriptor err / bound
    (shown with -s) and returns the Batch."""
    b = Batch(images, T)
    out = b.run(align)
    worst = 0.0
    for i, im in enumerate(images):
        r0, r1 = int(b.cu[i]), int(b.cu[i + 1])
        if len(im["kd"]["klines"]) == 0:
            assert r0 == r1
            continue
        want, ratio = check_image(im, T, align, {k: v[r0:r1] for k, v in out.items()}, f"{tag}:{i}")
        worst = max(worst, ratio)
        k0 = int(np.searchsorted(b.sub0, r0))
        A = want["mat_klines2sublines"][0].numpy()
        assert np.array_equal(b.sub0[k0:k0 + A.shape[0] + 1] - r0, adjacency_to_csr(A))
    print(f"\n{tag} align_corners={align}: worst descriptor err / bound {worst:.2f}")
    return b


# ------------------------------------------------------------------ GPU cases
@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(CONSTRUCTED)))
def test_constructed_lines_take_numpy_order_on_the_gpu(case):
    """Positions, cut points, a score pixel and a response that the fma-contracted order rounds differently, and a
    position where a pow-evaluated square of the slope would."""
    T, td, sp, ep, i, what = CONSTRUCTED[case]
    im = _image(klines_dict([_line(sp, ep)]), td, 640, 480, 40 + case)
    _check_batch([im], T, 0, "constructed")


@pytest.mark.gpu
@pytest.mark.parametrize("W,H,td,T", SHAPES)
@pytest.mark.parametrize("align", [0, 1])
def test_map_shapes_and_edge_lines(W, H, td, T, align):
    """SuperPoint-shaped maps at sizes that are and are not multiples of 8, lines along every branch, a zero
    descriptor patch under some tokens (the 1e-12 norm floor) and a second image of the same size in the batch."""
    lines = edge_lines(W, H, td, T)
    zero = (0, 0, max(W // 16, 1), max(H // 16, 1))           # the top-left cells: under the diagonal's first tokens
    images = [_image(klines_dict(lines), td, W, H, 1, zero), _image(klines_dict(lines[::-1]), td, W, H, 2)]
    b = _check_batch(images, T, align, f"{W}x{H}")
    if W >= 1600:
        assert np.diff(b.sub0).max() > 10                      # lines split into more than 10 sublines


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 7, 21, 128])
def test_token_slot_counts(T):
    """Per T: n_tok = 1, n_tok a multiple of T, one token short and past it, and lines cut into more than 10
    sublines (T <= 21)."""
    W, H, td = 1600, 1200, 4.0
    lines = [_line((10.0, 10.0 + 3 * j), (10.0 + n * td - 0.25 * td, 10.0 + 3 * j)) for j, n in
             enumerate([1, T, T + 1, max(T - 1, 1), 2 * T, 3 * T])]
    lines.append(_line((5.0, 900.0), (1590.0, 1190.0)))        # 200 tokens: 200 / T sublines
    b = _check_batch([_image(klines_dict(lines), td, W, H, 5)], T, 0, f"T{T}")
    if T <= 21:
        assert np.diff(b.sub0).max() > 10


@pytest.mark.gpu
@pytest.mark.parametrize("align", [0, 1])
def test_batch_of_300_images_equals_one_image_batches(align):
    """300 images (3 launches of up to 128) of mixed sizes and token distances; the images at 0, 127, 128, 255 and
    299 have no key lines.  Each image's rows against its own glue, its model and its one-image batch."""
    rng = np.random.Generator(np.random.PCG64(11))
    images = []
    for i in range(300):
        W, H = int(rng.integers(24, 200)), int(rng.integers(17, 160))
        td = float(rng.choice([3.0, 4.5, 8.0, 5.25]))
        lines = []
        if i not in (0, 127, 128, 255, 299):
            for _ in range(int(rng.integers(1, 5))):
                x0, x1 = np.sort(rng.uniform(0, W - 0.6, 2))
                y0, y1 = rng.uniform(0, H - 0.6, 2)
                lines.append(_line((x0, y0), (x1, y1)))
        images.append(_image(klines_dict(lines), td, W, H, 1000 + i))
    _check_batch(images, 7, align, "batch300")


# ------------------------------------------------------------------ GPU: refusals before any launch
def _refused(call, match):
    N.reset_launch_count()
    with pytest.raises(N.LtrError, match=match):
        call()
    torch.cuda.synchronize()
    assert N.launch_count() == 0


@pytest.mark.gpu
def test_batch_refusals_come_before_any_launch():
    ims = [_image(klines_dict(edge_lines(64, 48, 4.0, 7)), 4.0, 64, 48, 1),
           _image(klines_dict(edge_lines(40, 30, 3.0, 7)), 3.0, 40, 30, 2)]
    b = Batch(ims, 7)
    out = _outputs(b.S, 7)
    lib = N.load()

    def call(inp):
        return lambda: N.check(lib.ltr_tokenize_batch(C.byref(inp), *_ptrs(out), DEV.index, _stream()), "batch")

    cu = b.cu.copy()
    b.cu[0] = 1
    _refused(call(b.input(0)), "start at 0")
    b.cu[:] = cu
    b.cu[1] = b.cu[2] + 1
    _refused(call(b.input(0)), "must not decrease")
    b.cu[:] = cu
    b.tab[1] = N.LtrTokenizeImage(None, ims[1]["score"].data_ptr(), 3.0, 3, 5, 24, 40)
    _refused(call(b.input(0)), "null map")
    b.tab[1] = N.LtrTokenizeImage(ims[1]["dense"].data_ptr(), None, 3.0, 3, 5, 24, 40)
    _refused(call(b.input(0)), "null map")
    b = Batch(ims, 7)
    _refused(call(b.input(0, n_tokens=129)), "n_tokens in 1..128")
    for k in ("n_images", "n_keylines", "n_sublines"):
        _refused(call(b.input(0, **{k: -1})), "negative count")
    out_ok = b.run(0)                                          # the unmodified batch still runs
    assert not torch.isnan(out_ok["desc"]).any()
    sp = {"dense_descriptor": ims[0]["dense"][None], "dense_score": ims[0]["score"][None]}
    kd = {k: v.copy() for k, v in ims[0]["kd"].items()}
    _refused(lambda: LP.line_tokenizer_gpu(kd, 4.0, 129, sp, (48, 64)), "n_tokens in 1..128")


@pytest.mark.gpu
def test_reversed_key_line_refused_before_any_launch():
    from linetr_b200 import engine
    from linetr_b200.line_transformer import LineTransformer
    kd = klines_dict([_line((100, 100), (200, 150)), _line((300, 10), (100, 200), 300.0)])
    dense, score = superpoint_maps(0, 640, 480)
    sp = {"dense_descriptor": dense[None].to(DEV), "dense_score": score[None].to(DEV)}
    _refused(lambda: LP.line_tokenizer_gpu({k: v.copy() for k, v in kd.items()}, 8.0, 21, sp, (480, 640)),
             "runs right to left")
    up = klines_dict([_line((100, 100), (200, 150)), _line((300, 10), (400, -2))])   # would read row -2 of the map
    _refused(lambda: LP.line_tokenizer_gpu(up, 8.0, 21, sp, (480, 640)), "has a negative coordinate")
    eng = engine.PairEngine(LineTransformer({"mode": "train", "remove_borders": 0}), DEV)
    im = {"klines": {k: v.copy() for k, v in kd.items()}, "image_shape": (1, 1, 480, 640), **sp}
    _refused(lambda: eng.tokenize_images([im], auto_min_length=False), "runs right to left")
