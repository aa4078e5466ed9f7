"""Photometric augmentation (`photometric`): the numpy model against numpy's Philox, OpenCV and the reference's
additive shade (golden fixture), and `ltr_photometric` against the model on the GPU."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from linetr_b200 import _native as N, _ops, synthetic as syn
from linetr_b200 import photometric as PH
from linetr_b200.homography_pairs import homography_pairs, warp_pairs

DEV = torch.device("cuda", 0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "photometric.npz")
SHADE = PH.HOMOGRAPHY_PHOTOMETRIC["additive_shade"]
# a pre-truncation value this close to an integer may truncate either way under a 1-ulp change of the blurred mask
TOL = 2e-3
SIZES = [(480, 640), (37, 70), (17, 65), (9, 150), (3, 4), (1, 7), (1, 1)]


def _cv2():
    return pytest.importorskip("cv2")


def _golden():
    return np.load(GOLDEN)


def _builder_ellipses(rng, h, w, n):
    """n ellipses drawn with _py_additive_shade's bounds."""
    out, min_dim = [], min(h, w) / 4
    while len(out) < n:
        ax = int(max(rng.random() * min_dim, min_dim / 5))
        ay = int(max(rng.random() * min_dim, min_dim / 5))
        mr = max(ax, ay)
        out.append((ax, ay, int(rng.integers(mr, w - mr)), int(rng.integers(mr, h - mr)), rng.random() * 90))
    return out


def _compare(got, want, pre=None):
    """(differing bytes, of which near-integer pre-truncation values); raises on any other difference."""
    d = got != want
    if pre is None:
        assert not d.any(), f"{int(d.sum())} bytes differ"
        return 0
    near = np.abs(pre - np.rint(pre)) < TOL
    assert not (d & ~near).any(), f"{int((d & ~near).sum())} bytes differ away from an integer"
    return int(d.sum())


# ------------------------------------------------------------------ CPU: the model
@pytest.mark.parametrize("key,counter", [(0, [0, 0, 0, 0]), (12345, [5, 0, 0, 0]), (2 ** 64 - 1, [2 ** 64 - 2, 7, 3, 1]),
                                         (987654321987, [1234, 2 ** 40, 0, 9]), (2 ** 63 + 5, [0, 0, 2 ** 62, 2 ** 63])])
def test_philox_matches_numpy(key, counter):
    raw = np.random.Philox(key=key, counter=np.array(counter, dtype=np.uint64)).random_raw(12)
    ctr = [np.array(counter, dtype=np.uint64) for _ in range(3)]
    for j in range(3):
        ctr[j][0] = np.uint64((int(counter[0]) + j + 1) % 2 ** 64)
        if int(counter[0]) + j + 1 >= 2 ** 64:
            ctr[j][1] += np.uint64(1)
    got = PH.philox4x64(np.stack(ctr), np.array([key, 0], dtype=np.uint64)).reshape(-1)
    assert np.array_equal(got, raw)


def test_noise_words_are_per_pixel_and_application():
    w0 = PH.noise_words(77, 5, 7, 0)
    assert np.array_equal(w0[2, 3], PH.philox4x64(np.array([2 * 7 + 3, 0, 0, 0], np.uint64), np.array([77, 0], np.uint64)))
    assert not np.array_equal(w0, PH.noise_words(77, 5, 7, 1))
    z = PH.gaussian_from_words(*np.moveaxis(PH.noise_words(5, 300, 300, 0)[..., :2], -1, 0))
    assert abs(z.mean()) < 0.02 and abs(z.std() - 1) < 0.02


def test_sin_table_has_no_rounding_ties():
    """The device recomputes the table with its own sine; no entry is within 1e-6 of a tie at the 7th decimal, so a
    last-bit difference of the sine cannot change an entry."""
    s = np.sin(np.deg2rad(np.arange(451, dtype=np.float64))) * 1e7
    assert np.abs(np.abs(s - np.floor(s)) - 0.5).min() > 1e-6
    assert PH.SIN_TABLE[90] == 1 and PH.SIN_TABLE[0] == 0 and PH.SIN_TABLE[270] == -1


def test_ellipse_model_matches_cv2():
    cv2 = _cv2()
    rng = np.random.default_rng(3)
    n = 0
    for shape in [(480, 640)] * 6 + [(37, 70), (120, 160), (9, 150), (200, 31), (60, 61)]:
        h, w = shape
        for ax, ay, x, y, ang in _builder_ellipses(rng, h, w, 200):
            want = np.zeros(shape, np.uint8)
            cv2.ellipse(want, (x, y), (ax, ay), ang, 0, 360, 255, -1)
            got = PH.ellipse_mask(shape, [[ax, ay, x, y, int(np.rint(ang))]])
            assert np.array_equal(got, want), (shape, ax, ay, x, y, ang, int((got != want).sum()))
            n += 1
    assert n == 2200


def test_ellipse_polygon_is_not_fill_convex_poly():
    """cv2.ellipse's fill is not fillConvexPoly(ellipse2Poly(...)): the model follows the former."""
    cv2 = _cv2()
    want = np.zeros((480, 640), np.uint8)
    cv2.ellipse(want, (300, 200), (110, 47), 33, 0, 360, 255, -1)
    poly = np.zeros_like(want)
    cv2.fillConvexPoly(poly, cv2.ellipse2Poly((300, 200), (110, 47), 33, 0, 360, 5), 255)
    assert (poly != want).any()
    assert np.array_equal(PH.ellipse_mask(want.shape, [[110, 47, 300, 200, 33]]), want)


def test_gaussian_taps_match_cv2():
    cv2 = _cv2()
    for k in range(PH.MIN_KSIZE, PH.MAX_KSIZE + 1, 2):
        assert np.array_equal(PH.gaussian_taps(k), cv2.getGaussianKernel(k, 0, cv2.CV_32F).ravel()), k
    with pytest.raises(N.LtrError):
        PH.gaussian_taps(9)


@pytest.mark.parametrize("h,w", [(480, 640), (37, 70), (9, 150), (1, 7)])
def test_blur_model_matches_cv2(h, w):
    cv2 = _cv2()
    rng = np.random.default_rng(h * w)
    for k in (101, 125, 149):
        m = PH.ellipse_mask((h, w), PH.sample_photometric(1, (h, w), rng, additive_shade=SHADE)["ellipses"][0])
        m = m.astype(np.float32)
        if not m.any():
            m[rng.integers(0, h), rng.integers(0, w)] = 255
        want = cv2.GaussianBlur(m, (k, k), 0)
        assert np.abs(PH.gaussian_blur(m, PH.gaussian_taps(k)) - want).max() < 1e-3


def test_filter3x3_matches_cv2():
    cv2 = _cv2()
    rng = np.random.default_rng(5)
    for t in range(200):
        h, w = (int(v) for v in rng.integers(1, 50, 2))
        v = rng.integers(0, 256, (h, w)).astype(np.uint8)
        k = PH.motion_blur_kernel(rng.uniform(0, 360), rng.uniform(-1, 1))
        assert np.array_equal(PH.filter3x3(v, k), cv2.filter2D(v, -1, k)), (h, w)
    g = _golden()
    for j in range(5):
        v, k = g[f"filter2d/{j}/input"], g[f"filter2d/{j}/kernel"]
        assert np.array_equal(PH.filter3x3(v, k), g[f"filter2d/{j}/output"])


def test_motion_blur_kernel_is_normalised():
    for ang, d in [(0, 0), (45, -1), (90, 1), (200, 0.3)]:
        k = PH.motion_blur_kernel(ang, d)
        assert k.dtype == np.float32 and abs(float(k.sum()) - 1) < 1e-6 and k[1, 1] > 0


def _golden_record(g, name):
    a = g[f"shade/{name}/input"]
    h, w = a.shape
    ell = g[f"shade/{name}/ellipses"]
    rec = PH.sample_photometric(1, (h, w), np.random.default_rng(0), additive_shade=SHADE)
    k = int(g[f"shade/{name}/ksize"])
    rec["ellipses"] = ell[None].astype(np.int32)
    rec["transparency"] = np.array([float(g[f"shade/{name}/transparency"])])
    rec["ksize"] = np.array([k], np.int32)
    rec["taps"] = np.zeros((1, PH.MAX_KSIZE), np.float32)
    rec["taps"][0, :k] = PH.gaussian_taps(k)
    return a[None], rec


GOLDEN_SHADE = ("vga", "qvga", "ragged", "short", "tiny")


def test_model_matches_golden_shade():
    """The model reproduces the reference's additive_shade in the builder's chain; bytes may differ only where the
    pre-truncation value is within TOL of an integer (none do)."""
    g = _golden()
    differ = 0
    for name in GOLDEN_SHADE:
        a, rec = _golden_record(g, name)
        assert np.array_equal(rec["ellipses"][0, :, 4], np.rint(g[f"shade/{name}/angle"]))
        out, st = PH.photometric_host(a, rec, return_stages=True)
        differ += _compare(out[0], g[f"shade/{name}/output"], st["pre"][0])
        if name == "vga":
            assert (out[0] != a[0]).any()
    assert differ == 0


def test_model_blur_matches_golden_blur():
    g = _golden()
    for name in ("qvga", "ragged", "short", "tiny"):
        m, k = g[f"blur/{name}/input"], int(g[f"blur/{name}/ksize"])
        assert np.abs(PH.gaussian_blur(m.astype(np.float32), PH.gaussian_taps(k)) - g[f"blur/{name}/output"]).max() < 1e-3


def test_all_off_is_identity():
    g = np.arange(256, dtype=np.uint8).reshape(1, 16, 16)
    rec = PH.sample_photometric(1, (16, 16), np.random.default_rng(0))
    assert np.array_equal(PH.photometric_host(g, rec), g)
    # the builder's float chain itself is the identity on every grey level
    x = g.astype(np.float32) / np.float32(255) * np.float32(255)
    assert np.array_equal((np.clip(x, 0, 255) / np.float32(255)).astype(np.float64) * 255 // 1, g)
    assert np.array_equal((g / 255. * 255).astype(np.uint8), g)


def test_pointwise_primitives():
    """Each primitive alone, against the formulas of the contract."""
    img = np.arange(256, dtype=np.uint8).reshape(1, 16, 16)
    rec = PH.sample_photometric(1, (16, 16), np.random.default_rng(1), random_brightness={"max_abs_change": 50})
    d = int(rec["brightness"][0, 0])
    assert np.array_equal(PH.photometric_host(img, rec), np.clip(img.astype(int) + d, 0, 255))
    rec = PH.sample_photometric(1, (16, 16), np.random.default_rng(2), random_contrast={"strength_range": [0.3, 1.5]})
    al = rec["contrast"][0, 0]
    want = np.clip(np.float32(127.5) + al * (img.astype(np.float32) - np.float32(127.5)), 0, 255).astype(np.uint8)
    assert np.array_equal(PH.photometric_host(img, rec), want)
    rec = PH.sample_photometric(1, (16, 16), np.random.default_rng(3), additive_speckle_noise={"prob_range": [0.5, 0.6]})
    out = PH.photometric_host(img, rec)
    hit = out != img
    assert 0.3 < hit.mean() < 0.7
    assert ((out[hit] < 64) | (out[hit] > 191)).mean() > 0.5   # Beta(0.5, 0.5) puts most values near 0 and 255


def test_motion_blur_quirk():
    """max_kernel_size other than 3 builds no MotionBlur: the previous augmenter runs a second time."""
    rng = np.random.default_rng(4)
    p = dict(PH.HOMOGRAPHY_PHOTOMETRIC)
    rec = PH.sample_photometric(8, (48, 64), rng, **p)
    assert rec["reps"]["additive_speckle_noise"] == 1 and rec["blur"].any()
    p["motion_blur"] = {"max_kernel_size": 5}
    rec = PH.sample_photometric(8, (48, 64), rng, **p)
    assert rec["reps"]["additive_speckle_noise"] == 2 and not rec["blur"].any()
    assert (rec["speckle_p"][:, 1] > 0).all() and (rec["speckle_p"][:, 0] != rec["speckle_p"][:, 1]).all()
    rec = PH.sample_photometric(2, (48, 64), rng, random_brightness={"max_abs_change": 50},
                                motion_blur={"max_kernel_size": 7})
    assert rec["reps"]["random_brightness"] == 2
    img = np.full((2, 48, 64), 100, np.uint8)
    want = np.clip(np.clip(100 + rec["brightness"][:, 0], 0, 255) + rec["brightness"][:, 1], 0, 255)
    assert np.array_equal(PH.photometric_host(img, rec)[:, 0, 0], want)
    with pytest.raises(N.LtrError):
        PH.sample_photometric(2, (48, 64), rng, motion_blur={"max_kernel_size": 5})
    # a second impulse application draws its own pixels: counter word 1 is the application
    rec = PH.sample_photometric(1, (64, 64), rng, additive_speckle_noise={"prob_range": [0.2, 0.2001]},
                                motion_blur={"max_kernel_size": 4})
    once = dict(rec, reps=dict(rec["reps"], additive_speckle_noise=1))
    z = np.zeros((1, 64, 64), np.uint8)
    assert (PH.photometric_host(z, rec) != 0).sum() > (PH.photometric_host(z, once) != 0).sum()


def test_sample_ranges_and_refusals():
    rng = np.random.default_rng(6)
    rec = PH.sample_photometric(500, (480, 640), rng, **PH.HOMOGRAPHY_PHOTOMETRIC)
    assert np.abs(rec["brightness"][:, 0]).max() <= 50 and (rec["brightness"][:, 1] == 0).all()
    assert (rec["contrast"][:, 0] >= 0.3).all() and (rec["contrast"][:, 0] <= 1.5).all()
    assert (rec["noise_std"][:, 0] >= 0).all() and (rec["noise_std"][:, 0] <= 10).all()
    assert (rec["speckle_p"][:, 0] >= 0).all() and (rec["speckle_p"][:, 0] <= 0.0035).all()
    assert 0.4 < rec["blur"].mean() < 0.6
    k = rec["ksize"]
    assert (k % 2 == 1).all() and k.min() == 101 and k.max() == 149
    assert (rec["transparency"] >= -0.5).all() and (rec["transparency"] <= 0.5).all()
    ell = rec["ellipses"]
    assert ell.shape == (500, 20, 5)
    mr = ell[..., :2].max(-1)
    assert (ell[..., :2] >= 24).all() and (ell[..., :2] < 120).all()
    assert (ell[..., 2] >= mr).all() and (ell[..., 2] < 640 - mr).all()
    assert (ell[..., 3] >= mr).all() and (ell[..., 3] < 480 - mr).all()
    assert (ell[..., 4] >= 0).all() and (ell[..., 4] <= 90).all()
    for i in (0, 17):
        assert np.array_equal(rec["taps"][i, :k[i]], PH.gaussian_taps(k[i])) and not rec["taps"][i, k[i]:].any()
    assert len(np.unique(rec["key"])) == 500
    # the ellipse bounds are never empty on a non-empty image (max_rad < min(h, w) / 4); an empty one is refused
    PH.sample_photometric(1, (1, 1), rng, additive_shade=SHADE)
    with pytest.raises(N.LtrError):
        PH.sample_photometric(1, (0, 640), rng, additive_shade=SHADE)
    with pytest.raises(N.LtrError):
        PH.sample_photometric(1, (480, 640), rng, additive_shade={"kernel_size_range": [250, 350]})
    with pytest.raises(N.LtrError):
        PH.sample_photometric(1, (480, 640), rng, GaussianBlur={"sigma": 1})


def test_constants_agree():
    hdr = open(os.path.join(ROOT, "include", "linetr_b200.h")).read()
    cu = open(os.path.join(ROOT, "linetr_b200", "csrc", "photometric.cuh")).read()
    assert int(re.search(r"#define LTR_PHOTOMETRIC_PARAMS (\d+)", hdr).group(1)) == PH.N_PARAMS == N.PHOTOMETRIC_PARAMS
    assert int(re.search(r"#define LTR_PHOTOMETRIC_MAX_KSIZE (\d+)", hdr).group(1)) == PH.MAX_KSIZE
    assert int(re.search(r"PH_NPARAM = (\d+)", cu).group(1)) == PH.N_PARAMS
    for nm in ("BRIGHT", "CONTRAST", "NOISE", "SPECKLE", "BLUR", "KERNEL", "SHADE", "TRANSPARENCY", "KSIZE", "KEY_LO",
               "KEY_HI", "N_ELLIPSES"):
        assert int(re.search(rf"PH_P_{nm} = (\d+)", cu).group(1)) == getattr(PH, f"P_{nm}"), nm


# ------------------------------------------------------------------ GPU: the kernel against the model
def _run(gray, rec):
    got = PH.photometric_augment(torch.from_numpy(gray).to(DEV), rec).cpu().numpy()
    want, st = PH.photometric_host(gray, rec, return_stages=True)
    return got, want, st


def _check(gray, rec):
    got, want, st = _run(gray, rec)
    n = 0
    for i in range(len(gray)):
        n += _compare(got[i], want[i], st["pre"][i] if rec["shade"] else None)
    return n


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", SIZES)
def test_kernel_matches_model(h, w):
    gray, _ = syn.make_warp_images(h + 3 * w, 3 if h * w > 1000 else 6, h, w)
    rng = np.random.default_rng(h * 1000 + w)
    p = dict(PH.HOMOGRAPHY_PHOTOMETRIC)
    if h * w < 1000:   # strong noise so that the small images exercise every primitive
        p.update(additive_speckle_noise={"prob_range": [0.1, 0.3]})
    rec = PH.sample_photometric(len(gray), (h, w), rng, **p)
    rec["blur"][:] = True
    rec["blur_kernel"][:] = [PH.motion_blur_kernel(a, d) for a, d in zip(rng.uniform(0, 360, len(gray)),
                                                                         rng.uniform(-1, 1, len(gray)))]
    assert _check(gray, rec) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("prim", ["random_brightness", "random_contrast", "additive_gaussian_noise",
                                  "additive_speckle_noise", "motion_blur", "additive_shade", "quirk"])
def test_each_primitive_matches_model(prim):
    gray, _ = syn.make_warp_images(31, 2, 96, 130)
    if prim == "quirk":
        p = {"additive_speckle_noise": {"prob_range": [0.05, 0.1]}, "motion_blur": {"max_kernel_size": 5}}
    elif prim == "additive_speckle_noise":
        p = {prim: {"prob_range": [0.05, 0.1]}}
    else:
        p = {prim: PH.HOMOGRAPHY_PHOTOMETRIC[prim]}
    rec = PH.sample_photometric(2, (96, 130), np.random.default_rng(8), **p)
    if prim == "motion_blur":
        rec["blur"][:] = True
        rec["blur_kernel"][:] = PH.motion_blur_kernel(30, 0.4)
    got, want, st = _run(gray, rec)
    for i in range(2):
        _compare(got[i], want[i], st["pre"][i] if rec["shade"] else None)
    assert (got != gray).any()


@pytest.mark.gpu
def test_all_off_and_in_place():
    gray, _ = syn.make_warp_images(41, 2, 50, 60)
    rec = PH.sample_photometric(2, (50, 60), np.random.default_rng(0))
    assert np.array_equal(PH.photometric_augment(torch.from_numpy(gray).to(DEV), rec).cpu().numpy(), gray)
    rec = PH.sample_photometric(2, (50, 60), np.random.default_rng(1), **PH.HOMOGRAPHY_PHOTOMETRIC)
    t = torch.from_numpy(gray).to(DEV)
    dv = {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in
          (("params", PH.params_array(rec)), ("ellipses", rec["ellipses"]), ("taps", rec["taps"]))}
    ws = torch.empty(N.photometric_workspace_bytes(2, 50, 60), dtype=torch.uint8, device=DEV)
    _ops.photometric(t, t, PH.params_array(rec), dv["params"], dv["ellipses"], dv["taps"], ws)
    want, st = PH.photometric_host(gray, rec, return_stages=True)
    for i in range(2):
        _compare(t.cpu().numpy()[i], want[i], st["pre"][i])


@pytest.mark.gpu
def test_deterministic_and_independent_noise():
    h, w = 64, 80
    gray = np.full((4, h, w), 128, np.uint8)
    p = {"additive_gaussian_noise": {"stddev_range": [5, 5.0001]}, "additive_speckle_noise": {"prob_range": [0.01, 0.02]}}
    rec = PH.sample_photometric(4, (h, w), np.random.default_rng(2), **p)
    g = torch.from_numpy(gray).to(DEV)
    a, b = PH.photometric_augment(g, rec).cpu().numpy(), PH.photometric_augment(g, rec).cpu().numpy()
    assert np.array_equal(a, b)
    assert np.array_equal(a, PH.photometric_host(gray, rec))
    d = a.astype(np.float64) - 128
    for i in range(4):
        for j in range(i):
            assert abs(np.corrcoef(d[i].ravel(), d[j].ravel())[0, 1]) < 0.05


@pytest.mark.gpu
def test_kernel_matches_golden():
    g = _golden()
    for name in GOLDEN_SHADE:
        a, rec = _golden_record(g, name)
        got = PH.photometric_augment(torch.from_numpy(a).to(DEV), rec).cpu().numpy()
        _, st = PH.photometric_host(a, rec, return_stages=True)
        _compare(got[0], g[f"shade/{name}/output"], st["pre"][0])
    for j in range(5):
        v, k = g[f"filter2d/{j}/input"], g[f"filter2d/{j}/kernel"]
        rec = PH.sample_photometric(1, v.shape, np.random.default_rng(0))
        rec["blur"][:] = True
        rec["blur_kernel"][0] = k
        got = PH.photometric_augment(torch.from_numpy(v[None]).to(DEV), rec).cpu().numpy()
        assert np.array_equal(got[0], g[f"filter2d/{j}/output"])


@pytest.mark.gpu
def test_photometric_homography_pairs():
    gray, colour = syn.make_warp_images(51, 2, 120, 160)
    g, c = torch.from_numpy(gray).to(DEV), torch.from_numpy(colour).to(DEV)
    hp = dict(allow_artifacts=True, translation_overflow=0.1)
    image0, warped, mask, H = PH.photometric_homography_pairs(g, c, 3, np.random.default_rng(9), **hp)
    w_ref, m_ref, H_ref = homography_pairs(g, c, 3, np.random.default_rng(9), **hp)
    assert np.array_equal(H, H_ref)
    assert torch.equal(mask, m_ref)
    assert torch.equal(warped, warp_pairs(image0, image0[..., None], np.arange(6), H)[0])
    rng = np.random.default_rng(9)
    from linetr_b200.homography_pairs import sample_homographies
    sample_homographies(6, (120, 160), rng, **hp)
    rec = PH.sample_photometric(6, (120, 160), rng, **PH.HOMOGRAPHY_PHOTOMETRIC)
    want, st = PH.photometric_host(gray[np.arange(6) // 3], rec, return_stages=True)
    got = image0.cpu().numpy()
    for i in range(6):
        _compare(got[i], want[i], st["pre"][i])
    assert not torch.equal(image0[0], image0[1])   # every pair draws its own augmentation


@pytest.mark.gpu
def test_bad_input_raises_before_launch():
    gray, _ = syn.make_warp_images(61, 2, 40, 50)
    g = torch.from_numpy(gray).to(DEV)
    rec = PH.sample_photometric(2, (40, 50), np.random.default_rng(0), **PH.HOMOGRAPHY_PHOTOMETRIC)
    ph = PH.params_array(rec)
    dv = {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in
          (("params", ph), ("ellipses", rec["ellipses"]), ("taps", rec["taps"]))}
    out = torch.zeros_like(g)
    ws = torch.empty(N.photometric_workspace_bytes(2, 40, 50), dtype=torch.uint8, device=DEV)
    torch.cuda.synchronize()
    lib = N.load()

    def call(params_host=ph, n_params=N.PHOTOMETRIC_PARAMS, h=40, w=50, ws_bytes=ws.numel(), src=g, taps=dv["taps"]):
        return lib.ltr_photometric(_ops._ptr(src), _ops._ptr(out), 2, h, w, params_host.ctypes.data_as(C.c_void_p),
                                   _ops._ptr(dv["params"]), n_params, _ops._ptr(dv["ellipses"]), 20,
                                   _ops._ptr(taps), _ops._ptr(ws), ws_bytes, 0, None)

    n0 = N.launch_count()
    assert call(n_params=27) == -1
    assert call(h=0) == -4 and call(w=40000) == -4
    assert call(ws_bytes=100) == -3
    assert call(src=None) == -1 and call(taps=None) == -1
    for slot, v in ((PH.P_KSIZE, 150), (PH.P_KSIZE, 151), (PH.P_BRIGHT, 3), (PH.P_SPECKLE + 1, 1.5),
                    (PH.P_N_ELLIPSES, 21), (PH.P_TRANSPARENCY, np.nan), (PH.P_KEY_HI, 2.0 ** 32)):
        bad = ph.copy()
        bad[1, slot] = v
        assert call(params_host=bad) == -1, (slot, v)
    assert N.launch_count() == n0
    assert not out.any()
    with pytest.raises(N.LtrError):
        PH.photometric_augment(g, PH.sample_photometric(3, (40, 50), np.random.default_rng(0)))
    with pytest.raises(N.LtrError):
        PH.photometric_augment(g.cpu(), rec)
    bad = dict(rec, ellipses=rec["ellipses"].copy())
    bad["ellipses"][0, 0, 2] = 0
    with pytest.raises(N.LtrError):
        PH.photometric_augment(g, bad)
    assert call() == 0
    torch.cuda.synchronize()
