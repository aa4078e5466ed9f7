"""Homography image pairs (`homography_pairs`): the homography sampler, the numpy models of the warp and the mask
against OpenCV, and `ltr_warp_pairs` against the models and the OpenCV golden fixture."""
import os

import numpy as np
import pytest
import torch
from scipy import stats

from linetr_b200 import _native as N, _ops, engine, synthetic as syn
from linetr_b200.homography_pairs import (apply_valid_masks, get_perspective_transform, homography_pairs,
                                          sample_homographies, valid_mask_host, warp_pairs, warp_perspective_host)

DEV = torch.device("cuda", 0)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "homography_pairs.npz")
SIZES = [(480, 640), (60, 80), (37, 70), (17, 65), (16, 100), (9, 150), (5, 300), (3, 4), (1, 1)]


def _cv2():
    return pytest.importorskip("cv2")


def _special_maps(h, w):
    """Identity, a map that sends the whole frame outside, and one whose w crosses 0 inside the frame."""
    outside = np.array([[1., 0., 3.0 * w], [0., 1., 0.], [0., 0., 1.]])
    cross = np.array([[1., 0.1, 0.], [0.05, 1., 0.], [-2.0 / w, 0.3 / h, 1.]])   # inverse map, w = 0 near x = w/2
    return [np.eye(3), outside, np.linalg.inv(cross)]


def _cases(h, w, seed):
    rng = np.random.default_rng(seed)
    Hs = list(sample_homographies(2, (h, w), rng)[0]) + list(
        sample_homographies(2, (h, w), rng, allow_artifacts=True, translation_overflow=0.3)[0])
    return Hs + _special_maps(h, w)


def _builder_mask(cv2, colour, H):
    h, w = colour.shape[:2]
    wc = cv2.warpPerspective(colour.astype(np.float32), H, (w, h))
    m = np.ones((h, w), np.uint8)
    m[(wc == 0).all(-1) if wc.ndim == 3 else wc == 0] = 0
    return cv2.erode(m, np.ones((5, 5), np.uint8))


# ------------------------------------------------------------------ CPU: the models against OpenCV
@pytest.mark.parametrize("h,w", SIZES)
def test_warp_model_matches_cv2(h, w):
    cv2 = _cv2()
    gray, colour = syn.make_warp_images(h * 7 + w, 2, h, w)
    for k, H in enumerate(_cases(h, w, h + w)):
        M = np.linalg.inv(H)
        for src in (gray[k % 2], colour[k % 2]):
            want = cv2.warpPerspective(src, M, (w, h), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP)
            got = warp_perspective_host(src, M)
            assert np.array_equal(got, want), f"case {k}: {(got != want).sum()} pixels differ"
            # the builder's call on sampled homographies: cv2 inverts H itself (on the hand-made maps, whose w
            # crosses 0 in the frame, its inverse and np.linalg.inv's can differ in the last bit)
            if k < 4:
                assert np.array_equal(got, cv2.warpPerspective(src, H, (w, h)))


def test_warp_model_covers_edge_maps():
    h, w = 60, 80
    img = np.full((h, w), 200, np.uint8)
    ident, outside, cross = _special_maps(h, w)
    assert np.array_equal(warp_perspective_host(img, ident), img)
    assert not warp_perspective_host(img, np.linalg.inv(outside)).any()
    W = np.linalg.inv(cross)[2] @ np.stack([np.arange(w), np.full(w, h / 2), np.ones(w)])
    assert W.min() < 0 < W.max()   # the map's w changes sign inside the frame


@pytest.mark.parametrize("h,w", [(60, 80), (9, 150), (5, 300), (37, 70), (4, 3), (3, 4), (2, 2), (1, 7)])
def test_valid_mask_model_matches_builder(h, w):
    cv2 = _cv2()
    gray, colour = syn.make_warp_images(h * 11 + w, 2, h, w)
    colour[1, : max(h // 2, 1), : max(w // 2, 1)] = 0
    for k, H in enumerate(_cases(h, w, 3 * h + w)):
        c = colour[k % 2]
        M = np.linalg.inv(H)
        assert np.array_equal(valid_mask_host(c, M), _builder_mask(cv2, c, H)), f"case {k}"
        assert np.array_equal(valid_mask_host(gray[k % 2], M), _builder_mask(cv2, gray[k % 2][..., None], H))


def test_perspective_transform_matches_cv2():
    cv2 = _cv2()
    rng = np.random.default_rng(3)
    base = np.array([[-1., -1.], [-1., 1.], [1., 1.], [1., -1.]], np.float32)
    src = (base + rng.uniform(-0.3, 0.3, (200, 4, 2))).astype(np.float32)
    dst = (0.5 * base + rng.uniform(-0.4, 0.4, (200, 4, 2))).astype(np.float32)
    got = get_perspective_transform(src, dst)
    for g, s, d in zip(got, src, dst):
        want = cv2.getPerspectiveTransform(s, d)
        assert np.abs(g - want).max() <= 1e-12 * np.abs(want).max()


# ------------------------------------------------------------------ CPU: the sampler
def _patch_corners(H_inv, h, w):
    """Corners of the sampled patch in [0, 1] coordinates (the sampler's pts2): H_inv maps image 1's corners there."""
    c = np.array([[0., 0., 1.], [0., h, 1.], [w, h, 1.], [w, 0., 1.]])
    q = np.einsum("pij,cj->pci", H_inv, c)
    return q[..., :2] / q[..., 2:] / np.array([w, h])


@pytest.mark.parametrize("params", [{}, {"n_scales": 3, "n_angles": 7}, {"max_angle": 0.3, "patch_ratio": 0.7}])
def test_sampled_patches_stay_inside(params):
    h, w = 480, 640
    H, Hi = sample_homographies(2000, (h, w), np.random.default_rng(5), **params)
    pts = _patch_corners(Hi, h, w)
    assert pts.min() >= -1e-6 and pts.max() < 1 + 1e-6
    assert np.abs(H @ Hi - np.eye(3)).max() < 1e-9


def test_sampled_homographies_invert():
    H, Hi = sample_homographies(500, (240, 320), np.random.default_rng(6), allow_artifacts=True,
                                translation_overflow=0.2)
    assert np.abs(H @ Hi - np.eye(3)).max() < 1e-9
    assert np.array_equal(H, sample_homographies(500, (240, 320), np.random.default_rng(6), allow_artifacts=True,
                                                 translation_overflow=0.2)[0])


def test_everything_off_is_the_centred_crop():
    h, w = 480, 640
    H, Hi = sample_homographies(3, (h, w), np.random.default_rng(0), perspective=False, scaling=False, rotation=False,
                                translation=False)
    want = np.array([[2., 0., -w / 2], [0., 2., -h / 2], [0., 0., 1.]])
    assert np.abs(H - want).max() < 1e-9 and np.abs(Hi - np.linalg.inv(want)).max() < 1e-12


def _ks(x):
    return stats.kstest(x, stats.truncnorm(-2, 2).cdf).pvalue


def test_perturbation_marginals_are_truncated_normals():
    h, w, n, margin = 480, 640, 4000, 0.25
    rng = np.random.default_rng(7)
    _, Hi = sample_homographies(n, (h, w), rng, scaling=False, rotation=False, translation=False)
    pts = _patch_corners(Hi, h, w)
    amp = 0.1 / 2   # perspective_amplitude_x / y
    hl, pd, hr = pts[:, 0, 0] - margin, pts[:, 0, 1] - margin, pts[:, 2, 0] - (1 - margin)
    for v in (hl, pd, hr):
        assert _ks(v / amp) > 1e-3
    assert np.allclose(pts[:, 1, 1], 1 - margin - pd, atol=1e-6)   # the second corner moves by -pd
    _, Hi = sample_homographies(n, (h, w), rng, perspective=False, rotation=False, translation=False)
    pts = _patch_corners(Hi, h, w)
    scale = (pts[:, 2, 0] - pts[:, 0, 0]) / 0.5
    drawn = scale[np.abs(scale - 1) > 1e-6]   # the candidate scale 1 is picked 1 time in 6
    assert abs(len(drawn) / n - 5 / 6) < 0.03
    assert _ks((drawn - 1) / (0.1 / 2)) > 1e-3


def test_apply_valid_masks_filters_keypoints():
    h, w = 40, 50
    mask = np.zeros((h, w), np.uint8)
    mask[:, 20:] = 1
    kp = torch.tensor([[5.0, 3.0], [20.0, 10.0], [19.99, 10.0], [49.5, 39.9], [25.2, 0.0]])
    im = {"keypoints": kp, "scores": torch.arange(5.0), "descriptors": torch.arange(5.0)[None].repeat(4, 1),
          "image_shape": (1, 1, h, w)}
    out, same = apply_valid_masks([im, im], [torch.from_numpy(mask), None])
    assert out["keypoints"].tolist() == kp[[1, 3, 4]].tolist()
    assert out["scores"].tolist() == [1.0, 3.0, 4.0]
    assert out["descriptors"].shape == (4, 3) and out["descriptors"][0].tolist() == [1.0, 3.0, 4.0]
    assert np.array_equal(out["valid_mask"], mask) and "valid_mask" not in same and im["keypoints"] is kp


# ------------------------------------------------------------------ GPU
def _dev(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in arrays]


@pytest.mark.gpu
def test_warp_pairs_matches_golden():
    z = np.load(GOLDEN)
    for case in sorted({k.split("/")[0] for k in z.files}):
        g, c = _dev(z[f"{case}/gray"], z[f"{case}/colour"])
        warped, mask = warp_pairs(g, c, z[f"{case}/src_index"], z[f"{case}/H"])
        torch.cuda.synchronize()
        assert np.array_equal(warped.cpu().numpy(), z[f"{case}/warped"]), case
        assert np.array_equal(mask.cpu().numpy(), z[f"{case}/mask"]), case


def _check_against_models(gray, colour, src, H, warped, mask):
    w_np, m_np = warped.cpu().numpy(), mask.cpu().numpy()
    for p in range(len(src)):
        M = np.linalg.inv(H[p])
        assert np.array_equal(w_np[p], warp_perspective_host(gray[src[p]], M)), f"pair {p}: grey"
        assert np.array_equal(m_np[p], valid_mask_host(colour[src[p]], M)), f"pair {p}: mask"


@pytest.mark.gpu
def test_warp_pairs_matches_models_vga():
    h, w, n, P = 480, 640, 16, 256
    gray, colour = syn.make_warp_images(1, n, h, w)
    rng = np.random.default_rng(8)
    src = rng.integers(0, n, P)   # sources are reused across pairs
    H = np.concatenate([sample_homographies(P // 2, (h, w), rng)[0],
                        sample_homographies(P // 2, (h, w), rng, allow_artifacts=True, translation_overflow=0.2)[0]])
    warped, mask = warp_pairs(*_dev(gray, colour), src, H)
    _check_against_models(gray, colour, src, H, warped, mask)


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", SIZES[1:])
def test_warp_pairs_matches_models_ragged(h, w):
    n = 3
    gray, colour = syn.make_warp_images(h + 13 * w, n, h, w)
    Hs = _cases(h, w, 2 * h + w)
    src = np.arange(len(Hs)) % n
    H = np.stack(Hs)
    warped, mask = warp_pairs(*_dev(gray, colour), src, H)
    _check_against_models(gray, colour, src, H, warped, mask)
    # grey-only data: the grey image stands in for the colour image (C = 1)
    g = _dev(gray)[0]
    _, mask1 = warp_pairs(g, g[..., None], src, H)
    _check_against_models(gray, gray, src, H, warped, mask1)


@pytest.mark.gpu
def test_warp_pairs_rejects_bad_input():
    gray, colour = syn.make_warp_images(2, 2, 20, 30)
    g, c = _dev(gray, colour)
    H = np.repeat(np.eye(3)[None], 2, 0)
    with pytest.raises(N.LtrError, match="no CPU fallback"):
        warp_pairs(torch.from_numpy(gray), c, [0, 1], H)
    with pytest.raises(N.LtrError, match="src_index"):
        warp_pairs(g, c, [0, 2], H)
    with pytest.raises(N.LtrError, match="H must be"):
        warp_pairs(g, c, [0, 1, 1], H)
    with pytest.raises(N.LtrError, match="not invertible"):
        warp_pairs(g, c, [0, 1], np.zeros((2, 3, 3)))
    with pytest.raises(N.LtrError, match="colour"):
        warp_pairs(g, c[:, :, :10], [0, 1], H)
    with pytest.raises(N.LtrError, match="contiguous"):
        warp_pairs(g.float(), c, [0, 1], H)
    # the native entry's own checks, before any launch
    out = [torch.zeros((2, 20, 30), dtype=torch.uint8, device=DEV) for _ in range(2)]
    idx_d = torch.tensor([0, 5], dtype=torch.int32, device=DEV)
    M = torch.from_numpy(np.eye(3).reshape(1, 9).repeat(2, 0)).to(DEV)
    with pytest.raises(N.LtrError, match=r"code -1\).*src_index\[1\] = 5"):
        _ops.warp_pairs(g, c, np.array([0, 5], np.int32), idx_d, M, *out)
    with pytest.raises(N.LtrError, match=r"code -4\).*channels"):
        _ops.warp_pairs(g, c[..., :2].contiguous(), np.array([0, 1], np.int32), idx_d, M, *out)
    torch.cuda.synchronize()
    assert not out[0].any() and not out[1].any()   # nothing was launched
    warped, mask = warp_pairs(g, c, [], np.zeros((0, 3, 3)))
    assert warped.shape == (0, 20, 30) and mask.shape == (0, 20, 30)


@pytest.mark.gpu
def test_dots_land_at_H_p_and_masked_lines_are_dropped():
    h, w = 480, 640
    rng = np.random.default_rng(9)
    gx, gy = np.meshgrid(np.arange(200, 441, 40), np.arange(150, 331, 36))   # spaced so that windows do not overlap
    pts = np.stack([gx.ravel(), gy.ravel()], 1).astype(np.float64) + rng.integers(-3, 4, (gx.size, 2))
    gray = np.zeros((1, h, w), np.uint8)
    for x, y in pts.astype(int):
        gray[0, y - 1:y + 2, x - 1:x + 2] = 255
    colour = np.repeat(np.maximum(gray, 1)[..., None], 3, -1)   # no black source pixel
    warped, mask, H = homography_pairs(*_dev(gray, colour), 1, rng, patch_ratio=0.9, max_angle=0.3)
    img = warped[0].cpu().numpy().astype(np.float64)
    q = np.einsum("ij,nj->ni", H[0], np.concatenate([pts, np.ones((len(pts), 1))], 1))
    q = q[:, :2] / q[:, 2:]
    for x, y in q:
        y0, x0 = int(round(y)) - 4, int(round(x)) - 4
        win = img[y0:y0 + 9, x0:x0 + 9]
        yy, xx = np.mgrid[y0:y0 + 9, x0:x0 + 9]
        assert win.sum() > 0 and np.hypot((win * xx).sum() / win.sum() - x, (win * yy).sum() / win.sum() - y) < 1.0
    assert mask.all()   # without artifacts the frame maps inside the source

    # key lines of image 1 outside the valid mask are dropped by match_images
    from tests.test_image_pairs import _model
    m = np.ones((h, w), np.uint8)
    m[:, : w // 2] = 0
    im0, im1 = (syn.image_to(v, DEV) for v in syn.make_image_pair(4, 60, 300))
    model, _ = _model()
    eng = engine.PairEngine(model, DEV)
    (im1m,) = apply_valid_masks([im1], [torch.from_numpy(m).to(DEV)])
    assert (im1m["keypoints"][:, 0] >= w // 2).all() and len(im1m["keypoints"]) < len(im1["keypoints"])
    full, cut = eng.match_images([im0], [im1]), eng.match_images([im0], [im1m])
    k_full, k_cut = np.asarray(full.klines1[0]).reshape(-1, 2, 2), np.asarray(cut.klines1[0]).reshape(-1, 2, 2)
    assert 0 < len(k_cut) < len(k_full)
    x = np.floor(k_cut[..., 0]).astype(int)
    assert ((x[:, 0] >= w // 2) | (x[:, 1] >= w // 2)).all()   # every kept line has an end point in the mask
