"""The image-level front-end: `ltr_tokenize_batch` (many images per tokeniser call), its host preparation
(line_process.prepare_tokenizer_batch) and `PairEngine.match_images` (line and point matches of many image
pairs from detector + SuperPoint outputs), against the per-image call sequence of models/matching.py:18-86."""
import os
import sys

import numpy as np
import pytest
import torch

from linetr_b200 import _native as N
from linetr_b200 import engine, line_process as LP, synthetic as syn
from linetr_b200.match_io import dense_to_indices
from linetr_b200.line_transformer import LineTransformer
from linetr_b200.nn_matcher import adjacency_to_csr
from tests import helpers as H
from tests.test_tokenizer import CFGS, fake_lines, fake_superpoint

DIST_TOL = 2e-5
DEV = torch.device("cuda", 0)


def _cfg(extra, shape, auto=False):
    return LP.tokenizer_config({**LineTransformer.default_config, **extra}, shape, auto)


def _glue(lines, shape, sp, extra):
    """The per-image tokeniser: LineTransformer.preprocess with the settings `extra`."""
    m = LineTransformer({"mode": "train", **extra})
    return m.preprocess(lines, shape, sp, None)


# image set of the CPU preparation test: CFGS[0] and CFGS[2] (both T = 21) plus an image of another size and spacing
MIXED = [(7, 60, 640, 480, CFGS[0]), (7, 60, 640, 480, CFGS[2]), (11, 40, 800, 600, {"token_distance": 10})]


# ------------------------------------------------------------------ CPU
def test_batch_preparation_equals_cpu_glue():
    specs = [(fake_lines(s, n, w, h), (1, 1, h, w), None) for s, n, w, h, _ in MIXED]
    host = LP.prepare_tokenizer_batch(specs, [_cfg(c, sh) for (_, sh, _), (*_, c) in zip(specs, MIXED)])
    assert host.n_images == 3 and host.max_tokens == 21 and host.split
    assert len(set(host.token_distance.tolist())) == 2
    for i, (s, n, w, h, c) in enumerate(MIXED):
        want = _glue(fake_lines(s, n, w, h), (1, 1, h, w), fake_superpoint(s, h, w), c)
        A = want["mat_klines2sublines"][0].numpy()
        K, S = A.shape
        k0, k1, r0, r1 = host.cuk[i], host.cuk[i + 1], host.cu_lines[i], host.cu_lines[i + 1]
        assert (k1 - k0, r1 - r0) == (K, S)
        csr = adjacency_to_csr(A)
        assert np.array_equal(host.sub0[k0:k1 + 1] - r0, csr)
        assert np.array_equal(host.sub2line[r0:r1] - k0, A.argmax(axis=0))
        assert np.array_equal(host.line_image[k0:k1], np.full(K, i))
        # real tokens per key line = the glue's mask summed over the key line's sublines
        real = want["mask_sublines"][0, :, 1:, 0].numpy().sum(axis=1)
        assert np.array_equal(host.n_tok[k0:k1], np.add.reduceat(real, csr[:-1]).astype(np.int32))
        assert torch.equal(torch.from_numpy(host.klines[i]).float(), want["klines"][0])      # clipped in place
        assert torch.equal(torch.from_numpy(host.length_klines[i]).float(), want["length_klines"][0])
        assert torch.equal(torch.from_numpy(host.angles[i]).float(), want["angles"][0])


def test_batch_preparation_rejects_malformed_input():
    specs = [(fake_lines(7, 20), (1, 1, 480, 640), None)] * 2
    with pytest.raises(N.LtrError, match="max_tokens"):
        LP.prepare_tokenizer_batch(specs, [_cfg({}, specs[0][1]), _cfg(CFGS[1], specs[0][1])])
    eng = engine.PairEngine(LineTransformer({"mode": "train"}), "cuda:0")
    a, b = syn.make_image_pair(1, 10, 10)
    with pytest.raises(N.LtrError, match="side-1"):
        eng.match_images([a, a], [b])


def test_tokenizer_config_follows_matching():
    cfg = _cfg({}, (1, 1, 600, 800), auto=True)
    assert cfg["min_length"] == 20 and cfg["token_distance"] == 10 and cfg["max_tokens"] == 21
    cfg = _cfg({}, (1, 1, 480, 640), auto=True)
    assert cfg["min_length"] == 16 and cfg["token_distance"] == 8


# ------------------------------------------------------------------ GPU
_models = {}


def _model(tag="synthetic"):
    if tag not in _models:
        if tag == "synthetic":
            m = LineTransformer({"mode": "train"})
            sd = syn.make_state_dict(0, 1)
            m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
        else:
            if H.shipped_weights_path() is None:
                pytest.skip("shipped checkpoint not available")
            m = LineTransformer({"max_keylines": -1, "min_length": 16, "token_distance": 8, "nn_threshold": 0.8,
                                 "weights_path": H.shipped_weights_path()})
            sd = {k: v.numpy() for k, v in m.state_dict().items()}
        _models[tag] = (m.eval().to(DEV), sd)
    return _models[tag]


def _dev(im):
    return syn.image_to(im, DEV)


@pytest.mark.gpu
def test_tokenize_batch_equals_per_image_gpu_calls():
    """Sizes 640x480, 320x240 and 800x600 (token_distance 8, 8, 10 under auto_min_length), one image without key
    lines, vertical and split lines: the batch equals per-image GPU calls bit for bit."""
    model, _ = _model()
    eng = engine.PairEngine(model, DEV)
    sets = [(7, 60, 640, 480), (5, 30, 320, 240), (9, 0, 800, 600), (11, 50, 800, 600)]
    images = [{"klines": fake_lines(s, n, w, h) if n else [], "image_shape": (1, 1, h, w),
               **{k: v.to(DEV) for k, v in fake_superpoint(s, h, w).items()}} for s, n, w, h in sets]
    batch = eng.tokenize_images(images)
    assert batch.sub_off is not None and batch.n_images == 4
    assert batch.cu_lines[3] == batch.cu_lines[2]          # the image without key lines is an empty range
    fields = {"sublines": batch.sublines, "resp_sublines": batch.resp, "angle_sublines": batch.angle,
              "pnt_sublines": batch.pnt, "desc_sublines": batch.desc, "score_sublines": batch.score}
    for i, im in enumerate(images):
        cfg = LP.tokenizer_config(model.config, im["image_shape"], True)
        want = _glue(im["klines"], im["image_shape"], im, {k: cfg[k] for k in ("min_length", "token_distance")})
        r0, r1 = int(batch.cu_lines[i]), int(batch.cu_lines[i + 1])
        if r0 == r1:
            assert "sublines" not in want
            continue
        for k, t in fields.items():
            assert torch.equal(t[r0:r1], want[k][0]), (i, k)
        A = want["mat_klines2sublines"][0].cpu().numpy()
        k0, k1 = int(batch.cuk[i]), int(batch.cuk[i + 1])
        assert np.array_equal(batch.sub_off[k0:k1 + 1] - r0, adjacency_to_csr(A))


@pytest.mark.gpu
def test_tokenize_batch_against_reference_fixture():
    """tests/golden/tokenizer_outputs.npz (the reference tokeniser's outputs): cases c0 and c2 in one batch, c1 alone."""
    model, _ = _model()
    eng = engine.PairEngine(model, DEV)
    sp = {k: v.to(DEV) for k, v in fake_superpoint(7).items()}
    for group in ([0, 2], [1]):
        specs = [(fake_lines(7, 60), (1, 1, 480, 640), None) for _ in group]
        host = LP.prepare_tokenizer_batch(specs, [_cfg(CFGS[ci], (1, 1, 480, 640)) for ci in group])
        batch = eng.tokenize_prepared(host, [sp] * len(group))
        for j, ci in enumerate(group):
            ref, (rows, real, pad) = H.tokenizer_fixture(ci)
            r0, r1 = int(batch.cu_lines[j]), int(batch.cu_lines[j + 1])
            got = {"sublines": batch.sublines, "resp_sublines": batch.resp, "angle_sublines": batch.angle,
                   "pnt_sublines": batch.pnt, "score_sublines": batch.score}
            for k, t in got.items():
                assert np.array_equal(t[r0:r1].cpu().numpy(), ref[k][0]), (ci, k)
            assert np.array_equal(host.klines[j].astype(np.float32), ref["klines"][0])
            k0, k1 = int(host.cuk[j]), int(host.cuk[j + 1])
            assert np.array_equal(host.sub0[k0:k1 + 1] - r0, adjacency_to_csr(ref["mat_klines2sublines"][0]))
            desc = batch.desc[r0:r1].cpu().numpy()
            mask = ref["mask_sublines"][0, :, 1:, 0] > 0
            assert np.abs(desc[mask][rows] - real).max() < 2e-6
            assert np.abs(desc[~mask] - pad).max() < 2e-6


def _ragged_pairs():
    """P = 5 synthetic pairs of different sizes; pair 1's side 1 has no key lines, pair 3 has no keypoints, pair 4
    carries the real SuperPoint descriptors of tests/golden/plumbing_pnt.npz."""
    npz, _ = H.plumbing()
    out = []
    for p, (nl, npnt, w, h) in enumerate([(40, 300, 640, 480), (30, 200, 640, 480), (25, 150, 320, 240),
                                         (45, 0, 800, 600), (35, 100, 640, 480)]):
        a, b = syn.make_image_pair(100 + p, nl, npnt, w, h)
        if p == 1:
            b["klines"] = []
        if p == 4:
            a["descriptors"] = torch.from_numpy(npz["p0_desc_pnt0"])
            b["descriptors"] = torch.from_numpy(npz["p0_desc_pnt1"])
            a["keypoints"] = torch.zeros(a["descriptors"].shape[1], 2)
            b["keypoints"] = torch.zeros(b["descriptors"].shape[1], 2)
        out.append((_dev(a), _dev(b)))
    return out


def _per_image_sequence(model, a, b, thr_l=0.8, thr_p=0.7):
    """models/matching.py:29-84 for one pair: per-image config, preprocess, forward, get_dist_matrix,
    subline2keyline, nn_matcher_distmat; nn_matcher for the points."""
    from linetr_b200 import nn_matcher as nnm
    from linetr_b200.line_process import get_dist_matrix
    out = []
    for im in (a, b):
        shape = im["image_shape"]
        model.config["min_length"] = max(16, max(shape) / 40)
        model.config["token_distance"] = max(8, max(shape) / 80)
        out.append(model(model.preprocess(im["klines"], shape, im, None)))
    ta, tb = out
    mat_l, dist_l = H.matching_line_branch(get_dist_matrix, model.subline2keyline, nnm.nn_matcher_distmat,
                                           ta["line_desc"].cpu().numpy(), tb["line_desc"].cpu().numpy(),
                                           ta["mat_klines2sublines"][0], tb["mat_klines2sublines"][0], thr_l)
    mat_p, dist_p = nnm.nn_matcher(a["descriptors"].cpu().numpy(), b["descriptors"].cpu().numpy(), thr_p, True)
    return mat_l, np.asarray(dist_l), mat_p, dist_p


@pytest.mark.gpu
def test_match_images_equals_per_image_sequence_and_oracle():
    from oracle import linetr_oracle as orc
    model, sd = _model()
    eng = engine.PairEngine(model, DEV)
    pairs = _ragged_pairs()
    res = eng.match_images([a for a, _ in pairs], [b for _, b in pairs], want_scores=True)
    assert res.n_pairs == 5
    npz, _ = H.plumbing()
    for p, (a, b) in enumerate(pairs):
        mat_l, dist_l, mat_p, dist_p = _per_image_sequence(model, a, b)
        want_l, want_p = dense_to_indices(mat_l), dense_to_indices(mat_p)
        got_l, got_p = res.pair_lines(p).cpu().numpy(), res.pair_points(p).cpu().numpy()
        assert np.array_equal(got_l, want_l), p
        assert np.array_equal(got_p, want_p), p
        assert int(res.counts_l[p]) == int((want_l >= 0).sum()) and int(res.counts_p[p]) == int((want_p >= 0).sum())
        ref = res.reference_dict(p)
        K0, K1, N0, N1 = mat_l.shape[1], mat_l.shape[2], mat_p.shape[1], mat_p.shape[2]
        assert ref["matches_l"].dtype == torch.float64 and tuple(ref["matches_l"].shape) == (1, K0, K1)
        assert ref["matching_scores_l"].dtype == torch.float32 and tuple(ref["matching_scores_l"].shape) == (1, K0, K1)
        assert ref["matches_p"].dtype == torch.float64 and tuple(ref["matches_p"].shape) == (1, N0, N1)
        assert ref["matching_scores_p"].dtype == torch.float32 and tuple(ref["matching_scores_p"].shape) == (1, N0, N1)
        assert np.array_equal(ref["matches_l"].numpy(), mat_l) and np.array_equal(ref["matches_p"].numpy(), mat_p)
        if K0 and K1:
            assert np.abs(ref["matching_scores_l"].numpy() - dist_l).max() < DIST_TOL
        if N0 and N1:
            assert np.abs(ref["matching_scores_p"].numpy() - dist_p).max() < DIST_TOL
        # points against the numpy oracle
        assert np.array_equal(got_p, dense_to_indices(orc.nn_matcher(a["descriptors"].cpu().numpy().astype(np.float64),
                                                                       b["descriptors"].cpu().numpy().astype(np.float64),
                                                                       0.7, True)[0]))
        if p == 4:
            assert np.array_equal(got_p, npz["p0_matches_p"])
        if p == 1:
            assert int(res.counts_l[p]) == 0 and (got_l == -1).all()
        if p == 3:
            assert int(res.counts_p[p]) == 0 and len(got_p) == 0
        # lines against the oracle on the CPU tokeniser's dicts, on the rows whose decision has a margin
        if K0 and K1:
            sides = []
            for im in (a, b):
                shape = im["image_shape"]
                cpu_sp = {k: im[k].cpu() for k in ("dense_descriptor", "dense_score")}
                c = LP.tokenizer_config(model.config, shape, True)
                d = _glue(im["klines"], shape, cpu_sp, {k: c[k] for k in ("min_length", "token_distance")})
                sides.append({k: v.numpy() for k, v in d.items()})
            omat, odk, _, _ = orc.match_pair(sd, sides[0], sides[1], 0.8)
            dec = H.decisive_rows(odk[0], 0.8, 2e-3)
            assert np.array_equal(got_l[dec], orc.match_indices(omat)[dec]), p
    assert int(res.counts_l.sum()) > 0 and int(res.counts_p.sum()) > 0
    # P = 0
    empty = eng.match_images([], [])
    assert empty.n_pairs == 0 and empty.matches_l.numel() == 0 and empty.counts_p.numel() == 0


@pytest.mark.gpu
def test_match_images_launch_count_does_not_grow_with_pairs():
    model, _ = _model()
    eng = engine.PairEngine(model, DEV)
    pairs = [tuple(map(_dev, syn.make_image_pair(300 + p, 40 + 10 * p, 200))) for p in range(2)]
    counts = []
    for rep in (1, 4):
        i0, i1 = [a for a, _ in pairs] * rep, [b for _, b in pairs] * rep
        eng.match_images(i0, i1)                   # warm-up: weight packing, workspaces
        torch.cuda.synchronize()
        N.reset_launch_count()
        eng.match_images(i0, i1)
        torch.cuda.synchronize()
        counts.append(N.launch_count())
    assert counts[0] == counts[1] > 0, counts


@pytest.mark.gpu
def test_match_images_never_synchronises():
    model, _ = _model()
    eng = engine.PairEngine(model, DEV)
    pairs = _ragged_pairs()
    i0, i1 = [a for a, _ in pairs], [b for _, b in pairs]
    want = eng.match_images(i0, i1)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = eng.match_images(i0, i1)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(got.matches_l, want.matches_l) and torch.equal(got.matches_p, want.matches_p)


def _reference_superpoint():
    if not os.path.isdir(os.path.join(H.REF_DIR, "models")):
        pytest.skip("original project not staged under oracle/_ref/ (build())")
    sys.path.insert(0, H.REF_DIR)
    try:
        import importlib.util
        spec = importlib.util.spec_from_file_location("_ref_superpoint", os.path.join(H.REF_DIR, "models", "superpoint.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        sys.path.remove(H.REF_DIR)
    from tests.golden.make_plumbing_golden import reference_matching_config
    return mod.SuperPoint(reference_matching_config()["superpoint"]).eval().to(DEV)


@pytest.mark.gpu
def test_match_images_real_pairs_equal_per_image_sequence():
    """The four bundled pairs: reference SuperPoint (GPU) and the test LSD shim once per image; the same outputs go
    through the per-image sequence of models/matching.py and through match_images."""
    pytest.importorskip("cv2")
    from tests.golden.make_plumbing_golden import ShimLSD, read_image
    model, _ = _model("shipped")
    sp = _reference_superpoint()
    lsd = ShimLSD({"n_octave": 2})
    _, meta = H.plumbing()
    images = []
    with torch.no_grad():
        for info in meta["pairs"]:
            pair = []
            for name in info["names"]:
                im = read_image(os.path.join(H.REF_DIR, "assets", name))
                out = sp({"image": im.to(DEV)})
                pair.append({"klines": lsd.detect_torch(im), "image_shape": tuple(im.shape), **out})
            images.append(pair)
    eng = engine.PairEngine(model, DEV)
    res = eng.match_images([a for a, _ in images], [b for _, b in images])
    for p, (a, b) in enumerate(images):
        a1 = {**a, "descriptors": a["descriptors"][0]}
        b1 = {**b, "descriptors": b["descriptors"][0]}
        from oracle import linetr_oracle as orc
        mat_l, _, mat_p, _ = _per_image_sequence(model, a1, b1)
        assert np.array_equal(res.pair_lines(p).cpu().numpy(), dense_to_indices(mat_l)), p
        assert np.array_equal(res.pair_points(p).cpu().numpy(), dense_to_indices(mat_p)), p
        assert int(res.counts_l[p]) > 0 and int(res.counts_p[p]) > 0
