"""cfg[0] of BASELINE.json: the reference's `Matching` plugin / match_line_pairs.py path.

Three layers:
  * (CPU, everywhere) the oracle against what the UNMODIFIED reference `Matching` produced on the four
    bundled image pairs (tests/golden/plumbing_pairs.npz: real SuperPoint descriptors, real line geometry,
    key lines split into sublines) - pins the oracle on real data, not only on synthetic inputs;
  * (CPU, where build() staged the original project under oracle/_ref/) the reference's own `models/matching.py` executed
    UNCHANGED on top of `linetr_b200.install_as_reference_models()`: construction, per-image config
    mutation, `preprocess` (bit-identical tokeniser dicts), the full `forward` with the plugin's CUDA
    entry points routed to the oracle (test-only monkeypatch; the product has no CPU path and says so);
  * (GPU) the captured tokeniser dicts replayed through the real plugin: descriptors <= 1e-3, line and
    point matches identical (tests/test_gpu_parity.py::test_plumbing_*).
"""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import linetr_oracle as orc
from tests import helpers as H

REF = H.REF_DIR
needs_ref = pytest.mark.skipif(not os.path.isdir(REF), reason="original project not staged under oracle/_ref/ (build())")


def _weights():
    sd = H.load_shipped_weights()
    if sd is None:
        pytest.skip("shipped checkpoint not available")
    return sd


@pytest.mark.parametrize("pair", [0, 1, 2, 3])
def test_oracle_reproduces_reference_matching_on_real_pairs(pair):
    npz, meta = H.plumbing()
    sd = _weights()
    info = meta["pairs"][pair]
    a, want0 = H.plumbing_image(npz, f"p{pair}_0")
    b, want1 = H.plumbing_image(npz, f"p{pair}_1")
    assert a["sublines"].shape[1] == info["S0"] and a["klines"].shape[1] == info["K0"]
    d0 = orc.line_transformer_forward(sd, a)
    d1 = orc.line_transformer_forward(sd, b)
    assert np.abs(d0 - want0).max() < 2e-5 and np.abs(d1 - want1).max() < 2e-5
    # matcher on the REFERENCE descriptors: identical decisions, distances to fp32 rounding
    mat, dk = H.matching_line_branch(orc.get_dist_matrix, lambda d, A0, A1: orc.subline2keyline(d, A0, A1),
                                     orc.nn_matcher_distmat, want0, want1, a["mat_klines2sublines"][0],
                                     b["mat_klines2sublines"][0], 0.8)
    assert np.abs(dk[0] - npz[f"p{pair}_scores_l"]).max() < 1e-6
    assert np.array_equal(orc.match_indices(mat), npz[f"p{pair}_matches_l"])
    assert int(mat.sum()) == info["n_matches_l"]


def test_oracle_point_branch_on_real_superpoint_descriptors():
    npz, meta = H.plumbing()
    mat, _ = orc.nn_matcher(npz["p0_desc_pnt0"], npz["p0_desc_pnt1"], 0.7, True)
    assert np.array_equal(orc.match_indices(mat), npz["p0_matches_p"])
    assert int(mat.sum()) == meta["pairs"][0]["n_matches_p"]


# ------------------------------------------------------------------ reference Matching over the plugin
def _import_reference_matching_over_plugin():
    import linetr_b200
    for k in [k for k in sys.modules if k == "models" or k.startswith("models.")]:
        del sys.modules[k]
    sys.path.insert(0, REF)
    try:
        import models  # noqa: F401  (the reference package: superpoint, line_detector, matching stay stock)
        linetr_b200.install_as_reference_models()
        import models.matching as ref_matching
    finally:
        sys.path.remove(REF)
    from tests.golden.make_plumbing_golden import ShimLSD, read_image, reference_matching_config
    ref_matching.LSD = ShimLSD
    return ref_matching, read_image, reference_matching_config


@needs_ref
def test_reference_matching_constructs_and_preprocesses_over_plugin(monkeypatch):
    from linetr_b200 import _native as N
    from linetr_b200.line_transformer import LineTransformer as Ours
    # the plugin's LineTransformer(mode='test') loads the checkpoint build() staged with the reference
    monkeypatch.setenv("LINETR_WEIGHTS", H.shipped_weights_path())
    ref_matching, read_image, cfg = _import_reference_matching_over_plugin()
    assert ref_matching.LineTransformer is Ours          # models/matching.py:5 resolved to the plugin
    import linetr_b200.nn_matcher as our_nn
    assert ref_matching.nn_matcher is our_nn.nn_matcher and ref_matching.nn_matcher_distmat is our_nn.nn_matcher_distmat
    m = ref_matching.Matching(cfg()).eval()              # loads the shipped checkpoint through the plugin class
    assert isinstance(m.linetransformer, Ours)
    npz, meta = H.plumbing()
    names = meta["pairs"][0]["names"]
    im0 = read_image(os.path.join(REF, "assets", names[0]))
    im1 = read_image(os.path.join(REF, "assets", names[1]))
    with torch.no_grad():
        with pytest.raises(N.LtrError, match="CUDA"):     # forward reaches the plugin's CUDA boundary: no CPU fallback
            m({"image0": im0, "image1": im1})
        # everything before the boundary ran: SuperPoint, (shim) LSD, config mutation, the plugin's preprocess
        assert m.linetransformer.config["min_length"] == 16 and m.linetransformer.config["token_distance"] == 8
        sp = m.superpoint({"image": im0})
        kl = m.lsd.detect_torch(im0)
        tok = m.linetransformer.preprocess(kl, im0.shape, sp, torch.ones_like(im0))
    want, _ = H.plumbing_image(npz, "p0_0")
    for k, v in want.items():
        got = tok[k].numpy()
        if k == "desc_sublines":   # the fixture keeps the SuperPoint descriptors as float16 values
            got = got.astype(np.float16).astype(np.float32)
        if k in ("desc_sublines", "score_sublines"):
            # SuperPoint runs on the host CPU: its float results differ in the last bits between hosts (and the
            # float16 rounding of a descriptor can then land one step apart)
            assert np.allclose(got, v, rtol=1e-3, atol=1e-4), k
        else:
            assert np.array_equal(got, v), k      # identical to what the reference tokeniser fed its model


@needs_ref
def test_reference_matching_forward_unchanged_over_plugin_with_oracle_backend(monkeypatch):
    """The whole `Matching.forward` of the reference, unchanged, over the plugin's Python surface; only the
    three CUDA entry points are replaced by the oracle (there is no GPU in the build container).  Checks
    every dict key / shape / dtype the caller (match_line_pairs.py:91-104) reads."""
    from linetr_b200 import _ops, engine
    # the plugin's LineTransformer(mode='test') loads the checkpoint build() staged with the reference
    monkeypatch.setenv("LINETR_WEIGHTS", H.shipped_weights_path())
    ref_matching, read_image, cfg = _import_reference_matching_over_plugin()
    sd = _weights()

    def fake_encode(handle, sublines, resp, angle, pnt, desc, score, image_wh, *, lines_per_image=None, want_cf=True, **kw):
        L = int(lines_per_image)
        B = sublines.shape[0] // L
        T = desc.shape[1]
        data = {"sublines": sublines.reshape(B, L, 2, 2), "resp_sublines": resp.reshape(B, L, 1),
                "angle_sublines": angle.reshape(B, L, 2), "pnt_sublines": pnt.reshape(B, L, T, 2),
                # the fixture keeps the SuperPoint descriptors as float16 values (file size): the same rounding here
                "desc_sublines": np.asarray(desc).reshape(B, L, T, 256).astype(np.float16).astype(np.float32),
                "score_sublines": score.reshape(B, L, T, 1),
                "mask_sublines": np.ones((B, L, T + 1, 1), np.float32)}
        out = orc.line_transformer_forward(sd, {k: np.asarray(v) for k, v in data.items()}, (image_wh[1], image_wh[0]))
        return torch.from_numpy(out).reshape(-1), None

    def fake_match_descriptors(a, b, layout, n_pairs, thr, mutual=True, *, n0=0, n1=0, d=256, want_matches=True, **kw):
        A, Bm = a.numpy().reshape(n_pairs, d, n0), b.numpy().reshape(n_pairs, d, n1)
        dist = orc.get_dist_matrix(A, Bm)
        out = {"dist_key": torch.from_numpy(dist.reshape(-1)), "stride": n0 * n1}
        if want_matches:
            out["matches0"] = torch.from_numpy(orc.match_indices(orc.nn_matcher_distmat(dist[:1], thr, mutual)))
        return out

    def fake_match_distmat(dist, thr, mutual=True):
        return {"matches0": torch.from_numpy(orc.match_indices(orc.nn_matcher_distmat(dist.numpy(), thr, mutual)))[None]}

    def fake_merge(D, off0, off1, K0, K1):
        A = lambda off, K: np.stack([np.where((np.arange(off[-1]) >= off[k]) & (np.arange(off[-1]) < off[k + 1]),
                                              np.float32(1.0 / (off[k + 1] - off[k])), np.float32(0)) for k in range(K)])
        o0, o1 = off0.numpy(), off1.numpy()
        return torch.from_numpy(orc.subline2keyline(D.numpy(), A(o0, K0), A(o1, K1))[0])

    import linetr_b200.line_transformer as lt
    import linetr_b200.nn_matcher as nnm
    monkeypatch.setattr(_ops, "encode", fake_encode)
    monkeypatch.setattr(_ops, "match_descriptors", fake_match_descriptors)
    monkeypatch.setattr(_ops, "match_distmat", fake_match_distmat)
    monkeypatch.setattr(engine, "merge_sublines", fake_merge)
    monkeypatch.setattr(lt.LineTransformer, "_get_handle", lambda self, device: None)
    monkeypatch.setattr(_ops, "current_cuda_device", lambda: torch.device("cpu"))
    monkeypatch.setattr(_ops, "_req_cuda", lambda t, name: None)   # let CPU tensors pass the plugin's device guard
    m = ref_matching.Matching(cfg()).eval()
    npz, meta = H.plumbing()
    for p in (0, 3):
        names = meta["pairs"][p]["names"]
        with torch.no_grad():
            pred = m({"image0": read_image(os.path.join(REF, "assets", names[0])),
                      "image1": read_image(os.path.join(REF, "assets", names[1]))})
        for k in ("matches_l", "matching_scores_l", "matches_p", "matching_scores_p", "klines0", "klines1", "line_desc0",
                  "line_desc1", "keypoints0", "keypoints1", "mat_klines2sublines0", "sublines1"):
            assert k in pred, k
        K0, K1 = meta["pairs"][p]["K0"], meta["pairs"][p]["K1"]
        assert pred["matches_l"].shape == (1, K0, K1) and pred["matches_l"].dtype == torch.float64
        assert pred["matching_scores_l"].shape == (1, K0, K1) and pred["matching_scores_l"].dtype == torch.float32
        assert np.abs(pred["line_desc0"].numpy() - npz[f"p{p}_0_line_desc"]).max() < 2e-5
        got = np.where(pred["matches_l"][0].numpy().sum(1) > 0, pred["matches_l"][0].numpy().argmax(1), -1)
        assert np.array_equal(got, npz[f"p{p}_matches_l"])
        assert int(pred["matches_p"].sum()) == meta["pairs"][p]["n_matches_p"]
