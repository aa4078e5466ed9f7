"""Shared test helpers: golden fixtures, regenerated inputs, drift checks."""
import json
import os

import numpy as np

from linetr_b200 import synthetic as syn

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# the original project's models package, checkpoints and image pairs, staged by build() (oracle/stage_reference.py)
REF_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "reference")
_cache = {}


def golden():
    if "npz" not in _cache:
        _cache["npz"] = dict(np.load(os.path.join(GOLDEN_DIR, "reference_outputs.npz")))
        with open(os.path.join(GOLDEN_DIR, "reference_outputs.json")) as f:
            _cache["meta"] = json.load(f)
    return _cache["npz"], _cache["meta"]


def golden_full():
    """Full-size images (256 x 32, ragged 512 x 64) through the reference with the seeded weight set named in
    the fixture's metadata (tests/golden/make_golden.py::main_full)."""
    if "npz_full" not in _cache:
        _cache["npz_full"] = dict(np.load(os.path.join(GOLDEN_DIR, "reference_outputs_full.npz")))
        with open(os.path.join(GOLDEN_DIR, "reference_outputs_full.json")) as f:
            _cache["meta_full"] = json.load(f)
    return _cache["npz_full"], _cache["meta_full"]


FULL_CASES = ["real_enc_L256_T32", "real_enc_L512_T64_ragged"]


def checksum(d):
    return {k: float(np.asarray(v, dtype=np.float64).sum()) for k, v in sorted(d.items())}


def assert_checksum(d, want):
    got = checksum(d)
    assert got.keys() == want.keys()
    for k in got:
        assert abs(got[k] - want[k]) <= 1e-6 * max(1.0, abs(want[k])), f"input generator drift in {k}"


def weights_for(tag):
    kind, *rest = tag.split(":")
    if kind == "synthetic":
        return syn.make_state_dict(int(rest[0]), int(rest[1]))
    raise KeyError(tag)


def shipped_weights_path():
    """The reference checkpoint: $LINETR_WEIGHTS, or the copy build() staged under oracle/_ref/ (git-ignored)."""
    for p in (os.environ.get("LINETR_WEIGHTS", ""), os.path.join(REF_DIR, "models", "weights", "LineTR_weight.pth")):
        if p and os.path.exists(p):
            return p
    return None


def load_shipped_weights():
    p = shipped_weights_path()
    if p is None:
        return None
    import torch
    return {k: v.numpy() for k, v in torch.load(p, map_location="cpu").items()}


def case_inputs(case):
    ntok = case.get("ntok")
    ntok = tuple(ntok) if isinstance(ntok, list) else ntok
    return syn.make_image_inputs(case["seed"], case["L"], case["T"], ntok)


def stack(images):
    return {k: np.concatenate([im[k] for im in images], axis=0) for k in images[0]}


ENC_CASES = ["enc_L16_T21", "enc_L1_T21", "enc_L37_T5_ragged", "enc_L24_T32_ragged", "enc_L130_T21",
             "enc_L9_T21_nd2"]


# ---------------------------------------------------------------- cfg[0] plumbing / tokenizer fixtures
TOK_KEYS = ("klines", "length_klines", "angles", "sublines", "pnt_sublines", "mask_sublines", "resp_sublines",
            "angle_sublines", "score_sublines", "mat_klines2sublines")


def plumbing():
    """Fixtures of tests/golden/make_plumbing_golden.py: the reference `Matching` run on the four bundled pairs."""
    if "plumb" not in _cache:
        npz = {}
        for fn in sorted(os.listdir(GOLDEN_DIR)):   # plumbing_pairs / plumbing_img_<pair>_<side> / plumbing_pnt
            if fn.startswith("plumbing_") and fn.endswith(".npz"):
                npz.update(np.load(os.path.join(GOLDEN_DIR, fn)))
        # SuperPoint descriptors are stored as float16 values; the models consume them as float32
        _cache["plumb"] = {k: v.astype(np.float32) if v.dtype == np.float16 else v for k, v in npz.items()}
        with open(os.path.join(GOLDEN_DIR, "plumbing_pairs.json")) as f:
            _cache["plumb_meta"] = json.load(f)
    return _cache["plumb"], _cache["plumb_meta"]


def _rebuild_desc(mask_sublines, real, pad):
    """desc_sublines [1,S,T,256] from the real-token descriptors and the shared pad descriptor."""
    mask = mask_sublines[0, :, 1:, 0] > 0
    S, T = mask.shape
    desc = np.broadcast_to(pad.astype(np.float32), (S, T, 256)).copy()
    desc[mask] = real
    return desc[None]


def plumbing_image(npz, prefix):
    """Tokeniser dict (numpy, batch dim 1) of one captured image + the reference's line_desc."""
    d = {k: npz[f"{prefix}_{k}"] for k in TOK_KEYS}
    d["desc_sublines"] = _rebuild_desc(d["mask_sublines"], npz[f"{prefix}_desc_real"], npz[f"{prefix}_desc_pad"])
    return d, npz[f"{prefix}_line_desc"]


def tokenizer_fixture(ci):
    """-> (tokeniser fields except desc_sublines, (rows, real-token descriptors at those rows, pad descriptor)): the
    fixture keeps a fixed sample (every third row) of the real-token descriptors."""
    if "tok" not in _cache:
        _cache["tok"] = dict(np.load(os.path.join(GOLDEN_DIR, "tokenizer_outputs.npz")))
    npz = _cache["tok"]
    d = {k[len(f"c{ci}_"):]: v for k, v in npz.items() if k.startswith(f"c{ci}_") and not k.startswith(f"c{ci}_desc_")}
    return d, (npz[f"c{ci}_desc_real_rows"], npz[f"c{ci}_desc_real"], npz[f"c{ci}_desc_pad"])


def matching_line_branch(get_dist_matrix, subline2keyline, nn_matcher_distmat, line_desc0, line_desc1, A0, A1, thr):
    """The line branch of the reference's Matching.forward (models/matching.py:77-81), parameterised by
    the three functions it calls, so that tests can run it over the plugin or over the oracle."""
    distance_sublines = get_dist_matrix(line_desc0, line_desc1)[0]
    distance_matrix = subline2keyline(distance_sublines, A0, A1)
    match_mat = nn_matcher_distmat(distance_matrix, thr, True)
    return match_mat, distance_matrix


def decisive_rows(dist, thr, margin):
    """Rows of [K0,K1] distances whose decision does not hinge on differences below `margin`."""
    d = np.clip(np.asarray(dist, dtype=np.float64), 0.0, None)
    K0, K1 = d.shape
    srt = np.sort(d, axis=1)
    row_gap = srt[:, 1] - srt[:, 0] if K1 > 1 else np.full(K0, np.inf)
    idx = d.argmin(axis=1)
    csrt = np.sort(d, axis=0)
    col_gap = (csrt[1] - csrt[0]) if K0 > 1 else np.full(K1, np.inf)
    return (row_gap > margin) & (np.abs(srt[:, 0] - thr) > margin) & (col_gap[idx] > margin)
