"""Signature attention on uniform batches of 128-line images (`sig_attention_pipe_kernel`: one persistent CTA per SM,
all four heads of each of its images, P kept in registers).  It runs the per-element instruction sequence of
`sig_attention_tc_kernel`, so LTR_ATTN_PIPE=1 (the default) and LTR_ATTN_PIPE=0 must give the same bits: every
signature layer's attention output, the descriptors and the matches.  Every other batch keeps the old kernel."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from linetr_b200 import _native as N, _ops, engine, synthetic as syn
from tests import helpers as H
from tests.test_gemm_chain import _batch
from tests.test_image_pairs import _model

DEV = torch.device("cuda", 0)
T = 21


# ------------------------------------------------------------------ CPU: what ptxas made of the kernel
def test_pipe_kernel_keeps_its_state_in_registers():
    """The S and PV accumulators and the P fragments (64 + 32 + 64 registers per thread) fit the consumers' budget:
    no stack frame, no local memory, so nothing between the first and the last HGMMA of a head goes to memory."""
    lib = os.path.join(os.path.dirname(N._LIB_PATH), "liblinetr_b200.so")
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(lib) or not os.path.exists(tool):
        pytest.skip("needs the built library and cuobjdump")
    out = subprocess.check_output([tool, "-res-usage", lib], text=True, stderr=subprocess.STDOUT)
    lines = out.splitlines()
    idx = [i for i, l in enumerate(lines) if "Function" in l and "sig_attention_pipe_kernel" in l]
    assert len(idx) == 1, "sig_attention_pipe_kernel is not in the library"
    use = dict(kv.split(":", 1) for kv in lines[idx[0] + 1].split() if ":" in kv)
    assert use["STACK"] == "0" and use["LOCAL"] == "0", use
    assert int(use["REG"]) <= 168, use   # 384 threads, one CTA per SM


# ------------------------------------------------------------------ GPU
def _inputs(sizes, seed):
    ims = [syn.make_image_inputs(seed + i, L, T, None) for i, L in enumerate(sizes)]
    cat = lambda k: np.concatenate([np.asarray(im[k][0], np.float32) for im in ims], 0)
    host = dict(sublines=cat("sublines"), resp=cat("resp_sublines"), angle=cat("angle_sublines"),
                pnt=cat("pnt_sublines"), desc=cat("desc_sublines"), score=cat("score_sublines"))
    return {k: torch.from_numpy(v).contiguous().to(DEV) for k, v in host.items()}


def _encode(h, d, sizes, pipe):
    """ltr_encode of one batch -> (attention output xm[:, 256:] of the last signature layer as [tile, k-block, bytes]
    per plane, descriptor rows).  Uniform sizes go in as lines_per_image, others with cu."""
    lib = N.load()
    R = sum(sizes)
    uniform = len(set(sizes)) == 1
    cu = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    cu_dev = torch.from_numpy(cu).to(DEV)
    ws = torch.zeros(int(lib.ltr_encode_workspace_bytes(h.ptr, len(sizes), R, T)), dtype=torch.uint8, device=DEV)
    rows = torch.empty((R, 256), device=DEV)
    inp = N.LtrEncodeInput(*[d[k].data_ptr() for k in ("sublines", "resp", "angle", "pnt", "desc", "score")],
                           None if uniform else cu.ctypes.data, None if uniform else cu_dev.data_ptr(),
                           len(sizes), R, T, sizes[0] if uniform else 0, 640.0, 480.0)
    outp = N.LtrEncodeOutput(None, rows.data_ptr(), None)
    old = os.environ.get("LTR_ATTN_PIPE")
    os.environ["LTR_ATTN_PIPE"] = "1" if pipe else "0"
    try:
        rc = lib.ltr_encode(h.ptr, C.byref(inp), C.byref(outp), C.c_void_p(ws.data_ptr()), ws.numel(), None)
        torch.cuda.synchronize()
    finally:
        if old is None:
            del os.environ["LTR_ATTN_PIPE"]
        else:
            os.environ["LTR_ATTN_PIPE"] = old
    N.check(rc, "ltr_encode")
    hi, lo, kb = N.encode_images(h.ptr, R, ws.data_ptr())["xm"]
    n_tiles = -(-R // 128)
    planes = []
    for p in (hi, lo):
        off = p - ws.data_ptr()
        planes.append(ws[off:off + n_tiles * kb * 16384].view(n_tiles, kb, 16384)[:, 4:8].clone())
    return planes, rows


def _handle(n_sig):
    sd = H.weights_for("synthetic:0:1")
    d_inner = int(np.asarray(sd["klenc.desc_layers.0.pos_ffn.w_1.bias"]).shape[0])
    return _ops.ModelHandle(sd, 0, 256, 4, d_inner, 1, n_sig)


def _assert_same(h, d, sizes):
    (ph, pl), rp = _encode(h, d, sizes, True)
    (oh, ol), ro = _encode(h, d, sizes, False)
    for got, want in ((ph, oh), (pl, ol)):
        diff = (got != want).any(dim=2)
        assert not bool(diff.any()), f"attention output differs in (tile, head) {diff.nonzero()[:8].tolist()}"
    assert torch.equal(rp, ro)
    return ph


@pytest.mark.gpu
@pytest.mark.parametrize("n_sig", range(1, 8))
def test_every_signature_layer_bit_identical(n_sig):
    """cfg1's shape, 128 images x 128 lines: the attention output of signature layer n_sig - 1 (the last layer of an
    n_sig-layer model) is the same bits from either kernel."""
    d = _inputs([128] * 128, 10)
    h = _handle(n_sig)
    try:
        out = _assert_same(h, d, [128] * 128)
        assert bool((out != 0).any(dim=2).all())   # every (tile, head) block was written
    finally:
        h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n_images", [1, 150])
def test_image_counts(n_images):
    """One image (grid of one CTA), and more images than SMs (the CTAs' stride loop)."""
    d = _inputs([128] * n_images, 40)
    h = _handle(7)
    try:
        _assert_same(h, d, [128] * n_images)
    finally:
        h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("sizes", [[256] * 6, [128, 97, 128, 200, 33]], ids=["L256", "ragged"])
def test_other_batches_keep_the_old_kernel(sizes):
    """L = 256 and ragged batches take sig_attention_tc_kernel whatever LTR_ATTN_PIPE says."""
    d = _inputs(sizes, 70)
    h = _handle(2)
    try:
        _assert_same(h, d, sizes)
    finally:
        h.close()


def _run(eng, batch, P, pipe):
    os.environ["LTR_ATTN_PIPE"] = "1" if pipe else "0"
    try:
        N.reset_launch_count()
        rows, tiles = eng.encode(batch, want_tiles=True)
        torch.cuda.synchronize()
        launches = N.launch_count()
        res = eng.match_packed(batch, P, 0.8)
        torch.cuda.synchronize()
    finally:
        del os.environ["LTR_ATTN_PIPE"]
    return rows, tiles, res, launches


@pytest.mark.gpu
@pytest.mark.parametrize("pairs", [8, 64])
def test_encode_and_match_identical(pairs):
    """Pairs x 128 lines x 21 tokens through the engine: descriptor rows and tiles, matches and scores are equal, and
    a cfg1 encode (64 pairs) is still 20 launches."""
    batch, P = _batch([128] * pairs, 500, T)
    model, _ = _model()
    eng = engine.PairEngine(model, DEV)
    rp, tp, mp, lp = _run(eng, batch, P, True)
    ro, to, mo, lo = _run(eng, batch, P, False)
    assert lp == lo
    if pairs == 64:
        assert lp == 20
    assert torch.equal(rp, ro)
    assert torch.equal(tp, to)
    assert torch.equal(mp.matches0, mo.matches0)
    assert torch.equal(mp.scores0, mo.scores0)
    assert torch.equal(mp.counts, mo.counts)
