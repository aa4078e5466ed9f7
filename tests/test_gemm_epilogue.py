"""The image GEMM's fragment epilogue (`epi_frag_tile`): plain tiles whose op writes only a split-bf16 image take it
straight from the accumulator fragment and bulk-store each warp's 16 rows; ops that also write or read fp32 rows keep
the staged epilogue.

- The image the fragment path writes equals, bit for bit, the split (split8_bf16's rounding) of the fp32 rows the
  staged path writes for the same GEMM, at every tile width, activation and a row count that leaves a partial m-tile
  or more tiles than SMs; with and without a residual read from an image (written over in place, as mlp2 does).
- Rows at or past M of the last m-tile stay unwritten in every image an encode's GEMMs write, chained or not.
"""
import ctypes as C
import os

import numpy as np
import pytest

from linetr_b200 import _native as N, synthetic as syn
from tests import helpers as H

ACTS = {"none": 0, "relu": 1, "gelu": 2}


def _bf16_rn(v):
    """fp32 -> the fp32 value of its round-to-nearest-even bf16 (finite inputs)."""
    u = np.ascontiguousarray(v, np.float32).view(np.uint32)
    r = ((u + np.uint32(0x7FFF) + ((u >> 16) & np.uint32(1))) >> 16) << 16
    return r.astype(np.uint32).view(np.float32)


def _split_sum(y):
    """hi + lo of ptx::split2_bf16 (hi = bf16(y), lo = bf16(y - hi)), summed in fp32 as from_image_kernel does."""
    y = np.asarray(y, np.float32)
    hi = _bf16_rn(y)
    lo = _bf16_rn(y - hi)
    return (hi + lo).astype(np.float32)


def _linear_img(x, w, b, act, bn, image):
    """ltr_linear_img with one output: image only (fragment epilogue) or fp32 rows only (staged epilogue)."""
    import torch
    M, K = x.shape
    n = w.shape[0]
    out = torch.full((M, n), float("nan"), dtype=torch.float32, device=x.device)
    w_host = np.ascontiguousarray(w.cpu().numpy(), np.float32)
    y, y_img = (None, out.data_ptr()) if image else (out.data_ptr(), None)
    rc = N.load().ltr_linear_img(x.data_ptr(), K, w_host.ctypes.data, b.data_ptr(), None, n, y, n, y_img, M, n, K,
                                 act, bn, x.device.index, None)
    N.check(rc, "ltr_linear_img")
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 127, 130, 1000, 40000])
@pytest.mark.parametrize("act", sorted(ACTS))
@pytest.mark.parametrize("bn", [64, 128, 256])
def test_image_equals_split_of_rows(bn, act, M):
    import torch
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(1000 * bn + 10 * ACTS[act] + M % 7)
    K, n = 192, 256
    x = (torch.randn(M, K, generator=g) * 2.0).to(dev)
    w = torch.randn(n, K, generator=g) / K ** 0.5
    b = torch.randn(n, generator=g).to(dev)
    rows = _linear_img(x, w, b, ACTS[act], bn, image=False)
    img = _linear_img(x, w, b, ACTS[act], bn, image=True)
    assert np.isfinite(rows).all()
    want = _split_sum(rows)
    assert np.array_equal(img.view(np.uint32), want.view(np.uint32)), \
        (bn, act, M, int((img.view(np.uint32) != want.view(np.uint32)).sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 130, 1000, 40000])
@pytest.mark.parametrize("act", sorted(ACTS))
@pytest.mark.parametrize("bn", [64, 128, 256])
def test_residual_image_equals_split_of_rows(bn, act, M):
    """Residual read from a split-bf16 image (mlp2's x += delta): the fragment path, bulk-loading the residual and
    writing the output in place over it, equals the split of the staged path's fp32 rows bit for bit."""
    import torch
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(7000 + 1000 * bn + 10 * ACTS[act] + M % 7)
    K, n = 128, 256
    x = (torch.randn(M, K, generator=g) * 2.0).to(dev)
    w_host = np.ascontiguousarray((torch.randn(n, K, generator=g) / K ** 0.5).numpy(), np.float32)
    b = torch.randn(n, generator=g).to(dev)
    r = (torch.randn(M, n, generator=g) * 3.0).to(dev)
    lib = N.load()
    outs = []
    for image in (False, True):
        out = torch.full((M, n), float("nan"), dtype=torch.float32, device=dev)
        y, y_img = (None, out.data_ptr()) if image else (out.data_ptr(), None)
        rc = lib.ltr_debug_linear_img_res(x.data_ptr(), K, w_host.ctypes.data, b.data_ptr(), r.data_ptr(), y, y_img,
                                          M, n, K, ACTS[act], bn, 0, None)
        N.check(rc, "ltr_debug_linear_img_res")
        torch.cuda.synchronize()
        outs.append(out.cpu().numpy())
    rows, img = outs
    assert np.isfinite(rows).all()
    want = _split_sum(rows)
    assert np.array_equal(img.view(np.uint32), want.view(np.uint32)), \
        (bn, act, M, int((img.view(np.uint32) != want.view(np.uint32)).sum()))


SENTINEL = 0xA5
# images the encode's GEMMs write, with the k-blocks they write (xm[:, 256:] is the attention output, stored as whole
# tiles by sig_attention_tc)
GEMM_IMAGES = {"g": None, "hm": None, "qkv": None, "xm": 4}


@pytest.mark.gpu
@pytest.mark.parametrize("chain", [False, True])
def test_rows_past_m_stay_unwritten(chain):
    import torch
    from linetr_b200 import _ops
    dev = torch.device("cuda", 0)
    lib = N.load()
    sd = H.weights_for("synthetic:0:1")
    d_inner = int(np.asarray(sd["klenc.desc_layers.0.pos_ffn.w_1.bias"]).shape[0])
    h = _ops.ModelHandle(sd, 0, 256, 4, d_inner, 1, 2)
    Ls = [130, 101]   # 231 lines: the last m-tile holds rows 128 .. 230
    T = 21
    ims = [syn.make_image_inputs(7 + i, L, T, None) for i, L in enumerate(Ls)]
    cat = lambda k: np.concatenate([np.asarray(im[k][0], np.float32) for im in ims], 0)
    host = dict(sublines=cat("sublines"), resp=cat("resp_sublines"), angle=cat("angle_sublines"),
                pnt=cat("pnt_sublines"), desc=cat("desc_sublines"), score=cat("score_sublines"))
    d = {k: torch.from_numpy(v).contiguous().to(dev) for k, v in host.items()}
    R = sum(Ls)
    cu = np.concatenate([[0], np.cumsum(Ls)]).astype(np.int32)
    cu_dev = torch.from_numpy(cu).to(dev)
    ws = torch.full((int(lib.ltr_encode_workspace_bytes(h.ptr, len(Ls), R, T)),), SENTINEL, dtype=torch.uint8, device=dev)
    rows = torch.empty((R, 256), device=dev)
    tiles = torch.zeros(int(lib.ltr_desc_tiles_bytes(R)), dtype=torch.uint8, device=dev)
    inp = N.LtrEncodeInput(*[d[k].data_ptr() for k in ("sublines", "resp", "angle", "pnt", "desc", "score")],
                           cu.ctypes.data, cu_dev.data_ptr(), len(Ls), R, T, 0, 640.0, 480.0)
    outp = N.LtrEncodeOutput(None, rows.data_ptr(), tiles.data_ptr())
    old = os.environ.get("LTR_CHAIN_MIN_TILES")
    os.environ["LTR_CHAIN_MIN_TILES"] = "1" if chain else "0"
    try:
        rc = lib.ltr_encode(h.ptr, C.byref(inp), C.byref(outp), C.c_void_p(ws.data_ptr()), ws.numel(), None)
        torch.cuda.synchronize()
    finally:
        if old is None:
            del os.environ["LTR_CHAIN_MIN_TILES"]
        else:
            os.environ["LTR_CHAIN_MIN_TILES"] = old
    N.check(rc, "ltr_encode")
    assert np.isfinite(rows.cpu().numpy()).all()
    addr = N.encode_images(h.ptr, R, ws.data_ptr())
    base = ws.data_ptr()
    mt, m_in = R // 128, R % 128
    for name, kb_n in GEMM_IMAGES.items():
        hi, lo, kb = addr[name]
        kb_n = kb if kb_n is None else kb_n
        for plane in (hi, lo):
            off = plane - base + mt * kb * 16384
            t = ws[off:off + kb * 16384].view(kb, 128, 128)[:kb_n].cpu().numpy()   # [k-block, tile row, byte]
            assert (t[:, m_in:] == SENTINEL).all(), (name, chain, "rows >= M written")
            assert (t[:, :m_in] != SENTINEL).any(axis=2).all(), (name, chain, "rows < M not written")
