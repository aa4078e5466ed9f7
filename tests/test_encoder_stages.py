"""Every encoder kernel against a float64 model of its own stage, from its own GPU-produced inputs.

`ltr_debug_encode_images` tells where `ltr_encode` leaves each stage's activation image in the caller's workspace; a
test encodes with its own workspace, decodes the images (hi + lo, exact in fp64) and feeds a stage's GPU input to the
fp64 stage (tests/encoder_stage_model.py), then asserts |GPU output - fp64| <= bound element by element.  The bounds
are computed from the data by the precision model (split-bf16 operands, fp32 accumulation, image re-quantisation,
LayerNorm, GELU and softmax terms); the CPU tests below show that the fp64 stages compose to the reference forward and
that a subtly wrong kernel (a dropped split term, one skipped key, a bf16-only P, a token pooled into the wrong line,
an unbiased LayerNorm variance) lands outside its stage's bound.  n_sig_layers isolates a signature layer: a model
with l layers leaves x_l in xm, one with l + 1 leaves qkv_l, o_l, hm_l and x_{l+1}, computed from the same x_l.

Measured worst err / bound per stage over this file on one H100 SXM (seeded weights unless marked; the shipped
checkpoint where installed), printed at the end of a run with -s: token 0.31 (peaked CLS 0.06, shipped 0.05), V
projection 0.21, line positional head 0.82, l4 0.37, l5 0.26, fc + LN 0.24, w_1 GELU 0.17, w_2 + LN + pos 0.54, qkv
0.18 (shipped 0.23), attention 0.08 (peaked 0.01, shipped 0.07), mlp1 0.13 (0.16), mlp2 0.25 (0.31), final rows 0.11,
tiles vs rows 0.50, final_proj into yf 0.11, final_norm_kernel 0.22.  The file runs in about 80 s on the GPU.
"""
import ctypes as C
import os

import numpy as np
import pytest

from linetr_b200 import _native as N, synthetic as syn
from oracle import linetr_oracle as orc
from tests import helpers as H
from tests import encoder_stage_model as M

SEEDED = "synthetic:0:1"


# ------------------------------------------------------------------ CPU: the fp64 stages compose to the reference
def _compose(sm, data, width=640, height=480):
    """The fp64 stages end to end on one tokeniser dict (batch dim B, uniform lines) -> [B, 256, L]."""
    B, L, T = data["desc_sublines"].shape[:3]
    f = lambda k, *s: np.asarray(data[k], np.float64).reshape(B * L, *s)
    z, _, _ = sm.token(f("pnt_sublines", T, 2), f("score_sublines", T, 1), f("desc_sublines", T, 256), width, height)
    ctx, _ = sm.vproj(z)
    y1, _ = sm.fc_ln1(ctx)
    g, _ = sm.w1_gelu(y1)
    l128, _ = sm.line_pos_head(f("sublines", 2, 2), f("resp_sublines", 1), f("angle_sublines", 2), width, height)
    lpos, _ = sm.line_pos_l5(sm.line_pos_l4(l128)[0])
    x, _ = sm.w2_ln2(g, y1, lpos)
    cu = np.arange(B + 1) * L
    for l in range(len(sm.sig)):
        q, _ = sm.qkv(x, l)
        o, _ = M.attention(q, cu)
        hm, _ = sm.mlp1(x, o, l)
        x, _ = sm.mlp2(hm, x, l)
    u, _ = sm.final_rows(x)
    return u.reshape(B, L, 256).transpose(0, 2, 1)


@pytest.mark.parametrize("name", H.ENC_CASES)
def test_stage_model_composes_to_reference(name):
    """The fp64 stages, composed, equal the fp32 oracle and the reference's committed outputs to fp32 noise."""
    npz, meta = H.golden()
    case = meta["cases"][name]
    sd = H.weights_for(case["weights"])
    data = H.case_inputs(case)
    got = _compose(M.StageModel(sd), data)
    assert np.abs(got - orc.line_transformer_forward(sd, data)).max() < 1e-5
    assert np.abs(got - npz[name]).max() < 2e-5


def _stage_data():
    """fp64 activations of every stage on enc_L130_T21 (one image of 130 lines)."""
    _, meta = H.golden()
    case = meta["cases"]["enc_L130_T21"]
    sd = H.weights_for(case["weights"])
    d = H.case_inputs(case)
    sm = M.StageModel(sd)
    R, T = 130, 21
    f = lambda k, *s: np.asarray(d[k], np.float64).reshape(R, *s)
    raw = (f("pnt_sublines", T, 2), f("score_sublines", T, 1), f("desc_sublines", T, 256))
    z, _, _ = sm.token(*raw, 640, 480)
    ctx, _ = sm.vproj(z)
    y1, _ = sm.fc_ln1(ctx)
    g, _ = sm.w1_gelu(y1)
    q, _ = sm.qkv(sm.w2_ln2(g, y1, np.zeros_like(y1))[0], 0)
    return sm, raw, ctx, y1, g, q


def _worst(err, bound):
    return float((np.abs(err) / bound).max())


def test_planted_gemm_error_exceeds_bound():
    """The split-bf16 GEMM emulated on the CPU stays inside gemm_bound; without the a_lo * w_hi term it does not
    (K = 256: w_1, K = 1024: w_2)."""
    sm, _, _, y1, g, _ = _stage_data()
    for A, W, b in ((y1, sm.W1, sm.b1), (g, sm.W2, sm.b2)):
        good, a_img = M.emulate_gemm(A, W, b)
        bad, _ = M.emulate_gemm(A, W, b, drop_lo_hi=True)
        want = a_img @ W.T + b
        bound = M.gemm_bound(a_img, W, b, want)
        assert _worst(good - want, bound) <= 1.0
        assert _worst(bad - want, bound) > 1.0


def test_planted_attention_errors_exceed_bound():
    """One key skipped in one image, or P rounded to bf16 alone: both outside the attention bound."""
    _, _, _, _, _, q = _stage_data()
    cu = np.array([0, 130])
    o, e = M.attention(q, cu)
    for kw in (dict(skip_key=(0, 77)), dict(bf16_p=True)):
        bad, _ = M.attention(q, cu, **kw)
        assert _worst(bad - o, e) > 1.0, kw


def test_planted_token_pooling_error_exceeds_bound():
    """Token 3 of every line pooled into the next line's z: outside the token stage's bound."""
    sm, raw, _, _, _, _ = _stage_data()
    z, e, _ = sm.token(*raw, 640, 480)
    bad, _, _ = sm.token(*raw, 640, 480, pool_shift=3)
    assert _worst(bad - z, e) > 1.0


def test_planted_layer_norm_error_exceeds_bound():
    """LayerNorm with the unbiased variance (the biased / unbiased mix-up) is outside the fc + LN bound.  (Omitting
    eps = 1e-6 moves y by eps / (2 var) relative, below fp32 resolution at these variances.)"""
    sm, _, ctx, _, _, _ = _stage_data()
    y, e = sm.fc_ln1(ctx)
    bad, _ = sm.fc_ln1(ctx, ddof=1)
    assert _worst(bad - y, e) > 1.0


# ------------------------------------------------------------------ GPU
WORST_RATIO = {}


def _check(stage, got, want, bound):
    got = np.asarray(got, np.float64)
    assert got.shape == want.shape, (stage, got.shape, want.shape)
    assert np.isfinite(got).all(), stage
    r = np.abs(got - want) / bound
    worst = float(r.max()) if r.size else 0.0
    WORST_RATIO[stage] = max(WORST_RATIO.get(stage, 0.0), worst)
    assert worst <= 1.0, (stage, worst, np.unravel_index(int(r.argmax()), r.shape))


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST_RATIO:
        print("\nworst err/bound per stage:", {k: round(v, 4) for k, v in sorted(WORST_RATIO.items())})


_sd_cache = {}


def _state_dict(tag):
    if tag not in _sd_cache:
        if tag == "shipped":
            sd = H.load_shipped_weights()
            if sd is None:
                pytest.skip("shipped checkpoint not available")
        else:
            sd = H.weights_for(tag)
        _sd_cache[tag] = sd
    return _sd_cache[tag]


class Encoder:
    """One ModelHandle with n_sig signature layers, its fp64 stage model, and encodes into a workspace of its own."""

    def __init__(self, sd, n_sig):
        import torch
        from linetr_b200 import _ops
        self.torch = torch
        self.dev = torch.device("cuda", 0)
        d_inner = int(np.asarray(sd["klenc.desc_layers.0.pos_ffn.w_1.bias"]).shape[0])
        nd = 0
        while f"klenc.desc_layers.{nd}.slf_attn.w_qs.weight" in sd:
            nd += 1
        self.h = _ops.ModelHandle(sd, 0, 256, 4, d_inner, nd, n_sig)
        self.sm = M.StageModel(sd, n_sig)

    def run(self, images, width=640, height=480, uniform=False, cf=False, chain=None):
        """Encode the list of tokeniser dicts (batch dim 1 each); returns a dict of decoded images and outputs."""
        torch = self.torch
        lib = N.load()
        cat = lambda k: np.concatenate([np.asarray(im[k][0], np.float32) for im in images], 0)
        L = [im["desc_sublines"].shape[1] for im in images]
        T = images[0]["desc_sublines"].shape[2]
        R = sum(L)
        host = dict(sublines=cat("sublines"), resp=cat("resp_sublines"), angle=cat("angle_sublines"),
                    pnt=cat("pnt_sublines"), desc=cat("desc_sublines"), score=cat("score_sublines"))
        dev = {k: torch.from_numpy(v).contiguous().to(self.dev) for k, v in host.items()}
        cu = np.concatenate([[0], np.cumsum(L)]).astype(np.int32)
        cu_dev = torch.from_numpy(cu).to(self.dev)
        need = int(lib.ltr_encode_workspace_bytes(self.h.ptr, len(L), R, T))
        ws = torch.zeros(need, dtype=torch.uint8, device=self.dev)
        rows = torch.full((R, 256), float("nan"), device=self.dev)
        out_cf = torch.full((R * 256,), float("nan"), device=self.dev) if cf else None
        tiles = None if cf else torch.zeros(int(lib.ltr_desc_tiles_bytes(R)), dtype=torch.uint8, device=self.dev)
        inp = N.LtrEncodeInput(*[dev[k].data_ptr() for k in ("sublines", "resp", "angle", "pnt", "desc", "score")],
                               None if uniform else cu.ctypes.data, None if uniform else cu_dev.data_ptr(),
                               len(L), R, T, L[0] if uniform else 0, float(width), float(height))
        outp = N.LtrEncodeOutput(out_cf.data_ptr() if cf else None, rows.data_ptr(),
                                 tiles.data_ptr() if tiles is not None else None)
        old = os.environ.get("LTR_CHAIN_MIN_TILES")
        if chain is not None:
            os.environ["LTR_CHAIN_MIN_TILES"] = "1" if chain else "0"
        try:
            rc = lib.ltr_encode(self.h.ptr, C.byref(inp), C.byref(outp), C.c_void_p(ws.data_ptr()), ws.numel(), None)
            torch.cuda.synchronize()
        finally:
            if chain is not None:
                if old is None:
                    del os.environ["LTR_CHAIN_MIN_TILES"]
                else:
                    os.environ["LTR_CHAIN_MIN_TILES"] = old
        N.check(rc, "ltr_encode")
        addr = N.encode_images(self.h.ptr, R, ws.data_ptr())
        base = ws.data_ptr()
        widths = dict(z=1024, ctx=256, l128=128, l256=256, lpos=256, y1i=256, g=self.sm.W1.shape[0], xm=512, hm=512,
                      qkv=768)
        res = {k: _decode(ws, a[0] - base, a[1] - base, a[2], R, widths[k]) for k, a in addr.items() if k != "yf"}
        off = addr["yf"][0] - base
        res["yf"] = ws[off:off + R * 1024].view(torch.float32).reshape(R, 256).double().cpu().numpy()
        res["rows"] = rows.double().cpu().numpy()
        if cf:
            res["cf"] = out_cf.double().cpu().numpy()
        if tiles is not None:
            plane = (R + 127) // 128 * 128 * 256 * 2
            res["tiles"] = _decode(tiles, 0, plane, 4, R, 256)
        res.update(host=host, cu=cu, R=R, T=T)
        return res


def _decode(buf, off_hi, off_lo, kb, R, K):
    """Activation image (hi + lo planes at byte offsets of the uint8 tensor `buf`) -> fp64 [R, K]."""
    import torch
    r = torch.arange(R, device=buf.device)[:, None]
    k = torch.arange(K, device=buf.device)[None, :]
    rr = r & 127
    sw = (rr >> 3) * 1024 + (rr & 7) * 128 + ((((k & 63) >> 3) ^ (rr & 7)) & 7) * 16 + (k & 7) * 2
    idx = ((r >> 7) * kb + (k >> 6)) * 8192 + sw // 2
    n = ((R + 255) // 256 * 256) * kb * 64
    n = max(n, int(idx.max()) + 1) if R else n
    hi = buf[off_hi:off_hi + 2 * n].view(torch.bfloat16)
    lo = buf[off_lo:off_lo + 2 * n].view(torch.bfloat16)
    return (hi[idx].double() + lo[idx].double()).cpu().numpy()


_enc_cache = {}


def _encoder(tag, n_sig, scale=None):
    key = (tag, n_sig, tuple(sorted(scale.items())) if scale else None)
    if key not in _enc_cache:
        sd = _state_dict(tag)
        if scale is not None:
            sd = dict(sd)
            for k, f in scale.items():
                sd[k] = np.asarray(sd[k], np.float32) * np.float32(f)
        _enc_cache[key] = Encoder(sd, n_sig)
    return _enc_cache[key]


def _images(sizes, T, seed, ntok=None, width=640, height=480):
    return [syn.make_image_inputs(seed + i, n, T, ntok, width=width, height=height) for i, n in enumerate(sizes)]


def _check_token(enc, res, width, height, tag=""):
    h, R, T = res["host"], res["R"], res["T"]
    z, ez, sc = enc.sm.token(h["pnt"], h["score"], h["desc"], width, height)
    _check("token" + tag, res["z"], z, ez)
    ctx, ectx = enc.sm.vproj(res["z"])
    _check("vproj", res["ctx"], ctx, ectx)
    return sc


def _check_line(enc, res, width, height):
    sm, h = enc.sm, res["host"]
    l128, e = sm.line_pos_head(h["sublines"], h["resp"], h["angle"], width, height)
    _check("line_pos_head", res["l128"], l128, e)
    _check("line_pos_l4", res["l256"], *sm.line_pos_l4(res["l128"]))
    _check("line_pos_l5", res["lpos"], *sm.line_pos_l5(res["l256"]))
    _check("fc_ln1", res["y1i"], *sm.fc_ln1(res["ctx"]))
    _check("w1_gelu", res["g"], *sm.w1_gelu(res["y1i"]))
    _check("w2_ln2", res["xm"][:, :256], *sm.w2_ln2(res["g"], res["y1i"], res["lpos"]))


def _check_final_rows(enc, res):
    u, e = enc.sm.final_rows(res["xm"][:, :256])
    _check("final_rows", res["rows"], u, e)
    if "tiles" in res:
        # hi + lo of an fp32 value: within 2^-16 relative (tests/test_numeric_formulas.py::test_split_bf16_precision)
        _check("final_tiles", res["tiles"], res["rows"], 2.0 ** -16 * np.abs(res["rows"]) + 1e-30)


# token stage: T x R (R >= 3 rounds of 132 CTAs where lpt * 3 * 132 lines stay small, R % lpt != 0, R < lpt)
TOKEN_CASES = [
    (1, 1000, (640, 480), None), (2, 1000, (1241, 376), (1, 2)), (5, 9901, (640, 480), (2, 5)), (5, 7, (512, 512), None),
    (21, 2401, (640, 480), (3, 21)), (21, 4, (1241, 376), None), (42, 1189, (512, 512), (5, 42)),
    (43, 1191, (640, 480), None), (64, 801, (640, 480), (10, 64)), (65, 799, (1241, 376), None),
    (127, 400, (640, 480), (1, 127)), (128, 397, (512, 512), (60, 128)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("T, R, wh, ntok", TOKEN_CASES)
def test_token_stage_vs_fp64(T, R, wh, ntok):
    """token_fused_kernel (raw tokens -> z) and the V projection (z -> ctx) against fp64 from their inputs."""
    enc = _encoder(SEEDED, 0)
    res = enc.run(_images([R], T, 1000 + T, ntok, *wh), *wh, uniform=True)
    _check_token(enc, res, *wh)


@pytest.mark.gpu
def test_token_stage_peaked_cls_softmax():
    """CLS scores scaled up (W_q and b_q of the descriptive layer) until the largest logits reach about 30."""
    sd = _state_dict(SEEDED)
    imgs = _images([50, 37], 21, 77)
    sm = M.StageModel(sd, 0)
    f = lambda k, *s: np.concatenate([np.asarray(im[k][0], np.float64) for im in imgs]).reshape(87, *s)
    _, _, sc = sm.token(f("pnt_sublines", 21, 2), f("score_sublines", 21, 1), f("desc_sublines", 21, 256), 640, 480)
    s = 30.0 / float(np.abs(sc).max())
    p = "klenc.desc_layers.0.slf_attn.w_qs"
    enc = _encoder(SEEDED, 0, {p + ".weight": s, p + ".bias": s})
    res = enc.run(imgs)
    sc = _check_token(enc, res, 640, 480, "_peaked")
    assert np.abs(sc).max() > 25


@pytest.mark.gpu
@pytest.mark.parametrize("chain", [False, True])
@pytest.mark.parametrize("R", [1, 3, 4097, 12672, 12673, 30001])
def test_line_stage_vs_fp64(R, chain):
    """Line positional encoder (small_mlp_kernel<false> past its 396-CTA grid-stride threshold, then two GEMMs), fc +
    LN, w_1 GELU and w_2 + LN + position, per layer and chained, then final_proj + L2 on x_0 (rows and tiles)."""
    enc = _encoder(SEEDED, 0)
    res = enc.run(_images([R], 1, 3000 + R), uniform=True, chain=chain)
    _check_token(enc, res, 640, 480)
    _check_line(enc, res, 640, 480)
    _check_final_rows(enc, res)


@pytest.mark.gpu
def test_line_stage_shipped_checkpoint():
    enc = _encoder("shipped", 0)
    res = enc.run(_images([300, 45], 21, 11))
    _check_token(enc, res, 640, 480, "_shipped")
    _check_line(enc, res, 640, 480)
    _check_final_rows(enc, res)


ATTN_L = [1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 640, 1000, 2048]
ATTN_BATCHES = {
    "uniform128": ([128] * 6, True),                   # bulk-copy (TMA) operand tiles
    "uniform256": ([256] * 3, True),                   # cp.async gather, two key tiles
    "ragged_aligned": ([128, 5, 123, 128, 128], False),   # 128-line images at 128-aligned offsets under cu, one not
    "ragged_sizes": (ATTN_L, False),
    "ragged_empty": ([0, 3, 0, 129, 0, 0, 128, 0], False),
}


def _check_attention(enc, res, tag):
    o, e = M.attention(res["qkv"], res["cu"])
    _check("attention" + tag, res["xm"][:, 256:], o, e)


@pytest.mark.gpu
@pytest.mark.parametrize("batch", list(ATTN_BATCHES))
def test_sig_attention_vs_fp64(batch):
    """sig_attention_tc_kernel (qkv_0 -> o_0) on its three paths, segmented per image exactly as cu."""
    sizes, uniform = ATTN_BATCHES[batch]
    enc = _encoder(SEEDED, 1)
    _check_attention(enc, enc.run(_images(sizes, 1, 500), uniform=uniform), "")


@pytest.mark.gpu
def test_sig_attention_peaked_rows():
    """q of layer 0 scaled up until the largest logits reach about 30."""
    imgs = _images([300, 128, 77], 1, 600)
    res = _encoder(SEEDED, 1).run(imgs)
    q, k = res["qkv"][:, :256], res["qkv"][:, 256:512]
    s = max(float(np.abs(q[a:b, h * 64:(h + 1) * 64] @ k[a:b, h * 64:(h + 1) * 64].T).max())
            for a, b in zip(res["cu"][:-1], res["cu"][1:]) for h in range(4))
    p = "selfattn.layers.0.attn.proj.0"
    enc = _encoder(SEEDED, 1, {p + ".weight": 30.0 / s, p + ".bias": 30.0 / s})
    res = enc.run(imgs)
    _check_attention(enc, res, "_peaked")


@pytest.mark.gpu
@pytest.mark.parametrize("chain", [False, True])
@pytest.mark.parametrize("layer", [0, 6])
@pytest.mark.parametrize("batch", ["uniform", "ragged"])
def test_sig_layer_gemms_vs_fp64(layer, chain, batch):
    """qkv (x_l -> qkv_l), mlp1 ([x_l | o_l] -> hm_l, merge folded) and mlp2 (hm_l + x_l -> x_{l+1}), per layer and
    chained; with all seven layers also final_proj + L2 on x_7."""
    sizes, uniform = ([128] * 3, True) if batch == "uniform" else ([37, 300, 5, 190], False)
    imgs = _images(sizes, 5, 700)
    a = _encoder(SEEDED, layer).run(imgs, uniform=uniform, chain=chain)
    enc = _encoder(SEEDED, layer + 1)
    b = enc.run(imgs, uniform=uniform, chain=chain)
    x = a["xm"][:, :256]
    _check("qkv", b["qkv"], *enc.sm.qkv(x, layer))
    _check_attention(enc, b, "")
    _check("mlp1", b["hm"], *enc.sm.mlp1(x, b["xm"][:, 256:], layer))
    _check("mlp2", b["xm"][:, :256], *enc.sm.mlp2(b["hm"], x, layer))
    if layer + 1 == len(enc.sm.sig):
        _check_final_rows(enc, b)


@pytest.mark.gpu
def test_sig_layer_gemms_shipped_checkpoint():
    imgs = _images([200, 64], 5, 800)
    a = _encoder("shipped", 0).run(imgs)
    enc = _encoder("shipped", 1)
    b = enc.run(imgs)
    x = a["xm"][:, :256]
    _check("qkv_shipped", b["qkv"], *enc.sm.qkv(x, 0))
    _check_attention(enc, b, "_shipped")
    _check("mlp1_shipped", b["hm"], *enc.sm.mlp1(x, b["xm"][:, 256:], 0))
    _check("mlp2_shipped", b["xm"][:, :256], *enc.sm.mlp2(b["hm"], x, 0))


@pytest.mark.gpu
def test_final_channel_first_vs_fp64():
    """Channel-first output: final_proj into fp32 yf, then final_norm_kernel over grid (cdiv(max_l, 32), n_images) of
    ragged images, empty ones included: rows and [256, L_i] blocks against the fp64 L2 norm of yf."""
    sizes = [0, 40, 1, 0, 333, 65]
    enc = _encoder(SEEDED, 7)
    res = enc.run(_images(sizes, 5, 900), cf=True)
    _check("final_proj_cf", res["yf"], *enc.sm.final_proj(res["xm"][:, :256]))
    u, e = M.l2_rows_bound(res["yf"])
    _check("final_norm_rows", res["rows"], u, e)
    cu = res["cu"]
    for i in range(len(sizes)):
        a, b = int(cu[i]), int(cu[i + 1])
        blk = res["cf"][256 * a:256 * b].reshape(256, b - a)
        _check("final_norm_cf", blk.T, u[a:b], e[a:b])
