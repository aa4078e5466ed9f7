"""A float64 model of every encoder stage, in the kernels' conventions, with element-wise error bounds.

Each stage is restated from the state dict in fp64, folded the way `ltr_create` folds it (ltr_api.cu): BatchNorm into
the 1x1 convolutions, the CLS query into u_h = W_k,h^T q_h / 8, the CLS residual into the fc bias, 1/8 into W_q,
the signature heads re-ordered head-major (the reference's interleaved channel is c = d*4 + h), and `merge` into
mlp1 ([W1a | W1b Wm]).  Composing the stages reproduces oracle.line_transformer_forward (tests/test_encoder_stages.py).

The bounds come from the precision model of DESIGN.md section 3, evaluated on the test's own data:
* a split-bf16 value hi + lo carries x to 2^-17 relative (U17); a tensor-core product is the 3-term split product,
  accumulated in fp32, so a GEMM output is off by at most C_GEMM * U17 * (|A| |W|^T) plus the fp32 rounding of the
  bias, plus U17 |out| when the output is re-quantised into an activation image;
* CUDA-core fp32 arithmetic (narrow MLP layers, LayerNorm, softmax, L2 norm) costs a few U24 per operation; GELU's
  erfc approximation 3.3e-7 absolute; `ex2.approx` 2^-22 relative plus the fp32 rounding of its argument;
* inside a stage whose intermediates are not observable (the token stage's positional MLP, the line positional head)
  errors carry through W in quadrature (`_carry`); ReLU and GELU are 1- and 1.13-Lipschitz.  The inputs of a GPU
  stage test are the GPU's own images, decoded exactly (hi + lo in fp64), so they carry no error.
The constants C_* multiply terms whose size depends on how the hardware accumulates; they were set on an H100 and
tests/test_encoder_stages.py records the measured worst err / bound per stage.
"""
from __future__ import annotations

import numpy as np
from scipy.special import erf

U17 = 2.0 ** -17
U24 = 2.0 ** -24
C_GEMM = 2.0      # x U17 (|A| |W|^T): weight split + fp32 accumulation of a tensor-core GEMM
C_F32 = 8.0       # x U24 per fp32 CUDA-core layer / reduction
GELU_ABS = 3.3e-7
LN_EPS = 1e-6
BN_EPS = 1e-5


def _f(x):
    return np.asarray(x, dtype=np.float64)


def fold(sd, conv, bn=None):
    w = _f(sd[conv + ".weight"])
    w = w.reshape(w.shape[0], -1)
    b = _f(sd[conv + ".bias"])
    if bn is not None:
        s = _f(sd[bn + ".weight"]) / np.sqrt(_f(sd[bn + ".running_var"]) + BN_EPS)
        w = w * s[:, None]
        b = b * s + _f(sd[bn + ".bias"]) - _f(sd[bn + ".running_mean"]) * s
    return w, b


def _pos_encoder(sd, prefix):
    """5 layers (4 with BatchNorm + ReLU) of a positional encoder: [(W, b)]."""
    return [fold(sd, f"{prefix}.{3 * l}", f"{prefix}.{3 * l + 1}" if l < 4 else None) for l in range(5)]


def gemm_bound(A, W, b, out=None, c=C_GEMM):
    """Element-wise bound of act(A W^T + b) on the split-bf16 engine from exact operands A (fp64): the 3-term split
    product accumulated in fp32, the fp32 bias, and the re-quantisation of `out` into an image when given."""
    e = c * U17 * (np.abs(A) @ np.abs(W).T) + U24 * np.abs(b)
    if out is not None:
        e = e + U17 * np.abs(out)
    return e


def _carry(e, W):
    """An input error bound e carried through W inside a stage whose intermediates the tests cannot observe: rounding
    errors of different inputs are independent, so they add in quadrature (|W| |e| would compound the worst case of
    every layer of the 5-layer positional MLP into a bound far above any real error)."""
    return np.sqrt((e * e) @ (W * W).T)


def layer_norm(v, g, beta, eps=LN_EPS, ddof=0):
    mu = v.mean(-1, keepdims=True)
    sig = np.sqrt(v.var(-1, keepdims=True, ddof=ddof) + eps)
    return (v - mu) / sig * g + beta


def layer_norm_bound(v, e_v, g, beta, eps=LN_EPS):
    """Bound of LN(v) in fp32 when v is off by at most e_v: first-order propagation (the mean moves by at most mean e_v,
    sigma by at most rms e_v) plus C_F32 U24 of fp32 arithmetic on the normalised value."""
    mu = v.mean(-1, keepdims=True)
    sig = np.sqrt(v.var(-1, keepdims=True) + eps)
    n = (v - mu) / sig
    ag = np.abs(g)
    prop = ag / sig * (e_v + e_v.mean(-1, keepdims=True) + np.abs(n) * np.sqrt((e_v ** 2).mean(-1, keepdims=True)))
    return prop + C_F32 * U24 * (ag * (np.abs(n) + 1) + np.abs(beta))


def gelu(x):
    return 0.5 * x * (1.0 + erf(x / np.sqrt(2.0)))


def softmax(s, axis=-1):
    e = np.exp(s - s.max(axis, keepdims=True))
    return e / e.sum(axis, keepdims=True)


def image_size_norm(width, height):
    return np.array([width / 2.0, height / 2.0]), max(width, height) * 0.7


class StageModel:
    """fp64 stages of the encoder for one state dict (the last descriptive layer is the live one)."""

    def __init__(self, sd, n_sig=None):
        self.wpe = _pos_encoder(sd, "klenc.word_position_enc.encoder")
        self.lpe = _pos_encoder(sd, "klenc.line_position_enc.encoder")
        nd = 0
        while f"klenc.desc_layers.{nd}.slf_attn.w_qs.weight" in sd:
            nd += 1
        p = f"klenc.desc_layers.{nd - 1}"
        g = lambda k: _f(sd[f"{p}.{k}"])
        self.cls = _f(sd["klenc.cls_token"]).reshape(256)
        q = g("slf_attn.w_qs.weight") @ self.cls + g("slf_attn.w_qs.bias")
        wk = g("slf_attn.w_ks.weight")
        self.U = np.stack([wk[h * 64:(h + 1) * 64].T @ q[h * 64:(h + 1) * 64] / 8.0 for h in range(4)])   # [4, 256]
        self.s_cls = self.U @ self.cls
        self.Wv, self.bv = g("slf_attn.w_vs.weight"), g("slf_attn.w_vs.bias")
        self.Wfc, self.bfc = g("slf_attn.fc.weight"), g("slf_attn.fc.bias") + self.cls   # CLS residual in the bias
        self.ln1 = g("slf_attn.layer_norm.weight"), g("slf_attn.layer_norm.bias")
        self.W1, self.b1 = g("pos_ffn.w_1.weight"), g("pos_ffn.w_1.bias")
        self.W2, self.b2 = g("pos_ffn.w_2.weight"), g("pos_ffn.w_2.bias")
        self.ln2 = g("pos_ffn.layer_norm.weight"), g("pos_ffn.layer_norm.bias")
        self.sig = []
        li = 0
        while f"selfattn.layers.{li}.attn.merge.weight" in sd and (n_sig is None or li < n_sig):
            sp = f"selfattn.layers.{li}"
            perm = np.array([d * 4 + h for h in range(4) for d in range(64)])   # head-major row -> interleaved c
            ws, bs = [], []
            for t in range(3):
                w, b = fold(sd, f"{sp}.attn.proj.{t}")
                sc = 0.125 if t == 0 else 1.0
                ws.append(w[perm] * sc)
                bs.append(b[perm] * sc)
            Wm, bm = fold(sd, f"{sp}.attn.merge")
            Wm = Wm[:, perm]
            W1, B1 = fold(sd, f"{sp}.mlp.0", f"{sp}.mlp.1")
            W2, B2 = fold(sd, f"{sp}.mlp.3")
            W1f = np.concatenate([W1[:, :256], W1[:, 256:] @ Wm], axis=1)
            B1f = B1 + W1[:, 256:] @ bm
            self.sig.append(dict(Wqkv=np.concatenate(ws), bqkv=np.concatenate(bs), W1=W1f, B1=B1f, W2=W2, B2=B2))
            li += 1
        self.Wf, self.bf = fold(sd, "final_proj")

    # ------------------------------------------------------------------ token stage
    def token(self, pnt, score, desc, width, height, pool_shift=None):
        """Raw tokens -> z [R, 1024] (z_h = sum_n p_h[n] x[n] over CLS + T tokens, head-major) and its bound.
        pnt [R,T,2], score [R,T,1], desc [R,T,256].  `pool_shift` plants an error: token `pool_shift` of every line
        is pooled into the next line's z."""
        R, T = desc.shape[:2]
        c, s = image_size_norm(width, height)
        a = np.concatenate([(_f(pnt) - c) / s, _f(score)], -1).reshape(R * T, 3)
        e = 2 * U24 * np.abs(a)
        for l, (W, b) in enumerate(self.wpe):
            y = a @ W.T + b
            if l == 0:   # 3 -> 32 on CUDA cores in fp32
                e = _carry(e, W) + C_F32 * U24 * (np.abs(a) @ np.abs(W).T + np.abs(b))
            else:        # register-A split-bf16 wgmma
                e = _carry(e, W) + gemm_bound(a, W, b)
            a = np.maximum(y, 0) if l < 4 else y
        x = _f(desc).reshape(R * T, 256) + a
        e_x = (e + U24 * np.abs(x)).reshape(R, T, 256)
        x = x.reshape(R, T, 256)
        sc = np.concatenate([np.broadcast_to(self.s_cls, (R, 1, 4)), x @ self.U.T], 1)          # [R, T+1, 4]
        e_s = np.concatenate([C_F32 * U24 * np.broadcast_to(np.abs(self.U) @ np.abs(self.cls), (R, 1, 4)),
                              _carry(e_x, self.U) + 2 * C_F32 * U24 * (np.abs(x) @ np.abs(self.U).T)], 1)
        p = softmax(sc, axis=1)
        r = e_s + 2 * U24 * (np.abs(sc) + np.abs(sc).max(1, keepdims=True)) + 4 * U24
        dp = p * (r + (p * r).sum(1, keepdims=True) + (T + 2) * U24)
        xc = np.concatenate([np.broadcast_to(self.cls, (R, 1, 256)), x], 1)                     # [R, T+1, 256]
        exc = np.concatenate([np.zeros((R, 1, 256)), e_x], 1)
        if pool_shift is not None:
            moved = p[:, 1 + pool_shift, :, None] * xc[:, 1 + pool_shift, None, :]            # [R, 4, 256]
            p = p.copy()
            p[:, 1 + pool_shift] = 0
        z = np.einsum("rnh,rnc->rhc", p, xc)
        if pool_shift is not None:
            z[1:] += moved[:-1]
        e_z = (np.einsum("rnh,rnc->rhc", dp, np.abs(xc)) + np.einsum("rnh,rnc->rhc", p, exc)
               + (T + 2) * U24 * np.einsum("rnh,rnc->rhc", p, np.abs(xc)))
        z = z.reshape(R, 1024)
        return z, e_z.reshape(R, 1024) + U17 * np.abs(z), sc

    def vproj(self, z):
        """V projection (block diagonal over heads) -> ctx [R, 256] image and its bound."""
        out = np.concatenate([z[:, h * 256:(h + 1) * 256] @ self.Wv[h * 64:(h + 1) * 64].T + self.bv[h * 64:(h + 1) * 64]
                              for h in range(4)], 1)
        e = np.concatenate([gemm_bound(z[:, h * 256:(h + 1) * 256], self.Wv[h * 64:(h + 1) * 64],
                                       self.bv[h * 64:(h + 1) * 64]) for h in range(4)], 1)
        return out, e + U17 * np.abs(out)

    # ------------------------------------------------------------------ line positional encoder
    def line_pos_head(self, sublines, resp, angle, width, height):
        """5 -> 32 -> 64 -> 128 (fp32 CUDA cores, small_mlp_kernel<false>) -> l128 image and its bound."""
        c, s = image_size_norm(width, height)
        mid = (_f(sublines)[:, 0] + _f(sublines)[:, 1]) / 2.0
        a = np.concatenate([(mid - c) / s, _f(resp), _f(angle)], -1)
        e = 2 * U24 * np.abs(a)
        for W, b in self.lpe[:3]:
            e = _carry(e, W) + C_F32 * U24 * (np.abs(a) @ np.abs(W).T + np.abs(b))
            a = np.maximum(a @ W.T + b, 0)
        return a, e + U17 * np.abs(a)

    def lin(self, A, W, b, relu=False):
        y = A @ W.T + b
        if relu:
            y = np.maximum(y, 0)
        return y, gemm_bound(A, W, b, y)

    def line_pos_l4(self, l128):
        return self.lin(l128, *self.lpe[3], relu=True)

    def line_pos_l5(self, l256):
        return self.lin(l256, *self.lpe[4])

    # ------------------------------------------------------------------ line stage
    def fc_ln1(self, ctx, ddof=0):
        v = ctx @ self.Wfc.T + self.bfc
        y = layer_norm(v, *self.ln1, ddof=ddof)
        return y, layer_norm_bound(v, gemm_bound(ctx, self.Wfc, self.bfc), *self.ln1) + U17 * np.abs(y)

    def w1_gelu(self, y1):
        v = y1 @ self.W1.T + self.b1
        g = gelu(v)
        return g, 1.13 * gemm_bound(y1, self.W1, self.b1) + GELU_ABS + C_F32 * U24 * np.abs(v) + U17 * np.abs(g)

    def w2_ln2(self, g, y1, lpos, ddof=0):
        v = g @ self.W2.T + self.b2 + y1
        x = lpos + layer_norm(v, *self.ln2, ddof=ddof)
        e = layer_norm_bound(v, gemm_bound(g, self.W2, self.b2) + U24 * np.abs(v), *self.ln2)
        return x, e + U24 * np.abs(lpos) + U17 * np.abs(x)

    # ------------------------------------------------------------------ signature layers
    def qkv(self, x, l):
        L = self.sig[l]
        return self.lin(x, L["Wqkv"], L["bqkv"])

    def mlp1(self, x, o, l):
        L = self.sig[l]
        return self.lin(np.concatenate([x, o], 1), L["W1"], L["B1"], relu=True)

    def mlp2(self, hm, x, l):
        L = self.sig[l]
        y = hm @ L["W2"].T + L["B2"] + x
        return y, gemm_bound(hm, L["W2"], L["B2"]) + U24 * np.abs(y) + U17 * np.abs(y)

    def final_rows(self, x):
        """final_proj + L2 in the epilogue -> unit rows (fp32) and their bound."""
        y = x @ self.Wf.T + self.bf
        e_y = gemm_bound(x, self.Wf, self.bf)
        n = np.linalg.norm(y, axis=1, keepdims=True)
        u = y / np.maximum(n, 1e-12)
        return u, (e_y + np.abs(u) * np.linalg.norm(e_y, axis=1, keepdims=True)) / n + C_F32 * U24 * (np.abs(u) + 1 / 16)

    def final_proj(self, x):
        """final_proj alone, fp32 rows (the channel-first path's yf)."""
        y = x @ self.Wf.T + self.bf
        return y, gemm_bound(x, self.Wf, self.bf) + U24 * np.abs(y)


def attention(qkv, cu, skip_key=None, bf16_p=False):
    """Signature attention per image segment [cu[i], cu[i+1]) -> o [R, 256] head-major, and its bound.  qkv [R, 768]
    image values (q pre-scaled by 1/8).  Planted errors: `skip_key` = (image, key) drops one key of that image from
    every row's softmax; `bf16_p` keeps only the hi part of the probabilities (after normalisation)."""
    R = qkv.shape[0]
    o = np.zeros((R, 256))
    e = np.zeros((R, 256))
    for i in range(len(cu) - 1):
        a, b = int(cu[i]), int(cu[i + 1])
        if a == b:
            continue
        for h in range(4):
            q, k, v = (qkv[a:b, t * 256 + h * 64:t * 256 + (h + 1) * 64] for t in range(3))
            s = q @ k.T
            e_s = C_GEMM * U17 * (np.abs(q) @ np.abs(k).T)
            if skip_key is not None and skip_key[0] == i:
                s[:, skip_key[1]] = -np.inf
            p = softmax(s)
            if bf16_p:
                from tests.test_numeric_formulas import bf16_round
                p = bf16_round(p.astype(np.float32)).astype(np.float64)
            rr = e_s + 2 * U24 * (np.abs(np.where(np.isfinite(s), s, 0)) + np.abs(s.max(1, keepdims=True))) + 2.0 ** -21
            dp = p * (rr + (p * rr).sum(1, keepdims=True) + U17)
            oo = p @ v
            o[a:b, h * 64:(h + 1) * 64] = oo
            e[a:b, h * 64:(h + 1) * 64] = dp @ np.abs(v) + C_GEMM * U17 * (p @ np.abs(v)) + U17 * np.abs(oo)
    return o, e


def l2_rows_bound(y):
    """final_norm_kernel on fp32 rows y: unit rows and the fp32 bound of the normalisation itself."""
    n = np.linalg.norm(y, axis=1, keepdims=True)
    u = y / np.maximum(n, 1e-12)
    return u, C_F32 * U24 * (np.abs(u) + 1 / 16)


# ------------------------------------------------------------------ split-bf16 emulation (CPU, planted errors)
def split(x):
    from tests.test_numeric_formulas import split as _split
    hi, lo = _split(np.asarray(x, dtype=np.float32))
    return hi.astype(np.float64), lo.astype(np.float64)


def emulate_gemm(A, W, b, drop_lo_hi=False):
    """The tensor-core GEMM on the CPU: A split (as the producer's image holds it), W split, the 3-term product (or
    without a_lo w_hi), fp32 result and bias, then the output image's split.  Returns the decoded output image."""
    ah, al = split(A)
    wh, wl = split(W)
    acc = ah @ wh.T + ah @ wl.T + (0 if drop_lo_hi else al @ wh.T)
    y = (acc.astype(np.float32) + np.asarray(b, np.float32)).astype(np.float64)
    hi, lo = split(y)
    return hi + lo, ah + al
