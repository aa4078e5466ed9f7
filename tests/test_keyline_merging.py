"""Key-line merging against float64, stage by stage: the tensor-core subline distances `dist_sub`, the segment mean
`dist_key` (segmean_kernel) and the nearest-neighbour decisions taken on it (row_argmin / col_argmin / mutual_kernel).

The merged path never runs the matcher's exact re-check (match_exact_kernel): `dist_sub` comes straight from the
tensor cores, so its contract is a bound, not bits.  Each stage is fed the GPU's own output of the stage before:
1. `dist_sub` against the float64 distance of the fp32 descriptors, inside the element-wise bound `e_D` of the 3-term
   split-bf16 product (d = 256); bit for bit against the fp32 FMA model for other d (dist_kernel).
2. `dist_key` bit for bit against a C model of segmean_kernel run on the GPU's `dist_sub`, and against the float64
   merge A0 D64 A1^T inside `A0 e_D A1^T + 2 (n_a + n_b) U24 max D`.
3. matches0 / scores0 / nn1 / counts bit for bit against `decisions(dist_key)`, and against the float64 decisions on
   the rows whose float64 margins exceed twice the bound.  The other rows are counted and printed (`-s`).
Every GPU output buffer is filled with a NaN sentinel first: gaps between the pairs' blocks must keep it.
"""
import ctypes
import os
import re
import shutil
import subprocess
from fractions import Fraction

import numpy as np
import pytest
import torch

from linetr_b200 import _native as N
from linetr_b200 import _ops, nn_matcher as nnm
from linetr_b200.line_process import get_dist_matrix
from tests import helpers as H
from tests.encoder_stage_model import C_GEMM, U17, U24, split
from tests.test_matcher_edges import _round_f32, decisions, dist32_model, model32  # noqa: F401 (model32: fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda", 0)
ROWS, CF = N.LAYOUT_ROWS, N.LAYOUT_CHANNEL_FIRST
SENT = 0x7FC5A5A5            # a quiet-NaN bit pattern no kernel produces
MAXG = 65535                 # grid y / z limit


def _code(name):
    hdr = open(os.path.join(ROOT, "include", "linetr_b200.h")).read()
    return int(re.search(rf"#define\s+{name}\s+\((-?\d+)\)", hdr).group(1))


# ------------------------------------------------------------------ host references
_SEGMEAN_SRC = r"""
#include <math.h>
/* segmean_kernel (match_kernels.cuh) for one pair: D row-major [S0, ld], CSR offsets off0 [K0+1], off1 [K1+1] */
void model_segmean(const float* D, long ld, const int* off0, int K0, const int* off1, int K1, float* out) {
  for (int a = 0; a < K0; ++a)
    for (int b = 0; b < K1; ++b) {
      const int i0 = off0[a] - off0[0], i1 = off0[a + 1] - off0[0];
      const int j0 = off1[b] - off1[0], j1 = off1[b + 1] - off1[0];
      const float wa = 1.f / (float)(i1 - i0), wb = 1.f / (float)(j1 - j0);
      float acc = 0.f;
      for (int j = j0; j < j1; ++j) {
        float t = 0.f;
        for (int i = i0; i < i1; ++i) t = fmaf(wa, D[(long)i * ld + j], t);
        acc = fmaf(t, wb, acc);
      }
      out[(long)a * K1 + b] = acc;
    }
}
"""


@pytest.fixture(scope="module")
def segmean_model(tmp_path_factory):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler for the segmean model")
    td = tmp_path_factory.mktemp("segmean_model")
    src, so = str(td / "segmean.c"), str(td / "segmean.so")
    with open(src, "w") as f:
        f.write(_SEGMEAN_SRC)
    # no contraction, no fast-math: every operation rounds as written, the division correctly
    subprocess.check_call([cc, "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", "-o", so, src, "-lm"])
    lib = ctypes.CDLL(so)
    f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
    i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
    lib.model_segmean.argtypes = [f32p, ctypes.c_long, i32p, ctypes.c_int, i32p, ctypes.c_int, f32p]
    return lib


def segmean32(lib, D, off0, off1):
    """fp32 [S0, S1] and local CSR offsets -> the bits segmean_kernel writes, fp32 [K0, K1]."""
    D = np.ascontiguousarray(D, np.float32)
    off0, off1 = np.ascontiguousarray(off0, np.int32), np.ascontiguousarray(off1, np.int32)
    K0, K1 = len(off0) - 1, len(off1) - 1
    out = np.empty((K0, K1), np.float32)
    if out.size:
        lib.model_segmean(D, D.shape[1], off0, K0, off1, K1, out)
    return out


def dist64(a, b):
    s = np.asarray(a, np.float64) @ np.asarray(b, np.float64).T
    return np.maximum(2.0 - 2.0 * s, 0.0), s


def sub_bound(a, b, s):
    """e_D: 3-term split product (C_GEMM U17 |a| |b|^T) and its fp32 accumulation (U24 |s|), doubled by 2 - 2s, plus
    the rounding of 2 - 2s itself.  The clip at 0 is 1-Lipschitz and does not widen it."""
    ab = np.abs(np.asarray(a, np.float64)) @ np.abs(np.asarray(b, np.float64)).T
    return 2.0 * (C_GEMM * U17 * ab + U24 * np.abs(s)) + U24 * np.abs(2.0 - 2.0 * s)


def adjacency(off):
    off = np.asarray(off, np.int64)
    A = np.zeros((len(off) - 1, off[-1] - off[0]))
    for k in range(len(off) - 1):
        A[k, off[k] - off[0]:off[k + 1] - off[0]] = 1.0 / (off[k + 1] - off[k])
    return A


def merge64(D, off0, off1):
    return adjacency(off0) @ D @ adjacency(off1).T


def key_bound(e_D, D64, off0, off1):
    """A0 e_D A1^T + 2 (n_a + n_b) U24 max D over the block: the input bound carried through the mean, and the fp32
    rounding of the weights and of both fmaf chains."""
    off0, off1 = np.asarray(off0, np.int64) - off0[0], np.asarray(off1, np.int64) - off1[0]
    mx = np.maximum.reduceat(np.maximum.reduceat(D64 + e_D, off0[:-1], axis=0), off1[:-1], axis=1)
    n = np.diff(off0)[:, None] + np.diff(off1)[None, :]
    return merge64(e_D, off0, off1) + 2.0 * n * U24 * mx


def _top2(x, axis):
    if x.shape[axis] < 2:
        return np.full(x.shape[1 - axis], np.inf)
    s = np.sort(x, axis=axis)
    return s[1] - s[0] if axis == 0 else s[:, 1] - s[:, 0]


def decisive(k64, bnd, thr, mutual):
    """Rows whose float64 margins (top-2 gap, |best - thr|, with mutual the top-2 gap of the partner column) exceed
    twice the largest bound of the entries involved."""
    n0, n1 = k64.shape
    if n0 == 0 or n1 == 0:
        return np.ones(n0, bool)
    idx = np.argmin(k64, axis=1)
    margin = np.minimum(_top2(k64, 1), np.abs(k64[np.arange(n0), idx] - float(thr)))
    b = bnd.max(axis=1)
    if mutual:
        margin = np.minimum(margin, _top2(k64, 0)[idx])
        b = np.maximum(b, bnd.max(axis=0)[idx])
    return margin > 2.0 * b


def emulate_dist(a, b, drop_lo_hi=False):
    """The tensor-core distance on the CPU: both operands split into bf16 hi + lo, the 3-term product (or without
    a_lo b_hi) rounded once to fp32, then fmaf(-2, acc, 2) and the clip."""
    ah, al = split(a)
    bh, bl = split(b)
    acc = (ah @ bh.T + ah @ bl.T + (0 if drop_lo_hi else al @ bh.T)).astype(np.float32).astype(np.float64)
    return np.maximum((2.0 - 2.0 * acc).astype(np.float32), np.float32(0))


# ------------------------------------------------------------------ data
def _unit(rng, n, d=256):
    x = rng.standard_normal((n, d))
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def _csr(counts):
    return np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)


def make_image_pair(rng, c0, c1, d=256):
    """Unit descriptors for key lines with subline counts c0 / c1: side-0 sublines sit near a random side-1 subline,
    one side-1 key line is a copy of another (exact ties of dist_key), an eighth of side 0 is unrelated."""
    c0, c1 = np.asarray(c0, np.int64), np.asarray(c1, np.int64)
    S0, S1 = int(c0.sum()), int(c1.sum())
    b = _unit(rng, S1, d)
    off1 = _csr(c1)
    same = np.nonzero(c1[1:] == c1[:-1])[0]
    if len(same):
        k = int(same[0])
        b[off1[k + 1]:off1[k + 2]] = b[off1[k]:off1[k + 1]]
    if S1:
        a = b[rng.integers(0, S1, S0)] + _unit(rng, S0, d) * rng.uniform(0.3, 1.0, (S0, 1))
        far = rng.random(S0) < 0.125
        a[far] = _unit(rng, int(far.sum()), d)
        a /= np.linalg.norm(a, axis=1, keepdims=True)
    else:
        a = _unit(rng, S0, d)
    return dict(a=a.astype(np.float32), b=b.astype(np.float32), off0=_csr(c0), off1=off1)


def counts_random(rng, K, lo=1, hi=4):
    return rng.integers(lo, hi + 1, K)


def counts_summing(rng, S, hi=4):
    """Random subline counts in 1..hi that add up to exactly S."""
    out = []
    while S > 0:
        c = int(rng.integers(1, min(hi, S) + 1))
        out.append(c)
        S -= c
    return np.array(out, np.int64)


class Ref:
    """float64 references of one pair, computed once."""

    def __init__(self, p):
        self.D64, s = dist64(p["a"], p["b"])
        self.e_D = sub_bound(p["a"], p["b"], s)
        if self.D64.size:
            self.K64 = merge64(self.D64, p["off0"], p["off1"])
            self.e_K = key_bound(self.e_D, self.D64, p["off0"], p["off1"])
        else:
            self.K64 = self.e_K = np.zeros((len(p["off0"]) - 1, len(p["off1"]) - 1))


class Stats:
    def __init__(self, what):
        self.what, self.sub, self.key, self.nondec, self.rows = what, 0.0, 0.0, 0, 0

    def report(self):
        print(f"\n[{self.what}] worst err/bound: dist_sub {self.sub:.3f}, dist_key {self.key:.3f}; "
              f"non-decisive rows {self.nondec} of {self.rows}")


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def sentinel(n, offset=0):
    """A float32 device buffer of n elements starting `offset` elements into a fresh sentinel-filled allocation
    (offset 1: 4 bytes off 32-byte alignment)."""
    buf = torch.full((n + offset + 64,), SENT, dtype=torch.int32, device=DEV).view(torch.float32)
    return buf, buf[offset:]


def bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def check_blocks(flat, shapes, stride, what):
    """flat: the whole host copy of an output buffer view; blocks [r_p, c_p] at p * stride.  Returns the blocks and
    asserts that everything outside them holds the sentinel."""
    u = bits(flat)
    untouched = np.ones(len(u), bool)
    blocks = []
    for p, (r, c) in enumerate(shapes):
        untouched[p * stride:p * stride + r * c] = False
        blocks.append(flat[p * stride:p * stride + r * c].reshape(r, c))
    bad = np.nonzero(untouched & (u != SENT))[0]
    assert bad.size == 0, f"{what}: {bad.size} elements written outside the pairs' blocks, first at {bad[:4].tolist()}"
    return blocks


def check_pair(seg32, p, ref, ds, dk, m0, s0, nn1, cnt, thr, mutual, st, what):
    """Stages 1-3 of one pair (d = 256) from the GPU's dist_sub ds, dist_key dk and decisions (m0 None: bounds only)."""
    if ds.size:
        r = float((np.abs(ds.astype(np.float64) - ref.D64) / ref.e_D).max())
        st.sub = max(st.sub, r)
        assert r <= 1.0, f"{what}: dist_sub off by {r:.2f} x e_D"
    bad = np.nonzero(bits(dk) != bits(segmean32(seg32, ds, p["off0"], p["off1"])))
    assert bad[0].size == 0, f"{what}: dist_key differs from the segmean model at {list(zip(*bad))[:4]}"
    if dk.size:
        r = float((np.abs(dk.astype(np.float64) - ref.K64) / ref.e_K).max())
        st.key = max(st.key, r)
        assert r <= 1.0, f"{what}: dist_key off by {r:.2f} x its float64 bound"
    K0, K1 = dk.shape
    if m0 is None:
        return
    want, idx, wnn1 = decisions(dk, thr, mutual)
    assert np.array_equal(m0, want), f"{what}: matches0 rows {np.nonzero(m0 != want)[0][:8].tolist()}"
    assert int(cnt) == int((want >= 0).sum()), what
    if K1 == 0:
        assert np.isinf(s0).all(), what
    else:
        assert np.array_equal(bits(s0), bits(dk[np.arange(K0), idx])), what
    if mutual and K1:
        assert np.array_equal(nn1, wnn1 if K0 else np.full(K1, -1)), what
    ok = decisive(ref.K64, ref.e_K, thr, mutual)
    w64 = decisions(ref.K64, float(thr), mutual)[0]
    assert np.array_equal(m0[ok], w64[ok]), f"{what}: decisive rows differ from float64"
    st.nondec += int((~ok).sum())
    st.rows += K0


# ------------------------------------------------------------------ ltr_match on a batch
class Batch:
    def __init__(self, pairs):
        self.pairs = pairs
        self.S0 = [len(p["a"]) for p in pairs]
        self.S1 = [len(p["b"]) for p in pairs]
        self.K0 = [len(p["off0"]) - 1 for p in pairs]
        self.K1 = [len(p["off1"]) - 1 for p in pairs]
        self.cu0, self.cu1 = _csr(self.S0), _csr(self.S1)
        self.cuk0, self.cuk1 = _csr(self.K0), _csr(self.K1)
        self.sub_off0 = _csr(np.concatenate([np.diff(p["off0"]) for p in pairs]))
        self.sub_off1 = _csr(np.concatenate([np.diff(p["off1"]) for p in pairs]))
        self.refs = {}

    def ref(self, p, keep=True):
        if p in self.refs:
            return self.refs[p]
        r = Ref(self.pairs[p])
        if keep:
            self.refs[p] = r
        return r

    def pack(self, side, layout, d=256):
        xs = [p["a"] if side == 0 else p["b"] for p in self.pairs]
        flat = np.concatenate([(x if layout == ROWS else x.T).reshape(-1) for x in xs])
        return flat if flat.size else np.zeros(d, np.float32)


def run_batch(B, layout, thr, mutual, *, d=256, extra_n=0, extra_k=0, stride_key=0, offset=0):
    """ltr_match with merging into sentinel-filled buffers -> host (dist_sub, dist_key, outputs, strides)."""
    mx0, mx1 = max(B.S0) + extra_n, max(B.S1) + extra_n
    mk0, mk1 = max(B.K0) + extra_k, max(B.K1) + extra_k
    P = len(B.pairs)
    skey = stride_key or mk0 * mk1
    bs, ds = sentinel(P * mx0 * mx1, offset)
    bk, dk = sentinel(P * skey, offset)
    tk0, tk1 = int(B.cuk0[-1]), int(B.cuk1[-1])
    out = dict(dist_sub=ds, dist_key=dk, matches0=torch.full((tk0 + 1,), -7, dtype=torch.int32, device=DEV),
               scores0=torch.full((tk0 + 1,), SENT, dtype=torch.int32, device=DEV).view(torch.float32),
               nn1=torch.full((tk1 + 1,), -7, dtype=torch.int32, device=DEV),
               counts=torch.full((P,), -7, dtype=torch.int32, device=DEV))
    keep = [_t(B.pack(0, layout, d)), _t(B.pack(1, layout, d))] + [_t(x) for x in (
        B.cu0, B.cu1, B.sub_off0, B.sub_off1, B.cuk0, B.cuk1)]
    inp = dict(desc0=keep[0], desc1=keep[1], layout=layout, d=d, n_pairs=P, cu0=keep[2], cu1=keep[3],
               sub_off0=keep[4], sub_off1=keep[5], cuk0=keep[6], cuk1=keep[7], max_n0=mx0, max_n1=mx1,
               max_k0=mk0, max_k1=mk1, dist_pair_stride=stride_key, nn_thresh=float(thr), mutual=bool(mutual),
               total_n0=int(B.cu0[-1]), total_n1=int(B.cu1[-1]))
    _ops._match("ltr_match", DEV, inp, out)
    torch.cuda.synchronize()
    host = {k: v.cpu().numpy() for k, v in out.items()}
    host["dist_sub"] = bs.cpu().numpy()[offset:]
    host["dist_key"] = bk.cpu().numpy()[offset:]
    return host, mx0 * mx1, skey


def check_batch(seg32, B, host, ssub, skey, thr, mutual, st, what, keep_refs=True):
    dsub = check_blocks(host["dist_sub"], list(zip(B.S0, B.S1)), ssub, what + " dist_sub")
    dkey = check_blocks(host["dist_key"], list(zip(B.K0, B.K1)), skey, what + " dist_key")
    tk0, tk1 = int(B.cuk0[-1]), int(B.cuk1[-1])
    assert host["matches0"][tk0] == -7 and host["nn1"][tk1] == -7, what   # nothing past the last key line
    for p in range(len(B.pairs)):
        sl0, sl1 = slice(B.cuk0[p], B.cuk0[p + 1]), slice(B.cuk1[p], B.cuk1[p + 1])
        check_pair(seg32, B.pairs[p], B.ref(p, keep_refs), dsub[p], dkey[p], host["matches0"][sl0],
                   host["scores0"][sl0], host["nn1"][sl1], host["counts"][p], thr, mutual, st, f"{what} pair {p}")


def _case(name, seed):
    rng = np.random.default_rng(seed)
    R = counts_random
    if name == "ones_vs_split":        # the engine: one side all 1, the other split
        pairs = [make_image_pair(rng, np.ones(150, int), R(rng, 90)),
                 make_image_pair(rng, R(rng, 70), np.ones(140, int))]
    elif name == "random_1_4":
        pairs = [make_image_pair(rng, R(rng, k0), R(rng, k1)) for k0, k1 in ((60, 75), (90, 40), (33, 95))]
    elif name == "long":               # key lines spanning several 128-row tiles
        pairs = [make_image_pair(rng, [7, 1, 64, 129, 2, 300, 1], [300, 3, 129, 64, 7, 1]),
                 make_image_pair(rng, [129, 7], [1, 1, 64, 2, 300])]
    elif name == "single_keyline":     # K = 1: one key line holds every subline of its image
        pairs = [make_image_pair(rng, [257], R(rng, 40)), make_image_pair(rng, R(rng, 30), [130]),
                 make_image_pair(rng, [1], [1]), make_image_pair(rng, [200], [129])]
    elif name == "segmean_blocks":     # K0 around segmean's 8-row blocks x K1 around its 32-column blocks
        pairs = [make_image_pair(rng, R(rng, k0, 1, 2), R(rng, k1, 1, 2))
                 for k0 in (1, 7, 8, 9, 65) for k1 in (1, 31, 32, 33, 257)]
    elif name == "tile_edges":         # S around the 128-row tiles, S1 % 8 == 0 and != 0
        pairs = [make_image_pair(rng, counts_summing(rng, s0), counts_summing(rng, s1))
                 for s0, s1 in ((127, 128), (128, 129), (129, 256), (256, 257), (257, 136), (128, 127))]
    elif name == "ragged_empty":       # images without key lines on either side
        pairs = [make_image_pair(rng, R(rng, 20), []), make_image_pair(rng, [], R(rng, 30)),
                 make_image_pair(rng, R(rng, 45), R(rng, 50)), make_image_pair(rng, [], []),
                 make_image_pair(rng, [3, 1], R(rng, 9))]
    else:
        raise KeyError(name)
    return Batch(pairs)


CASES = ["ones_vs_split", "random_1_4", "long", "single_keyline", "segmean_blocks", "tile_edges", "ragged_empty"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_batch_chain(segmean_model, name):
    """ltr_match with merging, rows and channel-first, mutual on and off, aligned and 4 bytes off, with max_n / max_k
    and the caller's dist_pair_stride above every pair's own."""
    B = _case(name, seed=CASES.index(name) + 100)
    thr = np.float32(0.9)
    st = Stats(name)
    for layout in (ROWS, CF):
        for mutual in (True, False):
            extra = (3, 2) if mutual else (0, 0)
            skey = (max(B.K0) + extra[1]) * (max(B.K1) + extra[1]) + 37 if not mutual else 0
            runs = []
            for offset in (0, 1):
                host, ssub, sk = run_batch(B, layout, thr, mutual, extra_n=extra[0], extra_k=extra[1], stride_key=skey,
                                           offset=offset)
                what = f"{name} layout={layout} mutual={mutual} offset={offset}"
                check_batch(segmean_model, B, host, ssub, sk, thr, mutual, st, what)
                runs.append(host)
            for k in runs[0]:             # vector and scalar store paths: the same bits
                assert np.array_equal(bits(runs[0][k]) if runs[0][k].dtype == np.float32 else runs[0][k],
                                      bits(runs[1][k]) if runs[1][k].dtype == np.float32 else runs[1][k]), (name, k)
    st.report()


@pytest.mark.gpu
@pytest.mark.parametrize("d", [16, 272])
def test_batch_chain_fp32_dimension(segmean_model, model32, d):
    """d != 256 (dist_kernel): dist_sub equals the fp32 FMA model bit for bit, the rest of the chain as for d = 256."""
    rng = np.random.default_rng(d)
    B = Batch([make_image_pair(rng, counts_random(rng, k0), counts_random(rng, k1), d=d)
               for k0, k1 in ((40, 33), (1, 70), (65, 9))])
    for layout in (ROWS, CF):
        for mutual in (True, False):
            host, ssub, skey = run_batch(B, layout, np.float32(0.9), mutual, d=d)
            dsub = check_blocks(host["dist_sub"], list(zip(B.S0, B.S1)), ssub, "dist_sub")
            dkey = check_blocks(host["dist_key"], list(zip(B.K0, B.K1)), skey, "dist_key")
            for p, pp in enumerate(B.pairs):
                what = f"d={d} layout={layout} mutual={mutual} pair {p}"
                assert np.array_equal(bits(dsub[p]), bits(dist32_model(model32, pp["a"], pp["b"], 0))), what
                want = segmean32(segmean_model, dsub[p], pp["off0"], pp["off1"])
                assert np.array_equal(bits(dkey[p]), bits(want)), what
                sl0 = slice(B.cuk0[p], B.cuk0[p + 1])
                want = decisions(dkey[p], np.float32(0.9), mutual)[0]
                assert np.array_equal(host["matches0"][sl0], want), what
                assert host["counts"][p] == (want >= 0).sum(), what


# ------------------------------------------------------------------ the dense output without merging (get_dist_matrix)
@pytest.mark.gpu
@pytest.mark.parametrize("layout", [ROWS, CF])
def test_tc_dense_store_paths(layout):
    """dist_key of ltr_match with d = 256 and no merging: float64 bound, the same bits from the 256-bit vector store
    (nb % 8 == 0, stride % 8 == 0, 32-byte aligned) and the scalar store, nothing written outside a pair's block."""
    rng = np.random.default_rng(7 + layout)
    sizes = [(127, 128), (129, 136), (1, 8), (257, 256), (64, 0), (0, 16), (130, 255)]   # mx0 * mx1 % 8 == 0
    pairs = [make_image_pair(rng, np.ones(s0, int), np.ones(s1, int)) for s0, s1 in sizes]
    B = Batch(pairs)
    mx0, mx1 = max(B.S0), max(B.S1)
    st = Stats(f"dense layout={layout}")
    res = {}
    for stride in (0, mx0 * mx1 + 8, mx0 * mx1 + 3):
        for offset in (0, 1):
            sk = stride or mx0 * mx1
            bk, dk = sentinel(len(pairs) * sk, offset)
            keep = [_t(B.pack(0, layout)), _t(B.pack(1, layout)), _t(B.cu0), _t(B.cu1)]
            inp = dict(desc0=keep[0], desc1=keep[1], layout=layout, d=256, n_pairs=len(pairs), cu0=keep[2], cu1=keep[3],
                       max_n0=mx0, max_n1=mx1, dist_pair_stride=stride, nn_thresh=0.0, mutual=False,
                       total_n0=int(B.cu0[-1]), total_n1=int(B.cu1[-1]))
            _ops._match("ltr_match", DEV, inp, dict(dist_key=dk))
            flat = bk.cpu().numpy()[offset:]
            blocks = check_blocks(flat, sizes, sk, f"stride={stride} offset={offset}")
            for p in range(len(pairs)):
                ref = B.ref(p)
                if blocks[p].size:
                    r = float((np.abs(blocks[p].astype(np.float64) - ref.D64) / ref.e_D).max())
                    st.sub = max(st.sub, r)
                    assert r <= 1.0, (stride, offset, p, r)
            res[(stride, offset)] = [bits(b) for b in blocks]
    base = res[(0, 0)]
    for key, blocks in res.items():
        assert all(np.array_equal(x, y) for x, y in zip(base, blocks)), key
    st.report()


# ------------------------------------------------------------------ ltr_match_indexed on image pools
def _pool(images, layout):
    """Images (a or b of make_image_pair dicts, with CSR) -> device pool: descriptors, cu, tiles, cuk, sub_off."""
    x = [im[0] for im in images]
    cu = _csr([len(v) for v in x])
    cuk = _csr([len(im[1]) - 1 for im in images])
    sub_off = _csr(np.concatenate([np.diff(im[1]) for im in images]))
    flat = np.concatenate([(v if layout == ROWS else v.T).reshape(-1) for v in x])
    tile_off = _ops.tile_offsets(cu)
    desc, cu_d, to_d = _t(flat), _t(cu), _t(tile_off)
    tiles = _ops.image_tiles(desc, layout, cu, cu_d, to_d, int(tile_off[-1]))
    return dict(layout=layout, desc=desc, cu=cu, cu_d=cu_d, to_d=to_d, n_tiles=int(tile_off[-1]), tiles=tiles, cuk=cuk,
                cuk_d=_t(cuk), sub_off_d=_t(sub_off), S=[len(v) for v in x], K=[len(im[1]) - 1 for im in images])


def run_indexed(pool0, pool1, pr, thr, mutual, *, extra=0, stride_key=0, offset=0, maxes=None):
    P = len(pr)
    i0, i1 = np.array([p[0] for p in pr], np.int32), np.array([p[1] for p in pr], np.int32)
    S0, S1 = [pool0["S"][i] for i in i0], [pool1["S"][i] for i in i1]
    K0, K1 = [pool0["K"][i] for i in i0], [pool1["K"][i] for i in i1]
    mx0, mx1, mk0, mk1 = maxes or (max(S0) + extra, max(S1) + extra, max(K0) + extra, max(K1) + extra)
    skey = stride_key or mk0 * mk1
    oo0, oo1 = _csr(K0), _csr(K1)
    bs, ds = sentinel(P * mx0 * mx1, offset)
    bk, dk = sentinel(P * skey, offset)
    out = dict(dist_sub=ds, dist_key=dk,
               matches0=torch.full((int(oo0[-1]) + 1,), -7, dtype=torch.int32, device=DEV),
               scores0=torch.full((int(oo0[-1]) + 1,), SENT, dtype=torch.int32, device=DEV).view(torch.float32),
               nn1=torch.full((int(oo1[-1]) + 1,), -7, dtype=torch.int32, device=DEV),
               counts=torch.full((P,), -7, dtype=torch.int32, device=DEV))
    keep = [_t(i0), _t(i1), _t(oo0), _t(oo1)]
    inp = dict(desc0=pool0["desc"], desc1=pool1["desc"], layout=pool0["layout"], d=256, n_pairs=P, cu0=pool0["cu_d"],
               cu1=pool1["cu_d"], sub_off0=pool0["sub_off_d"], sub_off1=pool1["sub_off_d"], cuk0=pool0["cuk_d"],
               cuk1=pool1["cuk_d"], max_n0=mx0, max_n1=mx1, max_k0=mk0, max_k1=mk1, dist_pair_stride=stride_key,
               nn_thresh=float(thr), mutual=bool(mutual), total_n0=int(pool0["cu"][-1]), total_n1=int(pool1["cu"][-1]))
    idx = dict(img0=keep[0], img1=keep[1], tiles0=pool0["tiles"], tiles1=pool1["tiles"], tile_off0=pool0["to_d"],
               tile_off1=pool1["to_d"], n_tiles0=pool0["n_tiles"], n_tiles1=pool1["n_tiles"], out_off0=keep[2],
               out_off1=keep[3], total_out0=int(oo0[-1]), total_out1=int(oo1[-1]))
    _ops._match("ltr_match_indexed", DEV, inp, out, idx=idx)
    torch.cuda.synchronize()
    host = {k: v.cpu().numpy() for k, v in out.items()}
    host["dist_sub"] = bs.cpu().numpy()[offset:]
    host["dist_key"] = bk.cpu().numpy()[offset:]
    return host, dict(S0=S0, S1=S1, K0=K0, K1=K1, oo0=oo0, oo1=oo1, ssub=mx0 * mx1, skey=skey,
                      maxes=(mx0, mx1, mk0, mk1))


@pytest.mark.gpu
@pytest.mark.parametrize("same_pool", [False, True])
@pytest.mark.parametrize("layout", [ROWS, CF])
def test_indexed_pools(segmean_model, same_pool, layout):
    """ltr_match_indexed with merging: one image in several pairs, pool 0 = pool 1 with pairs (i, i), max_n / max_k
    above every pair's own, a caller stride and a misaligned output."""
    rng = np.random.default_rng(21 + 2 * same_pool + layout)
    shapes = [([7, 1, 64, 129], [2, 3, 1]), (counts_random(rng, 40), counts_random(rng, 130)), ([1], [300]),
              (counts_summing(rng, 128), counts_summing(rng, 136)), (counts_random(rng, 9), counts_random(rng, 33))]
    ims = [make_image_pair(rng, c0, c1) for c0, c1 in shapes]
    img0 = [(m["a"], m["off0"]) for m in ims]
    img1 = img0 if same_pool else [(m["b"], m["off1"]) for m in ims]
    pool0 = _pool(img0, layout)
    pool1 = pool0 if same_pool else _pool(img1, layout)
    pr = [(0, 1), (0, 0), (1, 0), (2, 3), (0, 4), (3, 3), (4, 2), (1, 1), (0, 2)]
    refs = {}
    st = Stats(f"indexed same_pool={same_pool} layout={layout}")
    thr = np.float32(0.9)
    for mutual in (True, False):
        runs = []
        for offset, extra, skey in ((0, 0, 0), (1, 5, 0), (0, 2, 100003)):
            host, g = run_indexed(pool0, pool1, pr, thr, mutual, extra=extra, stride_key=skey, offset=offset)
            what = f"mutual={mutual} offset={offset} extra={extra} stride={skey}"
            dsub = check_blocks(host["dist_sub"], list(zip(g["S0"], g["S1"])), g["ssub"], what + " dist_sub")
            dkey = check_blocks(host["dist_key"], list(zip(g["K0"], g["K1"])), g["skey"], what + " dist_key")
            assert host["matches0"][-1] == -7 and host["nn1"][-1] == -7, what
            for p, (a, b) in enumerate(pr):
                pp = dict(a=img0[a][0], b=img1[b][0], off0=img0[a][1], off1=img1[b][1])
                if (a, b) not in refs:
                    refs[(a, b)] = Ref(pp)
                sl0, sl1 = slice(g["oo0"][p], g["oo0"][p + 1]), slice(g["oo1"][p], g["oo1"][p + 1])
                check_pair(segmean_model, pp, refs[(a, b)], dsub[p], dkey[p], host["matches0"][sl0],
                           host["scores0"][sl0], host["nn1"][sl1], host["counts"][p], thr, mutual, st,
                           f"{what} pair {p} ({a}, {b})")
            runs.append((dsub, dkey, host["matches0"][:-1], host["scores0"][:-1], host["counts"]))
        for r in runs[1:]:
            for x, y in zip(runs[0][:2], r[:2]):
                assert all(np.array_equal(bits(u), bits(v)) for u, v in zip(x, y))
            assert all(np.array_equal(bits(u) if u.dtype == np.float32 else u, bits(v) if v.dtype == np.float32 else v)
                       for u, v in zip(runs[0][2:], r[2:]))
    st.report()


# ------------------------------------------------------------------ batched ltr_merge_sublines with explicit strides
@pytest.mark.gpu
def test_merge_sublines_batched_strides(segmean_model):
    rng = np.random.default_rng(9)
    c = [(counts_random(rng, 9), counts_random(rng, 33)), ([300], [1, 7, 64]), ([1] * 65, [129, 2]),
         (counts_random(rng, 8), counts_random(rng, 257, 1, 2)), ([], [3]), ([2], [])]
    off0 = [_csr(a) for a, _ in c]
    off1 = [_csr(b) for _, b in c]
    S = [(int(o0[-1]), int(o1[-1])) for o0, o1 in zip(off0, off1)]
    K = [(len(o0) - 1, len(o1) - 1) for o0, o1 in zip(off0, off1)]
    ssub = max(s0 * s1 for s0, s1 in S) + 13
    skey = max(k0 * k1 for k0, k1 in K) + 5
    D = np.zeros(len(c) * ssub + 7, np.float32)
    blocks = []
    for p, (s0, s1) in enumerate(S):   # distances of unit descriptors' range, with fp32 low bits in use
        blk = rng.uniform(0.0, 4.0, (s0, s1)).astype(np.float32)
        D[p * ssub:p * ssub + s0 * s1] = blk.reshape(-1)
        blocks.append(blk)
    cuk0, cuk1 = _csr([k for k, _ in K]), _csr([k for _, k in K])
    so0 = _csr(np.concatenate([np.diff(o) for o in off0]))
    so1 = _csr(np.concatenate([np.diff(o) for o in off1]))
    keep = [_t(D), _t(cuk0), _t(cuk1), _t(so0), _t(so1)]
    bk, dk = sentinel(len(c) * skey, 1)
    p_ = lambda t: ctypes.c_void_p(t.data_ptr())   # noqa: E731
    _ops._call("ltr_merge_sublines", DEV, p_(keep[0]), ssub, len(c), p_(keep[1]), p_(keep[2]), p_(keep[3]), p_(keep[4]),
               max(k for k, _ in K), max(k for _, k in K), p_(dk), skey)
    got = check_blocks(bk.cpu().numpy()[1:], K, skey, "merge_sublines")
    for p in range(len(c)):
        assert np.array_equal(bits(got[p]), bits(segmean32(segmean_model, blocks[p], off0[p], off1[p]))), p
    assert np.array_equal(D, keep[0].cpu().numpy())


# ------------------------------------------------------------------ the drop-in sequence and the real pairs
def _dropin(seg32, a_cf, b_cf, A0, A1, thr, st, what, ref_matches=None):
    """get_dist_matrix -> nn_matcher.subline2keyline -> nn_matcher_distmat on channel-first descriptors."""
    a, b = a_cf.T, b_cf.T
    off0, off1 = nnm.adjacency_to_csr(A0), nnm.adjacency_to_csr(A1)
    pp = dict(a=a, b=b, off0=off0, off1=off1)
    ref = Ref(pp)
    ds = get_dist_matrix(a_cf[None], b_cf[None])[0]
    dk = nnm.subline2keyline(ds, A0, A1)[0]
    check_pair(seg32, pp, ref, ds, dk, None, None, None, None, thr, True, st, what)
    for mutual in (True, False):
        mat = nnm.nn_matcher_distmat(dk[None], thr, mutual)
        m0 = np.where(mat[0].any(axis=1), mat[0].argmax(axis=1), -1).astype(np.int32)
        want = decisions(dk, np.float32(thr), mutual)[0]
        assert np.array_equal(m0, want), f"{what} mutual={mutual}"
        ok = decisive(ref.K64, ref.e_K, thr, mutual)
        assert np.array_equal(m0[ok], decisions(ref.K64, thr, mutual)[0][ok]), what
        if mutual:
            st.nondec += int((~ok).sum())
            st.rows += len(ok)
            if ref_matches is not None:
                assert np.array_equal(m0[ok], ref_matches[ok]), f"{what}: decisive rows differ from the reference"
    return ds, dk


@pytest.mark.gpu
def test_dropin_sequence(segmean_model):
    rng = np.random.default_rng(4)
    st = Stats("drop-in")
    for c0, c1 in (([7, 1, 64, 129, 2], counts_random(rng, 60)), (counts_summing(rng, 257), counts_summing(rng, 128)),
                   ([300], counts_random(rng, 31))):
        pp = make_image_pair(rng, c0, c1)
        _dropin(segmean_model, np.ascontiguousarray(pp["a"].T), np.ascontiguousarray(pp["b"].T),
                adjacency(pp["off0"]).astype(np.float32), adjacency(pp["off1"]).astype(np.float32), 0.9, st,
                f"K={len(c0)}x{len(c1)}")
    st.report()


@pytest.mark.gpu
def test_real_pairs(segmean_model):
    """The four bundled pairs: the reference's line descriptors and adjacencies through the drop-in sequence, and as one
    ltr_match batch (channel-first) whose merged distances must carry the same bits."""
    npz, _ = H.plumbing()
    st = Stats("real pairs")
    pairs, want = [], []
    for pair in range(4):
        a_cf, b_cf = npz[f"p{pair}_0_line_desc"][0], npz[f"p{pair}_1_line_desc"][0]
        A0, A1 = npz[f"p{pair}_0_mat_klines2sublines"][0], npz[f"p{pair}_1_mat_klines2sublines"][0]
        ds, dk = _dropin(segmean_model, a_cf, b_cf, A0, A1, 0.8, st, f"pair {pair}", npz[f"p{pair}_matches_l"])
        pairs.append(dict(a=np.ascontiguousarray(a_cf.T), b=np.ascontiguousarray(b_cf.T),
                          off0=nnm.adjacency_to_csr(A0), off1=nnm.adjacency_to_csr(A1)))
        want.append((ds, dk))
    B = Batch(pairs)
    host, ssub, skey = run_batch(B, CF, np.float32(0.8), True)
    dsub = check_blocks(host["dist_sub"], list(zip(B.S0, B.S1)), ssub, "real dist_sub")
    dkey = check_blocks(host["dist_key"], list(zip(B.K0, B.K1)), skey, "real dist_key")
    for p in range(4):
        assert np.array_equal(bits(dsub[p]), bits(want[p][0])), p
        assert np.array_equal(bits(dkey[p]), bits(want[p][1])), p
        m0 = host["matches0"][B.cuk0[p]:B.cuk0[p + 1]]
        assert np.array_equal(m0, decisions(dkey[p], np.float32(0.8), True)[0]), p
    st.report()


# ------------------------------------------------------------------ scale
@pytest.mark.gpu
def test_scale_32_pairs(segmean_model):
    rng = np.random.default_rng(32)
    cnt = lambda: rng.choice([1, 2, 3, 4], size=int(rng.integers(480, 521)), p=[0.35, 0.3, 0.2, 0.15])   # noqa: E731
    B = Batch([make_image_pair(rng, cnt(), cnt()) for _ in range(32)])
    assert 1000 < np.mean(B.S0) < 1200
    host, ssub, skey = run_batch(B, ROWS, np.float32(0.9), True)
    st = Stats("32 pairs x ~500 key lines")
    check_batch(segmean_model, B, host, ssub, skey, np.float32(0.9), True, st, "scale", keep_refs=False)
    st.report()


# ------------------------------------------------------------------ 65535 pairs: the grid limit itself
@pytest.mark.gpu
def test_max_pairs_equals_chunks(segmean_model):
    """Exactly 65535 pairs of images with 1-3 sublines in one ltr_match_indexed call equal the same pairs matched in
    chunks (the same max_n / max_k, so the same strides)."""
    rng = np.random.default_rng(65535)
    img = lambda: counts_summing(rng, int(rng.integers(1, 4)), hi=2)   # noqa: E731
    ims = [make_image_pair(rng, img(), img()) for _ in range(64)]
    pool0 = _pool([(m["a"], m["off0"]) for m in ims], ROWS)
    pool1 = _pool([(m["b"], m["off1"]) for m in ims], ROWS)
    pr = [tuple(x) for x in rng.integers(0, 64, (MAXG, 2))]
    thr = np.float32(0.9)
    whole, g = run_indexed(pool0, pool1, pr, thr, True)
    cuts = [0, 1, 20000, 40000, MAXG]
    for a, b in zip(cuts[:-1], cuts[1:]):
        part, h = run_indexed(pool0, pool1, pr[a:b], thr, True, maxes=g["maxes"])
        r0, r1 = slice(g["oo0"][a], g["oo0"][b]), slice(g["oo1"][a], g["oo1"][b])
        assert np.array_equal(part["matches0"][:-1], whole["matches0"][r0]), (a, b)
        assert np.array_equal(bits(part["scores0"][:-1]), bits(whole["scores0"][r0])), (a, b)
        assert np.array_equal(part["nn1"][:-1], whole["nn1"][r1]), (a, b)
        assert np.array_equal(part["counts"], whole["counts"][a:b]), (a, b)
        for k, sk in (("dist_sub", g["ssub"]), ("dist_key", g["skey"])):
            assert np.array_equal(bits(part[k][:(b - a) * sk]), bits(whole[k][a * sk:b * sk])), (a, b, k)
    # and the whole call against the segmean model and the decisions on a sample of pairs
    for p in rng.integers(0, MAXG, 200):
        i0, i1 = pr[p]
        ds = whole["dist_sub"][p * g["ssub"]:p * g["ssub"] + g["S0"][p] * g["S1"][p]].reshape(g["S0"][p], g["S1"][p])
        dk = whole["dist_key"][p * g["skey"]:p * g["skey"] + g["K0"][p] * g["K1"][p]].reshape(g["K0"][p], g["K1"][p])
        assert np.array_equal(bits(dk), bits(segmean32(segmean_model, ds, ims[i0]["off0"], ims[i1]["off1"]))), p
        assert np.array_equal(whole["matches0"][g["oo0"][p]:g["oo0"][p + 1]], decisions(dk, thr, True)[0]), p


# ------------------------------------------------------------------ host-only checks (no GPU)
def test_segmean_model_equals_exact_rational_evaluation(segmean_model):
    """The C model is the correctly rounded fmaf chain (weights 1 / n correctly rounded), checked against exact
    rationals rounded to float32 once per operation."""
    rng = np.random.default_rng(1)
    off0, off1 = _csr([3, 1, 7]), _csr([5, 2, 1, 3])
    D = (rng.uniform(0, 4, (off0[-1], off1[-1])) * 2.0 ** rng.integers(-8, 3, (off0[-1], off1[-1]))).astype(np.float32)
    got = segmean32(segmean_model, D, off0, off1)
    for a in range(3):
        for b in range(4):
            wa = _round_f32(Fraction(1, int(off0[a + 1] - off0[a])))
            wb = _round_f32(Fraction(1, int(off1[b + 1] - off1[b])))
            acc = Fraction(0)
            for j in range(off1[b], off1[b + 1]):
                t = Fraction(0)
                for i in range(off0[a], off0[a + 1]):
                    t = _round_f32(wa * Fraction(float(D[i, j])) + t)
                acc = _round_f32(t * wb + acc)
            assert got[a, b] == float(acc), (a, b)


def test_sub_bound_holds_for_split_product_and_has_teeth():
    rng = np.random.default_rng(2)
    pp = make_image_pair(rng, np.ones(96, int), np.ones(80, int))
    D64, s = dist64(pp["a"], pp["b"])
    e = sub_bound(pp["a"], pp["b"], s)
    r_ok = float((np.abs(emulate_dist(pp["a"], pp["b"]) - D64) / e).max())
    r_bad = float((np.abs(emulate_dist(pp["a"], pp["b"], drop_lo_hi=True) - D64) / e).max())
    print(f"\n3-term emulation {r_ok:.3f} x e_D, without a_lo b_hi {r_bad:.1f} x e_D")
    assert r_ok <= 1.0
    assert r_bad > 2.0


def _planted(D, off0, off1, kind, csr1_global=None, kb0=0, kb1=0):
    """float64 merges with a planted error: 'drop_last' leaves out the last subline of every key line with more than
    one, 'n_plus_1' weighs 1 / (n + 1), 'csr_offset' reads side 1's CSR at side 0's key-line offset."""
    if kind == "drop_last":
        A0, A1 = adjacency(off0), adjacency(off1)
        for A, off in ((A0, off0), (A1, off1)):
            for k in range(len(off) - 1):
                n = off[k + 1] - off[k]
                if n > 1:
                    A[k, off[k] - off[0]:off[k + 1] - off[0]] = 0
                    A[k, off[k] - off[0]:off[k + 1] - off[0] - 1] = 1.0 / (n - 1)
        return A0 @ D @ A1.T
    if kind == "n_plus_1":
        A0, A1 = adjacency(off0), adjacency(off1)
        n0, n1 = np.diff(off0)[:, None], np.diff(off1)[:, None]
        return (A0 * n0 / (n0 + 1)) @ D @ (A1 * n1 / (n1 + 1)).T
    if kind == "csr_offset":   # the key lines of side 1 whose misread sublines still lie inside the block
        K1 = len(off1) - 1
        o = csr1_global[kb0:kb0 + K1 + 1] - csr1_global[kb0]
        kept = int(np.searchsorted(o, D.shape[1], side="right")) - 1
        return merge64(D[:, :o[kept]], off0, o[:kept + 1]) if kept > 0 else None
    raise KeyError(kind)


@pytest.mark.parametrize("kind", ["drop_last", "n_plus_1", "csr_offset"])
def test_key_bound_has_teeth(kind):
    """Each planted merge error falls outside the dist_key bound on the data the GPU tests use, fed the exact float64
    subline distances (the bound's own input error is then all slack)."""
    B = _case("random_1_4", seed=CASES.index("random_1_4") + 100)
    worst = 0.0
    for p in range(len(B.pairs)):
        ref, pp = B.ref(p), B.pairs[p]
        bad = _planted(ref.D64, pp["off0"], pp["off1"], kind, B.sub_off1, int(B.cuk0[p]), int(B.cuk1[p]))
        if bad is None:
            continue
        k = bad.shape[1]
        worst = max(worst, float((np.abs(bad - ref.K64[:, :k]) / ref.e_K[:, :k]).max()))
    print(f"\nplanted {kind}: {worst:.1f} x the dist_key bound")
    assert worst > 2.0


def test_decisive_rule():
    k64 = np.array([[0.10, 0.10, 0.90], [0.80, 1.20, 1.30], [0.20, 0.60, 0.95], [0.70, 0.30, 0.30 + 1e-7]])
    bnd = np.full_like(k64, 1e-5)
    assert decisive(k64, bnd, 0.8, False).tolist() == [False, False, True, False]
    k64m = k64.copy()
    k64m[0, 0], k64m[3, 0] = 0.5, 0.2 + 1e-6   # row 2's partner column 0 gets a near-tie with row 3
    assert decisive(k64m, bnd, 0.8, True).tolist()[2] is False
    assert decisive(k64m, bnd, 0.8, False).tolist()[2] is True


def _lib():
    return N.load()


def _inp(**kw):
    base = dict(d=256, layout=ROWS, n_pairs=1, n0=1, n1=1)
    base.update(kw)
    return N.LtrMatchInput(**base)


FAKE = 0x1000   # a non-null pointer no refused call may dereference
SEG = dict(cu0=FAKE, cu1=FAKE, sub_off0=FAKE, sub_off1=FAKE, cuk0=FAKE, cuk1=FAKE, max_n0=2, max_n1=2, max_k0=1,
           max_k1=1, total_n0=2, total_n1=2)
IDX = dict(img0=FAKE, img1=FAKE, tiles0=FAKE, tiles1=FAKE, tile_off0=FAKE, tile_off1=FAKE, n_tiles0=1, n_tiles1=1,
           out_off0=FAKE, out_off1=FAKE, total_out0=1, total_out1=1)
UNS, INV = "unsupported", "invalid"
# (entry, LtrMatchInput fields, expected): the limits refuse with LTR_E_UNSUPPORTED; one below them the call goes on
# (workspace sizes) or stops at the next check with LTR_E_INVALID (null outputs) - in no case with a CUDA call
MATCH_TABLE = [
    ("ltr_match_workspace_bytes", dict(n_pairs=MAXG + 1), UNS),
    ("ltr_match_workspace_bytes", dict(n_pairs=MAXG), "ok"),
    ("ltr_match_workspace_bytes", dict(n_pairs=2 ** 31 - 1), UNS),
    ("ltr_match_workspace_bytes", dict(SEG, max_k0=8 * MAXG + 1), UNS),
    ("ltr_match_workspace_bytes", dict(SEG, max_k0=8 * MAXG), "ok"),
    ("ltr_match_workspace_bytes", dict(SEG, n_pairs=MAXG + 1), UNS),
    ("ltr_match", dict(n_pairs=MAXG + 1), UNS),
    ("ltr_match", dict(n_pairs=MAXG), INV),
    ("ltr_match", dict(n_pairs=MAXG + 1, d=16), UNS),
    ("ltr_match", dict(SEG, max_k0=8 * MAXG + 1), UNS),
    ("ltr_match", dict(SEG, max_k0=8 * MAXG), INV),
    ("ltr_match_indexed_workspace_bytes", dict(SEG, n_pairs=MAXG + 1), UNS),
    ("ltr_match_indexed_workspace_bytes", dict(SEG, n_pairs=MAXG), "ok"),
    ("ltr_match_indexed_workspace_bytes", dict(SEG, max_k0=8 * MAXG + 1), UNS),
    ("ltr_match_indexed", dict(SEG, n_pairs=MAXG + 1), UNS),
    ("ltr_match_indexed", dict(SEG, n_pairs=MAXG), INV),
    ("ltr_match_indexed", dict(SEG, max_k0=8 * MAXG + 1), UNS),
    ("ltr_match_indexed", dict(SEG, max_k0=8 * MAXG), INV),
]


@pytest.mark.parametrize("entry,fields,want", MATCH_TABLE)
def test_match_grid_limits_refused_on_host(entry, fields, want):
    lib = _lib()
    inp = _inp(**fields)
    args = [ctypes.byref(inp)]
    if "indexed" in entry:
        args.append(ctypes.byref(N.LtrPairIndex(**IDX)))
    if not entry.endswith("_workspace_bytes"):
        args += [ctypes.byref(N.LtrMatchOutput()), 0, None]   # no outputs: an accepted input stops at LTR_E_INVALID
    rc = int(getattr(lib, entry)(*args))
    if want == "ok":
        assert rc >= 0, (rc, lib.ltr_last_error())
    else:
        assert rc == _code("LTR_E_UNSUPPORTED" if want == UNS else "LTR_E_INVALID"), (rc, lib.ltr_last_error())
        if want == UNS:
            assert b"65535" in lib.ltr_last_error()


# (n_pairs, max_k0, expected) of ltr_merge_sublines and ltr_match_distmat, null buffers
OTHER_TABLE = [
    ("ltr_merge_sublines", MAXG + 1, 1, UNS),
    ("ltr_merge_sublines", MAXG, 1, INV),
    ("ltr_merge_sublines", 1, 8 * MAXG + 1, UNS),
    ("ltr_merge_sublines", 1, 8 * MAXG, INV),
    ("ltr_match_distmat", MAXG + 1, 1, UNS),
    ("ltr_match_distmat", MAXG, 1, INV),
]


@pytest.mark.parametrize("entry,n_pairs,max_k0,want", OTHER_TABLE)
def test_other_grid_limits_refused_on_host(entry, n_pairs, max_k0, want):
    lib = _lib()
    if entry == "ltr_merge_sublines":
        rc = lib.ltr_merge_sublines(None, 0, n_pairs, None, None, None, None, max_k0, 1, None, 0, 0, None)
    else:
        rc = lib.ltr_match_distmat(None, n_pairs, max_k0, 1, 0, 0.5, 1, None, None, None, None, 0, None)
    assert rc == _code("LTR_E_UNSUPPORTED" if want == UNS else "LTR_E_INVALID"), (rc, lib.ltr_last_error())
