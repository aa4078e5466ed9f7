"""Chained row-local GEMMs (`gemm_chain_kernel`): an encode whose batch has at least LTR_CHAIN_MIN_TILES 128-row
tiles runs fc -> w_1 -> w_2 -> qkv and every signature layer's mlp1 -> mlp2 -> qkv / final_proj as one launch each.
The chain performs the same per-tile arithmetic as one launch per layer, so both paths must agree bit for bit."""
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from linetr_b200 import _native as N, engine, synthetic as syn
from tests.test_image_pairs import _model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda", 0)


# ------------------------------------------------------------------ CPU: the chain's argument validation
_CHECK_SRC = r"""
#include <cstdio>
#include "gemm_img.cuh"
namespace ltr {   // the library state ltr_api.cu defines, which the headers' launch helpers refer to
thread_local std::string g_last_error;
std::atomic<int64_t> g_launches{0};
Profiler g_prof;
std::mutex g_state_mutex;
std::vector<std::pair<const void*, int>> g_smem_configured;
int set_error(int code, const std::string&) { return code; }
const char* kernel_class_name(int) { return ""; }
cudaEvent_t Profiler::get() { return nullptr; }
}
using namespace ltr;

static __nv_bfloat16 buf[8][2];   // stand-in image planes (the check compares pointers only)
static ActImg img(int i, int K) { return ActImg{&buf[i][0], &buf[i][1], K / 64}; }
static GemmImgArgs op(ActImg A, int N, int K, ActImg O) {
  GemmImgArgs a{};
  a.A = A; a.O = O; a.M = 1000; a.W.N = N; a.W.K = K;
  return a;
}
static void report(const char* name, const GemmImgArgs* ops, int n) {
  const char* why = gemm_chain_check(ops, n);
  std::printf("%s|%s\n", name, why ? why : "ok");
}

int main() {
  const ActImg xm = img(0, 512), hm = img(1, 512), qkv = img(2, 768), ctx = img(3, 256), y1 = img(4, 256),
               g = img(5, 1024), lpos = img(6, 256), big = img(7, 2048);
  {   // a signature layer: mlp1 -> mlp2 (+x in place) -> qkv of the next layer
    GemmImgArgs o[3] = {op(xm, 512, 512, hm), op(hm, 256, 512, xm), op(xm, 768, 256, qkv)};
    o[1].Rimg = xm;
    report("layer", o, 3);
    GemmImgArgs w = o[2]; w.A = hm; GemmImgArgs o2[3] = {o[0], o[1], w};
    report("other_image", o2, 3);                 // qkv would read an image mlp2 does not write
    w = o[2]; w.a_kb0 = 4; GemmImgArgs o3[3] = {o[0], o[1], w};
    report("shifted_kblocks", o3, 3);             // reads xm[:, 256:512], written by the previous launch
    w = o[1]; w.W.K = 256; GemmImgArgs o4[3] = {o[0], w, o[2]};
    report("partial_kblocks", o4, 3);             // mlp2 would read half of what mlp1 writes
    w = o[1]; w.M = 999; GemmImgArgs o5[3] = {o[0], w, o[2]};
    report("rows_differ", o5, 3);
    w = o[0]; w.a_kb_nb = 4; GemmImgArgs o6[3] = {w, o[1], o[2]};
    report("block_diagonal", o6, 3);
    w = o[0]; w.W.N = 448; GemmImgArgs o7[1] = {w};
    report("n_not_256", o7, 1);
    w = o[2]; w.a_kb0 = 8; GemmImgArgs o8[1] = {w};
    report("a_outside", o8, 1);
    GemmImgArgs o9[5] = {o[0], o[1], o[2], o[0], o[1]};
    report("too_many", o9, 5);
  }
  {   // the line stage: fc + LN -> w_1 GELU -> w_2 + LN + pos -> qkv of layer 0
    GemmImgArgs fc = op(ctx, 256, 256, y1), w1 = op(y1, 1024, 256, g), w2 = op(g, 256, 1024, xm), q = op(xm, 768, 256, qkv);
    static float par[256];
    fc.norm = NORM_LAYER; fc.ng = par; fc.nbeta = par;
    w1.act = ACT_GELU;
    w2.norm = NORM_LAYER; w2.ng = par; w2.nbeta = par; w2.Rimg = y1; w2.NaddImg = lpos;
    GemmImgArgs o[4] = {fc, w1, w2, q};
    report("line", o, 4);
    GemmImgArgs wide = op(y1, 2048, 256, big), w2w = op(big, 256, 2048, xm);
    GemmImgArgs o2[3] = {fc, wide, w2w};
    report("too_wide", o2, 3);                    // w_1 would hand 32 k-blocks to w_2
    GemmImgArgs bad = w2; bad.act = ACT_RELU; GemmImgArgs o3[3] = {fc, w1, bad};
    report("norm_with_act", o3, 3);
  }
  return 0;
}
"""

_EXPECT = {
    "layer": "ok", "line": "ok",
    "other_image": "row-local", "shifted_kblocks": "exactly the k-blocks", "partial_kblocks": "exactly the k-blocks",
    "rows_differ": "equal M", "block_diagonal": "plain A", "n_not_256": "N % 256", "a_outside": "exceeds",
    "too_many": "1..4 ops", "too_wide": "16 k-blocks", "norm_with_act": "row-norm",
}


def test_chain_check_rejects_non_chaining_ops():
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc) and shutil.which(nvcc) is None:
        pytest.skip("no nvcc for the host-side check")
    with tempfile.TemporaryDirectory() as td:
        src, exe = os.path.join(td, "chain_check.cu"), os.path.join(td, "chain_check")
        with open(src, "w") as f:
            f.write(_CHECK_SRC)
        subprocess.check_call([nvcc, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
                               "-I", os.path.join(ROOT, "linetr_b200", "csrc"), "-o", exe, src])
        out = subprocess.check_output([exe], text=True)
    got = dict(line.split("|", 1) for line in out.strip().splitlines())
    assert set(got) == set(_EXPECT)
    for name, want in _EXPECT.items():
        assert want in got[name], (name, got[name])


# ------------------------------------------------------------------ GPU: chained == one launch per layer, bit for bit
def _batch(sizes, seed, tokens):
    """Images [0, P) are side 0 of P pairs, [P, 2P) side 1; sizes = lines of each pair's two images."""
    pairs = [syn.make_pair_inputs(seed + i, n, tokens, n_real_tokens=(3, tokens))[:2] for i, n in enumerate(sizes)]
    return engine.LineBatch.from_images([a for a, _ in pairs] + [b for _, b in pairs]).to(DEV), len(pairs)


def _run(eng, batch, P, min_tiles):
    os.environ["LTR_CHAIN_MIN_TILES"] = str(min_tiles)
    try:
        N.reset_launch_count()
        if batch.uniform_lines is not None and batch.uniform_lines % 128 == 0:
            rows, tiles = eng.encode(batch, want_tiles=True)
        else:
            rows, tiles = eng.encode(batch), None
        torch.cuda.synchronize()
        launches = N.launch_count()
        res = eng.match_packed(batch, P, 0.8)
        torch.cuda.synchronize()
    finally:
        del os.environ["LTR_CHAIN_MIN_TILES"]
    return rows, tiles, res, launches


def _assert_equal_paths(batch, P, chain_tiles, expect_chain=True):
    model, _ = _model()
    eng = engine.PairEngine(model, DEV)
    rc, tc, mc, lc = _run(eng, batch, P, chain_tiles)
    rp, tp, mp, lp = _run(eng, batch, P, 0)
    saved = 3 + 2 * 7   # line stage fc, w_1, w_2, qkv -> 1 launch; per signature layer mlp1, mlp2, qkv -> 1
    assert lp - lc == (saved if expect_chain else 0), (lc, lp)
    assert torch.equal(rc, rp)
    if tc is not None:
        assert torch.equal(tc, tp)
    assert torch.equal(mc.matches0, mp.matches0)
    assert torch.equal(mc.scores0, mp.scores0)
    assert torch.equal(mc.counts, mp.counts)


@pytest.mark.gpu
def test_chain_equals_per_layer_cfg1_batch():
    """64 pairs x 128 lines x 21 tokens (128 m-tiles): the default threshold chains it."""
    batch, P = _batch([128] * 64, 100, 21)
    model, _ = _model()
    eng = engine.PairEngine(model, DEV)
    os.environ.pop("LTR_CHAIN_MIN_TILES", None)
    N.reset_launch_count()
    eng.encode(batch, want_tiles=True)
    torch.cuda.synchronize()
    assert N.launch_count() == 20
    _assert_equal_paths(batch, P, 1)


@pytest.mark.gpu
def test_chain_equals_per_layer_ragged_batch():
    """cfg3-like ragged sizes: the row count is not a multiple of 128, so the last m-tile is partial."""
    rng = np.random.Generator(np.random.PCG64(5))
    sizes = [int(x) for x in rng.integers(32, 513, size=12)]
    batch, P = _batch(sizes, 200, 64)
    assert batch.n_lines % 128 != 0 and batch.uniform_lines is None
    _assert_equal_paths(batch, P, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("pairs, chained", [(19, False), (20, True)])
def test_chain_threshold(pairs, chained):
    """LTR_CHAIN_MIN_TILES = 40: 2 x 19 x 128 lines are 38 tiles (one launch per layer), 2 x 20 x 128 are 40 (chained)."""
    batch, P = _batch([128] * pairs, 300, 21)
    _assert_equal_paths(batch, P, 40, expect_chain=chained)
