"""The k-block timeline gemm_chain_kernel's CTA 0 leaves in the debug trace (tools/gemm_chain_trace.py reads it):
one signature layer at 128 m-tiles, so CTA 0 walks one m-tile through mlp1 (2 tiles x 8 k-blocks), mlp2 (1 x 8) and
qkv (3 x 4).  Every stamp the tool reads must be written, and in causal order."""
import ctypes as C

import pytest

from linetr_b200 import _native as N

TRACE_KB, EPI = 36, 108          # CHAIN_TRACE_KB, CHAIN_TRACE_EPI (csrc/gemm_img.cuh)
T0 = EPI + 16                    # CHAIN_TRACE_T0
TILES = [(0, 2, 8), (1, 1, 8), (2, 3, 4)]   # (op, n-blocks, k-blocks per tile)


@pytest.mark.gpu
def test_chain_trace_timeline_is_complete_and_ordered():
    lib = N.load()
    lib.ltr_debug_trace_arm(1)
    try:
        ms = lib.ltr_gemm_chain_bench(128 * 128, 1, 1, 0)
        buf = (C.c_uint64 * 128)()
        rc = lib.ltr_debug_trace_read(buf)
    finally:
        lib.ltr_debug_trace_arm(0)
    assert ms > 0 and rc == 0
    t = [int(v) for v in buf]
    used = set(range(3 * TRACE_KB)) | {T0, T0 + 1}
    prev_done, it = t[T0 + 1], 0
    for o, nbl, nk in TILES:
        for nb in range(nbl):
            for _ in range(nk):
                issue, land, done = t[3 * it: 3 * it + 3]
                assert t[T0] <= issue < land <= done, it     # producer past pdl_wait, then issued, landed, MMAs done
                assert prev_done <= land, it                  # one consumer thread's stamps follow each other
                prev_done, it = done, it + 1
            epi = t[EPI + o * 4 + nb]
            used.add(EPI + o * 4 + nb)
            assert prev_done <= epi, (o, nb)
            prev_done = epi
    assert all(t[i] for i in used)
    assert not any(t[i] for i in range(128) if i not in used)   # no stray slots (ops 3.., n-blocks past the layer)
