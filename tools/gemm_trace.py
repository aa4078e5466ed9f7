"""Per-tile clock64 stamps of gemm_img_kernel CTA 0 on the signature-layer shapes (image output), from the debug
trace (slot layout under ltr_debug_trace_arm in include/linetr_b200_debug.h).  The launch time comes from a separate
unarmed call, so the timed loop carries no stamps."""
import ctypes as C
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from linetr_b200 import _native as N
lib = N.load()
names = {0: "mma:start", 2: "mma:done", 5: "epi:done", 6: "tma:slot_free"}
for name, m, n, k, bn, om in (("qkv", 16384, 768, 256, 256, 1), ("mlp1", 16384, 512, 512, 256, 1), ("mlp2", 16384, 256, 512, 128, 1),
                              ("mlp2", 16384, 256, 512, 256, 1), ("ffn_w1", 16384, 1024, 256, 256, 1)):
    ms = lib.ltr_gemm_bench(m, n, k, bn, om, 20, 0)
    lib.ltr_debug_trace_arm(1)
    traced = lib.ltr_gemm_bench(m, n, k, bn, om, 1, 0)
    buf = (C.c_uint64 * 128)()
    rc = lib.ltr_debug_trace_read(buf)
    lib.ltr_debug_trace_arm(0)
    if ms < 0 or traced < 0 or rc != 0:
        raise N.LtrError(f"{name}: gemm trace failed")
    vals = [int(v) for v in buf]
    base = min(v for v in vals if v)
    print(f"{name} M={m} N={n} K={k} BN={bn} out={om}: {ms*1e3:.1f} us/launch")
    for tl in range(3):
        print(f"  tile {tl}: " + "  ".join(f"{nm}={vals[tl*16+j]-base if vals[tl*16+j] else -1:7d}" for j, nm in names.items()))
