"""Host-side behaviour of the two matcher entry points, `ltr_match` and `ltr_match_indexed`, without a GPU: the return
code and error message of every malformed call that is refused before any CUDA call, and the scratch size
`ltr_match_workspace_bytes` / `ltr_match_indexed_workspace_bytes` report for valid inputs.  None of these calls
touches device memory, so the pointers are placeholders."""
import ctypes as C

import pytest

from linetr_b200 import _native as N

OK, INVALID, UNSUPPORTED = 0, -1, -4
PTR = 0x10000   # a non-null placeholder: these calls return before dereferencing anything


def _input(**kw):
    base = dict(desc0=PTR, desc1=PTR, layout=N.LAYOUT_ROWS, d=256, n_pairs=2, n0=128, n1=128, nn_thresh=0.8, mutual=1)
    base.update(kw)
    return N.LtrMatchInput(**base)


def _split(**kw):   # key-line merging over ragged pairs
    base = dict(cu0=PTR, cu1=PTR, sub_off0=PTR, sub_off1=PTR, cuk0=PTR, cuk1=PTR, max_n0=50, max_n1=40, max_k0=30,
                max_k1=20, total_n0=90, total_n1=70)
    base.update(kw)
    return base


def _index(**kw):
    base = dict(img0=PTR, img1=PTR, tiles0=PTR, tiles1=PTR, tile_off0=PTR, tile_off1=PTR, n_tiles0=4, n_tiles1=3,
                out_off0=PTR, out_off1=PTR, total_out0=300, total_out1=200)
    base.update(kw)
    return N.LtrPairIndex(**base)


def _pools(**kw):   # LtrMatchInput of a pair list over two image pools
    base = dict(cu0=PTR, cu1=PTR, max_n0=100, max_n1=90, total_n0=400, total_n1=300, n0=0, n1=0)
    base.update(kw)
    return _input(**base)


def _output(**kw):
    base = dict(matches0=PTR, scores0=PTR, nn1=PTR, counts=PTR, workspace=PTR, workspace_bytes=1 << 30)
    base.update(kw)
    return N.LtrMatchOutput(**base)


def _gather(**kw):
    base = dict(mc_base=PTR, peer_bases=None, rank=0, world=2, slot=0, epoch=1)
    base.update(kw)
    return C.pointer(N.LtrPeerGather(**base))


MERGE_OUT = dict(dist_key=PTR, dist_sub=PTR)

MATCH_CASES = {
    "dim_100": (_input(d=100), _output(), UNSUPPORTED),
    "dim_0": (_input(d=0), _output(), INVALID),
    "dim_negative": (_input(d=-16), _output(), INVALID),
    "dist_mode_2": (_input(dist_mode=2), _output(), INVALID),
    "dist_mode_1_dim_128": (_input(dist_mode=1, d=128), _output(dist_key=PTR), INVALID),
    "dist_mode_1_merging": (_input(dist_mode=1, **_split()), _output(**MERGE_OUT), INVALID),
    "merging_without_sub_off1": (_input(**_split(sub_off1=None)), _output(**MERGE_OUT), INVALID),
    "merging_without_sub_off0": (_input(**_split(sub_off0=None)), _output(**MERGE_OUT), INVALID),
    "merging_without_cuk1": (_input(**_split(cuk1=None)), _output(**MERGE_OUT), INVALID),
    "merging_without_cu": (_input(**_split(cu0=None, cu1=None)), _output(**MERGE_OUT), INVALID),
    "cu0_without_cu1": (_input(cu0=PTR, max_n0=10, max_n1=10), _output(), INVALID),
    "cu1_without_cu0": (_input(cu1=PTR, max_n0=10, max_n1=10), _output(), INVALID),
    "cu_without_total_n0": (_input(cu0=PTR, cu1=PTR, max_n0=10, max_n1=10, total_n0=-1, total_n1=5), _output(), INVALID),
    "cu_without_total_n1": (_input(cu0=PTR, cu1=PTR, max_n0=10, max_n1=10, total_n0=5, total_n1=-1), _output(), INVALID),
    "matches0_without_scores0": (_input(), _output(scores0=None), INVALID),
    "matches0_without_nn1": (_input(), _output(nn1=None), INVALID),
    "matches0_without_counts": (_input(), _output(counts=None), INVALID),
    "nothing_to_compute": (_input(), _output(matches0=None), INVALID),
    "merging_without_dist_sub": (_input(**_split()), _output(dist_key=PTR), INVALID),
    "merging_without_dist_key": (_input(**_split()), _output(dist_sub=PTR), INVALID),
    "dim_128_without_dist_key": (_input(d=128), _output(), INVALID),
    "gather_bad_rank": (_input(), _output(gather=_gather(rank=2)), INVALID),
    "gather_negative_rank": (_input(), _output(gather=_gather(rank=-1)), INVALID),
    "gather_bad_slot": (_input(), _output(gather=_gather(slot=N.GATHER_SLOTS)), INVALID),
    "gather_bad_epoch": (_input(), _output(gather=_gather(epoch=0)), INVALID),
    "gather_without_buffers": (_input(), _output(gather=_gather(mc_base=None)), INVALID),
    "gather_with_merging": (_input(**_split()), _output(gather=_gather(), **MERGE_OUT), UNSUPPORTED),
    "gather_dim_128": (_input(d=128), _output(gather=_gather(), dist_key=PTR), UNSUPPORTED),
    "gather_without_matches": (_input(), _output(gather=_gather(), matches0=None, dist_key=PTR), UNSUPPORTED),
    "gather_empty_side0": (_input(n0=0), _output(gather=_gather()), UNSUPPORTED),
    "gather_empty_side0_ragged": (_input(cu0=PTR, cu1=PTR, max_n0=0, max_n1=10), _output(gather=_gather()),
                                  UNSUPPORTED),
    # output checks come before the gather checks
    "gather_without_scores0": (_input(), _output(gather=_gather(rank=5), scores0=None), INVALID),
    "gather_with_merging_without_dist_sub": (_input(**_split()), _output(gather=_gather(), dist_key=PTR), INVALID),
    # no pairs: nothing is validated
    "no_pairs": (_input(n_pairs=0, d=100), _output(matches0=None), OK),
}

INDEXED_CASES = {
    "dim_128": (_pools(d=128), _index(), _output(), UNSUPPORTED),
    "dim_100": (_pools(d=100), _index(), _output(), UNSUPPORTED),
    "dist_mode_1": (_pools(dist_mode=1), _index(), _output(), UNSUPPORTED),
    "gather": (_pools(), _index(), _output(gather=_gather()), UNSUPPORTED),
    "gather_bad": (_pools(), _index(), _output(gather=_gather(rank=7, epoch=0)), UNSUPPORTED),
    "no_pairs_dim_100": (_pools(n_pairs=0, d=100), _index(), _output(), UNSUPPORTED),
    "no_pairs": (_pools(n_pairs=0, cu0=None), _index(img0=None), _output(matches0=None), OK),
    "without_cu0": (_pools(cu0=None), _index(), _output(), INVALID),
    "without_cu1": (_pools(cu1=None), _index(), _output(), INVALID),
    "merging_without_sub_off1": (_pools(sub_off0=PTR, cuk0=PTR, cuk1=PTR), _index(), _output(**MERGE_OUT), INVALID),
    "merging_without_sub_off0": (_pools(sub_off1=PTR, cuk0=PTR, cuk1=PTR), _index(), _output(**MERGE_OUT), INVALID),
    "merging_without_cuk0": (_pools(sub_off0=PTR, sub_off1=PTR, cuk1=PTR), _index(), _output(**MERGE_OUT), INVALID),
    "without_img0": (_pools(), _index(img0=None), _output(), INVALID),
    "without_img1": (_pools(), _index(img1=None), _output(), INVALID),
    "without_out_off0": (_pools(), _index(out_off0=None), _output(), INVALID),
    "without_out_off1": (_pools(), _index(out_off1=None), _output(), INVALID),
    "negative_max_n0": (_pools(max_n0=-1), _index(), _output(), INVALID),
    "negative_max_n1": (_pools(max_n1=-1), _index(), _output(), INVALID),
    "negative_n_tiles": (_pools(), _index(n_tiles1=-1), _output(), INVALID),
    "negative_total_out": (_pools(), _index(total_out0=-1), _output(), INVALID),
    "without_tiles0": (_pools(), _index(tiles0=None), _output(), INVALID),
    "without_tiles1": (_pools(), _index(tiles1=None), _output(), INVALID),
    "without_tile_off0": (_pools(), _index(tile_off0=None), _output(), INVALID),
    "without_tile_off1": (_pools(), _index(tile_off1=None), _output(), INVALID),
    "matches0_without_scores0": (_pools(), _index(), _output(scores0=None), INVALID),
    "matches0_without_nn1": (_pools(), _index(), _output(nn1=None), INVALID),
    "matches0_without_counts": (_pools(), _index(), _output(counts=None), INVALID),
    "nothing_to_compute": (_pools(), _index(), _output(matches0=None), INVALID),
    "merging_without_dist_sub": (_pools(sub_off0=PTR, sub_off1=PTR, cuk0=PTR, cuk1=PTR, max_k0=10, max_k1=10), _index(),
                                 _output(dist_key=PTR), INVALID),
    "without_desc0": (_pools(desc0=None), _index(), _output(), INVALID),
    "without_desc1": (_pools(desc1=None), _index(), _output(), INVALID),
    # the pool checks come before the output checks, the output checks before the descriptor check
    "without_img0_nothing_to_compute": (_pools(), _index(img0=None), _output(matches0=None), INVALID),
    "without_desc0_nothing_to_compute": (_pools(desc0=None), _index(), _output(matches0=None), INVALID),
}


def _error(lib) -> str:
    return lib.ltr_last_error().decode()


@pytest.mark.parametrize("case", sorted(MATCH_CASES))
def test_match_refuses_before_any_cuda_call(case):
    inp, out, want = MATCH_CASES[case]
    lib = N.load()
    rc = lib.ltr_match(C.byref(inp), C.byref(out), 0, None)
    assert rc == want, _error(lib)
    if want != OK:
        assert _error(lib).startswith("ltr_match: "), _error(lib)


@pytest.mark.parametrize("case", sorted(INDEXED_CASES))
def test_match_indexed_refuses_before_any_cuda_call(case):
    inp, idx, out, want = INDEXED_CASES[case]
    lib = N.load()
    rc = lib.ltr_match_indexed(C.byref(inp), C.byref(idx), C.byref(out), 0, None)
    assert rc == want, _error(lib)
    if want != OK:
        assert _error(lib).startswith("ltr_match_indexed: "), _error(lib)


def test_order_of_checks_pinned_by_messages():
    """Where one malformed call breaks two rules, the message says which check ran first."""
    lib = N.load()
    inp, out, _ = MATCH_CASES["gather_without_scores0"]
    lib.ltr_match(C.byref(inp), C.byref(out), 0, None)
    assert "matches0 needs scores0" in _error(lib)
    inp, idx, out, _ = INDEXED_CASES["without_img0_nothing_to_compute"]
    lib.ltr_match_indexed(C.byref(inp), C.byref(idx), C.byref(out), 0, None)
    assert "img0/1 and out_off0/1 are required" in _error(lib)
    inp, idx, out, _ = INDEXED_CASES["without_desc0_nothing_to_compute"]
    lib.ltr_match_indexed(C.byref(inp), C.byref(idx), C.byref(out), 0, None)
    assert "nothing to compute" in _error(lib)


def test_null_arguments():
    lib = N.load()
    inp, idx, out = _input(), _index(), _output()
    assert lib.ltr_match(None, C.byref(out), 0, None) == INVALID
    assert lib.ltr_match(C.byref(inp), None, 0, None) == INVALID
    assert _error(lib).startswith("ltr_match: ")
    assert lib.ltr_match_indexed(C.byref(inp), None, C.byref(out), 0, None) == INVALID
    assert _error(lib).startswith("ltr_match_indexed: ")
    assert lib.ltr_match_workspace_bytes(None) == INVALID
    assert lib.ltr_match_indexed_workspace_bytes(C.byref(inp), None) == INVALID


# Scratch sizes at the commit that folded the two entries' host code into one path; they must not move.
WORKSPACE_CASES = {
    "uniform": (_input(n_pairs=4, n0=128, n1=200), 1586176),
    "uniform_tiles_both": (_input(n_pairs=4, n0=128, n1=256, tiles0=PTR, tiles1=PTR, tiles_lines0=512,
                                  tiles_lines1=1024), 14336),
    "uniform_tiles_one_side": (_input(n_pairs=4, n0=128, n1=128, tiles0=PTR, tiles1=PTR, tiles_lines0=1024,
                                      tiles_lines1=1024, tiles_row0_0=512, tiles_row0_1=64), 534528),
    "uniform_tiles_past_the_end": (_input(n_pairs=4, n0=128, n1=128, tiles0=PTR, tiles1=PTR, tiles_lines0=384,
                                          tiles_lines1=512), 534528),
    "ragged": (_input(n_pairs=3, cu0=PTR, cu1=PTR, max_n0=300, max_n1=77, total_n0=500, total_n1=150), 1581056),
    "merging": (_input(n_pairs=3, **_split()), 790528),
    "dist_mode_1": (_input(n_pairs=2, n0=200, n1=100, dist_mode=1), 797696),
    "dist_mode_1_ragged": (_input(n_pairs=5, cu0=PTR, cu1=PTR, max_n0=129, max_n1=1, total_n0=300, total_n1=5,
                                  dist_mode=1), 1975296),
    "dim_128": (_input(d=128), 0),
    "no_pairs": (_input(n_pairs=0), 0),
}

INDEXED_WORKSPACE_CASES = {
    "plain": (_pools(n_pairs=33), _index(total_out0=1000, total_out1=700), 16384),
    "plain_empty_outputs": (_pools(n_pairs=2), _index(total_out0=0, total_out1=0), 4096),
    "merging": (_pools(n_pairs=33, sub_off0=PTR, sub_off1=PTR, cuk0=PTR, cuk1=PTR, max_k0=60, max_k1=50),
                _index(total_out0=1000, total_out1=700), 2048),
    "no_pairs": (_pools(n_pairs=0), _index(), 0),
}


@pytest.mark.parametrize("case", sorted(WORKSPACE_CASES))
def test_match_workspace_bytes(case):
    inp, want = WORKSPACE_CASES[case]
    assert N.load().ltr_match_workspace_bytes(C.byref(inp)) == want


@pytest.mark.parametrize("case", sorted(INDEXED_WORKSPACE_CASES))
def test_match_indexed_workspace_bytes(case):
    inp, idx, want = INDEXED_WORKSPACE_CASES[case]
    assert N.load().ltr_match_indexed_workspace_bytes(C.byref(inp), C.byref(idx)) == want
