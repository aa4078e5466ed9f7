"""Launch accounting: `ltr_launch_count` and the per-class profile (`ltr_profile_*`) count every kernel launch the library
issues exactly once, debug hooks included.  Each entry's count is its launch structure (include/linetr_b200.h), and over
a whole call the count, the profile's launches and the library kernels CUPTI records (torch.profiler) are equal."""
import re

import numpy as np
import pytest
import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile

from linetr_b200 import _native as N, _ops, bundle as BA, engine, geometry as G, retrieval as RT, synthetic as syn
from linetr_b200 import tracks as TR, triangulation as T
from linetr_b200.global_poses import global_poses

DEV = torch.device("cuda", 0)
LIBRARY_KERNEL = re.compile(r"(void )?(ltr::|debug_)")   # the library's kernels by the names CUPTI gives them


def _profiled(fn):
    """fn run once in a torch.profiler profile of its own with the library's profile armed.  -> ([(entry, inputs,
    launch count) of every `_ops.call_struct` call], {class: launches}, launch count, library kernels CUPTI recorded)."""
    calls = []
    call_struct = _ops.call_struct

    def counted(entry, inputs, outputs, *args, **kw):
        n0 = N.launch_count()
        out = call_struct(entry, inputs, outputs, *args, **kw)
        calls.append((entry, inputs, N.launch_count() - n0))
        return out

    torch.cuda.synchronize()
    _ops.call_struct = counted
    try:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            N.reset_launch_count()
            N.profile_begin()
            fn()
            classes = {k: n for k, (_, n) in N.profile_end().items()}   # synchronises
            launches = N.launch_count()
    finally:
        _ops.call_struct = call_struct
    kernels = sum(e.device_type == DeviceType.CUDA and LIBRARY_KERNEL.match(e.name) is not None for e in prof.events())
    return calls, classes, launches, kernels


def _accounted(fn, attempts=3):
    """Checks that the launch count of one run of fn equals the library kernels CUPTI recorded and the profile's
    launches summed over classes.  A profile session in which CUPTI delivered no kernel record at all is a profiler
    failure, not a count, and is run again.  -> (calls, classes) of `_profiled`."""
    for _ in range(attempts):
        calls, classes, launches, kernels = _profiled(fn)
        if kernels > 0:
            break
    assert launches > 0
    assert launches == kernels == sum(classes.values()), (launches, kernels, classes)
    return calls, classes


def _counts(calls, entry, select=lambda inputs: True):
    return [n for e, inputs, n in calls if e == entry and select(inputs)]


@pytest.mark.gpu
@pytest.mark.parametrize("iters", [0, 3])
def test_bundle_adjust_counts_four_launches_and_five_per_iteration(iters):
    from tests.test_bundle import _gpu_case, scene
    d, pairs, R, t = scene(11, V=10, n_pts=80, n_lines=16)
    trk = _gpu_case(d, pairs, R, t)
    calls, classes = _accounted(lambda: BA.bundle_adjust(d["keypoints"], d["klines"], d["K"], R, t, trk, max_iters=iters))
    assert _counts(calls, "ltr_bundle_adjust") == [4 + 5 * iters]
    assert classes == {"bundle": 4 + 5 * iters}


@pytest.mark.gpu
def test_global_poses_counts_two_launches_and_the_support_with_pairs():
    from tests.test_global_poses import ring, truth
    Rt, tt, _ = truth(40, 6)
    p = ring(6, 2)
    rp = syn.make_relative_poses(Rt, tt, p, noise_deg=0.5, seed=1)
    dp = {k: torch.as_tensor(v).to(DEV) for k, v in rp.items() if k != "outlier"}
    calls, _ = _accounted(lambda: global_poses(np.zeros((0, 2), np.int64), {k: v[:0] for k, v in dp.items()}, 1))
    assert _counts(calls, "ltr_global_poses") == [2]
    calls, _ = _accounted(lambda: global_poses(p, dp, 6))
    assert _counts(calls, "ltr_global_poses") == [3]


def _descriptor_set(seed):
    rng = np.random.default_rng(seed)
    rows = rng.standard_normal((300, 256))
    rows = (rows / np.linalg.norm(rows, axis=1, keepdims=True)).astype(np.float32)
    return RT.descriptor_set([rows[:150], rows[150:]], [rows[:10], rows[10:]], DEV)


@pytest.mark.gpu
def test_kmeans_update_counts_one_launch_with_init_rows_else_two():
    s = _descriptor_set(7)
    calls, _ = _accounted(lambda: RT.train_vocabulary(s, 6, 5, iters=1, seed=11))
    assert _counts(calls, "ltr_kmeans_update", lambda i: i["init_rows"] is not None) == [1, 1]
    assert _counts(calls, "ltr_kmeans_update", lambda i: i["init_rows"] is None) == [2, 2]


@pytest.mark.gpu
def test_vlad_and_retrieve_count_three_and_two_launches():
    s = _descriptor_set(8)
    voc = RT.train_vocabulary(s, 6, 5, iters=1, seed=11)
    out = {}
    calls, _ = _accounted(lambda: out.update(g=RT.global_descriptors(s, voc)))
    assert _counts(calls, "ltr_vlad") == [3]
    calls, classes = _accounted(lambda: RT.retrieve(out["g"], out["g"], 3))
    assert _counts(calls, "ltr_retrieve") == [2]
    assert classes == {"retrieval": 2}


@pytest.mark.gpu
def test_debug_hook_launch_is_counted_in_the_debug_class():
    from tests.test_posed_edges import hook
    A = np.tile(np.diag([4.0, 3.0, 2.0, 1.0]), (3, 1, 1))
    _, classes = _accounted(lambda: hook(A, np.ones((3, 4, 2)), shared=True))
    assert classes == {"debug": 1}


@pytest.mark.gpu
def test_pose_and_structure_entries_match_cupti():
    from tests.test_bundle import ring_matches, scene
    from tests.test_triangulation import _ragged, _res
    d, pairs, R, t = scene(3, V=8, n_pts=80, n_lines=16)
    res = ring_matches(d, pairs, DEV)
    calls, _ = _accounted(lambda: G.estimate_homographies(res))
    assert _counts(calls, "ltr_homography") == [2]
    calls, _ = _accounted(lambda: G.estimate_poses(res, d["K"], d["K"]))
    assert _counts(calls, "ltr_essential") == [2]
    d, pairs, mp, ml = _ragged(7)
    res = _res(d["keypoints"], d["klines"], pairs, mp, ml, DEV)
    calls, _ = _accounted(lambda: T.triangulate(d["keypoints"], d["klines"], pairs, res, d["K"], d["R"], d["t"]))
    assert _counts(calls, "ltr_triangulate") == [2]
    calls, _ = _accounted(lambda: TR.triangulate_tracks(d["keypoints"], d["klines"], pairs, res, d["K"], d["R"], d["t"]))
    assert _counts(calls, "ltr_tracks") == [6]


@pytest.mark.gpu
def test_encode_and_match_set_match_cupti():
    from tests.test_image_pairs import _model
    eng = engine.PairEngine(_model()[0], DEV)
    views = [syn.image_to(v, DEV) for v in syn.make_image_set(81, 4, 80, 200)]
    out = {}
    _accounted(lambda: out.update(s=eng.encode_images(views)))
    _accounted(lambda: eng.match_set(out["s"], engine.exhaustive_pairs(4)))
