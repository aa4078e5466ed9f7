"""The validation step's semi-hard triplet loss (`eval_criteria`, `ltr_triplet_loss`) against the reference's
descriptor_loss and Result.evaluate outputs in tests/golden/triplet_outputs.npz (tests/golden/make_triplet_golden.py),
against the host restatement, and against an fp32 FMA model of the distances the kernel promises.

`dist32_model` is the unclipped variant of tests/test_matcher_edges.py's model: d = 2 - 2 acc with acc an
ascending-k fmaf chain, compiled without contraction.  On its distances the host restatement must give every
anchor's pos, neg and state bit for bit."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from linetr_b200 import _native as N, eval_criteria as EC, eval_homography as EH, eval_matcher as em

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "triplet_outputs.npz")
DEV = torch.device("cuda", 0)
ROWS, CF = N.LAYOUT_ROWS, N.LAYOUT_CHANNEL_FIRST
F32_03 = EC.MATCH_THR_F32


def _golden():
    z = np.load(GOLDEN)
    cases = []
    for k, name in enumerate(z["names"]):
        g = {key[len(f"c{k}_"):]: z[key] for key in z.files if key.startswith(f"c{k}_")}
        g["name"] = str(name)
        g["raised"] = str(g["raised"])
        cases.append(g)
    return cases


def _same(a, b):
    """Bit-for-bit equality of float arrays, NaN where NaN."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(a[~na].view(np.int32), b[~nb].view(np.int32)))


# ------------------------------------------------------------------ CPU
def _ref_terms(g):
    """The reference's per-anchor terms stored with the case."""
    return {"pos": g["ref_pos"], "neg": g["ref_neg"], "state": g["ref_state"].astype(np.int32)}


def test_host_restatement_equals_golden():
    """On the reference's own distances (stored for the small cases) the restatement gives the stored per-anchor terms
    bit for bit; their valid anchors are the reference's outputs bit for bit in every case."""
    n_dist = 0
    for g in _golden():
        ref = _ref_terms(g)
        if "dist" in g:
            n_dist += 1
            t = EC.triplet_terms(list(g["dist"]), [a[:-1, :-1] for a in g["assign"]])
            assert _same(t["pos"], ref["pos"]) and _same(t["neg"], ref["neg"]), g["name"]
            assert np.array_equal(t["state"], ref["state"]), g["name"]
        t = dict(ref, **dict(zip(("loss", "hardest_pos", "hardest_neg", "n_valid"),
                                 EC.group_values(ref["pos"], ref["neg"], ref["state"]))))
        if g["raised"]:
            assert t["n_valid"] == 0 and np.isnan(t["loss"]), g["name"]
            if g["name"] == "nopos":
                assert not (t["state"] > 0).any()
            continue
        v = t["state"] == EC.STATE_VALID
        assert _same(t["pos"][v], g["dists_pos"]) and _same(t["neg"][v], g["dists_neg"]), g["name"]
        assert t["hardest_pos"] == g["hardest_pos"] and t["hardest_neg"] == g["hardest_neg"], g["name"]
        np.testing.assert_allclose(t["loss"], g["loss"], rtol=1e-6, atol=0, err_msg=g["name"])
        assert t["n_valid"] == len(g["dists_pos"])
    assert n_dist >= 5


def test_golden_covers_the_edges():
    """The fixtures exercise what the issue of the loss is about: 0.3f entries, the 10000 literal, pos near 0."""
    by = {g["name"]: g for g in _golden()}
    a = by["overlap"]["assign"][:, :-1, :-1]
    assert (a == np.float32(0.3)).any() and ((a > 0) & (a < np.float32(0.3))).any()
    assert (np.asarray(by["far"]["dists_neg"]) == np.float32(10000)).any()
    assert (np.asarray(by["duplicate"]["dists_pos"]) < 1e-6).any()
    assert {g["raised"] for g in by.values()} == {"", "RuntimeError"}


def test_drop_in_refuses_what_it_cannot_do():
    crit = EC.descriptor_loss()
    x = torch.zeros(1, 256, 4)
    a = torch.zeros(1, 5, 5)
    with pytest.raises(N.LtrError, match="require grad"):
        crit({"line_desc0": x.clone().requires_grad_(), "line_desc1": x}, {"mat_assign_sublines": a})
    with pytest.raises(N.LtrError, match="as many lines"):
        crit({"line_desc0": x, "line_desc1": torch.zeros(1, 256, 3)}, {"mat_assign_sublines": a})
    with pytest.raises(N.LtrError, match="mat_assign_sublines"):
        crit({"line_desc0": x, "line_desc1": x}, {"mat_assign_sublines": torch.zeros(1, 4, 4)})


def test_entry_return_codes():
    lib = N.load()

    def call(out=True, **kw):
        f = dict(d=256, n_pairs=1, n0=4, n1=4, n_groups=1, assign_stride=16)
        f.update(kw)
        inp = N.LtrTripletInput(**f)
        o = N.LtrTripletOutput()
        rc = lib.ltr_triplet_loss(ctypes.byref(inp), ctypes.byref(o) if out else None, 0, None)
        return rc, lib.ltr_last_error().decode()

    assert call(out=False) == (-1, "ltr_triplet_loss: null argument")
    rc, msg = call(d=128)
    assert rc == -4 and msg.startswith("ltr_triplet_loss: descriptor dim")
    assert call(d=128, layout=7)[0] == -4                    # the dimension is checked first
    assert call(layout=2)[1] == "ltr_triplet_loss: bad layout"
    for kw in ({"n_pairs": -1}, {"n0": -1}, {"max_n1": -1}, {"assign_ld": -1}, {"assign_stride": -1}):
        assert call(**kw) == (-1, "ltr_triplet_loss: negative count"), kw
    assert call(cu0=16)[1].startswith("ltr_triplet_loss: cu0/cu1")
    assert call(n_groups=0)[1].startswith("ltr_triplet_loss: n_groups")
    assert call(n_groups=2)[1].startswith("ltr_triplet_loss: n_groups")   # two groups need group_off
    assert call(n0=1 << 30, assign_stride=1 << 40)[1] == "ltr_triplet_loss: a pair side has 2^30 lines or more"
    assert call(assign_ld=3)[1] == "ltr_triplet_loss: assign_ld < max_n1"
    assert call(assign_stride=15)[1].startswith("ltr_triplet_loss: assign_stride")
    assert call(assign_ld=5, assign_stride=19)[1].startswith("ltr_triplet_loss: assign_stride")
    assert call(n_pairs=0)[0] == 0                            # nothing to do
    assert call()[1] == "ltr_triplet_loss: null output"


# ------------------------------------------------------------------ GPU
_MODEL_SRC = r"""
#include <math.h>
/* 2 - 2 acc, acc an ascending-k fmaf chain; not clipped */
void model_dist_raw(const float* a, const float* b, long n0, long n1, int d, float* out) {
  for (long i = 0; i < n0; ++i)
    for (long j = 0; j < n1; ++j) {
      float acc = 0.f;
      for (int k = 0; k < d; ++k) acc = fmaf(a[i * d + k], b[j * d + k], acc);
      out[i * n1 + j] = 2.f - 2.f * acc;
    }
}
"""


@pytest.fixture(scope="module")
def model32(tmp_path_factory):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler for the fp32 FMA model")
    td = tmp_path_factory.mktemp("fp32_model_raw")
    src, so = str(td / "model.c"), str(td / "model.so")
    with open(src, "w") as f:
        f.write(_MODEL_SRC)
    subprocess.check_call([cc, "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", "-o", so, src, "-lm"])
    lib = ctypes.CDLL(so)
    f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
    lib.model_dist_raw.argtypes = [f32p, f32p, ctypes.c_long, ctypes.c_long, ctypes.c_int, f32p]

    def dist(a, b):
        """rows a [n0, 256], b [n1, 256] -> fp32 [n0, n1]"""
        a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
        out = np.empty((len(a), len(b)), np.float32)
        if out.size:
            lib.model_dist_raw(a, b, len(a), len(b), a.shape[1], out)
        return out
    return dist


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _np(t):
    return t.cpu().numpy()


def _check_anchors(res, want, what):
    assert _same(_np(res.pos), want["pos"]), what
    assert _same(_np(res.neg), want["neg"]), what
    assert np.array_equal(_np(res.state), want["state"]), what


def _check_group(res, g, want, what):
    nv = int(res.n_valid[g])
    assert nv == want["n_valid"], what
    if nv == 0:
        assert np.isnan(_np(res.loss)[g]) and np.isnan(_np(res.hardest_pos)[g]) and np.isnan(_np(res.hardest_neg)[g])
        return
    assert _np(res.hardest_pos)[g] == want["hardest_pos"] and _np(res.hardest_neg)[g] == want["hardest_neg"], what
    np.testing.assert_allclose(_np(res.loss)[g], want["loss"], rtol=1e-6, atol=0, err_msg=what)


def _golden_batch(g):
    pred = {"line_desc0": _t(g["desc0"]), "line_desc1": _t(g["desc1"])}
    return pred, {"mat_assign_sublines": _t(g["assign"])}


@pytest.mark.gpu
def test_golden_bit_for_bit_against_fp32_model(model32):
    crit = EC.descriptor_loss()
    for g in _golden():
        x, y, a = g["desc0"], g["desc1"], g["assign"]
        want = EC.triplet_terms([model32(x[p].T, y[p].T) for p in range(len(x))], [m[:-1, :-1] for m in a], F32_03, 0.0)
        res = EC.triplet_loss(_t(x), _t(y), _t(a), layout=CF, match_thr=F32_03)
        _check_anchors(res, want, g["name"])
        _check_group(res, 0, want, g["name"])
        pred, target = _golden_batch(g)
        if want["n_valid"] == 0:
            with pytest.raises(N.LtrError):
                crit(pred, target)
            continue
        dp, dn = crit.compute_distances(pred, target)
        v = want["state"] == EC.STATE_VALID
        assert _same(_np(dp), want["pos"][v]) and _same(_np(dn), want["neg"][v]), g["name"]
        loss, hp, hn = crit(pred, target)
        assert loss.dim() == 0 and loss.dtype == torch.float32 and loss.device == DEV
        assert float(hp) == want["hardest_pos"] and float(hn) == want["hardest_neg"]
        assert float(loss) == float(res.loss[0])


def _decisive(x, y, assign, want_pos):
    """Anchors (in the reference's order) whose decisions no fp32 rounding can change: no candidate's float64 distance
    (or the literal 10000) within tol of pos or pos + 0.5, pos farther than tol from 0; tol = 1e-5 max(1, |a||b|)."""
    keep = []
    for p in range(len(x)):
        a, b = x[p].T.astype(np.float64), y[p].T.astype(np.float64)
        d = 2.0 - 2.0 * a @ b.T
        na, nb = np.linalg.norm(a, axis=1), np.linalg.norm(b, axis=1)
        m = assign[p][:-1, :-1].astype(np.float64)
        for D, M, s in ((d, m, na[:, None] * nb[None, :]), (d.T, m.T, (na[:, None] * nb[None, :]).T)):
            tol = 1e-5 * np.maximum(1.0, s.max(axis=1, initial=0))
            match, unmatch = M > F32_03, M <= 0
            pos = np.where(match, D, -np.inf).max(axis=1, initial=-np.inf)
            u = np.where(unmatch, D, 10000.0)
            near = lambda v: (np.abs(u - v[:, None]) <= tol[:, None]).any(axis=1)
            keep.append(~((np.abs(pos) <= tol) | near(pos) | near(pos + 0.5)))
    return np.concatenate(keep)


@pytest.mark.gpu
def test_golden_decisive_anchors_equal_reference():
    n_all = n_non = 0
    for g in _golden():
        ref = _ref_terms(g)
        res = EC.triplet_loss(_t(g["desc0"]), _t(g["desc1"]), _t(g["assign"]), layout=CF, match_thr=F32_03)
        dec = _decisive(g["desc0"], g["desc1"], g["assign"], ref["pos"])
        st, pos, neg = _np(res.state), _np(res.pos), _np(res.neg)
        assert np.array_equal(st[dec], ref["state"][dec]), g["name"]
        tol = 1e-5 * max(1.0, float(np.linalg.norm(g["desc0"], axis=1).max() * np.linalg.norm(g["desc1"], axis=1).max()))
        ok = dec & (st > 0)
        np.testing.assert_allclose(pos[ok], ref["pos"][ok], rtol=0, atol=tol, err_msg=g["name"])
        ok = dec & (st == 2)
        np.testing.assert_allclose(neg[ok], ref["neg"][ok], rtol=0, atol=tol, err_msg=g["name"])
        n_all += len(dec)
        n_non += int((~dec).sum())
        if not g["raised"] and dec.all():
            np.testing.assert_allclose(float(res.loss[0]), g["loss"], rtol=1e-5, err_msg=g["name"])
    print(f"\ntriplet golden: {n_all} anchors, {n_non} not decisive")
    assert n_non < n_all // 4


@pytest.mark.gpu
def test_threshold_semantics(model32):
    """An entry exactly 0.3f: no match in float32 (the drop-in), a match against the float64 0.3."""
    rng = np.random.default_rng(3)
    n = 24
    x = rng.normal(size=(n, 256)).astype(np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    y = (x + rng.normal(0, 0.15, x.shape)).astype(np.float32)
    y /= np.linalg.norm(y, axis=1, keepdims=True)
    a = np.zeros((1, n + 1, n + 1), np.float32)
    a[0, np.arange(n), np.arange(n)] = np.where(np.arange(n) % 2, np.float32(0.3), np.float32(1.0))
    d = model32(x, y)
    want32 = EC.triplet_terms(d, a[0, :-1, :-1], F32_03, 0.0)
    want64 = EC.triplet_terms(d, a[0, :-1, :-1], 0.3, 0.0)
    assert (want32["state"] == 0).sum() > (want64["state"] == 0).sum()
    xc, yc = _t(x.T[None]), _t(y.T[None])
    for thr, want in ((F32_03, want32), (0.3, want64)):
        _check_anchors(EC.triplet_loss(xc, yc, _t(a), layout=CF, match_thr=thr), want, thr)
    dp, _ = EC.descriptor_loss().compute_distances({"line_desc0": xc, "line_desc1": yc}, {"mat_assign_sublines": _t(a)})
    assert _same(_np(dp), want32["pos"][want32["state"] == 2])


def _segments(seed, n_pairs):
    from tests.test_line_gt import _ragged
    return _ragged(seed, n_pairs)


def _unit_rows(rng, n):
    x = rng.normal(size=(n, 256)).astype(np.float32)
    return x / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), 1e-12)


@pytest.mark.gpu
def test_line_ground_truth_in_place_equals_lmatches_matrix():
    """train.py's 0/1 matrix from lmatches (assign > 0.3) equals the raw overlaps at match_thr = unmatch_thr = 0.3."""
    l0s, l1s, hs = _segments(21, 12)
    cu0 = np.concatenate([[0], np.cumsum([len(v) for v in l0s])]).astype(np.int32)
    cu1 = np.concatenate([[0], np.cumsum([len(v) for v in l1s])]).astype(np.int32)
    gt = EH.homography_ground_truth(np.concatenate(l0s), np.concatenate(l1s), cu0, cu1, np.stack(hs), device=DEV)
    rng = np.random.default_rng(22)
    # a shared component puts unrelated lines about 1 apart, so that the semi-hard windows of matched lines fill
    common = _unit_rows(rng, 1)
    d0, d1 = _unit_rows(rng, cu0[-1]) + common, _unit_rows(rng, cu1[-1]) + common
    for p in range(len(l0s)):
        r, c = np.nonzero(gt.assign(p) > 0.3)
        d1[cu1[p] + c] = _unit_rows(rng, len(c)) * 1.1 + d0[cu0[p] + r]
    d0 /= np.linalg.norm(d0, axis=1, keepdims=True)
    d1 /= np.linalg.norm(d1, axis=1, keepdims=True)
    mx0, mx1 = int(np.diff(cu0).max()), int(np.diff(cu1).max())
    lm = np.zeros((len(l0s), mx0, mx1), np.float32)
    for p in range(len(l0s)):
        r, c = gt.lmatches(p).T
        lm[p, r, c] = 1
    a = EC.triplet_loss(_t(d0), _t(d1), gt, cu0=cu0, cu1=cu1, match_thr=0.3, unmatch_thr=0.3)
    b = EC.triplet_loss(_t(d0), _t(d1), _t(lm), cu0=cu0, cu1=cu1, match_thr=F32_03, unmatch_thr=0.0)
    for k in ("pos", "neg", "state", "loss", "hardest_pos", "hardest_neg", "n_valid"):
        assert torch.equal(getattr(a, k).view(torch.int32), getattr(b, k).view(torch.int32)), k
    assert int(a.n_valid[0]) > 100


def _ragged_batch(seed, n_pairs=64):
    rng = np.random.default_rng(seed)
    common = _unit_rows(rng, 1)
    d0s, d1s, asg = [], [], []
    for p in range(n_pairs):
        n0, n1 = (int(v) for v in rng.integers(0, 161, 2))
        if p % 16 == 3:
            n0 = 0
        if p % 16 == 7:
            n1 = 0
        # a shared component puts unrelated lines about 1 apart: semi-hard windows of matched lines fill
        x = _unit_rows(rng, n0) + common
        m = min(n0, n1) * 2 // 3
        y = _unit_rows(rng, n1) + common
        y[:m] = x[:m] + _unit_rows(rng, m) * rng.uniform(0.05, 1.5, (m, 1)).astype(np.float32)
        x /= np.linalg.norm(x, axis=1, keepdims=True)
        y /= np.linalg.norm(y, axis=1, keepdims=True)
        a = np.zeros((n0, n1), np.float32)
        if p % 16 != 5:   # pair 5, 21, ...: no match at all
            a[np.arange(m), np.arange(m)] = rng.choice([1.0, 0.6, 0.3, 0.2], m).astype(np.float32)
            a[rng.random((n0, n1)) < 0.02] = np.float32(0.1)
        perm = rng.permutation(n1)
        d0s.append(x); d1s.append(y[perm]); asg.append(a[:, perm])
    return d0s, d1s, asg


def _flat_assign(asg, mx0, mx1):
    out = np.zeros((len(asg), mx0, mx1), np.float32)
    for p, a in enumerate(asg):
        out[p, :a.shape[0], :a.shape[1]] = a
    return out


def _cu(arrs):
    return np.concatenate([[0], np.cumsum([len(v) for v in arrs])]).astype(np.int32)


@pytest.mark.gpu
def test_ragged_batch_against_model_layouts_groups_and_repeats(model32):
    d0s, d1s, asg = _ragged_batch(5)
    P = len(d0s)
    cu0, cu1 = _cu(d0s), _cu(d1s)
    mx0, mx1 = int(np.diff(cu0).max()), int(np.diff(cu1).max())
    A = _t(_flat_assign(asg, mx0, mx1))
    d0, d1 = np.concatenate(d0s), np.concatenate(d1s)
    rng = np.random.default_rng(6)
    pred = [np.where(rng.random(len(x)) < 0.8, rng.integers(-1, max(len(y), 1) + 2, len(x)), -1).astype(np.int32)
            for x, y in zip(d0s, d1s)]
    pred_dev = _t(np.concatenate(pred))
    want = EC.triplet_terms([model32(x, y) for x, y in zip(d0s, d1s)], asg, 0.3, 0.0)
    rows = EC.triplet_loss(_t(d0), _t(d1), A, cu0=cu0, cu1=cu1, pred0=pred_dev)
    _check_anchors(rows, want, "ragged rows")
    _check_group(rows, 0, want, "ragged rows")
    assert want["n_valid"] > 500 and (want["state"] == 1).any() and (want["state"] == 0).any()
    tfpn = _np(rows.tfpn)
    for p in range(P):
        score = np.zeros(asg[p].shape)
        r = np.nonzero((pred[p] >= 0) & (pred[p] < asg[p].shape[1]))[0]
        score[r, pred[p][r]] = 1
        assert tuple(tfpn[p]) == EH.calc_tfpn(score, (asg[p].astype(np.float64) > 0.3).astype(np.float64)), p
    # channel-first [256, n_p] per pair back to back gives the same bits
    cf = np.concatenate([x.T.reshape(-1) for x in d0s]), np.concatenate([y.T.reshape(-1) for y in d1s])
    chan = EC.triplet_loss(_t(cf[0]), _t(cf[1]), A, cu0=cu0, cu1=cu1, layout=CF, pred0=pred_dev)
    for k in ("pos", "neg", "state", "loss", "hardest_pos", "hardest_neg", "n_valid", "tfpn"):
        assert torch.equal(getattr(rows, k).view(torch.int32), getattr(chan, k).view(torch.int32)), k
    # groups equal one call per group; an identical call gives identical bits
    groups = np.array([0, 5, 6, 6, 30, P], np.int32)
    grp = EC.triplet_loss(_t(d0), _t(d1), A, cu0=cu0, cu1=cu1, groups=groups)
    again = EC.triplet_loss(_t(d0), _t(d1), A, cu0=cu0, cu1=cu1, groups=groups)
    for k in ("pos", "neg", "state", "loss", "hardest_pos", "hardest_neg", "n_valid"):
        assert torch.equal(getattr(grp, k).view(torch.int32), getattr(again, k).view(torch.int32)), k
    assert torch.equal(grp.pos.view(torch.int32), rows.pos.view(torch.int32))
    assert int(grp.n_valid[2]) == 0 and np.isnan(float(grp.loss[2]))   # an empty group
    for gi in range(len(groups) - 1):
        a, b = groups[gi], groups[gi + 1]
        one = EC.triplet_loss(_t(d0[cu0[a]:cu0[b]]), _t(d1[cu1[a]:cu1[b]]), A[a:b], cu0=cu0[a:b + 1] - cu0[a],
                              cu1=cu1[a:b + 1] - cu1[a])
        for k in ("loss", "hardest_pos", "hardest_neg", "n_valid"):
            assert getattr(one, k)[0].view(torch.int32) == getattr(grp, k)[gi].view(torch.int32), (gi, k)
        sub = EC.triplet_terms([model32(x, y) for x, y in zip(d0s[a:b], d1s[a:b])], asg[a:b], 0.3, 0.0)
        _check_group(grp, gi, sub, f"group {gi}")


@pytest.mark.gpu
def test_validation_metrics_equals_reference_evaluate():
    for g in _golden():
        x, y, a = g["desc0"], g["desc1"], g["assign"]
        res = EC.validation_metrics(_t(x), _t(y), _t(a), layout=CF, match_thr=F32_03)
        p, r, f = res.precision_recall()
        score = em.nn_matcher_batches(x, y, 0.7, is_mutual_NN=True)[:, :-1, :-1]
        # ground truth is the match class, Result.evaluate's `> 0` on train.py's 0/1 matrices
        gt = (a[:, :-1, :-1].astype(np.float64) > F32_03).astype(np.float64)
        hp, hr, hf = EH.get_precision_recall(score, gt)
        assert list(p) == hp and list(r) == hr and list(f) == hf, g["name"]
        if "pr" in g and np.isin(a, (0, 1)).all():
            assert np.array_equal(np.stack([p, r, f], 1), g["pr"]), g["name"]
        plain = EC.triplet_loss(_t(x), _t(y), _t(a), layout=CF, match_thr=F32_03)
        for k in ("pos", "neg", "state", "loss"):
            assert torch.equal(getattr(res, k).view(torch.int32), getattr(plain, k).view(torch.int32)), k


@pytest.mark.gpu
def test_no_valid_anchor_gives_nan_and_the_drop_in_raises():
    for g in _golden():
        if not g["raised"]:
            continue
        res = EC.triplet_loss(_t(g["desc0"]), _t(g["desc1"]), _t(g["assign"]), layout=CF, match_thr=F32_03)
        assert int(res.n_valid[0]) == 0
        assert all(np.isnan(float(getattr(res, k)[0])) for k in ("loss", "hardest_pos", "hardest_neg"))
        pred, target = _golden_batch(g)
        with pytest.raises(N.LtrError, match="no anchor"):
            EC.descriptor_loss()(pred, target)
