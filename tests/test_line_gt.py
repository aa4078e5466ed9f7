"""Homography ground truth and precision / recall of line matches (`eval_homography`, `ltr_line_gt`) against the
reference's find_line_matches / calculate_line_overlaps / Evaluate_PR outputs in tests/golden/line_gt_outputs.npz
(tests/golden/make_line_gt_golden.py) and against the host restatement."""
import ctypes
import os

import numpy as np
import pytest
import torch

from linetr_b200 import _native as N, eval_homography as EH, synthetic as syn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "line_gt_outputs.npz")
DEV = torch.device("cuda", 0)
THR_R, THR_A, MIN_OV = 3, 2, 0.3


def _golden():
    z = np.load(GOLDEN)
    cases = []
    for k, name in enumerate(z["names"]):
        g = {key[len(f"c{k}_"):]: z[key] for key in z.files if key.startswith(f"c{k}_")}
        g["name"] = str(name)
        cases.append(g)
    return cases


def _mask(g, key):
    m = np.zeros((len(g["lines0"]), len(g["lines1"])), bool)
    idx = g[key]
    if len(idx):
        m[idx[:, 0], idx[:, 1]] = True
    return m


def _dense(pred, n1):
    """Reference score matrix of int predictions; like the kernel, indices outside [0, n1) are no prediction."""
    m = np.zeros((len(pred), n1))
    r = np.nonzero((pred >= 0) & (pred < n1))[0]
    m[r, pred[r]] = 1
    return m


# ------------------------------------------------------------------ CPU
def test_golden_flags_are_few_and_near_the_angle_boundary():
    n_ang = n_pow = n_entries = 0
    for g in _golden():
        n_entries += len(g["lines0"]) * len(g["lines1"])
        n_ang += len(g["ang_flag"])
        n_pow += len(g["pow_flag"])
        near = {tuple(x): m for x, m in zip(g["ang_near"].tolist(), g["ang_margin"])}
        for e in g["ang_flag"].tolist():
            assert near.get(tuple(e), np.inf) < 1e-3, (g["name"], e)
    print(f"\nline gt golden: {n_entries} entries, {n_ang} angle-flagged, {n_pow} sensitive to libm powf squares")
    assert n_ang <= 16 and n_pow <= 16


def test_host_restatement_equals_golden():
    """With the reference's cv2 projections every matrix equals the reference's outside the flagged entries; on
    entries flagged for the reference's powf squares the ratios differ by at most a few ulp."""
    for g in _golden():
        terms = EH.assignment_terms(g["lines0"], g["lines1"], g["proj0"], g["proj1"], THR_R, THR_A)
        ang, pw = _mask(g, "ang_flag"), _mask(g, "pow_flag")
        want = (g["m0"].astype(np.float64), g["m1"].astype(np.float64), g["ov0"].astype(np.float64),
                g["ov1"].astype(np.float64), g["assign"].astype(np.float64))
        for nm, got, w in zip(("m0", "m1", "ov0", "ov1", "assign"), terms, want):
            assert got.dtype == np.float64 and got.shape == w.shape, (g["name"], nm)
            bad = (got != w) & ~ang & ~pw
            assert not bad.any(), (g["name"], nm, np.argwhere(bad)[:5])
            np.testing.assert_allclose(got[pw], w[pw], rtol=1e-6, atol=0, err_msg=f"{g['name']} {nm}")


def test_line_assignment_equals_golden():
    for g in _golden():
        p0 = EH.project_lines(g["lines0"], g["H"])
        p1 = EH.project_lines(g["lines1"], np.linalg.inv(g["H"]))
        ulp = lambda a, b: np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))
        assert p0.shape == g["proj0"].shape and p1.shape == g["proj1"].shape
        if p0.size:
            assert ulp(p0, g["proj0"]).max() <= 1, g["name"]
        if p1.size:
            assert ulp(p1, g["proj1"]).max() <= 1, g["name"]
        assign, lm = EH.line_assignment(g["lines0"], g["lines1"], g["H"])
        assert assign.dtype == np.float64 and lm.dtype == np.int64 and lm.shape[1:] == (2,)
        flagged = _mask(g, "ang_flag") | _mask(g, "pow_flag")
        if np.array_equal(p0, g["proj0"]) and np.array_equal(p1, g["proj1"]):
            bad = (assign != g["assign"]) & ~flagged
            assert not bad.any(), (g["name"], np.argwhere(bad)[:5])
        want = {tuple(x) for x in g["lmatches"].tolist() if not flagged[x[0], x[1]]}
        got = {tuple(x) for x in lm.tolist() if not flagged[x[0], x[1]]}
        assert got == want, g["name"]


def test_precision_recall_equals_golden():
    for g in _golden():
        n1 = len(g["lines1"])
        for tag in ("nn", "hand"):
            score = _dense(g[f"pred_{tag}"], n1)
            assert EH.calc_tfpn(score, g["assign"].astype(np.float64)) == tuple(g[f"tfpn_{tag}"]), (g["name"], tag)
            p, r, f = EH.get_precision_recall(score[None], g["assign"][None].astype(np.float64))
            assert [p[0], r[0], f[0]] == list(g[f"pr_{tag}"]), (g["name"], tag)
            pv, rv, fv = EH.precision_recall_from_counts(g[f"tfpn_{tag}"][None])
            assert [pv[0], rv[0], fv[0]] == list(g[f"pr_{tag}"])


def test_argument_validation():
    s = np.zeros((2, 2, 2), np.float32)
    with pytest.raises(N.LtrError, match=r"\[P, 3, 3\]"):
        EH.homography_ground_truth(s, s, [0, 2], [0, 2], np.eye(3))
    with pytest.raises(N.LtrError, match="finite"):
        EH.homography_ground_truth(s, s, [0, 2], [0, 2], np.full((1, 3, 3), np.nan))
    with pytest.raises(N.LtrError, match="cu0"):
        EH.homography_ground_truth(s, s, [0, 1], [0, 2], np.eye(3)[None])
    with pytest.raises(N.LtrError, match="cu1"):
        EH.homography_ground_truth(s, s, [0, 2], [0, 3, 2], np.eye(3)[None])
    with pytest.raises(N.LtrError, match="segs0"):
        EH.homography_ground_truth(np.zeros((2, 4)), s, [0, 2], [0, 2], np.eye(3)[None])
    lib = N.load()

    def call(**kw):
        inp = N.LtrLineGtInput(n_pairs=kw.get("n_pairs", 1), max_n0=kw.get("max_n0", 4), max_n1=kw.get("max_n1", 4))
        out = N.LtrLineGtOutput(assign=kw.get("assign"), assign_stride=kw.get("stride", 0))
        return lib.ltr_line_gt(ctypes.byref(inp), ctypes.byref(out), 0, None)

    assert call(n_pairs=-1) == -1
    assert call(max_n0=-1) == -1 and call(max_n1=-2) == -1
    assert call(assign=16, stride=15) == -1          # stride < max_n0 * max_n1
    assert call() == -1                               # null n_gt and inputs
    assert call(n_pairs=0) == 0


# ------------------------------------------------------------------ GPU
def _cat(arrs):
    return np.concatenate([np.asarray(a, np.float32).reshape(-1, 2, 2) for a in arrs]) if arrs else np.zeros((0, 2, 2), np.float32)


def _cu(arrs):
    return np.concatenate([[0], np.cumsum([len(a) for a in arrs])]).astype(np.int32)


def _run(l0s, l1s, hs, **kw):
    return EH.homography_ground_truth(torch.from_numpy(_cat(l0s)).to(DEV), torch.from_numpy(_cat(l1s)).to(DEV),
                                      _cu(l0s), _cu(l1s), np.stack(hs), **kw)


def _preds(cases, tag):
    return torch.from_numpy(np.concatenate([g[f"pred_{tag}"] for g in cases]).astype(np.int32)).to(DEV)


@pytest.mark.gpu
def test_kernel_with_stored_projections_equals_golden():
    cases = _golden()
    l0s, l1s, hs = [g["lines0"] for g in cases], [g["lines1"] for g in cases], [g["H"] for g in cases]
    proj = dict(proj0=torch.from_numpy(_cat([g["proj0"] for g in cases])).to(DEV),
                proj1=torch.from_numpy(_cat([g["proj1"] for g in cases])).to(DEV))
    for tag in ("nn", "hand"):
        res = _run(l0s, l1s, hs, pred0=_preds(cases, tag), **proj)
        tfpn = res.tfpn.cpu().numpy()
        counts = res.counts.cpu().numpy()
        for p, g in enumerate(cases):
            got = res.assign(p)
            ang, pw = _mask(g, "ang_flag"), _mask(g, "pow_flag")
            host = EH.assignment_terms(g["lines0"], g["lines1"], g["proj0"], g["proj1"], THR_R, THR_A)[4]
            bad = (got != g["assign"]) & ~ang & ~pw
            assert not bad.any(), (g["name"], np.argwhere(bad)[:5])
            assert np.array_equal(got[~ang], host[~ang]), g["name"]   # bit for bit, powf-sensitive entries included
            if not ang.any():
                assert counts[p] == len(g["lmatches"]), g["name"]
                assert tuple(tfpn[p]) == tuple(g[f"tfpn_{tag}"]), (g["name"], tag)
                lm = res.lmatches(p)
                assert np.array_equal(lm, g["lmatches"]) or pw.any(), g["name"]
            assert tuple(tfpn[p]) == EH.calc_tfpn(_dense(g[f"pred_{tag}"], len(g["lines1"])), got), (g["name"], tag)


@pytest.mark.gpu
def test_device_projection_equals_host_projection():
    """Without caller projections the kernel projects itself (cv2's rule in fp64): its results equal those from the
    host projections (which match cv2's to 1 ulp) bit for bit, and the golden's decisions outside flagged entries."""
    cases = _golden()
    l0s, l1s, hs = [g["lines0"] for g in cases], [g["lines1"] for g in cases], [g["H"] for g in cases]
    own = _run(l0s, l1s, hs)
    host = _run(l0s, l1s, hs, proj0=torch.from_numpy(_cat([EH.project_lines(g["lines0"], g["H"]) for g in cases])).to(DEV),
                proj1=torch.from_numpy(_cat([EH.project_lines(g["lines1"], np.linalg.inv(g["H"])) for g in cases])).to(DEV))
    assert torch.equal(own.assign_flat, host.assign_flat) and torch.equal(own.counts, host.counts)
    for p, g in enumerate(cases):
        flagged = _mask(g, "ang_flag") | _mask(g, "pow_flag")
        got = own.assign(p)
        assert np.array_equal((got > 0)[~flagged], (g["assign"] > 0)[~flagged]), g["name"]
        assert np.array_equal((got > MIN_OV)[~flagged], (g["assign"] > MIN_OV)[~flagged]), g["name"]


def _ragged(seed, n_pairs=64):
    rng = np.random.default_rng(seed)
    l0s, l1s, hs = [], [], []
    for p in range(n_pairs):
        n0, n1 = (int(x) for x in rng.integers(0, 301, 2))
        if p % 16 == 3:
            n0 = 0
        if p % 16 == 7:
            n1 = 0
        h = np.eye(3)
        h[:2, :2] += rng.normal(0, 0.05, (2, 2))
        h[:2, 2] = rng.normal(0, 15, 2)
        h[2, :2] = rng.normal(0, 1e-4, 2)
        sp = rng.random((n0, 2)) * [620, 460] + 10
        d = rng.normal(0, 60, (n0, 2))
        l0 = np.stack([sp, sp + d], 1).astype(np.float32)
        m = min(n0, n1) * 3 // 4
        mapped = EH.project_lines(l0[:m], h) + rng.normal(0, 0.3, (m, 2, 2)).astype(np.float32)
        l1 = np.concatenate([mapped, (rng.random((n1 - m, 2, 2)) * [640, 480]).astype(np.float32)])
        l0s.append(l0)
        l1s.append(l1[rng.permutation(n1)].astype(np.float32))
        hs.append(h)
    return l0s, l1s, hs


@pytest.mark.gpu
def test_ragged_batch_equals_host_and_per_pair_calls():
    l0s, l1s, hs = _ragged(11)
    rng = np.random.default_rng(12)
    pred = [np.where(rng.random(len(a)) < 0.7, rng.integers(-1, max(len(b), 1), len(a)), -1).astype(np.int32)
            for a, b in zip(l0s, l1s)]
    pred_dev = torch.from_numpy(np.concatenate(pred)).to(DEV)
    res = _run(l0s, l1s, hs, pred0=pred_dev)
    only = _run(l0s, l1s, hs, pred0=pred_dev, want_assign=False)
    assert only.assign_flat is None
    assert torch.equal(res.tfpn, only.tfpn) and torch.equal(res.counts, only.counts)
    counts, tfpn = res.counts.cpu().numpy(), res.tfpn.cpu().numpy()
    n_true = 0
    for p in range(len(l0s)):
        want, _ = EH.line_assignment(l0s[p], l1s[p], hs[p])
        got = res.assign(p)
        assert got.shape == want.shape and np.array_equal(got, want), p
        assert counts[p] == int((want > MIN_OV).sum()), p
        assert tuple(tfpn[p]) == EH.calc_tfpn(_dense(pred[p], len(l1s[p])), want), p
        n_true += int(counts[p])
    assert n_true > 1000
    for p in (0, 3, 7, 20, 63):   # the batched call equals per-pair calls bit for bit
        one = _run([l0s[p]], [l1s[p]], [hs[p]], pred0=torch.from_numpy(pred[p]).to(DEV))
        assert np.array_equal(one.assign(0), res.assign(p)) and np.array_equal(one.assign(0).view(np.int64),
                                                                                res.assign(p).view(np.int64)), p
        assert torch.equal(one.tfpn[0], res.tfpn[p]) and int(one.counts[0]) == counts[p]
    pr = res.precision_recall()
    assert all(np.array_equal(a, b) for a, b in zip(pr, EH.precision_recall_from_counts(tfpn)))


@pytest.mark.gpu
def test_score_line_matches_end_to_end():
    from linetr_b200 import LineTransformer, PairEngine
    m = LineTransformer({"mode": "train"})
    sd = syn.make_state_dict(0, 1)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    eng = PairEngine(m.eval().to(DEV), DEV)
    pairs = [tuple(syn.image_to(x, DEV) for x in syn.make_image_pair(500 + p, 60 + 20 * p, 100)) for p in range(4)]
    res = eng.match_images([a for a, _ in pairs], [b for _, b in pairs])
    hs = np.stack([np.eye(3)] * len(pairs))
    got = EH.score_line_matches(res, hs)
    ps, rs, fs = [], [], []
    for p in range(res.n_pairs):
        k0, k1 = np.asarray(res.klines0[p], np.float32), np.asarray(res.klines1[p], np.float32)
        assign, _ = EH.line_assignment(k0, k1, np.eye(3))
        score = _dense(res.pair_lines(p).cpu().numpy(), len(k1))
        a, b, c = EH.get_precision_recall(score[None], assign[None])
        ps.append(a[0]); rs.append(b[0]); fs.append(c[0])
    assert list(got["precision"]) == ps and list(got["recall"]) == rs and list(got["f1"]) == fs
    P = len(ps)
    assert (got["mean_precision"], got["mean_recall"], got["mean_f1"]) == (np.sum(ps) / P, np.sum(rs) / P, np.sum(fs) / P)
    assert got["mean_recall"] > 0
