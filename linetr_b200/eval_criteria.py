"""The descriptor loss of the reference's validation step (`evaluations/criteria.py`) on the CUDA library.

Drop-in, same name and call surface as the reference module (forward value only, no gradient):

    descriptor_loss().forward(pred, target) -> (t_loss, hardest_positive, hardest_negative)   (criteria.py:35-192)
    descriptor_loss().compute_distances(pred, target) -> (dists_pos, dists_neg)
        pred['line_desc0'] / pred['line_desc1'] [b, 256, n], target['mat_assign_sublines'] float32 [b, n+1, n+1]
        (read in place, dustbin included, with torch's float32 threshold semantics)

Host restatement, the oracle of the tests:

    triplet_terms(dist, assign, match_thr, unmatch_thr) -> per-anchor pos / neg / state and the group values

Batched on the GPU (`ltr_triplet_loss`):

    triplet_loss(desc0, desc1, assign, ...) -> TripletLoss       ragged pairs, groups of pairs, optional predictions
    validation_metrics(desc0, desc1, assign, ...) -> TripletLoss  train.py's run_epochs('val') after the forward:
        the loss terms plus precision / recall / F1 of nn_matcher_batches (distance mode 1, nn_thresh 0.7, mutual)

Semantics (include/linetr_b200.h, ltr_triplet_loss): d = 2 - 2 <a, b> in fp32, not clipped; an entry is a match if
its assignment value is > match_thr and an unmatch if it is <= unmatch_thr (compared in float64); anchors are the
side-0 lines then the side-1 lines of every pair; pos = max d over match candidates (a positive iff pos > 0);
neg = min over pos < u < pos + 0.5f of u = (unmatch ? d : 10000); valid iff that window is not empty;
loss = mean relu((pos - neg) + 1) over the valid anchors.  The reference thresholds a float32 tensor against 0.3,
which torch evaluates in float32: pass match_thr = MATCH_THR_F32 = float(np.float32(0.3)) for that.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from . import _native as N
from . import _ops
from .eval_homography import LineGroundTruth, precision_recall_from_counts

MATCH_THR_F32 = float(np.float32(0.3))   # criteria.py:63 `overlap_gt > 0.3` on a float32 tensor
FAR = np.float32(10000.0)                # criteria.py:95 max_dist
MARGIN = np.float32(0.5)                 # criteria.py:102
LOSS_MARGIN = np.float32(1.0)            # criteria.py:183

STATE_NO_POSITIVE, STATE_EMPTY_WINDOW, STATE_VALID = 0, 1, 2


# ------------------------------------------------------------------ host restatement
def _anchor_terms(dist, match, unmatch):
    """Rows of `dist` are anchors, columns their candidates: -> (pos, neg, state) float32 / float32 / int32."""
    n = dist.shape[0]
    if dist.shape[1] == 0:
        return np.full(n, np.nan, np.float32), np.full(n, np.nan, np.float32), np.zeros(n, np.int32)
    pos = np.where(match, dist, np.float32(-np.inf)).max(axis=1).astype(np.float32)
    has = pos > 0
    u = np.where(unmatch, dist, FAR).astype(np.float32)
    hi = (pos + MARGIN).astype(np.float32)
    win = (u > pos[:, None]) & (u < hi[:, None])
    neg = np.where(win, u, np.float32(np.inf)).min(axis=1).astype(np.float32)
    valid = has & win.any(axis=1)
    state = np.where(valid, STATE_VALID, np.where(has, STATE_EMPTY_WINDOW, STATE_NO_POSITIVE)).astype(np.int32)
    return np.where(has, pos, np.nan).astype(np.float32), np.where(valid, neg, np.nan).astype(np.float32), state


def group_values(pos, neg, state):
    """(loss, hardest_pos, hardest_neg, n_valid) of the anchors of one group: loss = float32(sum in float64 of the
    float32 terms relu((pos - neg) + 1) / n_valid); NaN for all three without a valid anchor."""
    v = np.asarray(state) == STATE_VALID
    n = int(v.sum())
    if n == 0:
        return np.float32(np.nan), np.float32(np.nan), np.float32(np.nan), 0
    p, q = np.asarray(pos, np.float32)[v], np.asarray(neg, np.float32)[v]
    terms = np.maximum((p - q) + LOSS_MARGIN, np.float32(0)).astype(np.float32)
    return np.float32(terms.astype(np.float64).sum() / n), p.max(), q.min(), n


def triplet_terms(dist, assign, match_thr=MATCH_THR_F32, unmatch_thr=0.0) -> dict:
    """descriptor_loss.compute_distances + forward on given distances.  dist / assign: one [n0, n1] matrix or a list of
    them (one per pair, float32 distances); -> dict of per-anchor 'pos', 'neg' (float32, NaN where undefined), 'state'
    (int32: 0 no positive, 1 empty window, 2 valid) in the reference's anchor order (pair-major, side-0 lines then
    side-1 lines) and the group's 'loss', 'hardest_pos', 'hardest_neg', 'n_valid'."""
    if isinstance(dist, np.ndarray) and dist.ndim == 2:
        dist, assign = [dist], [assign]
    parts = []
    for d, a in zip(dist, assign):
        d = np.asarray(d, np.float32)
        a = np.asarray(a, np.float64)
        match, unmatch = a > match_thr, a <= unmatch_thr
        parts.append(_anchor_terms(d, match, unmatch))
        parts.append(_anchor_terms(np.ascontiguousarray(d.T), match.T, unmatch.T))
    cat = lambda k, dt: np.concatenate([x[k] for x in parts]).astype(dt) if parts else np.zeros(0, dt)
    pos, neg, state = cat(0, np.float32), cat(1, np.float32), cat(2, np.int32)
    loss, hp, hn, nv = group_values(pos, neg, state)
    return {"pos": pos, "neg": neg, "state": state, "loss": loss, "hardest_pos": hp, "hardest_neg": hn, "n_valid": nv}


# ------------------------------------------------------------------ batched on the GPU
@dataclass
class TripletLoss:
    """Result of `triplet_loss` / `validation_metrics` (device tensors; nothing has been waited for).

    Per anchor (side-0 line i of pair p at a0[p] + i, side-1 line j at a0[p] + n0[p] + j, a0[p] = cu0[p] + cu1[p]):
    pos, neg float32 and state int32.  Per group: loss, hardest_pos, hardest_neg float32 (NaN without a valid anchor) and
    n_valid int32.  tfpn int32 [P, 4] (TP, FP, FN, TN) when predictions were given; matches0 the predictions of
    `validation_metrics`."""
    pos: torch.Tensor
    neg: torch.Tensor
    state: torch.Tensor
    loss: torch.Tensor
    hardest_pos: torch.Tensor
    hardest_neg: torch.Tensor
    n_valid: torch.Tensor
    tfpn: Optional[torch.Tensor]
    n0: np.ndarray
    n1: np.ndarray
    groups: np.ndarray
    matches0: Optional[torch.Tensor] = None

    @property
    def n_pairs(self) -> int:
        return len(self.n0)

    def anchors(self, p: int) -> slice:
        """Anchor range of pair p (its side-0 lines, then its side-1 lines)."""
        a0 = int(self.n0[:p].sum() + self.n1[:p].sum())
        return slice(a0, a0 + int(self.n0[p] + self.n1[p]))

    def precision_recall(self):
        """Per-pair (precision, recall, f1) float64 [P] from the counts, Evaluate_PR's formulas (host copy)."""
        if self.tfpn is None:
            raise N.LtrError("precision_recall() needs predictions (validation_metrics, or triplet_loss(..., pred0=...))")
        return precision_recall_from_counts(self.tfpn.cpu().numpy())


def _offsets(cu, n_pairs, n_lines, name) -> np.ndarray:
    cu = np.asarray(cu)
    if cu.ndim != 1 or len(cu) != n_pairs + 1 or not np.issubdtype(cu.dtype, np.integer):
        raise N.LtrError(f"triplet_loss: {name} must be integers [{n_pairs + 1}]")
    if cu[0] != 0 or cu[-1] != n_lines or np.any(np.diff(cu) < 0):
        raise N.LtrError(f"triplet_loss: {name} must rise from 0 to {n_lines}")
    return np.ascontiguousarray(cu, dtype=np.int32)


def _side(desc, cu, layout, name):
    """-> (float32 tensor, n_pairs, uniform n or None, host offsets or None)."""
    if not isinstance(desc, torch.Tensor) or not desc.is_cuda or desc.dtype != torch.float32:
        raise N.LtrError(f"triplet_loss: {name} must be a float32 CUDA tensor")
    desc = desc.contiguous()
    if cu is None:
        if desc.dim() != 3 or desc.shape[2 if layout == N.LAYOUT_ROWS else 1] != 256:
            raise N.LtrError(f"triplet_loss: without offsets {name} must be [P, n, 256] (rows) or [P, 256, n] "
                             "(channel-first)")
        return desc, int(desc.shape[0]), int(desc.shape[1 if layout == N.LAYOUT_ROWS else 2]), None
    if desc.numel() % 256:
        raise N.LtrError(f"triplet_loss: {name} must hold 256 channels per line")
    c = np.asarray(cu)
    return desc, len(c) - 1, None, _offsets(c, len(c) - 1, desc.numel() // 256, "cu" + name[-1])


def _prepare(desc0, desc1, assign, cu0, cu1, layout, assign_ld, groups):
    if layout not in (N.LAYOUT_ROWS, N.LAYOUT_CHANNEL_FIRST):
        raise N.LtrError("triplet_loss: layout must be LAYOUT_ROWS or LAYOUT_CHANNEL_FIRST")
    if (cu0 is None) != (cu1 is None):
        raise N.LtrError("triplet_loss: cu0 and cu1 must be given together")
    d0, P, u0, c0 = _side(desc0, cu0, layout, "desc0")
    d1, P1, u1, c1 = _side(desc1, cu1, layout, "desc1")
    if P1 != P:
        raise N.LtrError(f"triplet_loss: {P} pairs on side 0 but {P1} on side 1")
    n0 = np.full(P, u0, np.int64) if c0 is None else np.diff(c0).astype(np.int64)
    n1 = np.full(P, u1, np.int64) if c1 is None else np.diff(c1).astype(np.int64)
    mx0, mx1 = int(n0.max(initial=0)), int(n1.max(initial=0))
    if isinstance(assign, LineGroundTruth):
        if assign.assign_flat is None:
            raise N.LtrError("triplet_loss: the LineGroundTruth has no dense assignment (want_assign=False)")
        if not (np.array_equal(assign.n0, n0) and np.array_equal(assign.n1, n1)):
            raise N.LtrError("triplet_loss: the LineGroundTruth's line counts differ from the descriptors'")
        a, stride, ld = assign.assign_flat, int(assign.stride), 0
    else:
        if not isinstance(assign, torch.Tensor) or assign.dim() != 3 or assign.shape[0] != P:
            raise N.LtrError(f"triplet_loss: assign must be a LineGroundTruth or a tensor [{P}, rows, cols]")
        R, Cc = int(assign.shape[1]), int(assign.shape[2])
        ld = int(assign_ld) if assign_ld else Cc
        if R < mx0 or ld < mx1 or ld > Cc:
            raise N.LtrError(f"triplet_loss: assign [{P}, {R}, {Cc}] cannot hold [{mx0}, {mx1}] with row pitch {ld}")
        a, stride = assign, R * Cc
    if not (a.is_cuda and a.dtype == torch.float32) or a.device != d0.device:
        raise N.LtrError(f"triplet_loss: assign must be float32 on {d0.device}")
    a = a.contiguous()
    g = np.array([0, P], np.int32) if groups is None else _offsets(groups, len(np.asarray(groups)) - 1, P, "groups")
    if len(g) < 2:
        raise N.LtrError("triplet_loss: at least one group")
    host = {"groups": g}
    if c0 is not None:
        host.update(cu0=c0, cu1=c1)
    dv = _ops.stage(host, d0.device) if (c0 is not None or groups is not None) else {}
    return dict(d0=d0, d1=d1, P=P, u0=u0, u1=u1, n0=n0, n1=n1, mx0=mx0, mx1=mx1, assign=a, stride=stride, ld=ld, groups=g,
                cu0=dv.get("cu0"), cu1=dv.get("cu1"), group_off=dv.get("groups") if groups is not None else None)


def _run(b, layout, match_thr, unmatch_thr, pred0) -> TripletLoss:
    dev = b["d0"].device
    S = int(b["n0"].sum() + b["n1"].sum())
    G = len(b["groups"]) - 1
    f32, i32 = dict(dtype=torch.float32, device=dev), dict(dtype=torch.int32, device=dev)
    out = dict(pos=torch.empty(S, **f32), neg=torch.empty(S, **f32), state=torch.empty(S, **i32), loss=torch.empty(G, **f32),
               hardest_pos=torch.empty(G, **f32), hardest_neg=torch.empty(G, **f32), n_valid=torch.empty(G, **i32))
    if b["P"] == 0:   # nothing to mine: every group is empty; the kernel's NaN bits, so that results compare bitwise
        for k in ("loss", "hardest_pos", "hardest_neg"):
            out[k].view(torch.int32).fill_(0x7fffffff)
        out["n_valid"].zero_()
    tfpn = None
    if pred0 is not None:
        if not isinstance(pred0, torch.Tensor) or pred0.dim() != 1 or pred0.shape[0] != int(b["n0"].sum()):
            raise N.LtrError(f"triplet_loss: pred0 must be a CUDA tensor [{int(b['n0'].sum())}]")
        pred0 = pred0.to(device=dev, dtype=torch.int32).contiguous()
        tfpn = torch.zeros((b["P"], 4), **i32)
    _ops.call_struct("ltr_triplet_loss",
                     dict(desc0=b["d0"], desc1=b["d1"], layout=layout, d=256, n_pairs=b["P"], n0=b["u0"] or 0,
                          n1=b["u1"] or 0, cu0=b["cu0"], cu1=b["cu1"], max_n0=b["mx0"], max_n1=b["mx1"],
                          assign=b["assign"], assign_stride=b["stride"], assign_ld=b["ld"], match_thr=match_thr,
                          unmatch_thr=unmatch_thr, pred0=pred0, n_groups=G, group_off=b["group_off"]),
                     dict(out, tfpn=tfpn))
    return TripletLoss(tfpn=tfpn, n0=b["n0"], n1=b["n1"], groups=b["groups"], **out)


def triplet_loss(desc0, desc1, assign, cu0=None, cu1=None, layout=N.LAYOUT_ROWS, assign_ld=0, groups=None,
                 match_thr=0.3, unmatch_thr=0.0, pred0=None) -> TripletLoss:
    """The validation loss terms of P pairs in one `ltr_triplet_loss` call.

    desc0 / desc1: float32 CUDA descriptors.  Without offsets: [P, n, 256] (rows, e.g. `PairEngine.encode`) or
    [P, 256, n] (channel-first, the reference's line_desc).  With host offsets cu0 / cu1 [P+1] (side s of pair p =
    lines [cu_s[p], cu_s[p+1])): rows [S, 256] or channel-first [256, n_p] per pair back to back; n0_p != n1_p is
    allowed.  assign: a `LineGroundTruth` (dense, consumed in place) or a float32 CUDA tensor [P, rows, cols] read
    with row pitch assign_ld (0: cols), e.g. the reference's [b, n+1, n+1] with its dustbin.  groups: host pair
    offsets [G+1] (0 .. P) of the groups to reduce separately (one reference batch each); None = one group.
    match_thr / unmatch_thr: see the module docstring (0.3 / 0.3 on a LineGroundTruth reproduces train.py's 0/1
    matrix from lmatches).  pred0: CUDA int [S0] predicted side-1 index (local) or -1: also counts Evaluate_PR's
    TP / FP / FN / TN.  Host offsets go up in one pinned copy; the call never waits for the device."""
    b = _prepare(desc0, desc1, assign, cu0, cu1, layout, assign_ld, groups)
    return _run(b, layout, match_thr, unmatch_thr, pred0)


def validation_metrics(desc0, desc1, assign, cu0=None, cu1=None, layout=N.LAYOUT_ROWS, assign_ld=0, groups=None,
                       match_thr=0.3, unmatch_thr=0.0, nn_thresh=0.7, mutual=True) -> TripletLoss:
    """train.py's run_epochs('val') after the forward: nn_matcher_batches (`ltr_match`, distance mode 1) of the
    descriptors at nn_thresh, then `triplet_loss` with those matches as predictions.  Arguments as `triplet_loss`.
    The result's loss terms are per group, `precision_recall()` gives Result.evaluate's per-pair precision / recall /
    F1 (Evaluate_PR with the match class as ground truth) and `matches0` the predictions."""
    b = _prepare(desc0, desc1, assign, cu0, cu1, layout, assign_ld, groups)
    if b["P"] == 0:
        return _run(b, layout, match_thr, unmatch_thr, None)
    m = _ops.match_descriptors(b["d0"], b["d1"], layout, b["P"], float(nn_thresh), bool(mutual), n0=b["u0"] or 0,
                               n1=b["u1"] or 0, cu0=b["cu0"], cu1=b["cu1"], max_n0=b["mx0"], max_n1=b["mx1"],
                               want_dist=False, dist_mode=1)
    res = _run(b, layout, match_thr, unmatch_thr, m["matches0"])
    res.matches0 = m["matches0"]
    return res


# ------------------------------------------------------------------ drop-in
class descriptor_loss(torch.nn.Module):   # noqa: N801 - the reference's name
    """evaluations/criteria.py descriptor_loss, forward value only, on `ltr_triplet_loss`.

    Inputs as the reference: pred['line_desc0'], pred['line_desc1'] [b, 256, n] and target['mat_assign_sublines']
    float32 [b, n+1, n+1].  Outputs are float32 tensors on the descriptors' device.  Raises LtrError where the reference
    fails (n0 != n1, no anchor with a positive, no valid anchor) and for inputs that require grad: this loss has no
    backward pass."""

    def __init__(self):
        super().__init__()
        self.margin = 0.5

    def _terms(self, pred, target):
        desc0, desc1 = pred["line_desc0"], pred["line_desc1"]
        assign = target["mat_assign_sublines"]
        if any(isinstance(t, torch.Tensor) and t.requires_grad for t in (desc0, desc1, assign)):
            raise N.LtrError("descriptor_loss: inputs require grad, but this loss is forward-only (no backward pass)")
        desc0, desc1, assign = (torch.as_tensor(t) for t in (desc0, desc1, assign))
        if desc0.dim() != 3 or desc1.dim() != 3 or desc0.shape[1] != 256 or desc1.shape[1] != 256:
            raise N.LtrError("descriptor_loss: line_desc0 / line_desc1 must be [b, 256, n]")
        b, _, n0 = desc0.shape
        n1 = desc1.shape[2]
        if n0 != n1:
            raise N.LtrError(f"descriptor_loss: the reference needs as many lines on both sides ({n0} != {n1})")
        if tuple(assign.shape) != (b, n0 + 1, n1 + 1):
            raise N.LtrError(f"descriptor_loss: mat_assign_sublines must be [{b}, {n0 + 1}, {n1 + 1}]")
        home = desc0.device
        dev = home if home.type == "cuda" else _ops.current_cuda_device()
        f = lambda t: t.detach().to(device=dev, dtype=torch.float32).contiguous()
        res = triplet_loss(f(desc0), f(desc1), f(assign), layout=N.LAYOUT_CHANNEL_FIRST, match_thr=MATCH_THR_F32,
                           unmatch_thr=0.0)
        flags = torch.stack([(res.state > 0).any().to(torch.int32), res.n_valid[0]]).cpu()
        if not int(flags[0]):
            raise N.LtrError("descriptor_loss: no anchor has a positive (the reference's amax of an empty tensor)")
        if not int(flags[1]):
            raise N.LtrError("descriptor_loss: no anchor has a negative in the semi-hard window (the reference's "
                             "stack of an empty list)")
        return res, home

    def compute_distances(self, pred, target):
        res, home = self._terms(pred, target)
        valid = res.state == STATE_VALID
        return res.pos[valid].to(home), res.neg[valid].to(home)

    def forward(self, pred, target):
        res, home = self._terms(pred, target)
        return res.loss[0].to(home), res.hardest_pos[0].to(home), res.hardest_neg[0].to(home)
