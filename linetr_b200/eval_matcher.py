"""Training-side matchers of the reference (`evaluations/matcher.py`) on the CUDA library.

Same names, arguments and return values as the reference functions:

    nn_matcher(desc0 [d,n0], desc1 [d,n1], nn_thresh, is_mutual_NN=False) -> mat [n0,n1] float32   (:3-49)
    nn_matcher_batches(desc0 [b,d,n0], desc1 [b,d,n1], nn_thresh, is_mutual_NN=False)
        -> mat [b,n0+1,n1+1] float64 with dustbin row/column                                      (:51-102)
    nn_matcher_score(dist_mat [n0,n1], nn_thresh, is_mutual_NN=False) -> mat [n0,n1] float64      (:104-152)

The distance is ||a||^2 + ||b||^2 - 2 ab (no unit-norm assumption), clipped at 0 - `ltr_match` with
dist_mode = 1: the tensor-core contraction of match_tc.cuh with the norms added in its epilogue and
the same exact re-check tail as the inference matcher.  The batched variant is ONE launch sequence
for all b pairs (the reference loops over b in Python).  Host numpy in / host numpy out like the
reference; only the dense 0/1 (+ dustbin) matrices the API promises are assembled on the host.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _native as N
from . import _ops


def _match_batch(desc0, desc1, nn_thresh, mutual):
    desc0 = np.ascontiguousarray(desc0, dtype=np.float32)
    desc1 = np.ascontiguousarray(desc1, dtype=np.float32)
    b, d, n0 = desc0.shape
    n1 = desc1.shape[2]
    if d != 256:
        raise N.LtrError("linetr_b200.eval_matcher: descriptor dimension must be 256")
    if b == 0 or n0 == 0 or n1 == 0:
        return np.full((b, n0), -1, dtype=np.int32)
    dev = _ops.current_cuda_device()
    a = torch.from_numpy(desc0).to(dev, non_blocking=True)
    c = torch.from_numpy(desc1).to(dev, non_blocking=True)
    out = _ops.match_descriptors(a, c, N.LAYOUT_CHANNEL_FIRST, b, float(nn_thresh), bool(mutual), n0=n0, n1=n1, d=d,
                                 want_dist=False, dist_mode=1)
    return out["matches0"].view(b, n0).cpu().numpy()


def nn_matcher(desc0, desc1, nn_thresh, is_mutual_NN=False):
    d, n0 = desc0.shape
    n1 = desc1.shape[1]
    idx = _match_batch(np.asarray(desc0)[None], np.asarray(desc1)[None], nn_thresh, is_mutual_NN)[0]
    mat = np.zeros((n0, n1), dtype=np.result_type(np.asarray(desc0).dtype, np.float32))
    rows = np.nonzero(idx >= 0)[0]
    mat[rows, idx[rows]] = 1
    return mat


def nn_matcher_batches(desc0, desc1, nn_thresh, is_mutual_NN=False):
    b, d, n0 = desc0.shape
    n1 = desc1.shape[2]
    idx = _match_batch(desc0, desc1, nn_thresh, is_mutual_NN)
    mat = np.zeros((b, n0 + 1, n1 + 1))
    for i in range(b):
        rows = np.nonzero(idx[i] >= 0)[0]
        mat[i, rows, idx[i][rows]] = 1
        un0 = np.ones(n0 + 1, dtype=bool)
        un0[rows] = False                     # unmatched lines of image 0 (+ the dustbin row itself, :96-100)
        un1 = np.ones(n1 + 1, dtype=bool)
        un1[idx[i][rows]] = False
        mat[i, un0, -1] = 1
        mat[i, -1, un1] = 1
        mat[i, -1, -1] = 1
    return mat


def nn_matcher_score(dist_mat, nn_thresh, is_mutual_NN=False):
    dist_mat = np.asarray(dist_mat)
    n0, n1 = dist_mat.shape
    mat = np.zeros((n0, n1))
    if n0 == 0 or n1 == 0:
        return mat
    dev = _ops.current_cuda_device()
    out = _ops.match_distmat(torch.from_numpy(np.ascontiguousarray(dist_mat[None], dtype=np.float32)).to(dev),
                             float(nn_thresh), bool(is_mutual_NN))
    idx = out["matches0"][0].cpu().numpy()
    rows = np.nonzero(idx >= 0)[0]
    mat[rows, idx[rows]] = 1
    return mat
