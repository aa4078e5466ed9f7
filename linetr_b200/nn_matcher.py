"""Drop-in `nn_matcher` / `nn_matcher_distmat` (reference models/nn_matcher.py:3-43) and the
`subline2keyline` merge (reference models/line_transformer.py:277-282) on the CUDA library.

Same signatures, host numpy in / host numpy out, dense float64 0/1 match matrix [1,n0,n1] as
the reference returns it.  The arithmetic (distance GEMM, clip, argmin, threshold, mutual
check, segment means) runs in liblinetr_b200.so; the host only scatters the int32 match
indices into the dense matrix the reference API promises.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _native as N
from . import _ops


def _device():
    return _ops.current_cuda_device()


def _dense(matches0: np.ndarray, n0: int, n1: int) -> np.ndarray:
    mat = np.zeros((1, n0, n1))
    rows = np.nonzero(matches0 >= 0)[0]
    mat[0, rows, matches0[rows]] = 1
    return mat


def nn_matcher_distmat(dist_mat, nn_thresh, is_mutual_NN=True):
    """Nearest-neighbour matching on a distance matrix [1,n0,n1] (only batch 0 is matched, as in
    the reference where b = 1 is hard-coded, nn_matcher.py:7)."""
    n0, n1 = dist_mat.shape[1], dist_mat.shape[2]
    if n0 == 0 or n1 == 0:
        return np.zeros((1, n0, n1))
    d = torch.from_numpy(np.ascontiguousarray(dist_mat[0:1], dtype=np.float32)).to(_device())
    out = _ops.match_distmat(d, float(nn_thresh), bool(is_mutual_NN))
    return _dense(out["matches0"][0].cpu().numpy(), n0, n1)


def nn_matcher(desc0, desc1, nn_thresh=0.8, is_mutual_NN=True):
    """Nearest-neighbour matching of two descriptor sets [d,n0], [d,n1] -> (mat f64 [1,n0,n1],
    dist f32 [1,n0,n1])."""
    d, n0 = desc0.shape
    n1 = desc1.shape[1]
    if n0 == 0 or n1 == 0:
        return np.zeros((1, n0, n1)), np.zeros((1, n0, n1), dtype=np.float32)
    dev = _device()
    a = torch.from_numpy(np.ascontiguousarray(desc0, dtype=np.float32)).to(dev)
    b = torch.from_numpy(np.ascontiguousarray(desc1, dtype=np.float32)).to(dev)
    out = _ops.match_descriptors(a, b, N.LAYOUT_CHANNEL_FIRST, 1, float(nn_thresh), bool(is_mutual_NN),
                                 n0=n0, n1=n1, d=d)
    dist = out["dist_key"].view(1, n0, n1).cpu().numpy()
    return _dense(out["matches0"].cpu().numpy(), n0, n1), dist


def adjacency_to_csr(A: np.ndarray) -> np.ndarray:
    """Key-line -> subline adjacency [K,S] (rows 1/n_sub over contiguous sublines, reference
    models/line_process.py:163-167) -> CSR offsets int32 [K+1].  Raises if A is not of that form."""
    A = np.asarray(A)
    K, S = A.shape
    nz = A != 0
    cnt = nz.sum(axis=1)
    off = np.zeros(K + 1, dtype=np.int64)
    off[1:] = np.cumsum(cnt)
    ok = off[-1] == S and bool((cnt > 0).all())
    if ok:
        expect = np.zeros_like(A, dtype=np.float32)
        for k in range(K):
            expect[k, off[k]:off[k + 1]] = np.float32(1.0 / cnt[k])
        ok = np.array_equal(expect, A.astype(np.float32))
    if not ok:
        raise N.LtrError("subline2keyline: adjacency is not the tokenizer's block form (1/n_sub over "
                         "contiguous sublines)")
    return off.astype(np.int32)


def subline2keyline(distance_sublines, mat_klines2sublines0, mat_klines2sublines1):
    """A0 @ D @ A1^T for block-constant adjacencies -> np.float32 [1,K0,K1]."""
    to_np = lambda t: t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
    A0, A1 = to_np(mat_klines2sublines0), to_np(mat_klines2sublines1)
    D = np.ascontiguousarray(distance_sublines, dtype=np.float32)
    K0, K1 = A0.shape[0], A1.shape[0]
    if K0 == 0 or K1 == 0:
        return np.zeros((1, K0, K1), dtype=np.float32)
    off0, off1 = adjacency_to_csr(A0), adjacency_to_csr(A1)
    if off0[-1] == K0 and off1[-1] == K1:
        return D[None].copy()           # A0 = A1 = I: nothing to merge
    from . import engine
    dev = _device()
    out = engine.merge_sublines(torch.from_numpy(D).to(dev), torch.from_numpy(off0).to(dev),
                                torch.from_numpy(off1).to(dev), K0, K1)
    return out.cpu().numpy()[None]
