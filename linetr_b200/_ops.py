"""Device-level wrappers around the C ABI: CUDA torch tensors in, CUDA torch tensors out.

PyTorch is used here only for device memory, streams and dtype plumbing; all arithmetic
happens inside liblinetr_b200.so.  Every function raises if the tensors are not on a CUDA
device (no CPU fallback).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _native as N


def _stream_ptr(device) -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _req_cuda(t: torch.Tensor, name: str):
    if not t.is_cuda:
        raise N.LtrError(f"linetr_b200: '{name}' is on {t.device}; the CUDA path needs CUDA tensors "
                         "(there is no CPU fallback)")


def current_cuda_device() -> torch.device:
    """Device the host-numpy entry points (nn_matcher*, get_dist_matrix) compute on."""
    if not torch.cuda.is_available():
        raise N.LtrError("linetr_b200 needs a CUDA device (there is no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


def _f32c(t: torch.Tensor) -> torch.Tensor:
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def _i32c(t: torch.Tensor) -> torch.Tensor:
    if t.dtype != torch.int32:
        t = t.to(torch.int32)
    return t.contiguous()


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _call(entry: str, dev, *args):
    """C-ABI entry point `entry`(*args, device, stream) on the current stream of `dev`; raises on a non-zero return
    code."""
    with torch.cuda.device(dev):
        rc = getattr(N.load(), entry)(*args, dev.index, _stream_ptr(dev))
    N.check(rc, entry)


def _check_tensors(who: str, dev, specs):
    """Raises unless every tensor of `specs`, (name, tensor or None, dtype[, shape]), is None or a contiguous tensor
    of that dtype (and shape) on `dev`."""
    for nm, t, dt, *shape in specs:
        shape = shape[0] if shape else None
        if t is None:
            continue
        if t.dtype != dt or not t.is_contiguous() or t.device != dev or (shape is not None and tuple(t.shape) != shape):
            raise N.LtrError(f"{who}: '{nm}' must be a contiguous {dt} tensor on {dev}"
                             + (f" of shape {list(shape)}" if shape is not None else ""))


_staging = []   # (pinned host buffer, event behind its copy) until the copy has finished
_TORCH_DTYPE = {np.dtype(np.float64): torch.float64, np.dtype(np.float32): torch.float32,
                np.dtype(np.int32): torch.int32, np.dtype(np.uint8): torch.uint8}


def stage(arrays: dict, device) -> dict:
    """One pinned staging buffer, one non-blocking H2D copy on the current stream of `device`: -> device views of the
    host arrays (float64, float32, int32 or uint8).  The buffer is held (with an event behind the copy) until the copy has
    finished, so it is never reused early."""
    global _staging
    _staging = [(b, e) for b, e in _staging if not e.query()]
    layout, total = {}, 0
    for k, a in arrays.items():
        a = np.ascontiguousarray(a)
        total = (total + 15) // 16 * 16
        layout[k] = (total, a)
        total += a.nbytes
    host = torch.empty(max(total, 16), dtype=torch.uint8, pin_memory=True)
    hv = host.numpy()
    for o, a in layout.values():
        hv[o:o + a.nbytes] = a.reshape(-1).view(np.uint8)
    dev = host.to(device, non_blocking=True)
    ev = torch.cuda.Event()
    ev.record(torch.cuda.current_stream(device))
    _staging.append((host, ev))
    return {k: dev[o:o + a.nbytes].view(_TORCH_DTYPE[a.dtype]).view(a.shape) for k, (o, a) in layout.items()}


class ModelHandle:
    """Owns one LtrModel* (packed weights on one GPU)."""

    def __init__(self, state_dict: dict, device_index: int, d_model=256, n_heads=4, d_inner=1024,
                 n_desc_layers=1, n_sig_layers=7):
        lib = N.load()
        keep = []
        arr = (N.LtrTensor * len(state_dict))()
        i = 0
        for k, v in state_dict.items():
            a = np.ascontiguousarray(np.asarray(v), dtype=np.float32)
            keep.append(a)
            arr[i].name = k.encode()
            arr[i].data = a.ctypes.data
            arr[i].numel = a.size
            i += 1
        cfg = N.LtrConfig(d_model, n_heads, d_inner, n_desc_layers, n_sig_layers)
        h = C.c_void_p()
        N.check(lib.ltr_create(arr, len(state_dict), C.byref(cfg), int(device_index), C.byref(h)), "ltr_create")
        self._lib = lib
        self.ptr = h
        self.device_index = int(device_index)
        self._ws = {}   # one workspace per CUDA stream: calls on one stream are ordered, streams may overlap

    def close(self):
        if getattr(self, "ptr", None):
            self._lib.ltr_destroy(self.ptr)
            self.ptr = None

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    def workspace(self, n_images: int, n_lines: int, n_tokens: int) -> torch.Tensor:
        need = int(self._lib.ltr_encode_workspace_bytes(self.ptr, n_images, n_lines, n_tokens))
        if need < 0:
            N.check(need, "ltr_encode_workspace_bytes")
        dev = torch.device("cuda", self.device_index)
        key = torch.cuda.current_stream(dev).cuda_stream
        ws = self._ws.get(key)
        if ws is None or ws.numel() < need:
            if len(self._ws) >= 16:   # callers that keep creating streams: do not hoard one workspace per dead stream
                self._ws.clear()
            ws = self._ws[key] = torch.empty(need, dtype=torch.uint8, device=dev)
        return ws


def encode(handle: ModelHandle, sublines, resp, angle, pnt, desc, score, image_wh, *, lines_per_image=None,
           cu_lines_host=None, cu_lines_dev=None, want_cf=True, want_rows=False, want_tiles=False):
    """ltr_encode on flattened lines.

    sublines [R,2,2], resp [R,1], angle [R,2], pnt [R,T,2], desc [R,T,256], score [R,T,1]; either
    `lines_per_image` (uniform batch) or `cu_lines_host` (np.int32 [B+1]) + `cu_lines_dev`.
    Returns (desc_cf flat [256*R] or None, desc_rows [R,256] or None), plus the descriptor tile image
    (uint8 tensor, the matcher's operand format) as a third element when `want_tiles`.
    """
    for nm, t in (("sublines", sublines), ("resp_sublines", resp), ("angle_sublines", angle),
                  ("pnt_sublines", pnt), ("desc_sublines", desc), ("score_sublines", score)):
        _req_cuda(t, nm)
    dev = desc.device
    if dev.index != handle.device_index:
        raise N.LtrError(f"linetr_b200: inputs on cuda:{dev.index} but weights on cuda:{handle.device_index}")
    sublines, resp, angle, pnt, desc, score = map(_f32c, (sublines, resp, angle, pnt, desc, score))
    R, T = int(desc.shape[0]), int(desc.shape[1])
    if desc.shape[2] != 256:
        raise N.LtrError("linetr_b200: descriptor_dim must be 256")
    if cu_lines_host is not None:
        cu_lines_host = np.ascontiguousarray(cu_lines_host, dtype=np.int32)
        n_images = len(cu_lines_host) - 1
        cu_lines_dev = _i32c(cu_lines_dev)
        lpi = 0
    else:
        lpi = int(lines_per_image)
        n_images = R // lpi if lpi > 0 else 0
    out_cf = torch.empty(R * 256, dtype=torch.float32, device=dev) if want_cf else None
    out_rows = torch.empty((R, 256), dtype=torch.float32, device=dev) if want_rows else None
    out_tiles = None
    if want_tiles:
        if want_cf or not want_rows:
            raise N.LtrError("encode: want_tiles needs want_rows=True and want_cf=False")
        out_tiles = torch.empty(max(int(handle._lib.ltr_desc_tiles_bytes(R)), 1), dtype=torch.uint8, device=dev)
    if R == 0 or n_images == 0:
        return (out_cf, out_rows, out_tiles) if want_tiles else (out_cf, out_rows)
    ws = handle.workspace(n_images, R, T)
    inp = N.LtrEncodeInput(
        sublines.data_ptr(), resp.data_ptr(), angle.data_ptr(), pnt.data_ptr(), desc.data_ptr(), score.data_ptr(),
        cu_lines_host.ctypes.data if cu_lines_host is not None else None,
        cu_lines_dev.data_ptr() if cu_lines_host is not None else None,
        n_images, R, T, lpi, float(image_wh[0]), float(image_wh[1]))
    outp = N.LtrEncodeOutput(out_cf.data_ptr() if out_cf is not None else None,
                             out_rows.data_ptr() if out_rows is not None else None,
                             out_tiles.data_ptr() if out_tiles is not None else None)
    with torch.cuda.device(dev):   # ltr_encode takes no device argument, so it does not go through _call
        rc = handle._lib.ltr_encode(handle.ptr, C.byref(inp), C.byref(outp), _ptr(ws), ws.numel(), _stream_ptr(dev))
    N.check(rc, "ltr_encode")
    return (out_cf, out_rows, out_tiles) if want_tiles else (out_cf, out_rows)


_match_ws = {}   # (device index, stream) -> uint8 scratch tensor, grown on demand


def _match_workspace(dev, need: int) -> torch.Tensor:
    key = (dev.index, torch.cuda.current_stream(dev).cuda_stream)
    ws = _match_ws.get(key)
    if ws is None or ws.numel() < need:
        if len(_match_ws) >= 16:
            _match_ws.clear()
        ws = _match_ws[key] = torch.empty(max(need, 1), dtype=torch.uint8, device=dev)
    return ws


def _struct(cls, **fields):
    """A ctypes struct by field name: tensors go in as device pointers, None and fields not given as NULL / 0.  The
    caller keeps the tensors alive until the call."""
    return cls(**{k: v.data_ptr() if isinstance(v, torch.Tensor) else v for k, v in fields.items() if v is not None})


def _match(entry: str, dev, inp: dict, out: dict, idx=None, gather=None):
    """One matcher call on the current stream of `dev`: `entry` is ltr_match, or ltr_match_indexed with the pair index
    `idx`.  LtrMatchInput fields in `inp`, LtrPairIndex fields in `idx` and output tensors in `out`, all by field name;
    the scratch is the per-stream workspace, grown to what `entry`_workspace_bytes asks for."""
    lib = N.load()
    args = [C.byref(_struct(N.LtrMatchInput, **inp))]
    if idx is not None:
        args.append(C.byref(_struct(N.LtrPairIndex, **idx)))
    need = int(getattr(lib, entry + "_workspace_bytes")(*args))
    if need < 0:
        N.check(need, entry + "_workspace_bytes")
    ws = _match_workspace(dev, need)
    o = _struct(N.LtrMatchOutput, workspace=ws, workspace_bytes=ws.numel(),
                gather=C.pointer(gather) if gather is not None else None, **out)
    _call(entry, dev, *args, C.byref(o))


def match_descriptors(desc0, desc1, layout, n_pairs, nn_thresh, mutual=True, *, n0=0, n1=0, cu0=None, cu1=None,
                      max_n0=0, max_n1=0, sub_off0=None, sub_off1=None, cuk0=None, cuk1=None, max_k0=0, max_k1=0,
                      total_k0=None, total_k1=None, d=256, want_dist=True, want_matches=True, dist_mode=0,
                      tiles0=None, tiles1=None, tiles_lines=(0, 0), tiles_row0=(0, 0), gather=None):
    """ltr_match.  Returns dict(matches0, scores0, nn1, counts, dist_key, stride).

    want_dist=False (no key-line merging, d == 256) never materialises the distance matrix: the row
    argmin lives in the epilogue of the tensor-core contraction.  want_matches=False computes the
    distance matrices only (get_dist_matrix).  tiles0/tiles1: descriptor tile images from
    `encode(want_tiles=True)` (uniform batches with n % 128 == 0).  gather: an `N.LtrPeerGather` - the tail
    kernel then also publishes the per-pair counts to every rank (engine.PeerCounts)."""
    _req_cuda(desc0, "desc0")
    _req_cuda(desc1, "desc1")
    dev = desc0.device
    desc0, desc1 = _f32c(desc0), _f32c(desc1)
    seg = sub_off0 is not None
    varlen = cu0 is not None
    mx0 = max_n0 if varlen else n0
    mx1 = max_n1 if varlen else n1
    mk0, mk1 = (max_k0, max_k1) if seg else (mx0, mx1)
    total_n0 = int(desc0.numel() // d) if varlen else n_pairs * n0
    total_n1 = int(desc1.numel() // d) if varlen else n_pairs * n1
    if total_k0 is None:
        total_k0, total_k1 = total_n0, total_n1
    if seg or d != 256:
        want_dist = True
    stride = mk0 * mk1
    i32 = dict(dtype=torch.int32, device=dev)
    f32 = dict(dtype=torch.float32, device=dev)
    out = {"stride": stride}
    if want_matches:
        out["matches0"] = torch.empty(max(total_k0, 1), **i32)[:total_k0]
        out["scores0"] = torch.empty(max(total_k0, 1), **f32)[:total_k0]
        out["nn1"] = torch.empty(max(total_k1, 1), **i32)[:total_k1]
        out["counts"] = (torch.zeros if n_pairs == 0 else torch.empty)(max(n_pairs, 1), **i32)[:n_pairs]   # zeroed by the kernels
    out["dist_key"] = torch.empty(max(n_pairs * stride, 1), **f32)[:n_pairs * stride] if want_dist else None
    if n_pairs == 0:
        return out
    dist_sub = torch.empty(max(n_pairs * mx0 * mx1, 1), **f32) if seg else None
    cu0, cu1, sub_off0, sub_off1, cuk0, cuk1 = (_i32c(t) if t is not None else None
                                                for t in (cu0, cu1, sub_off0, sub_off1, cuk0, cuk1))
    _match("ltr_match", dev,
           dict(desc0=desc0, desc1=desc1, layout=layout, d=d, n_pairs=n_pairs, n0=n0, n1=n1, cu0=cu0, cu1=cu1,
                sub_off0=sub_off0, sub_off1=sub_off1, cuk0=cuk0, cuk1=cuk1, max_n0=max_n0, max_n1=max_n1, max_k0=max_k0,
                max_k1=max_k1, nn_thresh=nn_thresh, mutual=bool(mutual), total_n0=total_n0, total_n1=total_n1,
                dist_mode=dist_mode, tiles0=tiles0, tiles1=tiles1, tiles_lines0=tiles_lines[0],
                tiles_lines1=tiles_lines[1], tiles_row0_0=tiles_row0[0], tiles_row0_1=tiles_row0[1]),
           dict(matches0=out.get("matches0"), scores0=out.get("scores0"), nn1=out.get("nn1"), counts=out.get("counts"),
                dist_key=out["dist_key"], dist_sub=dist_sub),
           gather=gather)
    return out


def tile_offsets(cu: np.ndarray) -> np.ndarray:
    """First 128-row tile of every image in an image-aligned tile image: prefix sum of ceil(L_i / 128), int32 [n+1]."""
    n = np.diff(np.asarray(cu, dtype=np.int64))
    t = np.zeros(len(n) + 1, dtype=np.int64)
    t[1:] = np.cumsum((n + 127) // 128)
    return t.astype(np.int32)


def image_tiles(desc: torch.Tensor, layout: int, cu_host: np.ndarray, cu_dev: torch.Tensor, tile_off_dev: torch.Tensor,
                n_tiles: int) -> torch.Tensor:
    """ltr_image_tiles: the image-aligned tile image (uint8 tensor, the matcher's operand format) of a pool of
    images' descriptors, rows [R, 256] or channel-first [256, L_i] per image back to back."""
    _req_cuda(desc, "desc")
    dev = desc.device
    desc = _f32c(desc)
    cu_host = np.ascontiguousarray(cu_host, dtype=np.int32)
    n = len(cu_host) - 1
    lib = N.load()
    nbytes = int(lib.ltr_image_tiles_bytes(n, cu_host.ctypes.data_as(N.c_int32_p)))
    if nbytes < 0:
        N.check(nbytes, "ltr_image_tiles_bytes")
    out = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dev)
    _call("ltr_image_tiles", dev, _ptr(desc), int(layout), _ptr(cu_dev), _ptr(tile_off_dev), n,
          int(np.diff(cu_host).max(initial=0)), int(n_tiles), _ptr(out))
    return out


def match_indexed(desc0, desc1, layout, n_pairs, nn_thresh, *, cu0, cu1, max_n0, max_n1, img0, img1, tiles0, tiles1,
                  tile_off0, tile_off1, n_tiles0, n_tiles1, out_off0, out_off1, total_out0, total_out1,
                  matches0, scores0, nn1, counts, sub_off0=None, sub_off1=None, cuk0=None, cuk1=None, max_k0=0, max_k1=0,
                  dist_key=None, dist_stride=0, mutual=True):
    """ltr_match_indexed: P pairs over two image pools (pair p = image img0[p] of pool 0 against image img1[p] of
    pool 1) into caller-allocated outputs (matches0 / scores0 at out_off0[p] + k, nn1 at out_off1[p] + j,
    counts[p], dist_key at p * dist_stride when given).  Key-line merging when sub_off0 is given; its distance
    scratch (n_pairs * max_n0 * max_n1 floats) is allocated here."""
    _req_cuda(desc0, "desc0")
    _req_cuda(desc1, "desc1")
    dev = desc0.device
    desc0, desc1 = _f32c(desc0), _f32c(desc1)
    seg = sub_off0 is not None
    f32 = dict(dtype=torch.float32, device=dev)
    if seg and dist_key is None:
        dist_stride = max_k0 * max_k1
        dist_key = torch.empty(max(n_pairs * dist_stride, 1), **f32)
    dist_sub = torch.empty(max(n_pairs * max_n0 * max_n1, 1), **f32) if seg else None
    _match("ltr_match_indexed", dev,
           dict(desc0=desc0, desc1=desc1, layout=layout, d=256, n_pairs=n_pairs, cu0=cu0, cu1=cu1, sub_off0=sub_off0,
                sub_off1=sub_off1, cuk0=cuk0, cuk1=cuk1, max_n0=max_n0, max_n1=max_n1, max_k0=max_k0, max_k1=max_k1,
                dist_pair_stride=dist_stride, nn_thresh=nn_thresh, mutual=bool(mutual), total_n0=desc0.numel() // 256,
                total_n1=desc1.numel() // 256),
           dict(matches0=matches0, scores0=scores0, nn1=nn1, counts=counts, dist_key=dist_key, dist_sub=dist_sub),
           idx=dict(img0=img0, img1=img1, tiles0=tiles0, tiles1=tiles1, tile_off0=tile_off0, tile_off1=tile_off1,
                    n_tiles0=n_tiles0, n_tiles1=n_tiles1, out_off0=out_off0, out_off1=out_off1, total_out0=total_out0,
                    total_out1=total_out1))


def tokenize(dv: dict, maps, cu_lines: np.ndarray, max_tokens: int, dev) -> list:
    """ltr_tokenize_batch of the key lines staged in `dv` (device arrays sp, ep, epc, length, angle, n_tok, sub0,
    sub2line, line_image of `line_process.keyline_geometry`, image by image) -> sublines [S,2,2], pnt [S,T,2],
    mask [S,T+1,1], resp [S,1], angle [S,2], desc [S,T,256], score [S,T,1].  maps: per image (dense descriptor
    map, dense score map, token_distance), or None for an image without key lines; cu_lines [n+1]: host subline
    offsets."""
    S, T, n = int(cu_lines[-1]), int(max_tokens), len(maps)
    f32 = dict(dtype=torch.float32, device=dev)
    out = [torch.empty(shape, **f32) for shape in ((S, 2, 2), (S, T, 2), (S, T + 1, 1), (S, 1), (S, 2), (S, T, 256), (S, T, 1))]
    keep, tab = [], (N.LtrTokenizeImage * max(n, 1))()
    for i, m in enumerate(maps):
        if m is None:
            continue
        dense, smap = m[0].float().contiguous(), m[1].float().contiguous()
        if dense.shape[-3] != 256:
            raise N.LtrError(f"ltr_tokenize_batch: image {i} has {dense.shape[-3]} descriptor channels, 256 required")
        keep += [dense, smap]
        tab[i] = N.LtrTokenizeImage(dense.data_ptr(), smap.data_ptr(), float(m[2]), dense.shape[-2], dense.shape[-1],
                                    smap.shape[-2], smap.shape[-1])
    cu = np.ascontiguousarray(cu_lines, dtype=np.int32)
    ptr = lambda k: dv[k].data_ptr()   # noqa: E731
    # the reference keys grid_sample's align_corners on the third character of torch.__version__ (line_process.py:93)
    align = 1 if int(torch.__version__[2]) > 2 else 0
    inp = N.LtrTokenizeBatchInput(ptr("sp"), ptr("ep"), ptr("epc"), ptr("length"), ptr("angle"), ptr("n_tok"),
                                  ptr("sub0"), ptr("sub2line"), ptr("line_image"), n, len(dv["n_tok"]), S, T, 256, align,
                                  tab, cu.ctypes.data_as(N.c_int32_p))
    _call("ltr_tokenize_batch", dev, C.byref(inp), *[_ptr(t) for t in out])
    return out


def line_gt(segs0, segs1, n_pairs, *, cu0, cu1, max_n0, max_n1, homography, homography_inv, n_gt, assign=None,
            assign_stride=0, pred0=None, tfpn=None, proj0=None, proj1=None, thres_reprojected=3.0, thres_angdiff=2.0,
            min_overlap_ratio=0.3):
    """ltr_line_gt into caller-allocated outputs: homography ground truth of P line-segment pairs (segs [S,2,2] fp32,
    side s of pair p = [cu_s[p], cu_s[p+1]), homography [P,3,3] fp64 image 0 -> 1 and its inverse), n_gt [P] int32,
    optionally the dense assignment (pair p at p * assign_stride, row-major [n0_p, n1_p]) and, with pred0 (int32 [S0]
    local side-1 index or -1), tfpn [P,4] int32 (TP, FP, FN, TN)."""
    _req_cuda(segs0, "segs0")
    _req_cuda(segs1, "segs1")
    dev = segs0.device
    specs = (("segs0", segs0, torch.float32), ("segs1", segs1, torch.float32), ("cu0", cu0, torch.int32),
             ("cu1", cu1, torch.int32), ("homography", homography, torch.float64),
             ("homography_inv", homography_inv, torch.float64), ("n_gt", n_gt, torch.int32),
             ("assign", assign, torch.float32), ("pred0", pred0, torch.int32), ("tfpn", tfpn, torch.int32),
             ("proj0", proj0, torch.float32), ("proj1", proj1, torch.float32))
    for nm, t, _ in specs:
        if t is not None:
            _req_cuda(t, nm)
    _check_tensors("line_gt", dev, specs)
    inp = _struct(N.LtrLineGtInput, segs0=segs0, segs1=segs1, cu0=cu0, cu1=cu1, homography=homography,
                  homography_inv=homography_inv, proj0=proj0, proj1=proj1, pred0=pred0, n_pairs=int(n_pairs),
                  max_n0=int(max_n0), max_n1=int(max_n1), thres_reprojected=float(thres_reprojected),
                  thres_angdiff=float(thres_angdiff), min_overlap_ratio=float(min_overlap_ratio))
    out = _struct(N.LtrLineGtOutput, assign=assign, assign_stride=int(assign_stride), n_gt=n_gt, tfpn=tfpn)
    _call("ltr_line_gt", dev, C.byref(inp), C.byref(out))


def triplet_loss(desc0, desc1, layout, n_pairs, *, assign, assign_stride, pos, neg, state, loss, hardest_pos,
                 hardest_neg, n_valid, n0=0, n1=0, cu0=None, cu1=None, max_n0=0, max_n1=0, assign_ld=0, match_thr=0.3,
                 unmatch_thr=0.0, pred0=None, tfpn=None, n_groups=1, group_off=None):
    """ltr_triplet_loss into caller-allocated outputs: per anchor pos / neg (fp32) and state (int32) [S0 + S1], per
    group loss / hardest_pos / hardest_neg (fp32) and n_valid (int32), tfpn [P, 4] int32 with pred0."""
    _req_cuda(desc0, "desc0")
    _req_cuda(desc1, "desc1")
    dev = desc0.device
    _check_tensors("triplet_loss", dev, (
        ("desc0", desc0, torch.float32), ("desc1", desc1, torch.float32), ("assign", assign, torch.float32),
        ("cu0", cu0, torch.int32), ("cu1", cu1, torch.int32), ("pred0", pred0, torch.int32),
        ("group_off", group_off, torch.int32), ("pos", pos, torch.float32), ("neg", neg, torch.float32),
        ("state", state, torch.int32), ("loss", loss, torch.float32), ("hardest_pos", hardest_pos, torch.float32),
        ("hardest_neg", hardest_neg, torch.float32), ("n_valid", n_valid, torch.int32), ("tfpn", tfpn, torch.int32)))
    inp = _struct(N.LtrTripletInput, desc0=desc0, desc1=desc1, layout=int(layout), d=256, n_pairs=int(n_pairs), n0=int(n0),
                  n1=int(n1), cu0=cu0, cu1=cu1, max_n0=int(max_n0), max_n1=int(max_n1), assign=assign,
                  assign_stride=int(assign_stride), assign_ld=int(assign_ld), match_thr=float(match_thr),
                  unmatch_thr=float(unmatch_thr), pred0=pred0, n_groups=int(n_groups), group_off=group_off)
    out = _struct(N.LtrTripletOutput, pos=pos, neg=neg, state=state, loss=loss, hardest_pos=hardest_pos,
                  hardest_neg=hardest_neg, n_valid=n_valid, tfpn=tfpn)
    _call("ltr_triplet_loss", dev, C.byref(inp), C.byref(out))


def homography(n_pairs, *, pts0, pts1, pts_off0, pts_off1, n_pts1, matches_p, cu_p, max_rows_p, segs0, segs1, seg_off0,
               seg_off1, n_segs1, matches_l, cu_l, max_rows_l, H, valid, inliers_p, inliers_l, n_inliers_p, n_inliers_l,
               hypothesis, hypothesis_inliers, key, thresh=3.0, n_hypotheses=2048, seed=0, use_points=True,
               use_lines=True):
    """ltr_homography into caller-allocated outputs: keypoint pools [*,2] / segment pools [*,2,2] fp32, per-pair pool
    offsets and side-1 counts int32 [P], match rows int32 with offsets cu_p / cu_l [P+1]; H [P,3,3] fp64, valid [P]
    uint8, inliers_p / inliers_l uint8 aligned with the match rows, counts / hypothesis int32 [P], key [P] int64
    workspace."""
    _req_cuda(H, "H")
    dev = H.device
    _check_tensors("homography", dev, (
        ("pts0", pts0, torch.float32), ("pts1", pts1, torch.float32), ("pts_off0", pts_off0, torch.int32),
        ("pts_off1", pts_off1, torch.int32), ("n_pts1", n_pts1, torch.int32), ("matches_p", matches_p, torch.int32),
        ("cu_p", cu_p, torch.int32), ("segs0", segs0, torch.float32), ("segs1", segs1, torch.float32),
        ("seg_off0", seg_off0, torch.int32), ("seg_off1", seg_off1, torch.int32), ("n_segs1", n_segs1, torch.int32),
        ("matches_l", matches_l, torch.int32), ("cu_l", cu_l, torch.int32), ("H", H, torch.float64),
        ("valid", valid, torch.uint8), ("inliers_p", inliers_p, torch.uint8), ("inliers_l", inliers_l, torch.uint8),
        ("n_inliers_p", n_inliers_p, torch.int32), ("n_inliers_l", n_inliers_l, torch.int32),
        ("hypothesis", hypothesis, torch.int32), ("hypothesis_inliers", hypothesis_inliers, torch.int32),
        ("key", key, torch.int64)))
    inp = _struct(N.LtrHomographyInput, pts0=pts0, pts1=pts1, pts_off0=pts_off0, pts_off1=pts_off1, n_pts1=n_pts1,
                  matches_p=matches_p, cu_p=cu_p, segs0=segs0, segs1=segs1, seg_off0=seg_off0, seg_off1=seg_off1,
                  n_segs1=n_segs1, matches_l=matches_l, cu_l=cu_l, n_pairs=int(n_pairs), max_rows_p=int(max_rows_p),
                  max_rows_l=int(max_rows_l), thresh=float(thresh), n_hypotheses=int(n_hypotheses),
                  seed=int(seed) & 0xFFFFFFFFFFFFFFFF, use_points=int(bool(use_points)), use_lines=int(bool(use_lines)))
    out = _struct(N.LtrHomographyOutput, H=H, valid=valid, inliers_p=inliers_p, inliers_l=inliers_l,
                  n_inliers_p=n_inliers_p, n_inliers_l=n_inliers_l, hypothesis=hypothesis,
                  hypothesis_inliers=hypothesis_inliers, key=key)
    _call("ltr_homography", dev, C.byref(inp), C.byref(out))


def essential(n_pairs, *, pts0, pts1, pts_off0, pts_off1, n_pts1, matches_p, cu_p, max_rows_p, K0, K1, E, R, t, valid,
              inliers_p, n_inliers, n_cheirality, hypothesis, hypothesis_inliers, key, thresh=1.0, dist_thresh=1e9,
              n_hypotheses=1024, seed=0):
    """ltr_essential into caller-allocated outputs: keypoint pools [*,2] fp32, per-pair pool offsets and side-1 counts
    int32 [P], match rows int32 with offsets cu_p [P+1], intrinsics K0 / K1 fp64 [P,3,3]; E / R [P,3,3] and t [P,3]
    fp64, valid [P] uint8, inliers_p uint8 aligned with the match rows, counts / hypothesis int32 [P], key [P] int64
    workspace."""
    _req_cuda(E, "E")
    dev = E.device
    _check_tensors("essential", dev, (
        ("pts0", pts0, torch.float32), ("pts1", pts1, torch.float32), ("pts_off0", pts_off0, torch.int32),
        ("pts_off1", pts_off1, torch.int32), ("n_pts1", n_pts1, torch.int32), ("matches_p", matches_p, torch.int32),
        ("cu_p", cu_p, torch.int32), ("K0", K0, torch.float64), ("K1", K1, torch.float64), ("E", E, torch.float64),
        ("R", R, torch.float64), ("t", t, torch.float64), ("valid", valid, torch.uint8),
        ("inliers_p", inliers_p, torch.uint8), ("n_inliers", n_inliers, torch.int32),
        ("n_cheirality", n_cheirality, torch.int32), ("hypothesis", hypothesis, torch.int32),
        ("hypothesis_inliers", hypothesis_inliers, torch.int32), ("key", key, torch.int64)))
    inp = _struct(N.LtrEssentialInput, pts0=pts0, pts1=pts1, pts_off0=pts_off0, pts_off1=pts_off1, n_pts1=n_pts1,
                  matches_p=matches_p, cu_p=cu_p, K0=K0, K1=K1, n_pairs=int(n_pairs), max_rows_p=int(max_rows_p),
                  thresh=float(thresh), dist_thresh=float(dist_thresh), n_hypotheses=int(n_hypotheses),
                  seed=int(seed) & 0xFFFFFFFFFFFFFFFF)
    out = _struct(N.LtrEssentialOutput, E=E, R=R, t=t, valid=valid, inliers_p=inliers_p, n_inliers=n_inliers,
                  n_cheirality=n_cheirality, hypothesis=hypothesis, hypothesis_inliers=hypothesis_inliers, key=key)
    _call("ltr_essential", dev, C.byref(inp), C.byref(out))


def fundamental(n_pairs, *, pts0, pts1, pts_off0, pts_off1, n_pts1, matches_p, cu_p, max_rows_p, segs0, segs1,
                seg_off0, seg_off1, n_segs1, matches_l, cu_l, max_rows_l, F, valid, refit, inliers_p, lines_consistent,
                n_inliers, n_lines_consistent, hypothesis, hypothesis_inliers, key, thresh=3.0, min_overlap=0.5,
                n_hypotheses=2048, seed=0):
    """ltr_fundamental into caller-allocated outputs: keypoint pools [*,2] / segment pools [*,2,2] fp32, per-pair pool
    offsets and side-1 counts int32 [P], match rows int32 with offsets cu_p / cu_l [P+1]; F [P,3,3] fp64, valid / refit
    [P] uint8, inliers_p / lines_consistent uint8 aligned with the match rows, counts / hypothesis int32 [P], key [P]
    int64 workspace."""
    _req_cuda(F, "F")
    dev = F.device
    _check_tensors("fundamental", dev, (
        ("pts0", pts0, torch.float32), ("pts1", pts1, torch.float32), ("pts_off0", pts_off0, torch.int32),
        ("pts_off1", pts_off1, torch.int32), ("n_pts1", n_pts1, torch.int32), ("matches_p", matches_p, torch.int32),
        ("cu_p", cu_p, torch.int32), ("segs0", segs0, torch.float32), ("segs1", segs1, torch.float32),
        ("seg_off0", seg_off0, torch.int32), ("seg_off1", seg_off1, torch.int32), ("n_segs1", n_segs1, torch.int32),
        ("matches_l", matches_l, torch.int32), ("cu_l", cu_l, torch.int32), ("F", F, torch.float64),
        ("valid", valid, torch.uint8), ("refit", refit, torch.uint8), ("inliers_p", inliers_p, torch.uint8),
        ("lines_consistent", lines_consistent, torch.uint8), ("n_inliers", n_inliers, torch.int32),
        ("n_lines_consistent", n_lines_consistent, torch.int32), ("hypothesis", hypothesis, torch.int32),
        ("hypothesis_inliers", hypothesis_inliers, torch.int32), ("key", key, torch.int64)))
    inp = _struct(N.LtrFundamentalInput, pts0=pts0, pts1=pts1, pts_off0=pts_off0, pts_off1=pts_off1, n_pts1=n_pts1,
                  matches_p=matches_p, cu_p=cu_p, segs0=segs0, segs1=segs1, seg_off0=seg_off0, seg_off1=seg_off1,
                  n_segs1=n_segs1, matches_l=matches_l, cu_l=cu_l, n_pairs=int(n_pairs), max_rows_p=int(max_rows_p),
                  max_rows_l=int(max_rows_l), thresh=float(thresh), min_overlap=float(min_overlap),
                  n_hypotheses=int(n_hypotheses), seed=int(seed) & 0xFFFFFFFFFFFFFFFF)
    out = _struct(N.LtrFundamentalOutput, F=F, valid=valid, refit=refit, inliers_p=inliers_p,
                  lines_consistent=lines_consistent, n_inliers=n_inliers, n_lines_consistent=n_lines_consistent,
                  hypothesis=hypothesis, hypothesis_inliers=hypothesis_inliers, key=key)
    _call("ltr_fundamental", dev, C.byref(inp), C.byref(out))


def absolute_pose(n_pairs, n_groups, *, pts0, pts_off0, matches_p, cu_p, X1, x_off1, n_x1, segs0, seg_off0, matches_l,
                  cu_l, L1, l_off1, n_l1, groups, K0, max_rows_p, max_rows_l, R, t, valid, refit, inliers_p, inliers_l,
                  n_inliers_p, n_inliers_l, hypothesis, hypothesis_inliers, key, thresh=8.0, n_hypotheses=1024, seed=0,
                  use_lines=True):
    """ltr_absolute_pose into caller-allocated outputs: query keypoint pool [*,2] / segment pool [*,2,2] fp32 with
    per-pair first rows, world points X1 [*,3] / end points L1 [*,2,3] fp64 with per-pair first rows and counts int32
    [P], match rows int32 with offsets cu_p / cu_l [P+1], group offsets int32 [G+1], K0 fp64 [G,3,3]; R [G,3,3] / t
    [G,3] fp64, valid / refit [G] uint8, inliers_p / inliers_l uint8 aligned with the match rows, counts / hypothesis
    int32 [G], key [G] int64 workspace."""
    _req_cuda(R, "R")
    dev = R.device
    _check_tensors("absolute_pose", dev, (
        ("pts0", pts0, torch.float32), ("pts_off0", pts_off0, torch.int32), ("matches_p", matches_p, torch.int32),
        ("cu_p", cu_p, torch.int32), ("X1", X1, torch.float64), ("x_off1", x_off1, torch.int32),
        ("n_x1", n_x1, torch.int32), ("segs0", segs0, torch.float32), ("seg_off0", seg_off0, torch.int32),
        ("matches_l", matches_l, torch.int32), ("cu_l", cu_l, torch.int32), ("L1", L1, torch.float64),
        ("l_off1", l_off1, torch.int32), ("n_l1", n_l1, torch.int32), ("groups", groups, torch.int32),
        ("K0", K0, torch.float64), ("R", R, torch.float64), ("t", t, torch.float64), ("valid", valid, torch.uint8),
        ("refit", refit, torch.uint8), ("inliers_p", inliers_p, torch.uint8), ("inliers_l", inliers_l, torch.uint8),
        ("n_inliers_p", n_inliers_p, torch.int32), ("n_inliers_l", n_inliers_l, torch.int32),
        ("hypothesis", hypothesis, torch.int32), ("hypothesis_inliers", hypothesis_inliers, torch.int32),
        ("key", key, torch.int64)))
    inp = _struct(N.LtrAbsPoseInput, pts0=pts0, pts_off0=pts_off0, matches_p=matches_p, cu_p=cu_p, X1=X1,
                  x_off1=x_off1, n_x1=n_x1, segs0=segs0, seg_off0=seg_off0, matches_l=matches_l, cu_l=cu_l, L1=L1,
                  l_off1=l_off1, n_l1=n_l1, groups=groups, K0=K0, n_pairs=int(n_pairs), n_groups=int(n_groups),
                  max_rows_p=int(max_rows_p), max_rows_l=int(max_rows_l), thresh=float(thresh),
                  n_hypotheses=int(n_hypotheses), seed=int(seed) & 0xFFFFFFFFFFFFFFFF, use_lines=int(bool(use_lines)))
    out = _struct(N.LtrAbsPoseOutput, R=R, t=t, valid=valid, refit=refit, inliers_p=inliers_p, inliers_l=inliers_l,
                  n_inliers_p=n_inliers_p, n_inliers_l=n_inliers_l, hypothesis=hypothesis,
                  hypothesis_inliers=hypothesis_inliers, key=key)
    _call("ltr_absolute_pose", dev, C.byref(inp), C.byref(out))


def triangulate(*, kpts, kp_off, segs, seg_off, K, R, t, pairs, matches_p, cu_p, matches_l, cu_l, views, view_off,
                block_off, inv_off_p, inv_off_l, n_images, n_pairs, total_p, total_l, n_inv_p, n_inv_l, n_blocks,
                max_views, points3d, lines3d, n_views_p, n_views_l, inv_p, inv_l, thresh=4.0, min_angle=1.5,
                min_views=2):
    """ltr_triangulate into caller-allocated outputs: keypoint pool [*,2] / key-line pool [*,2,2] fp32 with image
    offsets [n+1], K / R [n,3,3] and t [n,3] fp64, pairs [P,2] and match rows int32 with offsets cu_p / cu_l [P+1],
    the observation lists (views, view_off), the block table block_off [2n+1] and the side-1 index offsets inv_off_*
    [P+1] int32; points3d [*,3] / lines3d [*,2,3] fp64, n_views_p / n_views_l int32, inv_p / inv_l int32 workspace."""
    _req_cuda(points3d, "points3d")
    dev = points3d.device
    _check_tensors("triangulate", dev, (
        ("kpts", kpts, torch.float32), ("kp_off", kp_off, torch.int32), ("segs", segs, torch.float32),
        ("seg_off", seg_off, torch.int32), ("K", K, torch.float64), ("R", R, torch.float64), ("t", t, torch.float64),
        ("pairs", pairs, torch.int32), ("matches_p", matches_p, torch.int32), ("cu_p", cu_p, torch.int32),
        ("matches_l", matches_l, torch.int32), ("cu_l", cu_l, torch.int32), ("views", views, torch.int32),
        ("view_off", view_off, torch.int32), ("block_off", block_off, torch.int32),
        ("inv_off_p", inv_off_p, torch.int32), ("inv_off_l", inv_off_l, torch.int32),
        ("points3d", points3d, torch.float64), ("lines3d", lines3d, torch.float64),
        ("n_views_p", n_views_p, torch.int32), ("n_views_l", n_views_l, torch.int32), ("inv_p", inv_p, torch.int32),
        ("inv_l", inv_l, torch.int32)))
    inp = _struct(N.LtrTriangulateInput, kpts=kpts, kp_off=kp_off, segs=segs, seg_off=seg_off, K=K, R=R, t=t,
                  pairs=pairs, matches_p=matches_p, cu_p=cu_p, matches_l=matches_l, cu_l=cu_l, views=views,
                  view_off=view_off, block_off=block_off, inv_off_p=inv_off_p, inv_off_l=inv_off_l,
                  n_images=int(n_images), n_pairs=int(n_pairs), total_p=int(total_p), total_l=int(total_l),
                  n_inv_p=int(n_inv_p), n_inv_l=int(n_inv_l), n_blocks=int(n_blocks), max_views=int(max_views),
                  thresh=float(thresh), min_angle=float(min_angle), min_views=int(min_views))
    out = _struct(N.LtrTriangulateOutput, points3d=points3d, lines3d=lines3d, n_views_p=n_views_p, n_views_l=n_views_l,
                  inv_p=inv_p, inv_l=inv_l)
    _call("ltr_triangulate", dev, C.byref(inp), C.byref(out))


_TRACK_OUTPUTS = (("track_p", torch.int32), ("track_l", torch.int32), ("n_tracks_p", torch.int32),
                  ("n_tracks_l", torch.int32), ("track_off_p", torch.int32), ("track_off_l", torch.int32),
                  ("obs_p", torch.int32), ("obs_l", torch.int32), ("points3d", torch.float64),
                  ("lines3d", torch.float64), ("n_obs_p", torch.int32), ("n_obs_l", torch.int32),
                  ("n_inliers_p", torch.int32), ("n_inliers_l", torch.int32), ("n_images_p", torch.int32),
                  ("n_images_l", torch.int32), ("status_p", torch.int32), ("status_l", torch.int32),
                  ("inlier_p", torch.uint8), ("inlier_l", torch.uint8), ("row_points3d", torch.float64),
                  ("row_lines3d", torch.float64), ("n_views_p", torch.int32), ("n_views_l", torch.int32),
                  ("workspace", torch.int32))


def tracks(*, kpts, kp_off, segs, seg_off, K, R, t, F, pairs, matches_p, cu_p, matches_l, cu_l, n_images, n_pairs,
           total_p, total_l, n_kp, n_kl, outputs: dict, thresh=4.0, min_angle=1.5, min_views=2, epi_thresh=4.0,
           min_overlap=0.5):
    """ltr_tracks into caller-allocated outputs: keypoint pool [*,2] / key-line pool [*,2,2] fp32 with image offsets
    [n+1], K / R [n,3,3], t [n,3] and the pairs' pixel fundamental matrices F [P,3,3] fp64, pairs [P,2] and match rows
    int32 with offsets cu_p / cu_l [P+1]; outputs {name: tensor} holds every LtrTracksOutput field (int32 workspace of
    5 (n_kp + n_kl))."""
    dev = outputs["workspace"].device
    _req_cuda(outputs["workspace"], "workspace")
    _check_tensors("tracks", dev, (
        ("kpts", kpts, torch.float32), ("kp_off", kp_off, torch.int32), ("segs", segs, torch.float32),
        ("seg_off", seg_off, torch.int32), ("K", K, torch.float64), ("R", R, torch.float64), ("t", t, torch.float64),
        ("F", F, torch.float64), ("pairs", pairs, torch.int32), ("matches_p", matches_p, torch.int32),
        ("cu_p", cu_p, torch.int32), ("matches_l", matches_l, torch.int32), ("cu_l", cu_l, torch.int32))
        + tuple((nm, outputs[nm], dt) for nm, dt in _TRACK_OUTPUTS))
    if outputs["workspace"].numel() < 5 * (int(n_kp) + int(n_kl)):
        raise N.LtrError("tracks: the workspace must hold 5 (n_kp + n_kl) int32")
    inp = _struct(N.LtrTracksInput, kpts=kpts, kp_off=kp_off, segs=segs, seg_off=seg_off, K=K, R=R, t=t, F=F,
                  pairs=pairs, matches_p=matches_p, cu_p=cu_p, matches_l=matches_l, cu_l=cu_l, n_images=int(n_images),
                  n_pairs=int(n_pairs), total_p=int(total_p), total_l=int(total_l), n_kp=int(n_kp), n_kl=int(n_kl),
                  thresh=float(thresh), min_angle=float(min_angle), min_views=int(min_views),
                  epi_thresh=float(epi_thresh), min_overlap=float(min_overlap))
    out = _struct(N.LtrTracksOutput, **{nm: outputs[nm] for nm, _ in _TRACK_OUTPUTS})
    _call("ltr_tracks", dev, C.byref(inp), C.byref(out))


_BUNDLE_INPUTS = (("kpts", torch.float32), ("kp_off", torch.int32), ("segs", torch.float32), ("seg_off", torch.int32),
                  ("K", torch.float64), ("R", torch.float64), ("t", torch.float64), ("hold", torch.int32),
                  ("fixed", torch.int32), ("n_tracks_p", torch.int32), ("n_tracks_l", torch.int32),
                  ("track_off_p", torch.int32), ("track_off_l", torch.int32), ("obs_p", torch.int32),
                  ("obs_l", torch.int32), ("status_p", torch.int32), ("status_l", torch.int32),
                  ("inlier_p", torch.uint8), ("inlier_l", torch.uint8), ("track_p", torch.int32),
                  ("track_l", torch.int32), ("n_views_p", torch.int32), ("n_views_l", torch.int32),
                  ("points3d", torch.float64), ("lines3d", torch.float64))
_BUNDLE_OUTPUTS = (("R", torch.float64), ("t", torch.float64), ("points3d", torch.float64), ("lines3d", torch.float64),
                   ("status_p", torch.int32), ("status_l", torch.int32), ("residual_p", torch.float64),
                   ("residual_l", torch.float64), ("row_points3d", torch.float64), ("row_lines3d", torch.float64),
                   ("n_views_p", torch.int32), ("n_views_l", torch.int32), ("stats", torch.float64),
                   ("workspace", torch.float64))


def bundle_adjust(*, inputs: dict, outputs: dict, n_images, n_fixed, n_kp, n_kl, t_p, t_l, max_iters=50, ftol=1e-10):
    """ltr_bundle_adjust into caller-allocated outputs: inputs {name: tensor} holds every LtrBundleInput pointer field
    (the set's rows and cameras, the held coordinates and fixed flags, and the ltr_tracks outputs), outputs every
    LtrBundleOutput field (an fp64 workspace of at least LTR_BA_WORKSPACE_BYTES)."""
    dev = outputs["workspace"].device
    _req_cuda(outputs["workspace"], "workspace")
    _check_tensors("bundle_adjust", dev, tuple((nm, inputs[nm], dt) for nm, dt in _BUNDLE_INPUTS)
                   + tuple((nm, outputs[nm], dt) for nm, dt in _BUNDLE_OUTPUTS))
    if outputs["workspace"].numel() * 8 < N.ba_workspace_bytes(n_images, n_kp, n_kl, t_p, t_l):
        raise N.LtrError("bundle_adjust: the workspace is smaller than LTR_BA_WORKSPACE_BYTES")
    inp = _struct(N.LtrBundleInput, **{nm: inputs[nm] for nm, _ in _BUNDLE_INPUTS}, n_images=int(n_images),
                  n_fixed=int(n_fixed), n_kp=int(n_kp), n_kl=int(n_kl), t_p=int(t_p), t_l=int(t_l),
                  max_iters=int(max_iters), ftol=float(ftol))
    out = _struct(N.LtrBundleOutput, **{nm: outputs[nm] for nm, _ in _BUNDLE_OUTPUTS})
    _call("ltr_bundle_adjust", dev, C.byref(inp), C.byref(out))


_GP_INPUTS = (("pairs", torch.int32), ("R", torch.float64), ("t", torch.float64), ("valid", torch.uint8),
              ("n_cheirality", torch.int32))
_GP_OUTPUTS = (("R", torch.float64), ("t", torch.float64), ("registered", torch.bool), ("edge_status", torch.int32),
               ("support", torch.int32), ("rot_residual", torch.float64), ("dir_cos", torch.float64),
               ("stats", torch.float64), ("workspace", torch.float64))


def global_poses(*, inputs: dict, outputs: dict, n_images, n_pairs, min_inliers, anchor, rot_iters, pos_iters, rot_tan,
                 dir_cos, ftol):
    """ltr_global_poses into caller-allocated outputs: inputs {name: tensor} holds every LtrGlobalPoseInput pointer
    field, outputs every LtrGlobalPoseOutput field (an fp64 workspace of at least LTR_GP_WORKSPACE_BYTES)."""
    dev = outputs["workspace"].device
    _req_cuda(outputs["workspace"], "workspace")
    _check_tensors("global_poses", dev, tuple((nm, inputs[nm], dt) for nm, dt in _GP_INPUTS)
                   + tuple((nm, outputs[nm], dt) for nm, dt in _GP_OUTPUTS))
    if outputs["workspace"].numel() * 8 < N.gp_workspace_bytes(n_images, n_pairs):
        raise N.LtrError("global_poses: the workspace is smaller than LTR_GP_WORKSPACE_BYTES")
    inp = _struct(N.LtrGlobalPoseInput, **{nm: inputs[nm] for nm, _ in _GP_INPUTS}, n_images=int(n_images),
                  n_pairs=int(n_pairs), min_inliers=int(min_inliers), anchor=int(anchor), rot_iters=int(rot_iters),
                  pos_iters=int(pos_iters), rot_tan=float(rot_tan), dir_cos=float(dir_cos), ftol=float(ftol))
    out = _struct(N.LtrGlobalPoseOutput, **{nm: outputs[nm] for nm, _ in _GP_OUTPUTS})
    _call("ltr_global_poses", dev, C.byref(inp), C.byref(out))


def warp_pairs(gray, colour, src_index_host: np.ndarray, src_index, inv_maps, warped, mask):
    """ltr_warp_pairs into caller-allocated outputs: gray uint8 [N,h,w], colour uint8 [N,h,w,C], src_index int32 [P]
    (host copy and device copy), inv_maps fp64 [P,9] on the device; warped / mask uint8 [P,h,w]."""
    dev = gray.device
    if gray.dim() != 3 or colour.dim() != 4 or tuple(colour.shape[:3]) != tuple(gray.shape):
        raise N.LtrError(f"warp_pairs: gray must be [N,h,w] and colour [N,h,w,C], got {list(gray.shape)} and "
                         f"{list(colour.shape)}")
    P = len(src_index_host)
    _check_tensors("warp_pairs", dev, (("gray", gray, torch.uint8), ("colour", colour, torch.uint8),
                                       ("src_index", src_index, torch.int32, (P,)),
                                       ("inv_maps", inv_maps, torch.float64, (P, 9)),
                                       ("warped", warped, torch.uint8, (P, *gray.shape[1:])),
                                       ("mask", mask, torch.uint8, (P, *gray.shape[1:]))))
    n, h, w = (int(s) for s in gray.shape)
    idx = np.ascontiguousarray(src_index_host, dtype=np.int32)
    _call("ltr_warp_pairs", dev, _ptr(gray), _ptr(colour), n, h, w, int(colour.shape[3]),
          idx.ctypes.data_as(N.c_int32_p), _ptr(src_index), _ptr(inv_maps), P, _ptr(warped), _ptr(mask))


def photometric(src, dst, params_host: np.ndarray, params, ellipses, taps, workspace):
    """ltr_photometric into a caller-allocated output: src / dst uint8 [N,h,w] (dst may be src), params fp64
    [N, PHOTOMETRIC_PARAMS] (host copy and device copy), ellipses int32 [N,E,5], taps float32 [N,149], workspace uint8
    of at least photometric_workspace_bytes(N, h, w)."""
    dev = src.device
    if src.dim() != 3:
        raise N.LtrError(f"photometric: images must be [N,h,w], got {list(src.shape)}")
    n, h, w = (int(s) for s in src.shape)
    ph = np.ascontiguousarray(params_host, dtype=np.float64)
    if ph.ndim != 2 or ph.shape[0] != n:
        raise N.LtrError(f"photometric: params must be [{n}, {N.PHOTOMETRIC_PARAMS}], got {list(ph.shape)}")
    E = int(ellipses.shape[1]) if ellipses.dim() == 3 else -1
    _check_tensors("photometric", dev, (("src", src, torch.uint8), ("dst", dst, torch.uint8, (n, h, w)),
                                        ("params", params, torch.float64, tuple(ph.shape)),
                                        ("ellipses", ellipses, torch.int32, (n, E, 5)),
                                        ("taps", taps, torch.float32, (n, N.PHOTOMETRIC_MAX_KSIZE)),
                                        ("workspace", workspace, torch.uint8)))
    _call("ltr_photometric", dev, _ptr(src), _ptr(dst), n, h, w, ph.ctypes.data_as(C.c_void_p), _ptr(params),
          int(ph.shape[1]), _ptr(ellipses), E, _ptr(taps), _ptr(workspace), int(workspace.numel()))


def match_distmat(dist: torch.Tensor, nn_thresh: float, mutual=True):
    """ltr_match_distmat on dist [P, n0, n1] (CUDA).  Returns dict(matches0 [P,n0], scores0, nn1, counts)."""
    _req_cuda(dist, "dist_mat")
    dev = dist.device
    dist = _f32c(dist)
    P, n0, n1 = (int(x) for x in dist.shape)
    i32 = dict(dtype=torch.int32, device=dev)
    out = {
        "matches0": torch.full((P, n0), -1, **i32),
        "scores0": torch.empty((P, n0), dtype=torch.float32, device=dev),
        "nn1": torch.full((P, n1), -1, **i32),
        "counts": torch.zeros(P, **i32),
    }
    if P == 0 or n0 == 0:
        return out
    _call("ltr_match_distmat", dev, _ptr(dist), P, n0, n1, 0, float(nn_thresh), int(bool(mutual)),
          _ptr(out["matches0"]), _ptr(out["scores0"]), _ptr(out["nn1"]), _ptr(out["counts"]))
    return out


def linear_img(x: torch.Tensor, w: torch.Tensor, bias=None, res=None, act=0, bn_hint=0):
    """ltr_linear_img (unit-test hook of the image-operand GEMM engine): returns (y_fp32, y_from_image)."""
    _req_cuda(x, "x")
    x = _f32c(x)
    w = _f32c(w).cpu()
    M, K = x.shape
    Nn = w.shape[0]
    y = torch.empty((M, Nn), dtype=torch.float32, device=x.device)
    y2 = torch.empty((M, Nn), dtype=torch.float32, device=x.device)
    bias = _f32c(bias) if bias is not None else None
    res = _f32c(res) if res is not None else None
    _call("ltr_linear_img", x.device, _ptr(x), K, _ptr(w), _ptr(bias), _ptr(res), Nn, _ptr(y), Nn, _ptr(y2), M, Nn, K,
          int(act), int(bn_hint))
    return y, y2


def linear_img_norm(x: torch.Tensor, w: torch.Tensor, bias=None, res=None, norm=1, eps=1e-6, gamma=None, beta=None, add=None):
    """ltr_linear_img_norm (unit-test hook of the row-normalising GEMM epilogue, N = 256):
    returns (y_fp32, y_from_image)."""
    _req_cuda(x, "x")
    x = _f32c(x)
    w = _f32c(w).cpu()
    M, K = x.shape
    if w.shape[0] != 256:
        raise N.LtrError("linear_img_norm: the row-norm epilogue is built for N = 256")
    y = torch.empty((M, 256), dtype=torch.float32, device=x.device)
    y2 = torch.empty((M, 256), dtype=torch.float32, device=x.device)
    f = lambda t: _f32c(t) if t is not None else None
    bias, res, gamma, beta, add = map(f, (bias, res, gamma, beta, add))
    _call("ltr_linear_img_norm", x.device, _ptr(x), K, _ptr(w), _ptr(bias), _ptr(res), 256, int(norm), float(eps),
          _ptr(gamma), _ptr(beta), _ptr(add), 256, _ptr(y), 256, _ptr(y2), M, K)
    return y, y2
