"""Device-level wrappers around the C ABI: CUDA torch tensors in, CUDA torch tensors out.

PyTorch is used here only for device memory, streams and dtype plumbing; all arithmetic
happens inside liblinetr_b200.so.  Every function raises if the tensors are not on a CUDA
device (no CPU fallback).
"""
from __future__ import annotations

import ctypes as C
import functools

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


# the tensor dtypes a pointer field takes by its pointee (_native._pointees_; a void* field takes any) and the
# conversion of each scalar field type
_POINTEE_DTYPES = {C.c_float: (torch.float32,), C.c_double: (torch.float64,), C.c_int32: (torch.int32,),
                   C.c_uint64: (torch.int64,), C.c_uint8: (torch.uint8, torch.bool)}
_SCALAR = {C.c_int32: int, C.c_int64: int, C.c_float: float, C.c_double: float,
           C.c_uint64: lambda v: int(v) & 0xFFFFFFFFFFFFFFFF}


@functools.cache
def _layout(cls):
    """(field names, pointer fields as (name, dtypes or None for void*), scalar fields as (name, conversion)) of a
    struct mirror."""
    ptrs = tuple((nm, _POINTEE_DTYPES[cls._pointees_[nm]] if nm in cls._pointees_ else None)
                 for nm, t in cls._fields_ if t is C.c_void_p)
    scalars = tuple((nm, _SCALAR[t]) for nm, t in cls._fields_ if t is not C.c_void_p)
    return frozenset(nm for nm, _ in cls._fields_), ptrs, scalars


def call_struct(entry: str, inputs: dict, outputs: dict, workspace_bytes=None, scalars=()):
    """`entry`(const In*, const Out*, *scalars, device, stream) with the fields of its In and Out structs by name (and
    the entry's own scalar arguments after the structs, in order): every scalar field is required; a pointer field
    takes None (NULL) or a contiguous CUDA tensor of the dtype its mirror names (any dtype for void*), on the device of
    the outputs.  Runs on that device's current stream.  workspace_bytes, when given, is the least size of the
    `workspace` output.  The caller keeps the tensors alive until the call."""
    who = entry[4:]
    _, (p_in, p_out, *_) = N.PROTOTYPES[entry]
    dev, structs = None, {}
    for cls, given in ((p_out._type_, outputs), (p_in._type_, inputs)):
        names, ptrs, fixed = _layout(cls)
        if not given.keys() <= names:
            raise N.LtrError(f"{who}: {cls.__name__} has no field {sorted(given.keys() - names)}")
        fields = {}
        for nm, dts in ptrs:
            t = given.get(nm)
            if t is None:
                continue
            _req_cuda(t, nm)
            dev = t.device if dev is None else dev
            if (dts is not None and t.dtype not in dts) or not t.is_contiguous() or t.device != dev:
                raise N.LtrError(f"{who}: '{nm}' must be a contiguous {f'{dts[0]} ' if dts else ''}tensor on {dev}")
            fields[nm] = t.data_ptr()
        for nm, conv in fixed:
            if nm not in given:
                raise N.LtrError(f"{who}: {cls.__name__}.{nm} is not given")
            fields[nm] = conv(given[nm])
        structs[cls] = cls(**fields)
    if workspace_bytes is not None:
        ws = outputs["workspace"]
        if ws.numel() * ws.element_size() < workspace_bytes:
            raise N.LtrError(f"{who}: the workspace holds {ws.numel() * ws.element_size()} bytes, {workspace_bytes} "
                             "needed")
    _call(entry, dev, C.byref(structs[p_in._type_]), C.byref(structs[p_out._type_]), *scalars)


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
