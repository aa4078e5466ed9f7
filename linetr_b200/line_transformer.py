"""Drop-in `LineTransformer` with the reference's call surface, computing on the CUDA library.

Mirrors yosungho/LineTR `models/line_transformer.py:185-291` (class LineTransformer):
same constructor/config dict, same state-dict keys (so the shipped `LineTR_weight.pth` loads
with `strict=True`), same `forward(dict) -> dict` contract (adds `'line_desc'` [B,256,L] and
returns the same dict object), same `preprocess` / `subline2keyline` / `default_ret` helpers.

The nn.Module tree below only *holds parameters* under the reference's names; no torch op
of it is ever executed.  `forward` hands the tensors to `ltr_encode` (include/linetr_b200.h).
"""
from __future__ import annotations

import os
from copy import deepcopy
from pathlib import Path

import numpy as np
import torch
from torch import nn

from . import _native as N
from . import _ops
from . import line_process as LP
from .line_process import get_dist_matrix  # noqa: F401  (reference re-exports it via `import *`)


def _mlp_container(channels):
    """Parameter container with the indices of the reference MLP() (line_transformer.py:9-20):
    Conv1d(k=1) at 3i, BatchNorm1d at 3i+1, ReLU at 3i+2, last layer conv only."""
    layers = []
    n = len(channels)
    for i in range(1, n):
        layers.append(nn.Conv1d(channels[i - 1], channels[i], kernel_size=1, bias=True))
        if i < n - 1:
            layers.append(nn.BatchNorm1d(channels[i]))
            layers.append(nn.ReLU())
    return nn.Sequential(*layers)


class _Holder(nn.Module):
    """Named parameter container; never called."""

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("parameter container - computation happens in liblinetr_b200.so")


def _pos_encoder(n_in, layers, feature_dim):
    h = _Holder()
    h.encoder = _mlp_container([n_in] + list(layers) + [feature_dim])
    nn.init.constant_(h.encoder[-1].bias, 0.0)
    return h


def _desc_layer(d, n_heads, d_inner):
    h = _Holder()
    h.slf_attn = _Holder()
    h.slf_attn.w_qs = nn.Linear(d, d, bias=True)
    h.slf_attn.w_ks = nn.Linear(d, d, bias=True)
    h.slf_attn.w_vs = nn.Linear(d, d, bias=True)
    h.slf_attn.fc = nn.Linear(d, d, bias=True)
    h.slf_attn.layer_norm = nn.LayerNorm(d, eps=1e-6)
    h.pos_ffn = _Holder()
    h.pos_ffn.w_1 = nn.Linear(d, d_inner)
    h.pos_ffn.w_2 = nn.Linear(d_inner, d)
    h.pos_ffn.layer_norm = nn.LayerNorm(d, eps=1e-6)
    return h


def _sig_layer(d):
    h = _Holder()
    h.attn = _Holder()
    h.attn.merge = nn.Conv1d(d, d, kernel_size=1)
    h.attn.proj = nn.ModuleList([deepcopy(h.attn.merge) for _ in range(3)])
    h.mlp = _mlp_container([2 * d, 2 * d, d])
    nn.init.constant_(h.mlp[-1].bias, 0.0)
    return h


def _find_weights(config):
    cands = [config.get("weights_path"), os.environ.get("LINETR_WEIGHTS"),
             str(Path(__file__).parent / "weights" / "LineTR_weight.pth")]
    for c in cands:
        if c and os.path.exists(c):
            return c
    raise FileNotFoundError(
        "LineTransformer(mode='test') needs the LineTR checkpoint: put LineTR_weight.pth into "
        f"{Path(__file__).parent / 'weights'} or set config['weights_path'] / $LINETR_WEIGHTS")


class LineTransformer(nn.Module):
    """Line-Transformer networks (line descriptive + line signature), H100-native."""

    default_config = {
        "mode": "test",
        "image_shape": [480, 640],
        "min_length": 16,
        "token_distance": 8,
        "max_tokens": 21,
        "remove_borders": 8,
        "max_keylines": -1,
        "descriptor_dim": 256,
        "keyline_encoder": [32, 64, 128, 256],
        "n_heads": 4,
        "n_line_descriptive_layers": 1,
        "d_inner": 1024,
    }
    # linetr_b200 extension, not part of default_config (which stays identical to the reference's): config
    # {'cuda_graph': True} replays the ~40 kernel launches of a forward from a CUDA graph captured per
    # (batch, lines, tokens) shape - single-image latency is launch-bound.

    def __init__(self, config):
        super().__init__()
        self.config = {**self.default_config, **config}
        self.image_shape = self.config["image_shape"]
        d = self.config["descriptor_dim"]
        if d != 256 or self.config["n_heads"] != 4 or list(self.config["keyline_encoder"]) != [32, 64, 128, 256]:
            raise N.LtrError("linetr_b200 kernels are specialised for descriptor_dim=256, n_heads=4, "
                             "keyline_encoder=[32,64,128,256] (the shipped LineTR architecture)")
        assert d % self.config["n_heads"] == 0
        # construction order mirrors the reference so that torch.manual_seed(s) gives the same init
        self.klenc = _Holder()
        self.klenc.feature_dim = d
        self.klenc.line_position_enc = _pos_encoder(5, self.config["keyline_encoder"], d)
        self.klenc.word_position_enc = _pos_encoder(3, self.config["keyline_encoder"], d)
        self.klenc.desc_layers = nn.ModuleList([
            _desc_layer(d, self.config["n_heads"], self.config["d_inner"])
            for _ in range(self.config["n_line_descriptive_layers"])])
        self.klenc.cls_token = nn.Parameter(torch.randn(1, 1, 1, d))
        self.selfattn = _Holder()
        self.selfattn.layers = nn.ModuleList([_sig_layer(d) for _ in range(7)])
        self.selfattn.names = ["self"] * 7
        self.final_proj = nn.Conv1d(d, d, kernel_size=1, bias=True)
        self._handle = None
        self._handle_sig = None
        self._tensors = None
        if self.config["mode"] == "test":
            self.load_state_dict(torch.load(_find_weights(self.config), map_location="cpu"))
            print("Loaded Line-Transformer model")

    # ------------------------------------------------------------------ packed weights
    def _apply(self, fn, *a, **k):
        # .to() / .cuda() / .float() replace parameter storage: the packed copy must be rebuilt
        self._tensors = None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self._tensors = None
        return super().load_state_dict(*a, **k)

    def _signature(self, device):
        """Cheap change detector of the weights behind the packed copy: in-place updates bump the tensors'
        version counters, storage swaps go through _apply / load_state_dict.  One pass over a cached list
        (198 tensors, ~15 us) instead of rebuilding parameter / buffer lists on every forward."""
        ts = getattr(self, "_tensors", None)
        if ts is None:
            ts = self._tensors = list(self.parameters()) + list(self.buffers())
            self._ptrs = tuple(t.data_ptr() for t in ts)
        v = 0
        for t in ts:
            v += t._version
        return (device.index, v, self._ptrs)

    def _get_handle(self, device) -> _ops.ModelHandle:
        sig = self._signature(device)
        if self._handle is None or sig != self._handle_sig:
            if tuple(t.data_ptr() for t in self._tensors) != self._ptrs:   # storage swapped behind our back (p.data = ...)
                self._tensors = None
                sig = self._signature(device)
            if self._handle is not None:
                self._handle.close()
            sd = {k: v.detach().float().cpu().numpy() for k, v in self.state_dict().items()}
            self._handle = _ops.ModelHandle(sd, device.index, 256, 4, int(self.config["d_inner"]),
                                            int(self.config["n_line_descriptive_layers"]), 7)
            self._handle_sig = sig
        return self._handle

    def _image_wh(self):
        shp = self.image_shape
        if len(shp) == 2:
            h, w = shp
        else:
            _, _, h, w = shp
        return float(w), float(h)

    # ------------------------------------------------------------------ reference API
    def forward(self, data):
        if len(data["klines"]) == 0:
            return self.default_ret()
        klines = data["sublines"]
        resp = data["resp_sublines"]
        angle = data["angle_sublines"]
        pnt = data["pnt_sublines"]
        desc = data["desc_sublines"]
        score = data["score_sublines"]
        data["mask_sublines"]  # read like the reference does; it cannot change the output (SURVEY §0.3)
        _ops._req_cuda(desc, "desc_sublines")   # CUDA only: there is no CPU fallback
        B, L, T = int(desc.shape[0]), int(desc.shape[1]), int(desc.shape[2])
        handle = self._get_handle(desc.device)
        flat = (klines.reshape(B * L, 2, 2), resp.reshape(B * L, 1), angle.reshape(B * L, 2), pnt.reshape(B * L, T, 2),
                desc.reshape(B * L, T, 256), score.reshape(B * L, T, 1))
        if self.config.get("cuda_graph") and B * L > 0:
            out_cf = self._forward_graphed(handle, flat, B, L, T)
        else:
            out_cf, _ = _ops.encode(handle, *flat, self._image_wh(), lines_per_image=L)
        data.update({"line_desc": out_cf.view(B, 256, L)})
        return data

    def _forward_graphed(self, handle, flat, B, L, T):
        """ltr_encode of one shape captured once in a CUDA graph (static input / output buffers); later calls
        copy the inputs in, replay, and hand out a copy of the result (callers keep the descriptors of
        several images alive - models/matching.py:41,59)."""
        dev = flat[4].device
        key = (id(handle), B, L, T, self._image_wh())
        graphs = self.__dict__.setdefault("_graphs", {})
        ent = graphs.get(key)
        if ent is None:
            if len(graphs) >= 32:
                graphs.clear()
            static_in = [_ops._f32c(t).clone() for t in flat]
            _ops.encode(handle, *static_in, self._image_wh(), lines_per_image=L)   # eager warm-up: attributes, workspace
            torch.cuda.current_stream(dev).synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                static_out, _ = _ops.encode(handle, *static_in, self._image_wh(), lines_per_image=L)
            ent = graphs[key] = (g, static_in, static_out)
        g, static_in, static_out = ent
        for dst, src in zip(static_in, flat):
            dst.copy_(src, non_blocking=True)
        g.replay()
        return static_out.clone()

    def preprocess(self, klines_cv, image_shape, pred_superpoint, valid_mask=None):
        """Line tokenisation (glue; reference models/line_transformer.py:251-275)."""
        klines = LP.change_cv2_T_np(klines_cv)
        _, _, height, width = self.config["image_shape"] = image_shape
        border = self.config["remove_borders"]
        if valid_mask is None:
            valid_mask = np.ones((height, width))
        klines = LP.remove_borders(klines, border, height, width, valid_mask)
        klines = LP.filter_by_length(klines, self.config["min_length"], self.config["max_keylines"])
        if len(klines["klines"]) == 0:
            return klines
        tok = LP.line_tokenizer_gpu if pred_superpoint["dense_descriptor"].is_cuda else LP.line_tokenizer
        return tok(klines, self.config["token_distance"], self.config["max_tokens"], pred_superpoint, image_shape[-2:])

    def subline2keyline(self, distance_sublines, mat_klines2sublines0, mat_klines2sublines1):
        """A0 @ D @ A1^T on the GPU (reference models/line_transformer.py:277-282) -> np [1,K0,K1]."""
        from .nn_matcher import subline2keyline
        return subline2keyline(distance_sublines, mat_klines2sublines0, mat_klines2sublines1)

    def default_ret(self):
        pred = {}
        pred["klines"] = torch.empty((1, 0, 2, 2))
        pred["sublines"] = torch.empty((1, 0, 2, 2))
        pred["line_desc"] = torch.empty((1, 256, 0))
        pred["mat_klines2sublines"] = torch.empty((1, 0, 0))
        return pred
