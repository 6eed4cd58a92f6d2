"""`ctranslate2.Encoder` for Device::CUDA on H100, on top of the C-ABI engine (include/ct2b200.h, encoder-only path).

Mirrors python/cpp/encoder.cc: `forward_batch(inputs, lengths=None, token_type_ids=None)` on a TransformerEncoderSpec model
(BERT, DistilBERT, RoBERTa, XLM-R class), returning the last hidden state and, for models with a pooler, the pooled first
position (models::EncoderReplica::forward_impl, src/models/language_model.cc:349-400).  Token strings are looked up in the
model's vocabulary here (unknown tokens map to `unk_token`); ids and outputs cross the boundary in HOST buffers."""
from __future__ import annotations

import ctypes
import json
import os
from dataclasses import dataclass
from typing import List, Optional

import numpy as np

from ._lib import GeneratorConfig, check, lib
from .generator import _COMPUTE, _F16, _F32, _non_negative_int, _rebatch
from .translator import _FLOAT_OF_WEIGHTS, _load_vocabulary


@dataclass
class EncoderForwardOutput:
    """last_hidden_state [batch, max_length, d_model] float32 (positions past a row's length hold unspecified values);
    pooler_output [batch, d_model] float32, or None when the model has no pooler."""
    last_hidden_state: np.ndarray
    pooler_output: Optional[np.ndarray] = None


def encoder_summary(model_path: str) -> dict:
    """Geometry of a TransformerEncoderSpec directory (host only, no GPU needed; ct2b200_encoder_summary).  Raises ValueError
    for what the engine does not run."""
    buf = ctypes.create_string_buffer(2048)
    check(lib().ct2b200_encoder_summary(model_path.encode(), buf, ctypes.c_size_t(len(buf))))
    return json.loads(buf.value.decode())


def _rows(x, what: str) -> List[list]:
    if isinstance(x, np.ndarray):
        if x.ndim != 2:
            raise ValueError(f"forward_batch: {what} must have 2 dimensions, got {x.ndim}")
        return [list(r) for r in x.tolist()]
    rows = [list(r) for r in x]
    for b, r in enumerate(rows):
        for v in r:
            if isinstance(v, str) or isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)):
                raise ValueError(f"forward_batch: {what} {b} holds {type(v).__name__} values instead of integer ids")
    return rows


class Encoder:
    def __init__(self, model_path: str, device: str = "cuda", device_index: int = 0, compute_type: str = "default",
                 max_batch_size: int = 64):
        """max_batch_size: rows per device pass; larger requests are split longest first and answered in request order."""
        if device not in ("cuda", "auto"):
            raise ValueError("ctranslate2_b200 runs on device='cuda' only (no CPU fallback)")
        if compute_type not in _COMPUTE:
            raise ValueError(f"Invalid compute type: {compute_type}")
        self.max_batch_size = _non_negative_int("max_batch_size", max_batch_size)
        if self.max_batch_size == 0:
            raise ValueError("max_batch_size must be >= 1")
        if not os.path.exists(os.path.join(model_path, "model.bin")):
            raise RuntimeError("Unable to open file 'model.bin' in model '%s'" % model_path)
        self.model_path = model_path
        cfg_path = os.path.join(model_path, "config.json")
        self._config = json.load(open(cfg_path)) if os.path.exists(cfg_path) else {}
        self._vocab = _load_vocabulary(model_path, "vocabulary")
        if self._vocab is None:
            raise RuntimeError("Cannot load the vocabulary from the model directory")
        self._to_id = {t: i for i, t in enumerate(self._vocab)}
        self._info = encoder_summary(model_path)
        dtype, weight_type = _COMPUTE[compute_type]
        if dtype is None:
            dtype = _FLOAT_OF_WEIGHTS.get(self._info["weights"], _F32)
            if compute_type == "auto" and dtype == _F32:
                dtype = _F16
        self.compute_type = compute_type
        cfg = GeneratorConfig(device_index, dtype, self.max_batch_size, 0, 0, 1, 0, 0, weight_type)
        L = lib()
        L.ct2b200_encoder_open.restype = ctypes.c_void_p
        self._h = L.ct2b200_encoder_open(model_path.encode(), ctypes.byref(cfg))
        if not self._h:
            raise RuntimeError(L.ct2b200_last_error().decode())

    def __del__(self):
        self.close()

    def close(self):
        if getattr(self, "_h", None):
            lib().ct2b200_encoder_close(ctypes.c_void_p(self._h))
            self._h = None

    @property
    def unk_token(self) -> str:
        return self._config.get("unk_token", "<unk>")

    def _ids(self, tokens) -> List[int]:
        unk = self._to_id.get(self.unk_token, 0)
        return [self._to_id.get(t, unk) for t in tokens]

    def forward_batch(self, inputs, lengths=None, token_type_ids=None) -> EncoderForwardOutput:
        """Encoder.forward_batch (python/cpp/encoder.cc): `inputs` = token-string lists, id lists, or a dense [batch, time]
        id array with `lengths` [batch] (required for a dense array, as in the reference).  token_type_ids: id lists or a
        [batch, time] array matching the inputs, None = zeros."""
        if isinstance(inputs, np.ndarray) or (lengths is not None):
            if lengths is None:
                raise ValueError("forward_batch: lengths is required when the inputs are a dense id array")
            ids = np.asarray(inputs)
            if ids.ndim != 2:
                raise ValueError(f"forward_batch: input ids must have 2 dimensions, got {ids.ndim}")
            if not np.issubdtype(ids.dtype, np.integer):
                raise ValueError("forward_batch: a dense input array must hold integer ids")
            lens = np.asarray(lengths)
            if lens.ndim != 1 or lens.shape[0] != ids.shape[0]:
                raise ValueError(f"forward_batch: expected lengths of size {ids.shape[0]}, got shape {lens.shape}")
            if np.any(lens > ids.shape[1]):
                raise ValueError("forward_batch: a length exceeds the width of the input array")
            rows = [ids[b, :int(lens[b])].tolist() for b in range(ids.shape[0])]
        else:
            rows = [list(r) for r in inputs]
            rows = [self._ids(r) if (r and isinstance(r[0], str)) else r for r in rows]
            rows = _rows(rows, "input")
        if not rows:
            raise ValueError("forward_batch: empty batch")
        types = None
        if token_type_ids is not None:
            if self._info["type_vocab_size"] == 0:
                raise ValueError("forward_batch: this model has no token-type embeddings")
            types = _rows(token_type_ids, "token_type_ids")
            if len(types) != len(rows):
                raise ValueError(f"forward_batch: {len(rows)} inputs but {len(types)} token_type_ids rows")
            for b, (r, t) in enumerate(zip(rows, types)):
                if len(t) < len(r):
                    raise ValueError(f"forward_batch: token_type_ids row {b} has {len(t)} values for {len(r)} tokens")
                types[b] = t[:len(r)]
        V, TV, P = self._info["vocab_size"], self._info["type_vocab_size"], self._info["max_positions"]
        for b, r in enumerate(rows):
            if len(r) == 0:
                raise ValueError(f"forward_batch: input {b} is empty")
            if len(r) > P:
                raise ValueError(f"forward_batch: input {b} has {len(r)} tokens, more than the {P} positions of the model")
            bad = [i for i in r if not 0 <= i < V]
            if bad:
                raise ValueError(f"forward_batch: id {bad[0]} of input {b} is outside the vocabulary [0, {V})")
            if types is not None:
                bad = [i for i in types[b] if not 0 <= i < TV]
                if bad:
                    raise ValueError(f"forward_batch: token type {bad[0]} of input {b} is outside [0, {TV})")
        T, d = max(len(r) for r in rows), self._info["d_model"]
        hidden = np.zeros((len(rows), T, d), np.float32)
        pooled = np.zeros((len(rows), d), np.float32) if self._info["pooler"] else None
        p = ctypes.c_void_p
        for idx in _rebatch([len(r) for r in rows], self.max_batch_size, "examples", self.max_batch_size):
            B, L = len(idx), max(len(rows[i]) for i in idx)
            ids = np.zeros((B, L), np.int32)
            tt = np.zeros((B, L), np.int32) if types is not None else None
            lens = np.array([len(rows[i]) for i in idx], np.int32)
            for j, i in enumerate(idx):
                ids[j, :lens[j]] = rows[i]
                if tt is not None:
                    tt[j, :lens[j]] = types[i]
            h = np.empty((B, L, d), np.float32)
            po = np.empty((B, d), np.float32) if pooled is not None else None
            check(lib().ct2b200_encoder_forward(
                p(self._h), ids.ctypes.data_as(p), lens.ctypes.data_as(p), None if tt is None else tt.ctypes.data_as(p),
                ctypes.c_int64(B), ctypes.c_int64(L), h.ctypes.data_as(p), None if po is None else po.ctypes.data_as(p)))
            for j, i in enumerate(idx):
                hidden[i, :L] = h[j]
                if pooled is not None:
                    pooled[i] = po[j]
        return EncoderForwardOutput(hidden, pooled)

    def bench(self, lengths, max_length: int, iters: int = 10, warmup: int = 2) -> float:
        """Median device time (ms) of one encoder pass over len(lengths) rows of the given lengths (synthetic ids)."""
        lens = np.asarray(lengths, np.int32)
        ms = ctypes.c_float()
        check(lib().ct2b200_encoder_bench(ctypes.c_void_p(self._h), lens.ctypes.data_as(ctypes.c_void_p),
                                          ctypes.c_int64(lens.size), ctypes.c_int64(max_length), ctypes.c_int64(iters),
                                          ctypes.c_int64(warmup), ctypes.byref(ms)))
        return ms.value
