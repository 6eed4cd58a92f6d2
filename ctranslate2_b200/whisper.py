"""`ctranslate2.models.Whisper` for Device::CUDA on H100, on top of the C-ABI engine (include/ct2b200.h, Whisper section).

Mirrors python/cpp/whisper.cc / include/ctranslate2/models/whisper.h: `encode(features)` and `generate(features, prompts, ...)`
with the WhisperOptions of whisper.h:11-60.  Vocabulary lookups and the model's config.json (suppress_ids,
suppress_ids_begin) are handled here, as WhisperReplica does (src/models/whisper.cc:61-92, 311-323).  Served prompts:
previous-text tokens, `<|startoftranscript|>` and the task tokens (no text after them); the timestamp rules
(whisper.cc:742-860) run on the device unless the prompt ends with `<|notimestamps|>`."""
from __future__ import annotations

import ctypes
import json
import os
from dataclasses import dataclass, field
from typing import List, Sequence

import numpy as np

from ._lib import GeneratorConfig, check, lib
from .generator import _COMPUTE, _F16, _F32
from .translator import _FLOAT_OF_WEIGHTS, translator_summary


@dataclass
class WhisperGenerationResult:
    sequences: List[List[str]]
    sequences_ids: List[List[int]]
    scores: List[float] = field(default_factory=list)
    no_speech_prob: float = 0.0


class Whisper:
    def __init__(self, model_path: str, device: str = "cuda", device_index: int = 0, compute_type: str = "default",
                 use_cuda_graph: bool = True):
        if device not in ("cuda", "auto"):
            raise ValueError("ctranslate2_b200 runs on device='cuda' only (no CPU fallback)")
        if compute_type not in _COMPUTE:
            raise ValueError(f"Invalid compute type: {compute_type}")
        if not os.path.exists(os.path.join(model_path, "model.bin")):
            raise RuntimeError("Unable to open file 'model.bin' in model '%s'" % model_path)
        self._tokens = json.load(open(os.path.join(model_path, "vocabulary.json"), encoding="utf-8"))
        self._ids = {t: i for i, t in enumerate(self._tokens)}
        cfg_path = os.path.join(model_path, "config.json")
        self._config = json.load(open(cfg_path)) if os.path.exists(cfg_path) else {}
        self.sot_id, self.eot_id = self._ids["<|startoftranscript|>"], self._ids["<|endoftext|>"]
        self.no_timestamps_id = self._ids["<|notimestamps|>"]
        self.no_speech_id = self._ids.get("<|nospeech|>", self._ids.get("<|nocaptions|>", -1))
        dtype, weight_type = _COMPUTE[compute_type]
        if dtype is None:
            dtype = _FLOAT_OF_WEIGHTS.get(translator_summary(model_path)["weights"], _F32)
            if compute_type == "auto" and dtype == _F32:
                dtype = _F16
        cfg = GeneratorConfig(device_index, dtype, 0, 0, 0, 1, int(use_cuda_graph), 0, weight_type)
        self._h = lib().ct2b200_translator_open(model_path.encode(), ctypes.byref(cfg))
        if not self._h:
            raise RuntimeError(lib().ct2b200_last_error().decode())
        v = [ctypes.c_int() for _ in range(4)]
        check(lib().ct2b200_whisper_info(ctypes.c_void_p(self._h), *[ctypes.byref(x) for x in v]))
        self.n_mels, self.max_frames, self.d_model, self.vocab_size = (x.value for x in v)

    def __del__(self):
        self.close()

    def close(self):
        if getattr(self, "_h", None):
            lib().ct2b200_translator_close(ctypes.c_void_p(self._h))
            self._h = None

    @property
    def is_multilingual(self) -> bool:
        return len(self._config.get("lang_ids", [])) > 1

    def _features(self, features) -> np.ndarray:
        f = np.ascontiguousarray(np.asarray(features, dtype=np.float32))
        if f.ndim != 3:
            raise ValueError("Expected input features to have 3 dimensions, but got %d dimension(s) instead" % f.ndim)
        if f.shape[1] != self.n_mels or (f.shape[2] + 1) // 2 > self.max_frames:
            raise ValueError("Invalid input features shape: expected an input with shape (%d, %d, %d), but got an input with "
                             "shape %s instead" % (f.shape[0], self.n_mels, min(f.shape[2], 2 * self.max_frames), tuple(f.shape)))
        return f

    def encode(self, features) -> np.ndarray:
        """WhisperEncoder output [batch, frames / 2, d_model] float32."""
        f = self._features(features)
        B, _, T = f.shape
        out = np.empty((B, (T + 1) // 2, self.d_model), np.float32)
        p = ctypes.c_void_p
        check(lib().ct2b200_whisper_encode(p(self._h), f.ctypes.data_as(p), ctypes.c_int64(B), ctypes.c_int64(T),
                                           out.ctypes.data_as(p)))
        return out

    def generate(self, features, prompts: Sequence[Sequence], *, beam_size: int = 5, patience: float = 1.0,
                 num_hypotheses: int = 1, length_penalty: float = 1.0, repetition_penalty: float = 1.0,
                 no_repeat_ngram_size: int = 0, max_length: int = 448, return_scores: bool = False,
                 return_logits_vocab: bool = False, return_no_speech_prob: bool = False,
                 max_initial_timestamp_index: int = 50, suppress_blank: bool = True,
                 suppress_tokens: Sequence[int] = (-1,), sampling_topk: int = 1,
                 sampling_temperature: float = 1.0) -> List[WhisperGenerationResult]:
        if repetition_penalty != 1 or no_repeat_ngram_size != 0 or return_logits_vocab or sampling_topk != 1 \
                or sampling_temperature != 1:
            raise ValueError("this engine implements the default repetition_penalty, no_repeat_ngram_size, return_logits_vocab, "
                             "sampling_topk and sampling_temperature only")
        f = self._features(features)
        rows = [[self._ids[t] if isinstance(t, str) else int(t) for t in r] for r in prompts]
        if not rows:
            return []
        if len(rows) != f.shape[0]:
            raise ValueError("one prompt per batch entry is required")
        P = len(rows[0])
        if any(len(r) != P for r in rows):
            raise ValueError("The generate method currently requires each batch to have the same number of task tokens")
        suppress = []
        for t in suppress_tokens:
            if t >= 0:
                suppress.append(int(t))
            elif t == -1:
                suppress += [int(x) for x in self._config.get("suppress_ids", [])]
        begin = [int(x) for x in self._config.get("suppress_ids_begin", [])] if suppress_blank else []
        B, _, T = f.shape
        pr = np.ascontiguousarray(np.array(rows, np.int32))
        sup, beg = np.array(suppress, np.int32), np.array(begin, np.int32)
        out = np.empty((B, num_hypotheses, max_length), np.int32)
        lens = np.empty((B, num_hypotheses), np.int32)
        scores = np.zeros((B, num_hypotheses), np.float32)
        nsp = np.zeros(B, np.float32)
        p = ctypes.c_void_p
        check(lib().ct2b200_whisper_generate(
            p(self._h), f.ctypes.data_as(p), ctypes.c_int64(B), ctypes.c_int64(T), pr.ctypes.data_as(p), ctypes.c_int64(P),
            int(beam_size), ctypes.c_float(patience), ctypes.c_float(length_penalty), ctypes.c_int64(max_length),
            int(num_hypotheses), sup.ctypes.data_as(p), int(sup.size), beg.ctypes.data_as(p), int(beg.size),
            ctypes.c_int32(self.sot_id), ctypes.c_int32(self.eot_id), ctypes.c_int32(self.no_speech_id),
            ctypes.c_int32(self.no_timestamps_id), int(max_initial_timestamp_index), out.ctypes.data_as(p),
            lens.ctypes.data_as(p), scores.ctypes.data_as(p), nsp.ctypes.data_as(p) if return_no_speech_prob else None))
        results = []
        for b in range(B):
            ids = [out[b, h, :lens[b, h]].tolist() for h in range(num_hypotheses) if lens[b, h] >= 0]
            results.append(WhisperGenerationResult([[self._tokens[i] for i in s] for s in ids], ids,
                                                   [float(scores[b, h]) for h in range(len(ids))] if return_scores else [],
                                                   float(nsp[b]) if return_no_speech_prob else 0.0))
        return results
