"""`ctranslate2.Translator` for Device::CUDA on H100, on top of the C-ABI engine (include/ct2b200.h, encoder-decoder path).

Mirrors python/cpp/translator.cc / include/ctranslate2/translator.h: `translate_batch(source, ...)` with the
TranslationOptions of include/ctranslate2/translation.h.  Token strings <-> ids (ctranslate2::Vocabulary: source /
target / shared vocabulary files, `add_source_bos` / `add_source_eos` / `decoder_start_token` of config.json) are handled
here, as in models::SequenceToSequenceModel (src/models/sequence_to_sequence.cc:19-100); ids cross the boundary in HOST
buffers.  The encoder, the decoder with cross-attention and the beam search run on the device."""
from __future__ import annotations

import ctypes
import json
import os
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Union

import numpy as np

from ._lib import GeneratorConfig, check, lib
from .generator import _COMPUTE, _F16, _F32, _is_neutral  # noqa: F401

_FLOAT_OF_WEIGHTS = {"float16": 1, "bfloat16": 2}


@dataclass
class TranslationResult:
    hypotheses: List[List[str]]
    hypotheses_ids: List[List[int]]
    scores: List[float] = field(default_factory=list)


def translator_summary(model_path: str) -> dict:
    """Geometry of an encoder-decoder model directory (host only, no GPU needed; ct2b200_translator_summary)."""
    buf = ctypes.create_string_buffer(2048)
    check(lib().ct2b200_translator_summary(model_path.encode(), buf, ctypes.c_size_t(len(buf))))
    return json.loads(buf.value.decode())


# TranslationOptions (include/ctranslate2/translation.h:14-98) this engine does not implement, with the only value it accepts
_NEUTRAL = {
    "coverage_penalty": 0, "repetition_penalty": 1, "no_repeat_ngram_size": 0, "disable_unk": False,
    "suppress_sequences": None, "prefix_bias_beta": 0, "sampling_topk": 1, "sampling_topp": 1, "sampling_temperature": 1,
    "use_vmap": False, "return_attention": False, "return_logits_vocab": False, "return_alternatives": False,
    "min_alternative_expansion_prob": 0, "replace_unknowns": False, "callback": None, "asynchronous": False,
    "max_batch_size": 0, "batch_type": "examples", "max_input_length": 1024,
}


def _neutral(name, value) -> bool:
    neutral = _NEUTRAL[name]
    if neutral is None:
        return value is None or (hasattr(value, "__len__") and len(value) == 0)
    if isinstance(neutral, bool):
        return isinstance(value, (bool, np.bool_)) and bool(value) == neutral
    if isinstance(neutral, str):
        return value == neutral
    return not isinstance(value, (bool, np.bool_)) and isinstance(value, (int, float, np.integer, np.floating)) \
        and float(value) == float(neutral)


def _load_vocabulary(model_path: str, name: str) -> Optional[List[str]]:
    for ext in (".json", ".txt"):
        p = os.path.join(model_path, name + ext)
        if os.path.exists(p):
            if ext == ".json":
                return json.load(open(p, encoding="utf-8"))
            with open(p, encoding="utf-8") as f:
                return [line.rstrip("\n") for line in f]
    return None


class Translator:
    def __init__(self, model_path: str, device: str = "cuda", device_index: int = 0, compute_type: str = "default",
                 use_cuda_graph: bool = True, max_positions: int = 512):
        if device not in ("cuda", "auto"):
            raise ValueError("ctranslate2_b200 runs on device='cuda' only (no CPU fallback)")
        if compute_type not in _COMPUTE:
            raise ValueError(f"Invalid compute type: {compute_type}")
        if not os.path.exists(os.path.join(model_path, "model.bin")):
            raise RuntimeError("Unable to open file 'model.bin' in model '%s'" % model_path)
        self.model_path = model_path
        cfg_path = os.path.join(model_path, "config.json")
        self._config = json.load(open(cfg_path)) if os.path.exists(cfg_path) else {}
        shared = _load_vocabulary(model_path, "shared_vocabulary")
        self._source = shared or _load_vocabulary(model_path, "source_vocabulary")
        self._target = shared or _load_vocabulary(model_path, "target_vocabulary")
        if self._source is None or self._target is None:
            raise RuntimeError("Cannot load the vocabulary from the model directory")
        self._src_to_id = {t: i for i, t in enumerate(self._source)}
        self._tgt_to_id = {t: i for i, t in enumerate(self._target)}
        dtype, weight_type = _COMPUTE[compute_type]
        if dtype is None:
            # "default" keeps the stored types: an int8 model with float32 norms / biases runs as int8_float32
            dtype = _FLOAT_OF_WEIGHTS.get(translator_summary(model_path)["weights"], _F32)
            if compute_type == "auto" and dtype == _F32:
                dtype = _F16
        self.compute_type = compute_type
        cfg = GeneratorConfig(device_index, dtype, 0, max_positions, 0, 1, int(use_cuda_graph), 0, weight_type)
        L = lib()
        L.ct2b200_translator_open.restype = ctypes.c_void_p
        self._h = L.ct2b200_translator_open(model_path.encode(), ctypes.byref(cfg))
        if not self._h:
            raise RuntimeError(L.ct2b200_last_error().decode())

    def __del__(self):
        self.close()

    def close(self):
        if getattr(self, "_h", None):
            lib().ct2b200_translator_close(ctypes.c_void_p(self._h))
            self._h = None

    # -- vocabulary (ctranslate2::Vocabulary, src/vocabulary.cc) -------------------------
    @property
    def unk_token(self):
        return self._config.get("unk_token", "<unk>")

    @property
    def bos_token(self):
        return self._config.get("bos_token", "<s>")

    @property
    def eos_token(self):
        return self._config.get("eos_token", "</s>")

    def source_ids(self, tokens: Sequence[str]) -> List[int]:
        """Vocabulary::to_ids with the model's add_source_bos / add_source_eos (sequence_to_sequence.cc:144-166)."""
        unk = self._src_to_id.get(self.unk_token, 0)
        ids = [self._src_to_id.get(t, unk) for t in tokens]
        if self._config.get("add_source_bos", False):
            ids = [self._src_to_id[self.bos_token]] + ids
        if self._config.get("add_source_eos", False):
            ids = ids + [self._src_to_id[self.eos_token]]
        return ids

    def info(self):
        v = [ctypes.c_int() for _ in range(6)]
        wb = ctypes.c_int64()
        check(lib().ct2b200_translator_info(ctypes.c_void_p(self._h), *[ctypes.byref(x) for x in v], ctypes.byref(wb)))
        return dict(encoder_layers=v[0].value, decoder_layers=v[1].value, num_heads=v[2].value, d_model=v[3].value,
                    source_vocab=v[4].value, target_vocab=v[5].value, weight_bytes=wb.value)

    # -- API ----------------------------------------------------------------------------
    def translate_batch(self, source, target_prefix=None, *, beam_size: int = 2, patience: float = 1.0,
                        num_hypotheses: int = 1, length_penalty: float = 1.0, max_decoding_length: int = 256,
                        min_decoding_length: int = 1, return_scores: bool = False, return_end_token: bool = False,
                        end_token: Union[None, str, Sequence[str], Sequence[int]] = None,
                        **unsupported) -> List[TranslationResult]:
        """source: list of token-string lists (looked up in the source vocabulary, special tokens added as the model asks)
        or list of id lists (taken as they are)."""
        if target_prefix is not None and any(len(p) for p in target_prefix):
            raise ValueError("target_prefix is not supported by this engine")
        for k, v in unsupported.items():
            if k not in _NEUTRAL:
                raise ValueError(f"unknown translation option: {k}")
            if not _neutral(k, v):
                raise ValueError(f"unsupported translation option: {k}={v!r} (this engine implements the default "
                                 f"{_NEUTRAL[k]!r} only)")
        if max_decoding_length == 0 or min_decoding_length > max_decoding_length:
            raise ValueError("max_decoding_length must be > 0 and min_decoding_length must be <= max_decoding_length")
        rows = [list(r) for r in source]
        if not rows:
            return []
        rows = [self.source_ids(r) if (r and isinstance(r[0], str)) else [int(i) for i in r] for r in rows]
        # an empty source (even with its special tokens) yields an empty translation (sequence_to_sequence.cc:288-303)
        keep = [b for b, r in enumerate(rows) if len(r) > 0]
        results: List[Optional[TranslationResult]] = [None] * len(rows)
        for b in range(len(rows)):
            if b not in keep:
                results[b] = TranslationResult([[] for _ in range(num_hypotheses)], [[] for _ in range(num_hypotheses)],
                                               [0.0] * num_hypotheses if return_scores else [])
        if keep:
            sub = [rows[b] for b in keep]
            ids, lens, scores = self.translate_ids(sub, beam_size=beam_size, patience=patience, num_hypotheses=num_hypotheses,
                                                   length_penalty=length_penalty, max_decoding_length=max_decoding_length,
                                                   min_decoding_length=min_decoding_length, return_end_token=return_end_token,
                                                   end_token=end_token)
            for j, b in enumerate(keep):
                hyp_ids = [ids[j, h, :lens[j, h]].tolist() for h in range(num_hypotheses) if lens[j, h] >= 0]
                results[b] = TranslationResult([[self._target[i] for i in h] for h in hyp_ids], hyp_ids,
                                               [float(scores[j, h]) for h in range(len(hyp_ids))] if return_scores else [])
        return results

    def _end_ids(self, end_token) -> List[int]:
        if end_token is None:
            end_token = self.eos_token
        if isinstance(end_token, str):
            return [self._tgt_to_id[end_token]]
        if len(end_token) and isinstance(end_token[0], str):
            return [self._tgt_to_id[t] for t in end_token]
        return [int(e) for e in end_token]

    def translate_ids(self, rows, *, beam_size=2, patience=1.0, num_hypotheses=1, length_penalty=1.0, max_decoding_length=256,
                      min_decoding_length=1, return_end_token=False, end_token=None, start_id: Optional[int] = None):
        """ids in, ids out: (ids [batch, num_hypotheses, max_decoding_length], lens, scores [batch, num_hypotheses])."""
        B = len(rows)
        lens = np.array([len(r) for r in rows], np.int32)
        S = int(lens.max())
        src = np.zeros((B, S), np.int32)
        for b, r in enumerate(rows):
            src[b, :len(r)] = r
        if start_id is None:
            start = self._config.get("decoder_start_token", "<s>")
            if start is None:
                raise ValueError("this model has no decoder start token: a target prefix would be required")
            start_id = self._tgt_to_id[start]
        end_ids = np.array(self._end_ids(end_token), np.int32)
        out = np.empty((B, num_hypotheses, max_decoding_length), np.int32)
        out_lens = np.empty((B, num_hypotheses), np.int32)
        scores = np.zeros((B, num_hypotheses), np.float32)
        p = ctypes.c_void_p
        check(lib().ct2b200_translate_batch(
            p(self._h), src.ctypes.data_as(p), lens.ctypes.data_as(p), ctypes.c_int64(B), ctypes.c_int64(S), int(beam_size),
            ctypes.c_float(patience), ctypes.c_float(length_penalty), ctypes.c_int64(max_decoding_length),
            ctypes.c_int64(min_decoding_length), int(num_hypotheses), ctypes.c_int32(start_id), end_ids.ctypes.data_as(p),
            int(end_ids.size), int(return_end_token), out.ctypes.data_as(p), out_lens.ctypes.data_as(p),
            scores.ctypes.data_as(p)))
        return out, out_lens, scores

    def encode(self, rows) -> np.ndarray:
        """TransformerEncoder output [batch, max_len, d_model] float32 (padded positions unspecified)."""
        B = len(rows)
        lens = np.array([len(r) for r in rows], np.int32)
        S = int(lens.max())
        src = np.zeros((B, S), np.int32)
        for b, r in enumerate(rows):
            src[b, :len(r)] = r
        d = self.info()["d_model"]
        mem = np.empty((B, S, d), np.float32)
        p = ctypes.c_void_p
        check(lib().ct2b200_translator_encode(p(self._h), src.ctypes.data_as(p), lens.ctypes.data_as(p), ctypes.c_int64(B),
                                              ctypes.c_int64(S), mem.ctypes.data_as(p)))
        return mem

    def bench(self, batch: int, source_len: int, beam_size: int, steps: int, warmup: int):
        enc, dec, n = ctypes.c_float(), ctypes.c_float(), ctypes.c_int64()
        check(lib().ct2b200_bench_translate(ctypes.c_void_p(self._h), ctypes.c_int64(batch), ctypes.c_int64(source_len),
                                            int(beam_size), ctypes.c_int64(steps), ctypes.c_int64(warmup), ctypes.byref(enc),
                                            ctypes.byref(dec), ctypes.byref(n)))
        return enc.value, dec.value, n.value
