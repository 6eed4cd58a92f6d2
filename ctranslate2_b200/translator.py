"""`ctranslate2.Translator` for Device::CUDA on H100, on top of the C-ABI engine (include/ct2b200.h, encoder-decoder path).

Mirrors python/cpp/translator.cc / include/ctranslate2/translator.h: `translate_batch(source, ...)` with the
TranslationOptions of include/ctranslate2/translation.h, and `score_batch(source, target, ...)`.  Token strings <-> ids (ctranslate2::Vocabulary: source /
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
from .generator import _COMPUTE, _F16, _F32, ScoringResult, _is_neutral, _non_negative_int, _rebatch, _truncate  # noqa: F401

_FLOAT_OF_WEIGHTS = {"float16": 1, "bfloat16": 2}


@dataclass
class TranslationResult:
    hypotheses: List[List[str]]
    hypotheses_ids: List[List[int]]
    scores: List[float] = field(default_factory=list)
    attention: List[List[List[float]]] = field(default_factory=list)


def translator_summary(model_path: str) -> dict:
    """Geometry of an encoder-decoder model directory (host only, no GPU needed; ct2b200_translator_summary)."""
    buf = ctypes.create_string_buffer(2048)
    check(lib().ct2b200_translator_summary(model_path.encode(), buf, ctypes.c_size_t(len(buf))))
    return json.loads(buf.value.decode())


# TranslationOptions (include/ctranslate2/translation.h:14-98) this engine does not implement, with the only value it accepts
_NEUTRAL = {
    "prefix_bias_beta": 0, "sampling_topk": 1, "sampling_topp": 1, "sampling_temperature": 1,
    "use_vmap": False, "return_logits_vocab": False, "return_alternatives": False,
    "min_alternative_expansion_prob": 0, "callback": None, "asynchronous": False,
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


# The engine's limits on the SuppressTokens / SuppressSequences tables (kMaxSuppressSequences, csrc/host/translator.h): larger
# tables are refused, never truncated
MAX_SUPPRESS_SEQUENCES = 4096
MAX_SUPPRESS_SEQUENCE_TOKENS = 65536


def _processor_options(repetition_penalty, no_repeat_ngram_size, disable_ids, suppress_sequences, vocab_size: int):
    """Checks the logits processors in id form (types as the reference's Python bindings take them) and returns
    (penalty, n, disabled ids, sequence offsets, sequence ids) for ct2b200_translate_batch_processors."""
    if isinstance(repetition_penalty, (bool, np.bool_)) or not isinstance(repetition_penalty, (int, float, np.integer, np.floating)):
        raise ValueError(f"repetition_penalty must be a number, not {type(repetition_penalty).__name__}")
    penalty = float(repetition_penalty)
    if not (np.isfinite(penalty) and penalty > 0):
        raise ValueError(f"repetition_penalty must be positive and finite, got {repetition_penalty!r}")
    if isinstance(no_repeat_ngram_size, (bool, np.bool_)) or not isinstance(no_repeat_ngram_size, (int, np.integer)) \
            or no_repeat_ngram_size < 0:
        raise ValueError(f"no_repeat_ngram_size must be a non-negative int, got {no_repeat_ngram_size!r}")
    ids = [_token_id(i, "disabled id", vocab_size) for i in disable_ids]
    offsets, flat = [0], []
    for seq in suppress_sequences:
        if isinstance(seq, (str, bytes)) or not hasattr(seq, "__len__"):
            raise ValueError(f"suppress_sequences must hold token sequences, not {type(seq).__name__}")
        flat += [_token_id(i, "suppressed sequence id", vocab_size) for i in seq]
        offsets.append(len(flat))
    if len(ids) > MAX_SUPPRESS_SEQUENCES or len(offsets) - 1 > MAX_SUPPRESS_SEQUENCES or len(flat) > MAX_SUPPRESS_SEQUENCE_TOKENS:
        raise ValueError(f"at most {MAX_SUPPRESS_SEQUENCES} disabled ids, {MAX_SUPPRESS_SEQUENCES} suppressed sequences and "
                         f"{MAX_SUPPRESS_SEQUENCE_TOKENS} suppressed tokens in all")
    return penalty, int(no_repeat_ngram_size), ids, (offsets if len(offsets) > 1 else []), flat


def _coverage_penalty(coverage_penalty) -> float:
    if isinstance(coverage_penalty, (bool, np.bool_)) or not isinstance(coverage_penalty, (int, float, np.integer, np.floating)):
        raise ValueError(f"coverage_penalty must be a number, not {type(coverage_penalty).__name__}")
    if not np.isfinite(float(coverage_penalty)):
        raise ValueError(f"coverage_penalty must be finite, got {coverage_penalty!r}")
    return float(coverage_penalty)


def _flag(name: str, value) -> bool:
    if not isinstance(value, (bool, np.bool_)):
        raise ValueError(f"{name} must be a bool, not {type(value).__name__}")
    return bool(value)


def _token_id(x, what: str, vocab_size: int) -> int:
    if isinstance(x, (bool, np.bool_)) or not isinstance(x, (int, np.integer)):
        raise ValueError(f"{what} must be an int, not {type(x).__name__}")
    if not 0 <= x < vocab_size:
        raise ValueError(f"{what} {x} is outside the target vocabulary [0, {vocab_size})")
    return int(x)


def _replace_unknowns(hypothesis: List[str], source: List[str], attention: np.ndarray, unk_token: str) -> None:
    """replace_unknown_tokens (sequence_to_sequence.cc:288-302): each unknown token becomes the source token of its
    attention row's first maximum."""
    for t, token in enumerate(hypothesis):
        if token == unk_token and source:
            hypothesis[t] = source[int(np.argmax(attention[t]))]


def _load_vocabulary(model_path: str, name: str) -> Optional[List[str]]:
    for ext in (".json", ".txt"):
        p = os.path.join(model_path, name + ext)
        if os.path.exists(p):
            if ext == ".json":
                return json.load(open(p, encoding="utf-8"))
            with open(p, encoding="utf-8") as f:
                return [line.rstrip("\n") for line in f]
    return None


def _index(x, side: str, row: int) -> int:
    if isinstance(x, (bool, np.bool_)) or not isinstance(x, (int, np.integer)):
        raise ValueError(f"score_batch: {side} {row} mixes token ids with {type(x).__name__} values")
    return int(x)


def _check_range(rows, vocab_size: int, side: str) -> None:
    for b, row in enumerate(rows):
        bad = [i for i in row if not 0 <= i < vocab_size]
        if bad:
            raise ValueError(f"score_batch: {side} id {bad[0]} of pair {b} is outside the vocabulary [0, {vocab_size})")


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
        enc_pos, dec_pos = ctypes.c_int64(), ctypes.c_int64()
        check(L.ct2b200_translator_positions(ctypes.c_void_p(self._h), ctypes.byref(enc_pos), ctypes.byref(dec_pos)))
        self._encoder_positions, self._decoder_positions = enc_pos.value, dec_pos.value
        # the model's embedding sizes: the reference appends <unk> to a vocabulary file that lacks it (src/vocabulary.cc:46-48)
        info = self.info()
        self._src_vocab_size, self._tgt_vocab_size = info["source_vocab"], info["target_vocab"]

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
                        repetition_penalty: float = 1, no_repeat_ngram_size: int = 0, disable_unk: bool = False,
                        suppress_sequences: Optional[List[List[str]]] = None, return_attention: bool = False,
                        replace_unknowns: bool = False, coverage_penalty: float = 0,
                        **unsupported) -> List[TranslationResult]:
        """source: list of token-string lists (looked up in the source vocabulary, special tokens added as the model asks)
        or list of id lists (taken as they are).  The logits processors run on the device in every search step, on each
        beam's tokens so far: repetition_penalty (> 0) rewrites them first, then no_repeat_ngram_size, disable_unk and
        suppress_sequences (token strings of the target vocabulary; an unknown one raises ValueError, the unknown-token
        string itself is accepted) disable tokens, as do the end tokens below min_decoding_length.

        The search keeps the alignment attention of every beam on the device (the mean of the normalised cross-attention of
        the model's alignment heads) when one of these asks for it:
          * return_attention: TranslationResult.attention holds, per hypothesis, one row per token over the source tokens
            (the special tokens the model adds are left out; sequence_to_sequence.cc:395-412);
          * replace_unknowns: each unknown-token string of a hypothesis becomes the source token it attends to most (the
            first of equal maxima).  Sources given as ids have no tokens to copy: ValueError (the reference has no id
            input);
          * coverage_penalty: the GNMT coverage term beta * sum(log(min(coverage, 1))) over the attended source positions
            joins each hypothesis's final score before the hypotheses are ranked (decoding.cc:176-254)."""
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
        disable_ids, sequences = self._suppressed_ids(disable_unk, suppress_sequences)
        _processor_options(repetition_penalty, no_repeat_ngram_size, disable_ids, sequences, self._tgt_vocab_size)
        return_attention = _flag("return_attention", return_attention)
        replace_unknowns = _flag("replace_unknowns", replace_unknowns)
        coverage_penalty = _coverage_penalty(coverage_penalty)
        tokens = [list(r) for r in source]
        is_text = [bool(r) and isinstance(r[0], str) for r in tokens]
        if replace_unknowns and any(r and not t for r, t in zip(tokens, is_text)):
            raise ValueError("replace_unknowns needs the source tokens: the sources were given as ids")
        if not tokens:
            return []
        rows = [self.source_ids(r) if t else [int(i) for i in r] for r, t in zip(tokens, is_text)]
        keep_attention = return_attention or replace_unknowns
        # an empty source (even with its special tokens) yields an empty translation (sequence_to_sequence.cc:288-303)
        keep = [b for b, r in enumerate(rows) if len(r) > 0]
        results: List[Optional[TranslationResult]] = [None] * len(rows)
        for b in range(len(rows)):
            if b not in keep:
                results[b] = TranslationResult([[] for _ in range(num_hypotheses)], [[] for _ in range(num_hypotheses)],
                                               [0.0] * num_hypotheses if return_scores else [],
                                               [[] for _ in range(num_hypotheses)] if return_attention else [])
        if keep:
            sub = [rows[b] for b in keep]
            extra = dict(return_attention=True) if keep_attention else {}
            if coverage_penalty != 0:
                extra["coverage_penalty"] = coverage_penalty
            out = self.translate_ids(sub, beam_size=beam_size, patience=patience, num_hypotheses=num_hypotheses,
                                     length_penalty=length_penalty, max_decoding_length=max_decoding_length,
                                     min_decoding_length=min_decoding_length, return_end_token=return_end_token,
                                     end_token=end_token, repetition_penalty=repetition_penalty,
                                     no_repeat_ngram_size=no_repeat_ngram_size, disable_ids=disable_ids,
                                     suppress_sequences=sequences, **extra)
            ids, lens, scores = out[:3]
            for j, b in enumerate(keep):
                hyp_ids = [ids[j, h, :lens[j, h]].tolist() for h in range(num_hypotheses) if lens[j, h] >= 0]
                hyps = [[self._target[i] for i in h] for h in hyp_ids]
                attention = []
                if keep_attention:
                    attention = [self._source_attention(out[3][j, h, :len(hyp_ids[h])], len(rows[b]),
                                                        len(tokens[b]) if is_text[b] else None)
                                 for h in range(len(hyp_ids))]
                    if replace_unknowns:
                        for h, att in zip(hyps, attention):
                            _replace_unknowns(h, tokens[b], att, self.unk_token)
                results[b] = TranslationResult(hyps, hyp_ids,
                                               [float(scores[j, h]) for h in range(len(hyp_ids))] if return_scores else [],
                                               [a.tolist() for a in attention] if return_attention else [])
        return results

    def _source_attention(self, rows: np.ndarray, input_len: int, original_len: Optional[int]) -> np.ndarray:
        """The attention rows of one hypothesis over its source (sequence_to_sequence.cc:395-412): cut to the entry's input
        length, special tokens included; for token sources the columns of the model's added <s> / </s> are dropped and the
        rows zero-padded to the token count.  Id sources keep the columns of their ids."""
        rows = rows[:, :input_len]
        if original_len is None:
            return rows
        if self._config.get("add_source_bos", False):
            rows = rows[:, 1:]
        if self._config.get("add_source_eos", False):
            rows = rows[:, :-1]
        out = np.zeros((rows.shape[0], original_len), np.float32)
        n = min(original_len, rows.shape[1])
        out[:, :n] = rows[:, :n]
        return out

    def score_batch(self, source, target, *, max_batch_size: int = 0, batch_type: str = "examples",
                    max_input_length: int = 1024, offset: int = 0, asynchronous: bool = False) -> List[ScoringResult]:
        """Translator.score_batch (python/cpp/translator.cc:504-531): the log-probability of every target token given the source
        and the target prefix, one ScoringResult per (source, target) pair in request order.  Sources are token-string lists
        (looked up with the model's special tokens, as translate_batch does) or id lists (taken as they are); targets are
        token-string lists or id lists, and get the decoder start token (when the model has one) and </s> either way.  An
        empty source is a token list: it gets the model's special tokens, as in the reference, and scores 0 for every
        target token only when it is still empty.  Both
        are truncated to max_input_length tokens, the target plus one for its start token, keeping </s> (Vocabulary::to_ids).
        Results cover target tokens offset + 1 .. (ScoringOptions::offset) and end with "</s>".  Pairs are re-batched
        longest source first by max_batch_size / batch_type; the scores do not depend on the batching."""
        if asynchronous:
            raise ValueError("score_batch: asynchronous=True is not supported (results are returned, not futures)")
        max_batch_size = _non_negative_int("max_batch_size", max_batch_size)
        max_input_length = _non_negative_int("max_input_length", max_input_length)
        offset = _non_negative_int("offset", offset)
        if batch_type not in ("examples", "tokens"):
            raise ValueError(f"Invalid batch type: {batch_type}")
        sources, targets = [list(r) for r in source], [list(r) for r in target]
        if len(sources) != len(targets):
            raise ValueError(f"score_batch: {len(sources)} sources but {len(targets)} targets")
        if not sources:
            return []
        src_eos = self._src_to_id.get(self.eos_token, -1)
        tgt_eos = self._tgt_to_id[self.eos_token]
        start = self._config.get("decoder_start_token", "<s>")
        start_ids = [] if start is None else [self._tgt_to_id[start]]
        tgt_unk = self._tgt_to_id.get(self.unk_token, 0)
        src_rows, tgt_rows = [], []
        for b, (s, t) in enumerate(zip(sources, targets)):
            s = self.source_ids(s) if (not s or isinstance(s[0], str)) else [_index(x, "source", b) for x in s]
            src_rows.append(_truncate(s, max_input_length, src_eos))
            if start is None and not t:
                tgt_rows.append(None)                  # skip_scoring: nothing to score without a start token
                continue
            t = [self._tgt_to_id.get(x, tgt_unk) for x in t] if (t and isinstance(t[0], str)) else [_index(x, "target", b) for x in t]
            tgt_rows.append(_truncate(start_ids + t + [tgt_eos], max_input_length + 1 if max_input_length else 0, tgt_eos))
        _check_range(src_rows, self._src_vocab_size, "source")
        _check_range([t for t in tgt_rows if t is not None], self._tgt_vocab_size, "target")
        for b, s in enumerate(src_rows):
            if len(s) > self._encoder_positions:
                raise ValueError(f"score_batch: source {b} has {len(s)} tokens, more than the {self._encoder_positions} "
                                 "positions of the encoder's position table (lower max_input_length)")
        for b, t in enumerate(tgt_rows):
            if t is not None and len(t) - 1 > self._decoder_positions:
                raise ValueError(f"score_batch: target {b} needs {len(t) - 1} decoder positions, more than the "
                                 f"{self._decoder_positions} of the model's position table (lower max_input_length)")
        results = [ScoringResult([], []) for _ in sources]
        run = []
        for b, (s, t) in enumerate(zip(src_rows, tgt_rows)):
            if t is None:
                continue
            if not s:                                  # skip_scoring: an empty source scores 0 for every target token
                results[b] = ScoringResult([self._target_token(i) for i in t[1:]], [0.0] * (len(t) - 1))
                continue
            run.append(b)
        p = ctypes.c_void_p
        for idx in _rebatch([len(src_rows[b]) for b in run], max_batch_size, batch_type, len(run)):
            idx = [run[i] for i in idx]
            B = len(idx)
            src_lens = np.array([len(src_rows[b]) for b in idx], np.int32)
            tgt_lens = np.array([len(tgt_rows[b]) for b in idx], np.int32)
            S, T = int(src_lens.max()), int(tgt_lens.max())
            src = np.zeros((B, S), np.int32)
            tgt = np.zeros((B, T), np.int32)
            for j, b in enumerate(idx):
                src[j, :src_lens[j]] = src_rows[b]
                tgt[j, :tgt_lens[j]] = tgt_rows[b]
            out = np.zeros((B, T - 1), np.float32)
            check(lib().ct2b200_translator_score_batch(
                p(self._h), src.ctypes.data_as(p), src_lens.ctypes.data_as(p), ctypes.c_int64(B), ctypes.c_int64(S),
                tgt.ctypes.data_as(p), tgt_lens.ctypes.data_as(p), ctypes.c_int64(T), ctypes.c_int64(offset),
                out.ctypes.data_as(p)))
            for j, b in enumerate(idx):
                n = max(0, int(tgt_lens[j]) - 1 - offset)
                results[b] = ScoringResult([self._target_token(i) for i in tgt_rows[b][1 + offset:]], out[j, :n].tolist())
        return results

    def _suppressed_ids(self, disable_unk, suppress_sequences):
        """disable_unk and suppress_sequences as target ids (sequence_to_sequence.cc:341-362: Vocabulary::to_ids with
        allow_unk = false).  The reference appends the unknown token to a vocabulary file that lacks it, past the output
        layer: such an id is never produced, so there is nothing to disable and a sequence holding it never completes —
        both are left out."""
        if not isinstance(disable_unk, (bool, np.bool_)):
            raise ValueError(f"disable_unk must be a bool, not {type(disable_unk).__name__}")
        unk = self._tgt_to_id.get(self.unk_token, len(self._target))
        disable = [unk] if disable_unk and unk < self._tgt_vocab_size else []
        if suppress_sequences is None:
            return disable, []
        if isinstance(suppress_sequences, (str, bytes)) or not isinstance(suppress_sequences, (list, tuple)):
            raise ValueError("suppress_sequences must be None or a list of token lists")
        sequences = []
        for seq in suppress_sequences:
            if isinstance(seq, (str, bytes)) or not isinstance(seq, (list, tuple)):
                raise ValueError("suppress_sequences must be None or a list of token lists")
            ids = []
            for tok in seq:
                if not isinstance(tok, str):
                    raise ValueError(f"suppress_sequences holds token strings, not {type(tok).__name__}")
                if tok not in self._tgt_to_id and tok != self.unk_token:
                    raise ValueError(f"Token {tok} is not in the vocabulary")
                ids.append(self._tgt_to_id.get(tok, unk))
            if all(i < self._tgt_vocab_size for i in ids):
                sequences.append(ids)
        return disable, sequences

    def _target_token(self, i: int) -> str:
        return self._target[i] if i < len(self._target) else self.unk_token

    def _end_ids(self, end_token) -> List[int]:
        if end_token is None:
            end_token = self.eos_token
        if isinstance(end_token, str):
            return [self._tgt_to_id[end_token]]
        if len(end_token) and isinstance(end_token[0], str):
            return [self._tgt_to_id[t] for t in end_token]
        return [int(e) for e in end_token]

    def translate_ids(self, rows, *, beam_size=2, patience=1.0, num_hypotheses=1, length_penalty=1.0, max_decoding_length=256,
                      min_decoding_length=1, return_end_token=False, end_token=None, start_id: Optional[int] = None,
                      repetition_penalty=1.0, no_repeat_ngram_size=0, disable_ids=(), suppress_sequences=(),
                      return_attention=False, coverage_penalty=0.0):
        """ids in, ids out: (ids [batch, num_hypotheses, max_decoding_length], lens, scores [batch, num_hypotheses]).
        The logits processors take target ids: disable_ids are disabled at every step, suppress_sequences are id lists.
        return_attention appends the raw attention [batch, num_hypotheses, max_decoding_length, max_source_len] float32:
        row t of a hypothesis comes from the step that produced token t, zeros past its tokens and past the entry's
        length.  coverage_penalty (finite) adds the coverage term to the final scores."""
        penalty, ngram, disable_ids, seq_offsets, seq_ids = _processor_options(
            repetition_penalty, no_repeat_ngram_size, disable_ids, suppress_sequences, self._tgt_vocab_size)
        return_attention = _flag("return_attention", return_attention)
        coverage = _coverage_penalty(coverage_penalty)
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
        args = (p(self._h), src.ctypes.data_as(p), lens.ctypes.data_as(p), ctypes.c_int64(B), ctypes.c_int64(S), int(beam_size),
                ctypes.c_float(patience), ctypes.c_float(length_penalty), ctypes.c_int64(max_decoding_length),
                ctypes.c_int64(min_decoding_length), int(num_hypotheses), ctypes.c_int32(start_id), end_ids.ctypes.data_as(p),
                int(end_ids.size), int(return_end_token))
        outs = (out.ctypes.data_as(p), out_lens.ctypes.data_as(p), scores.ctypes.data_as(p))
        if return_attention or coverage != 0:
            dis = np.array(disable_ids, np.int32)
            offsets = np.array(seq_offsets, np.int32)
            flat = np.array(seq_ids, np.int32)
            attention = np.zeros((B, num_hypotheses, max_decoding_length, S), np.float32) if return_attention else None
            check(lib().ct2b200_translate_batch_attention(
                *args, ctypes.c_float(penalty), int(ngram), dis.ctypes.data_as(p), int(dis.size), flat.ctypes.data_as(p),
                offsets.ctypes.data_as(p), max(0, int(offsets.size) - 1), ctypes.c_float(coverage), *outs,
                attention.ctypes.data_as(p) if return_attention else None))
            return (out, out_lens, scores, attention) if return_attention else (out, out_lens, scores)
        if penalty == 1 and ngram == 0 and not disable_ids and not seq_offsets:
            check(lib().ct2b200_translate_batch(*args, *outs))
        else:
            dis = np.array(disable_ids, np.int32)
            offsets = np.array(seq_offsets, np.int32)
            flat = np.array(seq_ids, np.int32)
            check(lib().ct2b200_translate_batch_processors(
                *args, ctypes.c_float(penalty), int(ngram), dis.ctypes.data_as(p), int(dis.size), flat.ctypes.data_as(p),
                offsets.ctypes.data_as(p), max(0, int(offsets.size) - 1), *outs))
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
