"""`ctranslate2.models.Whisper` for Device::CUDA on H100, on top of the C-ABI engine (include/ct2b200.h, Whisper section).

Mirrors python/cpp/whisper.cc / include/ctranslate2/models/whisper.h: `encode(features)`, `generate(features, prompts, ...)`
with the WhisperOptions of whisper.h:11-60, `detect_language(features)` and `align(features, start_sequence, text_tokens,
num_frames, median_filter_width)`.  Vocabulary lookups and the model's config.json (suppress_ids, suppress_ids_begin,
lang_ids, alignment_heads) are handled here, as WhisperReplica does (src/models/whisper.cc:61-92, 311-323, 440-448, 599-602).  Served prompts:
previous-text tokens, `<|startoftranscript|>` and the task tokens (no text after them); the timestamp rules
(whisper.cc:742-860) run on the device unless the prompt ends with `<|notimestamps|>`."""
from __future__ import annotations

import ctypes
import json
import os
from dataclasses import dataclass, field
from typing import List, Sequence, Tuple, Union

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


@dataclass
class WhisperAlignmentResult:
    alignments: List[Tuple[int, int]]
    text_token_probs: List[float]


_NO_ALIGNMENT_HEADS = ("The model configuration does not contain the field 'alignment_heads' which lists the cross-attention "
                       "heads that are highly correlated to the word-level timing. Please reconvert this model with the "
                       "current version of ctranslate2.")


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
        enc, dec = ctypes.c_int64(), ctypes.c_int64()
        check(lib().ct2b200_translator_positions(ctypes.c_void_p(self._h), ctypes.byref(enc), ctypes.byref(dec)))
        self.decoder_positions = dec.value

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
        """Whisper::generate.  sampling_topk != 1 with sampling_temperature != 0 selects random sampling (decoding.cc:1067-1074):
        beam_size must be 1, and each entry returns num_hypotheses (<= 32) independent samples, best first; the draws follow
        set_random_seed.  Otherwise the search is deterministic and the sampling options have no effect."""
        if repetition_penalty != 1 or no_repeat_ngram_size != 0 or return_logits_vocab:
            raise ValueError("this engine implements the default repetition_penalty, no_repeat_ngram_size and "
                             "return_logits_vocab only")
        sampling_topk, sampling_temperature = int(sampling_topk), float(sampling_temperature)
        if sampling_topk < 0 or sampling_temperature < 0:
            raise ValueError("sampling_topk and sampling_temperature must be >= 0")
        sampling = sampling_topk != 1 and sampling_temperature != 0
        if sampling and sampling_topk > self.vocab_size:         # checked by RandomSampler::sample only (sampling.cc:53-58)
            raise ValueError("sampling_topk option (%d) is greater than the vocabulary size (%d)" % (sampling_topk, self.vocab_size))
        if sampling and beam_size != 1:
            raise ValueError("random sampling with beam_size > 1 (sampled beam search) is not supported: use beam_size=1")
        if sampling and not 1 <= num_hypotheses <= 32:
            raise ValueError("num_hypotheses must be in [1, 32] when sampling")
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
        args = [p(self._h), f.ctypes.data_as(p), ctypes.c_int64(B), ctypes.c_int64(T), pr.ctypes.data_as(p), ctypes.c_int64(P),
                int(beam_size), ctypes.c_float(patience), ctypes.c_float(length_penalty), ctypes.c_int64(max_length),
                int(num_hypotheses), sup.ctypes.data_as(p), int(sup.size), beg.ctypes.data_as(p), int(beg.size),
                ctypes.c_int32(self.sot_id), ctypes.c_int32(self.eot_id), ctypes.c_int32(self.no_speech_id),
                ctypes.c_int32(self.no_timestamps_id), int(max_initial_timestamp_index)]
        outs = [out.ctypes.data_as(p), lens.ctypes.data_as(p), scores.ctypes.data_as(p),
                nsp.ctypes.data_as(p) if return_no_speech_prob else None]
        if sampling:
            check(lib().ct2b200_whisper_generate_sampling(*args, sampling_topk, ctypes.c_float(sampling_temperature), *outs))
        else:
            check(lib().ct2b200_whisper_generate(*args, *outs))
        results = []
        for b in range(B):
            ids = [out[b, h, :lens[b, h]].tolist() for h in range(num_hypotheses) if lens[b, h] >= 0]
            results.append(WhisperGenerationResult([[self._tokens[i] for i in s] for s in ids], ids,
                                                   [float(scores[b, h]) for h in range(len(ids))] if return_scores else [],
                                                   float(nsp[b]) if return_no_speech_prob else 0.0))
        return results

    def detect_language(self, features) -> List[List[Tuple[str, float]]]:
        """WhisperReplica::detect_language (whisper.cc:584-652): per entry, (language token, probability) pairs over
        config.json's lang_ids, most probable first (a stable sort: ties keep the lang_ids order)."""
        if not self.is_multilingual:
            raise RuntimeError("detect_language can only be called on multilingual models")
        f = self._features(features)
        B, _, T = f.shape
        if B == 0:
            return []
        lang_ids = np.ascontiguousarray(np.array([int(x) for x in self._config["lang_ids"]], np.int32))
        if lang_ids.min() < 0 or lang_ids.max() >= self.vocab_size:
            raise ValueError("lang_ids hold ids outside the vocabulary")
        probs = np.empty((B, lang_ids.size), np.float32)
        p = ctypes.c_void_p
        check(lib().ct2b200_whisper_detect_language(p(self._h), f.ctypes.data_as(p), ctypes.c_int64(B), ctypes.c_int64(T),
                                                    ctypes.c_int32(self.sot_id), lang_ids.ctypes.data_as(p), int(lang_ids.size),
                                                    probs.ctypes.data_as(p)))
        return [sorted(((self._tokens[int(i)], float(x)) for i, x in zip(lang_ids, row)), key=lambda e: -e[1]) for row in probs]

    def align(self, features, start_sequence: Sequence[Union[int, str]], text_tokens: Sequence[Sequence[Union[int, str]]],
              num_frames: Union[int, Sequence[int]], median_filter_width: int = 7) -> List[WhisperAlignmentResult]:
        """WhisperReplica::align (whisper.cc:424-582): word-level timings.  Every entry is start_sequence +
        <|notimestamps|> + text + <|endoftext|>; `alignments` are the (text index, time index) pairs of the DTW path through
        the alignment heads' cross-attention, `text_token_probs` the probability of each text token (SoftMax over the text
        vocabulary [0, <|endoftext|>)).  num_frames: input frames of each entry (one int for all)."""
        return self._align(features, start_sequence, text_tokens, num_frames, median_filter_width)[0]

    def _align(self, features, start_sequence, text_tokens, num_frames, median_filter_width, return_matrix=False):
        """align, and with return_matrix the DTW input of every entry: [batch, max_text + 1, (frames + 1) / 2] f32."""
        ids = lambda seq: [self._ids[t] if isinstance(t, str) else int(t) for t in seq]   # noqa: E731
        texts = [ids(t) for t in text_tokens]
        if not texts:
            return [], None
        B = len(texts)
        frames = [int(num_frames)] * B if isinstance(num_frames, (int, np.integer)) else [int(x) for x in num_frames]
        if len(frames) != B:
            raise ValueError("Invalid batch size for argument num_frames")
        heads = self._config.get("alignment_heads")
        if heads is None:
            raise RuntimeError(_NO_ALIGNMENT_HEADS)
        heads = [(int(layer), int(head)) for layer, head in heads]
        if not heads:
            raise ValueError("alignment_heads is empty")
        width = int(median_filter_width)
        if width > 1 and (width % 2 == 0 or width > 129):
            raise ValueError("median_filter_width must be odd and at most 129 (or <= 1 for no filter)")
        f = self._features(features)
        if f.shape[0] != B:
            raise ValueError("one text per batch entry is required")
        start = ids(start_sequence)
        if not start:
            raise ValueError("start_sequence must not be empty")
        for seq in [start] + texts:
            if any(i < 0 or i >= self.vocab_size for i in seq):
                raise ValueError("token id out of range [0, %d)" % self.vocab_size)
        longest = len(start) + max(len(t) for t in texts) + 2
        if longest > self.decoder_positions:
            raise ValueError("start_sequence + text + 2 special tokens need %d positions; the decoder has %d"
                             % (longest, self.decoder_positions))
        S = (f.shape[2] + 1) // 2
        if any(n < 0 or n // 2 > S for n in frames):
            raise ValueError("num_frames must be in [0, %d] (the frames of the features)" % (2 * S))
        T = f.shape[2]
        Nt = max(len(t) for t in texts)
        text = np.zeros((B, max(Nt, 1)), np.int32)
        for b, t in enumerate(texts):
            text[b, :len(t)] = t
        lens = np.array([len(t) for t in texts], np.int32)
        st = np.array(start, np.int32)
        nf = np.array(frames, np.int32)
        hd = np.ascontiguousarray(np.array(heads, np.int32).reshape(-1, 2))
        max_path = Nt + 1 + S
        path = np.zeros((B, max_path, 2), np.int32)
        path_lens = np.zeros(B, np.int32)
        probs = np.zeros((B, max(Nt, 1)), np.float32)
        matrix = np.zeros((B, Nt + 1, S), np.float32) if return_matrix else None
        p = ctypes.c_void_p
        check(lib().ct2b200_whisper_align(
            p(self._h), f.ctypes.data_as(p), ctypes.c_int64(B), ctypes.c_int64(T), st.ctypes.data_as(p), ctypes.c_int64(st.size),
            text.ctypes.data_as(p), lens.ctypes.data_as(p), ctypes.c_int64(Nt), nf.ctypes.data_as(p), width,
            hd.ctypes.data_as(p), int(hd.shape[0]), ctypes.c_int32(self.no_timestamps_id), ctypes.c_int32(self.eot_id),
            path.ctypes.data_as(p), path_lens.ctypes.data_as(p), probs.ctypes.data_as(p),
            matrix.ctypes.data_as(p) if return_matrix else None))
        return [WhisperAlignmentResult([(int(i), int(j)) for i, j in path[b, :path_lens[b]]],
                                       [float(x) for x in probs[b, :lens[b]]]) for b in range(B)], matrix
