"""`ctranslate2.Generator` for Device::CUDA on H100, on top of the C-ABI engine.

Mirrors python/cpp/generator.cc:15-96 / include/ctranslate2/generator.h: `generate_batch(start_tokens, ...)`,
`forward_batch(tokens)` and `score_batch(tokens, ...)`.  Token strings <-> ids (ctranslate2::Vocabulary, vocabulary.json) are
handled here; ids cross the boundary in HOST buffers (the engine does the host<->device copies)."""
from __future__ import annotations

import ctypes
import json
import os
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Union

import numpy as np

from ._lib import GeneratorConfig, check, lib

_F32, _F16, _BF16 = 0, 1, 2
_STORED, _INT8, _FLOAT = 0, 1, 2
# compute type -> (ct2b200_dtype of the activations or None = the model's stored float type, ct2b200_weight_type), following
# compute_type_to_data_type / resolve_compute_type of the reference (src/types.cc): "default" keeps what the model stores (an
# int8 model with float32 norms runs as int8_float32), "int8" means int8 weights with float32 activations, "auto" keeps the
# stored weights and runs float32 models in float16 (the fastest supported type).  Weights are converted at load, on the GPU.
_COMPUTE = {"default": (None, _STORED), "auto": (None, _STORED), "int8": (_F32, _INT8), "int8_float32": (_F32, _INT8),
            "int8_float16": (_F16, _INT8), "int8_bfloat16": (_BF16, _INT8), "float16": (_F16, _FLOAT),
            "bfloat16": (_BF16, _FLOAT), "float32": (_F32, _FLOAT)}
_FLOAT_IDS = {"float32": _F32, "float16": _F16, "bfloat16": _BF16}


@dataclass
class GenerationResult:
    sequences: List[List[str]]
    sequences_ids: List[List[int]]
    scores: List[float] = field(default_factory=list)


@dataclass
class ScoringResult:
    """ctranslate2.ScoringResult (include/ctranslate2/scoring.h): the scored tokens and their log-probabilities."""
    tokens: List[str]
    log_probs: List[float]


def _non_negative_int(name: str, value) -> int:
    if isinstance(value, (bool, np.bool_)) or not isinstance(value, (int, np.integer)) or value < 0:
        raise ValueError(f"{name} must be a non-negative integer")
    return int(value)


def _truncate(ids: List[int], max_length: int, eos: int) -> List[int]:
    """Vocabulary::to_ids(tokens, max_length) (src/vocabulary.cc:130-140): cut to max_length (0: no limit), keeping a final
    end token in the last position, or a final "end token, then one more token" pair in the last two."""
    if max_length == 0 or len(ids) <= max_length:
        return ids
    out = ids[:max_length]
    if ids[-1] == eos:
        out[-1] = eos
    elif ids[-2] == eos and max_length >= 2:
        out[-2:] = [eos, ids[-1]]
    return out


def _rebatch(lengths: Sequence[int], max_batch_size: int, batch_type: str, max_rows: int) -> List[List[int]]:
    """rebatch_input (src/batch_reader.cc:175-225): indices sorted longest first, split into batches of at most
    max_batch_size examples, or of at most max_batch_size tokens counting the padding (rows x longest length; the first row
    of a batch is always taken), 0 = no limit.  Every batch also has at most max_rows rows."""
    order = sorted(range(len(lengths)), key=lambda i: -lengths[i])
    batches: List[List[int]] = []
    for i in order:
        if batches:
            cur = batches[-1]
            rows = len(cur) + 1
            fits = rows <= max_rows
            if max_batch_size > 0:
                size = rows * max(lengths[j] for j in cur + [i]) if batch_type == "tokens" else rows
                fits = fits and size <= max_batch_size
            if fits:
                cur.append(i)
                continue
        batches.append([i])
    return batches


def model_summary(model_path: str) -> dict:
    """What the engine finds in a CTranslate2 model directory (host only, no GPU needed): spec, binary version, decoder
    geometry and the storage type of the linear layers (ct2b200_model_summary)."""
    buf = ctypes.create_string_buffer(2048)
    check(lib().ct2b200_model_summary(model_path.encode(), buf, ctypes.c_size_t(len(buf))))
    return json.loads(buf.value.decode())


# GenerationOptions (include/ctranslate2/generation.h:14-78) this engine does not implement, with the only value of each it
# accepts (the reference's default, under which the option is a no-op); everything else raises instead of being ignored.
_NEUTRAL_OPTIONS = {
    "patience": 1, "repetition_penalty": 1, "no_repeat_ngram_size": 0, "disable_unk": False, "suppress_sequences": None,
    "sampling_topp": 1, "sampling_temperature": 1, "num_hypotheses": 1, "return_logits_vocab": False,
    "return_alternatives": False, "min_alternative_expansion_prob": 0, "static_prompt": None, "cache_static_prompt": True,
    "callback": None, "asynchronous": False, "max_batch_size": 0, "batch_type": "examples",
}


def _is_neutral(name, value) -> bool:
    neutral = _NEUTRAL_OPTIONS[name]
    if neutral is None:                       # list-valued options: None or empty
        return value is None or (hasattr(value, "__len__") and len(value) == 0)
    if isinstance(neutral, bool):             # True == 1 in Python: compare flags as flags, not as numbers
        return isinstance(value, (bool, np.bool_)) and bool(value) == neutral
    if isinstance(neutral, str):
        return value == neutral
    return not isinstance(value, (bool, np.bool_)) and isinstance(value, (int, float, np.integer, np.floating)) \
        and float(value) == float(neutral)


def _check_options(options: dict, max_length: int, min_length: int) -> None:
    for k, v in options.items():
        if k not in _NEUTRAL_OPTIONS:
            raise ValueError(f"unknown generation option: {k}")
        if not _is_neutral(k, v):
            raise ValueError(f"unsupported generation option: {k}={v!r} (this engine implements the default "
                             f"{_NEUTRAL_OPTIONS[k]!r} only)")
    if max_length == 0 or min_length > max_length:
        # decoding.cc:1035-1040
        raise ValueError("max_length must be > 0 and min_length must be <= max_length")


def _validate_ids(rows, vocab_size: int) -> None:
    """Token ids index the embedding table on the device (layers::Embeddings gathers rows, common.cc:64-81): the C-ABI takes
    them as given, so the range check lives here, where ids can come from the caller instead of the vocabulary."""
    for b, row in enumerate(rows):
        a = np.asarray(row, dtype=np.int64)
        if a.size and (int(a.min()) < 0 or int(a.max()) >= vocab_size):
            bad = int(a[(a < 0) | (a >= vocab_size)][0])
            raise ValueError(f"token id {bad} of row {b} is outside the vocabulary [0, {vocab_size})")


class Generator:
    def __init__(self, model_path: str, device: str = "cuda", device_index: int = 0, compute_type: str = "default",
                 max_batch_size: int = 32, max_length: int = 4096, use_cuda_graph: bool = True, gemm_impl: int = 0,
                 tensor_parallel: bool = False, tp_rank: Optional[int] = None, tp_size: Optional[int] = None,
                 tp_group=None):
        """tensor_parallel=True (ctranslate2.Generator(..., tensor_parallel=True)): one process per GPU; rank and
        size default to torch.distributed's, whose default (or `tp_group`) group also carries the one-time exchange
        of the CUDA IPC handles.  Every rank must then make the same calls with the same inputs."""
        if device not in ("cuda", "auto"):
            raise ValueError("ctranslate2_b200 runs on device='cuda' only (no CPU fallback)")
        if compute_type not in _COMPUTE:
            raise ValueError(f"Invalid compute type: {compute_type}")
        self.model_path = model_path
        if not os.path.exists(os.path.join(model_path, "model.bin")):
            # same failure class as models::Model::load (std::runtime_error)
            raise RuntimeError("Unable to open file 'model.bin' in model '%s'" % model_path)
        vocab_path = os.path.join(model_path, "vocabulary.json")
        if os.path.exists(vocab_path):
            self._tokens = json.load(open(vocab_path))
        else:
            with open(os.path.join(model_path, "vocabulary.txt")) as f:
                self._tokens = [l.rstrip("\n") for l in f]
        self._token_to_id = None
        cfg_path = os.path.join(model_path, "config.json")
        self._config = json.load(open(cfg_path)) if os.path.exists(cfg_path) else {}
        self.tp_rank, self.tp_size = 0, 1
        if tensor_parallel:
            from .parallel import default_rank_and_size
            self.tp_rank, self.tp_size = default_rank_and_size(tp_rank, tp_size, tp_group)
        dtype, weight_type = _COMPUTE[compute_type]
        if dtype is None:
            summary = model_summary(model_path)
            dtype = _F16 if summary["weights"].startswith("awq") else _FLOAT_IDS[summary["float_type"]]
            if compute_type == "auto" and dtype == _F32:
                dtype = _F16
        self.compute_type = compute_type
        cfg = GeneratorConfig(device_index, dtype, max_batch_size, max_length, self.tp_rank,
                              self.tp_size, int(use_cuda_graph), gemm_impl, weight_type)
        self._h = lib().ct2b200_generator_open(model_path.encode(), ctypes.byref(cfg))
        if not self._h:
            raise RuntimeError(lib().ct2b200_last_error().decode())
        self.max_batch_size, self.max_length = max_batch_size, max_length
        self.vocab_size = lib().ct2b200_generator_vocab_size(ctypes.c_void_p(self._h))
        if self.tp_size > 1:
            from .parallel import exchange_handles
            self.tp_connect(exchange_handles(self.tp_handle(), self.tp_rank, self.tp_size, tp_group))

    # -- tensor parallel bootstrap ------------------------------------------------------
    def tp_handle(self) -> bytes:
        buf = ctypes.create_string_buffer(64)
        check(lib().ct2b200_generator_tp_handle(ctypes.c_void_p(self._h), buf))
        return buf.raw

    def tp_connect(self, handles: Sequence[bytes]):
        blob = b"".join(handles)
        if len(blob) != 64 * self.tp_size:
            raise ValueError("tp_connect needs one 64-byte handle per rank")
        check(lib().ct2b200_generator_tp_connect(ctypes.c_void_p(self._h), blob, len(handles)))

    def __del__(self):
        self.close()

    def close(self):
        if getattr(self, "_h", None):
            lib().ct2b200_generator_close(ctypes.c_void_p(self._h))
            self._h = None

    # -- vocabulary ---------------------------------------------------------------------
    def _ids(self, tokens: Sequence[str]) -> List[int]:
        if self._token_to_id is None:
            self._token_to_id = {t: i for i, t in enumerate(self._tokens)}
        unk = self._token_to_id.get(self._config.get("unk_token", "<unk>"), 0)
        return [self._token_to_id.get(t, unk) for t in tokens]

    def _end_ids(self, end_token) -> List[int]:
        if end_token is None:
            end_token = self._config.get("eos_token", "</s>")
        if isinstance(end_token, str):
            return self._ids([end_token])
        if len(end_token) and isinstance(end_token[0], str):
            return self._ids(end_token)
        return [int(e) for e in end_token]

    # -- API ----------------------------------------------------------------------------
    def generate_batch(self, start_tokens, max_length: int = 512, min_length: int = 0, beam_size: int = 1,
                       sampling_topk: int = 1, include_prompt_in_result: bool = False,
                       end_token: Union[None, str, Sequence[str], Sequence[int]] = None,
                       return_end_token: bool = False, return_scores: bool = False, length_penalty: float = 1.0,
                       **unsupported) -> List[GenerationResult]:
        """start_tokens: list of token-string lists, or list of id lists / int array [batch, len]."""
        if sampling_topk != 1:
            raise ValueError("this engine implements best-candidate search (sampling_topk=1)")
        if beam_size < 1:
            raise ValueError("The beam size must be > 0")
        if include_prompt_in_result:
            raise ValueError("include_prompt_in_result=True forces the prompt through the decode loop token by "
                             "token (decoding.cc:21-67); pass False (docs/performance.md)")
        patience = unsupported.pop("patience", 1) if beam_size > 1 else 1
        num_hypotheses = unsupported.pop("num_hypotheses", 1) if beam_size > 1 else 1
        # max_batch_size of the call (python/cpp/generator.cc: inputs beyond it are sorted by length and split into chunks of
        # that many examples); batch_type "tokens" is not implemented
        request_cap = unsupported.pop("max_batch_size", 0)
        if isinstance(request_cap, bool) or not isinstance(request_cap, (int, np.integer)) or request_cap < 0:
            raise ValueError("max_batch_size must be a non-negative integer")
        _check_options(unsupported, max_length, min_length)
        rows = [list(r) for r in start_tokens]
        if not rows:
            return []                       # an empty batch is an empty result (replica_pool.h: no job is posted)
        if rows[0] and isinstance(rows[0][0], str):
            rows = [self._ids(r) for r in rows]
        _validate_ids(rows, self.vocab_size)
        B = len(rows)
        cap = self.max_batch_size // beam_size
        if request_cap > 0:
            cap = min(cap, int(request_cap))
        if B > cap >= 1:
            # A request larger than the arena: the reference's replica pool re-batches it by max_batch_size, longest examples
            # first, and returns the results in request order (src/batch_reader.cc rebatch_input / load_examples).  Every row
            # equals the row decoded alone, so the split does not change any result.
            if beam_size > 1 and len({len(r) for r in rows}) > 1:
                raise ValueError("beam search needs prompts of equal length")
            order = sorted(range(B), key=lambda i: -len(rows[i]))
            results: List[Optional[GenerationResult]] = [None] * B
            for c in range(0, B, cap):
                idx = order[c:c + cap]
                sub = self.generate_batch([rows[i] for i in idx], max_length=max_length, min_length=min_length,
                                          beam_size=beam_size, end_token=end_token, return_end_token=return_end_token,
                                          return_scores=return_scores, length_penalty=length_penalty,
                                          **({"patience": patience, "num_hypotheses": num_hypotheses} if beam_size > 1 else {}))
                for i, r in zip(idx, sub):
                    results[i] = r
            return results
        lens = np.array([len(r) for r in rows], np.int32)
        P = int(lens.max())
        ids = np.zeros((B, P), np.int32)
        for b, r in enumerate(rows):
            ids[b, :len(r)] = r
        end_ids = np.array(self._end_ids(end_token), np.int32)
        if beam_size > 1:
            # BeamSearch::search on the device (ct2b200_generate_batch_beam): prompts of equal length
            if int(lens.min()) != P:
                raise ValueError("beam search needs prompts of equal length")
            if not 1 <= num_hypotheses <= beam_size:
                raise ValueError("The number of hypotheses cannot be greater than beam_size * patience")
            hyp = np.empty((B, num_hypotheses, max_length), np.int32)
            hyp_lens = np.empty((B, num_hypotheses), np.int32)
            hyp_scores = np.zeros((B, num_hypotheses), np.float32)
            p = ctypes.c_void_p
            check(lib().ct2b200_generate_batch_beam(
                p(self._h), ids.ctypes.data_as(p), ctypes.c_int64(B), ctypes.c_int64(P), ctypes.c_int64(max_length),
                ctypes.c_int64(min_length), end_ids.ctypes.data_as(p), int(end_ids.size), int(return_end_token), int(beam_size),
                ctypes.c_float(patience), ctypes.c_float(length_penalty), int(num_hypotheses), hyp.ctypes.data_as(p),
                hyp_lens.ctypes.data_as(p), hyp_scores.ctypes.data_as(p)))
            results = []
            for b in range(B):
                seqs = [hyp[b, h, :hyp_lens[b, h]].tolist() for h in range(num_hypotheses) if hyp_lens[b, h] >= 0]
                results.append(GenerationResult([[self._tokens[i] for i in s] for s in seqs], seqs,
                                                [float(hyp_scores[b, h]) for h in range(len(seqs))] if return_scores else []))
            return results
        out = np.empty((B, max_length), np.int32)
        out_lens = np.empty(B, np.int32)
        scores = np.zeros(B, np.float32)
        if return_scores:
            check(lib().ct2b200_generate_batch_scores(
                ctypes.c_void_p(self._h), ids.ctypes.data_as(ctypes.c_void_p), lens.ctypes.data_as(ctypes.c_void_p),
                ctypes.c_int64(B), ctypes.c_int64(P), ctypes.c_int64(max_length), ctypes.c_int64(min_length),
                end_ids.ctypes.data_as(ctypes.c_void_p), int(end_ids.size), int(return_end_token),
                ctypes.c_float(length_penalty), out.ctypes.data_as(ctypes.c_void_p),
                out_lens.ctypes.data_as(ctypes.c_void_p), scores.ctypes.data_as(ctypes.c_void_p)))
        else:
            check(lib().ct2b200_generate_batch(ctypes.c_void_p(self._h), ids.ctypes.data_as(ctypes.c_void_p),
                                               lens.ctypes.data_as(ctypes.c_void_p), ctypes.c_int64(B), ctypes.c_int64(P),
                                               ctypes.c_int64(max_length), ctypes.c_int64(min_length),
                                               end_ids.ctypes.data_as(ctypes.c_void_p), int(end_ids.size),
                                               int(return_end_token), out.ctypes.data_as(ctypes.c_void_p),
                                               out_lens.ctypes.data_as(ctypes.c_void_p)))
        results = []
        for b in range(B):
            seq = out[b, :out_lens[b]].tolist()
            results.append(GenerationResult([[self._tokens[i] for i in seq]], [seq],
                                            [float(scores[b])] if return_scores else []))
        return results

    def forward_batch(self, tokens, return_log_probs: bool = False) -> np.ndarray:
        """Full-sequence forward; returns logits (or log-probs) [batch, time, vocab] float32 (host)."""
        rows = [list(r) for r in tokens]
        if rows and rows[0] and isinstance(rows[0][0], str):
            rows = [self._ids(r) for r in rows]
        _validate_ids(rows, self.vocab_size)
        if not rows or min(len(r) for r in rows) == 0:
            raise ValueError("forward_batch: empty batch or empty sequence")
        # ragged batches (the reference passes `lengths`, models/language_model.cc:135-160): rows are padded on the right
        # with id 0; under the causal mask the positions < len(row) never see the padding, positions >= len(row) hold
        # unspecified values exactly as in the reference's padded output
        B, T = len(rows), max(len(r) for r in rows)
        ids = np.zeros((B, T), np.int32)
        for i, r in enumerate(rows):
            ids[i, :len(r)] = r
        logits = np.empty((B, T, self.vocab_size), np.float32)
        check(lib().ct2b200_forward_batch(ctypes.c_void_p(self._h), ids.ctypes.data_as(ctypes.c_void_p),
                                          ctypes.c_int64(B), ctypes.c_int64(T), int(return_log_probs),
                                          logits.ctypes.data_as(ctypes.c_void_p)))
        return logits

    def score_batch(self, tokens, *, max_batch_size: int = 0, batch_type: str = "examples", max_input_length: int = 1024,
                    asynchronous: bool = False, offset: int = 0) -> List[ScoringResult]:
        """Generator.score_batch (python/cpp/generator.cc:83-96): the log-probability of every token given its prefix, one
        ScoringResult per input in request order.  tokens: token-string lists or id lists.  Sequences of fewer than two
        tokens, before or after truncation to max_input_length, score nothing; results start at token offset + 1
        (ScoringOptions::offset).  Inputs are re-batched longest first by max_batch_size / batch_type, and by the arena's
        max_batch_size; the scores do not depend on the batching."""
        if asynchronous:
            raise ValueError("score_batch: asynchronous=True is not supported (results are returned, not futures)")
        max_batch_size = _non_negative_int("max_batch_size", max_batch_size)
        max_input_length = _non_negative_int("max_input_length", max_input_length)
        offset = _non_negative_int("offset", offset)
        if batch_type not in ("examples", "tokens"):
            raise ValueError(f"Invalid batch type: {batch_type}")
        rows = [list(r) for r in tokens]
        rows = [self._ids(r) if r and isinstance(r[0], str) else [int(t) for t in r] for r in rows]
        _validate_ids(rows, self.vocab_size)
        eos = self._end_ids(None)[0]
        # skip_scoring (language_model.cc:38-52): fewer than two tokens as given, or left after truncation
        seqs = [_truncate(r, max_input_length, eos) if len(r) >= 2 else [] for r in rows]
        seqs = [s if len(s) >= 2 else [] for s in seqs]
        for i, s in enumerate(seqs):
            if len(s) > self.max_length:
                raise ValueError(f"score_batch: sequence {i} has {len(s)} tokens, more than max_length={self.max_length} "
                                 "of the generator (lower max_input_length or open the generator with a larger max_length)")
        results = [ScoringResult([], []) for _ in rows]
        p = ctypes.c_void_p
        for idx in _rebatch([len(r) for r in rows], max_batch_size, batch_type, self.max_batch_size):
            idx = [i for i in idx if seqs[i]]
            if not idx:
                continue
            B, L = len(idx), max(len(seqs[i]) for i in idx)
            ids = np.zeros((B, L), np.int32)
            lens = np.array([len(seqs[i]) for i in idx], np.int32)
            for b, i in enumerate(idx):
                ids[b, :lens[b]] = seqs[i]
            out = np.zeros((B, L - 1), np.float32)
            check(lib().ct2b200_score_batch(p(self._h), ids.ctypes.data_as(p), lens.ctypes.data_as(p), ctypes.c_int64(B),
                                            ctypes.c_int64(L), ctypes.c_int64(offset), out.ctypes.data_as(p)))
            for b, i in enumerate(idx):
                n = max(0, int(lens[b]) - 1 - offset)
                results[i] = ScoringResult([self._tokens[t] for t in seqs[i][1 + offset:]], out[b, :n].tolist())
        return results

    def bench_decode(self, batch: int, prompt_len: int, steps: int, warmup: int):
        pre, dec, n = ctypes.c_float(), ctypes.c_float(), ctypes.c_int64()
        check(lib().ct2b200_bench_decode(ctypes.c_void_p(self._h), ctypes.c_int64(batch), ctypes.c_int64(prompt_len),
                                         ctypes.c_int64(steps), ctypes.c_int64(warmup), ctypes.byref(pre),
                                         ctypes.byref(dec), ctypes.byref(n)))
        return pre.value, dec.value, n.value

    def bench_last_logits(self, batch: int, vocab_size: int) -> np.ndarray:
        """Logits [batch, vocab_size] float32 (host) of the last decode step bench_decode ran."""
        out = np.empty((batch, vocab_size), np.float32)
        check(lib().ct2b200_bench_last_logits(ctypes.c_void_p(self._h), ctypes.c_int64(batch),
                                              out.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), ctypes.c_int64(out.size)))
        return out

    def info(self):
        v = [ctypes.c_int() for _ in range(5)]
        wb = ctypes.c_int64()
        check(lib().ct2b200_generator_info(ctypes.c_void_p(self._h), *[ctypes.byref(x) for x in v], ctypes.byref(wb)))
        return dict(num_layers=v[0].value, num_heads=v[1].value, num_heads_kv=v[2].value, head_dim=v[3].value,
                    d_model=v[4].value, weight_bytes=wb.value)
