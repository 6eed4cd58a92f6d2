"""ctypes binding of oracle/_ref/libct2ref_driver.so (the UNMODIFIED reference, CPU build) and of
oracle/_ref_cuda/libct2ref_cuda_driver.so (the UNMODIFIED reference WITH its CUDA backend: cuBLAS GEMM,
its own AWQ / FlashAttention-2 kernels, compiled for sm_90 by oracle/Makefile.ref_cuda).

TEST INFRASTRUCTURE: only tests/, tools/make_golden*.py, __graft_entry__.smoke() and bench.py's
reference legs import this.  `available()` / `cuda_available()` are False when the library was not built
(run `make -f oracle/Makefile.ref -j8` / `make -f oracle/Makefile.ref_cuda -j8` in a container that has
/root/reference).  `use_cuda(True)` switches the process to the CUDA build BEFORE the first call: the two
libraries define the same symbols and are never loaded together.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_PATH = os.path.join(_HERE, "_ref", "libct2ref_driver.so")
_PATH_CUDA = os.path.join(_HERE, "_ref_cuda", "libct2ref_cuda_driver.so")
_lib = None
_cuda = False


def available() -> bool:
    return os.path.exists(_PATH)


def cuda_available() -> bool:
    return os.path.exists(_PATH_CUDA)


def use_cuda(flash_attention: bool = False):
    """Route this process to the reference's CUDA build: generators / translators load on Device::CUDA (device 0)."""
    global _cuda
    if _lib is not None and not _cuda:
        raise RuntimeError("the CPU reference library is already loaded in this process")
    _cuda = True
    _check(lib().ref_set_device(1, int(flash_attention)))


def is_cuda() -> bool:
    return _cuda


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(_PATH_CUDA if _cuda else _PATH)
        _lib.ref_last_error.restype = ctypes.c_char_p
        _lib.ref_generator_open.restype = ctypes.c_void_p
        _lib.ref_generator_open.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int]
        _lib.ref_generator_close.argtypes = [ctypes.c_void_p]
        _lib.ref_vocab_size.argtypes = [ctypes.c_void_p]
    return _lib


def _p(a):
    return None if a is None else ctypes.c_void_p(a.ctypes.data)


def _check(rc):
    if rc != 0:
        raise RuntimeError("reference: " + lib().ref_last_error().decode())


def _c(a, dt):
    return None if a is None else np.ascontiguousarray(a, dtype=dt)


class RefGenerator:
    def __init__(self, model_dir: str, compute_type: str = "int8", threads: int = 0):
        self.h = lib().ref_generator_open(model_dir.encode(), compute_type.encode(), threads)
        if not self.h:
            raise RuntimeError("reference: " + lib().ref_last_error().decode())
        self.vocab = lib().ref_vocab_size(ctypes.c_void_p(self.h))

    def close(self):
        if self.h:
            lib().ref_generator_close(ctypes.c_void_p(self.h))
            self.h = None

    def forward(self, ids: np.ndarray, log_probs: bool = False) -> np.ndarray:
        ids = _c(ids, np.int32)
        B, T = ids.shape
        out = np.zeros((B, T, self.vocab), np.float32)
        _check(lib().ref_forward(ctypes.c_void_p(self.h), _p(ids), B, T, int(log_probs), _p(out),
                                 ctypes.c_int64(out.size)))
        return out

    def generate(self, prompts: np.ndarray, max_length: int, min_length: int = 0, end_id: int = 2):
        prompts = _c(prompts, np.int32)
        B, P = prompts.shape
        out = np.zeros((B, max_length), np.int32)
        lens = np.zeros(B, np.int32)
        _check(lib().ref_generate(ctypes.c_void_p(self.h), _p(prompts), B, P, max_length, min_length,
                                  end_id, _p(out), _p(lens)))
        return [out[b, :lens[b]].tolist() for b in range(B)]

    def generate_beam(self, prompts: np.ndarray, beam_size: int, max_length: int, min_length: int = 0, end_id: int = 2,
                      length_penalty: float = 1.0, num_hypotheses: int = 1, patience: float = 1.0):
        """Beam search: per prompt a list of (tokens, score), best first."""
        prompts = _c(prompts, np.int32)
        B, P = prompts.shape
        out = np.zeros((B, num_hypotheses, max_length), np.int32)
        lens = np.zeros((B, num_hypotheses), np.int32)
        scores = np.zeros((B, num_hypotheses), np.float32)
        _check(lib().ref_generate_beam(ctypes.c_void_p(self.h), _p(prompts), B, P, beam_size, num_hypotheses, max_length,
                                       min_length, end_id, ctypes.c_float(length_penalty), ctypes.c_float(patience),
                                       _p(out), _p(lens), _p(scores)))
        return [[(out[b, h, :lens[b, h]].tolist(), float(scores[b, h])) for h in range(num_hypotheses) if lens[b, h] >= 0]
                for b in range(B)]

    def generate_with_scores(self, prompts: np.ndarray, max_length: int, min_length: int = 0, end_id: int = 2,
                             length_penalty: float = 1.0):
        """(tokens, scores) with GenerationOptions::return_scores = true."""
        prompts = _c(prompts, np.int32)
        B, P = prompts.shape
        out = np.zeros((B, max_length), np.int32)
        lens = np.zeros(B, np.int32)
        scores = np.zeros(B, np.float32)
        _check(lib().ref_generate_scores(ctypes.c_void_p(self.h), _p(prompts), B, P, max_length, min_length, end_id,
                                         ctypes.c_float(length_penalty), _p(out), _p(lens), _p(scores)))
        return [out[b, :lens[b]].tolist() for b in range(B)], scores


def _generate_processors(self, prompts, max_length, min_length=0, end_id=2, repetition_penalty=1.0, no_repeat_ngram_size=0,
                         disable_unk=False, suppress_sequences=()):
    """(tokens, scores) of greedy generate_batch with the logits processors of GenerationOptions."""
    prompts = _c(prompts, np.int32)
    B, P = prompts.shape
    flat = []
    for seq in suppress_sequences:
        flat.extend(int(t) for t in seq)
        flat.append(-1)
    sup = np.array(flat if flat else [-1], np.int32)
    out = np.zeros((B, max_length), np.int32)
    lens = np.zeros(B, np.int32)
    scores = np.zeros(B, np.float32)
    _check(lib().ref_generate_processors(ctypes.c_void_p(self.h), _p(prompts), B, P, max_length, min_length, end_id,
                                         ctypes.c_float(repetition_penalty), int(no_repeat_ngram_size), int(bool(disable_unk)),
                                         _p(sup), int(len(flat)), _p(out), _p(lens), _p(scores)))
    return [out[b, :lens[b]].tolist() for b in range(B)], scores


RefGenerator.generate_processors = _generate_processors


def _generate_ragged(self, prompts, max_length, min_length=0, end_id=2):
    """(tokens, scores) of greedy generate_batch over prompts of different lengths (list of id lists)."""
    B = len(prompts)
    P = max(len(r) for r in prompts)
    ids = np.full((B, P), -1, np.int32)
    for b, r in enumerate(prompts):
        ids[b, :len(r)] = r
    width = max_length + P
    out = np.zeros((B, width), np.int32)
    lens = np.zeros(B, np.int32)
    scores = np.zeros(B, np.float32)
    _check(lib().ref_generate_ragged(ctypes.c_void_p(self.h), _p(ids), B, P, max_length, min_length, end_id, _p(out), _p(lens),
                                     _p(scores)))
    return [out[b, :lens[b]].tolist() for b in range(B)], scores


RefGenerator.generate_ragged = _generate_ragged


def _score(self, sequences, offset=0):
    """Generator::score_batch over id lists: per sequence the log-probabilities of tokens[offset + 1:] (list of float lists)."""
    B = len(sequences)
    P = max(2, max(len(r) for r in sequences))
    ids = np.full((B, P), -1, np.int32)
    for b, r in enumerate(sequences):
        ids[b, :len(r)] = r
    out = np.zeros((B, P - 1), np.float32)
    lens = np.zeros(B, np.int32)
    _check(lib().ref_score(ctypes.c_void_p(self.h), _p(ids), B, P, int(offset), _p(out), _p(lens)))
    return [out[b, :lens[b]].tolist() for b in range(B)]


RefGenerator.score = _score


class RefTranslator:
    """The unmodified reference's Translator (encoder-decoder models) over token ids."""

    def __init__(self, model_dir: str, compute_type: str = "int8", threads: int = 0):
        lib().ref_translator_open.restype = ctypes.c_void_p
        self.h = lib().ref_translator_open(model_dir.encode(), compute_type.encode(), threads)
        if not self.h:
            raise RuntimeError(lib().ref_last_error().decode())
        s, t = ctypes.c_int(), ctypes.c_int()
        _check(lib().ref_translator_vocab_sizes(ctypes.c_void_p(self.h), ctypes.byref(s), ctypes.byref(t)))
        self.source_vocab_size, self.target_vocab_size = s.value, t.value

    def close(self):
        if self.h:
            lib().ref_translator_close(ctypes.c_void_p(self.h))
            self.h = None

    def __del__(self):
        self.close()

    def encode(self, source_ids):
        """layers::TransformerEncoder over the padded batch -> memory [B, S, d] fp32 and the lengths."""
        B = len(source_ids)
        S = max(len(r) for r in source_ids)
        src = np.zeros((B, S), np.int32)
        for b, r in enumerate(source_ids):
            src[b, :len(r)] = r
        lens = np.array([len(r) for r in source_ids], np.int32)
        out = np.zeros((B, S, 4096), np.float32)
        _check(lib().ref_encoder_forward(ctypes.c_void_p(self.h), _p(src), _p(lens), B, S, _p(out), ctypes.c_int64(out.size)))
        return out, lens

    def translate(self, source_ids, beam_size=2, num_hypotheses=1, max_length=256, min_length=1, length_penalty=1.0):
        """source_ids: list of id lists.  Returns per sentence a list of (target ids, score), best first."""
        B = len(source_ids)
        S = max(len(r) for r in source_ids)
        src = np.full((B, S), -1, np.int32)
        for b, r in enumerate(source_ids):
            src[b, :len(r)] = r
        out = np.zeros((B, num_hypotheses, max_length), np.int32)
        lens = np.zeros((B, num_hypotheses), np.int32)
        scores = np.zeros((B, num_hypotheses), np.float32)
        _check(lib().ref_translate(ctypes.c_void_p(self.h), _p(src), B, S, beam_size, num_hypotheses, max_length, min_length,
                                   ctypes.c_float(length_penalty), _p(out), _p(lens), _p(scores)))
        return [[(out[b, h, :lens[b, h]].tolist(), float(scores[b, h])) for h in range(num_hypotheses) if lens[b, h] >= 0]
                for b in range(B)]



class RefWhisper:
    """The unmodified reference's models::Whisper (encode / generate) over features and prompt ids."""

    def __init__(self, model_dir: str, compute_type: str = "float32", threads: int = 0):
        lib().ref_whisper_open.restype = ctypes.c_void_p
        self.h = lib().ref_whisper_open(model_dir.encode(), compute_type.encode(), threads)
        if not self.h:
            raise RuntimeError(lib().ref_last_error().decode())

    def close(self):
        if self.h and lib is not None:
            lib().ref_whisper_close(ctypes.c_void_p(self.h))
            self.h = None

    def encode(self, features: np.ndarray, d_model: int) -> np.ndarray:
        f = np.ascontiguousarray(features, np.float32)
        B, M, T = f.shape
        out = np.zeros((B, (T + 1) // 2, d_model), np.float32)
        _check(lib().ref_whisper_encode(ctypes.c_void_p(self.h), _p(f), B, M, T, _p(out), ctypes.c_int64(out.size)))
        return out

    def generate(self, features: np.ndarray, prompts, beam_size=5, patience=1.0, num_hypotheses=1, length_penalty=1.0,
                 max_length=448, suppress_blank=True, suppress_default=True):
        """Returns (per entry [(ids, score), ...] best first, no_speech_probs [B])."""
        f = np.ascontiguousarray(features, np.float32)
        B, M, T = f.shape
        pr = np.ascontiguousarray(np.array(prompts, np.int32))
        out = np.zeros((B, num_hypotheses, max_length), np.int32)
        lens = np.zeros((B, num_hypotheses), np.int32)
        scores = np.zeros((B, num_hypotheses), np.float32)
        nsp = np.zeros(B, np.float32)
        _check(lib().ref_whisper_generate(ctypes.c_void_p(self.h), _p(f), B, M, T, _p(pr), pr.shape[1], beam_size,
                                          ctypes.c_float(patience), num_hypotheses, ctypes.c_float(length_penalty), max_length,
                                          int(suppress_blank), int(suppress_default), _p(out), _p(lens), _p(scores), _p(nsp)))
        res = [[(out[b, h, :lens[b, h]].tolist(), float(scores[b, h])) for h in range(num_hypotheses) if lens[b, h] >= 0]
               for b in range(B)]
        return res, nsp

def layer_norm(gamma, beta, x, eps=1e-5):
    x = _c(x, np.float32)
    r, c = x.shape
    y = np.zeros((r, c), np.float32)
    _check(lib().ref_layer_norm(_p(_c(gamma, np.float32)), _p(_c(beta, np.float32)), _p(x), r, c, ctypes.c_float(eps), _p(y)))
    return y


def quantize(x, round_before_cast=True):
    x = _c(x, np.float32)
    r, c = x.shape
    q = np.zeros((r, c), np.int8)
    s = np.zeros(r, np.float32)
    _check(lib().ref_quantize(_p(x), r, c, int(round_before_cast), _p(q), _p(s)))
    return q, s


def gemm_s8(a, b):
    a, b = _c(a, np.int8), _c(b, np.int8)
    m, k = a.shape
    n = b.shape[0]
    c = np.zeros((m, n), np.int32)
    _check(lib().ref_gemm_s8(_p(a), _p(b), m, n, k, _p(c)))
    return c


def gemm_f32(a, b, bias=None, residual=None, act=-1):
    a, b = _c(a, np.float32), _c(b, np.float32)
    bias, residual = _c(bias, np.float32), _c(residual, np.float32)
    m, k = a.shape
    n = b.shape[0]
    c = np.zeros((m, n), np.float32)
    _check(lib().ref_gemm_f32(_p(a), _p(b), _p(bias), _p(residual), act, m, n, k, _p(c)))
    return c


def dequantize_gemm(c, a_scale, b_scale, bias=None, act=-1):
    c = _c(c, np.int32)
    a_scale, b_scale, bias = _c(a_scale, np.float32), _c(b_scale, np.float32), _c(bias, np.float32)
    m, n = c.shape
    y = np.zeros((m, n), np.float32)
    _check(lib().ref_dequantize_gemm(_p(c), _p(a_scale), _p(b_scale), _p(bias), act, m, n, _p(y)))
    return y


def rms_norm(gamma, x, eps):
    gamma, x = _c(gamma, np.float32), _c(x, np.float32)
    r, c = x.shape
    y = np.zeros_like(x)
    _check(lib().ref_rms_norm(_p(gamma), _p(x), r, c, ctypes.c_float(eps), _p(y)))
    return y


def rotary(x, sin, cos, interleave):
    x, sin, cos = _c(x, np.float32), _c(sin, np.float32), _c(cos, np.float32)
    b, h, t, d = x.shape
    y = np.zeros_like(x)
    _check(lib().ref_rotary(_p(x), _p(sin), _p(cos), b, h, t, d, sin.shape[1], int(interleave), _p(y)))
    return y


def softmax(x, lengths=None, log=False):
    x = _c(x, np.float32)
    lengths = _c(lengths, np.int32)
    r, c = x.shape
    y = np.zeros_like(x)
    _check(lib().ref_softmax(_p(x), _p(lengths), r, c, int(log), _p(y)))
    return y


def topk(x, k):
    x = _c(x, np.float32)
    r, c = x.shape
    v = np.zeros((r, k), np.float32)
    i = np.zeros((r, k), np.int32)
    _check(lib().ref_topk(_p(x), r, c, k, _p(v), _p(i)))
    return v, i


def gather(data, ids):
    data, ids = _c(data, np.float32), _c(ids, np.int32)
    n, d = data.shape
    out = np.zeros((ids.size, d), np.float32)
    _check(lib().ref_gather(_p(data), n, d, _p(ids), ids.size, _p(out)))
    return out


def rotary_tables(num_positions, dim, base=10000.0, interleave=False, scaling_type=-1, scaling_factor=1.0,
                  low_freq_factor=1.0, high_freq_factor=4.0, original_max_position_embeddings=0):
    """sin/cos tables of the reference's layers::RotaryEmbeddings, recovered by rotating an all-ones input
    (non-interleaved: y_lo = cos - sin, y_hi = cos + sin)."""
    assert not interleave
    x = np.ones((num_positions, dim), np.float32)
    y = np.zeros_like(x)
    _check(lib().ref_rotary_embeddings(_p(x), num_positions, dim, 0, 0, scaling_type, ctypes.c_float(scaling_factor),
                                       ctypes.c_float(base), ctypes.c_float(low_freq_factor),
                                       ctypes.c_float(high_freq_factor), original_max_position_embeddings, _p(y)))
    h = dim // 2
    cos = (y[:, :h] + y[:, h:]) / 2
    sin = (y[:, h:] - y[:, :h]) / 2
    return np.concatenate([sin, sin], 1), np.concatenate([cos, cos], 1)


# ---- CUDA build only: the reference's GPU-only ops (AWQ) and its INT8 Dense chain, host arrays in and out ----
def _f16(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float16)


def cuda_gemm_awq(x, qweight, scales, qzeros, group):
    """ops::GemmAwq (AWQ_GEMM layout): x f16 [m,k], qweight int32 [k,n/8], scales f16 [k/g,n], qzeros int32 [k/g,n/8]."""
    x, scales = _f16(x), _f16(scales)
    qweight, qzeros = _c(qweight, np.int32), _c(qzeros, np.int32)
    m, k = x.shape
    n = qweight.shape[1] * 8
    y = np.zeros((m, n), np.float16)
    _check(lib().ref_cuda_gemm_awq(_p(x), _p(qweight), _p(scales), _p(qzeros), m, n, k, group, _p(y)))
    return y


def cuda_gemv_awq(x, qweight, scales, qzeros):
    """ops::GemvAwq (AWQ_GEMV layout): qweight int32 [n,k/8], scales f16 [n,sw], qzeros int32 [n,zw]."""
    x, scales = _f16(x), _f16(scales)
    qweight, qzeros = _c(qweight, np.int32), _c(qzeros, np.int32)
    m, k = x.shape
    n = qweight.shape[0]
    y = np.zeros((m, n), np.float16)
    _check(lib().ref_cuda_gemv_awq(_p(x), _p(qweight), _p(scales), _p(qzeros), m, n, k, scales.shape[1], qzeros.shape[1], _p(y)))
    return y


def cuda_dequantize_awq(qweight, scales, qzeros, group):
    """ops::DequantizeAwq (AWQ_GEMM layout) -> W f16 [k, n]."""
    scales = _f16(scales)
    qweight, qzeros = _c(qweight, np.int32), _c(qzeros, np.int32)
    k, n = qweight.shape[0], qweight.shape[1] * 8
    w = np.zeros((k, n), np.float16)
    _check(lib().ref_cuda_dequantize_awq(_p(qweight), _p(scales), _p(qzeros), n, k, group, _p(w)))
    return w


def cuda_dense_s8(x, w, w_scale, act=-1):
    """layers::Dense INT8 arm on the GPU: Quantize -> cublasGemmEx(s8) -> Dequantize(+act); x f16 [m,k], w int8 [n,k]."""
    x = _f16(x)
    w, w_scale = _c(w, np.int8), _c(w_scale, np.float32)
    m, k = x.shape
    n = w.shape[0]
    y = np.zeros((m, n), np.float16)
    _check(lib().ref_cuda_dense_s8(_p(x), _p(w), _p(w_scale), act, m, n, k, _p(y)))
    return y


def _generate_timed(self, prompts, max_length, end_id=2):
    """(tokens [B, max_length], seconds) of one greedy generate_batch of exactly max_length tokens (device-synchronised)."""
    prompts = _c(prompts, np.int32)
    B, P = prompts.shape
    out = np.zeros((B, max_length), np.int32)
    sec = ctypes.c_double()
    _check(lib().ref_generate_timed(ctypes.c_void_p(self.h), _p(prompts), B, P, max_length, end_id, _p(out), ctypes.byref(sec)))
    return out, sec.value


RefGenerator.generate_timed = _generate_timed


def _generate_steps(self, prompts, max_length, end_id=2):
    """(stamps [max_length], seconds): host time at which every step of batch entry 0 was delivered to the public per-step
    callback (generation.h:77) during one greedy generate_batch; stamps[0] is the end of the prompt pass."""
    prompts = _c(prompts, np.int32)
    B, P = prompts.shape
    stamps = np.zeros(max_length, np.float64)
    sec = ctypes.c_double()
    _check(lib().ref_generate_steps(ctypes.c_void_p(self.h), _p(prompts), B, P, max_length, end_id, _p(stamps), ctypes.byref(sec)))
    return stamps, sec.value


RefGenerator.generate_steps = _generate_steps
