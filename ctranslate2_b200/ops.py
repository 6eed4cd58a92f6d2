"""Host-side mirror of the reference's `ctranslate2::ops` operator classes for the decode path
(include/ctranslate2/ops/*.h), on top of the C-ABI.  Same names, same argument meaning, same error
behaviour (ValueError ~ std::invalid_argument, Ct2B200Error ~ std::runtime_error).  Tensors are torch
CUDA tensors used purely as device-memory handles; outputs are resized by the op, as the reference's
non-template `operator()` does before `compute` runs."""
from __future__ import annotations

import ctypes
from typing import Optional, Tuple

import torch

from ._lib import check, lib

F32, F16, BF16 = 0, 1, 2
_DT = {torch.float32: F32, torch.float16: F16, torch.bfloat16: BF16}

# ops::ActivationType (include/ctranslate2/ops/activation.h:9-17)
class ActivationType:
    ReLU, GELUTanh, Swish, GELU, GELUSigmoid, Tanh, Sigmoid = range(7)

GEMM_AUTO, GEMM_TCGEN05, GEMM_MMA_SYNC = 0, 1, 2


def _p(t: Optional[torch.Tensor]):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dt(t: torch.Tensor) -> int:
    if t.dtype not in _DT:
        raise ValueError(f"unsupported float type {t.dtype}")
    return _DT[t.dtype]


def _c(t: torch.Tensor) -> torch.Tensor:
    if not t.is_cuda:
        raise ValueError("ctranslate2_b200 ops run on Device::CUDA only (no CPU fallback)")
    return t.contiguous()


class Quantize:
    """ops::Quantize (int8 arm): q, scale = Quantize()(x)."""
    def __init__(self, round_before_cast: bool = True):
        self.round_before_cast = round_before_cast

    def __call__(self, x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        x = _c(x)
        cols = x.shape[-1]
        rows = x.numel() // cols if cols else 0
        q = torch.empty(x.shape, dtype=torch.int8, device=x.device)
        s = torch.empty(x.shape[:-1], dtype=torch.float32, device=x.device)
        check(lib().ct2b200_quantize_rows(_p(x), _dt(x), ctypes.c_int64(rows), ctypes.c_int64(cols),
                                          int(self.round_before_cast), _p(q), _p(s), _stream()))
        return q, s


class Gemm:
    """ops::Gemm for the form layers::Dense uses: alpha=1, beta=0, trans_a=False, trans_b=True.
    int8 x int8 -> int32 (exact) or float32/float16/bfloat16 -> same type (fp32 accumulate, + bias/activation/residual)."""
    def __init__(self, alpha=1.0, beta=0.0, trans_a=False, trans_b=True, activation_type: Optional[int] = None,
                 impl: int = GEMM_AUTO):
        if alpha != 1.0 or beta != 0.0 or trans_a or not trans_b:
            raise ValueError("Gemm: only alpha=1, beta=0, trans_a=false, trans_b=true is on the hot path")
        self.act = -1 if activation_type is None else activation_type
        self.impl = impl

    def __call__(self, a, b, bias=None, residual=None):
        a, b = _c(a), _c(b)
        m, k = a.shape
        n, kb = b.shape
        if k != kb:
            raise ValueError("Gemm: inner dimensions differ")
        if a.dtype == torch.int8:
            c = torch.empty((m, n), dtype=torch.int32, device=a.device)
            check(lib().ct2b200_gemm_s8(_p(a), _p(b), ctypes.c_int64(m), ctypes.c_int64(n), ctypes.c_int64(k), _p(c),
                                        self.impl, _stream()))
            return c
        c = torch.empty((m, n), dtype=a.dtype, device=a.device)
        if a.dtype == torch.float32:      # primitives<CUDA>::gemm<float, float>: true fp32 FMAs
            check(lib().ct2b200_gemm_f32(_p(a), _p(b), _p(bias), _p(residual), self.act, ctypes.c_int64(m), ctypes.c_int64(n),
                                         ctypes.c_int64(k), _p(c), _stream()))
            return c
        check(lib().ct2b200_gemm_f16(_p(a), _p(b), _p(bias), _p(residual), self.act, ctypes.c_int64(m),
                                     ctypes.c_int64(n), ctypes.c_int64(k), _p(c), _dt(a), _stream()))
        return c


class Dequantize:
    """ops::Dequantize: rows form (x, scale) and GEMM-output form (c, a_scale, b_scale, bias)."""
    def __init__(self, activation_type: Optional[int] = None):
        self.act = -1 if activation_type is None else activation_type

    def __call__(self, c, a_scale, b_scale=None, bias=None, dtype=torch.float16):
        c = _c(c)
        if b_scale is None:
            rows, cols = c.shape
            y = torch.empty(c.shape, dtype=dtype, device=c.device)
            check(lib().ct2b200_dequantize_rows(_p(c), _p(a_scale), ctypes.c_int64(rows), ctypes.c_int64(cols),
                                                _p(y), _DT[dtype], _stream()))
            return y
        m, n = c.shape
        y = torch.empty((m, n), dtype=dtype, device=c.device)
        check(lib().ct2b200_dequantize_gemm_output(_p(c), _p(a_scale), _p(b_scale), _p(bias), self.act,
                                                   ctypes.c_int64(m), ctypes.c_int64(n), _p(y), _DT[dtype], _stream()))
        return y


def dense_int8(xq, x_scale, w, w_scale, bias=None, residual=None, activation_type=None, dtype=torch.float16,
               impl=GEMM_AUTO):
    """layers::Dense::operator() quantized arm as one fused launch (src/layers/common.cc:353-401)."""
    xq, w = _c(xq), _c(w)
    m, k = xq.shape
    n = w.shape[0]
    y = torch.empty((m, n), dtype=dtype, device=xq.device)
    act = -1 if activation_type is None else activation_type
    check(lib().ct2b200_dense_s8(_p(xq), _p(x_scale), _p(w), _p(w_scale), _p(bias), _p(residual), act,
                                 ctypes.c_int64(m), ctypes.c_int64(n), ctypes.c_int64(k), _p(y), _DT[dtype], impl,
                                 _stream()))
    return y


def dense_int8_rows(x, w, w_scale, gamma=None, eps=1e-5, bias=None, residual=None, activation_type=None):
    """[RMSNorm +] Quantize + layers::Dense (INT8 arm) from rows in T: the row kernel, then the fused Dense.  Returns (y, xq, x_scale)."""
    x, w = _c(x), _c(w)
    m, k = x.shape
    n = w.shape[0]
    y = torch.empty((m, n), dtype=x.dtype, device=x.device)
    xq = torch.empty((m, k), dtype=torch.int8, device=x.device)
    xs = torch.empty((m,), dtype=torch.float32, device=x.device)
    act = -1 if activation_type is None else activation_type
    check(lib().ct2b200_dense_s8_rows(_p(x), _p(gamma), ctypes.c_float(eps), _p(w), _p(w_scale), _p(bias), _p(residual), act,
                                      ctypes.c_int64(m), ctypes.c_int64(n), ctypes.c_int64(k), _p(y), _dt(x), _p(xq), _p(xs),
                                      _stream()))
    return y, xq, xs


def dense_int8_glu_rows(x, w_gate, gate_scale, w_up, up_scale, gamma=None, eps=1e-5, activation_type=ActivationType.Swish):
    x = _c(x)
    m, k = x.shape
    n = w_gate.shape[0]
    h = torch.empty((m, n), dtype=x.dtype, device=x.device)
    xq = torch.empty((m, k), dtype=torch.int8, device=x.device)
    xs = torch.empty((m,), dtype=torch.float32, device=x.device)
    check(lib().ct2b200_dense_s8_glu_rows(_p(x), _p(gamma), ctypes.c_float(eps), _p(_c(w_gate)), _p(gate_scale), _p(_c(w_up)),
                                          _p(up_scale), activation_type, ctypes.c_int64(m), ctypes.c_int64(n),
                                          ctypes.c_int64(k), _p(h), _dt(x), _p(xq), _p(xs), _stream()))
    return h, xq, xs


def dense_int8_glu(xq, x_scale, w_gate, gate_scale, w_up, up_scale, activation_type=ActivationType.Swish,
                   dtype=torch.float16, impl=GEMM_AUTO):
    """FeedForwardNetwork gate/up pair fused (src/layers/transformer.cc:21-51)."""
    xq, w_gate, w_up = _c(xq), _c(w_gate), _c(w_up)
    m, k = xq.shape
    n = w_gate.shape[0]
    h = torch.empty((m, n), dtype=dtype, device=xq.device)
    check(lib().ct2b200_dense_s8_glu(_p(xq), _p(x_scale), _p(w_gate), _p(gate_scale), _p(w_up), _p(up_scale),
                                     activation_type, ctypes.c_int64(m), ctypes.c_int64(n), ctypes.c_int64(k), _p(h),
                                     _DT[dtype], impl, _stream()))
    return h


class RMSNorm:
    """ops::RMSNorm(epsilon, use_residual)(gamma, input) -> output."""
    def __init__(self, epsilon: float = 1e-6, use_residual: bool = False):
        self.eps, self.use_residual = epsilon, use_residual

    def __call__(self, gamma, x):
        x, gamma = _c(x), _c(gamma)
        cols = x.shape[-1]
        y = torch.empty_like(x)
        check(lib().ct2b200_rms_norm(_p(gamma), _p(x), ctypes.c_int64(x.numel() // cols), ctypes.c_int64(cols),
                                     ctypes.c_float(self.eps), int(self.use_residual), _p(y), _dt(x), _stream()))
        return y

    def quantize(self, gamma, x):
        """RMSNorm + Quantize fused."""
        x, gamma = _c(x), _c(gamma)
        cols = x.shape[-1]
        q = torch.empty(x.shape, dtype=torch.int8, device=x.device)
        s = torch.empty(x.shape[:-1], dtype=torch.float32, device=x.device)
        check(lib().ct2b200_rms_norm_quantize(_p(gamma), _p(x), ctypes.c_int64(x.numel() // cols),
                                              ctypes.c_int64(cols), ctypes.c_float(self.eps), int(self.use_residual),
                                              _p(q), _p(s), _dt(x), _stream()))
        return q, s


class Rotary:
    """ops::Rotary(ndims, interleave)(input [.., time, depth], sin, cos) -> output (is_transposed=True)."""
    def __init__(self, ndims: int, interleave: bool):
        self.ndims, self.interleave = ndims, interleave

    def __call__(self, x, sin, cos):
        x, sin, cos = _c(x), _c(sin), _c(cos)
        depth, time = x.shape[-1], x.shape[-2]
        nd = depth if self.ndims == 0 else self.ndims
        y = torch.empty_like(x)
        check(lib().ct2b200_rotary(_p(x), _p(sin), _p(cos), ctypes.c_int64(x.numel() // (time * depth)),
                                   ctypes.c_int64(time), ctypes.c_int64(depth), ctypes.c_int64(nd),
                                   int(self.interleave), _p(y), _dt(x), _stream()))
        return y


class SoftMax:
    """ops::SoftMax(log)(x, lengths=None) -> y."""
    def __init__(self, log: bool = False):
        self.log = log

    def __call__(self, x, lengths=None):
        x = _c(x)
        cols = x.shape[-1]
        y = torch.empty_like(x)
        check(lib().ct2b200_softmax(_p(x), _p(lengths), ctypes.c_int64(x.numel() // cols), ctypes.c_int64(cols),
                                    int(self.log), _p(y), _dt(x), _stream()))
        return y


class LogSoftMax(SoftMax):
    def __init__(self):
        super().__init__(True)


def log_softmax_gather(logits, ids):
    """ops::LogSoftMax then ops::Gather(axis=-1, batch_dims=1) as one launch (src/scoring.cc:50-56): logits [.., V] in T,
    ids int [..] -> float32 [..] = float(T(log_softmax(logits)[.., ids])); the log-probabilities are not materialised."""
    logits = _c(logits)
    cols = logits.shape[-1]
    rows = logits.numel() // cols if cols else 0
    ids = _c(ids).to(torch.int32)
    if ids.numel() != rows:
        raise ValueError("log_softmax_gather: one id per row is required")
    y = torch.empty(logits.shape[:-1], dtype=torch.float32, device=logits.device)
    check(lib().ct2b200_log_softmax_gather(_p(logits), _p(ids), ctypes.c_int64(rows), ctypes.c_int64(cols), _p(y),
                                           _dt(logits), _stream()))
    return y


class TopK:
    """ops::TopK(k)(x) -> (values, indices int32); ties: lowest index first."""
    def __init__(self, k: int, axis: int = -1):
        if axis != -1:
            raise ValueError("Unsupported TopK axis")   # same message class as the reference
        self.k = k

    def __call__(self, x):
        x = _c(x)
        cols = x.shape[-1]
        v = torch.empty(x.shape[:-1] + (self.k,), dtype=x.dtype, device=x.device)
        i = torch.empty(x.shape[:-1] + (self.k,), dtype=torch.int32, device=x.device)
        check(lib().ct2b200_topk(_p(x), ctypes.c_int64(x.numel() // cols), ctypes.c_int64(cols), self.k, _p(v),
                                 _p(i), _dt(x), _stream()))
        return v, i


def random_sample(logits, k: int, temperature: float, seed: int, counter: int, step: int = 0):
    """RandomSampler::sample on every row of logits [..., vocab]: keep the top k (0 = all), divide by the temperature, draw
    one id by inverse CDF against u = philox_uniform(seed, counter, row, step) (csrc/kernels/philox.h).  Returns (ids int32,
    log-probabilities f32 of the unscaled rows at those ids)."""
    x = _c(logits)
    cols = x.shape[-1]
    rows = x.numel() // cols
    ids = torch.empty(x.shape[:-1], dtype=torch.int32, device=x.device)
    logp = torch.empty(x.shape[:-1], dtype=torch.float32, device=x.device)
    check(lib().ct2b200_random_sample(_p(x), ctypes.c_int64(rows), ctypes.c_int64(cols), int(k), ctypes.c_float(temperature),
                                      ctypes.c_uint32(seed), ctypes.c_uint32(counter), ctypes.c_uint32(step), _p(ids),
                                      _p(logp), _dt(x), _stream()))
    return ids, logp


def philox4x32_10(counter, key):
    """Philox4x32-10 of four 32-bit counter words under two key words, computed on the host by the library's own code."""
    c = (ctypes.c_uint32 * 4)(*[int(v) & 0xFFFFFFFF for v in counter])
    k = (ctypes.c_uint32 * 2)(*[int(v) & 0xFFFFFFFF for v in key])
    out = (ctypes.c_uint32 * 4)()
    check(lib().ct2b200_philox4x32_host(c, k, out))
    return list(out)


class Gather:
    """ops::Gather(axis=0, batch_dims=0)(data, ids) -> rows."""
    def __init__(self, axis: int = 0, batch_dims: int = 0):
        if axis != 0 or batch_dims != 0:
            raise ValueError("Gather: only axis 0 / batch_dims 0 is on the hot path")

    def __call__(self, data, ids):
        data, ids = _c(data), _c(ids).to(torch.int32)
        row = data[0].numel() * data.element_size()
        out = torch.empty(tuple(ids.shape) + tuple(data.shape[1:]), dtype=data.dtype, device=data.device)
        check(lib().ct2b200_gather_rows(_p(data), _p(ids), ctypes.c_int64(ids.numel()), ctypes.c_int64(row), _p(out),
                                        _stream()))
        return out


def embedding_int8(weight, scale, ids, dtype=torch.float16):
    """layers::Embeddings::operator() for INT8 weights (src/layers/common.cc:64-81)."""
    ids = _c(ids).to(torch.int32)
    depth = weight.shape[1]
    y = torch.empty(tuple(ids.shape) + (depth,), dtype=dtype, device=weight.device)
    check(lib().ct2b200_embedding_s8(_p(weight), _p(scale), _p(ids), ctypes.c_int64(ids.numel()),
                                     ctypes.c_int64(depth), _p(y), _DT[dtype], _stream()))
    return y


def mul_quantize(gate, up):
    gate, up = _c(gate), _c(up)
    cols = gate.shape[-1]
    q = torch.empty(gate.shape, dtype=torch.int8, device=gate.device)
    s = torch.empty(gate.shape[:-1], dtype=torch.float32, device=gate.device)
    check(lib().ct2b200_mul_quantize(_p(gate), _p(up), ctypes.c_int64(gate.numel() // cols), ctypes.c_int64(cols),
                                     _p(q), _p(s), _dt(gate), _stream()))
    return q, s


def attention_decode_workspace_bytes(batch, num_heads, head_dim, max_len):
    """Bytes of the (zero-initialised, reusable) workspace of attention_decode."""
    return lib().ct2b200_attention_decode_workspace(ctypes.c_int64(batch), num_heads, head_dim, ctypes.c_int64(max_len))


def attention_decode(qkv, k_cache, v_cache, sin, cos, lens, num_heads, num_heads_kv, head_dim, interleave=False,
                     scale=None, workspace=None):
    """MultiHeadAttention decode step between the two Dense layers (attention.cc:485-602)."""
    batch = qkv.shape[0]
    max_len = k_cache.shape[2]
    scale = head_dim ** -0.5 if scale is None else scale
    if workspace is None:
        nbytes = lib().ct2b200_attention_decode_workspace(ctypes.c_int64(batch), num_heads, head_dim,
                                                          ctypes.c_int64(max_len))
        workspace = torch.zeros(nbytes, dtype=torch.uint8, device=qkv.device)
    out = torch.empty((batch, num_heads * head_dim), dtype=qkv.dtype, device=qkv.device)
    check(lib().ct2b200_attention_decode(_p(qkv), _p(k_cache), _p(v_cache), _p(sin), _p(cos), _p(lens),
                                         ctypes.c_int64(batch), num_heads, num_heads_kv, head_dim,
                                         ctypes.c_int64(max_len), int(interleave), ctypes.c_float(scale), _p(out),
                                         _p(workspace), ctypes.c_size_t(workspace.numel()), _dt(qkv), _stream()))
    return out


def attention_prefill(qkv, k_cache, v_cache, sin, cos, batch, time, offset, num_heads, num_heads_kv, head_dim,
                      interleave=False, scale=None, lengths=None):
    """MultiHeadAttention over `time` new tokens (causal).  NOTE: rotates the q part of qkv in place."""
    max_len = k_cache.shape[2]
    scale = head_dim ** -0.5 if scale is None else scale
    out = torch.empty((batch * time, num_heads * head_dim), dtype=qkv.dtype, device=qkv.device)
    check(lib().ct2b200_attention_prefill(_p(qkv), _p(k_cache), _p(v_cache), _p(sin), _p(cos), _p(lengths),
                                          ctypes.c_int64(batch), ctypes.c_int64(time), ctypes.c_int64(offset),
                                          num_heads, num_heads_kv, head_dim, ctypes.c_int64(max_len), int(interleave),
                                          ctypes.c_float(scale), _p(out), _dt(qkv), _stream()))
    return out


# ---------------- encoder-decoder attention and the beam-search row step (seq2seq.cu) ----------------
# Inputs are used where they lie (no copy), so that callers can pass views at any element offset; rows must be contiguous.
def _rows(t: torch.Tensor) -> torch.Tensor:
    if not t.is_cuda:
        raise ValueError("ctranslate2_b200 ops run on Device::CUDA only (no CPU fallback)")
    if not t.is_contiguous():
        raise ValueError("rows must be contiguous")
    return t


def attention_encoder(qkv, num_heads, head_dim, batch, lengths=None, scale=None):
    """Encoder self-attention with a padding mask: qkv [batch * S, 3d] -> out [batch * S, d]; lengths int32 [batch] or None."""
    qkv = _rows(qkv)
    d = num_heads * head_dim
    S = qkv.shape[0] // batch if batch else 0
    scale = head_dim ** -0.5 if scale is None else scale
    out = torch.empty((batch * S, d), dtype=qkv.dtype, device=qkv.device)
    check(lib().ct2b200_attention_encoder(_p(qkv), _p(lengths), ctypes.c_int64(batch), S, num_heads, head_dim,
                                          ctypes.c_float(scale), _p(out), _dt(qkv), _stream()))
    return out


def attention_encoder_mma(qkv, num_heads, head_dim, batch, lengths=None, scale=None):
    """attention_encoder on tensor cores (fp16 / bf16, head_dim 64 or 128; ValueError otherwise).  Rows past a length are
    unspecified but finite."""
    qkv = _rows(qkv)
    d = num_heads * head_dim
    S = qkv.shape[0] // batch if batch else 0
    scale = head_dim ** -0.5 if scale is None else scale
    out = torch.empty((batch * S, d), dtype=qkv.dtype, device=qkv.device)
    check(lib().ct2b200_attention_encoder_mma(_p(qkv), _p(lengths), ctypes.c_int64(batch), S, num_heads, head_dim,
                                              ctypes.c_float(scale), _p(out), _dt(qkv), _stream()))
    return out


def attention_causal(qkv, num_heads, head_dim, batch, scale=None):
    """Teacher-forced causal self-attention: qkv [batch * time, 3d] -> out [batch * time, d]."""
    qkv = _rows(qkv)
    d = num_heads * head_dim
    time = qkv.shape[0] // batch if batch else 0
    scale = head_dim ** -0.5 if scale is None else scale
    out = torch.empty((batch * time, d), dtype=qkv.dtype, device=qkv.device)
    check(lib().ct2b200_attention_causal(_p(qkv), ctypes.c_int64(batch), time, num_heads, head_dim, ctypes.c_float(scale),
                                         _p(out), _dt(qkv), _stream()))
    return out


def attention_beam_self(qkv, k_cache, v_cache, anc, step, num_heads, head_dim, scale=None):
    """One-token decoder self-attention over the beam-remapped cache: qkv [rows, 3d]; k_cache / v_cache [rows, max_len, d]
    (the rows' new k / v are written at position step); anc int32 [2, rows, max_len]; step: int32 [1] device tensor."""
    qkv, k_cache, v_cache, anc = _rows(qkv), _rows(k_cache), _rows(v_cache), _rows(anc)
    rows, max_len = k_cache.shape[0], k_cache.shape[1]
    scale = head_dim ** -0.5 if scale is None else scale
    out = torch.empty((rows, num_heads * head_dim), dtype=qkv.dtype, device=qkv.device)
    check(lib().ct2b200_attention_beam_self(_p(qkv), _p(k_cache), _p(v_cache), _p(anc), _p(step), ctypes.c_int64(rows), max_len,
                                            num_heads, head_dim, ctypes.c_float(scale), _p(out), _dt(qkv), _stream()))
    return out


def attention_cross(q, kv, num_heads, head_dim, beam, lengths=None, scale=None, capture=None, masks=None, first=0,
                    total=0):
    """Cross-attention: q [rows, d], kv [batch * S, 2d] with batch = rows / beam -> out [rows, d].  capture (float32
    [batch, total, beam, S]) with masks (uint32 as int32 [H]): also save the scores of the selected heads."""
    q, kv = _rows(q), _rows(kv)
    rows = q.shape[0]
    batch = rows // beam
    S = kv.shape[0] // batch if batch else 0
    scale = head_dim ** -0.5 if scale is None else scale
    out = torch.empty((rows, num_heads * head_dim), dtype=q.dtype, device=q.device)
    check(lib().ct2b200_attention_cross(_p(q), _p(kv), _p(lengths), ctypes.c_int64(rows), beam, S, num_heads, head_dim,
                                        ctypes.c_float(scale), _p(out), _p(capture), _p(masks), first, total, _dt(q),
                                        _stream()))
    return out


def beam_rows(logits, cum, step, beam, vocab, min_length=0, end_ids=None):
    """One beam-search step of every row: logits [batch * beam, vocab_ld] in T (the end ids are disabled in place while
    step < min_length), cum [batch * beam] T, step int32 [1] device tensor -> (scores T, ids int32) [batch * beam, 2 * beam],
    ids flattened over [beam, vocab]."""
    if beam < 1:
        raise ValueError("beam_rows: beam_size must be in [1, 8]")
    logits, cum = _rows(logits), _rows(cum)
    rows, vocab_ld = logits.shape
    num_end = 0 if end_ids is None else int(end_ids.numel())
    scores = torch.empty((rows, 2 * beam), dtype=logits.dtype, device=logits.device)
    ids = torch.empty((rows, 2 * beam), dtype=torch.int32, device=logits.device)
    check(lib().ct2b200_beam_rows(_p(logits), _p(cum), _p(step), rows // beam, beam, vocab, ctypes.c_int64(vocab_ld), min_length,
                                  _p(end_ids), num_end, _p(scores), _p(ids), _dt(logits), _stream()))
    return scores, ids


# ---------------- AWQ-INT4 (ops::GemmAwq / GemvAwq / DequantizeAwq) ----------------
AWQ_GEMM, AWQ_GEMV = 1, 2


class AwqWeight:
    """AWQ weight of a Dense layer repacked ONCE into the native K-major layout (ct2b200_awq_repack)."""
    def __init__(self, qweight, scales, qzeros, layout: int, group_size: int):
        qweight, scales, qzeros = _c(qweight), _c(scales), _c(qzeros)
        if layout == AWQ_GEMM:
            self.k, self.n = qweight.shape[0], qweight.shape[1] * 8
        elif layout == AWQ_GEMV:
            self.n, self.k = qweight.shape[0], qweight.shape[1] * 8
        else:
            raise ValueError("AWQ layout must be 1 (AWQ_GEMM) or 2 (AWQ_GEMV)")
        self.group_size = group_size
        ng = self.k // group_size
        dev = qweight.device
        self.wp = torch.empty((self.n, self.k // 8), dtype=torch.int32, device=dev)
        self.sc = torch.empty((self.n, ng), dtype=torch.float16, device=dev)
        self.zr = torch.empty((self.n, ng), dtype=torch.float16, device=dev)
        self.sz = torch.empty((ng, self.n, 2), dtype=torch.float16, device=dev)     # {scale, zero} pairs, group-major
        check(lib().ct2b200_awq_repack(_p(qweight), _p(scales), _p(qzeros), layout, group_size, ctypes.c_int64(self.n),
                                       ctypes.c_int64(self.k), _p(self.wp), _p(self.sc), _p(self.zr), _p(self.sz), _stream()))


def dequantize_awq(qweight, scales, qzeros, layout: int, group_size: int):
    """ops::DequantizeAwq: reference layout -> W float16 [K, N]."""
    qweight = _c(qweight)
    if layout == AWQ_GEMM:
        k, n = qweight.shape[0], qweight.shape[1] * 8
    else:
        n, k = qweight.shape[0], qweight.shape[1] * 8
    w = torch.empty((k, n), dtype=torch.float16, device=qweight.device)
    check(lib().ct2b200_dequantize_awq(_p(qweight), _p(_c(scales)), _p(_c(qzeros)), layout, group_size,
                                       ctypes.c_int64(n), ctypes.c_int64(k), _p(w), _stream()))
    return w


def dense_awq(x, w: AwqWeight, bias=None, residual=None, activation_type=None):
    """ops::GemmAwq / GemvAwq (+bias, activation, residual) on a repacked weight; x float16 [m, k]."""
    x = _c(x)
    m = x.shape[0]
    y = torch.empty((m, w.n), dtype=torch.float16, device=x.device)
    scratch = torch.empty((w.n, w.k), dtype=torch.float16, device=x.device) if m > 64 else None
    act = -1 if activation_type is None else activation_type
    check(lib().ct2b200_dense_awq(_p(x), _p(w.wp), _p(w.sc), _p(w.zr), _p(w.sz), w.group_size, _p(bias), _p(residual), act,
                                  ctypes.c_int64(m), ctypes.c_int64(w.n), ctypes.c_int64(w.k), _p(y), _p(scratch),
                                  _stream()))
    return y


def dense_awq_glu(x, wg: AwqWeight, wu: AwqWeight, activation_type=ActivationType.Swish):
    x = _c(x)
    m = x.shape[0]
    h = torch.empty((m, wg.n), dtype=torch.float16, device=x.device)
    s1 = torch.empty((wg.n, wg.k), dtype=torch.float16, device=x.device) if m > 64 else None
    s2 = torch.empty((m, wg.n), dtype=torch.float16, device=x.device) if m > 64 else None
    check(lib().ct2b200_dense_awq_glu(_p(x), _p(wg.wp), _p(wg.sc), _p(wg.zr), _p(wg.sz), _p(wu.wp), _p(wu.sc), _p(wu.zr), _p(wu.sz),
                                      wg.group_size, activation_type, ctypes.c_int64(m), ctypes.c_int64(wg.n),
                                      ctypes.c_int64(wg.k), _p(h), _p(s1), _p(s2), _stream()))
    return h


class LayerNorm:
    """ops::LayerNorm over the last axis (include/ctranslate2/ops/layer_norm.h): y = LayerNorm(axis=-1, epsilon)(beta, gamma, x).
    quantize=True also returns ops::Quantize of the normalised row from the same launch: (y, q, scale)."""
    def __init__(self, axis: int = -1, epsilon: float = 1e-5):
        if axis != -1:
            raise ValueError("LayerNorm: only the last axis is on the hot path")
        self.epsilon = epsilon

    def __call__(self, beta, gamma, x, quantize: bool = False, round_before_cast: bool = True):
        x = _c(x)
        cols = x.shape[-1]
        rows = x.numel() // cols if cols else 0
        y = torch.empty_like(x)
        q = torch.empty(x.shape, dtype=torch.int8, device=x.device) if quantize else None
        s = torch.empty(x.shape[:-1], dtype=torch.float32, device=x.device) if quantize else None
        check(lib().ct2b200_layer_norm(_p(x), _p(gamma), _p(beta), ctypes.c_int64(rows), ctypes.c_int64(cols),
                                       ctypes.c_float(self.epsilon), _p(y), _p(q), _p(s), int(round_before_cast), _dt(x),
                                       _stream()))
        return (y, q, s) if quantize else y
