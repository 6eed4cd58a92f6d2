"""Writer for CTranslate2 model directories (model.bin binary version 6 + config.json +
vocabulary.json) holding SYNTHETIC Llama-class decoders.

The on-disk format is the reference's own, so directories written here load unchanged in the
reference (python/ctranslate2/specs/model_spec.py:382-414 is the reference writer,
src/models/model.cc:561-660 the reader) and directories written by the reference converters load
unchanged in ctranslate2_b200.  There is no network in this environment, so the benchmark and the
tests use random-init weights of the named architecture (BASELINE.md §3).

Variable names follow TransformerDecoderSpec revision 8 as emitted for LlamaForCausalLM by
python/ctranslate2/converters/transformers.py:1697-1843.
"""
from __future__ import annotations

import json
import os
import struct
from dataclasses import dataclass
from typing import Dict, Optional

import numpy as np

BINARY_VERSION = 6
_TYPE_IDS = {"float32": 0, "int8": 1, "int16": 2, "int32": 3, "float16": 4, "bfloat16": 5}


@dataclass
class LlamaConfig:
    num_layers: int = 32
    num_heads: int = 32
    num_heads_kv: int = 8
    head_dim: int = 128
    ffn_dim: int = 14336
    vocab_size: int = 128256
    rotary_base: float = 500000.0
    rms_eps: float = 1e-5
    rotary_scaling_type: int = -1          # attention_spec.RotaryScalingType: Linear=0, Su=1, Llama3=2
    rotary_scaling_factor: float = 1.0
    rotary_low_freq_factor: float = 1.0
    rotary_high_freq_factor: float = 4.0
    original_max_position_embeddings: int = 0

    @property
    def d_model(self) -> int:
        return self.num_heads * self.head_dim


LLAMA3_8B = LlamaConfig()
LLAMA3_70B = LlamaConfig(num_layers=80, num_heads=64, num_heads_kv=8, head_dim=128, ffn_dim=28672)


def to_bf16_bits(x: np.ndarray) -> np.ndarray:
    """float32 -> bfloat16 bit pattern (uint16), round-to-nearest-even."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    r = ((u >> 16) & 1) + np.uint32(0x7FFF)
    return ((u + r) >> 16).astype(np.uint16)


def quantize_int8(w: np.ndarray):
    """Converter-side weight quantization (model_spec.py:222-243): scale = 127/amax per output row."""
    amax = np.max(np.abs(w), axis=1).astype(np.float32)
    amax[amax == 0] = 127.0
    scale = (np.float32(127.0) / amax).astype(np.float32)
    return np.rint(w * scale[:, None]).astype(np.int8), scale


class ModelWriter:
    """Streams variables into model.bin without holding the whole model in memory."""

    def __init__(self, model_dir: str, spec: str = "TransformerDecoderSpec", revision: int = 8):
        os.makedirs(model_dir, exist_ok=True)
        self.dir = model_dir
        self.f = open(os.path.join(model_dir, "model.bin"), "wb")
        self.count = 0
        self.aliases = []
        self.f.write(struct.pack("I", BINARY_VERSION))
        self._str(spec)
        self.f.write(struct.pack("I", revision))
        self._count_pos = self.f.tell()
        self.f.write(struct.pack("I", 0))

    def _str(self, s: str):
        b = s.encode("utf-8")
        self.f.write(struct.pack("H", len(b) + 1))
        self.f.write(b)
        self.f.write(b"\0")

    def add(self, name: str, value, dtype: Optional[str] = None):
        a = np.asarray(value)
        dtype = dtype or str(a.dtype)
        if dtype == "bfloat16" and a.dtype != np.uint16:
            a = to_bf16_bits(a.astype(np.float32))
        elif dtype != "bfloat16" and str(a.dtype) != dtype:
            a = a.astype(dtype)
        if a.ndim > 0:
            a = np.ascontiguousarray(a)   # (ascontiguousarray would promote a 0-d scalar to 1-d)
        if a.nbytes >= 2 ** 32:
            raise ValueError(f"variable {name} is too large for the model.bin format")
        self._str(name)
        self.f.write(struct.pack("B", a.ndim))
        for d in a.shape:
            self.f.write(struct.pack("I", d))
        self.f.write(struct.pack("B", _TYPE_IDS[dtype]))
        self.f.write(struct.pack("I", a.nbytes))
        self.f.write(memoryview(a).cast("B") if a.ndim > 0 else a.tobytes())
        self.count += 1

    def alias(self, alias: str, target: str):
        self.aliases.append((alias, target))

    def close(self, config: Dict, vocabulary):
        self.f.write(struct.pack("I", len(self.aliases)))
        for a, t in self.aliases:
            self._str(a)
            self._str(t)
        self.f.seek(self._count_pos)
        self.f.write(struct.pack("I", self.count))
        self.f.close()
        with open(os.path.join(self.dir, "config.json"), "w") as f:
            json.dump(config, f, indent=2, sort_keys=True)
        with open(os.path.join(self.dir, "vocabulary.json"), "w") as f:
            json.dump(list(vocabulary), f)


def write_llama_model(model_dir: str, cfg: LlamaConfig, quantization: str = "int8_float16",
                      seed: int = 1234, init_std: float = 0.02, fast_int8: bool = False,
                      extra: Optional[Dict] = None, omit=(), embedding_std: Optional[float] = None,
                      residual_std: Optional[float] = None) -> None:
    """Writes a random-init Llama-class model directory.

    quantization: "int8" / "int8_float32" / "int8_float16" / "int8_bfloat16" (int8 linear + embedding
    weights with fp32 row scales, norms in the float type), or "float32" / "float16" / "bfloat16".
    extra / omit: additional variables {name: numpy value} written after the standard ones / names left out (loader tests
    build model directories with features the engine must refuse).
    fast_int8: draw int8 weights and scales directly (same distribution as quantizing N(0, std^2)
    rows whose amax sits near 4 sigma) instead of quantizing an fp32 draw — used for the 8B bench
    model where generating 8e9 gaussians on the host would dominate the run.
    embedding_std / residual_std: standard deviation of the embedding rows and of the two matrices that write into the
    residual stream (attention linear_1, ffn linear_1); default init_std.  With init_std everywhere a deep random model is
    chaotic (every layer's update is ~100x the embedding it started from: fp16-level input differences grow to 20 % of
    the logits after 32 layers, measured against the reference's own float16 vs int8 runs), which no trained checkpoint is;
    embedding_std = 1 with a small residual_std keeps perturbations bounded so whole-model comparisons are meaningful.
    """
    emb_std = init_std if embedding_std is None else embedding_std
    res_std = init_std if residual_std is None else residual_std
    rng = np.random.default_rng(seed)
    awq_layout = {"awq_gemm": 1, "awq_gemv": 2}.get(quantization, 0)
    if awq_layout:
        return _write_llama_awq(model_dir, cfg, awq_layout, seed, init_std, fast_int8, emb_std, res_std)
    is_int8 = quantization.startswith("int8")
    ftype = {"int8": "float32", "int8_float32": "float32", "int8_float16": "float16",
             "int8_bfloat16": "bfloat16"}.get(quantization, quantization)
    d, D = cfg.d_model, cfg.head_dim
    w = ModelWriter(model_dir)
    _add = w.add
    if omit:
        w.add = lambda name, value, dtype=None: None if name in omit else _add(name, value, dtype)

    base = rng.integers(-127, 128, size=1 << 24, dtype=np.int8) if fast_int8 else None
    state = {"off": 0}

    def fast_block(count):
        # numpy's generators run at ~0.1 GB/s on the bench hosts; the 8 GB of int8 weights are instead tiled
        # from a 16 MiB random block at a different (odd) offset per matrix — memcpy speed, still no two rows alike
        out = np.empty(count, np.int8)
        pos = 0
        while pos < count:
            off = state["off"]
            take = min(count - pos, base.size - off)
            out[pos:pos + take] = base[off:off + take]
            pos += take
            state["off"] = (off + take + 12289) % base.size
        return out

    def linear(prefix, n, k, std=None):
        std = init_std if std is None else std
        if is_int8 and fast_int8:
            # uniform int8 in [-127,127] (std 73.3) with scale = 73.3/std: the dequantized weights have
            # standard deviation init_std; drawn directly as bytes (about 1 GB/s on one host core)
            q = fast_block(n * k).reshape(n, k)
            q[:, 0] = 127    # each row attains its amax, as a real quantized row does
            scale = np.full((n,), 73.3 / std, np.float32) * rng.uniform(0.9, 1.1, size=n).astype(np.float32)
            w.add(prefix + "/weight", q, "int8")
            w.add(prefix + "/weight_scale", scale, "float32")
            return
        wt = (rng.standard_normal((n, k), dtype=np.float32) * np.float32(std))
        if is_int8:
            q, scale = quantize_int8(wt)
            w.add(prefix + "/weight", q, "int8")
            w.add(prefix + "/weight_scale", scale, "float32")
        else:
            w.add(prefix + "/weight", wt, ftype)

    w.add("decoder/activation", np.int8(2))                      # common_spec.Activation.SWISH
    w.add("decoder/alibi", np.int8(0))
    w.add("decoder/alibi_use_positive_positions", np.int8(0))
    w.add("decoder/alignment_heads", np.int16(1))
    w.add("decoder/alignment_layer", np.int16(-1))
    linear("decoder/embeddings", cfg.vocab_size, d, emb_std)
    gamma0 = None
    for l in range(cfg.num_layers):
        p = f"decoder/layer_{l}/"
        g = (1.0 + 0.1 * rng.standard_normal(d)).astype(np.float32)
        w.add(p + "ffn/layer_norm/gamma", g, ftype)
        linear(p + "ffn/linear_0", cfg.ffn_dim, d)
        linear(p + "ffn/linear_0_noact", cfg.ffn_dim, d)
        linear(p + "ffn/linear_1", d, cfg.ffn_dim, res_std)
        g = (1.0 + 0.1 * rng.standard_normal(d)).astype(np.float32)
        w.add(p + "self_attention/layer_norm/gamma", g, ftype)
        linear(p + "self_attention/linear_0", (cfg.num_heads + 2 * cfg.num_heads_kv) * D, d)
        linear(p + "self_attention/linear_1", d, cfg.num_heads * D, res_std)
        w.add(p + "self_attention/num_heads_kv", np.int32(cfg.num_heads_kv))
        w.add(p + "self_attention/head_dim", np.int32(cfg.head_dim))
        w.add(p + "self_attention/rotary_base", np.float32(cfg.rotary_base))
        w.add(p + "self_attention/rotary_dim", np.int32(0))
        w.add(p + "self_attention/rotary_interleave", np.int8(0))
        if cfg.rotary_scaling_type >= 0:
            w.add(p + "self_attention/rotary_scaling_type", np.int8(cfg.rotary_scaling_type))
            w.add(p + "self_attention/rotary_scaling_factor", np.float32(cfg.rotary_scaling_factor))
            w.add(p + "self_attention/rotary_low_freq_factor", np.float32(cfg.rotary_low_freq_factor))
            w.add(p + "self_attention/rotary_high_freq_factor", np.float32(cfg.rotary_high_freq_factor))
            w.add(p + "self_attention/original_max_position_embeddings",
                  np.int32(cfg.original_max_position_embeddings))
    g = (1.0 + 0.1 * rng.standard_normal(d)).astype(np.float32)
    w.add("decoder/layer_norm/gamma", g, ftype)
    w.add("decoder/num_heads", np.int16(cfg.num_heads))
    w.add("decoder/pre_norm", np.int8(1))
    linear("decoder/projection", cfg.vocab_size, d)
    w.add("decoder/scale_alibi", np.int8(0))
    w.add("decoder/scale_embeddings", np.int8(0))
    w.add("decoder/start_from_zero_embedding", np.int8(0))
    for name, value in (extra or {}).items():
        _add(name, value)
    config = {"bos_token": "<t1>", "eos_token": "<t2>", "unk_token": "<t0>",
              "layer_norm_epsilon": cfg.rms_eps, "multi_query_attention": cfg.num_heads_kv != cfg.num_heads}
    w.close(config, (f"<t{i}>" for i in range(cfg.vocab_size)))


AWQ_ORDER = np.array([0, 4, 1, 5, 2, 6, 3, 7])


def _pack_nibbles(m: np.ndarray, order) -> np.ndarray:
    """[rows, cols] values 0..15 -> int32 [rows, cols/8]; element 8c+i goes to nibble order[i]."""
    r, c = m.shape
    m = m.reshape(r, c // 8, 8).astype(np.uint32)
    out = np.zeros((r, c // 8), np.uint32)
    for i in range(8):
        out |= (m[:, :, i] & 0xF) << np.uint32(4 * order[i])
    return out.view(np.int32)


def _write_llama_awq(model_dir, cfg, layout, seed, init_std, fast, emb_std=None, res_std=None):
    """AWQ-INT4 (group 128) Llama directory as the AutoAWQ -> CTranslate2 converter lays it out
    (converters/transformers.py:1697-1843 with quant_type AWQ_GEMM / AWQ_GEMV): linear layers carry int32
    `weight` + float16 `weight_scale` + int32 `weight_zero`; embeddings, norms and lm_head stay float16;
    config.json records quantization_type / bits / group size (src/models/model.cc:636-637)."""
    rng = np.random.default_rng(seed)
    emb_std = init_std if emb_std is None else emb_std
    res_std = init_std if res_std is None else res_std
    G = 128
    d, D = cfg.d_model, cfg.head_dim
    w = ModelWriter(model_dir)
    base = rng.integers(0, 16, size=1 << 22, dtype=np.uint8)
    off = [0]

    def nibbles(rows, cols):
        n = rows * cols
        reps = -(-(n + off[0]) // base.size)
        a = np.tile(base, reps)[off[0]:off[0] + n].reshape(rows, cols)
        off[0] = (off[0] + 7919) % base.size
        return a

    packed_cache = {}

    def linear(prefix, n, k, std=None):
        std = init_std if std is None else std
        if fast and (n, k, std) in packed_cache:
            # bench-sized models: layers of the same shape share one set of packed arrays (packing 7e9 nibbles in
            # numpy takes minutes; the values do not matter for a throughput measurement)
            for suffix, (arr, dt) in packed_cache[(n, k, std)].items():
                w.add(prefix + suffix, arr, dt)
            return
        _linear(prefix, n, k, std)

    def _linear(prefix, n, k, std):
        scales = (rng.uniform(0.6, 1.4, size=(k // G, n)) * (std / 2.5)).astype(np.float16)
        zeros = rng.integers(6, 10, size=(k // G, n))
        q = nibbles(k, n)                                   # [K, N] values 0..15
        if layout == 1:
            arrays = {"/weight": (_pack_nibbles(q, AWQ_ORDER), "int32"), "/weight_scale": (scales, "float16"),
                      "/weight_zero": (_pack_nibbles(zeros, AWQ_ORDER), "int32")}
        else:
            ng = k // G
            zw = -(-ng // 8)
            zp = np.zeros((n, zw * 8), np.int64)
            zp[:, :ng] = zeros.T
            sp = np.zeros((n, zw * 8), np.float16)
            sp[:, :ng] = scales.T
            arrays = {"/weight": (_pack_nibbles(np.ascontiguousarray(q.T), np.arange(8)), "int32"),
                      "/weight_scale": (sp, "float16"), "/weight_zero": (_pack_nibbles(zp, np.arange(8)), "int32")}
        for suffix, (arr, dt) in arrays.items():
            w.add(prefix + suffix, arr, dt)
        if fast:
            packed_cache[(n, k, std)] = arrays

    def dense_f16(prefix, n, k, std=None):
        reps = -(-(n * k) // (1 << 22))
        vals = (np.tile(base, reps)[:n * k].astype(np.float32) - 7.5) * ((init_std if std is None else std) / 4.6)
        w.add(prefix + "/weight", vals.reshape(n, k), "float16")

    w.add("decoder/activation", np.int8(2))
    w.add("decoder/alibi", np.int8(0))
    w.add("decoder/alibi_use_positive_positions", np.int8(0))
    w.add("decoder/alignment_heads", np.int16(1))
    w.add("decoder/alignment_layer", np.int16(-1))
    dense_f16("decoder/embeddings", cfg.vocab_size, d, emb_std)
    for l in range(cfg.num_layers):
        p = f"decoder/layer_{l}/"
        w.add(p + "ffn/layer_norm/gamma", (1.0 + 0.1 * rng.standard_normal(d)).astype(np.float32), "float16")
        linear(p + "ffn/linear_0", cfg.ffn_dim, d)
        linear(p + "ffn/linear_0_noact", cfg.ffn_dim, d)
        linear(p + "ffn/linear_1", d, cfg.ffn_dim, res_std)
        w.add(p + "self_attention/layer_norm/gamma", (1.0 + 0.1 * rng.standard_normal(d)).astype(np.float32), "float16")
        linear(p + "self_attention/linear_0", (cfg.num_heads + 2 * cfg.num_heads_kv) * D, d)
        linear(p + "self_attention/linear_1", d, cfg.num_heads * D, res_std)
        w.add(p + "self_attention/num_heads_kv", np.int32(cfg.num_heads_kv))
        w.add(p + "self_attention/head_dim", np.int32(cfg.head_dim))
        w.add(p + "self_attention/rotary_base", np.float32(cfg.rotary_base))
        w.add(p + "self_attention/rotary_dim", np.int32(0))
        w.add(p + "self_attention/rotary_interleave", np.int8(0))
        if cfg.rotary_scaling_type >= 0:
            w.add(p + "self_attention/rotary_scaling_type", np.int8(cfg.rotary_scaling_type))
            w.add(p + "self_attention/rotary_scaling_factor", np.float32(cfg.rotary_scaling_factor))
            w.add(p + "self_attention/rotary_low_freq_factor", np.float32(cfg.rotary_low_freq_factor))
            w.add(p + "self_attention/rotary_high_freq_factor", np.float32(cfg.rotary_high_freq_factor))
            w.add(p + "self_attention/original_max_position_embeddings",
                  np.int32(cfg.original_max_position_embeddings))
    w.add("decoder/layer_norm/gamma", (1.0 + 0.1 * rng.standard_normal(d)).astype(np.float32), "float16")
    w.add("decoder/num_heads", np.int16(cfg.num_heads))
    w.add("decoder/pre_norm", np.int8(1))
    dense_f16("decoder/projection", cfg.vocab_size, d)
    w.add("decoder/scale_alibi", np.int8(0))
    w.add("decoder/scale_embeddings", np.int8(0))
    w.add("decoder/start_from_zero_embedding", np.int8(0))
    config = {"bos_token": "<t1>", "eos_token": "<t2>", "unk_token": "<t0>", "layer_norm_epsilon": cfg.rms_eps,
              "multi_query_attention": cfg.num_heads_kv != cfg.num_heads, "quantization_type": layout,
              "quantization_bits": 4, "quantization_group_size": G}
    w.close(config, (f"<t{i}>" for i in range(cfg.vocab_size)))


# ---------------------------------------------------------------------------------------------
# Encoder-decoder Transformer directories (TransformerSpec revision 7, python/ctranslate2/specs/transformer_spec.py:477-560):
# the variable set the OpenNMT-py / Marian (OPUS-MT) converters emit — LayerNorm with beta, biased Dense layers, ReLU or
# Swish FFN, sinusoidal positions (no stored encodings), embeddings scaled by sqrt(d), optional shared vocabulary.
# ---------------------------------------------------------------------------------------------
@dataclass
class TransformerConfig:
    encoder_layers: int = 6
    decoder_layers: int = 6
    num_heads: int = 8
    d_model: int = 512
    ffn_dim: int = 2048
    source_vocab: int = 58101
    target_vocab: int = 58101
    pre_norm: bool = False                 # Marian / OPUS-MT transformers are post-norm (converters/marian.py:41)
    activation: int = 0                    # common_spec.Activation: RELU = 0, SWISH = 2
    start_from_zero_embedding: bool = False
    add_source_eos: bool = False
    layer_norm_epsilon: Optional[float] = None


OPUS_MT_BASE = TransformerConfig(pre_norm=False, activation=2, start_from_zero_embedding=True, add_source_eos=True)


def write_transformer_model(model_dir: str, cfg: TransformerConfig, quantization: str = "int8", seed: int = 1234,
                            init_std: float = 0.05, emb_std: float = 0.3, alignment_layer: int = -1,
                            alignment_heads: int = 1) -> None:
    """Writes a random-init encoder-decoder Transformer directory (model.bin v6 + config.json + vocabularies).
    alignment_layer / alignment_heads: the decoder's alignment attention (a negative layer counts from the end, 0 heads =
    all of them); the defaults are the converters' own."""
    rng = np.random.default_rng(seed)
    is_int8 = quantization.startswith("int8")
    ftype = {"int8": "float32", "int8_float32": "float32", "int8_float16": "float16",
             "int8_bfloat16": "bfloat16"}.get(quantization, quantization)
    d = cfg.d_model
    w = ModelWriter(model_dir, spec="TransformerSpec", revision=7)

    def linear(prefix, n, k, std=init_std, bias=True):
        wt = (rng.standard_normal((n, k), dtype=np.float32) * np.float32(std))
        if is_int8:
            q, scale = quantize_int8(wt)
            w.add(prefix + "/weight", q, "int8")
            w.add(prefix + "/weight_scale", scale, "float32")
        else:
            w.add(prefix + "/weight", wt, ftype)
        if bias:
            w.add(prefix + "/bias", (0.02 * rng.standard_normal(n)).astype(np.float32), ftype)

    def norm(prefix):
        w.add(prefix + "/gamma", (1.0 + 0.1 * rng.standard_normal(d)).astype(np.float32), ftype)
        w.add(prefix + "/beta", (0.05 * rng.standard_normal(d)).astype(np.float32), ftype)

    def attention(prefix, cross):
        norm(prefix + "/layer_norm")
        if cross:
            linear(prefix + "/linear_0", d, d)
            linear(prefix + "/linear_1", 2 * d, d)
            linear(prefix + "/linear_2", d, d)
        else:
            linear(prefix + "/linear_0", 3 * d, d)
            linear(prefix + "/linear_1", d, d)

    def ffn(prefix):
        norm(prefix + "/layer_norm")
        linear(prefix + "/linear_0", cfg.ffn_dim, d)
        linear(prefix + "/linear_1", d, cfg.ffn_dim)

    for scope, layers in (("encoder", cfg.encoder_layers), ("decoder", cfg.decoder_layers)):
        w.add(scope + "/num_heads", np.int16(cfg.num_heads))
        w.add(scope + "/pre_norm", np.int8(cfg.pre_norm))
        w.add(scope + "/activation", np.int8(cfg.activation))
        w.add(scope + "/scale_embeddings", np.int8(1))
        if scope == "encoder":
            w.add("encoder/embeddings_merge", np.int8(0))
            linear("encoder/embeddings_0", cfg.source_vocab, d, std=emb_std, bias=False)
        else:
            w.add("decoder/alignment_layer", np.int16(alignment_layer))
            w.add("decoder/alignment_heads", np.int16(alignment_heads))
            w.add("decoder/alibi", np.int8(0))
            w.add("decoder/alibi_use_positive_positions", np.int8(0))
            w.add("decoder/scale_alibi", np.int8(0))
            w.add("decoder/start_from_zero_embedding", np.int8(cfg.start_from_zero_embedding))
            linear("decoder/embeddings", cfg.target_vocab, d, std=emb_std, bias=False)
            linear("decoder/projection", cfg.target_vocab, d, std=emb_std / 4)
        if cfg.pre_norm:
            norm(scope + "/layer_norm")
        for l in range(layers):
            p = f"{scope}/layer_{l}"
            attention(p + "/self_attention", False)
            if scope == "decoder":
                attention(p + "/attention", True)
            ffn(p + "/ffn")
    config = {"bos_token": "<s>", "eos_token": "</s>", "unk_token": "<unk>", "add_source_bos": False,
              "add_source_eos": cfg.add_source_eos, "decoder_start_token": "<s>"}
    if cfg.layer_norm_epsilon is not None:
        config["layer_norm_epsilon"] = cfg.layer_norm_epsilon
    specials = ["<unk>", "<s>", "</s>"]
    w.close(config, [])
    os.remove(os.path.join(model_dir, "vocabulary.json"))
    for name, n in (("source_vocabulary", cfg.source_vocab), ("target_vocabulary", cfg.target_vocab)):
        with open(os.path.join(model_dir, name + ".json"), "w") as f:
            json.dump(specials + [f"<t{i}>" for i in range(3, n)], f)


# ---------------------------------------------------------------------------------------------
# Whisper directories (WhisperSpec revision 3, python/ctranslate2/specs/whisper_spec.py:26-78): Conv1D front-end (weights kept
# in float, as the reference does on CUDA, src/models/model.cc:204-223), pre-norm GELU encoder with stored positions, a
# TransformerDecoderSpec decoder with cross-attention, stored positions, unscaled embeddings tied to the output projection.
# ---------------------------------------------------------------------------------------------
@dataclass
class WhisperConfig:
    encoder_layers: int = 32
    decoder_layers: int = 32
    num_heads: int = 20
    d_model: int = 1280
    n_mels: int = 128
    max_source_positions: int = 1500       # frames after the stride-2 convolution (30 s of audio)
    max_target_positions: int = 448
    text_tokens: int = 50257               # ids below <|endoftext|>
    languages: int = 100
    timestamps: int = 1501


WHISPER_LARGE_V3 = WhisperConfig()


def whisper_vocabulary(cfg: WhisperConfig):
    """Token order of the Whisper tokenizers: text, <|endoftext|>, <|startoftranscript|>, languages, <|translate|>,
    <|transcribe|>, <|startoflm|>, <|startofprev|>, <|nospeech|>, <|notimestamps|>, timestamps (src/models/whisper.cc:75-80)."""
    toks = [f"<t{i}>" for i in range(cfg.text_tokens)] + ["<|endoftext|>", "<|startoftranscript|>"]
    toks += [f"<|l{i}|>" for i in range(cfg.languages)]
    toks += ["<|translate|>", "<|transcribe|>", "<|startoflm|>", "<|startofprev|>", "<|nospeech|>", "<|notimestamps|>"]
    toks += ["<|%.2f|>" % (0.02 * i) for i in range(cfg.timestamps)]
    return toks


def write_whisper_model(model_dir: str, cfg: WhisperConfig, quantization: str = "int8", seed: int = 1234,
                        init_std: float = 0.15, emb_std: float = 0.02) -> None:
    rng = np.random.default_rng(seed)
    is_int8 = quantization.startswith("int8")
    ftype = {"int8": "float32", "int8_float32": "float32", "int8_float16": "float16",
             "int8_bfloat16": "bfloat16"}.get(quantization, quantization)
    d, F = cfg.d_model, 4 * cfg.d_model
    vocab = whisper_vocabulary(cfg)
    V = len(vocab)
    w = ModelWriter(model_dir, spec="WhisperSpec", revision=3)

    def linear(prefix, n, k, std=init_std, bias=True):
        wt = (rng.standard_normal((n, k), dtype=np.float32) * np.float32(std))
        if is_int8:
            q, scale = quantize_int8(wt)
            w.add(prefix + "/weight", q, "int8")
            w.add(prefix + "/weight_scale", scale, "float32")
        else:
            w.add(prefix + "/weight", wt, ftype)
        if bias:
            w.add(prefix + "/bias", (0.02 * rng.standard_normal(n)).astype(np.float32), ftype)

    def norm(prefix):
        w.add(prefix + "/gamma", (1.0 + 0.1 * rng.standard_normal(d)).astype(np.float32), ftype)
        w.add(prefix + "/beta", (0.05 * rng.standard_normal(d)).astype(np.float32), ftype)

    def conv(prefix, cout, cin):
        w.add(prefix + "/weight", (rng.standard_normal((cout, cin, 3), dtype=np.float32) * np.float32(1.0 / np.sqrt(3 * cin))), ftype)
        w.add(prefix + "/bias", (0.02 * rng.standard_normal(cout)).astype(np.float32), ftype)

    w.add("encoder/num_heads", np.int16(cfg.num_heads))
    conv("encoder/conv1", d, cfg.n_mels)
    conv("encoder/conv2", d, d)
    w.add("encoder/position_encodings/encodings", (0.1 * rng.standard_normal((cfg.max_source_positions, d))).astype(np.float32), ftype)
    norm("encoder/layer_norm")
    for l in range(cfg.encoder_layers):
        p = f"encoder/layer_{l}"
        norm(p + "/self_attention/layer_norm")
        linear(p + "/self_attention/linear_0", 3 * d, d)
        linear(p + "/self_attention/linear_1", d, d)
        norm(p + "/ffn/layer_norm")
        linear(p + "/ffn/linear_0", F, d)
        linear(p + "/ffn/linear_1", d, F)
    w.add("decoder/num_heads", np.int16(cfg.num_heads))
    w.add("decoder/pre_norm", np.int8(1))
    w.add("decoder/activation", np.int8(3))                  # GELU
    w.add("decoder/alignment_layer", np.int16(-1))
    w.add("decoder/alignment_heads", np.int16(1))
    w.add("decoder/scale_embeddings", np.int8(0))
    w.add("decoder/alibi", np.int8(0))
    w.add("decoder/alibi_use_positive_positions", np.int8(0))
    w.add("decoder/scale_alibi", np.int8(0))
    w.add("decoder/start_from_zero_embedding", np.int8(0))
    # small embeddings: with the projection tied to them, large ones make every step repeat its input token
    linear("decoder/embeddings", V, d, std=emb_std, bias=False)
    w.add("decoder/position_encodings/encodings", (0.1 * rng.standard_normal((cfg.max_target_positions, d))).astype(np.float32), ftype)
    # a large output-norm gain gives the tied projection logits of order 1 (decisive, input-dependent tokens)
    w.add("decoder/layer_norm/gamma", (0.25 / emb_std * (1.0 + 0.1 * rng.standard_normal(d))).astype(np.float32), ftype)
    w.add("decoder/layer_norm/beta", (0.05 * rng.standard_normal(d)).astype(np.float32), ftype)
    for l in range(cfg.decoder_layers):
        p = f"decoder/layer_{l}"
        norm(p + "/self_attention/layer_norm")
        linear(p + "/self_attention/linear_0", 3 * d, d)
        linear(p + "/self_attention/linear_1", d, d)
        norm(p + "/attention/layer_norm")
        linear(p + "/attention/linear_0", d, d)
        linear(p + "/attention/linear_1", 2 * d, d)
        linear(p + "/attention/linear_2", d, d)
        norm(p + "/ffn/layer_norm")
        linear(p + "/ffn/linear_0", F, d)
        linear(p + "/ffn/linear_1", d, F)
    # the output projection is the embedding matrix (converters/transformers.py WhisperLoader ties them)
    w.alias("decoder/projection/weight", "decoder/embeddings/weight")
    eot = cfg.text_tokens
    config = {"suppress_ids": [1, 2, 7, 8, 9, eot + 1, eot + 2 + cfg.languages, eot + 3 + cfg.languages, eot + 4 + cfg.languages,
                               eot + 5 + cfg.languages, eot + 6 + cfg.languages],
              "suppress_ids_begin": [3, eot], "lang_ids": list(range(eot + 2, eot + 2 + cfg.languages)),
              "alignment_heads": [[cfg.decoder_layers - 1, 0]]}
    w.close(config, vocab)


# ---------------------------------------------------------------------------------------------
# Encoder-only directories (TransformerEncoderModelSpec revision 1, spec name TransformerEncoderSpec,
# python/ctranslate2/specs/transformer_spec.py:771-812), laid out as the BertLoader emits them
# (python/ctranslate2/converters/transformers.py:3295-3330): token and token-type embeddings merged by ADD, unscaled,
# stored positions, layernorm_embedding, post-norm GELU layers, pooler_dense + Tanh.
# ---------------------------------------------------------------------------------------------
@dataclass
class EncoderConfig:
    num_layers: int = 12
    num_heads: int = 12
    d_model: int = 768
    ffn_dim: int = 3072
    vocab_size: int = 30522
    type_vocab_size: int = 2               # 0 = one embedding table (no token types)
    max_positions: int = 512
    pre_norm: bool = False                 # pre-norm adds the final encoder/layer_norm
    activation: int = 3                    # common_spec.Activation: RELU = 0, GELUTanh = 1, GELU = 3
    pooler: bool = True
    layernorm_embedding: bool = True
    layer_norm_epsilon: float = 1e-12


BERT_BASE = EncoderConfig()


def write_encoder_model(model_dir: str, cfg: EncoderConfig, quantization: str = "int8", seed: int = 1234,
                        init_std: float = 0.05, emb_std: float = 0.5) -> None:
    """Writes a random-init TransformerEncoderSpec directory (model.bin v6 + config.json + vocabulary.json)."""
    rng = np.random.default_rng(seed)
    is_int8 = quantization.startswith("int8")
    ftype = {"int8": "float32", "int8_float32": "float32", "int8_float16": "float16",
             "int8_bfloat16": "bfloat16"}.get(quantization, quantization)
    d = cfg.d_model
    w = ModelWriter(model_dir, spec="TransformerEncoderSpec", revision=1)

    def linear(prefix, n, k, std=init_std, bias=True):
        wt = (rng.standard_normal((n, k), dtype=np.float32) * np.float32(std))
        if is_int8:
            q, scale = quantize_int8(wt)
            w.add(prefix + "/weight", q, "int8")
            w.add(prefix + "/weight_scale", scale, "float32")
        else:
            w.add(prefix + "/weight", wt, ftype)
        if bias:
            w.add(prefix + "/bias", (0.02 * rng.standard_normal(n)).astype(np.float32), ftype)

    def norm(prefix):
        w.add(prefix + "/gamma", (1.0 + 0.1 * rng.standard_normal(d)).astype(np.float32), ftype)
        w.add(prefix + "/beta", (0.05 * rng.standard_normal(d)).astype(np.float32), ftype)

    w.add("encoder/num_heads", np.int16(cfg.num_heads))
    w.add("encoder/pre_norm", np.int8(cfg.pre_norm))
    w.add("encoder/activation", np.int8(cfg.activation))
    w.add("encoder/embeddings_merge", np.int8(1))             # ADD
    w.add("encoder/scale_embeddings", np.int8(0))
    if cfg.type_vocab_size:
        linear("encoder/embeddings_0", cfg.vocab_size, d, std=emb_std, bias=False)
        linear("encoder/embeddings_1", cfg.type_vocab_size, d, std=emb_std, bias=False)
    else:
        linear("encoder/embeddings", cfg.vocab_size, d, std=emb_std, bias=False)
    w.add("encoder/position_encodings/encodings", (0.1 * rng.standard_normal((cfg.max_positions, d))).astype(np.float32), ftype)
    if cfg.layernorm_embedding:
        norm("encoder/layernorm_embedding")
    if cfg.pre_norm:
        norm("encoder/layer_norm")
    for l in range(cfg.num_layers):
        p = f"encoder/layer_{l}"
        norm(p + "/self_attention/layer_norm")
        linear(p + "/self_attention/linear_0", 3 * d, d)
        linear(p + "/self_attention/linear_1", d, d)
        norm(p + "/ffn/layer_norm")
        linear(p + "/ffn/linear_0", cfg.ffn_dim, d)
        linear(p + "/ffn/linear_1", d, cfg.ffn_dim)
    if cfg.pooler:
        linear("pooler_dense", d, d)
        w.add("pooler_activation", np.int8(5))                  # Tanh
    config = {"unk_token": "[UNK]", "bos_token": "[CLS]", "eos_token": "[SEP]", "multi_query_attention": False,
              "layer_norm_epsilon": cfg.layer_norm_epsilon}
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]"] + [f"<t{i}>" for i in range(4, cfg.vocab_size)]
    w.close(config, vocab)
