"""-m gpu, one device: what loading a decoder-only model puts on the GPU, read back through the C-ABI.  Every rank of a
tensor-parallel group is opened on the same device (tp_rank / tp_size set directly, no tp_connect, no forward pass), and its
weight_bytes is checked against the shard sizes computed here from the geometry: the replicated parts whole, the QKV_ROWS /
ROWS / COLS parts divided by the world size.  This pins the INT8, float and AWQ shard cuts on a one-GPU box."""
import ctypes

import pytest

from ctranslate2_b200._lib import GeneratorConfig, check, lib
from ctranslate2_b200.converters.synthetic import LlamaConfig, write_llama_model
from gpu_util import gpu

F32, F16, BF16 = 0, 1, 2
STORED, INT8, FLOAT = 0, 1, 2
ES = {F32: 4, F16: 2, BF16: 2}
AWQ_GROUP = 128
# heads, kv heads and FFN width divisible by 4; d_model / 4 and ffn / 4 multiples of the AWQ group size
CFG = LlamaConfig(num_layers=2, num_heads=8, num_heads_kv=4, head_dim=64, ffn_dim=1024, vocab_size=256)
# (storage, activation dtype, weight type): every compute type each storage accepts (AWQ runs float16 activations only)
CASES = [(q, d, wt) for q in ("int8", "float16") for d in (F32, F16, BF16) for wt in (STORED, INT8, FLOAT)] + \
        [(q, F16, wt) for q in ("awq_gemm", "awq_gemv") for wt in (STORED, INT8, FLOAT)]


@pytest.fixture(scope="module")
def models(tmp_path_factory):
    out = {}
    for q in ("int8", "float16", "awq_gemm", "awq_gemv"):
        d = str(tmp_path_factory.mktemp(q))
        write_llama_model(d, CFG, q, seed=5)
        out[q] = d
    return out


def expected_weight_bytes(storage, dtype, weight_type, world):
    es, d, F, V = ES[dtype], CFG.d_model, CFG.ffn_dim, CFG.vocab_size
    qkv, attn = (CFG.num_heads + 2 * CFG.num_heads_kv) * CFG.head_dim, CFG.num_heads * CFG.head_dim

    def dense(n, k, layer):
        if layer and storage.startswith("awq"):   # packed int32 [n, k / 8] + f16 scales and zeros [n, k / group]
            return n * (k // 8) * 4 + 2 * n * (k // AWQ_GROUP) * 2
        if weight_type == INT8 or (weight_type == STORED and storage == "int8"):
            return n * k + 4 * n                  # int8 [n, k] + f32 row scales
        return n * k * es

    per_layer = (dense(qkv // world, d, True) + dense(d, attn // world, True) + 2 * dense(F // world, d, True)
                 + dense(d, F // world, True) + 2 * d * es)
    return 2 * dense(V, d, False) + d * es + CFG.num_layers * per_layer


def weight_bytes(model_dir, dtype, weight_type, rank, world):
    cfg = GeneratorConfig(0, dtype, 1, 16, rank, world, 0, 0, weight_type)
    h = lib().ct2b200_generator_open(model_dir.encode(), ctypes.byref(cfg))
    if not h:
        raise RuntimeError(lib().ct2b200_last_error().decode())
    try:
        wb = ctypes.c_int64(0)
        check(lib().ct2b200_generator_info(ctypes.c_void_p(h), None, None, None, None, None, ctypes.byref(wb)))
        return wb.value
    finally:
        lib().ct2b200_generator_close(ctypes.c_void_p(h))


@gpu
@pytest.mark.parametrize("storage,dtype,weight_type", CASES)
def test_weight_bytes_of_every_shard(models, storage, dtype, weight_type):
    for world in (1, 2, 4):
        want = expected_weight_bytes(storage, dtype, weight_type, world)
        for rank in range(world):
            got = weight_bytes(models[storage], dtype, weight_type, rank, world)
            assert got == want, (storage, dtype, weight_type, world, rank, got, want)
