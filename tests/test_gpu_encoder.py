"""-m gpu: encoder-only models on the device.

  * ct2b200_attention_encoder_mma against a float64 restatement of dot_product_attention with a padding mask
    (src/layers/attention.cc:178-287).  Keys and values past every row's length are NaN, so reading one (a mask that is off
    by one upwards, a key tile that should have been skipped) turns a checked output into NaN; the last valid key of every
    row carries most of the weight and a value of +3, so dropping it (off by one downwards) moves the output by O(1).
  * Encoder.forward_batch against the reference's Encoder::forward_batch (tests/golden/encoder_ref.npz).
  * A BERT-base-shaped model (d 768, 12 heads of 64, 64 ragged rows up to 512 tokens) against EncoderOracle: the path that
    selects the tensor-core attention in float16 / int8_float16.
  * Batching invariance, and the Translator and Generator unchanged after an Encoder ran in the same process."""
import math
import os

import numpy as np
import pytest
import torch

import ctranslate2_b200 as ct2
from ctranslate2_b200 import ops
from ctranslate2_b200.converters.synthetic import EncoderConfig, write_encoder_model
from encoder_oracle import EncoderOracle, load_fixture
from gpu_util import DEV, TDT, TOL, gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIXTURE = load_fixture(os.path.join(GOLDEN, "encoder_ref.npz"))


# ---------------- the attention op ----------------
def _attention_inputs(B, T, H, D, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    lens = torch.randint(1, T + 1, (B,), generator=g)
    lens[0] = T
    lens[-1] = 1 if B > 1 else T
    q = torch.randn(B, T, H, D, generator=g, dtype=torch.float64)
    u = torch.randn(B, 1, H, D, generator=g, dtype=torch.float64)
    q = u + 0.3 * q                                              # every query shares a direction u per (b, h)
    k = 0.3 * torch.randn(B, T, H, D, generator=g, dtype=torch.float64)
    v = torch.randn(B, T, H, D, generator=g, dtype=torch.float64)
    for b in range(B):
        n = int(lens[b])
        a = math.log(n) + 1.0                                    # score of the last valid key ~ a, the others ~ 0
        k[b, n - 1] = u[b, 0] * (a * math.sqrt(D) / (u[b, 0] ** 2).sum(-1, keepdim=True))
        v[b, n - 1] = 3.0
        k[b, n:] = float("nan")
        v[b, n:] = float("nan")
    return q, k, v, lens


def _reference(q, k, v, lens):
    B, T, H, D = q.shape
    s = torch.einsum("bthd,bshd->bhts", q, k) / math.sqrt(D)
    mask = torch.arange(T)[None, :] >= lens[:, None]             # [B, S]
    s = s.masked_fill(mask[:, None, None, :], float("-inf"))
    p = torch.softmax(s, -1)
    return torch.einsum("bhts,bshd->bthd", p, torch.nan_to_num(v))


@gpu
@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("T", [1, 13, 64, 65, 512])
@pytest.mark.parametrize("B", [1, 7, 64])
def test_attention_mma_against_float64(B, T, D, dtype):
    H = 2
    q, k, v, lens = _attention_inputs(B, T, H, D, seed=B * 1000 + T * 10 + D)
    qkv = torch.cat([q, k, v], dim=2).reshape(B * T, 3 * H * D).to(DEV, TDT[dtype])
    # the reference sees the inputs the kernel sees (rounded to T)
    r = qkv.double().cpu().reshape(B, T, 3, H, D)
    ref = _reference(r[:, :, 0], r[:, :, 1], r[:, :, 2], lens)
    out = ops.attention_encoder_mma(qkv, H, D, B, lengths=lens.to(DEV, torch.int32)).double().cpu().reshape(B, T, H, D)
    assert torch.isfinite(out).all()                             # rows past the length too
    for b in range(B):
        n = int(lens[b])
        err = (out[b, :n] - ref[b, :n]).abs().max().item()
        assert err < TOL[dtype] * 3.0, (b, n, err)              # outputs reach |3|: tolerance class on that scale
    # power: dropping the last valid key moves the outputs by far more than the bound
    b = 0
    n = int(lens[b])
    if n > 1:
        short = _reference(r[b:b + 1, :, 0], r[b:b + 1, :, 1], r[b:b + 1, :, 2], torch.tensor([n - 1]))
        assert (short[0, :n] - ref[b, :n]).abs().max().item() > 10 * TOL[dtype] * 3.0


@gpu
def test_attention_mma_without_lengths_and_refusals():
    B, T, H, D = 3, 70, 4, 64
    q, k, v, _ = _attention_inputs(B, T, H, D, seed=5)
    lens = torch.full((B,), T)
    k, v = torch.nan_to_num(k), torch.nan_to_num(v)             # every key is valid without lengths
    qkv = torch.cat([q, k, v], dim=2).reshape(B * T, 3 * H * D).to(DEV, torch.float16)
    r = qkv.double().cpu().reshape(B, T, 3, H, D)
    ref = _reference(r[:, :, 0], r[:, :, 1], r[:, :, 2], lens)
    out = ops.attention_encoder_mma(qkv, H, D, B).double().cpu().reshape(B, T, H, D)
    assert (out - ref).abs().max().item() < TOL["float16"] * 3.0
    # the generic kernel on the same inputs agrees
    gen = ops.attention_encoder(qkv, H, D, B).double().cpu().reshape(B, T, H, D)
    assert (out - gen).abs().max().item() < TOL["float16"] * 3.0
    with pytest.raises(ValueError):
        ops.attention_encoder_mma(qkv.float(), H, D, B)             # fp32
    with pytest.raises(ValueError):
        ops.attention_encoder_mma(qkv, 2 * H, D // 2, B)            # head_dim 32


# ---------------- forward_batch against the reference ----------------
def _run_case(enc, case):
    out = enc.forward_batch(case["ids"], token_type_ids=case["token_type_ids"])
    errs = []
    for b, row in enumerate(case["ids"]):
        ref = np.array(case["last_hidden_state"][b])
        errs.append(float(np.abs(out.last_hidden_state[b, :len(row)].reshape(-1) - ref).max()))
    perr = None
    if case["pooler_output"] is not None:
        perr = float(np.abs(out.pooler_output - np.array(case["pooler_output"])).max())
    else:
        assert out.pooler_output is None
    return errs, perr


@gpu
@pytest.mark.parametrize("name", list(FIXTURE))
def test_forward_batch_float32_matches_the_reference(name):
    enc = ct2.Encoder(os.path.join(GOLDEN, name), compute_type="float32")
    for case in FIXTURE[name]:
        if case["compute_type"] != "float32":
            continue
        errs, perr = _run_case(enc, case)
        assert max(errs) < 2e-4, errs
        assert perr is None or perr < 2e-4, perr
    enc.close()


@gpu
@pytest.mark.parametrize("name", list(FIXTURE))
def test_forward_batch_int8_and_float16_within_bounds(name):
    """int8: the reference's int8 compute, up to the rounding flips of INT8 activations; float16 (the tensor-core attention
    runs here: head_dim 64): against the reference's float32, within the half-precision class of a LayerNorm output."""
    for compute, ref_compute, bound in (("int8", "int8", 0.1), ("float16", "float32", 0.05)):
        enc = ct2.Encoder(os.path.join(GOLDEN, name), compute_type=compute)
        for case in FIXTURE[name]:
            if case["compute_type"] != ref_compute:
                continue
            errs, perr = _run_case(enc, case)
            assert max(errs) < bound, (compute, errs)
            assert np.median(errs) < bound / 5, (compute, errs)
            assert perr is None or perr < bound, (compute, perr)
        enc.close()


# ---------------- BERT-base shape ----------------
@pytest.fixture(scope="module")
def bert_dir(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("bert") / "bert")
    write_encoder_model(path, EncoderConfig(num_layers=2, vocab_size=8000), "int8", seed=3)
    return path


def _rel_rms(a, b):
    return float(np.sqrt(np.mean((a - b) ** 2)) / np.sqrt(np.mean(b ** 2)))


@gpu
@pytest.mark.parametrize("compute,bound", [("float32", 1e-4), ("float16", 2e-2), ("int8_float16", 0.1)])
def test_bert_base_shape_against_the_oracle(bert_dir, compute, bound):
    rng = np.random.default_rng(1)
    B = 64
    lens = rng.integers(32, 513, B)
    lens[0], lens[1], lens[2] = 512, 1, 300
    ids = [rng.integers(0, 8000, n).tolist() for n in lens]
    types = [rng.integers(0, 2, n).tolist() for n in lens]
    enc = ct2.Encoder(bert_dir, compute_type=compute, max_batch_size=64)
    out = enc.forward_batch(ids, token_type_ids=types)
    enc.close()
    assert np.isfinite(out.last_hidden_state).all() and np.isfinite(out.pooler_output).all()
    oracle = EncoderOracle.from_dir(bert_dir, compute_type="float32")
    for b in (0, 1, 2, 17):                                      # rows are independent: check a few against the oracle alone
        n = int(lens[b])
        h, p = oracle.forward(np.array([ids[b]]), np.array([n]), np.array([types[b]]))
        assert _rel_rms(out.last_hidden_state[b, :n], h[0]) < bound, (b, compute)
        assert _rel_rms(out.pooler_output[b], p[0]) < bound, (b, compute)


# ---------------- batching ----------------
@gpu
@pytest.mark.parametrize("compute", ["float32", "float16"])
def test_a_row_alone_equals_the_row_in_a_batch_and_in_a_rebatched_request(compute):
    path = os.path.join(GOLDEN, "tiny_encoder")
    rng = np.random.default_rng(4)
    rows = [rng.integers(0, 50, int(n)).tolist() for n in rng.integers(1, 17, 13)]
    rows[5] = rows[5][:1]
    enc = ct2.Encoder(path, compute_type=compute, max_batch_size=64)
    small = ct2.Encoder(path, compute_type=compute, max_batch_size=3)
    batch = enc.forward_batch(rows)
    rebatched = small.forward_batch(rows)
    tol = 1e-5 if compute == "float32" else 1e-2
    for b in (0, 5, 12):
        alone = enc.forward_batch([rows[b]])
        n = len(rows[b])
        for other in (batch, rebatched):
            assert np.abs(other.last_hidden_state[b, :n] - alone.last_hidden_state[0, :n]).max() < tol
            assert np.abs(other.pooler_output[b] - alone.pooler_output[0]).max() < tol
    enc.close()
    small.close()


# ---------------- other engines ----------------
@gpu
def test_translator_and_generator_unchanged_after_an_encoder():
    enc = ct2.Encoder(os.path.join(GOLDEN, "tiny_encoder"), compute_type="float16")
    enc.forward_batch([[5, 6, 7], [8]])
    from ctranslate2_b200.translator import Translator
    t = Translator(os.path.join(GOLDEN, "aren-transliteration-i8"), compute_type="int8")
    tr = t.translate_batch([["آ", "ت", "ز", "م", "و", "ن"]], beam_size=2, num_hypotheses=2,
                           max_decoding_length=20, return_scores=True)
    assert tr[0].hypotheses[0] == ["a", "t", "z", "m", "o", "n"], tr[0].hypotheses
    assert abs(tr[0].scores[0] + 0.1553) < 0.03, tr[0].scores
    t.close()
    fx = np.load(os.path.join(GOLDEN, "tiny_llama_int8_ref.npz"), allow_pickle=True)
    gen = ct2.Generator(os.path.join(GOLDEN, "tiny_llama_int8"), compute_type="int8_float32", max_batch_size=4, max_length=64)
    res = gen.generate_batch(fx["prompts"].tolist(), max_length=12, min_length=12, end_token=[2])
    assert [x.sequences_ids[0] for x in res] == fx["generated_min12"].tolist()
    enc.close()
