"""-m gpu: Generator.score_batch (src/scoring.cc:6-66) and the fused LogSoftMax + Gather kernel behind it, against (1) the
committed scores of the unmodified reference on the tiny model, (2) float64 truth per kernel call, (3) the oracle over
sequences that need several prompt-pass chunks, (4) forward_batch's log-probabilities at full size (several lm_head slabs on
the prefill GEMM), (5) the same sequence scored alone and inside a ragged batch."""
import json
import os

import numpy as np
import pytest
import torch

import ctranslate2_b200 as ct2
from ctranslate2_b200 import ops
from ctranslate2_b200.converters.synthetic import LlamaConfig, write_llama_model
from oracle import ct2_oracle as O
from gpu_util import gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
TINY = os.path.join(GOLDEN, "tiny_llama_int8")
INT_VIEW = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16}


@gpu
def test_tiny_model_matches_reference_fixture():
    """Ragged batch, sequences of one and two tokens, offset 0 / 1 / 5: the reference's ScoringResult.log_probs."""
    fx = json.load(open(os.path.join(GOLDEN, "tiny_llama_int8_score_batch.json")))
    g = ct2.Generator(TINY, compute_type="int8_float32", max_batch_size=8, max_length=64)
    worst = 0.0
    for c in fx["cases"]:
        res = g.score_batch(c["sequences"], offset=c["offset"])
        assert [len(r.log_probs) for r in res] == [len(x) for x in c["log_probs"]]
        for seq, r, ref in zip(c["sequences"], res, c["log_probs"]):
            assert r.tokens == ["<t%d>" % t for t in seq[1 + c["offset"]:]]
            if ref:
                worst = max(worst, float(np.abs(np.array(r.log_probs) - np.array(ref)).max()))
    print("max |engine - reference| = %.3g" % worst)
    assert worst <= 5e-4, worst


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("vocab", [2000, 2001, 32000, 128256])
def test_log_softmax_gather_vs_float64(dtype, vocab):
    """float(T(log_softmax(x)[id])) within 1 ulp of T of the float64 value rounded to T.  V = 2001: a scalar tail on every row
    and rows that start off the 16-byte grid; the slab is also placed one element past an aligned address."""
    rows = 512 if vocab == 128256 else 4096
    g = torch.Generator(device="cuda").manual_seed(vocab)
    buf = torch.empty(rows * vocab + 1, dtype=dtype, device="cuda")
    x = buf[1:].view(rows, vocab)
    x.copy_(torch.randn(rows, vocab, generator=g, device="cuda") * 4)
    x[:, :7] += 12                                  # a few large logits per row, as a trained head has
    ids = torch.randint(0, vocab, (rows,), generator=g, device="cuda", dtype=torch.int32)
    got = ops.log_softmax_gather(x, ids)
    assert got.dtype == torch.float32 and got.shape == (rows,)
    truth = torch.log_softmax(x.double(), -1).gather(1, ids.long()[:, None])[:, 0].to(dtype)
    ulps = (got.to(dtype).view(INT_VIEW[dtype]).long() - truth.view(INT_VIEW[dtype]).long()).abs()
    assert torch.equal(got, got.to(dtype).float())          # the value is a T value
    assert int(ulps.max()) <= 1, int(ulps.max())
    # the unfused pair, LogSoftMax (softmax_kernel) then the gather, gives the same 16-bit values to the rounding step; in
    # fp32 it differs by its own fp32 running sums
    ref = ops.LogSoftMax()(x.contiguous()).gather(1, ids.long()[:, None])[:, 0]
    unfused = (got.to(dtype).view(INT_VIEW[dtype]).long() - ref.view(INT_VIEW[dtype]).long()).abs()
    assert int(unfused.max()) <= (1 if dtype != torch.float32 else 16), int(unfused.max())


@gpu
@pytest.mark.parametrize("quant", ["float32", "float16"])
def test_long_sequences_across_prompt_pass_chunks_vs_oracle(tmp_path, quant):
    """8 ragged sequences of 1100-1900 tokens (more than the 8192-row activation arena, so several time chunks of the prompt
    pass, which forward_batch refuses) with offset 3, against the oracle.  Float weights: no int8 activation rounding to flip
    over 1900 positions."""
    d = str(tmp_path / quant)
    cfg = LlamaConfig(num_layers=2, num_heads=8, num_heads_kv=2, head_dim=128, ffn_dim=1536, vocab_size=1000,
                      rotary_scaling_type=2, rotary_scaling_factor=8.0, rotary_low_freq_factor=1.0,
                      rotary_high_freq_factor=4.0, original_max_position_embeddings=64)
    write_llama_model(d, cfg, quant, seed=5, init_std=0.05)
    r = np.random.default_rng(12)
    seqs = [r.integers(3, 1000, size=int(n)).tolist() for n in r.integers(1100, 1901, size=8)]
    assert sum(len(s) - 1 for s in seqs) > 8192
    g = ct2.Generator(d, compute_type=quant, max_batch_size=8, max_length=2048)
    with pytest.raises(ValueError):
        g.forward_batch([s[:-1] for s in seqs])
    res = g.score_batch(seqs, offset=3, max_input_length=0)
    m = O.LlamaOracle(O.DecoderWeights.from_dir(d, "cuda"))
    ref = m.score(seqs, offset=3)
    got = np.concatenate([x.log_probs for x in res])
    want = np.concatenate(ref)
    assert [len(x.log_probs) for x in res] == [len(x) for x in ref] == [len(s) - 4 for s in seqs]
    tol = 1e-3 if quant == "float32" else 4e-2
    err = np.abs(got - want)
    print("%s: max |engine - oracle| = %.3g, rms %.3g" % (quant, err.max(), np.sqrt(np.mean(err ** 2))))
    assert err.max() <= tol * max(1.0, np.abs(want).max()), err.max()
    assert np.sqrt(np.mean(err ** 2)) <= tol / 3 * max(1.0, np.sqrt(np.mean(want ** 2)))


def _f16_ulp(v):
    e = np.floor(np.log2(np.maximum(np.abs(v), 2.0 ** -14)))
    return 2.0 ** (e - 10)


@gpu
def test_full_size_llama8b_matches_forward_batch():
    """Llama-3-8B geometry, INT8: 2 x 700 tokens = 1398 scored rows, i.e. two lm_head slabs on the prefill GEMM, against
    forward_batch(return_log_probs=True) gathered at the targets (lm_head on the decode GEMM, LogSoftMax written out)."""
    import bench
    g = ct2.Generator(bench.model_dir("8b"), compute_type="int8_float16", max_batch_size=2, max_length=1024)
    V = g.vocab_size
    seqs = np.random.default_rng(77).integers(3, V, size=(2, 700))
    res = g.score_batch(seqs.tolist())
    got = np.array([x.log_probs for x in res], np.float64)
    assert got.shape == (2, 699)
    assert np.isfinite(got).all() and (got <= 0).all()
    lp = g.forward_batch(seqs[:, :-1].tolist(), return_log_probs=True)
    want = np.take_along_axis(lp, seqs[:, 1:, None], axis=2)[..., 0].astype(np.float64)
    err = np.abs(got - want)
    ulps = err / _f16_ulp(want)
    print("max |score_batch - forward_batch| = %.3g (%.1f fp16 ulp); %d of %d differ"
          % (err.max(), ulps.max(), int((err > 0).sum()), err.size))
    assert (err <= 2 * _f16_ulp(want) + 1e-5).all(), (err.max(), ulps.max())


@gpu
def test_batch_independence_and_later_generation():
    """A sequence scored alone equals the same sequence inside a ragged batch with other rows and an offset; a score_batch
    call between two generate_batch calls leaves the greedy decode (and its CUDA graph) as it was."""
    g = ct2.Generator(TINY, compute_type="int8_float32", max_batch_size=4, max_length=64)
    r = np.random.default_rng(5)
    seq = r.integers(3, 200, size=23).tolist()
    others = [r.integers(3, 200, size=n).tolist() for n in (40, 7, 1)]
    prompts = [[5, 9, 11, 40, 7], [8, 3, 77, 12, 6]]
    before = [x.sequences_ids[0] for x in g.generate_batch(prompts, max_length=10, min_length=10, end_token=[2])]
    alone = g.score_batch([seq])[0].log_probs
    batch = g.score_batch([others[0], seq, others[1], others[2]], offset=2)
    np.testing.assert_allclose(batch[1].log_probs, alone[2:], rtol=0, atol=1e-5)
    assert len(batch[3].log_probs) == 0 and len(batch[2].log_probs) == 4
    after = [x.sequences_ids[0] for x in g.generate_batch(prompts, max_length=10, min_length=10, end_token=[2])]
    assert after == before
