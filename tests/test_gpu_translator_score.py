"""Translator.score_batch on the GPU: the teacher-forced decoder pass (causal self-attention over all target positions,
launch_attention_causal) against
  (a) Translator::score_batch of the UNMODIFIED reference (tests/golden/seq2seq_score_ref.json, tools/make_golden.py
      --translator-score-only), token strings in and out;
  (b) the oracle's cached one-token path with teacher forcing (tests/seq2seq_scoring.py) on targets long enough to need
      several logits slabs and several decoder passes;
  (c) the engine's own one-token path: the sum of the scores of a greedy translation equals its score.
Float32 has no activation quantization, so every score agrees to 2e-4.  INT8 on a d = 32 / 64 model turns a rounding flip
into ~1e-2 of a score now and then (see test_gpu_translator.py), so int8 scores are pinned by a bound on most of them and a
looser bound on all (on aren-transliteration-i8, whose binary version 2 truncates in the activation quantizer, fewer than half
of the int8 scores agree to 2e-2; the greatest difference seen is 0.16)."""
import json
import os

import numpy as np
import pytest

from ctranslate2_b200.translator import Translator
from oracle import ct2_oracle as O
from gpu_util import gpu
from seq2seq_scoring import oracle_score

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
POST = os.path.join(GOLDEN, "tiny_seq2seq_postnorm")
AREN = os.path.join(GOLDEN, "aren-transliteration")
START, END = 1, 2


@pytest.fixture(scope="module")
def fixture():
    with open(os.path.join(GOLDEN, "seq2seq_score_ref.json"), encoding="utf-8") as f:
        return json.load(f)


@gpu
@pytest.mark.parametrize("name", ["aren-float32", "aren-int8", "postnorm-float32", "postnorm-int8"])
def test_scores_match_the_reference(fixture, name):
    m = fixture["models"][name]
    t = Translator(os.path.join(GOLDEN, m["model"]), compute_type=m["compute_type"])
    got, want = [], []
    for c in m["cases"]:
        res = t.score_batch(c["source"], c["target"], max_input_length=c["max_input_length"], offset=c["offset"])
        for r, toks, lp in zip(res, c["tokens"], c["log_probs"]):
            assert r.tokens == toks
            assert len(r.log_probs) == len(lp)
            got += r.log_probs
            want += lp
    t.close()
    err = np.abs(np.array(got) - np.array(want))
    assert len(err) > 150
    if m["compute_type"] == "float32":
        assert err.max() <= 2e-4, err.max()
    else:
        assert np.mean(err <= 0.1) >= 0.9 and err.max() <= 0.3, (np.mean(err <= 0.1), np.median(err), err.max())


@gpu
@pytest.mark.parametrize("compute,atol", [("float32", 2e-4), ("float16", 0.1)])
def test_long_targets_match_the_oracle(compute, atol):
    """16 pairs with 100-400-token targets: several decoder passes and several logits slabs per pass."""
    rng = np.random.default_rng(3)
    srcs = [[int(x) for x in rng.integers(3, 120, size=int(rng.integers(5, 30)))] for _ in range(16)]
    tgts = [[int(x) for x in rng.integers(3, 96, size=int(rng.integers(100, 401)))] for _ in range(16)]
    t = Translator(POST, compute_type=compute)
    res = t.score_batch(srcs, tgts)
    t.close()
    oracle = O.Seq2SeqOracle.from_dir(POST, compute_type="float32")
    want = oracle_score(oracle, srcs, [[START] + x + [END] for x in tgts])
    err = np.concatenate([np.abs(np.array(r.log_probs) - np.array(w)) for r, w in zip(res, want)])
    assert len(err) == sum(len(x) + 1 for x in tgts)
    assert err.max() <= atol, err.max()
    if compute == "float16":
        assert err.mean() <= 0.02, err.mean()


@gpu
def test_sum_of_scores_equals_the_greedy_translation_score():
    """The cached one-token path (translate_batch) and the causal pass (score_batch) compute the same log-probabilities."""
    t = Translator(AREN, compute_type="float32")
    rng = np.random.default_rng(4)
    srcs = [[int(x) for x in rng.integers(4, 51, size=int(rng.integers(3, 12)))] for _ in range(16)]
    tr = t.translate_batch(srcs, beam_size=1, min_decoding_length=0, length_penalty=0, return_scores=True,
                           max_decoding_length=64)
    done = [b for b, r in enumerate(tr) if len(r.hypotheses_ids[0]) < 64]       # ended with </s>
    assert len(done) >= 12
    res = t.score_batch([srcs[b] for b in done], [tr[b].hypotheses_ids[0] for b in done])
    for b, r in zip(done, res):
        assert r.tokens == tr[b].hypotheses[0] + ["</s>"]
        assert abs(sum(r.log_probs) - tr[b].scores[0]) <= 1e-4, (b, sum(r.log_probs), tr[b].scores[0])
    t.close()


@gpu
@pytest.mark.parametrize("offset", [0, 2])
def test_a_pair_alone_equals_the_pair_in_a_ragged_batch(offset):
    rng = np.random.default_rng(6)
    srcs = [[int(x) for x in rng.integers(3, 120, size=int(rng.integers(1, 40)))] for _ in range(9)]
    tgts = [[int(x) for x in rng.integers(3, 96, size=int(rng.integers(0, 60)))] for _ in range(9)]
    t = Translator(POST, compute_type="float32")
    batch = t.score_batch(srcs, tgts, offset=offset)
    for s, g, r in zip(srcs, tgts, batch):
        alone = t.score_batch([s], [g], offset=offset)[0]
        assert alone.tokens == r.tokens
        np.testing.assert_allclose(alone.log_probs, r.log_probs, atol=1e-5, rtol=0)
    t.close()


@gpu
def test_scoring_between_translations_changes_nothing():
    t = Translator(os.path.join(GOLDEN, "aren-transliteration-i8"), compute_type="int8")
    rng = np.random.default_rng(8)
    srcs = [[int(x) for x in rng.integers(4, 51, size=int(rng.integers(3, 12)))] for _ in range(6)]
    first = t.translate_batch(srcs, beam_size=4, num_hypotheses=2, return_scores=True)
    long_src = [[int(x) for x in rng.integers(4, 51, size=200)]] * 3               # grows the arena past the translate one
    t.score_batch(long_src + srcs, [[int(x) for x in rng.integers(3, 30, size=300)]] * 3 + [r.hypotheses_ids[0] for r in first])
    second = t.translate_batch(srcs, beam_size=4, num_hypotheses=2, return_scores=True)
    assert [r.hypotheses_ids for r in first] == [r.hypotheses_ids for r in second]
    assert [r.scores for r in first] == [r.scores for r in second]
    t.close()


@gpu
def test_position_table_overflow_raises():
    t = Translator(POST, compute_type="float32", max_positions=512)
    positions = t._decoder_positions
    assert positions >= 500
    ok = [5] * (positions - 1)                                                     # <s> + tokens + </s>: `positions` inputs
    assert len(t.score_batch([[5, 6]], [ok], max_input_length=0)[0].log_probs) == positions
    with pytest.raises(ValueError):
        t.score_batch([[5, 6]], [ok + [7]], max_input_length=0)
    t.close()


@gpu
def test_scoring_many_short_pairs_leaves_the_search_state_alone():
    """A pass of short pairs holds up to 4096 / (longest side) pairs.  Scoring sizes only the encoder and activation rows of
    one pass and its logits slab; the beam-search state (beam arena, self-attention K/V of batch x beam x steps per decoder
    layer, logits) keeps the size the translations gave it, before and after scoring."""
    import torch
    torch.cuda.init()
    t = Translator(POST, compute_type="float32")
    rng = np.random.default_rng(9)
    srcs = [[int(x) for x in rng.integers(3, 120, size=int(rng.integers(3, 12)))] for _ in range(8)]
    first = t.translate_batch(srcs, beam_size=4, max_decoding_length=256, return_scores=True)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    short_src = [[int(x) for x in rng.integers(3, 120, size=int(rng.integers(1, 5)))] for _ in range(3000)]
    short_tgt = [[int(x) for x in rng.integers(3, 96, size=int(rng.integers(0, 3)))] for _ in range(3000)]
    res = t.score_batch(short_src, short_tgt)
    assert sum(len(r.log_probs) for r in res) == sum(len(x) + 1 for x in short_tgt)
    second = t.translate_batch(srcs, beam_size=4, max_decoding_length=256, return_scores=True)
    torch.cuda.synchronize()
    grown = free0 - torch.cuda.mem_get_info()[0]
    # one pass: 4096 activation / encoder rows of d = 64 (a few MB) and a 1024-row logits slab; search state for the ~1000
    # pairs of a pass would be 4 beams x 256 steps x 64 x 4 B x 2 (K, V) x 2 layers per pair, about 1 GB
    assert grown <= 96 << 20, grown
    assert [r.hypotheses_ids for r in first] == [r.hypotheses_ids for r in second]
    assert [r.scores for r in first] == [r.scores for r in second]
    t.close()
