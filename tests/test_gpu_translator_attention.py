"""Translator.translate_batch with return_attention, replace_unknowns and coverage_penalty on the GPU: the alignment attention
is written inside the captured search step (attention_generic_kernel's kAlign instantiation + align_mean_kernel), followed
through the beam reordering by the hypotheses' ancestry, and turned into coverage terms and returned rows at collect.
Against (a) the committed outputs of the UNMODIFIED reference (tests/golden/seq2seq_attention_ref.json), (b) the attention
oracle run live (tests/seq2seq_attention.py), and (c) invariants that hold in every compute type."""
import json
import os

import numpy as np
import pytest

from ctranslate2_b200.translator import Translator
from gpu_util import gpu
from seq2seq_attention import AttentionOracle, coverage_term, translate as oracle_translate

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
START, END = 1, 2
POSTNORM = os.path.join(GOLDEN, "tiny_seq2seq_postnorm")
ALIGN = os.path.join(GOLDEN, "tiny_seq2seq_align")


@pytest.fixture(scope="module")
def fixture():
    with open(os.path.join(GOLDEN, "seq2seq_attention_ref.json")) as f:
        return json.load(f)


def _run(t, c, **kw):
    res = t.translate_batch(c["sources"], beam_size=c["beam_size"], num_hypotheses=c["num_hypotheses"],
                            max_decoding_length=c["max_length"], min_decoding_length=c["min_length"],
                            length_penalty=c["length_penalty"], coverage_penalty=c["coverage_penalty"],
                            return_end_token=c["return_end_token"], return_attention=c["return_attention"],
                            replace_unknowns=c["replace_unknowns"], return_scores=True, **kw)
    return [r.hypotheses for r in res], [r.scores for r in res], [r.attention for r in res]


def _ragged(seed, n, lo, hi):
    rng = np.random.default_rng(seed)
    return [[int(x) for x in rng.integers(lo, hi, size=int(rng.integers(3, 16)))] for _ in range(n)]


@gpu
@pytest.mark.parametrize("name", ["aren", "postnorm", "align"])
def test_float32_equals_the_reference(fixture, name):
    entry = fixture[name]
    t = Translator(os.path.join(GOLDEN, entry["model"]), compute_type="float32")
    rows = 0
    for c in entry["cases"]:
        hyps, scores, attention = _run(t, c)
        assert hyps == c["hypotheses"], c
        for s, w in zip(scores, c["scores"]):
            np.testing.assert_allclose(s, w, atol=2e-4)
        assert len(attention) == len(c["attention"])
        for a, w in zip(attention, c["attention"]):
            assert len(a) == len(w)
            for x, y in zip(a, w):
                assert len(x) == len(y)
                rows += len(x)
                if x:
                    np.testing.assert_allclose(np.array(x), np.array(y), atol=1e-5)
    assert rows > 200
    t.close()


@gpu
@pytest.mark.parametrize("beam", [1, 4, 10])
def test_ragged_batches_match_the_oracle(beam):
    """16 ragged sources x 40 steps in float32 against the oracle: tokens, scores and raw attention rows."""
    t = Translator(ALIGN, compute_type="float32")
    oracle = AttentionOracle.from_dir(ALIGN, compute_type="float32")
    srcs = _ragged(40 + beam, 16, 3, 120)
    S = max(len(s) for s in srcs)
    for cov in (0.0, 0.3):
        ids, lens, scores, att = t.translate_ids(srcs, beam_size=beam, num_hypotheses=1, max_decoding_length=40,
                                                 min_decoding_length=40, return_end_token=True, return_attention=True,
                                                 coverage_penalty=cov)
        want = oracle_translate(oracle, srcs, beam_size=beam, max_length=40, min_length=40, coverage_penalty=cov,
                                return_end_token=True, bos=START, eos=END)
        for b, w in enumerate(want):
            toks, score, rows = w[0]
            assert ids[b, 0, :lens[b, 0]].tolist() == toks
            assert abs(float(scores[b, 0]) - score) < 2e-4
            np.testing.assert_allclose(att[b, 0, :len(toks), :S], np.array(rows), atol=1e-4)
    t.close()


@gpu
@pytest.mark.parametrize("compute", ["float16", "bfloat16", "int8_float16"])
def test_rows_are_distributions_over_the_source(compute):
    t = Translator(ALIGN, compute_type=compute)
    srcs = _ragged(7, 12, 3, 120)
    ids, lens, scores, att = t.translate_ids(srcs, beam_size=4, num_hypotheses=2, max_decoding_length=30,
                                             return_end_token=True, return_attention=True)
    tol = 2e-2 if compute == "bfloat16" else 4e-3
    for b, s in enumerate(srcs):
        for h in range(2):
            n = int(lens[b, h])
            assert n >= 1
            np.testing.assert_allclose(att[b, h, :n, :len(s)].sum(axis=1), 1.0, atol=tol)
            assert (att[b, h, :n, len(s):] == 0).all()
            assert (att[b, h, n:] == 0).all()
    t.close()


@gpu
def test_attention_leaves_ids_and_scores_bitwise_alone():
    t = Translator(POSTNORM, compute_type="float32")
    srcs = _ragged(11, 9, 3, 120)
    for beam in (1, 3, 8, 12):
        a = t.translate_ids(srcs, beam_size=beam, num_hypotheses=min(beam, 2), max_decoding_length=24)
        b = t.translate_ids(srcs, beam_size=beam, num_hypotheses=min(beam, 2), max_decoding_length=24, return_attention=True)
        for x, y in zip(a, b[:3]):
            np.testing.assert_array_equal(x, y)
    t.close()


@gpu
@pytest.mark.parametrize("lp", [1.0, 0.0])
def test_coverage_scores_follow_the_finalize_formula(lp):
    t = Translator(ALIGN, compute_type="float32")
    srcs = _ragged(13, 8, 3, 120)
    beta = 0.4
    plain = t.translate_ids(srcs, beam_size=5, num_hypotheses=5, max_decoding_length=20, length_penalty=lp,
                            return_end_token=True, return_attention=True)
    ids, lens, scores, att = t.translate_ids(srcs, beam_size=5, num_hypotheses=5, max_decoding_length=20, length_penalty=lp,
                                             return_end_token=True, return_attention=True, coverage_penalty=beta)
    for b in range(len(srcs)):
        got = [float(scores[b, h]) for h in range(5) if lens[b, h] >= 0]
        assert got == sorted(got, reverse=True)
        for h in range(len(got)):
            n = int(lens[b, h])
            toks = ids[b, h, :n].tolist()
            base = None
            for k in range(5):                               # the same hypothesis in the call without the penalty
                if plain[1][b, k] == n and plain[0][b, k, :n].tolist() == toks:
                    base = float(plain[2][b, k])
            if base is not None:
                np.testing.assert_allclose(got[h], base + beta * coverage_term(att[b, h, :n]), atol=1e-4)
    t.close()


@gpu
def test_graph_on_and_off_agree():
    srcs = _ragged(17, 6, 3, 120)
    out = []
    for graph in (True, False):
        t = Translator(ALIGN, compute_type="float32", use_cuda_graph=graph)
        out.append(t.translate_ids(srcs, beam_size=4, num_hypotheses=2, max_decoding_length=20, return_attention=True,
                                   coverage_penalty=0.2))
        t.close()
    for x, y in zip(*out):
        np.testing.assert_array_equal(x, y)


@gpu
def test_beam_32_and_a_source_at_the_encoder_positions():
    t = Translator(ALIGN, compute_type="float32", max_positions=512)
    srcs = _ragged(19, 3, 3, 120)
    ids, lens, scores, att = t.translate_ids(srcs, beam_size=32, num_hypotheses=3, max_decoding_length=16,
                                             return_attention=True, coverage_penalty=0.1)
    for b, s in enumerate(srcs):
        n = int(lens[b, 0])
        np.testing.assert_allclose(att[b, 0, :n, :len(s)].sum(axis=1), 1.0, atol=1e-5)
    full = [list(np.random.default_rng(5).integers(3, 120, size=t._encoder_positions))]
    ids, lens, scores, att = t.translate_ids(full + srcs, beam_size=4, max_decoding_length=12, return_attention=True)
    assert att.shape[-1] == t._encoder_positions
    np.testing.assert_allclose(att[0, 0, :int(lens[0, 0])].sum(axis=1), 1.0, atol=1e-5)
    t.close()


@gpu
def test_plain_calls_are_unchanged_after_an_attention_call():
    from ctranslate2_b200.whisper import Whisper
    whisper = os.path.join(GOLDEN, "tiny_whisper")
    w = Whisper(whisper, compute_type="float32")
    x = (np.random.default_rng(500).standard_normal((2, 16, 60)) * 2).astype(np.float32)
    prompts = [[101, 102, 106, 110], [101, 103, 105, 110]]
    gen_before = w.generate(x, prompts, beam_size=3, max_length=24, return_scores=True)
    align_before = w._align(x, [101, 102, 106], [[87, 44, 38], [56, 83]], [60, 50], 7)
    t = Translator(POSTNORM, compute_type="float32")
    srcs = _ragged(23, 5, 3, 120)
    before = t.translate_ids(srcs, beam_size=4, num_hypotheses=2, max_decoding_length=20)
    t.translate_batch([["<t5>", "<t9>"] * 20], beam_size=6, return_attention=True, replace_unknowns=True,
                      coverage_penalty=0.5, max_decoding_length=60)
    after = t.translate_ids(srcs, beam_size=4, num_hypotheses=2, max_decoding_length=20)
    for a, b in zip(before, after):
        np.testing.assert_array_equal(a, b)
    t.close()
    gen_after = w.generate(x, prompts, beam_size=3, max_length=24, return_scores=True)
    align_after = w._align(x, [101, 102, 106], [[87, 44, 38], [56, 83]], [60, 50], 7)
    assert [r.sequences_ids for r in gen_before] == [r.sequences_ids for r in gen_after]
    assert [r.scores for r in gen_before] == [r.scores for r in gen_after]
    assert repr(align_before) == repr(align_after)
    w.close()
