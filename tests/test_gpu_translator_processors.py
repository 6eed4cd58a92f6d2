"""Translator.translate_batch with repetition_penalty, no_repeat_ngram_size, disable_unk and suppress_sequences on the GPU
(the processors run inside beam_mask_row, in the captured search step), against (a) the committed outputs of the
UNMODIFIED reference (tests/golden/seq2seq_processors_ref.json, tools/make_golden.py --seq2seq-processors-only), (b) the
processor-aware oracle run live (tests/seq2seq_processors.py), (c) the reference's own SearchVariantTest cases
(tests/translator_test.cc:256-341), and (d) invariants that hold in every compute type.

Parity classes as in tests/test_gpu_translator.py: float32 hypotheses equal the reference's and scores agree to 2e-4; int8
on these d = 32 / 64 models is pinned by a majority agreement."""
import json
import os

import numpy as np
import pytest

from ctranslate2_b200.translator import Translator
from oracle import ct2_oracle as O
from gpu_util import gpu
from seq2seq_processors import translate as oracle_translate

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
START, END = 1, 2
AREN = os.path.join(GOLDEN, "aren-transliteration")
SOURCE = ["آ", "ت", "ز", "م", "و", "ن"]
COMPUTE = ["int8", "int8_float16", "float16", "bfloat16", "float32"]
OPTIONS = ("repetition_penalty", "no_repeat_ngram_size", "disable_unk", "suppress_sequences")


@pytest.fixture(scope="module")
def fixture():
    with open(os.path.join(GOLDEN, "seq2seq_processors_ref.json")) as f:
        return json.load(f)


def _run(t, c, **kw):
    opts = {k: c[k] for k in OPTIONS if k in c}
    res = t.translate_batch(c["sources"], beam_size=c["beam_size"], num_hypotheses=c["num_hypotheses"],
                            max_decoding_length=c["max_length"], min_decoding_length=c["min_length"],
                            length_penalty=c["length_penalty"], return_scores=True, **opts, **kw)
    return [r.hypotheses for r in res], [r.scores for r in res]


def _ngrams(tokens, n):
    return [tuple(tokens[i:i + n]) for i in range(len(tokens) - n + 1)]


def _contains(tokens, seq):
    return any(tokens[i:i + len(seq)] == seq for i in range(len(tokens) - len(seq) + 1))


@gpu
@pytest.mark.parametrize("name", ["aren", "postnorm"])
def test_float32_processors_equal_the_reference(fixture, name):
    entry = fixture[name]
    t = Translator(os.path.join(GOLDEN, entry["model"]), compute_type="float32")
    total = 0
    for c in entry["models"]["float32"]["cases"]:
        hyps, scores = _run(t, c)
        assert hyps == c["hypotheses"], c
        for s, w in zip(scores, c["scores"]):
            np.testing.assert_allclose(s, w, atol=2e-4)
            total += len(s)
    assert total > 200
    t.close()


@gpu
@pytest.mark.parametrize("name", ["aren", "postnorm"])
def test_int8_processors_agree_with_reference_statistically(fixture, name):
    entry = fixture[name]
    t = Translator(os.path.join(GOLDEN, entry["model"]), compute_type="int8")
    same = total = close = 0
    for c in entry["models"]["int8"]["cases"]:
        hyps, scores = _run(t, c)
        for b in range(len(hyps)):
            total += 1
            same += hyps[b][:1] == c["hypotheses"][b][:1]
            close += abs(scores[b][0] - c["scores"][b][0]) < 0.1
    assert same / total >= 0.7, (same, total)
    assert close / total >= 0.6, (close, total)
    t.close()


@gpu
@pytest.mark.parametrize("compute", COMPUTE)
def test_invariants_in_every_compute_type(compute):
    """No hypothesis holds a repeated n-gram, a suppressed sequence or <unk> under disable_unk, whatever the rounding."""
    t = Translator(os.path.join(GOLDEN, "tiny_seq2seq_postnorm"), compute_type=compute)
    rng = np.random.default_rng(11)
    srcs = [["<t%d>" % i for i in rng.integers(3, 120, size=int(rng.integers(3, 14)))] for _ in range(6)]
    plain = t.translate_batch(srcs, beam_size=4, max_decoding_length=30)
    top = [r.hypotheses[0] for r in plain]
    seqs = [top[0][:1], top[1][1:3], top[2][2:5]]
    for beam in (1, 4, 10):
        nh = min(beam, 2)
        for n in (1, 2, 3):
            for r in t.translate_batch(srcs, beam_size=beam, num_hypotheses=nh, max_decoding_length=30,
                                       no_repeat_ngram_size=n):
                for h in r.hypotheses:
                    assert len(set(_ngrams(h, n))) == len(_ngrams(h, n)), (compute, beam, n, h)
        for r in t.translate_batch(srcs, beam_size=beam, num_hypotheses=nh, max_decoding_length=30,
                                   suppress_sequences=seqs, disable_unk=True, repetition_penalty=1.3):
            for h in r.hypotheses:
                assert "<unk>" not in h and not any(_contains(h, s) for s in seqs), (compute, beam, h)
    t.close()


@gpu
@pytest.mark.parametrize("beam", [1, 4])
def test_reference_search_variant_cases(beam):
    """tests/translator_test.cc:256-341 (SearchVariantTest) on aren-transliteration."""
    t = Translator(AREN)
    res = t.translate_batch([SOURCE], beam_size=beam, suppress_sequences=[["o"], ["t", "z", "m"]])
    assert res[0].hypotheses[0] == ["a", "t", "z", "u", "m", "u", "n"]
    with pytest.raises(ValueError):
        t.translate_batch([SOURCE], beam_size=beam, suppress_sequences=[["o"], ["t", "oovtoken", "m"]])
    toks = t.translate_batch([["ن"] * 5], beam_size=beam, repetition_penalty=100)[0].hypotheses[0]
    assert len(set(toks)) == len(toks)
    out = "".join(t.translate_batch([["ن"] * 50], beam_size=beam, no_repeat_ngram_size=3)[0].hypotheses[0])
    assert len({out[i:i + 3] for i in range(len(out) - 3)}) == len(out) - 3
    t.close()


@gpu
@pytest.mark.parametrize("beam,nh", [(4, 3), (7, 2), (10, 2)])
def test_processors_match_oracle_on_long_batches(beam, nh):
    """16 sources, 40 steps, vs the processor-aware oracle live (float32); beam 4 and 7 take the one-pass scoring kernel,
    beam 10 the LogSoftMax + TopK path."""
    mdir = os.path.join(GOLDEN, "tiny_seq2seq_postnorm")
    t = Translator(mdir, compute_type="float32")
    oracle = O.Seq2SeqOracle.from_dir(mdir, compute_type="float32")
    rng = np.random.default_rng(5 + beam)
    srcs = [[int(x) for x in rng.integers(3, 120, size=int(rng.integers(3, 30)))] for _ in range(16)]
    opts = dict(repetition_penalty=1.25, no_repeat_ngram_size=2, disable_ids=[0], suppress_sequences=[[33], [13, 89], [5, 6, 7]])
    ids, lens, scores = t.translate_ids(srcs, beam_size=beam, num_hypotheses=nh, max_decoding_length=40, min_decoding_length=5,
                                        start_id=START, end_token=[END], **opts)
    want = oracle_translate(oracle, srcs, beam_size=beam, num_hypotheses=nh, max_length=40, min_length=5, bos=START, eos=END,
                            **opts)
    for b, w in enumerate(want):
        assert [ids[b, h, :lens[b, h]].tolist() for h in range(len(w))] == [x[0] for x in w]
        np.testing.assert_allclose(scores[b, :len(w)], [x[1] for x in w], atol=3e-4)
    t.close()


@gpu
def test_cuda_graph_and_eager_steps_agree(fixture):
    cases = fixture["postnorm"]["models"]["float32"]["cases"]
    mdir = os.path.join(GOLDEN, "tiny_seq2seq_postnorm")
    a = Translator(mdir, compute_type="float32", use_cuda_graph=True)
    b = Translator(mdir, compute_type="float32", use_cuda_graph=False)
    for c in cases[::3]:
        assert _run(a, c) == _run(b, c)
        assert _run(a, c)[0] == c["hypotheses"]
    a.close()
    b.close()


@gpu
def test_no_state_leaks_into_later_calls():
    """A call without processors after calls with them equals the same call on a fresh Translator, and the Generator's beam
    search and Whisper are unchanged by a processed translation."""
    import ctranslate2_b200 as ct2
    mdir = os.path.join(GOLDEN, "tiny_seq2seq_postnorm")
    rng = np.random.default_rng(3)
    srcs = [["<t%d>" % i for i in rng.integers(3, 120, size=int(rng.integers(3, 14)))] for _ in range(5)]
    kw = dict(beam_size=4, num_hypotheses=2, max_decoding_length=24, return_scores=True)
    fresh = Translator(mdir, compute_type="float16")
    want = fresh.translate_batch(srcs, **kw)
    fresh.close()

    gen = ct2.Generator(os.path.join(GOLDEN, "tiny_llama_int8"), compute_type="int8_float32", max_batch_size=4, max_length=64)
    prompts = [[5, 9, 13], [7, 8, 11]]
    gen_before = gen.generate_batch(prompts, max_length=10, beam_size=4, end_token=[2])
    whisper_dir = os.path.join(GOLDEN, "tiny_whisper")
    w = ct2.Whisper(whisper_dir, compute_type="float32")
    feats = (np.random.default_rng(1).standard_normal((1, w.n_mels, 2 * w.max_frames)) * 2).astype(np.float32)
    prompt = [["<|startoftranscript|>", "<|l0|>", "<|transcribe|>", "<|notimestamps|>"]]
    w_before = w.generate(feats, prompt, beam_size=3, max_length=40)

    t = Translator(mdir, compute_type="float16")
    t.translate_batch(srcs, repetition_penalty=0.6, no_repeat_ngram_size=1, disable_unk=True,
                      suppress_sequences=[["<t33>"], ["<t13>", "<t89>"]], **kw)
    t.translate_batch(srcs[:2], repetition_penalty=1.4, **kw)
    got = t.translate_batch(srcs, **kw)
    assert [r.hypotheses for r in got] == [r.hypotheses for r in want]
    assert [r.scores for r in got] == [r.scores for r in want]
    t.close()

    assert [r.sequences_ids for r in gen.generate_batch(prompts, max_length=10, beam_size=4, end_token=[2])] == \
        [r.sequences_ids for r in gen_before]
    assert [r.sequences_ids for r in w.generate(feats, prompt, beam_size=3, max_length=40)] == \
        [r.sequences_ids for r in w_before]
    w.close()
