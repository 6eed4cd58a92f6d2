"""The logits processors of Translator::translate_batch restated on the oracle (tests/seq2seq_processors.py) against the
unmodified reference: the committed outputs of tests/golden/seq2seq_processors_ref.json (tools/make_golden.py
--seq2seq-processors-only) and, where oracle/_ref has been built, the reference run live on new cases.

float32 compute has no activation quantization, so every hypothesis must equal the reference's token for token and scores
agree to 1e-4."""
import json
import os

import numpy as np
import pytest

from ctranslate2_b200.translator import _load_vocabulary
from oracle import ct2_oracle as O
from seq2seq_processors import processors_hook, translate

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
START, END = 1, 2
f32 = np.float32


@pytest.fixture(scope="module")
def fixture():
    with open(os.path.join(GOLDEN, "seq2seq_processors_ref.json")) as f:
        return json.load(f)


class Vocab:
    def __init__(self, model_dir):
        self.src = {t: i for i, t in enumerate(_load_vocabulary(model_dir, "source_vocabulary"))}
        self.tgt_list = _load_vocabulary(model_dir, "target_vocabulary")
        self.tgt = {t: i for i, t in enumerate(self.tgt_list)}

    def options(self, c):
        """The case's processors in id form (the unknown token of a vocabulary without it lies past the output layer)."""
        unk = self.tgt.get("<unk>", len(self.tgt_list))
        seqs = [[self.tgt.get(t, unk) for t in s] for s in c.get("suppress_sequences", [])]
        return dict(repetition_penalty=c.get("repetition_penalty", 1.0), no_repeat_ngram_size=c.get("no_repeat_ngram_size", 0),
                    disable_ids=[unk] if c.get("disable_unk") and unk < len(self.tgt_list) else [],
                    suppress_sequences=[s for s in seqs if all(i < len(self.tgt_list) for i in s)])


def run_oracle(oracle, vocab, c):
    srcs = [[vocab.src[t] for t in r] for r in c["sources"]]
    res = translate(oracle, srcs, beam_size=c["beam_size"], num_hypotheses=c["num_hypotheses"], max_length=c["max_length"],
                    min_length=c["min_length"], length_penalty=c["length_penalty"], bos=START, eos=END, **vocab.options(c))
    return [[[vocab.tgt_list[i] for i in h[0]] for h in r] for r in res], [[h[1] for h in r] for r in res]


@pytest.mark.parametrize("name", ["aren", "postnorm"])
def test_oracle_reproduces_the_float32_fixture(fixture, name):
    entry = fixture[name]
    mdir = os.path.join(GOLDEN, entry["model"])
    oracle, vocab = O.Seq2SeqOracle.from_dir(mdir, compute_type="float32"), Vocab(mdir)
    cases = entry["models"]["float32"]["cases"]
    assert {c["beam_size"] for c in cases} == {1, 2, 4, 10}
    total = 0
    for c in cases:
        hyps, scores = run_oracle(oracle, vocab, c)
        assert hyps == c["hypotheses"], c
        for s, w in zip(scores, c["scores"]):
            np.testing.assert_allclose(s, w, atol=1e-4)
            total += len(s)
    assert total > 200


def _row_hook(history, end_ids, min_length, step, logits, **kw):
    state = {"seq": [history], "raw": logits.copy()}
    masked = logits.copy()
    if step < min_length:
        masked[:, end_ids] = np.finfo(f32).min
    processors_hook(state, end_ids, min_length, **kw)(step, masked)
    return masked[0]


def test_penalty_runs_before_the_min_length_mask():
    """DisableTokens writes after the processors: an end id in the history stays at the lowest value under a penalty < 1
    below min_decoding_length; a penalty alone rewrites each token of the history once, from its unpenalised value."""
    lowest = np.finfo(f32).min
    x = np.array([[2.0, -1.0, 4.0, -3.0, 0.5]], f32)
    row = _row_hook([2, 1, 2, 3], [2], 5, 4, x, repetition_penalty=0.5)
    assert row[2] == lowest
    np.testing.assert_array_equal(row[[0, 1, 3, 4]], f32([2.0, -0.5, -1.5, 0.5]))
    row = _row_hook([2, 1, 2, 3], [2], 0, 4, x, repetition_penalty=0.5)    # past min_length: penalised once
    np.testing.assert_array_equal(row, f32([2.0, -0.5, 8.0, -1.5, 0.5]))


def test_ngram_and_sequences_on_one_row():
    lowest = np.finfo(f32).min
    x = np.zeros((1, 8), f32)
    row = _row_hook([3, 4, 5, 3, 4], [2], 0, 5, x, no_repeat_ngram_size=3)           # "3 4" was followed by 5
    assert row[5] == lowest and (row[[0, 1, 2, 3, 4, 6, 7]] == 0).all()
    row = _row_hook([3, 4, 5, 3, 4], [2], 0, 5, x, suppress_sequences=[[6], [3, 4, 7], [5, 3, 1], []])
    assert row[6] == lowest and row[7] == lowest and row[1] == 0
    row = _row_hook([], [2], 0, 0, x, no_repeat_ngram_size=1, repetition_penalty=2.0, suppress_sequences=[[3, 4]])
    assert (row == 0).all()                                                          # step 0: the history is empty


REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libct2ref.so")


def _reference_driver():
    """tools/make_golden.py's runner of the reference's translate_batch, where the reference CPU library and the sources it
    was built from (for the driver's headers) are present; None elsewhere."""
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_golden
    if not (os.path.exists(REF_LIB) and os.path.isdir(os.path.join(make_golden.REF, "include"))):
        return None
    return make_golden.ref_translate_processors


def test_oracle_matches_the_reference_live():
    """New requests on the post-norm model, run through the reference CPU build and the oracle."""
    ref_translate_processors = _reference_driver()
    if ref_translate_processors is None:
        pytest.skip("needs the reference CPU library (make -f oracle/Makefile.ref) and its sources")
    mdir = os.path.join(GOLDEN, "tiny_seq2seq_postnorm")
    oracle, vocab = O.Seq2SeqOracle.from_dir(mdir, compute_type="float32"), Vocab(mdir)
    rng = np.random.default_rng(77)
    src_tokens = list(vocab.src)[3:]
    tgt_tokens = vocab.tgt_list[3:]
    requests = []
    for beam, nh in ((1, 1), (3, 2), (5, 3), (12, 2)):
        srcs = [[src_tokens[int(i)] for i in rng.integers(0, len(src_tokens), size=int(rng.integers(2, 12)))] for _ in range(3)]
        seqs = [[tgt_tokens[int(i)] for i in rng.integers(0, len(tgt_tokens), size=k)] for k in (1, 2, 2, 3)]
        requests.append(dict(sources=srcs, beam_size=beam, num_hypotheses=nh, length_penalty=1.0, max_length=18, min_length=3,
                             repetition_penalty=float(rng.choice([0.8, 1.25])), no_repeat_ngram_size=int(rng.integers(1, 4)),
                             disable_unk=True, suppress_sequences=seqs))
    for r, ref in zip(requests, ref_translate_processors(mdir, "float32", requests)):
        hyps, scores = run_oracle(oracle, vocab, r)
        assert hyps == [x[0] for x in ref], r
        for s, (_, w) in zip(scores, ref):
            np.testing.assert_allclose(s, w, atol=1e-4)
