"""return_attention, replace_unknowns and coverage_penalty of Translator::translate_batch restated on the oracle
(tests/seq2seq_attention.py) against the unmodified reference: the committed outputs of
tests/golden/seq2seq_attention_ref.json (tools/make_golden.py --seq2seq-attention-only) and, where oracle/_ref has been built,
the reference run live on new cases.

float32 compute has no activation quantization: every hypothesis must equal the reference's token for token, scores agree to
2e-4 and attention to 1e-5."""
import json
import os

import numpy as np
import pytest

from ctranslate2_b200.translator import _load_vocabulary
from seq2seq_attention import AttentionOracle, replace_unknowns, source_columns, translate

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
START, END = 1, 2


@pytest.fixture(scope="module")
def fixture():
    with open(os.path.join(GOLDEN, "seq2seq_attention_ref.json")) as f:
        return json.load(f)


class Model:
    def __init__(self, mdir):
        self.oracle = AttentionOracle.from_dir(mdir, compute_type="float32")
        self.src = {t: i for i, t in enumerate(_load_vocabulary(mdir, "source_vocabulary"))}
        self.tgt = _load_vocabulary(mdir, "target_vocabulary")


def run_oracle(m: Model, c):
    """The case through the oracle, post-processed as run_translation does: (hypotheses, scores, attention) per source."""
    srcs = [[m.src[t] for t in r] for r in c["sources"]]
    res = translate(m.oracle, srcs, beam_size=c["beam_size"], num_hypotheses=c["num_hypotheses"], max_length=c["max_length"],
                    min_length=c["min_length"], length_penalty=c["length_penalty"], coverage_penalty=c["coverage_penalty"],
                    return_end_token=c["return_end_token"], bos=START, eos=END)
    hyps, scores, attention = [], [], []
    for r, tokens in zip(res, c["sources"]):
        h = [[m.tgt[i] for i in x[0]] for x in r]
        att = [source_columns(x[2], len(tokens), len(tokens), False, False) for x in r]
        if c["replace_unknowns"]:
            h = [replace_unknowns(x, tokens, a) for x, a in zip(h, att)]
        hyps.append(h)
        scores.append([x[1] for x in r])
        attention.append(att if c["return_attention"] else [])
    return hyps, scores, attention


def check(c, hyps, scores, attention, ref_hyps, ref_scores, ref_attention):
    assert hyps == ref_hyps, c
    for s, w in zip(scores, ref_scores):
        np.testing.assert_allclose(s, w, atol=2e-4)
    assert len(attention) == len(ref_attention)
    for a, w in zip(attention, ref_attention):
        assert len(a) == len(w)
        for x, y in zip(a, w):
            assert len(x) == len(y)
            if x:
                np.testing.assert_allclose(np.array(x), np.array(y), atol=1e-5)


@pytest.mark.parametrize("name", ["aren", "postnorm", "align"])
def test_oracle_reproduces_the_fixture(fixture, name):
    entry = fixture[name]
    m = Model(os.path.join(GOLDEN, entry["model"]))
    cases = entry["cases"]
    assert {c["beam_size"] for c in cases} == {1, 2, 4, 10}
    assert {c["coverage_penalty"] for c in cases} == {0.0, 0.2, 1.0}
    for c in cases:
        check(c, *run_oracle(m, c), c["hypotheses"], c["scores"], c["attention"])
    if name != "aren":
        # the <unk> case: replace_unknowns changes the hypothesis, and only at the <unk>
        before = next(c for c in cases if not c["replace_unknowns"] and "<unk>" in c["hypotheses"][0][0])
        after = next(c for c in cases if c["replace_unknowns"] and c["sources"] == before["sources"] and
                     c["beam_size"] == before["beam_size"])
        b, a = before["hypotheses"][0][0], after["hypotheses"][0][0]
        assert len(a) == len(b) and "<unk>" not in a
        assert all(x == y for x, y in zip(a, b) if y != "<unk>")


def test_the_align_model_averages_every_head_of_the_first_layer():
    m = AttentionOracle.from_dir(os.path.join(GOLDEN, "tiny_seq2seq_align"), compute_type="float32")
    assert m.align_layer == 0 and m.align_heads == m.num_heads == 4
    m = AttentionOracle.from_dir(os.path.join(GOLDEN, "tiny_seq2seq_postnorm"), compute_type="float32")
    assert m.align_layer == 1 and m.align_heads == 1


def test_source_columns():
    rows = [[0.1, 0.2, 0.3, 0.4, 0.0]]
    assert source_columns(rows, 4, 2, True, True) == [[np.float32(0.2), np.float32(0.3)]]
    assert source_columns(rows, 3, 4, False, True)[0][2:] == [0.0, 0.0]


REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libct2ref.so")


def _reference_driver():
    """tools/make_golden.py's runner of the reference's translate_batch, where the reference CPU library and the sources it
    was built from (for the driver's headers) are present; None elsewhere."""
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_golden
    if not (os.path.exists(REF_LIB) and os.path.isdir(os.path.join(make_golden.REF, "include"))):
        return None
    return make_golden.ref_translate_attention


def test_oracle_matches_the_reference_live():
    """New requests on the all-heads model, run through the reference CPU build and the oracle."""
    ref_translate_attention = _reference_driver()
    if ref_translate_attention is None:
        pytest.skip("needs the reference CPU library (make -f oracle/Makefile.ref) and its sources")
    mdir = os.path.join(GOLDEN, "tiny_seq2seq_align")
    m = Model(mdir)
    rng = np.random.default_rng(78)
    src_tokens = list(m.src)[3:]
    requests = []
    for beam, nh, cov, lp in ((1, 1, 0.5, 1.0), (3, 2, 0.3, 1.0), (5, 3, 0.7, 0.0), (12, 2, 0.1, 0.6)):
        # one source per beam search: the reference's first attention row of a batched beam search is another entry's
        # (tools/make_golden.py, make_seq2seq_attention_fixture)
        srcs = [[src_tokens[int(i)] for i in rng.integers(0, len(src_tokens), size=int(rng.integers(2, 12)))]
                for _ in range(3 if beam == 1 else 1)]
        requests.append(dict(sources=srcs, beam_size=beam, num_hypotheses=nh, length_penalty=lp, max_length=18, min_length=2,
                             coverage_penalty=cov, return_end_token=bool(beam % 2), return_attention=True,
                             replace_unknowns=False))
    for r, ref in zip(requests, ref_translate_attention(mdir, "float32", requests)):
        check(r, *run_oracle(m, r), [x[0] for x in ref], [x[1] for x in ref], [x[2] for x in ref])
