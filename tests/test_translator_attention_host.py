"""Host logic of Translator.translate_batch's return_attention, replace_unknowns and coverage_penalty without a device: the C-ABI
is replaced by a recording fake that answers with known attention rows, so what is checked is the Python side -- which entry
point is called with what, the row and column handling of run_translation (sequence_to_sequence.cc:381-412), the unknown-token
replacement (:288-302), empty sources and the argument checks before any library call.
tests/test_gpu_translator_attention.py covers the real library."""
import ctypes

import numpy as np
import pytest

import ctranslate2_b200.translator as TR
from test_translator_processors_host import FakeLib, SRC, TGT, _arr, _make


class AttentionFake(FakeLib):
    """ct2b200_translate_batch_attention: every hypothesis is `tokens`; attention row t of entry b, column s = t * 10 + s + 1
    over the entry's length (zeros past it), as many rows as tokens."""

    def __init__(self, tokens=(3, 4, 2)):
        super().__init__()
        self.tokens = list(tokens)

    def ct2b200_translate_batch_attention(self, *args):
        call = self._common(args[:15])
        penalty, n, dis, n_dis, seq_ids, seq_off, n_seq, cov = args[15:23]
        out_ids, out_lens, out_scores, out_att = args[23:27]
        call.update(penalty=penalty.value, ngram=n, disable=_arr(dis, ctypes.c_int32, n_dis).tolist(), coverage=cov.value,
                    attention=out_att is not None)
        self.calls.append(("translate_batch_attention", call))
        B, nh, L, S = len(call["lens"]), call["nh"], call["max_len"], max(call["lens"])
        ids = _arr(out_ids, ctypes.c_int32, B * nh * L).reshape(B, nh, L)
        toks = self.tokens if call["return_end"] else [x for x in self.tokens if x != 2]
        ids[:] = -1
        ids[:, :, :len(toks)] = toks
        _arr(out_lens, ctypes.c_int32, B * nh)[:] = len(toks)
        _arr(out_scores, ctypes.c_float, B * nh)[:] = -0.25
        if out_att is not None:
            att = np.ctypeslib.as_array((ctypes.c_float * (B * nh * L * S)).from_address(out_att.value)).reshape(B, nh, L, S)
            for b, n_src in enumerate(call["lens"]):
                for t in range(len(toks)):
                    att[b, :, t, :n_src] = [t * 10 + s + 1 for s in range(n_src)]
        return 0


@pytest.fixture
def tr(monkeypatch):
    t, _ = _make(monkeypatch)
    fake = AttentionFake()
    monkeypatch.setattr(TR, "lib", lambda: fake)
    yield t, fake
    t._h = None


def test_defaults_keep_the_existing_entries(tr):
    t, fake = tr
    t.translate_batch([["s1", "s2"]], return_attention=False, replace_unknowns=False, coverage_penalty=0)
    t.translate_batch([["s1"]], coverage_penalty=0.0, repetition_penalty=1.3)
    assert [c[0] for c in fake.calls] == ["translate_batch", "translate_batch_processors"]
    out = t.translate_ids([[4]])
    assert len(out) == 3 and fake.calls[-1][0] == "translate_batch"


@pytest.mark.parametrize("kw, attention, coverage", [
    (dict(return_attention=True), True, 0.0), (dict(replace_unknowns=True), True, 0.0),
    (dict(coverage_penalty=0.5), False, 0.5), (dict(coverage_penalty=1, return_attention=True), True, 1.0)])
def test_each_option_takes_the_attention_entry(tr, kw, attention, coverage):
    t, fake = tr
    t.translate_batch([["s1", "s2"]], beam_size=3, repetition_penalty=1.5, disable_unk=True, **kw)
    name, c = fake.calls[-1]
    assert name == "translate_batch_attention"
    assert c["attention"] is attention and c["coverage"] == coverage and c["beam"] == 3
    assert c["penalty"] == 1.5 and c["disable"] == [0]


def test_rows_follow_the_tokens_and_columns_the_source(tr):
    t, fake = tr
    res = t.translate_batch([["s1", "s2", "s3"], ["s4"]], return_attention=True)
    assert res[0].hypotheses == [["t0", "t1"]]                   # </s> stripped, and its row with it
    assert res[0].attention == [[[1.0, 2.0, 3.0], [11.0, 12.0, 13.0]]]
    assert res[1].attention == [[[1.0], [11.0]]]
    res = t.translate_batch([["s1", "s2"]], return_attention=True, return_end_token=True)
    assert res[0].hypotheses == [["t0", "t1", "</s>"]]
    assert res[0].attention == [[[1.0, 2.0], [11.0, 12.0], [21.0, 22.0]]]
    assert fake.calls[-1][1]["return_end"] == 1


@pytest.mark.parametrize("bos, eos, want", [
    (True, False, [[2.0, 3.0], [12.0, 13.0]]), (False, True, [[1.0, 2.0], [11.0, 12.0]]),
    (True, True, [[2.0, 3.0], [12.0, 13.0]])])
def test_the_added_special_tokens_lose_their_columns(tr, bos, eos, want):
    t, fake = tr
    t._config.update(add_source_bos=bos, add_source_eos=eos)
    res = t.translate_batch([["s1", "s2"]], return_attention=True)
    assert fake.calls[-1][1]["lens"] == [2 + bos + eos]
    assert res[0].attention == [want]


def test_id_sources_keep_their_columns(tr):
    t, fake = tr
    t._config.update(add_source_bos=True)
    res = t.translate_batch([[5, 6, 7]], return_attention=True)
    assert res[0].attention == [[[1.0, 2.0, 3.0], [11.0, 12.0, 13.0]]]


def test_replace_unknowns_copies_the_first_most_attended_token(monkeypatch):
    t, _ = _make(monkeypatch)
    fake = AttentionFake(tokens=(0, 5, 0, 2))                       # <unk> t2 <unk> </s>
    monkeypatch.setattr(TR, "lib", lambda: fake)
    try:
        res = t.translate_batch([["s1", "s2", "s3"]], replace_unknowns=True)
        # rows rise with the column: the last source token is the first maximum of every row
        assert res[0].hypotheses == [["s3", "t2", "s3"]] and res[0].hypotheses_ids == [[0, 5, 0]]
        assert res[0].attention == []
        res = t.translate_batch([["s1", "s2", "s3"]], replace_unknowns=True, return_attention=True)
        assert res[0].hypotheses == [["s3", "t2", "s3"]] and len(res[0].attention[0]) == 3
        res = t.translate_batch([["s1", "s2", "s3"]], return_attention=True)
        assert res[0].hypotheses == [["<unk>", "t2", "<unk>"]]
    finally:
        t._h = None


def test_first_maximum_wins():
    hyp = ["<unk>", "x", "<unk>"]
    TR._replace_unknowns(hyp, ["a", "b", "c"], np.array([[0.2, 0.4, 0.4], [1, 0, 0], [0.5, 0.1, 0.5]], np.float32), "<unk>")
    assert hyp == ["b", "x", "a"]


def test_empty_sources(tr):
    t, fake = tr
    res = t.translate_batch([[], ["s1"]], num_hypotheses=1, return_attention=True, return_scores=True)
    assert res[0].hypotheses == [[]] and res[0].attention == [[]] and res[0].scores == [0.0]
    assert res[1].attention == [[[1.0], [11.0]]]
    assert fake.calls[-1][1]["lens"] == [1]
    res = t.translate_batch([[]], return_attention=False)
    assert res[0].attention == []


@pytest.mark.parametrize("kw", [
    dict(coverage_penalty=True), dict(coverage_penalty="0.2"), dict(coverage_penalty=float("nan")),
    dict(coverage_penalty=float("inf")), dict(coverage_penalty=None),
    dict(return_attention=1), dict(return_attention="yes"), dict(return_attention=None),
    dict(replace_unknowns=0), dict(replace_unknowns="no"),
])
def test_bad_options_raise_before_any_call(tr, kw):
    t, fake = tr
    with pytest.raises(ValueError):
        t.translate_batch([["s1"]], **kw)
    with pytest.raises(ValueError):
        t.translate_batch([], **kw)
    assert fake.calls == []


def test_replace_unknowns_refuses_id_sources(tr):
    t, fake = tr
    with pytest.raises(ValueError):
        t.translate_batch([[4, 5]], replace_unknowns=True)
    with pytest.raises(ValueError):
        t.translate_batch([["s1"], [4, 5]], replace_unknowns=True)
    for kw in (dict(coverage_penalty=float("nan")), dict(return_attention=1)):
        with pytest.raises(ValueError):
            t.translate_ids([[4]], **kw)
    assert fake.calls == []
    t.translate_batch([[4, 5]], return_attention=True)
    assert fake.calls[-1][0] == "translate_batch_attention"


def test_translate_ids_returns_the_raw_rows(tr):
    t, fake = tr
    ids, lens, scores, att = t.translate_ids([[4, 5], [6]], return_attention=True, max_decoding_length=5)
    assert att.shape == (2, 1, 5, 2) and att.dtype == np.float32
    assert att[1, 0, 0].tolist() == [1.0, 0.0] and (att[:, :, 2:] == 0).all()
    out = t.translate_ids([[4]], coverage_penalty=0.3)
    assert len(out) == 3 and fake.calls[-1][1]["attention"] is False
