"""Host logic of ctranslate2_b200.Translator.score_batch without a device: the C-ABI is replaced by a recording fake, so what is
checked is the Python side -- source / target id construction (Vocabulary::to_ids with the model's special tokens and the
decoder start token, EncoderDecoderReplica::make_target_ids, src/models/sequence_to_sequence.cc:168-186), truncation that keeps
</s> (src/vocabulary.cc:108-147), offset, both skip rules (skip_scoring, :263-286), re-batching longest source first
(src/batch_reader.cc:175-225) answered in request order, and every argument check before any library call.  No compute is
claimed here; tests/test_gpu_translator_score.py covers the real library."""
import ctypes

import numpy as np
import pytest

import ctranslate2_b200.translator as TR
from ctranslate2_b200.generator import ScoringResult


def _arr(ptr, ctype, n):
    return np.ctypeslib.as_array((ctype * n).from_address(ptr.value))


def fake_score(src_row, tgt_id):
    """The fake's 'log-probability': identifies the target token and the source it was paired with."""
    return -tgt_id / 1000.0 - src_row[0] / 1e6


class FakeLib:
    def __init__(self):
        self.calls = []

    def ct2b200_translator_score_batch(self, h, src, src_lens, B, S, tgt, tgt_lens, T, offset, out):
        B, S, T, offset = B.value, S.value, T.value, offset.value
        src_a = _arr(src, ctypes.c_int32, B * S).reshape(B, S).copy()
        sl = _arr(src_lens, ctypes.c_int32, B).copy()
        tgt_a = _arr(tgt, ctypes.c_int32, B * T).reshape(B, T).copy()
        tl = _arr(tgt_lens, ctypes.c_int32, B).copy()
        self.calls.append(dict(src=src_a, src_lens=sl, tgt=tgt_a, tgt_lens=tl, offset=offset))
        o = _arr(out, ctypes.c_float, B * (T - 1)).reshape(B, T - 1)
        o[:] = 0
        for b in range(B):
            for t in range(offset, tl[b] - 1):
                o[b, t - offset] = fake_score(src_a[b], tgt_a[b, t + 1])
        return 0

    def ct2b200_translator_close(self, h):
        pass

    def ct2b200_last_error(self):
        return b""


SRC = ["<unk>", "<s>", "</s>"] + ["s%d" % i for i in range(60)]          # source vocabulary: s<i> has id i + 3
TGT = ["<unk>", "<s>", "</s>"] + ["t%d" % i for i in range(40)]          # target vocabulary: t<i> has id i + 3
BOS, EOS, UNK = 1, 2, 0


def _make(monkeypatch, config=None, positions=512, encoder_positions=512):
    fake = FakeLib()
    monkeypatch.setattr(TR, "lib", lambda: fake)
    t = object.__new__(TR.Translator)
    t._h = 1
    t._config = {"decoder_start_token": "<s>"} if config is None else config
    t._source, t._target = SRC, TGT
    t._src_to_id = {w: i for i, w in enumerate(SRC)}
    t._tgt_to_id = {w: i for i, w in enumerate(TGT)}
    t._decoder_positions = positions
    t._encoder_positions = encoder_positions
    t._src_vocab_size, t._tgt_vocab_size = len(SRC), len(TGT)
    return t, fake


@pytest.fixture
def tr(monkeypatch):
    t, fake = _make(monkeypatch)
    yield t, fake
    t._h = None


def s(*ids):
    return ["s%d" % (i - 3) for i in ids]


def t_(*ids):
    return ["t%d" % (i - 3) for i in ids]


def _sent(fake):
    """(source ids, full target ids) of every pair sent, in call order."""
    out = []
    for c in fake.calls:
        for b in range(len(c["src_lens"])):
            out.append((c["src"][b, :c["src_lens"][b]].tolist(), c["tgt"][b, :c["tgt_lens"][b]].tolist()))
    return out


def test_target_gets_start_and_end_tokens_and_results_end_with_eos(tr):
    t, fake = tr
    res = t.score_batch([s(5, 6, 7)], [t_(10, 11)])
    assert _sent(fake) == [([5, 6, 7], [BOS, 10, 11, EOS])]
    assert res[0].tokens == ["t7", "t8", "</s>"]
    np.testing.assert_allclose(res[0].log_probs, [fake_score([5], x) for x in (10, 11, EOS)])
    fake.calls.clear()
    # id lists: sources are taken as given, targets still get <s> and </s>
    res = t.score_batch([[5, 6, 7]], [[10, 11]])
    assert _sent(fake) == [([5, 6, 7], [BOS, 10, 11, EOS])] and res[0].tokens == ["t7", "t8", "</s>"]


def test_source_special_tokens_and_unknown_tokens(monkeypatch):
    t, fake = _make(monkeypatch, {"decoder_start_token": "<s>", "add_source_bos": True, "add_source_eos": True})
    res = t.score_batch([s(5) + ["nope"]], [t_(9) + ["missing"]])
    assert _sent(fake) == [([BOS, 5, UNK, EOS], [BOS, 9, UNK, EOS])]
    assert res[0].tokens == ["t6", "<unk>", "</s>"]


def test_no_decoder_start_token(monkeypatch):
    t, fake = _make(monkeypatch, {"decoder_start_token": None})
    res = t.score_batch([s(5, 6), s(7), s(8)], [t_(10, 11), [], t_(12)])
    # skip_scoring: an empty target scores nothing without a start token; the others have no <s>
    assert res[1] == ScoringResult([], [])
    assert sorted(_sent(fake)) == sorted([([5, 6], [10, 11, EOS]), ([8], [12, EOS])])
    assert res[0].tokens == ["t8", "</s>"] and res[2].tokens == ["</s>"]
    np.testing.assert_allclose(res[2].log_probs, [fake_score([8], EOS)])


def test_empty_target_with_a_start_token_scores_eos(tr):
    t, fake = tr
    res = t.score_batch([s(5)], [[]])
    assert _sent(fake) == [([5], [BOS, EOS])] and res[0].tokens == ["</s>"]


def test_empty_source_scores_zero_without_offset(tr):
    t, fake = tr
    res = t.score_batch([[], s(5)], [t_(10, 11, 12), t_(13)], offset=2)
    assert res[0] == ScoringResult(["t7", "t8", "t9", "</s>"], [0.0] * 4)       # the offset is not applied here
    assert _sent(fake) == [([5], [BOS, 13, EOS])]
    assert res[1] == ScoringResult([], [])                                     # offset 2 >= the 2 outputs of pair 1
    fake.calls.clear()
    assert t.score_batch([[]], [t_(10)])[0] == ScoringResult(["t7", "</s>"], [0.0, 0.0]) and fake.calls == []


@pytest.mark.parametrize("offset", [0, 1, 3, 7])
def test_offset(tr, offset):
    t, fake = tr
    tgts = [t_(10, 11, 12, 13), t_(14)]
    res = t.score_batch([s(5, 6), s(7)], tgts, offset=offset)
    assert all(c["offset"] == offset for c in fake.calls)
    for src, tg, r in zip(([5], [7]), tgts, res):
        full = [BOS] + [TGT.index(x) for x in tg] + [EOS]
        assert r.tokens == [TGT[i] for i in full[1 + offset:]]
        np.testing.assert_allclose(r.log_probs, [fake_score(src, x) for x in full[1 + offset:]])


def test_truncation(tr):
    t, fake = tr
    # source: cut to 3; target: <s> + 5 tokens + </s> cut to 3 + 1 = 4 keeping </s>
    res = t.score_batch([s(5, 6, 7, 8, 9)], [t_(10, 11, 12, 13, 14)], max_input_length=3)
    assert _sent(fake) == [([5, 6, 7], [BOS, 10, 11, EOS])]
    assert res[0].tokens == ["t7", "t8", "</s>"]
    fake.calls.clear()
    t.score_batch([s(5, 6, 7, 8, 9)], [t_(10, 11, 12, 13, 14)], max_input_length=0)       # 0: no limit
    assert _sent(fake) == [([5, 6, 7, 8, 9], [BOS, 10, 11, 12, 13, 14, EOS])]
    fake.calls.clear()
    t.score_batch([[5, 6, 7, EOS]], [t_(10)], max_input_length=2)                        # the source keeps its </s> too
    assert _sent(fake) == [([5, EOS], [BOS, 10, EOS])]
    fake.calls.clear()
    t.score_batch([s(5)], [t_(10, 11)], max_input_length=1)                              # target <s> </s>
    assert _sent(fake) == [([5], [BOS, EOS])]


def test_rebatching_longest_source_first_in_request_order(tr):
    t, fake = tr
    rng = np.random.default_rng(0)
    srcs = [[int(3 + i)] + rng.integers(3, 60, size=int(n)).tolist() for i, n in enumerate(rng.integers(0, 12, size=11))]
    tgts = [rng.integers(3, 40, size=int(n)).tolist() for n in rng.integers(0, 9, size=11)]
    res = t.score_batch(srcs, tgts)
    assert len(fake.calls) == 1
    assert fake.calls[0]["src_lens"].tolist() == sorted((len(x) for x in srcs), reverse=True)
    for src, tg, r in zip(srcs, tgts, res):
        full = [BOS] + tg + [EOS]
        assert r.tokens == [TGT[i] for i in full[1:]]
        np.testing.assert_allclose(r.log_probs, [fake_score(src, x) for x in full[1:]], rtol=1e-6)
    fake.calls.clear()
    res2 = t.score_batch(srcs, tgts, max_batch_size=3)
    assert [len(c["src_lens"]) for c in fake.calls] == [3, 3, 3, 2]
    served = [int(n) for c in fake.calls for n in c["src_lens"]]
    assert served == sorted((len(x) for x in srcs), reverse=True)
    assert res2 == res
    fake.calls.clear()
    res3 = t.score_batch(srcs, tgts, max_batch_size=20, batch_type="tokens")             # rows x longest source <= 20
    for c in fake.calls:
        assert len(c["src_lens"]) * int(c["src_lens"].max()) <= 20 or len(c["src_lens"]) == 1
    assert res3 == res
    for c in fake.calls:                                                                 # right-padded with 0
        for b in range(len(c["src_lens"])):
            assert (c["src"][b, c["src_lens"][b]:] == 0).all() and (c["tgt"][b, c["tgt_lens"][b]:] == 0).all()


def test_empty_batch(tr):
    t, fake = tr
    assert t.score_batch([], []) == [] and fake.calls == []


def test_refusals_happen_before_any_call(tr):
    t, fake = tr
    src, tgt = [s(5, 6)] * 3, [t_(10)] * 3
    for kw in (dict(asynchronous=True), dict(batch_type="sentences"), dict(max_batch_size=-1), dict(max_batch_size=1.5),
               dict(max_batch_size=True), dict(max_input_length=-1), dict(max_input_length=2.0), dict(offset=-1),
               dict(offset=0.5), dict(offset=None)):
        with pytest.raises(ValueError):
            t.score_batch(src, tgt, **kw)
    with pytest.raises(ValueError):
        t.score_batch(src, tgt[:2])                                    # count mismatch
    with pytest.raises(ValueError):
        t.score_batch(src + [[5, len(SRC)]], tgt + [[10]])             # source id outside the vocabulary
    with pytest.raises(ValueError):
        t.score_batch(src + [[-1]], tgt + [[10]])
    with pytest.raises(ValueError):
        t.score_batch(src + [[5]], tgt + [[len(TGT)]])                 # target id outside the vocabulary
    with pytest.raises(ValueError):
        t.score_batch(src + [[5]], tgt + [[10, -2]])
    with pytest.raises(ValueError):
        t.score_batch(src + [[5]], tgt + [[10, 1.5]])                  # not an id
    with pytest.raises(TypeError):
        t.score_batch(src, tgt, 4)                                     # options are keyword-only
    assert fake.calls == []


def test_position_table_overflow_is_refused_before_any_call(monkeypatch):
    t, fake = _make(monkeypatch, positions=6)
    ok = t_(*range(3, 8))                                              # <s> + 5 + </s>: 6 decoder positions
    t.score_batch([s(5)], [ok])
    assert len(fake.calls) == 1
    fake.calls.clear()
    with pytest.raises(ValueError):
        t.score_batch([s(5), s(6)], [ok, ok + ["t9"]])
    with pytest.raises(ValueError):
        t.score_batch([s(5)], [ok + ["t9"]], max_input_length=0)
    assert fake.calls == []
    t.score_batch([s(5)], [ok + ["t9", "t10"]], max_input_length=5)   # truncation brings it back within the table
    assert _sent(fake) == [([5], [BOS, 3, 4, 5, 6, EOS])]


def test_encoder_position_table_overflow_is_refused_before_any_call(monkeypatch):
    t, fake = _make(monkeypatch, encoder_positions=4)
    t.score_batch([s(5, 6, 7, 8)], [t_(10)])
    assert len(fake.calls) == 1
    fake.calls.clear()
    with pytest.raises(ValueError):
        t.score_batch([s(5), s(5, 6, 7, 8, 9)], [t_(10), t_(11)], max_input_length=0)
    assert fake.calls == []
    t.score_batch([s(5, 6, 7, 8, 9)], [t_(10)], max_input_length=4)           # truncated to the table
    assert _sent(fake) == [([5, 6, 7, 8], [BOS, 10, EOS])]


def test_an_empty_source_gets_the_special_tokens(monkeypatch):
    """Vocabulary::to_ids adds <s> / </s> to an empty token list too; only a source that stays empty scores zeros."""
    t, fake = _make(monkeypatch, {"decoder_start_token": "<s>", "add_source_eos": True})
    res = t.score_batch([[], s(5)], [t_(10), t_(11)])
    assert _sent(fake) == [([5, EOS], [BOS, 11, EOS]), ([EOS], [BOS, 10, EOS])]
    np.testing.assert_allclose(res[0].log_probs, [fake_score([EOS], x) for x in (10, EOS)])
