"""Host logic of Translator.translate_batch's logits processors without a device: the C-ABI is replaced by a recording fake,
so what is checked is the Python side -- token strings to target ids (Vocabulary::to_ids with allow_unk = false,
src/vocabulary.cc:67-75), the argument checks before any library call, and which entry point is called with what.  The
Generator's and Whisper's refusals of the same options are checked to hold.  tests/test_gpu_translator_processors.py covers
the real library."""
import ctypes

import numpy as np
import pytest

import ctranslate2_b200.translator as TR


def _arr(ptr, ctype, n):
    return np.ctypeslib.as_array((ctype * n).from_address(ptr.value)) if n else np.zeros(0, np.int32)


class FakeLib:
    def __init__(self):
        self.calls = []

    def _common(self, args):
        h, src, lens, B, S, beam, patience, lp, max_len, min_len, nh, start, end, n_end, ret_end = args
        B, S = B.value, S.value
        return dict(src=_arr(src, ctypes.c_int32, B * S).reshape(B, S).tolist(), lens=_arr(lens, ctypes.c_int32, B).tolist(),
                    beam=beam, patience=patience.value, length_penalty=lp.value, max_len=max_len.value,
                    min_len=min_len.value, nh=nh, start=start.value, end=_arr(end, ctypes.c_int32, n_end).tolist(),
                    return_end=ret_end)

    def _answer(self, call, out_ids, out_lens, out_scores):
        B, nh, L = len(call["lens"]), call["nh"], call["max_len"]
        _arr(out_ids, ctypes.c_int32, B * nh * L)[:] = 3
        _arr(out_lens, ctypes.c_int32, B * nh)[:] = 1
        _arr(out_scores, ctypes.c_float, B * nh)[:] = -0.5
        return 0

    def ct2b200_translate_batch(self, *args):
        call = self._common(args[:15])
        self.calls.append(("translate_batch", call))
        return self._answer(call, *args[15:])

    def ct2b200_translate_batch_processors(self, *args):
        call = self._common(args[:15])
        penalty, n, dis, n_dis, seq_ids, seq_off, n_seq = args[15:22]
        off = _arr(seq_off, ctypes.c_int32, n_seq + 1 if n_seq else 0).tolist()
        call.update(penalty=penalty.value, ngram=n, disable=_arr(dis, ctypes.c_int32, n_dis).tolist(), offsets=off,
                    seq_ids=_arr(seq_ids, ctypes.c_int32, off[-1] if off else 0).tolist())
        self.calls.append(("translate_batch_processors", call))
        return self._answer(call, *args[22:])

    def ct2b200_translator_close(self, h):
        pass

    def ct2b200_last_error(self):
        return b""


SRC = ["<unk>", "<s>", "</s>"] + ["s%d" % i for i in range(20)]
TGT = ["<unk>", "<s>", "</s>"] + ["t%d" % i for i in range(40)]          # t<i> has id i + 3


def _make(monkeypatch, target=TGT):
    fake = FakeLib()
    monkeypatch.setattr(TR, "lib", lambda: fake)
    t = object.__new__(TR.Translator)
    t._h = 1
    t._config = {"decoder_start_token": "<s>"}
    t._source, t._target = SRC, target
    t._src_to_id = {w: i for i, w in enumerate(SRC)}
    t._tgt_to_id = {w: i for i, w in enumerate(target)}
    t._decoder_positions = t._encoder_positions = 512
    t._src_vocab_size, t._tgt_vocab_size = len(SRC), len(target)
    return t, fake


@pytest.fixture
def tr(monkeypatch):
    t, fake = _make(monkeypatch)
    yield t, fake
    t._h = None


def test_neutral_values_call_the_existing_entry(tr):
    t, fake = tr
    t.translate_batch([["s1", "s2"]], beam_size=3)
    t.translate_batch([["s1", "s2"]], beam_size=3, repetition_penalty=1, no_repeat_ngram_size=0, disable_unk=False,
                      suppress_sequences=[])
    t.translate_batch([["s1", "s2"]], beam_size=3, repetition_penalty=1.0, suppress_sequences=None)
    assert [c[0] for c in fake.calls] == ["translate_batch"] * 3
    assert fake.calls[0][1] == fake.calls[1][1] == fake.calls[2][1]
    assert fake.calls[0][1]["src"] == [[4, 5]] and fake.calls[0][1]["beam"] == 3


def test_strings_map_to_target_ids(tr):
    t, fake = tr
    res = t.translate_batch([["s1"], ["s2", "s3"]], repetition_penalty=1.5, no_repeat_ngram_size=2, disable_unk=True,
                            suppress_sequences=[["t0"], ["t1", "t2"], [], ["<unk>", "t5", "t6"]])
    name, c = fake.calls[-1]
    assert name == "translate_batch_processors"
    assert c["penalty"] == 1.5 and c["ngram"] == 2 and c["disable"] == [0]
    assert c["offsets"] == [0, 1, 3, 3, 6] and c["seq_ids"] == [3, 4, 5, 0, 8, 9]
    assert c["src"] == [[4, 0], [5, 6]] and c["lens"] == [1, 2]
    assert res[0].hypotheses == [["t0"]]


@pytest.mark.parametrize("kw", [dict(repetition_penalty=0.7), dict(no_repeat_ngram_size=1), dict(disable_unk=True),
                                dict(suppress_sequences=[["t3"]])])
def test_each_option_alone_takes_the_processors_entry(tr, kw):
    t, fake = tr
    t.translate_batch([["s1"]], **kw)
    assert fake.calls[-1][0] == "translate_batch_processors"


def test_unknown_token_past_the_output_layer_is_left_out(monkeypatch):
    """A vocabulary without <unk>: the reference appends it after the last output id, which is never produced."""
    t, fake = _make(monkeypatch, target=TGT[1:])
    try:
        t.translate_batch([["s1"]], disable_unk=True, suppress_sequences=[["<unk>"], ["t0", "<unk>"]])
        assert fake.calls[-1][0] == "translate_batch"
        t.translate_batch([["s1"]], disable_unk=True, suppress_sequences=[["<unk>"], ["t0", "t1"]])
        assert fake.calls[-1][0] == "translate_batch_processors" and fake.calls[-1][1]["disable"] == []
        assert fake.calls[-1][1]["seq_ids"] == [2, 3]
    finally:
        t._h = None


@pytest.mark.parametrize("kw", [
    dict(suppress_sequences=[["t1", "oovtoken"]]),                 # SuppressSequenceOOV
    dict(suppress_sequences=["t1"]),                               # a list of strings, not of token lists
    dict(suppress_sequences="t1"),
    dict(suppress_sequences=[[3, 4]]),                             # ids, not token strings
    dict(repetition_penalty=0), dict(repetition_penalty=-1.2), dict(repetition_penalty=float("nan")),
    dict(repetition_penalty=float("inf")), dict(repetition_penalty=True), dict(repetition_penalty="1.2"),
    dict(no_repeat_ngram_size=-1), dict(no_repeat_ngram_size=2.0), dict(no_repeat_ngram_size=True),
    dict(disable_unk=1), dict(disable_unk="yes"),
    dict(suppress_sequences=[["t1"]] * (TR.MAX_SUPPRESS_SEQUENCES + 1)),
    dict(suppress_sequences=[["t1"] * 1000] * 66),                  # more than 65536 tokens in all
])
def test_bad_options_raise_before_any_call(tr, kw):
    t, fake = tr
    with pytest.raises(ValueError):
        t.translate_batch([["s1"]], **kw)
    with pytest.raises(ValueError):
        t.translate_batch([], **kw)
    assert fake.calls == []


def test_translate_ids_checks_ids(tr):
    t, fake = tr
    for kw in (dict(disable_ids=[len(TGT)]), dict(disable_ids=[-1]), dict(suppress_sequences=[[3, 99]]),
               dict(suppress_sequences=[["t1"]]), dict(repetition_penalty=0.0)):
        with pytest.raises(ValueError):
            t.translate_ids([[4]], **kw)
    assert fake.calls == []
    t.translate_ids([[4]], disable_ids=[5], suppress_sequences=[[3, 4]])
    assert fake.calls[-1][1]["disable"] == [5] and fake.calls[-1][1]["offsets"] == [0, 2]
    t.translate_ids([[4]])
    assert fake.calls[-1][0] == "translate_batch"


def test_the_caps_are_accepted_at_the_limit(tr):
    t, fake = tr
    t.translate_batch([["s1"]], suppress_sequences=[["t1"]] * TR.MAX_SUPPRESS_SEQUENCES)
    assert len(fake.calls[-1][1]["offsets"]) == TR.MAX_SUPPRESS_SEQUENCES + 1


@pytest.mark.parametrize("kw", [dict(repetition_penalty=1.2), dict(no_repeat_ngram_size=2), dict(disable_unk=True),
                                dict(suppress_sequences=[["a"]])])
def test_generator_and_whisper_still_refuse_the_processors(monkeypatch, kw):
    """Only the Translator takes the processors: the Generator's option check and Whisper.generate refuse them."""
    from ctranslate2_b200.generator import _check_options
    import ctranslate2_b200.whisper as W
    import test_whisper_sampling_host as WH
    with pytest.raises(ValueError):
        _check_options(kw, 8, 0)
    fake = WH.FakeLib()
    monkeypatch.setattr(W, "lib", lambda: fake)
    w = WH.make()
    try:
        with pytest.raises((ValueError, TypeError)):      # WhisperOptions has no disable_unk / suppress_sequences at all
            w.generate(WH.feats(), WH.PROMPT, beam_size=2, **kw)
        w.generate(WH.feats(), WH.PROMPT, beam_size=2)
        assert len(fake.calls) == 1
    finally:
        w._h = None                                       # the fake handle must not reach the real library's close
