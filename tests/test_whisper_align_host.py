"""Host logic of ctranslate2_b200.Whisper.align / detect_language without a device: the C-ABI is replaced by a recording fake,
so what is checked is the Python side -- num_frames as one int or one per entry, alignment_heads and lang_ids read from
config.json, every argument check (ValueError / RuntimeError) raised before any library call, an empty batch, and results
in request order with the padded outputs trimmed.  tests/test_gpu_whisper_align.py covers the real library."""
import ctypes

import numpy as np
import pytest

import ctranslate2_b200.whisper as W


def _arr(ptr, ctype, n):
    return np.ctypeslib.as_array((ctype * n).from_address(ptr.value))


class FakeLib:
    def __init__(self):
        self.calls = []

    def ct2b200_whisper_align(self, h, f, B, T, start, start_len, text, lens, Nt, nf, width, heads, nh, nt_id, eot, path,
                              path_lens, probs, matrix):
        B, T, Nt, start_len = B.value, T.value, Nt.value, start_len.value
        S = (T + 1) // 2
        lens_a = _arr(lens, ctypes.c_int32, B).copy()
        text_a = _arr(text, ctypes.c_int32, B * max(Nt, 1)).reshape(B, max(Nt, 1)).copy()
        self.calls.append(dict(kind="align", B=B, T=T, start=_arr(start, ctypes.c_int32, start_len).tolist(), text=text_a,
                               lens=lens_a.tolist(), Nt=Nt, nf=_arr(nf, ctypes.c_int32, B).tolist(), width=width,
                               heads=_arr(heads, ctypes.c_int32, 2 * nh).reshape(nh, 2).tolist(), nt=nt_id.value,
                               eot=eot.value, matrix=matrix is not None))
        mp = Nt + 1 + S
        pa = _arr(path, ctypes.c_int32, B * mp * 2).reshape(B, mp, 2)
        pl = _arr(path_lens, ctypes.c_int32, B)
        pr = _arr(probs, ctypes.c_float, B * max(Nt, 1)).reshape(B, max(Nt, 1))
        for b in range(B):
            pl[b] = lens_a[b] + 1
            for i in range(lens_a[b] + 1):
                pa[b, i] = (i, b)                     # identifies the entry
            pr[b, :lens_a[b]] = text_a[b, :lens_a[b]] / 1000.0
        return 0

    def ct2b200_whisper_detect_language(self, h, f, B, T, sot, ids, n, probs):
        B = B.value
        self.calls.append(dict(kind="lang", B=B, sot=sot.value, ids=_arr(ids, ctypes.c_int32, n).tolist()))
        out = _arr(probs, ctypes.c_float, B * n).reshape(B, n)
        for b in range(B):
            out[b] = [0.25, 0.5, 0.25] if b == 0 else [0.1, 0.2, 0.7]
        return 0

    def ct2b200_last_error(self):
        return b""


@pytest.fixture
def fake(monkeypatch):
    f = FakeLib()
    monkeypatch.setattr(W, "lib", lambda: f)
    return f


def make(config):
    w = object.__new__(W.Whisper)
    w._h = 1
    w._tokens = ["<t%d>" % i for i in range(100)] + ["<|endoftext|>", "<|startoftranscript|>", "<|l0|>", "<|l1|>", "<|l2|>",
                                                     "<|translate|>", "<|transcribe|>", "<|startoflm|>", "<|startofprev|>",
                                                     "<|nospeech|>", "<|notimestamps|>"]
    w._ids = {t: i for i, t in enumerate(w._tokens)}
    w._config = config
    w.sot_id, w.eot_id, w.no_timestamps_id = 101, 100, 110
    w.n_mels, w.max_frames, w.d_model, w.vocab_size, w.decoder_positions = 16, 30, 64, len(w._tokens), 64
    return w


CONFIG = {"alignment_heads": [[1, 2], [0, 1], [1, 0]], "lang_ids": [102, 103, 104]}


def feats(batch):
    return np.zeros((batch, 16, 60), np.float32)


def test_align_int_num_frames_and_results_in_order(fake):
    w = make(CONFIG)
    res = w.align(feats(3), ["<|startoftranscript|>", 102, "<|transcribe|>"], [[5, 6], [], ["<t7>"]], 60, median_filter_width=3)
    c = fake.calls[-1]
    assert c["start"] == [101, 102, 106] and c["nf"] == [60, 60, 60] and c["width"] == 3
    assert c["heads"] == [[1, 2], [0, 1], [1, 0]] and c["nt"] == 110 and c["eot"] == 100 and not c["matrix"]
    assert c["lens"] == [2, 0, 1] and c["Nt"] == 2 and c["text"][2, 0] == 7
    assert [r.alignments for r in res] == [[(0, 0), (1, 0), (2, 0)], [(0, 1)], [(0, 2), (1, 2)]]
    assert res[0].text_token_probs == pytest.approx([0.005, 0.006]) and res[1].text_token_probs == []
    assert isinstance(res[0], W.WhisperAlignmentResult)


def test_align_per_entry_num_frames(fake):
    w = make(CONFIG)
    w.align(feats(2), [101], [[1], [2, 3]], [60, 7])
    assert fake.calls[-1]["nf"] == [60, 7]


def test_empty_batch(fake):
    assert make(CONFIG).align(feats(0), [101], [], []) == []
    assert make(CONFIG).detect_language(feats(0)) == []
    assert fake.calls == []


@pytest.mark.parametrize("kwargs, error", [
    (dict(num_frames=[60]), ValueError),                                   # len(num_frames) != batch
    (dict(median_filter_width=4), ValueError),                             # even width
    (dict(median_filter_width=131), ValueError),                           # wider than 129
    (dict(start_sequence=[]), ValueError),
    (dict(start_sequence=[101, 500]), ValueError),                         # id outside the vocabulary
    (dict(text_tokens=[[1], [-1]]), ValueError),
    (dict(text_tokens=[[1], list(range(62))]), ValueError),                # 1 + 62 + 2 > 64 positions
    (dict(num_frames=[60, 62]), ValueError),                               # more frames than the features hold
    (dict(num_frames=[60, -2]), ValueError),
    (dict(features=feats(3)), ValueError),                                 # one text per entry
    (dict(features=np.zeros((2, 16))), ValueError),                        # rank
])
def test_align_argument_checks_before_any_call(fake, kwargs, error):
    args = dict(features=feats(2), start_sequence=[101], text_tokens=[[1], [2]], num_frames=60, median_filter_width=7)
    args.update(kwargs)
    with pytest.raises(error):
        make(CONFIG).align(args["features"], args["start_sequence"], args["text_tokens"], args["num_frames"],
                           args["median_filter_width"])
    assert fake.calls == []


def test_align_without_alignment_heads(fake):
    with pytest.raises(RuntimeError, match="alignment_heads"):
        make({"lang_ids": [102, 103, 104]}).align(feats(1), [101], [[1]], 60)
    assert fake.calls == []


def test_widths_that_pass_through_are_accepted(fake):
    for width in (0, 1, 129):
        make(CONFIG).align(feats(1), [101], [[1]], 60, median_filter_width=width)
    assert [c["width"] for c in fake.calls] == [0, 1, 129]


def test_detect_language_sorted_stable_and_in_lang_ids_order(fake):
    res = make(CONFIG).detect_language(feats(2))
    assert fake.calls[-1]["ids"] == [102, 103, 104] and fake.calls[-1]["sot"] == 101
    # ties keep the lang_ids order
    assert res[0] == [("<|l1|>", 0.5), ("<|l0|>", 0.25), ("<|l2|>", 0.25)]
    assert [t for t, _ in res[1]] == ["<|l2|>", "<|l1|>", "<|l0|>"]


def test_detect_language_on_a_model_without_languages(fake):
    with pytest.raises(RuntimeError, match="multilingual"):
        make({"alignment_heads": [[0, 0]], "lang_ids": [102]}).detect_language(feats(1))
    assert fake.calls == []
