"""Random sampling without a device: Philox4x32-10 known-answer vectors (the restatement and the library's own host code), the
exact sampler restatement on hand-made rows, and the host logic of Whisper.generate's sampler options over a recording fake
C-ABI -- every refusal raised before any library call, the sampled entry point reached with the right k, temperature and
num_hypotheses, and the deterministic entry point whenever the sampler is the best one.  tests/test_gpu_whisper_sampling.py
covers the device."""
import ctypes

import numpy as np
import pytest

import ctranslate2_b200.whisper as W
from sampling_ref import kept_set, philox4x32_10, philox_uniform, random_sample_rows

KAT = [
    ([0, 0, 0, 0], [0, 0], [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]),
    ([0xFFFFFFFF] * 4, [0xFFFFFFFF] * 2, [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]),
    ([0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344], [0xA4093822, 0x299F31D0],
     [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]),
]


@pytest.mark.parametrize("counter, key, expected", KAT)
def test_philox_known_answers(counter, key, expected):
    assert philox4x32_10(counter, key) == expected
    from ctranslate2_b200 import ops
    assert ops.philox4x32_10(counter, key) == expected


def test_uniform_takes_the_top_24_bits_of_word_0():
    w0 = philox4x32_10([7, 3, 2, 0], [11, 0])[0]
    assert philox_uniform(11, 2, 3, 7) == (w0 >> 8) / 2.0 ** 24
    us = [philox_uniform(5, 0, r, s) for r in range(64) for s in range(64)]
    assert 0.0 <= min(us) and max(us) < 1.0 and abs(np.mean(us) - 0.5) < 0.02


def test_kept_set_breaks_ties_by_lowest_index():
    x = np.array([1.0, 3.0, 2.0, 3.0, 2.0, -0.0, 0.0])
    assert kept_set(x, 3).tolist() == [1, 2, 3]
    assert kept_set(x, 6).tolist() == [0, 1, 2, 3, 4, 5]
    assert kept_set(x, 0).tolist() == list(range(7)) and kept_set(x, 7).tolist() == list(range(7))


def test_restated_sampler_follows_the_inverse_cdf():
    x = np.log(np.array([[1.0, 2.0, 1.0, 4.0]], np.float32))
    ids, logp, dist = random_sample_rows(x, 0, 1.0, seed=3, call=1)
    u = philox_uniform(3, 1, 0, 0)
    assert ids[0] == int(np.searchsorted(np.cumsum([1, 2, 1, 4]) / 8.0, u, side="right"))
    assert logp[0] == pytest.approx(np.log([1, 2, 1, 4][ids[0]] / 8.0), abs=1e-6)
    assert 0 <= dist[0] <= 0.5
    ids, _, _ = random_sample_rows(x, 1, 1.0, seed=3, call=1)
    assert ids[0] == 3


# ---- Whisper.generate host logic ----

def _arr(ptr, ctype, n):
    return np.ctypeslib.as_array((ctype * n).from_address(ptr.value))


class FakeLib:
    def __init__(self):
        self.calls = []

    def _record(self, kind, args, sampler):
        (h, f, B, T, pr, P, beam, patience, lp, max_length, nh, sup, nsup, beg, nbeg, sot, eot, nsp_id, nt, mit) = args
        out, lens, scores, nsp = sampler[-4:]
        B, nh, L = B.value, nh, max_length.value
        call = dict(kind=kind, B=B, beam=beam, num_hypotheses=nh)
        if kind == "sampling":
            call["topk"], call["temperature"] = sampler[0], sampler[1].value
        self.calls.append(call)
        o = _arr(out, ctypes.c_int32, B * nh * L).reshape(B, nh, L)
        ln = _arr(lens, ctypes.c_int32, B * nh).reshape(B, nh)
        sc = _arr(scores, ctypes.c_float, B * nh).reshape(B, nh)
        for b in range(B):
            for j in range(nh):
                ln[b, j] = 2
                o[b, j, :2] = [b, j]
                sc[b, j] = -float(j)
        return 0

    def ct2b200_whisper_generate(self, *args):
        return self._record("search", args[:20], args[20:])

    def ct2b200_whisper_generate_sampling(self, *args):
        return self._record("sampling", args[:20], args[20:])

    def ct2b200_translator_close(self, h):
        return 0

    def ct2b200_last_error(self):
        return b""


@pytest.fixture
def fake(monkeypatch):
    f = FakeLib()
    monkeypatch.setattr(W, "lib", lambda: f)
    return f


def make():
    w = object.__new__(W.Whisper)
    w._h = 1
    w._tokens = ["<t%d>" % i for i in range(100)] + ["<|endoftext|>", "<|startoftranscript|>", "<|l0|>", "<|l1|>", "<|l2|>",
                                                     "<|translate|>", "<|transcribe|>", "<|startoflm|>", "<|startofprev|>",
                                                     "<|nospeech|>", "<|notimestamps|>"]
    w._ids = {t: i for i, t in enumerate(w._tokens)}
    w._config = {}
    w.sot_id, w.eot_id, w.no_timestamps_id, w.no_speech_id = 101, 100, 110, 109
    w.n_mels, w.max_frames, w.d_model, w.vocab_size, w.decoder_positions = 16, 30, 64, len(w._tokens), 64
    return w


PROMPT = [[101, 102, 106, 110]]


def feats(batch=1):
    return np.zeros((batch, 16, 60), np.float32)


@pytest.mark.parametrize("kwargs", [
    dict(sampling_topk=-1),
    dict(sampling_temperature=-0.5),
    dict(sampling_topk=-1, sampling_temperature=0.0),
    dict(sampling_topk=112, beam_size=1),                       # more than the vocabulary (111 tokens)
    dict(sampling_topk=0, sampling_temperature=0.7, beam_size=5),   # sampled beam search
    dict(sampling_topk=5, beam_size=2, num_hypotheses=2),
    dict(sampling_topk=0, beam_size=1, num_hypotheses=33),
    dict(sampling_topk=0, beam_size=1, num_hypotheses=0),
    dict(sampling_topk=0, beam_size=1, repetition_penalty=1.2),
    dict(sampling_topk=0, beam_size=1, no_repeat_ngram_size=2),
    dict(sampling_topk=0, beam_size=1, return_logits_vocab=True),
])
def test_refusals_raise_before_any_call(fake, kwargs):
    with pytest.raises(ValueError):
        make().generate(feats(), PROMPT, **kwargs)
    assert fake.calls == []


@pytest.mark.parametrize("k, t, h", [(0, 1.0, 1), (0, 0.7, 5), (5, 1.5, 3), (111, 0.2, 32), (2, 1.0, 8)])
def test_random_sampler_reaches_the_sampled_entry_point(fake, k, t, h):
    res = make().generate(feats(2), PROMPT * 2, beam_size=1, num_hypotheses=h, sampling_topk=k, sampling_temperature=t,
                          return_scores=True)
    c = fake.calls[-1]
    assert c["kind"] == "sampling" and c["topk"] == k and c["temperature"] == pytest.approx(t)
    assert c["beam"] == 1 and c["num_hypotheses"] == h and c["B"] == 2
    assert [len(r.sequences_ids) for r in res] == [h, h]
    assert res[1].sequences_ids[-1] == [1, h - 1] and res[0].scores == [-float(j) for j in range(h)]


@pytest.mark.parametrize("kwargs", [
    dict(sampling_topk=1, sampling_temperature=0.3),
    dict(sampling_topk=1, sampling_temperature=2.0),
    dict(sampling_topk=0, sampling_temperature=0.0),
    dict(sampling_topk=5, sampling_temperature=0.0, beam_size=5),   # the best sampler: beam search stays available
    dict(sampling_topk=500, sampling_temperature=0.0, beam_size=1),  # k is only checked by the random sampler
    dict(),
])
def test_best_sampler_reaches_the_search_entry_point(fake, kwargs):
    make().generate(feats(), PROMPT, **kwargs)
    c = fake.calls[-1]
    assert c["kind"] == "search" and c["beam"] == kwargs.get("beam_size", 5)
