"""Host logic of ctranslate2_b200.Generator.score_batch without a device: the C-ABI is replaced by a recording fake, so what is
checked is the Python side — vocabulary lookup, truncation (Vocabulary::to_ids, src/vocabulary.cc:130-140), the skip of
sequences shorter than two tokens, re-batching (src/batch_reader.cc:18-77, 175-225: longest first, "examples" / "tokens" with
padding counted, answered in request order), the arena cap and the argument checks.  No compute is claimed here;
tests/test_gpu_score.py covers the real library."""
import ctypes

import numpy as np
import pytest

import ctranslate2_b200.generator as G


def _arr(ptr, ctype, n):
    return np.ctypeslib.as_array((ctype * n).from_address(ptr.value))


class FakeLib:
    """ct2b200_score_batch: the 'score' of a token is -id / 1000, so every result identifies the tokens it was given."""

    def __init__(self):
        self.calls = []

    def ct2b200_score_batch(self, h, ids, lens, B, L, offset, out):
        B, L, offset = B.value, L.value, offset.value
        ids_a = _arr(ids, ctypes.c_int32, B * L).reshape(B, L).copy()
        lens_a = _arr(lens, ctypes.c_int32, B).copy()
        self.calls.append((ids_a, lens_a, offset))
        out_a = _arr(out, ctypes.c_float, B * (L - 1)).reshape(B, L - 1)
        out_a[:] = 0
        for b in range(B):
            for t in range(offset, lens_a[b] - 1):
                out_a[b, t - offset] = -ids_a[b, t + 1] / 1000.0
        return 0

    def ct2b200_last_error(self):
        return b""


EOS = 2


@pytest.fixture
def gen(monkeypatch):
    fake = FakeLib()
    monkeypatch.setattr(G, "lib", lambda: fake)
    g = object.__new__(G.Generator)
    g._h, g.max_batch_size, g.max_length, g.vocab_size = 1, 4, 64, 1000
    g._tokens = ["<t%d>" % i for i in range(1000)]
    g._token_to_id, g._config = None, {"eos_token": "<t%d>" % EOS}
    yield g, fake
    g._h = None


def _expected(seq, offset=0):
    return [-t / 1000.0 for t in seq[1 + offset:]]


def test_scores_come_back_in_request_order_with_token_strings(gen):
    g, fake = gen
    seqs = [[5, 6, 7], [8, 9], [10, 11, 12, 13]]
    res = g.score_batch([["<t%d>" % t for t in s] for s in seqs])
    assert len(fake.calls) == 1
    for s, r in zip(seqs, res):
        assert isinstance(r, G.ScoringResult)
        assert r.tokens == ["<t%d>" % t for t in s[1:]]
        np.testing.assert_allclose(r.log_probs, _expected(s), rtol=1e-6)
    ids, lens, _ = fake.calls[0]
    assert lens.tolist() == [4, 3, 2]                                       # longest first
    for b in range(len(lens)):                                              # right-padded with 0
        assert (ids[b, lens[b]:] == 0).all()
    assert g.score_batch([]) == [] and len(fake.calls) == 1


def test_sequences_shorter_than_two_tokens_are_not_sent(gen):
    g, fake = gen
    res = g.score_batch([[7], [], [3, 4], [9]])
    assert [r.log_probs for r in res[:2]] == [[], []] and res[3].log_probs == [] and res[3].tokens == []
    np.testing.assert_allclose(res[2].log_probs, _expected([3, 4]))
    assert [c[1].tolist() for c in fake.calls] == [[2]]
    fake.calls.clear()
    assert g.score_batch([[1], [5]]) == [G.ScoringResult([], []), G.ScoringResult([], [])]
    assert fake.calls == []


@pytest.mark.parametrize("offset", [0, 1, 3, 9])
def test_offset_is_passed_through(gen, offset):
    g, fake = gen
    seqs = [[5, 6, 7, 8, 9], [10, 11, 12]]
    res = g.score_batch(seqs, offset=offset)
    assert fake.calls[0][2] == offset
    for s, r in zip(seqs, res):
        np.testing.assert_allclose(r.log_probs, _expected(s, offset), rtol=1e-6)
        assert r.tokens == ["<t%d>" % t for t in s[1 + offset:]]
        assert len(r.log_probs) == max(0, len(s) - 1 - offset)


def test_truncation_keeps_the_end_token(gen):
    g, fake = gen
    cases = [
        ([5, 6, 7, 8, 9], 3, [5, 6, 7]),                         # plain cut
        ([5, 6, 7, 8, EOS], 3, [5, 6, EOS]),                     # EOS last: kept in the last position
        ([5, 6, 7, EOS, 9], 3, [5, EOS, 9]),                     # EOS second to last: EOS, then the original last token
        ([5, 6, 7, EOS, 9], 1, None),                            # max_input_length 1: cut to [5], scores nothing
        ([5, 6, EOS], 2, [5, EOS]),
        ([5, 6, 7, 8, 9], 0, [5, 6, 7, 8, 9]),                   # 0 disables truncation
        ([5, 6, 7], 3, [5, 6, 7]),                               # not longer than the limit: unchanged
    ]
    for seq, limit, kept in cases:
        fake.calls.clear()
        r = g.score_batch([seq], max_input_length=limit)[0]
        if kept is None:
            assert r.log_probs == [] and fake.calls == []
            continue
        ids, lens, _ = fake.calls[0]
        assert ids[0, :lens[0]].tolist() == kept
        np.testing.assert_allclose(r.log_probs, _expected(kept), rtol=1e-6)
    # a sequence of 100 tokens does not fit a 64-position arena unless it is truncated
    long = list(range(3, 103))
    fake.calls.clear()
    with pytest.raises(ValueError):
        g.score_batch([long], max_input_length=0)
    assert fake.calls == []
    assert len(g.score_batch([long], max_input_length=64)[0].log_probs) == 63 and fake.calls[-1][1].tolist() == [64]
    assert len(g.score_batch([long], max_input_length=50)[0].log_probs) == 49


def test_examples_rebatching_and_the_arena_cap(gen):
    g, fake = gen
    r = np.random.default_rng(0)
    seqs = [[int(10 + i)] + r.integers(3, 900, size=int(n)).tolist() for i, n in enumerate(r.integers(1, 12, size=11))]
    res = g.score_batch(seqs)                                               # max_batch_size 0: the arena's 4 rows cap
    assert [len(c[1]) for c in fake.calls] == [4, 4, 3]
    served = [int(n) for c in fake.calls for n in c[1]]
    assert served == sorted((len(s) for s in seqs), reverse=True)
    for s, x in zip(seqs, res):
        np.testing.assert_allclose(x.log_probs, _expected(s), rtol=1e-6)
    fake.calls.clear()
    res2 = g.score_batch(seqs, max_batch_size=3)
    assert [len(c[1]) for c in fake.calls] == [3, 3, 3, 2]
    assert [x.log_probs for x in res2] == [x.log_probs for x in res]
    fake.calls.clear()
    g.score_batch(seqs, max_batch_size=100)                                 # the arena still caps every call
    assert [len(c[1]) for c in fake.calls] == [4, 4, 3]


def test_tokens_rebatching_counts_padding(gen):
    g, fake = gen
    lengths = [9, 3, 7, 7, 2, 5, 6, 4]
    seqs = [[100 + i] + [50] * (n - 1) for i, n in enumerate(lengths)]
    res = g.score_batch(seqs, max_batch_size=16, batch_type="tokens")
    # sorted: 9 (9 7 would be 2 x 9 = 18) | 7 7 (14; a third row 21) | 6 5 (12; 6 5 4 would be 18) | 4 3 2 (3 x 4 = 12)
    sizes = []
    order = sorted(lengths, reverse=True)
    i = 0
    while i < len(order):                   # the padding formula: rows_after_adding * longest <= max_batch_size
        n = 1
        while i + n < len(order) and (n + 1) * order[i] <= 16 and n + 1 <= 4:
            n += 1
        sizes.append(n)
        i += n
    assert [len(c[1]) for c in fake.calls] == sizes == [1, 2, 2, 3]
    for c in fake.calls:
        assert len(c[1]) * int(c[1].max()) <= 16 or len(c[1]) == 1
    for s, x in zip(seqs, res):
        np.testing.assert_allclose(x.log_probs, _expected(s), rtol=1e-6)
    fake.calls.clear()
    g.score_batch(seqs, max_batch_size=4, batch_type="tokens")              # smaller than the longest row: one row each
    assert [len(c[1]) for c in fake.calls] == [1] * len(seqs)


def test_refusals_happen_before_any_call(gen):
    g, fake = gen
    ok = [[5, 6, 7]] * 9
    for kw in (dict(asynchronous=True), dict(batch_type="sentences"), dict(max_batch_size=-1), dict(max_batch_size=1.5),
               dict(max_batch_size=True), dict(max_input_length=-1), dict(max_input_length=2.0), dict(offset=-1),
               dict(offset=0.5), dict(offset=None)):
        with pytest.raises(ValueError):
            g.score_batch(ok, **kw)
    with pytest.raises(ValueError):
        g.score_batch(ok + [[5, 1000]])                                     # id outside the vocabulary
    with pytest.raises(ValueError):
        g.score_batch(ok + [[-1, 5]])
    with pytest.raises(ValueError):
        g.score_batch(ok + [list(range(3, 70))], max_input_length=0)        # longer than the arena after truncation
    with pytest.raises(TypeError):
        g.score_batch(ok, 4)                                                # options are keyword-only
    assert fake.calls == []
