"""Random sampling on the GPU: the sampler op (ct2b200_random_sample) against the exact restatement of tests/sampling_ref.py,
its distribution, and Whisper.generate with sampling_topk / sampling_temperature on tiny_whisper against WhisperOracle
(teacher-forced scores of the sampled sequences, top-k membership, timestamp rules, first-token distribution), plus
reproducibility under set_random_seed and the state left for the other Whisper calls."""
import os

import numpy as np
import pytest
import torch
from scipy import stats

import ctranslate2_b200 as ct2
from ctranslate2_b200 import ops
from ctranslate2_b200.whisper import Whisper
from gpu_util import TDT, dev, gpu, round_through
from oracle import ct2_oracle as O
from sampling_ref import kept_set, random_sample_rows, whisper_teacher_forced

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MODEL = os.path.join(GOLDEN, "tiny_whisper")
LOWEST = {"float32": float(np.finfo(np.float32).min), "float16": -65504.0, "bfloat16": -3.3895313892515355e38}
NOTS = [101, 102, 106, 110]          # <|startoftranscript|><|l0|><|transcribe|><|notimestamps|>
TS = [101, 102, 106]                 # with timestamps


def rows_of(seed, n, vocab, dtype, spikes=0):
    """n rows of N(0, 9) logits; `spikes` entries per row raised by 40 (a peaked row, as a decoder's are: with a flat row of
    51 865 entries nearly every draw lands within 1e-5 of a cumulative boundary, where rounding decides the id)."""
    g = np.random.default_rng(seed)
    x = (g.standard_normal((n, vocab)) * 3).astype(np.float32)
    for r in range(n):
        x[r, g.choice(vocab, size=spikes, replace=False)] += 40
    for r in range(0, n, 2):                                   # suppressed entries on every other row
        x[r, g.choice(vocab, size=max(1, vocab // 10), replace=False)] = LOWEST[dtype]
    return round_through(x, dtype)


@gpu
@pytest.mark.parametrize("dtype", ["float32", "float16", "bfloat16"])
@pytest.mark.parametrize("vocab", [122, 51865, 51866])
def test_sampler_op_matches_the_restatement(dtype, vocab):
    x = rows_of(vocab, 8, vocab, dtype, spikes=4 if vocab > 1000 else 0)
    xt = dev(x, TDT[dtype])
    checked = total = 0
    for ki, k in enumerate([0, 1, 2, 40, 1000, vocab - 1, vocab]):
        if k > vocab:
            continue
        for ti, t in enumerate([0.1, 0.7, 1.0, 1.5]):
            counter = 16 * ki + ti
            ids, logp = ops.random_sample(xt, k, t, seed=1234, counter=counter, step=5)
            ids, logp = ids.cpu().numpy(), logp.cpu().numpy()
            rids, rlogp, dist = random_sample_rows(x, k, t, 1234, counter, 5, dtype)
            for r in range(x.shape[0]):
                assert ids[r] in set(kept_set(x[r], k).tolist()), (k, t, r)
                total += 1
                if dist[r] > 1e-5:
                    checked += 1
                    assert ids[r] == rids[r], (k, t, r, dist[r])
            lse = torch.logsumexp(torch.from_numpy(x.astype(np.float64)), dim=1).numpy()
            want = round_through((x[np.arange(x.shape[0]), ids] - lse).astype(np.float32), dtype)
            tol = 1e-5 if dtype == "float32" else 2e-2
            np.testing.assert_allclose(logp, want, rtol=tol, atol=tol)
    assert checked >= 0.99 * total, (checked, total)


@gpu
@pytest.mark.parametrize("dtype", ["float32", "float16", "bfloat16"])
def test_sampler_tiny_temperature_and_infinite_logits(dtype):
    """A temperature whose inverse overflows still draws a maximum of the row, and a row with an infinite logit draws it."""
    x = rows_of(3, 8, 51865, dtype, spikes=4)
    for k in (0, 2, 40):
        ids, _ = ops.random_sample(dev(x, TDT[dtype]), k, 1e-40, seed=5, counter=k)
        ids = ids.cpu().numpy()
        for r in range(x.shape[0]):
            assert x[r, ids[r]] == x[r].max(), (k, r)
    y = x.copy()
    y[:, 77] = np.inf
    for k, t in ((0, 1.0), (5, 0.7), (0, 1e-40)):
        ids, _ = ops.random_sample(dev(y, TDT[dtype]), k, t, seed=6, counter=k)
        assert (ids.cpu().numpy() == 77).all(), (k, t)


@gpu
@pytest.mark.parametrize("k, t", [(0, 1.0), (5, 0.7), (40, 1.5)])
def test_sampler_distribution(k, t):
    x = rows_of(7, 1, 122, "float32")[0]
    rows = 4096
    xt = dev(np.tile(x, (rows, 1)))
    counts = np.zeros(122)
    for counter in range(16):                                    # 2^16 draws
        ids, _ = ops.random_sample(xt, k, t, seed=99, counter=counter)
        counts += np.bincount(ids.cpu().numpy(), minlength=122)
    keep = kept_set(x, k)
    p = np.zeros(122)
    w = np.exp((x[keep].astype(np.float64) - x.max()) / t)
    p[keep] = w / w.sum()
    assert counts[p == 0].sum() == 0
    exp = p * counts.sum()
    big = exp >= 5
    obs = np.append(counts[big], counts[~big].sum())
    ex = np.append(exp[big], exp[~big].sum())
    if ex[-1] == 0:
        obs, ex = obs[:-1], ex[:-1]
    assert stats.chisquare(obs, ex).pvalue > 1e-3


# ---- Whisper.generate ----

def inputs(seed, batch, n_mels=16, frames=60):
    return (np.random.default_rng(seed).standard_normal((batch, n_mels, frames)) * 2).astype(np.float32)


@pytest.fixture(scope="module")
def model():
    w = Whisper(MODEL, compute_type="float32")
    yield w
    w.close()


@pytest.fixture(scope="module")
def oracle():
    return O.WhisperOracle.from_dir(MODEL, compute_type="float32")


def _pairs(res):
    return [(r.sequences_ids, r.scores) for r in res]


@gpu
@pytest.mark.parametrize("prompt", [NOTS, TS])
def test_best_sampler_is_the_deterministic_search(model, prompt):
    x = inputs(3, 3)
    base = _pairs(model.generate(x, [prompt] * 3, beam_size=1, max_length=24, return_scores=True))
    for kw in [dict(sampling_topk=1, sampling_temperature=0.3), dict(sampling_topk=1, sampling_temperature=2.0),
               dict(sampling_topk=0, sampling_temperature=0.0)]:
        assert _pairs(model.generate(x, [prompt] * 3, beam_size=1, max_length=24, return_scores=True, **kw)) == base


@gpu
def test_same_seed_same_results_with_and_without_the_graph(model):
    x = inputs(4, 3)
    kw = dict(beam_size=1, num_hypotheses=4, sampling_topk=0, sampling_temperature=1.5, max_length=24, return_scores=True)
    ct2.set_random_seed(17)
    a = [_pairs(model.generate(x, [NOTS] * 3, **kw)) for _ in range(2)]
    assert a[0] != a[1]                                          # the call counter advanced
    eager = Whisper(MODEL, compute_type="float32", use_cuda_graph=False)
    ct2.set_random_seed(17)
    b = [_pairs(eager.generate(x, [NOTS] * 3, **kw)) for _ in range(2)]
    eager.close()
    assert a == b
    ct2.set_random_seed(18)
    assert _pairs(model.generate(x, [NOTS] * 3, **kw)) != a[0]


@gpu
@pytest.mark.parametrize("prompt", [NOTS, TS])
@pytest.mark.parametrize("k", [0, 5])
def test_hypotheses_scores_and_membership(model, oracle, prompt, k):
    x = inputs(5, 2)
    max_length = 24
    steps = min(max_length // 2, max_length - (len(prompt) - 1))
    disable = list(oracle.config.get("suppress_ids", []))
    begin = list(oracle.config.get("suppress_ids_begin", []))
    lowest = np.finfo(np.float32).min
    ct2.set_random_seed(5 + k)
    for h in (1, 3, 8):
        for lp in (0.0, 1.0, 2.0):
            res = model.generate(x, [prompt] * 2, beam_size=1, num_hypotheses=h, sampling_topk=k, sampling_temperature=1.0,
                                 length_penalty=lp, max_length=max_length, return_scores=True)
            entries, seqs, scores = [], [], []
            for b, r in enumerate(res):
                assert len(r.sequences_ids) == h and len(r.scores) == h
                assert all(r.scores[j] >= r.scores[j + 1] for j in range(h - 1))
                entries += [b] * h
                seqs += r.sequences_ids
                scores += r.scores
            logits = whisper_teacher_forced(oracle, x, [prompt] * 2, entries, seqs, steps, disable, begin)
            for n, seq in enumerate(seqs):
                lps = O.softmax(logits[n], log=True)
                toks = seq + ([oracle.eot] if len(seq) < steps else [])
                total = sum(float(lps[s, tok]) for s, tok in enumerate(toks))
                if len(seq) == 0 and lp > 0:
                    continue
                np.testing.assert_allclose(scores[n], total / len(seq) ** lp, rtol=2e-4, atol=2e-4)
                for s, tok in enumerate(toks):
                    row = logits[n][s]
                    assert row[tok] > lowest, (n, s, tok)                       # allowed by the suppression / timestamp rules
                    if k:
                        assert (row > row[tok] + 1e-4).sum() < k, (n, s, tok)


@gpu
@pytest.mark.parametrize("k", [0, 5])
def test_first_token_distribution(model, oracle, k):
    B, H, t = 8, 32, 0.7
    x = inputs(6, B)
    disable = list(oracle.config.get("suppress_ids", []))
    begin = list(oracle.config.get("suppress_ids_begin", []))
    first = whisper_teacher_forced(oracle, x, [NOTS] * B, list(range(B)), [[]] * B, 1, disable, begin)
    expected = np.zeros(oracle.vocab)
    for b in range(B):
        row = first[b][0].astype(np.float64)
        keep = kept_set(row, k)
        w = np.exp((row[keep] - row.max()) / t)
        expected[keep] += w / w.sum()
    counts = np.zeros(oracle.vocab)
    seeds = 16
    for seed in range(seeds):
        ct2.set_random_seed(1000 + seed)
        res = model.generate(x, [NOTS] * B, beam_size=1, num_hypotheses=H, sampling_topk=k, sampling_temperature=t,
                             max_length=8, return_scores=True)
        for r in res:
            for s in r.sequences_ids:
                counts[s[0] if s else oracle.eot] += 1
    expected *= seeds * H
    assert counts[expected == 0].sum() == 0
    big = expected >= 5
    obs = np.append(counts[big], counts[~big].sum())
    ex = np.append(expected[big], expected[~big].sum())
    if ex[-1] == 0:
        obs, ex = obs[:-1], ex[:-1]
    assert stats.chisquare(obs, ex).pvalue > 1e-3


@gpu
def test_no_state_left_for_other_calls(model):
    x = inputs(8, 2)

    def others():
        g = _pairs(model.generate(x, [TS] * 2, beam_size=5, num_hypotheses=2, max_length=24, return_scores=True))
        a = [(r.alignments, r.text_token_probs) for r in model.align(x, [101, 102, 106], [[5, 6, 7], [8, 9]], 60)]
        return g, a, model.detect_language(x)

    before = others()
    ct2.set_random_seed(3)
    model.generate(x, [TS] * 2, beam_size=1, num_hypotheses=8, sampling_topk=0, sampling_temperature=1.0, max_length=24)
    assert others() == before
