"""The score convention of random sampling, pinned on the reference's own sampled sequences: tests/golden/whisper_sampling_ref.json
holds models::Whisper::generate with a RandomSampler of the unmodified reference (CPU, float32) on tiny_whisper
(tools/make_golden.py --whisper-sampling-only).  Without RNG parity the draws cannot be compared; what is compared is that the
oracle's teacher-forced processed log-probabilities (SuppressTokens, SuppressTokensBegin, the timestamp rules) of those very
sequences, the end token counted when the row ended with it, over length^length_penalty, give the reference's scores, and that
every sampled token was inside the top k of its processed row.  The GPU tests hold the engine to the same restatement."""
import json
import os

import numpy as np
import pytest

from oracle import ct2_oracle as O
from sampling_ref import whisper_teacher_forced

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def fixture():
    with open(os.path.join(GOLDEN, "whisper_sampling_ref.json")) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def oracle():
    return O.WhisperOracle.from_dir(os.path.join(GOLDEN, "tiny_whisper"), compute_type="float32")


def inputs(seed, batch, n_mels, frames):
    return (np.random.default_rng(seed).standard_normal((batch, n_mels, frames)) * 2).astype(np.float32)


def test_fixture_covers_the_sampler_options(fixture):
    cases = fixture["cases"]
    assert len(cases) == 48
    assert {c["sampling_topk"] for c in cases} == {0, 5} and {c["sampling_temperature"] for c in cases} == {0.5, 1.0, 1.5}
    assert {c["num_hypotheses"] for c in cases} == {1, 3} and {c["length_penalty"] for c in cases} == {0.0, 1.0}
    assert {len(c["prompt"]) for c in cases} == {3, 4}
    for c in cases:
        for hyps in c["results"]:
            assert len(hyps) == c["num_hypotheses"]
            assert all(hyps[j]["score"] >= hyps[j + 1]["score"] for j in range(len(hyps) - 1))   # best first


def test_reference_scores_are_teacher_forced_log_probabilities(fixture, oracle):
    B, L = fixture["batch"], fixture["max_length"]
    disable = list(oracle.config.get("suppress_ids", []))
    begin = list(oracle.config.get("suppress_ids_begin", []))
    lowest = np.finfo(np.float32).min
    checked = ended = 0
    for c in fixture["cases"]:
        prompt, k, lp = c["prompt"], c["sampling_topk"], c["length_penalty"]
        steps = min(L // 2, L - (len(prompt) - 1))
        entries = [b for b in range(B) for _ in c["results"][b]]
        seqs = [h["ids"] for b in range(B) for h in c["results"][b]]
        scores = [h["score"] for b in range(B) for h in c["results"][b]]
        x = inputs(c["seed"], B, fixture["n_mels"], fixture["frames"])
        logits = whisper_teacher_forced(oracle, x, [prompt] * B, entries, seqs, steps, disable, begin)
        for n, seq in enumerate(seqs):
            lps = O.softmax(logits[n], log=True)
            toks = seq + ([oracle.eot] if len(seq) < steps else [])
            ended += len(seq) < steps
            total = sum(float(lps[s, t]) for s, t in enumerate(toks))
            if len(seq) == 0 and lp > 0:
                continue
            assert scores[n] == pytest.approx(total / len(seq) ** lp, abs=1e-5, rel=1e-5), (c["seed"], n)
            for s, t in enumerate(toks):
                row = logits[n][s]
                assert row[t] > lowest, (c["seed"], n, s, t)
                if k:
                    assert (row > row[t]).sum() < k, (c["seed"], n, s, t)
            checked += 1
    assert checked >= 150 and ended >= 4, (checked, ended)          # rows that ended with <|endoftext|> pin its log-probability
