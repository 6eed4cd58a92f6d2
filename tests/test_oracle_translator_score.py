"""The scoring restatement (tests/seq2seq_scoring.py: Seq2SeqOracle's cached one-token path with teacher forcing) against
Translator::score_batch of the unmodified reference (tests/golden/seq2seq_score_ref.json, tools/make_golden.py
--translator-score-only), in float32 where nothing is quantized.  This pins the oracle the GPU tests use on longer targets."""
import json
import os

import numpy as np
import pytest

from oracle import ct2_oracle as O
from seq2seq_scoring import oracle_score, pair_ids

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def fixture():
    with open(os.path.join(GOLDEN, "seq2seq_score_ref.json"), encoding="utf-8") as f:
        return json.load(f)


@pytest.mark.parametrize("name", ["aren-float32", "postnorm-float32"])
def test_oracle_scores_match_the_reference(fixture, name):
    m = fixture["models"][name]
    mdir = os.path.join(GOLDEN, m["model"])
    oracle = O.Seq2SeqOracle.from_dir(mdir, compute_type="float32")
    checked = 0
    for c in m["cases"]:
        ids = [pair_ids(mdir, s, t, c["max_input_length"]) for s, t in zip(c["source"], c["target"])]
        run = [b for b, (s, _) in enumerate(ids) if s]
        got = oracle_score(oracle, [ids[b][0] for b in run], [ids[b][1] for b in run], c["offset"])
        for b, g in zip(run, got):
            np.testing.assert_allclose(g, c["log_probs"][b], atol=1e-5, rtol=0)
            checked += len(g)
        for b in set(range(len(ids))) - set(run):                  # an empty source scores 0 without the offset
            assert c["log_probs"][b] == [0.0] * (len(ids[b][1]) - 1)
    assert checked > 150
