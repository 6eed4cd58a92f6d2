"""CPU checks of the host side of Whisper.align: ct2b200_negative_dtw_host (the function the engine runs on its matrices)
against the numpy restatement of the reference's negative_dtw (src/dtw.cc) on random and tie-heavy matrices, the DTW and
median-filter edge cases, and the committed fixture of the UNMODIFIED reference (tests/golden/whisper_align_ref.json): its
alignments are DTW paths of the right shape, its detect_language results are sorted distributions, and the fp32 oracle
(whisper_align_ref.WhisperAlignOracle, the yardstick of tests/test_gpu_whisper_align.py) reproduces it: float32 alignments
identical, probabilities to 1e-5."""
import ctypes
import json
import os

import numpy as np
import pytest

from ctranslate2_b200._lib import check, lib
from whisper_align_ref import median_filter, negative_dtw

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def host_dtw(x):
    x = np.ascontiguousarray(x, np.float32)
    n, m = x.shape
    out = np.zeros((n + m, 2), np.int32)
    k = ctypes.c_int32()
    p = ctypes.c_void_p
    check(lib().ct2b200_negative_dtw_host(x.ctypes.data_as(p), ctypes.c_int64(n), ctypes.c_int64(m), out.ctypes.data_as(p),
                                          ctypes.byref(k)))
    return [(int(i), int(j)) for i, j in out[:k.value]]


@pytest.mark.parametrize("seed", range(6))
def test_host_dtw_equals_the_restatement_on_random_matrices(seed):
    r = np.random.default_rng(seed)
    for _ in range(20):
        n, m = (int(v) for v in r.integers(1, 16, size=2))
        x = r.standard_normal((n, m)).astype(np.float32)
        assert host_dtw(x) == negative_dtw(x)


@pytest.mark.parametrize("seed", range(4))
def test_host_dtw_equals_the_restatement_on_tie_heavy_matrices(seed):
    r = np.random.default_rng(100 + seed)
    for _ in range(20):
        n, m = (int(v) for v in r.integers(1, 12, size=2))
        x = r.integers(-1, 2, size=(n, m)).astype(np.float32)
        assert host_dtw(x) == negative_dtw(x)


def test_dtw_edge_cases():
    # one row: the path walks the columns
    assert host_dtw(np.zeros((1, 4))) == [(0, 0), (0, 1), (0, 2), (0, 3)]
    # one element
    assert host_dtw(np.ones((1, 1))) == [(0, 0)]
    # all ties: up and diagonal never win strictly, so the first step is the diagonal and the rest go left then up
    assert host_dtw(np.zeros((3, 3))) == negative_dtw(np.zeros((3, 3)))
    # one column
    assert host_dtw(np.zeros((3, 1))) == negative_dtw(np.zeros((3, 1)))
    # NaN (a constant frame column standardised with epsilon 0) falls through to "left", as in the reference
    x = np.full((4, 1), np.nan, np.float32)
    assert host_dtw(x) == negative_dtw(x)


def test_median_filter_edges():
    x = np.array([[5, 1, 4, 2, 3, 9, 0]], np.float32)
    # width 3 mirrors |j + k| at the start and depth - (read - depth) - 2 at the end
    assert median_filter(x, 3).tolist() == [[1, 4, 2, 3, 3, 3, 9]]
    # width 1 and widths whose half reaches the depth pass through
    assert median_filter(x, 1).tolist() == x.tolist()
    assert median_filter(x[:, :3], 7).tolist() == x[:, :3].tolist()
    # width 5 at both edges
    assert median_filter(x, 5)[0, 0] == 4 and median_filter(x, 5)[0, -1] == 3


def test_fixture_alignments_are_dtw_paths():
    fx = json.load(open(os.path.join(GOLDEN, "whisper_align_ref.json")))
    assert set(fx["models"]) == {"model-float32", "model-int8", "permuted-float32", "permuted-int8"}
    empty = 0
    for name, model in fx["models"].items():
        for c in model["cases"]:
            nf = [n // 2 for n in c["num_frames"]]
            assert len(c["results"]) == c["batch"]
            for b, r in enumerate(c["results"]):
                n = len(c["text_tokens"][b])
                assert len(r["text_token_probs"]) == n
                assert all(0 <= p <= 1 for p in r["text_token_probs"])
                # ids >= <|endoftext|> are outside the softmax: probability 0
                for t, tok in enumerate(c["text_tokens"][b]):
                    if tok >= 100:
                        assert r["text_token_probs"][t] == 0
                path = r["alignments"]
                if nf[b] == 0 or all(v == 0 for v in nf):
                    assert path == []
                    empty += 1
                    continue
                assert path[-1] == [n, nf[b] - 1]
                for (i0, j0), (i1, j1) in zip(path, path[1:]):
                    assert (i1 - i0, j1 - j0) in ((1, 1), (1, 0), (0, 1))
    assert empty >= 8


def test_fixture_detect_language_is_sorted_and_normalised():
    fx = json.load(open(os.path.join(GOLDEN, "whisper_align_ref.json")))
    for name in ("model-float32", "model-int8"):
        for c in fx["models"][name]["detect_language"]:
            for r in c["results"]:
                probs = [p for _, p in r]
                assert probs == sorted(probs, reverse=True)
                assert abs(sum(probs) - 1) < 1e-5
                assert sorted(t for t, _ in r) == ["<|l0|>", "<|l1|>", "<|l2|>"]


def _fixture_inputs(seed, batch):
    return (np.random.default_rng(seed).standard_normal((batch, 16, 60)) * 2).astype(np.float32)


@pytest.mark.parametrize("heads", ["model", "permuted"])
def test_oracle_float32_equals_the_reference(heads):
    """WhisperAlignOracle (fp32 restatement of whisper.cc:387-652) against the reference's CPU build: every alignment
    identical, text_token_probs and language probabilities to 1e-5."""
    from whisper_align_ref import WhisperAlignOracle
    fx = json.load(open(os.path.join(GOLDEN, "whisper_align_ref.json")))
    o = WhisperAlignOracle(os.path.join(GOLDEN, "tiny_whisper"), compute_type="float32")
    hl = None if heads == "model" else fx["permuted_heads"]
    entries = 0
    for c in fx["models"][heads + "-float32"]["cases"]:
        res, _ = o.align(_fixture_inputs(c["seed"], c["batch"]), c["start_sequence"], c["text_tokens"], c["num_frames"],
                         c["median_filter_width"], heads=hl)
        for b, ((path, probs), ref) in enumerate(zip(res, c["results"])):
            assert [list(p) for p in path] == ref["alignments"], (c["seed"], b)
            np.testing.assert_allclose(probs, ref["text_token_probs"], atol=1e-5, rtol=0)
            entries += 1
    assert entries >= 25
    if heads == "model":
        for c in fx["models"]["model-float32"]["detect_language"]:
            ids, probs = o.detect_language(_fixture_inputs(c["seed"], c["batch"]))
            tokens = ["<|l%d|>" % (i - 102) for i in ids]
            for row, ref in zip(probs, c["results"]):
                want = dict(ref)
                for t, p in zip(tokens, row):
                    assert abs(p - want[t]) <= 1e-5, (t, p, want[t])
