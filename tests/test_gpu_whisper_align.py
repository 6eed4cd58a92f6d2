"""Whisper.align and Whisper.detect_language on the GPU against the committed outputs of the UNMODIFIED reference's
models::Whisper (tests/golden/whisper_align_ref.json, CPU build): the tiny model with its own alignment_heads and with a copy
whose config.json lists heads of both decoder layers out of order.  float32: every alignment identical, text_token_probs and
language probabilities to 2e-4, and the DTW matrix against the fp32 oracle (tests/whisper_align_ref.py, pinned to the same
fixture on the CPU) to 1e-4; int8 / float16: most alignments identical (a d = 64 model amplifies single rounding flips into
different DTW paths), probabilities close.  A 1500-position model (multi-block standardisation, wide median rows, captures of
hundreds of positions, two passes) against the oracle in float32 and float16."""
import json
import os
import shutil

import numpy as np
import pytest

from ctranslate2_b200.whisper import Whisper
from gpu_util import gpu
from whisper_align_ref import WhisperAlignOracle, negative_dtw, path_cost

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MODEL = os.path.join(GOLDEN, "tiny_whisper")


def inputs(seed, batch, n_mels=16, frames=60):
    return (np.random.default_rng(seed).standard_normal((batch, n_mels, frames)) * 2).astype(np.float32)


@pytest.fixture(scope="module")
def fixture():
    with open(os.path.join(GOLDEN, "whisper_align_ref.json")) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def permuted(fixture, tmp_path_factory):
    d = str(tmp_path_factory.mktemp("whisper") / "tiny_whisper_heads")
    shutil.copytree(MODEL, d)
    cfg = json.load(open(os.path.join(MODEL, "config.json")))
    cfg["alignment_heads"] = fixture["permuted_heads"]
    json.dump(cfg, open(os.path.join(d, "config.json"), "w"))
    return d


def _align(w, c, matrix=False):
    return w._align(inputs(c["seed"], c["batch"]), c["start_sequence"], c["text_tokens"], c["num_frames"],
                    c["median_filter_width"], return_matrix=matrix)


@gpu
@pytest.mark.parametrize("heads", ["model", "permuted"])
def test_float32_alignments_equal_the_reference(fixture, permuted, heads):
    w = Whisper(MODEL if heads == "model" else permuted, compute_type="float32")
    oracle = WhisperAlignOracle(MODEL, compute_type="float32")
    hl = None if heads == "model" else fixture["permuted_heads"]
    entries = 0
    for c in fixture["models"][heads + "-float32"]["cases"]:
        res, matrix = _align(w, c, matrix=True)
        _, want = oracle.align(inputs(c["seed"], c["batch"]), c["start_sequence"], c["text_tokens"], c["num_frames"],
                               c["median_filter_width"], heads=hl)
        assert len(res) == c["batch"]
        for b, (r, ref) in enumerate(zip(res, c["results"])):
            assert [list(p) for p in r.alignments] == ref["alignments"], (c["seed"], b)
            np.testing.assert_allclose(r.text_token_probs, ref["text_token_probs"], atol=2e-4, rtol=0)
            nf = c["num_frames"][b] // 2
            if r.alignments and nf > 0:
                # the path is the DTW of the returned matrix, and nothing past the entry's rows / frames is set
                n = len(c["text_tokens"][b])
                assert negative_dtw(matrix[b, :n + 1, :nf]) == r.alignments
                assert not matrix[b, n + 1:].any() and not matrix[b, :, nf:].any()
                np.testing.assert_allclose(matrix[b, :n + 1, :nf], want[b], atol=1e-4, rtol=1e-4, equal_nan=True)
            entries += 1
    assert entries >= 25
    w.close()


@gpu
@pytest.mark.parametrize("compute", ["int8", "float16", "int8_float16"])
def test_reduced_precision_alignments_mostly_equal_the_reference(fixture, permuted, compute):
    ref_model = fixture["models"]["permuted-" + ("int8" if compute.startswith("int8") else "float32")]
    w = Whisper(permuted, compute_type=compute)
    same = total = 0
    diffs = []
    for c in ref_model["cases"]:
        res, matrix = _align(w, c, matrix=True)
        for b, (r, ref) in enumerate(zip(res, c["results"])):
            total += 1
            if [list(p) for p in r.alignments] == ref["alignments"]:
                same += 1
            elif r.alignments:
                # a different path must be as good a path through the engine's own matrix
                n, nf = len(c["text_tokens"][b]), c["num_frames"][b] // 2
                x = matrix[b, :n + 1, :nf]
                assert path_cost(x, r.alignments) >= path_cost(x, [tuple(p) for p in ref["alignments"]]) - 1e-3
            diffs += list(np.abs(np.array(r.text_token_probs) - np.array(ref["text_token_probs"])))
    assert same >= 0.6 * total, (same, total)
    assert np.median(diffs) < 2e-3 and max(diffs) < 0.1, (np.median(diffs), max(diffs))
    w.close()


@gpu
@pytest.mark.parametrize("compute", ["float32", "int8"])
def test_detect_language_equals_the_reference(fixture, compute):
    w = Whisper(MODEL, compute_type=compute)
    tol = 2e-4 if compute == "float32" else 2e-2
    for c in fixture["models"]["model-" + compute]["detect_language"]:
        res = w.detect_language(inputs(c["seed"], c["batch"]))
        assert len(res) == c["batch"]
        for r, ref in zip(res, c["results"]):
            probs = [p for _, p in r]
            assert probs == sorted(probs, reverse=True)
            got, want = dict(r), dict(ref)
            assert set(got) == set(want)
            for lang in want:
                assert abs(got[lang] - want[lang]) <= tol, (lang, got[lang], want[lang])
    w.close()


@gpu
def test_generate_is_unchanged_by_align(fixture):
    w = Whisper(MODEL, compute_type="float32")
    x = inputs(500, 2)
    prompts = [[101, 102, 106, 110], [101, 103, 105, 110]]
    before = w.generate(x, prompts, beam_size=3, max_length=24, return_scores=True)
    c = fixture["models"]["model-float32"]["cases"][6]       # the longest texts: grows the decoder rows
    _align(w, c)
    w.detect_language(inputs(420, 3))
    after = w.generate(x, prompts, beam_size=3, max_length=24, return_scores=True)
    assert [r.sequences_ids for r in before] == [r.sequences_ids for r in after]
    assert [r.scores for r in before] == [r.scores for r in after]
    w.close()


@gpu
def test_align_of_a_larger_model_against_the_oracle(tmp_path):
    """A synthetic Whisper with 1500 encoder positions, 4 + 4 layers, 8 heads and 6 alignment heads across 3 layers; 10 entries
    whose decoder rows (up to 445 positions each) need two passes; variable frames up to 1500 (several CTAs per standardised
    row, median rows wider than a CTA).  float32: matrices to 1e-4 of the fp32 oracle, alignments identical, probabilities to
    1e-4.  float16: matrices to a float16 tolerance, its paths as good as the oracle's through the oracle's matrix."""
    from ctranslate2_b200.converters.synthetic import WhisperConfig, write_whisper_model
    cfg = WhisperConfig(encoder_layers=4, decoder_layers=4, num_heads=8, d_model=256, n_mels=80, max_source_positions=1500,
                        max_target_positions=448, text_tokens=500, languages=4, timestamps=20)
    mdir = str(tmp_path / "whisper_large")
    write_whisper_model(mdir, cfg, "float32", seed=9)
    heads = [[3, 1], [1, 4], [2, 0], [3, 6], [1, 0], [2, 7]]
    conf = json.load(open(os.path.join(mdir, "config.json")))
    conf["alignment_heads"] = heads
    json.dump(conf, open(os.path.join(mdir, "config.json"), "w"))
    rng = np.random.default_rng(3)
    lengths = (440, 40, 7, 90, 1, 200, 60, 15, 300, 120)
    x = (rng.standard_normal((len(lengths), 80, 3000)) * 2).astype(np.float32)
    texts = [[int(t) for t in rng.integers(0, 500, size=n)] for n in lengths]
    frames = [3000, 2400, 800, 3000, 150, 2999, 1000, 3000, 2000, 517]
    start = [500 + 1, 500 + 2, 500 + 7]
    ref, want = WhisperAlignOracle(mdir, compute_type="float32").align(x, start, texts, frames, 7)
    for compute in ("float32", "float16"):
        w = Whisper(mdir, compute_type=compute)
        res, matrix = w._align(x, start, texts, frames, 7, return_matrix=True)
        w.close()
        for b in range(len(lengths)):
            n, nf = len(texts[b]), frames[b] // 2
            got, x32 = matrix[b, :n + 1, :nf], want[b]
            assert np.isfinite(x32).all()
            if compute == "float32":
                err = np.abs(got - x32) / np.maximum(1.0, np.abs(x32))
                assert err.max() <= 1e-4, (b, float(err.max()))
                assert res[b].alignments == ref[b][0], b
                np.testing.assert_allclose(res[b].text_token_probs, ref[b][1], atol=1e-4, rtol=0)
            else:
                d16 = np.abs(got - x32)
                assert np.median(d16) < 0.05 and d16.max() < 1.0, (b, float(np.median(d16)), float(d16.max()))
                assert path_cost(x32, res[b].alignments) >= path_cost(x32, ref[b][0]) - 0.05 * (n + nf), b
                # float16 logits carry about 3 significant digits: relative error of a few percent on a probability
                np.testing.assert_allclose(res[b].text_token_probs, ref[b][1], rtol=0.05, atol=5e-3)
