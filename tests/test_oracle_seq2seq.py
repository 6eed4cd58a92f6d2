"""Encoder-decoder restatement (SURVEY §8 f1: Translator::translate_batch) pinned against the unmodified reference.

The golden case is the reference's own tests/translator_test.cc:53-96 (aren-transliteration-i8: "آ ت ز م و ن" ->
"a t z m o n"), on the committed copy of its model (tests/golden/aren-transliteration-i8).  They run where the reference has
been compiled (oracle/_ref) and skip elsewhere.  Nothing here touches the product.
"""
import os
import struct

import numpy as np
import pytest

from oracle import ct2_oracle as O
from oracle import refapi

MODEL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "aren-transliteration-i8")
needs_reference = pytest.mark.skipif(not refapi.available(), reason="needs oracle/_ref")


def _vocab(name):
    with open(os.path.join(MODEL, name), encoding="utf-8") as f:
        return [line.rstrip("\n") for line in f]


def _random_sources(seed, cases):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(cases):
        batch = int(rng.integers(1, 4))
        out.append([[int(x) for x in rng.integers(4, 51, size=int(rng.integers(2, 9)))] for _ in range(batch)])
    return out


def test_sinusoidal_positions_and_layer_norm_shapes():
    pos = O.sinusoidal_position_encoding(7, 32)
    assert pos.shape == (7, 32)
    # position 0 is encoded as time 1 (common.cc:213): sin(1 * timescale_0) with timescale_0 = 1
    np.testing.assert_allclose(pos[0, 0], np.sin(np.float32(1)), rtol=1e-6)
    np.testing.assert_allclose(pos[0, 16], np.cos(np.float32(1)), rtol=1e-6)
    x = np.random.default_rng(0).standard_normal((3, 32)).astype(np.float32)
    y = O.layer_norm(x, np.ones(32, np.float32), np.zeros(32, np.float32))
    np.testing.assert_allclose(y.mean(-1), 0, atol=1e-6)
    np.testing.assert_allclose(y.var(-1), 1, atol=1e-3)


@needs_reference
def test_layer_norm_matches_reference_op():
    rng = np.random.default_rng(1)
    x = (rng.standard_normal((9, 48)) * 3 + 1).astype(np.float32)
    g, b = rng.standard_normal(48).astype(np.float32), rng.standard_normal(48).astype(np.float32)
    np.testing.assert_allclose(O.layer_norm(x, g, b, 1e-5), refapi.layer_norm(g, b, x, 1e-5), atol=2e-6)


@needs_reference
def test_golden_transliteration_int8():
    """tests/translator_test.cc:53-96 with the model's native int8 weights (binary version 2: the activation quantizer
    truncates, include/ctranslate2/models/model.h:87-89)."""
    src, tgt = _vocab("source_vocabulary.txt"), _vocab("target_vocabulary.txt")
    ids = [src.index(w) for w in ["آ", "ت", "ز", "م", "و", "ن"]]
    oracle = O.Seq2SeqOracle.from_dir(MODEL)
    assert not oracle.round_before_cast
    hyps = oracle.translate([ids], beam_size=2, num_hypotheses=2, max_length=20)[0]
    assert [tgt[i] for i in hyps[0][0]] == ["a", "t", "z", "m", "o", "n"]
    ref = refapi.RefTranslator(MODEL, "int8").translate([ids], beam_size=2, num_hypotheses=2, max_length=20)[0]
    assert [h[0] for h in hyps] == [h[0] for h in ref]
    # int8 activations: the score carries the quantization noise of a d=32 model, not fp32 round-off
    np.testing.assert_allclose([h[1] for h in hyps], [h[1] for h in ref], atol=5e-3)


@needs_reference
@pytest.mark.parametrize("beam,num_hyp,length_penalty", [(1, 1, 1.0), (2, 2, 1.0), (4, 2, 0.0), (3, 3, 0.6)])
def test_float32_translations_match_reference(beam, num_hyp, length_penalty):
    """compute_type float32 removes activation quantization, so every token and score must agree: encoder, cross-attention
    decoder, ragged batches, and BeamSearch::search (decoding.cc:402-760) through the Translator defaults."""
    oracle = O.Seq2SeqOracle.from_dir(MODEL, compute_type="float32")
    ref = refapi.RefTranslator(MODEL, "float32")
    hyps = 0
    for srcs in _random_sources(0, 10):
        got = oracle.translate(srcs, beam_size=beam, num_hypotheses=num_hyp, max_length=16, length_penalty=length_penalty)
        want = ref.translate(srcs, beam_size=beam, num_hypotheses=num_hyp, max_length=16, length_penalty=length_penalty)
        for g, w in zip(got, want):
            assert [h[0] for h in g] == [h[0] for h in w]
            np.testing.assert_allclose([h[1] for h in g], [h[1] for h in w], atol=1e-4)
            hyps += len(g)
    assert hyps >= 10 * num_hyp


@needs_reference
@pytest.mark.parametrize("variant", ["aren-transliteration", "aren-transliteration-i16", "aren-transliteration-i8"])
def test_model_variants_translate_the_golden_sentence(variant):
    """tests/translator_test.cc:53-96 (ModelVariantTest): the float32, int16 and int8 storage variants of the toy model all
    translate the golden sentence to "a t z m o n"; computed in float32 the oracle agrees with the reference on every
    hypothesis of a few random batches as well."""
    model = os.path.join(os.path.dirname(MODEL), variant)
    src, tgt = _vocab("source_vocabulary.txt"), _vocab("target_vocabulary.txt")
    ids = [src.index(w) for w in ["آ", "ت", "ز", "م", "و", "ن"]]
    oracle = O.Seq2SeqOracle.from_dir(model, compute_type="float32")
    ref = refapi.RefTranslator(model, "float32")
    assert [tgt[i] for i in oracle.translate([ids], beam_size=2)[0][0][0]] == ["a", "t", "z", "m", "o", "n"]
    for srcs in [[ids]] + _random_sources(3, 4):
        got = oracle.translate(srcs, beam_size=2, num_hypotheses=2, max_length=16)
        want = ref.translate(srcs, beam_size=2, num_hypotheses=2, max_length=16)
        for g, w in zip(got, want):
            assert [h[0] for h in g] == [h[0] for h in w]
            np.testing.assert_allclose([h[1] for h in g], [h[1] for h in w], atol=1e-4)


@needs_reference
def test_float32_min_length_and_encoder_memory():
    oracle = O.Seq2SeqOracle.from_dir(MODEL, compute_type="float32")
    ref = refapi.RefTranslator(MODEL, "float32")
    srcs = [[31, 10, 19, 13, 5, 7, 9], [38, 43, 12, 8]]
    memory, lengths = ref.encode(srcs)
    d = oracle.d
    memory = memory.reshape(-1)[:2 * 7 * d].reshape(2, 7, d)
    padded = np.zeros((2, 7), np.int64)
    padded[0], padded[1, :4] = srcs[0], srcs[1]
    mine = oracle.encode(padded, np.array([7, 4]))
    np.testing.assert_allclose(mine[0], memory[0], atol=2e-5)
    np.testing.assert_allclose(mine[1, :4], memory[1, :4], atol=2e-5)
    got = oracle.translate(srcs, beam_size=2, num_hypotheses=1, max_length=12, min_length=9)
    want = ref.translate(srcs, beam_size=2, num_hypotheses=1, max_length=12, min_length=9)
    assert [h[0][0] for h in got] == [h[0][0] for h in want]
    assert all(len(h[0][0]) >= 9 for h in got)


def _rewrite_binary_version_5(dst):
    """The same variables in a version-5 container: from version 5 on the activation quantizer rounds to nearest, which
    is the arithmetic of every model the converters write today."""
    spec, revision, variables, _ = O.read_model_bin(os.path.join(MODEL, "model.bin"))
    type_ids = {np.dtype(np.float32): 0, np.dtype(np.int8): 1, np.dtype(np.int16): 2, np.dtype(np.int32): 3}
    os.makedirs(dst, exist_ok=True)
    with open(os.path.join(dst, "model.bin"), "wb") as f:
        def put_string(s):
            raw = s.encode() + b"\0"
            f.write(struct.pack("H", len(raw)) + raw)
        f.write(struct.pack("I", 5))
        put_string(spec)
        f.write(struct.pack("II", revision, len(variables)))
        for name, a in variables.items():
            put_string(name)
            f.write(struct.pack("B", a.ndim))
            f.write(struct.pack("%dI" % a.ndim, *a.shape))
            f.write(struct.pack("B", type_ids[a.dtype]) + struct.pack("I", a.nbytes) + a.tobytes())
        f.write(struct.pack("I", 0))
    for name in ("source_vocabulary.txt", "target_vocabulary.txt"):
        with open(os.path.join(MODEL, name), "rb") as src, open(os.path.join(dst, name), "wb") as out:
            out.write(src.read())
    return dst


@needs_reference
def test_int8_rounding_quantizer_statistics(tmp_path):
    """INT8 compute: a d=32 model amplifies a single rounding flip (an activation within an ulp of k + 0.5, reached by a
    different fp32 summation order) to ~1e-2 in the output, so bit parity per sentence is not defined.  Most sentences
    have no flip and must agree to fp32 round-off; all must stay within the flip noise."""
    model = _rewrite_binary_version_5(str(tmp_path / "v5"))
    oracle = O.Seq2SeqOracle.from_dir(model)
    assert oracle.round_before_cast
    ref = refapi.RefTranslator(model, "int8")
    errs = []
    for srcs in _random_sources(2, 12):
        for row in srcs:
            memory, _ = ref.encode([row])
            memory = memory.reshape(-1)[:len(row) * oracle.d].reshape(len(row), oracle.d)
            mine = oracle.encode(np.array([row]), np.array([len(row)]))[0]
            errs.append(float(np.abs(mine - memory).max()))
    errs = np.array(errs)
    assert np.median(errs) < 5e-6, errs
    assert (errs < 5e-6).mean() >= 0.6, errs
    assert errs.max() < 0.1, errs
