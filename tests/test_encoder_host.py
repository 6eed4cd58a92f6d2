"""Encoder-only models without a device: the numpy oracle against the reference's Encoder::forward_batch
(tests/golden/encoder_ref.npz, written by tools/make_golden.py --encoder-only), what the loader reads from and refuses in a
TransformerEncoderSpec directory (host-only ct2b200_encoder_summary), and the Python side of Encoder.forward_batch over a
recording fake of the C-ABI (argument checks before any call, padding, re-batching longest first, request order)."""
import ctypes
import json
import os

import numpy as np
import pytest

import ctranslate2_b200.encoder as E
from ctranslate2_b200.converters.synthetic import EncoderConfig, ModelWriter, write_encoder_model
from encoder_oracle import EncoderOracle, load_fixture
from oracle import ct2_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIXTURE = load_fixture(os.path.join(GOLDEN, "encoder_ref.npz"))


def _batch(case):
    ids = case["ids"]
    lens = np.array([len(r) for r in ids])
    a = np.zeros((len(ids), lens.max()), np.int64)
    t = None if case["token_type_ids"] is None else np.zeros_like(a)
    for b, r in enumerate(ids):
        a[b, :len(r)] = r
        if t is not None:
            t[b, :len(r)] = case["token_type_ids"][b]
    return a, lens, t


def _errors(name, case):
    o = EncoderOracle.from_dir(os.path.join(GOLDEN, name), compute_type=case["compute_type"])
    a, lens, t = _batch(case)
    h, p = o.forward(a, lens, t)
    errs = [float(np.abs(h[b, :lens[b]].reshape(-1) - np.array(case["last_hidden_state"][b])).max()) for b in range(len(lens))]
    assert (p is None) == (case["pooler_output"] is None)
    if p is not None:
        errs.append(float(np.abs(p - np.array(case["pooler_output"])).max()))
    return errs


CASES = [(name, i) for name, m in FIXTURE.items() for i in range(len(m))]


def test_fixture_covers_what_it_claims():
    cases = [c for m in FIXTURE.values() for c in m]
    assert {c["compute_type"] for c in cases} == {"float32", "int8"}
    assert any(c["token_type_ids"] is not None for c in cases) and any(c["token_type_ids"] is None for c in cases)
    assert any(c["pooler_output"] is None for c in cases)
    for c in cases:
        assert 1 in [len(r) for r in c["ids"]] and 16 in [len(r) for r in c["ids"]]      # 16 = the position table
    assert E.encoder_summary(os.path.join(GOLDEN, "tiny_encoder_prenorm"))["pre_norm"] is True


@pytest.mark.parametrize("name,i", [c for c in CASES if FIXTURE[c[0]][c[1]]["compute_type"] == "float32"])
def test_oracle_matches_the_reference_float32(name, i):
    assert max(_errors(name, FIXTURE[name][i])) < 1e-5


def test_oracle_matches_the_reference_int8_statistically():
    """INT8 compute: a rounding flip of one activation (a value within an ulp of k + 0.5 reached by another fp32 summation
    order) moves a d=64 model's outputs by ~1e-2, so only most rows must agree to fp32 round-off (as DESIGN §2 pins the
    seq2seq INT8 oracle)."""
    errs = np.array([e for name, i in CASES if FIXTURE[name][i]["compute_type"] == "int8"
                     for e in _errors(name, FIXTURE[name][i])])
    assert np.median(errs) < 5e-6, errs
    assert (errs < 5e-6).mean() >= 0.6, errs
    assert errs.max() < 0.1, errs


# ---------------- loader: summary and refusals ----------------
def _write(tmp_path, name="m", **kw):
    cfg = EncoderConfig(num_layers=1, num_heads=2, d_model=64, ffn_dim=128, vocab_size=40, max_positions=16, **kw)
    path = str(tmp_path / name)
    write_encoder_model(path, cfg, "int8")
    return path


def _rewrite(src, dst, drop=(), add=None, spec="TransformerEncoderSpec"):
    """Copy of a model directory with variables removed / added."""
    _, _, variables, _ = O.read_model_bin(os.path.join(src, "model.bin"))
    w = ModelWriter(dst, spec=spec, revision=1)
    for k, v in variables.items():
        if k not in drop and k not in (add or {}):
            w.add(k, v)
    for k, v in (add or {}).items():
        w.add(k, v)
    w.close(json.load(open(os.path.join(src, "config.json"))), json.load(open(os.path.join(src, "vocabulary.json"))))
    return dst


@pytest.mark.parametrize("kw,expect", [
    ({}, dict(type_vocab_size=2, pre_norm=False, activation=3, layernorm_embedding=True, final_norm=False, pooler=True)),
    (dict(type_vocab_size=0), dict(type_vocab_size=0, pooler=True)),
    (dict(pooler=False), dict(pooler=False)),
    (dict(pre_norm=True, activation=0, layernorm_embedding=False), dict(pre_norm=True, activation=0, final_norm=True,
                                                                       layernorm_embedding=False)),
    (dict(activation=1), dict(activation=1)),
])
def test_summary_of_each_written_variant(tmp_path, kw, expect):
    s = E.encoder_summary(_write(tmp_path, **kw))
    assert s["spec"] == "TransformerEncoderSpec" and s["weights"] == "int8"
    assert (s["num_layers"], s["num_heads"], s["head_dim"], s["d_model"], s["ffn_dim"]) == (1, 2, 32, 64, 128)
    assert (s["vocab_size"], s["max_positions"], s["embeddings_scale"], s["pooler_activation"]) == (40, 16, 0, 5)
    assert s["layer_norm_epsilon"] == pytest.approx(1e-12)
    for k, v in expect.items():
        assert s[k] == v, k


@pytest.mark.parametrize("change,message", [
    (dict(add={"encoder/embeddings_merge": np.int8(0)}), "CONCAT"),
    (dict(add={"encoder/layer_0/self_attention/relative_position_keys": np.zeros((5, 32), np.float32)}), "relative position"),
    (dict(add={"encoder/layer_0/self_attention/relative_attention_bias": np.zeros((8, 2), np.float32)}), "relative attention"),
    (dict(add={"encoder/layer_0/self_attention/rotary_dim": np.int32(0)}), "rotary"),
    (dict(add={"encoder/layer_0/self_attention/num_heads_kv": np.int32(1)}), "multi-query"),
    (dict(add={"encoder/layer_0/ffn/linear_0_noact/weight": np.zeros((128, 64), np.float32)}), "gated"),
    (dict(add={"encoder/activation": np.int8(2)}), "activation"),
    (dict(drop=("encoder/position_encodings/encodings",)), "position encodings"),
    (dict(drop=("encoder/layer_0/self_attention/layer_norm/beta",)), "RMSNorm"),
    (dict(add={"encoder/embeddings_2/weight": np.zeros((3, 64), np.float32)}), "more than two"),
    (dict(spec="TransformerDecoderSpec"), "TransformerEncoderSpec"),
])
def test_unsupported_spec_features_are_refused(tmp_path, change, message):
    path = _rewrite(_write(tmp_path), str(tmp_path / "changed"), **change)
    with pytest.raises(ValueError, match=message):
        E.encoder_summary(path)


def test_the_translator_refuses_encoder_models():
    from ctranslate2_b200.translator import translator_summary
    with pytest.raises(ValueError, match="encoder-decoder"):
        translator_summary(os.path.join(GOLDEN, "tiny_encoder"))


# ---------------- Python side over a recording fake ----------------
def _i32(ptr, n):
    return np.ctypeslib.as_array((ctypes.c_int32 * n).from_address(ptr.value))


def _f32(ptr, n):
    return np.ctypeslib.as_array((ctypes.c_float * n).from_address(ptr.value))


class FakeLib:
    """ct2b200_encoder_forward: hidden[b, t, :] = ids[b, t] + 1000 * types[b, t], pooled[b, :] = lengths[b]."""

    def __init__(self, d):
        self.d, self.calls = d, []

    def ct2b200_encoder_forward(self, h, ids, lens, types, B, T, hidden, pooled):
        B, T, d = B.value, T.value, self.d
        ids_a = _i32(ids, B * T).reshape(B, T).copy()
        lens_a = _i32(lens, B).copy()
        types_a = None if types is None else _i32(types, B * T).reshape(B, T).copy()
        self.calls.append((ids_a, lens_a, types_a))
        out = _f32(hidden, B * T * d).reshape(B, T, d)
        out[:] = (ids_a + (0 if types_a is None else 1000 * types_a))[..., None]
        if pooled is not None:
            _f32(pooled, B * d).reshape(B, d)[:] = lens_a[:, None]
        return 0

    def ct2b200_last_error(self):
        return b""


@pytest.fixture
def enc(monkeypatch):
    fake = FakeLib(4)
    monkeypatch.setattr(E, "lib", lambda: fake)
    e = object.__new__(E.Encoder)
    e._h, e.max_batch_size = 1, 4
    e._info = dict(d_model=4, vocab_size=100, type_vocab_size=2, max_positions=16, pooler=True)
    e._vocab = ["[PAD]", "[UNK]"] + ["w%d" % i for i in range(2, 100)]
    e._to_id = {t: i for i, t in enumerate(e._vocab)}
    e._config = {"unk_token": "[UNK]"}
    yield e, fake
    e._h = None


def test_requests_larger_than_the_arena_are_rebatched_longest_first_and_answered_in_order(enc):
    e, fake = enc
    r = np.random.default_rng(0)
    rows = [r.integers(2, 100, size=int(n)).tolist() for n in r.integers(1, 17, size=11)]
    types = [r.integers(0, 2, size=len(x)).tolist() for x in rows]
    out = e.forward_batch(rows, token_type_ids=types)
    assert [len(c[1]) for c in fake.calls] == [4, 4, 3]
    assert [int(n) for c in fake.calls for n in c[1]] == sorted((len(x) for x in rows), reverse=True)
    T = max(len(x) for x in rows)
    assert out.last_hidden_state.shape == (11, T, 4) and out.pooler_output.shape == (11, 4)
    for b, (x, t) in enumerate(zip(rows, types)):
        assert (out.last_hidden_state[b, :len(x), 0] == np.array(x) + 1000 * np.array(t)).all()
        assert (out.pooler_output[b] == len(x)).all()
    for ids, lens, tt in fake.calls:
        for b in range(len(lens)):
            assert (ids[b, lens[b]:] == 0).all() and (tt[b, lens[b]:] == 0).all()


def test_token_strings_dense_arrays_and_no_types(enc):
    e, fake = enc
    out = e.forward_batch([["w5", "nope", "w7"], ["w9"]])
    assert fake.calls[-1][2] is None                                          # no types: the engine's zeros
    assert out.last_hidden_state[0, :, 0].tolist() == [5, 1, 7] and out.last_hidden_state[1, 0, 0] == 9
    ids = np.array([[5, 6, 7], [8, 0, 0]], np.int64)
    out = e.forward_batch(ids, lengths=np.array([3, 1]))
    assert fake.calls[-1][1].tolist() == [3, 1] and out.last_hidden_state[1, 0, 0] == 8


@pytest.mark.parametrize("args,kw", [
    (([[5, 100]],), {}),                                          # id outside the vocabulary
    (([[5, -1]],), {}),
    (([[5], []],), {}),                                           # a length of 0
    (([[5] * 17],), {}),                                          # longer than the position table
    (([[5, 6]],), dict(token_type_ids=[[0, 2]])),                 # token type outside [0, 2)
    (([[5, 6]],), dict(token_type_ids=[[0]])),                    # too few types
    (([[5, 6], [7]],), dict(token_type_ids=[[0, 1]])),            # a types row missing
    ((np.array([[5, 6]]),), {}),                                  # dense ids need lengths
    ((np.array([[5, 6]]),), dict(lengths=np.array([3]))),         # length wider than the array
    ((np.array([[5, 6]]),), dict(lengths=np.array([2, 1]))),      # lengths of another batch size
    (([[5, 6.5]],), {}),                                          # not ids
    (([],), {}),
])
def test_argument_checks_happen_before_any_call(enc, args, kw):
    e, fake = enc
    with pytest.raises(ValueError):
        e.forward_batch(*args, **kw)
    assert fake.calls == []


def test_types_for_a_model_without_token_types_are_refused(enc):
    e, fake = enc
    e._info["type_vocab_size"] = 0
    with pytest.raises(ValueError, match="token-type"):
        e.forward_batch([[5]], token_type_ids=[[0]])
    assert fake.calls == []
