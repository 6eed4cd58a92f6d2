"""-m "not gpu": the C-ABI library builds/loads and exports every symbol include/ct2b200.h declares;
host logic that needs no GPU (model-dir writer/reader round trip, error behaviour without a device)."""
import ctypes
import os

import numpy as np
import pytest

from ctranslate2_b200 import _lib


@pytest.fixture(scope="module")
def cdll():
    if not os.path.exists(_lib.LIB_PATH):
        from ctranslate2_b200.build import build
        build(verbose=False)
    return _lib.lib()


def test_exports_every_declared_symbol(cdll):
    names = _lib.declared_symbols()
    assert len(names) >= 30
    missing = [n for n in names if not hasattr(cdll, n)]
    assert not missing, missing


def test_version_and_no_cpu_fallback(cdll):
    assert b"sm_90a" in cdll.ct2b200_version()
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    # without a device every compute entry point must fail loudly (no CPU fallback)
    rc = cdll.ct2b200_quantize_rows(None, 1, ctypes.c_int64(1), ctypes.c_int64(8), 1, None, None, None)
    assert rc != 0 and b"no CPU fallback" in cdll.ct2b200_last_error()
    cfg = _lib.GeneratorConfig(0, 1, 1, 64, 0, 1, 0, 0)
    assert not cdll.ct2b200_generator_open(b"/nonexistent", ctypes.byref(cfg))


def test_synthetic_writer_matches_reference_layout(tmp_path):
    """Our model-dir writer vs the oracle's model.bin reader (format: model_spec.py:382-414)."""
    from ctranslate2_b200.converters.synthetic import LlamaConfig, write_llama_model
    from oracle.ct2_oracle import read_model_bin, quantize_weight
    cfg = LlamaConfig(num_layers=1, num_heads=2, num_heads_kv=1, head_dim=32, ffn_dim=96, vocab_size=50)
    d = str(tmp_path / "m")
    write_llama_model(d, cfg, "int8_float16", seed=3)
    spec, rev, v, _ = read_model_bin(os.path.join(d, "model.bin"))
    assert spec == "TransformerDecoderSpec" and rev == 8
    w = v["decoder/layer_0/self_attention/linear_0/weight"]
    assert w.dtype == np.int8 and w.shape == (128, 64)
    assert v["decoder/layer_0/self_attention/linear_0/weight_scale"].dtype == np.float32
    assert v["decoder/layer_0/ffn/layer_norm/gamma"].dtype == np.float16
    assert int(v["decoder/layer_0/self_attention/num_heads_kv"]) == 1
    assert np.abs(w).max(axis=1).min() == 127   # every quantized row attains +-127
    # converter-side quantization formula == oracle restatement of model.cc:304-369
    wf = np.random.default_rng(0).standard_normal((7, 33)).astype(np.float32)
    from ctranslate2_b200.converters.synthetic import quantize_int8
    q1, s1 = quantize_int8(wf)
    q2, s2 = quantize_weight(wf)
    np.testing.assert_array_equal(q1, q2)
    np.testing.assert_array_equal(s1, s2)


def test_generator_argument_errors():
    from ctranslate2_b200 import Generator
    with pytest.raises(ValueError):
        Generator("/nonexistent", device="cpu")
    with pytest.raises(ValueError):
        Generator("/nonexistent", compute_type="int4")
