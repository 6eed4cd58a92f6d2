"""-m gpu: the CUDA path against the UNMODIFIED reference's own CUDA build (cuBLAS GEMM, the reference's AWQ kernels, built for
sm_90 by oracle/Makefile.ref_cuda), through committed fixtures that tools/ref_cuda_worker.py wrote on an H100:

  * tests/golden/awq_ref_cuda.npz, dense_s8_ref_cuda.npz: outputs of the reference's GemmAwq / GemvAwq / DequantizeAwq kernels
    and of its INT8 Dense chain (Quantize -> cublasGemmEx -> Dequantize) on seeded inputs — this is what pins AWQ parity
    (the reference has no CPU implementation and no tests for AWQ);
  * tests/golden/llama8b_int8_ref_cuda.npz, opus_small_ref_cuda.json: BASELINE.json configs[2] at FULL size (Llama-3-8B
    geometry, INT8) — logits of the prompt pass and the first greedy tokens of the reference's `int8_float16` CUDA path — and
    the beam-4 translations of its CUDA Translator on an OPUS-MT-shaped model.  The models are rebuilt from their seeds.
"""
import json
import os
import sys

import numpy as np
import pytest
import torch

import ctranslate2_b200 as ct2
from ctranslate2_b200 import ops
from oracle import ct2_oracle as O
from gpu_util import dev, gpu, to_np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

sys.path.insert(0, os.path.join(ROOT, "tools"))
from ref_cuda_worker import AWQ_CASES, DEQ_CASES, awq_x, llama8b_inputs, make_awq, opus_small   # noqa: E402  (seeded input generators only)


def _fixture(name):
    p = os.path.join(GOLDEN, name)
    if not os.path.exists(p):
        pytest.skip("fixture %s not generated yet (tools/ref_cuda_worker.py on a GPU box)" % name)
    return np.load(p)


# fp16 outputs of two different summation orders (the reference: fp16 split-K partial planes + ops::Sum, or fp32 FMA per
# warp; ours: fp32 accumulation in the wgmma registers): the reference's own fp16 tolerance class (tests/ops_test.cc:1434-1445) on the
# scale of the output
def close_f16(got, ref, tol=1e-2):
    ref = ref.astype(np.float32)
    np.testing.assert_allclose(got, ref, rtol=tol, atol=tol * max(1e-3, np.abs(ref).max()))


@gpu
@pytest.mark.parametrize("case", AWQ_CASES, ids=lambda c: "m%d_n%d_k%d_g%d" % c[:4])
def test_dense_awq_vs_reference_cuda_kernels(case):
    fx = _fixture("awq_ref_cuda.npz")
    m, n, k, g, seed = case
    w_int, z_int, scales = make_awq(n, k, g, seed)
    x = awq_x(m, k, seed)
    key = "%d_%d_%d_%d_%d" % case
    qw, qz = O.awq_pack_gemm(w_int, z_int)
    y = to_np(ops.dense_awq(dev(x), ops.AwqWeight(dev(qw), dev(scales), dev(qz), ops.AWQ_GEMM, g)))
    close_f16(y, fx["gemm_" + key])                 # ops::GemmAwq (src/ops/awq/gemm_gpu.cu)
    qw2, qz2, sc2 = O.awq_pack_gemv(w_int.T.copy(), z_int.T.copy(), scales.T.copy(), g)
    y2 = to_np(ops.dense_awq(dev(x), ops.AwqWeight(dev(qw2), dev(sc2), dev(qz2), ops.AWQ_GEMV, g)))
    close_f16(y2, fx["gemv_" + key])                # ops::GemvAwq (src/ops/awq/gemv_gpu.cu: gemv m <= 8, gemv2 above)
    assert np.array_equal(y, y2)                    # both reference layouts repack to the same native weight


@gpu
def test_dequantize_awq_vs_reference_cuda_kernel():
    fx = _fixture("awq_ref_cuda.npz")
    n, k, g, seed = DEQ_CASES[0]
    w_int, z_int, scales = make_awq(n, k, g, seed)
    qw, qz = O.awq_pack_gemm(w_int, z_int)
    w = to_np(ops.dequantize_awq(dev(qw), dev(scales), dev(qz), ops.AWQ_GEMM, g))
    np.testing.assert_array_equal(w, fx["deq_%d_%d_%d_%d" % (n, k, g, seed)].astype(np.float32))    # bit-exact fp16


@gpu
def test_dense_int8_vs_reference_cuda_chain():
    """ours: one fused wgmma kernel; reference: quantize_kernel + cublasGemmEx(s8) + dequantize_gemm_output_kernel."""
    fx = _fixture("dense_s8_ref_cuda.npz")
    for key in fx.files:
        m, n, k, seed, act = [int(v) for v in key.split("_")[1:]]
        r = np.random.default_rng(seed)
        x = r.standard_normal((m, k)).astype(np.float16)
        w = r.integers(-127, 128, size=(n, k)).astype(np.int8)
        ws = r.uniform(500, 4000, size=n).astype(np.float32)
        xq, xs = ops.Quantize()(dev(x))
        y = to_np(ops.dense_int8(xq, xs, dev(w), dev(ws), activation_type=None if act < 0 else act, dtype=torch.float16))
        ref = fx[key].astype(np.float32)
        # same int32 accumulators, same fp32 scale product, __fdividef on both sides: at most one fp16 ulp apart
        np.testing.assert_allclose(y, ref, rtol=2e-3, atol=2e-3 * np.abs(ref).max())


@gpu
def test_llama8b_int8_full_size_vs_reference_cuda():
    """BASELINE.json configs[2] at full size: prompt-pass logits and greedy tokens vs the reference's CUDA int8_float16 path
    (llama8b_int8_ref_cuda.npz: its logits at 512 seeded vocabulary columns and its top 8 entries of every position)."""
    import bench
    fx = _fixture("llama8b_int8_ref_cuda.npz")
    ids, prompts, cols = llama8b_inputs()
    g = ct2.Generator(bench.model_dir("8b"), compute_type="int8_float16", max_batch_size=4, max_length=256)
    mine = g.forward_batch(ids.tolist())
    ref_cols, top_idx, top_val = fx["logits_cols"], fx["top_idx"], fx["top_val"]
    d_cols = mine[..., cols] - ref_cols
    d_top = np.take_along_axis(mine, top_idx.astype(np.int64), -1) - top_val
    rms = float(np.sqrt(np.mean(d_cols.astype(np.float64) ** 2)) / np.sqrt(np.mean(ref_cols.astype(np.float64) ** 2)))
    err = float(max(np.abs(d_cols).max(), np.abs(d_top).max()))
    # whole-model bound (32 layers of int8 activation rounding + fp16 GEMM accumulation on the reference side); the
    # bit-level claims are per op (test_gpu_ops.py)
    assert rms <= 8e-2, rms
    # greedy tokens: rows whose reference margin (top1 - top2) exceeds twice the observed logit error must agree
    margin = top_val[..., 0] - top_val[..., 1]
    decided = margin > 2 * err
    agree = mine.argmax(-1) == top_idx[..., 0]
    assert decided.any() and agree[decided].all()
    ref_tok = fx["tokens"]
    res = g.generate_batch(prompts.tolist(), max_length=8, min_length=8, end_token=[2])
    tok = np.array([x.sequences_ids[0] for x in res])
    print({"logits_rel_rms": rms, "logits_max_abs_err": err, "positions_decided": int(decided.sum()),
           "positions": int(decided.size), "argmax_agreement_all_positions": float(agree.mean()),
           "greedy_first_token_agreement": float((tok[:, 0] == ref_tok[:, 0]).mean()),
           "greedy_token_agreement_8": float((tok == ref_tok).mean())})


@gpu
def test_opus_mt_shape_translations_vs_reference_cuda(tmp_path):
    """BASELINE.json configs[1] geometry (Transformer-base 6+6, d 512, 8 heads, ffn 2048, post-norm / Swish / zero first
    embedding as converters/marian.py writes OPUS-MT; vocabulary cut to 4000 to keep the model small): beam-4 translations of
    16 sentences against those of the UNMODIFIED reference's CUDA Translator (opus_small_ref_cuda.json), float32 compute on
    both sides."""
    from ctranslate2_b200.translator import Translator
    p = os.path.join(GOLDEN, "opus_small_ref_cuda.json")
    if not os.path.exists(p):
        pytest.skip("fixture opus_small_ref_cuda.json not generated yet (tools/ref_cuda_worker.py on a GPU box)")
    ref = json.load(open(p))
    mdir = str(tmp_path / "opus_small")
    srcs = opus_small(mdir)
    t = Translator(mdir, compute_type="float32")
    ids, lens, scores = t.translate_ids(srcs, beam_size=4, num_hypotheses=2, max_decoding_length=24, start_id=1, end_token=[2])
    same = 0
    for b in range(len(srcs)):
        mine = ids[b, 0, :lens[b, 0]].tolist()
        same += mine == ref[b][0][0]
        if mine == ref[b][0][0]:
            assert abs(float(scores[b, 0]) - ref[b][0][1]) < 2e-3
    # random weights give near-uniform output distributions: a 1e-6 logit difference can reorder two candidates, so a
    # sentence or two may legitimately differ; a structural error would break all of them
    assert same >= len(srcs) - 2, {"sentences": len(srcs), "best_hypothesis_identical": same}
