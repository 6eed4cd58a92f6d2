#!/usr/bin/env python
"""tools/ref_cuda_worker.py — runs the UNMODIFIED reference's CUDA build (oracle/_ref_cuda, built by
oracle/Makefile.ref_cuda) on the GPU box, in its own process.  TEST / BENCH INFRASTRUCTURE: it is the GPU-side
oracle and the `ref_cuda` performance record; nothing under ctranslate2_b200/ imports it.

    python tools/ref_cuda_worker.py awq-golden OUT.npz            # GemmAwq / GemvAwq / DequantizeAwq outputs on seeded inputs
    python tools/ref_cuda_worker.py dense-s8 OUT.npz              # Quantize + cublasGemmEx(s8) + Dequantize on seeded inputs
    python tools/ref_cuda_worker.py model-golden OUT_DIR          # full-size Llama-3-8B INT8 logits / tokens, OPUS-shaped translations
    python tools/ref_cuda_worker.py forward MODEL_DIR COMPUTE IDS.npy OUT.npy [--flash]
    python tools/ref_cuda_worker.py generate MODEL_DIR COMPUTE PROMPTS.npy MAXLEN OUT.npy [--flash]
    python tools/ref_cuda_worker.py bench MODEL_DIR COMPUTE BATCH PROMPT_LEN G1 G2 [--flash]   # one JSON line
    python tools/ref_cuda_worker.py translate MODEL_DIR COMPUTE SOURCES.json BEAM NUM_HYP MAXLEN OUT.json
    python tools/ref_cuda_worker.py translate-bench MODEL_DIR COMPUTE SOURCES.json BEAM MAXLEN   # one JSON line

The seeded inputs of `awq-golden` are rebuilt by tests/test_gpu_awq.py::make_awq from (n, k, g, seed), so the fixture
holds only the reference's outputs.
"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import ct2_oracle as O   # noqa: E402
from oracle import refapi            # noqa: E402

AWQ_GEMM, AWQ_GEMV = 1, 2
# (m, n, k, g, seed): m <= 8 takes the reference's gemv kernel, m > 8 its gemv2 (split-K + Sum); GemmAwq covers all m
# (k / g >= 8 everywhere: the reference's gemv kernels read whole 32-bit words of 8 zero points per row, gemv_gpu.cu:305-307,
# 380-382; with fewer groups than that — k = 512, g = 128 — its own output is garbage / NaN)
AWQ_CASES = [(1, 256, 1024, 128, 11), (4, 256, 2048, 128, 12), (8, 384, 1024, 64, 13), (16, 256, 1024, 128, 14),
             (40, 384, 1024, 64, 15), (7, 1024, 4096, 128, 16), (32, 1024, 4096, 128, 17)]
DEQ_CASES = [(256, 512, 128, 21), (384, 1024, 64, 22)]


def make_awq(n, k, g, seed):
    """Same generator as tests/test_gpu_awq.py::make_awq."""
    r = np.random.default_rng(seed)
    w_int = r.integers(0, 16, size=(k, n))
    z_int = r.integers(0, 16, size=(k // g, n))
    scales = r.uniform(0.002, 0.02, size=(k // g, n)).astype(np.float16)
    return w_int, z_int, scales


def awq_x(m, k, seed):
    return np.random.default_rng(1000 + seed).standard_normal((m, k)).astype(np.float16)


def awq_golden(out):
    res, report = {}, []
    for (n, k, g, seed) in DEQ_CASES:
        w_int, z_int, scales = make_awq(n, k, g, seed)
        qw, qz = O.awq_pack_gemm(w_int, z_int)
        w = refapi.cuda_dequantize_awq(qw, scales, qz, g)
        mine = O.awq_dequantize_gemm(qw, scales, qz).astype(np.float16)
        report.append({"op": "DequantizeAwq", "n": n, "k": k, "g": g, "bit_exact_vs_oracle": bool(np.array_equal(w, mine)),
                       "max_abs_diff": float(np.abs(w.astype(np.float32) - mine.astype(np.float32)).max())})
        if n * k <= 256 * 512:
            res["deq_%d_%d_%d_%d" % (n, k, g, seed)] = w
    for (m, n, k, g, seed) in AWQ_CASES:
        w_int, z_int, scales = make_awq(n, k, g, seed)
        x = awq_x(m, k, seed)
        qw, qz = O.awq_pack_gemm(w_int, z_int)
        y = refapi.cuda_gemm_awq(x, qw, scales, qz, g)
        res["gemm_%d_%d_%d_%d_%d" % (m, n, k, g, seed)] = y
        qw2, qz2, sc2 = O.awq_pack_gemv(w_int.T.copy(), z_int.T.copy(), scales.T.copy(), g)
        y2 = refapi.cuda_gemv_awq(x, qw2, sc2, qz2)
        res["gemv_%d_%d_%d_%d_%d" % (m, n, k, g, seed)] = y2
        deq = (w_int - np.repeat(z_int, g, 0)).astype(np.float64) * np.repeat(scales.astype(np.float64), g, 0)
        truth = x.astype(np.float64) @ deq
        sc = np.abs(truth).max()
        report.append({"op": "GemmAwq/GemvAwq", "m": m, "n": n, "k": k, "g": g,
                       "gemm_max_err_over_max": float(np.abs(y - truth).max() / sc),
                       "gemv_max_err_over_max": float(np.abs(y2 - truth).max() / sc),
                       "oracle_gemm_vs_ref": float(np.abs(O.awq_gemm(x, qw, scales, qz) - y).max() / sc),
                       "oracle_gemv_vs_ref": float(np.abs(O.awq_gemv(x, qw2, sc2, qz2, g) - y2).max() / sc)})
    np.savez_compressed(out, **res)
    json.dump(report, open(os.path.splitext(out)[0] + "_report.json", "w"), indent=1)
    for r in report:
        print(json.dumps(r))


def dense_s8(out):
    res = {}
    for (m, n, k, seed) in [(1, 256, 512, 31), (32, 512, 1024, 32), (5, 1024, 4096, 33)]:
        r = np.random.default_rng(seed)
        x = r.standard_normal((m, k)).astype(np.float16)
        w = r.integers(-127, 128, size=(n, k)).astype(np.int8)
        ws = r.uniform(500, 4000, size=n).astype(np.float32)
        for act in (-1, 2):      # none, Swish (ops::ActivationType order: ReLU, GELUTanh, Swish, ...)
            res["y_%d_%d_%d_%d_%d" % (m, n, k, seed, act)] = refapi.cuda_dense_s8(x, w, ws, act)
    np.savez_compressed(out, **res)


# ---- whole-model fixtures (tests/golden/llama8b_int8_ref_cuda.npz, opus_small_ref_cuda.json): seeded inputs shared with
# tests/test_gpu_ref_cuda.py, which compares against what `model-golden` stored ----
LLAMA_VOCAB = 128256
LLAMA_SAMPLE_COLS = 512          # vocabulary columns of the reference logits that are stored (all 128256 would be 25 MB)
LLAMA_TOP = 8                    # plus the reference's top entries of every position (argmax and margin are exact)


def llama8b_inputs():
    r = np.random.default_rng(7)
    ids = r.integers(3, LLAMA_VOCAB, size=(2, 24)).astype(np.int32)
    prompts = r.integers(3, LLAMA_VOCAB, size=(4, 48)).astype(np.int32)
    cols = np.sort(np.random.default_rng(70).choice(LLAMA_VOCAB, LLAMA_SAMPLE_COLS, replace=False))
    return ids, prompts, cols


def opus_small(model_dir):
    """BASELINE.json configs[1] geometry with the vocabulary cut to 4000; returns the 16 source sentences."""
    from ctranslate2_b200.converters.synthetic import TransformerConfig, write_transformer_model
    cfg = TransformerConfig(source_vocab=4000, target_vocab=4000, pre_norm=False, activation=2, start_from_zero_embedding=True)
    write_transformer_model(model_dir, cfg, "int8", seed=3)
    r = np.random.default_rng(11)
    return [[int(x) for x in r.integers(3, 4000, size=int(r.integers(10, 50)))] for _ in range(16)]


def model_golden(out_dir):
    import tempfile
    import bench
    ids, prompts, cols = llama8b_inputs()
    g = open_generator(bench.model_dir("8b"), "int8_float16")
    logits = g.forward(ids)                                            # [2, 24, V] fp32
    top_idx = np.argsort(-logits, axis=-1, kind="stable")[..., :LLAMA_TOP].astype(np.int32)
    tokens, _ = g.generate_timed(prompts, 8, end_id=2)
    np.savez_compressed(os.path.join(out_dir, "llama8b_int8_ref_cuda.npz"), logits_cols=logits[..., cols].astype(np.float32),
                        top_idx=top_idx, top_val=np.take_along_axis(logits, top_idx, -1).astype(np.float32),
                        tokens=np.asarray(tokens, np.int32))
    del g
    with tempfile.TemporaryDirectory() as tmp:
        srcs = opus_small(os.path.join(tmp, "opus_small"))
        t = refapi.RefTranslator(os.path.join(tmp, "opus_small"), "float32", 0)
        res = t.translate(srcs, beam_size=4, num_hypotheses=2, max_length=24)
    json.dump([[[h[0], h[1]] for h in r] for r in res], open(os.path.join(out_dir, "opus_small_ref_cuda.json"), "w"))


def open_generator(model_dir, compute):
    return refapi.RefGenerator(model_dir, compute, 0)


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    flash = "--flash" in sys.argv
    task = args[0]
    if not refapi.cuda_available():
        print(json.dumps({"unavailable": "oracle/_ref_cuda is not built (make -f oracle/Makefile.ref_cuda)"}))
        return 3
    refapi.use_cuda(flash_attention=flash)
    if task == "awq-golden":
        awq_golden(args[1])
    elif task == "dense-s8":
        dense_s8(args[1])
    elif task == "model-golden":
        model_golden(args[1])
    elif task == "forward":
        g = open_generator(args[1], args[2])
        ids = np.load(args[3]).astype(np.int32)
        np.save(args[4], g.forward(ids))
    elif task == "generate":
        g = open_generator(args[1], args[2])
        prompts = np.load(args[3]).astype(np.int32)
        out, _ = g.generate_timed(prompts, int(args[4]), end_id=2)
        np.save(args[5], out)
    elif task == "bench":
        mdir, compute, B, P, G1, G2 = args[1], args[2], int(args[3]), int(args[4]), int(args[5]), int(args[6])
        t0 = time.time()
        g = open_generator(mdir, compute)
        load_s = time.time() - t0
        prompts = np.random.default_rng(42).integers(3, g.vocab, size=(B, P), dtype=np.int32)
        g.generate_timed(prompts, G1)                             # warm-up at the timed shapes (allocator pools, cuBLAS
        _, t1 = g.generate_timed(prompts, G1)                     # handles / heuristics, kernel loading)
        _, t2 = g.generate_timed(prompts, G2)
        dec = (t2 - t1) / max(1, G2 - G1)
        rec = {"impl": "reference-cuda", "flash_attention": flash, "compute_type": compute, "batch": B,
               "prompt_len": P, "generated": [G1, G2], "seconds": [round(t1, 4), round(t2, 4)],
               "decode_ms_per_step_by_difference": round(dec * 1e3, 4), "e2e_tokens_per_s": round(B * G2 / t2, 2),
               "load_seconds": round(load_s, 1)}
        # the decode step itself: slope of the per-step callback stamps of one run (the difference of two prompt-dominated
        # wall times above is only kept as a cross-check)
        stamps, t3 = g.generate_steps(prompts, G2)
        if (stamps >= 0).all() and G2 >= 8:
            lo = max(2, G2 // 8)
            dec = float(stamps[-1] - stamps[lo]) / (G2 - 1 - lo)
            rec["prefill_ms"] = round(float(stamps[0]) * 1e3, 2)
            rec["method"] = "per-step callback stamps, steps %d..%d" % (lo, G2 - 1)
        rec["decode_ms_per_step"] = round(dec * 1e3, 4)
        rec["decode_tokens_per_s"] = round(B / dec, 2)
        print(json.dumps(rec))
    elif task == "translate":
        t = refapi.RefTranslator(args[1], args[2], 0)
        srcs = json.load(open(args[3]))
        res = t.translate(srcs, beam_size=int(args[4]), num_hypotheses=int(args[5]), max_length=int(args[6]))
        json.dump([[[h[0], h[1]] for h in r] for r in res], open(args[7], "w"))
    elif task == "translate-bench":
        t = refapi.RefTranslator(args[1], args[2], 0)
        srcs = json.load(open(args[3]))
        beam, maxlen = int(args[4]), int(args[5])
        t.translate(srcs[:4], beam_size=beam, max_length=8)              # kernel loading, allocator pools
        t.translate(srcs, beam_size=beam, max_length=maxlen)             # warm-up at the timed shapes
        t0 = time.time()
        res = t.translate(srcs, beam_size=beam, max_length=maxlen)
        dt = time.time() - t0
        toks = sum(len(r[0][0]) for r in res)
        print(json.dumps({"impl": "reference-cuda", "compute_type": args[2], "batch": len(srcs), "beam_size": beam,
                          "max_decoding_length": maxlen, "target_tokens": toks, "seconds": round(dt, 4),
                          "tokens_per_s": round(toks / dt, 1)}))
    else:
        raise SystemExit("unknown task " + task)
    return 0


if __name__ == "__main__":
    sys.exit(main())
