#!/usr/bin/env python
"""Translator.score_batch on the encoder-decoder workload of bench.py: the OPUS-MT-shaped Transformer-base model
(bench.seq2seq_model_dir(), INT8 weights, int8_float16), 64 (source, target) pairs whose sources and targets hold U[10,50]
tokens, drawn from a fixed seed.  Prints one JSON line with

  * score_ms: host clock around score_batch (the call ends with a device synchronise), median of --repeats after a warm-up;
  * score_tokens_per_s: scored target tokens (every target token and </s>) / score_ms;
  * encode_ms: for context, Translator.bench's device-timed encoder pass (encoder + memory projections) of 64 x 51 tokens;
  * ref_cuda: the reference's CUDA build on the same pairs, or why it is unavailable: oracle/_ref_cuda is not built, or its
    C-ABI driver (oracle/ref_driver.cc) has no scoring entry to call;
  * the card's name and power limit, read in the same run.

usage: python tools/translate_score_bench.py [--pairs 64] [--repeats 5]"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from score_bench import card  # noqa: E402


def ref_cuda_record():
    driver = os.path.join(ROOT, "oracle", "_ref_cuda", "libct2ref_cuda_driver.so")
    if not os.path.exists(driver):
        return {"unavailable": "oracle/_ref_cuda is not built (make -f oracle/Makefile.ref_cuda)"}
    import ctypes
    if not hasattr(ctypes.CDLL(driver), "ref_translate_score"):
        return {"unavailable": "the reference's CUDA driver (oracle/ref_driver.cc) exposes no Translator::score_batch entry"}
    return {"unavailable": "no timing task for the reference's Translator::score_batch in tools/ref_cuda_worker.py"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    import numpy as np
    from ctranslate2_b200.translator import Translator
    mdir = bench.seq2seq_model_dir()
    rng = np.random.default_rng(7)
    V = 58101
    srcs = [[int(x) for x in rng.integers(3, V, size=int(rng.integers(10, 51)))] + [2] for _ in range(a.pairs)]
    tgts = [[int(x) for x in rng.integers(3, V, size=int(rng.integers(10, 51)))] for _ in range(a.pairs)]
    t = Translator(mdir, compute_type="int8_float16")
    res = t.score_batch(srcs, tgts)                                # warm-up: arena growth, slab allocation, first launches
    scored = sum(len(r.log_probs) for r in res)
    assert scored == sum(len(x) + 1 for x in tgts)
    assert all(np.isfinite(r.log_probs).all() for r in res)
    times = []
    for _ in range(a.repeats):
        t0 = time.perf_counter()
        t.score_batch(srcs, tgts)
        times.append((time.perf_counter() - t0) * 1e3)
    enc = [t.bench(a.pairs, 51, 1, 1, 0)[0] for _ in range(a.repeats)]
    score_ms, encode_ms = statistics.median(times), statistics.median(enc)
    rec = {"workload": "Translator.score_batch OPUS-MT-shaped Transformer-base INT8 (int8_float16), %d pairs, sources and "
                       "targets U[10,50] tokens" % a.pairs,
           "score_ms": round(score_ms, 2), "score_ms_min_max": [round(min(times), 2), round(max(times), 2)],
           "scored_tokens": scored, "score_tokens_per_s": round(scored / (score_ms * 1e-3), 1),
           "encode_ms": round(encode_ms, 3), "encode_ms_min_max": [round(min(enc), 3), round(max(enc), 3)],
           "repeats": a.repeats,
           "ref_cuda": ref_cuda_record()}
    rec.update(card())
    t.close()
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
