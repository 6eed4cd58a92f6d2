#!/usr/bin/env python
"""Translator.translate_batch with the alignment attention on the encoder-decoder workload of bench.py: the OPUS-MT-shaped
Transformer-base model (bench.seq2seq_model_dir(), INT8 weights, int8_float16), 32 sources of U[10,50] tokens drawn from a
fixed seed (token strings; the model adds </s>), beam 4, and a fixed number of decoding steps (min_decoding_length =
max_decoding_length = --steps), so every arm decodes the same number of steps whatever it translates.  Arms: off,
return_attention, coverage_penalty 0.2 and replace_unknowns.  The arms alternate within each round.  Prints one JSON line
with, per arm,

  * call_ms: host clock around translate_batch (the call ends with a device synchronise), median of --repeats after a
    warm-up, with its min / max;
  * ms_per_step: call_ms / steps (the call's encoder pass, about 1 % of it, included);

and the card's name and power limit, read in the same run.

usage: python tools/translate_attention_bench.py [--sources 32] [--beam 4] [--steps 256] [--repeats 5]"""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sources", type=int, default=32)
    ap.add_argument("--beam", type=int, default=4)
    ap.add_argument("--steps", type=int, default=256)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    import numpy as np
    from ctranslate2_b200.translator import Translator
    mdir = bench.seq2seq_model_dir()
    t = Translator(mdir, compute_type="int8_float16")
    V = t.info()["target_vocab"]
    rng = np.random.default_rng(7)
    srcs = [[t._source[int(x)] for x in rng.integers(3, V, size=int(rng.integers(10, 51)))] for _ in range(a.sources)]
    arms = {"off": {}, "return_attention": dict(return_attention=True), "coverage_penalty_0.2": dict(coverage_penalty=0.2),
            "replace_unknowns": dict(replace_unknowns=True)}
    kw = dict(beam_size=a.beam, max_decoding_length=a.steps, min_decoding_length=a.steps)
    times = {k: [] for k in arms}
    for k, o in arms.items():                                     # warm-up: arena growth, graph capture, first launches
        res = t.translate_batch(srcs, **kw, **o)
        assert all(len(r.hypotheses[0]) >= a.steps - 1 for r in res)
    for _ in range(a.repeats):
        for k, o in arms.items():
            t0 = time.perf_counter()
            t.translate_batch(srcs, **kw, **o)
            times[k].append((time.perf_counter() - t0) * 1e3)
    rec = {"workload": "Translator.translate_batch OPUS-MT-shaped Transformer-base INT8 (int8_float16), %d sources of "
                       "U[10,50] tokens, beam %d, %d decoding steps" % (a.sources, a.beam, a.steps),
           "repeats": a.repeats, "arms": {}}
    for k, v in times.items():
        med = statistics.median(v)
        rec["arms"][k] = {"call_ms": round(med, 2), "call_ms_min_max": [round(min(v), 2), round(max(v), 2)],
                          "ms_per_step": round(med / a.steps, 4)}
    rec.update(card())
    t.close()
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
