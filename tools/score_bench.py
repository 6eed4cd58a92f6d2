#!/usr/bin/env python
"""Generator.score_batch on the full-size workload: Llama-3-8B geometry, INT8 weights, int8_float16, 32 sequences x 1024
tokens.  Prints one JSON line with

  * score_ms: host clock around score_batch (the call ends with a device synchronise), median of --repeats after a warm-up;
  * score_tokens_per_s: scored tokens (32 x 1023) / score_ms;
  * prefill_ms: the device-timed prompt pass of the same tokens (bench_decode's prefill_ms, prompt_len 1025 = 1024 positions
    per row), median of --repeats;
  * ratio_to_prefill: score_ms / prefill_ms — what the lm_head, the LogSoftMax + Gather and the host round trip add;
  * the card's name and power limit, read in the same run.

usage: python tools/score_bench.py [--batch 32] [--tokens 1024] [--repeats 5]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402


def card():
    import torch
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        info["power_limit_w"] = float(q[0])
        info["sm_max_mhz"] = float(q[1])
    except Exception as e:           # the number is still reported, without the limit
        info["power_limit_w"] = "unavailable (%s)" % type(e).__name__
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--tokens", type=int, default=1024)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    import ctranslate2_b200 as ct2
    B, L = a.batch, a.tokens
    g = ct2.Generator(bench.model_dir("8b"), compute_type="int8_float16", max_batch_size=B, max_length=L + 16)
    seqs = bench.prompts_for("8b", B, L).tolist()
    res = g.score_batch(seqs, max_input_length=0)                  # warm-up: slab allocation, first-use kernel set-up
    scored = sum(len(r.log_probs) for r in res)
    assert scored == B * (L - 1)
    times = []
    for _ in range(a.repeats):
        t0 = time.perf_counter()
        g.score_batch(seqs, max_input_length=0)
        times.append((time.perf_counter() - t0) * 1e3)
    pre = [g.bench_decode(B, L + 1, 1, 0)[0] for _ in range(a.repeats)]
    score_ms, prefill_ms = statistics.median(times), statistics.median(pre)
    rec = {"workload": "score_batch %s int8_float16, %d x %d tokens" % (bench.NAMES["8b"], B, L),
           "score_ms": round(score_ms, 2), "score_ms_min_max": [round(min(times), 2), round(max(times), 2)],
           "score_tokens_per_s": round(scored / (score_ms * 1e-3), 1),
           "prefill_ms": round(prefill_ms, 2), "prefill_ms_min_max": [round(min(pre), 2), round(max(pre), 2)],
           "ratio_to_prefill": round(score_ms / prefill_ms, 3), "repeats": a.repeats}
    rec.update(card())
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
