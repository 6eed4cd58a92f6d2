#!/usr/bin/env python
"""Whisper.generate with random sampling against the beam search it replaces in a temperature fallback, on the
Whisper-small-shaped synthetic model of tools/whisper_align_bench.py (int8_float16), 8 windows of 3000 input frames.  The prompt
is <|startoftranscript|><|l0|><|transcribe|><|notimestamps|> with <|endoftext|> added to suppress_tokens, so every row runs all
224 decoding steps and the arms do the same number of steps.  Arms (CUDA graph on):

  * beam5:  beam_size=5 (40 decoder rows);
  * sample: beam_size=1, num_hypotheses=5, sampling_topk=0, sampling_temperature=0.8 (40 decoder rows);
  * greedy: beam_size=1 (8 rows).

Prints one JSON line with, per arm, call_ms (host clock around generate, which ends with a device synchronise; median of
--repeats after a warm-up) and step_ms = (call_ms - encode_ms) / 224, where encode_ms is Whisper.encode of the same batch;
then the search kernels per step from torch.profiler over one uncaptured call of each arm (beam_rows_kernel +
beam_update_kernel against beam_sample_kernel + beam_sample_update_kernel), and sampler_op_us, CUDA events over
ct2b200_random_sample on 40 x 51865 float16 rows (k=0 and k=50, T=0.8; *_kernel: the kernel's own time from
torch.profiler, without the gaps between launches); with the card's name and power limit read in the same
run.

usage: python tools/whisper_sample_bench.py [--repeats 5]"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from score_bench import card  # noqa: E402

STEPS = 224
SEARCH_KERNELS = ("beam_rows_kernel", "beam_update_kernel", "beam_sample_kernel", "beam_sample_update_kernel")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    from ctranslate2_b200 import ops, set_random_seed
    from ctranslate2_b200.converters.synthetic import WhisperConfig, write_whisper_model
    from ctranslate2_b200.whisper import Whisper
    cfg = WhisperConfig(encoder_layers=12, decoder_layers=12, num_heads=12, d_model=768, n_mels=80, max_source_positions=1500,
                        max_target_positions=448, text_tokens=50257, languages=99, timestamps=1501)
    rng = np.random.default_rng(5)
    x = (rng.standard_normal((8, 80, 3000)) * 2).astype(np.float32)
    set_random_seed(1)
    rec = {"workload": "Whisper.generate, Whisper-small-shaped synthetic model INT8 (int8_float16), 8 windows x 3000 frames, "
                       "notimestamps prompt, <|endoftext|> suppressed: 224 steps", "repeats": a.repeats}
    with tempfile.TemporaryDirectory() as tmp:
        mdir = os.path.join(tmp, "whisper_small_shaped")
        write_whisper_model(mdir, cfg, "int8_float16", seed=11)
        w = Whisper(mdir, compute_type="int8_float16")
        prompt = [[w.sot_id, w.sot_id + 1, w.sot_id + 101, w.no_timestamps_id]] * 8
        arms = {"beam5": dict(beam_size=5),
                "sample": dict(beam_size=1, num_hypotheses=5, sampling_topk=0, sampling_temperature=0.8),
                "greedy": dict(beam_size=1)}
        common = dict(max_length=448, suppress_tokens=[-1, w.eot_id])

        def timed(model, fn, n):
            fn()                                                       # warm-up: arena growth, graph capture
            ts = []
            for _ in range(n):
                t0 = time.perf_counter()
                fn()
                ts.append((time.perf_counter() - t0) * 1e3)
            return statistics.median(ts), [round(min(ts), 2), round(max(ts), 2)]

        encode_ms, _ = timed(w, lambda: w.encode(x), a.repeats)
        rec["encode_ms"] = round(encode_ms, 2)
        for name, kw in arms.items():
            res = w.generate(x, prompt, **kw, **common)
            assert all(len(s) == STEPS for r in res for s in r.sequences_ids), name
            ms, spread = timed(w, lambda: w.generate(x, prompt, **kw, **common), a.repeats)
            rec[name] = {"call_ms": round(ms, 2), "call_ms_min_max": spread, "step_ms": round((ms - encode_ms) / STEPS, 4)}
        w.close()

        eager = Whisper(mdir, compute_type="int8_float16", use_cuda_graph=False)
        for name in ("beam5", "sample"):
            eager.generate(x, prompt, **arms[name], **common)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                eager.generate(x, prompt, **arms[name], **common)
            per = {}
            for e in prof.key_averages():
                for k in SEARCH_KERNELS:
                    if k in e.key:
                        per[k] = per.get(k, 0.0) + e.device_time_total / STEPS
            rec[name]["search_kernels_us_per_step"] = {k: round(v, 2) for k, v in per.items()}
            rec[name]["search_us_per_step"] = round(sum(per.values()), 2)
        eager.close()

    logits = torch.randn(40, 51865, device="cuda").mul_(3).half()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    rec["sampler_op_us"] = {}
    for k in (0, 50):
        for i in range(20):
            ops.random_sample(logits, k, 0.8, seed=1, counter=i)
        ev0.record()
        n = 500
        for i in range(n):
            ops.random_sample(logits, k, 0.8, seed=1, counter=i)
        ev1.record()
        torch.cuda.synchronize()
        rec["sampler_op_us"]["k%d" % k] = round(ev0.elapsed_time(ev1) * 1e3 / n, 2)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:     # the kernel alone, without the launch gaps
            for i in range(n):
                ops.random_sample(logits, k, 0.8, seed=1, counter=i)
            torch.cuda.synchronize()
        kern = sum(e.device_time_total for e in prof.key_averages() if "random_sample_kernel" in e.key)
        rec["sampler_op_us"]["k%d_kernel" % k] = round(kern / n, 2)
    rec.update(card())
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
