"""Encoder-only throughput on a BERT-base-shaped synthetic INT8 model (12 layers, d 768, 12 heads of 64, FFN 3072, two
token types, pooler), compute type int8_float16, at 64 sequences x 512 tokens and 64 sequences of U[32, 512] tokens:

  * the median device-timed encoder pass (CUDA events around the whole pass, ct2b200_encoder_bench) and tokens/s over the
    valid tokens;
  * the tensor-core encoder attention next to the generic kernel on the same inputs (64 x 512, fp16), per-launch CUDA time
    from torch.profiler in a run of its own;
  * the card's name and power limit, read in the same process.

    python tools/encoder_bench.py [--out FILE.json] [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    name, power, clock = [x.strip() for x in r.stdout.strip().split("\n")[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def attention_times(iters):
    import torch
    from torch.profiler import ProfilerActivity, profile
    from ctranslate2_b200 import ops
    B, T, H, D = 64, 512, 12, 64
    g = torch.Generator(device="cpu").manual_seed(0)
    qkv = torch.randn(B * T, 3 * H * D, generator=g).to("cuda", torch.float16)
    lens = torch.full((B,), T, dtype=torch.int32, device="cuda")
    for _ in range(3):                                           # warm-up (module load, smem attribute)
        ops.attention_encoder(qkv, H, D, B, lengths=lens)
        ops.attention_encoder_mma(qkv, H, D, B, lengths=lens)
    torch.cuda.synchronize()
    diff = (ops.attention_encoder(qkv, H, D, B, lengths=lens).float()
            - ops.attention_encoder_mma(qkv, H, D, B, lengths=lens).float()).abs().max().item()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            ops.attention_encoder(qkv, H, D, B, lengths=lens)
            ops.attention_encoder_mma(qkv, H, D, B, lengths=lens)
        torch.cuda.synchronize()
    times = {}
    for e in prof.key_averages():
        if "attention_generic_kernel" in e.key:
            times["generic_ms"] = e.device_time_total / e.count / 1000.0
        elif "attention_prefill_mma_kernel" in e.key:
            times["mma_ms"] = e.device_time_total / e.count / 1000.0
    flops = 4.0 * B * T * T * H * D
    times.update({"shape": [B, T, H, D], "max_abs_diff": diff,
                  "mma_tflops": flops / times["mma_ms"] / 1e9, "generic_tflops": flops / times["generic_ms"] / 1e9})
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    import ctranslate2_b200 as ct2
    from ctranslate2_b200.converters.synthetic import BERT_BASE, write_encoder_model
    result = {"card": card(), "model": "BERT-base-shaped synthetic, int8 weights", "compute_type": "int8_float16"}
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "bert")
        write_encoder_model(path, BERT_BASE, "int8", seed=7)
        enc = ct2.Encoder(path, compute_type="int8_float16", max_batch_size=64)
        rng = np.random.default_rng(0)
        for name, lens in (("64x512", np.full(64, 512)), ("64xU[32,512]", rng.integers(32, 513, 64))):
            ms = enc.bench(lens, int(lens.max()), iters=args.iters, warmup=3)
            result[name] = {"median_ms": ms, "tokens": int(lens.sum()), "tokens_per_s": float(lens.sum()) / (ms / 1000.0)}
        enc.close()
    result["attention"] = attention_times(args.iters)
    result["card_after"] = card()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
