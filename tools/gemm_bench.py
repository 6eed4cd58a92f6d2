#!/usr/bin/env python
"""Micro-benchmarks of the decode-path kernels with CUDA events (weights rotated through > L2 worth of copies).
usage: python tools/gemm_bench.py [gemm] [awq] [attn] [sweep] [--rowsteps 8,1] [--rounds 3]

sweep: every INT8 decode Dense shape of Llama-3-8B alone, at m = 1, 16, 32, 64, for every planner row step
(CT2B200_GEMM_ROWSTEP); GB/s of algorithmic bytes (weights, their scales, activations, output), the median of --rounds
interleaved rounds.  Run it once per build (CT2B200_LIB) to compare builds."""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ctranslate2_b200 import ops  # noqa: E402


def hbm_peak():
    """HBM bandwidth the shares of peak are taken against: MEASURED_PEAKS.json if present, else the H100 SXM data sheet."""
    p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
    if os.path.exists(p):
        return float(json.load(open(p))["hbm_gbs"])
    return 3350.0


PEAK = hbm_peak()


def card():
    """name, power limit and max SM clock of GPU 0, as nvidia-smi reports them"""
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as ex:
        return "nvidia-smi unavailable: %s" % ex


def timeit(fn, iters):
    for i in range(3):
        fn(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3   # us


def bench_gemm():
    shapes = [("qkv", 6144, 4096, False), ("out", 4096, 4096, False), ("gate_up", 14336, 4096, True),
              ("down", 4096, 14336, False), ("lm_head", 128256, 4096, False)]
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, n, k, glu in shapes:
        nbytes = n * k * (2 if glu else 1)
        copies = max(2, int(300e6 // nbytes) + 1)
        ws = [torch.randint(-127, 128, (n, k), dtype=torch.int8, device="cuda", generator=g) for _ in range(copies * (2 if glu else 1))]
        sc = torch.full((n,), 3000.0, device="cuda")
        for m in (1, 8, 16, 32, 64):
            xq = torch.randint(-127, 128, (m, k), dtype=torch.int8, device="cuda", generator=g)
            xs = torch.full((m,), 40.0, device="cuda")
            res = torch.zeros((m, n), dtype=torch.float16, device="cuda")
            if glu:
                fn = lambda i: ops.dense_int8_glu(xq, xs, ws[2 * (i % copies)], sc, ws[2 * (i % copies) + 1], sc)
            else:
                fn = lambda i: ops.dense_int8(xq, xs, ws[i % copies], sc, residual=res)
            us = timeit(fn, 6 * copies)
            gbs = nbytes / us / 1e3
            print("gemm %-8s n=%6d k=%5d m=%2d: %7.2f us  %7.1f GB/s  %.3f of peak" % (name, n * (2 if glu else 1), k, m, us, gbs, gbs / PEAK), flush=True)
        del ws
        torch.cuda.empty_cache()


def bench_awq():
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, n, k, glu in [("qkv", 6144, 4096, False), ("gate_up", 14336, 4096, True), ("down", 4096, 14336, False)]:
        nbytes = n * k // 2 * (2 if glu else 1)
        copies = max(2, int(300e6 // nbytes) + 1)
        G = 128
        ws = []
        for _ in range(copies * (2 if glu else 1)):
            qw = torch.randint(-2**31, 2**31 - 1, (k, n // 8), dtype=torch.int32, device="cuda", generator=g)
            sc = torch.full((k // G, n), 0.01, dtype=torch.float16, device="cuda")
            qz = torch.randint(-2**31, 2**31 - 1, (k // G, n // 8), dtype=torch.int32, device="cuda", generator=g)
            ws.append(ops.AwqWeight(qw, sc, qz, ops.AWQ_GEMM, G))
        for m in (1, 16, 32):
            x = torch.randn((m, k), device="cuda").half()
            if glu:
                fn = lambda i: ops.dense_awq_glu(x, ws[2 * (i % copies)], ws[2 * (i % copies) + 1])
            else:
                fn = lambda i: ops.dense_awq(x, ws[i % copies])
            us = timeit(fn, 6 * copies)
            gbs = nbytes / us / 1e3
            print("awq  %-8s n=%6d k=%5d m=%2d: %7.2f us  %7.1f GB/s  %.3f of peak" % (name, n * (2 if glu else 1), k, m, us, gbs, gbs / PEAK), flush=True)
        del ws
        torch.cuda.empty_cache()


def bench_attn():
    H, Hkv, D = 32, 8, 128
    for B, ctx in [(1, 1024), (1, 2047), (32, 1024), (32, 2047)]:
        max_len = 2048
        layers = max(2, int(400e6 // (B * Hkv * max_len * D * 2 * 2)) + 1)
        kc = [torch.randn((B, Hkv, max_len, D), device="cuda").half() for _ in range(layers)]
        vc = [torch.randn((B, Hkv, max_len, D), device="cuda").half() for _ in range(layers)]
        qkv = torch.randn((B, (H + 2 * Hkv) * D), device="cuda").half()
        ang = torch.rand((max_len, D), device="cuda")
        sin, cos = torch.sin(ang), torch.cos(ang)
        lens = torch.full((B,), ctx, dtype=torch.int32, device="cuda")
        nb = ops.lib().ct2b200_attention_decode_workspace(B, H, D, max_len) if False else 64 << 20
        wsb = torch.zeros(nb, dtype=torch.uint8, device="cuda")
        fn = lambda i: ops.attention_decode(qkv, kc[i % layers], vc[i % layers], sin, cos, lens, H, Hkv, D, workspace=wsb)
        us = timeit(fn, 6 * layers)
        nbytes = B * Hkv * (ctx + 1) * D * 2 * 2
        gbs = nbytes / us / 1e3
        print("attn B=%2d ctx=%4d: %7.2f us  %7.1f GB/s  %.3f of peak" % (B, ctx, us, gbs, gbs / PEAK), flush=True)
        del kc, vc
        torch.cuda.empty_cache()


def _opt(name, default):
    return [int(v) for v in sys.argv[sys.argv.index(name) + 1].split(",")] if name in sys.argv else default


def bench_sweep():
    rowsteps, rounds = _opt("--rowsteps", [8, 1]), _opt("--rounds", [3])[0]
    shapes = [("qkv", 6144, 4096, False), ("out", 4096, 4096, False), ("gate_up", 14336, 4096, True), ("down", 4096, 14336, False)]
    g = torch.Generator(device="cuda").manual_seed(0)
    saved = os.environ.get("CT2B200_GEMM_ROWSTEP")
    results = []
    for name, n, k, glu in shapes:
        nw = 2 if glu else 1
        wbytes = n * k * nw
        copies = max(2, int(300e6 // wbytes) + 1)
        ws = [torch.randint(-127, 128, (n, k), dtype=torch.int8, device="cuda", generator=g) for _ in range(copies * nw)]
        sc = torch.full((n,), 3000.0, device="cuda")
        for m in (1, 16, 32, 64):
            xq = torch.randint(-127, 128, (m, k), dtype=torch.int8, device="cuda", generator=g)
            xs = torch.full((m,), 40.0, device="cuda")
            if glu:
                fn = lambda i: ops.dense_int8_glu(xq, xs, ws[2 * (i % copies)], sc, ws[2 * (i % copies) + 1], sc)
            else:
                fn = lambda i: ops.dense_int8(xq, xs, ws[i % copies], sc)
            alg = wbytes + n * nw * 4 + m * k + m * 4 + m * n * 2
            times = {r: [] for r in rowsteps}
            for _ in range(rounds):
                for r in rowsteps:
                    os.environ["CT2B200_GEMM_ROWSTEP"] = str(r)
                    times[r].append(timeit(fn, max(60, 6 * copies)))
            for r, ts in times.items():
                us = sorted(ts)[len(ts) // 2]
                gbs = alg / us / 1e3
                results.append({"shape": name, "n": n * nw, "k": k, "m": m, "rowstep": r, "us": round(us, 2),
                                "us_min": round(min(ts), 2), "us_max": round(max(ts), 2), "GBps": round(gbs, 1),
                                "frac": round(gbs / PEAK, 4)})
                print("sweep %-8s n=%6d k=%5d m=%2d rowstep=%d: %7.2f us [%7.2f, %7.2f]  %7.1f GB/s  %.3f of %.0f" % (
                    name, n * nw, k, m, r, us, min(ts), max(ts), gbs, gbs / PEAK, PEAK), flush=True)
        del ws
        torch.cuda.empty_cache()
    if saved is None:
        os.environ.pop("CT2B200_GEMM_ROWSTEP", None)
    else:
        os.environ["CT2B200_GEMM_ROWSTEP"] = saved
    print("SWEEP_JSON", json.dumps({"card": card(), "peak_gbs": PEAK, "results": results}), flush=True)


if __name__ == "__main__":
    what = [a for a in sys.argv[1:] if not a.startswith("--") and not a[0].isdigit()] or ["gemm", "awq", "attn"]
    print(torch.cuda.get_device_name(0), "|", card(), "| env:", {k: v for k, v in os.environ.items() if k.startswith("CT2B200")})
    if "sweep" in what:
        bench_sweep()
    if "gemm" in what:
        bench_gemm()
    if "awq" in what:
        bench_awq()
    if "attn" in what:
        bench_attn()
