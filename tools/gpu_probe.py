#!/usr/bin/env python
"""First-contact probe for a fresh H100 box: exercises each kernel family once with diagnostics
(prints what differs instead of just failing).  Usage: python tools/gpu_probe.py [tc|mma|attn|engine|all]"""
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ctranslate2_b200 import ops  # noqa: E402


def probe_gemm(impl, name):
    print("== int8 GEMM", name)
    for (m, n, k) in [(128, 256, 128), (128, 256, 512), (1, 128, 128), (16, 4096, 4096), (32, 6144, 4096),
                      (64, 512, 4096), (200, 1000, 2048), (1024, 4096, 4096)]:
        g = torch.Generator(device="cuda").manual_seed(m + n + k)
        a = torch.randint(-127, 128, (m, k), device="cuda", dtype=torch.int8, generator=g)
        b = torch.randint(-127, 128, (n, k), device="cuda", dtype=torch.int8, generator=g)
        t0 = time.time()
        c = ops.Gemm(impl=impl)(a, b)
        torch.cuda.synchronize()
        ref = (a.double() @ b.double().T).to(torch.int32)
        bad = (c != ref)
        print("  m=%d n=%d k=%d: %s (%.1f ms) mismatches=%d/%d" % (m, n, k, "OK" if not bad.any() else "FAIL",
                                                                   1e3 * (time.time() - t0), int(bad.sum()), bad.numel()))
        if bad.any():
            idx = bad.nonzero()[:5].tolist()
            print("    first bad:", [(i, j, int(c[i, j]), int(ref[i, j])) for i, j in idx])
            rows_bad = bad.any(1).nonzero().flatten()[:10].tolist()
            cols_bad = bad.any(0).nonzero().flatten()[:10].tolist()
            print("    bad rows (first):", rows_bad, " bad cols (first):", cols_bad)
            # does the output equal the reference of a K-prefix? (descriptor advance bug) or is it zero?
            print("    all-zero output:", bool((c == 0).all().item()))
            for kk in (32, 64, 96, 128):
                if kk <= k:
                    pref = (a[:, :kk].double() @ b[:, :kk].double().T).to(torch.int32)
                    if torch.equal(c, pref):
                        print("    output == GEMM over first %d of K" % kk)


def probe_f16():
    print("== f16/bf16 GEMM (wgmma)")
    for dt in (torch.float16, torch.bfloat16):
        for (m, n, k) in [(128, 256, 64), (8, 512, 1024), (300, 640, 512)]:
            a = torch.randn((m, k), device="cuda").to(dt)
            b = (torch.randn((n, k), device="cuda") * 0.05).to(dt)
            c = ops.Gemm()(a, b)
            ref = a.double() @ b.double().T
            err = (c.double() - ref).abs().max().item() / ref.abs().max().item()
            print("  %s m=%d n=%d k=%d rel err %.2e %s" % (dt, m, n, k, err, "OK" if err < 2e-2 else "FAIL"))


def main():
    what = sys.argv[1] if len(sys.argv) > 1 else "all"
    print(torch.cuda.get_device_name(0), torch.cuda.get_device_capability(0))
    if what in ("tc", "all"):
        probe_gemm(ops.GEMM_TCGEN05, "tcgen05")
        probe_f16()
    if what in ("mma", "all"):
        probe_gemm(ops.GEMM_MMA_SYNC, "mma.sync")


if __name__ == "__main__":
    main()
