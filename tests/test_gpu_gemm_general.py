"""-m gpu: the two general persistent wgmma GEMMs (gemm_tc.cu, awq.cu) at the shapes the specialised kernels decline.

Those shapes are what still reaches them: more output tiles than one wave at m <= 64 (a CTA's unit range then straddles
two tiles, and tiles are shared between CTAs), rows whose pitch is not a multiple of 16 bytes at m > 64, the raw int32
output of ops::Gemm, and AWQ with its weight-streaming kernel switched off.  Every group runs all its cases once, then
all of them again, and requires bitwise-identical results: a ticket counter or partial-tile slot that is not left clean
by one call changes a later one."""
import functools

import numpy as np
import pytest
import torch

from ctranslate2_b200 import ops
from oracle import ct2_oracle as O
from gpu_util import DEV, TDT, TOL, dev, gpu, round_through, to_np
from test_gpu_awq import make_awq, pack

TC = ops.GEMM_TCGEN05


def dense_ref(x, wq, ws, bias=None, act=O.ACT_NONE, res=None):
    """O.dense_int8 with the int8 product taken in float64, which is exact here (|sum| < 2^53) and fast."""
    xq, xs = O.quantize_rows(x)
    c = (xq.astype(np.float64) @ wq.astype(np.float64).T).astype(np.int32)
    y = O.dequantize_gemm_output(c, xs, ws, bias, act, "cuda")
    return y if res is None else (y + res.astype(np.float32)).astype(np.float32)


def close(y, ref, dt):
    tol = TOL[dt] if dt != "float32" else 2e-5
    np.testing.assert_allclose(to_np(y), ref, rtol=tol, atol=tol * max(1.0, float(np.abs(ref).max())))


def run_twice(cases):
    """cases: list of () -> (output tensor, check(output)).  All run, checked, then all run again: bitwise equal."""
    first = []
    for case in cases:
        y, check = case()
        check(y)
        first.append(y.clone())
    for case, y0 in zip(cases, first):
        assert torch.equal(case()[0], y0)


@functools.lru_cache(maxsize=4)
def int8_weight(n, k, seed):
    r = np.random.default_rng(seed)
    wq, ws = O.quantize_weight((r.standard_normal((n, k)) * 0.05).astype(np.float32))
    return wq, ws, dev(wq), dev(ws)


@functools.lru_cache(maxsize=4)
def f16_weight(n, k, dt):
    b = round_through(np.random.default_rng(n + k).standard_normal((n, k)) * 0.05, dt)
    return b, dev(b, TDT[dt])


def dense_case(m, n, k, dt, seed, glu=False):
    r = np.random.default_rng(seed)
    x = round_through(r.standard_normal((m, k)), dt)
    wq, ws, wq_d, ws_d = int8_weight(n, k, 1)
    xq, xs = ops.Quantize()(dev(x, TDT[dt]))
    if glu:
        wu, su, wu_d, su_d = int8_weight(n, k, 2)
        ref = round_through(dense_ref(x, wq, ws, act=O.ACT_SWISH), dt) * round_through(dense_ref(x, wu, su), dt)
        args = (xq, xs, wq_d, ws_d, wu_d, su_d)
        return lambda: (ops.dense_int8_glu(*args, ops.ActivationType.Swish, TDT[dt], TC), lambda y: close(y, ref, dt))
    bias = round_through(r.standard_normal(n) * 0.1, dt)
    res = round_through(r.standard_normal((m, n)), dt)
    ref = dense_ref(x, wq, ws, bias, O.ACT_GELU, res)
    args = (xq, xs, wq_d, ws_d, dev(bias, TDT[dt]), dev(res, TDT[dt]), ops.ActivationType.GELU, TDT[dt], TC)
    return lambda: (ops.dense_int8(*args), lambda y: close(y, ref, dt))


def f16_case(m, n, k, dt, seed):
    r = np.random.default_rng(seed)
    a = round_through(r.standard_normal((m, k)), dt)
    b, b_d = f16_weight(n, k, dt)
    bias = round_through(r.standard_normal(n), dt)
    ref = a.astype(np.float64) @ b.astype(np.float64).T + bias
    args = (dev(a, TDT[dt]), b_d)

    def check(y):
        np.testing.assert_allclose(to_np(y), ref, rtol=TOL[dt], atol=TOL[dt] * float(np.abs(ref).max()))
    return lambda: (ops.Gemm()(*args, bias=dev(bias, TDT[dt])), check)


@gpu
@pytest.mark.parametrize("k", [1024, 4096])
def test_general_straddling_tiles(k):
    """m <= 64 with 157 (n = 20000) or 133 (GLU, n = 17000) tiles of 128 channels on 132 SMs: stream-K, CTA ranges
    straddle two tiles and tiles are shared."""
    cases = []
    for m in (1, 16, 17, 33, 64):
        for dt in ("float32", "float16", "bfloat16"):
            cases.append(dense_case(m, 20000, k, dt, m * 10 + k))
        cases.append(dense_case(m, 17000, k, "float16", m + k, glu=True))
        for dt in ("float16", "bfloat16"):
            cases.append(f16_case(m, 20000, k, dt, m + 7 * k))
    run_twice(cases)


@gpu
def test_general_unaligned_rows():
    """m > 64 with n not a multiple of 8 (output rows not 16-byte aligned): the prefill kernel declines."""
    cases = []
    for m in (65, 100, 300):
        for n in (1001, 1003):
            for dt in ("float32", "float16", "bfloat16"):
                cases.append(dense_case(m, n, 1024, dt, m + n))
            cases.append(dense_case(m, n, 1024, "float16", m * n, glu=True))
            cases.append(f16_case(m, n, 1024, "bfloat16" if n == 1001 else "float16", n - m))
    run_twice(cases)


@gpu
def test_general_raw_int32():
    """ops::Gemm int8 -> int32: tile-partitioned split-K at (1, 4096, 4096) (32 tiles, 4 or 5 CTAs each) and stream-K with
    shared tiles at (64, 12000, 4096) (94 tiles on 132 CTAs).  Exact."""
    def case(m, n, k):
        g = torch.Generator(device=DEV).manual_seed(m * 7 + n)
        a = torch.randint(-127, 128, (m, k), device=DEV, dtype=torch.int8, generator=g)
        b = torch.randint(-127, 128, (n, k), device=DEV, dtype=torch.int8, generator=g)
        ref = (a.double() @ b.double().T).to(torch.int32)      # exact: |sum| < 2^53

        def check(c):
            assert torch.equal(c, ref), f"max abs diff {(c - ref).abs().max().item()}"
        return lambda: (ops.Gemm(impl=TC)(a, b), check)
    run_twice([case(1, 4096, 4096), case(64, 12000, 4096), case(17, 4096, 1024)])


@gpu
def test_general_awq(monkeypatch):
    """gemm_awq_tc_kernel (CT2B200_AWQ_DECODE=0; m >= 2 also skips the one-row GEMV) beyond one wave (n = 17000: 133
    tiles) and on a ragged n, Dense with bias + activation + residual and the fused gate/up, against float64 truth."""
    monkeypatch.setenv("CT2B200_AWQ_DECODE", "0")
    k, g = 2048, 128
    cases = []
    for n in (1000, 17000):
        w_int, z_int, scales, deq = make_awq(n, k, g, n)
        wt = ops.AwqWeight(*[dev(a) for a in pack(w_int, z_int, scales, g, ops.AWQ_GEMM)], ops.AWQ_GEMM, g)
        wu = make_awq(n, k, g, n + 1)
        ut = ops.AwqWeight(*[dev(a) for a in pack(*wu[:3], g, ops.AWQ_GEMV)], ops.AWQ_GEMV, g)
        for m in (2, 17, 64):
            r = np.random.default_rng(m + n)
            x = r.standard_normal((m, k)).astype(np.float16)
            bias = r.standard_normal(n).astype(np.float16)
            res = r.standard_normal((m, n)).astype(np.float16)
            prod = x.astype(np.float64) @ deq.astype(np.float64)
            ref = O.activation((prod + bias).astype(np.float32), O.ACT_SWISH) + res.astype(np.float32)
            gate = O.activation(prod.astype(np.float32), O.ACT_SWISH)
            ref_glu = gate * (x.astype(np.float64) @ wu[3].astype(np.float64)).astype(np.float32)

            def dense(x=dev(x), bias=dev(bias), res=dev(res), wt=wt, ref=ref):
                def check(y):
                    np.testing.assert_allclose(to_np(y), ref, rtol=1e-2, atol=1e-2 * max(1.0, np.abs(ref).max()))
                return ops.dense_awq(x, wt, bias=bias, residual=res, activation_type=ops.ActivationType.Swish), check

            def glu(x=dev(x), wt=wt, ut=ut, ref=ref_glu):
                def check(h):
                    np.testing.assert_allclose(to_np(h), ref, rtol=2e-2, atol=2e-2 * np.abs(ref).max())
                return ops.dense_awq_glu(x, wt, ut), check
            cases += [dense, glu]
    run_twice(cases)
