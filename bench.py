#!/usr/bin/env python
"""bench.py — generate_batch tokens/sec, Llama-3-8B INT8 (int8_float16), greedy, synthetic weights/prompts.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--batch B] [--impl ours|reference] [--model 8b|1b|tiny]

A "step" is one decode step of the whole batch (B generated tokens) of BASELINE.json configs[2]
("Llama-3-8B generate_batch INT8, seq 2048, bsz 1 and 32, on 1xH100"): prompt P=1024 then K generated
tokens per sequence.  One JSON line on stdout (rank 0):
  value    = B*K*N / device time of K decode steps, inputs already resident in HBM (CUDA events, max over ranks)
  e2e      = the same tokens/s through ctranslate2_b200.Generator.generate_batch with HOST prompt ids and HOST
             result ids (prefill + decode + host<->device copies inside the timed region)
  e2e_full = e2e at the NAMED workload (1024 generated tokens after the 1024-token prompt) whatever --steps is
  variants = the four points of BASELINE.json's metric — INT8 and AWQ-INT4 at bsz 1 and 32 — device-timed decode
             (ms/step, tokens/s, fraction of the HBM roofline of the step), each beside `ref_cuda`: the UNMODIFIED
             reference's own CUDA build (oracle/_ref_cuda: cuBLAS INT8 GEMM / its AWQ kernels) on the same GPU
  translate = BASELINE.json configs[1] (OPUS-MT-shaped Transformer-base INT8, 64 sentences, beam 4): device-timed decoding
             steps, end-to-end target tokens/s through Translator.translate_batch, beside the reference's CUDA Translator
  roofline = the weight-streaming wgmma GEMM timed alone with CUDA events over buffers larger than L2
  cpu_baseline = the unmodified reference (oracle/_ref, Ruy INT8) on the host cores, bounded sample
N>1: independent data-parallel replicas (one process per GPU, no data-path collective): scaling "weak"; the same line
also carries `tp`: ONE tensor-parallel generator over the N GPUs (heads / FFN columns sharded, collectives fused into
kernels over NVLink peer memory), strong scaling of the same step.
`--impl reference` times the reference's own CPU implementation (oracle/_ref) on the host cores.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

MODELS = {
    "8b": dict(num_layers=32, num_heads=32, num_heads_kv=8, head_dim=128, ffn_dim=14336, vocab_size=128256),
    "1b": dict(num_layers=16, num_heads=32, num_heads_kv=8, head_dim=64, ffn_dim=8192, vocab_size=128256),
    "tiny": dict(num_layers=2, num_heads=8, num_heads_kv=2, head_dim=128, ffn_dim=2048, vocab_size=2000),
}
NAMES = {"8b": "Llama-3-8B", "1b": "Llama-3.2-1B-shaped", "tiny": "tiny-llama-d128"}
PROMPT_LEN = 1024


def model_dir(name, quant="int8_float16"):
    """Synthetic model directory in the reference's on-disk format (written once per box)."""
    from ctranslate2_b200.converters.synthetic import LlamaConfig, write_llama_model
    base = os.environ.get("CT2B200_BENCH_DIR", os.path.join(tempfile.gettempdir(), "ct2b200_bench"))
    d = os.path.join(base, "llama_%s_%s" % (name, quant))
    done = os.path.join(d, ".complete")
    if not os.path.exists(done):
        os.makedirs(base, exist_ok=True)
        t0 = time.time()
        # embeddings of unit scale and small residual-stream matrices: a random 32-layer model with one init_std everywhere
        # is chaotic (synthetic.py), and the full-size parity tests compare whole-model logits with the reference's
        write_llama_model(d, LlamaConfig(**MODELS[name]), quant, seed=1234, fast_int8=True, embedding_std=1.0,
                          residual_std=0.002)
        open(done, "w").write("ok")
        print("[bench] wrote %s in %.1fs" % (d, time.time() - t0), file=sys.stderr)
    return d


def prompts_for(name, batch, plen, seed=42):
    import numpy as np
    v = MODELS[name]["vocab_size"]
    return np.random.default_rng(seed).integers(3, v, size=(batch, plen), dtype=np.int32)


class ClockSampler:
    """nvidia-smi clocks/throttle reasons during the timed region."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index):
        self.idx, self.rows, self.proc = gpu_index, [], None

    def __enter__(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.idx), "--query-gpu=" + self.Q,
                                          "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None
        return self

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def __exit__(self, *a):
        if self.proc:
            self.proc.terminate()
            try:
                self.proc.wait(timeout=2)
            except Exception:
                self.proc.kill()

    def summary(self):
        sm, mx, reasons = [], 0, set()
        for r in self.rows:
            try:
                sm.append(float(r[1]))
                mx = max(mx, float(r[2]))
                for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[4:8]):
                    if v.lower().startswith("active"):
                        reasons.add(name)
            except Exception:
                pass
        # median over the busier half of the samples (the sampler also sees idle gaps)
        sm.sort()
        busy = sm[len(sm) // 2:] if sm else []
        return {"sm_mhz": statistics.median(busy) if busy else None, "sm_max_mhz": mx or None,
                "reasons": sorted(reasons), "samples": len(sm)}


def measured_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        j = json.load(open(p))
        return float(j["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    return 3350.0, "fallback (H100 SXM data sheet, 3.35 TB/s HBM3)"


def step_bytes(name, batch, ctx, weights="int8"):
    """Algorithmic bytes of one decode step (SURVEY §8d): linear weights + their scales + KV read.
    int8: 1 B per weight + fp32 row scales; awq: 0.5 B per weight + fp16 scale and zero per group of 128, fp16 lm_head."""
    m = MODELS[name]
    d = m["num_heads"] * m["head_dim"]
    qkv = (m["num_heads"] + 2 * m["num_heads_kv"]) * m["head_dim"]
    per_layer = qkv * d + d * d + 3 * m["ffn_dim"] * d
    kv = 2 * m["num_heads_kv"] * m["head_dim"] * 2 * m["num_layers"]
    if weights == "awq":
        w = m["num_layers"] * per_layer // 2 + m["num_layers"] * per_layer // 128 * 4 + 2 * m["vocab_size"] * d
        return w + batch * ctx * kv
    w = m["num_layers"] * per_layer + m["vocab_size"] * d
    scales = 4 * (m["num_layers"] * (qkv + d + 2 * m["ffn_dim"] + d) + m["vocab_size"])
    return w + scales + batch * ctx * kv


def gemm_roofline(name, batch, device):
    """Times the dominant kernel (fused gate/up INT8 GEMM on wgmma, weight streaming) alone with CUDA
    events, cycling through more weight copies than fit in L2 (50 MB) so every launch streams from HBM."""
    import torch
    from ctranslate2_b200 import ops
    m = MODELS[name]
    d, f = m["num_heads"] * m["head_dim"], m["ffn_dim"]
    copies = max(3, int(400e6 // (2 * f * d)) + 1)
    g = torch.Generator(device=device).manual_seed(0)
    wg = [torch.randint(-127, 128, (f, d), dtype=torch.int8, device=device, generator=g) for _ in range(copies)]
    wu = [torch.randint(-127, 128, (f, d), dtype=torch.int8, device=device, generator=g) for _ in range(copies)]
    sg = torch.full((f,), 3000.0, device=device)
    xq = torch.randint(-127, 128, (batch, d), dtype=torch.int8, device=device, generator=g)
    xs = torch.full((batch,), 40.0, device=device)
    for i in range(copies):
        ops.dense_int8_glu(xq, xs, wg[i], sg, wu[i], sg)
    torch.cuda.synchronize()
    iters = 4 * copies
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        ops.dense_int8_glu(xq, xs, wg[i % copies], sg, wu[i % copies], sg)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    alg = 2 * f * d + 2 * f * 4 + batch * d + batch * 4 + batch * f * 2    # weights + scales + x + h(out)
    peak, how = measured_peaks()
    ach = alg / (ms * 1e-3) / 1e9
    traffic = None                # DRAM bytes of the kernel from a profiler capture: none taken on the H100
    return {"bound": "hbm", "kernel": "gemm_decode_kernel<s8, NB=2 gate/up + SwiGLU> (ffn gate/up %dx%d, m=%d)" % (2 * f, d, batch),
            "achieved": round(ach, 1), "peak": peak, "unit": "GB/s", "frac": round(ach / peak, 4),
            "traffic": traffic, "bytes_per_launch": alg, "us_per_launch": round(ms * 1e3, 2), "peak_source": how}


def awq_roofline(name, batch, device):
    """The dominant kernel of the AWQ variant: fused gate/up AWQ-INT4 GEMM (awq_decode.cu), timed alone like gemm_roofline."""
    import torch
    from ctranslate2_b200 import ops
    m = MODELS[name]
    d, f, G = m["num_heads"] * m["head_dim"], m["ffn_dim"], 128
    copies = max(3, int(400e6 // (f * d)) + 1)

    def weight():
        qw = torch.randint(-2 ** 31, 2 ** 31 - 1, (d, f // 8), dtype=torch.int32, device=device)
        sc = (torch.rand((d // G, f), device=device) * 0.01 + 0.005).to(torch.float16)
        qz = torch.randint(-2 ** 31, 2 ** 31 - 1, (d // G, f // 8), dtype=torch.int32, device=device)
        return ops.AwqWeight(qw, sc, qz, ops.AWQ_GEMM, G)

    wg, wu = [weight() for _ in range(copies)], [weight() for _ in range(copies)]
    x = torch.randn((batch, d), device=device, dtype=torch.float16)
    for i in range(copies):
        ops.dense_awq_glu(x, wg[i], wu[i])
    torch.cuda.synchronize()
    iters = 4 * copies
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        ops.dense_awq_glu(x, wg[i % copies], wu[i % copies])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    alg = 2 * (f * d // 2 + f * d // G * 4) + batch * d * 2 + batch * f * 2     # nibbles + scales/zeros + x + h
    peak, how = measured_peaks()
    ach = alg / (ms * 1e-3) / 1e9
    return {"bound": "hbm", "kernel": "awq_decode_kernel<NB=2 gate/up + SwiGLU> (ffn gate/up %dx%d int4 g128, m=%d)" % (2 * f, d, batch),
            "achieved": round(ach, 1), "peak": peak, "unit": "GB/s", "frac": round(ach / peak, 4), "traffic": None,
            "bytes_per_launch": alg, "us_per_launch": round(ms * 1e3, 2), "peak_source": how,
            "note": "the int4 -> fp16 conversion shares the SM with the stream"}


def _ref_thread_cache():
    base = os.environ.get("CT2B200_BENCH_DIR", os.path.join(tempfile.gettempdir(), "ct2b200_bench"))
    return os.path.join(base, "ref_threads.json")


def _ref_once(name, threads, batch, gen_tokens, prompt_len=8):
    """One reference generate_batch on `threads` host threads; returns (tokens/s, seconds, tokens)."""
    from oracle import refapi
    g = refapi.RefGenerator(model_dir(name), "int8", threads)
    prompts = prompts_for(name, batch, prompt_len)
    g.generate(prompts[:1, :2], max_length=1, min_length=1, end_id=2)     # touch the weights once
    t0 = time.time()
    out = g.generate(prompts, max_length=gen_tokens, min_length=gen_tokens, end_id=2)
    dt = time.time() - t0
    g.close()
    toks = sum(len(o) for o in out)
    return toks / dt, dt, toks


def reference_cpu(name, batch, steps, warmup, budget_s=100.0, calibrate=True):
    """The unmodified reference (oracle/_ref: CTranslate2 CPU build, Ruy INT8 GEMM, OpenMP) on the host cores:
    generate_batch of `batch` prompts — bounded sample: 8-token prompts, as many decode steps as fit the budget.
    "All the host threads it can use": Ruy + OpenMP oversubscribe badly at high thread counts, so the thread
    count is chosen by a short sweep (best tokens/s of {cores, cores/2, cores/4, 32, 16}) and cached per box."""
    from oracle import refapi
    if not refapi.available():
        return None
    cores = os.cpu_count() or 1
    cache = _ref_thread_cache()
    threads = int(os.environ.get("CT2B200_REF_THREADS", "0"))
    if not threads and os.path.exists(cache):
        threads = int(json.load(open(cache)).get(name, 0))
    if not threads and calibrate:
        best = (0.0, min(cores, 16))
        for th in sorted({cores, max(1, cores // 2), max(1, cores // 4), min(cores, 32), min(cores, 16)}):
            try:
                tps, dt, _ = _ref_once(name, th, 1, 2, prompt_len=2)
            except Exception:
                continue
            print("[bench] reference calibration: %d threads -> %.2f tok/s (%.1fs)" % (th, tps, dt), file=sys.stderr)
            if tps > best[0]:
                best = (tps, th)
        threads = best[1]
        try:
            os.makedirs(os.path.dirname(cache), exist_ok=True)
            d = json.load(open(cache)) if os.path.exists(cache) else {}
            d[name] = threads
            json.dump(d, open(cache, "w"))
        except Exception:
            pass
    if not threads:
        threads = min(cores, 32)
    # size the sample: one calibration step, then as many decode steps as fit the budget
    tps1, dt1, _ = _ref_once(name, threads, batch, 1)
    per_step = max(1e-3, dt1 / 2.0)      # prompt pass + 1 decode step
    k = int(max(1, min(steps, (budget_s - dt1) / per_step)))
    if k > 1:
        tps, dt, toks = _ref_once(name, threads, batch, k)
    else:
        tps, dt, toks, k = tps1, dt1, batch, 1
    return {"value": tps, "unit": "tokens/s", "cores": threads, "kind": "reference", "steps": k,
            "sample": "unmodified reference on CPU (Ruy int8, %d of %d host threads): generate_batch batch %d, "
                      "prompt 8 tokens, %d generated tokens per sequence, prompt pass included" % (threads, cores, batch, k),
            "seconds": dt}


def ref_cuda_bench(name, quant, compute, batch, plen, g1=8, g2=40, flash=False, timeout=900):
    """The unmodified reference's CUDA build (oracle/_ref_cuda) on the same GPU, in its own process: decode tokens/s from
    two generations of g1 and g2 tokens (the difference isolates the decode steps), e2e tokens/s of the longer one."""
    lib = os.path.join(ROOT, "oracle", "_ref_cuda", "libct2ref_cuda_driver.so")
    if not os.path.exists(lib):
        return {"unavailable": "oracle/_ref_cuda is not built (make -f oracle/Makefile.ref_cuda)"}
    cmd = [sys.executable, os.path.join(ROOT, "tools", "ref_cuda_worker.py"), "bench", model_dir(name, quant), compute,
           str(batch), str(plen), str(g1), str(g2)] + (["--flash"] if flash else [])
    try:
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout)
        line = [l for l in r.stdout.splitlines() if l.startswith("{")]
        if r.returncode != 0 or not line:
            return {"error": (r.stderr or r.stdout)[-300:]}
        return json.loads(line[-1])
    except Exception as ex:
        return {"error": str(ex)[-300:]}


def seq2seq_model_dir():
    """BASELINE.json configs[1]: OPUS-MT En-De geometry (Transformer-base 6+6, d 512, 8 heads, ffn 2048, V 58101, INT8, post-norm,
    Swish, zero first decoder embedding, source EOS — what converters/marian.py writes), random-init, written once per box."""
    from ctranslate2_b200.converters.synthetic import OPUS_MT_BASE, write_transformer_model
    base = os.environ.get("CT2B200_BENCH_DIR", os.path.join(tempfile.gettempdir(), "ct2b200_bench"))
    d = os.path.join(base, "opus_mt_base_int8")
    done = os.path.join(d, ".complete")
    if not os.path.exists(done):
        os.makedirs(base, exist_ok=True)
        write_transformer_model(d, OPUS_MT_BASE, "int8", seed=1234)
        open(done, "w").write("ok")
    return d


def translate_record(device_index, with_ref_cuda, batch=64, beam=4, max_len=256):
    """configs[1] (SURVEY §8d): translate_batch of 64 sentences of length U[10,50], beam 4, max_decoding_length 256, INT8
    weights / fp16 activations: device-timed decoding steps, end-to-end target tokens/s through Translator.translate_batch with
    HOST ids in and out, and the unmodified reference's CUDA Translator on the same GPU and sentences."""
    import numpy as np
    from ctranslate2_b200.translator import Translator
    mdir = seq2seq_model_dir()
    rng = np.random.default_rng(42)
    srcs = [[int(x) for x in rng.integers(3, 58101, size=int(rng.integers(10, 51)))] + [2] for _ in range(batch)]
    t = Translator(mdir, compute_type="int8_float16")
    enc_ms, dec_ms, launches = t.bench(batch, 51, beam, 64, 3)
    t.translate_ids(srcs, beam_size=beam, max_decoding_length=max_len, start_id=1, end_token=[2])      # warm-up at the timed shapes
    t0 = time.perf_counter()
    ids, lens, _ = t.translate_ids(srcs, beam_size=beam, max_decoding_length=max_len, start_id=1, end_token=[2])
    sec = time.perf_counter() - t0
    toks = int(lens[:, 0].sum())
    rec = {"workload": "OPUS-MT-shaped Transformer-base INT8 (int8_float16) translate_batch, %d sentences U[10,50], beam %d, "
                       "max_decoding_length %d (BASELINE.json configs[1])" % (batch, beam, max_len),
           "decode_ms_per_step": round(dec_ms / 64, 4), "rows_per_step": batch * beam, "encode_ms": round(enc_ms, 3),
           "launches_per_step": int(launches // 64), "e2e_target_tokens": toks, "e2e_seconds": round(sec, 4),
           "e2e_tokens_per_s": round(toks / sec, 1), "h2d_bytes": int(sum(len(r) for r in srcs) * 4), "d2h_bytes": toks * 4}
    t.close()
    return rec


def translate_reference(rec, batch=64, beam=4, max_len=256):
    """The unmodified reference's CUDA Translator on the same model and sentences (its own process)."""
    import numpy as np
    if not os.path.exists(os.path.join(ROOT, "oracle", "_ref_cuda", "libct2ref_cuda_driver.so")):
        return {"ref_cuda": {"unavailable": "oracle/_ref_cuda is not built (make -f oracle/Makefile.ref_cuda)"}}
    mdir = seq2seq_model_dir()
    rng = np.random.default_rng(42)
    srcs = [[int(x) for x in rng.integers(3, 58101, size=int(rng.integers(10, 51)))] for _ in range(batch)]
    src_path = os.path.join(os.path.dirname(mdir), "opus_sources.json")
    json.dump(srcs, open(src_path, "w"))                             # the reference appends </s> itself (add_source_eos)
    cmd = [sys.executable, os.path.join(ROOT, "tools", "ref_cuda_worker.py"), "translate-bench", mdir, "int8_float16",
           src_path, str(beam), str(max_len)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    line = [l for l in r.stdout.splitlines() if l.startswith("{")]
    out = {"ref_cuda": json.loads(line[-1]) if (r.returncode == 0 and line) else {"error": (r.stderr or r.stdout)[-300:]}}
    if "tokens_per_s" in out["ref_cuda"]:
        out["vs_ref_cuda"] = round(rec["e2e_tokens_per_s"] / out["ref_cuda"]["tokens_per_s"], 2)
    return out


class TpWatchdog:
    """Bounds the tensor-parallel side record of `--gpus N`.  Its collectives are spin waits on peer flags inside kernels
    (tp_rows.cu), so a rank that raised — or a world size the kernels misbehave at — blocks the other ranks on the device,
    where no Python exception can reach them.  On expiry (or fire()) rank 0 prints the line it already holds, with the reason
    under `tp.error`, and the process leaves with os._exit(0) (a blocked CUDA call cannot be unwound)."""

    def __init__(self, seconds, line):
        self.line, self.seconds = line, seconds
        self._done = threading.Event()
        self._lock = threading.Lock()
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()

    def _run(self):
        if not self._done.wait(self.seconds):
            self.fire("tensor-parallel record timed out after %.0f s (watchdog)" % self.seconds)

    def fire(self, why):
        with self._lock:
            if self._done.is_set():
                return
            self._done.set()
            if self.line is not None:
                self.line["tp"] = {"error": why[-300:]}
                self.line.setdefault("roofline", {"error": "not measured: the tensor-parallel record before it did not finish"})
                sys.stdout.write(json.dumps(self.line) + "\n")
                sys.stdout.flush()
            sys.stderr.write("bench.py: %s; leaving\n" % why)
            sys.stderr.flush()
            os._exit(0)

    def cancel(self):
        self._done.set()


def measure_variant(ct2, torch, name, weights, batch, plen, steps, warmup, device_index, peak, with_ref_cuda):
    """One point of the metric: device-timed decode of `steps` steps after the `plen`-token prompt."""
    awq = weights == "awq"
    quant = "awq_gemm" if awq else "int8_float16"
    gen = ct2.Generator(model_dir(name, quant), device_index=device_index, compute_type="float16" if awq else "int8_float16",
                        max_batch_size=batch, max_length=plen + steps + warmup + 16)
    pre_ms, dec_ms, launches = gen.bench_decode(batch, plen, steps, warmup)
    gen.close()
    del gen
    torch.cuda.empty_cache()
    ms = dec_ms / steps
    sb = step_bytes(name, batch, plen + steps / 2.0, weights)
    rec = {"ms_per_step": round(ms, 4), "tokens_per_s": round(batch / (ms * 1e-3), 1), "steps": steps,
           "context": "%d -> %d" % (plen, plen + steps), "prefill_ms": round(pre_ms, 2),
           "launches_per_step": int(launches // steps), "step_bytes_algorithmic": int(sb),
           "step_roofline_frac": round(sb / (ms * 1e-3) / 1e9 / peak, 4)}
    if with_ref_cuda:
        r = ref_cuda_bench(name, quant, "float16" if awq else "int8_float16", batch, plen)
        rec["ref_cuda"] = r
        if "decode_tokens_per_s" in r:
            rec["vs_ref_cuda"] = round(rec["tokens_per_s"] / r["decode_tokens_per_s"], 2)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    # default = the named workload: 1024 generated tokens after the 1024-token prompt ("seq 2048"); a few seconds on an H100
    ap.add_argument("--steps", type=int, default=1024)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--impl", default="ours")
    ap.add_argument("--model", default="8b", choices=list(MODELS))
    ap.add_argument("--prompt-len", type=int, default=PROMPT_LEN)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write what the last timed decode step computed (logits [batch, vocab], float32) to DIR/logits.npy")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-graph", action="store_true")
    ap.add_argument("--no-variants", action="store_true", help="skip the INT8/AWQ x bsz 1/32 sub-records and ref_cuda")
    ap.add_argument("--no-tp", action="store_true", help="N > 1: skip the tensor-parallel record")
    ap.add_argument("--side-budget", type=float, default=240.0,
                    help="seconds the variants / translate side records may spend before they stop launching reference CUDA runs")
    ap.add_argument("--weights", default="int8", choices=["int8", "awq"],
                    help="int8 = the headline INT8 configuration; awq = the AWQ-INT4 (group 128, AWQ_GEMM layout) variant")
    ap.add_argument("--tp-timeout", type=float, default=300.0,
                    help="N > 1: seconds the tensor-parallel side record may take before the replica line is printed without it")
    ap.add_argument("--tp", action="store_true",
                    help="N > 1: ONE tensor-parallel generator over the N GPUs (strong scaling) as the headline instead of N replicas")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    K, W, B, P = args.steps, max(3, args.warmup), args.batch, args.prompt_len
    awq = args.weights == "awq"
    config = {"workload": "%s generate_batch %s, greedy, bsz %d, prompt %d + %d generated "
                          "(BASELINE.json configs[2])" % (NAMES[args.model], "AWQ-INT4 g128 (float16)" if awq else
                                                          "INT8 (int8_float16)", B, P, K),
              "global_batch": B * (1 if args.tp else max(1, world)), "prompt_len": P,
              "parallelism": ("tp%d (heads / FFN columns sharded, collectives fused into kernels over NVLink peer memory)" % world)
              if args.tp and world > 1 else "dp%d (replicas, no collective)" % world,
              "l2": "every step streams %.1f GB of weights (> 50 MB L2) — no flush needed" % (step_bytes(args.model, 0, 0, args.weights) / 1e9)}

    if args.impl == "reference":
        if args.dump_outputs:
            ap.error("--dump-outputs records the GPU path; it has no meaning with --impl reference")
        if rank != 0:
            return
        r = reference_cpu(args.model, B, K, W)
        if r is None:
            print(json.dumps({"impl": "reference", "unavailable": "oracle/_ref is not built (make -f oracle/Makefile.ref)"}))
            return
        # the CPU arm runs a BOUNDED sample of the workload: say so in the label the driver compares
        config["workload"] = ("%s generate_batch INT8 (int8, Ruy), greedy, bsz %d, bounded sample: prompt 8 + %d generated "
                              "(BASELINE.json configs[2] has prompt %d + %d generated)" % (NAMES[args.model], B, r["steps"], P, K))
        config["prompt_len"] = 8
        config["parallelism"] = "host cores (%d threads)" % r["cores"]
        line = {"impl": "reference", "metric": "generate_batch tokens/sec", "value": round(r["value"], 3),
                "unit": "tokens/s", "n_gpus": 0, "steps": r["steps"], "warmup": W,
                "ms_per_step": round(1e3 * r["seconds"] / r["steps"], 3), "higher_is_better": True, "scaling": "weak",
                "vs_baseline": None, "dtype": "s8 (int8 weights/activations, fp32 epilogue)", "data": "synthetic",
                "config": config, "cpu_baseline": {k: r[k] for k in ("value", "unit", "cores", "kind", "sample")},
                "e2e": {"value": round(r["value"], 3), "unit": "tokens/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
        print(json.dumps(line))
        return

    import numpy as np
    import torch
    import ctranslate2_b200 as ct2
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    torch.cuda.set_device(local_rank)
    quant = "awq_gemm" if awq else "int8_float16"
    mdir = model_dir(args.model, quant) if local_rank == 0 else None
    if world > 1:
        torch.distributed.barrier()
        mdir = model_dir(args.model, quant)
    max_len = P + max(K, 8) + W + 8
    tp = args.tp and world > 1
    gen = ct2.Generator(mdir, device_index=local_rank, compute_type="float16" if awq else "int8_float16", max_batch_size=B,
                        max_length=max(max_len, P + 1024 + 16) if not tp else max_len, use_cuda_graph=not args.no_graph,
                        tensor_parallel=tp)
    units = 1 if tp else world             # independent batches processed per step
    info = gen.info()

    def sync_all():
        torch.cuda.synchronize()
        if world > 1:
            torch.distributed.barrier()
            torch.cuda.synchronize()

    def max_over_ranks(*vals):
        t = torch.tensor(list(vals), device="cuda", dtype=torch.float64)
        if world > 1:
            torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
        return [float(v) for v in t]

    # ---- device-timed decode (inputs resident), K steps after W warm-up steps ----
    sync_all()
    with ClockSampler(local_rank) as clocks:
        pre_ms, dec_ms, launches = gen.bench_decode(B, P, K, W)
        sync_all()
    if args.dump_outputs and rank == 0:
        # the prompt ids are a fixed function of their position, so two builds see identical inputs
        os.makedirs(args.dump_outputs, exist_ok=True)
        np.save(os.path.join(args.dump_outputs, "logits.npy"), gen.bench_last_logits(B, MODELS[args.model]["vocab_size"]))
    dec_ms, pre_ms = max_over_ranks(dec_ms, pre_ms)
    value = B * K * units / (dec_ms * 1e-3)

    # ---- end to end through the public API with host buffers ----
    prompts = prompts_for(args.model, B, P, seed=42 + (0 if tp else rank))
    gen.generate_batch(prompts[:, :8].tolist(), max_length=2, min_length=2, end_token=[0])   # warm the small path

    def e2e_run(tokens):
        sync_all()
        t0 = time.perf_counter()
        res = gen.generate_batch(prompts, max_length=tokens, min_length=tokens, end_token=[1])
        torch.cuda.synchronize()
        sec = time.perf_counter() - t0
        assert all(len(r.sequences_ids[0]) == tokens for r in res)
        sec, = max_over_ranks(sec)
        return {"value": round(B * tokens * units / sec, 2), "unit": "tokens/s", "h2d_bytes_per_step": round(B * P * 4 / tokens, 1),
                "d2h_bytes_per_step": B * 4, "seconds": round(sec, 4), "generated_tokens_per_sequence": tokens,
                "includes": "prompt H2D + prefill(P-1) + %d decode steps + ids D2H" % tokens}

    e2e = e2e_run(K)
    e2e_full = e2e if K == 1024 else (e2e_run(1024) if not tp else None)

    # ---- the replica / single-GPU line is complete here; rank 0 keeps it so that a failing side record cannot lose it ----
    line = None
    if rank == 0:
        peak, how = measured_peaks()
        ctx_mean = P + K / 2.0
        sb = step_bytes(args.model, B, ctx_mean, args.weights)
        step_gbs = sb / (dec_ms / K * 1e-3) / 1e9
        config.update({"step_bytes_algorithmic": int(sb), "step_GBps": round(step_gbs, 1),
                       "step_roofline_frac": round(step_gbs / peak, 4), "prefill_ms": round(pre_ms, 2),
                       "prefill_tokens_per_s": round(B * (P - 1) / (pre_ms * 1e-3), 1), "weight_bytes": info["weight_bytes"]})
        line = {"metric": "generate_batch tokens/sec", "value": round(value, 2), "unit": "tokens/s", "n_gpus": world,
                "steps": K, "warmup": W, "ms_per_step": round(dec_ms / K, 4), "higher_is_better": True,
                "scaling": "strong" if tp else "weak", "vs_baseline": None,
                "dtype": ("s4 weights -> f16 (wgmma f16, f32 accumulate)" if awq else
                          "s8 (int8 x int8 -> s32 on wgmma; f16 activations, f32 epilogue/softmax)"),
                "data": "synthetic", "config": config, "clocks": clocks.summary(), "e2e": e2e,
                "gpu_launches": int(launches)}
        if e2e_full is not None:
            line["e2e_full"] = e2e_full

    # ---- N > 1: ONE tensor-parallel generator over the same GPUs (strong scaling of the same step) ----
    # The collectives of that generator are spin waits on peer flags inside kernels: a rank that fails (or a world size the
    # fused kernels were never run at) would leave the others waiting forever and the driver without ANY line.  A watchdog
    # bounds the section: on expiry rank 0 prints the replica line with the failure recorded and every rank exits.
    tp_rec = None
    if world > 1 and not tp and not args.no_tp:
        watchdog = TpWatchdog(args.tp_timeout, line)
        gen.close()
        del gen
        torch.cuda.empty_cache()
        torch.distributed.barrier()
        try:
            tgen = ct2.Generator(mdir, device_index=local_rank, compute_type="float16" if awq else "int8_float16",
                                 max_batch_size=B, max_length=max_len, use_cuda_graph=not args.no_graph, tensor_parallel=True)
            sync_all()
            tpre, tdec, tl = tgen.bench_decode(B, P, K, W)
            sync_all()
            tdec, tpre = max_over_ranks(tdec, tpre)
            m = MODELS[args.model]
            d = m["num_heads"] * m["head_dim"]
            # per layer two reduced [B, d] tensors pulled from world-1 peers, plus two 8-byte {epoch, amax} words per row
            nvl = m["num_layers"] * 2 * (world - 1) * B * (d * 2 + 8)
            tp_rec = {"parallelism": "tp%d" % world, "scaling": "strong", "ms_per_step": round(tdec / K, 4),
                      "tokens_per_s": round(B * K / (tdec * 1e-3), 1), "prefill_ms": round(tpre, 2),
                      "speedup_vs_one_gpu_step": round((dec_ms / K) / (tdec / K), 3),
                      "nvlink_bytes_per_step_per_gpu": int(nvl), "launches_per_step": int(tl // K)}
            tgen.close()
        except Exception as ex:
            tp_rec = {"error": str(ex)[-300:]}
            # the peers of a failed rank wait for it inside a kernel: do not leave them (and the driver) hanging
            if "timed out" not in tp_rec["error"]:
                watchdog.fire("rank %d: %s" % (rank, tp_rec["error"]))
        try:
            sync_all()                        # every rank has left the section (a stuck peer trips the watchdog instead)
        finally:
            watchdog.cancel()
        gen = None

    if rank != 0:
        return
    if tp_rec is not None:
        line["tp"] = tp_rec
    if gen is not None:
        gen.close()
        del gen
    torch.cuda.empty_cache()
    try:
        line["roofline"] = awq_roofline(args.model, B, "cuda") if awq else gemm_roofline(args.model, B, "cuda")
    except Exception as ex:  # keep the headline even if the side measurement fails
        line["roofline"] = {"error": str(ex)}
    if world == 1 and not args.no_variants:
        # the four points BASELINE.json's metric names (device-timed, always), then the OPUS-MT-shaped translation record, then
        # the reference's own CUDA build beside each of them for as long as the side budget lasts (most important first)
        t_side = time.time()
        variants = {}
        for wname in ("int8", "awq"):
            for b in (1, 32):
                key = "%s_b%d" % (wname, b)
                try:
                    variants[key] = measure_variant(ct2, torch, args.model, wname, b, P, 64, W, local_rank, peak, False)
                except Exception as ex:
                    variants[key] = {"error": str(ex)[-300:]}
        line["variants"] = variants
        try:
            line["translate"] = translate_record(local_rank, False)
        except Exception as ex:
            line["translate"] = {"error": str(ex)[-300:]}
        for key in ("int8_b32", "awq_b32", "int8_b1", "awq_b1"):
            if time.time() - t_side > args.side_budget or "error" in variants[key]:
                variants[key].setdefault("ref_cuda", {"skipped": "side budget of %.0f s used up" % args.side_budget})
                continue
            wname, b = key.split("_b")
            quant = "awq_gemm" if wname == "awq" else "int8_float16"
            r = ref_cuda_bench(args.model, quant, "float16" if wname == "awq" else "int8_float16", int(b), P)
            variants[key]["ref_cuda"] = r
            if "decode_tokens_per_s" in r:
                variants[key]["vs_ref_cuda"] = round(variants[key]["tokens_per_s"] / r["decode_tokens_per_s"], 2)
        if "error" not in line["translate"] and time.time() - t_side <= args.side_budget:
            try:
                line["translate"].update(translate_reference(line["translate"]))
            except Exception as ex:
                line["translate"]["ref_cuda"] = {"error": str(ex)[-300:]}
        # SURVEY §8 a13: the reference's best attention (vendored FlashAttention-2 split-KV, flash_attention=True) on the headline
        # point, last in the side budget (with the cuBLAS GEMMs around it the reference's step is not attention-bound)
        for key in ("int8_b32", "int8_b1"):
            if time.time() - t_side > args.side_budget or "error" in variants[key]:
                continue
            r = ref_cuda_bench(args.model, "int8_float16", "int8_float16", int(key.split("_b")[1]), P, flash=True)
            variants[key]["ref_cuda_flash"] = r
            if "decode_tokens_per_s" in r:
                variants[key]["vs_ref_cuda_flash"] = round(variants[key]["tokens_per_s"] / r["decode_tokens_per_s"], 2)
    if awq:
        line["cpu_baseline"] = {"value": None, "unit": "tokens/s", "cores": 0, "kind": "reference",
                                "sample": "none: the reference has no CPU implementation of the AWQ ops "
                                          "(src/ops/awq/gemm_cpu.cc, gemv_cpu.cc, dequantize_cpu.cc throw)"}
    elif world == 1 and not args.no_cpu_baseline:
        r = reference_cpu(args.model, B, 64, 1, budget_s=25.0, calibrate=False)
        line["cpu_baseline"] = ({k: r[k] for k in ("value", "unit", "cores", "kind", "sample")} if r else
                                {"value": None, "kind": "reference", "sample": "oracle/_ref not built"})
    print(json.dumps(line))


if __name__ == "__main__":
    main()
