#!/usr/bin/env python
"""Whisper.align on a Whisper-small-shaped synthetic model (converters/synthetic.py: 12 + 12 layers, d 768, 12 heads, 80 mel
bins, 1500 encoder positions, INT8 weights, int8_float16), 8 windows of 3000 input frames x 120 text tokens, 6 alignment
heads across the upper decoder layers, median filter width 7.  The model is written to a temporary directory.  Prints one
JSON line with

  * align_ms: host clock around align (the call ends with a device synchronise), median of --repeats after a warm-up;
  * dtw_ms / dtw_share: the host DTW of the same 8 matrices (ct2b200_negative_dtw_host, the function align runs), and its
    share of align_ms;
  * encode_ms: for context, Whisper.encode of the same batch (host clock, includes the copy of the output to the host);
  * ref_cuda: null unless oracle/_ref_cuda is built (no timing task for the reference's align exists);
  * the card's name and power limit, read in the same run.

usage: python tools/whisper_align_bench.py [--repeats 5]"""
import argparse
import ctypes
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    import numpy as np
    from ctranslate2_b200._lib import check, lib
    from ctranslate2_b200.converters.synthetic import WhisperConfig, write_whisper_model
    from ctranslate2_b200.whisper import Whisper
    cfg = WhisperConfig(encoder_layers=12, decoder_layers=12, num_heads=12, d_model=768, n_mels=80, max_source_positions=1500,
                        max_target_positions=448, text_tokens=50257, languages=99, timestamps=1501)
    with tempfile.TemporaryDirectory() as tmp:
        mdir = os.path.join(tmp, "whisper_small_shaped")
        write_whisper_model(mdir, cfg, "int8_float16", seed=11)
        conf = json.load(open(os.path.join(mdir, "config.json")))
        conf["alignment_heads"] = [[5, 3], [6, 9], [8, 2], [9, 7], [10, 0], [11, 4]]
        json.dump(conf, open(os.path.join(mdir, "config.json"), "w"))
        w = Whisper(mdir, compute_type="int8_float16")
        rng = np.random.default_rng(5)
        x = (rng.standard_normal((8, 80, 3000)) * 2).astype(np.float32)
        texts = [[int(t) for t in rng.integers(0, 50257, size=120)] for _ in range(8)]
        start = [w.sot_id, w.sot_id + 1, w.sot_id + 101]          # <|startoftranscript|>, first language, <|transcribe|>
        res, matrix = w._align(x, start, texts, 3000, 7, return_matrix=True)     # warm-up: arena growth, first launches
        assert all(len(r.alignments) >= 1500 for r in res)
        times = []
        for _ in range(a.repeats):
            t0 = time.perf_counter()
            w.align(x, start, texts, 3000)
            times.append((time.perf_counter() - t0) * 1e3)
        dtw = []
        out = np.zeros((121 + 1500, 2), np.int32)
        n = ctypes.c_int32()
        p = ctypes.c_void_p
        for _ in range(a.repeats):
            t0 = time.perf_counter()
            for b in range(8):
                m = np.ascontiguousarray(matrix[b, :121, :1500])
                check(lib().ct2b200_negative_dtw_host(m.ctypes.data_as(p), ctypes.c_int64(121), ctypes.c_int64(1500),
                                                      out.ctypes.data_as(p), ctypes.byref(n)))
            dtw.append((time.perf_counter() - t0) * 1e3)
        enc = []
        for _ in range(a.repeats):
            t0 = time.perf_counter()
            w.encode(x)
            enc.append((time.perf_counter() - t0) * 1e3)
        w.close()
    align_ms, dtw_ms = statistics.median(times), statistics.median(dtw)
    ref_cuda = None
    if os.path.exists(os.path.join(ROOT, "oracle", "_ref_cuda", "libct2ref_cuda_driver.so")):
        ref_cuda = {"unavailable": "the reference's CUDA driver (oracle/ref_driver.cc) exposes no Whisper::align entry"}
    rec = {"workload": "Whisper.align, Whisper-small-shaped synthetic model INT8 (int8_float16), 8 windows x 3000 frames x 120 "
                       "text tokens, 6 alignment heads, width 7",
           "align_ms": round(align_ms, 2), "align_ms_min_max": [round(min(times), 2), round(max(times), 2)],
           "dtw_ms": round(dtw_ms, 2), "dtw_share": round(dtw_ms / align_ms, 3),
           "encode_ms": round(statistics.median(enc), 2), "repeats": a.repeats, "ref_cuda": ref_cuda}
    rec.update(card())
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
