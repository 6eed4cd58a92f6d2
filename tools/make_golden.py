#!/usr/bin/env python
"""Generates the committed fixtures under tests/golden/ from the reference itself.

Run in the build container (needs /root/reference and oracle/_ref built by oracle/Makefile.ref):

    python tools/make_golden.py

1. tests/golden/ref_gtest_vectors.json — the golden vectors the reference's own gtests hold for
   this path, extracted verbatim (by parsing, not by hand) from /root/reference/tests/ops_test.cc and
   layers_test.cc: every `StorageView name({shape}, std::vector<T>{...})` inside the named TEST_P blocks.
2. tests/golden/tiny_llama_int8/ — a 2-layer GQA/SwiGLU/RoPE decoder written by the REFERENCE's
   python spec writer (python/ctranslate2/specs), quantization="int8".
3. tests/golden/tiny_llama_int8_ref.npz — outputs of the UNMODIFIED reference (oracle/_ref, CPU):
   forward logits for a seeded prompt batch and greedy generate_batch tokens.
4. tests/golden/ref_ops_random.npz — reference op outputs (Quantize, Gemm s8, Dequantize, RMSNorm,
   Rotary, SoftMax, TopK, Gather) on seeded random inputs.

Nothing here runs at test time on the GPU box; the tests read only the files this script wrote.
"""
import json
import os
import re
import shutil
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
OUT = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)

GTESTS = {
    "ops_test.cc": ["GemmInt8", "TopK", "TopKVariableDepth", "TopKChangeK", "SoftMax", "LogSoftMax",
                    "MaskedSoftMax", "RMSNorm", "LayerNorm", "QuantizeINT8", "QuantizeINT8ZeroRow", "Swish", "ReLU",
                    "GELU", "GELUTanh", "GELUSigmoid", "Gemm", "GemmBias", "GemmResidual", "GemmGELU",
                    "GatherData1D", "GatherData1DIndex2D", "GatherData2D", "GatherData3D",
                    "GatherData2DIndex2D", "BiasAddGELU", "BiasAddAxisGELU"],
    "layers_test.cc": ["RotaryEmbedding"],
}


STATICS = ("gemm_a", "gemm_b", "gemm_y", "bias_value", "bias_bias")


def extract_gtest_vectors():
    out = {}
    sv = re.compile(r"StorageView\s+(\w+)\s*(?:=\s*StorageView)?\((\{[^}]*\}|\w+\.shape\(\)),\s*std::vector<(\w+)>\s*\{([^}]*)\}", re.S)
    for fname, names in GTESTS.items():
        text = open(os.path.join(REF, "tests", fname)).read()
        for name in names:
            m = re.search(r"TEST_P\(\w+,\s*%s\)\s*\{" % re.escape(name), text)
            if not m:
                print("  (no such test in this reference version: %s)" % name)
                continue
            nxt = re.search(r"\nTEST(_P|_F)?\(", text[m.end():])
            body = text[m.end(): m.end() + (nxt.start() if nxt else len(text))]
            items = []
            for v in sv.finditer(body):
                if v.group(2).startswith("{"):
                    shape = [int(s) for s in v.group(2).strip("{}").split(",") if s.strip()]
                else:   # `other.shape()`: same shape as the named vector of this test
                    other = v.group(2).split(".")[0]
                    shape = next(i["shape"] for i in items if i["name"] == other)
                vals = [float(t.rstrip("f")) for t in re.split(r"[,\s]+", v.group(4).strip()) if t]
                items.append({"name": v.group(1), "shape": shape, "ctype": v.group(3), "values": vals})
            out[name] = items
            print("  %-24s %d vectors" % (name, len(items)))
        # file-scope inputs shared by several tests (`static const StorageView gemm_a(...)`)
        static = re.compile(r"static const StorageView\s+(\w+)\((\{[^}]*\}),\s*std::vector<(\w+)>\s*\{([^}]*)\}", re.S)
        for v in static.finditer(text):
            if v.group(1) in STATICS:
                shape = [int(t) for t in v.group(2).strip("{}").split(",") if t.strip()]
                vals = [float(t.rstrip("f")) for t in re.split(r"[,\s]+", v.group(4).strip()) if t]
                out.setdefault("_static", []).append({"name": v.group(1), "shape": shape, "ctype": v.group(3), "values": vals})
                print("  static %-17s %s" % (v.group(1), shape))
    return out


def make_tiny_model(model_dir):
    sys.path.insert(0, os.path.join(REF, "python"))
    from ctranslate2.specs import common_spec, transformer_spec
    L, H, Hkv, D, F, V = 2, 4, 2, 32, 256, 200
    d = H * D
    spec = transformer_spec.TransformerDecoderModelSpec.from_config(
        L, H, activation=common_spec.Activation.SWISH, pre_norm=True, ffn_glu=True, rms_norm=True,
        rotary_dim=0, rotary_interleave=False, rotary_base=500000.0, num_heads_kv=Hkv)
    rng = np.random.default_rng(1234)

    def lin(s, n, k):
        s.weight = (rng.standard_normal((n, k)) * 0.05).astype(np.float32)

    dec = spec.decoder
    dec.scale_embeddings = False
    dec.embeddings.weight = (rng.standard_normal((V, d)) * 0.05).astype(np.float32)
    dec.layer_norm.gamma = (1 + 0.1 * rng.standard_normal(d)).astype(np.float32)
    for l in dec.layer:
        l.self_attention.layer_norm.gamma = (1 + 0.1 * rng.standard_normal(d)).astype(np.float32)
        l.ffn.layer_norm.gamma = (1 + 0.1 * rng.standard_normal(d)).astype(np.float32)
        lin(l.self_attention.linear[0], d + 2 * Hkv * D, d)
        lin(l.self_attention.linear[1], d, d)
        lin(l.ffn.linear_0, F, d)
        lin(l.ffn.linear_0_noact, F, d)
        lin(l.ffn.linear_1, d, F)
    lin(dec.projection, V, d)
    spec.register_vocabulary(["<t%d>" % i for i in range(V)])
    spec.config.bos_token = "<t1>"
    spec.config.eos_token = "<t2>"
    spec.config.unk_token = "<t0>"
    spec.config.layer_norm_epsilon = 1e-5
    spec.validate()
    spec.optimize(quantization="int8")
    shutil.rmtree(model_dir, ignore_errors=True)
    os.makedirs(model_dir)
    spec.save(model_dir)
    return V


def make_scores_fixture():
    """GenerationResult.scores of the unmodified reference on the committed tiny model (return_scores=true): sum of the
    chosen tokens' log-probabilities / length^length_penalty, incl. rows that end on the end token."""
    from oracle import refapi
    assert refapi.available(), "build oracle/_ref first: make -f oracle/Makefile.ref -j8"
    mdir = os.path.join(OUT, "tiny_llama_int8")
    fx = np.load(os.path.join(OUT, "tiny_llama_int8_ref.npz"), allow_pickle=True)
    prompts = fx["prompts"]
    g = refapi.RefGenerator(mdir, "int8", 4)
    gm = fx["generated_min12"]
    # end tokens that rows emit at different positions: rows then stop at step 0, mid-sequence, or never
    ends = [2, int(gm[0][3]), int(gm[1][2]), int(gm[2][5])]
    cases = []
    for lp in (1.0, 0.0, 0.6):
        for end in ends:
            for (mx, mn) in ((12, 12), (12, 0), (12, 3)):
                toks, scores = g.generate_with_scores(prompts, mx, mn, end, lp)
                cases.append({"max_length": mx, "min_length": mn, "end_id": end, "length_penalty": lp, "tokens": toks,
                              "scores": [float(x) for x in scores]})
    beams = []
    for beam in (2, 4):
        for lp in (1.0, 0.0):
            for end in ends[:3]:
                for (mx, mn, nh, pat) in ((10, 0, 2, 1.0), (10, 3, 2, 2.0), (6, 6, 1, 1.0)):
                    r = g.generate_beam(prompts, beam, mx, mn, end, lp, nh, pat)
                    beams.append({"beam_size": beam, "max_length": mx, "min_length": mn, "end_id": end,
                                  "length_penalty": lp, "num_hypotheses": nh, "patience": pat,
                                  "hypotheses": [[[t, sc] for t, sc in row] for row in r]})
    g.close()
    with open(os.path.join(OUT, "tiny_llama_int8_scores.json"), "w") as f:
        json.dump({"prompts": prompts.tolist(), "cases": cases, "beam_cases": beams}, f)
    print("wrote tiny_llama_int8_scores.json (%d greedy cases, %d beam cases)" % (len(cases), len(beams)))


def make_processors_fixture():
    """Greedy generate_batch of the unmodified reference with the logits processors of GenerationOptions (repetition_penalty,
    no_repeat_ngram_size, disable_unk, suppress_sequences) on the committed tiny model — it repeats tokens a lot, which is
    exactly what these options act on."""
    from oracle import refapi
    assert refapi.available(), "build oracle/_ref first: make -f oracle/Makefile.ref -j8"
    mdir = os.path.join(OUT, "tiny_llama_int8")
    fx = np.load(os.path.join(OUT, "tiny_llama_int8_ref.npz"), allow_pickle=True)
    prompts = fx["prompts"]
    gm = fx["generated_min12"]
    g = refapi.RefGenerator(mdir, "int8", 4)
    options = [dict(repetition_penalty=1.3), dict(repetition_penalty=0.7), dict(repetition_penalty=2.0, no_repeat_ngram_size=3),
               dict(no_repeat_ngram_size=1), dict(no_repeat_ngram_size=2), dict(no_repeat_ngram_size=4), dict(disable_unk=True),
               dict(suppress_sequences=[[int(gm[0][0])]]),
               dict(suppress_sequences=[[int(gm[0][0])], [int(gm[1][0]), int(gm[1][1])], [int(gm[2][1]), int(gm[2][2]), int(gm[2][3])]]),
               dict(suppress_sequences=[[int(gm[1][4]), int(gm[1][5])]], repetition_penalty=1.2, no_repeat_ngram_size=2)]
    cases = []
    for opt in options:
        for (mx, mn, end) in ((12, 12, 2), (12, 0, int(gm[0][4])), (10, 3, int(gm[1][2]))):
            toks, scores = g.generate_processors(prompts, mx, mn, end, **opt)
            cases.append({"max_length": mx, "min_length": mn, "end_id": end, "options": opt, "tokens": toks,
                          "scores": [float(x) for x in scores]})
    g.close()
    with open(os.path.join(OUT, "tiny_llama_int8_processors.json"), "w") as f:
        json.dump({"prompts": prompts.tolist(), "cases": cases}, f)
    print("wrote tiny_llama_int8_processors.json (%d cases)" % len(cases))


def make_ragged_fixture():
    """Greedy generate_batch of the unmodified reference over prompts of different lengths (include_prompt_in_result=false):
    the shortest prompt decides how much is forwarded at once, the rest of each prompt is forced through the loop
    (language_model.cc:217-238).  Also records the reference's behaviour when the shortest prompt is ONE token: it then keeps
    return_prefix = true and returns the forced prompt tokens as part of the result."""
    from oracle import refapi
    assert refapi.available(), "build oracle/_ref first: make -f oracle/Makefile.ref -j8"
    g = refapi.RefGenerator(os.path.join(OUT, "tiny_llama_int8"), "int8", 4)
    batches = [[[5, 9, 11, 40, 7], [8, 3, 77], [100, 23, 45, 67]],
               [[17, 4], [9, 9, 9, 9, 9, 9, 9], [150, 3, 8]],
               [[5, 9, 11, 40, 7], [8], [100, 23]],
               [[5], [8], [100]]]
    cases = []
    for prompts in batches:
        for (mx, mn, end) in ((6, 6, 2), (6, 0, 164), (5, 2, 18), (8, 3, 143)):
            toks, scores = g.generate_ragged(prompts, mx, mn, end)
            cases.append({"prompts": prompts, "max_length": mx, "min_length": mn, "end_id": end, "tokens": toks,
                          "scores": [float(x) for x in scores]})
    g.close()
    with open(os.path.join(OUT, "tiny_llama_int8_ragged.json"), "w") as f:
        json.dump({"cases": cases}, f)
    print("wrote tiny_llama_int8_ragged.json (%d cases)" % len(cases))


def make_score_fixture():
    """Generator::score_batch of the unmodified reference on the tiny model: log-probability of every token given its prefix,
    ragged batch, sequences too short to score, ScoringOptions::offset."""
    from oracle import refapi
    assert refapi.available(), "build oracle/_ref first: make -f oracle/Makefile.ref -j8"
    g = refapi.RefGenerator(os.path.join(OUT, "tiny_llama_int8"), "int8", 4)
    rng = np.random.default_rng(11)
    seqs = [[int(t) for t in rng.integers(3, 200, size=n)] for n in (12, 2, 1, 30, 7, 19)]
    cases = [{"sequences": seqs, "offset": off, "log_probs": g.score(seqs, off)} for off in (0, 1, 5)]
    g.close()
    with open(os.path.join(OUT, "tiny_llama_int8_score_batch.json"), "w") as f:
        json.dump({"cases": cases}, f)
    print("wrote tiny_llama_int8_score_batch.json (%d cases)" % len(cases))


SEQ2SEQ_CASES = [  # (beam, num_hypotheses, length_penalty, max_length, min_length)
    (1, 1, 1.0, 16, 1), (2, 2, 1.0, 16, 1), (4, 2, 0.0, 16, 1), (3, 3, 0.6, 12, 1), (4, 4, 1.0, 14, 9), (2, 1, 1.0, 5, 1)]


def seq2seq_sources(seed, cases, lo, hi):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(cases):
        batch = int(rng.integers(1, 5))
        out.append([[int(x) for x in rng.integers(lo, hi, size=int(rng.integers(2, 10)))] for _ in range(batch)])
    return out


def make_seq2seq_fixture():
    """Encoder-decoder path (SURVEY §8 f1): outputs of the UNMODIFIED reference's Translator (oracle/_ref, CPU) on
    (a) the reference's own golden model tests/data/models/v2/aren-transliteration-i8 (tests/translator_test.cc:53-96), copied
        to tests/golden/ as a data fixture (binary version 2: the activation quantizer truncates), and
    (b) a post-norm / Swish / start-from-zero-embedding model written by converters/synthetic.py (the OPUS-MT recipe in small),
    in float32 (no activation quantization: every token must agree) and int8."""
    from ctranslate2_b200.converters.synthetic import TransformerConfig, write_transformer_model
    from oracle import refapi
    src_dir = os.path.join(REF, "tests", "data", "models", "v2", "aren-transliteration-i8")
    aren = os.path.join(OUT, "aren-transliteration-i8")
    if os.path.isdir(aren):
        shutil.rmtree(aren)
    shutil.copytree(src_dir, aren)
    for root, _, files in os.walk(aren):          # the reference tree is read-only: the copy must not be
        os.chmod(root, 0o755)
        for name in files:
            os.chmod(os.path.join(root, name), 0o644)
    post = os.path.join(OUT, "tiny_seq2seq_postnorm")
    cfg = TransformerConfig(encoder_layers=2, decoder_layers=2, num_heads=4, d_model=64, ffn_dim=128, source_vocab=120,
                            target_vocab=96, pre_norm=False, activation=2, start_from_zero_embedding=True)
    write_transformer_model(post, cfg, "int8", seed=7)
    fixture = {}
    for name, mdir, lo, hi in (("aren", aren, 4, 51), ("postnorm", post, 3, 120)):
        entry = {"models": {}}
        for compute in ("float32", "int8"):
            t = refapi.RefTranslator(mdir, compute, 2)
            cases = []
            for ci, (beam, nh, lp, mx, mn) in enumerate(SEQ2SEQ_CASES):
                for srcs in seq2seq_sources(100 + ci, 4, lo, hi):
                    res = t.translate(srcs, beam_size=beam, num_hypotheses=nh, max_length=mx, min_length=mn, length_penalty=lp)
                    cases.append({"sources": srcs, "beam_size": beam, "num_hypotheses": nh, "length_penalty": lp,
                                  "max_length": mx, "min_length": mn,
                                  "hypotheses": [[h[0] for h in r] for r in res], "scores": [[h[1] for h in r] for r in res]})
            srcs = seq2seq_sources(9, 1, lo, hi)[0] + [[lo + 1, lo + 2, lo + 3, lo + 4, lo + 5, lo + 6, lo + 7]]
            memory, lens = t.encode(srcs)
            d = 32 if name == "aren" else 64
            S = max(len(r) for r in srcs)
            memory = memory.reshape(-1)[:len(srcs) * S * d].reshape(len(srcs), S, d)
            entry["models"][compute] = {"cases": cases, "encode_sources": srcs, "memory": memory.tolist()}
            t.close()
        fixture[name] = entry
    with open(os.path.join(OUT, "seq2seq_ref.json"), "w") as f:
        json.dump(fixture, f)
    print("seq2seq fixture:", sum(len(m["cases"]) for e in fixture.values() for m in e["models"].values()), "cases")


def _ref_translate_score(model_dir, compute, pairs, max_input_length, offset):
    """Translator::score_batch of the unmodified reference (CPU) through tools/ref_translate_score.cc, built by
    tools/ref_translate_score.mk against oracle/_ref/libct2ref.so into a temporary directory: one (tokens, log_probs) per
    (source tokens, target tokens) pair."""
    import subprocess
    import tempfile
    out_dir = os.path.join(tempfile.gettempdir(), "ct2ref_score")
    subprocess.run(["make", "-s", "-f", "tools/ref_translate_score.mk", "score", "SCORE_OUT=" + out_dir], cwd=ROOT, check=True)
    exe = os.path.join(out_dir, "ref_translate_score")
    text = "%s\t%s\t%d\t%d\t0\n" % (model_dir, compute, max_input_length, offset)
    text += "".join(" ".join(s) + "\t" + " ".join(t) + "\n" for s, t in pairs)
    out = subprocess.run([exe], input=text.encode(), capture_output=True, check=True).stdout.decode()
    res = []
    for line in out.split("\n")[:len(pairs)]:
        toks, scores = line.split("\t")
        res.append((toks.split(" ") if toks else [], [float(x) for x in scores.split(" ")] if scores else []))
    assert len(res) == len(pairs)
    return res


def make_translator_score_fixture():
    """Translator::score_batch of the UNMODIFIED reference (oracle/_ref, CPU) on token strings: aren-transliteration in float32,
    aren-transliteration-i8 in int8, and the post-norm / Swish / zero-first-embedding model in float32 and int8.  Ragged
    batches, offsets 0 / 1 / 3, a max_input_length that truncates both sides, an empty source, unknown target tokens (the
    post-norm model's vocabularies hold <unk>; the aren ones do not, and the reference maps unknown tokens past the output
    layer there)."""
    from ctranslate2_b200.translator import _load_vocabulary
    models = [("aren-float32", "aren-transliteration", "float32"), ("aren-int8", "aren-transliteration-i8", "int8"),
              ("postnorm-float32", "tiny_seq2seq_postnorm", "float32"), ("postnorm-int8", "tiny_seq2seq_postnorm", "int8")]
    fixture = {"models": {}}
    for name, mdir, compute in models:
        path = os.path.join(OUT, mdir)
        svocab = _load_vocabulary(path, "source_vocabulary")[3:]
        tvocab = _load_vocabulary(path, "target_vocabulary")[3:]
        svocab = [t for t in svocab if t not in ("<unk>", "<s>", "</s>", "<blank>")]
        tvocab = [t for t in tvocab if t not in ("<unk>", "<s>", "</s>", "<blank>")]
        rng = np.random.default_rng(21)
        pick = lambda vocab, n: [vocab[int(i)] for i in rng.integers(0, len(vocab), size=n)]   # noqa: E731
        ragged = [(pick(svocab, int(a)), pick(tvocab, int(b))) for a, b in zip(rng.integers(1, 14, size=7),
                                                                               rng.integers(0, 14, size=7))]
        edge = [([], pick(tvocab, 4)), (pick(svocab, 5), pick(tvocab, 6)), (pick(svocab, 2), [])]
        if name.startswith("aren"):
            # the pairs the reference's own Python test scores (python/tests/test_translator.py, test_score_api)
            edge.append((["\u0622", "\u062a", "\u0632", "\u0645", "\u0648", "\u0646"], ["a", "t", "z", "m", "o", "n"]))
        else:
            edge.append((pick(svocab, 6), pick(tvocab, 2) + ["not-a-token"] + pick(tvocab, 3) + ["also-unknown"]))
        cases = []
        for pairs, max_len, offset in ((ragged, 1024, 0), (ragged, 1024, 1), (ragged, 1024, 3), (ragged, 5, 0),
                                       (ragged, 5, 1), (edge, 1024, 0), (edge, 1024, 2)):
            res = _ref_translate_score(path, compute, pairs, max_len, offset)
            cases.append({"source": [p[0] for p in pairs], "target": [p[1] for p in pairs], "max_input_length": max_len,
                          "offset": offset, "tokens": [r[0] for r in res], "log_probs": [r[1] for r in res]})
        fixture["models"][name] = {"model": mdir, "compute_type": compute, "cases": cases}
    with open(os.path.join(OUT, "seq2seq_score_ref.json"), "w") as f:
        json.dump(fixture, f, ensure_ascii=False)
    print("translator score fixture:", sum(len(m["cases"]) for m in fixture["models"].values()), "cases")


def ref_translate_processors(model_dir, compute, requests):
    """Translator::translate_batch of the unmodified reference (CPU) with the logits processors, through
    tools/ref_translate_processors.cc, built by tools/ref_translate_processors.mk against oracle/_ref/libct2ref.so into a
    temporary directory.  requests: dicts of sources (token lists), beam_size, num_hypotheses, length_penalty, max_length,
    min_length, repetition_penalty, no_repeat_ngram_size, disable_unk, suppress_sequences (token lists).  Per request: per
    source (hypotheses as token lists, scores), or the reference's error message."""
    import subprocess
    import tempfile
    out_dir = os.path.join(tempfile.gettempdir(), "ct2ref_processors")
    subprocess.run(["make", "-s", "-f", "tools/ref_translate_processors.mk", "processors", "PROC_OUT=" + out_dir], cwd=ROOT,
                   check=True)
    lists = lambda ls: "|".join(" ".join(x) for x in ls)   # noqa: E731
    text = "%s\t%s\n" % (model_dir, compute)
    for r in requests:
        text += "\t".join(str(x) for x in (r["beam_size"], r["num_hypotheses"], r["length_penalty"], r["max_length"],
                                           r["min_length"], r["repetition_penalty"], r["no_repeat_ngram_size"],
                                           int(r["disable_unk"]), lists(r["suppress_sequences"]), lists(r["sources"]))) + "\n"
    lines = subprocess.run([os.path.join(out_dir, "ref_translate_processors")], input=text.encode(), capture_output=True,
                           check=True).stdout.decode().split("\n")
    res, k = [], 0
    for r in requests:
        if lines[k].startswith("ERROR\t"):
            res.append(lines[k].split("\t", 1)[1])
            k += 1
            continue
        entry = []
        for _ in r["sources"]:
            hyps, scores = lines[k].split("\t")
            entry.append(([h.split(" ") if h else [] for h in hyps.split("|")], [float(x) for x in scores.split(" ")]))
            k += 1
        res.append(entry)
    return res


PROCESSOR_BEAMS = [(1, 1), (2, 2), (4, 3), (10, 2)]   # (beam, num_hypotheses); beam 10 takes the LogSoftMax + TopK path


def processor_options(hyp, with_unk):
    """The option sets of the processors fixture: each processor alone, then combinations.  `hyp` is a translation the
    model makes without processors, so the suppressed sequences are ones it would produce."""
    one, two, three = [hyp[0]], hyp[1:3], hyp[2:5]
    opts = [dict(repetition_penalty=1.3), dict(repetition_penalty=0.7), dict(repetition_penalty=100.0),
            dict(no_repeat_ngram_size=1), dict(no_repeat_ngram_size=2), dict(no_repeat_ngram_size=3),
            dict(suppress_sequences=[one]), dict(suppress_sequences=[two]), dict(suppress_sequences=[three, []]),
            dict(suppress_sequences=[one, two, three]),
            dict(repetition_penalty=1.3, no_repeat_ngram_size=2, suppress_sequences=[two]),
            dict(repetition_penalty=0.7, min_length=8),                    # the penalty lands before the min-length mask
            dict(repetition_penalty=0.5, no_repeat_ngram_size=3, min_length=6, suppress_sequences=[one, three])]
    if with_unk:                                    # the aren vocabularies have no <unk>: its id lies past the output layer
        opts += [dict(disable_unk=True), dict(disable_unk=True, repetition_penalty=1.2, suppress_sequences=[["<unk>"], two])]
    return opts


def make_seq2seq_processors_fixture():
    """Translator::translate_batch with repetition_penalty, no_repeat_ngram_size, disable_unk and suppress_sequences, from
    the UNMODIFIED reference (oracle/_ref, CPU), on the models of seq2seq_ref.json (aren-transliteration-i8 and the post-norm
    model) in float32 and int8: ragged batches of token strings, beams 1 / 2 / 4 / 10, each processor alone and combined."""
    from ctranslate2_b200.translator import _load_vocabulary
    fixture = {}
    for name, mdir, lo, hi in (("aren", "aren-transliteration-i8", 4, 51), ("postnorm", "tiny_seq2seq_postnorm", 3, 120)):
        path = os.path.join(OUT, mdir)
        src_vocab = _load_vocabulary(path, "source_vocabulary")
        entry = {"model": mdir, "models": {}}
        for compute in ("float32", "int8"):
            srcs = [[src_vocab[i] for i in r] for r in seq2seq_sources(300, 1, lo, hi)[0]]
            srcs = (srcs + [[src_vocab[i] for i in r] for r in seq2seq_sources(301, 1, lo, hi)[0]])[:4]
            plain = dict(sources=srcs, beam_size=2, num_hypotheses=1, length_penalty=1.0, max_length=20, min_length=1,
                         repetition_penalty=1.0, no_repeat_ngram_size=0, disable_unk=False, suppress_sequences=[])
            hyp = max((h[0][0] for h in ref_translate_processors(path, compute, [plain])[0]), key=len)
            requests = []
            for beam, nh in PROCESSOR_BEAMS:
                for o in processor_options(hyp, name == "postnorm"):
                    r = dict(plain, beam_size=beam, num_hypotheses=nh, max_length=16 if beam < 10 else 12)
                    r.update(o)
                    requests.append(r)
            res = ref_translate_processors(path, compute, requests)
            cases = []
            for r, out in zip(requests, res):
                assert not isinstance(out, str), out
                cases.append(dict(r, hypotheses=[o[0] for o in out], scores=[o[1] for o in out]))
            entry["models"][compute] = {"cases": cases}
        fixture[name] = entry
    with open(os.path.join(OUT, "seq2seq_processors_ref.json"), "w") as f:
        json.dump(fixture, f, ensure_ascii=False)
    print("seq2seq processors fixture:", sum(len(m["cases"]) for e in fixture.values() for m in e["models"].values()), "cases")


def ref_translate_attention(model_dir, compute, requests):
    """Translator::translate_batch of the unmodified reference (CPU) with return_attention, replace_unknowns and
    coverage_penalty, through tools/ref_translate_attention.cc, built by tools/ref_translate_attention.mk against
    oracle/_ref/libct2ref.so into a temporary directory.  requests: dicts of sources (token lists), beam_size,
    num_hypotheses, length_penalty, max_length, min_length, coverage_penalty, return_end_token, return_attention,
    replace_unknowns.  Per request: per source (hypotheses as token lists, scores, attention [hyp][row][column]), or the
    reference's error message."""
    import subprocess
    import tempfile
    out_dir = os.path.join(tempfile.gettempdir(), "ct2ref_attention")
    subprocess.run(["make", "-s", "-f", "tools/ref_translate_attention.mk", "attention", "ATTN_OUT=" + out_dir], cwd=ROOT,
                   check=True)
    text = "%s\t%s\n" % (model_dir, compute)
    for r in requests:
        text += "\t".join(str(x) for x in (r["beam_size"], r["num_hypotheses"], r["length_penalty"], r["max_length"],
                                           r["min_length"], r["coverage_penalty"], int(r["return_end_token"]),
                                           int(r["return_attention"]), int(r["replace_unknowns"]),
                                           "|".join(" ".join(x) for x in r["sources"]))) + "\n"
    lines = subprocess.run([os.path.join(out_dir, "ref_translate_attention")], input=text.encode(), capture_output=True,
                           check=True).stdout.decode().split("\n")
    res, k = [], 0
    for r in requests:
        if lines[k].startswith("ERROR\t"):
            res.append(lines[k].split("\t", 1)[1])
            k += 1
            continue
        entry = []
        for _ in r["sources"]:
            hyps, scores, attn = lines[k].split("\t")
            matrices = [[[float(x) for x in row.split(" ")] if row else [] for row in m.split(";")] if m else []
                        for m in attn.split("|")] if attn else []
            entry.append(([h.split(" ") if h else [] for h in hyps.split("|")], [float(x) for x in scores.split(" ")],
                          matrices))
            k += 1
        res.append(entry)
    return res


ATTENTION_BEAMS = [(1, 1), (2, 2), (4, 3), (10, 2)]   # (beam, num_hypotheses); beam 10 takes the LogSoftMax + TopK path


def find_unk_source(path, compute, src_vocab, lo, hi, max_length):
    """A source of the random model's inputs for which the reference emits <unk> at beam 2."""
    rng = np.random.default_rng(500)
    pool = [[src_vocab[int(i)] for i in rng.integers(lo, hi, size=int(rng.integers(3, 10)))] for _ in range(400)]
    req = dict(sources=pool, beam_size=2, num_hypotheses=1, length_penalty=1.0, max_length=max_length, min_length=1,
               coverage_penalty=0.0, return_end_token=False, return_attention=False, replace_unknowns=False)
    for src, out in zip(pool, ref_translate_attention(path, compute, [req])[0]):
        if "<unk>" in out[0][0]:
            return src
    raise RuntimeError("no source of the pool makes the reference emit <unk>")


# (length_penalty, coverage_penalty) of each beam size; return_end_token alternates along the list
ATTENTION_PENALTIES = [(1.0, 0.0), (0.0, 0.2), (1.0, 1.0), (0.0, 0.0), (1.0, 0.2), (0.0, 1.0)]


def make_seq2seq_attention_fixture():
    """Translator::translate_batch with return_attention, replace_unknowns and coverage_penalty, from the UNMODIFIED
    reference (oracle/_ref, CPU) in float32, on aren-transliteration (default alignment heads), the post-norm model and
    tiny_seq2seq_align (the post-norm recipe with alignment_layer 0 and alignment_heads 0: the mean over every head of the
    first layer): beams 1 / 2 / 4 / 10, coverage_penalty 0 / 0.2 / 1 under length_penalty 1 and 0, return_end_token both
    ways, and a source the reference translates with <unk>, replace_unknowns both ways.

    Beam 1 runs a ragged batch (its padding columns are zeros) and returns the attention of every case (the reference's
    GreedySearch keeps no attention for a coverage penalty alone, decoding.cc:819-833).  Beam searches run one source per
    request: at the first step of a beam search over several sources the reference gathers the unexpanded attention with
    batch indices after repeat_batch expanded it (decoding.cc:565, 590-595), so entry i of its length-sorted batch gets the
    first row of entry i / beam_size (DESIGN §8).  They return the attention of two penalty settings out of six; the others
    pin the ranking the coverage penalty makes."""
    from ctranslate2_b200.converters.synthetic import TransformerConfig, write_transformer_model
    from ctranslate2_b200.translator import _load_vocabulary
    align = os.path.join(OUT, "tiny_seq2seq_align")
    cfg = TransformerConfig(encoder_layers=2, decoder_layers=2, num_heads=4, d_model=64, ffn_dim=128, source_vocab=120,
                            target_vocab=96, pre_norm=False, activation=2, start_from_zero_embedding=True)
    write_transformer_model(align, cfg, "int8", seed=7, alignment_layer=0, alignment_heads=0)
    max_length = 10
    fixture = {}
    for name, mdir, lo, hi in (("aren", "aren-transliteration", 4, 51), ("postnorm", "tiny_seq2seq_postnorm", 3, 120),
                               ("align", "tiny_seq2seq_align", 3, 120)):
        path = os.path.join(OUT, mdir)
        src_vocab = _load_vocabulary(path, "source_vocabulary")
        srcs = [[src_vocab[i] for i in r] for r in seq2seq_sources(310, 1, lo, hi)[0]]
        srcs = (srcs + [[src_vocab[i] for i in r] for r in seq2seq_sources(311, 1, lo, hi)[0]])[:3]
        base = dict(min_length=1, max_length=max_length, replace_unknowns=False)
        requests = []
        for beam, nh in ATTENTION_BEAMS:
            for k, (lp, cov) in enumerate(ATTENTION_PENALTIES):
                requests.append(dict(base, sources=srcs if beam == 1 else [srcs[k % len(srcs)]], beam_size=beam,
                                     num_hypotheses=nh, length_penalty=lp, coverage_penalty=cov, return_end_token=k % 2 == 1,
                                     return_attention=beam == 1 or k in (1, 2)))
        if name != "aren":                          # the aren vocabularies have no <unk>
            unk = find_unk_source(path, "float32", src_vocab, lo, hi, max_length)
            for beam, nh in ((1, 1), (2, 2)):
                for ret_attn in (False, True):
                    for rep in (False, True):
                        requests.append(dict(base, sources=[unk, srcs[0]] if beam == 1 else [unk], beam_size=beam,
                                             num_hypotheses=nh, length_penalty=1.0, coverage_penalty=0.0,
                                             return_end_token=False, return_attention=ret_attn, replace_unknowns=rep))
        res = ref_translate_attention(path, "float32", requests)
        cases = []
        for r, out in zip(requests, res):
            assert not isinstance(out, str), out
            cases.append(dict(r, hypotheses=[o[0] for o in out], scores=[o[1] for o in out], attention=[o[2] for o in out]))
        fixture[name] = {"model": mdir, "compute_type": "float32", "cases": cases}
    with open(os.path.join(OUT, "seq2seq_attention_ref.json"), "w") as f:
        json.dump(fixture, f, ensure_ascii=False, separators=(",", ":"))
    print("seq2seq attention fixture:", sum(len(e["cases"]) for e in fixture.values()), "cases")


WHISPER_CASES = [  # (beam, num_hypotheses, length_penalty, max_length, suppress_blank, timestamps)
    (1, 1, 1.0, 24, True, False), (3, 2, 1.0, 24, True, False), (5, 3, 1.0, 30, True, False), (5, 1, 0.0, 24, False, False),
    (2, 2, 0.7, 16, True, False), (1, 1, 1.0, 30, True, True), (5, 2, 1.0, 30, True, True), (3, 3, 1.0, 24, False, True)]


def whisper_inputs(seed, batch, n_mels, frames):
    return (np.random.default_rng(seed).standard_normal((batch, n_mels, frames)) * 2).astype(np.float32)


def make_whisper_fixture():
    """Whisper path (SURVEY §8 f3): outputs of the UNMODIFIED reference's models::Whisper (oracle/_ref, CPU) on a tiny WhisperSpec
    model written by converters/synthetic.py (2 + 2 layers, d 64, 4 heads, 16 mel bins, 60 frames): encoder output, generate
    (greedy and beam, several hypotheses, length penalties, suppress_blank on / off) and no-speech probabilities, in float32
    and int8.  The features are re-generated from their seeds by the tests."""
    from ctranslate2_b200.converters.synthetic import WhisperConfig, whisper_vocabulary, write_whisper_model
    from oracle import refapi
    cfg = WhisperConfig(encoder_layers=2, decoder_layers=2, num_heads=4, d_model=64, n_mels=16, max_source_positions=30,
                        max_target_positions=64, text_tokens=100, languages=3, timestamps=11)
    mdir = os.path.join(OUT, "tiny_whisper")
    write_whisper_model(mdir, cfg, "int8", seed=5)
    vocab = whisper_vocabulary(cfg)
    sot = vocab.index("<|startoftranscript|>")
    fixture = {"n_mels": 16, "frames": 60, "d_model": 64, "models": {}}
    for compute in ("float32", "int8"):
        w = refapi.RefWhisper(mdir, compute, 2)
        cases = []
        for ci, (beam, nh, lp, mx, blank, stamps) in enumerate(WHISPER_CASES):
            for rep in range(3):
                seed, batch = 300 + 10 * ci + rep, 1 + (ci + rep) % 4
                feats = whisper_inputs(seed, batch, 16, 60)
                # with timestamps the prompt ends with the task token and ApplyTimestampRules shapes the output
                prompts = [[sot, sot + 1 + (b % 3), vocab.index("<|transcribe|>" if b % 2 == 0 else "<|translate|>")] +
                           ([] if stamps else [vocab.index("<|notimestamps|>")]) for b in range(batch)]
                res, nsp = w.generate(feats, prompts, beam_size=beam, num_hypotheses=nh, length_penalty=lp, max_length=mx,
                                      suppress_blank=blank)
                cases.append({"seed": seed, "batch": batch, "prompts": prompts, "beam_size": beam, "num_hypotheses": nh,
                              "length_penalty": lp, "max_length": mx, "suppress_blank": blank, "timestamps": stamps,
                              "sequences": [[h[0] for h in r] for r in res], "scores": [[h[1] for h in r] for r in res],
                              "no_speech_prob": [float(x) for x in nsp]})
        enc = w.encode(whisper_inputs(7, 2, 16, 60), 64)
        fixture["models"][compute] = {"cases": cases, "encode_seed": 7, "encoder_output": enc.tolist()}
        w.close()
    with open(os.path.join(OUT, "whisper_ref.json"), "w") as f:
        json.dump(fixture, f)
    print("whisper fixture:", sum(len(m["cases"]) for m in fixture["models"].values()), "cases")


WHISPER_ALIGN_HEADS = [[1, 2], [0, 1], [1, 0]]   # both decoder layers, out of order: the copy's config.json


def whisper_align_cases():
    """(seed, batch, start_sequence, text rows, num_frames, median_filter_width) on tiny_whisper (60 input frames = 30
    encoder positions, 64 decoder positions; ids: text < 100, <|endoftext|> 100, <|startoftranscript|> 101, languages
    102-104, <|transcribe|> 106, <|notimestamps|> 110)."""
    rng = np.random.default_rng(33)
    text = lambda n: [int(x) for x in rng.integers(0, 100, size=n)]   # noqa: E731
    sot3, sot1 = [101, 102, 106], [101]
    return [
        (400, 1, sot3, [text(5)], [60], 7),                                        # one entry, equal full frames
        (401, 2, sot3, [text(4), text(9)], [60, 60], 7),                             # ragged texts, equal full frames
        (402, 3, sot1, [[], text(1), text(6)], [40, 40, 40], 3),                     # empty and one-token texts, partial
        (403, 4, sot3, [text(3), text(7), text(2), text(5)], [41, 41, 41, 41], 7),  # odd frame count
        (404, 4, sot3, [text(6), text(3), text(8), text(4)], [60, 3, 0, 37], 7),    # variable frames with 1 and 0
        (405, 2, sot1, [text(5), text(2)], [1, 0], 7),                               # all below 2: empty alignments
        (406, 2, sot3, [text(59), text(10)], [60, 50], 7),                           # fills the 64 positions, variable
        (407, 2, sot3, [text(59), text(3)], [60, 60], 3),                            # fills the 64 positions, equal
        (408, 3, sot3, [text(4), text(8), text(2)], [60, 44, 60], 1),                # width 1: pass-through
        (409, 2, sot1, [text(6), text(3)], [40, 40], 61),                            # wider than the frames
        (410, 2, sot3, [text(3) + [100, 105] + text(2), text(4)], [60, 60], 7),     # ids >= <|endoftext|> in a text
        (411, 3, sot1, [text(7), text(1), text(12)], [24, 58, 33], 3),               # variable, width 3
    ]


def _ref_whisper_align(model_dir, compute, requests):
    """models::Whisper::align / detect_language of the unmodified reference (CPU) through tools/ref_whisper_align.cc, built by
    tools/ref_whisper_align.mk against oracle/_ref/libct2ref.so into a temporary directory."""
    import subprocess
    import tempfile
    out_dir = os.path.join(tempfile.gettempdir(), "ct2ref_align")
    subprocess.run(["make", "-s", "-f", "tools/ref_whisper_align.mk", "align", "ALIGN_OUT=" + out_dir], cwd=ROOT, check=True)
    lines, counts = [], []
    for i, req in enumerate(requests):
        path = os.path.join(out_dir, "features_%d.f32" % i)
        req["features"].astype(np.float32).tofile(path)
        dims = " ".join(str(x) for x in req["features"].shape)
        if req["kind"] == "align":
            lines.append("\t".join(["align", path, dims, str(req["width"]), " ".join(map(str, req["start"])),
                                    ";".join(" ".join(map(str, t)) for t in req["text"]), " ".join(map(str, req["num_frames"]))]))
        else:
            lines.append("\t".join(["lang", path, dims]))
        counts.append(req["features"].shape[0])
    text = "%s\t%s\n" % (model_dir, compute) + "".join(x + "\n" for x in lines)
    out = subprocess.run([os.path.join(out_dir, "ref_whisper_align")], input=text.encode(), capture_output=True,
                         check=True).stdout.decode().split("\n")
    res, k = [], 0
    for req, n in zip(requests, counts):
        assert out[k] == "ok", out[k]
        rows = out[k + 1:k + 1 + n]
        k += 1 + n
        if req["kind"] == "align":
            entries = []
            for r in rows:
                a, p = r.split("\t")
                entries.append({"alignments": [[int(x) for x in pair.split(",")] for pair in a.split(" ")] if a else [],
                                "text_token_probs": [float(x) for x in p.split(" ")] if p else []})
            res.append(entries)
        else:
            res.append([[(t, float(v)) for t, v in zip(r.split(" ")[0::2], r.split(" ")[1::2])] for r in rows])
    return res


def make_whisper_align_fixture():
    """models::Whisper::align and ::detect_language of the UNMODIFIED reference (oracle/_ref, CPU) on tiny_whisper, in float32
    and int8: with the model's own alignment_heads, and with a temporary copy whose config.json lists heads of both layers out
    of order (WHISPER_ALIGN_HEADS; the tests recreate the copy).  Features are re-generated from their seeds."""
    import shutil
    import tempfile
    src = os.path.join(OUT, "tiny_whisper")
    tmp = tempfile.mkdtemp()
    permuted = os.path.join(tmp, "tiny_whisper_heads")
    shutil.copytree(src, permuted)
    cfg = json.load(open(os.path.join(src, "config.json")))
    cfg["alignment_heads"] = WHISPER_ALIGN_HEADS
    json.dump(cfg, open(os.path.join(permuted, "config.json"), "w"))
    # this reference calls a model multilingual when its vocabulary holds the empty token (whisper.cc:72): a second copy
    # renames the unused text token <t99> for detect_language
    multilingual = os.path.join(tmp, "tiny_whisper_multilingual")
    shutil.copytree(src, multilingual)
    vocab = json.load(open(os.path.join(src, "vocabulary.json"), encoding="utf-8"))
    vocab[99] = ""
    json.dump(vocab, open(os.path.join(multilingual, "vocabulary.json"), "w", encoding="utf-8"))
    fixture = {"n_mels": 16, "frames": 60, "permuted_heads": WHISPER_ALIGN_HEADS, "models": {}}
    lang_seeds = [(420, 3), (421, 1)]
    for heads, mdir in (("model", src), ("permuted", permuted)):
        for compute in ("float32", "int8"):
            reqs = [{"kind": "align", "features": whisper_inputs(seed, batch, 16, 60), "start": start, "text": text,
                     "num_frames": nf, "width": width} for seed, batch, start, text, nf, width in whisper_align_cases()]
            res = _ref_whisper_align(mdir, compute, reqs)
            cases = [{"seed": seed, "batch": batch, "start_sequence": start, "text_tokens": text, "num_frames": nf,
                      "median_filter_width": width, "results": r}
                     for (seed, batch, start, text, nf, width), r in zip(whisper_align_cases(), res)]
            entry = {"heads": heads, "compute_type": compute, "cases": cases}
            if heads == "model":
                res = _ref_whisper_align(multilingual, compute, [{"kind": "lang", "features": whisper_inputs(seed, batch, 16, 60)}
                                                                  for seed, batch in lang_seeds])
                entry["detect_language"] = [{"seed": seed, "batch": batch, "results": r} for (seed, batch), r in zip(lang_seeds, res)]
            fixture["models"]["%s-%s" % (heads, compute)] = entry
    shutil.rmtree(tmp)
    with open(os.path.join(OUT, "whisper_align_ref.json"), "w") as f:
        json.dump(fixture, f)
    print("whisper align fixture:", sum(len(m["cases"]) for m in fixture["models"].values()), "cases")


WHISPER_SAMPLING_SEED = 2024


def whisper_sampling_cases():
    """(features seed, prompt, sampling_topk, sampling_temperature, num_hypotheses, length_penalty) on tiny_whisper, batch 2,
    max_length 24: k in {0, 5}, T in {0.5, 1.0, 1.5}, H in {1, 3}, length penalties 0 and 1, with and without timestamps."""
    cases, seed = [], 430
    for prompt in ([101, 102, 106, 110], [101, 102, 106]):
        for k in (0, 5):
            for t in (0.5, 1.0, 1.5):
                for h in (1, 3):
                    for lp in (0.0, 1.0):
                        cases.append((seed, prompt, k, t, h, lp))
                        seed += 1
    return cases


def make_whisper_sampling_fixture():
    """models::Whisper::generate with a RandomSampler of the UNMODIFIED reference (oracle/_ref, CPU, float32) on tiny_whisper
    through tools/ref_whisper_sample.cc: the sampled sequences and their scores (no RNG parity: the tests check the score
    convention of these sequences and their top-k membership, not the draws).  Features are re-generated from their seeds."""
    import subprocess
    import tempfile
    out_dir = os.path.join(tempfile.gettempdir(), "ct2ref_sample")
    subprocess.run(["make", "-s", "-f", "tools/ref_whisper_sample.mk", "sample", "SAMPLE_OUT=" + out_dir], cwd=ROOT, check=True)
    cases, lines = whisper_sampling_cases(), []
    for i, (seed, prompt, k, t, h, lp) in enumerate(cases):
        path = os.path.join(out_dir, "features_%d.f32" % i)
        whisper_inputs(seed, 2, 16, 60).astype(np.float32).tofile(path)
        lines.append("\t".join([path, "2 16 60", ";".join([" ".join(map(str, prompt))] * 2), str(k), repr(t), str(h), repr(lp),
                                "24"]))
    text = "%s\tfloat32\t%d\n" % (os.path.join(OUT, "tiny_whisper"), WHISPER_SAMPLING_SEED) + "".join(x + "\n" for x in lines)
    out = subprocess.run([os.path.join(out_dir, "ref_whisper_sample")], input=text.encode(), capture_output=True,
                         check=True).stdout.decode().split("\n")
    fixture = {"n_mels": 16, "frames": 60, "batch": 2, "max_length": 24, "compute_type": "float32",
               "seed": WHISPER_SAMPLING_SEED, "cases": []}
    k_line = 0
    for seed, prompt, k, t, h, lp in cases:
        assert out[k_line] == "ok", out[k_line]
        rows = out[k_line + 1:k_line + 1 + 2 * h]
        k_line += 1 + 2 * h
        hyps = [[] for _ in range(2)]
        for r in rows:
            b, score, ids = r.split("\t")
            hyps[int(b)].append({"score": float(score), "ids": [int(x) for x in ids.split(" ")] if ids else []})
        fixture["cases"].append({"seed": seed, "prompt": prompt, "sampling_topk": k, "sampling_temperature": t,
                                 "num_hypotheses": h, "length_penalty": lp, "results": hyps})
    with open(os.path.join(OUT, "whisper_sampling_ref.json"), "w") as f:
        json.dump(fixture, f)
    print("whisper sampling fixture:", len(fixture["cases"]), "cases")


ENCODER_VARIANTS = {
    # BERT-like: tokens + token types, learned positions, layernorm_embedding, post-norm GELU, pooler
    "tiny_encoder": {},
    "tiny_encoder_prenorm": {"pre_norm": True, "activation": 0, "type_vocab_size": 0, "layernorm_embedding": False},
    "tiny_encoder_nopooler": {"pooler": False, "activation": 1},
}


def _ref_encoder(model_dir, compute, ids, types):
    """Encoder::forward_batch of the unmodified reference (CPU) through tools/ref_encoder.cc, built by tools/ref_encoder.mk
    against oracle/_ref/libct2ref.so into a temporary directory: per row, (hidden [len, d], pooled [d] or None)."""
    import subprocess
    import tempfile
    out_dir = os.path.join(tempfile.gettempdir(), "ct2ref_encoder")
    subprocess.run(["make", "-s", "-f", "tools/ref_encoder.mk", "encoder", "ENCODER_OUT=" + out_dir], cwd=ROOT, check=True)
    lines = ["%s\t%s" % (model_dir, compute)]
    for b, row in enumerate(ids):
        lines.append(" ".join(map(str, row)) + "\t" + (" ".join(map(str, types[b])) if types is not None else ""))
    r = subprocess.run([os.path.join(out_dir, "ref_encoder")], input="\n".join(lines) + "\n", capture_output=True, text=True,
                       check=True)
    res = []
    for line in r.stdout.rstrip("\n").split("\n"):
        h, p = line.split("\t")
        res.append(([float(x) for x in h.split(" ")], [float(x) for x in p.split(" ")] if p else None))
    return res


def make_encoder_fixture():
    """tests/golden/tiny_encoder*/ (synthetic TransformerEncoderSpec models, int8 storage, d 64 = 1 head of 64, 16 positions)
    and tests/golden/encoder_ref.npz: the reference's Encoder::forward_batch (CPU build) in float32 and int8 on ragged
    batches with a 1-token row and a row that fills the position table, with and without token types.  Case k is stored as
    c<k>_model, c<k>_compute, c<k>_ids [B, T] (right-padded), c<k>_lens [B], c<k>_types [B, T] (when given), c<k>_hidden
    [sum(lens), d] (the valid positions, row after row) and c<k>_pooled [B, d] (models with a pooler)."""
    from ctranslate2_b200.converters.synthetic import EncoderConfig, write_encoder_model
    rng = np.random.default_rng(2024)
    arrays, k = {}, 0
    for m, (name, kw) in enumerate(ENCODER_VARIANTS.items()):
        cfg = EncoderConfig(num_layers=2, num_heads=1, d_model=64, ffn_dim=128, vocab_size=50, max_positions=16,
                            layer_norm_epsilon=1e-12, **kw)
        path = os.path.join(OUT, name)
        write_encoder_model(path, cfg, "int8", seed=11 + m)
        for compute in ("float32", "int8"):
            for with_types in ((False, True) if cfg.type_vocab_size else (False,)):
                if compute == "int8" and not with_types and cfg.type_vocab_size:
                    continue
                lens = np.array([16, 1, 7], np.int32)
                ids = np.zeros((len(lens), lens.max()), np.int32)
                types = np.zeros_like(ids) if with_types else None
                for b, n in enumerate(lens):
                    ids[b, :n] = rng.integers(0, cfg.vocab_size, n)
                    if with_types:
                        types[b, :n] = rng.integers(0, cfg.type_vocab_size, n)
                res = _ref_encoder(os.path.abspath(path), compute, [ids[b, :n].tolist() for b, n in enumerate(lens)],
                                   None if types is None else [types[b, :n].tolist() for b, n in enumerate(lens)])
                c = "c%d_" % k
                arrays.update({c + "model": np.array(name), c + "compute": np.array(compute), c + "ids": ids, c + "lens": lens,
                               c + "hidden": np.array([v for h, _ in res for v in h], np.float32).reshape(-1, cfg.d_model)})
                if types is not None:
                    arrays[c + "types"] = types
                if res[0][1] is not None:
                    arrays[c + "pooled"] = np.array([p for _, p in res], np.float32)
                k += 1
    np.savez_compressed(os.path.join(OUT, "encoder_ref.npz"), **arrays)
    print("encoder fixture:", k, "cases")


def main():
    os.makedirs(OUT, exist_ok=True)
    if "--encoder-only" in sys.argv:
        make_encoder_fixture()
        return
    if "--whisper-sampling-only" in sys.argv:
        make_whisper_sampling_fixture()
        return
    if "--whisper-align-only" in sys.argv:
        make_whisper_align_fixture()
        return
    if "--scores-only" in sys.argv:
        make_scores_fixture()
        return
    if "--score-only" in sys.argv:
        make_score_fixture()
        return
    if "--ragged-only" in sys.argv:
        make_ragged_fixture()
        return
    if "--whisper-only" in sys.argv:
        make_whisper_fixture()
        return
    if "--seq2seq-only" in sys.argv:
        make_seq2seq_fixture()
        return
    if "--translator-score-only" in sys.argv:
        make_translator_score_fixture()
        return
    if "--seq2seq-processors-only" in sys.argv:
        make_seq2seq_processors_fixture()
        return
    if "--processors-only" in sys.argv:
        make_processors_fixture()
        return
    if "--seq2seq-attention-only" in sys.argv:
        make_seq2seq_attention_fixture()
        return
    if "--gtest-only" in sys.argv:
        with open(os.path.join(OUT, "ref_gtest_vectors.json"), "w") as f:
            json.dump(extract_gtest_vectors(), f)
        return
    print("extracting gtest golden vectors")
    with open(os.path.join(OUT, "ref_gtest_vectors.json"), "w") as f:
        json.dump(extract_gtest_vectors(), f)

    from oracle import refapi
    assert refapi.available(), "build oracle/_ref first: make -f oracle/Makefile.ref -j8"

    print("tiny model via the reference spec writer")
    mdir = os.path.join(OUT, "tiny_llama_int8")
    V = make_tiny_model(mdir)
    g = refapi.RefGenerator(mdir, "int8", 4)
    rng = np.random.default_rng(42)
    prompts = rng.integers(3, V, size=(3, 7), dtype=np.int32)
    logits = g.forward(prompts)
    gen = g.generate(prompts, max_length=12, min_length=0, end_id=2)
    gen_min = g.generate(prompts, max_length=12, min_length=12, end_id=2)
    np.savez(os.path.join(OUT, "tiny_llama_int8_ref.npz"), prompts=prompts, logits=logits,
             generated=np.array(gen, dtype=object), generated_min12=np.array(gen_min, dtype=np.int32),
             allow_pickle=True)
    g.close()

    print("reference ops on seeded random inputs")
    r = np.random.default_rng(7)
    d = {}
    x = (r.standard_normal((5, 96)) * 3).astype(np.float32)
    x[3] = 0
    d["q_x"] = x
    d["q_q"], d["q_s"] = refapi.quantize(x)
    a = r.integers(-127, 128, size=(5, 96), dtype=np.int8)
    b = r.integers(-127, 128, size=(24, 96), dtype=np.int8)
    d["g_a"], d["g_b"], d["g_c"] = a, b, refapi.gemm_s8(a, b)
    sa = r.uniform(1, 50, 5).astype(np.float32)
    sb = r.uniform(100, 900, 24).astype(np.float32)
    bias = r.standard_normal(24).astype(np.float32)
    d["dq_sa"], d["dq_sb"], d["dq_bias"] = sa, sb, bias
    for act in (-1, 0, 1, 2, 3, 4, 5, 6):
        d["dq_y_act%d" % act] = refapi.dequantize_gemm(d["g_c"], sa, sb, bias, act)
    d["dq_y_nobias"] = refapi.dequantize_gemm(d["g_c"], sa, sb, None, -1)
    gamma = r.standard_normal(96).astype(np.float32)
    d["rn_gamma"], d["rn_y"] = gamma, refapi.rms_norm(gamma, x, 1e-5)
    xr = r.standard_normal((2, 3, 4, 16)).astype(np.float32)
    ang = r.standard_normal((4, 16)).astype(np.float32)
    d["ro_x"], d["ro_sin"], d["ro_cos"] = xr, np.sin(ang), np.cos(ang)
    d["ro_y_interleave"] = refapi.rotary(xr, d["ro_sin"], d["ro_cos"], True)
    d["ro_y_half"] = refapi.rotary(xr, d["ro_sin"], d["ro_cos"], False)
    sx = r.standard_normal((6, 33)).astype(np.float32)
    lens = np.array([33, 1, 7, 20, 33, 2], np.int32)
    d["sm_x"], d["sm_len"] = sx, lens
    d["sm_y"], d["sm_y_len"] = refapi.softmax(sx), refapi.softmax(sx, lens)
    d["sm_logy"] = refapi.softmax(sx, None, True)
    tx = r.standard_normal((4, 1000)).astype(np.float32)
    tx[1, 17] = tx[1, 500] = 9.0   # exact tie: lowest index must win
    d["tk_x"] = tx
    d["tk_v1"], d["tk_i1"] = refapi.topk(tx, 1)
    d["tk_v4"], d["tk_i4"] = refapi.topk(tx, 4)
    gd = r.standard_normal((50, 8)).astype(np.float32)
    gi = r.integers(0, 50, 9).astype(np.int32)
    d["ga_d"], d["ga_i"], d["ga_y"] = gd, gi, refapi.gather(gd, gi)
    np.savez(os.path.join(OUT, "ref_ops_random.npz"), **d)
    make_scores_fixture()
    make_processors_fixture()
    make_ragged_fixture()
    make_score_fixture()
    make_seq2seq_fixture()
    make_translator_score_fixture()
    make_seq2seq_processors_fixture()
    make_seq2seq_attention_fixture()
    make_whisper_fixture()
    make_whisper_align_fixture()
    make_whisper_sampling_fixture()
    make_encoder_fixture()
    print("done")


if __name__ == "__main__":
    main()
