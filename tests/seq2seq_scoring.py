"""Translator::score_batch restated on the oracle, for the scoring tests: token strings to ids as the reference builds them
(Vocabulary::to_ids with add_source_bos / add_source_eos, the decoder start token and </s>, EOS-keeping truncation;
src/models/sequence_to_sequence.cc:168-186, src/vocabulary.cc:108-147), and the scores of Seq2SeqOracle's cached one-token
path run with teacher forcing, one target position at a time -- a different route from the engine's causal pass."""
import json
import os
from typing import List, Sequence

import numpy as np

from oracle import ct2_oracle as O


def _vocabulary(model_dir: str, name: str) -> List[str]:
    for n in ("shared_vocabulary", name):
        for ext in (".json", ".txt"):
            p = os.path.join(model_dir, n + ext)
            if os.path.exists(p):
                if ext == ".json":
                    with open(p, encoding="utf-8") as f:
                        return json.load(f)
                with open(p, encoding="utf-8") as f:
                    return [line.rstrip("\n") for line in f]
    raise FileNotFoundError(name)


def _truncate(ids: List[int], max_length: int, eos: int) -> List[int]:
    if max_length == 0 or len(ids) <= max_length:
        return ids
    out = ids[:max_length]
    if ids[-1] == eos:
        out[-1] = eos
    elif ids[-2] == eos and max_length >= 2:
        out[-2:] = [eos, ids[-1]]
    return out


def pair_ids(model_dir: str, source: Sequence[str], target: Sequence[str], max_input_length: int = 1024):
    """(source ids, full target ids) of one pair of token lists, as the reference's run_scoring makes them."""
    cfg_path = os.path.join(model_dir, "config.json")
    cfg = json.load(open(cfg_path)) if os.path.exists(cfg_path) else {}
    sv, tv = _vocabulary(model_dir, "source_vocabulary"), _vocabulary(model_dir, "target_vocabulary")
    s_id, t_id = {w: i for i, w in enumerate(sv)}, {w: i for i, w in enumerate(tv)}
    bos, eos, unk = cfg.get("bos_token", "<s>"), cfg.get("eos_token", "</s>"), cfg.get("unk_token", "<unk>")
    src = [s_id.get(w, s_id.get(unk, 0)) for w in source]
    if cfg.get("add_source_bos", False):
        src = [s_id[bos]] + src
    if cfg.get("add_source_eos", False):
        src = src + [s_id[eos]]
    start = cfg.get("decoder_start_token", "<s>")
    tgt = ([] if start is None else [t_id[start]]) + [t_id.get(w, t_id.get(unk, 0)) for w in target] + [t_id[eos]]
    return (_truncate(src, max_input_length, s_id.get(eos, -1)),
            _truncate(tgt, max_input_length + 1 if max_input_length else 0, t_id[eos]))


def oracle_score(oracle: O.Seq2SeqOracle, sources: Sequence[Sequence[int]], targets: Sequence[Sequence[int]],
                 offset: int = 0) -> List[List[float]]:
    """Log-probabilities of targets[b][offset + 1:] given sources[b] (non-empty id lists, special tokens included) and the
    target prefix: the encoder once, then Seq2SeqOracle.step on target position t for t = 0 .. len - 2 (the decoder
    appends each position to its self-attention cache), LogSoftMax of each step's logits, Gather of the next target id."""
    B = len(sources)
    lens = np.array([len(s) for s in sources])
    src = np.zeros((B, int(lens.max())), np.int64)
    for b, s in enumerate(sources):
        src[b, :len(s)] = s
    oracle.start(oracle.encode(src, lens), lens, 1)
    T = max(len(t) for t in targets)
    tgt = np.zeros((B, T), np.int64)
    for b, t in enumerate(targets):
        tgt[b, :len(t)] = t
    out: List[List[float]] = [[] for _ in range(B)]
    for t in range(T - 1):
        lp = O.softmax(oracle.step(tgt[:, t], t), log=True)
        for b in range(B):
            if offset <= t < len(targets[b]) - 1:
                out[b].append(float(lp[b, tgt[b, t + 1]]))
    return out
