"""Translator::translate_batch with the logits processors of TranslationOptions, restated on the oracle: Seq2SeqOracle's
encoder and cached decoder steps driven by ct2_oracle.beam_search, with a logits hook that keeps every beam's history of
chosen tokens (the gather indices of the search, as WhisperOracle.generate does) and applies the processors per row in the
reference's order.

BeamSearch::search (decoding.cc:505-527) collects every disabled entry — the end ids below min_decoding_length
(apply_min_length) and those of the processors — in DisableTokens and writes them after the processors ran, so the
RepetitionPenalty rewrites values that no disable has touched yet.  beam_search writes the min-length mask before its hook;
the hook therefore restores those entries from the step's logits, runs ct2_oracle.apply_logits_processors (penalty first, then
NoRepeatNgram, SuppressTokens, SuppressSequences) and writes the min-length mask again."""
from typing import Sequence

import numpy as np

from oracle import ct2_oracle as O

f32 = np.float32


def processors_hook(state, end_ids: Sequence[int], min_length: int, repetition_penalty: float = 1.0,
                    no_repeat_ngram_size: int = 0, disable_ids: Sequence[int] = (), suppress_sequences=()):
    """beam_search's logits_hook: state["seq"] [rows] = the histories, state["raw"] = the step's logits before any mask."""
    lowest = np.finfo(f32).min

    def hook(step, logits):
        if step < min_length:
            for e in end_ids:
                logits[:, e] = state["raw"][:, e]
        for n in range(logits.shape[0]):
            O.apply_logits_processors(logits[n], state["seq"][n], repetition_penalty, no_repeat_ngram_size,
                                      suppress_sequences, disable_ids)
        if step < min_length:
            for e in end_ids:
                logits[:, e] = lowest

    return hook


def translate(oracle: "O.Seq2SeqOracle", source_ids, beam_size: int = 2, num_hypotheses: int = 1, max_length: int = 256,
              min_length: int = 1, length_penalty: float = 1.0, bos: int = 1, eos: int = 2, repetition_penalty: float = 1.0,
              no_repeat_ngram_size: int = 0, disable_ids: Sequence[int] = (), suppress_sequences=()):
    """Seq2SeqOracle.translate with the processors (ids of the target vocabulary).  Per entry [(tokens, score), ...]."""
    B = len(source_ids)
    lengths = np.array([len(r) for r in source_ids])
    src = np.zeros((B, int(lengths.max())), np.int64)
    for b, r in enumerate(source_ids):
        src[b, :len(r)] = r
    oracle.start(oracle.encode(src, lengths), lengths, beam_size)
    V = oracle.v["decoder/projection/weight"].shape[0]
    state = {"seq": [[] for _ in range(B * beam_size)], "gather": None, "raw": None}

    def step_fn(ids, s):
        if s > 0:                                                # the search gathered the beams: ids are the new last tokens
            state["seq"] = [state["seq"][g] + [int(t)] for g, t in zip(state["gather"], ids)]
        state["raw"] = np.array(oracle.step(ids, s), f32)
        return state["raw"]

    def reorder(index):
        state["gather"] = [int(i) for i in index]
        oracle.reorder(index)

    hook = processors_hook(state, [eos], min_length, repetition_penalty, no_repeat_ngram_size, disable_ids, suppress_sequences)
    return O.beam_search(step_fn, reorder, np.full(B, bos), V, beam_size, max_length, min_length, [eos], length_penalty,
                         num_hypotheses, logits_hook=hook)
