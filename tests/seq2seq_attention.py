"""Translator::translate_batch with return_attention and coverage_penalty, restated on the oracle: Seq2SeqOracle's encoder and
cached decoder steps, with the cross-attention probabilities of the model's alignment heads kept per step, driven by a beam
search that follows ct2_oracle.beam_search and also keeps every beam's attention rows (alive_attention, decoding.cc:590-596),
hands a registered hypothesis the rows of its tokens (build_attention, :631-632) and adds the coverage penalty at finalize
(finalize_result, :176-254).  The oracle module itself is unchanged: AttentionOracle only records what its attention computes.

Also the host-side column handling of EncoderDecoderReplica::run_translation (sequence_to_sequence.cc:395-412), shared by the
fixture tests."""
import math
from typing import List, Sequence

import numpy as np

from oracle import ct2_oracle as O

f32 = np.float32


class AttentionOracle(O.Seq2SeqOracle):
    """Seq2SeqOracle that records the alignment attention of each decoder step: the mean of the normalised cross-attention
    of heads [0, alignment_heads) of decoder layer alignment_layer (transformer.cc:518-528, 811-838)."""

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        v = self.v

        def attr(name, default):
            for key in ("decoder/" + name, name):
                if key in v:
                    return int(v[key])
            return default
        layer, heads = attr("alignment_layer", -1), attr("alignment_heads", 1)
        self.align_layer = layer + self.dec_layers if layer < 0 else layer
        self.align_heads = heads if heads else self.num_heads
        self.attention = None                                    # [N, S] of the last step

    def _attend(self, q, k, v_, lens_rows):
        B, T, _ = q.shape
        S = k.shape[1]
        H, D = self.num_heads, self.d // self.num_heads
        qh = q.reshape(B, T, H, D).transpose(0, 2, 1, 3)
        kh = k.reshape(B, S, H, D).transpose(0, 2, 1, 3)
        vh = v_.reshape(B, S, H, D).transpose(0, 2, 1, 3)
        scores = (np.einsum("bhtd,bhsd->bhts", qh, kh) * f32(1.0 / math.sqrt(D))).astype(f32)
        probs = O.softmax(scores.reshape(-1, S), lens_rows).reshape(B, H, T, S)
        if T == 1 and getattr(self, "mem_k", None) and k is self.mem_k[self.align_layer]:
            self.attention = (probs[:, :self.align_heads, 0, :].sum(axis=1, dtype=f32) / f32(self.align_heads)).astype(f32)
        ctx = np.einsum("bhts,bhsd->bhtd", probs, vh).astype(f32)
        return ctx.transpose(0, 2, 1, 3).reshape(B, T, self.d)


def coverage_term(rows) -> float:
    """compute_coverage_penalty (decoding.cc:176-187) without its factor."""
    cov = np.sum(np.array(rows, f32), axis=0, dtype=f32)
    return float(np.log(np.minimum(cov[cov > 0], f32(1)), dtype=f32).sum(dtype=f32))


def translate(oracle: AttentionOracle, source_ids, beam_size: int = 2, num_hypotheses: int = 1, max_length: int = 256,
              min_length: int = 1, length_penalty: float = 1.0, coverage_penalty: float = 0.0, return_end_token: bool = False,
              bos: int = 1, eos: int = 2):
    """Per entry [(tokens, score, attention rows [len(tokens)][max source length]), ...], best first."""
    B = len(source_ids)
    lengths = np.array([len(r) for r in source_ids])
    src = np.zeros((B, int(lengths.max())), np.int64)
    for b, r in enumerate(source_ids):
        src[b, :len(r)] = r
    oracle.start(oracle.encode(src, lengths), lengths, beam_size)
    V = oracle.v["decoder/projection/weight"].shape[0]
    ids = np.repeat(np.full(B, bos), beam_size).astype(np.int64)
    lowest = np.finfo(f32).min
    scores = np.tile(np.array([0.0] + [lowest] * (beam_size - 1), f32), B)
    alive = [[([], []) for _ in range(beam_size)] for _ in range(B)]
    hyps: List[list] = [[] for _ in range(B)]
    finished, top_done = [False] * B, [False] * B
    ncand = 2 * beam_size
    early_exit = length_penalty == 0 and coverage_penalty == 0                       # decoding.cc:457
    for step in range(max_length):
        logits = np.array(oracle.step(ids, step), f32)
        attn = oracle.attention
        if step < min_length:
            logits[:, eos] = lowest
        with np.errstate(over="ignore"):
            lp = (O.softmax(logits, log=True) + scores[:, None]).astype(f32).reshape(B, beam_size * V)
        cand_scores, cand_ids = O.topk(lp, ncand)
        origin, word = cand_ids // V, cand_ids % V
        is_last = step + 1 == max_length
        new_ids = np.zeros((B, beam_size), np.int64)
        new_scores = np.zeros((B, beam_size), f32)
        gather = np.zeros((B, beam_size), np.int64)
        for i in range(B):
            seqs = []
            for j in range(ncand):
                o = int(origin[i, j])
                toks, rows = alive[i][o]
                seqs.append((toks + [int(word[i, j])], rows + [attn[i * beam_size + o]]))
            secondary, active = beam_size, []
            for k in range(beam_size):
                nxt = k
                if not finished[i] and (int(word[i, k]) == eos or is_last):
                    if k == 0:
                        top_done[i] = True
                    hyps[i].append((seqs[k][0], seqs[k][1], float(cand_scores[i, k])))
                    for j in range(secondary, ncand):
                        if int(word[i, j]) != eos:
                            nxt, secondary = j, j + 1
                            break
                active.append(nxt)
            if not finished[i]:
                if is_last:
                    finished[i] = True
                elif early_exit:
                    finished[i] = top_done[i] and len(hyps[i]) >= num_hypotheses
                else:
                    finished[i] = len(hyps[i]) >= max(1, int(math.floor(beam_size + 0.5)))
            alive[i] = [seqs[a] for a in active]
            new_ids[i] = word[i, active]
            new_scores[i] = cand_scores[i, active]
            gather[i] = i * beam_size + origin[i, active]
        if all(finished):
            break
        oracle.reorder(gather.reshape(-1))
        ids, scores = new_ids.reshape(-1), new_scores.reshape(-1).astype(f32)
    out = []
    for i in range(B):
        final = []
        for toks, rows, sc in hyps[i]:
            with np.errstate(divide="ignore"):
                s = f32(sc) / f32(f32(len(toks)) ** f32(length_penalty))
            if coverage_penalty != 0:
                s = f32(s + f32(coverage_penalty) * f32(coverage_term(rows)))
            final.append((toks, rows, float(s)))
        order = sorted(range(len(final)), key=lambda j: -final[j][2])
        best = []
        for j in order[:num_hypotheses]:
            toks, rows = list(final[j][0]), [np.asarray(r, f32) for r in final[j][1]]
            while not return_end_token and toks and toks[-1] == eos:
                toks.pop()
                rows.pop()
            best.append((toks, final[j][2], rows))
        out.append(best)
    return out


def source_columns(rows, input_len: int, original_len: int, add_bos: bool, add_eos: bool) -> List[List[float]]:
    """sequence_to_sequence.cc:395-412: cut to the input length, drop the added <s> / </s> columns, zero-pad to the tokens."""
    out = []
    for r in rows:
        r = list(np.asarray(r, f32)[:input_len])
        if add_bos:
            r = r[1:]
        if add_eos:
            r = r[:-1]
        out.append((r + [0.0] * original_len)[:original_len])
    return out


def replace_unknowns(hyp: Sequence[str], source: Sequence[str], attention, unk: str = "<unk>") -> List[str]:
    return [source[int(np.argmax(attention[t]))] if tok == unk else tok for t, tok in enumerate(hyp)]
