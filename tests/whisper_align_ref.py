"""numpy restatements of the host-side pieces of models::Whisper::align, for the tests: negative_dtw + backtrace (src/dtw.cc)
and ops::MedianFilter on the last axis (src/ops/median_filter_cpu.cc), and WhisperAlignOracle, the fp32 restatement of
models::Whisper::align / detect_language the tests compare the engine with."""
import math

import numpy as np


def negative_dtw(x):
    """dtw.cc:40-80: cost[i][j] = -x[i-1][j-1] + min(diagonal, up, left) with the reference's tie order (diagonal only if
    strictly below both, up only if strictly below both, otherwise left), then the backtrace of dtw.cc:8-38."""
    x = np.asarray(x, np.float32)
    n, m = x.shape
    cost = np.full((n + 1, m + 1), np.inf, np.float32)
    trace = np.full((n + 1, m + 1), -1, np.int8)
    cost[0, 0] = 0
    for j in range(1, m + 1):
        for i in range(1, n + 1):
            c0, c1, c2 = cost[i - 1, j - 1], cost[i - 1, j], cost[i, j - 1]
            if c0 < c1 and c0 < c2:
                c, t = c0, 0
            elif c1 < c0 and c1 < c2:
                c, t = c1, 1
            else:
                c, t = c2, 2
            cost[i, j] = np.float32(-x[i - 1, j - 1]) + c
            trace[i, j] = t
    trace[0, :] = 2
    trace[:, 0] = 1
    i, j, path = n, m, []
    while i > 0 or j > 0:
        path.append((i - 1, j - 1))
        t = trace[i, j]
        if t == 0:
            i, j = i - 1, j - 1
        elif t == 1:
            i -= 1
        else:
            j -= 1
    return path[::-1]


def path_cost(x, path):
    """Sum of the matrix values the path visits (entries with a -1 index are outside the matrix)."""
    return float(sum(x[i, j] for i, j in path if i >= 0 and j >= 0))


def median_filter(x, width):
    """median_filter_cpu.cc: a window of `width` around every element of the last axis, mirrored as |j + k| and
    depth - (read - depth) - 2; the input passes through when depth <= width // 2 (or width <= 1)."""
    x = np.asarray(x, np.float32)
    depth, rank = x.shape[-1], width // 2
    if width <= 1 or depth <= rank:
        return x.copy()
    out = np.empty_like(x)
    for j in range(depth):
        reads = []
        for k in range(-rank, rank + 1):
            read = abs(j + k)
            if read >= depth:
                read = depth - (read - depth) - 2
            reads.append(read)
        out[..., j] = np.sort(x[..., reads], axis=-1)[..., rank]
    return out


def softmax_rows(x):
    """ops::SoftMax on the last axis in fp32 (softmax_cpu: y = exp(x - max) * (1 / sum))."""
    x = np.asarray(x, np.float32)
    e = np.exp(x - x.max(-1, keepdims=True), dtype=np.float32)
    return (e * (np.float32(1) / e.sum(-1, keepdims=True, dtype=np.float32))).astype(np.float32)


def standardize_columns(x):
    """ops::LayerNorm(-2, 0) without gamma / beta (layer_norm_axis, cpu/kernels.cc): every column of x [.., T, F] over its
    T rows, summed in row order; var = max(sumsq / T - mean^2, 0), y = (x - mean) / sqrt(var) (NaN for a constant column)."""
    x = np.asarray(x, np.float32)
    s = np.zeros(x.shape[:-2] + x.shape[-1:], np.float32)
    sq = np.zeros_like(s)
    for t in range(x.shape[-2]):
        s = (s + x[..., t, :]).astype(np.float32)
        sq = (sq + x[..., t, :] * x[..., t, :]).astype(np.float32)
    n = np.float32(x.shape[-2])
    mean = (s / n).astype(np.float32)
    var = np.maximum(sq / n - mean * mean, np.float32(0)).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        rstd = (np.float32(1) / np.sqrt(var)).astype(np.float32)
        return ((x - mean[..., None, :]) * rstd[..., None, :]).astype(np.float32)


def _oracle_base():
    from oracle.ct2_oracle import WhisperOracle
    return WhisperOracle


class WhisperAlignOracle:
    """fp32 restatement of WhisperReplica::align (src/models/whisper.cc:387-582) and ::detect_language (:584-652) on top of
    oracle.ct2_oracle.WhisperOracle (encoder, decoder weights and layers).  Every entry runs through the decoder on its own
    (the reference's CPU build removes padding, transformer.cc:660-677), and in the equal-frames path the padded rows of
    shorter inputs are copies of the entry's last row, which is what Padder::add_padding gives back (src/padder.cc:33-44)."""

    def __init__(self, model_dir, compute_type="float32"):
        self.o = _oracle_base().from_dir(model_dir, compute_type=compute_type)
        self.config = self.o.config

    def decode_sequence(self, memory, ids, heads):
        """One entry: memory [S, d], ids [T] at positions 0 .. T - 1 with causal self-attention -> (logits [T, V], the
        pre-softmax cross-attention scores of `heads` [len(heads), T, S], layer order then list order)."""
        o = self.o
        T, H = len(ids), o.num_heads
        D = o.d // H
        x = (o._embed("decoder", np.asarray(ids).reshape(1, T)) + o.pos[:T][None]).astype(np.float32)
        mem = memory[None].astype(np.float32)
        causal = np.tile(np.arange(1, T + 1), H)
        per_layer = {}
        for layer, head in heads:
            per_layer.setdefault(layer, []).append(head)
        saved = []
        for l in range(o.dec_layers):
            p = f"decoder/layer_{l}/"

            def self_attn(h, res):
                q, k, v_ = np.split(o._dense(p + "self_attention/linear_0", h), 3, axis=-1)
                return o._dense(p + "self_attention/linear_1", o._attend(q, k, v_, causal), residual=res)

            def cross_attn(h, res):
                q = o._dense(p + "attention/linear_0", h)
                k, v_ = np.split(o._dense(p + "attention/linear_1", mem), 2, axis=-1)
                if l in per_layer:
                    qh = q[0].reshape(T, H, D).transpose(1, 0, 2)
                    kh = k[0].reshape(-1, H, D).transpose(1, 0, 2)
                    sc = (np.einsum("htd,hsd->hts", qh, kh) * np.float32(1.0 / math.sqrt(D))).astype(np.float32)
                    saved.extend(sc[hd] for hd in per_layer[l])
                return o._dense(p + "attention/linear_2", o._attend(q, k, v_, np.full(H * T, k.shape[1])), residual=res)

            def ffn(h, res):
                return o._dense(p + "ffn/linear_1", o._dense(p + "ffn/linear_0", h, act=o.act["decoder"]), residual=res)

            x = o._sublayer("decoder", p + "self_attention", x, self_attn)
            x = o._sublayer("decoder", p + "attention", x, cross_attn)
            x = o._sublayer("decoder", p + "ffn", x, ffn)
        if "decoder/layer_norm/gamma" in o.v:
            x = o._ln("decoder/layer_norm", x)
        return o._dense("decoder/projection", x)[0], (np.stack(saved) if saved else None)

    def align(self, features, start_sequence, text_tokens, num_frames, median_filter_width=7, heads=None):
        """-> (results [(alignments, text_token_probs)], matrices [per entry: [len(text) + 1, nf] or None])."""
        o = self.o
        heads = [tuple(h) for h in (heads if heads is not None else self.config["alignment_heads"])]
        B = len(text_tokens)
        nt, eot = o.no_timestamps, o.eot
        s0 = len(start_sequence)
        nf = [int(n) // 2 for n in (num_frames if not np.isscalar(num_frames) else [num_frames] * B)]
        inputs = [list(start_sequence) + [nt] + list(t) + [eot] for t in text_tokens]
        scores, probs = [], []
        for b in range(B):
            memory = o.encode_features(np.asarray(features[b:b + 1], np.float32))[0]
            logits, sc = self.decode_sequence(memory, inputs[b], heads)
            scores.append(sc)
            p = []
            for t, tok in enumerate(text_tokens[b]):     # SoftMax over [0, eot) at position s0 + t, Gather of text[t]
                p.append(float(softmax_rows(logits[s0 + t, :eot])[tok]) if tok < eot else 0.0)
            probs.append(p)
        matrices = [None] * B
        if any(n > 0 for n in nf):
            if all(n == nf[0] for n in nf):              # equal frames: all rows of the padded batch (whisper.cc:552-559)
                Tg = max(len(i) for i in inputs)
                for b in range(B):
                    sc = scores[b][:, :, :nf[b]]
                    sc = np.concatenate([sc, np.repeat(sc[:, -1:], Tg - sc.shape[1], axis=1)], axis=1)
                    matrices[b] = self._matrix(softmax_rows(sc), s0, len(text_tokens[b]), median_filter_width)
            else:                                        # variable frames: the entry's own rows and frames (:519-550)
                for b in range(B):
                    if nf[b] > 0:
                        matrices[b] = self._matrix(softmax_rows(scores[b][:, :, :nf[b]]), s0, len(text_tokens[b]),
                                                   median_filter_width)
        results = [(negative_dtw(m) if m is not None else [], probs[b]) for b, m in enumerate(matrices)]
        return results, matrices

    @staticmethod
    def _matrix(probs, s0, n, width):
        """compute_alignments (whisper.cc:387-418) on one entry's [heads, T, nf]: standardise, median filter, mean over heads,
        rows s0 .. s0 + n."""
        x = median_filter(standardize_columns(probs), width)
        return x.mean(0, dtype=np.float32)[s0:s0 + n + 1].astype(np.float32)

    def detect_language(self, features):
        """SoftMax over the logits of config.json's lang_ids at the first decoder position (input <|startoftranscript|>):
        per entry {language token: probability}."""
        o = self.o
        ids = [int(i) for i in self.config["lang_ids"]]
        out = []
        for b in range(len(features)):
            memory = o.encode_features(np.asarray(features[b:b + 1], np.float32))[0]
            logits, _ = self.decode_sequence(memory, [o.sot], [])
            out.append(softmax_rows(logits[0, ids]))
        return ids, out
