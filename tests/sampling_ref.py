"""Restatements of the random-sampling path for the tests: Philox4x32-10 and the uniform of one draw (csrc/kernels/philox.h),
RandomSampler::sample on rows in exact integer / float64 arithmetic (src/sampling.cc:34-101, as the sampling kernel orders it),
and the processed log-probabilities of given Whisper token sequences under WhisperOracle (the SuppressTokens /
SuppressTokensBegin / ApplyTimestampRules of models/whisper.cc:742-860, teacher-forced)."""
import numpy as np

from oracle import ct2_oracle as O

M32 = 0xFFFFFFFF
f32 = np.float32


def philox4x32_10(counter, key):
    c, k = [int(v) & M32 for v in counter], [int(v) & M32 for v in key]
    for r in range(10):
        if r:
            k = [(k[0] + 0x9E3779B9) & M32, (k[1] + 0xBB67AE85) & M32]
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [((p1 >> 32) ^ c[1] ^ k[0]) & M32, p1 & M32, ((p0 >> 32) ^ c[3] ^ k[1]) & M32, p0 & M32]
    return c


def philox_uniform(seed, call, row, step):
    """u of one draw: the top 24 bits of word 0 of Philox4x32-10({step, row, call, 0}, {seed, 0}), over 2^24."""
    return (philox4x32_10([step, row, call, 0], [seed, 0])[0] >> 8) / float(1 << 24)


def kept_set(x, k):
    """Indices of the top k of row x by (value desc, index asc); k = 0 or k >= len(x) keeps every index."""
    x = np.asarray(x, np.float64)
    if k <= 0 or k >= x.size:
        return np.arange(x.size)
    order = np.lexsort((np.arange(x.size), -x))
    return np.sort(order[:k])


def random_sample_rows(x, k, temperature, seed, call, step=0, dtype="float32"):
    """RandomSampler::sample per row of x [rows, V] (values as the device holds them).  Returns ids, the log-probabilities
    round_to(dtype)(x[id] - max - log sum exp(x - max)) of the unscaled rows, and the distance of u * sum to the nearest
    cumulative boundary of the kept weights, relative to the sum (rows closer than float rounding can tip either way)."""
    from gpu_util import round_through
    x = np.asarray(x, np.float32)
    ids, logp, dist = [], [], []
    for r, row in enumerate(x):
        xd = row.astype(np.float64)
        m = xd.max()
        keep = kept_set(xd, k)
        w = np.exp((xd[keep] - m) / float(temperature))
        cum = np.cumsum(w)
        total = cum[-1]
        target = philox_uniform(seed, call, r, step) * total
        j = int(np.searchsorted(cum, target, side="right"))
        j = min(j, keep.size - 1)
        ids.append(int(keep[j]))
        dist.append(float(np.min(np.abs(np.concatenate([[0.0], cum]) - target)) / total))
        lse = m + np.log(np.exp(xd - m).sum())
        logp.append(float(xd[keep[j]] - lse))
    logp = round_through(np.array(logp, np.float32), dtype) if dtype != "float32" else np.array(logp, np.float32)
    return np.array(ids), logp, np.array(dist)


def process_logits(o, logits, step, histories, disable, disable_begin, timestamps, max_initial=50):
    """DisableTokens of one search step on logits [N, V] in place (WhisperOracle.generate's hook): SuppressTokens,
    SuppressTokensBegin at step 0 and, with timestamps, ApplyTimestampRules on each row's own history."""
    lowest = np.finfo(f32).min
    ts_begin, ts_end = o.no_timestamps + 1, o.vocab - 1
    for t in disable:
        logits[:, t] = lowest
    if step == 0:
        for t in disable_begin:
            logits[:, t] = lowest
    if not timestamps:
        return
    check = []
    for n in range(logits.shape[0]):
        seq = histories[n]
        logits[n, o.no_timestamps] = lowest
        if step == 0:
            logits[n, :ts_begin] = lowest
            logits[n, ts_begin + max_initial + 1:ts_end + 1] = lowest
        else:
            last = seq[step - 1]
            if last >= ts_begin:
                penult = seq[step - 2] if step - 1 > 0 else last
                if penult >= ts_begin:
                    logits[n, ts_begin:ts_end + 1] = lowest
                else:
                    logits[n, :o.eot] = lowest
                    logits[n, ts_begin:last] = lowest
                    check.append(n)
            else:
                check.append(n)
                for t in range(step - 1, -1, -1):
                    if seq[t] >= ts_begin:
                        logits[n, ts_begin:seq[t] + 1] = lowest
                        break
    if check:
        with np.errstate(over="ignore"):
            lp = O.softmax(logits, log=True)
        for n in check:
            ts = lp[n, ts_begin:ts_end + 1]
            mx = ts.max()
            if f32(mx + np.log(np.exp(ts - mx, dtype=f32).sum(dtype=f32))) > lp[n, :ts_begin].max():
                logits[n, :ts_begin] = lowest


def whisper_teacher_forced(o, features, prompts, entries, sequences, steps, disable, disable_begin, max_initial=50):
    """Processed logits of every position of the given sequences: row n continues prompts[entries[n]] with sequences[n]
    (the hypothesis tokens, without the end token).  Position s < min(len + 1, steps) is scored; returns per row the
    processed logits [positions, V] f32 (the row the sampler saw at that step)."""
    prompts = np.asarray(prompts)
    P = prompts.shape[1]
    timestamps = prompts[0, -1] != o.no_timestamps
    memory = o.encode_features(features)[np.asarray(entries)]
    o.start(memory, np.full(len(entries), memory.shape[1]), 1)
    rows = prompts[np.asarray(entries)]
    for t in range(P - 1):
        o.step(rows[:, t], t)
    n_pos = [min(len(s) + 1, steps) for s in sequences]
    histories = [list(s) + [o.eot] * steps for s in sequences]      # rows past their end are not scored
    out = [[] for _ in sequences]
    ids = rows[:, -1].astype(np.int64)
    for s in range(max(n_pos)):
        logits = o.step(ids, P - 1 + s).astype(f32)
        process_logits(o, logits, s, histories, disable, disable_begin, timestamps, max_initial)
        for n in range(len(sequences)):
            if s < n_pos[n]:
                out[n].append(logits[n].copy())
        ids = np.array([seq[s] if s < len(seq) else o.eot for seq in sequences], np.int64)
    return [np.stack(r) for r in out]
