"""-m gpu: the encoder-decoder attention kernel (attention_generic_kernel, seq2seq.cu) op by op, at the head sizes and key
counts of real models, against a float64 numpy restatement of dot_product_attention (src/layers/attention.cc:178-287).

Two references per case:
  * mirror: rounds to T where the kernel does, T(scale * q.k), T(softmax), T(sum p.v).  The kernel accumulates in float32,
    so it may differ from the mirror by the rounding of its last step (one ulp of T of the output) plus rare one-ulp flips of
    a probability (an ulp of T of p times |v|, below an ulp of the output).  Bound: MIRROR_ULPS ulps of T at the largest
    |output| of the (row, head); float32 uses 2e-5, as the other op tests do.
  * truth: no rounding.  Bound: the reference's tolerance class TOL (float32 2e-5) on the scale of the output.

A tolerance cannot see one wrong key among 1500 (about 1e-3 of the output), so the inputs make such mistakes large:
  * NaN in every key / value the kernel must not read: padded positions (MODE 0, 2), cache slots no ancestry entry points to
    and the stale slot (row, step) (MODE 1).  A stray read turns a checked output into NaN.
  * the last valid key of every row has a score near 0 while the others sit near -A, A = log(keys) + 1, so it carries about
    half the weight, and its value row is about +3 everywhere: dropping it moves the output by O(1).
  * MODE 2: every batch entry's values carry their own offset, so reading another entry's memory moves the output by O(1).
  * MODE 3: keys are a slowly turning unit vector (AR(1), correlation 0.85 between neighbours) and query t is A times key t,
    so key t leads, key t - 1 and the future key t + 1 score -A * 0.15: including j = t + 1 moves the output by O(1).
Every case also checks that these edits would move its outputs by far more than the bounds (test power, not kernel output).
"""
import math

import numpy as np
import pytest
import torch

from ctranslate2_b200 import ops
from gpu_util import DEV, TDT, TOL, gpu

DTYPES = ["float32", "float16", "bfloat16"]
MANT = {"float32": 23, "float16": 10, "bfloat16": 7}
MIN_NORMAL = {"float32": 2.0 ** -126, "float16": 2.0 ** -14, "bfloat16": 2.0 ** -126}
MIRROR_ULPS = 4
TRUTH_TOL = {"float32": 2e-5, "float16": TOL["float16"], "bfloat16": TOL["bfloat16"]}
SPIKE_VALUE = 3.0
INT_VIEW = {"float32": torch.int32, "float16": torch.int16, "bfloat16": torch.int16}


# ---------------- rounding helpers ----------------
def f32(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


def rt(x, dt):
    """float64 -> float32 -> T -> float64: the kernel's float -> T conversion (round to nearest even)."""
    t = torch.from_numpy(np.ascontiguousarray(np.asarray(x, np.float64).astype(np.float32)))
    return t.to(TDT[dt]).double().numpy()


def ulp(x, dt):
    a = np.maximum(np.abs(np.asarray(x, np.float64)), MIN_NORMAL[dt])
    return 2.0 ** (np.floor(np.log2(a)) - MANT[dt])


def to_dev(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(DEV).to(TDT[dt])


def host(t):
    return t.detach().double().cpu().numpy()


def bits(t, dt):
    return t.contiguous().view(INT_VIEW[dt]).cpu()


def misaligned(t):
    """The same values one element past a 16-byte boundary: the kernel's scalar load forms."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    return v


# ---------------- the reference ----------------
def attend(q, K, V, scale, dt):
    """One (query row, all heads): q [H, D], K / V [n, H, D] float64 (values as T holds them) -> (mirror, truth) [H, D]."""
    H, D = q.shape
    if K.shape[0] == 0:
        z = np.zeros((H, D))
        return z, z
    sc = f32(scale)
    dots = np.einsum("hd,nhd->hn", q, K)
    s = rt(f32(f32(dots) * sc), dt)
    e = np.exp(s - s.max(axis=1, keepdims=True))
    p = rt(e / e.sum(axis=1, keepdims=True), dt)
    mirror = rt(np.einsum("hn,nhd->hd", p, V), dt)
    t = dots * sc
    e = np.exp(t - t.max(axis=1, keepdims=True))
    truth = np.einsum("hn,nhd->hd", e / e.sum(axis=1, keepdims=True), V)
    return mirror, truth


def truth_only(q, K, V, scale):
    if K.shape[0] == 0:
        return np.zeros(q.shape)
    t = np.einsum("hd,nhd->hn", q, K) * f32(scale)
    e = np.exp(t - t.max(axis=1, keepdims=True))
    return np.einsum("hn,nhd->hd", e / e.sum(axis=1, keepdims=True), V)


REPORT = {}


def check_row(got, q, K, V, scale, dt, what, drop_last=True, extra=None):
    """got [H, D] (kernel) against the mirror and the truth of q over K / V; `extra` = (k, v) [H, D] of the key that must NOT
    be read.  Also asserts that dropping the last key (and adding `extra`) would break the bounds many times over."""
    H, D = q.shape
    mirror, truth = attend(q, K, V, scale, dt)
    assert np.isfinite(got).all(), f"{what}: non-finite output (a masked key or value was read)"
    mscale = np.abs(mirror).max(axis=1, keepdims=True)
    if dt == "float32":
        mtol = 2e-5 * np.maximum(1.0, mscale)
    else:
        mtol = MIRROR_ULPS * ulp(mscale, dt)
    merr = np.abs(got - mirror)
    assert (merr <= mtol).all(), f"{what}: {merr.max()} from the mirror (bound {mtol.min()})"
    tscale = np.maximum(1.0, np.abs(truth).max(axis=1, keepdims=True))
    ttol = TRUTH_TOL[dt] * tscale
    terr = np.abs(got - truth)
    assert (terr <= ttol).all(), f"{what}: {terr.max()} from the truth (bound {ttol.min()})"
    key = (dt, D)
    REPORT[key] = max(REPORT.get(key, 0.0), float((merr / ulp(mscale, dt)).max()))
    if drop_last and K.shape[0] >= 2:
        moved = np.abs(truth_only(q, K[:-1], V[:-1], scale) - truth).max()
        assert moved > 4 * ttol.max(), f"{what}: the inputs do not expose a dropped last key ({moved})"
    if extra is not None:
        K2 = np.concatenate([K, extra[0][None]], 0)
        V2 = np.concatenate([V, extra[1][None]], 0)
        moved = np.abs(truth_only(q, K2, V2, scale) - truth).max()
        assert moved > 4 * ttol.max(), f"{what}: the inputs do not expose a read of the next key ({moved})"


@pytest.fixture(scope="module", autouse=True)
def mirror_report():
    yield
    if REPORT:
        print("\nlargest mirror error, in ulps of T at the (row, head) output scale:")
        for (dt, D), e in sorted(REPORT.items()):
            print(f"  {dt:9s} head_dim {D:4d}: {e:.2f}")


# ---------------- input builders ----------------
def spike_a(nkeys):
    return max(3.0, math.log(max(nkeys, 1)) + 1.0)


def bulk_keys(rng, n, H, D):
    """[n, H, D]: component 0 in [-0.3, 0.3], a random direction in 1 .. D-2, 1 in the last component."""
    k = np.zeros((n, H, D))
    k[..., 0] = rng.uniform(-0.3, 0.3, (n, H))
    if D > 2:
        k[..., 1:D - 1] = rng.standard_normal((n, H, D - 2)) / math.sqrt(D - 2)
    k[..., D - 1] = 1.0
    return k


def spike_key(H, D):
    k = np.zeros((H, D))
    k[:, 0] = 1.0
    k[:, D - 1] = 1.0
    return k


def queries(rng, n, H, D, A):
    """[n, H, D]: score of a bulk key = A (eta - 1) + noise, of the spike key about 0 (with scale 1 / sqrt(D))."""
    q = np.zeros((n, H, D))
    q[..., 0] = A + rng.normal(0, 0.2, (n, H))
    if D > 2:
        q[..., 1:D - 1] = rng.normal(0, 0.3, (n, H, D - 2))
    q[..., D - 1] = -A
    return q * math.sqrt(D)


def values(rng, n, H, D):
    return rng.standard_normal((n, H, D))


def spike_value(rng, H, D):
    return SPIKE_VALUE + rng.normal(0, 0.2, (H, D))


def rows_to_check(n, must, rng, extra=6):
    picks = set(int(x) for x in must if 0 <= x < n)
    if n > len(picks):
        picks.update(int(x) for x in rng.choice(n, size=min(extra, n), replace=False))
    return sorted(picks)


# ---------------- MODE 0: encoder self-attention ----------------
# (head_dim, heads, S, lengths): "ragged" = batch 3 with lengths S, about S / 2 and 0; None = every key valid (Whisper's encoder)
ENC_CASES = [(8, 8, 33, "ragged"), (20, 20, 31, "ragged"), (64, 8, 3100, "ragged"), (64, 20, 1500, None), (96, 1, 32, "ragged"),
             (128, 8, 1500, "ragged"), (256, 8, 33, "ragged"), (64, 8, 1, "ragged")]


def make_encoder(dt, D, H, S, spec, seed):
    rng = np.random.default_rng(seed)
    lens = [S, (S + 1) // 2, 0] if spec == "ragged" else [S, S]
    B, d = len(lens), H * D
    qkv = np.full((B, S, 3, H, D), np.nan)
    for b, L in enumerate(lens):
        qkv[b, :, 0] = queries(rng, S, H, D, spike_a(L))
        if L:
            qkv[b, :L, 1] = bulk_keys(rng, L, H, D)
            qkv[b, :L, 2] = values(rng, L, H, D)
            qkv[b, L - 1, 1] = spike_key(H, D)
            qkv[b, L - 1, 2] = spike_value(rng, H, D)
    qkv = rt(qkv.reshape(B * S, 3 * d), dt)
    return qkv, lens


def run_encoder(qkv_t, lens, spec, H, D):
    lengths = torch.tensor(lens, dtype=torch.int32, device=DEV) if spec == "ragged" else None
    return ops.attention_encoder(qkv_t, H, D, len(lens), lengths=lengths)


@gpu
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("D,H,S,spec", ENC_CASES)
def test_encoder_attention(dt, D, H, S, spec):
    qkv, lens = make_encoder(dt, D, H, S, spec, seed=D * 1000 + S)
    B, d = len(lens), H * D
    qkv_t = to_dev(qkv, dt)
    out_t = run_encoder(qkv_t, lens, spec, H, D)
    out = host(out_t).reshape(B, S, H, D)
    x = qkv.reshape(B, S, 3, H, D)
    rng = np.random.default_rng(1)
    for b, L in enumerate(lens):
        if L == 0:
            assert (out[b] == 0).all() and not np.signbit(out[b]).any(), "a length-0 entry must give +0 rows"
            continue
        for t in rows_to_check(S, [0, L - 1, L, S - 1], rng):       # rows t >= L are computed too (and ignored by callers)
            check_row(out[b, t], x[b, t, 0], x[b, :L, 1], x[b, :L, 2], D ** -0.5, dt, f"MODE 0 b={b} t={t}")
    assert np.isfinite(out).all()
    # the scalar load forms (row starts not 16-byte aligned) sum in the same order: bit-identical
    if D in (64, 256) or S == 33:
        again = run_encoder(misaligned(qkv_t), lens, spec, H, D)
        assert torch.equal(bits(again, dt), bits(out_t, dt))


@gpu
def test_encoder_over_the_shared_memory_limit_raises():
    """S = 13000 at head_dim 64 needs 4 * (13000 + 64) floats per block, above 200 KB: an argument error, not a fault."""
    qkv = torch.zeros((13000, 3 * 64), dtype=torch.float16, device=DEV)
    with pytest.raises(ValueError):
        ops.attention_encoder(qkv, 1, 64, 1)
    with pytest.raises(ValueError):
        ops.attention_cross(torch.zeros((1, 64), dtype=torch.float16, device=DEV), qkv[:, :128].contiguous(), 1, 64, 1)
    qkv, lens = make_encoder("float16", 64, 1, 31, "ragged", seed=5)
    out = host(run_encoder(to_dev(qkv, "float16"), lens, "ragged", 1, 64)).reshape(3, 31, 1, 64)
    x = qkv.reshape(3, 31, 3, 1, 64)
    check_row(out[0, 30], x[0, 30, 0], x[0, :31, 1], x[0, :31, 2], 64 ** -0.5, "float16", "after the refused call")


# ---------------- MODE 2: cross-attention ----------------
# (head_dim, heads, S, beam, lengths): "ragged" = batch 3 with lengths S, about S / 2 and 1
CROSS_CASES = [(8, 8, 31, 4, "ragged"), (20, 8, 33, 5, "ragged"), (64, 8, 1500, 1, None), (64, 20, 1500, 5, None),
               (64, 8, 3100, 4, "ragged"), (96, 8, 32, 1, "ragged"), (128, 8, 1500, 4, "ragged"), (256, 1, 33, 5, "ragged")]


def make_cross(dt, D, H, S, beam, spec, seed):
    rng = np.random.default_rng(seed)
    lens = [S, S // 2 + 1, 1] if spec == "ragged" else [S, S]
    B, d = len(lens), H * D
    kv = np.full((B, S, 2, H, D), np.nan)
    q = np.zeros((B, beam, H, D))
    for b, L in enumerate(lens):
        kv[b, :L, 0] = bulk_keys(rng, L, H, D)
        kv[b, :L, 1] = values(rng, L, H, D) + 2.0 * (b - 1)          # the entry's own offset
        kv[b, L - 1, 0] = spike_key(H, D)
        kv[b, L - 1, 1] = spike_value(rng, H, D) + 2.0 * (b - 1)
        q[b] = queries(rng, beam, H, D, spike_a(L))
    return rt(q.reshape(B * beam, d), dt), rt(kv.reshape(B * S, 2 * d), dt), lens


@gpu
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("D,H,S,beam,spec", CROSS_CASES)
def test_cross_attention(dt, D, H, S, beam, spec):
    q, kv, lens = make_cross(dt, D, H, S, beam, spec, seed=D * 1000 + S + beam)
    B = len(lens)
    q_t, kv_t = to_dev(q, dt), to_dev(kv, dt)
    lengths = torch.tensor(lens, dtype=torch.int32, device=DEV) if spec == "ragged" else None
    out_t = ops.attention_cross(q_t, kv_t, H, D, beam, lengths=lengths)
    out = host(out_t).reshape(B, beam, H, D)
    x = kv.reshape(B, S, 2, H, D)
    qq = q.reshape(B, beam, H, D)
    for b, L in enumerate(lens):
        for t in range(beam):
            check_row(out[b, t], qq[b, t], x[b, :L, 0], x[b, :L, 1], D ** -0.5, dt, f"MODE 2 b={b} beam={t}")
    if D in (64, 256) or S == 33:
        again = ops.attention_cross(misaligned(q_t), kv_t, H, D, beam, lengths=lengths)
        assert torch.equal(bits(again, dt), bits(out_t, dt))


def fma_scores(q, K, scale):
    """The kernel's own float32 scores: one fused multiply-add per element in head-dim order, then * scale.
    q [D], K [n, D] float64 (values as T holds them) -> float64 [n]."""
    dot = np.zeros(K.shape[0])
    for i in range(q.shape[0]):
        dot = f32(dot + q[i] * K[:, i])             # the product of two floats is exact in float64
    return f32(dot * f32(scale))


@gpu
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("D,S,beam", [(64, 1500, 1), (64, 200, 3), (20, 37, 2)])
def test_cross_attention_score_capture(dt, D, S, beam):
    """Whisper.align's capture: T(scale * q.k) of the selected heads, bit-for-bit; a head listed twice fills both slots;
    positions past the entry's length and unselected slots keep what was there; the context equals the plain call's."""
    H, first, total = 8, 1, 5
    q, kv, lens = make_cross(dt, D, H, S, beam, "ragged", seed=77 + D + S)
    B = len(lens)
    q_t, kv_t = to_dev(q, dt), to_dev(kv, dt)
    lengths = torch.tensor(lens, dtype=torch.int32, device=DEV)
    slots = {2: [0], 5: [1, 2], 7: [3]}                               # head 5 twice; slot `first + k` for bit k
    masks = np.zeros(H, np.int64)
    for h, ks in slots.items():
        for k in ks:
            masks[h] |= 1 << k
    masks_t = torch.tensor(masks.astype(np.int32), dtype=torch.int32, device=DEV)
    sentinel = -12345.0
    cap = torch.full((B, total, beam, S), sentinel, dtype=torch.float32, device=DEV)
    out_cap = ops.attention_cross(q_t, kv_t, H, D, beam, lengths=lengths, capture=cap, masks=masks_t, first=first,
                                  total=total)
    out = ops.attention_cross(q_t, kv_t, H, D, beam, lengths=lengths)
    assert torch.equal(bits(out_cap, dt), bits(out, dt))
    got = cap.cpu().numpy().astype(np.float64)
    x = kv.reshape(B, S, 2, H, D)
    qq = q.reshape(B, beam, H, D)
    written = np.zeros(got.shape, bool)
    for b, L in enumerate(lens):
        for t in range(beam):
            for h, ks in slots.items():
                want = rt(fma_scores(qq[b, t, h], x[b, :L, 0, h], D ** -0.5), dt)
                for k in ks:
                    np.testing.assert_array_equal(got[b, first + k, t, :L], want)
                    written[b, first + k, t, :L] = True
    assert (got[~written] == sentinel).all()


# ---------------- MODE 1: one-token decoder self-attention over the beam-remapped cache ----------------
# (head_dim, heads, keys = step + 1, batch, beam)
SELF_CASES = [(8, 8, 33, 2, 4), (20, 20, 32, 2, 5), (64, 8, 1500, 2, 4), (64, 8, 3100, 1, 4), (96, 8, 31, 2, 2),
              (128, 8, 1500, 1, 5), (256, 8, 33, 2, 4), (64, 1, 1, 2, 4)]


def ancestry(rng, batch, beam, step, max_len):
    """The read table a beam search leaves after `step` steps: every step each row continues a random beam of its entry
    (beam_update_kernel: anc_w[row][:t] = anc_r[parent][:t], anc_w[row][t] = parent)."""
    N = batch * beam
    anc = np.zeros((N, max_len), np.int64)
    for t in range(step):
        new = anc.copy()
        for r in range(N):
            parent = (r // beam) * beam + int(rng.integers(beam))
            new[r, :t] = anc[parent, :t]
            new[r, t] = parent
        anc = new
    return anc


@gpu
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("D,H,nkeys,batch,beam", SELF_CASES)
def test_beam_self_attention(dt, D, H, nkeys, batch, beam):
    rng = np.random.default_rng(D * 100 + nkeys + beam)
    step, max_len, N, d = nkeys - 1, nkeys + 3, batch * beam, H * D
    anc = ancestry(rng, batch, beam, step, max_len)
    tables = np.zeros((2, N, max_len), np.int64)
    tables[step & 1] = anc
    tables[1 - (step & 1)] = rng.integers(0, N, (N, max_len))         # the other parity: never read
    kc = np.full((N, max_len, H, D), np.nan)                          # unreferenced slots, (row, step) and j > step: NaN
    vc = np.full((N, max_len, H, D), np.nan)
    for j in range(step):
        for r in set(anc[:, j].tolist()):
            kc[r, j] = bulk_keys(rng, 1, H, D)[0]
            vc[r, j] = values(rng, 1, H, D)[0]
    qkv = np.zeros((N, 3, H, D))
    qkv[:, 0] = queries(rng, N, H, D, spike_a(nkeys))
    qkv[:, 1] = spike_key(H, D)[None]
    for n in range(N):
        qkv[n, 2] = spike_value(rng, H, D) + 0.5 * n                   # each row's own value: a swapped row shows
    qkv, kc, vc = rt(qkv, dt), rt(kc, dt), rt(vc, dt)
    qkv_t = to_dev(qkv.reshape(N, 3 * d), dt)
    kc_t, vc_t = to_dev(kc.reshape(N, max_len, d), dt), to_dev(vc.reshape(N, max_len, d), dt)
    kc0, vc0 = bits(kc_t, dt).clone(), bits(vc_t, dt).clone()
    anc_t = torch.tensor(tables.astype(np.int32), dtype=torch.int32, device=DEV)
    step_t = torch.tensor([step], dtype=torch.int32, device=DEV)
    out_t = ops.attention_beam_self(qkv_t, kc_t, vc_t, anc_t, step_t, H, D)
    out = host(out_t).reshape(N, H, D)
    for n in range(N):
        K = np.concatenate([kc[anc[n, :step], np.arange(step)], qkv[n, 1][None]], 0)
        V = np.concatenate([vc[anc[n, :step], np.arange(step)], qkv[n, 2][None]], 0)
        check_row(out[n], qkv[n, 0], K, V, D ** -0.5, dt, f"MODE 1 row={n}")
    # the rows' new k / v land at (row, step) bit-exactly and nothing else in the caches changes
    new = bits(qkv_t, dt).view(N, 3, d)
    kc0[:, step], vc0[:, step] = new[:, 1], new[:, 2]
    assert torch.equal(bits(kc_t, dt), kc0)
    assert torch.equal(bits(vc_t, dt), vc0)
    if D in (64, 256) or nkeys == 33:
        again = ops.attention_beam_self(misaligned(qkv_t), kc_t, vc_t, anc_t, step_t, H, D)
        assert torch.equal(bits(again, dt), bits(out_t, dt))


# ---------------- MODE 3: teacher-forced causal self-attention ----------------
# (head_dim, heads, time, batch); time 1 is Whisper.detect_language
CAUSAL_CASES = [(8, 8, 33, 2), (20, 20, 31, 2), (64, 8, 1500, 2), (64, 8, 3100, 1), (96, 8, 32, 3), (128, 8, 1500, 1),
                (256, 8, 33, 2), (64, 20, 1, 4)]


def make_causal(dt, D, H, T, B, seed):
    rng = np.random.default_rng(seed)
    A, rho = (9.0 if D >= 64 else 6.0), 0.85
    w = np.zeros((B, T, H, D - 1))
    w[:, 0] = rng.standard_normal((B, H, D - 1))
    for t in range(1, T):
        w[:, t] = rho * w[:, t - 1] / np.linalg.norm(w[:, t - 1], axis=-1, keepdims=True) \
            + math.sqrt(1 - rho * rho) * rng.standard_normal((B, H, D - 1)) / math.sqrt(D - 1)
    w /= np.linalg.norm(w, axis=-1, keepdims=True)
    qkv = np.zeros((B, T, 3, H, D))
    qkv[..., 0, :, :D - 1] = A * math.sqrt(D) * w
    qkv[..., 0, :, D - 1] = -A * math.sqrt(D)
    qkv[..., 1, :, :D - 1] = w
    qkv[..., 1, :, D - 1] = 1.0
    qkv[..., 2, :, :] = 2.0 * rng.standard_normal((B, T, H, D))
    return rt(qkv, dt)


@gpu
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("D,H,T,B", CAUSAL_CASES)
def test_causal_attention(dt, D, H, T, B):
    x = make_causal(dt, D, H, T, B, seed=D * 10 + T)
    d = H * D
    qkv_t = to_dev(x.reshape(B * T, 3 * d), dt)
    out_t = ops.attention_causal(qkv_t, H, D, B)
    out = host(out_t).reshape(B, T, H, D)
    rng = np.random.default_rng(2)
    for b in range(B):
        for t in rows_to_check(T, [0, 1, 31, 32, 33, T - 2, T - 1], rng):
            nxt = (x[b, t + 1, 1], x[b, t + 1, 2]) if t + 1 < T else None
            check_row(out[b, t], x[b, t, 0], x[b, :t + 1, 1], x[b, :t + 1, 2], D ** -0.5, dt, f"MODE 3 b={b} t={t}",
                      extra=nxt)
    if D in (64, 256) or T == 33:
        again = ops.attention_causal(misaligned(qkv_t), H, D, B)
        assert torch.equal(bits(again, dt), bits(out_t, dt))


# ---------------- the whole model at OPUS-MT size ----------------
# Bounds, from fp16 rounding (unit roundoff u = 2^-11): every encoder layer rounds its activations to T at about ten points
# (Q/K/V, scores, probabilities, context, output projection, residual, LayerNorm, the two FFN Dense, residual, LayerNorm); the
# post-norm LayerNorms keep the residual stream at unit scale, so independent roundings add in quadrature: about
# sqrt(10) * u / sqrt(3) = 9e-4 relative RMS per layer, sqrt(6) times that over the 6 encoder layers (2.2e-3), and a factor
# 4.5 for the gain of the random weights: 1e-2.  int8_float16 quantizes the input row of every Dense to int8: relative RMS
# error (amax / 127) / sqrt(12) / rms = 9e-3 per Dense for rows with amax / rms = 4, four Dense per layer, 24 in the
# encoder: sqrt(24) * 9e-3 = 4.4e-2, bound 0.1.  The decoder output adds the 6 decoder layers: sqrt(2) times the encoder
# bound.  A log-probability moves by that relative error times the spread of the logits (the standard deviation of the
# float32 log-probabilities of random targets), plus half an ulp of fp16 at |log p| (4e-3 at 8).
ENCODE_REL_RMS = {"float16": 1e-2, "int8_float16": 0.1}


@gpu
@pytest.mark.parametrize("compute", ["float16", "int8_float16"])
def test_opus_size_encode_and_score_half_precision(tmp_path, compute):
    """Transformer-base 6+6, d 512, 8 heads (head_dim 64), vocabulary cut to 4000: Translator.encode against the float32
    oracle and score_batch against the float32 Translator — the head_dim-64 half-precision attention as the engine calls it
    (scale, head split, source lengths)."""
    import os
    import sys
    from ctranslate2_b200.translator import Translator
    from oracle import ct2_oracle as O
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    from ref_cuda_worker import opus_small
    mdir = str(tmp_path / "opus_small")
    srcs = opus_small(mdir)
    t = Translator(mdir, compute_type=compute)
    mem = t.encode(srcs)
    oracle = O.Seq2SeqOracle.from_dir(mdir, compute_type="float32")
    S = max(len(r) for r in srcs)
    padded = np.zeros((len(srcs), S), np.int64)
    for b, r in enumerate(srcs):
        padded[b, :len(r)] = r
    want = oracle.encode(padded, np.array([len(r) for r in srcs]))
    diff = np.concatenate([(mem[b, :len(r)] - want[b, :len(r)]).ravel() for b, r in enumerate(srcs)])
    ref = np.concatenate([want[b, :len(r)].ravel() for b, r in enumerate(srcs)])
    rel = float(np.sqrt((diff.astype(np.float64) ** 2).sum() / (ref.astype(np.float64) ** 2).sum()))
    print(f"\n{compute}: encoder memory relative RMS vs float32 oracle {rel:.2e}")
    assert rel <= ENCODE_REL_RMS[compute], rel
    rng = np.random.default_rng(12)
    tgts = [[int(x) for x in rng.integers(3, 4000, size=int(rng.integers(10, 40)))] for _ in srcs]
    half = t.score_batch(srcs, tgts)
    t.close()
    t32 = Translator(mdir, compute_type="float32")
    full = t32.score_batch(srcs, tgts)
    t32.close()
    a = np.concatenate([r.log_probs for r in half])
    b = np.concatenate([r.log_probs for r in full])
    assert a.size == b.size == sum(len(x) + 1 for x in tgts)
    eps = np.sqrt(2.0) * ENCODE_REL_RMS[compute]
    spread = float(b.std())
    err = np.abs(a - b)
    print(f"{compute}: log-prob error max {err.max():.3e} mean {err.mean():.3e}, logit spread {spread:.3f}")
    assert err.mean() <= eps * spread + 4e-3, err.mean()
    assert err.max() <= 5 * eps * spread + 8e-3, err.max()
