"""-m gpu: the beam-search row kernel (beam_rows_kernel, seq2seq.cu) at real vocabulary sizes, against a numpy restatement of
one BeamSearch::search step (src/decoding.cc:425-720) per row: score = T(T(x - max - logsumexp) + cum), candidates ordered by
(score desc, flattened index asc), flattened index = (row % beam) * vocab + j, and (-inf, -1) past the vocabulary.

The kernel has two algorithms: a threshold fast path that ranks at most kCandCap = 1024 elements at or above a bound, and
per-thread sorted lists merged by block-wide arg-max rounds when more elements than that tie at the bound (every beam but the
first at the first step: their cumulative score is the lowest value of T).  Rows here take both, and rows with exactly 1023,
1024 and 1025 elements at the bound sit on both sides of the switch.

The kernel sums the exponentials in float32 (expf within 2 ulps, exp2f for 2-byte T) in its own order, so its log-sum-exp
carries an absolute error of about the relative error of that sum: at most (vocab / 512 + 16) float32 roundings, one per
term a thread adds in sequence plus the block tree and expf.  For 2-byte T that is far below an ulp of the score; in float32
it is up to a few ulps of a score near -log(vocab).  So where the logits do not tie the test asks for scores within one ulp
of T plus that error, a legal order and no omitted element above the last candidate by more than the same amount.  Where the rows
are built from exact ties, ids must match exactly.
"""
import numpy as np
import pytest
import torch

from ctranslate2_b200 import ops
from gpu_util import DEV, TDT, gpu

DTYPES = ["float32", "float16", "bfloat16"]
MANT = {"float32": 23, "float16": 10, "bfloat16": 7}
LOWEST = {"float32": -3.4028234663852886e38, "float16": -65504.0, "bfloat16": -3.3895313892515355e38}
PAD_VALUE = 100.0              # the columns between vocab and vocab_ld: a read of one would become the row's best element


def f32(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


def rt(x, dt):
    t = torch.from_numpy(np.ascontiguousarray(np.asarray(x, np.float64).astype(np.float32)))
    return t.to(TDT[dt]).double().numpy()


def ulp(x, dt):
    a = np.maximum(np.abs(np.asarray(x, np.float64)), 2.0 ** -100)
    return 2.0 ** (np.floor(np.log2(a)) - MANT[dt])


def tol(want, vocab, dt):
    """One ulp of T plus the float32 error of the kernel's log-sum-exp (module docstring)."""
    return ulp(want, dt) + (vocab / 512 + 16) * 2.0 ** -24


def ref_scores(x, cum, dt):
    """One row: x [vocab] float64 as T holds it, cum as T holds it -> the kernel's scores, float64."""
    m = x.max()
    logs = f32(np.log(np.exp(x - m).sum()))
    return rt(f32(rt(f32(f32(x - m) - logs), dt) + cum), dt)


def ref_order(ref, nc):
    order = np.lexsort((np.arange(ref.size), -ref))        # score desc, index asc
    return order[:nc]


def run(logits, cum, dt, beam, vocab, step=0, min_length=0, end_ids=None):
    x = torch.from_numpy(np.ascontiguousarray(logits, np.float32)).to(DEV).to(TDT[dt])
    c = torch.from_numpy(np.ascontiguousarray(cum, np.float32)).to(DEV).to(TDT[dt])
    step_t = torch.tensor([step], dtype=torch.int32, device=DEV)
    e = None if end_ids is None else torch.tensor(end_ids, dtype=torch.int32, device=DEV)
    s, i = ops.beam_rows(x, c, step_t, beam, vocab, min_length=min_length, end_ids=e)
    return s.double().cpu().numpy(), i.cpu().numpy(), x.double().cpu().numpy()


def check_relaxed(got_s, got_i, ref, base, what, dt):
    nc = got_s.size
    ids = got_i - base
    assert ((ids >= 0) & (ids < ref.size)).all(), f"{what}: id outside the row: {got_i}"
    assert np.unique(ids).size == nc, f"{what}: repeated id {got_i}"
    want = ref[ids]
    assert (np.abs(got_s - want) <= tol(want, ref.size, dt)).all(), f"{what}: scores {got_s} vs {want}"
    for k in range(nc - 1):
        assert got_s[k] > got_s[k + 1] or (got_s[k] == got_s[k + 1] and got_i[k] < got_i[k + 1]), f"{what}: order {k}"
    rest = np.delete(ref, ids)
    if rest.size:
        assert rest.max() <= got_s[-1] + tol(got_s[-1], ref.size, dt), f"{what}: omitted {rest.max()} > last {got_s[-1]}"


def check_exact(got_s, got_i, ref, base, what, dt):
    want = ref_order(ref, got_s.size)
    np.testing.assert_array_equal(got_i, base + want, err_msg=what)
    assert (np.abs(got_s - ref[want]) <= tol(ref[want], ref.size, dt)).all(), f"{what}: scores {got_s} vs {ref[want]}"


def tie_row(rng, vocab, count, above):
    """`count` elements at or above the bound: `above` distinct values above it, the rest tied at 2.0; all others lower."""
    x = rng.uniform(-3.0, -1.0, vocab)
    pos = rng.choice(vocab, size=count, replace=False)
    x[pos] = 2.0
    x[pos[:above]] = 3.0 + 0.25 * np.arange(above)
    return x


@gpu
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("vocab,vocab_ld", [(58101, 58101), (58101, 58104), (32000, 32000)])
@pytest.mark.parametrize("beam", [1, 2, 4, 5, 8])
def test_beam_rows(dt, vocab, vocab_ld, beam):
    """Entries: 0 random logits and scores; 1 the first step (beams > 0 at the lowest T: everything ties); 2.. rows with
    exactly 1023 / 1024 / 1025 elements at the bound, all tied or nc - 1 above and the rest tied."""
    rng = np.random.default_rng(vocab + 7 * beam + vocab_ld)
    nc = 2 * beam
    tie_kinds = [(count, above) for count in (1023, 1024, 1025) for above in (0, nc - 1)]
    batch = 2 + len(tie_kinds)
    N = batch * beam
    logits = np.full((N, vocab_ld), PAD_VALUE)
    cum = np.zeros(N)
    for k in range(beam):
        logits[k, :vocab] = rng.normal(0, 2, vocab)
        cum[k] = -rng.uniform(0, 5)
        logits[beam + k, :vocab] = rng.uniform(-1, 1, vocab)              # log-probs in [-12.1, -10.1]: no fp16 overflow edge
        cum[beam + k] = 0.0 if k == 0 else LOWEST[dt]
    for e, (count, above) in enumerate(tie_kinds):
        for k in range(beam):
            logits[(2 + e) * beam + k, :vocab] = tie_row(rng, vocab, count, above)
    logits, cum = rt(logits, dt), rt(cum, dt)
    got_s, got_i, _ = run(logits, cum, dt, beam, vocab)
    for r in range(N):
        e, k = divmod(r, beam)
        ref = ref_scores(logits[r, :vocab], cum[r], dt)
        what = f"{dt} vocab={vocab}/{vocab_ld} beam={beam} entry={e} row={k}"
        if e == 0 or (e == 1 and k == 0):
            check_relaxed(got_s[r], got_i[r], ref, k * vocab, what, dt)
        else:
            check_exact(got_s[r], got_i[r], ref, k * vocab, what, dt)
        if e == 1 and k > 0:
            np.testing.assert_array_equal(got_i[r], k * vocab + np.arange(nc), err_msg=what)


@gpu
@pytest.mark.parametrize("dt", DTYPES)
def test_beam_rows_min_length_masks_end_ids(dt):
    """DisableTokens of the end ids while step < min_length (decoding.cc:60-81): the best two logits are end ids."""
    vocab, beam = 58101, 4
    rng = np.random.default_rng(3)
    ends = [2, 40000]
    logits = rng.normal(0, 2, (2 * beam, vocab))
    logits[:, ends] = 12.0
    logits, cum = rt(logits, dt), rt(-rng.uniform(0, 3, 2 * beam), dt)
    for step, masked in ((0, True), (1, False)):
        got_s, got_i, after = run(logits, cum, dt, beam, vocab, step=step, min_length=1, end_ids=ends)
        for r in range(2 * beam):
            x = logits[r].copy()
            if masked:
                x[ends] = LOWEST[dt]
            ref = ref_scores(x, cum[r], dt)
            base = (r % beam) * vocab
            check_relaxed(got_s[r], got_i[r], ref, base, f"{dt} step={step} row={r}", dt)
            assert (np.isin(got_i[r] - base, ends).sum() == 0) == masked
            np.testing.assert_array_equal(after[r, ends], LOWEST[dt] if masked else logits[r, ends])


@gpu
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("vocab,vocab_ld,beam", [(5, 5, 4), (7, 8, 8), (3, 3, 2)])
def test_beam_rows_vocabulary_smaller_than_candidates(dt, vocab, vocab_ld, beam):
    rng = np.random.default_rng(vocab)
    N = 2 * beam
    logits = np.full((N, vocab_ld), PAD_VALUE)
    logits[:, :vocab] = rng.normal(0, 2, (N, vocab))
    cum = np.zeros(N)
    cum[beam + 1:] = LOWEST[dt]
    logits, cum = rt(logits, dt), rt(cum, dt)
    got_s, got_i, _ = run(logits, cum, dt, beam, vocab)
    for r in range(N):
        ref = ref_scores(logits[r, :vocab], cum[r], dt)
        base = (r % beam) * vocab
        if cum[r] == LOWEST[dt]:                                  # every element ties
            check_exact(got_s[r, :vocab], got_i[r, :vocab], ref, base, f"{dt} row={r}", dt)
        else:
            check_relaxed(got_s[r, :vocab], got_i[r, :vocab], ref, base, f"{dt} row={r}", dt)
        assert (got_i[r, vocab:] == -1).all() and np.isneginf(got_s[r, vocab:]).all()


@gpu
def test_beam_rows_refuses_more_than_eight_beams():
    x = torch.zeros((9, 100), dtype=torch.float16, device=DEV)
    c = torch.zeros(9, dtype=torch.float16, device=DEV)
    step = torch.zeros(1, dtype=torch.int32, device=DEV)
    with pytest.raises(ValueError):
        ops.beam_rows(x, c, step, 9, 100)
    s, i = ops.beam_rows(x[:8], c[:8], step, 8, 100)
    assert (i.cpu().numpy() == np.arange(16)[None] + 100 * np.arange(8)[:, None]).all()
