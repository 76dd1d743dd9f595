"""Checks of generated-token log-probabilities (b200_set_logprobs) that need no GPU: a float64 numpy restatement of the definition in
include/b200llama.h, which the GPU tests compare against, and the engine loops' logprobs entries over fake plans."""
import numpy as np
import pytest


def logprob_rows(logits, chosen, n_top):
    """The definition over float32 logits [n, V] and the emitted ids [n] -> (chosen float64 [n], top ids int32 [n, N],
    top logprobs float64 [n, N]).  m is the first strict maximum over the entries > -inf (-inf when there is none), S = sum_j
    exp(l_j - m) in double; the top list takes the entries > -inf by value descending, equal values by the lower index, then the
    others (-inf, NaN) by index."""
    lg = np.asarray(logits, dtype=np.float32).reshape(len(chosen), -1)
    n, V = lg.shape
    out_c = np.empty(n)
    out_i = np.empty((n, n_top), np.int32)
    out_l = np.empty((n, n_top))
    idx = np.arange(V)
    for r in range(n):
        row = lg[r]
        valid = row > -np.inf
        m = np.float64(row[valid].max()) if valid.any() else -np.inf
        with np.errstate(invalid="ignore", over="ignore"):
            d = row.astype(np.float64) - m
            log_s = np.log(np.exp(d).sum())
        order = np.lexsort((idx, -np.where(valid, row, 0.0), ~valid))[:n_top]
        out_c[r] = d[chosen[r]] - log_s
        out_i[r] = order
        out_l[r] = d[order] - log_s
    return out_c, out_i, out_l


def test_definition_is_the_float64_log_softmax():
    from scipy.special import log_softmax

    rng = np.random.default_rng(2)
    lg = (rng.standard_normal((4, 3000)) * 5).astype(np.float32)
    chosen = np.array([0, 2999, 1234, 7])
    c, ids, lps = logprob_rows(lg, chosen, 20)
    ref = log_softmax(lg.astype(np.float64), axis=1)
    assert np.allclose(c, ref[np.arange(4), chosen], rtol=0, atol=1e-12)
    assert np.allclose(lps, np.take_along_axis(ref, ids.astype(np.int64), 1), rtol=0, atol=1e-12)
    assert np.array_equal(ids, np.argsort(-lg, axis=1, kind="stable")[:, :20])
    assert np.array_equal(ids[:, 0], lg.argmax(axis=1))


def test_ties_take_the_lower_index_first():
    lg = np.array([[1, 3, 3, 2, 3, -0.0, 0.0]], np.float32)
    _, ids, lps = logprob_rows(lg, np.array([4]), 7)
    assert list(ids[0]) == [1, 2, 4, 3, 0, 5, 6]  # -0 and +0 are equal values
    assert lps[0, 0] == lps[0, 1] == lps[0, 2]


def test_rows_without_a_finite_maximum():
    inf = np.inf
    lg = np.array([[-inf, -inf, -inf, -inf], [np.nan, 2, np.nan, -inf], [np.nan] * 4], np.float32)
    _, ids, lps = logprob_rows(lg, np.array([0, 1, 0]), 4)
    assert list(ids[0]) == [0, 1, 2, 3]  # no entry > -inf: the lowest index not yet taken
    assert list(ids[1]) == [1, 0, 2, 3]  # the value first, then NaN / -inf by index
    assert list(ids[2]) == [0, 1, 2, 3]
    assert np.isnan(lps).all()  # a NaN logit makes S NaN, and with it every value; -inf rows give (-inf) - (-inf)


# ---- the engine loops over fake plans --------------------------------------------------------------------------------------------

V = 50


def _next(tok, pos):
    return (7 * tok + 3 * pos + 1) % V


def _entry(slot, tok, pos):
    """What the fake plans report for a row: chosen encodes (slot, position), the one alternative is the row's input token."""
    return float(1000 * slot + pos), [(int(tok), -float(pos))]


class FakeLogprobPlan:
    """Every emitting call of the plan: ids from _next, and a logprobs table whose rows identify the call's rows."""

    def __init__(self, n_slots=4, rows=4, on=True):
        self.n_slots, self.rows, self.top_n = n_slots, rows, (1 if on else -1)
        self.table = []

    def logprobs_top_n(self):
        return self.top_n

    def last_logprobs(self):
        assert self.top_n >= 0, "logprobs are off"
        c = np.array([e[0] for e in self.table])
        ids = np.array([[i for i, _ in e[1]] for e in self.table], np.int32).reshape(len(c), 1)
        lps = np.array([[v for _, v in e[1]] for e in self.table]).reshape(len(c), 1)
        return c, ids, lps

    def batch_info(self):
        return self.n_slots, 0, 0.0

    def decode_multi_rows(self):
        return self.rows

    def slot_reset(self, slot):
        pass

    def prefill_slots(self, slots, starts, pieces):
        pass

    def forward_batch_prefill(self, tokens, start):
        pass

    def forward_decode(self, tok, pos, logits=True):
        self.table = [_entry(0, tok, pos)]
        return None, _next(tok, pos)

    def forward_decode_batch(self, slots, tokens, positions, sampling=None, logits=False):
        self.table = [_entry(s, t, p) for s, t, p in zip(slots, tokens, positions)]
        return np.array([_next(t, p) for t, p in zip(tokens, positions)], np.int32), None

    def forward_decode_multi(self, slot, tokens, start, logits=False):
        self.table = [_entry(0, t, start + i) for i, t in enumerate(tokens)]
        return np.array([_next(t, start + i) for i, t in enumerate(tokens)], np.int32), None

    def forward_step(self, rows, logits=False):
        self.table = [_entry(r[0], r[1], r[2]) if r[3] else (float("nan"), [(-1, float("nan"))]) for r in rows]
        return np.array([_next(r[1], r[2]) if r[3] else -1 for r in rows], np.int32), None


def _solo(latest, start, prompt, max_tokens, ctx, qwen=False):
    """The request's ids and the (token, position) each id was emitted from, by the reference loop."""
    eng = _engine()
    rows = []

    def fwd(t, p):
        rows.append((t, p))
        return _next(t, p)

    loop = eng.generate_tokens_qwen3 if qwen else eng.generate_tokens_llama
    ids = loop(fwd, latest, start, prompt, [V + 1], max_tokens, ctx)
    return ids, rows[len(rows) - len(ids):]


def _engine():
    import __graft_entry__

    return __graft_entry__.import_package().engine


REQS = [(1, 0, [3, 4, 5]), (2, 0, [9]), (7, 0, [1, 2, 3, 4, 5, 6])]


@pytest.mark.parametrize("qwen", [False, True])
def test_batch_entries_follow_the_generated_ids(qwen):
    eng = _engine()
    plan = FakeLogprobPlan()
    lp = []
    res = eng.generate_tokens_batch(plan, "QWEN_3" if qwen else "LLAMA_3", REQS, [V + 1], 12, 32, logprobs=lp)
    assert len(lp) == len(REQS)
    for i, (latest, start, prompt) in enumerate(REQS):
        ids, src = _solo(latest, start, prompt, 12, 32, qwen)
        assert res[i] == ids and len(lp[i]) == len(ids)
        assert [e for e in lp[i]] == [_entry(i, t, p) for t, p in src]  # prompt rows excluded


def test_batch_prefill_entries_follow_the_generated_ids():
    eng = _engine()
    plan = FakeLogprobPlan()
    lp = []
    res = eng.generate_tokens_batch_prefill(plan, "LLAMA_3", REQS, [V + 1], 12, 32, 4, logprobs=lp)
    for i, (latest, start, prompt) in enumerate(REQS):
        ids, src = _solo(latest, start, prompt, 12, 32)
        assert res[i] == ids and lp[i] == [_entry(i, t, p) for t, p in src]
    lp1 = []
    one = eng.generate_tokens_llama_batch_prefill(plan, 7, 0, [1, 2, 3, 4, 5, 6], [V + 1], 12, 32, 4, logprobs=lp1)
    ids, src = _solo(7, 0, [1, 2, 3, 4, 5, 6], 12, 32)
    assert one == ids and lp1 == [_entry(0, t, p) for t, p in src]


def test_lookahead_entries_skip_rejected_drafts():
    eng = _engine()
    plan = FakeLogprobPlan(rows=4)
    lp, stats = [], {}
    draft = lambda h: [h[-1]] * 3  # mostly wrong drafts: rows after the first mismatch are dropped
    res = eng.generate_tokens_lookahead(plan, "LLAMA_3", 1, 0, [3, 4, 5], [V + 1], 20, 32, draft=draft, stats=stats, logprobs=lp)
    ids, src = _solo(1, 0, [3, 4, 5], 20, 32)
    assert res == ids and lp == [_entry(0, t, p) for t, p in src]
    assert stats["drafted"] > stats["accepted"]


@pytest.mark.parametrize("qwen", [False, True])
def test_continuous_entries_are_per_request(qwen):
    eng = _engine()
    plan = FakeLogprobPlan(n_slots=2, rows=4)
    lp = []
    res = eng.generate_tokens_continuous(plan, "QWEN_3" if qwen else "LLAMA_3", REQS, [0, 0, 1], [V + 1], 12, 32, logprobs=lp)
    for i, (latest, start, prompt) in enumerate(REQS):
        ids, src = _solo(latest, start, prompt, 12, 32, qwen)
        assert res[i] == ids
        assert [(e[1][0][0], int(e[0]) % 1000) for e in lp[i]] == src  # each entry is its id's row: (input token, position)


def test_no_entries_while_logprobs_are_off():
    eng = _engine()
    plan = FakeLogprobPlan(n_slots=2, on=False)
    cb = eng.ContinuousBatcher(plan, "LLAMA_3", [V + 1], 12, 32)
    rid = cb.submit(1, 0, [3, 4])
    while cb.pending() or cb.running():
        cb.step()
    assert cb.results[rid] and cb.logprobs[rid] == []
    # the loops take no entries unless asked for them, and then read the plan's table
    assert eng.generate_tokens_batch(plan, "LLAMA_3", REQS[:2], [V + 1], 12, 32) == [_solo(*r, 12, 32)[0] for r in REQS[:2]]
    with pytest.raises(AssertionError):
        eng.generate_tokens_batch(plan, "LLAMA_3", REQS[:2], [V + 1], 12, 32, logprobs=[])
