"""Checks of token scoring (b200_score_tokens) that need no GPU: a float64 numpy restatement of the definition in include/b200llama.h,
which the GPU tests compare against, and engine.score_sequence / engine.perplexity over a fake plan."""
import math

import numpy as np
import pytest


def score_rows(logits, targets):
    """The definition: greedy = the first index of the strict maximum m; S = sum_j exp(l_j - m) in double; logprob = (l_t - m) - log(S)
    for target t, NaN for t == -1.  logits float32 [n, vocab] -> (float64 [n], int32 [n])."""
    lg = np.asarray(logits, dtype=np.float32).reshape(len(targets), -1)
    ids = np.argmax(lg, axis=1).astype(np.int32)  # first occurrence of the maximum
    d = lg.astype(np.float64) - lg[np.arange(len(ids)), ids].astype(np.float64)[:, None]
    log_s = np.log(np.exp(d).sum(axis=1))
    t = np.asarray(targets)
    lp = np.where(t >= 0, d[np.arange(len(t)), np.maximum(t, 0)] - log_s, np.nan)
    return lp, ids


def test_definition_is_the_float64_log_softmax():
    from scipy.special import log_softmax

    rng = np.random.default_rng(1)
    lg = (rng.standard_normal((5, 1000)) * 4).astype(np.float32)
    t = np.array([0, 999, 17, -1, 500])
    lp, ids = score_rows(lg, t)
    ref = log_softmax(lg.astype(np.float64), axis=1)
    assert np.allclose(lp[t >= 0], ref[np.flatnonzero(t >= 0), t[t >= 0]], rtol=0, atol=1e-12)
    assert np.isnan(lp[3])
    assert np.array_equal(ids, lg.argmax(axis=1))


def test_ties_take_the_first_index():
    lg = np.array([[1, 3, 3, 2], [5, 5, 5, 5], [-np.inf, 0, 0, -np.inf]], np.float32)
    lp, ids = score_rows(lg, np.array([1, 3, 2]))
    assert list(ids) == [1, 0, 1]
    assert lp[0] == pytest.approx(-math.log(2 + math.exp(-1) + math.exp(-2)), abs=1e-15)
    assert lp[1] == pytest.approx(math.log(0.25), abs=1e-15)
    assert lp[2] == pytest.approx(math.log(0.5), abs=1e-15)


def test_saturated_softmax_is_finite():
    lg = np.zeros((1, 128256), np.float32)
    lg[0, 77] = 3.0e4
    lp, ids = score_rows(lg, np.array([77]))
    assert ids[0] == 77 and lp[0] == 0.0
    lp2, _ = score_rows(lg, np.array([5]))
    assert np.isfinite(lp2[0]) and lp2[0] == pytest.approx(-3.0e4, rel=1e-12)


class FakePlan:
    """Records score_tokens calls; row i's "log-probability" encodes (position, target) so the caller's assembly can be checked."""

    def __init__(self, prefill_batch_size):
        self.prefill_batch_size = prefill_batch_size
        self.calls = []
        self.resets = 0

    def kv_reset(self):
        self.resets += 1

    def score_tokens(self, tokens, start_pos, targets):
        tokens, targets = np.asarray(tokens), np.asarray(targets)
        limit = self.prefill_batch_size if self.prefill_batch_size > 1 else 10 ** 9
        assert 1 <= len(tokens) <= limit and len(targets) == len(tokens)
        self.calls.append((start_pos, tokens.tolist(), targets.tolist()))
        pos = start_pos + np.arange(len(tokens))
        lp = np.where(targets >= 0, -(pos + targets / 1000.0), np.nan)
        return lp, (tokens + 1).astype(np.int32)


@pytest.mark.parametrize("pb,n", [(16, 40), (16, 16), (16, 17), (1, 23), (0, 5), (64, 1)])
def test_score_sequence_chunks_and_cross_chunk_targets(pkg, pb, n):
    E = pkg.engine
    toks = [(7 * i + 3) % 101 for i in range(n)]
    plan = FakePlan(pb)
    lp, ids = E.score_sequence(plan, toks, start_pos=5)
    chunk = pb if pb > 1 else n
    assert [c[0] for c in plan.calls] == [5 + a for a in range(0, n, chunk)]
    assert sum(len(c[1]) for c in plan.calls) == n
    for start, t, tg in plan.calls:  # every row's target is the next token of the whole sequence, -1 at its end
        for k, tok in enumerate(t):
            i = start - 5 + k
            assert tok == toks[i] and tg[k] == (toks[i + 1] if i + 1 < n else -1)
    want = [-((5 + i) + toks[i + 1] / 1000.0) for i in range(n - 1)]
    assert np.array_equal(lp[:-1], want) and np.isnan(lp[-1])
    assert lp.dtype == np.float64 and ids.dtype == np.int32 and list(ids) == [t + 1 for t in toks]


def test_perplexity_resets_and_averages_positions_1_to_n_minus_1(pkg):
    E = pkg.engine
    toks = [3, 1, 4, 1, 5, 9, 2, 6]
    plan = FakePlan(3)
    ppl = E.perplexity(plan, toks)
    assert plan.resets == 1 and plan.calls[0][0] == 0
    mean = np.mean([-(i + toks[i + 1] / 1000.0) for i in range(len(toks) - 1)])
    assert ppl == pytest.approx(math.exp(-mean), rel=1e-15)
    with pytest.raises(ValueError):
        E.perplexity(plan, [1])
