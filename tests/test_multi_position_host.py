"""CPU checks of the multi-position step: engine.generate_tokens_lookahead equals generate_tokens_llama on a stand-in plan whose
forward_decode_multi runs a toy deterministic model over its own cache (so a rejected draft's rows are really written), for any
draft function; Qwen-loop types are refused; prompt_lookup proposes what followed the latest earlier occurrence."""
import pytest

V = 97


def _next(cache, pos):
    h = 0
    for t in cache[:pos + 1]:
        h = (h * 131 + t + 7) % 1000003
    return h % V


class _ToyPlan:
    """One sequence: row i writes tokens[i] at start + i, then its id reads positions 0 .. start + i."""

    def __init__(self, rows=8):
        self.rows, self.cache, self.calls = rows, {}, []

    def decode_multi_rows(self):
        return self.rows

    def forward_decode_multi(self, slot, tokens, start):
        assert slot == -1 and 1 <= len(tokens) <= self.rows
        self.calls.append(len(tokens))
        for i, t in enumerate(tokens):
            self.cache[start + i] = t
        cache = [self.cache.get(p, 0) for p in range(start + len(tokens))]
        return [_next(cache, start + i) for i in range(len(tokens))], None


def _reference(latest, start, prompt, stop, budget, ctx):
    from_cache = {}

    def fwd(t, p):
        from_cache[p] = t
        return _next([from_cache.get(q, 0) for q in range(p + 1)], p)
    return fwd


@pytest.mark.parametrize("drafter", ["prompt_lookup", "right", "wrong", "none", "half"])
@pytest.mark.parametrize("stop,budget", [([], 70), (None, 70), ([], 23), ([], -1)])
def test_lookahead_equals_llama_loop(pkg, drafter, stop, budget):
    E = pkg.engine
    prompt = [3, 4, 5, 3, 4, 6, 3, 4, 5, 9]
    ctx = 80
    full_run = E.generate_tokens_llama(_reference(1, 2, prompt, [], 70, ctx), 1, 2, prompt, [], 70, ctx)
    if stop is None:
        stop = [full_run[len(full_run) // 3]]
    want = E.generate_tokens_llama(_reference(1, 2, prompt, stop, budget, ctx), 1, 2, prompt, stop, budget, ctx)
    full = [1] + prompt + full_run
    draft = {"prompt_lookup": E.prompt_lookup,
             "right": lambda h: full[len(h):len(h) + 12],
             "wrong": lambda h: [(t + 1) % V for t in full[len(h):len(h) + 12]],
             "none": lambda h: [],
             "half": lambda h: full[len(h):len(h) + 2] + [(t + 1) % V for t in full[len(h) + 2:len(h) + 5]]}[drafter]
    plan = _ToyPlan()
    stats = {}
    got = E.generate_tokens_lookahead(plan, "LLAMA_3", 1, 2, prompt, stop, budget, ctx, draft=draft, stats=stats)
    assert got == want
    assert max(plan.calls) <= 8
    if drafter == "right":
        assert stats["accepted"] == stats["drafted"] and stats["steps"] < len(prompt) + len(want)
    if drafter == "wrong":
        assert stats["accepted"] == 0


def test_lookahead_refuses_the_qwen_loop(pkg):
    for t in ("QWEN_3", "QWEN_2", "QWEN_2_MOE", "DEEPSEEK_R1_DISTILL_QWEN"):
        with pytest.raises(ValueError, match="generate_tokens_qwen3"):
            pkg.engine.generate_tokens_lookahead(_ToyPlan(), t, 1, 0, [2, 3], [], 10, 16)
    with pytest.raises(ValueError, match="decode_multi_rows"):
        pkg.engine.generate_tokens_lookahead(_ToyPlan(0), "LLAMA_3", 1, 0, [2, 3], [], 10, 16)


def test_prompt_lookup(pkg):
    P = pkg.engine.prompt_lookup
    assert P([1, 2, 3, 9, 1, 2, 3]) == [9, 1, 2, 3]
    assert P([5, 1, 2, 7, 1, 2, 8, 2]) == [8, 2]  # "2" recurs most recently at index 5
    assert P([4, 1, 2, 5, 6, 1, 2], max_tokens=2) == [5, 6]
    assert P([1, 2, 3]) == []
    assert P([]) == []
