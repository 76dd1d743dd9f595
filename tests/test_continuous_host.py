"""Host side of continuous batching, without a GPU: engine.ContinuousBatcher / generate_tokens_continuous against the single-request
loops on a stand-in plan, the new entry point in the built library's symbol table, and k_sample_rows in the ptxas report."""
import ctypes
import random

import pytest

from test_batch_decode_build import _entries

V = 97


def _id(history: dict, token: int, pos: int) -> int:
    """A stand-in argmax that depends on the slot's K/V below pos (a dict position -> token), the token and the position."""
    h = 0
    for p in sorted(history):
        if p < pos:
            h = (h * 1000003 + p * 131 + history[p]) % (2 ** 61 - 1)
    return (h + token * 7 + pos) % V


class FakeStepPlan:
    """forward_step as the device runs it: every row writes its K/V (here its token) at (slot, position) before any row's id is
    computed.  A sampled row's id also depends on its uniform number.  Asserts the input contract of b200_forward_step."""

    def __init__(self, n_slots, rows=8):
        self.n_slots, self.rows = n_slots, rows
        self.kv = [dict() for _ in range(n_slots)]
        self.steps, self.resets = [], []

    def decode_multi_rows(self):
        return self.rows

    def batch_info(self):
        return self.n_slots, 7, 0.0

    def slot_reset(self, slot):
        assert 0 <= slot < self.n_slots
        self.kv[slot] = {}
        self.resets.append(slot)

    def forward_step(self, rows, logits=False):
        assert 1 <= len(rows) <= self.rows
        assert len({(r[0], r[2]) for r in rows}) == len(rows), "a (slot, position) repeats"
        for slot, token, pos, emit, t, topp, u in rows:
            assert 0 <= slot < self.n_slots and 0 <= token < V and pos >= 0
            assert emit in (0, 1)
            if emit:
                assert t >= 0.0 and 0.0 <= u < 1.0
            else:
                assert (t, topp, u) == (0.0, 0.0, 0.0)
        self.steps.append([tuple(r) for r in rows])
        for slot, token, pos, *_ in rows:
            self.kv[slot][pos] = token
        ids = []
        for slot, token, pos, emit, t, topp, u in rows:
            ids.append(-1 if not emit else (_id(self.kv[slot], token, pos) + (int(u * 1000) if t else 0)) % V)
        return ids, None


class FakeRng:
    def __init__(self, seed):
        self.r, self.draws = random.Random(seed), 0

    def next_float1(self):
        self.draws += 1
        return self.r.randrange(1 << 24) * 2.0 ** -24


class FakeSampler:
    def __init__(self, temperature, seed):
        self.temperature, self.topp, self.rng = temperature, 0.9, FakeRng(seed)


def _single(pkg, model_type, req, stop, budget, ctx, sampler=None):
    """The request's loop alone on one slot: prompt rows run without sampling, each generated token draws one uniform."""
    latest, start, prompt = req
    loop = pkg.engine.loop_for(model_type)
    kv_rows = len(prompt) if loop is pkg.engine.generate_tokens_llama else max(len(prompt) - 1, 0)
    history, seen = {}, [0]

    def forward(token, pos):
        history[pos] = token
        seen[0] += 1
        am = _id(history, token, pos)
        if seen[0] > kv_rows and sampler is not None and sampler.temperature:
            am = (am + int(sampler.rng.next_float1() * 1000)) % V
        return am

    return loop(forward, latest, start, prompt, stop, budget, ctx)


LOOPS = [("LLAMA_3", True), ("QWEN_3", False), ("MISTRAL", True), ("QWEN_2", False)]


@pytest.mark.parametrize("model_type,llama", LOOPS)
def test_random_traces_equal_each_request_alone(pkg, model_type, llama):
    rng = random.Random(17 if llama else 23)
    ctx = 96
    total = 0
    for trial in range(40):
        n_req = rng.randrange(1, 14)
        reqs = []
        for _ in range(n_req):
            n_prompt = rng.randrange(0 if llama else 1, 20)
            reqs.append((rng.randrange(V), rng.randrange(0, 40), [rng.randrange(V) for _ in range(n_prompt)]))
        arrivals = [rng.randrange(0, 30) for _ in reqs]
        stop = [rng.randrange(V) for _ in range(rng.randrange(3))]
        budget = rng.choice([-1, ctx + 50, rng.randrange(0, 80)])
        n_slots, rows = rng.randrange(1, 5), rng.randrange(4, 9)
        sampled = trial % 2 == 1
        samplers = [FakeSampler(rng.choice([0.0, 0.8]), 1000 + i) for i in range(n_req)] if sampled else None
        plan = FakeStepPlan(n_slots, rows)
        stats = {}
        got = pkg.engine.generate_tokens_continuous(plan, model_type, reqs, arrivals, stop, budget, ctx, samplers=samplers, stats=stats)
        for i, req in enumerate(reqs):
            ref_sampler = FakeSampler(samplers[i].temperature, 1000 + i) if sampled else None
            want = _single(pkg, model_type, req, stop, budget, ctx, ref_sampler)
            assert got[i] == want, (trial, i, req)
            total += len(want)
            if sampled:  # exactly one uniform per generated token (none for a greedy sampler)
                assert samplers[i].rng.draws == (len(want) if samplers[i].temperature else 0), (trial, i)
        assert stats["steps"] == len(plan.steps) and stats["rows"] == [len(s) for s in plan.steps]
        assert all(r <= rows for r in stats["rows"])
        for i in range(n_req):
            if got[i]:
                assert stats["submitted"][i] <= stats["first_token"][i] <= stats["done"][i]
    assert total > 500


def test_step_rows_decode_first_then_prompts_in_admission_order(pkg):
    plan = FakeStepPlan(3, rows=4)
    cb = pkg.engine.ContinuousBatcher(plan, "LLAMA_3", [], 64, 64)
    a = cb.submit(10, 0, [11, 12, 13, 14, 15])
    b = cb.submit(20, 0, [21])
    assert cb.pending() == 2 and cb.running() == 0
    assert cb.step() == []  # request a's prompt fills the step; b is admitted but gets no row yet
    assert plan.steps[-1] == [(0, 10, 0, 0, 0.0, 0.0, 0.0), (0, 11, 1, 0, 0.0, 0.0, 0.0), (0, 12, 2, 0, 0.0, 0.0, 0.0),
                              (0, 13, 3, 0, 0.0, 0.0, 0.0)]
    assert cb.running() == 2 and cb.pending() == 0
    ev = cb.step()  # a's last K/V row and its emitting row, then b's
    assert [r[:4] for r in plan.steps[-1]] == [(0, 14, 4, 0), (0, 15, 5, 1), (1, 20, 0, 0), (1, 21, 1, 1)]
    assert [(rid, fin) for rid, _, fin in ev] == [(a, False), (b, False)]
    ta, tb = ev[0][1], ev[1][1]
    c = cb.submit(30, 0, [31, 32, 33])
    ev = cb.step()  # the two decode rows first, then c's prompt in the rows left
    assert [r[:4] for r in plan.steps[-1]] == [(0, ta, 6, 1), (1, tb, 2, 1), (2, 30, 0, 0), (2, 31, 1, 0)]
    ta, tb = ev[0][1], ev[1][1]
    cb.step()
    assert [r[:4] for r in plan.steps[-1]] == [(0, ta, 7, 1), (1, tb, 3, 1), (2, 32, 2, 0), (2, 33, 3, 1)]
    assert plan.resets == [0, 1, 2]


def test_freed_slot_is_reused_in_the_same_step(pkg):
    plan = FakeStepPlan(1, rows=8)
    cb = pkg.engine.ContinuousBatcher(plan, "QWEN_3", [], 6, 64)
    reqs = [(1, 0, [2, 3]), (4, 0, [5, 6, 7]), (8, 3, [9])]
    rids = [cb.submit(*r) for r in reqs]
    assert cb.pending() == 3 and cb.running() == 0  # admission happens in step()
    finished = []
    while cb.pending() or cb.running():
        ev = cb.step()
        finished += [rid for rid, _, fin in ev if fin]
        if finished and cb.pending() + cb.running():
            assert cb.running() == 1  # the next request took the slot before step() returned
    assert finished == rids
    assert plan.resets == [0, 0, 0]
    for rid, req in zip(rids, reqs):
        assert cb.results[rid] == _single(pkg, "QWEN_3", req, [], 6, 64)


def test_budget_before_the_first_row(pkg):
    plan = FakeStepPlan(2, rows=8)
    got = pkg.engine.generate_tokens_continuous(plan, "LLAMA_3", [(1, 10, [2]), (3, 0, [4])], [0, 0], [], 10, 64)
    assert got[0] == [] and got[1] == _single(pkg, "LLAMA_3", (3, 0, [4]), [], 10, 64)
    assert plan.resets == [0]  # the request that cannot run is never admitted


def test_value_errors(pkg):
    E = pkg.engine
    with pytest.raises(ValueError, match="decode_multi_rows"):
        E.ContinuousBatcher(FakeStepPlan(2, rows=0), "LLAMA_3", [], 10, 64)
    with pytest.raises(ValueError, match="decode slots"):
        E.ContinuousBatcher(FakeStepPlan(0), "LLAMA_3", [], 10, 64)
    with pytest.raises(ValueError, match="start_position"):
        E.ContinuousBatcher(FakeStepPlan(2), "LLAMA_3", [], 10, 64).submit(1, -1, [2])
    reqs = [(1, 0, [2]), (3, 0, [4])]
    with pytest.raises(ValueError, match="arrival"):
        E.generate_tokens_continuous(FakeStepPlan(2), "LLAMA_3", reqs, [0], [], 10, 64)
    with pytest.raises(ValueError, match="samplers"):
        E.generate_tokens_continuous(FakeStepPlan(2), "LLAMA_3", reqs, [0, 0], [], 10, 64, samplers=[None])
    with pytest.raises(ValueError, match=">= 0"):
        E.generate_tokens_continuous(FakeStepPlan(2), "LLAMA_3", reqs, [0, -1], [], 10, 64)


def test_forward_step_is_exported(pkg):
    lib = ctypes.CDLL(pkg.native.LIB_PATH)
    assert hasattr(lib, "b200_forward_step")
    assert "b200_forward_step" in pkg.native.EXPORTS
    assert ctypes.sizeof(pkg.native.StepRow) == 28


def test_sample_rows_does_not_spill():
    e = _entries(r"k_sample")
    rows = [n for n in e if "k_sample_rows" in n]
    assert len(rows) == 1
    for name in e:
        assert e[name][1:] == (0, 0), f"{name}: spill stores / loads = {e[name][1:]}"
