"""Host side of the batched decode, without a GPU: engine.generate_tokens_batch against the single-request loops on a deterministic
fake forward, and the new entry points in the built library's symbol table."""
import ctypes
import random

import pytest


def _fake_argmax(token: int, pos: int, seed: int) -> int:
    return (token * 131 + pos * 17 + seed) % 97


class FakeBatchPlan:
    """Per-slot state is the request's seed; the fake forward depends on (seed, token, position) only, like a real sequence."""

    def __init__(self, n_slots, seeds):
        self.n_slots, self.seeds, self.calls = n_slots, seeds, []

    def batch_info(self):
        return self.n_slots, 0, 0.0

    def slot_reset(self, slot):
        assert 0 <= slot < self.n_slots

    def forward_decode_batch(self, slots, tokens, positions, sampling=None, logits=False):
        assert len(set(slots)) == len(slots) and 1 <= len(slots) <= self.n_slots
        self.calls.append(list(slots))
        return [_fake_argmax(t, p, self.seeds[s]) for s, t, p in zip(slots, tokens, positions)], None


REQUESTS = [(7, 0, [7, 11, 12]), (3, 0, [3]), (5, 4, [21, 22, 23, 24, 25, 26]), (9, 600, [1, 2]), (1, 0, [])]


@pytest.mark.parametrize("model_type,loop", [("LLAMA_3", "llama"), ("MISTRAL", "llama"), ("QWEN_3", "qwen3"), ("QWEN_2", "qwen3"),
                                             ("DEEPSEEK_R1_DISTILL_QWEN", "qwen3")])
@pytest.mark.parametrize("stop,max_tokens", [([], 20), ([5, 40], 30), ([], 606), ([0], -1)])
def test_generate_tokens_batch_equals_each_request_alone(pkg, model_type, loop, stop, max_tokens):
    reqs = [r for r in REQUESTS if loop == "llama" or r[2]]  # the Qwen3 loop needs a prompt
    seeds = list(range(len(reqs)))
    plan = FakeBatchPlan(8, seeds)
    got = pkg.engine.generate_tokens_batch(plan, model_type, reqs, stop, max_tokens, 640)
    single = pkg.engine.generate_tokens_llama if loop == "llama" else pkg.engine.generate_tokens_qwen3
    assert pkg.engine.loop_for(model_type) is single
    for i, (latest, start, prompt) in enumerate(reqs):
        ref = single(lambda t, p: _fake_argmax(t, p, seeds[i]), latest, start, prompt, stop, max_tokens, 640)
        assert got[i] == ref, f"request {i}"
    # rows leave as they finish: the batch shrinks, and the slots passed are those of the requests still running
    sizes = [len(c) for c in plan.calls]
    assert sizes == sorted(sizes, reverse=True) and sizes[0] <= len(reqs)


def test_generate_tokens_batch_random_requests(pkg):
    rng = random.Random(5)
    for _ in range(20):
        reqs = [(rng.randrange(97), rng.randrange(50), [rng.randrange(97) for _ in range(rng.randrange(1, 9))]) for _ in range(rng.randrange(1, 9))]
        stop = [rng.randrange(97) for _ in range(rng.randrange(3))]
        budget = rng.randrange(-1, 90)
        for mt, single in (("LLAMA_3", pkg.engine.generate_tokens_llama), ("QWEN_3", pkg.engine.generate_tokens_qwen3)):
            got = pkg.engine.generate_tokens_batch(FakeBatchPlan(8, list(range(len(reqs)))), mt, reqs, stop, budget, 96)
            for i, (latest, start, prompt) in enumerate(reqs):
                assert got[i] == single(lambda t, p: _fake_argmax(t, p, i), latest, start, prompt, stop, budget, 96)


def test_generate_tokens_batch_needs_enough_slots(pkg):
    with pytest.raises(ValueError):
        pkg.engine.generate_tokens_batch(FakeBatchPlan(2, [0, 1, 2]), "LLAMA_3", REQUESTS[:3], [], 10, 64)


def test_batch_entry_points_are_exported(pkg):
    lib = ctypes.CDLL(pkg.native.LIB_PATH)
    for sym in ("b200_set_decode_slots", "b200_forward_decode_batch", "b200_slot_reset", "b200_slot_copy_kv", "b200_batch_info"):
        assert hasattr(lib, sym), sym
        assert sym in pkg.native.EXPORTS
