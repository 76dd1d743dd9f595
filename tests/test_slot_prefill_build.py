"""CPU checks of the multi-slot prefill (b200_prefill_slots): its kernels compile for sm_90a without spills (the ptxas report build()
writes), and engine.generate_tokens_batch_prefill packs prompts into calls of at most batch_size tokens and decodes in lockstep,
checked on a stand-in plan that records its calls."""
import pytest

from test_batch_decode_build import _entries


def test_slot_prefill_kernels_do_not_spill():
    e = _entries(r"k_pf_rope_kv_packed|k_pf_attention_mma_packed|k_pf_kv_to_f16_packed|k_batch_rows_next")
    assert len([n for n in e if "k_pf_rope_kv_packed" in n]) == 2, sorted(e)
    assert len([n for n in e if "k_pf_attention_mma_packed" in n]) == 2, sorted(e)
    assert len([n for n in e if "k_pf_kv_to_f16_packed" in n]) == 1, sorted(e)
    assert len([n for n in e if "k_batch_rows_next" in n]) == 1, sorted(e)
    for name, (stack, st, ld) in e.items():
        assert (stack, st, ld) == (0, 0, 0), f"{name}: stack / spill stores / loads = {stack} / {st} / {ld}"


class _FakePlan:
    """Decodes every row to (token + 1) % 50 and records the prefill calls."""

    def __init__(self, n_slots):
        self.n_slots, self.calls, self.steps = n_slots, [], []

    def batch_info(self):
        return self.n_slots, 0, 0.0

    def prefill_slots(self, slots, starts, pieces):
        self.calls.append((list(slots), list(starts), [list(p) for p in pieces]))

    def forward_decode_batch(self, slots, tokens, positions):
        self.steps.append((list(slots), list(tokens), list(positions)))
        return [(t + 1) % 50 for t in tokens], None


def test_generate_tokens_batch_prefill_packs_and_decodes(pkg):
    E = pkg.engine
    plan = _FakePlan(4)
    reqs = [(7, 0, [7, 11, 12]), (3, 0, list(range(20, 40))), (5, 4, [5, 9]), (8, 0, [8, 2, 2, 2, 2])]
    got = E.generate_tokens_batch_prefill(plan, "LLAMA_3", reqs, [25], 30, 64, 16)
    for slots, starts, pieces in plan.calls:
        assert sum(len(p) for p in pieces) <= 16 and len(set(slots)) == len(slots)
    # each request's prefilled tokens, in order and at consecutive positions, are [latest] + prompt[:-1]
    for i, (latest, start, prompt) in enumerate(reqs):
        seq, pos = [], start
        for slots, starts, pieces in plan.calls:
            if i in slots:
                k = slots.index(i)
                assert starts[k] == pos
                seq += pieces[k]
                pos += len(pieces[k])
        assert seq == [latest] + prompt[:-1], i
    assert len(plan.calls) == 2  # 3 + 20 + 2 + 5 = 30 tokens: the 20-token prompt spans both calls
    # the single-sequence loop on the same stand-in decode
    for i, (latest, start, prompt) in enumerate(reqs):
        want, cur, pos = [], prompt[-1], start + len(prompt)
        while pos < 30:
            cur = (cur + 1) % 50
            want.append(cur)
            if cur == 25:
                break
            pos += 1
        assert got[i] == want, i
    with pytest.raises(ValueError, match="generate_tokens_batch"):
        E.generate_tokens_batch_prefill(plan, "QWEN_3", reqs, [], 30, 64, 16)
    with pytest.raises(ValueError, match="decode slots"):
        E.generate_tokens_batch_prefill(_FakePlan(2), "LLAMA_3", reqs, [], 30, 64, 16)


def test_generate_tokens_batch_prefill_clamps_to_the_budget(pkg):
    plan = _FakePlan(2)
    got = pkg.engine.generate_tokens_batch_prefill(plan, "LLAMA_3", [(1, 0, list(range(10))), (2, 3, [4, 5])], [], 6, 64, 4)
    assert sum(len(p) for _, _, ps in plan.calls for p in ps) == 6 + 2  # request 0 clamped to positions 0..5, request 1 to 3..4
    assert got == [[], [6]]  # request 1 decodes from position 5 only; request 0's prompt reaches the budget
