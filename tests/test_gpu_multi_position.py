"""GPU tests of the multi-position step: several consecutive positions of ONE sequence per weight stream.

The exact prefill (forward_batch_prefill, prefill_slots) and forward_decode_multi run rows that share a sequence through
k_rope_kv_batch + k_attention_cached_rows, so every row's K/V is written before any row attends.  Every K/V byte, logit and id is
held bit-equal (uint32) to the token-by-token path and to the CPU restatement."""
import os

import numpy as np
import pytest

from test_gpu_batch_decode import _model
from test_gpu_parity import assert_bit_equal
from test_gpu_slot_prefill import _exact_run, _oracle, _own_kv, _same_bytes

pytestmark = pytest.mark.gpu

SHAPES = ["tiny-llama", "tiny-qwen3", "tiny-phi3", "tiny-phi3-gqa", "tiny-qwen2", "tiny-granite", "tiny-llama-q4_k_m"]
CHUNKS = [2, 7, 8, 9, 17, 64]


def _plan(pkg, m, mode="graph"):
    plan = pkg.B200MasterPlan.initialize_plan(m)
    if mode == "persistent":
        try:
            plan.set_decode_mode("persistent")
        except pkg.native.UnsupportedOperation as e:
            plan.free()
            pytest.skip(str(e))
    return plan


def _buffers(plan, c):
    return [plan.read_buffer("x", c.dim), plan.read_buffer("qkv", c.dim), plan.read_buffer("xq", c.dim, np.int8).view(np.uint8).astype(np.uint32),
            plan.read_buffer("xs", c.dim // 32)]


def _prefill_vs_token_by_token(pkg, orc, m, starts, chunks, mode="graph", oracle=True):
    """Chunks through forward_batch_prefill on one plan, the same tokens one per call on another; K/V, the single-token buffers and
    the decode that follows compared between them after every chunk, and K/V against the oracle at the end."""
    c = m.configuration
    stream = orc.bench_tokens(c.vocab_size, c.context_length, seed=31)
    new, old = _plan(pkg, m, mode), _plan(pkg, m, mode)
    assert new.decode_multi_rows() > 0
    try:
        for start in starts:
            if start:  # the positions before start, as one chunk
                new.forward_batch_prefill(stream[:start], 0)
                for p in range(start):
                    old.forward_batch_prefill(stream[p:p + 1], p)
            pos = start
            for n in chunks:
                new.forward_batch_prefill(stream[pos:pos + n], pos)
                for p in range(pos, pos + n):
                    old.forward_batch_prefill(stream[p:p + 1], p)
                pos += n
                assert new.prefill_info()[0] == 0
                _same_bytes(_own_kv(new, c), _own_kv(old, c), f"K/V after the chunk of {n} at {pos - n}")
                _same_bytes(_buffers(new, c), _buffers(old, c), f"single-token buffers after the chunk of {n} at {pos - n}")
            lg_new, id_new = new.forward_decode(int(stream[pos]), pos)
            lg_old, id_old = old.forward_decode(int(stream[pos]), pos)
            assert_bit_equal(lg_new, lg_old, "decode after the prefill")
            assert id_new == id_old
        if oracle:
            om = _oracle(pkg, orc, m)
            try:
                for p in range(pos + 1):
                    ref = om.forward(int(stream[p]), p, want_logits=p == pos)
                assert_bit_equal(lg_new, ref, "decode after the prefill vs the oracle")
                nkv = c.context_length * c.kv_dim
                for l in range(c.n_layers):
                    assert_bit_equal(new.read_buffer("key_cache", nkv, layer=l), om.key_cache(l), f"key cache layer {l}")
                    assert_bit_equal(new.read_buffer("value_cache", nkv, layer=l), om.value_cache(l), f"value cache layer {l}")
            finally:
                om.close()
    finally:
        new.free()
        old.free()


@pytest.mark.parametrize("mode", ["graph", "persistent"])
@pytest.mark.parametrize("shape", SHAPES)
def test_exact_prefill_plan_cache_from_zero(pkg, orc, make_model, shape, mode):
    _prefill_vs_token_by_token(pkg, orc, _model(pkg, make_model, shape, 128), [0], CHUNKS, mode)


@pytest.mark.parametrize("shape", SHAPES)
def test_exact_prefill_plan_cache_continuing_at_600(pkg, orc, make_model, shape):
    _prefill_vs_token_by_token(pkg, orc, _model(pkg, make_model, shape, 720), [600], CHUNKS, oracle=False)


def test_exact_prefill_long_context_score_rows_in_global_memory(pkg, orc, make_model):
    m = _model(pkg, make_model, "tiny-llama", 4608)
    _prefill_vs_token_by_token(pkg, orc, m, [4500], [9, 64], oracle=False)


@pytest.mark.parametrize("shape", ["mid-llama", "mid-qwen3-4b", "mid-qwen2.5-7b"])
def test_exact_prefill_8_row_chunks_mid_geometries(pkg, orc, make_model, shape):
    m = _model(pkg, make_model, shape, 24)
    _prefill_vs_token_by_token(pkg, orc, m, [0], [8, 9], oracle=shape != "mid-qwen2.5-7b")


@pytest.mark.parametrize("shape", ["tiny-llama", "tiny-qwen3", "tiny-qwen2", "tiny-granite"])
def test_exact_prefill_slots_packs_rows(pkg, orc, make_model, shape):
    m = _model(pkg, make_model, shape, 192)
    L = m.configuration.n_layers
    # 1, 2 and 3 prompts of unequal length on 8 slots; the third call continues slots 2 and 5
    for slots, starts, lens in [([3], [0], [13]), ([2, 5], [0, 0], [9, 30]), ([2, 5, 0], [9, 30, 0], [4, 17, 1])]:
        mode, launches, _ = _exact_run(pkg, orc, m, 8, [(slots, starts, lens)] if starts[0] == 0 else
                                       [([2, 5], [0, 0], [9, 30]), (slots, starts, lens)], decode=True)
        T, R = sum(lens), 8
        steps = -(-T // R)
        assert steps * (1 + 7 * L) <= launches <= steps * (1 + 8 * L), (T, launches)


def _decode_ref(pkg, orc, m, stream, upto):
    om = _oracle(pkg, orc, m)
    out = [om.forward(int(stream[p]), p) for p in range(upto)]
    om.close()
    return out


@pytest.mark.parametrize("shape", ["tiny-llama", "tiny-qwen3", "tiny-phi3", "tiny-qwen2", "tiny-granite"])
def test_forward_decode_multi_bit_exact(pkg, orc, make_model, shape):
    m = _model(pkg, make_model, shape, 128)
    c = m.configuration
    stream = orc.bench_tokens(c.vocab_size, c.context_length, seed=5)
    plan = _plan(pkg, m)
    R = plan.decode_multi_rows()
    assert R == 8
    ref = _decode_ref(pkg, orc, m, stream, 1 + sum(range(1, R + 1)) + 1)
    try:
        plan.set_decode_slots(3)
        for slot in (-1, 1):
            pos = 0
            for n in range(1, R + 1):
                ids, lg = plan.forward_decode_multi(slot, stream[pos:pos + n], pos, logits=True)
                for i in range(n):
                    assert_bit_equal(lg[i], ref[pos + i], f"slot {slot}, n {n}, row {i}")
                    assert ids[i] == orc.argmax(ref[pos + i])
                pos += n
        # wrong drafts at pos..pos+5, then a re-verify from the first rejected position is still exact
        wrong = [(int(t) + 1) % c.vocab_size for t in stream[pos + 1:pos + 7]]
        plan.forward_decode_multi(-1, [int(stream[pos])] + wrong, pos)
        ids, lg = plan.forward_decode_multi(-1, stream[pos + 1:pos + 2], pos + 1, logits=True)
        assert_bit_equal(lg[0], ref[pos + 1], "re-verify after rejected drafts")
    finally:
        plan.free()


def test_forward_decode_multi_interleaves(pkg, orc, make_model):
    m = _model(pkg, make_model, "tiny-llama", 128)
    c = m.configuration
    streams = [orc.bench_tokens(c.vocab_size, c.context_length, seed=60 + s) for s in range(3)]
    refs = [_decode_ref(pkg, orc, m, s, 40) for s in streams]
    plan = _plan(pkg, m)
    try:
        plan.set_decode_slots(2)
        plan.prefill_slots([0], [0], [streams[0][:10]])
        for p in range(6):  # the plan's own sequence through forward_decode
            plan.forward_decode(int(streams[2][p]), p)
        pos = 6
        ids, lg = plan.forward_decode_multi(-1, streams[2][pos:pos + 5], pos, logits=True)
        for i in range(5):
            assert_bit_equal(lg[i], refs[2][pos + i], f"own row {i}")
        ids, lg = plan.forward_decode_batch([0, 1], [int(streams[0][10]), int(streams[1][0])], [10, 0], logits=True)
        assert_bit_equal(lg[0], refs[0][10], "batched slot 0")
        assert_bit_equal(lg[1], refs[1][0], "batched slot 1")
        ids, lg = plan.forward_decode_multi(1, streams[1][1:9], 1, logits=True)
        for i in range(8):
            assert_bit_equal(lg[i], refs[1][1 + i], f"slot 1 row {i}")
        lg, _ = plan.forward_decode(int(streams[2][11]), 11)
        assert_bit_equal(lg, refs[2][11], "forward_decode after multi steps")
        plan.set_decode_slots(0)  # the per-row buffers come back on first use
        ids, lg = plan.forward_decode_multi(-1, streams[2][12:14], 12, logits=True)
        assert_bit_equal(lg[1], refs[2][13], "after set_decode_slots(0)")
    finally:
        plan.free()


def _expect(pkg, fn, code, text):
    with pytest.raises(pkg.native.B200Error) as e:
        fn()
    assert e.value.code == code and text in str(e.value), str(e.value)


def test_forward_decode_multi_refusals(pkg, orc, make_model):
    m = _model(pkg, make_model, "tiny-llama", 64)
    plan = _plan(pkg, m)
    V = m.configuration.vocab_size
    try:
        _expect(pkg, lambda: plan.forward_decode_multi(-1, list(range(9)), 0), -1, "n = 9 rows")
        _expect(pkg, lambda: plan.forward_decode_multi(0, [1], 0), -1, "slot 0 out of range")
        _expect(pkg, lambda: plan.forward_decode_multi(-1, [1, 2, 3], 62), -1, "row 2: position 64")
        _expect(pkg, lambda: plan.forward_decode_multi(-1, [1, V], 0), -1, f"row 1: token {V}")
        lg, _ = plan.forward_decode(1, 0)
        assert np.isfinite(lg).all()
    finally:
        plan.free()
    fp16 = pkg.B200MasterPlan.initialize_plan(make_model("tiny-llama", pkg.gguf.GGMLType.F16, 64))
    try:
        assert fp16.decode_multi_rows() == 0
        _expect(pkg, lambda: fp16.forward_decode_multi(-1, [1, 2], 0), -2, "Q8_0 weights")
        assert np.isfinite(fp16.forward_decode(1, 0)[0]).all()
    finally:
        fp16.free()
    os.environ["B200_STREAM"] = "0"
    try:
        ns = pkg.B200MasterPlan.initialize_plan(m)
    finally:
        del os.environ["B200_STREAM"]
    try:
        _expect(pkg, lambda: ns.forward_decode_multi(-1, [1, 2], 0), -2, "streaming layout")
        assert np.isfinite(ns.forward_decode(1, 0)[0]).all()
    finally:
        ns.free()


def test_forward_decode_multi_refuses_moe(pkg, make_model):
    m = make_model("tiny-qwen2moe", pkg.gguf.GGMLType.Q8_0, 64)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    try:
        assert plan.decode_multi_rows() == 0
        _expect(pkg, lambda: plan.forward_decode_multi(-1, [1, 2], 0), -2, "Qwen2-MoE")
        assert np.isfinite(plan.forward_decode(1, 0)[0]).all()
    finally:
        plan.free()


@pytest.mark.parametrize("drafter", ["prompt_lookup", "right", "wrong"])
def test_generate_tokens_lookahead_equals_llama_loop(pkg, orc, make_model, drafter):
    E = pkg.engine
    m = _model(pkg, make_model, "tiny-llama", 96)
    c = m.configuration
    om = _oracle(pkg, orc, m)
    prompt = [5, 9, 5, 9, 7, 5, 9, 7, 3, 5, 9]
    try:
        want = E.generate_tokens_llama(lambda t, p: orc.argmax(om.forward(t, p)), 1, 0, prompt, [], 60, c.context_length)
        for stop, budget in [([], 60), ([want[len(want) // 2]], 60), ([], 40)]:
            om.reset()
            ref = E.generate_tokens_llama(lambda t, p: orc.argmax(om.forward(t, p)), 1, 0, prompt, stop, budget, c.context_length)
            full = [1] + prompt + want
            draft = {"prompt_lookup": E.prompt_lookup,
                     "right": lambda h: full[len(h):len(h) + 8],
                     "wrong": lambda h: [(full[len(h) + i] + 1) % c.vocab_size for i in range(min(8, len(full) - len(h)))]}[drafter]
            plan = _plan(pkg, m)
            try:
                stats = {}
                got = E.generate_tokens_lookahead(plan, "LLAMA_3", 1, 0, prompt, stop, budget, c.context_length, draft=draft, stats=stats)
            finally:
                plan.free()
            assert got == ref, (drafter, stop, budget)
            if drafter == "right":
                assert stats["accepted"] == stats["drafted"]
            if drafter == "wrong":
                assert stats["accepted"] == 0
    finally:
        om.close()
