"""Host side of the tensor-core chunk step (b200_forward_chunk), without a GPU: the entry points at every layer, the kernels the call
launches in the ptxas report, and ContinuousBatcher's chunked admission on a stand-in plan against the single-request loops."""
import ctypes
import inspect
import os
import random

import pytest

from test_batch_decode_build import _entries
from test_continuous_host import V, FakeSampler, FakeStepPlan, _single

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- build and wrappers ------------------------------------------------------------------------------------------------------

def test_chunk_entry_points_are_exported_and_wrapped(pkg):
    n = pkg.native
    lib = ctypes.CDLL(n.LIB_PATH)
    for name in ("b200_forward_chunk", "b200_chunk_rows"):
        assert hasattr(lib, name) and name in n.EXPORTS, name
    assert list(inspect.signature(n.NativePlan.forward_chunk).parameters) == ["self", "rows", "logits"]
    assert list(inspect.signature(n.NativePlan.chunk_rows).parameters) == ["self"]
    assert list(inspect.signature(pkg.B200MasterPlan.forward_chunk).parameters) == ["self", "rows", "logits"]
    assert list(inspect.signature(pkg.B200MasterPlan.chunk_rows).parameters) == ["self"]
    sig = inspect.signature(pkg.engine.ContinuousBatcher)
    assert sig.parameters["chunk_rows"].default == 0 and sig.parameters["min_chunk_rows"].default == 32
    sig = inspect.signature(pkg.engine.generate_tokens_continuous)
    assert sig.parameters["chunk_rows"].default == 0 and sig.parameters["min_chunk_rows"].default == 32
    hdr = open(os.path.join(ROOT, "include", "b200llama.h")).read()
    assert "int b200_forward_chunk(b200_plan *plan, int32_t n, const b200_step_row *rows, int32_t *ids_out" in hdr
    assert "int b200_chunk_rows(b200_plan *plan, int32_t *max_rows);" in hdr
    java = open(os.path.join(ROOT, "gpullama3.java_b200", "java", "B200MasterPlan.java")).read()
    assert 'fn("b200_forward_chunk"' in java and "public int[] forwardChunk(" in java
    assert 'fn("b200_chunk_rows"' in java and "public int chunkRows()" in java


def test_chunk_kernels_do_not_spill():
    """The kernels a chunk step launches: the int8 prefill's norm, RoPE / KV, attention and GEMMs, then the batched classifier."""
    e = _entries(r"k_i8_norm|k_i8_rope_kv|k_i8_attention|k_gemm_i8|k_rmsnorm_quant_batchILb0E|k_stream_matvec_q8_batch|k_argmax_batch")
    assert any("k_gemm_i8" in n for n in e) and any("k_i8_attention" in n for n in e) and any("k_argmax_batch" in n for n in e)
    for name, (stack, st, ld) in e.items():
        if "ILi32E" in name:  # head size 32 runs neither path's attention
            continue
        assert (st, ld) == (0, 0), f"{name}: spill stores / loads = {st} / {ld}"


# ---- the scheduler on a stand-in plan -----------------------------------------------------------------------------------------

class FakeChunkPlan(FakeStepPlan):
    """FakeStepPlan plus forward_chunk, which computes what forward_step computes on the same rows.  Asserts b200_forward_chunk's input
    contract: 1..chunk_rows() rows, at most 8 emitting, no (slot, position) twice, and the decode rows of generating slots first."""

    def __init__(self, n_slots, rows=8, chunk=0):
        super().__init__(n_slots, rows)
        self.chunk, self.kinds = chunk, []
        self.generating = set()  # slots whose request has emitted since their last reset

    def chunk_rows(self):
        return self.chunk

    def slot_reset(self, slot):
        super().slot_reset(slot)
        self.generating.discard(slot)

    def _note(self, rows, kind):
        self.kinds.append(kind)
        decode = [r[0] in self.generating for r in rows]
        assert decode == sorted(decode, reverse=True), "a decode row follows a prompt row"
        assert all(r[3] for r, d in zip(rows, decode) if d)
        self.generating |= {r[0] for r in rows if r[3]}

    def forward_step(self, rows, logits=False):
        self._note(rows, "step")
        return super().forward_step(rows, logits)

    def forward_chunk(self, rows, logits=False):
        assert 1 <= len(rows) <= self.chunk
        assert sum(r[3] for r in rows) <= 8
        self._note(rows, "chunk")
        saved, self.rows = self.rows, self.chunk
        try:
            return super().forward_step(rows, logits)
        finally:
            self.rows = saved


def _trace(rng, llama, ctx):
    n_req = rng.randrange(1, 14)
    reqs = []
    for _ in range(n_req):
        n_prompt = rng.randrange(0 if llama else 1, 60)
        reqs.append((rng.randrange(V), rng.randrange(0, 40), [rng.randrange(V) for _ in range(n_prompt)]))
    arrivals = [rng.randrange(0, 30) for _ in reqs]
    stop = [rng.randrange(V) for _ in range(rng.randrange(3))]
    budget = rng.choice([-1, ctx + 50, rng.randrange(0, 80)])
    return reqs, arrivals, stop, budget


LOOPS = [("LLAMA_3", True), ("QWEN_3", False)]


@pytest.mark.parametrize("model_type,llama", LOOPS)
def test_chunked_admission_equals_each_request_alone(pkg, model_type, llama):
    """Random traces, greedy and sampled: every request's ids are its loop's alone; chunks stay within chunk_rows (capped by the
    plan's chunk_rows()) and run only from min_chunk_rows rows; steps stay within decode_multi_rows()."""
    rng = random.Random(31 if llama else 37)
    ctx = 128
    total, chunks, steps = 0, 0, 0
    for trial in range(40):
        reqs, arrivals, stop, budget = _trace(rng, llama, ctx)
        rows = rng.randrange(4, 9)
        n_slots = rng.randrange(1, rows + 1)  # a plan holds at most decode_multi_rows() slots
        cap = rng.choice([16, 48, 512])
        chunk_rows, min_rows = rng.choice([8, 24, 64, 256]), rng.choice([1, 4, 12, 32])
        sampled = trial % 2 == 1
        samplers = [FakeSampler(rng.choice([0.0, 0.8]), 1000 + i) for i in range(len(reqs))] if sampled else None
        plan = FakeChunkPlan(n_slots, rows, cap)
        stats = {}
        got = pkg.engine.generate_tokens_continuous(plan, model_type, reqs, arrivals, stop, budget, ctx, samplers=samplers, stats=stats,
                                                    chunk_rows=chunk_rows, min_chunk_rows=min_rows)
        for i, req in enumerate(reqs):
            ref_sampler = FakeSampler(samplers[i].temperature, 1000 + i) if sampled else None
            want = _single(pkg, model_type, req, stop, budget, ctx, ref_sampler)
            assert got[i] == want, (trial, i, req)
            total += len(want)
            if sampled:
                assert samplers[i].rng.draws == (len(want) if samplers[i].temperature else 0), (trial, i)
        assert stats["kinds"] == plan.kinds and stats["rows"] == [len(s) for s in plan.steps]
        for kind, n in zip(stats["kinds"], stats["rows"]):
            if kind == "chunk":
                assert min_rows <= n <= min(chunk_rows, cap), (trial, n)
                chunks += 1
            else:
                assert n <= rows, (trial, n)
                steps += 1
    assert total > 500 and chunks > 50 and steps > 50


def test_chunk_rows_zero_is_todays_scheduler(pkg):
    """chunk_rows = 0: forward_chunk is never called and the forward_step calls are those of a plan without it, row for row."""
    rng = random.Random(5)
    for trial in range(20):
        llama = trial % 2 == 0
        model_type = "LLAMA_3" if llama else "QWEN_3"
        reqs, arrivals, stop, budget = _trace(rng, llama, 96)
        n_slots, rows = rng.randrange(1, 5), rng.randrange(4, 9)
        old, new = FakeStepPlan(n_slots, rows), FakeChunkPlan(n_slots, rows, 256)
        a = pkg.engine.generate_tokens_continuous(old, model_type, reqs, arrivals, stop, budget, 96)
        stats = {}
        b = pkg.engine.generate_tokens_continuous(new, model_type, reqs, arrivals, stop, budget, 96, stats=stats)
        assert a == b and old.steps == new.steps, trial
        assert set(new.kinds) <= {"step"} and set(stats["kinds"]) <= {"step"}


def test_chunk_layout_decode_rows_first(pkg):
    """Two generating requests and a long prompt admitted behind them: one chunk holds both decode rows, then the prompt in position
    order, its last row emitting."""
    plan = FakeChunkPlan(3, rows=4, chunk=64)
    cb = pkg.engine.ContinuousBatcher(plan, "LLAMA_3", [], 200, 200, chunk_rows=40, min_chunk_rows=8)
    cb.submit(10, 0, [11])
    cb.submit(20, 0, [21])
    cb.step()  # 4 rows: a step, not a chunk
    assert plan.kinds == ["step"] and cb.last_kind == "step"
    c = cb.submit(30, 0, list(range(40, 90)))
    cb.step()
    assert plan.kinds == ["step", "chunk"] and cb.last_kind == "chunk"
    got = [r[:4] for r in plan.steps[-1]]
    assert len(got) == 40 and [r[0] for r in got[:2]] == [0, 1] and all(r[3] for r in got[:2])
    assert got[2:] == [(2, 30, 0, 0)] + [(2, 40 + k, k + 1, 0) for k in range(37)]
    cb.step()  # 2 decode rows + the 13 rows left of the prompt (the last one emits): a chunk of 15
    got = [r[:4] for r in plan.steps[-1]]
    assert plan.kinds[-1] == "chunk" and len(got) == 15 and got[-1] == (2, 89, 50, 1)
    while cb.running():
        cb.step()
    assert plan.kinds[-1] == "step"  # three decode rows never reach min_chunk_rows
    assert cb.results[c] == _single(pkg, "LLAMA_3", (30, 0, list(range(40, 90))), [], 200, 200)


def test_chunk_value_errors(pkg):
    E = pkg.engine
    with pytest.raises(ValueError, match="chunk_rows"):
        E.ContinuousBatcher(FakeChunkPlan(2, chunk=0), "LLAMA_3", [], 10, 64, chunk_rows=64)
    with pytest.raises(ValueError, match="chunk_rows"):
        E.ContinuousBatcher(FakeChunkPlan(2, chunk=64), "LLAMA_3", [], 10, 64, chunk_rows=-1)
    with pytest.raises(ValueError, match="min_chunk_rows"):
        E.ContinuousBatcher(FakeChunkPlan(2, chunk=64), "LLAMA_3", [], 10, 64, chunk_rows=64, min_chunk_rows=0)
    cb = E.ContinuousBatcher(FakeChunkPlan(2, chunk=48), "LLAMA_3", [], 10, 64, chunk_rows=256)
    assert cb.chunk_rows == 48  # capped at the plan's chunk_rows()
