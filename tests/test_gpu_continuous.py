"""GPU tests of the mixed step (b200_forward_step) and the continuous-batching scheduler on top of it.

Decode rows and K/V-only prompt rows of several slots share one step; a slot may take several rows.  Every emitting row's logits
are held bit-equal (uint32) to the CPU restatement of that slot's sequence, with the same id; every slot's K/V after the steps too,
and the plan's own cache must not change.  generate_tokens_continuous must give each request the ids of its loop run alone."""
import numpy as np
import pytest

from devstral_oracle import DevstralOracle
from test_gpu_batch_decode import _model
from test_gpu_parity import assert_bit_equal
from test_gpu_slot_prefill import _kv, _oracle as _slot_oracle, _own_kv, _same_bytes

pytestmark = pytest.mark.gpu


def _oracle(pkg, orc, m):
    return DevstralOracle(orc, m) if m.configuration.arch == 6 else _slot_oracle(pkg, orc, m)


# Steps of (slot, rows, emit): rows consecutive positions of the slot, emit "none", "last" or "all" of them.  Covered: a prompt
# chunk whose last row emits, prompt chunks of one slot spanning steps, steps with no emitting row (split and not), emitting rows
# after K/V-only rows in call order, two emitting rows of one slot, and a full 8-row step.
SCHEDULE = [
    [(0, 5, "last")],
    [(0, 1, "all"), (1, 7, "none")],
    [(1, 3, "none")],
    [(1, 2, "last"), (0, 1, "all"), (2, 1, "all")],
    [(2, 1, "none"), (0, 1, "all"), (1, 1, "all")],
    [(0, 1, "all"), (1, 1, "all"), (2, 6, "last")],
    [(2, 1, "none")],
    [(0, 1, "all"), (2, 2, "all")],
]


def _run_mixed(pkg, orc, m, schedule, n_slots=3):
    c = m.configuration
    plan = pkg.B200MasterPlan.initialize_plan(m)
    streams = [orc.bench_tokens(c.vocab_size, c.context_length, seed=500 + s) for s in range(n_slots)]
    hist = [[] for _ in range(n_slots)]  # (token, position, logits or None, id) per slot
    nxt = [0] * n_slots
    om = _oracle(pkg, orc, m)
    try:
        plan.set_decode_slots(n_slots)
        own = _own_kv(plan, c)
        for step in schedule:
            rows = []
            for s, n, emit in step:
                for j in range(n):
                    e = emit == "all" or (emit == "last" and j == n - 1)
                    rows.append((s, int(streams[s][nxt[s] + j]), nxt[s] + j, int(e)))
                nxt[s] += n
            ids, lg = plan.forward_step(rows, logits=True)
            for i, (s, tok, pos, e) in enumerate(rows):
                if e:
                    hist[s].append((tok, pos, lg[i], int(ids[i])))
                else:
                    assert ids[i] == -1 and not lg[i].any(), f"K/V-only row {i} returned output"
                    hist[s].append((tok, pos, None, -1))
            split = any(len([r for r in rows if r[0] == s]) > 1 for s in range(n_slots))
            n_emit = sum(r[3] for r in rows)
            want = c.n_layers * (7 + split) + (3 if n_emit else 0)
            assert plan.batch_info()[1] == want, (step, plan.batch_info()[1], want)
        _same_bytes(_own_kv(plan, c), own, "the plan's own cache changed")
        for s in range(n_slots):
            om.reset()
            for tok, pos, lg, am in sorted(hist[s], key=lambda h: h[1]):
                if lg is None:
                    om.forward(tok, pos, want_logits=False)
                    continue
                ref = om.forward(tok, pos)
                assert_bit_equal(lg, ref, f"slot {s} logits pos {pos}")
                assert am == orc.argmax(ref), f"slot {s} id pos {pos}"
            nkv = c.context_length * c.kv_dim
            got = _kv(plan, c, s)
            for l in range(c.n_layers):
                assert_bit_equal(got[l], om.key_cache(l), f"slot {s} key cache layer {l}")
                assert_bit_equal(got[c.n_layers + l], om.value_cache(l), f"slot {s} value cache layer {l}")
            assert all(len(x) == nkv for x in got)
    finally:
        plan.free()
        om.close()


@pytest.mark.parametrize("shape", ["tiny-llama", "tiny-qwen3", "tiny-phi3", "tiny-qwen2", "tiny-granite", "tiny-devstral",
                                   "tiny-llama-q4_k_m", "mid-llama"])
def test_mixed_steps_bit_exact(pkg, orc, make_model, shape):
    m = _model(pkg, make_model, shape, 32 if shape.startswith("mid-") else 96)
    _run_mixed(pkg, orc, m, SCHEDULE)


def test_sampled_rows_equal_forward_decode_sample(pkg, orc, make_model):
    """Four slots on the same sequence; one step with a greedy, two top-p and a categorical row, and a K/V-only row of slot 0 after
    its emitting one.  Each id equals forward_decode_sample's (on the plan's own cache) and the oracle sampler's for the same
    uniform number, at a 128256-entry vocabulary."""
    m = make_model("tiny-llama-vocab128k", pkg.gguf.GGMLType.Q8_0, 24)
    c = m.configuration
    stream = orc.bench_tokens(c.vocab_size, c.context_length, seed=77)
    settings = [(0.0, 0.0, 0.0), (0.7, 0.9, 0.31), (1.0, 0.0, 0.77), (0.6, 0.95, 0.05)]
    P = 6
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = orc.OracleModel(m)
    try:
        plan.set_decode_slots(4)
        prompt = [(s, int(stream[p]), p, 0) for s in range(4) for p in range(P)]
        for k in range(0, len(prompt), 8):
            plan.forward_step(prompt[k:k + 8])
        rows = [(0, int(stream[P]), P, 1, *settings[0]), (0, int(stream[P + 1]), P + 1, 0)]
        rows += [(s, int(stream[P]), P, 1, *settings[s]) for s in (3, 1, 2)]
        ids, lg = plan.forward_step(rows, logits=True)
        for p in range(P):
            om.forward(int(stream[p]), p, want_logits=False)
            plan.forward_decode(int(stream[p]), p, logits=False)
        ref = om.forward(int(stream[P]), P)
        for i, r in enumerate(rows):
            if not r[3]:
                assert ids[i] == -1
                continue
            t, tp, u = r[4:]
            assert_bit_equal(lg[i], ref, f"row {i} logits")
            want = plan.forward_decode_sample(int(stream[P]), P, t, tp, u)
            assert ids[i] == want, (i, t, tp, u)
            assert ids[i] == (orc.argmax(ref) if t == 0.0 else orc.sample(ref, t, tp, u)), (i, t, tp, u)
    finally:
        plan.free()
        om.close()


def _requests(model_type, vocab, n=12, seed=3):
    rng = np.random.default_rng(seed)
    reqs = []
    for i in range(n):
        k = int(rng.integers(0 if model_type == "LLAMA_3" else 1, 13))
        reqs.append((int(rng.integers(vocab)), int(rng.integers(0, 4)), [int(t) for t in rng.integers(0, vocab, k)]))
    return reqs


ARRIVALS = [0, 0, 1, 2, 3, 5, 8, 8, 10, 13, 20, 30]


@pytest.mark.parametrize("shape", ["tiny-llama", "tiny-qwen3"])
def test_generate_tokens_continuous_greedy_equals_oracle_loop(pkg, orc, make_model, shape):
    m = make_model(shape, pkg.gguf.GGMLType.Q8_0, 64)
    c = m.configuration
    loop = pkg.engine.loop_for(m.model_type)
    reqs = _requests("QWEN_3" if loop is pkg.engine.generate_tokens_qwen3 else "LLAMA_3", c.vocab_size)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = orc.OracleModel(m)
    try:
        plan.set_decode_slots(4)
        refs = []
        for latest, start, prompt in reqs:
            om.reset()
            refs.append(loop(om.forward_argmax, latest, start, prompt, [], 40, 64))
        stop = [refs[3][2]]  # ends request 3 (and any other that meets it) early
        refs = []
        for latest, start, prompt in reqs:
            om.reset()
            refs.append(loop(om.forward_argmax, latest, start, prompt, stop, 40, 64))
        stats = {}
        got = pkg.engine.generate_tokens_continuous(plan, m.model_type, reqs, ARRIVALS, stop, 40, 64, stats=stats)
        assert got == refs
        assert max(stats["rows"]) == 8 and stats["steps"] < sum(len(r) for r in refs)
    finally:
        plan.free()
        om.close()


def _sampled_alone(pkg, plan, model_type, req, sampler, stop, budget, ctx):
    """The request's loop on the plan's own cache: prompt rows through forward_decode, each generated token through the sampler."""
    latest, start, prompt = req
    llama = pkg.engine.loop_for(model_type) is pkg.engine.generate_tokens_llama
    kv_rows = len(prompt) if llama else max(len(prompt) - 1, 0)
    seen = [0]

    def forward(tok, pos):
        seen[0] += 1
        if seen[0] <= kv_rows:
            return plan.forward_decode(tok, pos, logits=False)[1]
        return sampler.sample_token(plan, tok, pos)

    plan.kv_reset()
    return pkg.engine.loop_for(model_type)(forward, latest, start, prompt, stop, budget, ctx)


@pytest.mark.parametrize("shape", ["tiny-llama", "tiny-qwen3"])
def test_generate_tokens_continuous_sampled_equals_single_plan(pkg, orc, make_model, shape):
    m = make_model(shape, pkg.gguf.GGMLType.Q8_0, 64)
    c = m.configuration
    S = pkg.sampler
    llama = pkg.engine.loop_for(m.model_type) is pkg.engine.generate_tokens_llama
    reqs = _requests("LLAMA_3" if llama else "QWEN_3", c.vocab_size, seed=8)
    settings = [(0.8, 0.9), (1.0, 0.0), (0.0, 0.0), (0.6, 0.95)]
    make = lambda i: S.Sampler(c.vocab_size, *settings[i % 4], 100 + i)  # noqa: E731
    plan = pkg.B200MasterPlan.initialize_plan(m)
    try:
        plan.set_decode_slots(4)
        got = pkg.engine.generate_tokens_continuous(plan, m.model_type, reqs, ARRIVALS, [], 40, 64, samplers=[make(i) for i in range(len(reqs))])
        for i, req in enumerate(reqs):
            assert got[i] == _sampled_alone(pkg, plan, m.model_type, req, make(i), [], 40, 64), f"request {i}"
    finally:
        plan.free()


def test_batch_and_single_decode_after_mixed_steps(pkg, orc, make_model):
    m = make_model("tiny-llama", pkg.gguf.GGMLType.Q8_0, 64)
    c = m.configuration
    streams = [orc.bench_tokens(c.vocab_size, c.context_length, seed=90 + s) for s in range(4)]
    oms = [orc.OracleModel(m) for _ in range(4)]  # slots 0..2, then the plan's own sequence
    plan = pkg.B200MasterPlan.initialize_plan(m)
    try:
        plan.set_decode_slots(3)
        pos = [0, 0, 0]
        for it in range(6):
            rows = [(0, int(streams[0][pos[0]]), pos[0], 1), (0, int(streams[0][pos[0] + 1]), pos[0] + 1, 0),
                    (1, int(streams[1][pos[1]]), pos[1], 1)]
            ids, lg = plan.forward_step(rows, logits=True)
            oms[0].forward(rows[0][1], rows[0][2])
            oms[0].forward(rows[1][1], rows[1][2], want_logits=False)
            oms[1].forward(rows[2][1], rows[2][2])
            pos[0] += 2
            pos[1] += 1
            toks = [int(streams[2][pos[2]]), int(streams[1][pos[1]])]
            ids, blg = plan.forward_decode_batch([2, 1], toks, [pos[2], pos[1]], logits=True)
            assert plan.batch_info()[1] == 7 * c.n_layers + 3
            for k, s in enumerate((2, 1)):
                ref = oms[s].forward(toks[k], pos[s])
                assert_bit_equal(blg[k], ref, f"batched slot {s} step {it}")
                assert ids[k] == orc.argmax(ref)
                pos[s] += 1
            lg1, am = plan.forward_decode(int(streams[3][it]), it)
            ref = oms[3].forward(int(streams[3][it]), it)
            assert_bit_equal(lg1, ref, f"forward_decode step {it}")
            assert am == orc.argmax(ref)
    finally:
        plan.free()
        for o in oms:
            o.close()


def _expect(pkg, fn, code, text):
    with pytest.raises(pkg.native.B200Error) as e:
        fn()
    assert e.value.code == code and text in str(e.value), str(e.value)


def test_forward_step_refusals(pkg, make_model):
    m = make_model("tiny-llama", pkg.gguf.GGMLType.Q8_0, 64)
    V = m.configuration.vocab_size
    plan = pkg.B200MasterPlan.initialize_plan(m)
    try:
        _expect(pkg, lambda: plan.forward_step([(0, 1, 0, 1)]), -6, "b200_set_decode_slots")
        plan.set_decode_slots(3)
        _expect(pkg, lambda: plan.forward_step([]), -1, "n = 0 rows")
        _expect(pkg, lambda: plan.forward_step([(0, 1, p, 0) for p in range(9)]), -1, "n = 9 rows")
        _expect(pkg, lambda: plan.forward_step([(0, 1, 0, 1), (3, 1, 0, 1)]), -1, "row 1: slot 3 out of range")
        _expect(pkg, lambda: plan.forward_step([(-1, 1, 0, 1)]), -1, "row 0: slot -1 out of range")
        _expect(pkg, lambda: plan.forward_step([(0, V, 0, 1)]), -1, f"row 0: token {V} out of range")
        _expect(pkg, lambda: plan.forward_step([(1, 1, 0, 0), (0, 1, 64, 1)]), -1, "row 1: position 64 outside")
        _expect(pkg, lambda: plan.forward_step([(0, 1, 2, 0), (1, 1, 2, 0), (0, 5, 2, 1)]), -1, "row 2: slot 0 position 2 repeats row 0's")
        _expect(pkg, lambda: plan.forward_step([(0, 1, 0, 2)]), -1, "row 0: emit must be 0 or 1")
        _expect(pkg, lambda: plan.forward_step([(0, 1, 0, 0), (1, 1, 0, 1, -1.0, 0.9, 0.5)]), -1, "row 1: temperature")
        _expect(pkg, lambda: plan.forward_step([(0, 1, 0, 1, 0.7, 0.9, 1.0)]), -1, "row 0: temperature")
        _expect(pkg, lambda: plan.forward_step([(0, 1, 0, 1, float("nan"), 0.9, 0.5)]), -1, "row 0: temperature")
        plan.set_sampling_controls(1, pkg.sampler.SamplingControls(top_k=3))
        _expect(pkg, lambda: plan.forward_step([(1, 1, 0, 1), (0, 1, 0, 0), (1, 2, 1, 1)]), -1,
                "row 2: slot 1 has sampling controls and already emits in row 0")
        ids, _ = plan.forward_step([(2, 1, 0, 0), (2, 2, 1, 1)])  # a valid call still works after the rejected ones
        assert ids[0] == -1 and 0 <= ids[1] < V
        assert np.isfinite(plan.forward_decode(1, 0)[0]).all()
    finally:
        plan.free()
    fp16 = pkg.B200MasterPlan.initialize_plan(make_model("tiny-llama", pkg.gguf.GGMLType.F16, 64))
    try:
        _expect(pkg, lambda: fp16.forward_step([(0, 1, 0, 1)]), -2, "Q8_0 weights")
        assert np.isfinite(fp16.forward_decode(1, 0)[0]).all()
    finally:
        fp16.free()
    moe = pkg.B200MasterPlan.initialize_plan(make_model("tiny-qwen2moe", pkg.gguf.GGMLType.Q8_0, 64))
    try:
        _expect(pkg, lambda: moe.forward_step([(0, 1, 0, 1)]), -2, "Qwen2-MoE")
        assert np.isfinite(moe.forward_decode(1, 0)[0]).all()
    finally:
        moe.free()
