"""GPU tests of the tensor-core chunk step (b200_forward_chunk) and chunked admission in the continuous batcher.

A chunk runs forward_step's rows through the bit-exact int8 prefill and the batched classifier, so every comparison is bitwise
(uint32 views): each emitting row's logits and id against the same rows through forward_step on a second plan (in position order,
decode_multi_rows() rows per step) and against the CPU oracle, every named slot's K / V, and the bytes the call must not touch.  The
rows are also run shuffled and padded with other slots' prompt rows, since a row's result must not depend on the chunk's length or
on its place in it."""
import numpy as np
import pytest

from test_gpu_batch_decode import _model
from test_gpu_continuous import _expect, _oracle, _sampled_alone
from test_gpu_kquant_resident import _model as _kq_model, _resident_plan
from test_gpu_parity import assert_bit_equal
from test_gpu_q8_any_width import _model as _width_model
from test_gpu_slot_prefill import _kv, _own_kv, _same_bytes

pytestmark = pytest.mark.gpu

PAD_SLOTS = (4, 5)  # slots only the padded chunks name


def _rows(streams, spec):
    """spec: (slot, start, n, emit) with emit "none", "last" or "all" -> forward_step rows over the slot's token stream."""
    rows = []
    for s, start, n, emit in spec:
        for j in range(n):
            e = emit == "all" or (emit == "last" and j == n - 1)
            rows.append((s, int(streams[s][start + j]), start + j, int(e)))
    return rows


def _by_steps(plan, rows):
    """rows through forward_step in position order, decode_multi_rows() per step -> {(slot, position): (id, logits)} of the
    emitting rows."""
    R = plan.decode_multi_rows()
    order = sorted(rows, key=lambda r: r[2])
    out = {}
    for k in range(0, len(order), R):
        part = order[k:k + R]
        ids, lg = plan.forward_step(part, logits=True)
        for j, r in enumerate(part):
            if r[3]:
                out[(r[0], r[2])] = (int(ids[j]), lg[j].copy())
    return out


def _chunk(plan, rows, want):
    """One forward_chunk; every emitting row equal to want[(slot, position)], every other row -1 with its logits unwritten."""
    ids, lg = plan.forward_chunk(rows, logits=True)
    for i, r in enumerate(rows):
        if not r[3]:
            assert ids[i] == -1 and not lg[i].any(), f"K/V-only row {i} returned output"
            continue
        wid, wlg = want[(r[0], r[2])]
        assert_bit_equal(lg[i], wlg, f"row {i} (slot {r[0]} position {r[2]}) logits")
        assert ids[i] == wid, f"row {i} (slot {r[0]} position {r[2]}) id"


def _variant(calls, kind, rng, streams, ctx):
    """The calls as run: as given, each shuffled, or each padded with prompt rows of PAD_SLOTS at random places."""
    out, nxt = [], {s: 0 for s in PAD_SLOTS}
    for rows in calls:
        rows = list(rows)
        if kind == "padded":
            for s in PAD_SLOTS:
                k = int(rng.integers(1, 9))
                for _ in range(k):
                    if nxt[s] < ctx:
                        rows.insert(int(rng.integers(0, len(rows) + 1)), (s, int(streams[s][nxt[s]]), nxt[s], 0))
                        nxt[s] += 1
        elif kind == "shuffled":
            rows = [rows[i] for i in rng.permutation(len(rows))]
        out.append(rows)
    return out


def _run_mixed(pkg, orc, m, spec, batch, oracle=True):
    c = m.configuration
    streams = [orc.bench_tokens(c.vocab_size, c.context_length, seed=700 + s) for s in range(6)]
    calls = [_rows(streams, call) for call in spec]
    ref = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=batch)
    pt = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=batch)
    rng = np.random.default_rng(c.context_length + batch)
    try:
        ref.set_decode_slots(4)
        want = [_by_steps(ref, rows) for rows in calls]
        ref_kv = [_kv(ref, c, s) for s in range(4)]
        pt.set_decode_slots(6)
        assert pt.chunk_rows() == 0  # not in tensor_core_exact yet
        pt.set_prefill_mode("tensor_core_exact")
        assert pt.chunk_rows() == batch
        # bytes the calls must not touch: the plan's own cache after a few tokens, and the padding slots after a step of their own
        for pos in range(4):
            lg_own, id_own = pt.forward_decode(int(streams[0][pos]), pos)
        lg_own = lg_own.copy()
        own = _own_kv(pt, c)
        pt.forward_step([(s, int(streams[s][p]), p, 0) for s in PAD_SLOTS for p in range(3)])
        pads = [_kv(pt, c, s) for s in PAD_SLOTS]
        info = pt.prefill_info()
        for kind in ("plain", "shuffled", "padded"):
            if kind != "plain":
                for s in range(4):
                    pt.slot_reset(s)
            for rows, w in zip(_variant(calls, kind, rng, streams, c.context_length), want):
                _chunk(pt, rows, w)
                launches, ms = pt.batch_info()[1:]
                assert launches > 0 and ms > 0.0
            for s in range(4):
                _same_bytes(_kv(pt, c, s), ref_kv[s], f"{kind}: slot {s} K / V differ from forward_step's")
            if kind == "plain":
                for s, kv in zip(PAD_SLOTS, pads):
                    _same_bytes(_kv(pt, c, s), kv, f"slot {s}, named by no row, changed")
        assert pt.prefill_info() == info, "forward_chunk changed prefill_info"
        _same_bytes(_own_kv(pt, c), own, "the plan's own cache changed")
        lg, am = pt.forward_decode(int(streams[0][3]), 3)
        assert_bit_equal(lg, lg_own, "forward_decode on the plan's own cache after the chunks")
        assert am == id_own
    finally:
        ref.free()
        pt.free()
    if not oracle:
        return
    om = _oracle(pkg, orc, m)
    try:
        for s in range(4):
            om.reset()
            for tok_pos in sorted({(r[1], r[2], r[3]) for rows in calls for r in rows if r[0] == s}, key=lambda t: t[1]):
                tok, pos, e = tok_pos
                if not e:
                    om.forward(tok, pos, want_logits=False)
                    continue
                lg_ref = om.forward(tok, pos)
                wid, wlg = next(w[(s, pos)] for w in want if (s, pos) in w)
                assert_bit_equal(wlg, lg_ref, f"slot {s} position {pos} logits against the oracle")
                assert wid == orc.argmax(lg_ref), f"slot {s} position {pos} id against the oracle"
    finally:
        om.close()


# Three calls on slots 0..3: decode rows at several depths, a whole prompt whose last row emits (slots 0 and 2), a prompt prefilled
# in part (slot 1, 137 rows: two 128-row GEMM tiles) and continued later, and three consecutive emitting rows of slot 0.
SPEC = [
    [(0, 0, 20, "last"), (1, 0, 137, "none"), (2, 0, 9, "last")],
    [(0, 20, 1, "all"), (2, 9, 1, "all"), (1, 137, 24, "last"), (3, 0, 5, "none")],
    [(0, 21, 3, "all"), (1, 161, 1, "all"), (2, 10, 1, "all"), (3, 5, 8, "last")],
]


@pytest.mark.parametrize("shape", ["tiny-llama", "tiny-qwen3", "tiny-qwen2", "tiny-phi3", "tiny-granite", "tiny-devstral", "mid-llama"])
def test_mixed_chunks_bit_exact(pkg, orc, make_model, shape):
    _run_mixed(pkg, orc, _model(pkg, make_model, shape, 256), SPEC, 256)


def test_deep_rows_use_the_global_score_rows(pkg, orc, make_model):
    """A context above 4096 keys: decode and prompt rows past position 4096, whose attention scores live in global memory."""
    spec = [[(0, 0, 40, "none"), (1, 0, 40, "none"), (2, 0, 40, "last")],
            [(0, 4097, 24, "last"), (1, 4200, 1, "all"), (2, 4300, 1, "all"), (3, 0, 30, "none")]]
    _run_mixed(pkg, orc, make_model("tiny-llama", pkg.gguf.GGMLType.Q8_0, 4352), spec, 256)


def _same_logprobs(a, rows_a, b, rows_b):
    """last_logprobs() tables a and b, their rows matched by (slot, position); rows of a that do not emit: NaN and ids -1."""
    at = {(r[0], r[2]): i for i, r in enumerate(rows_b)}
    for i, r in enumerate(rows_a):
        if not r[3]:
            assert np.isnan(a[0][i]) and (a[1][i] == -1).all() and np.isnan(a[2][i]).all()
            continue
        j = at[(r[0], r[2])]
        assert a[0][i] == b[0][j] and np.array_equal(a[1][i], b[1][j]) and np.array_equal(a[2][i], b[2][j]), f"row {i} logprobs"


def test_sampled_rows_controls_and_logprobs(pkg, orc, make_model):
    """Four sequences with sampled and greedy emitting rows, two of them under per-slot controls (penalties, top-k, min-p, bias),
    logprobs on with 5 alternatives; each chunk also carries prompt rows of a fifth slot.  Ids, logprob rows and the controlled slots'
    counts equal forward_step's on the same rows."""
    m = make_model("tiny-llama", pkg.gguf.GGMLType.Q8_0, 128)
    c = m.configuration
    S = pkg.sampler
    controls = {0: S.SamplingControls(top_k=40, min_p=0.02, repetition_penalty=1.3, frequency_penalty=0.4, presence_penalty=0.2,
                                      logit_bias={3: 2.5, 17: -4.0}),
                1: S.SamplingControls(top_k=5, repetition_penalty=0.8, logit_bias={5: 1.0})}
    settings = [(0.8, 0.9), (1.0, 0.0), (0.7, 0.95), (0.0, 0.0)]
    streams = [orc.bench_tokens(c.vocab_size, c.context_length, seed=40 + s) for s in range(5)]
    plans = [pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=64) for _ in range(2)]
    ref, pt = plans
    rng = np.random.default_rng(12)
    try:
        for p in plans:
            p.set_decode_slots(5)
            for s, ctl in controls.items():
                p.set_sampling_controls(s, ctl)
                p.set_sample_history(s, [int(t) for t in streams[s][:6]])
            p.set_logprobs(5)
        pt.set_prefill_mode("tensor_core_exact")
        P = 6
        prompt = _rows(streams, [(s, 0, P, "none") for s in range(4)])
        _by_steps(ref, prompt)
        pt.forward_chunk(prompt)
        tok, pad = [int(streams[s][P]) for s in range(4)], 0
        for it in range(6):
            rows = [(s, tok[s], P + it, 1, settings[s][0], settings[s][1], float(rng.random())) for s in range(4)]
            ids_r, lg_r = ref.forward_step(rows, logits=True)
            lp_r = ref.last_logprobs()
            chunk = list(rows)
            for _ in range(int(rng.integers(3, 12))):
                chunk.insert(int(rng.integers(0, len(chunk) + 1)), (4, int(streams[4][pad]), pad, 0))
                pad += 1
            ids_t, lg_t = pt.forward_chunk(chunk, logits=True)
            lp_t = pt.last_logprobs()
            for i, r in enumerate(chunk):
                if r[0] == 4:
                    assert ids_t[i] == -1
                    continue
                assert ids_t[i] == ids_r[r[0]], (it, r)
                assert_bit_equal(lg_t[i], lg_r[r[0]], f"step {it} slot {r[0]} logits")
            _same_logprobs(lp_t, chunk, lp_r, rows)
            tok = [int(i) for i in ids_r]
        for s in controls:
            assert np.array_equal(pt.sample_counts(s), ref.sample_counts(s)), f"slot {s} counts"
    finally:
        for p in plans:
            p.free()


def _long_requests(model_type, vocab, seed):
    rng = np.random.default_rng(seed)
    return [(int(rng.integers(vocab)), int(rng.integers(0, 4)), [int(t) for t in rng.integers(0, vocab, int(rng.integers(5, 151)))])
            for _ in range(10)]


ARRIVALS = [0, 0, 0, 2, 5, 9, 14, 30, 31, 60]


@pytest.mark.parametrize("sampled", [False, True])
@pytest.mark.parametrize("shape", ["tiny-llama", "tiny-qwen3"])
def test_continuous_chunked_admission(pkg, orc, make_model, shape, sampled):
    """generate_tokens_continuous with chunk_rows = 64 on 4 slots: every request equals its loop alone and the chunk_rows = 0 run,
    and chunk steps ran."""
    m = make_model(shape, pkg.gguf.GGMLType.Q8_0, 256)
    c = m.configuration
    loop = pkg.engine.loop_for(m.model_type)
    reqs = _long_requests(m.model_type, c.vocab_size, 21 if sampled else 22)
    settings = [(0.8, 0.9), (1.0, 0.0), (0.0, 0.0), (0.6, 0.95)]
    make = (lambda i: pkg.sampler.Sampler(c.vocab_size, *settings[i % 4], 300 + i)) if sampled else None  # noqa: E731
    budget = 200
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=128)
    try:
        plan.set_decode_slots(4)
        plan.set_prefill_mode("tensor_core_exact")
        runs = {}
        for rows in (64, 0):
            stats = {}
            smp = [make(i) for i in range(len(reqs))] if sampled else None
            runs[rows] = pkg.engine.generate_tokens_continuous(plan, m.model_type, reqs, ARRIVALS, [], budget, 256, samplers=smp, stats=stats,
                                                               chunk_rows=rows)
            kinds = set(stats["kinds"])
            assert kinds == ({"chunk", "step"} if rows else {"step"}), kinds
            if rows:
                assert all(n <= 64 for n in stats["rows"]) and all(n >= 32 for k, n in zip(stats["kinds"], stats["rows"]) if k == "chunk")
        assert runs[64] == runs[0]
        if sampled:
            for i, req in enumerate(reqs):
                assert runs[64][i] == _sampled_alone(pkg, plan, m.model_type, req, make(i), [], budget, 256), f"request {i}"
        else:
            om = orc.OracleModel(m)
            try:
                for i, (latest, start, prompt) in enumerate(reqs):
                    om.reset()
                    assert runs[64][i] == loop(om.forward_argmax, latest, start, prompt, [], budget, 256), f"request {i}"
            finally:
                om.close()
    finally:
        plan.free()


def test_refusals(pkg, make_model):
    """Every refusal names its reason; a valid call works after them."""
    G = pkg.gguf.GGMLType
    m = make_model("tiny-llama", G.Q8_0, 64)
    V = m.configuration.vocab_size
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=16)
    try:
        _expect(pkg, lambda: plan.forward_chunk([(0, 1, 0, 1)]), -6, "b200_set_decode_slots")
        plan.set_decode_slots(3)
        for mode in ("exact", "tensor_core", "tensor_core_w8a16"):
            plan.set_prefill_mode(mode)
            assert plan.chunk_rows() == 0
            _expect(pkg, lambda: plan.forward_chunk([(0, 1, 0, 1)]), -6, f"prefill mode is {mode}")
        plan.set_prefill_mode("tensor_core_exact")
        assert plan.chunk_rows() == 16
        _expect(pkg, lambda: plan.forward_chunk([]), -1, "n = 0 rows")
        _expect(pkg, lambda: plan.forward_chunk([(0, 1, p, 0) for p in range(17)]), -1, "n = 17 rows")
        _expect(pkg, lambda: plan.forward_chunk([(s % 3, 1, s, 1) for s in range(9)]), -1, "row 8: more than 8 emitting rows")
        _expect(pkg, lambda: plan.forward_chunk([(0, 1, 0, 0), (1, 1, 0, 0), (0, 5, 0, 1)]), -1, "row 2: slot 0 position 0 repeats row 0's")
        _expect(pkg, lambda: plan.forward_chunk([(0, 1, 0, 2)]), -1, "row 0: emit must be 0 or 1")
        _expect(pkg, lambda: plan.forward_chunk([(0, 1, 0, 1), (3, 1, 0, 1)]), -1, "row 1: slot 3 out of range")
        _expect(pkg, lambda: plan.forward_chunk([(0, V, 0, 1)]), -1, f"row 0: token {V} out of range")
        _expect(pkg, lambda: plan.forward_chunk([(1, 1, 0, 0), (0, 1, 64, 1)]), -1, "row 1: position 64 outside")
        _expect(pkg, lambda: plan.forward_chunk([(0, 1, 0, 1, 0.7, 0.9, 1.0)]), -1, "row 0: temperature")
        plan.set_sampling_controls(1, pkg.sampler.SamplingControls(top_k=3))
        _expect(pkg, lambda: plan.forward_chunk([(1, 1, 0, 1), (2, 1, 0, 0), (1, 2, 1, 1)]), -1, "row 2: slot 1 has sampling controls")
        _expect(pkg, lambda: plan.forward_chunk([(2, 1, 0, 0), (1, 1, 0, 1), (1, 2, 1, 1)]), -1,
                "row 2: slot 1 has sampling controls and already emits in row 1")
        ids, _ = plan.forward_chunk([(2, 1, 0, 0), (2, 2, 1, 1), (0, 3, 0, 1), (0, 4, 1, 1)])  # a slot without controls may emit twice
        assert ids[0] == -1 and all(0 <= i < V for i in ids[1:])
        assert np.isfinite(plan.forward_decode(1, 0)[0]).all()
    finally:
        plan.free()
    for make, why in ((lambda: make_model("tiny-llama", G.F16, 64), "Q8_0 weights"), (lambda: make_model("tiny-qwen2moe", G.Q8_0, 64), "Qwen2-MoE"),
                      (lambda: _width_model(pkg, "hidden-2656"), "multiples of 64 columns")):
        p = pkg.B200MasterPlan.initialize_plan(make(), prefill_batch_size=16)
        try:
            if why == "multiples of 64 columns":
                p.set_decode_slots(2)
            _expect(pkg, lambda: p.forward_chunk([(0, 1, 0, 1)]), -2, why)
            assert p.chunk_rows() == 0
            assert np.isfinite(p.forward_decode(1, 0)[0]).all()
        finally:
            p.free()
    p = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=0)
    try:
        p.set_decode_slots(2)
        _expect(pkg, lambda: p.forward_chunk([(0, 1, 0, 1)]), -2, "prefill batch size")
    finally:
        p.free()
    p = _resident_plan(pkg, _kq_model(pkg, "tiny-llama"), prefill_batch_size=16)
    try:
        _expect(pkg, lambda: p.forward_chunk([(0, 1, 0, 1)]), -2, "resident")
    finally:
        p.free()
    cfg = pkg.plan.make_config(m)  # rank 0 of a two-way tensor-parallel plan, created without its peer
    cfg.tp_rank, cfg.tp_size = 0, 2
    p = pkg.native.NativePlan(cfg, m.tensors, 0, 0)
    try:
        _expect(pkg, lambda: p.forward_chunk([(0, 1, 0, 1)]), -2, "tensor-parallel")
    finally:
        p.free()
