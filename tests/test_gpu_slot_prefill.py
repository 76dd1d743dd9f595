"""GPU tests of the multi-slot prefill (b200_prefill_slots): prompts prefilled straight into decode slots, several per call.

Exact mode is the batched decode step without its classifier, so every slot's K/V (uint32) and the next batched step's logits are
bit-equal to the CPU restatement of that sequence alone.  The tensor-core modes pack every prompt into one chunk; where no residual
GEMM splits K, each slot's K/V is bit-equal to the same prompt prefilled alone, and the packed attention kernel is bit-equal to the
single-sequence kernel on each sequence."""
import numpy as np
import pytest

from granite_oracle import GraniteOracle
from test_gpu_batch_decode import _model
from test_gpu_batch_decode import _oracle as _batch_oracle
from test_gpu_parity import assert_bit_equal
from test_gpu_prefill import Q8_NOISE_TOL

pytestmark = pytest.mark.gpu


def _oracle(pkg, orc, m):
    return GraniteOracle(orc, m) if m.configuration.arch == 5 else _batch_oracle(pkg, orc, m)


def _kv(plan, c, slot):
    nkv = c.context_length * c.kv_dim
    return [plan.read_buffer(n, nkv, layer=slot * c.n_layers + l) for n in ("slot_key_cache", "slot_value_cache") for l in range(c.n_layers)]


def _own_kv(plan, c):
    nkv = c.context_length * c.kv_dim
    return [plan.read_buffer(n, nkv, layer=l) for n in ("key_cache", "value_cache") for l in range(c.n_layers)]


def _same_bytes(a, b, what):
    for x, y in zip(a, b):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), what


# Two calls on four slots: the first names slots 2, 0, 3 out of order (slot 1 untouched), the second continues slot 2 at start 37
# and starts slot 1, leaving slots 0 and 3 out.
CALLS = [([2, 0, 3], [0, 0, 0], [37, 7, 130]), ([1, 2], [0, 37], [1, 20])]


def _exact_run(pkg, orc, m, n_slots, calls, decode=True):
    c = m.configuration
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = _oracle(pkg, orc, m)
    streams = [orc.bench_tokens(c.vocab_size, c.context_length, seed=200 + s) for s in range(n_slots)]
    fed = [0] * n_slots
    try:
        plan.set_decode_slots(n_slots)
        own = _own_kv(plan, c)
        for slots, starts, lens in calls:
            named = set(slots)
            before = {s: _kv(plan, c, s) for s in range(n_slots) if s not in named}
            plan.prefill_slots(slots, starts, [streams[s][st:st + n] for s, st, n in zip(slots, starts, lens)])
            for s, st, n in zip(slots, starts, lens):
                assert st == fed[s]
                fed[s] = st + n
            for s, kv in before.items():
                _same_bytes(_kv(plan, c, s), kv, f"slot {s} was not named but changed")
            _same_bytes(_own_kv(plan, c), own, "the plan's own cache changed")
        lg = None
        rows = [s for s in range(n_slots) if fed[s]]
        if decode:
            ids, lg = plan.forward_decode_batch(rows, [int(streams[s][fed[s]]) for s in rows], [fed[s] for s in rows], logits=True)
        for i, s in enumerate(rows):
            om.reset()
            for p in range(fed[s]):
                om.forward(int(streams[s][p]), p, want_logits=False)
            if decode:
                ref = om.forward(int(streams[s][fed[s]]), fed[s])
                assert_bit_equal(lg[i], ref, f"slot {s}: logits of the first decode step")
                assert ids[i] == orc.argmax(ref)
            for l in range(c.n_layers):
                nkv = c.context_length * c.kv_dim
                assert_bit_equal(plan.read_buffer("slot_key_cache", nkv, layer=s * c.n_layers + l), om.key_cache(l), f"slot {s} key cache layer {l}")
                assert_bit_equal(plan.read_buffer("slot_value_cache", nkv, layer=s * c.n_layers + l), om.value_cache(l), f"slot {s} value cache layer {l}")
        return plan.prefill_info()
    finally:
        plan.free()
        om.close()


@pytest.mark.parametrize("shape", ["tiny-llama", "tiny-qwen3", "tiny-qwen2", "tiny-phi3", "tiny-granite", "tiny-llama-q4_k_m"])
def test_exact_prefill_slots_bit_exact(pkg, orc, make_model, shape):
    m = _model(pkg, make_model, shape, 192)
    mode, launches, ms = _exact_run(pkg, orc, m, 4, CALLS)
    assert mode == 0 and launches > 0 and ms > 0


@pytest.mark.parametrize("shape", ["mid-llama", "mid-qwen3-4b"])
def test_exact_prefill_slots_8_rows_mid_geometries(pkg, orc, make_model, shape):
    m = _model(pkg, make_model, shape, 16)
    _exact_run(pkg, orc, m, 8, [(list(range(8))[::-1], [0] * 8, [5, 1, 8, 3, 8, 2, 7, 4])], decode=False)


@pytest.mark.parametrize("hs", [64, 128])
@pytest.mark.parametrize("kv_mul", [1, 2, 4, 7, 8])
def test_packed_attention_matches_single_sequence(pkg, hs, kv_mul):
    N = pkg.native
    nkv = 2
    nh = nkv * kv_mul
    rng = np.random.default_rng(hs * 10 + kv_mul)
    lens, starts = [5, 70, 33, 64], [0, 17, 64, 3]
    qs = [rng.standard_normal((n, nh * hs)).astype(np.float32) for n in lens]
    ks = [rng.standard_normal((st + n, nkv * hs)).astype(np.float32) for n, st in zip(lens, starts)]
    vs = [rng.standard_normal((st + n, nkv * hs)).astype(np.float32) for n, st in zip(lens, starts)]
    packed = N.test_pf_attention_packed(qs, ks, vs, starts, nh, nkv)
    for i in range(len(lens)):
        alone = N.test_pf_attention(qs[i], ks[i], vs[i], nh, nkv, starts[i])
        assert np.array_equal(packed[i], alone), f"sequence {i} (n {lens[i]}, start {starts[i]}) differs from its single-sequence launch"


def _tc_plan(pkg, m, mode, slots, batch):
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=batch)
    plan.set_prefill_mode(mode)
    plan.set_decode_slots(slots)
    return plan


@pytest.mark.parametrize("shape", ["tiny-llama", "tiny-qwen3", "tiny-granite"])
@pytest.mark.parametrize("mode", ["tensor_core", "tensor_core_w8a16"])
def test_tensor_core_prefill_slots_equal_single_prompt(pkg, orc, make_model, shape, mode):
    """Every residual GEMM of these shapes has at most 8 k-blocks, so K is never split: each slot's K/V is bit-equal to its prompt
    prefilled alone through forward_batch_prefill in the same mode and chunks, continuation chunks (start > 0) included."""
    m = make_model(shape, pkg.gguf.GGMLType.Q8_0, 128)
    c = m.configuration
    calls = [([1, 0, 2], [0, 0, 0], [20, 9, 30]), ([0, 2], [9, 30], [25, 10])]
    streams = [orc.bench_tokens(c.vocab_size, c.context_length, seed=300 + s) for s in range(3)]
    plan, ref = _tc_plan(pkg, m, mode, 3, 64), _tc_plan(pkg, m, mode, 1, 64)
    try:
        own = _own_kv(plan, c)
        for slots, starts, lens in calls:
            plan.prefill_slots(slots, starts, [streams[s][st:st + n] for s, st, n in zip(slots, starts, lens)])
        _same_bytes(_own_kv(plan, c), own, "the plan's own cache changed")
        assert plan.prefill_info()[0] == {"tensor_core": 1, "tensor_core_w8a16": 2}[mode]
        for s in range(3):
            ref.kv_reset()
            for slots, starts, lens in calls:
                if s in slots:
                    k = slots.index(s)
                    ref.forward_batch_prefill(streams[s][starts[k]:starts[k] + lens[k]], starts[k])
            _same_bytes(_kv(plan, c, s), _own_kv(ref, c), f"{shape} {mode}: slot {s} differs from its prompt prefilled alone")
    finally:
        plan.free()
        ref.free()


def test_tensor_core_prefill_slots_mid_llama(pkg, orc):
    """Llama-3-8B layer geometry with 8 prompts in one chunk (split-K residual GEMMs): each slot's K/V and its first decode step's
    logits within the Q8_0 bar of tests/test_gpu_prefill.py against the CPU path, in both tensor-core modes."""
    sh = pkg.synth.SHAPES["mid-llama"]
    Q8 = pkg.gguf.GGMLType.Q8_0
    m = pkg.loader.model_from_tensors(sh, Q8, pkg.synth.build_tensors_fast(sh, Q8, seed=1234), 32)
    c = m.configuration
    lens = [12, 9, 3, 12, 5, 11, 7, 12]
    streams = [orc.bench_tokens(c.vocab_size, 16, seed=400 + s) for s in range(8)]
    nkv = c.context_length * c.kv_dim
    om = orc.OracleModel(m)
    refs = []
    for s in range(8):
        om.reset()
        for p in range(lens[s]):
            om.forward(int(streams[s][p]), p, want_logits=False)
        lg = om.forward(int(streams[s][lens[s]]), lens[s])
        refs.append(([om.key_cache(l)[:lens[s] * c.kv_dim] for l in range(c.n_layers)], [om.value_cache(l)[:lens[s] * c.kv_dim] for l in range(c.n_layers)], lg))
    om.close()
    for mode in ("tensor_core", "tensor_core_w8a16"):
        plan = _tc_plan(pkg, m, mode, 8, 128)
        try:
            slots = [3, 0, 7, 1, 6, 2, 5, 4]
            plan.prefill_slots(slots, [0] * 8, [streams[s][:lens[s]] for s in slots])
            ids, lg = plan.forward_decode_batch(list(range(8)), [int(streams[s][lens[s]]) for s in range(8)], lens, logits=True)
            for s in range(8):
                rk, rv, rl = refs[s]
                for l in range(c.n_layers):
                    for name, r in (("slot_key_cache", rk[l]), ("slot_value_cache", rv[l])):
                        got = plan.read_buffer(name, nkv, layer=s * c.n_layers + l)[:lens[s] * c.kv_dim]
                        err = float(np.max(np.abs(got - r)) / np.max(np.abs(r)))
                        assert err <= Q8_NOISE_TOL, f"{mode} slot {s} {name} layer {l}: rel err {err:.2e}"
                err = float(np.max(np.abs(lg[s] - rl)) / np.max(np.abs(rl)))
                assert err <= Q8_NOISE_TOL, f"{mode} slot {s}: first decode step logits rel err {err:.2e}"
        finally:
            plan.free()


@pytest.mark.parametrize("mode", ["exact", "tensor_core", "tensor_core_w8a16"])
def test_generate_tokens_batch_prefill(pkg, orc, make_model, mode):
    """Four requests, one stopping early; batch_size 16 makes the 20-token prompt span two prefill calls.  Each request's ids equal
    generate_tokens_llama_batch_prefill for it alone on the same plan and mode, and in exact mode the oracle loop's too."""
    m = make_model("tiny-llama", pkg.gguf.GGMLType.Q8_0, 96)
    E = pkg.engine
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=16)
    om = orc.OracleModel(m)
    reqs = [(7, 0, [7, 11, 12]), (3, 0, [3] + list(range(40, 59))), (5, 0, [5, 9]), (8, 0, [8, 2, 2, 2, 2])]
    try:
        if mode != "exact":
            plan.set_prefill_mode(mode)
        plan.set_decode_slots(4)
        first = E.generate_tokens_batch_prefill(plan, m.model_type, reqs, [], 40, 96, 16)
        stop = [first[1][3]]
        got = E.generate_tokens_batch_prefill(plan, m.model_type, reqs, stop, 40, 96, 16)
        assert len(got[1]) == 4
        for i, (latest, start, prompt) in enumerate(reqs):
            plan.kv_reset()
            alone = E.generate_tokens_llama_batch_prefill(plan, latest, start, prompt, stop, 40, 96, 16)
            assert got[i] == alone, f"request {i}"
            if mode == "exact":
                om.reset()
                assert got[i] == E.generate_tokens_llama(om.forward_argmax, latest, start, prompt, stop, 40, 96), f"request {i} vs the oracle"
        with pytest.raises(ValueError, match="generate_tokens_batch"):
            E.generate_tokens_batch_prefill(plan, "QWEN_3", reqs, stop, 40, 96, 16)
    finally:
        plan.free()
        om.close()


def test_prefill_slots_refusals(pkg, make_model):
    N = pkg.native
    m = make_model("tiny-llama", pkg.gguf.GGMLType.Q8_0, 32)
    V = m.configuration.vocab_size
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=8)
    try:
        with pytest.raises(N.B200Error, match="no decode slots") as e:
            plan.prefill_slots([0], [0], [[1]])
        assert e.value.code == -6
        plan.set_decode_slots(3)
        bad = [
            ([], [], [], "n_seqs = 0"),
            ([0, 1, 2, 0], [0] * 4, [[1]] * 4, "n_seqs = 4"),
            ([0, 3], [0, 0], [[1], [1]], "sequence 1: slot 3 out of range"),
            ([0, -1], [0, 0], [[1], [1]], "sequence 1: slot -1 out of range"),
            ([2, 2], [0, 0], [[1], [1]], "sequence 1: slot 2 repeats sequence 0"),
            ([0, 1], [0, 30], [[1], [1, 2, 3]], "sequence 1: positions 30..32 outside"),
            ([0, 1], [-1, 0], [[1], [1]], "sequence 0: positions -1"),
            ([0, 1], [0, 0], [[1], [1, V]], "sequence 1: token"),
            ([0, 1], [0, 0], [[-1], [1]], "sequence 0: token -1"),
        ]
        for slots, starts, toks, msg in bad:
            with pytest.raises(N.B200Error, match=msg) as e:
                plan.prefill_slots(slots, starts, toks)
            assert e.value.code == -1, msg
        s = np.array([0, 1], dtype=np.int32)
        st = np.zeros(2, dtype=np.int32)
        ln = np.array([1, -1], dtype=np.int32)
        t = np.ones(1, dtype=np.int32)
        rc = N.lib().b200_prefill_slots(plan._native._p, 2, s.ctypes.data, st.ctypes.data, ln.ctypes.data, t.ctypes.data)
        assert rc == -1 and "sequence 1: length -1 is negative" in N.lib().b200_last_error(plan._native._p).decode()
        plan.prefill_slots([2, 0], [0, 0], [list(range(1, 8)), [1, 2, 3]])  # exact mode: no chunk limit
        for mode in ("tensor_core", "tensor_core_w8a16"):
            plan.set_prefill_mode(mode)
            with pytest.raises(N.B200Error, match="sequence 1: the call's 10 tokens exceed prefill_batch_size 8") as e:
                plan.prefill_slots([2, 0], [0, 0], [list(range(1, 8)), [1, 2, 3]])
            assert e.value.code == -1
            plan.prefill_slots([2, 0], [0, 0], [list(range(1, 6)), [1, 2, 3]])  # a valid call still works after the rejected ones
    finally:
        plan.free()
    phi = pkg.B200MasterPlan.initialize_plan(make_model("tiny-phi3", pkg.gguf.GGMLType.Q8_0, 32), prefill_batch_size=8)
    try:  # head size 96: the tensor-core modes are refused, the exact multi-slot prefill runs
        with pytest.raises(N.UnsupportedOperation):
            phi.set_prefill_mode("tensor_core_w8a16")
        phi.set_decode_slots(2)
        phi.prefill_slots([1, 0], [0, 0], [[1, 2, 3, 4, 5, 6, 7, 8, 9, 10], [4]])
        assert phi.prefill_info()[0] == 0
    finally:
        phi.free()
