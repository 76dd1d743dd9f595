"""GPU tests of the batched decode (b200_forward_decode_batch, csrc/decode_batch.cuh): several sequences per step, each on its own KV
slot, every row held bit-exact (logits compared as uint32, equal ids) to the CPU restatement of its own sequence -- the C oracle's
OracleModel, tests/qwen2_oracle.py for Qwen2, the re-quantised Q8_0 twin for a K-quant file."""
import numpy as np
import pytest

from qwen2_oracle import Qwen2Oracle
from test_gpu_parity import assert_bit_equal

pytestmark = pytest.mark.gpu


def _oracle(pkg, orc, m):
    if m.configuration.arch == 3:
        return Qwen2Oracle(orc, m)
    G = pkg.gguf.GGMLType
    if any(t in G.K_QUANTS for t, _, _ in m.tensors.values()):  # the Q8_0 model the reference holds after loading a K-quant file
        twin = {n: ((G.Q8_0, d, orc.kquant_to_q8_0(t, np.asarray(r), int(np.prod(d)))) if t in G.K_QUANTS else (t, d, r)) for n, (t, d, r) in m.tensors.items()}
        m = pkg.loader.Model(None, m.configuration, m.model_type, twin)
    return orc.OracleModel(m)


def _model(pkg, make_model, shape, ctx):
    if shape == "tiny-llama-q4_k_m":
        sh = pkg.synth.SHAPES["tiny-llama"]
        return pkg.loader.model_from_tensors(sh, pkg.gguf.GGMLType.Q8_0, pkg.synth.build_tensors_kquant(sh, seed=11), ctx)
    if shape.startswith("mid-"):
        sh = pkg.synth.SHAPES[shape]
        return pkg.loader.model_from_tensors(sh, pkg.gguf.GGMLType.Q8_0, pkg.synth.build_tensors_fast(sh, pkg.gguf.GGMLType.Q8_0, seed=7), ctx)
    return make_model(shape, pkg.gguf.GGMLType.Q8_0, ctx)


def _run_schedule(pkg, orc, m, n_slots, schedule, starts, n_check_kv=True):
    """schedule: list of steps, each the slots of its rows in call order.  starts[s]: first position of slot s; positions below it
    enter the slot through the exact batched prefill into the plan's cache + slot_copy_kv.  Every row of every step is checked
    against that slot's sequence alone on the CPU; afterwards each slot's K/V cache too."""
    c = m.configuration
    plan = pkg.B200MasterPlan.initialize_plan(m)
    streams = [orc.bench_tokens(c.vocab_size, c.context_length, seed=100 + s) for s in range(n_slots)]
    rec = [[] for _ in range(n_slots)]  # (token, position, logits, id) per slot
    om = _oracle(pkg, orc, m)
    try:
        plan.set_decode_slots(n_slots)
        nkv = c.context_length * c.kv_dim
        for s in range(n_slots):
            if starts[s]:
                plan.kv_reset()
                plan.forward_batch_prefill(streams[s][: starts[s]], 0)
                plan.slot_copy_kv(s, starts[s])
        own_k = plan.read_buffer("key_cache", nkv, layer=0)
        nxt = list(starts)
        for rows in schedule:
            toks = [int(streams[s][nxt[s]]) for s in rows]
            ids, lg = plan.forward_decode_batch(rows, toks, [nxt[s] for s in rows], logits=True)
            for i, s in enumerate(rows):
                rec[s].append((toks[i], nxt[s], lg[i], int(ids[i])))
                nxt[s] += 1
        assert plan.batch_info()[0] == n_slots
        assert_bit_equal(plan.read_buffer("key_cache", nkv, layer=0), own_k, "the plan's own cache after batched steps")
        for s in range(n_slots):
            om.reset()
            for p in range(starts[s]):
                om.forward(int(streams[s][p]), p, want_logits=False)
            for tok, pos, lg, am in rec[s]:
                ref = om.forward(tok, pos)
                assert_bit_equal(lg, ref, f"slot {s} logits pos {pos}")
                assert am == orc.argmax(ref), f"slot {s} id pos {pos}"
            if n_check_kv:
                for l in range(c.n_layers):
                    assert_bit_equal(plan.read_buffer("slot_key_cache", nkv, layer=s * c.n_layers + l), om.key_cache(l), f"slot {s} key cache layer {l}")
                    assert_bit_equal(plan.read_buffer("slot_value_cache", nkv, layer=s * c.n_layers + l), om.value_cache(l), f"slot {s} value cache layer {l}")
    finally:
        plan.free()
        om.close()


# n changes between steps; slots out of order and with gaps; n = 1 and n = n_slots
SCHEDULE = [[0, 1, 2, 3], [3, 1], [2, 0, 3], [1], [0, 2], [3, 2, 1, 0], [1, 3], [0, 1, 2, 3], [2], [3, 0, 1, 2]]


@pytest.mark.parametrize("shape", ["tiny-llama", "tiny-qwen3", "tiny-phi3", "tiny-phi3-gqa", "tiny-qwen2", "tiny-llama-q4_k_m"])
def test_batch_decode_bit_exact(pkg, orc, make_model, shape):
    """Four slots, one of them starting ~600 positions deep (its prompt enters through the exact prefill + slot_copy_kv)."""
    m = _model(pkg, make_model, shape, 640)
    _run_schedule(pkg, orc, m, 4, SCHEDULE, [0, 5, 0, 600])


@pytest.mark.parametrize("shape", ["mid-llama", "mid-qwen3-4b", "mid-qwen2.5-7b"])
def test_batch_decode_8_rows_mid_geometries(pkg, orc, make_model, shape):
    """8 rows per step at the Llama-3-8B, Qwen3-4B and Qwen2.5-7B layer geometries (2 layers): the shapes that stress shared memory."""
    m = _model(pkg, make_model, shape, 16)
    _run_schedule(pkg, orc, m, 8, [list(range(8))] * 3, [0] * 8, n_check_kv=False)


@pytest.mark.parametrize("mode", ["graph", "persistent"])
def test_batch_isolation_and_interleaving(pkg, orc, make_model, mode):
    """A step on slots {0, 2} leaves slot 1's K/V bytes alone; single-sequence decode interleaved with batched steps stays exact on
    both sides, in both decode modes."""
    m = make_model("tiny-llama", pkg.gguf.GGMLType.Q8_0, 64)
    c = m.configuration
    nkv = c.context_length * c.kv_dim
    plan = pkg.B200MasterPlan.initialize_plan(m)
    plan.set_decode_mode(mode)
    single, batched = orc.OracleModel(m), [orc.OracleModel(m) for _ in range(3)]
    stream = orc.bench_tokens(c.vocab_size, 40, seed=3)
    try:
        plan.set_decode_slots(3)
        ids, _ = plan.forward_decode_batch([1], [5], [0])
        batched[1].forward(5, 0)
        k1 = [plan.read_buffer(n, nkv, layer=1 * c.n_layers + l) for n in ("slot_key_cache", "slot_value_cache") for l in range(c.n_layers)]
        for pos in range(12):
            lg, am = plan.forward_decode(int(stream[pos]), pos)
            ref = single.forward(int(stream[pos]), pos)
            assert_bit_equal(lg, ref, f"single-sequence logits pos {pos}")
            assert am == orc.argmax(ref)
            toks = [int(stream[pos + 20]), int(stream[pos + 10])]
            ids, blg = plan.forward_decode_batch([2, 0], toks, [pos, pos], logits=True)
            for i, s in enumerate([2, 0]):
                r = batched[s].forward(toks[i], pos)
                assert_bit_equal(blg[i], r, f"slot {s} logits pos {pos}")
                assert ids[i] == orc.argmax(r)
        k1b = [plan.read_buffer(n, nkv, layer=1 * c.n_layers + l) for n in ("slot_key_cache", "slot_value_cache") for l in range(c.n_layers)]
        for a, b in zip(k1, k1b):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), "slot 1 changed"
        for l in range(c.n_layers):
            assert_bit_equal(plan.read_buffer("key_cache", nkv, layer=l), single.key_cache(l), f"plan cache layer {l}")
    finally:
        plan.free()
        for o in [single, *batched]:
            o.close()


def test_slot_reuse_zeroes_the_tail_qwen3(pkg, orc, make_model):
    """A slot that held a 30-position sequence takes a second Qwen3 sequence through prefill + slot_copy_kv; the Qwen3 loop then
    skips position 5 and reads that row, which must be zero as in a fresh State."""
    m = make_model("tiny-qwen3", pkg.gguf.GGMLType.Q8_0, 64)
    c = m.configuration
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = orc.OracleModel(m)
    stream = orc.bench_tokens(c.vocab_size, 64, seed=9)
    try:
        plan.set_decode_slots(2)
        for pos in range(30):
            plan.forward_decode_batch([1, 0], [int(stream[pos]), int(stream[pos + 1])], [pos, pos])
        plan.kv_reset()
        plan.forward_batch_prefill(stream[40:45], 0)
        plan.slot_copy_kv(1, 5)
        for pos in range(5):
            om.forward(int(stream[40 + pos]), pos, want_logits=False)
        for pos in (6, 7, 8):
            ids, lg = plan.forward_decode_batch([1], [int(stream[50 + pos])], [pos], logits=True)
            ref = om.forward(int(stream[50 + pos]), pos)
            assert_bit_equal(lg[0], ref, f"reused slot logits pos {pos}")
            assert ids[0] == orc.argmax(ref)
    finally:
        plan.free()
        om.close()


@pytest.mark.parametrize("shape", ["tiny-llama", "tiny-llama-vocab128k"])
def test_batch_sampling_rows(pkg, orc, make_model, shape):
    """Greedy and sampled rows in one step: each sampled id is the oracle sampler's on the oracle logits with the same uniform number."""
    m = make_model(shape, pkg.gguf.GGMLType.Q8_0, 24)
    c = m.configuration
    plan = pkg.B200MasterPlan.initialize_plan(m)
    oms = [orc.OracleModel(m) for _ in range(4)]
    settings = [(0.0, 0.0, 0.0), (0.7, 0.9, 0.31), (1.0, 0.0, 0.77), (0.6, 0.95, 0.05)]
    try:
        plan.set_decode_slots(4)
        toks = [1, 2, 3, 4]
        for pos in range(6):
            ids, lg = plan.forward_decode_batch([0, 1, 2, 3], toks, [pos] * 4, sampling=settings, logits=True)
            for s in range(4):
                ref = oms[s].forward(toks[s], pos)
                assert_bit_equal(lg[s], ref, f"row {s} logits pos {pos}")
                t, p, u = settings[s]
                want = orc.argmax(ref) if t == 0.0 else orc.sample(ref, t, p, u)
                assert ids[s] == want, f"row {s} pos {pos}"
            toks = [int(i) for i in ids]
    finally:
        plan.free()
        for o in oms:
            o.close()


def test_batch_errors(pkg, make_model):
    N = pkg.native
    m = make_model("tiny-llama", pkg.gguf.GGMLType.Q8_0, 32)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    try:
        with pytest.raises(N.B200Error) as e:
            plan.forward_decode_batch([0], [1], [0])
        assert e.value.code == -6
        with pytest.raises(N.UnsupportedOperation, match="at most 8"):
            plan.set_decode_slots(9)
        plan.set_decode_slots(3)
        V = m.configuration.vocab_size
        bad = [([], [], []), ([0, 1, 2, 0], [1] * 4, [0] * 4), ([0, 0], [1, 1], [0, 0]), ([0, 3], [1, 1], [0, 0]), ([0, -1], [1, 1], [0, 0]),
               ([0, 1], [1, 1], [0, 32]), ([0, 1], [1, 1], [-1, 0]), ([0, 1], [1, V], [0, 0]), ([0, 1], [-1, 1], [0, 0])]
        for slots, toks, pos in bad:
            with pytest.raises(N.B200Error) as e:
                plan.forward_decode_batch(slots, toks, pos)
            assert e.value.code == -1, (slots, toks, pos)
        for smp in ([(0, 0, 0), (-1.0, 0.9, 0.5)], [(0, 0, 0), (0.7, 0.9, 1.0)], [(float("nan"), 0.9, 0.5), (0, 0, 0)], [(0.7, 0.9, -0.1), (0, 0, 0)]):
            with pytest.raises(N.B200Error, match="row") as e:
                plan.forward_decode_batch([0, 1], [1, 1], [0, 0], sampling=smp)
            assert e.value.code == -1
        with pytest.raises(N.B200Error) as e:
            plan.slot_copy_kv(3, 1)
        assert e.value.code == -1
        ids, _ = plan.forward_decode_batch([2, 0], [1, 1], [0, 0])  # a valid call still works after the rejected ones
        assert len(ids) == 2
        plan.set_decode_slots(0)
        with pytest.raises(N.B200Error) as e:
            plan.forward_decode_batch([0], [1], [0])
        assert e.value.code == -6
    finally:
        plan.free()
    f16 = pkg.B200MasterPlan.initialize_plan(make_model("tiny-llama", pkg.gguf.GGMLType.F16, 32))
    try:
        with pytest.raises(N.UnsupportedOperation, match="FP16"):
            f16.set_decode_slots(2)
    finally:
        f16.free()


@pytest.mark.parametrize("shape", ["tiny-llama", "tiny-qwen3"])
def test_generate_tokens_batch_on_device(pkg, orc, make_model, shape):
    m = make_model(shape, pkg.gguf.GGMLType.Q8_0, 64)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = orc.OracleModel(m)
    loop = pkg.engine.loop_for(m.model_type)
    reqs = [(7, 0, [7, 11, 12]), (3, 0, [3, 40, 41, 42, 43, 44, 45]), (5, 0, [5, 9]), (8, 0, [8, 2, 2, 2, 2])]
    try:
        plan.set_decode_slots(4)
        for stop, budget in (([], 14), (None, 40)):
            if stop is None:  # a stop token that ends one request early: the 4th id the first run produced for request 1
                stop = [first[1][3]]
            got = pkg.engine.generate_tokens_batch(plan, m.model_type, reqs, stop, budget, 64)
            for i, (latest, start, prompt) in enumerate(reqs):
                om.reset()
                assert got[i] == loop(om.forward_argmax, latest, start, prompt, stop, budget, 64), f"request {i}, stop {stop}"
            first = got
    finally:
        plan.free()
        om.close()
