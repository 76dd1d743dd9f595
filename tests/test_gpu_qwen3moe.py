"""GPU tests of Qwen3-MoE (B200_ARCH_QWEN3_MOE: Qwen3's attention, k_routed_route's renormalised top-k and the routed-only expert
streams k_routed_gateup / k_routed_down, csrc/moe.cuh) through the C ABI, against the CPU restatement (tests/qwen3moe_oracle.py).
Logits are compared as uint32; the routing buffers (selected ids and renormalised weights of every layer) and the KV cache bit for bit."""
import numpy as np
import pytest

from qwen3moe_oracle import Qwen3MoEOracle
from test_gpu_logprobs import test_every_emitting_call as _every_emitting_call
from test_gpu_parity import assert_bit_equal
from test_gpu_sampling_controls import _controls, _Host
from test_gpu_score import CHUNKS, _score_in_every_mode

pytestmark = pytest.mark.gpu


def _fast_model(pkg, shape_name, ctx, seed=1234, edit=None):
    sh = pkg.synth.SHAPES[shape_name]
    t = pkg.synth.build_tensors_fast(sh, pkg.gguf.GGMLType.Q8_0, seed=seed)
    if edit:
        edit(t)
    return pkg.loader.model_from_tensors(sh, pkg.gguf.GGMLType.Q8_0, t, ctx)


def _check_routing(plan, om, c, what):
    ids, w = plan.moe_routing()
    assert w.shape == (c.n_layers, c.n_experts_used), w.shape  # k weights per layer: no shared-expert weight
    for l in range(c.n_layers):
        rid, rw = om.routing[l]
        assert np.array_equal(ids[l], rid), f"{what}: layer {l} ids {ids[l]} != {rid}"
        assert_bit_equal(w[l], rw, f"{what}: layer {l} routing weights")
    return ids, w


def _check_kv(plan, om, c):
    nkv = c.context_length * c.kv_dim
    for l in range(c.n_layers):
        assert_bit_equal(plan.read_buffer("key_cache", nkv, layer=l), om.key_cache(l), f"key cache layer {l}")
        assert_bit_equal(plan.read_buffer("value_cache", nkv, layer=l), om.value_cache(l), f"value cache layer {l}")


def _decode_vs_oracle(pkg, orc, m, n, oracle_model=None, tok=1, toks=None):
    """n decode steps (greedy, or consuming toks[pos]): logits, argmax and the routing of every layer on every step, then the KV
    cache; returns the experts seen per layer."""
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = Qwen3MoEOracle(orc, oracle_model or m)
    c = m.configuration
    seen = [set() for _ in range(c.n_layers)]
    try:
        for pos in range(n):
            lg, am = plan.forward_decode(tok, pos)
            ref = om.forward(tok, pos)
            assert_bit_equal(lg, ref, f"logits pos {pos}")
            assert am == orc.argmax(ref), f"argmax pos {pos}"
            ids, _ = _check_routing(plan, om, c, f"pos {pos}")
            for l in range(c.n_layers):
                seen[l] |= set(int(e) for e in ids[l])
            tok = am if toks is None else int(toks[pos + 1]) if pos + 1 < n else am
        _check_kv(plan, om, c)
    finally:
        plan.free()
        om.close()
    return seen


@pytest.mark.parametrize("shape,n", [("tiny-qwen3moe", 48), ("tiny-qwen3moe-k8", 24), ("tiny-qwen3moe-tied", 32)])
def test_qwen3moe_decode_bit_exact(pkg, orc, make_model, shape, n):
    """GGUF written to disk, loaded through load_model: bit-exact logits, routing and KV cache."""
    m = make_model(shape, pkg.gguf.GGMLType.Q8_0, 64)
    assert m.model_type == "QWEN_3_MOE"
    toks = orc.bench_tokens(m.configuration.vocab_size, n)
    _decode_vs_oracle(pkg, orc, m, n, tok=int(toks[0]), toks=toks)


def test_qwen3moe_mid_30b_a3b_geometry_bit_exact(pkg, orc):
    """Qwen3-30B-A3B's layer geometry (dim 2048, 32 / 4 heads of 128, 128 experts, top-8, expert hidden 768; 2 layers, vocabulary
    151936)."""
    _decode_vs_oracle(pkg, orc, _fast_model(pkg, "mid-qwen3-30b-a3b", 16), 6)


def test_qwen3moe_mid_30b_a3b_every_expert_bit_exact(pkg, orc):
    """All 128 experts of the 30B-A3B geometry streamed: the embedding rows of tokens 0..127 are scaled up so they dominate the
    residual stream, and router row e of every layer is token e's (normalised, scaled) embedding row, so feeding tokens 0..127 puts
    expert e in the top-8 at step e.  Bit-exact on every step; every layer must select every expert."""
    sh = pkg.synth.SHAPES["mid-qwen3-30b-a3b"]
    E = sh.n_experts

    def align(t):
        tt, d, raw = t["token_embd.weight"]
        m0 = pkg.loader.model_from_tensors(sh, pkg.gguf.GGMLType.Q8_0, {"token_embd.weight": (tt, d, raw)}, 8)
        emb = pkg.loader.tensor_as_f32(m0, "token_embd.weight").reshape(sh.vocab, sh.dim).copy()
        emb[:E] *= np.float32(16.0)
        t["token_embd.weight"] = (tt, d, pkg.synth.encode(emb, tt))
        r = (emb[:E] / np.linalg.norm(emb[:E], axis=1, keepdims=True) * np.float32(4.0)).astype(np.float32)
        for l in range(sh.n_layers):
            rt, rd, _ = t[f"blk.{l}.ffn_gate_inp.weight"]
            t[f"blk.{l}.ffn_gate_inp.weight"] = (rt, rd, r.reshape(-1).view(np.uint8))
    m = _fast_model(pkg, "mid-qwen3-30b-a3b", E + 8, edit=align)
    seen = _decode_vs_oracle(pkg, orc, m, E, tok=0, toks=np.arange(E, dtype=np.int32))
    for l in range(sh.n_layers):
        assert seen[l] == set(range(E)), f"layer {l}: experts never selected: {sorted(set(range(E)) - seen[l])}"


def test_qwen3moe_kquant_decodes_like_its_q8_0_twin(pkg, orc):
    """A Q4_K_M file (Q4_K gate/up experts, Q6_K down experts; the router stays F32) against the oracle on its Q8_0 re-quantised twin."""
    G = pkg.gguf.GGMLType
    sh = pkg.synth.SHAPES["tiny-qwen3moe"]
    tensors = pkg.synth.build_tensors_kquant(sh, seed=21)
    assert tensors["blk.0.ffn_gate_exps.weight"][0] == G.Q4_K and tensors["blk.0.ffn_down_exps.weight"][0] == G.Q6_K
    twin = {n: ((G.Q8_0, d, orc.kquant_to_q8_0(t, np.asarray(r), int(np.prod(d)))) if t in G.K_QUANTS else (t, d, r)) for n, (t, d, r) in tensors.items()}
    m = pkg.loader.model_from_tensors(sh, G.Q8_0, tensors, 24)
    mt = pkg.loader.model_from_tensors(sh, G.Q8_0, twin, 24)
    _decode_vs_oracle(pkg, orc, m, 12, oracle_model=mt, tok=3)


def test_qwen3moe_exact_prefill_then_decode(pkg, orc, make_model):
    """600 positions through the exact batched prefill (the KV cache bit-equal to the oracle's), then greedy decode."""
    m = make_model("tiny-qwen3moe", pkg.gguf.GGMLType.Q8_0, 640)
    c = m.configuration
    n = 600
    toks = orc.bench_tokens(c.vocab_size, n)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=128)
    om = Qwen3MoEOracle(orc, m)
    try:
        assert plan.prefill_info()[0] == plan.PREFILL_EXACT
        for off in range(0, n, 128):
            plan.forward_batch_prefill(toks[off:off + 128], off)
        for pos in range(n):
            om.forward(int(toks[pos]), pos, want_logits=False)
        _check_kv(plan, om, c)
        tok = int(toks[-1])
        for pos in range(n, n + 8):
            lg, am = plan.forward_decode(tok, pos)
            assert_bit_equal(lg, om.forward(tok, pos), f"logits pos {pos}")
            _check_routing(plan, om, c, f"pos {pos}")
            tok = am
    finally:
        plan.free()
        om.close()


def test_qwen3moe_tied_router_rows_pick_the_lower_index(pkg, orc):
    """Router rows 1 and 5 are identical (their experts differ): their probabilities tie on every step, so wherever expert 5 is
    selected, expert 1 must be selected before it, and 1 is never passed over for 5."""
    sh = pkg.synth.SHAPES["tiny-qwen3moe"]

    def tie(t):
        for l in range(sh.n_layers):
            tt, d, raw = t[f"blk.{l}.ffn_gate_inp.weight"]
            r = np.asarray(raw).view(np.float32).reshape(sh.n_experts, sh.dim).copy()
            r[5] = r[1]
            t[f"blk.{l}.ffn_gate_inp.weight"] = (tt, d, r.view(np.uint8).reshape(-1))
    m = _fast_model(pkg, "tiny-qwen3moe", 48, edit=tie)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = Qwen3MoEOracle(orc, m)
    picked = 0
    try:
        tok = 1
        for pos in range(40):
            lg, am = plan.forward_decode(tok, pos)
            assert_bit_equal(lg, om.forward(tok, pos), f"logits pos {pos}")
            ids, _ = _check_routing(plan, om, m.configuration, f"pos {pos}")
            tok = am
            for l in range(sh.n_layers):
                row = [int(e) for e in ids[l]]
                if 5 in row:
                    assert 1 in row and row.index(1) < row.index(5), f"pos {pos} layer {l}: {row}"
                if 1 in row or 5 in row:
                    picked += 1
                    assert 1 in row, f"pos {pos} layer {l}: expert 5 chosen over its tied lower index 1: {row}"
        assert picked > 0, "the tied experts were never selected: the test saw nothing"
    finally:
        plan.free()
        om.close()


def test_qwen3moe_all_zero_router_picks_experts_0_to_7_at_one_eighth(pkg, orc):
    """All-zero router rows: every probability is 1/16, every scan keeps the lowest index, and the renormalised weights are exactly
    0.125 (top-8 of 16)."""
    sh = pkg.synth.SHAPES["tiny-qwen3moe-k8"]

    def zero(t):
        for l in range(sh.n_layers):
            tt, d, raw = t[f"blk.{l}.ffn_gate_inp.weight"]
            t[f"blk.{l}.ffn_gate_inp.weight"] = (tt, d, np.zeros_like(np.asarray(raw)))
    m = _fast_model(pkg, "tiny-qwen3moe-k8", 16, edit=zero)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = Qwen3MoEOracle(orc, m)
    try:
        tok = 2
        for pos in range(6):
            lg, am = plan.forward_decode(tok, pos)
            assert_bit_equal(lg, om.forward(tok, pos), f"logits pos {pos}")
            ids, w = _check_routing(plan, om, m.configuration, f"pos {pos}")
            assert np.array_equal(ids, np.tile(np.arange(8, dtype=np.int32), (sh.n_layers, 1))), ids
            assert np.all(w.view(np.uint32) == np.float32(0.125).view(np.uint32)), w
            tok = am
    finally:
        plan.free()
        om.close()


def test_qwen3moe_sampler_and_device_loop(pkg, orc, make_model):
    """forward_decode_sample against the oracle's sampler on the oracle's logits, and decode_sequence's greedy ids."""
    m = make_model("tiny-qwen3moe", pkg.gguf.GGMLType.Q8_0, 64)
    c = m.configuration
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = Qwen3MoEOracle(orc, m)
    try:
        toks = orc.bench_tokens(c.vocab_size, 24)
        ids, _ = plan.decode_sequence(toks, 24, 0)
        for pos in range(24):
            assert ids[pos] == orc.argmax(om.forward(int(toks[pos]), pos)), f"decode_sequence pos {pos}"
        plan.kv_reset()
        om.reset()
        ids, _ = plan.decode_sequence(np.array([7], dtype=np.int32), 16, 0, feedback=True)
        tok = 7
        for pos in range(16):
            tok = orc.argmax(om.forward(tok, pos))
            assert ids[pos] == tok, f"greedy loop pos {pos}"
        plan.kv_reset()
        om.reset()
        rng = np.random.default_rng(5)
        tok = 3
        for pos in range(12):
            u = float(rng.random())
            got = plan.forward_decode_sample(tok, pos, 0.8, 0.9, u)
            ref = orc.sample(om.forward(tok, pos), 0.8, 0.9, u)
            assert got == ref, f"sampled id pos {pos}"
            tok = got
    finally:
        plan.free()
        om.close()


def test_qwen3moe_scores_are_the_oracle(pkg, orc, make_model):
    """score_tokens in exact mode (the only prefill mode of an MoE plan) against the float64 log-softmax of the oracle's logits."""
    m = make_model("tiny-qwen3moe", pkg.gguf.GGMLType.Q8_0, ctx=96, seed=21)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=64)
    om = Qwen3MoEOracle(orc, m)
    try:
        assert set(_score_in_every_mode(pkg, plan, om, m.configuration, CHUNKS)) == {"exact"}
    finally:
        plan.free()
        om.close()


def test_qwen3moe_logprobs_on_every_emitting_call(pkg, make_model):
    """The logprobs table of every emitting call (single step, decode_sequence, sampled rows) against its float64 restatement and
    against score_tokens."""
    _every_emitting_call(pkg, make_model, "tiny-qwen3moe", pkg.gguf.GGMLType.Q8_0)


def test_qwen3moe_sampling_controls_on_slot_minus_one(pkg, orc, make_model):
    """Top-k, repetition / frequency penalties and a logit bias on slot -1: the device's choices and counts equal the host restatement
    of the controls applied to the oracle's logits."""
    m = make_model("tiny-qwen3moe", pkg.gguf.GGMLType.Q8_0, ctx=64, seed=24)
    V = m.configuration.vocab_size
    c = _controls(pkg, top_k=5, repetition_penalty=1.2, frequency_penalty=0.1, logit_bias={4: 1.0})
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = Qwen3MoEOracle(orc, m)
    try:
        for temp, topp in ((0.0, 0.0), (0.9, 0.9)):
            smp = pkg.sampler.Sampler(V, temp, topp, 9, controls=c, history=[4, 4])
            plan.kv_reset()
            toks = [2]
            for p in range(8):
                toks.append(smp.sample_token(plan, toks[-1], p))
            host = _Host(pkg, orc, V, c, temp, topp, 9, [4, 4])
            om.reset()
            want = [2]
            for p in range(8):
                want.append(host.choose(om.forward(want[-1], p)))
            assert toks == want, temp
            assert np.array_equal(plan.sample_counts(-1), host.counts), temp
    finally:
        plan.free()
        om.close()


def test_qwen3moe_engine_generation_loop(pkg, orc, make_model):
    """engine.loop_for picks the Qwen3 loop for Qwen3-MoE; driven by the plan it produces the tokens the same loop produces when driven
    by the oracle."""
    m = make_model("tiny-qwen3moe", pkg.gguf.GGMLType.Q8_0, 64)
    c = m.configuration
    loop = pkg.engine.loop_for(m.model_type)
    assert loop is pkg.engine.generate_tokens_qwen3
    prompt = [int(t) for t in orc.bench_tokens(c.vocab_size, 6)]
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = Qwen3MoEOracle(orc, m)
    try:
        got = loop(lambda tok, pos: plan.forward_decode(tok, pos, logits=False)[1], 0, 0, prompt, [], 20, c.context_length)
        want = loop(lambda tok, pos: orc.argmax(om.forward(tok, pos)), 0, 0, prompt, [], 20, c.context_length)
        assert got == want and len(got) > 0
    finally:
        plan.free()
        om.close()


def _expect(pkg, fn, code, needle):
    with pytest.raises(pkg.native.B200Error) as ei:
        fn()
    assert ei.value.code == code, str(ei.value)
    assert needle in str(ei.value), str(ei.value)
    assert "Qwen2-MoE" not in str(ei.value), str(ei.value)


def test_qwen3moe_refusals_name_qwen3moe(pkg, orc, make_model):
    N = pkg.native
    G = pkg.gguf.GGMLType
    sh = pkg.synth.SHAPES["tiny-qwen3moe"]
    m = make_model("tiny-qwen3moe", G.Q8_0, 64)
    c = m.configuration
    moe = N.MoeConfig(c.n_experts, c.n_experts_used, c.expert_hidden_dim, 0)

    def create(cfg=None, moe_cfg=moe, tensors=None):
        return N.NativePlan(cfg or pkg.plan.make_config(m), tensors or m.tensors, 0, 0, moe=moe_cfg)

    _expect(pkg, lambda: create(moe_cfg=None), -1, "B200_ARCH_QWEN3_MOE")
    _expect(pkg, lambda: create(moe_cfg=N.MoeConfig(c.n_experts, c.n_experts_used, c.expert_hidden_dim, 256)), -1, "Qwen3-MoE has no shared expert")
    for k in (0, 9):
        _expect(pkg, lambda: create(moe_cfg=N.MoeConfig(c.n_experts, k, c.expert_hidden_dim, 0)), -1, "n_experts_used")
    cfg = pkg.plan.make_config(m)
    cfg.tp_size = 2
    _expect(pkg, lambda: create(cfg=cfg), -2, "Qwen3-MoE plans are single-GPU")
    t = dict(m.tensors)
    del t["blk.1.ffn_down_exps.weight"]
    _expect(pkg, lambda: create(tensors=t), -1, "blk.1.ffn_down_exps.weight")
    mf = pkg.loader.model_from_tensors(sh, G.F16, pkg.synth.build_tensors_fast(sh, G.F16), 64)
    _expect(pkg, lambda: N.NativePlan(pkg.plan.make_config(mf), mf.tensors, 0, 0, moe=moe), -2, "Qwen3-MoE runs in Q8_0 only")
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=64)
    om = Qwen3MoEOracle(orc, m)
    try:
        assert plan.launches_per_decode == c.n_layers * 8 + 3
        for mode in ("tensor_core", "tensor_core_w8a16", "tensor_core_exact"):
            _expect(pkg, lambda: plan.set_prefill_mode(mode), -2, "Qwen3-MoE plans have no tensor-core prefill")
        plan.set_prefill_mode("exact")
        _expect(pkg, lambda: plan.set_decode_mode("persistent"), -2, "persistent decode kernel has no Qwen3-MoE layer")
        assert plan.decode_info()[0] == plan.DECODE_GRAPH
        _expect(pkg, lambda: plan.set_decode_slots(2), -2, "batched decode has no Qwen3-MoE layer")
        plan.set_decode_slots(0)
        assert plan.decode_multi_rows() == 0
        _expect(pkg, lambda: plan.forward_decode_multi(-1, np.array([1, 2], np.int32), 0), -2, "multi-position steps have no Qwen3-MoE layer")
        _expect(pkg, lambda: plan.time_kernel(0), -2, "a Qwen3-MoE plan has no dense FFN")
        tok = 1
        for pos in range(4):  # the plan still decodes bit-exactly after every refusal
            lg, am = plan.forward_decode(tok, pos)
            assert_bit_equal(lg, om.forward(tok, pos), f"logits pos {pos} after the refusals")
            _check_routing(plan, om, c, f"pos {pos} after the refusals")
            tok = am
    finally:
        plan.free()
        om.close()
