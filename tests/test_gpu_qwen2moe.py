"""GPU tests of Qwen2-MoE (B200_ARCH_QWEN2_MOE: the router, the shared + routed gate/up stream and the down streams with the ordered
combine, csrc/moe.cuh) through the C ABI, against the CPU restatement of forwardJavaQwen2MoE (tests/qwen2moe_oracle.py).  Logits are
compared as uint32; the routing buffers (selected ids and weights of every layer) bit for bit on every step."""
import os

import numpy as np
import pytest

from qwen2moe_oracle import Qwen2MoEOracle
from test_gpu_parity import assert_bit_equal

pytestmark = pytest.mark.gpu


def _fast_model(pkg, shape_name, ctx, seed=1234, edit=None):
    sh = pkg.synth.SHAPES[shape_name]
    t = pkg.synth.build_tensors_fast(sh, pkg.gguf.GGMLType.Q8_0, seed=seed)
    if edit:
        edit(t)
    return pkg.loader.model_from_tensors(sh, pkg.gguf.GGMLType.Q8_0, t, ctx)


def _check_routing(plan, om, c, what):
    ids, w = plan.moe_routing()
    for l in range(c.n_layers):
        rid, rw, rsw = om.routing[l]
        assert np.array_equal(ids[l], rid), f"{what}: layer {l} ids {ids[l]} != {rid}"
        assert_bit_equal(w[l, :-1], rw, f"{what}: layer {l} routing weights")
        assert_bit_equal(w[l, -1:], np.array([rsw], dtype=np.float32), f"{what}: layer {l} shared-expert weight")
    return ids


def _decode_vs_oracle(pkg, orc, m, n, oracle_model=None, tok=1, toks=None):
    """n decode steps (greedy, or consuming toks[pos]): logits, argmax and the routing of every layer on every step; returns the
    experts seen per layer."""
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = Qwen2MoEOracle(orc, oracle_model or m)
    c = m.configuration
    seen = [set() for _ in range(c.n_layers)]
    try:
        for pos in range(n):
            lg, am = plan.forward_decode(tok, pos)
            ref = om.forward(tok, pos)
            assert_bit_equal(lg, ref, f"logits pos {pos}")
            assert am == orc.argmax(ref), f"argmax pos {pos}"
            ids = _check_routing(plan, om, c, f"pos {pos}")
            for l in range(c.n_layers):
                seen[l] |= set(int(e) for e in ids[l])
            tok = am if toks is None else int(toks[pos + 1]) if pos + 1 < n else am
        nkv = c.context_length * c.kv_dim
        for l in range(c.n_layers):
            assert_bit_equal(plan.read_buffer("key_cache", nkv, layer=l), om.key_cache(l), f"key cache layer {l}")
            assert_bit_equal(plan.read_buffer("value_cache", nkv, layer=l), om.value_cache(l), f"value cache layer {l}")
    finally:
        plan.free()
        om.close()
    return seen


def _assert_every_expert(seen, E, layers):
    for l in layers:  # the stream-base tables are per layer: every layer must use every expert
        assert seen[l] == set(range(E)), f"layer {l}: experts never selected: {sorted(set(range(E)) - seen[l])}"


@pytest.mark.parametrize("shape,n", [("tiny-qwen2moe", 64), ("tiny-qwen2moe-gqa", 24)])
def test_qwen2moe_decode_bit_exact(pkg, orc, make_model, shape, n):
    """GGUF written to disk, loaded through load_model: bit-exact logits and routing, and every expert selected at least once in
    every layer."""
    m = make_model(shape, pkg.gguf.GGMLType.Q8_0, 64)
    assert m.model_type == "QWEN_2_MOE"
    toks = orc.bench_tokens(m.configuration.vocab_size, n)
    seen = _decode_vs_oracle(pkg, orc, m, n, tok=int(toks[0]), toks=toks)
    _assert_every_expert(seen, m.configuration.n_experts, range(m.configuration.n_layers))


def test_qwen2moe_mid_a27b_geometry_bit_exact(pkg, orc):
    """Qwen1.5-MoE-A2.7B's layer geometry (60 experts, top-4, expert hidden 1408, shared hidden 5632; 2 layers, vocabulary 8192)."""
    _decode_vs_oracle(pkg, orc, _fast_model(pkg, "mid-qwen1.5-moe-a2.7b", 16), 6)


def test_qwen2moe_mid_a27b_every_expert_bit_exact(pkg, orc):
    """All 60 experts of the A2.7B geometry streamed: the embedding rows of tokens 0..59 are scaled up so they dominate the residual
    stream, and router row e of every layer is token e's (normalised, scaled) embedding row, so feeding tokens 0..59 puts expert e in
    the top-4 at step e.  Bit-exact on every step; every layer must select every expert."""
    sh = pkg.synth.SHAPES["mid-qwen1.5-moe-a2.7b"]
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
    m = _fast_model(pkg, "mid-qwen1.5-moe-a2.7b", 64, edit=align)
    toks = np.arange(E, dtype=np.int32)
    seen = _decode_vs_oracle(pkg, orc, m, E, tok=0, toks=toks)
    _assert_every_expert(seen, E, range(sh.n_layers))


def test_qwen2moe_kquant_decodes_like_its_q8_0_twin(pkg, orc):
    """A K-quant file (Q4_K_M mix; router and shared gate stay F32) against the oracle on its Q8_0 re-quantised twin."""
    G = pkg.gguf.GGMLType
    sh = pkg.synth.SHAPES["tiny-qwen2moe"]
    tensors = pkg.synth.build_tensors_kquant(sh, seed=21)
    twin = {n: ((G.Q8_0, d, orc.kquant_to_q8_0(t, np.asarray(r), int(np.prod(d)))) if t in G.K_QUANTS else (t, d, r)) for n, (t, d, r) in tensors.items()}
    m = pkg.loader.model_from_tensors(sh, G.Q8_0, tensors, 24)
    mt = pkg.loader.model_from_tensors(sh, G.Q8_0, twin, 24)
    _decode_vs_oracle(pkg, orc, m, 12, oracle_model=mt, tok=3)


def test_qwen2moe_exact_prefill_then_decode(pkg, orc, make_model):
    """600 positions through the exact batched prefill (the KV cache bit-equal to the oracle's), then greedy decode."""
    m = make_model("tiny-qwen2moe", pkg.gguf.GGMLType.Q8_0, 640)
    c = m.configuration
    n = 600
    toks = orc.bench_tokens(c.vocab_size, n)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=128)
    om = Qwen2MoEOracle(orc, m)
    try:
        assert plan.prefill_info()[0] == plan.PREFILL_EXACT
        for off in range(0, n, 128):
            plan.forward_batch_prefill(toks[off:off + 128], off)
        for pos in range(n):
            om.forward(int(toks[pos]), pos, want_logits=False)
        nkv = c.context_length * c.kv_dim
        for l in range(c.n_layers):
            assert_bit_equal(plan.read_buffer("key_cache", nkv, layer=l), om.key_cache(l), f"key cache layer {l}")
            assert_bit_equal(plan.read_buffer("value_cache", nkv, layer=l), om.value_cache(l), f"value cache layer {l}")
        tok = int(toks[-1])
        for pos in range(n, n + 8):
            lg, am = plan.forward_decode(tok, pos)
            ref = om.forward(tok, pos)
            assert_bit_equal(lg, ref, f"logits pos {pos}")
            _check_routing(plan, om, c, f"pos {pos}")
            tok = am
    finally:
        plan.free()
        om.close()


def test_qwen2moe_tied_router_rows_pick_the_lower_index(pkg, orc):
    """Router rows 1 and 5 are identical (their experts differ): their probabilities tie on every step, so wherever expert 5 is
    selected, expert 1 must be selected before it, and 1 is never passed over for 5."""
    sh = pkg.synth.SHAPES["tiny-qwen2moe"]

    def tie(t):
        for l in range(sh.n_layers):
            tt, d, raw = t[f"blk.{l}.ffn_gate_inp.weight"]
            r = np.asarray(raw).view(np.float32).reshape(sh.n_experts, sh.dim).copy()
            r[5] = r[1]
            t[f"blk.{l}.ffn_gate_inp.weight"] = (tt, d, r.view(np.uint8).reshape(-1))
    m = _fast_model(pkg, "tiny-qwen2moe", 48, edit=tie)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = Qwen2MoEOracle(orc, m)
    picked = 0
    try:
        tok = 1
        for pos in range(40):
            lg, am = plan.forward_decode(tok, pos)
            assert_bit_equal(lg, om.forward(tok, pos), f"logits pos {pos}")
            ids = _check_routing(plan, om, m.configuration, f"pos {pos}")
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


def test_qwen2moe_sampler_and_device_loop(pkg, orc, make_model):
    """forward_decode_sample against the oracle's sampler on the oracle's logits, and decode_sequence's greedy ids."""
    m = make_model("tiny-qwen2moe", pkg.gguf.GGMLType.Q8_0, 64)
    c = m.configuration
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = Qwen2MoEOracle(orc, m)
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


def _expect(pkg, fn, code, needle):
    with pytest.raises(pkg.native.B200Error) as ei:
        fn()
    assert ei.value.code == code, str(ei.value)
    assert needle in str(ei.value), str(ei.value)


def test_qwen2moe_refusals(pkg, orc, make_model):
    N = pkg.native
    G = pkg.gguf.GGMLType
    sh = pkg.synth.SHAPES["tiny-qwen2moe"]
    m = make_model("tiny-qwen2moe", G.Q8_0, 64)
    c = m.configuration
    moe = N.MoeConfig(c.n_experts, c.n_experts_used, c.expert_hidden_dim, c.shared_hidden_dim)

    def create(cfg=None, moe_cfg=moe, tensors=None):
        return N.NativePlan(cfg or pkg.plan.make_config(m), tensors or m.tensors, 0, 0, moe=moe_cfg)

    # b200_plan_create with the MoE arch names the MoE entry point
    _expect(pkg, lambda: create(moe_cfg=None), -1, "b200_plan_create_moe")
    # k outside 1..min(E, 8)
    for k in (0, 9):
        _expect(pkg, lambda: create(moe_cfg=N.MoeConfig(c.n_experts, k, c.expert_hidden_dim, c.shared_hidden_dim)), -1, "n_experts_used")
    # tensor parallelism
    cfg = pkg.plan.make_config(m)
    cfg.tp_size = 2
    _expect(pkg, lambda: create(cfg=cfg), -2, "single-GPU")
    # a missing tensor, a router that is not F32, wrong dims
    t = dict(m.tensors)
    del t["blk.1.ffn_down_exps.weight"]
    _expect(pkg, lambda: create(tensors=t), -1, "blk.1.ffn_down_exps.weight")
    t = dict(m.tensors)
    tt, d, raw = t["blk.0.ffn_gate_inp.weight"]
    t["blk.0.ffn_gate_inp.weight"] = (G.F16, d, np.asarray(raw).view(np.float32).astype(np.float16).view(np.uint8))
    _expect(pkg, lambda: create(tensors=t), -2, "must be F32")
    _expect(pkg, lambda: create(moe_cfg=N.MoeConfig(c.n_experts, c.n_experts_used, c.expert_hidden_dim, 2 * c.shared_hidden_dim)), -1,
            "ffn_gate_shexp.weight")
    # n_experts outside 1..256, hidden sizes the Q8_0 stream cannot cut
    for e in (0, 257):
        _expect(pkg, lambda: create(moe_cfg=N.MoeConfig(e, 1, c.expert_hidden_dim, c.shared_hidden_dim)), -1, "n_experts")
    _expect(pkg, lambda: create(moe_cfg=N.MoeConfig(c.n_experts, c.n_experts_used, c.expert_hidden_dim + 16, c.shared_hidden_dim)), -2,
            "multiples of 32")
    # FP16 weights
    mf = pkg.loader.model_from_tensors(sh, G.F16, pkg.synth.build_tensors_fast(sh, G.F16), 64)
    _expect(pkg, lambda: N.NativePlan(pkg.plan.make_config(mf), mf.tensors, 0, 0, moe=moe), -2, "Q8_0 only")
    # on a working plan: tensor-core prefill, persistent decode, decode slots, the kernel timer
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=64)
    try:
        for mode in ("tensor_core", "tensor_core_w8a16"):
            _expect(pkg, lambda: plan.set_prefill_mode(mode), -2, "exact token-by-token prefill")
        plan.set_prefill_mode("exact")
        _expect(pkg, lambda: plan.set_decode_mode("persistent"), -2, "persistent decode kernel has no Qwen2-MoE layer")
        assert plan.decode_info()[0] == 0
        _expect(pkg, lambda: plan.set_decode_slots(2), -2, "batched decode has no Qwen2-MoE layer")
        plan.set_decode_slots(0)
        _expect(pkg, lambda: plan.time_kernel(0), -2, "no dense FFN")
        lg, _ = plan.forward_decode(1, 0)  # the plan still decodes after every refusal
        assert np.isfinite(lg).all()
    finally:
        plan.free()


def test_qwen2moe_persistent_env_falls_back_to_the_graph(pkg, make_model):
    m = make_model("tiny-qwen2moe", pkg.gguf.GGMLType.Q8_0, 64)
    os.environ["B200_DECODE"] = "persistent"
    try:
        plan = pkg.B200MasterPlan.initialize_plan(m)
    finally:
        del os.environ["B200_DECODE"]
    try:
        assert plan.decode_info()[0] == plan.DECODE_GRAPH
        assert plan.launches_per_decode == m.configuration.n_layers * 8 + 3
    finally:
        plan.free()


def test_qwen2moe_engine_generation_loop(pkg, orc, make_model):
    """engine.loop_for picks the Qwen3 loop for Qwen2-MoE (skipped position after the prompt); driven by the plan it produces the
    tokens the same loop produces when driven by the oracle."""
    m = make_model("tiny-qwen2moe", pkg.gguf.GGMLType.Q8_0, 64)
    c = m.configuration
    loop = pkg.engine.loop_for(m.model_type)
    assert loop is pkg.engine.generate_tokens_qwen3
    prompt = [int(t) for t in orc.bench_tokens(c.vocab_size, 6)]
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = Qwen2MoEOracle(orc, m)
    try:
        got = loop(lambda tok, pos: plan.forward_decode(tok, pos, logits=False)[1], 0, 0, prompt, [], 20, c.context_length)
        want = loop(lambda tok, pos: orc.argmax(om.forward(tok, pos)), 0, 0, prompt, [], 20, c.context_length)
        assert got == want and len(got) > 0
    finally:
        plan.free()
        om.close()
