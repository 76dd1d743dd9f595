"""GPU tests of the MoE tensor-core prefill (B200_PREFILL_TENSOR_CORE_EXACT_MOE: the chunk router k_xp_route, the grouping
k_xp_group / k_xp_gather, the grouped int8 expert GEMMs k_xp_gemm and the ordered combine k_xp_combine, csrc/moe.cuh and
csrc/prefill_i8.cuh).  Every comparison is bitwise: the KV cache and every row's chunk routing against the CPU oracles
(tests/qwen2moe_oracle.py, tests/qwen3moe_oracle.py), scores against exact mode on the same plan, the grouped GEMM against the
float32 restatement test_gpu_prefill_i8.py holds the int8 GEMM to."""
import numpy as np
import pytest

import test_gpu_score
from qwen2moe_oracle import Qwen2MoEOracle
from qwen3moe_oracle import Qwen3MoEOracle
from test_gpu_parity import assert_bit_equal
from test_gpu_prefill_i8 import _activations, _dot_q8, _swiglu_q8, _weights
from test_score_host import score_rows

pytestmark = pytest.mark.gpu

MOE = "tensor_core_exact_moe"
SHAPES = ["tiny-qwen2moe", "tiny-qwen2moe-gqa", "tiny-qwen3moe", "tiny-qwen3moe-k8", "tiny-qwen3moe-tied"]


def _oracle(orc, m):
    return (Qwen2MoEOracle if m.configuration.shared_hidden_dim else Qwen3MoEOracle)(orc, m)


def _fast_model(pkg, shape_name, ctx, seed=1234, edit=None):
    sh = pkg.synth.SHAPES[shape_name]
    t = pkg.synth.build_tensors_fast(sh, pkg.gguf.GGMLType.Q8_0, seed=seed)
    if edit:
        edit(t)
    return pkg.loader.model_from_tensors(sh, pkg.gguf.GGMLType.Q8_0, t, ctx)


def _oracle_routing(om, c):
    """The oracle's routing of its last position, per layer: (ids int32 [k], weights float32 [k (+1)])."""
    out = []
    for l in range(c.n_layers):
        r = om.routing[l]
        w = np.asarray(r[1], np.float32)
        if len(r) == 3:
            w = np.append(w, np.float32(r[2]))
        out.append((np.asarray(r[0], np.int32), w))
    return out


def _kv(plan, c):
    nkv = c.context_length * c.kv_dim
    return [plan.read_buffer(n, nkv, layer=l) for n in ("key_cache", "value_cache") for l in range(c.n_layers)]


def _check_kv(plan, om, c, what):
    nkv = c.context_length * c.kv_dim
    for l in range(c.n_layers):
        assert_bit_equal(plan.read_buffer("key_cache", nkv, layer=l), om.key_cache(l), f"{what}: key cache layer {l}")
        assert_bit_equal(plan.read_buffer("value_cache", nkv, layer=l), om.value_cache(l), f"{what}: value cache layer {l}")


def _chunk_then_oracle(plan, om, c, toks, chunks, what):
    """Each chunk through the plan in the new mode and position by position through the oracle: every row's chunk routing bit-equal
    to the oracle's routing at that position; returns the chunk routing of the last chunk."""
    for s, n in chunks:
        plan.forward_batch_prefill(toks[s:s + n], s)
        ids, w = plan.moe_chunk_routing()
        assert ids.shape == (c.n_layers, n, c.n_experts_used), ids.shape
        for v in range(n):
            om.forward(int(toks[s + v]), s + v, want_logits=False)
            for l, (rid, rw) in enumerate(_oracle_routing(om, c)):
                assert np.array_equal(ids[l, v], rid), f"{what}: chunk ({s}, {n}) row {v} layer {l} ids {ids[l, v]} != {rid}"
                assert_bit_equal(w[l, v], rw, f"{what}: chunk ({s}, {n}) row {v} layer {l} routing weights")
    return ids, w


def _decode_after(plan, om, c, tok, pos, steps, what):
    for p in range(pos, pos + steps):
        lg, am = plan.forward_decode(tok, p)
        assert_bit_equal(lg, om.forward(tok, p), f"{what}: logits pos {p}")
        ids, w = plan.moe_routing()
        for l, (rid, rw) in enumerate(_oracle_routing(om, c)):
            assert np.array_equal(ids[l], rid), f"{what}: decode pos {p} layer {l} ids"
            assert_bit_equal(w[l], rw, f"{what}: decode pos {p} layer {l} routing weights")
        tok = am


RUNS = [[(0, 1)], [(0, 37)], [(0, 64)], [(0, 128)], [(s, min(128, 600 - s)) for s in range(0, 600, 128)]]


@pytest.mark.parametrize("shape", SHAPES)
def test_chunks_against_the_oracle(pkg, orc, make_model, shape):
    """Chunks of 1, 37, 64 and 128 tokens from position 0, and 600 positions in 128-token chunks: every layer's K / V and every row's
    routing bit-equal to the oracle, then 8 greedy decode steps with bit-equal logits and routing."""
    m = make_model(shape, pkg.gguf.GGMLType.Q8_0, 640)
    c = m.configuration
    toks = orc.bench_tokens(c.vocab_size, 601)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=128)
    om = _oracle(orc, m)
    try:
        plan.set_prefill_mode(MOE)
        assert plan.prefill_info()[0] == plan.PREFILL_TENSOR_CORE_EXACT_MOE
        for run in RUNS:
            plan.kv_reset()
            om.reset()
            what = f"{shape} {run[0]}..{run[-1]}"
            _chunk_then_oracle(plan, om, c, toks, run, what)
            _check_kv(plan, om, c, what)
            end = run[-1][0] + run[-1][1]
            _decode_after(plan, om, c, int(toks[end]), end, 8, what)
    finally:
        plan.free()
        om.close()


@pytest.mark.parametrize("shape", ["tiny-qwen2moe", "tiny-qwen3moe", "tiny-qwen3moe-k8"])
def test_scores_are_exact_modes(pkg, orc, make_model, shape, monkeypatch):
    """score_tokens in the new mode: bit-equal to exact mode on the same plan, within 1e-9 of the oracle's float64 log-softmax."""
    monkeypatch.setattr(test_gpu_score, "MODES", ("exact", "tensor_core_exact", MOE))
    m = make_model(shape, pkg.gguf.GGMLType.Q8_0, ctx=96, seed=21)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=64)
    om = _oracle(orc, m)
    try:
        assert set(test_gpu_score._score_in_every_mode(pkg, plan, om, m.configuration, test_gpu_score.CHUNKS)) == {"exact", MOE}
    finally:
        plan.free()
        om.close()


def test_all_zero_router_fills_experts_0_to_7(pkg, orc):
    """All-zero router rows, one 200-token chunk: every row picks experts 0..7 at exactly 0.125, so each of them gets 200 grouped rows
    (two M tiles, the second partial) and the other 8 experts none."""
    sh = pkg.synth.SHAPES["tiny-qwen3moe-k8"]

    def zero(t):
        for l in range(sh.n_layers):
            tt, d, raw = t[f"blk.{l}.ffn_gate_inp.weight"]
            t[f"blk.{l}.ffn_gate_inp.weight"] = (tt, d, np.zeros_like(np.asarray(raw)))
    m = _fast_model(pkg, "tiny-qwen3moe-k8", 256, edit=zero)
    c = m.configuration
    toks = orc.bench_tokens(c.vocab_size, 201)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=200)
    om = Qwen3MoEOracle(orc, m)
    try:
        plan.set_prefill_mode(MOE)
        ids, w = _chunk_then_oracle(plan, om, c, toks, [(0, 200)], "all-zero router")
        assert np.array_equal(ids, np.broadcast_to(np.arange(8, dtype=np.int32), ids.shape))
        assert np.all(w.view(np.uint32) == np.float32(0.125).view(np.uint32))
        _check_kv(plan, om, c, "all-zero router")
        _decode_after(plan, om, c, int(toks[200]), 200, 4, "all-zero router")
    finally:
        plan.free()
        om.close()


def test_tied_router_rows_pick_the_lower_index(pkg, orc):
    """Router rows 1 and 5 identical: wherever a chunk row selects expert 5 it selected 1 before it, and 1 is never passed over."""
    sh = pkg.synth.SHAPES["tiny-qwen3moe"]

    def tie(t):
        for l in range(sh.n_layers):
            tt, d, raw = t[f"blk.{l}.ffn_gate_inp.weight"]
            r = np.asarray(raw).view(np.float32).reshape(sh.n_experts, sh.dim).copy()
            r[5] = r[1]
            t[f"blk.{l}.ffn_gate_inp.weight"] = (tt, d, r.view(np.uint8).reshape(-1))
    m = _fast_model(pkg, "tiny-qwen3moe", 128, edit=tie)
    c = m.configuration
    toks = orc.bench_tokens(c.vocab_size, 97)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=96)
    om = Qwen3MoEOracle(orc, m)
    try:
        plan.set_prefill_mode(MOE)
        ids, _ = _chunk_then_oracle(plan, om, c, toks, [(0, 96)], "tied router")
        picked = 0
        for row in ids.reshape(-1, c.n_experts_used).tolist():
            if 5 in row:
                assert 1 in row and row.index(1) < row.index(5), row
            if 1 in row or 5 in row:
                picked += 1
                assert 1 in row, row
        assert picked > 0, "the tied experts were never selected: the test saw nothing"
        _check_kv(plan, om, c, "tied router")
    finally:
        plan.free()
        om.close()


def test_mid_30b_a3b_every_expert_in_one_chunk(pkg):
    """Qwen3-30B-A3B's layer geometry with the aligned router of test_gpu_qwen3moe: tokens 0..127 in one chunk give every expert rows
    in every layer; the KV cache and the scores bit-equal to exact mode's on the same plan."""
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
    c = m.configuration
    toks = np.arange(E + 1, dtype=np.int32)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=E)
    try:
        plan.forward_batch_prefill(toks[:E], 0)
        want = [a.copy() for a in _kv(plan, c)]
        lp_e, ids_e = plan.score_tokens(toks[:E], 0, toks[1:])
        plan.set_prefill_mode(MOE)
        plan.kv_reset()
        plan.forward_batch_prefill(toks[:E], 0)
        for i, (a, b) in enumerate(zip(_kv(plan, c), want)):
            assert_bit_equal(a, b, f"{'KV'[i // c.n_layers]} cache layer {i % c.n_layers}")
        ids, _ = plan.moe_chunk_routing()
        for l in range(c.n_layers):
            assert set(ids[l].reshape(-1).tolist()) == set(range(E)), f"layer {l}: experts without rows"
        plan.kv_reset()
        lp, ids_s = plan.score_tokens(toks[:E], 0, toks[1:])
        assert np.array_equal(lp.view(np.uint64), lp_e.view(np.uint64)) and np.array_equal(ids_s, ids_e)
    finally:
        plan.free()


def test_mid_a27b_against_its_own_decode(pkg):
    """Qwen1.5-MoE-A2.7B's geometry (expert hidden 1408; the shared down projection's 5632 columns in four 1408-column segments):
    logprobs the float64 log-softmax of forward_decode's logits for the same tokens, ids its argmax, in both modes."""
    m = _fast_model(pkg, "mid-qwen1.5-moe-a2.7b", 80)
    c = m.configuration
    toks = np.random.default_rng(4).integers(0, c.vocab_size, 49).astype(np.int32)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=64)
    try:
        rows, ids_dec = [], []
        for p in range(48):
            lg, am = plan.forward_decode(int(toks[p]), p)
            rows.append(lg.copy())
            ids_dec.append(am)
        lp_ref, ids_ref = score_rows(np.stack(rows), toks[1:])
        assert list(ids_ref) == ids_dec
        for mode in ("exact", MOE):
            plan.set_prefill_mode(mode)
            plan.kv_reset()
            lp, ids = plan.score_tokens(toks[:48], 0, toks[1:])
            assert np.array_equal(ids, ids_ref), mode
            assert np.abs(lp - lp_ref).max() <= 1e-9, mode
    finally:
        plan.free()


def test_kquant_file_against_its_q8_0_twin(pkg, orc):
    """A Q4_K_M Qwen3-MoE file (its experts re-quantised to Q8_0 tiles at upload) against the oracle on its Q8_0 twin."""
    G = pkg.gguf.GGMLType
    sh = pkg.synth.SHAPES["tiny-qwen3moe"]
    tensors = pkg.synth.build_tensors_kquant(sh, seed=21)
    twin = {n: ((G.Q8_0, d, orc.kquant_to_q8_0(t, np.asarray(r), int(np.prod(d)))) if t in G.K_QUANTS else (t, d, r)) for n, (t, d, r) in tensors.items()}
    m = pkg.loader.model_from_tensors(sh, G.Q8_0, tensors, 128)
    mt = pkg.loader.model_from_tensors(sh, G.Q8_0, twin, 128)
    c = m.configuration
    toks = orc.bench_tokens(c.vocab_size, 102)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=64)
    om = Qwen3MoEOracle(orc, mt)
    try:
        plan.set_prefill_mode(MOE)
        _chunk_then_oracle(plan, om, c, toks, [(0, 64), (64, 37)], "Q4_K_M")
        _check_kv(plan, om, c, "Q4_K_M")
        _decode_after(plan, om, c, int(toks[101]), 101, 4, "Q4_K_M")
    finally:
        plan.free()
        om.close()


def test_mode_switching_gives_the_same_bits(pkg, make_model):
    m = make_model("tiny-qwen2moe", pkg.gguf.GGMLType.Q8_0, 128)
    c = m.configuration
    toks = np.random.default_rng(9).integers(0, c.vocab_size, 64).astype(np.int32)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=64)
    try:
        runs = []
        for mode in ("exact", MOE, "exact", MOE):
            plan.set_prefill_mode(mode)
            assert plan.prefill_info()[0] == {"exact": 0, MOE: 4}[mode]
            plan.kv_reset()
            plan.forward_batch_prefill(toks, 0)
            runs.append([a.copy() for a in _kv(plan, c)])
        for r in runs[1:]:
            for a, b in zip(r, runs[0]):
                assert_bit_equal(a, b, "KV cache after switching modes")
    finally:
        plan.free()


def test_refusals_then_decode_and_launch_count(pkg, orc, make_model):
    """A dense Q8_0 plan, an MoE plan without a prefill batch size (B200_ERR_UNSUPPORTED naming the reason) and mode 5
    (B200_ERR_BAD_ARG): the previous mode stays and the next decode step is bit-exact.  A chunk reports the documented launches:
    12 per layer (14 with a shared expert) when the attention runs in one launch."""
    N = pkg.native
    G = pkg.gguf.GGMLType
    cases = [(make_model("tiny-llama", G.Q8_0, 32), 16, "tensor_core_exact"), (make_model("tiny-qwen3moe", G.Q8_0, 32), 0, "prefill batch size"),
             (make_model("tiny-qwen2moe", G.Q8_0, 32), 16, None)]
    for m, batch, why in cases:
        plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=batch)
        om = _oracle(orc, m) if m.configuration.n_experts else orc.OracleModel(m)
        try:
            if why:
                with pytest.raises(N.UnsupportedOperation, match=why):
                    plan.set_prefill_mode(MOE)
            with pytest.raises(N.B200Error) as e:
                plan.set_prefill_mode(5)
            assert e.value.code == -1
            assert plan.prefill_info()[0] == plan.PREFILL_EXACT
            lg, _ = plan.forward_decode(3, 0)
            assert_bit_equal(lg, om.forward(3, 0), f"{m.model_type}: decode after the refusals")
        finally:
            plan.free()
            om.close()
    for shape, per_layer in (("tiny-qwen3moe", 12), ("tiny-qwen2moe", 14)):
        m = make_model(shape, G.Q8_0, 64)
        plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=48)
        try:
            plan.set_prefill_mode(MOE)
            plan.forward_batch_prefill(np.arange(1, 41, dtype=np.int32), 0)
            mode, launches, ms = plan.prefill_info()
            assert mode == 4 and launches == per_layer * m.configuration.n_layers and ms > 0, (mode, launches, ms)
            before = plan.moe_routing()
            plan.forward_batch_prefill(np.arange(2, 10, dtype=np.int32), 40)
            after = plan.moe_routing()
            assert all(np.array_equal(a, b) for a, b in zip(before, after)), "a chunk touched the decode routing buffers"
        finally:
            plan.free()


@pytest.mark.parametrize("mode,n,k", [("f32", 128, 512), ("f32", 64, 2048), ("gateup", 64, 512), ("gateup", 32, 2048)])
def test_gemm_i8_experts(pkg, mode, n, k):
    """Expert row counts 0, 1, 63, 64, 65, 128, 129 and 300 (empty experts between full ones, partial and multi-tile groups): every
    expert's rows bit-equal to the float32 block-order restatement against that expert's weights."""
    counts = np.array([65, 0, 1, 300, 63, 129, 0, 64, 128], np.int32)
    E, M = len(counts), int(counts.sum())
    rng = np.random.default_rng(n * 7 + k + len(mode))
    aq, a_scales = _activations(rng, M, k)
    bq = np.stack([_weights(rng, n, k) for _ in range(E)])
    off = np.concatenate([[0], np.cumsum(counts)])
    if mode == "gateup":
        bq2 = np.stack([_weights(rng, n, k) for _ in range(E)])
        hq0, hs0 = np.full((M, n), 0x5A, np.int8), np.full((M, n // 32), np.nan, np.float32)
        hq, hs = pkg.native.test_gemm_i8_experts(mode, counts, aq, a_scales, bq, bq2=bq2, hq=hq0, hs=hs0)
        for e in range(E):
            r = slice(off[e], off[e + 1])
            wq, ws = _swiglu_q8(_dot_q8(aq[r], a_scales[r], bq[e]), _dot_q8(aq[r], a_scales[r], bq2[e]))
            assert np.array_equal(hq[r], wq), f"expert {e}: quantised hidden rows differ"
            assert np.array_equal(hs[r].view(np.uint32), ws.view(np.uint32)), f"expert {e}: block scales differ"
        return
    c0 = np.full((M, n), np.nan, np.float32)
    got = pkg.native.test_gemm_i8_experts(mode, counts, aq, a_scales, bq, c=c0)
    for e in range(E):
        r = slice(off[e], off[e + 1])
        want = _dot_q8(aq[r], a_scales[r], bq[e])
        assert np.array_equal(got[r].view(np.uint32), want.view(np.uint32)), f"expert {e}: {int(np.sum(got[r].view(np.uint32) != want.view(np.uint32)))} differ"
