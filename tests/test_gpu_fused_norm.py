"""GPU tests of the RMSNorm fused into the Q8_0 weight streams that consume it (k_stream_matvec_q8_norm, csrc/norm_slots.cuh):
single-GPU Q8_0 streaming plans decode with 5 launches per layer + 2, bit-exact against the oracle (logits as uint32, ids, KV
cache) at widths that give 1, 2, 4 and 5 sixteen-byte slots per consumer thread; every other plan (FP16, tensor parallelism,
Qwen2-MoE) keeps the separate norm kernel."""
import numpy as np
import pytest

from granite_oracle import GraniteOracle
from qwen2moe_oracle import Qwen2MoEOracle
from test_gpu_parity import assert_bit_equal

pytestmark = pytest.mark.gpu


def _model(pkg, sh, quant, ctx, seed=11):
    return pkg.loader.model_from_tensors(sh, quant, pkg.synth.build_tensors_fast(sh, quant, seed=seed), ctx)


def _oracle(orc, m):
    if m.model_type == "GRANITE":
        return GraniteOracle(orc, m)
    if m.model_type == "QWEN_2_MOE":
        return Qwen2MoEOracle(orc, m)
    return orc.OracleModel(m)


def _decode_vs_oracle(pkg, orc, m, n, tok=1):
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = _oracle(orc, m)
    c = m.configuration
    try:
        assert plan.decode_info()[0] == 0  # the CUDA graph
        for pos in range(n):
            lg, am = plan.forward_decode(tok, pos)
            ref = om.forward(tok, pos)
            assert_bit_equal(lg, ref, f"logits pos {pos}")
            assert am == orc.argmax(ref), f"argmax pos {pos}"
            tok = am
        nkv = c.context_length * c.kv_dim
        for l in range(c.n_layers):
            assert_bit_equal(plan.read_buffer("key_cache", nkv, layer=l), om.key_cache(l), f"key cache layer {l}")
            assert_bit_equal(plan.read_buffer("value_cache", nkv, layer=l), om.value_cache(l), f"value cache layer {l}")
        return plan.launches_per_decode
    finally:
        plan.free()
        om.close()


@pytest.mark.parametrize("dim", [1024, 2048, 4096, 5120])  # 1, 2, 4 and 5 slots of 16 bytes per consumer thread
def test_fused_norm_widths_bit_exact(pkg, orc, dim):
    """Llama layers at each width, a vocabulary that is not a multiple of 4 (the lm_head's fused norm and its padded group)."""
    sh = pkg.synth.Shape("llama", dim, 1024, 2, dim // 128, dim // 512, 128, 515, False, 500000.0, 1e-5)
    m = _model(pkg, sh, pkg.gguf.GGMLType.Q8_0, 16)
    assert _decode_vs_oracle(pkg, orc, m, 6) == 5 * sh.n_layers + 2


def test_fused_norm_granite_bit_exact(pkg, orc, make_model):
    """Granite: layer 0's fused norm gathers the embedding row times the embedding scale, and CTA 0 writes it to x for Wo."""
    m = make_model("tiny-granite", pkg.gguf.GGMLType.Q8_0, 24)
    assert m.model_type == "GRANITE"
    assert _decode_vs_oracle(pkg, orc, m, 10) == 5 * m.configuration.n_layers + 2


def test_qwen2moe_keeps_the_separate_norm(pkg, orc, make_model):
    """Qwen2-MoE plans keep the norm kernel (its FFN norm writes float xb for the F32 router): 8 launches per layer + 3, bit-exact."""
    m = make_model("tiny-qwen2moe-gqa", pkg.gguf.GGMLType.Q8_0, 64)
    assert m.model_type == "QWEN_2_MOE"
    L = m.configuration.n_layers
    assert _decode_vs_oracle(pkg, orc, m, 10) == 8 * L + 3


def test_fused_norm_exact_prefill_kv_bit_exact(pkg, orc, make_model):
    """The exact token-by-token prefill runs the same fused graph (without the lm_head): its KV cache is the oracle's, bit for bit,
    and the decode that follows it is too."""
    m = make_model("tiny-llama", pkg.gguf.GGMLType.Q8_0, 64)
    c = m.configuration
    toks = orc.bench_tokens(c.vocab_size, 21)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=8)
    om = orc.OracleModel(m)
    try:
        plan.set_prefill_mode("exact")
        assert plan.prefill_info()[0] == plan.PREFILL_EXACT
        for off in range(0, 20, 8):
            plan.forward_batch_prefill(toks[off:min(off + 8, 20)], off)
        for pos in range(20):
            om.forward(int(toks[pos]), pos, want_logits=False)
        nkv = c.context_length * c.kv_dim
        for l in range(c.n_layers):
            assert_bit_equal(plan.read_buffer("key_cache", nkv, layer=l), om.key_cache(l), f"key cache layer {l}")
            assert_bit_equal(plan.read_buffer("value_cache", nkv, layer=l), om.value_cache(l), f"value cache layer {l}")
        lg, am = plan.forward_decode(int(toks[20]), 20)
        ref = om.forward(int(toks[20]), 20)
        assert_bit_equal(lg, ref, "logits after the prefill")
        assert am == orc.argmax(ref)
    finally:
        plan.free()
        om.close()


def test_launch_counts_of_the_other_plans(pkg, make_model):
    """5 L + 2 on a single-GPU Q8_0 plan; the FP16 rings keep the separate norm kernel: 7 L + 3."""
    q8 = make_model("tiny-llama", pkg.gguf.GGMLType.Q8_0, 24)
    f16 = make_model("tiny-llama", pkg.gguf.GGMLType.F16, 24)
    L = q8.configuration.n_layers
    plan = pkg.B200MasterPlan.initialize_plan(q8)
    try:
        assert plan.launches_per_decode == 5 * L + 2
        assert plan.decode_info()[1] == 5 * L + 2
    finally:
        plan.free()
    plan = pkg.B200MasterPlan.initialize_plan(f16, fp16_lanes=16)
    try:
        assert plan.launches_per_decode == 7 * L + 3
    finally:
        plan.free()


def test_stand_alone_fused_kernels_time(pkg, orc):
    """b200_time_kernel times the fused QKV, gate/up and lm_head on their own; their algorithmic bytes include the norm weights."""
    sh = pkg.synth.Shape("llama", 1024, 1024, 2, 8, 2, 128, 515, False, 500000.0, 1e-5)
    m = _model(pkg, sh, pkg.gguf.GGMLType.Q8_0, 16)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    try:
        plan.forward_decode(1, 0)
        q8 = lambda rows: rows * 1024 // 32 * 34  # Q8_0 bytes of a rows x 1024 matrix
        expect = {0: [q8(2 * 1024)], 2: [q8(1024 + 2 * 256)], 4: [q8(515), q8(516)]}  # gate/up, QKV, lm_head (its last group padded or not)
        for which, rows_bytes in expect.items():
            ms, nbytes = plan.time_kernel(which, 2)
            assert ms > 0
            assert nbytes in [b + 1024 * 4 for b in rows_bytes], (which, nbytes)
    finally:
        plan.free()
