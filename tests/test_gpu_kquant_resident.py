"""GPU tests of resident K-quant weights: a plan whose K-quant matrices do not fit the device as Q8_0 tiles keeps the raw super-blocks
in its weight streams, and the stream kernels rebuild the reference's Q8_0 blocks from them (csrc/stream_matvec.cuh, kq_q8_block in
csrc/kquant.cuh).  Bar: bit-identical logits, ids and KV cache against the oracle on the re-quantised Q8_0 twin, which is what the
reference computes with after ModelLoader.dequantizeToQ8_0TornadoTensor.

The residency rule reads the device's free memory; b200_test_set_memory_budget replaces that figure so a tiny model can be put on
either side of the threshold.  A plan created under a budget of 1 byte fails and names both figures (the Q8_0 form and the resident
form, each with what the plan allocates besides its weights), and the budget halfway between them builds the plan resident."""
import re

import numpy as np
import pytest

from devstral_oracle import DevstralOracle
from granite_oracle import GraniteOracle
from qwen2_oracle import Qwen2Oracle
from test_gpu_kquants import _requantised_twin
from test_gpu_parity import assert_bit_equal

pytestmark = pytest.mark.gpu

KB = {12: 144, 13: 176, 14: 210}


def _needs(msg):
    m = re.search(r"(\d+) bytes with Q8_0 tiles and (\d+) bytes with K-quant weights resident", msg)
    assert m, msg
    return int(m.group(1)), int(m.group(2))


def _figures(pkg, m, **kw):
    """(bytes the Q8_0 form needs, bytes the resident form needs) of model m, from the creation that fits neither."""
    n = pkg.native
    n.test_set_memory_budget(1)
    try:
        with pytest.raises(n.B200Error) as e:
            pkg.B200MasterPlan.initialize_plan(m, **kw)
    finally:
        n.test_set_memory_budget(0)
    assert e.value.code == -3, str(e.value)  # B200_ERR_OOM
    return _needs(str(e.value))


def _plan_under(pkg, m, budget, **kw):
    pkg.native.test_set_memory_budget(budget)
    try:
        return pkg.B200MasterPlan.initialize_plan(m, **kw)
    finally:
        pkg.native.test_set_memory_budget(0)


def _resident_plan(pkg, m, **kw):
    q8, res = _figures(pkg, m, **kw)
    assert res < q8
    plan = _plan_under(pkg, m, (q8 + res) // 2, **kw)
    assert plan.weight_info()["resident"]
    return plan


def _model(pkg, shape, mix="Q4_K_M", ctx=24, seed=11, tensors=None):
    sh = pkg.synth.SHAPES[shape]
    t = tensors if tensors is not None else pkg.synth.build_tensors_kquant(sh, seed=seed, mix=mix)
    return pkg.loader.model_from_tensors(sh, pkg.gguf.GGMLType.Q8_0, t, ctx)


def _oracle(pkg, orc, m):
    twin = _requantised_twin(pkg, orc, m)
    a, L = twin.configuration.arch, pkg.loader
    if a == L.ARCH_GRANITE:
        return GraniteOracle(orc, twin)
    if a == L.ARCH_DEVSTRAL:
        return DevstralOracle(orc, twin)
    if a == L.ARCH_QWEN2:
        return Qwen2Oracle(orc, twin)
    return orc.OracleModel(twin)


def _decode_matches(pkg, orc, m, n_tok, plan=None):
    c = m.configuration
    plan = plan or _resident_plan(pkg, m)
    om = _oracle(pkg, orc, m)
    try:
        tok = 3
        for pos in range(n_tok):
            lg, am = plan.forward_decode(tok, pos)
            ref = om.forward(tok, pos)
            assert_bit_equal(lg, ref, f"logits pos {pos}")
            assert am == orc.argmax(ref), f"argmax pos {pos}"
            tok = am
        nkv = c.context_length * c.kv_dim
        for l in range(c.n_layers):
            assert_bit_equal(plan.read_buffer("key_cache", nkv, layer=l), om.key_cache(l), f"key cache layer {l}")
            assert_bit_equal(plan.read_buffer("value_cache", nkv, layer=l), om.value_cache(l), f"value cache layer {l}")
    finally:
        plan.free()
        om.close()


@pytest.mark.parametrize("shape,mix,n_tok", [
    ("tiny-llama", "Q4_K_M", 10), ("tiny-llama-tied", "Q6_K", 10), ("tiny-qwen3", "Q5_K", 10), ("tiny-qwen3", "Q4_K_M", 10),
    ("tiny-qwen2-gqa6", "Q4_K_M", 8), ("tiny-phi3-gqa", "Q4_K_M", 8), ("mid-granite-3-2b", "Q4_K_M", 4), ("tiny-devstral", "Q4_K_M", 8),
    ("mid-llama", "Q4_K_M", 4), ("mid-llama-70b", "Q4_K_M", 3)])
def test_resident_plan_decodes_like_its_q8_0_twin(pkg, orc, shape, mix, n_tok):
    """Every format as a resident stream (Q4_K gate/up, Q5_K Wo, Q6_K down and classifier), a tied classifier built from the embedding's
    K-quant bytes, Qwen2 biases, Phi-3's fused qkv / gate-up tensors, Granite's 49155-row classifier (zero padding rows), Devstral's
    qd != dim, and the 8B / 70B layer geometries (56- and 112-super-block rows)."""
    _decode_matches(pkg, orc, _model(pkg, shape, mix), n_tok)


def test_resident_plan_700_positions(pkg, orc):
    """Long enough that the attention's score row leaves shared memory for the global scratch row."""
    _decode_matches(pkg, orc, _model(pkg, "tiny-llama", ctx=720, seed=12), 700)


def test_resident_exact_prefill_kv_matches_token_by_token(pkg, orc):
    m = _model(pkg, "tiny-llama", ctx=64, seed=13)
    c = m.configuration
    plan = _resident_plan(pkg, m, prefill_batch_size=32)
    om = _oracle(pkg, orc, m)
    try:
        toks = orc.bench_tokens(c.vocab_size, 40)
        plan.forward_batch_prefill(toks[:32], 0)
        plan.forward_batch_prefill(toks[32:], 32)
        for pos, t in enumerate(toks):
            om.forward(int(t), pos, want_logits=False)
        nkv = c.context_length * c.kv_dim
        for l in range(c.n_layers):
            assert_bit_equal(plan.read_buffer("key_cache", nkv, layer=l), om.key_cache(l), f"key cache layer {l}")
            assert_bit_equal(plan.read_buffer("value_cache", nkv, layer=l), om.value_cache(l), f"value cache layer {l}")
        lg, am = plan.forward_decode(int(toks[-1]), 40)
        ref = om.forward(int(toks[-1]), 40)
        assert_bit_equal(lg, ref, "logits after the prefill")
    finally:
        plan.free()
        om.close()


def test_resident_device_sampler_matches_the_q8_0_plan(pkg):
    """Same logits, so the device sampler draws the same ids with the same diagnostics as on the plan built with Q8_0 tiles."""
    m = _model(pkg, "tiny-qwen3", seed=14)
    res, q8 = _resident_plan(pkg, m), pkg.B200MasterPlan.initialize_plan(m)
    try:
        assert not q8.weight_info()["resident"]
        tok_r = tok_q = 5
        for pos, (temp, topp, u) in enumerate([(0.7, 0.9, 0.31), (1.0, 0.0, 0.77), (0.0, 0.9, 0.5), (1.3, 0.5, 0.02), (0.8, 0.95, 0.999)]):
            tok_r, info_r = res.forward_decode_sample(tok_r, pos, temp, topp, u, want_info=True)
            tok_q, info_q = q8.forward_decode_sample(tok_q, pos, temp, topp, u, want_info=True)
            assert (tok_r, info_r) == (tok_q, info_q), f"step {pos}"
        ids_r, _ = res.decode_sequence([tok_r], 8, 5, feedback=True)
        ids_q, _ = q8.decode_sequence([tok_q], 8, 5, feedback=True)
        assert np.array_equal(ids_r, ids_q)
    finally:
        res.free()
        q8.free()


def _set_f16(raw, off, v):
    raw[off:off + 2] = np.frombuffer(np.float16(v).tobytes(), dtype=np.uint8)


def _hostile(pkg, tensors):
    """Plant hostile super-blocks at the start of the Q4_K gate (resident gate/up stream), the Q5_K attention output and the Q6_K down
    projection of layer 0 of a Q4_K_M mix."""
    G = pkg.gguf.GGMLType
    for name, tt in (("blk.0.ffn_gate.weight", G.Q4_K), ("blk.0.attn_output.weight", G.Q5_K), ("blk.0.ffn_down.weight", G.Q6_K)):
        t, dims, raw = tensors[name]
        assert t == tt
        raw = np.array(raw, copy=True)
        kb = KB[tt]
        sb = [raw[i * kb:(i + 1) * kb] for i in range(7)]  # the first super-blocks of the tensor (views; rows 0.. of this shape)
        if tt == G.Q6_K:
            _set_f16(sb[0], 208, 2.0)                     # a large d with the largest scales ...
            sb[0][192:208] = np.frombuffer(np.array([127] * 8 + [-128] * 8, dtype=np.int8).tobytes(), dtype=np.uint8)
            sb[0][0:32] = 0x00                            # ... sub-block 0: code -32 (low nibble 0, high bits 0)
            sb[0][128:160] &= 0xFC
            sb[0][32:64] |= 0x0F                          # sub-block 1: code 31 (low nibble 15, high bits 3)
            sb[0][128:160] |= 0x0C
            _set_f16(sb[1], 208, 0.0)                     # d = 0
            _set_f16(sb[2], 208, -3e-5)                   # negative d
            sb[3][208:210] = [0x01, 0x00]                 # subnormal d
            sb[4][0:128] = 0x55                           # all-equal codes
            sb[4][128:192] = 0xAA
        else:
            qs = 16 if tt == G.Q4_K else 48
            _set_f16(sb[0], 0, 0.0)                       # d = 0: every value is -dmin * m
            _set_f16(sb[1], 2, 0.0)                       # dmin = 0
            _set_f16(sb[2], 0, -2e-4)                     # negative d
            sb[3][0:2] = [0x07, 0x00]                     # subnormal d
            sb[4][qs:qs + 128] = 0x77                     # all-equal nibbles
            if tt == G.Q5_K:
                sb[4][16:48] = 0x00
            sb[5][4] &= 0xC0                              # sub-block 0: scale 0 and min 0 -> an all-zero 32-block (scale 0, the 1/scale guard)
            sb[5][8] &= 0xC0
            _set_f16(sb[6], 0, 1e-5)                      # the maximum |v| on the dmin side: d * scale * q << dmin * m
            _set_f16(sb[6], 2, 0.05)
        tensors[name] = (t, dims, raw)
    return tensors


def test_hostile_kquant_blocks_in_resident_streams(pkg, orc):
    sh = pkg.synth.SHAPES["tiny-llama"]
    tensors = _hostile(pkg, pkg.synth.build_tensors_kquant(sh, seed=15))
    _decode_matches(pkg, orc, _model(pkg, "tiny-llama", tensors=tensors), 8)


def test_policy_thresholds(pkg):
    m = _model(pkg, "tiny-llama", seed=16)
    q8, res = _figures(pkg, m, prefill_batch_size=32)
    plan = _plan_under(pkg, m, q8, prefill_batch_size=32)  # Q8_0 tiles fit exactly: the plan is built as before
    try:
        info = plan.weight_info()
        assert not info["resident"] and info["weight_bytes"] == info["q8_weight_bytes"] > 0
        plan.set_decode_mode("persistent")
        plan.set_decode_mode("graph")
        plan.set_decode_slots(2)
        assert plan.decode_multi_rows() > 0
        plan.set_decode_slots(0)
        plan.set_prefill_mode("tensor_core_w8a16")
        plan.set_prefill_mode("exact")
    finally:
        plan.free()
    plan = _plan_under(pkg, m, q8 - 1, prefill_batch_size=32)
    try:
        info = plan.weight_info()
        assert info["resident"] and info["weight_bytes"] < info["q8_weight_bytes"]
        assert q8 - res == info["q8_weight_bytes"] - info["weight_bytes"]
    finally:
        plan.free()
    pkg.native.test_set_memory_budget(res - 1)
    try:
        with pytest.raises(pkg.native.B200Error) as e:
            pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=32)
    finally:
        pkg.native.test_set_memory_budget(0)
    assert str(q8) in str(e.value) and str(res) in str(e.value), str(e.value)


def _stream_bytes(rows, cols, fmt):
    q = 256 if fmt else 32
    nseg = next(n for n in range(1, cols // q + 1) if cols % n == 0 and (cols // n) % q == 0 and cols // n <= 2560)
    seg = cols // nseg
    unit = ((seg // 256 * KB[fmt]) if fmt else seg + seg // 16) + 15 & ~15
    return (rows + 3) // 4 * 4 * nseg * unit


def test_resident_footprint_is_the_layout_arithmetic(pkg):
    """mid-llama (8B layer geometry) in the Q4_K_M mix: QKV mixes Q4_K and Q6_K sources and stays Q8_0 tiles; Wo (Q5_K), gate/up (Q4_K),
    down and the classifier (Q6_K) are resident; the embedding keeps its Q8_0 planes."""
    G = pkg.gguf.GGMLType
    m = _model(pkg, "mid-llama", ctx=16, seed=17)
    c = m.configuration
    plan = _resident_plan(pkg, m)
    try:
        info = plan.weight_info()
    finally:
        plan.free()
    qd, kvd, d, h, v = c.n_heads * c.head_size, c.n_kv_heads * c.head_size, c.dim, c.hidden_dim, c.vocab_size
    layer = lambda fmt_wo, fmt_gu, fmt_dn, fmt_qkv: (_stream_bytes(qd + 2 * kvd, d, fmt_qkv) + _stream_bytes(d, qd, fmt_wo)
                                                    + _stream_bytes(2 * h, d, fmt_gu) + _stream_bytes(d, h, fmt_dn))
    emb = v * d // 32 * 34
    want = emb + _stream_bytes(v, d, G.Q6_K) + c.n_layers * layer(G.Q5_K, G.Q4_K, G.Q6_K, 0)
    want8 = emb + _stream_bytes(v, d, 0) + c.n_layers * layer(0, 0, 0, 0)
    assert info["weight_bytes"] == want and info["q8_weight_bytes"] == want8
    assert info["weight_bytes"] < 0.75 * info["q8_weight_bytes"]


def test_resident_plan_refusals(pkg, orc):
    """Each refused call raises UnsupportedOperation (-2) with its reason, and the plan decodes bit-exactly afterwards."""
    m = _model(pkg, "tiny-llama", seed=18)
    plan = _resident_plan(pkg, m, prefill_batch_size=16)
    U = pkg.native.UnsupportedOperation
    calls = [lambda: plan.set_decode_mode("persistent"), lambda: plan.set_decode_slots(1), lambda: plan.forward_decode_multi(-1, [1, 2], 0),
             lambda: plan.forward_step([(0, 1, 0, 1)]), lambda: plan.set_prefill_mode("tensor_core"),
             lambda: plan.set_prefill_mode("tensor_core_w8a16")]
    for i, call in enumerate(calls):
        with pytest.raises(U) as e:
            call()
        assert e.value.code == -2 and "resident" in str(e.value), f"call {i}: {e.value}"
    assert plan.decode_multi_rows() == 0
    assert plan.decode_info()[0] == 0
    _decode_matches(pkg, orc, m, 6, plan=plan)
