"""GPU tests of the Qwen2 family (B200_ARCH_QWEN2: q/k/v biases + NeoX RoPE, GQA ratios 5/6/7) through the C ABI, against the CPU
restatement of forwardJavaQwen2 (tests/qwen2_oracle.py).  Decode and the exact prefill are bit-exact (logits compared as uint32);
the tensor-core prefill is held to the bars of tests/test_gpu_prefill.py, and its attention kernels, at GQA ratios that do not
divide 64, to that file's float64 bound."""
import zlib

import numpy as np
import pytest

from qwen2_oracle import Qwen2Oracle
from test_gpu_parity import assert_bit_equal, set_mode
from test_gpu_prefill import ATT_KINDS, ATT_SENTINEL, FP16_TOL, Q8_NOISE_TOL, _attention_inputs, _check_attention

pytestmark = pytest.mark.gpu


def _fast_model(pkg, shape_name, quant, ctx, seed=1234):
    sh = pkg.synth.SHAPES[shape_name]
    return pkg.loader.model_from_tensors(sh, quant, pkg.synth.build_tensors_fast(sh, quant, seed=seed), ctx)


def _decode_vs_oracle(pkg, orc, m, n, mode="graph", lanes=16):
    plan = pkg.B200MasterPlan.initialize_plan(m, fp16_lanes=lanes)
    set_mode(pkg, plan, mode)
    om = Qwen2Oracle(orc, m, lanes=lanes)
    c = m.configuration
    tok = 1
    try:
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
    finally:
        plan.free()
        om.close()


@pytest.mark.parametrize("shape", ["tiny-qwen2", "tiny-qwen2-gqa6"])
@pytest.mark.parametrize("quant,mode", [("Q8_0", "graph"), ("Q8_0", "persistent"), ("F16", "graph")])
def test_qwen2_decode_bit_exact(pkg, orc, make_model, shape, quant, mode):
    m = make_model(shape, getattr(pkg.gguf.GGMLType, quant), 24)
    _decode_vs_oracle(pkg, orc, m, 16, mode)


@pytest.mark.parametrize("shape", ["mid-qwen2.5-0.5b", "mid-deepseek-r1-qwen-1.5b", "mid-qwen2.5-7b"])
@pytest.mark.parametrize("quant,mode", [("Q8_0", "graph"), ("Q8_0", "persistent"), ("F16", "graph")])
def test_qwen2_mid_geometries_bit_exact(pkg, orc, shape, quant, mode):
    """The real Qwen2.5-0.5B / DeepSeek-R1-Distill-Qwen-1.5B / Qwen2.5-7B layer geometries (2 layers, vocabulary 8192)."""
    _decode_vs_oracle(pkg, orc, _fast_model(pkg, shape, getattr(pkg.gguf.GGMLType, quant), 16), 6, mode)


def test_qwen2_kquant_decodes_like_its_q8_0_twin(pkg, orc):
    """A K-quant Qwen2 file (Q4_K_M mix; the biases stay F32) against the oracle on its Q8_0 re-quantised twin."""
    G = pkg.gguf.GGMLType
    sh = pkg.synth.SHAPES["tiny-qwen2-gqa6"]
    tensors = pkg.synth.build_tensors_kquant(sh, seed=21)
    twin = {n: ((G.Q8_0, d, orc.kquant_to_q8_0(t, np.asarray(r), int(np.prod(d)))) if t in G.K_QUANTS else (t, d, r)) for n, (t, d, r) in tensors.items()}
    m = pkg.loader.model_from_tensors(sh, G.Q8_0, tensors, 24)
    mt = pkg.loader.model_from_tensors(sh, G.Q8_0, twin, 24)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = Qwen2Oracle(orc, mt)
    try:
        tok = 3
        for pos in range(12):
            lg, am = plan.forward_decode(tok, pos)
            ref = om.forward(tok, pos)
            assert_bit_equal(lg, ref, f"logits pos {pos}")
            tok = am
    finally:
        plan.free()
        om.close()


@pytest.mark.parametrize("mode", ["graph", "persistent"])
def test_qwen2_long_context_bit_exact(pkg, orc, make_model, mode):
    """700 positions through b200_decode_sequence (the device-resident loop): every greedy id and the last logits."""
    n = 700
    m = make_model("tiny-qwen2", pkg.gguf.GGMLType.Q8_0, 720)
    c = m.configuration
    toks = orc.bench_tokens(c.vocab_size, n)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    set_mode(pkg, plan, mode)
    om = Qwen2Oracle(orc, m)
    try:
        ids, _ = plan.decode_sequence(toks, n, 0)
        for pos in range(n):
            ref = om.forward(int(toks[pos]), pos)
            assert ids[pos] == orc.argmax(ref), f"argmax pos {pos}"
        assert_bit_equal(plan.read_buffer("logits", c.vocab_size), ref, "logits of the last step")
        nkv = c.context_length * c.kv_dim
        assert_bit_equal(plan.read_buffer("key_cache", nkv, layer=1), om.key_cache(1), "key cache layer 1")
    finally:
        plan.free()
        om.close()


@pytest.mark.parametrize("shape", ["tiny-qwen2", "tiny-qwen2-gqa6"])
def test_qwen2_exact_batch_prefill_kv_bit_identical(pkg, orc, make_model, shape):
    m = make_model(shape, pkg.gguf.GGMLType.Q8_0, 64)
    c = m.configuration
    toks = orc.bench_tokens(c.vocab_size, 45)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=16)
    om = Qwen2Oracle(orc, m)
    try:
        assert plan.prefill_info()[0] == plan.PREFILL_EXACT
        for off in range(0, 45, 16):
            plan.forward_batch_prefill(toks[off:off + 16], off)
        for pos in range(45):
            om.forward(int(toks[pos]), pos, want_logits=False)
        nkv = c.context_length * c.kv_dim
        for l in range(c.n_layers):
            assert_bit_equal(plan.read_buffer("key_cache", nkv, layer=l), om.key_cache(l), f"key cache layer {l}")
            assert_bit_equal(plan.read_buffer("value_cache", nkv, layer=l), om.value_cache(l), f"value cache layer {l}")
    finally:
        plan.free()
        om.close()


def test_qwen2_device_sampler_at_vocab_152k(pkg, orc):
    sh = pkg.synth.SHAPES["tiny-qwen2-vocab152k"]
    assert sh.vocab == 151936
    m = _fast_model(pkg, "tiny-qwen2-vocab152k", pkg.gguf.GGMLType.Q8_0, 16)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = Qwen2Oracle(orc, m)
    rng = orc.JavaLXM(777)
    try:
        tok = 5
        for pos, (temp, topp) in enumerate([(0.7, 0.9), (1.0, 0.0), (0.6, 0.95), (0.0, 0.9), (0.8, 0.9)]):
            r = rng.next_float1()
            got = plan.forward_decode_sample(tok, pos, temp, topp, r)
            want = orc.sample(om.forward(tok, pos), temp, topp, r)
            assert got == want, (pos, temp, topp, got, want)
            tok = got
    finally:
        plan.free()
        om.close()


def test_qwen2_plan_without_a_bias_fails_and_names_it(pkg, make_model):
    m = make_model("tiny-qwen2", pkg.gguf.GGMLType.Q8_0, 16)
    t = dict(m.tensors)
    del t["blk.1.attn_v.bias"]
    bad = pkg.loader.Model(None, m.configuration, m.model_type, t)
    with pytest.raises(pkg.native.B200Error, match=r"blk\.1\.attn_v\.bias") as e:
        pkg.B200MasterPlan.initialize_plan(bad)
    assert e.value.code == -1  # B200_ERR_BAD_ARG
    tt, dims, raw = t["blk.0.attn_k.bias"]
    t["blk.0.attn_k.bias"] = (tt, (int(dims[0]) // 2,), raw)  # wrong length
    t["blk.1.attn_v.bias"] = m.tensors["blk.1.attn_v.bias"]
    with pytest.raises(pkg.native.B200Error, match=r"blk\.0\.attn_k\.bias") as e:
        pkg.B200MasterPlan.initialize_plan(pkg.loader.Model(None, m.configuration, m.model_type, t))
    assert e.value.code == -1
    t["blk.0.attn_k.bias"] = (pkg.gguf.GGMLType.F16, dims, raw)  # not F32
    with pytest.raises(pkg.native.B200Error, match=r"blk\.0\.attn_k\.bias"):
        pkg.B200MasterPlan.initialize_plan(pkg.loader.Model(None, m.configuration, m.model_type, t))


# ---- the tensor-core prefill at GQA ratios that do not divide 64 ---------------------------------------------------------

ATT_STARTS = [0, 1, 63, 64, 65, 200]


@pytest.mark.parametrize("impl", ["mma"])
@pytest.mark.parametrize("kv_mul", [3, 5, 6, 7, 12])
def test_pf_attention_any_gqa_ratio_matches_float64(pkg, impl, kv_mul):
    """QT = floor(64 / kv_mul) query tokens per CTA: rows QT * kv_mul .. 63 are padding.  n around QT and across tiles, several
    start positions, both head sizes; rows >= n must come back untouched (the check inside _check_attention)."""
    n_kv = 2
    n_heads = n_kv * kv_mul
    qt = 64 // kv_mul
    worst = 0.0
    for j, n in enumerate(sorted({1, qt - 1, qt, qt + 1, 130, 300} - {0})):
        for hs in (64, 128):
            start = ATT_STARTS[(j + kv_mul + hs // 64) % len(ATT_STARTS)]
            for kind in ATT_KINDS:
                rng = np.random.default_rng(zlib.crc32(repr(("qwen2", kv_mul, n, start, hs, kind)).encode()))
                q, k, v = _attention_inputs(kind, n, start, n_heads, n_kv, hs, rng)
                what = f"{impl} kv_mul={kv_mul} hs={hs} n={n} start={start} {kind}"
                worst = max(worst, _check_attention(pkg, impl, q, k, v, n_heads, n_kv, start, kind, what))
    print(f"attention {impl} kv_mul={kv_mul}: worst |err| / bound = {worst:.3g}")


def _tc_prefill(pkg, orc, m, n_tok, batch, tol, mode="tensor_core"):
    """Prefill n_tok tokens in chunks through the tensor-core mode, then check the KV cache per layer and the next decode step's
    logits against the oracle; returns the plan's K/V caches."""
    c = m.configuration
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=batch)
    om = Qwen2Oracle(orc, m)
    try:
        if c.quantization == "Q8_0":
            plan.set_prefill_mode(mode)
        assert plan.prefill_info()[0] == {"tensor_core": 1, "tensor_core_w8a16": 2}[mode]
        toks = orc.bench_tokens(c.vocab_size, n_tok + 1)
        for off in range(0, n_tok, batch):
            plan.forward_batch_prefill(toks[off:min(off + batch, n_tok)], off)
        assert plan.prefill_info()[1] > 0
        for pos in range(n_tok):
            om.forward(int(toks[pos]), pos, want_logits=False)
        nv, nkv = n_tok * c.kv_dim, c.context_length * c.kv_dim
        caches = []
        for l in range(c.n_layers):
            for name, ref in (("key_cache", om.key_cache(l)), ("value_cache", om.value_cache(l))):
                got = plan.read_buffer(name, nkv, layer=l)
                err = np.max(np.abs(got[:nv] - ref[:nv])) / np.max(np.abs(ref[:nv]))
                print(f"{name} layer {l}: rel err {err:.2e}")
                assert err <= tol, f"{name} layer {l}: rel err {err:.2e}"
                assert not np.any(got[nv:]), f"{name} layer {l}: rows past the prompt were written"
                caches.append(got)
        lg, _ = plan.forward_decode(int(toks[n_tok]), n_tok)
        ref = om.forward(int(toks[n_tok]), n_tok)
        err = np.max(np.abs(lg - ref)) / np.max(np.abs(ref))
        print(f"logits after prefill: rel err {err:.2e}")
        assert err <= tol, f"logits after prefill: rel err {err:.2e}"
        return caches
    finally:
        plan.free()
        om.close()


@pytest.mark.parametrize("shape,n_tok,batch", [("tiny-qwen2", 70, 32), ("tiny-qwen2-gqa6", 45, 32), ("tiny-qwen2", 300, 300)])
def test_qwen2_tensor_core_prefill_fp16(pkg, orc, make_model, shape, n_tok, batch):
    m = make_model(shape, pkg.gguf.GGMLType.F16, n_tok + 8)
    _tc_prefill(pkg, orc, m, n_tok, batch, FP16_TOL)


@pytest.mark.parametrize("shape", ["tiny-qwen2", "tiny-qwen2-gqa6"])
def test_qwen2_tensor_core_prefill_q8_twin_and_w8a16(pkg, orc, make_model, shape):
    """Q8_0 plans: twin mode within the Q8_0 noise bar; W8A16 against twin mode -- layer 0's K/V bit-identical (no GEMM feeding
    it splits K), the later layers within FP16 tolerance (the W2 GEMM of these shapes splits K, whose reduce-add order is free)."""
    m = make_model(shape, pkg.gguf.GGMLType.Q8_0, 80)
    twin = _tc_prefill(pkg, orc, m, 70, 32, Q8_NOISE_TOL, "tensor_core")
    w8 = _tc_prefill(pkg, orc, m, 70, 32, Q8_NOISE_TOL, "tensor_core_w8a16")
    assert np.array_equal(w8[0].view(np.uint32), twin[0].view(np.uint32)) and np.array_equal(w8[1].view(np.uint32), twin[1].view(np.uint32))
    for a, b in zip(w8[2:], twin[2:]):
        assert np.max(np.abs(a - b)) <= FP16_TOL * np.max(np.abs(b))
