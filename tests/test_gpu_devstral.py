"""GPU tests of the Devstral 2 family (B200_ARCH_DEVSTRAL: Llama's forward with an independent head size and a YaRN RoPE table) through
the C ABI, against the CPU restatement of forwardJavaDevstral (tests/devstral_oracle.py).  Decode and the exact prefill are bit-exact
(logits compared as uint32, ids equal); the tensor-core prefill is held to the bars of tests/test_gpu_prefill.py.  Also: the exact
RMSNorm at dims above 8192 (the Devstral 2 123B geometry, 12288) and the exact sequential sum up to 16384 terms."""
import dataclasses

import numpy as np
import pytest

from devstral_oracle import DevstralOracle, rope_table
from test_gpu_parity import _seq, assert_bit_equal
from test_gpu_prefill import FP16_TOL, Q8_NOISE_TOL

pytestmark = pytest.mark.gpu


def _fast_model(pkg, sh, quant, ctx, seed=1234):
    if isinstance(sh, str):
        sh = pkg.synth.SHAPES[sh]
    return pkg.loader.model_from_tensors(sh, quant, pkg.synth.build_tensors_fast(sh, quant, seed=seed), ctx)


def _decode_vs_oracle(pkg, orc, m, n, mode="graph", lanes=16, tok=1):
    plan = pkg.B200MasterPlan.initialize_plan(m, fp16_lanes=lanes)
    plan.set_decode_mode(mode)
    assert plan.decode_info()[0] == {"graph": 0, "persistent": 1}[mode]
    om = DevstralOracle(orc, m, lanes=lanes)
    c = m.configuration
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


@pytest.mark.parametrize("shape", ["tiny-devstral", "tiny-devstral-wide", "tiny-devstral-plain"])
@pytest.mark.parametrize("quant,mode,lanes", [("Q8_0", "graph", 16), ("Q8_0", "persistent", 16), ("F16", "graph", 16), ("F16", "graph", 8),
                                              ("F16", "graph", 0)])
def test_devstral_decode_bit_exact(pkg, orc, make_model, shape, quant, mode, lanes):
    """qd 256 < dim 512 with YaRN, qd 512 > dim 256 with YaRN, and qd == dim with the plain table: the Q8_0 stream (graph and
    persistent), the FP16 rings at 16 and 8 lanes and the scalar FP16 species on the fallback matvec.  The plans are loaded with
    load_model from GGUF files on disk."""
    m = make_model(shape, getattr(pkg.gguf.GGMLType, quant), 24)
    assert m.model_type == "DEVSTRAL_2" and m.configuration.arch == pkg.loader.ARCH_DEVSTRAL
    assert (m.configuration.yarn is None) == (shape == "tiny-devstral-plain")
    _decode_vs_oracle(pkg, orc, m, 10, mode, lanes)


@pytest.mark.parametrize("shape", ["tiny-devstral", "tiny-devstral-plain", "mid-devstral-2"])
def test_devstral_rope_table_bit_equal(pkg, make_model, shape):
    """The device's rope_cr / rope_ci against the oracle's independent restatement of precomputeFreqsCisYaRN / precomputeFreqsCis."""
    G = pkg.gguf.GGMLType
    if shape.startswith("mid"):  # only the table matters: a 1-layer cut of the 123B geometry's attention
        sh = dataclasses.replace(pkg.synth.SHAPES[shape], n_layers=1, hidden=1024)
        m = _fast_model(pkg, sh, G.Q8_0, 4096)
    else:
        m = make_model(shape, G.Q8_0, 1024)
    c = m.configuration
    plan = pkg.B200MasterPlan.initialize_plan(m)
    try:
        n = c.context_length * c.head_size // 2
        cr, ci = rope_table(c.context_length, c.head_size, c.rope_theta, c.yarn)
        assert_bit_equal(plan.read_buffer("rope_cr", n), cr, "rope_cr")
        assert_bit_equal(plan.read_buffer("rope_ci", n), ci, "rope_ci")
    finally:
        plan.free()


def test_devstral_kquant_decodes_like_its_q8_0_twin(pkg, orc):
    G = pkg.gguf.GGMLType
    sh = pkg.synth.SHAPES["tiny-devstral"]
    tensors = pkg.synth.build_tensors_kquant(sh, seed=21)
    twin = {n: ((G.Q8_0, d, orc.kquant_to_q8_0(t, np.asarray(r), int(np.prod(d)))) if t in G.K_QUANTS else (t, d, r)) for n, (t, d, r) in tensors.items()}
    m = pkg.loader.model_from_tensors(sh, G.Q8_0, tensors, 24)
    mt = pkg.loader.model_from_tensors(sh, G.Q8_0, twin, 24)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = DevstralOracle(orc, mt)
    try:
        tok = 3
        for pos in range(10):
            lg, am = plan.forward_decode(tok, pos)
            ref = om.forward(tok, pos)
            assert_bit_equal(lg, ref, f"logits pos {pos}")
            assert am == orc.argmax(ref)
            tok = am
    finally:
        plan.free()
        om.close()


@pytest.mark.parametrize("mode", ["graph", "persistent"])
def test_devstral_long_context_bit_exact(pkg, orc, make_model, mode):
    """700 positions (past the YaRN table's original context of 256) through the device-resident loop: every greedy id, the last
    logits and a KV cache layer."""
    n = 700
    m = make_model("tiny-devstral", pkg.gguf.GGMLType.Q8_0, 720)
    c = m.configuration
    toks = orc.bench_tokens(c.vocab_size, n)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    plan.set_decode_mode(mode)
    om = DevstralOracle(orc, m)
    try:
        ids, _ = plan.decode_sequence(toks, n, 0)
        for pos in range(n):
            ref = om.forward(int(toks[pos]), pos)
            assert ids[pos] == orc.argmax(ref), f"argmax pos {pos}"
        assert_bit_equal(plan.read_buffer("logits", c.vocab_size), ref, "logits of the last step")
        assert_bit_equal(plan.read_buffer("key_cache", c.context_length * c.kv_dim, layer=1), om.key_cache(1), "key cache layer 1")
    finally:
        plan.free()
        om.close()


def test_devstral_exact_batch_prefill_kv_bit_identical(pkg, orc, make_model):
    m = make_model("tiny-devstral", pkg.gguf.GGMLType.Q8_0, 64)
    c = m.configuration
    toks = orc.bench_tokens(c.vocab_size, 45)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=16)
    om = DevstralOracle(orc, m)
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
        lg, _ = plan.forward_decode(int(toks[44]), 45)
        assert_bit_equal(lg, om.forward(int(toks[44]), 45), "logits after the exact prefill")
    finally:
        plan.free()
        om.close()


def _tc_prefill(pkg, orc, m, n_tok, batch, tol, mode="tensor_core"):
    """Tensor-core prefill of n_tok tokens, then K, V and the next step's logits against the oracle within tol of max|ref|."""
    c = m.configuration
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=batch)
    om = DevstralOracle(orc, m)
    try:
        if c.quantization == "Q8_0":
            plan.set_prefill_mode(mode)
        assert plan.prefill_info()[0] == {"tensor_core": 1, "tensor_core_w8a16": 2}[mode]
        toks = orc.bench_tokens(c.vocab_size, n_tok + 1)
        for off in range(0, n_tok, batch):
            plan.forward_batch_prefill(toks[off:min(off + batch, n_tok)], off)
        for pos in range(n_tok):
            om.forward(int(toks[pos]), pos, want_logits=False)
        nv, nkv = n_tok * c.kv_dim, c.context_length * c.kv_dim
        for l in range(c.n_layers):
            for name, ref in (("key_cache", om.key_cache(l)), ("value_cache", om.value_cache(l))):
                got = plan.read_buffer(name, nkv, layer=l)
                err = np.max(np.abs(got[:nv] - ref[:nv])) / np.max(np.abs(ref[:nv]))
                print(f"{mode} {name} layer {l}: rel err {err:.2e}")
                assert err <= tol, f"{name} layer {l}: rel err {err:.2e}"
        lg, _ = plan.forward_decode(int(toks[n_tok]), n_tok)
        ref = om.forward(int(toks[n_tok]), n_tok)
        err = np.max(np.abs(lg - ref)) / np.max(np.abs(ref))
        print(f"{mode} logits after prefill: rel err {err:.2e}")
        assert err <= tol, f"logits after prefill: rel err {err:.2e}"
    finally:
        plan.free()
        om.close()


@pytest.mark.parametrize("shape", ["tiny-devstral", "tiny-devstral-wide"])
def test_devstral_tensor_core_prefill_fp16(pkg, orc, make_model, shape):
    _tc_prefill(pkg, orc, make_model(shape, pkg.gguf.GGMLType.F16, 80), 70, 32, FP16_TOL)


@pytest.mark.parametrize("mode", ["tensor_core", "tensor_core_w8a16"])
def test_devstral_tensor_core_prefill_q8(pkg, orc, make_model, mode):
    _tc_prefill(pkg, orc, make_model("tiny-devstral", pkg.gguf.GGMLType.Q8_0, 80), 70, 32, Q8_NOISE_TOL, mode)


def test_devstral_device_sampler_at_vocab_131072(pkg, orc):
    sh = dataclasses.replace(pkg.synth.SHAPES["tiny-devstral"], vocab=131072)
    m = _fast_model(pkg, sh, pkg.gguf.GGMLType.Q8_0, 16)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = DevstralOracle(orc, m)
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


def _batched_vs_single(pkg, orc, m, n_rows, n_steps):
    """n_rows sequences in lockstep on their own slots (staggered starts): every row's logits bit-equal to its own oracle sequence."""
    c = m.configuration
    plan = pkg.B200MasterPlan.initialize_plan(m)
    oms = [DevstralOracle(orc, m) for _ in range(n_rows)]
    try:
        plan.set_decode_slots(n_rows)
        toks = [int(t) for t in orc.bench_tokens(c.vocab_size, n_rows)]
        for step in range(n_steps):
            rows = [r for r in range(n_rows) if step >= r % 3]
            pos = [step - r % 3 for r in rows]
            ids, lg = plan.forward_decode_batch(rows, [toks[r] for r in rows], pos, logits=True)
            for i, r in enumerate(rows):
                ref = oms[r].forward(toks[r], pos[i])
                assert_bit_equal(lg[i], ref, f"row {r} step {step}")
                assert ids[i] == orc.argmax(ref), f"row {r} step {step}"
                toks[r] = int(ids[i])
    finally:
        plan.free()
        for om in oms:
            om.close()


def test_devstral_batched_decode_4_rows(pkg, orc, make_model):
    _batched_vs_single(pkg, orc, make_model("tiny-devstral", pkg.gguf.GGMLType.Q8_0, 24), 4, 8)


def test_devstral_batched_decode_8_rows_at_small_2_cut(pkg, orc):
    _batched_vs_single(pkg, orc, _fast_model(pkg, "mid-devstral-small-2", pkg.gguf.GGMLType.Q8_0, 8), 8, 3)


def test_devstral_prefill_slots_then_batched_decode(pkg, orc, make_model):
    """Two prompts prefilled straight into decode slots (exact prefill), then one batched step: K/V and logits bit-equal."""
    m = make_model("tiny-devstral", pkg.gguf.GGMLType.Q8_0, 64)
    c = m.configuration
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=16)
    prompts = [[int(t) for t in orc.bench_tokens(c.vocab_size, 9, seed=s)] for s in (1, 2)]
    oms = [DevstralOracle(orc, m) for _ in prompts]
    try:
        plan.set_decode_slots(2)
        plan.prefill_slots([0, 1], [0, 0], prompts)
        for om, p in zip(oms, prompts):
            for pos, t in enumerate(p):
                om.forward(t, pos, want_logits=False)
        ids, lg = plan.forward_decode_batch([0, 1], [7, 11], [9, 9], logits=True)
        for i, (om, t) in enumerate(zip(oms, (7, 11))):
            ref = om.forward(t, 9)
            assert_bit_equal(lg[i], ref, f"slot {i}")
            assert ids[i] == orc.argmax(ref)
    finally:
        plan.free()
        for om in oms:
            om.close()


def test_devstral_decode_multi_and_lookahead(pkg, orc, make_model):
    """forward_decode_multi: every row bit-equal to the oracle at its position; generate_tokens_lookahead returns the greedy ids."""
    m = make_model("tiny-devstral", pkg.gguf.GGMLType.Q8_0, 64)
    c = m.configuration
    toks = [int(t) for t in orc.bench_tokens(c.vocab_size, 6)]
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = DevstralOracle(orc, m)
    try:
        assert plan.decode_multi_rows() >= len(toks)
        ids, lg = plan.forward_decode_multi(-1, toks, 0, logits=True)
        for pos, t in enumerate(toks):
            ref = om.forward(t, pos)
            assert_bit_equal(lg[pos], ref, f"row {pos}")
            assert ids[pos] == orc.argmax(ref)
        prompt = [3, 17, 40, 3, 17]
        om.reset()
        want, tok = [], prompt[0]
        for pos in range(20):
            ref = om.forward(tok, pos)
            tok = prompt[pos + 1] if pos + 1 < len(prompt) else orc.argmax(ref)
            if pos + 1 >= len(prompt):
                want.append(tok)
        plan.kv_reset()
        got = pkg.engine.generate_tokens_lookahead(plan, "DEVSTRAL_2", prompt[0], 0, prompt[1:], [], 20, 64)
        assert got == want[:len(got)] and len(got) >= 10
    finally:
        plan.free()
        om.close()


# ---- the Devstral-Small-2 and Devstral 2 123B layer geometries ----------------------------------------------------------------

@pytest.mark.parametrize("quant,mode", [("Q8_0", "graph"), ("Q8_0", "persistent"), ("F16", "graph")])
def test_devstral_small_2_cut_bit_exact(pkg, orc, quant, mode):
    """dim 5120, qd 4096, hidden 32768: the fused RMSNorm covers dims up to 5120, so the Q8_0 graph runs 5 launches per layer + 2."""
    m = _fast_model(pkg, "mid-devstral-small-2", getattr(pkg.gguf.GGMLType, quant), 16)
    if quant == "Q8_0" and mode == "graph":
        plan = pkg.B200MasterPlan.initialize_plan(m)
        try:
            L = m.configuration.n_layers
            print(f"mid-devstral-small-2 Q8_0: {plan.launches_per_decode} launches per decode step")
            assert plan.launches_per_decode == 5 * L + 2  # the fused norm
        finally:
            plan.free()
    _decode_vs_oracle(pkg, orc, m, 4, mode)


@pytest.mark.parametrize("quant", ["Q8_0", "F16"])
def test_devstral_2_cut_dim_12288_bit_exact(pkg, orc, quant):
    """dim 12288 (Devstral 2 123B): the exact RMSNorm above 8192.  The persistent kernel is refused with its reason and the graph
    (separate norm kernel: 7 launches per layer + 3 on Q8_0) is bit-exact."""
    G = pkg.gguf.GGMLType
    m = _fast_model(pkg, "mid-devstral-2", getattr(G, quant), 8)
    if quant == "Q8_0":
        plan = pkg.B200MasterPlan.initialize_plan(m)
        try:
            with pytest.raises(pkg.native.UnsupportedOperation, match="dim <= 8192"):
                plan.set_decode_mode("persistent")
            assert plan.decode_info()[0] == 0
            assert plan.launches_per_decode == 7 * m.configuration.n_layers + 3
        finally:
            plan.free()
    _decode_vs_oracle(pkg, orc, m, 3)


# ---- the exact sequential sum at the new widths ------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [12288, 16384])
@pytest.mark.parametrize("threads", [1024, 512, 256])
def test_seqsum2_up_to_16384_terms(pkg, n, threads):
    """seqsum2.cuh at n = 12288 and 16384 on benign and adversarial inputs (ties, binade edges, zeros, huge dynamic range, sums parked
    next to a power of two): bit-equal to the literal chain; 16385 terms are refused."""
    rng = np.random.default_rng(n + threads)
    cases = []
    for kind in range(10):
        if kind == 0: x = rng.standard_normal(n)
        elif kind == 1: x = rng.standard_normal(n) * 10.0 ** rng.integers(-6, 6)
        elif kind == 2: x = rng.standard_cauchy(n)
        elif kind == 3: x = np.full(n, rng.standard_normal())
        elif kind == 4: x = 2.0 ** rng.integers(-10, 10, n)
        elif kind == 5:
            x = rng.standard_normal(n); x[rng.integers(0, n, n // 4)] = 0
        elif kind == 6: x = rng.standard_normal(n) * np.exp(rng.standard_normal(n) * 3)
        elif kind == 7: x = np.round(rng.standard_normal(n) * 8) / 8
        elif kind == 8:
            x = np.zeros(n); x[n // 2:] = rng.standard_normal(n - n // 2)
        else:
            x = rng.standard_normal(n) * 1e-3; x[rng.integers(40, n)] = 1e3
        cases.append((x.astype(np.float32) ** 2).astype(np.float32))
    for eps in (-3e-7, -1e-7, 0.0, 1e-7, 3e-7):
        cases.append(np.full(n, (1.0 + eps) / n, dtype=np.float64).astype(np.float32))
    for t in cases:
        got = np.float32(pkg.native.test_seqsum(t, threads=threads))
        ref = _seq(t)
        assert got.view(np.uint32) == ref.view(np.uint32), (len(t), got, ref)
    with pytest.raises(pkg.native.B200Error):
        pkg.native.test_seqsum(np.ones(16385, np.float32), threads=threads)


# ---- refusals ---------------------------------------------------------------------------------------------------------------

def test_devstral_refusals(pkg, make_model):
    N = pkg.native
    m = make_model("tiny-devstral", pkg.gguf.GGMLType.Q8_0, 16)
    cfg = pkg.plan.make_config(m)
    good = dict(factor=4.0, beta_fast=32.0, beta_slow=1.0, log_multiplier=1.0, original_context_length=256)
    for name in ("factor", "beta_fast", "beta_slow", "log_multiplier"):
        for bad in (float("nan"), float("inf"), float("-inf")):
            with pytest.raises(N.B200Error, match=name) as e:
                N.NativePlan(cfg, m.tensors, 0, 0, devstral=True, yarn=N.YarnConfig(**{**good, name: bad}))
            assert e.value.code == -1
    for name, bad in (("factor", 0.0), ("factor", -2.0), ("original_context_length", 0), ("original_context_length", -5)):
        with pytest.raises(N.B200Error, match=name) as e:
            N.NativePlan(cfg, m.tensors, 0, 0, devstral=True, yarn=N.YarnConfig(**{**good, name: bad}))
        assert e.value.code == -1
    with pytest.raises(N.B200Error, match="b200_plan_create_devstral") as e:  # arch 6 through b200_plan_create
        N.NativePlan(cfg, m.tensors, 0, 0)
    assert e.value.code == -1
    cfg.arch = pkg.loader.ARCH_LLAMA  # the Devstral creator with another arch
    with pytest.raises(N.B200Error, match="B200_ARCH_DEVSTRAL") as e:
        N.NativePlan(cfg, m.tensors, 0, 0, devstral=True, yarn=N.YarnConfig(**good))
    assert e.value.code == -1
    with pytest.raises(N.B200Error, match="B200_ARCH_DEVSTRAL") as e:
        N.NativePlan(cfg, m.tensors, 0, 0, devstral=True)
    assert e.value.code == -1
    cfg.arch = pkg.loader.ARCH_LLAMA  # and the Llama check still refuses qd != dim for every family but Qwen3 and Devstral
    with pytest.raises(N.B200Error, match="n_heads\\*head_size must equal dim"):
        N.NativePlan(cfg, m.tensors, 0, 0)
