"""GPU tests of the Granite family (B200_ARCH_GRANITE: Llama's forward with four muP scales) through the C ABI, against the CPU
restatement of forwardGranite (tests/granite_oracle.py), and of classifiers whose vocabulary is not a multiple of 4 on every family.
Decode and the exact prefill are bit-exact (logits compared as uint32, ids equal); the tensor-core prefill is held to the bars of
tests/test_gpu_prefill.py."""
import numpy as np
import pytest

from granite_oracle import GraniteOracle
from test_gpu_parity import assert_bit_equal, set_mode
from test_gpu_prefill import FP16_TOL, Q8_NOISE_TOL

pytestmark = pytest.mark.gpu


def _fast_model(pkg, shape_name, quant, ctx, seed=1234):
    sh = pkg.synth.SHAPES[shape_name]
    return pkg.loader.model_from_tensors(sh, quant, pkg.synth.build_tensors_fast(sh, quant, seed=seed), ctx)


def _oracle(orc, m, lanes=16):
    if m.configuration.arch == 5:
        return GraniteOracle(orc, m, lanes=lanes)
    return orc.OracleModel(m, lanes=lanes)


def _decode_vs_oracle(pkg, orc, m, n, mode="graph", lanes=16, tok=1):
    plan = pkg.B200MasterPlan.initialize_plan(m, fp16_lanes=lanes)
    set_mode(pkg, plan, mode)
    om = _oracle(orc, m, lanes)
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


@pytest.mark.parametrize("shape", ["tiny-granite", "tiny-granite-gqa"])
@pytest.mark.parametrize("quant,mode,lanes", [("Q8_0", "graph", 16), ("Q8_0", "persistent", 16), ("F16", "graph", 16), ("F16", "graph", 8),
                                              ("F16", "graph", 0), ("F16", "graph", 4)])
def test_granite_decode_bit_exact(pkg, orc, make_model, shape, quant, mode, lanes):
    """Multi-head / head 64 / vocabulary 515 and GQA / head 128 / vocabulary 512: the Q8_0 stream (graph and persistent), the FP16 rings
    at 16 and 8 lanes and the scalar / 4-lane FP16 species on the fallback matvec."""
    m = make_model(shape, getattr(pkg.gguf.GGMLType, quant), 24)
    assert m.model_type == "GRANITE"
    _decode_vs_oracle(pkg, orc, m, 12, mode, lanes)


@pytest.mark.parametrize("shape", ["mid-granite-3-2b", "mid-granite-3-8b"])
@pytest.mark.parametrize("quant,mode", [("Q8_0", "graph"), ("Q8_0", "persistent"), ("F16", "graph")])
def test_granite_mid_geometries_bit_exact(pkg, orc, shape, quant, mode):
    """2-layer cuts of the Granite-3.x-2B and -8B layer geometries with the 49155-token vocabulary."""
    m = _fast_model(pkg, shape, getattr(pkg.gguf.GGMLType, quant), 16)
    assert m.configuration.vocab_size == 49155
    _decode_vs_oracle(pkg, orc, m, 5, mode)


def test_granite_kquant_decodes_like_its_q8_0_twin(pkg, orc):
    G = pkg.gguf.GGMLType
    sh = pkg.synth.SHAPES["tiny-granite-gqa"]
    tensors = pkg.synth.build_tensors_kquant(sh, seed=21)
    twin = {n: ((G.Q8_0, d, orc.kquant_to_q8_0(t, np.asarray(r), int(np.prod(d)))) if t in G.K_QUANTS else (t, d, r)) for n, (t, d, r) in tensors.items()}
    m = pkg.loader.model_from_tensors(sh, G.Q8_0, tensors, 24)
    mt = pkg.loader.model_from_tensors(sh, G.Q8_0, twin, 24)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = GraniteOracle(orc, mt)
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
def test_granite_long_context_bit_exact(pkg, orc, make_model, mode):
    """700 positions through the device-resident loop: every greedy id, the last logits and a KV cache layer."""
    n = 700
    m = make_model("tiny-granite", pkg.gguf.GGMLType.Q8_0, 720)
    c = m.configuration
    toks = orc.bench_tokens(c.vocab_size, n)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    set_mode(pkg, plan, mode)
    om = GraniteOracle(orc, m)
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


def test_granite_exact_batch_prefill_kv_bit_identical(pkg, orc, make_model):
    m = make_model("tiny-granite-gqa", pkg.gguf.GGMLType.Q8_0, 64)
    c = m.configuration
    toks = orc.bench_tokens(c.vocab_size, 45)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=16)
    om = GraniteOracle(orc, m)
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


def _tc_prefill(pkg, orc, m, n_tok, batch, tol, mode="tensor_core"):
    """Tensor-core prefill of n_tok tokens, then K, V and the next step's logits against the oracle within tol of max|ref|."""
    c = m.configuration
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=batch)
    om = GraniteOracle(orc, m)
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


@pytest.mark.parametrize("shape", ["tiny-granite", "tiny-granite-gqa"])
def test_granite_tensor_core_prefill_fp16(pkg, orc, make_model, shape):
    _tc_prefill(pkg, orc, make_model(shape, pkg.gguf.GGMLType.F16, 80), 70, 32, FP16_TOL)


@pytest.mark.parametrize("mode", ["tensor_core", "tensor_core_w8a16"])
def test_granite_tensor_core_prefill_q8(pkg, orc, make_model, mode):
    _tc_prefill(pkg, orc, make_model("tiny-granite-gqa", pkg.gguf.GGMLType.Q8_0, 80), 70, 32, Q8_NOISE_TOL, mode)


def test_granite_device_sampler_at_vocab_49155(pkg, orc):
    m = _fast_model(pkg, "mid-granite-3-2b", pkg.gguf.GGMLType.Q8_0, 16)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = GraniteOracle(orc, m)
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
    oms = [_oracle(orc, m) for _ in range(n_rows)]
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


def test_granite_batched_decode_tiny(pkg, orc, make_model):
    _batched_vs_single(pkg, orc, make_model("tiny-granite", pkg.gguf.GGMLType.Q8_0, 24), 4, 8)


def test_granite_batched_decode_8_rows_at_8b_cut(pkg, orc):
    _batched_vs_single(pkg, orc, _fast_model(pkg, "mid-granite-3-8b", pkg.gguf.GGMLType.Q8_0, 8), 8, 4)


def test_granite_generate_tokens_stops(pkg, orc, make_model):
    """engine.loop_for("GRANITE") is the Llama loop: prompt, then greedy ids until a stop token (the oracle's 4th id)."""
    m = make_model("tiny-granite", pkg.gguf.GGMLType.Q8_0, 32)
    om = GraniteOracle(orc, m)
    prompt = [3, 17, 40]
    want, tok = [], prompt[0]
    for pos in range(12):
        ref = om.forward(tok, pos)
        tok = prompt[pos + 1] if pos + 1 < len(prompt) else orc.argmax(ref)
        if pos + 1 >= len(prompt):
            want.append(tok)
    om.close()
    stop = want[3]
    plan = pkg.B200MasterPlan.initialize_plan(m)
    loop = pkg.engine.loop_for("GRANITE")
    assert loop is pkg.engine.generate_tokens_llama
    try:
        got = loop(lambda t, p: plan.forward_decode(t, p, logits=False)[1], prompt[0], 0, prompt[1:], [stop], 20, 32)
    finally:
        plan.free()
    assert got == want[:want.index(stop) + 1]


# ---- vocabularies that are not a multiple of 4 --------------------------------------------------------------------------------

def test_odd_vocab_llama_streams_its_classifier(pkg, orc, make_model):
    """A Llama plan with vocabulary 509 streams its classifier in a zero-padded last group: the persistent kernel and decode slots
    are available; its logits stay bit-equal in both decode modes."""
    m = make_model("tiny-llama-vocab509", pkg.gguf.GGMLType.Q8_0, 24)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    try:
        plan.set_decode_mode("persistent")
        plan.set_decode_slots(8)
    finally:
        plan.free()
    _decode_vs_oracle(pkg, orc, m, 10, "graph")
    _decode_vs_oracle(pkg, orc, m, 10, "persistent")


def _all_negative_classifier(pkg, quant):
    """Llama, vocabulary 509: Wo = W2 = 0 (x stays the embedding row, whose element 0 is 1 for every token), the final norm keeps only
    element 0, and classifier column 0 is negative for every row -- every real logit is negative, the least negative being row 507.
    A padding row's 0 would win any argmax that let it in."""
    G = pkg.gguf.GGMLType
    sh = pkg.synth.SHAPES["tiny-llama-vocab509"]
    t = {n: (tt, d, raw) for n, tt, d, raw in pkg.synth.build_tensors(sh, quant, 99, 0.0)}
    V, D = sh.vocab, sh.dim
    for n in list(t):
        if n.endswith("attn_output.weight") or n.endswith("ffn_down.weight"):
            tt, d, _ = t[n]
            t[n] = (tt, d, pkg.synth.encode(np.zeros(int(np.prod(d)), np.float32), tt))
    rng = np.random.default_rng(5)
    emb = (rng.standard_normal((V, D)) * 0.5).astype(np.float32)
    emb[:, 0] = 1.0
    t["token_embd.weight"] = (quant, (D, V), pkg.synth.encode(emb.reshape(-1), quant))
    nw = np.zeros(D, np.float32)
    nw[0] = 1.0
    t["output_norm.weight"] = (G.F32, (D,), nw.view(np.uint8))
    out = np.zeros((V, D), np.float32)
    out[:, 0] = -1.0 - np.arange(V, dtype=np.float32) % 7 * 0.125
    out[V - 2, 0] = -0.5
    t["output.weight"] = (quant, (D, V), pkg.synth.encode(out.reshape(-1), quant))
    return pkg.loader.model_from_tensors(sh, quant, t, 16)


@pytest.mark.parametrize("quant,mode", [("Q8_0", "graph"), ("Q8_0", "persistent"), ("Q8_0", "batched"), ("F16", "graph")])
def test_padding_rows_never_win_the_argmax(pkg, orc, quant, mode):
    m = _all_negative_classifier(pkg, getattr(pkg.gguf.GGMLType, quant))
    V = m.configuration.vocab_size
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = orc.OracleModel(m)
    try:
        if mode == "batched":
            plan.set_decode_slots(2)
        else:
            set_mode(pkg, plan, mode)
        for pos, tok in enumerate([1, 77, 300]):
            ref = om.forward(tok, pos)
            assert ref.max() < 0 and orc.argmax(ref) == V - 2
            if mode == "batched":
                ids, lg = plan.forward_decode_batch([0, 1], [tok, tok], [pos, pos], logits=True)
                for i in range(2):
                    assert_bit_equal(lg[i], ref, f"row {i} pos {pos}")
                assert list(ids) == [V - 2, V - 2]
            else:
                lg, am = plan.forward_decode(tok, pos)
                assert_bit_equal(lg, ref, f"logits pos {pos}")
                assert am == V - 2
    finally:
        plan.free()
        om.close()


# ---- refusals ---------------------------------------------------------------------------------------------------------------

def test_granite_refusals(pkg, make_model):
    N = pkg.native
    m = make_model("tiny-granite", pkg.gguf.GGMLType.Q8_0, 16)
    cfg = pkg.plan.make_config(m)
    good = dict(embedding_scale=12.0, residual_scale=0.22, attention_scale=0.03, logit_scale=0.3)
    for name in good:
        for bad in (float("nan"), float("inf"), float("-inf")):
            g = N.GraniteConfig(**{**good, name: bad})
            with pytest.raises(N.B200Error, match=name) as e:
                N.NativePlan(cfg, m.tensors, 0, 0, granite=g)
            assert e.value.code == -1
    with pytest.raises(N.B200Error, match="b200_plan_create_granite") as e:  # arch 5 without its scales
        N.NativePlan(cfg, m.tensors, 0, 0)
    assert e.value.code == -1
    cfg.arch = pkg.loader.ARCH_LLAMA  # the Granite creator with another arch
    with pytest.raises(N.B200Error, match="B200_ARCH_GRANITE") as e:
        N.NativePlan(cfg, m.tensors, 0, 0, granite=N.GraniteConfig(**good))
    assert e.value.code == -1
