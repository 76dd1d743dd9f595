"""GPU tests of the W8A16 tensor-core prefill (B200_PREFILL_TENSOR_CORE_W8A16): the prefill GEMMs read B from the tile-major
Q8_0 stream and dequantise it to f16(q * d) in shared memory (csrc/prefill_gemm.cuh, BSRC = B_Q8).

With the same A, the same B values, the same wgmma sequence and the same k order the result must be bit-identical to the
f16-twin path (B200_PREFILL_TENSOR_CORE on a Q8_0 plan), which is therefore the reference here.  The one exception is the
reduce-add epilogue with K split over several CTAs: the order of the TMA f32 reduce-adds is not fixed in either path, so
there the float64 bound of test_gpu_prefill.py applies."""
import zlib

import numpy as np
import pytest

from test_gpu_prefill import FP16_TOL, GEMM_CASES, Q8_NOISE_TOL, U, F16_SENTINEL, F32_SENTINEL, _assert_within, _dequantised_f16_twin, _gemm_ref, _gemm_bound

pytestmark = pytest.mark.gpu

Q8_DEEP = 5  # the W8A16 ring's deep variant (6 stages do not fit next to the raw ring)


# ---- Q8_0 operands ------------------------------------------------------------------------------------------------

def _q8_blocks(rng, n, k):
    """GGUF Q8_0 blocks [n, k/32*34] with row scales spread over 2^-2 .. 2^2 (|w| ~ 1/sqrt(k)), and in every matrix: zero scales,
    subnormal scales, negative scales, and blocks of quants at -128, -127 and +127 (random quants cover the rest of [-128, 127])."""
    nb = k // 32
    q = rng.integers(-128, 128, size=(n, nb, 32)).astype(np.int8)
    d = (rng.uniform(0.5, 1.0, size=(n, nb)) * 2.0 ** rng.integers(-2, 3, size=(n, 1)) / np.sqrt(k) / 64).astype(np.float16)
    fd, fq = d.reshape(-1), q.reshape(-1, 32)
    per = max(1, fd.size // 16)
    sel = rng.permutation(fd.size)
    fd[sel[:per]] = np.float16(0.0)
    fd[sel[per:2 * per]] = rng.integers(1, 0x400, size=per).astype(np.uint16).view(np.float16)  # subnormal f16 scales
    fd[sel[2 * per:3 * per]] = -fd[sel[2 * per:3 * per]]
    fq[sel[3 * per:4 * per]] = -128
    fq[sel[4 * per:5 * per]] = 127
    fq[sel[5 * per:6 * per]] = -127
    fq[sel[6 * per:7 * per], ::2] = -128  # extremes next to each other inside one 8-quant chunk
    fq[sel[6 * per:7 * per], 1::2] = 127
    blocks = np.empty((n, nb, 34), dtype=np.uint8)
    blocks[:, :, :2] = d.view(np.uint8).reshape(n, nb, 2)
    blocks[:, :, 2:] = q.view(np.uint8)
    return blocks.reshape(n, nb * 34)


def _twin(blocks, k):
    """f16(q * d) of Q8_0 blocks, as k_tiles_to_f16 builds the twins (one rounding of the exact f32 product)."""
    b = np.ascontiguousarray(blocks).reshape(-1, 34)
    d = b[:, :2].copy().view("<f2").astype(np.float32)
    q = b[:, 2:].view(np.int8).astype(np.float32)
    return (q * d).astype(np.float16).reshape(blocks.shape[0], k)


def _a_operand(rng, m, k, m_valid):
    a = (rng.standard_normal((m, k)) * 2.0 ** rng.integers(-3, 4, size=(m, 1))).astype(np.float16)
    a[m_valid:] = np.float16(np.nan)
    return a


def _q8_case(pkg, mode, stages, splits, m, m_valid, n, k, seed):
    """W8A16 launch vs the f16 launch on the twins of the same blocks: bitwise where the k order is fixed, else the float64 bound."""
    rng = np.random.default_rng(seed)
    a = _a_operand(rng, m, k, m_valid)
    bq = _q8_blocks(rng, n, k)
    b = _twin(bq, k)
    q8_stages = Q8_DEEP if stages == 6 else stages
    what = f"w8a16 {mode} stages={q8_stages} splits={splits} M={m} m_valid={m_valid} N={n} K={k}"
    if mode == "gateup":
        bq2 = _q8_blocks(rng, n, k)
        c0 = np.full((m, n), F16_SENTINEL)
        got = pkg.native.test_gemm_q8(mode, a, bq, c0, bq2=bq2, m_valid=m_valid, stages=q8_stages)
        want = pkg.native.test_gemm(mode, a, b, c0, b2=_twin(bq2, k), m_valid=m_valid, stages=stages)
        assert np.array_equal(got.view(np.uint16), want.view(np.uint16)), f"{what}: differs from the twin path"
        assert np.array_equal(got[m_valid:].view(np.uint16), c0[m_valid:].view(np.uint16)), f"{what}: a row past m_valid was written"
        return
    if mode == "resid":
        c0 = (rng.uniform(0.5, 2.0, size=(m, n)) * rng.choice([-1.0, 1.0], size=(m, n)) * 2.0 ** rng.integers(-4, 2, size=(m, 1))).astype(np.float32)
    else:
        c0 = np.full((m, n), F32_SENTINEL)
    got = pkg.native.test_gemm_q8(mode, a, bq, c0, m_valid=m_valid, stages=q8_stages, splits=splits)
    if mode == "resid":
        assert np.array_equal(got[m_valid:].view(np.uint32), c0[m_valid:].view(np.uint32)), f"{what}: C0 changed in a row past m_valid"
    else:
        assert not np.any(got[m_valid:].view(np.uint32)), f"{what}: rows past m_valid are not +0"
    if mode == "resid" and splits > 1:
        ref, absprod = _gemm_ref(a[:m_valid], b)
        ref = ref + c0[:m_valid].astype(np.float64)
        bound = _gemm_bound(absprod, k) + (splits + 1) * U * (np.abs(c0[:m_valid].astype(np.float64)) + absprod)
        _assert_within(what, got[:m_valid], ref, bound)
        return
    want = pkg.native.test_gemm(mode, a, b, c0, m_valid=m_valid, stages=stages, splits=splits)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"{what}: differs from the twin path"


# ---- the GEMM ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode,stages,splits,m,m_valid,n,k", GEMM_CASES)
def test_gemm_q8_matches_twin_path(pkg, mode, stages, splits, m, m_valid, n, k):
    """Every GEMM_CASES row (6-stage rows run the W8A16 kernel at its deep ring, 5 stages: ring depth does not change the numbers)."""
    _q8_case(pkg, mode, stages, splits, m, m_valid, n, k, zlib.crc32(repr(("q8", mode, stages, splits, m, m_valid, n, k)).encode()))


# K spread over several stream segments, so the k-walk crosses segment boundaries inside the ring:
# 4096 = 2 x 2048, 14336 = 7 x 2048, 9728 = 4 x 2432 (the Llama-3-8B W2 and Qwen3-4B W2 widths)
@pytest.mark.parametrize("mode,stages,splits,m,m_valid,n,k", [
    ("f32", 4, 1, 128, 128, 128, 4096),
    ("f32", 6, 1, 128, 100, 256, 14336),
    ("f32", 4, 1, 128, 128, 128, 9728),
    ("gateup", 4, 1, 128, 77, 192, 4096),
    ("gateup", 6, 1, 128, 128, 64, 9728),
    ("resid", 4, 1, 128, 128, 128, 14336),
    ("resid", 6, 1, 128, 3, 128, 9728),
    ("resid", 4, 4, 128, 128, 256, 14336),
])
def test_gemm_q8_multi_segment(pkg, mode, stages, splits, m, m_valid, n, k):
    _q8_case(pkg, mode, stages, splits, m, m_valid, n, k, zlib.crc32(repr(("q8seg", mode, stages, splits, m, m_valid, n, k)).encode()))


def test_gemm_q8_hook_rejections(pkg):
    """A segment that is not a multiple of 64 columns (K = 2592: 3 segments of 864), K not a multiple of 64, and the split
    counts, row counts and ring depths b200_test_gemm rejects."""
    rng = np.random.default_rng(7)
    B200Error = pkg.native.B200Error
    c = np.zeros((128, 128), np.float32)
    for k in (2592, 288):
        with pytest.raises(B200Error) as e:
            pkg.native.test_gemm_q8("f32", _a_operand(rng, 128, k, 128), _q8_blocks(rng, 128, k), c)
        assert e.value.code == -1, k
    a, bq = _a_operand(rng, 128, 320, 128), _q8_blocks(rng, 128, 320)
    for mode, kw in (("f32", {"splits": 2}), ("gateup", {"splits": 2, "bq2": bq}), ("resid", {"splits": 4}),  # 5 k-blocks: 2+2+1+0
                     ("resid", {"m_valid": 0}), ("resid", {"m_valid": 129}), ("f32", {"stages": 6})):
        with pytest.raises(B200Error) as e:
            pkg.native.test_gemm_q8(mode, a, bq, c if mode != "gateup" else c.astype(np.float16), **kw)
        assert e.value.code == -1, (mode, kw)
    with pytest.raises(B200Error):
        pkg.native.test_gemm_q8("f32", a[:100], bq, c[:100])  # M not a multiple of 128


# ---- whole prefills ----------------------------------------------------------------------------------------------

def _prefill(plan, toks, batch):
    for off in range(0, len(toks), batch):
        plan.forward_batch_prefill(toks[off:off + batch], off)


def _snapshot(plan, c, n_last):
    """Every layer's K / V cache and the last chunk's rows of the f16 GEMM operands."""
    nkv, qd = c.context_length * c.kv_dim, c.n_heads * c.head_size
    bpad = (plan.prefill_batch_size + 127) // 128 * 128
    out = {}
    for l in range(c.n_layers):
        for name in ("key_cache", "value_cache"):
            out[f"{name}[{l}]"] = plan.read_buffer(name, nkv, layer=l)
    for name, width in (("pf_a16", c.dim), ("pf_att16", qd), ("pf_h16", c.hidden_dim)):
        out[name] = plan.read_buffer(name, bpad * width, dtype=np.float16).reshape(bpad, width)[:n_last]
    return out


def _run_modes(pkg, m, n_tok, batch, modes):
    c = m.configuration
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=batch)
    toks = np.random.default_rng(n_tok * 31 + batch).integers(0, c.vocab_size, n_tok).astype(np.int32)
    n_last = n_tok - (n_tok - 1) // batch * batch
    snaps = []
    try:
        assert plan.prefill_info()[0] == plan.PREFILL_EXACT
        for mode in modes:
            plan.set_prefill_mode(mode)
            assert plan.prefill_info()[0] == {"tensor_core": 1, "tensor_core_w8a16": 2}[mode]
            plan.kv_reset()
            _prefill(plan, toks, batch)
            snaps.append(_snapshot(plan, c, n_last))
    finally:
        plan.free()
    return snaps


def _kquant_tiny_llama(pkg):
    sh = pkg.synth.SHAPES["tiny-llama"]
    return pkg.loader.model_from_tensors(sh, pkg.gguf.GGMLType.Q8_0, pkg.synth.build_tensors_kquant(sh, seed=11, mix="Q4_K_M"), 64)


@pytest.mark.parametrize("shape,n_tok,batch,modes", [
    ("tiny-llama", 50, 16, ("tensor_core_w8a16", "tensor_core", "tensor_core_w8a16")),
    ("tiny-qwen3", 45, 32, ("tensor_core", "tensor_core_w8a16", "tensor_core")),
    ("kquant-tiny-llama", 40, 16, ("tensor_core_w8a16", "tensor_core")),
])
def test_w8a16_prefill_bit_equal_to_twin_mode(pkg, make_model, shape, n_tok, batch, modes):
    """Same plan, same chunks, both mode orders: every layer's KV cache and pf_a16 / pf_att16 / pf_h16 are bit-identical
    (these shapes run every residual GEMM unsplit: K / 64 < 16)."""
    m = _kquant_tiny_llama(pkg) if shape.startswith("kquant") else make_model(shape, pkg.gguf.GGMLType.Q8_0, 64)
    snaps = _run_modes(pkg, m, n_tok, batch, modes)
    for s in snaps[1:]:
        for name, ref in snaps[0].items():
            assert np.array_equal(s[name].view(np.uint16), ref.view(np.uint16)), f"{shape}: {name} differs between the modes"


def test_w8a16_prefill_phi3_fused_tensors(pkg, make_model):
    """Phi-3's fused qkv / gate-up source tensors.  Its W2 splits K two ways, so the bar is FP16_TOL against twin mode."""
    m = make_model("tiny-phi3-gqa", pkg.gguf.GGMLType.Q8_0, 64)
    w8, tw = _run_modes(pkg, m, 45, 32, ("tensor_core_w8a16", "tensor_core"))
    for name, ref in tw.items():
        if name.startswith(("key_cache", "value_cache")):
            ref64 = ref.astype(np.float64)
            err = np.max(np.abs(w8[name].astype(np.float64) - ref64)) / np.max(np.abs(ref64))
            assert err <= FP16_TOL, f"phi3 {name}: rel err {err:.2e} vs twin mode"


def test_w8a16_prefill_mid_llama(pkg, orc):
    """Llama-3-8B layer geometry (2 layers, split-K residual GEMMs, an 8-token tail): the bars of test_tensor_core_prefill_q8_model
    against the CPU oracle.  The next decode step's logits are held to Q8_NOISE_TOL against twin mode: the split-K reduce-add order
    is not fixed in either mode, and the Q8_0 decode step rounds its activations to int8, which turns last-bit KV differences into
    percent-level logit differences (twin mode against itself, run twice on an H100: 9.2e-3; W8A16 against twin mode: 9.3e-3)."""
    sh = pkg.synth.SHAPES["mid-llama"]
    Q8 = pkg.gguf.GGMLType.Q8_0
    m = pkg.loader.model_from_tensors(sh, Q8, pkg.synth.build_tensors_fast(sh, Q8, seed=1234), 144)
    c = m.configuration
    n_tok, batch = 136, 128
    toks = orc.bench_tokens(c.vocab_size, n_tok + 1)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=batch)
    om_twin = orc.OracleModel(_dequantised_f16_twin(pkg, m))
    om_q8 = orc.OracleModel(m)
    try:
        plan.set_prefill_mode("tensor_core_w8a16")
        _prefill(plan, toks[:n_tok], batch)
        for pos in range(n_tok):
            om_twin.forward(int(toks[pos]), pos, want_logits=False)
            om_q8.forward(int(toks[pos]), pos, want_logits=False)
        nv, nkv = n_tok * c.kv_dim, c.context_length * c.kv_dim
        worst_twin = worst_q8 = 0.0
        for l in range(c.n_layers):
            for name in ("key_cache", "value_cache"):
                got = plan.read_buffer(name, nkv, layer=l)[:nv]
                rt = (om_twin.key_cache(l) if name == "key_cache" else om_twin.value_cache(l))[:nv]
                rq = (om_q8.key_cache(l) if name == "key_cache" else om_q8.value_cache(l))[:nv]
                worst_twin = max(worst_twin, float(np.max(np.abs(got - rt)) / np.max(np.abs(rt))))
                worst_q8 = max(worst_q8, float(np.max(np.abs(got - rq)) / np.max(np.abs(rq))))
        assert worst_twin <= FP16_TOL, f"vs the oracle on the dequantised FP16 weights: rel err {worst_twin:.2e}"
        assert worst_q8 <= Q8_NOISE_TOL, f"vs the CPU path of the Q8_0 model: rel err {worst_q8:.2e}"
        lg_w8, _ = plan.forward_decode(int(toks[n_tok]), n_tok)
        lg_w8 = lg_w8.copy()
        plan.set_prefill_mode("tensor_core")
        plan.kv_reset()
        _prefill(plan, toks[:n_tok], batch)
        lg_tw, _ = plan.forward_decode(int(toks[n_tok]), n_tok)
        err = float(np.max(np.abs(lg_w8 - lg_tw)) / np.max(np.abs(lg_tw)))
        assert err <= Q8_NOISE_TOL, f"next-step logits vs twin mode: rel err {err:.2e}"
        print(f"w8a16 prefill mid-llama: {worst_twin:.2e} vs dequantised-FP16 oracle, {worst_q8:.2e} vs the Q8_0 CPU path, logits {err:.2e} vs twin mode")
    finally:
        plan.free()
        om_twin.close()
        om_q8.close()


def test_w8a16_allocates_only_the_prefill_scratch(pkg, make_model):
    """W8A16 adds the chunk scratch and nothing per weight, and nothing more on later chunks; twin mode afterwards adds the twins."""
    m = make_model("tiny-llama", pkg.gguf.GGMLType.Q8_0, 64)
    c = m.configuration
    batch = 32
    qd, kvd = c.n_heads * c.head_size, c.n_kv_heads * c.head_size
    nqkv, bpad = qd + 2 * kvd, (batch + 127) // 128 * 128
    scratch = bpad * (c.dim * 4 + nqkv * 4 + c.dim * 2 + qd * 2 + c.hidden_dim * 2 + 4) + 2 * c.context_length * kvd * 2
    twins = 2 * c.n_layers * (nqkv * c.dim + c.dim * qd + 2 * c.hidden_dim * c.dim + c.dim * c.hidden_dim)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=batch)
    try:
        b0 = plan.device_bytes
        plan.set_prefill_mode("tensor_core_w8a16")
        b1 = plan.device_bytes
        assert b1 - b0 == scratch, (b1 - b0, scratch)
        toks = np.arange(1, 60, dtype=np.int32)
        _prefill(plan, toks, batch)
        plan.set_prefill_mode("tensor_core_w8a16")
        _prefill(plan, toks[:20], batch)
        assert plan.device_bytes == b1
        plan.set_prefill_mode("tensor_core")
        assert plan.device_bytes - b1 == twins, (plan.device_bytes - b1, twins)
    finally:
        plan.free()


def test_w8a16_unsupported_is_loud(pkg, make_model):
    """Each unsupported plan raises with its reason and keeps running in exact mode."""
    G = pkg.gguf.GGMLType
    cases = [(make_model("tiny-llama", G.F16, 32), 16, "Q8_0 plan"), (make_model("tiny-llama", G.Q8_0, 32), 0, "prefill batch size"),
             (make_model("tiny-phi3", G.Q8_0, 32), 16, "head size")]
    for m, batch, why in cases:
        plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=batch)
        try:
            mode0 = plan.prefill_info()[0]
            with pytest.raises(Exception, match=why):
                plan.set_prefill_mode("tensor_core_w8a16")
            assert plan.prefill_info()[0] == mode0
            plan.set_prefill_mode("exact")
            plan.forward_batch_prefill(np.arange(1, 9, dtype=np.int32), 0)
            assert plan.prefill_info()[0] == plan.PREFILL_EXACT
        finally:
            plan.free()
