"""GPU tests of the bit-exact tensor-core prefill (B200_PREFILL_TENSOR_CORE_EXACT, csrc/prefill_i8.cuh): int8 wgmma GEMMs over the
chunk, each Q8_0 block's term fl(float(isum) * fl(wScale * aScale)) added in block order, so every comparison here is bitwise
(uint32 views): the GEMM against a float32 numpy restatement of Q8_0FloatTensor.dotQ8Activation, whole prefills against
B200_PREFILL_EXACT on a second plan (which the other suites hold to the CPU oracle)."""
import numpy as np
import pytest

import hostile
from test_gpu_prefill_w8a16 import _q8_blocks

pytestmark = pytest.mark.gpu


# ---- the GEMM ----------------------------------------------------------------------------------------------------------------

def _blocks(bq, k):
    b = np.ascontiguousarray(bq).reshape(bq.shape[0], k // 32, 34)
    return b[:, :, :2].copy().view("<f2").reshape(bq.shape[0], k // 32).astype(np.float32), b[:, :, 2:].view(np.int8).astype(np.int32)


def _dot_q8(aq, a_scales, bq):
    """result[i, j] = sum over blocks, from 0f in block order, of fl(float(isum) * fl(wScale * aScale)), all in float32, no FMA."""
    m, k = aq.shape
    d, q = _blocks(bq, k)
    a = aq.astype(np.int32).reshape(m, k // 32, 32)
    acc = np.zeros((m, bq.shape[0]), np.float32)
    for b in range(k // 32):
        isum = a[:, b, :] @ q[:, b, :].T
        acc = acc + isum.astype(np.float32) * (d[None, :, b] * a_scales[:, b, None])
    return acc


def _swiglu_q8(g, u):
    """swiglu_exact, then quant_block_lane per 32 units: (int8 [m][n], f32 scales [m][n/32])."""
    with np.errstate(over="ignore"):  # exp(-g) -> inf gives -0 for very negative g, as on the device; f16 scales may round to inf
        s = g / (1.0 + np.exp(-g.astype(np.float64))).astype(np.float32)
        h = (s * u).astype(np.float32)
        m, n = h.shape
        hb = h.reshape(m, n // 32, 32)
        qs = np.max(np.abs(hb), axis=2) / np.float32(127.0)
        ascale = qs.astype(np.float16).astype(np.float32)
    with np.errstate(divide="ignore"):
        ainv = np.where(qs != 0, np.float32(1.0) / qs, np.float32(0.0)).astype(np.float32)
    sc = hb * ainv[:, :, None]
    q = np.trunc(sc + np.copysign(np.float32(0.5), sc)).astype(np.int8)
    return q.reshape(m, n), ascale


def _activations(rng, m, k):
    """int8 quants over the full range and f16-representable scales, with all-zero blocks (quants and scale 0) mixed in."""
    aq = rng.integers(-128, 128, size=(m, k)).astype(np.int8)
    a_scales = (rng.uniform(0.5, 1.0, size=(m, k // 32)) * 2.0 ** rng.integers(-12, 3, size=(m, 1))).astype(np.float16).astype(np.float32)
    zero = rng.random((m, k // 32)) < 0.1
    a_scales[zero] = 0.0
    aq.reshape(m, k // 32, 32)[zero] = 0
    return aq, a_scales


def _weights(rng, n, k):
    """_q8_blocks' hostile blocks (d = 0, subnormal and negative d, q = -128, +-127) plus +-127 quants under a large d."""
    bq = _q8_blocks(rng, n, k)
    d, q = hostile.q8_split(bq)
    pick = rng.random(len(d)) < 0.03
    q[pick] = rng.choice(np.array([-127, 127], dtype=np.int8), (int(pick.sum()), 32))
    d[pick] = np.float16(8.0).view(np.uint16)
    return hostile.q8_raw(d, q).reshape(n, k // 32 * 34)


@pytest.mark.parametrize("m", [1, 63, 64, 130, 512])
@pytest.mark.parametrize("mode,n,k,oscale", [
    ("f32", 128, 256, 1.0), ("f32", 64, 4096, 1.0), ("f32", 64, 14336, 1.0),
    ("resid", 128, 256, 1.0), ("resid", 64, 4096, 0.22), ("resid", 64, 14336, 1.0),
    ("gateup", 64, 256, 1.0), ("gateup", 32, 4096, 1.0), ("gateup", 32, 14336, 1.0),
])
def test_gemm_i8_matches_dot_q8(pkg, m, mode, n, k, oscale):
    rng = np.random.default_rng(m * 1000003 + n * 101 + k + {"f32": 0, "resid": 1, "gateup": 2}[mode])
    aq, a_scales = _activations(rng, m, k)
    bq = _weights(rng, n, k)
    what = f"{mode} M={m} N={n} K={k} oscale={oscale}"
    if mode == "gateup":
        bq2 = _weights(rng, n, k)
        hq0, hs0 = np.full((m, n), 0x5A, np.int8), np.full((m, n // 32), np.nan, np.float32)
        hq, hs = pkg.native.test_gemm_i8(mode, aq, a_scales, bq, bq2=bq2, hq=hq0, hs=hs0)
        wq, ws = _swiglu_q8(_dot_q8(aq, a_scales, bq), _dot_q8(aq, a_scales, bq2))
        assert np.array_equal(hq, wq), f"{what}: quantised hidden rows differ"
        assert np.array_equal(hs.view(np.uint32), ws.view(np.uint32)), f"{what}: block scales differ"
        return
    c0 = (rng.standard_normal((m, n)) * 4).astype(np.float32) if mode == "resid" else np.full((m, n), np.nan, np.float32)
    got = pkg.native.test_gemm_i8(mode, aq, a_scales, bq, c=c0, oscale=oscale)
    acc = _dot_q8(aq, a_scales, bq)
    want = c0 + acc * np.float32(oscale) if mode == "resid" else acc
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"{what}: {int(np.sum(got.view(np.uint32) != want.view(np.uint32)))} elements differ"


def test_gemm_i8_hook_rejections(pkg):
    """A segment that is not a multiple of 64 columns (K = 2592: 3 segments of 864), K = 288, N not a multiple of 64 (32 for
    gate/up): B200_ERR_BAD_ARG."""
    rng = np.random.default_rng(5)
    for mode, n, k in (("f32", 64, 2592), ("f32", 64, 288), ("f32", 96, 256), ("resid", 32, 256), ("gateup", 48, 256)):
        aq, a_scales = _activations(rng, 8, k)
        bq = _q8_blocks(rng, n, k)
        with pytest.raises(pkg.native.B200Error) as e:
            pkg.native.test_gemm_i8(mode, aq, a_scales, bq, bq2=bq if mode == "gateup" else None)
        assert e.value.code == -1, (mode, n, k)


# ---- whole prefills ------------------------------------------------------------------------------------------------------------

def _kv(plan, c):
    nkv = c.context_length * c.kv_dim
    return [plan.read_buffer(n, nkv, layer=l) for n in ("key_cache", "value_cache") for l in range(c.n_layers)]


def _assert_same(a, b, what):
    assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32)), what


def _against_exact(pkg, m, batch, chunks, toks=None):
    """The same chunks through B200_PREFILL_EXACT on one plan and B200_PREFILL_TENSOR_CORE_EXACT on another: every layer's K / V,
    then the next decode step's logits and id, bit for bit."""
    c = m.configuration
    end = max(s + n for s, n in chunks)
    if toks is None:
        toks = np.random.default_rng(end * 7 + batch).integers(0, c.vocab_size, end + 1).astype(np.int32)
    pe = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=batch)
    pt = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=batch)
    try:
        pt.set_prefill_mode("tensor_core_exact")
        assert pt.prefill_info()[0] == pt.PREFILL_TENSOR_CORE_EXACT
        for s, n in chunks:
            pe.forward_batch_prefill(toks[s:s + n], s)
            pt.forward_batch_prefill(toks[s:s + n], s)
        for i, (a, b) in enumerate(zip(_kv(pe, c), _kv(pt, c))):
            _assert_same(b, a, f"{'KV'[i // c.n_layers]} cache layer {i % c.n_layers} differs from the exact prefill")
        lg_e, id_e = pe.forward_decode(int(toks[end]), end)
        lg_e = lg_e.copy()
        lg_t, id_t = pt.forward_decode(int(toks[end]), end)
        _assert_same(lg_t, lg_e, "next-step logits differ")
        assert id_t == id_e
        return pt.prefill_info()
    finally:
        pe.free()
        pt.free()


CHUNKS = [(0, 1), (1, 7), (8, 64), (72, 65), (137, 200), (600, 256)]


@pytest.mark.parametrize("shape", ["tiny-llama", "tiny-qwen3", "tiny-qwen2", "tiny-phi3", "tiny-phi3-gqa", "tiny-granite", "tiny-devstral"])
def test_prefill_bit_equal_to_exact(pkg, make_model, shape):
    """Chunks of 1, 7, 64, 65 and 200 tokens from position 0, then a chunk of prefill_batch_size tokens at 600."""
    info = _against_exact(pkg, make_model(shape, pkg.gguf.GGMLType.Q8_0, 1024), 256, CHUNKS)
    assert info[0] == 3 and info[1] > 0 and info[2] > 0


def test_prefill_kquant_on_q8_tiles(pkg):
    sh = pkg.synth.SHAPES["tiny-llama"]
    m = pkg.loader.model_from_tensors(sh, pkg.gguf.GGMLType.Q8_0, pkg.synth.build_tensors_kquant(sh, seed=11, mix="Q4_K_M"), 1024)
    _against_exact(pkg, m, 256, CHUNKS)


@pytest.mark.parametrize("shape", ["mid-llama", "mid-qwen3-4b", "mid-qwen2.5-7b"])
def test_prefill_mid_geometries(pkg, shape):
    sh = pkg.synth.SHAPES[shape]
    Q8 = pkg.gguf.GGMLType.Q8_0
    m = pkg.loader.model_from_tensors(sh, Q8, pkg.synth.build_tensors_fast(sh, Q8, seed=1234), 1024)
    _against_exact(pkg, m, 256, [(0, 65), (65, 200), (600, 256)])


def test_prefill_long_context_global_score_rows(pkg, make_model):
    """A context above 4096 keys: the attention's score rows live in global memory."""
    _against_exact(pkg, make_model("tiny-llama", pkg.gguf.GGMLType.Q8_0, 4352), 128, [(0, 64), (4200, 128)])


@pytest.mark.parametrize("kind", ["outlier", "extreme_q8"])
def test_prefill_hostile_values(pkg, kind):
    """The outlier / all-zero / binade-rotating embedding rows, and the hostile Q8_0 blocks in every tensor, through the whole model."""
    if kind == "outlier":
        m = hostile.outlier_embeddings("tiny-llama", pkg.gguf.GGMLType.Q8_0, ctx=128)
        toks = np.array(list(hostile.OUTLIER_TOKEN.values()) * 8, dtype=np.int32)
    else:
        m = hostile.extreme_q8_blocks("tiny-llama", ctx=128)
        toks = None
    n = 90 if toks is None else len(toks) - 1
    _against_exact(pkg, m, 64, [(0, 64), (64, n - 64)], toks)


def test_prefill_slots(pkg, make_model):
    """Three sequences of unequal length, two continuing earlier positions: each slot's K / V bit-equal to the same prompts through
    the exact prefill_slots on a second plan."""
    m = make_model("tiny-qwen2", pkg.gguf.GGMLType.Q8_0, 512)
    c = m.configuration
    rng = np.random.default_rng(3)
    calls = [([0, 1], [0, 0], [40, 13]), ([2, 0, 1], [0, 40, 13], [77, 9, 100])]
    plans = [pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=256) for _ in range(2)]
    try:
        plans[1].set_prefill_mode("tensor_core_exact")
        for p in plans:
            p.set_decode_slots(3)
        for slots, starts, lens in calls:
            lists = [rng.integers(0, c.vocab_size, n).astype(np.int32) for n in lens]
            for p in plans:
                p.prefill_slots(slots, starts, lists)
        nkv = c.context_length * c.kv_dim
        for s in range(3):
            for name in ("slot_key_cache", "slot_value_cache"):
                for l in range(c.n_layers):
                    _assert_same(plans[1].read_buffer(name, nkv, layer=s * c.n_layers + l), plans[0].read_buffer(name, nkv, layer=s * c.n_layers + l),
                                 f"slot {s} {name} layer {l}")
        assert plans[1].prefill_info()[0] == 3
    finally:
        for p in plans:
            p.free()


def test_generate_tokens_batch_prefill(pkg, make_model):
    """generate_tokens_batch_prefill in the new mode returns, per request, the ids of the exact mode."""
    m = make_model("tiny-llama", pkg.gguf.GGMLType.Q8_0, 96)
    E = pkg.engine
    reqs = [(1, 0, list(range(5, 25))), (2, 0, list(range(30, 37))), (3, 0, list(range(40, 52)))]
    out = {}
    for mode in ("exact", "tensor_core_exact"):
        plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=16)
        try:
            plan.set_prefill_mode(mode)
            plan.set_decode_slots(3)
            out[mode] = E.generate_tokens_batch_prefill(plan, m.model_type, reqs, [], 40, 96, 16)
        finally:
            plan.free()
    assert out["tensor_core_exact"] == out["exact"]


def test_refusals_and_mode_switching(pkg, make_model):
    """Every refusal names its reason, leaves the previous mode in force and the plan decoding; all four modes switch in any order on
    one plan, and each chunk afterwards matches the exact mode's."""
    G = pkg.gguf.GGMLType
    cases = [(make_model("tiny-llama", G.F16, 32), 16, "Q8_0 plan"), (make_model("tiny-llama", G.Q8_0, 32), 0, "prefill batch size"),
             (make_model("tiny-qwen2moe", G.Q8_0, 32), 16, "Qwen2-MoE")]
    for m, batch, why in cases:
        plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=batch)
        try:
            mode0 = plan.prefill_info()[0]
            with pytest.raises(Exception, match=why):
                plan.set_prefill_mode("tensor_core_exact")
            assert plan.prefill_info()[0] == mode0
            lg, _ = plan.forward_decode(3, 0)
            assert np.isfinite(lg).all()
        finally:
            plan.free()
    m = make_model("tiny-llama", G.Q8_0, 128)
    c = m.configuration
    toks = np.random.default_rng(9).integers(0, c.vocab_size, 40).astype(np.int32)
    ref = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=32)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=32)
    try:
        ref.forward_batch_prefill(toks[:32], 0)
        want = _kv(ref, c)
        for mode in ("tensor_core_exact", "tensor_core_w8a16", "tensor_core_exact", "exact", "tensor_core", "tensor_core_exact"):
            plan.set_prefill_mode(mode)
            assert plan.prefill_info()[0] == {"exact": 0, "tensor_core": 1, "tensor_core_w8a16": 2, "tensor_core_exact": 3}[mode]
            plan.kv_reset()
            plan.forward_batch_prefill(toks[:32], 0)
            if mode in ("exact", "tensor_core_exact"):
                for a, b in zip(_kv(plan, c), want):
                    _assert_same(a, b, f"{mode} after switching")
    finally:
        ref.free()
        plan.free()
