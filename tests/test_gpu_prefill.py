"""GPU tests of the tensor-core batched prefill (csrc/prefill.cuh, csrc/prefill_gemm.cuh) through the C ABI.

This is the one floating-point path that is NOT bit-exact, by design: activations are rounded to FP16 before each GEMM,
as in the reference's MMA prefill (TransformerBatchPrefillKernels.java:61,792-915).  Each kernel is held to a bound
derived from its own arithmetic, elementwise, against a float64 evaluation of the same operation on the same inputs:
  * GEMM (wgmma, f16 x f16 -> f32): |c - ref| <= K * 2^-23 * (|A| |B|^T)_ij -- products of f16 values are exact in
    f32, and the factor 2 over the round-to-nearest bound K * 2^-24 covers an accumulator that truncates.  The
    reduce-add epilogue adds (splits + 1) * 2^-24 * (|C0| + |A| |B|^T); the gate/up epilogue carries the accumulation
    bounds of g and u through silu (|silu'| <= 1.1), its own f32 arithmetic, and one f16 rounding.
  * attention (mma.sync, f16 Q / K / V / P, ex2.approx): against softmax attention on the kernel's rounded inputs, in
    log2 units; the bound sums the f16 output rounding, P rounded to f16 while l is not, the f32 score accumulation
    (a relative error of p), ex2.approx, and the f32 sums of l and P V.
  * every stage of the last layer of a real prefill chunk, against float64 evaluated from that stage's own inputs
    read back from the device, at the kernel bounds above.
Every kernel test prints its worst error / bound ratio.  The model-level tests then bound what all of it adds up to:
  * KV cache after prefill and the logits of the following decode step vs the CPU oracle:
    max|err| <= 2^-8 * max|ref| (SURVEY.md 8d "FP16-scale tolerance"; measured 2e-4 .. 1.2e-3)."""
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

FP16_TOL = 2.0 ** -8
Q8_NOISE_TOL = 0.03  # Q8_0 model vs the CPU path itself: the CPU path's own int8 activation rounding (measured 0.5-2.5 %), reported, not the parity bar
LOG2E = 1.4426950408889634
SILU_LIP = 1.1  # max |silu'(x)| = 1.0998
U = 2.0 ** -24  # f32 unit roundoff


# ---- float64 references and their bounds --------------------------------------------------------------------------

def _half_ulp_f16(x):
    """Half an f16 ulp at magnitude x (x >= 0), with the subnormal floor 2^-25."""
    e = np.floor(np.log2(np.maximum(x, 2.0 ** -14)))
    return 2.0 ** (e - 11)


def _gemm_ref(a, b):
    """(A B^T, |A| |B|^T) in float64 of f16 operands a [M,K], b [N,K]."""
    a64 = a.astype(np.float64)
    prod, absprod = np.empty((a.shape[0], b.shape[0])), np.empty((a.shape[0], b.shape[0]))
    for r in range(0, b.shape[0], 2048):  # bounded host memory at the 8B FFN width
        b64 = b[r:r + 2048].astype(np.float64)
        prod[:, r:r + 2048], absprod[:, r:r + 2048] = a64 @ b64.T, np.abs(a64) @ np.abs(b64).T
    return prod, absprod


def _gemm_bound(absprod, k):
    return k * 2.0 ** -23 * absprod


def _gateup_ref(a, w1, w3):
    """(f64 silu(a W1^T) * (a W3^T), elementwise bound of the kernel's f16 result)."""
    k = a.shape[1]
    g, ga = _gemm_ref(a, w1)
    u, ua = _gemm_ref(a, w3)
    eg, eu = _gemm_bound(ga, k), _gemm_bound(ua, k)
    with np.errstate(over="ignore"):
        sg = g / (1.0 + np.exp(-g))
    h = sg * u
    e_acc = SILU_LIP * eg * (np.abs(u) + eu) + np.abs(sg) * eu  # the accumulation errors of g and u carried through silu(g) * u
    e_f32 = 8 * U * (np.abs(h) + e_acc)                          # expf, 1 + e, the division and the product in f32
    return h, e_acc + e_f32 + _half_ulp_f16(np.abs(h) + e_acc + e_f32)


def _report(what, err, bound):
    ratio = float(np.max(err / bound)) if err.size else 0.0
    print(f"{what}: worst |err| / bound = {ratio:.3g}")
    return ratio


def _assert_within(what, got, ref, bound):
    assert not np.any(np.isnan(got)), f"{what}: NaN in the result"
    err = np.abs(got.astype(np.float64) - ref)
    ratio = _report(what, err, bound)
    if ratio > 1.0:
        i = np.unravel_index(np.argmax(err / bound), err.shape)
        raise AssertionError(f"{what}: |err| / bound = {ratio:.3g} at {i}: got {got[i]!r}, ref {ref[i]!r}, bound {bound[i]:.3g}")
    return ratio


# ---- the GEMM building block --------------------------------------------------------------------------------------

@pytest.mark.parametrize("m,n,k", [(128, 128, 64), (256, 384, 512), (384, 1024, 2240)])
def test_gemm_f16_timing_entry_matches_float64(pkg, m, n, k):
    """b200_gemm_f16 (the stand-alone timing entry, F32 epilogue) returns the product it timed."""
    rng = np.random.default_rng(m + n + k)
    a = (rng.standard_normal((m, k)) * 0.5).astype(np.float16)
    b = (rng.standard_normal((n, k)) * 0.5).astype(np.float16)
    ref, absprod = _gemm_ref(a, b)
    c, ms = pkg.native.gemm_f16(a, b, iters=2)
    _assert_within(f"gemm_f16 {m}x{n}x{k}", c, ref, _gemm_bound(absprod, k))
    assert ms > 0


def test_gemm_rejects_ragged_shapes(pkg):
    a = np.zeros((100, 64), dtype=np.float16)
    b = np.zeros((128, 64), dtype=np.float16)
    with pytest.raises(Exception):
        pkg.native.gemm_f16(a, b)


# (mode, ring stages, K splits, M, m_valid, N, K).  nk = K / 64 k-blocks: 1, 3 (fewer than the stages), = stages, and
# 20 / 32 (the ring wraps several times); splits 2-4 with a short last split (448 = 7 blocks -> 4+3, 3+3+1, 2+2+2+1);
# m_valid = M, M - 1, 1 and 129 of 256; gate/up with an odd count of 64-column tiles.
GEMM_CASES = [
    ("f32", 4, 1, 128, 128, 128, 64),
    ("f32", 4, 1, 256, 129, 384, 192),
    ("f32", 4, 1, 256, 256, 256, 256),
    ("f32", 6, 1, 128, 127, 256, 384),
    ("f32", 4, 1, 128, 1, 256, 1280),
    ("f32", 6, 1, 256, 256, 128, 1280),
    ("resid", 4, 1, 128, 128, 128, 64),
    ("resid", 4, 2, 128, 128, 128, 384),
    ("resid", 4, 2, 256, 129, 256, 448),
    ("resid", 4, 3, 128, 127, 128, 448),
    ("resid", 6, 4, 128, 1, 256, 448),
    ("resid", 6, 3, 256, 256, 128, 1280),
    ("resid", 4, 4, 128, 128, 384, 2048),
    ("gateup", 4, 1, 128, 128, 192, 64),
    ("gateup", 4, 1, 256, 129, 320, 192),
    ("gateup", 4, 1, 128, 128, 128, 256),
    ("gateup", 6, 1, 128, 127, 64, 384),
    ("gateup", 4, 1, 128, 1, 192, 1280),
    ("gateup", 6, 1, 256, 256, 448, 1280),
]
F32_SENTINEL = np.float32(-1234.5)
F16_SENTINEL = np.float16(-1234.0)


def _gemm_operands(rng, m, n, k, m_valid):
    """f16 operands with row scales spread over 2^-3 .. 2^3 (A) and 2^-2 .. 2^2 (B); A's rows >= m_valid are NaN."""
    a = rng.standard_normal((m, k)) * 2.0 ** rng.integers(-3, 4, size=(m, 1))
    b = rng.standard_normal((n, k)) * 2.0 ** rng.integers(-2, 3, size=(n, 1)) / np.sqrt(k)
    a = a.astype(np.float16)
    a[m_valid:] = np.float16(np.nan)
    return a, b.astype(np.float16)


@pytest.mark.parametrize("mode,stages,splits,m,m_valid,n,k", GEMM_CASES)
def test_gemm_modes_match_float64(pkg, mode, stages, splits, m, m_valid, n, k):
    """One launch of pg::gemm_launch<mode, stages> per case, elementwise against float64.  Rows past m_valid hold NaN in A:
    F32 must store +0 there, RESID must leave C0 bit for bit, GATEUP must not write (the sentinel stays)."""
    rng = np.random.default_rng(zlib.crc32(repr((mode, stages, splits, m, m_valid, n, k)).encode()))
    a, b = _gemm_operands(rng, m, n, k, m_valid)
    what = f"{mode} stages={stages} splits={splits} M={m} m_valid={m_valid} N={n} K={k}"
    if mode == "gateup":
        b2 = (rng.standard_normal((n, k)) * 2.0 ** rng.integers(-2, 3, size=(n, 1)) / np.sqrt(k)).astype(np.float16)
        c = pkg.native.test_gemm(mode, a, b, np.full((m, n), F16_SENTINEL), b2=b2, m_valid=m_valid, stages=stages, splits=splits)
        ref, bound = _gateup_ref(a[:m_valid], b, b2)
        _assert_within(what, c[:m_valid], ref, bound)
        assert np.array_equal(c[m_valid:].view(np.uint16), np.full((m - m_valid, n), F16_SENTINEL).view(np.uint16)), f"{what}: a row past m_valid was written"
        return
    ref, absprod = _gemm_ref(a[:m_valid], b)
    bound = _gemm_bound(absprod, k)
    if mode == "resid":
        c0 = rng.uniform(0.5, 2.0, size=(m, n)) * rng.choice([-1.0, 1.0], size=(m, n)) * 2.0 ** rng.integers(-4, 2, size=(m, 1))
        c0 = c0.astype(np.float32)
        c = pkg.native.test_gemm(mode, a, b, c0, m_valid=m_valid, stages=stages, splits=splits)
        ref = ref + c0[:m_valid].astype(np.float64)
        bound = bound + (splits + 1) * U * (np.abs(c0[:m_valid].astype(np.float64)) + absprod)
        assert np.array_equal(c[m_valid:].view(np.uint32), c0[m_valid:].view(np.uint32)), f"{what}: C0 changed in a row past m_valid"
    else:
        c = pkg.native.test_gemm(mode, a, b, np.full((m, n), F32_SENTINEL), m_valid=m_valid, stages=stages, splits=splits)
        assert not np.any(c[m_valid:].view(np.uint32)), f"{what}: rows past m_valid are not +0"
    _assert_within(what, c[:m_valid], ref, bound)


def test_gemm_hook_rejections(pkg):
    """Split-K only for the reduce-add epilogue, no split without a k-block, whole tiles only."""
    rng = np.random.default_rng(5)
    a, b = _gemm_operands(rng, 128, 128, 320, 128)
    c = np.zeros((128, 128), np.float32)
    B200Error = pkg.native.B200Error
    for mode, kw in (("f32", {"splits": 2}), ("gateup", {"splits": 2, "b2": b}), ("resid", {"splits": 4}),  # 5 k-blocks: 2+2+1+0
                     ("resid", {"m_valid": 0}), ("resid", {"m_valid": 129}), ("f32", {"stages": 5})):
        with pytest.raises(B200Error) as e:
            pkg.native.test_gemm(mode, a, b, c if mode != "gateup" else c.astype(np.float16), **kw)
        assert e.value.code == -1, (mode, kw)
    with pytest.raises(B200Error):
        pkg.native.test_gemm("f32", a[:, :300], b[:, :300], c)  # K not a multiple of 64
    with pytest.raises(B200Error):
        pkg.native.test_gemm("f32", a, b[:96], c[:, :96])  # N not a multiple of 128
    with pytest.raises(B200Error):
        pkg.native.test_gemm("f32", a[:100], b, c[:100])  # M not a multiple of 128


# ---- causal attention over one chunk -------------------------------------------------------------------------------

def _attention_ref(q, k, v, n_heads, n_kv, start, equal_scores=False):
    """(float64 causal softmax attention, elementwise bound of the kernel's f16 output) for queries at start .. start+n-1.

    The inputs are rounded as k_pf_attention_mma_packed rounds them -- qh = f16(f32(q) * f32(inv_sqrt_hs * log2e)),
    kh = f16(k), vh = f16(v) -- and scores are in log2 units.
    The bound, with vmax = max |v| over the row's visible keys:
      2^-11 |ref| + 2^-25           the f16 output rounding (subnormal floor)
      2^-10 vmax                     P rounded to f16 while l is summed unrounded
      2 (e^eps - 1) e^eps vmax       a relative error eps of every p: the f32 score accumulation, hs * 2^-23 * max sum|q||k|
                                     (times ln 2 in log2 units), plus 2^-21 for ex2.approx
      (3 keys + 64) 2^-23 vmax       the f32 sums of l and of P V, the rescales, the final 1 / l, the f32 rounding of s - m.
    equal_scores: every visible score of a row is the same f32 value, so every p is 2^0 (within ex2's error) and f16(p) = 1:
    only the ex2 share of eps and the f32 sums remain."""
    n, qd = q.shape
    hs = qd // n_heads
    kv_mul, nk = n_heads // n_kv, start + n
    inv = np.float32(1.0 / np.sqrt(hs))
    qh = (q * np.float32(inv * np.float32(LOG2E))).astype(np.float16).astype(np.float64)
    kh, vh = k.astype(np.float16).astype(np.float64), v.astype(np.float16).astype(np.float64)
    ln_base = np.log(2.0)
    pos = start + np.arange(n)
    visible = np.arange(nk)[None, :] <= pos[:, None]
    ref, bound = np.empty((n, qd)), np.empty((n, qd))
    e_p16 = 0.0 if equal_scores else 2.0 ** -10
    e_sums = (3 * (pos + 1) + 64) * 2.0 ** -23
    for g in range(n_kv):
        kg, vg = kh[:, g * hs:(g + 1) * hs], vh[:, g * hs:(g + 1) * hs]
        vmax = np.maximum.accumulate(np.abs(vg).max(axis=1))[pos]
        for h in range(g * kv_mul, (g + 1) * kv_mul):
            qg = qh[:, h * hs:(h + 1) * hs]
            s = np.where(visible, qg @ kg.T, -np.inf)
            p = np.exp(ln_base * (s - s.max(axis=1, keepdims=True)))
            o = (p @ vg) / p.sum(axis=1, keepdims=True)
            eps = 2.0 ** -21 + (0.0 if equal_scores else ln_base * hs * 2.0 ** -23 * np.where(visible, np.abs(qg) @ np.abs(kg).T, 0.0).max(axis=1))
            e_rel = 2 * np.expm1(eps) * np.exp(eps) + e_p16 + e_sums
            ref[:, h * hs:(h + 1) * hs] = o
            bound[:, h * hs:(h + 1) * hs] = 2.0 ** -11 * np.abs(o) + 2.0 ** -25 + (e_rel * vmax)[:, None]
    return ref, bound


def _attention_inputs(kind, n, start, n_heads, n_kv, hs, rng):
    """q [n, n_heads*hs], k / v [start+n, n_kv*hs] (f32).  v is random and different for every key and KV head.
    random:  scaled scores of a few log2 units.
    large:   scaled scores of about +-10^3: the row max jumps between key tiles (online max and rescale).
    equal:   every key of a KV head equal: the output is the exact average of the visible v.
    newest:  k_j = j * w_g along q's direction, so the scaled score of key j is c_h * j: the newest visible key dominates
             (any visible future key would take over), with a slope c_h in [1, 2) different for every head of a group."""
    nk, kv_mul = start + n, n_heads // n_kv
    v = rng.standard_normal((nk, n_kv * hs)).astype(np.float32)
    if kind in ("random", "large"):
        q = rng.standard_normal((n, n_heads * hs)) * (2.0 if kind == "random" else 700.0)
        k = rng.standard_normal((nk, n_kv * hs))
    elif kind == "equal":
        q = rng.standard_normal((n, n_heads * hs)) * 2.0
        k = np.tile(rng.standard_normal((1, n_kv * hs)), (nk, 1))
    else:
        w = rng.standard_normal((n_kv, hs))
        w /= np.linalg.norm(w, axis=1, keepdims=True)
        k = (np.arange(nk)[:, None, None] * w[None] + rng.standard_normal((nk, n_kv, hs)) * (0.05 / np.sqrt(hs))).reshape(nk, -1)
        c = 1.0 + (np.arange(n_heads) % kv_mul) / kv_mul
        qrow = (c[:, None] * np.sqrt(hs) * np.log(2.0) * w[np.arange(n_heads) // kv_mul]).reshape(-1)
        q = np.tile(qrow, (n, 1))
    return q.astype(np.float32), k.astype(np.float32), v


ATT_KINDS = ["random", "large", "equal", "newest"]
ATT_STARTS = [0, 1, 63, 64, 65, 200]
ATT_SENTINEL = 0x7E5A  # an f16 NaN: the kernels never produce one from finite inputs


def _attention_cases(kv_mul):
    """(n, start_pos, head_size) for one GQA ratio: n = 1, QT - 1, QT, QT + 1, 130, 300 (QT = 64 / kv_mul query tokens per
    CTA), start positions and both head sizes spread over them, and one 900-key context past many key tiles."""
    qt = 64 // kv_mul
    ns = sorted({x for x in (1, qt - 1, qt, qt + 1, 130, 300) if x >= 1})
    i0 = [1, 2, 4, 8, 16, 64].index(kv_mul)
    cases = [(n, ATT_STARTS[(i0 + j) % len(ATT_STARTS)], (64, 128)[(i0 + j) % 2]) for j, n in enumerate(ns)]
    cases.append((300, 600, (128, 64)[i0 % 2]))
    return cases


def _check_attention(pkg, q, k, v, n_heads, n_kv, start, kind, what):
    n = q.shape[0]
    out = pkg.native.test_pf_attention(q, k, v, n_heads, n_kv, start, out_rows=n + 64, sentinel=ATT_SENTINEL)
    assert np.all(out[n:] == ATT_SENTINEL), f"{what}: a padding row past n was written"
    assert not np.any(out[:n] == ATT_SENTINEL), f"{what}: a (row < n, head) slot was not written"
    ref, bound = _attention_ref(q, k, v, n_heads, n_kv, start, equal_scores=kind == "equal")
    return _assert_within(what, out[:n].view(np.float16), ref, bound)


@pytest.mark.parametrize("kv_mul", [1, 2, 4, 8, 16, 64])
def test_pf_attention_matches_float64(pkg, kv_mul):
    """k_pf_attention_mma_packed on a one-sequence chunk (what the prefill runs), elementwise against float64 softmax attention, at every GQA ratio
    the tensor-core prefill accepts (at 64 a query tile is one token), across key-tile boundaries."""
    n_kv = 2 if kv_mul <= 8 else 1
    n_heads = n_kv * kv_mul
    worst = 0.0
    for n, start, hs in _attention_cases(kv_mul):
        for kind in ATT_KINDS:
            rng = np.random.default_rng(zlib.crc32(repr((kv_mul, n, start, hs, kind)).encode()))
            q, k, v = _attention_inputs(kind, n, start, n_heads, n_kv, hs, rng)
            what = f"kv_mul={kv_mul} hs={hs} n={n} start={start} {kind}"
            worst = max(worst, _check_attention(pkg, q, k, v, n_heads, n_kv, start, kind, what))
    print(f"attention kv_mul={kv_mul}: worst |err| / bound over all cases = {worst:.3g}")


def _prefill_and_compare(pkg, orc, m, n_tok, batch, tol=FP16_TOL):
    c = m.configuration
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=batch)
    om = orc.OracleModel(m)
    try:
        assert plan.prefill_info()[0] == plan.PREFILL_TENSOR_CORE  # default for FP16 plans created with a batch size
        toks = orc.bench_tokens(c.vocab_size, n_tok + 1)
        for off in range(0, n_tok, batch):
            plan.forward_batch_prefill(toks[off:min(off + batch, n_tok)], off)
        assert plan.prefill_info()[1] > 0
        for pos in range(n_tok):
            om.forward(int(toks[pos]), pos, want_logits=False)
        nv = n_tok * c.kv_dim
        for l in range(c.n_layers):
            nkv = c.context_length * c.kv_dim
            for name, ref in (("key_cache", om.key_cache(l)), ("value_cache", om.value_cache(l))):
                got = plan.read_buffer(name, nkv, layer=l)
                err = np.max(np.abs(got[:nv] - ref[:nv])) / np.max(np.abs(ref[:nv]))
                assert err <= tol, f"{name} layer {l}: rel err {err:.2e}"
                assert not np.any(got[nv:]), f"{name} layer {l}: rows past the prompt were written"
        lg, _ = plan.forward_decode(int(toks[n_tok]), n_tok)
        ref = om.forward(int(toks[n_tok]), n_tok)
        err = np.max(np.abs(lg - ref)) / np.max(np.abs(ref))
        assert err <= tol, f"logits after prefill: rel err {err:.2e}"
        # the exact mode of the same plan stays bit-identical to the CPU path
        plan.set_prefill_mode("exact")
        plan.kv_reset()
        for off in range(0, n_tok, batch):
            plan.forward_batch_prefill(toks[off:min(off + batch, n_tok)], off)
        k = plan.read_buffer("key_cache", c.context_length * c.kv_dim, layer=c.n_layers - 1)
        assert np.array_equal(k.view(np.uint32)[:nv], om.key_cache(c.n_layers - 1).view(np.uint32)[:nv])
    finally:
        plan.free()
        om.close()


@pytest.mark.parametrize("shape,n_tok,batch", [("tiny-llama", 50, 32), ("tiny-qwen3", 37, 16), ("tiny-llama-tied", 130, 130), ("tiny-llama", 300, 300),
                                               ("tiny-qwen3", 520, 512), ("tiny-phi3-gqa", 45, 32), ("tiny-llama-mha", 70, 32),
                                               ("tiny-llama-gqa8", 100, 64), ("tiny-llama-gqa4-hs128", 90, 64)])
def test_tensor_core_prefill_within_fp16_tolerance(pkg, orc, make_model, shape, n_tok, batch):
    """Chunks that start at position > 0, a ragged last chunk, a chunk longer than one 128-row GEMM tile, chunks
    longer than 256 rows (ragged and full, then an 8-token tail at position 512),
    Llama (interleaved RoPE), Qwen3 (q/k norm + NeoX RoPE, q width != dim) and Phi-3 (fused qkv / gate-up source tensors, NeoX RoPE without norm);
    GQA ratios 1 (head size 64), 2, 4 (head size 128) and 8 (head size 64)."""
    m = make_model(shape, pkg.gguf.GGMLType.F16, n_tok + 8)
    _prefill_and_compare(pkg, orc, m, n_tok, batch)


def test_tensor_core_prefill_mid_llama(pkg, orc):
    """The real Llama-3-8B layer geometry (2 layers): 136 tokens in chunks of 128 (split-K residual GEMMs, an 8-token tail)."""
    sh = pkg.synth.SHAPES["mid-llama"]
    F16 = pkg.gguf.GGMLType.F16
    m = pkg.loader.model_from_tensors(sh, F16, pkg.synth.build_tensors_fast(sh, F16, seed=1234), 144)
    _prefill_and_compare(pkg, orc, m, 136, 128)


def _f16_rows(m, name, r0=0, r1=None):
    tt, dims, raw = m.tensors[name]
    assert int(tt) == 1, f"{name}: the stage check needs F16 weights"
    w = np.ascontiguousarray(raw).view(np.float16).reshape(int(dims[1]), int(dims[0]))
    return w[r0:r1]


def _rope_tables(c, positions):
    """cos / sin exactly as the plan builds them (RoPE.precomputeFreqsCis): f32 freq, f32 pos * freq, cos / sin in double narrowed."""
    i = np.arange(0, c.head_size, 2)
    freq = (1.0 / np.power(np.float64(np.float32(c.rope_theta)), i / np.float64(c.head_size))).astype(np.float32)
    val = (np.asarray(positions, dtype=np.float32)[:, None] * freq[None, :]).astype(np.float32)
    return np.cos(val.astype(np.float64)).astype(np.float32), np.sin(val.astype(np.float64)).astype(np.float32)


def _k_cache_ref(m, kpart, start, layer):
    """float64 RoPE (after the Qwen3 per-head k norm) of the k part of the QKV rows, and a bound of a few f32 roundings per pair."""
    c = m.configuration
    hs, half, n = c.head_size, c.head_size // 2, kpart.shape[0]
    x = kpart.astype(np.float64).reshape(n, -1, hs)
    qknorm = c.arch == 1
    if qknorm:
        nw = np.ascontiguousarray(m.tensors[f"blk.{layer}.attn_k_norm.weight"][2]).view(np.float32).astype(np.float64)
        x = x / np.sqrt((x * x).mean(axis=2, keepdims=True) + np.float64(np.float32(c.rms_norm_eps))) * nw
    neox = c.arch in (1, 2)
    i0 = np.arange(half) if neox else 2 * np.arange(half)
    i1 = i0 + half if neox else i0 + 1
    cr, ci = _rope_tables(c, start + np.arange(n))
    cr, ci = cr.astype(np.float64)[:, None, :], ci.astype(np.float64)[:, None, :]
    x0, x1 = x[:, :, i0], x[:, :, i1]
    ref, bound = np.empty_like(x), np.empty_like(x)
    ref[:, :, i0], ref[:, :, i1] = x0 * cr - x1 * ci, x0 * ci + x1 * cr
    pair = (4 + (16 if qknorm else 0)) * U * (np.abs(x0) + np.abs(x1))  # the rotation's 3 roundings; the norm's short f32 sums
    bound[:, :, i0], bound[:, :, i1] = pair, pair
    return ref.reshape(n, -1), bound.reshape(n, -1)


def _check_prefill_stages(pkg, m, first, second):
    """Prefill `first` tokens, then a chunk of `second` at start_pos = first; check every stage of the last layer of that
    chunk against float64 evaluated from the stage's own inputs as read back from the device."""
    c = m.configuration
    L, qd, kvd, hid = c.n_layers - 1, c.n_heads * c.head_size, c.n_kv_heads * c.head_size, c.hidden_dim
    nqkv = qd + 2 * kvd
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=max(first, second))
    try:
        assert plan.prefill_info()[0] == plan.PREFILL_TENSOR_CORE
        toks = np.random.default_rng(first * 1000 + second).integers(0, c.vocab_size, first + second).astype(np.int32)
        plan.forward_batch_prefill(toks[:first], 0)
        plan.forward_batch_prefill(toks[first:], first)
        n, start = second, first
        bpad = (max(first, second) + 127) // 128 * 128
        qkv = plan.read_buffer("pf_qkv", bpad * nqkv).reshape(bpad, nqkv)[:n]
        a16 = plan.read_buffer("pf_a16", bpad * c.dim, dtype=np.float16).reshape(bpad, c.dim)[:n]
        att16 = plan.read_buffer("pf_att16", bpad * qd, dtype=np.float16).reshape(bpad, qd)[:n]
        h16 = plan.read_buffer("pf_h16", bpad * hid, dtype=np.float16).reshape(bpad, hid)[:n]
        x = plan.read_buffer("pf_x", bpad * c.dim).reshape(bpad, c.dim)[:n]
        assert np.all(np.isfinite(x))
        kc = plan.read_buffer("key_cache", c.context_length * kvd, layer=L).reshape(-1, kvd)[:start + n]
        vc = plan.read_buffer("value_cache", c.context_length * kvd, layer=L).reshape(-1, kvd)[:start + n]
        name = f"{m.model_type} last layer"
        # V cache rows of the chunk: the v part of the QKV GEMM output, bit for bit
        assert np.array_equal(vc[start:].view(np.uint32), qkv[:, qd + kvd:].view(np.uint32)), f"{name}: V cache != v part of pf_qkv"
        # K cache rows of the chunk: RoPE (after the Qwen3 k norm) of the k part
        kref, kbound = _k_cache_ref(m, qkv[:, qd:qd + kvd], start, L)
        r_k = _assert_within(f"{name} K cache = RoPE(k)", kc[start:], kref, kbound)
        # attention over the rotated q and the KV cache, as k_pf_attention_mma_packed computes it
        aref, abound = _attention_ref(qkv[:, :qd], kc, vc, c.n_heads, c.n_kv_heads, start)
        r_a = _assert_within(f"{name} attention", att16, aref, abound)
        # gate/up + SwiGLU on the FFN input
        if c.arch == 2:
            w1, w3 = _f16_rows(m, f"blk.{L}.ffn_up.weight", 0, hid), _f16_rows(m, f"blk.{L}.ffn_up.weight", hid, 2 * hid)
        else:
            w1, w3 = _f16_rows(m, f"blk.{L}.ffn_gate.weight"), _f16_rows(m, f"blk.{L}.ffn_up.weight")
        href, hbound = _gateup_ref(a16, w1, w3)
        r_h = _assert_within(f"{name} gate/up", h16, href, hbound)
        print(f"prefill stages {name} (chunk of {n} at {start}): worst |err| / bound K cache {r_k:.3g}, attention {r_a:.3g}, gate/up {r_h:.3g}")
    finally:
        plan.free()


@pytest.mark.parametrize("shape,first,second", [("tiny-llama", 40, 50), ("tiny-qwen3", 70, 60), ("tiny-phi3-gqa", 30, 45)])
def test_tensor_core_prefill_stages(pkg, make_model, shape, first, second):
    """Each kernel of a real prefill chunk at start_pos > 0, in isolation, at the model's own geometry."""
    _check_prefill_stages(pkg, make_model(shape, pkg.gguf.GGMLType.F16, first + second + 8), first, second)


def test_tensor_core_prefill_stages_mid_llama(pkg):
    """The same stage checks at the Llama-3-8B layer geometry (32 heads, 8 KV heads, hidden 14336)."""
    sh = pkg.synth.SHAPES["mid-llama"]
    F16 = pkg.gguf.GGMLType.F16
    m = pkg.loader.model_from_tensors(sh, F16, pkg.synth.build_tensors_fast(sh, F16, seed=1234), 112)
    _check_prefill_stages(pkg, m, 64, 40)


def _dequantised_f16_twin(pkg, m):
    """The model the Q8_0 tensor-core prefill actually computes with: every matrix replaced by f16(q * scale) (Q8_0FloatTensor.getFloat
    rounded once, as k_tiles_to_f16 does on the device), norms untouched, embedding kept in Q8_0 (the gather dequantises in fp32)."""
    G = pkg.gguf.GGMLType
    tensors = {}
    for name, (tt, dims, raw) in m.tensors.items():
        if tt == G.Q8_0 and name != "token_embd.weight":
            blocks = np.ascontiguousarray(raw).reshape(-1, 34)
            d = blocks[:, :2].copy().view("<f2").astype(np.float32)
            q = blocks[:, 2:].view(np.int8).astype(np.float32)
            tensors[name] = (G.F16, dims, (q * d).astype(np.float16).view(np.uint8).reshape(-1))
        else:
            tensors[name] = (tt, dims, raw)
    cfg = m.configuration
    twin = pkg.loader.Model(None, type(cfg)(**{**cfg.__dict__, "quantization": "FP16"}), m.model_type, tensors)
    return twin


@pytest.mark.parametrize("shape", ["tiny-llama", "tiny-qwen3"])
def test_tensor_core_prefill_q8_model(pkg, orc, make_model, shape):
    """Opt-in on a Q8_0 plan: f16 twins of the matrices are dequantised on the device for the GEMMs (the reference's Q8_0 MMA prefill
    feeds FP16 tiles the same way, TransformerBatchPrefillKernels.java:1563-1574).  PARITY BAR: the KV cache must agree at FP16
    tolerance (2^-8) with the CPU oracle evaluated on exactly those dequantised FP16 weights -- that is what this path computes.
    Against the CPU path of the Q8_0 model itself the difference is the CPU path's own int8 activation rounding, which the tensor-core
    path (like the reference's GPU prefill) does not apply: percent-level, bounded loosely and reported, which is why this mode is not
    the default for Q8_0 plans."""
    m = make_model(shape, pkg.gguf.GGMLType.Q8_0, 48)
    c = m.configuration
    n_tok, batch = 40, 16
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=batch)
    om_twin = orc.OracleModel(_dequantised_f16_twin(pkg, m))
    om_q8 = orc.OracleModel(m)
    try:
        assert plan.prefill_info()[0] == plan.PREFILL_EXACT  # Q8_0 plans default to the exact path
        plan.set_prefill_mode("tensor_core")
        toks = orc.bench_tokens(c.vocab_size, n_tok + 1)
        for off in range(0, n_tok, batch):
            plan.forward_batch_prefill(toks[off:min(off + batch, n_tok)], off)
        for pos in range(n_tok):
            om_twin.forward(int(toks[pos]), pos, want_logits=False)
            om_q8.forward(int(toks[pos]), pos, want_logits=False)
        nv = n_tok * c.kv_dim
        worst_twin = worst_q8 = 0.0
        for l in range(c.n_layers):
            nkv = c.context_length * c.kv_dim
            for name in ("key_cache", "value_cache"):
                got = plan.read_buffer(name, nkv, layer=l)[:nv]
                rt = (om_twin.key_cache(l) if name == "key_cache" else om_twin.value_cache(l))[:nv]
                rq = (om_q8.key_cache(l) if name == "key_cache" else om_q8.value_cache(l))[:nv]
                worst_twin = max(worst_twin, float(np.max(np.abs(got - rt)) / np.max(np.abs(rt))))
                worst_q8 = max(worst_q8, float(np.max(np.abs(got - rq)) / np.max(np.abs(rq))))
        assert worst_twin <= FP16_TOL, f"vs the oracle on the dequantised FP16 weights: rel err {worst_twin:.2e}"
        assert worst_q8 <= Q8_NOISE_TOL, f"vs the CPU path of the Q8_0 model (its int8 activation rounding): rel err {worst_q8:.2e}"
        print(f"q8 tensor-core prefill {shape}: {worst_twin:.2e} vs dequantised-FP16 oracle, {worst_q8:.2e} vs the Q8_0 CPU path")
        # the exact mode of the same plan stays bit-identical to the CPU path of the Q8_0 model
        plan.set_prefill_mode("exact")
        plan.kv_reset()
        for off in range(0, n_tok, batch):
            plan.forward_batch_prefill(toks[off:min(off + batch, n_tok)], off)
        k = plan.read_buffer("key_cache", c.context_length * c.kv_dim, layer=c.n_layers - 1)
        assert np.array_equal(k.view(np.uint32)[:nv], om_q8.key_cache(c.n_layers - 1).view(np.uint32)[:nv])
    finally:
        plan.free()
        om_twin.close()
        om_q8.close()


def test_tensor_core_prefill_unsupported_is_loud(pkg, make_model):
    """A plan created without a prefill batch size keeps the exact path and says why the tensor-core one is unavailable."""
    m = make_model("tiny-llama", pkg.gguf.GGMLType.F16, 32)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=0)
    try:
        assert plan.prefill_info()[0] == plan.PREFILL_EXACT
        with pytest.raises(Exception, match="prefill batch size"):
            plan.set_prefill_mode("tensor_core")
        plan.set_prefill_mode("exact")
    finally:
        plan.free()


def test_tensor_core_refusal_allocates_nothing(pkg, make_model):
    """A Q8_0 plan whose shape the tensor-core prefill cannot run (Phi-3's head size 96) refuses "tensor_core" before it builds
    the f16 twins: the device bytes are unchanged and the previous mode stays in force."""
    m = make_model("tiny-phi3", pkg.gguf.GGMLType.Q8_0, 32)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=16)
    try:
        plan.set_prefill_mode("tensor_core_exact")
        b0 = plan.device_bytes
        with pytest.raises(pkg.native.UnsupportedOperation, match="head size"):
            plan.set_prefill_mode("tensor_core")
        assert plan.device_bytes == b0, (plan.device_bytes, b0)
        assert plan.prefill_info()[0] == plan.PREFILL_TENSOR_CORE_EXACT
    finally:
        plan.free()


def test_tensor_parallel_plan_refuses_tensor_core_modes(pkg, make_model):
    """Rank 0 of a two-way tensor-parallel plan with a prefill batch size, created without its peer: every tensor-core mode names
    the single-GPU rule and the exact mode stays in force."""
    m = make_model("tiny-qwen3", pkg.gguf.GGMLType.Q8_0, ctx=64, seed=28)
    cfg = pkg.plan.make_config(m)
    cfg.tp_rank, cfg.tp_size = 0, 2
    plan = pkg.native.NativePlan(cfg, m.tensors, 16, 0)
    P = pkg.B200MasterPlan
    try:
        for mode in (P.PREFILL_TENSOR_CORE, P.PREFILL_TENSOR_CORE_W8A16, P.PREFILL_TENSOR_CORE_EXACT):
            with pytest.raises(pkg.native.UnsupportedOperation, match="single-GPU"):
                plan.set_prefill_mode(mode)
            assert plan.prefill_info()[0] == P.PREFILL_EXACT
    finally:
        plan.free()
