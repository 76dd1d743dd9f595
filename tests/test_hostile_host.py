"""CPU tests of the hostile-value models (tests/hostile.py).  Two jobs, no GPU:

1. The oracle is the reference the GPU tests compare with, so its two restatements (oracle.c and the numpy one in oracle.py) are held
   to each other on the very blocks and rows the builders produce: extreme Q8_0 weight blocks, all-zero / outlier / signed-zero
   activations, dense FP16 subnormals at every lane count, the RMSNorm of the hostile rows, the attention softmax against float64.
2. "The test saw something": every builder's planted property is asserted on the oracle's own results, so a property that a quantiser
   or a rounding removed fails here instead of passing vacuously on the GPU."""
import ctypes as C

import numpy as np
import pytest

import hostile as H
from test_oracle import softmax_bound_violations

Q8, F16 = H.G.Q8_0, H.G.F16


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _rmsnorm_c(orc, x, w, eps):
    out = np.empty_like(x)
    t = orc.OTensor()
    t.data, t.type = w.ctypes.data, 0
    orc.lib().oracle_rmsnorm(out.ctypes.data, x.ctypes.data, C.byref(t), len(x), eps)
    return out


# ---- 1. the oracle's two restatements at the edges -----------------------------------------------------------------------------

def _hostile_activations(rng, n):
    x = rng.standard_normal(n).astype(np.float32)
    zero_block = x.copy()
    zero_block[32:64] = 0.0
    neg_zero = x.copy()
    neg_zero[64:96] = -0.0
    neg_zero[5] = -0.0
    outlier = x.copy()
    outlier[n // 2 + 5] = 4064.0
    tiny = (x * np.float32(1e-30)).astype(np.float32)  # amax / 127 is a float subnormal's neighbour; its f16 round trip is 0
    return {"normal": x, "zero_block": zero_block, "all_zero": np.zeros(n, np.float32), "neg_zero": neg_zero, "outlier": outlier,
            "tiny": tiny, "huge": (x * np.float32(1e30)).astype(np.float32)}


def test_q8_dot_restatements_agree_on_extreme_blocks(orc):
    """dotQ8Activation over weight blocks of every kind extreme_q8_blocks plants, against hostile activations."""
    rng = np.random.default_rng(1)
    cols, rows = 256, 10
    nb = rows * cols // 32
    d = (rng.random(nb) * 0.01 + 1e-4).astype(np.float16).view(np.uint16)
    q = rng.integers(-127, 128, (nb, 32)).astype(np.int8)
    d[0::5][:8] = 0
    d[1::5][:8] = 1
    d[2::5] ^= 0x8000
    q[3::5] = -128
    q[4::5] = rng.choice(np.array([-127, 127], dtype=np.int8), (len(q[4::5]), 32))
    d[7] = 0x7BFF  # 65504
    raw = H.q8_raw(d, q)
    with np.errstate(all="ignore"):  # "huge" against d = 65504 overflows to inf, and inf * 0 is NaN, in both restatements alike
        for name, x in _hostile_activations(rng, cols).items():
            for row in range(rows):
                a, b = np.float32(orc.q8_dot(raw, row * cols, x)), np.float32(orc.np_q8_dot(raw, row * cols, x))
                assert a.view(np.uint32) == b.view(np.uint32), (name, row, a, b)


def test_q8_quantize_restatements_agree_on_hostile_rows(orc):
    rng = np.random.default_rng(2)
    for name, x in _hostile_activations(rng, 256).items():
        aq, sc = orc.q8_quantize(x)
        for b in range(8):
            with np.errstate(over="ignore"):  # "huge": amax / 127 is beyond f16, the scale's round trip is inf
                qn, sn = orc.np_q8_quantize_block(x[b * 32:(b + 1) * 32])
            assert np.array_equal(aq[b * 32:(b + 1) * 32].astype(np.int64), qn), (name, b)
            assert np.float32(sc[b]).view(np.uint32) == np.float32(sn).view(np.uint32), (name, b)
        assert np.abs(aq.astype(np.int32)).max() <= 127
        if name == "all_zero":
            assert not aq.any() and not sc.any()


@pytest.mark.parametrize("lanes", [16, 8, 4, 0])
@pytest.mark.parametrize("n", [256, 16 * 5 + 7])
def test_f16_dot_restatements_agree_on_subnormals(orc, lanes, n):
    """Dense subnormals of both signs, -0 and +-65504: flushed in the vector loop, IEEE in the scalar tail and the scalar species."""
    rng = np.random.default_rng(3)
    w = (rng.standard_normal(n) * 0.02).astype(np.float16).view(np.uint16)
    u = rng.random(n)
    w[u < 0.3] = rng.integers(1, 0x400, int((u < 0.3).sum())).astype(np.uint16) | (rng.integers(0, 2, int((u < 0.3).sum())).astype(np.uint16) << 15)
    w[(u >= 0.3) & (u < 0.35)] = 0x8000
    w[3], w[n - 2] = 0x7BFF, 0xFBFF
    for name, x in _hostile_activations(rng, n).items():
        if name == "huge":
            continue  # 65504 * 1e30 overflows: an inf the forward pass never meets
        a, b = np.float32(orc.f16_dot(w, x, lanes)), np.float32(orc.np_f16_dot(w, x, lanes))
        assert a.view(np.uint32) == b.view(np.uint32), (name, a, b)


@pytest.mark.parametrize("dim", [256, 1536, 2848])
def test_rmsnorm_restatements_agree_on_outlier_rows(orc, dim):
    rng = np.random.default_rng(4)
    w = (1 + 0.02 * rng.standard_normal(dim)).astype(np.float32)
    for kind in H.OUTLIER_KINDS:
        d, q = H.outlier_row(kind, dim, rng)
        x = (q.astype(np.float32) * d[:, None]).reshape(-1)
        a, b = _rmsnorm_c(orc, x, w, 1e-5), orc.np_rmsnorm(x, w, 1e-5)
        assert np.array_equal(_bits(a), _bits(b)), kind
        if kind == "zero":
            assert not a.any()


def test_outlier_rows_have_their_property():
    rng = np.random.default_rng(5)
    for dim in (256, 1536, 4096, 12288):
        sums = {}
        for kind in H.OUTLIER_KINDS:
            d, q = H.outlier_row(kind, dim, rng)
            x = (q.astype(np.float64) * d[:, None]).reshape(-1)
            assert np.array_equal(x.astype(np.float16).astype(np.float64), x), kind  # exact in f16, and q * d in Q8_0
            sums[kind] = float(np.add.accumulate((x.astype(np.float32) ** 2).astype(np.float32), dtype=np.float32)[-1])
            if kind.startswith("outlier_"):
                a = np.sort(np.abs(x))
                assert a[-1] >= 1024 * a[-2], kind
        P = (1 << (dim.bit_length() - 1)) / 4
        assert sums["zero"] == 0.0 and sums["pow2_at"] == P
        assert P * (1 - 2.0 ** -9) <= sums["pow2_below"] < P < sums["pow2_above"] <= P * (1 + 2.0 ** -9)
        d, q = H.outlier_row("many_binades", dim, rng)
        e = np.frexp((q.astype(np.float64) * d[:, None]) ** 2)[1]
        assert e.max() - e.min() >= 30
        d, q = H.outlier_row("zero_head", dim, rng)
        assert not d[:dim // 64].any() and d[dim // 64:].all()


# ---- 2. every builder's property, on the oracle ----------------------------------------------------------------------------------

@pytest.mark.parametrize("shape,quant", [("tiny-llama", Q8), ("tiny-llama", F16), ("tiny-llama-tied", Q8), ("tiny-llama-vocab509", Q8),
                                         ("tiny-qwen3", F16), ("tiny-phi3", F16)])
@pytest.mark.parametrize("kind", ["group", "warps", "ctas", "padding"])
def test_tied_logits_tie_and_the_lowest_index_wins(orc, shape, quant, kind):
    m = H.tied_logits(shape, quant, kind)
    V = m.configuration.vocab_size
    A, B = H.tie_rows(kind, V)
    tied = "output.weight" not in m.tensors
    om = H.oracle_for(orc, m)
    try:
        for start in (4, 7):
            om.reset()
            tok, seen = start, set()
            for pos in range(16):
                lg = om.forward(tok, pos)
                even = tok % 2 == 0
                if tied and (tok in A or tok in B):  # a duplicated embedding row carries its set's column
                    even = tok in A
                want = A if even else B
                top = np.flatnonzero(lg == lg.max())
                assert list(top) == sorted(want), (kind, start, pos, tok, top)
                assert len(set(_bits(lg[top]))) == 1
                tok = orc.argmax(lg)
                assert tok == min(want)
                seen.add(tok)
            if min(A) % 2 == 1 and not tied:
                assert seen == {min(A), min(B)}  # the greedy loop alternates between the two sets
    finally:
        om.close()


@pytest.mark.parametrize("quant", [Q8, F16])
@pytest.mark.parametrize("kind", ["identical", "zero"])
def test_degenerate_classifiers_answer_zero(orc, quant, kind):
    m = H.tied_logits("tiny-llama", quant, kind)
    om = H.oracle_for(orc, m)
    try:
        for pos, tok in enumerate((4, 7, 300)):
            lg = om.forward(tok, pos)
            assert len(set(_bits(lg))) == 1 and orc.argmax(lg) == 0
            if kind == "zero":
                assert not lg.any()
    finally:
        om.close()
    raw = m.tensors["output.weight"][2]
    if kind == "zero":
        w = H.loader.tensor_as_f32(m, "output.weight")
        assert not w.any() and np.signbit(w).any() and not np.signbit(w).all()  # zeros of both signs
        if quant == Q8:
            assert H.q8_split(raw)[1].any()  # under quants that are not zero


@pytest.mark.parametrize("shape,quant", [("tiny-llama", Q8), ("tiny-llama", F16), ("tiny-qwen2moe", Q8)])
def test_outlier_embeddings_reach_every_norm(orc, shape, quant):
    """x is still the embedding row after the step (Wo = W2 = 0), so every norm of the step read it; the zero row gives all-zero
    activation blocks at the input of every matvec and all-zero logits."""
    m = H.outlier_embeddings(shape, quant)
    c = m.configuration
    emb = H.loader.tensor_as_f32(m, "token_embd.weight").reshape(c.vocab_size, c.dim)
    om = H.oracle_for(orc, m)
    try:
        for kind, tok in H.OUTLIER_TOKEN.items():
            lg = om.forward(tok, 0)
            assert np.isfinite(lg).all(), kind
            if hasattr(om, "x"):  # the C oracle normalises x in place for the classifier
                w = H.loader.tensor_as_f32(m, "output_norm.weight")
                assert np.array_equal(_bits(om.x()), _bits(orc.np_rmsnorm(emb[tok], w, c.rms_norm_eps))), kind
            if kind == "zero":
                assert not emb[tok].any() and not lg.any()
                aq, sc = orc.q8_quantize(orc.np_rmsnorm(emb[tok], np.ones(c.dim, np.float32), c.rms_norm_eps))
                assert not aq.any() and not sc.any()
            if kind == "outlier_mid":
                xn = orc.np_rmsnorm(emb[tok], np.ones(c.dim, np.float32), c.rms_norm_eps)
                aq, _ = orc.q8_quantize(xn)
                blk = (c.dim // 2 + 5) // 32
                assert np.count_nonzero(aq[blk * 32:(blk + 1) * 32]) == 1  # the outlier's block quantises everything else to 0
    finally:
        om.close()


def test_zero_qk_rows_give_the_head_norm_a_zero_vector(orc):
    m = H.zero_qk_rows("tiny-qwen3", Q8)
    c = m.configuration
    om = H.oracle_for(orc, m)
    try:
        for pos in range(3):
            om.forward(5 + pos, pos)
        for l in range(c.n_layers):
            k = om.key_cache(l).reshape(c.context_length, c.kv_dim)[:3]
            assert not k[:, :c.head_size].any() and k[:, c.head_size:].any()
        att = om.att(3)
        assert np.all(att[0] == np.float32(1) / np.float32(3))  # q = 0 in head 0: equal scores
    finally:
        om.close()


@pytest.mark.parametrize("shape,quant", [("tiny-llama", Q8), ("tiny-llama", F16), ("tiny-qwen3", Q8), ("tiny-phi3", Q8)])
def test_saturated_attention_underflows(orc, shape, quant):
    """Over 140 positions the last layer's softmax weights hold float subnormals, exact zeros and one-hot rows, and stay within the
    float64 softmax's error bound of the scores recomputed from the oracle's own K cache."""
    m = H.saturated_attention(shape, quant, "peaked", ctx=144)
    c = m.configuration
    om = H.oracle_for(orc, m)
    tiny = np.finfo(np.float32).tiny
    sub = zero = onehot = 0
    try:
        toks = orc.bench_tokens(c.vocab_size, 140)
        for pos in range(140):
            lg = om.forward(int(toks[pos]), pos)
            assert np.isfinite(lg).all()
            a = om.att(pos + 1)
            sub += int(((a > 0) & (a < tiny)).sum())
            zero += int((a == 0).sum())
            onehot += int(((a == 1).sum(axis=1) == 1).sum()) if pos else 0
            s = a.astype(np.float64).sum(axis=1)
            assert np.all(np.abs(s - 1) < 1e-5)
    finally:
        om.close()
    assert sub > 0 and zero > 0 and onehot > 0, (sub, zero, onehot)


def test_oracle_softmax_on_saturated_scores_matches_float64(orc):
    """softmaxInPlace as the attention uses it (temperature 1 through the sampler's entry) on score rows that span hundreds of nats."""
    rng = np.random.default_rng(9)
    for n in (2, 127, 128, 129, 511, 512, 513):
        for spread in (50.0, 250.0, 1000.0):
            x = (rng.standard_normal(n) * spread).astype(np.float32)
            _, p = orc.sample(x, 1.0, 0.0, 0.5, want_probs=True)
            assert softmax_bound_violations(x, p).size == 0, (n, spread)
        _, p = orc.sample(np.zeros(n, np.float32), 1.0, 0.0, 0.5, want_probs=True)
        assert np.all(p == np.float32(1) / np.float32(n))


@pytest.mark.parametrize("shape,quant", [("tiny-llama", Q8), ("tiny-qwen3", F16)])
def test_uniform_attention_is_one_over_n(orc, shape, quant):
    m = H.saturated_attention(shape, quant, "uniform", ctx=140)
    om = H.oracle_for(orc, m)
    try:
        for pos in range(129):
            om.forward(3 + pos % 50, pos, want_logits=pos in (127, 128))
            if pos in (127, 128):
                assert np.all(om.att(pos + 1) == np.float32(1) / np.float32(pos + 1))
    finally:
        om.close()


@pytest.mark.parametrize("shape,quant", [("tiny-llama", Q8), ("tiny-llama", F16), ("tiny-phi3", Q8)])
def test_saturated_swiglu_saturates(orc, shape, quant):
    """The down projection's input holds -0 (g / inf), +0 (g = 0) and values beyond +-100; a 32-block of it is not all zero, so the
    quantiser divides there."""
    m = H.saturated_swiglu(shape, quant)
    om = H.oracle_for(orc, m)
    neg0 = pos0 = big = 0
    try:
        for pos, tok in enumerate((1, 2, 3, 4)):
            assert np.isfinite(om.forward(tok, pos)).all()
            hb = om.hb()
            z = hb == 0
            neg0 += int((z & np.signbit(hb)).sum())
            pos0 += int((z & ~np.signbit(hb)).sum())
            big += int((np.abs(hb) > 100).sum())
            assert z[2::3].all()
    finally:
        om.close()
    assert neg0 > 0 and pos0 > 0 and big > 0, (neg0, pos0, big)


def test_extreme_q8_blocks_are_in_every_matrix(orc):
    m = H.extreme_q8_blocks("tiny-llama")
    for n, (tt, dims, raw) in m.tensors.items():
        if tt != Q8:
            continue
        d, q = H.q8_split(raw)
        df = d.view(np.float16).astype(np.float32)
        share = [(d == 0).mean() + (d == 0x8000).mean(), (d == 1).mean(), (df < 0).mean(), (q == -128).all(axis=1).mean(),
                 (np.abs(q.astype(np.int32)) == 127).all(axis=1).mean()]
        assert all(0.005 < s < 0.04 for s in share), (n, share)
    assert sorted(n.split(".")[-2] for n in m.tensors if m.tensors[n][0] == Q8 and "blk.0." in n) == \
        ["attn_k", "attn_output", "attn_q", "attn_v", "ffn_down", "ffn_gate", "ffn_up"]
    om = H.oracle_for(orc, m)
    ref = H.oracle_for(orc, H.loader.model_from_tensors(H.synth.SHAPES["tiny-llama"], Q8, H.base_tensors("tiny-llama", Q8, 51)[1], 16))
    try:
        a, b = om.forward(7, 0), ref.forward(7, 0)
        assert np.isfinite(a).all() and np.abs(a - b).max() > 0.05 * np.abs(b).max()  # the blocks matter to the logits
    finally:
        om.close()
        ref.close()


@pytest.mark.parametrize("shape", ["tiny-llama", "tiny-llama-tied"])
def test_extreme_f16_weights_are_dense_and_lane_visible(orc, shape):
    m = H.extreme_f16_weights(shape)
    for n, (tt, dims, raw) in m.tensors.items():
        if tt != F16:
            continue
        w = raw.view(np.uint16)
        e, man = (w >> 10) & 0x1F, w & 0x3FF
        sub = (e == 0) & (man != 0)
        assert sub.mean() >= 0.2 and (sub & (w >> 15 == 1)).any() and (sub & (w >> 15 == 0)).any(), n
        assert (w == 0x8000).any() and ((w == 0x7BFF) | (w == 0xFBFF)).any(), n
    vec, scalar = H.oracle_for(orc, m, lanes=16), H.oracle_for(orc, m, lanes=0)
    try:
        a, b = vec.forward(7, 0), scalar.forward(7, 0)
        assert np.isfinite(a).all() and np.isfinite(b).all()
        assert not np.array_equal(_bits(a), _bits(b))  # the flush is visible: the IEEE scalar order gives other logits
    finally:
        vec.close()
        scalar.close()
