"""CPU tests of the oracle (oracle/oracle.c) against (a) an independent numpy restatement of the
same reference lines, (b) numpy's IEEE half conversions, (c) the java.util.Random known answer,
(d) the committed golden fixtures.  No GPU."""
import hashlib
import json
import os

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "oracle_golden.json")


def test_f16_to_f32_all_halves(orc):
    L = orc.lib()
    bits = np.arange(65536, dtype=np.uint16)
    ref = bits.view(np.float16).astype(np.float32)
    got = np.array([L.oracle_f16_to_f32(int(b)) for b in bits], dtype=np.float32)
    ok = (got.view(np.uint32) == ref.view(np.uint32)) | (np.isnan(got) & np.isnan(ref))
    assert ok.all()


def test_f16_daz_matches_bit_trick(orc):
    L = orc.lib()
    bits = np.arange(65536, dtype=np.uint16)
    got = np.array([L.oracle_f16_to_f32_daz(int(b)) for b in bits], dtype=np.float32)
    ref = orc.np_f16_daz(bits)
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    # normal halves agree with IEEE, subnormal halves flush to (signed) zero
    ieee = bits.view(np.float16).astype(np.float32)
    exp = (bits >> 10) & 0x1F
    normal = (exp != 0) & (exp != 31)
    assert np.array_equal(got[normal], ieee[normal])
    assert np.all(got[exp == 0] == 0)


def test_f32_to_f16_rne(orc):
    L = orc.lib()
    rng = np.random.default_rng(0)
    xs = np.concatenate([
        rng.standard_normal(20000).astype(np.float32) * np.float32(10) ** rng.integers(-8, 5, 20000).astype(np.float32),
        np.array([0.0, -0.0, 65504.0, 65519.99, 65520.0, 70000.0, 5.96e-8, 2.98e-8, 2.9802322e-8, 2.9802326e-8, 6.1e-5, 6.0975e-5, 1e-10], dtype=np.float32),
        (np.arange(2048, dtype=np.uint32) * np.uint32(4099) + np.uint32(0x33000000)).view(np.float32),
    ])
    with np.errstate(over="ignore"):
        ref = xs.astype(np.float16).view(np.uint16)
    got = np.array([L.oracle_f32_to_f16(float(x)) for x in xs], dtype=np.uint16)
    assert np.array_equal(got, ref)


def test_java_random_known_answer(orc):
    # new Random(42).nextInt() == -1170105035 (the well-known first draw for seed 42)
    r = orc.JavaRandom(42)
    assert r.next_int() == -1170105035
    # new Random(42).nextInt(10) x10, as printed in countless Java tutorials
    assert list(orc.bench_tokens(10, 10)) == [0, 3, 8, 4, 0, 5, 5, 8, 9, 3]
    for vocab in (512, 128256, 151936, 1000, 7):
        c = orc.bench_tokens(vocab, 300)
        r = orc.JavaRandom(42)
        py = np.array([r.next_int(vocab) for _ in range(300)], dtype=np.int32)
        assert np.array_equal(c, py)
        assert c.min() >= 0 and c.max() < vocab


def _rand_q8_rows(pkg, rng, rows, cols, scale=0.02):
    w = rng.standard_normal(rows * cols).astype(np.float32) * np.float32(scale)
    return pkg.synth.quantize_q8_0(w)


def test_q8_dot_c_vs_numpy(orc, pkg):
    rng = np.random.default_rng(1)
    cols = 256
    raw = _rand_q8_rows(pkg, rng, 8, cols)
    for trial in range(6):
        x = rng.standard_normal(cols).astype(np.float32) * np.float32(10.0 ** rng.integers(-3, 3))
        if trial == 0:
            x[:32] = 0  # zero block: quantizationScale == 0 guard
        if trial == 1:
            x[32:64] = np.float32(1e-30)
        for row in range(8):
            a = np.float32(orc.q8_dot(raw, row * cols, x))
            b = orc.np_q8_dot(raw, row * cols, x)
            assert a.view(np.uint32) == np.float32(b).view(np.uint32)


def test_q8_quantize_matches_numpy(orc):
    rng = np.random.default_rng(2)
    x = rng.standard_normal(512).astype(np.float32)
    x[5] = 3.0
    x[64:96] = 0
    aq, sc = orc.q8_quantize(x)
    for b in range(16):
        q, s = orc.np_q8_quantize_block(x[b * 32:(b + 1) * 32])
        assert np.array_equal(aq[b * 32:(b + 1) * 32].astype(np.int64), q)
        assert np.float32(sc[b]).view(np.uint32) == np.float32(s).view(np.uint32)
    assert np.abs(aq.astype(np.int32)).max() <= 127


@pytest.mark.parametrize("lanes", [16, 8, 0])
def test_f16_dot_c_vs_numpy(orc, lanes):
    rng = np.random.default_rng(3)
    n = 256
    w = (rng.standard_normal(n) * 0.02).astype(np.float16)
    w[::17] = np.float16(3e-6)  # subnormal halves: DAZ in the vector loop, IEEE in the scalar one
    x = rng.standard_normal(n).astype(np.float32)
    a = np.float32(orc.f16_dot(w.view(np.uint16), x, lanes))
    b = orc.np_f16_dot(w.view(np.uint16), x, lanes)
    assert a.view(np.uint32) == np.float32(b).view(np.uint32)


def test_f16_dot_tail(orc):
    rng = np.random.default_rng(4)
    n = 16 * 5 + 7  # scalar tail after the vector loop (FP16FloatTensor.java:104-106)
    w = (rng.standard_normal(n) * 0.5).astype(np.float16)
    x = rng.standard_normal(n).astype(np.float32)
    a = np.float32(orc.f16_dot(w.view(np.uint16), x, 16))
    b = orc.np_f16_dot(w.view(np.uint16), x, 16)
    assert a.view(np.uint32) == np.float32(b).view(np.uint32)


def test_rmsnorm_c_vs_numpy(orc):
    rng = np.random.default_rng(5)
    x = rng.standard_normal(256).astype(np.float32) * 3
    w = (1 + 0.02 * rng.standard_normal(256)).astype(np.float32)
    out = np.empty(256, dtype=np.float32)
    t = orc.OTensor()
    t.data = w.ctypes.data
    t.type = 0
    import ctypes as C
    orc.lib().oracle_rmsnorm(out.ctypes.data, x.ctypes.data, C.byref(t), 256, 1e-5)
    ref = orc.np_rmsnorm(x, w, 1e-5)
    assert np.array_equal(out.view(np.uint32), ref.view(np.uint32))


def test_per_row_quant_is_bit_identical(orc, pkg, make_model):
    """Hoisting the activation quantisation out of the row loop (what the GPU does) must not
    change a single bit versus the reference's quantise-inside-every-dot (Q8_0FloatTensor.java:100-117)."""
    m = make_model("tiny-llama", pkg.gguf.GGMLType.Q8_0, 16)
    a = orc.OracleModel(m, per_row_quant=False)
    b = orc.OracleModel(m, per_row_quant=True)
    tok = 3
    for pos in range(4):
        la, lb = a.forward(tok, pos), b.forward(tok, pos)
        assert np.array_equal(la.view(np.uint32), lb.view(np.uint32))
        tok = orc.argmax(la)


def test_argmax_first_max(orc):
    v = np.array([1, 5, 5, 2, 5], dtype=np.float32)
    assert orc.argmax(v) == 1
    assert orc.argmax(np.full(4, -np.inf, dtype=np.float32)) == 0


def test_rope_table(orc):
    cr, ci = orc.rope_table(4, 8, 500000.0)
    assert cr[0] == 1.0 and ci[0] == 0.0
    for pos in range(4):
        for k in range(4):
            freq = np.float32(1.0 / (500000.0 ** (2 * k / 8.0)))
            val = np.float32(np.float32(pos) * freq)
            assert cr[pos * 4 + k] == np.float32(np.cos(np.float64(val)))
            assert ci[pos * 4 + k] == np.float32(np.sin(np.float64(val)))


def _golden_cases(pkg):
    Q, F = pkg.gguf.GGMLType.Q8_0, pkg.gguf.GGMLType.F16
    return [("tiny-llama", Q, 16), ("tiny-llama-tied", F, 16), ("tiny-llama", F, 8), ("tiny-llama", F, 0), ("tiny-qwen3", Q, 16), ("tiny-qwen3", F, 16),
            ("tiny-phi3", Q, 16), ("tiny-phi3-gqa", F, 16)]


def kquant_golden(orc, pkg):
    """sha256 of the Q8_0 bytes the K-quant re-quantiser produces for seeded synthetic super-blocks (ModelLoader.java:173-224)."""
    out = {}
    for name in ("Q4_K", "Q5_K", "Q6_K"):
        tt = getattr(pkg.gguf.GGMLType, name)
        raw = pkg.synth.random_kquant(tt, 256 * 64, np.random.Generator(np.random.PCG64(tt)), zero_blocks=1)
        out[name] = {"src_sha256": hashlib.sha256(raw.tobytes()).hexdigest(), "q8_0_sha256": hashlib.sha256(orc.kquant_to_q8_0(tt, raw, 256 * 64).tobytes()).hexdigest()}
    return out


def golden_run(orc, pkg, make_model, shape, quant, lanes, n=12):
    m = make_model(shape, quant, 24, seed=1234)
    om = orc.OracleModel(m, lanes=lanes)
    # teacher-forced LlamaBench token stream (random models collapse to one token under greedy feedback)
    stream = orc.bench_tokens(m.configuration.vocab_size, n)
    toks, h = [], hashlib.sha256()
    for pos in range(n):
        lg = om.forward(int(stream[pos]), pos)
        h.update(lg.tobytes())
        toks.append(orc.argmax(lg))
    return {"input": [int(t) for t in stream], "argmax": toks, "logits_sha256": h.hexdigest()}


def test_golden_fixture(orc, pkg, make_model):
    """Regression pin of the oracle itself: tokens and a hash of all logits for seeded tiny
    models.  Self-generated (tests/golden/make_golden.py) -- the reference has no vectors."""
    with open(GOLDEN) as f:
        gold = json.load(f)
    for shape, quant, lanes in _golden_cases(pkg):
        key = f"{shape}/{pkg.gguf.GGMLType.NAMES[quant]}/lanes{lanes}"
        got = golden_run(orc, pkg, make_model, shape, quant, lanes)
        assert got == gold[key], key
    assert kquant_golden(orc, pkg) == gold["kquant_to_q8_0"]


def test_sampler_restatements_agree(pkg, orc):
    """SURVEY 8(f) N3 (parity unpinned: no JDK): the product's Python restatement of L32X64MixRandom equals the oracle's C
    restatement, and the oracle's C sampler (Sampler.java / CategoricalSampler.java / ToppSampler.java line by line, heap
    included) equals an independent numpy formulation on random logits."""
    for seed in (0, 1, 42, -7, 2 ** 40 + 3):
        a, b = pkg.sampler.L32X64MixRandom(seed), orc.JavaLXM(seed)
        assert [a.next_int() for _ in range(50)] == [b.next_int() for _ in range(50)]
        assert abs(a.next_float1() - b.next_float1()) == 0.0
    rng = np.random.default_rng(3)
    for t in range(200):
        n = int(rng.choice([17, 512, 4096]))
        lg = (rng.standard_normal(n) * 3).astype(np.float32)
        temp = float(rng.choice([0.0, 0.5, 1.0, 1.5]))
        topp = float(rng.choice([0.0, 0.3, 0.9, 0.95, 1.0]))
        r = float(np.float32(rng.random()))
        assert orc.sample(lg, temp, topp, r) == orc.np_sample(lg, temp, topp, r), (n, temp, topp, r)
    # first strict maximum for temperature 0 (FloatTensor.argmax)
    assert orc.sample(np.array([1.0, 3.0, 3.0, 2.0], dtype=np.float32), 0.0, 0.9, 0.5) == 1
    # real vocabulary sizes and the edges: flat rows, ties, masked (-inf) ids, overflowing logits / temperature, topp just below 1
    for n in (2, 512, 32064, 128256):
        flat = np.zeros(n, dtype=np.float32)
        normal = (rng.standard_normal(n) * 3).astype(np.float32)
        ties = (rng.integers(-12, 13, n) * 0.25).astype(np.float32)
        masked = normal.copy()
        masked[::7] = -np.inf
        for r in (0.0, 0.5, TOPP_BELOW_1):
            # no candidate passes the cutoff: the reference returns indices[0], which its tail fill set to n - 1
            assert orc.sample(flat, 1.0, 1e-7, r) == orc.np_sample(flat, 1.0, 1e-7, r, want_info=True)[0] == n - 1, n
            assert orc.np_sample(flat, 1.0, 1e-7, r, want_info=True)[1:] == (0, 0)
            # NaN probabilities (logit / 1e-38 overflows to inf): no candidate either
            if n > 2:
                assert orc.sample(normal, 1e-38, 0.9, r) == orc.np_sample(normal, 1e-38, 0.9, r) == n - 1, n
        for lg in (normal, ties, masked, flat):
            for temp, topp in ((0.7, 0.9), (0.3, 0.95), (1.0, 0.0), (1.0, TOPP_BELOW_1), (2.0, 0.99)):
                r = float(np.float32(rng.random()))
                want, probs = orc.sample(lg, temp, topp, r, want_probs=True)
                if 0 < topp < 1 and np.count_nonzero(probs >= np.float32(1 - np.float32(topp)) / np.float32(n - 1)) > 4000:
                    continue  # the Python heap is too slow for ~1e5 candidates; the GPU tests cover these against the C oracle
                assert want == orc.np_sample(lg, temp, topp, r), (n, temp, topp, r)


TOPP_BELOW_1 = float(np.float32(1.0) - np.float32(2.0 ** -24))  # 0x1.fffffep-1, the largest float below 1


def softmax_bound_violations(x: np.ndarray, p: np.ndarray) -> np.ndarray:
    """Elements where the float32 probabilities p of the float32 scaled logits x = f32(l / T) leave the float64 softmax by more
    than the error of the reference's float evaluation (max, rounded x - m, (float)Math.exp, sequential float sum, division):
    |p_i - p64_i| <= 1.01 p64_i (d_i + max d_j + u sum_k S_k / S + 3u) + 2^-149 with u = 2^-24, d_i = u (1 + |x_i - m|) and
    S_k the partial sums of the sequential sum."""
    u = 2.0 ** -24
    x64 = x.astype(np.float64)
    m = x64.max()
    with np.errstate(invalid="ignore"):
        e = np.where(np.isneginf(x64), 0.0, np.exp(x64 - m))
    S = e.sum()
    p64 = e / S
    d = u * (1.0 + np.where(np.isneginf(x64), 0.0, np.abs(x64 - m)))
    bound = 1.01 * p64 * (d + d.max() + u * np.cumsum(e).sum() / S + 3 * u) + 2.0 ** -149
    return np.flatnonzero(~(np.abs(p.astype(np.float64) - p64) <= bound))


def test_oracle_softmax_matches_float64(orc):
    """The oracle's probabilities (Sampler.java's divideInPlace + softmaxInPlace in float32) against the float64 softmax of the
    same scaled logits, at real vocabulary sizes and on rows whose exponentials underflow (to zero or to subnormals)."""
    rng = np.random.default_rng(11)
    for n in (2, 1000, 32064, 151936):
        normal = rng.standard_normal(n).astype(np.float32)
        masked = (normal * 3).astype(np.float32)
        masked[::7] = -np.inf
        peaked = normal.copy()
        peaked[n // 3] = normal.max() + 30
        rows = {"normal": normal, "masked": masked, "peaked": peaked, "wide": (normal * 30).astype(np.float32),
                "ties": (rng.integers(-12, 13, n) * 0.25).astype(np.float32), "flat": np.zeros(n, dtype=np.float32)}
        for name, lg in rows.items():
            for temp in (0.05, 0.3, 1.0, 2.0):
                _, p = orc.sample(lg, temp, 0.0, 0.5, want_probs=True)
                x = (lg / np.float32(temp)).astype(np.float32)
                bad = softmax_bound_violations(x, p)
                assert bad.size == 0, (n, name, temp, bad[:5], p[bad[:5]])
                assert np.all(p[np.isneginf(lg)] == 0)
                if name == "flat":
                    assert np.all(p == np.float32(1) / np.float32(n))
