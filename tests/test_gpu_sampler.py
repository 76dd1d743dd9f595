"""SURVEY 8(f) N3: the device-side temperature / top-p sampler (csrc/sampler.cuh behind b200_forward_decode_sample) against the
oracle's restatement of Sampler.java / CategoricalSampler.java / ToppSampler.java: same logits (bit-exact forward), same uniform
number -> same token id, for greedy, categorical and top-p sampling.  The kernel alone (b200_test_sample) is held to the C oracle at
the real vocabulary sizes on rows built to hit its edges: probabilities bit-equal, same id, same candidate and kept counts."""
import math
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TOPP_BELOW_1 = float(np.float32(1.0) - np.float32(2.0 ** -24))  # 0x1.fffffep-1: the cumulative sum may never pass it
FAMILY_DEFAULTS = [(0.3, 0.95), (0.8, 0.9), (0.7, 0.9)]  # Llama, Qwen3, the other chat formats (defaultTemperature / defaultTopP)
MODES = ["graph", "persistent"]


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


# 2; not whole 1024-thread chunks; Phi-3 (E = 32 terms per thread, 16-byte loads); Llama-3 (E = 126); Qwen3 (E = 149)
VOCABS = [2, 1000, 4097, 32064, 128256, 151936]
ROWS = ["normal1", "normal3", "peaked", "ties", "flat", "masked", "wide", "drift"]
SETTINGS = FAMILY_DEFAULTS + [
    (1.0, 0.0), (1.0, 1.0),    # categorical
    (2.0, 0.99),               # many candidates
    (1.0, TOPP_BELOW_1),
    (1.0, 1e-7),               # no candidate on flat rows
    (1.0, 0.5),                # at n = 2 a flat row's probabilities equal the cutoff
    (1e-38, 0.9), (1e-38, 0.0),  # logit / T overflows: NaN probabilities
    (math.inf, 0.9),           # every row flat
    (0.05, 0.9),               # most exponentials underflow on the wide row
]


def make_row(kind: str, n: int, rng) -> np.ndarray:
    if kind in ("normal1", "normal3"):
        return (rng.standard_normal(n) * (1.0 if kind == "normal1" else 3.0)).astype(np.float32)
    if kind == "peaked":  # the sum is 1 plus terms below half an ulp
        lg = rng.standard_normal(n).astype(np.float32)
        lg[int(rng.integers(n))] = lg.max() + 30
        return lg
    if kind == "ties":  # many exactly equal probabilities: the heap's tie order decides
        return (rng.integers(-12, 13, n) * 0.25).astype(np.float32)
    if kind == "flat":
        return np.full(n, 0.5, dtype=np.float32)
    if kind == "masked":  # every 7th id, and Llama-3's reserved special tokens where the vocabulary has them
        lg = (rng.standard_normal(n) * 2).astype(np.float32)
        lg[::7] = -np.inf
        lg[128002:128256] = -np.inf
        return lg
    if kind == "drift":
        return drift_row(n)
    assert kind == "wide"
    return (rng.standard_normal(n) * 30).astype(np.float32)


def drift_row(n: int) -> np.ndarray:
    """At T = 1: 4096 terms 1.0 (the sum reaches 2^12 exactly), then terms t whose fraction of the binade's ulp 2^-11 is 0.55, so
    every sequential add rounds up by 0.45 ulp.  From n ~ 127500 on, the sequential sum crosses 2^13 while the exact prefix is still
    0.33 % below it -- past the 2^-9 margin of the exact sum's binade predictor (seqsum2.cuh), so only its verification keeps the
    result exact."""
    U = 2.0 ** -11
    c = np.float32(np.log(67.55 * U))
    assert 0.54 < float(np.float32(np.exp(np.float64(c)))) / U % 1.0 < 0.56
    lg = np.zeros(n, dtype=np.float32)
    lg[4096:] = c
    return lg


@pytest.mark.parametrize("n", VOCABS)
def test_sample_kernel_matches_oracle(pkg, orc, n):
    """Every row x (temperature, topp) x uniform number: the kernel's probabilities bit-equal to the oracle's (NaN where the
    reference produces NaN), the same token id, the same number of top-p candidates and of kept tokens.  At 128256 / 151936 tokens
    the softmax denominator is the exact sequential sum over 126 / 149 terms per thread, read from global memory."""
    rng = np.random.default_rng(n)
    lxm = orc.JavaLXM(2024)
    rs = [0.0, TOPP_BELOW_1, lxm.next_float1(), lxm.next_float1()]
    seqsum = {}
    for kind in ROWS:
        lg = make_row(kind, n, rng)
        t0 = time.perf_counter()
        checked_t = set()
        for temp, topp in SETTINGS:
            use_topp = 0 < topp < 1
            for r in rs:
                got, info, probs = pkg.native.test_sample(lg, temp, topp, r)
                want, ref = orc.sample(lg, temp, topp, r, want_probs=True)
                what = (n, kind, temp, topp, r, got, want, info)
                if temp not in checked_t:  # the probabilities depend on (row, T) only
                    checked_t.add(temp)
                    nan = np.isnan(ref)
                    assert np.array_equal(np.isnan(probs), nan), what
                    bad = np.flatnonzero(bits(probs)[~nan] != bits(ref)[~nan])
                    assert bad.size == 0, (what, bad[:5], probs[~nan][bad[:5]], ref[~nan][bad[:5]])
                    seqsum[(kind, temp)] = info[2:]
                assert got == want, what
                if not use_topp:
                    assert info[:2] == [n, n], what
                    continue
                cutoff = np.float32(np.float32(1.0) - np.float32(topp)) / np.float32(n - 1)
                n0 = int(np.count_nonzero(ref >= cutoff))
                assert info[0] == n0, what
                if n0 == 0:
                    assert got == n - 1 and info[1] == 0, what
                elif n0 <= 2000:
                    assert orc.np_sample(lg, temp, topp, r, want_info=True) == (want, n0, info[1]), what
                else:
                    assert 0 < info[1] <= n0, what
        print(f"\n  n={n} {kind}: {len(SETTINGS) * len(rs)} calls in {time.perf_counter() - t0:.2f} s", end="")
    if n >= 32064:
        worst = max(seqsum, key=lambda k: seqsum[k][1])
        print(f"\n  n={n} seqsum [items, fallbacks]: normal1 T=1 {seqsum[('normal1', 1.0)]}, drift T=1 {seqsum[('drift', 1.0)]}, "
              f"most fallbacks {worst} {seqsum[worst]}, "
              f"most items {max(v[0] for v in seqsum.values())}", end="")


def test_sample_hook_rejects_bad_arguments(pkg):
    lg = np.zeros(8, dtype=np.float32)
    for args in [(np.zeros(0, dtype=np.float32), 1.0, 0.9, 0.5), (lg, 0.0, 0.9, 0.5), (lg, -1.0, 0.9, 0.5), (lg, math.nan, 0.9, 0.5),
                 (lg, 1.0, 0.9, -0.25), (lg, 1.0, 0.9, 1.0), (lg, 1.0, 0.9, math.nan)]:
        with pytest.raises(pkg.native.B200Error) as e:
            pkg.native.test_sample(*args)
        assert e.value.code == -1, args
    assert pkg.native.test_sample(lg, 1.0, 0.9, 0.5)[0] in range(8)


CASES = [(0.0, 0.95), (1.0, 0.0), (0.7, 1.0), (1.0, 0.95), (0.1, 0.95), (1.3, 0.5), (0.8, 0.9), (2.0, 0.99)]
REAL_VOCAB_CASES = FAMILY_DEFAULTS + [(1.0, 0.0), (1.0, 1.0), (0.0, 0.9)]  # the chat defaults, categorical, greedy


def real_vocab_model(pkg, shape, ctx, classifier_zero=False):
    sh = pkg.synth.SHAPES[shape]
    Q8 = pkg.gguf.GGMLType.Q8_0
    tensors = pkg.synth.build_tensors_fast(sh, Q8, seed=1234)
    if classifier_zero:
        tt, dims, raw = tensors["output.weight"]
        tensors["output.weight"] = (tt, dims, np.zeros_like(raw))
    return pkg.loader.model_from_tensors(sh, Q8, tensors, ctx)


@pytest.mark.parametrize("shape", ["tiny-llama", "small-llama", "tiny-llama-vocab128k", "tiny-qwen3-vocab152k", "tiny-phi3-vocab32k"])
def test_device_sampler_matches_oracle(pkg, orc, make_model, shape):
    """Small vocabularies: 32 positions x 8 settings on the default decode path.  Real vocabularies (Llama-3 128256, Qwen3 151936,
    Phi-3 32064 on the tiny geometries): 16 positions through the chat defaults, categorical and greedy, in each decode mode."""
    real = pkg.synth.SHAPES[shape].vocab > 4096
    m = real_vocab_model(pkg, shape, 24) if real else make_model(shape, pkg.gguf.GGMLType.Q8_0, 48)
    c = m.configuration
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = orc.OracleModel(m)
    stream = orc.bench_tokens(c.vocab_size, 40)
    cases, n_pos, modes = (REAL_VOCAB_CASES, 16, MODES) if real else (CASES, 32, ["graph"])
    ran = []
    try:
        for mode in modes:
            try:
                plan.set_decode_mode(mode)
            except pkg.native.UnsupportedOperation:
                continue  # the persistent kernel needs head size 64 / 128 (Phi-3's 96 runs the graph only)
            ran.append(mode)
            rng = orc.JavaLXM(12345)
            for pos in range(n_pos):
                temp, topp = cases[pos % len(cases)]
                r = rng.next_float1()
                tok = int(stream[pos])
                got, info = plan.forward_decode_sample(tok, pos, temp, topp, r, want_info=True)
                want = orc.sample(om.forward(tok, pos), temp, topp, r)
                assert got == want, (mode, pos, temp, topp, r, got, want, info)
                if temp > 0 and 0 < topp < 1:
                    assert 0 < info[1] <= info[0] <= c.vocab_size
        assert "graph" in ran
    finally:
        plan.free()
        om.close()


def test_device_sampler_empty_topp_set_returns_last_id(pkg, orc):
    """A classifier of zeros makes every logit 0: with topp 1e-7 no token reaches the cutoff (1 - topp) / (n - 1) > 1 / n, and the
    reference returns n - 1 (its indices[0] after the tail fill).  The plan's index scratch still holds the previous call's heap."""
    m = real_vocab_model(pkg, "tiny-llama-vocab128k", 8, classifier_zero=True)
    n = m.configuration.vocab_size
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = orc.OracleModel(m)
    try:
        lg, _ = plan.forward_decode(5, 0)
        assert not np.any(lg) and not np.any(om.forward(5, 0))
        got, info = plan.forward_decode_sample(7, 1, 1.0, 0.9, 0.25, want_info=True)
        assert got == orc.sample(om.forward(7, 1), 1.0, 0.9, 0.25) and info[0] == n, (got, info)
        got, info = plan.forward_decode_sample(9, 2, 1.0, 1e-7, 0.25, want_info=True)
        assert orc.sample(om.forward(9, 2), 1.0, 1e-7, 0.25) == n - 1
        assert got == n - 1 and info[:2] == [0, 0], (got, info)
    finally:
        plan.free()
        om.close()


def test_sampler_object_drives_a_generation(pkg, orc, make_model):
    """Sampler.selectSampler's object over the plan vs the same loop over the oracle with the oracle's RNG restatement."""
    m = make_model("tiny-llama", pkg.gguf.GGMLType.Q8_0, 40)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = orc.OracleModel(m)
    smp = pkg.sampler.select_sampler(m.configuration.vocab_size, 0.8, 0.95, 42)
    rng = orc.JavaLXM(42)
    tok_g = tok_o = 3
    for pos in range(24):
        tok_g = smp.sample_token(plan, tok_g, pos)
        tok_o = orc.sample(om.forward(tok_o, pos), 0.8, 0.95, rng.next_float1())
        assert tok_g == tok_o, pos
    plan.free()
    om.close()
