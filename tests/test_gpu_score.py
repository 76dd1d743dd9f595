"""GPU tests of token scoring (b200_score_tokens, csrc/score.cuh): per-row log-probabilities and greedy ids from the prefill paths.
Bar: greedy ids equal the oracle's teacher-forced argmax, log-probabilities within 1e-9 of the float64 log-softmax of the oracle's
logits (test_score_host.score_rows), and every path's outputs bit-identical to every other's on one plan."""
import re

import numpy as np
import pytest

import hostile
from test_gpu_kquant_resident import _model, _oracle, _resident_plan
from test_gpu_parity import assert_bit_equal, mid_model
from test_score_host import score_rows

pytestmark = pytest.mark.gpu

G = hostile.G
MODES = ("exact", "tensor_core_exact")


def _modes(pkg, plan):
    """The scoring modes the plan admits."""
    out = []
    for mode in MODES:
        try:
            plan.set_prefill_mode(mode)
            out.append(mode)
        except pkg.native.UnsupportedOperation:
            pass
    return out


def _oracle_logits(om, toks, n):
    om.reset()
    return np.stack([om.forward(int(toks[p]), p) for p in range(n)])


def _bits(a):
    return np.asarray(a, np.float64).view(np.uint64)


def _score_in_every_mode(pkg, plan, om, c, chunks, seed=3):
    """Scores the chunks from position 0 in every mode the plan admits; each against the oracle, and all modes bit-equal."""
    end = max(s + n for s, n in chunks)
    toks = np.random.default_rng(seed).integers(0, c.vocab_size, end + 1).astype(np.int32)
    lp_ref, ids_ref = score_rows(_oracle_logits(om, toks, end), toks[1:end + 1])
    runs = {}
    for mode in _modes(pkg, plan):
        plan.set_prefill_mode(mode)
        plan.kv_reset()
        lp, ids = np.empty(end), np.empty(end, np.int32)
        for s, n in chunks:
            lp[s:s + n], ids[s:s + n] = plan.score_tokens(toks[s:s + n], s, toks[s + 1:s + n + 1])
        assert np.array_equal(ids, ids_ref), f"{mode}: greedy ids differ at {np.flatnonzero(ids != ids_ref)[:8]}"
        err = np.abs(lp - lp_ref)
        assert err.max() <= 1e-9, f"{mode}: logprob error {err.max()} at row {err.argmax()}"
        runs[mode] = (lp, ids)
    assert "exact" in runs
    for mode, (lp, ids) in runs.items():
        assert np.array_equal(_bits(lp), _bits(runs["exact"][0])) and np.array_equal(ids, runs["exact"][1]), f"{mode} differs from exact"
    return runs


CHUNKS = [(0, 40), (40, 37)]  # the second chunk's length is not a multiple of 64


@pytest.mark.parametrize("shape,quant", [("tiny-llama", G.Q8_0), ("tiny-llama-tied", G.Q8_0), ("tiny-qwen3", G.Q8_0), ("tiny-qwen2", G.Q8_0),
                                         ("tiny-phi3", G.Q8_0), ("tiny-phi3-gqa", G.Q8_0), ("tiny-granite", G.Q8_0), ("tiny-devstral", G.Q8_0),
                                         ("tiny-llama-vocab128k", G.Q8_0), ("tiny-qwen3-vocab152k", G.Q8_0), ("tiny-llama", G.F16),
                                         ("tiny-qwen2moe", G.Q8_0)])
def test_scores_are_the_oracle(pkg, orc, make_model, shape, quant):
    m = make_model(shape, quant, ctx=96, seed=21)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=64)
    om = hostile.oracle_for(orc, m)
    try:
        runs = _score_in_every_mode(pkg, plan, om, m.configuration, CHUNKS)
        if quant == G.Q8_0 and shape != "tiny-qwen2moe":
            assert set(runs) == set(MODES)
    finally:
        plan.free()
        om.close()


def test_mid_granite_vocab_49155(pkg, orc):
    m = mid_model(pkg, "mid-granite-3-2b", 96)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=64)
    om = hostile.oracle_for(orc, m)
    try:
        assert set(_score_in_every_mode(pkg, plan, om, m.configuration, CHUNKS)) == set(MODES)
    finally:
        plan.free()
        om.close()


@pytest.mark.parametrize("resident", [False, True])
def test_kquant_file(pkg, orc, resident):
    """A Q4_K_M file on its Q8_0-tile plan and on a resident plan (the classifier, Q6_K, expanded before its GEMM)."""
    m = _model(pkg, "tiny-llama", "Q4_K_M", ctx=96, seed=22)
    plan = _resident_plan(pkg, m, prefill_batch_size=64) if resident else pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=64)
    om = _oracle(pkg, orc, m)
    try:
        assert set(_score_in_every_mode(pkg, plan, om, m.configuration, CHUNKS)) == set(MODES)
    finally:
        plan.free()
        om.close()


@pytest.mark.parametrize("resident", [False, True])
def test_mid_llama_against_its_own_decode(pkg, resident):
    """8B layer geometry: logprobs are the float64 log-softmax of forward_decode's logits for the same tokens, ids its argmax."""
    if resident:
        m = _model(pkg, "mid-llama", "Q4_K_M", ctx=80, seed=23)
        plan = _resident_plan(pkg, m, prefill_batch_size=64)
    else:
        m = mid_model(pkg, "mid-llama", 80)
        plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=64)
    c = m.configuration
    toks = np.random.default_rng(4).integers(0, c.vocab_size, 49).astype(np.int32)
    try:
        rows, ids_dec = [], []
        for p in range(48):
            lg, am = plan.forward_decode(int(toks[p]), p)
            rows.append(lg.copy())
            ids_dec.append(am)
        lp_ref, ids_ref = score_rows(np.stack(rows), toks[1:])
        assert list(ids_ref) == ids_dec
        for mode in MODES:
            plan.set_prefill_mode(mode)
            plan.kv_reset()
            lp, ids = plan.score_tokens(toks[:48], 0, toks[1:])
            assert np.array_equal(ids, ids_ref), mode
            assert np.abs(lp - lp_ref).max() <= 1e-9, mode
    finally:
        plan.free()


def test_determinism_chunking_and_repeats(pkg, make_model):
    """One 96-token call, calls of 64 + 32, and a repeated call give the same bits, in both modes."""
    m = make_model("tiny-qwen3", G.Q8_0, ctx=128, seed=24)
    c = m.configuration
    toks = np.random.default_rng(5).integers(0, c.vocab_size, 97).astype(np.int32)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=96)
    try:
        outs = []
        for mode in MODES:
            plan.set_prefill_mode(mode)
            for split in ((96,), (64, 32), (96,)):
                plan.kv_reset()
                lp, ids, s = [], [], 0
                for n in split:
                    a, b = plan.score_tokens(toks[s:s + n], s, toks[s + 1:s + n + 1])
                    lp.append(a)
                    ids.append(b)
                    s += n
                outs.append((mode, split, np.concatenate(lp), np.concatenate(ids)))
        for mode, split, lp, ids in outs[1:]:
            assert np.array_equal(_bits(lp), _bits(outs[0][2])) and np.array_equal(ids, outs[0][3]), (mode, split)
    finally:
        plan.free()


@pytest.mark.parametrize("mode", MODES)
def test_cache_after_scoring_is_the_prefill_cache(pkg, make_model, mode):
    """After score_tokens the KV cache equals forward_batch_prefill's of the same tokens, and decoding continues with the same logits."""
    m = make_model("tiny-llama", G.Q8_0, ctx=96, seed=25)
    c = m.configuration
    toks = np.random.default_rng(6).integers(0, c.vocab_size, 51).astype(np.int32)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=64)
    nkv = c.context_length * c.kv_dim
    try:
        plan.set_prefill_mode(mode)
        state = []
        for score in (True, False):
            plan.kv_reset()
            if score:
                plan.score_tokens(toks[:50], 0)
            else:
                plan.forward_batch_prefill(toks[:50], 0)
            kv = [plan.read_buffer(n, nkv, layer=l).copy() for n in ("key_cache", "value_cache") for l in range(c.n_layers)]
            ids, _ = plan.decode_sequence(toks[50:], 8, 50, feedback=True)
            lg, _ = plan.forward_decode(int(ids[-1]), 58)
            state.append((kv, ids, lg))
        for i, (a, b) in enumerate(zip(state[0][0], state[1][0])):
            assert_bit_equal(a, b, f"cache buffer {i}")
        assert np.array_equal(state[0][1], state[1][1])
        assert_bit_equal(state[0][2], state[1][2], "logits after the greedy continuation")
    finally:
        plan.free()


@pytest.mark.parametrize("kind", ["group", "warps", "ctas", "padding"])
def test_tied_maxima_take_the_first_index(pkg, orc, kind):
    m = hostile.tied_logits("tiny-llama", G.Q8_0, kind, ctx=32)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=32)
    om = hostile.oracle_for(orc, m)
    try:
        runs = _score_in_every_mode(pkg, plan, om, m.configuration, [(0, 20)], seed=8)
        A, B = hostile.tie_rows(kind, m.configuration.vocab_size)
        assert set(runs["exact"][1].tolist()) <= {min(A), min(B)}, runs["exact"][1]
    finally:
        plan.free()
        om.close()


def test_saturated_softmax(pkg, orc):
    """Eight classifier rows scaled by 2^14: where one of them leads by far, logprob(greedy) is within 1e-12 of 0 and every other
    log-probability is finite and very negative."""
    sh, t = hostile.base_tensors("tiny-llama", G.Q8_0, 42)
    hostile.scale_rows(t["output.weight"], 0, 8, 14)
    m = pkg.loader.model_from_tensors(sh, G.Q8_0, t, 32)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=32)
    om = hostile.oracle_for(orc, m)
    try:
        c = m.configuration
        toks = np.random.default_rng(9).integers(0, c.vocab_size, 25).astype(np.int32)
        runs = _score_in_every_mode(pkg, plan, om, c, [(0, 24)], seed=9)
        lg = _oracle_logits(om, toks, 24)
        srt = np.sort(lg.astype(np.float64), axis=1)
        sat = srt[:, -1] - srt[:, -2] > 60
        assert sat.any(), "no row saturates"
        for mode, _ in runs.items():
            plan.set_prefill_mode(mode)
            plan.kv_reset()
            lp_g, ids = plan.score_tokens(toks[:24], 0, np.zeros(24, np.int32) - 1)
            plan.kv_reset()
            other = (ids + 1) % c.vocab_size
            lp_o, _ = plan.score_tokens(toks[:24], 0, other)
            plan.kv_reset()
            lp_self, _ = plan.score_tokens(toks[:24], 0, ids)
            assert np.isnan(lp_g).all()
            assert np.all(np.abs(lp_self[sat]) <= 1e-12), lp_self[sat]
            assert np.isfinite(lp_o).all() and np.all(lp_o[sat] < -60)
    finally:
        plan.free()
        om.close()


@pytest.mark.parametrize("mode", MODES)
def test_perplexity_700_positions(pkg, orc, make_model, mode):
    m = make_model("tiny-llama", G.Q8_0, ctx=720, seed=26)
    c = m.configuration
    toks = [int(t) for t in orc.bench_tokens(c.vocab_size, 700, seed=10)]
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=256)
    om = hostile.oracle_for(orc, m)
    try:
        plan.set_prefill_mode(mode)
        got = pkg.engine.perplexity(plan, toks)
        lp_ref, _ = score_rows(_oracle_logits(om, toks, 699), np.asarray(toks[1:]))
        want = float(np.exp(-lp_ref.mean()))
        assert abs(got - want) <= 1e-9 * want, (got, want)
    finally:
        plan.free()
        om.close()


def _decodes_like_the_oracle(plan, om, what):
    plan.kv_reset()
    om.reset()
    tok = 1
    for pos in range(4):
        lg, am = plan.forward_decode(tok, pos)
        assert_bit_equal(lg, om.forward(tok, pos), f"{what}: logits at {pos}")
        tok = am


def test_refusals_and_errors(pkg, orc, make_model):
    m = make_model("tiny-llama", G.Q8_0, ctx=64, seed=27)
    c = m.configuration
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=16)
    om = hostile.oracle_for(orc, m)
    toks = np.arange(1, 17, dtype=np.int32)
    try:
        for mode in ("tensor_core", "tensor_core_w8a16"):
            plan.set_prefill_mode(mode)
            with pytest.raises(pkg.native.UnsupportedOperation) as e:
                plan.score_tokens(toks, 0)
            assert "exact" in str(e.value) and "tensor_core_exact" in str(e.value), str(e.value)
            _decodes_like_the_oracle(plan, om, f"after the {mode} refusal")
        for mode in MODES:
            plan.set_prefill_mode(mode)
            for args, pat in (((toks, 0, np.full(16, c.vocab_size, np.int32)), "target"), ((toks, 0, np.full(16, -2, np.int32)), "target"),
                              ((np.full(16, c.vocab_size, np.int32), 0, None), "token"), ((toks, c.context_length - 8, None), "outside the KV cache"),
                              ((np.ones(17, np.int32), 0, None), "exceeds prefill_batch_size")):
                with pytest.raises(pkg.native.B200Error) as e:
                    plan.score_tokens(*args)
                assert e.value.code == -1 and pat in str(e.value), (mode, str(e.value))
            _decodes_like_the_oracle(plan, om, f"after the {mode} argument errors")
        plan.set_prefill_mode("tensor_core_exact")
        pkg.native.test_set_memory_budget(1)
        try:
            with pytest.raises(pkg.native.B200Error) as e:
                plan.score_tokens(toks, 0)
        finally:
            pkg.native.test_set_memory_budget(0)
        assert e.value.code == -3 and re.search(r"\b[1-9]\d* bytes of logits scratch", str(e.value)), str(e.value)
        _decodes_like_the_oracle(plan, om, "after the memory refusal")
        plan.kv_reset()
        plan.score_tokens(toks, 0)  # with the real figure the scratch is allocated
    finally:
        plan.free()
        om.close()


@pytest.mark.parametrize("resident", [False, True])
def test_launch_count(pkg, resident):
    """A tensor_core_exact score call launches the prefill's kernels plus the final norm, the classifier GEMM and the reduction (one
    group of up to 256 rows), and on a resident plan whose classifier is resident (Q6_K here) its expansion."""
    m = _model(pkg, "tiny-llama", "Q4_K_M", ctx=64, seed=28)
    plan = _resident_plan(pkg, m, prefill_batch_size=48) if resident else pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=48)
    toks = np.arange(3, 43, dtype=np.int32)
    try:
        plan.set_prefill_mode("tensor_core_exact")
        plan.forward_batch_prefill(toks, 0)
        base = plan.prefill_info()[1]
        plan.kv_reset()
        plan.score_tokens(toks, 0)
        assert plan.prefill_info()[1] == base + 3 + (1 if resident else 0), (base, plan.prefill_info())
    finally:
        plan.free()
