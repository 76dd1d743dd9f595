"""GPU tests on hostile values: every decode path against the CPU oracle, bit for bit (logits as uint32, ids equal, KV caches where the
model touches attention), on the models of tests/hostile.py -- tied logits, activation outliers and all-zero rows in every RMSNorm,
saturated softmax and SwiGLU, Q8_0 / FP16 weight blocks the project's own quantiser never writes.  tests/test_hostile_host.py shows on
the CPU that each model really has its property."""
import numpy as np
import pytest

import hostile as H
from test_gpu_parity import assert_bit_equal, set_mode
from test_gpu_prefill_w8a16 import _run_modes

pytestmark = pytest.mark.gpu

Q8, F16 = H.G.Q8_0, H.G.F16
S = H.synth.Shape

# (shape, quant, decode mode, FP16 lanes): the Q8_0 stream in both decode modes, the FP16 rings at 16 and 8 lanes, and the round-1
# FP16 kernels (tiny-phi3: dim 384 is not a multiple of 256), whose classifier is followed by the full-pass argmax
PATHS = [("tiny-llama", Q8, "graph", 16), ("tiny-llama", Q8, "persistent", 16), ("tiny-llama", F16, "graph", 16),
         ("tiny-llama", F16, "graph", 8), ("tiny-phi3", F16, "graph", 16)]
PATH_IDS = ["q8-graph", "q8-persistent", "f16-rings16", "f16-rings8", "f16-round1"]


def _check_kv(plan, om, c, n_pos=None):
    nkv = c.context_length * c.kv_dim
    n = nkv if n_pos is None else n_pos * c.kv_dim
    for l in range(c.n_layers):
        assert_bit_equal(plan.read_buffer("key_cache", nkv, layer=l)[:n], om.key_cache(l)[:n], f"key cache layer {l}")
        assert_bit_equal(plan.read_buffer("value_cache", nkv, layer=l)[:n], om.value_cache(l)[:n], f"value cache layer {l}")


def _decode(pkg, orc, m, toks, mode="graph", lanes=16, feedback=0, kv=True, check=None):
    """forward_decode over toks (then `feedback` more steps on its own greedy ids) against the oracle; check: the positions whose logits
    are compared (the others go through forward_prefill)."""
    plan = pkg.B200MasterPlan.initialize_plan(m, fp16_lanes=lanes)
    set_mode(pkg, plan, mode)
    om = H.oracle_for(orc, m, lanes)
    try:
        tok = None
        for pos in range(len(toks) + feedback):
            tok = int(toks[pos]) if pos < len(toks) else tok
            if check is not None and pos not in check:
                plan.forward_prefill(tok, pos)
                om.forward(tok, pos, want_logits=False)
                continue
            lg, am = plan.forward_decode(tok, pos)
            ref = om.forward(tok, pos)
            assert_bit_equal(lg, ref, f"logits pos {pos} (token {tok})")
            assert am == orc.argmax(ref), f"argmax pos {pos} (token {tok}): {am} != {orc.argmax(ref)}"
            tok = am
        if kv:
            _check_kv(plan, om, m.configuration, len(toks) + feedback)
    finally:
        plan.free()
        om.close()


def _batch(pkg, orc, m, row_tokens, n_steps, feedback=True, check_from=0):
    """len(row_tokens) sequences in lockstep on their own slots, row r starting from row_tokens[r] (feedback) or walking the list
    row_tokens[r] (no feedback): every row's ids and logits against its own oracle sequence."""
    n = len(row_tokens)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    oms = [H.oracle_for(orc, m) for _ in range(n)]
    try:
        plan.set_decode_slots(n)
        toks = [int(t if feedback else t[0]) for t in row_tokens]
        for step in range(n_steps):
            ids, lg = plan.forward_decode_batch(list(range(n)), toks, [step] * n, logits=True)
            for r in range(n):
                ref = oms[r].forward(toks[r], step)
                if step >= check_from:
                    assert_bit_equal(lg[r], ref, f"row {r} step {step} (token {toks[r]})")
                    assert ids[r] == orc.argmax(ref), f"row {r} step {step} (token {toks[r]})"
                toks[r] = int(ids[r]) if feedback else int(row_tokens[r][(step + 1) % len(row_tokens[r])])
    finally:
        plan.free()
        for om in oms:
            om.close()


def _multi_and_step(pkg, orc, m, toks):
    """forward_decode_multi over toks, decode_multi_rows() positions per step on the plan's own cache, then one forward_step that mixes a decode row of
    slot 0, three prompt rows and a decode row of slot 1: ids, logits and the KV cache against the oracle."""
    c = m.configuration
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om, om0, om1 = (H.oracle_for(orc, m) for _ in range(3))
    try:
        R = plan.decode_multi_rows()
        assert R >= 6
        for off in range(0, len(toks), R):
            chunk = [int(t) for t in toks[off:off + R]]
            ids, lg = plan.forward_decode_multi(-1, chunk, off, logits=True)
            for i, tok in enumerate(chunk):
                ref = om.forward(tok, off + i)
                assert_bit_equal(lg[i], ref, f"multi: position {off + i} (token {tok})")
                assert ids[i] == orc.argmax(ref), f"multi: position {off + i} (token {tok})"
        _check_kv(plan, om, c, len(toks))
        plan.set_decode_slots(2)
        t = [int(x) for x in toks[:6]]
        rows = [(0, t[0], 0, 1), (1, t[1], 0, 0), (1, t[2], 1, 0), (1, t[3], 2, 1), (0, t[4], 1, 0), (0, t[5], 2, 1)]
        ids, lg = plan.forward_step(rows, logits=True)
        for i, (s, tok, pos, emit) in enumerate(rows):
            ref = (om0 if s == 0 else om1).forward(tok, pos)
            if emit:
                assert_bit_equal(lg[i], ref, f"step: row {i} (token {tok})")
                assert ids[i] == orc.argmax(ref), f"step: row {i} (token {tok})"
            else:
                assert ids[i] == -1
    finally:
        plan.free()
        for o in (om, om0, om1):
            o.close()


# ---- tied logits ---------------------------------------------------------------------------------------------------------------

TIE_PATHS = PATHS + [("tiny-llama-tied", Q8, "graph", 16), ("tiny-llama-tied", Q8, "persistent", 16), ("tiny-llama-tied", F16, "graph", 8),
                     ("tiny-llama-vocab509", Q8, "graph", 16), ("tiny-llama-vocab509", Q8, "persistent", 16), ("tiny-qwen3", F16, "graph", 16)]
TIE_IDS = PATH_IDS + ["q8-tied-graph", "q8-tied-persistent", "f16-tied-rings8", "q8-vocab509-graph", "q8-vocab509-persistent", "f16-qwen3-tied"]


@pytest.mark.parametrize("kind", ["group", "warps", "ctas", "padding"])
@pytest.mark.parametrize("shape,quant,mode,lanes", TIE_PATHS, ids=TIE_IDS)
def test_tied_logits_lowest_index_wins(pkg, orc, shape, quant, mode, lanes, kind):
    """16 greedy steps from an even and from an odd token: at every step several rows share the maximum logit, and the id is the lowest."""
    m = H.tied_logits(shape, quant, kind)
    for start in (4, 7):
        _decode(pkg, orc, m, [start], mode, lanes, feedback=15)


@pytest.mark.parametrize("kind", ["identical", "zero"])
@pytest.mark.parametrize("shape,quant,mode,lanes", PATHS, ids=PATH_IDS)
def test_degenerate_classifier_answers_zero(pkg, orc, shape, quant, mode, lanes, kind):
    """Every logit equal (one row repeated, or an all-zero classifier with zeros of both signs): the id is 0 and the logits' signs match."""
    _decode(pkg, orc, H.tied_logits(shape, quant, kind), [4, 7, 300, 1], mode, lanes)


@pytest.mark.parametrize("mode", ["graph", "persistent"])
@pytest.mark.parametrize("shape,kind", [("tiny-llama", "group"), ("tiny-llama", "warps"), ("tiny-llama-vocab509", "padding"), ("tiny-llama-tied", "ctas")])
def test_tied_logits_device_loop_follows_the_oracle(pkg, orc, shape, kind, mode):
    """decode_sequence with feedback: the device-resident greedy loop, 20 steps on its own ids."""
    m = H.tied_logits(shape, Q8, kind)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    set_mode(pkg, plan, mode)
    om = H.oracle_for(orc, m)
    try:
        for start in (4, 7):
            om.reset()
            plan.kv_reset()
            ids, _ = plan.decode_sequence([start], 20, 0, feedback=True)
            tok = start
            for pos in range(20):
                tok = orc.argmax(om.forward(tok, pos))
                assert ids[pos] == tok, f"start {start} step {pos}: {ids[pos]} != {tok}"
    finally:
        plan.free()
        om.close()


@pytest.mark.parametrize("n_rows", [1, 3, 8])
@pytest.mark.parametrize("shape,kind", [("tiny-llama", "warps"), ("tiny-llama-vocab509", "padding"), ("tiny-llama", "zero")])
def test_tied_logits_batched(pkg, orc, shape, kind, n_rows):
    _batch(pkg, orc, H.tied_logits(shape, Q8, kind), [4, 7, 2, 9, 300, 301, 0, 5][:n_rows], 8)


@pytest.mark.parametrize("kind", ["warps", "ctas"])
def test_tied_logits_multi_position_and_mixed_step(pkg, orc, kind):
    _multi_and_step(pkg, orc, H.tied_logits("tiny-llama", Q8, kind), [4, 7, 2, 9, 300, 301, 0, 5, 6, 13, 8])


@pytest.mark.parametrize("kind", ["ctas", "identical"])
@pytest.mark.parametrize("quant,mode,lanes", [(Q8, "graph", 16), (Q8, "persistent", 16), (F16, "graph", 16)], ids=["q8-graph", "q8-persistent", "f16"])
def test_tied_logits_at_vocab_128k(pkg, orc, quant, mode, lanes, kind):
    """ctas: the first and the last of 128256 rows tie; every CTA of the classifier launch holds a partial, and the merge must keep row 0.
    identical: all 128256 logits are equal, so every lane's own running maximum meets ties among the many rows it walks (at 512 rows a
    warp sees one 4-row group and a lane one row) and must keep its first."""
    m = H.tied_logits("tiny-llama-vocab128k", quant, kind, ctx=8)
    _decode(pkg, orc, m, [4, 7, 128255], mode, lanes, feedback=2, kv=False)


# ---- activation outliers in every norm -----------------------------------------------------------------------------------------

ALL_KINDS = list(H.OUTLIER_TOKEN.values())


@pytest.mark.parametrize("shape,quant,mode,lanes", PATHS + [("tiny-qwen2moe", Q8, "graph", 16), ("tiny-qwen3", Q8, "graph", 16), ("small-llama", Q8, "graph", 16),
                                                            ("small-llama", Q8, "persistent", 16), ("tiny-llama-gqa8", Q8, "persistent", 16)],
                         ids=PATH_IDS + ["q8-moe-separate-norm", "q8-qwen3", "q8-dim1536-graph", "q8-dim1536-persistent", "q8-dim1024-persistent"])
def test_outlier_rows_through_every_norm(pkg, orc, shape, quant, mode, lanes):
    """One step per hostile embedding row (Wo = W2 = 0: the attention, FFN and final norm of both layers all read that row)."""
    _decode(pkg, orc, H.outlier_embeddings(shape, quant), ALL_KINDS, mode, lanes)


WIDE = {  # widths where the accumulator's chunk layouts differ; hidden and vocabulary cut down, 2 layers
    2848: S("qwen3", 2848, 1024, 2, 4, 2, 128, 640, True, 1000000.0, 1e-6),
    4096: S("llama", 4096, 1024, 2, 32, 8, 128, 512, False, 500000.0, 1e-5),
    5120: S("devstral", 5120, 1024, 2, 32, 8, 128, 512, False, 1000000.0, 1e-5, 4096, yarn=(16.0, 32.0, 1.0, 1.0, 2048)),
    12288: S("devstral", 12288, 1024, 2, 96, 8, 128, 512, False, 1000000.0, 1e-5, 4096, yarn=(16.0, 32.0, 1.0, 1.0, 2048)),
}


@pytest.mark.parametrize("dim,mode", [(2848, "graph"), (2848, "persistent"), (4096, "graph"), (4096, "persistent"), (5120, "graph"), (5120, "persistent"),
                                      (12288, "graph")])
def test_outlier_rows_at_wide_dims(pkg, orc, dim, mode):
    _decode(pkg, orc, H.outlier_embeddings(WIDE[dim], Q8, fast=True), ALL_KINDS, mode)


@pytest.mark.parametrize("n_rows", [1, 3, 8])
@pytest.mark.parametrize("shape", ["tiny-llama", "small-llama"])
def test_outlier_rows_do_not_leak_between_batch_rows(pkg, orc, shape, n_rows):
    """Every row of a batched step carries a different hostile token, and they rotate: the outlier row sits next to the all-zero row."""
    T = H.OUTLIER_TOKEN
    order = [T[k] for k in ("outlier_mid", "zero", "outlier_last", "benign", "many_binades", "pow2_at", "zero_head", "outlier_early", "pow2_below",
                            "pow2_above", "constant")]
    rows = [order[r:] + order[:r] for r in range(n_rows)]
    _batch(pkg, orc, H.outlier_embeddings(shape, Q8), rows, len(order), feedback=False)


@pytest.mark.parametrize("dim", [256, 4096])
def test_outlier_rows_multi_position_and_mixed_step(pkg, orc, dim):
    m = H.outlier_embeddings("tiny-llama", Q8) if dim == 256 else H.outlier_embeddings(WIDE[dim], Q8, fast=True)
    _multi_and_step(pkg, orc, m, ALL_KINDS)


@pytest.mark.parametrize("mode", ["graph", "persistent"])
def test_zero_qk_rows_through_the_head_norm(pkg, orc, mode):
    _decode(pkg, orc, H.zero_qk_rows("tiny-qwen3", Q8), [5, 6, 7, 8, 9, 10], mode)


@pytest.mark.parametrize("dim", [256, 4096])
def test_norm_kernel_walks_hostile_rows_without_misprediction(pkg, orc, dim):
    """plan.profile_norm() runs k_rmsnorm_quant over the plan's current x, which after a step of an outlier_embeddings model is still the
    hostile row, and reports {items walked, mispredicted runs} of its exact sum.  The predictor's 2^-9 margin exceeds what n <= 16384
    sequential roundings can drift (n 2^-24), so no run may be mispredicted on any row; what a hostile row costs is literal items: a
    zero prefix has no binade to predict, so the all-zero row is walked thread by thread and the zero-headed row half so."""
    m = H.outlier_embeddings("tiny-llama", Q8) if dim == 256 else H.outlier_embeddings(WIDE[dim], Q8, fast=True)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    items = {}
    try:
        for kind, tok in H.OUTLIER_TOKEN.items():
            plan.forward_decode(tok, 0, logits=False)
            prof = plan._native.profile_norm()
            items[kind] = int(prof[4])
            assert prof[5] == 0, f"{kind}: {prof[5]} mispredicted runs"
            assert prof[4] >= 1
    finally:
        plan.free()
    print(f"\n  dim {dim} items walked: {items}")
    assert items["zero"] > items["zero_head"] > items["benign"]


# ---- saturated softmax and SwiGLU ----------------------------------------------------------------------------------------------

EDGES = {0, 1, 2, 126, 127, 128, 129, 130}
HOSTILE_PREFILL_TOL = 0.15


@pytest.mark.parametrize("shape,quant,mode,lanes", PATHS + [("tiny-qwen3", Q8, "graph", 16), ("tiny-qwen3", Q8, "persistent", 16), ("tiny-phi3", Q8, "graph", 16),
                                                            ("tiny-granite", Q8, "graph", 16)],
                         ids=PATH_IDS + ["q8-qwen3-hs128-graph", "q8-qwen3-hs128-persistent", "q8-phi3-hs96", "q8-granite"])
@pytest.mark.parametrize("kind", ["peaked", "uniform"])
def test_saturated_attention_around_128_keys(pkg, orc, shape, quant, mode, lanes, kind):
    """Scores spread over hundreds of nats (subnormal and zero exponentials, one-hot rows) or all equal (the sum is exactly the number
    of keys), on both sides of the 128-key pass boundary; head sizes 64, 128 and 96."""
    m = H.saturated_attention(shape, quant, kind, ctx=136)
    toks = orc.bench_tokens(m.configuration.vocab_size, 131)
    _decode(pkg, orc, m, toks, mode, lanes, check=EDGES)


@pytest.mark.parametrize("mode,ctx", [("graph", 520), ("persistent", 520), ("graph", 20000)])
@pytest.mark.parametrize("kind", ["peaked", "uniform"])
def test_saturated_attention_around_512_keys(pkg, orc, mode, ctx, kind):
    """511 | 512 | 513 keys (the persistent kernel's softmax sum switches to the parallel accumulator at 512), and once with a
    20000-token context, where the score row lives in global memory."""
    m = H.saturated_attention("tiny-llama", Q8, kind, ctx=ctx)
    toks = orc.bench_tokens(m.configuration.vocab_size, 514)
    _decode(pkg, orc, m, toks, mode, check={0, 255, 256, 510, 511, 512, 513}, kv=ctx == 520)


@pytest.mark.parametrize("kind", ["peaked", "uniform"])
def test_saturated_attention_batched_slots(pkg, orc, kind):
    m = H.saturated_attention("tiny-llama", Q8, kind, ctx=136)
    V = m.configuration.vocab_size
    rows = [[int(t) for t in orc.bench_tokens(V, 131, seed=42 + r)] for r in range(3)]
    _batch(pkg, orc, m, rows, 131, feedback=False, check_from=126)


@pytest.mark.parametrize("shape,quant,mode,lanes", PATHS + [("tiny-phi3", Q8, "graph", 16)], ids=PATH_IDS + ["q8-phi3"])
def test_saturated_swiglu(pkg, orc, shape, quant, mode, lanes):
    """Gates of +-(100 ... 1000) and exact zeros: g / (float)(1 + exp(-g)) gives -0 and g itself, and the down projection quantises
    signed zeros next to values in the thousands."""
    _decode(pkg, orc, H.saturated_swiglu(shape, quant), [1, 2, 3, 4, 5, 6], mode, lanes)


def test_saturated_swiglu_batched_multi_and_mixed(pkg, orc):
    m = H.saturated_swiglu("tiny-llama", Q8)
    _batch(pkg, orc, m, [1, 2, 3], 5)
    _multi_and_step(pkg, orc, m, list(range(1, 12)))


# ---- extreme weight blocks -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("shape,mode", [("tiny-llama", "graph"), ("tiny-llama", "persistent"), ("tiny-llama-tied", "graph"), ("tiny-qwen3", "persistent"),
                                        ("tiny-phi3", "graph"), ("small-llama", "graph")])
def test_extreme_q8_blocks_decode(pkg, orc, shape, mode):
    """d = 0, a subnormal d, a negative d, q = -128 and q = +-127 under a large d in 8 % of the blocks of every matrix and of the embedding."""
    m = H.extreme_q8_blocks(shape)
    _decode(pkg, orc, m, orc.bench_tokens(m.configuration.vocab_size, 10), mode)


def test_extreme_q8_blocks_batched_multi_and_mixed(pkg, orc):
    m = H.extreme_q8_blocks("tiny-llama")
    _batch(pkg, orc, m, [1, 2, 3, 4, 5, 6, 7, 8], 5)
    _multi_and_step(pkg, orc, m, orc.bench_tokens(m.configuration.vocab_size, 11))


def test_extreme_q8_blocks_tensor_core_prefill(pkg, orc):
    """The W8A16 prefill reads the extreme blocks in place; it stays bit-identical to the f16-twin mode (no residual GEMM splits K at
    this shape).  Against the oracle both modes are held to HOSTILE_PREFILL_TOL, not to the Q8_0 prefill's 3e-2: the oracle rounds the
    activations to 8 bits per 32-block and the prefill keeps them in f16, and on this model (q = +-127 blocks under four times their d,
    activation outliers behind them) the two differ by 9.7e-2 of max |logit| (measured on an H100, the same in both modes)."""
    m = H.extreme_q8_blocks("tiny-llama", ctx=64)
    c = m.configuration
    a, b = _run_modes(pkg, m, 50, 16, ("tensor_core_w8a16", "tensor_core"))
    for name, ref in a.items():
        assert np.array_equal(b[name].view(np.uint16), ref.view(np.uint16)), f"{name} differs between the modes"
    toks = orc.bench_tokens(c.vocab_size, 51)
    om = H.oracle_for(orc, m)
    for pos in range(50):
        om.forward(int(toks[pos]), pos, want_logits=False)
    ref = om.forward(int(toks[50]), 50)
    om.close()
    for mode in ("tensor_core", "tensor_core_w8a16"):
        plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=16)
        try:
            plan.set_prefill_mode(mode)
            for off in range(0, 50, 16):
                plan.forward_batch_prefill(toks[off:min(off + 16, 50)], off)
            lg, _ = plan.forward_decode(int(toks[50]), 50)
        finally:
            plan.free()
        err = np.max(np.abs(lg - ref)) / np.max(np.abs(ref))
        print(f"{mode}: logits after prefill rel err {err:.2e}")
        assert err <= HOSTILE_PREFILL_TOL, f"{mode}: rel err {err:.2e}"


@pytest.mark.parametrize("shape,lanes", [("tiny-llama", 16), ("tiny-llama", 8), ("tiny-llama-tied", 16), ("tiny-llama-tied", 8), ("tiny-phi3", 16), ("tiny-llama", 0),
                                         ("tiny-qwen3", 16)])
def test_extreme_f16_weights_decode(pkg, orc, shape, lanes):
    """A quarter of every matrix subnormal (both signs), -0 and +-65504: the rings' flush, the round-1 kernels' bit trick, the IEEE
    embedding gather of the same tensor in the tied shapes, and the scalar species that does not flush."""
    m = H.extreme_f16_weights(shape)
    _decode(pkg, orc, m, orc.bench_tokens(m.configuration.vocab_size, 10), "graph", lanes)
