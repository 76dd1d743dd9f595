"""GPU tests of the bit-exact tensor-core prefill (B200_PREFILL_TENSOR_CORE_EXACT) on plans that keep K-quant weights resident: before
each resident matrix's int8 GEMM, k_kq_tiles_to_q8 (csrc/stream_matvec.cuh) expands it to the Q8_0 tiles a Q8_0-tile plan of the same
file holds, in one scratch the size of the largest.  Bar: the expansion byte for byte against b200_requant_kquant laid out as tiles,
and every prefill's KV cache, next logits and ids bit-equal (uint32 views) to the oracle on the re-quantised Q8_0 twin."""
import re

import numpy as np
import pytest

from test_gpu_kquant_resident import KB, _hostile, _model, _oracle, _resident_plan
from test_gpu_parity import assert_bit_equal

pytestmark = pytest.mark.gpu


# ---- the expansion -------------------------------------------------------------------------------------------------------------

def _q8_tiles(q8, rows, cols):
    """GGUF Q8_0 blocks [rows][cols / 32] in the tile-major layout of csrc/stream_matvec.cuh: units in (group, segment, slot) order,
    each a segment's quants, then its f16 scales, then zeros up to 16 bytes; a ragged last group is completed with zero rows."""
    nseg = next(n for n in range(1, cols // 32 + 1) if cols % n == 0 and (cols // n) % 32 == 0 and cols // n <= 2560)
    seg, groups = cols // nseg, (rows + 3) // 4
    unit = (seg + seg // 16 + 15) & ~15
    b = np.zeros((groups * 4, cols // 32, 34), np.uint8)
    b[:rows] = q8.reshape(rows, cols // 32, 34)
    b = b.reshape(groups, 4, nseg, seg // 32, 34).transpose(0, 2, 1, 3, 4)
    out = np.zeros((groups, nseg, 4, unit), np.uint8)
    out[..., :seg] = b[..., 2:].reshape(groups, nseg, 4, seg)
    out[..., seg:seg + seg // 16] = b[..., :2].reshape(groups, nseg, 4, seg // 16)
    return out.ravel()


def _expand_matches(pkg, tt, rows, cols, raw):
    got = pkg.native.test_kq_tiles_to_q8(tt, rows, cols, raw)
    want = _q8_tiles(pkg.native.requant_kquant(tt, raw, rows * cols), rows, cols)
    assert got.size == want.size == pkg.native.q8_tile_bytes(rows, cols)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"type {tt} {rows}x{cols}: {bad.size} bytes differ, first at {bad[0] if bad.size else None}"


@pytest.mark.parametrize("tt", [12, 13, 14])
@pytest.mark.parametrize("cols", [4096, 14336, 28672, 9728, 18944])
def test_expansion_is_the_requantiser_as_tiles(pkg, tt, cols):
    """Widths whose Q8_0 and resident segments agree (4096, 14336, 28672: 2048 / 2048 / 2048 columns) and differ (Qwen3-4B's 9728:
    2432 against 512; Qwen2.5-7B's 18944: 2368 against 512).  Six rows: the second 4-row group is completed with zero rows."""
    rng = np.random.default_rng(cols + tt)
    _expand_matches(pkg, tt, 6, cols, pkg.synth.random_kquant(tt, 6 * cols, rng, zero_blocks=1))


def test_expansion_of_hostile_blocks(pkg):
    """_hostile's super-blocks (d = 0, dmin = 0, negative and subnormal d, all-equal codes, an all-zero 32-block, Q6_K codes -32 / 31
    under the largest scales) at the start of a Q4_K, a Q5_K and a Q6_K matrix."""
    G = pkg.gguf.GGMLType
    rng = np.random.default_rng(21)
    rows, cols = 4, 2048
    tensors = {name: (tt, [cols, rows], pkg.synth.random_kquant(tt, rows * cols, rng))
               for name, tt in (("blk.0.ffn_gate.weight", G.Q4_K), ("blk.0.attn_output.weight", G.Q5_K), ("blk.0.ffn_down.weight", G.Q6_K))}
    for tt, _, raw in _hostile(pkg, tensors).values():
        _expand_matches(pkg, int(tt), rows, cols, raw)


def test_expansion_hook_rejections(pkg):
    n = pkg.native
    raw = np.zeros(4 * 2 * KB[12], np.uint8)
    out = np.zeros(n.q8_tile_bytes(4, 512), np.uint8)
    for tt, rows, cols, nbytes in ((12, 4, 500, out.size), (11, 4, 512, out.size), (12, 0, 512, out.size), (12, 4, 512, out.size - 16)):
        rc = n.lib().b200_test_kq_tiles_to_q8(tt, rows, cols, raw.ctypes.data, out.ctypes.data, nbytes)
        assert rc == -1, (tt, rows, cols, nbytes)


# ---- whole prefills ------------------------------------------------------------------------------------------------------------

def _kv_matches(plan, om, c, what):
    nkv = c.context_length * c.kv_dim
    for l in range(c.n_layers):
        assert_bit_equal(plan.read_buffer("key_cache", nkv, layer=l), om.key_cache(l), f"{what}: key cache layer {l}")
        assert_bit_equal(plan.read_buffer("value_cache", nkv, layer=l), om.value_cache(l), f"{what}: value cache layer {l}")


def _prefill_matches(pkg, orc, m, batch, chunks, plan=None, seed=5):
    """The chunks through mode 3 on a resident plan, the same tokens one by one through the oracle: every layer's K / V, then the next
    forward_decode's logits and id.  Returns prefill_info() after the last chunk."""
    c = m.configuration
    end = max(s + n for s, n in chunks)
    toks = np.random.default_rng(seed).integers(0, c.vocab_size, end + 1).astype(np.int32)
    own = plan is None
    plan = plan or _resident_plan(pkg, m, prefill_batch_size=batch)
    om = _oracle(pkg, orc, m)
    try:
        plan.set_prefill_mode("tensor_core_exact")
        for s, n in chunks:
            plan.forward_batch_prefill(toks[s:s + n], s)
        info = plan.prefill_info()
        for pos in range(end):
            om.forward(int(toks[pos]), pos, want_logits=False)
        _kv_matches(plan, om, c, "after the prefill")
        lg, am = plan.forward_decode(int(toks[end]), end)
        ref = om.forward(int(toks[end]), end)
        assert_bit_equal(lg, ref, "logits after the prefill")
        assert am == orc.argmax(ref)
        return info
    finally:
        if own:
            plan.free()
        om.close()


SHAPES = [("tiny-llama", "Q4_K_M"), ("tiny-llama-tied", "Q6_K"), ("tiny-qwen3", "Q5_K"), ("tiny-qwen3", "Q4_K_M"), ("tiny-qwen2-gqa6", "Q4_K_M"),
          ("tiny-phi3-gqa", "Q4_K_M"), ("mid-granite-3-2b", "Q4_K_M"), ("tiny-devstral", "Q4_K_M"), ("mid-llama", "Q4_K_M"), ("mid-llama-70b", "Q4_K_M")]


@pytest.mark.parametrize("shape,mix", SHAPES)
def test_resident_prefill_is_the_oracle(pkg, orc, shape, mix):
    """The shapes of test_resident_plan_decodes_like_its_q8_0_twin: a chunk from position 0, then one of 77 tokens (not a multiple of
    the 128-row tile) continuing it.  A shape whose Q8_0-tile plan refuses mode 3 must be refused with the same reason."""
    m = _model(pkg, shape, mix, ctx=160, seed=31)
    plan = _resident_plan(pkg, m, prefill_batch_size=128)
    try:
        try:
            plan.set_prefill_mode("tensor_core_exact")
        except pkg.native.UnsupportedOperation as e:
            q8 = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=128)
            try:
                with pytest.raises(pkg.native.UnsupportedOperation) as e8:
                    q8.set_prefill_mode("tensor_core_exact")
            finally:
                q8.free()
            assert str(e8.value) == str(e), (str(e8.value), str(e))
            return
        info = _prefill_matches(pkg, orc, m, 128, [(0, 64), (64, 77)], plan=plan)
        assert info[0] == 3 and info[2] > 0
    finally:
        plan.free()


def test_resident_prefill_700_positions(pkg, orc):
    """ctx 720 in chunks of 256, 256 and 188: the attention's score rows leave shared memory for the global scratch."""
    m = _model(pkg, "tiny-llama", ctx=720, seed=12)
    _prefill_matches(pkg, orc, m, 256, [(0, 256), (256, 256), (512, 188)])


def test_engine_batch_prefill_on_a_resident_plan(pkg, orc):
    """generate_tokens_llama_batch_prefill in mode 3 returns generate_tokens_llama's ids on the oracle."""
    m = _model(pkg, "tiny-llama", ctx=96, seed=33)
    c = m.configuration
    E = pkg.engine
    prompt = [int(t) for t in orc.bench_tokens(c.vocab_size, 45, seed=7)]
    plan = _resident_plan(pkg, m, prefill_batch_size=16)
    om = _oracle(pkg, orc, m)
    try:
        plan.set_prefill_mode("tensor_core_exact")
        got = E.generate_tokens_llama_batch_prefill(plan, prompt[0], 0, prompt, [], 80, c.context_length, 16)
        want = E.generate_tokens_llama(lambda t, p: orc.argmax(om.forward(t, p)), prompt[0], 0, prompt, [], 80, c.context_length)
        assert got == want
        assert plan.prefill_info()[0] == 3
    finally:
        plan.free()
        om.close()


# ---- plan behaviour ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mix,resident_per_layer", [("Q4_K_M", 3), ("Q6_K", 4)])
def test_launch_count(pkg, orc, mix, resident_per_layer):
    """One expansion per resident matrix on top of the Q8_0-tile plan's 8 launches per layer (two norms, four GEMMs, RoPE / KV and one
    attention wave): in the Q4_K_M mix Wo, gate/up and W2 are resident (QKV mixes Q4_K and Q6_K sources and stays Q8_0 tiles); in a
    single-format file all four are."""
    m = _model(pkg, "tiny-llama", mix, ctx=64, seed=34)
    info = _prefill_matches(pkg, orc, m, 32, [(0, 32), (32, 9)])
    assert info[0] == 3
    assert info[1] == m.configuration.n_layers * (8 + resident_per_layer), info


def test_switching_exact_and_tensor_core_exact(pkg, orc):
    """exact -> tensor_core_exact -> exact -> tensor_core_exact on one resident plan: the same chunk gives identical K / V each time."""
    m = _model(pkg, "tiny-qwen3", ctx=64, seed=35)
    c = m.configuration
    toks = orc.bench_tokens(c.vocab_size, 40, seed=3)
    plan = _resident_plan(pkg, m, prefill_batch_size=64)
    nkv = c.context_length * c.kv_dim
    try:
        kvs = []
        for mode in ("exact", "tensor_core_exact", "exact", "tensor_core_exact"):
            plan.set_prefill_mode(mode)
            assert plan.prefill_info()[0] == {"exact": 0, "tensor_core_exact": 3}[mode]
            plan.kv_reset()
            plan.forward_batch_prefill(toks, 0)
            kvs.append([plan.read_buffer(n, nkv, layer=l).copy() for n in ("key_cache", "value_cache") for l in range(c.n_layers)])
        for k in range(1, 4):
            for i, (a, b) in enumerate(zip(kvs[k], kvs[0])):
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), f"switch {k}: buffer {i} differs"
    finally:
        plan.free()


def test_scratch_must_fit(pkg, orc):
    """Under a 1-byte memory budget set_prefill_mode("tensor_core_exact") fails with B200_ERR_OOM naming the scratch (the Q8_0 tiles of
    the largest resident matrix: gate/up here) and the chunk buffers; the exact mode stays, and the plan still prefills and decodes
    bit-exactly.  With the real figure the mode is then accepted."""
    m = _model(pkg, "tiny-llama", ctx=64, seed=36)
    c = m.configuration
    plan = _resident_plan(pkg, m, prefill_batch_size=32)
    try:
        pkg.native.test_set_memory_budget(1)
        try:
            with pytest.raises(pkg.native.B200Error) as e:
                plan.set_prefill_mode("tensor_core_exact")
        finally:
            pkg.native.test_set_memory_budget(0)
        assert e.value.code == -3, str(e.value)
        msg = str(e.value)
        scratch = pkg.native.q8_tile_bytes(2 * c.hidden_dim, c.dim)
        assert re.search(rf"\b{scratch} bytes of Q8_0 scratch", msg) and re.search(r"\b[1-9]\d* bytes of chunk buffers", msg), msg
        assert plan.prefill_info()[0] == 0
        om = _oracle(pkg, orc, m)
        try:
            toks = orc.bench_tokens(c.vocab_size, 21, seed=4)
            plan.forward_batch_prefill(toks[:20], 0)
            for pos in range(20):
                om.forward(int(toks[pos]), pos, want_logits=False)
            _kv_matches(plan, om, c, "exact prefill after the refusal")
            lg, am = plan.forward_decode(int(toks[20]), 20)
            ref = om.forward(int(toks[20]), 20)
            assert_bit_equal(lg, ref, "logits after the refusal")
            assert am == orc.argmax(ref)
        finally:
            om.close()
        plan.set_prefill_mode("tensor_core_exact")
        assert plan.prefill_info()[0] == 3
    finally:
        plan.free()


def test_f16_and_w8a16_modes_stay_refused(pkg):
    m = _model(pkg, "tiny-llama", ctx=64, seed=37)
    plan = _resident_plan(pkg, m, prefill_batch_size=16)
    try:
        plan.set_prefill_mode("tensor_core_exact")
        for mode in ("tensor_core", "tensor_core_w8a16"):
            with pytest.raises(pkg.native.UnsupportedOperation) as e:
                plan.set_prefill_mode(mode)
            assert e.value.code == -2 and "resident" in str(e.value) and "tensor_core_exact" in str(e.value), str(e.value)
            assert plan.prefill_info()[0] == 3
    finally:
        plan.free()
