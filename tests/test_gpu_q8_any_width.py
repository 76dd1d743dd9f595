"""GPU tests of Q8_0 plans whose widths have no segment count up to 64 (csrc/stream_matvec.cuh, smv_pick_nseg): 2656 = 32 * 83 and
2848 = 32 * 89 are cut into 83 and 89 segments of 32 columns.  Decode is bit-exact against the oracle (logits as uint32, ids, both
KV caches) in both decode modes, through the weight streams and the fused norm; batched and multi-position steps match
single-sequence decode."""
import numpy as np
import pytest

from test_gpu_parity import assert_bit_equal

pytestmark = pytest.mark.gpu


def _model(pkg, name, ctx=32):
    S = pkg.synth.Shape
    sh = {
        # only ffn_down (2656 columns) gets 32-column segments
        "hidden-2656": S("llama", 256, 2656, 2, 4, 2, 64, 512, False, 500000.0, 1e-5),
        # QKV, gate/up and the tied lm_head (2848 columns) get 32-column segments, each behind the fused norm
        "dim-2848": S("qwen3", 2848, 1024, 2, 4, 2, 128, 640, True, 1000000.0, 1e-6),
    }[name]
    Q8 = pkg.gguf.GGMLType.Q8_0
    return pkg.loader.model_from_tensors(sh, Q8, pkg.synth.build_tensors_fast(sh, Q8, seed=17), ctx)


@pytest.mark.parametrize("mode", ["graph", "persistent"])
@pytest.mark.parametrize("name", ["hidden-2656", "dim-2848"])
def test_q8_32_column_segments_decode_bit_exact(pkg, orc, name, mode):
    m = _model(pkg, name)
    c = m.configuration
    plan = pkg.B200MasterPlan.initialize_plan(m)
    om = orc.OracleModel(m)
    try:
        plan.set_decode_mode(mode)
        assert plan.decode_info()[0] == {"graph": 0, "persistent": 1}[mode]
        if mode == "graph":
            assert plan.launches_per_decode == 5 * c.n_layers + 2  # the weight streams with the fused norm
        tok = 1
        for pos in range(12):
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


def test_q8_32_column_segments_batch_and_multi(pkg, orc):
    """A 2-slot forward_decode_batch gives each row the logits and id of single-sequence decode; one forward_decode_multi step
    gives the token-by-token ids."""
    m = _model(pkg, "hidden-2656")
    c = m.configuration
    n = 8
    streams = [orc.bench_tokens(c.vocab_size, n, seed=40 + s) for s in range(2)]
    plan = pkg.B200MasterPlan.initialize_plan(m)
    try:
        single = []
        for s in range(2):
            plan.kv_reset()
            single.append([plan.forward_decode(int(t), pos) for pos, t in enumerate(streams[s])])
        plan.set_decode_slots(2)
        for pos in range(n):
            ids, lg = plan.forward_decode_batch([0, 1], [int(streams[0][pos]), int(streams[1][pos])], [pos, pos], logits=True)
            for s in range(2):
                assert_bit_equal(lg[s], single[s][pos][0], f"slot {s} logits pos {pos}")
                assert int(ids[s]) == single[s][pos][1], f"slot {s} id pos {pos}"
        rows = plan.decode_multi_rows()
        assert rows >= 2
        plan.kv_reset()
        ids, lg = plan.forward_decode_multi(-1, [int(t) for t in streams[0][:rows]], 0, logits=True)
        assert [int(i) for i in ids] == [single[0][p][1] for p in range(rows)]
        assert_bit_equal(lg, np.stack([single[0][p][0] for p in range(rows)]), "multi-position logits")
    finally:
        plan.free()
