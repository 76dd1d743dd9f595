"""CPU checks of the exact-attention tests: the float32 restatement (tests/attention_oracle.py) agrees bit for bit with the oracle's own
forwards, b200_test_attention refuses what the plan would never launch before it touches the device, every GPU case reaches the
edge its name claims (a Python mirror of the plan's score-row rule, grid and chunk launches, checked against the hook's dry run),
and the exp sweep's checker reports what it should."""
import numpy as np
import pytest

import attention_oracle as ao
import test_gpu_attention as ga
from granite_oracle import GraniteOracle
from qwen2_oracle import Qwen2Oracle

f32 = np.float32
CHECK = (0, 1, 31, 32, 127, 128, 129, 255, 256, 257, 511, 512, 513, 599, 639)


def _bits(a):
    return np.ascontiguousarray(a, dtype=f32).view(np.uint32)


def _layer0_qkv(helper, token, cfg):
    """The layer-0 q | k | v of `token` before bias, norm and rotation, through the oracle's own embedding, RMSNorm and matmul."""
    m = helper.om.m
    dim, qd, kvd = cfg.dim, cfg.n_heads * cfg.head_size, cfg.n_kv_heads * cfg.head_size
    xb = helper._rmsnorm(helper._embedding(token), m.attn_norm[0])
    return np.concatenate([helper._matmul(m.wq[0], xb, qd, dim), helper._matmul(m.wk[0], xb, kvd, dim), helper._matmul(m.wv[0], xb, kvd, dim)])


ARCH = {"tiny-llama": 0, "tiny-qwen3": ao.KF_NEOX | ao.KF_QKNORM, "tiny-phi3": ao.KF_NEOX}


@pytest.mark.parametrize("shape", list(ARCH))
def test_restatement_matches_oracle_forwards(pkg, orc, make_model, shape):
    """640 positions of a tiny model through the C oracle: at every checked position the last layer's softmax rows and head outputs
    (from the oracle's rotated q and K / V cache) and the layer-0 K / V rows (from the oracle's unrotated projections) are the oracle's,
    bit for bit, and so are the Q8_0 activations the restatement quantises."""
    m = make_model(shape, pkg.gguf.GGMLType.Q8_0, 640)
    c = m.configuration
    om = orc.OracleModel(m)
    helper = GraniteOracle(orc, m, scales=dict(embedding_scale=1.0, residual_scale=1.0, attention_scale=1.0, logit_scale=1.0))
    hs, nh, nkv, ctx, L = c.head_size, c.n_heads, c.n_kv_heads, c.context_length, c.n_layers - 1
    cr, ci = orc.rope_table(ctx, hs, c.rope_theta)
    T = m.tensors
    qn = kn = None
    if ARCH[shape] & ao.KF_QKNORM:
        qn, kn = (np.asarray(T[f"blk.0.attn_{w}_norm.weight"][2]).view(f32) for w in "qk")
    toks = np.random.default_rng(3).integers(0, c.vocab_size, size=ctx)
    for pos in range(ctx):
        om.forward(int(toks[pos]), pos, want_logits=False)
        if pos not in CHECK:
            continue
        a, out = ao.attend(om.q().reshape(nh, hs), om.key_cache(L).reshape(ctx, nkv, hs), om.value_cache(L).reshape(ctx, nkv, hs), pos,
                           float(np.sqrt(np.float64(hs))))
        assert np.array_equal(_bits(a), _bits(om.att(pos + 1))), f"softmax rows differ at {pos}"
        assert np.array_equal(_bits(out.reshape(-1)), _bits(om.att_out())), f"head outputs differ at {pos}"
        _, k, v = ao.prologue(_layer0_qkv(helper, int(toks[pos]), c), pos, nh, nkv, hs, ARCH[shape], cr, ci, qn, kn, eps=c.rms_norm_eps)
        kvd = nkv * hs
        assert np.array_equal(_bits(k.reshape(-1)), _bits(om.key_cache(0)[pos * kvd:(pos + 1) * kvd])), f"K row differs at {pos}"
        assert np.array_equal(_bits(v.reshape(-1)), _bits(om.value_cache(0)[pos * kvd:(pos + 1) * kvd])), f"V row differs at {pos}"
    om.close()


def test_restatement_matches_qwen2_bias(pkg, orc, make_model):
    """The q | k | v bias before the NeoX rotation: layer-0 K / V rows equal the Qwen2 oracle's over 300 positions."""
    m = make_model("tiny-qwen2", pkg.gguf.GGMLType.Q8_0, 300)
    c = m.configuration
    q2 = Qwen2Oracle(orc, m)
    hs, nh, nkv, kvd = c.head_size, c.n_heads, c.n_kv_heads, c.n_kv_heads * c.head_size
    cr, ci = orc.rope_table(c.context_length, hs, c.rope_theta)
    bias = np.concatenate(q2._b[0])
    toks = np.random.default_rng(4).integers(0, c.vocab_size, size=300)
    for pos in (0, 1, 127, 128, 129, 299):
        q2.forward(int(toks[pos]), pos, want_logits=False)
        _, k, v = ao.prologue(_layer0_qkv(q2, int(toks[pos]), c), pos, nh, nkv, hs, ao.KF_NEOX | ao.KF_QKVBIAS, cr, ci, qkv_bias=bias)
        assert np.array_equal(_bits(k.reshape(-1)), _bits(np.asarray(q2.key_cache(0)).reshape(-1)[pos * kvd:(pos + 1) * kvd]))
        assert np.array_equal(_bits(v.reshape(-1)), _bits(np.asarray(q2.value_cache(0)).reshape(-1)[pos * kvd:(pos + 1) * kvd]))


def test_restatement_quantises_as_the_oracle():
    orc = ao._orc()
    x = np.random.default_rng(6).standard_normal(4096).astype(f32)
    x[::97] = -0.0
    aq, sc = orc.q8_quantize(x)
    for b in range(0, 128, 17):
        q, s = orc.np_q8_quantize_block(x[b * 32:(b + 1) * 32])
        assert np.array_equal(q.astype(np.int8), aq[b * 32:(b + 1) * 32]) and _bits(s) == _bits(sc[b])


def test_head_norm_matches_oracle_rmsnorm():
    orc = ao._orc()
    rng = np.random.default_rng(7)
    x = rng.standard_normal((6, 128)).astype(f32)
    x[1] = 0.0
    x[2] *= f32(1e-20)
    w = rng.standard_normal(128).astype(f32)
    got = ao.head_norm(x, w, 1e-6)
    for r in range(6):
        assert np.array_equal(_bits(got[r]), _bits(orc.np_rmsnorm(x[r], w, 1e-6)))


# ---- the hook's refusals and the cases' edges -----------------------------------------------------------------------------------
def _dry(pkg, form="single", hs=64, nh=4, nkv=2, ctx=64, slots=(0,), pos=(5,), n_slots=2, **kw):
    return pkg.native.test_attention(form, hs, nh, nkv, ctx, slots, pos, None, None, None, None, None, n_slots=n_slots, dry=True, **kw)


@pytest.mark.parametrize("bad", [
    dict(form="single", hs=48), dict(form="persistent", hs=32), dict(form="persistent", hs=96), dict(form="persistent", hs=256),
    dict(nh=6, nkv=4), dict(pos=(64,)), dict(pos=(-1,)), dict(slots=(2,)), dict(slots=(-1,)),
    dict(form="batch", slots=tuple(range(9)), pos=(1,) * 9, n_slots=9), dict(form="cached_rows", slots=tuple(range(9)), pos=(1,) * 9, n_slots=9),
    dict(form="single", slots=(0, 1), pos=(1, 1)), dict(form="persistent", slots=(0, 1), pos=(1, 1)),
    dict(form="chunk", slots=(0, 0), pos=(1, 2), att_tokens=0), dict(form="chunk", slots=(0, 0), pos=(1, 2), att_tokens=3),
    dict(form="batch", slots=(0, 1), pos=(1, 2), att_tokens=1),
    dict(form="batch", slots=(1, 1), pos=(1, 2)), dict(form="cached_rows", slots=(1, 1), pos=(2, 2)), dict(form="chunk", slots=(0, 0), pos=(3, 3), att_tokens=1),
    dict(arch=16), dict(ctx=0), dict(n_slots=0),
], ids=lambda d: "-".join(f"{k}{v}" for k, v in d.items()))
def test_refusals_need_no_device(pkg, bad):
    with pytest.raises(pkg.native.B200Error) as e:
        _dry(pkg, **bad)
    assert e.value.code == -1


def mirror(c):
    """The plan's launch of case c: score rows global (3 * head size + context > ATT_SMEM_FLOATS_MAX), grid, launches, shared memory."""
    glob = 3 * c["hs"] + c["ctx"] > ga.ATT_SMEM_FLOATS_MAX
    rows = len(c["rows"])
    gy = c["att_tokens"] if c["form"] == "chunk" else rows if c["form"] in ("batch", "cached_rows") else 1
    launches = -(-rows // c["att_tokens"]) if c["form"] == "chunk" else 1
    return {"grid_x": c["nh"], "grid_y": gy, "global_scores": int(glob), "launches": launches,
            "smem": None if c["form"] == "persistent" else (3 * c["hs"] + (0 if glob else c["ctx"])) * 4}


def edges(c):
    m = mirror(c)
    out = {"global" if m["global_scores"] else "shared"}
    if any(p > 128 for _, p in c["rows"]):
        out.add("v_rounds")
    if m["launches"] > 1:
        out.add("split")
    if c["form"] == "persistent" and c["ctx"] % 512 and (c["rows"][0][1] + 1) >= 512 and (c["rows"][0][1] + 1) % 512:
        out.add("pad")
    if any(s2 == s and p2 < p for i, (s, p) in enumerate(c["rows"]) for s2, p2 in c["rows"][:i]):
        out.add("reads_same_call")
    return out


@pytest.mark.parametrize("c", ga.CASES)
def test_case_reaches_its_edge(pkg, c):
    slots = [s for s, _ in c["rows"]]
    info = _dry(pkg, c["form"], c["hs"], c["nh"], c["nkv"], c["ctx"], slots, [p for _, p in c["rows"]], n_slots=max(slots) + 2, arch=c["arch"],
                att_tokens=c["att_tokens"])["info"]
    want = mirror(c)
    for k, v in want.items():
        if v is not None:
            assert info[k] == v, (k, info[k], v)
    assert set(c["edges"]) <= edges(c), (c["edges"], edges(c))
    if c["id"].endswith(("-ctx3328", "-ctx3712", "-ctx3808", "-ctx3904", "-ctx4000")):
        assert not info["global_scores"] and 3 * c["hs"] + c["ctx"] == ga.ATT_SMEM_FLOATS_MAX


def test_exp_sweep_reports_mismatches():
    orc = ao._orc()
    first = 0xC2AF0000  # around -87.5: the exps there are float subnormals
    x = (np.arange(1 << 16, dtype=np.uint32) + np.uint32(first)).view(f32)
    e = orc.exp_narrow(x)
    e1 = (1.0 + np.exp(x.astype(np.float64))).astype(f32)
    n, lows = orc.exp_sweep(first, e, e1)
    if n:  # numpy's exp may round differently from libm: mismatches can only be in e1 then; take the oracle's values
        e1 = (1.0 + e.astype(np.float64)).astype(f32)  # exp there is below 2^-24: 1 + exp rounds to 1 either way
        n, lows = orc.exp_sweep(first, e, e1)
    assert n == 0 and lows == []
    e2 = e.copy()
    e2[[5, 9, 60000]] = np.nextafter(e2[[5, 9, 60000]], f32(1))
    assert orc.exp_sweep(first, e2, e1, max_report=2) == (3, [first + 5, first + 9])
