"""The exact attention one launch at a time (b200_test_attention): every form -- the decode graph's k_attention, the batched step's
k_attention_batch, the multi-position step's k_rope_kv_batch + k_attention_cached_rows, the chunk's k_i8_rope_kv + k_i8_attention and
the persistent kernel's pd_attention_head -- held bit for bit to the float32 restatement of tests/attention_oracle.py, at head sizes,
positions, contexts, GQA ratios and values no model reaches.  Every cache row a launch must not read holds NaN (a read of one poisons
the output) and every cache float it must not write has to come back unchanged.  Each case names the edge it exists for;
tests/test_attention_host.py checks on the CPU that the launch configuration reaches it.

The exp sweep at the end holds the device's (float)exp((double)x) and (float)(1.0 + exp((double)x)) -- the softmaxes, the MoE routers,
the shared-expert gate and the SwiGLU denominator -- to the oracle's libm on every non-NaN float."""
import numpy as np
import pytest

import attention_oracle as ao

pytestmark = pytest.mark.gpu

f32 = np.float32
NEOX, QKNORM, QKVBIAS, ATTSCALE = ao.KF_NEOX, ao.KF_QKNORM, ao.KF_QKVBIAS, ao.KF_ATTSCALE
ATT_SMEM_FLOATS_MAX = 4096  # plan.cu: q | k | out | score row beyond this many floats -> the score row goes to a global scratch
GRANITE_SCALE = 0.015625


def C(id, form, hs, nh, nkv, ctx, rows, arch=0, values="gauss", att_tokens=0, edges=()):
    """One case: rows = [(slot, position)], values = the kind of data (make_inputs), edges = what test_attention_host.edges must find."""
    return pytest.param(dict(id=id, form=form, hs=hs, nh=nh, nkv=nkv, ctx=ctx, rows=list(rows), arch=arch, values=values, att_tokens=att_tokens,
                             edges=tuple(edges)), id=id)


GRAPH_FORMS = ("single", "batch", "cached_rows", "chunk")
HEAD_SIZES = (32, 64, 96, 128, 256)
POSITIONS = (0, 1, 31, 32, 127, 128, 129, 255, 256, 257, 511, 512, 513)


def _one(form, hs, nh, nkv, ctx, pos, **kw):
    return C(f"{form}-hs{hs}-pos{pos}", form, hs, nh, nkv, ctx, [(0, pos)], att_tokens=1 if form == "chunk" else 0, **kw)


CASES = (
    # every graph form at every compiled head size over the score passes and V rounds (128 keys per pass, 4 x 32 rows per round)
    [_one(f, hs, 4, 2, 600, p, edges=("v_rounds",) if p > 128 else ()) for f in GRAPH_FORMS for hs in HEAD_SIZES for p in (0, 1, 129, 257, 513)]
    + [_one(f, hs, 4, 2, 600, p) for f in ("single", "cached_rows") for hs in (64, 256) for p in (31, 32, 127, 128, 255, 256, 511, 512)]
    # the persistent form: every position, the switch to the parallel sum at 512 keys, and ctx - 1 with ctx not a multiple of 512
    + [_one("persistent", hs, 4, 2, 600, p) for hs in (64, 128) for p in POSITIONS]
    + [C(f"persistent-hs{hs}-pad-ctx1000", "persistent", hs, 4, 2, 1000, [(0, 999)], edges=("pad",)) for hs in (64, 128)]
    # the score row: the last context that fits shared memory and the first that does not, per head size, the row at its end
    + [C(f"{f}-hs{hs}-ctx{ATT_SMEM_FLOATS_MAX - 3 * hs + d}", f, hs, 2, 1, ATT_SMEM_FLOATS_MAX - 3 * hs + d, [(0, ATT_SMEM_FLOATS_MAX - 3 * hs + d - 1)],
         att_tokens=1 if f == "chunk" else 0, edges=("global",) if d else ("shared",))
       for f in GRAPH_FORMS for hs in HEAD_SIZES for d in (0, 1)]
    + [C(f"persistent-hs{hs}-ctx{ATT_SMEM_FLOATS_MAX - 3 * hs + d}", "persistent", hs, 2, 1, ATT_SMEM_FLOATS_MAX - 3 * hs + d,
         [(0, ATT_SMEM_FLOATS_MAX - 3 * hs + d - 1)], edges=("global",) if d else ("shared",)) for hs in (64, 128) for d in (0, 1)]
    + [C(f"{f}-ctx20011-long", f, 64, 4, 2, 20011, [(0, 20003)], att_tokens=1 if f == "chunk" else 0, edges=("global",))
       for f in GRAPH_FORMS + ("persistent",)]
    # GQA ratios, one KV head under 64 query heads, Devstral 2's 96 on 8
    + [C(f"{f}-gqa{r}", f, 64, 2 * r, 2, 300, [(0, 290)], att_tokens=1 if f == "chunk" else 0) for f in ("single", "batch", "chunk")
       for r in (1, 2, 4, 7, 8, 12, 16)]
    + [C(f"{f}-gqa64-one-kv-head", f, 128, 64, 1, 300, [(0, 200)], att_tokens=1 if f == "chunk" else 0) for f in GRAPH_FORMS + ("persistent",)]
    + [C(f"{f}-heads96-kv8", f, 128, 96, 8, 300, [(0, 150)], att_tokens=1 if f == "chunk" else 0) for f in GRAPH_FORMS + ("persistent",)]
    # the architecture flags
    + [C(f"{f}-hs{hs}-{name}", f, hs, 8, 2, 400, [(0, 300)], arch=a, att_tokens=1 if f == "chunk" else 0)
       for f in GRAPH_FORMS + ("persistent",) for hs in ((64, 128) if f == "persistent" else (32, 128, 256))
       for name, a in (("neox", NEOX), ("qknorm", NEOX | QKNORM), ("bias", NEOX | QKVBIAS), ("attscale", ATTSCALE))]
    # eight rows on distinct slots at unequal positions; one sequence's consecutive positions beside other slots
    + [C(f"batch-8-slots-hs{hs}", "batch", hs, 4, 2, 700, [(s, p) for s, p in enumerate((0, 700 - 1, 129, 1, 512, 257, 31, 640))],
         arch=NEOX | QKVBIAS) for hs in (32, 128, 256)]
    + [C(f"cached-rows-consecutive-hs{hs}", "cached_rows", hs, 4, 2, 700, [(1, 126 + i) for i in range(6)] + [(0, 3), (2, 511)], arch=NEOX | QKNORM,
         edges=("reads_same_call",)) for hs in (32, 128, 256)]
    # the chunk over several attention launches (v0 > 0), rows of two prompts
    + [C(f"chunk-att-tokens{k}", "chunk", 128, 8, 2, 300, [(0, 100 + i) for i in range(11)] + [(3, i) for i in range(9)], arch=NEOX | QKNORM,
         att_tokens=k, edges=("split", "reads_same_call")) for k in (1, 3, 19)]
    + [C("chunk-att-tokens3-global", "chunk", 64, 4, 2, 4300, [(1, 4000 + i) for i in range(7)], att_tokens=3, edges=("split", "global"))]
    # hostile values
    + [C(f"{f}-{v}", f, 64, 8, 2, 4100 if v == "equal" else 600, [(0, 4000 if v == "equal" else 530)], arch=NEOX | QKNORM if v == "zero_qk" else 0,
         values=v, att_tokens=1 if f == "chunk" else 0)
       for f in GRAPH_FORMS + ("persistent",) for v in ("dominant", "subnormal_exp", "equal", "ties", "huge", "zero_qk", "v_special")]
)


def make_inputs(c, seed=0):
    """(qkv rows, K cache, V cache, rope cr, ci, q_norm, k_norm, bias) for case c: every slot's rows below its first row's position hold
    data; every other cache float -- positions from there on, slots no row uses -- is NaN."""
    rng = np.random.default_rng(seed)
    hs, nh, nkv, ctx = c["hs"], c["nh"], c["nkv"], c["ctx"]
    qd, kvd = nh * hs, nkv * hs
    slots = max(s for s, _ in c["rows"]) + 2
    orc = ao._orc()
    cr, ci = orc.rope_table(ctx, hs, 10000.0)
    qn, kn = (1.0 + 0.25 * rng.standard_normal(hs)).astype(f32), (1.0 + 0.25 * rng.standard_normal(hs)).astype(f32)
    bias = (0.5 * rng.standard_normal(qd + 2 * kvd)).astype(f32)
    qkv = rng.standard_normal((len(c["rows"]), qd + 2 * kvd)).astype(f32)
    K = np.full((slots, ctx, kvd), np.nan, dtype=f32)
    V = np.full((slots, ctx, kvd), np.nan, dtype=f32)
    first = {}
    for s, p in c["rows"]:
        first[s] = min(p, first.get(s, p))
    for s, p0 in first.items():
        K[s, :p0] = rng.standard_normal((p0, kvd))
        V[s, :p0] = rng.standard_normal((p0, kvd))
    v = c["values"]
    if v == "zero_qk":
        qkv[:, :qd + kvd] = 0.0
    elif v == "equal":  # q = 0: every score is exactly 0
        qkv[:, :qd] = 0.0
    elif v == "v_special":
        special = np.array([-0.0, 0.0, 1e-40, -1e-40, 1.4e-45, -3e-39, 1.0], dtype=f32)
        V[~np.isnan(V)] = rng.choice(special, size=int((~np.isnan(V)).sum()))
        qkv[:, qd + kvd:] = rng.choice(special, size=qkv[:, qd + kvd:].shape)
    elif v in ("dominant", "subnormal_exp", "ties", "huge"):  # cache keys along each group's first rotated q: chosen scores
        s, p = c["rows"][0]
        q, k, _ = ao.prologue(qkv[0], p, nh, nkv, hs, c["arch"], cr, ci, qn, kn, bias)
        qkv[0, qd:qd + kvd] *= f32(0.01)  # the current key scores about 0
        kv_mul = nh // nkv
        for g in range(nkv):
            u = q[g * kv_mul].astype(np.float64)
            unit = u * np.sqrt(hs) / (u @ u)  # key t = score_t * unit scores about score_t
            if v == "dominant":
                scores = np.zeros(p)
                scores[p // 3] = 600.0
                K[s, :p, g * hs:(g + 1) * hs] *= 0.01
            elif v == "subnormal_exp":
                scores = 10.0 - rng.uniform(87.4, 103.9, size=p)
                scores[p // 2] = 10.0
            elif v == "ties":
                scores = rng.uniform(-5.0, 5.0, size=p)
                scores[::7] = 30.0
            else:
                scores = rng.choice([-1e30, 1e30, 3.0], size=p)
            sel = scores != 0.0
            K[s, :p, g * hs:(g + 1) * hs][sel] = (scores[sel, None] * unit[None, :]).astype(f32)
            if v == "ties":  # exact ties: the same key row
                K[s, :p:7, g * hs:(g + 1) * hs] = K[s, 0, g * hs:(g + 1) * hs]
    return qkv, K, V, cr, ci, qn, kn, bias


def run_case(pkg, c):
    qkv, K, V, cr, ci, qn, kn, bias = make_inputs(c)
    slots, pos = [s for s, _ in c["rows"]], [p for _, p in c["rows"]]
    kw = dict(arch=c["arch"], eps=1e-6, score_arg=GRANITE_SCALE if c["arch"] & ATTSCALE else None, q_norm=qn, k_norm=kn, qkv_bias=bias)
    got = pkg.native.test_attention(c["form"], c["hs"], c["nh"], c["nkv"], c["ctx"], slots, pos, qkv, K, V, cr, ci, att_tokens=c["att_tokens"],
                                    want_xb=c["form"] == "single", **kw)
    want = ao.reference(c["form"], c["hs"], c["nh"], c["nkv"], slots, pos, qkv, K, V, cr, ci, **kw)
    return got, want


def _bits(a):
    return np.ascontiguousarray(a, dtype=f32).view(np.uint32)


@pytest.mark.parametrize("c", CASES)
def test_attention_form(pkg, c):
    got, want = run_case(pkg, c)
    for name in ("k_cache", "v_cache", "qkv"):  # NaN rows compare by bit pattern: the launch must not touch them
        bad = np.argwhere(_bits(got[name]) != _bits(want[name]))
        assert bad.size == 0, f"{name}: {len(bad)} floats differ, first at {bad[0].tolist()}"
    assert np.array_equal(_bits(got["xs"]), _bits(want["xs"])), "xs differs"
    assert np.array_equal(got["xq"], want["xq"]), "xq differs"
    if c["form"] == "single":
        assert np.array_equal(_bits(got["xb"]), _bits(want["xb"])), "xb differs"
    assert not np.isnan(got["xs"]).any()


def test_attention_reports_launch(pkg):
    """The configuration a real launch reports is the one the dry run reports (the host test checks the dry run against the plan's rules)."""
    c = next(p.values[0] for p in CASES if p.values[0]["id"] == "chunk-att-tokens3-global")
    got, _ = run_case(pkg, c)
    assert got["info"] == {"grid_x": 4, "grid_y": 3, "smem": 3 * 64 * 4, "global_scores": 1, "launches": 3}


EXP_CHUNK = 1 << 26


def test_exp_matches_oracle_on_every_float(pkg, orc):
    """(float)exp((double)x) and (float)(1.0 + exp((double)x)) on the device against the oracle's libm for every non-NaN float: both signs,
    0 .. +inf.  The bit-exact paths assume they agree everywhere; nothing else checks it beyond the values random models produce."""
    total, worst = 0, []
    for base in (0x00000000, 0x80000000):
        end = base + 0x7F800000  # +-inf included; NaNs above it are not inputs of any path
        for first in range(base, end + 1, EXP_CHUNK):
            n = min(EXP_CHUNK, end + 1 - first)
            e, e1 = pkg.native.test_exp(first, n)
            bad, lows = orc.exp_sweep(first, e, e1)
            total += bad
            worst += lows
    assert total == 0, f"{total} inputs differ; lowest bit patterns {[hex(b) for b in sorted(worst)[:16]]}"
