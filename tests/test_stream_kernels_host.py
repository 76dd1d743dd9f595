"""CPU side of the single-stream tests (tests/test_gpu_stream_kernels.py): the float32 restatements they hold the kernels to equal the
oracle's C functions, b200_test_stream refuses what the plan would never launch before it touches the device, and every GPU case's
launch configuration reaches the edge it is named for -- by a Python mirror of the kernels' slicing and of smv_layout, checked against
the hook's own dry run and against b200_stream_rings."""
import numpy as np
import pytest

import hostile
import test_gpu_stream_kernels as sk
from test_gpu_prefill_i8 import _dot_q8, _weights

SMS = sk.SMS
WARPS = 8  # SMV_CONSUMER_WARPS: the groups of one producer round


# ---- mirrors of the launch geometry ------------------------------------------------------------------------------------------

def pick_nseg(cols, quantum=32):
    return next((n for n in range(1, cols // quantum + 1) if cols % n == 0 and (cols // n) % quantum == 0 and cols // n <= 2560), 0)


def slices(groups, grid):
    """[g0, g1) of every CTA: g0 = b * G / grid."""
    return [(b * groups // grid, (b + 1) * groups // grid) for b in range(grid)]


def smv_stages(cols, seg, budget, fmt=0):
    """smv_layout's ring depth (stream_matvec.cuh) for a plain single-row stream."""
    unit = (seg // 256 * sk.KQ_BYTES[fmt] + 15) & ~15 if fmt else (seg + seg // 16 + 15) & ~15
    stage = (4 * unit + 127) & ~127
    nbs_pad = ((seg // 32 + 3) & ~3) + 4
    o = 2 * 16 * 8 + 16 * 4 + cols + cols // 32 * 4
    o = (o + 15) & ~15
    o += WARPS * 4 * nbs_pad * 4 + 512 * 4
    o = (o + 127) & ~127
    return max(0, min(16, (budget - o) // stage))


def edges(s, info):
    """The edges a case's launch reaches, from its configuration (Q8_0 / resident / batched streams; F16 has none of these)."""
    if s["form"] == sk.F16:
        return set()
    fmt = 0 if s["form"] == sk.Q8 else s["form"]
    nseg = pick_nseg(s["cols"], 256 if fmt else 32)
    rows = 2 * s["rows"] if s["mode"] == "gateup" else s["rows"]
    sl = slices((rows + 3) // 4, info["grid"])
    n = [g1 - g0 for g0, g1 in sl]
    out = set()
    if max(n) * nseg >= 3 * info["stages"]:
        out.add("laps")  # the largest slice laps its ring at least twice
    if min(n) == 0:
        out.add("empty_cta")
    if any(k % WARPS == 1 for k in n):
        out.add("nw1")
    if any(k % WARPS == 7 for k in n):
        out.add("nw7")
    if info["stages"] > max(n) * nseg:
        out.add("stages_gt_slice")
    if s["mode"] == "gateup":
        for blk in range(s["rows"] // 32):
            owners = sum(1 for g0, g1 in sl if 2 * g0 < 32 * blk + 32 and 2 * g1 > 32 * blk)
            out.add(f"blocks_{min(owners, 3)}")
    return out


def _dry(pkg, s, grid=None):
    """The hook's dry run of a case: its checks and the configuration it would launch, without inputs."""
    L, cols = s.get("launches", 1), s["cols"]
    kw = dict(nrow=s.get("nrow", 0), grid=grid or s.get("grid", 0) or SMS, stages=s.get("stages", 0), argmax=s.get("argmax", False), launches=L,
              lanes=s.get("lanes", 16), budget=s.get("budget", 0), dry=True)
    if s["form"] == sk.F16 or (s.get("norm") and not s.get("from_emb")):
        kw["x"] = np.zeros(cols, np.float32)
    elif not s.get("norm"):
        kw["xq"], kw["xs"] = np.zeros(cols, np.int8), np.zeros(cols // 32, np.float32)
    if s.get("norm"):
        kw["norm_w"] = np.ones(cols, np.float32)
    if s.get("from_emb"):
        kw.update(emb=np.zeros(34, np.uint8), emb_rows=8, tokens=np.zeros(L, np.int32))
    if s["mode"] == "gateup":
        kw["w_up"] = np.zeros(1, np.uint8)
    if s["mode"] == "resid" or s.get("pair"):
        kw["out_init"] = np.zeros(1, np.float32)
    if s.get("pair"):
        kw.update(pair=True, down_rows=s["pair"], w_down=np.zeros(1, np.uint8))
    return pkg.native.test_stream(s["form"], s["mode"], np.zeros(1, np.uint8), s["rows"], cols, **kw)["info"]


@pytest.mark.parametrize("s", sk.CASES)
def test_case_reaches_its_configuration(pkg, s):
    info = _dry(pkg, s)
    for k, v in s["expect"].items():
        assert info[k] == v, f"{k}: {info}"
    assert set(s["edges"]) <= edges(s, info), f"{s['edges']} not all reached: {edges(s, info)} ({info})"
    if s["form"] != sk.F16:  # the mirror of the slicing gives the hook's group counts
        rows = 2 * s["rows"] if s["mode"] == "gateup" else s["rows"]
        n = [g1 - g0 for g0, g1 in slices((rows + 3) // 4, info["grid"])]
        assert (info["max_groups"], info["min_groups"]) == (max(n), min(n))
    if s["form"] != sk.F16 and not s.get("nrow") and not s.get("norm") and not s.get("stages"):
        fmt = 0 if s["form"] == sk.Q8 else s["form"]
        nseg = pick_nseg(s["cols"], 256 if fmt else 32)
        assert info["stages"] == smv_stages(s["cols"], s["cols"] // nseg, 96 * 1024, fmt)


def test_stage_mirror_matches_stream_rings(pkg):
    """smv_stages is the depth b200_stream_rings reports for the Wo and W2 streams (plain, flat 96 KB budget) of every synth shape."""
    for name, sh in pkg.synth.SHAPES.items():
        qd = sh.n_heads * sh.head_size
        for fmt in (0, sk.Q4K, sk.Q6K):
            fm = tuple(fmt if c % 256 == 0 else 0 for c in (sh.dim, qd, sh.dim, sh.hidden))
            try:
                r = pkg.native.stream_rings(sh.dim, qd, sh.n_kv_heads * sh.head_size, sh.hidden, SMS, False, fm, att_bytes=0)
            except pkg.native.UnsupportedOperation:
                continue
            for key, cols, f in (("wo", qd, fm[1]), ("w2", sh.hidden, fm[3])):
                nseg = pick_nseg(cols, 256 if f else 32)
                assert r[key]["stages"] == smv_stages(cols, cols // nseg, 96 * 1024, f), (name, fmt, key, r[key])


def test_stages_turn_into_the_budget_that_yields_them(pkg):
    for cols in (32, 544, 2592, 4096, 14336):
        for st in range(3, 17):
            s = dict(form=sk.Q8, mode="store", rows=64, cols=cols, stages=st)
            if smv_stages(cols, cols // pick_nseg(cols), 232448) < st:
                continue
            assert _dry(pkg, s)["stages"] == st


# ---- refusals before any CUDA call -------------------------------------------------------------------------------------------

REFUSED = [
    ("q8 width not whole blocks", dict(form=sk.Q8, mode="store", rows=64, cols=100)),
    ("kquant width not whole super-blocks", dict(form=sk.Q4K, mode="store", rows=64, cols=2080)),
    ("f16 width not whole segments", dict(form=sk.F16, mode="store", rows=64, cols=288)),
    ("f16 gateup rows ragged", dict(form=sk.F16, mode="gateup", rows=133, cols=512, lanes=8)),
    ("f16 lanes", dict(form=sk.F16, mode="store", rows=64, cols=512, lanes=4)),
    ("two stages", dict(form=sk.Q8, mode="store", rows=64, cols=4096, stages=2)),
    ("seventeen stages", dict(form=sk.Q8, mode="store", rows=64, cols=4096, stages=17)),
    ("f16 nine stages", dict(form=sk.F16, mode="store", rows=64, cols=512, stages=9)),
    ("budget under three stages", dict(form=sk.Q8, mode="store", rows=64, cols=4096, budget=20000)),
    ("gateup slice over the epilogue buffer", dict(form=sk.Q8, mode="gateup", rows=1024, cols=512, grid=1)),
    ("gateup hidden not whole blocks", dict(form=sk.Q8, mode="gateup", rows=48, cols=512)),
    ("norm with resid", dict(form=sk.Q8, mode="resid", rows=64, cols=2048, norm=True)),
    ("norm over 5120", dict(form=sk.Q8, mode="store", rows=64, cols=5632, norm=True)),
    ("nine batch rows", dict(form=sk.Q8, mode="store", rows=64, cols=2048, nrow=9)),
    ("batch on a resident form", dict(form=sk.Q4K, mode="store", rows=64, cols=2048, nrow=2)),
    ("batch on f16", dict(form=sk.F16, mode="store", rows=64, cols=2048, nrow=2)),
    ("batch budget over 112 KB", dict(form=sk.Q8, mode="store", rows=64, cols=14336, nrow=8, stages=16)),
    ("argmax on resid", dict(form=sk.Q8, mode="resid", rows=64, cols=2048, argmax=True)),
    ("three launches", dict(form=sk.Q8, mode="store", rows=64, cols=2048, launches=3)),
    ("pair on store", dict(form=sk.Q8, mode="store", rows=64, cols=2048, pair=64)),
]


@pytest.mark.parametrize("why,s", REFUSED, ids=[r[0] for r in REFUSED])
def test_refused_without_the_device(pkg, why, s):
    """B200_ERR_BAD_ARG from the checks alone: these run on a machine without a GPU, so no CUDA call may come before them."""
    for dry in (True, False):
        with pytest.raises(pkg.native.B200Error) as e:
            _dry(pkg, s) if dry else _dry_launch(pkg, s)
        assert e.value.code == -1, why


def _dry_launch(pkg, s):
    """The same arguments as a real launch (dry = 0, grid given): the refusal must still come before any CUDA call."""
    real = pkg.native.test_stream
    pkg.native.test_stream = lambda *a, **kw: real(*a, **{**kw, "dry": False})
    try:
        return _dry(pkg, s)
    finally:
        pkg.native.test_stream = real


# ---- the restatements against the oracle's C functions -----------------------------------------------------------------------

def _extreme(rng, n, k):
    """Every block one of hostile.Q8_BLOCK_KINDS, in rotation: d = 0, the smallest subnormal d, negated d, q = -128, +-127 under 4 d."""
    d, q = hostile.q8_split(_weights(rng, n, k))
    kind = np.arange(len(d)) % 5
    d[kind == 0] = 0
    d[kind == 1] = 1
    d[kind == 2] ^= 0x8000
    q[kind == 3] = -128
    q[kind == 4] = rng.choice(np.array([-127, 127], dtype=np.int8), (int((kind == 4).sum()), 32))
    return hostile.q8_raw(d, q).reshape(n, -1)


def test_q8_dot_matches_the_oracle(orc):
    """_dot_q8 on quantised activations equals oracle_q8_dot_ref on the floats they quantise from, row for row: random rows and the
    hostile Q8_0 blocks (zero, subnormal and negative scales, -128 / +-127 quants)."""
    rng = np.random.default_rng(1)
    for k in (32, 544, 2592, 4096):
        x = (rng.standard_normal(k) * 3).astype(np.float32)
        x[:32] = 0  # an all-zero activation block
        aq, xs = orc.q8_quantize(x)
        for bq in (_weights(rng, 24, k), _extreme(rng, 24, k)):
            want = np.array([orc.q8_dot(np.ascontiguousarray(bq[r]), 0, x) for r in range(bq.shape[0])], np.float32)
            got = _dot_q8(aq[None, :], xs[None, :], bq)[0]
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), k


def test_norm_act_matches_the_oracle(orc):
    """RMSNorm and block quantisation of the fused norm's restatement equal the oracle's C quantiser, on the outlier rows."""
    rng = np.random.default_rng(2)
    for kind in hostile.OUTLIER_KINDS:
        d, q = hostile.outlier_row(kind, 1024, rng)
        x = (q.astype(np.float32) * d[:, None]).reshape(-1)
        w = (rng.standard_normal(1024) * 0.5 + 1).astype(np.float32)
        aq, xs = sk.norm_act(orc, x, w, 1e-5)
        wq, ws = orc.q8_quantize(orc.np_rmsnorm(x, w, 1e-5))
        assert np.array_equal(aq, wq) and np.array_equal(xs.view(np.uint32), ws.view(np.uint32)), kind


@pytest.mark.parametrize("fmt", [sk.Q4K, sk.Q5K, sk.Q6K])
def test_resident_restatement_matches_the_oracle(pkg, orc, fmt):
    """The resident stream's blocks (orc.kquant_to_q8_0 row by row) through _dot_q8 equal oracle_q8_dot_ref on the re-quantised rows,
    for random super-blocks and for arbitrary bytes."""
    rng = np.random.default_rng(fmt)
    k = 2048
    x = (rng.standard_normal(k) * 2).astype(np.float32)
    aq, xs = orc.q8_quantize(x)
    for kind in ("random", "bits"):
        raw = sk._kq_rows(rng, pkg, fmt, 16, k, kind)
        bq = sk.q8_of(orc, fmt, raw, k)
        assert np.isfinite(bq.reshape(-1, 34)[:, :2].copy().view(np.float16).astype(np.float32)).all(), kind
        want = np.array([orc.q8_dot(np.ascontiguousarray(orc.kquant_to_q8_0(fmt, raw[r], k)), 0, x) for r in range(16)], np.float32)
        got = _dot_q8(aq[None, :], xs[None, :], bq)[0]
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), kind


@pytest.mark.parametrize("lanes", [16, 8])
def test_f16_dots_match_the_oracle(orc, lanes):
    """f16_dots equals oracle_f16_dot (C, fmaf) and orc.np_f16_dot row for row on the hostile FP16 weights: a quarter subnormal, -0,
    +-65504."""
    rng = np.random.default_rng(lanes)
    s = dict(id="host", form=sk.F16, mode="store", rows=24, cols=1024, lanes=lanes)
    ins, _ = sk._inputs(None, orc, s, rng)
    w, x = ins["w"], ins["x"][0]
    got = sk.f16_dots(orc, w, x, lanes)
    want = np.array([orc.f16_dot(w[r], x, lanes) for r in range(24)], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert np.array_equal(got.view(np.uint32), np.array([orc.np_f16_dot(w[r], x, lanes) for r in range(24)], np.float32).view(np.uint32))


def test_argmax_restatement(orc):
    """orc.argmax is the first strict maximum: ties inside a group, far apart, and all-negative rows."""
    v = np.full(1027, -3.0, np.float32)
    v[[5, 6, 1026]] = -1.0
    assert orc.argmax(v) == 5
    assert orc.argmax(np.full(9, -2.0, np.float32)) == 0
