"""The decode weight streams one launch at a time (b200_test_stream): every stream form -- Q8_0 tiles, resident K-quant tiles, the
batched stream and the FP16 rings -- against a float32 restatement of its dot products, bit for bit, at grids, ring depths and shapes
no model reaches.  Each case names the edge it exists for, and tests/test_stream_kernels_host.py checks on the CPU that the launch
configuration reaches it; here the configuration the hook reports is asserted as well."""
import zlib

import numpy as np
import pytest

import hostile
from test_gpu_prefill_i8 import _activations, _dot_q8, _swiglu_q8, _weights
from test_gpu_prefill_w8a16 import _q8_blocks

pytestmark = pytest.mark.gpu

Q8, F16, Q4K, Q5K, Q6K = 8, 1, 12, 13, 14
KQ_BYTES = {Q4K: 144, Q5K: 176, Q6K: 210}
SMS = 132  # H100 SXM: the grid of "grid 0" cases, for the host-side configuration checks
f32 = np.float32


def C(id, form, mode, rows, cols, expect=None, edges=(), **kw):
    """One case: the hook's arguments, the configuration it must report (expect) and the edges (test_stream_kernels_host.edges) it reaches."""
    return pytest.param(dict(id=id, form=form, mode=mode, rows=rows, cols=cols, expect=expect or {}, edges=tuple(edges), **kw), id=id)


# ---- the cases ----------------------------------------------------------------------------------------------------------------
RING = [
    C("q8-grid1-laps", Q8, "store", 256, 4096, {"grid": 1, "stages": 3}, ["laps"], grid=1, stages=3, argmax=True),
    C("q8-grid3-nw1", Q8, "resid", 100, 2592, {"grid": 3, "stages": 4}, ["nw1", "laps"], grid=3, stages=4, oscale=0.5),
    C("q8-empty-ctas", Q8, "store", 20, 544, {"grid": 8, "min_groups": 0}, ["empty_cta"], grid=8, argmax=True),
    C("q8-last-round-nw1", Q8, "store", 260, 2560, {"grid": 4}, ["nw1"], grid=4, stages=5, argmax=True),
    C("q8-last-round-nw7", Q8, "resid", 252, 2560, {"grid": 4}, ["nw7"], grid=4, stages=3),
    C("q8-stages3", Q8, "store", 1056, 4096, {"stages": 3}, [], stages=3),
    C("q8-stages4", Q8, "store", 1056, 4096, {"stages": 4}, [], stages=4),
    C("q8-stages5", Q8, "store", 1056, 4096, {"stages": 5}, [], stages=5),
    C("q8-stages-96k", Q8, "store", 1056, 4096, {"stages": 9}, []),
    C("q8-stages16-over-slice", Q8, "store", 1056, 4096, {"stages": 16}, ["stages_gt_slice"], stages=16),
    C("kq4-grid1-laps", Q4K, "store", 64, 4096, {"grid": 1, "stages": 3}, ["laps"], grid=1, stages=3, argmax=True),
    C("kq6-last-round-nw1", Q6K, "resid", 260, 2560, {"grid": 4}, ["nw1"], grid=4, stages=4, oscale=0.25),
    C("kq5-last-round-nw7", Q5K, "store", 252, 2048, {"grid": 4}, ["nw7"], grid=4),
    C("kq4-empty-ctas", Q4K, "store", 20, 1024, {"grid": 8, "min_groups": 0}, ["empty_cta"], grid=8, argmax=True),
    C("kq6-stages16-over-slice", Q6K, "store", 532, 4096, {"stages": 16}, ["stages_gt_slice"], stages=16),
    C("kq5-stages3", Q5K, "store", 532, 4096, {"stages": 3}, [], stages=3),
]
WIDTHS = [C(f"q8-width{k}", Q8, "store" if i % 2 == 0 else "resid", 132 * 4 + 3, k, {}, [], oscale=1.0 if i % 2 == 0 else 0.75)
          for i, k in enumerate((32, 96, 544, 2560, 2592, 2656, 4096, 14336, 18944))] + \
         [C(f"kq{f - 8}-width{k}", f, "store", 132 * 4 + 1, k, {}, []) for f, k in ((Q4K, 256), (Q5K, 2560), (Q6K, 14336))]
EPILOGUE = [
    C("q8-resid-oscale", Q8, "resid", 132 * 8, 4096, {}, [], oscale=0.22),
    C("q8-ragged1-negative", Q8, "store", 253, 2048, {}, [], argmax=True, weights="negative"),
    C("q8-ragged2-negative", Q8, "store", 254, 2048, {"grid": 64}, [], argmax=True, weights="negative", grid=64),
    C("q8-ragged3-negative", Q8, "store", 255, 2048, {}, [], argmax=True, weights="negative"),
    C("q8-tie-group", Q8, "store", 1059, 2048, {}, [], argmax=True, weights="tie-group"),
    C("q8-tie-warps", Q8, "store", 1059, 2048, {"grid": 2}, [], argmax=True, weights="tie-warps", grid=2),
    C("q8-tie-lane", Q8, "store", 1059, 2048, {"grid": 2}, [], argmax=True, weights="tie-lane", grid=2),
    C("q8-tie-ctas", Q8, "store", 1059, 2048, {}, [], argmax=True, weights="tie-ctas"),
    C("q8-tie-padding", Q8, "store", 1057, 2048, {}, [], argmax=True, weights="tie-padding"),
    C("q8-gateup-block-1cta", Q8, "gateup", 256, 2048, {"grid": 1, "stages": 3}, ["blocks_1"], grid=1, stages=3),
    C("q8-gateup-block-2ctas", Q8, "gateup", 96, 4096, {"grid": 2}, ["blocks_2"], grid=2),
    C("q8-gateup-block-3ctas", Q8, "gateup", 256, 2048, {"min_groups": 0}, ["blocks_3", "empty_cta"]),
    C("q8-gateup-wide", Q8, "gateup", 1024, 4096, {}, ["blocks_3"]),
    C("q8-gateup-launches2", Q8, "gateup", 256, 4096, {"grid": 24}, ["blocks_3"], grid=24, launches=2),
    C("q8-resid-launches2", Q8, "resid", 300, 4096, {}, [], launches=2, oscale=0.5),
    C("q8-store-argmax-launches2", Q8, "store", 1027, 2048, {}, [], launches=2, argmax=True),
    C("q8-pair", Q8, "gateup", 512, 2048, {}, ["blocks_3"], pair=2048, oscale=0.5),
    C("q8-pair-norm-launches2", Q8, "gateup", 256, 2048, {}, ["blocks_3"], pair=1024, norm=True, launches=2),
    C("kq4-pair", Q4K, "gateup", 512, 2048, {}, ["blocks_3"], pair=512),
]
NORM = [C(f"norm-{m}-dim{d}", Q8, m, 256 if m == "gateup" else 132 * 4 + 2, d, {}, [], norm=True, argmax=m == "store")
        for d in (256, 1024, 2048, 2848, 3072, 4096, 5120) for m in ("store", "gateup")] + \
       [C(f"norm-{k}", Q8, "store", 260, 2048, {}, [], norm=True, argmax=True, act=k) for k in ("zero", "zero_head", "outlier_mid", "pow2_below",
                                                                                             "pow2_at", "pow2_above")] + \
       [C("norm-from-emb-store", Q8, "store", 300, 2048, {}, [], norm=True, from_emb=True, argmax=True, launches=2),
        C("norm-from-emb-gateup", Q8, "gateup", 256, 3072, {}, [], norm=True, from_emb=True)]
KQUANT = [C(f"kq{f - 8}-{m}-{w}{'-norm' if n else ''}", f, m, 256 if m == "gateup" else 132 * 4 + 3, 2048 if n else 4096, {}, [], norm=n, weights=w,
            argmax=m == "store") for f in (Q4K, Q5K, Q6K) for m, n, w in (("store", False, "random"), ("gateup", True, "random"),
                                                                         ("store", True, "bits"), ("resid", False, "bits"))]
BATCH = [
    C("b1-store-544-grid1-s3", Q8, "store", 37, 544, {"grid": 1, "stages": 3}, ["laps"], nrow=1, grid=1, stages=3, argmax=True),
    C("b3-resid-14336-max", Q8, "resid", 260, 14336, {}, [], nrow=3, oscale=0.5),
    C("b8-gateup-2656-grid1-s3", Q8, "gateup", 256, 2656, {"grid": 1, "stages": 3}, ["blocks_1", "laps"], nrow=8, grid=1, stages=3),
    C("b8-store-2656-max", Q8, "store", 1027, 2656, {"stages": 16}, [], nrow=8, argmax=True),
    C("b8-gateup-544-s3", Q8, "gateup", 256, 544, {"stages": 3}, ["blocks_3"], nrow=8, stages=3, launches=2),
    C("b3-store-14336-grid1-s3", Q8, "store", 37, 14336, {"grid": 1, "stages": 3}, ["laps"], nrow=3, grid=1, stages=3, argmax=True),
    C("b8-resid-544-launches2", Q8, "resid", 531, 544, {}, [], nrow=8, launches=2, oscale=0.3),
    C("b1-gateup-14336-max", Q8, "gateup", 512, 14336, {}, ["blocks_3"], nrow=1),
    C("b8-store-14336-s3", Q8, "store", 133, 14336, {"stages": 3}, [], nrow=8, stages=3, argmax=True),
]
FP16 = [
    C("f16-l16-store-ragged-grid1-s3", F16, "store", 37, 512, {"grid": 1, "stages": 3}, [], lanes=16, grid=1, stages=3, argmax=True),
    C("f16-l8-store-ragged", F16, "store", 1027, 4096, {}, [], lanes=8, argmax=True),
    C("f16-l16-store-ragged-grid2", F16, "store", 1029, 2048, {"grid": 2}, [], lanes=16, grid=2, argmax=True),
    C("f16-l16-resid-grid2-s3", F16, "resid", 258, 2048, {"grid": 2, "stages": 3}, [], lanes=16, grid=2, stages=3, oscale=0.5),
    C("f16-l8-resid", F16, "resid", 1030, 4096, {}, [], lanes=8),
    C("f16-l16-gateup", F16, "gateup", 1024, 2048, {}, [], lanes=16),
    C("f16-l8-gateup-grid2-s3", F16, "gateup", 132, 2048, {"grid": 2, "stages": 3}, [], lanes=8, grid=2, stages=3),
    C("f16-l8-store-grid1", F16, "store", 35, 1024, {"grid": 1}, [], lanes=8, grid=1, argmax=True),
]
CASES = RING + WIDTHS + EPILOGUE + NORM + KQUANT + BATCH + FP16


# ---- inputs -------------------------------------------------------------------------------------------------------------------

def _kq_rows(rng, pkg, fmt, rows, cols, kind):
    """Raw K-quant rows: synth.random_kquant blocks, or arbitrary bytes whose f16 d / dmin fields are finite and below 1 in magnitude
    (every re-quantised Q8_0 scale then stays a finite f16)."""
    if kind == "random":
        return pkg.synth.random_kquant(fmt, rows * cols, rng, zero_blocks=3).reshape(rows, -1)
    b = rng.integers(0, 256, size=(rows * cols // 256, KQ_BYTES[fmt]), dtype=np.uint8)
    for col in ((0, 2) if fmt != Q6K else (208,)):
        b[:, col + 1] &= 0xBB
    return b.reshape(rows, -1)


def _q8_matrix(rng, rows, cols, kind, xq):
    """GGUF Q8_0 rows: hostile random blocks, all-negative dot products, rows tied byte for byte at the maximum, or (gate / up and down
    projections) _q8_blocks' hostile blocks at weight scale, so that most hidden values and their f16 block scales stay finite."""
    if kind == "small":
        return _q8_blocks(rng, rows, cols)
    if kind == "negative":  # activation quants are made positive: every term is negative
        q = -rng.integers(1, 128, size=(rows, cols // 32, 32))
        d = rng.uniform(0.01, 0.02, size=(rows * cols // 32,)).astype(np.float16)
        return hostile.q8_raw(d, q).reshape(rows, -1)
    bq = _weights(rng, rows, cols)
    if kind.startswith("tie-"):  # tie-lane: rows one consumer lane produces in turn (groups 7, 15, 31: warp 7 of CTA 0, lane 1)
        A = [29, 61, 125] if kind == "tie-lane" else hostile.tie_rows(kind[4:], rows)[0]
        top = hostile.q8_raw(np.full(cols // 32, 1.0, np.float16), np.where(xq.reshape(-1, 32) < 0, -127, 127)).reshape(-1)
        for r in A:
            bq[r] = top
    return bq


def _inputs(pkg, orc, s, rng):
    form, mode, rows, cols, L = s["form"], s["mode"], s["rows"], s["cols"], s.get("launches", 1)
    V = max(s.get("nrow", 0), 1)
    kw = dict(nrow=s.get("nrow", 0), grid=s.get("grid", 0), stages=s.get("stages", 0), argmax=s.get("argmax", False), launches=L,
              oscale=s.get("oscale", 1.0), lanes=s.get("lanes", 16))
    ins = {}
    if form == F16 or s.get("norm"):
        x = (rng.standard_normal((L, cols)) * 2).astype(f32)
        act = s.get("act")
        if act:
            d, q = hostile.outlier_row(act, cols, rng)
            x[0] = (q.astype(f32) * d[:, None]).reshape(-1)
        kw["x"] = ins["x"] = x
    else:
        xq, xs = _activations(rng, L * V, cols)
        if s.get("weights") == "negative":
            xq = np.abs(xq.astype(np.int32)).clip(1, 127).astype(np.int8)
            xs = np.abs(xs) + f32(2.0 ** -8)
        if V > 1:  # one all-zero activation row, one hostile row (full-range quants, large and subnormal-ish scales)
            xq[0], xs[0] = 0, 0
            xq[1] = np.where(np.arange(cols) % 2, 127, -128)
            xs[1] = np.where(np.arange(cols // 32) % 3, f32(2.0 ** 8), f32(2.0 ** -20))
        ins["xq"], ins["xs"] = xq.reshape(L, V, cols), xs.reshape(L, V, cols // 32)
        kw["xq"], kw["xs"] = ins["xq"], ins["xs"]
    if s.get("norm"):
        kw["norm_w"] = ins["norm_w"] = (rng.standard_normal(cols) * 0.5 + 1).astype(f32)
        kw["eps"] = ins["eps"] = 1e-5
        if s.get("from_emb"):
            E = 7
            emb_x = (rng.standard_normal((E, cols)) * 0.3).astype(f32)
            ins["emb"] = kw["emb"] = orc.np_requant_q8_0(emb_x.reshape(-1)).reshape(E, -1)
            ins["tokens"] = kw["tokens"] = np.array([3, 5][:L], np.int32)
            kw["emb_rows"] = E
            kw["emb_scale"] = ins["emb_scale"] = 12.0
            del kw["x"]
    nmat = 2 if mode == "gateup" else 1
    if form == F16:
        w = rng.standard_normal((nmat, rows, cols)).astype(np.float16).view(np.uint16)
        u = rng.random(w.shape)
        sub = u < 0.25
        w[sub] = rng.integers(1, 0x400, int(sub.sum())).astype(np.uint16) | (rng.integers(0, 2, int(sub.sum())).astype(np.uint16) << 15)
        w[(u >= 0.25) & (u < 0.27)] = 0x8000
        big = (u >= 0.27) & (u < 0.275)
        w[big] = 0x7BFF | (rng.integers(0, 2, int(big.sum())).astype(np.uint16) << 15)
        mats = list(w)
    elif form == Q8:
        kind = s.get("weights", "small" if mode == "gateup" else "random")
        mats = [_q8_matrix(rng, rows, cols, kind, ins["xq"][0, 0] if "xq" in ins else None) for _ in range(nmat)]
    else:
        mats = [_kq_rows(rng, pkg, form, rows, cols, s.get("weights", "random")) for _ in range(nmat)]
    ins["w"] = kw["w"] = mats[0]
    if mode == "gateup":
        ins["w_up"] = kw["w_up"] = mats[1]
    if mode == "resid":
        ins["out_init"] = kw["out_init"] = (rng.standard_normal((V, rows)) * 4).astype(f32)
    if s.get("pair"):
        D = s["pair"]
        kw["pair"], kw["down_rows"] = True, D
        ins["w_down"] = kw["w_down"] = (_q8_blocks(rng, D, rows) if form == Q8 else _kq_rows(rng, pkg, form, D, rows, "random"))
        ins["out_init"] = kw["out_init"] = (rng.standard_normal(D) * 4).astype(f32)
    return ins, kw


# ---- the restatement ----------------------------------------------------------------------------------------------------------

def q8_of(orc, form, raw, cols):
    """The Q8_0 blocks the stream computes with: the rows themselves, or the resident rows re-quantised as the load-time path does."""
    if form == Q8:
        return raw
    return orc.kquant_to_q8_0(form, np.ascontiguousarray(raw).reshape(-1), raw.shape[0] * cols).reshape(raw.shape[0], -1)


def f16_dots(orc, wbits, x, lanes):
    """orc.np_f16_dot for every row at once: lanes chains of fused multiply-adds over the flushed weights, summed in lane order."""
    w = np.asarray(wbits, np.uint16)
    rows, cols = w.shape
    wf = orc.np_f16_daz(w.reshape(-1)).reshape(rows, cols // lanes, lanes).astype(np.float64)
    xv = np.asarray(x, f32).reshape(cols // lanes, lanes).astype(np.float64)
    acc = np.zeros((rows, lanes), f32)
    for j in range(cols // lanes):
        acc = (wf[:, j, :] * xv[j] + acc.astype(np.float64)).astype(f32)
    r = np.zeros(rows, f32)
    for c in range(lanes):
        r = (r + acc[:, c]).astype(f32)
    return r


def swiglu(g, u):
    with np.errstate(over="ignore"):
        return ((g / (1.0 + np.exp(-g.astype(np.float64))).astype(f32)) * u).astype(f32)


def norm_act(orc, x, w, eps):
    """RMSNorm(x) * w quantised block by block (the fused norm's activation): (int8 [cols], f32 [cols / 32])."""
    h = orc.np_rmsnorm(x, w, eps)
    blocks = [orc.np_q8_quantize_block(h[b * 32:(b + 1) * 32]) for b in range(len(h) // 32)]
    return np.concatenate([q for q, _ in blocks]).astype(np.int8), np.array([s for _, s in blocks], f32)


def reference(orc, s, ins):
    """Per launch: the expected out [V][rows], hq / hs, out_down, x_out and ids."""
    form, mode, rows, cols = s["form"], s["mode"], s["rows"], s["cols"]
    oscale = f32(s.get("oscale", 1.0))
    L, V = s.get("launches", 1), max(s.get("nrow", 0), 1)
    mats = [q8_of(orc, form, ins["w"], cols)] if form != F16 else [ins["w"]]
    if mode == "gateup":
        mats.append(q8_of(orc, form, ins["w_up"], cols) if form != F16 else ins["w_up"])
    res, out = [], ins.get("out_init")
    down = ins.get("out_init") if s.get("pair") else None
    for l in range(L):
        r = {}
        if form == F16:
            accs = [f16_dots(orc, m, ins["x"][l], s["lanes"])[None, :] for m in mats]
        else:
            if s.get("norm"):
                if s.get("from_emb"):
                    d, q = hostile.q8_split(ins["emb"][ins["tokens"][l]])
                    x = (q.astype(f32) * d.view(np.float16).astype(f32)[:, None]).reshape(-1) * f32(ins["emb_scale"])
                    r["x_out"] = x.astype(f32)
                else:
                    x = ins["x"][l]
                aq, a_s = norm_act(orc, x, ins["norm_w"], ins["eps"])
                aq, a_s = aq[None, :], a_s[None, :]
            else:
                aq, a_s = ins["xq"][l], ins["xs"][l]
            accs = [_dot_q8(aq, a_s, m) for m in mats]
        if mode == "gateup":
            if form == F16:
                r["out"] = swiglu(accs[0], accs[1])
            else:
                r["hq"], r["hs"] = _swiglu_q8(accs[0], accs[1])
                r["out"] = swiglu(accs[0], accs[1])
                if s.get("pair"):
                    wd = q8_of(orc, form, ins["w_down"], rows)
                    down = (down + _dot_q8(r["hq"], r["hs"], wd)[0] * oscale).astype(f32)
                    r["out_down"] = down
        elif mode == "resid":
            out = (out + accs[0] * oscale).astype(f32)
            r["out"] = out
        else:
            r["out"] = (accs[0] * oscale).astype(f32)
            if s.get("argmax"):
                r["ids"] = np.array([orc.argmax(row) for row in r["out"]], np.int32)
        res.append(r)
    return res


def _same(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, what
    g, w = got.view(np.uint32 if got.dtype == np.float32 else got.dtype), want.view(np.uint32 if want.dtype == np.float32 else want.dtype)
    bad = np.argwhere(g != w)
    assert bad.size == 0, f"{what}: {len(bad)} of {g.size} differ, first at {tuple(bad[0])}: {got[tuple(bad[0])]!r} != {want[tuple(bad[0])]!r}"


@pytest.mark.parametrize("s", CASES)
def test_stream_bit_exact(pkg, orc, s):
    import test_stream_kernels_host as host
    rng = np.random.default_rng(zlib.crc32(s["id"].encode()))
    ins, kw = _inputs(pkg, orc, s, rng)
    got = pkg.native.test_stream(s["form"], s["mode"], rows=s["rows"], cols=s["cols"], **kw)
    info = got["info"]
    for k, v in s["expect"].items():
        assert info[k] == v, f"{k}: the hook ran {info}"
    for e in s["edges"]:
        assert e in host.edges(s, info), f"edge {e} not reached: {info}"
    for l, want in enumerate(reference(orc, s, ins)):
        for k, v in want.items():
            g = got[k][l]
            _same(g.reshape(np.asarray(v).shape), v, f"launch {l} {k}")
