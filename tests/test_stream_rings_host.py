"""The ring-size rule of the decode weight streams (plan.cu ring_budgets, DESIGN.md section 5a), on CPU through b200_stream_rings:
every shape in synth.SHAPES, in Q8_0 and resident K-quant tile forms, with and without the fused norm."""
import os
import re

import pytest

H100 = dict(sm_bytes=233472, reserve_bytes=1024, optin_bytes=232448)  # cudaDevAttr{MaxSharedMemoryPerMultiprocessor, ReservedSharedMemoryPerBlock, MaxSharedMemoryPerBlockOptin}
SMS = 132
FLOOR = 96 * 1024
Q4_K, Q5_K, Q6_K = 12, 13, 14
_HDR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpullama3.java_b200", "csrc", "stream_matvec.cuh")
MAX_STAGES = int(re.search(r"#define SMV_MAX_STAGES (\d+)", open(_HDR).read()).group(1))


def _att_bytes(head_size):  # k_attention's largest shared-memory score row (ATT_SMEM_FLOATS_MAX) plus room for its static arrays
    return 4096 * 4 + 256


def _fmts(shape, fmt):
    """A resident plan keeps a stream's K-quant tiles only when its width is a multiple of 256 (resident_fmt); else Q8_0 tiles."""
    qd, dim, hid = shape.n_heads * shape.head_size, shape.dim, shape.hidden
    return tuple(fmt if cols % 256 == 0 else 0 for cols in (dim, qd, dim, hid))


def _cases(pkg):
    for name, s in sorted(pkg.synth.SHAPES.items()):
        for fmt in (0, Q4_K, Q5_K, Q6_K):
            for fused in (True, False):
                yield name, s, fmt, fused


def _rings(pkg, s, fmt, fused, **dev):
    return pkg.native.stream_rings(s.dim, s.n_heads * s.head_size, s.n_kv_heads * s.head_size, s.hidden, SMS, fused, _fmts(s, fmt), **dev)


def test_pair_rule_holds_for_every_shape(pkg):
    sm, res, optin = H100["sm_bytes"], H100["reserve_bytes"], H100["optin_bytes"]
    for name, s, fmt, fused in _cases(pkg):
        att = _att_bytes(s.head_size)
        r = _rings(pkg, s, fmt, fused, att_bytes=att, **H100)
        floor = _rings(pkg, s, fmt, fused, att_bytes=att, sm_bytes=FLOOR, reserve_bytes=0, optin_bytes=optin)  # no room beside a neighbour: the flat budget
        tag = f"{name} fmt {fmt} fused {fused}: {r}"
        # each kernel of the chain W2 -> QKV -> attention -> Wo -> gate/up -> W2 fits beside the one before it
        for a, b in ((r["w2"]["smem"], r["qkv"]["smem"]), (r["qkv"]["smem"], att), (att, r["wo"]["smem"]),
                     (r["wo"]["smem"], r["gateup"]["smem"]), (r["gateup"]["smem"], r["w2"]["smem"])):
            assert a + b + 2 * res <= sm, tag
        for k, v in r.items():
            assert v["smem"] <= optin, tag
            assert v["stages"] >= 3, tag
            assert v["stages"] >= floor[k]["stages"], tag  # no stream has fewer stages than the flat 96 KB budget gave it
        assert r["wo"] == floor["wo"] and r["w2"] == floor["w2"], tag  # Wo and W2 keep the flat budget


def test_qkv_and_gateup_rings_are_the_largest_that_fit(pkg):
    """QKV and gate/up hold their whole CTA slice, or the most stages a ring has, or one stage more would break a pair with a
    neighbour: QKV's are W2 and the attention, gate/up's are Wo and W2."""
    sm, res, optin = H100["sm_bytes"], H100["reserve_bytes"], H100["optin_bytes"]
    for name, s, fmt, fused in _cases(pkg):
        att = _att_bytes(s.head_size)
        r = _rings(pkg, s, fmt, fused, att_bytes=att, **H100)
        for k, beside in (("qkv", max(r["w2"]["smem"], att)), ("gateup", max(r["wo"]["smem"], r["w2"]["smem"]))):
            v = r[k]
            if v["stages"] >= v["slice_tiles"] or v["stages"] == MAX_STAGES:
                continue
            more = v["smem"] + v["stage_bytes"]
            assert more > optin or more + beside + 2 * res > sm, f"{name} fmt {fmt} fused {fused}: {k} {r}"


def test_llama_3_8b_rings(pkg):
    """The bench shape on an H100: QKV and gate/up hold 12 stages of 8.7 KB each (7 at the flat 96 KB), Wo 9 and W2 8 as before."""
    s = pkg.synth.SHAPES["llama-3-8b"]
    r = _rings(pkg, s, 0, True, att_bytes=(3 * 128 + 144) * 4 + 64, **H100)
    assert r["qkv"]["stages"] == 12 and r["gateup"]["stages"] == 12
    assert r["wo"]["stages"] == 9 and r["w2"]["stages"] == 8


def test_bad_arguments_are_refused(pkg):
    with pytest.raises(pkg.native.B200Error):
        pkg.native.stream_rings(0, 4096, 1024, 14336, SMS, True, att_bytes=0)
    with pytest.raises(pkg.native.B200Error):
        pkg.native.stream_rings(4096, 4096, 1024, 14336, SMS, True, (3, 0, 0, 0), att_bytes=0)
