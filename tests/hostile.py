"""Model builders for the hostile-value tests (tests/test_hostile_host.py on the CPU, tests/test_gpu_hostile.py on the GPU).  TEST
INFRASTRUCTURE ONLY, like tests/qwen2_oracle.py.

synth.build_tensors draws i.i.d. Gaussian weights and quantises them with the project's own quantiser, so a suite built on it never
sees a tied logit, an activation outlier, a saturated softmax or SwiGLU, or a weight block another quantiser could have written.  Every
builder here starts from synth.build_tensors and edits tensors so that one such property is planted; all values stay finite and nothing
indexes out of range: the models change numbers only.  `assert_finite` (called by every builder) runs the CPU oracle over a few
positions and refuses a model whose logits are not finite.

Q8_0 tensors that need blocks our quantiser never emits are assembled as raw 34-byte blocks (`q8_raw`): f16 d + 32 int8.
"""
from __future__ import annotations

import numpy as np

import __graft_entry__ as ge

from devstral_oracle import DevstralOracle
from granite_oracle import GraniteOracle
from qwen2_oracle import Qwen2Oracle
from qwen2moe_oracle import Qwen2MoEOracle

pkg = ge.import_package()
G = pkg.gguf.GGMLType
synth, loader = pkg.synth, pkg.loader


def oracle_for(orc, m, lanes: int = 16):
    """The CPU restatement of the reference's forward pass for the model's architecture."""
    cls = {loader.ARCH_QWEN2: Qwen2Oracle, loader.ARCH_QWEN2_MOE: Qwen2MoEOracle, loader.ARCH_GRANITE: GraniteOracle,
           loader.ARCH_DEVSTRAL: DevstralOracle}.get(m.configuration.arch)
    return orc.OracleModel(m, lanes=lanes) if cls is None else cls(orc, m, lanes=lanes)


def assert_finite(m, tokens=(1, 2, 3)):
    orc = ge.import_oracle()
    om = oracle_for(orc, m)
    try:
        for pos, tok in enumerate(tokens):
            lg = om.forward(int(tok), pos)
            assert np.isfinite(lg).all(), f"the oracle's logits are not finite at position {pos} (token {tok})"
    finally:
        om.close()
    return m


# ---- raw tensors ---------------------------------------------------------------------------------------------------------------

def q8_raw(d, q) -> np.ndarray:
    """Q8_0 bytes of blocks with f16 scales d [nb] (or their uint16 bit patterns) and int8 quants q [nb, 32]."""
    d = np.asarray(d)
    q = np.ascontiguousarray(q, dtype=np.int8).reshape(-1, 32)
    out = np.empty((q.shape[0], 34), dtype=np.uint8)
    bits = d.astype(np.uint16) if d.dtype.kind in "ui" else d.astype(np.float16).view(np.uint16)
    out[:, :2] = bits.reshape(-1, 1).view(np.uint8)
    out[:, 2:] = q.view(np.uint8)
    return out.reshape(-1)


def q8_split(raw):
    """(d bits uint16 [nb], q int8 [nb, 32]) copies of a Q8_0 tensor's blocks."""
    b = np.asarray(raw).reshape(-1, 34)
    return b[:, :2].copy().view(np.uint16).reshape(-1), b[:, 2:].copy().view(np.int8)


def base_tensors(shape, quant: int, seed: int, w_std: float = 0.0, fast: bool = False):
    """(Shape, {name: (type, dims, writable bytes)}) of a synth shape (its name, or a Shape of the caller's own).  fast: generated with
    torch (synth.build_tensors_fast, fan-in scaled), for widths where numpy takes minutes."""
    sh = synth.SHAPES[shape] if isinstance(shape, str) else shape
    if fast:
        return sh, dict(synth.build_tensors_fast(sh, quant, seed=seed))  # host arrays of its own, writable
    return sh, {n: (tt, d, np.array(raw, copy=True)) for n, tt, d, raw in synth.build_tensors(sh, quant, seed, w_std)}


def zero_residual(t: dict):
    """Wo = W2 = 0 (zero bytes are zero weights in every type): x stays the embedding row through every norm of the step."""
    for n, (tt, d, raw) in t.items():
        if "attn_output" in n or "ffn_down" in n:
            t[n] = (tt, d, np.zeros_like(raw))


def row_bytes(tt: int, cols: int) -> int:
    return {G.F32: cols * 4, G.F16: cols * 2, G.Q8_0: cols // 32 * 34}[tt]


def scale_rows(entry, r0: int, r1: int, log2: int):
    """Rows [r0, r1) of a Q8_0 / F16 matrix times 2^log2, exactly (Q8_0: the block scales; every scaled value must stay a normal f16)."""
    tt, dims, raw = entry
    rb = row_bytes(tt, dims[0])
    part = raw[r0 * rb:r1 * rb]
    if tt == G.Q8_0:
        blk = part.reshape(-1, 34)
        d = blk[:, :2].copy().view(np.float16).astype(np.float32) * np.float32(2.0 ** log2)
        assert np.all(np.abs(d) < 65504) and np.all((np.abs(d) >= 2.0 ** -14) | (d == 0))
        blk[:, :2] = d.astype(np.float16).reshape(-1, 1).view(np.uint8)
    else:
        w = part.view(np.float16).astype(np.float32) * np.float32(2.0 ** log2)
        assert np.all(np.abs(w) < 65504)
        part.view(np.float16)[:] = w.astype(np.float16)
    return entry


def zero_rows(entry, rows):
    tt, dims, raw = entry
    rb = row_bytes(tt, dims[0])
    for r in rows:
        raw[r * rb:(r + 1) * rb] = 0
    return entry


# ---- tied logits ---------------------------------------------------------------------------------------------------------------

TIE_KINDS = ("group", "warps", "ctas", "padding", "identical", "zero")


def tie_rows(kind: str, V: int):
    """(A, B): the rows that share the maximum after an even / an odd input token.  group: two rows of one 4-row group; warps: rows of
    different groups at growing distances (neighbouring warps of the streaming classifier's CTA, whatever its row tile); ctas: the first
    and the last row of the vocabulary; padding: the last row (alone with the zero padding rows in its 4-row group when V % 4 == 1) and
    an earlier one."""
    A = {"group": [5, 6], "warps": [9, 13, 17, 29, 61, 125, 253], "ctas": [0, V - 1], "padding": [V - 3, V - 1]}[kind]
    return A, [2, V - 2]


def tied_logits(shape_name: str, quant: int, kind: str, ctx: int = 32, seed: int = 77):
    """Classifier rows duplicated byte for byte, so that their logits are bit-equal, with a boosted column that makes them the maximum:
    every even token's embedding row carries 4 in column 0, every odd token's in column 1; the rows of A carry a large column 0, those of
    B a large column 1.  FloatTensor.argmax is the first strict maximum: min(A) after an even token, min(B) = 2 after an odd one, so a
    greedy loop alternates between the two sets when min(A) is odd.  Tied-embedding shapes duplicate embedding rows instead.
    identical: every classifier row is the same row (answer 0).  zero: an all-zero classifier whose zeros carry both signs (Q8_0: d = 0
    under random quants; F16: +0 / -0), answer 0.  Both need an untied shape."""
    sh, t = base_tensors(shape_name, quant, seed, w_std=0.02)  # small layer outputs: the planted columns survive the residual stream
    V, D = sh.vocab, sh.dim
    rng = np.random.default_rng(seed)
    emb = (rng.standard_normal((V, D)) * 0.1).astype(np.float32)
    par = np.arange(V) % 2
    emb[:, 0] = np.where(par == 0, 4.0, 0.0)
    emb[:, 1] = np.where(par == 1, 4.0, 0.0)
    if kind in ("identical", "zero"):
        assert not sh.tied, "an identical / all-zero classifier needs a classifier of its own"
        A = B = []
    else:
        A, B = tie_rows(kind, V)
    if sh.tied:
        for rows, col in ((A, 0), (B, 1)):
            w = (rng.standard_normal(D) * 0.1).astype(np.float32)
            w[0:2] = 0.0
            w[col] = 8.0
            emb[rows] = w
    else:
        rb = row_bytes(quant, D)
        out = t["output.weight"][2]
        for rows, col in ((A, 0), (B, 1)):
            w = (rng.standard_normal(D) / np.sqrt(D)).astype(np.float32)
            w[0:2] = 0.0
            w[col] = 1.0
            enc = synth.encode(w, quant)
            for r in rows:
                out[r * rb:(r + 1) * rb] = enc
        if kind == "identical":
            out.reshape(V, rb)[:] = out[5 * rb:6 * rb]
        if kind == "zero":
            if quant == G.Q8_0:
                out[:] = q8_raw(np.zeros(V * D // 32, np.uint16), rng.integers(-127, 128, (V * D // 32, 32)))
            else:
                out.view(np.uint16)[:] = rng.integers(0, 2, V * D).astype(np.uint16) << 15
    t["token_embd.weight"] = (quant, (D, V), synth.encode(emb.reshape(-1), quant))
    return assert_finite(loader.model_from_tensors(sh, quant, t, ctx))


# ---- activation outliers -------------------------------------------------------------------------------------------------------

OUTLIER_KINDS = ("benign", "outlier_early", "outlier_mid", "outlier_last", "zero", "zero_head", "pow2_below", "pow2_at", "pow2_above",
                 "many_binades", "constant")
OUTLIER_TOKEN = {k: i + 1 for i, k in enumerate(OUTLIER_KINDS)}  # the token whose embedding row is of that kind


def outlier_row(kind: str, D: int, rng):
    """(d float32 [D/32] powers of two or 0, q int8 [D/32, 32]) of one embedding row, x = q * d: exact in Q8_0 blocks and in f16.
    The kinds mirror test_exact_parallel_sequential_sum's: one channel more than 2^10 times every other (early / middle / last index),
    an all-zero row (ss = 0: the norm multiplies by 1 / sqrt(eps), and every activation block is zero), a zero head then data, squares
    that sum to just below / exactly / just above a power of two, terms that rotate through 36 binades, a constant row."""
    nb = D // 32
    d = np.full(nb, 2.0 ** -6, dtype=np.float32)
    q = rng.integers(-127, 128, (nb, 32)).astype(np.int8)
    if kind.startswith("outlier_"):
        i = {"outlier_early": 3, "outlier_mid": D // 2 + 5, "outlier_last": D - 1}[kind]
        q[i // 32] = 0
        q[i // 32, i % 32] = 127
        d[i // 32] = 32.0  # 4064 against at most 127 / 64
    elif kind == "zero":
        d[:], q[:] = 0.0, 0
    elif kind == "zero_head":
        d[:nb // 2], q[:nb // 2] = 0.0, 0
    elif kind.startswith("pow2_"):
        P = 1 << (D.bit_length() - 1)  # P halves: the squares sum to P / 4 exactly
        d[:] = 2.0 ** -7
        flat = np.zeros(D, dtype=np.int8)
        flat[:P] = 64
        flat[P - 1] = {"pow2_below": 63, "pow2_at": 64, "pow2_above": 65}[kind]
        q = flat.reshape(nb, 32)
    elif kind == "many_binades":
        d = (2.0 ** ((np.arange(nb) * 5) % 13 - 7.0)).astype(np.float32)
        q = ((1 << rng.integers(0, 7, (nb, 32))) * rng.choice([-1, 1], (nb, 32))).astype(np.int8)
    elif kind == "constant":
        q[:] = 100
    return d, q


def outlier_embeddings(shape_name, quant: int, ctx: int = 16, seed: int = 31, fast: bool = False):
    """Wo = W2 = 0 and one embedding row per kind of OUTLIER_KINDS at token OUTLIER_TOKEN[kind]: every RMSNorm of a step over such a
    token (attention, FFN and final norm of every layer; the per-head q/k norm sees what Wq / Wk make of it) reads that row."""
    sh, t = base_tensors(shape_name, quant, seed, fast=fast)
    zero_residual(t)
    V, D = sh.vocab, sh.dim
    rng = np.random.default_rng(seed)
    tt, dims, raw = t["token_embd.weight"]
    rb = row_bytes(quant, D)
    for kind, tok in OUTLIER_TOKEN.items():
        d, q = outlier_row(kind, D, rng)
        if quant == G.Q8_0:
            raw[tok * rb:(tok + 1) * rb] = q8_raw(d, q)
        else:
            x = q.astype(np.float32) * d[:, None]
            assert np.array_equal(x.astype(np.float16).astype(np.float32), x)
            raw[tok * rb:(tok + 1) * rb] = x.astype(np.float16).reshape(-1).view(np.uint8)
    return assert_finite(loader.model_from_tensors(sh, quant, t, ctx), tokens=list(OUTLIER_TOKEN.values()))


def zero_qk_rows(shape_name: str, quant: int, ctx: int = 16, seed: int = 33):
    """Qwen3: Wq and Wk rows of head 0 zeroed in every layer, so its per-head q/k RMSNorm reads an all-zero vector (ss = 0)."""
    sh, t = base_tensors(shape_name, quant, seed)
    assert sh.arch == "qwen3"
    for l in range(sh.n_layers):
        zero_rows(t[f"blk.{l}.attn_q.weight"], range(sh.head_size))
        zero_rows(t[f"blk.{l}.attn_k.weight"], range(sh.head_size))
    return assert_finite(loader.model_from_tensors(sh, quant, t, ctx))


# ---- saturated softmax and SwiGLU ----------------------------------------------------------------------------------------------

def _qk_parts(sh, t, l):
    """[(entry, row0, row1)] of layer l's query and key projections (Phi-3: row ranges of the fused attn_qkv)."""
    if sh.arch == "phi3":
        e = t[f"blk.{l}.attn_qkv.weight"]
        return (e, 0, sh.q_dim), (e, sh.q_dim, sh.q_dim + sh.kv_dim)
    return (t[f"blk.{l}.attn_q.weight"], 0, sh.q_dim), (t[f"blk.{l}.attn_k.weight"], 0, sh.kv_dim)


def saturated_attention(shape_name: str, quant: int, kind: str = "peaked", ctx: int = 160, seed: int = 41):
    """peaked: Wq and Wk times 16 each, so the scores (O(1) in the synthetic models) spread over hundreds of nats: exp(score - max) lands
    in the float subnormals and at 0, and short rows are one-hot (the sum is exactly 1).  uniform: Wq = 0, so every score is 0, the sum
    is exactly the number of keys and every weight 1 / n.  Granite shapes scale through their attention multiplier as well, which the
    model keeps; the biases of Qwen2 shapes are left alone."""
    sh, t = base_tensors(shape_name, quant, seed)
    for l in range(sh.n_layers):
        (qe, q0, q1), (ke, k0, k1) = _qk_parts(sh, t, l)
        if kind == "uniform":
            zero_rows(qe, range(q0, q1))
        elif sh.arch == "qwen3":  # the per-head q/k norm undoes any scale of Wq / Wk: scale the norms' weights
            for n in (f"blk.{l}.attn_q_norm.weight", f"blk.{l}.attn_k_norm.weight"):
                t[n][2].view(np.float32)[:] *= np.float32(16)
        else:
            scale_rows(qe, q0, q1, 4)
            scale_rows(ke, k0, k1, 4)
    return assert_finite(loader.model_from_tensors(sh, quant, t, ctx))


def saturated_swiglu(shape_name: str, quant: int, ctx: int = 16, seed: int = 43):
    """Gate rows times 256 (row % 3 == 1: g reaches +-(100 ... 1000), exp(-g) overflows the float it is narrowed to and g / inf = -0 for
    the negative ones) or zeroed (row % 3 == 2: g = +0 exactly); rows % 3 == 0 stay as they were."""
    sh, t = base_tensors(shape_name, quant, seed)
    H = sh.hidden
    for l in range(sh.n_layers):
        e = t[f"blk.{l}.ffn_up.weight" if sh.arch == "phi3" else f"blk.{l}.ffn_gate.weight"]  # Phi-3: [gate; up] rows
        for r in range(1, H, 3):
            scale_rows(e, r, r + 1, 8)
        zero_rows(e, range(2, H, 3))
    return assert_finite(loader.model_from_tensors(sh, quant, t, ctx))


# ---- extreme weight blocks -----------------------------------------------------------------------------------------------------

Q8_BLOCK_KINDS = ("d_zero", "d_subnormal", "d_negative", "q_minus128", "q_pm127_large_d")


def extreme_q8_blocks(shape_name: str, ctx: int = 16, seed: int = 51, share: float = 0.08):
    """In every Q8_0 tensor (embedding, QKV, Wo, gate / up, W2, classifier) a seeded `share` of the blocks is replaced, the five kinds in
    rotation: d = 0 under the block's own quants; d = the smallest f16 subnormal; d negated; every q = -128; q = +-127 with four times
    the block's d.  All are legal GGUF; the project's quantiser emits none of them."""
    sh, t = base_tensors(shape_name, G.Q8_0, seed)
    rng = np.random.default_rng(seed)
    for n, (tt, dims, raw) in t.items():
        if tt != G.Q8_0:
            continue
        d, q = q8_split(raw)
        pick = np.flatnonzero(rng.random(len(d)) < share)
        kind = np.arange(len(pick)) % 5
        d[pick[kind == 0]] = 0
        d[pick[kind == 1]] = 1
        d[pick[kind == 2]] ^= 0x8000
        q[pick[kind == 3]] = -128
        p4 = pick[kind == 4]
        q[p4] = rng.choice(np.array([-127, 127], dtype=np.int8), (len(p4), 32))
        d[p4] = (d[p4].view(np.float16).astype(np.float32) * 4).astype(np.float16).view(np.uint16)
        raw[:] = q8_raw(d, q)
    return assert_finite(loader.model_from_tensors(sh, G.Q8_0, t, ctx))


def extreme_f16_weights(shape_name: str, ctx: int = 16, seed: int = 53):
    """In every F16 tensor: 25 % subnormals of both signs (the vector dot products flush them, the embedding gather and the scalar tails
    do not), 2 % -0, 1 % +0 and one value in 1024 at +-65504.  In a tied shape the same tensor is read both ways."""
    sh, t = base_tensors(shape_name, G.F16, seed)
    rng = np.random.default_rng(seed)
    for n, (tt, dims, raw) in t.items():
        if tt != G.F16:
            continue
        w = raw.view(np.uint16)
        u = rng.random(len(w))
        sub = u < 0.25
        w[sub] = rng.integers(1, 0x400, int(sub.sum())).astype(np.uint16) | (rng.integers(0, 2, int(sub.sum())).astype(np.uint16) << 15)
        w[(u >= 0.25) & (u < 0.27)] = 0x8000
        w[(u >= 0.27) & (u < 0.28)] = 0
        big = (u >= 0.28) & (u < 0.28 + 1.0 / 1024)
        w[big] = 0x7BFF | (rng.integers(0, 2, int(big.sum())).astype(np.uint16) << 15)
    return assert_finite(loader.model_from_tensors(sh, G.F16, t, ctx))
