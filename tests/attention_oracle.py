"""A float32 restatement of the CPU path's attention, in the oracle's order (oracle.c's forward, InferenceCore.java:75-137 and
:594-619; qwen2_oracle.py for the q|k|v bias, granite_oracle.py for the attention scale):

  bias add -> Qwen3 per-head RMSNorm (sequential sum) -> interleaved or NeoX rotation -> K / V row into the cache ->
  score_t = scalarDot(q, k_t) (one unfused chain per key) / sqrt(head size), or * scale -> softmax (max, (float)exp((double)(s - max))
  with the oracle's exp, sequential sum, divide) -> out = saxpyInPlace over t -> the oracle's Q8_0 quantisation of each row.

Every chain is sequential (numpy float32 operations round each step, np.add.accumulate sums in order); independent chains -- heads,
keys, output elements -- run as array operations, so a 20 000-key row takes seconds.  tests/test_attention_host.py pins it to the
oracle bit for bit; tests/test_gpu_attention.py holds b200_test_attention to it."""
from __future__ import annotations

import numpy as np

f32 = np.float32
KF_NEOX, KF_QKNORM, KF_QKVBIAS, KF_ATTSCALE = 1, 2, 4, 8


def _orc():
    import __graft_entry__ as ge
    return ge.import_oracle()


def head_norm(x: np.ndarray, w: np.ndarray, eps: float) -> np.ndarray:
    """oracle_rmsnorm on each row of x [n, hs]: ss = sequential sum of x * x, ss / hs + eps, (float)(1 / sqrt((double)ss)), w * (ss * x)."""
    x = np.asarray(x, dtype=f32)
    ss = np.add.accumulate((x * x).astype(f32), axis=1, dtype=f32)[:, -1]
    ss = ((ss / f32(x.shape[1])).astype(f32) + f32(eps)).astype(f32)
    ss = (1.0 / np.sqrt(ss.astype(np.float64))).astype(f32)
    return (np.asarray(w, dtype=f32)[None, :] * (ss[:, None] * x).astype(f32)).astype(f32)


def rotate(x: np.ndarray, cr: np.ndarray, ci: np.ndarray, neox: bool) -> np.ndarray:
    """RoPE of each row of x [n, hs] at one position (cr, ci: that position's [hs / 2] table row): pairs (2p, 2p + 1), or (p, p + hs / 2)
    for NeoX (Qwen3, Phi-3), each rotated as v0 * cr - v1 * ci, v0 * ci + v1 * cr with every product and sum rounded."""
    half = x.shape[1] // 2
    i0 = np.arange(half) if neox else 2 * np.arange(half)
    i1 = i0 + half if neox else i0 + 1
    v0, v1 = x[:, i0], x[:, i1]
    out = np.empty_like(x)
    out[:, i0] = ((v0 * cr).astype(f32) - (v1 * ci).astype(f32)).astype(f32)
    out[:, i1] = ((v0 * ci).astype(f32) + (v1 * cr).astype(f32)).astype(f32)
    return out


def prologue(qkv_row, pos: int, n_heads: int, n_kv_heads: int, hs: int, arch: int, rope_cr, rope_ci, q_norm=None, k_norm=None, qkv_bias=None,
             eps: float = 1e-6):
    """(q [n_heads, hs], k [n_kv_heads, hs], v [n_kv_heads, hs]) of one packed q|k|v row at position pos: what attention reads."""
    qd, kvd = n_heads * hs, n_kv_heads * hs
    x = np.asarray(qkv_row, dtype=f32)
    if arch & KF_QKVBIAS:
        x = (x + np.asarray(qkv_bias, dtype=f32)).astype(f32)
    q, k, v = x[:qd].reshape(n_heads, hs), x[qd:qd + kvd].reshape(n_kv_heads, hs), x[qd + kvd:qd + 2 * kvd].reshape(n_kv_heads, hs)
    if arch & KF_QKNORM:
        q, k = head_norm(q, q_norm, eps), head_norm(k, k_norm, eps)
    half = hs // 2
    cr = np.asarray(rope_cr, dtype=f32).reshape(-1, half)[pos]
    ci = np.asarray(rope_ci, dtype=f32).reshape(-1, half)[pos]
    neox = bool(arch & KF_NEOX)
    return rotate(q, cr, ci, neox), rotate(k, cr, ci, neox), v.copy()


def attend(q: np.ndarray, K: np.ndarray, V: np.ndarray, pos: int, score_arg: float, attscale: bool = False):
    """(softmax weights [n_heads, pos + 1], output [n_heads, hs]) of the rotated q [n_heads, hs] over the cache rows K, V [ctx][n_kv][hs]
    0..pos: only those rows are read."""
    nh, hs = q.shape
    nkv = K.shape[1]
    kvh = np.arange(nh) // (nh // nkv)
    nt = pos + 1
    Kt, Vt = np.asarray(K[:nt], dtype=f32), np.asarray(V[:nt], dtype=f32)
    s = np.zeros((nh, nt), dtype=f32)
    for i in range(hs):  # scalarDot: r += a[j] * b[j], in j order, per (head, key)
        s += q[:, i:i + 1] * Kt[:, kvh, i].T
    s = (s * f32(score_arg)).astype(f32) if attscale else (s / f32(score_arg)).astype(f32)
    mx = s.max(axis=1)
    e = _orc().exp_narrow((s - mx[:, None]).astype(f32))
    total = np.add.accumulate(e, axis=1, dtype=f32)[:, -1]
    a = (e / total[:, None]).astype(f32)
    out = np.zeros((nh, hs), dtype=f32)
    for t in range(nt):  # saxpyInPlace: out[i] = a * v[i] + out[i], in t order
        out = ((a[:, t:t + 1] * Vt[t, kvh, :]).astype(f32) + out).astype(f32)
    return a, out


def reference(form: str, head_size: int, n_heads: int, n_kv_heads: int, slots, positions, qkv, k_cache, v_cache, rope_cr, rope_ci, *, arch: int = 0,
              eps: float = 1e-6, score_arg: float | None = None, q_norm=None, k_norm=None, qkv_bias=None) -> dict:
    """What b200_test_attention must return for these arguments: every row's K / V written first (a chunk's and a multi-position
    step's rows read the rows earlier rows of their slot wrote), then each row's attention.  {"qkv": the rows after the launch (the
    rotated q written back; the persistent form writes nothing back), "k_cache", "v_cache", "xq", "xs", "xb" (row 0's float output),
    "att": each row's softmax weights}."""
    hs, qd = head_size, n_heads * head_size
    score_arg = float(np.sqrt(np.float64(hs))) if score_arg is None else score_arg
    kc, vc = np.array(k_cache, dtype=f32), np.array(v_cache, dtype=f32)
    ctx = kc.shape[1]
    qkv_out = np.array(qkv, dtype=f32)
    qs = []
    for r, (s, p) in enumerate(zip(slots, positions)):
        q, k, v = prologue(qkv[r], p, n_heads, n_kv_heads, hs, arch, rope_cr, rope_ci, q_norm, k_norm, qkv_bias, eps)
        kc[s, p], vc[s, p] = k.reshape(-1), v.reshape(-1)
        if form != "persistent":
            qkv_out[r, :qd] = q.reshape(-1)
        qs.append(q)
    outs, atts = [], []
    for r, (s, p) in enumerate(zip(slots, positions)):
        a, o = attend(qs[r], kc[s].reshape(ctx, n_kv_heads, hs), vc[s].reshape(ctx, n_kv_heads, hs), p, score_arg, bool(arch & KF_ATTSCALE))
        outs.append(o.reshape(-1))
        atts.append(a)
    xq, xs = zip(*[_orc().q8_quantize(o) for o in outs])
    return {"qkv": qkv_out, "k_cache": kc, "v_cache": vc, "xq": np.stack(xq), "xs": np.stack(xs), "xb": outs[0], "att": atts}
