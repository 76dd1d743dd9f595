"""ctypes binding of oracle/liboracle.so -- the CPU restatement of the reference's
onGPU=false path (oracle.c).  TEST INFRASTRUCTURE: imported only by tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.

Also holds a small, independent numpy restatement of the byte/integer arithmetic
(`np_q8_dot`, `np_f16_dot`, `np_rmsnorm`) used to cross-check the C code: two
implementations written separately from the same reference lines must agree bit for bit.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liboracle.so")


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "oracle.c")
    if force or not os.path.exists(LIB_PATH) or os.path.getmtime(src) > os.path.getmtime(LIB_PATH):
        subprocess.run(["make", "-C", _HERE, "-B", "liboracle.so"], check=True, capture_output=True)
    return LIB_PATH


class OTensor(C.Structure):
    _fields_ = [("data", C.c_void_p), ("type", C.c_int32), ("pad", C.c_int32)]


class OModel(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("arch", "dim", "hidden", "n_layers", "n_heads", "n_kv_heads", "head_size", "vocab", "ctx")] + \
               [("eps", C.c_float), ("theta", C.c_float), ("lanes", C.c_int32), ("per_row_quant", C.c_int32),
                ("token_embd", OTensor), ("output", OTensor), ("output_norm", OTensor)] + \
               [(n, C.POINTER(OTensor)) for n in ("attn_norm", "wq", "wk", "wv", "wo", "ffn_norm", "w1", "w2", "w3",
                                                  "attn_q_norm", "attn_k_norm")]


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB_PATH)
        vp, i32, f32 = C.c_void_p, C.c_int32, C.c_float
        L.oracle_state_new.argtypes = [C.POINTER(OModel)]
        L.oracle_state_new.restype = vp
        L.oracle_state_free.argtypes = [vp]
        L.oracle_state_reset.argtypes = [C.POINTER(OModel), vp]
        for fn in ("oracle_state_logits", "oracle_state_x", "oracle_state_key_cache", "oracle_state_value_cache"):
            getattr(L, fn).argtypes = [vp]
            getattr(L, fn).restype = C.POINTER(f32)
        L.oracle_forward.argtypes = [C.POINTER(OModel), vp, i32, i32, i32]
        L.oracle_forward.restype = C.POINTER(f32)
        L.oracle_argmax.argtypes = [vp, i32]
        L.oracle_q8_dot_ref.argtypes = [vp, C.c_int64, vp, i32]
        L.oracle_q8_dot_ref.restype = f32
        L.oracle_f16_dot.argtypes = [vp, vp, i32, i32]
        L.oracle_f16_dot.restype = f32
        L.oracle_q8_quantize.argtypes = [vp, i32, vp, vp]
        L.oracle_rmsnorm.argtypes = [vp, vp, C.POINTER(OTensor), i32, f32]
        L.oracle_rope_table.argtypes = [i32, i32, C.c_double, vp, vp]
        L.oracle_bench_tokens.argtypes = [C.c_int64, i32, i32, vp]
        L.oracle_quantize_q8_0.argtypes = [vp, C.c_int64, vp]
        L.oracle_kquant_dequantize.argtypes = [i32, vp, C.c_int64, vp]
        L.oracle_kquant_to_q8_0.argtypes = [i32, vp, C.c_int64, vp]
        L.oracle_f32_to_f16.argtypes = [f32]
        L.oracle_f32_to_f16.restype = C.c_uint16
        L.oracle_f16_to_f32.argtypes = [C.c_uint16]
        L.oracle_f16_to_f32.restype = f32
        L.oracle_f16_to_f32_daz.argtypes = [C.c_uint16]
        L.oracle_f16_to_f32_daz.restype = f32
        L.oracle_omp_threads.restype = i32
        L.oracle_set_threads.argtypes = [i32]
        L.oracle_lxm_seed.argtypes = [vp, C.c_int64]
        L.oracle_lxm_next_int.argtypes = [vp]
        L.oracle_lxm_next_int.restype = C.c_uint32
        L.oracle_lxm_next_float1.argtypes = [vp]
        L.oracle_lxm_next_float1.restype = f32
        L.oracle_sample.argtypes = [vp, i32, f32, f32, f32, vp]
        L.oracle_sample_categorical.argtypes = [vp, i32, f32]
        L.oracle_sample_topp.argtypes = [vp, i32, f32, f32, vp]
        _lib = L
    return _lib


class JavaLXM:
    """RandomGeneratorFactory.getDefault().create(seed) = L32X64MixRandom (Sampler.java:84), restated in oracle.c."""

    def __init__(self, seed: int):
        self._st = (C.c_uint32 * 4)()
        lib().oracle_lxm_seed(self._st, seed)

    def next_int(self) -> int:
        return int(lib().oracle_lxm_next_int(self._st))

    def next_float1(self) -> float:
        return float(lib().oracle_lxm_next_float1(self._st))


def sample(logits: np.ndarray, temperature: float, topp: float, r01: float, want_probs: bool = False):
    """Sampler.selectSampler's lambda on a COPY of the logits (the reference modifies them in place).  want_probs: also return
    that copy, which then holds the float32 probabilities (for temperature > 0)."""
    lg = np.ascontiguousarray(logits, dtype=np.float32).copy()
    idx = np.empty(len(lg), dtype=np.int32)
    tok = int(lib().oracle_sample(lg.ctypes.data, len(lg), temperature, topp, r01, idx.ctypes.data))
    return (tok, lg) if want_probs else tok


def np_sample(logits: np.ndarray, temperature: float, topp: float, r01: float, want_info: bool = False):
    """Second restatement of the same lines in numpy/Python (cross-check of the C code): sequential float32 sums via
    np.add.accumulate for the categorical walk, a statement-by-statement port of the top-p heap.  want_info: return
    (id, candidates n0, tokens kept) -- n, n for the categorical walk, 0, 0 for greedy."""
    lg = np.asarray(logits, dtype=np.float32)
    if temperature == 0.0:
        tok = int(np.argmax(lg))
        return (tok, 0, 0) if want_info else tok
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):  # x may overflow to inf (tiny T): NaN probabilities, as in Java
        x = (lg / np.float32(temperature)).astype(np.float32)
        e = np.exp((x - x.max()).astype(np.float64)).astype(np.float32)
        p = (e / np.add.accumulate(e, dtype=np.float32)[-1]).astype(np.float32)
    n = len(p)
    if topp <= 0 or topp >= 1:
        cdf = np.add.accumulate(p, dtype=np.float32)
        hit = np.flatnonzero(np.float32(r01) < cdf)
        tok = int(hit[0]) if len(hit) else n - 1
        return (tok, n, n) if want_info else tok
    # ToppSampler.sampleFromFloatTensor + processTopP, ported statement by statement (the popped order is NOT a perfect sort:
    # the reference sifts with heap size i - 1, ToppSampler.java:131, so the heap mechanics are part of the result).
    # indices: candidates from the head in index order, rejected ids from the tail (:71-77), so with no candidate the
    # final `return indices[lastIndex]` (:155) gives n - 1.
    cutoff = (np.float32(1.0) - np.float32(topp)) / np.float32(n - 1)
    keep = p >= cutoff
    idx = np.flatnonzero(keep).tolist() + np.flatnonzero(~keep)[::-1].tolist()
    n0 = int(keep.sum())
    pv = p.tolist()  # float32 values widened exactly: the comparisons are unchanged

    def less(x, y):  # comparator.compare(x, y) < 0  <=>  value(x) > value(y)
        return pv[x] > pv[y]

    def sift_down(frm, size):
        prev = frm
        while 2 * prev + 1 < size:
            nxt = 2 * prev + 1
            r = 2 * prev + 2
            if r < size and less(idx[r], idx[nxt]):
                nxt = r
            if less(idx[nxt], idx[prev]):
                idx[prev], idx[nxt] = idx[nxt], idx[prev]
                prev = nxt
            else:
                break

    for i in range(n0 // 2 - 1, -1, -1):
        sift_down(i, n0)
    cum, last = np.float32(0.0), 0
    for i in range(n0 - 1, -1, -1):
        idx[0], idx[i] = idx[i], idx[0]
        cum = np.float32(cum + p[idx[i]])
        if cum > np.float32(topp):
            last = i
            break
        sift_down(0, i - 1)
    r = np.float32(np.float32(r01) * cum)
    cdf = np.float32(0.0)
    tok = int(idx[last])
    for i in range(n0 - 1, last - 1, -1):
        cdf = np.float32(cdf + p[idx[i]])
        if r < cdf:
            tok = int(idx[i])
            break
    return (tok, n0, n0 - last) if want_info else tok


def use_all_cores() -> int:
    """Row-parallel over every host core this process may run on, whatever OMP_NUM_THREADS says (torchrun sets it to 1)."""
    try:
        n = len(os.sched_getaffinity(0))
    except AttributeError:
        n = os.cpu_count() or 1
    try:  # a container's CPU quota (cgroup v2 cpu.max = "<quota> <period>"): more OpenMP threads than that only fight each other
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()
        if quota != "max":
            n = max(1, min(n, int(quota) // int(period)))
    except (OSError, ValueError):
        pass
    lib().oracle_set_threads(n)
    return int(lib().oracle_omp_threads())


def _ot(entry) -> OTensor:
    tt, dims, raw = entry
    t = OTensor()
    t.data = raw.ctypes.data
    t.type = int(tt)
    return t


class OracleModel:
    """Wraps a loader.Model (anything with .configuration and .tensors) for the C oracle."""

    def __init__(self, model, lanes: int = 16, per_row_quant: bool = False):
        c = model.configuration
        self._model = model  # keeps the mmap alive
        m = OModel()
        m.arch, m.dim, m.hidden, m.n_layers = c.arch, c.dim, c.hidden_dim, c.n_layers
        m.n_heads, m.n_kv_heads, m.head_size, m.vocab, m.ctx = c.n_heads, c.n_kv_heads, c.head_size, c.vocab_size, c.context_length
        m.eps, m.theta, m.lanes, m.per_row_quant = c.rms_norm_eps, c.rope_theta, lanes, int(per_row_quant)
        T = model.tensors
        m.token_embd = _ot(T["token_embd.weight"])
        if "output.weight" in T:
            m.output = _ot(T["output.weight"])
        m.output_norm = _ot(T["output_norm.weight"])
        self._arrays = {}

        def arr(fmt):
            a = (OTensor * c.n_layers)(*[_ot(T[fmt.format(i)]) for i in range(c.n_layers)])
            self._arrays[fmt] = a
            return a

        def rows_of(fmt, key, row0, rows, cols):
            """Rows [row0, row0 + rows) of a fused tensor as tensors of their own (Phi-3: wqkv.matmul + copyTo, wGateUp.matmul + copyChunk)."""
            out = []
            for i in range(c.n_layers):
                tt, dims, raw = T[fmt.format(i)]
                rb = {0: cols * 4, 1: cols * 2, 8: cols // 32 * 34}[int(tt)]
                raw = np.asarray(raw).reshape(-1)
                out.append(_ot((tt, (cols, rows), raw[row0 * rb:(row0 + rows) * rb])))
            a = (OTensor * c.n_layers)(*out)
            self._arrays[key] = a
            return a

        m.attn_norm = arr("blk.{}.attn_norm.weight")
        if c.arch == 2:  # Phi-3: fused attn_qkv ([q; k; v] rows) and ffn_up ([gate; up] rows), InferenceCore.java:718-724,779-781
            qd, kvd = c.n_heads * c.head_size, c.n_kv_heads * c.head_size
            m.wq = rows_of("blk.{}.attn_qkv.weight", "q", 0, qd, c.dim)
            m.wk = rows_of("blk.{}.attn_qkv.weight", "k", qd, kvd, c.dim)
            m.wv = rows_of("blk.{}.attn_qkv.weight", "v", qd + kvd, kvd, c.dim)
            m.w1 = rows_of("blk.{}.ffn_up.weight", "g", 0, c.hidden_dim, c.dim)
            m.w3 = rows_of("blk.{}.ffn_up.weight", "u", c.hidden_dim, c.hidden_dim, c.dim)
            m.w2 = arr("blk.{}.ffn_down.weight")
        else:
            m.wq, m.wk, m.wv = arr("blk.{}.attn_q.weight"), arr("blk.{}.attn_k.weight"), arr("blk.{}.attn_v.weight")
            m.w1, m.w2, m.w3 = arr("blk.{}.ffn_gate.weight"), arr("blk.{}.ffn_down.weight"), arr("blk.{}.ffn_up.weight")
        m.wo = arr("blk.{}.attn_output.weight")
        m.ffn_norm = arr("blk.{}.ffn_norm.weight")
        if c.arch == 1:
            m.attn_q_norm, m.attn_k_norm = arr("blk.{}.attn_q_norm.weight"), arr("blk.{}.attn_k_norm.weight")
        self.m = m
        self.cfg = c
        self.state = lib().oracle_state_new(C.byref(m))

    def forward(self, token: int, pos: int, want_logits: bool = True):
        p = lib().oracle_forward(C.byref(self.m), self.state, token, pos, int(want_logits))
        if not want_logits:
            return None
        return np.ctypeslib.as_array(p, shape=(self.cfg.vocab_size,)).copy()

    def forward_argmax(self, token: int, pos: int) -> int:
        lg = self.forward(token, pos)
        return argmax(lg)

    def reset(self):
        lib().oracle_state_reset(C.byref(self.m), self.state)

    def key_cache(self, layer: int) -> np.ndarray:
        n = self.cfg.context_length * self.cfg.kv_dim
        p = lib().oracle_state_key_cache(self.state)
        return np.ctypeslib.as_array(p, shape=(self.cfg.n_layers * n,))[layer * n:(layer + 1) * n].copy()

    def value_cache(self, layer: int) -> np.ndarray:
        n = self.cfg.context_length * self.cfg.kv_dim
        p = lib().oracle_state_value_cache(self.state)
        return np.ctypeslib.as_array(p, shape=(self.cfg.n_layers * n,))[layer * n:(layer + 1) * n].copy()

    def x(self) -> np.ndarray:
        return np.ctypeslib.as_array(lib().oracle_state_x(self.state), shape=(self.cfg.dim,)).copy()

    def close(self):
        if self.state:
            lib().oracle_state_free(self.state)
            self.state = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def argmax(v: np.ndarray) -> int:
    v = np.ascontiguousarray(v, dtype=np.float32)
    return int(lib().oracle_argmax(v.ctypes.data, len(v)))


def bench_tokens(vocab: int, n: int, seed: int = 42) -> np.ndarray:
    """``new Random(42).nextInt(vocab)`` stream of LlamaBench.java:188-193."""
    out = np.empty(n, dtype=np.int32)
    lib().oracle_bench_tokens(seed, vocab, n, out.ctypes.data)
    return out


def q8_dot(raw: np.ndarray, row_off_elems: int, x: np.ndarray) -> float:
    x = np.ascontiguousarray(x, dtype=np.float32)
    return float(lib().oracle_q8_dot_ref(raw.ctypes.data, row_off_elems, x.ctypes.data, len(x)))


def f16_dot(w: np.ndarray, x: np.ndarray, lanes: int) -> float:
    w = np.ascontiguousarray(w, dtype=np.uint16)
    x = np.ascontiguousarray(x, dtype=np.float32)
    return float(lib().oracle_f16_dot(w.ctypes.data, x.ctypes.data, len(x), lanes))


def q8_quantize(x: np.ndarray):
    x = np.ascontiguousarray(x, dtype=np.float32)
    aq = np.empty(len(x), dtype=np.int8)
    sc = np.empty(len(x) // 32, dtype=np.float32)
    lib().oracle_q8_quantize(x.ctypes.data, len(x), aq.ctypes.data, sc.ctypes.data)
    return aq, sc


KQUANT_BLOCK_BYTES = {12: 144, 13: 176, 14: 210}  # Q4_K, Q5_K, Q6_K (tensor/GGMLType.java:18-20)


def kquant_dequantize(ggml_type: int, raw: np.ndarray, n: int) -> np.ndarray:
    """getFloat(i) of Q4_K/Q5_K/Q6_KFloatTensor for i in [0, n) (C restatement)."""
    raw = np.ascontiguousarray(raw, dtype=np.uint8)
    assert raw.size >= n // 256 * KQUANT_BLOCK_BYTES[ggml_type]
    out = np.empty(n, dtype=np.float32)
    lib().oracle_kquant_dequantize(ggml_type, raw.ctypes.data, n, out.ctypes.data)
    return out


def kquant_to_q8_0(ggml_type: int, raw: np.ndarray, n: int) -> np.ndarray:
    """ModelLoader.dequantizeToQ8_0TornadoTensor (ModelLoader.java:173-224): the Q8_0 bytes the reference's accelerator path computes with."""
    raw = np.ascontiguousarray(raw, dtype=np.uint8)
    out = np.empty((n + 31) // 32 * 34, dtype=np.uint8)
    lib().oracle_kquant_to_q8_0(ggml_type, raw.ctypes.data, n, out.ctypes.data)
    return out


def np_requant_q8_0(x: np.ndarray) -> np.ndarray:
    """Second restatement (numpy, vectorised) of the re-quantiser applied to already dequantised floats: ModelLoader.java:184-212."""
    x = np.ascontiguousarray(x, dtype=np.float32).reshape(-1, 32)
    max_abs = np.max(np.abs(x), axis=1)
    scale = (max_abs / np.float32(127.0)).astype(np.float32)
    with np.errstate(divide="ignore"):
        inv = np.where(scale != 0, (np.float32(1.0) / scale).astype(np.float32), np.float32(0.0)).astype(np.float32)
    t = (x * inv[:, None]).astype(np.float32)
    f = np.floor(t)
    q = f.astype(np.int64) + ((t - f) >= np.float32(0.5))  # Math.round(float): ties towards +infinity
    q = np.clip(q, -128, 127).astype(np.int8)
    out = np.empty((x.shape[0], 34), dtype=np.uint8)
    out[:, :2] = scale.astype(np.float16).view(np.uint8).reshape(-1, 2)  # Float.floatToFloat16: round to nearest even
    out[:, 2:] = q.view(np.uint8)
    return out.reshape(-1)


def rope_table(ctx: int, head_size: int, theta: float):
    cr = np.empty(ctx * head_size // 2, dtype=np.float32)
    ci = np.empty_like(cr)
    lib().oracle_rope_table(ctx, head_size, float(theta), cr.ctypes.data, ci.ctypes.data)
    return cr, ci


# --------------------------------------------------------------------------------------------
# Independent numpy restatement (cross-check of oracle.c; float32 scalars, no FMA by construction)
# --------------------------------------------------------------------------------------------
f32 = np.float32


def np_q8_quantize_block(x: np.ndarray):
    """Q8_0FloatTensor.java:100-117 for one 32-block."""
    amax = f32(0)
    for v in x:
        av = f32(abs(v))
        if av > amax:
            amax = av
    qs = f32(amax / f32(127))
    ascale = f32(np.float16(qs))  # floatToFloat16 (RNE) then float16ToFloat
    ainv = f32(f32(1) / qs) if qs != 0 else f32(0)
    aq = np.empty(32, dtype=np.int64)
    for i, v in enumerate(x):
        s = f32(v * ainv)
        aq[i] = int(f32(s + f32(np.copysign(f32(0.5), s))))  # (int) truncates
    return aq, ascale


def np_q8_dot(raw: np.ndarray, row_off_elems: int, x: np.ndarray) -> np.float32:
    """Q8_0FloatTensor.dotQ8Activation, Q8_0FloatTensor.java:90-123."""
    x = np.asarray(x, dtype=np.float32)
    result = f32(0)
    for b in range(len(x) // 32):
        off = (row_off_elems + b * 32) // 32 * 34
        ws = f32(raw[off:off + 2].view(np.float16)[0])
        wq = raw[off + 2:off + 34].view(np.int8).astype(np.int64)
        aq, ascale = np_q8_quantize_block(x[b * 32:(b + 1) * 32])
        isum = int((aq * wq).sum())
        result = f32(result + f32(f32(isum) * f32(ws * ascale)))
    return result


def np_f16_daz(bits: np.ndarray) -> np.ndarray:
    b = bits.astype(np.uint32)
    mask = np.where((b & 0x7C00) != 0, np.uint32(0xFFFFFFFF), np.uint32(0))
    out = ((b & 0x8000) << 16) | ((((b & 0x7FFF) + 0x1C000) << 13) & mask)
    return out.astype(np.uint32).view(np.float32)


def np_f16_dot(wbits: np.ndarray, x: np.ndarray, lanes: int) -> np.float32:
    """FP16FloatTensor.vectorDot, FP16FloatTensor.java:62-110 (fma emulated in float64:
    a float32 product is exact in float64, one rounding at the end == fused)."""
    x = np.asarray(x, dtype=np.float32)
    n = len(x)
    if lanes <= 0:
        r = f32(0)
        w = wbits.view(np.float16).astype(np.float32)
        for j in range(n):
            r = f32(r + f32(w[j] * x[j]))
        return r
    w = np_f16_daz(wbits)
    acc = np.zeros(lanes, dtype=np.float32)
    upper = n - n % lanes
    for i in range(0, upper, lanes):
        prod = w[i:i + lanes].astype(np.float64) * x[i:i + lanes].astype(np.float64) + acc.astype(np.float64)
        acc = prod.astype(np.float32)
    r = f32(0)
    for l in range(lanes):
        r = f32(r + acc[l])
    wt = wbits.view(np.float16).astype(np.float32)
    for j in range(upper, n):
        r = f32(r + f32(wt[j] * x[j]))
    return r


def np_rmsnorm(x: np.ndarray, w: np.ndarray, eps: float) -> np.ndarray:
    """InferenceCore.rmsnorm, InferenceCore.java:39-48."""
    x = np.asarray(x, dtype=np.float32)
    ss = f32(0)
    for v in x:
        ss = f32(ss + f32(v * v))
    ss = f32(ss / f32(len(x)))
    ss = f32(ss + f32(eps))
    ss = f32(1.0 / np.sqrt(np.float64(ss)))
    return (w.astype(np.float32) * (ss * x).astype(np.float32)).astype(np.float32)


class JavaRandom:
    """java.util.Random, independent Python restatement (cross-check of the C LCG)."""

    def __init__(self, seed: int):
        self.seed = (seed ^ 0x5DEECE66D) & ((1 << 48) - 1)

    def next(self, bits: int) -> int:
        self.seed = (self.seed * 0x5DEECE66D + 0xB) & ((1 << 48) - 1)
        v = self.seed >> (48 - bits)  # (int)(seed >>> (48 - bits)): wraps only when bits == 32
        if v >= 1 << 31:
            v -= 1 << 32
        return v

    def next_int(self, bound: int | None = None) -> int:
        if bound is None:
            return self.next(32)
        r = self.next(31)
        m = bound - 1
        if bound & m == 0:
            return (bound * r) >> 31
        u = r
        while True:
            r = u % bound
            t = u - r + m
            if t >= 1 << 31:  # int overflow -> negative in Java
                u = self.next(31)
                continue
            return r
