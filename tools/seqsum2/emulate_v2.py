"""Thread-accurate Python emulation of csrc/seqsum2.cuh::block_seqsum_exact_v2_t (T threads, warp shuffles with CUDA semantics)
against the literal float32 loop.  Without an argument: adversarial cases (ties, binade crossings, zeros, denormals, inf terms) at
n = 2048 / 4096 / 5120 / 8192 / 16384 and T = 256 / 512 / 1024 in the fused norm's chunk layout; with T: the exact inputs of
tests/test_gpu_parity.py::test_exact_parallel_sequential_sum at T threads.
Usage: python tools/seqsum2/emulate_v2.py [T]"""
import sys

import numpy as np

F = np.float32
LITERAL = -(2 ** 31)


def f32_exponent(f):
    return int((np.float32(f).view(np.uint32) >> 23) & 0xFF) - 127


def seq_pair(t, e):
    """csrc/seqsum2.cuh::seq_pair with scale = 2^(23-e): t * scale is exact, so the fused multiply-add's single rounding is
    the float64 sum rounded to float32."""
    t = F(t)
    scale = np.uint32((150 - e) << 23).view(F)
    with np.errstate(all="ignore"):
        kf = F(t * scale)
        r = F(np.float64(t) * np.float64(scale) + 2.0 ** 23)
        a0 = int(r.view(np.uint32)) - 0x4B000000
        d = F(F(r - F(2.0 ** 23)) - kf)
    a1 = (a0 - 1 if d > 0 else a0 + 1) if abs(d) == F(0.5) else a0
    return bool(kf < F(2.0 ** 23)), (a0, a1)


def compose(L, R):
    a0 = L[0] + (R[1] if (L[0] & 1) else R[0])
    a1 = L[1] + (R[1] if ((1 + L[1]) & 1) else R[0])
    return (min(a0, 1 << 26), min(a1, 1 << 26))


def warp_segscan(ps, fs):
    """ps, fs: lists of 32 (pair, flag); CUDA __shfl_up semantics (lane < d keeps its own value)."""
    ps, fs = list(ps), list(fs)
    d = 1
    while d < 32:
        ups = [ps[l - d] if l >= d else ps[l] for l in range(32)]
        ufs = [fs[l - d] if l >= d else fs[l] for l in range(32)]
        for l in range(32):
            if l >= d and not fs[l]:
                ps[l] = compose(ups[l], ps[l])
                fs[l] = ufs[l]
        d <<= 1
    return ps, fs


def v2(terms, T, S=None, m=2.0 ** -9):
    """Returns (sum, items walked, fallbacks, literal items).  m overrides the predictor's margin (0 or below: predictions that
    are wrong on purpose next to binade edges, which the resolver must catch)."""
    n = len(terms)
    E = (n + T - 1) // T
    S = E if S is None else S
    sq = np.zeros(T * S, dtype=F)
    for t in range(T):
        chunk = terms[t * E:(t + 1) * E]
        sq[t * S:t * S + len(chunk)] = chunk
    NW = T // 32
    loc = np.zeros(T, dtype=F)
    for t in range(T):
        s = F(0)
        for k in range(E):
            s = F(s + sq[t * S + k])
        loc[t] = s
    inc = loc.copy()
    for w in range(NW):
        v = inc[w * 32:(w + 1) * 32].copy()
        d = 1
        while d < 32:
            u = np.concatenate([v[:d], v[:-d]])
            for l in range(32):
                if l >= d:
                    v[l] = F(v[l] + u[l])
            d <<= 1
        inc[w * 32:(w + 1) * 32] = v
    wsum = [inc[w * 32 + 31] for w in range(NW)]
    # barrier 1; every warp: lane l holds wsum[l] if l < warp, then an xor butterfly (__shfl_xor_sync)
    wex = np.zeros(NW, dtype=F)
    for w in range(NW):
        v = np.array([wsum[l] if l < w else F(0) for l in range(32)], dtype=F)
        d = 16
        while d > 0:
            v = np.array([F(v[l] + v[l ^ d]) for l in range(32)], dtype=F)
            d >>= 1
        wex[w] = v[0]
    cls = [LITERAL] * T
    pr = [(0, 0)] * T
    for t in range(T):
        w = t >> 5
        p_end = F(wex[w] + inc[t])
        p_start = F(wex[w] + F(inc[t] - loc[t]))
        e = f32_exponent(p_start)
        if p_start > 0 and e > -100 and e < 128 and f32_exponent(p_end) == e:
            b = np.uint32((e + 127) << 23).view(F) if 0 <= e + 127 < 256 else F(np.inf)
            with np.errstate(all="ignore"):
                lo = F(b * F(1.0 + m))
                hi = F(F(2.0) * b) * F(1.0 - m)
            if p_start >= lo and p_end <= F(hi):
                ok, p = True, (0, 0)
                for k in range(E):
                    o, q = seq_pair(sq[t * S + k], e)
                    if not o:
                        ok = False
                        break
                    p = compose(p, q)
                if ok:
                    cls[t] = e
                    pr[t] = p
    # per warp: runs cut at the warp's edges, segmented scan, ballot compaction into slots [32 w, 32 w + count)
    items = [None] * T
    for w in range(NW):
        lo_t = w * 32
        f = [0] * 32
        isitem = [False] * 32
        for l in range(32):
            t = lo_t + l
            clean = cls[t] != LITERAL
            f[l] = 0 if (clean and l > 0 and cls[t - 1] == cls[t]) else 1
            isitem[l] = (not clean) or l == 31 or cls[t + 1] != cls[t]
        starts = [l for l in range(32) if f[l]]
        bal = [l for l in range(32) if isitem[l]]
        ps, _ = warp_segscan(pr[lo_t:lo_t + 32], f)
        for rank, l in enumerate(bal):
            first = lo_t + max(x for x in starts if x <= l)
            nxt = lo_t + rank + 1 if rank + 1 < len(bal) else lo_t + 32
            items[lo_t + rank] = (cls[lo_t + l], ps[l], first, lo_t + l, nxt)
    # barrier 2; the resolver (warp 0): runs step the float's bits, literal threads and mispredictions replay their terms
    sb = 0
    n_items = fallbacks = literals = 0
    i = 0
    with np.errstate(all="ignore"):
        while i < T:
            c, p, first, last, i = items[i]
            n_items += 1
            ebits = c + 127 if c != LITERAL else 0xFFFFFFFF
            nb = sb + (p[1] if (sb & 1) else p[0])
            if (sb >> 23) == ebits and (nb >> 23) == ebits:
                sb = nb
                continue
            fallbacks += c != LITERAL
            literals += c == LITERAL
            s = np.uint32(sb).view(F)
            for j in range(first, last + 1):
                for k in range(E):
                    s = F(s + sq[j * S + k])
            sb = int(np.float32(s).view(np.uint32))
    s = np.uint32(sb).view(F)
    return s, n_items, fallbacks, literals


def cases():
    rng = np.random.default_rng(0)
    out = []
    for trial in range(120):
        n = int(rng.choice([33, 64, 256, 1000, 1536, 2560, 4096, 8192]))
        kind = trial % 10
        if kind == 0: x = rng.standard_normal(n)
        elif kind == 1: x = rng.standard_normal(n) * 10.0 ** rng.integers(-6, 6)
        elif kind == 2: x = rng.standard_cauchy(n)
        elif kind == 3: x = np.full(n, rng.standard_normal())
        elif kind == 4: x = 2.0 ** rng.integers(-10, 10, n)
        elif kind == 5:
            x = rng.standard_normal(n); x[rng.integers(0, n, n // 4)] = 0
        elif kind == 6: x = rng.standard_normal(n) * np.exp(rng.standard_normal(n) * 3)
        elif kind == 7: x = np.round(rng.standard_normal(n) * 8) / 8
        elif kind == 8:
            x = np.zeros(n); x[n // 2:] = rng.standard_normal(n - n // 2)
        else:
            x = rng.standard_normal(n) * 1e-3; x[rng.integers(min(40, n - 1), n)] = 1e3
        out.append((x.astype(np.float32) ** 2).astype(np.float32))
    for n in (512, 4096):
        for eps in (-3e-7, -1e-7, 0.0, 1e-7, 3e-7):
            t = np.full(n, (1.0 + eps) / n, dtype=np.float64).astype(np.float32)
            out.append(t)
            out.append(np.concatenate([t, t]).astype(np.float32)[: min(2 * n, 8192)])
    out.append((4.0 ** (np.arange(300) % 150 - 75)).astype(np.float32))
    out.append(np.array([1.0] * 40 + [np.inf] + [1.0] * 40, dtype=np.float32))
    return out


def adversarial(n, rng):
    """Ties, binade crossings, sums parked next to a power of two, zeros, denormals, huge dynamic range and inf terms at n."""
    out = []
    x = rng.standard_normal(n)
    out.append(x)                                                  # RMSNorm-like squares
    out.append(np.round(x * 8) / 8)                                # few mantissa bits: exact ties on every binade
    out.append(2.0 ** rng.integers(-12, 12, n))                    # powers of two: ties and binade crossings
    z = x.copy(); z[rng.integers(0, n, n // 2)] = 0; out.append(z)  # zeros
    d = x * 1e-3; d[rng.integers(0, n, n // 4)] = 1e-22; out.append(d)  # squares 1e-44: denormal terms
    out.append(x * np.exp(rng.standard_normal(n) * 4))            # huge dynamic range
    i = x.copy(); i[n // 3] = 1e30; out.append(i)                  # 1e60 overflows: an inf term
    sq = [(v.astype(np.float32) ** 2).astype(np.float32) for v in out]
    for eps in (-3e-7, 0.0, 3e-7):                                 # the sum parked next to 1.0
        sq.append(np.full(n, (1.0 + eps) / n, dtype=np.float64).astype(np.float32))
    return sq


if __name__ == "__main__":
    # default: the adversarial cases at the widths of the decode norms, in the fused norm's chunk layout (seqsum2_stride);
    # with a thread count argument: the inputs of test_gpu_parity.py in the contiguous layout at that thread count
    def stride(E):
        return E + 4 if E % 4 == 0 and (E // 4) % 2 == 0 else E
    if len(sys.argv) > 1:
        runs = [(int(sys.argv[1]), t, False) for t in cases()]
    else:
        rng = np.random.default_rng(1)
        runs = [(T, t, True) for n in (2048, 4096, 5120, 8192, 16384) for t in adversarial(n, rng) for T in (256, 512, 1024)]
    bad = 0
    for i, (T, t, strided) in enumerate(runs):
        with np.errstate(all="ignore"):
            ref = np.add.accumulate(t, dtype=np.float32)[-1]
        E = (len(t) + T - 1) // T
        got, items, fb, _ = v2(t, T, stride(E) if strided else E)
        same = np.float32(got).view(np.uint32) == np.float32(ref).view(np.uint32) or (np.isnan(got) and np.isnan(ref))
        if not same:
            bad += 1
            print(f"case {i}: T={T} n={len(t)} got={got!r} ref={ref!r} items={items} fallbacks={fb}")
    print(f"{len(runs)} sums: {bad} mismatches")
