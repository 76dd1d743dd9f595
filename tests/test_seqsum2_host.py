"""CPU model of the exact sequential sum (tools/seqsum2/emulate_v2.py, the thread-accurate emulation of
csrc/seqsum2.cuh::block_seqsum_exact_v2_t) against the literal float32 loop, on sums whose chunk boundaries and exact ties sit right
at binade edges.  With the predictor's margin forced below zero, runs are predicted across binade edges on purpose: the resolver's
checks must catch every such run and replay it, so the result still matches bit for bit."""
import importlib.util
import os

import numpy as np
import pytest

_PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "seqsum2", "emulate_v2.py")
_spec = importlib.util.spec_from_file_location("seqsum2_emulate_v2", _PATH)
em = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(em)


def _stride(E):
    return E + 4 if E % 4 == 0 and (E // 4) % 2 == 0 else E


def _edge_cases(n, T, rng):
    """Sums that reach a power of two exactly at chunk boundaries and inside chunks, with exact half-ulp ties next to the edges."""
    E = (n + T - 1) // T
    out = []
    out.append(np.full(n, 1.0 / E, np.float32))                          # thread t ends at exactly t + 1: every power of two on a boundary
    out.append(np.full(n, 1.0 / (E - 2 if E > 2 else 1), np.float32))    # edges inside the chunks
    t = np.ones(n, np.float32)                                            # integers: then ties of half an ulp wherever the sum reaches 2^24
    t[::7] = 0.5
    out.append(t)
    k = np.arange(n)
    ties = np.where(k % 3 == 0, 2.0 ** -24, 1.0).astype(np.float32)      # 2^-24 is half an ulp of sums in [1, 2): a tie right after each edge
    out.append(ties)
    x = rng.standard_normal(n).astype(np.float32)
    out.append((x * x).astype(np.float32))                               # RMSNorm-like squares
    g = np.ones(n, np.float32)                                            # a binade edge in every chunk of one warp: the sum doubles per chunk
    for j in range(1, min(T, 40)):
        g[j * E:(j + 1) * E] = np.float32(2.0 ** j / E)
    out.append(g)
    return out


def _check(T, n, m, rng):
    E = (n + T - 1) // T
    fallbacks = 0
    for t in _edge_cases(n, T, rng):
        with np.errstate(all="ignore"):
            ref = np.add.accumulate(t, dtype=np.float32)[-1]
        got, items, fb, lits = em.v2(t, T, _stride(E)) if m is None else em.v2(t, T, _stride(E), m=m)
        assert np.float32(got).view(np.uint32) == np.float32(ref).view(np.uint32), (T, n, m, got, ref, items, fb)
        assert 1 <= items and lits <= items
        fallbacks += fb
    return fallbacks


@pytest.mark.parametrize("T", [256, 512, 1024])
@pytest.mark.parametrize("n", [2048, 4096, 5120])
def test_edge_cases_exact_at_the_margin(T, n):
    """The margin the kernel uses: bit-exact, and no run is mispredicted."""
    assert _check(T, n, None, np.random.default_rng(n + T)) == 0


@pytest.mark.parametrize("T", [256, 512, 1024])
def test_edge_cases_exact_with_wrong_predictions(T):
    """A negative margin puts runs across binade edges: the resolver's checks reject them and the replays keep the sum exact."""
    assert sum(_check(T, n, -2.0 ** -8, np.random.default_rng(n + T)) for n in (2048, 4096, 5120)) > 0


def test_adversarial_corpus_at_16384():
    """The adversarial kinds of emulate_v2.py at the largest dim, one thread count each."""
    rng = np.random.default_rng(1)
    for T, t in zip((256, 512, 1024) * 4, em.adversarial(16384, rng)):
        E = (len(t) + T - 1) // T
        with np.errstate(all="ignore"):
            ref = np.add.accumulate(t, dtype=np.float32)[-1]
        got = em.v2(t, T, _stride(E))[0]
        assert np.float32(got).view(np.uint32) == np.float32(ref).view(np.uint32) or (np.isnan(got) and np.isnan(ref)), (T, got, ref)
