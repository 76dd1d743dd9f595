"""Host-side mirror of the reference's benchmark harness ``bench/LlamaBench.java``:
llama-bench style ``pp N`` / ``tg N`` tests over a deterministic synthetic token stream
(``new Random(42).nextInt(vocab)``, LlamaBench.java:188-193), forward pass only, one untimed
warm-up repetition then ``-r`` timed ones, avg +- sample stddev (LlamaBench.java:200-254).
"""
from __future__ import annotations

import math
import time
from dataclasses import dataclass, field


class JavaRandom:
    """java.util.Random (48-bit LCG); only what LlamaBench uses."""

    def __init__(self, seed: int):
        self.seed = (seed ^ 0x5DEECE66D) & ((1 << 48) - 1)

    def _next(self, bits: int) -> int:
        self.seed = (self.seed * 0x5DEECE66D + 0xB) & ((1 << 48) - 1)
        v = self.seed >> (48 - bits)
        return v - (1 << 32) if v >= (1 << 31) else v

    def next_int(self, bound: int) -> int:
        r = self._next(31)
        m = bound - 1
        if bound & m == 0:
            return (bound * r) >> 31
        u = r
        while u - (u % bound) + m >= (1 << 31):  # Java int overflow -> retry
            u = self._next(31)
        return u % bound


def synthetic_tokens(vocab: int, n: int, seed: int = 42) -> list[int]:
    rng = JavaRandom(seed)
    return [rng.next_int(vocab) for _ in range(n)]


@dataclass
class TestSpec:
    """``pp<N>`` (prompt processing), ``tg<N>`` (generation) or ``pp<N>+tg<M>`` at ``depth``."""
    n_prompt: int
    n_gen: int
    depth: int = 0

    @property
    def tokens(self):
        return self.n_prompt + self.n_gen

    @property
    def name(self):
        if self.n_prompt and self.n_gen:
            base = f"pp{self.n_prompt}+tg{self.n_gen}"
        else:
            base = f"pp{self.n_prompt}" if self.n_prompt else f"tg{self.n_gen}"
        return base + (f" @ d{self.depth}" if self.depth else "")


@dataclass
class Result:
    test: str
    avg_ts: float
    stddev_ts: float
    samples: list = field(default_factory=list)


def _prefill(plan, toks, start: int, count: int, batch: int):
    """LlamaBench.prefill (LlamaBench.java:257-273)."""
    if count <= 0:
        return
    if batch > 1:
        for off in range(0, count, batch):
            n = min(batch, count - off)
            plan.forward_batch_prefill(toks[start + off:start + off + n], start + off)
    else:
        plan.decode_sequence(toks[start:start + count], count, start)


def run_test(plan, toks, t: TestSpec, batch: int) -> float:
    """One timed repetition (LlamaBench.runTest, LlamaBench.java:234-254): untimed depth prefill,
    then nPrompt prompt tokens (batched when batch > 1) and nGen single-token decodes."""
    _prefill(plan, toks, 0, t.depth, batch)
    base = t.depth
    t0 = time.perf_counter()
    _prefill(plan, toks, base, t.n_prompt, batch)
    if t.n_gen:
        plan.decode_sequence(toks[base + t.n_prompt:base + t.n_prompt + t.n_gen], t.n_gen, base + t.n_prompt)
    t1 = time.perf_counter()
    return t.tokens / (t1 - t0)


def bench_model(plan, vocab: int, tests: list[TestSpec], reps: int = 5, warmup: bool = True, batch: int = 1) -> list[Result]:
    max_tokens = max(t.depth + t.tokens for t in tests)
    toks = synthetic_tokens(vocab, max_tokens)
    out = []
    for t in tests:
        if warmup:
            run_test(plan, toks, t, batch)
        samples = [run_test(plan, toks, t, batch) for _ in range(reps)]
        avg = sum(samples) / len(samples)
        var = sum((s - avg) ** 2 for s in samples)
        sd = math.sqrt(var / (len(samples) - 1)) if len(samples) > 1 else 0.0
        out.append(Result(t.name + (f" b{batch}" if batch > 1 else ""), avg, sd, samples))
    return out


def to_markdown(results: list[Result], model: str, quant: str, backend: str = "H100 sm_90a") -> str:
    lines = ["| model | quant | backend | test | t/s |", "| --- | --- | --- | ---: | ---: |"]
    for r in results:
        lines.append(f"| {model} | {quant} | {backend} | {r.test} | {r.avg_ts:.2f} ± {r.stddev_ts:.2f} |")
    return "\n".join(lines)
