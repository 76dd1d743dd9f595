#!/usr/bin/env python
"""Chunked admission (ContinuousBatcher with chunk_rows > 0: prompt rows and decode rows share b200_forward_chunk on the tensor cores)
against exact admission (every step b200_forward_step), on the synthetic Llama-3-8B Q8_0 model of tools/continuous_bench.py with
prefill_batch_size 512, 8 decode slots and the tensor_core_exact prefill mode, alternated on the same plan.

    python tools/chunk_admission_bench.py [--requests 16] [--rounds 2] [--parity 2] [--seed 5] [--every 6]

The trace: prompt lengths 128-1024, generation budgets 64-128, request i arriving before step `every` * i of the scheduler.  As in
continuous_bench.py, max_tokens is the context and a request starts at CTX - len(prompt) - budget, so the Llama loop generates exactly
`budget` tokens.  Runs, in every round: (a) exact admission (chunk_rows = 0); (b) chunked admission at chunk_rows 128 and 256
(min_chunk_rows 32).  Prints one JSON line: per run the wall time, generated and prompt tok/s, time to first token and completion
time (median / p90, seconds from submission), and per step kind ("step" / "chunk") the count, median rows and median host / device
milliseconds per call; the parity gate (every request's ids equal across all runs, and the first --parity requests equal
generate_tokens_llama alone on the plan's own cache); and the GPU name and power limit from one read-only nvidia-smi query."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402
from continuous_bench import gpu_info, pct  # noqa: E402

CTX = 1160
SLOTS = 8
BATCH = 512


def trace(n: int, vocab: int, seed: int, every: int):
    rng = np.random.default_rng(seed)
    reqs, budgets = [], []
    for _ in range(n):
        k, b = int(rng.integers(128, 1025)), int(rng.integers(64, 129))
        reqs.append((int(rng.integers(vocab)), CTX - k - b, [int(t) for t in rng.integers(0, vocab, k)]))
        budgets.append(b)
    return reqs, budgets, [every * i for i in range(n)]


class Recorder:
    """The plan with every forward_step / forward_chunk call timed: host milliseconds around the call (it ends in a synchronise)
    and the device milliseconds b200_batch_info reports for it."""

    def __init__(self, plan):
        self._plan, self.calls = plan, []

    def __getattr__(self, name):
        return getattr(self._plan, name)

    def _timed(self, kind, fn, rows):
        t0 = time.perf_counter()
        out = fn(rows)
        self.calls.append((kind, len(rows), (time.perf_counter() - t0) * 1e3, self._plan.batch_info()[2]))
        return out

    def forward_step(self, rows, logits=False):
        return self._timed("step", self._plan.forward_step, rows)

    def forward_chunk(self, rows, logits=False):
        return self._timed("chunk", self._plan.forward_chunk, rows)


def run(pkg, plan, reqs, arrivals, chunk_rows):
    rec = Recorder(plan)
    stats = {}
    t0 = time.perf_counter()
    ids = pkg.engine.generate_tokens_continuous(rec, "LLAMA_3", reqs, arrivals, [], CTX, CTX, stats=stats, chunk_rows=chunk_rows)
    wall = time.perf_counter() - t0
    gen = sum(len(x) for x in ids)
    ttft = [f - s for f, s in zip(stats["first_token"], stats["submitted"])]
    done = [d - s for d, s in zip(stats["done"], stats["submitted"])]
    kinds = {}
    for kind in ("step", "chunk"):
        c = [x for x in rec.calls if x[0] == kind]
        kinds[kind] = {"calls": len(c), "median_rows": pct([x[1] for x in c], 50), "median_host_ms": pct([x[2] for x in c], 50),
                       "median_device_ms": pct([x[3] for x in c], 50)}
    return ids, {"chunk_rows": chunk_rows, "wall_s": wall, "generated": gen, "generated_tok_s": gen / wall,
                 "prompt_tok_s": sum(len(r[2]) for r in reqs) / wall, "ttft_s": {"median": pct(ttft, 50), "p90": pct(ttft, 90)},
                 "done_s": {"median": pct(done, 50), "p90": pct(done, 90)}, "steps": kinds}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--parity", type=int, default=2)
    ap.add_argument("--seed", type=int, default=5)
    ap.add_argument("--every", type=int, default=6)
    args = ap.parse_args()
    import torch

    pkg = ge.import_package()
    info = gpu_info()
    sh = pkg.synth.SHAPES["llama-3-8b"]
    Q8 = pkg.gguf.GGMLType.Q8_0
    model = pkg.loader.model_from_tensors(sh, Q8, pkg.synth.build_tensors_fast(sh, Q8, seed=1234, device="cuda:0"), CTX)
    plan = pkg.B200MasterPlan.initialize_plan(model, prefill_batch_size=BATCH)
    plan.set_prefill_mode("tensor_core_exact")
    plan.set_decode_slots(SLOTS)
    reqs, budgets, arrivals = trace(args.requests, sh.vocab, args.seed, args.every)
    out = {"metric": "llama-3-8b_q8_0_chunked_admission", "workload": f"llama-3-8b-shaped synthetic Q8_0, {sh.n_layers} layers", **info,
           "torch_device": torch.cuda.get_device_name(0), "requests": args.requests, "slots": SLOTS, "context": CTX,
           "prefill_batch_size": BATCH, "prompt_tokens": sum(len(r[2]) for r in reqs), "budget_tokens": sum(budgets),
           "arrival_every_steps": args.every, "min_chunk_rows": 32}

    # warm-up: the step graphs and the chunk path on a short trace of every configuration
    short = [(t, CTX - 200, p[:150]) for t, _, p in reqs[:SLOTS]]
    for chunk_rows in (0, 128, 256):
        pkg.engine.generate_tokens_continuous(plan, "LLAMA_3", short, [0] * len(short), [], CTX, CTX, chunk_rows=chunk_rows)

    configs = (0, 128, 256)
    runs = {str(c): [] for c in configs}
    ids = {}
    for _ in range(args.rounds):
        for c in configs:
            got, r = run(pkg, plan, reqs, arrivals, c)
            runs[str(c)].append(r)
            ids.setdefault(c, []).append(got)
    out["runs"] = runs

    alone = []
    for latest, start, prompt in reqs[:args.parity]:
        plan.kv_reset()
        alone.append(pkg.engine.generate_tokens_llama(lambda t, p: plan.forward_decode(t, p, logits=False)[1], latest, start, prompt, [], CTX, CTX))
    first = ids[0][0]
    ok_runs = all(g == first for c in configs for g in ids[c])
    ok_alone = first[:args.parity] == alone
    ok_budget = [len(x) for x in first] == budgets
    out["parity"] = {"requests_alone": args.parity, "runs_equal": ok_runs, "equals_alone": ok_alone, "budgets_met": ok_budget,
                     "ok": bool(ok_runs and ok_alone and ok_budget)}
    plan.free()
    print(json.dumps(out))
    if not out["parity"]["ok"]:
        sys.exit(1)


if __name__ == "__main__":
    main()
