#!/usr/bin/env python
"""Continuous batching (engine.generate_tokens_continuous over b200_forward_step) against arrival-order waves, on the synthetic
Llama-3-8B Q8_0 model of bench.py and a seeded request trace, alternated on the same plan.

    python tools/continuous_bench.py [--requests 32] [--rounds 2] [--parity 6] [--seed 11]

The trace: prompt lengths 16-256, generation budgets 32-128, request i arriving before step 3 i of the scheduler.  A request's
budget is expressed the way both loops clamp it: max_tokens is the context (400) and the request starts at position
400 - len(prompt) - budget, so the Llama loop generates exactly `budget` tokens (no stop token).  Runs, in every round:
  (a) generate_tokens_continuous on 8 slots: decode rows and exact prompt rows share every step;
  (b) the requests in arrival order, 8 per wave, through generate_tokens_batch_prefill in the exact prefill mode, each wave on
      zeroed slots -- every request of a wave is taken as available when the wave starts (arrival times are ignored, which
      favours this side);
  (c) the 8-row forward_decode_batch step alone (--steps steps), to show (a) left it unchanged.
Prints one JSON line: per run the wall time, generated tok/s, time to first token and completion time (median / p90, seconds from
the start of the run; for (a) also from submission), rows and launches per step; the parity gate (every request of the first
--parity requests from (a) equals generate_tokens_llama alone on the plan's own cache, and every request of (a) equals (b)); and
the GPU name and power limit from one read-only nvidia-smi query in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402

CTX = 400
SLOTS = 8


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": limit}
    except Exception as e:  # noqa: BLE001
        return {"gpu": None, "power_limit": None, "nvidia_smi_error": str(e)}


def trace(n: int, vocab: int, seed: int):
    rng = np.random.default_rng(seed)
    reqs, budgets = [], []
    for _ in range(n):
        k, b = int(rng.integers(16, 257)), int(rng.integers(32, 129))
        prompt = [int(t) for t in rng.integers(0, vocab, k)]
        reqs.append((int(rng.integers(vocab)), CTX - k - b, prompt))
        budgets.append(b)
    return reqs, budgets, [3 * i for i in range(n)]


def pct(v, q):
    v = [x for x in v if x is not None]
    return float(np.percentile(v, q)) if v else None


class Recorder:
    """The plan with every forward_decode_batch call timed: when each slot got a token."""

    def __init__(self, plan):
        self._plan, self.calls = plan, []

    def __getattr__(self, name):
        return getattr(self._plan, name)

    def forward_decode_batch(self, slots, tokens, positions, sampling=None, logits=False):
        out = self._plan.forward_decode_batch(slots, tokens, positions, sampling, logits)
        self.calls.append((time.perf_counter(), list(slots), self._plan.batch_info()[1]))
        return out


def run_continuous(pkg, plan, reqs, arrivals):
    stats = {}
    t0 = time.perf_counter()
    ids = pkg.engine.generate_tokens_continuous(plan, "LLAMA_3", reqs, arrivals, [], CTX, CTX, stats=stats)
    wall = time.perf_counter() - t0
    gen = sum(len(x) for x in ids)
    ttft = [f - t0 for f in stats["first_token"]]
    done = [d - t0 for d in stats["done"]]
    ttft_sub = [f - s for f, s in zip(stats["first_token"], stats["submitted"])]
    done_sub = [d - s for d, s in zip(stats["done"], stats["submitted"])]
    return ids, {"wall_s": wall, "generated": gen, "tok_s": gen / wall, "steps": stats["steps"],
                 "ttft_s": {"median": pct(ttft, 50), "p90": pct(ttft, 90)}, "done_s": {"median": pct(done, 50), "p90": pct(done, 90)},
                 "ttft_since_submit_s": {"median": pct(ttft_sub, 50), "p90": pct(ttft_sub, 90)},
                 "done_since_submit_s": {"median": pct(done_sub, 50), "p90": pct(done_sub, 90)},
                 "rows_per_step": float(np.mean(stats["rows"])), "launches_per_step": float(np.mean(stats["launches"]))}


def run_waves(pkg, plan, reqs):
    rec = Recorder(plan)
    ids, first, done = [], [], []
    t0 = time.perf_counter()
    for w in range(0, len(reqs), SLOTS):
        wave = reqs[w:w + SLOTS]
        rec.calls = []
        for s in range(len(wave)):  # the trace starts past position 0 and this loop reads a slot's rows below start: zero them,
            plan.slot_reset(s)      # as the continuous run's admission does
        ids += pkg.engine.generate_tokens_batch_prefill(rec, "LLAMA_3", wave, [], CTX, CTX, 8 * 256)
        for s in range(len(wave)):
            ts = [t for t, slots, _ in rec.calls if s in slots]
            first.append(ts[0] - t0 if ts else None)
            done.append(ts[-1] - t0 if ts else None)
        if w == 0:
            rows = [len(sl) for _, sl, _ in rec.calls]
            launches = [n for _, _, n in rec.calls]
    wall = time.perf_counter() - t0
    gen = sum(len(x) for x in ids)
    return ids, {"wall_s": wall, "generated": gen, "tok_s": gen / wall, "ttft_s": {"median": pct(first, 50), "p90": pct(first, 90)},
                 "done_s": {"median": pct(done, 50), "p90": pct(done, 90)}, "decode_rows_per_step_wave0": float(np.mean(rows)),
                 "decode_launches_per_step": float(np.mean(launches))}


def run_batch_step(plan, steps, vocab):
    rng = np.random.default_rng(5)
    slots = list(range(SLOTS))
    dev = []
    t0 = time.perf_counter()
    for k in range(steps):
        plan.forward_decode_batch(slots, [int(t) for t in rng.integers(0, vocab, SLOTS)], [200 + k] * SLOTS)
        dev.append(plan.batch_info()[2])
    wall = (time.perf_counter() - t0) * 1e3 / steps
    return {"wall_ms_per_step": wall, "device_ms_per_step": float(np.median(dev)), "tok_s_wall": SLOTS * 1e3 / wall,
            "launches_per_step": plan.batch_info()[1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--parity", type=int, default=6)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--seed", type=int, default=11)
    args = ap.parse_args()
    import torch

    pkg = ge.import_package()
    info = gpu_info()
    sh = pkg.synth.SHAPES["llama-3-8b"]
    Q8 = pkg.gguf.GGMLType.Q8_0
    model = pkg.loader.model_from_tensors(sh, Q8, pkg.synth.build_tensors_fast(sh, Q8, seed=1234, device="cuda:0"), CTX)
    plan = pkg.B200MasterPlan.initialize_plan(model)
    plan.set_prefill_mode("exact")
    plan.set_decode_slots(SLOTS)
    reqs, budgets, arrivals = trace(args.requests, sh.vocab, args.seed)
    out = {"metric": "llama-3-8b_q8_0_continuous_batching", "workload": f"llama-3-8b-shaped synthetic Q8_0, {sh.n_layers} layers", **info,
           "torch_device": torch.cuda.get_device_name(0), "requests": args.requests, "slots": SLOTS, "context": CTX,
           "prompt_tokens": sum(len(r[2]) for r in reqs), "budget_tokens": sum(budgets), "arrival_every_steps": 3}

    # warm-up: capture the graphs both runs use
    pkg.engine.generate_tokens_continuous(plan, "LLAMA_3", reqs[:SLOTS], [0] * SLOTS, [], CTX, CTX)
    pkg.engine.generate_tokens_batch_prefill(plan, "LLAMA_3", reqs[:SLOTS], [], CTX, CTX, 8 * 256)

    runs = {"continuous": [], "waves": [], "batch_step": []}
    ids_a = ids_b = None
    for _ in range(args.rounds):
        ids_a, ra = run_continuous(pkg, plan, reqs, arrivals)
        runs["continuous"].append(ra)
        ids_b, rb = run_waves(pkg, plan, reqs)
        runs["waves"].append(rb)
        runs["batch_step"].append(run_batch_step(plan, args.steps, sh.vocab))
    out["runs"] = runs
    out["continuous_vs_waves_tok_s"] = [a["tok_s"] / b["tok_s"] for a, b in zip(runs["continuous"], runs["waves"])]

    # parity gate: the first requests alone through the single-sequence loop on the plan's own cache
    alone = []
    for latest, start, prompt in reqs[:args.parity]:
        plan.kv_reset()
        alone.append(pkg.engine.generate_tokens_llama(lambda t, p: plan.forward_decode(t, p, logits=False)[1], latest, start, prompt, [], CTX, CTX))
    ok_alone = all(a == b for a, b in zip(ids_a[:args.parity], alone))
    ok_waves = ids_a == ids_b
    ok_budget = [len(x) for x in ids_a] == budgets
    out["parity"] = {"requests_alone": args.parity, "continuous_equals_alone": ok_alone, "continuous_equals_waves": ok_waves,
                     "budgets_met": ok_budget, "ok": bool(ok_alone and ok_waves and ok_budget)}
    plan.free()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
