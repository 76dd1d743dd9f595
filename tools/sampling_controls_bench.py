#!/usr/bin/env python
"""Sampling controls (b200_set_sampling_controls) on the H100:

  kernel_<vocab>_<setting>  k_sample_ctl against a one-row k_sample_rows on one random row at vocabularies 128256 and 151936,
                            temperature 0.8 with top-p 0.9 and without top-p; settings: penalties over a 512-token history with top-k off, and the
                            same with top-k 40.  b200_time_sample_controls: CUDA events around --kernel-reps launches of each
                            kernel, every launch on its own copy of the row and counts, ms per launch
  tg_<setting>              the Llama-3-8B-shaped Q8_0 model of bench.py, --tokens sampled tokens through forward_decode_sample
                            (temperature 0.8, top-p 0.9) with controls off and on (top-k 40, min-p 0.05, penalties, a 512-token
                            history), alternated within each repeat; host clock around the loop (every call ends in a stream
                            synchronise), median of --reps, ms per token
  step8_<setting>           one forward_step of 8 emitting sampled rows on 8 slots, no slot controlled against all 8: host clock,
                            median of --steps calls

    python tools/sampling_controls_bench.py [--tokens 128] [--reps 5] [--steps 50] [--kernel-reps 50]

Prints one JSON line with the card's name, power limit and max SM clock (nvidia-smi, read in the same run)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as ge  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--kernel-reps", type=int, default=50)
    args = ap.parse_args()
    pkg = ge.import_package()
    N, S = pkg.native, pkg.sampler.SamplingControls
    out = {"card": card()}
    rng = np.random.default_rng(0)

    for V in (128256, 151936):
        row = (rng.standard_normal(V) * 3).astype(np.float32)
        counts = np.bincount(rng.integers(0, V, 512), minlength=V).astype(np.int32)
        for topp in (0.9, 0.0):
            tag = f"kernel_{V}_topp{topp}"
            for name, c in (("penalties", S(repetition_penalty=1.1, frequency_penalty=0.1, presence_penalty=0.2)),
                            ("penalties_top_k40", S(top_k=40, repetition_penalty=1.1, frequency_penalty=0.1, presence_penalty=0.2))):
                ctl_ms, plain_ms = N.time_sample_controls(row, counts, c, 0.8, topp, 0.5, args.kernel_reps)
                out[f"{tag}_{name}_us"] = round(ctl_ms * 1e3, 1)
                out[f"{tag}_k_sample_rows_us"] = round(plain_ms * 1e3, 1)

    print(json.dumps(out), file=sys.stderr, flush=True)  # progress: each section's figures as soon as they exist
    n = args.tokens
    shape = pkg.synth.SHAPES["llama-3-8b"]
    Q8 = pkg.gguf.GGMLType.Q8_0
    model = pkg.loader.model_from_tensors(shape, Q8, pkg.synth.build_tensors_fast(shape, Q8, seed=1234, device="cuda:0"), n + 16)
    plan = pkg.B200MasterPlan.initialize_plan(model)
    V = model.configuration.vocab_size
    hist = [int(t) for t in rng.integers(0, V, 512)]
    ctl = S(top_k=40, min_p=0.05, repetition_penalty=1.1, frequency_penalty=0.1, presence_penalty=0.2)
    ms = {"off": [], "on": []}
    for r in range(1 + args.reps):
        for name, c in (("off", None), ("on", ctl)):
            smp = pkg.sampler.Sampler(V, 0.8, 0.9, 7, controls=c, history=hist if c else None)
            plan.kv_reset()
            tok = 1
            t0 = time.perf_counter()
            for p in range(n):
                tok = smp.sample_token(plan, tok, p)
            if r:
                ms[name].append((time.perf_counter() - t0) * 1e3 / n)
            # the plain sampler turned off the controls the previous repeat left on slot -1
            assert (plan.sampling_controls(-1) is None) == (c is None)
    for name in ms:
        out[f"tg{n}_{name}_ms_per_token"] = round(float(np.median(ms[name])), 4)
    out[f"tg{n}_on_vs_off_pct"] = round(100 * (np.median(ms["on"]) / np.median(ms["off"]) - 1), 2)
    print(json.dumps(out), file=sys.stderr, flush=True)

    plan.set_decode_slots(8)
    rows = [(s, 1 + s, 0, 1, 0.8, 0.9, 0.25 + 0.05 * s) for s in range(8)]
    for name, c in (("none", None), ("all", ctl)):
        for s in range(8):
            plan.set_sampling_controls(s, c)
        t = []
        for k in range(1 + args.steps):
            t0 = time.perf_counter()
            plan.forward_step(rows)
            if k:
                t.append((time.perf_counter() - t0) * 1e3)
        out[f"step8_{name}_ms"] = round(float(np.median(t)), 4)
    plan.free()
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
