#!/usr/bin/env python
"""Generated-token log-probabilities (b200_set_logprobs) on the Llama-3-8B-shaped Q8_0 model of bench.py, on ONE plan:

  tg_<setting>     b200_decode_sequence of --tokens greedy steps (feedback) with logprobs off, N = 0, N = 5 and N = 20, the settings
                   alternated within each repeat; device_ms of the call (CUDA events around the steps and, when on, the one
                   k_token_logprobs launch per step), median of --reps
  batch8_<setting> one forward_decode_batch step of 8 rows (greedy), logprobs off and N = 20: host clock around the call, which ends
                   in a stream synchronise, median of --steps calls
  kernel_<vocab>   k_token_logprobs alone (b200_test_logprobs) on a random row at vocabularies 128256 and 151936, N = 20: CUDA events
                   over --kernel-reps launches

    python tools/logprobs_bench.py [--tokens 128] [--reps 5] [--steps 50] [--kernel-reps 2000]

Prints one JSON line with the card's name, power limit and max SM clock (nvidia-smi, read in the same run).  Gate: the greedy ids
equal with logprobs off and on, and the chosen log-probabilities of the N = 20 run bit-equal to score_tokens (exact prefill mode) of
the generated sequence; a mismatch exits with status 1."""
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

SETTINGS = (("off", -1), ("n0", 0), ("n5", 5), ("n20", 20))


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--kernel-reps", type=int, default=2000)
    args = ap.parse_args()
    n = args.tokens
    pkg = ge.import_package()
    shape = pkg.synth.SHAPES["llama-3-8b"]
    Q8 = pkg.gguf.GGMLType.Q8_0
    model = pkg.loader.model_from_tensors(shape, Q8, pkg.synth.build_tensors_fast(shape, Q8, seed=1234, device="cuda:0"), n + 16)
    plan = pkg.B200MasterPlan.initialize_plan(model, prefill_batch_size=n)
    out = {"card": card(), "model": "llama-3-8b Q8_0 (synthetic)", "tokens": n}
    ok = True

    # tg<n>: the settings alternated within each repeat, one untimed round first
    ms, ids, chosen = {}, {}, None
    for r in range(1 + args.reps):
        for name, top_n in SETTINGS:
            plan.set_logprobs(top_n)
            plan.kv_reset()
            got, dms = plan.decode_sequence([1], n, 0, feedback=True)
            ids.setdefault(name, got)
            ok = ok and np.array_equal(got, ids["off"])
            if r:
                ms.setdefault(name, []).append(dms)
            if top_n == 20:
                chosen = plan.last_logprobs()[0]
    base = float(np.median(ms["off"]))
    for name, _ in SETTINGS:
        med = float(np.median(ms[name]))
        out[f"tg_{name}"] = {"ms_per_token": round(med / n, 4), "tok_s": round(n / (med / 1e3), 1), "vs_off_pct": round(100 * (med / base - 1), 2)}
    # the gate: chosen against score_tokens of the generated sequence
    plan.set_prefill_mode("exact")
    plan.kv_reset()
    seq = np.concatenate([[1], ids["off"][:-1]]).astype(np.int32)
    lp, _ = plan.score_tokens(seq, 0, ids["off"])
    ok = ok and np.array_equal(lp.view(np.uint64), chosen.view(np.uint64))

    # one 8-row batched step
    plan.set_decode_slots(8)
    slots = list(range(8))
    toks = [int(t) for t in ids["off"][:8]]
    for name, top_n in (("off", -1), ("n20", 20)):
        plan.set_logprobs(top_n)
        t = []
        for k in range(1 + args.steps):
            t0 = time.perf_counter()
            plan.forward_decode_batch(slots, toks, [k % 8] * 8)
            if k:
                t.append((time.perf_counter() - t0) * 1e3)
        out[f"batch8_{name}"] = {"ms": round(float(np.median(t)), 4), "device_ms": round(plan.batch_info()[2], 4)}
    plan.free()

    # the kernel alone
    rng = np.random.default_rng(0)
    for V in (128256, 151936):
        row = (rng.standard_normal(V) * 3).astype(np.float32)
        _, _, _, kms = pkg.native.test_logprobs(row, 5, 20, args.kernel_reps)
        out[f"kernel_{V}_us"] = round(kms * 1e3, 2)
    out["parity"] = "bit-equal" if ok else "MISMATCH"
    print(json.dumps(out))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
