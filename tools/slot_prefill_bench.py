#!/usr/bin/env python
"""Admitting 8 prompts into 8 decode slots on bench.py's synthetic Llama-3-8B Q8_0 model, three ways:

  (a) the path before b200_prefill_slots: per prompt kv_reset + forward_batch_prefill + slot_copy_kv (tensor-core modes);
  (b) one prefill_slots call for all 8 prompts, in twin (tensor_core) and W8A16 mode;
  (c) exact mode: prefill_slots against feeding the prompts through forward_decode_batch, one step per position.

    python tools/slot_prefill_bench.py [--prompts 64,16] [--ctx 2048] [--reps 5]

Prints one JSON line: per prompt length and method, wall-clock ms per admission of all 8 prompts (median of --reps after one
warm-up round; every call ends in a device synchronise), the device ms b200_prefill_info reports for the prefill_slots calls, and
tokens/s.  Parity gate, before timing: after each admission, the first forward_decode_batch step is compared with the
single-sequence path (kv_reset + forward_batch_prefill + forward_decode in the same mode).  Exact mode must give every slot the
same id.  The tensor-core modes split K in the residual GEMMs at this shape, and the order of the split-K reduce-adds is not fixed,
so their logits must stay within the 3 % of max|ref| bar of tests/test_gpu_prefill.py, and equal ids are reported, not required.
The GPU name and power limit come from one read-only nvidia-smi query in the same run."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import __graft_entry__ as ge  # noqa: E402
from batch_decode_bench import gpu_info  # noqa: E402

N_SLOTS = 8


def timed(fn, reps):
    fn()
    walls, devs = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        d = fn()
        walls.append((time.perf_counter() - t0) * 1e3)
        devs.append(d)
    return statistics.median(walls), (statistics.median(devs) if devs[0] is not None else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--prompts", default="64,16")
    ap.add_argument("--ctx", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    lengths = [int(x) for x in args.prompts.split(",")]
    pkg = ge.import_package()
    info = gpu_info()
    sh = pkg.synth.SHAPES["llama-3-8b"]
    Q8 = pkg.gguf.GGMLType.Q8_0
    model = pkg.loader.model_from_tensors(sh, Q8, pkg.synth.build_tensors_fast(sh, Q8, seed=1234, device="cuda:0"), args.ctx)
    batch = N_SLOTS * max(lengths)
    plan = pkg.B200MasterPlan.initialize_plan(model, prefill_batch_size=batch)
    plan.set_decode_slots(N_SLOTS)
    rng = np.random.default_rng(11)
    out = {"metric": "llama-3-8b_q8_0_slot_prefill", "workload": f"llama-3-8b-shaped synthetic Q8_0, {sh.n_layers} layers, ctx {args.ctx}, "
           f"{N_SLOTS} slots", **info, "reps": args.reps, "prefill_batch_size": batch}
    slots = list(range(N_SLOTS))
    parity, res = {}, {}
    for n in lengths:
        prompts = [rng.integers(0, sh.vocab, n + 1).astype(np.int32) for _ in slots]
        nxt = [int(p[n]) for p in prompts]

        def first_step_single():
            ids, lgs = [], []
            for s in slots:
                plan.kv_reset()
                plan.forward_batch_prefill(prompts[s][:n], 0)
                lg, am = plan.forward_decode(nxt[s], n)
                ids.append(int(am))
                lgs.append(lg.copy())
            return ids, lgs

        def admit_slots():
            plan.prefill_slots(slots, [0] * N_SLOTS, [p[:n] for p in prompts])
            return plan.prefill_info()[2]

        def admit_copy():
            d = 0.0
            for s in slots:
                plan.kv_reset()
                plan.forward_batch_prefill(prompts[s][:n], 0)
                d += plan.prefill_info()[2]
                plan.slot_copy_kv(s, n)
            return d

        def admit_decode_steps():
            for p in range(n):
                plan.forward_decode_batch(slots, [int(prompts[s][p]) for s in slots], [p] * N_SLOTS)

        r = {}
        for mode in ("exact", "tensor_core", "tensor_core_w8a16"):
            plan.set_prefill_mode(mode)
            want, want_lg = first_step_single()
            admit_slots()
            got, got_lg = plan.forward_decode_batch(slots, nxt, [n] * N_SLOTS, logits=True)
            err = max(float(np.max(np.abs(got_lg[s] - want_lg[s])) / np.max(np.abs(want_lg[s]))) for s in slots)
            same = [int(i) for i in got] == want
            parity[f"{mode}_{n}"] = {"ids_equal": same, "max_rel_logit_err": err,
                                     "ok": same and err == 0.0 if mode == "exact" else err <= 0.03}
            wall, dev = timed(admit_slots, args.reps)
            r[f"prefill_slots_{mode}"] = {"wall_ms": wall, "device_ms": dev, "tok_s_wall": N_SLOTS * n * 1e3 / wall,
                                          "launches": plan.prefill_info()[1]}
            if mode == "exact":
                wall, _ = timed(admit_decode_steps, args.reps)
                r["decode_batch_steps_exact"] = {"wall_ms": wall, "tok_s_wall": N_SLOTS * n * 1e3 / wall}
            else:
                wall, dev = timed(admit_copy, args.reps)
                r[f"prefill_copy_{mode}"] = {"wall_ms": wall, "prefill_device_ms": dev, "tok_s_wall": N_SLOTS * n * 1e3 / wall}
        res[f"8x{n}"] = r
    out["parity"] = {**parity, "ok": all(v["ok"] for v in parity.values())}
    out["admission"] = res
    plan.free()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
