#!/usr/bin/env python
"""Kernel-time breakdown of one tensor-core prefill chunk on the Llama-3-8B-shaped Q8_0 model, per prefill mode
(torch.profiler, CUDA kernel time summed by kernel name over `--reps` chunks, divided by the reps).

    python tools/pp_profile.py --pp-size 512 --modes tensor_core_w8a16,tensor_core

Prints one JSON object: {mode: {"ms_per_chunk": device ms per chunk (CUDA events), "kernels": [[name, ms per chunk, calls per chunk], ...]}}."""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as ge  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pp-size", type=int, default=512)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--modes", default="tensor_core_w8a16,tensor_core")
    ap.add_argument("--top", type=int, default=12)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    pkg = ge.import_package()
    shape = pkg.synth.SHAPES["llama-3-8b"]
    Q8 = pkg.gguf.GGMLType.Q8_0
    n = args.pp_size
    model = pkg.loader.model_from_tensors(shape, Q8, pkg.synth.build_tensors_fast(shape, Q8, seed=1234, device="cuda:0"), n + 8)
    plan = pkg.B200MasterPlan.initialize_plan(model, prefill_batch_size=n)
    toks = np.asarray(pkg.llama_bench.synthetic_tokens(shape.vocab, n), dtype=np.int32)
    out = {}
    for mode in args.modes.split(","):
        plan.set_prefill_mode(mode)
        for _ in range(2):
            plan.forward_batch_prefill(toks, 0)
        torch.cuda.synchronize()
        ms = []
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                plan.forward_batch_prefill(toks, 0)
                ms.append(plan.prefill_info()[2])
            torch.cuda.synchronize()
        rows = {}
        for e in prof.events():
            if e.device_type.name != "CUDA":
                continue
            r = rows.setdefault(e.name, [0.0, 0])
            r[0] += e.device_time / 1e3  # us -> ms
            r[1] += 1
        top = sorted(rows.items(), key=lambda kv: -kv[1][0])[:args.top]
        out[mode] = {"ms_per_chunk": float(np.mean(ms)), "kernels": [[name, t / args.reps, c // args.reps] for name, (t, c) in top]}
    plan.free()
    print(json.dumps({"pp": n, "device": torch.cuda.get_device_name(0), "modes": out}))


if __name__ == "__main__":
    main()
