#!/usr/bin/env python
"""Prompt processing on the Llama-3-8B-shaped Q8_0 model of bench.py in the four prefill modes, on ONE plan, chunks alternating:
exact (B200_PREFILL_EXACT: multi-position steps of the batched decode), tensor_core_exact (B200_PREFILL_TENSOR_CORE_EXACT: int8
wgmma GEMMs over the whole chunk), twin (B200_PREFILL_TENSOR_CORE) and w8a16 (B200_PREFILL_TENSOR_CORE_W8A16).

    python tools/pp_exact_bench.py [--pp 64,128,512] [--reps 3] [--profile]

Prints one JSON line: the card's name, power limit and max SM clock (nvidia-smi, read in the same run); per chunk length and mode
the ms per chunk (host clock around the call, which ends in a stream synchronise) and tok/s; the prefill_slots admission case
(8 prompts x 64 tokens into 8 decode slots) in the exact and tensor_core_exact modes; and, with --profile, a separate
torch.profiler run of one tensor_core_exact chunk of the longest length split into GEMM, norm and RoPE / attention kernel time.

Parity gate: after every tensor_core_exact chunk the last layer's K / V rows and the logits of the first decode step are bit-equal
to those after the exact chunk, and the slots' K / V too; a mismatch exits with status 1."""
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

MODES = {"exact": "exact", "tensor_core_exact": "tensor_core_exact", "twin": "tensor_core", "w8a16": "tensor_core_w8a16"}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pp", default="64,128,512", help="chunk lengths")
    ap.add_argument("--reps", type=int, default=3, help="timed chunks per mode and length (after one untimed round)")
    ap.add_argument("--profile", action="store_true", help="add the kernel-time split of one tensor_core_exact chunk")
    args = ap.parse_args()
    pp = [int(x) for x in args.pp.split(",")]
    pkg = ge.import_package()
    shape = pkg.synth.SHAPES["llama-3-8b"]
    Q8 = pkg.gguf.GGMLType.Q8_0
    big = max(pp + [512])  # the slots case packs 8 x 64 tokens into one chunk
    model = pkg.loader.model_from_tensors(shape, Q8, pkg.synth.build_tensors_fast(shape, Q8, seed=1234, device="cuda:0"), big + 8)
    plan = pkg.B200MasterPlan.initialize_plan(model, prefill_batch_size=big)
    toks = np.asarray(pkg.llama_bench.synthetic_tokens(shape.vocab, big + 1), dtype=np.int32)
    L = shape.n_layers - 1
    out = {"card": card(), "model": "llama-3-8b Q8_0 (synthetic)", "pp": {}}
    ok = True
    for n in pp:
        ms = {k: [] for k in MODES}
        ref = {}
        for r in range(1 + args.reps):
            for name, mode in MODES.items():
                plan.set_prefill_mode(mode)
                t0 = time.perf_counter()
                plan.forward_batch_prefill(toks[:n], 0)
                dt = (time.perf_counter() - t0) * 1e3
                if r:
                    ms[name].append(dt)
                if name in ("exact", "tensor_core_exact"):
                    kv = [plan.read_buffer(c, n * shape.kv_dim, layer=L) for c in ("key_cache", "value_cache")]
                    lg, _ = plan.forward_decode(int(toks[n]), n)
                    got = kv + [lg.copy()]
                    if name == "exact":
                        ref = got
                    elif not all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(got, ref)):
                        ok = False
        out["pp"][n] = {k: {"ms": round(float(np.median(v)), 3), "tok_s": round(n / (np.median(v) / 1e3), 1)} for k, v in ms.items()}
    # admission: 8 prompts of 64 tokens into 8 decode slots
    plan.set_decode_slots(8)
    lists = [toks[64 * i % big:64 * i % big + 64] if 64 * i % big + 64 <= big else toks[:64] for i in range(8)]
    slots = {}
    kv = {}
    for r in range(1 + args.reps):
        for name in ("exact", "tensor_core_exact"):
            plan.set_prefill_mode(name)
            plan.prefill_slots(list(range(8)), [0] * 8, lists)
            if r:
                slots.setdefault(name, []).append(plan.prefill_info()[2])
            kv[name] = [plan.read_buffer(c, 64 * shape.kv_dim, layer=7 * shape.n_layers + L) for c in ("slot_key_cache", "slot_value_cache")]
        if not all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(kv["exact"], kv["tensor_core_exact"])):
            ok = False
    out["slots_8x64"] = {k: {"ms": round(float(np.median(v)), 3), "tok_s": round(512 / (np.median(v) / 1e3), 1)} for k, v in slots.items()}
    if args.profile:
        import torch
        from torch.profiler import ProfilerActivity, profile

        plan.set_prefill_mode("tensor_core_exact")
        plan.forward_batch_prefill(toks[:big], 0)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            plan.forward_batch_prefill(toks[:big], 0)
            torch.cuda.synchronize()
        split = {"gemm": 0.0, "norm": 0.0, "rope_kv": 0.0, "attention": 0.0, "other": 0.0}
        for e in prof.key_averages():
            us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            key = next((k for k, s in (("gemm", "k_gemm_i8"), ("norm", "k_i8_norm"), ("rope_kv", "k_i8_rope_kv"), ("attention", "k_i8_attention")) if s in e.key), "other")
            split[key] += us / 1e3
        out["profile_pp%d_ms" % big] = {k: round(v, 3) for k, v in split.items()}
    plan.free()
    out["parity"] = "bit-equal" if ok else "MISMATCH"
    print(json.dumps(out))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
