#!/usr/bin/env python
"""Prompt prefill of a synthetic MoE model in the exact prefill mode and in tensor_core_exact_moe (the chunk routed on the device,
grouped int8 expert GEMMs), generated on the device as tools/qwen3moe_bench.py / tools/moe_bench.py build it: Qwen3-30B-A3B-shaped
(48 layers, 128 experts, top-8, expert hidden 768) by default, Qwen1.5-MoE-A2.7B-shaped with --shape qwen1.5-moe-a2.7b.

    python tools/moe_prefill_bench.py [--shape qwen3-30b-a3b] [--lengths 16,32,64,128,256,512] [--reps 3]

Prints one JSON line:
  * per chunk length and mode, after one warm-up chunk: tok/s from a host clock around b200_forward_batch_prefill (which ends in a
    device synchronise), and the device milliseconds and kernel launches b200_prefill_info reports for the chunk (exact mode runs
    no tensor-core chunk: its device time is not reported);
  * the crossover: the shortest measured length from which the new mode is faster at every longer measured length;
  * parity, in the same run: every layer's K / V after one chunk of the longest length, and the scores of a 128-token chunk, bit-equal
    between the two modes;
  * the GPU name and its power limit, read with one read-only nvidia-smi query in the same run."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import __graft_entry__ as ge  # noqa: E402
from qwen3moe_bench import gpu_info  # noqa: E402

MODES = ("exact", "tensor_core_exact_moe")


def kv(plan, c):
    nkv = c.context_length * c.kv_dim
    return [plan.read_buffer(n, nkv, layer=l) for n in ("key_cache", "value_cache") for l in range(c.n_layers)]


def time_chunk(plan, toks, reps):
    """[(host seconds, device ms, launches)] of reps chunks from position 0 after one warm-up."""
    plan.kv_reset()
    plan.forward_batch_prefill(toks, 0)
    out = []
    for _ in range(reps):
        plan.kv_reset()
        t0 = time.perf_counter()
        plan.forward_batch_prefill(toks, 0)
        dt = time.perf_counter() - t0
        _, launches, ms = plan.prefill_info()
        out.append((dt, ms, launches))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="qwen3-30b-a3b", choices=("qwen3-30b-a3b", "qwen1.5-moe-a2.7b"))
    ap.add_argument("--lengths", default="16,32,64,128,256,512")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    lengths = sorted(int(x) for x in args.lengths.split(","))
    import torch

    pkg = ge.import_package()
    info = gpu_info()
    sh = pkg.synth.SHAPES[args.shape]
    Q8 = pkg.gguf.GGMLType.Q8_0
    top = lengths[-1]
    ctx = max(top, 128) + 8
    model = pkg.loader.model_from_tensors(sh, Q8, pkg.synth.build_tensors_fast(sh, Q8, seed=1234, device="cuda:0"), ctx)
    torch.cuda.empty_cache()
    plan = pkg.B200MasterPlan.initialize_plan(model, prefill_batch_size=top)
    c = model.configuration
    toks = np.asarray(pkg.llama_bench.synthetic_tokens(sh.vocab, top + 1), dtype=np.int32)
    out = {"metric": f"{args.shape}_q8_0_prefill", "workload": f"{args.shape}-shaped synthetic Q8_0 ({sh.n_layers} layers, {sh.n_experts} experts, "
           f"top-{sh.n_experts_used}, expert hidden {sh.expert_hidden})", **info, "torch_device": torch.cuda.get_device_name(0)}
    try:
        # parity gate first: K / V of one chunk of the longest length, scores of a 128-token chunk
        runs = {}
        for mode in MODES:
            plan.set_prefill_mode(mode)
            plan.kv_reset()
            plan.forward_batch_prefill(toks[:top], 0)
            cache = [a.copy() for a in kv(plan, c)]
            plan.kv_reset()
            n = min(128, top)
            lp, ids = plan.score_tokens(toks[:n], 0, toks[1:n + 1])
            runs[mode] = (cache, lp, ids)
        (ka, la, ia), (kb, lb, ib) = runs[MODES[0]], runs[MODES[1]]
        kv_ok = all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(ka, kb))
        sc_ok = bool(np.array_equal(la.view(np.uint64), lb.view(np.uint64)) and np.array_equal(ia, ib))
        out["parity"] = {"kv_chunk": top, "kv_bit_equal": kv_ok, "score_chunk": min(128, top), "scores_bit_equal": sc_ok, "ok": kv_ok and sc_ok}

        res = {}
        for mode in MODES:
            plan.set_prefill_mode(mode)
            res[mode] = {}
            for n in lengths:
                r = time_chunk(plan, toks[:n], args.reps)
                sec = float(np.median([x[0] for x in r]))
                res[mode][n] = {"tok_s": n / sec, "host_ms": sec * 1e3, "runs_host_ms": [x[0] * 1e3 for x in r]}
                if mode != "exact":
                    res[mode][n].update({"device_ms": float(np.median([x[1] for x in r])), "launches": r[-1][2]})
        out["prefill"] = res
        faster = [res[MODES[1]][n]["tok_s"] > res[MODES[0]][n]["tok_s"] for n in lengths]
        cross = next((n for i, n in enumerate(lengths) if all(faster[i:])), None)
        out["crossover_chunk_length"] = cross
        out["speedup"] = {n: res[MODES[1]][n]["tok_s"] / res[MODES[0]][n]["tok_s"] for n in lengths}
    finally:
        plan.free()
    print(json.dumps(out))
    return 0 if out.get("parity", {}).get("ok") else 1


if __name__ == "__main__":
    sys.exit(main())
