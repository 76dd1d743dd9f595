#!/usr/bin/env python
"""Batched decode (b200_forward_decode_batch) on a synthetic Q8_0 model: ms per step and aggregate tok/s for n = 1, 2, 4, 8 rows,
alternated in the same run with single-sequence b200_forward_decode on the same plan.

    python tools/batch_decode_bench.py [--workload llama-3-8b|qwen3-4b|qwen2.5-7b] [--steps 128] [--warmup 8] [--parity-steps 4] [--profile]

Prints one JSON line:
  * per n: device ms per step (CUDA events around the step's graph, b200_batch_info; median), wall-clock ms per step over --steps
    steps after the warm-up (each call ends in a device synchronise), aggregate tok/s from both, and the same for single-sequence
    b200_forward_decode (wall clock);
  * the whole-step HBM roofline: weight bytes + n x the K/V bytes of the mean position, over 3.35 TB/s (H100 SXM data sheet);
  * parity gate: each row's first --parity-steps ids equal the single-sequence decode of the same token stream, and step 0's logits
    are bit-equal;
  * with --profile: device time per kernel over a few 8-row steps (torch.profiler, in a run of its own after the timing);
  * the GPU name and power limit, read with one read-only nvidia-smi query in the same run."""
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

PEAK_BW = 3.35e12
ROWS = (1, 2, 4, 8)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": limit}
    except Exception as e:  # noqa: BLE001
        return {"gpu": None, "power_limit": None, "nvidia_smi_error": str(e)}


def step_bytes(sh, n: int, pos: float) -> dict:
    w = sh.matmul_elements() * 34 // 32  # Q8_0 matrices and classifier, streamed once per step whatever n is
    kv = int(n * sh.n_layers * 2 * (pos + 1) * sh.kv_dim * 4)  # each row reads its own FP32 K / V rows
    return {"weights": w, "kv": kv, "total": w + kv}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="llama-3-8b", choices=["llama-3-8b", "qwen3-4b", "qwen2.5-7b"])
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--parity-steps", type=int, default=4)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    import torch

    pkg = ge.import_package()
    info = gpu_info()
    sh = pkg.synth.SHAPES[args.workload]
    Q8 = pkg.gguf.GGMLType.Q8_0
    ctx = args.warmup + args.steps + 8
    model = pkg.loader.model_from_tensors(sh, Q8, pkg.synth.build_tensors_fast(sh, Q8, seed=1234, device="cuda:0"), ctx)
    plan = pkg.B200MasterPlan.initialize_plan(model)
    plan.set_decode_slots(max(ROWS))
    out = {"metric": f"{args.workload}_q8_0_batched_decode", "workload": f"{args.workload}-shaped synthetic Q8_0, {sh.n_layers} layers", **info,
           "torch_device": torch.cuda.get_device_name(0), "steps": args.steps, "warmup": args.warmup}
    rng = np.random.default_rng(7)
    streams = rng.integers(0, sh.vocab, size=(max(ROWS), ctx), dtype=np.int64)

    # parity gate: every row of an 8-row batch against the single-sequence decode of its own stream
    P = args.parity_steps
    got_ids, got_lg0 = [], None
    for pos in range(P):
        ids, lg = plan.forward_decode_batch(list(range(8)), [int(streams[r, pos]) for r in range(8)], [pos] * 8, logits=(pos == 0))
        got_ids.append([int(i) for i in ids])
        if pos == 0:
            got_lg0 = lg
    ok_ids, ok_lg = True, True
    for r in range(8):
        plan.kv_reset()
        for pos in range(P):
            lg, am = plan.forward_decode(int(streams[r, pos]), pos, logits=(pos == 0))
            ok_ids &= am == got_ids[pos][r]
            if pos == 0:
                ok_lg &= bool(np.array_equal(lg.view(np.uint32), got_lg0[r].view(np.uint32)))
    out["parity"] = {"rows": 8, "steps": P, "ids_equal": bool(ok_ids), "step0_logits_bit_equal": bool(ok_lg), "ok": bool(ok_ids and ok_lg)}

    res = {}
    for n in ROWS:
        # single-sequence b200_forward_decode on the same plan, then n rows per step
        for k in range(args.warmup):
            plan.forward_decode(int(streams[0, k]), k, logits=False)
        t0 = time.perf_counter()
        for k in range(args.steps):
            plan.forward_decode(int(streams[0, args.warmup + k]), args.warmup + k, logits=False)
        single_ms = (time.perf_counter() - t0) * 1e3 / args.steps
        slots = list(range(n))
        for k in range(args.warmup):
            plan.forward_decode_batch(slots, [int(streams[r, k]) for r in slots], [k] * n)
        dev = []
        t0 = time.perf_counter()
        for k in range(args.steps):
            p = args.warmup + k
            plan.forward_decode_batch(slots, [int(streams[r, p]) for r in slots], [p] * n)
            dev.append(plan.batch_info()[2])
        wall_ms = (time.perf_counter() - t0) * 1e3 / args.steps
        dev_ms = float(np.median(dev))
        b = step_bytes(sh, n, args.warmup + args.steps / 2)
        res[n] = {"device_ms_per_step": dev_ms, "wall_ms_per_step": wall_ms, "tok_s_device": n * 1e3 / dev_ms, "tok_s_wall": n * 1e3 / wall_ms,
                  "launches_per_step": plan.batch_info()[1], "roofline_ms_per_step": b["total"] / PEAK_BW * 1e3, "bytes_per_step": b,
                  "single_wall_ms_per_step": single_ms, "single_tok_s_wall": 1e3 / single_ms}
    out["rows"] = res
    out["speedup_8_vs_1_device"] = res[8]["tok_s_device"] / res[1]["tok_s_device"]
    out["speedup_8_vs_single_wall"] = res[8]["tok_s_wall"] / res[1]["single_tok_s_wall"]

    if args.profile:
        from torch.profiler import ProfilerActivity, profile

        slots = list(range(8))
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for k in range(4):
                plan.forward_decode_batch(slots, [int(streams[r, k]) for r in slots], [k] * 8)
        agg = {}
        for e in prof.events():
            if e.device_type.name == "CUDA":
                name = e.name.split("<")[0].split("(")[0]
                agg[name] = agg.get(name, 0.0) + e.device_time / 1e3 / 4
        out["profile_ms_per_8row_step"] = dict(sorted(agg.items(), key=lambda kv: -kv[1]))
    plan.free()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
