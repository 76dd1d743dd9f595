#!/usr/bin/env python
"""Qwen1.5-MoE-A2.7B-shaped synthetic Q8_0 model (24 layers, 16 heads, 60 experts, top-4, expert hidden 1408, shared hidden 5632,
vocabulary 151936), generated on the device: decode speed and parity with the CPU restatement of forwardJavaQwen2MoE
(tests/qwen2moe_oracle.py).

    python tools/moe_bench.py [--tg 128] [--reps 3] [--parity-steps 3] [--profile-steps 16]

Prints one JSON line:
  * tg<N> through b200_decode_sequence (greedy, device-resident loop) in graph mode (the only decode mode of an MoE plan);
  * the whole-step HBM roofline on the ACTIVE bytes of one token: the Q8_0 matrices a token reads (attention, the shared expert,
    k routed experts, the classifier; 34/32 bytes per weight), the F32 routers and shared gates, biases, norms and the KV rows of
    the mean tg position, over the card's peak bandwidth (3.35 TB/s, H100 SXM data sheet);
  * a torch.profiler split of the decode step by kernel family (router, expert gate/up, expert down, the dense streams, attention,
    norms, the rest), in microseconds per token -- launch-to-exit durations, which overlap under programmatic dependent launch;
  * parity: the plan's greedy ids for the first steps equal the oracle's, step 0's logits are bit-equal, and the last parity step's
    routing (ids and weights of every layer) is bit-equal;
  * the GPU name and its power limit, read with one read-only nvidia-smi query in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import __graft_entry__ as ge  # noqa: E402

PEAK_BW = 3.35e12
FAMILIES = (("route", "k_moe_route"), ("expert_gateup", "k_moe_gateup"), ("expert_down", "k_moe_down"),
            ("dense_streams (qkv, attn out, lm_head)", "k_stream_matvec_q8"), ("attention", "k_attention"), ("norms", "k_rmsnorm"))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": limit}
    except Exception as e:  # noqa: BLE001
        return {"gpu": None, "power_limit": None, "nvidia_smi_error": str(e)}


def step_bytes(sh, pos: int) -> dict:
    """Bytes one decode step must read: only the k routed experts of each layer count (the active weights)."""
    w = sh.matmul_elements() * 34 // 32  # attention + shared expert + k routed experts per layer, classifier
    routers = sh.n_layers * (sh.n_experts + 1) * sh.dim * 4
    small = sh.n_layers * (sh.q_dim + 2 * sh.kv_dim + 2 * sh.dim) * 4 + sh.dim * 4
    kv = sh.n_layers * 2 * (pos + 1) * sh.kv_dim * 4
    return {"q8_0_weights": w, "routers": routers, "biases_norms": small, "kv": kv, "total": w + routers + small + kv}


def profile_split(plan, toks, n):
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        plan.decode_sequence(toks, n, 0, feedback=True)
        torch.cuda.synchronize()
    split = {name: 0.0 for name, _ in FAMILIES}
    split["other"] = 0.0
    seen = 0
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        seen += 1
        for name, key in FAMILIES:
            if key in ev.name:
                split[name] += us
                break
        else:
            split["other"] += us
    if not seen:
        return {"error": "the profiler recorded no device kernels"}
    return {k: v / n for k, v in split.items()} | {"unit": "us per token", "kernels_recorded": seen,
                                                   "note": "kernel durations from launch to exit; under programmatic dependent launch a kernel "
                                                           "is resident (and counted) while it waits for its predecessor, so the families "
                                                           "overlap and sum past the step time"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tg", type=int, default=128)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--parity-steps", type=int, default=3)
    ap.add_argument("--profile-steps", type=int, default=16)
    args = ap.parse_args()
    import torch

    pkg, orc = ge.import_package(), ge.import_oracle()
    from qwen2moe_oracle import Qwen2MoEOracle

    info = gpu_info()
    sh = pkg.synth.SHAPES["qwen1.5-moe-a2.7b"]
    Q8 = pkg.gguf.GGMLType.Q8_0
    ctx = max(args.tg, args.profile_steps, args.parity_steps) + 8
    model = pkg.loader.model_from_tensors(sh, Q8, pkg.synth.build_tensors_fast(sh, Q8, seed=1234, device="cuda:0"), ctx)
    torch.cuda.empty_cache()
    plan = pkg.B200MasterPlan.initialize_plan(model)
    out = {"metric": "qwen1.5-moe-a2.7b_q8_0", "workload": "Qwen1.5-MoE-A2.7B-shaped synthetic Q8_0 (24 layers, 60 experts, top-4, vocab 151936)",
           **info, "torch_device": torch.cuda.get_device_name(0), "launches_per_token": plan.launches_per_decode,
           "device_bytes": plan.device_bytes}

    # parity first, on a fresh KV cache
    om = Qwen2MoEOracle(orc, model)
    orc.use_all_cores()
    tok, ids, ref_ids, logits0 = 1, [], [], None
    for pos in range(args.parity_steps):
        lg, am = plan.forward_decode(tok, pos)
        ref = om.forward(tok, pos)
        if pos == 0:
            logits0 = bool(np.array_equal(lg.view(np.uint32), ref.view(np.uint32)))
        ids.append(int(am))
        ref_ids.append(orc.argmax(ref))
        tok = am
    rid, rw = plan.moe_routing()
    routing = all(np.array_equal(rid[l], om.routing[l][0]) and np.array_equal(rw[l, :-1].view(np.uint32), om.routing[l][1].view(np.uint32))
                  and rw[l, -1].view(np.uint32) == np.float32(om.routing[l][2]).view(np.uint32) for l in range(sh.n_layers))
    om.close()
    out["parity"] = {"steps": args.parity_steps, "greedy_ids_equal": ids == ref_ids, "step0_logits_bit_equal": logits0,
                     "last_step_routing_bit_equal": bool(routing), "ok": ids == ref_ids and logits0 and bool(routing)}

    # tg<N>: decode_sequence with greedy feedback
    toks = np.asarray(pkg.llama_bench.synthetic_tokens(sh.vocab, 1), dtype=np.int32)
    plan.kv_reset()
    plan.decode_sequence(toks, 8, 0, feedback=True)  # warm-up
    ms = [plan.decode_sequence(toks, args.tg, 0, feedback=True)[1] for _ in range(args.reps)]
    med = float(np.median(ms))
    b = step_bytes(sh, args.tg // 2)
    roof = b["total"] / PEAK_BW * 1e3
    out["tg"] = {"n": args.tg, "decode_mode": "graph", "tok_s": args.tg / (med / 1e3), "ms_per_token": med / args.tg, "runs_ms": ms,
                 "roofline_ms_per_token": roof, "roofline_frac": roof / (med / args.tg), "active_bytes_per_step": b}
    out["profile"] = profile_split(plan, toks, args.profile_steps)
    plan.free()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
