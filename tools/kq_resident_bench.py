#!/usr/bin/env python
"""Resident K-quant weights against their Q8_0 expansion (DESIGN.md sections 4, 6 and 10).

    python tools/kq_resident_bench.py [--tg 128] [--rounds 2] [--reps 3] [--parity-steps 4] [--tg70 32] [--ctx70 8192] [--skip-70b]

Prints one JSON line:
  * 8B: the synthetic Llama-3-8B-shaped Q4_K_M mix (synth.build_tensors_kquant), built resident (the free-memory figure of the
    residency rule set between the two forms with b200_test_set_memory_budget) and built as Q8_0 tiles from the same tensors.  tg<N>
    through b200_decode_sequence (greedy, device-resident loop), the two plans alternated for --rounds rounds of --reps runs each:
    tok/s, device ms per token, b200_weight_info, and the whole-step roofline (weight bytes streamed per token plus the K / V rows
    read, over the step's device time, against 3.35 TB/s).  Parity gate: the oracle on the re-quantised Q8_0 twin gives the plan's
    greedy ids for --parity-steps steps and step 0's logits bit-equal, for both forms;
  * 70B: the whole Llama-3-70B shape in the Q4_K_M mix on one GPU at context --ctx70, where the residency rule itself (no budget set)
    must pick the resident form: the form chosen, b200_weight_info and tg<--tg70>.  Every layer reuses layer 0's tensors (the device
    still holds 80 layers of weights; only the host copy is shared), so the host needs about 3 GB.  Parity at this geometry rests on
    the 2-layer cut in tests/test_gpu_kquant_resident.py: the C oracle cannot hold a 75 GB twin;
  * the GPU name and its power limit, read with one read-only nvidia-smi query in the same run."""
from __future__ import annotations

import argparse
import dataclasses
import json
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import __graft_entry__ as ge  # noqa: E402
from qwen2_bench import gpu_info  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def figures(pkg, model):
    """(bytes the Q8_0 form needs, bytes the resident form needs), from the creation that fits neither (budget 1 byte)."""
    pkg.native.test_set_memory_budget(1)
    try:
        pkg.B200MasterPlan.initialize_plan(model)
        raise RuntimeError("a plan was created under a 1-byte budget")
    except pkg.native.B200Error as e:
        m = re.search(r"(\d+) bytes with Q8_0 tiles and (\d+) bytes with K-quant weights resident", str(e))
        if not m:
            raise
        return int(m.group(1)), int(m.group(2))
    finally:
        pkg.native.test_set_memory_budget(0)


def resident_plan(pkg, model, **kw):
    q8, res = figures(pkg, model)
    pkg.native.test_set_memory_budget((q8 + res) // 2)
    try:
        return pkg.B200MasterPlan.initialize_plan(model, **kw)
    finally:
        pkg.native.test_set_memory_budget(0)


def parity(orc, plan, om, steps):
    tok, ids, ref_ids, logits0 = 1, [], [], None
    om.reset()
    for pos in range(steps):
        lg, am = plan.forward_decode(tok, pos)
        ref = om.forward(tok, pos)
        if pos == 0:
            logits0 = bool(np.array_equal(lg.view(np.uint32), ref.view(np.uint32)))
        ids.append(int(am))
        ref_ids.append(orc.argmax(ref))
        tok = am
    plan.kv_reset()
    return {"steps": steps, "greedy_ids_equal": ids == ref_ids, "step0_logits_bit_equal": logits0, "ok": ids == ref_ids and logits0}


def step_bytes(sh, weight_bytes: int, n: int) -> int:
    """Bytes one tg<n> step reads on average: the weight streams (the embedding planes are gathered one row per token) plus the
    F32 K / V rows attention reads, averaged over positions 0 .. n - 1."""
    emb = sh.vocab * sh.dim // 32 * 34
    kv = sh.n_layers * 2 * ((n + 1) / 2) * sh.kv_dim * 4
    return int(weight_bytes - emb + sh.dim // 32 * 34 + kv)


def tg_once(plan, toks, n):
    return plan.decode_sequence(toks, n, 0, feedback=True)[1]


def bench_8b(pkg, orc, args):
    sh = pkg.synth.SHAPES["llama-3-8b"]
    tensors = pkg.synth.build_tensors_kquant(sh, seed=1234, mix="Q4_K_M")
    model = pkg.loader.model_from_tensors(sh, pkg.gguf.GGMLType.Q8_0, tensors, args.tg + 16)
    plans = {"resident": resident_plan(pkg, model), "q8_0": pkg.B200MasterPlan.initialize_plan(model)}
    out = {"workload": "Llama-3-8B-shaped synthetic, Q4_K_M mix (Q4_K, Q5_K Wo, Q6_K attn_v / ffn_down / classifier / embedding)"}
    try:
        from test_gpu_kquants import _requantised_twin

        om = orc.OracleModel(_requantised_twin(pkg, orc, model))
        for name, plan in plans.items():
            out[name] = {"weight_info": plan.weight_info(), "parity": parity(orc, plan, om, args.parity_steps)}
        om.close()
        toks = np.asarray(pkg.llama_bench.synthetic_tokens(sh.vocab, 1), dtype=np.int32)
        for plan in plans.values():
            tg_once(plan, toks, 8)  # warm-up
        ms = {name: [] for name in plans}
        for _ in range(args.rounds):
            for name, plan in plans.items():
                ms[name] += [tg_once(plan, toks, args.tg) for _ in range(args.reps)]
        for name in plans:
            t = float(np.median(ms[name])) / args.tg
            b = step_bytes(sh, out[name]["weight_info"]["weight_bytes"], args.tg)
            out[name]["tg"] = {"n": args.tg, "tok_s": 1e3 / t, "ms_per_token": t, "runs_ms": ms[name], "bytes_per_step": b,
                               "roofline_whole_step": b / (t / 1e3) / HBM_BYTES_PER_S}
    finally:
        for plan in plans.values():
            plan.free()
    return out


def mem_available() -> int:
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def model_70b(pkg, ctx):
    """(model or None, report): the whole Llama-3-70B shape in the Q4_K_M mix, every layer reusing layer 0's host tensors; None with
    report["not_run"] when the host lacks the memory."""
    sh = pkg.synth.SHAPES["llama-3-70b"]
    one = pkg.synth.build_tensors_kquant(dataclasses.replace(sh, n_layers=1), seed=1234, mix="Q4_K_M")
    host = sum(np.asarray(r).nbytes for _, _, r in one.values())
    out = {"workload": f"Llama-3-70B shape (80 layers), Q4_K_M mix, one GPU, context {ctx}", "host_bytes": host}
    if host * 1.5 > mem_available():
        out["not_run"] = f"the host has {mem_available()} bytes available, the synthetic tensors need about {host}"
        return None, out
    tensors = {}
    for name, v in one.items():
        if name.startswith("blk.0."):
            for l in range(sh.n_layers):
                tensors[f"blk.{l}." + name[len("blk.0."):]] = v
        else:
            tensors[name] = v
    return pkg.loader.model_from_tensors(sh, pkg.gguf.GGMLType.Q8_0, tensors, ctx), out


def bench_70b(pkg, args):
    sh = pkg.synth.SHAPES["llama-3-70b"]
    model, out = model_70b(pkg, args.ctx70)
    if model is None:
        return out
    try:
        plan = pkg.B200MasterPlan.initialize_plan(model)
    except pkg.native.B200Error as e:
        out["not_run"] = f"plan creation failed: {e}"
        return out
    try:
        info = plan.weight_info()
        out["form"] = "resident" if info["resident"] else "q8_0"
        out["weight_info"] = info
        out["upload"] = plan.upload_info()
        toks = np.asarray(pkg.llama_bench.synthetic_tokens(sh.vocab, 1), dtype=np.int32)
        tg_once(plan, toks, 4)
        ms = [tg_once(plan, toks, args.tg70) for _ in range(args.reps)]
        t = float(np.median(ms)) / args.tg70
        b = step_bytes(sh, info["weight_bytes"], args.tg70)
        out["tg"] = {"n": args.tg70, "tok_s": 1e3 / t, "ms_per_token": t, "runs_ms": ms, "bytes_per_step": b,
                     "roofline_whole_step": b / (t / 1e3) / HBM_BYTES_PER_S}
    finally:
        plan.free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tg", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--parity-steps", type=int, default=4)
    ap.add_argument("--tg70", type=int, default=32)
    ap.add_argument("--ctx70", type=int, default=8192)
    ap.add_argument("--skip-70b", action="store_true")
    args = ap.parse_args()
    pkg, orc = ge.import_package(), ge.import_oracle()
    orc.use_all_cores()
    out = {"metric": "kq-resident", **gpu_info()}
    out["8b"] = bench_8b(pkg, orc, args)
    out["70b"] = {"not_run": "--skip-70b"} if args.skip_70b else bench_70b(pkg, args)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
