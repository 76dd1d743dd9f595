#!/usr/bin/env python
"""Granite-3.x-8B-shaped synthetic model (40 layers, 4096 / 12800, 32 / 8 heads, head 128, vocabulary 49155, tied classifier):
decode and prefill speed, and parity with the CPU restatement of forwardGranite (tests/granite_oracle.py).

    python tools/granite_bench.py [--tg 128] [--pp 512] [--reps 3] [--parity-steps 4] [--batch-steps 32]

Prints one JSON line:
  * Q8_0: tg<N> through b200_decode_sequence (greedy, device-resident loop) in the graph and the persistent decode mode; batched
    decode at 1, 2, 4 and 8 rows (device time of one step, aggregate tok/s); pp<N> in one chunk in the twin and the W8A16 mode;
  * FP16: tg<N> (graph) and pp<N> in the tensor-core mode;
  * parity, per weight format: the oracle's greedy ids for the first steps equal the plan's, and step 0's logits are bit-equal;
  * the GPU name and its power limit, read with one read-only nvidia-smi query in the same run."""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import __graft_entry__ as ge  # noqa: E402
from qwen2_bench import gpu_info  # noqa: E402


def parity(pkg, orc, plan, model, steps):
    from granite_oracle import GraniteOracle

    om = GraniteOracle(orc, model)
    tok, ids, ref_ids, logits0 = 1, [], [], None
    for pos in range(steps):
        lg, am = plan.forward_decode(tok, pos)
        ref = om.forward(tok, pos)
        if pos == 0:
            logits0 = bool(np.array_equal(lg.view(np.uint32), ref.view(np.uint32)))
        ids.append(int(am))
        ref_ids.append(orc.argmax(ref))
        tok = am
    om.close()
    plan.kv_reset()
    return {"steps": steps, "greedy_ids_equal": ids == ref_ids, "step0_logits_bit_equal": logits0, "ok": ids == ref_ids and logits0}


def tg(pkg, plan, sh, n, reps, modes):
    toks = np.asarray(pkg.llama_bench.synthetic_tokens(sh.vocab, 1), dtype=np.int32)
    out = {}
    for mode in modes:
        try:
            plan.set_decode_mode(mode)
        except pkg.native.UnsupportedOperation as e:
            out[mode] = {"unsupported": str(e)}
            continue
        plan.decode_sequence(toks, 8, 0, feedback=True)  # warm-up
        ms = [plan.decode_sequence(toks, n, 0, feedback=True)[1] for _ in range(reps)]
        out[mode] = {"tok_s": n / (float(np.median(ms)) / 1e3), "ms_per_token": float(np.median(ms)) / n}
    plan.set_decode_mode("graph")
    return out


def pp(pkg, plan, sh, n, reps, modes):
    ptoks = np.asarray(pkg.llama_bench.synthetic_tokens(sh.vocab, n), dtype=np.int32)
    out = {}
    for name, mode in modes:
        try:
            plan.set_prefill_mode(mode)
        except pkg.native.B200Error as e:
            out[name] = {"unsupported": str(e)}
            continue
        for _ in range(2):
            plan.forward_batch_prefill(ptoks, 0)
        d = []
        for _ in range(reps):
            plan.forward_batch_prefill(ptoks, 0)
            d.append(plan.prefill_info()[2])
        out[name] = {"tok_s": n / (float(np.median(d)) / 1e3), "ms_per_chunk": float(np.median(d))}
    return out


def batched(pkg, plan, sh, steps):
    plan.set_decode_slots(8)
    out = {}
    toks = [int(t) for t in pkg.llama_bench.synthetic_tokens(sh.vocab, 8)]
    for n in (1, 2, 4, 8):
        for s in range(8):
            plan.slot_reset(s)
        ms = []
        for step in range(steps + 4):
            ids, _ = plan.forward_decode_batch(list(range(n)), toks[:n], [step] * n)
            toks[:n] = [int(i) for i in ids]
            if step >= 4:  # the first steps warm up this row count's graph
                ms.append(plan.batch_info()[2])
        step_ms = float(np.median(ms))
        out[str(n)] = {"ms_per_step": step_ms, "tok_s_aggregate": n / (step_ms / 1e3)}
    plan.set_decode_slots(0)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tg", type=int, default=128)
    ap.add_argument("--pp", type=int, default=512)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--parity-steps", type=int, default=4)
    ap.add_argument("--batch-steps", type=int, default=32)
    args = ap.parse_args()
    import torch

    pkg, orc = ge.import_package(), ge.import_oracle()
    orc.use_all_cores()
    sh = pkg.synth.SHAPES["granite-3-8b"]
    G = pkg.gguf.GGMLType
    ctx = max(args.tg, args.pp, args.batch_steps + 4) + 8
    out = {"metric": "granite-3-8b", "workload": "Granite-3.x-8B-shaped synthetic (40 layers, 32/8 heads, head 128, vocab 49155, tied)",
           **gpu_info(), "torch_device": torch.cuda.get_device_name(0)}

    model = pkg.loader.model_from_tensors(sh, G.Q8_0, pkg.synth.build_tensors_fast(sh, G.Q8_0, seed=1234, device="cuda:0"), ctx)
    plan = pkg.B200MasterPlan.initialize_plan(model, prefill_batch_size=args.pp)
    out["q8_0"] = {"parity": parity(pkg, orc, plan, model, args.parity_steps),
                   "tg": {"n": args.tg, **tg(pkg, plan, sh, args.tg, args.reps, ("graph", "persistent"))},
                   "batched": batched(pkg, plan, sh, args.batch_steps),
                   "pp": {"n": args.pp, **pp(pkg, plan, sh, args.pp, args.reps, (("w8a16", "tensor_core_w8a16"), ("twin", "tensor_core")))}}
    plan.free()
    del model
    torch.cuda.empty_cache()

    model = pkg.loader.model_from_tensors(sh, G.F16, pkg.synth.build_tensors_fast(sh, G.F16, seed=1234, device="cuda:0"), ctx)
    plan = pkg.B200MasterPlan.initialize_plan(model, prefill_batch_size=args.pp)
    out["fp16"] = {"parity": parity(pkg, orc, plan, model, args.parity_steps),
                   "tg": {"n": args.tg, **tg(pkg, plan, sh, args.tg, args.reps, ("graph",))},
                   "pp": {"n": args.pp, **pp(pkg, plan, sh, args.pp, args.reps, (("fp16", "tensor_core"),))}}
    plan.free()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
