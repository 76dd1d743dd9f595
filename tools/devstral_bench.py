#!/usr/bin/env python
"""Devstral-Small-2-shaped synthetic model (40 layers, 5120 / 32768, 32 / 8 heads of 128 so q is 4096 wide, vocabulary 131072, YaRN
RoPE table): decode and prefill speed, and parity with the CPU restatement of forwardJavaDevstral (tests/devstral_oracle.py).

    python tools/devstral_bench.py [--tg 128] [--pp 512] [--reps 3] [--parity-steps 2] [--batch-steps 32] [--skip-fp16]

Prints one JSON line:
  * Q8_0: tg<N> through b200_decode_sequence in the graph and the persistent decode mode; batched decode at 1, 2, 4 and 8 rows;
    pp<N> in one chunk in the W8A16 mode and the twin mode (the twin mode's f16 copies need about 45 GB more; a plan that cannot
    allocate them reports why);
  * FP16: tg<N> (graph), when the host has the memory to generate the 47 GB of weights;
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
from granite_bench import batched, pp, tg  # noqa: E402
from qwen2_bench import gpu_info  # noqa: E402


def parity(orc, plan, model, steps):
    from devstral_oracle import DevstralOracle

    om = DevstralOracle(orc, model)
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


def host_available_bytes() -> int:
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tg", type=int, default=128)
    ap.add_argument("--pp", type=int, default=512)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--parity-steps", type=int, default=2)
    ap.add_argument("--batch-steps", type=int, default=32)
    ap.add_argument("--skip-fp16", action="store_true")
    args = ap.parse_args()
    import torch

    pkg, orc = ge.import_package(), ge.import_oracle()
    orc.use_all_cores()
    sh = pkg.synth.SHAPES["devstral-small-2"]
    G = pkg.gguf.GGMLType
    ctx = max(args.tg, args.pp, args.batch_steps + 4) + 8
    out = {"metric": "devstral-small-2", "workload": "Devstral-Small-2-shaped synthetic (40 layers, 5120/32768, 32/8 heads of 128, qd 4096, "
                                                     "vocab 131072, YaRN)", **gpu_info(), "torch_device": torch.cuda.get_device_name(0)}

    model = pkg.loader.model_from_tensors(sh, G.Q8_0, pkg.synth.build_tensors_fast(sh, G.Q8_0, seed=1234, device="cuda:0"), ctx)
    plan = pkg.B200MasterPlan.initialize_plan(model, prefill_batch_size=args.pp)
    out["q8_0"] = {"parity": parity(orc, plan, model, args.parity_steps),
                   "weight_bytes_per_token": int(sh.matmul_elements() // 32 * 34),
                   "tg": {"n": args.tg, **tg(pkg, plan, sh, args.tg, args.reps, ("graph", "persistent"))},
                   "batched": batched(pkg, plan, sh, args.batch_steps),
                   "pp": {"n": args.pp, **pp(pkg, plan, sh, args.pp, args.reps, (("w8a16", "tensor_core_w8a16"), ("twin", "tensor_core")))}}
    plan.free()
    del model
    torch.cuda.empty_cache()

    need = 2 * sh.matmul_elements() + 2 * sh.vocab * sh.dim  # f16 matrices and the embedding table, generated on the host
    if args.skip_fp16 or host_available_bytes() < 1.2 * need:
        out["fp16"] = {"not_measured": f"needs about {need / 1e9:.0f} GB of host memory for the weights (available "
                                       f"{host_available_bytes() / 1e9:.0f} GB)" if not args.skip_fp16 else "--skip-fp16"}
    else:
        model = pkg.loader.model_from_tensors(sh, G.F16, pkg.synth.build_tensors_fast(sh, G.F16, seed=1234, device="cuda:0"), ctx)
        plan = pkg.B200MasterPlan.initialize_plan(model)
        out["fp16"] = {"parity": parity(orc, plan, model, args.parity_steps),
                       "tg": {"n": args.tg, **tg(pkg, plan, sh, args.tg, args.reps, ("graph",))}}
        plan.free()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
