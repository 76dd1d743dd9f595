#!/usr/bin/env python
"""Qwen2.5-7B-shaped synthetic Q8_0 model (28 layers, 28 / 4 heads, GQA ratio 7, vocabulary 152064): decode and prefill speed,
and parity with the CPU restatement of forwardJavaQwen2 (tests/qwen2_oracle.py).

    python tools/qwen2_bench.py [--tg 128] [--pp 512] [--reps 3] [--parity-steps 4]

Prints one JSON line:
  * tg<N> through b200_decode_sequence (greedy, device-resident loop) in the graph and the persistent decode mode;
  * pp<N> in one chunk in the tensor-core twin mode and the W8A16 mode;
  * the whole-step HBM roofline: bytes one decode step must read (Q8_0 matrices at 34/32 bytes per weight, the biases, the norm
    weights, the KV rows of the mean tg position) over the card's peak bandwidth (3.35 TB/s, H100 SXM data sheet);
  * parity: the oracle's greedy ids for the first steps equal the plan's, and step 0's logits are bit-equal;
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


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": limit}
    except Exception as e:  # noqa: BLE001
        return {"gpu": None, "power_limit": None, "nvidia_smi_error": str(e)}


def step_bytes(sh, pos: int) -> int:
    w = sh.matmul_elements() * 34 // 32                        # Q8_0 matrices and classifier
    small = sh.n_layers * (sh.q_dim + 2 * sh.kv_dim + 2 * sh.dim) * 4 + sh.dim * 4  # biases, norms, final norm
    kv = sh.n_layers * 2 * (pos + 1) * sh.kv_dim * 4           # the FP32 K / V rows attention reads
    return w + small + kv


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tg", type=int, default=128)
    ap.add_argument("--pp", type=int, default=512)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--parity-steps", type=int, default=4)
    args = ap.parse_args()
    import torch

    pkg, orc = ge.import_package(), ge.import_oracle()
    from qwen2_oracle import Qwen2Oracle

    info = gpu_info()
    sh = pkg.synth.SHAPES["qwen2.5-7b"]
    Q8 = pkg.gguf.GGMLType.Q8_0
    ctx = max(args.tg, args.pp) + 8
    model = pkg.loader.model_from_tensors(sh, Q8, pkg.synth.build_tensors_fast(sh, Q8, seed=1234, device="cuda:0"), ctx)
    plan = pkg.B200MasterPlan.initialize_plan(model, prefill_batch_size=args.pp)
    out = {"metric": "qwen2.5-7b_q8_0", "workload": "Qwen2.5-7B-shaped synthetic Q8_0 (28 layers, 28/4 heads, vocab 152064)", **info,
           "torch_device": torch.cuda.get_device_name(0)}

    # parity first, on a fresh KV cache: greedy ids of the first steps and step 0's logits
    om = Qwen2Oracle(orc, model)
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
    om.close()
    out["parity"] = {"steps": args.parity_steps, "greedy_ids_equal": ids == ref_ids, "step0_logits_bit_equal": logits0,
                     "ok": ids == ref_ids and logits0}

    # tg<N>: decode_sequence with greedy feedback, each mode
    toks = np.asarray(pkg.llama_bench.synthetic_tokens(sh.vocab, 1), dtype=np.int32)
    tg = {}
    for mode in ("graph", "persistent"):
        try:
            plan.set_decode_mode(mode)
        except pkg.native.UnsupportedOperation as e:
            tg[mode] = {"unsupported": str(e)}
            continue
        plan.decode_sequence(toks, 8, 0, feedback=True)  # warm-up
        ms = [plan.decode_sequence(toks, args.tg, 0, feedback=True)[1] for _ in range(args.reps)]
        tg[mode] = {"tok_s": args.tg / (float(np.median(ms)) / 1e3), "ms_per_token": float(np.median(ms)) / args.tg}
    plan.set_decode_mode("graph")
    roof = step_bytes(sh, args.tg // 2) / PEAK_BW * 1e3
    out["tg"] = {"n": args.tg, **tg, "roofline_ms_per_token": roof, "roofline_tok_s": 1e3 / roof, "bytes_per_step": step_bytes(sh, args.tg // 2)}

    # pp<N>: one chunk from depth 0, each tensor-core mode
    ptoks = np.asarray(pkg.llama_bench.synthetic_tokens(sh.vocab, args.pp), dtype=np.int32)
    pp = {}
    for name, mode in (("w8a16", "tensor_core_w8a16"), ("twin", "tensor_core")):
        try:
            plan.set_prefill_mode(mode)
        except pkg.native.B200Error as e:
            pp[name] = {"unsupported": str(e)}
            continue
        for _ in range(2):
            plan.forward_batch_prefill(ptoks, 0)
        d = []
        for _ in range(args.reps):
            plan.forward_batch_prefill(ptoks, 0)
            d.append(plan.prefill_info()[2])
        pp[name] = {"tok_s": args.pp / (float(np.median(d)) / 1e3), "ms_per_chunk": float(np.median(d)), "device_bytes": plan.device_bytes}
    out["pp"] = {"n": args.pp, **pp}
    plan.free()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
