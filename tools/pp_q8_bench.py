#!/usr/bin/env python
"""pp<N> on the Llama-3-8B-shaped Q8_0 model in the two tensor-core prefill modes, on ONE plan, chunks alternating:
W8A16 (B200_PREFILL_TENSOR_CORE_W8A16: the GEMMs read the Q8_0 weights in place, dequantised in shared memory) and twin
mode (B200_PREFILL_TENSOR_CORE: f16 copies of every matrix).

    python tools/pp_q8_bench.py [--pp-size 512] [--reps 5] [--dump-outputs DIR]

Prints one JSON line.  Per mode: tok/s and ms per chunk (CUDA events on the plan's stream), and the plan's device bytes
once the mode has been enabled (W8A16 first, so its bytes exclude the twins); then the max relative difference of the last
layer's K / V between the modes (0 where no residual GEMM splits K).  --dump-outputs writes the W8A16 K / V as .npy."""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as ge  # noqa: E402

MODES = {"w8a16": "tensor_core_w8a16", "twin": "tensor_core"}
KV = ("key_cache", "value_cache")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pp-size", type=int, default=512, help="tokens in the one chunk (= --batch-prefill-size)")
    ap.add_argument("--reps", type=int, default=5, help="timed chunks per mode (after 2 untimed rounds)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None, help="write the W8A16 last-layer K / V as DIR/<name>.npy")
    args = ap.parse_args()
    import torch

    pkg = ge.import_package()
    shape = pkg.synth.SHAPES["llama-3-8b"]
    Q8 = pkg.gguf.GGMLType.Q8_0
    n = args.pp_size
    model = pkg.loader.model_from_tensors(shape, Q8, pkg.synth.build_tensors_fast(shape, Q8, seed=1234, device="cuda:0"), n + 8)
    plan = pkg.B200MasterPlan.initialize_plan(model, prefill_batch_size=n)
    toks = np.asarray(pkg.llama_bench.synthetic_tokens(shape.vocab, n), dtype=np.int32)
    base = plan.device_bytes
    dev_bytes, dev, kv = {}, {k: [] for k in MODES}, {}
    for name, mode in MODES.items():
        plan.set_prefill_mode(mode)
        dev_bytes[name] = plan.device_bytes
    nkv = n * shape.kv_dim
    for r in range(2 + args.reps):
        for name, mode in MODES.items():
            plan.set_prefill_mode(mode)
            plan.forward_batch_prefill(toks, 0)
            if r >= 2:
                dev[name].append(plan.prefill_info()[2])
            if r == 1 + args.reps:
                kv[name] = {c: plan.read_buffer(c, nkv, layer=shape.n_layers - 1) for c in KV}
    plan.free()
    diff = {}
    for c in KV:
        ref = kv["twin"][c].astype(np.float64)
        diff[c] = float(np.max(np.abs(kv["w8a16"][c] - ref)) / np.max(np.abs(ref)))
    out = {"metric": "prefill_tokens_per_s", "pp": n, "reps": args.reps, "device": torch.cuda.get_device_name(0),
           "workload": f"Llama-3-8B-shaped synthetic GGUF, Q8_0, pp{n} in one chunk from depth 0, KV cache only; the modes alternate on one plan",
           "device_bytes_before_prefill": base, "max_rel_diff_last_layer_kv": diff}
    for name in MODES:
        d = float(np.mean(dev[name]))
        out[name] = {"tok_s": n / d * 1e3, "ms_per_chunk": d, "device_bytes": dev_bytes[name]}
    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        for c in KV:
            np.save(os.path.join(args.dump_outputs, f"pp{n}_w8a16_{c}_last_layer.npy"), kv["w8a16"][c])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
