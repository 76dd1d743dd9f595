#!/usr/bin/env python
"""Token scoring (b200_score_tokens) on the Llama-3-8B-shaped Q8_0 model of bench.py, 512-token chunks, on ONE plan:

  score_<mode>    plan.score_tokens of the chunk in the exact and tensor_core_exact prefill modes
  prefill_<mode>  plan.forward_batch_prefill of the same chunk in the same mode (no logits): the classifier's cost is the difference
  decode_loop     what a user writes without score_tokens: forward_decode per token with its logits row copied to the host and a
                  float64 log-softmax in numpy (--decode-tokens tokens, rate per token)

    python tools/score_bench.py [--chunk 512] [--reps 3] [--decode-tokens 128]

Prints one JSON line: the card's name, power limit and max SM clock (nvidia-smi, read in the same run), ms per call (host clock around
calls that end in a stream synchronise; median of --reps after one untimed round) and tok/s.  Parity gate: both modes' logprobs and
ids bit-equal, and within 1e-9 (ids equal) of the decode loop's for the positions it covers; a mismatch exits with status 1."""
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

MODES = ("exact", "tensor_core_exact")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def rate(n, ms):
    return {"ms": round(float(np.median(ms)), 3), "tok_s": round(n / (float(np.median(ms)) / 1e3), 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunk", type=int, default=512)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--decode-tokens", type=int, default=128)
    args = ap.parse_args()
    n = args.chunk
    pkg = ge.import_package()
    shape = pkg.synth.SHAPES["llama-3-8b"]
    Q8 = pkg.gguf.GGMLType.Q8_0
    model = pkg.loader.model_from_tensors(shape, Q8, pkg.synth.build_tensors_fast(shape, Q8, seed=1234, device="cuda:0"), n + 8)
    plan = pkg.B200MasterPlan.initialize_plan(model, prefill_batch_size=n)
    toks = np.asarray(pkg.llama_bench.synthetic_tokens(shape.vocab, n + 1), dtype=np.int32)
    out = {"card": card(), "model": "llama-3-8b Q8_0 (synthetic)", "chunk": n}
    ms = {}
    scores = {}
    for r in range(1 + args.reps):
        for mode in MODES:
            plan.set_prefill_mode(mode)
            for what in ("score", "prefill"):
                plan.kv_reset()
                t0 = time.perf_counter()
                if what == "score":
                    scores[mode] = plan.score_tokens(toks[:n], 0, toks[1:n + 1])
                else:
                    plan.forward_batch_prefill(toks[:n], 0)
                if r:
                    ms.setdefault(f"{what}_{mode}", []).append((time.perf_counter() - t0) * 1e3)
    for k, v in ms.items():
        out[k] = rate(n, v)
    # the per-token loop: logits row to the host, float64 log-softmax there
    d = min(args.decode_tokens, n)
    plan.kv_reset()
    plan.forward_decode(int(toks[0]), 0)  # warm-up
    plan.kv_reset()
    lp_dec, ids_dec = np.empty(d), np.empty(d, np.int32)
    t0 = time.perf_counter()
    for p in range(d):
        lg, am = plan.forward_decode(int(toks[p]), p)
        x = lg.astype(np.float64)
        m = x.max()
        lp_dec[p] = (x[toks[p + 1]] - m) - np.log(np.exp(x - m).sum())
        ids_dec[p] = am
    out["decode_loop"] = {"tokens": d, **rate(d, [(time.perf_counter() - t0) * 1e3])}
    plan.free()
    a, b = scores["exact"], scores["tensor_core_exact"]
    ok = np.array_equal(a[0].view(np.uint64), b[0].view(np.uint64)) and np.array_equal(a[1], b[1])
    ok = ok and np.array_equal(b[1][:d], ids_dec) and float(np.abs(b[0][:d] - lp_dec).max()) <= 1e-9
    out["mean_logprob"] = round(float(b[0].mean()), 6)
    out["parity"] = "bit-equal" if ok else "MISMATCH"
    print(json.dumps(out))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
