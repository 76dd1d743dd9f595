#!/usr/bin/env python
"""Several positions of one sequence per weight stream, on bench.py's synthetic Llama-3-8B Q8_0 model:

  (a) the exact prefill of one --chunk-token chunk (forward_batch_prefill: multi-position steps, then the last token through the
      single-token graph) against --chunk one-token forward_batch_prefill calls (the token-by-token path);
  (b) one forward_decode_multi step at n = 1, 2, 4, 8 on the plan's own cache;
  (c) generate_tokens_lookahead with an oracle draft (every draft right: the upper bound) and with prompt_lookup, against
      generate_tokens_llama driven by forward_decode, with the acceptance rate.

    python tools/multi_position_bench.py [--ctx 2048] [--chunk 512] [--gen 96] [--reps 3]

Prints one JSON line.  Wall-clock ms are medians of --reps after one warm-up; every call ends in a device synchronise.  Parity gate,
in the same run: the K/V of layers 0 and L-1 after the chunk equals (uint32) the token-by-token path's, every multi-step row's id
equals forward_decode's, and both lookahead runs return the ids of generate_tokens_llama.  The GPU name and power limit come from
one read-only nvidia-smi query in the same run."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import __graft_entry__ as ge  # noqa: E402
from batch_decode_bench import gpu_info  # noqa: E402


def timed(fn, reps):
    fn()
    walls = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        walls.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(walls)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ctx", type=int, default=2048)
    ap.add_argument("--chunk", type=int, default=512)
    ap.add_argument("--gen", type=int, default=96)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    pkg = ge.import_package()
    E = pkg.engine
    info = gpu_info()
    sh = pkg.synth.SHAPES["llama-3-8b"]
    Q8 = pkg.gguf.GGMLType.Q8_0
    model = pkg.loader.model_from_tensors(sh, Q8, pkg.synth.build_tensors_fast(sh, Q8, seed=1234, device="cuda:0"), args.ctx)
    plan = pkg.B200MasterPlan.initialize_plan(model)
    c = model.configuration
    R = plan.decode_multi_rows()
    rng = np.random.default_rng(5)
    toks = rng.integers(0, sh.vocab, args.ctx).astype(np.int32)
    n = args.chunk
    out = {"metric": "llama-3-8b_q8_0_multi_position", "workload": f"llama-3-8b-shaped synthetic Q8_0, {sh.n_layers} layers, ctx {args.ctx}",
           **info, "reps": args.reps, "rows_per_step": R}
    parity = {}

    def kv_of(layers):
        nkv = c.context_length * c.kv_dim
        return [plan.read_buffer(b, nkv, layer=l).view(np.uint32).copy() for b in ("key_cache", "value_cache") for l in layers]

    def prefill_chunk():
        plan.forward_batch_prefill(toks[:n], 0)

    def prefill_tokens():
        for p in range(n):
            plan.forward_batch_prefill(toks[p:p + 1], p)

    layers = [0, c.n_layers - 1]
    plan.kv_reset()
    prefill_tokens()
    want = kv_of(layers)
    plan.kv_reset()
    prefill_chunk()
    parity["prefill_kv_equal"] = all(np.array_equal(a, b) for a, b in zip(kv_of(layers), want))
    res = {}
    wall = timed(prefill_chunk, args.reps)
    res["exact_prefill_chunk"] = {"tokens": n, "wall_ms": wall, "tok_s": n * 1e3 / wall, "ms_per_token": wall / n}
    wall = timed(prefill_tokens, 1)
    res["one_token_calls"] = {"tokens": n, "wall_ms": wall, "tok_s": n * 1e3 / wall, "ms_per_token": wall / n}

    # (b) one step at n rows, positions n .. on top of the chunk; ids against forward_decode
    start = n
    ids, _ = plan.forward_decode_multi(-1, toks[start:start + R], start)
    single = [plan.forward_decode(int(toks[start + i]), start + i, logits=False)[1] for i in range(R)]
    parity["multi_ids_equal"] = [int(i) for i in ids] == [int(i) for i in single]
    steps = {}
    for k in (1, 2, 4, 8):
        if k > R:
            continue
        wall = timed(lambda: plan.forward_decode_multi(-1, toks[start:start + k], start), max(args.reps, 10))
        steps[str(k)] = {"wall_ms": wall, "ms_per_position": wall / k}
    res["forward_decode_multi"] = steps

    # (c) generation after a 64-token prompt whose second half repeats its first (so prompt lookup has something to find)
    half = [int(t) for t in toks[:32]]
    prompt = half + half
    budget = len(prompt) + 1 + args.gen

    def loop():
        return E.generate_tokens_llama(lambda t, p: plan.forward_decode(t, p, logits=False)[1], 1, 0, prompt, [], budget, c.context_length)

    ref = loop()
    full = [1] + prompt + ref
    gen = {}
    wall = timed(loop, 1)
    gen["generate_tokens_llama"] = {"wall_ms": wall, "tok_s": (len(prompt) + len(ref)) * 1e3 / wall}
    for name, draft in (("oracle_draft", lambda h: full[len(h):len(h) + R]), ("prompt_lookup", E.prompt_lookup)):
        stats = {}
        got = E.generate_tokens_lookahead(plan, "LLAMA_3", 1, 0, prompt, [], budget, c.context_length, draft=draft, stats=stats)
        parity[f"lookahead_{name}_equal"] = got == ref
        wall = timed(lambda: E.generate_tokens_lookahead(plan, "LLAMA_3", 1, 0, prompt, [], budget, c.context_length, draft=draft), 1)
        gen[name] = {"wall_ms": wall, "tok_s": (len(prompt) + len(ref)) * 1e3 / wall, "steps": stats["steps"],
                     "acceptance": stats["accepted"] / stats["drafted"] if stats["drafted"] else None}
    res["generation"] = {"prompt": len(prompt), "generated": len(ref), **gen}
    out["parity"] = {**parity, "ok": all(parity.values())}
    out["results"] = res
    plan.free()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
