#!/usr/bin/env python
"""The bit-exact tensor-core prefill (B200_PREFILL_TENSOR_CORE_EXACT) on plans that keep K-quant weights resident (DESIGN.md sections
5b and 6).

    python tools/kq_prefill_bench.py [--pp 32,128,512] [--reps 3] [--ctx70 8192] [--skip-8b] [--skip-70b]

Prints one JSON line:
  * 8B: the synthetic Llama-3-8B-shaped Q4_K_M mix built resident (kq_resident_bench.resident_plan) and built as Q8_0 tiles from the
    same tensors, both with prefill_batch_size 512 in tensor_core_exact, chunks alternating between the two plans: ms per chunk
    (host clock around the call, which ends in a stream synchronise) and tok/s at each --pp length; the resident plan's exact prefill
    over one 512-token chunk; parity gate: after the resident tensor_core_exact chunk, the K / V of the first and last layer and the
    logits of the first decode step are bit-equal to those after the resident exact chunk (and to the Q8_0-tile plan's mode 3);
  * profile: a separate torch.profiler run of one resident pp512 chunk split into expansion (k_kq_tiles_to_q8), int8 GEMMs, attention
    (with RoPE / KV) and norms, the expansion's share of the chunk, and its achieved bytes/s (resident bytes read plus Q8_0 bytes
    written, computed from the shapes, over its kernel time);
  * 70B: the whole Llama-3-70B shape in the Q4_K_M mix on one GPU at context --ctx70 (kq_resident_bench.model_70b), prefill batch 512:
    pp512 in tensor_core_exact and the exact prefill of 32 tokens;
  * the GPU name and its power limit, read in the same run.
A parity mismatch exits with status 1."""
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
from kq_resident_bench import model_70b, resident_plan  # noqa: E402
from qwen2_bench import gpu_info  # noqa: E402

BATCH = 512
KB = {12: 144, 13: 176, 14: 210}


def resident_bytes(rows, cols, fmt):
    """Bytes of a resident K-quant stream (csrc/stream_matvec.cuh: segments of multiples of 256 columns, at most 2560)."""
    nseg = next(n for n in range(1, cols // 256 + 1) if cols % n == 0 and (cols // n) % 256 == 0 and cols // n <= 2560)
    return (rows + 3) // 4 * 4 * nseg * ((cols // nseg // 256 * KB[fmt] + 15) & ~15)


def expansion_bytes(pkg, sh):
    """Bytes one chunk's expansions move in the Q4_K_M mix, whose resident layer matrices are Wo (Q5_K), gate/up (Q4_K) and W2 (Q6_K):
    every resident byte read once plus every Q8_0 tile byte written, over all layers."""
    mats = [(sh.dim, sh.q_dim, 13), (2 * sh.hidden, sh.dim, 12), (sh.dim, sh.hidden, 14)]
    return sh.n_layers * sum(resident_bytes(r, c, f) + pkg.native.q8_tile_bytes(r, c) for r, c, f in mats)


def timed(plan, toks, start=0):
    t0 = time.perf_counter()
    plan.forward_batch_prefill(toks, start)
    return (time.perf_counter() - t0) * 1e3


def snapshot(plan, sh, n, tok):
    """K / V rows 0 .. n - 1 of the first and last layer, then the logits of the decode step at position n."""
    kv = [plan.read_buffer(c, n * sh.kv_dim, layer=l).copy() for c in ("key_cache", "value_cache") for l in (0, sh.n_layers - 1)]
    lg, _ = plan.forward_decode(int(tok), n)
    return kv + [lg.copy()]


def same(a, b):
    return all(np.array_equal(x.view(np.uint32), y.view(np.uint32)) for x, y in zip(a, b))


def bench_8b(pkg, args, pp):
    sh = pkg.synth.SHAPES["llama-3-8b"]
    tensors = pkg.synth.build_tensors_kquant(sh, seed=1234, mix="Q4_K_M")
    model = pkg.loader.model_from_tensors(sh, pkg.gguf.GGMLType.Q8_0, tensors, BATCH + 8)
    toks = np.asarray(pkg.llama_bench.synthetic_tokens(sh.vocab, BATCH + 1), dtype=np.int32)
    plans = {"resident": resident_plan(pkg, model, prefill_batch_size=BATCH), "q8_0": pkg.B200MasterPlan.initialize_plan(model, prefill_batch_size=BATCH)}
    out = {"workload": "Llama-3-8B-shaped synthetic, Q4_K_M mix (Q4_K, Q5_K Wo, Q6_K attn_v / ffn_down / classifier / embedding)", "pp": {}}
    res = plans["resident"]
    try:
        assert res.weight_info()["resident"] and not plans["q8_0"].weight_info()["resident"]
        out["weight_info"] = {k: p.weight_info() for k, p in plans.items()}
        # parity: the resident exact chunk first (the reference), then mode 3 on both plans
        res.set_prefill_mode("exact")
        out["resident_exact_pp512_ms"] = round(timed(res, toks[:BATCH]), 1)
        out["resident_exact_pp512_tok_s"] = round(BATCH / (out["resident_exact_pp512_ms"] / 1e3), 1)
        ref = snapshot(res, sh, BATCH, toks[BATCH])
        ok = True
        for name, plan in plans.items():
            plan.set_prefill_mode("tensor_core_exact")
            plan.kv_reset()
            plan.forward_batch_prefill(toks[:BATCH], 0)
            ok = ok and same(snapshot(plan, sh, BATCH, toks[BATCH]), ref)
        out["parity"] = "bit-equal" if ok else "MISMATCH"
        out["resident_launches_pp512"] = res.prefill_info()[1]
        for n in pp:
            ms = {k: [] for k in plans}
            dev = {k: [] for k in plans}
            for r in range(1 + args.reps):
                for name, plan in plans.items():
                    t = timed(plan, toks[:n])
                    if r:
                        ms[name].append(t)
                        dev[name].append(plan.prefill_info()[2])
            out["pp"][n] = {k: {"ms": round(float(np.median(v)), 3), "device_ms": round(float(np.median(dev[k])), 3),
                                "tok_s": round(n / (np.median(v) / 1e3), 1), "runs_ms": [round(x, 3) for x in v]} for k, v in ms.items()}
            out["pp"][n]["resident_over_q8_0"] = round(float(np.median(ms["resident"]) / np.median(ms["q8_0"])), 4)
        plans.pop("q8_0").free()
        out["profile_pp512"] = profile(pkg, sh, res, toks)
    finally:
        for plan in plans.values():
            plan.free()
    return out, ok


def profile(pkg, sh, plan, toks):
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile

    plan.forward_batch_prefill(toks[:BATCH], 0)
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        plan.forward_batch_prefill(toks[:BATCH], 0)
        torch.cuda.synchronize()
    split = {"expansion": 0.0, "gemm": 0.0, "attention": 0.0, "norm": 0.0, "other": 0.0}
    kinds = (("expansion", "k_kq_tiles_to_q8"), ("gemm", "k_gemm_i8"), ("attention", "k_i8_attention"), ("attention", "k_i8_rope_kv"),
             ("norm", "k_i8_norm"))
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        split[next((k for k, s in kinds if s in e.key), "other")] += us / 1e3
    total = sum(split.values())
    b = expansion_bytes(pkg, sh)
    return {"ms": {k: round(v, 3) for k, v in split.items()}, "expansion_share": round(split["expansion"] / total, 4),
            "expansion_bytes": b, "expansion_bytes_per_s": b / (split["expansion"] / 1e3) if split["expansion"] else None}


def bench_70b(pkg, args):
    model, out = model_70b(pkg, args.ctx70)
    if model is None:
        return out
    sh = pkg.synth.SHAPES["llama-3-70b"]
    try:
        plan = pkg.B200MasterPlan.initialize_plan(model, prefill_batch_size=BATCH)
    except pkg.native.B200Error as e:
        out["not_run"] = f"plan creation failed: {e}"
        return out
    try:
        out["form"] = "resident" if plan.weight_info()["resident"] else "q8_0"
        toks = np.asarray(pkg.llama_bench.synthetic_tokens(sh.vocab, BATCH), dtype=np.int32)
        plan.set_prefill_mode("exact")
        timed(plan, toks[:4])
        out["exact_pp32_ms"] = round(timed(plan, toks[:32]), 1)
        out["exact_pp32_tok_s"] = round(32 / (out["exact_pp32_ms"] / 1e3), 2)
        plan.set_prefill_mode("tensor_core_exact")
        timed(plan, toks[:BATCH])
        ms = [timed(plan, toks[:BATCH]) for _ in range(args.reps)]
        out["tensor_core_exact_pp512_ms"] = round(float(np.median(ms)), 1)
        out["tensor_core_exact_pp512_tok_s"] = round(BATCH / (np.median(ms) / 1e3), 1)
        out["runs_ms"] = [round(x, 1) for x in ms]
        out["launches"] = plan.prefill_info()[1]
    finally:
        plan.free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pp", default="32,128,512", help="chunk lengths (at most 512)")
    ap.add_argument("--reps", type=int, default=3, help="timed chunks per plan and length (after one untimed round)")
    ap.add_argument("--ctx70", type=int, default=8192)
    ap.add_argument("--skip-8b", action="store_true")
    ap.add_argument("--skip-70b", action="store_true")
    args = ap.parse_args()
    pp = [int(x) for x in args.pp.split(",")]
    if max(pp) > BATCH:
        ap.error(f"chunk lengths above the prefill batch size {BATCH}")
    pkg = ge.import_package()
    out = {"metric": "kq-resident-prefill", **gpu_info()}
    out["8b"], ok = ({"not_run": "--skip-8b"}, True) if args.skip_8b else bench_8b(pkg, args, pp)
    out["70b"] = {"not_run": "--skip-70b"} if args.skip_70b else bench_70b(pkg, args)
    print(json.dumps(out))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
