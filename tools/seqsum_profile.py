"""Cycles of the exact RMSNorm sum (csrc/seqsum2.cuh) at 256 / 512 / 1024 threads, cold and warm instruction cache, on the
squares of a real residual row: the residual stream x of the synthetic Llama-3-8B Q8_0 model of bench.py after a few decode steps
(dim 4096), and that row extended by its own first 1024 values (dim 5120, the Devstral-Small-2 width).  Next to the cycles: the
items the resolver walked, how many of them were literal stretches, and how many runs were mispredicted and replayed.
Usage: python tools/seqsum_profile.py [steps] [repeats]"""
import os, subprocess, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge

pkg = ge.import_package()
steps = int(sys.argv[1]) if len(sys.argv) > 1 else 16
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip())
sh = pkg.synth.SHAPES["llama-3-8b"]
m = pkg.loader.model_from_tensors(sh, 8, pkg.synth.build_tensors_fast(sh, 8, seed=1234, device="cuda:0"), steps + 8)
plan = pkg.B200MasterPlan.initialize_plan(m, device=0)
toks = pkg.llama_bench.synthetic_tokens(sh.vocab, steps)
plan.decode_sequence(toks, steps, 0)
x = plan._native.read_buffer("x", sh.dim)
plan.free()
rows = {4096: x, 5120: np.concatenate([x, x[:1024]])}


def seq(t):
    s = np.float32(0)
    for v in t:
        s = np.float32(s + v)
    return s


print("dim   threads  cold cycles  warm cycles  items  literals  fallbacks   (median of %d launches)" % reps)
for dim, row in rows.items():
    sq = (row * row).astype(np.float32)
    ref = seq(sq)
    for T in (256, 512, 1024):
        runs = [pkg.native.profile_seqsum(sq, threads=T) for _ in range(reps)]
        for _, _, a, b, *_ in runs:
            assert np.float32(a).view(np.uint32) == ref.view(np.uint32) == np.float32(b).view(np.uint32), (dim, T, a, b, ref)
        cold = int(np.median([r[0] for r in runs]))
        warm = int(np.median([r[1] for r in runs]))
        items, lits, fbs = runs[-1][4:]
        print(f"{dim:5d} {T:8d} {cold:12d} {warm:12d} {items:6d} {lits:9d} {fbs:10d}")
