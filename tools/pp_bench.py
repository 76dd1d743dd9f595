"""pp<N> on the tensor-core batched prefill: usage python tools/pp_bench.py [shape] [n_tokens] [reps]"""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from __graft_entry__ import import_oracle, import_package  # noqa: E402

pkg = import_package()
orc = import_oracle()
shape = sys.argv[1] if len(sys.argv) > 1 else "llama-3-8b"
n = int(sys.argv[2]) if len(sys.argv) > 2 else 512
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 5
sh = pkg.synth.SHAPES[shape]
F16 = pkg.gguf.GGMLType.F16
t0 = time.time()
m = pkg.loader.model_from_tensors(sh, F16, pkg.synth.build_tensors_fast(sh, F16, seed=1234), n + 8)
t1 = time.time()
plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=n)
t2 = time.time()
toks = orc.bench_tokens(sh.vocab, n)
ms = []
for r in range(reps + 2):
    w0 = time.time()
    plan.forward_batch_prefill(toks, 0)
    w1 = time.time()
    info = plan.prefill_info()
    if r >= 2:
        ms.append((info[2], (w1 - w0) * 1e3))
dev = float(np.mean([a for a, _ in ms]))
wall = float(np.mean([b for _, b in ms]))
gemm_flops = 2.0 * sh.n_layers * (2 * sh.q_dim * sh.dim + 2 * sh.kv_dim * sh.dim + 3 * sh.hidden * sh.dim) * n
att_flops = 4.0 * sh.q_dim * sh.n_layers * (n * (n + 1) / 2)
rec = {"shape": shape, "n": n, "mode": info[0], "launches": info[1], "device_ms": dev, "wall_ms": wall, "tok_s_device": n / dev * 1e3, "tok_s_e2e": n / wall * 1e3,
       "tflops": (gemm_flops + att_flops) / (dev * 1e-3) / 1e12, "gemm_tflop": gemm_flops / 1e12, "att_tflop": att_flops / 1e12, "build_s": t1 - t0, "plan_s": t2 - t1}
print(json.dumps(rec), flush=True)
os.makedirs("results", exist_ok=True)
json.dump(rec, open(f"results/pp_bench_{shape}_{n}.json", "w"), indent=1)
plan.free()
