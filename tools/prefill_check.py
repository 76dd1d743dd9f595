"""Tensor-core batched prefill vs the CPU oracle (KV cache + next-token logits), with timings.
usage: python tools/prefill_check.py [shape ...]"""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from __graft_entry__ import import_oracle, import_package  # noqa: E402

pkg = import_package()
orc = import_oracle()

shapes = sys.argv[1:] or ["tiny-llama", "tiny-qwen3", "mid-llama"]
out = []
for shape in shapes:
    n_tok, batch = (160, 128) if shape.startswith("mid") else (50, 32)
    ctx = n_tok + 8
    sh = pkg.synth.SHAPES[shape]
    F16 = pkg.gguf.GGMLType.Q8_0 if os.environ.get("PREFILL_QUANT") == "q8" else pkg.gguf.GGMLType.F16
    m = pkg.loader.model_from_tensors(sh, F16, pkg.synth.build_tensors_fast(sh, F16, seed=1234), ctx)
    c = m.configuration
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=batch)
    if os.environ.get("PREFILL_QUANT") == "q8":
        plan.set_prefill_mode("tensor_core")
    mode = plan.prefill_info()[0]
    toks = orc.bench_tokens(c.vocab_size, n_tok + 1)
    t0 = time.time()
    for off in range(0, n_tok, batch):
        plan.forward_batch_prefill(toks[off:off + batch][: n_tok - off], off)
    info = plan.prefill_info()
    lg, am = plan.forward_decode(int(toks[n_tok]), n_tok)
    om = orc.OracleModel(m)
    for pos in range(n_tok):
        om.forward(int(toks[pos]), pos, want_logits=False)
    ref_lg = om.forward(int(toks[n_tok]), n_tok)
    rec = {"shape": shape, "mode": mode, "launches": info[1], "last_chunk_ms": info[2]}
    for l in range(c.n_layers):
        nkv = c.context_length * c.kv_dim
        for name in ("key_cache", "value_cache"):
            got = plan.read_buffer(name, nkv, layer=l)[: (n_tok + 1) * c.kv_dim]
            ref = (om.key_cache(l) if name == "key_cache" else om.value_cache(l))[: (n_tok + 1) * c.kv_dim]
            rec[f"{name}{l}_relmax"] = float(np.max(np.abs(got - ref)) / np.max(np.abs(ref)))
    rec["logit_relmax"] = float(np.max(np.abs(lg - ref_lg)) / np.max(np.abs(ref_lg)))
    rec["argmax_same"] = bool(int(np.argmax(ref_lg)) == am)
    # exact mode must still be bit-identical
    plan.set_prefill_mode("exact")
    plan.kv_reset()
    for off in range(0, n_tok, batch):
        plan.forward_batch_prefill(toks[off:off + batch][: n_tok - off], off)
    k0 = plan.read_buffer("key_cache", c.context_length * c.kv_dim, layer=c.n_layers - 1)
    nv = n_tok * c.kv_dim
    rec["exact_mode_bit_equal"] = bool(np.array_equal(k0.view(np.uint32)[:nv], om.key_cache(c.n_layers - 1).view(np.uint32)[:nv]))
    print(json.dumps(rec), flush=True)
    out.append(rec)
    plan.free()
os.makedirs("results", exist_ok=True)
json.dump(out, open("results/prefill_check%s.json" % ("_q8" if os.environ.get("PREFILL_QUANT") == "q8" else ""), "w"), indent=1)
