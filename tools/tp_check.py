"""Tensor-parallel parity check, one process per GPU:
   torchrun --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29511 tools/tp_check.py [shape] [steps]
Every rank builds the same seeded model, uploads its share, decodes a teacher-forced stream and a greedy
stream with BOTH decode implementations (CUDA graph / persistent kernel); rank 0 compares every argmax with the
CPU oracle (token-exact expected: row sharding keeps the reference's summation order) and the residual stream bit
for bit, and writes results/tp_check_<shape>_tp<N>.json."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import torch.distributed as dist

import __graft_entry__ as ge

pkg = ge.import_package()
rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
shape = sys.argv[1] if len(sys.argv) > 1 else "mid-llama"
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 8
sh = pkg.synth.SHAPES[shape]
m = pkg.loader.model_from_tensors(sh, 8, pkg.synth.build_tensors_fast(sh, 8, seed=5, device=f"cuda:{local}"), steps + 8)
plan = pkg.B200MasterPlan(m, device=local, tp_rank=rank, tp_size=world)
toks = pkg.llama_bench.synthetic_tokens(sh.vocab, steps)
report = {"shape": shape, "tp": world, "steps": steps, "modes": {}}
ok = True
ref = refg = refx = None
if rank == 0:
    orc = ge.import_oracle()
    orc.use_all_cores()
    om = orc.OracleModel(m)
    ref = [orc.argmax(om.forward(int(toks[p]), p)) for p in range(steps)]
    om.reset()
    for p in range(steps):
        om.forward(int(toks[p]), p, want_logits=False)
    refx = om.x().copy()  # the residual stream after the last layer of the last step
    om.reset()
    tok, refg = int(toks[0]), []
    for p in range(steps):
        tok = orc.argmax(om.forward(tok, p))
        refg.append(tok)
for mode in ("graph", "persistent"):
    try:
        plan.set_decode_mode(mode)
    except pkg.native.UnsupportedOperation as e:
        if rank == 0:
            print(f"[tp{world}] {mode}: unsupported ({e})", flush=True)
        continue
    plan.kv_reset()
    dist.barrier()
    ids, ms = plan.decode_sequence(toks, steps, 0)
    x = plan.read_buffer("x", sh.dim)
    plan.kv_reset()
    g, _ = plan.decode_sequence(toks[:1], steps, 0, feedback=True)
    all_g = [None] * world
    dist.all_gather_object(all_g, [int(t) for t in g])
    if rank == 0:
        r = {"teacher_forced_ids_equal_oracle": list(ids) == ref, "residual_stream_bit_exact": bool(np.array_equal(refx.view(np.uint32), x.view(np.uint32))),
             "greedy_ranks_agree": all(a == all_g[0] for a in all_g), "greedy_ids_equal_oracle": all_g[0] == refg, "us_per_token": ms / steps * 1e3}
        report["modes"][mode] = r
        ok &= all(v for k, v in r.items() if k != "us_per_token")
        print(f"[tp{world}] {mode}: {r}", flush=True)
if rank == 0:
    report["ok"] = bool(ok)
    os.makedirs(os.path.join(ROOT, "results"), exist_ok=True)
    with open(os.path.join(ROOT, "results", f"tp_check_{shape}_tp{world}.json"), "w") as f:
        json.dump(report, f, indent=1)
    print("RESULT", "OK" if ok else "MISMATCH", flush=True)
plan.free()
dist.barrier()
dist.destroy_process_group()
