"""Host-side logic of the tensor-parallel path, on CPU: the row-sharding plan and the rank-ordered
handle exchange over a world_size-2 gloo group (the device side is exercised by tools/tp_check.py
with torchrun on 2 GPUs)."""
import os
import socket
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_shard_plan_covers_every_row_once(pkg):
    from types import SimpleNamespace
    c = SimpleNamespace(n_heads=32, n_kv_heads=8, head_size=128, dim=4096, hidden_dim=14336, vocab_size=128256)
    for n in (1, 2, 4, 8):
        plan = pkg.plan.tp_shard_plan(c, n)
        assert len(plan) == n
        for key, total in (("q_rows", 4096), ("kv_rows", 1024), ("residual_rows", 4096), ("hidden_units", 14336), ("vocab_rows", 128256), ("heads", 32), ("kv_heads", 8)):
            edges = [p[key] for p in plan]
            assert edges[0][0] == 0 and edges[-1][1] == total
            assert all(edges[i][1] == edges[i + 1][0] for i in range(n - 1))
        # slices stay aligned to what the kernels need: whole heads, 32-unit activation blocks, 4-row groups
        for p in plan:
            assert (p["hidden_units"][1] - p["hidden_units"][0]) % 32 == 0
            assert (p["residual_rows"][1] - p["residual_rows"][0]) % 4 == 0
            assert (p["vocab_rows"][1] - p["vocab_rows"][0]) % 4 == 0
    with pytest.raises(pkg.native.UnsupportedOperation):
        pkg.plan.tp_shard_plan(c, 3)
    c70 = SimpleNamespace(n_heads=64, n_kv_heads=8, head_size=128, dim=8192, hidden_dim=28672, vocab_size=128256)
    assert pkg.plan.tp_shard_plan(c70, 8)[7]["kv_heads"] == (7, 8)


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    import __graft_entry__ as ge
    pkg = ge.import_package()
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    handle = bytes([rank]) * 64
    got = pkg.plan.exchange_handles(handle)
    q.put((rank, [h[0] for h in got], all(len(h) == 64 for h in got)))
    dist.barrier()
    dist.destroy_process_group()


def test_handle_exchange_gloo_world2():
    import torch.multiprocessing as mp

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert res == [(0, [0, 1], True), (1, [0, 1], True)]  # every rank sees the handles in rank order


def test_sharded_host_tensors_equal_the_full_model_on_the_ranks_rows(pkg):
    """bench.py --gpus N keeps only each rank's rows on the host (70B: 74 GB -> ~10 GB per rank); the kept rows must be
    byte-identical to the single-GPU model, whatever the world size (same seeded stream)."""
    import numpy as np
    sh = pkg.synth.SHAPES["tiny-qwen3"]
    Q = pkg.gguf.GGMLType.Q8_0
    full = pkg.synth.build_tensors_fast(sh, Q, seed=9, device="cpu")
    for n in (2,):  # tiny-qwen3 has 2 KV heads
        for r in range(n):
            part = pkg.synth.build_tensors_fast(sh, Q, seed=9, device="cpu", tp_rank=r, tp_size=n)
            rng = pkg.synth.tp_row_ranges(sh, r, n)
            plan = pkg.plan.tp_shard_plan(type("C", (), dict(n_heads=sh.n_heads, n_kv_heads=sh.n_kv_heads, head_size=sh.head_size, dim=sh.dim,
                                                            hidden_dim=sh.hidden, vocab_size=sh.vocab))(), n)[r]
            assert rng["blk.0.attn_q.weight"] == plan["q_rows"] and rng["blk.0.ffn_gate.weight"] == plan["hidden_units"]
            assert rng["blk.1.ffn_down.weight"] == plan["residual_rows"] and rng["blk.0.attn_v.weight"] == plan["kv_rows"]
            for name, (tt, dims, raw) in full.items():
                praw = part[name][2]
                assert praw.shape == raw.shape
                if name in rng:
                    rb = pkg.gguf.GGMLType.byte_size_for(tt, int(dims[0]))
                    lo, hi = rng[name][0] * rb, rng[name][1] * rb
                    assert np.array_equal(praw[lo:hi], raw[lo:hi]), name
                else:
                    assert np.array_equal(praw, raw), name
