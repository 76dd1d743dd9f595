#!/usr/bin/env python
"""Phase timeline of the persistent decode kernel (b200_trace_persistent): where one token's time goes.

    python tools/trace_persistent.py [workload] [depth] > decode_timeline.txt

Every CTA stamps %globaltimer at ten points per layer (include/b200llama.h).  Reported per phase, averaged over the
layers 1..L-1 (layer 0 starts from the embedding row): the mean and the slowest CTA's duration, and for every grid-wide
dependency the exposed wait = (first CTA through the wait) - (last CTA arriving), i.e. the barrier's own latency.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402

PHASES = ["attn norm (x -> xq in smem)", "QKV stream", "QKV sync + attention + gather", "stage att + Wo stream", "Wo sync (x gather)",
          "ffn norm", "gate/up stream (+SwiGLU, quantise)", "gate/up sync + stage hidden act", "W2 stream", "W2 sync (x gather) -> next layer"]


def main():
    workload = sys.argv[1] if len(sys.argv) > 1 else "llama-3-8b"
    depth = int(sys.argv[2]) if len(sys.argv) > 2 else 64
    pkg = ge.import_package()
    shape = pkg.synth.SHAPES[workload]
    Q = pkg.gguf.GGMLType.Q8_0
    model = pkg.loader.model_from_tensors(shape, Q, pkg.synth.build_tensors_fast(shape, Q, seed=1234, device="cuda:0"), depth + 16)
    plan = pkg.B200MasterPlan.initialize_plan(model)
    plan.set_decode_mode("persistent")
    toks = np.asarray(pkg.llama_bench.synthetic_tokens(shape.vocab, depth + 8), dtype=np.int32)
    plan.decode_sequence(toks[:depth], depth, 0)
    for i in range(3):
        st = plan.trace_persistent(int(toks[depth + i]), depth + i).astype(np.float64)
    nL = shape.n_layers
    t0 = st[:, 0, 0].min()
    st = (st - t0) / 1e3  # us
    lay = st[:, :nL, :]  # [cta][layer][10]
    print(f"# {workload} Q8_0, persistent decode kernel, position {depth + 2}; decode_info = {plan.decode_info()}")
    nxt = np.concatenate([lay[:, 1:, 0], st[:, nL:nL + 1, 0]], axis=1)  # start of the next layer (or of the lm_head row)
    ends = np.concatenate([lay[:, :, 1:10], nxt[:, :, None]], axis=2)   # end stamp of phase k = stamp k+1
    dur = ends - lay[:, :, :10]                                          # [cta][layer][10]
    sel = slice(1, nL) if nL > 1 else slice(0, 1)
    print(f"{'phase':44s} {'mean us':>9s} {'slowest CTA':>12s}")
    for k, name in enumerate(PHASES):
        d = dur[:, sel, k]
        print(f"{name:44s} {d.mean():9.2f} {d.max(axis=0).mean():12.2f}")
    # inside the attn norm (every CTA) and the attention (head CTAs only: stamps 12-15 are zero elsewhere)
    print(f"{'  attn norm: load x,w + squares':44s} {(lay[:, sel, 10] - lay[:, sel, 0]).mean():9.2f}")
    print(f"{'  attn norm: exact sequential sum':44s} {(lay[:, sel, 11] - lay[:, sel, 10]).mean():9.2f}")
    print(f"{'  attn norm: scale + normalise + quantise':44s} {(lay[:, sel, 1] - lay[:, sel, 11]).mean():9.2f}")
    heads = np.flatnonzero(st[:, 1 if nL > 1 else 0, 12] > -1e6)  # unstamped slots are zero, i.e. hugely negative after the shift
    if len(heads):
        hl = lay[heads][:, sel, :]
        print(f"{'  attention: QKV barrier (arrive -> all in)':44s} {(hl[:, :, 12] - hl[:, :, 2]).mean():9.2f}")
        print(f"{'  attention: rope + scores + max':44s} {(hl[:, :, 13] - hl[:, :, 12]).mean():9.2f}")
        print(f"{'  attention: exp + sum + normalise':44s} {(hl[:, :, 14] - hl[:, :, 13]).mean():9.2f}")
        print(f"{'  attention: weighted value sum + quantise':44s} {(hl[:, :, 15] - hl[:, :, 14]).mean():9.2f}")
        print(f"{'  attention: ATT barrier (head done -> gathered)':44s} {(hl[:, :, 3] - hl[:, :, 15]).mean():9.2f}")
    if st.shape[2] > 17 and nL > 1:
        cold = (lay[:, 1, 11] - lay[:, 1, 10]).mean()
        warm = (lay[:, 1, 17] - lay[:, 1, 16]).mean()
        print(f"{'  exact sum of layer 1: first run / immediate re-run':52s} {cold:6.2f} / {warm:5.2f}   (same code, same data: the difference is instruction fetch)")
    per_layer = (nxt[:, sel] - lay[:, sel, 0])
    print(f"{'layer total (CTA mean)':44s} {per_layer.mean():9.2f}")
    # exposed barrier latency: last arrival -> first departure, per dependency
    print("\n# grid-wide dependencies: (first CTA past the wait) - (last CTA done producing), mean over layers [us]")
    deps = [("QKV+attention -> Wo", 2, 3), ("Wo -> ffn norm", 4, 5), ("gate/up -> W2 (incl. staging the activation)", 7, 8)]
    for name, a, b in deps:
        last_arrive = lay[:, sel, a].max(axis=0)
        first_leave = lay[:, sel, b].min(axis=0)
        print(f"  {name:46s} {np.mean(first_leave - last_arrive):8.2f}")
    last_arrive = lay[:, sel, 9].max(axis=0)
    first_leave = nxt[:, sel].min(axis=0)
    print(f"  {'W2 -> next layer':46s} {np.mean(first_leave - last_arrive):8.2f}")
    lm = st[:, nL, :]
    print(f"\n# lm_head row: final norm {np.mean(lm[:, 1] - lm[:, 0]):.2f} us, lm_head stream {np.mean(lm[:, 2] - lm[:, 1]):.2f} us (slowest CTA {np.max(lm[:, 2] - lm[:, 1]):.2f}), "
          f"argmax + advance {lm[0, 3] - lm[:, 2].max():.2f} us")
    print(f"# token total (first stamp -> step advanced): {lm[0, 3]:.1f} us; layers {st[:, nL, 0].mean():.1f} us")
    plan.free()


if __name__ == "__main__":
    main()
