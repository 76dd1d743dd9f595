"""Qwen2-MoE checks that need no GPU: the loader against Qwen2MoEModelLoader.createConfiguration, the synthetic writer against gguf-py,
the oracle's routing restatement against a literal Java-order loop, the new export and the ptxas report of the new kernels."""
import os
import re

import numpy as np
import pytest

from qwen2moe_oracle import route, shared_weight

LOG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpullama3.java_b200", "csrc", "ptxas.log")


def test_architecture_key_wins_over_name(pkg):
    L = pkg.loader
    assert L.detect_model_type({"general.architecture": "qwen2moe", "general.name": "Qwen2 Llama MoE"}) == "QWEN_2_MOE"
    assert L.detect_model_type({"general.architecture": "qwen2", "general.name": "Qwen2 MoE"}) == "QWEN_2"
    assert pkg.engine.loop_for("QWEN_2_MOE") is pkg.engine.generate_tokens_qwen3


def test_loader_maps_qwen2moe_metadata(pkg, tmp_path):
    path = str(tmp_path / "m.gguf")
    sh = pkg.synth.write_model(path, "tiny-qwen2moe", pkg.gguf.GGMLType.Q8_0)
    m = pkg.load_model(path, 100000)  # clamped to the model's context
    c = m.configuration
    assert m.model_type == "QWEN_2_MOE"
    assert (c.arch, c.quantization, c.dim, c.hidden_dim, c.n_layers) == (pkg.loader.ARCH_QWEN2_MOE, "Q8_0", sh.dim, 0, sh.n_layers)
    assert (c.n_heads, c.n_kv_heads, c.head_size, c.vocab_size, c.context_length) == (sh.n_heads, sh.n_kv_heads, sh.dim // sh.n_heads, sh.vocab, sh.model_ctx)
    assert (c.n_experts, c.n_experts_used, c.expert_hidden_dim, c.shared_hidden_dim) == (sh.n_experts, sh.n_experts_used, sh.expert_hidden, sh.hidden)
    assert c.rms_norm_eps == np.float32(sh.eps) and c.rope_theta == sh.rope_theta
    m2 = pkg.load_model(path, 32)
    assert m2.configuration.context_length == 32
    tok = pkg.tokenizer.from_metadata(m.gguf.metadata, m.model_type)
    assert tok.kind == pkg.tokenizer.KIND_QWEN3


def test_feed_forward_length_mismatch_is_refused(pkg, tmp_path):
    G = pkg.gguf.GGMLType
    sh = pkg.synth.SHAPES["tiny-qwen2moe"]
    md = pkg.synth.metadata_for(sh, G.Q8_0, "Qwen MoE mismatch")
    md["qwen2moe.feed_forward_length"] = sh.hidden + 256
    path = str(tmp_path / "bad.gguf")
    pkg.gguf.write_gguf(path, md, pkg.synth.build_tensors(sh, G.Q8_0, 1, 0.0))
    with pytest.raises(pkg.loader.UnsupportedModel, match="feed_forward_length"):
        pkg.load_model(path, 64)


def test_synth_writer_matches_gguf_py(pkg, tmp_path):
    gguf_py = pytest.importorskip("gguf")
    path = str(tmp_path / "w.gguf")
    sh = pkg.synth.write_model(path, "tiny-qwen2moe", pkg.gguf.GGMLType.Q8_0, seed=3)
    want = {n: (tt, d, raw) for n, tt, d, raw in pkg.synth.build_tensors(sh, pkg.gguf.GGMLType.Q8_0, 3, 0.0)}
    r = gguf_py.GGUFReader(path)
    assert r.fields["general.architecture"].contents() == "qwen2moe"
    assert r.fields["qwen2moe.expert_count"].contents() == sh.n_experts
    got = {t.name: t for t in r.tensors}
    assert set(got) == set(want)
    for name, (tt, dims, raw) in want.items():
        t = got[name]
        assert int(t.tensor_type) == int(tt), name
        assert [int(d) for d in t.shape] == list(dims), name
        assert np.array_equal(np.asarray(t.data).view(np.uint8).reshape(-1), np.asarray(raw).reshape(-1)), name
    assert list(got["blk.0.ffn_down_exps.weight"].shape) == [sh.expert_hidden, sh.dim, sh.n_experts]


def _java_route(logits, k):
    """softmaxInPlace + the top-k loop of forwardJavaQwen2MoE, one float at a time."""
    p = [np.float32(v) for v in logits]
    mx = np.float32(-np.inf)
    for v in p:
        mx = max(mx, v)
    p = [np.float32(np.exp(np.float64(np.float32(v - mx)))) for v in p]
    s = np.float32(0.0)
    for v in p:
        s = np.float32(s + v)
    p = [np.float32(v / s) for v in p]
    ids, w = [], []
    for _ in range(k):
        best, index = np.float32(-np.inf), -1
        for j, v in enumerate(p):
            if v > best:
                best, index = v, j
        ids.append(index)
        w.append(best)
        p[index] = np.float32(-np.inf)
    return ids, w


def test_routing_restatement_matches_java_order_with_ties():
    rng = np.random.default_rng(0)
    for trial in range(200):
        E, k = int(rng.integers(2, 64)), 0
        k = int(rng.integers(1, min(E, 8) + 1))
        lg = (rng.standard_normal(E) * 2).astype(np.float32)
        for _ in range(int(rng.integers(0, 4))):  # exact ties: the first index must win
            a, b = rng.integers(0, E, 2)
            lg[b] = lg[a]
        if trial % 10 == 0:
            lg[:] = lg[0]  # every row tied
        ids, w = route(lg, k)
        jid, jw = _java_route(lg, k)
        assert list(ids) == jid
        assert np.array_equal(np.asarray(w, dtype=np.float32).view(np.uint32), np.asarray(jw, dtype=np.float32).view(np.uint32))
        for i in range(1, k):
            if w[i] == w[i - 1]:
                assert ids[i] > ids[i - 1], "tied probabilities must be taken in index order"
    for g in (np.float32(-30.0), np.float32(-0.5), np.float32(0.0), np.float32(3.25), np.float32(90.0)):
        want = np.float32(np.float32(1.0) / np.float32(np.float32(1.0) + np.float32(np.exp(np.float64(-g)))))
        assert shared_weight(g).view(np.uint32) == want.view(np.uint32)


def test_moe_export_declared(pkg):
    assert "b200_plan_create_moe" in pkg.native.EXPORTS
    hdr = open(os.path.join(os.path.dirname(LOG), "..", "..", "include", "b200llama.h")).read()
    assert re.search(r"int b200_plan_create_moe\(", hdr)
    assert "#define B200_ARCH_QWEN2_MOE 4" in hdr


def test_moe_kernels_do_not_spill():
    if not os.path.exists(LOG):
        pytest.skip("no ptxas report: the library was not built in this tree")
    lines = open(LOG).read().splitlines()
    found = {}
    for i, line in enumerate(lines):
        m = re.search(r"Compiling entry function '(\S*k_moe_\S+)'", line)
        if m:
            props = next((x for x in lines[i + 1:i + 4] if "spill stores" in x), "")
            s = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", props)
            found[m.group(1)] = tuple(int(v) for v in s.groups())
    assert len(found) == 3, found
    for name, (stack, st, ld) in found.items():
        assert (stack, st, ld) == (0, 0, 0), f"{name}: stack / spill stores / loads = {stack} / {st} / {ld}"
