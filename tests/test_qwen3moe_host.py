"""Qwen3-MoE checks that need no GPU: type detection and the configuration read from a synthetic qwen3moe GGUF, the loader's refusals,
the tokenizer and generation loop the family runs, the routing restatement (renormalised top-k) against a literal Java-order loop, the
header and the ptxas report of the new kernels."""
import os
import re

import numpy as np
import pytest

from qwen3moe_oracle import renormalise, route
from test_batch_decode_build import _entries

HDR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "b200llama.h")


def test_qwen3moe_architecture_wins_over_the_qwen3_name(pkg):
    L = pkg.loader
    assert L.detect_model_type({"general.architecture": "qwen3moe", "general.name": "Qwen3-30B-A3B-Instruct"}) == "QWEN_3_MOE"
    assert L.detect_model_type({"general.architecture": "qwen3", "general.name": "Qwen3 MoE"}) == "QWEN_3"
    assert L.ARCH_QWEN3_MOE == 7


def test_loader_maps_qwen3moe_metadata(pkg, tmp_path):
    path = str(tmp_path / "m.gguf")
    sh = pkg.synth.write_model(path, "tiny-qwen3moe", pkg.gguf.GGMLType.Q8_0)
    m = pkg.load_model(path, 100000)  # clamped to the model's context
    c = m.configuration
    assert "qwen3" in m.gguf.metadata["general.name"].lower()  # the name alone would say dense Qwen3
    assert m.model_type == "QWEN_3_MOE"
    assert (c.arch, c.quantization, c.dim, c.hidden_dim, c.n_layers) == (pkg.loader.ARCH_QWEN3_MOE, "Q8_0", sh.dim, 0, sh.n_layers)
    assert (c.n_heads, c.n_kv_heads, c.head_size, c.vocab_size, c.context_length) == (sh.n_heads, sh.n_kv_heads, sh.head_size, sh.vocab, sh.model_ctx)
    assert c.q_dim != c.dim
    assert (c.n_experts, c.n_experts_used, c.expert_hidden_dim, c.shared_hidden_dim) == (sh.n_experts, sh.n_experts_used, sh.expert_hidden, 0)
    assert c.rms_norm_eps == np.float32(sh.eps) and c.rope_theta == sh.rope_theta
    assert pkg.load_model(path, 32).configuration.context_length == 32
    assert not any("shexp" in n for n in m.tensors)
    assert m.tensors["blk.0.ffn_down_exps.weight"][1] == (sh.expert_hidden, sh.dim, sh.n_experts)
    # the native configuration: b200_plan_create_moe without a shared expert
    cfg = pkg.plan.make_config(m)
    assert (cfg.arch, cfg.hidden_dim, cfg.head_size) == (7, 0, sh.head_size)


def test_qwen3moe_fp16_file_loads(pkg, tmp_path):
    """FP16 files load (the plan refuses them, as it refuses FP16 Qwen2-MoE)."""
    path = str(tmp_path / "f16.gguf")
    pkg.synth.write_model(path, "tiny-qwen3moe", pkg.gguf.GGMLType.F16)
    c = pkg.load_model(path, 32).configuration
    assert c.quantization == "FP16" and c.arch == pkg.loader.ARCH_QWEN3_MOE


def _write_edited(pkg, tmp_path, edit):
    G = pkg.gguf.GGMLType
    sh = pkg.synth.SHAPES["tiny-qwen3moe"]
    md = pkg.synth.metadata_for(sh, G.Q8_0, "Qwen3 MoE edited")
    edit(md)
    path = str(tmp_path / "bad.gguf")
    pkg.gguf.write_gguf(path, md, pkg.synth.build_tensors(sh, G.Q8_0, 1, 0.0))
    return path


def test_value_length_mismatch_is_refused(pkg, tmp_path):
    path = _write_edited(pkg, tmp_path, lambda md: md.__setitem__("qwen3moe.attention.value_length", 64))
    with pytest.raises(pkg.loader.UnsupportedModel, match="value_length"):
        pkg.load_model(path, 64)


def test_expert_size_mismatch_is_refused(pkg, tmp_path):
    path = _write_edited(pkg, tmp_path, lambda md: md.__setitem__("qwen3moe.expert_feed_forward_length", 512))
    with pytest.raises(pkg.loader.UnsupportedModel, match="expert_feed_forward_length"):
        pkg.load_model(path, 64)


def test_qwen3moe_tokenizer_and_loop(pkg, tmp_path):
    path = str(tmp_path / "t.gguf")
    pkg.synth.write_model(path, "tiny-qwen3moe", pkg.gguf.GGMLType.Q8_0)
    m = pkg.load_model(path, 32)
    tok = pkg.tokenizer.from_metadata(m.gguf.metadata, m.model_type)
    assert isinstance(tok, pkg.tokenizer.Qwen3Tokenizer) and tok.kind == pkg.tokenizer.KIND_QWEN3
    ids = tok.encode_as_list("the quick brown fox")
    assert ids and tok.decode(ids) == "the quick brown fox"
    assert pkg.engine.loop_for("QWEN_3_MOE") is pkg.engine.generate_tokens_qwen3


def _java_route_renorm(logits, k):
    """softmaxInPlace, the top-k loop of forwardJavaQwen2MoE, then s = 0f, s += p_j, w_j = p_j / s, one float at a time."""
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
    t = np.float32(0.0)
    for v in w:
        t = np.float32(t + v)
    return ids, [np.float32(v / t) for v in w]


def test_renormalised_routing_matches_java_order_with_ties():
    rng = np.random.default_rng(1)
    for trial in range(200):
        E = int(rng.integers(2, 160))
        k = int(rng.integers(1, min(E, 8) + 1))
        lg = (rng.standard_normal(E) * 3).astype(np.float32)
        for _ in range(int(rng.integers(0, 4))):
            a, b = rng.integers(0, E, 2)
            lg[b] = lg[a]
        if trial % 10 == 0:
            lg[:] = 0.0  # all-zero router rows: experts 0..k-1, each weight 1/k
        ids, p = route(lg, k)
        w = renormalise(p)
        jid, jw = _java_route_renorm(lg, k)
        assert list(ids) == jid
        assert np.array_equal(w.view(np.uint32), np.asarray(jw, dtype=np.float32).view(np.uint32))
        if trial % 10 == 0:
            assert list(ids) == list(range(k))
            if E & (E - 1) == 0:  # p = 1/E exactly, so every sum of picks is exact
                assert np.all(w == np.float32(1.0 / k))


def test_qwen3moe_header():
    hdr = open(HDR).read()
    assert "#define B200_ARCH_QWEN3_MOE 7" in hdr
    assert re.search(r"int b200_plan_create_moe\(", hdr)


def test_qwen3moe_kernels_do_not_spill():
    e = _entries(r"k_routed_")
    assert len(e) == 3, e
    for name, (stack, st, ld) in e.items():
        assert (stack, st, ld) == (0, 0, 0), f"{name}: stack / spill stores / loads = {stack} / {st} / {ld}"
