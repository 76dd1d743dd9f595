"""Qwen2 / Qwen2.5 / DeepSeek-R1-Distill-Qwen on the host (no GPU): the loader (Qwen2ModelLoader.createConfiguration,
Qwen2ModelLoader.java:48-73), the tokenizer routing (:35-43) and the CPU restatement of forwardJavaQwen2 (tests/qwen2_oracle.py)
against Hugging Face transformers' Qwen2ForCausalLM in float64 on the same synthetic weights, biases included."""
import numpy as np
import pytest

from qwen2_oracle import Qwen2Oracle


def _write(pkg, path, shape_name, quant, edit=None, name=None):
    """A synthetic Qwen2 GGUF whose metadata `edit` may change first."""
    s = pkg.synth
    sh = s.SHAPES[shape_name]
    md = s.metadata_for(sh, quant, name or f"Qwen2 synthetic {shape_name}")
    if edit:
        edit(md)
    pkg.gguf.write_gguf(path, md, s.build_tensors(sh, quant, 1234, 0.0))
    return sh


def test_qwen2_loader_configuration(pkg, tmp_path):
    path = str(tmp_path / "q2.gguf")
    sh = _write(pkg, path, "tiny-qwen2", pkg.gguf.GGMLType.Q8_0)
    m = pkg.load_model(path, 64)
    c = m.configuration
    assert m.model_type == "QWEN_2" and c.arch == pkg.loader.ARCH_QWEN2 == 3 and c.quantization == "Q8_0"
    assert (c.dim, c.hidden_dim, c.n_layers, c.n_heads, c.n_kv_heads, c.head_size) == (896, 1024, 2, 14, 2, 64)
    assert c.head_size == c.dim // c.n_heads and c.kv_dim == c.dim * c.n_kv_heads // c.n_heads
    assert (c.rms_norm_eps, c.rope_theta) == (np.float32(1e-6), 1000000.0)
    assert c.context_length == 64                          # min(model context, requested)
    assert pkg.load_model(path, 10 ** 6).configuration.context_length == sh.model_ctx == 32768
    assert pkg.load_model(path).configuration.context_length == 32768
    for l in range(c.n_layers):
        for w, n in (("q", c.q_dim), ("k", c.kv_dim), ("v", c.kv_dim)):
            tt, dims, raw = m.tensors[f"blk.{l}.attn_{w}.bias"]
            assert int(tt) == pkg.gguf.GGMLType.F32 and tuple(int(d) for d in dims) == (n,)
            b = np.asarray(raw).view(np.float32)
            assert np.sum(np.abs(b) == 20.0) == max(1, n // 32)  # the large entries that make a missing bias visible


def test_deepseek_distill_loader_vocab_from_token_list_and_defaults(pkg, tmp_path):
    path = str(tmp_path / "ds.gguf")

    def edit(md):
        md["tokenizer.ggml.tokens"] = md["tokenizer.ggml.tokens"] + ["<｜end▁of▁sentence｜>"]
        md["tokenizer.ggml.token_type"] = md["tokenizer.ggml.token_type"] + [3]
        md["general.basename"] = "DeepSeek-R1-Distill-Qwen"
        del md["qwen2.attention.head_count_kv"]
    _write(pkg, path, "tiny-qwen2", pkg.gguf.GGMLType.F16, edit, name="DeepSeek R1 Distill Qwen 1.5B synthetic")
    m = pkg.load_model(path, 48)
    c = m.configuration
    assert m.model_type == "DEEPSEEK_R1_DISTILL_QWEN" and c.arch == 3 and c.quantization == "FP16"
    assert c.vocab_size == 513 != m.gguf.metadata["qwen2.vocab_size"]  # the token list's size, not qwen2.vocab_size
    assert c.n_kv_heads == c.n_heads == 14                             # head_count_kv defaults to head_count
    tok = pkg.tokenizer.from_metadata(m.gguf.metadata, m.model_type)
    assert isinstance(tok, pkg.tokenizer.Qwen3Tokenizer)
    first = min(tok.special_tokens.values())
    assert tok.tokens[first] == "<｜end▁of▁sentence｜>" and first == 512


def test_qwen2_tokenizer_routing(pkg, tmp_path):
    path = str(tmp_path / "q2.gguf")
    _write(pkg, path, "tiny-qwen2", pkg.gguf.GGMLType.Q8_0, lambda md: md.__setitem__("general.basename", "Qwen2.5"))
    m = pkg.load_model(path, 32)
    tok = pkg.tokenizer.from_metadata(m.gguf.metadata, m.model_type)
    assert isinstance(tok, pkg.tokenizer.Qwen3Tokenizer)
    assert tok.tokens[min(tok.special_tokens.values())] == "<|endoftext|>"
    assert tok.decode(tok.encode("the quick brown fox")) == "the quick brown fox"


@pytest.mark.parametrize("key", ["qwen2.attention.layer_norm_rms_epsilon", "qwen2.rope.freq_base"])
def test_qwen2_loader_requires_eps_and_theta(pkg, tmp_path, key):
    path = str(tmp_path / "bad.gguf")
    _write(pkg, path, "tiny-qwen2", pkg.gguf.GGMLType.Q8_0, lambda md: md.pop(key))
    with pytest.raises(KeyError, match=key.replace(".", r"\.")):
        pkg.load_model(path, 32)


def test_qwen2_biases_are_not_sharded(pkg):
    """Tensor parallelism splits the matrices by rows; the host passes the biases whole (each rank reads its heads' rows)."""
    sh = pkg.synth.SHAPES["tiny-qwen2"]
    r = pkg.synth.tp_row_ranges(sh, 1, 2)
    assert "blk.0.attn_q.weight" in r and not any(k.endswith(".bias") for k in r)


# ---- the oracle against transformers ---------------------------------------------------------------------------------

torch = pytest.importorskip("torch")
transformers = pytest.importorskip("transformers")


def _hf_qwen2(pkg, m):
    c = m.configuration
    cfg = transformers.Qwen2Config(hidden_size=c.dim, intermediate_size=c.hidden_dim, num_hidden_layers=c.n_layers,
                                   num_attention_heads=c.n_heads, num_key_value_heads=c.n_kv_heads, vocab_size=c.vocab_size,
                                   rms_norm_eps=c.rms_norm_eps, max_position_embeddings=c.context_length, tie_word_embeddings=False,
                                   rope_theta=c.rope_theta, use_sliding_window=False)
    hf = transformers.Qwen2ForCausalLM(cfg)

    def W(name, rows, cols):
        return pkg.loader.tensor_as_f32(m, name).reshape(rows, cols).astype(np.float64)

    def V(name):
        return pkg.loader.tensor_as_f32(m, name).astype(np.float64)
    sd = {"model.embed_tokens.weight": W("token_embd.weight", c.vocab_size, c.dim), "model.norm.weight": V("output_norm.weight")}
    sd["lm_head.weight"] = W("output.weight", c.vocab_size, c.dim) if "output.weight" in m.tensors else sd["model.embed_tokens.weight"]
    qd, kvd = c.q_dim, c.kv_dim
    for l in range(c.n_layers):  # Qwen2 GGUF files keep the rotate-half (NeoX) row order: no un-permute
        g, h = f"blk.{l}.", f"model.layers.{l}."
        sd[h + "self_attn.q_proj.weight"] = W(g + "attn_q.weight", qd, c.dim)
        sd[h + "self_attn.k_proj.weight"] = W(g + "attn_k.weight", kvd, c.dim)
        sd[h + "self_attn.v_proj.weight"] = W(g + "attn_v.weight", kvd, c.dim)
        sd[h + "self_attn.q_proj.bias"] = V(g + "attn_q.bias")
        sd[h + "self_attn.k_proj.bias"] = V(g + "attn_k.bias")
        sd[h + "self_attn.v_proj.bias"] = V(g + "attn_v.bias")
        sd[h + "self_attn.o_proj.weight"] = W(g + "attn_output.weight", c.dim, qd)
        sd[h + "mlp.gate_proj.weight"] = W(g + "ffn_gate.weight", c.hidden_dim, c.dim)
        sd[h + "mlp.up_proj.weight"] = W(g + "ffn_up.weight", c.hidden_dim, c.dim)
        sd[h + "mlp.down_proj.weight"] = W(g + "ffn_down.weight", c.dim, c.hidden_dim)
        sd[h + "input_layernorm.weight"] = V(g + "attn_norm.weight")
        sd[h + "post_attention_layernorm.weight"] = V(g + "ffn_norm.weight")
    hf = hf.to(torch.float64)
    missing, unexpected = hf.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in sd.items()}, strict=False)
    assert not unexpected and all("rotary" in k or "inv_freq" in k for k in missing), (missing, unexpected)
    return hf.eval()


def _oracle_logits(orc, m, toks, **kw):
    om = Qwen2Oracle(orc, m, **kw)
    try:
        return np.stack([om.forward(int(toks[p]), p) for p in range(len(toks))])
    finally:
        om.close()


@pytest.mark.parametrize("shape,quant,tol", [("tiny-qwen2", "F16", 2e-4), ("tiny-qwen2-gqa6", "F16", 2e-4), ("tiny-qwen2", "Q8_0", 5e-2)])
def test_qwen2_oracle_agrees_with_transformers(pkg, orc, make_model, shape, quant, tol):
    n_tok = 20
    m = make_model(shape, getattr(pkg.gguf.GGMLType, quant), 32)
    toks = orc.bench_tokens(m.configuration.vocab_size, n_tok)
    ours = _oracle_logits(orc, m, toks)
    with torch.no_grad():
        theirs = _hf_qwen2(pkg, m)(torch.tensor(toks[None, :].astype(np.int64))).logits[0].numpy()
    scale = np.abs(theirs).max()
    err = np.abs(ours - theirs).max() / scale
    print(f"{shape} {quant}: oracle vs transformers max|d| / max|logit| = {err:.3e}")
    assert err <= tol, f"{shape} {quant}: oracle vs transformers max|d| / max|logit| = {err:.3e}"
    if quant == "F16":
        margin = np.sort(theirs, axis=1)
        clear = (margin[:, -1] - margin[:, -2]) > 10 * tol * scale
        assert np.array_equal(ours.argmax(axis=1)[clear], theirs.argmax(axis=1)[clear]) and clear.sum() >= n_tok // 2


def test_qwen2_oracle_check_has_teeth(pkg, orc, make_model):
    """The two ways to get Qwen2 wrong -- dropping the biases, or rotating interleaved instead of NeoX pairs -- each move the
    oracle's logits by far more than the tolerance above, and dropping the biases changes the greedy tokens."""
    m = make_model("tiny-qwen2", pkg.gguf.GGMLType.F16, 32)
    toks = orc.bench_tokens(m.configuration.vocab_size, 12)
    good = _oracle_logits(orc, m, toks)
    scale = np.abs(good).max()
    no_bias = _oracle_logits(orc, m, toks, bias=False)
    interleaved = _oracle_logits(orc, m, toks, neox=False)
    assert np.abs(good - no_bias).max() / scale > 1e-2
    assert np.abs(good - interleaved).max() / scale > 1e-2
    assert not np.array_equal(good.argmax(axis=1), no_bias.argmax(axis=1))


def test_qwen2_oracle_reuses_the_c_oracle_for_llama_steps(pkg, orc, make_model):
    """Cross-check of the numpy attention / softmax / SwiGLU steps: a Llama model run through Qwen2Oracle's code with zero
    biases and interleaved pairs is exactly the C oracle's forwardJava, bit for bit."""
    m = make_model("tiny-llama", pkg.gguf.GGMLType.Q8_0, 24)
    c = m.configuration
    z = {}
    for l in range(c.n_layers):
        for w, n in (("q", c.q_dim), ("k", c.kv_dim), ("v", c.kv_dim)):
            z[f"blk.{l}.attn_{w}.bias"] = (pkg.gguf.GGMLType.F32, (n,), np.full(n, -0.0, dtype=np.float32).view(np.uint8))
    m2 = pkg.loader.Model(None, c, m.model_type, {**m.tensors, **z})
    toks = orc.bench_tokens(c.vocab_size, 16)
    ours = _oracle_logits(orc, m2, toks, neox=False)
    om = orc.OracleModel(m)
    try:
        ref = np.stack([om.forward(int(toks[p]), p) for p in range(len(toks))])
    finally:
        om.close()
    assert np.array_equal(ours.view(np.uint32), ref.view(np.uint32))

