"""The CPU restatement of forwardGranite (tests/granite_oracle.py) against Hugging Face transformers' GraniteForCausalLM in float64 on
the same synthetic weights, and against the C oracle on a plain Llama model.

Logit scale: the reference MULTIPLIES the logits by granite.logit_scale (InferenceCore.java:917-918); transformers DIVIDES by
logits_scaling (modeling_granite.py), the value llama.cpp's converter stores in that key.  This project follows the reference, so the
pin hands transformers logits_scaling = 1 / logit_scale (DESIGN.md section 10)."""
import numpy as np
import pytest

from granite_oracle import GraniteOracle

torch = pytest.importorskip("torch")
transformers = pytest.importorskip("transformers")

SCALES = ("embedding_scale", "residual_scale", "attention_scale", "logit_scale")


def _unpermute(w, n_head):
    """Inverse of llama.cpp's permute(): GGUF (interleaved pairs 2i, 2i+1) -> HF (i, i + head/2)."""
    rows, cols = w.shape
    hs = rows // n_head
    return w.reshape(n_head, hs // 2, 2, cols).swapaxes(1, 2).reshape(rows, cols)


def _hf_granite(pkg, m):
    c = m.configuration
    cfg = transformers.GraniteConfig(hidden_size=c.dim, intermediate_size=c.hidden_dim, num_hidden_layers=c.n_layers, num_attention_heads=c.n_heads,
                                     num_key_value_heads=c.n_kv_heads, vocab_size=c.vocab_size, rms_norm_eps=c.rms_norm_eps,
                                     max_position_embeddings=c.context_length, tie_word_embeddings=True, rope_theta=c.rope_theta,
                                     embedding_multiplier=c.embedding_scale, residual_multiplier=c.residual_scale,
                                     attention_multiplier=c.attention_scale, logits_scaling=1.0 / c.logit_scale)
    hf = transformers.GraniteForCausalLM(cfg)

    def W(name, rows, cols):
        return pkg.loader.tensor_as_f32(m, name).reshape(rows, cols).astype(np.float64)

    def V(name):
        return pkg.loader.tensor_as_f32(m, name).astype(np.float64)
    sd = {"model.embed_tokens.weight": W("token_embd.weight", c.vocab_size, c.dim), "model.norm.weight": V("output_norm.weight")}
    sd["lm_head.weight"] = sd["model.embed_tokens.weight"]
    qd, kvd = c.q_dim, c.kv_dim
    for l in range(c.n_layers):
        g, h = f"blk.{l}.", f"model.layers.{l}."
        sd[h + "self_attn.q_proj.weight"] = _unpermute(W(g + "attn_q.weight", qd, c.dim), c.n_heads)
        sd[h + "self_attn.k_proj.weight"] = _unpermute(W(g + "attn_k.weight", kvd, c.dim), c.n_kv_heads)
        sd[h + "self_attn.v_proj.weight"] = W(g + "attn_v.weight", kvd, c.dim)
        sd[h + "self_attn.o_proj.weight"] = W(g + "attn_output.weight", c.dim, qd)
        sd[h + "mlp.gate_proj.weight"] = W(g + "ffn_gate.weight", c.hidden_dim, c.dim)
        sd[h + "mlp.up_proj.weight"] = W(g + "ffn_up.weight", c.hidden_dim, c.dim)
        sd[h + "mlp.down_proj.weight"] = W(g + "ffn_down.weight", c.dim, c.hidden_dim)
        sd[h + "input_layernorm.weight"] = V(g + "attn_norm.weight")
        sd[h + "post_attention_layernorm.weight"] = V(g + "ffn_norm.weight")
    hf = hf.to(torch.float64)
    missing, unexpected = hf.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in sd.items()}, strict=False)
    assert not unexpected and all("rotary" in k or "inv_freq" in k or k == "lm_head.weight" for k in missing), (missing, unexpected)
    return hf.eval()


def _oracle_logits(orc, m, toks, **kw):
    om = GraniteOracle(orc, m, **kw)
    try:
        return np.stack([om.forward(int(toks[p]), p) for p in range(len(toks))])
    finally:
        om.close()


@pytest.mark.parametrize("shape,quant,tol", [("tiny-granite", "F16", 2e-4), ("tiny-granite-gqa", "F16", 2e-4), ("tiny-granite", "Q8_0", 1.7e-2)])
def test_granite_oracle_agrees_with_transformers(pkg, orc, make_model, shape, quant, tol):
    """Within the FP16 / Q8_0 bars; dropping any one of the four scales moves the logits by more than 1e-2 of max|logit|."""
    n_tok = 16
    m = make_model(shape, getattr(pkg.gguf.GGMLType, quant), 32)
    toks = orc.bench_tokens(m.configuration.vocab_size, n_tok)
    ours = _oracle_logits(orc, m, toks)
    with torch.no_grad():
        theirs = _hf_granite(pkg, m)(torch.tensor(toks[None, :].astype(np.int64))).logits[0].numpy()
    scale = np.abs(theirs).max()
    err = np.abs(ours - theirs).max() / scale
    print(f"{shape} {quant}: oracle vs transformers max|d| / max|logit| = {err:.3e}")
    assert err <= tol
    for s in SCALES:
        moved = np.abs(_oracle_logits(orc, m, toks, drop=(s,)) - theirs).max() / scale
        print(f"  without {s}: {moved:.3e}")
        assert moved > 1e-2, f"dropping {s} moves the logits by only {moved:.3e}"


def test_granite_oracle_on_llama_matches_the_c_oracle(pkg, orc, make_model):
    """Scales 1, 1, 1/sqrt(head size), 1 on a Llama model: the forward is the C oracle's except that the score is MULTIPLIED by the
    rounded 1/sqrt(hs) instead of divided by sqrt(hs), so the two agree to float rounding (not bit for bit)."""
    m = make_model("tiny-llama-tied", pkg.gguf.GGMLType.F16, 32)
    hs = m.configuration.head_size
    scales = {"embedding_scale": 1.0, "residual_scale": 1.0, "attention_scale": float(np.float32(1.0 / np.sqrt(hs))), "logit_scale": 1.0}
    toks = orc.bench_tokens(m.configuration.vocab_size, 12)
    ours = _oracle_logits(orc, m, toks, scales=scales)
    om = orc.OracleModel(m)
    try:
        ref = np.stack([om.forward(int(toks[p]), p) for p in range(len(toks))])
    finally:
        om.close()
    err = np.abs(ours - ref).max() / np.abs(ref).max()
    print(f"granite oracle (llama scales) vs C oracle: {err:.3e}")
    assert err <= 1e-5
