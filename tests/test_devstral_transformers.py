"""The CPU restatement of forwardJavaDevstral and its YaRN RoPE table (tests/devstral_oracle.py) against Hugging Face transformers'
MistralForCausalLM in float64 on the same synthetic weights.

transformers is configured to compute what the reference computes: head_dim set explicitly (q is n_heads * head_dim wide, not dim),
rope_parameters of type yarn with truncate=False (by default transformers floors / ceils the correction range; RoPE.java uses the
float correction dims as they are) and attention_factor = the reference's mscale (transformers' default is 0.1 * ln(factor) + 1,
without the log multiplier).  The synthetic shapes keep the correction range inside [0, head_dim - 1], where transformers' clamp is
inactive."""
import numpy as np
import pytest

from devstral_oracle import DevstralOracle, yarn_freqs, yarn_mscale

torch = pytest.importorskip("torch")
transformers = pytest.importorskip("transformers")


def _unpermute(w, n_head):
    """Inverse of llama.cpp's permute(): GGUF (interleaved pairs 2i, 2i+1) -> HF (i, i + head/2)."""
    rows, cols = w.shape
    hs = rows // n_head
    return w.reshape(n_head, hs // 2, 2, cols).swapaxes(1, 2).reshape(rows, cols)


def _hf_config(c):
    rope = {"rope_type": "default", "rope_theta": c.rope_theta}
    if c.yarn is not None:
        y = c.yarn
        rope = {"rope_type": "yarn", "rope_theta": c.rope_theta, "factor": y.factor, "beta_fast": y.beta_fast, "beta_slow": y.beta_slow,
                "original_max_position_embeddings": y.original_context_length, "truncate": False,
                "attention_factor": float(yarn_mscale(y.factor, y.log_multiplier))}
    return transformers.MistralConfig(hidden_size=c.dim, intermediate_size=c.hidden_dim, num_hidden_layers=c.n_layers, num_attention_heads=c.n_heads,
                                      num_key_value_heads=c.n_kv_heads, head_dim=c.head_size, vocab_size=c.vocab_size, rms_norm_eps=c.rms_norm_eps,
                                      max_position_embeddings=c.context_length, tie_word_embeddings=False, rope_parameters=rope, sliding_window=None)


def _hf_mistral(pkg, m):
    c = m.configuration
    hf = transformers.MistralForCausalLM(_hf_config(c))

    def W(name, rows, cols):
        return pkg.loader.tensor_as_f32(m, name).reshape(rows, cols).astype(np.float64)

    def V(name):
        return pkg.loader.tensor_as_f32(m, name).astype(np.float64)
    sd = {"model.embed_tokens.weight": W("token_embd.weight", c.vocab_size, c.dim), "model.norm.weight": V("output_norm.weight"),
          "lm_head.weight": W("output.weight", c.vocab_size, c.dim)}
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
    assert not unexpected and all("rotary" in k or "inv_freq" in k for k in missing), (missing, unexpected)
    return hf.eval()


def _oracle_logits(orc, m, toks, **kw):
    om = DevstralOracle(orc, m, **kw)
    try:
        return np.stack([om.forward(int(toks[p]), p) for p in range(len(toks))])
    finally:
        om.close()


@pytest.mark.parametrize("shape,quant,tol,mistakes", [
    ("tiny-devstral", "F16", 2e-4, ("mscale", "ramp")),
    # Q8_0: the CPU path rounds every activation block to int8 (the algorithm, not an error); at this shape that alone moves the
    # logits by about 2.3e-2 of max|logit|, inside the Q8_0 bar of the Llama pin (tests/test_oracle_vs_transformers.py)
    ("tiny-devstral", "Q8_0", 5e-2, ("mscale", "ramp")),
    ("tiny-devstral-wide", "F16", 2e-4, ("mscale", "ramp", "qdim")),
    ("tiny-devstral-plain", "F16", 2e-4, ()),
])
def test_devstral_oracle_agrees_with_transformers(pkg, orc, make_model, shape, quant, tol, mistakes):
    """Within the FP16 / Q8_0 bars of max|logit|; dropping the YaRN attention factor, dropping the ramp (the plain table) or rotating q
    over dim instead of qDim each moves the logits by more than 1e-2 of max|logit|."""
    n_tok = 24
    m = make_model(shape, getattr(pkg.gguf.GGMLType, quant), 32)
    assert m.model_type == "DEVSTRAL_2"
    toks = orc.bench_tokens(m.configuration.vocab_size, n_tok)
    ours = _oracle_logits(orc, m, toks)
    with torch.no_grad():
        theirs = _hf_mistral(pkg, m)(torch.tensor(toks[None, :].astype(np.int64))).logits[0].numpy()
    scale = np.abs(theirs).max()
    err = np.abs(ours - theirs).max() / scale
    print(f"{shape} {quant}: oracle vs transformers max|d| / max|logit| = {err:.3e}")
    assert err <= tol
    for d in mistakes:
        moved = np.abs(_oracle_logits(orc, m, toks, drop=(d,)) - theirs).max() / scale
        print(f"  without {d}: {moved:.3e}")
        assert moved > 1e-2, f"dropping {d} moves the logits by only {moved:.3e}"


def test_yarn_frequencies_match_transformers(pkg, make_model):
    """The oracle's per-pair YaRN frequencies against transformers' float32 inv_freq, and the correction range is unclamped there."""
    c = make_model("tiny-devstral", pkg.gguf.GGMLType.F16, 32).configuration
    from transformers.modeling_rope_utils import ROPE_INIT_FUNCTIONS
    inv, att = ROPE_INIT_FUNCTIONS["yarn"](_hf_config(c), "cpu")
    ours, mscale = yarn_freqs(c.head_size, c.rope_theta, c.yarn)
    assert np.abs(ours - inv.numpy()).max() / np.abs(ours).max() < 1e-6
    assert np.float32(att) == mscale
    plain, _ = yarn_freqs(c.head_size, c.rope_theta, c.yarn, ("ramp",))
    assert (plain != ours).sum() >= c.head_size // 2 - 2   # only the pairs below the low correction dim keep their frequency
