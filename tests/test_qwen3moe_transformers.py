"""The Qwen3-MoE oracle (tests/qwen3moe_oracle.py) against Hugging Face transformers' Qwen3MoeForCausalLM in float64 on the same
synthetic weights, with norm_topk_prob=True as every Qwen3-MoE release sets it: Qwen3's attention (q/k RMSNorm per head, NeoX RoPE, a
q width that differs from dim), the router orientation, the per-expert slices of the stacked tensors, SwiGLU per expert and the
renormalised top-k without a shared expert are pinned by a third party, at the Qwen2-MoE pin's tolerances and routing-margin rule
(tests/test_qwen2moe_transformers.py): both sides must choose the same experts wherever transformers' top-k margin exceeds the
tolerance; tokens where a near-tie flips are excluded from the logit comparison and must stay rare."""
import numpy as np
import pytest

from qwen3moe_oracle import Qwen3MoEOracle
from test_qwen2moe_transformers import _hf_run, _routing_flips

torch = pytest.importorskip("torch")
transformers = pytest.importorskip("transformers")


def _hf_qwen3moe(pkg, m, norm_topk: bool = True):
    c = m.configuration
    cfg = transformers.Qwen3MoeConfig(hidden_size=c.dim, intermediate_size=c.expert_hidden_dim, num_hidden_layers=c.n_layers,
                                      num_attention_heads=c.n_heads, num_key_value_heads=c.n_kv_heads, head_dim=c.head_size,
                                      vocab_size=c.vocab_size, rms_norm_eps=c.rms_norm_eps, max_position_embeddings=c.context_length,
                                      tie_word_embeddings=False, rope_theta=c.rope_theta, use_sliding_window=False,
                                      moe_intermediate_size=c.expert_hidden_dim, num_experts=c.n_experts, num_experts_per_tok=c.n_experts_used,
                                      norm_topk_prob=norm_topk, decoder_sparse_step=1, mlp_only_layers=[], attention_bias=False)
    hf = transformers.Qwen3MoeForCausalLM(cfg)
    hf.set_experts_implementation("eager")  # the per-expert loop (the grouped GEMM has no float64 form)

    def F(name):
        return pkg.loader.tensor_as_f32(m, name).astype(np.float64)
    E, he, d = c.n_experts, c.expert_hidden_dim, c.dim
    sd = {"model.embed_tokens.weight": F("token_embd.weight").reshape(c.vocab_size, d), "model.norm.weight": F("output_norm.weight")}
    sd["lm_head.weight"] = F("output.weight").reshape(c.vocab_size, d) if "output.weight" in m.tensors else sd["model.embed_tokens.weight"]
    qd, kvd = c.q_dim, c.kv_dim
    for l in range(c.n_layers):
        g, h = f"blk.{l}.", f"model.layers.{l}."
        sd[h + "self_attn.q_proj.weight"] = F(g + "attn_q.weight").reshape(qd, d)
        sd[h + "self_attn.k_proj.weight"] = F(g + "attn_k.weight").reshape(kvd, d)
        sd[h + "self_attn.v_proj.weight"] = F(g + "attn_v.weight").reshape(kvd, d)
        sd[h + "self_attn.o_proj.weight"] = F(g + "attn_output.weight").reshape(d, qd)
        sd[h + "self_attn.q_norm.weight"] = F(g + "attn_q_norm.weight")
        sd[h + "self_attn.k_norm.weight"] = F(g + "attn_k_norm.weight")
        sd[h + "input_layernorm.weight"] = F(g + "attn_norm.weight")
        sd[h + "post_attention_layernorm.weight"] = F(g + "ffn_norm.weight")
        sd[h + "mlp.gate.weight"] = F(g + "ffn_gate_inp.weight").reshape(E, d)
        sd[h + "mlp.experts.gate_up_proj"] = np.concatenate([F(g + "ffn_gate_exps.weight").reshape(E, he, d),
                                                             F(g + "ffn_up_exps.weight").reshape(E, he, d)], axis=1)
        sd[h + "mlp.experts.down_proj"] = F(g + "ffn_down_exps.weight").reshape(E, d, he)
    hf = hf.to(torch.float64)
    missing, unexpected = hf.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in sd.items()}, strict=False)
    assert not unexpected and all("rotary" in k or "inv_freq" in k for k in missing), (missing, unexpected)
    return hf.eval()


def _oracle_run(orc, m, toks):
    om = Qwen3MoEOracle(orc, m)
    try:
        lg, ids = [], []
        for p in range(len(toks)):
            lg.append(om.forward(int(toks[p]), p))
            ids.append([om.routing[l][0].copy() for l in range(m.configuration.n_layers)])
        return np.stack(lg), ids
    finally:
        om.close()


# Q8_0 runs on the shapes whose 20 tokens have no flip that also moves the later tokens: on tiny-qwen3moe a near-tie flip at token 15
# (margin 2e-3) changes the K/V rows the next tokens attend to, which the exclusion rule does not cover (F16 pins that shape).
@pytest.mark.parametrize("shape,quant,tol", [("tiny-qwen3moe", "F16", 2e-4), ("tiny-qwen3moe-k8", "F16", 2e-4), ("tiny-qwen3moe-tied", "F16", 2e-4),
                                             ("tiny-qwen3moe-k8", "Q8_0", 5e-2), ("tiny-qwen3moe-tied", "Q8_0", 5e-2)])
def test_qwen3moe_oracle_agrees_with_transformers(pkg, orc, make_model, shape, quant, tol):
    n_tok = 20
    m = make_model(shape, getattr(pkg.gguf.GGMLType, quant), 32)
    c = m.configuration
    toks = orc.bench_tokens(c.vocab_size, n_tok)
    ours, ids = _oracle_run(orc, m, toks)
    theirs, probs = _hf_run(_hf_qwen3moe(pkg, m), toks)
    flipped = _routing_flips(probs, ids, c.n_experts_used, tol)
    assert len(flipped) <= n_tok // 10, f"routing differs on tokens {sorted(flipped)}"
    if quant == "F16":
        assert not flipped, f"routing differs on tokens {sorted(flipped)}"
    keep = [t for t in range(n_tok) if t not in flipped]
    scale = np.abs(theirs).max()
    err = np.abs(ours[keep] - theirs[keep]).max() / scale
    print(f"{shape} {quant}: oracle vs transformers max|d| / max|logit| = {err:.3e}")
    assert err <= tol, f"{shape} {quant}: oracle vs transformers max|d| / max|logit| = {err:.3e}"


def test_qwen3moe_transformers_check_has_teeth(pkg, orc, make_model):
    """Leaving the top-k weights unnormalised (norm_topk_prob=False) moves transformers' logits far beyond the F16 tolerance above, so
    the pin sees a missing renormalisation."""
    m = make_model("tiny-qwen3moe", pkg.gguf.GGMLType.F16, 32)
    toks = orc.bench_tokens(m.configuration.vocab_size, 12)
    ours, _ = _oracle_run(orc, m, toks)
    theirs, _ = _hf_run(_hf_qwen3moe(pkg, m, norm_topk=False), toks)
    assert np.abs(ours - theirs).max() / np.abs(theirs).max() > 100 * 2e-4
