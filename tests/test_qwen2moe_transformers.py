"""The Qwen2-MoE oracle (tests/qwen2moe_oracle.py) against Hugging Face transformers' Qwen2MoeForCausalLM in float64 on the same
synthetic weights: the router orientation ([E][dim]), the per-expert slices of the stacked [E][rows][cols] tensors, SwiGLU per
expert, top-k without renormalisation and the sigmoid-gated shared expert are pinned by a third party, at the tolerances the Qwen2
pin uses (tests/test_qwen2.py).  Before the logits are compared, the routing is: both sides must choose the same experts wherever
transformers' top-k margin (k-th minus (k+1)-th probability) exceeds the tolerance.  Where it does not, Q8_0's int8 activations may
flip a near-tied expert; such tokens are excluded from the logit comparison and must stay rare."""
import numpy as np
import pytest

from qwen2moe_oracle import Qwen2MoEOracle

torch = pytest.importorskip("torch")
transformers = pytest.importorskip("transformers")


def _hf_qwen2moe(pkg, m, norm_topk: bool = False):
    c = m.configuration
    cfg = transformers.Qwen2MoeConfig(hidden_size=c.dim, intermediate_size=c.shared_hidden_dim, num_hidden_layers=c.n_layers,
                                      num_attention_heads=c.n_heads, num_key_value_heads=c.n_kv_heads, vocab_size=c.vocab_size,
                                      rms_norm_eps=c.rms_norm_eps, max_position_embeddings=c.context_length, tie_word_embeddings=False,
                                      rope_theta=c.rope_theta, use_sliding_window=False, moe_intermediate_size=c.expert_hidden_dim,
                                      shared_expert_intermediate_size=c.shared_hidden_dim, num_experts=c.n_experts,
                                      num_experts_per_tok=c.n_experts_used, norm_topk_prob=norm_topk, decoder_sparse_step=1,
                                      mlp_only_layers=[], qkv_bias=True)
    hf = transformers.Qwen2MoeForCausalLM(cfg)
    hf.set_experts_implementation("eager")  # the per-expert loop of Qwen2MoeExperts (the grouped GEMM has no float64 form)

    def F(name):
        return pkg.loader.tensor_as_f32(m, name).astype(np.float64)
    E, he, hs, d = c.n_experts, c.expert_hidden_dim, c.shared_hidden_dim, c.dim
    sd = {"model.embed_tokens.weight": F("token_embd.weight").reshape(c.vocab_size, d), "model.norm.weight": F("output_norm.weight")}
    sd["lm_head.weight"] = F("output.weight").reshape(c.vocab_size, d) if "output.weight" in m.tensors else sd["model.embed_tokens.weight"]
    qd, kvd = c.q_dim, c.kv_dim
    for l in range(c.n_layers):
        g, h = f"blk.{l}.", f"model.layers.{l}."
        sd[h + "self_attn.q_proj.weight"] = F(g + "attn_q.weight").reshape(qd, d)
        sd[h + "self_attn.k_proj.weight"] = F(g + "attn_k.weight").reshape(kvd, d)
        sd[h + "self_attn.v_proj.weight"] = F(g + "attn_v.weight").reshape(kvd, d)
        for w in "qkv":
            sd[h + f"self_attn.{w}_proj.bias"] = F(g + f"attn_{w}.bias")
        sd[h + "self_attn.o_proj.weight"] = F(g + "attn_output.weight").reshape(d, qd)
        sd[h + "input_layernorm.weight"] = F(g + "attn_norm.weight")
        sd[h + "post_attention_layernorm.weight"] = F(g + "ffn_norm.weight")
        sd[h + "mlp.gate.weight"] = F(g + "ffn_gate_inp.weight").reshape(E, d)
        sd[h + "mlp.experts.gate_up_proj"] = np.concatenate([F(g + "ffn_gate_exps.weight").reshape(E, he, d),
                                                             F(g + "ffn_up_exps.weight").reshape(E, he, d)], axis=1)
        sd[h + "mlp.experts.down_proj"] = F(g + "ffn_down_exps.weight").reshape(E, d, he)
        sd[h + "mlp.shared_expert.gate_proj.weight"] = F(g + "ffn_gate_shexp.weight").reshape(hs, d)
        sd[h + "mlp.shared_expert.up_proj.weight"] = F(g + "ffn_up_shexp.weight").reshape(hs, d)
        sd[h + "mlp.shared_expert.down_proj.weight"] = F(g + "ffn_down_shexp.weight").reshape(d, hs)
        sd[h + "mlp.shared_expert_gate.weight"] = F(g + "ffn_gate_inp_shexp.weight").reshape(1, d)
    hf = hf.to(torch.float64)
    missing, unexpected = hf.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in sd.items()}, strict=False)
    assert not unexpected and all("rotary" in k or "inv_freq" in k for k in missing), (missing, unexpected)
    return hf.eval()


def _hf_run(hf, toks):
    """Logits and, per layer, the router's softmax probabilities of every token."""
    probs = {}
    hooks = [layer.mlp.gate.register_forward_hook(lambda mod, inp, out, l=l: probs.__setitem__(l, out[0].detach().double().numpy()))
             for l, layer in enumerate(hf.model.layers)]
    try:
        with torch.no_grad():
            lg = hf(torch.tensor(toks[None, :].astype(np.int64))).logits[0].numpy()
    finally:
        for hk in hooks:
            hk.remove()
    return lg, probs


def _oracle_run(orc, m, toks):
    om = Qwen2MoEOracle(orc, m)
    try:
        lg, ids = [], []
        for p in range(len(toks)):
            lg.append(om.forward(int(toks[p]), p))
            ids.append([om.routing[l][0].copy() for l in range(m.configuration.n_layers)])
        return np.stack(lg), ids
    finally:
        om.close()


def _routing_flips(probs, ids, k, tol):
    """Tokens where the two sides selected different experts in some layer; each such difference must be a near-tie of
    transformers' k-th and (k+1)-th probabilities (margin <= tol)."""
    flipped = set()
    for l, p in probs.items():
        for t in range(p.shape[0]):
            if set(np.argsort(-p[t], kind="stable")[:k].tolist()) != set(ids[t][l].tolist()):
                srt = np.sort(p[t])[::-1]
                assert srt[k - 1] - srt[k] <= tol, f"token {t} layer {l}: experts differ at a top-k margin of {srt[k - 1] - srt[k]:.3e}"
                flipped.add(t)
    return flipped


@pytest.mark.parametrize("shape,quant,tol", [("tiny-qwen2moe", "F16", 2e-4), ("tiny-qwen2moe-gqa", "F16", 2e-4), ("tiny-qwen2moe", "Q8_0", 5e-2)])
def test_qwen2moe_oracle_agrees_with_transformers(pkg, orc, make_model, shape, quant, tol):
    n_tok = 20
    m = make_model(shape, getattr(pkg.gguf.GGMLType, quant), 32)
    c = m.configuration
    toks = orc.bench_tokens(c.vocab_size, n_tok)
    ours, ids = _oracle_run(orc, m, toks)
    theirs, probs = _hf_run(_hf_qwen2moe(pkg, m), toks)
    flipped = _routing_flips(probs, ids, c.n_experts_used, tol)
    assert len(flipped) <= n_tok // 10, f"routing differs on tokens {sorted(flipped)}"
    if quant == "F16":
        assert not flipped, f"routing differs on tokens {sorted(flipped)}"
    keep = [t for t in range(n_tok) if t not in flipped]
    scale = np.abs(theirs).max()
    err = np.abs(ours[keep] - theirs[keep]).max() / scale
    print(f"{shape} {quant}: oracle vs transformers max|d| / max|logit| = {err:.3e}")
    assert err <= tol, f"{shape} {quant}: oracle vs transformers max|d| / max|logit| = {err:.3e}"


def test_qwen2moe_transformers_check_has_teeth(pkg, orc, make_model):
    """Renormalising the top-k weights (norm_topk_prob=True) moves transformers' logits far beyond the F16 tolerance above, so the
    pin sees that mistake."""
    m = make_model("tiny-qwen2moe", pkg.gguf.GGMLType.F16, 32)
    toks = orc.bench_tokens(m.configuration.vocab_size, 12)
    ours, _ = _oracle_run(orc, m, toks)
    theirs, _ = _hf_run(_hf_qwen2moe(pkg, m, norm_topk=True), toks)
    assert np.abs(ours - theirs).max() / np.abs(theirs).max() > 100 * 2e-4
