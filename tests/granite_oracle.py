"""CPU restatement of the reference's Granite forward pass, InferenceCore.forwardGranite (InferenceCore.java:814-921), for the tests and
tools/granite_bench.py.  TEST INFRASTRUCTURE ONLY, like oracle/oracle.c.

It is the Llama forward of oracle.c with four muP scalars, each one float32 multiply evaluated where the reference makes it:
  * x = emb[token] * embeddingScale                (:826-829, after copyTo);
  * score = q.k * attentionScale                   (:868-873, in place of score / sqrt(headSize));
  * x = x + (Wo.xb) * residualScale, and the same for W2 (:889-892, :907-910: mapInPlace, then addInPlace);
  * logits = (wcls.x) * logitScale                 (:917-918).
Every other step uses the C oracle's own code (oracle_matmul, oracle_rmsnorm, its RoPE table) and tests/qwen2_oracle.py's
order-exact sums, so the matmul and norm arithmetic is exactly the one the other architectures are pinned to.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from qwen2_oracle import Qwen2Oracle, _seqsum

f32 = np.float32


class GraniteOracle(Qwen2Oracle):
    """Same interface as the C oracle's OracleModel for a Granite loader.Model (or any Llama-shaped model with explicit `scales`).
    scales: {"embedding_scale", "residual_scale", "attention_scale", "logit_scale"}; default: the model configuration's.
    drop: names of scales evaluated as if absent (the embedding / residual / logit multiply skipped, the attention score divided by
    sqrt(head size) again) -- the mistakes the tests must be able to see."""

    def __init__(self, orc, model, lanes: int = 16, per_row_quant: bool = False, scales: dict | None = None, drop: tuple = ()):
        # Qwen2Oracle's state without its q/k/v biases (a Granite file has none); RoPE on interleaved pairs, as forwardGranite (:845-857)
        self.orc, self.model = orc, model
        self.cfg = c = model.configuration
        self.om = orc.OracleModel(model, lanes=lanes, per_row_quant=per_row_quant)
        L = orc.lib()
        L.oracle_matmul.argtypes = [C.POINTER(orc.OModel), C.c_void_p, C.POINTER(orc.OTensor), C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]
        self._lib = L
        self.bias, self.neox = False, False
        self._rope_cr, self._rope_ci = orc.rope_table(c.context_length, c.head_size, c.rope_theta)
        self._kc = np.zeros((c.n_layers, c.context_length, c.kv_dim), dtype=np.float32)
        self._vc = np.zeros_like(self._kc)
        self._emb = model.tensors["token_embd.weight"]
        s = scales or {k: getattr(c, k) for k in ("embedding_scale", "residual_scale", "attention_scale", "logit_scale")}
        self.es, self.rs, self.as_, self.ls = (f32(s[k]) for k in ("embedding_scale", "residual_scale", "attention_scale", "logit_scale"))
        self.drop = set(drop)

    def forward(self, token: int, pos: int, want_logits: bool = True):
        c, m = self.cfg, self.om.m
        dim, hs, nh, nkv = c.dim, c.head_size, c.n_heads, c.n_kv_heads
        qd, kvd, kv_mul = nh * hs, nkv * hs, nh // nkv
        sqrt_hs = f32(np.sqrt(np.float64(hs)))
        x = self._embedding(token)
        if "embedding_scale" not in self.drop:
            x = x * self.es                                                                     # x[i] = x[i] * embeddingScale
        resid = (lambda v: v) if "residual_scale" in self.drop else (lambda v: v * self.rs)
        for l in range(c.n_layers):
            xb = self._rmsnorm(x, m.attn_norm[l])
            q, k, v = self._matmul(m.wq[l], xb, qd, dim), self._matmul(m.wk[l], xb, kvd, dim), self._matmul(m.wv[l], xb, kvd, dim)
            q, k = self._rope(q, nh, pos), self._rope(k, nkv, pos)
            self._kc[l, pos], self._vc[l, pos] = k, v
            K = self._kc[l, :pos + 1].reshape(pos + 1, nkv, hs)[:, np.arange(nh) // kv_mul].transpose(1, 0, 2)  # [head][t][hs]
            V = self._vc[l, :pos + 1].reshape(pos + 1, nkv, hs)[:, np.arange(nh) // kv_mul].transpose(1, 0, 2)
            dot = _seqsum(q.reshape(nh, 1, hs) * K, axis=2)                                     # scalarDot
            score = dot / sqrt_hs if "attention_scale" in self.drop else dot * self.as_         # score *= attentionScale
            e = np.exp((score - score.max(axis=1, keepdims=True)).astype(np.float64)).astype(np.float32)
            att = e / _seqsum(e, axis=1)[:, None]                                               # softmaxInPlace
            xb = _seqsum(att[:, :, None] * V, axis=1).reshape(-1)
            x = x + resid(self._matmul(m.wo[l], xb, dim, qd))                                   # xb2 * residualScale, then x += xb2
            xb = self._rmsnorm(x, m.ffn_norm[l])
            hb, hb2 = self._matmul(m.w1[l], xb, c.hidden_dim, dim), self._matmul(m.w3[l], xb, c.hidden_dim, dim)
            hb = hb / (1.0 + np.exp(-hb.astype(np.float64))).astype(np.float32)
            x = x + resid(self._matmul(m.w2[l], hb * hb2, dim, c.hidden_dim))
        if not want_logits:
            return None
        x = self._rmsnorm(x, m.output_norm)
        logits = self._matmul(m.output if m.output.data else m.token_embd, x, c.vocab_size, dim)
        return logits if "logit_scale" in self.drop else logits * self.ls                      # logits * logitScale
