"""CPU restatement of a Qwen3-MoE forward pass, for the tests and tools/qwen3moe_bench.py.  TEST INFRASTRUCTURE ONLY, like
oracle/oracle.c.

The reference has no Qwen3-MoE path, so this one is composed of the reference's pieces:
  * attention is forwardJavaQwen3's (InferenceCore.java:565-697), as oracle.c runs the QWEN3 arch: the C oracle's matmuls, a
    per-head RMSNorm of q and of k (oracle_rmsnorm over head_size floats), NeoX RoPE, then the same attention as every other family;
  * the FFN is forwardJavaQwen2MoE's (InferenceCore.java:366-424, tests/qwen2moe_oracle.py) without the shared expert: router logits
    by scalarDot, softmaxInPlace, k scans for the first strict maximum, then the renormalisation s = 0f; s += p_j over the picks in
    selection order; w_j = p_j / s, and each selected expert's SwiGLU through the Q8_0 matmul added as x = w_j * y + x in selection
    order.
Expert slices are cut lazily from the stacked tensors (no copy), so the whole 48-layer model is never materialised as float.
"""
from __future__ import annotations

import ctypes as C
import dataclasses

import numpy as np

from qwen2_oracle import _seqsum
from qwen2moe_oracle import Qwen2MoEOracle, route, scalar_dot_rows

f32 = np.float32


def renormalise(weights: np.ndarray) -> np.ndarray:
    """s = 0f; s = s + w_j in selection order; w_j / s (float32 throughout)."""
    w = np.asarray(weights, dtype=np.float32)
    s = f32(0.0)
    for v in w:
        s = f32(s + v)
    return (w / s).astype(np.float32)


class Qwen3MoEOracle(Qwen2MoEOracle):
    """Same interface as Qwen2MoEOracle; after each forward, `routing[l]` holds (ids, renormalised weights) of layer l."""

    def __init__(self, orc, model, lanes: int = 16):
        c = model.configuration
        T = model.tensors
        # The C oracle's model wrapper supplies the matrices, norms, q/k norms and matmul scratch.  It expects a dense FFN, so its
        # FFN slots point at the stacked expert tensors (never used through them) and its hidden size covers one expert's activation.
        shim_t = dict(T)
        for l in range(c.n_layers):
            for w in ("gate", "up", "down"):
                shim_t[f"blk.{l}.ffn_{w}.weight"] = T[f"blk.{l}.ffn_{w}_exps.weight"]
        shim_c = dataclasses.replace(c, arch=1, hidden_dim=c.expert_hidden_dim)

        class _Shim:
            configuration = shim_c
            tensors = shim_t
        self.orc, self.model = orc, model
        self.cfg = c
        self.om = orc.OracleModel(_Shim(), lanes=lanes)
        L = orc.lib()
        L.oracle_matmul.argtypes = [C.POINTER(orc.OModel), C.c_void_p, C.POINTER(orc.OTensor), C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]
        self._lib = L
        self.neox = True
        self._rope_cr, self._rope_ci = orc.rope_table(c.context_length, c.head_size, c.rope_theta)
        self._kc = np.zeros((c.n_layers, c.context_length, c.kv_dim), dtype=np.float32)  # Java arrays start zeroed
        self._vc = np.zeros_like(self._kc)
        self._emb = T["token_embd.weight"]
        self._T = T
        self._router = [np.asarray(T[f"blk.{l}.ffn_gate_inp.weight"][2]).view(np.float32).reshape(c.n_experts, c.dim) for l in range(c.n_layers)]
        self._ot = {}
        self.routing = [None] * c.n_layers

    def _head_norm(self, vec: np.ndarray, n_heads: int, w) -> np.ndarray:
        hs = self.cfg.head_size
        return np.concatenate([self._rmsnorm(vec[h * hs:(h + 1) * hs], w) for h in range(n_heads)])

    def ffn(self, l: int, x: np.ndarray, xb: np.ndarray) -> np.ndarray:
        c = self.cfg
        he = c.expert_hidden_dim
        ids, p = route(scalar_dot_rows(self._router[l], xb), c.n_experts_used)
        wts = renormalise(p)
        self.routing[l] = (ids, wts)
        pre = f"blk.{l}."
        for j, e in enumerate(ids):
            y = self._swiglu_expert(self._slice(pre + "ffn_gate_exps.weight", int(e), he, c.dim), self._slice(pre + "ffn_up_exps.weight", int(e), he, c.dim),
                                    self._slice(pre + "ffn_down_exps.weight", int(e), c.dim, he), xb, he)
            x = (wts[j] * y + x).astype(np.float32)
        return x

    def forward(self, token: int, pos: int, want_logits: bool = True):
        c, m = self.cfg, self.om.m
        dim, hs, nh, nkv = c.dim, c.head_size, c.n_heads, c.n_kv_heads
        qd, kvd, kv_mul = nh * hs, nkv * hs, nh // nkv
        sqrt_hs = f32(np.sqrt(np.float64(hs)))
        x = self._embedding(token)
        for l in range(c.n_layers):
            xb = self._rmsnorm(x, m.attn_norm[l])
            q, k, v = self._matmul(m.wq[l], xb, qd, dim), self._matmul(m.wk[l], xb, kvd, dim), self._matmul(m.wv[l], xb, kvd, dim)
            q, k = self._head_norm(q, nh, m.attn_q_norm[l]), self._head_norm(k, nkv, m.attn_k_norm[l])
            q, k = self._rope(q, nh, pos), self._rope(k, nkv, pos)
            self._kc[l, pos], self._vc[l, pos] = k, v
            K = self._kc[l, :pos + 1].reshape(pos + 1, nkv, hs)[:, np.arange(nh) // kv_mul].transpose(1, 0, 2)
            V = self._vc[l, :pos + 1].reshape(pos + 1, nkv, hs)[:, np.arange(nh) // kv_mul].transpose(1, 0, 2)
            score = _seqsum(q.reshape(nh, 1, hs) * K, axis=2) / sqrt_hs
            e = np.exp((score - score.max(axis=1, keepdims=True)).astype(np.float64)).astype(np.float32)
            att = e / _seqsum(e, axis=1)[:, None]
            xb = _seqsum(att[:, :, None] * V, axis=1).reshape(-1)
            x = x + self._matmul(m.wo[l], xb, dim, qd)
            x = self.ffn(l, x, self._rmsnorm(x, m.ffn_norm[l]))
        if not want_logits:
            return None
        x = self._rmsnorm(x, m.output_norm)
        return self._matmul(m.output if m.output.data else m.token_embd, x, c.vocab_size, dim)

