"""CPU restatement of the reference's Qwen2-MoE forward pass, InferenceCore.forwardJavaQwen2MoE (InferenceCore.java:263-432), for the
tests and tools/moe_bench.py.  TEST INFRASTRUCTURE ONLY, like oracle/oracle.c.

Attention is Qwen2Oracle's (q/k/v biases, NeoX RoPE).  The FFN is restated step by step:
  * router logits: FloatTensor.scalarDot over the F32 router rows (result += w * x, float, index order);
  * softmaxInPlace: max; (float) Math.exp(f - max) (float64 exp, narrowed); a sequential sum from 0f; a divide;
  * top-k: k scans for the first strict maximum, each pick then set to -inf; the weight is the probability (no renormalisation);
  * each selected expert's gate/up/down are the C oracle's oracle_matmul on an OTensor pointing at the expert's slice of the stacked
    tensor (matmulExpert, :430-432: the same per-32-block activation quantisation as every other Q8_0 matmul);
  * x = w * y + x per expert in selection order (saxpyInPlace: a float multiply, then a float add), then the shared expert with
    weight 1f / (1f + (float) Math.exp(-g)), g the F32 scalarDot of ffn_gate_inp_shexp and xb.
"""
from __future__ import annotations

import ctypes as C
import dataclasses

import numpy as np

from qwen2_oracle import Qwen2Oracle, _seqsum

f32 = np.float32


def scalar_dot_rows(w: np.ndarray, x: np.ndarray) -> np.ndarray:
    """FloatTensor.scalarDot of every row of w with x: float products, summed element after element from 0f."""
    return _seqsum(w.astype(np.float32) * x.astype(np.float32)[None, :], axis=1)


def route(logits: np.ndarray, k: int):
    """softmaxInPlace over the router logits, then the reference's top-k scans.  Returns (ids, weights) as int32 / float32 arrays."""
    lg = np.asarray(logits, dtype=np.float32)
    mx = lg.max()
    e = np.exp((lg - mx).astype(np.float64)).astype(np.float32)
    p = (e / _seqsum(e[None, :], axis=1)[0]).astype(np.float32)
    ids, wts = [], []
    for _ in range(k):
        best, idx = f32(-np.inf), -1
        for j in range(len(p)):
            if p[j] > best:
                best, idx = p[j], j
        ids.append(idx)
        wts.append(best)
        p[idx] = -np.inf
    return np.array(ids, dtype=np.int32), np.array(wts, dtype=np.float32)


def shared_weight(g: np.float32) -> np.float32:
    """1f / (1f + (float) Math.exp(-g))"""
    return f32(f32(1.0) / (f32(1.0) + f32(np.exp(np.float64(-f32(g))))))


class Qwen2MoEOracle(Qwen2Oracle):
    """Qwen2Oracle with the MoE FFN.  After each forward, `routing[l]` holds (ids, weights, shared weight) of layer l."""

    def __init__(self, orc, model, lanes: int = 16):
        c = model.configuration
        T = model.tensors
        # The C oracle's model wrapper supplies the matrices, norms and matmul scratch; it expects a dense FFN, so it gets the shared
        # expert's tensors in those slots (never used here) and a hidden size that covers every expert's activation.
        shim_t = dict(T)
        for l in range(c.n_layers):
            for a, b in (("gate", "gate"), ("up", "up"), ("down", "down")):
                shim_t[f"blk.{l}.ffn_{a}.weight"] = T[f"blk.{l}.ffn_{b}_shexp.weight"]
        shim_c = dataclasses.replace(c, arch=3, hidden_dim=max(c.shared_hidden_dim, c.expert_hidden_dim))

        class _Shim:
            configuration = shim_c
            tensors = shim_t
        super().__init__(orc, _Shim(), lanes=lanes)
        self.cfg = c
        self.model = model
        self._T = T
        self._router = [np.asarray(T[f"blk.{l}.ffn_gate_inp.weight"][2]).view(np.float32).reshape(c.n_experts, c.dim) for l in range(c.n_layers)]
        self._shgate = [np.asarray(T[f"blk.{l}.ffn_gate_inp_shexp.weight"][2]).view(np.float32).reshape(c.dim) for l in range(c.n_layers)]
        self._ot = {}
        self.routing = [None] * c.n_layers

    def _slice(self, name: str, e: int, rows: int, cols: int):
        """OTensor of expert e of a stacked [E][rows][cols] tensor."""
        key = (name, e)
        if key not in self._ot:
            tt, dims, raw = self._T[name]
            rb = {0: cols * 4, 1: cols * 2, 8: cols // 32 * 34}[int(tt)]
            raw = np.asarray(raw).reshape(-1)[e * rows * rb:(e + 1) * rows * rb]
            t = self.orc.OTensor()
            t.data = raw.ctypes.data
            t.type = int(tt)
            self._ot[key] = (t, raw)
        return self._ot[key][0]

    def _whole(self, name: str):
        return self._slice(name, 0, *self._rows_cols(name))

    def _rows_cols(self, name):
        dims = self._T[name][1]
        return int(dims[1]), int(dims[0])

    def _swiglu_expert(self, wg, wu, wd, xb, hidden):
        c = self.cfg
        hb, hb2 = self._matmul(wg, xb, hidden, c.dim), self._matmul(wu, xb, hidden, c.dim)
        hb = hb / (1.0 + np.exp(-hb.astype(np.float64))).astype(np.float32)
        return self._matmul(wd, hb * hb2, c.dim, hidden)

    def ffn(self, l: int, x: np.ndarray, xb: np.ndarray) -> np.ndarray:
        c = self.cfg
        he, hs = c.expert_hidden_dim, c.shared_hidden_dim
        ids, wts = route(scalar_dot_rows(self._router[l], xb), c.n_experts_used)
        g = scalar_dot_rows(self._shgate[l][None, :], xb)[0]
        sw = shared_weight(g)
        self.routing[l] = (ids, wts, sw)
        pre = f"blk.{l}."
        for j, e in enumerate(ids):
            y = self._swiglu_expert(self._slice(pre + "ffn_gate_exps.weight", int(e), he, c.dim), self._slice(pre + "ffn_up_exps.weight", int(e), he, c.dim),
                                    self._slice(pre + "ffn_down_exps.weight", int(e), c.dim, he), xb, he)
            x = (wts[j] * y + x).astype(np.float32)
        y = self._swiglu_expert(self._whole(pre + "ffn_gate_shexp.weight"), self._whole(pre + "ffn_up_shexp.weight"),
                                self._whole(pre + "ffn_down_shexp.weight"), xb, hs)
        return (sw * y + x).astype(np.float32)

    def forward(self, token: int, pos: int, want_logits: bool = True):
        c, m = self.cfg, self.om.m
        dim, hs, nh, nkv = c.dim, c.head_size, c.n_heads, c.n_kv_heads
        qd, kvd, kv_mul = nh * hs, nkv * hs, nh // nkv
        sqrt_hs = f32(np.sqrt(np.float64(hs)))
        x = self._embedding(token)
        for l in range(c.n_layers):
            xb = self._rmsnorm(x, m.attn_norm[l])
            q, k, v = self._matmul(m.wq[l], xb, qd, dim), self._matmul(m.wk[l], xb, kvd, dim), self._matmul(m.wv[l], xb, kvd, dim)
            bq, bk, bv = self._b[l]
            q, k, v = q + bq, k + bk, v + bv
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
