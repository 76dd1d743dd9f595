"""CPU restatement of the reference's Qwen2 forward pass, InferenceCore.forwardJavaQwen2 (InferenceCore.java:434-563), for the
tests and tools/qwen2_bench.py.  TEST INFRASTRUCTURE ONLY, like oracle/oracle.c.

It is the Llama forward of oracle.c with two differences, both restated here line by line:
  * q, k and v get their F32 biases right after the three matmuls (q.addInPlace(q_bias) etc., :456-459: one float add each);
  * RoPE rotates NeoX pairs (ic, ic + head/2) per head, without a q/k norm (:463-478).
Every other step uses the C oracle's own code (oracle_matmul, oracle_rmsnorm, its RoPE table), so the matmul and norm arithmetic is
exactly the one the other architectures are pinned to.  Attention, softmax and SwiGLU are evaluated in numpy float32 in the
reference's order: the sequential sums (scalarDot :86-92, softmaxInPlace :211-219, saxpyInPlace :221-227) run through
np.add.accumulate, which adds element after element, from an explicit 0.0f start; Math.exp is evaluated in float64 and narrowed.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

f32 = np.float32


def _seqsum(terms: np.ndarray, axis: int) -> np.ndarray:
    """`float r = 0; for (i) r += t[i];` along `axis`: element after element from +0.0f."""
    shape = list(terms.shape)
    shape[axis] = 1
    z = np.zeros(shape, dtype=np.float32)
    return np.take(np.add.accumulate(np.concatenate([z, terms.astype(np.float32)], axis=axis), axis=axis, dtype=np.float32), -1, axis=axis)


class Qwen2Oracle:
    """Same interface as the C oracle's OracleModel (forward / reset / key_cache / value_cache / close) for a Qwen2 loader.Model.
    bias=False or neox=False evaluate the forward pass WITHOUT the biases / with interleaved pairs instead: the structural mistakes
    the tests must be able to see."""

    def __init__(self, orc, model, lanes: int = 16, per_row_quant: bool = False, bias: bool = True, neox: bool = True):
        self.orc, self.model = orc, model
        self.cfg = c = model.configuration
        self.om = orc.OracleModel(model, lanes=lanes, per_row_quant=per_row_quant)  # the matrices, norms and matmul scratch
        L = orc.lib()
        L.oracle_matmul.argtypes = [C.POINTER(orc.OModel), C.c_void_p, C.POINTER(orc.OTensor), C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]
        self._lib = L
        self.bias, self.neox = bias, neox
        T = model.tensors
        self._b = [[np.asarray(T[f"blk.{l}.attn_{w}.bias"][2]).view(np.float32).copy() for w in "qkv"] for l in range(c.n_layers)]
        self._rope_cr, self._rope_ci = orc.rope_table(c.context_length, c.head_size, c.rope_theta)
        self._kc = np.zeros((c.n_layers, c.context_length, c.kv_dim), dtype=np.float32)  # Java arrays start zeroed
        self._vc = np.zeros_like(self._kc)
        self._emb = T["token_embd.weight"]

    # ---- C oracle pieces
    def _matmul(self, w, x: np.ndarray, d0: int, d1: int) -> np.ndarray:
        x = np.ascontiguousarray(x, dtype=np.float32)
        out = np.empty(d0, dtype=np.float32)
        self._lib.oracle_matmul(C.byref(self.om.m), self.om.state, C.byref(w), x.ctypes.data, out.ctypes.data, d0, d1)
        return out

    def _rmsnorm(self, x: np.ndarray, w) -> np.ndarray:
        x = np.ascontiguousarray(x, dtype=np.float32)
        out = np.empty_like(x)
        self._lib.oracle_rmsnorm(out.ctypes.data, x.ctypes.data, C.byref(w), len(x), self.cfg.rms_norm_eps)
        return out

    def _embedding(self, token: int) -> np.ndarray:
        """token_embedding_table.copyTo (getFloat per element)."""
        tt, dims, raw = self._emb
        dim, raw = self.cfg.dim, np.asarray(raw).reshape(-1)
        if int(tt) == 0:
            return raw[token * dim * 4:(token + 1) * dim * 4].view(np.float32).copy()
        if int(tt) == 1:
            return raw[token * dim * 2:(token + 1) * dim * 2].view(np.float16).astype(np.float32)
        blk = raw[token * dim // 32 * 34:(token + 1) * dim // 32 * 34].reshape(-1, 34)
        d = blk[:, :2].copy().view(np.float16).astype(np.float32)
        return (blk[:, 2:].view(np.int8).astype(np.float32) * d).reshape(-1)  # (float) q * float16ToFloat(scale)

    def _rope(self, vec: np.ndarray, n_heads: int, pos: int) -> np.ndarray:
        hs = self.cfg.head_size
        half = hs // 2
        fcr, fci = self._rope_cr[pos * half:(pos + 1) * half], self._rope_ci[pos * half:(pos + 1) * half]
        v = vec.reshape(n_heads, hs).copy()
        if self.neox:  # pairs (ic, ic + head/2), frequency index ic (:463-478)
            v0, v1 = v[:, :half].copy(), v[:, half:].copy()
            v[:, :half] = v0 * fcr - v1 * fci
            v[:, half:] = v0 * fci + v1 * fcr
        else:  # interleaved pairs (2i, 2i + 1), frequency index i (forwardJava :75-87)
            v0, v1 = v[:, 0::2].copy(), v[:, 1::2].copy()
            v[:, 0::2] = v0 * fcr - v1 * fci
            v[:, 1::2] = v0 * fci + v1 * fcr
        return v.reshape(-1)

    def forward(self, token: int, pos: int, want_logits: bool = True):
        c, m = self.cfg, self.om.m
        dim, hs, nh, nkv = c.dim, c.head_size, c.n_heads, c.n_kv_heads
        qd, kvd, kv_mul = nh * hs, nkv * hs, nh // nkv
        sqrt_hs = f32(np.sqrt(np.float64(hs)))
        x = self._embedding(token)
        for l in range(c.n_layers):
            xb = self._rmsnorm(x, m.attn_norm[l])
            q, k, v = self._matmul(m.wq[l], xb, qd, dim), self._matmul(m.wk[l], xb, kvd, dim), self._matmul(m.wv[l], xb, kvd, dim)
            if self.bias:
                bq, bk, bv = self._b[l]
                q, k, v = q + bq, k + bk, v + bv
            q, k = self._rope(q, nh, pos), self._rope(k, nkv, pos)
            self._kc[l, pos], self._vc[l, pos] = k, v
            K = self._kc[l, :pos + 1].reshape(pos + 1, nkv, hs)[:, np.arange(nh) // kv_mul].transpose(1, 0, 2)  # [head][t][hs]
            V = self._vc[l, :pos + 1].reshape(pos + 1, nkv, hs)[:, np.arange(nh) // kv_mul].transpose(1, 0, 2)
            score = _seqsum(q.reshape(nh, 1, hs) * K, axis=2) / sqrt_hs                      # scalarDot, then score /= sqrtHeadSize
            e = np.exp((score - score.max(axis=1, keepdims=True)).astype(np.float64)).astype(np.float32)
            att = e / _seqsum(e, axis=1)[:, None]                                              # softmaxInPlace
            xb = _seqsum(att[:, :, None] * V, axis=1).reshape(-1)                              # xb[i] = a * v[i] + xb[i], t ascending
            x = x + self._matmul(m.wo[l], xb, dim, qd)
            xb = self._rmsnorm(x, m.ffn_norm[l])
            hb, hb2 = self._matmul(m.w1[l], xb, c.hidden_dim, dim), self._matmul(m.w3[l], xb, c.hidden_dim, dim)
            hb = hb / (1.0 + np.exp(-hb.astype(np.float64))).astype(np.float32)                # value / (float) (1.0 + Math.exp(-value))
            x = x + self._matmul(m.w2[l], hb * hb2, dim, c.hidden_dim)
        if not want_logits:
            return None
        x = self._rmsnorm(x, m.output_norm)
        return self._matmul(m.output if m.output.data else m.token_embd, x, c.vocab_size, dim)

    def reset(self):
        self._kc[:] = 0.0
        self._vc[:] = 0.0

    def key_cache(self, layer: int) -> np.ndarray:
        return self._kc[layer].reshape(-1).copy()

    def value_cache(self, layer: int) -> np.ndarray:
        return self._vc[layer].reshape(-1).copy()

    def close(self):
        self.om.close()
