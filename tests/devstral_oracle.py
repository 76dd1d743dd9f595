"""CPU restatement of the reference's Devstral 2 forward pass, InferenceCore.forwardJavaDevstral (InferenceCore.java:178-261), and of its
RoPE table (DevstralModelLoader.precomputeRopeFrequencies, RoPE.precomputeFreqsCisYaRN, RoPE.java:39-83), for the tests and
tools/devstral_bench.py.  TEST INFRASTRUCTURE ONLY, like oracle/oracle.c.

The forward is Llama's with qDim = n_heads * head_size in place of dim wherever q is concerned: the Q projection has qDim rows, RoPE
rotates interleaved pairs over qDim (k over kvDim), and Wo takes qDim columns.  No biases, no q/k norm.  It runs on Qwen2Oracle's
pieces (the C oracle's matmul and RMSNorm, order-exact attention sums) with biases off and interleaved pairs.

The YaRN table is restated here independently of csrc/plan.cu, one float32 rounding per Java float operation: numpy float32 scalars
for the float arithmetic, and math.log / math.pow / math.cos / math.sin (libm, as plan.cu calls it) for Java's double Math calls.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np

from qwen2_oracle import Qwen2Oracle

f32 = np.float32


def _jmax(a, b):
    """Math.max(float, float): NaN wins, -0.0f < 0.0f."""
    if a != a:
        return a
    if a == 0 and b == 0 and math.copysign(1.0, float(a)) < 0:
        return b
    return a if a >= b else b


def _jmin(a, b):
    """Math.min(float, float): NaN wins, -0.0f < 0.0f."""
    if a != a:
        return a
    if a == 0 and b == 0 and math.copysign(1.0, float(b)) < 0:
        return b
    return a if a <= b else b


def _corr_dim(n_dims: int, n_ctx_orig: int, n_rot, base) -> np.float32:
    """yarnCorrDim: nDims * (float) Math.log(nCtxOrig / (nRot * 2.0f * (float) Math.PI)) / (2.0f * (float) Math.log(base))."""
    denom = f32(f32(n_rot) * f32(2.0)) * f32(math.pi)
    num = f32(n_dims) * f32(math.log(float(f32(n_ctx_orig) / denom)))
    return num / (f32(2.0) * f32(math.log(float(base))))


def _ramp(low, high, i0: int) -> np.float32:
    """yarnRamp: 1 - min(1, max(0, (i0 - low) / max(0.001f, high - low)))."""
    y = (f32(i0) - low) / _jmax(f32(0.001), f32(high - low))
    return f32(1.0) - _jmin(f32(1.0), _jmax(f32(0.0), f32(y)))


def yarn_mscale(factor, log_multiplier) -> np.float32:
    """1.0f + 0.1f * logMultiplier * (float) Math.log(1.0f / freqScale) with freqScale = 1.0f / factor (1.0f when logMultiplier <= 0)."""
    factor, lm = f32(factor), f32(log_multiplier)
    if not lm > 0:
        return f32(1.0)
    freq_scale = f32(1.0) / factor
    return f32(1.0) + f32(f32(0.1) * lm) * f32(math.log(float(f32(1.0) / freq_scale)))


def yarn_freqs(head_size: int, theta: float, yarn, drop: tuple = ()) -> tuple[np.ndarray, np.float32]:
    """(per-pair frequencies, mscale) of precomputeFreqsCisYaRN.  drop: "mscale" -> mscale 1, "ramp" -> the plain frequencies."""
    th = float(f32(theta))                                      # DevstralConfiguration.ropeTheta() is a float
    extrap = [f32(1.0 / math.pow(th, i / float(head_size))) for i in range(0, head_size, 2)]
    mscale = f32(1.0) if "mscale" in drop else yarn_mscale(yarn.factor, yarn.log_multiplier)
    if "ramp" in drop:
        return np.array(extrap, dtype=np.float32), mscale
    freq_scale = f32(1.0) / f32(yarn.factor)
    c0 = _corr_dim(head_size, yarn.original_context_length, yarn.beta_fast, f32(th))
    c1 = _corr_dim(head_size, yarn.original_context_length, yarn.beta_slow, f32(th))
    out = []
    for j, fe in enumerate(extrap):
        fi = freq_scale * fe
        r = _ramp(c0, c1, j)
        out.append(f32(fi * f32(f32(1.0) - r)) + f32(fe * r))   # two rounded products, then a rounded sum
    return np.array(out, dtype=np.float32), mscale


def rope_table(context_length: int, head_size: int, theta: float, yarn=None, drop: tuple = ()) -> tuple[np.ndarray, np.ndarray]:
    """The table DevstralModelLoader builds: precomputeFreqsCisYaRN when yarn is given, else precomputeFreqsCis (no scaling).
    cr = (float) Math.cos(pos * freq) * mscale, narrowed to float before the multiply."""
    if yarn is None:
        freqs, mscale = yarn_freqs(head_size, theta, None, ("ramp", "mscale"))
    else:
        freqs, mscale = yarn_freqs(head_size, theta, yarn, drop)
    half = head_size // 2
    cr = np.empty(context_length * half, dtype=np.float32)
    ci = np.empty_like(cr)
    k = 0
    for pos in range(context_length):
        for j in range(half):
            val = float(f32(pos) * freqs[j])
            cr[k] = f32(math.cos(val)) * mscale
            ci[k] = f32(math.sin(val)) * mscale
            k += 1
    return cr, ci


class DevstralOracle(Qwen2Oracle):
    """Same interface as the C oracle's OracleModel for a Devstral loader.Model.
    drop: mistakes the tests must be able to see -- "mscale" (the YaRN table without its attention factor), "ramp" (the plain table
    in place of the YaRN one), "qdim" (q rotated over its first dim entries only, as forwardJava's loop over dim would)."""

    def __init__(self, orc, model, lanes: int = 16, per_row_quant: bool = False, drop: tuple = ()):
        self.orc, self.model = orc, model
        self.cfg = c = model.configuration
        self.om = orc.OracleModel(model, lanes=lanes, per_row_quant=per_row_quant)
        L = orc.lib()
        L.oracle_matmul.argtypes = [C.POINTER(orc.OModel), C.c_void_p, C.POINTER(orc.OTensor), C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]
        self._lib = L
        self.bias, self.neox = False, False
        self.drop = set(drop)
        if c.yarn is None and self.drop & {"mscale", "ramp"}:
            raise ValueError("a plain-table model has no YaRN terms to drop")
        self._rope_cr, self._rope_ci = rope_table(c.context_length, c.head_size, c.rope_theta, c.yarn, tuple(self.drop & {"mscale", "ramp"}))
        self._kc = np.zeros((c.n_layers, c.context_length, c.kv_dim), dtype=np.float32)
        self._vc = np.zeros_like(self._kc)
        self._emb = model.tensors["token_embd.weight"]

    def _rope(self, vec: np.ndarray, n_heads: int, pos: int) -> np.ndarray:
        out = super()._rope(vec, n_heads, pos)
        if "qdim" in self.drop and len(vec) > self.cfg.dim:
            out[self.cfg.dim:] = vec[self.cfg.dim:]  # `for (i = 0; i < dim; i += 2)`: the heads past dim stay unrotated
        return out
