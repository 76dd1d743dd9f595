"""Host-side mirror of the reference's sampler selection (``inference/sampler/Sampler.java:74-122``).

The reference copies the logits row to the host whenever ``temperature > 0`` and samples there
(``CategoricalSampler.java:28-40``, ``ToppSampler.java:62-156``).  Here the arithmetic runs on the device
(``csrc/sampler.cuh`` behind ``b200_forward_decode_sample``): per token 4 bytes go in -- the uniform number -- and 4 bytes
come out.  What stays on the host is the random stream itself, because it is host state in the reference too:
``RandomGeneratorFactory.getDefault().create(seed)`` = ``L32X64MixRandom`` (Sampler.java:84), restated below from the published
LXM algorithm (Steele & Vigna, OOPSLA 2021).  No JDK is available here, so the stream is unpinned against a JVM; the test suite
checks this restatement against the oracle's independent C restatement.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

M32 = 0xFFFFFFFF
MAX_LOGIT_BIAS = 1024  # B200_MAX_LOGIT_BIAS


def _mix_murmur32(z: int) -> int:
    z = ((z ^ (z >> 16)) * 0x85EBCA6B) & M32
    z = ((z ^ (z >> 13)) * 0xC2B2AE35) & M32
    return z ^ (z >> 16)


def _mix_lea32(z: int) -> int:
    z = ((z ^ (z >> 16)) * 0xD36D884B) & M32
    z = ((z ^ (z >> 16)) * 0xD36D884B) & M32
    return z ^ (z >> 16)


def _rotl32(v: int, k: int) -> int:
    return ((v << k) | (v >> (32 - k))) & M32


class L32X64MixRandom:
    """java.util.random default generator: 32-bit LCG (multiplier 0xadb4a92d) + xoroshiro64, mixed with mixLea32."""

    def __init__(self, seed: int):
        sd = (seed ^ 0x6A09E667F3BCC909) & 0xFFFFFFFFFFFFFFFF  # SILVER_RATIO_64
        self.a = _mix_murmur32(sd >> 32) | 1
        self.s = 1
        self.x0 = _mix_lea32(sd & M32)
        self.x1 = _mix_lea32(((sd & M32) + 0x9E3779B9) & M32)  # GOLDEN_RATIO_32
        if (self.x0 | self.x1) == 0:
            self.x0, self.x1 = 0x9E3779B9, 0x3C6EF372

    def next_int(self) -> int:
        result = _mix_lea32((self.s + self.x0) & M32)
        self.s = (0xADB4A92D * self.s + self.a) & M32
        q0, q1 = self.x0, self.x1
        q1 ^= q0
        q0 = _rotl32(q0, 26)
        q0 = q0 ^ q1 ^ ((q1 << 9) & M32)
        q1 = _rotl32(q1, 13)
        self.x0, self.x1 = q0, q1
        return result

    def next_float1(self) -> float:
        """RandomGenerator.nextFloat(1f): (nextInt() >>> 8) * 2^-24 (times the bound 1, always below it)."""
        return (self.next_int() >> 8) * (2.0 ** -24)


@dataclass(frozen=True)
class SamplingControls:
    """One sequence's sampling controls (b200_sampling_controls, include/b200llama.h): logit bias, llama.cpp's repetition /
    frequency / presence penalties over the sequence's token counts, top-k (every token tied at the k-th value is kept) and min-p
    (logit space, before temperature), applied on the device to the raw row before the sampler.  The defaults change nothing.
    logit_bias: {token id: added logit}."""
    top_k: int = 0
    min_p: float = 0.0
    repetition_penalty: float = 1.0
    frequency_penalty: float = 0.0
    presence_penalty: float = 0.0
    logit_bias: dict | None = None

    def validate(self, vocabulary_size: int) -> "SamplingControls":
        """Raises ValueError where b200_set_sampling_controls returns B200_ERR_BAD_ARG; returns self."""
        if not 0 <= int(self.top_k) <= vocabulary_size:
            raise ValueError(f"top_k = {self.top_k} outside [0, {vocabulary_size}]")
        if not 0.0 <= self.min_p <= 1.0:
            raise ValueError(f"min_p = {self.min_p} outside [0, 1]")
        if not (math.isfinite(self.repetition_penalty) and self.repetition_penalty > 0.0):
            raise ValueError(f"repetition_penalty = {self.repetition_penalty}: must be finite and > 0")
        if not (math.isfinite(self.frequency_penalty) and math.isfinite(self.presence_penalty)):
            raise ValueError(f"frequency_penalty = {self.frequency_penalty}, presence_penalty = {self.presence_penalty}: must be finite")
        bias = self.logit_bias or {}
        if len(bias) > MAX_LOGIT_BIAS:
            raise ValueError(f"{len(bias)} logit_bias entries: at most {MAX_LOGIT_BIAS}")
        for i, b in bias.items():
            if not 0 <= int(i) < vocabulary_size:
                raise ValueError(f"logit_bias id {i} out of range")
            if not math.isfinite(b):
                raise ValueError(f"logit_bias[{i}] = {b} is not finite")
        return self


class Sampler:
    """``Sampler.selectSampler(vocabulary_size, temperature, topp, rngSeed)``: greedy when temperature == 0, otherwise
    temperature + softmax + categorical (topp outside (0,1)) or top-p sampling.  ``sample_token`` runs one decode forward and
    returns the sampled id; the logits never leave the GPU.

    controls (optional SamplingControls) and history (optional token ids, e.g. the prompt, counted by the penalties): with controls,
    every token goes through forward_decode_sample, temperature 0 included, and the device applies them to the plan's own sequence
    (slot -1).  The sampler's counts are its history plus every id it has emitted; whenever slot -1 does not hold this sampler's
    controls and counts (another sampler or the caller set controls there, or kv_reset cleared the counts), sample_token installs
    them again first.  Without controls, sample_token first turns off any controls left on slot -1, so a plain sampler samples the
    raw model whatever ran before it.  The RNG draws one next_float1() per token when temperature > 0 and none otherwise, with or
    without controls."""

    def __init__(self, vocabulary_size: int, temperature: float, topp: float, rng_seed: int, controls: SamplingControls | None = None,
                 history=None):
        self.vocabulary_size = vocabulary_size
        self.temperature = float(temperature)
        self.topp = float(topp)
        self.rng = None if self.temperature == 0.0 else L32X64MixRandom(rng_seed)
        self.controls = None if controls is None else controls.validate(vocabulary_size)
        self.history = [int(t) for t in (history or [])]
        if any(not 0 <= t < vocabulary_size for t in self.history):
            raise ValueError("history token out of range")
        self.counted = list(self.history)  # then each id sample_token emits

    def sample_token(self, plan, token: int, position: int) -> int:
        if self.controls is not None:
            if plan.sampling_controls_owner(-1) is not self:
                plan.set_sampling_controls(-1, self.controls, owner=self)
                plan.set_sample_history(-1, self.counted)
            u = 0.0 if self.temperature == 0.0 else self.rng.next_float1()
            tok = plan.forward_decode_sample(token, position, self.temperature, self.topp, u)
            self.counted.append(tok)
            return tok
        if getattr(plan, "sampling_controls", lambda slot: None)(-1) is not None:  # a stand-in plan without controls: none to clear
            plan.set_sampling_controls(-1, None)
        if self.temperature == 0.0:
            return plan.forward_decode(token, position, logits=False)[1]
        return plan.forward_decode_sample(token, position, self.temperature, self.topp, self.rng.next_float1())


def select_sampler(vocabulary_size: int, temperature: float, topp: float, rng_seed: int) -> Sampler:
    return Sampler(vocabulary_size, temperature, topp, rng_seed)
