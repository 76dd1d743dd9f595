"""Token-generation loops over the plan: the callers of the hot path.

Position/token conventions decide parity, so they are restated exactly:
``generate_tokens_llama``  <- InferenceEngine.generateTokensGPULlama / generateTokensLlama
                              (inference/InferenceEngine.java:81-154, 293-381)
``generate_tokens_qwen3``  <- InferenceEngine.generateTokensQwen3 (InferenceEngine.java:156-234),
                              including its skipped position after the last prompt token
``generate_tokens_llama_batch_prefill`` <- InferenceEngineWithBatchPrefillDecode.generateTokensGPULlama
                              (InferenceEngineWithBatchPrefillDecode.java:163-251)
The sampler is greedy (temperature 0 -> FloatTensor.argmax, Sampler.java:124-132) and runs on
the device; ``forward`` is any callable (token, position) -> argmax so the same loops drive
the oracle in the tests.
"""
from __future__ import annotations

from typing import Callable, Iterable

Forward = Callable[[int, int], int]


def generate_tokens_llama(forward: Forward, latest_token: int, start_position: int, prompt_tokens: list[int],
                          stop_tokens: Iterable[int], max_tokens: int, context_length: int) -> list[int]:
    if max_tokens < 0 or context_length < max_tokens:
        max_tokens = context_length
    stop = set(stop_tokens)
    generated: list[int] = []
    current, prompt_index, pos = latest_token, 0, start_position
    while pos < max_tokens:
        am = forward(current, pos)
        if prompt_index < len(prompt_tokens):
            nxt = prompt_tokens[prompt_index]
            prompt_index += 1
        else:
            nxt = am
            generated.append(nxt)
            if nxt in stop:
                break
        current = nxt
        pos += 1
    return generated


def generate_tokens_qwen3(forward: Forward, latest_token: int, start_position: int, prompt_tokens: list[int],
                          stop_tokens: Iterable[int], max_tokens: int, context_length: int) -> list[int]:
    if max_tokens < 0 or context_length < max_tokens:
        max_tokens = context_length
    stop = set(stop_tokens)
    generated: list[int] = []
    current, prompt_index = latest_token, 0
    position = start_position
    while position < max_tokens:
        if prompt_index < len(prompt_tokens):
            am = forward(prompt_tokens[prompt_index], position)
            prompt_index += 1
            if prompt_index < len(prompt_tokens):
                position += 1
                continue
            position += 1  # "The current logit belongs to the next position" (InferenceEngine.java:194)
        else:
            am = forward(current, position)
        nxt = am
        generated.append(nxt)
        if nxt in stop:
            break
        current = nxt
        position += 1
    return generated


def loop_for(model_type: str):
    """The generation loop the reference's model class uses: Qwen3, Qwen2 and DeepSeek-R1-Distill-Qwen run generateTokensQwen3
    (Qwen3.java, Qwen2.java:95-115), the others generateTokensLlama."""
    return generate_tokens_qwen3 if model_type.upper() in ("QWEN_3", "QWEN_2", "DEEPSEEK_R1_DISTILL_QWEN") else generate_tokens_llama


def generate_tokens_llama_batch_prefill(plan, latest_token: int, start_position: int, prompt_tokens: list[int],
                                        stop_tokens: Iterable[int], max_tokens: int, context_length: int, batch_size: int) -> list[int]:
    """prefillSeq = [latestToken, prompt[0..N-2]] at positions startPosition.. in chunks of B through the batched
    prefill, clamped to the token budget, then decode from the last prompt token at startPosition+N
    (InferenceEngineWithBatchPrefillDecode.java:163-251; the chunk clamp is :204-205)."""
    if max_tokens < 0 or context_length < max_tokens:
        max_tokens = context_length
    stop = set(stop_tokens)
    n = len(prompt_tokens)
    if n == 0:
        raise IndexError("empty prompt (the reference's promptTokens.get(N - 1) throws as well)")
    seq = [latest_token] + list(prompt_tokens[: n - 1])
    pos = start_position
    chunk_start = 0
    while chunk_start < n and pos + chunk_start < max_tokens:
        chunk_end = min(chunk_start + batch_size, n, max_tokens - pos)
        plan.forward_batch_prefill(seq[chunk_start:chunk_end], pos + chunk_start)
        chunk_start += batch_size
    generated: list[int] = []
    current, pos = prompt_tokens[n - 1], start_position + n
    while pos < max_tokens:
        _, nxt = plan.forward_decode(current, pos, logits=False)
        generated.append(nxt)
        if nxt in stop:
            break
        current = nxt
        pos += 1
    return generated
