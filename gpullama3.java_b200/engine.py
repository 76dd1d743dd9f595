"""Token-generation loops over the plan: the callers of the hot path.

Position/token conventions decide parity, so they are restated exactly:
``generate_tokens_llama``  <- InferenceEngine.generateTokensGPULlama / generateTokensLlama
                              (inference/InferenceEngine.java:81-154, 293-381)
``generate_tokens_qwen3``  <- InferenceEngine.generateTokensQwen3 (InferenceEngine.java:156-234),
                              including its skipped position after the last prompt token
``generate_tokens_llama_batch_prefill`` <- InferenceEngineWithBatchPrefillDecode.generateTokensGPULlama
                              (InferenceEngineWithBatchPrefillDecode.java:163-251)
``generate_tokens_batch``  several requests through the first two loops in lockstep on the plan's decode slots
``generate_tokens_batch_prefill`` the third loop for several requests: prompts prefilled straight into the decode slots
                              (prefill_slots), then lockstep decode
``generate_tokens_lookahead`` the first loop, several positions verified per step (forward_decode_multi): the rest of the
                              prompt, or drafted tokens, checked in one weight stream; the same ids for any draft
The sampler is greedy (temperature 0 -> FloatTensor.argmax, Sampler.java:124-132) and runs on
the device; ``forward`` is any callable (token, position) -> argmax so the same loops drive
the oracle in the tests.
"""
from __future__ import annotations

from typing import Callable, Iterable

Forward = Callable[[int, int], int]


def _llama_steps(latest_token: int, start_position: int, prompt_tokens: list[int], stop_tokens: Iterable[int], max_tokens: int,
                 context_length: int):
    """generate_tokens_llama as a generator: yields each forward's (token, position), receives its argmax, returns the ids."""
    if max_tokens < 0 or context_length < max_tokens:
        max_tokens = context_length
    stop = set(stop_tokens)
    generated: list[int] = []
    current, prompt_index, pos = latest_token, 0, start_position
    while pos < max_tokens:
        am = yield current, pos
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


def _qwen3_steps(latest_token: int, start_position: int, prompt_tokens: list[int], stop_tokens: Iterable[int], max_tokens: int,
                 context_length: int):
    """generate_tokens_qwen3 as a generator (see _llama_steps)."""
    if max_tokens < 0 or context_length < max_tokens:
        max_tokens = context_length
    stop = set(stop_tokens)
    generated: list[int] = []
    current, prompt_index = latest_token, 0
    position = start_position
    while position < max_tokens:
        if prompt_index < len(prompt_tokens):
            am = yield prompt_tokens[prompt_index], position
            prompt_index += 1
            if prompt_index < len(prompt_tokens):
                position += 1
                continue
            position += 1  # "The current logit belongs to the next position" (InferenceEngine.java:194)
        else:
            am = yield current, position
        nxt = am
        generated.append(nxt)
        if nxt in stop:
            break
        current = nxt
        position += 1
    return generated


def _drive(steps, forward: Forward) -> list[int]:
    try:
        req = next(steps)
        while True:
            req = steps.send(forward(*req))
    except StopIteration as done:
        return done.value


def generate_tokens_llama(forward: Forward, latest_token: int, start_position: int, prompt_tokens: list[int],
                          stop_tokens: Iterable[int], max_tokens: int, context_length: int) -> list[int]:
    return _drive(_llama_steps(latest_token, start_position, prompt_tokens, stop_tokens, max_tokens, context_length), forward)


def generate_tokens_qwen3(forward: Forward, latest_token: int, start_position: int, prompt_tokens: list[int],
                          stop_tokens: Iterable[int], max_tokens: int, context_length: int) -> list[int]:
    return _drive(_qwen3_steps(latest_token, start_position, prompt_tokens, stop_tokens, max_tokens, context_length), forward)


def loop_for(model_type: str):
    """The generation loop the reference's model class uses: Qwen3, Qwen2, Qwen2-MoE and DeepSeek-R1-Distill-Qwen run
    generateTokensQwen3 (Qwen3.java, Qwen2.java:95-115, Qwen2MoE.java:84-98), the others generateTokensLlama (Granite's
    generateTokensGranite is generateTokensLlama with forwardGranite, InferenceEngine.java:554-616)."""
    return generate_tokens_qwen3 if _is_qwen_loop(model_type) else generate_tokens_llama


def _is_qwen_loop(model_type: str) -> bool:
    return model_type.upper() in ("QWEN_3", "QWEN_2", "QWEN_2_MOE", "DEEPSEEK_R1_DISTILL_QWEN")


def generate_tokens_batch(plan, model_type: str, requests: list, stop_tokens: Iterable[int], max_tokens: int,
                          context_length: int) -> list[list[int]]:
    """Several independent generations in lockstep on the plan's decode slots (request i on slot i, reset first): one
    forward_decode_batch per step for every request still running.  Each request is (latest_token, start_position,
    prompt_tokens) and follows the loop loop_for(model_type) runs, so each result equals that loop's for the request alone;
    a request leaves the batch at its stop token or budget."""
    n_slots = plan.batch_info()[0]
    if len(requests) > n_slots:
        raise ValueError(f"{len(requests)} requests but the plan has {n_slots} decode slots (set_decode_slots)")
    make = _qwen3_steps if _is_qwen_loop(model_type) else _llama_steps
    stop = list(stop_tokens)
    results: list = [None] * len(requests)
    live: dict = {}  # request index -> (generator, pending (token, position))
    for i, (latest, start, prompt) in enumerate(requests):
        plan.slot_reset(i)
        g = make(latest, start, list(prompt), stop, max_tokens, context_length)
        try:
            live[i] = (g, next(g))
        except StopIteration as done:
            results[i] = done.value
    while live:
        rows = sorted(live)
        ids, _ = plan.forward_decode_batch(rows, [live[i][1][0] for i in rows], [live[i][1][1] for i in rows])
        for i, am in zip(rows, ids):
            g = live[i][0]
            try:
                live[i] = (g, g.send(int(am)))
            except StopIteration as done:
                results[i] = done.value
                del live[i]
    return results


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


def generate_tokens_batch_prefill(plan, model_type: str, requests: list, stop_tokens: Iterable[int], max_tokens: int,
                                  context_length: int, batch_size: int) -> list[list[int]]:
    """The batched counterpart of generate_tokens_llama_batch_prefill on the plan's decode slots (request i on slot i).  Each request
    (latest_token, start_position, prompt_tokens) prefills [latest] + prompt[:-1] into its slot, clamped to the token budget as that
    function clamps it; the prompts of all requests are packed into prefill_slots calls of at most batch_size tokens (a prompt may
    span two calls).  Then every request decodes in lockstep through forward_decode_batch from prompt[-1] at start + len(prompt)
    until its stop token or the budget, so each result equals generate_tokens_llama_batch_prefill for the request alone.  Only the
    Llama loop has this form: a slot's rows past its prompt are never read, so the slots are not reset first."""
    if _is_qwen_loop(model_type):
        raise ValueError(f"{model_type} runs the Qwen3 loop, which has no batched-prefill form: use generate_tokens_batch")
    n_slots = plan.batch_info()[0]
    if len(requests) > n_slots:
        raise ValueError(f"{len(requests)} requests but the plan has {n_slots} decode slots (set_decode_slots)")
    if batch_size < 1:
        raise ValueError("batch_size must be >= 1")
    if max_tokens < 0 or context_length < max_tokens:
        max_tokens = context_length
    stop = set(stop_tokens)
    todo = []  # per request: (slot, first position, tokens still to prefill)
    for i, (latest, start, prompt) in enumerate(requests):
        n = len(prompt)
        if n == 0:
            raise IndexError("empty prompt (the reference's promptTokens.get(N - 1) throws as well)")
        seq = [latest] + list(prompt[: n - 1])
        todo.append([i, start, seq[: max(0, min(n, max_tokens - start))]])
    while any(t[2] for t in todo):
        slots, starts, pieces, room = [], [], [], batch_size
        for t in todo:
            if room == 0:
                break
            if t[2]:
                take = min(room, len(t[2]))
                slots.append(t[0]); starts.append(t[1]); pieces.append(t[2][:take])
                t[1] += take
                t[2] = t[2][take:]
                room -= take
        plan.prefill_slots(slots, starts, pieces)
    results: list = [[] for _ in requests]
    live = {i: (int(prompt[-1]), start + len(prompt)) for i, (_, start, prompt) in enumerate(requests) if start + len(prompt) < max_tokens}
    while live:
        rows = sorted(live)
        ids, _ = plan.forward_decode_batch(rows, [live[i][0] for i in rows], [live[i][1] for i in rows])
        for i, am in zip(rows, ids):
            nxt = int(am)
            results[i].append(nxt)
            pos = live[i][1] + 1
            if nxt in stop or pos >= max_tokens:
                del live[i]
            else:
                live[i] = (nxt, pos)
    return results


def prompt_lookup(history: list[int], max_tokens: int = 8) -> list[int]:
    """Draft by prompt lookup: the tokens that followed the most recent earlier occurrence of the history's last 3, 2 or 1 tokens
    (the longest suffix that recurs wins), at most max_tokens of them; [] when none recurs."""
    n = len(history)
    for k in (3, 2, 1):
        if n <= k:
            continue
        tail = history[n - k:]
        for j in range(n - k - 1, -1, -1):
            if history[j:j + k] == tail:
                return list(history[j + k:j + k + max_tokens])
    return []


def generate_tokens_lookahead(plan, model_type: str, latest_token: int, start_position: int, prompt_tokens: list[int],
                              stop_tokens: Iterable[int], max_tokens: int, context_length: int,
                              draft: Callable[[list[int]], list[int]] = prompt_lookup, stats: dict | None = None) -> list[int]:
    """generate_tokens_llama on the plan's own cache, verifying several positions per step with forward_decode_multi.

    Each step runs [current] + drafts (up to decode_multi_rows() - 1 drafts) at consecutive positions.  While prompt tokens remain
    the drafts are the rest of the prompt; after that draft(history) proposes them, history being [latest_token] + prompt + the
    tokens generated so far.  The rows are then walked as generate_tokens_llama walks its steps: a prompt token is taken whatever
    the id says, a generated token is the row's id, and the walk goes on to the next row only while that row's input equals the
    token just taken.  A stop token or the budget ends generation at the same token as there.  Every row is bit-identical to
    forward_decode of its token over the same cache prefix, and a rejected draft's K/V rows are rewritten before any later row
    reads them, so the result equals generate_tokens_llama for any draft function.  stats (optional dict) receives the steps run,
    the drafted tokens that were generated rather than forced, and how many of those were accepted.

    Llama loop only: the Qwen3 loop reads a skipped position as a zero row, which a rejected draft may have written."""
    if _is_qwen_loop(model_type):
        raise ValueError(f"{model_type} runs the Qwen3 loop, which has no lookahead form: use generate_tokens_qwen3")
    rows = plan.decode_multi_rows()
    if rows < 1:
        raise ValueError("the plan cannot run multi-position steps (decode_multi_rows() == 0)")
    if max_tokens < 0 or context_length < max_tokens:
        max_tokens = context_length
    stop = set(stop_tokens)
    prompt = list(prompt_tokens)
    history = [latest_token] + prompt
    generated: list[int] = []
    current, prompt_index, pos = latest_token, 0, start_position
    steps = drafted = accepted = 0
    while pos < max_tokens:
        forced = prompt_index < len(prompt)
        guesses = prompt[prompt_index:] if forced else list(draft(list(history)))
        guesses = [int(t) for t in guesses[:min(rows, max_tokens - pos) - 1]]
        ids, _ = plan.forward_decode_multi(-1, [current] + guesses, pos)
        steps += 1
        for i, am in enumerate(ids):
            if prompt_index < len(prompt):
                nxt = prompt[prompt_index]
                prompt_index += 1
            else:
                nxt = int(am)
                generated.append(nxt)
                history.append(nxt)
                if i < len(guesses) and not forced:
                    drafted += 1
                    accepted += guesses[i] == nxt
                if nxt in stop:
                    pos = max_tokens  # ends the outer loop too
                    break
            current = nxt
            pos += 1
            if i == len(guesses) or guesses[i] != nxt:
                break
    if stats is not None:
        stats.update(steps=steps, drafted=drafted, accepted=accepted)
    return generated
