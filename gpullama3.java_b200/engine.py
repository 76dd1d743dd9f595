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
``ContinuousBatcher`` / ``generate_tokens_continuous`` the first two loops for a stream of requests: decode rows of running
                              requests and prompt rows of newly admitted ones share each forward_step (or, opted in, each
                              forward_chunk on the tensor cores), and freed slots are refilled from a queue
``score_sequence`` / ``perplexity`` teacher-forced scoring of a given text (plan.score_tokens) in chunks the plan accepts
The plan-driven loops take an optional ``logprobs`` list: with the plan's log-probabilities on (plan.set_logprobs(N)) it receives
one entry (chosen, [(id, logprob), ...]) per generated id -- per request, one list per request -- from plan.last_logprobs().
``generate_tokens_llama`` / ``_qwen3`` take a callable; it reads them itself, e.g.
    def forward(tok, pos):
        _, am = plan.forward_decode(tok, pos, logits=False)
        rows.append(plan.last_logprobs())  # the row of the id just emitted
        return am
The sampler is greedy (temperature 0 -> FloatTensor.argmax, Sampler.java:124-132) and runs on
the device; ``forward`` is any callable (token, position) -> argmax so the same loops drive
the oracle in the tests.
"""
from __future__ import annotations

import math
import time
from collections import deque
from typing import Callable, Iterable

import numpy as np

Forward = Callable[[int, int], int]


def _llama_steps(latest_token: int, start_position: int, prompt_tokens: list[int], stop_tokens: Iterable[int], max_tokens: int,
                 context_length: int, generated: list | None = None):
    """generate_tokens_llama as a generator: yields each forward's (token, position), receives its argmax, returns the ids
    (`generated` if given, so a caller can see which results became ids)."""
    if max_tokens < 0 or context_length < max_tokens:
        max_tokens = context_length
    stop = set(stop_tokens)
    generated = [] if generated is None else generated
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
                 context_length: int, generated: list | None = None):
    """generate_tokens_qwen3 as a generator (see _llama_steps)."""
    if max_tokens < 0 or context_length < max_tokens:
        max_tokens = context_length
    stop = set(stop_tokens)
    generated = [] if generated is None else generated
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
    """The generation loop the reference's model class uses: Qwen3, Qwen3-MoE, Qwen2, Qwen2-MoE and DeepSeek-R1-Distill-Qwen run
    generateTokensQwen3 (Qwen3.java, Qwen2.java:95-115, Qwen2MoE.java:84-98), the others generateTokensLlama (Granite's
    generateTokensGranite is generateTokensLlama with forwardGranite, InferenceEngine.java:554-616)."""
    return generate_tokens_qwen3 if _is_qwen_loop(model_type) else generate_tokens_llama


def _is_qwen_loop(model_type: str) -> bool:
    return model_type.upper() in ("QWEN_3", "QWEN_3_MOE", "QWEN_2", "QWEN_2_MOE", "DEEPSEEK_R1_DISTILL_QWEN")


def _logprob_rows(plan) -> list:
    """plan.last_logprobs() as one (chosen, [(id, logprob), ...]) entry per row of the last emitting call."""
    chosen, ids, lps = plan.last_logprobs()
    return [(float(chosen[r]), [(int(i), float(v)) for i, v in zip(ids[r], lps[r])]) for r in range(len(chosen))]


def generate_tokens_batch(plan, model_type: str, requests: list, stop_tokens: Iterable[int], max_tokens: int,
                          context_length: int, logprobs: list | None = None) -> list[list[int]]:
    """Several independent generations in lockstep on the plan's decode slots (request i on slot i, reset first): one
    forward_decode_batch per step for every request still running.  Each request is (latest_token, start_position,
    prompt_tokens) and follows the loop loop_for(model_type) runs, so each result equals that loop's for the request alone;
    a request leaves the batch at its stop token or budget.  logprobs (optional list, plan.set_logprobs on) receives one list per
    request, one entry per generated id."""
    n_slots = plan.batch_info()[0]
    if len(requests) > n_slots:
        raise ValueError(f"{len(requests)} requests but the plan has {n_slots} decode slots (set_decode_slots)")
    make = _qwen3_steps if _is_qwen_loop(model_type) else _llama_steps
    stop = list(stop_tokens)
    results: list = [None] * len(requests)
    gen = [[] for _ in requests]
    lp = [[] for _ in requests]
    if logprobs is not None:
        logprobs.extend(lp)
    live: dict = {}  # request index -> (generator, pending (token, position))
    for i, (latest, start, prompt) in enumerate(requests):
        plan.slot_reset(i)
        g = make(latest, start, list(prompt), stop, max_tokens, context_length, gen[i])
        try:
            live[i] = (g, next(g))
        except StopIteration as done:
            results[i] = done.value
    while live:
        rows = sorted(live)
        ids, _ = plan.forward_decode_batch(rows, [live[i][1][0] for i in rows], [live[i][1][1] for i in rows])
        entries = _logprob_rows(plan) if logprobs is not None else None
        for k, (i, am) in enumerate(zip(rows, ids)):
            g = live[i][0]
            n0 = len(gen[i])
            try:
                live[i] = (g, g.send(int(am)))
            except StopIteration as done:
                results[i] = done.value
                del live[i]
            if entries is not None and len(gen[i]) > n0:  # the row's id became a generated token
                lp[i].append(entries[k])
    return results


def generate_tokens_llama_batch_prefill(plan, latest_token: int, start_position: int, prompt_tokens: list[int],
                                        stop_tokens: Iterable[int], max_tokens: int, context_length: int, batch_size: int,
                                        logprobs: list | None = None) -> list[int]:
    """prefillSeq = [latestToken, prompt[0..N-2]] at positions startPosition.. in chunks of B through the batched
    prefill, clamped to the token budget, then decode from the last prompt token at startPosition+N
    (InferenceEngineWithBatchPrefillDecode.java:163-251; the chunk clamp is :204-205).  logprobs (optional list, plan.set_logprobs
    on) receives one entry per generated id."""
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
        if logprobs is not None:
            logprobs.extend(_logprob_rows(plan))
        if nxt in stop:
            break
        current = nxt
        pos += 1
    return generated


def generate_tokens_batch_prefill(plan, model_type: str, requests: list, stop_tokens: Iterable[int], max_tokens: int,
                                  context_length: int, batch_size: int, logprobs: list | None = None) -> list[list[int]]:
    """The batched counterpart of generate_tokens_llama_batch_prefill on the plan's decode slots (request i on slot i).  Each request
    (latest_token, start_position, prompt_tokens) prefills [latest] + prompt[:-1] into its slot, clamped to the token budget as that
    function clamps it; the prompts of all requests are packed into prefill_slots calls of at most batch_size tokens (a prompt may
    span two calls).  Then every request decodes in lockstep through forward_decode_batch from prompt[-1] at start + len(prompt)
    until its stop token or the budget, so each result equals generate_tokens_llama_batch_prefill for the request alone.  Only the
    Llama loop has this form: a slot's rows past its prompt are never read, so the slots are not reset first.  logprobs (optional
    list, plan.set_logprobs on) receives one list per request, one entry per generated id."""
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
    lp = [[] for _ in requests]
    if logprobs is not None:
        logprobs.extend(lp)
    live = {i: (int(prompt[-1]), start + len(prompt)) for i, (_, start, prompt) in enumerate(requests) if start + len(prompt) < max_tokens}
    while live:
        rows = sorted(live)
        ids, _ = plan.forward_decode_batch(rows, [live[i][0] for i in rows], [live[i][1] for i in rows])
        entries = _logprob_rows(plan) if logprobs is not None else None
        for k, (i, am) in enumerate(zip(rows, ids)):
            nxt = int(am)
            results[i].append(nxt)
            if entries is not None:
                lp[i].append(entries[k])
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
                              draft: Callable[[list[int]], list[int]] = prompt_lookup, stats: dict | None = None,
                              logprobs: list | None = None) -> list[int]:
    """generate_tokens_llama on the plan's own cache, verifying several positions per step with forward_decode_multi.

    Each step runs [current] + drafts (up to decode_multi_rows() - 1 drafts) at consecutive positions.  While prompt tokens remain
    the drafts are the rest of the prompt; after that draft(history) proposes them, history being [latest_token] + prompt + the
    tokens generated so far.  The rows are then walked as generate_tokens_llama walks its steps: a prompt token is taken whatever
    the id says, a generated token is the row's id, and the walk goes on to the next row only while that row's input equals the
    token just taken.  A stop token or the budget ends generation at the same token as there.  Every row is bit-identical to
    forward_decode of its token over the same cache prefix, and a rejected draft's K/V rows are rewritten before any later row
    reads them, so the result equals generate_tokens_llama for any draft function.  stats (optional dict) receives the steps run,
    the drafted tokens that were generated rather than forced, and how many of those were accepted.

    logprobs (optional list, plan.set_logprobs on) receives one entry per generated id: the accepted rows' only.

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
        entries = _logprob_rows(plan) if logprobs is not None else None
        steps += 1
        for i, am in enumerate(ids):
            if prompt_index < len(prompt):
                nxt = prompt[prompt_index]
                prompt_index += 1
            else:
                nxt = int(am)
                generated.append(nxt)
                history.append(nxt)
                if entries is not None:
                    logprobs.append(entries[i])
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


class _Request:
    __slots__ = ("rid", "steps", "sampler", "kv_left", "limit", "row", "slot", "generated")

    def __init__(self, rid, steps, sampler, kv_rows, limit):
        self.rid, self.steps, self.sampler, self.kv_left = rid, steps, sampler, kv_rows
        self.limit = limit  # the loop's clamped max_tokens: it yields positions below it only
        self.row = None  # the (token, position) the loop asks for next
        self.slot = -1
        self.generated = 0

    def rows_left(self) -> int:
        """Rows the request can put into one step: its decode row, or its prompt rows up to and including the emitting one (prompt
        rows sit at consecutive positions, and the loop ends at the first position >= limit)."""
        if self.generated:
            return 1
        return min(self.kv_left + 1, self.limit - self.row[1])


class ContinuousBatcher:
    """Continuous batching over the plan's decode slots: requests queue, are admitted first in, first out into free slots, and share
    each forward_step with the requests already generating.

    A step holds at most decode_multi_rows() rows: first one emitting row for every request that has generated a token, then the
    prompt rows of the requests still in their prompt, in admission order, as many as fit.  A request's rows are exactly the
    (token, position) sequence loop_for(model_type) runs for it -- the Llama loop's K/V-only rows are latest + prompt[:-1], the
    Qwen3 loop's prompt[:-1] -- so a prompt may span several steps, and its last row, which yields the first generated token,
    emits.  Both loops' budget clamps and the Qwen3 loop's skipped position come with the loop; slot_reset at admission makes the
    skipped row read as zero.  A request ends at its stop token or budget and its slot takes the next queued request in the same
    step().  Every forward_step row is bit-identical to forward_decode of its sequence alone, so each request's ids equal its loop
    run alone on one slot, greedy or sampled with the same seed, whatever else shares the steps.

    chunk_rows > 0 admits prompts on the tensor cores (the plan in set_prefill_mode("tensor_core_exact")): a step gathers its rows
    the same way with a budget of chunk_rows, capped at plan.chunk_rows(), and runs them as one forward_chunk when at least
    min_chunk_rows rows are available; otherwise it is today's step of decode_multi_rows() rows through forward_step.  forward_chunk
    is bit-identical to forward_step on the same rows, so every request's ids are its loop's alone whichever call a step takes.  The
    default of 32 rows is where the int8 prefill overtakes the exact multi-position step on prompts alone (DESIGN.md section 6); a
    starting point, not a tuned value.  chunk_rows = 0 (the default) never calls forward_chunk.

    sampler (optional, per request): a sampler.Sampler; one next_float1() is drawn per generated token, never for a prompt row, as
    generateTokensLlama draws it (InferenceEngine.java:81-154).  Without chunk_rows the steps are always the exact mixed steps,
    whatever the plan's prefill mode.  A sampler's controls (sampler.SamplingControls) and history go onto the request's slot at
    admission, after slot_reset (a request without controls turns its slot's off); the device applies them to the request's emitting
    rows.

    When the plan's log-probabilities are on (plan.set_logprobs), logprobs[rid] receives one entry (chosen, [(id, logprob), ...])
    per generated id, next to results[rid]."""

    def __init__(self, plan, model_type: str, stop_tokens: Iterable[int], max_tokens: int, context_length: int, chunk_rows: int = 0,
                 min_chunk_rows: int = 32):
        self.plan = plan
        self.rows = plan.decode_multi_rows()
        if self.rows < 1:
            raise ValueError("the plan cannot run mixed steps (decode_multi_rows() == 0)")
        n_slots = plan.batch_info()[0]
        if n_slots < 1:
            raise ValueError("the plan has no decode slots (set_decode_slots)")
        if chunk_rows < 0 or min_chunk_rows < 1:
            raise ValueError(f"chunk_rows = {chunk_rows} must be >= 0 and min_chunk_rows = {min_chunk_rows} >= 1")
        self.chunk_rows = 0
        if chunk_rows:
            cap = plan.chunk_rows()
            if cap < 1:
                raise ValueError("the plan cannot run chunk steps (chunk_rows() == 0: set_prefill_mode('tensor_core_exact') first)")
            self.chunk_rows = min(chunk_rows, cap)
        self.min_chunk_rows = min_chunk_rows
        self.qwen = _is_qwen_loop(model_type)
        self.stop = list(stop_tokens)
        self.max_tokens, self.context_length = max_tokens, context_length
        self.results: dict = {}  # request id -> generated ids so far
        self.logprobs: dict = {}  # request id -> their log-probability entries (the plan's logprobs on)
        self.last_rows = 0  # rows of the last step() (0: no step ran)
        self.last_kind = None  # "step" (forward_step) or "chunk" (forward_chunk) of the last step() that ran
        self._queue: deque = deque()
        self._free = list(range(n_slots))
        self._running: list = []  # admitted requests, in admission order
        self._next_id = 0

    def submit(self, latest_token: int, start_position: int, prompt_tokens: list[int], sampler=None) -> int:
        """Queue one request (the arguments of generate_tokens_llama / generate_tokens_qwen3); returns its id."""
        if start_position < 0:
            raise ValueError(f"start_position {start_position} is negative")
        prompt = [int(t) for t in prompt_tokens]
        make = _qwen3_steps if self.qwen else _llama_steps
        steps = make(int(latest_token), int(start_position), prompt, self.stop, self.max_tokens, self.context_length)
        rid = self._next_id
        self._next_id += 1
        self.results[rid] = []
        self.logprobs[rid] = []
        limit = self.context_length if self.max_tokens < 0 or self.context_length < self.max_tokens else self.max_tokens
        self._queue.append(_Request(rid, steps, sampler, max(len(prompt) - 1, 0) if self.qwen else len(prompt), limit))
        return rid

    def pending(self) -> int:
        """Requests queued but not admitted."""
        return len(self._queue)

    def running(self) -> int:
        """Requests holding a slot."""
        return len(self._running)

    def _admit(self, out: list):
        while self._queue and self._free:
            r = self._queue.popleft()
            try:
                r.row = next(r.steps)
            except StopIteration:  # the budget ends it before its first row
                out.append((r.rid, None, True))
                continue
            r.slot = self._free.pop(0)
            self.plan.slot_reset(r.slot)
            controls = getattr(r.sampler, "controls", None)
            if controls is not None or hasattr(self.plan, "set_sampling_controls"):  # a stand-in plan without them: no controls
                self.plan.set_sampling_controls(r.slot, controls)
                if controls is not None:
                    self.plan.set_sample_history(r.slot, r.sampler.history)
            self._running.append(r)

    def _advance(self, r: _Request, am) -> bool:
        """Send the row's result to the loop; False when the loop has ended."""
        try:
            r.row = r.steps.send(am)
            return True
        except StopIteration:
            r.row = None
            return False

    def step(self) -> list:
        """Admit what fits, run one mixed step, and return (request id, token, finished) per generated token, in row order.  A
        request that ends without generating a token (its budget) is reported as (request id, None, True).  A step with no rows
        is not run."""
        out: list = []
        self._admit(out)
        rows, emit = [], []  # rows: (slot, token, position, emit, temperature, topp, uniform01); emit: the emitting rows' requests
        ended = []  # requests whose loop ended on a K/V-only row of this step

        def add(r, emitting):
            smp = r.sampler if emitting else None
            if smp is not None and smp.temperature != 0.0:
                rows.append((r.slot, r.row[0], r.row[1], 1, smp.temperature, smp.topp, smp.rng.next_float1()))
            else:
                rows.append((r.slot, r.row[0], r.row[1], int(emitting), 0.0, 0.0, 0.0))
            if emitting:
                emit.append(r)

        budget, chunk = self.rows, False
        if self.chunk_rows:
            chunk = min(sum(r.rows_left() for r in self._running if r.row is not None), self.chunk_rows) >= self.min_chunk_rows
            if chunk:
                budget = self.chunk_rows
        for r in self._running:  # one decode row per generating request
            if r.generated:
                add(r, True)
        for r in self._running:  # then the prompts, in admission order
            while not r.generated and r.row is not None and len(rows) < budget:
                if r.kv_left == 0:
                    add(r, True)
                    break
                add(r, False)
                r.kv_left -= 1
                if not self._advance(r, -1):  # a K/V-only row: the loop does not read its result
                    ended.append(r)
        self.last_rows = len(rows)
        if rows:
            ids, _ = (self.plan.forward_chunk if chunk else self.plan.forward_step)(rows)
            self.last_kind = "chunk" if chunk else "step"
            lp_on = getattr(self.plan, "logprobs_top_n", lambda: -1)() >= 0  # a stand-in plan without log-probabilities: off
            entries = _logprob_rows(self.plan) if lp_on else None
            done = list(ended)
            k = 0
            for j, (row, am) in enumerate(zip(rows, ids)):
                if not row[3]:
                    continue
                r = emit[k]
                k += 1
                tok = int(am)
                self.results[r.rid].append(tok)
                if entries is not None:
                    self.logprobs[r.rid].append(entries[j])
                r.generated += 1
                alive = self._advance(r, tok)
                out.append((r.rid, tok, not alive))
                if not alive:
                    done.append(r)
            for r in ended:
                out.append((r.rid, None, True))
            for r in done:
                self._running.remove(r)
                self._free.append(r.slot)
            self._free.sort()
        self._admit(out)
        return out


def generate_tokens_continuous(plan, model_type: str, requests: list, arrivals: list, stop_tokens: Iterable[int], max_tokens: int,
                               context_length: int, samplers: list | None = None, stats: dict | None = None,
                               logprobs: list | None = None, chunk_rows: int = 0, min_chunk_rows: int = 32) -> list[list[int]]:
    """Replays a request trace through a ContinuousBatcher: request i = (latest_token, start_position, prompt_tokens) is submitted
    before step arrivals[i] (requests of the same step in index order), with samplers[i] if given.  Steps with no rows still count.
    Returns each request's ids, equal to loop_for(model_type) for the request alone.  stats (optional dict) receives the steps run,
    the rows, launches and kind ("step" or "chunk") of each, and per request its submission, first-token and completion times
    (time.perf_counter seconds, None where it generated no token).  logprobs (optional list, plan.set_logprobs on) receives one list
    per request, one entry per generated id.  chunk_rows / min_chunk_rows: ContinuousBatcher's chunked admission (0: off)."""
    if len(arrivals) != len(requests):
        raise ValueError(f"{len(requests)} requests but {len(arrivals)} arrival steps")
    if samplers is not None and len(samplers) != len(requests):
        raise ValueError(f"{len(requests)} requests but {len(samplers)} samplers")
    if any(a < 0 for a in arrivals):
        raise ValueError("arrival steps must be >= 0")
    cb = ContinuousBatcher(plan, model_type, stop_tokens, max_tokens, context_length, chunk_rows, min_chunk_rows)
    order = sorted(range(len(requests)), key=lambda i: (arrivals[i], i))
    rid_of: dict = {}
    t_sub, t_first, t_done = [None] * len(requests), [None] * len(requests), [None] * len(requests)
    rows, launches, kinds = [], [], []
    nxt, k = 0, 0
    while nxt < len(order) or cb.pending() or cb.running():
        while nxt < len(order) and arrivals[order[nxt]] <= k:
            i = order[nxt]
            latest, start, prompt = requests[i]
            rid_of[cb.submit(latest, start, prompt, samplers[i] if samplers is not None else None)] = i
            t_sub[i] = time.perf_counter()
            nxt += 1
        events = cb.step()
        now = time.perf_counter()
        if cb.last_rows:
            rows.append(cb.last_rows)
            launches.append(plan.batch_info()[1])
            kinds.append(cb.last_kind)
        for rid, tok, finished in events:
            i = rid_of[rid]
            if tok is not None and t_first[i] is None:
                t_first[i] = now
            if finished:
                t_done[i] = now
        k += 1
    if stats is not None:
        stats.update(steps=len(rows), rows=rows, launches=launches, kinds=kinds, submitted=t_sub, first_token=t_first, done=t_done)
    rids = sorted(rid_of, key=lambda r: rid_of[r])
    if logprobs is not None:
        logprobs.extend(cb.logprobs[rid] for rid in rids)
    return [cb.results[rid] for rid in rids]


def score_sequence(plan, tokens: list[int], start_pos: int = 0):
    """Score tokens[i] at start_pos + i through plan.score_tokens, in chunks of the plan's prefill batch size (the whole sequence when
    the plan has none).  Row i's target is tokens[i + 1] -- for a chunk's last row, the next chunk's first token -- and -1 for the
    sequence's last row.  Returns (logprobs float64 [n], NaN in the last row; greedy ids int32 [n])."""
    t = np.asarray(tokens, dtype=np.int32).reshape(-1)
    n = len(t)
    targets = np.append(t[1:], np.int32(-1))
    pb = getattr(plan, "prefill_batch_size", 0) or 0
    chunk = pb if pb > 1 else max(n, 1)
    lp = np.empty(n, dtype=np.float64)
    ids = np.empty(n, dtype=np.int32)
    for a in range(0, n, chunk):
        b = min(a + chunk, n)
        lp[a:b], ids[a:b] = plan.score_tokens(t[a:b], start_pos + a, targets[a:b])
    return lp, ids


def perplexity(plan, tokens: list[int]) -> float:
    """exp(-mean log p(tokens[i] | tokens[:i])) over i = 1 .. n-1, scored from position 0 after plan.kv_reset()."""
    if len(tokens) < 2:
        raise ValueError("perplexity needs at least two tokens")
    plan.kv_reset()
    lp, _ = score_sequence(plan, tokens, 0)
    return math.exp(-float(lp[:-1].mean()))
