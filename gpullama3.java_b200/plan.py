"""Host-side mirror of the reference's plan interface.

``B200MasterPlan`` stands where ``TornadoVMMasterPlan`` does
(``tornadovm/TornadoVMMasterPlan.java:30-85``): same factory, same three forward entry
points, same ``free`` -- but each call is one C-ABI call into libb200llama.so instead of
N+2 TornadoVM TaskGraph executions (``TornadoVMMasterPlanSingleToken.java:68-95``).
The flag names follow the reference's system properties (``TornadoVMMasterPlan.java:32-41``).
"""
from __future__ import annotations

import os

import numpy as np

from . import native
from .loader import ARCH_DEVSTRAL, ARCH_GRANITE, Model


def _flag(name: str, default: str) -> str:
    # -Dllama.xxx system properties become LLAMA_XXX environment variables here
    return os.environ.get(name.upper().replace(".", "_"), default)


WITH_PREFILL_DECODE = _flag("llama.withPrefillDecode", "false").lower() == "true"
PREFILL_BATCH_SIZE = int(_flag("llama.prefillBatchSize", "1"))
FP16_LANES = int(_flag("llama.VectorBitSize", "512")) // 32  # FloatTensor.java:21 (species width / 32-bit lanes)


def tp_shard_plan(c, n: int) -> list[dict]:
    """Row ranges every rank owns under n-way tensor parallelism (mirrors csrc/plan.cu).  Every matrix is
    split by OUTPUT rows -- query/KV heads, FFN hidden units, residual rows, vocabulary rows -- so each dot
    product keeps its full column range and therefore the reference's summation order; what the usual
    column split turns into an all-reduce is an all-gather of the output slices here."""
    if n < 1 or n > 8 or c.n_heads % n or c.n_kv_heads % n or c.dim % (4 * n) or c.hidden_dim % (32 * n) or c.vocab_size % (4 * n):
        raise native.UnsupportedOperation(-2, f"shape does not split {n} ways")
    hs = c.head_size
    out = []
    for r in range(n):
        nh, nkv = c.n_heads // n, c.n_kv_heads // n
        out.append({
            "q_rows": (r * nh * hs, (r + 1) * nh * hs), "kv_rows": (r * nkv * hs, (r + 1) * nkv * hs),
            "heads": (r * nh, (r + 1) * nh), "kv_heads": (r * nkv, (r + 1) * nkv),
            "residual_rows": (r * c.dim // n, (r + 1) * c.dim // n),          # rows of Wo and W2
            "hidden_units": (r * c.hidden_dim // n, (r + 1) * c.hidden_dim // n),  # rows of gate/up
            "vocab_rows": (r * c.vocab_size // n, (r + 1) * c.vocab_size // n),
        })
    return out


def exchange_handles(handle: bytes, group=None) -> list[bytes]:
    """All-gather the 64-byte CUDA IPC handles in rank order (any torch.distributed backend)."""
    import torch.distributed as dist

    world = dist.get_world_size(group)
    out = [None] * world
    dist.all_gather_object(out, handle, group=group)
    return out


def make_config(model: Model, fp16_lanes: int | None = None) -> native.Config:
    c = model.configuration
    cfg = native.Config()
    cfg.arch = c.arch
    cfg.dim, cfg.hidden_dim, cfg.n_layers = c.dim, c.hidden_dim, c.n_layers
    cfg.n_heads, cfg.n_kv_heads, cfg.head_size = c.n_heads, c.n_kv_heads, c.head_size
    cfg.vocab_size, cfg.context_length = c.vocab_size, c.context_length
    cfg.rms_norm_eps, cfg.rope_theta = c.rms_norm_eps, c.rope_theta
    cfg.fp16_lanes = FP16_LANES if fp16_lanes is None else fp16_lanes
    cfg.tp_rank, cfg.tp_size = 0, 1
    return cfg


class B200MasterPlan:
    """One plan per model, used from one thread at a time (InferenceService.java:31,58)."""

    def __init__(self, model: Model, prefill_batch_size: int | None = None, device: int = 0, fp16_lanes: int | None = None,
                 tp_rank: int = 0, tp_size: int = 1, tp_group=None):
        self.model = model
        self.prefill_batch_size = PREFILL_BATCH_SIZE if prefill_batch_size is None else prefill_batch_size
        cfg = make_config(model, fp16_lanes)
        cfg.tp_rank, cfg.tp_size = tp_rank, tp_size
        if tp_size > 1:
            tp_shard_plan(model.configuration, tp_size)  # raises early on shapes that do not split
        c = model.configuration
        moe = granite = None
        if c.n_experts:  # Qwen2-MoE / Qwen3-MoE (shared_hidden_dim 0): b200_plan_create_moe
            moe = native.MoeConfig(c.n_experts, c.n_experts_used, c.expert_hidden_dim, c.shared_hidden_dim)
        if c.arch == ARCH_GRANITE:  # Granite: b200_plan_create_granite
            granite = native.GraniteConfig(c.embedding_scale, c.residual_scale, c.attention_scale, c.logit_scale)
        y = c.yarn  # Devstral: b200_plan_create_devstral, YaRN table or (None) the plain one
        yarn = native.YarnConfig(y.factor, y.beta_fast, y.beta_slow, y.log_multiplier, y.original_context_length) if y is not None else None
        self._native = native.NativePlan(cfg, model.tensors, self.prefill_batch_size, device, moe=moe, granite=granite,
                                         devstral=c.arch == ARCH_DEVSTRAL, yarn=yarn)
        self.tp_rank, self.tp_size = tp_rank, tp_size
        self._controls = {}  # slot -> (the SamplingControls set there, who set them); the device state lives in the plan
        if tp_size > 1:
            # one process per GPU: swap IPC handles of the communication buffers, then wire the peers
            import torch.distributed as dist

            handles = exchange_handles(self._native.tp_handle(), tp_group)
            self._native.tp_attach(handles)
            dist.barrier(group=tp_group)

    # TornadoVMMasterPlan.initializeTornadoVMPlan(state, model)  (TornadoVMMasterPlan.java:55-70)
    @staticmethod
    def initialize_plan(model: Model, **kw) -> "B200MasterPlan":
        plan = B200MasterPlan(model, **kw)
        model.plan = plan  # model.setTornadoVMPlan(plan)
        return plan

    # FloatArray tornadoVMForwardDecode(int position) + the embedding gather of
    # InferenceCore.forwardTornadoVM (InferenceCore.java:956-980)
    def forward_decode(self, token: int, position: int, logits: bool = True):
        lg, am = self._native.forward_decode(token, position, want_logits=logits, want_argmax=True)
        return lg, am

    # forward + Sampler.sampleToken on the device (Sampler.java:74-122): 4 bytes in (the uniform number), 4 bytes out
    def forward_decode_sample(self, token: int, position: int, temperature: float, topp: float, uniform01: float, want_info: bool = False):
        return self._native.forward_decode_sample(token, position, temperature, topp, uniform01, want_info)

    # void tornadoVMForwardPrefill(int position)  (TornadoVMMasterPlanPrefillDecode.java:116)
    def forward_prefill(self, token: int, position: int):
        self._native.forward_prefill(token, position)

    # void tornadoVMForwardBatchPrefill()  (TornadoVMMasterPlanBatchPrefillDecode.java:107-123)
    def forward_batch_prefill(self, tokens, start_pos: int):
        self._native.forward_batch_prefill(np.asarray(tokens, dtype=np.int32), start_pos)

    def score_tokens(self, tokens, start_pos: int, targets=None):
        """Score tokens[i] at start_pos + i -> (logprobs float64 [n], greedy ids int32 [n]): logprobs[i] is the log-probability of
        targets[i] (default: the next token, -1 = NaN for the last row) under logits bit-identical to forward_decode's, in double;
        the K/V go into the cache as forward_batch_prefill writes them.  Prefill modes "exact" and "tensor_core_exact" only, and at
        most forward_batch_prefill's chunk length (engine.score_sequence splits longer sequences)."""
        return self._native.score_tokens(tokens, start_pos, targets)

    def set_logprobs(self, top_n: int):
        """Log-probabilities of generated tokens (b200_set_logprobs): -1 off (the default), 0..20 alternatives per row.  While on, every
        call that emits ids (forward_decode, forward_decode_sample, decode_sequence, forward_decode_batch, forward_decode_multi,
        forward_step) records one row per emitted id, read back with last_logprobs().  Single-GPU plans only."""
        self._native.set_logprobs(top_n)

    def logprobs_top_n(self) -> int:
        """The set_logprobs setting: -1 off, else the alternatives per row."""
        return self._native.logprobs_top_n()

    def last_logprobs(self):
        """The last emitting call's rows -> (chosen float64 [rows], top_ids int32 [rows, N], top_logprobs float64 [rows, N]): the
        emitted id's log-probability under the raw logits (temperature 1, in double; bit-equal to score_tokens') and the N most
        likely ids, ties to the lower index, with theirs.  Rows of forward_step that do not emit: NaN and ids -1."""
        return self._native.last_logprobs()

    # TensorCoreSupport.java's switch between the MMA and the plain batch-prefill layer families
    PREFILL_EXACT, PREFILL_TENSOR_CORE, PREFILL_TENSOR_CORE_W8A16, PREFILL_TENSOR_CORE_EXACT = 0, 1, 2, 3
    PREFILL_TENSOR_CORE_EXACT_MOE = 4

    def set_sampling_controls(self, slot: int, controls, owner=None):
        """Sampling controls (sampler.SamplingControls, or None to turn them off) for one sequence: a decode slot, or -1 for the plan's
        own cache.  forward_decode_sample (slot -1), forward_decode_batch with sampling and forward_step's emitting rows apply them
        on the device and count each emitted id; every other call ignores them.  Single-GPU plans only.  owner: who holds the
        sequence's controls and counts (a sampler.Sampler), until they are replaced or a reset clears the counts."""
        self._native.set_sampling_controls(slot, controls)
        self._controls[slot] = (controls, owner) if controls is not None else None

    def sampling_controls(self, slot: int):
        """The controls set on the sequence through set_sampling_controls, or None."""
        e = self._controls.get(slot)
        return e[0] if e else None

    def sampling_controls_owner(self, slot: int):
        """The owner given with the sequence's controls; None once slot_reset / kv_reset / set_decode_slots cleared its counts."""
        e = self._controls.get(slot)
        return e[1] if e else None

    def _counts_cleared(self, slots):
        for s in slots:
            if self._controls.get(s):
                self._controls[s] = (self._controls[s][0], None)

    def set_sample_history(self, slot: int, tokens):
        """Replace the sequence's token counts with those of tokens (e.g. the prompt); slot_reset / kv_reset clear them."""
        self._native.set_sample_history(slot, tokens)

    def sample_counts(self, slot: int):
        """The sequence's count per token id (int32 [vocab])."""
        return self._native.sample_counts(slot)

    def set_prefill_mode(self, mode):
        """"exact" (token-by-token graph, bit-identical KV cache), "tensor_core" (wgmma GEMMs, FP16 tolerance; a Q8_0 plan
        builds f16 twins of its matrices) or "tensor_core_w8a16" (Q8_0 plans: the same GEMMs reading the Q8_0 weights in
        place, dequantised in shared memory; bit-identical to "tensor_core" where no residual GEMM splits K) or "tensor_core_exact"
        (Q8_0 plans: the whole chunk through int8 tensor-core GEMMs summing each Q8_0 block's term in the CPU path's order;
        KV cache bit-identical to "exact").  On a plan that keeps K-quant weights resident (weight_info()["resident"]) only
        "exact" and "tensor_core_exact" are available: the latter expands each resident matrix to its Q8_0 tiles on the device
        just before its GEMM, in one scratch the size of the largest resident matrix's Q8_0 tiles, and raises B200Error
        (B200_ERR_OOM) naming the bytes when that scratch and the chunk buffers do not fit the free memory.
        "tensor_core_exact_moe" is "tensor_core_exact" for Qwen2-MoE / Qwen3-MoE plans (which refuse the other tensor-core modes;
        dense plans refuse this one): the chunk's rows are routed on the device, each expert's rows run as one grouped int8 GEMM, and
        the results are combined in the decode's order, so the KV cache is bit-identical to "exact" and score_tokens' results are
        exact mode's; moe_chunk_routing() returns each row's routing of the last chunk."""
        if isinstance(mode, str):
            mode = {"exact": 0, "tensor_core": 1, "tensor_core_w8a16": 2, "tensor_core_exact": 3, "tensor_core_exact_moe": 4}[mode]
        self._native.set_prefill_mode(int(mode))

    def prefill_info(self):
        """(active mode, kernels launched, device ms) of the last tensor-core prefill chunk."""
        return self._native.prefill_info()

    # -Dllama.cudaGraphs-style switch of the decode implementation (both bit-identical): "graph" = one CUDA graph of
    # ~7 kernels per layer, "persistent" = one persistent kernel per token (csrc/decode_persistent.cuh)
    DECODE_GRAPH, DECODE_PERSISTENT = 0, 1

    def set_decode_mode(self, mode):
        if isinstance(mode, str):
            mode = {"graph": 0, "persistent": 1}[mode]
        self._native.set_decode_mode(int(mode))

    def decode_info(self):
        return self._native.decode_info()

    def trace_persistent(self, token: int, position: int):
        return self._native.trace_persistent(token, position)

    def decode_sequence(self, tokens, n: int, start_pos: int, feedback: bool = False):
        return self._native.decode_sequence(tokens, n, start_pos, feedback)

    def time_kernel(self, which: int, reps: int = 3):
        return self._native.time_kernel(which, reps)

    # Batched decode (csrc/decode_batch.cuh): up to 8 independent sequences per step, each on its own KV-cache slot, every weight
    # matrix streamed once per step; each row bit-identical to forward_decode of the same token stream.  Q8_0 plans only.
    def set_decode_slots(self, n_slots: int):
        """Allocate n_slots zeroed KV-cache slots (0 frees them); UnsupportedOperation beyond what the plan can run."""
        self._native.set_decode_slots(n_slots)
        self._counts_cleared([s for s in self._controls if s >= 0])

    def forward_decode_batch(self, slots, tokens, positions, sampling=None, logits: bool = False):
        """One step for len(slots) rows -> (ids, logits [n, vocab] or None).  sampling: None (greedy) or one
        (temperature, topp, uniform01) per row, with forward_decode_sample's contract."""
        return self._native.forward_decode_batch(slots, tokens, positions, sampling, logits)

    def slot_reset(self, slot: int):
        self._native.slot_reset(slot)
        self._counts_cleared([slot])

    def slot_copy_kv(self, slot: int, n_positions: int):
        """Copy positions [0, n_positions) of the plan's own KV cache (e.g. after forward_batch_prefill) into the slot; zero the rest."""
        self._native.slot_copy_kv(slot, n_positions)

    def prefill_slots(self, slots, start_positions, token_lists):
        """Prefill token_lists[i] straight into decode slot slots[i] at positions start_positions[i].. in one call (K/V only, the
        plan's prefill mode; at most prefill_batch_size tokens in all in a tensor-core mode).  The plan's own cache and the other
        slots are left as they are."""
        self._native.prefill_slots(slots, start_positions, token_lists)

    def batch_info(self):
        """(decode slots, kernels of the last batched step, its device milliseconds)."""
        return self._native.batch_info()

    def forward_decode_multi(self, slot: int, tokens, start_pos: int, logits: bool = False):
        """Run tokens[i] at position start_pos + i of ONE sequence in one step (slot >= 0: a decode slot; -1: the plan's own cache)
        -> (ids, logits [n, vocab] or None); ids[i] is the greedy id after position start_pos + i.  Every row is bit-identical to
        forward_decode of the same token at the same position over the same cache prefix: the verification step of draft-and-verify
        decoding.  1 <= len(tokens) <= decode_multi_rows(); single-GPU Q8_0 plans without MoE only."""
        return self._native.forward_decode_multi(slot, tokens, start_pos, logits)

    def forward_step(self, rows, logits: bool = False):
        """One mixed step over the decode slots -> (ids, logits [n, vocab] or None).  Each row is (slot, token, position, emit) or
        (slot, token, position, emit, temperature, topp, uniform01); a slot may take several rows at distinct positions, and every
        row's K/V is written before any row attends.  emit 0: K/V only (a prompt position), id -1; emit 1: the id after the row,
        greedy (temperature 0) or forward_decode_sample's for the triple, with logits bit-identical to forward_decode of that
        sequence.  1 <= len(rows) <= decode_multi_rows(); needs set_decode_slots."""
        return self._native.forward_step(rows, logits)

    def decode_multi_rows(self) -> int:
        """Positions per forward_decode_multi step (8 at the 8B shapes); 0 where the plan cannot run it."""
        return self._native.decode_multi_rows()

    def forward_chunk(self, rows, logits: bool = False):
        """forward_step on the tensor cores -> (ids, logits [n, vocab] or None): the same row tuples and results, every emitting row
        bit-identical to forward_decode of its sequence, run as one chunk of the tensor_core_exact prefill, so prompt rows of newly
        admitted sequences ride in the chunk's GEMMs with the decode rows.  1 <= len(rows) <= chunk_rows(), at most 8 of them
        emitting; needs set_prefill_mode("tensor_core_exact") and set_decode_slots."""
        return self._native.forward_chunk(rows, logits)

    def chunk_rows(self) -> int:
        """Rows per forward_chunk call: prefill_batch_size in tensor_core_exact with decode slots; 0 where the plan cannot run it."""
        return self._native.chunk_rows()

    def moe_routing(self):
        """MoE plans: (ids [layer, k], weights [layer, k + 1]) of the last step (selected experts in selection order, their
        routing weights, then the shared-expert weight); Qwen3-MoE has no shared expert, its weights are [layer, k]."""
        return self._native.moe_routing()

    def moe_chunk_routing(self, rows=None):
        """MoE plans after a tensor_core_exact_moe chunk: (ids [layer, rows, k], weights [layer, rows, k + 1]) of every row of the
        last chunk, as moe_routing() reports one step's (Qwen3-MoE: weights [layer, rows, k]); rows defaults to the last chunk's."""
        return self._native.moe_chunk_routing(rows)

    def kv_reset(self):
        self._native.kv_reset()
        self._counts_cleared([-1])

    def read_buffer(self, *a, **kw):
        return self._native.read_buffer(*a, **kw)

    def upload_info(self):
        """Seconds / bytes of the weight upload pipeline of plan creation (load-time metric, ModelLoader.java:102-106)."""
        return self._native.upload_info()

    def weight_info(self):
        """{"resident", "weight_bytes", "q8_weight_bytes"}: whether plan creation kept the K-quant weights resident because their
        Q8_0 expansion did not fit the device (decode stays bit-identical; batched steps, the persistent kernel and the tensor-core
        prefill are then refused), and the weight footprints of the chosen and of the all-Q8_0 form."""
        return self._native.weight_info()

    @property
    def launches_per_decode(self):
        return self._native.launches_per_decode

    @property
    def device_bytes(self):
        return self._native.device_bytes

    # void freeTornadoExecutionPlan()
    def free(self):
        self._native.free()
