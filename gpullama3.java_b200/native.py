"""ctypes binding of libb200llama.so (the C ABI in include/b200llama.h).

There is deliberately NO fallback: if the CUDA library is missing or a call fails, this
module raises.  Nothing here (or anywhere in the package) touches ``oracle/``.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .sampler import SamplingControls

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libb200llama.so")

B200_OK = 0
ERRORS = {-1: "BAD_ARG", -2: "UNSUPPORTED", -3: "OOM", -4: "CUDA", -5: "NCCL", -6: "STATE"}


class B200Error(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"b200llama error {ERRORS.get(code, code)}: {msg}")
        self.code = code


class UnsupportedOperation(B200Error):
    """Counterpart of the reference's UnsupportedOperationException (ForwardPlanFactory.java:84-87)."""


class Config(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("arch", "dim", "hidden_dim", "n_layers", "n_heads", "n_kv_heads", "head_size",
                                        "vocab_size", "context_length")] + \
               [("rms_norm_eps", C.c_float), ("rope_theta", C.c_float), ("fp16_lanes", C.c_int32),
                ("tp_rank", C.c_int32), ("tp_size", C.c_int32)]


class MoeConfig(C.Structure):
    """b200_moe_config: the expert configuration of a B200_ARCH_QWEN2_MOE or B200_ARCH_QWEN3_MOE plan (shared_hidden_dim 0)."""
    _fields_ = [(n, C.c_int32) for n in ("n_experts", "n_experts_used", "expert_hidden_dim", "shared_hidden_dim")]


class GraniteConfig(C.Structure):
    """b200_granite_config: the four muP scales of a B200_ARCH_GRANITE plan."""
    _fields_ = [(n, C.c_float) for n in ("embedding_scale", "residual_scale", "attention_scale", "logit_scale")]


class YarnConfig(C.Structure):
    """b200_yarn_config: the YaRN parameters of a B200_ARCH_DEVSTRAL plan's RoPE table."""
    _fields_ = [(n, C.c_float) for n in ("factor", "beta_fast", "beta_slow", "log_multiplier")] + [("original_context_length", C.c_int32)]


class StepRow(C.Structure):
    """b200_step_row: one row of a mixed step (b200_forward_step)."""
    _fields_ = [(n, C.c_int32) for n in ("slot", "token", "position", "emit")] + [(n, C.c_float) for n in ("temperature", "topp", "uniform01")]


class SamplingControlsC(C.Structure):
    """b200_sampling_controls."""
    _fields_ = [("top_k", C.c_int32)] + [(n, C.c_float) for n in ("min_p", "repetition_penalty", "frequency_penalty", "presence_penalty")] + \
               [("n_bias", C.c_int32), ("bias_ids", C.c_void_p), ("bias_values", C.c_void_p)]


def _controls_c(c: SamplingControls):
    """(b200_sampling_controls, the arrays its pointers reference: keep them alive across the call)."""
    bias = c.logit_bias or {}
    ids = np.ascontiguousarray(list(bias.keys()), dtype=np.int32)
    vals = np.ascontiguousarray(list(bias.values()), dtype=np.float32)
    s = SamplingControlsC(int(c.top_k), c.min_p, c.repetition_penalty, c.frequency_penalty, c.presence_penalty, len(ids),
                          ids.ctypes.data if len(ids) else None, vals.ctypes.data if len(ids) else None)
    return s, (ids, vals)


class StreamTest(C.Structure):
    """b200_stream_test: the arguments and the reported configuration of b200_test_stream."""
    _fields_ = [(n, C.c_int32) for n in ("form", "mode", "norm", "nrow", "lanes", "rows", "cols", "grid", "stages")] + [("budget", C.c_int64)] + \
               [(n, C.c_int32) for n in ("argmax", "launches", "pair", "down_rows", "from_emb", "emb_rows", "dry")] + \
               [(n, C.c_float) for n in ("oscale", "eps", "emb_scale")] + \
               [(n, C.c_void_p) for n in ("w", "w_up", "w_down", "xq", "xs", "x", "norm_w", "emb", "tokens", "out_init", "out", "hq", "hs", "out_down",
                                          "x_out", "ids")] + [("info", C.c_int64 * 5)]


class AttentionTest(C.Structure):
    """b200_attention_test: the arguments and the reported configuration of b200_test_attention."""
    _fields_ = [(n, C.c_int32) for n in ("form", "head_size", "n_heads", "n_kv_heads", "arch", "ctx", "rows", "slots", "att_tokens", "dry")] + \
               [(n, C.c_float) for n in ("eps", "score_arg")] + \
               [(n, C.c_void_p) for n in ("slot", "pos", "qkv", "k_cache", "v_cache", "rope_cr", "rope_ci", "q_norm", "k_norm", "qkv_bias", "qkv_out",
                                          "k_out", "v_out", "xq", "xs", "xb")] + [("info", C.c_int64 * 5)]


class Tensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.c_void_p), ("ggml_type", C.c_int32), ("n_dims", C.c_int32),
                ("dims", C.c_int64 * 4)]


EXPORTS = ["b200_plan_create", "b200_plan_create_moe", "b200_plan_create_granite", "b200_plan_create_devstral", "b200_forward_decode", "b200_forward_prefill", "b200_forward_batch_prefill", "b200_score_tokens", "b200_set_logprobs", "b200_read_logprobs", "b200_test_logprobs", "b200_set_sampling_controls", "b200_set_sample_history", "b200_read_sample_counts", "b200_test_sample_controls", "b200_time_sample_controls", "b200_set_prefill_mode", "b200_prefill_info",
           "b200_set_decode_mode", "b200_decode_info", "b200_trace_persistent", "b200_test_seqsum2", "b200_profile_seqsum2", "b200_test_sample", "b200_forward_decode_sample", "b200_upload_info", "b200_requant_kquant", "b200_test_kq_tiles_to_q8",
           "b200_decode_sequence", "b200_time_kernel", "b200_tp_handle", "b200_tp_attach", "b200_trace_decode", "b200_profile_norm", "b200_gemm_f16", "b200_test_gemm", "b200_test_gemm_q8", "b200_test_gemm_i8", "b200_test_gemm_i8_experts", "b200_kv_reset", "b200_read_buffer", "b200_launches_per_decode",
           "b200_set_decode_slots", "b200_forward_decode_batch", "b200_slot_reset", "b200_slot_copy_kv", "b200_prefill_slots", "b200_test_pf_attention_packed", "b200_batch_info",
           "b200_forward_decode_multi", "b200_decode_multi_rows", "b200_forward_step", "b200_forward_chunk", "b200_chunk_rows", "b200_weight_info", "b200_test_set_memory_budget", "b200_stream_rings",
           "b200_test_stream", "b200_test_attention", "b200_test_exp", "b200_device_bytes", "b200_plan_free", "b200_last_error", "b200_version"]

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    vp, i32 = C.c_void_p, C.c_int32
    L.b200_plan_create.argtypes = [C.POINTER(Config), C.POINTER(Tensor), i32, i32, i32, C.POINTER(vp), C.c_char_p, C.c_size_t]
    L.b200_plan_create_moe.argtypes = [C.POINTER(Config), C.POINTER(MoeConfig), C.POINTER(Tensor), i32, i32, i32, C.POINTER(vp), C.c_char_p, C.c_size_t]
    L.b200_plan_create_granite.argtypes = [C.POINTER(Config), C.POINTER(GraniteConfig), C.POINTER(Tensor), i32, i32, i32, C.POINTER(vp), C.c_char_p, C.c_size_t]
    L.b200_plan_create_devstral.argtypes = [C.POINTER(Config), C.POINTER(YarnConfig), C.POINTER(Tensor), i32, i32, i32, C.POINTER(vp), C.c_char_p, C.c_size_t]
    L.b200_forward_decode.argtypes = [vp, i32, i32, vp, C.POINTER(i32)]
    L.b200_forward_prefill.argtypes = [vp, i32, i32]
    L.b200_forward_decode_sample.argtypes = [vp, i32, i32, C.c_float, C.c_float, C.c_float, C.POINTER(i32), C.POINTER(i32)]
    L.b200_forward_batch_prefill.argtypes = [vp, vp, i32, i32]
    L.b200_score_tokens.argtypes = [vp, vp, vp, i32, i32, vp, vp]
    L.b200_set_logprobs.argtypes = [vp, i32]
    L.b200_read_logprobs.argtypes = [vp, i32, C.POINTER(i32), vp, vp, vp]
    L.b200_test_logprobs.argtypes = [vp, i32, i32, i32, i32, vp, vp, vp, C.POINTER(C.c_float)]
    L.b200_set_sampling_controls.argtypes = [vp, i32, C.POINTER(SamplingControlsC)]
    L.b200_set_sample_history.argtypes = [vp, i32, vp, i32]
    L.b200_read_sample_counts.argtypes = [vp, i32, vp]
    L.b200_test_sample_controls.argtypes = [vp, i32, vp, C.POINTER(SamplingControlsC), C.c_float, C.c_float, C.c_float, C.POINTER(i32), C.POINTER(i32), vp]
    L.b200_time_sample_controls.argtypes = [vp, i32, vp, C.POINTER(SamplingControlsC), C.c_float, C.c_float, C.c_float, i32, C.POINTER(C.c_float),
                                            C.POINTER(C.c_float)]
    L.b200_decode_sequence.argtypes = [vp, vp, i32, i32, i32, vp, C.POINTER(C.c_float)]
    L.b200_kv_reset.argtypes = [vp]
    L.b200_profile_norm.argtypes = [vp, C.POINTER(C.c_int64)]
    L.b200_trace_decode.argtypes = [vp, i32, i32, vp, i32, C.POINTER(i32)]
    L.b200_tp_handle.argtypes = [vp, vp]
    L.b200_tp_attach.argtypes = [vp, vp, i32]
    L.b200_set_prefill_mode.argtypes = [vp, i32]
    L.b200_set_decode_mode.argtypes = [vp, i32]
    L.b200_decode_info.argtypes = [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]
    L.b200_trace_persistent.argtypes = [vp, i32, i32, vp, C.c_int64, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]
    L.b200_test_seqsum2.argtypes = [vp, i32, i32, C.POINTER(C.c_float), C.POINTER(i32)]
    L.b200_profile_seqsum2.argtypes = [vp, i32, i32, C.POINTER(C.c_int64), C.POINTER(C.c_float)]
    L.b200_test_sample.argtypes = [vp, i32, C.c_float, C.c_float, C.c_float, C.POINTER(i32), C.POINTER(i32), vp]
    L.b200_prefill_info.argtypes = [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(C.c_float)]
    L.b200_gemm_f16.argtypes = [vp, vp, vp, i32, i32, i32, i32, C.POINTER(C.c_float)]
    L.b200_test_gemm.argtypes = [i32, i32, i32, i32, i32, i32, i32, vp, vp, vp, vp]
    L.b200_test_gemm_q8.argtypes = [i32, i32, i32, i32, i32, i32, i32, vp, vp, vp, vp]
    L.b200_test_gemm_i8.argtypes = [i32, i32, i32, i32, vp, vp, vp, vp, C.c_float, vp, vp, vp]
    L.b200_test_gemm_i8_experts.argtypes = [i32, i32, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp]
    L.b200_time_kernel.argtypes = [vp, i32, i32, C.POINTER(C.c_float), C.POINTER(C.c_int64)]
    L.b200_read_buffer.argtypes = [vp, C.c_char_p, i32, vp, C.c_size_t]
    L.b200_set_decode_slots.argtypes = [vp, i32]
    L.b200_forward_decode_batch.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp]
    L.b200_slot_reset.argtypes = [vp, i32]
    L.b200_slot_copy_kv.argtypes = [vp, i32, i32]
    L.b200_prefill_slots.argtypes = [vp, i32, vp, vp, vp, vp]
    L.b200_test_pf_attention_packed.argtypes = [i32, vp, vp, vp, vp, vp, i32, i32, i32, i32, vp]
    L.b200_batch_info.argtypes = [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(C.c_float)]
    L.b200_forward_decode_multi.argtypes = [vp, i32, i32, vp, i32, vp, vp]
    L.b200_decode_multi_rows.argtypes = [vp, C.POINTER(i32)]
    L.b200_forward_step.argtypes = [vp, i32, C.POINTER(StepRow), vp, vp]
    L.b200_forward_chunk.argtypes = [vp, i32, C.POINTER(StepRow), vp, vp]
    L.b200_chunk_rows.argtypes = [vp, C.POINTER(i32)]
    L.b200_upload_info.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int64)]
    L.b200_weight_info.argtypes = [vp, C.POINTER(i32), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    L.b200_test_set_memory_budget.argtypes = [C.c_int64]
    L.b200_test_kq_tiles_to_q8.argtypes = [i32, i32, i32, vp, vp, C.c_int64]
    L.b200_stream_rings.argtypes = [C.POINTER(i32), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    L.b200_test_stream.argtypes = [C.POINTER(StreamTest)]
    L.b200_test_attention.argtypes = [C.POINTER(AttentionTest)]
    L.b200_test_exp.argtypes = [C.c_uint32, C.c_int64, vp, vp]
    L.b200_launches_per_decode.argtypes = [vp]
    L.b200_device_bytes.argtypes = [vp]
    L.b200_device_bytes.restype = C.c_int64
    L.b200_plan_free.argtypes = [vp]
    L.b200_plan_free.restype = None
    L.b200_last_error.argtypes = [vp]
    L.b200_last_error.restype = C.c_char_p
    L.b200_version.restype = C.c_char_p
    _lib = L
    return L


def _raise(code: int, msg: str):
    if code == -2:
        raise UnsupportedOperation(code, msg)
    raise B200Error(code, msg)


def test_seqsum(terms, want_info: bool = False, threads: int = 1024):
    """The exact sequential sum (seqsum2.cuh) with 1024 / 512 / 256 threads: the norm kernel's / persistent kernel's form."""
    t = np.ascontiguousarray(terms, dtype=np.float32)
    out = C.c_float(0)
    info = (C.c_int32 * 2)()
    rc = lib().b200_test_seqsum2(t.ctypes.data, len(t), threads, C.byref(out), info)
    if rc != B200_OK:
        _raise(rc, "b200_test_seqsum2 failed")
    return (out.value, info[0], info[1]) if want_info else out.value


def profile_seqsum(terms, threads: int = 256):
    """Cycles of the exact sequential sum in the fused norm's chunk layout, two calls in one launch:
    (cold, warm, sum, sum, items, literal items, fallbacks)."""
    t = np.ascontiguousarray(terms, dtype=np.float32)
    cyc = (C.c_int64 * 5)()
    out = (C.c_float * 2)()
    rc = lib().b200_profile_seqsum2(t.ctypes.data, len(t), threads, cyc, out)
    if rc != B200_OK:
        _raise(rc, "b200_profile_seqsum2 failed")
    return cyc[0], cyc[1], out[0], out[1], cyc[2], cyc[3], cyc[4]


def test_sample(logits, temperature: float, topp: float, uniform01: float):
    """One launch of the device sampler (csrc/sampler.cuh) as b200_forward_decode_sample issues it, on host logits.
    Returns (token id, [top-p candidates, kept, seqsum items, seqsum fallbacks], float32 probabilities)."""
    lg = np.ascontiguousarray(logits, dtype=np.float32)
    probs = np.empty(len(lg), dtype=np.float32)
    out = C.c_int32(-1)
    info = (C.c_int32 * 4)()
    rc = lib().b200_test_sample(lg.ctypes.data, len(lg), temperature, topp, uniform01, C.byref(out), info, probs.ctypes.data)
    if rc != B200_OK:
        _raise(rc, "b200_test_sample failed")
    return out.value, list(info), probs


def test_sample_controls(logits, counts, controls: SamplingControls, temperature: float, topp: float, uniform01: float):
    """One launch of the controlled sampler (k_sample_ctl, csrc/sampler.cuh) as the plans issue it, on host logits and counts.
    temperature 0 takes the first maximum of the modified row.  Returns (token id, the sampler's four diagnostics, the modified row
    float32 before the choice, the counts after the launch)."""
    lg = np.ascontiguousarray(logits, dtype=np.float32)
    cnt = np.array(counts, dtype=np.int32, copy=True)
    if cnt.shape != lg.shape:
        raise ValueError("one count per logit")
    row = np.empty(len(lg), dtype=np.float32)
    out = C.c_int32(-1)
    info = (C.c_int32 * 4)()
    cs, keep = _controls_c(controls)
    rc = lib().b200_test_sample_controls(lg.ctypes.data, len(lg), cnt.ctypes.data, C.byref(cs), temperature, topp, uniform01, C.byref(out), info,
                                         row.ctypes.data)
    if rc != B200_OK:
        _raise(rc, "b200_test_sample_controls failed")
    return out.value, list(info), row, cnt


def time_sample_controls(logits, counts, controls: SamplingControls, temperature: float, topp: float, uniform01: float, reps: int):
    """b200_time_sample_controls: CUDA-event ms per launch of (k_sample_ctl under controls, one-row k_sample_rows) on the same row, reps each."""
    lg = np.ascontiguousarray(logits, dtype=np.float32)
    cnt = np.ascontiguousarray(counts, dtype=np.int32)
    if cnt.shape != lg.shape:
        raise ValueError("one count per logit")
    cs, keep = _controls_c(controls)
    a, b = C.c_float(0), C.c_float(0)
    rc = lib().b200_time_sample_controls(lg.ctypes.data, len(lg), cnt.ctypes.data, C.byref(cs), temperature, topp, uniform01, int(reps),
                                         C.byref(a), C.byref(b))
    if rc != B200_OK:
        _raise(rc, "b200_time_sample_controls failed")
    return a.value, b.value


def test_set_memory_budget(n_bytes: int):
    """Test hook: the device free-memory figure the weight-form rule of plan creation reads, for every later plan in the process
    (0 restores the real figure).  Puts a budget on either side of the K-quant residency threshold without filling the GPU."""
    rc = lib().b200_test_set_memory_budget(int(n_bytes))
    if rc != B200_OK:
        _raise(rc, f"b200_test_set_memory_budget({n_bytes}) failed")


def stream_rings(dim: int, q_width: int, kv_width: int, hidden: int, n_sms: int, fused_norm: bool, fmts=(0, 0, 0, 0),
                 sm_bytes: int = 233472, reserve_bytes: int = 1024, optin_bytes: int = 232448, att_bytes: int = 0) -> dict:
    """b200_stream_rings: the rings plan creation gives one layer's QKV, Wo, gate/up and W2 streams (fmts: their tile formats,
    0 or a resident K-quant type) on a device with these shared-memory figures (defaults: H100).  Per stream: smem (dynamic
    shared memory of the launch), stages, stage_bytes and slice_tiles (the largest CTA slice)."""
    shape = (C.c_int32 * 10)(dim, q_width, kv_width, hidden, n_sms, 1 if fused_norm else 0, *fmts)
    dev = (C.c_int64 * 4)(sm_bytes, reserve_bytes, optin_bytes, att_bytes)
    out = (C.c_int64 * 16)()
    rc = lib().b200_stream_rings(shape, dev, out)
    if rc != B200_OK:
        _raise(rc, "b200_stream_rings failed")
    keys = ("smem", "stages", "stage_bytes", "slice_tiles")
    return {name: dict(zip(keys, out[4 * k:4 * k + 4])) for k, name in enumerate(("qkv", "wo", "gateup", "w2"))}


def requant_kquant(ggml_type: int, raw, n_elems: int) -> np.ndarray:
    """Device K-quant (Q4_K = 12 / Q5_K = 13 / Q6_K = 14) -> GGUF Q8_0 bytes (csrc/kquant.cuh; ModelLoader.java:173-224)."""
    raw = np.ascontiguousarray(raw, dtype=np.uint8)
    out = np.empty(n_elems // 32 * 34, dtype=np.uint8)
    lib().b200_requant_kquant.argtypes = [C.c_int32, C.c_void_p, C.c_int64, C.c_void_p]
    rc = lib().b200_requant_kquant(int(ggml_type), raw.ctypes.data, int(n_elems), out.ctypes.data)
    if rc != B200_OK:
        _raise(rc, "b200_requant_kquant failed")
    return out


def q8_tile_bytes(rows: int, cols: int) -> int:
    """Bytes of the tile-major Q8_0 stream of a rows x cols matrix (csrc/stream_matvec.cuh: the fewest segments of at most 2560
    columns, each a multiple of 32; a unit is a segment's quants and f16 scales padded to 16 bytes; whole 4-row groups)."""
    nseg = next(n for n in range(1, cols // 32 + 1) if cols % n == 0 and (cols // n) % 32 == 0 and cols // n <= 2560)
    seg = cols // nseg
    return (rows + 3) // 4 * 4 * nseg * ((seg + seg // 16 + 15) & ~15)


def test_kq_tiles_to_q8(ggml_type: int, rows: int, cols: int, raw) -> np.ndarray:
    """b200_test_kq_tiles_to_q8: row-major K-quant rows (Q4_K = 12 / Q5_K = 13 / Q6_K = 14) repacked into resident tiles and expanded
    on the device to the matrix's tile-major Q8_0 stream (uint8, q8_tile_bytes(rows, cols) bytes), as the bit-exact tensor-core
    prefill expands a resident matrix."""
    raw = np.ascontiguousarray(raw, dtype=np.uint8)
    if cols % 256 or raw.size != rows * (cols // 256) * {12: 144, 13: 176, 14: 210}.get(int(ggml_type), 0):
        raise ValueError(f"{raw.size} bytes are not {rows} rows of {cols} type-{ggml_type} elements")
    out = np.empty(q8_tile_bytes(rows, cols), dtype=np.uint8)
    rc = lib().b200_test_kq_tiles_to_q8(int(ggml_type), int(rows), int(cols), raw.ctypes.data, out.ctypes.data, out.size)
    if rc != B200_OK:
        _raise(rc, "b200_test_kq_tiles_to_q8 failed")
    return out


def gemm_f16(a, b, iters: int = 0):
    """C = A @ B.T on the wgmma prefill GEMM (A [m,k], B [n,k] float16) -> (C float32, ms per launch or None)."""
    a = np.ascontiguousarray(a, dtype=np.float16)
    b = np.ascontiguousarray(b, dtype=np.float16)
    m, k = a.shape
    n, k2 = b.shape
    if k != k2:
        raise ValueError("inner dimensions differ")
    c = np.empty((m, n), dtype=np.float32)
    ms = C.c_float(0)
    rc = lib().b200_gemm_f16(a.ctypes.data, b.ctypes.data, c.ctypes.data, m, n, k, iters, C.byref(ms))
    if rc != B200_OK:
        _raise(rc, "b200_gemm_f16 failed")
    return c, (ms.value if iters > 0 else None)


GEMM_MODES = {"f32": 0, "resid": 1, "gateup": 2}


def test_gemm(mode: str, a, b, c, b2=None, m_valid: int | None = None, stages: int = 4, splits: int = 1) -> np.ndarray:
    """One launch of the prefill GEMM (csrc/prefill_gemm.cuh) as the prefill issues it.  a [M,K], b (and b2 for "gateup") [N,K]
    float16; c is the initial output: float32 [M,N] for "f32" / "resid" (resid adds to it), float16 [M,N] for "gateup".
    Returns the output after the launch (a new array)."""
    a = np.ascontiguousarray(a, dtype=np.float16)
    b = np.ascontiguousarray(b, dtype=np.float16)
    gateup = mode == "gateup"
    c = np.array(c, dtype=np.float16 if gateup else np.float32, order="C", copy=True)
    m, k = a.shape
    n = b.shape[0]
    if b.shape != (n, k) or c.shape != (m, n):
        raise ValueError("shapes do not match")
    if gateup:
        b2 = np.ascontiguousarray(b2, dtype=np.float16)
        if b2.shape != b.shape:
            raise ValueError("b2 must have the shape of b")
    rc = lib().b200_test_gemm(GEMM_MODES[mode], stages, splits, m, m if m_valid is None else m_valid, n, k, a.ctypes.data, b.ctypes.data,
                              b2.ctypes.data if gateup else None, c.ctypes.data)
    if rc != B200_OK:
        _raise(rc, "b200_test_gemm failed")
    return c


def test_gemm_q8(mode: str, a, bq, c, bq2=None, m_valid: int | None = None, stages: int = 4, splits: int = 1) -> np.ndarray:
    """One launch of the W8A16 prefill GEMM (B dequantised from the tile-major Q8_0 stream in shared memory) as the
    B200_PREFILL_TENSOR_CORE_W8A16 prefill issues it.  As test_gemm, but bq (and bq2 for "gateup") are GGUF Q8_0 blocks:
    uint8 [N, K / 32 * 34].  stages 4 or 5."""
    a = np.ascontiguousarray(a, dtype=np.float16)
    bq = np.ascontiguousarray(bq, dtype=np.uint8)
    gateup = mode == "gateup"
    c = np.array(c, dtype=np.float16 if gateup else np.float32, order="C", copy=True)
    m, k = a.shape
    n = bq.shape[0]
    if bq.shape != (n, k // 32 * 34) or k % 32 or c.shape != (m, n):
        raise ValueError("shapes do not match")
    if gateup:
        bq2 = np.ascontiguousarray(bq2, dtype=np.uint8)
        if bq2.shape != bq.shape:
            raise ValueError("bq2 must have the shape of bq")
    rc = lib().b200_test_gemm_q8(GEMM_MODES[mode], stages, splits, m, m if m_valid is None else m_valid, n, k, a.ctypes.data, bq.ctypes.data,
                                 bq2.ctypes.data if gateup else None, c.ctypes.data)
    if rc != B200_OK:
        _raise(rc, "b200_test_gemm_q8 failed")
    return c


def test_gemm_i8(mode: str, aq, a_scales, bq, c=None, bq2=None, oscale: float = 1.0, hq=None, hs=None):
    """One launch of the int8 GEMM of B200_PREFILL_TENSOR_CORE_EXACT (csrc/prefill_i8.cuh) as the prefill issues it.  aq int8 [M,K],
    a_scales float32 [M, K/32], bq (and bq2, the up projection, for "gateup") GGUF Q8_0 blocks uint8 [N, K/32*34].  "f32" / "resid":
    c float32 [M,N] (resid adds fl(acc * oscale) to it); returns the new c.  "gateup": N hidden units, hq int8 [M,N] and hs float32
    [M, N/32] initial contents; returns the new (hq, hs)."""
    aq = np.ascontiguousarray(aq, dtype=np.int8)
    a_scales = np.ascontiguousarray(a_scales, dtype=np.float32)
    bq = np.ascontiguousarray(bq, dtype=np.uint8)
    m, k = aq.shape
    n = bq.shape[0]
    if a_scales.shape != (m, k // 32) or bq.shape != (n, k // 32 * 34) or k % 32:
        raise ValueError("shapes do not match")
    if mode == "gateup":
        bq2 = np.ascontiguousarray(bq2, dtype=np.uint8)
        hq = np.array(np.zeros((m, n), np.int8) if hq is None else hq, dtype=np.int8, order="C", copy=True)
        hs = np.array(np.zeros((m, n // 32), np.float32) if hs is None else hs, dtype=np.float32, order="C", copy=True)
        if bq2.shape != bq.shape or hq.shape != (m, n) or hs.shape != (m, n // 32):
            raise ValueError("shapes do not match")
        rc = lib().b200_test_gemm_i8(GEMM_MODES[mode], m, n, k, aq.ctypes.data, a_scales.ctypes.data, bq.ctypes.data, bq2.ctypes.data, oscale, None,
                                     hq.ctypes.data, hs.ctypes.data)
        if rc != B200_OK:
            _raise(rc, "b200_test_gemm_i8 failed")
        return hq, hs
    c = np.array(np.zeros((m, n), np.float32) if c is None else c, dtype=np.float32, order="C", copy=True)
    if c.shape != (m, n):
        raise ValueError("shapes do not match")
    rc = lib().b200_test_gemm_i8(GEMM_MODES[mode], m, n, k, aq.ctypes.data, a_scales.ctypes.data, bq.ctypes.data, None, oscale, c.ctypes.data, None, None)
    if rc != B200_OK:
        _raise(rc, "b200_test_gemm_i8 failed")
    return c


def test_gemm_i8_experts(mode: str, counts, aq, a_scales, bq, bq2=None, c=None, hq=None, hs=None):
    """One launch of the grouped expert GEMM of B200_PREFILL_TENSOR_CORE_EXACT_MOE (csrc/prefill_i8.cuh) as the prefill issues it.
    counts: grouped rows per expert (M = their sum, expert after expert); aq int8 [M,K], a_scales float32 [M, K/32]; bq (and bq2, the
    up projections, for "gateup") every expert's GGUF Q8_0 blocks uint8 [E, N, K/32*34].  "f32": returns c float32 [M,N] (initial
    contents c, default zeros).  "gateup": N hidden units; returns (hq int8 [M,N], hs float32 [M, N/32]) from the given initial
    contents."""
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    aq = np.ascontiguousarray(aq, dtype=np.int8)
    a_scales = np.ascontiguousarray(a_scales, dtype=np.float32)
    bq = np.ascontiguousarray(bq, dtype=np.uint8)
    m, k = aq.shape
    e, n = bq.shape[:2]
    if counts.shape != (e,) or int(counts.sum()) != m or a_scales.shape != (m, k // 32) or bq.shape != (e, n, k // 32 * 34) or k % 32:
        raise ValueError("shapes do not match")
    if mode == "gateup":
        bq2 = np.ascontiguousarray(bq2, dtype=np.uint8)
        hq = np.array(np.zeros((m, n), np.int8) if hq is None else hq, dtype=np.int8, order="C", copy=True)
        hs = np.array(np.zeros((m, n // 32), np.float32) if hs is None else hs, dtype=np.float32, order="C", copy=True)
        if bq2.shape != bq.shape or hq.shape != (m, n) or hs.shape != (m, n // 32):
            raise ValueError("shapes do not match")
        rc = lib().b200_test_gemm_i8_experts(GEMM_MODES[mode], e, counts.ctypes.data, n, k, aq.ctypes.data, a_scales.ctypes.data, bq.ctypes.data,
                                             bq2.ctypes.data, None, hq.ctypes.data, hs.ctypes.data)
        if rc != B200_OK:
            _raise(rc, "b200_test_gemm_i8_experts failed")
        return hq, hs
    c = np.array(np.zeros((m, n), np.float32) if c is None else c, dtype=np.float32, order="C", copy=True)
    if c.shape != (m, n):
        raise ValueError("shapes do not match")
    rc = lib().b200_test_gemm_i8_experts(GEMM_MODES[mode], e, counts.ctypes.data, n, k, aq.ctypes.data, a_scales.ctypes.data, bq.ctypes.data, None,
                                         c.ctypes.data, None, None)
    if rc != B200_OK:
        _raise(rc, "b200_test_gemm_i8_experts failed")
    return c


STREAM_MODES = {"store": 0, "resid": 1, "gateup": 2}
STREAM_INFO = ("stages", "grid", "max_groups", "min_groups", "smem")


def test_stream(form: int, mode: str, w, rows: int, cols: int, *, w_up=None, w_down=None, down_rows: int = 0, xq=None, xs=None, x=None,
                norm_w=None, eps: float = 1e-5, emb=None, emb_rows: int = 0, tokens=None, emb_scale: float = 1.0, out_init=None,
                oscale: float = 1.0, nrow: int = 0, lanes: int = 16, grid: int = 0, stages: int = 0, budget: int = 0, argmax: bool = False,
                launches: int = 1, pair: bool = False, dry: bool = False) -> dict:
    """b200_test_stream: one decode weight stream launched as the plan launches it, at any grid and ring depth.  form: 8 (Q8_0 tiles),
    12 / 13 / 14 (resident K-quant tiles) or 1 (F16 rings); w (and w_up for "gateup", w_down for pair) are raw GGUF rows of that type.
    Activations per launch: xq int8 [launches][V][cols] and xs [launches][V][cols / 32] (V = max(nrow, 1)), or x float32 [launches][cols]
    for F16 and the fused norm (norm_w given; emb + tokens instead of x: the embedding rows).  Returns {"info": the configuration run,
    and per launch "out", "hq", "hs", "out_down", "x_out", "ids" where they apply}.  dry: only the checks and "info" (grid must be given)."""
    V = max(nrow, 1)
    keep = []

    def arr(a, dtype):
        if a is None:
            return None
        a = np.ascontiguousarray(a, dtype=dtype)
        keep.append(a)
        return a.ctypes.data

    t = StreamTest()
    t.form, t.mode, t.norm, t.nrow, t.lanes, t.rows, t.cols = form, STREAM_MODES[mode], norm_w is not None, nrow, lanes, rows, cols
    t.grid, t.stages, t.budget, t.argmax, t.launches, t.pair, t.down_rows = grid, stages, budget, argmax, launches, pair, down_rows
    t.from_emb, t.emb_rows, t.dry, t.oscale, t.eps, t.emb_scale = emb is not None, emb_rows, dry, oscale, eps, emb_scale
    t.w, t.w_up, t.w_down = arr(w, np.uint8 if form != 1 else np.uint16), arr(w_up, np.uint8 if form != 1 else np.uint16), arr(w_down, np.uint8)
    t.xq, t.xs, t.x, t.norm_w, t.emb, t.tokens = arr(xq, np.int8), arr(xs, np.float32), arr(x, np.float32), arr(norm_w, np.float32), arr(emb, np.uint8), \
        arr(tokens, np.int32)
    t.out_init = arr(out_init, np.float32)
    res = {}
    if not dry:
        res["out"] = np.empty((launches, V, rows), np.float32)
        t.out = res["out"].ctypes.data
        if mode == "gateup" and form != 1:
            res["hq"], res["hs"] = np.empty((launches, V, rows), np.int8), np.empty((launches, V, rows // 32), np.float32)
            t.hq, t.hs = res["hq"].ctypes.data, res["hs"].ctypes.data
        if pair:
            res["out_down"] = np.empty((launches, down_rows), np.float32)
            t.out_down = res["out_down"].ctypes.data
        if emb is not None:
            res["x_out"] = np.empty((launches, cols), np.float32)
            t.x_out = res["x_out"].ctypes.data
        if argmax:
            res["ids"] = np.empty((launches, V), np.int32)
            t.ids = res["ids"].ctypes.data
    else:  # the pointer checks of a real launch, without the buffers
        t.out = t.hq = t.hs = t.x_out = t.ids = t.out_down = 1
    rc = lib().b200_test_stream(C.byref(t))
    if rc != B200_OK:
        _raise(rc, "b200_test_stream failed")
    res["info"] = dict(zip(STREAM_INFO, t.info))
    return res


ATTENTION_FORMS = {"single": 0, "batch": 1, "cached_rows": 2, "chunk": 3, "persistent": 4}
ATTENTION_INFO = ("grid_x", "grid_y", "smem", "global_scores", "launches")


def test_attention(form: str, head_size: int, n_heads: int, n_kv_heads: int, ctx: int, slots, positions, qkv, k_cache, v_cache, rope_cr,
                   rope_ci, *, arch: int = 0, eps: float = 1e-6, score_arg: float | None = None, q_norm=None, k_norm=None, qkv_bias=None,
                   att_tokens: int = 0, want_xb: bool = False, n_slots: int | None = None, dry: bool = False) -> dict:
    """b200_test_attention: one exact attention form launched as the plan launches it.  form: a key of ATTENTION_FORMS; row r is
    (slots[r], positions[r]); qkv float32 [rows][q | k | v]; caches float32 [n_slots][ctx][kv width]; rope tables [ctx][head_size / 2].
    score_arg: sqrt(head_size) by default (Granite: its attention multiplier with arch & 8).  Returns {"info": the configuration run, and
    "qkv", "k_cache", "v_cache" after the launch, "xq" [rows][q width], "xs" [rows][q width / 32], "xb" (want_xb, single form)}.
    dry: only the checks and "info" (n_slots then stands for the caches' first dimension)."""
    slots = np.ascontiguousarray(slots, dtype=np.int32)
    positions = np.ascontiguousarray(positions, dtype=np.int32)
    keep = [slots, positions]

    def arr(a):
        if a is None:
            return None
        a = np.ascontiguousarray(a, dtype=np.float32)
        keep.append(a)
        return a.ctypes.data

    rows, qd = len(slots), n_heads * head_size
    t = AttentionTest()
    t.form, t.head_size, t.n_heads, t.n_kv_heads, t.arch, t.ctx = ATTENTION_FORMS[form], head_size, n_heads, n_kv_heads, arch, ctx
    t.rows, t.att_tokens, t.dry, t.eps = rows, att_tokens, dry, eps
    t.score_arg = float(np.sqrt(np.float64(head_size))) if score_arg is None else score_arg
    t.slot, t.pos = slots.ctypes.data, positions.ctypes.data
    t.qkv, t.rope_cr, t.rope_ci, t.q_norm, t.k_norm, t.qkv_bias = arr(qkv), arr(rope_cr), arr(rope_ci), arr(q_norm), arr(k_norm), arr(qkv_bias)
    res = {}
    if dry:  # the pointer checks of a real launch, without the buffers
        t.slots = n_slots
        t.qkv = t.k_cache = t.v_cache = t.rope_cr = t.rope_ci = t.qkv_out = t.k_out = t.v_out = t.xq = t.xs = 1
        t.q_norm, t.k_norm, t.qkv_bias = t.q_norm or 1, t.k_norm or 1, t.qkv_bias or 1
    else:
        kc, vc = np.ascontiguousarray(k_cache, dtype=np.float32), np.ascontiguousarray(v_cache, dtype=np.float32)
        keep += [kc, vc]
        t.slots = kc.shape[0]
        t.k_cache, t.v_cache = kc.ctypes.data, vc.ctypes.data
        res["qkv"], res["k_cache"], res["v_cache"] = np.empty((rows, qkv.shape[-1]), np.float32), np.empty_like(kc), np.empty_like(vc)
        res["xq"], res["xs"] = np.empty((rows, qd), np.int8), np.empty((rows, qd // 32), np.float32)
        t.qkv_out, t.k_out, t.v_out = res["qkv"].ctypes.data, res["k_cache"].ctypes.data, res["v_cache"].ctypes.data
        t.xq, t.xs = res["xq"].ctypes.data, res["xs"].ctypes.data
        if want_xb:
            res["xb"] = np.empty(qd, np.float32)
            t.xb = res["xb"].ctypes.data
    rc = lib().b200_test_attention(C.byref(t))
    if rc != B200_OK:
        _raise(rc, "b200_test_attention failed")
    res["info"] = dict(zip(ATTENTION_INFO, t.info))
    return res


def test_exp(first: int, n: int):
    """b200_test_exp: ((float)exp((double)x), (float)(1.0 + exp((double)x))) on the device for the n float bit patterns from `first`."""
    e, e1 = np.empty(n, np.float32), np.empty(n, np.float32)
    rc = lib().b200_test_exp(first, n, e.ctypes.data, e1.ctypes.data)
    if rc != B200_OK:
        _raise(rc, "b200_test_exp failed")
    return e, e1


def _pf_attention_packed(qs, ks, vs, starts, n_heads: int, n_kv_heads: int, out_rows: int | None, sentinel: int) -> np.ndarray:
    lens = np.array([len(q) for q in qs], dtype=np.int32)
    st = np.ascontiguousarray(starts, dtype=np.int32)
    hs = qs[0].shape[1] // n_heads
    q = np.ascontiguousarray(np.concatenate(qs), dtype=np.float32)
    k = np.ascontiguousarray(np.concatenate(ks), dtype=np.float32)
    v = np.ascontiguousarray(np.concatenate(vs), dtype=np.float32)
    if len(st) != len(qs) or any(np.shape(ks[i]) != (st[i] + lens[i], n_kv_heads * hs) or np.shape(vs[i]) != np.shape(ks[i]) for i in range(len(qs))):
        raise ValueError("ks[i] / vs[i] must be [starts[i] + n_i, n_kv_heads * head_size]")
    out = np.full((int(lens.sum()) if out_rows is None else out_rows, n_heads * hs), sentinel, dtype=np.uint16)
    rc = lib().b200_test_pf_attention_packed(len(qs), lens.ctypes.data, st.ctypes.data, q.ctypes.data, k.ctypes.data, v.ctypes.data, n_heads,
                                             n_kv_heads, hs, len(out), out.ctypes.data)
    if rc != B200_OK:
        _raise(rc, "b200_test_pf_attention_packed failed")
    return out


def test_pf_attention_packed(qs, ks, vs, starts, n_heads: int, n_kv_heads: int, sentinel: int = 0x7E5A) -> list:
    """The prefill's causal attention (k_pf_attention_mma_packed, csrc/prefill.cuh) over several sequences in one launch.  qs[i]
    float32 [n_i, n_heads*hs]; ks[i], vs[i] float32 [starts[i]+n_i, n_kv_heads*hs].  Returns each sequence's f16 bits [n_i, n_heads*hs]."""
    lens = [len(q) for q in qs]
    return np.split(_pf_attention_packed(qs, ks, vs, starts, n_heads, n_kv_heads, None, sentinel), np.cumsum(lens)[:-1])


def test_pf_attention(q, k, v, n_heads: int, n_kv_heads: int, start_pos: int, out_rows: int | None = None, sentinel: int = 0x7E5A) -> np.ndarray:
    """The prefill's causal attention over one sequence: a chunk that holds it alone.  q float32 [n, n_heads*hs]; k, v float32
    [start_pos+n, n_kv_heads*hs].  Returns the f16 bits (uint16) of [out_rows, n_heads*hs]: rows >= n keep `sentinel`."""
    return _pf_attention_packed([q], [k], [v], [start_pos], n_heads, n_kv_heads, out_rows, sentinel)


GGML_SIZES = {0: (4, 1), 1: (2, 1), 8: (34, 32), 12: (144, 256), 13: (176, 256), 14: (210, 256)}  # (bytes, elements) per block, GGMLType.java:5-20


def test_logprobs(logits, chosen_id: int, top_n: int, reps: int = 1):
    """b200_test_logprobs: k_token_logprobs on one row -> (chosen, top ids int32 [top_n], top logprobs float64 [top_n], ms per launch)."""
    lg = np.ascontiguousarray(logits, dtype=np.float32).reshape(-1)
    c = C.c_double(0)
    ids = np.empty(top_n, np.int32)
    lps = np.empty(top_n, np.float64)
    ms = C.c_float(0)
    rc = lib().b200_test_logprobs(lg.ctypes.data, len(lg), int(chosen_id), int(top_n), int(reps), C.byref(c), ids.ctypes.data, lps.ctypes.data, C.byref(ms))
    if rc != B200_OK:
        _raise(rc, "b200_test_logprobs failed")
    return c.value, ids, lps, ms.value


class NativePlan:
    """Owns one ``b200_plan*``."""

    def __init__(self, cfg: Config, tensors: dict, prefill_batch_size: int = 0, device: int = 0, moe: MoeConfig | None = None,
                 granite: GraniteConfig | None = None, devstral: bool = False, yarn: YarnConfig | None = None):
        """devstral: create through b200_plan_create_devstral, with `yarn` (None: the plain RoPE table)."""
        L = lib()
        arr = (Tensor * len(tensors))()
        self._keep = []
        for i, (name, (tt, dims, raw)) in enumerate(tensors.items()):
            raw = np.ascontiguousarray(raw)
            ts_bs = GGML_SIZES.get(int(tt))
            n_el = int(np.prod(dims))
            if ts_bs is not None and (n_el % ts_bs[1] or raw.nbytes != n_el // ts_bs[1] * ts_bs[0]):
                # the C ABI takes plain pointers: a short buffer would be read past its end on the device side of the upload
                raise B200Error(-1, f"tensor {name}: {raw.nbytes} bytes do not hold {n_el} elements of ggml type {int(tt)}")
            self._keep.append(raw)
            arr[i].name = name.encode()
            arr[i].data = raw.ctypes.data
            arr[i].ggml_type = int(tt)
            arr[i].n_dims = len(dims)
            for k, d in enumerate(dims):
                arr[i].dims[k] = int(d)
        out = C.c_void_p()
        err = C.create_string_buffer(512)
        if devstral:
            rc = L.b200_plan_create_devstral(C.byref(cfg), C.byref(yarn) if yarn is not None else None, arr, len(tensors), prefill_batch_size,
                                             device, C.byref(out), err, 512)
        elif granite is not None:
            rc = L.b200_plan_create_granite(C.byref(cfg), C.byref(granite), arr, len(tensors), prefill_batch_size, device, C.byref(out), err, 512)
        elif moe is not None:
            rc = L.b200_plan_create_moe(C.byref(cfg), C.byref(moe), arr, len(tensors), prefill_batch_size, device, C.byref(out), err, 512)
        else:
            rc = L.b200_plan_create(C.byref(cfg), arr, len(tensors), prefill_batch_size, device, C.byref(out), err, 512)
        self._keep = None  # the library never touches the host pointers again
        if rc != B200_OK:
            _raise(rc, err.value.decode())
        self._p = out
        self.cfg = cfg
        self.moe = moe

    def _ck(self, rc: int):
        if rc != B200_OK:
            _raise(rc, lib().b200_last_error(self._p).decode())

    def forward_decode(self, token: int, position: int, want_logits: bool = True, want_argmax: bool = True):
        logits = np.empty(self.cfg.vocab_size, dtype=np.float32) if want_logits else None
        am = C.c_int32(-1)
        self._ck(lib().b200_forward_decode(self._p, token, position, logits.ctypes.data if want_logits else None,
                                           C.byref(am) if want_argmax else None))
        return logits, (am.value if want_argmax else None)

    def forward_decode_sample(self, token: int, position: int, temperature: float, topp: float, uniform01: float, want_info: bool = False):
        out = C.c_int32(-1)
        info = (C.c_int32 * 4)()
        self._ck(lib().b200_forward_decode_sample(self._p, token, position, temperature, topp, uniform01, C.byref(out), info))
        return (out.value, list(info)) if want_info else out.value

    def forward_prefill(self, token: int, position: int):
        self._ck(lib().b200_forward_prefill(self._p, token, position))

    def set_prefill_mode(self, mode: int):
        self._ck(lib().b200_set_prefill_mode(self._p, mode))

    def set_decode_mode(self, mode: int):
        self._ck(lib().b200_set_decode_mode(self._p, mode))

    def decode_info(self):
        """(mode, kernels per decode step, ring stages, shared-memory bytes of the persistent kernel)."""
        a, b, c, d = C.c_int32(0), C.c_int32(0), C.c_int32(0), C.c_int32(0)
        self._ck(lib().b200_decode_info(self._p, C.byref(a), C.byref(b), C.byref(c), C.byref(d)))
        return a.value, b.value, c.value, d.value

    def trace_persistent(self, token: int, position: int) -> np.ndarray:
        """uint64 %globaltimer stamps [cta][row][k] of one traced step of the persistent decode kernel."""
        cap = 200 * (self.cfg.n_layers + 1) * 32
        buf = np.zeros(cap, dtype=np.uint64)
        a, b, c = C.c_int32(0), C.c_int32(0), C.c_int32(0)
        self._ck(lib().b200_trace_persistent(self._p, token, position, buf.ctypes.data, cap, C.byref(a), C.byref(b), C.byref(c)))
        return buf[: a.value * b.value * c.value].reshape(a.value, b.value, c.value)

    def prefill_info(self):
        mode, launches, ms = C.c_int32(0), C.c_int32(0), C.c_float(0)
        self._ck(lib().b200_prefill_info(self._p, C.byref(mode), C.byref(launches), C.byref(ms)))
        return mode.value, launches.value, ms.value

    def forward_batch_prefill(self, tokens, start_pos: int):
        t = np.ascontiguousarray(tokens, dtype=np.int32)
        self._ck(lib().b200_forward_batch_prefill(self._p, t.ctypes.data, len(t), start_pos))
        self._chunk_rows = len(t)

    def score_tokens(self, tokens, start_pos: int, targets=None):
        """b200_score_tokens: run tokens[i] at start_pos + i (K/V into the plan's cache) and score each row.  targets[i] is the token
        whose log-probability row i reports (-1: none, NaN); the default is the next token of `tokens`, -1 for the last row.
        Returns (logprobs float64 [n], greedy ids int32 [n])."""
        t = np.ascontiguousarray(tokens, dtype=np.int32).reshape(-1)
        n = len(t)
        tg = np.append(t[1:], np.int32(-1)) if targets is None else np.ascontiguousarray(targets, dtype=np.int32).reshape(-1)
        if len(tg) != n:
            raise ValueError("targets must have one entry per token")
        lp = np.empty(n, dtype=np.float64)
        ids = np.empty(n, dtype=np.int32)
        self._ck(lib().b200_score_tokens(self._p, t.ctypes.data, tg.ctypes.data, n, start_pos, lp.ctypes.data, ids.ctypes.data))
        self._chunk_rows = n
        return lp, ids

    MAX_TOP_LOGPROBS = 20  # B200_MAX_TOP_LOGPROBS

    def set_logprobs(self, top_n: int):
        """b200_set_logprobs: -1 off (the default); 0..20 alternatives per emitted row while on."""
        self._ck(lib().b200_set_logprobs(self._p, int(top_n)))
        self._top_n = int(top_n)

    def logprobs_top_n(self) -> int:
        return getattr(self, "_top_n", -1)

    def last_logprobs(self):
        """b200_read_logprobs: the last emitting call's rows -> (chosen float64 [rows], top_ids int32 [rows, N],
        top_logprobs float64 [rows, N])."""
        n_top = max(self.logprobs_top_n(), 0)
        rows = C.c_int32(0)
        self._ck(lib().b200_read_logprobs(self._p, 0, C.byref(rows), None, None, None))  # the row count alone
        r = rows.value
        chosen = np.empty(r, dtype=np.float64)
        ids = np.empty((r, n_top), dtype=np.int32)
        lps = np.empty((r, n_top), dtype=np.float64)
        self._ck(lib().b200_read_logprobs(self._p, r, C.byref(rows), chosen.ctypes.data, ids.ctypes.data, lps.ctypes.data))
        return chosen, ids, lps

    def set_sampling_controls(self, slot: int, controls: SamplingControls | None):
        """b200_set_sampling_controls: controls for one sequence (slot -1: the plan's own cache); None turns them off."""
        if controls is None:
            self._ck(lib().b200_set_sampling_controls(self._p, slot, None))
            return
        cs, keep = _controls_c(controls)
        self._ck(lib().b200_set_sampling_controls(self._p, slot, C.byref(cs)))

    def set_sample_history(self, slot: int, tokens):
        """b200_set_sample_history: the sequence's counts become those of tokens."""
        t = np.ascontiguousarray(tokens, dtype=np.int32).reshape(-1)
        self._ck(lib().b200_set_sample_history(self._p, slot, t.ctypes.data if len(t) else None, len(t)))

    def sample_counts(self, slot: int) -> np.ndarray:
        """b200_read_sample_counts: the sequence's count per token id, int32 [vocab]."""
        out = np.empty(self.cfg.vocab_size, dtype=np.int32)
        self._ck(lib().b200_read_sample_counts(self._p, slot, out.ctypes.data))
        return out

    def decode_sequence(self, tokens, n: int, start_pos: int, feedback: bool = False):
        t = np.ascontiguousarray(tokens, dtype=np.int32)
        out = np.empty(n, dtype=np.int32)
        ms = C.c_float(0)
        self._ck(lib().b200_decode_sequence(self._p, t.ctypes.data, n, start_pos, 1 if feedback else 0, out.ctypes.data, C.byref(ms)))
        return out, ms.value

    def set_decode_slots(self, n_slots: int):
        self._ck(lib().b200_set_decode_slots(self._p, n_slots))

    def forward_decode_batch(self, slots, tokens, positions, sampling=None, want_logits: bool = False):
        """One batched step (b200_forward_decode_batch): row i = tokens[i] at positions[i] on slot slots[i].  sampling: None or
        n x (temperature, topp, uniform01).  Returns (ids int32 [n], logits float32 [n, vocab] or None)."""
        s = np.ascontiguousarray(slots, dtype=np.int32)
        t = np.ascontiguousarray(tokens, dtype=np.int32)
        p = np.ascontiguousarray(positions, dtype=np.int32)
        n = len(s)
        if len(t) != n or len(p) != n:
            raise ValueError("slots, tokens and positions must have the same length")
        smp = None
        if sampling is not None:
            smp = np.ascontiguousarray(sampling, dtype=np.float32).reshape(-1)
            if smp.size != 3 * n:
                raise ValueError("sampling must hold (temperature, topp, uniform01) per row")
        ids = np.empty(n, dtype=np.int32)
        lg = np.empty((n, self.cfg.vocab_size), dtype=np.float32) if want_logits else None
        self._ck(lib().b200_forward_decode_batch(self._p, n, s.ctypes.data, t.ctypes.data, p.ctypes.data, smp.ctypes.data if smp is not None else None,
                                                 ids.ctypes.data, lg.ctypes.data if want_logits else None))
        return ids, lg

    def slot_reset(self, slot: int):
        self._ck(lib().b200_slot_reset(self._p, slot))

    def slot_copy_kv(self, slot: int, n_positions: int):
        self._ck(lib().b200_slot_copy_kv(self._p, slot, n_positions))

    def prefill_slots(self, slots, start_positions, token_lists):
        """b200_prefill_slots: token_lists[i] into slot slots[i] at positions start_positions[i].. (K/V only)."""
        s = np.ascontiguousarray(slots, dtype=np.int32)
        st = np.ascontiguousarray(start_positions, dtype=np.int32)
        if len(st) != len(s) or len(token_lists) != len(s):
            raise ValueError("slots, start_positions and token_lists must have the same length")
        ln = np.array([len(t) for t in token_lists], dtype=np.int32)
        toks = np.ascontiguousarray(np.concatenate([np.asarray(t, dtype=np.int32).reshape(-1) for t in token_lists]) if len(s) else np.zeros(0), dtype=np.int32)
        self._ck(lib().b200_prefill_slots(self._p, len(s), s.ctypes.data, st.ctypes.data, ln.ctypes.data, toks.ctypes.data))

    def batch_info(self):
        """(decode slots, kernels of the last batched step, its device milliseconds)."""
        a, b, ms = C.c_int32(0), C.c_int32(0), C.c_float(0)
        self._ck(lib().b200_batch_info(self._p, C.byref(a), C.byref(b), C.byref(ms)))
        return a.value, b.value, ms.value

    def forward_decode_multi(self, slot: int, tokens, start_pos: int, want_logits: bool = False):
        """b200_forward_decode_multi: tokens[i] at start_pos + i of one sequence (slot -1: the plan's own cache) in one step.
        Returns (ids int32 [n], logits float32 [n, vocab] or None)."""
        t = np.ascontiguousarray(tokens, dtype=np.int32).reshape(-1)
        n = len(t)
        ids = np.empty(max(n, 1), dtype=np.int32)
        lg = np.empty((n, self.cfg.vocab_size), dtype=np.float32) if want_logits else None
        self._ck(lib().b200_forward_decode_multi(self._p, slot, n, t.ctypes.data, start_pos, ids.ctypes.data, lg.ctypes.data if want_logits else None))
        return ids[:n], lg

    def forward_step(self, rows, logits: bool = False):
        """b200_forward_step: one mixed step.  rows: (slot, token, position, emit[, temperature, topp, uniform01]) per row.  Returns
        (ids int32 [n], -1 where emit is 0; logits float32 [n, vocab] or None, rows with emit 0 left unwritten)."""
        return self._step_rows(lib().b200_forward_step, rows, logits)

    def forward_chunk(self, rows, logits: bool = False):
        """b200_forward_chunk: forward_step's rows and results, run as one chunk of the tensor_core_exact prefill."""
        return self._step_rows(lib().b200_forward_chunk, rows, logits)

    def _step_rows(self, fn, rows, logits):
        n = len(rows)
        arr = (StepRow * max(n, 1))()
        for i, r in enumerate(rows):
            if len(r) not in (4, 7):
                raise ValueError(f"row {i}: (slot, token, position, emit) or (slot, token, position, emit, temperature, topp, uniform01)")
            arr[i] = StepRow(*[int(v) for v in r[:4]], *[float(v) for v in r[4:]])
        ids = np.empty(max(n, 1), dtype=np.int32)
        lg = np.zeros((n, self.cfg.vocab_size), dtype=np.float32) if logits else None
        self._ck(fn(self._p, n, arr, ids.ctypes.data, lg.ctypes.data if logits else None))
        return ids[:n], lg

    def chunk_rows(self) -> int:
        r = C.c_int32(0)
        self._ck(lib().b200_chunk_rows(self._p, C.byref(r)))
        return r.value

    def decode_multi_rows(self) -> int:
        r = C.c_int32(0)
        self._ck(lib().b200_decode_multi_rows(self._p, C.byref(r)))
        return r.value

    def time_kernel(self, which: int, reps: int = 3):
        ms, nbytes = C.c_float(0), C.c_int64(0)
        self._ck(lib().b200_time_kernel(self._p, which, reps, C.byref(ms), C.byref(nbytes)))
        return ms.value, nbytes.value

    def tp_handle(self) -> bytes:
        buf = C.create_string_buffer(64)
        self._ck(lib().b200_tp_handle(self._p, buf))
        return buf.raw

    def tp_attach(self, handles: list):
        blob = b"".join(handles)
        self._ck(lib().b200_tp_attach(self._p, blob, len(handles)))

    def trace_decode(self, token: int, position: int):
        cap = self.launches_per_decode + 8
        rec = np.zeros((cap, 4), dtype=np.uint64)
        n = C.c_int32(0)
        self._ck(lib().b200_trace_decode(self._p, token, position, rec.ctypes.data, cap, C.byref(n)))
        return rec[: n.value]

    def profile_norm(self):
        a = (C.c_int64 * 16)()
        self._ck(lib().b200_profile_norm(self._p, a))
        return list(a)

    def kv_reset(self):
        self._ck(lib().b200_kv_reset(self._p))

    def read_buffer(self, name: str, n: int, dtype=np.float32, layer: int = 0) -> np.ndarray:
        out = np.empty(n, dtype=dtype)
        self._ck(lib().b200_read_buffer(self._p, name.encode(), layer, out.ctypes.data, out.nbytes))
        return out

    def moe_routing(self):
        """(ids int32 [layer, k], weights float32 [layer, k + 1]) of the last step: the selected experts in selection order, their
        routing weights, then the shared-expert weight.  Without a shared expert (Qwen3-MoE) the weights are [layer, k]."""
        k = self.moe.n_experts_used
        nw = k + 1 if self.moe.shared_hidden_dim else k
        ids = self.read_buffer("moe_ids", self.cfg.n_layers * k, np.int32).reshape(self.cfg.n_layers, k)
        w = self.read_buffer("moe_weights", self.cfg.n_layers * nw).reshape(self.cfg.n_layers, nw)
        return ids, w

    def moe_chunk_routing(self, rows: int | None = None):
        """(ids int32 [layer, rows, k], weights float32 [layer, rows, k + 1]) of the last tensor_core_exact_moe chunk: every row's
        selected experts in selection order, their routing weights, then the shared-expert weight (Qwen3-MoE: [layer, rows, k]).
        rows defaults to the length of the last forward_batch_prefill / score_tokens call."""
        rows = getattr(self, "_chunk_rows", 0) if rows is None else rows
        k = self.moe.n_experts_used
        nw = k + 1 if self.moe.shared_hidden_dim else k
        L = self.cfg.n_layers
        ids = np.stack([self.read_buffer("moe_chunk_ids", rows * k, np.int32, layer=l).reshape(rows, k) for l in range(L)])
        w = np.stack([self.read_buffer("moe_chunk_weights", rows * nw, layer=l).reshape(rows, nw) for l in range(L)])
        return ids, w

    def upload_info(self) -> dict:
        a, b, c = C.c_double(0), C.c_double(0), C.c_int64(0)
        self._ck(lib().b200_upload_info(self._p, C.byref(a), C.byref(b), C.byref(c)))
        return {"seconds": a.value, "host_copy_seconds": b.value, "h2d_bytes": c.value,
                "GB/s": (c.value / a.value / 1e9) if a.value > 0 else None}

    def weight_info(self) -> dict:
        """b200_weight_info: whether the plan keeps K-quant weights resident, its weight bytes and those of its all-Q8_0 form."""
        r, w, w8 = C.c_int32(0), C.c_int64(0), C.c_int64(0)
        self._ck(lib().b200_weight_info(self._p, C.byref(r), C.byref(w), C.byref(w8)))
        return {"resident": bool(r.value), "weight_bytes": w.value, "q8_weight_bytes": w8.value}

    @property
    def launches_per_decode(self) -> int:
        return lib().b200_launches_per_decode(self._p)

    @property
    def device_bytes(self) -> int:
        return lib().b200_device_bytes(self._p)

    def free(self):
        if self._p:
            lib().b200_plan_free(self._p)
            self._p = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass
