"""Host-side mirror of the reference model loaders (metadata -> Configuration, tensor names ->
weight slots).  Mirrors ``model/loader/ModelLoader.java:47-108`` (type detection on
``general.name``), ``LlamaModelLoader.java:47-63`` / ``Qwen3ModelLoader.java:48-74`` / ``Qwen2ModelLoader.java:48-73`` / ``GraniteLoader.java:48-92``
(configuration keys), ``AbstractModelLoader.java:40-50`` (file_type -> quantisation) and
``AbstractModelLoader.java:186-195`` (tied output falls back to ``token_embd.weight``).
Weights stay in GGUF block layout; the native library repacks at upload.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from .gguf import GGMLType, GGUFFile

ARCH_LLAMA = 0
ARCH_QWEN3 = 1
ARCH_PHI3 = 2
ARCH_QWEN2 = 3  # Qwen2 / Qwen2.5 / DeepSeek-R1-Distill-Qwen: Llama's forward + q/k/v biases, NeoX RoPE (InferenceCore.java:434-563)
ARCH_QWEN2_MOE = 4  # Qwen1.5-MoE: Qwen2's attention + a routed mixture-of-experts FFN with a shared expert (InferenceCore.java:263-432)
ARCH_GRANITE = 5  # Granite 3.x: Llama's forward with four muP scales (InferenceCore.forwardGranite, InferenceCore.java:814-921)

# GraniteLoader.createConfiguration's defaults for the four scales (GraniteLoader.java:55-58)
GRANITE_DEFAULT_SCALES = {"embedding_scale": 12.0, "residual_scale": 0.22, "attention_scale": 0.0078125, "logit_scale": 16.0}


@dataclass
class Configuration:
    arch: int
    quantization: str  # "FP16" | "Q8_0"
    dim: int
    hidden_dim: int
    n_layers: int
    n_heads: int
    n_kv_heads: int
    head_size: int
    vocab_size: int
    context_length: int
    rms_norm_eps: float
    rope_theta: float
    # Qwen2-MoE only (Qwen2MoEConfiguration); 0 for every dense model
    n_experts: int = 0
    n_experts_used: int = 0
    expert_hidden_dim: int = 0
    shared_hidden_dim: int = 0
    # Granite only (GraniteConfiguration); 1.0 for every other family
    embedding_scale: float = 1.0
    residual_scale: float = 1.0
    attention_scale: float = 1.0
    logit_scale: float = 1.0

    @property
    def q_dim(self):
        return self.n_heads * self.head_size

    @property
    def kv_dim(self):
        return self.n_kv_heads * self.head_size


class UnsupportedModel(Exception):
    """Maps to the reference's UnsupportedOperationException (ForwardPlanFactory.java:84-87)."""


def detect_model_type(metadata: dict) -> str:
    if metadata.get("general.architecture") == "qwen2moe":  # checked before the name (ModelLoader.java:50)
        return "QWEN_2_MOE"
    name = metadata.get("general.name")
    if name is not None:
        low = name.lower()
        for key, typ in (("granite", "GRANITE"), ("devstral", "DEVSTRAL_2"), ("mistral", "MISTRAL"),
                         ("llama", "LLAMA_3"), ("qwen2", "QWEN_2"), ("qwen3", "QWEN_3"),
                         ("deepseek r1 distill", "DEEPSEEK_R1_DISTILL_QWEN"), ("phi3", "PHI_3"), ("phi-3", "PHI_3")):
            if key in low:
                return typ
    return "UNKNOWN"


def _quantization(metadata: dict) -> str:
    ft = int(metadata["general.file_type"])
    if ft == 1:
        return "FP16"
    if ft == 7:
        return "Q8_0"
    if ft in (14, 15, 16, 17, 18):  # Q4_K_S/M, Q5_K_S/M, Q6_K: the accelerator path computes in Q8_0 (AbstractModelLoader.java:45-47)
        return "Q8_0"
    raise UnsupportedModel(f"Unsupported quantization format: {ft} (as int).")


class Model:
    """Configuration + raw tensor views.  ``tensors[name] = (ggml_type, dims, uint8 ndarray)``."""

    def __init__(self, gguf: GGUFFile | None, config: Configuration, model_type: str, tensors: dict | None = None):
        self.gguf = gguf
        self.configuration = config
        self.model_type = model_type
        self.tensors = dict(tensors) if tensors is not None else {}
        if gguf is not None:
            for name, ti in gguf.tensor_infos.items():
                if name == "rope_freqs.weight":  # GGUF.java:121-124
                    continue
                self.tensors[name] = (ti.ggml_type, ti.dims, gguf.tensor_bytes(name))
        self.plan = None  # Model.setTornadoVMPlan
        self.latest_token = None


def model_from_tensors(shape, quant: int, tensors: dict, context_length: int) -> Model:
    """In-memory model (bench: synthetic weights never touch the disk)."""
    arch = {"llama": ARCH_LLAMA, "qwen3": ARCH_QWEN3, "phi3": ARCH_PHI3, "qwen2": ARCH_QWEN2, "qwen2moe": ARCH_QWEN2_MOE, "granite": ARCH_GRANITE}[shape.arch]
    moe = shape.arch == "qwen2moe"
    cfg = Configuration(arch, "Q8_0" if quant == GGMLType.Q8_0 else "FP16",
                        shape.dim, 0 if moe else shape.hidden, shape.n_layers, shape.n_heads, shape.n_kv_heads, shape.head_size,
                        shape.vocab, context_length, float(shape.eps), float(shape.rope_theta))
    if moe:
        cfg.n_experts, cfg.n_experts_used = shape.n_experts, shape.n_experts_used
        cfg.expert_hidden_dim, cfg.shared_hidden_dim = shape.expert_hidden, shape.hidden
    if shape.arch == "granite":
        for k, v in shape.granite_scales.items():
            setattr(cfg, k, float(np.float32(v)))
    typ = {"llama": "LLAMA_3", "qwen3": "QWEN_3", "phi3": "PHI_3", "qwen2": "QWEN_2", "qwen2moe": "QWEN_2_MOE", "granite": "GRANITE"}[shape.arch]
    return Model(None, cfg, typ, tensors)


def load_model(path: str, context_length: int = -1) -> Model:
    """``ModelLoader.loadModel(Path,int,boolean,boolean)`` (ModelLoader.java:113-120)."""
    g = GGUFFile(path)
    md = g.metadata
    typ = detect_model_type(md)
    q = _quantization(md)
    if typ == "LLAMA_3" or typ == "MISTRAL":
        # Mistral runs the same forward as Llama (Mistral.java -> InferenceCore.forwardJava; weights in the same
        # LlamaStandardWeights slots, MistralModelLoader.java:92-113).  Differences are host-side only: the context is
        # clamped to the model's (MistralModelLoader.java:45-46) and the vocabulary size may come from the token list.
        vocab = md.get("llama.vocab_size")
        if vocab is None:
            vocab = len(md["tokenizer.ggml.tokens"])
        model_ctx = int(md["llama.context_length"])
        n_heads = int(md["llama.attention.head_count"])
        dim = int(md["llama.embedding_length"])
        if typ == "MISTRAL":
            ctx = model_ctx if (context_length < 0 or model_ctx < context_length) else context_length
        else:  # withContextLength(contextLength): LlamaConfiguration keeps the requested length when >= 0
            ctx = model_ctx if context_length < 0 else context_length
        cfg = Configuration(
            ARCH_LLAMA, q, dim, int(md["llama.feed_forward_length"]), int(md["llama.block_count"]), n_heads,
            int(md.get("llama.attention.head_count_kv", n_heads)), dim // n_heads, int(vocab), ctx,
            float(md.get("llama.attention.layer_norm_rms_epsilon", 1e-5)), float(md.get("llama.rope.freq_base", 10000.0)))
    elif typ == "QWEN_3":
        model_ctx = int(md["qwen3.context_length"])
        ctx = model_ctx if (context_length < 0 or model_ctx < context_length) else context_length
        vocab = md.get("qwen3.vocab_size")
        if vocab is None:
            vocab = len(md["tokenizer.ggml.tokens"])
        n_heads = int(md["qwen3.attention.head_count"])
        if int(md["qwen3.attention.key_length"]) != int(md["qwen3.attention.value_length"]):
            raise UnsupportedModel("key_length != value_length")
        cfg = Configuration(
            ARCH_QWEN3, q, int(md["qwen3.embedding_length"]), int(md["qwen3.feed_forward_length"]),
            int(md["qwen3.block_count"]), n_heads, int(md.get("qwen3.attention.head_count_kv", n_heads)),
            int(md["qwen3.attention.key_length"]), int(vocab), ctx,
            float(md["qwen3.attention.layer_norm_rms_epsilon"]), float(md["qwen3.rope.freq_base"]))
    elif typ == "PHI_3":
        # Phi3ModelLoader.createConfiguration (Phi3ModelLoader.java:51-71): head size = dim / heads, the context is the requested one
        # (the RoPE table is precomputed for the model's), the vocabulary size is the token list's.
        n_heads = int(md["phi3.attention.head_count"])
        dim = int(md["phi3.embedding_length"])
        model_ctx = int(md["phi3.context_length"])
        vocab = len(md["tokenizer.ggml.tokens"]) if "tokenizer.ggml.tokens" in md else int(md["phi3.vocab_size"])
        cfg = Configuration(
            ARCH_PHI3, q, dim, int(md["phi3.feed_forward_length"]), int(md["phi3.block_count"]), n_heads,
            int(md.get("phi3.attention.head_count_kv", n_heads)), dim // n_heads, int(vocab), model_ctx if context_length < 0 else context_length,
            float(md.get("phi3.attention.layer_norm_rms_epsilon", 1e-5)), float(md.get("phi3.rope.freq_base", 10000.0)))
    elif typ in ("QWEN_2", "DEEPSEEK_R1_DISTILL_QWEN"):
        # Qwen2ModelLoader.createConfiguration (Qwen2ModelLoader.java:48-73): qwen2.* keys, head_count_kv defaults to head_count, the
        # vocabulary size is the token list's, the context is clamped to the model's, eps and theta have no defaults;
        # head size = dim / heads (Qwen2Configuration.java:25-32).
        model_ctx = int(md["qwen2.context_length"])
        ctx = model_ctx if (context_length < 0 or model_ctx < context_length) else context_length
        n_heads = int(md["qwen2.attention.head_count"])
        dim = int(md["qwen2.embedding_length"])
        cfg = Configuration(
            ARCH_QWEN2, q, dim, int(md["qwen2.feed_forward_length"]), int(md["qwen2.block_count"]), n_heads,
            int(md.get("qwen2.attention.head_count_kv", n_heads)), dim // n_heads, len(md["tokenizer.ggml.tokens"]), ctx,
            float(md["qwen2.attention.layer_norm_rms_epsilon"]), float(md["qwen2.rope.freq_base"]))
    elif typ == "QWEN_2_MOE":
        cfg = _qwen2moe_configuration(md, g, q, context_length)
    elif typ == "GRANITE":
        cfg = granite_configuration(md, q, context_length)
    else:
        raise UnsupportedModel(f"model type {typ} is outside the hot-path scope (Llama / Mistral / Qwen3 / Phi-3 / Qwen2 / Qwen2-MoE / Granite forward passes only)")
    return Model(g, cfg, typ)


def _qwen2moe_configuration(md: dict, g: GGUFFile, q: str, context_length: int) -> Configuration:
    """Qwen2MoEModelLoader.createConfiguration: qwen2moe.* keys, head_count_kv required, the vocabulary size is the token list's, the
    context is clamped to the model's, hidden_dim is 0, the expert hidden size comes from ffn_down_exps dims[0].  The shared expert's
    hidden size is taken from the ffn_gate_shexp tensor; where it differs from feed_forward_length (which the reference uses) the
    reference would read the shared expert with the wrong row count, so such a file is refused.  FP16 files load (as in the reference);
    the plan refuses them."""
    model_ctx = int(md["qwen2moe.context_length"])
    ctx = model_ctx if (context_length < 0 or model_ctx < context_length) else context_length
    n_heads = int(md["qwen2moe.attention.head_count"])
    dim = int(md["qwen2moe.embedding_length"])
    ti = g.tensor_infos
    expert_hidden = int(ti["blk.0.ffn_down_exps.weight"].dims[0])
    shared_hidden = int(ti["blk.0.ffn_gate_shexp.weight"].dims[1])
    ffl = int(md["qwen2moe.feed_forward_length"])
    if shared_hidden != ffl:
        raise UnsupportedModel(f"qwen2moe.feed_forward_length is {ffl} but the shared expert (blk.0.ffn_gate_shexp.weight) has {shared_hidden} rows: "
                               "the reference sizes the shared expert by feed_forward_length and would read the wrong bytes")
    return Configuration(
        ARCH_QWEN2_MOE, q, dim, 0, int(md["qwen2moe.block_count"]), n_heads, int(md["qwen2moe.attention.head_count_kv"]), dim // n_heads,
        len(md["tokenizer.ggml.tokens"]), ctx, float(md["qwen2moe.attention.layer_norm_rms_epsilon"]), float(md["qwen2moe.rope.freq_base"]),
        n_experts=int(md["qwen2moe.expert_count"]), n_experts_used=int(md["qwen2moe.expert_used_count"]),
        expert_hidden_dim=expert_hidden, shared_hidden_dim=shared_hidden)


def granite_configuration(md: dict, q: str, context_length: int) -> Configuration:
    """GraniteLoader.createConfiguration (GraniteLoader.java:48-92): granite.* keys; the vocabulary size is granite.vocab_size, else the
    token list's length; the four scales default to 12.0 / 0.22 / 0.0078125 / 16.0 (read as Java floats); head_count_kv is a scalar or a
    per-layer array whose first element the reference takes -- a non-uniform array is refused here, because the reference would run
    every layer with layer 0's count; eps defaults to 1e-5 and theta to 10000; the context is the requested one when >= 0
    (GraniteConfiguration.withContextLength), else the model's; head size = dim / heads; the classifier is tied."""
    n_heads = int(md["granite.attention.head_count"])
    dim = int(md["granite.embedding_length"])
    kv = md.get("granite.attention.head_count_kv", n_heads)
    if isinstance(kv, (list, tuple, np.ndarray)):
        kv = [int(v) for v in kv]
        if not kv or any(v != kv[0] for v in kv):
            raise UnsupportedModel(f"granite.attention.head_count_kv varies across layers ({kv}): the reference runs every layer with the "
                                   "first layer's count, which would compute the other layers wrongly")
        kv = kv[0]
    vocab = md.get("granite.vocab_size")
    if vocab is None:
        vocab = len(md["tokenizer.ggml.tokens"])
    model_ctx = int(md["granite.context_length"])
    f = lambda key, default: float(np.float32(md.get(key, default)))  # (float) metadata.getOrDefault(key, <float literal>)
    return Configuration(
        ARCH_GRANITE, q, dim, int(md["granite.feed_forward_length"]), int(md["granite.block_count"]), n_heads, int(kv), dim // n_heads,
        int(vocab), model_ctx if context_length < 0 else context_length, f("granite.attention.layer_norm_rms_epsilon", 1e-5),
        f("granite.rope.freq_base", 10000.0),
        embedding_scale=f("granite.embedding_scale", GRANITE_DEFAULT_SCALES["embedding_scale"]),
        residual_scale=f("granite.residual_scale", GRANITE_DEFAULT_SCALES["residual_scale"]),
        attention_scale=f("granite.attention.scale", GRANITE_DEFAULT_SCALES["attention_scale"]),
        logit_scale=f("granite.logit_scale", GRANITE_DEFAULT_SCALES["logit_scale"]))


def tensor_as_f32(model: Model, name: str) -> np.ndarray:
    """Dequantise a whole tensor the way ``FloatTensor.getFloat`` does (tests / debugging)."""
    tt, dims, raw = model.tensors[name]
    if tt == GGMLType.F32:
        return raw.view("<f4").copy()
    if tt == GGMLType.F16:
        return raw.view("<f2").astype(np.float32)
    blocks = raw.reshape(-1, 34)
    d = blocks[:, :2].copy().view("<f2").astype(np.float32)
    q = blocks[:, 2:].view(np.int8).astype(np.float32)
    return (q * d).reshape(-1)
