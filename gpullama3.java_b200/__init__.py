"""gpullama3.java_b200 -- H100-native replacement for the TornadoVM execution layer of
beehive-lab/GPULlama3.java: the single-token decode forward and batched prefill of
Llama/Qwen3 GGUF models (Q8_0 / FP16) as hand-written sm_90a CUDA behind a C ABI
(include/b200llama.h).  The directory name contains a dot, so import it through
``__graft_entry__.import_package()`` (registers it as ``gpullama3_java_b200``)."""
from . import chat_format, engine, gguf, llama_bench, loader, native, plan, sampler, synth, tokenizer  # noqa: F401
from .loader import load_model  # noqa: F401
from .plan import B200MasterPlan  # noqa: F401
