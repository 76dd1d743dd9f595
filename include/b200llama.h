/*
 * b200llama.h -- C ABI of libb200llama.so: the H100-native replacement for the
 * TornadoVM execution-plan layer of beehive-lab/GPULlama3.java.
 *
 * One `b200_plan` plays the role of one `TornadoVMMasterPlan` instance
 * (reference: src/main/java/org/beehive/gpullama3/tornadovm/TornadoVMMasterPlan.java:30-85).
 * It owns the device copies of the weights (repacked from GGUF block layout at
 * creation), the FP32 KV cache ([layer][ctx][kvDim], LlamaState.java:46-47,69-70) and all
 * activation buffers.  Plain pointers and sizes only; no C++/torch types.
 *
 * Threading: a plan is single-owner (one thread at a time, like the reference where the
 * server serialises on a lock, InferenceService.java:31,58).  Several plans may coexist;
 * there is no process-global state.
 *
 * Errors: every entry point returns B200_OK (0) or a negative B200_ERR_* code;
 * b200_last_error(plan) gives the message.  The Java shim maps B200_ERR_UNSUPPORTED to
 * UnsupportedOperationException (ForwardPlanFactory.java:84-87) and B200_ERR_OOM to the
 * reference's out-of-memory error (README.md:262-265).
 */
#ifndef B200LLAMA_H
#define B200LLAMA_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_OK 0
#define B200_ERR_BAD_ARG (-1)
#define B200_ERR_UNSUPPORTED (-2)
#define B200_ERR_OOM (-3)
#define B200_ERR_CUDA (-4)
#define B200_ERR_NCCL (-5)
#define B200_ERR_STATE (-6)

#define B200_ARCH_LLAMA 0 /* InferenceCore.forwardJava,      InferenceCore.java:50-172  */
#define B200_ARCH_QWEN3 1 /* InferenceCore.forwardJavaQwen3, InferenceCore.java:565-697 */
#define B200_ARCH_PHI3 2  /* InferenceCore.forwardJavaPhi3,  InferenceCore.java:699-800: fused blk.N.attn_qkv.weight ([q; k; v] rows) and
                           * blk.N.ffn_up.weight ([gate; up] rows), NeoX-pair RoPE without q/k norm; n_heads * head_size == dim */
#define B200_ARCH_QWEN2 3 /* InferenceCore.forwardJavaQwen2, InferenceCore.java:434-563 (Qwen2, Qwen2.5, DeepSeek-R1-Distill-Qwen): Llama's
                           * tensors plus F32 biases blk.N.attn_q.bias (n_heads * head_size floats), attn_k.bias and attn_v.bias
                           * (n_kv_heads * head_size each), added to q, k and v right after their matmuls; NeoX-pair RoPE without q/k
                           * norm; n_heads * head_size == dim.  Under tensor parallelism a rank reads the bias rows of its own heads. */
#define B200_ARCH_QWEN2_MOE 4 /* InferenceCore.forwardJavaQwen2MoE, InferenceCore.java:263-432 (Qwen1.5-MoE-A2.7B): Qwen2's attention (q/k/v
                               * biases, NeoX RoPE) and a mixture-of-experts FFN.  Created with b200_plan_create_moe only. */
#define B200_ARCH_GRANITE 5 /* InferenceCore.forwardGranite, InferenceCore.java:814-921 (Granite 3.x): Llama's tensors and forward with four
                             * muP scalars (b200_granite_config).  Created with b200_plan_create_granite only. */

/* GGML tensor type ids accepted for weights (tensor/GGMLType.java:5-20) */
#define B200_GGML_F32 0
#define B200_GGML_F16 1
#define B200_GGML_Q8_0 8
/* K-quants are accepted for weight matrices and the embedding table of a Q8_0 plan: they are re-quantised to Q8_0 on the device while
 * the upload pipeline streams them in, byte-identical to ModelLoader.dequantizeToQ8_0TornadoTensor (model/loader/ModelLoader.java:163,
 * 173-224); the plan then computes exactly as for a Q8_0 file (AbstractModelLoader.java:45-59). */
#define B200_GGML_Q4_K 12
#define B200_GGML_Q5_K 13
#define B200_GGML_Q6_K 14

/* Model configuration: the fields of Configuration the forward pass reads
 * (LlamaModelLoader.java:47-63, Qwen3ModelLoader.java:48-74). */
typedef struct b200_config {
    int32_t arch;           /* B200_ARCH_* */
    int32_t dim;            /* embedding_length */
    int32_t hidden_dim;     /* feed_forward_length */
    int32_t n_layers;       /* block_count */
    int32_t n_heads;        /* attention.head_count */
    int32_t n_kv_heads;     /* attention.head_count_kv */
    int32_t head_size;      /* dim/n_heads (Llama) or attention.key_length (Qwen3) */
    int32_t vocab_size;
    int32_t context_length; /* KV-cache positions to allocate (Options.maxTokens) */
    float rms_norm_eps;
    float rope_theta;
    int32_t fp16_lanes;     /* FP16 weights only: lane count of the CPU path's vector species the
                               results are pinned to (FP16FloatTensor.java:62-110, FloatTensor.java:21);
                               8, 16 or 0 (scalar).  Ignored for Q8_0. */
    int32_t tp_rank;        /* tensor-parallel rank of this process, 0 when tp_size == 1 */
    int32_t tp_size;        /* 1, 2, 4 or 8 */
} b200_config;

/* One named GGUF tensor: raw host bytes exactly as mapped from the file
 * (GGUF.loadTensorsStandard, GGUF.java:105-137).  dims[0] is the innermost dimension. */
typedef struct b200_tensor {
    const char *name; /* GGUF name, e.g. "blk.0.attn_q.weight" (LlamaModelLoader.java:78-99) */
    const void *data;
    int32_t ggml_type;
    int32_t n_dims;
    int64_t dims[4];
} b200_tensor;

/* Expert configuration of a B200_ARCH_QWEN2_MOE plan (Qwen2MoEModelLoader.createConfiguration).  b200_config.hidden_dim is unused
 * (0, as the reference's configuration has it). */
typedef struct b200_moe_config {
    int32_t n_experts;         /* expert_count (E), 1..256 */
    int32_t n_experts_used;    /* expert_used_count (k), 1..min(E, 8) */
    int32_t expert_hidden_dim; /* ffn_down_exps dims[0] (He) */
    int32_t shared_hidden_dim; /* ffn_gate_shexp dims[1] (Hs) */
} b200_moe_config;

/* The four scalars of a B200_ARCH_GRANITE plan (GraniteConfiguration).  Each is ONE float multiply, rounded once, where the CPU path
 * makes it: the embedding row (x = emb[token] * embedding_scale), every attention score (q.k * attention_scale, in place of
 * / sqrt(head_size)), both residual branches (x += (W*v) * residual_scale: Wo and W2) and the logits (logits * logit_scale, the
 * greedy argmax taken on the scaled values).  The reference MULTIPLIES by logit_scale; see DESIGN.md section 10. */
typedef struct b200_granite_config {
    float embedding_scale; /* granite.embedding_scale, default 12.0 */
    float residual_scale;  /* granite.residual_scale, default 0.22 */
    float attention_scale; /* granite.attention.scale, default 0.0078125 */
    float logit_scale;     /* granite.logit_scale, default 16.0 */
} b200_granite_config;

typedef struct b200_plan b200_plan;

/* TornadoVMMasterPlan.initializeTornadoVMPlan(state, model) (TornadoVMMasterPlan.java:55-70)
 * + forceCopyInReadOnlyData (TornadoVMMasterPlanSingleToken.java:100-117): copies/repacks every
 * tensor to `device`, allocates KV cache and activations, captures the decode CUDA graph.
 * The host pointers are not retained.  prefill_batch_size mirrors -Dllama.prefillBatchSize
 * (TornadoVMMasterPlan.java:41); 0/1 = no batched-prefill buffers.
 * On failure *out is NULL and err (if non-NULL) receives the message. */
int b200_plan_create(const b200_config *cfg, const b200_tensor *tensors, int32_t n_tensors,
                     int32_t prefill_batch_size, int32_t device, b200_plan **out, char *err, size_t err_len);

/* b200_plan_create for cfg->arch == B200_ARCH_QWEN2_MOE (b200_plan_create refuses that arch with B200_ERR_BAD_ARG, and this call
 * every other).  Per layer it requires, besides Qwen2's attention tensors and biases and the two norms (dims[0] innermost, as
 * llama.cpp writes them):
 *   blk.N.ffn_gate_inp.weight        F32 [dim, E]          the router
 *   blk.N.ffn_gate_inp_shexp.weight  F32 [dim]             the shared-expert gate
 *   blk.N.ffn_{gate,up}_exps.weight  [dim, He, E]          the routed experts, stacked [E][He][dim]
 *   blk.N.ffn_down_exps.weight       [He, dim, E]          stacked [E][dim][He]
 *   blk.N.ffn_{gate,up}_shexp.weight [dim, Hs]             the shared expert
 *   blk.N.ffn_down_shexp.weight      [Hs, dim]
 * Matrices are Q8_0 or K-quants (re-quantised to Q8_0 at upload).  Each layer's FFN runs the reference's order: F32 router dot
 * products (sequential, no FMA), softmax, top-k by first strict maximum with the probabilities as weights (no renormalisation), the k
 * routed experts' SwiGLU FFNs added to x in selection order (x[i] = w * y[i] + x[i]), then the shared expert with weight
 * 1 / (1 + exp(-g)).  B200_ERR_BAD_ARG: a missing tensor, wrong dims, n_experts_used outside 1..min(E, 8).  B200_ERR_UNSUPPORTED
 * (reason in the message): a router or shared gate that is not F32, FP16 weights, tp_size > 1, the non-streaming Q8_0 layout,
 * hidden sizes the stream layout cannot cut.  The plan decodes through the CUDA graph (not the persistent kernel), prefills through
 * the exact path only, and refuses b200_set_decode_slots (n_slots > 0) and b200_time_kernel with B200_ERR_UNSUPPORTED. */
int b200_plan_create_moe(const b200_config *cfg, const b200_moe_config *moe, const b200_tensor *tensors, int32_t n_tensors,
                         int32_t prefill_batch_size, int32_t device, b200_plan **out, char *err, size_t err_len);

/* b200_plan_create for cfg->arch == B200_ARCH_GRANITE (b200_plan_create refuses that arch with B200_ERR_BAD_ARG, and this call every
 * other).  The tensors are Llama's (tied classifier: output.weight may be absent).  A scale that is not finite fails with
 * B200_ERR_BAD_ARG and names the scale.  Every decode mode, weight format and prefill mode of a Llama plan is available. */
int b200_plan_create_granite(const b200_config *cfg, const b200_granite_config *granite, const b200_tensor *tensors, int32_t n_tensors,
                             int32_t prefill_batch_size, int32_t device, b200_plan **out, char *err, size_t err_len);

/* TornadoVMMasterPlan.tornadoVMForwardDecode(position) with the embedding gather moved
 * device-side (replaces InferenceCore.forwardTornadoVM, InferenceCore.java:956-980, which copies
 * the embedding row H2D every token).  Runs one single-token forward at `position`.
 * logits (vocab_size floats, host) may be NULL: then only 4 bytes cross PCIe.
 * argmax (host) may be NULL; otherwise receives FloatTensor.argmax semantics
 * (first strict maximum, FloatTensor.java:138-151), computed on the device. */
int b200_forward_decode(b200_plan *plan, int32_t token, int32_t position, float *logits, int32_t *argmax);

/* b200_forward_decode + Sampler.sampleToken on the DEVICE (inference/sampler/Sampler.java:74-122, CategoricalSampler.java:28-40,
 * ToppSampler.java:62-156): the reference copies the whole logits row to the host whenever temperature > 0; here 4 bytes go in
 * (the uniform number the host-side Java RNG produced for this token, in [0,1)) and 4 bytes come out.  temperature == 0 is
 * FloatTensor.argmax; otherwise logits/temperature, softmax, then categorical sampling (topp <= 0 or >= 1) or top-p.  Every
 * float is evaluated in the reference's order (csrc/sampler.cuh), so the same uniform number yields the same token id.
 * info (nullable, 4 ints): {top-p candidates after the cutoff, tokens kept, items / fallbacks of the exact softmax sum}.
 * Single-GPU plans only (B200_ERR_UNSUPPORTED under tensor parallelism). */
int b200_forward_decode_sample(b200_plan *plan, int32_t token, int32_t position, float temperature, float topp, float uniform01,
                               int32_t *token_out, int32_t *info);

/* TornadoVMMasterPlanPrefillDecode.tornadoVMForwardPrefill(position)
 * (TornadoVMMasterPlanPrefillDecode.java:116): single-token forward that only fills the KV
 * cache -- final norm, lm_head and argmax are skipped. */
int b200_forward_prefill(b200_plan *plan, int32_t token, int32_t position);

/* TornadoVMMasterPlanBatchPrefillDecode.tornadoVMForwardBatchPrefill()
 * (TornadoVMMasterPlanBatchPrefillDecode.java:107-123) with explicit arguments instead of
 * state.embeddingXBatch/batchStartPosHolder: tokens[b] is processed at start_pos+b,
 * n <= prefill_batch_size.  KV cache only, no logits (InferenceCoreBatchPrefillDecode.java:166-167).
 * In B200_PREFILL_EXACT on plans that run b200_forward_decode_multi, positions start_pos .. start_pos + n - 2 run as multi-position
 * steps of b200_decode_multi_rows rows into the plan's cache (no classifier) and the last token runs through the single-token
 * prefill graph, so the single-token buffers and step state are left as the token-by-token loop leaves them; other plans run
 * every token through that graph.  Either way the KV cache is bit-identical to the CPU path. */
int b200_forward_batch_prefill(b200_plan *plan, const int32_t *tokens, int32_t n, int32_t start_pos);

/* How b200_forward_batch_prefill computes (the reference has the same two families:
 * LlamaFP16LayersBatchPrefill vs ...BatchPrefillMMA, selected by TensorCoreSupport.java):
 *   B200_PREFILL_EXACT       multi-position steps, then the single-token prefill graph for the chunk's last token (the
 *                            graph per token on FP16, tensor-parallel, MoE and non-streaming plans): KV cache
 *                            bit-identical to the CPU path;
 *   B200_PREFILL_TENSOR_CORE TMA + wgmma GEMMs over the whole chunk, FP16 operands / FP32 accumulation:
 *                            KV cache within FP16 tolerance of the CPU path.  Default for FP16 plans created
 *                            with prefill_batch_size > 1.  Opt-in for single-GPU Q8_0 plans: the first call
 *                            dequantises f16 twins of the weight matrices on the device (+2 bytes/weight);
 *                            there the CPU path additionally rounds activations to int8, so agreement is
 *                            percent-level, not FP16-level -- hence not the default.  Returns
 *                            B200_ERR_UNSUPPORTED with the reason in b200_last_error when unavailable.
 *   B200_PREFILL_TENSOR_CORE_W8A16  the same batched prefill on a single-GPU Q8_0 plan (K-quant plans included) on the
 *                            streaming layout, with the GEMMs' B operand dequantised to f16(q * scale) in shared memory
 *                            from the tile-major Q8_0 stream the decode kernels read: no f16 twins, 1.06 instead of
 *                            2 bytes per weight streamed.  Bit-identical to B200_PREFILL_TENSOR_CORE except where a
 *                            residual GEMM splits K (the order of the f32 reduce-adds is not fixed in either mode).
 *                            The first call allocates the prefill scratch and builds tensor maps only.  Needs every
 *                            stream segment to be a multiple of 64 columns; B200_ERR_UNSUPPORTED with the reason
 *                            otherwise.  The two tensor-core modes can be switched in either order on one plan. */
#define B200_PREFILL_EXACT 0
#define B200_PREFILL_TENSOR_CORE 1
#define B200_PREFILL_TENSOR_CORE_W8A16 2
int b200_set_prefill_mode(b200_plan *plan, int32_t mode);

/* Active mode, kernels launched and device milliseconds of the last tensor-core chunk (any pointer may be NULL). */
int b200_prefill_info(b200_plan *plan, int32_t *mode, int32_t *launches, float *device_ms);

/* How the single-token forwards (b200_forward_decode / _prefill / b200_decode_sequence) run.  Both replace
 * TornadoVMMasterPlanSingleToken.tornadoVMForwardDecode's N+2 TaskGraph executions
 * (TornadoVMMasterPlanSingleToken.java:68-95) and produce bit-identical results:
 *   B200_DECODE_GRAPH       one CUDA graph of ~7 kernels per layer with programmatic-dependent-launch edges (the default:
 *                           every plan can run it; DESIGN.md section 6 has both measured);
 *   B200_DECODE_PERSISTENT  ONE persistent kernel per token (csrc/decode_persistent.cuh): one CTA per SM streams the
 *                           weights of every matrix through a shared-memory ring while epoch counters order the phases.
 *                           Available when the plan fits (Q8_0 streaming layout, head size 64/128); the environment
 *                           variable B200_DECODE=persistent selects it at creation.
 * Returns B200_ERR_UNSUPPORTED with the reason in b200_last_error when the plan cannot run the requested mode.
 * Under tensor parallelism every rank must switch at the same point of the call sequence. */
#define B200_DECODE_GRAPH 0
#define B200_DECODE_PERSISTENT 1
int b200_set_decode_mode(b200_plan *plan, int32_t mode);

/* Active decode mode, kernels per decode step, and the persistent kernel's ring depth / shared memory (0 if unsupported). */
int b200_decode_info(b200_plan *plan, int32_t *mode, int32_t *launches, int32_t *ring_stages, int32_t *smem_bytes);

/* Device-resident token loop (what LlamaBench.runTest times, LlamaBench.java:234-254, and the
 * greedy generation loop InferenceEngine.java:96-145 with the sampler on the device):
 * runs n single-token forwards at positions start_pos..start_pos+n-1 without host round trips.
 * feedback == 0: step i consumes tokens[i] (n entries).  feedback != 0: step 0 consumes
 * tokens[0], step i>0 consumes the argmax of step i-1 (greedy generation).
 * out_ids (n ints, may be NULL) receives each step's argmax.  device_ms (may be NULL)
 * receives the CUDA-event time of the n steps on the plan's stream. */
int b200_decode_sequence(b200_plan *plan, const int32_t *tokens, int32_t n, int32_t start_pos,
                         int32_t feedback, int32_t *out_ids, float *device_ms);

/* Zero the KV cache (a fresh State in the reference: Java arrays start zeroed,
 * LlamaState.java:46-47; matters because the Qwen3 loop skips a position,
 * InferenceEngine.java:175-225). */
int b200_kv_reset(b200_plan *plan);

/* ---- batched decode: up to B200_MAX_DECODE_SLOTS independent sequences per step ---------------------------------------------
 * One step streams every weight matrix from HBM once for all its rows (csrc/decode_batch.cuh); every dot product keeps its own
 * row, activation vector and block order, so each row is bit-identical to b200_forward_decode of the same token stream.  Single-GPU
 * Q8_0 plans on the streaming layout only (K-quant files included; every architecture and head size); FP16 plans, the
 * non-streaming Q8_0 layout and tensor-parallel plans get B200_ERR_UNSUPPORTED.  Batched steps always run as a multi-kernel CUDA
 * graph with programmatic-dependent-launch edges, whatever b200_set_decode_mode selected; the plan's own KV cache, step state and
 * graphs are not touched, so single-sequence calls can be interleaved with batched ones. */
#define B200_MAX_DECODE_SLOTS 8

/* Allocates n_slots zeroed KV caches ([layer][ctx][kvDim] f32 each, the plan's context_length), per-row activation buffers and,
 * lazily, one graph per row count.  0 frees them.  B200_ERR_UNSUPPORTED (the message names the maximum) when the plan cannot
 * run n_slots rows per step.  Calling it again replaces every slot with a zeroed one. */
int b200_set_decode_slots(b200_plan *plan, int32_t n_slots);

/* One forward step of n rows: row i consumes tokens[i] at positions[i] against slot slots[i]'s cache.  sampling is NULL (all rows
 * greedy: FloatTensor.argmax, first strict maximum) or n x {temperature, topp, uniform01}: a row with temperature 0 takes the argmax,
 * any other row runs b200_forward_decode_sample's sampler on its own logits.  ids_out receives n ids; logits (nullable) n x vocab_size
 * floats.  B200_ERR_BAD_ARG naming the row for: n outside [1, n_slots], a repeated slot, a slot or position out of range, a bad
 * token or sampling triple.  B200_ERR_STATE before b200_set_decode_slots. */
int b200_forward_decode_batch(b200_plan *plan, int32_t n, const int32_t *slots, const int32_t *tokens, const int32_t *positions,
                              const float *sampling /* nullable, 3n */, int32_t *ids_out, float *logits /* nullable, n x vocab */);

/* Zero one slot's K/V cache (a fresh State). */
int b200_slot_reset(b200_plan *plan, int32_t slot);

/* Copy positions [0, n_positions) of the plan's own K/V cache into the slot and zero positions [n_positions, ctx): how a prompt
 * prefilled with b200_forward_batch_prefill enters a slot.  The copy is exact after the exact prefill; after a tensor-core prefill it
 * carries that mode's FP16 tolerance.  b200_prefill_slots prefills prompts straight into their slots, several per call, without
 * the plan's own cache or this copy. */
int b200_slot_copy_kv(b200_plan *plan, int32_t slot, int32_t n_positions);

/* Prefill n_seqs prompts, each into its own decode slot: sequence i's tokens tokens[off_i .. off_i + lengths[i]) (concatenated in
 * call order) are processed at positions start_positions[i] .. start_positions[i] + lengths[i] - 1 of slot slots[i].  KV only, no
 * logits.  The mode is the plan's prefill mode (b200_set_prefill_mode):
 *   exact: the batched decode step without its final norm, lm_head and argmax.  The call's T tokens, sequence after sequence, fill
 *          ceil(T / b200_decode_multi_rows) steps, a sequence taking several consecutive positions of a step when rows are free
 *          (such steps write every row's K/V before any row attends); each slot's K/V is bit-identical to the CPU path;
 *   tensor-core modes: one chunk of all the tokens through the GEMMs, at most prefill_batch_size tokens per call; each slot's K/V is
 *          what b200_forward_batch_prefill of that prompt alone followed by b200_slot_copy_kv gives, wherever the GEMMs split K
 *          the same way (the split depends on the chunk's total length).
 * Only the named slots' rows at the named positions are written: the plan's own cache, the other slots and a named slot's rows
 * outside its range keep their bytes, so a later call may continue a slot's prompt (start_positions[i] > 0).  A length of 0 takes
 * no part.  B200_ERR_STATE without decode slots; B200_ERR_BAD_ARG (naming the sequence) for n_seqs outside 1..n_slots, a slot out
 * of range or repeated, a negative length, positions outside the KV cache, a token out of range, or more tokens than
 * prefill_batch_size in a tensor-core mode.  b200_prefill_info reports the call's launches and device milliseconds. */
int b200_prefill_slots(b200_plan *plan, int32_t n_seqs, const int32_t *slots, const int32_t *start_positions, const int32_t *lengths,
                       const int32_t *tokens);

/* Run tokens[i] at position start_pos + i, i < n, of ONE sequence in one step: slot >= 0 is a decode slot, slot == -1 the plan's own
 * cache.  ids_out[i] = greedy id (FloatTensor.argmax) after position start_pos + i; logits (nullable) n x vocab_size floats.  Every
 * row is bit-identical to b200_forward_decode of the same token at the same position over the same cache prefix; K/V is written at
 * all n positions, each before any row attends to it, so rows written past an accepted draft are rewritten by the next call before
 * they are read.  Greedy only: the verification step of draft-and-verify (speculative) decoding.  With slot == -1 the plan's
 * single-token buffers and step state are not touched.  B200_ERR_BAD_ARG (naming the row) for n outside 1..b200_decode_multi_rows,
 * a slot out of range, positions outside the KV cache or a bad token; B200_ERR_UNSUPPORTED with the reason on plans that cannot run
 * it (FP16, tensor-parallel, Qwen2-MoE, the non-streaming Q8_0 layout).  The per-row buffers are allocated on first use. */
int b200_forward_decode_multi(b200_plan *plan, int32_t slot, int32_t n, const int32_t *tokens, int32_t start_pos, int32_t *ids_out,
                              float *logits /* nullable, n x vocab */);

/* Rows per b200_forward_decode_multi step (and per step of the exact prefills): 8 at the 8B shapes; 0 where unsupported. */
int b200_decode_multi_rows(b200_plan *plan, int32_t *max_rows);

/* Decode slots, kernels of the last batched step and its device milliseconds (CUDA events around the graph); any pointer may be NULL. */
int b200_batch_info(b200_plan *plan, int32_t *n_slots, int32_t *launches_per_step, float *device_ms_last_step);

/* Test/diagnostic read-back of a named device buffer into host memory.  Names:
 * "x","xb","q","k","v","hb","logits","key_cache","value_cache","xq","xs", and "slot_key_cache" / "slot_value_cache" with
 * layer = slot * n_layers + layer.  "q" (= "qkv") is the packed q|k|v vector of the
 * last layer: its q part rotated (Qwen2: bias added, then rotated), its k and v parts as the matmul produced them, BEFORE any
 * Qwen2 bias (the KV caches hold the biased k, v).  `layer` selects the
 * layer for the KV caches (ignored otherwise).  The tensor-core prefill scratch, as the last layer of the last
 * chunk left it, rows padded to a multiple of 128: "pf_x" (f32 residual, dim wide), "pf_qkv" (f32, q + k + v wide,
 * q rotated in place (after its Qwen2 bias), k before RoPE and v, both before their Qwen2 bias), "pf_a16" (f16 bits, the FFN input), "pf_att16" (f16 bits, attention output),
 * "pf_h16" (f16 bits, SwiGLU output).  Qwen2-MoE plans: "hb", "hq", "hs" hold the virtual hidden vector of the last layer (the shared
 * expert's units, then each routed slot's, shared_hidden_dim + n_experts_used * expert_hidden_dim units), "moe_ids" (int32 [layer][k], the experts the last step selected, in
 * selection order) and "moe_weights" (f32 [layer][k + 1], their routing weights, then the shared-expert weight).
 * Copies min(bytes, buffer size). */
int b200_read_buffer(b200_plan *plan, const char *name, int32_t layer, void *dst, size_t bytes);

/* Measurement hook for bench.py's roofline line: launches ONE kernel family of the decode step
 * stand-alone, `reps` times per layer, cycling over all layers so every launch streams weights
 * that are not L2-resident, and returns the average duration of one launch (CUDA events on the
 * plan's stream).  which: 0 = fused gate/up+SwiGLU, 1 = down projection (+residual),
 * 2 = fused QKV, 3 = attention output projection (+residual), 4 = lm_head.
 * The residual stream is restored afterwards; the KV cache is not touched. */
int b200_time_kernel(b200_plan *plan, int32_t which, int32_t reps, float *avg_ms, int64_t *algorithmic_bytes);

/* ---- tensor parallelism (one process per GPU; cfg.tp_size in {2,4,8}) ----------------------------
 * Nothing like this exists in the reference (docs/GPULlama3_ROADMAP.md:21 lists multi-GPU as open).
 * Every rank holds ROWS of every matrix (its query/KV heads, its slice of the FFN and of the
 * vocabulary), so each dot product keeps the reference's summation order and the tokens stay
 * bit-identical to the single-GPU path; slices are all-gathered by the kernels themselves through
 * peer-mapped buffers.  Protocol: every rank calls b200_plan_create (with the FULL tensors; the
 * library uploads only its share), then b200_tp_handle; the 64-byte handles are exchanged by the
 * host (torch.distributed / MPI / anything), then every rank calls b200_tp_attach with the n handles
 * in rank order.  After that all ranks must issue the same forward calls with the same arguments.
 * Under TP b200_forward_decode returns the argmax only (logits must be NULL). */
int b200_tp_handle(b200_plan *plan, void *handle64);
int b200_tp_attach(b200_plan *plan, const void *handles, int32_t n);

/* Diagnostic: runs ONE decode step through a traced copy of the decode graph (same kernels, same
 * programmatic-dependent-launch edges) and returns one record per kernel launch, in launch order:
 * {kernel id, earliest CTA entry, latest dependency-wait return, latest CTA exit}, the times in
 * %globaltimer nanoseconds.  ids: 1 rmsnorm, 2 qkv, 3 rope+kv, 4 attention, 5 attn-out, 6 gate/up,
 * 7 down, 8 lm_head, 9 argmax/advance; Qwen2-MoE layers: 1 for the FFN norm, then 10 router, 11 expert gate/up, 12 expert down.
 * records holds 4*cap uint64. */
int b200_trace_decode(b200_plan *plan, int32_t token, int32_t position, uint64_t *records, int32_t cap, int32_t *n_out);

/* Diagnostic: ONE decode step through the persistent kernel with phase stamps: stamps[cta][row][k] (uint64, %globaltimer ns),
 * rows 0..n_layers-1 = layers with k = {0 layer start, 1 attn norm done, 2 QKV rows done, 3 attention gathered, 4 Wo rows done,
 * 5 x gathered, 6 ffn norm done, 7 gate/up done, 8 hidden activation gathered+staged, 9 W2 rows done, 10/11 attn norm: squares staged /
 * exact sum done, 12-15 (head CTAs) attention: QKV gathered / scores+max / softmax / output quantised}; row n_layers = lm_head
 * {0 start, 1 final norm done, 2 lm_head rows done, 3 (CTA 0) step advanced}.  cap = capacity of stamps in uint64. */
int b200_trace_persistent(b200_plan *plan, int32_t token, int32_t position, uint64_t *stamps, int64_t cap, int32_t *n_ctas, int32_t *n_rows, int32_t *n_stamps);

/* Diagnostic: SM-clock cycles of the RMSNorm kernel's phases {launch->dependency wait, load+square,
 * exact sequential sum, normalise+quantise+store} followed by {items walked, fallbacks} of the exact
 * sequential sum (csrc/seqsum2.cuh).  cycles holds 16 int64; [6..15] are set to 0. */
int b200_profile_norm(b200_plan *plan, int64_t *cycles);

/* Test hook for the exact parallel evaluation of the reference's sequential float sum (csrc/seqsum2.cuh; the RMSNorm
 * accumulator of InferenceCore.java:39-48): sums n <= 8192 non-negative host floats on the device exactly as
 * `for (i) s += t[i]` would, run by `threads` = 1024 (the RMSNorm kernel's form), 512 (the persistent decode kernel's form)
 * or 256 threads; info = {items walked, fallbacks}. */
int b200_test_seqsum2(const float *terms, int32_t n, int32_t threads, float *out, int32_t *info /* nullable */);

/* Test hook for the device-side sampler (csrc/sampler.cuh): ONE launch of k_sample as b200_forward_decode_sample issues it (same
 * grid and shared memory, a logits buffer of whole 1024-float chunks with a zero pad) on n host logits.  Returns the sampled id, the
 * diagnostics {top-p candidates, tokens kept, seqsum items, seqsum fallbacks} and the n probabilities the kernel leaves in place.
 * The index scratch starts as 0xFF bytes, so a slot the kernel did not write in this call reads as -1.  temperature must be > 0
 * (0 is the plan's argmax path, not this kernel), uniform01 in [0, 1), n >= 1; B200_ERR_BAD_ARG otherwise. */
int b200_test_sample(const float *logits, int32_t n, float temperature, float topp, float uniform01,
                     int32_t *token_out, int32_t *info /* nullable, 4 */, float *probs_out /* nullable, n */);

/* Test hook for the device-side K-quant -> Q8_0 re-quantiser the upload pipeline applies to Q4_K / Q5_K / Q6_K tensors (csrc/kquant.cuh;
 * replaces ModelLoader.dequantizeToQ8_0TornadoTensor, model/loader/ModelLoader.java:173-224): host K-quant blocks in, host GGUF Q8_0
 * blocks (34 bytes per 32 elements) out, byte-identical to the reference's.  n_elems % 256 == 0. */
int b200_requant_kquant(int32_t ggml_type, const void *src, int64_t n_elems, void *dst_q8_0);

/* Batched-prefill GEMM building block (csrc/prefill_gemm.cuh; replaces the reference's mma.sync GEMMs
 * gemmMMA / gemmMMAQKV / gemmMMAGateUp, TransformerBatchPrefillKernels.java:792-1132) exposed for
 * tests and measurement: C[m][n] (f32) = A[m][k] (f16 bits) x B[n][k]^T (f16 bits) on the Hopper tensor
 * cores (wgmma), FP32 accumulation.  Host pointers; m % 128 == n % 128 == k % 64 == 0.
 * iters > 0 additionally times `iters` back-to-back launches (device events) into *ms. */
int b200_gemm_f16(const uint16_t *a, const uint16_t *b, float *c, int32_t m, int32_t n, int32_t k, int32_t iters, float *ms /* nullable */);

/* Test hook: ONE launch of the prefill GEMM exactly as b200_forward_batch_prefill launches it (pg::gemm_launch<mode, stages>).
 *   mode 0 (F32):    c (f32 [m][n]) = a[m][k] x b[n][k]^T; rows >= m_valid are stored as 0.
 *   mode 1 (RESID):  c (f32 [m][n]) += a x b^T, K split `splits` ways, every split reduce-adding its partial product;
 *                    rows >= m_valid add 0.
 *   mode 2 (GATEUP): c (f16 bits [m][n]) = f16(silu(a x b^T) * (a x b2^T)), b = W1, b2 = W3, N tiles of 64 columns;
 *                    rows >= m_valid are not written.
 * a, b, b2: f16 bits.  c is in/out: its content is uploaded first.  stages = 4 or 6 (ring depth); m % 128 == 0, k % 64 == 0,
 * n % 128 == 0 (n % 64 == 0 for GATEUP), 1 <= m_valid <= m.  splits > 1 outside RESID, or a split left without a
 * 64-wide k-block, is rejected with B200_ERR_BAD_ARG. */
int b200_test_gemm(int32_t mode, int32_t stages, int32_t splits, int32_t m, int32_t m_valid, int32_t n, int32_t k, const uint16_t *a, const uint16_t *b,
                   const uint16_t *b2 /* GATEUP only */, void *c);

/* Test hook: ONE launch of the W8A16 prefill GEMM exactly as B200_PREFILL_TENSOR_CORE_W8A16 launches it.  As b200_test_gemm,
 * but B (and B2 = W3 for GATEUP) are GGUF Q8_0 blocks (34 bytes per 32 weights, row-major [n][k]); they are repacked into
 * the tile-major stream by the plan's upload kernel (gate/up interleaved as in the plan) and dequantised inside the GEMM
 * to f16(q * scale).  stages = 4 or 5.  K whose stream segment (smv_pick_nseg) is not a multiple of 64 columns is
 * rejected with B200_ERR_BAD_ARG, like the shapes and split counts b200_test_gemm rejects. */
int b200_test_gemm_q8(int32_t mode, int32_t stages, int32_t splits, int32_t m, int32_t m_valid, int32_t n, int32_t k, const uint16_t *a, const void *bq,
                      const void *bq2 /* GATEUP only */, void *c);

/* Test hook: the causal attention of the tensor-core prefill over one chunk of n query tokens at positions start_pos ..
 * start_pos + n - 1.  q: f32 [n][n_heads * head_size] (rotated); k, v: f32 [start_pos + n][n_kv_heads * head_size] (the KV cache
 * rows), run by k_pf_attention_mma on f16 K / V copies built by k_pf_kv_to_f16, as in the prefill.  q is placed in rows of
 * stride q + 2 * kv width whose k / v columns hold NaN; grid and shared memory are the prefill's.  out: f16 bits [out_rows][n_heads * head_size], out_rows >= n, in/out: rows >= n must come back untouched.
 * head_size 64 or 128, n_heads % n_kv_heads == 0 and n_heads / n_kv_heads <= 64 (any ratio: a CTA serves floor(64 / ratio) query
 * tokens, the remaining rows of its 64-row tile are padding). */
int b200_test_pf_attention(const float *q, const float *k, const float *v, int32_t n, int32_t start_pos, int32_t n_heads,
                           int32_t n_kv_heads, int32_t head_size, int32_t out_rows, uint16_t *out);

/* Test hook: the packed form of the same attention (k_pf_attention_mma_packed, as b200_prefill_slots runs it) over n_seqs sequences
 * at once.  Sequence i has lengths[i] >= 1 query tokens at positions start_positions[i]..; q: f32 [sum lengths][n_heads * head_size]
 * (the sequences' rows back to back); k, v: f32 [sum (start_positions[i] + lengths[i])][n_kv_heads * head_size] (each sequence's
 * rows 0 .. start + length - 1, back to back).  out: f16 bits [sum lengths][n_heads * head_size], in/out. */
int b200_test_pf_attention_packed(int32_t n_seqs, const int32_t *lengths, const int32_t *start_positions, const float *q, const float *k,
                                  const float *v, int32_t n_heads, int32_t n_kv_heads, int32_t head_size, uint16_t *out);

/* Weight upload of b200_plan_create (the counterpart of the reference's load-time metrics, ModelLoader.java:102-106 and the
 * copy-in timing of TornadoVMMasterPlanSingleToken.java:51-54): wall seconds from the first tensor to the last repack kernel,
 * seconds the host spent copying mapped/pageable bytes into the pinned double buffer, and bytes sent over PCIe (a tensor-parallel
 * rank sends only its row ranges).  The pipeline: pinned double buffer filled by several host threads -> async H2D on a copy
 * stream -> double-buffered device staging -> repack kernel on the plan's stream. */
int b200_upload_info(b200_plan *plan, double *seconds, double *host_copy_seconds, int64_t *h2d_bytes);

/* Number of kernels one decode step launches (bench.py's gpu_launches). */
int b200_launches_per_decode(b200_plan *plan);

/* Bytes of device memory held by the plan (weights + KV + activations). */
int64_t b200_device_bytes(b200_plan *plan);

/* TornadoVMMasterPlan.freeTornadoExecutionPlan() */
void b200_plan_free(b200_plan *plan);

const char *b200_last_error(b200_plan *plan);

/* Library build id, e.g. "b200llama 0.1 sm_90a". */
const char *b200_version(void);

#ifdef __cplusplus
}
#endif
#endif /* B200LLAMA_H */
