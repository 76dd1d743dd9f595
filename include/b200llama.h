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
#define B200_ARCH_DEVSTRAL 6 /* InferenceCore.forwardJavaDevstral, InferenceCore.java:178-261 (Devstral 2, GGUF architecture mistral3): Llama's
                              * tensors and forward with an independent head size (n_heads * head_size may differ from dim: q has that
                              * width, RoPE rotates interleaved pairs over it, Wo takes it as columns) and a RoPE table that may be
                              * YaRN-scaled (b200_yarn_config).  Created with b200_plan_create_devstral only. */
#define B200_ARCH_QWEN3_MOE 7 /* Qwen3-MoE (GGUF architecture qwen3moe: Qwen3-30B-A3B, Qwen3-Coder-30B-A3B): Qwen3's attention (q/k
                               * RMSNorm, NeoX RoPE, head size of its own) and a mixture-of-experts FFN without a shared expert, the
                               * top-k weights renormalised to sum to one.  Created with b200_plan_create_moe only, shared_hidden_dim 0. */

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
    int32_t head_size;      /* dim/n_heads (Llama) or attention.key_length (Qwen3, Devstral) */
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

/* Expert configuration of a B200_ARCH_QWEN2_MOE or B200_ARCH_QWEN3_MOE plan (Qwen2MoEModelLoader.createConfiguration).
 * b200_config.hidden_dim is unused (0, as the reference's configuration has it). */
typedef struct b200_moe_config {
    int32_t n_experts;         /* expert_count (E), 1..256 */
    int32_t n_experts_used;    /* expert_used_count (k), 1..min(E, 8) */
    int32_t expert_hidden_dim; /* ffn_down_exps dims[0] (He) */
    int32_t shared_hidden_dim; /* ffn_gate_shexp dims[1] (Hs), > 0; B200_ARCH_QWEN3_MOE: 0 (no shared expert) */
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

/* YaRN parameters of a B200_ARCH_DEVSTRAL plan's RoPE table (mistral3.rope.scaling.*, read when rope.scaling.type is "yarn";
 * DevstralModelLoader.precomputeRopeFrequencies).  The table is RoPE.precomputeFreqsCisYaRN evaluated with Java's float / double
 * boundaries: per pair i, freq = (freq_extrap / factor) * (1 - ramp_i) + freq_extrap * ramp_i, cos / sin narrowed to float, then times
 * mscale = 1 + 0.1 * log_multiplier * ln(factor) (1 when log_multiplier <= 0). */
typedef struct b200_yarn_config {
    float factor;                    /* rope.scaling.factor, > 0 */
    float beta_fast;                 /* rope.scaling.yarn_beta_fast */
    float beta_slow;                 /* rope.scaling.yarn_beta_slow */
    float log_multiplier;            /* rope.scaling.yarn_log_multiplier, default 0 */
    int32_t original_context_length; /* rope.scaling.original_context_length, > 0 */
} b200_yarn_config;

typedef struct b200_plan b200_plan;

/* TornadoVMMasterPlan.initializeTornadoVMPlan(state, model) (TornadoVMMasterPlan.java:55-70)
 * + forceCopyInReadOnlyData (TornadoVMMasterPlanSingleToken.java:100-117): copies/repacks every
 * tensor to `device`, allocates KV cache and activations, captures the decode CUDA graph.
 * The host pointers are not retained.  prefill_batch_size mirrors -Dllama.prefillBatchSize
 * (TornadoVMMasterPlan.java:41); 0/1 = no batched-prefill buffers.
 * On failure *out is NULL and err (if non-NULL) receives the message. */
int b200_plan_create(const b200_config *cfg, const b200_tensor *tensors, int32_t n_tensors,
                     int32_t prefill_batch_size, int32_t device, b200_plan **out, char *err, size_t err_len);

/* b200_plan_create for cfg->arch == B200_ARCH_QWEN2_MOE or B200_ARCH_QWEN3_MOE (b200_plan_create refuses those archs with
 * B200_ERR_BAD_ARG, and this call every other).  B200_ARCH_QWEN2_MOE:  Per layer it requires, besides Qwen2's attention tensors and biases and the two norms (dims[0] innermost, as
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
 * (reason in the message): a router or shared gate that is not F32, FP16 weights, tp_size > 1, hidden sizes the stream layout
 * cannot cut.  The plan decodes through the CUDA graph (not the persistent kernel), prefills through
 * the exact path only, and refuses b200_set_decode_slots (n_slots > 0) and b200_time_kernel with B200_ERR_UNSUPPORTED.
 *
 * B200_ARCH_QWEN3_MOE (moe->shared_hidden_dim must be 0, else B200_ERR_BAD_ARG): Qwen3's attention tensors (no biases; the F32
 * blk.N.attn_q_norm.weight and attn_k_norm.weight of head_size floats, head_size = attention.key_length, so n_heads * head_size may
 * differ from dim) and, per layer, only
 *   blk.N.ffn_gate_inp.weight        F32 [dim, E]          the router
 *   blk.N.ffn_{gate,up}_exps.weight  [dim, He, E]          the routed experts, stacked [E][He][dim]
 *   blk.N.ffn_down_exps.weight       [He, dim, E]          stacked [E][dim][He]
 * Each layer's FFN: the F32 router dot products (sequential, no FMA), softmax, top-k by first strict maximum (ties to the lower
 * index), then the renormalisation s = 0, s += p_j over the picks in selection order, w_j = p_j / s, and the k routed experts'
 * SwiGLU FFNs added to x in selection order (x[i] = w_j * y[i] + x[i]).  The refusals are those of B200_ARCH_QWEN2_MOE, naming
 * Qwen3-MoE. */
int b200_plan_create_moe(const b200_config *cfg, const b200_moe_config *moe, const b200_tensor *tensors, int32_t n_tensors,
                         int32_t prefill_batch_size, int32_t device, b200_plan **out, char *err, size_t err_len);

/* b200_plan_create for cfg->arch == B200_ARCH_GRANITE (b200_plan_create refuses that arch with B200_ERR_BAD_ARG, and this call every
 * other).  The tensors are Llama's (tied classifier: output.weight may be absent).  A scale that is not finite fails with
 * B200_ERR_BAD_ARG and names the scale.  Every decode mode, weight format and prefill mode of a Llama plan is available. */
int b200_plan_create_granite(const b200_config *cfg, const b200_granite_config *granite, const b200_tensor *tensors, int32_t n_tensors,
                             int32_t prefill_batch_size, int32_t device, b200_plan **out, char *err, size_t err_len);

/* b200_plan_create for cfg->arch == B200_ARCH_DEVSTRAL (b200_plan_create refuses that arch with B200_ERR_BAD_ARG, and this call every
 * other).  The tensors are Llama's; blk.N.attn_q.weight has n_heads * head_size rows and attn_output.weight that many columns.
 * yarn == NULL: the plain RoPE table (RoPE.precomputeFreqsCis).  A YaRN field that is not finite, factor <= 0 or
 * original_context_length <= 0 fails with B200_ERR_BAD_ARG naming the field.  Every decode mode, weight format and prefill mode of a
 * Llama plan is available; the persistent decode kernel needs dim <= 8192 (b200_set_decode_mode reports the reason otherwise). */
int b200_plan_create_devstral(const b200_config *cfg, const b200_yarn_config *yarn, const b200_tensor *tensors, int32_t n_tensors,
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
 *                            graph per token on FP16, tensor-parallel and MoE plans): KV cache
 *                            bit-identical to the CPU path;
 *   B200_PREFILL_TENSOR_CORE TMA + wgmma GEMMs over the whole chunk, FP16 operands / FP32 accumulation:
 *                            KV cache within FP16 tolerance of the CPU path.  Default for FP16 plans created
 *                            with prefill_batch_size > 1.  Opt-in for single-GPU Q8_0 plans: the first call the
 *                            plan can run dequantises f16 twins of the weight matrices on the device (+2 bytes/weight);
 *                            there the CPU path additionally rounds activations to int8, so agreement is
 *                            percent-level, not FP16-level -- hence not the default.  Returns
 *                            B200_ERR_UNSUPPORTED with the reason in b200_last_error when unavailable.
 *   B200_PREFILL_TENSOR_CORE_W8A16  the same batched prefill on a single-GPU Q8_0 plan (K-quant plans included), with the
 *                            GEMMs' B operand dequantised to f16(q * scale) in shared memory
 *                            from the tile-major Q8_0 stream the decode kernels read: no f16 twins, 1.06 instead of
 *                            2 bytes per weight streamed.  Bit-identical to B200_PREFILL_TENSOR_CORE except where a
 *                            residual GEMM splits K (the order of the f32 reduce-adds is not fixed in either mode).
 *                            The first call allocates the prefill scratch and builds tensor maps only.  Needs every
 *                            stream segment to be a multiple of 64 columns; B200_ERR_UNSUPPORTED with the reason
 *                            otherwise.  The two tensor-core modes can be switched in either order on one plan.
 *   B200_PREFILL_TENSOR_CORE_EXACT  the whole chunk (<= prefill_batch_size tokens) on a single-GPU Q8_0 plan (K-quant files
 *                            expanded to Q8_0 tiles included) through int8 tensor-core GEMMs (wgmma s8 x s8 -> s32, one per
 *                            32-column Q8_0 block) that read the tile-major Q8_0 streams in place and add each block's term
 *                            fl(isum * fl(wScale * aScale)) in the CPU path's block order; norms, RoPE / KV and attention run
 *                            the exact per-row bodies over the chunk.  KV cache bit-identical to the CPU path, as
 *                            B200_PREFILL_EXACT.  Any head size the plan decodes.  The first call allocates the chunk buffers
 *                            and builds tensor maps only.  On a plan that keeps K-quant weights resident (b200_weight_info)
 *                            each resident matrix is expanded on the device to the Q8_0 tiles a Q8_0-tile plan of the same
 *                            file holds, just before its GEMM, into one scratch the size of the largest resident matrix's Q8_0
 *                            tiles, allocated by the first call and kept until b200_plan_free; B200_ERR_OOM naming both
 *                            figures (the previous mode stays in force) when that scratch and the chunk buffers exceed the
 *                            device's free memory.  B200_ERR_UNSUPPORTED with the reason (the previous mode stays in
 *                            force) on FP16, tensor-parallel and Qwen2-MoE plans, plans created without a prefill batch size,
 *                            and plans whose dim, q or q+k+v widths or Q8_0 stream segments are not multiples of 64 columns.
 *                            Applies to b200_forward_batch_prefill and b200_prefill_slots (a resident plan has no decode
 *                            slots: its prompts go to the plan's own cache).
 *   B200_PREFILL_TENSOR_CORE_EXACT_MOE  B200_PREFILL_TENSOR_CORE_EXACT for Qwen2-MoE / Qwen3-MoE plans (K-quant files included: their
 *                            experts are Q8_0 tiles), whose tensor_core_exact stays refused.  Per layer the attention half is
 *                            tensor_core_exact's; the FFN half routes every row of the chunk on the device (each router logit one
 *                            float dot product in index order, then the decode routers' own softmax / top-k / renormalisation /
 *                            shared-gate tail), sorts the n * k assignments by expert (stable: token order within each expert),
 *                            gathers each assignment's int8 row, runs every expert's rows as one grouped int8 gate/up and one
 *                            grouped down GEMM (the int8 GEMM's block order and epilogues, B read from that expert's tile-major
 *                            Q8_0 stream in place), the shared expert's GEMMs on the token rows (Qwen2-MoE), and adds the results
 *                            in the decode's order: x = fl(fl(w_j * y_j) + x) for j in selection order, the shared expert last.
 *                            KV cache bit-identical to B200_PREFILL_EXACT; b200_score_tokens' results bit-identical to exact
 *                            mode's; the decode routing buffers (b200_read_buffer "moe_ids") are left as they were.  Needs
 *                            prefill_batch_size > 1, dim, q width and q+k+v width multiples of 64 and every Q8_0 stream segment
 *                            (attention, every expert's gate/up and down, the shared expert's) a multiple of 64 columns.  The first
 *                            call allocates the chunk buffers and encodes 4 tensor maps per expert per layer into device memory.
 *                            Dense plans refuse it with B200_ERR_UNSUPPORTED (their mode is B200_PREFILL_TENSOR_CORE_EXACT). */
#define B200_PREFILL_EXACT 0
#define B200_PREFILL_TENSOR_CORE 1
#define B200_PREFILL_TENSOR_CORE_W8A16 2
#define B200_PREFILL_TENSOR_CORE_EXACT 3
#define B200_PREFILL_TENSOR_CORE_EXACT_MOE 4
int b200_set_prefill_mode(b200_plan *plan, int32_t mode);

/* Active mode, kernels launched and device milliseconds of the last tensor-core chunk (any pointer may be NULL). */
int b200_prefill_info(b200_plan *plan, int32_t *mode, int32_t *launches, float *device_ms);

/* Score a token sequence: the model's log-probability of each row's target and its greedy id, for perplexity, log-likelihood
 * evaluation and prompt log-probabilities.  Definition (every path below gives these bits):
 *   - tokens[0..n) run at positions start_pos .. start_pos + n - 1, and their K/V go into the plan's cache exactly as
 *     b200_forward_batch_prefill writes them, so decoding continues at start_pos + n;
 *   - row i's logits l are the ones b200_forward_decode(tokens[i], start_pos + i) returns, bit for bit (Granite's logit scale
 *     included; the classifier's padding rows are never part of l);
 *   - greedy_ids[i] = the first index of the strict maximum m of l (FloatTensor.argmax, b200_forward_decode's argmax);
 *   - S = sum_j exp((double)l_j - (double)m) in double, in an order fixed by vocab_size alone (not by n, the mode or the launch);
 *   - logprobs[i] = ((double)l_t - (double)m) - log(S) for t = targets[i], NaN for targets[i] == -1.  No temperature.
 * Limits and validation are b200_forward_batch_prefill's: n <= prefill_batch_size when that is > 1, positions inside the KV cache,
 * tokens inside the vocabulary; a target other than -1 or a token id fails with B200_ERR_BAD_ARG.  The path follows the prefill
 * mode (b200_set_prefill_mode):
 *   B200_PREFILL_TENSOR_CORE_EXACT  the int8 tensor-core prefill of the chunk, then the final norm, the classifier as one int8 GEMM
 *                                   per 256 rows (expanded from the resident tiles first on a resident plan) and the per-row
 *                                   reduction.  The first call allocates a logits scratch of 256 rows and, on a resident plan whose
 *                                   classifier's Q8_0 tiles exceed the prefill's expansion scratch, grows that scratch; B200_ERR_OOM
 *                                   naming the bytes when they exceed the device's free memory;
 *   B200_PREFILL_EXACT              on plans that run b200_forward_decode_multi: multi-position steps with the classifier on every row;
 *                                   on every other single-GPU plan (FP16, Qwen2-MoE, resident): the single-token decode graph per
 *                                   position.  n <= context_length + 8.
 * B200_ERR_UNSUPPORTED with the reason on tensor-parallel plans (full logits are not gathered) and in the tensor_core and
 * tensor_core_w8a16 modes (their f16 activations do not give the reference's logits: use exact or tensor_core_exact).  A refused
 * or failed call leaves the plan able to decode. */
int b200_score_tokens(b200_plan *plan, const int32_t *tokens, const int32_t *targets, int32_t n, int32_t start_pos, double *logprobs,
                      int32_t *greedy_ids);

/* Log-probabilities of generated tokens: each emitted id's log-probability and its top-N alternatives, computed on the device, for
 * OpenAI-style logprobs / top_logprobs, confidence filtering and evaluation harnesses that record completion likelihoods.
 * b200_set_logprobs(plan, top_n): -1 turns them off (the default), 0..B200_MAX_TOP_LOGPROBS turns them on with top_n alternatives per
 * row.  While on, each call that emits ids fills the plan's result table with its rows, and b200_read_logprobs reads it:
 *   b200_forward_decode, b200_forward_decode_sample      one row;
 *   b200_decode_sequence                                  n rows, one per step;
 *   b200_forward_decode_batch, _multi, b200_forward_step  n rows in the call's row order.
 * Every other call leaves the table alone; b200_set_logprobs empties it.  Definition, for an emitting row whose logits l[0, vocab) are
 * exactly the row the call returns through its `logits` argument and whose id c is exactly the id it returns (the argmax or the
 * sampler's id):
 *   - m and S are b200_score_tokens' (its sum order, fixed by vocab_size alone);
 *   - chosen = ((double)l_c - m) - log(S): bit-equal to b200_score_tokens' logprob of target c at the same position over the same
 *     cache prefix;
 *   - t_k, k = 1..top_n: the first index of the strict maximum among the entries not yet taken; when no remaining entry is > -inf
 *     (NaN rows included), the lowest index not yet taken.  t_1 is the greedy id.  top_logprob_k = ((double)l_{t_k} - m) - log(S);
 *   - the raw logits' values: temperature 1, no top-p truncation, Granite's logit scale included, so a sampled token's value is the
 *     model's probability, not the sampler's; the classifier's padding rows never appear;
 *   - rows of b200_forward_step with emit == 0: chosen NaN, ids -1, logprobs NaN.
 * The kernel (k_token_logprobs, one block per row) runs on the plan's stream after the call's graph and is never part of a graph:
 * b200_decode_info's and b200_batch_info's launch counts and b200_batch_info's device time are unchanged, while
 * b200_decode_sequence's device_ms includes the one launch per step.  Sampled rows are copied before the sampler turns them into
 * probabilities; the sampler reads the copy, so the ids equal those with logprobs off for the same uniform numbers.  The results
 * reach pinned host memory inside the call's own synchronise.  The table holds max(the plan's sequence capacity, prefill_batch_size,
 * 8) rows.  b200_forward_chunk fills one row per call row, as b200_forward_step does.
 * B200_ERR_BAD_ARG for top_n outside -1..20 or above vocab_size; B200_ERR_UNSUPPORTED on tensor-parallel plans (full logits are
 * not gathered). */
#define B200_MAX_TOP_LOGPROBS 20
int b200_set_logprobs(b200_plan *plan, int32_t top_n);
/* The last emitting call's table: *n_rows rows; chosen[i], top_ids[i * top_n + k] and top_logprobs[i * top_n + k] (any of the
 * three may be NULL; with all three NULL only *n_rows is set).  B200_ERR_STATE while logprobs are off; B200_ERR_BAD_ARG if the table
 * has more than max_rows rows. */
int b200_read_logprobs(b200_plan *plan, int32_t max_rows, int32_t *n_rows, double *chosen, int32_t *top_ids /* max_rows x top_n */,
                       double *top_logprobs /* max_rows x top_n */);
/* Test and measurement hook (no plan): k_token_logprobs on one host row logits[0, vocab) with emitted id chosen_id, run reps times on
 * the default stream after one warm-up; *avg_ms = the CUDA-event time per launch (any output may be NULL). */
int b200_test_logprobs(const float *logits, int32_t vocab, int32_t chosen_id, int32_t top_n, int32_t reps, double *chosen, int32_t *top_ids,
                       double *top_logprobs, float *avg_ms);

/* ---- sampling controls: logit bias, repetition / frequency / presence penalties, top-k and min-p, per sequence ------------------
 * A sequence is a decode slot, or slot -1 for the plan's own cache.  For an emitting row of a sequence with controls, l[0, vocab)
 * the raw logits of the step (Granite's logit scale included) and cnt[i] the sequence's count of token i, the row is modified in
 * float32, every operation rounded once (csrc/sampler.cuh, k_sample_ctl):
 *   1. logit bias: l[i] = fl(l[i] + b) for each (i, b) of the bias list;
 *   2. where cnt[i] > 0 (llama.cpp's penalties): l[i] = l[i] <= 0 ? fl(l[i] * rep) : fl(l[i] / rep), then
 *      l[i] = fl(l[i] - fl(fl((float)cnt[i] * freq) + pres));
 *   3. both masks on the row of step 2, applied together, masked entries -inf: top-k keeps l[i] >= v_k, v_k the top_k-th largest
 *      value counting repeats, and EVERY token tied at v_k (more than top_k can survive; llama.cpp keeps the first in sort order
 *      instead); min-p keeps l[i] >= fl(m + (float)log((double)min_p)), m the row maximum (llama.cpp's min-p in logit space, before
 *      temperature).  The maximum passes both, so no row is empty;
 *   4. temperature 0: the first strict maximum; otherwise b200_forward_decode_sample's sampler, unchanged, on the modified row.  A
 *      -inf entry has probability 0, so it never passes the top-p cutoff and the categorical walk never stops on it, with the
 *      reference's two fallbacks as the only exception: when the float cdf ends at or below the uniform number, or no probability
 *      reaches the top-p cutoff, the sampler returns vocab_size - 1, masked or not (CategoricalSampler.java:28-40,
 *      ToppSampler.java:71-77);
 *   5. the emitted id's count is incremented on the device.
 * Neutral values (top_k 0, min_p 0, rep 1, freq 0, pres 0, no bias) give exactly the ids of a sequence without controls.  The
 * controls apply on the calls whose ids are generated tokens: b200_forward_decode_sample (slot -1), b200_forward_decode_batch with
 * non-NULL sampling, and the emitting rows of b200_forward_step.  Every other call (b200_forward_decode, the batch without sampling,
 * b200_decode_sequence, b200_forward_decode_multi, b200_score_tokens, the prefills) neither reads nor changes them.  The logits
 * outputs and the log-probabilities stay those of the raw logits.  b200_forward_step refuses (B200_ERR_BAD_ARG, naming the row) two
 * emitting rows of one slot with controls: the second row's counts would depend on the first row's id.  Rows of sequences without
 * controls run exactly as before. */
#define B200_MAX_LOGIT_BIAS 1024
typedef struct b200_sampling_controls {
    int32_t top_k;      /* 0 = off; 1..vocab_size */
    float min_p;        /* [0, 1]; 0 = off */
    float repetition_penalty, frequency_penalty, presence_penalty; /* rep finite > 0 (1 = off); freq, pres finite (0 = off) */
    int32_t n_bias;     /* 0..B200_MAX_LOGIT_BIAS entries of distinct ids in [0, vocab_size) and finite values */
    const int32_t *bias_ids;
    const float *bias_values;
} b200_sampling_controls;
/* Set (c non-NULL, copied) or turn off (c NULL) the controls of one sequence; they stay until replaced, through b200_slot_reset,
 * b200_kv_reset and b200_set_decode_slots.  The first call that sets controls allocates the count tables, one vocab_size-int32 row
 * for slot -1 and for each of B200_MAX_DECODE_SLOTS slots, and the modified-row scratch; plans that never set controls hold none of
 * it.  Slot -1 works on every single-GPU plan (Q8_0, FP16, Qwen2-MoE, resident K-quant).  B200_ERR_BAD_ARG naming the field for a
 * slot or value out of range; B200_ERR_UNSUPPORTED on tensor-parallel plans (the sampler needs the whole row on one GPU). */
int b200_set_sampling_controls(b200_plan *plan, int32_t slot, const b200_sampling_controls *c);
/* Replace one sequence's counts with those of tokens[0, n) (how a caller counts the prompt, which is not counted otherwise).
 * b200_slot_reset clears its slot's counts, b200_kv_reset slot -1's and b200_set_decode_slots every slot's.  B200_ERR_STATE before
 * the first b200_set_sampling_controls that set controls; B200_ERR_BAD_ARG for a slot or token out of range. */
int b200_set_sample_history(b200_plan *plan, int32_t slot, const int32_t *tokens, int32_t n);
/* One sequence's counts, vocab_size int32 into counts.  B200_ERR_STATE before the count tables exist. */
int b200_read_sample_counts(b200_plan *plan, int32_t slot, int32_t *counts);
/* Test hook (no plan): ONE launch of k_sample_ctl as the plans issue it, on n host logits, the host counts (in/out: the emitted id's
 * is incremented) and controls c (validated as b200_set_sampling_controls does).  temperature 0 is allowed.  Returns the id, the
 * sampler's four diagnostics (zeros at temperature 0) and, in row_out (nullable, n floats), the modified row before the choice. */
int b200_test_sample_controls(const float *logits, int32_t n, int32_t *counts, const b200_sampling_controls *c, float temperature, float topp,
                              float uniform01, int32_t *token_out, int32_t *info, float *row_out);
/* Measurement hook (no plan): CUDA-event time per launch of k_sample_ctl under controls c and of k_sample_rows on one row (b200_test_sample's launch)
 * on the same host row, reps launches of each after one warm-up, each launch on its own copy of the row and counts.  temperature
 * must be > 0 (the plain sampler's range). */
int b200_time_sample_controls(const float *logits, int32_t n, const int32_t *counts, const b200_sampling_controls *c, float temperature, float topp,
                              float uniform01, int32_t reps, float *ctl_ms, float *plain_ms);

/* How the single-token forwards (b200_forward_decode / _prefill / b200_decode_sequence) run.  Both replace
 * TornadoVMMasterPlanSingleToken.tornadoVMForwardDecode's N+2 TaskGraph executions
 * (TornadoVMMasterPlanSingleToken.java:68-95) and produce bit-identical results:
 *   B200_DECODE_GRAPH       one CUDA graph of ~7 kernels per layer with programmatic-dependent-launch edges (the default:
 *                           every plan can run it; DESIGN.md section 6 has both measured);
 *   B200_DECODE_PERSISTENT  ONE persistent kernel per token (csrc/decode_persistent.cuh): one CTA per SM streams the
 *                           weights of every matrix through a shared-memory ring while epoch counters order the phases.
 *                           Available when the plan fits (Q8_0 weights, head size 64/128); the environment
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
 * Q8_0 plans only (K-quant files included; every architecture and head size); FP16 plans and tensor-parallel plans get
 * B200_ERR_UNSUPPORTED.  Batched steps always run as a multi-kernel CUDA
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
 * it (FP16, tensor-parallel, Qwen2-MoE).  The per-row buffers are allocated on first use. */
int b200_forward_decode_multi(b200_plan *plan, int32_t slot, int32_t n, const int32_t *tokens, int32_t start_pos, int32_t *ids_out,
                              float *logits /* nullable, n x vocab */);

/* Rows per b200_forward_decode_multi step (and per step of the exact prefills): 8 at the 8B shapes; 0 where unsupported. */
int b200_decode_multi_rows(b200_plan *plan, int32_t *max_rows);

/* One row of a mixed step (b200_forward_step). */
typedef struct b200_step_row {
    int32_t slot, token, position;
    int32_t emit;                        /* 0: K/V only (a prompt position); 1: this row's next token is wanted */
    float temperature, topp, uniform01;  /* emit rows only: b200_forward_decode_sample's triple; temperature 0 = FloatTensor.argmax */
} b200_step_row;

/* One mixed step of n rows over the decode slots: decode rows of running sequences and prompt rows of newly admitted ones share
 * one weight stream.  Row i consumes rows[i].token at rows[i].position of slot rows[i].slot; a slot may appear in several rows (at
 * distinct positions).  Every row writes its K/V at (slot, position) before any row of the step attends, so each emitting row's
 * logits are bit-identical to b200_forward_decode of the same token at the same position over the same slot prefix, and its id is
 * that call's argmax (temperature 0) or b200_forward_decode_sample's id for the same triple.  ids_out receives n ids, -1 where emit
 * is 0; logits (nullable) n x vocab_size floats, rows with emit 0 not written.  The final norm, lm_head and argmax run over the
 * emitting rows only, and all sampled rows in one sampler launch.  The plan's own cache, its single-token buffers and the slots
 * not named are not touched.  B200_ERR_UNSUPPORTED with the reason on plans that cannot run it (FP16, tensor-parallel,
 * Qwen2-MoE); B200_ERR_STATE before b200_set_decode_slots; B200_ERR_BAD_ARG naming the row for: n outside
 * 1..b200_decode_multi_rows, a slot, token or position out of range, the same (slot, position) twice, an emit flag other than 0 / 1,
 * or a bad sampling triple on an emitting row. */
int b200_forward_step(b200_plan *plan, int32_t n, const b200_step_row *rows, int32_t *ids_out /* n; -1 where emit == 0 */,
                      float *logits /* nullable, n x vocab; rows with emit == 0 are not written */);

/* b200_forward_step on the tensor cores: the same rows and outputs, run as one chunk of the bit-exact int8 prefill
 * (B200_PREFILL_TENSOR_CORE_EXACT), so prompt rows of newly admitted sequences and decode rows of running ones share the chunk's
 * GEMMs.  Up to prefill_batch_size rows (b200_chunk_rows), at most B200_MAX_DECODE_SLOTS of them emitting; any mix of slots, a slot
 * at several distinct positions.  The chunk runs the emitting rows first; their final residual rows then go through the batched
 * step's classifier (final norm, Q8_0 lm_head stream, argmax), so each emitting row's logits are bit-identical to
 * b200_forward_decode of that token at that position over the same slot prefix, whatever the chunk's length or the row's place in
 * it, and its id, sampling controls, log-probabilities (one row per call row) and counts are b200_forward_step's.  Only the named
 * (slot, position) K/V rows are written; the plan's own cache, its single-token buffers and the other slots are not touched.
 * b200_batch_info reports the call (its launches, and CUDA events around the chunk and the classifier); b200_prefill_info is left
 * alone.  One synchronise per call.
 * B200_ERR_UNSUPPORTED with the reason on plans that cannot run it (FP16, tensor-parallel, Qwen2-MoE, resident K-quant, created
 * without a prefill batch size, or a shape the int8 prefill refuses); B200_ERR_STATE without decode slots or when the prefill mode
 * is not tensor_core_exact (the message names the mode); B200_ERR_BAD_ARG naming the row for: n outside 1..prefill_batch_size,
 * more emitting rows than b200_decode_multi_rows, and every refusal of b200_forward_step's rows. */
int b200_forward_chunk(b200_plan *plan, int32_t n, const b200_step_row *rows, int32_t *ids_out /* n; -1 where emit == 0 */,
                       float *logits /* nullable, n x vocab; rows with emit == 0 are not written */);
/* Rows per b200_forward_chunk call: prefill_batch_size when the call can run (tensor_core_exact and decode slots), else 0. */
int b200_chunk_rows(b200_plan *plan, int32_t *max_rows);

/* Decode slots, kernels of the last batched step with a classifier (b200_forward_decode_batch, b200_forward_decode_multi,
 * b200_forward_step or b200_forward_chunk, whichever ran last) and its device milliseconds (CUDA events around the graph, or around
 * the chunk and its classifier); any pointer may be NULL. */
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
 * selection order) and "moe_weights" (f32 [layer][k + 1], their routing weights, then the shared-expert weight).  Qwen3-MoE plans: the
 * same without the shared expert: n_experts_used * expert_hidden_dim units, and "moe_weights" is f32 [layer][k], the renormalised weights.
 * "moe_chunk_ids" (int32 [rows][k]) and "moe_chunk_weights" (f32 [rows][k], + 1 with a shared expert) of layer `layer`: the routing of
 * every row of the last B200_PREFILL_TENSOR_CORE_EXACT_MOE chunk (B200_ERR_STATE before the mode's buffers exist).
 * "rope_cr" / "rope_ci": the RoPE table every decode and prefill kernel reads (f32 [context_length][head_size / 2]).
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
 * accumulator of InferenceCore.java:39-48): sums n <= 16384 non-negative host floats on the device exactly as
 * `for (i) s += t[i]` would, run by `threads` = 1024 (the RMSNorm kernel's form), 512 (the persistent decode kernel's form)
 * or 256 threads; info = {items walked, fallbacks}. */
int b200_test_seqsum2(const float *terms, int32_t n, int32_t threads, float *out, int32_t *info /* nullable */);

/* Diagnostic: SM-clock cycles of the same exact sum in the fused norm's chunk layout, called twice in one launch of `threads`
 * = 1024, 512 or 256 threads: cycles[0] on a cold instruction cache, cycles[1] warm, cycles[2..4] = {items walked, literal
 * items, fallbacks} of the second call (cycles holds 5 int64); out[0..1] = the two sums. */
int b200_profile_seqsum2(const float *terms, int32_t n, int32_t threads, int64_t *cycles, float *out);

/* Test hook for the device-side sampler (csrc/sampler.cuh): ONE one-row launch of k_sample_rows as b200_forward_decode_sample issues it
 * (same block and shared memory, a logits buffer of whole 1024-float chunks with a zero pad) on n host logits.  Returns the sampled id, the
 * diagnostics {top-p candidates, tokens kept, seqsum items, seqsum fallbacks} and the n probabilities the kernel leaves in place.
 * The index scratch starts as 0xFF bytes, so a slot the kernel did not write in this call reads as -1.  temperature must be > 0
 * (0 is the plan's argmax path, not this kernel), uniform01 in [0, 1), n >= 1; B200_ERR_BAD_ARG otherwise. */
int b200_test_sample(const float *logits, int32_t n, float temperature, float topp, float uniform01,
                     int32_t *token_out, int32_t *info /* nullable, 4 */, float *probs_out /* nullable, n */);

/* Test hook for the device-side K-quant -> Q8_0 re-quantiser the upload pipeline applies to Q4_K / Q5_K / Q6_K tensors (csrc/kquant.cuh;
 * replaces ModelLoader.dequantizeToQ8_0TornadoTensor, model/loader/ModelLoader.java:173-224): host K-quant blocks in, host GGUF Q8_0
 * blocks (34 bytes per 32 elements) out, byte-identical to the reference's.  n_elems % 256 == 0. */
int b200_requant_kquant(int32_t ggml_type, const void *src, int64_t n_elems, void *dst_q8_0);

/* Test hook for the expansion B200_PREFILL_TENSOR_CORE_EXACT runs on a resident plan (k_kq_tiles_to_q8, csrc/stream_matvec.cuh):
 * kq_rows, `rows` row-major rows of cols / 256 K-quant super-blocks (ggml_type 12 / 13 / 14), are repacked into resident tiles by
 * the upload's kernel, expanded on the device, and the matrix's tile-major Q8_0 stream is copied to q8_tiles_out: `bytes` bytes,
 * exactly the stream's size (4-row groups x segments x units, the layout of csrc/stream_matvec.cuh).  Each Q8_0 block is the one
 * b200_requant_kquant gives.  B200_ERR_BAD_ARG on a null pointer, rows < 1, cols not a positive multiple of 256, an unknown
 * type or a wrong `bytes`. */
int b200_test_kq_tiles_to_q8(int32_t ggml_type, int32_t rows, int32_t cols, const void *kq_rows, void *q8_tiles_out, int64_t bytes);

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

/* Test hook: ONE launch of the int8 GEMM of B200_PREFILL_TENSOR_CORE_EXACT exactly as the prefill launches it, on m activation
 * rows (any m >= 1; padded to whole 128-row tiles with rows that must never be stored).  aq: int8 [m][k]; as: their f32 block
 * scales [m][k / 32]; bq (and bq2 = the up projection for GATEUP): GGUF Q8_0 blocks [n][k / 32 * 34], repacked into the
 * tile-major stream by the plan's upload kernel.  mode 0 (STORE): c = f32 [m][n] out; 1 (RESID): c[i][j] = fl(c + fl(acc * oscale))
 * in/out; n a multiple of 64.  2 (GATEUP): n hidden units (a multiple of 32), hq = int8 [m][n] and hs = f32 [m][n / 32], the
 * Q8_0 quantisation of swiglu(gate, up), in/out.  K whose stream segment is not a multiple of 64 columns: B200_ERR_BAD_ARG. */
int b200_test_gemm_i8(int32_t mode, int32_t m, int32_t n, int32_t k, const int8_t *aq, const float *as, const void *bq, const void *bq2, float oscale,
                      float *c, int8_t *hq, float *hs);

/* Test hook: ONE launch of the grouped expert GEMM of B200_PREFILL_TENSOR_CORE_EXACT_MOE exactly as the prefill launches it.
 * n_experts experts; counts[e] >= 0 grouped rows of expert e, expert after expert (m = sum of counts).  aq: int8 [m][k]; as: f32
 * [m][k / 32]; bq (and bq2 = the up projections for GATEUP): each expert's GGUF Q8_0 blocks, [n_experts][n][k / 32 * 34], repacked
 * into one tile-major stream per expert by the plan's upload kernel, with one tensor map pair per expert in device memory; the
 * tile table is the one the prefill's grouping kernel writes for these counts.  mode 0 (STORE): c = f32 [m][n] out, n a multiple
 * of 64; 2 (GATEUP): n hidden units (a multiple of 32), hq = int8 [m][n], hs = f32 [m][n / 32] in/out.  B200_ERR_BAD_ARG for any
 * other mode, a negative count, more than 256 experts, or K whose stream segment is not a multiple of 64 columns. */
int b200_test_gemm_i8_experts(int32_t mode, int32_t n_experts, const int32_t *counts, int32_t n, int32_t k, const int8_t *aq, const float *as,
                              const void *bq, const void *bq2, float *c, int8_t *hq, float *hs);

/* One decode weight stream launched on its own (b200_test_stream).  Arrays are indexed [launch][row][...]; V = max(nrow, 1). */
typedef struct b200_stream_test {
    int32_t form;      /* B200_GGML_Q8_0 (Q8_0 tiles), B200_GGML_Q4_K / Q5_K / Q6_K (resident tiles) or B200_GGML_F16 (row-major rings) */
    int32_t mode;      /* 0 STORE, 1 RESID, 2 GATEUP */
    int32_t norm;      /* 1: the fused-RMSNorm kernel (STORE or GATEUP, Q8_0 or resident tiles, cols <= 5120) */
    int32_t nrow;      /* 0: the single-row stream; 1..8: the batched Q8_0 stream over nrow activation rows */
    int32_t lanes;     /* F16: 16 or 8 */
    int32_t rows;      /* output rows; GATEUP: hidden units (the gate and the up matrix have `rows` rows each) */
    int32_t cols;
    int32_t grid;      /* CTAs; 0: what the plan launches */
    int32_t stages;    /* ring stages, turned into the budget that yields them (F16: SfArgs::stages); 0: from `budget` */
    int64_t budget;    /* Q8_0 / resident ring budget in bytes; 0: the plan's (96 KB single-row, 112 KB batched, sf_layout for F16) */
    int32_t argmax;    /* STORE: per-CTA argmax partials, then the plan's merge (k_argmax_advance / k_argmax_batch) into ids */
    int32_t launches;  /* 1 or 2: the second launch reuses every buffer (blk_cnt too) with the second set of activations */
    int32_t pair;      /* GATEUP, single row: then a RESID stream of w_down [down_rows][rows] reading its hq / hs, both under PDL */
    int32_t down_rows;
    int32_t from_emb;  /* norm: the activation is row tokens[launch] of emb (GGUF Q8_0, emb_rows x cols) times emb_scale */
    int32_t emb_rows;
    int32_t dry;       /* 1: return after the checks with info filled in; makes no CUDA call (grid must be given) */
    float oscale, eps, emb_scale;
    const void *w;        /* GGUF Q8_0 rows, raw K-quant rows or f16 rows [rows][cols]; GATEUP: the gate matrix */
    const void *w_up;     /* GATEUP: the up matrix, same format */
    const void *w_down;   /* pair: [down_rows][rows], same format */
    const int8_t *xq;     /* Q8_0 / resident without norm: the quantised activation [launches][V][cols] ... */
    const float *xs;      /* ... and its block scales [launches][V][cols / 32] */
    const float *x;       /* norm (without from_emb) and F16: the activation [launches][cols] */
    const float *norm_w;  /* norm: [cols] */
    const void *emb;
    const int32_t *tokens;   /* from_emb: [launches] */
    const float *out_init;   /* RESID: the initial out [V][rows]; pair: the initial residual [down_rows] */
    float *out;              /* out: [launches][V][rows] after each launch (GATEUP: the float hidden values) */
    int8_t *hq;              /* GATEUP out: [launches][V][rows] ... */
    float *hs;               /* ... and [launches][V][rows / 32] */
    float *out_down;         /* pair out: the residual after each launch [launches][down_rows] */
    float *x_out;            /* from_emb out: CTA 0's write of x [launches][cols] */
    int32_t *ids;            /* argmax out: [launches][V] */
    int64_t info[5];         /* out: ring stages, grid, largest and smallest 4-row groups (F16: row groups) per CTA, dynamic shared memory */
} b200_stream_test;

/* Test hook: the decode weight stream of `form` launched as the plan launches it (upload repack, layout, kernel, shared-memory
 * attribute), but at any grid and ring depth the caller asks for.  B200_ERR_BAD_ARG, before any CUDA call, for what the plan would
 * never launch: a width that is not whole segments of the form, stages outside 3..SMV_MAX_STAGES (F16: SF_MAX_STAGES), a GATEUP whose
 * largest CTA slice exceeds the epilogue buffer at that grid, a fused norm with RESID or cols > 5120, nrow > 8 or a batch on a
 * resident or F16 form; and, once the device is known, a ring above its opt-in shared-memory limit.  B200_ERR_STATE when a store
 * reached the guard words past `out` (a padding row of a ragged STORE). */
int b200_test_stream(b200_stream_test *t);

/* The exact attention forms of b200_test_attention. */
enum {
    B200_ATT_SINGLE = 0,      /* k_attention: the decode graph (one row) */
    B200_ATT_BATCH = 1,       /* k_attention_batch: a batched step over distinct slots (rows 1..8) */
    B200_ATT_CACHED_ROWS = 2, /* k_rope_kv_batch + k_attention_cached_rows: multi-position steps, the exact multi-slot prefill (rows 1..8) */
    B200_ATT_CHUNK = 3,       /* k_i8_rope_kv + k_i8_attention: the bit-exact tensor-core prefill (any rows, att_tokens rows per launch) */
    B200_ATT_PERSISTENT = 4   /* pd_attention_head, the persistent decode kernel's copy of the body (one row, head size 64 or 128) */
};

/* One exact attention launched on its own (b200_test_attention).  One layer; row r is (slot[r], pos[r]).  The caches hold
 * `slots` slots of [ctx][n_kv_heads * head_size] floats each. */
typedef struct b200_attention_test {
    int32_t form;          /* B200_ATT_* */
    int32_t head_size;     /* 32, 64, 96, 128 or 256 (persistent: 64 or 128) */
    int32_t n_heads, n_kv_heads;
    int32_t arch;          /* KF_* flags: 1 NeoX rotation, 2 Qwen3 q/k RMSNorm, 4 Qwen2 q|k|v bias, 8 Granite's attention scale */
    int32_t ctx;           /* context length: picks shared or global score rows as the plan does (3 * head_size + ctx > 4096: global) */
    int32_t rows;          /* single / persistent: 1; batch / cached rows: 1..8; chunk: any >= 1 */
    int32_t slots;         /* cache slots (>= 1) */
    int32_t att_tokens;    /* chunk: rows per attention launch, 1..rows (the plan's rule for its scratch bound); other forms: 0 */
    int32_t dry;           /* 1: return after the checks with info filled in; makes no CUDA call */
    float eps;             /* the q/k RMSNorm's epsilon */
    float score_arg;       /* sqrt(head_size) (scores are divided by it), or with arch & 8 Granite's attention multiplier */
    const int32_t *slot;   /* [rows] */
    const int32_t *pos;    /* [rows], each < ctx */
    const float *qkv;      /* [rows][q | k | v width]: unrotated, without bias */
    const float *k_cache;  /* [slots][ctx][kv width] before the launch */
    const float *v_cache;
    const float *rope_cr;  /* [ctx][head_size / 2] */
    const float *rope_ci;
    const float *q_norm;   /* arch & 2: [head_size] */
    const float *k_norm;
    const float *qkv_bias; /* arch & 4: [q | k | v width] */
    float *qkv_out;        /* out: the qkv rows after the launch (rotated q written back) */
    float *k_out;          /* out: both caches after the launch */
    float *v_out;
    int8_t *xq;            /* out: each row's attention output quantised to Q8_0, [rows][q width] ... */
    float *xs;             /* ... and its block scales [rows][q width / 32] */
    float *xb;             /* single form, nullable: the float output [q width] (an FP16 plan's form) */
    int64_t info[5];       /* out: grid x (heads), grid y (rows per attention launch), dynamic shared memory, score rows in global
                              memory (0 / 1), attention launches */
} b200_attention_test;

/* Test hook: one exact attention form launched as the plan launches it (grid, dynamic shared memory and its attribute, score-row
 * scratch rule and indexing).  B200_ERR_BAD_ARG, before any CUDA call, for what the plan would never launch or what could read out
 * of bounds: a head size without a kernel of that form, n_heads % n_kv_heads != 0, a position outside 0..ctx-1, a slot outside
 * the caches, rows outside the form's range, att_tokens outside 1..rows, two batch rows on one slot or two rows of a slot at one
 * position.  B200_ERR_STATE when the launch wrote past the end of an output. */
int b200_test_attention(b200_attention_test *t);

/* Test hook: the two exp expressions of the bit-exact paths on the device, for the n float bit patterns first, first + 1, ...:
 * e[i] = (float)exp((double)x) (softmaxes, routers, the shared-expert gate) and e1[i] = (float)(1.0 + exp((double)x)) (the SwiGLU
 * denominator), computed as the kernels compute them.  Host arrays of n floats; first + n - 1 must not wrap. */
int b200_test_exp(uint32_t first, int64_t n, float *e, float *e1);

/* Test hook: the causal attention of the tensor-core prefill (k_pf_attention_mma_packed, on f16 K / V copies built by
 * k_pf_kv_to_f16_packed, as a chunk runs it) over n_seqs sequences at once.  Sequence i has lengths[i] >= 1 query tokens at positions
 * start_positions[i]..; q: f32 [sum lengths][n_heads * head_size] (rotated; the sequences' rows back to back, placed in rows of
 * stride q + 2 * kv width whose k / v columns hold NaN); k, v: f32 [sum (start_positions[i] + lengths[i])][n_kv_heads * head_size]
 * (each sequence's KV cache rows 0 .. start + length - 1, back to back); grid and shared memory are the prefill's.  out: f16 bits
 * [out_rows][n_heads * head_size], out_rows >= sum lengths, in/out: rows >= sum lengths must come back untouched.  head_size 64 or
 * 128, n_heads % n_kv_heads == 0 and n_heads / n_kv_heads <= 64 (any ratio: a CTA serves floor(64 / ratio) query tokens, the
 * remaining rows of its 64-row tile are padding). */
int b200_test_pf_attention_packed(int32_t n_seqs, const int32_t *lengths, const int32_t *start_positions, const float *q, const float *k,
                                  const float *v, int32_t n_heads, int32_t n_kv_heads, int32_t head_size, int32_t out_rows, uint16_t *out);

/* Weight upload of b200_plan_create (the counterpart of the reference's load-time metrics, ModelLoader.java:102-106 and the
 * copy-in timing of TornadoVMMasterPlanSingleToken.java:51-54): wall seconds from the first tensor to the last repack kernel,
 * seconds the host spent copying mapped/pageable bytes into the pinned double buffer, and bytes sent over PCIe (a tensor-parallel
 * rank sends only its row ranges).  The pipeline: pinned double buffer filled by several host threads -> async H2D on a copy
 * stream -> double-buffered device staging -> repack kernel on the plan's stream. */
int b200_upload_info(b200_plan *plan, double *seconds, double *host_copy_seconds, int64_t *h2d_bytes);

/* The weight form b200_plan_create chose (any pointer may be NULL).  A single-GPU dense plan whose tensors hold a K-quant matrix
 * (Q4_K / Q5_K / Q6_K) computes two weight footprints from the shapes and tile layouts: q8_weight_bytes with every matrix re-quantised
 * to Q8_0 tiles, and the resident form, where every weight stream whose sources share one K-quant format keeps the raw K-quant
 * super-blocks and the decode kernels rebuild the reference's Q8_0 blocks from them on the fly (bit-identical results).  It adds
 * what the plan allocates besides the weights (KV cache, activations, upload staging) and a 1 GiB margin, and compares with the
 * device's free memory: Q8_0 tiles when they fit (*resident = 0), else the resident form (*resident = 1), else creation fails with
 * B200_ERR_OOM naming both figures.  weight_bytes is the footprint of the chosen form.  Other Q8_0 plans report *resident = 0 and
 * weight_bytes == q8_weight_bytes; FP16, tensor-parallel and Qwen2-MoE plans report 0 for both (they never go resident).
 * A resident plan decodes through the CUDA graph (b200_forward_decode, _sample, b200_decode_sequence, b200_trace_decode) and
 * prefills through B200_PREFILL_EXACT, one token per step.  It refuses with B200_ERR_UNSUPPORTED and the reason: the persistent
 * decode kernel, b200_set_decode_slots (n_slots > 0), b200_forward_decode_multi, b200_forward_step (b200_decode_multi_rows reports 0)
 * and both tensor-core prefill modes. */
int b200_weight_info(b200_plan *plan, int32_t *resident, int64_t *weight_bytes, int64_t *q8_weight_bytes);

/* Test hook: replaces the device free-memory figure the weight-form rule of b200_plan_create reads (see b200_weight_info), and
 * the one b200_set_prefill_mode(B200_PREFILL_TENSOR_CORE_EXACT) checks a resident plan's Q8_0 scratch against, by `bytes` for
 * every later plan or call in the process; 0 restores the real figure.  Lets tests put a budget on either side of the
 * threshold without filling a shared GPU.  bytes < 0: B200_ERR_BAD_ARG. */
int b200_test_set_memory_budget(int64_t bytes);

/* The shared-memory rings plan creation gives one layer's decode weight streams (a host computation: no device is needed).  QKV's
 * and gate/up's rings are the largest that fit beside their neighbours under programmatic dependent launch (DESIGN.md §5a).
 * shape[10]: dim, q width (n_heads * head_size), kv width, hidden, SMs, fused norm (0 / 1), then the tile format of QKV, Wo, gate/up
 * and W2 (0: Q8_0 tiles; 12 / 13 / 14: resident Q4_K / Q5_K / Q6_K tiles).  dev[4]: shared memory per SM, reserved per resident
 * CTA, opt-in limit per CTA, and the attention CTA's shared memory.  out[16]: for QKV, Wo, gate/up and W2 in turn, the launch's
 * dynamic shared memory, its ring stages, the bytes of one stage and the tiles of the largest CTA slice.
 * B200_ERR_BAD_ARG on a null pointer, a non-positive size or an unknown format; B200_ERR_UNSUPPORTED when a width has no tiling. */
int b200_stream_rings(const int32_t *shape, const int64_t *dev, int64_t *out);

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
