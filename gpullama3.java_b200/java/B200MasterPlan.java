// B200MasterPlan.java -- java.lang.foreign (Panama, JDK 22+) shim that puts libb200llama.so behind
// the reference's TornadoVMMasterPlan interface (tornadovm/TornadoVMMasterPlan.java:30-85).
//
// SHIPPED AS SOURCE: this image has no JDK, so the file is not compiled or exercised here; the
// identical C ABI (include/b200llama.h) is exercised from Python ctypes in tests/.  Drop it into
// src/main/java/org/beehive/gpullama3/tornadovm/ of the reference (see INTEGRATION.md).
package org.beehive.gpullama3.tornadovm;

import org.beehive.gpullama3.inference.state.State;
import org.beehive.gpullama3.model.Configuration;
import org.beehive.gpullama3.model.Model;
import org.beehive.gpullama3.tensor.GGMLTensorEntry;

import java.lang.foreign.Arena;
import java.lang.foreign.FunctionDescriptor;
import java.lang.foreign.Linker;
import java.lang.foreign.MemoryLayout;
import java.lang.foreign.MemorySegment;
import java.lang.foreign.StructLayout;
import java.lang.foreign.SymbolLookup;
import java.lang.invoke.MethodHandle;
import java.util.Map;

import static java.lang.foreign.ValueLayout.ADDRESS;
import static java.lang.foreign.ValueLayout.JAVA_FLOAT;
import static java.lang.foreign.ValueLayout.JAVA_INT;
import static java.lang.foreign.ValueLayout.JAVA_LONG;

/** One native plan = one TornadoVMMasterPlan: create, forward*, free. Single-owner, like the reference. */
public final class B200MasterPlan implements AutoCloseable {

    private static final Linker LINKER = Linker.nativeLinker();
    private static final SymbolLookup LIB = SymbolLookup.libraryLookup(System.getProperty("b200.lib", "libb200llama.so"), Arena.global());

    // struct b200_config: 9 x int32, 2 x float, 3 x int32
    private static final StructLayout CONFIG = MemoryLayout.structLayout(
            JAVA_INT.withName("arch"), JAVA_INT.withName("dim"), JAVA_INT.withName("hidden_dim"), JAVA_INT.withName("n_layers"),
            JAVA_INT.withName("n_heads"), JAVA_INT.withName("n_kv_heads"), JAVA_INT.withName("head_size"), JAVA_INT.withName("vocab_size"),
            JAVA_INT.withName("context_length"), JAVA_FLOAT.withName("rms_norm_eps"), JAVA_FLOAT.withName("rope_theta"),
            JAVA_INT.withName("fp16_lanes"), JAVA_INT.withName("tp_rank"), JAVA_INT.withName("tp_size"));
    // struct b200_tensor: char* name, void* data, int32 type, int32 n_dims, int64 dims[4]
    private static final StructLayout TENSOR = MemoryLayout.structLayout(
            ADDRESS.withName("name"), ADDRESS.withName("data"), JAVA_INT.withName("ggml_type"), JAVA_INT.withName("n_dims"),
            MemoryLayout.sequenceLayout(4, JAVA_LONG).withName("dims"));

    // struct b200_moe_config: 4 x int32 (Qwen2-MoE and Qwen3-MoE plans)
    private static final StructLayout MOE_CONFIG = MemoryLayout.structLayout(
            JAVA_INT.withName("n_experts"), JAVA_INT.withName("n_experts_used"), JAVA_INT.withName("expert_hidden_dim"), JAVA_INT.withName("shared_hidden_dim"));

    // struct b200_granite_config: 4 x float (Granite plans)
    private static final StructLayout GRANITE_CONFIG = MemoryLayout.structLayout(
            JAVA_FLOAT.withName("embedding_scale"), JAVA_FLOAT.withName("residual_scale"), JAVA_FLOAT.withName("attention_scale"), JAVA_FLOAT.withName("logit_scale"));

    // struct b200_yarn_config: 4 x float, int32 (Devstral plans with a YaRN RoPE table)
    private static final StructLayout YARN_CONFIG = MemoryLayout.structLayout(
            JAVA_FLOAT.withName("factor"), JAVA_FLOAT.withName("beta_fast"), JAVA_FLOAT.withName("beta_slow"), JAVA_FLOAT.withName("log_multiplier"),
            JAVA_INT.withName("original_context_length"));

    private static MethodHandle fn(String name, FunctionDescriptor fd) {
        return LINKER.downcallHandle(LIB.find(name).orElseThrow(), fd);
    }

    private static final MethodHandle CREATE = fn("b200_plan_create",
            FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, JAVA_INT, JAVA_INT, JAVA_INT, ADDRESS, ADDRESS, JAVA_LONG));
    private static final MethodHandle CREATE_MOE = fn("b200_plan_create_moe",
            FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, ADDRESS, JAVA_INT, JAVA_INT, JAVA_INT, ADDRESS, ADDRESS, JAVA_LONG));
    private static final MethodHandle CREATE_GRANITE = fn("b200_plan_create_granite",
            FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, ADDRESS, JAVA_INT, JAVA_INT, JAVA_INT, ADDRESS, ADDRESS, JAVA_LONG));
    private static final MethodHandle CREATE_DEVSTRAL = fn("b200_plan_create_devstral",
            FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, ADDRESS, JAVA_INT, JAVA_INT, JAVA_INT, ADDRESS, ADDRESS, JAVA_LONG));
    private static final MethodHandle DECODE = fn("b200_forward_decode", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, JAVA_INT, ADDRESS, ADDRESS));
    private static final MethodHandle PREFILL = fn("b200_forward_prefill", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, JAVA_INT));
    private static final MethodHandle BATCH_PREFILL = fn("b200_forward_batch_prefill", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, JAVA_INT, JAVA_INT));
    private static final MethodHandle SCORE_TOKENS = fn("b200_score_tokens", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, ADDRESS, JAVA_INT, JAVA_INT, ADDRESS, ADDRESS));
    private static final MethodHandle SET_LOGPROBS = fn("b200_set_logprobs", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT));
    private static final MethodHandle READ_LOGPROBS = fn("b200_read_logprobs", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle SET_SAMPLING_CONTROLS = fn("b200_set_sampling_controls", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS));
    private static final MethodHandle SET_SAMPLE_HISTORY = fn("b200_set_sample_history", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, JAVA_INT));
    private static final MethodHandle SET_PREFILL_MODE = fn("b200_set_prefill_mode", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT));
    private static final MethodHandle SET_DECODE_MODE = fn("b200_set_decode_mode", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT));
    private static final MethodHandle DECODE_SAMPLE = fn("b200_forward_decode_sample",
            FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, JAVA_INT, JAVA_FLOAT, JAVA_FLOAT, JAVA_FLOAT, ADDRESS, ADDRESS));
    private static final MethodHandle DECODE_SEQUENCE = fn("b200_decode_sequence",
            FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, JAVA_INT, JAVA_INT, JAVA_INT, ADDRESS, ADDRESS));
    private static final MethodHandle TP_HANDLE = fn("b200_tp_handle", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS));
    private static final MethodHandle TP_ATTACH = fn("b200_tp_attach", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, JAVA_INT));
    private static final MethodHandle KV_RESET = fn("b200_kv_reset", FunctionDescriptor.of(JAVA_INT, ADDRESS));
    private static final MethodHandle SET_DECODE_SLOTS = fn("b200_set_decode_slots", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT));
    private static final MethodHandle DECODE_BATCH = fn("b200_forward_decode_batch",
            FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle FORWARD_STEP = fn("b200_forward_step", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle FORWARD_CHUNK = fn("b200_forward_chunk", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle CHUNK_ROWS = fn("b200_chunk_rows", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS));
    private static final MethodHandle SLOT_RESET = fn("b200_slot_reset", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT));
    private static final MethodHandle SLOT_COPY_KV = fn("b200_slot_copy_kv", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, JAVA_INT));
    private static final MethodHandle PREFILL_SLOTS = fn("b200_prefill_slots", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle DECODE_MULTI = fn("b200_forward_decode_multi", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, JAVA_INT, ADDRESS, JAVA_INT, ADDRESS, ADDRESS));
    private static final MethodHandle MULTI_ROWS = fn("b200_decode_multi_rows", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS));
    private static final MethodHandle WEIGHT_INFO = fn("b200_weight_info", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, ADDRESS, ADDRESS));
    private static final MethodHandle FREE = fn("b200_plan_free", FunctionDescriptor.ofVoid(ADDRESS));
    private static final MethodHandle LAST_ERROR = fn("b200_last_error", FunctionDescriptor.of(ADDRESS, ADDRESS));

    private final Arena arena = Arena.ofConfined();
    private final MemorySegment plan;
    private final MemorySegment logits;   // vocab floats, reused every token (state.wrapLogits in the reference)
    private final MemorySegment argmax;

    /** TornadoVMMasterPlan.initializeTornadoVMPlan(state, model): tensors are the plain mmap slices of GGUF.loadTensorsStandard.
     *  archId: 0 = Llama / Mistral, 1 = Qwen3, 2 = Phi-3 (pass blk.N.attn_qkv.weight and blk.N.ffn_up.weight fused, as in the file). */
    public B200MasterPlan(State state, Model model, Map<String, GGMLTensorEntry> tensors, int archId, int headSize) throws Throwable {
        this(state, model, tensors, archId, headSize, 0, 1);
    }

    /** One plan per GPU for tensor-parallel decode: every rank passes the same tensors, the library uploads its row slices. */
    public B200MasterPlan(State state, Model model, Map<String, GGMLTensorEntry> tensors, int archId, int headSize, int tpRank, int tpSize) throws Throwable {
        this(state, model, tensors, archId, headSize, tpRank, tpSize, null, null, false, null, 0);
    }

    /** Qwen2-MoE (archId = ARCH_QWEN2_MOE, single GPU): moe = {numberOfExperts, numberOfExpertsUsed, moeHiddenDim, sharedExpertHiddenDim}
     *  (Qwen2MoEConfiguration); the router, shared-expert gate, stacked experts and shared expert go in `tensors` as in the file. */
    public B200MasterPlan(State state, Model model, Map<String, GGMLTensorEntry> tensors, int headSize, int[] moe) throws Throwable {
        this(state, model, tensors, ARCH_QWEN2_MOE, headSize, 0, 1, moe, null, false, null, 0);
    }

    /** Qwen2-MoE or Qwen3-MoE (archId = ARCH_QWEN2_MOE or ARCH_QWEN3_MOE, single GPU).  Qwen3-MoE: moe = {numberOfExperts,
     *  numberOfExpertsUsed, moeHiddenDim, 0} (no shared expert), headSize = attention.key_length; `tensors` holds Qwen3's attention
     *  tensors (with attn_q_norm / attn_k_norm), the router and the stacked experts, as in the file.  The top-k weights are
     *  renormalised to sum to one, and b200_read_buffer("moe_weights") gives k weights per layer. */
    public B200MasterPlan(State state, Model model, Map<String, GGMLTensorEntry> tensors, int archId, int headSize, int[] moe) throws Throwable {
        this(state, model, tensors, archId, headSize, 0, 1, moe, null, false, null, 0);
    }

    /** Granite (archId = ARCH_GRANITE): granite = {embeddingScale, residualScale, attentionScale, logitScale} (GraniteConfiguration);
     *  Llama's tensors, tied classifier. */
    public B200MasterPlan(State state, Model model, Map<String, GGMLTensorEntry> tensors, int headSize, int tpRank, int tpSize, float[] granite) throws Throwable {
        this(state, model, tensors, ARCH_GRANITE, headSize, tpRank, tpSize, null, granite, false, null, 0);
    }

    /** Devstral 2 (archId = ARCH_DEVSTRAL): headSize = mistral3.attention.key_length (DevstralConfiguration.headDim()); Llama's tensors;
     *  yarn = {factor, betaFast, betaSlow, logMultiplier} and originalContextLength when mistral3.rope.scaling.type is "yarn"
     *  (DevstralModelLoader.precomputeRopeFrequencies), yarn = null for the plain RoPE table. */
    public B200MasterPlan(State state, Model model, Map<String, GGMLTensorEntry> tensors, int headSize, int tpRank, int tpSize, float[] yarn,
                          int originalContextLength) throws Throwable {
        this(state, model, tensors, ARCH_DEVSTRAL, headSize, tpRank, tpSize, null, null, true, yarn, originalContextLength);
    }

    private B200MasterPlan(State state, Model model, Map<String, GGMLTensorEntry> tensors, int archId, int headSize, int tpRank, int tpSize, int[] moe,
                           float[] granite, boolean devstral, float[] yarn, int yarnContextLength) throws Throwable {
        Configuration c = model.configuration();
        MemorySegment cfg = arena.allocate(CONFIG);
        int[] ints = {archId, c.dim(), c.hiddenDim(), c.numberOfLayers(), c.numberOfHeads(), c.numberOfKeyValueHeads(), headSize,
                c.vocabularySize(), c.contextLength()};
        for (int i = 0; i < ints.length; i++) cfg.setAtIndex(JAVA_INT, i, ints[i]);
        cfg.set(JAVA_FLOAT, 36, c.rmsNormEps());
        cfg.set(JAVA_FLOAT, 40, c.ropeTheta());
        cfg.set(JAVA_INT, 44, Integer.getInteger("llama.VectorBitSize", 512) / 32); // FloatTensor.java:21
        cfg.set(JAVA_INT, 48, tpRank);
        cfg.set(JAVA_INT, 52, tpSize);

        MemorySegment arr = arena.allocate(TENSOR, tensors.size());
        int i = 0;
        for (var e : tensors.entrySet()) {
            MemorySegment t = arr.asSlice((long) i * TENSOR.byteSize(), TENSOR.byteSize());
            t.set(ADDRESS, 0, arena.allocateFrom(e.getKey()));
            t.set(ADDRESS, 8, e.getValue().memorySegment());       // MemorySegment.address() of the mapping
            t.set(JAVA_INT, 16, e.getValue().ggmlType().ordinal()); // GGMLType ordinal == ggml type id (F32 0, F16 1, Q8_0 8, Q4_K 12, Q5_K 13, Q6_K 14: GGMLType.java:5-20); K-quants are re-quantised on the device
            int[] shape = e.getValue().shape();
            t.set(JAVA_INT, 20, shape.length);
            for (int d = 0; d < shape.length; d++) t.set(JAVA_LONG, 24 + 8L * d, shape[d]);
            i++;
        }
        MemorySegment out = arena.allocate(ADDRESS);
        MemorySegment err = arena.allocate(512);
        int batch = TornadoVMMasterPlan.WITH_PREFILL_DECODE ? TornadoVMMasterPlan.PREFILL_BATCH_SIZE : 0;
        int rc;
        if (devstral) {
            MemorySegment yc = MemorySegment.NULL;
            if (yarn != null) {
                yc = arena.allocate(YARN_CONFIG);
                for (int k = 0; k < 4; k++) yc.setAtIndex(JAVA_FLOAT, k, yarn[k]);
                yc.set(JAVA_INT, 16, yarnContextLength);
            }
            rc = (int) CREATE_DEVSTRAL.invokeExact(cfg, yc, arr, tensors.size(), batch, Integer.getInteger("b200.device", tpRank), out, err, 512L);
        } else if (moe != null) {
            MemorySegment mc = arena.allocate(MOE_CONFIG);
            for (int k = 0; k < 4; k++) mc.setAtIndex(JAVA_INT, k, moe[k]);
            rc = (int) CREATE_MOE.invokeExact(cfg, mc, arr, tensors.size(), batch, Integer.getInteger("b200.device", tpRank), out, err, 512L);
        } else if (granite != null) {
            MemorySegment gc = arena.allocate(GRANITE_CONFIG);
            for (int k = 0; k < 4; k++) gc.setAtIndex(JAVA_FLOAT, k, granite[k]);
            rc = (int) CREATE_GRANITE.invokeExact(cfg, gc, arr, tensors.size(), batch, Integer.getInteger("b200.device", tpRank), out, err, 512L);
        } else {
            rc = (int) CREATE.invokeExact(cfg, arr, tensors.size(), batch, Integer.getInteger("b200.device", tpRank), out, err, 512L);
        }
        check(rc, err.getString(0));
        plan = out.get(ADDRESS, 0);
        logits = arena.allocate(JAVA_FLOAT, c.vocabularySize());
        argmax = arena.allocate(JAVA_INT);
    }

    private static void check(int rc, String msg) {
        if (rc == 0) return;
        if (rc == -2) throw new UnsupportedOperationException(msg);            // ForwardPlanFactory.java:84-87
        if (rc == -3) throw new OutOfMemoryError("device memory: " + msg); // README.md:262-265
        throw new IllegalStateException("b200llama error " + rc + ": " + msg);
    }

    private String lastError() throws Throwable {
        return ((MemorySegment) LAST_ERROR.invokeExact(plan)).reinterpret(512).getString(0);
    }

    /** FloatArray tornadoVMForwardDecode(int position) + the embedding gather of InferenceCore.forwardTornadoVM (InferenceCore.java:956-980). */
    public MemorySegment forwardDecode(int token, int position) throws Throwable {
        int rc = (int) DECODE.invokeExact(plan, token, position, logits, argmax);
        if (rc != 0) check(rc, lastError());
        return logits;
    }

    /** Greedy path: only the argmax (4 bytes) crosses PCIe. */
    public int forwardDecodeArgmax(int token, int position) throws Throwable {
        int rc = (int) DECODE.invokeExact(plan, token, position, MemorySegment.NULL, argmax);
        if (rc != 0) check(rc, lastError());
        return argmax.get(JAVA_INT, 0);
    }

    /** void tornadoVMForwardPrefill(int position) (TornadoVMMasterPlanPrefillDecode.java:116). */
    public void forwardPrefill(int token, int position) throws Throwable {
        int rc = (int) PREFILL.invokeExact(plan, token, position);
        if (rc != 0) check(rc, lastError());
    }

    /** void tornadoVMForwardBatchPrefill() (TornadoVMMasterPlanBatchPrefillDecode.java:107-123). */
    public void forwardBatchPrefill(int[] tokens, int startPos) throws Throwable {
        try (Arena a = Arena.ofConfined()) {
            int rc = (int) BATCH_PREFILL.invokeExact(plan, a.allocateFrom(JAVA_INT, tokens), tokens.length, startPos);
            if (rc != 0) check(rc, lastError());
        }
    }

    /** Scores tokens[i] at startPos + i (their K/V go into the cache as forwardBatchPrefill writes them): logprobs[i] = the model's
     *  log-probability of targets[i] (-1: NaN) computed in double from logits bit-identical to forwardDecode's, greedyIds[i] = their
     *  argmax.  Prefill modes exact and tensor_core_exact only; tokens.length within forwardBatchPrefill's limit. */
    public void scoreTokens(int[] tokens, int[] targets, int startPos, double[] logprobs, int[] greedyIds) throws Throwable {
        if (targets.length != tokens.length || logprobs.length < tokens.length || greedyIds.length < tokens.length)
            throw new IllegalArgumentException("targets, logprobs and greedyIds must hold tokens.length entries");
        try (Arena a = Arena.ofConfined()) {
            MemorySegment lp = a.allocate(java.lang.foreign.ValueLayout.JAVA_DOUBLE, tokens.length);
            MemorySegment ids = a.allocate(JAVA_INT, tokens.length);
            int rc = (int) SCORE_TOKENS.invokeExact(plan, a.allocateFrom(JAVA_INT, tokens), a.allocateFrom(JAVA_INT, targets), tokens.length, startPos, lp, ids);
            if (rc != 0) check(rc, lastError());
            MemorySegment.copy(lp, java.lang.foreign.ValueLayout.JAVA_DOUBLE, 0, logprobs, 0, tokens.length);
            MemorySegment.copy(ids, JAVA_INT, 0, greedyIds, 0, tokens.length);
        }
    }

    /** The last emitting call's log-probabilities: chosen[i] for its i-th emitted id, topIds[i][k] / topLogprobs[i][k] for the k-th
     *  most likely alternative (ties to the lower id).  Rows of forwardStep that do not emit hold NaN and id -1. */
    public record Logprobs(double[] chosen, int[][] topIds, double[][] topLogprobs) {}

    private int logprobsTopN = -1;

    /** Log-probabilities of generated tokens (b200_set_logprobs): -1 off (the default), 0..20 alternatives per emitted id.  While on,
     *  every call that emits ids records one row per id, in double and under the raw logits (temperature 1), read with lastLogprobs.
     *  Single-GPU plans only. */
    public void setLogprobs(int topN) throws Throwable {
        int rc = (int) SET_LOGPROBS.invokeExact(plan, topN);
        if (rc != 0) check(rc, lastError());
        logprobsTopN = topN;
    }

    /** The rows the last emitting call recorded (b200_read_logprobs); setLogprobs must be on. */
    public Logprobs lastLogprobs() throws Throwable {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment nRows = a.allocate(JAVA_INT);
            int rc = (int) READ_LOGPROBS.invokeExact(plan, 0, nRows, MemorySegment.NULL, MemorySegment.NULL, MemorySegment.NULL);
            if (rc != 0) check(rc, lastError());
            int rows = nRows.get(JAVA_INT, 0), n = Math.max(logprobsTopN, 0);
            MemorySegment ch = a.allocate(java.lang.foreign.ValueLayout.JAVA_DOUBLE, Math.max(rows, 1));
            MemorySegment ids = a.allocate(JAVA_INT, Math.max(rows * n, 1));
            MemorySegment lps = a.allocate(java.lang.foreign.ValueLayout.JAVA_DOUBLE, Math.max(rows * n, 1));
            rc = (int) READ_LOGPROBS.invokeExact(plan, rows, nRows, ch, ids, lps);
            if (rc != 0) check(rc, lastError());
            double[] chosen = new double[rows];
            int[][] topIds = new int[rows][n];
            double[][] topLogprobs = new double[rows][n];
            MemorySegment.copy(ch, java.lang.foreign.ValueLayout.JAVA_DOUBLE, 0, chosen, 0, rows);
            for (int i = 0; i < rows; i++) {
                MemorySegment.copy(ids, JAVA_INT, (long) i * n * 4, topIds[i], 0, n);
                MemorySegment.copy(lps, java.lang.foreign.ValueLayout.JAVA_DOUBLE, (long) i * n * 8, topLogprobs[i], 0, n);
            }
            return new Logprobs(chosen, topIds, topLogprobs);
        }
    }

    /** One sequence's sampling controls (b200_sampling_controls): top-k (0 off; every token tied at the k-th value kept), min-p in
     *  logit space (0 off), llama.cpp's repetition (1 off) / frequency / presence (0 off) penalties over the sequence's token counts,
     *  and a logit bias per token id (biasIds / biasValues of equal length, distinct ids, finite values; at most 1024). */
    public record SamplingControls(int topK, float minP, float repetitionPenalty, float frequencyPenalty, float presencePenalty,
                                   int[] biasIds, float[] biasValues) {}

    /** b200_set_sampling_controls: controls for one sequence (slot -1: the plan's own cache), applied on the device by
     *  forwardDecodeSample, forwardDecodeBatch with sampling and forwardStep's emitting rows; null turns them off. */
    public void setSamplingControls(int slot, SamplingControls c) throws Throwable {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment s = MemorySegment.NULL;
            if (c != null) {
                int nb = c.biasIds() == null ? 0 : c.biasIds().length;
                if (nb != (c.biasValues() == null ? 0 : c.biasValues().length)) throw new IllegalArgumentException("biasIds and biasValues differ in length");
                s = a.allocate(40, 8); // {int32 top_k; float min_p, rep, freq, pres; int32 n_bias; const int32_t *ids; const float *values}
                s.set(JAVA_INT, 0, c.topK());
                s.set(java.lang.foreign.ValueLayout.JAVA_FLOAT, 4, c.minP());
                s.set(java.lang.foreign.ValueLayout.JAVA_FLOAT, 8, c.repetitionPenalty());
                s.set(java.lang.foreign.ValueLayout.JAVA_FLOAT, 12, c.frequencyPenalty());
                s.set(java.lang.foreign.ValueLayout.JAVA_FLOAT, 16, c.presencePenalty());
                s.set(JAVA_INT, 20, nb);
                s.set(ADDRESS, 24, nb == 0 ? MemorySegment.NULL : a.allocateFrom(JAVA_INT, c.biasIds()));
                s.set(ADDRESS, 32, nb == 0 ? MemorySegment.NULL : a.allocateFrom(java.lang.foreign.ValueLayout.JAVA_FLOAT, c.biasValues()));
            }
            int rc = (int) SET_SAMPLING_CONTROLS.invokeExact(plan, slot, s);
            if (rc != 0) check(rc, lastError());
        }
    }

    /** b200_set_sample_history: the sequence's token counts become those of tokens (e.g. the prompt). */
    public void setSampleHistory(int slot, int[] tokens) throws Throwable {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment t = tokens.length == 0 ? MemorySegment.NULL : a.allocateFrom(JAVA_INT, tokens);
            int rc = (int) SET_SAMPLE_HISTORY.invokeExact(plan, slot, t, tokens.length);
            if (rc != 0) check(rc, lastError());
        }
    }

    /** Forward + Sampler.sampleToken on the device (Sampler.java:74-122): the caller draws uniform01 = rng.nextFloat(1f) from the
     *  sampler's own RandomGenerator (Sampler.java:84) and gets the token id back; the logits row never crosses PCIe. */
    public int forwardDecodeSample(int token, int position, float temperature, float topp, float uniform01) throws Throwable {
        int rc = (int) DECODE_SAMPLE.invokeExact(plan, token, position, temperature, topp, uniform01, argmax, MemorySegment.NULL);
        if (rc != 0) check(rc, lastError());
        return argmax.get(JAVA_INT, 0);
    }

    /** 0 = CUDA graph of ~7 kernels per layer, 1 = one persistent kernel per token (default when the plan supports it); bit-identical. */
    public void setDecodeMode(int mode) throws Throwable {
        int rc = (int) SET_DECODE_MODE.invokeExact(plan, mode);
        if (rc != 0) check(rc, lastError());
    }

    public static final int PREFILL_EXACT = 0, PREFILL_TENSOR_CORE = 1, PREFILL_TENSOR_CORE_W8A16 = 2, PREFILL_TENSOR_CORE_EXACT = 3;
    /** PREFILL_TENSOR_CORE_EXACT for Qwen2-MoE / Qwen3-MoE plans: the chunk routed on the device, grouped int8 expert GEMMs, KV cache bit-identical to PREFILL_EXACT. */
    public static final int PREFILL_TENSOR_CORE_EXACT_MOE = 4;
    // b200_config.arch (include/b200llama.h): Qwen2 / Qwen2.5 / DeepSeek-R1-Distill-Qwen pass blk.N.attn_{q,k,v}.bias (F32) with the weights
    public static final int ARCH_LLAMA = 0, ARCH_QWEN3 = 1, ARCH_PHI3 = 2, ARCH_QWEN2 = 3, ARCH_QWEN2_MOE = 4, ARCH_GRANITE = 5, ARCH_DEVSTRAL = 6,
            ARCH_QWEN3_MOE = 7;

    /** TensorCoreSupport.java's switch: 0 = exact token-by-token prefill (bit-identical KV cache), 1 = TMA + wgmma GEMMs (a Q8_0
     *  plan first builds f16 twins of its matrices, +2 bytes per weight), 2 = the same GEMMs on a Q8_0 plan reading the Q8_0 weights
     *  in place and dequantising them in shared memory (no twins; bit-identical to 1 where no residual GEMM splits K). */
    public void setPrefillMode(int mode) throws Throwable {
        int rc = (int) SET_PREFILL_MODE.invokeExact(plan, mode);
        if (rc != 0) check(rc, lastError());
    }

    /** The greedy loop of InferenceEngine.generateTokensGPULlama with sampler and token feedback on the device (feedback = true),
     *  or LlamaBench's teacher-forced loop (feedback = false): n steps from startPos, returns the argmax of every step. */
    public int[] decodeSequence(int[] tokens, int n, int startPos, boolean feedback) throws Throwable {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment ids = a.allocate(JAVA_INT, n);
            int rc = (int) DECODE_SEQUENCE.invokeExact(plan, a.allocateFrom(JAVA_INT, tokens), n, startPos, feedback ? 1 : 0, ids, MemorySegment.NULL);
            if (rc != 0) check(rc, lastError());
            return ids.toArray(JAVA_INT);
        }
    }

    /** 64-byte CUDA-IPC handle of this rank's communication buffer; exchange with the other ranks, then attach(all handles in rank order). */
    public byte[] tpHandle() throws Throwable {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment h = a.allocate(64);
            int rc = (int) TP_HANDLE.invokeExact(plan, h);
            if (rc != 0) check(rc, lastError());
            return h.toArray(java.lang.foreign.ValueLayout.JAVA_BYTE);
        }
    }

    public void tpAttach(byte[][] handles) throws Throwable {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment all = a.allocate(64L * handles.length);
            for (int r = 0; r < handles.length; r++) MemorySegment.copy(handles[r], 0, all, java.lang.foreign.ValueLayout.JAVA_BYTE, 64L * r, 64);
            int rc = (int) TP_ATTACH.invokeExact(plan, all, handles.length);
            if (rc != 0) check(rc, lastError());
        }
    }

    public void kvReset() throws Throwable {
        int rc = (int) KV_RESET.invokeExact(plan);
        if (rc != 0) check(rc, lastError());
    }

    /** Up to 8 KV-cache slots (one State per conversation) for forwardDecodeBatch; 0 frees them.  Q8_0 plans only. */
    public void setDecodeSlots(int nSlots) throws Throwable {
        int rc = (int) SET_DECODE_SLOTS.invokeExact(plan, nSlots);
        if (rc != 0) check(rc, lastError());
    }

    /** One step for tokens.length independent sequences: row i = tokens[i] at positions[i] on slot slots[i].  sampling is null
     *  (greedy) or {temperature, topp, rng.nextFloat(1f)} per row.  Returns one token id per row; each row is bit-identical to
     *  forwardDecode / forwardDecodeSample of its own sequence. */
    public int[] forwardDecodeBatch(int[] slots, int[] tokens, int[] positions, float[] sampling) throws Throwable {
        try (Arena a = Arena.ofConfined()) {
            int n = tokens.length;
            MemorySegment ids = a.allocate(JAVA_INT, n);
            MemorySegment smp = sampling == null ? MemorySegment.NULL : a.allocateFrom(java.lang.foreign.ValueLayout.JAVA_FLOAT, sampling);
            int rc = (int) DECODE_BATCH.invokeExact(plan, n, a.allocateFrom(JAVA_INT, slots), a.allocateFrom(JAVA_INT, tokens),
                    a.allocateFrom(JAVA_INT, positions), smp, ids, MemorySegment.NULL);
            if (rc != 0) check(rc, lastError());
            return ids.toArray(JAVA_INT);
        }
    }

    /** One mixed step: row i = tokens[i] at positions[i] on slot slots[i]; a slot may take several rows at distinct positions.  emit[i]
     *  false: K/V only (a prompt position), id -1; true: the id after the row, greedy or, with sampling non-null, sampled from
     *  {temperature, topp, rng.nextFloat(1f)} of row i (temperature 0 = argmax).  Every row's K/V is written before any row attends,
     *  so each emitting row is bit-identical to forwardDecode / forwardDecodeSample of its own sequence (b200_forward_step). */
    public int[] forwardStep(int[] slots, int[] tokens, int[] positions, boolean[] emit, float[] sampling) throws Throwable {
        return stepRows(FORWARD_STEP, slots, tokens, positions, emit, sampling);
    }

    /** forwardStep on the tensor cores: the same rows and ids, run as one chunk of the bit-exact int8 prefill (the plan's prefill
     *  mode must be tensor_core_exact), so prompt rows ride in the chunk's GEMMs with the decode rows.  Up to chunkRows() rows, at
     *  most 8 of them emitting (b200_forward_chunk). */
    public int[] forwardChunk(int[] slots, int[] tokens, int[] positions, boolean[] emit, float[] sampling) throws Throwable {
        return stepRows(FORWARD_CHUNK, slots, tokens, positions, emit, sampling);
    }

    private int[] stepRows(MethodHandle call, int[] slots, int[] tokens, int[] positions, boolean[] emit, float[] sampling) throws Throwable {
        try (Arena a = Arena.ofConfined()) {
            int n = tokens.length;
            MemorySegment rows = a.allocate(28L * Math.max(1, n), 4); // b200_step_row: 4 int32 + 3 float
            for (int i = 0; i < n; i++) {
                long o = 28L * i;
                rows.set(JAVA_INT, o, slots[i]);
                rows.set(JAVA_INT, o + 4, tokens[i]);
                rows.set(JAVA_INT, o + 8, positions[i]);
                rows.set(JAVA_INT, o + 12, emit[i] ? 1 : 0);
                for (int k = 0; k < 3; k++)
                    rows.set(JAVA_FLOAT, o + 16 + 4L * k, sampling == null ? 0f : sampling[3 * i + k]);
            }
            MemorySegment ids = a.allocate(JAVA_INT, Math.max(1, n));
            int rc = (int) call.invokeExact(plan, n, rows, ids, MemorySegment.NULL);
            if (rc != 0) check(rc, lastError());
            return ids.asSlice(0, 4L * n).toArray(JAVA_INT);
        }
    }

    public void slotReset(int slot) throws Throwable {
        int rc = (int) SLOT_RESET.invokeExact(plan, slot);
        if (rc != 0) check(rc, lastError());
    }

    /** Positions [0, nPositions) of the plan's own KV cache (a prompt after forwardBatchPrefill) into the slot; the rest of it zeroed. */
    public void slotCopyKv(int slot, int nPositions) throws Throwable {
        int rc = (int) SLOT_COPY_KV.invokeExact(plan, slot, nPositions);
        if (rc != 0) check(rc, lastError());
    }

    /** Prefill prompts[i] straight into slot slots[i] at positions startPositions[i].. (K/V only), all in one call, in the plan's
     *  prefill mode; a tensor-core mode takes at most prefill_batch_size tokens per call.  The plan's own cache and the other slots
     *  are not touched. */
    public void prefillSlots(int[] slots, int[] startPositions, int[][] prompts) throws Throwable {
        try (Arena a = Arena.ofConfined()) {
            int n = slots.length, total = 0;
            int[] lengths = new int[n];
            for (int i = 0; i < n; i++) { lengths[i] = prompts[i].length; total += lengths[i]; }
            int[] tokens = new int[total];
            for (int i = 0, o = 0; i < n; o += lengths[i], i++) System.arraycopy(prompts[i], 0, tokens, o, lengths[i]);
            int rc = (int) PREFILL_SLOTS.invokeExact(plan, n, a.allocateFrom(JAVA_INT, slots), a.allocateFrom(JAVA_INT, startPositions),
                    a.allocateFrom(JAVA_INT, lengths), total == 0 ? MemorySegment.NULL : a.allocateFrom(JAVA_INT, tokens));
            if (rc != 0) check(rc, lastError());
        }
    }

    /** tokens[i] at position startPos + i of ONE sequence in one step (slot -1: the plan's own cache); returns the greedy id after
     *  each position, every row bit-identical to forwardDecode of the same token over the same cache prefix (draft verification). */
    public int[] forwardDecodeMulti(int slot, int[] tokens, int startPos) throws Throwable {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment ids = a.allocate(JAVA_INT, Math.max(1, tokens.length));
            int rc = (int) DECODE_MULTI.invokeExact(plan, slot, tokens.length, a.allocateFrom(JAVA_INT, tokens), startPos, ids, MemorySegment.NULL);
            if (rc != 0) check(rc, lastError());
            return ids.asSlice(0, 4L * tokens.length).toArray(JAVA_INT);
        }
    }

    /** Positions per forwardDecodeMulti step; 0 where the plan cannot run it. */
    public int decodeMultiRows() throws Throwable {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment r = a.allocate(JAVA_INT);
            int rc = (int) MULTI_ROWS.invokeExact(plan, r);
            if (rc != 0) check(rc, lastError());
            return r.get(JAVA_INT, 0);
        }
    }

    /** Rows per forwardChunk call: prefill_batch_size in tensor_core_exact with decode slots, else 0 (b200_chunk_rows). */
    public int chunkRows() throws Throwable {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment r = a.allocate(JAVA_INT);
            int rc = (int) CHUNK_ROWS.invokeExact(plan, r);
            if (rc != 0) check(rc, lastError());
            return r.get(JAVA_INT, 0);
        }
    }

    /** {resident (0 / 1), weight bytes, weight bytes of the all-Q8_0 form}: a K-quant model whose Q8_0 expansion does not fit the
     *  device keeps its K-quant weights resident (same logits; batched steps, the persistent kernel and the tensor-core prefill are
     *  then refused with UnsupportedOperationException). */
    public long[] weightInfo() throws Throwable {
        try (Arena a = Arena.ofConfined()) {
            MemorySegment r = a.allocate(JAVA_INT), w = a.allocate(JAVA_LONG), w8 = a.allocate(JAVA_LONG);
            int rc = (int) WEIGHT_INFO.invokeExact(plan, r, w, w8);
            if (rc != 0) check(rc, lastError());
            return new long[] {r.get(JAVA_INT, 0), w.get(JAVA_LONG, 0), w8.get(JAVA_LONG, 0)};
        }
    }

    /** void freeTornadoExecutionPlan() */
    @Override
    public void close() {
        try {
            FREE.invokeExact(plan);
        } catch (Throwable t) {
            throw new IllegalStateException(t);
        } finally {
            arena.close();
        }
    }
}
