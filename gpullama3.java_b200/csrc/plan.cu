// plan.cu -- libb200llama.so: plan lifecycle, weight upload/repack, CUDA-graph capture and the
// C ABI declared in include/b200llama.h.  Plays the role of TornadoVMMasterPlan*.java +
// tornadovm/plan/** + tornadovm/layers/** of the reference (one native context and one CUDA
// graph per token instead of N+2 TaskGraph executions, TornadoVMMasterPlanSingleToken.java:68-95).
#include "../../include/b200llama.h"
#include "decode_kernels.cuh"
#include "prefill.cuh"
#include "stream_matvec.cuh"
#include "stream_matvec_f16.cuh"
#include "kquant.cuh"
#include "decode_persistent.cuh"
#include "sampler.cuh"
#include "decode_batch.cuh"
#include "moe.cuh"
#include "prefill_i8.cuh"
#include "score.cuh"
#include "logprobs.cuh"

#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <string>
#include <thread>
#include <type_traits>
#include <unordered_map>
#include <utility>
#include <vector>

namespace {

struct LayerW {
    DevMat qkv, wo, w1, w3, w2;
    TileMat tqkv{}, two{}, tgu{}, tw2{}; // tile-major copies for the streaming kernel (Q8_0)
    size_t ring_qkv = 0, ring_gu = 0;    // dynamic shared memory of the QKV and gate/up stream launches (ring_budgets)
    float *attn_norm = nullptr, *ffn_norm = nullptr, *q_norm = nullptr, *k_norm = nullptr;
    float *qkv_bias = nullptr; // Qwen2: this rank's q|k|v bias, laid out like the packed q|k|v vector
    // Qwen2-MoE / Qwen3-MoE (moe.cuh): the shared expert's streams (Qwen2-MoE only), the routed experts' geometry and the device
    // tables of their stream bases
    TileMat sgu{}, sdn{}, xgu{}, xdn{};
    const unsigned char **gu_bases = nullptr, **dn_bases = nullptr;
    float *router = nullptr, *shared_gate = nullptr; // F32 [n_experts][dim] and [dim]
};

// A captured CUDA graph and the kernel launches it holds.
struct Graph {
    cudaGraphExec_t exec = nullptr;
    int launches = 0;
};

// The single-token graphs of one decode implementation: with logits, without (the prefill form), and with trace records.
struct TokenGraphs {
    Graph decode, prefill, trace;
};

// The form of a batched step (enqueue_batch), three independent bits.  SCHED: a step of the exact prefills, its rows copied from
// the call's schedule by k_batch_rows_next, without the classifier.  SPLIT: a slot repeats, so the attention runs as
// k_rope_kv_batch + k_attention_cached_rows.  OWN: the K / V target is the plan's own cache instead of the decode slots.
enum StepForm { SCHED = 1, SPLIT = 2, OWN = 4, STEP_FORMS = 8 };

} // namespace

// Weight upload pipeline (SURVEY 8f N1; replaces the reference's lazy FIRST_EXECUTION copy-in, LlamaQ8_0FFNLayers.java:122-132,
// timed by TornadoVMMasterPlanSingleToken.java:51-54): pageable/mmapped host bytes -> pinned double buffer (several host
// threads) -> async H2D on a copy stream -> device staging (double buffered) -> repack kernel on the plan's stream.  The host
// copy of chunk i+1, the DMA of chunk i and the repack of the previous matrix overlap; nothing synchronises per matrix.
struct Uploader {
    cudaStream_t copy = nullptr;
    unsigned char *pin[2] = {nullptr, nullptr};
    size_t pin_bytes = 0;
    cudaEvent_t pin_done[2] = {nullptr, nullptr};
    bool pin_used[2] = {false, false};
    int pi = 0;
    unsigned char *dst[2] = {nullptr, nullptr};
    size_t dst_bytes = 0;
    cudaEvent_t d_ready[2] = {nullptr, nullptr}, d_free[2] = {nullptr, nullptr};
    bool d_used[2] = {false, false};
    int di = 0;
    int threads = 4;
    double host_copy_s = 0.0, total_s = 0.0;
    int64_t h2d_bytes = 0;
};

struct b200_plan {
    b200_config cfg{};
    Uploader up;
    int device = 0;
    int wtype = 0; // B200_GGML_Q8_0 or B200_GGML_F16 (matrix type)
    int qd = 0, kvd = 0;
    int prefill_batch = 0;
    cudaStream_t stream = nullptr;
    std::vector<void *> allocs;
    int64_t bytes = 0;
    std::string err;

    DevMat emb{}, out{};
    TileMat tout{};
    bool use_pdl = false;
    bool fuse_norm = false; // single-GPU Q8_0 streams: QKV, gate/up and lm_head compute their RMSNorm themselves (k_stream_matvec_q8_norm)
    int kflags = 0; // KF_* (common.cuh): what the attention prologues do for this architecture
    size_t kq_off = 0; // K-quant files: offset of the raw (K-quant bytes) area inside each staging buffer; 0 = no K-quant tensor in the file
    // K-quant files whose Q8_0 expansion does not fit the device (weight_policy): every stream whose sources share one K-quant format
    // keeps the raw super-blocks (TileMat::fmt); w_bytes is the plan's weight footprint, w8_bytes the one of its all-Q8_0 form
    bool resident = false;
    int64_t w_bytes = 0, w8_bytes = 0;
    bool use_f16_stream = false; // FP16 plans: per-warp bulk-copy rings (stream_matvec_f16.cuh) instead of k_matvec_f16
    bool f16_copies = false; // Q8_0 plan that also holds f16 weight matrices for the tensor-core prefill
    int n_sms = 148;
    unsigned *blk_cnt = nullptr;
    float *part_val = nullptr;
    int *part_idx = nullptr;
    float *out_norm = nullptr;
    std::vector<LayerW> layers;
    float *rope_cr = nullptr, *rope_ci = nullptr;

    // activations
    float *x = nullptr, *xb = nullptr, *qkv = nullptr, *hb = nullptr, *hb2 = nullptr, *logits = nullptr;
    int8_t *xq = nullptr, *hq = nullptr;
    float *xs = nullptr, *hs = nullptr;
    float *key_cache = nullptr, *value_cache = nullptr;
    StepState *st = nullptr;
    int *seq_tokens = nullptr, *out_ids = nullptr;
    int seq_cap = 0;
    StepState *h_st = nullptr; // pinned
    int *h_ids = nullptr;      // pinned, seq_cap (also the single-token calls' step_outputs block, 9 ints)

    TokenGraphs graph; // the multi-kernel decode graph (round 1)
    TokenGraphs pers;  // one persistent kernel per token (decode_persistent.cuh)
    unsigned long long *trace_rec = nullptr;
    int decode_mode = B200_DECODE_GRAPH; // which of the two the forward entry points launch
    float *att_scratch = nullptr; // [heads][ctx] score rows when the context does not fit shared memory
    int *smp_indices = nullptr, *smp_out = nullptr; // device-side sampler scratch (sampler.cuh): candidate list, {id, info[4]}

    // tensor parallelism (tp.n == 1: single GPU).  *_l = this rank's share.
    TpCtx tp{};
    unsigned char *comm = nullptr; // IPC-exported communication buffer (x, gathered activations, flags)
    size_t comm_bytes = 0;
    bool attached = false;
    int nh_l = 0, nkv_l = 0, qd_l = 0, kvd_l = 0, hid_l = 0, dim_l = 0, voc_l = 0;
    int8_t *attq = nullptr; // gathered attention output (quantised) feeding the Wo matvec
    float *atts = nullptr;
    void *peer_open[TP_MAX] = {nullptr};
    int launches_prefill = 0;
    float prefill_ms = 0.f; // device time of the last tensor-core prefill chunk
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;

    // Qwen2-MoE / Qwen3-MoE: the routing buffers [layer][k] ids and [layer][moe_nw] weights of the last step, the router logits
    // scratch and arrival counters, the down projection's shared-memory layout
    bool is_moe = false;
    bool moe_shared = false; // Qwen2-MoE: a shared expert with its sigmoid gate; Qwen3-MoE: none, the top-k weights renormalised
    int moe_nw = 0;          // routing weights per layer: k, plus the shared-expert weight on Qwen2-MoE
    const char *moe_name = ""; // the family the MoE refusals name
    b200_moe_config moe{};
    int moe_hv = 0; // units of the virtual hidden vector: shared_hidden_dim + n_experts_used * expert_hidden_dim
    int *moe_ids = nullptr;
    float *moe_w = nullptr, *moe_logits = nullptr;
    unsigned *moe_done = nullptr;
    MoeDownSmem moe_dl{};

    // Granite's µP scales (b200_plan_create_granite); 1.0f for every other family, where each multiply leaves its operand unchanged
    b200_granite_config mup{1.0f, 1.0f, 1.0f, 1.0f};
    // Devstral's YaRN RoPE table (b200_plan_create_devstral with a non-NULL b200_yarn_config); every other plan uses the plain table
    bool has_yarn = false;
    b200_yarn_config yarn{};

    // The prefill modes (B200_PREFILL_*, PREFILL_MODE_NAMES): the active one, and per mode whether its buffers and tensor maps are
    // built or why not.  exact is always ready; b200_set_prefill_mode builds the others (build() an FP16 plan's tensor_core) and
    // selects a mode only once it is ready.
    int pf_mode = B200_PREFILL_EXACT;
    struct PrefillMode { bool ready; const char *why; } pf[5] = {{true, ""}, {false, ""}, {false, ""}, {false, ""}, {false, ""}};
    PrefillCtx prefill; // tensor_core and tensor_core_w8a16 (prefill.cuh)
    PrefillI8Ctx pi8;   // tensor_core_exact and, on MoE plans, tensor_core_exact_moe (prefill_i8.cuh)
    // persistent decode kernel
    bool pd_ok = false;           // the plan fits the kernel's restrictions
    std::string pd_why;           // ... or why not
    PdSmem pd_L{};
    PdLayer *pd_layers = nullptr; // device copies of the per-layer descriptors
    unsigned *pd_sync = nullptr;  // epoch counters, ticks, error word
    unsigned *h_err = nullptr;    // mapped pinned host word written by a timed-out wait
    unsigned *d_err = nullptr;    // its device alias
    unsigned long long *pd_trace = nullptr;
    unsigned pd_flags_off = 0;
    bool pd_coop = true;          // launched with the cooperative attribute (co-residency guaranteed by the driver)

    // batched decode (decode_batch.cuh): n_slots KV caches [slot][layer][ctx][kvDim] and per-row activations, one graph per step
    // form and row count, captured on first use
    struct Batch {
        int n_slots = 0;
        std::vector<void *> allocs;
        float *slot_k = nullptr, *slot_v = nullptr;
        float *x = nullptr, *qkv = nullptr, *hb = nullptr, *logits = nullptr, *xs = nullptr, *hs = nullptr, *att_scratch = nullptr;
        int8_t *xq = nullptr, *hq = nullptr;
        float *part_val = nullptr;
        int *part_idx = nullptr, *ids = nullptr, *smp_out = nullptr;
        unsigned *blk_cnt = nullptr;
        BatchRows *rows = nullptr, *h_rows = nullptr; // device / pinned host
        int *h_out = nullptr;                         // pinned: step_outputs' readback block, 9 ints a row
        // the exact prefills: the per-step rows of the call [context_length], the device step index
        BatchRows *sched = nullptr;
        int *step = nullptr;
        int *smp_indices = nullptr; // the sampler's candidate lists, [row][vocab]
        Graph g[STEP_FORMS][SMB_MAX_ROWS + 1][SMB_MAX_ROWS + 1]; // [form][rows][rows that run the classifier]
        int last_launches = 0; // of the last step with the classifier (batch_step)
        float last_ms = 0.f;
    } bt;

    // b200_score_tokens (score.cuh): the call's targets and per-row results on the device (cap rows, allocated on the first call);
    // tensor_core_exact adds the classifier's maps and a logits scratch of SCORE_GROUP_ROWS rows of ldl floats
    struct Score {
        int cap = 0;
        int *tgt = nullptr;
        ScoreOut *out = nullptr;
        float *logits = nullptr;
        int ldl = 0;
        CUtensorMap cls_q, cls_s;
    } sc;

    // b200_set_logprobs (logprobs.cuh): top_n < 0 is off.  While on, each emitting call runs k_token_logprobs on its rows after its
    // graph into out (cap rows) and copies them to the pinned h_out inside its synchronise; smp holds the copies of sampled rows
    // that the sampler turns into probabilities (SMB_MAX_ROWS padded rows), so k_token_logprobs reads the untouched logits
    struct Logprobs {
        int top_n = -1, cap = 0, rows = 0;
        LogprobRow *out = nullptr, *h_out = nullptr;
        float *smp = nullptr;
    } lp;

    // b200_set_sampling_controls (sampler.cuh, k_sample_ctl): sequence s = slot + 1 (s = 0: the plan's own cache).  The host keeps
    // each sequence's controls; the device buffers are allocated by the first call that sets controls and hold a row for every
    // sequence the plan can address, so b200_set_decode_slots never reallocates them.  rows: the modified rows of one call.
    struct Controls {
        bool on[SMB_MAX_ROWS + 1] = {};
        b200_sampling_controls c[SMB_MAX_ROWS + 1] = {}; // bias pointers cleared: the list lives in bias_id / bias_val
        float min_p_log[SMB_MAX_ROWS + 1] = {};
        int *cnt = nullptr;        // [sequence][vocab]
        int *bias_id = nullptr;    // [sequence][B200_MAX_LOGIT_BIAS]
        float *bias_val = nullptr; // [sequence][B200_MAX_LOGIT_BIAS]
        float *rows = nullptr;     // [SMB_MAX_ROWS][sampler_padded(vocab)]
    } ctl;
};

namespace {

int fail(b200_plan *p, int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (p) p->err = buf;
    return code;
}

#define CK(call)                                                                                     \
    do {                                                                                             \
        cudaError_t e_ = (call);                                                                     \
        if (e_ != cudaSuccess)                                                                       \
            return fail(p, e_ == cudaErrorMemoryAllocation ? B200_ERR_OOM : B200_ERR_CUDA, "%s: %s (%s:%d)", #call, \
                        cudaGetErrorString(e_), __FILE__, __LINE__);                                 \
    } while (0)

// Largest dynamic shared memory a kernel may ask for = the device opt-in limit minus the kernel's own static shared memory.
template <typename K> cudaError_t set_max_dyn(K kern, int maxdyn) {
    cudaFuncAttributes fa;
    cudaError_t e = cudaFuncGetAttributes(&fa, kern);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, maxdyn - (int)fa.sharedSizeBytes);
}

// f(std::integral_constant<int, HS>()) for a head size the decode attention kernels are compiled for (k_attention,
// k_attention_batch, k_rope_kv_batch, k_attention_cached_rows); build() refuses every other size.
template <typename F> int with_decode_head_size(b200_plan *p, int hs, F &&f) {
    switch (hs) {
    case 32: return f(std::integral_constant<int, 32>());
    case 64: return f(std::integral_constant<int, 64>());
    case 96: return f(std::integral_constant<int, 96>());
    case 128: return f(std::integral_constant<int, 128>());
    case 256: return f(std::integral_constant<int, 256>());
    }
    return fail(p, B200_ERR_UNSUPPORTED, "head size %d has no decode attention kernel", hs);
}

// The same for the sizes of the tensor-core prefill attention (k_pf_*) and the persistent decode kernel.
template <typename F> int with_mma_head_size(b200_plan *p, int hs, F &&f) {
    switch (hs) {
    case 64: return f(std::integral_constant<int, 64>());
    case 128: return f(std::integral_constant<int, 128>());
    }
    return fail(p, B200_ERR_UNSUPPORTED, "head size %d has no tensor-core prefill or persistent decode kernel", hs);
}

template <typename T> int dalloc(b200_plan *p, T **ptr, size_t n_bytes) {
    void *d = nullptr;
    if (n_bytes == 0) n_bytes = 16;
    CK(cudaMalloc(&d, n_bytes));
    p->allocs.push_back(d);
    p->bytes += (int64_t)n_bytes;
    *ptr = reinterpret_cast<T *>(d);
    return B200_OK;
}

void par_memcpy(void *dst, const void *src, size_t n, int threads) {
    if (threads <= 1 || n < (size_t)(4u << 20)) { memcpy(dst, src, n); return; }
    std::vector<std::thread> th;
    const size_t per = ((n + threads - 1) / threads + 4095) & ~(size_t)4095;
    for (int i = 0; i < threads; i++) {
        const size_t o = (size_t)i * per;
        if (o >= n) break;
        const size_t m = n - o < per ? n - o : per;
        th.emplace_back([=] { memcpy((unsigned char *)dst + o, (const unsigned char *)src + o, m); });
    }
    for (auto &t : th) t.join();
}

int up_init(b200_plan *p, size_t dst_bytes) {
    Uploader &u = p->up;
    const char *t = getenv("B200_UPLOAD_THREADS");
    u.threads = t ? atoi(t) : 4;
    u.pin_bytes = (size_t)64 << 20;
    u.dst_bytes = dst_bytes;
    CK(cudaStreamCreateWithFlags(&u.copy, cudaStreamNonBlocking));
    for (int i = 0; i < 2; i++) {
        CK(cudaHostAlloc((void **)&u.pin[i], u.pin_bytes, cudaHostAllocDefault));
        CK(cudaMalloc((void **)&u.dst[i], dst_bytes));
        CK(cudaEventCreateWithFlags(&u.pin_done[i], cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&u.d_ready[i], cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&u.d_free[i], cudaEventDisableTiming));
    }
    return B200_OK;
}

void up_destroy(b200_plan *p) {
    Uploader &u = p->up;
    if (u.copy) cudaStreamSynchronize(u.copy);
    for (int i = 0; i < 2; i++) {
        if (u.pin[i]) cudaFreeHost(u.pin[i]);
        if (u.dst[i]) cudaFree(u.dst[i]);
        if (u.pin_done[i]) cudaEventDestroy(u.pin_done[i]);
        if (u.d_ready[i]) cudaEventDestroy(u.d_ready[i]);
        if (u.d_free[i]) cudaEventDestroy(u.d_free[i]);
        u.pin[i] = nullptr; u.dst[i] = nullptr; u.pin_done[i] = u.d_ready[i] = u.d_free[i] = nullptr;
    }
    if (u.copy) cudaStreamDestroy(u.copy);
    u.copy = nullptr;
}

// host bytes -> device, through the pinned double buffer, on the copy stream (asynchronous with respect to the caller except
// for the wait on a pinned buffer still in flight)
int up_h2d(b200_plan *p, void *dst, const void *src, size_t bytes) {
    Uploader &u = p->up;
    for (size_t o = 0; o < bytes; o += u.pin_bytes) {
        const size_t n = bytes - o < u.pin_bytes ? bytes - o : u.pin_bytes;
        const int i = u.pi;
        if (u.pin_used[i]) CK(cudaEventSynchronize(u.pin_done[i]));
        const auto t0 = std::chrono::steady_clock::now();
        par_memcpy(u.pin[i], (const unsigned char *)src + o, n, u.threads);
        u.host_copy_s += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        CK(cudaMemcpyAsync((unsigned char *)dst + o, u.pin[i], n, cudaMemcpyHostToDevice, u.copy));
        CK(cudaEventRecord(u.pin_done[i], u.copy));
        u.pin_used[i] = true;
        u.pi ^= 1;
        u.h2d_bytes += (int64_t)n;
    }
    return B200_OK;
}
// device staging buffer protocol: begin (copy stream waits until the repack that last read this buffer is done) -> h2d... ->
// ready (plan stream waits for the copies) -> [repack kernel on the plan stream] -> release
int up_stage_begin(b200_plan *p, unsigned char **stage) {
    Uploader &u = p->up;
    if (u.d_used[u.di]) CK(cudaStreamWaitEvent(u.copy, u.d_free[u.di], 0));
    *stage = u.dst[u.di];
    return B200_OK;
}
int up_stage_ready(b200_plan *p) {
    Uploader &u = p->up;
    CK(cudaEventRecord(u.d_ready[u.di], u.copy));
    CK(cudaStreamWaitEvent(p->stream, u.d_ready[u.di], 0));
    return B200_OK;
}
int up_stage_release(b200_plan *p) {
    Uploader &u = p->up;
    CK(cudaEventRecord(u.d_free[u.di], p->stream));
    u.d_used[u.di] = true;
    u.di ^= 1;
    return B200_OK;
}

// GGUF Q8_0 blocks (f16 scale + 32 int8, 34 bytes, GGMLType.java:13) -> split planes.
// One thread per 16-bit word of the raw stream: word 0 of each block is the scale.
__global__ void k_repack_q8(const uint16_t *__restrict__ raw, uint16_t *__restrict__ qs, uint16_t *__restrict__ sc,
                            size_t n_words) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_words) return;
    size_t blk = i / 17;
    int w = (int)(i % 17);
    uint16_t v = raw[i];
    if (w == 0) sc[blk] = v;
    else qs[blk * 16 + (w - 1)] = v;
}

const b200_tensor *find(const b200_tensor *t, int n, const std::string &name) {
    for (int i = 0; i < n; i++)
        if (name == t[i].name) return &t[i];
    return nullptr;
}

int64_t n_elems(const b200_tensor *t) {
    int64_t n = 1;
    for (int i = 0; i < t->n_dims; i++) n *= t->dims[i];
    return n;
}

static inline int eff_type(int t) { return kq_is_kquant(t) ? B200_GGML_Q8_0 : t; } // AbstractModelLoader.effectiveGpuWeightType (:58-64)

// Upload rows [0, rows) of a [rows][cols] GGUF matrix into dst at row offset `row_off`.  K-quant sources are re-quantised to Q8_0 on
// the device (kquant.cuh) between the copy and the repack.
int upload_matrix(b200_plan *p, const b200_tensor *t, int rows, int cols, DevMat &dst, int row_off, int src_row = 0,
                  int src_full_rows = -1) { // rows [src_row, src_row + rows) of a source tensor with src_full_rows rows (Phi-3's fused wqkv / gate-up)
    if (!t) return fail(p, B200_ERR_BAD_ARG, "missing tensor");
    if (src_full_rows < 0) src_full_rows = rows;
    if (n_elems(t) != (int64_t)src_full_rows * cols || src_row < 0 || src_row + rows > src_full_rows)
        return fail(p, B200_ERR_BAD_ARG, "tensor %s has %lld elements, expected %lld", t->name, (long long)n_elems(t),
                    (long long)src_full_rows * cols);
    const size_t src_row_bytes = kq_is_kquant(t->ggml_type) ? (size_t)cols / 256 * kq_block_bytes(t->ggml_type)
                                 : t->ggml_type == B200_GGML_Q8_0 ? (size_t)cols / 32 * 34 : (size_t)cols * (t->ggml_type == B200_GGML_F16 ? 2 : 4);
    const unsigned char *tdata = (const unsigned char *)t->data + (size_t)src_row * src_row_bytes;
    if (eff_type(t->ggml_type) != dst.type)
        return fail(p, B200_ERR_UNSUPPORTED, "tensor %s has ggml type %d, plan weight type is %d", t->name, t->ggml_type,
                    dst.type);
    if (dst.type == B200_GGML_Q8_0) {
        const bool kq = kq_is_kquant(t->ggml_type);
        if (kq && (cols % 256 || !p->kq_off)) return fail(p, B200_ERR_BAD_ARG, "K-quant tensor %s: rows must be multiples of 256 elements", t->name);
        const size_t kb = kq ? (size_t)kq_block_bytes(t->ggml_type) : 0;
        size_t nblk = (size_t)rows * cols / 32;
        int8_t *qs = (int8_t *)dst.qs + (size_t)row_off * cols;
        __half *sc = (__half *)dst.sc + (size_t)row_off * (cols / 32);
        // chunked through the staging buffer (multiple of 34 bytes; of 8 blocks = one super-block for K-quants)
        const size_t q8_area = p->kq_off ? p->kq_off : p->up.dst_bytes;
        size_t blk_per_chunk = (q8_area / 34) & ~(size_t)7;
        for (size_t b0 = 0; b0 < nblk; b0 += blk_per_chunk) {
            size_t nb = nblk - b0 < blk_per_chunk ? nblk - b0 : blk_per_chunk;
            const unsigned char *hsrc = kq ? tdata + b0 / 8 * kb : tdata + b0 * 34;
            const size_t hbytes = kq ? nb / 8 * kb : nb * 34;
            int rc;
            unsigned char *stage = nullptr;
            if ((rc = up_stage_begin(p, &stage))) return rc;
            if ((rc = up_h2d(p, stage + (kq ? p->kq_off : 0), hsrc, hbytes))) return rc;
            if ((rc = up_stage_ready(p))) return rc;
            if (kq) CK(launch_requant_kquant(t->ggml_type, stage + p->kq_off, stage, (long long)nb, p->stream));
            size_t words = nb * 17;
            k_repack_q8<<<(unsigned)((words + 255) / 256), 256, 0, p->stream>>>((const uint16_t *)stage, (uint16_t *)(qs + b0 * 32),
                                                                                  (uint16_t *)(sc + b0), words);
            CK(cudaGetLastError());
            if ((rc = up_stage_release(p))) return rc;
        }
    } else {
        size_t esz = dst.type == B200_GGML_F16 ? 2 : 4;
        return up_h2d(p, (uint8_t *)dst.qs + (size_t)row_off * cols * esz, tdata, (size_t)rows * cols * esz); // ordered by the final synchronize
    }
    return B200_OK;
}

const size_t SMV_SMEM_BUDGET_MAX = 96 * 1024;

// Segments, unit size and format of a tile-major stream (fmt 0: Q8_0 tiles; a K-quant type: resident tiles).
TileMat tile_geometry(int rows, int cols, int fmt) {
    TileMat t{};
    t.rows = rows;
    t.cols = cols;
    t.fmt = fmt;
    t.nseg = smv_pick_nseg(cols, fmt ? 256 : 32);
    t.seg = t.nseg ? cols / t.nseg : 0;
    t.unit_bytes = smv_unit_bytes(t.seg, fmt);
    return t;
}
int64_t tile_bytes(const TileMat &t) { return (int64_t)tile_groups(t) * 4 * t.nseg * t.unit_bytes; }

// ---- ring sizes of the decode weight streams (DESIGN.md section 5a) -----------------------------------------------------------
// Under PDL the next kernel of the chain becomes resident while its predecessor still runs, and a stream kernel's producer fills
// its ring before the dependency wait returns.  During the chain's latency phases (the fused norm's exact sum, the attention) the
// resident rings are all that keep HBM busy, so a ring is sized for the kernels it must stay resident beside: its CTA and each
// neighbour's, with a per-CTA reserve each, within the SM's shared memory.  QKV sits between W2 (before it) and the attention
// (after it); gate/up between Wo and W2.  Wo, W2 and lm_head keep SMV_SMEM_BUDGET_MAX, which is also the floor of every budget
// and what the shape checks use, so a device with less shared memory refuses no plan it ran before.
struct SmDev {
    size_t sm, reserve, optin; // shared memory per SM, reserved per resident CTA, opt-in limit per CTA
};

size_t stream_smem(const TileMat &W, bool norm, size_t budget) {
    unsigned a, b;
    return (norm ? smv_layout_norm(W.cols, W.seg, budget, &a, &b, W.fmt) : smv_layout(W.cols, W.seg, budget, W.fmt)).total;
}
int slice_tiles(const TileMat &W, int n_sms) { return (tile_groups(W) + n_sms - 1) / n_sms * W.nseg; } // the largest CTA slice

// The budget of stream W between CTAs that take `before` and `after` bytes of shared memory: as many stages as fit beside the
// larger of the two, but no more than its largest CTA slice (a stage it never fills would only crowd out its neighbours).
size_t ring_budget(const SmDev &d, const TileMat &W, bool norm, int n_sms, size_t before, size_t after) {
    const size_t nb = (before > after ? before : after) + 2 * d.reserve;
    size_t room = d.sm > nb ? d.sm - nb : 0;
    if (room > d.optin) room = d.optin;
    if (room <= SMV_SMEM_BUDGET_MAX) return SMV_SMEM_BUDGET_MAX;
    unsigned a, b;
    const SmvSmem L = norm ? smv_layout_norm(W.cols, W.seg, room, &a, &b, W.fmt) : smv_layout(W.cols, W.seg, room, W.fmt);
    const int s = L.stages < slice_tiles(W, n_sms) ? L.stages : slice_tiles(W, n_sms);
    const size_t need = L.off_ring + (size_t)s * L.stage_bytes;
    return need > SMV_SMEM_BUDGET_MAX ? need : SMV_SMEM_BUDGET_MAX;
}

// The streams that open with a latency phase get the larger rings: QKV (the attention norm's exact sum) between W2 of layer prev
// (l - 1; layer 0 takes its own) and the attention (att bytes), and gate/up (the FFN norm's) between Wo and W2.  Their neighbours
// keep SMV_SMEM_BUDGET_MAX: a larger Wo would keep gate/up from entering beside it, and measured slower (DESIGN.md section 6).
// norm: the plan's QKV and gate/up compute their RMSNorm (k_stream_matvec_q8_norm).
void ring_budgets(const SmDev &d, int n_sms, bool norm, size_t att, const LayerW &prev, LayerW &L) {
    // a Qwen2-MoE layer has no tw2 / tgu: its down and gate/up streams (moe.cuh) take at most SMV_SMEM_BUDGET_MAX
    auto at_floor = [](const TileMat &W, bool nrm) { return W.nseg ? stream_smem(W, nrm, SMV_SMEM_BUDGET_MAX) : SMV_SMEM_BUDGET_MAX; };
    L.ring_qkv = ring_budget(d, L.tqkv, norm, n_sms, at_floor(prev.tw2, false), att);
    L.ring_gu = L.tgu.nseg ? ring_budget(d, L.tgu, norm, n_sms, at_floor(L.two, false), at_floor(L.tw2, false)) : SMV_SMEM_BUDGET_MAX;
}

// The format a stream of these stacked sources keeps on a resident plan: their common K-quant type when every present source has
// it and the resident layout leaves at least 3 ring stages; else 0 (the stream is re-quantised to Q8_0 tiles at upload).
int resident_fmt(const b200_tensor *const ts[3], const int rs[3], int rows, int cols) {
    int fmt = -1;
    for (int k = 0; k < 3; k++) {
        if (!rs[k]) continue;
        if (!ts[k] || !kq_is_kquant(ts[k]->ggml_type) || (fmt >= 0 && ts[k]->ggml_type != fmt)) return 0;
        fmt = ts[k]->ggml_type;
    }
    if (fmt < 0 || cols % 256) return 0;
    const TileMat t = tile_geometry(rows, cols, fmt);
    return t.nseg && smv_layout(cols, t.seg, SMV_SMEM_BUDGET_MAX, fmt).stages >= 3 ? fmt : 0;
}

// Upload up to three stacked GGUF Q8_0 or K-quant matrices (or the gate/up pair) into tile-major layout: Q8_0 tiles, or on a
// resident plan resident tiles when resident_fmt allows.
int upload_tiles(b200_plan *p, const b200_tensor *t0, const b200_tensor *t1, const b200_tensor *t2, int r0, int r1, int r2, int cols,
                 bool gateup, TileMat &out, const int *row0 = nullptr, const int *full = nullptr) {
    const b200_tensor *ts[3] = {t0, t1, t2};
    int rs[3] = {r0, r1, r2};
    const int rows = gateup ? r0 + r1 : r0 + r1 + r2;
    const int fmt = p->resident ? resident_fmt(ts, rs, rows, cols) : 0;
    RepackSrc src;
    size_t off = 0;
    int rc;
    unsigned char *stage = nullptr;
    if ((rc = up_stage_begin(p, &stage))) return rc;
    const size_t stage_bytes = p->up.dst_bytes;
    const size_t q8_area = p->kq_off ? p->kq_off : stage_bytes;
    size_t roff = 0; // cursor inside the raw (K-quant) area
    struct Requant { int type; const unsigned char *raw; unsigned char *q8; long long nblk; } rq[3];
    int n_rq = 0;
    for (int k = 0; k < 3; k++) {
        src.raw[k] = nullptr;
        src.rows[k] = rs[k];
        src.row0[k] = 0; // only this rank's row range [row0, row0 + rows) crosses PCIe (rows are contiguous in GGUF)
        if (rs[k] == 0) continue;
        const int full_rows = full ? full[k] : rs[k];
        const int first = row0 ? row0[k] : 0;
        const b200_tensor *t = ts[k];
        if (!t) return fail(p, B200_ERR_BAD_ARG, "missing tensor");
        const bool kq = kq_is_kquant(t->ggml_type);
        if (t->ggml_type != B200_GGML_Q8_0 && !kq) return fail(p, B200_ERR_UNSUPPORTED, "tensor %s has ggml type %d, plan weight type is Q8_0", t->name, t->ggml_type);
        if (kq && (cols % 256 || !p->kq_off)) return fail(p, B200_ERR_BAD_ARG, "K-quant tensor %s: rows must be multiples of 256 elements", t->name);
        if (n_elems(t) != (int64_t)full_rows * cols) return fail(p, B200_ERR_BAD_ARG, "tensor %s has %lld elements, expected %lld", t->name, (long long)n_elems(t), (long long)full_rows * cols);
        if (first < 0 || first + rs[k] > full_rows) return fail(p, B200_ERR_BAD_ARG, "row range of tensor %s out of bounds", t->name);
        // resident: the K-quant rows are staged as they are, and the repack copies them
        const size_t row_bytes = fmt ? (size_t)cols / 256 * kq_block_bytes(fmt) : (size_t)cols / 32 * 34, nbytes = (size_t)rs[k] * row_bytes;
        if (off + nbytes > q8_area) return fail(p, B200_ERR_STATE, "staging buffer too small");
        if (kq && !fmt) { // the K-quant bytes land in the raw area; the Q8_0 blocks are produced on the device once the copies are in
            const size_t raw_row = (size_t)cols / 256 * kq_block_bytes(t->ggml_type), raw_bytes = (size_t)rs[k] * raw_row;
            const unsigned char *hsrc = (const unsigned char *)t->data + (size_t)first * raw_row;
            if (p->kq_off + roff + raw_bytes > stage_bytes) return fail(p, B200_ERR_STATE, "staging buffer too small");
            unsigned char *rdst = stage + p->kq_off + roff;
            if ((rc = up_h2d(p, rdst, hsrc, raw_bytes))) return rc;
            rq[n_rq++] = Requant{t->ggml_type, rdst, stage + off, (long long)rs[k] * (cols / 32)};
            roff += (raw_bytes + 255) & ~(size_t)255;
        } else {
            const unsigned char *hsrc = (const unsigned char *)t->data + (size_t)first * row_bytes;
            if ((rc = up_h2d(p, stage + off, hsrc, nbytes))) return rc;
        }
        src.raw[k] = stage + off;
        off += (nbytes + 255) & ~(size_t)255;
    }
    if ((rc = up_stage_ready(p))) return rc;
    for (int i = 0; i < n_rq; i++) CK(launch_requant_kquant(rq[i].type, rq[i].raw, rq[i].q8, rq[i].nblk, p->stream));
    src.gateup = gateup ? 1 : 0;
    out = tile_geometry(rows, cols, fmt);
    const size_t stored_rows = (size_t)tile_groups(out) * 4; // whole 4-row groups: a ragged classifier gets zero padding rows
    unsigned char *d;
    rc = dalloc(p, &d, (size_t)tile_bytes(out));
    if (rc) return rc;
    out.base = d;
    if (fmt) k_repack_kq_tiles<<<(unsigned)(stored_rows * out.nseg), 128, 0, p->stream>>>(src, d, rows, cols, out.seg, out.nseg, out.unit_bytes, kq_block_bytes(fmt));
    else k_repack_tiles<<<(unsigned)(stored_rows * out.nseg), 128, 0, p->stream>>>(src, d, rows, cols, out.seg, out.nseg, out.unit_bytes);
    CK(cudaGetLastError());
    return up_stage_release(p);
}

int alloc_matrix(b200_plan *p, DevMat &m, int rows, int cols, int type) {
    m.rows = rows;
    m.cols = cols;
    m.type = type;
    m.sc = nullptr;
    void *q = nullptr;
    int rc;
    if (type == B200_GGML_Q8_0) {
        if ((rc = dalloc(p, (int8_t **)&q, (size_t)rows * cols))) return rc;
        __half *s;
        if ((rc = dalloc(p, &s, (size_t)rows * (cols / 32) * 2))) return rc;
        m.sc = s;
    } else {
        if ((rc = dalloc(p, (uint8_t **)&q, (size_t)rows * cols * (type == B200_GGML_F16 ? 2 : 4)))) return rc;
    }
    m.qs = q;
    return B200_OK;
}

int upload_f32(b200_plan *p, const b200_tensor *t, int n, float **dst, const char *what) {
    if (!t) return fail(p, B200_ERR_BAD_ARG, "missing tensor %s", what);
    if (t->ggml_type != B200_GGML_F32) return fail(p, B200_ERR_UNSUPPORTED, "tensor %s must be F32", what);
    if (n_elems(t) != n) return fail(p, B200_ERR_BAD_ARG, "tensor %s has wrong size", what);
    int rc = dalloc(p, dst, (size_t)n * 4);
    if (rc) return rc;
    CK(cudaMemcpy(*dst, t->data, (size_t)n * 4, cudaMemcpyHostToDevice));
    return B200_OK;
}

// Qwen2's blk.N.attn_{q,k,v}.bias (F32, one dimension of qd / kvd / kvd floats) as one packed q|k|v vector of this rank's heads:
// q rows rank * qd_l .., k and v rows rank * kvd_l .. (the biases are row-sharded with the heads, like the matrices).
int upload_qkv_bias(b200_plan *p, const b200_tensor *tensors, int n_tensors, int layer, float **dst) {
    const std::string pre = "blk." + std::to_string(layer) + ".";
    const char *names[3] = {"attn_q.bias", "attn_k.bias", "attn_v.bias"};
    const int full[3] = {p->qd, p->kvd, p->kvd}, local[3] = {p->qd_l, p->kvd_l, p->kvd_l};
    std::vector<float> h((size_t)p->qd_l + 2 * p->kvd_l);
    size_t o = 0;
    for (int i = 0; i < 3; i++) {
        const std::string name = pre + names[i];
        const b200_tensor *t = find(tensors, n_tensors, name);
        if (!t) return fail(p, B200_ERR_BAD_ARG, "missing tensor %s", name.c_str());
        if (t->ggml_type != B200_GGML_F32) return fail(p, B200_ERR_UNSUPPORTED, "tensor %s must be F32 (ggml type %d)", name.c_str(), t->ggml_type);
        if (t->n_dims != 1 || t->dims[0] != full[i] || !t->data)
            return fail(p, B200_ERR_BAD_ARG, "tensor %s must have one dimension of %d floats (n_dims %d, dims[0] %lld)", name.c_str(), full[i], t->n_dims,
                        (long long)(t->n_dims > 0 ? t->dims[0] : 0));
        memcpy(h.data() + o, (const float *)t->data + (size_t)p->tp.rank * local[i], (size_t)local[i] * 4);
        o += local[i];
    }
    int rc = dalloc(p, dst, h.size() * 4);
    if (rc) return rc;
    CK(cudaMemcpy(*dst, h.data(), h.size() * 4, cudaMemcpyHostToDevice));
    return B200_OK;
}

// Output scale of a STORE / RESID epilogue: Granite's residualScale on the Wo / W2 branch, its logitScale on the classifier, else 1.
float out_scale(const b200_plan *p, bool resid, bool classifier) { return resid ? p->mup.residual_scale : classifier ? p->mup.logit_scale : 1.0f; }
// The attention kernels' score argument: the divisor sqrt(head size), or (KF_ATTSCALE) Granite's attentionScale multiplier.
float att_score_arg(const b200_plan *p) { return (p->kflags & KF_ATTSCALE) ? p->mup.attention_scale : (float)sqrt((double)p->cfg.head_size); }

size_t f16_smem_bytes(int cols, int lanes) {
    int L = lanes > 0 ? lanes : 1;
    return (size_t)cols * 4 + (size_t)8 * (32 / L) * 256 * 2;
}

template <int MODE> int launch_matvec_f16(b200_plan *p, const DevMat &m, const float *x, float *out) {
    int L = p->cfg.fp16_lanes > 0 ? p->cfg.fp16_lanes : 1;
    int rw = 32 / L;
    int warps = (m.rows + rw - 1) / rw;
    int ctas = (warps + 7) / 8;
    k_matvec_f16<MODE><<<ctas, 256, f16_smem_bytes(m.cols, p->cfg.fp16_lanes), p->stream>>>((const __half *)m.qs, x, m.rows,
                                                                                            m.cols, p->cfg.fp16_lanes, out,
                                                                                            out_scale(p, MODE == MODE_RESID, &m == &p->out));
    CK(cudaGetLastError());
    return B200_OK;
}

// FP16 plans on the streaming path (stream_matvec_f16.cuh); m2 = ffn_up for SF_GATEUP.
template <typename... KA, typename... A> int launch_k(b200_plan *p, bool pdl, void (*kern)(KA...), dim3 grid, dim3 block, size_t smem, A... args);
int sf_grid(int n_sms, int lanes, int rows, int cols, bool gateup) { // CTAs of an FP16 streaming launch
    const SfLayout L = sf_layout(rows, cols, lanes, gateup);
    const int rw = 64 / lanes, mr = gateup ? rw / 2 : rw;
    const int grid = L.ctas_per_sm * n_sms;
    const int groups = (rows + mr - 1) / mr; // a ragged classifier ends in a partial group
    return grid > groups ? groups : grid;
}
template <int MODE> int launch_stream_f16(b200_plan *p, const DevMat &m, const DevMat *m2, const float *x, float *out, TraceBuf tr = TraceBuf{nullptr, 0, 0},
                                          bool argmax = false) {
    const int lanes = p->cfg.fp16_lanes;
    const SfLayout L = sf_layout(m.rows, m.cols, lanes, MODE == SF_GATEUP);
    if (!L.ok) return fail(p, B200_ERR_STATE, "f16 streaming layout does not fit %d x %d", m.rows, m.cols);
    SfArgs a;
    a.w0 = (const __half *)m.qs; a.w1 = m2 ? (const __half *)m2->qs : nullptr; a.x = x; a.out = out; a.rows = m.rows; a.cols = m.cols;
    a.oscale = out_scale(p, MODE == SF_RESID, &m == &p->out);
    a.seg = L.seg; a.nseg = L.nseg; a.stages = L.stages; a.tr = tr;
    a.part_val = argmax ? p->part_val : nullptr;
    a.part_idx = argmax ? p->part_idx : nullptr;
    const int grid = sf_grid(p->n_sms, lanes, m.rows, m.cols, MODE == SF_GATEUP);
    if (lanes == 16) return launch_k(p, p->use_pdl, k_stream_matvec_f16<16, MODE>, dim3(grid), dim3(SF_THREADS), L.total, a);
    return launch_k(p, p->use_pdl, k_stream_matvec_f16<8, MODE>, dim3(grid), dim3(SF_THREADS), L.total, a);
}

// Kernel launch with the programmatic-dependent-launch attribute (captured into the CUDA graph as
// a programmatic edge): the kernel may become resident while its predecessor is still running.
template <typename... KA, typename... A>
cudaError_t launch_on(cudaStream_t stream, bool pdl, void (*kern)(KA...), dim3 grid, dim3 block, size_t smem, A... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KA>(args)...);
}
template <typename... KA, typename... A>
int launch_k(b200_plan *p, bool pdl, void (*kern)(KA...), dim3 grid, dim3 block, size_t smem, A... args) {
    CK(launch_on(p->stream, pdl, kern, grid, block, smem, args...));
    return B200_OK;
}

// Read ONCE per plan (b200_plan_create), never inside a launch helper.
void read_knobs(b200_plan *p) {
    const char *d = getenv("B200_DECODE");
    // default: the CUDA graph, which every plan can run (on one H100, with the fused norm, it measured ~2.5 % faster than the persistent kernel for 8B Q8_0, DESIGN.md section 6).  B200_DECODE=persistent or b200_set_decode_mode select the one-kernel-per-token path.
    p->decode_mode = (d && !strcmp(d, "persistent")) ? B200_DECODE_PERSISTENT : B200_DECODE_GRAPH;
}

// The stream kernels of a tile format (TileMat::fmt): the Q8_0 kernels, or their resident K-quant instantiations.
template <int MODE> void (*smv_kernel(int fmt))(SmvArgs, SmvSmem) {
    switch (fmt) {
    case B200_GGML_Q4_K: return k_stream_matvec_kq<MODE, B200_GGML_Q4_K>;
    case B200_GGML_Q5_K: return k_stream_matvec_kq<MODE, B200_GGML_Q5_K>;
    case B200_GGML_Q6_K: return k_stream_matvec_kq<MODE, B200_GGML_Q6_K>;
    }
    return k_stream_matvec_q8<MODE>;
}
template <int MODE> void (*smv_norm_kernel(int fmt))(SmvArgs, SmvSmem, SmvNormArgs) {
    switch (fmt) {
    case B200_GGML_Q4_K: return k_stream_matvec_kq_norm<MODE, B200_GGML_Q4_K>;
    case B200_GGML_Q5_K: return k_stream_matvec_kq_norm<MODE, B200_GGML_Q5_K>;
    case B200_GGML_Q6_K: return k_stream_matvec_kq_norm<MODE, B200_GGML_Q6_K>;
    }
    return k_stream_matvec_q8_norm<MODE>;
}

template <int MODE>
int launch_stream(b200_plan *p, const TileMat &W, size_t budget, const int8_t *xq, const float *xs, float *out, int8_t *hq, float *hs, bool argmax = false,
                  TraceBuf tr = TraceBuf{nullptr, 0, 0}, int wait_slot = -1, unsigned wait_op = 0, int out_slot = -1, unsigned out_op = 0,
                  int row_base = 0) {
    SmvSmem L = smv_layout(W.cols, W.seg, budget, W.fmt);
    SmvArgs a;
    a.W = W; a.xq = xq; a.xs = xs; a.out = out; a.hq = hq; a.hs = hs; a.blk_cnt = p->blk_cnt;
    a.oscale = out_scale(p, MODE == SMV_RESID, &W == &p->tout);
    a.part_val = argmax ? p->part_val : nullptr;
    a.part_idx = argmax ? p->part_idx : nullptr;
    a.tr = tr;
    a.tp = p->tp;
    a.wait_slot = wait_slot; a.wait_op = wait_op; a.out_slot = out_slot; a.out_op = out_op; a.row_base = row_base;
    return launch_k(p, p->use_pdl, smv_kernel<MODE>(W.fmt), dim3(p->n_sms), dim3(SMV_THREADS), L.total, a, L);
}

// A stream kernel behind a fused RMSNorm of the residual stream x (weights w; from_emb: layer 0, the embedding row, which CTA 0
// also writes to x).  MODE is SMV_STORE (QKV, lm_head) or SMV_GATEUP.
template <int MODE>
int launch_stream_norm(b200_plan *p, const TileMat &W, size_t budget, const float *w, bool from_emb, float *out, int8_t *hq, float *hs, bool argmax, TraceBuf tr,
                       int row_base = 0) {
    SmvNormArgs n;
    const SmvSmem L = smv_layout_norm(W.cols, W.seg, budget, &n.off_sq, &n.off_seq, W.fmt);
    n.x = p->x; n.w = w; n.st = p->st; n.emb = p->emb; n.emb_scale = p->mup.embedding_scale; n.eps = p->cfg.rms_norm_eps;
    n.from_emb = from_emb ? 1 : 0; n.x_out = p->x;
    SmvArgs a;
    a.W = W; a.xq = nullptr; a.xs = nullptr; a.out = out; a.hq = hq; a.hs = hs; a.blk_cnt = p->blk_cnt;
    a.oscale = out_scale(p, false, &W == &p->tout);
    a.part_val = argmax ? p->part_val : nullptr;
    a.part_idx = argmax ? p->part_idx : nullptr;
    a.tr = tr;
    a.tp = p->tp;
    a.wait_slot = -1; a.wait_op = 0; a.out_slot = -1; a.out_op = 0; a.row_base = row_base;
    return launch_k(p, p->use_pdl, smv_norm_kernel<MODE>(W.fmt), dim3(p->n_sms), dim3(SMV_THREADS), L.total, a, L, n);
}

// The fused norm needs 256 x ceil(dim / 256) squares and the accumulator's scratch next to the ring: at least 3 stages must remain.
bool norm_fusion_ok(int dim) {
    const int nseg = smv_pick_nseg(dim);
    if (!nseg || dim % 32 || dim > 5 * 4 * 256) return false; // at most 5 slots of 16 bytes per consumer thread (registers)
    unsigned a, b;
    return smv_layout_norm(dim, dim / nseg, SMV_SMEM_BUDGET_MAX, &a, &b).stages >= 3;
}

bool stream_shape_ok(int rows, int cols) {
    if (rows % 4 || cols % 32) return false;
    int nseg = smv_pick_nseg(cols);
    if (!nseg) return false;
    return smv_layout(cols, cols / nseg, SMV_SMEM_BUDGET_MAX).stages >= 3;
}

bool gateup_fits(int hidden, int n_sms) { // epilogue buffer holds this CTA's hidden units
    return 2 * ((hidden / 2) / n_sms + 1) <= SMV_HVALS;
}

// k_attention's dynamic shared memory: q | k | out | score row (the row lives in a global scratch buffer for long contexts).
size_t att_smem_bytes(int head_size, int ctx, bool scratch) { return (size_t)(3 * head_size + (scratch ? 0 : ctx)) * 4; }

// The FFN half of a Qwen2-MoE or Qwen3-MoE layer (moe.cuh): the FFN norm (float xb for the F32 router, xq/xs for the experts), the
// router, the (shared +) routed gate/up stream and the down streams with the ordered combine.  Four launches, all under PDL; `tr` is
// the norm's trace record, the three MoE kernels take the next three (trace ids 10, 11, 12).
int enqueue_moe_ffn(b200_plan *p, int l, TraceBuf tr) {
    const b200_config &c = p->cfg;
    const LayerW &L = p->layers[l];
    const int E = p->moe.n_experts, k = p->moe.n_experts_used;
    int rc;
    if ((rc = launch_k(p, p->use_pdl, k_rmsnorm_quant<false>, dim3(1), dim3(NORM_THREADS), norm_smem_bytes(c.dim), p->x, (const StepState *)p->st, p->emb,
                       p->mup.embedding_scale, (const float *)L.ffn_norm, c.rms_norm_eps, c.dim, p->xq, p->xs, p->xb, (long long *)nullptr, tr, p->tp, -1)))
        return rc;
    const bool sh = p->moe_shared;
    int *ids = p->moe_ids + (size_t)l * k;
    float *w = p->moe_w + (size_t)l * p->moe_nw;
    MoeRouteArgs ra;
    ra.router = L.router; ra.shared_gate = L.shared_gate; ra.xb = p->xb; ra.logits = p->moe_logits + (size_t)l * (E + 1); ra.done = p->moe_done + l;
    ra.ids = ids; ra.weights = w; ra.dim = c.dim; ra.n_experts = E; ra.k = k; ra.tr = TraceBuf{tr.rec, tr.slot + 1, 10};
    if ((rc = launch_k(p, p->use_pdl, sh ? k_moe_route : k_routed_route, dim3(sh ? E + 1 : E), dim3(MOE_ROUTE_THREADS), (size_t)c.dim * 4, ra))) return rc;
    MoeStreamArgs a;
    a.S = L.sgu; a.X = L.xgu; a.bases = L.gu_bases; a.ids = ids; a.weights = w; a.k = k;
    a.xq = p->xq; a.xs = p->xs; a.out = p->hb; a.hq = p->hq; a.hs = p->hs; a.blk_cnt = p->blk_cnt; a.tr = TraceBuf{tr.rec, tr.slot + 2, 11};
    const SmvSmem GL = smv_layout(c.dim, (sh ? L.sgu : L.xgu).seg, SMV_SMEM_BUDGET_MAX);
    if ((rc = launch_k(p, p->use_pdl, sh ? k_moe_gateup : k_routed_gateup, dim3(p->n_sms), dim3(SMV_THREADS), GL.total, a, GL))) return rc;
    a.S = L.sdn; a.X = L.xdn; a.bases = L.dn_bases;
    a.xq = p->hq; a.xs = p->hs; a.out = p->x; a.hq = nullptr; a.hs = nullptr; a.blk_cnt = nullptr; a.tr = TraceBuf{tr.rec, tr.slot + 3, 12};
    return launch_k(p, p->use_pdl, sh ? k_moe_down : k_routed_down, dim3(p->n_sms), dim3(SMV_THREADS), p->moe_dl.total, a, p->moe_dl);
}

// Enqueue one single-token forward on p->stream (captured into a CUDA graph at creation).
// with_logits=false is the prefill variant (InferenceCoreBatchPrefillDecode.java:166-167).
int enqueue_forward(b200_plan *p, bool with_logits, int *launches, bool trace = false) {
    const b200_config &c = p->cfg;
    const bool q8 = p->wtype == B200_GGML_Q8_0;
    const bool pdl = p->use_pdl, sf = p->use_f16_stream;
    const bool tpar = p->tp.n > 1;
    const bool fz = p->fuse_norm; // attention / FFN / final norm inside QKV / gate-up / lm_head: 5 launches per layer instead of 7
    int n = 0;
    auto TR = [&](int id) { return TraceBuf{trace ? p->trace_rec : nullptr, n, id}; };
    const size_t norm_smem = norm_smem_bytes(c.dim);
    int8_t *xq = q8 ? p->xq : nullptr;
    float *xs = q8 ? p->xs : nullptr;
    float *xbf = q8 ? nullptr : p->xb;
    const size_t ctx_kv = (size_t)c.context_length * p->kvd_l;
    const int rank = p->tp.rank;
    auto norm = [&](bool embed, const float *w, int wait_op) {
        auto go = [&](auto kern) {
            return launch_k(p, pdl, kern, dim3(1), dim3(NORM_THREADS), norm_smem, p->x, (const StepState *)p->st, p->emb, p->mup.embedding_scale, w, c.rms_norm_eps, c.dim, xq, xs, xbf, (long long *)nullptr, TR(1), p->tp, wait_op);
        };
        return embed ? go(k_rmsnorm_quant<true>) : go(k_rmsnorm_quant<false>);
    };
    for (int l = 0; l < c.n_layers; l++) {
        LayerW &L = p->layers[l];
        int rc;
        // TP flag epochs inside one forward: op = 4*l + {0: attention out, 1: x after Wo, 2: hb, 3: x after W2}
        if (fz) rc = launch_stream_norm<SMV_STORE>(p, L.tqkv, L.ring_qkv, L.attn_norm, l == 0, p->qkv, nullptr, nullptr, false, TR(2)); // attention norm + QKV
        else {
            if ((rc = norm(l == 0, L.attn_norm, l == 0 ? -1 : 4 * (l - 1) + 3))) return rc;
            n++;
            if (q8) rc = launch_stream<SMV_STORE>(p, L.tqkv, L.ring_qkv, p->xq, p->xs, p->qkv, nullptr, nullptr, false, TR(2));
            else if (sf) rc = launch_stream_f16<SF_STORE>(p, L.qkv, nullptr, p->xb, p->qkv, TR(2));
            else rc = launch_matvec_f16<MODE_STORE>(p, L.qkv, p->xb, p->qkv);
        }
        if (rc) return rc; n++;
        float *kc = p->key_cache + (size_t)l * ctx_kv, *vc = p->value_cache + (size_t)l * ctx_kv;
        const size_t att_smem = att_smem_bytes(c.head_size, c.context_length, p->att_scratch != nullptr);
        rc = with_decode_head_size(p, c.head_size, [&](auto HS) {
            return launch_k(p, pdl, k_attention<HS>, dim3(p->nh_l), dim3(ATT_THREADS), att_smem, p->qkv, kc, vc, (const StepState *)p->st,
                            (const float *)p->rope_cr, (const float *)p->rope_ci, p->nh_l, p->nkv_l, p->kflags, (const float *)L.q_norm,
                            (const float *)L.k_norm, (const float *)L.qkv_bias, c.rms_norm_eps, att_score_arg(p), q8 ? p->attq : nullptr, q8 ? p->atts : nullptr, xbf, TR(4),
                            p->tp, (unsigned)(4 * l + 0), rank * p->nh_l, p->att_scratch, c.context_length);
        });
        if (rc) return rc; n++;
        if (q8) rc = launch_stream<SMV_RESID>(p, L.two, SMV_SMEM_BUDGET_MAX, p->attq, p->atts, p->x, nullptr, nullptr, false, TR(5), tpar ? TP_SLOT_ATT : -1, 4 * l + 0, tpar ? TP_SLOT_X : -1, 4 * l + 1, rank * p->dim_l);
        else if (sf) rc = launch_stream_f16<SF_RESID>(p, L.wo, nullptr, p->xb, p->x, TR(5));
        else rc = launch_matvec_f16<MODE_RESID>(p, L.wo, p->xb, p->x);
        if (rc) return rc; n++;
        if (p->is_moe) {
            if ((rc = enqueue_moe_ffn(p, l, TR(1)))) return rc;
            n += 4;
            continue;
        }
        if (!fz) {
            if ((rc = norm(false, L.ffn_norm, 4 * l + 1))) return rc;
            n++;
        }
        if (q8) {
            if (fz) rc = launch_stream_norm<SMV_GATEUP>(p, L.tgu, L.ring_gu, L.ffn_norm, false, p->hb, p->hq, p->hs, false, TR(6)); // FFN norm + gate/up
            else rc = launch_stream<SMV_GATEUP>(p, L.tgu, L.ring_gu, p->xq, p->xs, p->hb, p->hq, p->hs, false, TR(6), -1, 0, tpar ? TP_SLOT_HQ : -1, 4 * l + 2, rank * p->hid_l);
            if (rc) return rc; n++;
            if ((rc = launch_stream<SMV_RESID>(p, L.tw2, SMV_SMEM_BUDGET_MAX, p->hq, p->hs, p->x, nullptr, nullptr, false, TR(7), tpar ? TP_SLOT_HQ : -1, 4 * l + 2, tpar ? TP_SLOT_X : -1, 4 * l + 3, rank * p->dim_l))) return rc; n++;
        } else if (sf) { // gate, up and SwiGLU in one launch; then the down projection
            if ((rc = launch_stream_f16<SF_GATEUP>(p, L.w1, &L.w3, p->xb, p->hb, TR(6)))) return rc; n++;
            if ((rc = launch_stream_f16<SF_RESID>(p, L.w2, nullptr, p->hb, p->x, TR(7)))) return rc; n++;
        } else {
            if ((rc = launch_matvec_f16<MODE_STORE>(p, L.w1, p->xb, p->hb))) return rc; n++;
            if ((rc = launch_matvec_f16<MODE_STORE>(p, L.w3, p->xb, p->hb2))) return rc; n++;
            k_swiglu<<<(c.hidden_dim + 255) / 256, 256, 0, p->stream>>>(p->hb, p->hb2, c.hidden_dim);
            CK(cudaGetLastError()); n++;
            if ((rc = launch_matvec_f16<MODE_RESID>(p, L.w2, p->hb, p->x))) return rc; n++;
        }
    }
    const int last_x_op = 4 * (c.n_layers - 1) + 3;
    if (with_logits) {
        // rmsnorm(x, x, rms_final_weight) then wcls.matmul (InferenceCore.java:167-169)
        int rc;
        if (fz) rc = launch_stream_norm<SMV_STORE>(p, p->tout, SMV_SMEM_BUDGET_MAX, p->out_norm, false, p->logits, nullptr, nullptr, true, TR(8)); // final norm + lm_head
        else {
            if ((rc = norm(false, p->out_norm, last_x_op))) return rc;
            n++;
            if (q8) rc = launch_stream<SMV_STORE>(p, p->tout, SMV_SMEM_BUDGET_MAX, p->xq, p->xs, p->logits, nullptr, nullptr, true, TR(8), -1, 0, -1, 0, rank * p->voc_l);
            else if (sf) rc = launch_stream_f16<SF_STORE>(p, p->out, nullptr, p->xb, p->logits, TR(8), true);
            else rc = launch_matvec_f16<MODE_STORE>(p, p->out, p->xb, p->logits);
        }
        if (rc) return rc; n++;
    }
    {
        int rc;
        if ((rc = launch_k(p, pdl, k_argmax_advance, dim3(1), dim3(1024), (size_t)0, (const float *)p->logits, c.vocab_size, p->st, (const int *)p->seq_tokens, p->out_ids, with_logits ? 1 : 0,
                           (const float *)(q8 || sf ? p->part_val : nullptr), (const int *)(q8 || sf ? p->part_idx : nullptr),
                           sf ? sf_grid(p->n_sms, c.fp16_lanes, c.vocab_size, c.dim, false) : p->n_sms, TR(9), p->tp, with_logits ? -1 : last_x_op))) return rc;
        n++;
    }
    if (launches) *launches = n;
    return B200_OK;
}

// ---- one persistent kernel per token (decode_persistent.cuh) ---------------------------------------------------------------
// Checks the kernel's restrictions and allocates its descriptors; never launches (the KV cache must stay zero-initialised).
// Leaves p->pd_ok / p->pd_why; a plan that does not fit simply keeps the multi-kernel graph.
int pd_prepare(b200_plan *p) {
    const b200_config &c = p->cfg;
    p->pd_ok = false;
    if (p->is_moe) {
        p->pd_why = p->moe_shared ? "the persistent decode kernel has no Qwen2-MoE layer (MoE plans decode through the CUDA graph)"
                                  : "the persistent decode kernel has no Qwen3-MoE layer (MoE plans decode through the CUDA graph)";
        return B200_OK;
    }
    if (p->resident) { p->pd_why = "the persistent decode kernel reads Q8_0 tiles only (this plan keeps K-quant weights resident: it decodes through the CUDA graph)"; return B200_OK; }
    if (c.dim > 8192) { p->pd_why = "the persistent decode kernel's register-resident RMSNorm supports dim <= 8192"; return B200_OK; }
    if (p->wtype != B200_GGML_Q8_0) { p->pd_why = "the persistent decode kernel needs Q8_0 weights"; return B200_OK; }
    if (c.head_size != 64 && c.head_size != 128) { p->pd_why = "the persistent decode kernel supports head sizes 64 and 128"; return B200_OK; }
    if (p->nh_l > p->n_sms) { p->pd_why = "more attention heads than SMs"; return B200_OK; }
    if (!gateup_fits(p->hid_l, p->n_sms)) { p->pd_why = "hidden slice per CTA exceeds the epilogue buffer"; return B200_OK; }
    int max_seg = p->tout.seg;
    for (const LayerW &L : p->layers) {
        const int segs[4] = {L.tqkv.seg, L.two.seg, L.tgu.seg, L.tw2.seg};
        for (int k = 0; k < 4; k++) if (segs[k] > max_seg) max_seg = segs[k];
    }
    int maxdyn = 0;
    CK(cudaDeviceGetAttribute(&maxdyn, cudaDevAttrMaxSharedMemoryPerBlockOptin, p->device));
    const int att_floats = 3 * c.head_size + (p->att_scratch ? 0 : (c.context_length + PD_CT - 1) / PD_CT * PD_CT); // score row padded to whole accumulator chunks
    const PdSmem L = pd_layout(c.dim, p->qd, c.hidden_dim, c.head_size, att_floats, max_seg, (size_t)maxdyn);
    if (L.stages < 4) { p->pd_why = "shape leaves fewer than 4 ring stages of shared memory"; return B200_OK; }
    int rc;
    if (!p->pd_layers) {
        std::vector<PdLayer> h(c.n_layers);
        const size_t ctx_kv = (size_t)c.context_length * p->kvd_l;
        for (int l = 0; l < c.n_layers; l++) {
            const LayerW &W = p->layers[l];
            h[l].qkv = W.tqkv; h[l].wo = W.two; h[l].gu = W.tgu; h[l].w2 = W.tw2;
            h[l].attn_norm = W.attn_norm; h[l].ffn_norm = W.ffn_norm; h[l].q_norm = W.q_norm; h[l].k_norm = W.k_norm;
            h[l].qkv_bias = W.qkv_bias;
            h[l].kc = p->key_cache + (size_t)l * ctx_kv;
            h[l].vc = p->value_cache + (size_t)l * ctx_kv;
        }
        if ((rc = dalloc(p, &p->pd_layers, h.size() * sizeof(PdLayer)))) return rc;
        CK(cudaMemcpy(p->pd_layers, h.data(), h.size() * sizeof(PdLayer), cudaMemcpyHostToDevice));
        if ((rc = dalloc(p, &p->pd_trace, (size_t)p->n_sms * (c.n_layers + 1) * PD_STAMPS * 8))) return rc;
        CK(cudaMemset(p->pd_trace, 0, (size_t)p->n_sms * (c.n_layers + 1) * PD_STAMPS * 8));
    }
    if ((rc = with_mma_head_size(p, c.head_size, [&](auto HS) { CK(set_max_dyn(k_decode_persistent<HS>, maxdyn)); return B200_OK; }))) return rc;
    p->pd_L = L;
    p->pd_ok = true;
    p->pd_why = "";
    return B200_OK;
}

int enqueue_persistent(b200_plan *p, bool with_logits, int *launches, bool trace) {
    const b200_config &c = p->cfg;
    PdArgs a;
    memset(&a, 0, sizeof a);
    a.layers = p->pd_layers; a.n_layers = c.n_layers; a.lm_head = p->tout; a.out_norm = p->out_norm; a.emb = p->emb;
    a.dim = c.dim; a.hidden = c.hidden_dim; a.qd = p->qd; a.n_heads = p->nh_l; a.n_kv_heads = p->nkv_l;
    a.head_size = c.head_size; a.arch = p->kflags; a.ctx = c.context_length;
    a.eps = c.rms_norm_eps; a.sqrt_hs = att_score_arg(p);
    a.emb_scale = p->mup.embedding_scale; a.res_scale = p->mup.residual_scale; a.logit_scale = p->mup.logit_scale;
    a.rope_cr = p->rope_cr; a.rope_ci = p->rope_ci;
    a.st = p->st; a.seq_tokens = p->seq_tokens; a.out_ids = p->out_ids;
    a.x = p->x; a.qkv = p->qkv; a.hb = p->hb; a.logits = p->logits;
    a.attq = p->attq; a.atts = p->atts; a.hq = p->hq; a.hs = p->hs; a.blk_cnt = p->blk_cnt;
    a.part_val = p->part_val; a.part_idx = p->part_idx; a.sync = p->pd_sync; a.host_err = p->d_err;
    a.att_scratch = p->att_scratch; a.trace = trace ? p->pd_trace : nullptr;
    a.with_logits = with_logits ? 1 : 0;
    a.tp = p->tp; a.pd_flags_off = p->pd_flags_off;
    a.head_base = p->tp.rank * p->nh_l; a.dim_base = p->tp.rank * p->dim_l; a.hid_base = p->tp.rank * p->hid_l; a.voc_base = p->tp.rank * p->voc_l;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(p->n_sms);
    cfg.blockDim = dim3(PD_THREADS);
    cfg.dynamicSmemBytes = p->pd_L.total;
    cfg.stream = p->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative; // every CTA spins on its peers: the driver must guarantee co-residency
    attr[0].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = p->pd_coop ? 1 : 0;
    if (launches) *launches = 1;
    return with_mma_head_size(p, c.head_size, [&](auto HS) { CK(cudaLaunchKernelEx(&cfg, k_decode_persistent<HS>, a, p->pd_L)); return B200_OK; });
}

// Captures what enqueue(&g.launches) puts on p->stream into g.
template <typename Enqueue> int capture(b200_plan *p, Graph &g, Enqueue &&enqueue) {
    cudaGraph_t cg = nullptr;
    CK(cudaStreamBeginCapture(p->stream, cudaStreamCaptureModeThreadLocal));
    int rc = enqueue(&g.launches);
    cudaError_t e = cudaStreamEndCapture(p->stream, &cg);
    if (rc) { if (cg) cudaGraphDestroy(cg); return rc; }
    if (e != cudaSuccess) return fail(p, B200_ERR_CUDA, "cudaStreamEndCapture: %s", cudaGetErrorString(e));
    e = cudaGraphInstantiate(&g.exec, cg, 0);
    cudaGraphDestroy(cg);
    if (e != cudaSuccess) return fail(p, B200_ERR_CUDA, "cudaGraphInstantiate: %s", cudaGetErrorString(e));
    return B200_OK;
}

void destroy(Graph &g) {
    if (g.exec) cudaGraphExecDestroy(g.exec);
    g = Graph{};
}

void destroy(TokenGraphs &t) {
    for (Graph *g : {&t.decode, &t.prefill, &t.trace}) destroy(*g);
}

// Both decode implementations are captured; b200_set_decode_mode picks which one the forward calls launch.
int capture_all(b200_plan *p) {
    auto token = [&](Graph &g, bool persistent, bool with_logits, bool trace) {
        return capture(p, g, [&](int *launches) {
            return persistent ? enqueue_persistent(p, with_logits, launches, trace) : enqueue_forward(p, with_logits, launches, trace);
        });
    };
    TokenGraphs &G = p->graph, &P = p->pers;
    int rc;
    if ((rc = token(G.decode, false, true, false)) || (rc = token(G.prefill, false, false, false))) return rc;
    if (p->wtype == B200_GGML_Q8_0 || p->use_f16_stream) {
        if ((rc = dalloc(p, &p->trace_rec, (size_t)(G.decode.launches + 8) * 32)) || (rc = token(G.trace, false, true, true))) return rc;
    }
    if ((rc = pd_prepare(p))) return rc;
    if (p->pd_ok) {
        // grid = one CTA per SM with (almost) all of its shared memory: co-resident on an idle GPU either way; the cooperative
        // attribute makes the driver check it.  Should a driver refuse cooperative kernel nodes in a graph, retry without.
        for (int attempt = 0; attempt < 2; attempt++) {
            p->pd_coop = attempt == 0;
            if (!(rc = token(P.decode, true, true, false)) && !(rc = token(P.prefill, true, false, false)) && !(rc = token(P.trace, true, true, true))) break;
            cudaGetLastError();
            destroy(P);
        }
        if (rc) { p->pd_ok = false; p->pd_why = "persistent decode kernel could not be captured: " + p->err; }
    }
    if (!p->pd_ok && p->decode_mode == B200_DECODE_PERSISTENT) p->decode_mode = B200_DECODE_GRAPH;
    return B200_OK;
}

// ---- batched decode (decode_batch.cuh) -------------------------------------------------------------------------------------
// 112 KB: two batched-stream CTAs (the gate/up and down projections, back to back under PDL) still fit on one SM together.
const size_t SMB_SMEM_BUDGET = 112 * 1024;

// Largest row count whose batched stream keeps at least 3 ring stages on every matrix of the plan.
int batch_max_rows(const b200_plan *p) {
    const LayerW &L0 = p->layers[0];
    const int segs[5] = {L0.tqkv.seg, L0.two.seg, L0.tgu.seg, L0.tw2.seg, p->tout.seg};
    for (int n = SMB_MAX_ROWS; n > 0; n--) {
        bool ok = true;
        for (int s : segs) ok = ok && smb_layout(s, n, SMB_SMEM_BUDGET).stages >= 3;
        if (ok) return n;
    }
    return 0;
}

template <int MODE>
int launch_stream_batch(b200_plan *p, const TileMat &W, int n, const int8_t *xq, const float *xs, float *out, int ostride, int8_t *hq = nullptr,
                        float *hs = nullptr, bool argmax = false) {
    const SmbSmem L = smb_layout(W.seg, n, SMB_SMEM_BUDGET);
    SmbArgs a;
    a.W = W; a.nrow = n; a.xq = xq; a.xs = xs; a.out = out; a.ostride = ostride; a.hq = hq; a.hs = hs; a.blk_cnt = p->bt.blk_cnt;
    a.oscale = out_scale(p, MODE == SMV_RESID, &W == &p->tout);
    a.part_val = argmax ? p->bt.part_val : nullptr;
    a.part_idx = argmax ? p->bt.part_idx : nullptr;
    return launch_k(p, p->use_pdl, k_stream_matvec_q8_batch<MODE>, dim3(p->n_sms), dim3(SMV_THREADS), L.total, a, L);
}

// The classifier of a batched step over its first e rows, whose final residuals are rows [0, e) of x (dim floats apart): the final
// norm (k_rmsnorm_quant_batch), the Q8_0 lm_head stream with per-row argmax partials, and k_argmax_batch -> bt.logits / bt.ids rows
// [0, e).  enqueue_batch ends with it over bt.x, b200_forward_chunk over the chunk's residual rows (pi8.X).
const int CLASSIFIER_LAUNCHES = 3;
int enqueue_classifier(b200_plan *p, float *x, int e) {
    const b200_config &c = p->cfg;
    auto &B = p->bt;
    TpCtx solo{};
    solo.n = 1;
    int rc;
    if ((rc = launch_k(p, p->use_pdl, k_rmsnorm_quant_batch<false>, dim3(e), dim3(NORM_THREADS), norm_smem_bytes(c.dim), x, (const BatchRows *)B.rows, p->emb,
                       p->mup.embedding_scale, (const float *)p->out_norm, c.rms_norm_eps, c.dim, B.xq, B.xs, TraceBuf{nullptr, 0, 0}, solo)))
        return rc;
    if ((rc = launch_stream_batch<SMV_STORE>(p, p->tout, e, B.xq, B.xs, B.logits, sampler_padded(c.vocab_size), nullptr, nullptr, true))) return rc;
    return launch_k(p, p->use_pdl, k_argmax_batch, dim3(e), dim3(32), (size_t)0, (const float *)B.part_val, (const int *)B.part_idx, p->n_sms, B.ids);
}

// One forward step of n rows in the given form (StepForm bits): the single-sequence graph's kernel sequence, every launch serving
// all n rows.  The final norm, lm_head and argmax run over the first e rows only (e = 0: not at all, as in the prefills).  SPLIT
// costs one more launch per layer.  OWN writes key_cache / value_cache, whose layout is slot 0's.
int enqueue_batch(b200_plan *p, int n, int e, int form, int *launches) {
    const bool sched = form & SCHED, split = form & SPLIT, own = form & OWN;
    const b200_config &c = p->cfg;
    auto &B = p->bt;
    const bool pdl = p->use_pdl;
    const int qkvd = p->qd + 2 * p->kvd;
    const size_t ctx_kv = (size_t)c.context_length * p->kvd, slot_stride = (size_t)c.n_layers * ctx_kv;
    const size_t norm_smem = norm_smem_bytes(c.dim);
    TpCtx solo{};
    solo.n = 1;
    int k = 0, rc;
    if (sched) {
        k_batch_rows_next<<<1, 32, 0, p->stream>>>(B.sched, B.step, B.rows);
        CK(cudaGetLastError());
        k++;
    }
    auto norm = [&](bool embed, const float *w, int rows) {
        auto go = [&](auto kern) { // the first norm of a SCHED step waits for k_batch_rows_next in full: the rows are read before any PDL wait
            return launch_k(p, pdl && !(sched && embed), kern, dim3(rows), dim3(NORM_THREADS), norm_smem, B.x, (const BatchRows *)B.rows, p->emb, p->mup.embedding_scale, w, c.rms_norm_eps, c.dim, B.xq, B.xs, TraceBuf{nullptr, 0, 0}, solo);
        };
        k++;
        return embed ? go(k_rmsnorm_quant_batch<true>) : go(k_rmsnorm_quant_batch<false>);
    };
    for (int l = 0; l < c.n_layers; l++) {
        const LayerW &L = p->layers[l];
        if ((rc = norm(l == 0, L.attn_norm, n))) return rc;
        if ((rc = launch_stream_batch<SMV_STORE>(p, L.tqkv, n, B.xq, B.xs, B.qkv, qkvd))) return rc;
        float *kc = (own ? p->key_cache : B.slot_k) + (size_t)l * ctx_kv, *vc = (own ? p->value_cache : B.slot_v) + (size_t)l * ctx_kv;
        const size_t att_smem = att_smem_bytes(c.head_size, c.context_length, B.att_scratch != nullptr);
        rc = with_decode_head_size(p, c.head_size, [&](auto HS) {
            if (!split)
                return launch_k(p, pdl, k_attention_batch<HS>, dim3(p->nh_l, n), dim3(ATT_THREADS), att_smem, B.qkv, qkvd, kc, vc, slot_stride,
                                (const BatchRows *)B.rows, (const float *)p->rope_cr, (const float *)p->rope_ci, p->nh_l, p->nkv_l, p->kflags,
                                (const float *)L.q_norm, (const float *)L.k_norm, (const float *)L.qkv_bias, c.rms_norm_eps, att_score_arg(p), B.xq,
                                B.xs, B.att_scratch, c.context_length, TraceBuf{nullptr, 0, 0}, solo);
            // split: the two launches of a step whose rows may share a sequence
            const int r = launch_k(p, pdl, k_rope_kv_batch<HS>, dim3(p->nh_l, n), dim3(2 * HS), (size_t)0, B.qkv, qkvd, kc, vc, slot_stride, (const BatchRows *)B.rows,
                                   (const float *)p->rope_cr, (const float *)p->rope_ci, p->nh_l, p->nkv_l, p->kflags, (const float *)L.q_norm,
                                   (const float *)L.k_norm, (const float *)L.qkv_bias, c.rms_norm_eps);
            k++;
            return r ? r : launch_k(p, pdl, k_attention_cached_rows<HS>, dim3(p->nh_l, n), dim3(ATT_THREADS), att_smem, B.qkv, qkvd, kc, vc, slot_stride,
                                    (const BatchRows *)B.rows, p->nh_l, p->nkv_l, p->kflags, att_score_arg(p), B.xq, B.xs, B.att_scratch, c.context_length,
                                    TraceBuf{nullptr, 0, 0}, solo);
        });
        if (rc) return rc;
        if ((rc = launch_stream_batch<SMV_RESID>(p, L.two, n, B.xq, B.xs, B.x, c.dim))) return rc;
        if ((rc = norm(false, L.ffn_norm, n))) return rc;
        if ((rc = launch_stream_batch<SMV_GATEUP>(p, L.tgu, n, B.xq, B.xs, B.hb, c.hidden_dim, B.hq, B.hs))) return rc;
        if ((rc = launch_stream_batch<SMV_RESID>(p, L.tw2, n, B.hq, B.hs, B.x, c.dim))) return rc;
        k += 5;
    }
    if (e && (rc = enqueue_classifier(p, B.x, e))) return rc;
    if (launches) *launches = k + (e ? CLASSIFIER_LAUNCHES : 0);
    return B200_OK;
}

// The step graph of `form` for n rows, e of them with the classifier, captured on first use.
int batch_graph(b200_plan *p, int form, int n, int e, const Graph **out) {
    Graph &g = p->bt.g[form][n][e];
    int rc;
    if (!g.exec && (rc = capture(p, g, [&](int *launches) { return enqueue_batch(p, n, e, form, launches); }))) return rc;
    *out = &g;
    return B200_OK;
}

// The form of a step of n rows writing the decode slots, or with own the plan's cache (every row slot 0): SPLIT when a slot
// repeats, because k_attention_batch writes a row's K / V inside its attention CTA and rows of one sequence would race.
int step_form(const BatchRows &r, int n, bool own) {
    const int target = own ? OWN : 0;
    for (int i = 1; i < n; i++)
        for (int j = 0; j < i; j++)
            if (r.slot[j] == r.slot[i]) return target | SPLIT;
    return target;
}

void batch_free(b200_plan *p) {
    auto &B = p->bt;
    for (auto &by_form : B.g)
        for (auto &by_rows : by_form)
            for (Graph &g : by_rows) destroy(g);
    for (void *d : B.allocs) cudaFree(d);
    if (B.h_rows) cudaFreeHost(B.h_rows);
    if (B.h_out) cudaFreeHost(B.h_out);
    B = b200_plan::Batch{};
}

template <typename T> int balloc(b200_plan *p, T **ptr, size_t n_bytes) {
    void *d = nullptr;
    CK(cudaMalloc(&d, n_bytes ? n_bytes : 16));
    p->bt.allocs.push_back(d);
    CK(cudaMemsetAsync(d, 0, n_bytes ? n_bytes : 16, p->stream));
    *ptr = reinterpret_cast<T *>(d);
    return B200_OK;
}

// ns decode slots (0: none) and the per-row scratch of batch_max_rows rows, whatever the slot count: a step of the exact prefills
// or of b200_forward_decode_multi fills every row however many slots there are.
int batch_alloc(b200_plan *p, int ns) {
    const b200_config &c = p->cfg;
    auto &B = p->bt;
    const int big = c.dim > p->qd ? c.dim : p->qd;
    const size_t N = (size_t)batch_max_rows(p), kv = (size_t)c.n_layers * c.context_length * p->kvd * 4;
    int rc;
    if ((rc = balloc(p, &B.slot_k, (size_t)ns * kv)) || (rc = balloc(p, &B.slot_v, (size_t)ns * kv)) || (rc = balloc(p, &B.x, N * c.dim * 4)) ||
        (rc = balloc(p, &B.qkv, N * (p->qd + 2 * p->kvd) * 4)) || (rc = balloc(p, &B.hb, N * c.hidden_dim * 4)) ||
        (rc = balloc(p, &B.logits, N * sampler_padded(c.vocab_size) * 4)) || (rc = balloc(p, &B.xq, N * big)) || (rc = balloc(p, &B.xs, N * (big / 32) * 4)) ||
        (rc = balloc(p, &B.hq, N * c.hidden_dim)) || (rc = balloc(p, &B.hs, N * (c.hidden_dim / 32) * 4)) ||
        (rc = balloc(p, &B.part_val, N * p->n_sms * 4)) || (rc = balloc(p, &B.part_idx, N * p->n_sms * 4)) || (rc = balloc(p, &B.ids, N * 4)) ||
        (rc = balloc(p, &B.smp_out, N * 8 * 4)) || (rc = balloc(p, &B.smp_indices, N * c.vocab_size * 4)) || (rc = balloc(p, &B.blk_cnt, N * (c.hidden_dim / 32) * 4)) || (rc = balloc(p, &B.rows, sizeof(BatchRows))) ||
        (rc = balloc(p, &B.sched, (size_t)c.context_length * sizeof(BatchRows))) || (rc = balloc(p, &B.step, 4)))
        return rc;
    if (p->att_scratch && (rc = balloc(p, &B.att_scratch, N * p->nh_l * c.context_length * 4))) return rc;
    CK(cudaMallocHost(&B.h_rows, sizeof(BatchRows)));
    CK(cudaMallocHost(&B.h_out, (size_t)SMB_MAX_ROWS * 9 * 4));
    CK(cudaStreamSynchronize(p->stream));
    B.n_slots = ns;
    return B200_OK;
}

// ---- steps whose rows may share a sequence: b200_forward_decode_multi and the exact prefills ------------------------------
// Why a plan cannot run them (nullptr: it can): the conditions of batched decode.
const char *const RESIDENT_MULTI_WHY = "batched and multi-position steps read Q8_0 tiles only (this plan keeps K-quant weights resident: it runs one position per step)";
const char *multi_why(const b200_plan *p) {
    if (p->is_moe)
        return p->moe_shared ? "multi-position steps have no Qwen2-MoE layer (MoE plans run one position per step)"
                             : "multi-position steps have no Qwen3-MoE layer (MoE plans run one position per step)";
    if (p->resident) return RESIDENT_MULTI_WHY;
    if (p->cfg.tp_size > 1) return "multi-position steps run on single-GPU plans only (this plan is tensor-parallel)";
    if (p->wtype != B200_GGML_Q8_0) return "multi-position steps need Q8_0 weights (FP16 plans run one position per step)";
    if (!batch_max_rows(p)) return "no row count of the batched Q8_0 stream fits this plan's shapes";
    return nullptr;
}

// The per-row scratch: a plan without decode slots allocates it on first use.
int multi_ready(b200_plan *p) {
    if (p->bt.x) return B200_OK;
    const int rc = batch_alloc(p, 0);
    if (rc) batch_free(p);
    return rc;
}

// Enqueues the steps of one call back to back: the schedule is uploaded once and k_batch_rows_next feeds each step its entry, so
// the caller synchronises once.  p->ev0 / ev1 bracket the steps.  own: every row writes the plan's cache (slot 0) instead of the
// decode slots.  Without scored the steps run no classifier; with it every row of every step runs it, and scored(s, r0) enqueues
// after step s, whose rows are the call's rows from r0 on, the work that reads its logits.
template <typename Scored = std::nullptr_t>
int run_steps(b200_plan *p, const std::vector<BatchRows> &sched, const std::vector<int> &nrows, bool own, int *launches, Scored scored = nullptr) {
    constexpr bool classify = !std::is_same_v<Scored, std::nullptr_t>;
    auto &B = p->bt;
    const int steps = (int)sched.size();
    std::vector<const Graph *> graphs(steps);
    int rc;
    for (int s = 0; s < steps; s++)
        if ((rc = batch_graph(p, SCHED | step_form(sched[s], nrows[s], own), nrows[s], classify ? nrows[s] : 0, &graphs[s]))) return rc;
    CK(cudaMemcpyAsync(B.sched, sched.data(), (size_t)steps * sizeof(BatchRows), cudaMemcpyHostToDevice, p->stream));
    CK(cudaMemsetAsync(B.step, 0, 4, p->stream));
    CK(cudaEventRecord(p->ev0, p->stream));
    int k = 0;
    for (int s = 0, r0 = 0; s < steps; r0 += nrows[s++]) {
        CK(cudaGraphLaunch(graphs[s]->exec, p->stream));
        k += graphs[s]->launches;
        if constexpr (classify)
            if ((rc = scored(s, r0))) return rc;
    }
    CK(cudaEventRecord(p->ev1, p->stream));
    if (launches) *launches = k;
    return B200_OK;
}

// Appends positions start .. start + len - 1 of one sequence to a schedule of rows-wide steps, filling the last step first.
void pack_rows(std::vector<BatchRows> &sched, std::vector<int> &nrows, int rows, const int *tokens, int start, int len, int slot) {
    for (int j = 0; j < len; j++) {
        if (nrows.empty() || nrows.back() == rows) { sched.emplace_back(); nrows.push_back(0); }
        const int v = nrows.back()++;
        sched.back().token[v] = tokens[j];
        sched.back().pos[v] = start + j;
        sched.back().slot[v] = slot;
    }
}

// cudaFuncSetAttribute is per function and process-wide: every kernel gets the device opt-in maximum ONCE, so a later plan
// with a smaller context never lowers the limit under an earlier plan's instantiated graphs.
const int ATT_SMEM_FLOATS_MAX = 4096; // q|k|out|scores beyond this: the score row goes to a global scratch row

int set_smem_attrs(b200_plan *p) {
    const b200_config &c = p->cfg;
    int maxdyn = 0;
    CK(cudaDeviceGetAttribute(&maxdyn, cudaDevAttrMaxSharedMemoryPerBlockOptin, p->device));
    if (c.dim > 16384) return fail(p, B200_ERR_UNSUPPORTED, "dim > 16384 not supported by the RMSNorm kernel");
    size_t need_norm = norm_smem_bytes(c.dim);
    size_t need_att = att_smem_bytes(c.head_size, c.context_length, p->att_scratch != nullptr);
    int maxcols = c.hidden_dim > c.dim ? c.hidden_dim : c.dim;
    if (p->qd > maxcols) maxcols = p->qd;
    size_t need_f16 = f16_smem_bytes(maxcols, p->cfg.fp16_lanes);
    if (need_norm > (size_t)maxdyn || need_att > (size_t)maxdyn || (p->wtype == B200_GGML_F16 && need_f16 > (size_t)maxdyn))
        return fail(p, B200_ERR_UNSUPPORTED, "shape needs more shared memory than the device offers (%d bytes)", maxdyn);
    static bool done = false; // process-wide, like the attribute itself (plans are created from one thread at a time per process)
    if (done) return B200_OK;
    CK(set_max_dyn(k_rmsnorm_quant<true>, maxdyn));
    CK(set_max_dyn(k_rmsnorm_quant<false>, maxdyn));
    for (int hs : {32, 64, 96, 128, 256}) {
        const int rc = with_decode_head_size(p, hs, [&](auto HS) {
            CK(set_max_dyn(k_attention<HS>, maxdyn));
            CK(set_max_dyn(k_attention_batch<HS>, maxdyn));
            CK(set_max_dyn(k_attention_cached_rows<HS>, maxdyn));
            CK(set_max_dyn(k_i8_attention<HS>, maxdyn));
            return B200_OK;
        });
        if (rc) return rc;
    }
    for (int fmt : {0, B200_GGML_Q4_K, B200_GGML_Q5_K, B200_GGML_Q6_K}) { // the single-token streams: budgets up to the opt-in limit (ring_budgets)
        CK(set_max_dyn(smv_kernel<SMV_STORE>(fmt), maxdyn));
        CK(set_max_dyn(smv_kernel<SMV_RESID>(fmt), maxdyn));
        CK(set_max_dyn(smv_kernel<SMV_GATEUP>(fmt), maxdyn));
        CK(set_max_dyn(smv_norm_kernel<SMV_STORE>(fmt), maxdyn));
        CK(set_max_dyn(smv_norm_kernel<SMV_GATEUP>(fmt), maxdyn));
    }
    CK(set_max_dyn(k_matvec_f16<MODE_STORE>, maxdyn));
    CK(set_max_dyn(k_matvec_f16<MODE_RESID>, maxdyn));
    CK(set_max_dyn(k_stream_matvec_f16<16, SF_STORE>, maxdyn));
    CK(set_max_dyn(k_stream_matvec_f16<16, SF_RESID>, maxdyn));
    CK(set_max_dyn(k_stream_matvec_f16<16, SF_GATEUP>, maxdyn));
    CK(set_max_dyn(k_stream_matvec_f16<8, SF_STORE>, maxdyn));
    CK(set_max_dyn(k_stream_matvec_f16<8, SF_RESID>, maxdyn));
    CK(set_max_dyn(k_stream_matvec_f16<8, SF_GATEUP>, maxdyn));
    CK(set_max_dyn(k_rmsnorm_quant_batch<true>, maxdyn));
    CK(set_max_dyn(k_rmsnorm_quant_batch<false>, maxdyn));
    CK(set_max_dyn(k_i8_norm<true>, maxdyn));
    CK(set_max_dyn(k_i8_norm<false>, maxdyn));
    CK(cudaFuncSetAttribute(k_stream_matvec_q8_batch<SMV_STORE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMB_SMEM_BUDGET));
    CK(cudaFuncSetAttribute(k_stream_matvec_q8_batch<SMV_RESID>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMB_SMEM_BUDGET));
    CK(cudaFuncSetAttribute(k_stream_matvec_q8_batch<SMV_GATEUP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMB_SMEM_BUDGET));
    CK(cudaFuncSetAttribute(k_moe_gateup, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMV_SMEM_BUDGET_MAX));
    CK(cudaFuncSetAttribute(k_moe_down, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMV_SMEM_BUDGET_MAX));
    CK(cudaFuncSetAttribute(k_routed_gateup, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMV_SMEM_BUDGET_MAX));
    CK(cudaFuncSetAttribute(k_routed_down, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMV_SMEM_BUDGET_MAX));
    CK(cudaFuncSetAttribute(k_sample_rows, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sampler_smem_bytes()));
    CK(cudaFuncSetAttribute(k_sample_ctl, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sampler_smem_bytes()));
    done = true;
    return B200_OK;
}

// Every layer's QKV and gate/up ring budget (ring_budgets), from the device's shared-memory figures and this plan's attention launch.
int size_rings(b200_plan *p) {
    const b200_config &c = p->cfg;
    if (p->wtype != B200_GGML_Q8_0) return B200_OK; // no tile-major streams
    int sm = 0, reserve = 0, optin = 0;
    CK(cudaDeviceGetAttribute(&sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, p->device));
    CK(cudaDeviceGetAttribute(&reserve, cudaDevAttrReservedSharedMemoryPerBlock, p->device));
    CK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, p->device));
    size_t att = att_smem_bytes(c.head_size, c.context_length, p->att_scratch != nullptr);
    const int rc = with_decode_head_size(p, c.head_size, [&](auto HS) {
        cudaFuncAttributes fa;
        CK(cudaFuncGetAttributes(&fa, k_attention<HS>));
        att += fa.sharedSizeBytes;
        return B200_OK;
    });
    if (rc) return rc;
    const SmDev d{(size_t)sm, (size_t)reserve, (size_t)optin};
    for (int l = 0; l < c.n_layers; l++) ring_budgets(d, p->n_sms, p->fuse_norm, att, p->layers[l ? l - 1 : 0], p->layers[l]);
    return B200_OK;
}

const char *prefill_why(const b200_plan *p, int mode);
int prefill_init(b200_plan *p);

// RoPE.precomputeFreqsCisYaRN (RoPE.java:39-83) with Java's float / double boundaries taken literally: every float expression is
// rounded to float after each operation (the library is built with -ffp-contract=off, so nothing here becomes an FMA), each
// Math.log / Math.pow / Math.cos / Math.sin is a double libm call on a widened float, and (float) casts narrow where Java's do.
// yarnCorrDim(nDims, nCtxOrig, nRot, base) = nDims * (float)log(nCtxOrig / (nRot * 2f * (float)PI)) / (2f * (float)log(base))
float yarn_corr_dim(int n_dims, int n_ctx_orig, float n_rot, float base) {
    const float pi_f = (float)3.14159265358979323846;
    const float denom = n_rot * 2.0f * pi_f;                       // nRot * 2.0f * (float) Math.PI, left to right
    const float ratio = (float)n_ctx_orig / denom;                  // int / float: the int widens to float
    const float num = (float)n_dims * (float)log((double)ratio);
    return num / (2.0f * (float)log((double)base));
}

// Java's Math.max / Math.min (float): a NaN operand wins, and -0.0f orders below 0.0f (fmaxf / fminf return the other operand)
float java_maxf(float a, float b) {
    if (a != a) return a;
    if (a == 0.0f && b == 0.0f && std::signbit(a)) return b;
    return a >= b ? a : b;
}
float java_minf(float a, float b) {
    if (a != a) return a;
    if (a == 0.0f && b == 0.0f && std::signbit(b)) return b;
    return a <= b ? a : b;
}

// yarnRamp(low, high, i0) = 1 - min(1, max(0, (i0 - low) / max(0.001f, high - low)))
float yarn_ramp(float low, float high, int i0) {
    const float y = ((float)i0 - low) / java_maxf(0.001f, high - low);
    return 1.0f - java_minf(1.0f, java_maxf(0.0f, y));
}

void rope_table_yarn(const b200_config &c, const b200_yarn_config &y, std::vector<float> &cr, std::vector<float> &ci) {
    const int hs = c.head_size, half = hs / 2;
    cr.resize((size_t)c.context_length * half);
    ci.resize((size_t)c.context_length * half);
    const double theta = (double)c.rope_theta;                      // DevstralConfiguration.ropeTheta() is a float, widened
    const float freq_scale = 1.0f / y.factor;
    const float corr0 = yarn_corr_dim(hs, y.original_context_length, y.beta_fast, (float)theta);
    const float corr1 = yarn_corr_dim(hs, y.original_context_length, y.beta_slow, (float)theta);
    // mscale = 1 + 0.1f * logMultiplier * (float)Math.log(1.0f / freqScale): 1/(1/factor) in float, not factor
    const float mscale = y.log_multiplier > 0.0f ? 1.0f + 0.1f * y.log_multiplier * (float)log((double)(1.0f / freq_scale)) : 1.0f;
    std::vector<float> freq(half);
    for (int i = 0; i < hs; i += 2) {
        const float extrap = (float)(1.0 / pow(theta, i / (double)hs));
        const float interp = freq_scale * extrap;
        const float ramp = yarn_ramp(corr0, corr1, i / 2);
        const float a = interp * (1.0f - ramp), b = extrap * ramp;  // two rounded products, then a rounded sum
        freq[i / 2] = a + b;
    }
    size_t k = 0;
    for (int pos = 0; pos < c.context_length; pos++)
        for (int j = 0; j < half; j++) {
            const float val = (float)pos * freq[j];
            cr[k] = (float)cos((double)val) * mscale;               // narrowed first, then one float multiply
            ci[k] = (float)sin((double)val) * mscale;
            k++;
        }
}

// MoE FFN tensors of one layer (llama.cpp's names and shapes, dims[0] innermost): the F32 router, the stacked routed experts
// [E][rows][cols] and, on Qwen2-MoE, the shared-expert gate and the shared expert (Qwen3-MoE has neither).  Every routed expert
// becomes a TileMat of its own, cut from its row range of the stacked tensor (K-quant experts are re-quantised on the way like any
// matrix).
int upload_moe_layer(b200_plan *p, const b200_tensor *tensors, int n_tensors, int l) {
    const b200_config &c = p->cfg;
    LayerW &L = p->layers[l];
    const int E = p->moe.n_experts, He = p->moe.expert_hidden_dim, Hs = p->moe.shared_hidden_dim, D = c.dim;
    struct Want { const char *name; int n_dims; int64_t d[3]; bool f32; };
    const Want want[8] = {{"ffn_gate_inp.weight", 2, {D, E, 0}, true},     {"ffn_gate_inp_shexp.weight", 1, {D, 0, 0}, true},
                          {"ffn_gate_exps.weight", 3, {D, He, E}, false},  {"ffn_up_exps.weight", 3, {D, He, E}, false},
                          {"ffn_down_exps.weight", 3, {He, D, E}, false},  {"ffn_gate_shexp.weight", 2, {D, Hs, 0}, false},
                          {"ffn_up_shexp.weight", 2, {D, Hs, 0}, false},   {"ffn_down_shexp.weight", 2, {Hs, D, 0}, false}};
    const b200_tensor *t[8];
    for (int i = 0; i < 8; i++) {
        if (!p->moe_shared && (i == 1 || i >= 5)) continue; // the shared-expert tensors
        const std::string name = "blk." + std::to_string(l) + "." + want[i].name;
        t[i] = find(tensors, n_tensors, name);
        if (!t[i]) return fail(p, B200_ERR_BAD_ARG, "missing tensor %s", name.c_str());
        if (want[i].f32 && t[i]->ggml_type != B200_GGML_F32)
            return fail(p, B200_ERR_UNSUPPORTED, "tensor %s must be F32 (ggml type %d)", name.c_str(), t[i]->ggml_type);
        // the shared-expert gate may also come as [dim, 1]
        const int nd = (i == 1 && t[i]->n_dims == 2 && t[i]->dims[1] == 1) ? 1 : t[i]->n_dims;
        bool ok = nd == want[i].n_dims && t[i]->data;
        for (int k = 0; ok && k < nd; k++) ok = t[i]->dims[k] == want[i].d[k];
        if (!ok)
            return fail(p, B200_ERR_BAD_ARG, "tensor %s must have dims [%lld, %lld, %lld] (first %d used; got n_dims %d, dims [%lld, %lld, %lld])", name.c_str(),
                        (long long)want[i].d[0], (long long)want[i].d[1], (long long)want[i].d[2], want[i].n_dims, t[i]->n_dims, (long long)t[i]->dims[0],
                        (long long)(t[i]->n_dims > 1 ? t[i]->dims[1] : 0), (long long)(t[i]->n_dims > 2 ? t[i]->dims[2] : 0));
    }
    int rc;
    if ((rc = dalloc(p, &L.router, (size_t)E * D * 4))) return rc;
    CK(cudaMemcpy(L.router, t[0]->data, (size_t)E * D * 4, cudaMemcpyHostToDevice));
    if (p->moe_shared) {
        if ((rc = dalloc(p, &L.shared_gate, (size_t)D * 4))) return rc;
        CK(cudaMemcpy(L.shared_gate, t[1]->data, (size_t)D * 4, cudaMemcpyHostToDevice));
        if ((rc = upload_tiles(p, t[5], t[6], nullptr, Hs, Hs, 0, D, true, L.sgu))) return rc;
        if ((rc = upload_tiles(p, t[7], nullptr, nullptr, D, 0, 0, Hs, false, L.sdn))) return rc;
    }
    std::vector<const unsigned char *> hg(E), hd(E);
    for (int e = 0; e < E; e++) {
        const int gr0[3] = {e * He, e * He, 0}, gfu[3] = {E * He, E * He, 0};
        if ((rc = upload_tiles(p, t[2], t[3], nullptr, He, He, 0, D, true, L.xgu, gr0, gfu))) return rc;
        const int dr0[3] = {e * D, 0, 0}, dfu[3] = {E * D, 0, 0};
        if ((rc = upload_tiles(p, t[4], nullptr, nullptr, D, 0, 0, He, false, L.xdn, dr0, dfu))) return rc;
        hg[e] = L.xgu.base;
        hd[e] = L.xdn.base;
    }
    if ((rc = dalloc(p, &L.gu_bases, (size_t)E * sizeof(void *)))) return rc;
    if ((rc = dalloc(p, &L.dn_bases, (size_t)E * sizeof(void *)))) return rc;
    CK(cudaMemcpy(L.gu_bases, hg.data(), (size_t)E * sizeof(void *), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(L.dn_bases, hd.data(), (size_t)E * sizeof(void *), cudaMemcpyHostToDevice));
    return B200_OK;
}

// Weight bytes of a dense single-GPU Q8_0 plan: the embedding's Q8_0 planes plus every stream, as Q8_0 tiles or (resident) in the
// form upload_tiles gives it on a resident plan.  The one function behind both footprints of the residency rule.
int64_t weight_footprint(const b200_plan *p, const b200_tensor *tensors, int n_tensors, bool resident) {
    const b200_config &c = p->cfg;
    const bool phi3 = c.arch == B200_ARCH_PHI3;
    auto T = [&](const std::string &s) { return find(tensors, n_tensors, s); };
    auto stream = [&](const b200_tensor *a, const b200_tensor *b, const b200_tensor *d, int r0, int r1, int r2, int cols, bool gateup) {
        const b200_tensor *ts[3] = {a, b, d};
        const int rs[3] = {r0, r1, r2}, rows = gateup ? r0 + r1 : r0 + r1 + r2;
        return tile_bytes(tile_geometry(rows, cols, resident ? resident_fmt(ts, rs, rows, cols) : 0));
    };
    const b200_tensor *outw = T("output.weight");
    int64_t b = (int64_t)c.vocab_size * c.dim / 32 * 34; // embedding: int8 plane + f16 scale plane (row gather)
    b += stream(outw ? outw : T("token_embd.weight"), nullptr, nullptr, c.vocab_size, 0, 0, c.dim, false);
    for (int l = 0; l < c.n_layers; l++) {
        const std::string pre = "blk." + std::to_string(l) + ".";
        const b200_tensor *tq = T(pre + (phi3 ? "attn_qkv.weight" : "attn_q.weight"));
        const b200_tensor *tk = phi3 ? tq : T(pre + "attn_k.weight"), *tv = phi3 ? tq : T(pre + "attn_v.weight");
        const b200_tensor *tg = T(pre + (phi3 ? "ffn_up.weight" : "ffn_gate.weight")), *tu = T(pre + "ffn_up.weight");
        b += stream(tq, tk, tv, p->qd, p->kvd, p->kvd, c.dim, false);
        b += stream(T(pre + "attn_output.weight"), nullptr, nullptr, c.dim, 0, 0, p->qd, false);
        b += stream(tg, tu, nullptr, c.hidden_dim, c.hidden_dim, 0, c.dim, true);
        b += stream(T(pre + "ffn_down.weight"), nullptr, nullptr, c.dim, 0, 0, c.hidden_dim, false);
    }
    return b;
}

// Room kept free beyond what rest_footprint counts: the CUDA graphs, the scratch of the exact prefill's multi-position steps and of
// the persistent kernel, allocator rounding, and what other processes on the device may take meanwhile.
const int64_t RESIDENT_MARGIN = (int64_t)1 << 30;
int64_t g_memory_budget = 0; // b200_test_set_memory_budget: replaces the free-memory figure of memory_free (0: off)

// The device's free memory as the weight-form rule and the resident plan's prefill scratch read it.
int memory_free(b200_plan *p, int64_t *avail) {
    *avail = g_memory_budget;
    if (!*avail) {
        size_t fr = 0, tot = 0;
        CK(cudaMemGetInfo(&fr, &tot));
        *avail = (int64_t)fr;
    }
    return B200_OK;
}

// What a plan allocates besides its weights: both KV caches, the upload's two device staging buffers (live while the weights are
// allocated), the activations, the attention score scratch and the RoPE tables.
int64_t rest_footprint(const b200_plan *p, size_t stage_bytes) {
    const b200_config &c = p->cfg;
    const int64_t big = c.dim > p->qd ? c.dim : p->qd;
    const int64_t kv = 2LL * c.n_layers * c.context_length * p->kvd * 4;
    const int64_t act = 4LL * (c.dim + big + p->qd + 2 * p->kvd + 2LL * c.hidden_dim + sampler_padded(c.vocab_size) + c.vocab_size) +
                        (big + c.hidden_dim) * 33 / 8; // + int8 activations and their f32 block scales
    const int64_t att = 3 * c.head_size + c.context_length > ATT_SMEM_FLOATS_MAX ? 4LL * c.n_heads * ((c.context_length + PD_CT - 1) / PD_CT * PD_CT) : 0;
    const int64_t rope = 4LL * c.context_length * c.head_size;
    return kv + 2 * (int64_t)stage_bytes + act + att + rope;
}

// The residency rule of a single-GPU dense plan with K-quant matrices: Q8_0 tiles throughout when they fit the device's free memory
// (less RESIDENT_MARGIN) next to everything else the plan allocates; else resident streams where resident_fmt allows; else an error
// naming both figures.  No option selects the form: the rule reads only the shapes, the tensor types and the free memory.
int weight_policy(b200_plan *p, const b200_tensor *tensors, int n_tensors, size_t stage_bytes) {
    p->w8_bytes = weight_footprint(p, tensors, n_tensors, false);
    const int64_t wr = weight_footprint(p, tensors, n_tensors, true);
    const int64_t rest = rest_footprint(p, stage_bytes) + RESIDENT_MARGIN;
    int64_t avail;
    int rc;
    if ((rc = memory_free(p, &avail))) return rc;
    if (p->w8_bytes + rest <= avail) { p->w_bytes = p->w8_bytes; return B200_OK; }
    if (wr + rest <= avail) { p->resident = true; p->w_bytes = wr; return B200_OK; }
    return fail(p, B200_ERR_OOM, "the model does not fit the device: %lld bytes with Q8_0 tiles and %lld bytes with K-quant weights resident are needed "
                "(weights plus %lld bytes of KV cache, activations, upload staging and margin), %lld bytes are free",
                (long long)(p->w8_bytes + rest), (long long)(wr + rest), (long long)rest, (long long)avail);
}

int build(b200_plan *p, const b200_tensor *tensors, int n_tensors) {
    const b200_config &c = p->cfg;
    if (c.arch != B200_ARCH_LLAMA && c.arch != B200_ARCH_QWEN3 && c.arch != B200_ARCH_PHI3 && c.arch != B200_ARCH_QWEN2 && c.arch != B200_ARCH_QWEN2_MOE &&
        c.arch != B200_ARCH_GRANITE && c.arch != B200_ARCH_DEVSTRAL && c.arch != B200_ARCH_QWEN3_MOE)
        return fail(p, B200_ERR_UNSUPPORTED, "unknown arch %d", c.arch);
    const bool qwen3_attn = c.arch == B200_ARCH_QWEN3 || c.arch == B200_ARCH_QWEN3_MOE; // q/k RMSNorm, NeoX RoPE, head size of its own
    p->kflags = qwen3_attn ? (KF_NEOX | KF_QKNORM) : c.arch == B200_ARCH_PHI3 ? KF_NEOX
              : (c.arch == B200_ARCH_QWEN2 || c.arch == B200_ARCH_QWEN2_MOE) ? (KF_NEOX | KF_QKVBIAS) : c.arch == B200_ARCH_GRANITE ? KF_ATTSCALE : 0;
    if (p->is_moe) {
        const b200_moe_config &m = p->moe;
        if (c.tp_size > 1) return fail(p, B200_ERR_UNSUPPORTED, "%s plans are single-GPU (tensor parallelism has no expert layout)", p->moe_name);
        if (m.n_experts < 1 || m.n_experts > MOE_MAX_EXPERTS) return fail(p, B200_ERR_BAD_ARG, "n_experts = %d: need 1..%d", m.n_experts, MOE_MAX_EXPERTS);
        const int kmax = m.n_experts < MOE_MAX_K ? m.n_experts : MOE_MAX_K;
        if (m.n_experts_used < 1 || m.n_experts_used > kmax)
            return fail(p, B200_ERR_BAD_ARG, "n_experts_used = %d: need 1..%d (min(n_experts, %d))", m.n_experts_used, kmax, MOE_MAX_K);
        if (p->moe_shared && (m.expert_hidden_dim <= 0 || m.shared_hidden_dim <= 0 || m.expert_hidden_dim % 32 || m.shared_hidden_dim % 32))
            return fail(p, B200_ERR_UNSUPPORTED, "expert hidden %d / shared hidden %d: the Q8_0 stream needs positive multiples of 32", m.expert_hidden_dim,
                        m.shared_hidden_dim);
        if (!p->moe_shared && m.shared_hidden_dim != 0)
            return fail(p, B200_ERR_BAD_ARG, "shared_hidden_dim = %d: Qwen3-MoE has no shared expert (pass 0)", m.shared_hidden_dim);
        if (!p->moe_shared && (m.expert_hidden_dim <= 0 || m.expert_hidden_dim % 32))
            return fail(p, B200_ERR_UNSUPPORTED, "expert hidden %d: the Q8_0 stream needs a positive multiple of 32", m.expert_hidden_dim);
        if (c.dim > 8192) // k_moe_route stages dim floats in (default-sized) dynamic shared memory, as the RMSNorm kernel caps dim
            return fail(p, B200_ERR_UNSUPPORTED, "dim %d: the MoE router kernel supports dim <= 8192", c.dim);
        p->moe_hv = m.shared_hidden_dim + m.n_experts_used * m.expert_hidden_dim;
    }
    if (c.dim <= 0 || c.dim % 32 || c.hidden_dim % 32 || (c.head_size != 32 && c.head_size != 64 && c.head_size != 96 && c.head_size != 128 && c.head_size != 256) || c.n_heads % c.n_kv_heads ||
        c.n_layers <= 0 || c.vocab_size <= 0 || c.context_length <= 0)
        return fail(p, B200_ERR_BAD_ARG, "unsupported shape (dim/hidden must be multiples of 32, head_size one of 32/64/96/128/256)");
    if (c.fp16_lanes != 0 && c.fp16_lanes != 8 && c.fp16_lanes != 16 && c.fp16_lanes != 4 && c.fp16_lanes != 32)
        return fail(p, B200_ERR_BAD_ARG, "fp16_lanes must be 0, 4, 8, 16 or 32");
    p->qd = c.n_heads * c.head_size;
    p->kvd = c.n_kv_heads * c.head_size;
    if (!qwen3_attn && c.arch != B200_ARCH_DEVSTRAL && p->qd != c.dim)
        return fail(p, B200_ERR_BAD_ARG, "llama / phi3 / qwen2: n_heads*head_size must equal dim");
    {
        const int tn = c.tp_size;
        if (tn < 1 || tn > TP_MAX || c.tp_rank < 0 || c.tp_rank >= tn) return fail(p, B200_ERR_BAD_ARG, "bad tp_rank/tp_size %d/%d", c.tp_rank, tn);
        if (tn > 1 && (c.n_heads % tn || c.n_kv_heads % tn || c.dim % (4 * tn) || c.hidden_dim % (32 * tn) || c.vocab_size % (4 * tn)))
            return fail(p, B200_ERR_UNSUPPORTED, "shape does not split %d ways (heads, kv heads, dim/4, hidden/32 and vocab/4 must be divisible)", tn);
        p->nh_l = c.n_heads / tn; p->nkv_l = c.n_kv_heads / tn;
        p->qd_l = p->nh_l * c.head_size; p->kvd_l = p->nkv_l * c.head_size;
        p->hid_l = c.hidden_dim / tn; p->dim_l = c.dim / tn; p->voc_l = c.vocab_size / tn;
        p->tp.rank = c.tp_rank; p->tp.n = 1; // n becomes tp_size once the peers are attached
        p->tp.ops_per_fwd = 4u * (unsigned)c.n_layers + 1u;
    }

    const b200_tensor *emb = find(tensors, n_tensors, "token_embd.weight");
    if (!emb) return fail(p, B200_ERR_BAD_ARG, "missing tensor token_embd.weight");
    const b200_tensor *wq0 = find(tensors, n_tensors, c.arch == B200_ARCH_PHI3 ? "blk.0.attn_qkv.weight" : "blk.0.attn_q.weight");
    if (!wq0) return fail(p, B200_ERR_BAD_ARG, "missing tensor blk.0.attn_q.weight (Phi-3: blk.0.attn_qkv.weight)");
    p->wtype = eff_type(wq0->ggml_type); // K-quant matrices become Q8_0 while they are uploaded (kquant.cuh)
    if (p->wtype != B200_GGML_Q8_0 && p->wtype != B200_GGML_F16)
        return fail(p, B200_ERR_UNSUPPORTED, "Type: %d currently not supported by this engine (Q8_0, F16 and the K-quants Q4_K/Q5_K/Q6_K only)", wq0->ggml_type);
    if (p->is_moe && p->wtype != B200_GGML_Q8_0)
        return fail(p, B200_ERR_UNSUPPORTED, "%s runs in Q8_0 only (FP16 MoE plans are not supported, as in the reference)", p->moe_name);
    bool any_kq = false;
    for (int i = 0; i < n_tensors; i++) any_kq = any_kq || kq_is_kquant(tensors[i].ggml_type);

    CK(cudaSetDevice(p->device));
    read_knobs(p);
    CK(cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking));
    CK(cudaEventCreate(&p->ev0));
    CK(cudaEventCreate(&p->ev1));
    int rc;
    CK(cudaDeviceGetAttribute(&p->n_sms, cudaDevAttrMultiProcessorCount, p->device));
    const bool q8 = p->wtype == B200_GGML_Q8_0; // every Q8_0 weight matrix is a tile-major stream (stream_matvec.cuh)
    {
        if (c.tp_size > 1 && !q8) return fail(p, B200_ERR_UNSUPPORTED, "tensor parallelism needs Q8_0 weights");
        if (q8) {
            const struct { const char *name; int rows, cols; } mats[5] = {
                {"attn_qkv", p->qd_l + 2 * p->kvd_l, c.dim}, {"attn_output", p->dim_l, p->qd}, {"output", (p->voc_l + 3) & ~3, c.dim},
                {"ffn_gate/ffn_up", 2 * p->hid_l, c.dim}, {"ffn_down", p->dim_l, c.hidden_dim}}; // the MoE FFN has its own streams (below)
            for (int i = 0; i < (p->is_moe ? 3 : 5); i++)
                if (!stream_shape_ok(mats[i].rows, mats[i].cols))
                    return fail(p, B200_ERR_UNSUPPORTED, "Q8_0 matrix %s is %d columns wide: too wide for 3 ring stages of the weight stream", mats[i].name, mats[i].cols);
            if (!gateup_fits(p->hid_l, p->n_sms))
                return fail(p, B200_ERR_UNSUPPORTED, "Q8_0 matrix ffn_gate/ffn_up: hidden dim %d puts more hidden units on one CTA than the stream's epilogue buffer holds (%d)",
                            c.hidden_dim, SMV_HVALS);
        }
        p->use_f16_stream = p->wtype == B200_GGML_F16 && c.tp_size == 1 && sf_layout(p->qd + 2 * p->kvd, c.dim, c.fp16_lanes, false).ok &&
                            sf_layout(c.dim, p->qd, c.fp16_lanes, false).ok && sf_layout(c.hidden_dim, c.dim, c.fp16_lanes, true).ok &&
                            sf_layout(c.dim, c.hidden_dim, c.fp16_lanes, false).ok && sf_layout(c.vocab_size, c.dim, c.fp16_lanes, false).ok;
        if (p->is_moe) { // the MoE FFN has its own streams (the dense FFN checks above are skipped)
            const b200_moe_config &m = p->moe;
            const int hs = m.shared_hidden_dim, he = m.expert_hidden_dim;
            const bool cut = (!p->moe_shared || (stream_shape_ok(2 * hs, c.dim) && stream_shape_ok(c.dim, hs))) && stream_shape_ok(2 * he, c.dim) &&
                             stream_shape_ok(c.dim, he) && gateup_fits(p->moe_hv, p->n_sms);
            if (!cut) return fail(p, B200_ERR_UNSUPPORTED, "expert hidden %d / shared hidden %d at dim %d: the Q8_0 stream layout cannot cut these matrices", he, hs, c.dim);
            const int seg_x = he / smv_pick_nseg(he);
            p->moe_dl = moe_down_layout(p->moe_hv, p->moe_shared ? hs / smv_pick_nseg(hs) : seg_x, seg_x, SMV_SMEM_BUDGET_MAX);
            if (p->moe_dl.stages < 3) return fail(p, B200_ERR_UNSUPPORTED, "the expert down projection leaves fewer than 3 ring stages of shared memory");
        }
        p->use_pdl = q8 || p->use_f16_stream;
        // Tensor parallelism keeps the separate norm: its read of x waits on every rank's slice (TP_SLOT_X).  So does MoE,
        // whose FFN norm must write float xb for the F32 router anyway; its plans keep 8 launches per layer.
        p->fuse_norm = q8 && c.tp_size == 1 && !p->is_moe && norm_fusion_ok(c.dim);
    }
    size_t stage_bytes = (size_t)34 * (8u << 20); // 8 Mi blocks = 272 MiB
    if (q8) {
        size_t m1 = (size_t)c.vocab_size * c.dim, m2 = (size_t)2 * c.hidden_dim * c.dim, m3 = (size_t)(p->qd + 2 * p->kvd) * c.dim;
        size_t mx = m1 > m2 ? m1 : m2;
        if (m3 > mx) mx = m3;
        const size_t m4 = (size_t)2 * p->moe.shared_hidden_dim * c.dim;
        if (m4 > mx) mx = m4;
        size_t need = mx / 32 * 34 + 4096;
        if (need > stage_bytes) stage_bytes = need;
    }
    if (any_kq) { // second half of each staging buffer receives the raw K-quant bytes (always fewer than their Q8_0 form)
        stage_bytes = (stage_bytes + 255) & ~(size_t)255;
        p->kq_off = stage_bytes;
        stage_bytes *= 2;
    }
    if (q8 && c.tp_size == 1 && !p->is_moe) {
        if (any_kq) {
            if ((rc = weight_policy(p, tensors, n_tensors, stage_bytes))) return rc;
        } else p->w_bytes = p->w8_bytes = weight_footprint(p, tensors, n_tensors, false);
    }
    const auto t_up0 = std::chrono::steady_clock::now();
    if ((rc = up_init(p, stage_bytes))) return rc;
    struct StageGuard { b200_plan *pl; ~StageGuard() { up_destroy(pl); } } guard{p};

    // embedding table (+ tied classifier: AbstractModelLoader.java:186-195)
    if ((rc = alloc_matrix(p, p->emb, c.vocab_size, c.dim, eff_type(emb->ggml_type)))) return rc;
    if ((rc = upload_matrix(p, emb, c.vocab_size, c.dim, p->emb, 0))) return rc;
    const b200_tensor *outw = find(tensors, n_tensors, "output.weight");
    if (!outw && eff_type(emb->ggml_type) != p->wtype) return fail(p, B200_ERR_UNSUPPORTED, "tied output weight type differs from the matrix type");
    if (q8) {
        const int r0[3] = {c.tp_rank * p->voc_l, 0, 0}, fu[3] = {c.vocab_size, 0, 0};
        if ((rc = upload_tiles(p, outw ? outw : emb, nullptr, nullptr, p->voc_l, 0, 0, c.dim, false, p->tout, r0, fu))) return rc;
        p->out = p->emb;
        if ((rc = dalloc(p, &p->part_val, (size_t)p->n_sms * 4))) return rc;
        if ((rc = dalloc(p, &p->part_idx, (size_t)p->n_sms * 4))) return rc;
        const int hid = c.hidden_dim > p->moe_hv ? c.hidden_dim : p->moe_hv;
        if ((rc = dalloc(p, &p->blk_cnt, (size_t)(hid / 32) * 4))) return rc;
        CK(cudaMemset(p->blk_cnt, 0, (size_t)(hid / 32) * 4));
    } else {
        if (p->use_f16_stream) { // per-CTA argmax partials of the classifier launch (at most 3 CTAs per SM)
            if ((rc = dalloc(p, &p->part_val, (size_t)p->n_sms * 4 * 4))) return rc;
            if ((rc = dalloc(p, &p->part_idx, (size_t)p->n_sms * 4 * 4))) return rc;
        }
        if (!outw) p->out = p->emb;
        else if ((rc = alloc_matrix(p, p->out, c.vocab_size, c.dim, p->wtype)) || (rc = upload_matrix(p, outw, c.vocab_size, c.dim, p->out, 0))) return rc;
    }
    if ((rc = upload_f32(p, find(tensors, n_tensors, "output_norm.weight"), c.dim, &p->out_norm, "output_norm.weight"))) return rc;

    p->layers.resize(c.n_layers);
    for (int l = 0; l < c.n_layers; l++) {
        LayerW &L = p->layers[l];
        std::string pre = "blk." + std::to_string(l) + ".";
        auto T = [&](const char *s) { return find(tensors, n_tensors, pre + s); };
        if ((rc = upload_f32(p, T("attn_norm.weight"), c.dim, &L.attn_norm, "attn_norm.weight"))) return rc;
        if ((rc = upload_f32(p, T("ffn_norm.weight"), c.dim, &L.ffn_norm, "ffn_norm.weight"))) return rc;
        if (qwen3_attn) {
            if ((rc = upload_f32(p, T("attn_q_norm.weight"), c.head_size, &L.q_norm, "attn_q_norm.weight"))) return rc;
            if ((rc = upload_f32(p, T("attn_k_norm.weight"), c.head_size, &L.k_norm, "attn_k_norm.weight"))) return rc;
        }
        if ((c.arch == B200_ARCH_QWEN2 || c.arch == B200_ARCH_QWEN2_MOE) && (rc = upload_qkv_bias(p, tensors, n_tensors, l, &L.qkv_bias))) return rc;
        // Phi-3 stores wqkv and gate|up fused (Phi3StandardWeights: attn_qkv.weight = [q; k; v] rows, ffn_up.weight = [gate; up] rows,
        // InferenceCore.java:718-724,779-781): the row ranges below address the same source tensor; rows are independent dot products, so
        // splitting a fused matrix by rows changes nothing in the arithmetic.
        const bool phi3 = c.arch == B200_ARCH_PHI3;
        const b200_tensor *tq = T(phi3 ? "attn_qkv.weight" : "attn_q.weight"), *tk = phi3 ? tq : T("attn_k.weight"), *tv = phi3 ? tq : T("attn_v.weight");
        const b200_tensor *tg = T(phi3 ? "ffn_up.weight" : "ffn_gate.weight"), *tu = T("ffn_up.weight");
        const int q_full = phi3 ? p->qd + 2 * p->kvd : p->qd, k_full = phi3 ? q_full : p->kvd, g_full = phi3 ? 2 * c.hidden_dim : c.hidden_dim;
        const int k_src = phi3 ? p->qd : 0, v_src = phi3 ? p->qd + p->kvd : 0, u_src = phi3 ? c.hidden_dim : 0;
        if (q8) {
            const int rk = c.tp_rank;
            const int qr0[3] = {rk * p->qd_l, k_src + rk * p->kvd_l, v_src + rk * p->kvd_l}, qfu[3] = {q_full, k_full, k_full};
            if ((rc = upload_tiles(p, tq, tk, tv, p->qd_l, p->kvd_l, p->kvd_l, c.dim, false, L.tqkv, qr0, qfu))) return rc;
            const int dr0[3] = {rk * p->dim_l, 0, 0}, dfu[3] = {c.dim, 0, 0};
            if ((rc = upload_tiles(p, T("attn_output.weight"), nullptr, nullptr, p->dim_l, 0, 0, p->qd, false, L.two, dr0, dfu))) return rc;
            if (p->is_moe) {
                if ((rc = upload_moe_layer(p, tensors, n_tensors, l))) return rc;
                continue;
            }
            const int gr0[3] = {rk * p->hid_l, u_src + rk * p->hid_l, 0}, gfu[3] = {g_full, g_full, 0};
            if ((rc = upload_tiles(p, tg, tu, nullptr, p->hid_l, p->hid_l, 0, c.dim, true, L.tgu, gr0, gfu))) return rc;
            if ((rc = upload_tiles(p, T("ffn_down.weight"), nullptr, nullptr, p->dim_l, 0, 0, c.hidden_dim, false, L.tw2, dr0, dfu))) return rc;
            continue;
        }
        // FP16: row-major matrices, fused [Wq; Wk; Wv] so one launch produces the packed q|k|v vector
        if ((rc = alloc_matrix(p, L.qkv, p->qd + 2 * p->kvd, c.dim, p->wtype))) return rc;
        if ((rc = upload_matrix(p, tq, p->qd, c.dim, L.qkv, 0, 0, q_full))) return rc;
        if ((rc = upload_matrix(p, tk, p->kvd, c.dim, L.qkv, p->qd, k_src, k_full))) return rc;
        if ((rc = upload_matrix(p, tv, p->kvd, c.dim, L.qkv, p->qd + p->kvd, v_src, k_full))) return rc;
        if ((rc = alloc_matrix(p, L.wo, c.dim, p->qd, p->wtype))) return rc;
        if ((rc = upload_matrix(p, T("attn_output.weight"), c.dim, p->qd, L.wo, 0))) return rc;
        if ((rc = alloc_matrix(p, L.w1, c.hidden_dim, c.dim, p->wtype))) return rc;
        if ((rc = upload_matrix(p, tg, c.hidden_dim, c.dim, L.w1, 0, 0, g_full))) return rc;
        if ((rc = alloc_matrix(p, L.w3, c.hidden_dim, c.dim, p->wtype))) return rc;
        if ((rc = upload_matrix(p, tu, c.hidden_dim, c.dim, L.w3, 0, u_src, g_full))) return rc;
        if ((rc = alloc_matrix(p, L.w2, c.dim, c.hidden_dim, p->wtype))) return rc;
        if ((rc = upload_matrix(p, T("ffn_down.weight"), c.dim, c.hidden_dim, L.w2, 0))) return rc;
    }

    // drain the pipeline: every copy and every repack has finished before the first forward
    CK(cudaStreamSynchronize(p->up.copy));
    CK(cudaStreamSynchronize(p->stream));
    p->up.total_s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_up0).count();
    {
        const double hs = p->up.host_copy_s, ts = p->up.total_s;
        const int64_t hb = p->up.h2d_bytes;
        up_destroy(p); // pinned buffers and device staging are not needed any more
        p->up.host_copy_s = hs; p->up.total_s = ts; p->up.h2d_bytes = hb;
    }
    // RoPE table exactly as RoPE.precomputeFreqsCis (RoPE.java:6-37, ropeScaling=false):
    // freq = (float)(1.0 / Math.pow(theta, i / (double) headSize)); val = pos * freq (float);
    // cos/sin evaluated in double and narrowed.  Devstral plans with YaRN parameters use rope_table_yarn instead.
    {
        std::vector<float> cr, ci;
        if (p->has_yarn) {
            rope_table_yarn(c, p->yarn, cr, ci);
        } else {
            int half = c.head_size / 2;
            cr.resize((size_t)c.context_length * half);
            ci.resize((size_t)c.context_length * half);
            size_t k = 0;
            for (int pos = 0; pos < c.context_length; pos++)
                for (int i = 0; i < c.head_size; i += 2) {
                    float freq = (float)(1.0 / pow((double)c.rope_theta, i / (double)c.head_size));
                    float val = (float)pos * freq;
                    cr[k] = (float)cos((double)val);
                    ci[k] = (float)sin((double)val);
                    k++;
                }
        }
        if ((rc = dalloc(p, &p->rope_cr, cr.size() * 4))) return rc;
        if ((rc = dalloc(p, &p->rope_ci, ci.size() * 4))) return rc;
        CK(cudaMemcpy(p->rope_cr, cr.data(), cr.size() * 4, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(p->rope_ci, ci.data(), ci.size() * 4, cudaMemcpyHostToDevice));
    }

    int big = c.dim > p->qd ? c.dim : p->qd;
    if (c.tp_size > 1) {
        // one IPC-exportable allocation: x | attq | atts | hq | hs | argmax partials | flags | tick | done counters
        auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
        size_t o = 0;
        p->tp.off_x = (unsigned)o; o = al(o + (size_t)c.dim * 4);
        p->tp.off_attq = (unsigned)o; o = al(o + (size_t)p->qd);
        p->tp.off_atts = (unsigned)o; o = al(o + (size_t)(p->qd / 32) * 4);
        p->tp.off_hq = (unsigned)o; o = al(o + (size_t)c.hidden_dim);
        p->tp.off_hs = (unsigned)o; o = al(o + (size_t)(c.hidden_dim / 32) * 4);
        p->tp.off_pv = (unsigned)o; o = al(o + TP_MAX * 4);
        p->tp.off_pi = (unsigned)o; o = al(o + TP_MAX * 4);
        p->tp.off_flags = (unsigned)o; o = al(o + TP_SLOTS * TP_MAX * 4);
        p->tp.off_tick = (unsigned)o; o = al(o + 4);
        p->tp.off_done = (unsigned)o; o = al(o + TP_SLOTS * 4);
        p->pd_flags_off = (unsigned)o; o = al(o + PD_S_SLOTS * TP_MAX * 4); // epoch flags of the persistent decode kernel
        p->comm_bytes = o;
        if ((rc = dalloc(p, &p->comm, o))) return rc;
        CK(cudaMemset(p->comm, 0, o));
        p->x = reinterpret_cast<float *>(p->comm + p->tp.off_x);
    } else if ((rc = dalloc(p, &p->x, (size_t)c.dim * 4))) return rc;
    if ((rc = dalloc(p, &p->xb, (size_t)big * 4))) return rc;
    if ((rc = dalloc(p, &p->qkv, (size_t)(p->qd_l + 2 * p->kvd_l) * 4))) return rc;
    const int hid_alloc = c.hidden_dim > p->moe_hv ? c.hidden_dim : p->moe_hv; // MoE: the virtual hidden vector (moe.cuh)
    if ((rc = dalloc(p, &p->hb, (size_t)hid_alloc * 4))) return rc;
    if ((rc = dalloc(p, &p->hb2, (size_t)c.hidden_dim * 4))) return rc;
    if ((rc = dalloc(p, &p->logits, (size_t)sampler_padded(c.vocab_size) * 4))) return rc; // zero pad: the sampler's exact sum runs over whole thread chunks
    if ((rc = dalloc(p, &p->xq, (size_t)big))) return rc;
    if ((rc = dalloc(p, &p->xs, (size_t)(big / 32) * 4))) return rc;
    if (c.tp_size > 1) {
        p->hq = reinterpret_cast<int8_t *>(p->comm + p->tp.off_hq);
        p->hs = reinterpret_cast<float *>(p->comm + p->tp.off_hs);
        p->attq = reinterpret_cast<int8_t *>(p->comm + p->tp.off_attq);
        p->atts = reinterpret_cast<float *>(p->comm + p->tp.off_atts);
    } else {
        if ((rc = dalloc(p, &p->hq, (size_t)hid_alloc))) return rc;
        if ((rc = dalloc(p, &p->hs, (size_t)(hid_alloc / 32) * 4))) return rc;
        p->attq = p->xq; // the attention output is the activation of the Wo matvec
        p->atts = p->xs;
    }
    size_t kv_bytes = (size_t)c.n_layers * c.context_length * p->kvd_l * 4;
    if ((rc = dalloc(p, &p->key_cache, kv_bytes))) return rc;
    if ((rc = dalloc(p, &p->value_cache, kv_bytes))) return rc;
    CK(cudaMemset(p->key_cache, 0, kv_bytes));
    CK(cudaMemset(p->value_cache, 0, kv_bytes));
    CK(cudaMemset(p->logits, 0, (size_t)sampler_padded(c.vocab_size) * 4));
    if ((rc = dalloc(p, &p->smp_indices, (size_t)c.vocab_size * 4))) return rc;
    if ((rc = dalloc(p, &p->smp_out, 8 * 4))) return rc;
    p->seq_cap = c.context_length + 8;
    if ((rc = dalloc(p, &p->st, sizeof(StepState)))) return rc;
    if ((rc = dalloc(p, &p->seq_tokens, (size_t)p->seq_cap * 4))) return rc;
    if ((rc = dalloc(p, &p->out_ids, (size_t)p->seq_cap * 4))) return rc;
    CK(cudaMemset(p->st, 0, sizeof(StepState)));
    CK(cudaMemset(p->seq_tokens, 0, (size_t)p->seq_cap * 4));
    CK(cudaMallocHost(&p->h_st, sizeof(StepState)));
    CK(cudaMallocHost(&p->h_ids, (size_t)p->seq_cap * 4));
    if (p->is_moe) {
        const int E = p->moe.n_experts, k = p->moe.n_experts_used;
        if ((rc = dalloc(p, &p->moe_ids, (size_t)c.n_layers * k * 4))) return rc;
        if ((rc = dalloc(p, &p->moe_w, (size_t)c.n_layers * p->moe_nw * 4))) return rc;
        if ((rc = dalloc(p, &p->moe_logits, (size_t)c.n_layers * (E + 1) * 4))) return rc;
        if ((rc = dalloc(p, &p->moe_done, (size_t)c.n_layers * 4))) return rc;
        CK(cudaMemset(p->moe_ids, 0, (size_t)c.n_layers * k * 4));
        CK(cudaMemset(p->moe_w, 0, (size_t)c.n_layers * p->moe_nw * 4));
        CK(cudaMemset(p->moe_done, 0, (size_t)c.n_layers * 4));
    }

    // epoch counters of the persistent kernel + the error word every bounded device-side wait reports through
    if ((rc = dalloc(p, &p->pd_sync, PD_S_WORDS * 4))) return rc;
    CK(cudaMemset(p->pd_sync, 0, PD_S_WORDS * 4));
    CK(cudaHostAlloc(&p->h_err, 64, cudaHostAllocMapped));
    *p->h_err = 0u;
    CK(cudaHostGetDevicePointer((void **)&p->d_err, p->h_err, 0));
    p->tp.err = p->pd_sync + PD_S_ERR;
    p->tp.host_err = p->d_err;
    if (3 * c.head_size + c.context_length > ATT_SMEM_FLOATS_MAX) { // long context: score rows in global memory
        if ((rc = dalloc(p, &p->att_scratch, (size_t)p->nh_l * ((c.context_length + PD_CT - 1) / PD_CT * PD_CT) * 4))) return rc;
    }
    if ((rc = size_rings(p))) return rc;
    if ((rc = set_smem_attrs(p))) return rc;
    // tensor_core: why the plan cannot run it, or on a Q8_0 plan that it is opt-in; an FP16 plan that can run it builds and selects it
    auto &tc = p->pf[B200_PREFILL_TENSOR_CORE];
    if (!(tc.why = prefill_why(p, B200_PREFILL_TENSOR_CORE)) && p->wtype == B200_GGML_Q8_0)
        tc.why = "Q8_0 plan: the tensor-core prefill is opt-in (b200_set_prefill_mode builds f16 twins of the weight matrices, +2 bytes per weight)";
    if (c.tp_size > 1) { CK(cudaStreamSynchronize(p->stream)); return B200_OK; } // graphs are captured by b200_tp_attach
    if ((rc = capture_all(p))) return rc;
    if (!tc.why) {
        if ((rc = prefill_init(p))) return rc;
        if (tc.ready) p->pf_mode = B200_PREFILL_TENSOR_CORE;
    }
    CK(cudaStreamSynchronize(p->stream));
    return B200_OK;
}

// ---- batched prefill on the tensor cores (prefill.cuh) -------------------------------------------
static const char *const MOE_PREFILL_WHY = "Qwen2-MoE plans have no tensor-core prefill in this mode: prompts go through the exact token-by-token "
                                           "prefill, or through tensor_core_exact_moe on the tensor cores";
static const char *const MOE3_PREFILL_WHY = "Qwen3-MoE plans have no tensor-core prefill in this mode: prompts go through the exact token-by-token "
                                            "prefill, or through tensor_core_exact_moe on the tensor cores";
static const char *moe_prefill_why(const b200_plan *p) { return p->moe_shared ? MOE_PREFILL_WHY : MOE3_PREFILL_WHY; }

// The geometry of W as Q8_0 tiles: W itself, or for a resident matrix the tiles a Q8_0-tile plan of the same file holds, which
// k_kq_tiles_to_q8 writes into the prefill's scratch before W's GEMM.
TileMat q8_geometry(const TileMat &W) { return W.fmt ? tile_geometry(W.rows, W.cols, 0) : W; }

// Why the plan cannot run prefill mode `mode` (nullptr: it can), decided before anything is allocated: MoE, then resident weights,
// then the prefill batch size, the weight type, tensor parallelism, the shape, the stream segments and the tensor-map encoder, in
// the order each mode has always checked them.  tensor_core_exact_moe: MoE plans only (always single-GPU Q8_0 tiles), then the
// prefill batch size, the shape, every stream's segments (the experts' and the shared expert's included) and the encoder.
const char *prefill_why(const b200_plan *p, int mode) {
    const b200_config &g = p->cfg;
    const int kv_mul = g.n_heads / g.n_kv_heads, nqkv = p->qd + 2 * p->kvd;
    const bool exact = mode == B200_PREFILL_TENSOR_CORE_EXACT, w8a16 = mode == B200_PREFILL_TENSOR_CORE_W8A16;
    auto segs_ok = [&] { // every Q8_0 stream's segment (as Q8_0 tiles) a whole number of GEMM k-blocks (an absent stream has none)
        for (const LayerW &L : p->layers)
            for (const TileMat *t : {&L.tqkv, &L.two, &L.tgu, &L.tw2, &L.sgu, &L.sdn, &L.xgu, &L.xdn})
                if (q8_geometry(*t).seg % pg::BK) return false;
        return true;
    };
    if (mode == B200_PREFILL_EXACT) return nullptr;
    if (mode == B200_PREFILL_TENSOR_CORE_EXACT_MOE) {
        if (!p->is_moe)
            return "tensor_core_exact_moe runs the MoE FFN of Qwen2-MoE / Qwen3-MoE plans: a dense Q8_0 plan's bit-exact tensor-core prefill is tensor_core_exact";
        if (p->prefill_batch <= 1) return "the plan was created without a prefill batch size (prefill_batch_size <= 1)";
        if (g.dim % 64 || p->qd % 64 || nqkv % 64) return "the bit-exact tensor-core prefill needs dim, q width and q+k+v width multiples of 64";
        if (!segs_ok()) return "the bit-exact tensor-core prefill needs Q8_0 stream segments (every expert's included) that are multiples of 64 columns";
        return pg::encode_fn() ? nullptr : "cuTensorMapEncodeTiled not available from the driver";
    }
    if (p->is_moe) return moe_prefill_why(p);
    if (p->resident && !exact)
        return "this plan keeps K-quant weights resident: the f16 and W8A16 tensor-core prefills read f16 matrices or Q8_0 tiles it does not "
               "hold; tensor_core_exact expands each resident matrix to Q8_0 tiles before its GEMM";
    if (p->prefill_batch <= 1) return "the plan was created without a prefill batch size (prefill_batch_size <= 1)";
    if (w8a16 && p->wtype != B200_GGML_Q8_0) return "W8A16 prefill needs a Q8_0 plan (FP16 plans run the tensor-core prefill on their own f16 matrices)";
    if (exact && p->wtype != B200_GGML_Q8_0)
        return "the bit-exact tensor-core prefill needs a Q8_0 plan (an FP16 plan's CPU dot products are FP16 lane chains, not int8 block sums)";
    if (g.tp_size > 1) return "tensor-core prefill is single-GPU";
    if (exact) {
        if (g.dim % 64 || p->qd % 64 || nqkv % 64) return "the bit-exact tensor-core prefill needs dim, q width and q+k+v width multiples of 64";
        if (!segs_ok()) return "the bit-exact tensor-core prefill needs Q8_0 stream segments that are multiples of 64 columns";
        return pg::encode_fn() ? nullptr : "cuTensorMapEncodeTiled not available from the driver";
    }
    if (g.head_size != 64 && g.head_size != 128) return "tensor-core prefill supports head sizes 64 and 128";
    if (g.n_heads % g.n_kv_heads || kv_mul > 64) return "tensor-core prefill needs n_heads % n_kv_heads == 0 and a GQA ratio <= 64";
    if (g.dim % 128 || p->qd % 128 || nqkv % 128 || g.hidden_dim % 64) return "tensor-core prefill needs dim, q width and q+k+v width multiples of 128, hidden a multiple of 64";
    if (!pg::encode_fn()) return "cuTensorMapEncodeTiled not available from the driver";
    if (w8a16 && !segs_ok()) return "W8A16 prefill needs Q8_0 stream segments that are multiples of 64 columns";
    return nullptr;
}

// The end of a mode's init: the mode is ready, or refused with the encoder's rejection if one of its tensor maps was not accepted.
int prefill_built(b200_plan *p, int mode, bool maps_ok) {
    p->pf[mode] = maps_ok ? b200_plan::PrefillMode{true, ""} : b200_plan::PrefillMode{false, "cuTensorMapEncodeTiled rejected a tensor map"};
    return B200_OK;
}

// The chunk's scratch buffers, their tensor maps, both modes' per-layer map slots and the attention kernels' shared-memory
// attributes: allocated once per plan, shared by both tensor-core modes.  *ok = false if a tensor map was rejected.
static int prefill_scratch(b200_plan *p, bool *ok) {
    PrefillCtx &c = p->prefill;
    const b200_config &g = p->cfg;
    const int nqkv = p->qd + 2 * p->kvd;
    *ok = true;
    if (c.bpad) return B200_OK;
    c.bpad = (p->prefill_batch + pg::BM - 1) / pg::BM * pg::BM; // whole 128-row GEMM tiles
    c.maps.resize(g.n_layers);
    c.maps_q8.resize(g.n_layers);
    int rc;
    if ((rc = dalloc(p, &c.X, (size_t)c.bpad * g.dim * 4))) return rc;
    if ((rc = dalloc(p, &c.QKV, (size_t)c.bpad * nqkv * 4))) return rc;
    if ((rc = dalloc(p, &c.A16, (size_t)c.bpad * g.dim * 2))) return rc;
    if ((rc = dalloc(p, &c.ATT16, (size_t)c.bpad * p->qd * 2))) return rc;
    if ((rc = dalloc(p, &c.H16, (size_t)c.bpad * g.hidden_dim * 2))) return rc;
    if ((rc = dalloc(p, &c.tok, (size_t)c.bpad * 4))) return rc;
    if ((rc = dalloc(p, &c.KH, (size_t)g.context_length * p->kvd * 2))) return rc; // f16 K / V of the layer being processed
    if ((rc = dalloc(p, &c.VH, (size_t)g.context_length * p->kvd * 2))) return rc;
    CK(cudaMemset(c.X, 0, (size_t)c.bpad * g.dim * 4));
    CK(cudaMemset(c.QKV, 0, (size_t)c.bpad * nqkv * 4));
    CK(cudaMemset(c.A16, 0, (size_t)c.bpad * g.dim * 2));
    CK(cudaMemset(c.ATT16, 0, (size_t)c.bpad * p->qd * 2));
    CK(cudaMemset(c.H16, 0, (size_t)c.bpad * g.hidden_dim * 2));
    CK(cudaMemset(c.tok, 0, (size_t)c.bpad * 4));
    *ok = pg::make_map(&c.mA, c.A16, c.bpad, g.dim, pg::BM) == 0 && pg::make_map(&c.mATT, c.ATT16, c.bpad, p->qd, pg::BM) == 0 &&
          pg::make_map(&c.mH, c.H16, c.bpad, g.hidden_dim, pg::BM) == 0 && pg::make_map_c(&c.mX, c.X, c.bpad, g.dim) == 0 &&
          pg::make_map_c(&c.mQKV, c.QKV, c.bpad, nqkv) == 0;
    return with_mma_head_size(p, g.head_size, [&](auto HS) {
        CK(cudaFuncSetAttribute(k_pf_attention_mma_packed<HS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pm_smem_bytes<HS>()));
        return B200_OK;
    });
}

// W8A16: the GEMMs read B from the tile-major Q8_0 streams the decode kernels use (L.tqkv, L.two, L.tgu, L.tw2) -- no
// per-weight memory.  Built on the first b200_set_prefill_mode(TENSOR_CORE_W8A16).
int prefill_init_q8(b200_plan *p) {
    PrefillCtx &c = p->prefill;
    const b200_config &g = p->cfg;
    bool ok;
    int rc;
    if ((rc = prefill_scratch(p, &ok))) return rc;
    for (int l = 0; ok && l < g.n_layers; l++) {
        const LayerW &L = p->layers[l];
        PrefillQ8Maps &m = c.maps_q8[l];
        auto mk = [](CUtensorMap *q, CUtensorMap *s, const TileMat &t) {
            return pg::make_map_q8(q, t.base, (uint64_t)t.rows, t.nseg, t.unit_bytes, 0) == 0 && pg::make_map_q8(s, t.base, (uint64_t)t.rows, t.nseg, t.unit_bytes, 1) == 0;
        };
        ok = mk(&m.qkv_q, &m.qkv_s, L.tqkv) && mk(&m.wo_q, &m.wo_s, L.two) && mk(&m.gu_q, &m.gu_s, L.tgu) && mk(&m.w2_q, &m.w2_s, L.tw2);
    }
    return prefill_built(p, B200_PREFILL_TENSOR_CORE_W8A16, ok);
}

// Q8_0 plan: f16 twins of the weight matrices, dequantised on the device from the tile-major stream (value = f16(q * scale),
// Q8_0FloatTensor.getFloat rounded once) -- the B operands of the tensor-core GEMMs; the reference's Q8_0 MMA prefill also
// feeds FP16 tiles (LlamaQ8_0LayersBatchPrefillMMA.java).  Built once the plan is found able to run tensor_core.
int build_f16_twins(b200_plan *p) {
    const b200_config &c = p->cfg;
    if (p->f16_copies) return B200_OK;
    for (int l = 0; l < c.n_layers; l++) {
        LayerW &L = p->layers[l];
        int rc;
        if ((rc = alloc_matrix(p, L.qkv, p->qd + 2 * p->kvd, c.dim, B200_GGML_F16))) return rc;
        if ((rc = alloc_matrix(p, L.wo, c.dim, p->qd, B200_GGML_F16))) return rc;
        if ((rc = alloc_matrix(p, L.w1, c.hidden_dim, c.dim, B200_GGML_F16))) return rc;
        if ((rc = alloc_matrix(p, L.w3, c.hidden_dim, c.dim, B200_GGML_F16))) return rc;
        if ((rc = alloc_matrix(p, L.w2, c.dim, c.hidden_dim, B200_GGML_F16))) return rc;
        auto run = [&](const TileMat &t, int gateup, const DevMat &o0, const DevMat &o1) {
            k_tiles_to_f16<<<(unsigned)((size_t)t.rows * t.nseg), 128, 0, p->stream>>>(t, gateup, (__half *)o0.qs, (__half *)o1.qs);
        };
        run(L.tqkv, 0, L.qkv, L.qkv);
        run(L.two, 0, L.wo, L.wo);
        run(L.tgu, 1, L.w1, L.w3);
        run(L.tw2, 0, L.w2, L.w2);
        CK(cudaGetLastError());
    }
    CK(cudaStreamSynchronize(p->stream));
    p->f16_copies = true;
    return B200_OK;
}

// tensor_core: on a Q8_0 plan the f16 twins first, then the chunk scratch and the f16 matrices' tensor maps.
int prefill_init(b200_plan *p) {
    PrefillCtx &c = p->prefill;
    const b200_config &g = p->cfg;
    const int nqkv = p->qd + 2 * p->kvd;
    int rc;
    if (p->wtype == B200_GGML_Q8_0 && (rc = build_f16_twins(p))) return rc;
    bool ok;
    if ((rc = prefill_scratch(p, &ok))) return rc;
    for (int l = 0; ok && l < g.n_layers; l++) {
        const LayerW &L = p->layers[l];
        PrefillLayerMaps &m = c.maps[l];
        ok = pg::make_map(&m.qkv, L.qkv.qs, nqkv, g.dim, pg::BN) == 0 && pg::make_map(&m.wo, L.wo.qs, g.dim, p->qd, pg::BN) == 0 &&
             pg::make_map(&m.w1, L.w1.qs, g.hidden_dim, g.dim, pg::BN / 2) == 0 && pg::make_map(&m.w3, L.w3.qs, g.hidden_dim, g.dim, pg::BN / 2) == 0 &&
             pg::make_map(&m.w2, L.w2.qs, g.dim, g.hidden_dim, pg::BN) == 0;
    }
    return prefill_built(p, B200_PREFILL_TENSOR_CORE, ok);
}

// A chunk of the tensor-core prefill (prefill_chunk): the device tables of prefill.cuh, the f16 scratch the sequences' regions live
// in, and the K / V target: the plan's own cache (own, one sequence in slot 0) or the decode slots
struct PfChunk {
    const PfTok *tok;
    const PfTile *tiles;
    int n_tiles;
    const PfHist *hist; // sequences with start > 0
    int n_hist, max_start;
    __half *KH, *VH;
    bool own;
};

// The chunk's n tokens already in c.tok (device).  Times the chunk (p->prefill_ms) and counts its launches (p->launches_prefill).
int prefill_forward(b200_plan *p, int n, const PfChunk &ck) {
    PrefillCtx &c = p->prefill;
    const b200_config &g = p->cfg;
    cudaStream_t s = p->stream;
    const int nqkv = p->qd + 2 * p->kvd, mt = (n + pg::BM - 1) / pg::BM, kv_mul = g.n_heads / g.n_kv_heads;
    const size_t ctx_kv = (size_t)g.context_length * p->kvd, slot_stride = (size_t)g.n_layers * ctx_kv;
    // k_pf_attention_mma_packed scales q by this times log2(e): 1/sqrt(head size), or Granite's attentionScale
    const float inv_sqrt_hs = (p->kflags & KF_ATTSCALE) ? p->mup.attention_scale : (float)(1.0 / sqrt((double)g.head_size));
    int nl = 0, rc;
    constexpr int ST = pg::GEMM_STAGES;
    const bool q8 = p->pf_mode == B200_PREFILL_TENSOR_CORE_W8A16;
    // One GEMM, counted: B through the f16 matrices' maps b / b2 (gate/up: W1, W3; c.maps) or, W8A16, through the quant / scale
    // maps bq / bs of the Q8_0 stream W (c.maps_q8)
    auto gemm = [&](auto MODE, const char *name, const CUtensorMap &a, const CUtensorMap &b, const CUtensorMap &b2, const CUtensorMap &bq,
                    const CUtensorMap &bs, const TileMat &W, const CUtensorMap &mc, void *C, int ldc, int n_tiles, int K, int sp, float oscale) {
        constexpr int M = decltype(MODE)::value;
        if (q8 ? pg::gemm_launch<M, ST, pg::B_Q8>(a, bq, bs, mc, C, ldc, n, mt, n_tiles, K, s, sp, W.seg, oscale)
               : pg::gemm_launch<M, ST>(a, b, b2, mc, C, ldc, n, mt, n_tiles, K, s, sp, 0, oscale))
            return fail(p, B200_ERR_CUDA, "%s GEMM launch failed", name);
        nl++;
        return B200_OK;
    };
    using F32 = std::integral_constant<int, pg::GEMM_F32>;
    using RESID = std::integral_constant<int, pg::GEMM_RESID>;
    using GATEUP = std::integral_constant<int, pg::GEMM_GATEUP>;
    // the x += A W^T GEMMs (N = dim only) split K until the grid fills the SMs -- every split reduce-adds its partial
    // product through TMA -- keeping at least 8 k-blocks per split
    auto splits = [&](int n_tiles, int K) {
        const int nk = K / pg::BK;
        int sp = p->n_sms / (mt * n_tiles);
        if (sp > 4) sp = 4;
        while (sp > 1 && (nk / sp < 8 || (sp - 1) * ((nk + sp - 1) / sp) >= nk)) sp--;
        return sp < 1 ? 1 : sp;
    };
    CK(cudaEventRecord(p->ev0, s));
    k_pf_embed<<<n, 256, 0, s>>>(c.tok, p->emb, p->mup.embedding_scale, c.X, g.dim); nl++;
    for (int l = 0; l < g.n_layers; l++) {
        const LayerW &L = p->layers[l];
        const PrefillLayerMaps &m = c.maps[l];
        const PrefillQ8Maps &mq = c.maps_q8[l];
        float *kc = (ck.own ? p->key_cache : p->bt.slot_k) + (size_t)l * ctx_kv, *vc = (ck.own ? p->value_cache : p->bt.slot_v) + (size_t)l * ctx_kv;
        k_pf_rmsnorm_f16<<<n, 256, 0, s>>>(c.X, L.attn_norm, g.rms_norm_eps, g.dim, c.A16); nl++;
        if ((rc = gemm(F32(), "QKV", c.mA, m.qkv, m.qkv, mq.qkv_q, mq.qkv_s, L.tqkv, c.mQKV, c.QKV, nqkv, nqkv / pg::BN, g.dim, 1, 1.0f))) return rc;
        if (ck.n_hist) { // rows written by earlier chunks / decode steps
            const size_t n4 = (size_t)ck.max_start * p->kvd / 4;
            const dim3 hg((unsigned)((n4 + 255) / 256 < 1184 ? (n4 + 255) / 256 : 1184), ck.n_hist);
            k_pf_kv_to_f16_packed<<<hg, 256, 0, s>>>(kc, vc, slot_stride, ck.KH, ck.VH, p->kvd, ck.hist);
            nl++;
        }
        const dim3 ag(ck.n_tiles, g.n_kv_heads);
        rc = with_mma_head_size(p, g.head_size, [&](auto HS) {
            k_pf_rope_kv_packed<HS><<<n, 256, 0, s>>>(c.QKV, nqkv, kc, vc, slot_stride, ck.KH, ck.VH, p->kvd, g.n_heads, g.n_kv_heads, p->kflags, L.q_norm, L.k_norm, L.qkv_bias, g.rms_norm_eps, p->rope_cr, p->rope_ci, ck.tok);
            k_pf_attention_mma_packed<HS><<<ag, PM_THREADS, pm_smem_bytes<HS>(), s>>>(c.QKV, nqkv, ck.KH, ck.VH, p->kvd, kv_mul, ck.tiles, inv_sqrt_hs, c.ATT16, p->qd);
            return B200_OK;
        });
        if (rc) return rc;
        nl += 2;
        const int sp_wo = splits(g.dim / pg::BN, p->qd), sp_w2 = splits(g.dim / pg::BN, g.hidden_dim);
        const float rs = p->mup.residual_scale;
        if ((rc = gemm(RESID(), "Wo", c.mATT, m.wo, m.wo, mq.wo_q, mq.wo_s, L.two, c.mX, c.X, g.dim, g.dim / pg::BN, p->qd, sp_wo, rs))) return rc;
        k_pf_rmsnorm_f16<<<n, 256, 0, s>>>(c.X, L.ffn_norm, g.rms_norm_eps, g.dim, c.A16); nl++;
        if ((rc = gemm(GATEUP(), "gate/up", c.mA, m.w1, m.w3, mq.gu_q, mq.gu_s, L.tgu, c.mX, c.H16, g.hidden_dim, g.hidden_dim / (pg::BN / 2), g.dim, 1, 1.0f)))
            return rc;
        if ((rc = gemm(RESID(), "W2", c.mH, m.w2, m.w2, mq.w2_q, mq.w2_s, L.tw2, c.mX, c.X, g.dim, g.dim / pg::BN, g.hidden_dim, sp_w2, rs))) return rc;
    }
    CK(cudaGetLastError());
    CK(cudaEventRecord(p->ev1, s));
    CK(cudaStreamSynchronize(s));
    CK(cudaEventElapsedTime(&p->prefill_ms, p->ev0, p->ev1));
    p->launches_prefill = nl;
    return B200_OK;
}

// ---- the bit-exact tensor-core prefill (prefill_i8.cuh) -----------------------------------------------------------------------
cudaError_t launch_kq_tiles_to_q8(const TileMat &W, const TileMat &Q, unsigned char *out, cudaStream_t s) {
    const long long n = (long long)tile_groups(Q) * 4 * Q.nseg * (Q.seg / 32);
    const unsigned grid = (unsigned)((n + 127) / 128);
    if (W.fmt == 12) k_kq_tiles_to_q8<12><<<grid, 128, 0, s>>>(W, Q.seg, Q.nseg, Q.unit_bytes, out);
    else if (W.fmt == 13) k_kq_tiles_to_q8<13><<<grid, 128, 0, s>>>(W, Q.seg, Q.nseg, Q.unit_bytes, out);
    else if (W.fmt == 14) k_kq_tiles_to_q8<14><<<grid, 128, 0, s>>>(W, Q.seg, Q.nseg, Q.unit_bytes, out);
    else return cudaErrorInvalidValue;
    return cudaGetLastError();
}

// The quant / scale maps of W's Q8_0 tiles: W itself, or for a resident W the expansion scratch.
bool i8_b_maps(const b200_plan *p, CUtensorMap *q, CUtensorMap *s, const TileMat &w) {
    const TileMat t = q8_geometry(w);
    const unsigned char *base = w.fmt ? p->pi8.kq8 : w.base;
    const uint64_t rows = (uint64_t)tile_groups(t) * 4; // a classifier's last 4-row group is stored zero-padded
    return pg::make_map_i8_q8(q, base, rows, t.nseg, t.unit_bytes, 0) == 0 && pg::make_map_i8_q8(s, base, rows, t.nseg, t.unit_bytes, 1) == 0;
}

// Every layer's stream maps (pi8.maps); false if a tensor map was rejected.  An MoE layer has no dense FFN: its gate/up and W2
// slots hold the shared expert's streams (Qwen2-MoE) or nothing (Qwen3-MoE).
bool i8_weight_maps(b200_plan *p) {
    PrefillI8Ctx &c = p->pi8;
    c.maps.resize(p->cfg.n_layers);
    for (int l = 0; l < p->cfg.n_layers; l++) {
        const LayerW &L = p->layers[l];
        PrefillQ8Maps &m = c.maps[l];
        if (!(i8_b_maps(p, &m.qkv_q, &m.qkv_s, L.tqkv) && i8_b_maps(p, &m.wo_q, &m.wo_s, L.two)))
            return false;
        if (p->is_moe && !p->moe_shared) continue;
        const TileMat &gu = p->is_moe ? L.sgu : L.tgu, &w2 = p->is_moe ? L.sdn : L.tw2;
        if (!(i8_b_maps(p, &m.gu_q, &m.gu_s, gu) && i8_b_maps(p, &m.w2_q, &m.w2_s, w2))) return false;
    }
    return true;
}

// The FFN hidden width of the chunk's HQ / HS rows: the dense hidden dim, or an MoE plan's shared expert's (0 on Qwen3-MoE).
int i8_hidden(const b200_plan *p) { return p->is_moe ? p->moe.shared_hidden_dim : p->cfg.hidden_dim; }

// tensor_core_exact_moe's buffers (pi8.xp) for bpad chunk rows, and the per-expert tensor maps: 4 per expert per layer, encoded
// on the host from each layer's stream-base tables and copied to the device once.  *ok = false if a tensor map was rejected.
int prefill_init_xp(b200_plan *p, bool *ok) {
    PrefillI8Ctx &c = p->pi8;
    XpCtx &x = c.xp;
    const b200_config &g = p->cfg;
    const int E = p->moe.n_experts, k = p->moe.n_experts_used, He = p->moe.expert_hidden_dim, nl = g.n_layers;
    const size_t na = (size_t)c.bpad * k, ga = na + pg::BM; // grouped rows, and what a tile of the last one may read
    const int lds_d = pg::i8_lds(g.dim), lds_e = pg::i8_lds(He);
    *ok = true;
    if (x.maps) return B200_OK;
    int rc;
    auto zero = [&](auto **ptr, size_t bytes) {
        int r = dalloc(p, ptr, bytes);
        if (!r && cudaMemset(*ptr, 0, bytes) != cudaSuccess) r = fail(p, B200_ERR_CUDA, "cudaMemset failed");
        return r;
    };
    if ((rc = zero(&x.XB, (size_t)c.bpad * g.dim * 4)) || (rc = zero(&x.ids, (size_t)nl * na * 4)) || (rc = zero(&x.w, (size_t)nl * c.bpad * p->moe_nw * 4)) ||
        (rc = zero(&x.row_of, na * 4)) || (rc = zero(&x.offsets, (size_t)(E + 1) * 4)) || (rc = zero(&x.n_tiles, 4)) ||
        (rc = zero(&x.tiles, (size_t)pg::xp_max_tiles((int)na, E) * sizeof(pg::XpTile))) || (rc = zero(&x.GQ, ga * g.dim)) ||
        (rc = zero(&x.GS, ga * lds_d * 4)) || (rc = zero(&x.HQg, ga * He)) || (rc = zero(&x.HSg, ga * lds_e * 4)) || (rc = zero(&x.Yg, na * g.dim * 4)) ||
        (p->moe_shared && (rc = zero(&x.Ys, (size_t)c.bpad * g.dim * 4))))
        return rc;
    *ok = pg::make_map_i8_a(&x.a_g, x.GQ, ga, g.dim) == 0 && pg::make_map_i8_s(&x.s_g, x.GS, ga, lds_d) == 0 && pg::make_map_i8_a(&x.a_hg, x.HQg, ga, He) == 0 &&
          pg::make_map_i8_s(&x.s_hg, x.HSg, ga, lds_e) == 0;
    std::vector<CUtensorMap> h((size_t)nl * E * 4);
    std::vector<const unsigned char *> gu(E), dn(E);
    for (int l = 0; l < nl && *ok; l++) {
        const LayerW &L = p->layers[l];
        CK(cudaMemcpy(gu.data(), L.gu_bases, (size_t)E * sizeof(void *), cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(dn.data(), L.dn_bases, (size_t)E * sizeof(void *), cudaMemcpyDeviceToHost));
        for (int e = 0; e < E && *ok; e++) {
            TileMat tg = L.xgu, td = L.xdn;
            tg.base = gu[e];
            td.base = dn[e];
            CUtensorMap *m = &h[((size_t)l * E + e) * 4];
            *ok = i8_b_maps(p, m, m + 1, tg) && i8_b_maps(p, m + 2, m + 3, td);
        }
    }
    if (!*ok) return B200_OK;
    CUtensorMap *maps = nullptr;
    if ((rc = dalloc(p, &maps, h.size() * sizeof(CUtensorMap)))) return rc;
    CK(cudaMemcpy(maps, h.data(), h.size() * sizeof(CUtensorMap), cudaMemcpyHostToDevice));
    x.maps = maps;
    return B200_OK;
}

// Built on the first b200_set_prefill_mode(TENSOR_CORE_EXACT): the chunk buffers and tensor maps over the plan's own Q8_0 streams,
// nothing per weight.  A resident plan adds one scratch, the Q8_0 tiles of its largest resident matrix, and its resident matrices'
// maps point there; the scratch and the chunk buffers must fit the free memory (memory_free) or the call fails with
// B200_ERR_OOM.
int prefill_init_i8(b200_plan *p) {
    PrefillI8Ctx &c = p->pi8;
    const b200_config &g = p->cfg;
    const int nqkv = p->qd + 2 * p->kvd;
    int64_t kq8_bytes = 0;
    for (const LayerW &L : p->layers)
        for (const TileMat *t : {&L.tqkv, &L.two, &L.tgu, &L.tw2})
            if (t->fmt && tile_bytes(q8_geometry(*t)) > kq8_bytes) kq8_bytes = tile_bytes(q8_geometry(*t));
    const int bpad = (p->prefill_batch + pg::BM - 1) / pg::BM * pg::BM, big = g.dim > p->qd ? g.dim : p->qd, hid = i8_hidden(p);
    const int lds_big = pg::i8_lds(big), lds_h = pg::i8_lds(hid);
    int att_tokens = bpad;
    if (p->att_scratch) {
        const size_t row = (size_t)p->nh_l * g.context_length * 4;
        att_tokens = I8_ATT_SCRATCH_MAX / row < 1 ? 1 : (int)(I8_ATT_SCRATCH_MAX / row < (size_t)bpad ? I8_ATT_SCRATCH_MAX / row : bpad);
    }
    const size_t sizes[7] = {(size_t)bpad * g.dim * 4, (size_t)bpad * nqkv * 4, (size_t)bpad * big, (size_t)bpad * lds_big * 4,
                             (size_t)bpad * hid, (size_t)bpad * lds_h * 4, (size_t)bpad * sizeof(ChunkTok)};
    const size_t att_bytes = p->att_scratch ? (size_t)att_tokens * p->nh_l * g.context_length * 4 : 0;
    int rc;
    if (kq8_bytes && !c.kq8) {
        int64_t chunk_bytes = 0, avail;
        if (!c.bpad) {
            for (size_t b : sizes) chunk_bytes += (int64_t)b;
            chunk_bytes += (int64_t)att_bytes;
        }
        if ((rc = memory_free(p, &avail))) return rc;
        if (kq8_bytes + chunk_bytes > avail)
            return fail(p, B200_ERR_OOM, "the bit-exact tensor-core prefill of this resident plan needs %lld bytes of Q8_0 scratch for its largest resident "
                        "matrix and %lld bytes of chunk buffers, %lld bytes are free", (long long)kq8_bytes, (long long)chunk_bytes, (long long)avail);
    }
    if (!c.bpad) {
        c.att_tokens = att_tokens;
        void **dst[7] = {(void **)&c.X, (void **)&c.QKV, (void **)&c.XQ, (void **)&c.XS, (void **)&c.HQ, (void **)&c.HS, (void **)&c.tok};
        for (int i = 0; i < 7; i++) {
            if ((rc = dalloc(p, (unsigned char **)dst[i], sizes[i]))) return rc;
            CK(cudaMemset(*dst[i], 0, sizes[i]));
        }
        if (p->att_scratch && (rc = dalloc(p, &c.att, att_bytes))) return rc;
        c.bpad = bpad;
    }
    if (kq8_bytes && !c.kq8) {
        if ((rc = dalloc(p, &c.kq8, (size_t)kq8_bytes))) return rc;
        c.kq8_bytes = kq8_bytes;
    }
    bool ok = pg::make_map_i8_a(&c.a_dim, c.XQ, c.bpad, g.dim) == 0 && pg::make_map_i8_s(&c.s_dim, c.XS, c.bpad, pg::i8_lds(g.dim)) == 0 &&
              pg::make_map_i8_a(&c.a_qd, c.XQ, c.bpad, p->qd) == 0 && pg::make_map_i8_s(&c.s_qd, c.XS, c.bpad, pg::i8_lds(p->qd)) == 0 &&
              (!hid || (pg::make_map_i8_a(&c.a_h, c.HQ, c.bpad, hid) == 0 && pg::make_map_i8_s(&c.s_h, c.HS, c.bpad, lds_h) == 0));
    if (p->is_moe) {
        bool xp_ok = false;
        if ((rc = prefill_init_xp(p, &xp_ok))) return rc;
        ok = ok && xp_ok;
    }
    return prefill_built(p, p->is_moe ? B200_PREFILL_TENSOR_CORE_EXACT_MOE : B200_PREFILL_TENSOR_CORE_EXACT, ok && i8_weight_maps(p));
}

// k_i8_norm over chunk rows [0, n) of c.X into XQ / XS (and the float rows into xb, if given); embed (layer 0): each row's
// embedding is gathered into c.X first.
void i8_norm(b200_plan *p, int n, bool embed, const float *w, float *xb = nullptr) {
    PrefillI8Ctx &c = p->pi8;
    const b200_config &g = p->cfg;
    const size_t norm_smem = norm_smem_bytes(g.dim);
    const int lds_d = pg::i8_lds(g.dim);
    const TraceBuf tr{nullptr, 0, 0};
    TpCtx solo{};
    solo.n = 1;
    if (embed) k_i8_norm<true><<<n, NORM_THREADS, norm_smem, p->stream>>>(c.X, c.tok, p->emb, p->mup.embedding_scale, w, g.rms_norm_eps, g.dim, c.XQ, c.XS, lds_d, xb, tr, solo);
    else k_i8_norm<false><<<n, NORM_THREADS, norm_smem, p->stream>>>(c.X, c.tok, p->emb, p->mup.embedding_scale, w, g.rms_norm_eps, g.dim, c.XQ, c.XS, lds_d, xb, tr, solo);
}

// The routed experts of MoE layer l over the chunk's n rows (tensor_core_exact_moe), after the FFN norm (XQ / XS and the float rows
// xp.XB) and, on Qwen2-MoE, the shared expert's down projection into xp.Ys: the chunk router, the grouping of the n * k
// assignments by expert, the gather of each assignment's activation row, the grouped gate/up and down GEMMs, and the ordered
// combine into c.X.  Six launches.
int enqueue_chunk_moe(b200_plan *p, int l, int n, int *nl) {
    PrefillI8Ctx &c = p->pi8;
    XpCtx &x = c.xp;
    const b200_config &g = p->cfg;
    const LayerW &L = p->layers[l];
    cudaStream_t s = p->stream;
    const int E = p->moe.n_experts, k = p->moe.n_experts_used, He = p->moe.expert_hidden_dim, nw = p->moe_nw, na = n * k;
    int *ids = x.ids + (size_t)l * c.bpad * k;
    float *w = x.w + (size_t)l * c.bpad * nw;
    XpRouteArgs ra{L.router, L.shared_gate, x.XB, ids, w, n, g.dim, E, k, nw};
    const unsigned rg = (unsigned)((n + XP_ROUTE_TOKENS - 1) / XP_ROUTE_TOKENS);
    if (p->moe_shared) k_xp_route<true><<<rg, MOE_ROUTE_THREADS, 0, s>>>(ra);
    else k_xp_route<false><<<rg, MOE_ROUTE_THREADS, 0, s>>>(ra);
    pg::k_xp_group<<<1, pg::XP_GROUP_THREADS, 0, s>>>(ids, na, E, x.row_of, x.offsets, x.tiles, x.n_tiles);
    pg::k_xp_gather<<<na, 128, 0, s>>>(c.XQ, c.XS, g.dim, pg::i8_lds(g.dim), k, x.row_of, x.GQ, x.GS);
    CK(cudaGetLastError());
    const CUtensorMap *maps = x.maps + (size_t)l * E * 4;
    const int gm = pg::xp_max_tiles(na, E);
    pg::I8Out o{};
    o.hq = x.HQg; o.hs = x.HSg; o.ldq = He; o.lds = pg::i8_lds(He); o.K = g.dim; o.seg = L.xgu.seg; o.oscale = 1.0f;
    if (pg::xp_gemm_launch<pg::GEMM_GATEUP>(x.a_g, x.s_g, maps, x.tiles, x.n_tiles, o, gm, L.xgu.rows / pg::I8_BN, s))
        return fail(p, B200_ERR_CUDA, "grouped expert gate/up GEMM launch failed");
    o = pg::I8Out{};
    o.C = x.Yg; o.ldc = g.dim; o.K = He; o.seg = L.xdn.seg; o.oscale = 1.0f;
    if (pg::xp_gemm_launch<pg::GEMM_F32>(x.a_hg, x.s_hg, maps, x.tiles, x.n_tiles, o, gm, L.xdn.rows / pg::I8_BN, s))
        return fail(p, B200_ERR_CUDA, "grouped expert down GEMM launch failed");
    pg::k_xp_combine<<<n, 256, 0, s>>>(c.X, g.dim, x.Yg, x.row_of, w, k, nw, p->moe_shared ? x.Ys : nullptr);
    CK(cudaGetLastError());
    *nl += 6;
    return B200_OK;
}

// The layers of one chunk over its n rows, whose ChunkTok entries (token, position, KV offset) are already in c.tok: the batched
// step's graph (enqueue_batch) over the whole chunk, its Q8_0 streams replaced by k_gemm_i8.  own: the K / V go to the plan's cache,
// else to the decode slots.  Leaves each row's final residual in row v of c.X and adds its launches to *nl; enqueued only (no events,
// no synchronise), so prefill_forward_i8 and b200_forward_chunk wrap it in their own tails.
int enqueue_chunk_i8(b200_plan *p, int n, bool own, int *nl_out) {
    PrefillI8Ctx &c = p->pi8;
    const b200_config &g = p->cfg;
    cudaStream_t s = p->stream;
    const int nqkv = p->qd + 2 * p->kvd, mt = (n + pg::BM - 1) / pg::BM, hid = i8_hidden(p);
    const int lds_q = pg::i8_lds(p->qd), lds_h = pg::i8_lds(hid);
    const size_t ctx_kv = (size_t)g.context_length * p->kvd;
    const size_t att_smem = att_smem_bytes(g.head_size, g.context_length, c.att != nullptr);
    const TraceBuf tr{nullptr, 0, 0};
    TpCtx solo{};
    solo.n = 1;
    int &nl = *nl_out, rc = 0;
    auto norm = [&](bool embed, const float *w) {
        i8_norm(p, n, embed, w);
        nl++;
    };
    // one k_gemm_i8 over the stream W; n_tiles from W's rows (64 stream rows per tile).  A resident W is first expanded to its Q8_0
    // tiles in c.kq8, where its maps point; stream order (k_gemm_i8 is launched without PDL) orders the expansion between the
    // previous GEMM's reads of the scratch and this GEMM's.
    auto gemm = [&](auto MODE, const CUtensorMap &a, const CUtensorMap &as, const CUtensorMap &bq, const CUtensorMap &bs, const TileMat &W, float *C, int ldc,
                    float oscale) {
        const TileMat Q = q8_geometry(W);
        if (W.fmt) {
            CK(launch_kq_tiles_to_q8(W, Q, c.kq8, s));
            nl++;
        }
        pg::I8Out o{};
        o.C = C; o.ldc = ldc; o.hq = c.HQ; o.hs = c.HS; o.ldq = hid; o.lds = lds_h;
        o.m_valid = n; o.K = Q.cols; o.seg = Q.seg; o.oscale = oscale;
        nl++;
        return pg::gemm_i8_launch<decltype(MODE)::value>(a, as, bq, bs, o, mt, Q.rows / pg::I8_BN, s) ? fail(p, B200_ERR_CUDA, "int8 GEMM launch failed") : B200_OK;
    };
    using F32 = std::integral_constant<int, pg::GEMM_F32>;
    using RESID = std::integral_constant<int, pg::GEMM_RESID>;
    using GATEUP = std::integral_constant<int, pg::GEMM_GATEUP>;
    const float rs = p->mup.residual_scale;
    for (int l = 0; l < g.n_layers; l++) {
        const LayerW &L = p->layers[l];
        const PrefillQ8Maps &m = c.maps[l];
        float *kc = (own ? p->key_cache : p->bt.slot_k) + (size_t)l * ctx_kv, *vc = (own ? p->value_cache : p->bt.slot_v) + (size_t)l * ctx_kv;
        norm(l == 0, L.attn_norm);
        if ((rc = gemm(F32(), c.a_dim, c.s_dim, m.qkv_q, m.qkv_s, L.tqkv, c.QKV, nqkv, 1.0f))) return rc;
        rc = with_decode_head_size(p, g.head_size, [&](auto HS) {
            k_i8_rope_kv<HS><<<dim3(p->nh_l, n), 2 * HS, 0, s>>>(c.QKV, nqkv, kc, vc, c.tok, p->rope_cr, p->rope_ci, p->nh_l, p->nkv_l, p->kflags, L.q_norm,
                                                              L.k_norm, L.qkv_bias, g.rms_norm_eps);
            nl++;
            for (int v0 = 0; v0 < n; v0 += c.att_tokens, nl++) // every K / V row of the chunk is in the cache before any attention reads it
                k_i8_attention<HS><<<dim3(p->nh_l, n - v0 < c.att_tokens ? n - v0 : c.att_tokens), ATT_THREADS, att_smem, s>>>(
                    c.QKV, nqkv, kc, vc, c.tok, v0, p->nh_l, p->nkv_l, p->kflags, att_score_arg(p), c.XQ, c.XS, lds_q, c.att, g.context_length, tr, solo);
            return B200_OK;
        });
        if (rc) return rc;
        if ((rc = gemm(RESID(), c.a_qd, c.s_qd, m.wo_q, m.wo_s, L.two, c.X, g.dim, rs))) return rc;
        if (p->is_moe) { // the MoE FFN over the chunk: the FFN norm with float rows for the router, then enqueue_chunk_moe
            i8_norm(p, n, false, L.ffn_norm, c.xp.XB);
            nl++;
            if (p->moe_shared) { // the shared expert on the token rows: gate/up into HQ / HS, down into Ys
                if ((rc = gemm(GATEUP(), c.a_dim, c.s_dim, m.gu_q, m.gu_s, L.sgu, nullptr, 0, 1.0f))) return rc;
                if ((rc = gemm(F32(), c.a_h, c.s_h, m.w2_q, m.w2_s, L.sdn, c.xp.Ys, g.dim, 1.0f))) return rc;
            }
            if ((rc = enqueue_chunk_moe(p, l, n, &nl))) return rc;
            continue;
        }
        norm(false, L.ffn_norm);
        if ((rc = gemm(GATEUP(), c.a_dim, c.s_dim, m.gu_q, m.gu_s, L.tgu, nullptr, 0, 1.0f))) return rc;
        if ((rc = gemm(RESID(), c.a_h, c.s_h, m.w2_q, m.w2_s, L.tw2, c.X, g.dim, rs))) return rc;
    }
    CK(cudaGetLastError());
    return B200_OK;
}

// One chunk: tab[v] = (token, position, KV offset) of chunk row v; own: the K / V go to the plan's cache, else to the decode slots.
// enqueue_chunk_i8, timed (p->prefill_ms) with its launches counted (p->launches_prefill).  score (b200_score_tokens, after
// score_init_i8): then the final norm, the classifier (expanded first on a resident plan) into p->sc.logits SCORE_GROUP_ROWS rows at
// a time, and k_score_rows over each group into p->sc.out.
int prefill_forward_i8(b200_plan *p, const std::vector<ChunkTok> &tab, bool own, bool score = false) {
    PrefillI8Ctx &c = p->pi8;
    const b200_config &g = p->cfg;
    cudaStream_t s = p->stream;
    const int n = (int)tab.size(), lds_d = pg::i8_lds(g.dim);
    CK(cudaMemcpyAsync(c.tok, tab.data(), (size_t)n * sizeof(ChunkTok), cudaMemcpyHostToDevice, s));
    if (p->is_moe) c.xp.rows = n;
    CK(cudaEventRecord(p->ev0, s));
    int nl = 0, rc;
    if ((rc = enqueue_chunk_i8(p, n, own, &nl))) return rc;
    if (score) {
        auto &S = p->sc;
        const TileMat Q = q8_geometry(p->tout);
        i8_norm(p, n, false, p->out_norm);
        nl++;
        if (p->tout.fmt) {
            CK(launch_kq_tiles_to_q8(p->tout, Q, c.kq8, s));
            nl++;
        }
        for (int r0 = 0; r0 < n; r0 += SCORE_GROUP_ROWS) {
            const int rows = n - r0 < SCORE_GROUP_ROWS ? n - r0 : SCORE_GROUP_ROWS;
            CUtensorMap a, as; // the group's activation rows
            if (pg::make_map_i8_a(&a, c.XQ + (size_t)r0 * g.dim, c.bpad - r0, g.dim) || pg::make_map_i8_s(&as, c.XS + (size_t)r0 * lds_d, c.bpad - r0, lds_d))
                return fail(p, B200_ERR_CUDA, "cuTensorMapEncodeTiled rejected a tensor map");
            pg::I8Out o{};
            o.C = S.logits; o.ldc = S.ldl; o.m_valid = rows; o.K = Q.cols; o.seg = Q.seg; o.oscale = out_scale(p, false, true);
            if (pg::gemm_i8_launch<pg::I8_LOGITS>(a, as, S.cls_q, S.cls_s, o, (rows + pg::BM - 1) / pg::BM, S.ldl / pg::I8_BN, s))
                return fail(p, B200_ERR_CUDA, "int8 classifier GEMM launch failed");
            k_score_rows<<<rows, SCORE_THREADS, 0, s>>>(S.logits, S.ldl, g.vocab_size, S.tgt + r0, S.out + r0);
            nl += 2;
        }
    }
    CK(cudaGetLastError());
    CK(cudaEventRecord(p->ev1, s));
    CK(cudaStreamSynchronize(s));
    CK(cudaEventElapsedTime(&p->prefill_ms, p->ev0, p->ev1));
    p->launches_prefill = nl;
    return B200_OK;
}

const char *const PREFILL_MODE_NAMES[5] = {"exact", "tensor_core", "tensor_core_w8a16", "tensor_core_exact", "tensor_core_exact_moe"};

// The chunk path the plan's prefill mode runs: the bit-exact int8 one (prefill_i8.cuh), the f16 / W8A16 one (prefill.cuh), or
// none (the exact token-by-token and multi-position paths).
enum ChunkPath { CHUNK_NONE, CHUNK_TC, CHUNK_I8 };
ChunkPath chunk_path(const b200_plan *p) {
    constexpr ChunkPath PATHS[5] = {CHUNK_NONE, CHUNK_TC, CHUNK_TC, CHUNK_I8, CHUNK_I8};
    return PATHS[p->pf_mode];
}

// One chunk on the tensor-core path chunk_path selects: the tokens of ns sequences back to back (call order, no padding),
// sequence i at positions start[i] .. start[i] + len[i] - 1 of slot slots[i] -- of the decode slots, or, own, of the plan's cache
// (one sequence, slot 0).  Sequences of length 0 take no part.  score: see prefill_forward_i8.
int prefill_chunk(b200_plan *p, int ns, const int *slots, const int *start, const int *len, const int *tokens, bool own, bool score = false) {
    const b200_config &g = p->cfg;
    if (chunk_path(p) == CHUNK_I8) {
        const size_t slot_stride = (size_t)g.n_layers * g.context_length * p->kvd;
        std::vector<ChunkTok> tab;
        for (int i = 0, off = 0; i < ns; off += len[i++])
            for (int j = 0; j < len[i]; j++) tab.push_back(ChunkTok{tokens[off + j], start[i] + j, (long long)(slots[i] * slot_stride)});
        return prefill_forward_i8(p, tab, own, score);
    }
    // Sequence i's f16 K / V region holds its rows [0, start + len) from scratch row hrow[i].
    PrefillCtx &c = p->prefill;
    std::vector<int> n, st, row0, hrow;
    std::vector<PfTok> tok;
    std::vector<PfHist> hist;
    size_t rows = 0;
    int total = 0, max_start = 0;
    for (int i = 0; i < ns; total += len[i++]) {
        if (!len[i]) continue;
        n.push_back(len[i]); st.push_back(start[i]); row0.push_back(total); hrow.push_back((int)rows);
        for (int j = 0; j < len[i]; j++) tok.push_back(PfTok{start[i] + j, slots[i], (int)rows + start[i] + j});
        if (start[i] > 0) {
            hist.push_back(PfHist{slots[i], start[i], (int)rows});
            if (start[i] > max_start) max_start = start[i];
        }
        rows += (size_t)start[i] + len[i];
    }
    const std::vector<PfTile> tiles = pf_tiles((int)n.size(), n.data(), st.data(), row0.data(), hrow.data(), g.n_heads / g.n_kv_heads);
    auto up16 = [](size_t x) { return (x + 15) & ~(size_t)15; };
    const size_t o_tiles = up16(tok.size() * sizeof(PfTok)), o_hist = o_tiles + up16(tiles.size() * sizeof(PfTile));
    const size_t bytes = o_hist + hist.size() * sizeof(PfHist) + 16;
    const bool big = rows > (size_t)g.context_length; // more than one sequence's worth: the grown regions
    if ((big && rows > c.pk_rows) || bytes > c.ptab_bytes) CK(cudaStreamSynchronize(p->stream)); // the buffers below are reallocated
    if (big && rows > c.pk_rows) {
        CK(cudaFree(c.PKH)); CK(cudaFree(c.PVH));
        c.PKH = c.PVH = nullptr; c.pk_rows = 0;
        CK(cudaMalloc(&c.PKH, rows * p->kvd * 2));
        CK(cudaMalloc(&c.PVH, rows * p->kvd * 2));
        c.pk_rows = rows;
    }
    if (bytes > c.ptab_bytes) {
        CK(cudaFree(c.ptab));
        c.ptab = nullptr; c.ptab_bytes = 0;
        CK(cudaMalloc(&c.ptab, bytes));
        c.ptab_bytes = bytes;
    }
    std::vector<unsigned char> h(bytes, 0);
    memcpy(h.data(), tok.data(), tok.size() * sizeof(PfTok));
    memcpy(h.data() + o_tiles, tiles.data(), tiles.size() * sizeof(PfTile));
    if (!hist.empty()) memcpy(h.data() + o_hist, hist.data(), hist.size() * sizeof(PfHist));
    // pageable sources: both copies are staged before cudaMemcpyAsync returns
    CK(cudaMemcpyAsync(c.ptab, h.data(), bytes, cudaMemcpyHostToDevice, p->stream));
    CK(cudaMemcpyAsync(c.tok, tokens, (size_t)total * 4, cudaMemcpyHostToDevice, p->stream));
    PfChunk ck{};
    ck.tok = reinterpret_cast<const PfTok *>(c.ptab);
    ck.tiles = reinterpret_cast<const PfTile *>(c.ptab + o_tiles);
    ck.n_tiles = (int)tiles.size();
    ck.hist = reinterpret_cast<const PfHist *>(c.ptab + o_hist);
    ck.n_hist = (int)hist.size();
    ck.max_start = max_start;
    ck.KH = big ? c.PKH : c.KH;
    ck.VH = big ? c.PVH : c.VH;
    ck.own = own;
    return prefill_forward(p, total, ck);
}

// The single-token graphs the forward calls launch: the persistent kernel's when that mode is selected and captured.
const TokenGraphs &active_graphs(const b200_plan *p) { return p->decode_mode == B200_DECODE_PERSISTENT && p->pers.decode.exec ? p->pers : p->graph; }
cudaGraphExec_t decode_graph(const b200_plan *p) { return active_graphs(p).decode.exec; }
cudaGraphExec_t prefill_graph(const b200_plan *p) { return active_graphs(p).prefill.exec; }

// The checks b200_set_sampling_controls and b200_test_sample_controls share (p may be NULL).
int check_controls(b200_plan *p, const b200_sampling_controls &c, int vocab) {
    if (c.top_k < 0 || c.top_k > vocab) return fail(p, B200_ERR_BAD_ARG, "top_k = %d outside [0, %d]", c.top_k, vocab);
    if (!(c.min_p >= 0.0f && c.min_p <= 1.0f)) return fail(p, B200_ERR_BAD_ARG, "min_p = %g outside [0, 1]", c.min_p);
    if (!(isfinite(c.repetition_penalty) && c.repetition_penalty > 0.0f))
        return fail(p, B200_ERR_BAD_ARG, "repetition_penalty = %g: must be finite and > 0", c.repetition_penalty);
    if (!isfinite(c.frequency_penalty) || !isfinite(c.presence_penalty))
        return fail(p, B200_ERR_BAD_ARG, "frequency_penalty = %g, presence_penalty = %g: must be finite", c.frequency_penalty, c.presence_penalty);
    if (c.n_bias < 0 || c.n_bias > B200_MAX_LOGIT_BIAS) return fail(p, B200_ERR_BAD_ARG, "n_bias = %d outside [0, %d]", c.n_bias, B200_MAX_LOGIT_BIAS);
    if (c.n_bias && (!c.bias_ids || !c.bias_values)) return fail(p, B200_ERR_BAD_ARG, "n_bias = %d with a NULL bias list", c.n_bias);
    std::vector<char> seen(c.n_bias ? vocab : 0, 0);
    for (int b = 0; b < c.n_bias; b++) {
        const int i = c.bias_ids[b];
        if (i < 0 || i >= vocab) return fail(p, B200_ERR_BAD_ARG, "bias entry %d: id %d out of range", b, i);
        if (seen[i]++) return fail(p, B200_ERR_BAD_ARG, "bias entry %d: id %d repeats an earlier entry", b, i);
        if (!isfinite(c.bias_values[b])) return fail(p, B200_ERR_BAD_ARG, "bias entry %d: value %g is not finite", b, c.bias_values[b]);
    }
    return B200_OK;
}

float min_p_log(float min_p) { return (float)log((double)min_p); } // -inf for 0: the min-p mask keeps everything

// One k_sample_ctl row: sequence s's controls and counts, raw row src, modified row dst, the sampler's scratch and outputs.
SampleCtlRow ctl_row(b200_plan *p, int s, const float *src, float *dst, int *indices, int *out, float temperature, float topp, float uniform01) {
    const auto &S = p->ctl;
    const b200_sampling_controls &c = S.c[s];
    SampleCtlRow r;
    r.src = src; r.dst = dst; r.row_out = nullptr; r.cnt = S.cnt + (size_t)s * p->cfg.vocab_size;
    r.bias_id = S.bias_id + (size_t)s * B200_MAX_LOGIT_BIAS; r.bias_val = S.bias_val + (size_t)s * B200_MAX_LOGIT_BIAS; r.n_bias = c.n_bias;
    r.top_k = c.top_k; r.min_p_log = S.min_p_log[s]; r.rep = c.repetition_penalty; r.freq = c.frequency_penalty; r.pres = c.presence_penalty;
    r.temperature = temperature; r.topp = topp; r.r01 = uniform01;
    r.indices = indices; r.out = out;
    return r;
}

// Zero the counts of sequences [s0, s1) if the tables exist (on the plan's stream; the caller synchronises).
int clear_counts(b200_plan *p, int s0, int s1) {
    if (p->ctl.cnt) CK(cudaMemsetAsync(p->ctl.cnt + (size_t)s0 * p->cfg.vocab_size, 0, (size_t)(s1 - s0) * p->cfg.vocab_size * 4, p->stream));
    return B200_OK;
}

// k_token_logprobs on n rows: row k of logits (stride floats apart) emitted *ids[k] and fills result row out_row[k].
int launch_logprobs(b200_plan *p, const float *logits, long long stride, int n, const int *const *ids, const int *out_row) {
    static_assert(SMB_MAX_ROWS <= LOGPROB_MAX_ROWS, "k_token_logprobs takes every row of a batched step");
    static_assert(B200_MAX_TOP_LOGPROBS == LOGPROB_MAX_TOP, "the header's limit is the kernel's");
    LogprobArgs a{};
    a.logits = logits; a.stride = stride; a.vocab = p->cfg.vocab_size; a.n_top = p->lp.top_n; a.out = p->lp.out;
    for (int k = 0; k < n; k++) { a.ids[k] = ids[k]; a.out_row[k] = out_row[k]; }
    k_token_logprobs<<<n, SCORE_THREADS, 0, p->stream>>>(a);
    CK(cudaGetLastError());
    return B200_OK;
}

// One step of b200_decode_sequence: p->logits, the id at *id, result row `row`.
int launch_logprobs_one(b200_plan *p, const int *id, int row) { return launch_logprobs(p, p->logits, 0, 1, &id, &row); }

// The result rows [0, n) to the pinned table; the caller's synchronise completes the copy.
int copy_logprobs(b200_plan *p, int n) {
    CK(cudaMemcpyAsync(p->lp.h_out, p->lp.out, (size_t)n * sizeof(LogprobRow), cudaMemcpyDeviceToHost, p->stream));
    return B200_OK;
}

// After a synchronize: did a device-side wait of the persistent kernel (or a tensor-parallel flag wait) give up?
int check_device_error(b200_plan *p) {
    if (p->h_err && *reinterpret_cast<volatile unsigned *>(p->h_err)) {
        const unsigned code = *reinterpret_cast<volatile unsigned *>(p->h_err);
        return fail(p, B200_ERR_STATE, "a device-side wait timed out (code %u: 1+phase of the persistent decode kernel, 100+slot of a tensor-parallel flag): a peer "
                                       "rank is missing or the ranks' call sequences diverged; the plan must be freed", code);
    }
    return B200_OK;
}

int set_state(b200_plan *p, int token, int pos, int n_seq, int feedback, int step = 0) {
    StepState *h = p->h_st;
    h->token = token; h->pos = pos; h->step = step; h->n_seq = n_seq; h->feedback = feedback;
    CK(cudaMemcpyAsync(p->st, h, sizeof(StepState), cudaMemcpyHostToDevice, p->stream));
    return B200_OK;
}

int check_pos(b200_plan *p, int token, int pos) {
    if (token < 0 || token >= p->cfg.vocab_size) return fail(p, B200_ERR_BAD_ARG, "token %d out of range", token);
    if (pos < 0 || pos >= p->cfg.context_length) return fail(p, B200_ERR_BAD_ARG, "position %d outside the KV cache (%d)", pos, p->cfg.context_length);
    return B200_OK;
}

// The index of the first of tokens[0, n) outside the vocabulary, or -1; each caller names it in its own terms.
int bad_token(const b200_plan *p, const int32_t *tokens, int n) {
    for (int i = 0; i < n; i++)
        if (tokens[i] < 0 || tokens[i] >= p->cfg.vocab_size) return i;
    return -1;
}

// The checks b200_forward_batch_prefill and b200_score_tokens make of a chunk: its length against prefill_batch_size, its positions,
// its tokens, and on the token-by-token path the step buffers' capacity.
int check_chunk(b200_plan *p, const int32_t *tokens, int32_t n, int32_t start_pos) {
    if (p->prefill_batch > 1 && n > p->prefill_batch) return fail(p, B200_ERR_BAD_ARG, "chunk of %d tokens exceeds prefill_batch_size %d", n, p->prefill_batch);
    if (start_pos < 0 || start_pos + n > p->cfg.context_length) return fail(p, B200_ERR_BAD_ARG, "positions %d..%d outside the KV cache", start_pos, start_pos + n - 1);
    if (const int i = bad_token(p, tokens, n); i >= 0) return fail(p, B200_ERR_BAD_ARG, "token %d out of range", tokens[i]);
    if (chunk_path(p) == CHUNK_NONE && n > p->seq_cap) return fail(p, B200_ERR_BAD_ARG, "chunk too long");
    return B200_OK;
}

// The refusals b200_forward_decode_batch and b200_forward_step share for row i: slot, token and position out of range, and an
// emitting row's bad sampling triple.
int check_row(b200_plan *p, int i, const b200_step_row &r) {
    const b200_config &c = p->cfg;
    if (r.slot < 0 || r.slot >= p->bt.n_slots) return fail(p, B200_ERR_BAD_ARG, "row %d: slot %d out of range (%d slots)", i, r.slot, p->bt.n_slots);
    if (bad_token(p, &r.token, 1) >= 0) return fail(p, B200_ERR_BAD_ARG, "row %d: token %d out of range", i, r.token);
    if (r.position < 0 || r.position >= c.context_length)
        return fail(p, B200_ERR_BAD_ARG, "row %d: position %d outside the KV cache (%d)", i, r.position, c.context_length);
    if (r.emit && (!(r.temperature >= 0.0f) || !(r.uniform01 >= 0.0f && r.uniform01 < 1.0f)))
        return fail(p, B200_ERR_BAD_ARG, "row %d: temperature must be >= 0 and the uniform number in [0, 1)", i);
    return B200_OK;
}

// The refusals b200_forward_step and b200_forward_chunk share, for the first offending row: an emit flag other than 0 / 1, check_row,
// a (slot, position) pair that repeats, more than max_emit emitting rows, and a second emitting row of a slot with sampling controls.
int check_step_rows(b200_plan *p, int n, const b200_step_row *rows, int max_emit) {
    int rc, e = 0, emits[SMB_MAX_ROWS]; // emits[s]: the first emitting row of slot s, or -1
    for (int s = 0; s < SMB_MAX_ROWS; s++) emits[s] = -1;
    std::unordered_map<long long, int> seen; // slot * context_length + position -> row
    for (int i = 0; i < n; i++) {
        const b200_step_row &r = rows[i];
        if (r.emit != 0 && r.emit != 1) return fail(p, B200_ERR_BAD_ARG, "row %d: emit must be 0 or 1 (got %d)", i, r.emit);
        if ((rc = check_row(p, i, r))) return rc;
        const auto at = seen.emplace((long long)r.slot * p->cfg.context_length + r.position, i);
        if (!at.second) return fail(p, B200_ERR_BAD_ARG, "row %d: slot %d position %d repeats row %d's", i, r.slot, r.position, at.first->second);
        if (!r.emit) continue;
        if (++e > max_emit) return fail(p, B200_ERR_BAD_ARG, "row %d: more than %d emitting rows in one call", i, max_emit);
        if (emits[r.slot] >= 0 && p->ctl.on[r.slot + 1])
            return fail(p, B200_ERR_BAD_ARG, "row %d: slot %d has sampling controls and already emits in row %d (its counts would depend on "
                                             "that row's id)", i, r.slot, emits[r.slot]);
        if (emits[r.slot] < 0) emits[r.slot] = i;
    }
    return B200_OK;
}

// The emitting rows first (stable), then the others: order[k] = the caller's index of step row k; returns the emitting rows' count.
int emit_first(int n, const b200_step_row *rows, int *order) {
    int e = 0;
    for (int i = 0; i < n; i++)
        if (rows[i].emit) order[e++] = i;
    for (int i = 0, k = e; i < n; i++)
        if (!rows[i].emit) order[k++] = i;
    return e;
}

// The buffers step_outputs works on: logits rows sampler_padded(vocab) floats apart and their argmax ids, the sampler's outputs
// (8 ints a row: the id, then its four diagnostics) and candidate lists (vocab ints a row), and a pinned block of 9 ints a row
// that receives the e ids, then the e rows of sampler outputs.  The batched steps pass bt's, the single-token calls the plan's own.
struct RowBufs {
    float *logits;
    int *ids, *smp_out, *smp_indices, *h_out;
};

// What a step with the classifier does after it, for every emitting call but b200_decode_sequence: R's rows [0, e) hold the
// emitting rows (step row k is the caller's row order[k], order from emit_first over n rows).  Their logits go back to the caller's
// row order, ids -1 where a row does not emit.  Rows with a temperature run the device sampler, all in one launch.  With controls,
// the emitting rows of sequences with sampling controls (slot + 1; slot -1 is the plan's own) run k_sample_ctl instead, all in one
// launch of their own.  Then the log-probabilities, the readback and the call's one synchronise.  info_out (nullable, 4 ints per
// caller row): an emitting row's sampler diagnostics, zeros where it takes the argmax.
int step_outputs(b200_plan *p, int n, const b200_step_row *rows, const int *order, int e, bool controls, const RowBufs &R, int32_t *ids_out,
                 float *logits, int32_t *info_out = nullptr) {
    static_assert(SMB_MAX_ROWS <= SAMPLER_MAX_ROWS, "k_sample_rows and k_sample_ctl take every row of a batched step");
    static_assert(B200_MAX_LOGIT_BIAS == SAMPLER_CTL_MAX_BIAS, "the header's limit is the kernel's");
    const b200_config &c = p->cfg;
    int rc;
    const size_t vpad = (size_t)sampler_padded(c.vocab_size);
    if (logits) // before the sampler turns sampled rows into probabilities
        for (int k = 0; k < e; k++)
            CK(cudaMemcpyAsync(logits + (size_t)order[k] * c.vocab_size, R.logits + k * vpad, (size_t)c.vocab_size * 4, cudaMemcpyDeviceToHost, p->stream));
    int m = 0, mc = 0;
    bool ctl[SMB_MAX_ROWS];
    SamplerRowsArgs sa;
    SampleCtlArgs ca;
    for (int k = 0; k < e; k++) {
        const b200_step_row &r = rows[order[k]];
        ctl[k] = controls && p->ctl.on[r.slot + 1];
        if (ctl[k]) {
            ca.row[mc++] = ctl_row(p, r.slot + 1, R.logits + k * vpad, p->ctl.rows + k * vpad, R.smp_indices + (size_t)k * c.vocab_size, R.smp_out + 8 * k,
                                   r.temperature, r.topp, r.uniform01);
            continue;
        }
        if (r.temperature == 0.0f) continue; // Sampler.selectSampler: temperature 0 -> FloatTensor.argmax, already computed
        sa.row[m] = k; sa.temperature[m] = r.temperature; sa.topp[m] = r.topp; sa.r01[m] = r.uniform01;
        m++;
    }
    if (mc) {
        ca.n = c.vocab_size;
        k_sample_ctl<<<mc, SAMPLER_THREADS, sampler_smem_bytes(), p->stream>>>(ca);
        CK(cudaGetLastError());
    }
    const bool lp = p->lp.top_n >= 0;
    sa.logits = R.logits; sa.stride = (int)vpad; sa.n = c.vocab_size; sa.indices = R.smp_indices; sa.out = R.smp_out;
    if (lp && m) { // the sampler overwrites its rows with probabilities: it samples copies (zero pad included) in the same layout
        sa.logits = p->lp.smp;
        for (int j = 0; j < m; j++) CK(cudaMemcpyAsync(sa.logits + sa.row[j] * vpad, R.logits + sa.row[j] * vpad, vpad * 4, cudaMemcpyDeviceToDevice, p->stream));
    }
    if (m) {
        k_sample_rows<<<m, SAMPLER_THREADS, sampler_smem_bytes(), p->stream>>>(sa);
        CK(cudaGetLastError());
    }
    if (lp && e) {
        const int *ids[SMB_MAX_ROWS];
        for (int k = 0; k < e; k++) ids[k] = ctl[k] || rows[order[k]].temperature != 0.0f ? R.smp_out + 8 * k : R.ids + k;
        if ((rc = launch_logprobs(p, R.logits, (long long)vpad, e, ids, order))) return rc;
    }
    if (lp && (rc = copy_logprobs(p, n))) return rc;
    if (e) CK(cudaMemcpyAsync(R.h_out, R.ids, (size_t)e * 4, cudaMemcpyDeviceToHost, p->stream));
    if (m || mc) CK(cudaMemcpyAsync(R.h_out + e, R.smp_out, (size_t)e * 8 * 4, cudaMemcpyDeviceToHost, p->stream));
    CK(cudaStreamSynchronize(p->stream));
    if (lp) {
        for (int k = e; k < n; k++) { // rows that do not emit
            LogprobRow &r = p->lp.h_out[order[k]];
            r.chosen = NAN;
            for (int j = 0; j < LOGPROB_MAX_TOP; j++) { r.id[j] = -1; r.lp[j] = NAN; }
        }
        p->lp.rows = n;
    }
    for (int i = 0; i < n; i++) ids_out[i] = -1;
    for (int k = 0; k < e; k++) {
        const bool sampled = ctl[k] || rows[order[k]].temperature != 0.0f;
        ids_out[order[k]] = sampled ? R.h_out[e + 8 * k] : R.h_out[k];
        if (info_out)
            for (int d = 0; d < 4; d++) info_out[4 * order[k] + d] = rows[order[k]].temperature != 0.0f ? R.h_out[e + 8 * k + 1 + d] : 0;
    }
    return B200_OK;
}

// One batched step with the classifier over checked rows: against the decode slots, or with own the plan's cache (every row
// slot 0).  The emitting rows go first, so the final norm, lm_head and argmax run over rows [0, e) and no kernel indexes through a
// row map; step_outputs does the rest.  b200_batch_info reports the step.
int batch_step(b200_plan *p, int n, const b200_step_row *rows, bool own, bool controls, int32_t *ids_out, float *logits) {
    auto &B = p->bt;
    int order[SMB_MAX_ROWS];
    const int e = emit_first(n, rows, order);
    BatchRows br{};
    for (int k = 0; k < n; k++) {
        const b200_step_row &r = rows[order[k]];
        br.token[k] = r.token; br.pos[k] = r.position; br.slot[k] = r.slot;
    }
    int rc;
    const Graph *g;
    if ((rc = batch_graph(p, step_form(br, n, own), n, e, &g))) return rc;
    *B.h_rows = br;
    CK(cudaMemcpyAsync(B.rows, B.h_rows, sizeof(BatchRows), cudaMemcpyHostToDevice, p->stream));
    CK(cudaEventRecord(p->ev0, p->stream));
    CK(cudaGraphLaunch(g->exec, p->stream));
    CK(cudaEventRecord(p->ev1, p->stream));
    if ((rc = step_outputs(p, n, rows, order, e, controls, RowBufs{B.logits, B.ids, B.smp_out, B.smp_indices, B.h_out}, ids_out, logits))) return rc;
    CK(cudaEventElapsedTime(&B.last_ms, p->ev0, p->ev1));
    B.last_launches = g->launches;
    return B200_OK;
}

// b200_forward_chunk over checked rows in the tensor_core_exact mode: the chunk laid out with the emitting rows first, as batch_step
// lays out its step, runs enqueue_chunk_i8 (K / V to the decode slots); its first e residual rows go through the batched step's
// classifier, read in place from pi8.X, and step_outputs does the rest.  b200_batch_info reports the call (CUDA events around the
// chunk and the classifier); b200_prefill_info is left alone.
int chunk_step(b200_plan *p, int n, const b200_step_row *rows, int32_t *ids_out, float *logits) {
    const b200_config &g = p->cfg;
    auto &B = p->bt;
    std::vector<int> order(n);
    const int e = emit_first(n, rows, order.data());
    const size_t slot_stride = (size_t)g.n_layers * g.context_length * p->kvd;
    std::vector<ChunkTok> tab(n);
    for (int k = 0; k < n; k++) {
        const b200_step_row &r = rows[order[k]];
        tab[k] = ChunkTok{r.token, r.position, (long long)(r.slot * slot_stride)};
    }
    int rc, nl = 0;
    CK(cudaMemcpyAsync(p->pi8.tok, tab.data(), (size_t)n * sizeof(ChunkTok), cudaMemcpyHostToDevice, p->stream));
    CK(cudaEventRecord(p->ev0, p->stream));
    if ((rc = enqueue_chunk_i8(p, n, false, &nl))) return rc;
    if (e) {
        if ((rc = enqueue_classifier(p, p->pi8.X, e))) return rc;
        nl += CLASSIFIER_LAUNCHES;
    }
    CK(cudaEventRecord(p->ev1, p->stream));
    if ((rc = step_outputs(p, n, rows, order.data(), e, true, RowBufs{B.logits, B.ids, B.smp_out, B.smp_indices, B.h_out}, ids_out, logits))) return rc;
    CK(cudaEventElapsedTime(&B.last_ms, p->ev0, p->ev1));
    B.last_launches = nl;
    return B200_OK;
}

// b200_forward_decode and b200_forward_decode_sample over a checked row r of slot -1: the single-token decode graph, then
// step_outputs on its one row in the plan's own buffers (h_ids as the readback block).
int decode_one(b200_plan *p, const b200_step_row &r, bool controls, int32_t *id, float *logits, int32_t *info) {
    CK(cudaSetDevice(p->device));
    int rc;
    if ((rc = set_state(p, r.token, r.position, 0, 0))) return rc;
    CK(cudaGraphLaunch(decode_graph(p), p->stream));
    const int order = 0;
    if ((rc = step_outputs(p, 1, &r, &order, 1, controls, RowBufs{p->logits, p->out_ids, p->smp_out, p->smp_indices, p->h_ids}, id, logits, info))) return rc;
    return check_device_error(p);
}

// ---- b200_score_tokens (score.cuh) ----------------------------------------------------------------------------------------------
// The per-row targets and results: rows for the longest call any mode takes.
int score_ready(b200_plan *p) {
    auto &S = p->sc;
    if (S.tgt) return B200_OK;
    const int cap = p->prefill_batch > p->seq_cap ? p->prefill_batch : p->seq_cap;
    int rc;
    if ((rc = dalloc(p, &S.tgt, (size_t)cap * 4)) || (rc = dalloc(p, &S.out, (size_t)cap * sizeof(ScoreOut)))) return rc;
    S.cap = cap;
    return B200_OK;
}

// tensor_core_exact: the logits scratch and the classifier's maps, built on the first score call.  A resident classifier is
// expanded into pi8.kq8, which then grows to its Q8_0 tiles if they are larger than every layer matrix's (the layer maps are
// rebuilt over the new scratch).  Both must fit the free memory (memory_free), or the call fails with B200_ERR_OOM.
int score_init_i8(b200_plan *p) {
    auto &S = p->sc;
    PrefillI8Ctx &c = p->pi8;
    if (S.logits) return B200_OK;
    const TileMat Q = q8_geometry(p->tout);
    if (Q.seg % pg::BK) return fail(p, B200_ERR_UNSUPPORTED, "the classifier's Q8_0 stream segments are not multiples of 64 columns: score in the exact prefill mode");
    const int ldl = (p->cfg.vocab_size + pg::I8_BN - 1) / pg::I8_BN * pg::I8_BN; // whole 64-column tiles
    const int64_t logit_bytes = (int64_t)SCORE_GROUP_ROWS * ldl * 4;
    const int64_t cls_bytes = p->tout.fmt ? tile_bytes(Q) : 0, grow = cls_bytes > c.kq8_bytes ? cls_bytes - c.kq8_bytes : 0;
    int64_t avail;
    int rc;
    if ((rc = memory_free(p, &avail))) return rc;
    if (logit_bytes + grow > avail)
        return fail(p, B200_ERR_OOM, "scoring in tensor_core_exact needs %lld bytes of logits scratch and %lld more bytes of Q8_0 scratch for the classifier, "
                    "%lld bytes are free", (long long)logit_bytes, (long long)grow, (long long)avail);
    if (grow) {
        if (c.kq8) {
            CK(cudaFree(c.kq8));
            for (size_t i = 0; i < p->allocs.size(); i++)
                if (p->allocs[i] == c.kq8) { p->allocs.erase(p->allocs.begin() + i); break; }
            p->bytes -= c.kq8_bytes;
            c.kq8 = nullptr;
            c.kq8_bytes = 0;
        }
        if ((rc = dalloc(p, &c.kq8, (size_t)cls_bytes))) return rc;
        c.kq8_bytes = cls_bytes;
        if (!i8_weight_maps(p)) return fail(p, B200_ERR_CUDA, "cuTensorMapEncodeTiled rejected a tensor map");
    }
    if (!i8_b_maps(p, &S.cls_q, &S.cls_s, p->tout)) return fail(p, B200_ERR_CUDA, "cuTensorMapEncodeTiled rejected the classifier's tensor map");
    if ((rc = dalloc(p, &S.logits, (size_t)logit_bytes))) return rc;
    S.ldl = ldl;
    return B200_OK;
}

// exact mode on a plan that runs multi-position steps: steps of batch_max_rows rows with the classifier on every row, each followed
// by k_score_rows over its logits rows.  The schedule is uploaded once (k_batch_rows_next feeds each step its rows).
int score_multi(b200_plan *p, const int32_t *tokens, int n, int start_pos) {
    int rc;
    if ((rc = multi_ready(p))) return rc;
    std::vector<BatchRows> sched;
    std::vector<int> nrows;
    pack_rows(sched, nrows, batch_max_rows(p), tokens, start_pos, n, 0);
    return run_steps(p, sched, nrows, true, nullptr, [&](int s, int r0) {
        k_score_rows<<<nrows[s], SCORE_THREADS, 0, p->stream>>>(p->bt.logits, sampler_padded(p->cfg.vocab_size), p->cfg.vocab_size, p->sc.tgt + r0, p->sc.out + r0);
        CK(cudaGetLastError());
        return B200_OK;
    });
}

// exact mode on every other single-GPU plan: the single-token decode graph per position (it computes p->logits), each followed by
// k_score_rows over that row.  The step state walks seq_tokens as b200_decode_sequence's does.
int score_single(b200_plan *p, const int32_t *tokens, int n, int start_pos) {
    int rc;
    memcpy(p->h_ids, tokens, (size_t)n * 4);
    CK(cudaMemcpyAsync(p->seq_tokens, p->h_ids, (size_t)n * 4, cudaMemcpyHostToDevice, p->stream));
    if ((rc = set_state(p, tokens[0], start_pos, n, 0))) return rc;
    for (int i = 0; i < n; i++) {
        CK(cudaGraphLaunch(decode_graph(p), p->stream));
        k_score_rows<<<1, SCORE_THREADS, 0, p->stream>>>(p->logits, 0, p->cfg.vocab_size, p->sc.tgt + i, p->sc.out + i);
        CK(cudaGetLastError());
    }
    return B200_OK;
}

// Device memory and the result code of an entry point without a plan.  ok() keeps the first failure (an allocation failure is
// B200_ERR_OOM, any other B200_ERR_CUDA) and answers whether everything so far succeeded; the allocations are freed at scope exit.
struct Scratch {
    int rc = B200_OK;
    std::vector<void *> mem;
    bool ok(cudaError_t e) {
        if (e != cudaSuccess && rc == B200_OK) rc = e == cudaErrorMemoryAllocation ? B200_ERR_OOM : B200_ERR_CUDA;
        return rc == B200_OK;
    }
    template <typename T> bool alloc(T **ptr, size_t bytes) {
        void *d = nullptr;
        const cudaError_t e = cudaMalloc(&d, bytes);
        if (e == cudaSuccess) mem.push_back(d);
        *ptr = reinterpret_cast<T *>(d);
        return ok(e);
    }
    ~Scratch() {
        for (void *d : mem) cudaFree(d);
    }
};

// f(std::integral_constant<int, MODE>()) for a checked run-time pg::GEMM_* mode.
template <typename F> int with_gemm_mode(int mode, F &&f) {
    if (mode == pg::GEMM_F32) return f(std::integral_constant<int, pg::GEMM_F32>());
    if (mode == pg::GEMM_RESID) return f(std::integral_constant<int, pg::GEMM_RESID>());
    return f(std::integral_constant<int, pg::GEMM_GATEUP>());
}

} // namespace

// b200_plan_create, b200_plan_create_moe, b200_plan_create_granite and b200_plan_create_devstral (moe / granite == nullptr: neither;
// devstral: called by b200_plan_create_devstral, whose yarn may be nullptr)
static int plan_create(const b200_config *cfg, const b200_moe_config *moe, const b200_granite_config *granite, bool devstral,
                       const b200_yarn_config *yarn, const b200_tensor *tensors, int32_t n_tensors, int32_t prefill_batch_size, int32_t device,
                       b200_plan **out, char *err, size_t err_len) {
    if (out) *out = nullptr;
    if (!cfg || !tensors || !out || n_tensors <= 0) {
        if (err && err_len) snprintf(err, err_len, "null argument");
        return B200_ERR_BAD_ARG;
    }
    if ((cfg->arch == B200_ARCH_QWEN2_MOE || cfg->arch == B200_ARCH_QWEN3_MOE) != (moe != nullptr)) {
        if (err && err_len)
            snprintf(err, err_len, moe ? "b200_plan_create_moe needs arch B200_ARCH_QWEN2_MOE or B200_ARCH_QWEN3_MOE (got %d)"
                     : cfg->arch == B200_ARCH_QWEN2_MOE ? "arch %d (B200_ARCH_QWEN2_MOE) needs its expert configuration: create the plan with b200_plan_create_moe"
                                                        : "arch %d (B200_ARCH_QWEN3_MOE) needs its expert configuration: create the plan with b200_plan_create_moe",
                     cfg->arch);
        return B200_ERR_BAD_ARG;
    }
    if ((cfg->arch == B200_ARCH_GRANITE) != (granite != nullptr)) {
        if (err && err_len)
            snprintf(err, err_len, granite ? "b200_plan_create_granite needs arch B200_ARCH_GRANITE (got %d)"
                                           : "arch %d (B200_ARCH_GRANITE) needs its scales: create the plan with b200_plan_create_granite", cfg->arch);
        return B200_ERR_BAD_ARG;
    }
    if (granite) {
        const float v[4] = {granite->embedding_scale, granite->residual_scale, granite->attention_scale, granite->logit_scale};
        const char *names[4] = {"embedding_scale", "residual_scale", "attention_scale", "logit_scale"};
        for (int i = 0; i < 4; i++)
            if (!isfinite(v[i])) {
                if (err && err_len) snprintf(err, err_len, "Granite %s is not finite (%g)", names[i], (double)v[i]);
                return B200_ERR_BAD_ARG;
            }
    }
    if ((cfg->arch == B200_ARCH_DEVSTRAL) != devstral) {
        if (err && err_len)
            snprintf(err, err_len, devstral ? "b200_plan_create_devstral needs arch B200_ARCH_DEVSTRAL (got %d)"
                                            : "arch %d (B200_ARCH_DEVSTRAL) needs its RoPE parameters: create the plan with b200_plan_create_devstral", cfg->arch);
        return B200_ERR_BAD_ARG;
    }
    if (yarn) {
        const float v[4] = {yarn->factor, yarn->beta_fast, yarn->beta_slow, yarn->log_multiplier};
        const char *names[4] = {"factor", "beta_fast", "beta_slow", "log_multiplier"};
        for (int i = 0; i < 4; i++)
            if (!isfinite(v[i])) {
                if (err && err_len) snprintf(err, err_len, "YaRN %s is not finite (%g)", names[i], (double)v[i]);
                return B200_ERR_BAD_ARG;
            }
        if (!(yarn->factor > 0.0f) || yarn->original_context_length <= 0) {
            if (err && err_len)
                snprintf(err, err_len, "YaRN %s must be > 0 (factor %g, original_context_length %d)", yarn->factor > 0.0f ? "original_context_length" : "factor",
                         (double)yarn->factor, yarn->original_context_length);
            return B200_ERR_BAD_ARG;
        }
    }
    b200_plan *p = new b200_plan();
    p->cfg = *cfg;
    if (moe) {
        p->is_moe = true;
        p->moe = *moe;
        p->moe_shared = cfg->arch == B200_ARCH_QWEN2_MOE;
        p->moe_nw = moe->n_experts_used + (p->moe_shared ? 1 : 0);
        p->moe_name = p->moe_shared ? "Qwen2-MoE" : "Qwen3-MoE";
    }
    if (granite) p->mup = *granite;
    if (yarn) { p->has_yarn = true; p->yarn = *yarn; }
    if (p->cfg.tp_size <= 0) p->cfg.tp_size = 1;
    p->device = device;
    p->prefill_batch = prefill_batch_size;
    int rc = build(p, tensors, n_tensors);
    if (rc != B200_OK) {
        if (err && err_len) snprintf(err, err_len, "%s", p->err.c_str());
        b200_plan_free(p);
        return rc;
    }
    *out = p;
    return B200_OK;
}

template <int T>
cudaError_t launch_profile_seqsum2(const float *d, int n, long long *cyc, float *o) {
    const size_t smem = (size_t)T * seqsum2_stride((n + T - 1) / T) * 4 + seqsum2_scratch_bytes(T);
    cudaError_t e = cudaFuncSetAttribute(k_profile_seqsum2<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) k_profile_seqsum2<T><<<1, T, smem>>>(d, n, cyc, o);
    return e;
}

extern "C" {

int b200_plan_create(const b200_config *cfg, const b200_tensor *tensors, int32_t n_tensors, int32_t prefill_batch_size,
                     int32_t device, b200_plan **out, char *err, size_t err_len) {
    return plan_create(cfg, nullptr, nullptr, false, nullptr, tensors, n_tensors, prefill_batch_size, device, out, err, err_len);
}

int b200_plan_create_moe(const b200_config *cfg, const b200_moe_config *moe, const b200_tensor *tensors, int32_t n_tensors, int32_t prefill_batch_size,
                         int32_t device, b200_plan **out, char *err, size_t err_len) {
    if (!moe) {
        if (out) *out = nullptr;
        if (err && err_len) snprintf(err, err_len, "null argument");
        return B200_ERR_BAD_ARG;
    }
    return plan_create(cfg, moe, nullptr, false, nullptr, tensors, n_tensors, prefill_batch_size, device, out, err, err_len);
}

int b200_plan_create_granite(const b200_config *cfg, const b200_granite_config *granite, const b200_tensor *tensors, int32_t n_tensors,
                             int32_t prefill_batch_size, int32_t device, b200_plan **out, char *err, size_t err_len) {
    if (!granite) {
        if (out) *out = nullptr;
        if (err && err_len) snprintf(err, err_len, "null argument");
        return B200_ERR_BAD_ARG;
    }
    return plan_create(cfg, nullptr, granite, false, nullptr, tensors, n_tensors, prefill_batch_size, device, out, err, err_len);
}

int b200_plan_create_devstral(const b200_config *cfg, const b200_yarn_config *yarn, const b200_tensor *tensors, int32_t n_tensors,
                              int32_t prefill_batch_size, int32_t device, b200_plan **out, char *err, size_t err_len) {
    return plan_create(cfg, nullptr, nullptr, true, yarn, tensors, n_tensors, prefill_batch_size, device, out, err, err_len);
}

int b200_forward_decode(b200_plan *p, int32_t token, int32_t position, float *logits, int32_t *argmax) {
    if (!p) return B200_ERR_BAD_ARG;
    if (!p->graph.decode.exec) return fail(p, B200_ERR_STATE, "tensor-parallel plan: call b200_tp_attach on every rank first");
    if (logits && p->tp.n > 1) return fail(p, B200_ERR_UNSUPPORTED, "full logits are not gathered under tensor parallelism (argmax is)");
    int rc, id;
    if ((rc = check_pos(p, token, position))) return rc;
    if ((rc = decode_one(p, b200_step_row{-1, token, position, 1, 0.0f, 0.0f, 0.0f}, false, &id, logits, nullptr))) return rc; // sequence 0's controls stay unused
    if (argmax) *argmax = id;
    return B200_OK;
}

int b200_forward_decode_sample(b200_plan *p, int32_t token, int32_t position, float temperature, float topp, float uniform01, int32_t *token_out, int32_t *info) {
    if (!p || !token_out) return B200_ERR_BAD_ARG;
    if (!p->graph.decode.exec) return fail(p, B200_ERR_STATE, "tensor-parallel plan: call b200_tp_attach on every rank first");
    if (p->tp.n > 1) return fail(p, B200_ERR_UNSUPPORTED, "the device-side temperature/top-p sampler needs the whole logits row on one GPU (tensor-parallel plans sample greedily)");
    if (!(temperature >= 0.0f) || !(uniform01 >= 0.0f && uniform01 < 1.0f)) return fail(p, B200_ERR_BAD_ARG, "temperature must be >= 0 and the uniform number in [0, 1)");
    int rc, id;
    if ((rc = check_pos(p, token, position))) return rc;
    if ((rc = decode_one(p, b200_step_row{-1, token, position, 1, temperature, topp, uniform01}, true, &id, nullptr, info))) return rc;
    *token_out = id;
    return B200_OK;
}

int b200_forward_prefill(b200_plan *p, int32_t token, int32_t position) {
    if (!p) return B200_ERR_BAD_ARG;
    if (!p->graph.prefill.exec) return fail(p, B200_ERR_STATE, "tensor-parallel plan: call b200_tp_attach on every rank first");
    int rc;
    if ((rc = check_pos(p, token, position))) return rc;
    CK(cudaSetDevice(p->device));
    if ((rc = set_state(p, token, position, 0, 0))) return rc;
    CK(cudaGraphLaunch(prefill_graph(p), p->stream));
    CK(cudaStreamSynchronize(p->stream));
    return check_device_error(p);
}

int b200_forward_batch_prefill(b200_plan *p, const int32_t *tokens, int32_t n, int32_t start_pos) {
    if (!p || !tokens) return B200_ERR_BAD_ARG;
    if (n <= 0) return B200_OK;
    if (!p->graph.prefill.exec) return fail(p, B200_ERR_STATE, "tensor-parallel plan: call b200_tp_attach on every rank first");
    int rc;
    if ((rc = check_chunk(p, tokens, n, start_pos))) return rc;
    CK(cudaSetDevice(p->device));
    if (chunk_path(p) != CHUNK_NONE) { // the whole chunk on the tensor cores into the plan's cache
        const int slot = 0;
        return prefill_chunk(p, 1, &slot, &start_pos, &n, tokens, true);
    }
    // Exact path (bit-identical KV cache to the CPU batchForwardJavaPrefill, InferenceCoreBatchPrefillDecode.java:62-168).  Plans
    // that run multi-position steps take positions start .. start + n - 2 in steps of batch_max_rows rows into the plan's cache;
    // the last token, and every token elsewhere, runs through the single-token prefill graph, with the step state as the
    // token-by-token loop leaves it before its last step.
    memcpy(p->h_ids, tokens, (size_t)n * 4);
    CK(cudaMemcpyAsync(p->seq_tokens, p->h_ids, (size_t)n * 4, cudaMemcpyHostToDevice, p->stream));
    int first = 0;
    if (n > 1 && !multi_why(p)) {
        if ((rc = multi_ready(p))) return rc;
        std::vector<BatchRows> sched;
        std::vector<int> nrows;
        pack_rows(sched, nrows, batch_max_rows(p), tokens, start_pos, n - 1, 0);
        if ((rc = run_steps(p, sched, nrows, true, nullptr))) return rc;
        first = n - 1;
    }
    if ((rc = set_state(p, tokens[first], start_pos + first, n, 0, first))) return rc;
    for (int i = first; i < n; i++) CK(cudaGraphLaunch(prefill_graph(p), p->stream));
    CK(cudaStreamSynchronize(p->stream));
    return check_device_error(p);
}

int b200_score_tokens(b200_plan *p, const int32_t *tokens, const int32_t *targets, int32_t n, int32_t start_pos, double *logprobs, int32_t *greedy_ids) {
    if (!p || !tokens || !targets || !logprobs || !greedy_ids) return B200_ERR_BAD_ARG;
    if (n <= 0) return B200_OK;
    if (p->cfg.tp_size > 1)
        return fail(p, B200_ERR_UNSUPPORTED, "full logits are not gathered under tensor parallelism: scoring runs on single-GPU plans");
    const ChunkPath path = chunk_path(p);
    if (path == CHUNK_TC)
        return fail(p, B200_ERR_UNSUPPORTED, "the %s prefill keeps f16 activations, so its logits are not the reference's: score in the exact, "
                    "tensor_core_exact or tensor_core_exact_moe prefill mode", PREFILL_MODE_NAMES[p->pf_mode]);
    int rc;
    if ((rc = check_chunk(p, tokens, n, start_pos))) return rc;
    for (int i = 0; i < n; i++)
        if (targets[i] != -1 && (targets[i] < 0 || targets[i] >= p->cfg.vocab_size))
            return fail(p, B200_ERR_BAD_ARG, "target %d of row %d out of range (-1 or a token id)", targets[i], i);
    const bool tc = path == CHUNK_I8;
    CK(cudaSetDevice(p->device));
    if ((rc = score_ready(p)) || (tc && (rc = score_init_i8(p)))) return rc;
    CK(cudaMemcpyAsync(p->sc.tgt, targets, (size_t)n * 4, cudaMemcpyHostToDevice, p->stream));
    if (tc) {
        const int slot = 0;
        rc = prefill_chunk(p, 1, &slot, &start_pos, &n, tokens, true, true);
    } else rc = multi_why(p) ? score_single(p, tokens, n, start_pos) : score_multi(p, tokens, n, start_pos);
    if (rc) return rc;
    std::vector<ScoreOut> out(n);
    CK(cudaMemcpyAsync(out.data(), p->sc.out, (size_t)n * sizeof(ScoreOut), cudaMemcpyDeviceToHost, p->stream));
    CK(cudaStreamSynchronize(p->stream));
    if ((rc = check_device_error(p))) return rc;
    for (int i = 0; i < n; i++) { logprobs[i] = out[i].logprob; greedy_ids[i] = out[i].greedy; }
    return B200_OK;
}

int b200_decode_sequence(b200_plan *p, const int32_t *tokens, int32_t n, int32_t start_pos, int32_t feedback,
                         int32_t *out_ids, float *device_ms) {
    if (!p || !tokens) return B200_ERR_BAD_ARG;
    if (n <= 0) return B200_OK;
    if (!p->graph.decode.exec) return fail(p, B200_ERR_STATE, "tensor-parallel plan: call b200_tp_attach on every rank first");
    if (n > p->seq_cap) return fail(p, B200_ERR_BAD_ARG, "sequence of %d steps exceeds capacity %d", n, p->seq_cap);
    if (start_pos < 0 || start_pos + n > p->cfg.context_length) return fail(p, B200_ERR_BAD_ARG, "positions %d..%d outside the KV cache (%d)", start_pos, start_pos + n - 1, p->cfg.context_length);
    int nt = feedback ? 1 : n;
    if (const int i = bad_token(p, tokens, nt); i >= 0) return fail(p, B200_ERR_BAD_ARG, "token %d out of range", tokens[i]);
    CK(cudaSetDevice(p->device));
    memcpy(p->h_ids, tokens, (size_t)nt * 4);
    CK(cudaMemcpyAsync(p->seq_tokens, p->h_ids, (size_t)nt * 4, cudaMemcpyHostToDevice, p->stream));
    int rc;
    if ((rc = set_state(p, tokens[0], start_pos, nt, feedback))) return rc;
    const bool lp = p->lp.top_n >= 0;
    CK(cudaEventRecord(p->ev0, p->stream));
    for (int i = 0; i < n; i++) {
        CK(cudaGraphLaunch(decode_graph(p), p->stream));
        if (lp && (rc = launch_logprobs_one(p, p->out_ids + i, i))) return rc; // before the next step overwrites p->logits
    }
    CK(cudaEventRecord(p->ev1, p->stream));
    if (lp && (rc = copy_logprobs(p, n))) return rc;
    if (out_ids) CK(cudaMemcpyAsync(p->h_ids, p->out_ids, (size_t)n * 4, cudaMemcpyDeviceToHost, p->stream));
    CK(cudaStreamSynchronize(p->stream));
    if ((rc = check_device_error(p))) return rc;
    if (lp) p->lp.rows = n;
    if (out_ids) memcpy(out_ids, p->h_ids, (size_t)n * 4);
    if (device_ms) CK(cudaEventElapsedTime(device_ms, p->ev0, p->ev1));
    return B200_OK;
}

int b200_set_decode_mode(b200_plan *p, int32_t mode) {
    if (!p || (mode != B200_DECODE_GRAPH && mode != B200_DECODE_PERSISTENT)) return B200_ERR_BAD_ARG;
    if (!p->graph.decode.exec) return fail(p, B200_ERR_STATE, "tensor-parallel plan: call b200_tp_attach on every rank first");
    if (mode == B200_DECODE_PERSISTENT && !p->pd_ok) return fail(p, B200_ERR_UNSUPPORTED, "%s", p->pd_why.c_str());
    p->decode_mode = mode;
    return B200_OK;
}

int b200_decode_info(b200_plan *p, int32_t *mode, int32_t *launches, int32_t *ring_stages, int32_t *smem_bytes) {
    if (!p) return B200_ERR_BAD_ARG;
    const TokenGraphs &t = active_graphs(p);
    if (mode) *mode = &t == &p->pers ? B200_DECODE_PERSISTENT : B200_DECODE_GRAPH;
    if (launches) *launches = t.decode.launches;
    if (ring_stages) *ring_stages = p->pd_ok ? p->pd_L.stages : 0;
    if (smem_bytes) *smem_bytes = p->pd_ok ? (int32_t)p->pd_L.total : 0;
    return B200_OK;
}

int b200_trace_persistent(b200_plan *p, int32_t token, int32_t position, uint64_t *stamps, int64_t cap, int32_t *n_ctas, int32_t *n_rows, int32_t *n_stamps) {
    if (!p || !stamps) return B200_ERR_BAD_ARG;
    if (!p->pers.trace.exec) return fail(p, B200_ERR_UNSUPPORTED, "%s", p->pd_ok ? "no traced persistent graph" : p->pd_why.c_str());
    int rc;
    if ((rc = check_pos(p, token, position))) return rc;
    CK(cudaSetDevice(p->device));
    const size_t words = (size_t)p->n_sms * (p->cfg.n_layers + 1) * PD_STAMPS;
    if ((size_t)cap < words) return fail(p, B200_ERR_BAD_ARG, "stamp buffer too small: need %zu uint64", words);
    CK(cudaMemsetAsync(p->pd_trace, 0, words * 8, p->stream));
    if ((rc = set_state(p, token, position, 0, 0))) return rc;
    CK(cudaGraphLaunch(p->pers.trace.exec, p->stream));
    CK(cudaStreamSynchronize(p->stream));
    if ((rc = check_device_error(p))) return rc;
    CK(cudaMemcpy(stamps, p->pd_trace, words * 8, cudaMemcpyDeviceToHost));
    if (n_ctas) *n_ctas = p->n_sms;
    if (n_rows) *n_rows = p->cfg.n_layers + 1;
    if (n_stamps) *n_stamps = PD_STAMPS;
    return B200_OK;
}

int b200_set_prefill_mode(b200_plan *p, int32_t mode) {
    if (!p || mode < B200_PREFILL_EXACT || mode > B200_PREFILL_TENSOR_CORE_EXACT_MOE) return B200_ERR_BAD_ARG;
    const b200_plan::PrefillMode &m = p->pf[mode];
    if (!m.ready) { // refused before anything is allocated, else built (each init leaves the mode ready or says why not)
        if (const char *why = prefill_why(p, mode)) return fail(p, B200_ERR_UNSUPPORTED, "%s", why);
        CK(cudaSetDevice(p->device));
        const int rc = mode == B200_PREFILL_TENSOR_CORE ? prefill_init(p) : mode == B200_PREFILL_TENSOR_CORE_W8A16 ? prefill_init_q8(p) : prefill_init_i8(p);
        if (rc) return rc;
        if (!m.ready) return fail(p, B200_ERR_UNSUPPORTED, "%s", m.why);
    }
    p->pf_mode = mode;
    return B200_OK;
}

int b200_prefill_info(b200_plan *p, int32_t *mode, int32_t *launches, float *device_ms) {
    if (!p) return B200_ERR_BAD_ARG;
    if (mode) *mode = p->pf_mode;
    if (launches) *launches = p->launches_prefill;
    if (device_ms) *device_ms = p->prefill_ms;
    return B200_OK;
}

int b200_kv_reset(b200_plan *p) {
    if (!p) return B200_ERR_BAD_ARG;
    CK(cudaSetDevice(p->device));
    size_t kv_bytes = (size_t)p->cfg.n_layers * p->cfg.context_length * p->kvd_l * 4;
    CK(cudaMemsetAsync(p->key_cache, 0, kv_bytes, p->stream));
    CK(cudaMemsetAsync(p->value_cache, 0, kv_bytes, p->stream));
    int rc;
    if ((rc = clear_counts(p, 0, 1))) return rc;
    CK(cudaStreamSynchronize(p->stream));
    return B200_OK;
}

int b200_set_decode_slots(b200_plan *p, int32_t n_slots) {
    if (!p) return B200_ERR_BAD_ARG;
    if (n_slots < 0) return fail(p, B200_ERR_BAD_ARG, "n_slots must be >= 0");
    CK(cudaSetDevice(p->device));
    CK(cudaStreamSynchronize(p->stream));
    if (n_slots == 0) { batch_free(p); return clear_counts(p, 1, SMB_MAX_ROWS + 1); } // the memset orders before any later call's work
    if (p->is_moe) return fail(p, B200_ERR_UNSUPPORTED, "batched decode has no %s layer (MoE plans decode one sequence per step)", p->moe_name);
    if (p->cfg.tp_size > 1) return fail(p, B200_ERR_UNSUPPORTED, "batched decode runs on single-GPU plans only (this plan is tensor-parallel)");
    if (p->wtype != B200_GGML_Q8_0) return fail(p, B200_ERR_UNSUPPORTED, "batched decode needs Q8_0 weights (FP16 plans decode one sequence per step)");
    if (p->resident) return fail(p, B200_ERR_UNSUPPORTED, "%s", RESIDENT_MULTI_WHY);
    const int mx = batch_max_rows(p);
    if (n_slots > mx) return fail(p, B200_ERR_UNSUPPORTED, "at most %d decode slots on this plan (asked for %d)", mx, n_slots);
    batch_free(p);
    const int rc = batch_alloc(p, n_slots);
    if (rc) { batch_free(p); return rc; }
    return clear_counts(p, 1, SMB_MAX_ROWS + 1);
}

int b200_forward_decode_batch(b200_plan *p, int32_t n, const int32_t *slots, const int32_t *tokens, const int32_t *positions, const float *sampling,
                              int32_t *ids_out, float *logits) {
    if (!p) return B200_ERR_BAD_ARG;
    auto &B = p->bt;
    if (!B.n_slots) return fail(p, B200_ERR_STATE, "no decode slots: call b200_set_decode_slots first");
    if (!slots || !tokens || !positions || !ids_out) return fail(p, B200_ERR_BAD_ARG, "slots, tokens, positions and ids_out must not be NULL");
    if (n < 1 || n > B.n_slots) return fail(p, B200_ERR_BAD_ARG, "n = %d rows: need 1 <= n <= %d (the plan's decode slots)", n, B.n_slots);
    b200_step_row r[SMB_MAX_ROWS];
    int rc;
    for (int i = 0; i < n; i++) {
        for (int j = 0; j < i; j++)
            if (slots[j] == slots[i]) return fail(p, B200_ERR_BAD_ARG, "row %d: slot %d repeats row %d's", i, slots[i], j);
        const float *s = sampling ? sampling + 3 * i : nullptr;
        r[i] = b200_step_row{slots[i], tokens[i], positions[i], 1, s ? s[0] : 0.0f, s ? s[1] : 0.0f, s ? s[2] : 0.0f};
        if ((rc = check_row(p, i, r[i]))) return rc;
    }
    CK(cudaSetDevice(p->device));
    return batch_step(p, n, r, false, sampling != nullptr, ids_out, logits);
}

int b200_slot_reset(b200_plan *p, int32_t slot) {
    if (!p) return B200_ERR_BAD_ARG;
    if (slot < 0 || slot >= p->bt.n_slots) return fail(p, B200_ERR_BAD_ARG, "slot %d out of range (%d slots)", slot, p->bt.n_slots);
    CK(cudaSetDevice(p->device));
    const size_t kv = (size_t)p->cfg.n_layers * p->cfg.context_length * p->kvd;
    CK(cudaMemsetAsync(p->bt.slot_k + (size_t)slot * kv, 0, kv * 4, p->stream));
    CK(cudaMemsetAsync(p->bt.slot_v + (size_t)slot * kv, 0, kv * 4, p->stream));
    int rc;
    if ((rc = clear_counts(p, slot + 1, slot + 2))) return rc;
    CK(cudaStreamSynchronize(p->stream));
    return B200_OK;
}

int b200_slot_copy_kv(b200_plan *p, int32_t slot, int32_t n_positions) {
    if (!p) return B200_ERR_BAD_ARG;
    const b200_config &c = p->cfg;
    if (slot < 0 || slot >= p->bt.n_slots) return fail(p, B200_ERR_BAD_ARG, "slot %d out of range (%d slots)", slot, p->bt.n_slots);
    if (n_positions < 0 || n_positions > c.context_length) return fail(p, B200_ERR_BAD_ARG, "n_positions %d outside [0, %d]", n_positions, c.context_length);
    CK(cudaSetDevice(p->device));
    const size_t ctx_kv = (size_t)c.context_length * p->kvd, head = (size_t)n_positions * p->kvd;
    for (int l = 0; l < c.n_layers; l++) {
        const size_t o = ((size_t)slot * c.n_layers + l) * ctx_kv;
        float *dk = p->bt.slot_k + o, *dv = p->bt.slot_v + o;
        if (head) {
            CK(cudaMemcpyAsync(dk, p->key_cache + (size_t)l * ctx_kv, head * 4, cudaMemcpyDeviceToDevice, p->stream));
            CK(cudaMemcpyAsync(dv, p->value_cache + (size_t)l * ctx_kv, head * 4, cudaMemcpyDeviceToDevice, p->stream));
        }
        if (head < ctx_kv) { // beyond the prefix the slot must read like a fresh State (the Qwen3 / Qwen2 loop reads a skipped, zero position)
            CK(cudaMemsetAsync(dk + head, 0, (ctx_kv - head) * 4, p->stream));
            CK(cudaMemsetAsync(dv + head, 0, (ctx_kv - head) * 4, p->stream));
        }
    }
    CK(cudaStreamSynchronize(p->stream));
    return B200_OK;
}

namespace {
// Exact b200_prefill_slots: the batched step without the classifier.  The call's tokens, sequence after sequence, are cut into
// steps of batch_max_rows rows, so a sequence contributes several consecutive positions to a step when rows are free and T tokens
// take ceil(T / rows) steps.  Steps in which a slot repeats run the split attention form (k_rope_kv_batch, then
// k_attention_cached_rows); the others the plain batched step.
int prefill_slots_exact(b200_plan *p, int ns, const int *slots, const int *start, const int *len, const int *off, const int *tokens) {
    std::vector<BatchRows> sched;
    std::vector<int> nrows;
    const int rows = batch_max_rows(p);
    for (int i = 0; i < ns; i++) pack_rows(sched, nrows, rows, tokens + off[i], start[i], len[i], slots[i]);
    int rc, launches = 0;
    if ((rc = run_steps(p, sched, nrows, false, &launches))) return rc;
    CK(cudaStreamSynchronize(p->stream));
    CK(cudaEventElapsedTime(&p->prefill_ms, p->ev0, p->ev1));
    p->launches_prefill = launches;
    return B200_OK;
}
} // namespace

int b200_prefill_slots(b200_plan *p, int32_t n_seqs, const int32_t *slots, const int32_t *start_positions, const int32_t *lengths, const int32_t *tokens) {
    if (!p) return B200_ERR_BAD_ARG;
    auto &B = p->bt;
    const b200_config &c = p->cfg;
    if (!B.n_slots) return fail(p, B200_ERR_STATE, "no decode slots: call b200_set_decode_slots first");
    if (!slots || !start_positions || !lengths) return fail(p, B200_ERR_BAD_ARG, "slots, start_positions and lengths must not be NULL");
    if (n_seqs < 1 || n_seqs > B.n_slots) return fail(p, B200_ERR_BAD_ARG, "n_seqs = %d: need 1 <= n_seqs <= %d (the plan's decode slots)", n_seqs, B.n_slots);
    std::vector<int> off(n_seqs);
    int64_t total = 0;
    for (int i = 0; i < n_seqs; i++) {
        if (slots[i] < 0 || slots[i] >= B.n_slots) return fail(p, B200_ERR_BAD_ARG, "sequence %d: slot %d out of range (%d slots)", i, slots[i], B.n_slots);
        for (int j = 0; j < i; j++)
            if (slots[j] == slots[i]) return fail(p, B200_ERR_BAD_ARG, "sequence %d: slot %d repeats sequence %d's", i, slots[i], j);
        if (lengths[i] < 0) return fail(p, B200_ERR_BAD_ARG, "sequence %d: length %d is negative", i, lengths[i]);
        if (start_positions[i] < 0 || (int64_t)start_positions[i] + lengths[i] > c.context_length)
            return fail(p, B200_ERR_BAD_ARG, "sequence %d: positions %d..%lld outside the KV cache (%d)", i, start_positions[i],
                        (long long)start_positions[i] + lengths[i] - 1, c.context_length);
        off[i] = (int)total;
        total += lengths[i];
    }
    if (total && !tokens) return fail(p, B200_ERR_BAD_ARG, "tokens must not be NULL");
    for (int i = 0; i < n_seqs; i++)
        if (const int j = bad_token(p, tokens + off[i], lengths[i]); j >= 0)
            return fail(p, B200_ERR_BAD_ARG, "sequence %d: token %d (index %d) out of range", i, tokens[off[i] + j], j);
    const bool tc = chunk_path(p) != CHUNK_NONE;
    if (tc && total > p->prefill_batch) {
        int i = 0;
        while (off[i] + lengths[i] <= p->prefill_batch) i++;
        return fail(p, B200_ERR_BAD_ARG, "sequence %d: the call's %lld tokens exceed prefill_batch_size %d (split the prompts into chunks)", i, (long long)total,
                    p->prefill_batch);
    }
    if (!total) return B200_OK;
    CK(cudaSetDevice(p->device));
    return tc ? prefill_chunk(p, n_seqs, slots, start_positions, lengths, tokens, false)
              : prefill_slots_exact(p, n_seqs, slots, start_positions, lengths, off.data(), tokens);
}

int b200_decode_multi_rows(b200_plan *p, int32_t *max_rows) {
    if (!p || !max_rows) return B200_ERR_BAD_ARG;
    *max_rows = multi_why(p) ? 0 : batch_max_rows(p);
    return B200_OK;
}

int b200_forward_decode_multi(b200_plan *p, int32_t slot, int32_t n, const int32_t *tokens, int32_t start_pos, int32_t *ids_out, float *logits) {
    if (!p) return B200_ERR_BAD_ARG;
    if (const char *why = multi_why(p)) return fail(p, B200_ERR_UNSUPPORTED, "%s", why);
    auto &B = p->bt;
    const b200_config &c = p->cfg;
    const int R = batch_max_rows(p);
    if (!tokens || !ids_out) return fail(p, B200_ERR_BAD_ARG, "tokens and ids_out must not be NULL");
    if (n < 1 || n > R) return fail(p, B200_ERR_BAD_ARG, "n = %d rows: need 1 <= n <= %d (b200_decode_multi_rows)", n, R);
    if (slot < -1 || slot >= B.n_slots) return fail(p, B200_ERR_BAD_ARG, "slot %d out of range (%d slots; -1 is the plan's own cache)", slot, B.n_slots);
    if (const int i = bad_token(p, tokens, n); i >= 0) return fail(p, B200_ERR_BAD_ARG, "row %d: token %d out of range", i, tokens[i]);
    b200_step_row r[SMB_MAX_ROWS];
    for (int i = 0; i < n; i++) {
        if (start_pos < 0 || (int64_t)start_pos + i >= c.context_length)
            return fail(p, B200_ERR_BAD_ARG, "row %d: position %lld outside the KV cache (%d)", i, (long long)start_pos + i, c.context_length);
        r[i] = b200_step_row{slot < 0 ? 0 : slot, tokens[i], start_pos + i, 1, 0.0f, 0.0f, 0.0f};
    }
    CK(cudaSetDevice(p->device));
    int rc;
    if ((rc = multi_ready(p))) return rc;
    return batch_step(p, n, r, slot < 0, false, ids_out, logits);
}

int b200_forward_step(b200_plan *p, int32_t n, const b200_step_row *rows, int32_t *ids_out, float *logits) {
    if (!p) return B200_ERR_BAD_ARG;
    if (const char *why = multi_why(p)) return fail(p, B200_ERR_UNSUPPORTED, "%s", why);
    auto &B = p->bt;
    if (!B.n_slots) return fail(p, B200_ERR_STATE, "no decode slots: call b200_set_decode_slots first");
    if (!rows || !ids_out) return fail(p, B200_ERR_BAD_ARG, "rows and ids_out must not be NULL");
    const int R = batch_max_rows(p);
    if (n < 1 || n > R) return fail(p, B200_ERR_BAD_ARG, "n = %d rows: need 1 <= n <= %d (b200_decode_multi_rows)", n, R);
    int rc;
    if ((rc = check_step_rows(p, n, rows, R))) return rc;
    CK(cudaSetDevice(p->device));
    return batch_step(p, n, rows, false, true, ids_out, logits);
}

namespace {
// Why a plan can never run b200_forward_chunk (nullptr: it can, in tensor_core_exact with decode slots): what rules out batched
// steps, then what rules out the bit-exact tensor-core prefill.
const char *chunk_why(const b200_plan *p) {
    const char *why = multi_why(p);
    return why ? why : prefill_why(p, B200_PREFILL_TENSOR_CORE_EXACT);
}
} // namespace

int b200_chunk_rows(b200_plan *p, int32_t *max_rows) {
    if (!p || !max_rows) return B200_ERR_BAD_ARG;
    *max_rows = !chunk_why(p) && p->bt.n_slots && chunk_path(p) == CHUNK_I8 ? p->prefill_batch : 0;
    return B200_OK;
}

int b200_forward_chunk(b200_plan *p, int32_t n, const b200_step_row *rows, int32_t *ids_out, float *logits) {
    if (!p) return B200_ERR_BAD_ARG;
    if (const char *why = chunk_why(p)) return fail(p, B200_ERR_UNSUPPORTED, "%s", why);
    auto &B = p->bt;
    if (!B.n_slots) return fail(p, B200_ERR_STATE, "no decode slots: call b200_set_decode_slots first");
    if (const int mode = p->pf_mode; mode != B200_PREFILL_TENSOR_CORE_EXACT)
        return fail(p, B200_ERR_STATE, "the plan's prefill mode is %s%s: b200_forward_chunk runs in tensor_core_exact (b200_set_prefill_mode)",
                    PREFILL_MODE_NAMES[mode], mode == B200_PREFILL_EXACT ? "" : ", whose f16 GEMMs are not bit-exact");
    if (!rows || !ids_out) return fail(p, B200_ERR_BAD_ARG, "rows and ids_out must not be NULL");
    if (n < 1 || n > p->prefill_batch) return fail(p, B200_ERR_BAD_ARG, "n = %d rows: need 1 <= n <= %d (b200_chunk_rows)", n, p->prefill_batch);
    int rc;
    if ((rc = check_step_rows(p, n, rows, batch_max_rows(p)))) return rc; // at most the batched classifier's rows emit
    CK(cudaSetDevice(p->device));
    return chunk_step(p, n, rows, ids_out, logits);
}

int b200_batch_info(b200_plan *p, int32_t *n_slots, int32_t *launches_per_step, float *device_ms_last_step) {
    if (!p) return B200_ERR_BAD_ARG;
    if (n_slots) *n_slots = p->bt.n_slots;
    if (launches_per_step) *launches_per_step = p->bt.last_launches;
    if (device_ms_last_step) *device_ms_last_step = p->bt.last_ms;
    return B200_OK;
}

int b200_set_logprobs(b200_plan *p, int32_t top_n) {
    if (!p) return B200_ERR_BAD_ARG;
    if (top_n < -1 || top_n > B200_MAX_TOP_LOGPROBS)
        return fail(p, B200_ERR_BAD_ARG, "top_n = %d: -1 (off) or 0..%d alternatives", top_n, B200_MAX_TOP_LOGPROBS);
    auto &L = p->lp;
    if (top_n >= 0) {
        if (p->cfg.tp_size > 1) return fail(p, B200_ERR_UNSUPPORTED, "full logits are not gathered under tensor parallelism: logprobs run on single-GPU plans");
        if (top_n > p->cfg.vocab_size) return fail(p, B200_ERR_BAD_ARG, "top_n = %d exceeds the vocabulary (%d)", top_n, p->cfg.vocab_size);
        // each buffer on its own: a call that failed part-way leaves the rest to the next call, and logprobs stay off until all exist
        CK(cudaSetDevice(p->device));
        const int cap = std::max({p->seq_cap, p->prefill_batch, SMB_MAX_ROWS}); // b200_forward_chunk: a row per chunk row
        int rc;
        if (!L.out && (rc = dalloc(p, &L.out, (size_t)cap * sizeof(LogprobRow)))) return rc;
        if (!L.smp && (rc = dalloc(p, &L.smp, (size_t)SMB_MAX_ROWS * sampler_padded(p->cfg.vocab_size) * 4))) return rc;
        if (!L.h_out) {
            if (cudaMallocHost(&L.h_out, (size_t)cap * sizeof(LogprobRow)) != cudaSuccess) {
                L.h_out = nullptr;
                return fail(p, B200_ERR_OOM, "pinned host memory for the logprobs table (%zu bytes)", (size_t)cap * sizeof(LogprobRow));
            }
        }
        L.cap = cap;
    }
    L.top_n = top_n;
    L.rows = 0;
    return B200_OK;
}

int b200_read_logprobs(b200_plan *p, int32_t max_rows, int32_t *n_rows, double *chosen, int32_t *top_ids, double *top_logprobs) {
    if (!p || !n_rows) return B200_ERR_BAD_ARG;
    const auto &L = p->lp;
    if (L.top_n < 0) return fail(p, B200_ERR_STATE, "logprobs are off: call b200_set_logprobs first");
    *n_rows = L.rows;
    if (!chosen && !top_ids && !top_logprobs) return B200_OK; // the row count alone
    if (max_rows < L.rows) return fail(p, B200_ERR_BAD_ARG, "the table has %d rows, max_rows is %d", L.rows, max_rows);
    const int N = L.top_n;
    for (int i = 0; i < L.rows; i++) {
        const LogprobRow &r = L.h_out[i];
        if (chosen) chosen[i] = r.chosen;
        for (int k = 0; k < N; k++) {
            if (top_ids) top_ids[(size_t)i * N + k] = r.id[k];
            if (top_logprobs) top_logprobs[(size_t)i * N + k] = r.lp[k];
        }
    }
    return B200_OK;
}

// The slot argument of the sampling-control calls: -1 (the plan's own cache) or a decode slot.
static int check_ctl_slot(b200_plan *p, int slot) {
    if (p->cfg.tp_size > 1) return fail(p, B200_ERR_UNSUPPORTED, "sampling controls run on single-GPU plans only: the sampler needs the whole logits row on one GPU");
    if (slot < -1 || slot >= p->bt.n_slots) return fail(p, B200_ERR_BAD_ARG, "slot %d out of range (%d slots; -1 is the plan's own cache)", slot, p->bt.n_slots);
    return B200_OK;
}

int b200_set_sampling_controls(b200_plan *p, int32_t slot, const b200_sampling_controls *c) {
    if (!p) return B200_ERR_BAD_ARG;
    int rc;
    if ((rc = check_ctl_slot(p, slot))) return rc;
    auto &S = p->ctl;
    const int s = slot + 1, V = p->cfg.vocab_size;
    if (!c) { S.on[s] = false; return B200_OK; }
    if ((rc = check_controls(p, *c, V))) return rc;
    CK(cudaSetDevice(p->device));
    CK(cudaStreamSynchronize(p->stream));
    // each buffer on its own: a call that failed part-way leaves the rest to the next call, and no sequence has controls until all exist
    const size_t seqs = SMB_MAX_ROWS + 1;
    if (!S.cnt) {
        int *cnt = nullptr;
        if ((rc = dalloc(p, &cnt, seqs * V * 4))) return rc;
        CK(cudaMemsetAsync(cnt, 0, seqs * V * 4, p->stream));
        CK(cudaStreamSynchronize(p->stream));
        S.cnt = cnt;
    }
    if (!S.bias_id && (rc = dalloc(p, &S.bias_id, seqs * B200_MAX_LOGIT_BIAS * 4))) return rc;
    if (!S.bias_val && (rc = dalloc(p, &S.bias_val, seqs * B200_MAX_LOGIT_BIAS * 4))) return rc;
    if (!S.rows && (rc = dalloc(p, &S.rows, (size_t)SMB_MAX_ROWS * sampler_padded(V) * 4))) return rc;
    if (c->n_bias) { // on the plan's stream, which k_sample_ctl runs on, and complete before the caller's lists may change
        CK(cudaMemcpyAsync(S.bias_id + (size_t)s * B200_MAX_LOGIT_BIAS, c->bias_ids, (size_t)c->n_bias * 4, cudaMemcpyHostToDevice, p->stream));
        CK(cudaMemcpyAsync(S.bias_val + (size_t)s * B200_MAX_LOGIT_BIAS, c->bias_values, (size_t)c->n_bias * 4, cudaMemcpyHostToDevice, p->stream));
        CK(cudaStreamSynchronize(p->stream));
    }
    S.c[s] = *c;
    S.c[s].bias_ids = nullptr;
    S.c[s].bias_values = nullptr;
    S.min_p_log[s] = min_p_log(c->min_p);
    S.on[s] = true;
    return B200_OK;
}

int b200_set_sample_history(b200_plan *p, int32_t slot, const int32_t *tokens, int32_t n) {
    if (!p) return B200_ERR_BAD_ARG;
    int rc;
    if ((rc = check_ctl_slot(p, slot))) return rc;
    if (!p->ctl.cnt) return fail(p, B200_ERR_STATE, "no count tables yet: call b200_set_sampling_controls first");
    if (n < 0 || (n && !tokens)) return fail(p, B200_ERR_BAD_ARG, "n = %d history tokens with %s", n, tokens ? "a list" : "a NULL list");
    if (const int i = bad_token(p, tokens, n); i >= 0) return fail(p, B200_ERR_BAD_ARG, "history token %d: %d out of range", i, tokens[i]);
    const int V = p->cfg.vocab_size;
    std::vector<int32_t> h(V, 0);
    for (int i = 0; i < n; i++) h[tokens[i]]++;
    CK(cudaSetDevice(p->device));
    CK(cudaMemcpyAsync(p->ctl.cnt + (size_t)(slot + 1) * V, h.data(), (size_t)V * 4, cudaMemcpyHostToDevice, p->stream));
    CK(cudaStreamSynchronize(p->stream)); // h is freed on return
    return B200_OK;
}

int b200_read_sample_counts(b200_plan *p, int32_t slot, int32_t *counts) {
    if (!p || !counts) return B200_ERR_BAD_ARG;
    int rc;
    if ((rc = check_ctl_slot(p, slot))) return rc;
    if (!p->ctl.cnt) return fail(p, B200_ERR_STATE, "no count tables yet: call b200_set_sampling_controls first");
    const int V = p->cfg.vocab_size;
    CK(cudaSetDevice(p->device));
    CK(cudaMemcpyAsync(counts, p->ctl.cnt + (size_t)(slot + 1) * V, (size_t)V * 4, cudaMemcpyDeviceToHost, p->stream));
    CK(cudaStreamSynchronize(p->stream));
    return B200_OK;
}

int b200_read_buffer(b200_plan *p, const char *name, int32_t layer, void *dst, size_t bytes) {
    if (!p || !name || !dst) return B200_ERR_BAD_ARG;
    const b200_config &c = p->cfg;
    const void *src = nullptr;
    size_t sz = 0;
    std::string s = name;
    size_t ctx_kv = (size_t)c.context_length * p->kvd_l;
    if (s == "x") { src = p->x; sz = (size_t)c.dim * 4; }
    else if (s == "xb") { src = p->xb; sz = (size_t)(c.dim > p->qd ? c.dim : p->qd) * 4; }
    else if (s == "q" || s == "qkv") { src = p->qkv; sz = (size_t)(p->qd_l + 2 * p->kvd_l) * 4; }
    else if (s == "hb") { src = p->hb; sz = (size_t)(c.hidden_dim > p->moe_hv ? c.hidden_dim : p->moe_hv) * 4; }
    else if (s == "logits") { src = p->logits; sz = (size_t)c.vocab_size * 4; }
    else if (s == "xq") { src = p->xq; sz = (size_t)(c.dim > p->qd ? c.dim : p->qd); }
    else if (s == "xs") { src = p->xs; sz = (size_t)((c.dim > p->qd ? c.dim : p->qd) / 32) * 4; }
    else if (s == "hq") { src = p->hq; sz = (size_t)(c.hidden_dim > p->moe_hv ? c.hidden_dim : p->moe_hv); }
    else if (s == "hs") { src = p->hs; sz = (size_t)((c.hidden_dim > p->moe_hv ? c.hidden_dim : p->moe_hv) / 32) * 4; }
    else if (s == "rope_cr") { src = p->rope_cr; sz = (size_t)c.context_length * (c.head_size / 2) * 4; }
    else if (s == "rope_ci") { src = p->rope_ci; sz = (size_t)c.context_length * (c.head_size / 2) * 4; }
    else if (s == "moe_ids" || s == "moe_weights") {
        if (!p->is_moe) return fail(p, B200_ERR_BAD_ARG, "%s: not a Qwen2-MoE plan", name);
        const size_t k = (size_t)p->moe.n_experts_used;
        if (s == "moe_ids") { src = p->moe_ids; sz = (size_t)c.n_layers * k * 4; }
        else { src = p->moe_w; sz = (size_t)c.n_layers * p->moe_nw * 4; }
    }
    else if (s == "moe_chunk_ids" || s == "moe_chunk_weights") { // the last tensor_core_exact_moe chunk's routing of layer `layer`
        if (!p->is_moe || !p->pi8.xp.maps)
            return fail(p, B200_ERR_STATE, "%s: the plan has no tensor_core_exact_moe buffers (b200_set_prefill_mode)", name);
        if (layer < 0 || layer >= c.n_layers) return fail(p, B200_ERR_BAD_ARG, "layer out of range");
        const XpCtx &x = p->pi8.xp;
        const size_t k = (size_t)p->moe.n_experts_used, rows = (size_t)x.rows, bpad = (size_t)p->pi8.bpad;
        if (s == "moe_chunk_ids") { src = x.ids + (size_t)layer * bpad * k; sz = rows * k * 4; }
        else { src = x.w + (size_t)layer * bpad * p->moe_nw; sz = rows * p->moe_nw * 4; }
    }
    else if (s == "key_cache" || s == "value_cache") {
        if (layer < 0 || layer >= c.n_layers) return fail(p, B200_ERR_BAD_ARG, "layer out of range");
        src = (s == "key_cache" ? p->key_cache : p->value_cache) + (size_t)layer * ctx_kv;
        sz = ctx_kv * 4;
    } else if (s == "slot_key_cache" || s == "slot_value_cache") {
        if (layer < 0 || layer >= p->bt.n_slots * c.n_layers) return fail(p, B200_ERR_BAD_ARG, "slot layer %d out of range (%d slots)", layer, p->bt.n_slots);
        src = (s == "slot_key_cache" ? p->bt.slot_k : p->bt.slot_v) + (size_t)layer * ctx_kv;
        sz = ctx_kv * 4;
    } else if (s.rfind("pf_", 0) == 0) { // tensor-core prefill scratch: [padded rows][width], the last layer of the last chunk
        const PrefillCtx &pc = p->prefill;
        if (!p->pf[B200_PREFILL_TENSOR_CORE].ready && !p->pf[B200_PREFILL_TENSOR_CORE_W8A16].ready)
            return fail(p, B200_ERR_STATE, "%s: the plan has no tensor-core prefill buffers (%s)", name, p->pf[B200_PREFILL_TENSOR_CORE].why);
        const size_t rows = (size_t)pc.bpad;
        if (s == "pf_x") { src = pc.X; sz = rows * c.dim * 4; }
        else if (s == "pf_qkv") { src = pc.QKV; sz = rows * (p->qd + 2 * p->kvd) * 4; }
        else if (s == "pf_a16") { src = pc.A16; sz = rows * c.dim * 2; }
        else if (s == "pf_att16") { src = pc.ATT16; sz = rows * p->qd * 2; }
        else if (s == "pf_h16") { src = pc.H16; sz = rows * c.hidden_dim * 2; }
        else return fail(p, B200_ERR_BAD_ARG, "unknown buffer %s", name);
    } else return fail(p, B200_ERR_BAD_ARG, "unknown buffer %s", name);
    if (bytes < sz) sz = bytes;
    CK(cudaSetDevice(p->device));
    CK(cudaStreamSynchronize(p->stream));
    CK(cudaMemcpy(dst, src, sz, cudaMemcpyDeviceToHost));
    return B200_OK;
}

int b200_time_kernel(b200_plan *p, int32_t which, int32_t reps, float *avg_ms, int64_t *algorithmic_bytes) {
    if (!p || !avg_ms || reps <= 0) return B200_ERR_BAD_ARG;
    if (p->cfg.tp_size > 1) return fail(p, B200_ERR_UNSUPPORTED, "b200_time_kernel is single-GPU only");
    if (p->is_moe) return fail(p, B200_ERR_UNSUPPORTED, "b200_time_kernel times the dense FFN and attention matrices; a %s plan has no dense FFN", p->moe_name);
    if (which < 0 || which > 4) return fail(p, B200_ERR_BAD_ARG, "unknown kernel id %d", which);
    const b200_config &c = p->cfg;
    const bool q8 = p->wtype == B200_GGML_Q8_0, sf = p->use_f16_stream, fz = p->fuse_norm;
    auto tb = [&](const TileMat &m) -> int64_t { return (int64_t)m.rows * m.cols / 32 * 34; };
    auto mat_bytes = [&](const DevMat &m) -> int64_t { return (int64_t)m.rows * m.cols * 2; }; // FP16
    const int64_t nw = fz ? (int64_t)c.dim * 4 : 0; // a fused norm also reads its weights (x: an L2 hit)
    const TraceBuf none{nullptr, 0, 0};
    int64_t bytes = 0;
    auto stream = [&](LayerW &L) -> int { // Q8_0 streaming kernels
        switch (which) {
        case 0:
            bytes = tb(L.tgu) + nw;
            return fz ? launch_stream_norm<SMV_GATEUP>(p, L.tgu, L.ring_gu, L.ffn_norm, false, p->hb, p->hq, p->hs, false, none)
                      : launch_stream<SMV_GATEUP>(p, L.tgu, L.ring_gu, p->xq, p->xs, p->hb, p->hq, p->hs);
        case 1: bytes = tb(L.tw2); return launch_stream<SMV_RESID>(p, L.tw2, SMV_SMEM_BUDGET_MAX, p->hq, p->hs, p->x, nullptr, nullptr);
        case 2:
            bytes = tb(L.tqkv) + nw;
            return fz ? launch_stream_norm<SMV_STORE>(p, L.tqkv, L.ring_qkv, L.attn_norm, false, p->qkv, nullptr, nullptr, false, none)
                      : launch_stream<SMV_STORE>(p, L.tqkv, L.ring_qkv, p->xq, p->xs, p->qkv, nullptr, nullptr);
        case 3: bytes = tb(L.two); return launch_stream<SMV_RESID>(p, L.two, SMV_SMEM_BUDGET_MAX, p->xq, p->xs, p->x, nullptr, nullptr);
        default:
            bytes = tb(p->tout) + nw;
            return fz ? launch_stream_norm<SMV_STORE>(p, p->tout, SMV_SMEM_BUDGET_MAX, p->out_norm, false, p->logits, nullptr, nullptr, false, none)
                      : launch_stream<SMV_STORE>(p, p->tout, SMV_SMEM_BUDGET_MAX, p->xq, p->xs, p->logits, nullptr, nullptr);
        }
    };
    auto f16_stream = [&](LayerW &L) -> int { // FP16 streaming kernels
        switch (which) {
        case 0: bytes = mat_bytes(L.w1) + mat_bytes(L.w3); return launch_stream_f16<SF_GATEUP>(p, L.w1, &L.w3, p->xb, p->hb);
        case 1: bytes = mat_bytes(L.w2); return launch_stream_f16<SF_RESID>(p, L.w2, nullptr, p->hb, p->x);
        case 2: bytes = mat_bytes(L.qkv); return launch_stream_f16<SF_STORE>(p, L.qkv, nullptr, p->xb, p->qkv);
        case 3: bytes = mat_bytes(L.wo); return launch_stream_f16<SF_RESID>(p, L.wo, nullptr, p->xb, p->x);
        default: bytes = mat_bytes(p->out); return launch_stream_f16<SF_STORE>(p, p->out, nullptr, p->xb, p->logits);
        }
    };
    auto matvec = [&](LayerW &L) -> int { // the FP16 fallback kernels
        switch (which) {
        case 0: {
            int rc;
            if ((rc = launch_matvec_f16<MODE_STORE>(p, L.w1, p->xb, p->hb))) return rc;
            if ((rc = launch_matvec_f16<MODE_STORE>(p, L.w3, p->xb, p->hb2))) return rc;
            bytes = mat_bytes(L.w1) + mat_bytes(L.w3);
            return B200_OK;
        }
        case 1: bytes = mat_bytes(L.w2); return launch_matvec_f16<MODE_RESID>(p, L.w2, p->hb, p->x);
        case 2: bytes = mat_bytes(L.qkv); return launch_matvec_f16<MODE_STORE>(p, L.qkv, p->xb, p->qkv);
        case 3: bytes = mat_bytes(L.wo); return launch_matvec_f16<MODE_RESID>(p, L.wo, p->xb, p->x);
        default: bytes = mat_bytes(p->out); return launch_matvec_f16<MODE_STORE>(p, p->out, p->xb, p->logits);
        }
    };
    // one launch on layer l's matrix; the streaming kernels run stand-alone (no PDL overlap)
    auto one = [&](int l) -> int {
        LayerW &L = p->layers[l];
        if (!q8 && !sf) return matvec(L);
        const bool keep = p->use_pdl;
        p->use_pdl = false;
        const int r = q8 ? stream(L) : f16_stream(L);
        p->use_pdl = keep;
        return r;
    };
    CK(cudaSetDevice(p->device));
    std::vector<float> save(c.dim);
    CK(cudaStreamSynchronize(p->stream));
    CK(cudaMemcpy(save.data(), p->x, (size_t)c.dim * 4, cudaMemcpyDeviceToHost));
    int rc, launches = 0;
    for (int l = 0; l < c.n_layers; l++) if ((rc = one(l))) return rc; // warm-up pass (also defeats L2 for pass 1)
    CK(cudaEventRecord(p->ev0, p->stream));
    for (int r = 0; r < reps; r++)
        for (int l = 0; l < c.n_layers; l++) { if ((rc = one(l))) return rc; launches++; }
    CK(cudaEventRecord(p->ev1, p->stream));
    CK(cudaStreamSynchronize(p->stream));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, p->ev0, p->ev1));
    *avg_ms = ms / launches;
    if (algorithmic_bytes) *algorithmic_bytes = bytes;
    CK(cudaMemcpy(p->x, save.data(), (size_t)c.dim * 4, cudaMemcpyHostToDevice));
    return B200_OK;
}

int b200_tp_handle(b200_plan *p, void *handle64) {
    if (!p || !handle64) return B200_ERR_BAD_ARG;
    if (p->cfg.tp_size <= 1 || !p->comm) return fail(p, B200_ERR_STATE, "not a tensor-parallel plan");
    CK(cudaSetDevice(p->device));
    cudaIpcMemHandle_t h;
    CK(cudaIpcGetMemHandle(&h, p->comm));
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    memcpy(handle64, &h, 64);
    return B200_OK;
}

int b200_tp_attach(b200_plan *p, const void *handles, int32_t n) {
    if (!p || !handles) return B200_ERR_BAD_ARG;
    if (p->cfg.tp_size <= 1 || !p->comm) return fail(p, B200_ERR_STATE, "not a tensor-parallel plan");
    if (n != p->cfg.tp_size) return fail(p, B200_ERR_BAD_ARG, "expected %d handles, got %d", p->cfg.tp_size, n);
    if (p->attached) return fail(p, B200_ERR_STATE, "already attached");
    CK(cudaSetDevice(p->device));
    for (int k = 0; k < n; k++) {
        if (k == p->cfg.tp_rank) { p->tp.peer[k] = p->comm; continue; }
        cudaIpcMemHandle_t h;
        memcpy(&h, (const unsigned char *)handles + (size_t)k * 64, 64);
        void *ptr = nullptr;
        CK(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
        p->peer_open[k] = ptr;
        p->tp.peer[k] = (unsigned char *)ptr;
    }
    p->tp.n = n;
    p->attached = true;
    int rc;
    if ((rc = capture_all(p))) return rc;
    CK(cudaStreamSynchronize(p->stream));
    return B200_OK;
}

int b200_trace_decode(b200_plan *p, int32_t token, int32_t position, uint64_t *records, int32_t cap, int32_t *n_out) {
    if (!p || !records || !n_out) return B200_ERR_BAD_ARG;
    if (!p->graph.trace.exec) return fail(p, B200_ERR_UNSUPPORTED, "tracing needs a streaming path (Q8_0 tiles or the FP16 rings)");
    int rc;
    if ((rc = check_pos(p, token, position))) return rc;
    CK(cudaSetDevice(p->device));
    int n = p->graph.trace.launches;
    std::vector<unsigned long long> init((size_t)n * 4);
    for (int i = 0; i < n; i++) { init[i * 4] = 0; init[i * 4 + 1] = ~0ull; init[i * 4 + 2] = 0; init[i * 4 + 3] = 0; }
    CK(cudaMemcpyAsync(p->trace_rec, init.data(), init.size() * 8, cudaMemcpyHostToDevice, p->stream));
    if ((rc = set_state(p, token, position, 0, 0))) return rc;
    CK(cudaGraphLaunch(p->graph.trace.exec, p->stream));
    CK(cudaStreamSynchronize(p->stream));
    int m = n < cap ? n : cap;
    CK(cudaMemcpy(records, p->trace_rec, (size_t)m * 32, cudaMemcpyDeviceToHost));
    *n_out = m;
    return B200_OK;
}

int b200_profile_norm(b200_plan *p, int64_t *cycles4) {
    if (!p || !cycles4) return B200_ERR_BAD_ARG;
    CK(cudaSetDevice(p->device));
    long long *d = nullptr;
    CK(cudaMalloc(&d, 128));
    const b200_config &c = p->cfg;
    const size_t norm_smem = norm_smem_bytes(c.dim);
    const bool q8 = p->wtype == B200_GGML_Q8_0;
    for (int i = 0; i < 3; i++)
        k_rmsnorm_quant<false><<<1, NORM_THREADS, norm_smem, p->stream>>>(p->x, p->st, p->emb, 1.0f, p->layers[0].attn_norm, c.rms_norm_eps, c.dim,
                                                                 q8 ? p->xq : nullptr, q8 ? p->xs : nullptr, q8 ? nullptr : p->xb, d, TraceBuf{nullptr, 0, 0}, p->tp, -1);
    cudaError_t e = cudaStreamSynchronize(p->stream);
    long long h[6] = {0};
    if (e == cudaSuccess) e = cudaMemcpy(h, d, sizeof(h), cudaMemcpyDeviceToHost);
    cudaFree(d);
    for (int i = 0; i < 16; i++) cycles4[i] = i < 6 ? h[i] : 0;
    return e == cudaSuccess ? B200_OK : B200_ERR_CUDA;
}

int b200_test_seqsum2(const float *terms, int32_t n, int32_t threads, float *out, int32_t *info) {
    if (!terms || !out || n <= 0 || n > 16384) return B200_ERR_BAD_ARG;
    if (threads != 256 && threads != 512 && threads != 1024) return B200_ERR_BAD_ARG;
    Scratch s;
    float *d = nullptr, *o = nullptr;
    if (!s.alloc(&d, (size_t)n * 4) || !s.alloc(&o, 16)) return B200_ERR_OOM;
    cudaError_t e = cudaMemcpy(d, terms, (size_t)n * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        if (threads == 1024) {
            const size_t smem = (size_t)1024 * ((n + 1023) / 1024) * 4 + seqsum2_scratch_bytes(1024);
            e = cudaFuncSetAttribute(k_test_seqsum2<1024>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e == cudaSuccess) k_test_seqsum2<1024><<<1, 1024, smem>>>(d, n, o, reinterpret_cast<int *>(o) + 1);
        } else if (threads == 512) {
            const size_t smem = (size_t)512 * ((n + 511) / 512) * 4 + seqsum2_scratch_bytes(512);
            e = cudaFuncSetAttribute(k_test_seqsum2<512>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e == cudaSuccess) k_test_seqsum2<512><<<1, 512, smem>>>(d, n, o, reinterpret_cast<int *>(o) + 1);
        } else {
            const size_t smem = (size_t)256 * ((n + 255) / 256) * 4 + seqsum2_scratch_bytes(256);
            e = cudaFuncSetAttribute(k_test_seqsum2<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e == cudaSuccess) k_test_seqsum2<256><<<1, 256, smem>>>(d, n, o, reinterpret_cast<int *>(o) + 1);
        }
    }
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    int32_t host[3] = {0, 0, 0};
    if (e == cudaSuccess) e = cudaMemcpy(host, o, 12, cudaMemcpyDeviceToHost);
    memcpy(out, host, 4);
    if (info) { info[0] = host[1]; info[1] = host[2]; }
    return e == cudaSuccess ? B200_OK : B200_ERR_CUDA;
}

int b200_test_logprobs(const float *logits, int32_t vocab, int32_t chosen_id, int32_t top_n, int32_t reps, double *chosen, int32_t *top_ids,
                       double *top_logprobs, float *avg_ms) {
    if (!logits || vocab <= 0 || chosen_id < 0 || chosen_id >= vocab || top_n < 0 || top_n > LOGPROB_MAX_TOP || top_n > vocab || reps < 1)
        return B200_ERR_BAD_ARG;
    Scratch s;
    float *d = nullptr;
    int *id = nullptr;
    LogprobRow *out = nullptr;
    if (!s.alloc(&d, (size_t)vocab * 4) || !s.alloc(&id, 4) || !s.alloc(&out, sizeof(LogprobRow))) return s.rc;
    LogprobArgs a{};
    a.logits = d; a.stride = 0; a.vocab = vocab; a.n_top = top_n; a.ids[0] = id; a.out_row[0] = 0; a.out = out;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    s.ok(cudaMemcpy(d, logits, (size_t)vocab * 4, cudaMemcpyHostToDevice)) && s.ok(cudaMemcpy(id, &chosen_id, 4, cudaMemcpyHostToDevice)) &&
        s.ok(cudaEventCreate(&e0)) && s.ok(cudaEventCreate(&e1));
    if (s.rc == B200_OK) {
        k_token_logprobs<<<1, SCORE_THREADS>>>(a); // warm-up
        s.ok(cudaEventRecord(e0));
        for (int r = 0; r < reps; r++) k_token_logprobs<<<1, SCORE_THREADS>>>(a);
        s.ok(cudaEventRecord(e1)) && s.ok(cudaGetLastError()) && s.ok(cudaEventSynchronize(e1));
    }
    float ms = 0.f;
    LogprobRow h{};
    if (s.rc == B200_OK && s.ok(cudaEventElapsedTime(&ms, e0, e1)) && s.ok(cudaMemcpy(&h, out, sizeof(LogprobRow), cudaMemcpyDeviceToHost))) {
        if (avg_ms) *avg_ms = ms / reps;
        if (chosen) *chosen = h.chosen;
        for (int k = 0; k < top_n; k++) {
            if (top_ids) top_ids[k] = h.id[k];
            if (top_logprobs) top_logprobs[k] = h.lp[k];
        }
    }
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    return s.rc;
}

int b200_profile_seqsum2(const float *terms, int32_t n, int32_t threads, int64_t *cycles, float *out) {
    if (!terms || !cycles || !out || n <= 0 || n > 16384) return B200_ERR_BAD_ARG;
    if (threads != 256 && threads != 512 && threads != 1024) return B200_ERR_BAD_ARG;
    Scratch s;
    float *d = nullptr, *o = nullptr;
    long long *cyc = nullptr;
    if (!s.alloc(&d, (size_t)n * 4) || !s.alloc(&o, 16) || !s.alloc(&cyc, 40)) return B200_ERR_OOM;
    cudaError_t e = cudaMemcpy(d, terms, (size_t)n * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = threads == 1024 ? launch_profile_seqsum2<1024>(d, n, cyc, o)
                            : threads == 512 ? launch_profile_seqsum2<512>(d, n, cyc, o) : launch_profile_seqsum2<256>(d, n, cyc, o);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(cycles, cyc, 40, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(out, o, 8, cudaMemcpyDeviceToHost);
    return e == cudaSuccess ? B200_OK : B200_ERR_CUDA;
}

int b200_test_sample(const float *logits, int32_t n, float temperature, float topp, float uniform01, int32_t *token_out, int32_t *info, float *probs_out) {
    if (!logits || !token_out || n < 1) return B200_ERR_BAD_ARG;
    if (!(temperature > 0.0f) || !(uniform01 >= 0.0f && uniform01 < 1.0f)) return B200_ERR_BAD_ARG;
    const size_t padded = (size_t)sampler_padded(n) * 4;
    float *dl = nullptr;
    int *di = nullptr, *dout = nullptr;
    Scratch s;
    // the index scratch starts as 0xFF bytes: a slot the kernel did not write in this call reads as -1
    if (s.alloc(&dl, padded) && s.alloc(&di, (size_t)n * 4) && s.alloc(&dout, 8 * 4) && s.ok(cudaMemset(dl, 0, padded)) &&
        s.ok(cudaMemcpy(dl, logits, (size_t)n * 4, cudaMemcpyHostToDevice)) && s.ok(cudaMemset(di, 0xFF, (size_t)n * 4)) && s.ok(cudaMemset(dout, 0xFF, 8 * 4)) &&
        s.ok(cudaFuncSetAttribute(k_sample_rows, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sampler_smem_bytes()))) {
        SamplerRowsArgs a;
        a.logits = dl; a.stride = 0; a.n = n; a.indices = di; a.out = dout;
        a.row[0] = 0; a.temperature[0] = temperature; a.topp[0] = topp; a.r01[0] = uniform01;
        k_sample_rows<<<1, SAMPLER_THREADS, sampler_smem_bytes()>>>(a);
        int32_t h[5];
        if (s.ok(cudaGetLastError()) && s.ok(cudaDeviceSynchronize()) && s.ok(cudaMemcpy(h, dout, 5 * 4, cudaMemcpyDeviceToHost))) {
            *token_out = h[0];
            if (info) for (int k = 0; k < 4; k++) info[k] = h[1 + k];
            if (probs_out) s.ok(cudaMemcpy(probs_out, dl, (size_t)n * 4, cudaMemcpyDeviceToHost));
        }
    }
    return s.rc;
}

int b200_test_sample_controls(const float *logits, int32_t n, int32_t *counts, const b200_sampling_controls *c, float temperature, float topp,
                              float uniform01, int32_t *token_out, int32_t *info, float *row_out) {
    if (!logits || !counts || !c || !token_out || n < 1) return B200_ERR_BAD_ARG;
    if (!(temperature >= 0.0f) || !(uniform01 >= 0.0f && uniform01 < 1.0f)) return B200_ERR_BAD_ARG;
    if (check_controls(nullptr, *c, n)) return B200_ERR_BAD_ARG;
    const size_t padded = (size_t)sampler_padded(n) * 4, nb = (size_t)(c->n_bias ? c->n_bias : 1) * 4;
    float *dl = nullptr, *drow = nullptr, *dout_row = nullptr, *dbv = nullptr;
    int *dcnt = nullptr, *di = nullptr, *dout = nullptr, *dbi = nullptr;
    Scratch s;
    if (s.alloc(&dl, (size_t)n * 4) && s.alloc(&drow, padded) && s.alloc(&dout_row, (size_t)n * 4) && s.alloc(&dcnt, (size_t)n * 4) &&
        s.alloc(&di, (size_t)n * 4) && s.alloc(&dout, 8 * 4) && s.alloc(&dbi, nb) && s.alloc(&dbv, nb) &&
        s.ok(cudaMemcpy(dl, logits, (size_t)n * 4, cudaMemcpyHostToDevice)) && s.ok(cudaMemcpy(dcnt, counts, (size_t)n * 4, cudaMemcpyHostToDevice)) &&
        s.ok(cudaMemset(dout, 0xFF, 8 * 4)) &&
        (!c->n_bias || (s.ok(cudaMemcpy(dbi, c->bias_ids, nb, cudaMemcpyHostToDevice)) && s.ok(cudaMemcpy(dbv, c->bias_values, nb, cudaMemcpyHostToDevice)))) &&
        s.ok(cudaFuncSetAttribute(k_sample_ctl, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sampler_smem_bytes()))) {
        SampleCtlArgs a;
        a.n = n;
        SampleCtlRow &r = a.row[0];
        r.src = dl; r.dst = drow; r.row_out = dout_row; r.cnt = dcnt; r.bias_id = dbi; r.bias_val = dbv; r.n_bias = c->n_bias;
        r.top_k = c->top_k; r.min_p_log = min_p_log(c->min_p); r.rep = c->repetition_penalty; r.freq = c->frequency_penalty; r.pres = c->presence_penalty;
        r.temperature = temperature; r.topp = topp; r.r01 = uniform01; r.indices = di; r.out = dout;
        k_sample_ctl<<<1, SAMPLER_THREADS, sampler_smem_bytes()>>>(a);
        int32_t h[5];
        if (s.ok(cudaGetLastError()) && s.ok(cudaDeviceSynchronize()) && s.ok(cudaMemcpy(h, dout, 5 * 4, cudaMemcpyDeviceToHost)) &&
            s.ok(cudaMemcpy(counts, dcnt, (size_t)n * 4, cudaMemcpyDeviceToHost))) {
            *token_out = h[0];
            if (info) for (int k = 0; k < 4; k++) info[k] = h[1 + k];
            if (row_out) s.ok(cudaMemcpy(row_out, dout_row, (size_t)n * 4, cudaMemcpyDeviceToHost));
        }
    }
    return s.rc;
}

int b200_time_sample_controls(const float *logits, int32_t n, const int32_t *counts, const b200_sampling_controls *c, float temperature, float topp,
                              float uniform01, int32_t reps, float *ctl_ms, float *plain_ms) {
    if (!logits || !counts || !c || !ctl_ms || !plain_ms || n < 1 || reps < 1) return B200_ERR_BAD_ARG;
    if (!(temperature > 0.0f) || !(uniform01 >= 0.0f && uniform01 < 1.0f)) return B200_ERR_BAD_ARG;
    if (check_controls(nullptr, *c, n)) return B200_ERR_BAD_ARG;
    // k_sample_rows turns its row into probabilities and k_sample_ctl counts its id: every launch, the warm-up's included, gets its own copy
    const size_t pad = (size_t)sampler_padded(n), copies = (size_t)reps + 1, nb = (size_t)(c->n_bias ? c->n_bias : 1) * 4;
    float *dl = nullptr, *drow = nullptr, *dbv = nullptr;
    int *dcnt = nullptr, *di = nullptr, *dout = nullptr, *dbi = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr, e2 = nullptr;
    Scratch s;
    if (!(s.alloc(&dl, copies * pad * 4) && s.alloc(&drow, pad * 4) && s.alloc(&dcnt, copies * n * 4) && s.alloc(&di, (size_t)n * 4) &&
          s.alloc(&dout, 8 * 4) && s.alloc(&dbi, nb) && s.alloc(&dbv, nb) && s.ok(cudaMemset(dl, 0, copies * pad * 4)) &&
          s.ok(cudaMemcpy(dl, logits, (size_t)n * 4, cudaMemcpyHostToDevice)) && s.ok(cudaMemcpy(dcnt, counts, (size_t)n * 4, cudaMemcpyHostToDevice)) &&
          (!c->n_bias || (s.ok(cudaMemcpy(dbi, c->bias_ids, nb, cudaMemcpyHostToDevice)) && s.ok(cudaMemcpy(dbv, c->bias_values, nb, cudaMemcpyHostToDevice)))) &&
          s.ok(cudaFuncSetAttribute(k_sample_ctl, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sampler_smem_bytes())) &&
          s.ok(cudaFuncSetAttribute(k_sample_rows, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sampler_smem_bytes())) &&
          s.ok(cudaEventCreate(&e0)) && s.ok(cudaEventCreate(&e1)) && s.ok(cudaEventCreate(&e2))))
        return s.rc;
    for (size_t r = 1; r < copies && s.rc == B200_OK; r++)
        s.ok(cudaMemcpy(dl + r * pad, dl, (size_t)n * 4, cudaMemcpyDeviceToDevice)) && s.ok(cudaMemcpy(dcnt + r * n, dcnt, (size_t)n * 4, cudaMemcpyDeviceToDevice));
    float ms_ctl = 0.f, ms_plain = 0.f;
    if (s.rc == B200_OK) {
        SampleCtlArgs a;
        a.n = n;
        SampleCtlRow &w = a.row[0];
        w.dst = drow; w.row_out = nullptr; w.bias_id = dbi; w.bias_val = dbv; w.n_bias = c->n_bias;
        w.top_k = c->top_k; w.min_p_log = min_p_log(c->min_p); w.rep = c->repetition_penalty; w.freq = c->frequency_penalty; w.pres = c->presence_penalty;
        w.temperature = temperature; w.topp = topp; w.r01 = uniform01; w.indices = di; w.out = dout;
        SamplerRowsArgs b;
        b.stride = 0; b.n = n; b.indices = di; b.out = dout;
        b.row[0] = 0; b.temperature[0] = temperature; b.topp[0] = topp; b.r01[0] = uniform01;
        auto ctl = [&](size_t r) { w.src = dl + r * pad; w.cnt = dcnt + r * n; k_sample_ctl<<<1, SAMPLER_THREADS, sampler_smem_bytes()>>>(a); };
        auto plain = [&](size_t r) { b.logits = dl + r * pad; k_sample_rows<<<1, SAMPLER_THREADS, sampler_smem_bytes()>>>(b); };
        ctl(reps); // warm-up on the last copy: k_sample_ctl only reads the row, so k_sample_rows' warm-up can follow on it
        plain(reps);
        s.ok(cudaEventRecord(e0));
        for (int r = 0; r < reps; r++) ctl(r);
        s.ok(cudaEventRecord(e1));
        for (int r = 0; r < reps; r++) plain(r);
        s.ok(cudaEventRecord(e2)) && s.ok(cudaGetLastError()) && s.ok(cudaEventSynchronize(e2)) && s.ok(cudaEventElapsedTime(&ms_ctl, e0, e1)) &&
            s.ok(cudaEventElapsedTime(&ms_plain, e1, e2));
    }
    if (s.rc == B200_OK) { *ctl_ms = ms_ctl / reps; *plain_ms = ms_plain / reps; }
    for (cudaEvent_t e : {e0, e1, e2})
        if (e) cudaEventDestroy(e);
    return s.rc;
}

int b200_requant_kquant(int32_t ggml_type, const void *src, int64_t n_elems, void *dst_q8_0) {
    if (!src || !dst_q8_0 || n_elems <= 0 || n_elems % 256 || !kq_is_kquant(ggml_type)) return B200_ERR_BAD_ARG;
    const size_t raw = (size_t)(n_elems / 256) * kq_block_bytes(ggml_type), q8 = (size_t)(n_elems / 32) * 34;
    unsigned char *ds = nullptr, *dd = nullptr;
    Scratch s;
    if (s.alloc(&ds, raw) && s.alloc(&dd, q8) && s.ok(cudaMemcpy(ds, src, raw, cudaMemcpyHostToDevice)) &&
        s.ok(launch_requant_kquant(ggml_type, ds, dd, n_elems / 32, 0)) && s.ok(cudaDeviceSynchronize()))
        s.ok(cudaMemcpy(dst_q8_0, dd, q8, cudaMemcpyDeviceToHost));
    return s.rc;
}

int b200_test_kq_tiles_to_q8(int32_t ggml_type, int32_t rows, int32_t cols, const void *kq_rows, void *q8_tiles_out, int64_t bytes) {
    if (!kq_rows || !q8_tiles_out || rows < 1 || cols < 256 || cols % 256 || !kq_is_kquant(ggml_type)) return B200_ERR_BAD_ARG;
    TileMat W = tile_geometry(rows, cols, ggml_type);
    const TileMat Q = tile_geometry(rows, cols, 0);
    if (!W.nseg || !Q.nseg) return B200_ERR_BAD_ARG;
    if (bytes != tile_bytes(Q)) return B200_ERR_BAD_ARG;
    const size_t raw = (size_t)rows * (cols / 256) * kq_block_bytes(ggml_type);
    unsigned char *draw = nullptr, *dres = nullptr, *dq8 = nullptr;
    Scratch s;
    // the resident tiles as upload_tiles lays them out, then the expansion as prefill_forward_i8 launches it
    if (s.alloc(&draw, raw) && s.alloc(&dres, (size_t)tile_bytes(W)) && s.alloc(&dq8, (size_t)bytes) &&
        s.ok(cudaMemcpy(draw, kq_rows, raw, cudaMemcpyHostToDevice)) && s.ok(cudaMemset(dq8, 0xA5, (size_t)bytes))) {
        RepackSrc src{};
        src.raw[0] = draw;
        src.rows[0] = rows;
        k_repack_kq_tiles<<<(unsigned)((size_t)tile_groups(W) * 4 * W.nseg), 128>>>(src, dres, rows, cols, W.seg, W.nseg, W.unit_bytes, kq_block_bytes(ggml_type));
        W.base = dres;
        if (s.ok(cudaGetLastError()) && s.ok(launch_kq_tiles_to_q8(W, Q, dq8, 0)) && s.ok(cudaDeviceSynchronize()))
            s.ok(cudaMemcpy(q8_tiles_out, dq8, (size_t)bytes, cudaMemcpyDeviceToHost));
    }
    return s.rc;
}

int b200_gemm_f16(const uint16_t *a, const uint16_t *b, float *c, int32_t m, int32_t n, int32_t k, int32_t iters, float *ms) {
    const int stages = getenv("B200_GEMM_STAGES") ? atoi(getenv("B200_GEMM_STAGES")) : 0;
    // B200_GEMM_RESID=s: the reduce-add epilogue with K split s ways; C starts at 0 and accumulates over the timed launches
    const int resid = getenv("B200_GEMM_RESID") ? atoi(getenv("B200_GEMM_RESID")) : 0;
    if (!a || !b || !c || m <= 0 || n <= 0 || k <= 0 || m % 128 || n % 128 || k % 64) return B200_ERR_BAD_ARG;
    __half *da = nullptr, *db = nullptr;
    float *dc = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    Scratch s;
    if (s.alloc(&da, (size_t)m * k * 2) && s.alloc(&db, (size_t)n * k * 2) && s.alloc(&dc, (size_t)m * n * 4) &&
        s.ok(cudaMemcpy(da, a, (size_t)m * k * 2, cudaMemcpyHostToDevice)) && s.ok(cudaMemcpy(db, b, (size_t)n * k * 2, cudaMemcpyHostToDevice)) &&
        s.ok(cudaMemset(dc, resid ? 0 : 0xFF, (size_t)m * n * 4))) {
        if (pg::gemm_f16(da, db, dc, m, n, k, stages, resid, 0)) s.rc = B200_ERR_CUDA;
        s.ok(cudaDeviceSynchronize());
        if (s.rc == B200_OK && iters > 0 && ms && s.ok(cudaEventCreate(&e0)) && s.ok(cudaEventCreate(&e1)) && s.ok(cudaEventRecord(e0, 0))) {
            for (int i = 0; i < iters && s.rc == B200_OK; i++)
                if (pg::gemm_f16(da, db, dc, m, n, k, stages, resid, 0)) s.rc = B200_ERR_CUDA;
            float t = 0.f;
            if (s.ok(cudaEventRecord(e1, 0)) && s.ok(cudaEventSynchronize(e1)) && s.ok(cudaEventElapsedTime(&t, e0, e1))) *ms = t / iters;
            if (s.rc == B200_OK && resid) { // C accumulated 1 + iters products: return exactly one
                if (s.ok(cudaMemset(dc, 0, (size_t)m * n * 4)) && pg::gemm_f16(da, db, dc, m, n, k, stages, resid, 0)) s.rc = B200_ERR_CUDA;
                s.ok(cudaDeviceSynchronize());
            }
        }
        if (s.rc == B200_OK) s.ok(cudaMemcpy(c, dc, (size_t)m * n * 4, cudaMemcpyDeviceToHost));
    }
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    return s.rc;
}

int b200_test_gemm(int32_t mode, int32_t stages, int32_t splits, int32_t m, int32_t m_valid, int32_t n, int32_t k, const uint16_t *a, const uint16_t *b,
                   const uint16_t *b2, void *c) {
    const bool gateup = mode == pg::GEMM_GATEUP;
    if (mode < pg::GEMM_F32 || mode > pg::GEMM_GATEUP || (stages != pg::GEMM_STAGES && stages != pg::GEMM_STAGES_DEEP)) return B200_ERR_BAD_ARG;
    if (!a || !b || !c || (gateup && !b2) || m <= 0 || n <= 0 || k <= 0 || m % pg::BM || k % pg::BK || n % (gateup ? pg::BN / 2 : pg::BN)) return B200_ERR_BAD_ARG;
    if (m_valid < 1 || m_valid > m || splits < 1) return B200_ERR_BAD_ARG;
    const size_t c_bytes = (size_t)m * n * (gateup ? 2 : 4);
    __half *da = nullptr, *db = nullptr, *db2 = nullptr;
    void *dc = nullptr;
    Scratch s;
    if (s.alloc(&da, (size_t)m * k * 2) && s.alloc(&db, (size_t)n * k * 2) && (!gateup || s.alloc(&db2, (size_t)n * k * 2)) &&
        s.alloc(&dc, c_bytes) && s.ok(cudaMemcpy(da, a, (size_t)m * k * 2, cudaMemcpyHostToDevice)) &&
        s.ok(cudaMemcpy(db, b, (size_t)n * k * 2, cudaMemcpyHostToDevice)) && (!gateup || s.ok(cudaMemcpy(db2, b2, (size_t)n * k * 2, cudaMemcpyHostToDevice))) &&
        s.ok(cudaMemcpy(dc, c, c_bytes, cudaMemcpyHostToDevice))) {
        // the same maps prefill_forward builds: A boxes of 128 rows, B boxes of 128 rows (64 for each half of the gate/up tile), C boxes 128 x 32 f32
        CUtensorMap ma, mb, mb2, mc;
        const uint32_t b_rows = gateup ? pg::BN / 2 : pg::BN;
        if (pg::make_map(&ma, da, (uint64_t)m, (uint64_t)k, pg::BM) || pg::make_map(&mb, db, (uint64_t)n, (uint64_t)k, b_rows) ||
            pg::make_map(&mb2, gateup ? db2 : db, (uint64_t)n, (uint64_t)k, b_rows) || (!gateup && pg::make_map_c(&mc, dc, (uint64_t)m, (uint64_t)n)))
            s.rc = B200_ERR_CUDA;
        if (gateup) mc = mb; // unused by the gate/up epilogue, which stores f16 through plain pointers
        if (s.rc == B200_OK) {
            const int mt = m / pg::BM, nt = n / (gateup ? pg::BN / 2 : pg::BN);
            const bool deep = stages == pg::GEMM_STAGES_DEEP;
            const int lr = with_gemm_mode(mode, [&](auto MODE) {
                return deep ? pg::gemm_launch<MODE, pg::GEMM_STAGES_DEEP>(ma, mb, mb2, mc, dc, n, m_valid, mt, nt, k, 0, splits)
                            : pg::gemm_launch<MODE, pg::GEMM_STAGES>(ma, mb, mb2, mc, dc, n, m_valid, mt, nt, k, 0, splits);
            });
            if (lr == -6) s.rc = B200_ERR_BAD_ARG; // splits > 1 outside GEMM_RESID, or a split with no k-block
            else if (lr) s.rc = B200_ERR_CUDA;
        }
        if (s.ok(cudaDeviceSynchronize()) && s.rc == B200_OK) s.ok(cudaMemcpy(c, dc, c_bytes, cudaMemcpyDeviceToHost));
    }
    return s.rc;
}

int b200_test_gemm_q8(int32_t mode, int32_t stages, int32_t splits, int32_t m, int32_t m_valid, int32_t n, int32_t k, const uint16_t *a, const void *bq,
                      const void *bq2, void *c) {
    const bool gateup = mode == pg::GEMM_GATEUP;
    if (mode < pg::GEMM_F32 || mode > pg::GEMM_GATEUP || (stages != pg::GEMM_STAGES && stages != pg::GEMM_STAGES_DEEP_Q8)) return B200_ERR_BAD_ARG;
    if (!a || !bq || !c || (gateup && !bq2) || m <= 0 || n <= 0 || k <= 0 || m % pg::BM || k % pg::BK || n % (gateup ? pg::BN / 2 : pg::BN)) return B200_ERR_BAD_ARG;
    if (m_valid < 1 || m_valid > m || splits < 1) return B200_ERR_BAD_ARG;
    // the stream exactly as upload_tiles lays it out; W8A16 needs whole 64-column k-blocks inside each segment
    const int nseg = smv_pick_nseg(k);
    if (!nseg || (k / nseg) % pg::BK) return B200_ERR_BAD_ARG;
    const int seg = k / nseg, unit = smv_unit_bytes(seg), rows = gateup ? 2 * n : n;
    const size_t c_bytes = (size_t)m * n * (gateup ? 2 : 4), q8_bytes = (size_t)n * (k / 32) * 34, stream_bytes = (size_t)rows * nseg * unit;
    __half *da = nullptr;
    unsigned char *draw = nullptr, *dstream = nullptr;
    void *dc = nullptr;
    Scratch s;
    if (s.alloc(&da, (size_t)m * k * 2) && s.alloc(&draw, q8_bytes * (gateup ? 2 : 1)) && s.alloc(&dstream, stream_bytes) &&
        s.alloc(&dc, c_bytes) && s.ok(cudaMemcpy(da, a, (size_t)m * k * 2, cudaMemcpyHostToDevice)) && s.ok(cudaMemcpy(draw, bq, q8_bytes, cudaMemcpyHostToDevice)) &&
        (!gateup || s.ok(cudaMemcpy(draw + q8_bytes, bq2, q8_bytes, cudaMemcpyHostToDevice))) && s.ok(cudaMemcpy(dc, c, c_bytes, cudaMemcpyHostToDevice))) {
        RepackSrc src{};
        src.raw[0] = draw;
        src.rows[0] = n;
        if (gateup) { src.raw[1] = draw + q8_bytes; src.rows[1] = n; }
        src.gateup = gateup ? 1 : 0;
        k_repack_tiles<<<(unsigned)((size_t)rows * nseg), 128>>>(src, dstream, rows, k, seg, nseg, unit);
        s.ok(cudaGetLastError());
        // the maps prefill_init_q8 builds and the A / C maps of the prefill scratch
        CUtensorMap ma, mq, ms, mc;
        if (s.rc == B200_OK && (pg::make_map(&ma, da, (uint64_t)m, (uint64_t)k, pg::BM) || pg::make_map_q8(&mq, dstream, (uint64_t)rows, nseg, unit, 0) ||
                                pg::make_map_q8(&ms, dstream, (uint64_t)rows, nseg, unit, 1) || (!gateup && pg::make_map_c(&mc, dc, (uint64_t)m, (uint64_t)n))))
            s.rc = B200_ERR_CUDA;
        if (gateup) mc = mq; // unused by the gate/up epilogue
        if (s.rc == B200_OK) {
            using pg::B_Q8;
            const int mt = m / pg::BM, nt = n / (gateup ? pg::BN / 2 : pg::BN);
            const bool deep = stages == pg::GEMM_STAGES_DEEP_Q8;
            const int lr = with_gemm_mode(mode, [&](auto MODE) {
                return deep ? pg::gemm_launch<MODE, pg::GEMM_STAGES_DEEP_Q8, B_Q8>(ma, mq, ms, mc, dc, n, m_valid, mt, nt, k, 0, splits, seg)
                            : pg::gemm_launch<MODE, pg::GEMM_STAGES, B_Q8>(ma, mq, ms, mc, dc, n, m_valid, mt, nt, k, 0, splits, seg);
            });
            if (lr == -6) s.rc = B200_ERR_BAD_ARG;
            else if (lr) s.rc = B200_ERR_CUDA;
        }
        if (s.ok(cudaDeviceSynchronize()) && s.rc == B200_OK) s.ok(cudaMemcpy(c, dc, c_bytes, cudaMemcpyDeviceToHost));
    }
    return s.rc;
}

int b200_test_gemm_i8(int32_t mode, int32_t m, int32_t n, int32_t k, const int8_t *aq, const float *as, const void *bq, const void *bq2, float oscale,
                      float *c, int8_t *hq, float *hs) {
    const bool gateup = mode == pg::GEMM_GATEUP;
    if (mode < pg::GEMM_F32 || mode > pg::GEMM_GATEUP || !aq || !as || !bq || m < 1 || n < 1 || k < 1 || k % 32) return B200_ERR_BAD_ARG;
    if (gateup ? (!bq2 || !hq || !hs || n % 32) : (!c || n % pg::I8_BN)) return B200_ERR_BAD_ARG;
    const int nseg = smv_pick_nseg(k);
    if (!nseg || (k / nseg) % pg::BK) return B200_ERR_BAD_ARG;
    const int seg = k / nseg, unit = smv_unit_bytes(seg), rows = gateup ? 2 * n : n, mpad = (m + pg::BM - 1) / pg::BM * pg::BM;
    const int lds = pg::i8_lds(k), nb = k / 32;
    const size_t q8_bytes = (size_t)n * nb * 34, stream_bytes = (size_t)rows * nseg * unit;
    int8_t *daq = nullptr, *dhq = nullptr;
    float *das = nullptr, *dc = nullptr, *dhs = nullptr;
    unsigned char *draw = nullptr, *dstream = nullptr;
    Scratch s;
    // rows m .. mpad - 1 of A hold large quants and scales: a tile row past m_valid is computed but must never be stored
    if (s.alloc(&daq, (size_t)mpad * k) && s.alloc(&das, (size_t)mpad * lds * 4) && s.alloc(&draw, q8_bytes * (gateup ? 2 : 1)) &&
        s.alloc(&dstream, stream_bytes) && s.ok(cudaMemset(daq, 0x7F, (size_t)mpad * k)) && s.ok(cudaMemset(das, 0x7F, (size_t)mpad * lds * 4)) &&
        s.ok(cudaMemcpy(daq, aq, (size_t)m * k, cudaMemcpyHostToDevice)) &&
        s.ok(cudaMemcpy2D(das, (size_t)lds * 4, as, (size_t)nb * 4, (size_t)nb * 4, m, cudaMemcpyHostToDevice)) &&
        s.ok(cudaMemcpy(draw, bq, q8_bytes, cudaMemcpyHostToDevice)) && (!gateup || s.ok(cudaMemcpy(draw + q8_bytes, bq2, q8_bytes, cudaMemcpyHostToDevice))) &&
        (gateup ? s.alloc(&dhq, (size_t)m * n) && s.alloc(&dhs, (size_t)m * (n / 32) * 4) && s.ok(cudaMemcpy(dhq, hq, (size_t)m * n, cudaMemcpyHostToDevice)) &&
                      s.ok(cudaMemcpy(dhs, hs, (size_t)m * (n / 32) * 4, cudaMemcpyHostToDevice))
                : s.alloc(&dc, (size_t)m * n * 4) && s.ok(cudaMemcpy(dc, c, (size_t)m * n * 4, cudaMemcpyHostToDevice)))) {
        RepackSrc src{};
        src.raw[0] = draw;
        src.rows[0] = n;
        if (gateup) { src.raw[1] = draw + q8_bytes; src.rows[1] = n; }
        src.gateup = gateup ? 1 : 0;
        k_repack_tiles<<<(unsigned)((size_t)rows * nseg), 128>>>(src, dstream, rows, k, seg, nseg, unit);
        s.ok(cudaGetLastError());
        // the maps prefill_init_i8 builds
        CUtensorMap ma, ms, mq, mqs;
        if (s.rc == B200_OK && (pg::make_map_i8_a(&ma, daq, (uint64_t)mpad, (uint64_t)k) || pg::make_map_i8_s(&ms, das, (uint64_t)mpad, (uint64_t)lds) ||
                                pg::make_map_i8_q8(&mq, dstream, (uint64_t)rows, nseg, unit, 0) || pg::make_map_i8_q8(&mqs, dstream, (uint64_t)rows, nseg, unit, 1)))
            s.rc = B200_ERR_CUDA;
        if (s.rc == B200_OK) {
            pg::I8Out o{};
            o.C = dc; o.ldc = n; o.hq = dhq; o.hs = dhs; o.ldq = n; o.lds = n / 32;
            o.m_valid = m; o.K = k; o.seg = seg; o.oscale = oscale;
            const int lr = with_gemm_mode(mode, [&](auto MODE) { return pg::gemm_i8_launch<MODE>(ma, ms, mq, mqs, o, mpad / pg::BM, rows / pg::I8_BN, 0); });
            if (lr == -6) s.rc = B200_ERR_BAD_ARG;
            else if (lr) s.rc = B200_ERR_CUDA;
        }
        if (s.ok(cudaDeviceSynchronize()) && s.rc == B200_OK) {
            if (gateup) s.ok(cudaMemcpy(hq, dhq, (size_t)m * n, cudaMemcpyDeviceToHost)) && s.ok(cudaMemcpy(hs, dhs, (size_t)m * (n / 32) * 4, cudaMemcpyDeviceToHost));
            else s.ok(cudaMemcpy(c, dc, (size_t)m * n * 4, cudaMemcpyDeviceToHost));
        }
    }
    return s.rc;
}

int b200_test_gemm_i8_experts(int32_t mode, int32_t n_experts, const int32_t *counts, int32_t n, int32_t k, const int8_t *aq, const float *as,
                              const void *bq, const void *bq2, float *c, int8_t *hq, float *hs) {
    const bool gateup = mode == pg::GEMM_GATEUP;
    if ((mode != pg::GEMM_F32 && !gateup) || n_experts < 1 || n_experts > MOE_MAX_EXPERTS || !counts || !bq || n < 1 || k < 1 || k % 32) return B200_ERR_BAD_ARG;
    if (gateup ? (!bq2 || n % 32) : n % pg::I8_BN) return B200_ERR_BAD_ARG;
    const int E = n_experts;
    std::vector<int> off(E + 1, 0);
    for (int e = 0; e < E; e++) {
        if (counts[e] < 0) return B200_ERR_BAD_ARG;
        off[e + 1] = off[e] + counts[e];
    }
    const int m = off[E];
    if (m && (!aq || !as || (gateup ? !hq || !hs : !c))) return B200_ERR_BAD_ARG;
    const int nseg = smv_pick_nseg(k);
    if (!nseg || (k / nseg) % pg::BK) return B200_ERR_BAD_ARG;
    if (!m) return B200_OK;
    const int seg = k / nseg, unit = smv_unit_bytes(seg), rows = gateup ? 2 * n : n, ga = m + pg::BM; // a tile of the last rows reads up to BM past them
    const int lds = pg::i8_lds(k), nb = k / 32;
    const size_t q8_bytes = (size_t)n * nb * 34, stream_bytes = (size_t)rows * nseg * unit;
    std::vector<pg::XpTile> tiles(pg::xp_max_tiles(m, E));
    const int nt = pg::xp_tile_table(counts, off.data(), E, tiles.data());
    int8_t *daq = nullptr, *dhq = nullptr;
    float *das = nullptr, *dc = nullptr, *dhs = nullptr;
    unsigned char *draw = nullptr, *dstream = nullptr;
    CUtensorMap *dmaps = nullptr;
    pg::XpTile *dtiles = nullptr;
    int *dnt = nullptr;
    Scratch s;
    // rows m .. ga - 1 of A hold large quants and scales: a tile row past its expert's rows is computed but must never be stored
    if (s.alloc(&daq, (size_t)ga * k) && s.alloc(&das, (size_t)ga * lds * 4) && s.alloc(&draw, q8_bytes * (gateup ? 2 : 1)) &&
        s.alloc(&dstream, stream_bytes * E) && s.alloc(&dmaps, (size_t)E * 4 * sizeof(CUtensorMap)) && s.alloc(&dtiles, tiles.size() * sizeof(pg::XpTile)) &&
        s.alloc(&dnt, 4) && s.ok(cudaMemset(daq, 0x7F, (size_t)ga * k)) && s.ok(cudaMemset(das, 0x7F, (size_t)ga * lds * 4)) &&
        s.ok(cudaMemcpy(daq, aq, (size_t)m * k, cudaMemcpyHostToDevice)) &&
        s.ok(cudaMemcpy2D(das, (size_t)lds * 4, as, (size_t)nb * 4, (size_t)nb * 4, m, cudaMemcpyHostToDevice)) &&
        s.ok(cudaMemcpy(dtiles, tiles.data(), tiles.size() * sizeof(pg::XpTile), cudaMemcpyHostToDevice)) && s.ok(cudaMemcpy(dnt, &nt, 4, cudaMemcpyHostToDevice)) &&
        (gateup ? s.alloc(&dhq, (size_t)m * n) && s.alloc(&dhs, (size_t)m * (n / 32) * 4) && s.ok(cudaMemcpy(dhq, hq, (size_t)m * n, cudaMemcpyHostToDevice)) &&
                      s.ok(cudaMemcpy(dhs, hs, (size_t)m * (n / 32) * 4, cudaMemcpyHostToDevice))
                : s.alloc(&dc, (size_t)m * n * 4) && s.ok(cudaMemcpy(dc, c, (size_t)m * n * 4, cudaMemcpyHostToDevice)))) {
        // each expert's stream as the upload repacks it, and its quant / scale maps (entries 0 / 1 for GATEUP, 2 / 3 for STORE)
        std::vector<CUtensorMap> h((size_t)E * 4);
        for (int e = 0; e < E && s.rc == B200_OK; e++) {
            const unsigned char *src0 = static_cast<const unsigned char *>(bq) + (size_t)e * q8_bytes;
            if (!s.ok(cudaMemcpy(draw, src0, q8_bytes, cudaMemcpyHostToDevice)) ||
                (gateup && !s.ok(cudaMemcpy(draw + q8_bytes, static_cast<const unsigned char *>(bq2) + (size_t)e * q8_bytes, q8_bytes, cudaMemcpyHostToDevice))))
                break;
            RepackSrc src{};
            src.raw[0] = draw;
            src.rows[0] = n;
            if (gateup) { src.raw[1] = draw + q8_bytes; src.rows[1] = n; }
            src.gateup = gateup ? 1 : 0;
            unsigned char *dst = dstream + (size_t)e * stream_bytes;
            k_repack_tiles<<<(unsigned)((size_t)rows * nseg), 128>>>(src, dst, rows, k, seg, nseg, unit);
            if (!s.ok(cudaGetLastError()) || !s.ok(cudaDeviceSynchronize())) break; // draw is reused by the next expert
            CUtensorMap *mm = &h[(size_t)e * 4 + (gateup ? 0 : 2)];
            if (pg::make_map_i8_q8(mm, dst, (uint64_t)rows, nseg, unit, 0) || pg::make_map_i8_q8(mm + 1, dst, (uint64_t)rows, nseg, unit, 1)) s.rc = B200_ERR_CUDA;
        }
        CUtensorMap ma, ms;
        if (s.rc == B200_OK && (pg::make_map_i8_a(&ma, daq, (uint64_t)ga, (uint64_t)k) || pg::make_map_i8_s(&ms, das, (uint64_t)ga, (uint64_t)lds)))
            s.rc = B200_ERR_CUDA;
        if (s.rc == B200_OK) s.ok(cudaMemcpy(dmaps, h.data(), h.size() * sizeof(CUtensorMap), cudaMemcpyHostToDevice));
        if (s.rc == B200_OK) {
            pg::I8Out o{};
            o.C = dc; o.ldc = n; o.hq = dhq; o.hs = dhs; o.ldq = n; o.lds = n / 32;
            o.K = k; o.seg = seg; o.oscale = 1.0f;
            const int gm = pg::xp_max_tiles(m, E), nn = rows / pg::I8_BN;
            const int lr = gateup ? pg::xp_gemm_launch<pg::GEMM_GATEUP>(ma, ms, dmaps, dtiles, dnt, o, gm, nn, 0)
                                  : pg::xp_gemm_launch<pg::GEMM_F32>(ma, ms, dmaps, dtiles, dnt, o, gm, nn, 0);
            if (lr == -6) s.rc = B200_ERR_BAD_ARG;
            else if (lr) s.rc = B200_ERR_CUDA;
        }
        if (s.ok(cudaDeviceSynchronize()) && s.rc == B200_OK) {
            if (gateup) s.ok(cudaMemcpy(hq, dhq, (size_t)m * n, cudaMemcpyDeviceToHost)) && s.ok(cudaMemcpy(hs, dhs, (size_t)m * (n / 32) * 4, cudaMemcpyDeviceToHost));
            else s.ok(cudaMemcpy(c, dc, (size_t)m * n * 4, cudaMemcpyDeviceToHost));
        }
    }
    return s.rc;
}

} // extern "C"

namespace {
// What b200_test_stream launches, decided from its arguments alone (grid 0 with n_sms 0: the grid is not known yet).
struct StreamTest {
    TileMat W, Wd;   // Q8_0 / resident: the stream and, in pair mode, the down projection (bases unset)
    SmvSmem L, Ld;   // single-row layouts
    SmbSmem B;       // batched layout
    SfLayout F;      // F16 layout
    unsigned off_sq = 0, off_seq = 0;
    int stages = 0, grid = 0, gmax = 0, gmin = 0;
    size_t total = 0;
};

int stream_test_plan(const b200_stream_test &t, int n_sms, StreamTest &c) {
    const bool f16 = t.form == B200_GGML_F16, kq = kq_is_kquant(t.form), batch = t.nrow > 0, gateup = t.mode == SMV_GATEUP;
    const bool norm_in = t.norm && !t.from_emb;
    if (!f16 && !kq && t.form != B200_GGML_Q8_0) return B200_ERR_BAD_ARG;
    if (t.mode < SMV_STORE || t.mode > SMV_GATEUP || t.rows < 1 || t.cols < 32 || t.grid < 0 || t.stages < 0 || t.budget < 0) return B200_ERR_BAD_ARG;
    if (t.nrow < 0 || t.nrow > SMB_MAX_ROWS || (batch && (kq || f16 || t.norm))) return B200_ERR_BAD_ARG;
    if (t.launches != 1 && t.launches != 2) return B200_ERR_BAD_ARG;
    if (t.norm && (t.mode == SMV_RESID || f16 || !norm_fusion_ok(t.cols) || !t.norm_w)) return B200_ERR_BAD_ARG;
    if (t.from_emb && (!t.norm || !t.emb || !t.tokens || !t.x_out || t.emb_rows < 1)) return B200_ERR_BAD_ARG;
    for (int l = 0; t.from_emb && l < t.launches; l++)
        if (t.tokens[l] < 0 || t.tokens[l] >= t.emb_rows) return B200_ERR_BAD_ARG;
    if (t.argmax && (t.mode != SMV_STORE || !t.ids)) return B200_ERR_BAD_ARG;
    if (t.pair && (!gateup || batch || f16 || !t.w_down || t.down_rows < 1 || !t.out_init || !t.out_down)) return B200_ERR_BAD_ARG;
    if (!t.w || !t.out || (gateup && !t.w_up) || (gateup && !f16 && (!t.hq || !t.hs)) || (t.mode == SMV_RESID && !t.out_init)) return B200_ERR_BAD_ARG;
    if ((f16 || norm_in) ? !t.x : (!t.norm && (!t.xq || !t.xs))) return B200_ERR_BAD_ARG;
    if (f16) {
        c.F = sf_layout(t.rows, t.cols, t.lanes, gateup);
        if (!c.F.ok || t.budget) return B200_ERR_BAD_ARG;
        c.stages = t.stages ? t.stages : c.F.stages;
        if (c.stages < 3 || c.stages > SF_MAX_STAGES) return B200_ERR_BAD_ARG;
        const int rw = 64 / t.lanes, mr = gateup ? rw / 2 : rw, ngroups = (t.rows + mr - 1) / mr;
        c.total = (size_t)t.cols * 4 + SF_WARPS * SF_MAX_STAGES * 8 + 256 + (size_t)SF_WARPS * c.stages * ((size_t)rw * (c.F.seg * 2 + SF_ROW_PAD));
        c.grid = t.grid ? t.grid : n_sms ? sf_grid(n_sms, t.lanes, t.rows, t.cols, gateup) : 0;
        for (int b = 0; b < c.grid; b++) { // k_stream_matvec_f16's warp-interleaved assignment
            int g = 0;
            for (int w = 0; w < SF_WARPS; w++) {
                const int gw = w * c.grid + b, G = c.grid * SF_WARPS;
                g += gw < ngroups ? (ngroups - gw + G - 1) / G : 0;
            }
            c.gmax = b ? std::max(c.gmax, g) : g;
            c.gmin = b ? std::min(c.gmin, g) : g;
        }
        return B200_OK;
    }
    if (gateup && t.rows % 32) return B200_ERR_BAD_ARG; // whole 32-unit blocks of hq
    if (t.stages && (t.stages < 3 || t.stages > SMV_MAX_STAGES)) return B200_ERR_BAD_ARG;
    c.W = tile_geometry(gateup ? 2 * t.rows : t.rows, t.cols, kq ? t.form : 0);
    if (!c.W.nseg) return B200_ERR_BAD_ARG;
    if (batch) {
        const size_t budget = t.stages ? smb_layout(c.W.seg, t.nrow, 0).off_ring + (size_t)t.stages * smb_layout(c.W.seg, t.nrow, 0).stage_bytes
                              : t.budget ? (size_t)t.budget : SMB_SMEM_BUDGET;
        if (budget > SMB_SMEM_BUDGET) return B200_ERR_BAD_ARG; // the batched kernels are set up for at most this much
        c.B = smb_layout(c.W.seg, t.nrow, budget);
        c.stages = c.B.stages;
        c.total = c.B.total;
    } else {
        const int fmt = c.W.fmt;
        auto lay = [&](size_t b) { return t.norm ? smv_layout_norm(t.cols, c.W.seg, b, &c.off_sq, &c.off_seq, fmt) : smv_layout(t.cols, c.W.seg, b, fmt); };
        const SmvSmem L0 = lay(0);
        c.L = lay(t.stages ? L0.off_ring + (size_t)t.stages * L0.stage_bytes : t.budget ? (size_t)t.budget : SMV_SMEM_BUDGET_MAX);
        c.stages = c.L.stages;
        c.total = c.L.total;
        if (t.pair) {
            c.Wd = tile_geometry(t.down_rows, t.rows, fmt);
            if (!c.Wd.nseg) return B200_ERR_BAD_ARG;
            c.Ld = smv_layout(t.rows, c.Wd.seg, SMV_SMEM_BUDGET_MAX, fmt);
            if (c.Ld.stages < 3) return B200_ERR_BAD_ARG;
        }
    }
    if (c.stages < 3 || (t.stages && c.stages != t.stages)) return B200_ERR_BAD_ARG;
    c.grid = t.grid ? t.grid : n_sms;
    if (gateup && c.grid && !gateup_fits(t.rows, c.grid)) return B200_ERR_BAD_ARG;
    const int G = tile_groups(c.W);
    for (int b = 0; b < c.grid; b++) { // the kernels' static slice [g0, g1)
        const int g = (int)(((long long)(b + 1) * G) / c.grid - ((long long)b * G) / c.grid);
        c.gmax = b ? std::max(c.gmax, g) : g;
        c.gmin = b ? std::min(c.gmin, g) : g;
    }
    return B200_OK;
}

template <typename F> void with_stream_mode(int mode, F &&f) { // SMV_* and SF_* share their values
    if (mode == SMV_STORE) f(std::integral_constant<int, SMV_STORE>());
    else if (mode == SMV_RESID) f(std::integral_constant<int, SMV_RESID>());
    else f(std::integral_constant<int, SMV_GATEUP>());
}
} // namespace

extern "C" {

int b200_test_stream(b200_stream_test *t) {
    if (!t) return B200_ERR_BAD_ARG;
    StreamTest c;
    int rc = stream_test_plan(*t, 0, c);
    if (rc) return rc;
    auto report = [&] {
        const int64_t v[5] = {c.stages, c.grid, c.gmax, c.gmin, (int64_t)c.total};
        for (int k = 0; k < 5; k++) t->info[k] = v[k];
    };
    if (t->dry) {
        if (!t->grid) return B200_ERR_BAD_ARG;
        report();
        return B200_OK;
    }
    int dev = 0, n_sms = 0, optin = 0;
    Scratch s;
    if (!s.ok(cudaGetDevice(&dev)) || !s.ok(cudaDeviceGetAttribute(&n_sms, cudaDevAttrMultiProcessorCount, dev)) ||
        !s.ok(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev)))
        return s.rc;
    if ((rc = stream_test_plan(*t, n_sms, c))) return rc;
    if (c.total > (size_t)optin) return B200_ERR_BAD_ARG;
    report();

    const bool f16 = t->form == B200_GGML_F16, batch = t->nrow > 0, gateup = t->mode == SMV_GATEUP;
    const int V = batch ? t->nrow : 1, rows = t->rows, cols = t->cols, nb = cols / 32, fmt = f16 ? 0 : c.W.fmt;
    const size_t rb = f16 ? (size_t)cols * 2 : fmt ? (size_t)cols / 256 * kq_block_bytes(fmt) : (size_t)nb * 34;
    const size_t wbytes = (size_t)rows * rb, obytes = (size_t)V * rows * 4;
    TpCtx solo{};
    solo.n = 1;
    const TraceBuf none{nullptr, 0, 0};
    unsigned char *dw = nullptr, *dtile = nullptr, *dwd = nullptr, *dtd = nullptr;
    int8_t *dxq = nullptr, *dhq = nullptr, *dembq = nullptr;
    float *dxs = nullptr, *dx = nullptr, *dnw = nullptr, *dout = nullptr, *dhs = nullptr, *dres = nullptr, *dpv = nullptr;
    __half *dembs = nullptr;
    int *dpi = nullptr, *dids = nullptr;
    unsigned *dblk = nullptr;
    StepState *dst = nullptr;
    // the weights: raw rows (gate then up), repacked as upload_tiles repacks them
    // out ends in GUARD words that no store may reach (a padding row of a ragged STORE would land there)
    const int GUARD = 4;
    if (!s.alloc(&dw, wbytes * (gateup ? 2 : 1)) || !s.ok(cudaMemcpy(dw, t->w, wbytes, cudaMemcpyHostToDevice)) ||
        (gateup && !s.ok(cudaMemcpy(dw + wbytes, t->w_up, wbytes, cudaMemcpyHostToDevice))) || !s.alloc(&dout, obytes + GUARD * 4) ||
        !s.ok(cudaMemset(dout, 0xFF, obytes + GUARD * 4)) || (t->mode == SMV_RESID && !s.ok(cudaMemcpy(dout, t->out_init, obytes, cudaMemcpyHostToDevice))))
        return s.rc;
    auto repack = [&](const TileMat &W, const unsigned char *raw, int nrows, int ncols, bool gu, unsigned char **tiles) {
        RepackSrc src{};
        src.raw[0] = raw;
        src.rows[0] = nrows;
        if (gu) { src.raw[1] = raw + (size_t)nrows * rb; src.rows[1] = nrows; }
        src.gateup = gu ? 1 : 0;
        if (!s.alloc(tiles, (size_t)tile_bytes(W))) return false;
        const unsigned n = (unsigned)((size_t)tile_groups(W) * 4 * W.nseg);
        if (W.fmt) k_repack_kq_tiles<<<n, 128>>>(src, *tiles, W.rows, ncols, W.seg, W.nseg, W.unit_bytes, kq_block_bytes(W.fmt));
        else k_repack_tiles<<<n, 128>>>(src, *tiles, W.rows, ncols, W.seg, W.nseg, W.unit_bytes);
        return s.ok(cudaGetLastError());
    };
    if (!f16) {
        if (!repack(c.W, dw, rows, cols, gateup, &dtile)) return s.rc;
        c.W.base = dtile;
    }
    if (t->pair) {
        const size_t db = (size_t)t->down_rows * (fmt ? (size_t)rows / 256 * kq_block_bytes(fmt) : (size_t)rows / 32 * 34);
        if (!s.alloc(&dwd, db) || !s.ok(cudaMemcpy(dwd, t->w_down, db, cudaMemcpyHostToDevice)) || !repack(c.Wd, dwd, t->down_rows, rows, false, &dtd) ||
            !s.alloc(&dres, (size_t)t->down_rows * 4) || !s.ok(cudaMemcpy(dres, t->out_init, (size_t)t->down_rows * 4, cudaMemcpyHostToDevice)))
            return s.rc;
        c.Wd.base = dtd;
    }
    // activations, epilogue buffers, the step state and the argmax partials
    if (f16 || t->norm) {
        if (!s.alloc(&dx, (size_t)cols * 4)) return s.rc;
    } else if (!s.alloc(&dxq, (size_t)V * cols) || !s.alloc(&dxs, (size_t)V * nb * 4)) return s.rc;
    if (t->norm && (!s.alloc(&dnw, (size_t)cols * 4) || !s.ok(cudaMemcpy(dnw, t->norm_w, (size_t)cols * 4, cudaMemcpyHostToDevice)))) return s.rc;
    DevMat emb{};
    if (t->from_emb) { // the embedding as the plan keeps a Q8_0 one: quants and f16 scales in separate planes
        const size_t n = (size_t)t->emb_rows * cols;
        std::vector<int8_t> q(n);
        std::vector<uint16_t> sc(n / 32);
        const unsigned char *raw = (const unsigned char *)t->emb;
        for (size_t b = 0; b < n / 32; b++) {
            memcpy(&sc[b], raw + b * 34, 2);
            memcpy(&q[b * 32], raw + b * 34 + 2, 32);
        }
        if (!s.alloc(&dembq, n) || !s.alloc(&dembs, n / 32 * 2) || !s.ok(cudaMemcpy(dembq, q.data(), n, cudaMemcpyHostToDevice)) ||
            !s.ok(cudaMemcpy(dembs, sc.data(), n / 32 * 2, cudaMemcpyHostToDevice)))
            return s.rc;
        emb = DevMat{dembq, dembs, t->emb_rows, cols, B200_GGML_Q8_0};
    }
    if (gateup && !f16 &&
        (!s.alloc(&dhq, (size_t)V * rows) || !s.alloc(&dhs, (size_t)V * (rows / 32) * 4) || !s.alloc(&dblk, (size_t)V * (rows / 32) * 4) ||
         !s.ok(cudaMemset(dhq, 0x5A, (size_t)V * rows)) || !s.ok(cudaMemset(dhs, 0xFF, (size_t)V * (rows / 32) * 4)) ||
         !s.ok(cudaMemset(dblk, 0, (size_t)V * (rows / 32) * 4))))
        return s.rc;
    if (!s.alloc(&dst, sizeof(StepState))) return s.rc;
    if (t->argmax && (!s.alloc(&dpv, (size_t)V * c.grid * 4) || !s.alloc(&dpi, (size_t)V * c.grid * 4) || !s.alloc(&dids, (size_t)t->launches * V * 4)))
        return s.rc;

    // the shared-memory attributes set_smem_attrs gives every plan
    with_stream_mode(t->mode, [&](auto M) {
        constexpr int MODE = decltype(M)::value;
        if (f16) s.ok(t->lanes == 16 ? set_max_dyn(k_stream_matvec_f16<16, MODE>, optin) : set_max_dyn(k_stream_matvec_f16<8, MODE>, optin));
        else if (batch) s.ok(cudaFuncSetAttribute(k_stream_matvec_q8_batch<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMB_SMEM_BUDGET));
        else if (!t->norm) s.ok(set_max_dyn(smv_kernel<MODE>(fmt), optin));
        else if constexpr (MODE != SMV_RESID) s.ok(set_max_dyn(smv_norm_kernel<MODE>(fmt), optin));
    });
    if (t->pair) s.ok(set_max_dyn(smv_kernel<SMV_RESID>(fmt), optin));
    if (s.rc) return s.rc;

    for (int l = 0; l < t->launches; l++) {
        const StepState st{t->from_emb ? t->tokens[l] : 0, 0, l, 0, 0, {0, 0, 0}};
        if (!s.ok(cudaMemcpy(dst, &st, sizeof st, cudaMemcpyHostToDevice))) return s.rc;
        if (t->from_emb) {
            if (!s.ok(cudaMemset(dx, 0xFF, (size_t)cols * 4))) return s.rc;
        } else if (dx) {
            if (!s.ok(cudaMemcpy(dx, t->x + (size_t)l * cols, (size_t)cols * 4, cudaMemcpyHostToDevice))) return s.rc;
        } else if (!s.ok(cudaMemcpy(dxq, t->xq + (size_t)l * V * cols, (size_t)V * cols, cudaMemcpyHostToDevice)) ||
                   !s.ok(cudaMemcpy(dxs, t->xs + (size_t)l * V * nb, (size_t)V * nb * 4, cudaMemcpyHostToDevice)))
            return s.rc;
        with_stream_mode(t->mode, [&](auto M) {
            constexpr int MODE = decltype(M)::value;
            const dim3 grid(c.grid);
            if (f16) {
                SfArgs a{};
                a.w0 = (const __half *)dw; a.w1 = gateup ? (const __half *)(dw + wbytes) : nullptr; a.x = dx; a.out = dout; a.oscale = t->oscale;
                a.rows = rows; a.cols = cols; a.seg = c.F.seg; a.nseg = c.F.nseg; a.stages = c.stages; a.tr = none;
                a.part_val = dpv; a.part_idx = dpi;
                s.ok(t->lanes == 16 ? launch_on(0, true, k_stream_matvec_f16<16, MODE>, grid, dim3(SF_THREADS), c.total, a)
                                    : launch_on(0, true, k_stream_matvec_f16<8, MODE>, grid, dim3(SF_THREADS), c.total, a));
            } else if (batch) {
                SmbArgs a{};
                a.W = c.W; a.nrow = t->nrow; a.xq = dxq; a.xs = dxs; a.out = dout; a.oscale = t->oscale; a.ostride = rows; a.hq = dhq; a.hs = dhs;
                a.blk_cnt = dblk; a.part_val = dpv; a.part_idx = dpi;
                s.ok(launch_on(0, true, k_stream_matvec_q8_batch<MODE>, grid, dim3(SMV_THREADS), c.total, a, c.B));
            } else {
                SmvArgs a{};
                a.W = c.W; a.xq = dxq; a.xs = dxs; a.out = dout; a.oscale = t->oscale; a.hq = dhq; a.hs = dhs; a.blk_cnt = dblk;
                a.part_val = dpv; a.part_idx = dpi; a.tr = none; a.tp = solo; a.wait_slot = -1; a.out_slot = -1;
                if (!t->norm) s.ok(launch_on(0, true, smv_kernel<MODE>(fmt), grid, dim3(SMV_THREADS), c.total, a, c.L));
                else if constexpr (MODE != SMV_RESID) {
                    SmvNormArgs n{};
                    n.x = dx; n.w = dnw; n.st = dst; n.emb = emb; n.emb_scale = t->emb_scale; n.eps = t->eps; n.from_emb = t->from_emb ? 1 : 0;
                    n.x_out = dx; n.off_sq = c.off_sq; n.off_seq = c.off_seq;
                    s.ok(launch_on(0, true, smv_norm_kernel<MODE>(fmt), grid, dim3(SMV_THREADS), c.total, a, c.L, n));
                }
            }
        });
        if (t->pair && s.rc == B200_OK) { // W2 after gate/up, as the decode graph chains them
            SmvArgs a{};
            a.W = c.Wd; a.xq = dhq; a.xs = dhs; a.out = dres; a.oscale = t->oscale; a.tr = none; a.tp = solo; a.wait_slot = -1; a.out_slot = -1;
            s.ok(launch_on(0, true, smv_kernel<SMV_RESID>(fmt), dim3(c.grid), dim3(SMV_THREADS), c.Ld.total, a, c.Ld));
        }
        if (t->argmax && s.rc == B200_OK) {
            if (batch) s.ok(launch_on(0, true, k_argmax_batch, dim3(V), dim3(32), (size_t)0, (const float *)dpv, (const int *)dpi, c.grid, dids + (size_t)l * V));
            else
                s.ok(launch_on(0, true, k_argmax_advance, dim3(1), dim3(1024), (size_t)0, (const float *)dout, rows, dst, (const int *)nullptr, dids, 1,
                               (const float *)dpv, (const int *)dpi, c.grid, none, solo, -1));
        }
        unsigned guard[GUARD];
        if (!s.ok(cudaGetLastError()) || !s.ok(cudaDeviceSynchronize()) ||
            !s.ok(cudaMemcpy(t->out + (size_t)l * V * rows, dout, obytes, cudaMemcpyDeviceToHost)) ||
            !s.ok(cudaMemcpy(guard, (const unsigned char *)dout + obytes, sizeof guard, cudaMemcpyDeviceToHost)))
            return s.rc;
        for (unsigned g : guard)
            if (g != 0xFFFFFFFFu) return B200_ERR_STATE;
        if (dhq && (!s.ok(cudaMemcpy(t->hq + (size_t)l * V * rows, dhq, (size_t)V * rows, cudaMemcpyDeviceToHost)) ||
                    !s.ok(cudaMemcpy(t->hs + (size_t)l * V * (rows / 32), dhs, (size_t)V * (rows / 32) * 4, cudaMemcpyDeviceToHost))))
            return s.rc;
        if (t->pair && !s.ok(cudaMemcpy(t->out_down + (size_t)l * t->down_rows, dres, (size_t)t->down_rows * 4, cudaMemcpyDeviceToHost))) return s.rc;
        if (t->from_emb && !s.ok(cudaMemcpy(t->x_out + (size_t)l * cols, dx, (size_t)cols * 4, cudaMemcpyDeviceToHost))) return s.rc;
        if (t->argmax && !s.ok(cudaMemcpy(t->ids + (size_t)l * V, batch ? dids + (size_t)l * V : dids + l, (size_t)V * 4, cudaMemcpyDeviceToHost))) return s.rc;
    }
    return s.rc;
}

} // extern "C"

namespace {
// What b200_test_attention launches, decided from its arguments alone.
struct AttTest {
    int qd = 0, kvd = 0, nqkv = 0, grid_y = 0, launches = 0;
    bool global = false;   // score rows in a global scratch (the plan's rule: 3 * head size + context > ATT_SMEM_FLOATS_MAX)
    size_t smem = 0;       // dynamic shared memory of the attention launch
    size_t scratch = 0;    // floats of that scratch, as the plan sizes it for the form
    PdSmem L{};            // persistent form: the offsets pd_attention_head uses
};

int att_test_plan(const b200_attention_test &t, AttTest &c) {
    const int f = t.form, hs = t.head_size;
    if (f < B200_ATT_SINGLE || f > B200_ATT_PERSISTENT) return B200_ERR_BAD_ARG;
    const bool pers = f == B200_ATT_PERSISTENT;
    if (pers ? hs != 64 && hs != 128 : hs != 32 && hs != 64 && hs != 96 && hs != 128 && hs != 256) return B200_ERR_BAD_ARG;
    if (t.n_heads < 1 || t.n_kv_heads < 1 || t.n_heads % t.n_kv_heads || t.ctx < 1 || t.slots < 1) return B200_ERR_BAD_ARG;
    if (t.arch & ~(KF_NEOX | KF_QKNORM | KF_QKVBIAS | KF_ATTSCALE)) return B200_ERR_BAD_ARG;
    const int max_rows = f == B200_ATT_BATCH || f == B200_ATT_CACHED_ROWS ? SMB_MAX_ROWS : f == B200_ATT_CHUNK ? 1 << 20 : 1;
    if (t.rows < 1 || t.rows > max_rows) return B200_ERR_BAD_ARG;
    if (f == B200_ATT_CHUNK ? t.att_tokens < 1 || t.att_tokens > t.rows : t.att_tokens != 0) return B200_ERR_BAD_ARG;
    if (!t.slot || !t.pos || !t.qkv || !t.k_cache || !t.v_cache || !t.rope_cr || !t.rope_ci || !t.qkv_out || !t.k_out || !t.v_out || !t.xq ||
        !t.xs || ((t.arch & KF_QKNORM) && (!t.q_norm || !t.k_norm)) || ((t.arch & KF_QKVBIAS) && !t.qkv_bias))
        return B200_ERR_BAD_ARG;
    for (int r = 0; r < t.rows; r++) {
        if (t.slot[r] < 0 || t.slot[r] >= t.slots || t.pos[r] < 0 || t.pos[r] >= t.ctx) return B200_ERR_BAD_ARG;
        for (int q = 0; q < r; q++) // a batch row writes its K / V inside its attention CTAs: one slot per row; no two rows write one cache row
            if (t.slot[q] == t.slot[r] && (f == B200_ATT_BATCH || t.pos[q] == t.pos[r])) return B200_ERR_BAD_ARG;
    }
    c.qd = t.n_heads * hs; c.kvd = t.n_kv_heads * hs; c.nqkv = c.qd + 2 * c.kvd;
    c.global = 3 * hs + t.ctx > ATT_SMEM_FLOATS_MAX;
    const int ctx_pad = (t.ctx + PD_CT - 1) / PD_CT * PD_CT; // the plan's scratch rows are padded for the persistent kernel
    c.grid_y = f == B200_ATT_CHUNK ? t.att_tokens : f == B200_ATT_BATCH || f == B200_ATT_CACHED_ROWS ? t.rows : 1;
    c.launches = f == B200_ATT_CHUNK ? (t.rows + t.att_tokens - 1) / t.att_tokens : 1;
    if (pers) {
        c.L = pd_layout(c.qd, c.qd, c.qd, hs, 3 * hs + (c.global ? 0 : ctx_pad), 32, 0); // no ring: the offsets before it
        c.smem = c.L.total;
        c.scratch = c.global ? (size_t)t.n_heads * ctx_pad : 0;
    } else {
        c.smem = att_smem_bytes(hs, t.ctx, c.global);
        c.scratch = !c.global ? 0 : f == B200_ATT_SINGLE ? (size_t)t.n_heads * ctx_pad : (size_t)c.grid_y * t.n_heads * t.ctx;
    }
    return B200_OK;
}
} // namespace

extern "C" {

int b200_test_attention(b200_attention_test *t) {
    if (!t) return B200_ERR_BAD_ARG;
    AttTest c;
    int rc = att_test_plan(*t, c);
    if (rc) return rc;
    const int64_t info[5] = {t->n_heads, c.grid_y, (int64_t)c.smem, c.global ? 1 : 0, c.launches};
    for (int k = 0; k < 5; k++) t->info[k] = info[k];
    if (t->dry) return B200_OK;
    int dev = 0, optin = 0;
    Scratch s;
    if (!s.ok(cudaGetDevice(&dev)) || !s.ok(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev))) return s.rc;
    if (c.smem > (size_t)optin) return B200_ERR_BAD_ARG;

    const int R = t->rows, hs = t->head_size, nh = t->n_heads, nkv = t->n_kv_heads, f = t->form;
    const size_t slot_stride = (size_t)t->ctx * c.kvd, cache = (size_t)t->slots * slot_stride, rope = (size_t)t->ctx * (hs / 2);
    const int lds = pg::i8_lds(c.qd); // the chunk form's block-scale row stride (the plan's XS rows)
    const size_t xs_rows = f == B200_ATT_CHUNK ? (size_t)lds : (size_t)c.qd / 32;
    // Every output sits between GUARD bytes of 0xA5 that no store may reach; outputs start as 0xFF bytes (xs, xb: NaN).
    const size_t GUARD = 256;
    std::vector<std::pair<unsigned char *, size_t>> guarded;
    auto buf = [&](auto **p, size_t bytes, const void *init) {
        unsigned char *d = nullptr;
        if (!s.alloc(&d, bytes + 2 * GUARD) || !s.ok(cudaMemset(d, 0xA5, bytes + 2 * GUARD)) ||
            !s.ok(init ? cudaMemcpy(d + GUARD, init, bytes, cudaMemcpyHostToDevice) : cudaMemset(d + GUARD, 0xFF, bytes)))
            return false;
        guarded.push_back({d, bytes});
        *p = reinterpret_cast<std::remove_pointer_t<decltype(p)>>(d + GUARD);
        return true;
    };
    float *dqkv = nullptr, *dk = nullptr, *dv = nullptr, *dxs = nullptr, *dxb = nullptr, *dcr = nullptr, *dci = nullptr, *dqn = nullptr, *dkn = nullptr;
    float *dbias = nullptr, *datt = nullptr;
    int8_t *dxq = nullptr;
    StepState *dst = nullptr;
    BatchRows *drows = nullptr;
    ChunkTok *dtok = nullptr;
    if (!buf(&dqkv, (size_t)R * c.nqkv * 4, t->qkv) || !buf(&dk, cache * 4, t->k_cache) || !buf(&dv, cache * 4, t->v_cache) ||
        !buf(&dxq, (size_t)R * c.qd, nullptr) || !buf(&dxs, (size_t)R * xs_rows * 4, nullptr) || (t->xb && !buf(&dxb, (size_t)c.qd * 4, nullptr)))
        return s.rc;
    if (!s.alloc(&dcr, rope * 4) || !s.alloc(&dci, rope * 4) || !s.ok(cudaMemcpy(dcr, t->rope_cr, rope * 4, cudaMemcpyHostToDevice)) ||
        !s.ok(cudaMemcpy(dci, t->rope_ci, rope * 4, cudaMemcpyHostToDevice)))
        return s.rc;
    if ((t->arch & KF_QKNORM) && (!s.alloc(&dqn, (size_t)hs * 4) || !s.alloc(&dkn, (size_t)hs * 4) ||
                                  !s.ok(cudaMemcpy(dqn, t->q_norm, (size_t)hs * 4, cudaMemcpyHostToDevice)) ||
                                  !s.ok(cudaMemcpy(dkn, t->k_norm, (size_t)hs * 4, cudaMemcpyHostToDevice))))
        return s.rc;
    if ((t->arch & KF_QKVBIAS) && (!s.alloc(&dbias, (size_t)c.nqkv * 4) || !s.ok(cudaMemcpy(dbias, t->qkv_bias, (size_t)c.nqkv * 4, cudaMemcpyHostToDevice))))
        return s.rc;
    if (c.scratch && (!s.alloc(&datt, c.scratch * 4) || !s.ok(cudaMemset(datt, 0xFF, c.scratch * 4)))) return s.rc;
    if (f == B200_ATT_SINGLE || f == B200_ATT_PERSISTENT) {
        const StepState st{0, t->pos[0], 0, 0, 0, {0, 0, 0}};
        if (!s.alloc(&dst, sizeof st) || !s.ok(cudaMemcpy(dst, &st, sizeof st, cudaMemcpyHostToDevice))) return s.rc;
    } else if (f == B200_ATT_CHUNK) {
        std::vector<ChunkTok> tab(R);
        for (int r = 0; r < R; r++) tab[r] = ChunkTok{0, t->pos[r], (long long)(t->slot[r] * slot_stride)};
        if (!s.alloc(&dtok, (size_t)R * sizeof(ChunkTok)) || !s.ok(cudaMemcpy(dtok, tab.data(), (size_t)R * sizeof(ChunkTok), cudaMemcpyHostToDevice)))
            return s.rc;
    } else {
        BatchRows br{};
        for (int r = 0; r < R; r++) { br.pos[r] = t->pos[r]; br.slot[r] = t->slot[r]; }
        if (!s.alloc(&drows, sizeof br) || !s.ok(cudaMemcpy(drows, &br, sizeof br, cudaMemcpyHostToDevice))) return s.rc;
    }

    const TraceBuf none{nullptr, 0, 0};
    TpCtx solo{};
    solo.n = 1;
    const float eps = t->eps, sa = t->score_arg;
    const int arch = t->arch, ctx = t->ctx;
    if (f == B200_ATT_PERSISTENT) {
        PdArgs a;
        memset(&a, 0, sizeof a);
        a.qd = c.qd; a.n_heads = nh; a.n_kv_heads = nkv; a.head_size = hs; a.arch = arch; a.ctx = ctx; a.eps = eps; a.sqrt_hs = sa;
        a.rope_cr = dcr; a.rope_ci = dci; a.qkv = dqkv; a.attq = dxq; a.atts = dxs; a.att_scratch = datt; a.tp.n = 1;
        PdLayer Ly;
        memset(&Ly, 0, sizeof Ly);
        Ly.q_norm = dqn; Ly.k_norm = dkn; Ly.qkv_bias = dbias;
        Ly.kc = dk + (size_t)t->slot[0] * slot_stride; Ly.vc = dv + (size_t)t->slot[0] * slot_stride;
        with_mma_head_size(nullptr, hs, [&](auto HS) {
            if (s.ok(cudaFuncSetAttribute(k_test_pd_attention<HS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c.smem)))
                k_test_pd_attention<HS><<<nh, PD_THREADS, c.smem>>>(a, c.L, Ly, t->pos[0]);
            return B200_OK;
        });
    } else {
        with_decode_head_size(nullptr, hs, [&](auto HS) { // the shared-memory attributes set_smem_attrs gives every plan, then the plan's launches
            const size_t sm = c.smem;
            if (f == B200_ATT_SINGLE) {
                float *kc = dk + (size_t)t->slot[0] * slot_stride, *vc = dv + (size_t)t->slot[0] * slot_stride;
                if (s.ok(set_max_dyn(k_attention<HS>, optin)))
                    s.ok(launch_on(0, true, k_attention<HS>, dim3(nh), dim3(ATT_THREADS), sm, dqkv, kc, vc, (const StepState *)dst, (const float *)dcr,
                                   (const float *)dci, nh, nkv, arch, (const float *)dqn, (const float *)dkn, (const float *)dbias, eps, sa, dxq, dxs, dxb,
                                   none, solo, 0u, 0, datt, ctx));
            } else if (f == B200_ATT_BATCH) {
                if (s.ok(set_max_dyn(k_attention_batch<HS>, optin)))
                    s.ok(launch_on(0, true, k_attention_batch<HS>, dim3(nh, R), dim3(ATT_THREADS), sm, dqkv, c.nqkv, dk, dv, slot_stride,
                                   (const BatchRows *)drows, (const float *)dcr, (const float *)dci, nh, nkv, arch, (const float *)dqn, (const float *)dkn,
                                   (const float *)dbias, eps, sa, dxq, dxs, datt, ctx, none, solo));
            } else if (f == B200_ATT_CACHED_ROWS) {
                if (s.ok(set_max_dyn(k_attention_cached_rows<HS>, optin)) &&
                    s.ok(launch_on(0, true, k_rope_kv_batch<HS>, dim3(nh, R), dim3(2 * HS), (size_t)0, dqkv, c.nqkv, dk, dv, slot_stride,
                                   (const BatchRows *)drows, (const float *)dcr, (const float *)dci, nh, nkv, arch, (const float *)dqn, (const float *)dkn,
                                   (const float *)dbias, eps)))
                    s.ok(launch_on(0, true, k_attention_cached_rows<HS>, dim3(nh, R), dim3(ATT_THREADS), sm, dqkv, c.nqkv, dk, dv, slot_stride,
                                   (const BatchRows *)drows, nh, nkv, arch, sa, dxq, dxs, datt, ctx, none, solo));
            } else if (s.ok(set_max_dyn(k_i8_attention<HS>, optin))) { // the chunk: enqueue_chunk_i8's two launches
                k_i8_rope_kv<HS><<<dim3(nh, R), 2 * HS, 0>>>(dqkv, c.nqkv, dk, dv, dtok, dcr, dci, nh, nkv, arch, dqn, dkn, dbias, eps);
                for (int v0 = 0; v0 < R; v0 += t->att_tokens)
                    k_i8_attention<HS><<<dim3(nh, R - v0 < t->att_tokens ? R - v0 : t->att_tokens), ATT_THREADS, sm>>>(
                        dqkv, c.nqkv, dk, dv, dtok, v0, nh, nkv, arch, sa, dxq, dxs, lds, datt, ctx, none, solo);
            }
            return B200_OK;
        });
    }
    if (s.rc || !s.ok(cudaGetLastError()) || !s.ok(cudaDeviceSynchronize())) return s.rc;
    if (!s.ok(cudaMemcpy(t->qkv_out, dqkv, (size_t)R * c.nqkv * 4, cudaMemcpyDeviceToHost)) || !s.ok(cudaMemcpy(t->k_out, dk, cache * 4, cudaMemcpyDeviceToHost)) ||
        !s.ok(cudaMemcpy(t->v_out, dv, cache * 4, cudaMemcpyDeviceToHost)) || !s.ok(cudaMemcpy(t->xq, dxq, (size_t)R * c.qd, cudaMemcpyDeviceToHost)) ||
        !s.ok(cudaMemcpy2D(t->xs, (size_t)c.qd / 32 * 4, dxs, xs_rows * 4, (size_t)c.qd / 32 * 4, R, cudaMemcpyDeviceToHost)) ||
        (t->xb && !s.ok(cudaMemcpy(t->xb, dxb, (size_t)c.qd * 4, cudaMemcpyDeviceToHost))))
        return s.rc;
    std::vector<unsigned char> g(GUARD);
    for (const auto &b : guarded)
        for (size_t off : {(size_t)0, GUARD + b.second}) {
            if (!s.ok(cudaMemcpy(g.data(), b.first + off, GUARD, cudaMemcpyDeviceToHost))) return s.rc;
            for (unsigned char x : g)
                if (x != 0xA5) return B200_ERR_STATE;
        }
    return B200_OK;
}

int b200_test_exp(uint32_t first, int64_t n, float *e, float *e1) {
    if (!e || !e1 || n < 1 || n > ((int64_t)1 << 31) || (uint64_t)first + (uint64_t)n - 1 > 0xFFFFFFFFull) return B200_ERR_BAD_ARG;
    Scratch s;
    float *de = nullptr, *de1 = nullptr;
    if (!s.alloc(&de, (size_t)n * 4) || !s.alloc(&de1, (size_t)n * 4)) return s.rc;
    k_test_exp<<<(unsigned)std::min<int64_t>((n + 255) / 256, 65536), 256>>>(first, (unsigned)n, de, de1);
    if (s.ok(cudaGetLastError()) && s.ok(cudaMemcpy(e, de, (size_t)n * 4, cudaMemcpyDeviceToHost))) s.ok(cudaMemcpy(e1, de1, (size_t)n * 4, cudaMemcpyDeviceToHost));
    return s.rc;
}

int b200_test_pf_attention_packed(int32_t n_seqs, const int32_t *lengths, const int32_t *start_positions, const float *q, const float *k, const float *v,
                                  int32_t n_heads, int32_t n_kv_heads, int32_t head_size, int32_t out_rows, uint16_t *out) {
    if (!lengths || !start_positions || !q || !k || !v || !out || n_seqs < 1 || n_kv_heads < 1 || n_heads % n_kv_heads) return B200_ERR_BAD_ARG;
    const int kv_mul = n_heads / n_kv_heads, hs = head_size;
    if ((hs != 64 && hs != 128) || kv_mul > 64) return B200_ERR_BAD_ARG; // what prefill_why accepts for tensor_core
    const int qd = n_heads * hs, kvd = n_kv_heads * hs, ldq = qd + 2 * kvd;
    std::vector<int> row0(n_seqs), hrow(n_seqs);
    int n = 0, rows = 0;
    for (int i = 0; i < n_seqs; i++) {
        if (lengths[i] < 1 || start_positions[i] < 0) return B200_ERR_BAD_ARG;
        row0[i] = n; hrow[i] = rows;
        n += lengths[i]; rows += start_positions[i] + lengths[i];
    }
    if (out_rows < n) return B200_ERR_BAD_ARG;
    const std::vector<PfTile> tiles = pf_tiles(n_seqs, lengths, start_positions, row0.data(), hrow.data(), kv_mul);
    const PfHist hist{0, rows, 0}; // every K / V row, in place
    const size_t kv_elems = (size_t)rows * kvd;
    float *dqkv = nullptr, *dk = nullptr, *dv = nullptr;
    __half *dkh = nullptr, *dvh = nullptr, *dout = nullptr;
    PfTile *dt = nullptr;
    PfHist *dh = nullptr;
    Scratch s;
    // q rows of every sequence back to back in the q columns of QKV rows (as after k_pf_rope_kv_packed; the k / v columns hold NaN,
    // which the kernel must never read), K / V rows [0, start + n) of each sequence back to back: the layout a chunk gives the kernel
    if (s.alloc(&dqkv, (size_t)n * ldq * 4) && s.alloc(&dk, kv_elems * 4) && s.alloc(&dv, kv_elems * 4) &&
        s.alloc(&dkh, kv_elems * 2) && s.alloc(&dvh, kv_elems * 2) && s.alloc(&dout, (size_t)out_rows * qd * 2) &&
        s.alloc(&dt, tiles.size() * sizeof(PfTile)) && s.alloc(&dh, sizeof(PfHist)) &&
        s.ok(cudaMemset(dqkv, 0xFF, (size_t)n * ldq * 4)) && s.ok(cudaMemcpy2D(dqkv, (size_t)ldq * 4, q, (size_t)qd * 4, (size_t)qd * 4, n, cudaMemcpyHostToDevice)) &&
        s.ok(cudaMemcpy(dk, k, kv_elems * 4, cudaMemcpyHostToDevice)) && s.ok(cudaMemcpy(dv, v, kv_elems * 4, cudaMemcpyHostToDevice)) &&
        s.ok(cudaMemcpy(dout, out, (size_t)out_rows * qd * 2, cudaMemcpyHostToDevice)) &&
        s.ok(cudaMemcpy(dt, tiles.data(), tiles.size() * sizeof(PfTile), cudaMemcpyHostToDevice)) && s.ok(cudaMemcpy(dh, &hist, sizeof(PfHist), cudaMemcpyHostToDevice))) {
        const float inv_sqrt_hs = (float)(1.0 / sqrt((double)hs));
        const dim3 ag((unsigned)tiles.size(), n_kv_heads);
        // f16 K / V copies as a chunk makes them (k_pf_kv_to_f16_packed and k_pf_rope_kv_packed round the same way)
        const size_t n4 = kv_elems / 4;
        k_pf_kv_to_f16_packed<<<(unsigned)((n4 + 255) / 256 < 1184 ? (n4 + 255) / 256 : 1184), 256, 0, 0>>>(dk, dv, 0, dkh, dvh, kvd, dh);
        with_mma_head_size(nullptr, hs, [&](auto HS) {
            if (s.ok(cudaFuncSetAttribute(k_pf_attention_mma_packed<HS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pm_smem_bytes<HS>())))
                k_pf_attention_mma_packed<HS><<<ag, PM_THREADS, pm_smem_bytes<HS>(), 0>>>(dqkv, ldq, dkh, dvh, kvd, kv_mul, dt, inv_sqrt_hs, dout, qd);
            return B200_OK;
        });
        if (s.ok(cudaGetLastError()) && s.ok(cudaDeviceSynchronize())) s.ok(cudaMemcpy(out, dout, (size_t)out_rows * qd * 2, cudaMemcpyDeviceToHost));
    }
    return s.rc;
}

int b200_weight_info(b200_plan *p, int32_t *resident, int64_t *weight_bytes, int64_t *q8_weight_bytes) {
    if (!p) return B200_ERR_BAD_ARG;
    if (resident) *resident = p->resident ? 1 : 0;
    if (weight_bytes) *weight_bytes = p->w_bytes;
    if (q8_weight_bytes) *q8_weight_bytes = p->w8_bytes;
    return B200_OK;
}

int b200_stream_rings(const int32_t *shape, const int64_t *dev, int64_t *out) {
    if (!shape || !dev || !out) return B200_ERR_BAD_ARG;
    const int dim = shape[0], qd = shape[1], kvd = shape[2], hidden = shape[3], n_sms = shape[4];
    if (dim <= 0 || qd <= 0 || kvd <= 0 || hidden <= 0 || n_sms <= 0) return B200_ERR_BAD_ARG;
    for (int k = 0; k < 4; k++) {
        const int f = shape[6 + k];
        if (f != 0 && !kq_is_kquant(f)) return B200_ERR_BAD_ARG;
    }
    LayerW L;
    L.tqkv = tile_geometry(qd + 2 * kvd, dim, shape[6]);
    L.two = tile_geometry(dim, qd, shape[7]);
    L.tgu = tile_geometry(2 * hidden, dim, shape[8]);
    L.tw2 = tile_geometry(dim, hidden, shape[9]);
    const TileMat *ms[4] = {&L.tqkv, &L.two, &L.tgu, &L.tw2};
    for (const TileMat *m : ms)
        if (!m->nseg) return B200_ERR_UNSUPPORTED;
    const bool norm = shape[5] != 0;
    ring_budgets(SmDev{(size_t)dev[0], (size_t)dev[1], (size_t)dev[2]}, n_sms, norm, (size_t)dev[3], L, L);
    const size_t budgets[4] = {L.ring_qkv, SMV_SMEM_BUDGET_MAX, L.ring_gu, SMV_SMEM_BUDGET_MAX};
    const bool norms[4] = {norm, false, norm, false};
    for (int k = 0; k < 4; k++) {
        const TileMat &W = *ms[k];
        unsigned a, b;
        const SmvSmem S = norms[k] ? smv_layout_norm(W.cols, W.seg, budgets[k], &a, &b, W.fmt) : smv_layout(W.cols, W.seg, budgets[k], W.fmt);
        out[4 * k + 0] = (int64_t)S.total;
        out[4 * k + 1] = S.stages;
        out[4 * k + 2] = S.stage_bytes;
        out[4 * k + 3] = slice_tiles(W, n_sms);
    }
    return B200_OK;
}

int b200_test_set_memory_budget(int64_t bytes) {
    if (bytes < 0) return B200_ERR_BAD_ARG;
    g_memory_budget = bytes;
    return B200_OK;
}

int b200_upload_info(b200_plan *p, double *seconds, double *host_copy_seconds, int64_t *h2d_bytes) {
    if (!p) return B200_ERR_BAD_ARG;
    if (seconds) *seconds = p->up.total_s;
    if (host_copy_seconds) *host_copy_seconds = p->up.host_copy_s;
    if (h2d_bytes) *h2d_bytes = p->up.h2d_bytes;
    return B200_OK;
}

int b200_launches_per_decode(b200_plan *p) {
    if (!p) return 0;
    return active_graphs(p).decode.launches;
}
int64_t b200_device_bytes(b200_plan *p) { return p ? p->bytes : 0; }

void b200_plan_free(b200_plan *p) {
    if (!p) return;
    cudaSetDevice(p->device);
    if (p->stream) cudaStreamSynchronize(p->stream);
    prefill_free(p->prefill);
    batch_free(p);
    destroy(p->graph);
    destroy(p->pers);
    if (p->h_err) cudaFreeHost(p->h_err);
    for (int k = 0; k < TP_MAX; k++) if (p->peer_open[k]) cudaIpcCloseMemHandle(p->peer_open[k]);
    for (void *d : p->allocs) cudaFree(d);
    if (p->h_st) cudaFreeHost(p->h_st);
    if (p->h_ids) cudaFreeHost(p->h_ids);
    if (p->lp.h_out) cudaFreeHost(p->lp.h_out);
    if (p->ev0) cudaEventDestroy(p->ev0);
    if (p->ev1) cudaEventDestroy(p->ev1);
    if (p->stream) cudaStreamDestroy(p->stream);
    delete p;
}

const char *b200_last_error(b200_plan *p) { return p ? p->err.c_str() : "null plan"; }
const char *b200_version(void) { return "b200llama 0.1 sm_90a"; }

} // extern "C"
