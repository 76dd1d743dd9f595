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

#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <chrono>
#include <string>
#include <thread>
#include <utility>
#include <vector>

namespace {

struct LayerW {
    DevMat qkv, wo, w1, w3, w2;
    TileMat tqkv{}, two{}, tgu{}, tw2{}; // tile-major copies for the streaming kernel (Q8_0)
    float *attn_norm = nullptr, *ffn_norm = nullptr, *q_norm = nullptr, *k_norm = nullptr;
    float *qkv_bias = nullptr; // Qwen2: this rank's q|k|v bias, laid out like the packed q|k|v vector
    // Qwen2-MoE (moe.cuh): the shared expert's streams, the routed experts' geometry and the device tables of their stream bases
    TileMat sgu{}, sdn{}, xgu{}, xdn{};
    const unsigned char **gu_bases = nullptr, **dn_bases = nullptr;
    float *router = nullptr, *shared_gate = nullptr; // F32 [n_experts][dim] and [dim]
};

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
    bool use_stream = false, use_pdl = false;
    bool fuse_norm = false; // single-GPU Q8_0 streams: QKV, gate/up and lm_head compute their RMSNorm themselves (k_stream_matvec_q8_norm)
    int kflags = 0; // KF_* (common.cuh): what the attention prologues do for this architecture
    size_t kq_off = 0; // K-quant files: offset of the raw (K-quant bytes) area inside each staging buffer; 0 = no K-quant tensor in the file
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
    int *h_ids = nullptr;      // pinned, seq_cap

    cudaGraphExec_t g_decode = nullptr, g_prefill = nullptr, g_trace = nullptr; // the multi-kernel decode graph (round 1)
    cudaGraphExec_t g_pdecode = nullptr, g_pprefill = nullptr, g_ptrace = nullptr; // one persistent kernel per token (decode_persistent.cuh)
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
    int launches_decode = 0, launches_prefill = 0;
    float prefill_ms = 0.f; // device time of the last tensor-core prefill chunk
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;

    // Qwen2-MoE: the routing buffers [layer][k] ids and [layer][k + 1] weights of the last step, the router logits scratch and
    // arrival counters, the down projection's shared-memory layout
    bool is_moe = false;
    b200_moe_config moe{};
    int moe_hv = 0; // units of the virtual hidden vector: shared_hidden_dim + n_experts_used * expert_hidden_dim
    int *moe_ids = nullptr;
    float *moe_w = nullptr, *moe_logits = nullptr;
    unsigned *moe_done = nullptr;
    MoeDownSmem moe_dl{};

    // Granite's µP scales (b200_plan_create_granite); 1.0f for every other family, where each multiply leaves its operand unchanged
    b200_granite_config mup{1.0f, 1.0f, 1.0f, 1.0f};

    PrefillCtx prefill;
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

    // batched decode (decode_batch.cuh): n_slots KV caches [slot][layer][ctx][kvDim] and per-row activations, one graph per row count
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
        int *h_out = nullptr;                         // pinned: ids [SMB_MAX_ROWS] then sampler outputs [SMB_MAX_ROWS][8]
        cudaGraphExec_t g[SMB_MAX_ROWS + 1] = {};
        int launches[SMB_MAX_ROWS + 1] = {};
        // exact b200_prefill_slots: the per-step rows of the call [context_length], the device step index, the step graphs without the
        // classifier (one per row count)
        BatchRows *sched = nullptr;
        int *step = nullptr;
        cudaGraphExec_t gp[SMB_MAX_ROWS + 1] = {};
        int launches_p[SMB_MAX_ROWS + 1] = {};
        // steps whose rows may share a sequence (k_rope_kv_batch + k_attention_cached_rows), captured on first use:
        // [target: 0 the decode slots, 1 the plan's own cache][0 schedule-driven without the classifier, 1 with it][rows]
        cudaGraphExec_t gs[2][2][SMB_MAX_ROWS + 1] = {};
        int launches_s[2][2][SMB_MAX_ROWS + 1] = {};
        int last_n = 0;
        float last_ms = 0.f;
    } bt;
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

// Upload up to three stacked GGUF Q8_0 matrices (or the gate/up pair) into tile-major layout.
int upload_tiles(b200_plan *p, const b200_tensor *t0, const b200_tensor *t1, const b200_tensor *t2, int r0, int r1, int r2, int cols,
                 bool gateup, TileMat &out, const int *row0 = nullptr, const int *full = nullptr) {
    const b200_tensor *ts[3] = {t0, t1, t2};
    int rs[3] = {r0, r1, r2};
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
        const size_t row_bytes = (size_t)cols / 32 * 34, nbytes = (size_t)rs[k] * row_bytes;
        if (off + nbytes > q8_area) return fail(p, B200_ERR_STATE, "staging buffer too small");
        if (kq) { // the K-quant bytes land in the raw area; the Q8_0 blocks are produced on the device once the copies are in
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
    const int rows = gateup ? r0 + r1 : r0 + r1 + r2;
    out.rows = rows;
    out.cols = cols;
    out.nseg = smv_pick_nseg(cols);
    out.seg = cols / out.nseg;
    out.unit_bytes = smv_unit_bytes(out.seg);
    const size_t stored_rows = (size_t)tile_groups(out) * 4; // whole 4-row groups: a ragged classifier gets zero padding rows
    size_t total = stored_rows * out.nseg * out.unit_bytes;
    unsigned char *d;
    rc = dalloc(p, &d, total);
    if (rc) return rc;
    out.base = d;
    k_repack_tiles<<<(unsigned)(stored_rows * out.nseg), 128, 0, p->stream>>>(src, d, rows, cols, out.seg, out.nseg, out.unit_bytes);
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

template <int MODE> int launch_matvec_q8(b200_plan *p, const DevMat &m, const int8_t *xq, const float *xs, float *out) {
    int R = (m.rows % 4 == 0 && m.rows >= 32768) ? 4 : (m.rows % 2 == 0 ? 2 : 1);
    int warps = m.rows / R;
    int ctas = (warps + 7) / 8;
    size_t smem = q8_smem_bytes(m.cols, R, 8);
    const int8_t *qs = (const int8_t *)m.qs;
    const float os = out_scale(p, MODE == MODE_RESID, &m == &p->out);
    if (R == 4) k_matvec_q8<4, MODE><<<ctas, 256, smem, p->stream>>>(qs, m.sc, xq, xs, m.rows, m.cols, out, os);
    else if (R == 2) k_matvec_q8<2, MODE><<<ctas, 256, smem, p->stream>>>(qs, m.sc, xq, xs, m.rows, m.cols, out, os);
    else k_matvec_q8<1, MODE><<<ctas, 256, smem, p->stream>>>(qs, m.sc, xq, xs, m.rows, m.cols, out, os);
    CK(cudaGetLastError());
    return B200_OK;
}

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
int sf_grid(const b200_plan *p, int rows, int cols, bool gateup) { // CTAs of an FP16 streaming launch
    const int lanes = p->cfg.fp16_lanes;
    const SfLayout L = sf_layout(rows, cols, lanes, gateup);
    const int rw = 64 / lanes, mr = gateup ? rw / 2 : rw;
    const int grid = L.ctas_per_sm * p->n_sms;
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
    const int grid = sf_grid(p, m.rows, m.cols, MODE == SF_GATEUP);
    if (lanes == 16) return launch_k(p, p->use_pdl, k_stream_matvec_f16<16, MODE>, dim3(grid), dim3(SF_THREADS), L.total, a);
    return launch_k(p, p->use_pdl, k_stream_matvec_f16<8, MODE>, dim3(grid), dim3(SF_THREADS), L.total, a);
}

// Kernel launch with the programmatic-dependent-launch attribute (captured into the CUDA graph as
// a programmatic edge): the kernel may become resident while its predecessor is still running.
template <typename... KA, typename... A>
int launch_k(b200_plan *p, bool pdl, void (*kern)(KA...), dim3 grid, dim3 block, size_t smem, A... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = p->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    CK(cudaLaunchKernelEx(&cfg, kern, static_cast<KA>(args)...));
    return B200_OK;
}

const size_t SMV_SMEM_BUDGET_MAX = 96 * 1024;
// Read ONCE per plan (b200_plan_create), never inside a launch helper.
void read_knobs(b200_plan *p) {
    const char *d = getenv("B200_DECODE");
    // default: the CUDA graph, which every plan can run (on one H100, with the fused norm, it measured ~2.5 % faster than the persistent kernel for 8B Q8_0, DESIGN.md section 6).  B200_DECODE=persistent or b200_set_decode_mode select the one-kernel-per-token path.
    p->decode_mode = (d && !strcmp(d, "persistent")) ? B200_DECODE_PERSISTENT : B200_DECODE_GRAPH;
}

template <int MODE>
int launch_stream(b200_plan *p, const TileMat &W, const int8_t *xq, const float *xs, float *out, int8_t *hq, float *hs, bool argmax = false,
                  TraceBuf tr = TraceBuf{nullptr, 0, 0}, int wait_slot = -1, unsigned wait_op = 0, int out_slot = -1, unsigned out_op = 0,
                  int row_base = 0) {
    SmvSmem L = smv_layout(W.cols, W.seg, SMV_SMEM_BUDGET_MAX);
    SmvArgs a;
    a.W = W; a.xq = xq; a.xs = xs; a.out = out; a.hq = hq; a.hs = hs; a.blk_cnt = p->blk_cnt;
    a.oscale = out_scale(p, MODE == SMV_RESID, &W == &p->tout);
    a.part_val = argmax ? p->part_val : nullptr;
    a.part_idx = argmax ? p->part_idx : nullptr;
    a.tr = tr;
    a.tp = p->tp;
    a.wait_slot = wait_slot; a.wait_op = wait_op; a.out_slot = out_slot; a.out_op = out_op; a.row_base = row_base;
    return launch_k(p, p->use_pdl, k_stream_matvec_q8<MODE>, dim3(p->n_sms), dim3(SMV_THREADS), L.total, a, L);
}

// A stream kernel behind a fused RMSNorm of the residual stream x (weights w; from_emb: layer 0, the embedding row, which CTA 0
// also writes to x).  MODE is SMV_STORE (QKV, lm_head) or SMV_GATEUP.
template <int MODE>
int launch_stream_norm(b200_plan *p, const TileMat &W, const float *w, bool from_emb, float *out, int8_t *hq, float *hs, bool argmax, TraceBuf tr, int row_base = 0) {
    SmvNormArgs n;
    const SmvSmem L = smv_layout_norm(W.cols, W.seg, SMV_SMEM_BUDGET_MAX, &n.off_sq, &n.off_seq);
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
    return launch_k(p, p->use_pdl, k_stream_matvec_q8_norm<MODE>, dim3(p->n_sms), dim3(SMV_THREADS), L.total, a, L, n);
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

// The FFN half of a Qwen2-MoE layer (moe.cuh): the FFN norm (float xb for the F32 router, xq/xs for the experts), the router,
// the shared + routed gate/up stream and the down streams with the ordered combine.  Four launches, all under PDL; `tr` is the
// norm's trace record, the three MoE kernels take the next three (trace ids 10, 11, 12).
int enqueue_moe_ffn(b200_plan *p, int l, TraceBuf tr) {
    const b200_config &c = p->cfg;
    const LayerW &L = p->layers[l];
    const int E = p->moe.n_experts, k = p->moe.n_experts_used;
    int rc;
    if ((rc = launch_k(p, p->use_pdl, k_rmsnorm_quant<false>, dim3(1), dim3(NORM_THREADS), norm_smem_bytes(c.dim), p->x, (const StepState *)p->st, p->emb,
                       p->mup.embedding_scale, (const float *)L.ffn_norm, c.rms_norm_eps, c.dim, p->xq, p->xs, p->xb, (long long *)nullptr, tr, p->tp, -1)))
        return rc;
    int *ids = p->moe_ids + (size_t)l * k;
    float *w = p->moe_w + (size_t)l * (k + 1);
    MoeRouteArgs ra;
    ra.router = L.router; ra.shared_gate = L.shared_gate; ra.xb = p->xb; ra.logits = p->moe_logits + (size_t)l * (E + 1); ra.done = p->moe_done + l;
    ra.ids = ids; ra.weights = w; ra.dim = c.dim; ra.n_experts = E; ra.k = k; ra.tr = TraceBuf{tr.rec, tr.slot + 1, 10};
    if ((rc = launch_k(p, p->use_pdl, k_moe_route, dim3(E + 1), dim3(MOE_ROUTE_THREADS), (size_t)c.dim * 4, ra))) return rc;
    MoeStreamArgs a;
    a.S = L.sgu; a.X = L.xgu; a.bases = L.gu_bases; a.ids = ids; a.weights = w; a.k = k;
    a.xq = p->xq; a.xs = p->xs; a.out = p->hb; a.hq = p->hq; a.hs = p->hs; a.blk_cnt = p->blk_cnt; a.tr = TraceBuf{tr.rec, tr.slot + 2, 11};
    const SmvSmem GL = smv_layout(c.dim, L.sgu.seg, SMV_SMEM_BUDGET_MAX);
    if ((rc = launch_k(p, p->use_pdl, k_moe_gateup, dim3(p->n_sms), dim3(SMV_THREADS), GL.total, a, GL))) return rc;
    a.S = L.sdn; a.X = L.xdn; a.bases = L.dn_bases;
    a.xq = p->hq; a.xs = p->hs; a.out = p->x; a.hq = nullptr; a.hs = nullptr; a.blk_cnt = nullptr; a.tr = TraceBuf{tr.rec, tr.slot + 3, 12};
    return launch_k(p, p->use_pdl, k_moe_down, dim3(p->n_sms), dim3(SMV_THREADS), p->moe_dl.total, a, p->moe_dl);
}

// Enqueue one single-token forward on p->stream (captured into a CUDA graph at creation).
// with_logits=false is the prefill variant (InferenceCoreBatchPrefillDecode.java:166-167).
int enqueue_forward(b200_plan *p, bool with_logits, int *launches, bool trace = false) {
    const b200_config &c = p->cfg;
    const bool q8 = p->wtype == B200_GGML_Q8_0;
    const bool st = p->use_stream, pdl = p->use_pdl, sf = p->use_f16_stream;
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
        if (fz) rc = launch_stream_norm<SMV_STORE>(p, L.tqkv, L.attn_norm, l == 0, p->qkv, nullptr, nullptr, false, TR(2)); // attention norm + QKV
        else {
            if ((rc = norm(l == 0, L.attn_norm, l == 0 ? -1 : 4 * (l - 1) + 3))) return rc;
            n++;
            if (st) rc = launch_stream<SMV_STORE>(p, L.tqkv, p->xq, p->xs, p->qkv, nullptr, nullptr, false, TR(2));
            else if (q8) rc = launch_matvec_q8<MODE_STORE>(p, L.qkv, p->xq, p->xs, p->qkv);
            else if (sf) rc = launch_stream_f16<SF_STORE>(p, L.qkv, nullptr, p->xb, p->qkv, TR(2));
            else rc = launch_matvec_f16<MODE_STORE>(p, L.qkv, p->xb, p->qkv);
        }
        if (rc) return rc; n++;
        float *kc = p->key_cache + (size_t)l * ctx_kv, *vc = p->value_cache + (size_t)l * ctx_kv;
        {
            const size_t att_smem = att_smem_bytes(c.head_size, c.context_length, p->att_scratch != nullptr);
            auto att = [&](auto kern) {
                return launch_k(p, pdl, kern, dim3(p->nh_l), dim3(ATT_THREADS), att_smem, p->qkv, kc, vc, (const StepState *)p->st,
                                (const float *)p->rope_cr, (const float *)p->rope_ci, p->nh_l, p->nkv_l, p->kflags, (const float *)L.q_norm,
                                (const float *)L.k_norm, (const float *)L.qkv_bias, c.rms_norm_eps, att_score_arg(p), q8 ? p->attq : nullptr, q8 ? p->atts : nullptr, xbf, TR(4),
                                p->tp, (unsigned)(4 * l + 0), rank * p->nh_l, p->att_scratch, c.context_length);
            };
            if (c.head_size == 128) rc = att(k_attention<128>);
            else if (c.head_size == 64) rc = att(k_attention<64>);
            else if (c.head_size == 256) rc = att(k_attention<256>);
            else if (c.head_size == 96) rc = att(k_attention<96>);
            else rc = att(k_attention<32>);
            if (rc) return rc;
            n++;
        }
        if (st) rc = launch_stream<SMV_RESID>(p, L.two, p->attq, p->atts, p->x, nullptr, nullptr, false, TR(5), tpar ? TP_SLOT_ATT : -1, 4 * l + 0, tpar ? TP_SLOT_X : -1, 4 * l + 1, rank * p->dim_l);
        else if (q8) rc = launch_matvec_q8<MODE_RESID>(p, L.wo, p->xq, p->xs, p->x);
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
        if (st) {
            if (fz) rc = launch_stream_norm<SMV_GATEUP>(p, L.tgu, L.ffn_norm, false, p->hb, p->hq, p->hs, false, TR(6)); // FFN norm + gate/up
            else rc = launch_stream<SMV_GATEUP>(p, L.tgu, p->xq, p->xs, p->hb, p->hq, p->hs, false, TR(6), -1, 0, tpar ? TP_SLOT_HQ : -1, 4 * l + 2, rank * p->hid_l);
            if (rc) return rc; n++;
            if ((rc = launch_stream<SMV_RESID>(p, L.tw2, p->hq, p->hs, p->x, nullptr, nullptr, false, TR(7), tpar ? TP_SLOT_HQ : -1, 4 * l + 2, tpar ? TP_SLOT_X : -1, 4 * l + 3, rank * p->dim_l))) return rc; n++;
        } else if (q8) {
            k_gateup_q8<<<c.hidden_dim / 32, 256, q8_smem_bytes(c.dim, 4, 8), p->stream>>>(
                (const int8_t *)L.w1.qs, L.w1.sc, (const int8_t *)L.w3.qs, L.w3.sc, p->xq, p->xs, c.hidden_dim, c.dim, p->hq, p->hs, p->hb);
            CK(cudaGetLastError()); n++;
            if ((rc = launch_matvec_q8<MODE_RESID>(p, L.w2, p->hq, p->hs, p->x))) return rc; n++;
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
        if (fz) rc = launch_stream_norm<SMV_STORE>(p, p->tout, p->out_norm, false, p->logits, nullptr, nullptr, true, TR(8)); // final norm + lm_head
        else {
            if ((rc = norm(false, p->out_norm, last_x_op))) return rc;
            n++;
            if (st) rc = launch_stream<SMV_STORE>(p, p->tout, p->xq, p->xs, p->logits, nullptr, nullptr, true, TR(8), -1, 0, -1, 0, rank * p->voc_l);
            else if (q8) rc = launch_matvec_q8<MODE_STORE>(p, p->out, p->xq, p->xs, p->logits);
            else if (sf) rc = launch_stream_f16<SF_STORE>(p, p->out, nullptr, p->xb, p->logits, TR(8), true);
            else rc = launch_matvec_f16<MODE_STORE>(p, p->out, p->xb, p->logits);
        }
        if (rc) return rc; n++;
    }
    {
        int rc;
        if ((rc = launch_k(p, pdl, k_argmax_advance, dim3(1), dim3(1024), (size_t)0, (const float *)p->logits, c.vocab_size, p->st, (const int *)p->seq_tokens, p->out_ids, with_logits ? 1 : 0,
                           (const float *)(st || sf ? p->part_val : nullptr), (const int *)(st || sf ? p->part_idx : nullptr),
                           sf ? sf_grid(p, c.vocab_size, c.dim, false) : p->n_sms, TR(9), p->tp, with_logits ? -1 : last_x_op))) return rc;
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
    if (p->is_moe) { p->pd_why = "the persistent decode kernel has no Qwen2-MoE layer (MoE plans decode through the CUDA graph)"; return B200_OK; }
    if (!p->use_stream) { p->pd_why = "the persistent decode kernel needs the Q8_0 streaming layout"; return B200_OK; }
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
    CK(set_max_dyn(k_decode_persistent<128>, maxdyn));
    CK(set_max_dyn(k_decode_persistent<64>, maxdyn));
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
    if (c.head_size == 128) CK(cudaLaunchKernelEx(&cfg, k_decode_persistent<128>, a, p->pd_L));
    else CK(cudaLaunchKernelEx(&cfg, k_decode_persistent<64>, a, p->pd_L));
    if (launches) *launches = 1;
    return B200_OK;
}

int capture(b200_plan *p, bool with_logits, cudaGraphExec_t *exec, int *launches, bool trace = false, bool persistent = false) {
    cudaGraph_t g = nullptr;
    CK(cudaStreamBeginCapture(p->stream, cudaStreamCaptureModeThreadLocal));
    int rc = persistent ? enqueue_persistent(p, with_logits, launches, trace) : enqueue_forward(p, with_logits, launches, trace);
    cudaError_t e = cudaStreamEndCapture(p->stream, &g);
    if (rc) { if (g) cudaGraphDestroy(g); return rc; }
    if (e != cudaSuccess) return fail(p, B200_ERR_CUDA, "cudaStreamEndCapture: %s", cudaGetErrorString(e));
    e = cudaGraphInstantiate(exec, g, 0);
    cudaGraphDestroy(g);
    if (e != cudaSuccess) return fail(p, B200_ERR_CUDA, "cudaGraphInstantiate: %s", cudaGetErrorString(e));
    return B200_OK;
}

// Both decode implementations are captured; b200_set_decode_mode picks which one the forward calls launch.
int capture_all(b200_plan *p) {
    int rc;
    if ((rc = capture(p, true, &p->g_decode, &p->launches_decode))) return rc;
    if ((rc = capture(p, false, &p->g_prefill, nullptr))) return rc;
    if (p->use_stream || p->use_f16_stream) {
        if ((rc = dalloc(p, &p->trace_rec, (size_t)(p->launches_decode + 8) * 32))) return rc;
        if ((rc = capture(p, true, &p->g_trace, nullptr, true))) return rc;
    }
    if ((rc = pd_prepare(p))) return rc;
    if (p->pd_ok) {
        // grid = one CTA per SM with (almost) all of its shared memory: co-resident on an idle GPU either way; the cooperative
        // attribute makes the driver check it.  Should a driver refuse cooperative kernel nodes in a graph, retry without.
        for (int attempt = 0; attempt < 2; attempt++) {
            p->pd_coop = attempt == 0;
            rc = capture(p, true, &p->g_pdecode, nullptr, false, true);
            if (!rc) rc = capture(p, false, &p->g_pprefill, nullptr, false, true);
            if (!rc) rc = capture(p, true, &p->g_ptrace, nullptr, true, true);
            if (!rc) break;
            cudaGetLastError();
            for (cudaGraphExec_t *g : {&p->g_pdecode, &p->g_pprefill, &p->g_ptrace})
                if (*g) { cudaGraphExecDestroy(*g); *g = nullptr; }
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

// One forward step of n rows: the single-sequence graph's kernel sequence, every launch serving all n rows.  prefill: a step of
// b200_prefill_slots -- the rows come from the call's schedule (k_batch_rows_next) and there is no final norm, lm_head or argmax.
// split: rows may share a sequence, so the attention runs as k_rope_kv_batch + k_attention_cached_rows (one more launch per
// layer).  own: the K / V target is the plan's cache (key_cache / value_cache, slot 0's layout) instead of the decode slots.
int enqueue_batch(b200_plan *p, int n, int *launches, bool prefill = false, bool split = false, bool own = false) {
    const b200_config &c = p->cfg;
    auto &B = p->bt;
    const bool pdl = p->use_pdl;
    const int qkvd = p->qd + 2 * p->kvd;
    const size_t ctx_kv = (size_t)c.context_length * p->kvd, slot_stride = (size_t)c.n_layers * ctx_kv;
    const size_t norm_smem = norm_smem_bytes(c.dim);
    TpCtx solo{};
    solo.n = 1;
    int k = 0, rc;
    if (prefill) {
        k_batch_rows_next<<<1, 32, 0, p->stream>>>(B.sched, B.step, B.rows);
        CK(cudaGetLastError());
        k++;
    }
    auto norm = [&](bool embed, const float *w) {
        auto go = [&](auto kern) { // the first norm of a prefill step waits for k_batch_rows_next in full: the rows are read before any PDL wait
            return launch_k(p, pdl && !(prefill && embed), kern, dim3(n), dim3(NORM_THREADS), norm_smem, B.x, (const BatchRows *)B.rows, p->emb, p->mup.embedding_scale, w, c.rms_norm_eps, c.dim, B.xq, B.xs, TraceBuf{nullptr, 0, 0}, solo);
        };
        k++;
        return embed ? go(k_rmsnorm_quant_batch<true>) : go(k_rmsnorm_quant_batch<false>);
    };
    for (int l = 0; l < c.n_layers; l++) {
        const LayerW &L = p->layers[l];
        if ((rc = norm(l == 0, L.attn_norm))) return rc;
        if ((rc = launch_stream_batch<SMV_STORE>(p, L.tqkv, n, B.xq, B.xs, B.qkv, qkvd))) return rc;
        float *kc = (own ? p->key_cache : B.slot_k) + (size_t)l * ctx_kv, *vc = (own ? p->value_cache : B.slot_v) + (size_t)l * ctx_kv;
        // split: the two launches of a step whose rows may share a sequence
        auto att2 = [&](auto rope_kern, auto att_kern, int hs) {
            const int r = launch_k(p, pdl, rope_kern, dim3(p->nh_l, n), dim3(2 * hs), (size_t)0, B.qkv, qkvd, kc, vc, slot_stride, (const BatchRows *)B.rows,
                                   (const float *)p->rope_cr, (const float *)p->rope_ci, p->nh_l, p->nkv_l, p->kflags, (const float *)L.q_norm,
                                   (const float *)L.k_norm, (const float *)L.qkv_bias, c.rms_norm_eps);
            k++;
            return r ? r : launch_k(p, pdl, att_kern, dim3(p->nh_l, n), dim3(ATT_THREADS), att_smem_bytes(c.head_size, c.context_length, B.att_scratch != nullptr),
                                    B.qkv, qkvd, kc, vc, slot_stride, (const BatchRows *)B.rows, p->nh_l, p->nkv_l, p->kflags, att_score_arg(p), B.xq, B.xs,
                                    B.att_scratch, c.context_length, TraceBuf{nullptr, 0, 0}, solo);
        };
        auto att = [&](auto kern) {
            return launch_k(p, pdl, kern, dim3(p->nh_l, n), dim3(ATT_THREADS), att_smem_bytes(c.head_size, c.context_length, B.att_scratch != nullptr), B.qkv, qkvd,
                            kc, vc, slot_stride, (const BatchRows *)B.rows, (const float *)p->rope_cr, (const float *)p->rope_ci, p->nh_l, p->nkv_l, p->kflags,
                            (const float *)L.q_norm, (const float *)L.k_norm, (const float *)L.qkv_bias, c.rms_norm_eps, att_score_arg(p), B.xq,
                            B.xs, B.att_scratch, c.context_length, TraceBuf{nullptr, 0, 0}, solo);
        };
        if (split) {
            if (c.head_size == 128) rc = att2(k_rope_kv_batch<128>, k_attention_cached_rows<128>, 128);
            else if (c.head_size == 64) rc = att2(k_rope_kv_batch<64>, k_attention_cached_rows<64>, 64);
            else if (c.head_size == 256) rc = att2(k_rope_kv_batch<256>, k_attention_cached_rows<256>, 256);
            else if (c.head_size == 96) rc = att2(k_rope_kv_batch<96>, k_attention_cached_rows<96>, 96);
            else rc = att2(k_rope_kv_batch<32>, k_attention_cached_rows<32>, 32);
        } else if (c.head_size == 128) rc = att(k_attention_batch<128>);
        else if (c.head_size == 64) rc = att(k_attention_batch<64>);
        else if (c.head_size == 256) rc = att(k_attention_batch<256>);
        else if (c.head_size == 96) rc = att(k_attention_batch<96>);
        else rc = att(k_attention_batch<32>);
        if (rc) return rc;
        if ((rc = launch_stream_batch<SMV_RESID>(p, L.two, n, B.xq, B.xs, B.x, c.dim))) return rc;
        if ((rc = norm(false, L.ffn_norm))) return rc;
        if ((rc = launch_stream_batch<SMV_GATEUP>(p, L.tgu, n, B.xq, B.xs, B.hb, c.hidden_dim, B.hq, B.hs))) return rc;
        if ((rc = launch_stream_batch<SMV_RESID>(p, L.tw2, n, B.hq, B.hs, B.x, c.dim))) return rc;
        k += 5;
    }
    if (prefill) {
        if (launches) *launches = k;
        return B200_OK;
    }
    if ((rc = norm(false, p->out_norm))) return rc;
    if ((rc = launch_stream_batch<SMV_STORE>(p, p->tout, n, B.xq, B.xs, B.logits, sampler_padded(c.vocab_size), nullptr, nullptr, true))) return rc;
    if ((rc = launch_k(p, pdl, k_argmax_batch, dim3(n), dim3(32), (size_t)0, (const float *)B.part_val, (const int *)B.part_idx, p->n_sms, B.ids))) return rc;
    if (launches) *launches = k + 2;
    return B200_OK;
}

int capture_batch(b200_plan *p, int n, bool prefill = false, bool split = false, bool own = false) {
    auto &B = p->bt;
    cudaGraph_t g = nullptr;
    CK(cudaStreamBeginCapture(p->stream, cudaStreamCaptureModeThreadLocal));
    int *launches = split ? &B.launches_s[own][!prefill][n] : prefill ? &B.launches_p[n] : &B.launches[n];
    int rc = enqueue_batch(p, n, launches, prefill, split, own);
    cudaError_t e = cudaStreamEndCapture(p->stream, &g);
    if (rc) { if (g) cudaGraphDestroy(g); return rc; }
    if (e != cudaSuccess) return fail(p, B200_ERR_CUDA, "cudaStreamEndCapture: %s", cudaGetErrorString(e));
    e = cudaGraphInstantiate(split ? &B.gs[own][!prefill][n] : prefill ? &B.gp[n] : &B.g[n], g, 0);
    cudaGraphDestroy(g);
    if (e != cudaSuccess) return fail(p, B200_ERR_CUDA, "cudaGraphInstantiate: %s", cudaGetErrorString(e));
    return B200_OK;
}

void batch_free(b200_plan *p) {
    auto &B = p->bt;
    for (cudaGraphExec_t &g : B.g)
        if (g) { cudaGraphExecDestroy(g); g = nullptr; }
    for (cudaGraphExec_t &g : B.gp)
        if (g) { cudaGraphExecDestroy(g); g = nullptr; }
    for (auto &by_target : B.gs)
        for (auto &by_kind : by_target)
            for (cudaGraphExec_t &g : by_kind)
                if (g) { cudaGraphExecDestroy(g); g = nullptr; }
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
        (rc = balloc(p, &B.smp_out, N * 8 * 4)) || (rc = balloc(p, &B.blk_cnt, N * (c.hidden_dim / 32) * 4)) || (rc = balloc(p, &B.rows, sizeof(BatchRows))) ||
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
const char *multi_why(const b200_plan *p) {
    if (p->is_moe) return "multi-position steps have no Qwen2-MoE layer (MoE plans run one position per step)";
    if (p->cfg.tp_size > 1) return "multi-position steps run on single-GPU plans only (this plan is tensor-parallel)";
    if (p->wtype != B200_GGML_Q8_0) return "multi-position steps need Q8_0 weights (FP16 plans run one position per step)";
    if (!p->use_stream) return "multi-position steps need the Q8_0 streaming layout (this plan uses the non-streaming matvecs)";
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

// Enqueues the steps of one call back to back without the classifier: the schedule is uploaded once and k_batch_rows_next
// feeds each step its entry, so the caller synchronises once.  p->ev0 / ev1 bracket the steps.  own: every row writes the plan's cache (slot 0); otherwise a
// step whose rows name distinct slots runs the b200_prefill_slots graph, and one with a repeated slot the split form.
int run_steps(b200_plan *p, const std::vector<BatchRows> &sched, const std::vector<int> &nrows, bool own, int *launches) {
    auto &B = p->bt;
    const int steps = (int)sched.size();
    std::vector<char> split(steps, own);
    for (int s = 0; s < steps; s++)
        for (int i = 0; i < nrows[s] && !split[s]; i++)
            for (int j = 0; j < i; j++)
                if (sched[s].slot[j] == sched[s].slot[i]) { split[s] = 1; break; }
    int rc;
    for (int s = 0; s < steps; s++) {
        const int n = nrows[s];
        if (split[s] ? !B.gs[own][0][n] && (rc = capture_batch(p, n, true, true, own)) : !B.gp[n] && (rc = capture_batch(p, n, true))) return rc;
    }
    CK(cudaMemcpyAsync(B.sched, sched.data(), (size_t)steps * sizeof(BatchRows), cudaMemcpyHostToDevice, p->stream));
    CK(cudaMemsetAsync(B.step, 0, 4, p->stream));
    CK(cudaEventRecord(p->ev0, p->stream));
    int k = 0;
    for (int s = 0; s < steps; s++) {
        const int n = nrows[s];
        CK(cudaGraphLaunch(split[s] ? B.gs[own][0][n] : B.gp[n], p->stream));
        k += split[s] ? B.launches_s[own][0][n] : B.launches_p[n];
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
    if (c.dim > 8192) return fail(p, B200_ERR_UNSUPPORTED, "dim > 8192 not supported by the RMSNorm kernel");
    size_t need_norm = norm_smem_bytes(c.dim);
    size_t need_att = att_smem_bytes(c.head_size, c.context_length, p->att_scratch != nullptr);
    int maxcols = c.hidden_dim > c.dim ? c.hidden_dim : c.dim;
    if (p->qd > maxcols) maxcols = p->qd;
    size_t need_mv = q8_smem_bytes(maxcols, 4, 8);
    size_t need_f16 = f16_smem_bytes(maxcols, p->cfg.fp16_lanes);
    if (need_norm > (size_t)maxdyn || need_att > (size_t)maxdyn || (p->wtype == B200_GGML_Q8_0 && need_mv > (size_t)maxdyn) ||
        (p->wtype == B200_GGML_F16 && need_f16 > (size_t)maxdyn))
        return fail(p, B200_ERR_UNSUPPORTED, "shape needs more shared memory than the device offers (%d bytes)", maxdyn);
    static bool done = false; // process-wide, like the attribute itself (plans are created from one thread at a time per process)
    if (done) return B200_OK;
    CK(set_max_dyn(k_rmsnorm_quant<true>, maxdyn));
    CK(set_max_dyn(k_rmsnorm_quant<false>, maxdyn));
    CK(set_max_dyn(k_attention<32>, maxdyn));
    CK(set_max_dyn(k_attention<64>, maxdyn));
    CK(set_max_dyn(k_attention<128>, maxdyn));
    CK(set_max_dyn(k_attention<96>, maxdyn));
    CK(set_max_dyn(k_attention<256>, maxdyn));
    CK(set_max_dyn(k_matvec_q8<1, MODE_STORE>, maxdyn));
    CK(set_max_dyn(k_matvec_q8<2, MODE_STORE>, maxdyn));
    CK(set_max_dyn(k_matvec_q8<4, MODE_STORE>, maxdyn));
    CK(set_max_dyn(k_matvec_q8<1, MODE_RESID>, maxdyn));
    CK(set_max_dyn(k_matvec_q8<2, MODE_RESID>, maxdyn));
    CK(set_max_dyn(k_matvec_q8<4, MODE_RESID>, maxdyn));
    CK(set_max_dyn(k_gateup_q8, maxdyn));
    CK(cudaFuncSetAttribute(k_stream_matvec_q8<SMV_STORE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMV_SMEM_BUDGET_MAX));
    CK(cudaFuncSetAttribute(k_stream_matvec_q8<SMV_RESID>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMV_SMEM_BUDGET_MAX));
    CK(cudaFuncSetAttribute(k_stream_matvec_q8<SMV_GATEUP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMV_SMEM_BUDGET_MAX));
    CK(cudaFuncSetAttribute(k_stream_matvec_q8_norm<SMV_STORE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMV_SMEM_BUDGET_MAX));
    CK(cudaFuncSetAttribute(k_stream_matvec_q8_norm<SMV_GATEUP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMV_SMEM_BUDGET_MAX));
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
    CK(set_max_dyn(k_attention_batch<32>, maxdyn));
    CK(set_max_dyn(k_attention_batch<64>, maxdyn));
    CK(set_max_dyn(k_attention_batch<128>, maxdyn));
    CK(set_max_dyn(k_attention_batch<96>, maxdyn));
    CK(set_max_dyn(k_attention_batch<256>, maxdyn));
    CK(set_max_dyn(k_attention_cached_rows<32>, maxdyn));
    CK(set_max_dyn(k_attention_cached_rows<64>, maxdyn));
    CK(set_max_dyn(k_attention_cached_rows<128>, maxdyn));
    CK(set_max_dyn(k_attention_cached_rows<96>, maxdyn));
    CK(set_max_dyn(k_attention_cached_rows<256>, maxdyn));
    CK(cudaFuncSetAttribute(k_stream_matvec_q8_batch<SMV_STORE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMB_SMEM_BUDGET));
    CK(cudaFuncSetAttribute(k_stream_matvec_q8_batch<SMV_RESID>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMB_SMEM_BUDGET));
    CK(cudaFuncSetAttribute(k_stream_matvec_q8_batch<SMV_GATEUP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMB_SMEM_BUDGET));
    CK(cudaFuncSetAttribute(k_moe_gateup, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMV_SMEM_BUDGET_MAX));
    CK(cudaFuncSetAttribute(k_moe_down, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMV_SMEM_BUDGET_MAX));
    done = true;
    return B200_OK;
}

int prefill_init(b200_plan *p);

// Qwen2-MoE FFN tensors of one layer (llama.cpp's names and shapes, dims[0] innermost): the F32 router and shared-expert gate, the
// stacked routed experts [E][rows][cols] and the shared expert.  Every routed expert becomes a TileMat of its own, cut from its
// row range of the stacked tensor (K-quant experts are re-quantised on the way like any matrix).
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
    if ((rc = dalloc(p, &L.shared_gate, (size_t)D * 4))) return rc;
    CK(cudaMemcpy(L.shared_gate, t[1]->data, (size_t)D * 4, cudaMemcpyHostToDevice));
    if ((rc = upload_tiles(p, t[5], t[6], nullptr, Hs, Hs, 0, D, true, L.sgu))) return rc;
    if ((rc = upload_tiles(p, t[7], nullptr, nullptr, D, 0, 0, Hs, false, L.sdn))) return rc;
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

int build(b200_plan *p, const b200_tensor *tensors, int n_tensors) {
    const b200_config &c = p->cfg;
    if (c.arch != B200_ARCH_LLAMA && c.arch != B200_ARCH_QWEN3 && c.arch != B200_ARCH_PHI3 && c.arch != B200_ARCH_QWEN2 && c.arch != B200_ARCH_QWEN2_MOE &&
        c.arch != B200_ARCH_GRANITE)
        return fail(p, B200_ERR_UNSUPPORTED, "unknown arch %d", c.arch);
    p->kflags = c.arch == B200_ARCH_QWEN3 ? (KF_NEOX | KF_QKNORM) : c.arch == B200_ARCH_PHI3 ? KF_NEOX
              : (c.arch == B200_ARCH_QWEN2 || c.arch == B200_ARCH_QWEN2_MOE) ? (KF_NEOX | KF_QKVBIAS) : c.arch == B200_ARCH_GRANITE ? KF_ATTSCALE : 0;
    if (p->is_moe) {
        const b200_moe_config &m = p->moe;
        if (c.tp_size > 1) return fail(p, B200_ERR_UNSUPPORTED, "Qwen2-MoE plans are single-GPU (tensor parallelism has no expert layout)");
        if (m.n_experts < 1 || m.n_experts > MOE_MAX_EXPERTS) return fail(p, B200_ERR_BAD_ARG, "n_experts = %d: need 1..%d", m.n_experts, MOE_MAX_EXPERTS);
        const int kmax = m.n_experts < MOE_MAX_K ? m.n_experts : MOE_MAX_K;
        if (m.n_experts_used < 1 || m.n_experts_used > kmax)
            return fail(p, B200_ERR_BAD_ARG, "n_experts_used = %d: need 1..%d (min(n_experts, %d))", m.n_experts_used, kmax, MOE_MAX_K);
        if (m.expert_hidden_dim <= 0 || m.shared_hidden_dim <= 0 || m.expert_hidden_dim % 32 || m.shared_hidden_dim % 32)
            return fail(p, B200_ERR_UNSUPPORTED, "expert hidden %d / shared hidden %d: the Q8_0 stream needs positive multiples of 32", m.expert_hidden_dim,
                        m.shared_hidden_dim);
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
    if (c.arch != B200_ARCH_QWEN3 && p->qd != c.dim) return fail(p, B200_ERR_BAD_ARG, "llama / phi3 / qwen2: n_heads*head_size must equal dim");
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
        return fail(p, B200_ERR_UNSUPPORTED, "Qwen2-MoE runs in Q8_0 only (FP16 MoE plans are not supported, as in the reference)");
    bool any_kq = false;
    for (int i = 0; i < n_tensors; i++) any_kq = any_kq || kq_is_kquant(tensors[i].ggml_type);

    CK(cudaSetDevice(p->device));
    read_knobs(p);
    CK(cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking));
    CK(cudaEventCreate(&p->ev0));
    CK(cudaEventCreate(&p->ev1));
    int rc;
    CK(cudaDeviceGetAttribute(&p->n_sms, cudaDevAttrMultiProcessorCount, p->device));
    {
        const char *e = getenv("B200_STREAM");
        bool want = !(e && e[0] == '0');
        p->use_stream = want && p->wtype == B200_GGML_Q8_0 && stream_shape_ok(p->qd_l + 2 * p->kvd_l, c.dim) && stream_shape_ok(p->dim_l, p->qd) &&
                        (p->is_moe || (stream_shape_ok(2 * p->hid_l, c.dim) && stream_shape_ok(p->dim_l, c.hidden_dim))) && stream_shape_ok((p->voc_l + 3) & ~3, c.dim) &&
                        gateup_fits(p->hid_l, p->n_sms);
        const char *e3 = getenv("B200_F16_STREAM"); // FP16 plans: 0 = the round-1 k_matvec_f16 launches
        p->use_f16_stream = !(e3 && e3[0] == '0') && p->wtype == B200_GGML_F16 && c.tp_size == 1 && sf_layout(p->qd + 2 * p->kvd, c.dim, c.fp16_lanes, false).ok &&
                            sf_layout(c.dim, p->qd, c.fp16_lanes, false).ok && sf_layout(c.hidden_dim, c.dim, c.fp16_lanes, true).ok &&
                            sf_layout(c.dim, c.hidden_dim, c.fp16_lanes, false).ok && sf_layout(c.vocab_size, c.dim, c.fp16_lanes, false).ok;
        if (p->is_moe) { // the MoE FFN has its own streams (the dense FFN checks above are skipped)
            const b200_moe_config &m = p->moe;
            const int hs = m.shared_hidden_dim, he = m.expert_hidden_dim;
            const bool cut = stream_shape_ok(2 * hs, c.dim) && stream_shape_ok(c.dim, hs) && stream_shape_ok(2 * he, c.dim) && stream_shape_ok(c.dim, he) &&
                             gateup_fits(p->moe_hv, p->n_sms);
            if (!cut) return fail(p, B200_ERR_UNSUPPORTED, "expert hidden %d / shared hidden %d at dim %d: the Q8_0 stream layout cannot cut these matrices", he, hs, c.dim);
            p->moe_dl = moe_down_layout(p->moe_hv, hs / smv_pick_nseg(hs), he / smv_pick_nseg(he), SMV_SMEM_BUDGET_MAX);
            if (p->moe_dl.stages < 3) return fail(p, B200_ERR_UNSUPPORTED, "the expert down projection leaves fewer than 3 ring stages of shared memory");
            if (!p->use_stream) return fail(p, B200_ERR_UNSUPPORTED, "Qwen2-MoE needs the Q8_0 streaming layout (this plan would use the non-streaming matvecs)");
        }
        p->use_pdl = p->use_stream || p->use_f16_stream;
        // Tensor parallelism keeps the separate norm: its read of x waits on every rank's slice (TP_SLOT_X).  So does Qwen2-MoE,
        // whose FFN norm must write float xb for the F32 router anyway; its plans keep 8 launches per layer.
        p->fuse_norm = p->use_stream && c.tp_size == 1 && !p->is_moe && norm_fusion_ok(c.dim);
        if (c.tp_size > 1 && !p->use_stream) return fail(p, B200_ERR_UNSUPPORTED, "tensor parallelism needs the Q8_0 streaming path");
    }
    size_t stage_bytes = (size_t)34 * (8u << 20); // 8 Mi blocks = 272 MiB
    if (p->use_stream) {
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
    const auto t_up0 = std::chrono::steady_clock::now();
    if ((rc = up_init(p, stage_bytes))) return rc;
    struct StageGuard { b200_plan *pl; ~StageGuard() { up_destroy(pl); } } guard{p};

    // embedding table (+ tied classifier: AbstractModelLoader.java:186-195)
    if ((rc = alloc_matrix(p, p->emb, c.vocab_size, c.dim, eff_type(emb->ggml_type)))) return rc;
    if ((rc = upload_matrix(p, emb, c.vocab_size, c.dim, p->emb, 0))) return rc;
    const b200_tensor *outw = find(tensors, n_tensors, "output.weight");
    if (p->use_stream) {
        if (!outw && eff_type(emb->ggml_type) != p->wtype) return fail(p, B200_ERR_UNSUPPORTED, "tied output weight type differs from the matrix type");
        {
            const int r0[3] = {c.tp_rank * p->voc_l, 0, 0}, fu[3] = {c.vocab_size, 0, 0};
            if ((rc = upload_tiles(p, outw ? outw : emb, nullptr, nullptr, p->voc_l, 0, 0, c.dim, false, p->tout, r0, fu))) return rc;
        }
        p->out = p->emb;
        if ((rc = dalloc(p, &p->part_val, (size_t)p->n_sms * 4))) return rc;
        if ((rc = dalloc(p, &p->part_idx, (size_t)p->n_sms * 4))) return rc;
        const int hid = c.hidden_dim > p->moe_hv ? c.hidden_dim : p->moe_hv;
        if ((rc = dalloc(p, &p->blk_cnt, (size_t)(hid / 32) * 4))) return rc;
        CK(cudaMemset(p->blk_cnt, 0, (size_t)(hid / 32) * 4));
    } else if (outw) {
        if (p->use_f16_stream) { // per-CTA argmax partials of the classifier launch (at most 3 CTAs per SM)
            if ((rc = dalloc(p, &p->part_val, (size_t)p->n_sms * 4 * 4))) return rc;
            if ((rc = dalloc(p, &p->part_idx, (size_t)p->n_sms * 4 * 4))) return rc;
        }
        if ((rc = alloc_matrix(p, p->out, c.vocab_size, c.dim, p->wtype))) return rc;
        if ((rc = upload_matrix(p, outw, c.vocab_size, c.dim, p->out, 0))) return rc;
    } else {
        if (eff_type(emb->ggml_type) != p->wtype) return fail(p, B200_ERR_UNSUPPORTED, "tied output weight type differs from the matrix type");
        p->out = p->emb;
        if (p->use_f16_stream) {
            if ((rc = dalloc(p, &p->part_val, (size_t)p->n_sms * 4 * 4))) return rc;
            if ((rc = dalloc(p, &p->part_idx, (size_t)p->n_sms * 4 * 4))) return rc;
        }
    }
    if ((rc = upload_f32(p, find(tensors, n_tensors, "output_norm.weight"), c.dim, &p->out_norm, "output_norm.weight"))) return rc;

    p->layers.resize(c.n_layers);
    for (int l = 0; l < c.n_layers; l++) {
        LayerW &L = p->layers[l];
        std::string pre = "blk." + std::to_string(l) + ".";
        auto T = [&](const char *s) { return find(tensors, n_tensors, pre + s); };
        if ((rc = upload_f32(p, T("attn_norm.weight"), c.dim, &L.attn_norm, "attn_norm.weight"))) return rc;
        if ((rc = upload_f32(p, T("ffn_norm.weight"), c.dim, &L.ffn_norm, "ffn_norm.weight"))) return rc;
        if (c.arch == B200_ARCH_QWEN3) {
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
        if (p->use_stream) {
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
        // fused [Wq; Wk; Wv] so one launch produces the packed q|k|v vector
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
    // cos/sin evaluated in double and narrowed.
    {
        int half = c.head_size / 2;
        std::vector<float> cr((size_t)c.context_length * half), ci((size_t)c.context_length * half);
        size_t k = 0;
        for (int pos = 0; pos < c.context_length; pos++)
            for (int i = 0; i < c.head_size; i += 2) {
                float freq = (float)(1.0 / pow((double)c.rope_theta, i / (double)c.head_size));
                float val = (float)pos * freq;
                cr[k] = (float)cos((double)val);
                ci[k] = (float)sin((double)val);
                k++;
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
        if ((rc = dalloc(p, &p->moe_w, (size_t)c.n_layers * (k + 1) * 4))) return rc;
        if ((rc = dalloc(p, &p->moe_logits, (size_t)c.n_layers * (E + 1) * 4))) return rc;
        if ((rc = dalloc(p, &p->moe_done, (size_t)c.n_layers * 4))) return rc;
        CK(cudaMemset(p->moe_ids, 0, (size_t)c.n_layers * k * 4));
        CK(cudaMemset(p->moe_w, 0, (size_t)c.n_layers * (k + 1) * 4));
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
    if ((rc = set_smem_attrs(p))) return rc;
    if (c.tp_size > 1) { CK(cudaStreamSynchronize(p->stream)); return B200_OK; } // graphs are captured by b200_tp_attach
    if ((rc = capture_all(p))) return rc;
    if (p->prefill_batch > 1)
        if ((rc = prefill_init(p))) return rc;
    CK(cudaStreamSynchronize(p->stream));
    return B200_OK;
}

// ---- batched prefill on the tensor cores (prefill.cuh) -------------------------------------------
static const char *const MOE_PREFILL_WHY = "Qwen2-MoE plans have no tensor-core prefill: prompts go through the exact token-by-token prefill";
// What both tensor-core modes need of the plan's shape; nullptr when the chunk GEMMs and the attention can run it.
static const char *prefill_shape_why(const b200_plan *p) {
    const b200_config &g = p->cfg;
    const int kv_mul = g.n_heads / g.n_kv_heads, nqkv = p->qd + 2 * p->kvd;
    if (p->is_moe) return MOE_PREFILL_WHY;
    if (g.tp_size > 1) return "tensor-core prefill is single-GPU";
    if (g.head_size != 64 && g.head_size != 128) return "tensor-core prefill supports head sizes 64 and 128";
    if (g.n_heads % g.n_kv_heads || kv_mul > 64) return "tensor-core prefill needs n_heads % n_kv_heads == 0 and a GQA ratio <= 64";
    if (g.dim % 128 || p->qd % 128 || nqkv % 128 || g.hidden_dim % 64) return "tensor-core prefill needs dim, q width and q+k+v width multiples of 128, hidden a multiple of 64";
    if (!pg::encode_fn()) return "cuTensorMapEncodeTiled not available from the driver";
    return nullptr;
}

// The chunk's scratch buffers, their tensor maps and the attention kernels' shared-memory attributes: allocated once per
// plan, shared by both tensor-core modes.  *ok = false if a tensor map was rejected.
static int prefill_scratch(b200_plan *p, bool *ok) {
    PrefillCtx &c = p->prefill;
    const b200_config &g = p->cfg;
    const int nqkv = p->qd + 2 * p->kvd;
    *ok = true;
    if (c.bpad) return B200_OK;
    c.bpad = (c.batch + pg::BM - 1) / pg::BM * pg::BM; // whole 128-row GEMM tiles
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
    if (g.head_size == 128) {
        CK(cudaFuncSetAttribute(k_pf_attention_mma<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pm_smem_bytes<128>()));
        CK(cudaFuncSetAttribute(k_pf_attention_mma_packed<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pm_smem_bytes<128>()));
    } else {
        CK(cudaFuncSetAttribute(k_pf_attention_mma<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pm_smem_bytes<64>()));
        CK(cudaFuncSetAttribute(k_pf_attention_mma_packed<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pm_smem_bytes<64>()));
    }
    return B200_OK;
}

int prefill_init(b200_plan *p) {
    PrefillCtx &c = p->prefill;
    const b200_config &g = p->cfg;
    c.batch = p->prefill_batch;
    c.ready = false;
    if (c.mode == B200_PREFILL_TENSOR_CORE) c.mode = B200_PREFILL_EXACT;
    const int nqkv = p->qd + 2 * p->kvd;
    if (p->wtype != B200_GGML_F16 && !p->f16_copies) {
        c.why = p->use_stream ? "Q8_0 plan: the tensor-core prefill is opt-in (b200_set_prefill_mode builds f16 twins of the weight matrices, +2 bytes per weight)"
                              : "tensor-core prefill needs FP16 weight matrices or a Q8_0 plan on the streaming path";
        return B200_OK;
    }
    if ((c.why = prefill_shape_why(p))) return B200_OK;
    bool ok;
    int rc;
    if ((rc = prefill_scratch(p, &ok))) return rc;
    c.maps.resize(g.n_layers);
    for (int l = 0; ok && l < g.n_layers; l++) {
        const LayerW &L = p->layers[l];
        PrefillLayerMaps &m = c.maps[l];
        ok = pg::make_map(&m.qkv, L.qkv.qs, nqkv, g.dim, pg::BN) == 0 && pg::make_map(&m.wo, L.wo.qs, g.dim, p->qd, pg::BN) == 0 &&
             pg::make_map(&m.w1, L.w1.qs, g.hidden_dim, g.dim, pg::BN / 2) == 0 && pg::make_map(&m.w3, L.w3.qs, g.hidden_dim, g.dim, pg::BN / 2) == 0 &&
             pg::make_map(&m.w2, L.w2.qs, g.dim, g.hidden_dim, pg::BN) == 0;
    }
    if (!ok) { c.why = "cuTensorMapEncodeTiled rejected a tensor map"; return B200_OK; }
    c.ready = true;
    c.mode = B200_PREFILL_TENSOR_CORE;
    c.why = "";
    return B200_OK;
}

// W8A16: the GEMMs read B from the tile-major Q8_0 streams the decode kernels use (L.tqkv, L.two, L.tgu, L.tw2) -- no
// per-weight memory.  Built on the first b200_set_prefill_mode(TENSOR_CORE_W8A16).
int prefill_init_q8(b200_plan *p) {
    PrefillCtx &c = p->prefill;
    const b200_config &g = p->cfg;
    c.batch = p->prefill_batch;
    if (p->prefill_batch <= 1) { c.why_q8 = "the plan was created without a prefill batch size (prefill_batch_size <= 1)"; return B200_OK; }
    if (p->wtype != B200_GGML_Q8_0) { c.why_q8 = "W8A16 prefill needs a Q8_0 plan (FP16 plans run the tensor-core prefill on their own f16 matrices)"; return B200_OK; }
    if (g.tp_size > 1) { c.why_q8 = "tensor-core prefill is single-GPU"; return B200_OK; }
    if (!p->use_stream) { c.why_q8 = "W8A16 prefill reads the tile-major Q8_0 streams: the plan must use the streaming layout"; return B200_OK; }
    if ((c.why_q8 = prefill_shape_why(p))) return B200_OK;
    for (int l = 0; l < g.n_layers; l++) {
        const LayerW &L = p->layers[l];
        for (const TileMat *t : {&L.tqkv, &L.two, &L.tgu, &L.tw2})
            if (t->seg % pg::BK) { c.why_q8 = "W8A16 prefill needs Q8_0 stream segments that are multiples of 64 columns"; return B200_OK; }
    }
    bool ok;
    int rc;
    if ((rc = prefill_scratch(p, &ok))) return rc;
    c.maps_q8.resize(g.n_layers);
    for (int l = 0; ok && l < g.n_layers; l++) {
        const LayerW &L = p->layers[l];
        PrefillQ8Maps &m = c.maps_q8[l];
        auto mk = [](CUtensorMap *q, CUtensorMap *s, const TileMat &t) {
            return pg::make_map_q8(q, t.base, (uint64_t)t.rows, t.nseg, t.unit_bytes, 0) == 0 && pg::make_map_q8(s, t.base, (uint64_t)t.rows, t.nseg, t.unit_bytes, 1) == 0;
        };
        ok = mk(&m.qkv_q, &m.qkv_s, L.tqkv) && mk(&m.wo_q, &m.wo_s, L.two) && mk(&m.gu_q, &m.gu_s, L.tgu) && mk(&m.w2_q, &m.w2_s, L.tw2);
    }
    if (!ok) { c.why_q8 = "cuTensorMapEncodeTiled rejected a tensor map"; return B200_OK; }
    c.q8_ready = true;
    c.why_q8 = "";
    return B200_OK;
}

// Q8_0 plan: f16 twins of the weight matrices, dequantised on the device from the tile-major stream (value = f16(q * scale),
// Q8_0FloatTensor.getFloat rounded once) -- the B operands of the tensor-core GEMMs; the reference's Q8_0 MMA prefill also
// feeds FP16 tiles (LlamaQ8_0LayersBatchPrefillMMA.java).  Built on the first b200_set_prefill_mode(TENSOR_CORE).
int build_f16_twins(b200_plan *p) {
    const b200_config &c = p->cfg;
    if (p->f16_copies) return B200_OK;
    if (p->wtype != B200_GGML_Q8_0 || !p->use_stream || c.tp_size > 1) return fail(p, B200_ERR_UNSUPPORTED, "f16 twins need a single-GPU Q8_0 plan on the streaming path");
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

// A packed chunk of b200_prefill_slots: the device tables of prefill.cuh and the f16 scratch the sequences' regions live in
struct PfPacked {
    const PfTok *tok;
    const PfTile *tiles;
    int n_tiles;
    const PfHist *hist; // sequences with start > 0
    int n_hist, max_start;
    __half *KH, *VH;
};

// n tokens already in c.tok (device), positions start_pos .. start_pos + n - 1 of the plan's cache; or, with pk, the packed
// tokens of several sequences, each written to its own decode slot (start_pos unused)
int prefill_forward(b200_plan *p, int n, int start_pos, int *launches, const PfPacked *pk = nullptr) {
    PrefillCtx &c = p->prefill;
    const b200_config &g = p->cfg;
    cudaStream_t s = p->stream;
    const int nqkv = p->qd + 2 * p->kvd, mt = (n + pg::BM - 1) / pg::BM, kv_mul = g.n_heads / g.n_kv_heads;
    const size_t ctx_kv = (size_t)g.context_length * p->kvd;
    // k_pf_attention_mma scales q by this times log2(e): 1/sqrt(head size), or Granite's attentionScale
    const float inv_sqrt_hs = (p->kflags & KF_ATTSCALE) ? p->mup.attention_scale : (float)(1.0 / sqrt((double)g.head_size));
    int nl = 0;
    constexpr int ST = pg::GEMM_STAGES;
    const bool q8 = c.mode == B200_PREFILL_TENSOR_CORE_W8A16; // B from the Q8_0 streams (c.maps_q8) instead of the f16 matrices (c.maps)
    using pg::B_Q8;
    // the x += A W^T GEMMs (N = dim only) split K until the grid fills the SMs -- every split reduce-adds its partial
    // product through TMA -- keeping at least 8 k-blocks per split
    auto splits = [&](int n_tiles, int K) {
        const int nk = K / pg::BK;
        int sp = p->n_sms / (mt * n_tiles);
        if (sp > 4) sp = 4;
        while (sp > 1 && (nk / sp < 8 || (sp - 1) * ((nk + sp - 1) / sp) >= nk)) sp--;
        return sp < 1 ? 1 : sp;
    };
    k_pf_embed<<<n, 256, 0, s>>>(c.tok, p->emb, p->mup.embedding_scale, c.X, g.dim); nl++;
    for (int l = 0; l < g.n_layers; l++) {
        const LayerW &L = p->layers[l];
        const PrefillLayerMaps *m = q8 ? nullptr : &c.maps[l];
        const PrefillQ8Maps *mq = q8 ? &c.maps_q8[l] : nullptr;
        float *kc = (pk ? p->bt.slot_k : p->key_cache) + (size_t)l * ctx_kv, *vc = (pk ? p->bt.slot_v : p->value_cache) + (size_t)l * ctx_kv;
        k_pf_rmsnorm_f16<<<n, 256, 0, s>>>(c.X, L.attn_norm, g.rms_norm_eps, g.dim, c.A16); nl++;
        if (q8 ? pg::gemm_launch<pg::GEMM_F32, ST, B_Q8>(c.mA, mq->qkv_q, mq->qkv_s, c.mQKV, c.QKV, nqkv, n, mt, nqkv / pg::BN, g.dim, s, 1, L.tqkv.seg)
               : pg::gemm_launch<pg::GEMM_F32, ST>(c.mA, m->qkv, m->qkv, c.mQKV, c.QKV, nqkv, n, mt, nqkv / pg::BN, g.dim, s))
            return fail(p, B200_ERR_CUDA, "QKV GEMM launch failed");
        nl++;
        const int qt = PM_ROWS / kv_mul;
        if (pk) {
            const size_t slot_stride = (size_t)g.n_layers * ctx_kv;
            if (pk->n_hist) {
                const size_t n4 = (size_t)pk->max_start * p->kvd / 4;
                const dim3 hg((unsigned)((n4 + 255) / 256 < 1184 ? (n4 + 255) / 256 : 1184), pk->n_hist);
                k_pf_kv_to_f16_packed<<<hg, 256, 0, s>>>(kc, vc, slot_stride, pk->KH, pk->VH, p->kvd, pk->hist);
                nl++;
            }
            const dim3 ag(pk->n_tiles, g.n_kv_heads);
            if (g.head_size == 128) {
                k_pf_rope_kv_packed<128><<<n, 256, 0, s>>>(c.QKV, nqkv, kc, vc, slot_stride, pk->KH, pk->VH, p->kvd, g.n_heads, g.n_kv_heads, p->kflags, L.q_norm, L.k_norm, L.qkv_bias, g.rms_norm_eps, p->rope_cr, p->rope_ci, pk->tok);
                k_pf_attention_mma_packed<128><<<ag, PM_THREADS, pm_smem_bytes<128>(), s>>>(c.QKV, nqkv, pk->KH, pk->VH, p->kvd, kv_mul, pk->tiles, inv_sqrt_hs, c.ATT16, p->qd);
            } else {
                k_pf_rope_kv_packed<64><<<n, 256, 0, s>>>(c.QKV, nqkv, kc, vc, slot_stride, pk->KH, pk->VH, p->kvd, g.n_heads, g.n_kv_heads, p->kflags, L.q_norm, L.k_norm, L.qkv_bias, g.rms_norm_eps, p->rope_cr, p->rope_ci, pk->tok);
                k_pf_attention_mma_packed<64><<<ag, PM_THREADS, pm_smem_bytes<64>(), s>>>(c.QKV, nqkv, pk->KH, pk->VH, p->kvd, kv_mul, pk->tiles, inv_sqrt_hs, c.ATT16, p->qd);
            }
        } else {
            const dim3 ag((n + qt - 1) / qt, g.n_kv_heads);
            if (start_pos > 0) { // rows written by earlier chunks / decode steps
                const size_t n4 = (size_t)start_pos * p->kvd / 4;
                k_pf_kv_to_f16<<<(unsigned)((n4 + 255) / 256 < 1184 ? (n4 + 255) / 256 : 1184), 256, 0, s>>>(kc, vc, c.KH, c.VH, n4);
                nl++;
            }
            if (g.head_size == 128) {
                k_pf_rope_kv<128><<<n, 256, 0, s>>>(c.QKV, nqkv, kc, vc, c.KH, c.VH, p->kvd, g.n_heads, g.n_kv_heads, p->kflags, L.q_norm, L.k_norm, L.qkv_bias, g.rms_norm_eps, p->rope_cr, p->rope_ci, start_pos);
                k_pf_attention_mma<128><<<ag, PM_THREADS, pm_smem_bytes<128>(), s>>>(c.QKV, nqkv, c.KH, c.VH, p->kvd, kv_mul, n, start_pos, inv_sqrt_hs, c.ATT16, p->qd);
            } else {
                k_pf_rope_kv<64><<<n, 256, 0, s>>>(c.QKV, nqkv, kc, vc, c.KH, c.VH, p->kvd, g.n_heads, g.n_kv_heads, p->kflags, L.q_norm, L.k_norm, L.qkv_bias, g.rms_norm_eps, p->rope_cr, p->rope_ci, start_pos);
                k_pf_attention_mma<64><<<ag, PM_THREADS, pm_smem_bytes<64>(), s>>>(c.QKV, nqkv, c.KH, c.VH, p->kvd, kv_mul, n, start_pos, inv_sqrt_hs, c.ATT16, p->qd);
            }
        }
        nl += 2;
        const int sp_wo = splits(g.dim / pg::BN, p->qd), sp_w2 = splits(g.dim / pg::BN, g.hidden_dim);
        const float rs = p->mup.residual_scale;
        if (q8 ? pg::gemm_launch<pg::GEMM_RESID, ST, B_Q8>(c.mATT, mq->wo_q, mq->wo_s, c.mX, c.X, g.dim, n, mt, g.dim / pg::BN, p->qd, s, sp_wo, L.two.seg, rs)
               : pg::gemm_launch<pg::GEMM_RESID, ST>(c.mATT, m->wo, m->wo, c.mX, c.X, g.dim, n, mt, g.dim / pg::BN, p->qd, s, sp_wo, 0, rs))
            return fail(p, B200_ERR_CUDA, "Wo GEMM launch failed");
        nl++;
        k_pf_rmsnorm_f16<<<n, 256, 0, s>>>(c.X, L.ffn_norm, g.rms_norm_eps, g.dim, c.A16); nl++;
        if (q8 ? pg::gemm_launch<pg::GEMM_GATEUP, ST, B_Q8>(c.mA, mq->gu_q, mq->gu_s, c.mX, c.H16, g.hidden_dim, n, mt, g.hidden_dim / (pg::BN / 2), g.dim, s, 1, L.tgu.seg)
               : pg::gemm_launch<pg::GEMM_GATEUP, ST>(c.mA, m->w1, m->w3, c.mX, c.H16, g.hidden_dim, n, mt, g.hidden_dim / (pg::BN / 2), g.dim, s))
            return fail(p, B200_ERR_CUDA, "gate/up GEMM launch failed");
        nl++;
        if (q8 ? pg::gemm_launch<pg::GEMM_RESID, ST, B_Q8>(c.mH, mq->w2_q, mq->w2_s, c.mX, c.X, g.dim, n, mt, g.dim / pg::BN, g.hidden_dim, s, sp_w2, L.tw2.seg, rs)
               : pg::gemm_launch<pg::GEMM_RESID, ST>(c.mH, m->w2, m->w2, c.mX, c.X, g.dim, n, mt, g.dim / pg::BN, g.hidden_dim, s, sp_w2, 0, rs))
            return fail(p, B200_ERR_CUDA, "W2 GEMM launch failed");
        nl++;
    }
    CK(cudaGetLastError());
    if (launches) *launches = nl;
    return B200_OK;
}

cudaGraphExec_t decode_graph(b200_plan *p) { return p->decode_mode == B200_DECODE_PERSISTENT && p->g_pdecode ? p->g_pdecode : p->g_decode; }
cudaGraphExec_t prefill_graph(b200_plan *p) { return p->decode_mode == B200_DECODE_PERSISTENT && p->g_pprefill ? p->g_pprefill : p->g_prefill; }

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

} // namespace

// b200_plan_create, b200_plan_create_moe and b200_plan_create_granite (moe / granite == nullptr: neither)
static int plan_create(const b200_config *cfg, const b200_moe_config *moe, const b200_granite_config *granite, const b200_tensor *tensors, int32_t n_tensors,
                       int32_t prefill_batch_size, int32_t device, b200_plan **out, char *err, size_t err_len) {
    if (out) *out = nullptr;
    if (!cfg || !tensors || !out || n_tensors <= 0) {
        if (err && err_len) snprintf(err, err_len, "null argument");
        return B200_ERR_BAD_ARG;
    }
    if ((cfg->arch == B200_ARCH_QWEN2_MOE) != (moe != nullptr)) {
        if (err && err_len)
            snprintf(err, err_len, moe ? "b200_plan_create_moe needs arch B200_ARCH_QWEN2_MOE (got %d)"
                                       : "arch %d (B200_ARCH_QWEN2_MOE) needs its expert configuration: create the plan with b200_plan_create_moe", cfg->arch);
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
    b200_plan *p = new b200_plan();
    p->cfg = *cfg;
    if (moe) { p->is_moe = true; p->moe = *moe; }
    if (granite) p->mup = *granite;
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

extern "C" {

int b200_plan_create(const b200_config *cfg, const b200_tensor *tensors, int32_t n_tensors, int32_t prefill_batch_size,
                     int32_t device, b200_plan **out, char *err, size_t err_len) {
    return plan_create(cfg, nullptr, nullptr, tensors, n_tensors, prefill_batch_size, device, out, err, err_len);
}

int b200_plan_create_moe(const b200_config *cfg, const b200_moe_config *moe, const b200_tensor *tensors, int32_t n_tensors, int32_t prefill_batch_size,
                         int32_t device, b200_plan **out, char *err, size_t err_len) {
    if (!moe) {
        if (out) *out = nullptr;
        if (err && err_len) snprintf(err, err_len, "null argument");
        return B200_ERR_BAD_ARG;
    }
    return plan_create(cfg, moe, nullptr, tensors, n_tensors, prefill_batch_size, device, out, err, err_len);
}

int b200_plan_create_granite(const b200_config *cfg, const b200_granite_config *granite, const b200_tensor *tensors, int32_t n_tensors,
                             int32_t prefill_batch_size, int32_t device, b200_plan **out, char *err, size_t err_len) {
    if (!granite) {
        if (out) *out = nullptr;
        if (err && err_len) snprintf(err, err_len, "null argument");
        return B200_ERR_BAD_ARG;
    }
    return plan_create(cfg, nullptr, granite, tensors, n_tensors, prefill_batch_size, device, out, err, err_len);
}

int b200_forward_decode(b200_plan *p, int32_t token, int32_t position, float *logits, int32_t *argmax) {
    if (!p) return B200_ERR_BAD_ARG;
    if (!p->g_decode) return fail(p, B200_ERR_STATE, "tensor-parallel plan: call b200_tp_attach on every rank first");
    if (logits && p->tp.n > 1) return fail(p, B200_ERR_UNSUPPORTED, "full logits are not gathered under tensor parallelism (argmax is)");
    int rc;
    if ((rc = check_pos(p, token, position))) return rc;
    CK(cudaSetDevice(p->device));
    if ((rc = set_state(p, token, position, 0, 0))) return rc;
    CK(cudaGraphLaunch(decode_graph(p), p->stream));
    if (argmax) CK(cudaMemcpyAsync(p->h_ids, p->out_ids, 4, cudaMemcpyDeviceToHost, p->stream));
    if (logits) CK(cudaMemcpyAsync(logits, p->logits, (size_t)p->cfg.vocab_size * 4, cudaMemcpyDeviceToHost, p->stream));
    CK(cudaStreamSynchronize(p->stream));
    if ((rc = check_device_error(p))) return rc;
    if (argmax) *argmax = p->h_ids[0];
    return B200_OK;
}

int b200_forward_decode_sample(b200_plan *p, int32_t token, int32_t position, float temperature, float topp, float uniform01, int32_t *token_out, int32_t *info) {
    if (!p || !token_out) return B200_ERR_BAD_ARG;
    if (!p->g_decode) return fail(p, B200_ERR_STATE, "tensor-parallel plan: call b200_tp_attach on every rank first");
    if (p->tp.n > 1) return fail(p, B200_ERR_UNSUPPORTED, "the device-side temperature/top-p sampler needs the whole logits row on one GPU (tensor-parallel plans sample greedily)");
    if (!(temperature >= 0.0f) || !(uniform01 >= 0.0f && uniform01 < 1.0f)) return fail(p, B200_ERR_BAD_ARG, "temperature must be >= 0 and the uniform number in [0, 1)");
    int rc;
    if ((rc = check_pos(p, token, position))) return rc;
    CK(cudaSetDevice(p->device));
    if ((rc = set_state(p, token, position, 0, 0))) return rc;
    CK(cudaGraphLaunch(decode_graph(p), p->stream));
    const bool greedy = temperature == 0.0f; // Sampler.selectSampler: temperature 0 -> FloatTensor.argmax, already computed by the forward
    if (!greedy) {
        static bool attr = false;
        if (!attr) { CK(cudaFuncSetAttribute(k_sample, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sampler_smem_bytes())); attr = true; }
        SamplerArgs a;
        a.logits = p->logits; a.n = p->cfg.vocab_size; a.temperature = temperature; a.topp = topp; a.r01 = uniform01;
        a.indices = p->smp_indices; a.out_id = p->smp_out; a.info = p->smp_out + 1;
        k_sample<<<1, SAMPLER_THREADS, sampler_smem_bytes(), p->stream>>>(a);
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(p->h_ids, p->smp_out, 5 * 4, cudaMemcpyDeviceToHost, p->stream));
    } else CK(cudaMemcpyAsync(p->h_ids, p->out_ids, 4, cudaMemcpyDeviceToHost, p->stream));
    CK(cudaStreamSynchronize(p->stream));
    if ((rc = check_device_error(p))) return rc;
    *token_out = p->h_ids[0];
    if (info) for (int k = 0; k < 4; k++) info[k] = greedy ? 0 : p->h_ids[1 + k];
    return B200_OK;
}

int b200_forward_prefill(b200_plan *p, int32_t token, int32_t position) {
    if (!p) return B200_ERR_BAD_ARG;
    if (!p->g_prefill) return fail(p, B200_ERR_STATE, "tensor-parallel plan: call b200_tp_attach on every rank first");
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
    if (!p->g_prefill) return fail(p, B200_ERR_STATE, "tensor-parallel plan: call b200_tp_attach on every rank first");
    if (p->prefill_batch > 1 && n > p->prefill_batch) return fail(p, B200_ERR_BAD_ARG, "chunk of %d tokens exceeds prefill_batch_size %d", n, p->prefill_batch);
    if (start_pos < 0 || start_pos + n > p->cfg.context_length) return fail(p, B200_ERR_BAD_ARG, "positions %d..%d outside the KV cache", start_pos, start_pos + n - 1);
    for (int i = 0; i < n; i++)
        if (tokens[i] < 0 || tokens[i] >= p->cfg.vocab_size) return fail(p, B200_ERR_BAD_ARG, "token %d out of range", tokens[i]);
    CK(cudaSetDevice(p->device));
    if ((p->prefill.ready && p->prefill.mode == B200_PREFILL_TENSOR_CORE) ||
        (p->prefill.q8_ready && p->prefill.mode == B200_PREFILL_TENSOR_CORE_W8A16)) { // tensor-core GEMM path (prefill.cuh)
        memcpy(p->h_ids, tokens, (size_t)n * 4);
        CK(cudaMemcpyAsync(p->prefill.tok, p->h_ids, (size_t)n * 4, cudaMemcpyHostToDevice, p->stream));
        CK(cudaEventRecord(p->ev0, p->stream));
        int rc2 = prefill_forward(p, n, start_pos, &p->launches_prefill);
        if (rc2) return rc2;
        CK(cudaEventRecord(p->ev1, p->stream));
        CK(cudaStreamSynchronize(p->stream));
        CK(cudaEventElapsedTime(&p->prefill_ms, p->ev0, p->ev1));
        return B200_OK;
    }
    // Exact path (bit-identical KV cache to the CPU batchForwardJavaPrefill, InferenceCoreBatchPrefillDecode.java:62-168).  Plans
    // that run multi-position steps take positions start .. start + n - 2 in steps of batch_max_rows rows into the plan's cache;
    // the last token, and every token elsewhere, runs through the single-token prefill graph, with the step state as the
    // token-by-token loop leaves it before its last step.
    if (n > p->seq_cap) return fail(p, B200_ERR_BAD_ARG, "chunk too long");
    memcpy(p->h_ids, tokens, (size_t)n * 4);
    CK(cudaMemcpyAsync(p->seq_tokens, p->h_ids, (size_t)n * 4, cudaMemcpyHostToDevice, p->stream));
    int rc, first = 0;
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

int b200_decode_sequence(b200_plan *p, const int32_t *tokens, int32_t n, int32_t start_pos, int32_t feedback,
                         int32_t *out_ids, float *device_ms) {
    if (!p || !tokens) return B200_ERR_BAD_ARG;
    if (n <= 0) return B200_OK;
    if (!p->g_decode) return fail(p, B200_ERR_STATE, "tensor-parallel plan: call b200_tp_attach on every rank first");
    if (n > p->seq_cap) return fail(p, B200_ERR_BAD_ARG, "sequence of %d steps exceeds capacity %d", n, p->seq_cap);
    if (start_pos < 0 || start_pos + n > p->cfg.context_length) return fail(p, B200_ERR_BAD_ARG, "positions %d..%d outside the KV cache (%d)", start_pos, start_pos + n - 1, p->cfg.context_length);
    int nt = feedback ? 1 : n;
    for (int i = 0; i < nt; i++)
        if (tokens[i] < 0 || tokens[i] >= p->cfg.vocab_size) return fail(p, B200_ERR_BAD_ARG, "token %d out of range", tokens[i]);
    CK(cudaSetDevice(p->device));
    memcpy(p->h_ids, tokens, (size_t)nt * 4);
    CK(cudaMemcpyAsync(p->seq_tokens, p->h_ids, (size_t)nt * 4, cudaMemcpyHostToDevice, p->stream));
    int rc;
    if ((rc = set_state(p, tokens[0], start_pos, nt, feedback))) return rc;
    CK(cudaEventRecord(p->ev0, p->stream));
    for (int i = 0; i < n; i++) CK(cudaGraphLaunch(decode_graph(p), p->stream));
    CK(cudaEventRecord(p->ev1, p->stream));
    if (out_ids) CK(cudaMemcpyAsync(p->h_ids, p->out_ids, (size_t)n * 4, cudaMemcpyDeviceToHost, p->stream));
    CK(cudaStreamSynchronize(p->stream));
    if ((rc = check_device_error(p))) return rc;
    if (out_ids) memcpy(out_ids, p->h_ids, (size_t)n * 4);
    if (device_ms) CK(cudaEventElapsedTime(device_ms, p->ev0, p->ev1));
    return B200_OK;
}

int b200_set_decode_mode(b200_plan *p, int32_t mode) {
    if (!p || (mode != B200_DECODE_GRAPH && mode != B200_DECODE_PERSISTENT)) return B200_ERR_BAD_ARG;
    if (!p->g_decode) return fail(p, B200_ERR_STATE, "tensor-parallel plan: call b200_tp_attach on every rank first");
    if (mode == B200_DECODE_PERSISTENT && !p->pd_ok) return fail(p, B200_ERR_UNSUPPORTED, "%s", p->pd_why.c_str());
    p->decode_mode = mode;
    return B200_OK;
}

int b200_decode_info(b200_plan *p, int32_t *mode, int32_t *launches, int32_t *ring_stages, int32_t *smem_bytes) {
    if (!p) return B200_ERR_BAD_ARG;
    const bool pers = p->decode_mode == B200_DECODE_PERSISTENT && p->g_pdecode;
    if (mode) *mode = pers ? B200_DECODE_PERSISTENT : B200_DECODE_GRAPH;
    if (launches) *launches = pers ? 1 : p->launches_decode;
    if (ring_stages) *ring_stages = p->pd_ok ? p->pd_L.stages : 0;
    if (smem_bytes) *smem_bytes = p->pd_ok ? (int32_t)p->pd_L.total : 0;
    return B200_OK;
}

int b200_trace_persistent(b200_plan *p, int32_t token, int32_t position, uint64_t *stamps, int64_t cap, int32_t *n_ctas, int32_t *n_rows, int32_t *n_stamps) {
    if (!p || !stamps) return B200_ERR_BAD_ARG;
    if (!p->g_ptrace) return fail(p, B200_ERR_UNSUPPORTED, "%s", p->pd_ok ? "no traced persistent graph" : p->pd_why.c_str());
    int rc;
    if ((rc = check_pos(p, token, position))) return rc;
    CK(cudaSetDevice(p->device));
    const size_t words = (size_t)p->n_sms * (p->cfg.n_layers + 1) * PD_STAMPS;
    if ((size_t)cap < words) return fail(p, B200_ERR_BAD_ARG, "stamp buffer too small: need %zu uint64", words);
    CK(cudaMemsetAsync(p->pd_trace, 0, words * 8, p->stream));
    if ((rc = set_state(p, token, position, 0, 0))) return rc;
    CK(cudaGraphLaunch(p->g_ptrace, p->stream));
    CK(cudaStreamSynchronize(p->stream));
    if ((rc = check_device_error(p))) return rc;
    CK(cudaMemcpy(stamps, p->pd_trace, words * 8, cudaMemcpyDeviceToHost));
    if (n_ctas) *n_ctas = p->n_sms;
    if (n_rows) *n_rows = p->cfg.n_layers + 1;
    if (n_stamps) *n_stamps = PD_STAMPS;
    return B200_OK;
}

int b200_set_prefill_mode(b200_plan *p, int32_t mode) {
    if (!p || (mode != B200_PREFILL_EXACT && mode != B200_PREFILL_TENSOR_CORE && mode != B200_PREFILL_TENSOR_CORE_W8A16)) return B200_ERR_BAD_ARG;
    if (p->is_moe && mode != B200_PREFILL_EXACT) return fail(p, B200_ERR_UNSUPPORTED, "%s", MOE_PREFILL_WHY);
    if (mode == B200_PREFILL_TENSOR_CORE_W8A16) {
        if (!p->prefill.q8_ready) {
            CK(cudaSetDevice(p->device));
            int rc = prefill_init_q8(p);
            if (rc) return rc;
            if (!p->prefill.q8_ready) return fail(p, B200_ERR_UNSUPPORTED, "%s", p->prefill.why_q8);
        }
        p->prefill.mode = mode;
        return B200_OK;
    }
    if (mode == B200_PREFILL_TENSOR_CORE && !p->prefill.ready && p->prefill_batch > 1 && p->wtype == B200_GGML_Q8_0 && p->use_stream && p->cfg.tp_size == 1) {
        CK(cudaSetDevice(p->device)); // opt-in on a Q8_0 plan: build the f16 twins, then the GEMM context
        int rc = build_f16_twins(p);
        if (rc) return rc;
        if ((rc = prefill_init(p))) return rc;
    }
    if (mode == B200_PREFILL_TENSOR_CORE && !p->prefill.ready) return fail(p, B200_ERR_UNSUPPORTED, "%s", p->prefill.why);
    p->prefill.mode = mode;
    return B200_OK;
}

int b200_prefill_info(b200_plan *p, int32_t *mode, int32_t *launches, float *device_ms) {
    if (!p) return B200_ERR_BAD_ARG;
    if (mode) *mode = p->prefill.ready || p->prefill.q8_ready ? p->prefill.mode : B200_PREFILL_EXACT;
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
    CK(cudaStreamSynchronize(p->stream));
    return B200_OK;
}

int b200_set_decode_slots(b200_plan *p, int32_t n_slots) {
    if (!p) return B200_ERR_BAD_ARG;
    if (n_slots < 0) return fail(p, B200_ERR_BAD_ARG, "n_slots must be >= 0");
    CK(cudaSetDevice(p->device));
    CK(cudaStreamSynchronize(p->stream));
    if (n_slots == 0) { batch_free(p); return B200_OK; }
    if (p->is_moe) return fail(p, B200_ERR_UNSUPPORTED, "batched decode has no Qwen2-MoE layer (MoE plans decode one sequence per step)");
    if (p->cfg.tp_size > 1) return fail(p, B200_ERR_UNSUPPORTED, "batched decode runs on single-GPU plans only (this plan is tensor-parallel)");
    if (p->wtype != B200_GGML_Q8_0) return fail(p, B200_ERR_UNSUPPORTED, "batched decode needs Q8_0 weights (FP16 plans decode one sequence per step)");
    if (!p->use_stream) return fail(p, B200_ERR_UNSUPPORTED, "batched decode needs the Q8_0 streaming layout (this plan uses the non-streaming matvecs)");
    const int mx = batch_max_rows(p);
    if (n_slots > mx) return fail(p, B200_ERR_UNSUPPORTED, "at most %d decode slots on this plan (asked for %d)", mx, n_slots);
    batch_free(p);
    const int rc = batch_alloc(p, n_slots);
    if (rc) { batch_free(p); return rc; }
    return B200_OK;
}

int b200_forward_decode_batch(b200_plan *p, int32_t n, const int32_t *slots, const int32_t *tokens, const int32_t *positions, const float *sampling,
                              int32_t *ids_out, float *logits) {
    if (!p) return B200_ERR_BAD_ARG;
    auto &B = p->bt;
    if (!B.n_slots) return fail(p, B200_ERR_STATE, "no decode slots: call b200_set_decode_slots first");
    if (!slots || !tokens || !positions || !ids_out) return fail(p, B200_ERR_BAD_ARG, "slots, tokens, positions and ids_out must not be NULL");
    if (n < 1 || n > B.n_slots) return fail(p, B200_ERR_BAD_ARG, "n = %d rows: need 1 <= n <= %d (the plan's decode slots)", n, B.n_slots);
    const b200_config &c = p->cfg;
    for (int i = 0; i < n; i++) {
        if (slots[i] < 0 || slots[i] >= B.n_slots) return fail(p, B200_ERR_BAD_ARG, "row %d: slot %d out of range (%d slots)", i, slots[i], B.n_slots);
        for (int j = 0; j < i; j++)
            if (slots[j] == slots[i]) return fail(p, B200_ERR_BAD_ARG, "row %d: slot %d repeats row %d's", i, slots[i], j);
        if (tokens[i] < 0 || tokens[i] >= c.vocab_size) return fail(p, B200_ERR_BAD_ARG, "row %d: token %d out of range", i, tokens[i]);
        if (positions[i] < 0 || positions[i] >= c.context_length)
            return fail(p, B200_ERR_BAD_ARG, "row %d: position %d outside the KV cache (%d)", i, positions[i], c.context_length);
        if (sampling) {
            const float t = sampling[3 * i], u = sampling[3 * i + 2];
            if (!(t >= 0.0f) || !(u >= 0.0f && u < 1.0f))
                return fail(p, B200_ERR_BAD_ARG, "row %d: temperature must be >= 0 and the uniform number in [0, 1)", i);
        }
    }
    CK(cudaSetDevice(p->device));
    int rc;
    if (!B.g[n] && (rc = capture_batch(p, n))) return rc;
    for (int i = 0; i < n; i++) { B.h_rows->token[i] = tokens[i]; B.h_rows->pos[i] = positions[i]; B.h_rows->slot[i] = slots[i]; }
    CK(cudaMemcpyAsync(B.rows, B.h_rows, sizeof(BatchRows), cudaMemcpyHostToDevice, p->stream));
    CK(cudaEventRecord(p->ev0, p->stream));
    CK(cudaGraphLaunch(B.g[n], p->stream));
    CK(cudaEventRecord(p->ev1, p->stream));
    const size_t vpad = (size_t)sampler_padded(c.vocab_size);
    if (logits) // before the sampler turns sampled rows into probabilities
        for (int i = 0; i < n; i++) CK(cudaMemcpyAsync(logits + (size_t)i * c.vocab_size, B.logits + i * vpad, (size_t)c.vocab_size * 4, cudaMemcpyDeviceToHost, p->stream));
    bool any_sampled = false;
    for (int i = 0; i < n; i++) {
        if (!sampling || sampling[3 * i] == 0.0f) continue; // Sampler.selectSampler: temperature 0 -> FloatTensor.argmax, already computed
        static bool attr = false;
        if (!attr) { CK(cudaFuncSetAttribute(k_sample, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sampler_smem_bytes())); attr = true; }
        SamplerArgs a;
        a.logits = B.logits + i * vpad; a.n = c.vocab_size; a.temperature = sampling[3 * i]; a.topp = sampling[3 * i + 1]; a.r01 = sampling[3 * i + 2];
        a.indices = p->smp_indices; a.out_id = B.smp_out + 8 * i; a.info = B.smp_out + 8 * i + 1;
        k_sample<<<1, SAMPLER_THREADS, sampler_smem_bytes(), p->stream>>>(a);
        CK(cudaGetLastError());
        any_sampled = true;
    }
    CK(cudaMemcpyAsync(B.h_out, B.ids, (size_t)n * 4, cudaMemcpyDeviceToHost, p->stream));
    if (any_sampled) CK(cudaMemcpyAsync(B.h_out + SMB_MAX_ROWS, B.smp_out, (size_t)n * 8 * 4, cudaMemcpyDeviceToHost, p->stream));
    CK(cudaStreamSynchronize(p->stream));
    for (int i = 0; i < n; i++) ids_out[i] = (sampling && sampling[3 * i] != 0.0f) ? B.h_out[SMB_MAX_ROWS + 8 * i] : B.h_out[i];
    CK(cudaEventElapsedTime(&B.last_ms, p->ev0, p->ev1));
    B.last_n = n;
    return B200_OK;
}

int b200_slot_reset(b200_plan *p, int32_t slot) {
    if (!p) return B200_ERR_BAD_ARG;
    if (slot < 0 || slot >= p->bt.n_slots) return fail(p, B200_ERR_BAD_ARG, "slot %d out of range (%d slots)", slot, p->bt.n_slots);
    CK(cudaSetDevice(p->device));
    const size_t kv = (size_t)p->cfg.n_layers * p->cfg.context_length * p->kvd;
    CK(cudaMemsetAsync(p->bt.slot_k + (size_t)slot * kv, 0, kv * 4, p->stream));
    CK(cudaMemsetAsync(p->bt.slot_v + (size_t)slot * kv, 0, kv * 4, p->stream));
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

// Tensor-core b200_prefill_slots: one chunk of the concatenated tokens (call order, no padding).  Sequence i's f16 K / V region
// holds its rows [0, start + len) from scratch row hrow[i]; sequences of length 0 take no part.
int prefill_slots_tc(b200_plan *p, int ns, const int *slots, const int *start, const int *len, const int *off, const int *tokens, int total) {
    PrefillCtx &c = p->prefill;
    const b200_config &g = p->cfg;
    std::vector<int> n, st, row0, hrow;
    std::vector<PfTok> tok(total);
    std::vector<PfHist> hist;
    size_t rows = 0;
    int max_start = 0;
    for (int i = 0; i < ns; i++) {
        if (!len[i]) continue;
        n.push_back(len[i]); st.push_back(start[i]); row0.push_back(off[i]); hrow.push_back((int)rows);
        for (int j = 0; j < len[i]; j++) tok[off[i] + j] = PfTok{start[i] + j, slots[i], (int)rows + start[i] + j};
        if (start[i] > 0) {
            hist.push_back(PfHist{slots[i], start[i], (int)rows});
            if (start[i] > max_start) max_start = start[i];
        }
        rows += (size_t)start[i] + len[i];
    }
    const std::vector<PfTile> tiles = pf_tiles((int)n.size(), n.data(), st.data(), row0.data(), hrow.data(), g.n_heads / g.n_kv_heads);
    CK(cudaStreamSynchronize(p->stream)); // the buffers below may be reallocated
    PfPacked pk{};
    pk.KH = c.KH; pk.VH = c.VH;
    if (rows > (size_t)g.context_length) { // more than one sequence's worth: the grown regions
        if (rows > c.pk_rows) {
            CK(cudaFree(c.PKH)); CK(cudaFree(c.PVH));
            c.PKH = c.PVH = nullptr; c.pk_rows = 0;
            CK(cudaMalloc(&c.PKH, rows * p->kvd * 2));
            CK(cudaMalloc(&c.PVH, rows * p->kvd * 2));
            c.pk_rows = rows;
        }
        pk.KH = c.PKH; pk.VH = c.PVH;
    }
    auto up16 = [](size_t x) { return (x + 15) & ~(size_t)15; };
    const size_t o_tiles = up16(tok.size() * sizeof(PfTok)), o_hist = o_tiles + up16(tiles.size() * sizeof(PfTile));
    const size_t bytes = o_hist + hist.size() * sizeof(PfHist) + 16;
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
    CK(cudaMemcpyAsync(c.ptab, h.data(), bytes, cudaMemcpyHostToDevice, p->stream));
    pk.tok = reinterpret_cast<const PfTok *>(c.ptab);
    pk.tiles = reinterpret_cast<const PfTile *>(c.ptab + o_tiles);
    pk.n_tiles = (int)tiles.size();
    pk.hist = reinterpret_cast<const PfHist *>(c.ptab + o_hist);
    pk.n_hist = (int)hist.size();
    pk.max_start = max_start;
    // pageable sources: both copies are staged before cudaMemcpyAsync returns (the pinned p->h_ids holds one sequence's worth)
    CK(cudaMemcpyAsync(c.tok, tokens, (size_t)total * 4, cudaMemcpyHostToDevice, p->stream));
    CK(cudaEventRecord(p->ev0, p->stream));
    int rc = prefill_forward(p, total, 0, &p->launches_prefill, &pk);
    if (rc) return rc;
    CK(cudaEventRecord(p->ev1, p->stream));
    CK(cudaStreamSynchronize(p->stream));
    CK(cudaEventElapsedTime(&p->prefill_ms, p->ev0, p->ev1));
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
        for (int j = 0; j < lengths[i]; j++)
            if (tokens[off[i] + j] < 0 || tokens[off[i] + j] >= c.vocab_size)
                return fail(p, B200_ERR_BAD_ARG, "sequence %d: token %d (index %d) out of range", i, tokens[off[i] + j], j);
    const PrefillCtx &pc = p->prefill;
    const bool tc = (pc.ready && pc.mode == B200_PREFILL_TENSOR_CORE) || (pc.q8_ready && pc.mode == B200_PREFILL_TENSOR_CORE_W8A16);
    if (tc && total > p->prefill_batch) {
        int i = 0;
        while (off[i] + lengths[i] <= p->prefill_batch) i++;
        return fail(p, B200_ERR_BAD_ARG, "sequence %d: the call's %lld tokens exceed prefill_batch_size %d (split the prompts into chunks)", i, (long long)total,
                    p->prefill_batch);
    }
    if (!total) return B200_OK;
    CK(cudaSetDevice(p->device));
    return tc ? prefill_slots_tc(p, n_seqs, slots, start_positions, lengths, off.data(), tokens, (int)total)
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
    for (int i = 0; i < n; i++) {
        if (tokens[i] < 0 || tokens[i] >= c.vocab_size) return fail(p, B200_ERR_BAD_ARG, "row %d: token %d out of range", i, tokens[i]);
        if (start_pos < 0 || (int64_t)start_pos + i >= c.context_length)
            return fail(p, B200_ERR_BAD_ARG, "row %d: position %lld outside the KV cache (%d)", i, (long long)start_pos + i, c.context_length);
    }
    CK(cudaSetDevice(p->device));
    int rc;
    if ((rc = multi_ready(p))) return rc;
    const bool own = slot < 0;
    if (!B.gs[own][1][n] && (rc = capture_batch(p, n, false, true, own))) return rc;
    for (int i = 0; i < n; i++) { B.h_rows->token[i] = tokens[i]; B.h_rows->pos[i] = start_pos + i; B.h_rows->slot[i] = own ? 0 : slot; }
    CK(cudaMemcpyAsync(B.rows, B.h_rows, sizeof(BatchRows), cudaMemcpyHostToDevice, p->stream));
    CK(cudaGraphLaunch(B.gs[own][1][n], p->stream));
    const size_t vpad = (size_t)sampler_padded(c.vocab_size);
    if (logits)
        for (int i = 0; i < n; i++) CK(cudaMemcpyAsync(logits + (size_t)i * c.vocab_size, B.logits + i * vpad, (size_t)c.vocab_size * 4, cudaMemcpyDeviceToHost, p->stream));
    CK(cudaMemcpyAsync(B.h_out, B.ids, (size_t)n * 4, cudaMemcpyDeviceToHost, p->stream));
    CK(cudaStreamSynchronize(p->stream));
    memcpy(ids_out, B.h_out, (size_t)n * 4);
    return B200_OK;
}

int b200_batch_info(b200_plan *p, int32_t *n_slots, int32_t *launches_per_step, float *device_ms_last_step) {
    if (!p) return B200_ERR_BAD_ARG;
    if (n_slots) *n_slots = p->bt.n_slots;
    if (launches_per_step) *launches_per_step = p->bt.last_n ? p->bt.launches[p->bt.last_n] : 0;
    if (device_ms_last_step) *device_ms_last_step = p->bt.last_ms;
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
    else if (s == "moe_ids" || s == "moe_weights") {
        if (!p->is_moe) return fail(p, B200_ERR_BAD_ARG, "%s: not a Qwen2-MoE plan", name);
        const size_t k = (size_t)p->moe.n_experts_used;
        if (s == "moe_ids") { src = p->moe_ids; sz = (size_t)c.n_layers * k * 4; }
        else { src = p->moe_w; sz = (size_t)c.n_layers * (k + 1) * 4; }
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
        if (!pc.ready && !pc.q8_ready) return fail(p, B200_ERR_STATE, "%s: the plan has no tensor-core prefill buffers (%s)", name, pc.why);
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
    if (p->is_moe) return fail(p, B200_ERR_UNSUPPORTED, "b200_time_kernel times the dense FFN and attention matrices; a Qwen2-MoE plan has no dense FFN");
    const b200_config &c = p->cfg;
    const bool q8 = p->wtype == B200_GGML_Q8_0;
    CK(cudaSetDevice(p->device));
    std::vector<float> save(c.dim);
    CK(cudaStreamSynchronize(p->stream));
    CK(cudaMemcpy(save.data(), p->x, (size_t)c.dim * 4, cudaMemcpyDeviceToHost));
    if (p->use_stream) {
        auto tb = [&](const TileMat &m) -> int64_t { return (int64_t)m.rows * m.cols / 32 * 34; };
        int64_t bytes = 0;
        int launches = 0, rc;
        auto one = [&](int l) -> int {
            LayerW &L = p->layers[l];
            bool keep = p->use_pdl;
            p->use_pdl = false;
            int r;
            const bool fz = p->fuse_norm;
            const int64_t nw = fz ? (int64_t)c.dim * 4 : 0; // a fused norm also reads its weights (x: an L2 hit)
            switch (which) {
            case 0:
                bytes = tb(L.tgu) + nw;
                r = fz ? launch_stream_norm<SMV_GATEUP>(p, L.tgu, L.ffn_norm, false, p->hb, p->hq, p->hs, false, TraceBuf{nullptr, 0, 0})
                       : launch_stream<SMV_GATEUP>(p, L.tgu, p->xq, p->xs, p->hb, p->hq, p->hs);
                break;
            case 1: bytes = tb(L.tw2); r = launch_stream<SMV_RESID>(p, L.tw2, p->hq, p->hs, p->x, nullptr, nullptr); break;
            case 2:
                bytes = tb(L.tqkv) + nw;
                r = fz ? launch_stream_norm<SMV_STORE>(p, L.tqkv, L.attn_norm, false, p->qkv, nullptr, nullptr, false, TraceBuf{nullptr, 0, 0})
                       : launch_stream<SMV_STORE>(p, L.tqkv, p->xq, p->xs, p->qkv, nullptr, nullptr);
                break;
            case 3: bytes = tb(L.two); r = launch_stream<SMV_RESID>(p, L.two, p->xq, p->xs, p->x, nullptr, nullptr); break;
            default:
                bytes = tb(p->tout) + nw;
                r = fz ? launch_stream_norm<SMV_STORE>(p, p->tout, p->out_norm, false, p->logits, nullptr, nullptr, false, TraceBuf{nullptr, 0, 0})
                       : launch_stream<SMV_STORE>(p, p->tout, p->xq, p->xs, p->logits, nullptr, nullptr);
                break;
            }
            p->use_pdl = keep;
            return r;
        };
        if (which < 0 || which > 4) return fail(p, B200_ERR_BAD_ARG, "unknown kernel id %d", which);
        for (int l = 0; l < c.n_layers; l++) if ((rc = one(l))) return rc;
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
    auto mat_bytes = [&](const DevMat &m) -> int64_t {
        int64_t e = (int64_t)m.rows * m.cols;
        return q8 ? e / 32 * 34 : e * 2;
    };
    int64_t bytes = 0;
    int launches = 0;
    const bool sf = p->use_f16_stream;
    auto one = [&](int l) -> int {
        LayerW &L = p->layers[l];
        if (sf) { // FP16 streaming kernels, stand-alone (no PDL overlap)
            const bool keep = p->use_pdl;
            p->use_pdl = false;
            int r;
            switch (which) {
            case 0: bytes = mat_bytes(L.w1) + mat_bytes(L.w3); r = launch_stream_f16<SF_GATEUP>(p, L.w1, &L.w3, p->xb, p->hb); break;
            case 1: bytes = mat_bytes(L.w2); r = launch_stream_f16<SF_RESID>(p, L.w2, nullptr, p->hb, p->x); break;
            case 2: bytes = mat_bytes(L.qkv); r = launch_stream_f16<SF_STORE>(p, L.qkv, nullptr, p->xb, p->qkv); break;
            case 3: bytes = mat_bytes(L.wo); r = launch_stream_f16<SF_RESID>(p, L.wo, nullptr, p->xb, p->x); break;
            default: bytes = mat_bytes(p->out); r = launch_stream_f16<SF_STORE>(p, p->out, nullptr, p->xb, p->logits); break;
            }
            p->use_pdl = keep;
            return r;
        }
        switch (which) {
        case 0:
            if (q8) {
                k_gateup_q8<<<c.hidden_dim / 32, 256, q8_smem_bytes(c.dim, 4, 8), p->stream>>>(
                    (const int8_t *)L.w1.qs, L.w1.sc, (const int8_t *)L.w3.qs, L.w3.sc, p->xq, p->xs, c.hidden_dim, c.dim, p->hq, p->hs, p->hb);
                CK(cudaGetLastError());
            } else {
                int rc;
                if ((rc = launch_matvec_f16<MODE_STORE>(p, L.w1, p->xb, p->hb))) return rc;
                if ((rc = launch_matvec_f16<MODE_STORE>(p, L.w3, p->xb, p->hb2))) return rc;
            }
            bytes = mat_bytes(L.w1) + mat_bytes(L.w3);
            return B200_OK;
        case 1: bytes = mat_bytes(L.w2); return q8 ? launch_matvec_q8<MODE_RESID>(p, L.w2, p->hq, p->hs, p->x) : launch_matvec_f16<MODE_RESID>(p, L.w2, p->hb, p->x);
        case 2: bytes = mat_bytes(L.qkv); return q8 ? launch_matvec_q8<MODE_STORE>(p, L.qkv, p->xq, p->xs, p->qkv) : launch_matvec_f16<MODE_STORE>(p, L.qkv, p->xb, p->qkv);
        case 3: bytes = mat_bytes(L.wo); return q8 ? launch_matvec_q8<MODE_RESID>(p, L.wo, p->xq, p->xs, p->x) : launch_matvec_f16<MODE_RESID>(p, L.wo, p->xb, p->x);
        default: bytes = mat_bytes(p->out); return q8 ? launch_matvec_q8<MODE_STORE>(p, p->out, p->xq, p->xs, p->logits) : launch_matvec_f16<MODE_STORE>(p, p->out, p->xb, p->logits);
        }
    };
    if (which < 0 || which > 4) return fail(p, B200_ERR_BAD_ARG, "unknown kernel id %d", which);
    int rc;
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
    if (!p->g_trace) return fail(p, B200_ERR_UNSUPPORTED, "tracing needs a streaming path (Q8_0 tiles or the FP16 rings)");
    int rc;
    if ((rc = check_pos(p, token, position))) return rc;
    CK(cudaSetDevice(p->device));
    int n = p->launches_decode;
    std::vector<unsigned long long> init((size_t)n * 4);
    for (int i = 0; i < n; i++) { init[i * 4] = 0; init[i * 4 + 1] = ~0ull; init[i * 4 + 2] = 0; init[i * 4 + 3] = 0; }
    CK(cudaMemcpyAsync(p->trace_rec, init.data(), init.size() * 8, cudaMemcpyHostToDevice, p->stream));
    if ((rc = set_state(p, token, position, 0, 0))) return rc;
    CK(cudaGraphLaunch(p->g_trace, p->stream));
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
    if (!terms || !out || n <= 0 || n > 8192) return B200_ERR_BAD_ARG;
    if (threads != 256 && threads != 512 && threads != 1024) return B200_ERR_BAD_ARG;
    float *d = nullptr, *o = nullptr;
    if (cudaMalloc(&d, (size_t)n * 4) != cudaSuccess) return B200_ERR_OOM;
    if (cudaMalloc(&o, 16) != cudaSuccess) { cudaFree(d); return B200_ERR_OOM; }
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
    cudaFree(d);
    cudaFree(o);
    return e == cudaSuccess ? B200_OK : B200_ERR_CUDA;
}

int b200_test_sample(const float *logits, int32_t n, float temperature, float topp, float uniform01, int32_t *token_out, int32_t *info, float *probs_out) {
    if (!logits || !token_out || n < 1) return B200_ERR_BAD_ARG;
    if (!(temperature > 0.0f) || !(uniform01 >= 0.0f && uniform01 < 1.0f)) return B200_ERR_BAD_ARG;
    const size_t padded = (size_t)sampler_padded(n) * 4;
    float *dl = nullptr;
    int *di = nullptr, *dout = nullptr;
    int rc = B200_OK;
    auto ok = [&](cudaError_t e) { if (e != cudaSuccess && rc == B200_OK) rc = e == cudaErrorMemoryAllocation ? B200_ERR_OOM : B200_ERR_CUDA; return rc == B200_OK; };
    // the index scratch starts as 0xFF bytes: a slot the kernel did not write in this call reads as -1
    if (ok(cudaMalloc(&dl, padded)) && ok(cudaMalloc(&di, (size_t)n * 4)) && ok(cudaMalloc(&dout, 8 * 4)) && ok(cudaMemset(dl, 0, padded)) &&
        ok(cudaMemcpy(dl, logits, (size_t)n * 4, cudaMemcpyHostToDevice)) && ok(cudaMemset(di, 0xFF, (size_t)n * 4)) && ok(cudaMemset(dout, 0xFF, 8 * 4)) &&
        ok(cudaFuncSetAttribute(k_sample, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sampler_smem_bytes()))) {
        SamplerArgs a;
        a.logits = dl; a.n = n; a.temperature = temperature; a.topp = topp; a.r01 = uniform01;
        a.indices = di; a.out_id = dout; a.info = dout + 1;
        k_sample<<<1, SAMPLER_THREADS, sampler_smem_bytes()>>>(a);
        int32_t h[5];
        if (ok(cudaGetLastError()) && ok(cudaDeviceSynchronize()) && ok(cudaMemcpy(h, dout, 5 * 4, cudaMemcpyDeviceToHost))) {
            *token_out = h[0];
            if (info) for (int k = 0; k < 4; k++) info[k] = h[1 + k];
            if (probs_out) ok(cudaMemcpy(probs_out, dl, (size_t)n * 4, cudaMemcpyDeviceToHost));
        }
    }
    cudaFree(dl); cudaFree(di); cudaFree(dout);
    return rc;
}

int b200_requant_kquant(int32_t ggml_type, const void *src, int64_t n_elems, void *dst_q8_0) {
    if (!src || !dst_q8_0 || n_elems <= 0 || n_elems % 256 || !kq_is_kquant(ggml_type)) return B200_ERR_BAD_ARG;
    const size_t raw = (size_t)(n_elems / 256) * kq_block_bytes(ggml_type), q8 = (size_t)(n_elems / 32) * 34;
    unsigned char *ds = nullptr, *dd = nullptr;
    int rc = B200_OK;
    auto ok = [&](cudaError_t e) { if (e != cudaSuccess && rc == B200_OK) rc = e == cudaErrorMemoryAllocation ? B200_ERR_OOM : B200_ERR_CUDA; return rc == B200_OK; };
    if (ok(cudaMalloc(&ds, raw)) && ok(cudaMalloc(&dd, q8)) && ok(cudaMemcpy(ds, src, raw, cudaMemcpyHostToDevice)) &&
        ok(launch_requant_kquant(ggml_type, ds, dd, n_elems / 32, 0)) && ok(cudaDeviceSynchronize()))
        ok(cudaMemcpy(dst_q8_0, dd, q8, cudaMemcpyDeviceToHost));
    cudaFree(ds); cudaFree(dd);
    return rc;
}

int b200_gemm_f16(const uint16_t *a, const uint16_t *b, float *c, int32_t m, int32_t n, int32_t k, int32_t iters, float *ms) {
    const int stages = getenv("B200_GEMM_STAGES") ? atoi(getenv("B200_GEMM_STAGES")) : 0;
    // B200_GEMM_RESID=s: the reduce-add epilogue with K split s ways; C starts at 0 and accumulates over the timed launches
    const int resid = getenv("B200_GEMM_RESID") ? atoi(getenv("B200_GEMM_RESID")) : 0;
    if (!a || !b || !c || m <= 0 || n <= 0 || k <= 0 || m % 128 || n % 128 || k % 64) return B200_ERR_BAD_ARG;
    __half *da = nullptr, *db = nullptr;
    float *dc = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    int rc = B200_OK;
    auto ok = [&](cudaError_t e) { if (e != cudaSuccess && rc == B200_OK) rc = e == cudaErrorMemoryAllocation ? B200_ERR_OOM : B200_ERR_CUDA; return rc == B200_OK; }; // first failure wins
    if (ok(cudaMalloc(&da, (size_t)m * k * 2)) && ok(cudaMalloc(&db, (size_t)n * k * 2)) && ok(cudaMalloc(&dc, (size_t)m * n * 4)) &&
        ok(cudaMemcpy(da, a, (size_t)m * k * 2, cudaMemcpyHostToDevice)) && ok(cudaMemcpy(db, b, (size_t)n * k * 2, cudaMemcpyHostToDevice)) &&
        ok(cudaMemset(dc, resid ? 0 : 0xFF, (size_t)m * n * 4))) {
        if (pg::gemm_f16(da, db, dc, m, n, k, stages, resid, 0)) rc = B200_ERR_CUDA;
        ok(cudaDeviceSynchronize());
        if (rc == B200_OK && iters > 0 && ms && ok(cudaEventCreate(&e0)) && ok(cudaEventCreate(&e1)) && ok(cudaEventRecord(e0, 0))) {
            for (int i = 0; i < iters && rc == B200_OK; i++)
                if (pg::gemm_f16(da, db, dc, m, n, k, stages, resid, 0)) rc = B200_ERR_CUDA;
            float t = 0.f;
            if (ok(cudaEventRecord(e1, 0)) && ok(cudaEventSynchronize(e1)) && ok(cudaEventElapsedTime(&t, e0, e1))) *ms = t / iters;
            if (rc == B200_OK && resid) { // C accumulated 1 + iters products: return exactly one
                if (ok(cudaMemset(dc, 0, (size_t)m * n * 4)) && pg::gemm_f16(da, db, dc, m, n, k, stages, resid, 0)) rc = B200_ERR_CUDA;
                ok(cudaDeviceSynchronize());
            }
        }
        if (rc == B200_OK) ok(cudaMemcpy(c, dc, (size_t)m * n * 4, cudaMemcpyDeviceToHost));
    }
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    cudaFree(da); cudaFree(db); cudaFree(dc);
    return rc;
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
    int rc = B200_OK;
    auto ok = [&](cudaError_t e) { if (e != cudaSuccess && rc == B200_OK) rc = e == cudaErrorMemoryAllocation ? B200_ERR_OOM : B200_ERR_CUDA; return rc == B200_OK; };
    if (ok(cudaMalloc(&da, (size_t)m * k * 2)) && ok(cudaMalloc(&db, (size_t)n * k * 2)) && (!gateup || ok(cudaMalloc(&db2, (size_t)n * k * 2))) &&
        ok(cudaMalloc(&dc, c_bytes)) && ok(cudaMemcpy(da, a, (size_t)m * k * 2, cudaMemcpyHostToDevice)) &&
        ok(cudaMemcpy(db, b, (size_t)n * k * 2, cudaMemcpyHostToDevice)) && (!gateup || ok(cudaMemcpy(db2, b2, (size_t)n * k * 2, cudaMemcpyHostToDevice))) &&
        ok(cudaMemcpy(dc, c, c_bytes, cudaMemcpyHostToDevice))) {
        // the same maps prefill_forward builds: A boxes of 128 rows, B boxes of 128 rows (64 for each half of the gate/up tile), C boxes 128 x 32 f32
        CUtensorMap ma, mb, mb2, mc;
        const uint32_t b_rows = gateup ? pg::BN / 2 : pg::BN;
        if (pg::make_map(&ma, da, (uint64_t)m, (uint64_t)k, pg::BM) || pg::make_map(&mb, db, (uint64_t)n, (uint64_t)k, b_rows) ||
            pg::make_map(&mb2, gateup ? db2 : db, (uint64_t)n, (uint64_t)k, b_rows) || (!gateup && pg::make_map_c(&mc, dc, (uint64_t)m, (uint64_t)n)))
            rc = B200_ERR_CUDA;
        if (gateup) mc = mb; // unused by the gate/up epilogue, which stores f16 through plain pointers
        int lr = 0;
        if (rc == B200_OK) {
            const int mt = m / pg::BM, nt = n / (gateup ? pg::BN / 2 : pg::BN);
            const bool deep = stages == pg::GEMM_STAGES_DEEP;
            if (mode == pg::GEMM_F32)
                lr = deep ? pg::gemm_launch<pg::GEMM_F32, pg::GEMM_STAGES_DEEP>(ma, mb, mb2, mc, dc, n, m_valid, mt, nt, k, 0, splits)
                          : pg::gemm_launch<pg::GEMM_F32, pg::GEMM_STAGES>(ma, mb, mb2, mc, dc, n, m_valid, mt, nt, k, 0, splits);
            else if (mode == pg::GEMM_RESID)
                lr = deep ? pg::gemm_launch<pg::GEMM_RESID, pg::GEMM_STAGES_DEEP>(ma, mb, mb2, mc, dc, n, m_valid, mt, nt, k, 0, splits)
                          : pg::gemm_launch<pg::GEMM_RESID, pg::GEMM_STAGES>(ma, mb, mb2, mc, dc, n, m_valid, mt, nt, k, 0, splits);
            else
                lr = deep ? pg::gemm_launch<pg::GEMM_GATEUP, pg::GEMM_STAGES_DEEP>(ma, mb, mb2, mc, dc, n, m_valid, mt, nt, k, 0, splits)
                          : pg::gemm_launch<pg::GEMM_GATEUP, pg::GEMM_STAGES>(ma, mb, mb2, mc, dc, n, m_valid, mt, nt, k, 0, splits);
            if (lr == -6) rc = B200_ERR_BAD_ARG; // splits > 1 outside GEMM_RESID, or a split with no k-block
            else if (lr) rc = B200_ERR_CUDA;
        }
        if (ok(cudaDeviceSynchronize()) && rc == B200_OK) ok(cudaMemcpy(c, dc, c_bytes, cudaMemcpyDeviceToHost));
    }
    cudaFree(da); cudaFree(db); cudaFree(db2); cudaFree(dc);
    return rc;
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
    int rc = B200_OK;
    auto ok = [&](cudaError_t e) { if (e != cudaSuccess && rc == B200_OK) rc = e == cudaErrorMemoryAllocation ? B200_ERR_OOM : B200_ERR_CUDA; return rc == B200_OK; };
    if (ok(cudaMalloc(&da, (size_t)m * k * 2)) && ok(cudaMalloc(&draw, q8_bytes * (gateup ? 2 : 1))) && ok(cudaMalloc(&dstream, stream_bytes)) &&
        ok(cudaMalloc(&dc, c_bytes)) && ok(cudaMemcpy(da, a, (size_t)m * k * 2, cudaMemcpyHostToDevice)) && ok(cudaMemcpy(draw, bq, q8_bytes, cudaMemcpyHostToDevice)) &&
        (!gateup || ok(cudaMemcpy(draw + q8_bytes, bq2, q8_bytes, cudaMemcpyHostToDevice))) && ok(cudaMemcpy(dc, c, c_bytes, cudaMemcpyHostToDevice))) {
        RepackSrc src{};
        src.raw[0] = draw;
        src.rows[0] = n;
        if (gateup) { src.raw[1] = draw + q8_bytes; src.rows[1] = n; }
        src.gateup = gateup ? 1 : 0;
        k_repack_tiles<<<(unsigned)((size_t)rows * nseg), 128>>>(src, dstream, rows, k, seg, nseg, unit);
        ok(cudaGetLastError());
        // the maps prefill_init_q8 builds and the A / C maps of the prefill scratch
        CUtensorMap ma, mq, ms, mc;
        if (rc == B200_OK && (pg::make_map(&ma, da, (uint64_t)m, (uint64_t)k, pg::BM) || pg::make_map_q8(&mq, dstream, (uint64_t)rows, nseg, unit, 0) ||
                              pg::make_map_q8(&ms, dstream, (uint64_t)rows, nseg, unit, 1) || (!gateup && pg::make_map_c(&mc, dc, (uint64_t)m, (uint64_t)n))))
            rc = B200_ERR_CUDA;
        if (gateup) mc = mq; // unused by the gate/up epilogue
        int lr = 0;
        if (rc == B200_OK) {
            using pg::B_Q8;
            constexpr int S4 = pg::GEMM_STAGES, S5 = pg::GEMM_STAGES_DEEP_Q8;
            const int mt = m / pg::BM, nt = n / (gateup ? pg::BN / 2 : pg::BN);
            const bool deep = stages == S5;
            if (mode == pg::GEMM_F32)
                lr = deep ? pg::gemm_launch<pg::GEMM_F32, S5, B_Q8>(ma, mq, ms, mc, dc, n, m_valid, mt, nt, k, 0, splits, seg)
                          : pg::gemm_launch<pg::GEMM_F32, S4, B_Q8>(ma, mq, ms, mc, dc, n, m_valid, mt, nt, k, 0, splits, seg);
            else if (mode == pg::GEMM_RESID)
                lr = deep ? pg::gemm_launch<pg::GEMM_RESID, S5, B_Q8>(ma, mq, ms, mc, dc, n, m_valid, mt, nt, k, 0, splits, seg)
                          : pg::gemm_launch<pg::GEMM_RESID, S4, B_Q8>(ma, mq, ms, mc, dc, n, m_valid, mt, nt, k, 0, splits, seg);
            else
                lr = deep ? pg::gemm_launch<pg::GEMM_GATEUP, S5, B_Q8>(ma, mq, ms, mc, dc, n, m_valid, mt, nt, k, 0, splits, seg)
                          : pg::gemm_launch<pg::GEMM_GATEUP, S4, B_Q8>(ma, mq, ms, mc, dc, n, m_valid, mt, nt, k, 0, splits, seg);
            if (lr == -6) rc = B200_ERR_BAD_ARG;
            else if (lr) rc = B200_ERR_CUDA;
        }
        if (ok(cudaDeviceSynchronize()) && rc == B200_OK) ok(cudaMemcpy(c, dc, c_bytes, cudaMemcpyDeviceToHost));
    }
    cudaFree(da); cudaFree(draw); cudaFree(dstream); cudaFree(dc);
    return rc;
}

int b200_test_pf_attention(const float *q, const float *k, const float *v, int32_t n, int32_t start_pos, int32_t n_heads, int32_t n_kv_heads,
                           int32_t head_size, int32_t out_rows, uint16_t *out) {
    if (!q || !k || !v || !out || n < 1 || start_pos < 0 || out_rows < n || n_kv_heads < 1 || n_heads % n_kv_heads) return B200_ERR_BAD_ARG;
    const int kv_mul = n_heads / n_kv_heads, hs = head_size;
    if ((hs != 64 && hs != 128) || kv_mul > 64) return B200_ERR_BAD_ARG; // what prefill_init accepts
    const int qd = n_heads * hs, kvd = n_kv_heads * hs, ldq = qd + 2 * kvd, nkeys = start_pos + n;
    const size_t kv_elems = (size_t)nkeys * kvd;
    float *dqkv = nullptr, *dk = nullptr, *dv = nullptr;
    __half *dkh = nullptr, *dvh = nullptr, *dout = nullptr;
    int rc = B200_OK;
    auto ok = [&](cudaError_t e) { if (e != cudaSuccess && rc == B200_OK) rc = e == cudaErrorMemoryAllocation ? B200_ERR_OOM : B200_ERR_CUDA; return rc == B200_OK; };
    // q sits in the q columns of a QKV row as after k_pf_rope_kv; the k / v columns hold NaN, which the kernels must never read
    if (ok(cudaMalloc(&dqkv, (size_t)n * ldq * 4)) && ok(cudaMalloc(&dk, kv_elems * 4)) && ok(cudaMalloc(&dv, kv_elems * 4)) &&
        ok(cudaMalloc(&dkh, kv_elems * 2)) && ok(cudaMalloc(&dvh, kv_elems * 2)) && ok(cudaMalloc(&dout, (size_t)out_rows * qd * 2)) &&
        ok(cudaMemset(dqkv, 0xFF, (size_t)n * ldq * 4)) && ok(cudaMemcpy2D(dqkv, (size_t)ldq * 4, q, (size_t)qd * 4, (size_t)qd * 4, n, cudaMemcpyHostToDevice)) &&
        ok(cudaMemcpy(dk, k, kv_elems * 4, cudaMemcpyHostToDevice)) && ok(cudaMemcpy(dv, v, kv_elems * 4, cudaMemcpyHostToDevice)) &&
        ok(cudaMemcpy(dout, out, (size_t)out_rows * qd * 2, cudaMemcpyHostToDevice))) {
        const float inv_sqrt_hs = (float)(1.0 / sqrt((double)hs));
        const int qt = PM_ROWS / kv_mul;
        const dim3 ag((n + qt - 1) / qt, n_kv_heads);
        // f16 K / V copies as prefill_forward makes them (k_pf_kv_to_f16 and k_pf_rope_kv round the same way)
        const size_t n4 = kv_elems / 4;
        k_pf_kv_to_f16<<<(unsigned)((n4 + 255) / 256 < 1184 ? (n4 + 255) / 256 : 1184), 256, 0, 0>>>(dk, dv, dkh, dvh, n4);
        if (hs == 128) {
            if (ok(cudaFuncSetAttribute(k_pf_attention_mma<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pm_smem_bytes<128>())))
                k_pf_attention_mma<128><<<ag, PM_THREADS, pm_smem_bytes<128>(), 0>>>(dqkv, ldq, dkh, dvh, kvd, kv_mul, n, start_pos, inv_sqrt_hs, dout, qd);
        } else {
            if (ok(cudaFuncSetAttribute(k_pf_attention_mma<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pm_smem_bytes<64>())))
                k_pf_attention_mma<64><<<ag, PM_THREADS, pm_smem_bytes<64>(), 0>>>(dqkv, ldq, dkh, dvh, kvd, kv_mul, n, start_pos, inv_sqrt_hs, dout, qd);
        }
        if (ok(cudaGetLastError()) && ok(cudaDeviceSynchronize())) ok(cudaMemcpy(out, dout, (size_t)out_rows * qd * 2, cudaMemcpyDeviceToHost));
    }
    cudaFree(dqkv); cudaFree(dk); cudaFree(dv); cudaFree(dkh); cudaFree(dvh); cudaFree(dout);
    return rc;
}

int b200_test_pf_attention_packed(int32_t n_seqs, const int32_t *lengths, const int32_t *start_positions, const float *q, const float *k, const float *v,
                                  int32_t n_heads, int32_t n_kv_heads, int32_t head_size, uint16_t *out) {
    if (!lengths || !start_positions || !q || !k || !v || !out || n_seqs < 1 || n_kv_heads < 1 || n_heads % n_kv_heads) return B200_ERR_BAD_ARG;
    const int kv_mul = n_heads / n_kv_heads, hs = head_size;
    if ((hs != 64 && hs != 128) || kv_mul > 64) return B200_ERR_BAD_ARG;
    const int qd = n_heads * hs, kvd = n_kv_heads * hs, ldq = qd + 2 * kvd;
    std::vector<int> row0(n_seqs), hrow(n_seqs);
    int n = 0, rows = 0;
    for (int i = 0; i < n_seqs; i++) {
        if (lengths[i] < 1 || start_positions[i] < 0) return B200_ERR_BAD_ARG;
        row0[i] = n; hrow[i] = rows;
        n += lengths[i]; rows += start_positions[i] + lengths[i];
    }
    const std::vector<PfTile> tiles = pf_tiles(n_seqs, lengths, start_positions, row0.data(), hrow.data(), kv_mul);
    const size_t kv_elems = (size_t)rows * kvd;
    float *dqkv = nullptr, *dk = nullptr, *dv = nullptr;
    __half *dkh = nullptr, *dvh = nullptr, *dout = nullptr;
    PfTile *dt = nullptr;
    int rc = B200_OK;
    auto ok = [&](cudaError_t e) { if (e != cudaSuccess && rc == B200_OK) rc = e == cudaErrorMemoryAllocation ? B200_ERR_OOM : B200_ERR_CUDA; return rc == B200_OK; };
    // q rows of every sequence back to back in the q columns of QKV rows, K / V rows [0, start + n) of each sequence back to back: the
    // layout b200_prefill_slots gives the packed kernel
    if (ok(cudaMalloc(&dqkv, (size_t)n * ldq * 4)) && ok(cudaMalloc(&dk, kv_elems * 4)) && ok(cudaMalloc(&dv, kv_elems * 4)) &&
        ok(cudaMalloc(&dkh, kv_elems * 2)) && ok(cudaMalloc(&dvh, kv_elems * 2)) && ok(cudaMalloc(&dout, (size_t)n * qd * 2)) &&
        ok(cudaMalloc(&dt, tiles.size() * sizeof(PfTile))) &&
        ok(cudaMemset(dqkv, 0xFF, (size_t)n * ldq * 4)) && ok(cudaMemcpy2D(dqkv, (size_t)ldq * 4, q, (size_t)qd * 4, (size_t)qd * 4, n, cudaMemcpyHostToDevice)) &&
        ok(cudaMemcpy(dk, k, kv_elems * 4, cudaMemcpyHostToDevice)) && ok(cudaMemcpy(dv, v, kv_elems * 4, cudaMemcpyHostToDevice)) &&
        ok(cudaMemcpy(dout, out, (size_t)n * qd * 2, cudaMemcpyHostToDevice)) &&
        ok(cudaMemcpy(dt, tiles.data(), tiles.size() * sizeof(PfTile), cudaMemcpyHostToDevice))) {
        const float inv_sqrt_hs = (float)(1.0 / sqrt((double)hs));
        const dim3 ag((unsigned)tiles.size(), n_kv_heads);
        const size_t n4 = kv_elems / 4;
        k_pf_kv_to_f16<<<(unsigned)((n4 + 255) / 256 < 1184 ? (n4 + 255) / 256 : 1184), 256, 0, 0>>>(dk, dv, dkh, dvh, n4);
        if (hs == 128) {
            if (ok(cudaFuncSetAttribute(k_pf_attention_mma_packed<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pm_smem_bytes<128>())))
                k_pf_attention_mma_packed<128><<<ag, PM_THREADS, pm_smem_bytes<128>(), 0>>>(dqkv, ldq, dkh, dvh, kvd, kv_mul, dt, inv_sqrt_hs, dout, qd);
        } else {
            if (ok(cudaFuncSetAttribute(k_pf_attention_mma_packed<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pm_smem_bytes<64>())))
                k_pf_attention_mma_packed<64><<<ag, PM_THREADS, pm_smem_bytes<64>(), 0>>>(dqkv, ldq, dkh, dvh, kvd, kv_mul, dt, inv_sqrt_hs, dout, qd);
        }
        if (ok(cudaGetLastError()) && ok(cudaDeviceSynchronize())) ok(cudaMemcpy(out, dout, (size_t)n * qd * 2, cudaMemcpyDeviceToHost));
    }
    cudaFree(dqkv); cudaFree(dk); cudaFree(dv); cudaFree(dkh); cudaFree(dvh); cudaFree(dout); cudaFree(dt);
    return rc;
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
    return (p->decode_mode == B200_DECODE_PERSISTENT && p->g_pdecode) ? 1 : p->launches_decode;
}
int64_t b200_device_bytes(b200_plan *p) { return p ? p->bytes : 0; }

void b200_plan_free(b200_plan *p) {
    if (!p) return;
    cudaSetDevice(p->device);
    if (p->stream) cudaStreamSynchronize(p->stream);
    prefill_free(p->prefill);
    batch_free(p);
    if (p->g_decode) cudaGraphExecDestroy(p->g_decode);
    if (p->g_prefill) cudaGraphExecDestroy(p->g_prefill);
    if (p->g_trace) cudaGraphExecDestroy(p->g_trace);
    if (p->g_pdecode) cudaGraphExecDestroy(p->g_pdecode);
    if (p->g_pprefill) cudaGraphExecDestroy(p->g_pprefill);
    if (p->g_ptrace) cudaGraphExecDestroy(p->g_ptrace);
    if (p->h_err) cudaFreeHost(p->h_err);
    for (int k = 0; k < TP_MAX; k++) if (p->peer_open[k]) cudaIpcCloseMemHandle(p->peer_open[k]);
    for (void *d : p->allocs) cudaFree(d);
    if (p->h_st) cudaFreeHost(p->h_st);
    if (p->h_ids) cudaFreeHost(p->h_ids);
    if (p->ev0) cudaEventDestroy(p->ev0);
    if (p->ev1) cudaEventDestroy(p->ev1);
    if (p->stream) cudaStreamDestroy(p->stream);
    delete p;
}

const char *b200_last_error(b200_plan *p) { return p ? p->err.c_str() : "null plan"; }
const char *b200_version(void) { return "b200llama 0.1 sm_90a"; }

} // extern "C"
