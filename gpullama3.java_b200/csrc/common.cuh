// common.cuh -- shared device helpers for libb200llama (sm_90a).
//
// Numerics contract: every kernel reproduces the float evaluation order of the reference's
// CPU path (see DESIGN.md "Exactness").  The translation unit is compiled with -fmad=false
// and, belt and braces, all order-sensitive arithmetic uses the __f*_rn intrinsics, which
// the compiler never contracts or reassociates.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define B200_WARP 32

// Device-resident step descriptor read by every kernel of the captured decode graph, so one
// graph serves every (token, position) and on-device greedy loops need no host round trip.
struct StepState {
    int token;    // token consumed by this step
    int pos;      // sequence position of this step
    int step;     // index into seq_tokens / out_ids
    int n_seq;    // number of valid entries in seq_tokens
    int feedback; // !=0: next token = this step's argmax (greedy generation)
    int pad[3];
};

// Programmatic dependent launch (PDL): launch_dependents lets the next kernel of the stream become
// resident early (it may only touch immutable weights until it executes pdl_wait, which blocks
// until the preceding kernel has completed and flushed).  Both are no-ops without the launch attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---- tensor parallelism over NVLink peer memory ------------------------------------------------
// Every rank owns ROWS of every matrix, so each dot product keeps its full sequential order and the
// results stay bit-identical to the single-GPU (and CPU) path; what would be an all-reduce becomes an
// all-gather: the producing kernel's epilogue stores its slice straight into every rank's
// communication buffer (peer-mapped via CUDA IPC) and then raises a monotonically increasing flag;
// the consuming kernel spins on the flags of all ranks.  n == 1 turns every helper into a no-op.
#define TP_MAX 8
enum { TP_SLOT_X = 0, TP_SLOT_ATT = 1, TP_SLOT_HQ = 2, TP_SLOT_ARG = 3, TP_SLOTS = 4 };
struct TpCtx {
    int rank, n;
    unsigned ops_per_fwd;          // 4 * layers + 1
    unsigned char *peer[TP_MAX];   // base of each rank's communication buffer (peer[rank] = own)
    unsigned off_x, off_attq, off_atts, off_hq, off_hs, off_pv, off_pi, off_flags, off_tick, off_done;
    unsigned *err;      // device word: != 0 once any wait of this plan gave up (every later wait returns at once)
    unsigned *host_err; // mapped pinned host alias the host checks after each synchronize
};
#define TP_TIMEOUT_NS 4000000000ull // a peer that has not signalled after 4 s is gone (or the ranks' call sequences diverged)
template <typename T> __device__ __forceinline__ T *tp_ptr(const TpCtx &t, int k, unsigned off) {
    return reinterpret_cast<T *>(t.peer[k] + off);
}
__device__ __forceinline__ unsigned tp_seq(const TpCtx &t, unsigned op) {
    const unsigned tick = *reinterpret_cast<volatile unsigned *>(t.peer[t.rank] + t.off_tick);
    return tick * t.ops_per_fwd + op + 1u;
}
__device__ __forceinline__ unsigned long long gtime_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// one thread; bounded: a rank that errored out or died must not leave the others spinning inside a captured graph
__device__ __noinline__ void tp_wait(const TpCtx &t, int slot, unsigned seq) {
    const unsigned *f = reinterpret_cast<const unsigned *>(t.peer[t.rank] + t.off_flags) + slot * TP_MAX;
    unsigned it = 0;
    unsigned long long t0 = 0;
    for (int k = 0; k < t.n; k++) {
        for (;;) {
            unsigned v; // relaxed polls, ONE acquire fence after the last flag: ld.acquire in the loop is a load + CCTL.IVALL (an L1 flush per poll)
            asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(f + k) : "memory");
            if ((int)(v - seq) >= 0) break;
            if ((++it & 255u) == 0u && t.err) {
                if (*reinterpret_cast<volatile unsigned *>(t.err)) return;
                const unsigned long long now = gtime_ns();
                if (!t0) t0 = now;
                else if (now - t0 > TP_TIMEOUT_NS) {
                    atomicCAS(t.err, 0u, 100u + (unsigned)slot);
                    *reinterpret_cast<volatile unsigned *>(t.host_err) = 100u + (unsigned)slot;
                    return;
                }
            }
        }
    }
    { // one acquire load after the relaxed polls (flags are monotone); a fence.acq_rel.sys here is a MEMBAR.SYS per wait
        unsigned v;
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(f) : "memory");
    }
}
__device__ __forceinline__ void tp_signal(const TpCtx &t, int slot, unsigned seq) { // one thread, after the data stores
    __threadfence_system();
    for (int k = 0; k < t.n; k++) {
        unsigned *f = reinterpret_cast<unsigned *>(t.peer[k] + t.off_flags) + slot * TP_MAX + t.rank;
        asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(f), "r"(seq) : "memory"); // ordered by the fence above
    }
}
// Grid-wide "last CTA signals": every CTA calls this (one thread, after a CTA barrier that follows the
// CTA's peer stores + __threadfence_system()); the last one to arrive raises the flag on every rank.
__device__ __forceinline__ void tp_cta_done(const TpCtx &t, int slot, unsigned seq, unsigned n_ctas) {
    unsigned *cnt = reinterpret_cast<unsigned *>(t.peer[t.rank] + t.off_done) + slot;
    __threadfence();
    if (atomicAdd(cnt, 1u) == n_ctas - 1u) {
        *cnt = 0u;
        tp_signal(t, slot, seq);
    }
}
__device__ __forceinline__ float ldcg_f32c(const float *p) {
    float v;
    asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(v) : "l"(p));
    return v;
}

// What the attention prologues do per architecture (the kernels take these flags, not the architecture id):
//   Llama / Mistral: interleaved-pair RoPE (InferenceCore.java:75-87); Qwen3: NeoX pairs + per-head q/k RMSNorm (:594-619);
//   Phi-3: NeoX pairs, no q/k norm (forwardJavaPhi3, :726-742); Qwen2: F32 biases added to q, k and v right after their matmuls
//   (q.addInPlace(q_bias) etc., :456-459), then NeoX pairs without q/k norm (:463-478).
//   Granite: the attention score is multiplied by the model's attentionScale instead of divided by sqrt(head size)
//   (forwardGranite, :868-873); the kernels' `sqrt_hs` argument then carries that multiplier.
#define KF_NEOX 1
#define KF_QKNORM 2
#define KF_QKVBIAS 4
#define KF_ATTSCALE 8

// In-graph timeline tracing (diagnostic graph only; rec == nullptr in the production graphs, so the
// branch is uniform and free).  One record per launch: {kernel id, earliest CTA entry, latest
// dependency-wait return, latest CTA exit} in %globaltimer nanoseconds.
struct TraceBuf {
    unsigned long long *rec;
    int slot, id;
};
__device__ __forceinline__ unsigned long long gtime() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void trace_entry(const TraceBuf &tr) {
    if (tr.rec && threadIdx.x == 0) { tr.rec[tr.slot * 4] = (unsigned long long)tr.id; atomicMin(&tr.rec[tr.slot * 4 + 1], gtime()); }
}
__device__ __forceinline__ void trace_mark(const TraceBuf &tr, int k) {
    if (tr.rec && threadIdx.x == 0) atomicMax(&tr.rec[tr.slot * 4 + k], gtime());
}

__device__ __forceinline__ float warp_max_f(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Activation quantisation of one 32-element block held one element per lane.
// Restates Q8_0FloatTensor.dotQ8Activation's per-block quantiser (Q8_0FloatTensor.java:100-117):
// amax -> qs = amax/127f -> aScale = f16 round trip of qs -> aInv = qs != 0 ? 1/qs : 0 ->
// aq = (int)(x*aInv + copySign(0.5f, .)).
__device__ __forceinline__ int quant_block_lane(float v, float &ascale) {
    float amax = warp_max_f(fabsf(v));
    float qs = __fdiv_rn(amax, 127.0f);
    ascale = __half2float(__float2half_rn(qs));
    float ainv = qs != 0.0f ? __fdiv_rn(1.0f, qs) : 0.0f;
    float s = __fmul_rn(v, ainv);
    return __float2int_rz(__fadd_rn(s, copysignf(0.5f, s)));
}

// One whole Q8_0 quant block (32 bytes) per lane as two 128-bit read-only streaming loads
// (sm_90 has no 256-bit global load).
__device__ __forceinline__ void ldg256_stream(const void *p, int (&r)[8]) {
    asm("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "l"(p));
    asm("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
        : "=r"(r[4]), "=r"(r[5]), "=r"(r[6]), "=r"(r[7])
        : "l"(reinterpret_cast<const char *>(p) + 16));
}

__device__ __forceinline__ int4 ldg128_stream(const void *p) {
    int4 r;
    asm("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

// FP16FloatTensor.vectorDot's bit trick (FP16FloatTensor.java:88-98): denormals-are-zero,
// no inf/nan handling.  Used for FP16 weight matrices only; embedding lookups use IEEE.
__device__ __forceinline__ float f16_bits_to_f32_daz(unsigned h) {
    unsigned mask = (h & 0x7C00u) ? 0xFFFFFFFFu : 0u;
    unsigned bits = ((h & 0x8000u) << 16) | ((((h & 0x7FFFu) + 0x1C000u) << 13) & mask);
    return __uint_as_float(bits);
}

// Weight matrix as stored on the device.
//   Q8_0: qs = int8 [rows][cols] row-major, sc = f16 scale [rows][cols/32]
//         (GGUF's 34-byte blocks split at upload so the quants are 32-byte aligned: same
//          1.0625 B/element, one LDG.256 per block).
//   F16 : qs = f16 [rows][cols], sc unused.  F32: qs = float.
struct DevMat {
    const void *qs;
    const __half *sc;
    int rows, cols, type;
};
