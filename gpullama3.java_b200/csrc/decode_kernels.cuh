// decode_kernels.cuh -- single-token decode kernels, bit-exact with the reference's CPU path: the RMSNorm, the attention
// and the FP16 matvecs (the Q8_0 matvecs are the weight streams of stream_matvec.cuh).  One CUDA graph strings them together
// per token (plan.cu).
//
// Replaces (reference kernel inventory, SURVEY.md 2.K):
//   k_rmsnorm_quant  <- reductionOneBlockWithLayer + reductionOneBlock2WithLayer / mapContextWithQuantize
//                       (TransformerComputeKernelsLayered.java:387-454) + convertQ8_0toFP32 embedding
//   k_rope_kv        <- ropeRotationWithCacheCopy (:495-542), Qwen3 fusedQKRmsNorm + NeoX rope (Qwen3Kernels.java:302-361,973-1064)
//   k_attention      <- processHeadsFlashAttention (:784-906)
//   k_argmax_advance <- argmaxLogits (TransformerComputeKernels.java:25-56), with CPU tie-break semantics
// but the arithmetic they implement is the CPU path's (InferenceCore.java:50-172, 565-697).
#pragma once
#include "common.cuh"
#include "seqsum2.cuh"

enum { MODE_STORE = 0, MODE_RESID = 1 };

// ------------------------------------------------------------------------------------------
// Embedding row lookup: FloatTensor.copyTo -> getFloat per element (InferenceCore.java:61).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float emb_get_raw(const DevMat &e, int token, int i) {
    size_t idx = (size_t)token * e.cols + i;
    if (e.type == 8) { // Q8_0FloatTensor.getFloat: quant * scale (Q8_0FloatTensor.java:55-63)
        float q = (float)((const int8_t *)e.qs)[idx];
        return __fmul_rn(q, __half2float(e.sc[idx >> 5]));
    } else if (e.type == 1) { // FP16FloatTensor.getFloat: Float.float16ToFloat (IEEE, subnormals kept)
        return __half2float(((const __half *)e.qs)[idx]);
    }
    return ((const float *)e.qs)[idx];
}
// The embedding row times the model's embedding scale: Granite's x[i] = x[i] * embeddingScale (InferenceCore.java:826-829), one
// rounding; every other family passes 1.0f, which leaves each value bit for bit as it is.
__device__ __forceinline__ float emb_get(const DevMat &e, int token, int i, float es) { return __fmul_rn(emb_get_raw(e, token, i), es); }

// ------------------------------------------------------------------------------------------
// RMSNorm (+ optional embedding gather, + Q8_0 activation quantisation).
// InferenceCore.rmsnorm (InferenceCore.java:39-48): ss = sequential float sum of x*x;
// ss = ss/size + eps; ss = (float)(1.0/Math.sqrt(ss)); out = w * (ss * x).
// The sum is order-sensitive, so one thread walks it (squares precomputed in parallel).
// One CTA.  Outputs: xq/xs (Q8_0 activation for the following matvec) and/or xb (float).
// ------------------------------------------------------------------------------------------
#define NORM_THREADS SEQSUM2_THREADS
__host__ __device__ inline int norm_padded(int dim) { return (dim + SEQSUM2_THREADS - 1) / SEQSUM2_THREADS * SEQSUM2_THREADS; }
__host__ __device__ inline size_t norm_smem_bytes(int dim) { return (size_t)norm_padded(dim) * 4 + 16 + seqsum2_scratch_bytes(); }

// The body of k_rmsnorm_quant for one vector; `tok` is read after the dependency wait (the batched step, decode_batch.cuh,
// runs it once per row with that row's x, token and outputs).
template <bool EMBED>
__device__ __forceinline__ void rmsnorm_quant_row(float *__restrict__ x, const int *__restrict__ tok, const DevMat &emb, float emb_scale,
                                                  const float *__restrict__ w, float eps, int dim, int8_t *__restrict__ xq,
                                                  float *__restrict__ xs, float *__restrict__ xb, long long *__restrict__ prof,
                                                  const TraceBuf &tr, const TpCtx &tp, int tp_wait_op) {
    extern __shared__ __align__(16) float sm[];
    float *sq = sm;
    __shared__ float s_ss;
    const int tid = threadIdx.x;
    long long t0 = 0, t1 = 0, t2 = 0, t3 = 0;
    if (prof) t0 = clock64();
    trace_entry(tr);
    pdl_launch_dependents();
    pdl_wait();
    trace_mark(tr, 2);
    if (prof) t1 = clock64();
    if (tp.n > 1 && tp_wait_op >= 0) { // x is gathered from all ranks: wait for their slices
        if (tid == 0) tp_wait(tp, TP_SLOT_X, tp_seq(tp, (unsigned)tp_wait_op));
        __syncthreads();
    }
    int token = 0;
    if (EMBED) token = *tok;
    for (int i = tid; i < dim; i += NORM_THREADS) {
        float v;
        if (EMBED) { v = emb_get(emb, token, i, emb_scale); x[i] = v; }
        else v = ldcg_f32c(x + i);
        sq[i] = __fmul_rn(v, v);
    }
    for (int i = dim + tid; i < norm_padded(dim); i += NORM_THREADS) sq[i] = 0.0f;
    __syncthreads();
    if (prof) t2 = clock64();
    // ss = sequential float sum of the squares (exact, parallel)
    int info0 = 0, info1 = 0;
    SeqSum2Scratch scratch = seqsum2_carve(reinterpret_cast<unsigned char *>(sm + norm_padded(dim)));
    float ss = block_seqsum_exact_v2(sq, dim, scratch);
    if (prof && tid == 0) { info0 = scratch.info[0]; info1 = scratch.info[1]; }
    if (prof) t3 = clock64();
    if (EMBED) __threadfence_block(); // x[] written above by other threads of this block
    if (tid == 0) {
        ss = __fdiv_rn(ss, (float)dim);
        ss = __fadd_rn(ss, eps);
        s_ss = (float)(1.0 / sqrt((double)ss));
    }
    __syncthreads();
    ss = s_ss;
    const int lane = tid & 31, warp = tid >> 5;
    constexpr int NWN = NORM_THREADS / 32;
    const int nb = dim / 32;
#pragma unroll 1
    for (int b0 = warp; b0 < nb; b0 += 4 * NWN) { // 8 loads in flight per lane
        float xv[4], wv[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int b = b0 + u * NWN;
            xv[u] = 0.0f; wv[u] = 0.0f;
            if (b < nb) { xv[u] = ldcg_f32c(x + b * 32 + lane); wv[u] = w[b * 32 + lane]; } // x: L2 hit (or this block's own store)
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int b = b0 + u * NWN;
            if (b < nb) {
                const int i = b * 32 + lane;
                const float v = __fmul_rn(wv[u], __fmul_rn(ss, xv[u]));
                if (xb) xb[i] = v;
                if (xq) {
                    float as;
                    int q = quant_block_lane(v, as);
                    xq[i] = (int8_t)q;
                    if (lane == 0) xs[b] = as;
                }
            }
        }
    }
    trace_mark(tr, 3);
    if (prof) {
        __syncthreads();
        if (tid == 0) { long long t4 = clock64(); prof[0] = t1 - t0; prof[1] = t2 - t1; prof[2] = t3 - t2; prof[3] = t4 - t3;
                        prof[4] = info0; prof[5] = info1; prof[6] = 0; }
    }
}

template <bool EMBED>
__global__ void __launch_bounds__(NORM_THREADS, 1) k_rmsnorm_quant(float *__restrict__ x, const StepState *__restrict__ st,
                                                               DevMat emb, float emb_scale, const float *__restrict__ w, float eps, int dim,
                                                               int8_t *__restrict__ xq, float *__restrict__ xs,
                                                               float *__restrict__ xb, long long *__restrict__ prof, TraceBuf tr, TpCtx tp, int tp_wait_op) {
    // One CTA of 1024 threads.  Under PDL this CTA only has to fit next to ONE streaming-matvec CTA
    // (the following matvec's CTA for this SM simply starts a little later).
    rmsnorm_quant_row<EMBED>(x, &st->token, emb, emb_scale, w, eps, dim, xq, xs, xb, prof, tr, tp, tp_wait_op);
}

// Test hook: the sequential-sum emulation on arbitrary non-negative terms (padded with zeros: adding +0 never changes a sum
// of non-negative floats), seqsum2.cuh with T threads (1024: the norm kernel's form; 256: the persistent decode kernel's form)
template <int T>
__global__ void __launch_bounds__(T, 1) k_test_seqsum2(const float *__restrict__ terms, int n, float *__restrict__ out, int *__restrict__ info) {
    extern __shared__ __align__(16) float sm[];
    float *sq = sm;
    const int E = (n + T - 1) / T, np = T * E;
    SeqSum2Scratch scratch = seqsum2_carve(reinterpret_cast<unsigned char *>(sm + np), T);
    for (int i = threadIdx.x; i < np; i += T) sq[i] = i < n ? terms[i] : 0.0f;
    if (threadIdx.x == 0) { scratch.info[0] = -1; scratch.info[1] = -2; }
    __syncthreads();
    const float s = block_seqsum_exact_v2_t<T>(sq, n, scratch, (int)threadIdx.x, SeqSum2BlockSync());
    if (threadIdx.x == 0) { out[0] = s; info[0] = scratch.info[0]; info[1] = scratch.info[1]; }
}

// Profiling hook: the accumulator in the fused norm's form (chunks at seqsum2_stride, one out-of-line copy as smv_seqsum and
// pd_seqsum have), called twice in one launch: the first call runs on a cold instruction cache, the second on a warm one.  Each
// call is timed in clock64 cycles from a barrier before it to a barrier after it; the second call's {items, literal items,
// fallbacks} follow the two cycle counts.
template <int T>
__device__ __noinline__ float profile_seqsum2_call(const float *sq, int n, int S, unsigned char *scratch) {
    return block_seqsum_exact_v2_t<T>(sq, n, seqsum2_carve(scratch, T), (int)threadIdx.x, SeqSum2BlockSync(), S);
}
template <int T>
__global__ void __launch_bounds__(T, 1) k_profile_seqsum2(const float *__restrict__ terms, int n, long long *__restrict__ cycles, float *__restrict__ out) {
    extern __shared__ __align__(16) float sm[];
    const int E = (n + T - 1) / T, S = seqsum2_stride(E);
    unsigned char *scratch = reinterpret_cast<unsigned char *>(sm + T * S);
    for (int i = threadIdx.x; i < T * E; i += T) sm[(i / E) * S + (i % E)] = i < n ? terms[i] : 0.0f;
    __syncthreads();
    const long long t0 = clock64();
    const float s0 = profile_seqsum2_call<T>(sm, n, S, scratch);
    __syncthreads();
    const long long t1 = clock64();
    const float s1 = profile_seqsum2_call<T>(sm, n, S, scratch);
    __syncthreads();
    const long long t2 = clock64();
    if (threadIdx.x == 0) {
        const int *info = seqsum2_carve(scratch, T).info;
        cycles[0] = t1 - t0; cycles[1] = t2 - t1; cycles[2] = info[0]; cycles[3] = info[2]; cycles[4] = info[1];
        out[0] = s0; out[1] = s1;
    }
}

// ------------------------------------------------------------------------------------------
// SwiGLU of one hidden unit, InferenceCore.java:150-158: hb = hb / (float)(1.0 + Math.exp(-hb)); hb *= hb2.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float swiglu(float g, float u) {
    float s = __fdiv_rn(g, (float)(1.0 + exp((double)(-g))));
    return __fmul_rn(s, u);
}

// Test hook: the two exp expressions of the bit-exact paths (the softmaxes and routers, swiglu's denominator) on the n float bit
// patterns first, first + 1, ...
__global__ void __launch_bounds__(256) k_test_exp(unsigned first, unsigned n, float *__restrict__ e, float *__restrict__ e1) {
    for (unsigned i = blockIdx.x * 256u + threadIdx.x; i < n; i += gridDim.x * 256u) {
        const double d = exp((double)__uint_as_float(first + i));
        e[i] = (float)d;
        e1[i] = (float)(1.0 + d);
    }
}

// ------------------------------------------------------------------------------------------
// FP16 dequant-matvec, bit-exact with FP16FloatTensor.vectorDot (FP16FloatTensor.java:62-110)
// for an L-lane species: L independent strided FMA chains (fused, as FloatVector.fma), then
// reduceLanes(ADD) in ascending lane order, then the IEEE scalar tail.
// A warp owns 32/L rows at a time... see k_matvec_f16 below: thread (r, c) owns chain c of row r;
// the warp stages 16-byte coalesced loads through shared memory so every thread reads its
// stride-L elements from there.
// ------------------------------------------------------------------------------------------
template <int MODE>
__global__ void __launch_bounds__(256) k_matvec_f16(const __half *__restrict__ w, const float *__restrict__ x, int rows,
                                                    int cols, int lanes, float *__restrict__ out, float oscale) {
    // Each warp processes RW = 32/lanes rows at once; thread t of the warp: row r = t / lanes, chain c = t % lanes.
    // Shared: activation x (cols floats) + per-warp weight tile RW x TC halves.
    extern __shared__ __align__(16) unsigned char smraw[];
    float *sx = reinterpret_cast<float *>(smraw);
    constexpr int TC = 256; // columns per staged tile
    __half *tiles = reinterpret_cast<__half *>(smraw + (size_t)cols * 4);
    for (int i = threadIdx.x; i < cols; i += blockDim.x) sx[i] = x[i];
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int L = lanes > 0 ? lanes : 1;
    const int RW = 32 / L;
    __half *tile = tiles + (size_t)warp * RW * TC;
    const int r = lane / L, c = lane % L;
    const int nwarps_total = gridDim.x * (blockDim.x >> 5);
    const int upper = lanes > 0 ? cols - (cols % L) : 0;
    for (size_t row0 = (size_t)(blockIdx.x * (blockDim.x >> 5) + warp) * RW; row0 < (size_t)rows; row0 += (size_t)nwarps_total * RW) {
        float acc = 0.0f;
        for (int c0 = 0; c0 < cols; c0 += TC) {
            int tc = min(TC, cols - c0);
            // coalesced stage: RW rows x tc halves, 8 halves (16 B) per lane per load
            int chunks_per_row = tc >> 3;
            for (int q = lane; q < RW * chunks_per_row; q += 32) {
                int rr = q / chunks_per_row, cc = q % chunks_per_row;
                size_t row = row0 + rr;
                int4 v = make_int4(0, 0, 0, 0);
                if (row < (size_t)rows) v = ldg128_stream(w + row * (size_t)cols + c0 + cc * 8);
                *reinterpret_cast<int4 *>(tile + rr * TC + cc * 8) = v;
            }
            __syncwarp();
            if (lanes > 0) {
                int lim = min(tc, upper - c0);
                for (int i = c; i < lim; i += L) {
                    float wf = f16_bits_to_f32_daz(__half_as_ushort(tile[r * TC + i]));
                    acc = fmaf(wf, sx[c0 + i], acc);
                }
            } else {
                // llama.VectorBitSize=0: FloatTensor.scalarDot, sequential, IEEE conversion, unfused
                for (int i = 0; i < tc; i++) acc = __fadd_rn(acc, __fmul_rn(__half2float(tile[r * TC + i]), sx[c0 + i]));
            }
            __syncwarp();
        }
        // reduceLanes(ADD), ascending lane order starting from the identity, then scalar tail
        float result = acc;
        if (lanes > 0) {
            result = 0.0f;
            for (int k = 0; k < L; k++) {
                float a = __shfl_sync(0xffffffffu, acc, r * L + k);
                result = __fadd_rn(result, a);
            }
            size_t row = row0 + r;
            if (row < (size_t)rows)
                for (int j = upper; j < cols; j++)
                    result = __fadd_rn(result, __fmul_rn(__half2float(w[row * (size_t)cols + j]), sx[j]));
        }
        size_t row = row0 + r;
        if (c == 0 && row < (size_t)rows) {
            result = __fmul_rn(result, oscale); // Granite's residualScale / logitScale (1.0f: unchanged)
            if (MODE == MODE_RESID) out[row] = __fadd_rn(out[row], result);
            else out[row] = result;
        }
    }
}

// SwiGLU over separately computed gate/up vectors (FP16 path): hb = silu(hb) * hb2.
__global__ void k_swiglu(float *__restrict__ hb, const float *__restrict__ hb2, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) hb[i] = swiglu(hb[i], hb2[i]);
}

// ------------------------------------------------------------------------------------------
// Fused RoPE + KV-cache write + attention, one query head per CTA, exact CPU-path order.
//   prologue : (Qwen3: per-head RMSNorm of q and k, InferenceCore.java:594-600) then RoPE of this
//              head's q and of its KV head's k (InferenceCore.java:75-87 interleaved pairs / :604-619 NeoX);
//              every query head of a KV group rotates the same k redundantly (cheaper than a
//              kernel boundary); the group's first head writes k,v into the cache (:92-93)
//   scores   : score_t = scalarDot(q, k_t) / sqrt(head)   (sequential unfused mul/add, FloatTensor.java:86-92)
//   softmax  : max, (float)Math.exp(f - max), sequential sum, divide        (FloatTensor.java:211-219)
//   output   : xb = sum_t a_t * v_t, sequentially over t per element (saxpyInPlace, FloatTensor.java:221-227)
// The current position's k/v come from shared memory / the packed qkv vector, older ones from the
// FP32 cache.  Output as floats (xb) and/or quantised to Q8_0 (activation of the Wo matvec).
// ------------------------------------------------------------------------------------------
#define ATT_THREADS 512 // four threads per key (scores) and per output element (weighted sum): head size <= ATT_THREADS / 4

// The prologue of attention_head for query head h at position pos: threads [0,HALF) rotate q pairs, threads [HALF,HS) rotate
// k pairs, threads [HS,2HS) take v.  The rotated q goes to sq and back into qkv, the rotated k to sk; the group's first head
// writes k / v into the cache.  sk / so are the Qwen3 norm's scratch; Qwen2 stages its biased v in so.  k_rope_kv_batch
// (decode_batch.cuh) runs it on its own, ahead of an attention that takes every key from the cache.
// qsrc / ksrc / vsrc: this head's q, its KV head's k and v in qkv.
template <int HS>
__device__ __forceinline__ void rope_kv_prologue(float *qkv, const float *qsrc, const float *ksrc, const float *vsrc, float *kc, float *vc, int pos,
                                                 int h, int kv_mul, int kvh, int qd, int kvd, const float *cr, const float *ci, int arch,
                                                 const float *qnorm_w, const float *knorm_w, const float *qkv_bias, float eps, float *sq, float *sk,
                                                 float *so, float *s_val) {
    const int tid = threadIdx.x;
    constexpr int HALF = HS / 2;
    if (tid < HS) {
        const bool is_q = tid < HALF;
        const int p = is_q ? tid : tid - HALF;
        const float *src = is_q ? qsrc : ksrc;
        int i0, i1;
        if (arch & KF_NEOX) { i0 = p; i1 = p + HALF; } else { i0 = 2 * p; i1 = 2 * p + 1; }
        float v0 = src[i0], v1 = src[i1];
        if (arch & KF_QKVBIAS) { // Qwen2: q / k bias (laid out like q|k|v) before the rotation
            const float *b = qkv_bias + (is_q ? h * HS : qd + kvh * HS);
            v0 = __fadd_rn(v0, b[i0]);
            v1 = __fadd_rn(v1, b[i1]);
        }
        if (arch & KF_QKNORM) { // Qwen3 per-head RMSNorm: literal sequential sum over the head
            float *sqr = is_q ? so : sk; // scratch: HS squares each
            sqr[i0] = __fmul_rn(v0, v0);
            sqr[i1] = __fmul_rn(v1, v1);
        }
        if (arch & KF_QKNORM) {
            asm volatile("bar.sync 3, %0;" ::"n"(HS) : "memory");
            if (p == 0) {
                const float *sqr = is_q ? so : sk;
                float ss = 0.0f;
                for (int i = 0; i < HS; i++) ss = __fadd_rn(ss, sqr[i]);
                ss = __fdiv_rn(ss, (float)HS);
                ss = __fadd_rn(ss, eps);
                s_val[is_q ? 0 : 1] = (float)(1.0 / sqrt((double)ss));
            }
            asm volatile("bar.sync 3, %0;" ::"n"(HS) : "memory");
            const float ss = s_val[is_q ? 0 : 1];
            const float *nw = is_q ? qnorm_w : knorm_w;
            v0 = __fmul_rn(nw[i0], __fmul_rn(ss, v0));
            v1 = __fmul_rn(nw[i1], __fmul_rn(ss, v1));
            asm volatile("bar.sync 3, %0;" ::"n"(HS) : "memory"); // scratch reads done before sk/so are overwritten
        }
        const float fcr = cr[(size_t)pos * HALF + p], fci = ci[(size_t)pos * HALF + p];
        const float r0 = __fsub_rn(__fmul_rn(v0, fcr), __fmul_rn(v1, fci));
        const float r1 = __fadd_rn(__fmul_rn(v0, fci), __fmul_rn(v1, fcr));
        float *dst = is_q ? sq : sk;
        dst[i0] = r0;
        dst[i1] = r1;
        if (h % kv_mul == 0) { // first query head of the KV group owns the cache / debug write-back
            if (!is_q) {
                const size_t o = (size_t)pos * kvd + kvh * HS;
                kc[o + i0] = r0;
                kc[o + i1] = r1;
                // (the rotated k is NOT written back into qkv: the other query heads of this group read the
                //  unrotated k from there concurrently)
            }
        }
        if (is_q) { qkv[h * HS + i0] = r0; qkv[h * HS + i1] = r1; }
    } else if (tid < 2 * HS) { // v: the group's first head writes the cache; Qwen2 adds the bias and stages v for the weighted sum
        const int j = tid - HS;
        float w = vsrc[j];
        if (arch & KF_QKVBIAS) {
            w = __fadd_rn(w, qkv_bias[qd + kvd + kvh * HS + j]);
            so[j] = w; // (so is scratch of the q/k norm only, which Qwen2 does not have)
        }
        if (h % kv_mul == 0) vc[(size_t)pos * kvd + kvh * HS + j] = w;
    }
}

// K / V cache loads of attention_head: read-only path, or L2 (ld.global.cg) for rows the previous grid wrote.
template <bool CG, typename T> __device__ __forceinline__ T kv_ld(const T *p) {
    if constexpr (CG) return __ldcg(p);
    else return __ldg(p);
}

// The body of k_attention for query head blockIdx.x of one sequence; `posp` is read after the dependency wait (the batched
// step, decode_batch.cuh, runs it per (head, row) with that row's position, cache, qkv vector, outputs and score rows).
// CACHED: k_rope_kv_batch has run the prologue, so q is read rotated from qkv and every key t <= pos, the current one
// included, comes from the cache -- the same floats the prologue would hold in sk / so, in the same order.  Those rows were
// written by the previous grid, so they are read through L2 (ld.global.cg), never through the non-coherent path.
template <int HS, bool CACHED = false>
__device__ __forceinline__ void attention_head(float *__restrict__ qkv, float *__restrict__ kc, float *__restrict__ vc,
                                               const int *__restrict__ posp, const float *__restrict__ cr, const float *__restrict__ ci,
                                               int n_heads, int n_kv_heads, int arch, const float *__restrict__ qnorm_w,
                                               const float *__restrict__ knorm_w, const float *__restrict__ qkv_bias, float eps, float sqrt_hs,
                                               int8_t *__restrict__ xq, float *__restrict__ xs, float *__restrict__ xb, const TraceBuf &tr,
                                               const TpCtx &tp, unsigned tp_out_op, int head_base, float *att_scratch, int ctx) {
    extern __shared__ __align__(16) float sm[]; // q[HS] | k[HS] | out[HS] | att[ctx] (att in global scratch for long contexts)
    __shared__ float red[ATT_THREADS / 32];
    __shared__ float s_val[2];
    float *sq = sm, *sk = sm + HS, *so = sm + 2 * HS;
    float *att = att_scratch ? att_scratch + (size_t)blockIdx.x * ctx : sm + 3 * HS;
    const int h = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    trace_entry(tr);
    pdl_launch_dependents();
    const int kv_mul = n_heads / n_kv_heads, kvh = h / kv_mul;
    const int qd = n_heads * HS, kvd = n_kv_heads * HS;
    pdl_wait();
    trace_mark(tr, 2);
    const int pos = *posp, nt = pos + 1;
    { // K/V rows of the earlier positions -> L2, one 128-byte line per request, so the score loads below hit L2 (the weight stream carries an
      // evict_first policy; without the prefetch these rows come from HBM every layer)
        constexpr int LINES = HS / 32;
        for (int i = tid; i < pos * LINES; i += ATT_THREADS) {
            const size_t off = (size_t)(i / LINES) * kvd + kvh * HS + (i % LINES) * 32;
            asm volatile("prefetch.global.L2 [%0];" ::"l"(kc + off));
            asm volatile("prefetch.global.L2 [%0];" ::"l"(vc + off));
        }
    }
    const float *qsrc = qkv + h * HS, *ksrc = qkv + qd + kvh * HS, *vsrc = qkv + qd + kvd + kvh * HS;
    if (CACHED) {
        if (tid < HS) sq[tid] = qsrc[tid];
    } else {
        rope_kv_prologue<HS>(qkv, qsrc, ksrc, vsrc, kc, vc, pos, h, kv_mul, kvh, qd, kvd, cr, ci, arch, qnorm_w, knorm_w, qkv_bias, eps, sq, sk,
                             so, s_val);
    }
    __syncthreads();
    // ---- scores (scalarDot, FloatTensor.java:86-92: one sequential unfused mul/add chain per key).  Four threads share a key: each loads
    // ITS quarter of the K row at once (one round trip per pass of ATT_THREADS/4 keys), then the chain runs through the quad in element
    // order, handed on by shuffle.  The V rows of the first round of the weighted sum are requested here too (they do not depend on the scores).
    constexpr int QE = HS / 4, QV = HS / 16, VB = 32;
    const int quad = tid & 3, qbase = lane & ~3, vd = tid >> 2;
    const bool vlive = vd < HS;
    float vv[VB];
    {
        const float *vcol = vc + kvh * HS + vd;
#pragma unroll
        for (int u = 0; u < VB; u++) vv[u] = (vlive && quad * VB + u < pos) ? kv_ld<CACHED>(vcol + (size_t)(quad * VB + u) * kvd) : 0.0f;
    }
    float lmax = -INFINITY;
#pragma unroll 1
    for (int t0 = 0; t0 < nt; t0 += ATT_THREADS / 4) {
        const int t = t0 + (tid >> 2);
        float4 kk[QV];
        if (t < pos || (CACHED && t == pos)) {
            const float4 *k = reinterpret_cast<const float4 *>(kc + (size_t)t * kvd + kvh * HS + quad * QE);
#pragma unroll
            for (int u = 0; u < QV; u++) kk[u] = kv_ld<CACHED>(k + u);
        } else {
#pragma unroll
            for (int u = 0; u < QV; u++) kk[u] = t == pos ? *reinterpret_cast<const float4 *>(sk + quad * QE + 4 * u) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        float acc = 0.0f;
#pragma unroll 1
        for (int qd4 = 0; qd4 < 4; qd4++) {
            if (quad == qd4) {
                const float *qq = sq + qd4 * QE;
#pragma unroll
                for (int u = 0; u < QV; u++) {
                    acc = __fadd_rn(acc, __fmul_rn(qq[4 * u + 0], kk[u].x));
                    acc = __fadd_rn(acc, __fmul_rn(qq[4 * u + 1], kk[u].y));
                    acc = __fadd_rn(acc, __fmul_rn(qq[4 * u + 2], kk[u].z));
                    acc = __fadd_rn(acc, __fmul_rn(qq[4 * u + 3], kk[u].w));
                }
            }
            acc = __shfl_sync(0xffffffffu, acc, qbase + qd4);
        }
        if (quad == 0 && t < nt) {
            const float s = (arch & KF_ATTSCALE) ? __fmul_rn(acc, sqrt_hs) : __fdiv_rn(acc, sqrt_hs); // Granite: score *= attentionScale
            att[t] = s;
            lmax = fmaxf(lmax, s);
        }
    }
    lmax = warp_max_f(lmax);
    if (lane == 0) red[warp] = lmax;
    __syncthreads();
    float mx = red[0];
#pragma unroll
    for (int w = 1; w < ATT_THREADS / 32; w++) mx = fmaxf(mx, red[w]);
    for (int t = tid; t < nt; t += ATT_THREADS) att[t] = (float)exp((double)__fsub_rn(att[t], mx));
    __syncthreads();
    if (tid == 0) {
        float sum = 0.0f;
        int t = 0;
        for (; t + 4 <= nt; t += 4) {
            const float a0 = att[t], a1 = att[t + 1], a2 = att[t + 2], a3 = att[t + 3];
            sum = __fadd_rn(sum, a0); sum = __fadd_rn(sum, a1); sum = __fadd_rn(sum, a2); sum = __fadd_rn(sum, a3);
        }
        for (; t < nt; t++) sum = __fadd_rn(sum, att[t]);
        s_val[0] = sum;
    }
    __syncthreads();
    const float sum = s_val[0];
    for (int t = tid; t < nt; t += ATT_THREADS) att[t] = __fdiv_rn(att[t], sum);
    __syncthreads();
    // ---- output: xb = sum_t a_t * v_t sequentially over t per element (saxpyInPlace, FloatTensor.java:221-227); four threads per element, thread
    // `quad` holds rows [128 r + 32 quad, +32) of round r, the chain runs through the quad in row order
#pragma unroll 1
    for (int vd0 = 0; vd0 < HS; vd0 += ATT_THREADS / 4) { // one pass for head sizes up to 128
        const int d = vd0 + vd;
        const bool live = d < HS;
        const float *vcol = vc + kvh * HS + d;
        const float vcur = !live ? 0.0f
                           : CACHED ? kv_ld<true>(vcol + (size_t)pos * kvd)
                                    : ((arch & KF_QKVBIAS) ? so[d] : vsrc[d]); // current position: the packed qkv vector (biased: staged)
        float acc = 0.0f;
#pragma unroll 1
        for (int r0 = 0; r0 < pos; r0 += 4 * VB) {
            if (r0 > 0 || vd0 > 0) { // (round 0 of the first pass was requested before the scores)
                const int vt0 = r0 + quad * VB;
#pragma unroll
                for (int u = 0; u < VB; u++) vv[u] = (live && vt0 + u < pos) ? kv_ld<CACHED>(vcol + (size_t)(vt0 + u) * kvd) : 0.0f;
            }
#pragma unroll 1
            for (int qd4 = 0; qd4 < 4; qd4++) {
                if (quad == qd4) {
                    const int vt0 = r0 + qd4 * VB;
#pragma unroll
                    for (int u = 0; u < VB; u++)
                        if (vt0 + u < pos) acc = __fadd_rn(__fmul_rn(att[vt0 + u], vv[u]), acc);
                }
                acc = __shfl_sync(0xffffffffu, acc, qbase + qd4);
            }
        }
        if (live && quad == 0) {
            acc = __fadd_rn(__fmul_rn(att[pos], vcur), acc);
            so[d] = acc;
            if (xb) xb[h * HS + d] = acc;
        }
    }
    __syncthreads();
    if (xq) {
        for (int b = warp; b < HS / 32; b += ATT_THREADS / 32) {
            float as;
            int q = quant_block_lane(so[b * 32 + lane], as);
            if (tp.n > 1) { // all-gather: this head's quantised output goes straight into every rank's buffer
                const int gh = head_base + h;
                for (int k = 0; k < tp.n; k++) {
                    tp_ptr<int8_t>(tp, k, tp.off_attq)[gh * HS + b * 32 + lane] = (int8_t)q;
                    if (lane == 0) tp_ptr<float>(tp, k, tp.off_atts)[(gh * HS) / 32 + b] = as;
                }
            } else {
                xq[h * HS + b * 32 + lane] = (int8_t)q;
                if (lane == 0) xs[(h * HS) / 32 + b] = as;
            }
        }
    }
    if (tp.n > 1) {
        __syncthreads();
        if (tid == 0) tp_cta_done(tp, TP_SLOT_ATT, tp_seq(tp, tp_out_op), gridDim.x);
    }
    trace_mark(tr, 3);
}

template <int HS>
__global__ void __launch_bounds__(ATT_THREADS) k_attention(float *__restrict__ qkv, float *__restrict__ kc, float *__restrict__ vc,
                                                          const StepState *__restrict__ st, const float *__restrict__ cr,
                                                          const float *__restrict__ ci, int n_heads, int n_kv_heads, int arch /* KF_* flags */,
                                                          const float *__restrict__ qnorm_w, const float *__restrict__ knorm_w,
                                                          const float *__restrict__ qkv_bias, float eps, float sqrt_hs, int8_t *__restrict__ xq,
                                                          float *__restrict__ xs, float *__restrict__ xb, TraceBuf tr, TpCtx tp,
                                                          unsigned tp_out_op, int head_base, float *att_scratch, int ctx) {
    attention_head<HS>(qkv, kc, vc, &st->pos, cr, ci, n_heads, n_kv_heads, arch, qnorm_w, knorm_w, qkv_bias, eps, sqrt_hs, xq, xs, xb, tr, tp,
                       tp_out_op, head_base, att_scratch, ctx);
}

// ------------------------------------------------------------------------------------------
// Greedy sampler + step advance.  FloatTensor.argmax (FloatTensor.java:138-151): first strict
// maximum.  One CTA; each thread keeps (max, lowest index) over a strided slice, then a tree
// merge that prefers the lower index on ties -- equal to the sequential scan for NaN-free input.
// Also advances the device-resident StepState so graph replays chain without the host.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void argmax_merge(float &v, int &i, float ov, int oi) {
    if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
}

__global__ void __launch_bounds__(1024) k_argmax_advance(const float *__restrict__ logits, int vocab, StepState *st,
                                                        const int *__restrict__ seq_tokens, int *__restrict__ out_ids,
                                                        int do_argmax, const float *__restrict__ part_val,
                                                        const int *__restrict__ part_idx, int n_part, TraceBuf tr, TpCtx tp, int tp_wait_x_op) {
    __shared__ float sv[32];
    __shared__ int si[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    trace_entry(tr);
    pdl_launch_dependents();
    pdl_wait();
    trace_mark(tr, 2);
    int best_i = 0;
    if (do_argmax) {
        float best = -INFINITY;
        best_i = 0x7fffffff;
        if (part_val) { // per-CTA (max, first index) pairs produced by the lm_head kernel
            for (int i = tid; i < n_part; i += blockDim.x) {
                float v = part_val[i];
                int ix = part_idx[i];
                argmax_merge(best, best_i, v, ix);
            }
        } else {
            for (int i = tid; i < vocab; i += blockDim.x) {
                float v = logits[i];
                if (v > best) { best = v; best_i = i; }
            }
        }
        // a thread that saw nothing > -inf keeps INT_MAX; index 0 wins below if all are -inf
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            float ov = __shfl_xor_sync(0xffffffffu, best, o);
            int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
            argmax_merge(best, best_i, ov, oi);
        }
        if (lane == 0) { sv[warp] = best; si[warp] = best_i; }
        __syncthreads();
        if (warp == 0) {
            int nw = blockDim.x >> 5;
            best = lane < nw ? sv[lane] : -INFINITY;
            best_i = lane < nw ? si[lane] : 0x7fffffff;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                float ov = __shfl_xor_sync(0xffffffffu, best, o);
                int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
                argmax_merge(best, best_i, ov, oi);
            }
            if (tp.n > 1) { // exchange every rank's (max, lowest global index) and merge identically everywhere
                const unsigned seq = tp_seq(tp, tp.ops_per_fwd - 1u);
                if (lane == 0) {
                    for (int k = 0; k < tp.n; k++) {
                        tp_ptr<float>(tp, k, tp.off_pv)[tp.rank] = best;
                        tp_ptr<int>(tp, k, tp.off_pi)[tp.rank] = best_i;
                    }
                    tp_signal(tp, TP_SLOT_ARG, seq);
                    tp_wait(tp, TP_SLOT_ARG, seq);
                }
                __syncwarp();
                best = lane < tp.n ? ldcg_f32c(tp_ptr<float>(tp, tp.rank, tp.off_pv) + lane) : -INFINITY;
                best_i = lane < tp.n ? (int)__float_as_int(ldcg_f32c(reinterpret_cast<const float *>(tp_ptr<int>(tp, tp.rank, tp.off_pi)) + lane)) : 0x7fffffff;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    float ov = __shfl_xor_sync(0xffffffffu, best, o);
                    int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
                    argmax_merge(best, best_i, ov, oi);
                }
            }
            if (best_i == 0x7fffffff) best_i = 0;
        }
    } else if (tp.n > 1 && tp_wait_x_op >= 0) {
        // prefill graph: no argmax exchange, but the next forward's embedding write must not race the peers'
        // last residual-stream pushes of this forward
        if (tid == 0) tp_wait(tp, TP_SLOT_X, tp_seq(tp, (unsigned)tp_wait_x_op));
        __syncthreads();
    }
    if (tid == 0) {
        int step = st->step;
        if (do_argmax && out_ids) out_ids[step] = best_i;
        int next = step + 1;
        if (st->feedback && do_argmax) st->token = best_i;
        else if (next < st->n_seq) st->token = seq_tokens[next];
        st->step = next;
        st->pos = st->pos + 1;
        if (tp.n > 1) *reinterpret_cast<volatile unsigned *>(tp.peer[tp.rank] + tp.off_tick) += 1u; // next forward's flag epoch
    }
    trace_mark(tr, 3);
}
