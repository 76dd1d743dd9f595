// moe.cuh -- the FFN half of a Qwen2-MoE decode layer (InferenceCore.forwardJavaQwen2MoE, InferenceCore.java:366-424): the router,
// the gate/up projections of the shared expert and the k routed experts, and their down projections with the ordered combine.
//
// Every other weight stream of the decode step has addresses that never depend on activations, so its producer starts copying
// before the previous kernel has finished (programmatic dependent launch).  Here the router's top-k, computed in the same step,
// picks which expert matrices are streamed.  The two stream kernels therefore treat the shared expert, whose addresses are
// static, first: their producers issue its tiles before the dependency wait and the routed experts' tiles after it, once the
// routing buffer can be read.
//
// Device layout: every expert is a TileMat of its own (stream_matvec.cuh), gate/up interleaved as in the dense plan's L.tgu,
// down as in L.tw2; a per-layer device table holds the base of each routed expert's two streams, indexed by expert id.  The
// hidden activations of one step form one "virtual" vector of Hs + k * He units: [shared | routed slot 0 | ... | slot k-1].
// Both Hs and He are multiples of 32, so no Q8_0 activation block straddles two experts and each expert's down projection reads
// exactly the per-32-block quantisation of its own hidden vector (Q8_0FloatTensor.java:100-117).
#pragma once
#include "stream_matvec.cuh"

#define MOE_MAX_K 8            // experts used per token (the routing table and the per-slot weights live in shared memory)
#define MOE_MAX_EXPERTS 256
#define MOE_ROUTE_THREADS 256

// ---- router --------------------------------------------------------------------------------------------------------------
// One CTA per router row plus one for the shared-expert gate (blockIdx.x == n_experts): each evaluates FloatTensor.scalarDot
// (FloatTensor.java:86-92) -- result += w[j] * x[j], one float multiply and one float add per term, strictly in index order.
// The products are formed in parallel; one thread walks the sum.  The last CTA to finish runs softmaxInPlace, the top-k scans
// and the shared-expert sigmoid on one thread, in the reference's order.
struct MoeRouteArgs {
    const float *router;      // [n_experts][dim] F32 (ffn_gate_inp)
    const float *shared_gate; // [dim] F32 (ffn_gate_inp_shexp)
    const float *xb;          // rmsnorm(x, ffn_norm), float
    float *logits;            // [n_experts + 1] scratch of this layer
    unsigned *done;           // arrival counter of this layer (self-resetting)
    int *ids;                 // [k] selected experts, in selection order
    float *weights;           // [k + 1] routing weights, then the shared-expert weight
    int dim, n_experts, k;
    TraceBuf tr;
};

__global__ void __launch_bounds__(MOE_ROUTE_THREADS, 1) k_moe_route(MoeRouteArgs a) {
    extern __shared__ __align__(16) float t[]; // dim terms
    __shared__ float pr[MOE_MAX_EXPERTS];
    __shared__ unsigned s_last;
    const int tid = threadIdx.x, e = blockIdx.x;
    const float *w = e < a.n_experts ? a.router + (size_t)e * a.dim : a.shared_gate;
    trace_entry(a.tr);
    for (int i = tid; i < a.dim; i += MOE_ROUTE_THREADS) t[i] = w[i]; // the router is immutable: read before the dependency wait
    pdl_launch_dependents();
    pdl_wait();
    trace_mark(a.tr, 2);
    for (int i = tid; i < a.dim; i += MOE_ROUTE_THREADS) t[i] = __fmul_rn(t[i], ldcg_f32(a.xb + i));
    __syncthreads();
    if (tid == 0) {
        a.logits[e] = pd_walk_terms(0.0f, t, a.dim); // float result = 0f; result += ... in index order
        __threadfence();
        s_last = atomicAdd(a.done, 1u) == (unsigned)a.n_experts ? 1u : 0u;
    }
    __syncthreads();
    if (!s_last || tid != 0) { trace_mark(a.tr, 3); return; }
    __threadfence();
    *a.done = 0u;
    const int E = a.n_experts;
    // softmaxInPlace (FloatTensor.java:211-219): max; (float) Math.exp(f - max); sequential sum from 0f; divide
    float mx = -INFINITY;
    for (int j = 0; j < E; j++) { pr[j] = ldcg_f32(a.logits + j); mx = fmaxf(mx, pr[j]); }
    for (int j = 0; j < E; j++) pr[j] = (float)exp((double)__fsub_rn(pr[j], mx));
    float sum = 0.0f;
    for (int j = 0; j < E; j++) sum = __fadd_rn(sum, pr[j]);
    for (int j = 0; j < E; j++) pr[j] = __fdiv_rn(pr[j], sum);
    // top-k: k scans for the first strict maximum, each pick then set to -inf; the weight is the probability itself (no renormalisation)
    for (int i = 0; i < a.k; i++) {
        float best = -INFINITY;
        int idx = 0;
        for (int j = 0; j < E; j++)
            if (pr[j] > best) { best = pr[j]; idx = j; }
        a.ids[i] = idx;
        a.weights[i] = best;
        pr[idx] = -INFINITY;
    }
    // shared-expert weight: 1f / (1f + (float) Math.exp(-g))
    const float g = ldcg_f32(a.logits + E);
    a.weights[a.k] = __fdiv_rn(1.0f, __fadd_rn(1.0f, (float)exp((double)(-g))));
    trace_mark(a.tr, 3);
}

// ---- the expert streams --------------------------------------------------------------------------------------------------
struct MoeStreamArgs {
    TileMat S;                         // shared expert: gate/up (rows 2 * Hs) or down (rows dim, cols Hs)
    TileMat X;                         // geometry of every routed expert's stream (base unused)
    const unsigned char *const *bases; // [n_experts] stream bases of this layer's routed experts
    const int *ids;                    // [k] routing buffer of this layer
    const float *weights;              // [k + 1]
    int k;
    const int8_t *xq;                  // gate/up: quantised xb [dim]; down: the quantised virtual hidden vector
    const float *xs;
    float *out;                        // gate/up: the virtual hidden vector (float); down: the residual stream x
    int8_t *hq;                        // gate/up: quantised virtual hidden vector
    float *hs;
    unsigned *blk_cnt;                 // gate/up: per-32-block arrival counters (self-resetting)
    TraceBuf tr;
};

// Stream geometry of one matrix of the down projection's sequence: shared (m = 0) or routed slot m - 1.
struct MoeMat {
    int seg, nseg, unit_bytes, act_off; // act_off: first unit of its activation in the virtual hidden vector
};
__device__ __forceinline__ MoeMat moe_mat(const MoeStreamArgs &a, int m) {
    const TileMat &T = m == 0 ? a.S : a.X;
    return MoeMat{T.seg, T.nseg, T.unit_bytes, m == 0 ? 0 : a.S.cols + (m - 1) * a.X.cols};
}

struct MoeDownSmem {
    size_t off_bar, off_xq, off_xs, off_terms, off_ring, total;
    int stages, stage_bytes, nbs_pad;
};

__host__ __device__ inline MoeDownSmem moe_down_layout(int hv, int seg_s, int seg_x, size_t budget) {
    MoeDownSmem L;
    const int ub = smv_unit_bytes(seg_s) > smv_unit_bytes(seg_x) ? smv_unit_bytes(seg_s) : smv_unit_bytes(seg_x);
    const int seg = seg_s > seg_x ? seg_s : seg_x;
    L.stage_bytes = (4 * ub + 127) & ~127;
    L.nbs_pad = ((seg / 32 + 3) & ~3) + 4;
    size_t o = 0;
    L.off_bar = o; o += 2 * SMV_MAX_STAGES * 8 + SMV_MAX_STAGES * 4;
    L.off_xq = o; o += (size_t)hv;
    o = (o + 15) & ~(size_t)15;
    L.off_xs = o; o += (size_t)(hv / 32) * 4;
    o = (o + 15) & ~(size_t)15;
    L.off_terms = o; o += (size_t)SMV_CONSUMER_WARPS * 4 * L.nbs_pad * 4;
    o = (o + 127) & ~(size_t)127;
    L.off_ring = o;
    long room = (long)budget - (long)o;
    int s = room > 0 ? (int)(room / L.stage_bytes) : 0;
    if (s > SMV_MAX_STAGES) s = SMV_MAX_STAGES;
    L.stages = s;
    L.total = o + (size_t)s * L.stage_bytes;
    return L;
}

// The int8 dot products of one tile (4 rows x one segment) against the staged activation, one term per (row, block), as the
// dense stream computes them (stream_matvec.cuh).
__device__ __forceinline__ void moe_tile_terms(const unsigned char *tile, const unsigned char *sact, const float *sxs, int unit_bytes, int seg,
                                               int nbs, float *terms, int nbs_pad, int lane) {
    const int hsel = (lane >> 2) & 1;
    for (int b = lane; b < nbs; b += 32) {
        const unsigned char *ab = sact + ((size_t)b << 5);
        const int4 a0 = *reinterpret_cast<const int4 *>(ab + 16 * hsel);
        const int4 a1 = *reinterpret_cast<const int4 *>(ab + 16 * (hsel ^ 1));
        const float as = sxs[b];
#pragma unroll
        for (int r = 0; r < 4; r++) {
            const unsigned char *wb = tile + (size_t)r * unit_bytes + ((size_t)b << 5);
            const int4 w0 = *reinterpret_cast<const int4 *>(wb + 16 * hsel);
            const int4 w1 = *reinterpret_cast<const int4 *>(wb + 16 * (hsel ^ 1));
            const __half sc = *reinterpret_cast<const __half *>(tile + (size_t)r * unit_bytes + seg + 2 * b);
            int isum = __dp4a(w0.x, a0.x, 0);
            isum = __dp4a(w0.y, a0.y, isum);
            isum = __dp4a(w0.z, a0.z, isum);
            isum = __dp4a(w0.w, a0.w, isum);
            isum = __dp4a(w1.x, a1.x, isum);
            isum = __dp4a(w1.y, a1.y, isum);
            isum = __dp4a(w1.z, a1.z, isum);
            isum = __dp4a(w1.w, a1.w, isum);
            terms[r * nbs_pad + b] = __fmul_rn((float)isum, __fmul_rn(__half2float(sc), as));
        }
    }
}

// Ring bookkeeping shared by both kernels (the dense stream's protocol): full[s] / empty[s] mbarriers and release counters.
__device__ __forceinline__ void moe_ring_init(unsigned char *smem, size_t off_bar, int S) {
    volatile unsigned *rel = reinterpret_cast<volatile unsigned *>(smem + off_bar + 2 * SMV_MAX_STAGES * 8);
    const unsigned bar0 = smem_u32(smem + off_bar);
    if (threadIdx.x == 0) {
        for (int s = 0; s < S; s++) {
            mbar_init(bar0 + 8 * s, 1);
            mbar_init(bar0 + 8 * (SMV_MAX_STAGES + s), 1);
            rel[s] = 0u;
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
}

// Gate/up of the shared expert and the k routed experts as ONE virtual gate/up matrix: groups [0, Hs/2) are the shared expert's,
// then He/2 groups per routed slot.  Output unit u of the virtual hidden vector = silu(gate) * up of group u / 2, exactly as
// k_stream_matvec_q8<SMV_GATEUP> computes a dense layer's; its Q8_0 epilogue is the dense one over the virtual vector.
__global__ void __launch_bounds__(SMV_THREADS, 1) k_moe_gateup(MoeStreamArgs a, SmvSmem L) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ const unsigned char *s_base[MOE_MAX_K];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int S = L.stages;
    const unsigned bar0 = smem_u32(smem + L.off_bar);
    const int gs = a.S.rows >> 2, gx = a.X.rows >> 2;
    const int ngroups = gs + a.k * gx;
    const int g0 = (int)(((long long)blockIdx.x * ngroups) / gridDim.x);
    const int g1 = (int)(((long long)(blockIdx.x + 1) * ngroups) / gridDim.x);
    const int nseg = a.S.nseg; // the shared and the routed gate/up streams have the same columns (dim), so the same tiles
    const unsigned tile_bytes = 4u * (unsigned)a.S.unit_bytes;
    volatile unsigned *rel = reinterpret_cast<volatile unsigned *>(smem + L.off_bar + 2 * SMV_MAX_STAGES * 8);
    moe_ring_init(smem, L.off_bar, S);
    __syncthreads();
    trace_entry(a.tr);
    pdl_launch_dependents();

    if (warp == SMV_CONSUMER_WARPS) {
        if (lane == 0) {
            unsigned seq = 0;
            bool routed = false;
            const unsigned long long pol = l2_policy_evict_first();
            for (int gb = g0; gb < g1; gb += SMV_CONSUMER_WARPS) {
                int nw = min(SMV_CONSUMER_WARPS, g1 - gb);
                for (int s = 0; s < nseg; s++)
#pragma unroll 1
                    for (int w = 0; w < nw; w++, seq++) {
                        const int G = gb + w;
                        const unsigned char *base;
                        int lg;
                        if (G < gs) { base = a.S.base; lg = G; }
                        else {
                            if (!routed) { // the routed experts' addresses are known once the router has finished
                                pdl_wait();
                                for (int j = 0; j < a.k; j++) s_base[j] = a.bases[__ldcg(a.ids + j)];
                                routed = true;
                            }
                            const int j = (G - gs) / gx;
                            lg = G - gs - j * gx;
                            base = s_base[j];
                        }
                        const int st = seq % S;
                        const unsigned ph = (seq / S) & 1u;
                        mbar_wait(bar0 + 8 * (SMV_MAX_STAGES + st), ph ^ 1u);
                        const unsigned full = bar0 + 8 * st;
                        mbar_expect_tx(full, tile_bytes);
                        bulk_g2s_evict_first(smem_u32(smem + L.off_ring + (size_t)st * L.stage_bytes), base + ((size_t)lg * nseg + s) * tile_bytes, tile_bytes,
                                             full, pol);
                    }
            }
        }
        return;
    }

    pdl_wait();
    trace_mark(a.tr, 2);
    const int cols = a.S.cols;
    {
        int4 *sxq = reinterpret_cast<int4 *>(smem + L.off_xq);
        float *sxs = reinterpret_cast<float *>(smem + L.off_xs);
        const int4 *src = reinterpret_cast<const int4 *>(a.xq);
        for (int c = tid; c < cols / 16; c += SMV_CONSUMER_WARPS * 32) sxq[c] = __ldcg(src + c);
        for (int b = tid; b < cols / 32; b += SMV_CONSUMER_WARPS * 32) sxs[b] = __ldcg(a.xs + b);
    }
    consumer_bar_sync();

    const int seg = a.S.seg, nbs = seg >> 5;
    float *terms = reinterpret_cast<float *>(smem + L.off_terms) + (size_t)warp * 4 * L.nbs_pad;
    const unsigned char *sact = smem + L.off_xq;
    const float *sxs = reinterpret_cast<const float *>(smem + L.off_xs);
    float *hvals = reinterpret_cast<float *>(smem + L.off_hvals);

    unsigned seq_base = 0;
    for (int gb = g0; gb < g1; gb += SMV_CONSUMER_WARPS) {
        const int nw = min(SMV_CONSUMER_WARPS, g1 - gb);
        if (warp < nw) {
            const int G = gb + warp;
            float acc = 0.0f;
            for (int s = 0; s < nseg; s++) {
                const unsigned seq = seq_base + (unsigned)(s * nw + warp);
                const int st = seq % S;
                const unsigned lap = seq / S;
                if (lane == 0)
                    while (rel[st] != lap) {}
                __syncwarp();
                mbar_wait(bar0 + 8 * st, lap & 1u);
                const unsigned char *tile = smem + L.off_ring + (size_t)st * L.stage_bytes;
                moe_tile_terms(tile, sact + ((size_t)s * seg), sxs + s * nbs, a.S.unit_bytes, seg, nbs, terms, L.nbs_pad, lane);
                __syncwarp();
                if (lane == 0) {
                    rel[st] = lap + 1u;
                    mbar_arrive(bar0 + 8 * (SMV_MAX_STAGES + st));
                }
                if (lane < 4) acc = pd_walk_terms(acc, terms + lane * L.nbs_pad, nbs);
                __syncwarp();
            }
            const float up = __shfl_down_sync(0xffffffffu, acc, 2);
            if (lane < 2) {
                const int unit = 2 * G + lane;
                const float hval = swiglu_exact(acc, up);
                a.out[unit] = hval;
                hvals[unit - 2 * g0] = hval;
            }
        }
        seq_base += (unsigned)(nseg * nw);
    }

    // Q8_0 of the virtual hidden vector: whole 32-unit blocks from shared memory, blocks shared with a neighbouring CTA by the
    // CTA that arrives last (the dense gate/up epilogue)
    consumer_bar_sync();
    const int u0 = 2 * g0, u1 = 2 * g1;
    if (u1 > u0) {
        for (int blk = (u0 >> 5) + warp; blk <= ((u1 - 1) >> 5); blk += SMV_CONSUMER_WARPS) {
            const int lo = max(blk << 5, u0), hi = min((blk << 5) + 32, u1);
            float v = 0.0f;
            bool mine = true;
            if (hi - lo == 32) v = hvals[(blk << 5) + lane - u0];
            else {
                unsigned old = 0;
                if (lane == 0) {
                    __threadfence();
                    old = atomicAdd(&a.blk_cnt[blk], (unsigned)(hi - lo));
                }
                old = __shfl_sync(0xffffffffu, old, 0);
                mine = (old + (unsigned)(hi - lo) == 32u);
                if (mine) {
                    __threadfence();
                    v = ldcg_f32(a.out + (blk << 5) + lane);
                    if (lane == 0) a.blk_cnt[blk] = 0u;
                }
            }
            if (mine) {
                float as;
                const int q = quant_block_lane(v, as);
                a.hq[(blk << 5) + lane] = (int8_t)q;
                if (lane == 0) a.hs[blk] = as;
            }
        }
    }
    trace_mark(a.tr, 3);
}

// Down projections of the shared expert and the k routed experts, one CTA owning rows [4 g0, 4 g1) of all k + 1 matrices, and
// the combine as the epilogue: saxpyInPlace (FloatTensor.java:221-227) x[i] = w_j * y_j[i] + x[i] -- a float multiply, then a
// float add -- for j in selection order, then the shared expert with its sigmoid weight (InferenceCore.java:404-423).
__global__ void __launch_bounds__(SMV_THREADS, 1) k_moe_down(MoeStreamArgs a, MoeDownSmem L) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ const unsigned char *s_base[MOE_MAX_K];
    __shared__ float s_w[MOE_MAX_K + 1];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int S = L.stages;
    const unsigned bar0 = smem_u32(smem + L.off_bar);
    const int ngroups = a.S.rows >> 2; // rows = dim for every matrix
    const int g0 = (int)(((long long)blockIdx.x * ngroups) / gridDim.x);
    const int g1 = (int)(((long long)(blockIdx.x + 1) * ngroups) / gridDim.x);
    const int nm = a.k + 1;
    volatile unsigned *rel = reinterpret_cast<volatile unsigned *>(smem + L.off_bar + 2 * SMV_MAX_STAGES * 8);
    moe_ring_init(smem, L.off_bar, S);
    __syncthreads();
    trace_entry(a.tr);
    pdl_launch_dependents();

    if (warp == SMV_CONSUMER_WARPS) {
        if (lane == 0) {
            unsigned seq = 0;
            bool routed = false;
            const unsigned long long pol = l2_policy_evict_first();
            for (int gb = g0; gb < g1; gb += SMV_CONSUMER_WARPS) {
                const int nw = min(SMV_CONSUMER_WARPS, g1 - gb);
                for (int m = 0; m < nm; m++) {
                    const unsigned char *base = a.S.base;
                    if (m > 0) {
                        if (!routed) {
                            pdl_wait();
                            for (int j = 0; j < a.k; j++) s_base[j] = a.bases[__ldcg(a.ids + j)];
                            routed = true;
                        }
                        base = s_base[m - 1];
                    }
                    const MoeMat M = moe_mat(a, m);
                    const unsigned tile_bytes = 4u * (unsigned)M.unit_bytes;
                    for (int s = 0; s < M.nseg; s++)
#pragma unroll 1
                        for (int w = 0; w < nw; w++, seq++) {
                            const int st = seq % S;
                            const unsigned ph = (seq / S) & 1u;
                            mbar_wait(bar0 + 8 * (SMV_MAX_STAGES + st), ph ^ 1u);
                            const unsigned full = bar0 + 8 * st;
                            mbar_expect_tx(full, tile_bytes);
                            bulk_g2s_evict_first(smem_u32(smem + L.off_ring + (size_t)st * L.stage_bytes), base + ((size_t)(gb + w) * M.nseg + s) * tile_bytes,
                                                 tile_bytes, full, pol);
                        }
                }
            }
        }
        return;
    }

    pdl_wait();
    trace_mark(a.tr, 2);
    const int hv = a.S.cols + a.k * a.X.cols;
    {
        int4 *sxq = reinterpret_cast<int4 *>(smem + L.off_xq);
        float *sxs = reinterpret_cast<float *>(smem + L.off_xs);
        const int4 *src = reinterpret_cast<const int4 *>(a.xq);
        for (int c = tid; c < hv / 16; c += SMV_CONSUMER_WARPS * 32) sxq[c] = __ldcg(src + c);
        for (int b = tid; b < hv / 32; b += SMV_CONSUMER_WARPS * 32) sxs[b] = __ldcg(a.xs + b);
        if (tid < nm) s_w[tid] = __ldcg(a.weights + tid);
    }
    consumer_bar_sync();

    float *terms = reinterpret_cast<float *>(smem + L.off_terms) + (size_t)warp * 4 * L.nbs_pad;
    const unsigned char *sact = smem + L.off_xq;
    const float *sxs = reinterpret_cast<const float *>(smem + L.off_xs);

    unsigned seq_base = 0;
    for (int gb = g0; gb < g1; gb += SMV_CONSUMER_WARPS) {
        const int nw = min(SMV_CONSUMER_WARPS, g1 - gb);
        unsigned off = 0; // tiles of this chunk issued before matrix m
        if (warp < nw) {
            const int row = 4 * (gb + warp) + (lane & 3);
            float xv = lane < 4 ? ldcg_f32(a.out + row) : 0.0f, ysh = 0.0f;
            for (int m = 0; m < nm; m++) {
                const MoeMat M = moe_mat(a, m);
                const int nbs = M.seg >> 5;
                float acc = 0.0f;
                for (int s = 0; s < M.nseg; s++) {
                    const unsigned seq = seq_base + off + (unsigned)(s * nw + warp);
                    const int st = seq % S;
                    const unsigned lap = seq / S;
                    if (lane == 0)
                        while (rel[st] != lap) {}
                    __syncwarp();
                    mbar_wait(bar0 + 8 * st, lap & 1u);
                    const unsigned char *tile = smem + L.off_ring + (size_t)st * L.stage_bytes;
                    const int c0 = M.act_off + s * M.seg;
                    moe_tile_terms(tile, sact + c0, sxs + (c0 >> 5), M.unit_bytes, M.seg, nbs, terms, L.nbs_pad, lane);
                    __syncwarp();
                    if (lane == 0) {
                        rel[st] = lap + 1u;
                        mbar_arrive(bar0 + 8 * (SMV_MAX_STAGES + st));
                    }
                    if (lane < 4) acc = pd_walk_terms(acc, terms + lane * L.nbs_pad, nbs);
                    __syncwarp();
                }
                off += (unsigned)(M.nseg * nw);
                if (m == 0) ysh = acc;                              // the shared expert is added last
                else xv = __fadd_rn(__fmul_rn(s_w[m - 1], acc), xv); // routed slot m - 1, in selection order
            }
            xv = __fadd_rn(__fmul_rn(s_w[a.k], ysh), xv);
            if (lane < 4) a.out[row] = xv;
        } else {
            for (int m = 0; m < nm; m++) off += (unsigned)(moe_mat(a, m).nseg * nw);
        }
        seq_base += off;
    }
    trace_mark(a.tr, 3);
}
