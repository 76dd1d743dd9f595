// decode_batch.cuh -- the batched step: up to SMB_MAX_ROWS rows, each a (slot, token, position), advance together while every
// weight matrix streams from HBM once (b200_forward_decode_batch, b200_forward_decode_multi, b200_forward_step and the exact
// prefills, plan.cu).  Each dot product keeps its own row, its own activation vector and its own block order, so every row stays
// bit-identical to the single-sequence decode (and the CPU path).
//
//   k_rmsnorm_quant_batch      one CTA per row: rmsnorm_quant_row (decode_kernels.cuh) on that row's x / token / outputs
//   k_stream_matvec_q8_batch   the tile-major Q8_0 stream of stream_matvec.cuh; each tile is applied to every row's activation
//   k_attention_batch          grid (heads, rows): attention_head (decode_kernels.cuh) on the row's slot cache and position
//   k_rope_kv_batch + k_attention_cached_rows   the same attention split in two, for steps whose rows share a sequence
//   k_argmax_batch             one CTA per row: merges that row's lm_head partials (first strict maximum)
#pragma once
#include "decode_kernels.cuh"
#include "stream_matvec.cuh"

#define SMB_MAX_ROWS 8 // one warp walks 4 weight rows x SMB_MAX_ROWS activation rows = 32 sequential chains, one per lane
#define SMB_TSTRIDE 36 // floats per chain in the per-warp term buffer: 32 terms, 16-byte aligned rows, conflict-free LDS.128 walks

// Per-step inputs of the batched graph, uploaded before each launch.
struct BatchRows {
    int token[SMB_MAX_ROWS];
    int pos[SMB_MAX_ROWS];
    int slot[SMB_MAX_ROWS];
};

// Exact multi-slot prefill (b200_prefill_slots): the first node of each step's graph copies entry *step of the schedule uploaded
// with the call into rows and advances *step, so the steps of one call are enqueued back to back with no host round trip.
__global__ void __launch_bounds__(32) k_batch_rows_next(const BatchRows *__restrict__ sched, int *step, BatchRows *__restrict__ rows) {
    const int s = *step;
    const int *src = reinterpret_cast<const int *>(sched + s);
    int *dst = reinterpret_cast<int *>(rows);
    for (int i = threadIdx.x; i < (int)(sizeof(BatchRows) / 4); i += 32) dst[i] = src[i];
    __syncwarp();
    if (threadIdx.x == 0) *step = s + 1;
}

// The norm and attention kernels take the (unused: tr.rec == nullptr, tp.n == 1) trace and tensor-parallel contexts as kernel
// parameters, as the single-row kernels do: a zero-initialised local copy would be placed in local memory.

// ---- RMSNorm + quantisation, one CTA per row ------------------------------------------------------------------------------
template <bool EMBED>
__global__ void __launch_bounds__(NORM_THREADS, 1) k_rmsnorm_quant_batch(float *__restrict__ x, const BatchRows *__restrict__ rows, DevMat emb,
                                                                     float emb_scale, const float *__restrict__ w, float eps, int dim,
                                                                     int8_t *__restrict__ xq, float *__restrict__ xs, TraceBuf tr, TpCtx tp) {
    const int v = blockIdx.x;
    rmsnorm_quant_row<EMBED>(x + (size_t)v * dim, rows->token + v, emb, emb_scale, w, eps, dim, xq + (size_t)v * dim, xs + (size_t)v * (dim / 32),
                             nullptr, nullptr, tr, tp, -1);
}

// ---- attention, grid (heads, rows) ----------------------------------------------------------------------------------------
// kc / vc: this layer's rows of slot 0's cache; slot s starts slot_stride floats further.
template <int HS>
__global__ void __launch_bounds__(ATT_THREADS) k_attention_batch(float *__restrict__ qkv, int qkv_stride, float *__restrict__ kc, float *__restrict__ vc,
                                                                size_t slot_stride, const BatchRows *__restrict__ rows, const float *__restrict__ cr,
                                                                const float *__restrict__ ci, int n_heads, int n_kv_heads, int arch,
                                                                const float *__restrict__ qnorm_w, const float *__restrict__ knorm_w,
                                                                const float *__restrict__ qkv_bias, float eps, float sqrt_hs,
                                                                int8_t *__restrict__ xq, float *__restrict__ xs, float *att_scratch, int ctx,
                                                                TraceBuf tr, TpCtx tp) {
    const int v = blockIdx.y, qd = n_heads * HS;
    const size_t base = (size_t)rows->slot[v] * slot_stride; // host-written before the graph launch: readable before the dependency wait
    attention_head<HS>(qkv + (size_t)v * qkv_stride, kc + base, vc + base, rows->pos + v, cr, ci, n_heads, n_kv_heads, arch, qnorm_w, knorm_w,
                       qkv_bias, eps, sqrt_hs, xq + (size_t)v * qd, xs + (size_t)v * (qd / 32), nullptr, tr, tp, 0u, 0,
                       att_scratch ? att_scratch + (size_t)v * n_heads * ctx : nullptr, ctx);
}

// ---- same-sequence steps: RoPE / KV write, then attention from the cache ----------------------------------------------------
// Rows of one step may be consecutive positions of ONE sequence (b200_forward_decode_multi, the exact prefills): row i attends to
// the K / V rows i' < i write.  k_attention_batch writes its row's K / V inside the attention CTA, so those rows would race;
// here a separate grid writes every row's K / V first, and the attention reads them only after its dependency wait (the
// previous grid complete), with no CTA ever waiting on another of its own grid.
//   k_rope_kv_batch            grid (heads, rows), 2 x HS threads: rope_kv_prologue, rotated q back into qkv, k / v into the cache
//   k_attention_cached_rows   grid (heads, rows): attention_head<HS, true>, every key t <= pos from the cache
template <int HS>
__global__ void __launch_bounds__(2 * HS) k_rope_kv_batch(float *__restrict__ qkv, int qkv_stride, float *__restrict__ kc, float *__restrict__ vc,
                                                         size_t slot_stride, const BatchRows *__restrict__ rows, const float *__restrict__ cr,
                                                         const float *__restrict__ ci, int n_heads, int n_kv_heads, int arch,
                                                         const float *__restrict__ qnorm_w, const float *__restrict__ knorm_w,
                                                         const float *__restrict__ qkv_bias, float eps) {
    __shared__ __align__(16) float sq[HS], sk[HS], so[HS];
    __shared__ float s_val[2];
    const int v = blockIdx.y, h = blockIdx.x;
    const size_t base = (size_t)rows->slot[v] * slot_stride;
    const int kv_mul = n_heads / n_kv_heads, kvh = h / kv_mul;
    pdl_launch_dependents();
    pdl_wait();
    const int qd = n_heads * HS, kvd = n_kv_heads * HS;
    float *q = qkv + (size_t)v * qkv_stride;
    rope_kv_prologue<HS>(q, q + h * HS, q + qd + kvh * HS, q + qd + kvd + kvh * HS, kc + base, vc + base, rows->pos[v], h, kv_mul, kvh, qd, kvd, cr,
                         ci, arch, qnorm_w, knorm_w, qkv_bias, eps, sq, sk, so, s_val);
}

template <int HS>
__global__ void __launch_bounds__(ATT_THREADS) k_attention_cached_rows(float *__restrict__ qkv, int qkv_stride, float *__restrict__ kc,
                                                                       float *__restrict__ vc, size_t slot_stride, const BatchRows *__restrict__ rows,
                                                                       int n_heads, int n_kv_heads, int arch, float sqrt_hs, int8_t *__restrict__ xq,
                                                                       float *__restrict__ xs, float *att_scratch, int ctx, TraceBuf tr, TpCtx tp) {
    const int v = blockIdx.y, qd = n_heads * HS;
    const size_t base = (size_t)rows->slot[v] * slot_stride;
    attention_head<HS, true>(qkv + (size_t)v * qkv_stride, kc + base, vc + base, rows->pos + v, nullptr, nullptr, n_heads, n_kv_heads, arch, nullptr,
                             nullptr, nullptr, 0.0f, sqrt_hs, xq + (size_t)v * qd, xs + (size_t)v * (qd / 32), nullptr, tr, tp, 0u, 0,
                             att_scratch ? att_scratch + (size_t)v * n_heads * ctx : nullptr, ctx);
}

// ---- the batched Q8_0 stream ----------------------------------------------------------------------------------------------
// Shared memory: the ring and the producer are those of k_stream_matvec_q8.  Of the activations only the SEGMENT being consumed is
// staged (all rows of it): staging whole vectors, as the single-row kernel does, would take rows x 1.125 x cols bytes (129 KB for
// 8 rows of a 14336-column down projection).  The producer issues the tiles of a round of (up to) eight row groups segment by
// segment, so the consumer warps walk the segments in step anyway; two consumer barriers per segment swap the staged segment.
// Block terms are walked 32 blocks at a time, lane l holding the chain of (activation row l / 4, weight row l % 4).
struct SmbSmem {
    size_t off_bar, off_act, off_terms, off_cand, off_ring, total;
    int stages, stage_bytes;
};

__host__ __device__ inline SmbSmem smb_layout(int seg, int nrow, size_t budget) {
    SmbSmem L;
    L.stage_bytes = (4 * smv_unit_bytes(seg) + 127) & ~127;
    size_t o = 0;
    L.off_bar = o; o += ring_bar_bytes(SMV_MAX_STAGES);
    o = (o + 15) & ~(size_t)15;
    L.off_act = o; o += (size_t)nrow * seg + (size_t)nrow * (seg / 32) * 4; // quants [row][seg], then scales [row][seg / 32]
    o = (o + 15) & ~(size_t)15;
    L.off_terms = o; o += (size_t)SMV_CONSUMER_WARPS * 4 * nrow * SMB_TSTRIDE * 4;
    L.off_cand = o; o += (size_t)SMV_CONSUMER_WARPS * 32 * 8; // lm_head: per-lane (max, first index)
    ring_fit<SMV_MAX_STAGES>(L, o, budget);
    return L;
}

struct SmbArgs {
    TileMat W;
    int nrow;           // activation rows (sequences) of this launch
    const int8_t *xq;   // [nrow][cols] quantised activations
    const float *xs;    // [nrow][cols / 32] their block scales
    float *out;         // STORE: out[v][row] = r * oscale; RESID: out[v][row] += r * oscale; GATEUP: hb[v][unit]
    float oscale;       // Granite's logitScale / residualScale (SmvArgs::oscale); 1.0f otherwise
    int ostride;        // floats between two rows' outputs
    int8_t *hq;         // GATEUP: quantised hb [nrow][ostride]
    float *hs;          // GATEUP: its block scales [nrow][ostride / 32]
    unsigned *blk_cnt;  // GATEUP: per-(row, 32-block) arrival counters [nrow][ostride / 32] (self-resetting)
    float *part_val;    // STORE (lm_head): per-(row, CTA) maximum [nrow][gridDim.x] ...
    int *part_idx;      // ... and the lowest index attaining it, or NULL
};

template <int MODE>
__global__ void __launch_bounds__(SMV_THREADS, 1) k_stream_matvec_q8_batch(SmbArgs a, SmbSmem L) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const TileMat W = a.W;
    const int S = L.stages, nrow = a.nrow;
    const unsigned bar0 = smem_u32(smem + L.off_bar);
    const int ngroups = tile_groups(W);
    const int g0 = (int)(((long long)blockIdx.x * ngroups) / gridDim.x);
    const int g1 = (int)(((long long)(blockIdx.x + 1) * ngroups) / gridDim.x);
    const int nseg = W.nseg;
    const unsigned tile_bytes = 4u * (unsigned)W.unit_bytes;
    volatile unsigned *rel = reinterpret_cast<volatile unsigned *>(smem + L.off_bar + 2 * SMV_MAX_STAGES * 8);
    if (tid == 0) { // stream_ring_init's work, written out: through the shared helper this kernel's machine code changes
        for (int s = 0; s < S; s++) {
            mbar_init(bar0 + 8 * s, 1);
            mbar_init(bar0 + 8 * (SMV_MAX_STAGES + s), 1);
            rel[s] = 0u;
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    pdl_launch_dependents();

    if (warp == SMV_CONSUMER_WARPS) { // producer: k_stream_matvec_q8's walk
        if (lane == 0) {
            unsigned seq = 0;
            const unsigned long long pol = l2_policy_evict_first();
            for (int gb = g0; gb < g1; gb += SMV_CONSUMER_WARPS) {
                const int nw = min(SMV_CONSUMER_WARPS, g1 - gb);
                for (int s = 0; s < nseg; s++)
                    for (int w = 0; w < nw; w++, seq++) {
                        const int st = seq % S;
                        mbar_wait(bar0 + 8 * (SMV_MAX_STAGES + st), ((seq / S) & 1u) ^ 1u);
                        const unsigned full = bar0 + 8 * st;
                        mbar_expect_tx(full, tile_bytes);
                        const unsigned char *src = W.base + ((size_t)(gb + w) * nseg + s) * tile_bytes;
                        bulk_g2s_evict_first(smem_u32(smem + L.off_ring + (size_t)st * L.stage_bytes), src, tile_bytes, full, pol);
                    }
            }
        }
        return;
    }

    pdl_wait(); // activations come from the previous kernel
    const int seg = W.seg, nbs = seg >> 5, nb = W.cols >> 5;
    unsigned char *sact = smem + L.off_act;
    float *sxs = reinterpret_cast<float *>(sact + (size_t)nrow * seg);
    float *terms = reinterpret_cast<float *>(smem + L.off_terms) + (size_t)warp * 4 * nrow * SMB_TSTRIDE;
    const int hsel = (lane >> 2) & 1;
    const int nchain = 4 * nrow;
    float best = -INFINITY;
    int best_i = 0x7fffffff;

    unsigned seq_base = 0;
    for (int gb = g0; gb < g1; gb += SMV_CONSUMER_WARPS) {
        const int nw = min(SMV_CONSUMER_WARPS, g1 - gb);
        const bool live = warp < nw;
        const int G = gb + warp;
        float acc = 0.0f; // lane l < nchain: row 4G + l % 4 against activation row l / 4
        for (int s = 0; s < nseg; s++) {
            consumer_bar_sync(); // every warp is done with the previous segment
            {
                const int q16 = seg >> 4;
                for (int c = tid; c < nrow * q16; c += SMV_CONSUMER_WARPS * 32) {
                    const int v = c / q16, k = c - v * q16;
                    reinterpret_cast<int4 *>(sact)[c] = __ldcg(reinterpret_cast<const int4 *>(a.xq + (size_t)v * W.cols + (size_t)s * seg) + k);
                }
                for (int c = tid; c < nrow * nbs; c += SMV_CONSUMER_WARPS * 32) {
                    const int v = c / nbs, k = c - v * nbs;
                    sxs[c] = __ldcg(a.xs + (size_t)v * nb + (size_t)s * nbs + k);
                }
            }
            consumer_bar_sync();
            if (!live) continue;
            const unsigned seq = seq_base + (unsigned)(s * nw + warp);
            const int st = seq % S;
            const unsigned lap = seq / S;
            if (lane == 0)
                while (rel[st] != lap) {}
            __syncwarp();
            mbar_wait(bar0 + 8 * st, lap & 1u);
            const unsigned char *tile = smem + L.off_ring + (size_t)st * L.stage_bytes;
            for (int b0 = 0; b0 < nbs; b0 += 32) {
                const int b = b0 + lane;
                if (b < nbs) {
                    int4 w0[4], w1[4];
                    float wsc[4];
#pragma unroll
                    for (int r = 0; r < 4; r++) {
                        const unsigned char *wb = tile + (size_t)r * W.unit_bytes + ((size_t)b << 5);
                        w0[r] = *reinterpret_cast<const int4 *>(wb + 16 * hsel);
                        w1[r] = *reinterpret_cast<const int4 *>(wb + 16 * (hsel ^ 1));
                        wsc[r] = __half2float(*reinterpret_cast<const __half *>(tile + (size_t)r * W.unit_bytes + seg + 2 * b));
                    }
#pragma unroll 1
                    for (int v = 0; v < nrow; v++) {
                        const unsigned char *ab = sact + (size_t)v * seg + ((size_t)b << 5);
                        const int4 a0 = *reinterpret_cast<const int4 *>(ab + 16 * hsel);
                        const int4 a1 = *reinterpret_cast<const int4 *>(ab + 16 * (hsel ^ 1));
                        const float as = sxs[v * nbs + b];
#pragma unroll
                        for (int r = 0; r < 4; r++) {
                            int isum = __dp4a(w0[r].x, a0.x, 0);
                            isum = __dp4a(w0[r].y, a0.y, isum);
                            isum = __dp4a(w0[r].z, a0.z, isum);
                            isum = __dp4a(w0[r].w, a0.w, isum);
                            isum = __dp4a(w1[r].x, a1.x, isum);
                            isum = __dp4a(w1[r].y, a1.y, isum);
                            isum = __dp4a(w1[r].z, a1.z, isum);
                            isum = __dp4a(w1[r].w, a1.w, isum);
                            terms[(v * 4 + r) * SMB_TSTRIDE + lane] = __fmul_rn((float)isum, __fmul_rn(wsc[r], as));
                        }
                    }
                }
                __syncwarp();
                if (b0 + 32 >= nbs && lane == 0) { // last chunk read: the tile goes back to the producer
                    rel[st] = lap + 1u;
                    mbar_arrive(bar0 + 8 * (SMV_MAX_STAGES + st));
                }
                if (lane < nchain) acc = pd_walk_terms(acc, terms + lane * SMB_TSTRIDE, min(32, nbs - b0)); // strictly in block order
                __syncwarp();
            }
        }
        if (live) {
            const int v = lane >> 2, r = lane & 3;
            if (MODE == SMV_GATEUP) {
                const float up = __shfl_down_sync(0xffffffffu, acc, 2); // lanes 4v, 4v+1: gate rows; 4v+2, 4v+3: up rows
                if (lane < nchain && r < 2) a.out[(size_t)v * a.ostride + 2 * G + r] = swiglu_exact(acc, up);
            } else if (lane < nchain && 4 * G + r < W.rows) {
                const int row = 4 * G + r;
                float *o = a.out + (size_t)v * a.ostride + row;
                acc = __fmul_rn(acc, a.oscale);
                if (MODE == SMV_RESID) *o = __fadd_rn(*o, acc);
                else {
                    *o = acc;
                    if (acc > best) { best = acc; best_i = row; } // rows ascend per lane: first maximum kept
                }
            }
        }
        seq_base += (unsigned)(nseg * nw);
    }

    if (MODE == SMV_GATEUP) {
        // Quantise hb per row as k_stream_matvec_q8 does: 32-unit blocks inside this CTA's range from its own stores (ordered by the
        // barrier), blocks shared with a neighbouring CTA by whichever CTA arrives last.
        consumer_bar_sync();
        const int u0 = 2 * g0, u1 = 2 * g1;
        if (u1 > u0) {
            const int blo = u0 >> 5, nblk = ((u1 - 1) >> 5) - blo + 1, hblk = a.ostride >> 5;
            for (int k = warp; k < nrow * nblk; k += SMV_CONSUMER_WARPS) {
                const int v = k / nblk, blk = blo + k - v * nblk;
                const int lo = max(blk << 5, u0), hi = min((blk << 5) + 32, u1);
                float *hb = a.out + (size_t)v * a.ostride;
                float val = 0.0f;
                bool mine = true;
                if (hi - lo == 32) val = hb[(blk << 5) + lane];
                else {
                    unsigned old = 0;
                    if (lane == 0) {
                        __threadfence();
                        old = atomicAdd(&a.blk_cnt[v * hblk + blk], (unsigned)(hi - lo));
                    }
                    old = __shfl_sync(0xffffffffu, old, 0);
                    mine = (old + (unsigned)(hi - lo) == 32u);
                    if (mine) {
                        __threadfence();
                        val = ldcg_f32(hb + (blk << 5) + lane);
                        if (lane == 0) a.blk_cnt[v * hblk + blk] = 0u;
                    }
                }
                if (mine) {
                    float as;
                    const int q = quant_block_lane(val, as);
                    a.hq[(size_t)v * a.ostride + (blk << 5) + lane] = (int8_t)q;
                    if (lane == 0) a.hs[(size_t)v * hblk + blk] = as;
                }
            }
        }
    } else if (MODE == SMV_STORE && a.part_val) { // per-(row, CTA) (max, first index) for k_argmax_batch
        float *cv = reinterpret_cast<float *>(smem + L.off_cand);
        int *ci = reinterpret_cast<int *>(cv + SMV_CONSUMER_WARPS * 32);
        cv[warp * 32 + lane] = best;
        ci[warp * 32 + lane] = best_i;
        consumer_bar_sync();
        if (tid < nrow) {
            float bv = -INFINITY;
            int bi = 0x7fffffff;
            for (int w = 0; w < SMV_CONSUMER_WARPS; w++)
                for (int r = 0; r < 4; r++) {
                    const float x = cv[w * 32 + tid * 4 + r];
                    const int ix = ci[w * 32 + tid * 4 + r];
                    if (x > bv || (x == bv && ix < bi)) { bv = x; bi = ix; }
                }
            a.part_val[(size_t)tid * gridDim.x + blockIdx.x] = bv;
            a.part_idx[(size_t)tid * gridDim.x + blockIdx.x] = bi;
        }
    }
}

// ---- greedy ids: FloatTensor.argmax per row over the lm_head partials (k_argmax_advance's merge) ---------------------------
__global__ void __launch_bounds__(32) k_argmax_batch(const float *__restrict__ part_val, const int *__restrict__ part_idx, int n_part,
                                                     int *__restrict__ ids) {
    pdl_launch_dependents();
    pdl_wait();
    const int v = blockIdx.x, lane = threadIdx.x;
    float best = -INFINITY;
    int best_i = 0x7fffffff;
    for (int i = lane; i < n_part; i += 32) argmax_merge(best, best_i, part_val[(size_t)v * n_part + i], part_idx[(size_t)v * n_part + i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
        argmax_merge(best, best_i, ov, oi);
    }
    if (lane == 0) ids[v] = best_i == 0x7fffffff ? 0 : best_i;
}
