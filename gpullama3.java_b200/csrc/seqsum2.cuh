// seqsum2.cuh -- exact, parallel evaluation of a SEQUENTIAL float32 sum of non-negative terms: the accumulator of the decode
// path's RMSNorms and of the sampler's softmax (the algorithm is validated on the CPU by tools/seqsum2/proto.c, on the GPU by
// tests/test_gpu_parity.py).
//
// The reference's RMSNorm accumulates  s = ((0 + t0) + t1) + ...  one float add at a time (InferenceCore.rmsnorm,
// InferenceCore.java:39-48 via FloatTensor.reduce, FloatTensor.java:110-116).  Float addition is not associative, so a tree
// reduction gives different bits, and a literal chain costs ~8-10 cycles per term on one thread.  This file returns the
// chain's bit-exact value, evaluated by one CTA:
//
//   While the running sum s stays inside one binade [2^e, 2^(e+1)) its mantissa M is an integer in units of u = 2^(e-23), and
//   adding a term t rounds to  M + k + [f > 1/2]  with t/u = k + f (on an exact tie, f == 1/2, round-half-even makes the
//   increment depend on the parity of M; real activations produce 3-30 ties per 4096 terms).  So inside a binade a step is the
//   integer map  M -> M + a[M & 1], and such maps compose associatively.  The evaluation takes three barriers and a short
//   serial walk:
//   1. float prefix P over per-thread sums (E consecutive terms per thread): a warp scan, barrier 1, and every warp adds
//      the totals of the warps before it                                                  -> predicted binade per thread
//   2. a thread whose P range lies well inside one binade composes its E steps  M -> M + a[M & 1]  (SeqPair)
//      into one pair ("clean"); any other thread is "literal"
//   3. inside each warp: segmented scan of the pairs over runs of clean threads with equal binade (pairs compose
//      associatively), and ballot/popc compaction into the warp's own item slots: one item per literal thread and one
//      per run; a run that spans warps becomes one item per warp.  Barrier 2.
//   4. warp 0 walks the items: literal = E real float adds; run = verify (exponent on entry, mantissa < 2^24 on exit) and
//      add the integer; a failed check replays the item literally.  Each item is verified on its own, so where runs are
//      cut and what the predictor says decide speed, never the result.  Barrier 3 hands the sum to every thread.
// CPU model (tools/seqsum2/emulate_v2.py, adversarial cases up to n = 16384 at 256 / 512 / 1024 threads): 0 mismatches.
#pragma once
#include "common.cuh"

#define SEQSUM2_THREADS 1024
#define SEQSUM2_LITERAL INT_MIN

struct SeqPair { // the step  M -> M + a[M & 1]
    unsigned a0, a1;
};
__device__ __forceinline__ SeqPair seq_compose(SeqPair L, SeqPair R) { // apply L, then R
    SeqPair o;
    o.a0 = L.a0 + ((L.a0 & 1u) ? R.a1 : R.a0);
    o.a1 = L.a1 + (((1u + L.a1) & 1u) ? R.a1 : R.a0);
    o.a0 = min(o.a0, 1u << 26); // saturate: anything >= 2^24 fails verification anyway
    o.a1 = min(o.a1, 1u << 26);
    return o;
}

__device__ __forceinline__ int f32_exponent(float f) { return (int)((__float_as_uint(f) >> 23) & 0xffu) - 127; }

// Parity pair of adding t to a running sum in binade e, with scale = 2^(23-e): t / ulp = t * scale is exact, and one fused
// multiply-add rounds it to an integer with ties to even, which is the step when M is even.  When M is odd only an exact tie
// (rounding error +-1/2) steps differently: to the other, odd, neighbour.  Returns false when t * scale >= 2^23, i.e.
// t >= 2^e (no step of a sum that stays inside [2^e, 2^(e+1)) with margin), or t is inf / NaN.  Zero and denormal terms
// give (0, 0).
__device__ __forceinline__ bool seq_pair(float t, float scale, SeqPair &pr) {
    const float kf = __fmul_rn(t, scale), r = __fmaf_rn(t, scale, 0x1p23f);
    const unsigned a0 = __float_as_uint(r) - 0x4b000000u; // r = 2^23 + the rounded integer
    const float d = __fsub_rn(__fsub_rn(r, 0x1p23f), kf);  // exact: the rounding error, in [-1/2, 1/2]
    pr.a0 = a0;
    pr.a1 = fabsf(d) == 0.5f ? (d > 0.0f ? a0 - 1u : a0 + 1u) : a0;
    return kf < 0x1p23f;
}

struct SeqItem {
    unsigned ebits;   // a run in binade e: e + 127, the exponent field of every sum inside it; a literal thread: ~0u
    unsigned a0, a1;  // the run's composed pair
    unsigned idx;     // first thread | last thread << 10 | slot of the next item << 20 (T: the end of the list)
};

// Warp w writes its items to items[32 w ..]; every warp has at least one (its lane 31 always closes an item).
struct SeqSum2Scratch {
    SeqItem *items;   // [T]
    float *wsum;      // [32] warp totals of the per-thread sums
    int *info;        // [3] {items, fallbacks, literal items}, written by thread 0 (valid in that thread on return)
    float *result;    // [1]
};
__host__ __device__ inline size_t seqsum2_scratch_bytes(int T = SEQSUM2_THREADS) { // T = threads that run the accumulator
    return (size_t)T * sizeof(SeqItem) + 32 * 4 + 16;
}
__device__ __forceinline__ SeqSum2Scratch seqsum2_carve(unsigned char *p, int T = SEQSUM2_THREADS) { // p 16-byte aligned
    SeqSum2Scratch s;
    s.items = reinterpret_cast<SeqItem *>(p); p += (size_t)T * sizeof(SeqItem);
    s.wsum = reinterpret_cast<float *>(p); p += 32 * 4;
    s.info = reinterpret_cast<int *>(p);
    s.result = reinterpret_cast<float *>(p + 12);
    return s;
}

struct SeqSum2BlockSync {
    __device__ __forceinline__ void operator()() const { __syncthreads(); }
};

// Chunk stride that makes the 16-byte reads of consecutive threads hit distinct shared-memory banks (E = terms per thread):
// thread t's terms live at sq[t * S .. t * S + E).  E = 16 -> 20, 8 -> 12, 32 -> 36, 4 -> 4.
__host__ __device__ inline int seqsum2_stride(int E) { return (E % 4 == 0 && (E / 4) % 2 == 0) ? E + 4 : E; }

// literal adds of one thread's E terms (16-byte loads when the layout allows, 16 terms requested before their adds start)
__device__ __forceinline__ float seq2_literal(float s, const float *q, int E, bool vec) {
    int k = 0;
    if (vec) {
#pragma unroll 1
        for (; k + 16 <= E; k += 16) {
            const float4 v0 = *reinterpret_cast<const float4 *>(q + k), v1 = *reinterpret_cast<const float4 *>(q + k + 4);
            const float4 v2 = *reinterpret_cast<const float4 *>(q + k + 8), v3 = *reinterpret_cast<const float4 *>(q + k + 12);
            s = __fadd_rn(s, v0.x); s = __fadd_rn(s, v0.y); s = __fadd_rn(s, v0.z); s = __fadd_rn(s, v0.w);
            s = __fadd_rn(s, v1.x); s = __fadd_rn(s, v1.y); s = __fadd_rn(s, v1.z); s = __fadd_rn(s, v1.w);
            s = __fadd_rn(s, v2.x); s = __fadd_rn(s, v2.y); s = __fadd_rn(s, v2.z); s = __fadd_rn(s, v2.w);
            s = __fadd_rn(s, v3.x); s = __fadd_rn(s, v3.y); s = __fadd_rn(s, v3.z); s = __fadd_rn(s, v3.w);
        }
#pragma unroll 1
        for (; k + 4 <= E; k += 4) {
            const float4 v = *reinterpret_cast<const float4 *>(q + k);
            s = __fadd_rn(s, v.x); s = __fadd_rn(s, v.y); s = __fadd_rn(s, v.z); s = __fadd_rn(s, v.w);
        }
    }
#pragma unroll 1
    for (; k < E; k++) s = __fadd_rn(s, q[k]);
    return s;
}

// sq: n terms, thread t's E = ceil(n / T) consecutive terms at sq[t * S + k] (S >= E; S = E is the plain contiguous layout),
// zero-padded up to T whole chunks.  Exactly T threads (a multiple of 32, at most SEQSUM2_THREADS) call this with tid in
// [0, T); `sync` is a barrier over those T threads (the whole CTA, or a named barrier over a subset of its warps as in the
// persistent decode kernel).  When S and E are multiples of 4 and sq is 16-byte aligned the terms are read with 16-byte loads.
// Every thread returns the sum.
template <int T, class Sync>
__device__ float block_seqsum_exact_v2_t(const float *sq, int n, SeqSum2Scratch sc, int tid, Sync sync, int S = 0) {
    static_assert(T % 32 == 0 && T <= SEQSUM2_THREADS, "T threads = T/32 whole warps");
    const int lane = tid & 31, warp = tid >> 5;
    const int E = (n + T - 1) / T;
    if (S == 0) S = E;
    const bool vec = ((E | S) & 3) == 0 && (reinterpret_cast<uintptr_t>(sq) & 15) == 0;
    const float *mine = sq + tid * S;

    // ---- 1. float prefix over per-thread sums (a predictor: plain adds in any order)
    float loc = 0.0f;
    {
        int k = 0;
        if (vec) {
#pragma unroll 1
            for (; k < E; k += 4) {
                const float4 v = *reinterpret_cast<const float4 *>(mine + k);
                loc += v.x; loc += v.y; loc += v.z; loc += v.w;
            }
        }
#pragma unroll 1
        for (; k < E; k++) loc += mine[k];
    }
    float inc = loc;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const float u = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += u;
    }
    if (lane == 31) sc.wsum[warp] = inc;
    sync(); // barrier 1: the warp totals
    float wex = lane < warp ? sc.wsum[lane] : 0.0f; // every warp forms its own offset
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) wex += __shfl_xor_sync(0xffffffffu, wex, d);
    const float p_end = wex + inc, p_start = wex + (inc - loc);

    // ---- 2. classify, compose the thread's own steps
    int cls = SEQSUM2_LITERAL;
    SeqPair pr;
    pr.a0 = pr.a1 = 0u;
    {
        const int e = f32_exponent(p_start);
        if (p_start > 0.0f && e > -100 && e < 128 && f32_exponent(p_end) == e) { // e == 128: inf/nan prefix -> literal adds
            const float b = __uint_as_float((unsigned)(e + 127) << 23), scale = __uint_as_float((unsigned)(150 - e) << 23);
            // margin 2^-9: the sequential sum deviates from any exact prefix by < n * 2^-24 relative (n <= 16384 -> 2^-10)
            if (p_start >= b * (1.0f + 0x1p-9f) && p_end <= 2.0f * b * (1.0f - 0x1p-9f)) {
                bool ok = true;
                int k = 0;
                if (vec)
#pragma unroll 1
                    for (; k < E; k += 4) { // four independent pair evaluations, composed as a tree: the dependent chain is E/4 + 2 composes, not E
                        const float4 v = *reinterpret_cast<const float4 *>(mine + k);
                        SeqPair q0, q1, q2, q3;
                        const bool o0 = seq_pair(v.x, scale, q0), o1 = seq_pair(v.y, scale, q1), o2 = seq_pair(v.z, scale, q2), o3 = seq_pair(v.w, scale, q3);
                        ok = ok && o0 && o1 && o2 && o3; // composing an invalid pair is harmless: the result is discarded
                        pr = seq_compose(pr, seq_compose(seq_compose(q0, q1), seq_compose(q2, q3)));
                    }
#pragma unroll 1
                for (; ok && k < E; k++) {
                    SeqPair q;
                    if (!seq_pair(mine[k], scale, q)) { ok = false; break; }
                    pr = seq_compose(pr, q);
                }
                if (ok) cls = e;
            }
        }
    }

    // ---- 3. runs of clean threads with equal binade, cut at warp boundaries: segmented scan of the pairs inside the warp,
    // then one item per literal thread and one per run, compacted into the warp's own slots
    const bool clean = cls != SEQSUM2_LITERAL;
    const int prev_cls = __shfl_up_sync(0xffffffffu, cls, 1), next_cls = __shfl_down_sync(0xffffffffu, cls, 1);
    int f = (clean && lane > 0 && prev_cls == cls) ? 0 : 1; // 1 = a run (or a literal thread) starts here
    const bool is_item = !clean || lane == 31 || next_cls != cls;
    const unsigned starts = __ballot_sync(0xffffffffu, f), bal = __ballot_sync(0xffffffffu, is_item);
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const unsigned u0 = __shfl_up_sync(0xffffffffu, pr.a0, d), u1 = __shfl_up_sync(0xffffffffu, pr.a1, d);
        const int fu = __shfl_up_sync(0xffffffffu, f, d);
        if (lane >= d && !f) {
            SeqPair L;
            L.a0 = u0; L.a1 = u1;
            pr = seq_compose(L, pr);
            f = fu;
        }
    }
    if (is_item) {
        const int slot = warp * 32 + __popc(bal & ((1u << lane) - 1u));
        const int first = warp * 32 + 31 - __clz(starts & (0xffffffffu >> (31 - lane)));
        const int next = (bal >> lane) > 1u ? slot + 1 : (warp + 1) * 32;
        SeqItem it;
        it.ebits = clean ? (unsigned)(cls + 127) : ~0u; it.a0 = pr.a0; it.a1 = pr.a1; it.idx = (unsigned)first | ((unsigned)tid << 10) | ((unsigned)next << 20);
        sc.items[slot] = it;
    }
    sync(); // barrier 2: the items

    // ---- 4. resolver: warp 0 walks the items (every lane the same; one warp alone keeps the whole issue rate of its
    // scheduler), barrier 3 hands the sum to the other warps
    if (warp == 0) {
        unsigned sb = 0u; // the bits of the running sum (s >= 0)
        int items = 0, fallbacks = 0, literals = 0;
        SeqItem nxt = sc.items[0];
#pragma unroll 1
        for (int i = 0; i < T; items++) {
            const SeqItem it = nxt;
            i = (int)(it.idx >> 20);
            nxt = sc.items[min(i, T - 1)]; // in flight while this item is resolved
            // a run on the float's bits: the mantissa's parity is the bit pattern's, and M + a < 2^24 exactly when the add
            // leaves the exponent field alone; a denormal, inf or NaN sum and a literal thread never match ebits
            const unsigned nb = sb + ((sb & 1u) ? it.a1 : it.a0);
            if ((sb >> 23) == it.ebits && (nb >> 23) == it.ebits) {
                sb = nb;
                continue;
            }
            fallbacks += it.ebits != ~0u; // a misprediction; otherwise a literal thread: replay the item's threads literally
            literals += it.ebits == ~0u;
            const int last = (int)((it.idx >> 10) & 1023u);
            float s = __uint_as_float(sb);
#pragma unroll 1
            for (int j = (int)(it.idx & 1023u); j <= last; j++) s = seq2_literal(s, sq + j * S, E, vec);
            sb = __float_as_uint(s);
        }
        if (lane == 0) { sc.info[0] = items; sc.info[1] = fallbacks; sc.info[2] = literals; sc.result[0] = __uint_as_float(sb); }
    }
    sync(); // barrier 3: the sum
    return sc.result[0];
}

// The whole-CTA form used by k_rmsnorm_quant: SEQSUM2_THREADS threads, __syncthreads.
__device__ __forceinline__ float block_seqsum_exact_v2(const float *sq, int n, SeqSum2Scratch sc) {
    return block_seqsum_exact_v2_t<SEQSUM2_THREADS>(sq, n, sc, (int)threadIdx.x, SeqSum2BlockSync());
}
