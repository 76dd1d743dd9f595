// sampler.cuh -- device-side temperature / top-p sampler (SURVEY.md 8f N3): the reference copies the whole logits row to the
// host whenever temperature > 0 and samples there (Sampler.selectSampler, inference/sampler/Sampler.java:74-122;
// CategoricalSampler.java:28-40; ToppSampler.java:62-156); here only the sampled id (4 bytes) leaves the GPU.
//
// Exactness: the kernel evaluates the reference's floats in the reference's order, so for the same uniform number r it
// returns the same token id:
//   logits[i] / temperature                       (divideInPlace, FloatTensor.java:203-205)           parallel
//   max, (float)Math.exp(x - max)                 (softmaxInPlace, FloatTensor.java:211-219)          parallel
//   sum = sequential float sum of the exps        exact + parallel: seqsum2.cuh (non-negative terms)
//   p[i] = e[i] / sum                                                                                  parallel
//   categorical: first i with r < cdf_i, cdf the sequential float prefix sum   -- one thread walks (early exit)
//   top-p: candidates p >= (1-topp)/(n-1) compacted in index order (parallel ordered scan), then the reference's own heap
//          (siftDown / pop until the cumulative probability exceeds topp, including its siftDown(..., i - 1)) and the final
//          cdf walk, by one thread: tie order among equal probabilities depends on the heap's mechanics, so the mechanics
//          are kept (n0 is a few hundred to a few thousand after the cutoff).
// The uniform number comes from the host (the Java RNG is host state: RandomGeneratorFactory.getDefault(), Sampler.java:84);
// 4 bytes in, 4 bytes out per token.
#pragma once
#include "common.cuh"
#include "seqsum2.cuh"

#define SAMPLER_THREADS 1024

struct SamplerArgs {
    float *logits;   // [n_pad] in/out: becomes the probability vector (as in the reference); n_pad = SAMPLER_THREADS * ceil(n / SAMPLER_THREADS), pad zero
    int n;
    float temperature, topp, r01;
    int *indices;    // [n] scratch (ToppSampler.indices)
    int *out_id;     // [1]
    int *info;       // [4] diagnostics: {n0 candidates, kept, seqsum items, seqsum fallbacks}
};

__host__ __device__ inline int sampler_padded(int n) { return (n + SAMPLER_THREADS - 1) / SAMPLER_THREADS * SAMPLER_THREADS; }
__host__ __device__ inline size_t sampler_smem_bytes() { return seqsum2_scratch_bytes(SAMPLER_THREADS) + 96 * 4; } // + red[32], redi[33]

__device__ __forceinline__ int sampler_cmp(const float *p, int a, int b) { // Comparator.comparingDouble(getFloat).reversed()
    const float va = p[a], vb = p[b];
    return vb < va ? -1 : (vb > va ? 1 : 0);
}
__device__ void sampler_sift_down(int *arr, int from, int n, const float *p) { // ToppSampler.siftDown (:32-46)
    int prev = from, next;
    while ((next = 2 * prev + 1) < n) {
        const int r = 2 * prev + 2;
        if (r < n && sampler_cmp(p, arr[r], arr[next]) < 0) next = r;
        if (sampler_cmp(p, arr[next], arr[prev]) < 0) {
            const int t = arr[prev]; arr[prev] = arr[next]; arr[next] = t;
            prev = next;
        } else break;
    }
}

// The sampler on one logits row, by one SAMPLER_THREADS-thread block with sampler_smem_bytes() of dynamic shared memory at smp_sm.
__device__ __forceinline__ void sample_row(const SamplerArgs &a, unsigned char *smp_sm) {
    SeqSum2Scratch scratch = seqsum2_carve(smp_sm, SAMPLER_THREADS);
    float *red = reinterpret_cast<float *>(smp_sm + seqsum2_scratch_bytes(SAMPLER_THREADS)); // [32] floats + [33] ints
    int *redi = reinterpret_cast<int *>(red + 32);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n = a.n;
    float *p = a.logits;

    // ---- temperature scaling + max
    float mx = -INFINITY;
    for (int i = tid; i < n; i += SAMPLER_THREADS) {
        const float v = __fdiv_rn(p[i], a.temperature);
        p[i] = v;
        mx = fmaxf(mx, v);
    }
    mx = warp_max_f(mx);
    if (lane == 0) red[warp] = mx;
    __syncthreads();
    mx = red[0];
    for (int w = 1; w < SAMPLER_THREADS / 32; w++) mx = fmaxf(mx, red[w]);
    // ---- exp (double, narrowed), exact sequential sum, normalise
    for (int i = tid; i < n; i += SAMPLER_THREADS) p[i] = (float)exp((double)__fsub_rn(p[i], mx));
    __syncthreads();
    const float sum = block_seqsum_exact_v2_t<SAMPLER_THREADS>(p, n, scratch, tid, SeqSum2BlockSync());
    if (tid == 0 && a.info) { a.info[2] = scratch.info[0]; a.info[3] = scratch.info[1]; }
    __syncthreads();
    for (int i = tid; i < n; i += SAMPLER_THREADS) p[i] = __fdiv_rn(p[i], sum);
    __syncthreads();

    const bool use_topp = a.topp > 0.0f && a.topp < 1.0f;
    if (!use_topp) { // CategoricalSampler (:28-40)
        if (tid == 0) {
            float cdf = 0.0f;
            int id = n - 1;
            for (int i = 0; i < n; i++) {
                cdf = __fadd_rn(cdf, p[i]);
                if (a.r01 < cdf) { id = i; break; }
            }
            *a.out_id = id;
            if (a.info) { a.info[0] = n; a.info[1] = n; }
        }
        return;
    }
    // ---- top-p: ordered compaction of the candidates (ToppSampler.java:70-78; the rejected tail is not written, see n0 == 0 below)
    const float cutoff = __fdiv_rn(__fsub_rn(1.0f, a.topp), (float)(n - 1));
    __shared__ int s_base;
    if (tid == 0) s_base = 0;
    __syncthreads();
    for (int c0 = 0; c0 < n; c0 += SAMPLER_THREADS) {
        const int i = c0 + tid;
        const bool keep = i < n && p[i] >= cutoff;
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) redi[warp] = __popc(bal);
        __syncthreads();
        if (warp == 0) {
            const int c = redi[lane];
            int v = c;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int u = __shfl_up_sync(0xffffffffu, v, d);
                if (lane >= d) v += u;
            }
            redi[lane] = v - c; // exclusive offset of each warp
            if (lane == 31) redi[32] = v; // chunk total
        }
        __syncthreads();
        if (keep) a.indices[s_base + redi[warp] + __popc(bal & ((1u << lane) - 1u))] = i;
        __syncthreads();
        if (tid == 0) s_base += redi[32];
        __syncthreads();
    }
    if (tid != 0) return;
    // ---- the reference's heap, verbatim mechanics (processTopP :114-156)
    int *idx = a.indices;
    const int n0 = s_base;
    if (n0 == 0) {
        // No candidate (a flat row with topp < 1/n, or NaN probabilities): the reference fills rejected ids in from the tail
        // (ToppSampler.java:71-77), so its indices[0] is n - 1, and with lastIndex = 0 it returns that slot (:155).  This kernel
        // writes only the candidates; every other path reads idx[0, n0) alone (last <= n0 - 1, siftDown(..., i - 1) < n0).
        *a.out_id = n - 1;
        if (a.info) { a.info[0] = 0; a.info[1] = 0; }
        return;
    }
    for (int i = n0 / 2 - 1; i >= 0; --i) sampler_sift_down(idx, i, n0, p);
    float cumulative = 0.0f;
    int last = 0;
    for (int i = n0 - 1; i >= 0; i--) {
        const int t = idx[0]; idx[0] = idx[i]; idx[i] = t;
        cumulative = __fadd_rn(cumulative, p[idx[i]]);
        if (cumulative > a.topp) { last = i; break; }
        sampler_sift_down(idx, 0, i - 1, p);
    }
    const float r = __fmul_rn(a.r01, cumulative);
    float cdf = 0.0f;
    int id = idx[last];
    for (int i = n0 - 1; i >= last; i--) {
        cdf = __fadd_rn(cdf, p[idx[i]]);
        if (r < cdf) { id = idx[i]; break; }
    }
    *a.out_id = id;
    if (a.info) { a.info[0] = n0; a.info[1] = n0 - last; }
}

// Every sampled row of a step in one launch: block j samples logits row row[j] (of rows stride floats apart) into
// out[8 * row[j]] (the id, then the four diagnostics), with that row's own triple and its own indices scratch (n ints per row).
#define SAMPLER_MAX_ROWS 8

struct SamplerRowsArgs {
    float *logits;
    int stride, n;
    int *indices; // [row][n]
    int *out;     // [row][8]
    int row[SAMPLER_MAX_ROWS];
    float temperature[SAMPLER_MAX_ROWS], topp[SAMPLER_MAX_ROWS], r01[SAMPLER_MAX_ROWS];
};

__global__ void __launch_bounds__(SAMPLER_THREADS, 1) k_sample_rows(SamplerRowsArgs a) {
    extern __shared__ __align__(16) unsigned char smp_sm[];
    const int j = blockIdx.x, r = a.row[j];
    SamplerArgs s;
    s.logits = a.logits + (size_t)r * a.stride;
    s.indices = a.indices + (size_t)r * a.n;
    // Opaque to the optimiser: otherwise it keeps the row offsets as separate 64-bit terms and adds them back on every p[idx[i]]
    // load of sample_row's single-thread top-p heap and CDF walk, which makes those latency-bound loops measurably slower.
    asm("mov.b64 %0, %0;" : "+l"(s.logits));
    asm("mov.b64 %0, %0;" : "+l"(s.indices));
    s.n = a.n;
    s.temperature = a.temperature[j]; s.topp = a.topp[j]; s.r01 = a.r01[j];
    s.out_id = a.out + 8 * r;
    s.info = a.out + 8 * r + 1;
    sample_row(s, smp_sm);
}

// ---- sampling controls (b200_set_sampling_controls): logit bias, repetition / frequency / presence penalties, top-k and min-p on
// the raw row of a sequence with controls, then the choice and the count of the emitted id, all in one launch with one block per
// row.  The raw row is only read: the modified row goes to dst (the sampler then turns it into probabilities there), so the logits
// output and k_token_logprobs still see the model's values.  Every operation is rounded once, in include/b200llama.h's order:
//   l = fl(l + bias);  where cnt > 0: l = l <= 0 ? fl(l * rep) : fl(l / rep), then l = fl(l - fl(fl(cnt * freq) + pres));
//   keep l >= v_k (the top_k-th largest value, ties at it all kept) and l >= fl(m + log(min_p)), the rest -inf;
//   temperature 0: the first strict maximum; otherwise sample_row on the modified row;  cnt[id] += 1.
// v_k comes from a radix select over order-preserving integer keys: four 8-bit digit passes, each a shared-memory histogram of
// the keys that share the digits found so far (warp-aggregated with __match_any_sync), no sort and no host work.
#define SAMPLER_CTL_MAX_BIAS 1024

struct SampleCtlRow {
    const float *src; // the raw logits row [n]
    float *dst;       // [sampler_padded(n)]: the modified row with a zero pad, then the sampler's probabilities
    float *row_out;   // nullable: a copy of the modified row before the choice (the test hook)
    int *cnt;         // the sequence's counts [n]; the emitted id's is incremented
    const int *bias_id;
    const float *bias_val;
    int n_bias, top_k;
    float min_p_log, rep, freq, pres; // min_p_log = (float)log((double)min_p): -inf for min_p 0
    float temperature, topp, r01;
    int *indices; // [n] the sampler's candidate list
    int *out;     // [5]: the id, then the sampler's four diagnostics (zeros at temperature 0)
};

struct SampleCtlArgs {
    int n;
    SampleCtlRow row[SAMPLER_MAX_ROWS];
};

__device__ __forceinline__ unsigned ctl_key(float v) { // ordered like the floats, -0 just below +0
    const unsigned u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ctl_unkey(unsigned k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

__global__ void __launch_bounds__(SAMPLER_THREADS, 1) k_sample_ctl(SampleCtlArgs args) {
    extern __shared__ __align__(16) unsigned char smp_sm[];
    __shared__ int hist[256];
    __shared__ float s_max[32];
    __shared__ int s_idx[32], s_digit, s_above;
    const int j = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n = args.n, npad = sampler_padded(n);
    const float *src = args.row[j].src;
    float *dst = args.row[j].dst, *row_out = args.row[j].row_out;
    int *cnt = args.row[j].cnt;
    const float rep = args.row[j].rep, freq = args.row[j].freq, pres = args.row[j].pres;

    // ---- 1. logit bias (the ids are distinct)
    for (int i = tid; i < npad; i += SAMPLER_THREADS) dst[i] = i < n ? src[i] : 0.0f;
    __syncthreads();
    for (int b = tid; b < args.row[j].n_bias; b += SAMPLER_THREADS) {
        const int i = args.row[j].bias_id[b];
        dst[i] = __fadd_rn(dst[i], args.row[j].bias_val[b]);
    }
    __syncthreads();
    // ---- 2. penalties, and the row maximum m
    float mx = -INFINITY;
    for (int i = tid; i < n; i += SAMPLER_THREADS) {
        float v = dst[i];
        const int c = cnt[i];
        if (c > 0) {
            v = v <= 0.0f ? __fmul_rn(v, rep) : __fdiv_rn(v, rep);
            v = __fsub_rn(v, __fadd_rn(__fmul_rn(__int2float_rn(c), freq), pres));
            dst[i] = v;
        }
        mx = fmaxf(mx, v);
    }
    mx = warp_max_f(mx);
    if (lane == 0) s_max[warp] = mx;
    __syncthreads();
    mx = s_max[0];
    for (int w = 1; w < SAMPLER_THREADS / 32; w++) mx = fmaxf(mx, s_max[w]);
    // ---- 3. v_k: the key with fewer than top_k keys above it and at least top_k at or above it
    float vk = -INFINITY;
    const int top_k = args.row[j].top_k;
    if (top_k > 0 && top_k < n) {
        unsigned prefix = 0, pmask = 0;
        int krem = top_k;
        for (int shift = 24; shift >= 0; shift -= 8) {
            if (tid < 256) hist[tid] = 0;
            __syncthreads();
            for (int i = tid; i < npad; i += SAMPLER_THREADS) { // npad is whole blocks: every lane runs every iteration
                const unsigned key = i < n ? ctl_key(dst[i]) : 0u;
                const bool in = i < n && (key & pmask) == prefix;
                const int bin = in ? (int)((key >> shift) & 255u) : 256;
                const unsigned peers = __match_any_sync(0xffffffffu, bin);
                if (in && lane == __ffs(peers) - 1) atomicAdd(&hist[bin], __popc(peers));
            }
            __syncthreads();
            if (warp == 0) { // lane l holds digits 255 - 8 l down to 248 - 8 l; the first lane whose running count reaches krem has v_k's
                int s = 0;
#pragma unroll
                for (int d = 0; d < 8; d++) s += hist[255 - 8 * lane - d];
                int incl = s;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const int u = __shfl_up_sync(0xffffffffu, incl, d);
                    if (lane >= d) incl += u;
                }
                const int hit = __ffs(__ballot_sync(0xffffffffu, incl >= krem)) - 1;
                if (lane == hit) {
                    int c = incl - s;
                    for (int d = 0; d < 8; d++) {
                        const int b = 255 - 8 * lane - d, h = hist[b];
                        if (c + h >= krem) { s_digit = b; s_above = c; break; }
                        c += h;
                    }
                }
            }
            __syncthreads();
            prefix |= (unsigned)s_digit << shift;
            pmask |= 255u << shift;
            krem -= s_above;
        }
        vk = ctl_unkey(prefix);
    }
    // ---- 4. masks (the maximum passes both), and the first index of the maximum
    const float thr = __fadd_rn(mx, args.row[j].min_p_log);
    int best = 0x7fffffff;
    for (int i = tid; i < n; i += SAMPLER_THREADS) {
        float v = dst[i];
        if (!(v >= vk && v >= thr)) { v = -INFINITY; dst[i] = v; }
        if (row_out) row_out[i] = v;
        if (v == mx && i < best) best = i;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, d));
    if (lane == 0) s_idx[warp] = best;
    __syncthreads();
    int *out = args.row[j].out;
    // ---- 5. the choice and the count
    if (args.row[j].temperature == 0.0f) {
        if (tid == 0) {
            for (int w = 1; w < SAMPLER_THREADS / 32; w++) best = min(best, s_idx[w]);
            best = min(best, s_idx[0]);
            out[0] = best;
            for (int k = 1; k < 5; k++) out[k] = 0;
            cnt[best] += 1;
        }
        return;
    }
    SamplerArgs s;
    s.logits = dst; s.n = n;
    s.temperature = args.row[j].temperature; s.topp = args.row[j].topp; s.r01 = args.row[j].r01;
    s.indices = args.row[j].indices; s.out_id = out; s.info = out + 1;
    sample_row(s, smp_sm);
    if (tid == 0) cnt[*out] += 1;
}
