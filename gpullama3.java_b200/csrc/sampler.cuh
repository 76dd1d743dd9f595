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

__global__ void __launch_bounds__(SAMPLER_THREADS, 1) k_sample(SamplerArgs a) {
    extern __shared__ __align__(16) unsigned char smp_sm[];
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
