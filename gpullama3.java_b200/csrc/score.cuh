// score.cuh -- per-row scores of b200_score_tokens: greedy id, and the log-probability of a target token under the row's logits.
//
// For a row l[0, vocab) with target t (include/b200llama.h states the definition):
//   m, greedy = the first index of the strict maximum (FloatTensor.argmax, k_argmax_advance's tie rule)
//   S         = sum_j exp((double)l_j - (double)m), in double
//   logprob   = ((double)l_t - (double)m) - log(S);  NaN for t == -1
//
// k_score_rows: one CTA per row.  Thread i reduces the fixed strided slice i, i + SCORE_THREADS, ... in index order (the max and
// its first index in float, then the sum in double), and a fixed-shape tree (warp shuffles, then warp 0 over the warps' values)
// combines the slices.  The order depends only on vocab, so every path of b200_score_tokens -- the tensor-core classifier's
// scratch rows, the batched step's rows and the single-token graph's row -- gives the same bits for the same logits.  Rows are
// read with an arbitrary stride (the batched step pads to sampler_padded(vocab), the GEMM scratch to whole 64-column tiles).
#pragma once
#include "decode_kernels.cuh"

constexpr int SCORE_THREADS = 256;
// tensor_core_exact: rows of classifier logits per GEMM into the scratch (256 rows x 128256 columns = 131 MB); a longer chunk
// re-reads the classifier once per group
constexpr int SCORE_GROUP_ROWS = 256;

struct ScoreOut {
    double logprob;
    int greedy, pad;
};

// Row blockIdx.x's maximum m and the first index of it (s_m, s_i) and S = sum_j exp((double)l_j - m), by a SCORE_THREADS-thread
// block over its shared scratch sv / si / ss; thread 0 then runs tail(row, S, m).  k_score_rows and k_token_logprobs (logprobs.cuh)
// both call it, so their m and S are the same code and the same bits.
template <typename Tail>
__device__ __forceinline__ void score_row(const float *logits, long long stride, int vocab, float (&sv)[SCORE_THREADS / 32], int (&si)[SCORE_THREADS / 32],
                                          double (&ss)[SCORE_THREADS / 32], float &s_m, int &s_i, Tail &&tail) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float *l = logits + (size_t)blockIdx.x * stride;
    int best_i = 0x7fffffff;
    float best = -INFINITY;
    for (int j = tid; j < vocab; j += SCORE_THREADS) {
        const float v = l[j];
        if (v > best) { best = v; best_i = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) argmax_merge(best, best_i, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, best_i, o));
    if (lane == 0) { sv[warp] = best; si[warp] = best_i; }
    __syncthreads();
    if (warp == 0) {
        best = lane < SCORE_THREADS / 32 ? sv[lane] : -INFINITY;
        best_i = lane < SCORE_THREADS / 32 ? si[lane] : 0x7fffffff;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) argmax_merge(best, best_i, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, best_i, o));
        if (lane == 0) { s_m = best; s_i = best_i == 0x7fffffff ? 0 : best_i; } // every logit -inf: index 0, as k_argmax_advance
    }
    __syncthreads();
    const double m = (double)s_m;
    double sum = 0.0;
#pragma unroll 1 // the adds form one chain anyway; unrolled, ptxas spills a register pair around the inlined exp()
    for (int j = tid; j < vocab; j += SCORE_THREADS) sum = __dadd_rn(sum, exp(__dsub_rn((double)l[j], m)));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum = __dadd_rn(sum, __shfl_xor_sync(0xffffffffu, sum, o));
    if (lane == 0) ss[warp] = sum;
    __syncthreads();
    if (tid == 0) {
        double S = 0.0;
#pragma unroll
        for (int w = 0; w < SCORE_THREADS / 32; w++) S = __dadd_rn(S, ss[w]);
        tail(l, S, m);
    }
}

__global__ void __launch_bounds__(SCORE_THREADS) k_score_rows(const float *__restrict__ logits, long long stride, int vocab,
                                                              const int *__restrict__ targets, ScoreOut *__restrict__ out) {
    __shared__ float sv[SCORE_THREADS / 32];
    __shared__ int si[SCORE_THREADS / 32];
    __shared__ double ss[SCORE_THREADS / 32];
    __shared__ float s_m;
    __shared__ int s_i;
    score_row(logits, stride, vocab, sv, si, ss, s_m, s_i, [&](const float *l, double S, double m) {
        const int t = targets[blockIdx.x];
        out[blockIdx.x].logprob = t < 0 ? __longlong_as_double(0x7ff8000000000000ll) : __dsub_rn(__dsub_rn((double)l[t], m), log(S));
        out[blockIdx.x].greedy = s_i;
    });
}
