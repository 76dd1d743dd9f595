// logprobs.cuh -- per emitted token: its log-probability and the top-N alternatives (b200_set_logprobs; include/b200llama.h states
// the definition).  For a row l[0, vocab) and the id c the call emits:
//   m, S      = score_row's (score.cuh), the same code as b200_score_tokens' k_score_rows, so chosen has its bits
//   chosen    = ((double)l_c - (double)m) - log(S)
//   t_1..t_N  = repeated first-strict-maximum selection among the entries not yet taken; once no remaining entry is > -inf (NaN
//               never is), the lowest index not yet taken.  t_1 is the greedy id.
//   lp_k      = ((double)l_{t_k} - (double)m) - log(S)
//
// The selection is a sort by one 64-bit key per entry, descending: the high word orders the value (0 for -inf and NaN, -0 read as
// +0 so that equal values tie), the low word is ~index (the lower index first).  Keys are distinct, so the top N keys are the
// definition's t_1..t_N.  k_token_logprobs finds them without a per-entry sort:
//   1. each thread's largest key over its strided slice; T = the N-th largest of these SCORE_THREADS keys.  They are N distinct
//      entries with key >= T, so every one of the row's top N keys is >= T;
//   2. the keys >= T go to a shared candidate list (only the N slices whose maximum is >= T can contribute, each at most
//      ceil(vocab / SCORE_THREADS) entries; a few dozen entries on real logits), and each candidate's rank among them is its place;
//   3. a list that overflows LOGPROB_CAND falls back to N rounds of "the largest key below the previous one" over the whole row.
//      Overflow takes more than LOGPROB_CAND / ceil(vocab / SCORE_THREADS) slices lying largely above T -- at least three slices
//      at vocab 128256, two at 151936; one slice never does.  Both give the same result; only the time differs.
#pragma once
#include "score.cuh"

constexpr int LOGPROB_MAX_TOP = 20;   // B200_MAX_TOP_LOGPROBS
constexpr int LOGPROB_MAX_ROWS = 8;   // rows per launch: every emitting row of a batched step
constexpr int LOGPROB_CAND = 1024;    // candidate keys held in shared memory

struct LogprobRow {
    double chosen;
    double lp[LOGPROB_MAX_TOP];
    int id[LOGPROB_MAX_TOP];
};

// Block b reads logits row b (stride floats apart), its emitted id at *ids[b], and writes out[out_row[b]].
struct LogprobArgs {
    const float *logits;
    long long stride;
    int vocab, n_top;
    const int *ids[LOGPROB_MAX_ROWS];
    int out_row[LOGPROB_MAX_ROWS];
    LogprobRow *out;
};

__device__ __forceinline__ unsigned long long logprob_key(float v, int j) {
    unsigned hi = 0;
    if (v > -INFINITY) {
        const unsigned b = v == 0.0f ? 0u : __float_as_uint(v);
        hi = (b & 0x80000000u) ? ~b : (b | 0x80000000u); // > 0 for every value above -inf
    }
    return ((unsigned long long)hi << 32) | (unsigned)~j;
}

__global__ void __launch_bounds__(SCORE_THREADS) k_token_logprobs(LogprobArgs a) {
    __shared__ float sv[SCORE_THREADS / 32];
    __shared__ int si[SCORE_THREADS / 32];
    __shared__ double ss[SCORE_THREADS / 32];
    __shared__ float s_m;
    __shared__ int s_i;
    __shared__ double s_ls;
    __shared__ unsigned long long cand[LOGPROB_CAND];
    __shared__ unsigned long long s_t;
    __shared__ int s_n;
    const int b = blockIdx.x, tid = threadIdx.x, vocab = a.vocab, n_top = a.n_top;
    const int *id = nullptr;
    int row = 0;
#pragma unroll
    for (int k = 0; k < LOGPROB_MAX_ROWS; k++) // constant indices: the parameter arrays stay in the constant bank
        if (k == b) { id = a.ids[k]; row = a.out_row[k]; }
    LogprobRow &o = a.out[row];
    score_row(a.logits, a.stride, vocab, sv, si, ss, s_m, s_i, [&](const float *l, double S, double m) {
        const double ls = log(S);
        s_ls = ls;
        o.chosen = __dsub_rn(__dsub_rn((double)l[*id], m), ls);
    });
    if (n_top == 0) return;
    const float *l = a.logits + (size_t)b * a.stride;
    __syncthreads();
    const double m = (double)s_m, ls = s_ls;
    auto put = [&](int r, unsigned long long k) {
        const int j = (int)~(unsigned)k;
        o.id[r] = j;
        o.lp[r] = __dsub_rn(__dsub_rn((double)l[j], m), ls);
    };

    // 1. the threshold
    unsigned long long mine = 0; // an empty slice: below every entry's key
    for (int j = tid; j < vocab; j += SCORE_THREADS) {
        const unsigned long long k = logprob_key(l[j], j);
        if (k > mine) mine = k;
    }
    cand[tid] = mine;
    if (tid == 0) { s_t = ~0ull; s_n = 0; }
    __syncthreads();
    int above = 0;
    for (int t = 0; t < SCORE_THREADS; t++) above += cand[t] > mine;
    if (above < n_top) atomicMin(&s_t, mine);
    __syncthreads();
    const unsigned long long T = s_t;
    __syncthreads();

    // 2. the candidates and their ranks
    for (int j = tid; j < vocab; j += SCORE_THREADS) {
        const unsigned long long k = logprob_key(l[j], j);
        if (k >= T) {
            const int q = atomicAdd(&s_n, 1);
            if (q < LOGPROB_CAND) cand[q] = k;
        }
    }
    __syncthreads();
    const int nc = s_n;
    if (nc <= LOGPROB_CAND) {
        for (int q = tid; q < nc; q += SCORE_THREADS) {
            const unsigned long long k = cand[q];
            int r = 0;
            for (int t = 0; t < nc; t++) r += cand[t] > k;
            if (r < n_top) put(r, k);
        }
        return;
    }

    // 3. the fallback: n_top block-wide maxima, each below the previous one
    const int lane = tid & 31, warp = tid >> 5;
    unsigned long long prev = ~0ull;
    for (int r = 0; r < n_top; r++) {
        unsigned long long best = 0;
        for (int j = tid; j < vocab; j += SCORE_THREADS) {
            const unsigned long long k = logprob_key(l[j], j);
            if (k < prev && k > best) best = k;
        }
#pragma unroll
        for (int o2 = 16; o2 > 0; o2 >>= 1) {
            const unsigned long long v = __shfl_xor_sync(0xffffffffu, best, o2);
            if (v > best) best = v;
        }
        __syncthreads(); // the previous round's reads of cand
        if (lane == 0) cand[warp] = best;
        __syncthreads();
        best = cand[0];
        for (int w = 1; w < SCORE_THREADS / 32; w++)
            if (cand[w] > best) best = cand[w];
        if (tid == 0) put(r, best);
        prev = best;
    }
}
