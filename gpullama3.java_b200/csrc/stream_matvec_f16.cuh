// stream_matvec_f16.cuh -- FP16-weight matvec of the decode step on per-warp bulk-copy rings (FP16 plans, SURVEY 8(a) a4/a6/a9/a10,
// BASELINE configs 1 and 3).  Bit-exact with FP16FloatTensor.vectorDot (FP16FloatTensor.java:62-110) for an L-lane species, like
// k_matvec_f16 (decode_kernels.cuh) which stays as the fallback for odd shapes and the scalar (L = 0) order:
//   * per output row L independent chains  acc_c = fma(w[L j + c], x[L j + c], acc_c), j ascending   (FloatVector.fma: fused),
//   * reduceLanes(ADD) in ascending lane order starting from the identity,
//   * the FP16 -> FP32 widening flushes FP16 subnormals to (signed) zero, as the reference's vector conversion does.
// A row therefore offers only L-way parallelism of strictly sequential chains, and the arithmetic is one FMA per weight: the kernel is
// about keeping bytes in flight and instructions per weight low.
// Layout: the weights stay ROW-MAJOR exactly as in the GGUF file (no repack pass for FP16 plans).  Every warp owns a private ring of
// `stages` shared-memory stages and its own mbarriers: lane 0 issues one cp.async.bulk per row segment (seg columns of each of the
// warp's rows), the warp waits on the stage's mbarrier, consumes it from shared memory, __syncwarp()s and lane 0 refills the stage --
// no producer warp, no CTA-wide synchronisation after the activation has been staged.
// Lane mapping: a lane owns the chain PAIR (2u, 2u+1) of one row, so one 32-bit shared load delivers both weights as a half2 and one
// 64-bit load both activations; L/2 lanes cover a row and a warp works on 64/L rows at once (4 for the 16-lane species).  The subnormal
// flush is ONE packed instruction per pair: add.ftz.f16x2 w, -0 (x + -0 = x exactly for every other value; .ftz flushes subnormal
// inputs to sign-preserving zero) -- 3.5 instructions per weight instead of the 10 of the integer-arithmetic widening (v1 of the
// kernel was issue-bound).  The rows of a stage are SF_ROW_PAD bytes
// apart modulo 128 so the row groups of a warp hit different banks.
//   SF_GATEUP: half of the warp's row slots are ffn_gate rows, the other half the same rows of ffn_up; SwiGLU (InferenceCore.java:150-158)
//   is applied in the epilogue, so w1, w3 and the SwiGLU kernel of the round-1 FP16 graph collapse into one launch.
// PDL: the rings are filled before griddepcontrol.wait (weights are immutable); x, and out in SF_RESID, are touched only after it.
// Ragged rows (SF_STORE / SF_RESID; in practice a classifier whose vocabulary is not a multiple of the warp's row slots): the slots
// of the last group past the matrix re-read its last row, so no copy leaves the matrix (a tied classifier is the embedding table
// itself), and they are never stored nor offered to the argmax.
#pragma once
#include "stream_matvec.cuh"

#define SF_WARPS 8
#define SF_THREADS (SF_WARPS * 32)
#define SF_MAX_STAGES 8
#define SF_ROW_PAD 32

enum { SF_STORE = 0, SF_RESID = 1, SF_GATEUP = 2 };

struct SfArgs {
    const __half *w0, *w1; // [rows][cols] row-major; w1 = ffn_up (SF_GATEUP only)
    const float *x;        // activation, cols floats
    float *out;            // rows floats: r * oscale (SF_STORE), out + r * oscale (SF_RESID)
    float oscale;          // Granite's logitScale (classifier) / residualScale (Wo, W2), one rounding; 1.0f otherwise
    int rows, cols;        // of ONE matrix
    int seg, nseg;         // columns per stage, stages per row
    int stages;            // ring depth per warp
    float *part_val;       // SF_STORE on the classifier: per-CTA (max, first index) of the rows this CTA produced (FloatTensor.argmax, first
    int *part_idx;         // strict maximum), merged by k_argmax_advance instead of a pass over all logits; nullptr otherwise
    TraceBuf tr;
};

struct SfLayout {
    int seg, nseg, stages, ctas_per_sm;
    size_t total;
    bool ok;
};

// Host: pick the segment, the ring depth and the CTAs per SM that maximise the bytes in flight per SM.
static inline SfLayout sf_layout(int rows, int cols, int lanes, bool gateup) {
    SfLayout o{};
    o.ok = false;
    if (lanes != 8 && lanes != 16) return o;
    const int rw = 64 / lanes; // a lane owns two chains: L/2 lanes per row
    if (cols % 256 || cols < 256) return o;
    if (gateup && rows % (rw / 2)) return o; // other matrices may end in a partial row group
    const size_t fixed = (size_t)cols * 4 + SF_WARPS * SF_MAX_STAGES * 8 + 256;
    const size_t per_sm = 220 * 1024;
    size_t best = 0;
    for (int seg = 256; seg <= 512; seg += 256) { // bytes in flight per SM = occ * warps * (stages - 1) * stage bytes; ties -> more CTAs
        if (cols % seg) continue;
        const size_t stage = (size_t)rw * (seg * 2 + SF_ROW_PAD);
        for (int occ = 1; occ <= 3; occ++) {
            if (per_sm / occ <= fixed + 1024) continue;
            int s = (int)((per_sm / occ - 1024 - fixed) / (SF_WARPS * stage));
            if (s > SF_MAX_STAGES) s = SF_MAX_STAGES;
            if (s < 3) continue;
            const size_t score = (size_t)occ * (s - 1) * stage * (occ >= 2 ? 5 : 4); // a second CTA (8 more warps) is worth 25 % of the bytes
            if (score >= best) { best = score; o.stages = s; o.ctas_per_sm = occ; o.seg = seg; }
        }
    }
    if (!best) return o;
    o.nseg = cols / o.seg;
    o.total = fixed + (size_t)SF_WARPS * o.stages * ((size_t)rw * (o.seg * 2 + SF_ROW_PAD));
    o.ok = true;
    return o;
}

__device__ __forceinline__ unsigned f16x2_flush_subnormals(unsigned w) { // both halves: subnormal -> sign-preserving zero, anything else unchanged
    unsigned r;
    asm("add.ftz.f16x2 %0, %1, %2;" : "=r"(r) : "r"(w), "r"(0x80008000u));
    return r;
}

template <int L, int MODE>
__global__ void __launch_bounds__(SF_THREADS) k_stream_matvec_f16(SfArgs a) {
    constexpr int LPR = L / 2;         // lanes per row (a lane owns chains 2u and 2u+1)
    constexpr int RW = 32 / LPR;       // row slots per warp
    constexpr int MR = MODE == SF_GATEUP ? RW / 2 : RW; // matrix rows per warp step
    extern __shared__ __align__(128) unsigned char sf_smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float *sx = reinterpret_cast<float *>(sf_smem);
    const size_t off_bar = ((size_t)a.cols * 4 + 127) & ~(size_t)127;
    const unsigned row_b = (unsigned)(a.seg * 2 + SF_ROW_PAD), stage_b = RW * row_b;
    const unsigned bar0 = smem_u32(sf_smem + off_bar) + (unsigned)warp * SF_MAX_STAGES * 8;
    unsigned char *ring = sf_smem + off_bar + SF_WARPS * SF_MAX_STAGES * 8 + (size_t)warp * a.stages * stage_b;
    const unsigned ring_u = smem_u32(ring);
    const int S = a.stages, nseg = a.nseg, seg = a.seg;

    // warp-interleaved assignment: group g belongs to global warp (g mod G); consecutive groups go to different SMs
    const int G = gridDim.x * SF_WARPS, gw = warp * gridDim.x + blockIdx.x;
    const int ngroups = (a.rows + MR - 1) / MR;
    const int my_groups = gw < ngroups ? (ngroups - gw + G - 1) / G : 0;
    const int n_items = my_groups * nseg;
    const size_t row_bytes = (size_t)a.cols * 2;
    const unsigned long long pol = l2_policy_evict_first();

    auto issue = [&](int k) { // lane 0 only
        const int st = k % S, gi = k / nseg, s = k - gi * nseg;
        const size_t row0 = (size_t)(gw + gi * G) * MR;
        const unsigned bar = bar0 + 8u * st;
        mbar_expect_tx(bar, RW * (unsigned)seg * 2u);
#pragma unroll
        for (int r = 0; r < RW; r++) {
            const __half *m = (MODE == SF_GATEUP && r >= MR) ? a.w1 : a.w0;
            const size_t rr = row0 + (MODE == SF_GATEUP ? r % MR : r), row = rr < (size_t)a.rows ? rr : (size_t)a.rows - 1;
            bulk_g2s_evict_first(ring_u + st * stage_b + r * row_b, reinterpret_cast<const unsigned char *>(m) + row * row_bytes + (size_t)s * seg * 2,
                                 (unsigned)seg * 2u, bar, pol);
        }
    };

    if (lane == 0) {
        for (int s = 0; s < S; s++) mbar_init(bar0 + 8u * s, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    trace_entry(a.tr);
    pdl_launch_dependents();
    if (lane == 0)
        for (int k = 0; k < S && k < n_items; k++) issue(k);
    pdl_wait(); // the activation (and out, SF_RESID) come from the previous kernel
    for (int i = tid * 4; i < a.cols; i += SF_THREADS * 4) *reinterpret_cast<float4 *>(sx + i) = *reinterpret_cast<const float4 *>(a.x + i);
    __syncthreads();
    trace_mark(a.tr, 2);

    const int r = lane / LPR, u = lane % LPR;
    float acc0 = 0.0f, acc1 = 0.0f; // chains 2u and 2u+1 of row slot r
    float best = -INFINITY;          // (a lane's rows ascend, so a strict comparison keeps the first maximum)
    int best_i = 0x7fffffff;
    for (int k = 0; k < n_items; k++) {
        const int st = k % S, gi = k / nseg, s = k - gi * nseg;
        mbar_wait(bar0 + 8u * st, (unsigned)(k / S) & 1u);
        const unsigned *wr = reinterpret_cast<const unsigned *>(ring + st * stage_b + r * row_b) + u; // half2 (L j + 2u, L j + 2u + 1)
        const float2 *xs = reinterpret_cast<const float2 *>(sx + s * seg) + u;
#pragma unroll 8
        for (int j = 0; j < seg / L; j++) {
            const unsigned w2 = f16x2_flush_subnormals(wr[j * LPR]);
            const float2 xv = xs[j * LPR];
            const __half2 h2 = *reinterpret_cast<const __half2 *>(&w2);
            acc0 = fmaf(__low2float(h2), xv.x, acc0);
            acc1 = fmaf(__high2float(h2), xv.y, acc1);
        }
        __syncwarp(); // every lane has consumed the stage: lane 0 may overwrite it
        if (lane == 0 && k + S < n_items) issue(k + S);
        if (s == nseg - 1) {
            float result = 0.0f; // reduceLanes(ADD): ascending lanes from the identity
#pragma unroll
            for (int q = 0; q < LPR; q++) {
                result = __fadd_rn(result, __shfl_sync(0xffffffffu, acc0, r * LPR + q));
                result = __fadd_rn(result, __shfl_sync(0xffffffffu, acc1, r * LPR + q));
            }
            const size_t row = (size_t)(gw + gi * G) * MR + (MODE == SF_GATEUP ? r % MR : r);
            if (MODE == SF_GATEUP) {
                const float up = __shfl_sync(0xffffffffu, result, ((r + MR) % RW) * LPR);
                if (r < MR && u == 0) a.out[row] = swiglu(result, up);
            } else if (u == 0 && row < (size_t)a.rows) {
                result = __fmul_rn(result, a.oscale);
                a.out[row] = MODE == SF_RESID ? __fadd_rn(a.out[row], result) : result; // x[i] = x[i] + xb2[i] (InferenceCore.java:143,164)
                if (MODE == SF_STORE && result > best) { best = result; best_i = (int)row; }
            }
            acc0 = acc1 = 0.0f;
        }
    }
    if (MODE == SF_STORE && a.part_val) { // uniform over the grid
        __shared__ float pv[SF_WARPS];
        __shared__ int pi[SF_WARPS];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
            argmax_merge(best, best_i, ov, oi);
        }
        if (lane == 0) { pv[warp] = best; pi[warp] = best_i; }
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < SF_WARPS; w++) argmax_merge(best, best_i, pv[w], pi[w]);
            a.part_val[blockIdx.x] = best;
            a.part_idx[blockIdx.x] = best_i;
        }
    }
    trace_mark(a.tr, 3);
}
