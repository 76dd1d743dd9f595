// prefill_gemm.cuh -- the batched-prefill building block: C[M,N] (fp32) = A[M,K] (fp16) * B[N,K]^T (fp16)
// on the Hopper tensor cores (sm_90a): TMA (cp.async.bulk.tensor, SWIZZLE_128B) -> shared-memory ring
// guarded by mbarriers -> wgmma.mma_async (m64n128k16, f16 x f16 -> f32, both operands read from shared
// memory, accumulator in registers) -> epilogue.  Replaces the reference's mma.sync m16n8k16 GEMMs gemmMMA /
// gemmMMAQKV / gemmMMAGateUp (TransformerBatchPrefillKernels.java:792-915, 971, 1132), which stage BK=16
// through a single shared-memory buffer.  A = activations rounded to FP16 (batchedRmsApplyFP16, :61), B = the
// FP16 weight matrix exactly as stored in GGUF ([N][K], K contiguous = "K-major" for both operands).
//
// Warp groups (384 threads): warp group 0 = TMA producer (one elected thread), warp groups 1 and 2 = consumers;
// consumer c issues the wgmmas for rows 64*c .. 64*c+63 of the 128 x 128 tile and runs their epilogue.
//
// W8A16 (BSRC = B_Q8): B comes straight from the decode kernels' tile-major Q8_0 stream (stream_matvec.cuh), as the
// reference's gemmMMAQ8 family does with packQ8Halves (TransformerBatchPrefillKernels.java:1544-1580).  Per k-block the
// producer thread loads 128 rows x (64 int8 quants + the 16-byte line holding their two f16 scales) into a raw ring next
// to the operand ring; warps 1-3 of the producer warp group turn it into the f16 B tile f16(q * d) in exactly the
// SWIZZLE_128B layout TMA gives the f16 path, then arrive on the stage's full barrier.  The wgmma loop and the
// epilogues are the same code for both sources.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace pg {

constexpr int BM = 128, BK = 64, BN = 128;
constexpr int GEMM_THREADS = 384;
// Epilogue modes: F32 store (QKV), F32 reduce-add (x += A*W^T: Wo and W2, split-K partials add up), and the gate/up
// pair: the B tile is 64 rows of W1 and 64 rows of W3 for the same 64 hidden units, so accumulator columns
// [0,64) = gate, [64,128) = up, and the epilogue emits f16(silu(gate)*up) (InferenceCore.java:150-158).
enum { GEMM_F32 = 0, GEMM_RESID = 1, GEMM_GATEUP = 2 };
// B operand sources: an f16 [N][K] matrix through TMA, or the tile-major Q8_0 stream dequantised in shared memory
enum { B_F16 = 0, B_Q8 = 1 };
// W8A16 raw stage: 128 rows x 64 quants, then 128 rows x the 16-byte scale line holding the k-block's two scales
constexpr int Q8_QUANT_BYTES = BN * BK, Q8_SCALE_BYTES = BN * 16, Q8_RAW_BYTES = Q8_QUANT_BYTES + Q8_SCALE_BYTES;
constexpr int Q8_CONVERTERS = 96; // warps 1-3 of the producer warp group

__device__ __forceinline__ uint32_t s32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t cnt) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(cnt)); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "PG_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra PG_DONE;\n"
        "bra PG_WAIT;\n"
        "PG_DONE:\n"
        "}\n" ::"r"(bar), "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *map, int c0, int c1, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
                 "l"(map), "r"(c0), "r"(c1), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap *map, int c0, int c1, int c2, int c3, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];" ::"r"(dst),
                 "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(bar)
                 : "memory");
}

// 8 int8 quants (two words, lowest byte = lowest column) -> 8 f16 values f16(q * d), as one 16-byte chunk.  q ^ 0x80 is
// q + 128 as an unsigned byte; under the exponent byte 0x64 it reads as the f16 1024 + (q + 128), and subtracting 1152
// leaves q exactly.  The f16 product q * d is rounded once, so the value is __float2half_rn((float)q * (float)d): the
// f32 product of an 8-bit and an 11-bit significand is exact.
__device__ __forceinline__ uint4 q8_chunk_to_f16(uint2 q, __half2 d) {
    const __half2 bias = __half2half2(__ushort_as_half((unsigned short)0x6480)); // 1152
    const uint32_t u0 = q.x ^ 0x80808080u, u1 = q.y ^ 0x80808080u;
    uint32_t w[4] = {__byte_perm(u0, 0x64646464u, 0x4140), __byte_perm(u0, 0x64646464u, 0x4342), __byte_perm(u1, 0x64646464u, 0x4140),
                     __byte_perm(u1, 0x64646464u, 0x4342)};
    uint4 o;
    uint32_t *po = reinterpret_cast<uint32_t *>(&o);
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const __half2 v = __hmul2_rn(__hsub2(*reinterpret_cast<const __half2 *>(&w[i]), bias), d);
        po[i] = *reinterpret_cast<const uint32_t *>(&v);
    }
    return o;
}
// wgmma shared-memory matrix descriptor, K-major operand, 128-byte swizzle: start address >> 4 (bits 0-13) | LBO (unused for
// swizzled K-major, 1) << 16 | SBO = 8 rows * 128 B >> 4 << 32 | layout SWIZZLE_128B (1) << 62.  The tile base is 1024-byte aligned.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}

// d[64 rows x 128 cols] (+)= A[64 x 16] * B[128 x 16]^T.  Thread t of the warp group holds, for j = 0..15, columns
// 8j + 2(t%4) + {0,1} of row 16(t/32) + (t%32)/4 in d[4j], d[4j+1] and of that row + 8 in d[4j+2], d[4j+3].
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t da, uint64_t db, int accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
        "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
        "%64, %65, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
          "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
          "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]),
          "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]),
          "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]),
          "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(accumulate)
        : "memory");
}

// W8A16 raw ring depth: as deep as the 227 KB budget allows next to the operand ring (at most 8), so the weight bytes are
// requested from HBM well before the converters need them
template <int STAGES> __host__ __device__ constexpr int q8_raw_stages() {
    return (227 * 1024 - STAGES * (BM * BK * 2 + BN * BK * 2) - 2048) / Q8_RAW_BYTES < 8 ? (227 * 1024 - STAGES * (BM * BK * 2 + BN * BK * 2) - 2048) / Q8_RAW_BYTES : 8;
}
template <int STAGES, int BSRC = B_F16> constexpr size_t smem_bytes() {
    return (size_t)STAGES * (BM * BK * 2 + BN * BK * 2) + (BSRC == B_Q8 ? (size_t)q8_raw_stages<STAGES>() * (Q8_RAW_BYTES + 8) : 0) + 2 * STAGES * 8 + 1024;
}

// grid = (M tiles, N tiles, K splits): the CTAs that share a weight (B) tile are adjacent in launch order, so the
// tile comes from HBM once and from L2 for the others; A (activations, a few MB) lives in L2.
// C: row stride ldc (elements); rows >= m_valid are not stored (GEMM_F32 / GEMM_RESID write zeros / add zeros there,
// inside the padded buffer).  GEMM_GATEUP: N tiles index 64 hidden units.  Split z owns k-blocks [z * kb_per_split, +kb_per_split).
// BSRC = B_Q8: tma_b / tma_b2 are the quant / scale maps of the Q8_0 stream (make_map_q8), seg its segment width.
template <int MODE, int STAGES, int BSRC = B_F16>
__global__ void __launch_bounds__(GEMM_THREADS, 1) k_gemm_f16_wgmma(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                                                                 const __grid_constant__ CUtensorMap tma_b2, const __grid_constant__ CUtensorMap tma_c,
                                                                 void *__restrict__ Cv, int ldc, int m_valid, int K, int kb_per_split, int seg,
                                                                 float oscale) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023); // SWIZZLE_128B tiles need 1024-byte alignment
    constexpr int A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2, RAW_BYTES = BSRC == B_Q8 ? Q8_RAW_BYTES : 0;
    constexpr int RSTAGES = BSRC == B_Q8 ? q8_raw_stages<STAGES>() : 0;
    static_assert(STAGES * (A_BYTES + B_BYTES) >= BM * BN * 4, "the C tile is staged in the operand ring");
    uint8_t *sA = smem, *sB = smem + STAGES * A_BYTES, *sR = sB + STAGES * B_BYTES;
    uint64_t *bars = reinterpret_cast<uint64_t *>(sR + RSTAGES * RAW_BYTES);
    // raw: a W8A16 raw stage has landed.  The converters own the raw ring: they refill a stage once all of them have
    // converted it, so its loads run up to RSTAGES k-blocks ahead, independent of the operand ring.
    const uint32_t full0 = s32(bars), empty0 = s32(bars + STAGES), raw0 = s32(bars + 2 * STAGES);
    const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        // empty: one arrival per consumer warp once its wgmmas have read the stage.  full (W8A16): the A load's expect_tx
        // and one arrival for the converted B tile.
        for (int s = 0; s < STAGES; s++) { mbar_init(full0 + 8 * s, BSRC == B_Q8 ? 2 : 1); mbar_init(empty0 + 8 * s, 8); }
        for (int s = 0; s < RSTAGES; s++) mbar_init(raw0 + 8 * s, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int nk_all = (K + BK - 1) / BK, kb0 = blockIdx.z * kb_per_split;
    const int nk = nk_all - kb0 < kb_per_split ? nk_all - kb0 : kb_per_split;
    const int m0 = blockIdx.x * BM;
    const int n0 = blockIdx.y * (MODE == GEMM_GATEUP ? BN / 2 : BN);

    if (wg == 0) {
        // ===== TMA producer =====
        if (warp == 0 && lane == 0) {
            for (int kb = 0; kb < nk; kb++) {
                const int st = kb % STAGES;
                mbar_wait(empty0 + 8 * st, ((kb / STAGES) & 1) ^ 1);
                const int kc = (kb0 + kb) * BK;
                if (BSRC == B_Q8) { // B arrives through the converters
                    mbar_expect_tx(full0 + 8 * st, A_BYTES);
                    tma_load_2d(s32(sA + st * A_BYTES), &tma_a, kc, m0, full0 + 8 * st);
                    continue;
                }
                mbar_expect_tx(full0 + 8 * st, A_BYTES + B_BYTES);
                tma_load_2d(s32(sA + st * A_BYTES), &tma_a, kc, m0, full0 + 8 * st);
                if (MODE == GEMM_GATEUP) {
                    tma_load_2d(s32(sB + st * B_BYTES), &tma_b, kc, n0, full0 + 8 * st);
                    tma_load_2d(s32(sB + st * B_BYTES + B_BYTES / 2), &tma_b2, kc, n0, full0 + 8 * st);
                } else {
                    tma_load_2d(s32(sB + st * B_BYTES), &tma_b, kc, n0, full0 + 8 * st);
                }
            }
        } else if constexpr (BSRC == B_Q8) {
            // ===== W8A16 converters: raw stage -> f16 B tile.  Stream row n of the tile -> B row n (gate/up: slots 0, 1 of
            // group n / 4 are gate rows, 2, 3 up rows -> rows 2(n/4) + (n&1), +64 for up).  Work item i = (row i / 8,
            // 8-column chunk i % 8): a warp reads 256 consecutive quant bytes and writes four whole 128-byte rows. =====
            if (warp == 0) return;
            const int ct = threadIdx.x - 32;
            const int g0 = (MODE == GEMM_GATEUP ? 2 * n0 : n0) / 4; // stream rows 4 g0 .. 4 g0 + 127 (gate/up: the 64 hidden units from n0 on)
            // k-block kb -> raw stage kb % RSTAGES: the quants of segment s, columns j .. j+63, and the 16-byte aligned line of
            // 8 scales (256 columns) holding their two (a box starting at an unaligned byte faults; the line never passes
            // the unit's 16-byte padded end)
            auto load_raw = [&](int kb) {
                const int kc = (kb0 + kb) * BK, s = kc / seg, j = kc - s * seg, rs = kb % RSTAGES;
                mbar_expect_tx(raw0 + 8 * rs, RAW_BYTES);
                tma_load_4d(s32(sR + rs * RAW_BYTES), &tma_b, j, 0, s, g0, raw0 + 8 * rs);
                tma_load_4d(s32(sR + rs * RAW_BYTES + Q8_QUANT_BYTES), &tma_b2, seg + ((j >> 8) << 4), 0, s, g0, raw0 + 8 * rs);
            };
            if (ct == 0)
                for (int kb = 0; kb < RSTAGES && kb < nk; kb++) load_raw(kb);
            for (int kb = 0; kb < nk; kb++) {
                const int st = kb % STAGES, rs = kb % RSTAGES;
                mbar_wait(raw0 + 8 * rs, (kb / RSTAGES) & 1);
                mbar_wait(empty0 + 8 * st, ((kb / STAGES) & 1) ^ 1); // the consumers have read the B tile this stage held
                const int j = (kb0 + kb) * BK % seg;                 // column of the k-block in its segment
                const uint8_t *rq = sR + rs * RAW_BYTES, *rsc = rq + Q8_QUANT_BYTES + ((j & 255) >> 4); // its first scale in the line
                uint8_t *dst = sB + st * B_BYTES;
#pragma unroll 4
                for (int i = ct; i < BN * 8; i += Q8_CONVERTERS) {
                    const int n = i >> 3, ch = i & 7;
                    const int row = MODE == GEMM_GATEUP ? ((n & 2) << 5) + ((n >> 2) << 1) + (n & 1) : n;
                    const uint2 q = *reinterpret_cast<const uint2 *>(rq + 64 * n + 8 * ch);
                    const __half d = *reinterpret_cast<const __half *>(rsc + 16 * n + 2 * (ch >> 2));
                    *reinterpret_cast<uint4 *>(dst + 128 * row + ((ch ^ (row & 7)) << 4)) = q8_chunk_to_f16(q, __half2half2(d));
                }
                // the generic-proxy stores (and raw reads) are ordered before wgmma's reads (and the raw stage's refill), then
                // one thread signals the tile and refills the raw stage every converter is done with
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                asm volatile("bar.sync 2, %0;" ::"n"(Q8_CONVERTERS) : "memory");
                if (ct == 0) {
                    mbar_arrive(full0 + 8 * st);
                    if (kb + RSTAGES < nk) load_raw(kb + RSTAGES);
                }
            }
        }
        return; // the producer warp group takes no part in the epilogue (named barrier 1 counts the 256 consumer threads)
    }

    // ===== consumers: warp group c = wg - 1 owns tile rows 64c .. 64c+63 =====
    const int c = wg - 1, t = threadIdx.x & 127;
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; i++) acc[i] = 0.0f;
    int prev = -1;
    for (int kb = 0; kb < nk; kb++) {
        const int st = kb % STAGES;
        mbar_wait(full0 + 8 * st, (kb / STAGES) & 1);
        asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
        const uint64_t da = wgmma_desc_sw128(s32(sA + st * A_BYTES + c * (64 * 128))), db = wgmma_desc_sw128(s32(sB + st * B_BYTES));
#pragma unroll
        for (int k = 0; k < BK / 16; k++) // K step of 16 fp16 = 32 bytes = +2 in the (addr >> 4) field, inside the 128-byte swizzle atom
            wgmma_m64n128k16(acc, da + 2 * k, db + 2 * k, (kb | k) != 0);
        asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
        asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); // the previous stage's wgmmas are done: hand it back
        if (prev >= 0 && lane == 0) mbar_arrive(empty0 + 8 * prev);
        prev = st;
    }
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");

    const int r_lo = c * 64 + (t >> 5) * 16 + ((t & 31) >> 2); // tile row of acc[4j], acc[4j+1]; acc[4j+2], acc[4j+3] are row r_lo + 8
    const int cq = 2 * (t & 3);                                 // column offset inside each 8-column group
    if (MODE == GEMM_GATEUP) {
        __half *C = reinterpret_cast<__half *>(Cv);
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int row = m0 + r_lo + 8 * h;
            if (row < m_valid) {
                __half2 *dst = reinterpret_cast<__half2 *>(C + (size_t)row * ldc + n0 + cq);
#pragma unroll
                for (int j = 0; j < 8; j++) { // gate column 8j + cq (+1) sits in acc[4j + 2h (+1)], its up partner 64 columns on in acc[32 + ...]
                    const float g0 = acc[4 * j + 2 * h], g1 = acc[4 * j + 2 * h + 1];
                    const float h0 = (g0 / (1.0f + expf(-g0))) * acc[32 + 4 * j + 2 * h];
                    const float h1 = (g1 / (1.0f + expf(-g1))) * acc[32 + 4 * j + 2 * h + 1];
                    dst[4 * j] = __floats2half2_rn(h0, h1);
                }
            }
        }
    } else {
        // FP32 tile -> shared memory (the ring is idle once BOTH consumer warp groups have finished their wgmmas: every
        // TMA load has landed and been read) in the SWIZZLE_128B layout of the C tensor map: four 128 x 32 boxes, row r of
        // box b at b * 16 KB + 128 r, 16-byte chunk q at (q ^ (r & 7)) << 4.  Then ONE thread hands the boxes to TMA: a plain
        // tensor store (QKV) or an f32 reduce-add performed by the memory system (x += A W^T for Wo / W2 -- no
        // read-modify-write through the SM, and split-K partials add up).  Rows past m_valid store / add 0.  GEMM_RESID scales
        // the tile by oscale first (Granite's residualScale: under split-K each partial is scaled, within the FP16 tolerance).
        asm volatile("bar.sync 1, 256;" ::: "memory");
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int rloc = r_lo + 8 * h;
            const bool live = m0 + rloc < m_valid;
#pragma unroll
            for (int j = 0; j < 16; j++) {
                const int col = 8 * j + cq, b = col >> 5, q = (col & 31) >> 2;
                float2 o = live ? make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]) : make_float2(0.0f, 0.0f);
                if (MODE == GEMM_RESID) o = make_float2(__fmul_rn(o.x, oscale), __fmul_rn(o.y, oscale));
                *reinterpret_cast<float2 *>(smem + b * (BM * 32 * 4) + rloc * 128 + ((q ^ (rloc & 7)) << 4) + (col & 3) * 4) = o;
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (t == 0 && c == 0) {
#pragma unroll
            for (int b = 0; b < BN / 32; b++) {
                const uint32_t src = s32(smem + b * (BM * 32 * 4));
                if (MODE == GEMM_RESID)
                    asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.bulk_group [%0, {%2, %3}], [%1];" ::"l"(&tma_c), "r"(src),
                                 "r"(n0 + b * 32), "r"(m0)
                                 : "memory");
                else
                    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(&tma_c), "r"(src), "r"(n0 + b * 32),
                                 "r"(m0)
                                 : "memory");
            }
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
        }
    }
}

// ---- host side ----
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                  const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess && qr == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

// [rows][K] fp16 row-major, box = {BK (inner, 128 bytes), box_rows}, 128-byte swizzle
inline int make_map(CUtensorMap *map, const void *base, uint64_t rows, uint64_t K, uint32_t box_rows) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return -1;
    cuuint64_t dims[2] = {K, rows};
    cuuint64_t strides[1] = {K * 2};
    cuuint32_t box[2] = {(cuuint32_t)BK, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : -2;
}

// C / x as [rows][cols] fp32 row-major, box = 32 columns (128 bytes) x 128 rows, 128-byte swizzle (matches the epilogue's staging)
inline int make_map_c(CUtensorMap *map, const void *base, uint64_t rows, uint64_t cols) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return -1;
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {cols * 4};
    cuuint32_t box[2] = {32, (cuuint32_t)BM};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : -2;
}

// The tile-major Q8_0 stream (stream_matvec.cuh) as a 4-D byte tensor {unit byte, slot r, segment s, group G}: every
// stride a multiple of 16.  which = 0: the quant box {64, 4, 1, 32} (128 rows x one k-block); which = 1: the scale box
// {16, 4, 1, 32} (128 rows x the 16-byte aligned line of 8 scales that holds the k-block's two).
inline int make_map_q8(CUtensorMap *map, const void *base, uint64_t rows, int nseg, int unit_bytes, int which) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return -1;
    cuuint64_t dims[4] = {(cuuint64_t)unit_bytes, 4, (cuuint64_t)nseg, rows / 4};
    cuuint64_t strides[3] = {(cuuint64_t)unit_bytes, 4ull * unit_bytes, 4ull * unit_bytes * nseg};
    cuuint32_t box[4] = {which ? 16u : (cuuint32_t)BK, 4, 1, BN / 4};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : -2;
}

// 4 stages x 32 KB of operands: the default ring (the C tile, 64 KB, is staged in it).  6 stages (192 KB) is the deep
// variant the GEMM test also runs, so a ring that wraps at a different k-block is exercised too.  W8A16 adds a 10 KB
// raw stage per stage, so its deep variant is 5 stages (211 KB).
constexpr int GEMM_STAGES = 4, GEMM_STAGES_DEEP = 6, GEMM_STAGES_DEEP_Q8 = 5;
static_assert(smem_bytes<GEMM_STAGES_DEEP_Q8, B_Q8>() <= 227 * 1024, "W8A16 deep ring exceeds the shared-memory budget");

// m_tiles x n_tiles output tiles, K split into `splits` ranges (GEMM_RESID only: every split reduce-adds its partial product).
// B maps have box rows BN (BN / 2 for the W1 / W3 maps of GEMM_GATEUP).  BSRC = B_Q8: b / b2 are the make_map_q8 quant /
// scale maps of one stream, seg its segment width (a multiple of BK, so no k-block straddles two segments).
template <int MODE, int STAGES, int BSRC = B_F16>
inline int gemm_launch(const CUtensorMap &a, const CUtensorMap &b, const CUtensorMap &b2, const CUtensorMap &c, void *C, int ldc, int m_valid, int m_tiles,
                       int n_tiles, int K, cudaStream_t stream, int splits = 1, int seg = 0, float oscale = 1.0f) {
    static bool attr = false; // one flag per instantiation
    if (!attr) {
        if (cudaFuncSetAttribute(k_gemm_f16_wgmma<MODE, STAGES, BSRC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes<STAGES, BSRC>()) != cudaSuccess)
            return -4;
        attr = true;
    }
    if (splits < 1 || (splits > 1 && MODE != GEMM_RESID)) return -6;
    if (BSRC == B_Q8 && (seg <= 0 || seg % BK || K % seg)) return -6;
    const int nk = (K + BK - 1) / BK, per = (nk + splits - 1) / splits;
    if ((splits - 1) * per >= nk) return -6; // an empty split would store an unwritten accumulator
    k_gemm_f16_wgmma<MODE, STAGES, BSRC><<<dim3(m_tiles, n_tiles, splits), GEMM_THREADS, smem_bytes<STAGES, BSRC>(), stream>>>(a, b, b2, c, C, ldc, m_valid, K,
                                                                                                                          per, seg, oscale);
    return cudaGetLastError() == cudaSuccess ? 0 : -5;
}

// Test/measurement entry: C[M,N] (+)= A[M,K] * B[N,K]^T ; M, N multiples of 128, K multiple of 64.  Device pointers.
// resid > 0: reduce-add into C with K split resid ways.
inline int gemm_f16(const __half *A, const __half *B, float *C, int M, int N, int K, int stages, int resid, cudaStream_t stream) {
    if (M % BM || N % BN || K % BK) return -3;
    CUtensorMap ma, mb, mc;
    int rc;
    if ((rc = make_map(&ma, A, (uint64_t)M, (uint64_t)K, BM))) return rc;
    if ((rc = make_map(&mb, B, (uint64_t)N, (uint64_t)K, BN))) return rc;
    if ((rc = make_map_c(&mc, C, (uint64_t)M, (uint64_t)N))) return rc;
    if (resid && stages == GEMM_STAGES_DEEP) return gemm_launch<GEMM_RESID, GEMM_STAGES_DEEP>(ma, mb, mb, mc, C, N, M, M / BM, N / BN, K, stream, resid);
    if (resid) return gemm_launch<GEMM_RESID, GEMM_STAGES>(ma, mb, mb, mc, C, N, M, M / BM, N / BN, K, stream, resid);
    if (stages == GEMM_STAGES_DEEP) return gemm_launch<GEMM_F32, GEMM_STAGES_DEEP>(ma, mb, mb, mc, C, N, M, M / BM, N / BN, K, stream);
    return gemm_launch<GEMM_F32, GEMM_STAGES>(ma, mb, mb, mc, C, N, M, M / BM, N / BN, K, stream);
}

} // namespace pg
