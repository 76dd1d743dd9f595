// prefill_i8.cuh -- the bit-exact tensor-core prefill (B200_PREFILL_TENSOR_CORE_EXACT) for Q8_0 plans.
//
// The CPU path's Q8_0 dot product (Q8_0FloatTensor.dotQ8Activation, Q8_0FloatTensor.java:90-123) is, per 32-element block, an exact
// int8 x int8 -> int32 sum isum, one float term fl(float(isum) * fl(wScale * aScale)), and result += term from 0f in block order.  Over
// a chunk of tokens that is a GEMM whose K loop is the block loop:
//
//   k_gemm_i8   per 32-column block ONE wgmma.m64n64k32.s32.s8.s8 with scale-d = 0 gives every isum of a 64 x 64 tile exactly
//               (|isum| <= 32 * 128 * 128 < 2^22); the thread that owns an output element then adds its term in registers, block
//               after block, as the CPU path does.  K is never split, so no element's order depends on the tiling.
//
// A = the chunk's int8 activations [rows][K] and their f32 block scales [rows][lds] (lds = K / 32 rounded up to 4: a 16-byte TMA
// box holds the k-block's two scales).  B = the tile-major Q8_0 stream the decode kernels read (stream_matvec.cuh), in place:
// the quant box lands with a 64-byte swizzle the wgmma descriptor reads directly, the 16-byte scale line next to it.  Warp groups:
// 0 = the TMA producer (one thread), 1 and 2 = consumers of tile rows 0-63 and 64-127.  Each consumer keeps two s32 accumulator
// sets: the wgmma of a k-block's second 32-column block runs while the terms of its first are added, and so on.
//
// Epilogues: STORE (QKV: out = acc), I8_LOGITS (k_gemm_i8_logits, the classifier of b200_score_tokens: out = fl(acc * oscale),
// Granite's logitScale or 1, as the streaming classifier stores it; every column of the tile is written, so C's row stride covers
// whole 64-column tiles), RESID (Wo, W2: x = fl(x + fl(acc * oscale)), Granite's residualScale or 1), GATEUP (the
// interleaved gate/up stream: a 64-row tile is 32 gate and 32 up rows of the same 32 hidden units, so swiglu_exact and the Q8_0
// quantisation of that 32-unit block (quant_block_lane) both finish inside the tile).  These are the batched step's epilogues
// (decode_batch.cuh), element for element.
//
// The chunk forms of the exact per-row bodies run around the GEMMs over a per-token table (ChunkTok): k_i8_norm
// (rmsnorm_quant_row, one CTA per token), k_i8_rope_kv (rope_kv_prologue, grid heads x tokens) and k_i8_attention
// (attention_head<HS, true>, grid heads x tokens, after every K / V row of the chunk is in the cache).
//
// MoE plans (B200_PREFILL_TENSOR_CORE_EXACT_MOE) run the same attention half; their FFN half groups the chunk's (token, expert)
// assignments by expert (k_xp_group, k_xp_gather) and runs gemm_i8_body over every expert's rows as one grouped launch per
// projection (k_xp_gemm), then adds the results in the decode's order (k_xp_combine).  The chunk router is in moe.cuh (k_xp_route).
//
// On a plan that keeps K-quant weights resident, each resident matrix is first expanded to the Q8_0 tiles a Q8_0-tile plan of the
// same file holds (k_kq_tiles_to_q8, stream_matvec.cuh) in one scratch the size of the largest, and its GEMM reads them there.
#pragma once
#include "decode_kernels.cuh"
#include "moe.cuh"
#include "prefill.cuh"
#include "stream_matvec.cuh"

namespace pg {

constexpr int I8_BN = 64, I8_STAGES = 8;
constexpr int I8_LOGITS = 3; // the epilogue of k_gemm_i8_logits, next to GEMM_F32 / GEMM_RESID / GEMM_GATEUP (prefill_gemm.cuh)
// one stage: A quants (128 rows x 64 bytes, 64-byte swizzle), B quants (64 rows x 64 bytes, same swizzle), A scale lines (128 x 16
// bytes), B scale lines (64 x 16 bytes).  Every part starts on a 1024-byte boundary of the stage.
constexpr int I8_A_BYTES = BM * BK, I8_B_BYTES = I8_BN * BK, I8_AS_BYTES = BM * 16, I8_BS_BYTES = I8_BN * 16;
constexpr int I8_STAGE_BYTES = I8_A_BYTES + I8_B_BYTES + I8_AS_BYTES + I8_BS_BYTES;
constexpr int I8_HBUF_BYTES = BM * 32 * 4; // GATEUP: the tile's 128 rows x 32 hidden units before quantisation
constexpr size_t i8_smem_bytes() { return (size_t)I8_STAGES * I8_STAGE_BYTES + I8_HBUF_BYTES + 2 * I8_STAGES * 8 + 1024; }
static_assert(I8_STAGE_BYTES % 1024 == 0, "stage parts keep the swizzle atoms aligned");
static_assert(i8_smem_bytes() <= 227 * 1024, "the int8 GEMM ring exceeds the shared-memory budget");

// f32 block scales per activation row: K / 32 rounded up to whole 16-byte lines
__host__ __device__ inline int i8_lds(int K) { return (K / 32 + 3) & ~3; }

struct I8Out {
    float *C;    // STORE / RESID: f32 [rows][ldc]
    int ldc;
    int8_t *hq;  // GATEUP: quantised hidden rows [rows][ldq] and their block scales [rows][lds]
    float *hs;
    int ldq, lds;
    int m_valid; // k_gemm_i8: rows >= m_valid are never written (the grouped kernel k_xp_gemm takes its bound from its tile table)
    int K, seg;  // K: a multiple of seg; seg: the stream's segment width, a multiple of 64
    float oscale;
};

// wgmma shared-memory descriptor, K-major, 64-byte swizzle: start >> 4 | LBO 1 (unused) | SBO = 8 rows x 64 B >> 4 | SWIZZLE_64B (2) << 62
__device__ __forceinline__ uint64_t wgmma_desc_sw64(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | (32ull << 32) | (2ull << 62);
}

// d[64 x 64] = A[64 x 32] * B[64 x 32]^T (int8 -> int32, scale-d = 0: the previous contents are ignored).  Thread t holds, for
// j = 0..7, columns 8j + 2(t%4) + {0,1} of row 16(t/32) + (t%32)/4 in d[4j], d[4j+1] and of that row + 8 in d[4j+2], d[4j+3].
__device__ __forceinline__ void wgmma_i8_m64n64k32(int (&d)[32], uint64_t da, uint64_t db) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
        "%32, %33, p;\n"
        "}\n"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]),
          "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]),
          "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]),
          "+r"(d[31])
        : "l"(da), "l"(db), "r"(0)
        : "memory");
}

// The accumulator registers are read only after the wgmma that writes them has completed (wgmma.wait_group): tie them to a volatile
// statement after the wait so that no read is scheduled above it.
__device__ __forceinline__ void i8_fence_regs(int (&d)[32]) {
#pragma unroll
    for (int i = 0; i < 32; i++) asm volatile("" : "+r"(d[i])::"memory");
}

// float(isum) exactly for |isum| < 2^22: isum added to the bit pattern of 1.5 * 2^23 is the float 1.5 * 2^23 + isum, and the
// subtraction of 1.5 * 2^23 is exact (isum = 0 gives +0, as (float)0 does)
__device__ __forceinline__ float i8_to_float(int isum) { return __fsub_rn(__int_as_float(isum + 0x4B400000), 12582912.0f); }

// The GEMM of the kernels below: k_gemm_i8 (the prefill's epilogues), k_gemm_i8_logits (I8_LOGITS) and k_xp_gemm (the grouped
// expert GEMMs): the 128-row tile from A row m0, rows >= m_valid never written.  A consumer warp group whose 64 rows all lie at or
// past m_valid computes nothing: it only releases each stage once it has landed (so its arrival counts for that stage's lap).
template <int MODE>
__device__ __forceinline__ void gemm_i8_body(const CUtensorMap &tma_a, const CUtensorMap &tma_as, const CUtensorMap &tma_bq, const CUtensorMap &tma_bs,
                                             const I8Out &o, int m0, int m_valid) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    float *hbuf = reinterpret_cast<float *>(smem + I8_STAGES * I8_STAGE_BYTES);
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + I8_STAGES * I8_STAGE_BYTES + I8_HBUF_BYTES);
    const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + I8_STAGES);
    const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        // full: the producer's expect_tx; empty: one arrival per consumer warp once it has read the stage (operands and scales)
        for (int s = 0; s < I8_STAGES; s++) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int nk = o.K / BK, g0 = blockIdx.y * (I8_BN / 4);

    if (wg == 0) {
        if (warp == 0 && lane == 0) {
            for (int kb = 0; kb < nk; kb++) {
                const int st = kb % I8_STAGES;
                mbar_wait(empty0 + 8 * st, ((kb / I8_STAGES) & 1) ^ 1);
                const int kc = kb * BK, s = kc / o.seg, j = kc - s * o.seg;
                const uint32_t base = smem_u32(smem + st * I8_STAGE_BYTES), full = full0 + 8 * st;
                mbar_expect_tx(full, I8_STAGE_BYTES);
                tma_load_2d(base, &tma_a, kc, m0, full);
                tma_load_4d(base + I8_A_BYTES, &tma_bq, j, 0, s, g0, full);
                tma_load_2d(base + I8_A_BYTES + I8_B_BYTES, &tma_as, (2 * kb) & ~3, m0, full);
                tma_load_4d(base + I8_A_BYTES + I8_B_BYTES + I8_AS_BYTES, &tma_bs, o.seg + ((j >> 8) << 4), 0, s, g0, full);
            }
        }
        return;
    }

    // ===== consumers: warp group c = wg - 1 owns tile rows 64c .. 64c+63 =====
    const int c = wg - 1, t = threadIdx.x & 127;
    if (m0 + c * 64 >= m_valid) {
        for (int kb = 0; kb < nk; kb++) {
            const int st = kb % I8_STAGES;
            mbar_wait(full0 + 8 * st, (kb / I8_STAGES) & 1);
            __syncwarp();
            if (lane == 0) mbar_arrive(empty0 + 8 * st);
        }
        return;
    }
    const int r_lo = c * 64 + (t >> 5) * 16 + ((t & 31) >> 2); // tile row of d[4j], d[4j+1]; d[4j+2], d[4j+3] are row r_lo + 8
    const int cq = 2 * (t & 3);
    float acc[32];
    int da[32], db[32];
#pragma unroll
    for (int i = 0; i < 32; i++) { acc[i] = 0.0f; da[i] = 0; db[i] = 0; }
    auto issue = [&](int (&d)[32], int st, int sub) { // sub: the k-block's first or second 32-column block (+32 bytes = +2 in the address field)
        const uint32_t base = smem_u32(smem + st * I8_STAGE_BYTES);
        asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
        wgmma_i8_m64n64k32(d, wgmma_desc_sw64(base + c * 64 * BK) + 2 * sub, wgmma_desc_sw64(base + I8_A_BYTES) + 2 * sub);
        asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    };
    // result += fl(float(isum) * fl(wScale * aScale)) for block 2 kb + sub of every element this thread owns
    auto terms = [&](const int (&d)[32], int st, int kb, int sub) {
        const uint8_t *base = smem + st * I8_STAGE_BYTES;
        const float *as = reinterpret_cast<const float *>(base + I8_A_BYTES + I8_B_BYTES);
        const int ai = 2 * (kb & 1) + sub; // the box starts at block (2 kb) & ~3
        const float a0 = as[4 * r_lo + ai], a1 = as[4 * (r_lo + 8) + ai];
        const int j = kb * BK % o.seg; // column of the k-block in its segment: its scales start at ((j & 255) >> 5) in the 8-scale line
        const uint8_t *bs = base + I8_A_BYTES + I8_B_BYTES + I8_AS_BYTES + 2 * (((j & 255) >> 5) + sub);
#pragma unroll
        for (int jj = 0; jj < 8; jj++)
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const float w = __half2float(*reinterpret_cast<const __half *>(bs + 16 * (8 * jj + cq + e)));
                acc[4 * jj + e] = __fadd_rn(acc[4 * jj + e], __fmul_rn(i8_to_float(d[4 * jj + e]), __fmul_rn(w, a0)));
                acc[4 * jj + 2 + e] = __fadd_rn(acc[4 * jj + 2 + e], __fmul_rn(i8_to_float(d[4 * jj + 2 + e]), __fmul_rn(w, a1)));
            }
    };
    mbar_wait(full0, 0);
    issue(da, 0, 0);
    for (int kb = 0; kb < nk; kb++) {
        const int st = kb % I8_STAGES;
        issue(db, st, 1);
        asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); // da (block 2 kb) is complete
        i8_fence_regs(da);
        terms(da, st, kb, 0);
        if (kb + 1 < nk) {
            const int st1 = (kb + 1) % I8_STAGES;
            mbar_wait(full0 + 8 * st1, ((kb + 1) / I8_STAGES) & 1);
            issue(da, st1, 0);
            asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); // db (block 2 kb + 1) is complete
        } else {
            asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
        }
        i8_fence_regs(db);
        terms(db, st, kb, 1);
        __syncwarp();
        if (lane == 0) mbar_arrive(empty0 + 8 * st);
    }

    const int n0 = blockIdx.y * I8_BN;
    if (MODE == GEMM_GATEUP) {
        // column 8jj + cq + e is stream row 4 (2jj + cq / 4) + cq % 4 + e: even lanes (cq = 0, 4) hold gate units 4jj + cq / 2 + e,
        // their odd neighbours the up rows of the same units
        float *hb = hbuf + c * 64 * 32;
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int jj = 0; jj < 8; jj++)
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const float g = acc[4 * jj + 2 * h + e];
                    const float u = __shfl_xor_sync(0xffffffffu, g, 1);
                    if (!(t & 1)) hb[(r_lo - c * 64 + 8 * h) * 32 + 4 * jj + (cq >> 1) + e] = swiglu_exact(g, u);
                }
        asm volatile("bar.sync %0, 128;" ::"r"(2 + c) : "memory");
        for (int r = (t >> 5); r < 64; r += 4) {
            const int row = m0 + c * 64 + r;
            if (row >= m_valid) break; // warp-uniform
            float as;
            const int q = quant_block_lane(hb[r * 32 + lane], as);
            o.hq[(size_t)row * o.ldq + blockIdx.y * 32 + lane] = (int8_t)q;
            if (lane == 0) o.hs[(size_t)row * o.lds + blockIdx.y] = as;
        }
    } else {
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int row = m0 + r_lo + 8 * h;
            if (row < m_valid) {
                float *dst = o.C + (size_t)row * o.ldc + n0 + cq;
#pragma unroll
                for (int jj = 0; jj < 8; jj++)
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        const float v = acc[4 * jj + 2 * h + e];
                        if (MODE == GEMM_RESID) dst[8 * jj + e] = __fadd_rn(dst[8 * jj + e], __fmul_rn(v, o.oscale));
                        else if (MODE == I8_LOGITS) dst[8 * jj + e] = __fmul_rn(v, o.oscale);
                        else dst[8 * jj + e] = v;
                    }
            }
        }
    }
}

template <int MODE>
__global__ void __launch_bounds__(GEMM_THREADS, 1) k_gemm_i8(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_as,
                                                          const __grid_constant__ CUtensorMap tma_bq, const __grid_constant__ CUtensorMap tma_bs,
                                                          const I8Out o) {
    gemm_i8_body<MODE>(tma_a, tma_as, tma_bq, tma_bs, o, blockIdx.x * BM, o.m_valid);
}

__global__ void __launch_bounds__(GEMM_THREADS, 1) k_gemm_i8_logits(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_as,
                                                                 const __grid_constant__ CUtensorMap tma_bq, const __grid_constant__ CUtensorMap tma_bs,
                                                                 const I8Out o) {
    gemm_i8_body<I8_LOGITS>(tma_a, tma_as, tma_bq, tma_bs, o, blockIdx.x * BM, o.m_valid);
}

template <int MODE> constexpr auto gemm_i8_kernel() {
    if constexpr (MODE == I8_LOGITS) return k_gemm_i8_logits;
    else return k_gemm_i8<MODE>;
}


// ---- the grouped expert GEMMs of B200_PREFILL_TENSOR_CORE_EXACT_MOE ----------------------------------------------------------
// The chunk's n * k (token, slot) assignments, grouped by expert (k_xp_group), form the rows of one A operand: expert e's rows are
// [offset[e], offset[e] + count[e]), in token order.  Each expert's rows are cut into 128-row M tiles; one tile table entry per tile.
struct XpTile {
    int expert, row0, rows, pad;
};
// Upper bound of the tile table: every expert's last tile may be partial.
__host__ __device__ inline int xp_max_tiles(int assignments, int n_experts) {
    return (assignments + BM - 1) / BM + (n_experts < assignments ? n_experts : assignments);
}
// The tile table of per-expert row counts and offsets, experts in index order; returns its length.  k_xp_group and the test hook
// build it with this one function.
__host__ __device__ inline int xp_tile_table(const int *count, const int *offset, int E, XpTile *tiles) {
    int nt = 0;
    for (int e = 0; e < E; e++)
        for (int r = 0; r < count[e]; r += BM) tiles[nt++] = XpTile{e, offset[e] + r, count[e] - r < BM ? count[e] - r : BM, 0};
    return nt;
}

// The grouped kernel: blockIdx.x indexes the tile table (CTAs past its length return before any barrier), blockIdx.y the 64-column
// N tile.  maps: the layer's per-expert tensor maps [expert][4] = gate/up quants, gate/up scales, down quants, down scales, written
// by the host before the first launch; GATEUP reads entries 0 / 1, STORE entries 2 / 3.
template <int MODE>
__global__ void __launch_bounds__(GEMM_THREADS, 1) k_xp_gemm(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_as,
                                                          const CUtensorMap *__restrict__ maps, const XpTile *__restrict__ tiles,
                                                          const int *__restrict__ n_tiles, const I8Out o) {
    if ((int)blockIdx.x >= *n_tiles) return;
    const XpTile tl = tiles[blockIdx.x];
    const CUtensorMap *m = maps + 4 * tl.expert + (MODE == GEMM_GATEUP ? 0 : 2);
    if (threadIdx.x == 0) // the maps live in global memory: acquire them for the tensor-map proxy before the producer's first copy
        asm volatile("fence.proxy.tensormap::generic.acquire.sys [%0], 128;\n\tfence.proxy.tensormap::generic.acquire.sys [%1], 128;" ::"l"(m), "l"(m + 1)
                     : "memory");
    gemm_i8_body<MODE>(tma_a, tma_as, m[0], m[1], o, tl.row0, tl.row0 + tl.rows);
}

// grid_m = xp_max_tiles(...) M slots, n_tiles N tiles.  -6: a shape the kernel does not take.
template <int MODE>
inline int xp_gemm_launch(const CUtensorMap &a, const CUtensorMap &as, const CUtensorMap *maps, const XpTile *tiles, const int *n_tiles, const I8Out &o,
                          int grid_m, int n_tiles_n, cudaStream_t stream) {
    static bool attr = false; // one flag per instantiation
    if (!attr) {
        if (cudaFuncSetAttribute(k_xp_gemm<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)i8_smem_bytes()) != cudaSuccess) return -4;
        attr = true;
    }
    if (o.seg <= 0 || o.seg % BK || o.K <= 0 || o.K % o.seg || grid_m < 1 || n_tiles_n < 1) return -6;
    k_xp_gemm<MODE><<<dim3(grid_m, n_tiles_n), GEMM_THREADS, i8_smem_bytes(), stream>>>(a, as, maps, tiles, n_tiles, o);
    return cudaGetLastError() == cudaSuccess ? 0 : -5;
}

// Deterministic, stable counting sort of the na = n * k assignments (ids [n][k], assignment a = t * k + j) by expert, on one CTA:
// XP_SLICES slices of the assignments, one thread per (slice, expert) counting, then placing its slice's assignments in order.
// row_of[a]: the assignment's grouped row; offsets[e] (e <= E): first grouped row of expert e; tiles / *n_tiles: the tile table.
constexpr int XP_GROUP_THREADS = 1024, XP_SLICES = XP_GROUP_THREADS / MOE_MAX_EXPERTS;
__global__ void __launch_bounds__(XP_GROUP_THREADS, 1) k_xp_group(const int *__restrict__ ids, int na, int E, int *__restrict__ row_of,
                                                                  int *__restrict__ offsets, XpTile *__restrict__ tiles, int *__restrict__ n_tiles) {
    __shared__ int cnt[XP_SLICES][MOE_MAX_EXPERTS], base[XP_SLICES][MOE_MAX_EXPERTS], tot[MOE_MAX_EXPERTS], off[MOE_MAX_EXPERTS + 1];
    const int e = threadIdx.x % MOE_MAX_EXPERTS, s = threadIdx.x / MOE_MAX_EXPERTS;
    const int a0 = (int)((long long)na * s / XP_SLICES), a1 = (int)((long long)na * (s + 1) / XP_SLICES);
    int c = 0;
    if (e < E)
        for (int i = a0; i < a1; i++) c += ids[i] == e;
    cnt[s][e] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        int o = 0;
        for (int x = 0; x < E; x++) {
            off[x] = o;
            for (int q = 0; q < XP_SLICES; q++) { base[q][x] = o; o += cnt[q][x]; }
            tot[x] = o - off[x];
        }
        off[E] = o;
        *n_tiles = xp_tile_table(tot, off, E, tiles);
    }
    __syncthreads();
    if (e < E) {
        int r = base[s][e];
        for (int i = a0; i < a1; i++)
            if (ids[i] == e) row_of[i] = r++;
    }
    if ((int)threadIdx.x <= E) offsets[threadIdx.x] = off[threadIdx.x];
}

// One CTA per assignment: token t's int8 row (dim bytes) and its block scales (lds floats) into grouped row row_of[a].
__global__ void __launch_bounds__(128) k_xp_gather(const int8_t *__restrict__ xq, const float *__restrict__ xs, int dim, int lds, int k,
                                                   const int *__restrict__ row_of, int8_t *__restrict__ gq, float *__restrict__ gs) {
    const int a = blockIdx.x, t = a / k, r = row_of[a];
    const int4 *src = reinterpret_cast<const int4 *>(xq + (size_t)t * dim);
    int4 *dst = reinterpret_cast<int4 *>(gq + (size_t)r * dim);
    for (int i = threadIdx.x; i < dim / 16; i += blockDim.x) dst[i] = src[i];
    for (int i = threadIdx.x; i < lds; i += blockDim.x) gs[(size_t)r * lds + i] = xs[(size_t)t * lds + i];
}

// The ordered combine, one CTA per chunk row (moe_down's epilogue order): x = fl(fl(w_j * Yg[row(t, j)]) + x) for j in selection
// order, then with a shared expert x = fl(fl(w_shared * Ys[t]) + x).
__global__ void __launch_bounds__(256) k_xp_combine(float *__restrict__ x, int dim, const float *__restrict__ yg, const int *__restrict__ row_of,
                                                    const float *__restrict__ w, int k, int nw, const float *__restrict__ ys) {
    __shared__ int rows[MOE_MAX_K];
    __shared__ float ws[MOE_MAX_K + 1];
    const int t = blockIdx.x;
    if ((int)threadIdx.x < k) rows[threadIdx.x] = row_of[(size_t)t * k + threadIdx.x];
    if ((int)threadIdx.x < nw) ws[threadIdx.x] = w[(size_t)t * nw + threadIdx.x];
    __syncthreads();
    float *xr = x + (size_t)t * dim;
    for (int i = threadIdx.x; i < dim; i += blockDim.x) {
        float v = xr[i];
        for (int j = 0; j < k; j++) v = __fadd_rn(__fmul_rn(ws[j], yg[(size_t)rows[j] * dim + i]), v);
        if (ys) v = __fadd_rn(__fmul_rn(ws[k], ys[(size_t)t * dim + i]), v);
        xr[i] = v;
    }
}

// ---- host side ----
inline int i8_encode(CUtensorMap *map, CUtensorMapDataType type, int rank, const void *base, const cuuint64_t *dims, const cuuint64_t *strides,
                     const cuuint32_t *box, CUtensorMapSwizzle swz) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return -1;
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    return fn(map, type, rank, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS
               ? 0
               : -2;
}
// int8 activations [rows][K]: box {64 bytes, 128 rows}, 64-byte swizzle
inline int make_map_i8_a(CUtensorMap *map, const int8_t *base, uint64_t rows, uint64_t K) {
    const cuuint64_t dims[2] = {K, rows}, strides[1] = {K};
    const cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)BM};
    return i8_encode(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, base, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_64B);
}
// their f32 block scales [rows][lds]: box {4 scales (16 bytes), 128 rows}
inline int make_map_i8_s(CUtensorMap *map, const float *base, uint64_t rows, uint64_t lds) {
    const cuuint64_t dims[2] = {lds, rows}, strides[1] = {lds * 4};
    const cuuint32_t box[2] = {4, (cuuint32_t)BM};
    return i8_encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, base, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE);
}
// The tile-major Q8_0 stream as make_map_q8 describes it, with 64-row boxes: which = 0, the quants of one k-block (64-byte swizzle,
// the wgmma B operand as it lands); which = 1, the 16-byte scale lines
inline int make_map_i8_q8(CUtensorMap *map, const void *base, uint64_t rows, int nseg, int unit_bytes, int which) {
    const cuuint64_t dims[4] = {(cuuint64_t)unit_bytes, 4, (cuuint64_t)nseg, rows / 4};
    const cuuint64_t strides[3] = {(cuuint64_t)unit_bytes, 4ull * unit_bytes, 4ull * unit_bytes * nseg};
    const cuuint32_t box[4] = {which ? 16u : (cuuint32_t)BK, 4, 1, I8_BN / 4};
    return i8_encode(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, base, dims, strides, box, which ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_64B);
}

// m_tiles x n_tiles tiles of 128 x 64 (GATEUP: 64 stream rows = 32 hidden units per tile).  -6: a shape the kernel does not take.
template <int MODE>
inline int gemm_i8_launch(const CUtensorMap &a, const CUtensorMap &as, const CUtensorMap &bq, const CUtensorMap &bs, const I8Out &o, int m_tiles,
                          int n_tiles, cudaStream_t stream) {
    static bool attr = false; // one flag per instantiation
    if (!attr) {
        if (cudaFuncSetAttribute(gemm_i8_kernel<MODE>(), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)i8_smem_bytes()) != cudaSuccess) return -4;
        attr = true;
    }
    if (o.seg <= 0 || o.seg % BK || o.K <= 0 || o.K % o.seg || m_tiles < 1 || n_tiles < 1) return -6;
    gemm_i8_kernel<MODE>()<<<dim3(m_tiles, n_tiles), GEMM_THREADS, i8_smem_bytes(), stream>>>(a, as, bq, bs, o);
    return cudaGetLastError() == cudaSuccess ? 0 : -5;
}

} // namespace pg

// ---- chunk forms of the exact per-row bodies ----------------------------------------------------------------------------------
// One entry per chunk token: its token id, position, and the float offset of its KV cache (0: the plan's own cache; slot s of
// b200_prefill_slots: s * slot_stride).
struct ChunkTok {
    int token, pos;
    long long kv;
};

// B200_PREFILL_TENSOR_CORE_EXACT_MOE (MoE plans, built with the chunk buffers): the FFN norm's float rows XB (the router's input), the
// chunk routing of every layer (ids [layer][bpad][k], w [layer][bpad][nw]), the grouping (row_of, offsets, the tile table), the
// grouped A rows GQ / GS and hidden rows HQg / HSg (n * k + 128 rows: a tile may read past its expert's rows), the grouped down
// outputs Yg [n * k][dim], the shared expert's down outputs Ys [bpad][dim] (Qwen2-MoE) and the per-expert tensor maps.
struct XpCtx {
    float *XB = nullptr, *w = nullptr, *GS = nullptr, *HSg = nullptr, *Yg = nullptr, *Ys = nullptr;
    int *ids = nullptr, *row_of = nullptr, *offsets = nullptr, *n_tiles = nullptr;
    int8_t *GQ = nullptr, *HQg = nullptr;
    pg::XpTile *tiles = nullptr;
    CUtensorMap *maps = nullptr;      // device [layer][expert][4]: make_map_i8_q8 quant / scale maps of gate/up, then of down
    CUtensorMap a_g, s_g, a_hg, s_hg; // A operands of the grouped gate/up (K = dim) and down (K = expert hidden) GEMMs
    int rows = 0;                     // rows of the last chunk (b200_read_buffer "moe_chunk_ids" / "moe_chunk_weights")
};

// The mode's chunk buffers for bpad rows (built on the first b200_set_prefill_mode(TENSOR_CORE_EXACT)): X and QKV as the batched
// step keeps them per row; XQ / XS the int8 activations of the QKV, gate/up (row stride dim) and Wo (row stride q width) GEMMs, HQ /
// HS those of W2 (MoE: of the shared expert's down projection, K = shared hidden); the token table; score rows for ATT_TOKENS tokens
// at a time when the context needs global score rows.
struct PrefillI8Ctx {
    int bpad = 0, att_tokens = 0;
    float *X = nullptr, *QKV = nullptr, *XS = nullptr, *HS = nullptr, *att = nullptr;
    int8_t *XQ = nullptr, *HQ = nullptr;
    ChunkTok *tok = nullptr;
    unsigned char *kq8 = nullptr;                   // resident plans: the Q8_0 tiles of the resident matrix the next GEMM reads
    int64_t kq8_bytes = 0;                          // its size (b200_score_tokens grows it to the classifier's tiles)
    CUtensorMap a_dim, s_dim, a_qd, s_qd, a_h, s_h; // A operands: K = dim (XQ), K = q width (XQ), K = hidden (HQ)
    std::vector<PrefillQ8Maps> maps;                // per layer: make_map_i8_q8 quant / scale maps of the four streams (over kq8
                                                    // for a resident stream); MoE layers: the shared expert's gate/up
                                                    // and down (Qwen2-MoE) in the gate/up and W2 slots, or none
    XpCtx xp;
};
// Global score rows of one attention launch are bounded by this many bytes (att_tokens = max(1, bound / (heads x context x 4))).
constexpr size_t I8_ATT_SCRATCH_MAX = (size_t)64 << 20;

template <bool EMBED>
__global__ void __launch_bounds__(NORM_THREADS, 1) k_i8_norm(float *__restrict__ x, const ChunkTok *__restrict__ tok, DevMat emb, float emb_scale,
                                                         const float *__restrict__ w, float eps, int dim, int8_t *__restrict__ xq,
                                                         float *__restrict__ xs, int lds, float *__restrict__ xb, TraceBuf tr, TpCtx tp) {
    const int v = blockIdx.x;
    rmsnorm_quant_row<EMBED>(x + (size_t)v * dim, &tok[v].token, emb, emb_scale, w, eps, dim, xq + (size_t)v * dim, xs + (size_t)v * lds,
                             xb ? xb + (size_t)v * dim : nullptr, nullptr, tr, tp, -1);
}

template <int HS>
__global__ void __launch_bounds__(2 * HS) k_i8_rope_kv(float *__restrict__ qkv, int qkv_stride, float *__restrict__ kc, float *__restrict__ vc,
                                                      const ChunkTok *__restrict__ tok, const float *__restrict__ cr, const float *__restrict__ ci,
                                                      int n_heads, int n_kv_heads, int arch, const float *__restrict__ qnorm_w,
                                                      const float *__restrict__ knorm_w, const float *__restrict__ qkv_bias, float eps) {
    __shared__ __align__(16) float sq[HS], sk[HS], so[HS];
    __shared__ float s_val[2];
    const int v = blockIdx.y, h = blockIdx.x;
    const ChunkTok t = tok[v];
    const int kv_mul = n_heads / n_kv_heads, kvh = h / kv_mul, qd = n_heads * HS, kvd = n_kv_heads * HS;
    float *q = qkv + (size_t)v * qkv_stride;
    rope_kv_prologue<HS>(q, q + h * HS, q + qd + kvh * HS, q + qd + kvd + kvh * HS, kc + t.kv, vc + t.kv, t.pos, h, kv_mul, kvh, qd, kvd, cr, ci, arch,
                         qnorm_w, knorm_w, qkv_bias, eps, sq, sk, so, s_val);
}

// Tokens v0 .. v0 + gridDim.y - 1; att_scratch (long contexts): one score row per (head, token of this launch)
template <int HS>
__global__ void __launch_bounds__(ATT_THREADS) k_i8_attention(float *__restrict__ qkv, int qkv_stride, float *__restrict__ kc, float *__restrict__ vc,
                                                             const ChunkTok *__restrict__ tok, int v0, int n_heads, int n_kv_heads, int arch, float sqrt_hs,
                                                             int8_t *__restrict__ xq, float *__restrict__ xs, int lds, float *att_scratch, int ctx,
                                                             TraceBuf tr, TpCtx tp) {
    const int v = v0 + blockIdx.y, qd = n_heads * HS;
    const ChunkTok *t = tok + v;
    attention_head<HS, true>(qkv + (size_t)v * qkv_stride, kc + t->kv, vc + t->kv, &t->pos, nullptr, nullptr, n_heads, n_kv_heads, arch, nullptr,
                             nullptr, nullptr, 0.0f, sqrt_hs, xq + (size_t)v * qd, xs + (size_t)v * lds, nullptr, tr, tp, 0u, 0,
                             att_scratch ? att_scratch + (size_t)blockIdx.y * n_heads * ctx : nullptr, ctx);
}
