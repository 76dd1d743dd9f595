// kquant.cuh -- load-time re-quantisation of K-quant tensors (Q4_K / Q5_K / Q6_K) to Q8_0 ON THE DEVICE, inside the upload pipeline
// (SURVEY 8(f) N4).  The reference does this on the host, one element at a time, while loading
// (ModelLoader.dequantizeToQ8_0TornadoTensor, model/loader/ModelLoader.java:173-224); here the K-quant bytes cross PCIe as they are
// (4.5-6.6 bits per weight instead of 8.5) and one thread per 32-element block produces the GGUF Q8_0 block the repack kernels expect.
// Byte-identical to the reference's output:
//   element read  = getFloat of tensor/standard/Q4_KFloatTensor.java:90-120, Q5_KFloatTensor.java:84-122, Q6_KFloatTensor.java:64-116
//                   (float products left to right, every operation rounded: __fmul_rn / __fsub_rn, never contracted);
//   block         : maxAbs over the 32 reads, scale = maxAbs / 127f (IEEE division), stored with Float.floatToFloat16 (round to nearest
//                   even), inv = 1f / scale (of the FLOAT scale, not the stored one), q = clamp(Math.round(x * inv), -128, 127) where
//                   Math.round(float) = floor(x + 1/2) evaluated exactly (ties towards +infinity).
#pragma once
#include "common.cuh"

__host__ __device__ inline int kq_block_bytes(int ggml_type) { return ggml_type == 12 ? 144 : ggml_type == 13 ? 176 : ggml_type == 14 ? 210 : 0; }
__host__ __device__ inline bool kq_is_kquant(int ggml_type) { return ggml_type >= 12 && ggml_type <= 14; }

__device__ __forceinline__ float kq_f16(const unsigned char *p) { return __half2float(__ushort_as_half((unsigned short)(p[0] | (p[1] << 8)))); }
__device__ __forceinline__ int kq_scale4(int j, const unsigned char *sc) { return j < 4 ? (sc[j] & 63) : ((sc[j + 4] & 0xF) | ((sc[j - 4] >> 6) << 4)); }
__device__ __forceinline__ int kq_min4(int j, const unsigned char *sc) { return j < 4 ? (sc[j + 4] & 63) : ((sc[j + 4] >> 4) | ((sc[j] >> 6) << 4)); }

// The 32 elements [32 * sub, 32 * sub + 32) of one 256-element super-block.  A Q8_0 block never straddles the sub-block structure of any
// of the three formats, so the per-sub-block constants are read once.
template <int TYPE> __device__ __forceinline__ void kq_read32(const unsigned char *b, int sub, float (&v)[32]) {
    if (TYPE == 12 || TYPE == 13) {
        const float d = kq_f16(b), dmin = kq_f16(b + 2);
        const int pair = sub >> 1, hi_nib = sub & 1;
        const float a = __fmul_rn(d, (float)kq_scale4(sub, b + 4)), c = __fmul_rn(dmin, (float)kq_min4(sub, b + 4));
        const unsigned char *qs = b + (TYPE == 12 ? 16 : 48) + pair * 32;
#pragma unroll
        for (int i = 0; i < 32; i++) {
            int q = hi_nib ? (qs[i] >> 4) : (qs[i] & 0xF);
            if (TYPE == 13) q += ((b[16 + i] >> sub) & 1) * 16; // bit (pair * 2 + nibble) of qh
            v[i] = __fsub_rn(__fmul_rn(a, (float)q), c);
        }
    } else {
        const float d = kq_f16(b + 208);
        const int half = sub >> 2, grp = sub & 3;
        const unsigned char *ql = b + half * 64 + (grp & 1) * 32, *qh = b + 128 + half * 32;
        const signed char *sc = reinterpret_cast<const signed char *>(b + 192 + half * 8 + grp * 2);
#pragma unroll
        for (int i = 0; i < 32; i++) {
            const int lo = grp < 2 ? (ql[i] & 0xF) : (ql[i] >> 4);
            const int qv = (lo | (((qh[i] >> (2 * grp)) & 3) << 4)) - 32;
            v[i] = __fmul_rn(__fmul_rn(d, (float)sc[i >> 4]), (float)qv);
        }
    }
}

// The Q8_0 block the reference builds from elements [32 * sub, 32 * sub + 32) of super-block b: q[k] holds quants 4k..4k+3 packed
// little-endian (the byte order of the GGUF block, and dp4a's operand order), the return value is the f16 scale as stored.  Shared by
// the load-time re-quantiser and the resident weight streams (stream_matvec.cuh), so both produce the same bytes.
template <int TYPE> __device__ __forceinline__ __half kq_q8_block(const unsigned char *b, int sub, int (&q)[8]) {
    float v[32];
    kq_read32<TYPE>(b, sub, v);
    float max_abs = 0.0f;
#pragma unroll
    for (int i = 0; i < 32; i++) { const float a = fabsf(v[i]); max_abs = a > max_abs ? a : max_abs; } // Math.max(maxAbs, Math.abs(x))
    const float scale = __fdiv_rn(max_abs, 127.0f);
    const float inv = scale != 0.0f ? __fdiv_rn(1.0f, scale) : 0.0f;
#pragma unroll
    for (int w = 0; w < 8; w++) {
        unsigned packed = 0u;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const float t = __fmul_rn(v[4 * w + k], inv), f = floorf(t);
            int r = (int)f + (__fsub_rn(t, f) >= 0.5f ? 1 : 0);
            if (t != t) r = 0;
            r = r < -128 ? -128 : (r > 127 ? 127 : r);
            packed |= (unsigned)(r & 0xFF) << (8 * k);
        }
        q[w] = (int)packed;
    }
    return __float2half_rn(scale);
}

// One thread per Q8_0 block; src = K-quant super-blocks (contiguous), dst = GGUF Q8_0 blocks (34 bytes each, 2-byte aligned).
template <int TYPE> __global__ void k_requant_kquant(const unsigned char *__restrict__ src, unsigned char *__restrict__ dst, long long n_blocks) {
    const long long blk = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (blk >= n_blocks) return;
    int q[8];
    const __half sc = kq_q8_block<TYPE>(src + (blk >> 3) * kq_block_bytes(TYPE), (int)(blk & 7), q);
    unsigned short *o = reinterpret_cast<unsigned short *>(dst + blk * 34);
    o[0] = __half_as_ushort(sc);
#pragma unroll
    for (int w = 0; w < 8; w++) {
        o[1 + 2 * w] = (unsigned short)((unsigned)q[w] & 0xFFFFu);
        o[2 + 2 * w] = (unsigned short)((unsigned)q[w] >> 16);
    }
}

static inline cudaError_t launch_requant_kquant(int ggml_type, const unsigned char *src, unsigned char *dst, long long n_blocks, cudaStream_t stream) {
    if (n_blocks <= 0) return cudaSuccess;
    const unsigned grid = (unsigned)((n_blocks + 127) / 128);
    if (ggml_type == 12) k_requant_kquant<12><<<grid, 128, 0, stream>>>(src, dst, n_blocks);
    else if (ggml_type == 13) k_requant_kquant<13><<<grid, 128, 0, stream>>>(src, dst, n_blocks);
    else if (ggml_type == 14) k_requant_kquant<14><<<grid, 128, 0, stream>>>(src, dst, n_blocks);
    else return cudaErrorInvalidValue;
    return cudaGetLastError();
}
