// norm_slots.cuh -- RMSNorm + Q8_0 quantisation of the residual stream straight into a CTA's shared-memory activation buffer,
// computed redundantly by every CTA that consumes it.  Shared by the persistent decode kernel (512 consumer threads,
// decode_persistent.cuh) and the normalising stream matvec (256 consumer threads, stream_matvec.cuh); the arithmetic is
// k_rmsnorm_quant's (InferenceCore.rmsnorm, InferenceCore.java:39-48, then Q8_0FloatTensor.java:100-117 per 32-block).
//
// Thread t of the T consumer threads owns the 16-byte slots i4 = u * T + t (u < U) of the vector: x and the norm weights stay in
// REGISTERS between the two passes; a 32-element quantisation block is eight consecutive slots = eight consecutive lanes, so its
// amax is three shuffles.  Only the squares go through shared memory (the exact accumulator's chunk layout, seqsum2.cuh).
#pragma once
#include "common.cuh"
#include "seqsum2.cuh"

__device__ __forceinline__ float4 ldcg_f32x4(const float *p) {
    float4 v;
    asm volatile("ld.global.cg.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}

// Floats of the squares buffer: T chunks of seqsum2_stride(E) floats, E = ceil(dim / T).
__host__ __device__ inline int norm_slots_sq_floats(int dim, int T) { return T * seqsum2_stride((dim + T - 1) / T); }

// Ops supplies what differs between the callers:
//   sync()                  barrier over the T consumer threads
//   seqsum(sq, n, S)        block_seqsum_exact_v2_t<T> over them (one out-of-line copy per kernel)
//   emb(token, i)           element i of the embedding row times the embedding scale (emb_get)
//   x4(i4)                  slot i4 of the residual stream, read past L1 (written by the previous phase / kernel)
//   store_x(i4, v)          layer 0: where the gathered embedding row has to be written back to x (or nothing)
//   scale(ss, dim, eps)     ss -> (float)(1.0 / sqrt((double)(ss / dim + eps))), the same value in every thread (every thread
//                           holds the same sum; the persistent kernel lets one thread compute it and broadcasts it)
//   w4(wv, u, i4)           slot i4 of the norm weights (wv[u] when they are in registers)
//   stamp(k)                trace hook
// xv: this thread's slots of x, in registers; wv: its slots of the norm weights when the caller keeps them in registers.  On return sxq / sxs hold the quantised vector, visible to all T threads.
template <int T, int U, class Ops>
__device__ __forceinline__ void norm_quant_slots(const Ops &ops, bool from_emb, int token, int dim, float eps, const float4 (&wv)[U], float *sq,
                                                 unsigned *sxq, float *sxs, int tid) {
    const int n4 = dim >> 2;
    const int E = (dim + T - 1) / T, S = seqsum2_stride(E);
    float4 xv[U];
#pragma unroll
    for (int u = 0; u < U; u++) { // every load of this thread in flight at once: one L2 round trip
        const int i4 = u * T + tid;
        xv[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i4 < n4) {
            if (from_emb) { // first layer: the embedding row (quantised table: element-wise, FloatTensor.copyTo)
                xv[u] = make_float4(ops.emb(token, 4 * i4), ops.emb(token, 4 * i4 + 1), ops.emb(token, 4 * i4 + 2), ops.emb(token, 4 * i4 + 3));
                ops.store_x(i4, xv[u]);
            } else xv[u] = ops.x4(i4);
        }
    }
    // squares -> chunk layout: element i belongs to accumulator thread i / E at offset i % E of its S-float chunk
    for (int i = dim + tid; i < T * E; i += T) sq[(i / E) * S + (i % E)] = 0.0f; // zero padding of the last chunks
#pragma unroll
    for (int u = 0; u < U; u++) {
        const int i4 = u * T + tid;
        if (i4 < n4) {
            const int i = 4 * i4;
            const float4 q = make_float4(__fmul_rn(xv[u].x, xv[u].x), __fmul_rn(xv[u].y, xv[u].y), __fmul_rn(xv[u].z, xv[u].z), __fmul_rn(xv[u].w, xv[u].w));
            if ((E & 3) == 0) *reinterpret_cast<float4 *>(sq + (i / E) * S + (i % E)) = q; // the four elements share a chunk
            else {
                sq[(i / E) * S + (i % E)] = q.x; sq[((i + 1) / E) * S + ((i + 1) % E)] = q.y;
                sq[((i + 2) / E) * S + ((i + 2) % E)] = q.z; sq[((i + 3) / E) * S + ((i + 3) % E)] = q.w;
            }
        }
    }
    ops.sync();
    ops.stamp(10);
    float ss = ops.seqsum(sq, dim, S);
    ops.stamp(11);
    ss = ops.scale(ss, dim, eps); // (float)(1.0 / Math.sqrt(ss / size + eps))
#pragma unroll
    for (int u = 0; u < U; u++) { // out = w * (ss * x) (InferenceCore.java:45-47), then Q8_0FloatTensor.java:100-117 per 32-block
        const int i4 = u * T + tid;
        if (u * T < n4) { // warp-uniform (n4 is a multiple of 8 and whole 8-lane groups are in or out)
            float v0 = 0.f, v1 = 0.f, v2 = 0.f, v3 = 0.f;
            if (i4 < n4) {
                const float4 w = ops.w4(wv, u, i4);
                v0 = __fmul_rn(w.x, __fmul_rn(ss, xv[u].x)); v1 = __fmul_rn(w.y, __fmul_rn(ss, xv[u].y));
                v2 = __fmul_rn(w.z, __fmul_rn(ss, xv[u].z)); v3 = __fmul_rn(w.w, __fmul_rn(ss, xv[u].w));
            }
            float amax = fmaxf(fmaxf(fabsf(v0), fabsf(v1)), fmaxf(fabsf(v2), fabsf(v3)));
            amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
            amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
            amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 4));
            const float qs = __fdiv_rn(amax, 127.0f);
            const float ascale = __half2float(__float2half_rn(qs));
            const float ainv = qs != 0.0f ? __fdiv_rn(1.0f, qs) : 0.0f;
            const float s0 = __fmul_rn(v0, ainv), s1 = __fmul_rn(v1, ainv), s2 = __fmul_rn(v2, ainv), s3 = __fmul_rn(v3, ainv);
            const int q0 = __float2int_rz(__fadd_rn(s0, copysignf(0.5f, s0))), q1 = __float2int_rz(__fadd_rn(s1, copysignf(0.5f, s1)));
            const int q2 = __float2int_rz(__fadd_rn(s2, copysignf(0.5f, s2))), q3 = __float2int_rz(__fadd_rn(s3, copysignf(0.5f, s3)));
            if (i4 < n4) {
                sxq[i4] = (unsigned)(q0 & 0xff) | ((unsigned)(q1 & 0xff) << 8) | ((unsigned)(q2 & 0xff) << 16) | ((unsigned)(q3 & 0xff) << 24);
                if ((tid & 7) == 0) sxs[i4 >> 3] = ascale;
            }
        }
    }
    ops.sync();
}
