/*
 * oracle.c -- CPU restatement of GPULlama3.java's onGPU=false forward pass.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under gpullama3.java_b200/ may link,
 * import or call this file; only tests/, __graft_entry__.smoke() and the
 * cpu_baseline / --impl reference legs of bench.py use it, as the checker /
 * reported CPU baseline.
 *
 * PARITY UNPINNED: the reference ships no golden vectors or known-answer
 * tests for this path (its only unit test is ToolCallParserUtilsTest) and it
 * cannot be executed here (needs JDK 21 + TornadoVM, neither present).  This
 * file is a line-by-line restatement; every function cites the reference
 * file:line it follows (paths relative to
 * src/main/java/org/beehive/gpullama3/ of the reference).
 * What third parties pin instead (everything but the float summation order):
 * the data formats against gguf-py (tests/test_kquants.py) and the structure
 * of the forward pass against Hugging Face transformers in float64
 * (tests/test_oracle_vs_transformers.py).
 *
 * Build: gcc -O2 -ffp-contract=off -fopenmp -shared -fPIC  (see Makefile)
 *   -ffp-contract=off is REQUIRED: Java never contracts a*b+c into an FMA;
 *   the only fused operations in the reference are the explicit
 *   FloatVector.fma calls in FP16FloatTensor.vectorDot, restated with fmaf().
 *
 * Pinned host-dependent choices (see DESIGN.md "Oracle pins"):
 *   - FP16 vector dot lane count: `lanes` in the model config (16 = 512-bit
 *     species, 8 = 256-bit, 0 = llama.VectorBitSize=0 scalar path).
 *   - FloatVector.reduceLanes(ADD) order: ascending lane order (JDK 21 C2
 *     x86 lowering of AddReductionVF is strictly ordered).
 *   - Math.exp/cos/sin/pow: glibc libm in double (both <1 ulp; the (float)
 *     cast makes a disagreement a ~2^-29 event per call).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define GGML_F32 0
#define GGML_F16 1
#define GGML_Q8_0 8

#define ARCH_LLAMA 0
#define ARCH_QWEN3 1
#define ARCH_PHI3 2 /* forwardJavaPhi3 (InferenceCore.java:699-800): the caller passes wq/wk/wv and w1/w3 as row ranges of the fused
                     * attn_qkv / ffn_up tensors (rows of a matmul are independent dot products: wqkv.matmul + copyTo :718-724 and
                     * wGateUp.matmul + copyChunk :779-781 produce exactly these vectors) */

typedef struct {
    const void *data; /* raw GGUF tensor bytes (block layout for Q8_0) */
    int32_t type;     /* GGML type id */
    int32_t pad;
} otensor;

typedef struct {
    int32_t arch;
    int32_t dim, hidden, n_layers, n_heads, n_kv_heads, head_size, vocab, ctx;
    float eps, theta;
    int32_t lanes;         /* FP16 vector-dot lane count (0 = scalar) */
    int32_t per_row_quant; /* 1: re-quantise the activation inside every row dot, as the
                              reference does (slow, bit-identical); 0: hoist per matmul */
    otensor token_embd, output, output_norm;
    otensor *attn_norm, *wq, *wk, *wv, *wo, *ffn_norm, *w1, *w2, *w3;
    otensor *attn_q_norm, *attn_k_norm; /* qwen3 only */
} omodel;

typedef struct {
    float *x, *xb, *xb2, *q, *k, *v, *hb, *hb2, *att, *logits;
    float *xo;                      /* the attention output of the last layer, before wo ([n_heads * head_size]) */
    float *key_cache, *value_cache; /* [L][ctx][kvDim] */
    float *rope_cr, *rope_ci;       /* [ctx][head/2] */
    int8_t *aq;                     /* hoisted activation quants */
    float *ascale;
} ostate;

/* ---- Float.float16ToFloat (IEEE, subnormals kept) : Q8_0FloatTensor.java:61, FP16FloatTensor.java:50 */
static inline float f16_to_f32(uint16_t h) {
    uint32_t sign = (uint32_t)(h & 0x8000) << 16;
    uint32_t exp = (h >> 10) & 0x1F, man = h & 0x3FF, bits;
    if (exp == 0) {
        if (man == 0) bits = sign;
        else { /* subnormal: normalise */
            int e = -1;
            do { e++; man <<= 1; } while ((man & 0x400) == 0);
            man &= 0x3FF;
            bits = sign | ((uint32_t)(127 - 15 - e) << 23) | (man << 13);
        }
    } else if (exp == 31) bits = sign | 0x7F800000u | (man << 13);
    else bits = sign | ((exp + 112) << 23) | (man << 13);
    float f; memcpy(&f, &bits, 4); return f;
}

/* ---- FP16FloatTensor.vectorDot bit trick (FP16FloatTensor.java:88-98): DAZ, no inf/nan */
static inline float f16_to_f32_daz(uint16_t h) {
    uint32_t b = h;
    uint32_t mask = (b & 0x7C00) ? 0xFFFFFFFFu : 0u; /* (-exp) >> 31 */
    uint32_t bits = ((b & 0x8000) << 16) | ((((b & 0x7FFF) + 0x1C000) << 13) & mask);
    float f; memcpy(&f, &bits, 4); return f;
}

/* ---- Float.floatToFloat16 (round-to-nearest-even) : Q8_0FloatTensor.java:109 */
static inline uint16_t f32_to_f16(float f) {
    uint32_t x; memcpy(&x, &f, 4);
    uint32_t sign = (x >> 16) & 0x8000;
    uint32_t ax = x & 0x7FFFFFFF;
    if (ax >= 0x7F800000) return (uint16_t)(sign | 0x7C00 | ((ax > 0x7F800000) ? 0x200 | ((ax >> 13) & 0x3FF) : 0));
    if (ax >= 0x477FF000) return (uint16_t)(sign | 0x7C00); /* rounds to >= 65520 -> inf */
    if (ax < 0x33000001) return (uint16_t)sign;             /* < 2^-25 (or ==2^-25 tie->even 0) */
    int32_t e = (int32_t)(ax >> 23) - 127;
    uint32_t m = (ax & 0x7FFFFF) | 0x800000;
    int shift;
    uint32_t base;
    if (e < -14) { shift = 13 + (-14 - e); base = 0; }      /* subnormal half */
    else { shift = 13; base = (uint32_t)(e + 15) << 10; m &= 0x7FFFFF; }
    uint32_t r = m >> shift;
    uint32_t rem = m & ((1u << shift) - 1), half = 1u << (shift - 1);
    if (rem > half || (rem == half && (r & 1))) r++;
    return (uint16_t)(sign | (base + r)); /* mantissa carry bumps the exponent correctly */
}

uint16_t oracle_f32_to_f16(float f) { return f32_to_f16(f); }
float oracle_f16_to_f32(uint16_t h) { return f16_to_f32(h); }
float oracle_f16_to_f32_daz(uint16_t h) { return f16_to_f32_daz(h); }

/* ---- FloatTensor.getFloat per type */
static inline float t_get(const otensor *t, int64_t i) {
    if (t->type == GGML_F32) return ((const float *)t->data)[i];
    if (t->type == GGML_F16) return f16_to_f32(((const uint16_t *)t->data)[i]);
    /* Q8_0FloatTensor.getFloat, Q8_0FloatTensor.java:55-63 */
    const uint8_t *blk = (const uint8_t *)t->data + (i / 32) * 34;
    uint16_t s; memcpy(&s, blk, 2);
    return (float)((const int8_t *)blk)[2 + (i % 32)] * f16_to_f32(s);
}

/* ---- activation quantisation of one 32-block : Q8_0FloatTensor.java:100-117 */
static inline float q8_quant_block(const float *x, int8_t *aq) {
    float amax = 0.0f;
    for (int i = 0; i < 32; i++) { float av = fabsf(x[i]); if (av > amax) amax = av; }
    float qs = amax / 127.0f;
    float ascale = f16_to_f32(f32_to_f16(qs));
    float ainv = qs != 0.0f ? 1.0f / qs : 0.0f;
    for (int i = 0; i < 32; i++) {
        float s = x[i] * ainv;
        aq[i] = (int8_t)(int)(s + copysignf(0.5f, s)); /* (int) truncates toward zero */
    }
    return ascale;
}

void oracle_q8_quantize(const float *x, int n, int8_t *aq, float *ascale) {
    for (int b = 0; b < n / 32; b++) ascale[b] = q8_quant_block(x + b * 32, aq + b * 32);
}

/* ---- Q8_0FloatTensor.dotQ8Activation, Q8_0FloatTensor.java:90-123 (faithful: quantises per call) */
float oracle_q8_dot_ref(const void *w, int64_t woff, const float *x, int n) {
    float result = 0.0f;
    int8_t aq[32];
    for (int b = 0; b < n / 32; b++) {
        const uint8_t *blk = (const uint8_t *)w + ((woff + b * 32) / 32) * 34;
        uint16_t s; memcpy(&s, blk, 2);
        float ws = f16_to_f32(s);
        float as = q8_quant_block(x + b * 32, aq);
        int isum = 0;
        for (int i = 0; i < 32; i++) isum += (int)aq[i] * (int)((const int8_t *)blk)[2 + i];
        result += (float)isum * (ws * as);
    }
    return result;
}

/* same arithmetic with the (row-independent) activation quantisation hoisted */
static float q8_dot_hoisted(const void *w, int64_t woff, const int8_t *aq, const float *ascale, int n) {
    float result = 0.0f;
    for (int b = 0; b < n / 32; b++) {
        const uint8_t *blk = (const uint8_t *)w + ((woff + b * 32) / 32) * 34;
        uint16_t s; memcpy(&s, blk, 2);
        float ws = f16_to_f32(s);
        const int8_t *wq = (const int8_t *)blk + 2;
        int isum = 0;
        for (int i = 0; i < 32; i++) isum += (int)aq[b * 32 + i] * (int)wq[i];
        result += (float)isum * (ws * ascale[b]);
    }
    return result;
}

/* ---- FloatTensor.scalarDot, FloatTensor.java:86-92 */
static float scalar_dot_t(const otensor *t, int64_t off, const float *x, int n) {
    float r = 0.0f;
    for (int j = 0; j < n; j++) r += t_get(t, off + j) * x[j];
    return r;
}
static inline float scalar_dot_ff(const float *a, const float *b, int n) {
    float r = 0.0f;
    for (int j = 0; j < n; j++) r += a[j] * b[j];
    return r;
}

/* ---- FP16FloatTensor.vectorDot, FP16FloatTensor.java:62-110 with `lanes`-wide species */
float oracle_f16_dot(const uint16_t *w, const float *x, int n, int lanes) {
    if (lanes <= 0) { /* USE_VECTOR_API == false -> scalarDot with IEEE getFloat */
        float r = 0.0f;
        for (int j = 0; j < n; j++) r += f16_to_f32(w[j]) * x[j];
        return r;
    }
    float acc[64];
    for (int l = 0; l < lanes; l++) acc[l] = 0.0f;
    int upper = n - (n % lanes); /* F_SPECIES.loopBound(size) */
    for (int i = 0; i < upper; i += lanes)
        for (int l = 0; l < lanes; l++) acc[l] = fmaf(f16_to_f32_daz(w[i + l]), x[i + l], acc[l]);
    float result = 0.0f; /* reduceLanes(ADD): ordered, identity first */
    for (int l = 0; l < lanes; l++) result += acc[l];
    for (int j = upper; j < n; j++) result += f16_to_f32(w[j]) * x[j]; /* scalar tail, :104-106 */
    return result;
}

/* ---- FloatTensor.matmul, FloatTensor.java:98-100 (rows in parallel; each row independent) */
static void matmul(const omodel *m, ostate *s, const otensor *w, const float *x, float *out, int d0, int d1) {
    if (w->type == GGML_Q8_0) {
        if (m->per_row_quant) {
#pragma omp parallel for schedule(static)
            for (int i = 0; i < d0; i++) out[i] = oracle_q8_dot_ref(w->data, (int64_t)i * d1, x, d1);
        } else {
            oracle_q8_quantize(x, d1, s->aq, s->ascale);
#pragma omp parallel for schedule(static)
            for (int i = 0; i < d0; i++) out[i] = q8_dot_hoisted(w->data, (int64_t)i * d1, s->aq, s->ascale, d1);
        }
    } else if (w->type == GGML_F16) {
#pragma omp parallel for schedule(static)
        for (int i = 0; i < d0; i++) out[i] = oracle_f16_dot((const uint16_t *)w->data + (int64_t)i * d1, x, d1, m->lanes);
    } else {
#pragma omp parallel for schedule(static)
        for (int i = 0; i < d0; i++) out[i] = scalar_dot_t(w, (int64_t)i * d1, x, d1);
    }
}
void oracle_matmul(const omodel *m, ostate *s, const otensor *w, const float *x, float *out, int d0, int d1) {
    matmul(m, s, w, x, out, d0, d1);
}

/* ---- InferenceCore.rmsnorm, InferenceCore.java:39-48 (out may alias x) */
void oracle_rmsnorm(float *out, const float *x, const otensor *w, int size, float eps) {
    float ss = 0.0f;
    for (int i = 0; i < size; i++) ss = ss + x[i] * x[i];
    ss /= (float)size;
    ss += eps;
    ss = (float)(1.0 / sqrt((double)ss));
    for (int i = 0; i < size; i++) out[i] = t_get(w, i) * (ss * x[i]);
}

/* ---- RoPE.precomputeFreqsCis, RoPE.java:6-37 with ropeScaling=false (LlamaModelLoader.java:68) */
void oracle_rope_table(int ctx, int head_size, double theta, float *cr, float *ci) {
    int n = 0;
    for (int pos = 0; pos < ctx; pos++)
        for (int i = 0; i < head_size; i += 2) {
            float freq = (float)(1.0 / pow(theta, i / (double)head_size));
            float val = (float)pos * freq;
            cr[n] = (float)cos((double)val);
            ci[n] = (float)sin((double)val);
            n++;
        }
}

/* ---- FloatTensor.softmaxInPlace, FloatTensor.java:211-219 */
static void softmax(float *a, int n) {
    float mx = -INFINITY;
    for (int i = 0; i < n; i++) mx = fmaxf(mx, a[i]); /* Float.max; no NaNs on this path */
    for (int i = 0; i < n; i++) a[i] = (float)exp((double)(a[i] - mx));
    float sum = 0.0f;
    for (int i = 0; i < n; i++) sum += a[i];
    for (int i = 0; i < n; i++) a[i] = a[i] / sum;
}

/* ---- (float)Math.exp(double) over n floats: the softmax's exp (and, at -g, the shared-expert gate's), for restatements of it */
void oracle_exp_narrow(const float *x, float *y, int64_t n) {
    for (int64_t i = 0; i < n; i++) y[i] = (float)exp((double)x[i]);
}

/* Checks a device's evaluation of the exp expressions of the bit-exact paths against this library's exp: for the float x with
 * bit pattern first + i, e[i] must equal (float)exp((double)x) (softmaxes, routers, shared-expert gate) and e1[i]
 * (float)(1.0 + exp((double)x)) (the SwiGLU denominator), bit for bit.  Returns the number of inputs where either differs; the
 * lowest max_report of them go to bad (bit patterns, ascending). */
int64_t oracle_exp_sweep(uint32_t first, int64_t n, const float *e, const float *e1, uint32_t *bad, int32_t max_report) {
    int64_t count = 0;
    int32_t nbad = 0;
#pragma omp parallel for schedule(static, 65536) reduction(+ : count)
    for (int64_t i = 0; i < n; i++) {
        const uint32_t b = first + (uint32_t)i;
        float x, r, r1;
        memcpy(&x, &b, 4);
        const double d = exp((double)x);
        r = (float)d;
        r1 = (float)(1.0 + d);
        if (memcmp(&r, e + i, 4) == 0 && memcmp(&r1, e1 + i, 4) == 0) continue;
        count++;
#pragma omp critical(oracle_exp_sweep)
        { /* keep the lowest max_report patterns, sorted */
            int k = nbad < max_report ? nbad++ : max_report;
            if (k == max_report && (max_report == 0 || b > bad[max_report - 1])) k = -1;
            else if (k == max_report) k = max_report - 1;
            if (k >= 0) {
                while (k > 0 && bad[k - 1] > b) { bad[k] = bad[k - 1]; k--; }
                bad[k] = b;
            }
        }
    }
    return count;
}

/* ---- FloatTensor.argmax, FloatTensor.java:138-151 (first strict maximum) */
int oracle_argmax(const float *v, int n) {
    int mi = 0; float mv = v[0];
    for (int i = 0; i < n; i++) if (v[i] > mv) { mv = v[i]; mi = i; }
    return mi;
}

static inline int q_dim(const omodel *m) { return m->n_heads * m->head_size; }
static inline int kv_dim(const omodel *m) { return m->n_kv_heads * m->head_size; }

ostate *oracle_state_new(const omodel *m) {
    ostate *s = (ostate *)calloc(1, sizeof(ostate));
    int qd = q_dim(m), kvd = kv_dim(m);
    int big = m->dim > m->hidden ? m->dim : m->hidden;
    if (qd > big) big = qd;
    s->x = calloc(m->dim, 4); s->xb = calloc(big, 4); s->xb2 = calloc(m->dim, 4);
    s->q = calloc(qd > m->dim ? qd : m->dim, 4); s->k = calloc(m->dim > kvd ? m->dim : kvd, 4);
    s->v = calloc(m->dim > kvd ? m->dim : kvd, 4);
    s->hb = calloc(m->hidden, 4); s->hb2 = calloc(m->hidden, 4);
    s->att = calloc((size_t)m->n_heads * m->ctx, 4); s->logits = calloc(m->vocab, 4); s->xo = calloc(qd, 4);
    s->key_cache = calloc((size_t)m->n_layers * m->ctx * kvd, 4);   /* Java arrays are zero-filled */
    s->value_cache = calloc((size_t)m->n_layers * m->ctx * kvd, 4);
    s->rope_cr = malloc((size_t)m->ctx * (m->head_size / 2) * 4);
    s->rope_ci = malloc((size_t)m->ctx * (m->head_size / 2) * 4);
    oracle_rope_table(m->ctx, m->head_size, (double)m->theta, s->rope_cr, s->rope_ci);
    s->aq = malloc(big); s->ascale = malloc((big / 32 + 1) * 4);
    return s;
}
void oracle_state_free(ostate *s) {
    free(s->x); free(s->xb); free(s->xb2); free(s->q); free(s->k); free(s->v); free(s->hb); free(s->hb2);
    free(s->att); free(s->logits); free(s->xo); free(s->key_cache); free(s->value_cache); free(s->rope_cr); free(s->rope_ci);
    free(s->aq); free(s->ascale); free(s);
}
void oracle_state_reset(const omodel *m, ostate *s) {
    size_t n = (size_t)m->n_layers * m->ctx * kv_dim(m) * 4;
    memset(s->key_cache, 0, n); memset(s->value_cache, 0, n);
}
float *oracle_state_logits(ostate *s) { return s->logits; }
float *oracle_state_x(ostate *s) { return s->x; }
float *oracle_state_key_cache(ostate *s) { return s->key_cache; }
float *oracle_state_value_cache(ostate *s) { return s->value_cache; }
/* read-only views of the last layer's intermediates after a forward: the softmax weights ([n_heads][ctx], entries 0..pos of each
 * head), the SwiGLU output that w2 multiplies ([hidden]), the rotated q ([n_heads * head_size]) and the attention output that wo
 * multiplies ([n_heads * head_size]) */
float *oracle_state_att(ostate *s) { return s->att; }
float *oracle_state_hb(ostate *s) { return s->hb; }
float *oracle_state_q(ostate *s) { return s->q; }
float *oracle_state_att_out(ostate *s) { return s->xo; }

/*
 * InferenceCore.forwardJava (InferenceCore.java:50-172) and
 * InferenceCore.forwardJavaQwen3 (InferenceCore.java:565-697).
 * `want_logits` = 0 stops after the last layer (prefill: logits are never computed,
 * InferenceCoreBatchPrefillDecode.java:166-167; the KV cache is identical).
 */
float *oracle_forward(const omodel *m, ostate *s, int token, int pos, int want_logits) {
    const int dim = m->dim, hs = m->head_size, qd = q_dim(m), kvd = kv_dim(m);
    const int kv_mul = m->n_heads / m->n_kv_heads;
    const float sqrt_hs = (float)sqrt((double)hs);
    const int half = hs / 2;

    /* token_embedding_table.copyTo(token*dim, x, 0, dim) : InferenceCore.java:61 */
    for (int i = 0; i < dim; i++) s->x[i] = t_get(&m->token_embd, (int64_t)token * dim + i);

    for (int l = 0; l < m->n_layers; l++) {
        oracle_rmsnorm(s->xb, s->x, &m->attn_norm[l], dim, m->eps);
        matmul(m, s, &m->wq[l], s->xb, s->q, qd, dim);
        matmul(m, s, &m->wk[l], s->xb, s->k, kvd, dim);
        matmul(m, s, &m->wv[l], s->xb, s->v, kvd, dim);

        if (m->arch == ARCH_QWEN3) {
            /* per-head RMSNorm of q and k : InferenceCore.java:594-600 */
            for (int h = 0; h < m->n_heads; h++) oracle_rmsnorm(s->q + h * hs, s->q + h * hs, &m->attn_q_norm[l], hs, m->eps);
            for (int h = 0; h < m->n_kv_heads; h++) oracle_rmsnorm(s->k + h * hs, s->k + h * hs, &m->attn_k_norm[l], hs, m->eps);
            /* NeoX RoPE, pairs (ic, ic+half) : InferenceCore.java:604-619 */
            for (int h = 0; h < m->n_heads; h++) {
                int rotn = h < m->n_kv_heads ? 2 : 1;
                for (int ic = 0; ic < half; ic++) {
                    float fcr = s->rope_cr[pos * half + ic], fci = s->rope_ci[pos * half + ic];
                    for (int vi = 0; vi < rotn; vi++) {
                        float *vec = vi == 0 ? s->q : s->k;
                        float v0 = vec[h * hs + ic], v1 = vec[h * hs + ic + half];
                        vec[h * hs + ic] = v0 * fcr - v1 * fci;
                        vec[h * hs + ic + half] = v0 * fci + v1 * fcr;
                    }
                }
            }
        } else if (m->arch == ARCH_PHI3) {
            /* InferenceCore.java:726-742: pairs (ic, ic + headSize/2) with ic = head base + head_dim/2, no q/k norm */
            for (int i = 0; i < dim; i += 2) {
                int head_dim = i % hs, base = i - head_dim, ic = base + head_dim / 2;
                float fcr = s->rope_cr[pos * half + head_dim / 2], fci = s->rope_ci[pos * half + head_dim / 2];
                int rotn = i < kvd ? 2 : 1;
                for (int v = 0; v < rotn; v++) {
                    float *vec = v == 0 ? s->q : s->k;
                    float v0 = vec[ic], v1 = vec[ic + half];
                    vec[ic] = v0 * fcr - v1 * fci;
                    vec[ic + half] = v0 * fci + v1 * fcr;
                }
            }
        } else {
            /* interleaved-pair RoPE : InferenceCore.java:75-87 */
            for (int i = 0; i < dim; i += 2) {
                int hd = i % hs;
                float fcr = s->rope_cr[pos * half + hd / 2], fci = s->rope_ci[pos * half + hd / 2];
                int rotn = i < kvd ? 2 : 1;
                for (int v = 0; v < rotn; v++) {
                    float *vec = v == 0 ? s->q : s->k;
                    float v0 = vec[i], v1 = vec[i + 1];
                    vec[i] = v0 * fcr - v1 * fci;
                    vec[i + 1] = v0 * fci + v1 * fcr;
                }
            }
        }

        /* KV write : InferenceCore.java:92-93 */
        float *kc = s->key_cache + (size_t)l * m->ctx * kvd, *vc = s->value_cache + (size_t)l * m->ctx * kvd;
        memcpy(kc + (size_t)pos * kvd, s->k, kvd * 4);
        memcpy(vc + (size_t)pos * kvd, s->v, kvd * 4);

        /* attention : InferenceCore.java:98-137 */
#pragma omp parallel for schedule(static)
        for (int h = 0; h < m->n_heads; h++) {
            const float *q = s->q + h * hs;
            float *att = s->att + (size_t)h * m->ctx;
            for (int t = 0; t <= pos; t++) {
                float score = scalar_dot_ff(q, kc + (size_t)t * kvd + (h / kv_mul) * hs, hs);
                score /= sqrt_hs;
                att[t] = score;
            }
            softmax(att, pos + 1);
            float *xb = s->xb + h * hs;
            for (int i = 0; i < hs; i++) xb[i] = 0.0f;
            for (int t = 0; t <= pos; t++) {
                const float *v = vc + (size_t)t * kvd + (h / kv_mul) * hs;
                float a = att[t];
                for (int i = 0; i < hs; i++) xb[i] = a * v[i] + xb[i]; /* saxpyInPlace, FloatTensor.java:221-227 */
            }
        }
        memcpy(s->xo, s->xb, (size_t)qd * 4);

        matmul(m, s, &m->wo[l], s->xb, s->xb2, dim, qd);
        for (int i = 0; i < dim; i++) s->x[i] = s->x[i] + s->xb2[i];

        oracle_rmsnorm(s->xb, s->x, &m->ffn_norm[l], dim, m->eps);
        matmul(m, s, &m->w1[l], s->xb, s->hb, m->hidden, dim);
        matmul(m, s, &m->w3[l], s->xb, s->hb2, m->hidden, dim);
        /* SwiGLU : InferenceCore.java:150-158 */
        for (int i = 0; i < m->hidden; i++) {
            float v = s->hb[i];
            v = v / (float)(1.0 + exp((double)(-v)));
            s->hb[i] = v * s->hb2[i];
        }
        matmul(m, s, &m->w2[l], s->hb, s->xb, dim, m->hidden);
        for (int i = 0; i < dim; i++) s->x[i] = s->x[i] + s->xb[i];
    }
    if (!want_logits) return NULL;
    oracle_rmsnorm(s->x, s->x, &m->output_norm, dim, m->eps);
    matmul(m, s, m->output.data ? &m->output : &m->token_embd, s->x, s->logits, m->vocab, dim);
    return s->logits;
}

/* ---- java.util.Random (48-bit LCG) as used by LlamaBench.java:188-193 */
typedef struct { uint64_t seed; } jrandom;
void jrandom_init(jrandom *r, int64_t seed) { r->seed = ((uint64_t)seed ^ 0x5DEECE66DULL) & ((1ULL << 48) - 1); }
static int32_t jnext(jrandom *r, int bits) {
    r->seed = (r->seed * 0x5DEECE66DULL + 0xBULL) & ((1ULL << 48) - 1);
    return (int32_t)((int64_t)r->seed >> (48 - bits));
}
int32_t jrandom_next_int(jrandom *r) { return jnext(r, 32); }
int32_t jrandom_next_int_bound(jrandom *r, int32_t bound) {
    int32_t rr = jnext(r, 31);
    int32_t m = bound - 1;
    if ((bound & m) == 0) return (int32_t)(((int64_t)bound * (int64_t)rr) >> 31);
    for (int32_t u = rr; (int32_t)((uint32_t)u - (uint32_t)(rr = u % bound) + (uint32_t)m) < 0; u = jnext(r, 31)) {}
    return rr;
}
void oracle_bench_tokens(int64_t seed, int32_t vocab, int32_t n, int32_t *out) {
    jrandom r; jrandom_init(&r, seed);
    for (int i = 0; i < n; i++) out[i] = jrandom_next_int_bound(&r, vocab);
}

/* ---- ggml-style Q8_0 quantiser used to synthesise weights (amax/127, roundf, f16 scale) */
void oracle_quantize_q8_0(const float *x, int64_t n, uint8_t *out) {
#pragma omp parallel for schedule(static)
    for (int64_t b = 0; b < n / 32; b++) {
        const float *xb = x + b * 32;
        float amax = 0.0f;
        for (int i = 0; i < 32; i++) { float a = fabsf(xb[i]); if (a > amax) amax = a; }
        float d = amax / 127.0f, id = d != 0.0f ? 1.0f / d : 0.0f;
        uint16_t h = f32_to_f16(d);
        memcpy(out + b * 34, &h, 2);
        for (int i = 0; i < 32; i++) ((int8_t *)out)[b * 34 + 2 + i] = (int8_t)roundf(xb[i] * id);
    }
}

/* ================================================================================================================
 * K-quants (SURVEY 8f N4): the reference's accelerator path never computes with Q4_K/Q5_K/Q6_K -- ModelLoader.loadTornadoTensor
 * (model/loader/ModelLoader.java:163) re-quantises such tensors to Q8_0 at load time (dequantizeToQ8_0TornadoTensor, :173-224) and
 * AbstractModelLoader.java:45-59 reports the model as Q8_0.  Restated here: the element read of each format (getFloat of
 * tensor/standard/Q4_KFloatTensor.java:90-120, Q5_KFloatTensor.java:84-122, Q6_KFloatTensor.java:64-116; float products evaluated left
 * to right, no contraction) and the re-quantiser (per 32 elements: maxAbs, scale = maxAbs / 127f stored as Float.floatToFloat16,
 * q = clamp(Math.round(x * (1f / scale)), -128, 127) with Math.round = floor(x + 1/2) computed exactly).  The element reads are
 * pinned against the gguf-py package (llama.cpp's own Python implementation of the formats, tests/test_kquants.py).
 * ================================================================================================================ */
static inline int k4_scale(int j, const uint8_t *sc) { return j < 4 ? (sc[j] & 63) : ((sc[j + 4] & 0xF) | ((sc[j - 4] >> 6) << 4)); }
static inline int k4_min(int j, const uint8_t *sc) { return j < 4 ? (sc[j + 4] & 63) : ((sc[j + 4] >> 4) | ((sc[j] >> 6) << 4)); }
static inline uint16_t rd16(const uint8_t *p) { return (uint16_t)(p[0] | (p[1] << 8)); }

static float q4k_get(const uint8_t *base, int64_t index) {
    const uint8_t *b = base + (index / 256) * 144;
    const int within = (int)(index % 256), pair = within / 64, pos = within % 64;
    const float d = f16_to_f32(rd16(b)), dmin = f16_to_f32(rd16(b + 2));
    int sub, q;
    if (pos < 32) { sub = pair * 2; q = b[16 + pair * 32 + pos] & 0xF; }
    else { sub = pair * 2 + 1; q = (b[16 + pair * 32 + (pos - 32)] >> 4) & 0xF; }
    const int sc = k4_scale(sub, b + 4), m = k4_min(sub, b + 4);
    const float a = d * (float)sc, a2 = a * (float)q, c = dmin * (float)m;
    return a2 - c;
}
static float q5k_get(const uint8_t *base, int64_t index) {
    const uint8_t *b = base + (index / 256) * 176;
    const int within = (int)(index % 256), pair = within / 64, pos = within % 64;
    const float d = f16_to_f32(rd16(b)), dmin = f16_to_f32(rd16(b + 2));
    int sub, q, hi;
    if (pos < 32) { sub = pair * 2; q = b[48 + pair * 32 + pos] & 0xF; hi = (b[16 + pos] >> (pair * 2)) & 1; }
    else { sub = pair * 2 + 1; q = (b[48 + pair * 32 + (pos - 32)] >> 4) & 0xF; hi = (b[16 + (pos - 32)] >> (pair * 2 + 1)) & 1; }
    q += hi * 16;
    const int sc = k4_scale(sub, b + 4), m = k4_min(sub, b + 4);
    const float a = d * (float)sc, a2 = a * (float)q, c = dmin * (float)m;
    return a2 - c;
}
static float q6k_get(const uint8_t *base, int64_t index) {
    const uint8_t *b = base + (index / 256) * 210;
    const int within = (int)(index % 256), half = within / 128, ph = within % 128, grp = ph / 32, pg = ph % 32, is = pg / 16;
    const float d = f16_to_f32(rd16(b + 208));
    const uint8_t *ql = b + half * 64, *qh = b + 128 + half * 32;
    const int8_t *sc = (const int8_t *)(b + 192 + half * 8);
    int qv, s;
    switch (grp) {
    case 0: qv = ((ql[pg] & 0xF) | (((qh[pg] >> 0) & 3) << 4)) - 32; s = sc[is]; break;
    case 1: qv = ((ql[32 + pg] & 0xF) | (((qh[pg] >> 2) & 3) << 4)) - 32; s = sc[is + 2]; break;
    case 2: qv = ((ql[pg] >> 4) | (((qh[pg] >> 4) & 3) << 4)) - 32; s = sc[is + 4]; break;
    default: qv = ((ql[32 + pg] >> 4) | (((qh[pg] >> 6) & 3) << 4)) - 32; s = sc[is + 6]; break;
    }
    const float a = d * (float)s;
    return a * (float)qv;
}
/* ggml type ids: Q4_K = 12, Q5_K = 13, Q6_K = 14 (tensor/GGMLType.java:18-20 in enum order) */
float oracle_kquant_get(int type, const uint8_t *src, int64_t index) {
    return type == 12 ? q4k_get(src, index) : type == 13 ? q5k_get(src, index) : q6k_get(src, index);
}
void oracle_kquant_dequantize(int type, const uint8_t *src, int64_t n, float *out) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; i++) out[i] = oracle_kquant_get(type, src, i);
}
static inline int java_round_f(float a) { /* Math.round(float): floor(a + 1/2), ties towards +infinity, NaN -> 0 */
    if (a != a) return 0;
    const float f = floorf(a);
    return (int)f + ((a - f) >= 0.5f ? 1 : 0);
}
void oracle_kquant_to_q8_0(int type, const uint8_t *src, int64_t n, uint8_t *dst) { /* ModelLoader.java:184-212 */
#pragma omp parallel for schedule(static)
    for (int64_t b = 0; b < (n + 31) / 32; b++) {
        const int64_t start = b * 32, end = start + 32 < n ? start + 32 : n;
        float max_abs = 0.0f;
        for (int64_t i = start; i < end; i++) { const float a = fabsf(oracle_kquant_get(type, src, i)); max_abs = a > max_abs ? a : max_abs; }
        const float scale = max_abs / 127.0f;
        const uint16_t h = f32_to_f16(scale);
        dst[b * 34] = (uint8_t)(h & 0xFF);
        dst[b * 34 + 1] = (uint8_t)(h >> 8);
        const float inv = scale != 0.0f ? 1.0f / scale : 0.0f;
        for (int64_t i = start; i < end; i++) {
            int q = java_round_f(oracle_kquant_get(type, src, i) * inv);
            q = q < -128 ? -128 : (q > 127 ? 127 : q);
            dst[b * 34 + 2 + (i - start)] = (uint8_t)(int8_t)q;
        }
        for (int64_t i = end; i < start + 32; i++) dst[b * 34 + 2 + (i - start)] = 0;
    }
}

/* ================================================================================================================
 * Sampler (SURVEY 8f N3): Sampler.selectSampler (inference/sampler/Sampler.java:74-122), CategoricalSampler.java:28-40,
 * ToppSampler.java:26-156.  Temperature 0 -> FloatTensor.argmax; otherwise logits / temperature, softmaxInPlace, then
 * either the categorical walk or the top-p heap.  PARITY UNPINNED (no JDK here): the uniform numbers come from
 * RandomGeneratorFactory.getDefault() = L32X64MixRandom, restated below from the published LXM algorithm (Steele & Vigna,
 * OOPSLA 2021) and the JDK 17 description of its seeding; its output stream could not be compared with a JVM's.  Everything
 * after the uniform number is plain float arithmetic restated line by line (including the top-p loop's siftDown(..., i - 1)).
 * ================================================================================================================ */
typedef struct { uint32_t a, s, x0, x1; } lxm32;

static inline uint32_t mix_murmur32(uint32_t z) { z = (z ^ (z >> 16)) * 0x85ebca6bu; z = (z ^ (z >> 13)) * 0xc2b2ae35u; return z ^ (z >> 16); }
static inline uint32_t mix_lea32(uint32_t z) { z = (z ^ (z >> 16)) * 0xd36d884bu; z = (z ^ (z >> 16)) * 0xd36d884bu; return z ^ (z >> 16); }
static inline uint32_t rotl32(uint32_t v, int k) { return (v << k) | (v >> (32 - k)); }

/* new L32X64MixRandom(long seed): a = mixMurmur32(high half of seed ^ SILVER_RATIO_64) | 1, s = 1,
 * x0 = mixLea32(low half), x1 = mixLea32(low half + GOLDEN_RATIO_32) */
void oracle_lxm_seed(lxm32 *r, int64_t seed) {
    uint64_t sd = (uint64_t)seed ^ 0x6A09E667F3BCC909ULL;
    r->a = mix_murmur32((uint32_t)(sd >> 32)) | 1u;
    r->s = 1u;
    r->x0 = mix_lea32((uint32_t)sd);
    r->x1 = mix_lea32((uint32_t)sd + 0x9e3779b9u);
    if ((r->x0 | r->x1) == 0u) { r->x0 = 0x9e3779b9u; r->x1 = 0x3c6ef372u; } /* never all-zero xoroshiro state */
}
uint32_t oracle_lxm_next_int(lxm32 *r) {
    const uint32_t z = r->s + r->x0;
    const uint32_t result = mix_lea32(z);
    r->s = 0xadb4a92du * r->s + r->a;                 /* LCG */
    uint32_t q0 = r->x0, q1 = r->x1;                  /* xoroshiro64 */
    q1 ^= q0; q0 = rotl32(q0, 26); q0 = q0 ^ q1 ^ (q1 << 9); q1 = rotl32(q1, 13);
    r->x0 = q0; r->x1 = q1;
    return result;
}
/* RandomGenerator.nextFloat(1f): (nextInt() >>> 8) * 2^-24, times the bound, clamped below the bound */
float oracle_lxm_next_float1(lxm32 *r) {
    float f = (float)(oracle_lxm_next_int(r) >> 8) * 0x1.0p-24f;
    f = f * 1.0f;
    if (f >= 1.0f) f = 0x1.fffffep-1f;
    return f;
}

/* CategoricalSampler.sampleFromFloatTensor (:28-40) on probabilities p[0..n) */
int oracle_sample_categorical(const float *p, int n, float r01) {
    float cdf = 0.0f;
    for (int i = 0; i < n; i++) { cdf += p[i]; if (r01 < cdf) return i; }
    return n - 1;
}

/* Comparator.comparingDouble(logits::getFloat).reversed(): negative when value(a) > value(b) */
static inline int topp_cmp(const float *p, int a, int b) { const double va = p[a], vb = p[b]; return vb < va ? -1 : (vb > va ? 1 : 0); }
static void topp_sift_down(int *arr, int from, int n, const float *p) { /* ToppSampler.siftDown :32-46 */
    int prev = from, next;
    while ((next = 2 * prev + 1) < n) {
        int r = 2 * prev + 2;
        if (r < n && topp_cmp(p, arr[r], arr[next]) < 0) next = r;
        if (topp_cmp(p, arr[next], arr[prev]) < 0) { int t = arr[prev]; arr[prev] = arr[next]; arr[next] = t; prev = next; }
        else break;
    }
}
/* ToppSampler.sampleFromFloatTensor + processTopP (:62-156); indices = scratch of n ints */
int oracle_sample_topp(const float *p, int n, float topp, float r01, int *indices) {
    int head = 0, tail = n - 1;
    const float cutoff = (1.0f - topp) / (float)(n - 1);
    for (int i = 0; i < n; i++) { if (p[i] >= cutoff) indices[head++] = i; else indices[tail--] = i; }
    const int n0 = head;
    for (int i = n0 / 2 - 1; i >= 0; --i) topp_sift_down(indices, i, n0, p);
    float cumulative = 0.0f;
    int last = 0;
    for (int i = n0 - 1; i >= 0; i--) {
        int t = indices[0]; indices[0] = indices[i]; indices[i] = t;
        cumulative += p[indices[i]];
        if (cumulative > topp) { last = i; break; }
        topp_sift_down(indices, 0, i - 1, p); /* i - 1, as in the reference (:131) */
    }
    const float r = r01 * cumulative;
    float cdf = 0.0f;
    for (int i = n0 - 1; i >= last; i--) { cdf += p[indices[i]]; if (r < cdf) return indices[i]; }
    return indices[last];
}

/* Sampler.selectSampler's lambda (:97-118): logits are modified in place exactly as the reference does.
 * r01 = the uniform number the RNG produced for this token (ignored for temperature 0). */
int oracle_sample(float *logits, int n, float temperature, float topp, float r01, int *indices) {
    if (temperature == 0.0f) return oracle_argmax(logits, n);
    for (int i = 0; i < n; i++) logits[i] = logits[i] / temperature; /* divideInPlace, FloatTensor.java:203-205 */
    softmax(logits, n);
    if (topp <= 0.0f || topp >= 1.0f) return oracle_sample_categorical(logits, n, r01);
    return oracle_sample_topp(logits, n, topp, r01, indices);
}

/* torchrun exports OMP_NUM_THREADS=1: the bench's CPU legs set the thread count explicitly (all host cores, like
 * Parallel.parallelFor's ForkJoin common pool, Parallel.java:9-11). */
void oracle_set_threads(int n) {
#ifdef _OPENMP
    extern void omp_set_num_threads(int);
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

int oracle_omp_threads(void) {
#ifdef _OPENMP
    extern int omp_get_max_threads(void);
    return omp_get_max_threads();
#else
    return 1;
#endif
}
