/* proto.c -- CPU model of the exact RMSNorm accumulator (csrc/seqsum2.cuh), checked against the literal loop.
 *
 * Goal: the bit-exact value of   s = 0; for (i) s = s + t[i];   (float32, round-to-nearest-even, t[i] >= 0)
 * -- InferenceCore.rmsnorm's accumulator (InferenceCore.java:39-48) -- with O(log n) parallel depth plus a
 * short serial walk (csrc/seqsum2.cuh implements it).
 *
 * Model of the CUDA kernel (T threads, E consecutive terms per thread), every step written as the loop the
 * threads would execute in parallel:
 *   1. P[j] = approximate sum of all terms before thread j (a parallel float prefix; any summation order).
 *   2. thread j is CLEAN in binade e when P[j] and P[j+1] both lie well inside [2^e, 2^(e+1)) and every term is
 *      below 2^(e+1); it then composes its E steps  M -> M + a[M & 1]  (integer mantissa steps, the pair captures
 *      round-half-even ties) into one pair.  Otherwise the thread is LITERAL.
 *   3. maximal runs of clean threads with equal e are composed by a segmented scan (associative).
 *   4. one thread walks the items in order: literal threads are E real float adds; a run is applied to the exact
 *      state after VERIFYING its premise (exponent of s == e before, mantissa < 2^24 after); a failed check
 *      falls back to the literal loop over that run.  The prediction only decides speed, never the result.
 * Build:  gcc -O2 -ffp-contract=off -o proto proto.c -lm      Run: ./proto [n] [T] [cases]
 */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

typedef struct { uint32_t a0, a1; } Pair;
static uint32_t fbits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static float bitsf(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static int fexp(float f) { return (int)((fbits(f) >> 23) & 0xff) - 127; }

static Pair compose(Pair L, Pair R) { /* apply L, then R */
    Pair o;
    o.a0 = L.a0 + ((L.a0 & 1u) ? R.a1 : R.a0);
    o.a1 = L.a1 + (((1u + L.a1) & 1u) ? R.a1 : R.a0);
    if (o.a0 > (1u << 26)) o.a0 = 1u << 26; /* saturate: >= 2^24 fails verification anyway */
    if (o.a1 > (1u << 26)) o.a1 = 1u << 26;
    return o;
}
/* pair of adding t to a sum in binade e; 0 when t >= 2^(e+1) */
static int seq_pair(float t, int e, Pair *pr) {
    uint32_t tb = fbits(t);
    int et = (int)(tb >> 23);
    pr->a0 = pr->a1 = 0;
    if (et == 0) return 1;
    uint32_t m = (tb & 0x7fffffu) | 0x800000u;
    int shift = (e + 127) - et;
    if (shift < 0) return 0;
    if (shift > 25) shift = 25;
    uint32_t k = m >> shift, rem = m & ((1u << shift) - 1u), half = shift ? (1u << (shift - 1)) : 0u;
    if (shift && rem == half) { pr->a0 = k + (k & 1u); pr->a1 = k + ((k + 1u) & 1u); }
    else pr->a0 = pr->a1 = k + ((shift && rem > half) ? 1u : 0u);
    return 1;
}

static long g_items, g_literal_items, g_fallbacks, g_head;

static float seqsum_v2(const float *t, int n, int T) {
    const int E = (n + T - 1) / T;
    float *P = malloc(sizeof(float) * (T + 1));
    int *cls = malloc(sizeof(int) * T);      /* binade of a clean thread, or INT32_MIN for literal */
    Pair *pr = malloc(sizeof(Pair) * T);
    /* 1. float prefix over per-thread sums (tree order inside a thread does not matter for the prediction) */
    P[0] = 0.f;
    for (int j = 0; j < T; j++) {
        float loc = 0.f;
        for (int k = 0; k < E; k++) { int i = j * E + k; if (i < n) loc += t[i]; }
        P[j + 1] = P[j] + loc;
    }
    /* 2. classify + thread-local composition */
    for (int j = 0; j < T; j++) {
        cls[j] = INT32_MIN;
        const float lo = P[j], hi = P[j + 1];
        if (!(lo > 0.f) || fexp(lo) != fexp(hi) || fexp(lo) < -100 || fexp(lo) >= 128) continue; /* inf/nan prefix: literal adds */
        const int e = fexp(lo);
        const float b = ldexpf(1.0f, e);
        /* margin 2^-9: the sequential sum deviates from the exact prefix by < n * 2^-24 relative (n <= 8192 -> 2^-11) */
#ifndef NO_MARGIN /* -DNO_MARGIN exercises the resolver's verification + fallback */
        if (lo < b * (1.0f + 0x1p-9f) || hi > 2.0f * b * (1.0f - 0x1p-9f)) continue;
#endif
        Pair acc = {0, 0};
        int ok = 1;
        for (int k = 0; k < E && ok; k++) {
            int i = j * E + k;
            if (i >= n) break;
            Pair p;
            ok = seq_pair(t[i], e, &p);
            if (ok) acc = compose(acc, p);
        }
        if (!ok) continue;
        cls[j] = e;
        pr[j] = acc;
    }
    /* 3. segmented inclusive scan: run = consecutive clean threads with equal binade */
    Pair *run = malloc(sizeof(Pair) * T);
    int *run_start = malloc(sizeof(int) * T);
    for (int j = 0; j < T; j++) {
        if (cls[j] == INT32_MIN) continue;
        if (j > 0 && cls[j - 1] == cls[j]) { run[j] = compose(run[j - 1], pr[j]); run_start[j] = run_start[j - 1]; }
        else { run[j] = pr[j]; run_start[j] = j; }
    }
    /* 4. resolver */
    float s = 0.f;
    int j = 0;
    /* tight literal head: everything before the first clean thread */
    while (j < T && cls[j] == INT32_MIN) { for (int k = 0; k < E; k++) { int i = j * E + k; if (i < n) s = s + t[i]; } j++; g_head++; }
    while (j < T) {
        g_items++;
        if (cls[j] == INT32_MIN) {
            for (int k = 0; k < E; k++) { int i = j * E + k; if (i < n) s = s + t[i]; }
            g_literal_items++;
            j++;
            continue;
        }
        int last = j;
        while (last + 1 < T && cls[last + 1] == cls[j]) last++;
        const int e = cls[j];
        const uint32_t sb = fbits(s);
        int ok = fexp(s) == e && (sb >> 23) != 0;
        if (ok) {
            const uint32_t M = (sb & 0x7fffffu) | 0x800000u;
            const uint32_t M2 = M + ((M & 1u) ? run[last].a1 : run[last].a0);
            if (M2 < (1u << 24)) s = bitsf(((uint32_t)(e + 127) << 23) | (M2 & 0x7fffffu));
            else ok = 0;
        }
        if (!ok) { /* misprediction: literal over the run */
            g_fallbacks++;
            for (int q = j; q <= last; q++) for (int k = 0; k < E; k++) { int i = q * E + k; if (i < n) s = s + t[i]; }
        }
        j = last + 1;
    }
    free(P); free(cls); free(pr); free(run); free(run_start);
    return s;
}

static float literal(const float *t, int n) { float s = 0.f; for (int i = 0; i < n; i++) s = s + t[i]; return s; }

static uint64_t rng = 88172645463325252ull;
static uint32_t xr(void) { rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17; return (uint32_t)(rng >> 16); }
static float urand(void) { return (xr() & 0xffffff) / 16777216.0f; }
static float nrand(void) { float u = urand() + 1e-7f, v = urand(); return sqrtf(-2.f * logf(u)) * cosf(6.2831853f * v); }

int main(int argc, char **argv) {
    int n = argc > 1 ? atoi(argv[1]) : 4096, T = argc > 2 ? atoi(argv[2]) : 1024, cases = argc > 3 ? atoi(argv[3]) : 20000;
    float *t = malloc(sizeof(float) * n);
    long bad = 0;
    for (int c = 0; c < cases; c++) {
        const int kind = c % 10;
        for (int i = 0; i < n; i++) {
            float x;
            switch (kind) {
            case 0: x = nrand(); break;                                         /* activations ~ N(0,1) */
            case 1: x = nrand() * 0.02f; break;
            case 2: x = nrand() * (i % 97 == 0 ? 30.f : 1.f); break;            /* outlier channels */
            case 3: x = ldexpf(1.0f, (int)(xr() % 12) - 6); break;              /* powers of two: ties everywhere */
            case 4: x = (float)(xr() % 8) * 0.25f; break;                       /* small dyadic values: many ties, zeros */
            case 5: x = (i < n / 2) ? 1e-3f * urand() : 50.f * urand(); break;   /* late jump over many binades */
            case 6: x = (xr() % 50 == 0) ? nrand() * 100.f : 0.f; break;         /* sparse */
            case 7: x = sqrtf(ldexpf(1.0f + urand() * 1e-3f, (int)(xr() % 3))); break; /* sum hugs powers of two */
            case 8: x = nrand() * expf(nrand()); break;                         /* heavy tailed */
            default: x = (c & 16) ? 1.0f : 0.5f; break;                         /* constant: exact boundary hits */
            }
            t[i] = x * x;
        }
        float a = seqsum_v2(t, n, T), b = literal(t, n);
        if (fbits(a) != fbits(b)) { if (bad < 5) printf("MISMATCH case %d kind %d: v2 %.9g literal %.9g\n", c, kind, a, b); bad++; }
    }
    printf("n=%d T=%d cases=%d mismatches=%ld | per case: head threads %.1f, items %.1f (literal %.1f), fallbacks %.3f\n", n, T, cases, bad,
           (double)g_head / cases, (double)g_items / cases, (double)g_literal_items / cases, (double)g_fallbacks / cases);
    return bad != 0;
}
