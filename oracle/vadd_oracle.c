/*
 * oracle/vadd_oracle.c -- CPU restatement of the reference's vectorAdd hot path.
 *
 * THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it.  The product
 * (k8s-gpu-hpa_b200/csrc, the vectorAdd CLI) never links, loads or calls anything here.
 *
 * PARITY UNPINNED BY THE REFERENCE.  The reference repository holds no source and no tests
 * for this path: the arithmetic lives in the third-party container image
 *     k8s.gcr.io/cuda-vector-add:v0.1        (cuda-test-deployment.yaml:18)
 * which the reference only *invokes*:
 *     for (( c=1; c<=5000; c++ )); do ./vectorAdd; done   (cuda-test-deployment.yaml:19,
 *                                                          README.md:115)
 * That image is the NVIDIA CUDA Samples 8.0 `0_Simple/vectorAdd` program (SURVEY.md
 * section 8(a), recalled -- not on disk, not fetchable).  What this file restates is
 * its published algorithm:
 *     a2  h_A[i] = rand()/(float)RAND_MAX; h_B[i] = rand()/(float)RAND_MAX  (no srand)
 *     a4  C[i] = A[i] + B[i]          IEEE-754 binary32, round-to-nearest-even
 *     a6  fabs(h_A[i] + h_B[i] - h_C[i]) > 1e-5  -> "Result verification failed"
 * (Its launch shape -- N = 50000, 256 threads, (N+255)/256 blocks, guard i < N -- is
 * corroborated by NVIDIA's int-typed derivatives shipped with this toolkit:
 * /usr/local/cuda/extras/CUPTI/samples/cupti_nvtx/cupti_nvtx.cu:41-53,71,150-153; and the
 * FLOAT recipe itself by another NVIDIA derivative of the same sample on this disk,
 * /usr/local/cuda/extras/CUPTI/samples/cuda_memory_trace/memory_trace.cu:
 *   :23-35    __global__ VectorAdd(const float*, const float*, float*, int N):
 *             i = blockIdx.x * blockDim.x + threadIdx.x; if (i < N) pC[i] = pA[i] + pB[i];
 *   :101-105  pHostA[n] = rand() / (float)RAND_MAX; pHostB[n] = rand() / (float)RAND_MAX;
 *             interleaved per index, and no srand() anywhere in the file
 *   :116-118  dim3 block(256); grid = ceil(nElements / 256).
 * That is NVIDIA's code, not the reference's image: it corroborates a2 and a4 as restated
 * here (tests/test_oracle.py re-reads those lines when the file is present); it does not
 * pin the reference.)
 * Because binary32 RNE addition has exactly one correct result for non-NaN operands,
 * the oracle is pinned by the IEEE-754 standard instead: oracle_softfloat_add_f32()
 * below is an integer-only implementation written from the standard, and
 * tests/test_oracle.py checks the hardware `addss` loop against it and against the
 * known-answer vectors of SURVEY.md section 8(c) (glibc seed-1 rand() stream).
 *
 * Build: see oracle/Makefile (gcc -O2, NO -ffast-math: fast-math links crtfastmath.o
 * which sets FTZ/DAZ and breaks subnormal bit-exactness).
 */
#define _GNU_SOURCE
#include <math.h>
#include <pthread.h>
#include <sched.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <unistd.h>
#if defined(__x86_64__)
#include <immintrin.h>
#endif

/* ------------------------------------------------------------------ a4: the add */

/* Reference kernel body, one element per "thread": C[i] = A[i] + B[i]
 * (CUDA sample vectorAdd.cu kernel; invoked at cuda-test-deployment.yaml:19). */
void oracle_vadd_f32(const float *a, const float *b, float *c, size_t n)
{
    for (size_t i = 0; i < n; ++i)
        c[i] = a[i] + b[i];
}

/* Integer-only IEEE-754 binary32 addition, round-to-nearest-even, no FTZ.
 * Written from the standard (clause 4.3.1 roundTiesToEven, 6.3 sign of zero, 7.2
 * invalid -> quiet NaN); independent of the host FPU.  NaN results are returned as
 * the canonical quiet NaN 0x7fc00000; callers compare NaNs as a class. */
uint32_t oracle_softfloat_add_f32(uint32_t ua, uint32_t ub)
{
    const uint32_t QNAN = 0x7fc00000u;
    uint32_t sa = ua >> 31, sb = ub >> 31;
    int32_t ea = (int32_t)((ua >> 23) & 0xff), eb = (int32_t)((ub >> 23) & 0xff);
    uint32_t ma = ua & 0x7fffffu, mb = ub & 0x7fffffu;

    if (ea == 0xff) {
        if (ma) return QNAN;                               /* NaN + x */
        if (eb == 0xff) {
            if (mb) return QNAN;                           /* Inf + NaN */
            return (sa == sb) ? ua : QNAN;                 /* Inf + Inf / Inf - Inf */
        }
        return ua;                                         /* Inf + finite */
    }
    if (eb == 0xff) return mb ? QNAN : ub;

    /* finite operands: significands with hidden bit, exponent of subnormals = 1 */
    uint64_t xa = ea ? (ma | 0x800000u) : ma;
    uint64_t xb = eb ? (mb | 0x800000u) : mb;
    if (!ea) ea = 1;
    if (!eb) eb = 1;
    if (xa == 0 && xb == 0)
        return (sa & sb) << 31;                            /* +0 unless both -0 (RNE) */

    /* 3 guard bits below the significand + sticky */
    xa <<= 3; xb <<= 3;
    int32_t e;
    if (ea >= eb) {
        int32_t d = ea - eb; e = ea;
        if (d) {
            if (d > 30) xb = (xb != 0);
            else xb = (xb >> d) | ((xb & ((1ull << d) - 1)) != 0);
        }
    } else {
        int32_t d = eb - ea; e = eb;
        if (d > 30) xa = (xa != 0);
        else xa = (xa >> d) | ((xa & ((1ull << d) - 1)) != 0);
    }

    uint32_t s;
    uint64_t x;
    if (sa == sb) { s = sa; x = xa + xb; }
    else if (xa > xb) { s = sa; x = xa - xb; }
    else if (xb > xa) { s = sb; x = xb - xa; }
    else return 0;                                         /* exact cancel -> +0 under RNE */

    /* normalise so that the hidden bit sits at bit 26 (23 + 3 guard bits) */
    if (x & (1ull << 27)) {                                /* carry out */
        x = (x >> 1) | (x & 1);
        e += 1;
    }
    while (!(x & (1ull << 26)) && e > 1) { x <<= 1; e -= 1; }

    /* round to nearest even on the 3 guard bits */
    uint32_t grs = (uint32_t)(x & 7);
    x >>= 3;
    if (grs > 4 || (grs == 4 && (x & 1))) x += 1;
    if (x & (1ull << 24)) { x >>= 1; e += 1; }             /* rounding carried out */

    if (!(x & (1ull << 23)))                               /* still subnormal */
        return (s << 31) | (uint32_t)x;                    /* exponent field 0 */
    if (e >= 0xff) return (s << 31) | 0x7f800000u;         /* overflow -> Inf */
    return (s << 31) | ((uint32_t)e << 23) | ((uint32_t)x & 0x7fffffu);
}

/* Whole-vector soft-float add on bit patterns (for cross-checking oracle_vadd_f32). */
void oracle_softfloat_vadd_f32(const uint32_t *a, const uint32_t *b, uint32_t *c, size_t n)
{
    for (size_t i = 0; i < n; ++i)
        c[i] = oracle_softfloat_add_f32(a[i], b[i]);
}

/* ------------------------------------------------------------ a2: input recipes */

/* The sample's input recipe: interleaved rand() fill, never seeded (== srand(1)).
 * Reseeds to 1 first so that repeated calls inside one test process reproduce what a
 * fresh ./vectorAdd process sees (each loop iteration of cuda-test-deployment.yaml:19
 * is a fresh process). */
void oracle_fill_rand_f32(float *a, float *b, size_t n)
{
    srand(1);
    for (size_t i = 0; i < n; ++i) {
        a[i] = rand() / (float)RAND_MAX;
        b[i] = rand() / (float)RAND_MAX;
    }
}

static inline uint64_t splitmix64(uint64_t z)
{
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

/* Stateless counter generator for the large configs (SURVEY.md section 8(d)):
 * x[i] = (float)(splitmix64(seed*PHI + first+i) >> 40) * 2^-24, uniform on [0,1). */
void oracle_fill_ctr_f32(float *x, size_t n, uint64_t seed, uint64_t first)
{
    const uint64_t base = seed * 0x9E3779B97F4A7C15ull + first;
    for (size_t i = 0; i < n; ++i)
        x[i] = (float)(splitmix64(base + i) >> 40) * 0x1.0p-24f;
}

/* ------------------------------------------------------------ a6: self-verify */

/* The sample's own check: fabs(h_A[i] + h_B[i] - h_C[i]) > 1e-5 fails.
 * Returns -1 if all pass, else the first failing index. */
long long oracle_verify_sample_tolerance(const float *a, const float *b, const float *c, size_t n)
{
    for (size_t i = 0; i < n; ++i)
        if (fabs(a[i] + b[i] - c[i]) > 1e-5)
            return (long long)i;
    return -1;
}

/* Bit-exact compare of two result vectors; NaNs match as a class (PTX add.f32 returns
 * the canonical NaN 0x7fffffff, SSE addss propagates a quieted payload).
 * Returns -1 if identical, else the first differing index. */
long long oracle_first_mismatch_f32(const float *x, const float *y, size_t n)
{
    const uint32_t *ux = (const uint32_t *)x, *uy = (const uint32_t *)y;
    for (size_t i = 0; i < n; ++i) {
        if (ux[i] == uy[i]) continue;
        int nx = (ux[i] & 0x7fffffffu) > 0x7f800000u, ny = (uy[i] & 0x7fffffffu) > 0x7f800000u;
        if (nx && ny) continue;
        return (long long)i;
    }
    return -1;
}

/* ------------------------------------------------------------ digests */

uint64_t oracle_fnv1a64(const void *p, size_t nbytes)
{
    const unsigned char *s = (const unsigned char *)p;
    uint64_t h = 1469598103934665603ull;
    for (size_t i = 0; i < nbytes; ++i) { h ^= s[i]; h *= 1099511628211ull; }
    return h;
}

/* out[0] = sum of the uint32 bit patterns (mod 2^64), out[1] = xor of them. */
void oracle_bits_digest_u32(const float *x, size_t n, uint64_t out[2])
{
    const uint32_t *u = (const uint32_t *)x;
    uint64_t s = 0; uint32_t xo = 0;
    for (size_t i = 0; i < n; ++i) { s += u[i]; xo ^= u[i]; }
    out[0] = s; out[1] = xo;
}

/* Digest of A+B without materialising C: the "checksum of checksums" used at
 * BASELINE.json's full sizes, where the device result stays in HBM. */
void oracle_vadd_digest_f32(const float *a, const float *b, size_t n, uint64_t out[2])
{
    uint64_t s = 0; uint32_t xo = 0;
    for (size_t i = 0; i < n; ++i) {
        float c = a[i] + b[i];
        uint32_t u; memcpy(&u, &c, 4);
        s += u; xo ^= u;
    }
    out[0] = s; out[1] = xo;
}

/* ------------------------------------------------------------ all-cores baseline */

int oracle_num_cpus(void)
{
    cpu_set_t set;
    if (sched_getaffinity(0, sizeof set, &set) == 0) {
        int c = CPU_COUNT(&set);
        if (c > 0) return c;
    }
    long c = sysconf(_SC_NPROCESSORS_ONLN);
    return c > 0 ? (int)c : 1;
}

/* CPU bandwidth quota of the container in whole CPUs (cgroup v2 cpu.max or v1 cfs quota),
 * 0 if unlimited/unknown.  More runnable threads than this only get throttled. */
double oracle_cpu_quota(void)
{
    FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r");
    if (f) {
        char q[64]; double period = 0;
        int n = fscanf(f, "%63s %lf", q, &period);
        fclose(f);
        if (n == 2 && strcmp(q, "max") != 0 && period > 0) return atof(q) / period;
        return 0.0;
    }
    double quota = -1, period = 0;
    if ((f = fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r"))) { if (fscanf(f, "%lf", &quota) != 1) quota = -1; fclose(f); }
    if ((f = fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r"))) { if (fscanf(f, "%lf", &period) != 1) period = 0; fclose(f); }
    return (quota > 0 && period > 0) ? quota / period : 0.0;
}

typedef struct {
    const float *a, *b; float *c; size_t lo, hi;
    uint64_t seed_a, seed_b, first; int op;                /* 0 add, 1 fill, 2 digest, 3 add with non-temporal stores */
    uint64_t dig[2];
} span_t;

__attribute__((target_clones("avx2", "default")))
static void add_span(const float *a, const float *b, float *c, size_t lo, size_t hi)
{
    for (size_t i = lo; i < hi; ++i)
        c[i] = a[i] + b[i];
}

/* Non-temporal-store variants of the same add, for the reported CPU baseline only: a
 * regular store to a line that is not in cache first READS it (write-allocate), so the
 * scalar/AVX2 loop above moves ~16 B per element through DRAM, not 12.  Streaming stores
 * (movntps / vmovntps) skip that read.  vaddps is the same correctly-rounded IEEE add per
 * lane as addss, so the results are bit-identical (checked in tests/test_oracle.py).
 * The widest ISA the host supports is picked at run time. */
#if defined(__x86_64__)
__attribute__((target("avx512f")))
static void add_span_nt512(const float *a, const float *b, float *c, size_t lo, size_t hi)
{
    size_t i = lo;
    for (; i < hi && ((uintptr_t)(c + i) & 63u); ++i) c[i] = a[i] + b[i];
    for (; i + 16 <= hi; i += 16)
        _mm512_stream_ps(c + i, _mm512_add_ps(_mm512_loadu_ps(a + i), _mm512_loadu_ps(b + i)));
    for (; i < hi; ++i) c[i] = a[i] + b[i];
    _mm_sfence();
}

__attribute__((target("avx")))
static void add_span_nt256(const float *a, const float *b, float *c, size_t lo, size_t hi)
{
    size_t i = lo;
    for (; i < hi && ((uintptr_t)(c + i) & 31u); ++i) c[i] = a[i] + b[i];
    for (; i + 8 <= hi; i += 8)
        _mm256_stream_ps(c + i, _mm256_add_ps(_mm256_loadu_ps(a + i), _mm256_loadu_ps(b + i)));
    for (; i < hi; ++i) c[i] = a[i] + b[i];
    _mm_sfence();
}

static void add_span_nt128(const float *a, const float *b, float *c, size_t lo, size_t hi)
{
    size_t i = lo;
    for (; i < hi && ((uintptr_t)(c + i) & 15u); ++i) c[i] = a[i] + b[i];
    for (; i + 4 <= hi; i += 4)
        _mm_stream_ps(c + i, _mm_add_ps(_mm_loadu_ps(a + i), _mm_loadu_ps(b + i)));
    for (; i < hi; ++i) c[i] = a[i] + b[i];
    _mm_sfence();
}

/* 512 / 256 / 128: the vector width the non-temporal variant uses on this host. */
int oracle_nt_width(void)
{
    __builtin_cpu_init();
    if (__builtin_cpu_supports("avx512f")) return 512;
    if (__builtin_cpu_supports("avx")) return 256;
    return 128;
}

static void add_span_nt(const float *a, const float *b, float *c, size_t lo, size_t hi)
{
    switch (oracle_nt_width()) {
        case 512: add_span_nt512(a, b, c, lo, hi); break;
        case 256: add_span_nt256(a, b, c, lo, hi); break;
        default:  add_span_nt128(a, b, c, lo, hi); break;
    }
}
#else
int oracle_nt_width(void) { return 0; }
static void add_span_nt(const float *a, const float *b, float *c, size_t lo, size_t hi) { add_span(a, b, c, lo, hi); }
#endif

static void *span_main(void *arg)
{
    span_t *s = (span_t *)arg;
    if (s->op == 0) {
        add_span(s->a, s->b, s->c, s->lo, s->hi);
    } else if (s->op == 3) {
        add_span_nt(s->a, s->b, s->c, s->lo, s->hi);
    } else if (s->op == 1) {                               /* first-touch + fill */
        oracle_fill_ctr_f32((float *)s->a + s->lo, s->hi - s->lo, s->seed_a, s->first + s->lo);
        oracle_fill_ctr_f32((float *)s->b + s->lo, s->hi - s->lo, s->seed_b, s->first + s->lo);
        if (s->c) memset(s->c + s->lo, 0, (s->hi - s->lo) * sizeof(float));
    } else {
        oracle_vadd_digest_f32(s->a + s->lo, s->b + s->lo, s->hi - s->lo, s->dig);
    }
    return NULL;
}

static void run_spans(span_t proto, size_t n, int threads, uint64_t dig[2])
{
    if (threads < 1) threads = 1;
    if ((size_t)threads > n && n) threads = (int)n;
    pthread_t *tid = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)threads);
    span_t *sp = (span_t *)malloc(sizeof(span_t) * (size_t)threads);
    /* contiguous static partition, chunk boundaries on 16-float (64 B line) multiples */
    size_t chunk = (n + (size_t)threads - 1) / (size_t)threads;
    chunk = (chunk + 15) & ~(size_t)15;
    for (int t = 0; t < threads; ++t) {
        sp[t] = proto;
        sp[t].lo = (size_t)t * chunk < n ? (size_t)t * chunk : n;
        sp[t].hi = sp[t].lo + chunk < n ? sp[t].lo + chunk : n;
        sp[t].dig[0] = sp[t].dig[1] = 0;
        pthread_create(&tid[t], NULL, span_main, &sp[t]);
    }
    uint64_t s = 0, x = 0;
    for (int t = 0; t < threads; ++t) {
        pthread_join(tid[t], NULL);
        s += sp[t].dig[0]; x ^= sp[t].dig[1];
    }
    if (dig) { dig[0] = s; dig[1] = x; }
    free(tid); free(sp);
}

/* C = A + B on `threads` host threads (static contiguous partition). */
void oracle_vadd_f32_mt(const float *a, const float *b, float *c, size_t n, int threads)
{
    span_t p; memset(&p, 0, sizeof p);
    p.a = a; p.b = b; p.c = c; p.op = 0;
    run_spans(p, n, threads, NULL);
}

/* The same with non-temporal stores (timing variant of the CPU baseline; same bits). */
void oracle_vadd_f32_mt_nt(const float *a, const float *b, float *c, size_t n, int threads)
{
    span_t p; memset(&p, 0, sizeof p);
    p.a = a; p.b = b; p.c = c; p.op = 3;
    run_spans(p, n, threads, NULL);
}

/* Multi-threaded ctr fill of A and B (and zero of C if non-NULL): the worker that will
 * later add a span also first-touches it. */
void oracle_fill_ctr_pair_mt(float *a, float *b, float *c, size_t n, uint64_t seed_a,
                             uint64_t seed_b, uint64_t first, int threads)
{
    span_t p; memset(&p, 0, sizeof p);
    p.a = a; p.b = b; p.c = c; p.op = 1; p.seed_a = seed_a; p.seed_b = seed_b; p.first = first;
    run_spans(p, n, threads, NULL);
}

void oracle_vadd_digest_f32_mt(const float *a, const float *b, size_t n, int threads, uint64_t out[2])
{
    span_t p; memset(&p, 0, sizeof p);
    p.a = a; p.b = b; p.op = 2;
    run_spans(p, n, threads, out);
}

static double now_s(void)
{
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

/* Times `reps` passes of the all-cores add over n elements; writes per-pass seconds to
 * secs[reps].  Buffers are allocated and first-touched by the worker threads here. */
int oracle_time_vadd_mt_ex(size_t n, int threads, int warmup, int reps, int nt_stores, double *secs);

int oracle_time_vadd_mt(size_t n, int threads, int warmup, int reps, double *secs)
{
    return oracle_time_vadd_mt_ex(n, threads, warmup, reps, 0, secs);
}

/* nt_stores: 0 regular (write-allocate) stores, 1 non-temporal stores. */
int oracle_time_vadd_mt_ex(size_t n, int threads, int warmup, int reps, int nt_stores, double *secs)
{
    void (*add)(const float *, const float *, float *, size_t, int) = nt_stores ? oracle_vadd_f32_mt_nt : oracle_vadd_f32_mt;
    float *a = NULL, *b = NULL, *c = NULL;
    if (posix_memalign((void **)&a, 64, n * sizeof(float) + 64) ||
        posix_memalign((void **)&b, 64, n * sizeof(float) + 64) ||
        posix_memalign((void **)&c, 64, n * sizeof(float) + 64)) {
        free(a); free(b); free(c);
        return -1;
    }
    oracle_fill_ctr_pair_mt(a, b, c, n, 0x0A, 0x0B, 0, threads);
    for (int i = 0; i < warmup; ++i) add(a, b, c, n, threads);
    for (int i = 0; i < reps; ++i) {
        double t0 = now_s();
        add(a, b, c, n, threads);
        secs[i] = now_s() - t0;
    }
    free(a); free(b); free(c);
    return 0;
}

/* ============================================================================ f4 oracle
 * STREAM-style ops of the generalised core (SURVEY.md 8(f) row 4; not in the reference,
 * whose only operation is the f32 add above).  Semantics restated from include/b200va.h:
 *   COPY c=a   SCALE c=s*a   ADD c=a+b   TRIAD c=fma(s,b,a)
 * f32/f64 natively (RNE); f16/bf16: widen exactly to f32, op in f32 (s rounded to f32),
 * round to nearest-even into the storage type.  The half conversions below are integer
 * code written from the formats' definitions, independent of compiler half types. */
static float half_to_float(uint16_t h)
{
    uint32_t s = (uint32_t)(h >> 15) << 31, e = (h >> 10) & 0x1f, m = h & 0x3ff, u;
    if (e == 0x1f) u = s | 0x7f800000u | (m << 13);                 /* Inf / NaN */
    else if (e) u = s | ((e + 112) << 23) | (m << 13);              /* normal: bias 15 -> 127 */
    else if (m) {                                                   /* subnormal: renormalise */
        int sh = 0;
        while (!(m & 0x400)) { m <<= 1; ++sh; }
        u = s | ((uint32_t)(113 - sh) << 23) | ((m & 0x3ff) << 13);
    } else u = s;
    float f; memcpy(&f, &u, 4); return f;
}

static uint16_t float_to_half_rne(float f)
{
    uint32_t u; memcpy(&u, &f, 4);
    uint16_t s = (uint16_t)((u >> 16) & 0x8000);
    uint32_t a = u & 0x7fffffffu;
    if (a > 0x7f800000u) return (uint16_t)(s | 0x7fff);             /* NaN (class only) */
    if (a >= 0x47800000u) return (uint16_t)(s | 0x7c00);            /* >= 65536 -> Inf (also Inf) */
    int32_t e = (int32_t)(a >> 23) - 127;
    uint32_t m = (a & 0x7fffffu) | 0x800000u;                       /* 24-bit significand */
    int shift;                                                      /* bits to drop */
    uint32_t base;
    if (e >= -14) { shift = 13; base = (uint32_t)(e + 15) << 10; m &= 0x7fffffu; }
    else { shift = 13 + (-14 - e); base = 0; if (shift > 25) return s; }   /* subnormal or zero */
    uint32_t q = m >> shift, rem = m & ((1u << shift) - 1), half = 1u << (shift - 1);
    uint32_t r = base + q;
    if (rem > half || (rem == half && (r & 1))) r += 1;             /* carries ripple into the exponent */
    return (uint16_t)(s | r);                                       /* 0x7c00 if it rounded up to Inf */
}

static float bf16_to_float(uint16_t h) { uint32_t u = (uint32_t)h << 16; float f; memcpy(&f, &u, 4); return f; }

static uint16_t float_to_bf16_rne(float f)
{
    uint32_t u; memcpy(&u, &f, 4);
    if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x7fff);   /* NaN */
    uint32_t lsb = (u >> 16) & 1;
    u += 0x7fffu + lsb;                                             /* RNE; overflow rounds to Inf */
    return (uint16_t)(u >> 16);
}

#include <math.h>
enum { ORC_COPY = 0, ORC_SCALE = 1, ORC_ADD = 2, ORC_TRIAD = 3 };
enum { ORC_F32 = 0, ORC_F64 = 1, ORC_F16 = 2, ORC_BF16 = 3 };

static inline float stream_f32(int op, float a, float b, float s)
{
    switch (op) {
        case ORC_SCALE: return s * a;
        case ORC_ADD:   return a + b;
        case ORC_TRIAD: return fmaf(s, b, a);
        default:        return a;
    }
}

/* Returns 0, or -1 for an unknown op/dtype. */
int oracle_stream(int op, int dtype, const void *a, const void *b, void *c, size_t n, double scalar)
{
    if (op < 0 || op > 3 || dtype < 0 || dtype > 3) return -1;
    const int binary = (op == ORC_ADD || op == ORC_TRIAD);
    if (op == ORC_COPY) { memcpy(c, a, n * (dtype == ORC_F64 ? 8 : dtype == ORC_F32 ? 4 : 2)); return 0; }
    if (dtype == ORC_F32) {
        const float *x = (const float *)a, *y = (const float *)b; float *z = (float *)c; const float s = (float)scalar;
        for (size_t i = 0; i < n; ++i) z[i] = stream_f32(op, x[i], binary ? y[i] : 0.f, s);
    } else if (dtype == ORC_F64) {
        const double *x = (const double *)a, *y = (const double *)b; double *z = (double *)c;
        for (size_t i = 0; i < n; ++i)
            z[i] = op == ORC_SCALE ? scalar * x[i] : op == ORC_ADD ? x[i] + y[i] : fma(scalar, y[i], x[i]);
    } else {
        const uint16_t *x = (const uint16_t *)a, *y = (const uint16_t *)b; uint16_t *z = (uint16_t *)c;
        const float s = (float)scalar;
        for (size_t i = 0; i < n; ++i) {
            if (dtype == ORC_F16)
                z[i] = float_to_half_rne(stream_f32(op, half_to_float(x[i]), binary ? half_to_float(y[i]) : 0.f, s));
            else
                z[i] = float_to_bf16_rne(stream_f32(op, bf16_to_float(x[i]), binary ? bf16_to_float(y[i]) : 0.f, s));
        }
    }
    return 0;
}

void oracle_half_to_float(const uint16_t *h, float *f, size_t n) { for (size_t i = 0; i < n; ++i) f[i] = half_to_float(h[i]); }
void oracle_float_to_half(const float *f, uint16_t *h, size_t n) { for (size_t i = 0; i < n; ++i) h[i] = float_to_half_rne(f[i]); }
void oracle_bf16_to_float(const uint16_t *h, float *f, size_t n) { for (size_t i = 0; i < n; ++i) f[i] = bf16_to_float(h[i]); }
void oracle_float_to_bf16(const float *f, uint16_t *h, size_t n) { for (size_t i = 0; i < n; ++i) h[i] = float_to_bf16_rne(f[i]); }
