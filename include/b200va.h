/*
 * b200va.h -- C ABI of libb200va.so: the H100 (sm_90a) vectorAdd hot path.
 *
 * The reference (ashrafgt/k8s-gpu-hpa) has NO library/plugin API for this path: the
 * kernel is statically linked into the `vectorAdd` executable inside the third-party
 * image k8s.gcr.io/cuda-vector-add:v0.1, and the reference only invokes it:
 *
 *     image:   "k8s.gcr.io/cuda-vector-add:v0.1"                     cuda-test-deployment.yaml:18
 *     command: for (( c=1; c<=5000; c++ )); do ./vectorAdd; done     cuda-test-deployment.yaml:19
 *     (same loop started by hand to raise utilisation)               README.md:113-116
 *
 * The outer drop-in boundary is therefore the `vectorAdd` executable
 * (k8s-gpu-hpa_b200/host/vectorAdd.cpp).  This header is the inner boundary the
 * executable -- and any other host language via cgo/JNI/ctypes -- binds: each entry
 * point below names the step of that process (SURVEY.md section 8(a), rows a1-a7) it
 * replaces.  See INTEGRATION.md for the binding stubs.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no C++ or torch types, no exceptions.
 *   - Functions return 0 (B200VA_OK) or a negative code; they never print or abort.
 *     CUDA runtime failures are returned as  -(1000 + cudaError_t).
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).
 *     Device entry points are asynchronous on that stream: no hidden synchronisation,
 *     no hidden allocation; the caller owns every buffer.
 *   - The current CUDA device of the calling thread is used (cudaSetDevice first);
 *     the library is re-entrant and keeps only immutable per-device attribute caches.
 *     Entry points that take a `device` argument (stager, b200va_add_f32_host, b200va_query)
 *     restore the caller's current device before returning, on every path.
 *   - Element type is IEEE-754 binary32; the add is add.rn.f32 without FTZ, so results
 *     are bit-identical to a scalar C loop on the same inputs (NaN payloads excepted:
 *     PTX returns the canonical NaN 0x7fffffff).
 */
#ifndef B200VA_H
#define B200VA_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200VA_ABI_VERSION 2   /* 2: b200va_tune_t grew early_loads/scheduler; *_ex, stager modes 4/AUTO */

/* ---- status codes ------------------------------------------------------------- */
#define B200VA_OK               0
#define B200VA_ERR_INVALID     (-1)   /* NULL pointer with n > 0, bad argument            */
#define B200VA_ERR_ALIGN       (-2)   /* pointer not 4-byte aligned                       */
#define B200VA_ERR_OVERLAP     (-3)   /* C partially overlaps A or B (exact alias is ok)  */
#define B200VA_ERR_VARIANT     (-4)   /* unknown kernel variant / unsupported tune combo  */
#define B200VA_ERR_NO_DEVICE   (-5)   /* no CUDA device / not an sm_90 device             */
#define B200VA_ERR_VERIFY      (-6)   /* result verification failed (a6)                  */
#define B200VA_ERR_NOMEM       (-7)   /* host allocation failed; captured-counter pool empty */
#define B200VA_ERR_CUDA_BASE   (-1000) /* code = -(1000 + cudaError_t)                    */
/* Which combinations a library carries: libb200va.so ships the production set (what
 * B200VA_K_AUTO and the named variants resolve to, plus a few neighbours); the full
 * A/B matrix of b200va_tune_t lives in libb200va_tune.so (same ABI, development only).
 * A combination the loaded library does not carry returns B200VA_ERR_VARIANT. */

/* ---- kernel variants (argument `variant`) ---------------------------------------- */
#define B200VA_K_AUTO      0   /* the tuned production choice for this n                */
#define B200VA_K0_SCALAR   1   /* reference-shape control: 1 elem/thread, 256-thread CTAs,
                                  (n+255)/256 CTAs  (CUDA sample launch geometry, a5)   */
#define B200VA_K1_VEC128   2   /* 128-bit ld/st.global.v4.f32, unrolled, cache-hinted   */
#define B200VA_K2_TMA      3   /* cp.async.bulk (TMA) smem ring; tiles handed out by the
                                  dynamic tile scheduler (store_mode 2)                  */
#define B200VA_K3_VEC256   4   /* 32-byte vectors per thread: two adjacent 128-bit
                                  ld/st.global.v4.f32 (sm_90 has no 256-bit access)     */
#define B200VA_K4_SCALAR_MLP 5 /* 32-bit accesses, `unroll` (4|8|16) independent loads per array
                                  per thread in flight: the mixed-misalignment path, also
                                  selectable through b200va_add_f32_tuned for A/B runs   */

/* Explicit geometry for A/B experiments (b200va_add_f32_tuned). Zero = default.      */
typedef struct b200va_tune {
    int kind;         /* B200VA_K0_SCALAR .. B200VA_K3_VEC256                           */
    int threads;      /* CTA size (vec kernels) or consumer threads (TMA kernel)        */
    int unroll;       /* vec: vectors per thread per tile: 1,2,4,8                      */
    int ctas_per_sm;  /* 0: one tile per CTA; >0: persistent grid = SMs * ctas_per_sm   */
    int ld_hint;      /* 0 plain, 1 L1::no_allocate, 2 .cs, 3 no_allocate+L2 evict_first, 4 .nc+no_allocate, 5 no_allocate+L2::256B */
    int st_hint;      /* 0 plain, 1 L1::no_allocate,   2 .cs, 3 no_allocate+L2 evict_first */
    int stages;       /* TMA: ring depth (2..16)                                        */
    int tile_bytes;   /* TMA: bytes per array per stage (multiple of 2048)              */
    int store_mode;   /* TMA: 0 = st.global from registers, 1 = bulk store from smem,
                         2 = register stores + dynamic tile scheduler (persistent grid,
                             tiles claimed from an atomic ticket counter)               */
    int early_loads;  /* vec: what a CTA does about its first tile before the programmatic
                         dependency on the previous launch resolves:
                         1 = issue the loads themselves (only the stores wait).  Requires that
                             the previous launch on the stream does not write A or B; replaced
                             by 2 when C aliases A or B.  See b200va_add_f32_ex.
                         2 = bulk-prefetch the A and B tiles into L2 (cp.async.bulk.prefetch.L2);
                             loads and stores wait.  Always legal (L2 is the coherence point);
                             pays off on data that is not already in L2.                     */
    int scheduler;    /* vec: 0 = hardware block scheduler (one CTA per tile, or the static
                         persistent split of ctas_per_sm), 1 = dynamic tile scheduler:
                         a persistent grid whose CTAs claim tiles from an atomic ticket
                         counter (K1d)                                                  */
} b200va_tune_t;

typedef struct b200va_devinfo {
    int device;
    int cc_major, cc_minor;
    int sm_count;
    int max_smem_optin;        /* bytes                                                 */
    int l2_bytes;
    size_t global_mem_bytes;
    char name[64];
} b200va_devinfo_t;

/* ---- library ----------------------------------------------------------------------- */
int         b200va_abi_version(void);
const char *b200va_strerror(int code);
/* Attributes of `device` (does not change the current device). */
int         b200va_query(int device, b200va_devinfo_t *out);
/* The geometry B200VA_K_AUTO (or a named variant) resolves to for n elements; the _ex form
 * takes the B200VA_F_* hints b200va_add_f32_ex takes. */
int         b200va_resolve(int variant, size_t n, b200va_tune_t *out);
int         b200va_resolve_ex(int variant, size_t n, unsigned flags, b200va_tune_t *out);

/* Launch geometry of b200va_add_f32_tuned(tune) on `device` for n elements with distinct,
 * 256-byte-aligned pointers (what "CUDA kernel launch with %d blocks of %d threads" prints,
 * a5).  Planned exactly as that call plans its launch: for a tune it would launch, the
 * geometry it launches with; for a tune it refuses, its error code. */
int         b200va_geometry(const b200va_tune_t *tune, size_t n, int device,
                            unsigned *grid, unsigned *block, unsigned *dyn_smem_bytes);

/* ---- a4 + a5: the vectorAdd kernel and its launch geometry -------------------------
 * Replaces `vectorAdd<<<blocksPerGrid, threadsPerBlock>>>(d_A, d_B, d_C, numElements)`
 * of the image's binary (invoked at cuda-test-deployment.yaml:19).
 * dA, dB, dC: device pointers, 4-byte aligned; any n >= 0; dC may equal dA or dB.
 * Capture.  b200va_add_f32, b200va_add_f32_ex and b200va_add_f32_tuned are capturable in a CUDA graph, also as
 * the first call of a process and under every capture mode: the one-time setup of the dynamic tile scheduler's
 * counters runs in relaxed capture mode on a private stream.  A dynamically scheduled launch (variant K2,
 * scheduler = 1) captured into a graph takes a ticket counter that the graph holds until it and every executable
 * instance of it are destroyed; no direct launch is handed it meanwhile.  So the executable instances of one
 * captured graph must not run at the same time, and each device lends at most 16384 such counters at once: one
 * more is refused with B200VA_ERR_NOMEM.  b200va_add_f32_loop with graph_batch > 1 and b200va_loop_create
 * allocate and synchronize, and are not capturable: the former returns -(1000 + cudaErrorStreamCaptureUnsupported)
 * when `stream` is capturing. */
int b200va_add_f32(const float *dA, const float *dB, float *dC, size_t n,
                   int variant, void *stream);
int b200va_add_f32_tuned(const float *dA, const float *dB, float *dC, size_t n,
                         const b200va_tune_t *tune, void *stream);
/* Same as b200va_add_f32 with launch-ordering hints (`flags`, OR of B200VA_F_*).
 * B200VA_F_INPUTS_STABLE: the caller promises that the launch immediately preceding this
 * one on `stream` does not write A or B (e.g. it is another add into a different or the
 * same C).  The kernel then issues its loads while that launch is still draining and only
 * its stores wait for it (programmatic dependent launch), which removes most of the
 * ~2 us bubble between back-to-back launches.  The library's kernels release their
 * successor only after their own wait, so the immediately preceding launch is the only
 * one that can still be running.  Results and stream order of C are unchanged; the flag
 * is ignored when C aliases A or B. */
#define B200VA_F_INPUTS_STABLE 1u
/* B200VA_F_COLD: the operands are not L2-resident (fresh from a copy engine, or one of many
 * buffer sets touched in rotation): B200VA_K_AUTO then resolves to the geometry tuned on
 * rotating buffers instead of the one tuned for relaunching the same buffers -- in particular
 * the launch prefetches its first tiles into L2 while the previous launch is still draining
 * (early_loads = 2; no promise about the previous launch is needed for that).  A hint only;
 * vectors of 2^25 elements and more can never be L2-resident and are always treated as cold. */
#define B200VA_F_COLD          2u
int b200va_add_f32_ex(const float *dA, const float *dB, float *dC, size_t n,
                      int variant, unsigned flags, void *stream);

/* ---- a1: the launch loop, in-process -----------------------------------------------
 * Replaces the 5000-process bash loop (cuda-test-deployment.yaml:19): `iters`
 * back-to-back launches on `stream`; graph_batch > 1 captures that many launches into
 * one CUDA graph and replays it (launch-bound sizes).  Asynchronous, except that the
 * graph form (graph_batch > 1) drains the stream before returning; any capturable or
 * legacy stream is accepted (the capture happens on a private stream).
 * Launches 2..iters of a loop know their predecessor (the same add, which writes only C),
 * so unless C aliases A or B they run with early loads (see B200VA_F_INPUTS_STABLE). */
int b200va_add_f32_loop(const float *dA, const float *dB, float *dC, size_t n,
                        int variant, int iters, int graph_batch, void *stream);
/* Persistent form for a long-running load generator: the graph of `graph_batch` launches
 * is captured once; b200va_loop_run replays it floor(iters/graph_batch) times plus
 * iters%graph_batch direct launches, asynchronously on `stream`.  Destroy only after
 * the stream has drained.  One handle must not be run on two streams at the same time:
 * every replay of its graph uses the same scratch memory (the ticket counters of the
 * dynamically scheduled kernels), so two replays in flight at once would share it.
 * Separate handles are independent. */
typedef struct b200va_loop b200va_loop_t;
int b200va_loop_create(b200va_loop_t **out, const float *dA, const float *dB, float *dC,
                       size_t n, int variant, int graph_batch);
int b200va_loop_run(b200va_loop_t *loop, int iters, void *stream);
int b200va_loop_destroy(b200va_loop_t *loop);

/* ---- a2: input recipes ---------------------------------------------------------------
 * Host: the sample's recipe  h_A[i] = rand()/(float)RAND_MAX; h_B[i] = ... interleaved,
 * never seeded.  Reseeds glibc to 1 so every call equals a fresh ./vectorAdd process. */
int b200va_host_fill_rand_f32(float *hA, float *hB, size_t n);
/* Counter generator for large n (index-addressable, shard-invariant):
 * x[i] = (float)(splitmix64(seed*0x9E3779B97F4A7C15 + first + i) >> 40) * 2^-24.       */
int b200va_host_fill_ctr_f32(float *h, size_t n, uint64_t seed, uint64_t first);
int b200va_fill_ctr_f32(float *d, size_t n, uint64_t seed, uint64_t first, void *stream);

/* ---- a6: verification ----------------------------------------------------------------
 * Host: the sample's check made strict: bitwise C[i] == A[i]+B[i] (NaNs as a class).
 * Returns B200VA_OK or B200VA_ERR_VERIFY with *first_bad = failing index.            */
int b200va_host_verify_f32(const float *hA, const float *hB, const float *hC, size_t n,
                           size_t *first_bad);
/* Device: recompute + bit-compare in HBM.  d_result[0] = mismatch count,
 * d_result[1] = first mismatching index (UINT64_MAX if none).  Asynchronous; the
 * caller zero-inits nothing (the call resets d_result on the stream first).          */
int b200va_verify_f32(const float *dA, const float *dB, const float *dC, size_t n,
                      uint64_t *d_result, void *stream);
/* Device digest of a vector's bit patterns: d_out[0] = sum of uint32 patterns mod 2^64,
 * d_out[1] = xor of them.  Order-independent, so shards combine by + and ^.          */
int b200va_digest_f32(const float *d, size_t n, uint64_t *d_out, void *stream);

/* ---- a3 + a4 + a6(copy) : host-buffer path -------------------------------------------
 * Replaces cudaMalloc x3 / cudaMemcpy H2D x2 / kernel / cudaMemcpy D2H of one
 * ./vectorAdd run, for host arrays of any size: a staged, double-direction pipeline
 * (H2D of chunk k+1, add of chunk k, D2H of chunk k-1 overlap on separate streams).
 * A stager owns its device staging buffers and streams; create one per device/thread. */
typedef struct b200va_stager b200va_stager_t;
/* mode 0: copy-engine pipeline through HBM staging buffers;
 * mode 1: zero-copy kernel reading/writing pinned host memory directly over PCIe
 *         (requires all three host buffers pinned/registered);
 * mode 2: "lanes" pipeline: one stream per direction plus one for the adds, event edges
 *         per slot, so the H2D queue never waits behind another chunk's kernel or D2H;
 * mode 3: pageable host arrays (plain malloc): host threads copy chunks through pinned
 *         bounce buffers around the lanes pipeline.  b200va_add_f32_host picks 2 or 3
 *         by asking the runtime whether the arrays are pinned.
 * mode 4: register-once: pageable arrays are page-locked in place (cudaHostRegister) the
 *         first time the stager sees them and the registration is cached by address range,
 *         so a long-lived loop over the same malloc'd arrays -- the reference process's
 *         shape -- runs the lanes pipeline at the pinned rate from the second call on.
 *         The first call pays the pinning (~0.3 ms/MiB).  Registered arrays must stay
 *         allocated until b200va_stager_release_host / b200va_stager_destroy.  Falls back
 *         to mode 3 if the registration is refused (RLIMIT_MEMLOCK, exotic mappings).
 * mode -1 (B200VA_STAGE_AUTO): mode 2 for pinned arrays, mode 4 for pageable arrays of at
 *         least 8 MiB in total, mode 3 below that. */
#define B200VA_STAGE_AUTO      (-1)
#define B200VA_STAGE_SLOTS       0
#define B200VA_STAGE_ZEROCOPY    1
#define B200VA_STAGE_LANES       2
#define B200VA_STAGE_BOUNCE      3
#define B200VA_STAGE_REGISTER    4
/* chunk_elems = 0 -> 32 Mi elements (128 MiB per array per slot), depth = 0 -> 3 slots.
 * The lanes pipeline tapers the last chunk (1/2, 1/4, ... ~1 Mi) so the D2H tail is short. */
int b200va_stager_create(b200va_stager_t **out, int device, size_t chunk_elems, int depth);
/* Synchronous.  On an error in the middle of the pipeline every stream of the stager is
 * drained before the call returns, so no copy is still touching the caller's arrays. */
int b200va_stager_add_f32(b200va_stager_t *s, const float *hA, const float *hB, float *hC,
                          size_t n, int variant, int mode);
/* Device-side time of the last b200va_stager_add_f32 call, milliseconds (events). */
int b200va_stager_last_ms(b200va_stager_t *s, float *ms);
/* The mode the last b200va_stager_add_f32 call actually ran (after AUTO / fallbacks). */
int b200va_stager_last_mode(b200va_stager_t *s, int *mode);
/* Unregister every host range the stager page-locked (mode 4); call before freeing them
 * if the stager outlives the arrays.  b200va_stager_destroy does this too. */
int b200va_stager_release_host(b200va_stager_t *s);
int b200va_stager_destroy(b200va_stager_t *s);
/* One-shot convenience: create, add, destroy (synchronous). */
int b200va_add_f32_host(const float *hA, const float *hB, float *hC, size_t n,
                        int device, int variant);
/* Pinned, mapped host memory for the pipeline (cudaHostAlloc / cudaFreeHost), placed on
 * the NUMA node of the current CUDA device.  write_combined != 0 adds
 * cudaHostAllocWriteCombined: meant for H2D *sources* the CPU only writes. */
int b200va_host_alloc(void **out, size_t bytes);
int b200va_host_alloc_ex(void **out, size_t bytes, int write_combined);
int b200va_host_free(void *p);
/* NUMA node that holds the page at p, or -1 if it cannot be determined. */
int b200va_host_node_of(const void *p);
/* NUMA node the current CUDA device is attached to, or -1. */
int b200va_device_numa_node(void);
/* Same for `device`, without making it current (no context is created). */
int b200va_device_numa_node_of(int device);

/* ---- generalised streaming element-wise core (SURVEY.md 8(f) row 4) -------------------
 * The tuned 128-bit streaming skeleton of the vectorAdd kernel over other element types
 * and STREAM operations.  Not part of the reference's surface (its only op is the f32
 * add, for which  b200va_stream(ADD, F32, ...)  is bit-identical to  b200va_add_f32).
 *   COPY  c = a            SCALE c = s*a          ADD c = a + b      TRIAD c = fma(s, b, a)
 * f32/f64: native IEEE arithmetic, round-to-nearest-even, no FTZ.  f16/bf16: operands
 * widened exactly to f32, op in f32 (s rounded to f32), result rounded to nearest-even.
 * dB is ignored (may be NULL) for COPY and SCALE.  Pointers aligned to the element size. */
#define B200VA_OP_COPY   0
#define B200VA_OP_SCALE  1
#define B200VA_OP_ADD    2
#define B200VA_OP_TRIAD  3
#define B200VA_DT_F32    0
#define B200VA_DT_F64    1
#define B200VA_DT_F16    2
#define B200VA_DT_BF16   3
int b200va_stream(int op, int dtype, const void *dA, const void *dB, void *dC, size_t n,
                  double scalar, void *stream);

/* c[i] = a[i] rounded once to dst_dtype (B200VA_DT_* codes on both sides): IEEE round-to-
 * nearest-even as if the exponent range were unbounded, then overflow to +-inf.  No FTZ on
 * either side: subnormal inputs and results stay.  Widening is exact; +-0 and +-inf are kept;
 * a NaN gives a NaN (payload and sign unspecified).  f16 <-> bf16 widen exactly to f32 and round
 * once; f64 -> f16/bf16 never goes through f32.  src_dtype == dst_dtype is a bit copy, NaN
 * payloads included (the COPY of b200va_stream).
 * B200VA_ERR_VARIANT: bad dtype code.  B200VA_ERR_INVALID: NULL dA/dC with n > 0, n > 2^40.
 * B200VA_ERR_ALIGN: a pointer not aligned to its own element size.  B200VA_ERR_OVERLAP: C meets A
 * anywhere, except dC == dA when both element sizes are equal (the same type, f16 <-> bf16).
 * Asynchronous on `stream`: one kernel launch, no allocation, synchronisation or memset;
 * capturable in a CUDA graph. */
int b200va_convert(int src_dtype, const void *dA, int dst_dtype, void *dC, size_t n, void *stream);

/* ---- FP8 quantize and dequantize (row f4) ---------------------------------------------------
 * The two OCP FP8 formats of the H100's FP8 tensor cores, one byte per element: */
#define B200VA_F8_E4M3 0   /* OCP FP8 E4M3 ("e4m3fn"): bias 7, no infinities, max finite 448, NaN = S.1111.111 */
#define B200VA_F8_E5M2 1   /* OCP FP8 E5M2: bias 15, IEEE-style +-inf and NaNs, max finite 57344 */
/* Quantize: c[i] = sat(RN(a[i] * 2^scale_exp)), src_dtype a B200VA_DT_* code.  The product is exact and is
 * rounded once to the FP8 format (round-to-nearest-even, the format's subnormals, no FTZ on either side).  A
 * magnitude above the largest finite value -- values that round past it and +-inf included -- gives +-max finite
 * (448 or 57344: the hardware's .satfinite); a NaN gives a NaN; +-0 and values that round to zero keep their sign.
 * d_amax (may be NULL) max-accumulates the largest unscaled magnitude: *d_amax = max(*d_amax, max_i |a_i|), the a_i
 * widened exactly to f64, a NaN anywhere making it a NaN.  Set *d_amax to +0.0 before the first call; shards and
 * repeated calls then combine.  The max is exact, so the result does not depend on the order of reduction.
 * Dequantize: c[i] = a[i] * 2^-scale_exp rounded once to dst_dtype by b200va_convert's rules (RNE, no FTZ,
 * overflow to +-inf); E5M2 +-inf stays +-inf, a NaN gives a NaN.  Dequantizing with the scale_exp a tensor was
 * quantized with gives its FP8 values scaled back, exactly whenever the destination can hold them.
 * scale_exp must lie in [-126, 126].
 * B200VA_ERR_VARIANT: bad dtype or FP8 code.  B200VA_ERR_INVALID: scale_exp out of range, NULL dA/dC with n > 0,
 * n > 2^40.  B200VA_ERR_ALIGN: dA/dC not aligned to their element size, d_amax not 8-byte aligned.
 * B200VA_ERR_OVERLAP: C meets A anywhere, or d_amax meets A or C.  n = 0 writes nothing.
 * Asynchronous on `stream`: one kernel launch, no allocation, synchronisation or memset; capturable in a CUDA
 * graph.  The d_amax update is one atomic per CTA. */
int b200va_quantize_fp8(int src_dtype, const void *dA, int fp8, void *dC, size_t n,
                        int scale_exp, double *d_amax, void *stream);
int b200va_dequantize_fp8(int fp8, const void *dA, int dst_dtype, void *dC, size_t n,
                          int scale_exp, void *stream);
/* The same casts with the scale exponent k in device memory, chosen there from the tensor's amax ("current
 * scaling"), or from a running amax the caller keeps in *d_amax, with no host read between the passes.
 * Quantize is two launches on `stream`:
 *   1. Amax pass: *d_amax = max(*d_amax, M), M the largest FINITE |a_i| widened exactly to f64 (0 when there is
 *      none).  NaN and +-inf do not take part: this is the MXFP8 block-maximum rule, not the NaN-propagating amax of
 *      b200va_quantize_fp8.  One atomic per CTA on the f64 bits, so it is exact and independent of order.  Set
 *      *d_amax = +0.0 before the call for current scaling; left as it is, the scale follows the running max.
 *   2. Scale: from the value m in *d_amax after the amax pass, K(m) is the largest integer k with
 *      m * 2^k <= max finite (448 / 57344), K(0) = +inf; with emax = 8 (E4M3) / 15 (E5M2) it reads off the bits as
 *      K = emax - floor(log2 m) - (m * 2^-floor(log2 m) > 1.75), the negated B200VA_MX_SCALE_NOSAT exponent.
 *      k = clamp(K(m) - margin, -126, 126); k = 0 if *d_amax does not hold +0.0 or a positive finite value, which
 *      happens only when the caller left a NaN, +inf or a value with the sign bit set (-0.0 included) there: the
 *      amax pass's maximum is taken on the bit patterns as unsigned integers, so it keeps those.  Every CTA computes k
 *      once the amax pass has completed; one thread writes it to *d_scale_exp.
 *   3. Quantize: c[i] = sat(RN(a[i] * 2^k)) by exactly the rules of b200va_quantize_fp8.  With margin >= 0 and k not
 *      clamped, no finite element saturates (|a_i| * 2^k <= max finite); only +-inf does.
 * Dequantize is one launch: c[i] = a[i] * 2^-k rounded once by b200va_dequantize_fp8's rules, k read from
 * *d_scale_exp once the launch before it has completed.  A k outside [-126, 126] makes every element a NaN (the
 * device-side counterpart of the E8M0 0xFF rule: the host cannot check a value that lives on the device).
 * 2^-k in f32 is the per-tensor dequantization scale an FP8 GEMM takes from a device tensor.
 * margin lies in [0, 126]; d_amax is 8-byte and d_scale_exp 4-byte aligned, both non-NULL.
 * B200VA_ERR_VARIANT: bad dtype or FP8 code.  B200VA_ERR_INVALID: margin out of range, NULL d_amax or d_scale_exp,
 * NULL dA/dC with n > 0, n > 2^40.  B200VA_ERR_ALIGN: dA/dC not aligned to their element size, d_amax or d_scale_exp
 * misaligned.  B200VA_ERR_OVERLAP: C meets A, or d_amax (quantize) or d_scale_exp meets A, C or the other.  A
 * rejected call writes nothing; n = 0 writes nothing and launches nothing (*d_scale_exp keeps its value).
 * Asynchronous on `stream`: no allocation, synchronisation or memset; capturable in a CUDA graph. */
int b200va_quantize_fp8_auto(int src_dtype, const void *dA, int fp8, void *dC, size_t n,
                             int margin, double *d_amax, int32_t *d_scale_exp, void *stream);
int b200va_dequantize_fp8_auto(int fp8, const void *dA, int dst_dtype, void *dC, size_t n,
                               const int32_t *d_scale_exp, void *stream);
/* Quantize-transpose: the FP8 bytes of a 2-D tensor and their transpose in one pass over it, the operands an H100
 * FP8 GEMM takes K-major on both sides (the forward product uses C, the backward products Ct).  A is row-major
 * rows x cols, contiguous (row stride cols); C is row-major rows x cols and Ct row-major cols x rows.  With
 * n = rows * cols:
 *   - C holds exactly the bytes b200va_quantize_fp8 (or b200va_quantize_fp8_auto) writes for n elements of A, and
 *     Ct[j * rows + i] == C[i * cols + j].
 *   - *d_amax ends with exactly the bits the 1-D call leaves: the NaN-propagating amax here (d_amax may be NULL),
 *     the finite-only amax pass in the _auto form, which also writes k to *d_scale_exp by the same rule.
 * The _auto form is two launches, the amax pass and one quantize-transpose, and captures into one graph.
 * Arguments: the rules, order and codes of the 1-D call with this n, plus: dCt non-NULL when n > 0
 * (B200VA_ERR_INVALID); rows * cols must not overflow and is at most 2^40 (B200VA_ERR_INVALID); A, C, Ct, d_amax and
 * d_scale_exp must not meet one another (B200VA_ERR_OVERLAP).  A rejected call writes nothing; rows == 0 or
 * cols == 0 writes nothing and launches nothing.
 * Fast path: rows % 16 == 0, cols % 16 == 0 and A, C and Ct on 16-byte boundaries -- every operand torch._scaled_mm
 * accepts.  Any other shape or placement gives the same bytes through a per-element path that is not tuned.
 * Asynchronous on `stream`: no allocation, synchronisation or memset; capturable in a CUDA graph. */
int b200va_quantize_fp8_transpose(int src_dtype, const void *dA, int fp8, void *dC, void *dCt,
                                  size_t rows, size_t cols, int scale_exp, double *d_amax, void *stream);
int b200va_quantize_fp8_transpose_auto(int src_dtype, const void *dA, int fp8, void *dC, void *dCt,
                                       size_t rows, size_t cols, int margin, double *d_amax,
                                       int32_t *d_scale_exp, void *stream);

/* ---- block-scaled FP8 (MXFP8) quantize and dequantize (row f4) --------------------------------
 * The same two FP8 formats with one scale per block of `block` elements, block one of 32 (OCP Microscaling MXFP8),
 * 64 and 128.  Block b is the elements [b*block, min(n, (b+1)*block)), counted from element 0 of the arrays and not
 * from an address boundary: the result does not depend on where A, C or S sit in memory.  The last block may be
 * short.  dS holds b200va_mxfp8_scale_bytes(n, block) = ceil(n / block) bytes, one per block, in E8M0: dS[b] is the
 * value 2^(dS[b] - 127), and 0xFF is NaN.  With emax = 8 for E4M3 and 15 for E5M2 (the largest finite value of
 * both formats is 1.75 * 2^emax), the scale rules are: */
#define B200VA_MX_SCALE_OCP    0   /* e = floor(log2 m) - emax: the OCP MX v1.0 rule; block values whose magnitude lies
                                      in (max finite, 2^(emax+1)) * 2^e saturate                                      */
#define B200VA_MX_SCALE_NOSAT  1   /* the smallest e with m * 2^-e <= max finite (the OCP e, plus 1 when
                                      m * 2^-floor(log2 m) > 1.75): only +-inf saturates, and f64 blocks whose e
                                      was clamped at 127                                                              */
/* Quantize, per block and in one pass over the source: m = max |a_i| over the block's finite elements, widened
 * exactly (NaN and +-inf do not take part); e by the scale rule, then clamped to [-127, 127]; m = 0, or no finite
 * element, gives e = -127.  dS[b] = e + 127, so quantize never writes 0xFF.  Then c[i] = sat(RN(a[i] * 2^-e)) by
 * exactly the rules of b200va_quantize_fp8: the product is exact and rounded once (round-to-nearest-even, the
 * format's subnormals, no FTZ on either side), +-max finite beyond it and for +-inf, a NaN gives a NaN, +-0 and
 * values that round to zero keep their sign.  e = 127 is reached from f64 only.  The result is a function of the
 * values, n, block and the rule only.
 * Dequantize: c[i] = a[i] * 2^(dS[b] - 127) rounded once to dst_dtype by b200va_convert's rules (RNE, no FTZ,
 * overflow to +-inf); dS[b] == 0xFF makes every element of block b a NaN.  Dequantizing what quantize wrote gives
 * the FP8 values scaled back, exactly whenever the destination can hold them.
 * src_dtype / dst_dtype: a B200VA_DT_* code; fp8: a B200VA_F8_* code.
 * B200VA_ERR_VARIANT: bad dtype, FP8 or scale_rule code.  B200VA_ERR_INVALID: block not 32, 64 or 128, NULL
 * dA/dC/dS with n > 0, n > 2^40.  B200VA_ERR_ALIGN: dA/dC not aligned to their element size (S is bytes: any
 * address).  B200VA_ERR_OVERLAP: C meets A, or S meets A or C.  A rejected call writes nothing; n = 0 writes nothing.
 * Asynchronous on `stream`: one kernel launch, no allocation, synchronisation or memset; capturable in a CUDA
 * graph.  The vector path runs when dA and dC are both 16-byte aligned; any other placement gives the same bytes
 * through a slower path. */
int b200va_quantize_mxfp8(int src_dtype, const void *dA, int fp8, void *dC, void *dS, size_t n,
                          int block, int scale_rule, void *stream);
int b200va_dequantize_mxfp8(int fp8, const void *dA, const void *dS, int dst_dtype, void *dC, size_t n,
                            int block, void *stream);
/* Scale bytes for n elements: ceil(n / block); 0 for n = 0 or a block that is not 32, 64 or 128. */
size_t b200va_mxfp8_scale_bytes(size_t n, int block);

/* ---- blockwise FP8 quantize and dequantize for H100 FP8 GEMMs (row f4) -------------------------------
 * The block-scaled operands of the H100's FP8 GEMMs (cuBLASLt's sm_90 blockwise scaling, torch's
 * ScalingType.BlockWise1x128 / BlockWise128x128): f32 scales, one per block of: */
#define B200VA_FP8_BLOCK_1X128    0   /* one scale per row and 128 columns: activations, gradients */
#define B200VA_FP8_BLOCK_128X128  1   /* one scale per 128 x 128 tile: weights                    */
/* A is row-major rows x cols, contiguous, of any B200VA_DT_* type.  C is row-major rows x cols FP8 and Ct row-major
 * cols x rows FP8 (the transposed operand); S and St hold their f32 scales.
 * Blocks.  1x128 row-wise (C, S): block (i, b) is A[i, 128b .. min(cols, 128b + 128)).  1x128 column-wise (Ct, St):
 * the 1x128 blocks of A^T, A[128b .. min(rows, 128b + 128), j].  128x128: block (p, q) is the tile
 * A[128p .., 128q ..] clipped at the edges; Ct is then exactly the byte transpose of C and St the same scales in the
 * transposed operand's layout.  The last block in each direction may be short.
 * Scale rule.  m is the largest finite |a| in the block, widened exactly; NaN and +-inf do not take part (the MXFP8
 * and _auto rule).  k = clamp(K(m), -126, 126), K(m) the largest k with m * 2^k <= max finite (448 / 57344),
 * K(0) = +inf: an all-zero block, or one with no finite element, gets k = 126.  k is the negated
 * B200VA_MX_SCALE_NOSAT exponent clamped to [-126, 126], and b200va_quantize_fp8_auto's k with margin 0.  The block's
 * scale is the f32 2^-k -- the dequantization factor the GEMM multiplies by; exact and always a normal f32.  Each
 * element is sat(RN(a * 2^k)) by exactly the rules of b200va_quantize_fp8: one rounding, the format's subnormals, no
 * FTZ, +-max finite for overflow and +-inf, NaN stays NaN, signed zeros kept.  With k unclamped no finite element
 * saturates.
 * Scale layouts (the ones torch.nn.functional.scaled_mm checks).  For an R x K operand (C: R = rows, K = cols; Ct:
 * R = cols, K = rows), with nkb = ceil(K / 128), and L4 = ceil(nkb / 4) * 4:
 *   1x128    S[b * R + r] for block b of row r: MN-major, an [R, nkb] view with strides [1, R];
 *   128x128  S[p * L4 + q] for tile (p, q), p down R and q along K: an [L4, ceil(R / 128)] view with strides
 *            [1, L4]; the padding entries q >= nkb are not written.
 * Outputs.  (dC, dS) and (dCt, dSt) are each both NULL or both non-NULL: row-wise only, column-wise only, or both.
 * Dequantize: c = RN_dst(q * s), s the f32 scale of q's block in the quantize's layout for (rows, cols, block_kind);
 * to dequantize Ct pass St and (cols, rows).  s may be any f32, not only a power of two (scales from other producers,
 * such as amax / 448, dequantize correctly): the product is exact (an FP8 value has at most 4 significant bits) and
 * rounded once to dst_dtype by b200va_convert's rules (RNE, no FTZ, overflow to +-inf).  A NaN, +-inf or 0 scale gives
 * the IEEE product.
 * Arguments, in this order: B200VA_ERR_VARIANT: bad dtype, FP8 code or block kind.  B200VA_ERR_INVALID: a pair with
 * one pointer NULL, nothing requested (or NULL dA) with rows * cols > 0, rows * cols overflowing or above 2^40
 * (dequantize: NULL dA, dS or dC with rows * cols > 0, or the size rule).  B200VA_ERR_ALIGN: dA (quantize) or dC
 * (dequantize) not aligned to its element size, dS or dSt not 4-byte aligned.  B200VA_ERR_OVERLAP: any two of A, C,
 * S, Ct and St meet, scale padding included (dequantize: C meets A or S).  A rejected call writes nothing;
 * rows == 0 or cols == 0 launches nothing.
 * Both calls are one launch each: asynchronous on `stream`, no allocation, synchronisation or memset; capturable in a
 * CUDA graph.  Fast path: cols % 128 == 0, rows % 16 == 0 and A, C and Ct on 16-byte boundaries; it reads A once
 * from HBM and writes each output byte and scale once.  Any other shape or placement gives the same bytes through a
 * per-block path that is not tuned.  Dequantize's fast path: cols % 16 == 0, A and C on 16-byte boundaries. */
/* f32 scales of a rows x cols operand: 1x128: rows * ceil(cols/128); 128x128: ceil(rows/128) * L4,
 * L4 = ceil(ceil(cols/128) / 4) * 4.  The transposed operand's count is this with rows and cols swapped.
 * 0 for rows == 0, cols == 0 or a bad kind. */
size_t b200va_fp8_blockwise_scales(size_t rows, size_t cols, int block_kind);
int b200va_quantize_fp8_blockwise(int src_dtype, const void *dA, int fp8, int block_kind, size_t rows, size_t cols,
                                  void *dC, float *dS, void *dCt, float *dSt, void *stream);
int b200va_dequantize_fp8_blockwise(int fp8, const void *dA, const float *dS, int block_kind, int dst_dtype,
                                    void *dC, size_t rows, size_t cols, void *stream);

/* ---- row-wise FP8 quantize and dequantize for H100 FP8 GEMMs (row f4) --------------------------------
 * The operands of torch's ScalingType.RowWise scaled_mm (cuBLASLt's sm_90 outer-vector scaling): one f32 scale per
 * row of each operand.  A is row-major rows x cols, contiguous, of any B200VA_DT_* type.  C is row-major rows x cols
 * FP8 and S holds rows f32 scales; Ct is row-major cols x rows FP8 (the transposed operand) and St holds cols f32
 * scales.  (dC, dS) and (dCt, dSt) are each both NULL or both non-NULL: row-wise only, column-wise only, or both.
 * Scale rule.  The blockwise rule above with one block per row (C) or per column (Ct): m is the largest finite |a| of
 * the row, widened exactly (NaN and +-inf do not take part); k = clamp(K(m), -126, 126) with _auto's margin-0 K, and
 * k = 126 for an all-zero row or one with no finite element; the stored scale is the f32 2^-k; each element is
 * sat(RN(a * 2^k)) by exactly the rules of b200va_quantize_fp8.  This is the power-of-two row-wise scale (448 / amax
 * rounded down to a power of two) with the library's clamp.  S[r] is the largest of the row's 1x128 block scales.
 * Scale layout.  S and St are plain f32 vectors: S viewed as [rows, 1] is scaled_mm's scale_a and St viewed as
 * [1, cols] its scale_b (and S as [1, rows] when C is the second operand).  A linear layer Y = X W^T takes:
 *   forward          Y  = X W^T    (C_X, S_X)   x (C_W^T, S_W)
 *   data gradient    dX = dY W     (C_dY, S_dY) x (Ct_W^T, St_W)
 *   weight gradient  dW = dY^T X   (Ct_dY, St_dY) x (Ct_X^T, St_X)
 * so one call per tensor, both sides requested, makes everything that tensor contributes.
 * Workspace.  d_work is caller-owned scratch of at least b200va_fp8_rowwise_workspace(rows, cols) bytes; its contents
 * before and after the call are unspecified.  The call allocates nothing and needs no memset.
 * Arguments, in this order: B200VA_ERR_VARIANT: bad dtype or FP8 code.  B200VA_ERR_INVALID: a pair with one pointer
 * NULL; with rows * cols > 0, nothing requested, NULL dA, rows * cols overflowing or above 2^40, NULL d_work or
 * work_bytes below the workspace size.  B200VA_ERR_ALIGN: dA not aligned to its element size, dS, dSt or d_work not
 * 4-byte aligned.  B200VA_ERR_OVERLAP: any two of A, C, S, Ct, St and the workspace meet.  A rejected call writes
 * nothing, the workspace included; rows == 0 or cols == 0 launches nothing.
 * Quantize is three launches chained by programmatic dependent launch (the 1x128 block maxima of the requested sides
 * into the workspace, their reduction to S and St, the cast), asynchronous on `stream` and capturable in a CUDA graph.
 * Fast path: cols % 128 == 0, rows % 16 == 0 and A, C and Ct on 16-byte boundaries; it reads A twice (the second
 * time mostly from HBM) and writes each output byte and scale once.  Any other shape or placement gives the same
 * bytes through a path that is not tuned.
 * Dequantize: c = RN_dst(q * S[r]), one scale per row, S any f32 (not only a power of two): the product is exact and
 * rounded once by b200va_convert's rules, as in b200va_dequantize_fp8_blockwise, whose argument rules it follows (S
 * holds rows scales).  To dequantize Ct pass St and (cols, rows).  One launch; fast path: cols % 16 == 0, A and C on
 * 16-byte boundaries. */
/* Workspace bytes: 4 * (rows * ceil(cols/128) + cols * ceil(rows/128)); 0 for rows == 0 or cols == 0. */
size_t b200va_fp8_rowwise_workspace(size_t rows, size_t cols);
int b200va_quantize_fp8_rowwise(int src_dtype, const void *dA, int fp8, size_t rows, size_t cols,
                                void *dC, float *dS, void *dCt, float *dSt,
                                void *d_work, size_t work_bytes, void *stream);
int b200va_dequantize_fp8_rowwise(int fp8, const void *dA, const float *dS, int dst_dtype,
                                  void *dC, size_t rows, size_t cols, void *stream);

/* ---- stochastic rounding from f32 (row f4) ------------------------------------------------------
 * Narrowing that keeps, in expectation, what round-to-nearest drops: an f32 value rounds to one of its two
 * neighbours in the destination with probability given by its position between them, so an update smaller than
 * half an ulp of the narrow value survives on average.  The random bits come from a counter-based generator, so the
 * bytes depend only on the value, the seed and the element's global index.
 * Random bits.  Element i has the global index m = first + i, taken mod 2^64.  splitmix64(z) is the mixing step of the
 * counter generator above: z += 0x9E3779B97F4A7C15, z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9,
 * z = (z ^ (z >> 27)) * 0x94D049BB133111EB, z ^= z >> 31.  key = splitmix64(seed) and w_j = splitmix64(key + j) (mod
 * 2^64).  r_m is the low 32 bits of w_(m>>1) when m is even and the high 32 bits when m is odd: one hash serves two
 * adjacent global indices.  Hashing the seed first keeps these bits unrelated to what b200va_fill_ctr_f32 makes from
 * the same seed.
 * Rounding.  y = a_i for bf16/f16 and y = a_i * 2^scale_exp for FP8.  D is the destination's set of values, with its
 * subnormals and with the exponent range unbounded above.  For finite nonzero y: lo is the element of D nearest y
 * toward zero and hi the next element of D away from zero; f = (|y| - |lo|) / (|hi| - |lo|), in [0, 1), and
 * t = floor(f * 2^32).  The result is hi if t + r_m >= 2^32, else lo, with y's sign (a zero result is +-0 with y's
 * sign).  Then bf16/f16: a magnitude beyond max finite is +-inf, and +-inf stays +-inf (b200va_convert's overflow
 * rule).  FP8: |y| beyond max finite, +-inf included, gives +-max finite (448 / 57344), as b200va_quantize_fp8 does.
 * +-0 stays +-0; a NaN gives a NaN.  No FTZ on either side: f32 subnormal sources and the destination's subnormals
 * take part.
 * Consequences:
 *   - A y already in D never moves.
 *   - Where neither overflow nor saturation applies, the expected result differs from y by less than 2^-32 of the
 *     gap hi - lo.
 *   - The result depends only on (a_i, seed, first + i, scale_exp, destination): not on n, on where A or C sit, on how
 *     the array is split across calls (call k with first + offset_k on its slice gives the matching bytes), or on
 *     graph replay.
 *   - For f32 -> bf16 with y normal, t is the low 16 bits of y's pattern shifted left by 16, and the rule is the
 *     familiar idiom: add the high 16 bits of r_m to the f32 pattern and clear its low 16 bits.
 * Arguments, in this order with these codes, as in b200va_convert / b200va_quantize_fp8:
 * B200VA_ERR_VARIANT: dst_dtype not B200VA_DT_F16 / B200VA_DT_BF16, or fp8 not a B200VA_F8_* code.
 * B200VA_ERR_INVALID: scale_exp outside [-126, 126], NULL dA/dC with n > 0, n > 2^40.  B200VA_ERR_ALIGN: dA not
 * 4-byte aligned, dC not aligned to its element size, d_amax not 8-byte aligned.  B200VA_ERR_OVERLAP: C meets A,
 * or d_amax meets A or C.  A rejected call writes nothing; n = 0 writes nothing.  d_amax (may be NULL)
 * max-accumulates max_i |a_i| exactly as in b200va_quantize_fp8.
 * Asynchronous on `stream`: one kernel launch, no allocation, synchronisation or memset; capturable in a CUDA graph. */
/* c[i] = a[i] stochastically rounded to dst_dtype (B200VA_DT_F16 or B200VA_DT_BF16) */
int b200va_convert_sr_f32(const float *dA, int dst_dtype, void *dC, size_t n,
                          uint64_t seed, uint64_t first, void *stream);
/* c[i] = sat(SR(a[i] * 2^scale_exp)) to E4M3 / E5M2, d_amax as in b200va_quantize_fp8 (may be NULL) */
int b200va_quantize_fp8_sr_f32(const float *dA, int fp8, void *dC, size_t n, int scale_exp,
                               uint64_t seed, uint64_t first, double *d_amax, void *stream);

/* ---- reproducible dot product (row f4) --------------------------------------------------
 * *d_out = sum_i a_i b_i as a binary64 value in device memory, written asynchronously on `stream`
 * (not rounded to the storage type; dtype is a B200VA_DT_* code).  Every operand is widened
 * exactly to f64 (f16/bf16 as the stream ops widen them, no FTZ: f32 and f16 subnormals stay).
 * The result is a function of the values and n only, defined by three rules:
 *   1. Lane chain: the elements i of chunk k with the same i mod LANES form one lane, which
 *      accumulates them in increasing index order: acc = +0.0; acc = fma(a_i, b_i, acc) in binary64
 *      RNE.  For f32/f16/bf16 the product is exact in f64, so this is acc + a_i*b_i rounded once;
 *      for f64 it is a true fma.
 *   2. Chunk value: the LANES lane values summed as a pairwise tree over aligned dyadic blocks (the
 *      value of an aligned block of 2^l entries is the sum of its two halves).  A lane with no
 *      elements, in the last chunk, is +0.0.
 *   3. Total: the ceil(n / CHUNK) chunk values summed with the same aligned dyadic tree; where a
 *      block's upper half is empty, its value is its lower half.  For n = 0 the result is +0.0.
 * Consequences:
 *   - The result is never -0.0: the chain starts at +0 and RNE never makes -0 from a sum that is not
 *     (-0) + (-0).  So "empty lane = +0.0" and "empty lane = absent" give the same bits.
 *   - The aligned dyadic tree decomposes: any aligned block can be reduced by a different CTA or
 *     launch and combined later, so how chunks and lanes map onto the GPU does not change the bits.
 *   - The result is the same at every element offset and any relative alignment of A and B.
 * Arguments: dA == dB is legal (a sum of squares).  d_workspace is device scratch of at least
 * b200va_dot_workspace_bytes(n) bytes (NULL allowed when that is 0); only those bytes are written.
 * B200VA_ERR_VARIANT: bad dtype.  B200VA_ERR_INVALID: NULL d_out, NULL dA/dB/d_workspace with n > 0,
 * workspace_bytes too small, n > 2^40.  B200VA_ERR_ALIGN: dA/dB not aligned to the element size,
 * d_out/d_workspace not 8-byte aligned.  B200VA_ERR_OVERLAP: d_out or the workspace overlapping A, B
 * or each other.  The call never allocates, synchronises or memsets, and is capturable in a CUDA graph:
 * it is two or more kernel launches on `stream` (a pass over the chunks, then the tree over their
 * values), the second and later ones behind a programmatic dependency on the one before. */
#define B200VA_DOT_LANES 2048          /* elements i of a chunk with the same i mod LANES form one lane   */
#define B200VA_DOT_CHUNK 65536         /* chunk k = indices [k*CHUNK, min(n, (k+1)*CHUNK))                */
/* Device scratch b200va_dot needs for n elements: 8 * ceil(n / B200VA_DOT_CHUNK) bytes (0 for n = 0). */
size_t b200va_dot_workspace_bytes(size_t n);
int b200va_dot(int dtype, const void *dA, const void *dB, size_t n, double *d_out,
               void *d_workspace, size_t workspace_bytes, void *stream);

/* ---- ceiling probes (measurement aids; not part of the reference's surface) -------------
 * The production launch geometry with one side of the add's traffic removed, so a harness can
 * measure on the spot what the HBM gives each kind of stream (bench.py reports the add as a
 * fraction of the READ2 rate).  n is rounded down to a multiple of 4; pointers 16-byte aligned.
 *   READ2  load A and B, store one float per CTA into C (8 B/element read)
 *   FILL   C = 1.0f, nothing is read                       (4 B/element written)
 *   COPY   C = A                                            (4 B read + 4 B written per element) */
#define B200VA_PROBE_READ2  0
#define B200VA_PROBE_FILL   1
#define B200VA_PROBE_COPY   2
int b200va_probe_f32(int kind, const float *dA, const float *dB, float *dC, size_t n, void *stream);

/* ---- shard arithmetic (8(e)): contiguous equal shards, starts on 16-byte multiples --- */
int b200va_shard_range(size_t n, int world, int rank, size_t *begin, size_t *end);

#ifdef __cplusplus
}
#endif
#endif /* B200VA_H */
