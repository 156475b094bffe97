// b200va_fp8.cuh -- b200va_quantize_fp8 and b200va_dequantize_fp8 (include/b200va.h): casts between f32, f64,
// f16, bf16 and the two OCP FP8 formats, with a power-of-two scale 2^k and an optional fused amax.
//
//   quantize    c[i] = sat(RN(a[i] 2^k))   rounded once to E4M3 / E5M2, saturating at +-max finite
//   dequantize  c[i] = RN(a[i] 2^-k)       rounded once to the destination, overflow to +-inf
//
// One kernel per non-FP8 type, fp8_quant_vec<SRC> and fp8_dequant_vec<DST>, each carrying a body per format that a
// uniform argument picks at the top (16 pairs in 8 kernels).  The same kernels carry b200va_quantize_fp8_auto and
// b200va_dequantize_fp8_auto, whose scale exponent k lives in device memory:
//   amax pass   fp8_quant_vec with C = nullptr: the largest finite |a_i| max-accumulated into *amax, nothing stored
//   quantize    fp8_quant_vec with amax_in: k = auto_scale_exp(*amax_in), read after the dependency wait, and
//               written to *k_out by one thread
//   dequantize  fp8_dequant_vec with k_in: k = *k_in, read after the dependency wait; outside [-126, 126] the
//               scale is a NaN
// How one rounding is reached:
// - f32, f16, bf16 sources widen exactly to f32 and are scaled there; cvt.rn.satfinite.{e4m3x2,e5m2x2}.f32 rounds.
//   Where the f32 product is inexact (below 2^-126) the exact value lies far below half the smallest FP8
//   subnormal, so the result is +-0 either way; where it overflows, the exact value saturates either way.
// - f64 sources are scaled in f64 and rounded to f32 with round-to-odd (cvt.rz, then the last bit set when that
//   was inexact).  Round-to-odd to 24 bits followed by RN to p <= 22 bits rounds once (Boldo-Melquiond).
// - Dequantize widens with cvt.rn.f16x2.{e4m3x2,e5m2x2} (exact), then to f32 and scales there (exact: FP8
//   values have at most 4 significant bits and the smallest one times 2^-126 is a multiple of 2^-149), then
//   rounds once to f16 / bf16.  An f64 destination widens to f64 and scales there.
//
// Layout.  Quantize works in groups of G = 16 elements (the FP8 side is one 16-byte vector, the source side
// sizeof SRC of them), like convert_vec.  Dequantize gives each lane a slice of 16 / sizeof DST elements, so its
// widened result is one 16-byte vector and a warp's store covers 512 contiguous bytes; the loads are 8, 4 or 2
// bytes per lane.
#pragma once
#include <type_traits>

#include "b200va_convert.cuh"

namespace b200va {

enum : int { F8_E4M3 = 0, F8_E5M2 = 1, F8_COUNT = 2 };

// The format (fmt, uniform across the launch) to a template argument: f(F8) for the one that matches, so a kernel
// takes one branch at the top and both formats share it.
template <class F>
__device__ __forceinline__ void with_f8(int fmt, F f)
{
    if (fmt == F8_E4M3) f(std::integral_constant<int, F8_E4M3>{});
    else f(std::integral_constant<int, F8_E5M2>{});
}

// 2^k in DT's arithmetic type (f64 for f64, f32 otherwise), for k in [-126, 126] (a normal number either way).
template <int DT>
__device__ __forceinline__ typename dt_traits<DT>::scalar pow2(int k)
{
    if constexpr (DT == DT_F64) return __longlong_as_double(static_cast<long long>(1023 + k) << 52);
    else return __int_as_float((127 + k) << 23);
}

// Two f32 rounded (RN, saturating at +-max finite) to FP8: lo in bits 0..7, hi in bits 8..15.
template <int F8>
__device__ __forceinline__ uint32_t f8x2_from_f32(float lo, float hi)
{
    unsigned short r;
    if constexpr (F8 == F8_E4M3) asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
    else asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
    return r;
}

// Two FP8 values (bits 0..7 and 8..15 of v) widened exactly to f16: lo in bits 0..15, hi in bits 16..31.
template <int F8>
__device__ __forceinline__ uint32_t f16x2_from_f8x2(uint32_t v)
{
    uint32_t r;
    const unsigned short s = static_cast<unsigned short>(v);
    if constexpr (F8 == F8_E4M3) asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(r) : "h"(s));
    else asm("cvt.rn.f16x2.e5m2x2 %0, %1;" : "=r"(r) : "h"(s));
    return r;
}

// An f64 rounded to f32 with round-to-odd: toward zero, then the last bit set if that was inexact.  NaN stays
// NaN, +-inf stays +-inf, and a finite value past FLT_MAX gives +-FLT_MAX (which saturates all the same).
__device__ __forceinline__ float f32_round_odd(double x)
{
    float r;
    asm("cvt.rz.f32.f64 %0, %1;" : "=f"(r) : "d"(x));
    return __uint_as_float(__float_as_uint(r) | static_cast<uint32_t>(static_cast<double>(r) != x));
}

// ---- quantize ---------------------------------------------------------------------------------------------
// The amax a thread tracks: the largest |a_i| bit pattern, as f32 bits for the f32 family (the exact widening
// keeps the order) and as f64 bits for f64.  Every NaN pattern sorts above +inf.
template <int SRC>
using amax_bits_t = std::conditional_t<SRC == DT_F64, unsigned long long, uint32_t>;

// The magnitude bit pattern of element e of the source words s if it is finite, else 0 (NaN and +-inf do not take
// part in a finite maximum): f32 bits for the f32 family, f64 bits for f64, as amax_bits_t.
template <int SRC>
__device__ __forceinline__ amax_bits_t<SRC> finite_mag(const uint32_t* s, int e)
{
    if constexpr (SRC == DT_F64) {
        const unsigned long long v = static_cast<unsigned long long>(__double_as_longlong(elem_f64(s, e))) & 0x7fffffffffffffffull;
        return v < 0x7ff0000000000000ull ? v : 0ull;
    } else {
        const uint32_t v = __float_as_uint(elem_f32<SRC>(s, e)) & 0x7fffffffu;
        return v < 0x7f800000u ? v : 0u;
    }
}

// The scale exponent b200va_quantize_fp8_auto takes from the value m its amax pass left: with m = s 2^e (s in
// [1, 2)), K = emax - e - (s > 1.75) is the largest k with m 2^k <= max finite = 1.75 2^emax, and k = K - margin
// clamped to [-126, 126].  An f64 subnormal m or m = +0 reads as e = -1023, which clamps to 126 as K(0) = +inf
// does.  m whose pattern is not that of a finite value with the sign bit clear (a NaN, +inf, or a negative value
// or -0.0 the caller left, which the amax pass's unsigned maximum keeps) gives 0.
__device__ __forceinline__ int auto_scale_exp(double m, int fmt, int margin)
{
    const unsigned long long b = static_cast<unsigned long long>(__double_as_longlong(m));
    if (b >= 0x7ff0000000000000ull) return 0;
    const int K = (fmt == F8_E4M3 ? 8 : 15) - (static_cast<int>(b >> 52) - 1023) - ((b & 0x000fffffffffffffull) > 0x000c000000000000ull);
    return min(max(K - margin, -126), 126);
}

// Elements e0 and e0 + 1 of the source words s, scaled by 2^k0 and 2^k1 and rounded to two FP8 bytes (bits 0..15); m
// takes their magnitudes.  With `one`, only e0 (the high byte is 0).
template <int SRC, int F8, bool ONE = false>
__device__ __forceinline__ uint32_t quant_pair(const uint32_t* s, int e0, int k0, int k1, amax_bits_t<SRC>& m)
{
    float q[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < (ONE ? 1 : 2); ++j) {
        if constexpr (SRC == DT_F64) {
            const double x = elem_f64(s, e0 + j);
            m = max(m, static_cast<unsigned long long>(__double_as_longlong(x)) & 0x7fffffffffffffffull);
            q[j] = f32_round_odd(__dmul_rn(x, pow2<SRC>(j ? k1 : k0)));
        } else {
            const float x = elem_f32<SRC>(s, e0 + j);
            m = max(m, __float_as_uint(x) & 0x7fffffffu);
            q[j] = __fmul_rn(x, pow2<SRC>(j ? k1 : k0));
        }
    }
    return f8x2_from_f32<F8>(q[0], q[1]);
}

// The same with one scale exponent k for both elements.
template <int SRC, int F8, bool ONE = false>
__device__ __forceinline__ uint32_t quant_pair(const uint32_t* s, int e0, int k, amax_bits_t<SRC>& m)
{
    return quant_pair<SRC, F8, ONE>(s, e0, k, k, m);
}

// One group: the 16 elements in the source words s, scaled by 2^k and rounded to the 16 FP8 bytes of the words d; m
// takes their magnitudes.
template <int SRC, int F8>
__device__ __forceinline__ void quant_group(const uint32_t* s, int k, amax_bits_t<SRC>& m, uint32_t* d)
{
#pragma unroll
    for (int w = 0; w < 4; ++w)
        d[w] = quant_pair<SRC, F8>(s, 4 * w, k, m) | (quant_pair<SRC, F8>(s, 4 * w + 2, k, m) << 16);
}

// One element at p (element-size aligned), the same way: its FP8 byte.
template <int SRC, int F8>
__device__ __forceinline__ unsigned char quant_elem(const unsigned char* p, int k, amax_bits_t<SRC>& m)
{
    uint32_t s[2];
    ld_elem<dt_traits<SRC>::size>(p, s);
    return static_cast<unsigned char>(quant_pair<SRC, F8, true>(s, 0, k, m));
}

template <class T>
__device__ __forceinline__ T warp_max(T v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// The CTA's magnitudes m (every thread's) max-accumulated into *amax as f64 bits with one atomic; called by every
// thread of the CTA, after the dependency wait like every other access.
template <int SRC>
__device__ __forceinline__ void cta_amax(double* amax, amax_bits_t<SRC> m)
{
    __shared__ unsigned long long part[32];
    unsigned long long v;
    if constexpr (SRC == DT_F64) v = m;
    else v = static_cast<unsigned long long>(__double_as_longlong(static_cast<double>(__uint_as_float(m)))) & 0x7fffffffffffffffull;
    v = warp_max(v);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (unsigned w = 1; w < blockDim.x / 32; ++w) v = max(v, part[w]);
        atomicMax(reinterpret_cast<unsigned long long*>(amax), v);
    }
}

// Quantize's body after the dependency wait: elements [head, head + 16 ngroups) are the vector body, one group of 16
// per unit, on 16-byte boundaries in A and in C; the others go through cast_edges.
template <int SRC, int F8>
__device__ __forceinline__ void quant_body(const unsigned char* a, unsigned char* c, size_t n, size_t head,
                                           size_t ngroups, int unroll, int k, amax_bits_t<SRC>& m)
{
    constexpr int ES = dt_traits<SRC>::size;      // also the 16-byte source vectors per group
    const unsigned char* ab = a + head * ES;
    unsigned char* cb = c + head;
    cast_tiles(unroll, ngroups, [=](size_t g) { return ld_vecs<ES>(ab, g); }, [&](size_t g, const vecs<ES>& in) {
        uint32_t s[4 * ES], d[4];
        unpack<ES>(in.v, s);
        quant_group<SRC, F8>(s, k, m, d);
        stg128_bits<ST_NA>(cb + g * 16, u32x4{d[0], d[1], d[2], d[3]});
    });
    cast_edges(n, head, head + ngroups * 16, [&](size_t e) { c[e] = quant_elem<SRC, F8>(a + e * ES, k, m); });
}

// The amax pass's body after the dependency wait: quant_body's tiles and edges over A alone (elements [head, head +
// 16 ngroups) on 16-byte boundaries in A), each element's finite magnitude folded into m and nothing stored.
template <int SRC>
__device__ __forceinline__ void amax_body(const unsigned char* a, size_t n, size_t head, size_t ngroups, int unroll,
                                          amax_bits_t<SRC>& m)
{
    constexpr int ES = dt_traits<SRC>::size;
    const unsigned char* ab = a + head * ES;
    cast_tiles(unroll, ngroups, [=](size_t g) { return ld_vecs<ES>(ab, g); }, [&](size_t, const vecs<ES>& in) {
        uint32_t s[4 * ES];
        unpack<ES>(in.v, s);
#pragma unroll
        for (int e = 0; e < 16; ++e) m = max(m, finite_mag<SRC>(s, e));
    });
    cast_edges(n, head, head + ngroups * 16, [&](size_t e) {
        uint32_t s[2];
        ld_elem<ES>(a + e * ES, s);
        m = max(m, finite_mag<SRC>(s, 0));
    });
}

// ---- quantize-transpose ---------------------------------------------------------------------------------
// b200va_quantize_fp8_transpose: A is rows x cols (row-major, n = rows cols), C gets quant_body's bytes and Ct
// (cols x rows, row-major) their transpose, Ct[j rows + i] = C[i cols + j], in one pass over A.
//
// Tiled path (rows and cols multiples of 16, A, C and Ct on 16-byte boundaries): tiles of T8 x T8 elements, row-major
// over the matrix and grid-strided, FP8T_THREADS = (T8 / 16) T8 threads per CTA.  Thread t first takes group t % 4
// of tile row t / 4: it rounds those 16 elements with quant_group, stores the 16 bytes to C, and stores each byte
// into the shared-memory tile, which holds the tile transposed (tile row j is Ct's row, tile column i is A's row).
// After the barrier it takes tile row j = t / 4, columns 16 (t % 4) .. + 15: one 16-byte shared load and one 16-byte
// store to Ct.  So 4 lanes cover the 64 bytes of a Ct row (two whole 32-byte sectors) and a warp 8 Ct rows.  The
// tile is swizzled: 16-byte chunk h of tile row j sits at chunk h ^ (j / 16), so the byte stores of the 4 lanes of a
// group (16 tile rows apart) fall in 4 different banks, and a quarter warp's 16-byte loads cover 128 contiguous
// bytes.  Tiles on the right and bottom edges are partial in steps of 16.  Two tile buffers alternate, so one
// barrier per tile keeps a tile's reads apart from the writes two tiles later.
//
// Element path (every other shape or placement): cast_edges with head = n; element e to C[e] and to
// Ct[(e % cols) rows + e / cols].  For correctness, not speed.
constexpr int FP8T_TILE = 64;                                         // T8
constexpr int FP8T_THREADS = FP8T_TILE / 16 * FP8T_TILE;              // 256
constexpr int FP8T_SMEM = 2 * FP8T_TILE * FP8T_TILE;                  // two tile buffers, 8 KiB (dynamic)

// The tiled path's body after the dependency wait, one format, n = rows cols elements, k the scale exponent.
template <int SRC, int F8>
__device__ __forceinline__ void quant_t_tiles(const unsigned char* a, unsigned char* c, unsigned char* ct, size_t rows,
                                              size_t cols, int k, amax_bits_t<SRC>& m)
{
    constexpr int ES = dt_traits<SRC>::size, T8 = FP8T_TILE;
    extern __shared__ __align__(16) unsigned char fp8t_tile[];
    // at most 2^36 / T8 tile columns and 2^40 / (16 T8) tiles (n <= 2^40, rows and cols multiples of 16)
    const unsigned tiles_c = static_cast<unsigned>((cols + T8 - 1) / T8);
    const unsigned ntiles = static_cast<unsigned>((rows + T8 - 1) / T8) * tiles_c;
    const unsigned r = threadIdx.x / 4, q = threadIdx.x % 4;          // phase 1: tile row, group; phase 2: column, rows
    unsigned buf = 0;
    for (unsigned t = blockIdx.x; t < ntiles; t += gridDim.x, buf ^= T8 * T8) {
        const size_t i0 = static_cast<size_t>(t / tiles_c) * T8, j0 = static_cast<size_t>(t % tiles_c) * T8;
        const unsigned tr = static_cast<unsigned>(min(rows - i0, size_t{T8})), tc = static_cast<unsigned>(min(cols - j0, size_t{T8}));
        unsigned char* tile = fp8t_tile + buf;
        if (r < tr && 16 * q < tc) {
            const size_t e = (i0 + r) * cols + j0 + 16 * q;
            uint32_t s[4 * ES], d[4];
            unpack<ES>(ld_vecs<ES>(a + e * ES, 0).v, s);
            quant_group<SRC, F8>(s, k, m, d);
            stg128_bits<ST_NA>(c + e, u32x4{d[0], d[1], d[2], d[3]});
            // byte b goes to tile column 16 q + b, at row r of its swizzled chunk
            unsigned char* col = tile + 16 * q * T8 + 16 * ((r / 16) ^ q) + r % 16;
#pragma unroll
            for (int b = 0; b < 16; ++b) col[b * T8] = static_cast<unsigned char>(d[b / 4] >> (8 * (b % 4)));
        }
        __syncthreads();
        if (r < tc && 16 * q < tr)
            stg128_bits<ST_NA>(ct + (j0 + r) * rows + i0 + 16 * q,
                               *reinterpret_cast<const u32x4*>(tile + r * T8 + 16 * (q ^ (r / 16))));
    }
}

// The transposed body after the dependency wait: the tiled path for ngroups = n / 16 (head = 0), else the element
// path (head = n, ngroups = 0).
template <int SRC, int F8>
__device__ __forceinline__ void quant_t_body(const unsigned char* a, unsigned char* c, unsigned char* ct, size_t n,
                                             size_t cols, size_t head, size_t ngroups, int k, amax_bits_t<SRC>& m)
{
    constexpr int ES = dt_traits<SRC>::size;
    const size_t rows = n / cols;
    if (ngroups) quant_t_tiles<SRC, F8>(a, c, ct, rows, cols, k, m);
    // e = i cols + j without a 64-bit division, whose call would raise the kernel's register count: e < 2^40, so
    // e / cols in f64 (by the rounded reciprocal) is within 2^-11 of the quotient, and i is its truncation corrected
    // by at most one.
    const double rc = __drcp_rn(static_cast<double>(cols));
    cast_edges(n, head, head + ngroups * 16, [&](size_t e) {
        const unsigned char b = quant_elem<SRC, F8>(a + e * ES, k, m);
        c[e] = b;
        long long i = static_cast<long long>(static_cast<double>(e) * rc);
        long long j = static_cast<long long>(e) - i * static_cast<long long>(cols);
        if (j < 0) { --i; j += cols; }
        else if (j >= static_cast<long long>(cols)) { ++i; j -= cols; }
        ct[j * rows + i] = b;
    });
}

// One kernel per source type, the format picking one of its two bodies (with_f8).  unroll (1 or 2) and prefetch_first
// are the launch's geometry, as in convert_vec.  With amax, each CTA max-accumulates its largest |a_i| (as f64 bits)
// into *amax with one atomic, after the dependency wait like every other access; every body reaches that one atomic.
// Without C the kernel is b200va_quantize_fp8_auto's amax pass (amax_body: finite magnitudes only, fmt and k unused).
// With amax_in, k is auto_scale_exp(*amax_in, fmt, margin) instead of the argument, and thread 0 of CTA 0 writes it
// to *k_out.  With Ct the kernel is b200va_quantize_fp8_transpose's (quant_t_body; A has `cols` columns, and the
// launch gives FP8T_THREADS threads and FP8T_SMEM bytes of dynamic shared memory on the tiled path).
template <int SRC>
__global__ void fp8_quant_vec(const void* A, void* C, size_t n, size_t head, size_t ngroups, int unroll,
                              int prefetch_first, int fmt, int k, double* amax, const double* amax_in, int margin,
                              int32_t* k_out, void* Ct, size_t cols)
{
    const unsigned char* a = static_cast<const unsigned char*>(A);
    unsigned char* c = static_cast<unsigned char*>(C);
    unsigned char* ct = static_cast<unsigned char*>(Ct);
    prefetch_first_tile<16, dt_traits<SRC>::size>(prefetch_first, a, head, ngroups, unroll);
    pdl_wait();

    amax_bits_t<SRC> m = 0;
    if (!c) {
        amax_body<SRC>(a, n, head, ngroups, unroll, m);
    } else {
        if (amax_in) {
            k = auto_scale_exp(*amax_in, fmt, margin);
            if (blockIdx.x == 0 && threadIdx.x == 0) *k_out = k;
        }
        if (ct) with_f8(fmt, [&](auto F8) { quant_t_body<SRC, F8>(a, c, ct, n, cols, head, ngroups, k, m); });
        else with_f8(fmt, [&](auto F8) { quant_body<SRC, F8>(a, c, n, head, ngroups, unroll, k, m); });
    }
    if (amax) cta_amax<SRC>(amax, m);
}

// ---- dequantize -------------------------------------------------------------------------------------------
// W = 16 / sizeof DST FP8 values, in the low bytes of v, to one 16-byte vector of DST scaled by s (a power of two,
// or a NaN), in f64 for an f64 destination and in f32 otherwise.
template <int F8, int DST>
__device__ __forceinline__ u32x4 dequant_slice(unsigned long long v, typename dt_traits<DST>::scalar s)
{
    uint32_t d[4];
    if constexpr (DST == DT_F64) {
        const uint32_t h = f16x2_from_f8x2<F8>(static_cast<uint32_t>(v));
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const double x = __dmul_rn(static_cast<double>(widen_f16(h >> (16 * e) & 0xffffu)), s);
            d[2 * e] = static_cast<uint32_t>(__double2loint(x));
            d[2 * e + 1] = static_cast<uint32_t>(__double2hiint(x));
        }
    } else {
#pragma unroll
        for (int p = 0; p < (DST == DT_F32 ? 2 : 4); ++p) {
            const uint32_t h = f16x2_from_f8x2<F8>(static_cast<uint32_t>(v >> (16 * p)));
            const float lo = __fmul_rn(widen_f16(h & 0xffffu), s), hi = __fmul_rn(widen_f16(h >> 16), s);
            if constexpr (DST == DT_F32) { d[2 * p] = __float_as_uint(lo); d[2 * p + 1] = __float_as_uint(hi); }
            else d[p] = narrow2_f32<DST>(lo, hi);
        }
    }
    return u32x4{d[0], d[1], d[2], d[3]};
}

// A dequantize unit as a tile holds it: the slice's FP8 bytes and its scale.
template <int DST>
struct dequant_unit { unsigned long long v; typename dt_traits<DST>::scalar scale; };

// Dequantize's body after the dependency wait, per tensor and block-scaled: elements [head, head + 16 ngroups) are the
// vector body, whose units are slices of W = 16 / sizeof DST elements (sizeof DST per group of 16), so lane-consecutive
// 16-byte stores; the others go through cast_edges.  scale_of(e) is the scale of the slice, or the element, that
// starts at element e; a tile calls it beside the load of the FP8 bytes, so what it reads is in flight before the
// tile's first store.
template <int F8, int DST, class ScaleOf>
__device__ __forceinline__ void dequant_body(const unsigned char* a, unsigned char* c, size_t n, size_t head,
                                             size_t ngroups, int unroll, ScaleOf scale_of)
{
    constexpr int ES = dt_traits<DST>::size, W = 16 / ES;
    const unsigned char* ab = a + head;
    unsigned char* cb = c + head * ES;
    cast_tiles(unroll, ngroups * ES,
               [=](size_t u) { return dequant_unit<DST>{ld_bits<W>(ab + u * W), scale_of(head + u * W)}; },
               [=](size_t u, const dequant_unit<DST>& in) {
        stg128_bits<ST_NA>(cb + u * 16, dequant_slice<F8, DST>(in.v, in.scale));
    });
    cast_edges(n, head, head + ngroups * 16, [=](size_t e) {
        const u32x4 r = dequant_slice<F8, DST>(ld_bits<1>(a + e), scale_of(e));
        st_elem<ES>(c + e * ES, r.x, r.y);
    });
}

// One kernel per destination type, the format picked at the top as in fp8_quant_vec; every slice has the scale 2^-k.
// With k_in, k is *k_in, read once per thread after the dependency wait, and a k outside [-126, 126] scales by a NaN.
template <int DST>
__global__ void fp8_dequant_vec(const void* A, void* C, size_t n, size_t head, size_t ngroups, int unroll,
                                int prefetch_first, int fmt, int k, const int32_t* k_in)
{
    using S = typename dt_traits<DST>::scalar;
    constexpr int ES = dt_traits<DST>::size;
    const unsigned char* a = static_cast<const unsigned char*>(A);
    unsigned char* c = static_cast<unsigned char*>(C);
    prefetch_first_tile<16 / ES, 1>(prefetch_first, a, head, ngroups * ES, unroll);
    pdl_wait();

    S s = pow2<DST>(-k);
    if (k_in) {
        const int kd = *k_in;
        if constexpr (DST == DT_F64) s = kd >= -126 && kd <= 126 ? pow2<DST>(-kd) : __longlong_as_double(0x7ff8000000000000ll);
        else s = kd >= -126 && kd <= 126 ? pow2<DST>(-kd) : __uint_as_float(0x7fc00000u);
    }
    with_f8(fmt, [=](auto F8) { dequant_body<F8, DST>(a, c, n, head, ngroups, unroll, [=](size_t) { return s; }); });
}

}  // namespace b200va
