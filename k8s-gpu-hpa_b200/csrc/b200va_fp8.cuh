// b200va_fp8.cuh -- b200va_quantize_fp8 and b200va_dequantize_fp8 (include/b200va.h): casts between f32, f64,
// f16, bf16 and the two OCP FP8 formats, with a power-of-two scale 2^k and an optional fused amax.
//
//   quantize    c[i] = sat(RN(a[i] 2^k))   rounded once to E4M3 / E5M2, saturating at +-max finite
//   dequantize  c[i] = RN(a[i] 2^-k)       rounded once to the destination, overflow to +-inf
//
// One kernel per non-FP8 type, fp8_quant_vec<SRC> and fp8_dequant_vec<DST>, each carrying a body per format that a
// uniform argument picks at the top (16 pairs in 8 kernels).  How one rounding is reached:
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

// 2^k as an f32 / f64, for k in [-126, 126] (a normal number either way).
__device__ __forceinline__ float pow2_f32(int k) { return __int_as_float((127 + k) << 23); }
__device__ __forceinline__ double pow2_f64(int k) { return __longlong_as_double(static_cast<long long>(1023 + k) << 52); }

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

// Elements e0 and e0 + 1 of the source words s, scaled by 2^k and rounded to two FP8 bytes (bits 0..15); m takes
// their magnitudes.  With `one`, only e0 (the high byte is 0).
template <int SRC, int F8, bool ONE = false>
__device__ __forceinline__ uint32_t quant_pair(const uint32_t* s, int e0, int k, amax_bits_t<SRC>& m)
{
    float q[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < (ONE ? 1 : 2); ++j) {
        if constexpr (SRC == DT_F64) {
            const double x = elem_f64(s, e0 + j);
            m = max(m, static_cast<unsigned long long>(__double_as_longlong(x)) & 0x7fffffffffffffffull);
            q[j] = f32_round_odd(__dmul_rn(x, pow2_f64(k)));
        } else {
            const float x = elem_f32<SRC>(s, e0 + j);
            m = max(m, __float_as_uint(x) & 0x7fffffffu);
            q[j] = __fmul_rn(x, pow2_f32(k));
        }
    }
    return f8x2_from_f32<F8>(q[0], q[1]);
}

template <class T>
__device__ __forceinline__ T warp_max(T v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
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
#pragma unroll
        for (int w = 0; w < 4; ++w)
            d[w] = quant_pair<SRC, F8>(s, 4 * w, k, m) | (quant_pair<SRC, F8>(s, 4 * w + 2, k, m) << 16);
        stg128_bits<ST_NA>(cb + g * 16, u32x4{d[0], d[1], d[2], d[3]});
    });
    cast_edges(n, head, head + ngroups * 16, [&](size_t e) {
        const unsigned long long x = ld_bits<ES>(a + e * ES);
        const uint32_t s[2] = {static_cast<uint32_t>(x), static_cast<uint32_t>(x >> 32)};
        st_bits<1>(c + e, quant_pair<SRC, F8, true>(s, 0, k, m));
    });
}

// One kernel per source type; the format (fmt, uniform) picks one of two bodies at the top, so both formats share
// a kernel.  unroll (1 or 2) and prefetch_first are the launch's geometry, as in convert_vec.  With amax, each CTA
// max-accumulates its largest |a_i| (as f64 bits) into *amax with one atomic, after the dependency wait like every
// other access.
template <int SRC>
__global__ void fp8_quant_vec(const void* A, void* C, size_t n, size_t head, size_t ngroups, int unroll,
                              int prefetch_first, int fmt, int k, double* amax)
{
    const unsigned char* a = static_cast<const unsigned char*>(A);
    unsigned char* c = static_cast<unsigned char*>(C);
    prefetch_first_tile<16, dt_traits<SRC>::size>(prefetch_first, a, head, ngroups, unroll);
    pdl_wait();

    amax_bits_t<SRC> m = 0;
    if (fmt == F8_E4M3) quant_body<SRC, F8_E4M3>(a, c, n, head, ngroups, unroll, k, m);
    else quant_body<SRC, F8_E5M2>(a, c, n, head, ngroups, unroll, k, m);

    if (amax) {
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
}

// ---- dequantize -------------------------------------------------------------------------------------------
// W = 16 / sizeof DST FP8 values, in the low bytes of v, to one 16-byte vector of DST scaled by 2^-k.
template <int F8, int DST>
__device__ __forceinline__ u32x4 dequant_slice(unsigned long long v, int k)
{
    uint32_t d[4];
    if constexpr (DST == DT_F64) {
        const uint32_t h = f16x2_from_f8x2<F8>(static_cast<uint32_t>(v));
        const double s = pow2_f64(-k);
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const double x = __dmul_rn(static_cast<double>(widen_f16(h >> (16 * e) & 0xffffu)), s);
            d[2 * e] = static_cast<uint32_t>(__double2loint(x));
            d[2 * e + 1] = static_cast<uint32_t>(__double2hiint(x));
        }
    } else {
        const float s = pow2_f32(-k);
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

// Dequantize's body after the dependency wait: elements [head, head + 16 ngroups) are the vector body, whose units are
// slices of W = 16 / sizeof DST elements (sizeof DST per group of 16), so lane-consecutive 16-byte stores; the others
// go through cast_edges.
template <int F8, int DST>
__device__ __forceinline__ void dequant_body(const unsigned char* a, unsigned char* c, size_t n, size_t head,
                                             size_t ngroups, int unroll, int k)
{
    constexpr int ES = dt_traits<DST>::size, W = 16 / ES;
    const unsigned char* ab = a + head;
    unsigned char* cb = c + head * ES;
    cast_tiles(unroll, ngroups * ES, [=](size_t u) { return ld_bits<W>(ab + u * W); },
               [=](size_t u, unsigned long long v) { stg128_bits<ST_NA>(cb + u * 16, dequant_slice<F8, DST>(v, k)); });
    cast_edges(n, head, head + ngroups * 16, [=](size_t e) {
        const u32x4 r = dequant_slice<F8, DST>(ld_bits<1>(a + e), k);
        st_bits<ES>(c + e * ES, r.x | static_cast<unsigned long long>(r.y) << 32);
    });
}

// One kernel per destination type, the format picked at the top as in fp8_quant_vec.
template <int DST>
__global__ void fp8_dequant_vec(const void* A, void* C, size_t n, size_t head, size_t ngroups, int unroll,
                                int prefetch_first, int fmt, int k)
{
    constexpr int ES = dt_traits<DST>::size;
    const unsigned char* a = static_cast<const unsigned char*>(A);
    unsigned char* c = static_cast<unsigned char*>(C);
    prefetch_first_tile<16 / ES, 1>(prefetch_first, a, head, ngroups * ES, unroll);
    pdl_wait();

    if (fmt == F8_E4M3) dequant_body<F8_E4M3, DST>(a, c, n, head, ngroups, unroll, k);
    else dequant_body<F8_E5M2, DST>(a, c, n, head, ngroups, unroll, k);
}

}  // namespace b200va
