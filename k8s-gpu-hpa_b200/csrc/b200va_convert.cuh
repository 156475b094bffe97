// b200va_convert.cuh -- b200va_convert (include/b200va.h): c[i] = a[i] rounded once to another of f32, f64,
// f16 and bf16 (IEEE round-to-nearest-even, no FTZ on either side, overflow to +-inf).
//
// One kernel per ordered pair of distinct types.  A thread works in groups of G = 16 / min(sizeof SRC,
// sizeof DST) elements: per group the narrow side is one 16-byte vector and the wide side 2 or 4.  The
// rounding is the hardware's, once: cvt.rn.{f16,bf16}.f64 and cvt.rn.f32.f64 from f64 (never through
// f32), the paired cvt.rn.{f16x2,bf16x2}.f32 from f32, and f16 <-> bf16 through the exact f32 widening.
// Widening is exact.  The same-type copy is not here: b200va_convert sends it to the COPY stream kernel.
#pragma once
#include "b200va_stream.cuh"

namespace b200va {

template <int SRC, int DST>
struct convert_shape {
    static_assert(SRC != DST, "a same-type convert is a COPY");
    static constexpr int ESS = dt_traits<SRC>::size, ESD = dt_traits<DST>::size;
    static constexpr int G = 16 / (ESS < ESD ? ESS : ESD);       // elements per group
    static constexpr int VS = G * ESS / 16, VD = G * ESD / 16;   // 16-byte vectors per group, each side
};

// ---- one element, from the 32-bit words of a group ------------------------------------------------
// Element e of SRC in the words w: f32/f16/bf16 widened exactly to f32, f64 as the double.
template <int SRC>
__device__ __forceinline__ float elem_f32(const uint32_t* w, int e)
{
    if constexpr (SRC == DT_F32) return __uint_as_float(w[e]);
    else if constexpr (SRC == DT_F16) return widen_f16((w[e / 2] >> (16 * (e % 2))) & 0xffffu);
    else return widen_bf16((w[e / 2] >> (16 * (e % 2))) & 0xffffu);
}

__device__ __forceinline__ double elem_f64(const uint32_t* w, int e)
{
    return __hiloint2double(static_cast<int>(w[2 * e + 1]), static_cast<int>(w[2 * e]));
}

// One f64 rounded once to f16 / bf16: the 16 bits, in the low half.
template <int DST>
__device__ __forceinline__ uint32_t narrow_f64(double x)
{
    unsigned short r;
    if constexpr (DST == DT_F16) asm("cvt.rn.f16.f64 %0, %1;" : "=h"(r) : "d"(x));
    else asm("cvt.rn.bf16.f64 %0, %1;" : "=h"(r) : "d"(x));
    return r;
}

// Two f32 rounded to f16 / bf16 in one instruction: lo in bits 0..15, hi in bits 16..31.
template <int DST>
__device__ __forceinline__ uint32_t narrow2_f32(float lo, float hi)
{
    uint32_t r;
    if constexpr (DST == DT_F16) asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    else asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}

// N elements of SRC in the words s to N elements of DST in the words d (an odd last 16-bit element
// leaves the high half of its word 0).
template <int SRC, int DST, int N>
__device__ __forceinline__ void convert_words(const uint32_t* s, uint32_t* d)
{
    if constexpr (DST == DT_F64) {
#pragma unroll
        for (int e = 0; e < N; ++e) {
            const double x = static_cast<double>(elem_f32<SRC>(s, e));
            d[2 * e] = static_cast<uint32_t>(__double2loint(x));
            d[2 * e + 1] = static_cast<uint32_t>(__double2hiint(x));
        }
    } else if constexpr (DST == DT_F32) {
#pragma unroll
        for (int e = 0; e < N; ++e) d[e] = __float_as_uint(SRC == DT_F64 ? __double2float_rn(elem_f64(s, e)) : elem_f32<SRC>(s, e));
    } else {
#pragma unroll
        for (int k = 0; k < (N + 1) / 2; ++k) {
            if constexpr (SRC == DT_F64)
                d[k] = narrow_f64<DST>(elem_f64(s, 2 * k)) | (2 * k + 1 < N ? narrow_f64<DST>(elem_f64(s, 2 * k + 1)) << 16 : 0u);
            else
                d[k] = narrow2_f32<DST>(elem_f32<SRC>(s, 2 * k), 2 * k + 1 < N ? elem_f32<SRC>(s, 2 * k + 1) : 0.f);
        }
    }
}

// One group: VS source vectors in, VD destination vectors out.
template <int SRC, int DST>
__device__ __forceinline__ void convert_group(const u32x4* in, u32x4* out)
{
    using S = convert_shape<SRC, DST>;
    uint32_t s[4 * S::VS], d[4 * S::VD];
#pragma unroll
    for (int k = 0; k < S::VS; ++k) {
        s[4 * k] = in[k].x; s[4 * k + 1] = in[k].y; s[4 * k + 2] = in[k].z; s[4 * k + 3] = in[k].w;
    }
    convert_words<SRC, DST, S::G>(s, d);
#pragma unroll
    for (int k = 0; k < S::VD; ++k) out[k] = u32x4{d[4 * k], d[4 * k + 1], d[4 * k + 2], d[4 * k + 3]};
}

// One element at byte pointers a, c (element-size aligned).
template <int SRC, int DST>
__device__ __forceinline__ void convert_elem(const unsigned char* a, unsigned char* c)
{
    using S = convert_shape<SRC, DST>;
    uint32_t s[2] = {0, 0}, d[2];
    if constexpr (S::ESS == 8) {
        const unsigned long long x = *reinterpret_cast<const unsigned long long*>(a);
        s[0] = static_cast<uint32_t>(x);
        s[1] = static_cast<uint32_t>(x >> 32);
    } else if constexpr (S::ESS == 4) {
        s[0] = *reinterpret_cast<const uint32_t*>(a);
    } else {
        s[0] = *reinterpret_cast<const unsigned short*>(a);
    }
    convert_words<SRC, DST, 1>(s, d);
    if constexpr (S::ESD == 8) *reinterpret_cast<unsigned long long*>(c) = d[0] | (static_cast<unsigned long long>(d[1]) << 32);
    else if constexpr (S::ESD == 4) *reinterpret_cast<uint32_t*>(c) = d[0];
    else *reinterpret_cast<unsigned short*>(c) = static_cast<unsigned short>(d[0]);
}

// ---- the vector body --------------------------------------------------------------------------------
// Tiles of blockDim.x * U groups, grid-strided; thread t takes groups t + j blockDim.x of a tile.  A full
// tile issues all U * VS loads before its first store.
template <int SRC, int DST, int U>
__device__ __forceinline__ void convert_tiles(const unsigned char* a, unsigned char* c, size_t ngroups)
{
    using S = convert_shape<SRC, DST>;
    const size_t tile = static_cast<size_t>(blockDim.x) * U;
    for (size_t t = blockIdx.x; t * tile < ngroups; t += gridDim.x) {
        const size_t g0 = t * tile + threadIdx.x;
        if ((t + 1) * tile <= ngroups) {
            u32x4 in[U][S::VS];
#pragma unroll
            for (int j = 0; j < U; ++j)
#pragma unroll
                for (int k = 0; k < S::VS; ++k)
                    in[j][k] = ldg128_bits<LD_PLAIN>(a + ((g0 + static_cast<size_t>(j) * blockDim.x) * S::VS + k) * 16);
#pragma unroll
            for (int j = 0; j < U; ++j) {
                u32x4 out[S::VD];
                convert_group<SRC, DST>(in[j], out);
#pragma unroll
                for (int k = 0; k < S::VD; ++k)
                    stg128_bits<ST_NA>(c + ((g0 + static_cast<size_t>(j) * blockDim.x) * S::VD + k) * 16, out[k]);
            }
        } else {
#pragma unroll
            for (int j = 0; j < U; ++j) {
                const size_t g = g0 + static_cast<size_t>(j) * blockDim.x;
                if (g < ngroups) {
                    u32x4 in[S::VS], out[S::VD];
#pragma unroll
                    for (int k = 0; k < S::VS; ++k) in[k] = ldg128_bits<LD_PLAIN>(a + (g * S::VS + k) * 16);
                    convert_group<SRC, DST>(in, out);
#pragma unroll
                    for (int k = 0; k < S::VD; ++k) stg128_bits<ST_NA>(c + (g * S::VD + k) * 16, out[k]);
                }
            }
        }
    }
}

// ---- the kernel -------------------------------------------------------------------------------------
// Elements [head, head + G ngroups) are the vector body, at 16-byte boundaries in A and in C; the others
// (the head, the tail, or all n when A and C have no common boundary and the dispatcher passes head = n)
// go through a grid-stride scalar loop.  unroll (1 or 2) and prefetch_first are the launch's geometry:
// with prefetch_first, thread 0 bulk-prefetches the CTA's first A tile into L2 ahead of the programmatic
// dependency (always legal: L2 is the point of coherence).
template <int SRC, int DST>
__global__ void convert_vec(const void* A, void* C, size_t n, size_t head, size_t ngroups, int unroll, int prefetch_first)
{
    using S = convert_shape<SRC, DST>;
    const unsigned char* a = static_cast<const unsigned char*>(A);
    unsigned char* c = static_cast<unsigned char*>(C);
    if (prefetch_first && threadIdx.x == 0) {
        const size_t tile = static_cast<size_t>(blockDim.x) * unroll, g0 = blockIdx.x * tile;
        if (g0 < ngroups)
            bulk_prefetch_l2(a + (head + g0 * S::G) * S::ESS,
                             static_cast<uint32_t>((ngroups - g0 < tile ? ngroups - g0 : tile) * S::G * S::ESS));
    }
    pdl_wait();

    if (unroll == 2) convert_tiles<SRC, DST, 2>(a + head * S::ESS, c + head * S::ESD, ngroups);
    else convert_tiles<SRC, DST, 1>(a + head * S::ESS, c + head * S::ESD, ngroups);

    const size_t body_end = head + ngroups * S::G, edges = head + (n - body_end);
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < edges; i += stride) {
        const size_t e = i < head ? i : body_end + (i - head);
        convert_elem<SRC, DST>(a + e * S::ESS, c + e * S::ESD);
    }
}

}  // namespace b200va
