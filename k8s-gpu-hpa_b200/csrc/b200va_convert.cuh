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

// ---- the pieces every cast kernel shares -------------------------------------------------------------
// The BYTES (1, 2, 4 or 8) bytes at p, BYTES-aligned, zero-extended; and the low BYTES bytes of v stored to p.
template <int BYTES>
__device__ __forceinline__ unsigned long long ld_bits(const unsigned char* p)
{
    if constexpr (BYTES == 8) return *reinterpret_cast<const unsigned long long*>(p);
    else if constexpr (BYTES == 4) return *reinterpret_cast<const uint32_t*>(p);
    else if constexpr (BYTES == 2) return *reinterpret_cast<const unsigned short*>(p);
    else return *p;
}

template <int BYTES>
__device__ __forceinline__ void st_bits(unsigned char* p, unsigned long long v)
{
    if constexpr (BYTES == 8) *reinterpret_cast<unsigned long long*>(p) = v;
    else if constexpr (BYTES == 4) *reinterpret_cast<uint32_t*>(p) = static_cast<uint32_t>(v);
    else if constexpr (BYTES == 2) *reinterpret_cast<unsigned short*>(p) = static_cast<unsigned short>(v);
    else *p = static_cast<unsigned char>(v);
}

// One element as the words a group holds it in: the ES (2, 4 or 8) bytes at p, ES-aligned, to s[0] and s[1] (the
// bytes it does not have are 0); and the low ES bytes of lo, hi stored to p.
template <int ES>
__device__ __forceinline__ void ld_elem(const unsigned char* p, uint32_t* s)
{
    const unsigned long long x = ld_bits<ES>(p);
    s[0] = static_cast<uint32_t>(x);
    s[1] = static_cast<uint32_t>(x >> 32);
}

template <int ES>
__device__ __forceinline__ void st_elem(unsigned char* p, uint32_t lo, uint32_t hi)
{
    st_bits<ES>(p, lo | static_cast<unsigned long long>(hi) << 32);
}

// V consecutive 16-byte vectors, as a value a tile can hold per unit.
template <int V>
struct vecs { u32x4 v[V]; };

// Unit u of a body of V-vector units at p.
template <int V>
__device__ __forceinline__ vecs<V> ld_vecs(const unsigned char* p, size_t u)
{
    vecs<V> r;
#pragma unroll
    for (int k = 0; k < V; ++k) r.v[k] = ldg128_bits<LD_PLAIN>(p + (u * V + k) * 16);
    return r;
}

// The 32-bit words of V vectors, in memory order.
template <int V>
__device__ __forceinline__ void unpack(const u32x4* v, uint32_t* w)
{
#pragma unroll
    for (int k = 0; k < V; ++k) {
        w[4 * k] = v[k].x; w[4 * k + 1] = v[k].y; w[4 * k + 2] = v[k].z; w[4 * k + 3] = v[k].w;
    }
}

// With prefetch_first, thread 0 bulk-prefetches the CTA's first tile of A into L2 (units of PER_UNIT elements of
// ES bytes, from element head on) ahead of the programmatic dependency: always legal, L2 is the point of coherence.
template <int PER_UNIT, int ES>
__device__ __forceinline__ void prefetch_first_tile(int prefetch_first, const unsigned char* a, size_t head, size_t nunits,
                                                    int unroll)
{
    if (prefetch_first && threadIdx.x == 0) {
        const size_t tile = static_cast<size_t>(blockDim.x) * unroll, u0 = blockIdx.x * tile;
        if (u0 < nunits)
            bulk_prefetch_l2(a + (head + u0 * PER_UNIT) * ES,
                             static_cast<uint32_t>((nunits - u0 < tile ? nunits - u0 : tile) * PER_UNIT * ES));
    }
}

// The vector body: tiles of blockDim.x * U units, grid-strided; thread t takes units t + j blockDim.x of a tile.
// load(u) reads unit u and put(u, x) computes and stores it.  A full tile issues all U loads before its first store;
// a partial tile guards each unit.
template <int U, class Load, class Put>
__device__ __forceinline__ void cast_tiles(size_t nunits, Load load, Put put)
{
    const size_t tile = static_cast<size_t>(blockDim.x) * U;
    for (size_t t = blockIdx.x; t * tile < nunits; t += gridDim.x) {
        const size_t u0 = t * tile + threadIdx.x;
        if ((t + 1) * tile <= nunits) {
            decltype(load(u0)) in[U];
#pragma unroll
            for (int j = 0; j < U; ++j) in[j] = load(u0 + static_cast<size_t>(j) * blockDim.x);
#pragma unroll
            for (int j = 0; j < U; ++j) put(u0 + static_cast<size_t>(j) * blockDim.x, in[j]);
        } else {
#pragma unroll
            for (int j = 0; j < U; ++j) {
                const size_t u = u0 + static_cast<size_t>(j) * blockDim.x;
                if (u < nunits) put(u, load(u));
            }
        }
    }
}

// The launch's unroll (1 or 2) to cast_tiles.
template <class Load, class Put>
__device__ __forceinline__ void cast_tiles(int unroll, size_t nunits, Load load, Put put)
{
    if (unroll == 2) cast_tiles<2>(nunits, load, put);
    else cast_tiles<1>(nunits, load, put);
}

// The elements outside the vector body [head, body_end) -- the head and the tail, or all n in mixed phase (head = n)
// -- grid-strided, elem(e) for each.
template <class Elem>
__device__ __forceinline__ void cast_edges(size_t n, size_t head, size_t body_end, Elem elem)
{
    const size_t edges = head + (n - body_end);
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < edges; i += stride)
        elem(i < head ? i : body_end + (i - head));
}

// One group: VS source vectors in, VD destination vectors out.
template <int SRC, int DST>
__device__ __forceinline__ void convert_group(const u32x4* in, u32x4* out)
{
    using S = convert_shape<SRC, DST>;
    uint32_t s[4 * S::VS], d[4 * S::VD];
    unpack<S::VS>(in, s);
    convert_words<SRC, DST, S::G>(s, d);
#pragma unroll
    for (int k = 0; k < S::VD; ++k) out[k] = u32x4{d[4 * k], d[4 * k + 1], d[4 * k + 2], d[4 * k + 3]};
}

// One element at byte pointers a, c (element-size aligned).
template <int SRC, int DST>
__device__ __forceinline__ void convert_elem(const unsigned char* a, unsigned char* c)
{
    using S = convert_shape<SRC, DST>;
    uint32_t s[2], d[2] = {0, 0};
    ld_elem<S::ESS>(a, s);
    convert_words<SRC, DST, 1>(s, d);
    st_elem<S::ESD>(c, d[0], d[1]);
}

// ---- the kernel -------------------------------------------------------------------------------------
// Elements [head, head + G ngroups) are the vector body, one group per unit, at 16-byte boundaries in A and in C;
// the others go through cast_edges.  unroll (1 or 2) and prefetch_first are the launch's geometry.
template <int SRC, int DST>
__global__ void convert_vec(const void* A, void* C, size_t n, size_t head, size_t ngroups, int unroll, int prefetch_first)
{
    using S = convert_shape<SRC, DST>;
    const unsigned char* a = static_cast<const unsigned char*>(A);
    unsigned char* c = static_cast<unsigned char*>(C);
    prefetch_first_tile<S::G, S::ESS>(prefetch_first, a, head, ngroups, unroll);
    pdl_wait();

    const unsigned char* ab = a + head * S::ESS;
    unsigned char* cb = c + head * S::ESD;
    cast_tiles(unroll, ngroups, [=](size_t g) { return ld_vecs<S::VS>(ab, g); }, [=](size_t g, const vecs<S::VS>& in) {
        u32x4 out[S::VD];
        convert_group<SRC, DST>(in.v, out);
#pragma unroll
        for (int k = 0; k < S::VD; ++k) stg128_bits<ST_NA>(cb + (g * S::VD + k) * 16, out[k]);
    });
    cast_edges(n, head, head + ngroups * S::G, [=](size_t e) { convert_elem<SRC, DST>(a + e * S::ESS, c + e * S::ESD); });
}

}  // namespace b200va
