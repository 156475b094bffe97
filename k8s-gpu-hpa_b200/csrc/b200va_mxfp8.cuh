// b200va_mxfp8.cuh -- b200va_quantize_mxfp8 and b200va_dequantize_mxfp8 (include/b200va.h): the FP8 casts of
// b200va_fp8.cuh with one E8M0 scale byte per block of 32, 64 or 128 elements (OCP MXFP8 and its wider cousins),
// the scale chosen and applied in one pass over the source.
//
//   quantize    per block: m = max |a_i| over the finite a_i, e from m by the scale rule, S[b] = e + 127,
//               c[i] = sat(RN(a[i] 2^-e))          rounded once, by the rules of b200va_quantize_fp8
//   dequantize  c[i] = RN(a[i] 2^(S[b] - 127))      rounded once to the destination; S[b] = 0xFF gives NaNs
//
// Blocks are counted from element 0 of the arrays.  Three kernels per direction, mx_quant_vec<ES> and
// mx_dequant_vec<ES> over the element size of the non-FP8 side: f16 and bf16 share the ES = 2 kernels (the same
// layout; they differ in the widening or narrowing instruction), and a uniform argument picks the type and the
// format at the top, one body per pair.  block and scale_rule are uniform arguments too.
//
// The exponent.  e = floor(log2 m) - emax (+ 1 under NOSAT when m's significand exceeds 1.75), clamped to
// [-127, 127], is read from m's bit pattern: the exponent field minus the bias, and the mantissa field compared
// with 0.75.  The field is not floor(log2 m) for a subnormal m or for m = 0, but there it does not matter: an f32
// subnormal is below 2^-126 and an f64 one below 2^-1022, so with the field read as the smallest normal exponent
// e is still below -127 - emax + 1 < -127 and the clamp gives -127, which is also the rule for m = 0.  f16 and bf16
// widen to f32 first (f16 subnormals become f32 normals, bf16 subnormals are f32 subnormals).
//
// One rounding, as in b200va_fp8.cuh, with the scale exponent -e per block:
// - f32, f16, bf16: -e lies in [-120, 127], so 2^-e is an f32 normal.  |a_i| <= m < 2^(e + emax + 1) unless e was
//   clamped up to -127, and then |a_i| 2^127 is smaller still: the product never overflows.  Where it is inexact
//   (below 2^-126) the exact value lies far below half the smallest FP8 subnormal and the result is +-0 either way.
// - f64: the product is formed in f64 and rounded to odd into f32.  With e clamped down to 127 the block holds
//   values up to 2^1024 2^-127, far outside f32: cvt.rz gives +-FLT_MAX there, which saturates as the exact value
//   does.  A product below the f64 or f32 normal range is far below half the smallest FP8 subnormal; round-to-odd
//   keeps it nonzero with its sign, and it rounds to +-0.  The product never overflows f64 (e = 127 only shrinks).
// - Dequantize scales by 2^(S - 127) in [2^-127, 2^127].  2^-127 is an f32 subnormal (0x00400000); the product with
//   an FP8 value is still exact (at most 4 significant bits, and the smallest one, 2^-16, times 2^-127 is a
//   multiple of 2^-149).  S = 0xFF scales by NaN, which makes every element, +-0 and +-inf included, a NaN.
//
// Layout.  The vector body runs when A and C both sit on a 16-byte boundary at element 0 (what an allocator
// returns), so groups of 16 and blocks coincide.  Quantize: a unit is a group of 16 elements per thread, a block is
// 2, 4 or 8 adjacent lanes, and the block maximum is 1-3 __shfl_xor_sync steps over the magnitude bit patterns.
// Tiles are multiples of 32 units and a unit's lane is its index mod 32, so a block never straddles a warp or a
// tile; the body is padded to whole warps, with the loads and stores guarded and the shuffle not.  The first lane
// of a block stores its scale byte.  Dequantize keeps fp8_dequant_vec's lane-contiguous 16-byte output slices; a
// slice lies inside one block, whose scale byte the lane loads beside its FP8 bytes.
// Everything else -- every block when A or C is off the boundary, and the short last block -- takes the edge
// path in the same kernel: quantize gives one thread one whole block (two passes of element-size loads: the
// maximum, then the cast), dequantize goes element by element.  It is the correctness path and is not tuned.
#pragma once
#include "b200va_fp8.cuh"

namespace b200va {

enum : int { MX_SCALE_OCP = 0, MX_SCALE_NOSAT = 1, MX_SCALE_COUNT = 2 };

// The block's scale exponent e from its finite maximum m (see "The exponent" above).
template <int SRC, int F8>
__device__ __forceinline__ int mx_exponent(amax_bits_t<SRC> m, int rule)
{
    constexpr int EMAX = F8 == F8_E4M3 ? 8 : 15;
    if constexpr (SRC == DT_F64) {
        const int up = rule == MX_SCALE_NOSAT && (m & 0x000fffffffffffffull) > 0x000c000000000000ull;
        return min(max(static_cast<int>(m >> 52) - 1023 - EMAX + up, -127), 127);
    } else {
        const int up = rule == MX_SCALE_NOSAT && (m & 0x007fffffu) > 0x00600000u;
        return max(static_cast<int>(m >> 23) - 127 - EMAX + up, -127);      // at most 127 - 8 + 1
    }
}

// The largest m over the `lanes` (2, 4 or 8) adjacent lanes that hold one block.  Every lane of the warp calls it.
template <class T>
__device__ __forceinline__ T block_max(T m, int lanes)
{
    m = max(m, __shfl_xor_sync(0xffffffffu, m, 1));
    if (lanes >= 4) m = max(m, __shfl_xor_sync(0xffffffffu, m, 2));
    if (lanes >= 8) m = max(m, __shfl_xor_sync(0xffffffffu, m, 4));
    return m;
}

// Quantize's body after the dependency wait.  Elements [0, 16 ngroups) are the vector body: whole blocks, one group
// of 16 per unit; blocks from 16 ngroups / block on take the edge path, one thread each.
template <int SRC, int F8>
__device__ __forceinline__ void mx_quant_body(const unsigned char* a, unsigned char* c, unsigned char* sc, size_t n,
                                              size_t ngroups, int unroll, int block, int rule)
{
    constexpr int ES = dt_traits<SRC>::size;      // also the 16-byte source vectors per group
    const int lanes = block / 16;
    const size_t padded = (ngroups + 31) & ~size_t{31};
    cast_tiles(unroll, padded, [=](size_t g) { return g < ngroups ? ld_vecs<ES>(a, g) : vecs<ES>{}; },
               [=](size_t g, const vecs<ES>& in) {
        uint32_t s[4 * ES], d[4];
        unpack<ES>(in.v, s);
        amax_bits_t<SRC> m = 0, unused = 0;
#pragma unroll
        for (int e = 0; e < 16; ++e) m = max(m, finite_mag<SRC>(s, e));
        const int ex = mx_exponent<SRC, F8>(block_max(m, lanes), rule);
        quant_group<SRC, F8>(s, -ex, unused, d);
        if (g < ngroups) {
            stg128_bits<ST_NA>(c + g * 16, u32x4{d[0], d[1], d[2], d[3]});
            if (g % lanes == 0) sc[g / lanes] = static_cast<unsigned char>(ex + 127);
        }
    });
    const size_t nblocks = (n + block - 1) / block;
    cast_edges(nblocks, 0, ngroups / lanes, [=](size_t b) {
        const size_t e0 = b * block, e1 = e0 + block < n ? e0 + block : n;
        amax_bits_t<SRC> m = 0, unused = 0;
        for (size_t e = e0; e < e1; ++e) {
            uint32_t s[2];
            ld_elem<ES>(a + e * ES, s);
            m = max(m, finite_mag<SRC>(s, 0));
        }
        const int ex = mx_exponent<SRC, F8>(m, rule);
        sc[b] = static_cast<unsigned char>(ex + 127);
        for (size_t e = e0; e < e1; ++e) c[e] = quant_elem<SRC, F8>(a + e * ES, -ex, unused);
    });
}

// The type (dt, a DT_* code of element size ES) and the format (fmt) to template arguments: f(SRC, F8) for the one
// pair that matches.  Both are uniform, so a kernel takes one branch at the top.
template <int ES, class F>
__device__ __forceinline__ void mx_with_pair(int dt, int fmt, F f)
{
    auto with_fmt = [=](auto T) { with_f8(fmt, [=](auto F8) { f(T, F8); }); };
    if constexpr (ES == 4) with_fmt(std::integral_constant<int, DT_F32>{});
    else if constexpr (ES == 8) with_fmt(std::integral_constant<int, DT_F64>{});
    else if (dt == DT_F16) with_fmt(std::integral_constant<int, DT_F16>{});
    else with_fmt(std::integral_constant<int, DT_BF16>{});
}

// One kernel per source element size.  unroll (1 or 2) and prefetch_first are the launch's geometry, as in
// convert_vec; the prefetch covers the CTA's first tile of the vector body.
template <int ES>
__global__ void mx_quant_vec(const void* A, void* C, void* S, size_t n, size_t ngroups, int unroll, int prefetch_first,
                             int src, int fmt, int block, int rule)
{
    const unsigned char* a = static_cast<const unsigned char*>(A);
    unsigned char* c = static_cast<unsigned char*>(C);
    unsigned char* sc = static_cast<unsigned char*>(S);
    prefetch_first_tile<16, ES>(prefetch_first, a, 0, ngroups, unroll);
    pdl_wait();

    mx_with_pair<ES>(src, fmt, [=](auto SRC, auto F8) { mx_quant_body<SRC, F8>(a, c, sc, n, ngroups, unroll, block, rule); });
}

// ---- dequantize -------------------------------------------------------------------------------------------
// The scale 2^(b - 127) of the E8M0 byte b in DST's arithmetic type; NaN for b = 0xFF.  As f32 bits it is b << 23
// for 1 <= b <= 254 and the subnormal 2^-127 for b = 0.
template <int DST>
__device__ __forceinline__ typename dt_traits<DST>::scalar mx_scale(uint32_t b)
{
    if constexpr (DST == DT_F64) return b == 0xffu ? __longlong_as_double(0x7ff8000000000000ll) : pow2<DST>(static_cast<int>(b) - 127);
    else return __uint_as_float(b == 0xffu ? 0x7fc00000u : b == 0u ? 0x00400000u : b << 23);
}

// One kernel per destination element size, the type and the format picked at the top as in mx_quant_vec.  The body is
// fp8_dequant_vec's from element 0 (elements [0, 16 ngroups), each slice inside one block), with the scale of the
// block an element lies in.
template <int ES>
__global__ void mx_dequant_vec(const void* A, const void* S, void* C, size_t n, size_t ngroups, int unroll,
                               int prefetch_first, int dst, int fmt, int block)
{
    const unsigned char* a = static_cast<const unsigned char*>(A);
    const unsigned char* sc = static_cast<const unsigned char*>(S);
    unsigned char* c = static_cast<unsigned char*>(C);
    prefetch_first_tile<16 / ES, 1>(prefetch_first, a, 0, ngroups * ES, unroll);
    pdl_wait();

    const int shift = 31 - __clz(block);
    mx_with_pair<ES>(dst, fmt, [=](auto DST, auto F8) {
        dequant_body<F8, DST>(a, c, n, 0, ngroups, unroll, [=](size_t e) { return mx_scale<DST>(sc[e >> shift]); });
    });
}

}  // namespace b200va
