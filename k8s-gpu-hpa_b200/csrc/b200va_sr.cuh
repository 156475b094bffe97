// b200va_sr.cuh -- b200va_convert_sr_f32 and b200va_quantize_fp8_sr_f32 (include/b200va.h): f32 rounded
// stochastically to f16, bf16, E4M3 or E5M2, with random bits that depend only on a seed and the element's global
// index, so the bytes do not depend on how the array is split across calls or launched.
//
//   convert   c[i] = SR(a[i])            to f16 / bf16, past max finite +-inf
//   quantize  c[i] = sat(SR(a[i] 2^k))   to E4M3 / E5M2, saturating at +-max finite
//
// Random bits.  Element i has the global index m = first + i (mod 2^64).  With key = splitmix64(seed) (the host
// derives it) and w_j = splitmix64(key + j), r_m is the low half of w_(m>>1) for even m and the high half for odd m.
// A group of G elements starting at global index m0 takes the words of the pairs m0>>1 .. (m0+G-1)>>1: G/2 of them
// for even m0, G/2 + 1 for odd m0.  m0 = first + head + G g with G even, so the parity is uniform across the launch.
//
// Rounding, exactly, in integer operations on the f32 pattern of y (y = a for f16/bf16, the f32 product a 2^k for
// FP8).  With E the exponent field, E' = max(E, 1) and sig the significand (with its implicit bit when E > 0),
// |y| = sig 2^(E'-150).  The destination's quantum at |y| is 2^(E'-150+s), s = (24 - P) + max(0, EMIN - E'), where P
// is its significand width and EMIN its smallest normal exponent in f32's bias; the quantum is fixed below its
// normal range, which gives its subnormals.  So lo = sig with its low s bits cleared and hi = lo + 2^s (in units of
// 2^(E'-150)), f = (sig mod 2^s) / 2^s, and t = floor(f 2^32) is the low word of (sig 2^32) >> s:
// - s <= 23: lo is the pattern with its low s bits cleared and hi that plus 2^s; a carry moves into the exponent,
//   as the element of D above the largest one of a binade is the next binade's first.
// - s >= 24: |y| lies below the destination's smallest subnormal q = 2^(E'-150+s), so lo = 0 and hi = q.  t is 0
//   once s >= 56 (sig < 2^24), which covers every f32 subnormal source for f16 and FP8.
// The result is hi when t + r carries out of 32 bits (r >= 2^32 - t), else lo, with y's sign put back.  That value,
// in D or one step past its largest finite value, is narrowed with the RN conversions b200va_convert and
// b200va_quantize_fp8 use, which are exact on it: f16 / bf16 give +-inf past max finite, the FP8 .satfinite gives
// +-max finite.  An exponent field of 255 bypasses the rounding: +-inf becomes +-inf or +-max finite, a NaN a NaN.
// For bf16 EMIN = 1 <= E', so s = 16 throughout and the rule is the familiar idiom: add the high 16 bits of r to the
// pattern and clear its low 16 bits.
//
// Why the f32 product is enough for FP8.  a 2^k (k in [-126, 126]) is exact in f32 unless it falls below 2^-126 or
// overflows.  Below 2^-126, f < 2^-32 for both formats (their smallest subnormals are 2^-9 and 2^-16), so t = 0 and
// the result is +-0 for the exact value and for the product alike (the product lies below 2^-126 too, or on it, where
// s >= 110 and t = 0 as well).  On overflow the product is +-inf, and the exact value saturates all the same.
//
// Layout.  One kernel, sr_cast_vec, the destination a uniform argument that picks one of four bodies at the top.  A
// group is G = 8 elements to a 2-byte destination and 16 to FP8: one 16-byte vector of C and 2 or 4 of A, as in
// convert_vec and fp8_quant_vec; the elements outside the vector body go through cast_edges.
#pragma once
#include "b200va_fp8.cuh"

namespace b200va {

// The kernel's destinations.
enum : int { SR_F16 = 0, SR_BF16 = 1, SR_E4M3 = 2, SR_E5M2 = 3 };

template <int D>
struct sr_traits {
    static constexpr bool fp8 = D == SR_E4M3 || D == SR_E5M2;
    static constexpr int G = fp8 ? 16 : 8;                  // elements per group
    static constexpr int VS = G / 4;                        // 16-byte source vectors per group
    static constexpr int ESC = fp8 ? 1 : 2;                 // destination bytes per element
    static constexpr uint32_t P = D == SR_F16 ? 11 : D == SR_BF16 ? 8 : D == SR_E4M3 ? 4 : 3;
    static constexpr uint32_t EMIN = D == SR_BF16 ? 1 : D == SR_E4M3 ? 121 : 113;
    static constexpr uint32_t QSUB = (EMIN - P + 1) << 23;  // the smallest subnormal's f32 pattern (not bf16's)
};

// The destination (dst, uniform across the launch) to a template argument, as with_f8 does for the format.
template <class F>
__device__ __forceinline__ void with_sr(int dst, F f)
{
    if (dst == SR_F16) f(std::integral_constant<int, SR_F16>{});
    else if (dst == SR_BF16) f(std::integral_constant<int, SR_BF16>{});
    else if (dst == SR_E4M3) f(std::integral_constant<int, SR_E4M3>{});
    else f(std::integral_constant<int, SR_E5M2>{});
}

// r for the G global indices m0 .. m0 + G - 1 (mod 2^64).  Word t serves the pair (m0 >> 1) + t, taken mod 2^63 as
// the pair index of an index mod 2^64 is: a group that runs past 2^64 - 1 continues with pair 0.
template <int G>
__device__ __forceinline__ void sr_bits(uint64_t key, uint64_t m0, uint32_t* r)
{
    const uint64_t p0 = m0 >> 1;
    const bool odd = m0 & 1;
    auto word = [=](int t) { return splitmix64(key + ((p0 + t) & 0x7fffffffffffffffull)); };
    uint32_t w[G + 1];
#pragma unroll
    for (int t = 0; t < G / 2; ++t) {
        const uint64_t x = word(t);
        w[2 * t] = static_cast<uint32_t>(x);
        w[2 * t + 1] = static_cast<uint32_t>(x >> 32);
    }
    w[G] = 0;
    if (odd) w[G] = static_cast<uint32_t>(word(G / 2));
#pragma unroll
    for (int j = 0; j < G; ++j) r[j] = odd ? w[j + 1] : w[j];
}

// r for the global index m.
__device__ __forceinline__ uint32_t sr_bits1(uint64_t key, uint64_t m)
{
    const uint64_t x = splitmix64(key + (m >> 1));
    return static_cast<uint32_t>(m & 1 ? x >> 32 : x);
}

// y rounded stochastically with r onto D (unbounded above), as an f32 value.
template <int D>
__device__ __forceinline__ float sr_round(float y, uint32_t r)
{
    using T = sr_traits<D>;
    const uint32_t u = __float_as_uint(y), a = u & 0x7fffffffu, E = a >> 23;
    const uint32_t Ep = max(E, 1u);
    const uint32_t s = (24 - T::P) + (T::EMIN > Ep ? T::EMIN - Ep : 0u);
    const uint32_t sig = a - ((Ep - 1) << 23);
    const uint32_t t = static_cast<uint32_t>((static_cast<uint64_t>(sig) << 32) >> min(s, 63u));
    const bool up = t + r < r;                              // t + r >= 2^32
    const bool sub = s >= 24;                               // |y| < q: lo = 0, hi = q
    const uint32_t step = sub ? T::QSUB : 1u << min(s, 23u);
    uint32_t res = (sub ? 0u : a & (0u - step)) + (up ? step : 0u);
    if (E == 255) res = a;
    return __uint_as_float(res | (u & 0x80000000u));
}

// Two source words x0, x1 with their bits r0, r1 to two elements of D: bits 0..15 and 16..31 of a 2-byte
// destination, bits 0..7 and 8..15 of FP8.  FP8 scales by 2^k first and takes the magnitudes into m.
template <int D>
__device__ __forceinline__ uint32_t sr_pair(uint32_t x0, uint32_t x1, uint32_t r0, uint32_t r1, int k, uint32_t& m)
{
    float y0 = __uint_as_float(x0), y1 = __uint_as_float(x1);
    if constexpr (sr_traits<D>::fp8) {
        m = max(m, max(x0 & 0x7fffffffu, x1 & 0x7fffffffu));
        y0 = __fmul_rn(y0, pow2<DT_F32>(k));
        y1 = __fmul_rn(y1, pow2<DT_F32>(k));
    }
    const float z0 = sr_round<D>(y0, r0), z1 = sr_round<D>(y1, r1);
    if constexpr (D == SR_F16) return narrow2_f32<DT_F16>(z0, z1);
    else if constexpr (D == SR_BF16) return narrow2_f32<DT_BF16>(z0, z1);
    else return f8x2_from_f32<D == SR_E4M3 ? F8_E4M3 : F8_E5M2>(z0, z1);
}

// The body after the dependency wait: elements [head, head + G ngroups) are the vector body, one group per unit, on
// 16-byte boundaries in A and in C; the others go through cast_edges.
template <int D>
__device__ __forceinline__ void sr_body(const unsigned char* a, unsigned char* c, size_t n, size_t head, size_t ngroups,
                                        int unroll, int k, uint64_t key, uint64_t first, uint32_t& m)
{
    using T = sr_traits<D>;
    constexpr int G = T::G;
    const unsigned char* ab = a + head * 4;
    unsigned char* cb = c + head * T::ESC;
    const uint64_t m0 = first + head;
    cast_tiles(unroll, ngroups, [=](size_t g) { return ld_vecs<T::VS>(ab, g); }, [&](size_t g, const vecs<T::VS>& in) {
        uint32_t s[G], r[G], d[4];
        unpack<T::VS>(in.v, s);
        sr_bits<G>(key, m0 + g * G, r);
#pragma unroll
        for (int w = 0; w < 4; ++w) {
            if constexpr (T::fp8)
                d[w] = sr_pair<D>(s[4 * w], s[4 * w + 1], r[4 * w], r[4 * w + 1], k, m) |
                       sr_pair<D>(s[4 * w + 2], s[4 * w + 3], r[4 * w + 2], r[4 * w + 3], k, m) << 16;
            else
                d[w] = sr_pair<D>(s[2 * w], s[2 * w + 1], r[2 * w], r[2 * w + 1], k, m);
        }
        stg128_bits<ST_NA>(cb + g * 16, u32x4{d[0], d[1], d[2], d[3]});
    });
    cast_edges(n, head, head + ngroups * G, [&](size_t e) {
        const uint32_t x = static_cast<uint32_t>(ld_bits<4>(a + e * 4));
        st_bits<T::ESC>(c + e * T::ESC, sr_pair<D>(x, 0u, sr_bits1(key, first + e), 0u, k, m));
    });
}

// The kernel: dst one of SR_*, k the FP8 scale exponent (0 otherwise), key = splitmix64(seed), first the global
// index of element 0.  unroll (1 or 2) and prefetch_first are the launch's geometry, as in convert_vec.  With amax
// (FP8 only), each CTA max-accumulates its largest |a_i| into *amax as fp8_quant_vec<DT_F32> does.
__global__ void sr_cast_vec(const void* A, void* C, size_t n, size_t head, size_t ngroups, int unroll, int prefetch_first,
                            int dst, int k, uint64_t key, uint64_t first, double* amax)
{
    const unsigned char* a = static_cast<const unsigned char*>(A);
    unsigned char* c = static_cast<unsigned char*>(C);
    uint32_t m = 0;
    with_sr(dst, [&](auto D) {
        prefetch_first_tile<sr_traits<decltype(D)::value>::G, 4>(prefetch_first, a, head, ngroups, unroll);
        pdl_wait();
        sr_body<D>(a, c, n, head, ngroups, unroll, k, key, first, m);
    });
    if (amax) cta_amax<DT_F32>(amax, m);
}

}  // namespace b200va
