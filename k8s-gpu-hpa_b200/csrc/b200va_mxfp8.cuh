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

// ---- blockwise FP8 (b200va_quantize_fp8_blockwise) -----------------------------------------------------
// A is rows x cols, row-major.  C (rows x cols) and Ct (cols x rows) are FP8, each with f32 scales S and St; either
// pair may be absent.  Blocks are 1 x 128 (C's run along A's rows, Ct's along A's columns, so 128 x 1 blocks of A) or
// 128 x 128 tiles of A (one scale for C and Ct).  Per block: m = the largest finite |a_i|, k = clamp(K(m), -126, 126)
// with K(m) the largest k with m 2^k <= max finite (the negated NOSAT exponent), the scale 2^-k stored as an f32, and
// every element rounded once as sat(RN(a 2^k)) by quant_pair.  Scale layouts (torch's scaled_mm, MN-major):
//   1 x 128    S[b rows + i] for block b of row i; St[b cols + j] for block b of column j
//   128 x 128  S[p L4 + q] for tile (p, q), L4 = ceil(ceil(cols / 128) / 4) 4; St[q L4t + p], L4t from rows alike
//
// Tiled path (cols % 128 == 0, rows % 16 == 0, A, C and Ct on 16-byte boundaries): one 128 x 128 tile of A per CTA,
// FP8B_THREADS threads.  Warp w, lane l takes group g = l % 8 (columns 16 g .. 16 g + 15) of tile
// rows 32 s + 4 w + l / 8, s = 0..3; the bottom tile row may hold 16..112 rows, whole warps' rows dropping out.
//   1 x 128     without Ct, one sweep: the row's maximum over the 8 lanes of its row (block_max), its scale and
//               quant_group to C.  With Ct, sweep 1 loads each group once and takes the column maxima over the
//               warp's 4 rows by __shfl_xor, max-accumulated into the warp's row of shared memory (kept out of
//               registers, where 16 more live values spilled); the 8 warps' rows give the 128 column exponents and
//               512 contiguous bytes of St.  Sweep 2 reloads the groups (from L2: the CTA read them just before),
//               rounds each element by its column's exponent into the transposed byte tile, and C's row as above.
//   128 x 128   sweep 1 takes the maximum only; one exponent per tile (warp_max, then the 8 warps); sweep 2 reloads
//               and rounds each group with quant_group to C and into the byte tile.
// The byte tile holds Ct's 128 rows of the tile, swizzled as in quant_t_tiles: 16-byte chunk h of tile row j sits at
// chunk h ^ (j / 16), so the 8 groups of a warp's byte stores fall in 8 different bank quads, and 8 lanes read a Ct
// row's 128 bytes, stored as one 128-byte line.
// Per-block path (every other shape or placement): one thread per block, two passes of element loads (the maximum,
// then the cast) -- the correctness path, not tuned, reading A once per block kind it writes.
enum : int { FP8B_1X128 = 0, FP8B_128X128 = 1, FP8B_COUNT = 2 };
// The row-wise cast (b200va_quantize_fp8_rowwise) is three launches of the same kernel, told apart by kind:
//   FP8R_MAXIMA  the 1 x 128 block scales of the requested sides into the workspace, in the 1 x 128 layouts (W[b rows
//                + i] for block b of row i, then W'[b cols + j] for block b of column j), no bytes: the 1 x 128 cast's
//                sweep 1 (fp8b_tiles) or its per-block path without the cast.  C and Ct only say which sides.
//   FP8R_REDUCE  S[i] = max_b W[b rows + i], St[j] = max_b W'[b cols + j] (fp8r_reduce).  K is monotone and the clamp
//                commutes with min, so a row's k is the min of its blocks' k: its scale, the max of theirs.
//   FP8R_ROWS    every element rounded with its row's k (C) and its column's k (Ct), k = 127 - (S bits >> 23); the
//                dequantize's kind too, one scale per row.
enum : int { FP8R_MAXIMA = FP8B_COUNT, FP8R_REDUCE, FP8R_ROWS };
constexpr int FP8B_TILE = 128;
constexpr int FP8B_THREADS = 256;
// the byte tile, then the warps' column maxima (8 x 128 as f64 bits at most), then the 128 column exponents
constexpr int FP8B_SMEM = FP8B_TILE * FP8B_TILE + 8 * FP8B_TILE * 8 + FP8B_TILE * 4;      // 25 088 bytes (dynamic)

// The shape of a blockwise cast: A rows x cols, nkb_r and nkb_c blocks of 128 down and across, and the row pitch of
// the 128 x 128 scale layouts of C (l4) and Ct (l4t).
struct fp8b_shape { size_t rows, cols, nkb_r, nkb_c, l4, l4t; };

// k of a block with finite maximum m (amax_bits_t): clamp(K(m), -126, 126), K(0) = +inf.
template <int SRC, int F8>
__device__ __forceinline__ int fp8b_exponent(amax_bits_t<SRC> m)
{
    return min(max(-mx_exponent<SRC, F8>(m, MX_SCALE_NOSAT), -126), 126);
}

// The f32 scale 2^-k a block stores, k in [-126, 126].
__device__ __forceinline__ float fp8b_scale(int k) { return __int_as_float((127 - k) << 23); }

// x / d, and x % d into r, for x < 2^42 and rd = __drcp_rn(d), without a 64-bit division (whose call would raise the
// kernel's register count): x rd in f64 is within 2^-10 of the quotient, and its truncation is corrected by one.
__device__ __forceinline__ size_t fp8b_div(size_t x, size_t d, double rd, size_t& r)
{
    long long q = static_cast<long long>(static_cast<double>(x) * rd);
    long long s = static_cast<long long>(x) - q * static_cast<long long>(d);
    if (s < 0) { --q; s += d; }
    else if (s >= static_cast<long long>(d)) { ++q; s -= d; }
    r = static_cast<size_t>(s);
    return static_cast<size_t>(q);
}

// A group's row-wise 1 x 128 cast: gm its finite maximum, the block's maximum over the 8 lanes of the row (every lane
// of the warp calls it), the 16 bytes to c and, from the row's first lane (g = 0), the scale to *s.
template <int SRC, int F8>
__device__ __forceinline__ void fp8b_row(const uint32_t* v, amax_bits_t<SRC> gm, unsigned char* c, float* s, unsigned g)
{
    amax_bits_t<SRC> unused = 0;
    const int k = fp8b_exponent<SRC, F8>(block_max(gm, 8));
    uint32_t d[4];
    quant_group<SRC, F8>(v, k, unused, d);
    stg128_bits<ST_NA>(c, u32x4{d[0], d[1], d[2], d[3]});
    if (g == 0) *s = fp8b_scale(k);
}

// Byte b of d (b = 0..15) is A's column 16 g + b at tile row i: into the byte tile, at tile row 16 g + b and row i of
// its swizzled chunk.
__device__ __forceinline__ void fp8b_put_t(unsigned char* tile, const uint32_t* d, unsigned i, unsigned g)
{
    unsigned char* col = tile + 16 * g * FP8B_TILE + 16 * ((i / 16) ^ g) + i % 16;
#pragma unroll
    for (int b = 0; b < 16; ++b) col[b * FP8B_TILE] = static_cast<unsigned char>(d[b / 4] >> (8 * (b % 4)));
}

// The byte tile to Ct's rows j0 .. j0 + 127, columns i0 .. i0 + tr: 8 lanes per 128-byte row.
__device__ __forceinline__ void fp8b_store_t(const unsigned char* tile, unsigned char* ct, size_t rows, size_t i0,
                                             size_t j0, unsigned tr)
{
#pragma unroll
    for (int u = 0; u < FP8B_TILE * FP8B_TILE / 16 / FP8B_THREADS; ++u) {
        const unsigned chunk = threadIdx.x + u * FP8B_THREADS, j = chunk / 8, h = chunk % 8;
        if (16 * h < tr)
            stg128_bits<ST_NA>(ct + (j0 + j) * rows + i0 + 16 * h,
                               *reinterpret_cast<const u32x4*>(tile + j * FP8B_TILE + 16 * (h ^ (j / 16))));
    }
}

// The tiled path, one format and one block kind.  With kind FP8R_MAXIMA (1 x 128 only) it is sweep 1 alone: the row
// blocks' scales to sc when c is set, the column blocks' to sct when ct is set, and no bytes.
template <int SRC, int F8, int KIND>
__device__ __forceinline__ void fp8b_tiles(const unsigned char* a, unsigned char* c, float* sc, unsigned char* ct,
                                           float* sct, const fp8b_shape& sh, int kind)
{
    constexpr int ES = dt_traits<SRC>::size, T = FP8B_TILE;
    using M = amax_bits_t<SRC>;
    extern __shared__ __align__(16) unsigned char fp8b_smem[];
    unsigned char* tile = fp8b_smem;                                              // T x T bytes, Ct's rows
    M* part = reinterpret_cast<M*>(fp8b_smem + T * T);                            // [8 warps][T] column maxima
    int* kcol = reinterpret_cast<int*>(fp8b_smem + T * T + 8 * T * 8);            // [T] column exponents
    const size_t rows = sh.rows, cols = sh.cols;
    const unsigned w = threadIdx.x / 32, l = threadIdx.x % 32, g = l % 8, r = 4 * w + l / 8;
    // one CTA per tile: the launch has as many CTAs as tiles, at most 2^40 / (16 T) = 2^29 (and at most 2^36 / T tile
    // columns, rows >= 16)
    const unsigned tiles_c = static_cast<unsigned>(sh.nkb_c), p = blockIdx.x / tiles_c, q = blockIdx.x % tiles_c;
    const size_t i0 = static_cast<size_t>(p) * T, j0 = static_cast<size_t>(q) * T;
    const unsigned tr = static_cast<unsigned>(min(rows - i0, size_t{T}));
    M tm = 0, unused = 0;
    // sweep 1: A's groups once
#pragma unroll 1
    for (int s = 0; s < 4; ++s) {
        const unsigned i = 32 * s + r;
        if (i >= tr) continue;                                                // whole warps (tr % 16 == 0)
        const size_t e = (i0 + i) * cols + j0 + 16 * g;
        uint32_t v[4 * ES];
        unpack<ES>(ld_vecs<ES>(a + e * ES, 0).v, v);
        M gm = 0;
#pragma unroll
        for (int x = 0; x < 16; ++x) gm = max(gm, finite_mag<SRC>(v, x));
        if constexpr (KIND == FP8B_1X128) {
            if (kind == FP8R_MAXIMA) {
                if (c) {
                    const int kr = fp8b_exponent<SRC, F8>(block_max(gm, 8));
                    if (g == 0) sc[q * rows + i0 + i] = fp8b_scale(kr);
                }
                if (!ct) continue;
            } else if (!ct) {
                fp8b_row<SRC, F8>(v, gm, c + e, sc + q * rows + i0 + i, g);
                continue;
            }
            // the column maxima over the warp's 4 rows, max-accumulated into the warp's own row of part
#pragma unroll
            for (int x = 0; x < 16; ++x) {
                M f = finite_mag<SRC>(v, x);
                f = max(f, __shfl_xor_sync(0xffffffffu, f, 8));
                f = max(f, __shfl_xor_sync(0xffffffffu, f, 16));
                if (l < 8) part[w * T + 16 * g + x] = s ? max(part[w * T + 16 * g + x], f) : f;
            }
        } else {
            tm = max(tm, gm);
        }
    }
    // the exponents the second sweep needs
    int k = 0;
    if constexpr (KIND == FP8B_1X128) {
        if (!ct) return;
        if (l < 8 && 4 * w >= tr) {                       // a warp below the tile's rows adds nothing
#pragma unroll
            for (int x = 0; x < 16; ++x) part[w * T + 16 * g + x] = 0;
        }
        __syncthreads();
        if (threadIdx.x < T) {
            M m = part[threadIdx.x];
#pragma unroll
            for (int u = 1; u < 8; ++u) m = max(m, part[u * T + threadIdx.x]);
            const int kx = fp8b_exponent<SRC, F8>(m);
            kcol[threadIdx.x] = kx;
            sct[p * cols + j0 + threadIdx.x] = fp8b_scale(kx);
        }
        __syncthreads();
        if (kind == FP8R_MAXIMA) return;                  // sweep 1 only
    } else {
        tm = warp_max(tm);
        if (l == 0) part[w] = tm;
        __syncthreads();
        M m = part[0];
#pragma unroll
        for (int u = 1; u < 8; ++u) m = max(m, part[u]);
        k = fp8b_exponent<SRC, F8>(m);
        if (threadIdx.x == 0) {
            if (c) sc[p * sh.l4 + q] = fp8b_scale(k);
            if (ct) sct[q * sh.l4t + p] = fp8b_scale(k);
        }
    }
    // sweep 2: the groups again, rounded for Ct (and C for 128 x 128)
#pragma unroll 1
    for (int s = 0; s < 4; ++s) {
        const unsigned i = 32 * s + r;
        if (i >= tr) continue;
        const size_t e = (i0 + i) * cols + j0 + 16 * g;
        uint32_t v[4 * ES], d[4];
        unpack<ES>(ld_vecs<ES>(a + e * ES, 0).v, v);
        if constexpr (KIND == FP8B_1X128) {
            const int* kc = kcol + 16 * g;                    // the 16 columns' exponents
#pragma unroll
            for (int x = 0; x < 4; ++x)
                d[x] = quant_pair<SRC, F8>(v, 4 * x, kc[4 * x], kc[4 * x + 1], unused) |
                       (quant_pair<SRC, F8>(v, 4 * x + 2, kc[4 * x + 2], kc[4 * x + 3], unused) << 16);
        } else {
            quant_group<SRC, F8>(v, k, unused, d);
            if (c) stg128_bits<ST_NA>(c + e, u32x4{d[0], d[1], d[2], d[3]});
        }
        if (ct) fp8b_put_t(tile, d, i, g);
        if constexpr (KIND == FP8B_1X128) {
            if (c) {
                M gm = 0;
#pragma unroll
                for (int x = 0; x < 16; ++x) gm = max(gm, finite_mag<SRC>(v, x));
                fp8b_row<SRC, F8>(v, gm, c + e, sc + q * rows + i0 + i, g);
            }
        }
    }
    __syncthreads();
    if (!ct) return;
    fp8b_store_t(tile, ct, rows, i0, j0, tr);
}

// k from a scale 2^-k that FP8R_REDUCE left (a normal f32 power of two, k in [-126, 126]).
__device__ __forceinline__ int fp8r_k(float s) { return 127 - static_cast<int>(__float_as_uint(s) >> 23); }

// FP8R_ROWS on the tiled path: fp8b_tiles' tiles, threads and byte tile, one sweep (the k are known, no maxima).  Each
// group is rounded with its row's k into C (quant_group) and with its 16 columns' k (kcol, from St) into the byte tile
// (quant_pair).
template <int SRC, int F8>
__device__ __forceinline__ void fp8r_tiles(const unsigned char* a, unsigned char* c, const float* sc, unsigned char* ct,
                                           const float* sct, const fp8b_shape& sh)
{
    constexpr int ES = dt_traits<SRC>::size, T = FP8B_TILE;
    extern __shared__ __align__(16) unsigned char fp8b_smem[];
    unsigned char* tile = fp8b_smem;
    int* kcol = reinterpret_cast<int*>(fp8b_smem + T * T + 8 * T * 8);
    const size_t rows = sh.rows, cols = sh.cols;
    const unsigned w = threadIdx.x / 32, l = threadIdx.x % 32, g = l % 8, r = 4 * w + l / 8;
    const unsigned tiles_c = static_cast<unsigned>(sh.nkb_c), p = blockIdx.x / tiles_c, q = blockIdx.x % tiles_c;
    const size_t i0 = static_cast<size_t>(p) * T, j0 = static_cast<size_t>(q) * T;
    const unsigned tr = static_cast<unsigned>(min(rows - i0, size_t{T}));
    amax_bits_t<SRC> unused = 0;
    if (ct) {
        if (threadIdx.x < T) kcol[threadIdx.x] = fp8r_k(sct[j0 + threadIdx.x]);
        __syncthreads();
    }
#pragma unroll 1
    for (int s = 0; s < 4; ++s) {
        const unsigned i = 32 * s + r;
        if (i >= tr) continue;
        const size_t e = (i0 + i) * cols + j0 + 16 * g;
        uint32_t v[4 * ES], d[4];
        unpack<ES>(ld_vecs<ES>(a + e * ES, 0).v, v);
        if (ct) {
            const int* kc = kcol + 16 * g;
#pragma unroll
            for (int x = 0; x < 4; ++x)
                d[x] = quant_pair<SRC, F8>(v, 4 * x, kc[4 * x], kc[4 * x + 1], unused) |
                       (quant_pair<SRC, F8>(v, 4 * x + 2, kc[4 * x + 2], kc[4 * x + 3], unused) << 16);
            fp8b_put_t(tile, d, i, g);
        }
        if (c) {
            quant_group<SRC, F8>(v, fp8r_k(sc[i0 + i]), unused, d);
            stg128_bits<ST_NA>(c + e, u32x4{d[0], d[1], d[2], d[3]});
        }
    }
    if (!ct) return;
    __syncthreads();
    fp8b_store_t(tile, ct, rows, i0, j0, tr);
}

// FP8R_ROWS on every other shape or placement: one thread per element of A, its byte to C and / or Ct (untuned).
template <int SRC, int F8>
__device__ __forceinline__ void fp8r_elems(const unsigned char* a, unsigned char* c, const float* sc, unsigned char* ct,
                                           const float* sct, const fp8b_shape& sh)
{
    constexpr int ES = dt_traits<SRC>::size;
    const size_t n = sh.rows * sh.cols;
    const double rd = __drcp_rn(static_cast<double>(sh.cols));
    cast_edges(n, n, n, [=](size_t e) {
        size_t j;
        const size_t i = fp8b_div(e, sh.cols, rd, j);
        amax_bits_t<SRC> unused = 0;
        if (c) c[e] = quant_elem<SRC, F8>(a + e * ES, fp8r_k(sc[i]), unused);
        if (ct) ct[j * sh.rows + i] = quant_elem<SRC, F8>(a + e * ES, fp8r_k(sct[j]), unused);
    });
}

// FP8R_REDUCE: one thread per row (S, when set), then per column (St, when set), walking its blocks' scales in the
// workspace w; consecutive threads read consecutive entries.  The scales are positive normals, so their bit patterns
// order as they do.
__device__ __forceinline__ void fp8r_reduce(const float* w, float* s, float* st, const fp8b_shape& sh)
{
    const size_t nr = s ? sh.rows : 0, n = nr + (st ? sh.cols : 0);
    const float* wt = w + sh.rows * sh.nkb_c;
    cast_edges(n, n, n, [=](size_t t) {
        const bool row = t < nr;
        const size_t u = row ? t : t - nr, pitch = row ? sh.rows : sh.cols, nb = row ? sh.nkb_c : sh.nkb_r;
        const float* p = (row ? w : wt) + u;
        uint32_t m = 0;
#pragma unroll 4
        for (size_t b = 0; b < nb; ++b) m = max(m, __float_as_uint(p[b * pitch]));
        (row ? s : st)[u] = __uint_as_float(m);
    });
}

// A block of the per-block path: the h x w elements (h, w <= 128) of A from pa on, row pitch cols; its maximum, then
// its bytes to C from pc on (row pitch cols) and / or to Ct from pct on (row pitch rows), either may be null, and its
// scale to *s and / or *st.
template <int SRC, int F8>
__device__ __forceinline__ void fp8b_rect(const unsigned char* pa, unsigned char* pc, unsigned char* pct, size_t rows,
                                          size_t cols, unsigned h, unsigned w, float* s, float* st)
{
    constexpr int ES = dt_traits<SRC>::size;
    amax_bits_t<SRC> m = 0, unused = 0;
#pragma unroll 1
    for (unsigned y = 0; y < h; ++y)
#pragma unroll 1
        for (unsigned x = 0; x < w; ++x) {
            uint32_t v[2];
            ld_elem<ES>(pa + (y * cols + x) * ES, v);
            m = max(m, finite_mag<SRC>(v, 0));
        }
    const int k = fp8b_exponent<SRC, F8>(m);
    if (s) *s = fp8b_scale(k);
    if (st) *st = fp8b_scale(k);
    if (!pc && !pct) return;
#pragma unroll 1
    for (unsigned y = 0; y < h; ++y)
#pragma unroll 1
        for (unsigned x = 0; x < w; ++x) {
            const unsigned char b = quant_elem<SRC, F8>(pa + (y * cols + x) * ES, k, unused);
            if (pc) pc[y * cols + x] = b;
            if (pct) pct[x * rows + y] = b;
        }
}

// The per-block path: 1 x 128 gives C's blocks (row i, block b) as items [0, nrow) and Ct's (column j, block b) as
// the next ncol; 128 x 128 gives one item per tile, writing both.  Without `bytes` (FP8R_MAXIMA) only the scales.
template <int SRC, int F8>
__device__ __forceinline__ void fp8b_blocks(const unsigned char* a, unsigned char* c, float* sc, unsigned char* ct,
                                            float* sct, const fp8b_shape& sh, int kind, bool bytes = true)
{
    constexpr int ES = dt_traits<SRC>::size;
    constexpr size_t B = FP8B_TILE;
    const size_t rows = sh.rows, cols = sh.cols;
    // items: 1 x 128 row blocks (nrow), then column blocks; 128 x 128 tiles.  An item is (u, b): u the row, column
    // or tile row, b the block along it, u = t / nb by the reciprocal.
    const bool tiles = kind != FP8B_1X128;
    const size_t nrow = tiles ? sh.nkb_r * sh.nkb_c : c ? rows * sh.nkb_c : 0;
    const size_t nitems = nrow + (tiles || !ct ? 0 : cols * sh.nkb_r);
    cast_edges(nitems, nitems, nitems, [=](size_t t) {
        const bool along = t < nrow;                                  // C's row blocks, or a tile
        const size_t nb = along ? sh.nkb_c : sh.nkb_r;
        size_t b;
        const size_t u = fp8b_div(along ? t : t - nrow, nb, __drcp_rn(static_cast<double>(nb)), b);
        // the block's first element (i, j) and extent
        const size_t i = tiles ? u * B : along ? u : b * B, j = tiles ? b * B : along ? b * B : u;
        const unsigned h = static_cast<unsigned>(tiles || !along ? min(rows - i, B) : 1),
                       w = static_cast<unsigned>(tiles || along ? min(cols - j, B) : 1);
        float* s = tiles ? (c ? sc + u * sh.l4 + b : nullptr) : along ? sc + b * rows + u : nullptr;
        float* st = tiles ? (ct ? sct + b * sh.l4t + u : nullptr) : along ? nullptr : sct + b * cols + u;
        fp8b_rect<SRC, F8>(a + (i * cols + j) * ES, bytes && (tiles || along) && c ? c + i * cols + j : nullptr,
                           !bytes ? nullptr : tiles ? (ct ? ct + j * rows + i : nullptr) : along ? nullptr : ct + j * rows + i,
                           rows, cols, h, w, s, st);
    });
}

// The blockwise quantize, and the row-wise cast's launches, after the dependency wait: the tiled path when ngroups
// (= n / 16) is set, else the per-block (or per-element) path.
template <int SRC, int F8>
__device__ __forceinline__ void fp8b_quant_body(const unsigned char* a, unsigned char* c, float* sc, unsigned char* ct,
                                                float* sct, size_t ngroups, const fp8b_shape& sh, int kind)
{
    if (!ngroups && kind == FP8R_ROWS) fp8r_elems<SRC, F8>(a, c, sc, ct, sct, sh);
    else if (!ngroups) fp8b_blocks<SRC, F8>(a, c, sc, ct, sct, sh, kind == FP8R_MAXIMA ? FP8B_1X128 : kind, kind != FP8R_MAXIMA);
    else if (kind == FP8R_ROWS) fp8r_tiles<SRC, F8>(a, c, sc, ct, sct, sh);
    else if (kind == FP8B_128X128) fp8b_tiles<SRC, F8, FP8B_128X128>(a, c, sc, ct, sct, sh, kind);
    else fp8b_tiles<SRC, F8, FP8B_1X128>(a, c, sc, ct, sct, sh, kind);
}

// The shape of a rows x cols blockwise cast, as the host's b200va_fp8_blockwise_scales counts it.
__device__ __forceinline__ fp8b_shape fp8b_make_shape(size_t rows, size_t cols)
{
    fp8b_shape sh;
    sh.rows = rows;
    sh.cols = cols;
    sh.nkb_r = (rows + FP8B_TILE - 1) / FP8B_TILE;
    sh.nkb_c = (cols + FP8B_TILE - 1) / FP8B_TILE;
    sh.l4 = (sh.nkb_c + 3) / 4 * 4;
    sh.l4t = (sh.nkb_r + 3) / 4 * 4;
    return sh;
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
// With cols != 0 the kernel is b200va_quantize_fp8_blockwise's (fp8b_quant_body): A is rows x cols, S and St are
// f32, Ct and St may be null (and C and S), kind is an FP8B_* code, and block and rule are unused; the launch gives
// FP8B_THREADS threads and FP8B_SMEM bytes of dynamic shared memory on the tiled path, and no prefetch.  With an
// FP8R_* kind it is one of b200va_quantize_fp8_rowwise's three launches; FP8R_REDUCE reads the workspace at A and
// writes S to C and St to Ct.
// The launch bounds keep the register count at the 1-D launches' occupancy (two 512-thread CTAs per SM, one for f64),
// which the blockwise body alone would exceed.
template <int ES>
__global__ void __launch_bounds__(512, ES == 8 ? 1 : 2)
mx_quant_vec(const void* A, void* C, void* S, size_t n, size_t ngroups, int unroll, int prefetch_first, int src, int fmt,
             int block, int rule, void* Ct, void* St, size_t rows, size_t cols, int kind)
{
    const unsigned char* a = static_cast<const unsigned char*>(A);
    unsigned char* c = static_cast<unsigned char*>(C);
    unsigned char* sc = static_cast<unsigned char*>(S);
    prefetch_first_tile<16, ES>(prefetch_first, a, 0, ngroups, unroll);
    pdl_wait();

    if (cols) {
        const fp8b_shape sh = fp8b_make_shape(rows, cols);
        if (kind == FP8R_REDUCE) {
            fp8r_reduce(static_cast<const float*>(A), static_cast<float*>(C), static_cast<float*>(Ct), sh);
            return;
        }

        mx_with_pair<ES>(src, fmt, [=](auto SRC, auto F8) {
            fp8b_quant_body<SRC, F8>(a, c, static_cast<float*>(S), static_cast<unsigned char*>(Ct), static_cast<float*>(St),
                                     ngroups, sh, kind);
        });
        return;
    }
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

// b200va_dequantize_fp8_blockwise: W = 16 / sizeof DST FP8 values (low bytes of v) times an f32 scale s of any value,
// rounded once to DST.  The FP8 value has at most 4 significant bits, so q s is exact in f64: f32 and f64 take
// dequant_slice (__fmul_rn rounds once; the f64 product is exact), f16 and bf16 round the exact f64 product to odd in
// f32 and then to nearest, one rounding by Boldo-Melquiond (24 >= 11 + 2 bits).
template <int F8, int DST>
__device__ __forceinline__ u32x4 fp8b_dequant_slice(unsigned long long v, float s)
{
    if constexpr (DST == DT_F32 || DST == DT_F64) {
        return dequant_slice<F8, DST>(v, s);
    } else {
        uint32_t d[4];
        const double sd = static_cast<double>(s);
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            const uint32_t h = f16x2_from_f8x2<F8>(static_cast<uint32_t>(v >> (16 * p)));
            d[p] = narrow2_f32<DST>(f32_round_odd(__dmul_rn(static_cast<double>(widen_f16(h & 0xffffu)), sd)),
                                    f32_round_odd(__dmul_rn(static_cast<double>(widen_f16(h >> 16)), sd)));
        }
        return u32x4{d[0], d[1], d[2], d[3]};
    }
}

// The blockwise dequantize after the dependency wait: dequant_body's layout (the vector body when cols % 16 == 0 and
// A and C sit on 16-byte boundaries, ngroups = n / 16; a slice then lies in one row and one block) with the f32 scale
// of the block element e = i cols + j lies in: sf[(j / 128) rows + i] (1 x 128), sf[(i / 128) L4 + j / 128] (128 x 128)
// or sf[i] (FP8R_ROWS).
template <int F8, int DST>
__device__ __forceinline__ void fp8b_dequant_body(const unsigned char* a, const float* sf, unsigned char* c, size_t n,
                                                  size_t ngroups, int unroll, const fp8b_shape& sh, int kind)
{
    constexpr int ES = dt_traits<DST>::size, W = 16 / ES;
    const double rd = __drcp_rn(static_cast<double>(sh.cols));
    const int jshift = kind == FP8R_ROWS ? 63 : 7;                // one scale per row: j >> 63 = 0
    auto scale_of = [=](size_t e) {
        size_t j;
        const size_t i = fp8b_div(e, sh.cols, rd, j);
        return sf[kind != FP8B_128X128 ? (j >> jshift) * sh.rows + i : (i / FP8B_TILE) * sh.l4 + j / FP8B_TILE];
    };
    struct unit { unsigned long long v; float s; };
    cast_tiles(unroll, ngroups * ES, [=](size_t u) { return unit{ld_bits<W>(a + u * W), scale_of(u * W)}; },
               [=](size_t u, const unit& in) { stg128_bits<ST_NA>(c + u * 16, fp8b_dequant_slice<F8, DST>(in.v, in.s)); });
    cast_edges(n, 0, ngroups * 16, [=](size_t e) {
        const u32x4 r = fp8b_dequant_slice<F8, DST>(ld_bits<1>(a + e), scale_of(e));
        st_elem<ES>(c + e * ES, r.x, r.y);
    });
}

// One kernel per destination element size, the type and the format picked at the top as in mx_quant_vec.  The body is
// fp8_dequant_vec's from element 0 (elements [0, 16 ngroups), each slice inside one block), with the scale of the
// block an element lies in.  With cols != 0 it is b200va_dequantize_fp8_blockwise's (fp8b_dequant_body): S holds f32
// scales, A is rows x cols, kind an FP8B_* code, and block is unused.
template <int ES>
__global__ void mx_dequant_vec(const void* A, const void* S, void* C, size_t n, size_t ngroups, int unroll,
                               int prefetch_first, int dst, int fmt, int block, size_t rows, size_t cols, int kind)
{
    const unsigned char* a = static_cast<const unsigned char*>(A);
    const unsigned char* sc = static_cast<const unsigned char*>(S);
    unsigned char* c = static_cast<unsigned char*>(C);
    prefetch_first_tile<16 / ES, 1>(prefetch_first, a, 0, ngroups * ES, unroll);
    pdl_wait();

    if (cols) {
        const fp8b_shape sh = fp8b_make_shape(rows, cols);
        mx_with_pair<ES>(dst, fmt, [=](auto DST, auto F8) {
            fp8b_dequant_body<F8, DST>(a, static_cast<const float*>(S), c, n, ngroups, unroll, sh, kind);
        });
        return;
    }
    const int shift = 31 - __clz(block);
    mx_with_pair<ES>(dst, fmt, [=](auto DST, auto F8) {
        dequant_body<F8, DST>(a, c, n, 0, ngroups, unroll, [=](size_t e) { return mx_scale<DST>(sc[e >> shift]); });
    });
}

}  // namespace b200va
