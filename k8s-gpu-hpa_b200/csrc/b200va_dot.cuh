// b200va_dot.cuh -- the reproducible dot product of row f4 (b200va_dot, include/b200va.h).
//
// The result is a function of the values and n only (never of the grid, the SM count, the
// alignment, the stream or the run), defined by three rules over LANES = 2048, CHUNK = 65536:
//   1. lane chain   lane l of chunk k holds the elements i of the chunk with i mod LANES == l and
//                   accumulates them in increasing order: acc = +0.0; acc = fma(a_i, b_i, acc) in
//                   binary64 RNE, operands widened exactly (no FTZ)
//   2. chunk value  the 2048 lane values summed as an aligned dyadic (pairwise) tree
//   3. total        the chunk values summed with the same tree; an empty upper half passes the
//                   lower half up unchanged (equivalently: padded with +0.0, as nothing is -0.0)
// Pass 1 (dot_vec, or dot_scalar when A and B sit in different 16-byte phases) runs one CTA per
// chunk: each thread owns a fixed set of lanes and runs their chains in f64 registers, then the
// CTA sums its 2048 lanes with the tree and writes one f64 partial per chunk into the workspace.
// Pass 2 (dot_final, a second launch behind a programmatic dependency) sums the partials with the
// tree; more than DOT_FINAL_BLOCK partials take one more launch per level, each summing aligned
// blocks of DOT_FINAL_BLOCK.  Both passes keep no state between calls.
#pragma once
#include <type_traits>

#include "b200va_stream.cuh"

namespace b200va {

constexpr int DOT_LANES = 2048;
constexpr int DOT_CHUNK = 65536;
constexpr int DOT_ROWS = DOT_CHUNK / DOT_LANES;          // elements per lane of a full chunk
constexpr int DOT_FINAL_THREADS = 1024;
constexpr int DOT_FINAL_PER_THREAD = 8;
constexpr int DOT_FINAL_BLOCK = DOT_FINAL_THREADS * DOT_FINAL_PER_THREAD;   // partials per pass-2 CTA
constexpr int DOT_SCALAR_THREADS = 512;
constexpr int DOT_SCALAR_ROWS = 4;

// The pass-1 form per dtype: CTA size, rows (16-byte loads per array per owned column) in flight,
// and the CTAs an SM must hold (caps registers at 65536 / (threads * min_ctas)).  Lanes per thread
// are LANES / threads: 4 for f32 and f64, 8 for f16 and bf16.
template <int DT> struct dot_form;
template <> struct dot_form<DT_F32>  { static constexpr int threads = 512, rows = 4, min_ctas = 2; };
template <> struct dot_form<DT_F64>  { static constexpr int threads = 512, rows = 2, min_ctas = 2; };
template <> struct dot_form<DT_F16>  { static constexpr int threads = 256, rows = 4, min_ctas = 4; };
template <> struct dot_form<DT_BF16> { static constexpr int threads = 256, rows = 4, min_ctas = 4; };

// ---- one lane step: acc = fma(a, b, acc) over the exact f64 widenings ------------------------------
// f32 and bf16 products are exact in f64, so the fma rounds once, as acc + a*b would.  An f16 product
// (11 x 11 significant bits, exponents within f32's range) is already exact in f32, which saves one
// widening per element and gives the same bits.
template <int DT>
__device__ __forceinline__ double dot_step(double acc, uint32_t a, uint32_t b)
{
    if constexpr (DT == DT_F32)
        return __fma_rn(static_cast<double>(__uint_as_float(a)), static_cast<double>(__uint_as_float(b)), acc);
    else if constexpr (DT == DT_F16)
        return __dadd_rn(acc, static_cast<double>(__fmul_rn(widen_f16(a), widen_f16(b))));
    else
        return __fma_rn(static_cast<double>(widen_bf16(a)), static_cast<double>(widen_bf16(b)), acc);
}

__device__ __forceinline__ double dot_step64(double acc, double a, double b) { return __fma_rn(a, b, acc); }

// Element e (0 .. 16/ES - 1, a constant after unrolling) of a 16-byte vector pair.
template <int DT>
__device__ __forceinline__ double dot_step_vec(double acc, const u32x4& a, const u32x4& b, int e)
{
    const uint32_t wa[4] = {a.x, a.y, a.z, a.w}, wb[4] = {b.x, b.y, b.z, b.w};
    if constexpr (DT == DT_F64)
        return dot_step64(acc, __hiloint2double(static_cast<int>(wa[2 * e + 1]), static_cast<int>(wa[2 * e])),
                          __hiloint2double(static_cast<int>(wb[2 * e + 1]), static_cast<int>(wb[2 * e])));
    else if constexpr (DT == DT_F32)
        return dot_step<DT>(acc, wa[e], wb[e]);
    else
        return dot_step<DT>(acc, (wa[e / 2] >> (16 * (e % 2))) & 0xffffu, (wb[e / 2] >> (16 * (e % 2))) & 0xffffu);
}

// One element at byte pointers a, b (element-size aligned).
template <int DT>
__device__ __forceinline__ double dot_step_elem(double acc, const unsigned char* a, const unsigned char* b)
{
    if constexpr (DT == DT_F64)
        return dot_step64(acc, *reinterpret_cast<const double*>(a), *reinterpret_cast<const double*>(b));
    else if constexpr (DT == DT_F32)
        return dot_step<DT>(acc, *reinterpret_cast<const uint32_t*>(a), *reinterpret_cast<const uint32_t*>(b));
    else
        return dot_step<DT>(acc, *reinterpret_cast<const unsigned short*>(a), *reinterpret_cast<const unsigned short*>(b));
}

// ---- the aligned dyadic tree -----------------------------------------------------------------------
// x[0 .. N) of one thread: blocks of 2, 4, ... N, each the sum of its two halves.
template <int N>
__device__ __forceinline__ double tree_serial(double* x)
{
#pragma unroll
    for (int w = 1; w < N; w *= 2)
#pragma unroll
        for (int i = 0; i < N; i += 2 * w) x[i] = __dadd_rn(x[i], x[i + w]);
    return x[0];
}

// Lane 0 of the warp gets the tree over the 32 lanes' values in lane order.  Step `off` adds to each
// lane the block that starts `off` lanes higher; the lanes read at the next step are multiples of
// 2 * off, whose values are then exactly their aligned blocks.
__device__ __forceinline__ double tree_warp(double v)
{
#pragma unroll
    for (int off = 1; off < 32; off *= 2) v = __dadd_rn(v, __shfl_down_sync(0xffffffffu, v, off));
    return v;
}

// Tree over the CTA's values in thread order, PER consecutive values per thread in `x`.  The result is
// valid in thread 0.  THREADS / 32 <= 32 warps; missing warps are +0.0, which leaves every sum as it is.
template <int THREADS, int PER>
__device__ __forceinline__ double tree_cta(double* x, double* warp_sums)
{
    double v = tree_warp(tree_serial<PER>(x));
    const unsigned warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    if (lane == 0) warp_sums[warp] = v;
    __syncthreads();
    if (warp == 0) v = tree_warp(lane < THREADS / 32 ? warp_sums[lane] : 0.0);
    return v;
}

// In the HBM class (prefetch_first), thread 0 bulk-prefetches the first `bytes` of each operand's
// chunk into L2 ahead of the programmatic dependency (always legal: L2 is the point of coherence).
__device__ __forceinline__ void dot_prefetch(const unsigned char* a, const unsigned char* b, size_t len_bytes, size_t bytes)
{
    // 16-byte-aligned starts; the operands may sit in different phases
    const unsigned char* pa = reinterpret_cast<const unsigned char*>((reinterpret_cast<uintptr_t>(a) + 15) & ~uintptr_t{15});
    const unsigned char* pb = reinterpret_cast<const unsigned char*>((reinterpret_cast<uintptr_t>(b) + 15) & ~uintptr_t{15});
    const size_t skip = (pa - a) > (pb - b) ? (pa - a) : (pb - b);
    if (len_bytes <= skip) return;
    if (bytes > len_bytes - skip) bytes = len_bytes - skip;
    bytes &= ~size_t{15};
    if (bytes == 0) return;
    bulk_prefetch_l2(pa, static_cast<uint32_t>(bytes));
    bulk_prefetch_l2(pb, static_cast<uint32_t>(bytes));
}

// ---- pass 1, vector form ---------------------------------------------------------------------------
// A and B in the same 16-byte phase; `head` = elements before the first 16-byte boundary (the same in
// every chunk, as a chunk is a multiple of 16 bytes).  In chunk-relative element indices the 16-byte
// vectors start at e0 + EPV v, with e0 = head - EPV if head > 0 (the first vector straddles the chunk
// start) and 0 otherwise.  Vector v is column v mod NC of row v / NC; every column holds the same EPV
// lanes in every row, so a thread that owns columns and walks their rows in order runs the lane chains
// in index order.  With head > 0 a vector can straddle the chunk's start or end, and column 0 has one
// more row (the chunk's last EPV - head elements); vectors not wholly inside [0, len) load only their
// elements that are.
template <int DT, int THREADS, int ROWS>
__global__ void __launch_bounds__(THREADS, dot_form<DT>::min_ctas)
dot_vec(const void* A, const void* B, size_t n, size_t head, double* partials, int prefetch_first)
{
    constexpr int ES = dt_traits<DT>::size;
    constexpr int EPV = 16 / ES;
    constexpr int NC = DOT_LANES / EPV;                  // 16-byte columns of a row
    constexpr int COLS = NC / THREADS;                   // columns per thread
    constexpr int PER = DOT_LANES / THREADS;             // lanes per thread
    static_assert(COLS * THREADS == NC && DOT_ROWS % ROWS == 0, "dot_vec geometry");
    __shared__ double lane_val[DOT_LANES];
    __shared__ double warp_sums[32];

    const size_t base = static_cast<size_t>(blockIdx.x) * DOT_CHUNK;
    const int len = n - base < static_cast<size_t>(DOT_CHUNK) ? static_cast<int>(n - base) : DOT_CHUNK;
    const unsigned char* a = static_cast<const unsigned char*>(A) + base * ES;
    const unsigned char* b = static_cast<const unsigned char*>(B) + base * ES;
    const int e0 = head ? static_cast<int>(head) - EPV : 0;
    if (prefetch_first && threadIdx.x == 0) dot_prefetch(a, b, static_cast<size_t>(len) * ES, size_t{ROWS} * DOT_LANES * ES);
    pdl_wait();

    double acc[COLS][EPV];
#pragma unroll
    for (int q = 0; q < COLS; ++q)
#pragma unroll
        for (int e = 0; e < EPV; ++e) acc[q][e] = 0.0;

    // the vectors of the elements that exist, one element at a time
    auto partial = [&](int s, int q) {
#pragma unroll
        for (int e = 0; e < EPV; ++e)
            if (s + e >= 0 && s + e < len) acc[q][e] = dot_step_elem<DT>(acc[q][e], a + (s + e) * ES, b + (s + e) * ES);
    };
    const int c0 = e0 + EPV * static_cast<int>(threadIdx.x);          // chunk index of column threadIdx.x, row 0
    for (int r0 = 0; r0 < DOT_ROWS; r0 += ROWS) {
        const int first = c0 + DOT_LANES * r0;
        const int last = c0 + EPV * THREADS * (COLS - 1) + DOT_LANES * (r0 + ROWS - 1);
        if (first >= 0 && last + EPV <= len) {
            u32x4 ra[ROWS][COLS], rb[ROWS][COLS];
#pragma unroll
            for (int r = 0; r < ROWS; ++r)
#pragma unroll
                for (int q = 0; q < COLS; ++q) ra[r][q] = ldg128_bits<LD_PLAIN>(a + (first + DOT_LANES * r + EPV * THREADS * q) * ES);
#pragma unroll
            for (int r = 0; r < ROWS; ++r)
#pragma unroll
                for (int q = 0; q < COLS; ++q) rb[r][q] = ldg128_bits<LD_PLAIN>(b + (first + DOT_LANES * r + EPV * THREADS * q) * ES);
#pragma unroll
            for (int r = 0; r < ROWS; ++r)
#pragma unroll
                for (int q = 0; q < COLS; ++q)
#pragma unroll
                    for (int e = 0; e < EPV; ++e) acc[q][e] = dot_step_vec<DT>(acc[q][e], ra[r][q], rb[r][q], e);
        } else {
            for (int r = 0; r < ROWS; ++r)
#pragma unroll
                for (int q = 0; q < COLS; ++q) partial(first + DOT_LANES * r + EPV * THREADS * q, q);
        }
    }
    if (head && threadIdx.x == 0) partial(e0 + DOT_CHUNK, 0);         // column 0, row DOT_ROWS

#pragma unroll
    for (int q = 0; q < COLS; ++q)
#pragma unroll
        for (int e = 0; e < EPV; ++e)
            lane_val[(e0 + DOT_LANES + EPV * (static_cast<int>(threadIdx.x) + THREADS * q) + e) & (DOT_LANES - 1)] = acc[q][e];
    __syncthreads();
    double x[PER];
#pragma unroll
    for (int i = 0; i < PER; ++i) x[i] = lane_val[threadIdx.x * PER + i];
    const double v = tree_cta<THREADS, PER>(x, warp_sums);
    if (threadIdx.x == 0) partials[blockIdx.x] = v;
}

// ---- pass 1, scalar form ---------------------------------------------------------------------------
// A and B in different 16-byte phases: thread t owns lanes t + DOT_SCALAR_THREADS j and loads one
// element at a time, ROWS rows in flight.
template <int DT>
__global__ void __launch_bounds__(DOT_SCALAR_THREADS)
dot_scalar(const void* A, const void* B, size_t n, double* partials, int prefetch_first)
{
    constexpr int ES = dt_traits<DT>::size;
    constexpr int PER = DOT_LANES / DOT_SCALAR_THREADS;
    constexpr int ROWS = DOT_SCALAR_ROWS;
    __shared__ double lane_val[DOT_LANES];
    __shared__ double warp_sums[32];

    const size_t base = static_cast<size_t>(blockIdx.x) * DOT_CHUNK;
    const int len = n - base < static_cast<size_t>(DOT_CHUNK) ? static_cast<int>(n - base) : DOT_CHUNK;
    const unsigned char* a = static_cast<const unsigned char*>(A) + base * ES;
    const unsigned char* b = static_cast<const unsigned char*>(B) + base * ES;
    if (prefetch_first && threadIdx.x == 0) dot_prefetch(a, b, static_cast<size_t>(len) * ES, size_t{ROWS} * DOT_LANES * ES);
    pdl_wait();

    double acc[PER];
#pragma unroll
    for (int j = 0; j < PER; ++j) acc[j] = 0.0;
    for (int r0 = 0; r0 < DOT_ROWS; r0 += ROWS) {
        if (DOT_LANES * (r0 + ROWS) <= len) {
            if constexpr (DT == DT_F64) {
                double xa[ROWS][PER], xb[ROWS][PER];
#pragma unroll
                for (int r = 0; r < ROWS; ++r)
#pragma unroll
                    for (int j = 0; j < PER; ++j) {
                        const int i = DOT_LANES * (r0 + r) + threadIdx.x + DOT_SCALAR_THREADS * j;
                        xa[r][j] = reinterpret_cast<const double*>(a)[i];
                        xb[r][j] = reinterpret_cast<const double*>(b)[i];
                    }
#pragma unroll
                for (int r = 0; r < ROWS; ++r)
#pragma unroll
                    for (int j = 0; j < PER; ++j) acc[j] = dot_step64(acc[j], xa[r][j], xb[r][j]);
            } else {
                using W = std::conditional_t<ES == 4, uint32_t, unsigned short>;
                uint32_t xa[ROWS][PER], xb[ROWS][PER];
#pragma unroll
                for (int r = 0; r < ROWS; ++r)
#pragma unroll
                    for (int j = 0; j < PER; ++j) {
                        const int i = DOT_LANES * (r0 + r) + threadIdx.x + DOT_SCALAR_THREADS * j;
                        xa[r][j] = reinterpret_cast<const W*>(a)[i];
                        xb[r][j] = reinterpret_cast<const W*>(b)[i];
                    }
#pragma unroll
                for (int r = 0; r < ROWS; ++r)
#pragma unroll
                    for (int j = 0; j < PER; ++j) acc[j] = dot_step<DT>(acc[j], xa[r][j], xb[r][j]);
            }
        } else {
            for (int r = r0; r < r0 + ROWS; ++r)
#pragma unroll
                for (int j = 0; j < PER; ++j) {
                    const int i = DOT_LANES * r + threadIdx.x + DOT_SCALAR_THREADS * j;
                    if (i < len) acc[j] = dot_step_elem<DT>(acc[j], a + i * ES, b + i * ES);
                }
        }
    }
#pragma unroll
    for (int j = 0; j < PER; ++j) lane_val[threadIdx.x + DOT_SCALAR_THREADS * j] = acc[j];
    __syncthreads();
    double x[PER];
#pragma unroll
    for (int i = 0; i < PER; ++i) x[i] = lane_val[threadIdx.x * PER + i];
    const double v = tree_cta<DOT_SCALAR_THREADS, PER>(x, warp_sums);
    if (threadIdx.x == 0) partials[blockIdx.x] = v;
}

// ---- pass 2 ----------------------------------------------------------------------------------------
// CTA i sums entries [i DOT_FINAL_BLOCK, (i + 1) DOT_FINAL_BLOCK) of the k values at p[j * stride]
// (entries past k are +0.0) and writes the sum to *out (one CTA) or over its own first entry,
// p[i DOT_FINAL_BLOCK stride], which the next level reads at stride DOT_FINAL_BLOCK * stride.
__global__ void __launch_bounds__(DOT_FINAL_THREADS)
dot_final(double* p, size_t k, size_t stride, double* out)
{
    __shared__ double warp_sums[32];
    pdl_wait();
    const size_t j0 = static_cast<size_t>(blockIdx.x) * DOT_FINAL_BLOCK + static_cast<size_t>(threadIdx.x) * DOT_FINAL_PER_THREAD;
    double x[DOT_FINAL_PER_THREAD];
#pragma unroll
    for (int i = 0; i < DOT_FINAL_PER_THREAD; ++i) x[i] = j0 + i < k ? p[(j0 + i) * stride] : 0.0;
    const double v = tree_cta<DOT_FINAL_THREADS, DOT_FINAL_PER_THREAD>(x, warp_sums);
    if (threadIdx.x == 0) {
        if (out) *out = v;
        else p[static_cast<size_t>(blockIdx.x) * DOT_FINAL_BLOCK * stride] = v;
    }
}

}  // namespace b200va
