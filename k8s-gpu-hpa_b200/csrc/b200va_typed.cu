// b200va_typed.cu -- the STREAM ops (copy, scale, add, triad), the reproducible dot product, the
// conversions between f32, f64, f16 and bf16, and the FP8 quantize and dequantize.  The only unit that
// includes the STREAM, dot, convert and FP8 kernels (b200va_dot.cuh and b200va_fp8.cuh, which include
// b200va_convert.cuh and b200va_stream.cuh).
#include "b200va_internal.h"
#include "b200va_fp8.cuh"
#include "b200va_dot.cuh"

using namespace b200va;

namespace {

// Bytes per element of a dtype.
size_t dtype_size(int dtype) { return dtype == DT_F64 ? 8 : dtype == DT_F32 ? 4 : 2; }

// Elements of `es` bytes before the first 16-byte boundary at or after address `a`: the scalar head
// a vector body peels off.
size_t head_peel(uintptr_t a, size_t es) { return ((16u - (a & 15u)) & 15u) / es; }

// The stream_vec forms each library carries (every DT): the production library only the two plain forms and
// the ST_NA form the HBM class picks, the tune library every form B200VA_STREAM_GEOMETRY can ask for.
template <int OP, int UNROLL, int ST>
constexpr bool carries_stream()
{
#ifdef B200VA_TUNE_MATRIX
    return true;
#else
    return UNROLL <= 2 && (ST == ST_PLAIN || UNROLL == (OP == OP_ADD || OP == OP_TRIAD ? 1 : 2));
#endif
}

template <int DT, int OP>
int launch_stream_typed(const void* dA, const void* dB, void* dC, size_t n, double scalar, cudaStream_t st)
{
    using S = typename dt_traits<DT>::scalar;
    constexpr size_t ES = dt_traits<DT>::size;
    constexpr bool binary = (OP == OP_ADD || OP == OP_TRIAD);
    const S s = static_cast<S>(scalar);
    const uintptr_t a = reinterpret_cast<uintptr_t>(dA), b = reinterpret_cast<uintptr_t>(dB),
                    c = reinterpret_cast<uintptr_t>(dC);
    const bool vec_ok = (a & 15u) == (c & 15u) && (!binary || (b & 15u) == (a & 15u));
    if (!vec_ok) {
        const size_t blocks = (n + 255) / 256;
        if (blocks > 0x7fffffffull) return B200VA_ERR_INVALID;
        stream_scalar<DT, OP><<<static_cast<unsigned>(blocks), 256, 0, st>>>(dA, dB, dC, n, s);
        return cuda_err(cudaGetLastError());
    }
    size_t head = head_peel(a, ES);
    if (head > n) head = n;
    const size_t nvec = (n - head) * ES / 16;
    // same footprint classes as the f32 add (default_tune), in 4-byte units
    const size_t m = n * ES / 4;
    const bool hbm = hbm_class(n, ES);
    unsigned threads = 128;
    int unroll = 1, st_hint = ST_PLAIN;
    if (hbm) {
        // three-array ops like the add: 512 x 1; two-array ops (copy, scale) want twice the bytes in
        // flight per thread: 1024 x 2; stores skip L1
        threads = binary ? 512 : 1024;
        unroll = binary ? 1 : 2;
        st_hint = ST_NA;
    } else if (m > (size_t{1} << 23)) { threads = 128; unroll = 2; }
    else if (m >= (size_t{1} << 21)) { threads = 256; unroll = 2; }
    else if (m >= (size_t{1} << 19)) { threads = 512; }
#ifdef B200VA_TUNE_MATRIX
    // development knob for A/B runs (tune library only): B200VA_STREAM_GEOMETRY="threads,unroll,skip_l1_stores"
    static const struct Override { int threads = 0, unroll = 0, na = 0; } ov = [] {
        Override o;
        if (const char* e = std::getenv("B200VA_STREAM_GEOMETRY")) std::sscanf(e, "%d,%d,%d", &o.threads, &o.unroll, &o.na);
        return o;
    }();
    if (ov.threads >= 32 && ov.threads <= 1024 && (ov.threads & 31) == 0 && (ov.unroll == 1 || ov.unroll == 2 || ov.unroll == 4)) {
        threads = static_cast<unsigned>(ov.threads);
        unroll = ov.unroll;
        st_hint = ov.na ? ST_NA : ST_PLAIN;
    }
#endif
    const size_t tile_vecs = static_cast<size_t>(threads) * unroll;
    const size_t ntiles = (nvec + tile_vecs - 1) / tile_vecs;
    const size_t grid = std::max<size_t>(std::min<size_t>(ntiles, 0x7fffffff), 1);
    using fn_t = void (*)(const void*, const void*, void*, size_t, size_t, size_t, size_t, S, int);
    const int prefetch_first = hbm ? 1 : 0;
    fn_t fn = nullptr;
    with_value<1, 2, 4>(unroll, [&](auto U) {
    with_value<ST_PLAIN, ST_NA>(st_hint, [&](auto ST) {
        if constexpr (carries_stream<OP, U, ST>()) fn = stream_vec<DT, OP, U, LD_PLAIN, ST>;
    }); });
    if (!fn) return B200VA_ERR_VARIANT;
    return launch_kernel(fn, static_cast<unsigned>(grid), threads, 0, st, pdl_enabled(), dA, dB, dC, n, head, nvec, ntiles, s, prefetch_first);
}

// Pass 1 of b200va_dot: one CTA per chunk, one f64 partial each into ws.  The vector form when A and
// B share a 16-byte phase, else the scalar form; the HBM class prefetches each CTA's first rows into L2
// ahead of the programmatic dependency.
template <int DT>
int launch_dot_typed(const void* dA, const void* dB, size_t n, double* ws, cudaStream_t st)
{
    constexpr size_t ES = dt_traits<DT>::size;
    const uintptr_t a = reinterpret_cast<uintptr_t>(dA), b = reinterpret_cast<uintptr_t>(dB);
    const unsigned grid = static_cast<unsigned>((n + DOT_CHUNK - 1) / DOT_CHUNK);
    const int prefetch_first = hbm_class(n, ES) ? 1 : 0;
    if ((a & 15u) != (b & 15u))
        return launch_kernel(dot_scalar<DT>, grid, DOT_SCALAR_THREADS, 0, st, pdl_enabled(), dA, dB, n, ws, prefetch_first);
    using F = dot_form<DT>;
    return launch_kernel(dot_vec<DT, F::threads, F::rows>, grid, F::threads, 0, st, pdl_enabled(), dA, dB, n, head_peel(a, ES),
                         ws, prefetch_first);
}

// The launch of a cast kernel (convert_vec, fp8_quant_vec, fp8_dequant_vec) over n elements of esa bytes at a to
// esc bytes at c.  A group is G = 16 / min(esa, esc) elements, one 16-byte vector on the narrow side, and a thread's
// unit of work is 1 / units_per_group of a group.  The head is the smallest h < G at which A and C both sit on a
// 16-byte boundary; with none (mixed phase) head = n, and the kernel's edge loop takes every element.  The geometry
// follows the HBM class of the wider operand: 512 x 2 with the L2 prefetch there, 256 x 1 below it (neither
// measured yet).
struct cast_plan {
    size_t head, ngroups;
    unsigned grid, threads;
    int unroll, prefetch_first;
};

cast_plan plan_cast(uintptr_t a, size_t esa, uintptr_t c, size_t esc, size_t n, size_t units_per_group)
{
    const size_t G = 16 / std::min(esa, esc);
    cast_plan p;
    p.head = n;
    for (size_t h = head_peel(a, esa); h < G; h += 16 / esa)
        if (((c + h * esc) & 15u) == 0) { p.head = h; break; }
    if (p.head > n) p.head = n;
    p.ngroups = (n - p.head) / G;
    const size_t units = p.ngroups * units_per_group, edges = n - p.ngroups * G;
    const bool hbm = hbm_class(n, std::max(esa, esc));
    p.threads = hbm ? 512 : 256;
    p.unroll = hbm ? 2 : 1;
    p.prefetch_first = hbm ? 1 : 0;
    const size_t tile = static_cast<size_t>(p.threads) * p.unroll;
    const size_t blocks = std::max((units + tile - 1) / tile, (edges + p.threads - 1) / p.threads);
    p.grid = static_cast<unsigned>(std::max<size_t>(std::min<size_t>(blocks, 0x7fffffff), 1));
    return p;
}

// b200va_convert between two distinct types: one convert_vec launch, a group per unit.
template <int SRC, int DST>
int launch_convert_typed(const void* dA, void* dC, size_t n, cudaStream_t st)
{
    const cast_plan p = plan_cast(reinterpret_cast<uintptr_t>(dA), dt_traits<SRC>::size, reinterpret_cast<uintptr_t>(dC),
                                  dt_traits<DST>::size, n, 1);
    return launch_kernel(convert_vec<SRC, DST>, p.grid, p.threads, 0, st, pdl_enabled(), dA, dC, n, p.head, p.ngroups,
                         p.unroll, p.prefetch_first);
}

// b200va_quantize_fp8 (QUANT: T -> fmt) and b200va_dequantize_fp8 (fmt -> T): one fp8_quant_vec<T> or
// fp8_dequant_vec<T> launch, the format passed to the kernel.  A unit is a group of 16 when quantizing and a 16-byte
// output slice (sizeof T per group) when dequantizing.
template <bool QUANT, int T>
int launch_fp8_typed(const void* dA, void* dC, size_t n, int fmt, int k, double* amax, cudaStream_t st)
{
    constexpr size_t ES = dt_traits<T>::size;
    const cast_plan p = plan_cast(reinterpret_cast<uintptr_t>(dA), QUANT ? ES : 1, reinterpret_cast<uintptr_t>(dC),
                                  QUANT ? 1 : ES, n, QUANT ? 1 : ES);
    if constexpr (QUANT)
        return launch_kernel(fp8_quant_vec<T>, p.grid, p.threads, 0, st, pdl_enabled(), dA, dC, n, p.head, p.ngroups,
                             p.unroll, p.prefetch_first, fmt, k, amax);
    else
        return launch_kernel(fp8_dequant_vec<T>, p.grid, p.threads, 0, st, pdl_enabled(), dA, dC, n, p.head, p.ngroups,
                             p.unroll, p.prefetch_first, fmt, k);
}

// The argument rules the two FP8 entry points share, after the dtype and format codes: scale_exp in [-126, 126],
// then A and C as b200va_convert checks them (1-byte FP8 elements), then d_amax (may be NULL) 8-byte aligned and
// meeting neither A nor C.
int check_fp8_args(size_t es, const void* dA, size_t esc, const void* dC, size_t n, int k, const double* d_amax)
{
    if (k < -126 || k > 126) return B200VA_ERR_INVALID;
    RC_TRY(check_convert_operands(es, dA, esc, dC, n));
    const uintptr_t m = reinterpret_cast<uintptr_t>(d_amax), a = reinterpret_cast<uintptr_t>(dA),
                    c = reinterpret_cast<uintptr_t>(dC);
    if (m & 7u) return B200VA_ERR_ALIGN;
    auto meet = [&](uintptr_t x, size_t bytes) { return m && n && m < x + bytes && x < m + 8; };
    if (meet(a, n * es) || meet(c, n * esc)) return B200VA_ERR_OVERLAP;
    return B200VA_OK;
}

}  // namespace

// ========================================= ABI (C linkage from the declarations in include/b200va.h)
// ------------------------------------------------------------------ f4: STREAM-style ops
int b200va_stream(int op, int dtype, const void* dA, const void* dB, void* dC, size_t n, double scalar, void* stream)
{
    if (op < 0 || op >= OP_COUNT || dtype < 0 || dtype >= DT_COUNT) return B200VA_ERR_VARIANT;
    RC_TRY(current_dev_info(nullptr));
    RC_TRY(check_operands(dtype_size(dtype), dA, dB, dC, n, op == OP_ADD || op == OP_TRIAD));
    if (n == 0) return B200VA_OK;
    int rc = B200VA_ERR_VARIANT;
    with_value<DT_F32, DT_F64, DT_F16, DT_BF16>(dtype, [&](auto DT) {
    with_value<OP_COPY, OP_SCALE, OP_ADD, OP_TRIAD>(op, [&](auto OP) {
        rc = launch_stream_typed<DT, OP>(dA, dB, dC, n, scalar, static_cast<cudaStream_t>(stream));
    }); });
    return rc;
}

int b200va_convert(int src_dtype, const void* dA, int dst_dtype, void* dC, size_t n, void* stream)
{
    if (src_dtype < 0 || src_dtype >= DT_COUNT || dst_dtype < 0 || dst_dtype >= DT_COUNT) return B200VA_ERR_VARIANT;
    RC_TRY(current_dev_info(nullptr));
    RC_TRY(check_convert_operands(dtype_size(src_dtype), dA, dtype_size(dst_dtype), dC, n));
    if (n == 0) return B200VA_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc = B200VA_ERR_VARIANT;
    with_value<DT_F32, DT_F64, DT_F16, DT_BF16>(src_dtype, [&](auto SRC) {
        if (src_dtype == dst_dtype) { rc = launch_stream_typed<SRC, OP_COPY>(dA, nullptr, dC, n, 0.0, st); return; }
        with_value<DT_F32, DT_F64, DT_F16, DT_BF16>(dst_dtype, [&](auto DST) {
            if constexpr (SRC != DST) rc = launch_convert_typed<SRC, DST>(dA, dC, n, st);
        });
    });
    return rc;
}

int b200va_quantize_fp8(int src_dtype, const void* dA, int fp8, void* dC, size_t n, int scale_exp, double* d_amax,
                        void* stream)
{
    if (src_dtype < 0 || src_dtype >= DT_COUNT || fp8 < 0 || fp8 >= F8_COUNT) return B200VA_ERR_VARIANT;
    RC_TRY(current_dev_info(nullptr));
    RC_TRY(check_fp8_args(dtype_size(src_dtype), dA, 1, dC, n, scale_exp, d_amax));
    if (n == 0) return B200VA_OK;
    int rc = B200VA_ERR_VARIANT;
    with_value<DT_F32, DT_F64, DT_F16, DT_BF16>(src_dtype, [&](auto SRC) {
        rc = launch_fp8_typed<true, SRC>(dA, dC, n, fp8, scale_exp, d_amax, static_cast<cudaStream_t>(stream));
    });
    return rc;
}

int b200va_dequantize_fp8(int fp8, const void* dA, int dst_dtype, void* dC, size_t n, int scale_exp, void* stream)
{
    if (dst_dtype < 0 || dst_dtype >= DT_COUNT || fp8 < 0 || fp8 >= F8_COUNT) return B200VA_ERR_VARIANT;
    RC_TRY(current_dev_info(nullptr));
    RC_TRY(check_fp8_args(1, dA, dtype_size(dst_dtype), dC, n, scale_exp, nullptr));
    if (n == 0) return B200VA_OK;
    int rc = B200VA_ERR_VARIANT;
    with_value<DT_F32, DT_F64, DT_F16, DT_BF16>(dst_dtype, [&](auto DST) {
        rc = launch_fp8_typed<false, DST>(dA, dC, n, fp8, scale_exp, nullptr, static_cast<cudaStream_t>(stream));
    });
    return rc;
}

size_t b200va_dot_workspace_bytes(size_t n)
{
    return 8 * (n / DOT_CHUNK + (n % DOT_CHUNK != 0));
}

int b200va_dot(int dtype, const void* dA, const void* dB, size_t n, double* d_out, void* d_workspace,
               size_t workspace_bytes, void* stream)
{
    if (dtype < 0 || dtype >= DT_COUNT) return B200VA_ERR_VARIANT;
    RC_TRY(current_dev_info(nullptr));
    if (n > (size_t{1} << 40)) return B200VA_ERR_INVALID;
    const size_t need = b200va_dot_workspace_bytes(n);
    if (!d_out || (n && (!dA || !dB)) || (need && !d_workspace) || workspace_bytes < need) return B200VA_ERR_INVALID;
    const size_t es = dtype_size(dtype);
    const uintptr_t a = reinterpret_cast<uintptr_t>(dA), b = reinterpret_cast<uintptr_t>(dB),
                    o = reinterpret_cast<uintptr_t>(d_out), w = reinterpret_cast<uintptr_t>(d_workspace);
    if (n && ((a | b) & (es - 1)) != 0) return B200VA_ERR_ALIGN;
    if ((o & 7u) || (need && (w & 7u))) return B200VA_ERR_ALIGN;
    // what the call writes (d_out, the needed workspace) must not meet what it reads or each other
    auto meet = [](uintptr_t x, size_t xn, uintptr_t y, size_t yn) { return xn && yn && x < y + yn && y < x + xn; };
    const size_t bytes = n * es;
    if (meet(o, 8, a, bytes) || meet(o, 8, b, bytes) || meet(o, 8, w, need) || meet(w, need, a, bytes) ||
        meet(w, need, b, bytes))
        return B200VA_ERR_OVERLAP;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    double* ws = static_cast<double*>(d_workspace);
    int rc = B200VA_OK;
    if (n) with_value<DT_F32, DT_F64, DT_F16, DT_BF16>(dtype, [&](auto DT) { rc = launch_dot_typed<DT>(dA, dB, n, ws, st); });
    RC_TRY(rc);
    // pass 2: aligned blocks of DOT_FINAL_BLOCK partials per CTA, one level per launch, until one CTA
    // writes *d_out (for n = 0 it sums nothing and writes +0.0)
    size_t k = need / 8, stride = 1;
    while (k > static_cast<size_t>(DOT_FINAL_BLOCK)) {
        const size_t grid = (k + DOT_FINAL_BLOCK - 1) / DOT_FINAL_BLOCK;
        RC_TRY(launch_kernel(dot_final, static_cast<unsigned>(grid), DOT_FINAL_THREADS, 0, st, pdl_enabled(), ws, k, stride,
                             static_cast<double*>(nullptr)));
        k = grid;
        stride *= DOT_FINAL_BLOCK;
    }
    return launch_kernel(dot_final, 1u, DOT_FINAL_THREADS, 0, st, pdl_enabled(), ws, k, stride, d_out);
}
