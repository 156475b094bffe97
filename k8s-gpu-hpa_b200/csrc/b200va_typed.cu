// b200va_typed.cu -- the STREAM ops (copy, scale, add, triad), the reproducible dot product, the
// conversions between f32, f64, f16 and bf16, the FP8 quantize and dequantize, per tensor and block-scaled, and the
// stochastically rounded casts from f32.
// The only unit that includes the STREAM, dot, convert, FP8 and SR kernels (b200va_dot.cuh, b200va_mxfp8.cuh and
// b200va_sr.cuh, which include b200va_fp8.cuh, b200va_convert.cuh and b200va_stream.cuh).
#include "b200va_internal.h"
#include "b200va_mxfp8.cuh"
#include "b200va_sr.cuh"
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

// What a cast launch is made of: the vector body (ngroups groups from element head on) and the launch geometry.
struct cast_plan {
    size_t head, ngroups;
    unsigned grid, threads;
    int unroll, prefetch_first;
};

// The geometry of a cast launch with `units` units of work in the vector body and `edges` items in the edge loop:
// 512 x 2 with the L2 prefetch in the HBM class, 256 x 1 below it (neither measured yet), and enough CTAs that every
// tile and every edge item has a thread.
void plan_geometry(cast_plan& p, bool hbm, size_t units, size_t edges)
{
    p.threads = hbm ? 512 : 256;
    p.unroll = hbm ? 2 : 1;
    p.prefetch_first = hbm ? 1 : 0;
    const size_t tile = static_cast<size_t>(p.threads) * p.unroll;
    const size_t blocks = std::max((units + tile - 1) / tile, (edges + p.threads - 1) / p.threads);
    p.grid = static_cast<unsigned>(std::max<size_t>(std::min<size_t>(blocks, 0x7fffffff), 1));
}

// Where the vector body of a cast over n elements of esa bytes at a to esc bytes at c lies (the geometry is not set).
// A group is G = 16 / min(esa, esc) elements, one 16-byte vector on the narrow side.  The head is the smallest h < G at
// which A and C both sit on a 16-byte boundary; with none (mixed phase) head = n, and the kernel's edge loop takes
// every element.
cast_plan cast_body(uintptr_t a, size_t esa, uintptr_t c, size_t esc, size_t n)
{
    const size_t G = 16 / std::min(esa, esc);
    cast_plan p{};
    p.head = n;
    for (size_t h = head_peel(a, esa); h < G; h += 16 / esa)
        if (((c + h * esc) & 15u) == 0) { p.head = h; break; }
    if (p.head > n) p.head = n;
    p.ngroups = (n - p.head) / G;
    return p;
}

// The launch of a cast kernel (convert_vec, fp8_quant_vec, fp8_dequant_vec): the body of cast_body, a thread's unit
// of work being 1 / units_per_group of a group and every element outside the body an edge item.  The geometry follows
// the HBM class of the wider operand.
cast_plan plan_cast(uintptr_t a, size_t esa, uintptr_t c, size_t esc, size_t n, size_t units_per_group)
{
    const size_t G = 16 / std::min(esa, esc);
    cast_plan p = cast_body(a, esa, c, esc, n);
    plan_geometry(p, hbm_class(n, std::max(esa, esc)), p.ngroups * units_per_group, n - p.ngroups * G);
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

// The arguments of one fp8_quant_vec launch besides its plan, set by name; a launch that sets only a, c, n, fmt, k and
// amax is the 1-D quantize by the host's k.  The kernel's mode follows from which pointers are set (b200va_fp8.cuh):
//   amax pass   c NULL: max-accumulates A's largest finite |a_i| into *amax and stores nothing (fmt and k unused)
//   auto k      amax_in: k = auto_scale_exp(*amax_in, fmt, margin), written to *k_out
//   transpose   ct: C's transpose also goes to Ct, A having `cols` columns
struct fp8_quant_args {
    const void* a = nullptr;
    void* c = nullptr;
    size_t n = 0;
    int fmt = 0, k = 0;
    double* amax = nullptr;
    const double* amax_in = nullptr;
    int margin = 0;
    int32_t* k_out = nullptr;
    void* ct = nullptr;
    size_t cols = 0;
};

using fp8_quant_fn = decltype(&fp8_quant_vec<DT_F32>);

// The one launch site of fp8_quant_vec: fn = fp8_quant_vec<T> under plan p, with smem bytes of dynamic shared memory.
int launch_fp8_quant(fp8_quant_fn fn, const cast_plan& p, size_t smem, const fp8_quant_args& q, cudaStream_t st)
{
    return launch_kernel(fn, p.grid, p.threads, smem, st, pdl_enabled(), q.a, q.c, q.n, p.head, p.ngroups, p.unroll,
                         p.prefetch_first, q.fmt, q.k, q.amax, q.amax_in, q.margin, q.k_out, q.ct, q.cols);
}

// The amax pass's plan, over n elements of es bytes at a.  There is no C to share a phase with, so the vector body
// starts at the head that puts A alone on a 16-byte boundary; a unit is a group of 16, and every element outside the
// body an edge item.  The geometry follows A's HBM class.
cast_plan plan_fp8_amax(uintptr_t a, size_t es, size_t n)
{
    cast_plan p{};
    p.head = std::min(head_peel(a, es), n);
    p.ngroups = (n - p.head) / 16;
    plan_geometry(p, hbm_class(n, es), p.ngroups, n - p.ngroups * 16);
    return p;
}

// The quantize-transpose's plan, n = rows cols > 0 elements of es bytes.  The tiled path runs when rows and cols are
// multiples of 16 and A, C and Ct sit on 16-byte boundaries: head 0, every group in the body, FP8T_THREADS threads per
// CTA (one per group of a tile), one tile per CTA and FP8T_SMEM bytes of dynamic shared memory (smem).  Otherwise the
// element path: head = n, every element an edge item, plan_geometry's threads and grid for A's HBM class.  Neither
// path prefetches a first tile, and neither geometry was tuned.
cast_plan plan_fp8_transpose(uintptr_t a, uintptr_t c, uintptr_t ct, size_t es, size_t rows, size_t cols, size_t& smem)
{
    constexpr size_t T8 = FP8T_TILE;
    const size_t n = rows * cols;
    cast_plan p{};
    smem = 0;
    if (rows % 16 == 0 && cols % 16 == 0 && ((a | c | ct) & 15u) == 0) {
        p.ngroups = n / 16;
        p.threads = FP8T_THREADS;
        p.unroll = 1;
        p.grid = static_cast<unsigned>(std::min<size_t>((rows + T8 - 1) / T8 * ((cols + T8 - 1) / T8), 0x7fffffff));
        smem = FP8T_SMEM;
    } else {
        p.head = n;
        plan_geometry(p, hbm_class(n, es), 0, n);
        p.prefetch_first = 0;
    }
    return p;
}

// The argument rules of every per-tensor FP8 cast after the dtype and format codes, in the order they apply.  A holds
// n elements of esa bytes and C n of esc, one side FP8 (a quantize has esc = 1).
//   1. k is the host's scale exponent, in [-126, 126]; with auto_k it is the margin, in [0, 126], d_scale_exp is
//      non-NULL, and a quantize's d_amax is non-NULL.
//   2. A and C as b200va_convert checks them.
//   3. d_amax (may be NULL) 8-byte aligned and meeting neither A nor C.
//   4. d_scale_exp (may be NULL) 4-byte aligned and meeting neither A, C nor d_amax.
//   5. For a quantize-transpose with n > 0: dCt non-NULL, and its n bytes meeting none of the others.
int check_fp8_args(size_t esa, const void* dA, size_t esc, const void* dC, size_t n, int k, bool auto_k,
                   const double* d_amax, const int32_t* d_scale_exp, bool transpose, const void* dCt)
{
    if (k < (auto_k ? 0 : -126) || k > 126 || (auto_k && (!d_scale_exp || (esc == 1 && !d_amax))))
        return B200VA_ERR_INVALID;
    RC_TRY(check_convert_operands(esa, dA, esc, dC, n));
    const size_t abytes = n * esa, cbytes = n * esc, mbytes = d_amax ? 8 : 0, sbytes = d_scale_exp ? 4 : 0;
    if (reinterpret_cast<uintptr_t>(d_amax) & 7u) return B200VA_ERR_ALIGN;
    if (ranges_meet(d_amax, mbytes, dA, abytes) || ranges_meet(d_amax, mbytes, dC, cbytes)) return B200VA_ERR_OVERLAP;
    if (reinterpret_cast<uintptr_t>(d_scale_exp) & 3u) return B200VA_ERR_ALIGN;
    if (ranges_meet(d_scale_exp, sbytes, dA, abytes) || ranges_meet(d_scale_exp, sbytes, dC, cbytes) ||
        ranges_meet(d_scale_exp, sbytes, d_amax, mbytes))
        return B200VA_ERR_OVERLAP;
    if (!transpose || n == 0) return B200VA_OK;
    if (!dCt) return B200VA_ERR_INVALID;
    if (ranges_meet(dCt, n, dA, abytes) || ranges_meet(dCt, n, dC, cbytes) || ranges_meet(dCt, n, d_amax, mbytes) ||
        ranges_meet(dCt, n, d_scale_exp, sbytes))
        return B200VA_ERR_OVERLAP;
    return B200VA_OK;
}

// Every per-tensor FP8 quantize.  The shape is n = rows cols elements; with `transpose`, C's transpose also goes to
// dCt, A having `cols` columns.  The scale is the host's k; with auto_k, k is the margin, and an amax pass into
// *d_amax comes first, from which the quantize launch chooses the exponent and writes it to *d_scale_exp.
int quantize_fp8(int src_dtype, const void* dA, int fp8, void* dC, size_t rows, size_t cols, void* dCt, bool transpose,
                 int k, bool auto_k, double* d_amax, int32_t* d_scale_exp, void* stream)
{
    if (src_dtype < 0 || src_dtype >= DT_COUNT || fp8 < 0 || fp8 >= F8_COUNT) return B200VA_ERR_VARIANT;
    RC_TRY(current_dev_info(nullptr));
    // rows cols, saturated at 2^40 + 1 when the product overflows, so that the operand checks reject it as n > 2^40
    constexpr size_t past = (size_t{1} << 40) + 1;
    const size_t es = dtype_size(src_dtype), n = cols && rows > past / cols ? past : rows * cols;
    RC_TRY(check_fp8_args(es, dA, 1, dC, n, k, auto_k, d_amax, d_scale_exp, transpose, dCt));
    if (n == 0) return B200VA_OK;
    fp8_quant_fn fn = nullptr;
    with_value<DT_F32, DT_F64, DT_F16, DT_BF16>(src_dtype, [&](auto SRC) { fn = fp8_quant_vec<SRC>; });
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const uintptr_t a = reinterpret_cast<uintptr_t>(dA), c = reinterpret_cast<uintptr_t>(dC);
    fp8_quant_args q;
    q.a = dA;
    q.n = n;
    if (auto_k) {
        q.amax = d_amax;                                                    // the amax pass: no C yet
        RC_TRY(launch_fp8_quant(fn, plan_fp8_amax(a, es, n), 0, q, st));
        q.amax = nullptr;
        q.amax_in = d_amax;
        q.margin = k;
        q.k_out = d_scale_exp;
    } else {
        q.k = k;
        q.amax = d_amax;
    }
    q.c = dC;
    q.fmt = fp8;
    if (!transpose) return launch_fp8_quant(fn, plan_cast(a, es, c, 1, n, 1), 0, q, st);
    q.ct = dCt;
    q.cols = cols;
    size_t smem = 0;
    const cast_plan p = plan_fp8_transpose(a, c, reinterpret_cast<uintptr_t>(dCt), es, rows, cols, smem);
    return launch_fp8_quant(fn, p, smem, q, st);
}

// Every per-tensor FP8 dequantize: one fp8_dequant_vec<T> launch, a unit being a 16-byte output slice (sizeof T per
// group of 16).  The scale is the host's k; with auto_k the kernel reads k from *k_in.
int dequantize_fp8(int fp8, const void* dA, int dst_dtype, void* dC, size_t n, int k, bool auto_k, const int32_t* k_in,
                   void* stream)
{
    if (dst_dtype < 0 || dst_dtype >= DT_COUNT || fp8 < 0 || fp8 >= F8_COUNT) return B200VA_ERR_VARIANT;
    RC_TRY(current_dev_info(nullptr));
    const size_t es = dtype_size(dst_dtype);
    RC_TRY(check_fp8_args(1, dA, es, dC, n, k, auto_k, nullptr, k_in, false, nullptr));
    if (n == 0) return B200VA_OK;
    decltype(&fp8_dequant_vec<DT_F32>) fn = nullptr;
    with_value<DT_F32, DT_F64, DT_F16, DT_BF16>(dst_dtype, [&](auto DST) { fn = fp8_dequant_vec<DST>; });
    const cast_plan p = plan_cast(reinterpret_cast<uintptr_t>(dA), 1, reinterpret_cast<uintptr_t>(dC), es, n, es);
    return launch_kernel(fn, p.grid, p.threads, 0, static_cast<cudaStream_t>(stream), pdl_enabled(), dA, dC, n, p.head,
                         p.ngroups, p.unroll, p.prefetch_first, fp8, k, k_in);
}

// b200va_convert_sr_f32 and b200va_quantize_fp8_sr_f32: one sr_cast_vec launch, a group per unit, dst one of SR_*.
// The key of the random bits is derived from the seed here, once per call.
int launch_sr(const void* dA, int dst, void* dC, size_t n, int k, uint64_t seed, uint64_t first, double* amax,
              cudaStream_t st)
{
    const size_t esc = dst == SR_F16 || dst == SR_BF16 ? 2 : 1;
    const cast_plan p = plan_cast(reinterpret_cast<uintptr_t>(dA), 4, reinterpret_cast<uintptr_t>(dC), esc, n, 1);
    return launch_kernel(sr_cast_vec, p.grid, p.threads, 0, st, pdl_enabled(), dA, dC, n, p.head, p.ngroups, p.unroll,
                         p.prefetch_first, dst, k, splitmix64(seed), first, amax);
}

// b200va_quantize_mxfp8 (QUANT: T -> fmt) and b200va_dequantize_mxfp8 (fmt -> T), T of ES bytes: one mx_quant_vec<ES>
// or mx_dequant_vec<ES> launch, the type, format, block and rule passed to the kernel.  The vector body runs only
// with A and C both on a 16-byte boundary at element 0 (cast_body finds no head), where groups of 16 and blocks
// coincide: the whole blocks when quantizing (a unit is a group; each further block is one edge item), the whole
// groups when dequantizing (a unit is a 16-byte output slice; each further element is one edge item).  Otherwise
// every block, or element, is an edge item.  The geometry is plan_cast's.
template <bool QUANT, int ES>
int launch_mx_typed(const void* dA, void* dS, void* dC, size_t n, int dt, int fmt, int block, int rule, cudaStream_t st)
{
    cast_plan p = cast_body(reinterpret_cast<uintptr_t>(dA), QUANT ? ES : 1, reinterpret_cast<uintptr_t>(dC),
                            QUANT ? 1 : ES, n);
    if (p.head != 0) p = {};      // no vector body: every block, or element, is an edge item
    if constexpr (QUANT) {
        const size_t per_block = block / 16;
        p.ngroups -= p.ngroups % per_block;
        plan_geometry(p, hbm_class(n, ES), p.ngroups, (n + block - 1) / block - p.ngroups / per_block);
        return launch_kernel(mx_quant_vec<ES>, p.grid, p.threads, 0, st, pdl_enabled(), dA, dC, dS, n, p.ngroups, p.unroll,
                             p.prefetch_first, dt, fmt, block, rule, static_cast<void*>(nullptr), static_cast<void*>(nullptr),
                             size_t{0}, size_t{0}, 0);
    } else {
        plan_geometry(p, hbm_class(n, ES), p.ngroups * ES, n - p.ngroups * 16);
        return launch_kernel(mx_dequant_vec<ES>, p.grid, p.threads, 0, st, pdl_enabled(), dA, dS, dC, n, p.ngroups, p.unroll,
                             p.prefetch_first, dt, fmt, block, size_t{0}, size_t{0}, 0);
    }
}

// The argument rules the two MXFP8 entry points share, after the dtype, format and rule codes: block one of 32, 64
// and 128, then A and C as b200va_convert checks them (1-byte FP8 elements), dS non-NULL, and the ceil(n / block)
// scale bytes (any address) meeting neither A nor C.
int check_mx_args(size_t es, const void* dA, size_t esc, const void* dC, const void* dS, size_t n, int block)
{
    if (block != 32 && block != 64 && block != 128) return B200VA_ERR_INVALID;
    if (n && !dS) return B200VA_ERR_INVALID;
    RC_TRY(check_convert_operands(es, dA, esc, dC, n));
    const size_t sbytes = b200va_mxfp8_scale_bytes(n, block);
    if (ranges_meet(dS, sbytes, dA, n * es) || ranges_meet(dS, sbytes, dC, n * esc)) return B200VA_ERR_OVERLAP;
    return B200VA_OK;
}

// rows cols, saturated at 2^40 + 1 when the product overflows, so that the operand checks reject it as n > 2^40.
size_t matrix_elems(size_t rows, size_t cols)
{
    constexpr size_t past = (size_t{1} << 40) + 1;
    return cols && rows > past / cols ? past : rows * cols;
}

// The blockwise quantize's plan, n = rows cols > 0 elements of es bytes, C and / or Ct requested.  The tiled path runs
// when cols % 128 == 0, rows % 16 == 0 and A, C and Ct (those requested) sit on 16-byte boundaries: ngroups = n / 16,
// FP8B_THREADS threads, one CTA per 128 x 128 tile and FP8B_SMEM bytes of dynamic shared memory (smem).  Otherwise the
// per-block path: ngroups = 0, one edge item per block (1 x 128: C's blocks, then Ct's; 128 x 128: one per tile) under
// plan_geometry for A's HBM class.  Neither prefetches a first tile, and neither geometry was tuned.
cast_plan plan_fp8_blockwise(uintptr_t a, uintptr_t c, uintptr_t ct, size_t es, size_t rows, size_t cols, int kind,
                             size_t& smem)
{
    constexpr size_t T = FP8B_TILE;
    const size_t n = rows * cols, nkb_r = (rows + T - 1) / T, nkb_c = (cols + T - 1) / T;
    cast_plan p{};
    smem = 0;
    if (cols % T == 0 && rows % 16 == 0 && ((a | c | ct) & 15u) == 0) {
        p.ngroups = n / 16;
        p.threads = FP8B_THREADS;
        p.unroll = 1;
        p.grid = static_cast<unsigned>(std::min<size_t>(nkb_r * nkb_c, 0x7fffffff));
        smem = FP8B_SMEM;
    } else {
        const size_t items = kind == FP8B_1X128 ? (c ? rows * nkb_c : 0) + (ct ? cols * nkb_r : 0) : nkb_r * nkb_c;
        plan_geometry(p, hbm_class(n, es), 0, items);
        p.prefetch_first = 0;
    }
    return p;
}

// The argument rules of b200va_quantize_fp8_blockwise and b200va_quantize_fp8_rowwise after the dtype, format and
// kind codes, in the order they apply (A of es bytes per element, rows x cols; S and St of sbytes and stbytes; the
// caller has checked that the two pairs are each all-NULL or all-non-NULL).  The row-wise call's workspace dW of
// wbytes needs `need` bytes; the blockwise call has none (need = wbytes = 0).
//   1. with n = rows cols > 0: something requested, dA non-NULL, and n (saturated on overflow) at most 2^40; dW
//      non-NULL and wbytes >= need;
//   2. A aligned to its element size, S, St and dW 4-byte aligned (C and Ct are bytes: any address);
//   3. no two of A, C, S, Ct, St and the needed workspace meeting, the scales' padding included.
int check_fp8_2d_args(size_t es, const void* dA, const void* dC, const float* dS, size_t sbytes, const void* dCt,
                      const float* dSt, size_t stbytes, size_t rows, size_t cols, const void* dW = nullptr,
                      size_t need = 0, size_t wbytes = 0)
{
    const size_t n = matrix_elems(rows, cols);
    if (n && ((!dC && !dCt) || !dA || n > (size_t{1} << 40) || (need && !dW) || wbytes < need)) return B200VA_ERR_INVALID;
    if ((reinterpret_cast<uintptr_t>(dA) & (es - 1)) || (reinterpret_cast<uintptr_t>(dS) & 3u) ||
        (reinterpret_cast<uintptr_t>(dSt) & 3u) || (reinterpret_cast<uintptr_t>(dW) & 3u))
        return B200VA_ERR_ALIGN;
    const void* p[6] = {dA, dC, dS, dCt, dSt, dW};
    const size_t bytes[6] = {n * es, dC ? n : 0, dS ? sbytes : 0, dCt ? n : 0, dSt ? stbytes : 0, need};
    for (int x = 0; x < 6; ++x)
        for (int y = x + 1; y < 6; ++y)
            if (ranges_meet(p[x], bytes[x], p[y], bytes[y])) return B200VA_ERR_OVERLAP;
    return B200VA_OK;
}

// The blockwise and row-wise dequantize: one mx_dequant_vec<ES> launch, kind an FP8B_* code or FP8R_ROWS, S of sbytes
// (the layout's count, 0 when rows cols = 0).  The vector body runs when cols % 16 == 0 and A and C sit on 16-byte
// boundaries; a unit is a 16-byte output slice, every other element an edge item.
int dequantize_fp8_2d(int fp8, const void* dA, const float* dS, size_t sbytes, int kind, int dst_dtype, void* dC,
                      size_t rows, size_t cols, void* stream)
{
    if (dst_dtype < 0 || dst_dtype >= DT_COUNT || fp8 < 0 || fp8 >= F8_COUNT) return B200VA_ERR_VARIANT;
    RC_TRY(current_dev_info(nullptr));
    const size_t es = dtype_size(dst_dtype), n = matrix_elems(rows, cols);
    if (n && (!dA || !dS || !dC || n > (size_t{1} << 40))) return B200VA_ERR_INVALID;
    const uintptr_t a = reinterpret_cast<uintptr_t>(dA), c = reinterpret_cast<uintptr_t>(dC);
    if ((c & (es - 1)) || (reinterpret_cast<uintptr_t>(dS) & 3u)) return B200VA_ERR_ALIGN;
    if (ranges_meet(dC, n * es, dA, n) || ranges_meet(dC, n * es, dS, sbytes)) return B200VA_ERR_OVERLAP;
    if (n == 0) return B200VA_OK;
    cast_plan p{};
    if (cols % 16 == 0 && ((a | c) & 15u) == 0) p.ngroups = n / 16;
    plan_geometry(p, hbm_class(n, es), p.ngroups * es, n - p.ngroups * 16);
    int rc = B200VA_ERR_VARIANT;
    with_value<4, 8, 2>(static_cast<int>(es), [&](auto ES) {
        rc = launch_kernel(mx_dequant_vec<ES>, p.grid, p.threads, 0, static_cast<cudaStream_t>(stream), pdl_enabled(), dA,
                           static_cast<const void*>(dS), dC, n, p.ngroups, p.unroll, p.prefetch_first, dst_dtype, fp8, 0,
                           rows, cols, kind);
    });
    return rc;
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
    return quantize_fp8(src_dtype, dA, fp8, dC, n, 1, nullptr, false, scale_exp, false, d_amax, nullptr, stream);
}

int b200va_dequantize_fp8(int fp8, const void* dA, int dst_dtype, void* dC, size_t n, int scale_exp, void* stream)
{
    return dequantize_fp8(fp8, dA, dst_dtype, dC, n, scale_exp, false, nullptr, stream);
}

int b200va_quantize_fp8_auto(int src_dtype, const void* dA, int fp8, void* dC, size_t n, int margin, double* d_amax,
                             int32_t* d_scale_exp, void* stream)
{
    return quantize_fp8(src_dtype, dA, fp8, dC, n, 1, nullptr, false, margin, true, d_amax, d_scale_exp, stream);
}

int b200va_dequantize_fp8_auto(int fp8, const void* dA, int dst_dtype, void* dC, size_t n, const int32_t* d_scale_exp,
                               void* stream)
{
    return dequantize_fp8(fp8, dA, dst_dtype, dC, n, 0, true, d_scale_exp, stream);
}

int b200va_quantize_fp8_transpose(int src_dtype, const void* dA, int fp8, void* dC, void* dCt, size_t rows, size_t cols,
                                  int scale_exp, double* d_amax, void* stream)
{
    return quantize_fp8(src_dtype, dA, fp8, dC, rows, cols, dCt, true, scale_exp, false, d_amax, nullptr, stream);
}

int b200va_quantize_fp8_transpose_auto(int src_dtype, const void* dA, int fp8, void* dC, void* dCt, size_t rows,
                                       size_t cols, int margin, double* d_amax, int32_t* d_scale_exp, void* stream)
{
    return quantize_fp8(src_dtype, dA, fp8, dC, rows, cols, dCt, true, margin, true, d_amax, d_scale_exp, stream);
}

int b200va_convert_sr_f32(const float* dA, int dst_dtype, void* dC, size_t n, uint64_t seed, uint64_t first,
                          void* stream)
{
    if (dst_dtype != DT_F16 && dst_dtype != DT_BF16) return B200VA_ERR_VARIANT;
    RC_TRY(current_dev_info(nullptr));
    RC_TRY(check_convert_operands(4, dA, 2, dC, n));
    if (n == 0) return B200VA_OK;
    return launch_sr(dA, dst_dtype == DT_F16 ? SR_F16 : SR_BF16, dC, n, 0, seed, first, nullptr,
                     static_cast<cudaStream_t>(stream));
}

int b200va_quantize_fp8_sr_f32(const float* dA, int fp8, void* dC, size_t n, int scale_exp, uint64_t seed, uint64_t first,
                               double* d_amax, void* stream)
{
    if (fp8 < 0 || fp8 >= F8_COUNT) return B200VA_ERR_VARIANT;
    RC_TRY(current_dev_info(nullptr));
    RC_TRY(check_fp8_args(4, dA, 1, dC, n, scale_exp, false, d_amax, nullptr, false, nullptr));
    if (n == 0) return B200VA_OK;
    return launch_sr(dA, fp8 == F8_E4M3 ? SR_E4M3 : SR_E5M2, dC, n, scale_exp, seed, first, d_amax,
                     static_cast<cudaStream_t>(stream));
}

size_t b200va_mxfp8_scale_bytes(size_t n, int block)
{
    return block == 32 || block == 64 || block == 128 ? n / block + (n % block != 0) : 0;
}

int b200va_quantize_mxfp8(int src_dtype, const void* dA, int fp8, void* dC, void* dS, size_t n, int block, int scale_rule,
                          void* stream)
{
    if (src_dtype < 0 || src_dtype >= DT_COUNT || fp8 < 0 || fp8 >= F8_COUNT || scale_rule < 0 || scale_rule >= MX_SCALE_COUNT)
        return B200VA_ERR_VARIANT;
    RC_TRY(current_dev_info(nullptr));
    RC_TRY(check_mx_args(dtype_size(src_dtype), dA, 1, dC, dS, n, block));
    if (n == 0) return B200VA_OK;
    int rc = B200VA_ERR_VARIANT;
    with_value<4, 8, 2>(static_cast<int>(dtype_size(src_dtype)), [&](auto ES) {
        rc = launch_mx_typed<true, ES>(dA, dS, dC, n, src_dtype, fp8, block, scale_rule, static_cast<cudaStream_t>(stream));
    });
    return rc;
}

int b200va_dequantize_mxfp8(int fp8, const void* dA, const void* dS, int dst_dtype, void* dC, size_t n, int block,
                            void* stream)
{
    if (dst_dtype < 0 || dst_dtype >= DT_COUNT || fp8 < 0 || fp8 >= F8_COUNT) return B200VA_ERR_VARIANT;
    RC_TRY(current_dev_info(nullptr));
    RC_TRY(check_mx_args(1, dA, dtype_size(dst_dtype), dC, dS, n, block));
    if (n == 0) return B200VA_OK;
    int rc = B200VA_ERR_VARIANT;
    with_value<4, 8, 2>(static_cast<int>(dtype_size(dst_dtype)), [&](auto ES) {
        rc = launch_mx_typed<false, ES>(dA, const_cast<void*>(dS), dC, n, dst_dtype, fp8, block, 0, static_cast<cudaStream_t>(stream));
    });
    return rc;
}

size_t b200va_fp8_blockwise_scales(size_t rows, size_t cols, int block_kind)
{
    constexpr size_t T = FP8B_TILE;
    if (!rows || !cols || block_kind < 0 || block_kind >= FP8B_COUNT) return 0;
    const size_t nkb_c = (cols + T - 1) / T;
    return block_kind == FP8B_1X128 ? rows * nkb_c : (rows + T - 1) / T * ((nkb_c + 3) / 4 * 4);
}

int b200va_quantize_fp8_blockwise(int src_dtype, const void* dA, int fp8, int block_kind, size_t rows, size_t cols,
                                  void* dC, float* dS, void* dCt, float* dSt, void* stream)
{
    if (src_dtype < 0 || src_dtype >= DT_COUNT || fp8 < 0 || fp8 >= F8_COUNT || block_kind < 0 || block_kind >= FP8B_COUNT)
        return B200VA_ERR_VARIANT;
    RC_TRY(current_dev_info(nullptr));
    if (!dC != !dS || !dCt != !dSt) return B200VA_ERR_INVALID;
    const size_t es = dtype_size(src_dtype);
    RC_TRY(check_fp8_2d_args(es, dA, dC, dS, 4 * b200va_fp8_blockwise_scales(rows, cols, block_kind), dCt, dSt,
                             4 * b200va_fp8_blockwise_scales(cols, rows, block_kind), rows, cols));
    if (rows == 0 || cols == 0) return B200VA_OK;
    size_t smem = 0;
    const cast_plan p = plan_fp8_blockwise(reinterpret_cast<uintptr_t>(dA), reinterpret_cast<uintptr_t>(dC),
                                           reinterpret_cast<uintptr_t>(dCt), es, rows, cols, block_kind, smem);
    int rc = B200VA_ERR_VARIANT;
    with_value<4, 8, 2>(static_cast<int>(es), [&](auto ES) {
        rc = launch_kernel(mx_quant_vec<ES>, p.grid, p.threads, smem, static_cast<cudaStream_t>(stream), pdl_enabled(), dA,
                           dC, static_cast<void*>(dS), rows * cols, p.ngroups, p.unroll, p.prefetch_first, src_dtype, fp8, 0,
                           0, dCt, static_cast<void*>(dSt), rows, cols, block_kind);
    });
    return rc;
}

int b200va_dequantize_fp8_blockwise(int fp8, const void* dA, const float* dS, int block_kind, int dst_dtype, void* dC,
                                    size_t rows, size_t cols, void* stream)
{
    if (block_kind < 0 || block_kind >= FP8B_COUNT) return B200VA_ERR_VARIANT;
    return dequantize_fp8_2d(fp8, dA, dS, 4 * b200va_fp8_blockwise_scales(rows, cols, block_kind), block_kind, dst_dtype,
                             dC, rows, cols, stream);
}

size_t b200va_fp8_rowwise_workspace(size_t rows, size_t cols)
{
    return 4 * (b200va_fp8_blockwise_scales(rows, cols, FP8B_1X128) + b200va_fp8_blockwise_scales(cols, rows, FP8B_1X128));
}

// Three mx_quant_vec<ES> launches chained by PDL, each waiting for the one before: FP8R_MAXIMA (the 1 x 128 block
// scales into the workspace, under the 1 x 128 blockwise cast's plan), FP8R_REDUCE (one thread per row and column) and
// FP8R_ROWS (the tiled plan's tiles, or one edge item per element).
int b200va_quantize_fp8_rowwise(int src_dtype, const void* dA, int fp8, size_t rows, size_t cols, void* dC, float* dS,
                                void* dCt, float* dSt, void* d_work, size_t work_bytes, void* stream)
{
    if (src_dtype < 0 || src_dtype >= DT_COUNT || fp8 < 0 || fp8 >= F8_COUNT) return B200VA_ERR_VARIANT;
    RC_TRY(current_dev_info(nullptr));
    if (!dC != !dS || !dCt != !dSt) return B200VA_ERR_INVALID;
    const size_t es = dtype_size(src_dtype), n = matrix_elems(rows, cols);
    const size_t need = n <= (size_t{1} << 40) ? b200va_fp8_rowwise_workspace(rows, cols) : 0;
    RC_TRY(check_fp8_2d_args(es, dA, dC, dS, n ? 4 * rows : 0, dCt, dSt, n ? 4 * cols : 0, rows, cols, d_work, need,
                             work_bytes));
    if (n == 0) return B200VA_OK;
    const uintptr_t a = reinterpret_cast<uintptr_t>(dA), c = reinterpret_cast<uintptr_t>(dC),
                    ct = reinterpret_cast<uintptr_t>(dCt);
    size_t smem = 0;
    const cast_plan pm = plan_fp8_blockwise(a, c, ct, es, rows, cols, FP8B_1X128, smem);
    cast_plan pr{}, pq = pm;
    plan_geometry(pr, false, 0, (dC ? rows : 0) + (dCt ? cols : 0));
    if (!pq.ngroups) plan_geometry(pq, hbm_class(n, es), 0, n);
    float* w = static_cast<float*>(d_work);
    float* wt = w + b200va_fp8_blockwise_scales(rows, cols, FP8B_1X128);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc = B200VA_ERR_VARIANT;
    with_value<4, 8, 2>(static_cast<int>(es), [&](auto ES) {
        auto launch = [&](const cast_plan& p, size_t sm, const void* A, void* C, void* S, void* Ct, void* St, int kind) {
            return launch_kernel(mx_quant_vec<ES>, p.grid, p.threads, sm, st, pdl_enabled(), A, C, S, n, p.ngroups, p.unroll,
                                 0, src_dtype, fp8, 0, 0, Ct, St, rows, cols, kind);
        };
        rc = launch(pm, smem, dA, dC, dC ? w : nullptr, dCt, dCt ? wt : nullptr, FP8R_MAXIMA);
        if (rc == B200VA_OK) rc = launch(pr, 0, w, dS, nullptr, dSt, nullptr, FP8R_REDUCE);
        if (rc == B200VA_OK) rc = launch(pq, pq.ngroups ? smem : 0, dA, dC, dS, dCt, dSt, FP8R_ROWS);
    });
    return rc;
}

int b200va_dequantize_fp8_rowwise(int fp8, const void* dA, const float* dS, int dst_dtype, void* dC, size_t rows,
                                  size_t cols, void* stream)
{
    return dequantize_fp8_2d(fp8, dA, dS, rows && cols ? 4 * rows : 0, FP8R_ROWS, dst_dtype, dC, rows, cols, stream);
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
    const size_t bytes = n * es;
    if (ranges_meet(d_out, 8, dA, bytes) || ranges_meet(d_out, 8, dB, bytes) || ranges_meet(d_out, 8, d_workspace, need) ||
        ranges_meet(d_workspace, need, dA, bytes) || ranges_meet(d_workspace, need, dB, bytes))
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
