// b200va_typed.cu -- the STREAM ops (copy, scale, add, triad) and the reproducible dot product over
// f32, f64, f16 and bf16.  The only unit that includes the STREAM and dot kernels (b200va_dot.cuh,
// which includes b200va_stream.cuh).
#include "b200va_internal.h"
#include "b200va_dot.cuh"

using namespace b200va;

namespace {

// Bytes per element of a dtype.
size_t dtype_size(int dtype) { return dtype == DT_F64 ? 8 : dtype == DT_F32 ? 4 : 2; }

// Elements of `es` bytes before the first 16-byte boundary at or after address `a`: the scalar head
// a vector body peels off.
size_t head_peel(uintptr_t a, size_t es) { return ((16u - (a & 15u)) & 15u) / es; }

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
    int unroll = 1;
    bool skip_l1_stores = false;
    if (hbm) {
        // three-array ops like the add: 512 x 1; two-array ops (copy, scale) want twice the bytes in
        // flight per thread: 1024 x 2
        threads = binary ? 512 : 1024;
        unroll = binary ? 1 : 2;
        skip_l1_stores = true;
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
        skip_l1_stores = ov.na != 0;
    }
#endif
    const size_t tile_vecs = static_cast<size_t>(threads) * unroll;
    const size_t ntiles = (nvec + tile_vecs - 1) / tile_vecs;
    const size_t grid = std::max<size_t>(std::min<size_t>(ntiles, 0x7fffffff), 1);
    using fn_t = void (*)(const void*, const void*, void*, size_t, size_t, size_t, size_t, S, int);
    const int prefetch_first = hbm ? 1 : 0;
    fn_t fn = nullptr;
#ifdef B200VA_TUNE_MATRIX
    if (unroll == 4) fn = skip_l1_stores ? stream_vec<DT, OP, 4, LD_PLAIN, ST_NA> : stream_vec<DT, OP, 4, LD_PLAIN, ST_PLAIN>;
    else if (skip_l1_stores) fn = unroll == 2 ? stream_vec<DT, OP, 2, LD_PLAIN, ST_NA> : stream_vec<DT, OP, 1, LD_PLAIN, ST_NA>;
#else
    // the production library carries only the ST_NA form the HBM class above picks
    if (skip_l1_stores) {
        if constexpr (binary) fn = stream_vec<DT, OP, 1, LD_PLAIN, ST_NA>;
        else fn = stream_vec<DT, OP, 2, LD_PLAIN, ST_NA>;
    }
#endif
    if (!fn) fn = unroll == 2 ? stream_vec<DT, OP, 2, LD_PLAIN, ST_PLAIN> : stream_vec<DT, OP, 1, LD_PLAIN, ST_PLAIN>;
    return launch_kernel(fn, static_cast<unsigned>(grid), threads, 0, st, pdl_enabled(), dA, dB, dC, n, head, nvec, ntiles, s, prefetch_first);
}

template <int DT>
int launch_stream_op(int op, const void* dA, const void* dB, void* dC, size_t n, double scalar, cudaStream_t st)
{
    switch (op) {
        case OP_COPY:  return launch_stream_typed<DT, OP_COPY>(dA, dB, dC, n, scalar, st);
        case OP_SCALE: return launch_stream_typed<DT, OP_SCALE>(dA, dB, dC, n, scalar, st);
        case OP_ADD:   return launch_stream_typed<DT, OP_ADD>(dA, dB, dC, n, scalar, st);
        case OP_TRIAD: return launch_stream_typed<DT, OP_TRIAD>(dA, dB, dC, n, scalar, st);
    }
    return B200VA_ERR_VARIANT;
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

}  // namespace

// ========================================= ABI (C linkage from the declarations in include/b200va.h)
// ------------------------------------------------------------------ f4: STREAM-style ops
int b200va_stream(int op, int dtype, const void* dA, const void* dB, void* dC, size_t n, double scalar, void* stream)
{
    if (op < 0 || op >= OP_COUNT || dtype < 0 || dtype >= DT_COUNT) return B200VA_ERR_VARIANT;
    RC_TRY(current_dev_info(nullptr));
    RC_TRY(check_operands(dtype_size(dtype), dA, dB, dC, n, op == OP_ADD || op == OP_TRIAD));
    if (n == 0) return B200VA_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    switch (dtype) {
        case DT_F32:  return launch_stream_op<DT_F32>(op, dA, dB, dC, n, scalar, st);
        case DT_F64:  return launch_stream_op<DT_F64>(op, dA, dB, dC, n, scalar, st);
        case DT_F16:  return launch_stream_op<DT_F16>(op, dA, dB, dC, n, scalar, st);
        case DT_BF16: return launch_stream_op<DT_BF16>(op, dA, dB, dC, n, scalar, st);
    }
    return B200VA_ERR_VARIANT;
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
    if (n) {
        switch (dtype) {
            case DT_F32:  RC_TRY(launch_dot_typed<DT_F32>(dA, dB, n, ws, st)); break;
            case DT_F64:  RC_TRY(launch_dot_typed<DT_F64>(dA, dB, n, ws, st)); break;
            case DT_F16:  RC_TRY(launch_dot_typed<DT_F16>(dA, dB, n, ws, st)); break;
            case DT_BF16: RC_TRY(launch_dot_typed<DT_BF16>(dA, dB, n, ws, st)); break;
        }
    }
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
