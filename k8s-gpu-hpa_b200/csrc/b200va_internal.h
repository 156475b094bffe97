// b200va_internal.h -- what the translation units of libb200va.so share: error plumbing, the
// device-info cache, the launch helper, the argument and size-class rules, and the f32 add entry
// points the host-buffer stager calls, plus the standard headers most units use.  No kernel header.
//
// Everything here has external linkage but hidden visibility: it never enters the libraries'
// dynamic symbol tables, which carry the C ABI of include/b200va.h.  The units define the ABI's
// entry points after including this header, so they take C linkage from those declarations.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <type_traits>

#include "../../include/b200va.h"

// This body of the project namespace is hidden; the kernel headers reopen it with default visibility.
namespace b200va __attribute__((visibility("hidden"))) {

constexpr int kMaxDevices = 64;

inline int cuda_err(cudaError_t e) { return e == cudaSuccess ? B200VA_OK : -(1000 + static_cast<int>(e)); }

#define CU_TRY(expr)                                   \
    do {                                               \
        cudaError_t e__ = (expr);                      \
        if (e__ != cudaSuccess) return cuda_err(e__);  \
    } while (0)

#define RC_TRY(expr)                   \
    do {                               \
        int rc__ = (expr);             \
        if (rc__ != B200VA_OK) return rc__; \
    } while (0)

// ---- b200va_capi.cu
// The cached attributes of `device`; B200VA_ERR_NO_DEVICE unless it is a CC 9.0 part.
int dev_info(int device, const b200va_devinfo_t** out);

inline int current_dev_info(const b200va_devinfo_t** out)
{
    int device = -1;
    CU_TRY(cudaGetDevice(&device));
    return dev_info(device, out);
}

// Programmatic stream serialization lets launch k+1 ramp up behind launch k's tail.  The kernels call
// griddepcontrol.wait before their first global access, except the early-load forms (vadd_vec and
// vadd_vec_dyn with EARLY = 1), which load their first tile before it; each kernel releases its successor
// only after its own wait (b200va_ptx.cuh: pdl_wait), so launch k is the only launch that can still be
// running beside launch k+1.  Every hot-path launch uses it unless B200VA_NO_PDL=1.
bool pdl_enabled();

// Restores the calling thread's current device on every exit path of the entry points that
// take a `device` argument (include/b200va.h: "restore the caller's current device").
struct DeviceGuard {
    int prev = -1;
    cudaError_t err = cudaSuccess;
    explicit DeviceGuard(int device)
    {
        if (cudaGetDevice(&prev) != cudaSuccess) { prev = -1; cudaGetLastError(); }
        if (prev != device) err = cudaSetDevice(device);
    }
    ~DeviceGuard()
    {
        int now = -1;
        if (prev >= 0 && cudaGetDevice(&now) == cudaSuccess && now != prev) cudaSetDevice(prev);
    }
    DeviceGuard(const DeviceGuard&) = delete;
    DeviceGuard& operator=(const DeviceGuard&) = delete;
};

template <class... KArgs, class... Args>
int launch_kernel(void (*fn)(KArgs...), unsigned grid, unsigned block, size_t smem, cudaStream_t stream, bool pdl, Args... args)
{
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(block);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, fn, static_cast<KArgs>(args)...);
    if (e != cudaSuccess) cudaGetLastError();   // a refused launch must not stay latched for the next caller
    return cuda_err(e);
}

// Calls f(std::integral_constant<int, V>{}) for the V in Vs that equals v, and nothing if none does: turns a
// runtime field into a template argument.  Nested calls pick a kernel from a tune.
template <int... Vs, class F>
void with_value(int v, F&& f)
{
    (void)((v == Vs && (f(std::integral_constant<int, Vs>{}), true)) || ...);
}

// ---- the rules the f32 add and the STREAM ops share
// The HBM size class: at least 2^25 four-byte words (128 MiB) per operand of `es`-byte elements,
// never L2-resident.  Written as a bound on n so that no n overflows.
constexpr bool hbm_class(size_t n, size_t es) { return n >= (size_t{1} << 25) * 4 / es; }

// C = f(A[, B]) over n elements of `es` bytes: the operands are element-aligned, n is at most 2^40
// and C either is an input or does not meet it.  `has_b`: B is an operand (otherwise it is ignored).
inline int check_operands(size_t es, const void* pa, const void* pb, const void* pc, size_t n, bool has_b)
{
    if (n == 0) return B200VA_OK;
    if (!pa || !pc || (has_b && !pb)) return B200VA_ERR_INVALID;
    const uintptr_t a = reinterpret_cast<uintptr_t>(pa), b = has_b ? reinterpret_cast<uintptr_t>(pb) : 0,
                    c = reinterpret_cast<uintptr_t>(pc);
    if ((a | b | c) & (es - 1)) return B200VA_ERR_ALIGN;
    if (n > (size_t{1} << 40)) return B200VA_ERR_INVALID;
    const uintptr_t bytes = n * es;
    auto partial = [&](uintptr_t x) { return x != c && x < c + bytes && c < x + bytes; };
    if (partial(a) || (has_b && partial(b))) return B200VA_ERR_OVERLAP;
    return B200VA_OK;
}

// C = convert(A), A of `esa`-byte and C of `esc`-byte elements: the rules of check_operands, except that
// operands of different element sizes must not meet at all.  With exact aliasing the wide side's stores
// would overwrite elements of the narrow side that other threads have not read yet.
inline int check_convert_operands(size_t esa, const void* pa, size_t esc, const void* pc, size_t n)
{
    if (esa == esc) return check_operands(esa, pa, nullptr, pc, n, false);
    if (n == 0) return B200VA_OK;
    if (!pa || !pc) return B200VA_ERR_INVALID;
    const uintptr_t a = reinterpret_cast<uintptr_t>(pa), c = reinterpret_cast<uintptr_t>(pc);
    if ((a & (esa - 1)) || (c & (esc - 1))) return B200VA_ERR_ALIGN;
    if (n > (size_t{1} << 40)) return B200VA_ERR_INVALID;
    if (a < c + n * esc && c < a + n * esa) return B200VA_ERR_OVERLAP;
    return B200VA_OK;
}

// ---- b200va_add.cu: the f32 add, as the host-buffer stager calls it
void default_tune(int variant, size_t n, b200va_tune_t* t, unsigned flags = 0);
int check_variant(int variant, unsigned flags = 0);
// `ctr`: the dynamic tile scheduler's two-word ticket counter (zeroed; the kernel leaves it zeroed
// again); nullptr takes the next slot of the device's ring.
int launch(const float* dA, const float* dB, float* dC, size_t n, const b200va_tune_t& t, cudaStream_t stream, bool pdl,
           unsigned int* ctr = nullptr);

}  // namespace b200va
