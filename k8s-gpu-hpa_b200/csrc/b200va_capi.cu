// b200va_capi.cu -- the C ABI of libb200va.so (declared in include/b200va.h): the shared core.
//
// The library's host side is split by concern: this unit holds the device-info cache and the
// entry points that launch nothing; b200va_add.cu the f32 add (dispatch, alignment peeling,
// geometry, the in-process launch loop, the a2/a6 support kernels, the ceiling probes);
// b200va_typed.cu the STREAM ops and the dot product; b200va_stager.cu the host-buffer staging
// pipeline.  Each entry point names the step of the reference's `./vectorAdd` process it replaces
// (cuda-test-deployment.yaml:18-19; SURVEY.md section 8(a)).
//
// There is deliberately NO CPU fallback: without a CUDA device every compute entry
// point returns an error code.
#include "b200va_internal.h"

using namespace b200va;

struct DevCache {
    std::once_flag once;
    int rc = B200VA_ERR_NO_DEVICE;
    b200va_devinfo_t info{};
};
static DevCache g_dev[kMaxDevices];

int b200va::dev_info(int device, const b200va_devinfo_t** out)
{
    if (device < 0 || device >= kMaxDevices) return B200VA_ERR_INVALID;
    DevCache& dc = g_dev[device];
    std::call_once(dc.once, [&] {
        // individual attributes, not cudaGetDeviceProperties: the latter queries everything
        // and costs tens of milliseconds of every short-lived ./vectorAdd process
        int major = 0, minor = 0, sms = 0, smem = 0, l2 = 0;
        cudaError_t e = cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device);
        if (e == cudaSuccess) e = cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device);
        if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
        if (e == cudaSuccess) e = cudaDeviceGetAttribute(&smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
        if (e == cudaSuccess) e = cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, device);
        if (e != cudaSuccess) { dc.rc = cuda_err(e); return; }
        dc.info.device = device;
        dc.info.cc_major = major;
        dc.info.cc_minor = minor;
        dc.info.sm_count = sms;
        dc.info.max_smem_optin = smem;
        dc.info.l2_bytes = l2;
        // the cubin is sm_90a SASS (+ compute_90a PTX): architecture-specific, it runs on CC 9.0 only
        dc.rc = (major == 9 && minor == 0) ? B200VA_OK : B200VA_ERR_NO_DEVICE;
    });
    if (out) *out = &dc.info;
    return dc.rc;
}

bool b200va::pdl_enabled()
{
    static const bool on = [] {
        const char* e = std::getenv("B200VA_NO_PDL");
        return !(e && e[0] == '1');
    }();
    return on;
}

// ========================================= ABI (C linkage from the declarations in include/b200va.h)
int b200va_abi_version(void) { return B200VA_ABI_VERSION; }

const char* b200va_strerror(int code)
{
    switch (code) {
        case B200VA_OK:            return "success";
        case B200VA_ERR_INVALID:   return "invalid argument";
        case B200VA_ERR_ALIGN:     return "pointer not 4-byte aligned";
        case B200VA_ERR_OVERLAP:   return "output partially overlaps an input";
        case B200VA_ERR_VARIANT:   return "unknown kernel variant or unsupported geometry";
        case B200VA_ERR_NO_DEVICE: return "no sm_90 CUDA device";
        case B200VA_ERR_VERIFY:    return "result verification failed";
        case B200VA_ERR_NOMEM:     return "host allocation failed, or no captured-launch counter left";
    }
    if (code <= B200VA_ERR_CUDA_BASE) return cudaGetErrorString(static_cast<cudaError_t>(-code - 1000));
    return "unknown error";
}

int b200va_query(int device, b200va_devinfo_t* out)
{
    if (!out) return B200VA_ERR_INVALID;
    const b200va_devinfo_t* di = nullptr;
    const int rc = dev_info(device, &di);
    if (!di || di->sm_count <= 0) return rc;
    *out = *di;
    cudaDeviceProp p;                       // name and memory size: only this (cold) call pays for them
    if (cudaGetDeviceProperties(&p, device) == cudaSuccess) {
        out->global_mem_bytes = p.totalGlobalMem;
        std::snprintf(out->name, sizeof out->name, "%s", p.name);
    }
    return rc;
}

// ------------------------------------------------------------------ shard arithmetic
int b200va_shard_range(size_t n, int world, int rank, size_t* begin, size_t* end)
{
    if (world < 1 || rank < 0 || rank >= world || !begin || !end) return B200VA_ERR_INVALID;
    size_t chunk = (n + static_cast<size_t>(world) - 1) / static_cast<size_t>(world);
    chunk = (chunk + 7) & ~size_t{7};  // shard starts stay 32-byte aligned (256-bit body)
    size_t b = static_cast<size_t>(rank) * chunk;
    if (b > n) b = n;
    size_t e = b + chunk;
    if (e > n) e = n;
    *begin = b;
    *end = e;
    return B200VA_OK;
}
