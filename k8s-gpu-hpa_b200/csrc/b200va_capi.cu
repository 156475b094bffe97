// b200va_capi.cu -- the C ABI of libb200va.so (declared in include/b200va.h).
//
// Host-side dispatch for the sm_90a vectorAdd kernels: argument checking, alignment
// peeling, geometry resolution, the in-process launch loop, the host-buffer staging
// pipeline.  Each entry point names the step of the reference's `./vectorAdd` process
// it replaces (cuda-test-deployment.yaml:18-19; SURVEY.md section 8(a)).
//
// There is deliberately NO CPU fallback: without a CUDA device every compute entry
// point returns an error code.
#include <cuda_runtime.h>

#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <atomic>
#include <cctype>
#include <condition_variable>
#include <functional>
#include <map>
#include <thread>
#include <utility>
#include <vector>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>

#include "../../include/b200va.h"
#include "b200va_kernels.cuh"
#include "b200va_stream.cuh"
#include "b200va_dot.cuh"

using namespace b200va;

namespace {

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

struct DevCache {
    std::once_flag once;
    int rc = B200VA_ERR_NO_DEVICE;
    b200va_devinfo_t info{};
};
DevCache g_dev[kMaxDevices];

int dev_info(int device, const b200va_devinfo_t** out)
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

int current_dev_info(const b200va_devinfo_t** out)
{
    int device = -1;
    CU_TRY(cudaGetDevice(&device));
    return dev_info(device, out);
}

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

// ----------------------------------------------------------------------- vec dispatch
// libb200va.so carries the production set only (what AUTO and the named variants resolve to,
// plus close neighbours used by the parity tests); -DB200VA_TUNE_MATRIX (libb200va_tune.so, the
// A/B tool's library) instantiates every combination of b200va_tune_t.  A combination that is
// not compiled in makes the pick functions return nullptr -> B200VA_ERR_VARIANT.
using vec_fn = void (*)(const float*, const float*, float*, size_t, size_t, size_t, size_t);
using dyn_fn = void (*)(const float*, const float*, float*, size_t, size_t, size_t, size_t, unsigned int*);

// The vec kernel a tune selects: `plain` under the hardware block scheduler, `dyn` under the
// dynamic tile scheduler (scheduler = 1); at most one is set.
struct VecFn {
    vec_fn plain = nullptr;
    dyn_fn dyn = nullptr;
    const void* key() const { return plain ? reinterpret_cast<const void*>(plain) : reinterpret_cast<const void*>(dyn); }
};

template <int VW, int UNROLL, int LD, int ST>
VecFn pick_early_hw(int early)
{
    VecFn f;
    switch (early) {
        case 0: f.plain = vadd_vec<VW, UNROLL, LD, ST, 0>; break;
        case 1: f.plain = vadd_vec<VW, UNROLL, LD, ST, 1>; break;
        case 2: f.plain = vadd_vec<VW, UNROLL, LD, ST, 2>; break;
    }
    return f;
}

template <int VW, int UNROLL, int LD, int ST>
VecFn pick_early_dyn(int early)
{
    VecFn f;
    switch (early) {
        case 0: f.dyn = vadd_vec_dyn<VW, UNROLL, LD, ST, 0>; break;
        case 1: f.dyn = vadd_vec_dyn<VW, UNROLL, LD, ST, 1>; break;
        case 2: f.dyn = vadd_vec_dyn<VW, UNROLL, LD, ST, 2>; break;
    }
    return f;
}

template <int VW, int UNROLL, int LD, int ST>
VecFn pick_sched(int early, int sched)
{
    if (sched == 1) {
#ifdef B200VA_TUNE_MATRIX
        return pick_early_dyn<VW, UNROLL, LD, ST>(early);
#else
        if constexpr (VW == 4 && LD == LD_PLAIN && ST == ST_NA && (UNROLL == 2 || UNROLL == 4))
            return pick_early_dyn<VW, UNROLL, LD, ST>(early);
        else
            return VecFn{};
#endif
    }
    return pick_early_hw<VW, UNROLL, LD, ST>(early);
}

template <int VW, int UNROLL, int LD>
VecFn pick_st(int st, int early, int sched)
{
    switch (st) {
        case ST_PLAIN: return pick_sched<VW, UNROLL, LD, ST_PLAIN>(early, sched);
        case ST_NA:    return pick_sched<VW, UNROLL, LD, ST_NA>(early, sched);
#ifdef B200VA_TUNE_MATRIX
        case ST_CS:    return pick_sched<VW, UNROLL, LD, ST_CS>(early, sched);
        case ST_NA_EF: return pick_sched<VW, UNROLL, LD, ST_NA_EF>(early, sched);
#endif
    }
    return VecFn{};
}

template <int VW, int UNROLL>
VecFn pick_ld(int ld, int st, int early, int sched)
{
    switch (ld) {
        case LD_PLAIN: return pick_st<VW, UNROLL, LD_PLAIN>(st, early, sched);
        case LD_NA_EF: return pick_st<VW, UNROLL, LD_NA_EF>(st, early, sched);
#ifdef B200VA_TUNE_MATRIX
        case LD_NA:    return pick_st<VW, UNROLL, LD_NA>(st, early, sched);
        case LD_NC_NA: return pick_st<VW, UNROLL, LD_NC_NA>(st, early, sched);
        case LD_CS:    return pick_st<VW, UNROLL, LD_CS>(st, early, sched);
        case LD_NA_256: return pick_st<VW, UNROLL, LD_NA_256>(st, early, sched);
#endif
    }
    return VecFn{};
}

template <int VW>
VecFn pick_unroll(int unroll, int ld, int st, int early, int sched)
{
    switch (unroll) {
        case 1: return pick_ld<VW, 1>(ld, st, early, sched);
        case 2: return pick_ld<VW, 2>(ld, st, early, sched);
        case 4: return pick_ld<VW, 4>(ld, st, early, sched);
#ifdef B200VA_TUNE_MATRIX
        case 8: return pick_ld<VW, 8>(ld, st, early, sched);
#endif
    }
    return VecFn{};
}

VecFn pick_vec(int vw, int unroll, int ld, int st, int early, int sched)
{
    return vw == 8 ? pick_unroll<8>(unroll, ld, st, early, sched) : pick_unroll<4>(unroll, ld, st, early, sched);
}

// ----------------------------------------------------------------------- tma dispatch
using tma_fn = void (*)(const float*, const float*, float*, size_t, size_t, size_t, uint32_t, uint32_t);
using tma_dyn_fn = void (*)(const float*, const float*, float*, size_t, size_t, size_t, uint32_t, uint32_t, unsigned int*);

#ifdef B200VA_TUNE_MATRIX
template <int MODE, bool HINT>
tma_fn pick_tma_st(int st)
{
    switch (st) {
        case ST_PLAIN: return vadd_tma<MODE, HINT, ST_PLAIN>;
        case ST_NA:    return vadd_tma<MODE, HINT, ST_NA>;
        case ST_CS:    return vadd_tma<MODE, HINT, ST_CS>;
        case ST_NA_EF: return vadd_tma<MODE, HINT, ST_NA_EF>;
    }
    return nullptr;
}
#endif

// store_mode 2: the dynamic tile scheduler, register stores
template <bool HINT>
tma_dyn_fn pick_tma_dyn_st(int st)
{
    switch (st) {
        case ST_PLAIN: return vadd_tma_dyn<HINT, ST_PLAIN>;
        case ST_NA:    return vadd_tma_dyn<HINT, ST_NA>;
#ifdef B200VA_TUNE_MATRIX
        case ST_CS:    return vadd_tma_dyn<HINT, ST_CS>;
        case ST_NA_EF: return vadd_tma_dyn<HINT, ST_NA_EF>;
#endif
    }
    return nullptr;
}

tma_dyn_fn pick_tma_dyn(bool l2_hint, int st)
{
    return l2_hint ? pick_tma_dyn_st<true>(st) : pick_tma_dyn_st<false>(st);
}

tma_fn pick_tma(int store_mode, bool l2_hint, int st)
{
#ifdef B200VA_TUNE_MATRIX
    if (store_mode == 1)  // st hint is meaningless for bulk stores: one instantiation
        return l2_hint ? vadd_tma<1, true, ST_PLAIN> : vadd_tma<1, false, ST_PLAIN>;
    return l2_hint ? pick_tma_st<0, true>(st) : pick_tma_st<0, false>(st);
#else
    // the static-split ring (store modes 0/1) is not a production default: the tune library carries its
    // matrix, this library two forms
    if (store_mode == 1 && !l2_hint) return vadd_tma<1, false, ST_PLAIN>;   // kept: the bulk-store (UBLKCP.G.S) form
    if (store_mode == 0 && !l2_hint && st == ST_NA) return vadd_tma<0, false, ST_NA>;
    return nullptr;
#endif
}

// ----------------------------------------------------------------------- geometry
// Production choices per size class.  K_AUTO is always the 128-bit kernel; thread count / unroll /
// cache hints follow the footprint (12 n bytes) AND what the caller says about the data:
//
//  default (the same buffers may be launched again: the a1 loop)
//   n >= 2^25         HBM streaming, never L2-resident   512 thr x1, stores skip L1, L2 bulk prefetch ahead of the wait
//   2^23 < n < 2^25   footprint several x L2             128 thr x2, L2 evict-first loads
//   6 Mi <= n <= 2^23 footprint ~ 1.5-2 x L2             256 thr x2, stores skip L1
//   2^21 <= n < 6 Mi  partly L2-resident                 256 thr x2, plain hints (L2 keeps what fits)
//   n < 2^21          launch-bound                       512 thr (>= 2^19) / 128 thr, x1
//
//  B200VA_F_COLD (operands not in L2: the stager's chunks, rotating buffers).  The launch boundary is what
//  costs here (the previous grid's tail, then a full DRAM round trip before the first store), and the
//  always-legal L2 bulk prefetch ahead of griddepcontrol.wait (early_loads = 2) hides it without any promise
//  from the caller:
//   n >= 12 Mi         512 thr x1
//   3 Mi <= n < 12 Mi  512 thr x2
//   n < 3 Mi           256 thr x1
//  B200VA_F_COLD | B200VA_F_INPUTS_STABLE: from 3 Mi the prefetch form; below, register loads ahead of the
//  wait (early_loads = 1): 256 thr x4 from 1.5 Mi, 128 thr x2 from 0.5 Mi.
//  The class boundaries below 2^25 were chosen against the footprint; the 2^28 class is the one bench.py times.
void default_tune(int variant, size_t n, b200va_tune_t* t, unsigned flags = 0)
{
    std::memset(t, 0, sizeof *t);
    const bool cold = (flags & B200VA_F_COLD) != 0, early = (flags & B200VA_F_INPUTS_STABLE) != 0;
    t->early_loads = early ? 1 : 0;      // vec kernels only; K0 / K2 ignore it
    switch (variant) {
        case B200VA_K0_SCALAR:
            t->kind = B200VA_K0_SCALAR;
            t->threads = 256;
            t->unroll = 1;
            return;
        case B200VA_K2_TMA:               // TMA ring + dynamic tile scheduler
            t->kind = B200VA_K2_TMA;
            t->threads = n >= (size_t{1} << 25) ? 512 : 128;   // consumer threads (+32 producer)
            t->ctas_per_sm = 1;
            t->ld_hint = LD_PLAIN;
            t->st_hint = ST_NA;
            t->stages = n >= (size_t{1} << 25) ? 8 : 3;
            t->tile_bytes = 8192;
            t->store_mode = 2;
            return;
        case B200VA_K1_VEC128:
            t->kind = B200VA_K1_VEC128;
            t->threads = n < (size_t{1} << 19) ? 128 : 512;
            t->unroll = 1;
            t->ld_hint = LD_PLAIN;
            t->st_hint = ST_NA;
            return;
        case B200VA_K3_VEC256:
            t->kind = B200VA_K3_VEC256;
            t->threads = n < (size_t{1} << 26) ? 128 : 1024;
            t->unroll = 1;
            t->ld_hint = n < (size_t{1} << 26) ? LD_NA_EF : LD_PLAIN;
            t->st_hint = n < (size_t{1} << 26) ? ST_PLAIN : ST_NA;
            return;
        default:
            break;
    }
    // B200VA_K_AUTO
    t->kind = B200VA_K1_VEC128;
    t->unroll = 1;
    const size_t Mi = size_t{1} << 20;
    if (n >= 32 * Mi) {
        t->threads = 512; t->ld_hint = LD_PLAIN; t->st_hint = ST_NA;
        if (!early) t->early_loads = 2;
    } else if (cold) {
        t->ld_hint = LD_PLAIN; t->st_hint = ST_PLAIN;
        if (early && n < 3 * Mi) {                       // launch-latency dominated: register loads ahead of the wait
            if (n >= 3 * Mi / 2) { t->threads = 256; t->unroll = 4; }
            else if (n >= Mi / 2) { t->threads = 128; t->unroll = 2; }
            else t->threads = 128;
        } else {                                          // L2 bulk prefetch ahead of the wait
            t->early_loads = 2;
            if (n >= 12 * Mi) t->threads = 512;
            else if (n >= 3 * Mi) { t->threads = 512; t->unroll = 2; }
            else t->threads = n >= Mi / 2 ? 256 : 128;
        }
    } else if (n > 8 * Mi) {
        t->threads = 128; t->unroll = 2; t->ld_hint = LD_NA_EF; t->st_hint = ST_PLAIN;
    } else if (n >= 2 * Mi) {
        t->threads = 256; t->unroll = early ? 4 : 2; t->ld_hint = LD_PLAIN;
        t->st_hint = n >= 6 * Mi ? ST_NA : ST_PLAIN;            // from 6 Mi elements the output no longer fits next to the inputs
    } else if (n >= Mi / 2) {
        t->threads = 512; t->ld_hint = LD_PLAIN; t->st_hint = ST_PLAIN;
    } else {
        t->threads = 128; t->ld_hint = LD_PLAIN; t->st_hint = ST_PLAIN;
    }
}

// The named variants and B200VA_F_* hints the entry points accept.
int check_variant(int variant, unsigned flags = 0)
{
    if (variant < B200VA_K_AUTO || variant > B200VA_K3_VEC256) return B200VA_ERR_VARIANT;
    return (flags & ~(B200VA_F_INPUTS_STABLE | B200VA_F_COLD)) ? B200VA_ERR_INVALID : B200VA_OK;
}

// The tune b200va_add_f32_tuned runs for `in`: K_AUTO takes the whole AUTO tune for n, other zero
// fields the defaults of the tune's kind.
int complete_tune(const b200va_tune_t& in, size_t n, b200va_tune_t* out)
{
    b200va_tune_t t = in;
    b200va_tune_t d;
    default_tune(t.kind, n, &d);
    if (t.kind == B200VA_K_AUTO) t = d;
    if (t.kind == B200VA_K4_SCALAR_MLP) {
        if (t.threads == 0) t.threads = 256;
        if (t.unroll == 0) t.unroll = 8;
    }
    if (t.threads == 0) t.threads = d.threads;
    if (t.unroll == 0) t.unroll = d.unroll ? d.unroll : 1;
    if (t.stages == 0) t.stages = d.stages;
    if (t.tile_bytes == 0) t.tile_bytes = d.tile_bytes;
    if (t.early_loads < 0 || t.early_loads > 2 || (t.scheduler & ~1)) return B200VA_ERR_VARIANT;
    *out = t;
    return B200VA_OK;
}

inline bool is_pow2(int x) { return x > 0 && (x & (x - 1)) == 0; }

int check_args(const float* dA, const float* dB, const float* dC, size_t n)
{
    if (n == 0) return B200VA_OK;
    if (!dA || !dB || !dC) return B200VA_ERR_INVALID;
    const uintptr_t a = reinterpret_cast<uintptr_t>(dA), b = reinterpret_cast<uintptr_t>(dB),
                    c = reinterpret_cast<uintptr_t>(dC);
    if ((a | b | c) & 3u) return B200VA_ERR_ALIGN;
    if (n > (size_t{1} << 40)) return B200VA_ERR_INVALID;
    const uintptr_t bytes = n * sizeof(float);
    auto partial = [&](uintptr_t x) { return x != c && x < c + bytes && c < x + bytes; };
    if (partial(a) || partial(b)) return B200VA_ERR_OVERLAP;
    return B200VA_OK;
}

// ----------------------------------------------------------------------- launch plan
// The kernel forms of an add: the scalar control K0, the 4-byte kernel K4, the vec kernels of K1/K3 under
// the block scheduler or the dynamic tile scheduler (K1d), K2's TMA ring with a static or dynamic (K2d) split.
enum class Form { Scalar, K4, Vec, VecDyn, Tma, TmaDyn };

using scalar_fn = void (*)(const float*, const float*, float*, size_t);

// One launch as plan_launch decides it: run by launch(), reported by b200va_geometry().
struct Plan {
    Form form = Form::Scalar;
    scalar_fn scalar = nullptr;      // Scalar, K4
    VecFn vec;                       // Vec, VecDyn
    tma_fn tma = nullptr;
    tma_dyn_fn tma_dyn = nullptr;
    unsigned grid = 1, block = 0;
    size_t smem = 0, head = 0, nvec = 0, ntiles = 0;   // Scalar, K4: a tile is one CTA's threads x unroll elements
    bool ctr = false;                // dynamically scheduled: takes a two-word ticket counter
};

// Validates the tune for the plan's form and sets block, dynamic shared memory and tile count.
int plan_block(const b200va_tune_t& t, const b200va_devinfo_t* di, size_t n, Plan* p)
{
    if (t.threads < 32 || t.threads > 1024 || (t.threads & 31)) return B200VA_ERR_VARIANT;
    p->block = static_cast<unsigned>(t.threads);
    switch (p->form) {
        case Form::K4:
            if (t.unroll != 4 && t.unroll != 8 && t.unroll != 16) return B200VA_ERR_VARIANT;
            [[fallthrough]];
        case Form::Scalar: {
            const size_t per_cta = static_cast<size_t>(t.threads) * t.unroll;
            p->ntiles = (n + per_cta - 1) / per_cta;
            break;
        }
        case Form::Tma:
        case Form::TmaDyn: {
            if (t.threads > 992 || t.stages < 2 || t.stages > 32) return B200VA_ERR_VARIANT;
            if (t.tile_bytes < 2048 || (t.tile_bytes & 2047)) return B200VA_ERR_VARIANT;
            if (t.st_hint < 0 || t.st_hint >= ST_HINTS) return B200VA_ERR_VARIANT;
            if (t.store_mode < 0 || t.store_mode > 2) return B200VA_ERR_VARIANT;
            // ring + full/empty barriers; the dynamic-scheduler form adds a tile slot per stage
            const long long smem = static_cast<long long>(t.stages) * 2 * t.tile_bytes +
                                   (t.store_mode == 2 ? 20LL : 16LL) * t.stages;
            if (smem > di->max_smem_optin) return B200VA_ERR_VARIANT;
            p->smem = static_cast<size_t>(smem);
            p->ntiles = (p->nvec * 16u + t.tile_bytes - 1) / t.tile_bytes;
            p->block += 32;                                   // + the producer warp
            break;
        }
        case Form::Vec:
        case Form::VecDyn: {
            if (!is_pow2(t.unroll) || t.unroll > 8) return B200VA_ERR_VARIANT;
            if (t.ld_hint < 0 || t.ld_hint >= LD_HINTS || t.st_hint < 0 || t.st_hint >= ST_HINTS) return B200VA_ERR_VARIANT;
            if (t.scheduler < 0 || t.scheduler > 1 || (t.scheduler == 1 && t.ctas_per_sm != 0)) return B200VA_ERR_VARIANT;
            const size_t tile_vecs = static_cast<size_t>(t.threads) * t.unroll;
            p->ntiles = (p->nvec + tile_vecs - 1) / tile_vecs;
            break;
        }
    }
    if (p->ctr && p->ntiles > 0x7fffffffull) return B200VA_ERR_INVALID;   // 32-bit tile tickets
    return B200VA_OK;
}

// The grid: one CTA per tile, capped for the persistent forms at the CTAs that fit at once --
// `resident` per SM (the occupancy calculator's answer) under the dynamic scheduler, else ctas_per_sm.
int plan_grid(const b200va_tune_t& t, const b200va_devinfo_t* di, int resident, Plan* p)
{
    const size_t sms = static_cast<size_t>(di->sm_count);
    size_t grid = p->ntiles;
    if (p->form == Form::Tma || p->form == Form::TmaDyn) {
        grid = sms * static_cast<size_t>(p->ctr ? resident : t.ctas_per_sm > 0 ? t.ctas_per_sm : 1);
        if (grid > 0x7fffffffull) return B200VA_ERR_INVALID;
        if (grid > p->ntiles) grid = p->ntiles;
    } else if (p->form == Form::Vec || p->form == Form::VecDyn) {
        if (p->ctr && grid > sms * resident) grid = sms * resident;
        if (t.ctas_per_sm > 0 && grid > sms * t.ctas_per_sm) grid = sms * t.ctas_per_sm;
        if (grid > 0x7fffffffull) grid = 0x7fffffffull;   // the kernel loops tile += gridDim.x
    } else if (grid > 0x7fffffffull) {
        return B200VA_ERR_INVALID;
    }
    p->grid = static_cast<unsigned>(grid ? grid : 1);
    return B200VA_OK;
}

// Ticket counters of the dynamic tile scheduler for direct launches: a ring of kSchedSlots two-word
// slots per device, zeroed once and handed out round-robin, one per launch; the kernel's last CTA
// zeroes its slot again (b200va_ptx.cuh: sched_retire).  Launches on one stream are ordered (every
// counter access follows griddepcontrol.wait), so a slot is only ever shared by direct launches that
// are kSchedSlots apart in issue order and run concurrently on different streams.  A captured graph
// would keep its slots for every replay while the ring moves on and hands them to other launches,
// so a loop handle's graph takes its counters from the handle instead (b200va_loop::ctr).
constexpr unsigned kSchedSlots = 4096;

struct SchedPool {
    std::once_flag once;
    int rc = B200VA_OK;
    unsigned int* ctr = nullptr;
    std::atomic<unsigned> next{0};
};
SchedPool g_sched[kMaxDevices];

int sched_slot(int device, unsigned int** out)
{
    SchedPool& p = g_sched[device];
    std::call_once(p.once, [&] {
        void* d = nullptr;
        cudaError_t e = cudaMalloc(&d, size_t{kSchedSlots} * 2 * sizeof(unsigned int));
        if (e == cudaSuccess) e = cudaMemset(d, 0, size_t{kSchedSlots} * 2 * sizeof(unsigned int));
        if (e != cudaSuccess) { cudaGetLastError(); if (d) cudaFree(d); p.rc = cuda_err(e); return; }
        p.ctr = static_cast<unsigned int*>(d);
    });
    if (p.rc != B200VA_OK) return p.rc;
    *out = p.ctr + 2 * (p.next.fetch_add(1, std::memory_order_relaxed) % kSchedSlots);
    return B200VA_OK;
}

// The runtime's answers about one kernel on one device.
struct KernelAttrs {
    int max_block = 0, smem_optin = 0, resident = 0;
    unsigned res_block = 0;
    size_t res_smem = 0;
};
std::mutex g_attr_mu;
std::map<std::pair<const void*, int>, KernelAttrs> g_attrs;

// Refuses a CTA larger than `fn` runs (register-limited for the deep unrolls), opts in to `smem` bytes of
// dynamic shared memory and, given `resident`, returns the CTAs of this shape resident on one SM at once
// (cached for the last shape asked).  A cached answer makes no CUDA call.
int kernel_attrs(const void* fn, int device, unsigned block, size_t smem, int* resident)
{
    std::lock_guard<std::mutex> lk(g_attr_mu);
    KernelAttrs* k = nullptr;
    try {
        k = &g_attrs[{fn, device}];
    } catch (...) {
        return B200VA_ERR_NOMEM;
    }
    if (k->max_block == 0) {
        cudaFuncAttributes fa;
        CU_TRY(cudaFuncGetAttributes(&fa, fn));
        k->max_block = fa.maxThreadsPerBlock;
    }
    if (block > static_cast<unsigned>(k->max_block)) return B200VA_ERR_VARIANT;
    if (smem > static_cast<size_t>(k->smem_optin)) {
        CU_TRY(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
        k->smem_optin = static_cast<int>(smem);
    }
    if (resident) {
        if (k->resident == 0 || k->res_block != block || k->res_smem != smem) {
            int r = 0;
            CU_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&r, fn, static_cast<int>(block), smem));
            k->resident = r > 0 ? r : 1;
            k->res_block = block;
            k->res_smem = smem;
        }
        *resident = k->resident;
    }
    return B200VA_OK;
}

// The one place an add kernel and its geometry are decided, for C = A + B at these addresses (never
// dereferenced).  Each step runs once: alias rules, vector width and head peel, tune validation, kernel
// pick, register limit, shared-memory opt-in, occupancy, grid.
int plan_launch(b200va_tune_t t, const b200va_devinfo_t* di, const void* pa, const void* pb, const void* pc, size_t n,
                Plan* p)
{
    const uintptr_t a = reinterpret_cast<uintptr_t>(pa), b = reinterpret_cast<uintptr_t>(pb),
                    c = reinterpret_cast<uintptr_t>(pc);
    if (a == c || b == c) {
        // .nc (non-coherent) loads require data that is read-only for the kernel's lifetime
        if (t.ld_hint == LD_NC_NA) t.ld_hint = LD_PLAIN;
        // early register loads (1) read A and B while the previous launch may still be running: the
        // always-legal L2 prefetch (2) takes their place
        if (t.early_loads == 1) t.early_loads = 2;
    }

    int vw = 0;
    if (t.kind == B200VA_K3_VEC256) vw = 8;
    else if (t.kind == B200VA_K1_VEC128 || t.kind == B200VA_K2_TMA) vw = 4;
    else if (t.kind != B200VA_K0_SCALAR && t.kind != B200VA_K4_SCALAR_MLP) return B200VA_ERR_VARIANT;
    // vector body needs A, B, C equally misaligned w.r.t. the vector width (K3 falls back to 16 bytes)
    for (; vw; vw = vw == 8 ? 4 : 0) {
        const uintptr_t mask = static_cast<uintptr_t>(vw) * 4u - 1u;
        if ((a & mask) == (b & mask) && (a & mask) == (c & mask)) {
            p->head = ((static_cast<uintptr_t>(vw) * 4u - (a & mask)) & mask) / 4u;
            break;
        }
    }
    if (p->head > n) p->head = n;
    if (vw) p->nvec = (n - p->head) / static_cast<size_t>(vw);
    if (t.kind == B200VA_K0_SCALAR) {
        p->form = Form::Scalar;
        t.threads = 256;                  // the sample's launch shape
        t.unroll = 1;
    } else if (vw == 0) {
        // the explicit K4 variant, and the path taken when A, B, C share no 16-byte phase (no vector
        // body exists): 256 threads x 8 loads per array in flight
        if (t.kind != B200VA_K4_SCALAR_MLP) { t.threads = 256; t.unroll = 8; }
        p->form = Form::K4;
    } else if (t.kind == B200VA_K2_TMA) {
        p->form = t.store_mode == 2 ? Form::TmaDyn : Form::Tma;
    } else {
        p->form = t.scheduler == 1 ? Form::VecDyn : Form::Vec;
    }
    p->ctr = p->form == Form::VecDyn || p->form == Form::TmaDyn;

    RC_TRY(plan_block(t, di, n, p));

    const void* fn = nullptr;
    switch (p->form) {
        case Form::Scalar:
        case Form::K4:
            p->scalar = p->form == Form::Scalar ? vadd_scalar : t.unroll == 4 ? vadd_scalar_unrolled<4>
                      : t.unroll == 8 ? vadd_scalar_unrolled<8> : vadd_scalar_unrolled<16>;
            fn = reinterpret_cast<const void*>(p->scalar);
            break;
        case Form::Vec:
        case Form::VecDyn:
            p->vec = pick_vec(vw, t.unroll, t.ld_hint, t.st_hint, t.early_loads, t.scheduler);
            fn = p->vec.key();
            break;
        case Form::Tma:
            p->tma = pick_tma(t.store_mode, t.ld_hint == LD_NA_EF, t.st_hint);
            fn = reinterpret_cast<const void*>(p->tma);
            break;
        case Form::TmaDyn:
            p->tma_dyn = pick_tma_dyn(t.ld_hint == LD_NA_EF, t.st_hint);
            fn = reinterpret_cast<const void*>(p->tma_dyn);
            break;
    }
    if (!fn) return B200VA_ERR_VARIANT;   // not compiled into this library
    // CTAs of up to 256 threads are never register-limited (255 registers per thread fit)
    int resident = 1;
    if (p->block > 256 || p->smem || p->ctr)
        RC_TRY(kernel_attrs(fn, di->device, p->block, p->smem, p->ctr ? &resident : nullptr));
    return plan_grid(t, di, resident, p);
}

// Programmatic stream serialization lets launch k+1 ramp up behind launch k's tail (the kernels
// call griddepcontrol.wait before their first global access, so stream order is unchanged).  Every
// hot-path launch uses it unless B200VA_NO_PDL=1.
bool pdl_enabled()
{
    static const bool on = [] {
        const char* e = std::getenv("B200VA_NO_PDL");
        return !(e && e[0] == '1');
    }();
    return on;
}

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

// `ctr`: the dynamic tile scheduler's two-word ticket counter (zeroed; the kernel leaves it zeroed
// again); nullptr takes the next slot of the device's ring.
int launch(const float* dA, const float* dB, float* dC, size_t n, const b200va_tune_t& t, cudaStream_t stream, bool pdl,
           unsigned int* ctr = nullptr)
{
    RC_TRY(check_args(dA, dB, dC, n));
    const b200va_devinfo_t* di = nullptr;
    RC_TRY(current_dev_info(&di));
    if (n == 0) return B200VA_OK;
    Plan p;
    RC_TRY(plan_launch(t, di, dA, dB, dC, n, &p));
    if (p.ctr && !ctr) RC_TRY(sched_slot(di->device, &ctr));
    const uint32_t tile = static_cast<uint32_t>(t.tile_bytes), stages = static_cast<uint32_t>(t.stages);
    switch (p.form) {
        case Form::Scalar:   // the control keeps the sample's plain launch (no programmatic dependent launch)
            p.scalar<<<p.grid, p.block, 0, stream>>>(dA, dB, dC, n);
            return cuda_err(cudaGetLastError());
        case Form::K4:
            return launch_kernel(p.scalar, p.grid, p.block, 0, stream, pdl, dA, dB, dC, n);
        case Form::Vec:
            return launch_kernel(p.vec.plain, p.grid, p.block, 0, stream, pdl, dA, dB, dC, n, p.head, p.nvec, p.ntiles);
        case Form::VecDyn:
            return launch_kernel(p.vec.dyn, p.grid, p.block, 0, stream, pdl, dA, dB, dC, n, p.head, p.nvec, p.ntiles, ctr);
        case Form::Tma:
            return launch_kernel(p.tma, p.grid, p.block, p.smem, stream, pdl, dA, dB, dC, n, p.head, p.nvec, tile, stages);
        case Form::TmaDyn:
            return launch_kernel(p.tma_dyn, p.grid, p.block, p.smem, stream, pdl, dA, dB, dC, n, p.head, p.nvec, tile,
                                 stages, ctr);
    }
    return B200VA_ERR_VARIANT;
}

// `count` launches of the same add on `stream`.  One that follows what the caller queued runs `t`; one
// that follows the same add (`after_same` for the first), which writes only C, runs with early_loads = 1.
// `ctr`, if set, gives launch i the ticket counter at ctr + 2 i instead of a ring slot.
int launch_chain(const float* dA, const float* dB, float* dC, size_t n, const b200va_tune_t& t, bool after_same,
                 int count, cudaStream_t stream, bool pdl, unsigned int* ctr = nullptr)
{
    b200va_tune_t follow = t;
    follow.early_loads = 1;
    for (int i = 0; i < count; ++i)
        RC_TRY(launch(dA, dB, dC, n, i || after_same ? follow : t, stream, pdl, ctr ? ctr + 2 * i : nullptr));
    return B200VA_OK;
}

unsigned support_grid(const b200va_devinfo_t* di, size_t n, int threads)
{
    size_t want = (n + threads - 1) / threads;
    size_t cap = static_cast<size_t>(di->sm_count) * 16;
    if (want > cap) want = cap;
    if (want == 0) want = 1;
    return static_cast<unsigned>(want);
}

}  // namespace

// ----------------------------------------------------------------------- f4 dispatch
namespace {

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
    size_t head = ((16u - (a & 15u)) & 15u) / ES;
    if (head > n) head = n;
    const size_t nvec = (n - head) * ES / 16;
    // same footprint classes as the f32 add (default_tune), in 4-byte units
    const size_t m = n * ES / 4;
    unsigned threads = 128;
    int unroll = 1;
    bool skip_l1_stores = false;
    if (m >= (size_t{1} << 25)) {
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
    size_t grid = (nvec + tile_vecs - 1) / tile_vecs;
    if (grid > 0x7fffffffull) grid = 0x7fffffffull;
    if (grid == 0) grid = 1;
    const size_t ntiles = (nvec + tile_vecs - 1) / tile_vecs;
    using fn_t = void (*)(const void*, const void*, void*, size_t, size_t, size_t, size_t, S, int);
    const int prefetch_first = m >= (size_t{1} << 25) ? 1 : 0;      // >= 128 MiB per array: never L2-resident
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
// B share a 16-byte phase, else the scalar form; the HBM class of launch_stream_typed (>= 2^25 words
// per operand) prefetches each CTA's first rows into L2 ahead of the programmatic dependency.
template <int DT>
int launch_dot_typed(const void* dA, const void* dB, size_t n, double* ws, cudaStream_t st)
{
    constexpr size_t ES = dt_traits<DT>::size;
    const uintptr_t a = reinterpret_cast<uintptr_t>(dA), b = reinterpret_cast<uintptr_t>(dB);
    const unsigned grid = static_cast<unsigned>((n + DOT_CHUNK - 1) / DOT_CHUNK);
    const int prefetch_first = n * ES / 4 >= (size_t{1} << 25) ? 1 : 0;
    if ((a & 15u) != (b & 15u))
        return launch_kernel(dot_scalar<DT>, grid, DOT_SCALAR_THREADS, 0, st, pdl_enabled(), dA, dB, n, ws, prefetch_first);
    using F = dot_form<DT>;
    const size_t head = ((16u - (a & 15u)) & 15u) / ES;
    return launch_kernel(dot_vec<DT, F::threads, F::rows>, grid, F::threads, 0, st, pdl_enabled(), dA, dB, n, head, ws,
                         prefetch_first);
}

}  // namespace

// =============================================================================== ABI
extern "C" {

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
        case B200VA_ERR_NOMEM:     return "host allocation failed";
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

int b200va_resolve(int variant, size_t n, b200va_tune_t* out)
{
    return b200va_resolve_ex(variant, n, 0, out);
}

int b200va_resolve_ex(int variant, size_t n, unsigned flags, b200va_tune_t* out)
{
    if (!out) return B200VA_ERR_VARIANT;
    RC_TRY(check_variant(variant, flags));
    default_tune(variant, n, out, flags);
    return B200VA_OK;
}

int b200va_geometry(const b200va_tune_t* tune, size_t n, int device, unsigned* grid, unsigned* block,
                    unsigned* dyn_smem_bytes)
{
    if (!tune || !grid || !block) return B200VA_ERR_INVALID;
    const b200va_devinfo_t* di = nullptr;
    RC_TRY(dev_info(device, &di));
    b200va_tune_t t;
    RC_TRY(complete_tune(*tune, n, &t));
    DeviceGuard guard(device);
    CU_TRY(guard.err);
    // notional operands, distinct and 256-byte aligned: the plan reads only their values
    const float* base = reinterpret_cast<const float*>(uintptr_t{256});
    Plan p;
    RC_TRY(plan_launch(t, di, base, base + 64, base + 128, n, &p));
    *grid = p.grid;
    *block = p.block;
    if (dyn_smem_bytes) *dyn_smem_bytes = static_cast<unsigned>(p.smem);
    return B200VA_OK;
}

int b200va_add_f32(const float* dA, const float* dB, float* dC, size_t n, int variant, void* stream)
{
    return b200va_add_f32_ex(dA, dB, dC, n, variant, 0, stream);
}

int b200va_add_f32_ex(const float* dA, const float* dB, float* dC, size_t n, int variant, unsigned flags, void* stream)
{
    RC_TRY(check_variant(variant, flags));
    b200va_tune_t t;
    default_tune(variant, n, &t, flags);
    return launch(dA, dB, dC, n, t, static_cast<cudaStream_t>(stream), pdl_enabled());
}

int b200va_add_f32_tuned(const float* dA, const float* dB, float* dC, size_t n,
                         const b200va_tune_t* tune, void* stream)
{
    if (!tune) return B200VA_ERR_INVALID;
    b200va_tune_t t;
    RC_TRY(complete_tune(*tune, n, &t));
    return launch(dA, dB, dC, n, t, static_cast<cudaStream_t>(stream), pdl_enabled());
}

// ---- a1: the launch loop --------------------------------------------------------------
struct b200va_loop {
    const float *dA = nullptr, *dB = nullptr;
    float* dC = nullptr;
    size_t n = 0;
    b200va_tune_t tune{};
    int batch = 1;
    int device = 0;
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    // ticket counters of the graph's nodes (two words per node) when the tune is dynamically
    // scheduled: owned by the handle, so no other launch can be handed them while the graph replays
    unsigned int* ctr = nullptr;
};

static int capture_batch(b200va_loop* l, cudaStream_t cap, bool pdl)
{
    CU_TRY(cudaStreamBeginCapture(cap, cudaStreamCaptureModeThreadLocal));
    // node 0 follows an unknown predecessor
    const int rc = launch_chain(l->dA, l->dB, l->dC, l->n, l->tune, false, l->batch, cap, pdl, l->ctr);
    cudaGraph_t g = nullptr;
    const cudaError_t e = cudaStreamEndCapture(cap, &g);
    if (rc != B200VA_OK || e != cudaSuccess) {
        if (g) cudaGraphDestroy(g);
        cudaGetLastError();
        return rc != B200VA_OK ? rc : cuda_err(e);
    }
    cudaGraphExec_t x = nullptr;
    const cudaError_t e2 = cudaGraphInstantiate(&x, g, 0);
    if (e2 != cudaSuccess) { cudaGraphDestroy(g); cudaGetLastError(); return cuda_err(e2); }
    l->graph = g;
    l->exec = x;
    return B200VA_OK;
}

// The handle's device, counters and graph.  A failure leaves what was made to b200va_loop_destroy.
static int loop_init(b200va_loop* l)
{
    CU_TRY(cudaGetDevice(&l->device));
    if (l->batch <= 1 || l->n == 0) return B200VA_OK;
    cudaStream_t cap = nullptr;
    CU_TRY(cudaStreamCreateWithFlags(&cap, cudaStreamNonBlocking));
    cudaError_t e = cudaSuccess;
    if (l->tune.scheduler == 1 || (l->tune.kind == B200VA_K2_TMA && l->tune.store_mode == 2)) {
        const size_t bytes = static_cast<size_t>(l->batch) * 2 * sizeof(unsigned int);
        void* d = nullptr;
        e = cudaMalloc(&d, bytes);
        l->ctr = static_cast<unsigned int*>(d);
        if (e == cudaSuccess) e = cudaMemsetAsync(d, 0, bytes, cap);
        if (e == cudaSuccess) e = cudaStreamSynchronize(cap);   // zero before the first replay, on any stream
        if (e != cudaSuccess) cudaGetLastError();
    }
    int rc = cuda_err(e);
    if (rc == B200VA_OK) {
        rc = capture_batch(l, cap, pdl_enabled());
        // older drivers: capture without programmatic edges (same counters: a failed capture ran nothing)
        if (rc != B200VA_OK && pdl_enabled()) rc = capture_batch(l, cap, false);
    }
    cudaStreamDestroy(cap);
    return rc;
}

int b200va_loop_destroy(b200va_loop_t* l)
{
    if (!l) return B200VA_OK;
    if (l->exec) cudaGraphExecDestroy(l->exec);
    if (l->graph) cudaGraphDestroy(l->graph);
    if (l->ctr) cudaFree(l->ctr);
    delete l;
    return B200VA_OK;
}

int b200va_loop_create(b200va_loop_t** out, const float* dA, const float* dB, float* dC, size_t n, int variant,
                       int graph_batch)
{
    if (!out || graph_batch < 0) return B200VA_ERR_INVALID;
    *out = nullptr;
    RC_TRY(check_variant(variant));
    RC_TRY(check_args(dA, dB, dC, n));
    b200va_loop* l = new (std::nothrow) b200va_loop;
    if (!l) return B200VA_ERR_NOMEM;
    l->dA = dA; l->dB = dB; l->dC = dC; l->n = n;
    l->batch = graph_batch > 1 ? graph_batch : 1;
    default_tune(variant, n, &l->tune);
    const int rc = loop_init(l);
    if (rc != B200VA_OK) { b200va_loop_destroy(l); return rc; }
    *out = l;
    return B200VA_OK;
}

int b200va_loop_run(b200va_loop_t* l, int iters, void* stream)
{
    if (!l || iters < 0) return B200VA_ERR_INVALID;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int left = iters;
    if (l->exec)
        for (; left >= l->batch; left -= l->batch) CU_TRY(cudaGraphLaunch(l->exec, st));
    // the rest are direct launches; the first follows whatever the caller queued unless a replay ran
    return launch_chain(l->dA, l->dB, l->dC, l->n, l->tune, left < iters, left, st, pdl_enabled());
}

int b200va_add_f32_loop(const float* dA, const float* dB, float* dC, size_t n, int variant, int iters,
                        int graph_batch, void* stream)
{
    if (iters < 0 || graph_batch < 0) return B200VA_ERR_INVALID;
    RC_TRY(check_variant(variant));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (graph_batch <= 1 || iters < graph_batch) {
        b200va_tune_t t;
        default_tune(variant, n, &t);
        return launch_chain(dA, dB, dC, n, t, false, iters, st, pdl_enabled());
    }
    b200va_loop_t* l = nullptr;
    RC_TRY(b200va_loop_create(&l, dA, dB, dC, n, variant, graph_batch));
    int rc = b200va_loop_run(l, iters, stream);
    // the executable graph must outlive its launches: the one-shot form drains the stream
    const cudaError_t e = cudaStreamSynchronize(st);
    b200va_loop_destroy(l);
    if (rc == B200VA_OK) rc = cuda_err(e);
    return rc;
}

// ------------------------------------------------------------------ a2: input recipes
int b200va_host_fill_rand_f32(float* hA, float* hB, size_t n)
{
    if (n && (!hA || !hB)) return B200VA_ERR_INVALID;
    srand(1);  // a fresh ./vectorAdd process never calls srand: glibc default seed is 1
    for (size_t i = 0; i < n; ++i) {
        hA[i] = rand() / (float)RAND_MAX;
        hB[i] = rand() / (float)RAND_MAX;
    }
    return B200VA_OK;
}

static inline uint64_t host_splitmix64(uint64_t z)
{
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

int b200va_host_fill_ctr_f32(float* h, size_t n, uint64_t seed, uint64_t first)
{
    if (n && !h) return B200VA_ERR_INVALID;
    const uint64_t base = seed * 0x9E3779B97F4A7C15ull + first;
    for (size_t i = 0; i < n; ++i)
        h[i] = static_cast<float>(static_cast<uint32_t>(host_splitmix64(base + i) >> 40)) * 0x1.0p-24f;
    return B200VA_OK;
}

int b200va_fill_ctr_f32(float* d, size_t n, uint64_t seed, uint64_t first, void* stream)
{
    if (n && !d) return B200VA_ERR_INVALID;
    const b200va_devinfo_t* di = nullptr;
    RC_TRY(current_dev_info(&di));
    if (n == 0) return B200VA_OK;
    const uint64_t base = seed * 0x9E3779B97F4A7C15ull + first;
    if ((reinterpret_cast<uintptr_t>(d) & 15u) == 0)      // the usual case: one STG.128 per four elements
        fill_ctr_vec<<<support_grid(di, (n + 3) / 4, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(d, n, base);
    else
        fill_ctr<<<support_grid(di, n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(d, n, base);
    return cuda_err(cudaGetLastError());
}

// ------------------------------------------------------------------ a6: verification
int b200va_host_verify_f32(const float* hA, const float* hB, const float* hC, size_t n, size_t* first_bad)
{
    if (n && (!hA || !hB || !hC)) return B200VA_ERR_INVALID;
    for (size_t i = 0; i < n; ++i) {
        const float want = hA[i] + hB[i];
        uint32_t uw, ug;
        std::memcpy(&uw, &want, 4);
        std::memcpy(&ug, &hC[i], 4);
        if (uw == ug) continue;
        const bool nw = (uw & 0x7fffffffu) > 0x7f800000u, ng = (ug & 0x7fffffffu) > 0x7f800000u;
        if (nw && ng) continue;
        if (first_bad) *first_bad = i;
        return B200VA_ERR_VERIFY;
    }
    return B200VA_OK;
}

int b200va_verify_f32(const float* dA, const float* dB, const float* dC, size_t n,
                      uint64_t* d_result, void* stream)
{
    if (!d_result || (n && (!dA || !dB || !dC))) return B200VA_ERR_INVALID;
    const b200va_devinfo_t* di = nullptr;
    RC_TRY(current_dev_info(&di));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    auto* res = reinterpret_cast<unsigned long long*>(d_result);
    reset_verify<<<1, 1, 0, st>>>(res);
    const bool aligned = ((reinterpret_cast<uintptr_t>(dA) | reinterpret_cast<uintptr_t>(dB) | reinterpret_cast<uintptr_t>(dC)) & 15u) == 0;
    if (n && aligned) verify_bits_vec<<<support_grid(di, (n + 3) / 4, 256), 256, 0, st>>>(dA, dB, dC, n, res);
    else if (n) verify_bits<<<support_grid(di, n, 256), 256, 0, st>>>(dA, dB, dC, n, res);
    return cuda_err(cudaGetLastError());
}

int b200va_digest_f32(const float* d, size_t n, uint64_t* d_out, void* stream)
{
    if (!d_out || (n && !d)) return B200VA_ERR_INVALID;
    const b200va_devinfo_t* di = nullptr;
    RC_TRY(current_dev_info(&di));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    auto* out = reinterpret_cast<unsigned long long*>(d_out);
    reset_digest<<<1, 1, 0, st>>>(out);
    if (n && (reinterpret_cast<uintptr_t>(d) & 15u) == 0) digest_bits_vec<<<support_grid(di, (n + 3) / 4, 256), 256, 0, st>>>(d, n, out);
    else if (n) digest_bits<<<support_grid(di, n, 256), 256, 0, st>>>(d, n, out);
    return cuda_err(cudaGetLastError());
}

// ------------------------------------------------------------------ f4: STREAM-style ops
int b200va_stream(int op, int dtype, const void* dA, const void* dB, void* dC, size_t n, double scalar, void* stream)
{
    if (op < 0 || op >= OP_COUNT || dtype < 0 || dtype >= DT_COUNT) return B200VA_ERR_VARIANT;
    const b200va_devinfo_t* di = nullptr;
    RC_TRY(current_dev_info(&di));
    if (n == 0) return B200VA_OK;
    const bool binary = (op == OP_ADD || op == OP_TRIAD);
    if (!dA || !dC || (binary && !dB)) return B200VA_ERR_INVALID;
    const size_t es = dtype == DT_F64 ? 8 : dtype == DT_F32 ? 4 : 2;
    const uintptr_t a = reinterpret_cast<uintptr_t>(dA), b = reinterpret_cast<uintptr_t>(dB),
                    c = reinterpret_cast<uintptr_t>(dC);
    if (((a | c | (binary ? b : 0)) & (es - 1)) != 0) return B200VA_ERR_ALIGN;
    if (n > (size_t{1} << 40)) return B200VA_ERR_INVALID;
    const uintptr_t bytes = n * es;
    auto partial = [&](uintptr_t x) { return x != c && x < c + bytes && c < x + bytes; };
    if (partial(a) || (binary && partial(b))) return B200VA_ERR_OVERLAP;
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
    const b200va_devinfo_t* di = nullptr;
    RC_TRY(current_dev_info(&di));
    if (n > (size_t{1} << 40)) return B200VA_ERR_INVALID;
    const size_t need = b200va_dot_workspace_bytes(n);
    if (!d_out || (n && (!dA || !dB)) || (need && !d_workspace) || workspace_bytes < need) return B200VA_ERR_INVALID;
    const size_t es = dtype == DT_F64 ? 8 : dtype == DT_F32 ? 4 : 2;
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

// ------------------------------------------------------------------ ceiling probes
int b200va_probe_f32(int kind, const float* dA, const float* dB, float* dC, size_t n, void* stream)
{
    if (kind < B200VA_PROBE_READ2 || kind > B200VA_PROBE_COPY) return B200VA_ERR_VARIANT;
    const b200va_devinfo_t* di = nullptr;
    RC_TRY(current_dev_info(&di));
    const size_t nvec = n / 4;
    if (nvec == 0) return B200VA_OK;
    if (!dC || (kind != B200VA_PROBE_FILL && !dA) || (kind == B200VA_PROBE_READ2 && !dB)) return B200VA_ERR_INVALID;
    const uintptr_t bits = reinterpret_cast<uintptr_t>(dC) | (kind != B200VA_PROBE_FILL ? reinterpret_cast<uintptr_t>(dA) : 0) |
                           (kind == B200VA_PROBE_READ2 ? reinterpret_cast<uintptr_t>(dB) : 0);
    if (bits & 15u) return B200VA_ERR_ALIGN;
    const size_t blocks = (nvec + 511) / 512;
    if (blocks > 0x7fffffffull) return B200VA_ERR_INVALID;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const unsigned grid = static_cast<unsigned>(blocks);
    switch (kind) {
        case B200VA_PROBE_READ2: return launch_kernel(probe_read2, grid, 512u, 0, st, pdl_enabled(), dA, dB, dC, nvec);
        case B200VA_PROBE_FILL:  return launch_kernel(probe_fill, grid, 512u, 0, st, pdl_enabled(), dC, nvec, 1.0f);
        default:                 return launch_kernel(probe_copy, grid, 512u, 0, st, pdl_enabled(), dA, dC, nvec);
    }
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

// ------------------------------------------------------------------ host-buffer path
// Fork-join pool for the pageable path: T persistent workers, each copies one slice.
// Construction may throw (std::system_error from std::thread under a pids limit, bad_alloc):
// make_copy_pool() catches and degrades, nothing propagates through the C ABI.
class CopyPool {
public:
    explicit CopyPool(int threads) : n_(threads < 1 ? 1 : threads)
    {
        th_.reserve(static_cast<size_t>(n_));
        try {
            for (int i = 1; i < n_; ++i) th_.emplace_back([this, i] { worker(i); });
        } catch (...) {
            n_ = static_cast<int>(th_.size()) + 1;          // run with the workers that did start
        }
    }
    ~CopyPool()
    {
        { std::lock_guard<std::mutex> lk(m_); stop_ = true; ++gen_; }
        cv_.notify_all();
        for (auto& t : th_) t.join();
    }
    int size() const { return n_; }
    // dst[0..bytes) = src[0..bytes), split in 64-byte-aligned slices over the pool (caller = slice 0)
    void copy(void* dst, const void* src, size_t bytes)
    {
        if (bytes < (size_t{1} << 20) || n_ == 1) { std::memcpy(dst, src, bytes); return; }
        {
            std::lock_guard<std::mutex> lk(m_);
            dst_ = static_cast<unsigned char*>(dst); src_ = static_cast<const unsigned char*>(src); bytes_ = bytes;
            pending_ = n_ - 1;
            ++gen_;
        }
        cv_.notify_all();
        slice(0);
        std::unique_lock<std::mutex> lk(m_);
        done_.wait(lk, [this] { return pending_ == 0; });
    }

private:
    void slice(int i)
    {
        size_t per = (bytes_ + static_cast<size_t>(n_) - 1) / static_cast<size_t>(n_);
        per = (per + 63) & ~size_t{63};
        const size_t lo = std::min(bytes_, per * static_cast<size_t>(i)), hi = std::min(bytes_, lo + per);
        if (hi > lo) std::memcpy(dst_ + lo, src_ + lo, hi - lo);
    }
    void worker(int i)
    {
        unsigned long seen = 0;
        for (;;) {
            {
                std::unique_lock<std::mutex> lk(m_);
                cv_.wait(lk, [&] { return gen_ != seen; });
                seen = gen_;
                if (stop_) return;
            }
            if (i < n_) slice(i);
            std::lock_guard<std::mutex> lk(m_);
            if (--pending_ == 0) done_.notify_one();
        }
    }
    int n_;
    std::vector<std::thread> th_;
    std::mutex m_;
    std::condition_variable cv_, done_;
    unsigned long gen_ = 0;
    int pending_ = 0;
    bool stop_ = false;
    unsigned char* dst_ = nullptr;
    const unsigned char* src_ = nullptr;
    size_t bytes_ = 0;
};

// Copy threads: the CPUs this process may use (affinity mask, cgroup v2 bandwidth quota), at
// most 16; B200VA_COPY_THREADS overrides (clamped to 1..64).  Never throws: returns nullptr
// only if even a single-threaded pool cannot be allocated.
static CopyPool* make_copy_pool()
{
    unsigned hw = std::thread::hardware_concurrency();
    cpu_set_t set;
    if (sched_getaffinity(0, sizeof set, &set) == 0 && CPU_COUNT(&set) > 0) hw = static_cast<unsigned>(CPU_COUNT(&set));
    if (FILE* f = std::fopen("/sys/fs/cgroup/cpu.max", "r")) {
        char q[64];
        double period = 0;
        if (std::fscanf(f, "%63s %lf", q, &period) == 2 && std::strcmp(q, "max") != 0 && period > 0)
            hw = std::min(hw, static_cast<unsigned>(std::max(1.0, std::atof(q) / period)));
        std::fclose(f);
    }
    unsigned want = std::max(1u, std::min(16u, hw));
    if (const char* e = std::getenv("B200VA_COPY_THREADS")) want = static_cast<unsigned>(std::min(64, std::max(1, std::atoi(e))));
    for (; want >= 1; want /= 2) {
        try {
            return new CopyPool(static_cast<int>(want));
        } catch (...) {
            // bad_alloc / system_error while building the pool: retry smaller
        }
        if (want == 1) break;
    }
    return nullptr;
}

struct HostRange { uintptr_t lo, hi; };     // [lo, hi) page-locked by this stager (mode 4)

struct b200va_stager {
    int device = 0;
    size_t chunk = 0;
    int depth = 0;
    float* d_buf = nullptr;            // depth * 3 * chunk floats
    cudaStream_t main = nullptr;
    cudaStream_t* slot = nullptr;
    cudaEvent_t* slot_done = nullptr;
    cudaEvent_t ev_start = nullptr, ev_stop = nullptr;
    // "lanes" pipeline (mode 2): one stream per direction + one for the kernel, events per slot
    cudaStream_t lane_h2d = nullptr, lane_k = nullptr, lane_d2h = nullptr;
    cudaEvent_t *ev_in = nullptr, *ev_sum = nullptr, *ev_out = nullptr;
    // pageable path (mode 3): pinned bounce chunks (depth * 3 * bounce_chunk floats) + copy threads, made on first use
    float* bounce = nullptr;
    size_t bounce_chunk = 0;
    CopyPool* pool = nullptr;
    // register-once path (mode 4): host ranges this stager page-locked
    std::vector<HostRange>* regs = nullptr;
    float last_ms = 0.f;
    int last_mode = -1;
};

// NUMA node a CUDA device hangs off (sysfs), or -1.  B200VA_NUMA_NODE overrides.
static int device_numa_node_of(int dev)
{
    if (const char* e = std::getenv("B200VA_NUMA_NODE")) return std::atoi(e);
    char bus[32] = {0}, path[128];
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, dev) != cudaSuccess) { cudaGetLastError(); return -1; }
    for (char* c = bus; *c; ++c) *c = static_cast<char>(std::tolower(*c));
    std::snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
    int node = -1;
    if (FILE* f = std::fopen(path, "r")) {
        if (std::fscanf(f, "%d", &node) != 1) node = -1;
        std::fclose(f);
    }
    return node;
}

static int device_numa_node()
{
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return -1; }
    return device_numa_node_of(dev);
}

// Parses a sysfs cpulist ("0-31,64-95") into a cpu_set_t restricted to `allowed`.
static bool node_cpuset(int node, const cpu_set_t& allowed, cpu_set_t* out)
{
    char path[96], buf[4096];
    std::snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
    FILE* f = std::fopen(path, "r");
    if (!f) return false;
    const bool ok = std::fgets(buf, sizeof buf, f) != nullptr;
    std::fclose(f);
    if (!ok) return false;
    CPU_ZERO(out);
    int count = 0;
    for (char* p = buf; *p && *p != '\n';) {
        char* end = nullptr;
        long lo = std::strtol(p, &end, 10), hi = lo;
        if (end == p) break;
        if (*end == '-') hi = std::strtol(end + 1, &end, 10);
        for (long c = lo; c <= hi && c < CPU_SETSIZE; ++c)
            if (CPU_ISSET(c, &allowed)) { CPU_SET(c, out); ++count; }
        p = (*end == ',') ? end + 1 : end;
    }
    return count > 0;
}

// Pinned, mapped host memory whose pages sit on the NUMA node local to the current GPU:
// the calling thread is moved onto that node's CPUs (and its memory policy set to prefer
// the node) for the duration of the allocation, so the first touch inside cudaHostAlloc
// lands there; a PCIe DMA then never crosses the inter-socket link.  Affinity and memory
// policy of the caller (e.g. numactl --interleave) are saved and put back.
int b200va_host_alloc_ex(void** out, size_t bytes, int write_combined)
{
    if (!out) return B200VA_ERR_INVALID;
    const int node = device_numa_node();
    cpu_set_t old_set, node_set;
    bool moved = false, policy = false;
    int old_mode = 0;
    unsigned long old_mask[16] = {0};                       // 1024 nodes
    constexpr unsigned long kMaxNode = sizeof old_mask * 8;
    if (node >= 0 && sched_getaffinity(0, sizeof old_set, &old_set) == 0 && node_cpuset(node, old_set, &node_set)) {
        moved = sched_setaffinity(0, sizeof node_set, &node_set) == 0;
        if (node < 64 && syscall(SYS_get_mempolicy, &old_mode, old_mask, kMaxNode, nullptr, 0ul) == 0) {
            unsigned long mask = 1ul << node;
            policy = syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, &mask, 65ul) == 0;
        }
    }
    unsigned flags = cudaHostAllocPortable | cudaHostAllocMapped;
    if (write_combined) flags |= cudaHostAllocWriteCombined;   // H2D sources only: CPU reads of WC memory crawl
    const cudaError_t e = cudaHostAlloc(out, bytes ? bytes : 1, flags);
    if (policy) {
        bool any = false;
        for (unsigned long w : old_mask) any = any || w != 0;
        if (syscall(SYS_set_mempolicy, old_mode, any ? old_mask : nullptr, any ? kMaxNode : 0ul) != 0)
            syscall(SYS_set_mempolicy, 0 /* MPOL_DEFAULT */, nullptr, 0ul);
    }
    if (moved) sched_setaffinity(0, sizeof old_set, &old_set);
    CU_TRY(e);
    return B200VA_OK;
}

int b200va_host_alloc(void** out, size_t bytes) { return b200va_host_alloc_ex(out, bytes, 0); }

// NUMA node the current CUDA device is attached to (sysfs), or -1.
int b200va_device_numa_node(void) { return device_numa_node(); }
int b200va_device_numa_node_of(int device) { return device_numa_node_of(device); }

// NUMA node holding the page at `p` (get_mempolicy(MPOL_F_NODE | MPOL_F_ADDR)), or -1.
int b200va_host_node_of(const void* p)
{
    int node = -1;
    if (!p) return -1;
    if (syscall(SYS_get_mempolicy, &node, nullptr, 0ul, const_cast<void*>(p), 3ul /* F_NODE|F_ADDR */) != 0) return -1;
    return node;
}

int b200va_host_free(void* p)
{
    if (!p) return B200VA_OK;
    CU_TRY(cudaFreeHost(p));
    return B200VA_OK;
}

static void stager_release_host(b200va_stager* s)
{
    if (!s->regs) return;
    for (const HostRange& r : *s->regs)
        if (cudaHostUnregister(reinterpret_cast<void*>(r.lo)) != cudaSuccess) cudaGetLastError();
    s->regs->clear();
}

int b200va_stager_release_host(b200va_stager_t* s)
{
    if (!s) return B200VA_ERR_INVALID;
    DeviceGuard g(s->device);
    stager_release_host(s);
    return B200VA_OK;
}

int b200va_stager_destroy(b200va_stager_t* s)
{
    if (!s) return B200VA_OK;
    DeviceGuard g(s->device);
    stager_release_host(s);
    delete s->regs;
    if (s->slot) {
        for (int i = 0; i < s->depth; ++i) {
            if (s->slot[i]) cudaStreamDestroy(s->slot[i]);
            if (s->slot_done && s->slot_done[i]) cudaEventDestroy(s->slot_done[i]);
        }
    }
    for (cudaStream_t st : {s->lane_h2d, s->lane_k, s->lane_d2h})
        if (st) cudaStreamDestroy(st);
    for (cudaEvent_t* arr : {s->ev_in, s->ev_sum, s->ev_out}) {
        if (!arr) continue;
        for (int i = 0; i < s->depth; ++i)
            if (arr[i]) cudaEventDestroy(arr[i]);
        delete[] arr;
    }
    if (s->main) cudaStreamDestroy(s->main);
    if (s->ev_start) cudaEventDestroy(s->ev_start);
    if (s->ev_stop) cudaEventDestroy(s->ev_stop);
    if (s->d_buf) cudaFree(s->d_buf);
    if (s->bounce) cudaFreeHost(s->bounce);
    delete s->pool;
    delete[] s->slot;
    delete[] s->slot_done;
    delete s;
    return B200VA_OK;
}

int b200va_stager_create(b200va_stager_t** out, int device, size_t chunk_elems, int depth)
{
    if (!out) return B200VA_ERR_INVALID;
    *out = nullptr;
    if (chunk_elems == 0) chunk_elems = size_t{1} << 25;   // 128 MiB per array per slot (the lanes pipeline tapers the tail)
    if (depth == 0) depth = 3;
    if (depth < 1 || depth > 16) return B200VA_ERR_INVALID;
    chunk_elems = (chunk_elems + 63) & ~size_t{63};        // slots stay 256-B aligned
    RC_TRY(dev_info(device, nullptr));
    DeviceGuard guard(device);
    CU_TRY(guard.err);
    b200va_stager* s = new (std::nothrow) b200va_stager;
    if (!s) return B200VA_ERR_NOMEM;
    s->device = device;
    s->chunk = chunk_elems;
    s->depth = depth;
    s->slot = new (std::nothrow) cudaStream_t[depth]();
    s->slot_done = new (std::nothrow) cudaEvent_t[depth]();
    s->regs = new (std::nothrow) std::vector<HostRange>();
    if (!s->slot || !s->slot_done || !s->regs) { b200va_stager_destroy(s); return B200VA_ERR_NOMEM; }
    cudaError_t e = cudaMalloc(&s->d_buf, static_cast<size_t>(depth) * 3 * chunk_elems * sizeof(float));
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s->main, cudaStreamNonBlocking);
    for (int i = 0; i < depth && e == cudaSuccess; ++i) {
        e = cudaStreamCreateWithFlags(&s->slot[i], cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->slot_done[i], cudaEventDisableTiming);
    }
    if (e == cudaSuccess) e = cudaEventCreate(&s->ev_start);
    if (e == cudaSuccess) e = cudaEventCreate(&s->ev_stop);
    s->ev_in = new (std::nothrow) cudaEvent_t[depth]();
    s->ev_sum = new (std::nothrow) cudaEvent_t[depth]();
    s->ev_out = new (std::nothrow) cudaEvent_t[depth]();
    if (!s->ev_in || !s->ev_sum || !s->ev_out) { b200va_stager_destroy(s); return B200VA_ERR_NOMEM; }
    for (cudaStream_t* st : {&s->lane_h2d, &s->lane_k, &s->lane_d2h})
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(st, cudaStreamNonBlocking);
    for (int i = 0; i < depth && e == cudaSuccess; ++i) {
        e = cudaEventCreateWithFlags(&s->ev_in[i], cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->ev_sum[i], cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->ev_out[i], cudaEventDisableTiming);
    }
    if (e != cudaSuccess) { b200va_stager_destroy(s); return cuda_err(e); }
    *out = s;
    return B200VA_OK;
}

// ---- the pipelines (device already current; a non-OK return leaves work in flight: the caller drains)
static int stage_zero_copy(b200va_stager* s, const float* hA, const float* hB, float* hC, size_t n, int variant)
{
    // the kernel streams A and B from pinned host memory over PCIe and writes C back the same
    // way -- both link directions busy, no staging latency.
    const float *dA = nullptr, *dB = nullptr;
    float* dC = nullptr;
    if (n) {
        CU_TRY(cudaHostGetDevicePointer(reinterpret_cast<void**>(const_cast<float**>(&dA)), const_cast<float*>(hA), 0));
        CU_TRY(cudaHostGetDevicePointer(reinterpret_cast<void**>(const_cast<float**>(&dB)), const_cast<float*>(hB), 0));
        CU_TRY(cudaHostGetDevicePointer(reinterpret_cast<void**>(&dC), hC, 0));
    }
    b200va_tune_t t;
    default_tune(variant == B200VA_K_AUTO ? B200VA_K1_VEC128 : variant, n, &t);
    return launch(dA, dB, dC, n, t, s->main, pdl_enabled());
}

static int stage_slots(b200va_stager* s, const float* hA, const float* hB, float* hC, size_t n, int variant)
{
    const size_t nchunks = (n + s->chunk - 1) / s->chunk;
    for (int i = 0; i < s->depth; ++i) CU_TRY(cudaStreamWaitEvent(s->slot[i], s->ev_start, 0));
    b200va_tune_t t;
    for (size_t k = 0; k < nchunks; ++k) {
        const int i = static_cast<int>(k % static_cast<size_t>(s->depth));
        const size_t off = k * s->chunk;
        const size_t m = (n - off < s->chunk) ? n - off : s->chunk;
        float* dA = s->d_buf + static_cast<size_t>(i) * 3 * s->chunk;
        float* dB = dA + s->chunk;
        float* dC = dB + s->chunk;
        CU_TRY(cudaMemcpyAsync(dA, hA + off, m * sizeof(float), cudaMemcpyHostToDevice, s->slot[i]));
        CU_TRY(cudaMemcpyAsync(dB, hB + off, m * sizeof(float), cudaMemcpyHostToDevice, s->slot[i]));
        default_tune(variant, m, &t, B200VA_F_COLD);      // a chunk fresh off the copy engine is never in L2
        RC_TRY(launch(dA, dB, dC, m, t, s->slot[i], pdl_enabled()));
        CU_TRY(cudaMemcpyAsync(hC + off, dC, m * sizeof(float), cudaMemcpyDeviceToHost, s->slot[i]));
    }
    for (int i = 0; i < s->depth; ++i) {
        CU_TRY(cudaEventRecord(s->slot_done[i], s->slot[i]));
        CU_TRY(cudaStreamWaitEvent(s->main, s->slot_done[i], 0));
    }
    return B200VA_OK;
}

// Fault injection for the error-path test (tests/test_gpu_host_path.py): with
// B200VA_TEST_FAIL_CHUNK=k in the environment the lanes pipeline fails ONCE per process, right
// after it has queued chunk k's H2D copies -- i.e. with DMA in flight on the caller's arrays.
static bool inject_fault_at_chunk(size_t k)
{
    static const long at = [] { const char* e = std::getenv("B200VA_TEST_FAIL_CHUNK"); return e ? std::atol(e) : -1L; }();
    static std::atomic<bool> fired{false};
    return at >= 0 && static_cast<long>(k) == at && !fired.exchange(true);
}

static int stage_lanes(b200va_stager* s, const float* hA, const float* hB, float* hC, size_t n, int variant)
{
    // lanes: every H2D copy queues on one stream, every add on a second, every D2H on a
    // third; slot reuse and data flow are event edges.  The H2D queue -- the bottleneck
    // direction -- never waits behind a kernel or a D2H of another chunk.
    for (cudaStream_t st : {s->lane_h2d, s->lane_k, s->lane_d2h}) CU_TRY(cudaStreamWaitEvent(st, s->ev_start, 0));
    b200va_tune_t t;
    // Full-size chunks, then a tapered tail (1/2, 1/4, ... down to ~1 Mi elements): what is left
    // after the last H2D byte has arrived is one small add and one small D2H, not a full chunk.
    const size_t taper_min = size_t{1} << 20;
    size_t off = 0;
    for (size_t k = 0; off < n; ++k) {
        const size_t left = n - off;
        size_t m = s->chunk;
        if (left <= s->chunk && s->depth > 1) {
            m = left / 2;
            m = (m + 63) & ~size_t{63};                      // chunk starts stay 256-byte aligned
            if (m < taper_min || m >= left) m = left;
        }
        if (m > left) m = left;
        const int i = static_cast<int>(k % static_cast<size_t>(s->depth));
        float* dA = s->d_buf + static_cast<size_t>(i) * 3 * s->chunk;
        float* dB = dA + s->chunk;
        float* dC = dB + s->chunk;
        if (k >= static_cast<size_t>(s->depth)) CU_TRY(cudaStreamWaitEvent(s->lane_h2d, s->ev_out[i], 0));  // slot drained
        CU_TRY(cudaMemcpyAsync(dA, hA + off, m * sizeof(float), cudaMemcpyHostToDevice, s->lane_h2d));
        CU_TRY(cudaMemcpyAsync(dB, hB + off, m * sizeof(float), cudaMemcpyHostToDevice, s->lane_h2d));
        CU_TRY(cudaEventRecord(s->ev_in[i], s->lane_h2d));
        if (inject_fault_at_chunk(k)) return B200VA_ERR_INVALID;   // test hook: fail with copies in flight
        CU_TRY(cudaStreamWaitEvent(s->lane_k, s->ev_in[i], 0));
        default_tune(variant, m, &t, B200VA_F_COLD);      // a chunk fresh off the copy engine is never in L2
        RC_TRY(launch(dA, dB, dC, m, t, s->lane_k, pdl_enabled()));
        CU_TRY(cudaEventRecord(s->ev_sum[i], s->lane_k));
        CU_TRY(cudaStreamWaitEvent(s->lane_d2h, s->ev_sum[i], 0));
        CU_TRY(cudaMemcpyAsync(hC + off, dC, m * sizeof(float), cudaMemcpyDeviceToHost, s->lane_d2h));
        CU_TRY(cudaEventRecord(s->ev_out[i], s->lane_d2h));
        off += m;
    }
    CU_TRY(cudaEventRecord(s->slot_done[0], s->lane_d2h));   // the D2H lane finishes last
    CU_TRY(cudaStreamWaitEvent(s->main, s->slot_done[0], 0));
    return B200VA_OK;
}

static int stage_bounce(b200va_stager* s, const float* hA, const float* hB, float* hC, size_t n, int variant)
{
    // Pageable host arrays (plain malloc, what one ./vectorAdd process has): a cudaMemcpy from
    // pageable memory is staged by the driver on one thread at ~10 GB/s.  Here a pool of host
    // threads copies chunk k+1 into pinned bounce buffers and chunk k-2 out of them while the
    // copy engines and the add work on the chunks in between (lanes as in mode 2).
    const size_t bc = std::min(s->chunk, size_t{1} << 23);          // 32 MiB bounce chunks
    if (!s->pool) {
        s->pool = make_copy_pool();
        if (!s->pool) return B200VA_ERR_NOMEM;
    }
    if (!s->bounce || s->bounce_chunk != bc) {
        if (s->bounce) { cudaFreeHost(s->bounce); s->bounce = nullptr; }
        void* p = nullptr;
        RC_TRY(b200va_host_alloc(&p, static_cast<size_t>(s->depth) * 3 * bc * sizeof(float)));
        s->bounce = static_cast<float*>(p);
        s->bounce_chunk = bc;
    }
    for (cudaStream_t st : {s->lane_h2d, s->lane_k, s->lane_d2h}) CU_TRY(cudaStreamWaitEvent(st, s->ev_start, 0));
    const size_t nchunks = (n + bc - 1) / bc;
    const size_t depth = static_cast<size_t>(s->depth);
    b200va_tune_t t;
    auto span = [&](size_t k, size_t* off, size_t* m) { *off = k * bc; *m = std::min(bc, n - *off); };
    for (size_t k = 0; k < nchunks + depth - 1 || k < nchunks; ++k) {
        if (k < nchunks) {
            size_t off, m;
            span(k, &off, &m);
            const size_t i = k % depth;
            float* pA = s->bounce + i * 3 * bc;
            float* dA = s->d_buf + i * 3 * s->chunk;
            // slot i was drained (copied out) at iteration k-1 below, or never used
            s->pool->copy(pA, hA + off, m * sizeof(float));
            s->pool->copy(pA + bc, hB + off, m * sizeof(float));
            CU_TRY(cudaMemcpyAsync(dA, pA, m * sizeof(float), cudaMemcpyHostToDevice, s->lane_h2d));
            CU_TRY(cudaMemcpyAsync(dA + s->chunk, pA + bc, m * sizeof(float), cudaMemcpyHostToDevice, s->lane_h2d));
            CU_TRY(cudaEventRecord(s->ev_in[i], s->lane_h2d));
            CU_TRY(cudaStreamWaitEvent(s->lane_k, s->ev_in[i], 0));
            default_tune(variant, m, &t, B200VA_F_COLD);
            RC_TRY(launch(dA, dA + s->chunk, dA + 2 * s->chunk, m, t, s->lane_k, pdl_enabled()));
            CU_TRY(cudaEventRecord(s->ev_sum[i], s->lane_k));
            CU_TRY(cudaStreamWaitEvent(s->lane_d2h, s->ev_sum[i], 0));
            CU_TRY(cudaMemcpyAsync(pA + 2 * bc, dA + 2 * s->chunk, m * sizeof(float), cudaMemcpyDeviceToHost, s->lane_d2h));
            CU_TRY(cudaEventRecord(s->ev_out[i], s->lane_d2h));
        }
        if (k + 1 >= depth) {                                       // retire chunk j = k - (depth - 1)
            const size_t j = k + 1 - depth;
            if (j < nchunks) {
                size_t off, m;
                span(j, &off, &m);
                const size_t i = j % depth;
                CU_TRY(cudaEventSynchronize(s->ev_out[i]));
                s->pool->copy(hC + off, s->bounce + i * 3 * bc + 2 * bc, m * sizeof(float));
            }
        }
    }
    CU_TRY(cudaEventRecord(s->slot_done[0], s->lane_d2h));
    CU_TRY(cudaStreamWaitEvent(s->main, s->slot_done[0], 0));
    return B200VA_OK;
}

static bool host_is_pinned(const void* p)
{
    cudaPointerAttributes at{};
    const bool ok = cudaPointerGetAttributes(&at, p) == cudaSuccess && at.type != cudaMemoryTypeUnregistered;
    if (!ok) cudaGetLastError();
    return ok;
}

// Page-locks [p, p+bytes) in place unless the runtime already knows it (cudaHostAlloc'd,
// registered by the caller, or by this stager earlier).  Returns false if the range cannot be
// registered -- the caller then falls back to the bounce path.
static bool ensure_registered(b200va_stager* s, const void* p, size_t bytes)
{
    if (bytes == 0) return true;
    const uintptr_t lo = reinterpret_cast<uintptr_t>(p), hi = lo + bytes;
    for (const HostRange& r : *s->regs)
        if (r.lo <= lo && hi <= r.hi) return true;                  // cached
    if (host_is_pinned(p) && host_is_pinned(reinterpret_cast<const void*>(hi - 1))) return true;
    // a cached range that overlaps without containing the new one (the caller's buffer moved or grew): drop it
    for (size_t i = 0; i < s->regs->size();) {
        const HostRange r = (*s->regs)[i];
        if (r.lo < hi && lo < r.hi) {
            if (cudaHostUnregister(reinterpret_cast<void*>(r.lo)) != cudaSuccess) cudaGetLastError();
            s->regs->erase(s->regs->begin() + static_cast<long>(i));
        } else {
            ++i;
        }
    }
    const cudaError_t e = cudaHostRegister(const_cast<void*>(p), bytes, cudaHostRegisterPortable);
    if (e != cudaSuccess) { cudaGetLastError(); return false; }
    try {
        s->regs->push_back(HostRange{lo, hi});
    } catch (...) {
        cudaHostUnregister(const_cast<void*>(p));
        return false;
    }
    return true;
}

static void stager_drain(b200va_stager* s)
{
    // after a failure in the middle of a pipeline: nothing may still be reading or writing the
    // caller's arrays (or the bounce ring) when the error code is returned
    for (int i = 0; i < s->depth; ++i)
        if (s->slot && s->slot[i]) cudaStreamSynchronize(s->slot[i]);
    for (cudaStream_t st : {s->lane_h2d, s->lane_k, s->lane_d2h, s->main})
        if (st) cudaStreamSynchronize(st);
    cudaGetLastError();
}

int b200va_stager_add_f32(b200va_stager_t* s, const float* hA, const float* hB, float* hC, size_t n,
                          int variant, int mode)
{
    if (!s || (n && (!hA || !hB || !hC))) return B200VA_ERR_INVALID;
    RC_TRY(check_variant(variant));
    if (mode < B200VA_STAGE_AUTO || mode > B200VA_STAGE_REGISTER) return B200VA_ERR_INVALID;
    DeviceGuard guard(s->device);
    CU_TRY(guard.err);
    const size_t bytes = n * sizeof(float);
    if (mode == B200VA_STAGE_AUTO) {
        const bool pinned = n == 0 || (host_is_pinned(hA) && host_is_pinned(hB) && host_is_pinned(hC));
        mode = pinned ? B200VA_STAGE_LANES : (3 * bytes >= (size_t{8} << 20) ? B200VA_STAGE_REGISTER : B200VA_STAGE_BOUNCE);
    }
    if (mode == B200VA_STAGE_REGISTER) {
        // page-lock the caller's arrays once (outside the timed pipeline: it is a one-off cost of the first call)
        const bool ok = ensure_registered(s, hA, bytes) && ensure_registered(s, hB, bytes) && ensure_registered(s, hC, bytes);
        if (!ok) mode = B200VA_STAGE_BOUNCE;
    }
    s->last_mode = mode;
    CU_TRY(cudaEventRecord(s->ev_start, s->main));
    int rc = B200VA_OK;
    switch (mode) {
        case B200VA_STAGE_ZEROCOPY: rc = stage_zero_copy(s, hA, hB, hC, n, variant); break;
        case B200VA_STAGE_SLOTS:    rc = stage_slots(s, hA, hB, hC, n, variant); break;
        case B200VA_STAGE_LANES:
        case B200VA_STAGE_REGISTER: rc = stage_lanes(s, hA, hB, hC, n, variant); break;
        case B200VA_STAGE_BOUNCE:   rc = stage_bounce(s, hA, hB, hC, n, variant); break;
    }
    if (rc == B200VA_OK) rc = cuda_err(cudaEventRecord(s->ev_stop, s->main));
    if (rc == B200VA_OK) rc = cuda_err(cudaStreamSynchronize(s->main));
    if (rc != B200VA_OK) { stager_drain(s); return rc; }
    CU_TRY(cudaEventElapsedTime(&s->last_ms, s->ev_start, s->ev_stop));
    return B200VA_OK;
}

int b200va_stager_last_ms(b200va_stager_t* s, float* ms)
{
    if (!s || !ms) return B200VA_ERR_INVALID;
    *ms = s->last_ms;
    return B200VA_OK;
}

int b200va_stager_last_mode(b200va_stager_t* s, int* mode)
{
    if (!s || !mode) return B200VA_ERR_INVALID;
    *mode = s->last_mode;
    return B200VA_OK;
}

int b200va_add_f32_host(const float* hA, const float* hB, float* hC, size_t n, int device, int variant)
{
    b200va_stager_t* s = nullptr;
    size_t chunk = size_t{1} << 25;
    if (n < chunk) chunk = n ? n : 1;
    RC_TRY(dev_info(device, nullptr));
    DeviceGuard guard(device);          // cudaPointerGetAttributes below needs a current device; restored on return
    CU_TRY(guard.err);
    // pinned/registered arrays go straight to the copy engines; pageable ones through the bounce pool
    // (one-shot: page-locking 3 arrays for a single pass costs more than bouncing them)
    const bool pageable = n && !(host_is_pinned(hA) && host_is_pinned(hB) && host_is_pinned(hC));
    // pinning the bounce ring costs ~0.35 ms/MiB, so keep it small (9 x 8 MiB)
    if (pageable && chunk > (size_t{1} << 21)) chunk = size_t{1} << 21;
    RC_TRY(b200va_stager_create(&s, device, chunk, n > chunk ? 3 : 1));
    const int rc = b200va_stager_add_f32(s, hA, hB, hC, n, variant, pageable ? B200VA_STAGE_BOUNCE : B200VA_STAGE_LANES);
    b200va_stager_destroy(s);
    return rc;
}

}  // extern "C"
