// b200va_add.cu -- the f32 add of libb200va.so: the tune defaults, the kernel pick, the one launch
// plan, the ticket ring, the in-process launch loop, the a2/a6 support kernels and the ceiling
// probes.  The only unit that includes b200va_kernels.cuh.
#include <map>
#include <utility>

#include "b200va_internal.h"
#include "b200va_kernels.cuh"

using namespace b200va;

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
void b200va::default_tune(int variant, size_t n, b200va_tune_t* t, unsigned flags)
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
            t->threads = hbm_class(n, sizeof(float)) ? 512 : 128;   // consumer threads (+32 producer)
            t->ctas_per_sm = 1;
            t->ld_hint = LD_PLAIN;
            t->st_hint = ST_NA;
            t->stages = hbm_class(n, sizeof(float)) ? 8 : 3;
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
    if (hbm_class(n, sizeof(float))) {
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
int b200va::check_variant(int variant, unsigned flags)
{
    if (variant < B200VA_K_AUTO || variant > B200VA_K3_VEC256) return B200VA_ERR_VARIANT;
    return (flags & ~(B200VA_F_INPUTS_STABLE | B200VA_F_COLD)) ? B200VA_ERR_INVALID : B200VA_OK;
}

namespace {

// ----------------------------------------------------------------------- kernel pick
// What each library carries.  libb200va.so carries the production set: what AUTO and the named variants
// resolve to, plus close neighbours the parity tests run.  -DB200VA_TUNE_MATRIX (libb200va_tune.so, the A/B
// tool's library) carries every combination of b200va_tune_t.  The pick below instantiates exactly the
// kernels these predicates admit; any other combination gives nullptr, and so B200VA_ERR_VARIANT.
template <int VW, int UNROLL, int LD, int ST, int EARLY, int SCHED>
constexpr bool carries_vec()
{
#ifdef B200VA_TUNE_MATRIX
    return true;
#else
    if (SCHED == 1) return VW == 4 && LD == LD_PLAIN && ST == ST_NA && (UNROLL == 2 || UNROLL == 4);
    return UNROLL <= 4 && (LD == LD_PLAIN || LD == LD_NA_EF) && (ST == ST_PLAIN || ST == ST_NA);
#endif
}

// The static-split ring (store modes 0 and 1) is no production default: the production library keeps the
// bulk-store (UBLKCP.G.S) form and one register-store form.  A bulk store takes no store hint, so store
// mode 1 has its ST_PLAIN form only.
template <int MODE, bool HINT, int ST>
constexpr bool carries_tma()
{
    if (MODE == 1 && ST != ST_PLAIN) return false;
#ifdef B200VA_TUNE_MATRIX
    return true;
#else
    return !HINT && (MODE == 1 || ST == ST_NA);
#endif
}

// K2d, the TMA production form: both load hints, plain and L1::no_allocate stores.
template <bool HINT, int ST>
constexpr bool carries_tma_dyn()
{
#ifdef B200VA_TUNE_MATRIX
    return true;
#else
    return ST == ST_PLAIN || ST == ST_NA;
#endif
}

using vec_fn = void (*)(const float*, const float*, float*, size_t, size_t, size_t, size_t);
using dyn_fn = void (*)(const float*, const float*, float*, size_t, size_t, size_t, size_t, unsigned int*);

// The vec kernel a tune selects: `plain` under the hardware block scheduler, `dyn` under the
// dynamic tile scheduler (scheduler = 1); at most one is set.
struct VecFn {
    vec_fn plain = nullptr;
    dyn_fn dyn = nullptr;
    const void* key() const { return plain ? reinterpret_cast<const void*>(plain) : reinterpret_cast<const void*>(dyn); }
};

VecFn pick_vec(int vw, int unroll, int ld, int st, int early, int sched)
{
    VecFn f;
    with_value<4, 8>(vw, [&](auto VW) {
    with_value<1, 2, 4, 8>(unroll, [&](auto U) {
    with_value<LD_PLAIN, LD_NA, LD_CS, LD_NA_EF, LD_NC_NA, LD_NA_256>(ld, [&](auto LD) {
    with_value<ST_PLAIN, ST_NA, ST_CS, ST_NA_EF>(st, [&](auto ST) {
    with_value<0, 1, 2>(early, [&](auto E) {
    with_value<0, 1>(sched, [&](auto S) {
        if constexpr (carries_vec<VW, U, LD, ST, E, S>()) {
            if constexpr (S == 1) f.dyn = vadd_vec_dyn<VW, U, LD, ST, E>;
            else f.plain = vadd_vec<VW, U, LD, ST, E>;
        }
    }); }); }); }); }); });
    return f;
}

using tma_fn = void (*)(const float*, const float*, float*, size_t, size_t, size_t, uint32_t, uint32_t);
using tma_dyn_fn = void (*)(const float*, const float*, float*, size_t, size_t, size_t, uint32_t, uint32_t, unsigned int*);

tma_fn pick_tma(int store_mode, bool l2_hint, int st)
{
    tma_fn f = nullptr;
    with_value<0, 1>(store_mode, [&](auto M) {
    with_value<0, 1>(l2_hint, [&](auto H) {
    with_value<ST_PLAIN, ST_NA, ST_CS, ST_NA_EF>(M == 1 ? ST_PLAIN : st, [&](auto ST) {
        if constexpr (carries_tma<M, H != 0, ST>()) f = vadd_tma<M, H != 0, ST>;
    }); }); });
    return f;
}

// store_mode 2: the dynamic tile scheduler, register stores
tma_dyn_fn pick_tma_dyn(bool l2_hint, int st)
{
    tma_dyn_fn f = nullptr;
    with_value<0, 1>(l2_hint, [&](auto H) {
    with_value<ST_PLAIN, ST_NA, ST_CS, ST_NA_EF>(st, [&](auto ST) {
        if constexpr (carries_tma_dyn<H != 0, ST>()) f = vadd_tma_dyn<H != 0, ST>;
    }); });
    return f;
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

}  // namespace

int b200va::launch(const float* dA, const float* dB, float* dC, size_t n, const b200va_tune_t& t,
                           cudaStream_t stream, bool pdl, unsigned int* ctr)
{
    RC_TRY(check_operands(sizeof(float), dA, dB, dC, n, true));
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
static int launch_chain(const float* dA, const float* dB, float* dC, size_t n, const b200va_tune_t& t, bool after_same,
                        int count, cudaStream_t stream, bool pdl, unsigned int* ctr = nullptr)
{
    b200va_tune_t follow = t;
    follow.early_loads = 1;
    for (int i = 0; i < count; ++i)
        RC_TRY(launch(dA, dB, dC, n, i || after_same ? follow : t, stream, pdl, ctr ? ctr + 2 * i : nullptr));
    return B200VA_OK;
}

static unsigned support_grid(const b200va_devinfo_t* di, size_t n, int threads)
{
    const size_t want = (n + threads - 1) / threads, cap = static_cast<size_t>(di->sm_count) * 16;
    return static_cast<unsigned>(std::max<size_t>(std::min(want, cap), 1));
}

// ========================================= ABI (C linkage from the declarations in include/b200va.h)
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
    RC_TRY(check_operands(sizeof(float), dA, dB, dC, n, true));
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

int b200va_host_fill_ctr_f32(float* h, size_t n, uint64_t seed, uint64_t first)
{
    if (n && !h) return B200VA_ERR_INVALID;
    const uint64_t base = seed * 0x9E3779B97F4A7C15ull + first;
    for (size_t i = 0; i < n; ++i) h[i] = ctr_value(base + i);
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

// ------------------------------------------------------------------ ceiling probes
int b200va_probe_f32(int kind, const float* dA, const float* dB, float* dC, size_t n, void* stream)
{
    if (kind < B200VA_PROBE_READ2 || kind > B200VA_PROBE_COPY) return B200VA_ERR_VARIANT;
    RC_TRY(current_dev_info(nullptr));
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
