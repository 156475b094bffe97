// b200va_ptx.cuh -- hand-written PTX primitives for the sm_90a vectorAdd kernels.
//
// Everything here is a thin wrapper over one PTX instruction so that the SASS the
// kernels produce is predictable (LDG.E.128, UBLKCP, SYNCS.*): no CCCL, no CUTLASS.
// Compiled only for -gencode arch=compute_90a,code=sm_90a.
#pragma once
#include <cstdint>

namespace b200va {

// ---------------------------------------------------------------- cache-hint enums
// Load hints (tune.ld_hint)
enum : int {
    LD_PLAIN = 0,   // ld.global
    LD_NA    = 1,   // ld.global.L1::no_allocate               (streaming: skip L1)
    LD_CS    = 2,   // ld.global.cs                             (evict-first streaming)
    LD_NA_EF = 3,   // L1::no_allocate + L2 evict_first         (createpolicy operand)
    LD_NC_NA = 4,   // ld.global.nc.L1::no_allocate             (read-only path; NOTE ptxas is then free to
                    //   sink the loads next to their use, which serialises the batch -- kept as a control)
    LD_NA_256 = 5,  // L1::no_allocate + L2::256B prefetch size (SASS LTC256B): L2 fetches 256-B granules
    LD_HINTS = 6
};
// Store hints (tune.st_hint)
enum : int {
    ST_PLAIN = 0,   // st.global
    ST_NA    = 1,   // st.global.L1::no_allocate
    ST_CS    = 2,   // st.global.cs
    ST_NA_EF = 3,   // L1::no_allocate + L2 evict_first
    ST_HINTS = 4
};

struct f32x4 { float x, y, z, w; };
struct f32x8 { float v[8]; };

__device__ __forceinline__ uint64_t l2_evict_first_policy()
{
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}

// ---------------------------------------------------------------- 128-bit global
template <int HINT>
__device__ __forceinline__ f32x4 ldg128(const float* p, uint64_t pol)
{
    f32x4 r;
    if constexpr (HINT == LD_PLAIN)
        asm volatile("ld.global.v4.f32 {%0,%1,%2,%3}, [%4];"
                     : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p) : "memory");
    else if constexpr (HINT == LD_NA)
        asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                     : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p) : "memory");
    else if constexpr (HINT == LD_NC_NA)
        asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                     : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p) : "memory");
    else if constexpr (HINT == LD_CS)
        asm volatile("ld.global.cs.v4.f32 {%0,%1,%2,%3}, [%4];"
                     : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p) : "memory");
    else if constexpr (HINT == LD_NA_256)
        asm volatile("ld.global.L1::no_allocate.L2::256B.v4.f32 {%0,%1,%2,%3}, [%4];"
                     : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p) : "memory");
    else
        asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;"
                     : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p), "l"(pol) : "memory");
    return r;
}

template <int HINT>
__device__ __forceinline__ void stg128(float* p, const f32x4& v, uint64_t pol)
{
    if constexpr (HINT == ST_PLAIN)
        asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};"
                     :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
    else if constexpr (HINT == ST_NA)
        asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};"
                     :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
    else if constexpr (HINT == ST_CS)
        asm volatile("st.global.cs.v4.f32 [%0], {%1,%2,%3,%4};"
                     :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
    else
        asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.f32 [%0], {%1,%2,%3,%4}, %5;"
                     :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol) : "memory");
}

// ---------------------------------------------------------------- 32-byte vectors
// sm_90 has no 256-bit global access: a 32-byte vector (K3) is two adjacent 128-bit accesses
// with the same hint, issued back to back, so a warp still moves 1 KiB per instruction pair.
template <int HINT>
__device__ __forceinline__ f32x8 ldg256(const float* p, uint64_t pol)
{
    const f32x4 lo = ldg128<HINT>(p, pol), hi = ldg128<HINT>(p + 4, pol);
    return f32x8{{lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w}};
}

template <int HINT>
__device__ __forceinline__ void stg256(float* p, const f32x8& r, uint64_t pol)
{
    stg128<HINT>(p, f32x4{r.v[0], r.v[1], r.v[2], r.v[3]}, pol);
    stg128<HINT>(p + 4, f32x4{r.v[4], r.v[5], r.v[6], r.v[7]}, pol);
}

// ---------------------------------------------------------------- shared memory
__device__ __forceinline__ uint32_t smem_u32(const void* p)
{
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ f32x4 lds128(uint32_t saddr)
{
    f32x4 r;
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "r"(saddr) : "memory");
    return r;
}

__device__ __forceinline__ void sts128(uint32_t saddr, const f32x4& v)
{
    asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};"
                 :: "r"(saddr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar), "r"(count) : "memory");
}

__device__ __forceinline__ void mbar_fence_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void mbar_arrive(uint32_t bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(bar) : "memory");
}

__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;"
                 :: "r"(bar), "r"(bytes) : "memory");
}

// Blocks (hardware-suspended try_wait, re-armed in a loop) until the phase with the
// given parity has completed.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" :: "r"(bar), "r"(parity) : "memory");
}

// ---------------------------------------------------------------- TMA 1-D bulk copies
// global -> shared, completion counted in bytes on an mbarrier (SASS: UBLKCP.S.G).
// dst/src 16-B aligned, bytes a multiple of 16.
template <bool L2_HINT>
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes,
                                         uint32_t bar, uint64_t pol)
{
    if constexpr (L2_HINT)
        asm volatile(
            "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint "
            "[%0], [%1], %2, [%3], %4;"
            :: "r"(dst_smem), "l"(src), "r"(bytes), "r"(bar), "l"(pol) : "memory");
    else
        asm volatile(
            "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
            :: "r"(dst_smem), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// shared -> global, tracked by the issuing thread's bulk async-group (SASS: UBLKCP.G.S).
template <bool L2_HINT>
__device__ __forceinline__ void bulk_s2g(void* dst, uint32_t src_smem, uint32_t bytes, uint64_t pol)
{
    if constexpr (L2_HINT)
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;"
                     :: "l"(dst), "r"(src_smem), "r"(bytes), "l"(pol) : "memory");
    else
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                     :: "l"(dst), "r"(src_smem), "r"(bytes) : "memory");
}

// Bulk prefetch of [src, src + bytes) into L2 (no destination, nothing to wait for).  src 16-B
// aligned, bytes a multiple of 16.  L2 is the point of coherence, so prefetching data that an
// earlier kernel is still writing is harmless.
__device__ __forceinline__ void bulk_prefetch_l2(const void* src, uint32_t bytes)
{
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" :: "l"(src), "r"(bytes) : "memory");
}

__device__ __forceinline__ void bulk_commit()
{
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}

// Wait until at most N of this thread's bulk groups still have their *source reads*
// outstanding (the shared-memory stage may then be overwritten).
template <int N>
__device__ __forceinline__ void bulk_wait_read()
{
    asm volatile("cp.async.bulk.wait_group.read %0;" :: "n"(N) : "memory");
}

// Wait until at most N bulk groups are still incomplete (writes performed).
template <int N>
__device__ __forceinline__ void bulk_wait_all()
{
    asm volatile("cp.async.bulk.wait_group %0;" :: "n"(N) : "memory");
}

// Generic-proxy shared-memory writes -> visible to the async proxy (TMA) reads.
__device__ __forceinline__ void fence_proxy_async_smem()
{
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// Programmatic dependent launch (sm_90+).  `pdl_wait` blocks until the PREVIOUS grid has completed
// and its memory operations are visible, and then lets the NEXT kernel in the stream start
// scheduling its CTAs once every CTA of this grid has done the same (or exited).  This hides
// launch latency and CTA ramp-up behind the previous launch's tail.  The release comes only after
// the wait, so when a kernel starts, every launch before the one immediately preceding it has
// completed: an early-load kernel (vadd_vec EARLY = 1) can overlap that one launch and no older
// one.  A no-op for a launch without the programmatic-stream-serialization attribute.
__device__ __forceinline__ void pdl_wait()
{
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// ---------------------------------------------------------------- dynamic tile scheduler
// Work stealing for persistent grids: every CTA starts on tile blockIdx.x, then takes tickets
// from a per-launch counter in global memory (ctr[0]); ticket t is tile gridDim.x + t.  When a
// CTA has run out of tiles it counts itself out on ctr[1]; the last CTA to do so zeroes both
// words, so the slot is clean for the next launch that is handed it.  Every access happens
// after griddepcontrol.wait, i.e. after every earlier launch on the stream has completed.
__device__ __forceinline__ uint32_t sched_next_tile(unsigned int* ctr)
{
    return gridDim.x + atomicAdd(ctr, 1u);
}

__device__ __forceinline__ void sched_retire(unsigned int* ctr)
{
    __threadfence();                                  // this CTA's last ticket precedes its count
    if (atomicAdd(ctr + 1, 1u) == gridDim.x - 1) {
        ctr[0] = 0u;
        ctr[1] = 0u;
        __threadfence();
    }
}

// Named barrier over a subset of the CTA's warps (id 1..15; 0 is __syncthreads).
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads)
{
    asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(nthreads) : "memory");
}

}  // namespace b200va
