// b200va_stager.cu -- the host-buffer path of libb200va.so: the copy pool, NUMA-local pinned
// allocation, register-once and the chunk pipelines that feed the f32 add from host arrays.
// Host code only: the adds go through the same launch as b200va_add_f32 (b200va_add.cu).
#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <cctype>
#include <condition_variable>
#include <thread>
#include <vector>

#include "b200va_internal.h"

using namespace b200va;

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

namespace {    // internal linkage: std::vector<Slot>'s code stays out of the libraries' symbol tables
// One of the `depth` device slots a chunk rotates through.
struct Slot {
    float* d = nullptr;                  // A, B and C of one chunk, `chunk` floats each (in d_buf)
    cudaStream_t stream = nullptr;       // mode 0: the chunk's copies and add
    cudaEvent_t in = nullptr, sum = nullptr, out = nullptr;   // A and B arrived, C computed, C copied out
    size_t off = 0, m = 0;               // the chunk it holds: where it sits in the caller's arrays, its length
};
}  // namespace

struct b200va_stager {
    int device = 0;
    size_t chunk = 0;
    float* d_buf = nullptr;              // the slots: depth * 3 * chunk floats
    std::vector<Slot> slots;
    cudaStream_t main = nullptr;
    // modes 2, 3 and 4: one stream for the H2D copies, one for the adds, one for the D2H copies
    cudaStream_t lane_h2d = nullptr, lane_k = nullptr, lane_d2h = nullptr;
    cudaEvent_t ev_start = nullptr, ev_stop = nullptr;
    // pageable path (mode 3): pinned bounce slots (depth * 3 * bounce_chunk(s) floats) + copy threads, made on first use
    float* bounce = nullptr;
    CopyPool* pool = nullptr;
    // register-once path (mode 4): host ranges this stager page-locked
    std::vector<HostRange> regs;
    float last_ms = 0.f;
    int last_mode = -1;
};

// Mode 3's chunk length, and the length of each array of a bounce slot: 32 MiB at most.
static size_t bounce_chunk(const b200va_stager* s) { return std::min(s->chunk, size_t{1} << 23); }

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
    for (const HostRange& r : s->regs)
        if (cudaHostUnregister(reinterpret_cast<void*>(r.lo)) != cudaSuccess) cudaGetLastError();
    s->regs.clear();
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
    for (const Slot& sl : s->slots) {
        if (sl.stream) cudaStreamDestroy(sl.stream);
        for (cudaEvent_t ev : {sl.in, sl.sum, sl.out})
            if (ev) cudaEventDestroy(ev);
    }
    for (cudaStream_t st : {s->main, s->lane_h2d, s->lane_k, s->lane_d2h})
        if (st) cudaStreamDestroy(st);
    for (cudaEvent_t ev : {s->ev_start, s->ev_stop})
        if (ev) cudaEventDestroy(ev);
    if (s->d_buf) cudaFree(s->d_buf);
    if (s->bounce) cudaFreeHost(s->bounce);
    delete s->pool;
    delete s;
    return B200VA_OK;
}

// Makes everything a stager owns; on failure the caller destroys what was made.
static int stager_make(b200va_stager* s, int device, size_t chunk, int depth)
{
    s->device = device;
    s->chunk = chunk;
    try {
        s->slots.resize(static_cast<size_t>(depth));
    } catch (const std::bad_alloc&) {
        return B200VA_ERR_NOMEM;
    }
    CU_TRY(cudaMalloc(&s->d_buf, s->slots.size() * 3 * s->chunk * sizeof(float)));
    for (cudaStream_t* st : {&s->main, &s->lane_h2d, &s->lane_k, &s->lane_d2h})
        CU_TRY(cudaStreamCreateWithFlags(st, cudaStreamNonBlocking));
    CU_TRY(cudaEventCreate(&s->ev_start));
    CU_TRY(cudaEventCreate(&s->ev_stop));
    for (size_t i = 0; i < s->slots.size(); ++i) {
        Slot& sl = s->slots[i];
        sl.d = s->d_buf + i * 3 * s->chunk;
        CU_TRY(cudaStreamCreateWithFlags(&sl.stream, cudaStreamNonBlocking));
        for (cudaEvent_t* ev : {&sl.in, &sl.sum, &sl.out})
            CU_TRY(cudaEventCreateWithFlags(ev, cudaEventDisableTiming));
    }
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
    const int rc = s ? stager_make(s, device, chunk_elems, depth) : B200VA_ERR_NOMEM;
    if (rc != B200VA_OK) { b200va_stager_destroy(s); return rc; }
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

// Fault injection for the error-path test (tests/test_gpu_host_path.py): with
// B200VA_TEST_FAIL_CHUNK=k in the environment the chunk loop fails ONCE per process, right
// after it has queued chunk k's H2D copies -- i.e. with DMA in flight on the caller's arrays.
static bool inject_fault_at_chunk(size_t k)
{
    static const long at = [] { const char* e = std::getenv("B200VA_TEST_FAIL_CHUNK"); return e ? std::atol(e) : -1L; }();
    static std::atomic<bool> fired{false};
    return at >= 0 && static_cast<long>(k) == at && !fired.exchange(true);
}

// The length of the next chunk when `left` elements are still to be staged.
static size_t chunk_len(const b200va_stager* s, int mode, size_t left)
{
    if (mode == B200VA_STAGE_BOUNCE) return std::min(bounce_chunk(s), left);
    if (mode == B200VA_STAGE_SLOTS || left > s->chunk || s->slots.size() == 1) return std::min(s->chunk, left);
    // Modes 2 and 4: full-size chunks, then a tapered tail (1/2, 1/4, ... down to ~1 Mi elements): what is left
    // after the last H2D byte has arrived is one small add and one small D2H, not a full chunk.
    const size_t m = (left / 2 + 63) & ~size_t{63};          // chunk starts stay 256-byte aligned
    return m < (size_t{1} << 20) || m >= left ? left : m;
}

// Modes 0, 2, 3 and 4: the vector in chunks that rotate through the slots; each chunk is two H2D copies, the add
// and a D2H copy.  Mode 0 queues a chunk's work on its slot's stream.  The other modes queue every H2D copy on one
// lane, every add on a second and every D2H copy on a third, with data flow and slot reuse as event edges, so the
// H2D lane -- the bottleneck direction -- never waits behind another chunk's add or D2H.
// Mode 3 takes pageable arrays (plain malloc, what one ./vectorAdd process has), which the driver would stage on
// one thread at ~10 GB/s: a pool of host threads copies each chunk into a pinned bounce slot before its H2D, and
// out of it depth - 1 chunks later, while the copy engines and the add work on the chunks in between.
static int stage_chunks(b200va_stager* s, const float* hA, const float* hB, float* hC, size_t n, int variant, int mode)
{
    const bool lanes = mode != B200VA_STAGE_SLOTS, bounce = mode == B200VA_STAGE_BOUNCE;
    const size_t depth = s->slots.size(), bc = bounce_chunk(s);
    if (bounce && !s->pool && !(s->pool = make_copy_pool())) return B200VA_ERR_NOMEM;
    if (bounce && !s->bounce) {
        void* p = nullptr;
        RC_TRY(b200va_host_alloc(&p, depth * 3 * bc * sizeof(float)));
        s->bounce = static_cast<float*>(p);
    }
    // mode 3: chunk j's result leaves its bounce slot for the caller's C once its D2H has landed
    auto retire = [&](size_t j) -> int {
        const Slot& sl = s->slots[j % depth];
        CU_TRY(cudaEventSynchronize(sl.out));
        s->pool->copy(hC + sl.off, s->bounce + (j % depth) * 3 * bc + 2 * bc, sl.m * sizeof(float));
        return B200VA_OK;
    };
    b200va_tune_t t;
    size_t k = 0;
    for (size_t off = 0; off < n; ++k) {
        const size_t i = k % depth, m = chunk_len(s, mode, n - off);
        Slot& sl = s->slots[i];
        cudaStream_t h2d = lanes ? s->lane_h2d : sl.stream, add = lanes ? s->lane_k : sl.stream,
                     d2h = lanes ? s->lane_d2h : sl.stream;
        // A slot's first chunk in this call follows the call's start, a later one the previous chunk's D2H out of
        // the slot (in mode 0 that is stream order; in mode 3 the host has already waited for it, in retire).
        CU_TRY(cudaStreamWaitEvent(h2d, k < depth ? s->ev_start : sl.out, 0));
        sl.off = off;
        sl.m = m;
        const float *srcA = hA + off, *srcB = hB + off;
        float* dstC = hC + off;
        if (bounce) {                                        // the bounce slot was retired at iteration k-1, or never used
            float* p = s->bounce + i * 3 * bc;
            s->pool->copy(p, srcA, m * sizeof(float));
            s->pool->copy(p + bc, srcB, m * sizeof(float));
            srcA = p;
            srcB = p + bc;
            dstC = p + 2 * bc;
        }
        float *dA = sl.d, *dB = dA + s->chunk, *dC = dB + s->chunk;
        CU_TRY(cudaMemcpyAsync(dA, srcA, m * sizeof(float), cudaMemcpyHostToDevice, h2d));
        CU_TRY(cudaMemcpyAsync(dB, srcB, m * sizeof(float), cudaMemcpyHostToDevice, h2d));
        CU_TRY(cudaEventRecord(sl.in, h2d));
        if (inject_fault_at_chunk(k)) return B200VA_ERR_INVALID;   // test hook: fail with copies in flight
        CU_TRY(cudaStreamWaitEvent(add, sl.in, 0));
        default_tune(variant, m, &t, B200VA_F_COLD);      // a chunk fresh off the copy engine is never in L2
        RC_TRY(launch(dA, dB, dC, m, t, add, pdl_enabled()));
        CU_TRY(cudaEventRecord(sl.sum, add));
        CU_TRY(cudaStreamWaitEvent(d2h, sl.sum, 0));
        CU_TRY(cudaMemcpyAsync(dstC, dC, m * sizeof(float), cudaMemcpyDeviceToHost, d2h));
        CU_TRY(cudaEventRecord(sl.out, d2h));
        if (bounce && k + 1 >= depth) RC_TRY(retire(k + 1 - depth));
        off += m;
    }
    if (bounce)                                              // the last depth - 1 chunks are still in the ring
        for (size_t j = k + 1 > depth ? k + 1 - depth : 0; j < k; ++j) RC_TRY(retire(j));
    // the call ends after every used slot's last D2H (on the D2H lane, the last one follows all the others)
    for (size_t i = 0; i < std::min(k, depth); ++i) CU_TRY(cudaStreamWaitEvent(s->main, s->slots[i].out, 0));
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
    for (const HostRange& r : s->regs)
        if (r.lo <= lo && hi <= r.hi) return true;                  // cached
    if (host_is_pinned(p) && host_is_pinned(reinterpret_cast<const void*>(hi - 1))) return true;
    // a cached range that overlaps without containing the new one (the caller's buffer moved or grew): drop it
    for (size_t i = 0; i < s->regs.size();) {
        const HostRange r = s->regs[i];
        if (r.lo < hi && lo < r.hi) {
            if (cudaHostUnregister(reinterpret_cast<void*>(r.lo)) != cudaSuccess) cudaGetLastError();
            s->regs.erase(s->regs.begin() + static_cast<long>(i));
        } else {
            ++i;
        }
    }
    const cudaError_t e = cudaHostRegister(const_cast<void*>(p), bytes, cudaHostRegisterPortable);
    if (e != cudaSuccess) { cudaGetLastError(); return false; }
    try {
        s->regs.push_back(HostRange{lo, hi});
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
    for (const Slot& sl : s->slots) cudaStreamSynchronize(sl.stream);
    for (cudaStream_t st : {s->lane_h2d, s->lane_k, s->lane_d2h, s->main}) cudaStreamSynchronize(st);
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
    int rc = mode == B200VA_STAGE_ZEROCOPY ? stage_zero_copy(s, hA, hB, hC, n, variant)
                                           : stage_chunks(s, hA, hB, hC, n, variant, mode);
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
